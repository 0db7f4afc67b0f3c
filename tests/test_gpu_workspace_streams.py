"""GPU test: the packed GEMM's per-stream workspace serves every stream torch's pool hands out, plus the default stream.
A process that builds many models (each MTAD_GAT takes a side stream from the pool, e.g. one model per live detector)
runs GEMMs on all 32 pooled streams of one priority level and on the default stream."""
import pytest
import torch

pytestmark = pytest.mark.gpu


def test_gemms_run_on_every_pooled_stream_and_the_default_stream():
    import mtad_gat_pytorch_b200 as mg
    from mtad_gat_pytorch_b200._lib import lib
    lin = mg.Forecasting_Model(64, 64, 64, 1, 0.0).cuda().eval()
    x = torch.rand(300, 64, device="cuda")
    ref = lin(x)
    streams = [torch.cuda.Stream() for _ in range(40)]              # the pool wraps: all 32 streams of the level
    assert len({s.cuda_stream for s in streams}) == 32
    outs = []
    for s in streams:
        s.wait_stream(torch.cuda.current_stream())
        with torch.cuda.stream(s):
            outs.append(lin(x))
    torch.cuda.synchronize()
    for out in outs:
        assert torch.equal(out, ref)
    lib.mtadgat_workspace_release()
