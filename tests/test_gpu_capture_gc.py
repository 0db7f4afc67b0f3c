"""The scorers' CUDA-graph captures (scoring.SeriesScorer, scoring.MultiStreamScorer through a FleetDetector) run with
the garbage collector held off: a collection inside a capture would run finalizers of unreachable CUDA objects while
the stream captures.  The collector is enabled again afterwards, and a caller's disabled collector stays disabled."""
import gc

import numpy as np
import pytest
import torch

pytestmark = pytest.mark.gpu


def _rows(rng, n, k=5):
    return torch.from_numpy(rng.random((n, k)).astype(np.float32))


def test_captures_hold_off_the_garbage_collector(monkeypatch):
    import mtad_gat_pytorch_b200 as mg
    from mtad_gat_pytorch_b200 import prediction, scoring
    seen = []
    begin = torch.cuda.CUDAGraph.capture_begin

    def recording(self, *args, **kw):
        seen.append(gc.isenabled())
        return begin(self, *args, **kw)
    monkeypatch.setattr(torch.cuda.CUDAGraph, "capture_begin", recording)
    torch.manual_seed(0)
    model = mg.MTAD_GAT(5, 20, 5, kernel_size=3, gru_hid_dim=16, forecast_hid_dim=12, recon_hid_dim=10).cuda().eval()
    rng = np.random.default_rng(0)
    assert gc.isenabled()
    scoring.SeriesScorer(model, batch=64).score(_rows(rng, 200))
    n_series = len(seen)
    fleet = prediction.FleetDetector(model, [_rows(rng, 300), _rows(rng, 320)], q=1e-3, level=0.9)
    fleet.push(_rows(rng, 6), np.array([0, 1, 0, 1, 1, 0]))
    assert n_series >= 1 and len(seen) > n_series + 1                  # series graphs, then a fleet push graph
    assert not any(seen)
    assert gc.isenabled()
    gc.disable()
    try:
        scoring.SeriesScorer(model, batch=32).score(_rows(rng, 100))
        assert not gc.isenabled()
    finally:
        gc.enable()
