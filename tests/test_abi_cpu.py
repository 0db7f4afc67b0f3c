"""CPU tests: the C-ABI library builds, loads without a GPU and exports every symbol include/mtadgat.h
declares; host-side logic (state-dict contract, shape queries, dispatch by tensor device)."""
import ctypes
import os
import re

import numpy as np
import pytest
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


@pytest.fixture(scope="module")
def mg():
    import __graft_entry__ as ge
    ge.build()
    import mtad_gat_pytorch_b200 as m
    return m


def header_functions():
    txt = open(os.path.join(ROOT, "include", "mtadgat.h")).read()
    txt = re.sub(r"/\*.*?\*/", "", txt, flags=re.S)
    return sorted(set(re.findall(r"\b(mtadgat_\w+)\s*\(", txt)))


def test_library_exports_every_declared_symbol_at_abi_3(mg):
    lib = ctypes.CDLL(mg.LIB_PATH)
    names = header_functions()
    assert len(names) >= 20
    for n in names:
        assert hasattr(lib, n), f"{n} declared in include/mtadgat.h but not exported"
    from mtad_gat_pytorch_b200 import _lib
    assert sorted(_lib.SIGNATURES) == names            # the ctypes table mirrors the header one to one
    assert lib.mtadgat_abi_version() == 3


def test_gemm_impl_is_tensor_core_or_fp32_only(mg):
    """The GEMM dispatch has two paths (1 = packed tensor-core, 0 = SIMT fp32) and the GAT forward one."""
    from mtad_gat_pytorch_b200._lib import lib
    try:
        assert lib.mtadgat_set_gemm_impl(2) != 0
        assert "set_gemm_impl" in lib.mtadgat_last_error().decode()
        assert lib.mtadgat_get_gemm_impl() == 1
        assert lib.mtadgat_set_gemm_impl(0) == 0
    finally:
        assert lib.mtadgat_set_gemm_impl(1) == 0
    assert not hasattr(ctypes.CDLL(mg.LIB_PATH), "mtadgat_set_gat_impl")


def test_host_side_queries_need_no_gpu(mg):
    from mtad_gat_pytorch_b200._lib import lib
    # scrambled-repeat span (modules.py:279): at most 2 distinct h entries per row for (n,H)=(100,150)
    assert lib.mtadgat_rep_J(100, 150) == 2
    assert lib.mtadgat_rep_J(512, 150) == 2
    assert lib.mtadgat_rep_J(10, 150) == 15
    assert lib.mtadgat_gru_saved_floats(4, 10, 8, 0) == 3 * 8 * 8
    assert lib.mtadgat_gru_saved_floats(4, 10, 8, 1) == 3 * 8 * 8 + 16 * 10 * 4 * 8   # windows padded to 16 (tiled layout)
    a = lib.mtadgat_gat_saved_floats(2, 100, 38, 76, 0, 1, 0)
    b = lib.mtadgat_gat_saved_floats(2, 100, 38, 76, 0, 1, 1)
    assert b - a == 2 * 100 * 100                      # attention (B,K,Kp) kept only when gradients are needed


def test_state_dict_contract_matches_reference_fixture(mg):
    """Keys/shapes of the drop-in module == what the reference produced (golden fixture + shipped checkpoint)."""
    m = mg.MTAD_GAT(38, 100, 38, forecast_n_layers=3, dropout=0.3)
    g = np.load(os.path.join(ROOT, "tests", "golden", "smd_1_1_replay.npz"))
    ref = {k[len("param."):]: g[k].shape for k in g.files if k.startswith("param.")}
    mine = {k: tuple(v.shape) for k, v in m.state_dict().items()}
    assert mine == ref
    m.load_state_dict({k[len("param."):]: torch.from_numpy(g[k]) for k in g.files if k.startswith("param.")}, strict=True)
    g2 = np.load(os.path.join(ROOT, "tests", "golden", "msl_smap_bias.npz"))
    for which, k in (("msl", 55), ("smap", 25)):
        mm = mg.MTAD_GAT(k, 100, 1, forecast_n_layers=3)
        for key, v in mm.state_dict().items():
            assert tuple(g2[f"{which}.shape.{key}"]) == tuple(v.shape), key


def test_constructor_signature_matches_reference_call_site(mg):
    """train.py:74-90 passes three positionals + these kwargs."""
    m = mg.MTAD_GAT(25, 100, 1, kernel_size=7, use_gatv2=True, feat_gat_embed_dim=None, time_gat_embed_dim=None,
                    gru_n_layers=1, gru_hid_dim=150, forecast_n_layers=3, forecast_hid_dim=150, recon_n_layers=1,
                    recon_hid_dim=150, dropout=0.3, alpha=0.2)
    assert sum(p.numel() for p in m.parameters()) > 0
    with pytest.raises(ValueError):
        mg.ConvLayer(5, 4)                             # even kernel sizes change the window length


def test_device_dispatch_is_by_tensor_device_only(mg):
    """Host tensors run the library's CPU backend (returning host tensors); the CUDA bridges refuse host tensors, so a
    CUDA model can never silently compute on the CPU."""
    from mtad_gat_pytorch_b200 import functional as F
    m = mg.MTAD_GAT(5, 12, 5).eval()
    with torch.no_grad():
        p, r = m(torch.rand(2, 12, 5))
    assert p.shape == (2, 5) and r.shape == (2, 12, 5) and p.device.type == "cpu"
    w, b = m.conv.conv.weight, m.conv.conv.bias
    with pytest.raises(mg.MtadGatLibraryError):
        F.ConvReluFn.apply(torch.rand(2, 12, 5), w, b)             # the CUDA bridge itself never accepts host tensors


def test_product_never_imports_oracle():
    pkg = os.path.join(ROOT, "mtad_gat_pytorch_b200")
    for dp, _, fs in os.walk(pkg):
        for f in fs:
            if f.endswith((".py", ".cu", ".cuh", ".h")):
                assert "oracle" not in open(os.path.join(dp, f)).read(), f


def test_shard_batch():
    from mtad_gat_pytorch_b200.training import shard_batch
    for gb, w in ((256, 8), (1024, 8), (10, 4), (7, 3)):
        spans = [shard_batch(gb, w, r) for r in range(w)]
        assert spans[0][0] == 0 and spans[-1][1] == gb
        assert all(a[1] == b[0] for a, b in zip(spans, spans[1:]))
