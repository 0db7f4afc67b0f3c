"""The factored float64 GAT reference of tests/gat_reference.py against the materialised oracle (orc.gat_fwd /
orc.gat_bwd), and its restatement of the GAT dispatch against the table DESIGN §4 gives.  No GPU."""
import numpy as np
import pytest

from oracle import mtad_gat_oracle as orc
from tests import gat_reference as gr


def problem(B, n, k, E, feature, v2, seed, bias=True):
    rng = np.random.default_rng(seed)
    K, D, _, _, _ = gr.dims(n, k, E, feature, v2)
    x = rng.standard_normal((B, n, k))
    lin_w = rng.standard_normal((E, 2 * D if v2 else D)) / np.sqrt(D)
    lin_b = rng.standard_normal(E) * 0.1
    a = rng.standard_normal((E if v2 else 2 * E, 1)) * 0.5
    b = rng.standard_normal((K, K)) * 0.1 if bias else None
    return x, lin_w, lin_b, a, b


def rel(a, b):
    return float(np.abs(a - b).max() / max(np.abs(b).max(), 1e-300))


@pytest.mark.parametrize("layer", ["feature", "temporal"])
@pytest.mark.parametrize("v2", [True, False])
@pytest.mark.parametrize("bias,drop", [(True, True), (False, False)])
def test_factored_reference_equals_oracle(layer, v2, bias, drop):
    feature = layer == "feature"
    B, n, k, E = 3, 11, 7, 6
    x, lin_w, lin_b, a, b = problem(B, n, k, E, feature, v2, seed=n + k + 2 * v2 + feature, bias=bias)
    K = k if feature else n
    rng = np.random.default_rng(1)
    mask = (rng.uniform(size=(B, K, K)) >= 0.3) / 0.7 if drop else None
    alpha = 0.2
    out_o, cache_o = orc.gat_fwd(x, lin_w, lin_b, a, b, alpha, feature, v2, mask)
    out_f, cache_f = gr.gat_fwd(x, lin_w, lin_b, a, b, alpha, feature, v2, mask=mask, rows=4)
    assert rel(out_f, out_o) < 1e-12
    dout = rng.standard_normal(x.shape)
    ref = orc.gat_bwd(dout, cache_o)
    got = gr.gat_bwd(dout, cache_f)
    for name, g, r in zip(("dx", "dlin_w", "dlin_b", "da", "dbias"), got, ref):
        if r is None:
            assert g is None
            continue
        assert rel(np.asarray(g).reshape(-1), np.asarray(r).reshape(-1)) < 1e-12, name


@pytest.mark.parametrize("layer", ["feature", "temporal"])
@pytest.mark.parametrize("v2", [True, False])
def test_own_slopes_reproduce_oracle(layer, v2):
    """A slope array taken from the reference's own z > 0 gives bitwise the reference's own-branch results, and the
    oracle's to 1e-12; the opposite branches do not (so the array is really used)."""
    feature = layer == "feature"
    B, n, k, E = 2, 9, 5, 4
    x, lin_w, lin_b, a, b = problem(B, n, k, E, feature, v2, seed=5)
    K = k if feature else n
    P, Q = gr._proj(gr.nodes(x, feature), lin_w, lin_b, v2)
    z = gr._pre(P, Q, a.reshape(-1), v2, 0, K)
    assert 0.2 < (z > 0).mean() < 0.8
    dout = np.random.default_rng(2).standard_normal(x.shape)
    _, cache_o = orc.gat_fwd(x, lin_w, lin_b, a, b, 0.2, feature, v2)
    ref = orc.gat_bwd(dout, cache_o)
    own = gr.gat_bwd(dout, gr.gat_fwd(x, lin_w, lin_b, a, b, 0.2, feature, v2)[1])
    for slope, same in ((z > 0, True), (z <= 0, False)):
        out, cache = gr.gat_fwd(x, lin_w, lin_b, a, b, 0.2, feature, v2, slope=slope)
        got = gr.gat_bwd(dout, cache)
        assert all(np.array_equal(g, r) for g, r in zip(got, own)) == same
        errs = [rel(np.asarray(g).reshape(-1), np.asarray(r).reshape(-1)) for g, r in zip(got, ref)]
        assert (max(errs) < 1e-12) == same, errs


def test_saved_layout():
    L = gr.saved_layout(3, 100, 38, 76, False, True)
    K, D, Ew, NC, Kp = gr.dims(100, 38, 76, False, True)
    assert (K, D, Ew, NC, Kp) == (100, 38, 76, 154, 100)
    assert L["meta"] % 4 == 0 and L["pqt"] % 4 == 0 and L["meta"] >= D * NC + NC
    assert L["att"] - L["pqt"] == 3 * NC * Kp and L["total"] - L["att"] == 3 * K * Kp


# rows of DESIGN §4's GAT dispatch table: (layer, v2, n, k, E, B) -> the paths it names
TABLE = [
    (("temporal", True, 100, 38, 76, 256), dict(fwd="win<4,10>", bwd1="bwd1<4>", bwd2="bwd2_win", param="tc")),
    (("feature", True, 100, 38, 200, 256), dict(fwd="win<2,4>", bwd1="bwd1<2>", bwd2="bwd2_win", dv="T", param="tc")),
    (("temporal", True, 100, 55, 110, 256), dict(fwd="tiled<4,4>", bwd2="bwd2", param="tc")),
    (("temporal", True, 100, 25, 50, 256), dict(fwd="win<4,10>", bwd2="bwd2_win", param="simt", colsum=True)),
    (("temporal", False, 100, 38, 38, 256), dict(param="simt", colsum=True)),
    (("feature", False, 100, 38, 100, 256), dict(param="simt", colsum=True)),
    (("feature", True, 100, 5, 200, 256), dict(fwd="win<2,2>", proj="simt", dv2="simt")),
    (("feature", True, 100, 13, 200, 256), dict(fwd="win<2,2>", proj="simt", dv2="simt")),
    (("temporal", True, 512, 38, 76, 256), dict(fwd="tiled<2,4>", split=("rows", "JT<K", "DT<E"), param="tc")),
    (("feature", True, 100, 512, 200, 256), dict(fwd="tiled<4,4>", split=("rows", "JT<K", "DT<E"), param="tc")),
    (("temporal", True, 100, 512, 1024, 2), dict(bwd1="bwd1<2>", bwd1_split=("JT<K",))),
]


@pytest.mark.parametrize("case,want", TABLE, ids=[f"{c[0]}-v{2 if c[1] else 1}-n{c[2]}-k{c[3]}" for c, _ in TABLE])
def test_expected_paths_table(case, want):
    layer, v2, n, k, E, B = case
    got = gr.expected_paths(layer, v2, n, k, E, "tc", B)
    assert {key: got[key] for key in want} == want, got
    fp32 = gr.expected_paths(layer, v2, n, k, E, "fp32", B)
    assert fp32["proj"] == fp32["param"] == fp32["dv1"] == fp32["dv2"] == "simt" and fp32["colsum"]


# the window limit of DESIGN §4: (layer, v2, n, k, E, B, mode) -> kernel launches per call.  Windows on gridDim.x (the
# whole-window kernels) take one launch at any B; on gridDim.y (tiled score, bwd1) or gridDim.z (two-pass bwd2, the
# batched GEMMs) they are launched in chunks of at most 65 535
LAUNCHES = [
    # B = 65 535: one chunk everywhere
    (("temporal", True, 16, 32, 8, 65535, "tc"), dict(fwd=1, bwd1=1, bwd2=1, proj=1, dv1=1, dv2=1)),
    # B = 65 573 on the whole-window kernels: only bwd1 and the GEMMs see two chunks (65 535 + 38)
    (("temporal", True, 16, 32, 8, 65573, "tc"), dict(fwd=1, bwd1=2, bwd2=1, proj=2, dv1=2, dv2=2)),
    # K = 130 (tiled, rows split, two-pass bwd2): tiled score 2, bwd2 2 passes x 2 chunks
    (("feature", True, 4, 130, 1, 65573, "tc"), dict(fwd=2, bwd1=2, bwd2=4, proj=2, dv1=2, dv2=2)),
    # three chunks past 2 x 65 535, fp32 mode (SIMT GEMMs)
    (("feature", True, 4, 130, 1, 131071, "fp32"), dict(fwd=3, bwd1=3, bwd2=6, proj=3, dv1=3, dv2=3)),
]


@pytest.mark.parametrize("case,want", LAUNCHES, ids=[f"{c[0]}-k{c[3]}-B{c[5]}-{c[6]}" for c, _ in LAUNCHES])
def test_expected_launches_past_65535_windows(case, want):
    layer, v2, n, k, E, B, mode = case
    got = gr.expected_paths(layer, v2, n, k, E, mode, B)
    assert got["launches"] == want, got
