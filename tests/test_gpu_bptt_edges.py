"""The unit-split cluster BPTT (gru_cl_bwd_kernel) copies each step's saved gates, dout and out[t-1] 4 / WPT steps ahead
into a per-thread shared-memory ring (4, 2 or 1 slots at 1, 2 or 4 clusters per 16-window tile), which at H >= 72 lies
over the part of W_hh^T that the MMA warpgroup keeps in registers (H >= 65), and folds dh_last into the last step.  These cases run
the ring at its edges: with and without dout and dh_last, sequences of 1-4 steps (no longer than the ring), batches that
leave the last 16-window tile partly empty, hidden sizes whose last CTA has idle epilogue threads, odd H (out rows not
16-byte aligned), a hidden size small enough for the ring to sit after the staging buffer (H = 40), and every split.
Each result is checked per window against the fp64 oracle with test_gpu_recurrence.py's fp16 gate, and a second run
must give bitwise the same gradients."""
import numpy as np
import pytest

from tests.test_gpu_recurrence import TOL, _cu, bwd_views, k_bwd, oracle_bwd, oracle_fwd, problem, report, upstream
from tests import oracle_tools as ot

pytestmark = pytest.mark.gpu


@pytest.fixture(autouse=True)
def _cluster_unit_split():
    import mtad_gat_pytorch_b200 as mg
    mg.set_mode("tc"); mg.set_gru_impl("tc"); mg.set_gru_bptt("unitsplit"); mg.set_gru_split(0)
    yield
    mg.set_mode("tc"); mg.set_gru_split(0)


@pytest.mark.parametrize("split", [1, 2, 4])
@pytest.mark.parametrize("H,B,n", [(150, 17, 100), (97, 40, 3), (161, 15, 2), (200, 33, 1), (150, 1, 4), (40, 20, 5)])
def test_bptt_edges_vs_fp64_oracle(H, B, n, split):
    import mtad_gat_pytorch_b200 as mg
    mg.set_gru_split(split)
    gi, w_hh, b_hh, dout, dh_last = problem(H, B, n, seed=7 * H + B + n)
    cache = oracle_fwd(gi, w_hh, b_hh)
    gates = _cu(ot.tile(np.concatenate(cache[2:6], axis=2)))
    out, W = _cu(cache[1]), _cu(w_hh)
    for style in ("all", "last", "both"):
        do, dl = upstream(style, dout, dh_last)
        ref = dict(zip(("dgi", "dghn"), oracle_bwd(cache, do, dl)))
        first = bwd_views(*k_bwd(gates, out, W, _cu(do), _cu(dl), B, n, H), B)
        report(f"ring split={split} {style} H={H} B={B} n={n}", first, ref, TOL)
        again = bwd_views(*k_bwd(gates, out, W, _cu(do), _cu(dl), B, n, H), B)
        for k in first:
            assert np.array_equal(first[k], again[k]), (k, style, H, B, n, split)
