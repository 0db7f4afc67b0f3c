"""CPU tests of anomaly diagnosis (thresholding.rank_features / diagnosis_eval): the rule the device states against
TranAD's literal hit_att / ndcg and sklearn's ndcg_score, and every host-side argument check raising ValueError before
anything is launched."""
import os
import subprocess

import numpy as np
import pytest
import torch
from sklearn.metrics import ndcg_score

from tests import diagnosis_reference as ref


def _tie_free(rng, m, out):
    a = rng.permutation(m * out).reshape(m, out).astype(np.float64) / (m * out) + rng.random((m, out)) * 1e-9
    lab = (rng.random((m, out)) < rng.uniform(0.02, 0.4, (m, 1))).astype(np.float32)
    lab[::7] = 0                                                       # rows without a labelled feature are skipped
    return a, lab


@pytest.mark.parametrize("out", [2, 5, 38])
def test_restated_rule_equals_literal_code_without_ties(out):
    rng = np.random.default_rng(out)
    a, lab = _tie_free(rng, 300, out)
    assert all(len(set(r)) == out for r in a)
    ps = [100, 150, 250, 137.5]
    want, got = ref.literal(a, lab, ps), ref.restated(a, lab, ps)
    for p in ps:
        assert got[f"Hit@{p}%"] == want[f"Hit@{p}%"]
        assert got[f"NDCG@{p}%"] == pytest.approx(want[f"NDCG@{p}%"], rel=1e-12, abs=0)
    assert got["rows"] == sum(1 for r in lab if r.any())


def test_restated_ndcg_equals_sklearn_with_ties():
    rng = np.random.default_rng(3)
    checked = 0
    for _ in range(400):
        out = int(rng.integers(2, 40))
        a = rng.integers(0, 4, out).astype(np.float64)
        a[rng.random(out) < 0.2] = -0.0                               # sklearn refuses infinite scores
        l = (rng.random(out) < 0.3).astype(np.float64)
        if not l.any():
            continue
        for p in (100, 150, 333):
            k = ref.cutoff(p, int(l.sum()), out)
            assert ref.row_ndcg(a, l, k) == pytest.approx(ndcg_score(l[None], a[None], k=k), rel=1e-12, abs=0)
            checked += 1
    assert checked > 500


def test_rank_is_stable_descending_with_signed_zeros_and_nan():
    a = np.array([0.0, np.nan, -0.0, 2.0, np.inf, 2.0, -np.inf, np.nan])
    assert ref.rank(a).tolist() == [4, 3, 5, 0, 2, 6, 1, 7]


class NoLib:
    def __getattr__(self, name):
        raise AssertionError(f"{name} launched")


@pytest.fixture
def th(monkeypatch):
    """thresholding with every library function refusing to run."""
    from mtad_gat_pytorch_b200 import thresholding
    monkeypatch.setattr(thresholding, "lib", NoLib())
    return thresholding


def _host_cuda(monkeypatch, th):
    """Host scores taken as they come, so that the checks after the score check run here."""
    monkeypatch.setattr(th, "_diag_scores", lambda a, what: a)


SCORE_BAD = [
    (np.zeros((4, 3), np.float32), "must be a CUDA tensor"),
    (torch.zeros(4, 3, dtype=torch.float16), "float32 or float64"),
    (torch.zeros(12), r"an \(m, out\) score matrix"),
    (torch.zeros(0, 3), r"an \(m, out\) score matrix"),
    (torch.zeros(4, 1), "at least 2"),
    (torch.zeros(2, 1025), "1024 features"),
    (torch.zeros(4, 3), "must be a CUDA tensor"),
]


@pytest.mark.parametrize("a, match", SCORE_BAD)
def test_score_checks(th, a, match):
    for fn in (th.rank_features, lambda x: th.diagnosis_eval(x, np.zeros((4, 3), np.float32))):
        with pytest.raises(ValueError, match=match):
            fn(a)


OTHER_BAD = [  # (labels, ps, rows, match)
    (np.zeros((4, 3), np.float64), (100,), None, "labels must be float32, integer or bool"),
    (torch.zeros(4, 3, dtype=torch.float64), (100,), None, "labels must be float32, integer or bool"),
    (np.zeros((3, 4), np.float32), (100,), None, r"labels of shape \(3, 4\)"),
    (np.full((4, 3), 2, np.int64), (100,), None, "must be 0 or 1"),
    (np.full((4, 3), 0.5, np.float32), (100,), None, "must be 0 or 1"),
    (torch.full((4, 3), -1, dtype=torch.int32), (100,), None, "must be 0 or 1"),
    (np.zeros((4, 3), np.float32), (99.9,), None, ">= 100"),
    (np.zeros((4, 3), np.float32), (100, 50), None, ">= 100"),
    (np.zeros((4, 3), np.float32), (float("nan"),), None, ">= 100"),
    (np.zeros((4, 3), np.float32), (True,), None, ">= 100"),
    (np.zeros((4, 3), np.float32), ("100",), None, ">= 100"),
    (np.zeros((4, 3), np.float32), 100, None, "list of percentages"),
    (np.zeros((4, 3), np.float32), (), None, "1 to 16"),
    (np.zeros((4, 3), np.float32), tuple(range(100, 117)), None, "17 percentages"),
    (np.zeros((4, 3), np.float32), (100,), np.zeros(4, np.float32), "rows must be bool or integer"),
    (np.zeros((4, 3), np.float32), (100,), torch.zeros(4), "rows must be bool or integer"),
    (np.zeros((4, 3), np.float32), (100,), np.zeros(5, bool), r"rows must be \(m,\) or \(R, m\)"),
    (np.zeros((4, 3), np.float32), (100,), np.zeros((2, 3), bool), r"rows must be \(m,\) or \(R, m\)"),
    (np.zeros((4, 3), np.float32), (100,), np.zeros((2, 2, 4), bool), r"rows must be \(m,\) or \(R, m\)"),
    (np.zeros((4, 3), np.float32), (100,), np.zeros((0, 4), bool), "0 row masks"),
    (np.zeros((4, 3), np.float32), (100,), torch.zeros(65536, 4, dtype=torch.bool), "65536 row masks"),
]


@pytest.mark.parametrize("labels, ps, rows, match", OTHER_BAD)
def test_argument_checks_before_any_launch(th, monkeypatch, labels, ps, rows, match):
    import mtad_gat_pytorch_b200 as mg
    _host_cuda(monkeypatch, th)
    mg.reset_launch_count()
    with pytest.raises(ValueError, match=match):
        th.diagnosis_eval(torch.zeros(4, 3), labels, ps=ps, rows=rows)
    assert mg.launch_count() == 0


def test_host_labels_and_masks_as_the_kernel_reads_them(th):
    dev = torch.device("cpu")
    for lab in (np.eye(3, dtype=np.float32), np.eye(3, dtype=np.int64), np.eye(3, dtype=bool),
                torch.eye(3, dtype=torch.int16), torch.eye(3).bool()):
        t = th._diag_labels(lab, 3, 3, dev, "x")
        assert t.dtype == torch.uint8 and t.tolist() == np.eye(3, dtype=np.uint8).tolist()
    sel, R, two = th._diag_rows(np.array([0, 2, -1, 0]), 4, dev, "x")
    assert (sel.tolist(), R, two) == ([[0, 1, 1, 0]], 1, False)
    sel, R, two = th._diag_rows(torch.tensor([[0, 1, 2, 0], [1, 0, 0, 0]], dtype=torch.uint8), 4, dev, "x")
    assert (sel.tolist(), R, two) == ([[0, 1, 2, 0], [1, 0, 0, 0]], 2, True)   # any nonzero byte selects
    assert th._diag_rows(None, 4, dev, "x") == (None, 1, False)


def test_diagnose_kernels_are_built_for_sm_90a():
    import __graft_entry__ as ge
    ge.build()
    nvcc = os.environ.get("NVCC", "/usr/local/cuda/bin/nvcc")
    out = subprocess.run([os.path.join(os.path.dirname(nvcc), "cuobjdump"), "-sass",
                          os.path.join(ge.OBJDIR, "diagnose.o")], capture_output=True, text=True, check=True).stdout
    assert "sm_90a" in out
    for k in ("rank_kernel", "diag_rows_kernel", "diag_select_kernel", "diag_mean_kernel"):
        assert k in out, k
    import mtad_gat_pytorch_b200._lib as L
    for name in ("mtadgat_rank_features", "mtadgat_rank_features_f64", "mtadgat_diagnose", "mtadgat_diagnose_f64",
                 "mtadgat_diagnose_scratch_words"):
        assert hasattr(L.lib, name)


@pytest.mark.parametrize("p", [99.5, 0.0, float("nan"), float("inf"), -100.0])
def test_the_library_refuses_percentages_below_100(p):
    """A cutoff of 0 would index the discount sums at -1: mtadgat_diagnose refuses such P before launching."""
    import ctypes
    import mtad_gat_pytorch_b200 as mg
    from mtad_gat_pytorch_b200._lib import lib
    ps = (ctypes.c_double * 2)(150.0, p)
    mg.reset_launch_count()
    for entry in (lib.mtadgat_diagnose, lib.mtadgat_diagnose_f64):
        assert entry(8, 4, 3, 3, 8, 3, None, 1, ps, 2, 8, 8, 8, 8, None) != 0   # checked before any pointer is read
        assert "percentages must be finite and >= 100" in lib.mtadgat_last_error().decode()
    assert mg.launch_count() == 0
