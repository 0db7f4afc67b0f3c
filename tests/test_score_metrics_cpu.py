"""CPU tests of the score metrics (thresholding.auc_eval, pak_search, pak_eval): the host definitions in
score_metrics_reference against sklearn and the reference's adjust_predicts, and every host-side argument check before
any launch."""
import warnings

import numpy as np
import pytest
import torch
from sklearn.metrics import average_precision_score, roc_auc_score

from oracle import evaluation_oracle as orc
from tests import score_metrics_reference as ref


def _inputs(rng, n, kind):
    lab = (rng.random(n) < 0.2).astype(np.int64)
    s = rng.gamma(2.0, 1.0, n).astype(np.float32)
    if kind == "rounded":                                              # heavy ties within and across classes
        s = np.round(s, 1).astype(np.float32)
    elif kind == "zeros":                                              # -0.0 and +0.0 tie
        s = np.where(rng.random(n) < 0.5, np.float32(-0.0), np.float32(0.0))
        s[rng.random(n) < 0.3] = 1.0
    return s, lab


@pytest.mark.parametrize("kind", ["random", "rounded", "zeros"])
@pytest.mark.parametrize("n", [7, 300, 5000])
def test_roc_and_ap_references_agree_with_sklearn(kind, n):
    rng = np.random.default_rng(n + len(kind))
    s, lab = _inputs(rng, n, kind)
    if lab.min() == lab.max():
        lab[0] = 1 - lab[0]
    roc, want = ref.roc_exact(s, lab), roc_auc_score(lab, s)
    assert abs(roc - want) <= 1e-12 * want
    a, want = ref.ap(s, lab), average_precision_score(lab, s)
    assert abs(a - want) <= 1e-13 * want


def test_degenerate_labels_as_sklearn():
    s = np.array([0.3, 0.1, 0.2], np.float32)
    with warnings.catch_warnings():
        warnings.simplefilter("ignore")
        assert ref.ap(s, np.zeros(3, np.int64)) == average_precision_score(np.zeros(3, np.int64), s) == 0.0
        assert ref.ap(s, np.ones(3, np.int64)) == average_precision_score(np.ones(3, np.int64), s) == 1.0
    assert np.isnan(ref.roc_exact(s, np.zeros(3))) and np.isnan(ref.roc_exact(s, np.ones(3)))


def _segment_labels(rng, n):
    lab = np.zeros(n, np.float32)
    for _ in range(int(rng.integers(0, 6))):
        s = int(rng.integers(0, n))
        lab[s:s + int(rng.integers(1, 12))] = 1
    if rng.random() < 0.5:
        lab[:int(rng.integers(1, 5))] = 1                             # a segment at index 0
    return lab


@pytest.mark.parametrize("seed", range(60))
def test_pak_at_0_is_adjust_predicts_and_at_100_pointwise(seed):
    rng = np.random.default_rng(seed)
    n = int(rng.integers(1, 80))
    lab, s = _segment_labels(rng, n), rng.random(n).astype(np.float32)
    for t in (0.2, 0.5, 0.9):
        pred = s > np.float32(t)
        c0, c100 = ref.pak_counts(pred, lab, [0, 100])
        adj = orc.adjust_predicts(s, lab, np.float32(t))
        _, _, _, TP, TN, FP, FN = orc.calc_point2point(adj, lab)
        assert c0 == (int(TP), int(TN), int(FP), int(FN))
        actual = lab > 0.1
        assert c100 == (int((pred & actual).sum()), int((~pred & ~actual).sum()), int((pred & ~actual).sum()),
                        int((~pred & actual).sum()))


def test_pak_counts_a_segment_by_its_share():
    lab = np.array([1, 1, 1, 1, 0, 0, 1, 1, 0, 1], np.float32)           # segments of 4 (at 0), 2 and 1
    pred = np.array([0, 1, 0, 0, 1, 0, 1, 0, 0, 0])                      # d = 1, 1, 0
    (c0, c25, c50), = [ref.pak_counts(pred, lab, [0, 25, 50])]
    assert c0 == (3 + 2, 2, 1, 2)                                        # index 0 unpredicted: 4 - 1
    assert c25 == (1 + 2, 2, 1, 4)                                       # 100 * 1 > 25 * 4 fails: d = 1
    assert c50 == (1 + 1, 2, 1, 5)


class NoLib:
    def __getattr__(self, name):
        raise AssertionError(f"{name} launched")


@pytest.fixture
def th(monkeypatch):
    """thresholding with every library function refusing to run, and host score tensors taken as they come."""
    from mtad_gat_pytorch_b200 import thresholding
    monkeypatch.setattr(thresholding, "lib", NoLib())
    return thresholding


def test_scores_must_be_cuda_float32(th):
    for fn in (th.auc_eval, lambda s, l: th.pak_search(s, l, 0.5)):
        with pytest.raises(ValueError, match="CUDA tensor"):
            fn(np.zeros(4, np.float32), np.zeros(4))
        with pytest.raises(ValueError, match="CUDA tensor"):
            fn(torch.zeros(4), np.zeros(4))


def _host_scores(monkeypatch, th):
    monkeypatch.setattr(th, "_scores", lambda s, what: s.reshape(-1))


AUC_BAD = [  # (scores, labels, match)
    (torch.zeros(0), np.zeros(0), "empty scores"),
    (torch.zeros(4), np.zeros(5, np.float32), "4 scores but 5 labels"),
    (torch.zeros(4), np.zeros(4, np.float64), "labels must be float32, integer or bool"),
    (torch.zeros(4), np.array([0, 1, 2, 0]), "labels must be 0 or 1"),
    (torch.zeros(4), np.array([0, 0.5, 1, 0], np.float32), "labels must be 0 or 1"),
    (torch.zeros(4), torch.tensor([0, -1, 1, 0]), "labels must be 0 or 1"),
]


@pytest.mark.parametrize("scores, labels, match", AUC_BAD)
def test_auc_argument_checks_before_any_launch(th, monkeypatch, scores, labels, match):
    _host_scores(monkeypatch, th)
    with pytest.raises(ValueError, match=match):
        th.auc_eval(scores, labels)


def test_auc_refuses_2_27_scores(th, monkeypatch):
    monkeypatch.setattr(th, "_scores", lambda s, what: s)
    big = torch.zeros(1).expand(1 << 27)                               # no storage behind the 2^27 elements
    with pytest.raises(ValueError, match="2\\^27"):
        th.auc_eval(big, np.zeros(1))


KS_BAD = [((), "0 K values"), (range(102), "102 K values"), ((0, 101), r"\[0, 100\]"), ((-1,), r"\[0, 100\]"),
          ((10, 5), "strictly increasing"), ((5, 5), "strictly increasing"), ((0.5,), "integers"), ((True,), "integers"),
          (10, "list of integers"), ("10", "list of integers")]


@pytest.mark.parametrize("ks, match", KS_BAD)
def test_pak_ks_checks_before_any_launch(th, monkeypatch, ks, match):
    _host_scores(monkeypatch, th)
    with pytest.raises(ValueError, match=match):
        th.pak_search(torch.zeros(4), np.zeros(4), 0.1, 0.9, 4, ks=ks)
    with pytest.raises(ValueError, match=match):
        th.pak_eval(np.zeros(4, bool), np.zeros(4), ks=ks)


PAK_SEARCH_BAD = [  # (scores, labels, end, step_num, match)
    (torch.zeros(0), np.zeros(0), 1.0, 4, "empty scores"),
    (torch.zeros(4), np.zeros(3, np.float32), 1.0, 4, "4 scores but 3 labels"),
    (torch.zeros(4), np.zeros(4, np.float64), 1.0, 4, "labels must be float32"),
    (torch.zeros(4), np.zeros(4), 1.0, 0, "step_num must be a positive integer"),
    (torch.zeros(4), np.zeros(4), 1.0, 2.5, "step_num must be a positive integer"),
    (torch.zeros(4), np.zeros(4), 1.0, 65535 * 8 + 1, "thresholds; at most"),
]


@pytest.mark.parametrize("scores, labels, end, step_num, match", PAK_SEARCH_BAD)
def test_pak_search_argument_checks_before_any_launch(th, monkeypatch, scores, labels, end, step_num, match):
    _host_scores(monkeypatch, th)
    with pytest.raises(ValueError, match=match):
        th.pak_search(scores, labels, 0.0, end, step_num)


PAK_EVAL_BAD = [  # (pred, labels, match)
    (np.zeros(4, np.float32), np.zeros(4), "pred must be bool or integer"),
    (np.zeros((2, 2, 4), bool), np.zeros(4), r"pred must be \(m,\) or \(R, m\)"),
    (np.zeros(0, bool), np.zeros(0), r"pred must be \(m,\) or \(R, m\) with m >= 1"),
    (np.zeros((0, 4), bool), np.zeros(4), "0 row masks"),
    (torch.zeros(65536, 4, dtype=torch.bool), np.zeros(4), "65536 row masks"),
    (np.zeros(4, bool), np.zeros(5, np.float32), "4 scores but 5 labels"),
    (np.zeros(4, bool), np.zeros(4, np.float64), "labels must be float32"),
]


@pytest.mark.parametrize("pred, labels, match", PAK_EVAL_BAD)
def test_pak_eval_argument_checks_before_any_launch(th, monkeypatch, pred, labels, match):
    monkeypatch.setattr(torch.Tensor, "to", lambda self, *a, **k: self)   # host tensors stay on the host
    with pytest.raises(ValueError, match=match):
        th.pak_eval(pred, labels)


def test_score_metric_kernels_are_built_for_sm_90a():
    import os
    import subprocess
    import __graft_entry__ as ge
    ge.build()
    cuobjdump = os.path.join(os.path.dirname(os.environ.get("NVCC", "/usr/local/cuda/bin/nvcc")), "cuobjdump")
    out = subprocess.run([cuobjdump, "-sass", os.path.join(ge.OBJDIR, "auc.o")], capture_output=True, text=True,
                         check=True).stdout
    assert "sm_90a" in out
    for k in ("split_count_kernel", "radix_hist_kernel", "radix_scatter_kernel", "auc_count_kernel", "ap_terms_kernel",
              "auc_finish_kernel"):
        assert k in out, k
    out = subprocess.run([cuobjdump, "-sass", os.path.join(ge.OBJDIR, "evaluate.o")], capture_output=True, text=True,
                         check=True).stdout
    assert "pak_count_kernel" in out and "pak_finish_kernel" in out
