"""CPU tests of affiliation precision and recall: the O(n) integer restatement equals the Fraction definition in every
integer word on random small series (half-integer zone boundaries, units straddling a boundary, events at both ends,
one-point events, zones without predictions); the closed forms; the exactness bound; and the host-side argument
checks of thresholding.affiliation_eval / affiliation_search, which raise before anything is launched."""
from fractions import Fraction

import numpy as np
import pytest
import torch

from tests import affiliation_reference as ref


def _case(rng):
    n = int(rng.integers(1, 40))
    lab = (rng.random(n) < rng.random()).astype(np.float32)
    if rng.random() < 0.3:                                             # one-point events with odd and even gaps
        lab = np.zeros(n, np.float32)
        lab[rng.integers(0, n, size=int(rng.integers(1, 4)))] = 1
    if lab.sum() == 0:
        lab[rng.integers(0, n)] = 1
    pred = rng.random(n) < rng.random()
    return pred, lab


def test_integer_words_are_the_fraction_definition():
    rng = np.random.default_rng(2024)
    straddles = edges = 0
    for _ in range(2500):
        pred, lab = _case(rng)
        words, probs = ref.definition(pred, lab)
        got = ref.integer_words(pred, lab)
        assert all(f.denominator == 1 for w in words for f in w)
        assert np.array_equal(got, np.array([[int(f) for f in w] for w in words], np.int64).reshape(-1, 3))
        r = ref.affiliation(pred, lab)
        for j, (p, rc) in enumerate(probs):
            assert (p is None and np.isnan(r["P"][j])) or float(p) == r["P"][j]
            assert float(rc) == r["R"][j]
        S, E, LO, HI = ref.zone_bounds(lab, lab.size)
        straddles += int(np.any((HI[:-1] % 4 == 2) & pred[np.minimum(HI[:-1] // 4, lab.size - 1)]))
        edges += int(lab[0] == 1) + int(lab[-1] == 1)
    assert straddles > 100 and edges > 500                              # the cases reach what they are meant to


def test_closed_forms():
    lab = np.zeros(33, np.float32)
    lab[10:13] = 1
    r = ref.affiliation(np.ones(33, bool), lab)                       # p0 + (1 - p0)^2 / 2 with p0 = 3 / 33
    assert r["recall"] == 1.0 and r["precision"] == float(Fraction(61, 121))
    rng = np.random.default_rng(1)
    for _ in range(50):
        _, lab = _case(rng)
        r = ref.affiliation(lab != 0, lab)
        assert r["precision"] == 1.0 and r["recall"] == 1.0 and r["f1"] == 1.0
        r = ref.affiliation(np.zeros(lab.size, bool), lab)
        assert np.isnan(r["precision"]) and r["recall"] == 0.0 and np.isnan(r["f1"]) and r["predicted_zones"] == 0
    assert ref.f1(0.0, 0.0) == 0.0


def test_every_integer_stays_exact_in_a_double():
    n = (1 << 24) - 1                                                  # the longest series the entry points take
    assert 16 * n * n < 1 << 53
    lab = np.zeros(1 << 12, np.float32)
    lab[7] = 1
    w = ref.integer_words(np.ones(lab.size, bool), lab)                # the largest words: one event, all predicted
    assert w.max() <= 16 * lab.size ** 2


@pytest.fixture(scope="module")
def th():
    import __graft_entry__ as ge
    ge.build()
    from mtad_gat_pytorch_b200 import thresholding
    return thresholding


EVAL_BAD = [  # (pred, labels, match)
    (np.zeros(4, np.float32), np.ones(4), "pred must be bool or integer"),
    (np.zeros((2, 2, 4), bool), np.ones(4), r"pred must be \(n,\) or \(R, n\)"),
    (np.zeros(0, bool), np.zeros(0), r"pred must be \(n,\) or \(R, n\) with n >= 1"),
    (np.zeros((0, 4), bool), np.ones(4), "0 row masks"),
    (torch.zeros(65536, 4, dtype=torch.bool), np.ones(4), "65536 row masks"),
    (np.zeros(4, bool), np.ones(5, np.float32), "4 scores but 5 labels"),
    (np.zeros(4, bool), np.ones(4, np.float64), "labels must be float32"),
    (np.zeros(4, bool), np.array([0, 1, 2, 0], np.float32), "labels must be 0 or 1"),
    (np.zeros(4, bool), torch.tensor([0, 1, 0.5, 0]), "labels must be 0 or 1"),
    (np.zeros(4, bool), np.zeros(4, np.float32), "no anomaly"),
    (np.zeros(4, bool), torch.zeros(4, dtype=torch.int64), "no anomaly"),
]


@pytest.mark.parametrize("pred, labels, match", EVAL_BAD)
def test_affiliation_eval_argument_checks_before_any_launch(th, monkeypatch, pred, labels, match):
    monkeypatch.setattr(torch.Tensor, "to", lambda self, *a, **k: self)   # host tensors stay on the host
    with pytest.raises(ValueError, match=match):
        th.affiliation_eval(pred, labels)


def test_affiliation_length_limit_before_any_launch(th, monkeypatch):
    monkeypatch.setattr(torch.Tensor, "to", lambda self, *a, **k: self)
    big = torch.zeros(1 << 24, dtype=torch.bool)
    with pytest.raises(ValueError, match="at most 2"):
        th.affiliation_eval(big, torch.ones(1 << 24))
    monkeypatch.setattr(torch.Tensor, "is_cuda", property(lambda self: True))   # host scores pass _scores' check
    with pytest.raises(ValueError, match="at most 2"):
        th.affiliation_search(torch.zeros(1 << 24), torch.ones(1 << 24), 0.5)


SEARCH_BAD = [  # (scores, labels, end, step_num, match)
    (torch.zeros(0), np.zeros(0), 1.0, 4, "empty scores"),
    (torch.zeros(4), np.ones(3, np.float32), 1.0, 4, "4 scores but 3 labels"),
    (torch.zeros(4), np.ones(4, np.float64), 1.0, 4, "labels must be float32"),
    (torch.zeros(4), np.array([0, 1, 3, 0], np.int64), 1.0, 4, "labels must be 0 or 1"),
    (torch.zeros(4), np.zeros(4, bool), 1.0, 4, "no anomaly"),
    (torch.zeros(4), np.ones(4), 1.0, 0, "step_num must be a positive integer"),
    (torch.zeros(4), np.ones(4), 1.0, 2.5, "step_num must be a positive integer"),
    (torch.zeros(4), np.ones(4), 1.0, 65536, "65536 thresholds; at most 65535"),
]


@pytest.mark.parametrize("scores, labels, end, step_num, match", SEARCH_BAD)
def test_affiliation_search_argument_checks_before_any_launch(th, monkeypatch, scores, labels, end, step_num, match):
    monkeypatch.setattr(torch.Tensor, "to", lambda self, *a, **k: self)
    monkeypatch.setattr(torch.Tensor, "is_cuda", property(lambda self: True))
    with pytest.raises(ValueError, match=match):
        th.affiliation_search(scores, labels, 0.0, end, step_num)


def test_affiliation_kernels_are_built_for_sm_90a(th):
    import os
    import subprocess
    import __graft_entry__ as ge
    cuobjdump = os.path.join(os.path.dirname(os.environ.get("NVCC", "/usr/local/cuda/bin/nvcc")), "cuobjdump")
    out = subprocess.run([cuobjdump, "-sass", os.path.join(ge.OBJDIR, "affiliation.o")], capture_output=True, text=True,
                         check=True).stdout
    assert "sm_90a" in out
    for k in ("aff_zone_index_kernel", "aff_ends_kernel", "aff_carry_kernel", "aff_accum_kernel", "aff_zone_kernel",
              "aff_mean_kernel"):
        assert k in out, k
    assert th.lib.mtadgat_affiliation_rows(None, 4, 1, 4, None, 1, None, None, None, None, None) != 0
    assert th.lib.mtadgat_affiliation_rows(1, 1 << 24, 1, 1 << 24, 1, 1, 1, 1, 1, 1, None) != 0
    assert "2^24" in th.lib.mtadgat_last_error().decode()
