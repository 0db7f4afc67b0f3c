"""CPU tests of replays (thresholding.replay_eval, csrc/evaluate.cu's mtadgat_eval_counts_rows): a host restatement of
the batched point-adjusted counts against the oracle's adjust_predicts(pred=...) + calc_point2point, turned into the
reference's dict by thresholding's own host expressions, for random alarm rows (two-sided codes included) and float32,
int64 and bool labels with segments at index 0 and at the end; and configurations refused before anything launches."""
import numpy as np
import pytest
import torch

from oracle import evaluation_oracle as ev


def count_rows(pred, label):
    """mtadgat_eval_counts_rows restated: {TP, TN, FP, FN, latency_sum, n_detected} per row of `pred` (nonzero =
    predicted) from the label segments alone; -1s for labels other than 0 / 1."""
    lab = np.asarray(label, np.float32)
    n, a = lab.size, lab > 0.1
    if np.any((lab != 0) & (lab != 1)):
        return np.full((len(pred), 6), -1, np.int64)
    edges = np.diff(np.concatenate([[0], a.astype(np.int8), [0]]))
    segs = list(zip(np.flatnonzero(edges == 1), np.flatnonzero(edges == -1) - 1))
    P = int(a.sum())
    out = []
    for row in np.asarray(pred):
        hit = row != 0
        fp = int(np.count_nonzero(hit & ~a))
        tp = lat = nd = 0
        for s, e in segs:
            f = np.flatnonzero(hit[s:e + 1])
            if f.size:
                f = s + int(f[0])
                tp += e - s + 1 - (1 if s == 0 and f > 0 else 0)     # index 0 is never back-filled
                lat += max(f - max(s, 1), 0)
                nd += 1
        out.append([tp, n - P - fp, fp, P - tp, lat, nd])
    return np.array(out, np.int64)


def _labels(rng, n):
    lab = np.zeros(n, np.float32)
    lab[:rng.integers(1, 6)] = 1                                       # a segment at index 0
    lab[n - rng.integers(1, 6):] = 1                                   # and one at the end
    for s in rng.integers(5, n - 10, 6):
        lab[s:s + rng.integers(1, 8)] = 1
    return lab


@pytest.mark.parametrize("dtype", [np.float32, np.int64, np.bool_])
@pytest.mark.parametrize("seed", range(4))
def test_restated_counts_are_the_reference(seed, dtype):
    from mtad_gat_pytorch_b200 import thresholding as th
    rng = np.random.default_rng(seed)
    n = int(rng.integers(40, 300))
    lab = _labels(rng, n).astype(dtype)
    rows = (rng.random((12, n)) < rng.random((12, 1)) * 0.2) * rng.integers(1, 3, (12, n))   # codes 0 / 1 / 2
    rows[0] = 0
    rows[1, 0], rows[1, 1:] = 0, 0
    rows[1, 3] = 2                                                     # the index-0 segment found late
    rows[2, 0] = 1                                                     # and found at 0
    counts = count_rows(rows, lab)
    dts = th._sum_dtypes(np.dtype(dtype))
    for row, c in zip(rows, counts):
        p, latency = ev.adjust_predicts(None, lab, 0.0, pred=row != 0, calc_latency=True)
        want = ev.calc_point2point(p, lab)
        got = th._point2point(c, dts)
        for g, w in zip(got, want):
            assert g == w and type(g) is type(w)
        assert th._latency(c) == latency


def test_restated_counts_refuse_other_labels():
    assert (count_rows(np.ones((2, 3)), [0, 2, 1]) == -1).all()


BAD = [
    ([], "1 to 65535 configurations"),
    ([{"q": 0}], "q must be > 0"),
    ([{"level": 1.0}], r"level must be in \(0, 1\)"),
    ([{"level": 0}], r"level must be in \(0, 1\)"),
    ([{"level": 0.4, "bidirectional": True}], "level > 0.5"),
    ([{"depth": 4097}], "depth must be None or an integer"),
    ([{"depth": -1}], "depth must be None or an integer"),
    ([{"depth": 2.5}], "depth must be None or an integer"),
    ([{"depth": 100}], "needs more than 100"),
    ([{"level": 0.9}, {"spam": 1}], "configuration 1: a mapping"),
    ([{"level": 0.9}, 0.9], "configuration 1: a mapping"),
]


@pytest.mark.parametrize("configs,match", BAD)
def test_bad_configurations_are_refused_before_any_launch(configs, match, monkeypatch):
    """replay / replay_eval check every configuration before the first library call: scores are taken as they come
    (no device here) and every library function raises if reached."""
    from mtad_gat_pytorch_b200 import thresholding as th

    class NoLib:
        def __getattr__(self, name):
            raise AssertionError(f"{name} launched")
    monkeypatch.setattr(th, "lib", NoLib())
    monkeypatch.setattr(th, "_scores", lambda x, what: x.reshape(-1))
    tr, s = torch.zeros(100), torch.zeros(50)
    with pytest.raises(ValueError, match=match):
        th.replay(tr, s, configs)
    with pytest.raises(ValueError, match=match):
        th.replay_eval(tr, s, np.zeros(50, np.float32), configs)
    with pytest.raises(ValueError, match=match):
        th.replay_configs(configs, 100)


def test_good_configurations_normalise():
    from mtad_gat_pytorch_b200 import thresholding as th
    got = th.replay_configs([{}, {"depth": 0, "bidirectional": True, "level": 0.95}, {"depth": 99, "q": 1e-2,
                                                                                      "with_alarm": False}], 100)
    assert got == [(1e-3, 0.99, None, False, True), (1e-3, 0.95, None, True, True), (1e-2, 0.99, 99, False, False)]
