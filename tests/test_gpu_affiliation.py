"""GPU tests of thresholding.affiliation_eval and affiliation_search against the host restatement of
affiliation_reference: per-zone integer words, P_j and R_j bit for bit, the means bit for bit against np.mean, at SMD,
MSL and SMAP lengths for one and 128 rows; rows against single-row calls, the search against the rows entry point,
strided views and label dtypes, run-to-run equality, one device-to-host copy per call and bad CUDA labels."""
import numpy as np
import pytest
import torch

from tests import affiliation_reference as ref

pytestmark = pytest.mark.gpu

LENGTHS = [1, 50, 2049, 28479, 73729, 427617]                           # SMD, MSL and SMAP test lengths


def _labels(rng, n, cover=0.1):
    lab = np.zeros(n, np.float32)
    while lab.sum() < max(cover * n, 1):
        s = int(rng.integers(0, n))
        lab[s:s + int(rng.integers(1, max(2, n // 50)))] = 1
    if n >= 8:
        lab[0], lab[-1] = 1, 1                                          # events at index 0 and at n - 1
    return lab


def _preds(rng, n, R):
    """R rows: sparse, dense and clustered alarms."""
    rows = np.zeros((R, n), bool)
    for r in range(R):
        kind = r % 3
        if kind == 0:
            rows[r] = rng.random(n) < 0.01
        elif kind == 1:
            rows[r] = rng.random(n) < 0.3
        else:
            for _ in range(max(1, n // 500)):
                s = int(rng.integers(0, n))
                rows[r, s:s + int(rng.integers(1, 40))] = True
    return rows


def _device(th, pred, lab):
    """mtadgat_affiliation_rows' words, probabilities and per-row words for a host (R, n) bool array."""
    sel = torch.from_numpy(pred.view(np.uint8)).cuda()
    labd, cap = th._aff_labels(lab, pred.shape[1], sel.device, "test")
    words, probs, host = th._aff_launch(sel, None, None, labd, cap, pred.shape[0], "test")
    return words.cpu().numpy(), probs.cpu().numpy(), host


def _same(a, b):
    return np.array_equal(np.asarray(a, np.float64).view(np.int64), np.asarray(b, np.float64).view(np.int64))


@pytest.mark.parametrize("R", [1, 128])
@pytest.mark.parametrize("n", LENGTHS)
def test_rows_are_the_integer_restatement_bit_for_bit(n, R):
    from mtad_gat_pytorch_b200 import thresholding as th
    rng = np.random.default_rng(n + R)
    lab = _labels(rng, n)
    pred = _preds(rng, n, R)
    words, probs, host = _device(th, pred, lab)
    m = int(host[0])
    rows = host[2:].reshape(R, 3)
    for r in range(R):
        want = ref.affiliation(pred[r], lab)
        assert m == want["zones"]
        assert np.array_equal(words[r, :m], want["words"]), r
        assert _same(probs[r, 0, :m], want["P"]) and _same(probs[r, 1, :m], want["R"]), r
        assert _same(rows[r, :2].view(np.float64), [want["precision"], want["recall"]]), r
        assert rows[r, 2] == want["predicted_zones"]


def test_public_dicts_rows_and_single_rows():
    from mtad_gat_pytorch_b200 import thresholding as th
    rng = np.random.default_rng(3)
    n = 28479
    lab = _labels(rng, n)
    pred = torch.from_numpy(_preds(rng, n, 16)).cuda()
    got = th.affiliation_eval(pred, lab)
    assert len(got) == 16
    for r in range(16):
        want = ref.affiliation(pred[r].cpu().numpy(), lab)
        one = th.affiliation_eval(pred[r], lab)
        for d in (got[r], one):
            assert d["zones"] == want["zones"] and d["predicted_zones"] == want["predicted_zones"]
            assert _same([d["precision"], d["recall"], d["f1"]], [want["precision"], want["recall"], want["f1"]])
            for key, w in (("individual_precision_probabilities", want["P"]),
                           ("individual_recall_probabilities", want["R"])):
                assert d[key].is_cuda and d[key].dtype == torch.float64 and _same(d[key].cpu().numpy(), w)


def test_search_is_the_rows_entry_point_on_every_threshold():
    from mtad_gat_pytorch_b200 import thresholding as th
    rng = np.random.default_rng(5)
    n = 28479
    lab = _labels(rng, n)
    s = rng.gamma(2.0, 1.0, n).astype(np.float32)
    s[lab != 0] += 1.5
    s[::997] = np.nan                                                    # NaN never predicts
    sd = torch.from_numpy(s).cuda()
    start, end, steps = 0.0, 12.0, 100
    thresholds = th._bf_thresholds(start, end, steps)
    pred = np.stack([s > np.float32(t) for t in thresholds])
    words, probs, host = _device(th, pred, lab)
    labd, cap = th._aff_labels(lab, n, sd.device, "test")
    thr = torch.tensor([th._compare_value(t) for t in thresholds], dtype=torch.float64).cuda()
    w2, p2, h2 = th._aff_launch(None, sd, thr, labd, cap, len(thresholds), "test")
    assert np.array_equal(w2.cpu().numpy(), words) and _same(p2.cpu().numpy(), probs) and np.array_equal(h2, host)
    got = th.affiliation_search(sd, lab, start, end, steps)
    rows = [ref.affiliation(p, lab) for p in pred]
    best = 0
    for t, d in enumerate(rows):
        if d["predicted_zones"] and (not rows[best]["predicted_zones"] or d["f1"] > rows[best]["f1"]):
            best = t
    assert got["threshold"] == thresholds[best] and got["f1"] == rows[best]["f1"]
    none = th.affiliation_search(sd, lab, 1e9)                           # nothing predicted: the first threshold
    assert none["predicted_zones"] == 0 and np.isnan(none["precision"]) and none["recall"] == 0.0


def test_strided_views_and_label_dtypes():
    from mtad_gat_pytorch_b200 import thresholding as th
    rng = np.random.default_rng(7)
    n = 2049
    lab = _labels(rng, n)
    big = torch.from_numpy(_preds(rng, 2 * n, 16)).cuda()
    view = big[::2, ::2]                                                 # non-contiguous rows and columns
    host = view.cpu().numpy()
    want = [ref.affiliation(host[r], lab) for r in range(8)]
    for l in (lab, lab.astype(np.int64), lab.astype(bool), torch.from_numpy(lab).cuda(),
              torch.from_numpy(lab.astype(np.uint8)).cuda()):
        for p in (view, view.to(torch.int32), host.astype(np.int8) * 3):
            got = th.affiliation_eval(p, l)
            for g, w in zip(got, want):
                assert _same([g["precision"], g["recall"]], [w["precision"], w["recall"]])
                assert _same(g["individual_recall_probabilities"].cpu().numpy(), w["R"])


def test_two_runs_are_bitwise_equal():
    from mtad_gat_pytorch_b200 import thresholding as th
    rng = np.random.default_rng(9)
    n = 427617
    lab = _labels(rng, n)
    pred = _preds(rng, n, 32)
    a, b = _device(th, pred, lab), _device(th, pred, lab)
    assert np.array_equal(a[0], b[0]) and _same(a[1], b[1]) and np.array_equal(a[2], b[2])


def test_one_read_back_per_call(monkeypatch):
    import mtad_gat_pytorch_b200 as mg
    from mtad_gat_pytorch_b200 import thresholding as th
    rng = np.random.default_rng(11)
    n = 5000
    s = torch.from_numpy(rng.gamma(2.0, 1.0, n).astype(np.float32)).cuda()
    lab = _labels(rng, n)
    pred = (s > 2.0).view(1, -1).repeat(4, 1)
    calls = []
    real_cpu = torch.Tensor.cpu

    def counting_cpu(self, *args, **kw):
        calls.append(self.device.type)
        return real_cpu(self, *args, **kw)

    def refuse(fn):
        def wrapped(self, *args, **kw):
            assert not self.is_cuda, f"{fn.__name__} on a CUDA tensor"
            return fn(self, *args, **kw)
        return wrapped
    for name in ("item", "tolist", "numpy"):
        monkeypatch.setattr(torch.Tensor, name, refuse(getattr(torch.Tensor, name)))
    monkeypatch.setattr(torch.Tensor, "cpu", counting_cpu)
    for labels in (lab, torch.from_numpy(lab).cuda()):
        for fn in (lambda: th.affiliation_eval(pred, labels), lambda: th.affiliation_search(s, labels, 0.0, 5.0, 30)):
            calls.clear()
            mg.reset_launch_count()
            fn()
            assert calls == ["cuda"]
            assert mg.launch_count() == 10                               # 4 segment-pass launches + 6


def test_bad_and_empty_cuda_labels_raise():
    from mtad_gat_pytorch_b200 import thresholding as th
    pred = torch.ones(6, dtype=torch.bool).cuda()
    s = torch.arange(6, dtype=torch.float32).cuda()
    for bad in (torch.tensor([0, 1, 2, 1, 0, 0]).cuda(), torch.tensor([0, 1, 0.5, 1, 0, 0]).cuda()):
        with pytest.raises(ValueError, match="0 or 1"):
            th.affiliation_eval(pred, bad)
        with pytest.raises(ValueError, match="0 or 1"):
            th.affiliation_search(s, bad, 1.0)
    for empty in (torch.zeros(6).cuda(), torch.zeros(6, dtype=torch.uint8).cuda()):
        with pytest.raises(ValueError, match="no anomaly"):
            th.affiliation_eval(pred, empty)
        with pytest.raises(ValueError, match="no anomaly"):
            th.affiliation_search(s, empty, 1.0, 3.0, 4)
