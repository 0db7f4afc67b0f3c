"""GPU tests of thresholding.auc_eval, pak_search and pak_eval against the host definitions of
score_metrics_reference: the exact ROC (Fraction) and the restated AP bit for bit at small, SMD, MSL and SMAP lengths
with ties and signed zeros; PA%K counts bit for bit against the literal per-segment loop, K = 0 against bf_search and
replay_eval; run-to-run equality and one device-to-host copy per call."""
import ctypes

import numpy as np
import pytest
import torch

from tests import score_metrics_reference as ref

pytestmark = pytest.mark.gpu

LENGTHS = [1, 50, 2049, 28479, 73729, 427617]                           # SMD, MSL and SMAP test lengths


def _segment_labels(rng, n, cover=0.1):
    lab = np.zeros(n, np.float32)
    while lab.sum() < cover * n:
        s = int(rng.integers(0, n))
        lab[s:s + int(rng.integers(1, max(2, n // 50)))] = 1
    return lab


def _scores(rng, n, kind):
    s = rng.gamma(2.0, 1.0, n).astype(np.float32)
    if kind == "rounded":
        s = np.round(s, 1).astype(np.float32)
    elif kind == "zeros":
        s = np.round(s, 0).astype(np.float32) - 2                       # many -0.0 and +0.0 after the sign flips
        s = np.where(rng.random(n) < 0.5, -s, s).astype(np.float32)
    return s


def _same(a, b):
    return (np.isnan(a) and np.isnan(b)) or np.float64(a).tobytes() == np.float64(b).tobytes()


@pytest.mark.parametrize("kind", ["random", "rounded", "zeros"])
@pytest.mark.parametrize("n", LENGTHS)
def test_auc_is_the_exact_roc_and_the_restated_ap(n, kind):
    from mtad_gat_pytorch_b200 import thresholding as th
    rng = np.random.default_rng(n + 7 * len(kind))
    s = _scores(rng, n, kind)
    lab = _segment_labels(rng, n) if n > 1 else np.ones(1, np.float32)
    got = th.auc_eval(torch.from_numpy(s).cuda(), lab)
    assert got["positives"] == int(lab.sum()) and got["negatives"] == n - int(lab.sum())
    assert _same(got["roc_auc"], ref.roc_exact(s, lab)), (got, ref.roc_exact(s, lab))
    assert _same(got["average_precision"], ref.ap(s, lab)), (got, ref.ap(s, lab))


def test_auc_label_dtypes_strided_views_and_one_class():
    from mtad_gat_pytorch_b200 import thresholding as th
    rng = np.random.default_rng(3)
    big = torch.from_numpy(_scores(rng, 20000, "rounded")).cuda()
    view = big[::2]
    s = view.cpu().numpy()
    lab = _segment_labels(rng, s.size)
    want = (ref.roc_exact(s, lab), ref.ap(s, lab))
    for l in (lab, lab.astype(np.int64), lab.astype(bool), torch.from_numpy(lab).cuda(),
              torch.from_numpy(lab.astype(np.uint8)).cuda()):
        got = th.auc_eval(view, l)
        assert _same(got["roc_auc"], want[0]) and _same(got["average_precision"], want[1])
    neg = th.auc_eval(view, np.zeros(s.size, np.float32))
    assert np.isnan(neg["roc_auc"]) and neg["average_precision"] == 0.0 and neg["positives"] == 0
    pos = th.auc_eval(view, np.ones(s.size, np.float32))
    assert np.isnan(pos["roc_auc"]) and pos["average_precision"] == 1.0 and pos["negatives"] == 0


def test_auc_refuses_non_finite_scores_and_bad_cuda_labels():
    from mtad_gat_pytorch_b200 import thresholding as th
    lab = np.array([0, 1, 0, 1, 1], np.float32)
    for bad in (np.nan, np.inf, -np.inf):
        s = torch.tensor([0.1, 0.2, bad, 0.3, 0.0]).cuda()
        with pytest.raises(ValueError, match="NaN or infinity"):
            th.auc_eval(s, lab)
    s = torch.tensor([0.1, 0.2, 0.5, 0.3, 0.0]).cuda()
    for bad in (torch.tensor([0, 1, 2, 1, 0]).cuda(), torch.tensor([0, 1, 0.5, 1, 0]).cuda()):
        with pytest.raises(ValueError, match="0 or 1"):
            th.auc_eval(s, bad)


def _device_pak_counts(th, s, lab, thresholds, ks):
    """mtadgat_eval_pak_counts' full (K, T, 4) counts."""
    n, T, K = s.numel(), len(thresholds), len(ks)
    labd, _ = th._labels(lab, n, s.device, "test")
    segs = th._segments(s, None, labd)
    thr = torch.tensor([th._compare_value(t) for t in thresholds], dtype=torch.float64).cuda()
    counts = torch.empty((K, T, 4), dtype=torch.int64, device=s.device)
    scratch = torch.empty(max(int(th.lib.mtadgat_eval_pak_scratch_words(n, T, K)), 1), dtype=torch.int64,
                          device=s.device)
    th.check(th.lib.mtadgat_eval_pak_counts(s.data_ptr(), n, segs.data_ptr(), thr.data_ptr(), T,
                                            (ctypes.c_int * K)(*ks), K, counts.data_ptr(), scratch.data_ptr(),
                                            th._stream()))
    return counts.cpu().numpy()


GRIDS = [(0.0, 1.0, 7, [0, 10, 50, 100]), (0.5, 3.0, 20, list(range(0, 101, 10))), (1.0, None, 1, [0]),
         (0.0, 6.0, 33, [0, 1, 33, 99, 100]), (-1.0, 8.0, 100, list(range(101)))]


@pytest.mark.parametrize("n", [1, 5, 300, 28479])
@pytest.mark.parametrize("grid", range(len(GRIDS)))
def test_pak_search_counts_are_the_literal_loop(n, grid):
    from mtad_gat_pytorch_b200 import thresholding as th
    start, end, steps, ks = GRIDS[grid]
    rng = np.random.default_rng(n + grid)
    s = _scores(rng, n, "rounded")
    lab = _segment_labels(rng, n, 0.2)
    if n >= 5:
        lab[:3], lab[-2:], lab[n // 2] = 1, 1, 1                        # segments at index 0, at the end, of length 1
        lab[n // 2 - 1], lab[n // 2 + 1] = 0, 0
    sd = torch.from_numpy(s).cuda()
    thresholds = th._bf_thresholds(start, end, steps)
    want = ref.pak_score_counts(s, lab, thresholds, ks)
    assert np.array_equal(_device_pak_counts(th, sd, lab, thresholds, ks), want)
    got = th.pak_search(sd, lab, start, end, steps, ks=ks)
    dts = th._sum_dtypes(np.dtype(np.float32))
    for k, d in enumerate(got["per_k"]):
        best = max(range(len(thresholds)), key=lambda t: (th._point2point(want[k, t], dts)[0], -t))
        assert d["threshold"] == thresholds[best]
        assert [d[key] for key in ("TP", "TN", "FP", "FN")] == list(want[k, best])
    bf = th.bf_search(sd, lab, start, end, steps)
    if ks[0] == 0:
        d0 = got["per_k"][0]
        assert set(d0) == set(bf) - {"latency"}
        for key, v in d0.items():
            assert v == bf[key] and type(v) is type(bf[key]), key
    f1 = np.array([d["f1"] for d in got["per_k"]], np.float64)
    assert got["f1_auc"] == float(np.trapezoid(f1, np.array(ks, np.float64) / 100)) and got["ks"] == ks


def test_pak_eval_on_replay_alarms_and_replay_eval_at_0():
    from mtad_gat_pytorch_b200 import thresholding as th
    from scripts.replay_speed import configs, series
    rng = np.random.default_rng(11)
    tr, te, lab = series(rng, 3000, 20000)
    lab[:40] = 1                                                        # a segment at index 0
    cfgs = configs(128)
    trd, ted = torch.from_numpy(tr).cuda(), torch.from_numpy(te).cuda()
    alarms = th.replay(trd, ted, cfgs)["alarms"]
    ks = list(range(0, 101, 10))
    got = th.pak_eval(alarms, lab, ks=ks)
    ev = th.replay_eval(trd, ted, lab, cfgs)
    host = alarms.cpu().numpy()
    assert len(got) == 128
    for r in range(128):
        want = ref.pak_counts(host[r], lab, ks)
        assert [tuple(int(d[k]) for k in ("TP", "TN", "FP", "FN")) for d in got[r]["per_k"]] == want, r
        for key in ("f1", "precision", "recall", "TP", "TN", "FP", "FN"):
            assert got[r]["per_k"][0][key] == ev[r][key] and type(got[r]["per_k"][0][key]) is type(ev[r][key])
    one = th.pak_eval(alarms[5], lab, ks=ks)
    assert one == got[5]
    assert th.pak_eval(host[5].astype(np.int64), lab, ks=ks) == got[5]


def test_two_runs_are_bitwise_equal():
    from mtad_gat_pytorch_b200 import thresholding as th
    rng = np.random.default_rng(5)
    s = torch.from_numpy(_scores(rng, 427617, "rounded")).cuda()
    lab = _segment_labels(rng, 427617)
    a, b = th.auc_eval(s, lab), th.auc_eval(s, lab)
    assert all(_same(a[k], b[k]) for k in a)
    assert th.pak_search(s, lab, 0.0, 5.0, 50) == th.pak_search(s, lab, 0.0, 5.0, 50)


def test_one_read_back_per_call(monkeypatch):
    import mtad_gat_pytorch_b200 as mg
    from mtad_gat_pytorch_b200 import thresholding as th
    rng = np.random.default_rng(9)
    s = torch.from_numpy(_scores(rng, 5000, "random")).cuda()
    lab = torch.from_numpy(_segment_labels(rng, 5000)).cuda()
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
    for fn, launches in ((lambda: th.auc_eval(s, lab), 19), (lambda: th.pak_search(s, lab, 0.0, 5.0, 30), 6),
                         (lambda: th.pak_eval(pred, lab), 6)):
        calls.clear()
        mg.reset_launch_count()
        fn()
        assert calls == ["cuda"]
        assert mg.launch_count() == launches
