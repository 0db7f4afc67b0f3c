"""Point-adjusted evaluation on the device (csrc/evaluate.cu, thresholding.adjust_predicts / bf_search / epsilon_eval /
threshold_eval / feature_epsilons) against the restatement of eval_methods.py in oracle/evaluation_oracle.py.  Counts
are integers and the ratios are formed with the reference's own expressions, so everything but the epsilon itself is
compared with `==`."""
import os

import numpy as np
import pytest
import torch

from oracle import evaluation_oracle as ev
from oracle import thresholding_oracle as tho
from tests.test_oracle_golden import _score_series

pytestmark = pytest.mark.gpu
GOLD = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden")


def _case(n, pattern, seed=0):
    """Scores in [0, 1) with raised segments; `sparse`: few short segments, `dense`: most points anomalous,
    `spanning`: segments longer than a 2048-index chunk; all but `sparse` have segments at both ends."""
    rng = np.random.default_rng(seed + n)
    score = rng.random(n).astype(np.float32)
    label = np.zeros(n, np.float32)
    gap, length = {"sparse": (400, 20), "dense": (3, 12), "spanning": (1500, 5000)}[pattern]
    i = int(rng.integers(1, gap + 1)) if pattern == "sparse" else 0
    while i < n:
        ln = int(rng.integers(1, length + 1))
        label[i:i + ln] = 1
        score[i:i + ln] += np.float32(rng.random() * 0.4)
        i += ln + int(rng.integers(1, gap + 1))
    if pattern != "sparse":
        label[-min(n, 3):] = 1
    return score, label


def _thresholds(score, T, rng):
    """Python floats: exact score values, their float32 neighbours, values strictly between float32(t) and t, and
    quantiles; padded / cut to T."""
    vals = score[rng.integers(0, len(score), size=max(T // 4, 1))]
    out = []
    for v in vals:
        up, dn = np.nextafter(v, np.float32(np.inf)), np.nextafter(v, np.float32(-np.inf))
        out += [float(v), float(up), float(dn), float(v) + (float(up) - float(v)) / 3]
    out += [float(q) for q in np.quantile(score, np.linspace(0, 1, 9))] + [-1.0, 9.0]
    return [out[i % len(out)] for i in range(T)]


def _device_counts(score, label, thresholds, ge=False):
    from mtad_gat_pytorch_b200 import thresholding as th
    counts, _ = th._eval_thresholds(torch.from_numpy(score).cuda(), label, [th._compare_value(t) for t in thresholds],
                                    int(ge), "test")
    return counts


@pytest.mark.parametrize("pattern", ["sparse", "dense", "spanning"])
@pytest.mark.parametrize("n", [1, 2, 255, 256, 257, 4097, 28479, 427617])
def test_counts_equal_oracle(n, pattern):
    score, label = _case(n, pattern)
    rng = np.random.default_rng(n)
    Ts = (1, 100, 4096) if n in (4097, 28479) else (1, 100)
    for T in Ts:
        thr = _thresholds(score, T, rng)
        for ge in ((False, True) if T == 100 else (False,)):
            got = _device_counts(score, label, thr, ge)
            exp = ev.point_adjusted_counts(score, label, thr, ge=ge)
            assert np.array_equal(got, exp), (n, pattern, T, ge, np.argwhere(got != exp)[:5])
    # the literal loops on two thresholds
    for t in _thresholds(score, 2, rng):
        p, lat = ev.adjust_predicts(score, label, t, calc_latency=True)
        a = label > 0.1
        row = _device_counts(score, label, [t])[0]
        assert tuple(row[:4]) == (np.sum(p & a), np.sum(~p & ~a), np.sum(p & ~a), np.sum(~p & a))
        assert row[4] / (row[5] + 1e-4) == lat


def _same_dict(a, b):
    assert a.keys() == b.keys()
    for k in a:
        assert type(a[k]) is type(b[k]) and a[k] == b[k], (k, a[k], b[k])


@pytest.mark.parametrize("ldt", [np.float32, np.int64])
def test_bf_search_and_threshold_eval_equal_oracle(ldt):
    from mtad_gat_pytorch_b200 import thresholding as th
    for n, pattern in ((4097, "dense"), (28479, "sparse")):
        score, label = _case(n, pattern, seed=1)
        lab = label.astype(ldt)
        s = torch.from_numpy(score).cuda()
        _same_dict(th.bf_search(s, lab, start=0.01, end=2, step_num=100), ev.bf_search(score, lab, 0.01, 2, 100))
        _same_dict(th.bf_search(s, torch.from_numpy(lab).cuda(), start=0.5), ev.bf_search(score, lab, 0.5))
        for t in (0.7, np.float64(0.7), float(score[17])):
            _same_dict(th.threshold_eval(s, lab, t), ev.threshold_eval(score, lab, t))


def test_adjust_predicts_bit_exact():
    from mtad_gat_pytorch_b200 import thresholding as th
    score, label = _case(28479, "dense", seed=2)
    s = torch.from_numpy(score).cuda()
    for t in (0.3, 0.9, float(score[0])):
        p, lat = th.adjust_predicts(s, label, t, calc_latency=True)
        q, lat_ref = ev.adjust_predicts(score, label, t, calc_latency=True)
        assert p.dtype == torch.bool and np.array_equal(p.cpu().numpy(), q) and lat == lat_ref
        raw = score >= t                                                 # prediction.py: A_Pred_Global, then pred=
        q2, lat2 = ev.adjust_predicts(None, label, t, pred=raw.astype(int), calc_latency=True)
        for pred in (raw, torch.from_numpy(raw).cuda(), torch.from_numpy(raw.astype(np.int64)).cuda()):
            p2, l2 = th.adjust_predicts(None, label, t, pred=pred, calc_latency=True)
            assert np.array_equal(p2.cpu().numpy(), q2.astype(bool)) and l2 == lat2
        assert np.array_equal(th.adjust_predicts(s, label, t).cpu().numpy(), q)


@pytest.mark.parametrize("reg_level", [0, 1, 2])
def test_epsilon_eval(reg_level):
    from mtad_gat_pytorch_b200 import thresholding as th
    for seed, n in ((0, 3000), (3, 28479)):
        train = _score_series(seed, n)
        test, label = _case(n, "sparse", seed=seed)
        got = th.epsilon_eval(torch.from_numpy(train).cuda(), torch.from_numpy(test).cuda(), label, reg_level)
        ref = ev.epsilon_eval(train, test, label, reg_level)
        assert abs(got["threshold"] - ref["threshold"]) <= 2e-6 * max(1.0, abs(ref["threshold"]))
        at = ev.threshold_eval(test, label, got["threshold"])           # everything else at the device's epsilon
        at["reg_level"] = reg_level
        _same_dict(got, at)
    flat = np.full(500, 0.25, np.float32)                                 # no candidate qualifies: max, as np.float32
    got = th.epsilon_eval(torch.from_numpy(flat).cuda(), torch.from_numpy(flat).cuda(), np.zeros(500, np.int64))
    assert type(got["threshold"]) is np.float32 and got["threshold"] == np.float32(0.25)


def test_feature_epsilons():
    from mtad_gat_pytorch_b200 import thresholding as th
    from mtad_gat_pytorch_b200._lib import lib, check
    n, C = 3000, 38
    a = np.stack([_score_series(c, n) for c in range(C)], 1)
    b = np.stack([_score_series(100 + c, 2000) for c in range(C)], 1)
    wide = torch.zeros((n, C + 5), device="cuda")
    wide[:, 2:2 + C] = torch.from_numpy(a).cuda()
    x = wide[:, 2:2 + C]                                                 # row-strided view, read in place
    eps, ptr, pte = th.feature_epsilons(x, torch.from_numpy(b).cuda())
    eps_h = eps.cpu().numpy()
    for c in range(C):
        ref = float(tho.find_epsilon(a[:, c], 2))
        assert abs(eps_h[c] - ref) <= 2e-6 * max(1.0, abs(ref)), c
        one, _, _ = th.feature_epsilons(torch.from_numpy(np.ascontiguousarray(a[:, c])).cuda())
        assert one.cpu().numpy()[0] == eps_h[c]                            # bitwise
        out = torch.empty(3, dtype=torch.float32, device="cuda")
        scratch = torch.empty(int(lib.mtadgat_find_epsilon_scratch_doubles(n)), dtype=torch.float64, device="cuda")
        col = torch.from_numpy(np.ascontiguousarray(a[:, c])).cuda()
        check(lib.mtadgat_find_epsilon(col.data_ptr(), n, 2, out.data_ptr(), scratch.data_ptr(),
                                       torch.cuda.current_stream().cuda_stream))
        assert out.cpu().numpy()[0] == np.float32(eps_h[c])               # the float entry is its rounding
    assert np.array_equal(ptr.cpu().numpy(), a >= eps_h[None, :])
    assert np.array_equal(pte.cpu().numpy(), b >= eps_h[None, :])


def test_find_epsilon_outputs_unchanged():
    """mtadgat_find_epsilon's float outputs equal, bit for bit, those the library gave before the column generalisation
    (tests/golden/find_epsilon_outputs.npz, recorded on an H100)."""
    from mtad_gat_pytorch_b200 import thresholding as th
    g = np.load(os.path.join(GOLD, "find_epsilon_outputs.npz"))
    for key in g.files:
        seed, n, reg = (int(v) for v in key.split("_"))
        got = np.array(th.find_epsilon(torch.from_numpy(_score_series(seed, n)).cuda(), reg), np.float32)
        assert np.array_equal(got, g[key]), (key, got, g[key])


def test_runs_agree_and_graph_replay():
    from mtad_gat_pytorch_b200 import thresholding as th
    score, label = _case(427617, "spanning", seed=4)
    thr = _thresholds(score, 100, np.random.default_rng(4))
    s = torch.from_numpy(score).cuda()
    lab = torch.from_numpy(label).cuda()
    n = s.numel()
    tv = torch.tensor([th._compare_value(t) for t in thr], dtype=torch.float64, device="cuda")
    counts = torch.empty((100, 6), dtype=torch.int64, device="cuda")
    scratch = th._counts_scratch(n, 100, s.device)
    segs = th._segments(s, None, lab)
    th._launch_counts(s, None, segs, n, tv, 0, counts, scratch)
    first = counts.clone()
    th._launch_counts(s, None, th._segments(s, None, lab), n, tv, 0, counts, scratch)
    assert torch.equal(first, counts)
    stream = torch.cuda.Stream()
    stream.wait_stream(torch.cuda.current_stream())
    g = torch.cuda.CUDAGraph()
    with torch.cuda.stream(stream):
        with torch.cuda.graph(g, stream=stream):
            segs_g = th._segments(s, None, lab)
            th._launch_counts(s, None, segs_g, n, tv, 0, counts, scratch)
    counts.zero_()
    g.replay()
    torch.cuda.synchronize()
    assert torch.equal(first, counts)
    assert np.array_equal(first.cpu().numpy(), ev.point_adjusted_counts(score, label, thr))


def test_end_to_end_on_scored_series():
    """score_series on the SMD-1-1 replay rows (shipped checkpoint), synthetic labels, then bf_search / epsilon_eval on
    the device scores == the restatement on the same scores."""
    import mtad_gat_pytorch_b200 as mg
    from mtad_gat_pytorch_b200 import scoring, thresholding as th
    g = np.load(os.path.join(GOLD, "smd_1_1_replay.npz"))
    m = mg.MTAD_GAT(38, 100, 38, forecast_n_layers=3, dropout=0.3)
    m.load_state_dict({k[len("param."):]: torch.from_numpy(g[k]) for k in g.files if k.startswith("param.")})
    m.cuda().eval()
    res = scoring.score_series(m, torch.from_numpy(g["rows"]), batch=128)
    a = res["a_global"]
    ah = a.cpu().numpy()
    n = ah.shape[0]
    label = np.zeros(n, np.float32)
    for s0 in range(5, n, max(n // 7, 2)):
        label[s0:s0 + max(n // 40, 1)] = 1
    _same_dict(th.bf_search(a, label, start=0.01, end=2, step_num=100), ev.bf_search(ah, label, 0.01, 2, 100))
    half = n // 2
    got = th.epsilon_eval(a[:half].contiguous(), a[half:].contiguous(), label[half:], 1)
    ref = ev.epsilon_eval(ah[:half], ah[half:], label[half:], 1)
    assert abs(got["threshold"] - ref["threshold"]) <= 2e-6 * max(1.0, abs(ref["threshold"]))
    at = ev.threshold_eval(ah[half:], label[half:], got["threshold"])
    at["reg_level"] = 1
    _same_dict(got, at)


def test_bad_inputs_raise():
    from mtad_gat_pytorch_b200 import thresholding as th
    s = torch.rand(100, device="cuda")
    lab = np.zeros(100, np.float32)
    bad = lab.copy()
    bad[7] = 0.5
    with pytest.raises(ValueError):
        th.bf_search(s, bad, 0.5)                                        # label other than 0 / 1
    with pytest.raises(ValueError):
        th.threshold_eval(s, torch.full((100,), 2, dtype=torch.int64, device="cuda"), 0.5)
    with pytest.raises(ValueError):
        th.adjust_predicts(s, bad, 0.5)
    with pytest.raises(ValueError):
        th.bf_search(s, lab[:99], 0.5)                                   # length mismatch
    with pytest.raises(ValueError):
        th.bf_search(s.cpu(), lab, 0.5)                                  # host scores
    with pytest.raises(ValueError):
        th.bf_search(s.cpu().numpy(), lab, 0.5)
    with pytest.raises(ValueError):
        th.threshold_eval(s.double(), lab, 0.5)                          # float64 scores
    with pytest.raises(ValueError):
        th.bf_search(s, lab.astype(np.float64), 0.5)                     # float64 labels
    with pytest.raises(ValueError):
        th.feature_epsilons(s.double().view(50, 2))
