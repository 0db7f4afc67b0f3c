"""Replays on the device (thresholding.replay / replay_eval, prediction.replay_detectors; csrc's mtadgat_*_replay and
mtadgat_eval_counts_rows): every configuration of a grid of SPOT, dSPOT (depths 1, 16, 129), biSPOT and bidSPOT, two
levels, two q values and both with_alarm, bitwise a SpotStream initialised alone and pushed the whole series (in one
push and in ragged pushes); the evaluation dicts equal to the oracle's evaluation of those alarms for float32, int64 and
bool labels; results independent of the chunk size and of the run; C = 1 and C = 300; stopped configurations; the
detectors' replay against StreamDetectors; and the read-back count."""
import numpy as np
import pytest
import torch

from oracle import evaluation_oracle as ev
from tests.test_stream_cpu import gpd

pytestmark = pytest.mark.gpu
KEEP = [w for w in range(24) if w not in (5, 6)]                       # all but the peak array's address, capacity
PERSIST = [w for w in KEEP if w not in (8, 9, 10)]                     # and the counts of the last push
RULES = [dict(), dict(depth=1), dict(depth=16), dict(depth=129), dict(bidirectional=True),
         dict(bidirectional=True, depth=16)]


def _grid():
    return [dict(rule, q=q, level=level, with_alarm=wa) for rule in RULES for level in (0.9, 0.98)
            for q in (1e-3, 1e-2) for wa in (True, False)]


def _series(seed, n_init, m):
    """Two-sided heavy tails on a slow ramp, so every rule refits on both sides and alarms."""
    rng = np.random.default_rng(seed)
    ramp = np.linspace(0, 0.3, n_init + m).astype(np.float32)
    x = (gpd(rng, n_init + m) - gpd(rng, n_init + m) + ramp).astype(np.float32)
    return torch.from_numpy(x[:n_init]).cuda(), torch.from_numpy(x[n_init:]).cuda()


def _labels(m, seed):
    """0 / 1 labels with a segment at index 0, one at the end and some in between."""
    rng = np.random.default_rng(seed)
    lab = np.zeros(m, np.float32)
    lab[:25] = 1
    lab[-40:] = 1
    for s in rng.integers(50, m - 100, 12):
        lab[s:s + rng.integers(1, 60)] = 1
    return lab


def _bits(x):
    return x.contiguous().view(torch.int64) if x.dtype == torch.float64 else x


def _eq(a, b):
    return a.shape == b.shape and torch.equal(_bits(a), _bits(b))


def _solo(tr, s, cfg, pieces=None):
    """SpotStream with `cfg` pushed `s` whole (or in `pieces`): (alarm codes uint8, thresholds, lower or None, state
    (2, 24) with a zero lower block when one-sided)."""
    from mtad_gat_pytorch_b200 import thresholding as th
    sp = th.SpotStream(tr, cfg.get("q", 1e-3), cfg.get("level", 0.99), cfg.get("with_alarm", True),
                       depth=cfg.get("depth"), bidirectional=cfg.get("bidirectional", False))
    bounds = [0] + list(np.cumsum(pieces or [s.numel()]))
    outs = [sp.push(s[a:b]) for a, b in zip(bounds[:-1], bounds[1:])]
    cat = [torch.cat([o[j] for o in outs]) for j in range(len(outs[0]))]
    state = torch.zeros(2, 24, dtype=torch.int64, device="cuda")
    if sp.bidirectional:
        state.copy_(sp.state)
        return cat[2], cat[0], cat[1], state
    state[0] = sp.state
    return cat[1].to(torch.uint8), cat[0], None, state


def _oracle(alarms, label):
    """eval_methods.py adjust_predicts(pred=alarms != 0) + calc_point2point, restated (oracle/)."""
    pred = np.asarray(alarms) != 0
    p, latency = ev.adjust_predicts(None, label, 0.0, pred=pred, calc_latency=True)
    f1, precision, recall, TP, TN, FP, FN = ev.calc_point2point(p, label)
    return {"f1": f1, "precision": precision, "recall": recall, "TP": TP, "TN": TN, "FP": FP, "FN": FN,
            "latency": latency}


def _same_eval(got, want):
    for key, v in want.items():
        assert got[key] == v and type(got[key]) is type(v), (key, got[key], v)


def test_grid_is_spot_streams_bitwise():
    from mtad_gat_pytorch_b200 import thresholding as th
    tr, s = _series(0, 2000, 3000)
    grid = _grid()
    rep = th.replay(tr, s, grid, thresholds=True, chunk=1000)
    assert not rep["flags"].any()
    lab = _labels(s.numel(), 1)
    evals = {dt: th.replay_eval(tr, s, lab.astype(dt), grid) for dt in (np.float32, np.int64, np.bool_)}
    pieces = [1, 700, 13, 1286, 1000]
    for c, cfg in enumerate(grid):
        al, thr, low, state = _solo(tr, s, cfg)
        assert _eq(rep["alarms"][c], al), c
        assert _eq(rep["thresholds"][c], thr), c
        if low is not None:
            assert _eq(rep["lower_thresholds"][c], low), c
        else:
            assert torch.isnan(rep["lower_thresholds"][c]).all()
        assert torch.equal(rep["state"][:, c][:, KEEP], state[:, KEEP]), c
        al2, thr2, low2, state2 = _solo(tr, s, cfg, pieces)
        assert _eq(al2, al) and _eq(thr2, thr) and (low is None or _eq(low2, low)), c
        assert torch.equal(rep["state"][:, c][:, PERSIST], state2[:, PERSIST]), c
        codes = al.cpu().numpy()
        for dt, res in evals.items():
            _same_eval(res[c], _oracle(codes, lab.astype(dt)))
            assert res[c]["alarms"] == int(np.count_nonzero(codes)) and res[c]["flags"] == 0
            assert res[c]["refits"] == int(state[0, 9] + state[1, 9]) > 0
    assert any(r["TP"] > 0 for r in evals[np.float32]) and any(r["FP"] > 0 for r in evals[np.float32])
    assert (rep["alarms"] == 2).any() and (rep["alarms"] == 1).any()


def test_chunk_size_and_runs_do_not_change_bits():
    from mtad_gat_pytorch_b200 import thresholding as th
    tr, s = _series(2, 1500, 2500)
    grid = _grid()
    runs = [th.replay(tr, s, grid, thresholds=True, chunk=c) for c in (333, 65536, 333)]
    for r in runs[1:]:
        for key in ("alarms", "thresholds", "lower_thresholds", "flags"):
            assert _eq(r[key], runs[0][key]), key
        assert torch.equal(r["state"][..., KEEP], runs[0]["state"][..., KEEP])
    lab = _labels(s.numel(), 3)
    assert th.replay_eval(tr, s, lab, grid, chunk=333) == th.replay_eval(tr, s, lab, grid, chunk=100000)


def test_one_and_more_configurations_than_resident_ctas():
    """C = 300 (more CTAs than two per SM on 132 SMs) against C = 1 runs and against SpotStreams."""
    from mtad_gat_pytorch_b200 import thresholding as th
    tr, s = _series(4, 800, 700)
    grid = _grid()
    big = [dict(grid[c % len(grid)], level=0.9 + 0.0003 * c) for c in range(300)]
    rep = th.replay(tr, s, big, thresholds=True, chunk=256)
    for c in range(0, 300, 23):
        one = th.replay(tr, s, [big[c]], thresholds=True)
        for key in ("alarms", "thresholds"):
            assert _eq(one[key][0], rep[key][c]), (c, key)
        assert torch.equal(one["state"][:, 0][:, KEEP], rep["state"][:, c][:, KEEP]), c
        al, thr, _, state = _solo(tr, s, big[c])
        assert _eq(rep["alarms"][c], al) and _eq(rep["thresholds"][c], thr), c
        assert torch.equal(rep["state"][:, c][:, KEEP], state[:, KEEP]), c


def test_stopped_configurations(monkeypatch):
    """A NaN score stops every walk where a SpotStreams(errors="flag") stops; a configuration whose peak array runs
    out stops alone and leaves the others bitwise intact."""
    from mtad_gat_pytorch_b200 import thresholding as th
    tr, s = _series(5, 1000, 1200)
    grid = _grid()[::3]
    bad = s.clone()
    bad[700] = float("nan")
    rep = th.replay(tr, bad, grid, thresholds=True, chunk=500)
    for c, cfg in enumerate(grid):
        sp = th.SpotStreams([tr], cfg["q"], cfg["level"], cfg["with_alarm"], "flag", cfg.get("depth"),
                            cfg.get("bidirectional", False))
        out = sp.push(bad, [0, bad.numel()])
        assert _eq(rep["thresholds"][c], out[0]) and _eq(rep["alarms"][c], out[-1].to(torch.uint8)), c
        assert int(rep["flags"][c]) == int(sp.flags[0]) == 1
        assert int(rep["state"][0, c, 10]) == 700
    res = th.replay_eval(tr, bad, _labels(bad.numel(), 6), grid)
    assert all(r["flags"] == 1 for r in res)
    with pytest.raises(ValueError, match="configuration 0: NaN scores"):
        th.replay_eval(tr, bad, _labels(bad.numel(), 6), grid, errors="raise")

    clean = th.replay(tr, s, grid, thresholds=True, chunk=500)
    room = th._replay_room

    def keys(g):                                                       # (n_init, k) of each side's peak array
        n = tr.numel() - (g.get("depth") or 0)
        up = (n, int(g["level"] * n))
        return [up, (n, n - 1 - int((1 - g["level"]) * n))] if g.get("bidirectional") else [up]
    every = [key for g in grid for key in keys(g)]
    target = next(c for c, g in enumerate(grid) if len(keys(g)) == 1 and every.count(keys(g)[0]) == 1)
    small = keys(grid[target])[0]
    monkeypatch.setattr(th, "_replay_room", lambda ni, k, m: ni - k + 3 if (ni, k) == small else room(ni, k, m))
    full = th.replay(tr, s, grid, thresholds=True, chunk=500)
    assert int(full["flags"][target]) & 16
    for c in range(len(grid)):
        if c != target:
            for key in ("alarms", "thresholds", "flags"):
                assert _eq(full[key][c], clean[key][c]), (c, key)
            assert torch.equal(full["state"][:, c][:, KEEP], clean["state"][:, c][:, KEEP])


def test_replay_detectors_are_stream_detectors():
    """replay_detectors' scores are a StreamDetector's training and pushed scores bit for bit, so every configuration's
    alarms, thresholds and state are the detector's, and its evaluation is the oracle's evaluation of them."""
    from mtad_gat_pytorch_b200 import prediction, scoring, thresholding as th
    from tests.test_gpu_fleet import _model
    model = _model()
    rng = np.random.default_rng(7)
    x_train = torch.from_numpy(rng.random((900, 5)).astype(np.float32))
    x_test = rng.random((700, 5)).astype(np.float32)
    x_test[300:310] += 2.0
    x_test[500:503] -= 1.0
    x_test = torch.from_numpy(x_test)
    configs = [dict(level=0.9), dict(level=0.95, depth=16, with_alarm=False), dict(level=0.9, bidirectional=True),
               dict(q=1e-2, level=0.98, bidirectional=True, depth=16)]
    lab = _labels(700 - 20, 8).astype(np.int64)
    res = prediction.replay_detectors(model, x_train, x_test, lab, configs, gamma=0.7)
    sc = scoring.SeriesScorer(model)
    tr, te = (scoring.row_mean(sc.score(x, 0.7)["a_score"]) for x in (x_train, x_test))
    rep = th.replay(tr, te, configs, thresholds=True)
    bad = []
    for c, cfg in enumerate(configs):
        det = prediction.StreamDetector(model, x_train, gamma=0.7, **cfg)
        out = det.push(x_test)
        two = cfg.get("bidirectional", False)
        codes = out["alarm"].to(torch.uint8) + (out["lower_alarm"].to(torch.uint8) if two else 0)
        words = torch.zeros(2, 24, dtype=torch.int64, device="cuda")
        words[:2 if two else 1] = det.spot._state.view(-1, 24)
        checks = {"train scores": _eq(det.train_scores, tr), "scores": _eq(out["a_global"], te),
                  "alarms": _eq(rep["alarms"][c], codes), "thresholds": _eq(rep["thresholds"][c], out["threshold"]),
                  "lower": not two or _eq(rep["lower_thresholds"][c], out["lower_threshold"]),
                  "state": torch.equal(rep["state"][:, c][:, KEEP], words[:, KEEP])}
        bad += [(c, k) for k, ok in checks.items() if not ok]
        want = _oracle(codes.cpu().numpy(), lab)
        want.update(alarms=int(out["alarm"].sum()), refits=int(words[:, 9].sum()), flags=0)
        if res[c] != want:
            bad.append((c, "evaluation", res[c], want))
    assert not bad, bad


def test_replay_eval_reads_back_once(monkeypatch):
    """After the checks, replay_eval copies one buffer to the host: counts and state words of every configuration."""
    from mtad_gat_pytorch_b200 import thresholding as th
    tr, s = _series(9, 1000, 5000)
    lab = _labels(s.numel(), 10)
    grid = _grid()
    th.replay_eval(tr, s, lab, grid, chunk=1024)                       # warm-up
    torch.cuda.synchronize()
    calls = []
    real_cpu = torch.Tensor.cpu

    def counting_cpu(self, *a, **k):
        calls.append(self.device)
        return real_cpu(self, *a, **k)

    def refuse(fn):
        def wrapped(self, *a, **k):
            assert not self.is_cuda, f"{fn.__name__} on a CUDA tensor"
            return fn(self, *a, **k)
        return wrapped
    for name in ("item", "tolist", "numpy"):
        monkeypatch.setattr(torch.Tensor, name, refuse(getattr(torch.Tensor, name)))
    monkeypatch.setattr(torch.Tensor, "cpu", counting_cpu)
    res = th.replay_eval(tr, s, lab, grid, chunk=1024)
    assert [d.type for d in calls] == ["cuda"]
    assert len(res) == len(grid)
