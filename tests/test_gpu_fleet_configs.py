"""Fleets whose streams each run their own configuration (FleetDetector / thresholding.SpotStreams with configs,
csrc/spot_mixed.cu): every stream bitwise its own StreamDetector through ragged pushes, equal configs bitwise a uniform
fleet, launch and read-back counts independent of S and of the rule mix, membership changes, records (saved, loaded,
imported from uniform fleets and refused by them), per-feature streams, errors, and a replay's winners deployed."""
import io

import numpy as np
import pytest
import torch

from tests.test_gpu_fleet import _model, _same, _schedule, _series

pytestmark = pytest.mark.gpu
K, N = 5, 20
KEYS = ("index", "a_score", "a_global", "threshold", "alarm")
LOWER = ("lower_threshold", "lower_alarm")
RULES = [{}, {"depth": 1}, {"depth": 16}, {"depth": 129}, {"bidirectional": True},
         {"bidirectional": True, "depth": 16}]


def _configs(S):
    """S configurations cycling through SPOT, dSPOT at depths 1, 16, 129, biSPOT and bidSPOT at depth 16, with q,
    level and with_alarm varying independently."""
    return [{**RULES[s % 6], "q": (1e-3, 1e-4)[s % 2], "level": (0.98, 0.99, 0.995)[s % 3],
             "with_alarm": s % 4 < 2} for s in range(S)]


def _data(S, seed=0, length=1200):
    rng = np.random.default_rng(seed)
    train = _series(rng, S, K, [length + 7 * s for s in range(S)])
    test = _series(rng, S, K, [300] * S, bump=True)
    return rng, train, test


def _pieces(schedule, s):
    return [rows[ids == s] for rows, ids in schedule]


def _solo(model, train, pieces, cfg, per_feature=False):
    from mtad_gat_pytorch_b200 import prediction
    det = prediction.StreamDetector(model, torch.from_numpy(train), per_feature=per_feature, **cfg)
    outs = [det.push(torch.from_numpy(p)) for p in pieces]
    return det, {key: torch.cat([o[key] for o in outs]) for key in outs[0]}


def _fleet_results(fleet, schedule, keys):
    S, got = fleet.n_streams, None
    for rows, ids in schedule:
        res = fleet.push(torch.from_numpy(rows), ids)
        off = res["offsets"].cpu().numpy()
        part = [{key: res[key][off[s]:off[s + 1]] for key in keys} for s in range(S)]
        got = part if got is None else [{key: torch.cat([g[key], p[key]]) for key in keys} for g, p in zip(got, part)]
    return got


def _check_stream(fleet, s, got, det, want, cfg):
    for key in KEYS:
        assert _same(got[key], want[key]), (s, key, cfg)
    if cfg.get("bidirectional"):
        for key in LOWER:
            assert _same(got[key], want[key]), (s, key, cfg)
        for name in ("t_lower", "quantile_lower"):
            assert np.array_equal(np.asarray(getattr(fleet, name)[s]), np.asarray(getattr(det, name)), equal_nan=True)
    else:
        assert torch.isnan(got["lower_threshold"]).all() and not got["lower_alarm"].any(), (s, cfg)
        assert np.isnan(fleet.t_lower[s]) and np.isnan(fleet.quantile_lower[s]) and fleet.n_peaks_lower[s] == 0
    assert np.array_equal(fleet.t[s:s + 1], np.atleast_1d(det.t))
    assert fleet.quantile[s].tobytes() == np.float64(det.quantile).tobytes()
    assert fleet.n[s] == det.spot.n and fleet.n_peaks[s] == det.spot.n_peaks
    for name, v in fleet.fit.items():
        assert v[s].tobytes() == np.float64(det.fit[name]).tobytes(), (s, name)


def test_each_stream_is_its_own_stream_detector():
    from mtad_gat_pytorch_b200 import prediction
    S = 12
    model = _model(K, N)
    rng, train, test = _data(S)
    cfgs = _configs(S)
    schedule, _ = _schedule(rng, test, N, 8)
    fleet = prediction.FleetDetector(model, [torch.from_numpy(x) for x in train], configs=cfgs)
    assert fleet.configs == [{"q": c["q"], "level": c["level"], "depth": c.get("depth"),
                              "bidirectional": c.get("bidirectional", False), "with_alarm": c["with_alarm"]}
                             for c in cfgs]
    assert fleet.depth is None and fleet.bidirectional is None and fleet.spots.q is None
    got = _fleet_results(fleet, schedule, KEYS + LOWER)
    for s in range(S):
        det, want = _solo(model, train[s], _pieces(schedule, s), cfgs[s])
        _check_stream(fleet, s, got[s], det, want, cfgs[s])


@pytest.mark.parametrize("rule", RULES[:3:2] + RULES[4:])
def test_equal_configs_equal_a_uniform_fleet(rule):
    from mtad_gat_pytorch_b200 import prediction
    S = 5
    model = _model(K, N)
    rng, train, test = _data(S, 1)
    schedule, _ = _schedule(rng, test, N, 5)
    xs = [torch.from_numpy(x) for x in train]
    mixed = prediction.FleetDetector(model, xs, configs=[dict(rule, level=0.98)] * S)
    uniform = prediction.FleetDetector(model, xs, level=0.98, **rule)
    for rows, ids in schedule:
        a = mixed.push(torch.from_numpy(rows), ids)
        b = uniform.push(torch.from_numpy(rows), ids)
        for key in b:
            if isinstance(b[key], torch.Tensor):
                assert _same(a[key], b[key]), key
    for name in ("t", "quantile", "n", "n_peaks", "flags"):
        assert getattr(mixed, name).tobytes() == getattr(uniform, name).tobytes(), name


def _warm(fleet, S, rng):
    for _ in range(2):
        fleet.push(torch.from_numpy(rng.random((S * (N + 2), K)).astype(np.float32)), np.repeat(np.arange(S), N + 2))


def test_costs_do_not_grow_with_streams_or_mix(monkeypatch):
    import mtad_gat_pytorch_b200 as mg
    from mtad_gat_pytorch_b200 import prediction
    model = _model(K, N)
    counts = []
    # level 0.9 leaves every peak array room enough that no push here grows one
    for S, kw in ((4, {"configs": _configs(4)}), (64, {"configs": _configs(64)}), (64, {"bidirectional": True})):
        kw = {"configs": [dict(c, level=0.9) for c in kw["configs"]]} if "configs" in kw else dict(kw, level=0.9)
        rng, train, _ = _data(S, 2, length=300)
        fleet = prediction.FleetDetector(model, [torch.from_numpy(x) for x in train], **kw)
        _warm(fleet, S, rng)
        rows = torch.from_numpy(rng.random((3 * S, K)).astype(np.float32))
        mg.reset_launch_count()
        fleet.push(rows, np.repeat(np.arange(S), 3))
        counts.append(mg.launch_count())
    assert counts[0] == counts[1] == counts[2], counts
    calls, real_cpu = [], torch.Tensor.cpu

    def counting_cpu(self, *a, **kw):
        calls.append(self.device.type)
        return real_cpu(self, *a, **kw)
    monkeypatch.setattr(torch.Tensor, "cpu", counting_cpu)
    rng, train, _ = _data(8, 3, length=300)
    f = prediction.FleetDetector(model, [torch.from_numpy(x) for x in train],
                                 configs=[dict(c, level=0.9) for c in _configs(8)])
    _warm(f, 8, rng)
    calls.clear()
    f.push(torch.from_numpy(rng.random((16, K)).astype(np.float32)), np.repeat(np.arange(8), 2))
    assert calls == ["cuda"]


def test_membership_changes_keep_streams_bitwise():
    from mtad_gat_pytorch_b200 import prediction
    S = 6
    model = _model(K, N)
    rng, train, test = _data(S + 3, 4)
    cfgs = _configs(S + 3)
    fleet = prediction.FleetDetector(model, [torch.from_numpy(x) for x in train[:S]], configs=cfgs[:S])
    first, _ = _schedule(rng, test[:S], N, 3)
    _fleet_results(fleet, first, KEYS)
    fleet.add_streams([torch.from_numpy(train[s]) for s in (S + 1, S + 2, S)],
                      configs=[cfgs[S + 1], cfgs[S + 2], cfgs[S]])
    mapping = fleet.remove_streams([1, 4])
    order = [s for s in range(S) if mapping[s] >= 0] + [S + 1, S + 2, S]
    assert [c["depth"] for c in fleet.configs] == [cfgs[s].get("depth") for s in order]
    used = [int(sum((ids == s).sum() for _, ids in first)) if s < S else 0 for s in order]
    later, _ = _schedule(rng, [test[s][u:] for s, u in zip(order, used)], N, 4)
    got = _fleet_results(fleet, later, KEYS + LOWER)
    for j, s in enumerate(order):
        det, want = _solo(model, train[s], (_pieces(first, s) if s < S else []) + _pieces(later, j), cfgs[s])
        tail = {key: v[v.shape[0] - got[j][key].shape[0]:] for key, v in want.items()}
        _check_stream(fleet, j, got[j], det, tail, cfgs[s])


def _push_both(a, b, rng, S, pushes=3):
    for _ in range(pushes):
        rows = torch.from_numpy(rng.random((2 * S + 3, K)).astype(np.float32))
        ids = rng.integers(0, S, 2 * S + 3)
        ra, rb = a.push(rows, ids), b.push(rows, ids)
        for key in rb:
            if isinstance(rb[key], torch.Tensor) and key in ra:
                assert _same(ra[key], rb[key]), key


def test_records_round_trip_and_uniform_records_import():
    import mtad_gat_pytorch_b200 as mg
    from mtad_gat_pytorch_b200 import prediction
    S = 6
    model = _model(K, N)
    rng, train, test = _data(S, 5)
    xs = [torch.from_numpy(x) for x in train]
    fleet = prediction.FleetDetector(model, xs, configs=_configs(S))
    schedule, _ = _schedule(rng, test, N, 3)
    _fleet_results(fleet, schedule, KEYS)
    buf = io.BytesIO()
    torch.save(fleet.state_dict(), buf)
    buf.seek(0)
    rec = torch.load(buf, weights_only=True)
    assert rec["configs"] == fleet.configs and rec["window_offsets"].shape == (S + 1,)
    assert "with_alarm" not in rec and "depth" not in rec and rec["spot_lower"].shape == (S, 24)
    resumed = prediction.FleetDetector.from_state_dict(model, rec)
    _push_both(fleet, resumed, rng, S)

    # uniform fleets' and a StreamDetector's records enter a per-stream fleet and continue bitwise
    for kw in ({}, {"depth": 8}, {"bidirectional": True}):
        uni = prediction.FleetDetector(model, xs[:3], **kw)
        _fleet_results(uni, _schedule(rng, test[:3], N, 2)[0], KEYS)
        target = prediction.FleetDetector(model, xs[:2], configs=_configs(2))
        ids = target.import_streams(uni.state_dict())
        assert list(ids) == [2, 3, 4]
        assert target.configs[2]["depth"] == kw.get("depth") and \
            target.configs[2]["bidirectional"] == kw.get("bidirectional", False)
        for _ in range(3):
            rows = torch.from_numpy(rng.random((7, K)).astype(np.float32))
            sid = rng.integers(0, 3, 7)
            ra, rb = target.push(rows, sid + 2), uni.push(rows, sid)
            for key in ("a_global", "threshold", "alarm"):
                assert _same(ra[key], rb[key]), (kw, key)
        again = prediction.FleetDetector.from_state_dict(model, uni.state_dict(), per_stream=True)
        assert again.configs is not None
    det = prediction.StreamDetector(model, xs[0], depth=4, bidirectional=True, level=0.98)
    det.push(torch.from_numpy(test[0][:N + 9]))
    target = prediction.FleetDetector(model, xs[:2], configs=_configs(2))
    target.import_streams(det.state_dict())
    for _ in range(3):
        rows = rng.random((4, K)).astype(np.float32)
        ra, rb = target.push(torch.from_numpy(rows), np.full(4, 2)), det.push(torch.from_numpy(rows))
        for key in ("threshold", "lower_threshold", "alarm", "lower_alarm"):
            assert _same(ra[key], rb[key]), key

    # uniform detectors refuse a per-stream record, launching nothing and changing nothing
    uni = prediction.FleetDetector(model, xs[:2])
    before, one = uni.spots._words.copy(), fleet.state_dict([0])
    mg.reset_launch_count()
    with pytest.raises(ValueError, match="configs"):
        uni.import_streams(rec)
    with pytest.raises(ValueError, match="configs"):
        prediction.StreamDetector.from_state_dict(model, one)
    assert mg.launch_count() == 0 and uni.n_streams == 2 and np.array_equal(uni.spots._words, before)


def test_per_feature_streams_run_their_stream_configuration():
    from mtad_gat_pytorch_b200 import prediction
    S = 6
    model = _model(K, N)
    rng, train, test = _data(S, 6)
    cfgs = _configs(S)
    fleet = prediction.FleetDetector(model, [torch.from_numpy(x) for x in train], configs=cfgs, per_feature=True)
    schedule, _ = _schedule(rng, test, N, 4)
    fkeys = ("feature_threshold", "feature_alarm", "feature_lower_threshold", "feature_lower_alarm")
    got = _fleet_results(fleet, schedule, KEYS + fkeys)
    for s in range(S):
        _, want = _solo(model, train[s], _pieces(schedule, s), cfgs[s], per_feature=True)
        for key in ("feature_threshold", "feature_alarm") + (fkeys[2:] if cfgs[s].get("bidirectional") else ()):
            assert _same(got[s][key], want[key]), (s, key)
        if not cfgs[s].get("bidirectional"):
            assert torch.isnan(got[s]["feature_lower_threshold"]).all()
    rec = fleet.state_dict([4, 1])
    resumed = prediction.FleetDetector.from_state_dict(model, rec)
    assert resumed.configs == [fleet.configs[4], fleet.configs[1]]


def test_errors_name_the_stream():
    import mtad_gat_pytorch_b200 as mg
    from mtad_gat_pytorch_b200 import prediction
    S = 4
    model = _model(K, N)
    rng, train, test = _data(S, 7)
    xs = [torch.from_numpy(x) for x in train]
    mg.reset_launch_count()
    for bad, match in (({"depht": 3}, "stream 1"), ({"depth": 2000}, "stream 1"),
                       ({"bidirectional": True, "level": 0.5}, "stream 1")):
        with pytest.raises(ValueError, match=match):
            prediction.FleetDetector(model, xs[:2], configs=[{}, bad])
    assert mg.launch_count() == 0
    for errors in ("flag", "raise"):
        fleet = prediction.FleetDetector(model, xs, configs=_configs(S), errors=errors)
        rows = np.concatenate([test[s][:N + 4] for s in range(S)])
        ids = np.repeat(np.arange(S), N + 4)
        rows[ids == 2] = np.nan
        if errors == "flag":
            res = fleet.push(torch.from_numpy(rows), ids)
            assert [bool(f) for f in res["flags"]] == [False, False, True, False]
        else:
            with pytest.raises(ValueError, match="stream 2"):
                fleet.push(torch.from_numpy(rows), ids)


def test_replay_winners_deploy_bitwise():
    from mtad_gat_pytorch_b200 import prediction, scoring, thresholding as th
    S = 3
    model = _model(K, N)
    rng, train, test = _data(S, 8)
    grid = [{"q": 1e-3, "level": 0.98}, {"depth": 16, "level": 0.99, "with_alarm": False},
            {"bidirectional": True, "level": 0.98}, {"bidirectional": True, "depth": 8, "q": 1e-4}]
    sc = scoring.SeriesScorer(model)
    chosen, alarms = [1, 2, 3], []
    for s in range(S):
        tr = scoring.row_mean(sc.score(torch.from_numpy(train[s]), 1.0, None)["a_score"])
        te = scoring.row_mean(sc.score(torch.from_numpy(test[s]), 1.0, None)["a_score"])
        alarms.append(th.replay(tr, te, grid)["alarms"][chosen[s]] != 0)
    fleet = prediction.FleetDetector(model, [torch.from_numpy(x) for x in train],
                                     configs=[grid[c] for c in chosen])
    rows = np.concatenate(test)
    ids = np.repeat(np.arange(S), [t.shape[0] for t in test])
    res = fleet.push(torch.from_numpy(rows), ids)
    off = res["offsets"].cpu().numpy()
    for s in range(S):
        assert torch.equal(res["alarm"][off[s]:off[s + 1]], alarms[s]), s
