"""Replays over many labelled streams on the device (thresholding.replay_streams / replay_streams_eval,
prediction.replay_fleet / replay_channels; csrc/spot_mixed.cu's mtadgat_spot_fleet_replay): every (stream,
configuration) walk bitwise a SpotStream of that configuration pushed the whole stream; the evaluation dicts equal to
the oracle's evaluation of those alarms for float32, int64 and bool labels; results independent of the chunk size and
of the run; more walks than resident CTAs; stopped walks; one read-back and one walk launch per chunk; and the
model-level replays against replay_detectors and FleetDetector.from_channels."""
import numpy as np
import pytest
import torch

from tests.test_gpu_replay import KEEP, _eq, _grid, _labels, _oracle, _same_eval, _series, _solo

pytestmark = pytest.mark.gpu
# (training, test) lengths: one shorter than the chunk, one over several chunks, one training set just longer than
# depth 129 of the grid
SHAPES = [(1500, 700), (1200, 3500), (160, 2000), (1000, 1000), (800, 2600)]


def _streams(shapes, seed=0):
    trs, ss = zip(*(_series(seed + s, n, m) for s, (n, m) in enumerate(shapes)))
    return list(trs), list(ss)


def _same_replay(got, want):
    """One stream's replay_streams dicts of two runs, bitwise."""
    for key in ("alarms", "thresholds", "lower_thresholds", "flags"):
        assert (got[key] is None) == (want[key] is None), key
        assert want[key] is None or _eq(got[key], want[key]), key
    assert torch.equal(got["state"][..., KEEP], want["state"][..., KEEP])


def _reference(tr, x, cfg):
    """`_solo`'s (alarm codes, thresholds, lower thresholds or None, state (2, 24)) for `cfg` on one stream, and None;
    or, for a configuration SpotStream refuses to initialise, no alarms, NaN thresholds, the state words its
    initialisation left and SpotStream's ValueError."""
    from mtad_gat_pytorch_b200 import thresholding as th
    try:
        return _solo(tr, x, cfg) + (None,)
    except ValueError as err:
        bi = cfg.get("bidirectional", False)
        init = th._initialise([tr], cfg["level"], cfg["q"], cfg.get("depth"), bi, lambda n, k: n - k + 1, tr.device)[0]
        state = torch.zeros(2, 24, dtype=torch.int64, device="cuda")
        state[:2 if bi else 1] = init[:, 0]
        nan = torch.full((x.numel(),), float("nan"), dtype=torch.float64, device="cuda")
        return torch.zeros(x.numel(), dtype=torch.uint8, device="cuda"), nan, nan if bi else None, state, err


def _same_walk(got, c, cfg, ref):
    """Configuration c of one stream's replay_streams dict against `_reference`'s result: bitwise, or for a refused
    configuration a walk stopped for SpotStream's reason that processed nothing."""
    from mtad_gat_pytorch_b200 import thresholding as th
    al, thr, low, state, err = ref
    assert _eq(got["alarms"][c], al), c
    if err is None:
        assert _eq(got["thresholds"][c], thr) and (low is None or _eq(got["lower_thresholds"][c], low)), c
    else:
        with pytest.raises(ValueError) as reason:
            th._stream_status(got["state"][:, c:c + 1].cpu().numpy()[:1 if low is None else 2], 0, "")
        assert str(err).endswith(str(reason.value)), (c, str(err))
        assert bool(torch.isnan(got["thresholds"][c]).all()), c
        assert low is None or bool(torch.isnan(got["lower_thresholds"][c]).all()), c
    if low is None:                                                    # one-sided: a NaN row, or no lower matrix
        assert got["lower_thresholds"] is None or bool(torch.isnan(got["lower_thresholds"][c]).all()), c
    assert torch.equal(got["state"][:, c][:, KEEP], state[:, KEEP]), c
    assert int(got["flags"][c]) == int(state[0, 4] | state[1, 4]), c


def test_every_stream_is_its_single_stream_replay_bitwise():
    """Every (stream, configuration) walk against a SpotStream initialised on that stream alone, and every evaluation
    dict against the oracle's evaluation of the SpotStream's alarms."""
    from mtad_gat_pytorch_b200 import thresholding as th
    trs, ss = _streams(SHAPES)
    grid = _grid()
    got = th.replay_streams(trs, ss, grid, thresholds=True, chunk=1000)
    assert len(got) == len(SHAPES)
    refs = [[_reference(tr, x, cfg) for cfg in grid] for tr, x in zip(trs, ss)]
    for s, x in enumerate(ss):
        assert got[s]["alarms"].shape == (len(grid), x.numel())
        for c, cfg in enumerate(grid):
            _same_walk(got[s], c, cfg, refs[s][c])
    assert sum(r[-1] is None for rs in refs for r in rs) > 0.9 * len(SHAPES) * len(grid)
    assert any(bool((g["alarms"] == 2).any()) for g in got) and any(bool((g["alarms"] == 1).any()) for g in got)
    for dt in (np.float32, np.int64, np.bool_):
        labs = [_labels(x.numel(), 10 + s).astype(dt) for s, x in enumerate(ss)]
        res = th.replay_streams_eval(trs, ss, labs, grid, chunk=1000)
        for s, lab in enumerate(labs):
            assert len(res[s]) == len(grid)
            for c, (al, _, _, state, _) in enumerate(refs[s]):
                codes = al.cpu().numpy()
                want = _oracle(codes, lab)
                want.update(alarms=int(np.count_nonzero(codes)), refits=int(state[0, 9] + state[1, 9]),
                            flags=int(state[0, 4] | state[1, 4]))
                assert res[s][c] == want, (dt, s, c)
                _same_eval(res[s][c], want)


def test_chunk_size_and_runs_do_not_change_bits():
    from mtad_gat_pytorch_b200 import thresholding as th
    trs, ss = _streams(SHAPES[:4], 20)
    grid = _grid()
    runs = [th.replay_streams(trs, ss, grid, thresholds=True, chunk=c) for c in (333, 65536, 333)]
    for r in runs[1:]:
        for s in range(len(ss)):
            _same_replay(r[s], runs[0][s])
    labs = [_labels(x.numel(), 30 + s) for s, x in enumerate(ss)]
    evals = [th.replay_streams_eval(trs, ss, labs, grid, chunk=c) for c in (333, 65536, 65536)]
    assert evals[0] == evals[1] == evals[2]


def test_more_walks_than_resident_ctas():
    """S * C = 7 * 48 walks (two CTAs per SM on 132 SMs keep 264 resident), streams whose scales and lengths give very
    different refit counts; walks spot-checked against SpotStream."""
    from mtad_gat_pytorch_b200 import thresholding as th
    trs, ss = _streams([(900, 400), (700, 1800), (1200, 250), (600, 900), (1000, 1300), (500, 600), (800, 2200)], 40)
    ss[1] = ss[1] * 3.0                                                # a stream far beyond its training tail
    grid = _grid()
    got = th.replay_streams(trs, ss, grid, thresholds=True, chunk=512)
    refits = []
    for s, (tr, x) in enumerate(zip(trs, ss)):
        refits.append(int(got[s]["state"][:, :, 9].sum()))
        for c in range(s % 5, len(grid), 5):
            _same_walk(got[s], c, grid[c], _reference(tr, x, grid[c]))
    assert max(refits) > 2 * min(refits), refits


def test_stopped_walks():
    """A NaN in one stream's test scores stops every configuration of that stream where SpotStreams(errors="flag")
    stops; the other streams are bitwise a clean run."""
    from mtad_gat_pytorch_b200 import thresholding as th
    trs, ss = _streams([SHAPES[0], SHAPES[1], SHAPES[3]], 50)
    grid = _grid()[::3]
    bad = [x.clone() for x in ss]
    bad[1][700] = float("nan")
    clean = th.replay_streams(trs, ss, grid, thresholds=True, chunk=500)
    got = th.replay_streams(trs, bad, grid, thresholds=True, chunk=500)
    for s in (0, 2):
        _same_replay(got[s], clean[s])
        assert not got[s]["flags"].any()
    for c, cfg in enumerate(grid):
        sp = th.SpotStreams([trs[1]], cfg["q"], cfg["level"], cfg["with_alarm"], "flag", cfg.get("depth"),
                            cfg.get("bidirectional", False))
        out = sp.push(bad[1], [0, bad[1].numel()])
        assert _eq(got[1]["thresholds"][c], out[0]), c
        assert int(got[1]["flags"][c]) == int(sp.flags[0]) == 1
        assert int(got[1]["state"][0, c, 10]) == 700
    labs = [_labels(x.numel(), 60 + s) for s, x in enumerate(bad)]
    res = th.replay_streams_eval(trs, bad, labs, grid)
    assert all(r["flags"] == 1 for r in res[1]) and all(r["flags"] == 0 for s in (0, 2) for r in res[s])
    with pytest.raises(ValueError, match="stream 1, configuration 0: NaN scores"):
        th.replay_streams_eval(trs, bad, labs, grid, errors="raise")


class _Counting:
    """th.lib with the calls of one entry point counted."""

    def __init__(self, lib, name):
        self.lib, self.name, self.calls = lib, name, 0

    def __getattr__(self, attr):
        fn = getattr(self.lib, attr)
        if attr != self.name:
            return fn

        def counted(*a):
            self.calls += 1
            return fn(*a)
        return counted


@pytest.mark.parametrize("S", [2, 16])
def test_one_walk_launch_per_chunk_and_one_read_back(S, monkeypatch):
    from mtad_gat_pytorch_b200 import thresholding as th
    shapes = [(600 + 37 * s, 300 + 211 * s) for s in range(S)]
    trs, ss = _streams(shapes, 70)
    labs = [_labels(x.numel(), 80 + s) for s, x in enumerate(ss)]
    grid = _grid()[::5]
    th.replay_streams_eval(trs, ss, labs, grid, chunk=256)             # warm-up
    torch.cuda.synchronize()
    counter = _Counting(th.lib, "mtadgat_spot_fleet_replay")
    monkeypatch.setattr(th, "lib", counter)
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
    res = th.replay_streams_eval(trs, ss, labs, grid, chunk=256)
    assert [d.type for d in calls] == ["cuda"]
    assert len(res) == S and all(len(r) == len(grid) for r in res)
    assert counter.calls == -(-max(x.numel() for x in ss) // 256)
    counter.calls = 0
    th.replay_streams(trs, ss, grid[1:2], chunk=1000)                  # one configuration, one rule
    assert counter.calls == -(-max(x.numel() for x in ss) // 1000)


def _fleet_data(rng, S, k=5):
    from tests.test_gpu_fleet import _series as rows
    train = rows(rng, S, k, [700 + 90 * s for s in range(S)])
    test = rows(rng, S, k, [260 + 70 * s for s in range(S)], bump=True)
    return [torch.from_numpy(x) for x in train], [torch.from_numpy(x) for x in test]


CONFIGS = [dict(level=0.9), dict(level=0.95, depth=16, with_alarm=False), dict(level=0.9, bidirectional=True),
           dict(q=1e-2, level=0.98, bidirectional=True, depth=16), dict(level=0.98, depth=1)]


def test_replay_fleet_is_replay_detectors_per_stream():
    from mtad_gat_pytorch_b200 import prediction
    from tests.test_gpu_fleet import _model
    model = _model()
    rng = np.random.default_rng(3)
    train, test = _fleet_data(rng, 3)
    labs = [_labels(x.shape[0] - 20, 90 + s).astype(np.int64) for s, x in enumerate(test)]
    got = prediction.replay_fleet(model, train, test, labs, CONFIGS, gamma=0.7)
    for s in range(3):
        assert got[s] == prediction.replay_detectors(model, train[s], test[s], labs[s], CONFIGS, gamma=0.7), s


def test_replay_channels_and_their_winners_deployed(tmp_path):
    """replay_channels on a synthetic SMAP metadata directory is replay_fleet on the split series, and its winners
    passed to FleetDetector.from_channels give every channel bitwise the StreamDetector of its winning
    configuration."""
    from mtad_gat_pytorch_b200 import prediction
    from tests.test_gpu_fleet import _model
    from tests.test_prediction_cpu import write_metadata
    model = _model()
    rng = np.random.default_rng(5)
    train, test = _fleet_data(rng, 3)
    write_metadata(str(tmp_path), "SMAP", [x.shape[0] for x in train], [x.shape[0] for x in test])
    d = str(tmp_path / "datasets" / "data")
    x_train, x_test = torch.cat(train), torch.cat(test)
    label = np.concatenate([np.concatenate([np.zeros(20, np.float32), _labels(x.shape[0] - 20, 100 + s)])
                            for s, x in enumerate(test)])
    got = prediction.replay_channels(model, x_train, x_test, label, "SMAP", CONFIGS, data_dir=d)
    b = np.concatenate([[0], np.cumsum([x.shape[0] for x in test])])
    want = prediction.replay_fleet(model, train, test, [label[b[s] + 20:b[s + 1]] for s in range(3)], CONFIGS)
    assert got == want
    best = [CONFIGS[max(range(len(CONFIGS)), key=lambda c: (r[c]["f1"], -c))] for r in got]
    fleet = prediction.FleetDetector.from_channels(model, x_train, "SMAP", data_dir=d, configs=best)
    rows = [x[:60].numpy() for x in test]
    res = fleet.push(torch.from_numpy(np.concatenate(rows)), np.repeat(np.arange(3), 60))
    off = res["offsets"].cpu().numpy()
    for s in range(3):
        det = prediction.StreamDetector(model, train[s], **best[s])
        want = det.push(torch.from_numpy(rows[s]))
        for key in ("a_global", "threshold", "alarm"):
            assert _eq(res[key][off[s]:off[s + 1]], want[key]), (s, key)
