"""CPU tests of replays over many labelled streams (thresholding.replay_streams / replay_streams_eval,
prediction.replay_fleet; csrc/spot_mixed.cu's mtadgat_spot_fleet_replay): every bad argument refused with a ValueError
naming the stream before anything is launched, the host walk table and ragged offsets against a plain-Python
restatement, the fleet replay kernel in the sm_90a build, and the per-rule replay entry points gone."""
import os
import subprocess

import numpy as np
import pytest
import torch


class NoLib:
    def __getattr__(self, name):
        raise AssertionError(f"{name} launched")


@pytest.fixture
def no_launch(monkeypatch):
    """Scores are taken as they come (no device here) and every thresholding library function raises if reached."""
    import mtad_gat_pytorch_b200 as mg
    from mtad_gat_pytorch_b200 import thresholding as th
    monkeypatch.setattr(th, "lib", NoLib())
    monkeypatch.setattr(th, "_scores", lambda x, what: x.reshape(-1))
    mg.reset_launch_count()
    yield
    assert mg.launch_count() == 0


def _streams(lengths):
    return [torch.zeros(n) for n in lengths]


BAD = [  # (training lengths, test lengths, label lengths, configs, match)
    ([100, 100], [50, 60, 70], [50, 60, 70], [{}], "2 training series but 3 test series"),
    ([], [], [], [{}], "0 training series but 0 test series"),
    ([100, 100], [50, 0], [50, 0], [{}], "stream 1: empty scores"),
    ([100, 0], [50, 60], [50, 60], [{}], "stream 1: empty scores"),
    ([100, 100, 30], [50, 60, 70], [50, 60, 70], [{}, {"depth": 30}], "stream 2: configuration 1: 30 training scores"),
    ([100, 100], [50, 60], [50, 60], [{}] * 65536, "stream 0: 1 to 65535 configurations"),
    ([100, 100], [50, 60], [50, 60], [], "stream 0: 1 to 65535 configurations"),
    ([100, 100], [50, 60], [50, 60], [{"level": 0.9}, {"spam": 1}], "stream 0: configuration 1: a mapping"),
]


@pytest.mark.parametrize("ns,ms,ls,configs,match", BAD)
def test_bad_streams_are_refused_before_any_launch(ns, ms, ls, configs, match, no_launch):
    from mtad_gat_pytorch_b200 import thresholding as th
    labels = [np.zeros(n, np.float32) for n in ls]
    with pytest.raises(ValueError, match=match):
        th.replay_streams(_streams(ns), _streams(ms), configs)
    with pytest.raises(ValueError, match=match):
        th.replay_streams_eval(_streams(ns), _streams(ms), labels, configs)


@pytest.mark.parametrize("labels,match", [
    ([np.zeros(50, np.float32)], "a list of 2 label vectors"),
    (np.zeros((2, 50), np.float32), "a list of 2 label vectors"),
    ([np.zeros(50, np.float32), np.zeros(59, np.float32)], "stream 1: 60 scores but 59 labels"),
    ([np.zeros(50, np.float32), np.zeros(60, np.float64)], "stream 1: labels must be float32, integer or bool"),
])
def test_bad_labels_are_refused_before_any_launch(labels, match, no_launch):
    from mtad_gat_pytorch_b200 import thresholding as th
    with pytest.raises(ValueError, match=match):
        th.replay_streams_eval(_streams([100, 100]), _streams([50, 60]), labels, [{}])


def test_bad_arguments_of_the_model_replay_are_refused_before_scoring(no_launch, monkeypatch):
    from mtad_gat_pytorch_b200 import prediction, scoring

    def refuse(*a, **k):
        raise AssertionError("scored")
    monkeypatch.setattr(scoring, "SeriesScorer", refuse)
    monkeypatch.setattr(prediction, "_model_config", lambda model, what: (None, {"n": 10, "k": 3, "out": 3}))
    x = [np.zeros((110, 3), np.float32), np.zeros((40, 3), np.float32)]
    t = [np.zeros((60, 3), np.float32), np.zeros((70, 3), np.float32)]
    lab = [np.zeros(50, np.float32), np.zeros(60, np.float32)]
    cases = [
        ((x, t[:1], lab), [{}], "2 training series, 1 test series and 2 label vectors"),
        ((x, t, lab[:1]), [{}], "2 training series, 2 test series and 1 label vectors"),
        ((x, [t[0], t[1][:10]], lab), [{}], r"stream 1: x_test must be \(N, 3\) with N > window size 10"),
        ((x, [t[0], t[1][:, :2]], lab), [{}], r"stream 1: x_test must be \(N, 3\)"),
        ((x, t, [lab[0], lab[1][:59]]), [{}], "stream 1: 60 scored test timestamps but 59 labels"),
        ((x, t, lab), [{}, {"depth": 30}], "stream 1: configuration 1: 30 training scores"),
        ((x, t, lab), [{}] * 65536, "stream 0: 1 to 65535 configurations"),
        ((x[0], t, lab), [{}], "must be lists"),
    ]
    for (xs, ts, ls), configs, match in cases:
        with pytest.raises(ValueError, match=match):
            prediction.replay_fleet(None, xs, ts, ls, configs)


def restated_layout(n, m, cfgs, chunk, thresholds):
    """_fleet_layout restated with plain loops: walk w = (stream w // C, configuration w % C)."""
    S, C = len(n), len(cfgs)
    W = S * C
    order = []                                                         # (walk, side) of each block
    for q in dict.fromkeys(cfg[0] for cfg in cfgs):
        walks = [w for w in range(W) if cfgs[w % C][0] == q]
        order += [(w, 0) for w in walks] + [(w, 1) for w in walks if cfgs[w % C][3]]
    B = len(order)
    block = {key: i for i, key in enumerate(order)}
    ks, caps = [], []
    for w, side in order:
        s, (q, level, depth, bi, wa) = w // C, cfgs[w % C]
        ni = n[s] - (depth or 0)
        k = ni - 1 - int((1 - level) * ni) if side else int(level * ni)
        ks.append(k)
        caps.append(ni - k + m[s])
    win, pos = {}, 0
    for d in sorted({cfg[2] for cfg in cfgs if cfg[2]}):
        for w in range(W):
            if cfgs[w % C][2] == d:
                win[w] = pos
                pos += d
    two = any(cfg[3] for cfg in cfgs)
    tab, row, part, soff = [], 0, 0, 0
    for w in range(W):
        s, (q, level, depth, bi, wa) = w // C, cfgs[w % C]
        if w % C == 0 and w:
            soff += m[s - 1]
        rule = {(False, None): 0, (True, None): 2}.get((bi, depth), 3 if bi else 1)
        tab.append([rule, depth or 0, win.get(w, 0), int(wa), block[(w, 0)], block.get((w, 1), B), soff, m[s], row,
                    row if thresholds else part, row if thresholds and two else part])
        row += m[s]                                                    # stream-major: rows follow one another
        part += min(chunk, m[s])
    return np.array(tab, np.int64), np.array(ks, np.int64), np.array(caps, np.int64), row, part, pos


@pytest.mark.parametrize("thresholds", [False, True])
@pytest.mark.parametrize("grid", ["mixed", "one-sided"])
def test_walk_table_and_ragged_offsets(thresholds, grid):
    from mtad_gat_pytorch_b200 import thresholding as th
    n, m, chunk = [40, 17, 25], [30, 5, 12], 8
    configs = [dict(level=0.9), dict(depth=3, q=1e-2), dict(bidirectional=True, level=0.8),
               dict(bidirectional=True, depth=5, with_alarm=False), dict(depth=3, level=0.95, q=1e-2),
               dict(depth=5, q=1e-4)]
    if grid == "one-sided":
        configs = [c for c in configs if not c.get("bidirectional")]
    cfgs = th.replay_configs(configs, min(n))
    plan = th._fleet_layout(n, m, cfgs, chunk, thresholds)
    tab, ks, caps, rows, part, wins = restated_layout(n, m, cfgs, chunk, thresholds)
    assert np.array_equal(plan["tab"], tab)
    assert np.array_equal(plan["ks"], ks) and np.array_equal(plan["caps"], caps)
    C = len(cfgs)
    B = ks.size
    assert np.array_equal(plan["index"], np.concatenate([tab[:, 4], tab[:, 5]]))
    assert plan["alarms"] == rows == C * sum(m) and plan["windows"] == wins
    assert plan["upper"] == (rows if thresholds else part)
    two = grid == "mixed"
    assert plan["lower"] == (rows if thresholds and two else part)
    assert sum(nb for _, _, nb in plan["groups"]) == B
    assert [q for q, _, _ in plan["groups"]] == list(dict.fromkeys(c[0] for c in cfgs))
    for s in range(len(n)):                                            # stream s's C rows: contiguous, ld = m[s]
        r = tab[s * C:(s + 1) * C, 8]
        assert np.array_equal(r, r[0] + m[s] * np.arange(C)) and r[0] == C * sum(m[:s])


def test_the_fleet_replay_kernel_is_built_for_sm_90a():
    import __graft_entry__ as ge
    ge.build()
    nvcc = os.environ.get("NVCC", "/usr/local/cuda/bin/nvcc")
    out = subprocess.run([os.path.join(os.path.dirname(nvcc), "cuobjdump"), "-sass",
                          os.path.join(ge.OBJDIR, "spot_mixed.o")], capture_output=True, text=True, check=True).stdout
    assert "spot_fleet_replay_kernel" in out and "sm_90a" in out
    import mtad_gat_pytorch_b200._lib as L
    assert hasattr(L.lib, "mtadgat_spot_fleet_replay")


def test_the_per_rule_replay_entry_points_are_gone():
    """replay runs as the one-stream case of mtadgat_spot_fleet_replay, so the per-rule replay entry points are not
    exported."""
    import ctypes
    import __graft_entry__ as ge
    ge.build()
    lib = ctypes.CDLL(ge.LIB)
    for name in ("mtadgat_spot_replay", "mtadgat_dspot_replay", "mtadgat_bispot_replay"):
        assert not hasattr(lib, name), name
