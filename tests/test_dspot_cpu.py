"""Host restatement of streaming dSPOT (thresholding.SpotStream with a depth, csrc/dspot.cu): `DSpotModel` is spot.py's
backMean + dSPOT.initialize + dSPOT.run with an injectable fit, float32 residuals and peaks, and SPOT's `level`.  With
the scipy fit it equals the restated spot.py (tests/dspot_reference.py dSPOT.run); with the device's fit rule
(`device_fit`) it is what the GPU tests compare the device against.  Also: the device's order of numpy's pairwise sum
(leaves, then the recursion over their sums, on the window as a ring) against numpy, and the validation of dSPOT and
SPOT stream state records."""
import copy
import os
import sys
from math import floor

import numpy as np
import pytest
import torch

from tests import dspot_reference as dr
from tests.test_stream_cpu import device_fit, gpd, scipy_fit
from tests.test_stream_state_cpu import EXPECT, _record

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
REF_DIR = os.path.join(ROOT, "baseline", "_ref")
DEPTHS = [1, 7, 8, 9, 128, 129, 300]


# ---------------------------------------------------------------------------------------------------------------------
# numpy's pairwise sum in the device's order

def pw_leaves(n, c0=0):
    """The leaves (start, length) of numpy's pairwise sum of n values, left to right: blocks of at most 128, split at
    the first half rounded down to a multiple of 8."""
    if n <= 128:
        return [(c0, n)]
    h = n // 2 - (n // 2) % 8
    return pw_leaves(h, c0) + pw_leaves(n - h, c0 + h)


def pw_leaf(v):
    """One leaf: a plain float32 loop below 8 values, else 8 accumulators, their fixed tree, then the tail."""
    v = np.asarray(v, np.float32)
    n = v.size
    if n < 8:
        res = np.float32(0)
        for x in v:
            res = np.float32(res + x)
        return res
    r = v[:8].copy()
    i = 8
    while i < n - n % 8:
        r = (r + v[i:i + 8]).astype(np.float32)
        i += 8
    res = np.float32((r[0] + r[1]) + (r[2] + r[3])) + np.float32((r[4] + r[5]) + (r[6] + r[7]))
    res = np.float32(res)
    for x in v[i:]:
        res = np.float32(res + x)
    return res


def pw_combine(n, sums, c0=0):
    """The recursion over precomputed leaf sums (sums: leaf start -> its sum)."""
    if n <= 128:
        return sums[c0]
    h = n // 2 - (n // 2) % 8
    return np.float32(pw_combine(h, sums, c0) + pw_combine(n - h, sums, c0 + h))


def device_sum(ring, head):
    """np.sum of the window W = ring[head:] + ring[:head] (oldest first) as csrc/spot_walk.cuh adds it: each leaf of
    W's pairwise sum on its own, then the recursion over the leaf sums, then added to +0.0."""
    d = ring.size
    at = lambda c: ring[(head + c) % d]                                  # noqa: E731
    sums = {c0: pw_leaf([at(c0 + i) for i in range(n)]) for c0, n in pw_leaves(d)}
    return np.float32(np.float32(0) + pw_combine(d, sums))


def back_mean_model(X, d):
    """csrc/dspot.cu's backMean: the first sum in pairwise order, then one float32 subtraction and addition per step."""
    X = np.asarray(X, np.float32)
    w = device_sum(X[:d], 0)
    M = [np.float32(w / np.float32(d))]
    for i in range(d, X.size):
        w = np.float32(np.float32(w - X[i - d]) + X[i])
        M.append(np.float32(w / np.float32(d)))
    return np.array(M, np.float32)


@pytest.mark.parametrize("d", DEPTHS)
def test_back_mean_and_window_mean_equal_numpy(d):
    rng = np.random.default_rng(d)
    X = (rng.standard_normal(2 * d + 257) * 3 + 10).astype(np.float32)
    want = dr.backMean(X, d)
    assert want.dtype == np.float32
    assert np.array_equal(back_mean_model(X, d).view(np.int32), want.view(np.int32))
    assert X[:d].sum() == device_sum(X[:d], 0)
    for head in sorted({0, 1, d // 2, d - 1}):
        ring = X[d:2 * d].copy()
        W = np.concatenate([ring[head:], ring[:head]])
        got = np.float32(device_sum(ring, head) / np.float32(d))
        assert got.view(np.int32) == W.mean().view(np.int32) and W.mean().dtype == np.float32, head


def test_leaves_cover_the_window():
    for d in DEPTHS + [4096, 4095, 1000]:
        leaves = pw_leaves(d)
        assert sum(n for _, n in leaves) == d and all(c0 % 8 == 0 for c0, _ in leaves)
        assert len(leaves) <= max(1, 4096 // 64) and (d <= 128 or min(n for _, n in leaves) >= 64)


# ---------------------------------------------------------------------------------------------------------------------
# dSPOT, restated with an injectable fit

class DSpotModel:
    """spot.py backMean + dSPOT.initialize + dSPOT.run(with_alarm), statement for statement, with t at `level` as
    SPOT.initialize takes it (spot.py's dSPOT is level = 0.98), continued over any number of `run` calls.  `joins`
    records the stream indices that became peaks; `T` holds the training residuals, `W` the window (oldest first)."""

    def __init__(self, depth, q=1e-3, fit=device_fit):
        self.depth, self.q, self.fit = depth, q, fit
        self.joins, self.seen = [], 0

    def initialize(self, init, level=0.98):
        init = np.asarray(init, np.float32)
        level = level - floor(level)
        d = self.depth
        n_init = init.size - d
        M = dr.backMean(init, d)
        self.T = init[d:] - M[:-1]
        self.t = np.sort(self.T)[int(level * n_init)]
        self.peaks = self.T[self.T > self.t] - self.t
        self.Nt, self.n = self.peaks.size, n_init
        self.quantile = self.fit(self.peaks, self.t, self.n, self.q)
        self.W = init[-d:]
        return self

    def _join(self, r, i):
        self.peaks = np.append(self.peaks, r - self.t)                  # (x - Mi) - t: a float32 peak
        self.Nt += 1
        self.n += 1
        self.quantile = self.fit(self.peaks, self.t, self.n, self.q)
        self.joins.append(i)

    def run(self, data, with_alarm=True):
        th, alarm = [], []
        for x in np.asarray(data, np.float32):
            i = self.seen
            self.seen += 1
            Mi = self.W.mean()
            r = x - Mi
            if r > self.quantile:
                if with_alarm:
                    alarm.append(i)
                else:
                    self._join(r, i)
                    self.W = np.append(self.W[1:], x)
            elif r > self.t:
                self._join(r, i)
                self.W = np.append(self.W[1:], x)
            else:
                self.n += 1
                self.W = np.append(self.W[1:], x)
            th.append(self.quantile + Mi)
        return {"thresholds": np.array(th, np.float64), "alarms": alarm}


def drift_case(seed, n_init=500, n=90, drift=2.0, d=10):
    """Training scores and a stream on a rising baseline (heavy-tailed noise on a ramp), with alarm runs, an alarm
    immediately followed by a peak, and points between t and the quantile above the moving mean."""
    rng = np.random.default_rng(seed)
    ramp = np.linspace(0, drift, n_init + n).astype(np.float32)
    init = (gpd(rng, n_init) + ramp[:n_init]).astype(np.float32)
    data = (gpd(rng, n) + ramp[n_init:]).astype(np.float32)
    m = DSpotModel(d).initialize(init)
    W = list(init[-d:])
    for j in range(n):                                                  # the window as the stream would see it
        Mi = np.float32(np.mean(np.array(W[-d:], np.float32)))
        if j in (20, 21, 22, 60):
            data[j] = Mi + np.float32(m.quantile) * np.float32(1.5 + j % 3)
        elif j in (23, 61, 62):
            data[j] = Mi + np.float32((float(m.t) + float(m.quantile)) / 2)
        if j not in (20, 21, 22, 60):
            W.append(data[j])
    return init, data, d


@pytest.mark.parametrize("with_alarm", [True, False])
@pytest.mark.parametrize("seed", [0, 1])
def test_dspot_model_is_dspot_run(seed, with_alarm):
    """DSpotModel with spot.py's scipy fit gives spot.py's dSPOT run, threshold for threshold and alarm for alarm."""
    init, data, d = drift_case(seed)
    ref = dr.dSPOT(1e-3, depth=d)
    ref.fit(init, data)
    ref.initialize()
    m = DSpotModel(d, 1e-3, fit=scipy_fit).initialize(init, 0.98)
    assert m.t == ref.init_threshold and m.Nt == ref.Nt and m.n == ref.n and m.quantile == ref.extreme_quantile
    want = ref.run(with_alarm=with_alarm)
    got = m.run(data, with_alarm)
    assert got["alarms"] == want["alarms"]
    assert np.array_equal(got["thresholds"], np.array(want["thresholds"], np.float64))
    assert len(m.joins) >= 3
    if with_alarm:
        assert len(want["alarms"]) >= 3


def test_dspot_model_chunks():
    """run() continued over chunks is run() over the whole stream."""
    init, data, d = drift_case(5)
    whole = DSpotModel(d).initialize(init, 0.95).run(data)
    m = DSpotModel(d).initialize(init, 0.95)
    parts = [m.run(data[i:i + 7]) for i in range(0, data.size, 7)]
    assert np.array_equal(np.concatenate([p["thresholds"] for p in parts]), whole["thresholds"])
    assert sum((p["alarms"] for p in parts), []) == whole["alarms"]


def test_oracle_dspot_is_the_staged_reference():
    """When the reference is staged, the oracle's backMean and dSPOT are its own, output for output."""
    if not os.path.exists(os.path.join(REF_DIR, "spot.py")):
        pytest.skip("reference not present")
    saved = dict(sys.modules)
    import types
    stubs = {}
    for name in ("tqdm", "matplotlib", "matplotlib.pyplot", "pandas"):
        try:
            __import__(name)
        except ImportError:
            stubs[name] = types.ModuleType(name)
    if "tqdm" in stubs:
        stubs["tqdm"].tqdm = lambda x, *a, **k: x
    sys.modules.update(stubs)
    sys.path.insert(0, REF_DIR)
    try:
        import spot as ref_spot
        for d in DEPTHS[:5]:
            X = np.random.default_rng(d).random(d + 50).astype(np.float32)
            assert np.array_equal(ref_spot.backMean(X, d), dr.backMean(X, d))
        init, data, d = drift_case(2)
        for with_alarm in (True, False):
            ref = ref_spot.dSPOT(1e-3, depth=d)
            ref.fit(init, data)
            ref.initialize(verbose=False)
            want = ref.run(with_alarm=with_alarm)
            orc = dr.dSPOT(1e-3, depth=d)
            orc.fit(init, data)
            orc.initialize()
            got = orc.run(with_alarm=with_alarm)
            assert got["alarms"] == want["alarms"] and np.array_equal(got["thresholds"], want["thresholds"])
    finally:
        sys.path.remove(REF_DIR)
        for name in list(sys.modules):
            if name not in saved:
                sys.modules.pop(name, None)


# ---------------------------------------------------------------------------------------------------------------------
# stream state records

def _drift_record(B=3, depth=5):
    rec = _record(B)
    rec["depth"] = depth
    rec["window"] = torch.from_numpy(np.random.default_rng(1).random((B, depth)).astype(np.float32))
    return rec


def _check(rec, expect):
    from mtad_gat_pytorch_b200 import prediction
    return prediction.check_state_record(rec, expect, lambda: "abc", "import")


def test_drift_and_spot_records():
    got = _check(_drift_record(), dict(EXPECT, depth=5))
    assert got["depth"] == 5 and got["window"].shape == (3, 5)
    assert _check(_drift_record(), {"n": 6})["depth"] == 5             # depth left out of expect: only type-checked
    got = _check(_record(), dict(EXPECT, depth=None))
    assert got["depth"] is None and got["window"] is None
    with pytest.raises(ValueError, match="^import: a dSPOT record .* SPOT detector"):
        _check(_drift_record(), dict(EXPECT, depth=None))
    with pytest.raises(ValueError, match="^import: a SPOT record .* dSPOT detector"):
        _check(_record(), dict(EXPECT, depth=5))
    with pytest.raises(ValueError, match="^import: the record's depth 5 does not match the detector's 6"):
        _check(_drift_record(), dict(EXPECT, depth=6))


@pytest.mark.parametrize("case", ["no window", "window shape", "window dtype", "window numpy", "depth 0",
                                  "depth too large", "depth float", "depth bool", "window without depth"])
def test_bad_drift_records_are_refused(case):
    rec = copy.deepcopy(_drift_record())
    if case == "no window":
        rec.pop("window")
    elif case == "window shape":
        rec["window"] = rec["window"][:, :-1]
    elif case == "window dtype":
        rec["window"] = rec["window"].double()
    elif case == "window numpy":
        rec["window"] = rec["window"].numpy()
    elif case == "depth 0":
        rec["depth"] = 0
    elif case == "depth too large":
        rec["depth"] = 4097
    elif case == "depth float":
        rec["depth"] = 5.0
    elif case == "depth bool":
        rec["depth"] = True
    else:
        rec.pop("depth")
    with pytest.raises(ValueError, match="^import: "):
        _check(rec, EXPECT)


def test_depth_arguments():
    from mtad_gat_pytorch_b200 import thresholding as th
    assert th.check_depth(None, "x") is None and th.check_depth(np.int64(7), "x") == 7
    assert th.check_depth(th.DSPOT_MAX_DEPTH, "x") == 4096
    for bad in (0, -1, 4097, 2.0, True, "8"):
        with pytest.raises(ValueError, match="^x: depth"):
            th.check_depth(bad, "x")
