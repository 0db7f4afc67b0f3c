"""Host restatement of streaming biSPOT / bidSPOT (thresholding.SpotStream(s) with bidirectional=True,
csrc/bispot.cu): `BiSpotModel` is spot.py's biSPOT (bidSPOT with a depth) initialize + run with an injectable fit,
float32 peaks and `level` / `1 - level`.  With spot.py's scipy fit it equals the restated spot.py
(tests/bispot_reference.py); with the device's fit rule (`device_fit`) it is what the GPU tests compare the device
against.  Also: the negation identities the device's lower side rests on, two-sided stream state records and the
argument checks."""
import copy
import os
import sys
import types
from math import floor, log

import numpy as np
import pytest
import torch

from oracle import pot_oracle as po
from tests import bispot_reference as br
from tests import dspot_reference as dr
from tests.test_stream_cpu import device_fit, gpd
from tests.test_stream_state_cpu import EXPECT, _record

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
REF_DIR = os.path.join(ROOT, "baseline", "_ref")


def bi_scipy_fit(peaks, t, n, q):
    """spot.py's biSPOT._grimshaw (scipy's L-BFGS-B, n_points = 8) and the upper _quantile at t."""
    g, s, _ = br._side_grimshaw(peaks)
    sp = po.SPOT(q)
    sp.init_threshold, sp.n, sp.Nt = t, n, peaks.size
    return sp._quantile(g, s)


class BiSpotModel:
    """spot.py biSPOT.initialize + run(with_alarm) (bidSPOT's with a depth), statement for statement, with the levels
    `level` and `1 - level`, continued over any number of `run` calls.  fit(peaks, t, n, q) is the upper side's
    quantile; the lower side's is -fit(its peaks, -t_down, n, q), which is spot.py's lower formula exactly.  `joins`
    records (index, side) of every new peak."""

    def __init__(self, q=1e-3, fit=device_fit, depth=None):
        self.q, self.fit, self.depth = q, fit, depth
        self.joins, self.seen = [], 0

    def _refit(self, side):
        if side == 0:
            self.Q[0] = self.fit(self.peaks[0], self.t[0], self.n, self.q)
        else:
            self.Q[1] = -self.fit(self.peaks[1], -self.t[1], self.n, self.q)

    def initialize(self, init, level=0.98):
        init = np.asarray(init, np.float32)
        level = level - floor(level)
        X = init
        if self.depth is not None:
            d = self.depth
            X = init[d:] - dr.backMean(init, d)[:-1]
            self.W = init[-d:]
        self.T = X
        n = X.size
        S = np.sort(X)
        self.t = [S[int(level * n)], S[int((1 - level) * n)]]
        self.peaks = [X[X > self.t[0]] - self.t[0], -(X[X < self.t[1]] - self.t[1])]
        self.n = n
        self.Q = [None, None]
        self._refit(0)
        self._refit(1)
        return self

    @property
    def Nt(self):
        return [p.size for p in self.peaks]

    def _join(self, side, r, i):
        self.peaks[side] = np.append(self.peaks[side], r - self.t[0] if side == 0 else -(r - self.t[1]))
        self.n += 1
        self._refit(side)
        self.joins.append((i, side))

    def run(self, data, with_alarm=True):
        up, low, codes = [], [], []
        for x in np.asarray(data, np.float32):
            i = self.seen
            self.seen += 1
            Mi = self.W.mean() if self.depth is not None else None
            r = x - Mi if Mi is not None else x
            code = 0
            if r > self.Q[0]:
                if with_alarm:
                    code = 1
                else:
                    self._join(0, r, i)
            elif r > self.t[0]:
                self._join(0, r, i)
            elif r < self.Q[1]:
                if with_alarm:
                    code = 2
                else:
                    self._join(1, r, i)
            elif r < self.t[1]:
                self._join(1, r, i)
            else:
                self.n += 1
            if self.depth is not None and not code:
                self.W = np.append(self.W[1:], x)
            codes.append(code)
            up.append(self.Q[0] + Mi if Mi is not None else self.Q[0])
            low.append(self.Q[1] + Mi if Mi is not None else self.Q[1])
        return {"upper": np.array(up, np.float64), "lower": np.array(low, np.float64),
                "codes": np.array(codes, np.uint8)}


def bi_case(seed, n_init=500, n=90, depth=None, drift=0.0, level=0.95):
    """Training scores and a stream with two heavy tails (a ramp under them with a depth) that take every branch on
    both sides: alarm runs above and below, an alarm followed by a peak, and points between t and Q on each side."""
    rng = np.random.default_rng(seed)
    ramp = np.linspace(0, drift, n_init + n).astype(np.float32)
    init = (gpd(rng, n_init) - gpd(rng, n_init) + ramp[:n_init]).astype(np.float32)
    data = (gpd(rng, n) - gpd(rng, n) + ramp[n_init:]).astype(np.float32)
    m = BiSpotModel(depth=depth).initialize(init, level)
    tu, Qu, td, Qd = (float(v) for v in (m.t[0], m.Q[0], m.t[1], m.Q[1]))
    W = list(init[-depth:]) if depth else []
    for j in range(n):
        Mi = np.float32(np.mean(np.array(W[-depth:], np.float32))) if depth else np.float32(0)
        alarm = j in (10, 11, 40, 50, 51, 70)
        if j in (10, 11, 40):
            data[j] = Mi + np.float32(Qu + (Qu - tu) * (1 + j % 3))
        elif j in (12, 41):
            data[j] = Mi + np.float32((tu + Qu) / 2)
        elif j in (50, 51, 70):
            data[j] = Mi + np.float32(Qd - (td - Qd) * (1 + j % 3))
        elif j in (52, 71, 72):
            data[j] = Mi + np.float32((td + Qd) / 2)
        if depth and not alarm:
            W.append(data[j])
    return init, data


def _reference(depth, level, q=1e-3):
    return br.biSPOT(q, level) if depth is None else br.bidSPOT(q, depth, level)


@pytest.mark.parametrize("with_alarm", [True, False])
@pytest.mark.parametrize("depth", [None, 10])
@pytest.mark.parametrize("seed", [0, 1])
def test_bispot_model_is_bispot_run(seed, depth, with_alarm):
    """BiSpotModel with spot.py's scipy fit gives spot.py's biSPOT / bidSPOT run, threshold for threshold on both
    sides and alarm for alarm."""
    init, data = bi_case(seed, depth=depth, drift=2.0 if depth else 0.0, level=0.98)
    ref = _reference(depth, 0.98)
    ref.fit(init, data)
    ref.initialize()
    m = BiSpotModel(1e-3, fit=bi_scipy_fit, depth=depth).initialize(init, 0.98)
    assert m.t[0] == ref.init_threshold["up"] and m.t[1] == ref.init_threshold["down"]
    assert m.Nt == [ref.Nt["up"], ref.Nt["down"]] and m.n == ref.n
    assert m.Q[0] == ref.extreme_quantile["up"] and m.Q[1] == ref.extreme_quantile["down"]
    want = ref.run(with_alarm=with_alarm)
    got = m.run(data, with_alarm)
    assert np.nonzero(got["codes"])[0].tolist() == want["alarms"]
    assert np.array_equal(got["upper"], np.array(want["upper_thresholds"], np.float64))
    assert np.array_equal(got["lower"], np.array(want["lower_thresholds"], np.float64))
    sides = {s for _, s in m.joins}
    assert sides == {0, 1}
    if with_alarm:
        assert {1, 2} <= set(got["codes"].tolist())


@pytest.mark.parametrize("depth", [None, 7])
def test_bispot_model_chunks(depth):
    """run() continued over chunks is run() over the whole stream."""
    init, data = bi_case(5, depth=depth)
    whole = BiSpotModel(depth=depth).initialize(init, 0.95).run(data)
    m = BiSpotModel(depth=depth).initialize(init, 0.95)
    parts = [m.run(data[i:i + 7]) for i in range(0, data.size, 7)]
    for key in ("upper", "lower", "codes"):
        assert np.array_equal(np.concatenate([p[key] for p in parts]), whole[key])


def test_oracle_bispot_is_the_staged_reference():
    """When the reference is staged, the restated biSPOT and bidSPOT are its own, output for output (at its levels)."""
    if not os.path.exists(os.path.join(REF_DIR, "spot.py")):
        pytest.skip("reference not present")
    saved = dict(sys.modules)
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
        for depth in (None, 10):
            init, data = bi_case(2, depth=depth, level=0.98)
            for with_alarm in (True, False):
                ref = ref_spot.biSPOT(1e-3) if depth is None else ref_spot.bidSPOT(1e-3, depth=depth)
                ref.fit(init, data)
                ref.initialize(verbose=False)
                want = ref.run(with_alarm=with_alarm, plot=False) if depth is not None else \
                    ref.run(with_alarm=with_alarm)
                orc = _reference(depth, 0.98)
                orc.fit(init, data)
                orc.initialize()
                got = orc.run(with_alarm=with_alarm)
                assert got["alarms"] == want["alarms"]
                assert np.array_equal(got["upper_thresholds"], want["upper_thresholds"])
                assert np.array_equal(got["lower_thresholds"], want["lower_thresholds"])
    finally:
        sys.path.remove(REF_DIR)
        for name in list(sys.modules):
            if name not in saved:
                sys.modules.pop(name, None)


# ---------------------------------------------------------------------------------------------------------------------
# the negation identities of the lower side (csrc/bispot.cu)

def test_negation_identities():
    rng = np.random.default_rng(0)
    x = (rng.standard_normal(20000) * np.exp(rng.uniform(-20, 20, 20000))).astype(np.float32)
    t = (rng.standard_normal(20000) * np.exp(rng.uniform(-20, 20, 20000))).astype(np.float32)
    # (-x) - (-t) == -(x - t), bit for bit
    assert np.array_equal((-x - -t).view(np.int32), (-(x - t)).view(np.int32))
    # x < Q  <=>  -x > -Q for a float32 x and a float64 Q
    Q = x.astype(np.float64) + rng.standard_normal(x.size) * np.abs(x) * 1e-7
    Q[::7] = x[::7]
    assert np.array_equal(x < Q, -x > -Q)
    # the lower quantile is minus the upper formula at -t_down: the float64 branch and the float32 gamma = 0 branch
    sigma, gamma = rng.uniform(0.01, 3, x.size), rng.uniform(-0.5, 0.5, x.size)
    r = rng.uniform(1e-4, 0.5, x.size)
    for i in range(0, x.size, 97):
        td, s, g, ri = t[i], sigma[i], gamma[i], r[i]
        low = td - (s / g) * (pow(ri, -g) - 1)
        up = -td + (s / g) * (pow(ri, -g) - 1)
        assert np.float64(low).view(np.int64) == np.float64(-up).view(np.int64)
        s32 = np.float32(s)
        lr = log(float(ri))                                           # spot.py: math.log, a Python float
        low0, up0 = td + s32 * lr, -td - s32 * lr
        assert low0.dtype == np.float32 and up0.dtype == np.float32
        assert low0.view(np.int32) == (-up0).view(np.int32)
    # t_down = S[k] is -(sorted(-x)[n - 1 - k]) (up to the sign of a zero)
    for n in (1, 2, 7, 100, 1001):
        v = x[:n]
        k = int((1 - 0.98) * n)
        assert np.sort(v)[k] == -np.sort(-v)[n - 1 - k]


def test_bispot_model_lower_side_is_spot_on_negated_scores():
    """The lower side of BiSpotModel with the device fit is SPOT's upper side on -x: the peaks, t and quantile."""
    init, _ = bi_case(3)
    m = BiSpotModel().initialize(init, 0.95)
    neg = -np.asarray(init, np.float32)
    n = neg.size
    t_lo = np.sort(neg)[n - 1 - int((1 - 0.95) * n)]
    assert t_lo == -m.t[1]
    assert np.array_equal(neg[neg > t_lo] - t_lo, m.peaks[1])
    q = device_fit(neg[neg > t_lo] - t_lo, t_lo, n, 1e-3)
    assert np.float64(-q).view(np.int64) == np.float64(m.Q[1]).view(np.int64)


# ---------------------------------------------------------------------------------------------------------------------
# two-sided stream state records

def _bi_record(B=3, seed=1):
    rec = _record(B)
    rng = np.random.default_rng(seed)
    nt = rng.integers(0, 9, B)
    low = torch.from_numpy(rng.integers(0, 1 << 40, (B, 24)).astype(np.int64))
    low[:, 2] = torch.from_numpy(nt)
    low[:, 1] = rec["spot"][:, 1]
    rec.update(bidirectional=True, spot_lower=low,
               peak_offsets_lower=torch.from_numpy(np.concatenate([[0], np.cumsum(nt)]).astype(np.int64)),
               peaks_lower=torch.from_numpy(rng.random(int(nt.sum())).astype(np.float32)))
    return rec


def _check(rec, expect):
    from mtad_gat_pytorch_b200 import prediction
    return prediction.check_state_record(rec, expect, lambda: "abc", "import")


def test_two_sided_and_one_sided_records():
    got = _check(_bi_record(), dict(EXPECT, bidirectional=True))
    assert got["bidirectional"] and got["spot_lower"].shape == (3, 24)
    assert np.array_equal(got["peak_offsets_lower"], _bi_record()["peak_offsets_lower"].numpy())
    assert not _check(_record(), dict(EXPECT, bidirectional=False))["bidirectional"]
    with pytest.raises(ValueError, match="^import: a two-sided record does not enter a one-sided detector"):
        _check(_bi_record(), dict(EXPECT, bidirectional=False))
    with pytest.raises(ValueError, match="^import: a one-sided record does not enter a two-sided detector"):
        _check(_record(), dict(EXPECT, bidirectional=True))


@pytest.mark.parametrize("case", ["lower Nt", "lower N", "offsets", "offsets short", "peaks dtype", "spot shape",
                                  "missing peaks", "not two-sided", "bidirectional False"])
def test_bad_two_sided_records_are_refused(case):
    rec = copy.deepcopy(_bi_record())
    if case == "lower Nt":
        rec["spot_lower"][1, 2] += 1
    elif case == "lower N":
        rec["spot_lower"][2, 1] += 1
    elif case == "offsets":
        rec["peak_offsets_lower"][1] = rec["peak_offsets_lower"][2] + 1
    elif case == "offsets short":
        rec["peak_offsets_lower"] = rec["peak_offsets_lower"][:-1]
    elif case == "peaks dtype":
        rec["peaks_lower"] = rec["peaks_lower"].double()
    elif case == "spot shape":
        rec["spot_lower"] = rec["spot_lower"][:, :-1]
    elif case == "missing peaks":
        rec.pop("peaks_lower")
    elif case == "not two-sided":
        rec.pop("bidirectional")
    else:
        rec["bidirectional"] = False
    with pytest.raises(ValueError, match="^import: "):
        _check(rec, dict(EXPECT, bidirectional=True))


# ---------------------------------------------------------------------------------------------------------------------
# argument checks (before anything touches the device)

def test_level_argument():
    from mtad_gat_pytorch_b200 import thresholding as th
    assert th.check_level(0.98, True, "x") == 0.98 and th.check_level(1.25, False, "x") == 0.25
    for bad in (0.5, 0.3, 1.5, 2.0):
        with pytest.raises(ValueError, match="^x: a two-sided stream needs level > 0.5"):
            th.check_level(bad, True, "x")
    with pytest.raises(ValueError, match="^SpotStream: a two-sided stream needs level > 0.5"):
        th.SpotStream(torch.zeros(10), level=0.5, bidirectional=True)
    with pytest.raises(ValueError, match="^SpotStreams: a two-sided stream needs level > 0.5"):
        th.SpotStreams([torch.zeros(10)], level=0.4, bidirectional=True)
    with pytest.raises(ValueError, match="^SpotStream: depth"):
        th.SpotStream(torch.zeros(10), depth=0, bidirectional=True)
    with pytest.raises(ValueError, match="^SpotStreams: depth"):
        th.SpotStreams([torch.zeros(10)], depth=4097, bidirectional=True)


def test_detector_arguments():
    from mtad_gat_pytorch_b200 import prediction
    model = types.SimpleNamespace(temporal_gat=types.SimpleNamespace(window_size=5))
    x = torch.zeros(16, 3)
    with pytest.raises(ValueError, match="^StreamDetector: a two-sided stream needs level > 0.5"):
        prediction.StreamDetector(model, x, level=0.2, bidirectional=True)
    with pytest.raises(ValueError, match="^StreamDetector: 16 rows give 11 training scores; dSPOT with depth 11"):
        prediction.StreamDetector(model, x, depth=11, bidirectional=True)
    with pytest.raises(ValueError, match="^FleetDetector: a two-sided stream needs level > 0.5"):
        prediction.FleetDetector(model, [x], level=0.5, bidirectional=True)
    with pytest.raises(ValueError, match="^FleetDetector: depth"):
        prediction.FleetDetector(model, [x], depth=0, bidirectional=True)
