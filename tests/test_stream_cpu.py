"""Host restatement of the streaming SPOT update (thresholding.SpotStream, csrc/spot_stream.cu): `SpotModel` is spot.py's
SPOT.initialize + SPOT.run(dynamic=True) with an injectable fit and float32 peaks.  With the scipy fit it equals the
restated spot.py (oracle/pot_oracle.py SPOT.run); with the device's fit rule (`device_fit`) it is what the GPU tests
compare the device against."""
from math import floor

import numpy as np
import pytest

from oracle import pot_oracle as po


def device_fit(peaks, t, n, q):
    """The device's Grimshaw fit and quantile, typed as spot.py's: np.float64, or np.float32 for the gamma = 0 baseline."""
    g, s, _, _, ym = po.grimshaw_model(peaks)
    v = po.quantile_model(t, n, q, peaks.size, g, s, ym)
    return np.float64(v) if g != 0 else np.float32(v)


def scipy_fit(peaks, t, n, q):
    """spot.py's own _grimshaw (scipy's L-BFGS-B) and _quantile."""
    sp = po.SPOT(q)
    sp.peaks, sp.init_threshold, sp.n, sp.Nt = peaks, t, n, peaks.size
    g, s, _ = sp._grimshaw()
    return sp._quantile(g, s)


class SpotModel:
    """spot.py SPOT.initialize(level) + SPOT.run(with_alarm, dynamic=True), statement for statement, continued over any
    number of `run` calls; `joins` records the stream indices that became peaks."""

    def __init__(self, q=1e-3, fit=device_fit):
        self.q, self.fit = q, fit
        self.joins, self.seen = [], 0

    def initialize(self, init, level=0.99):
        init = np.asarray(init, np.float32)
        level = level - floor(level)
        self.t = np.sort(init)[int(level * init.size)]
        self.peaks = init[init > self.t] - self.t
        self.Nt, self.n = self.peaks.size, init.size
        self.quantile = self.fit(self.peaks, self.t, self.n, self.q)
        return self

    def _join(self, x, i):
        self.peaks = np.append(self.peaks, x - self.t)                  # float32 - float32: a float32 peak
        self.Nt += 1
        self.n += 1
        self.quantile = self.fit(self.peaks, self.t, self.n, self.q)
        self.joins.append(i)

    def run(self, data, with_alarm=True):
        th, alarm = [], []
        for x in np.asarray(data, np.float32):
            i = self.seen
            self.seen += 1
            if x > self.quantile:
                if with_alarm:
                    alarm.append(i)
                else:
                    self._join(x, i)
            elif x > self.t:
                self._join(x, i)
            else:
                self.n += 1
            th.append(self.quantile)
        return {"thresholds": np.array(th, np.float64), "alarms": alarm}


def gpd(rng, m, xi=0.25, scale=0.05):
    """Generalised-Pareto scores: heavy-tailed, so the fits choose a gamma != 0 candidate."""
    return (scale * ((1 - rng.random(m)) ** -xi - 1) / xi).astype(np.float32)


def alarm_case(seed, n_init=400, n=80):
    """Training scores and a stream with alarm runs, one alarm immediately followed by a peak (t < x <= quantile), and
    points between t and the quantile."""
    rng = np.random.default_rng(seed)
    init, data = gpd(rng, n_init), gpd(rng, n)
    m = SpotModel(fit=device_fit).initialize(init, 0.95)
    t, Q = float(m.t), float(m.quantile)
    data[10:14] = Q * np.array([1.5, 2.0, 1.2, 3.0], np.float32)          # an alarm run
    data[14] = (t + Q) / 2                                               # ... immediately followed by a peak
    data[40] = Q * 4                                                     # a single alarm
    data[41:43] = (t + Q) / 2
    return init, data


@pytest.mark.parametrize("with_alarm", [True, False])
@pytest.mark.parametrize("seed", [0, 1])
def test_spot_model_is_spot_run(seed, with_alarm):
    """SpotModel with spot.py's scipy fit gives spot.py's run, threshold for threshold and alarm for alarm."""
    init, data = alarm_case(seed)
    ref = po.SPOT(1e-3)
    ref.fit(init, data)
    ref.initialize(level=0.95)
    want = ref.run(with_alarm=with_alarm, dynamic=True)
    got = SpotModel(1e-3, fit=scipy_fit).initialize(init, 0.95).run(data, with_alarm)
    assert got["alarms"] == want["alarms"]
    assert np.array_equal(got["thresholds"], np.array(want["thresholds"], np.float64))
    if with_alarm:
        assert len(want["alarms"]) >= 3


def test_spot_model_continues_pot_model():
    """With the device's fit and no alarms, SpotModel gives pot_model's dynamic thresholds where pot_model's premise
    holds, and runs on where it does not."""
    rng = np.random.default_rng(3)
    init, data = gpd(rng, 1500), gpd(rng, 300)
    pm = po.pot_model(init, data, q=1e-3, level=0.95, dynamic=True)
    assert pm["first_violation"] == -1
    sm = SpotModel(1e-3).initialize(init, 0.95)
    assert sm.t == pm["t"] and sm.Nt == pm["Nt0"]
    assert np.array_equal(sm.run(data, with_alarm=False)["thresholds"], pm["thresholds"])

    # test_gpu_pot's "test point 3" stream: the quantile is below t, so a point at or below t joins the peaks
    init = np.random.default_rng(4).gamma(2.0, 1.0, 1000).astype(np.float32)
    st = po.pot_model(init, init[:10], q=0.05, level=0.99)
    t, Q = float(st["t"]), st["pot_th"]
    data = np.array([t - 10.0, t + 1.0, t - 10.0, (t + Q) / 2, t + 2.0, (t + Q) / 2], np.float32)
    assert po.pot_model(init, data, q=0.05, level=0.99, dynamic=True)["first_violation"] == 3
    sm = SpotModel(0.05).initialize(init, 0.99)
    r = sm.run(data, with_alarm=False)
    assert sm.joins[:3] == [1, 3, 4] and np.all(np.isfinite(r["thresholds"]))


def test_spot_model_chunks():
    """run() continued over chunks is run() over the whole stream."""
    init, data = alarm_case(5)
    whole = SpotModel().initialize(init, 0.95).run(data)
    m = SpotModel().initialize(init, 0.95)
    parts = [m.run(data[i:i + 7]) for i in range(0, data.size, 7)]
    assert np.array_equal(np.concatenate([p["thresholds"] for p in parts]), whole["thresholds"])
    assert sum((p["alarms"] for p in parts), []) == whole["alarms"]
