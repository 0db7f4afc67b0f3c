"""CPU tests of the POT threshold's oracle: the restatement of spot.py / pot_eval against the reference (when staged),
the device fit rule's model against the scipy Grimshaw on a seeded sweep, the level / k semantics and the check of
the dynamic decomposition on hand-built streams."""
import os
import sys
import types
from math import floor, log

import numpy as np
import pytest

from oracle import pot_oracle as po

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
REF_DIR = os.path.join(ROOT, "baseline", "_ref")


def gpd(rng, xi, scale, m):
    """m float32 generalised-Pareto draws (shape xi, scale), shifted off 0 so that no peak is 0."""
    u = rng.random(m)
    y = scale * (((1 - u) ** (-xi) - 1) / xi if xi != 0 else -np.log(1 - u))
    return y.astype(np.float32) + np.float32(1e-6)


def sweep_cases():
    rng = np.random.default_rng(1)
    for m in (2, 20, 200, 2000):
        for scale in (0.01, 0.05, 1.0):
            for xi in (-0.3, -0.1, 0.0, 0.1, 0.3, 0.6):
                yield xi, scale, m, gpd(rng, xi, scale, m)


def scipy_grimshaw(peaks):
    s = po.SPOT(1e-3)
    s.peaks = peaks
    with np.errstate(all="ignore"):
        return s._grimshaw()


def test_model_ll_at_least_scipy():
    """The device rule's fit never has a lower log-likelihood than the scipy search's (1e-9 relative); where both
    choose the gamma = 0 baseline, the quantiles are equal."""
    worse, baseline_pairs, rels = [], 0, []
    for xi, scale, m, Y in sweep_cases():
        gs, ss, ls = scipy_grimshaw(Y)
        gm, sm, lm, zm, ym = po.grimshaw_model(Y)
        if lm < ls - 1e-9 * abs(ls) and not (gs == 0 and gm == 0):  # both baselines: compared as quantiles below
            worse.append((xi, scale, m, ls, lm))
        s = po.SPOT(1e-3)
        s.init_threshold, s.n, s.Nt = np.float32(0.5), 28479, m
        q_ref = s._quantile(gs, ss)
        q_mod = po.quantile_model(np.float32(0.5), 28479, 1e-3, m, gm, sm, ym)
        if gs == 0 and gm == 0:
            # equal where the means are; the device's mean (double sum, rounded) can be ulps off numpy's float32 one
            baseline_pairs += 1
            if ym == Y.mean():
                assert q_mod == q_ref, (xi, scale, m, q_mod, q_ref)
            else:
                assert abs(q_mod - q_ref) <= 4 * abs(np.spacing(np.float32(q_ref))),(xi, scale, m, q_mod, q_ref)
        rels.append(abs(q_mod - q_ref) / abs(q_ref))
    assert not worse, worse
    assert baseline_pairs > 0
    print(f"max rel quantile difference {max(rels):.1e}, median {np.median(rels):.1e}")


def test_model_edge_cases():
    with pytest.raises(ValueError):
        po.grimshaw_model(np.zeros(0, np.float32))
    with pytest.raises(ValueError):
        po.grimshaw_model(np.full(5, 0.25, np.float32))
    # two peaks: a fit exists and its ll is finite
    g, s, ll, z, ym = po.grimshaw_model(np.array([0.1, 0.3], np.float32))
    assert np.isfinite(ll) and ym == np.float32(0.2)


def test_bounds_follow_numpy_float32():
    """The model's interval ends are spot.py's float32 expressions (mean aside)."""
    rng = np.random.default_rng(3)
    for scale in (1e-3, 1.0, 1e9):
        Y = gpd(rng, 0.2, scale, 100)
        (l, r), Ym, YM, Ymean = po.bounds_f32(Y)
        assert all(np.asarray(v).dtype == np.float32 for v in (*l, *r, Ymean))
        a = -1 / Y.max()
        eps = 1e-8 if abs(a) >= 2e-8 else abs(a) / 10
        a = a + eps
        assert l == (a + eps, -eps) or scale == 1e9
        Ym_ = Y.min()
        assert r == (2 * (Ymean - Ym_) / (Ymean * Ym_), 2 * (Ymean - Ym_) / (Ym_ ** 2))


@pytest.mark.parametrize("level,n", [(0.99, 1000), (1.7, 1000), (0.9999, 28479), (0.5, 7), (2.0, 10)])
def test_level_and_k(level, n):
    """spot.py initialize: level -= floor(level) (1.7 -> 0.7000000000000002, 2.0 -> 0.0), t = sort(init)[int(level *
    n_init)], peaks = init[init > t] - t; the model and the restated SPOT agree on all three."""
    rng = np.random.default_rng(n)
    init = rng.normal(size=n).astype(np.float32)
    k = int((level - floor(level)) * n)
    if level == 1.7:
        assert k == int(0.7000000000000002 * n) == 700
    m = po.pot_model(init, init[:5], q=1e-3, level=level)
    assert m["k"] == k and m["t"] == np.sort(init)[k] and m["Nt0"] == int(np.sum(init > np.sort(init)[k]))
    s = po.SPOT(1e-3)
    s.fit(init, init[:5])
    with np.errstate(all="ignore"):
        s.initialize(level=level)
    assert s.init_threshold == m["t"] and s.Nt == m["Nt0"] and s.n == n


def _stream_case(seed=0, n_init=2000, n=600):
    rng = np.random.default_rng(seed)
    return rng.gamma(2.0, 1.0, n_init).astype(np.float32), rng.gamma(2.0, 1.0, n).astype(np.float32)


def test_dynamic_model_equals_spot_run():
    """Where the premise holds, the parallel decomposition is SPOT.run: every refit fits a prefix of one peak array, and
    the per-point thresholds are those of the refits in order (SPOT.run driven with the model's fit rule)."""
    init, data = _stream_case()
    m = po.pot_model(init, data, q=1e-3, level=0.95, dynamic=True)
    assert m["first_violation"] == -1

    class ModelSPOT(po.SPOT):
        def _grimshaw(self, epsilon=1e-8, n_points=10):
            g, s, ll, z, ym = po.grimshaw_model(self.peaks)
            self._ym = ym
            return g, s, ll

        def _quantile(self, gamma, sigma):
            return po.quantile_model(self.init_threshold, self.n, self.proba, self.Nt, gamma, sigma, self._ym)

    s = ModelSPOT(1e-3)
    s.fit(init, data)
    s.initialize(level=0.95)
    ret = s.run(dynamic=True, with_alarm=False)
    assert np.array_equal(np.asarray(ret["thresholds"], np.float64), m["thresholds"])
    assert len(m["fits"]) == 1 + int(np.sum(data > m["t"]))


def test_dynamic_premise_violation():
    """n q > Nt puts the extreme quantile below t: a point between them is where SPOT.run appends a peak that x > t does
    not see; the model reports the first such index, and the static threshold is unaffected."""
    rng = np.random.default_rng(4)
    init = rng.gamma(2.0, 1.0, 1000).astype(np.float32)
    m0 = po.pot_model(init, init[:10], q=0.05, level=0.99, dynamic=False)
    t, Q = float(m0["t"]), m0["pot_th"]
    assert Q < t
    data = np.array([t - 10.0, t + 1.0, t - 10.0, (t + Q) / 2, t + 2.0, (t + Q) / 2], np.float32)
    m = po.pot_model(init, data, q=0.05, level=0.99, dynamic=True)
    assert m["first_violation"] == 3
    # the premise holds: no point between the quantile and t
    m = po.pot_model(init, data[:3], q=0.05, level=0.99, dynamic=True)
    assert m["first_violation"] == -1
    assert po.pot_model(init, data, q=0.05, level=0.99, dynamic=False)["first_violation"] == -1


def test_dynamic_all_baseline_threshold_is_float32():
    """Scale-1 exponential-like peaks make every fit choose gamma = 0; numpy's mean of float32 thresholds is float32."""
    rng = np.random.default_rng(9)
    init = (rng.exponential(3.0, 400)).astype(np.float32)
    data = (rng.exponential(3.0, 50)).astype(np.float32)
    m = po.pot_model(init, data, q=1e-3, level=0.9, dynamic=True)
    if all(f[0] == 0 for f in m["fits"]):
        assert m["pot_th"] == float(np.float32(m["pot_th"]))


def _load_ref_spot():
    if not os.path.exists(os.path.join(REF_DIR, "spot.py")):
        pytest.skip("reference not present")
    saved = dict(sys.modules)
    for name in ("tqdm", "pandas"):
        try:
            __import__(name)
        except ImportError:
            mod = types.ModuleType(name)
            if name == "tqdm":
                mod.tqdm = lambda it, *a, **k: it
            else:
                mod.Series = type("Series", (), {})
            sys.modules[name] = mod
    sys.path.insert(0, REF_DIR)
    return saved


def _unload_ref(saved):
    sys.path.remove(REF_DIR)
    for name in ("spot", "tqdm", "pandas"):
        if name not in saved:
            sys.modules.pop(name, None)


def test_spot_oracle_equals_reference(capsys):
    """The restated SPOT equals spot.py's: thresholds and every fit's (gamma, sigma, ll), static and dynamic."""
    saved = _load_ref_spot()
    try:
        import spot as ref
        rng = np.random.default_rng(2)
        for n_init, n, level, q in ((500, 120, 0.95, 1e-3), (2000, 200, 0.99, 1e-3), (300, 80, 1.9, 0.01)):
            init = rng.gamma(2.0, 1.0, n_init).astype(np.float32)
            data = rng.gamma(2.0, 1.0, n).astype(np.float32)
            for dynamic in (False, True):
                a, b = po.SPOT(q), ref.SPOT(q)
                with np.errstate(all="ignore"):
                    a.fit(init, data); a.initialize(level=level)
                    b.fit(init, data); b.initialize(level=level, verbose=False)
                    ra, rb = a.run(dynamic=dynamic, with_alarm=False), b.run(dynamic=dynamic, with_alarm=False)
                assert ra["thresholds"] == rb["thresholds"] and ra["alarms"] == rb["alarms"]
                assert a.init_threshold == b.init_threshold and a.Nt == b.Nt and a.n == b.n
                assert np.array_equal(a.peaks, b.peaks)
    finally:
        _unload_ref(saved)
