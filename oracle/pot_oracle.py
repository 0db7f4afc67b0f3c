"""CPU restatement of the reference's POT threshold -- TEST INFRASTRUCTURE, NOT PRODUCT CODE.

- `SPOT` / `pot_eval` restate spot.py's SPOT (fit, initialize, _rootsFinder, _log_likelihood, _grimshaw, _quantile,
  run) and eval_methods.py pot_eval statement for statement, scipy's L-BFGS-B included (printing, tqdm and the pandas /
  list input forms are left out).  `SPOT.fits` records (gamma, sigma, ll) of every Grimshaw fit.
- `grimshaw_model` / `pot_model` are a float64 numpy model of the device's fit rule (csrc/pot.cu, DESIGN §1): the same
  float32 bounds, w at 353 nodes per interval, 60 bisection steps per sign change, the maximum-likelihood candidate
  among the roots and each interval's outermost nodes where w is finite (its ends, unless 1 + zY <= 0 there).
  Sums are numpy's (pairwise), the device's are thread-strided then a fixed tree: the two agree to rounding."""
from math import floor, log

import numpy as np

NODES = 352
BISECT = 60


# ---------------------------------------------------------------------------------------------------------------------
# spot.py / eval_methods.py, restated

class SPOT:
    def __init__(self, q=1e-4):
        self.proba = q
        self.extreme_quantile = None
        self.data = None
        self.init_data = None
        self.init_threshold = None
        self.peaks = None
        self.n = 0
        self.Nt = 0
        self.fits = []

    def fit(self, init_data, data):
        self.data = np.asarray(data)
        self.init_data = np.asarray(init_data)

    def initialize(self, level=0.98, min_extrema=False):
        if min_extrema:
            self.init_data = -self.init_data
            self.data = -self.data
            level = 1 - level
        level = level - floor(level)
        n_init = self.init_data.size
        S = np.sort(self.init_data)
        self.init_threshold = S[int(level * n_init)]
        self.peaks = self.init_data[self.init_data > self.init_threshold] - self.init_threshold
        self.Nt = self.peaks.size
        self.n = n_init
        g, s, l = self._grimshaw()
        self.extreme_quantile = self._quantile(g, s)

    @staticmethod
    def _rootsFinder(fun, jac, bounds, npoints, method):
        from scipy.optimize import minimize
        if method == "regular":
            step = (bounds[1] - bounds[0]) / (npoints + 1)
            X0 = np.arange(bounds[0] + step, bounds[1], step)
        elif method == "random":
            X0 = np.random.uniform(bounds[0], bounds[1], npoints)

        def objFun(X, f, jac):
            g = 0
            j = np.zeros(X.shape)
            i = 0
            for x in X:
                fx = f(x)
                g = g + fx ** 2
                j[i] = 2 * fx * jac(x)
                i = i + 1
            return g, j

        opt = minimize(lambda X: objFun(X, fun, jac), X0, method="L-BFGS-B", jac=True, bounds=[bounds] * len(X0))
        X = opt.x
        np.round(X, decimals=5)
        return np.unique(X)

    @staticmethod
    def _log_likelihood(Y, gamma, sigma):
        n = Y.size
        if gamma != 0:
            tau = gamma / sigma
            L = -n * log(sigma) - (1 + (1 / gamma)) * (np.log(1 + tau * Y)).sum()
        else:
            L = n * (1 + log(Y.mean()))
        return L

    def _grimshaw(self, epsilon=1e-8, n_points=10):
        def u(s):
            return 1 + np.log(s).mean()

        def v(s):
            return np.mean(1 / s)

        def w(Y, t):
            s = 1 + t * Y
            us = u(s)
            vs = v(s)
            return us * vs - 1

        def jac_w(Y, t):
            s = 1 + t * Y
            us = u(s)
            vs = v(s)
            jac_us = (1 / t) * (1 - vs)
            jac_vs = (1 / t) * (-vs + np.mean(1 / s ** 2))
            return us * jac_vs + vs * jac_us

        Ym = self.peaks.min()
        YM = self.peaks.max()
        Ymean = self.peaks.mean()
        a = -1 / YM
        if abs(a) < 2 * epsilon:
            epsilon = abs(a) / n_points
        a = a + epsilon
        b = 2 * (Ymean - Ym) / (Ymean * Ym)
        c = 2 * (Ymean - Ym) / (Ym ** 2)
        left_zeros = SPOT._rootsFinder(lambda t: w(self.peaks, t), lambda t: jac_w(self.peaks, t),
                                       (a + epsilon, -epsilon), n_points, "regular")
        right_zeros = SPOT._rootsFinder(lambda t: w(self.peaks, t), lambda t: jac_w(self.peaks, t), (b, c), n_points,
                                        "regular")
        zeros = np.concatenate((left_zeros, right_zeros))
        gamma_best = 0
        sigma_best = Ymean
        ll_best = SPOT._log_likelihood(self.peaks, gamma_best, sigma_best)
        for z in zeros:
            gamma = u(1 + z * self.peaks) - 1
            sigma = gamma / z
            ll = SPOT._log_likelihood(self.peaks, gamma, sigma)
            if ll > ll_best:
                gamma_best = gamma
                sigma_best = sigma
                ll_best = ll
        self.fits.append((gamma_best, sigma_best, ll_best))
        return gamma_best, sigma_best, ll_best

    def _quantile(self, gamma, sigma):
        r = self.n * self.proba / self.Nt
        if gamma != 0:
            return self.init_threshold + (sigma / gamma) * (pow(r, -gamma) - 1)
        else:
            return self.init_threshold - sigma * log(r)

    def run(self, with_alarm=True, dynamic=True):
        if self.n > self.init_data.size:
            return {}
        th = []
        alarm = []
        for i in range(self.data.size):
            if not dynamic:
                if self.data[i] > self.init_threshold and with_alarm:
                    self.extreme_quantile = self.init_threshold
                    alarm.append(i)
            else:
                if self.data[i] > self.extreme_quantile:
                    if with_alarm:
                        alarm.append(i)
                    else:
                        self.peaks = np.append(self.peaks, self.data[i] - self.init_threshold)
                        self.Nt += 1
                        self.n += 1
                        g, s, l = self._grimshaw()
                        self.extreme_quantile = self._quantile(g, s)
                elif self.data[i] > self.init_threshold:
                    self.peaks = np.append(self.peaks, self.data[i] - self.init_threshold)
                    self.Nt += 1
                    self.n += 1
                    g, s, l = self._grimshaw()
                    self.extreme_quantile = self._quantile(g, s)
                else:
                    self.n += 1
            th.append(self.extreme_quantile)
        return {"thresholds": th, "alarms": alarm}


def pot_eval(init_score, score, label, q=1e-3, level=0.99, dynamic=False):
    """eval_methods.py pot_eval; the tail (adjust_predicts + calc_point2point) is evaluation_oracle.threshold_eval's.
    Returns (the reference's dict, the SPOT object)."""
    from oracle.evaluation_oracle import threshold_eval
    s = SPOT(q)
    s.fit(init_score, score)
    s.initialize(level=level, min_extrema=False)
    ret = s.run(dynamic=dynamic, with_alarm=False)
    pot_th = np.mean(ret["thresholds"])
    if label is not None:
        return threshold_eval(score, label, pot_th), s
    return {"threshold": pot_th}, s


# ---------------------------------------------------------------------------------------------------------------------
# the device's fit rule

def bounds_f32(peaks):
    """spot.py _grimshaw's two search intervals, with Ymean the float64 sum / Nt rounded to float32 (the device's)."""
    peaks = np.asarray(peaks, np.float32)
    Ym, YM = peaks.min(), peaks.max()
    Ymean = np.float32(np.sum(peaks, dtype=np.float64) / peaks.size)
    a = np.float32(-1) / YM
    eps = np.float32(1e-8)
    if abs(a) < np.float32(2e-8):
        eps = abs(a) / np.float32(10)
    a = a + eps
    d = np.float32(2) * (Ymean - Ym)
    return ((a + eps, -eps), (d / (Ymean * Ym), d / (Ym * Ym))), Ym, YM, Ymean


def _w(Y, x):
    """w(x) = u v - 1 as L + V + L V (L = mean log1p(xY), V = -mean(xY / (1 + xY))); x may be a vector."""
    ty = np.multiply.outer(np.atleast_1d(x), Y)
    L = np.sum(np.log1p(ty), axis=-1) / Y.size
    V = -np.sum(ty / (1.0 + ty), axis=-1) / Y.size
    return L + V + L * V


def _candidate(Y, z, ll0):
    gamma = np.sum(np.log1p(z * Y)) / Y.size
    sigma = gamma / z
    if gamma == 0:
        return gamma, sigma, ll0
    tau = gamma / sigma
    return gamma, sigma, -Y.size * np.log(sigma) - (1.0 + 1.0 / gamma) * np.sum(np.log1p(tau * Y))


def grimshaw_model(peaks):
    """The device's Grimshaw fit of float32 `peaks` -> (gamma, sigma, ll, z, Ymean); z = 0 for the baseline.
    Raises ValueError for no peaks or all peaks equal (where spot.py raises)."""
    peaks = np.asarray(peaks, np.float32)
    if peaks.size == 0:
        raise ValueError("no peaks")
    ivs, Ym, YM, Ymean = bounds_f32(peaks)
    if Ym == YM:
        raise ValueError("all peaks equal")
    Y = peaks.astype(np.float64)
    ll0 = Y.size * (1 + log(float(Ymean)))
    best = (0.0, float(Ymean), ll0, 0.0)
    with np.errstate(all="ignore"):
        for lo, hi in ivs:
            lo, hi = float(lo), float(hi)
            j = np.arange(NODES + 1, dtype=np.float64)
            x = lo + (hi - lo) * j / NODES
            x[0], x[-1] = lo, hi
            w = _w(Y, x)
            fin = np.flatnonzero(np.isfinite(w))
            ends = (x[fin[0]], x[fin[-1]]) if fin.size else (lo, hi)   # outermost nodes where w is defined
            cands = [ends[0]]
            for i in range(NODES):
                if np.isfinite(w[i]) and np.isfinite(w[i + 1]) and (w[i] < 0) != (w[i + 1] < 0):
                    a, b, neg = x[i], x[i + 1], w[i] < 0
                    for _ in range(BISECT):
                        m = 0.5 * (a + b)
                        if (_w(Y, m)[0] < 0) == neg:
                            a = m
                        else:
                            b = m
                    cands.append(0.5 * (a + b))
            cands.append(ends[1])
            for z in cands:
                g, s, ll = _candidate(Y, z, ll0)
                if ll > best[2]:
                    best = (g, s, ll, z)
    return best + (Ymean,)


def quantile_model(t, n, q, Nt, gamma, sigma, Ymean):
    """spot.py _quantile with numpy 2's types: the gamma = 0 branch is float32 arithmetic on the float32 Ymean."""
    r = n * q / Nt
    if gamma != 0:
        return float(t) + (sigma / gamma) * (pow(r, -gamma) - 1)
    return float(np.float32(t) - np.float32(Ymean) * np.float32(log(r)))


def pot_model(init, data, q=1e-3, level=0.99, dynamic=False):
    """The device's pot_eval threshold.  Returns a dict: t, k, Nt0, fits [(gamma, sigma, ll, z, quantile)], thresholds
    (per test point, float64), pot_th, first_violation (-1 if none)."""
    init, data = np.asarray(init, np.float32), np.asarray(data, np.float32)
    level = level - floor(level)
    k = int(level * init.size)
    t = np.sort(init)[k]
    P0 = init[init > t] - t
    g, s, ll, z, ym = grimshaw_model(P0)
    fits = [(g, s, ll, z, quantile_model(t, init.size, q, P0.size, g, s, ym))]
    n = data.size
    if not dynamic:
        thr = np.full(n, fits[0][4])
        return {"t": t, "k": k, "Nt0": P0.size, "fits": fits, "thresholds": thr, "pot_th": fits[0][4],
                "first_violation": -1}
    exc = data > t
    idx = np.flatnonzero(exc)
    P = np.concatenate([P0, data[idx] - t])
    for m, i in enumerate(idx, 1):
        g, s, ll, z, ym = grimshaw_model(P[:P0.size + m])
        fits.append((g, s, ll, z, quantile_model(t, init.size + i + 1, q, P0.size + m, g, s, ym)))
    Q = np.array([f[4] for f in fits])
    thr = Q[np.cumsum(exc)]
    bad = np.flatnonzero(~exc & (data.astype(np.float64) > thr))
    pot_th = thr.mean()
    if all(f[0] == 0 for f in fits):
        pot_th = float(np.float32(pot_th))
    return {"t": t, "k": k, "Nt0": P0.size, "fits": fits, "thresholds": thr, "pot_th": pot_th,
            "first_violation": int(bad[0]) if bad.size else -1}
