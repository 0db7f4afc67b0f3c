"""spot.py's backMean and dSPOT (SPOT with drift: fit, initialize, run), restated statement for statement, scipy's
L-BFGS-B included (printing, tqdm and the pandas / list input forms are left out).  Test infrastructure only: the
reference for csrc/dspot.cu and thresholding.SpotStream(s) with a depth.  dSPOT's _rootsFinder, _log_likelihood,
_grimshaw and _quantile are SPOT's, statement for statement, so they come from oracle/pot_oracle.py's restated SPOT."""
import numpy as np

from oracle.pot_oracle import SPOT


def backMean(X, d):
    M = []
    w = X[:d].sum()
    M.append(w / d)
    for i in range(d, len(X)):
        w = w - X[i - d] + X[i]
        M.append(w / d)
    return np.array(M)


class dSPOT(SPOT):
    def __init__(self, q=1e-4, depth=10):
        super().__init__(q)
        self.depth = depth

    def fit(self, init_data, data):
        self.data = np.asarray(data)
        self.init_data = np.asarray(init_data)

    def initialize(self):
        n_init = self.init_data.size - self.depth
        M = backMean(self.init_data, self.depth)
        T = self.init_data[self.depth:] - M[:-1]
        S = np.sort(T)
        self.init_threshold = S[int(0.98 * n_init)]
        self.peaks = T[T > self.init_threshold] - self.init_threshold
        self.Nt = self.peaks.size
        self.n = n_init
        g, s, l = self._grimshaw()
        self.extreme_quantile = self._quantile(g, s)

    def run(self, with_alarm=True):
        if self.n > self.init_data.size:
            return {}
        W = self.init_data[-self.depth:]
        th = []
        alarm = []
        for i in range(self.data.size):
            Mi = W.mean()
            if (self.data[i] - Mi) > self.extreme_quantile:
                if with_alarm:
                    alarm.append(i)
                else:
                    self.peaks = np.append(self.peaks, self.data[i] - Mi - self.init_threshold)
                    self.Nt += 1
                    self.n += 1
                    g, s, l = self._grimshaw()
                    self.extreme_quantile = self._quantile(g, s)
                    W = np.append(W[1:], self.data[i])
            elif (self.data[i] - Mi) > self.init_threshold:
                self.peaks = np.append(self.peaks, self.data[i] - Mi - self.init_threshold)
                self.Nt += 1
                self.n += 1
                g, s, l = self._grimshaw()
                self.extreme_quantile = self._quantile(g, s)
                W = np.append(W[1:], self.data[i])
            else:
                self.n += 1
                W = np.append(W[1:], self.data[i])
            th.append(self.extreme_quantile + Mi)
        return {"thresholds": th, "alarms": alarm}
