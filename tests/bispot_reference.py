"""spot.py's biSPOT and bidSPOT (two-sided SPOT, and two-sided SPOT with drift: fit, initialize, _grimshaw, _quantile,
run), restated statement for statement, scipy's L-BFGS-B included (printing, tqdm, plotting and the pandas / list input
forms are left out).  Test infrastructure only: the reference for csrc/bispot.cu and thresholding.SpotStream(s) with
bidirectional=True.  spot.py fixes the levels at 0.98 and 0.02; here they are `level` and `1 - level` (level = 0.98 is
spot.py's).  The per-side fit is spot.py's biSPOT._grimshaw: SPOT's search on that side's peaks with biSPOT's own
defaults (n_points = 8), on oracle/pot_oracle.py's restated _rootsFinder and _log_likelihood."""
from math import log

import numpy as np

from oracle.pot_oracle import SPOT
from tests.dspot_reference import backMean


def _side_grimshaw(peaks, epsilon=1e-8, n_points=8):
    """biSPOT._grimshaw(side): SPOT._grimshaw's statements on the side's peaks, with biSPOT's defaults."""
    sp = SPOT()
    sp.peaks = peaks
    g, s, ll = sp._grimshaw(epsilon, n_points)
    return g, s, ll


class biSPOT:
    def __init__(self, q=1e-4, level=0.98):
        self.proba = q
        self.level = level
        self.data = None
        self.init_data = None
        self.n = 0
        self.extreme_quantile = {"up": None, "down": None}
        self.init_threshold = {"up": None, "down": None}
        self.peaks = {"up": None, "down": None}
        self.Nt = {"up": 0, "down": 0}

    def fit(self, init_data, data):
        self.data = np.asarray(data)
        self.init_data = np.asarray(init_data)

    def _init_on(self, X):
        n_init = X.size
        S = np.sort(X)
        self.init_threshold["up"] = S[int(self.level * n_init)]
        self.init_threshold["down"] = S[int((1 - self.level) * n_init)]
        self.peaks["up"] = X[X > self.init_threshold["up"]] - self.init_threshold["up"]
        self.peaks["down"] = -(X[X < self.init_threshold["down"]] - self.init_threshold["down"])
        self.Nt["up"] = self.peaks["up"].size
        self.Nt["down"] = self.peaks["down"].size
        self.n = n_init
        for side in ["up", "down"]:
            g, s, l = self._grimshaw(side)
            self.extreme_quantile[side] = self._quantile(side, g, s)

    def initialize(self):
        self._init_on(self.init_data)

    def _grimshaw(self, side):
        return _side_grimshaw(self.peaks[side])

    def _quantile(self, side, gamma, sigma):
        if side == "up":
            r = self.n * self.proba / self.Nt[side]
            if gamma != 0:
                return self.init_threshold["up"] + (sigma / gamma) * (pow(r, -gamma) - 1)
            else:
                return self.init_threshold["up"] - sigma * log(r)
        elif side == "down":
            r = self.n * self.proba / self.Nt[side]
            if gamma != 0:
                return self.init_threshold["down"] - (sigma / gamma) * (pow(r, -gamma) - 1)
            else:
                return self.init_threshold["down"] + sigma * log(r)

    def _peak(self, side, value):
        self.peaks[side] = np.append(self.peaks[side], value)
        self.Nt[side] += 1
        self.n += 1
        g, s, l = self._grimshaw(side)
        self.extreme_quantile[side] = self._quantile(side, g, s)

    def run(self, with_alarm=True):
        thup, thdown, alarm = [], [], []
        for i in range(self.data.size):
            x = self.data[i]
            if x > self.extreme_quantile["up"]:
                if with_alarm:
                    alarm.append(i)
                else:
                    self._peak("up", x - self.init_threshold["up"])
            elif x > self.init_threshold["up"]:
                self._peak("up", x - self.init_threshold["up"])
            elif x < self.extreme_quantile["down"]:
                if with_alarm:
                    alarm.append(i)
                else:
                    self._peak("down", -(x - self.init_threshold["down"]))
            elif x < self.init_threshold["down"]:
                self._peak("down", -(x - self.init_threshold["down"]))
            else:
                self.n += 1
            thup.append(self.extreme_quantile["up"])
            thdown.append(self.extreme_quantile["down"])
        return {"upper_thresholds": thup, "lower_thresholds": thdown, "alarms": alarm}


class bidSPOT(biSPOT):
    def __init__(self, q=1e-4, depth=10, level=0.98):
        super().__init__(q, level)
        self.depth = depth

    def initialize(self):
        M = backMean(self.init_data, self.depth)
        T = self.init_data[self.depth:] - M[:-1]
        self._init_on(T)

    def run(self, with_alarm=True):
        W = self.init_data[-self.depth:]
        thup, thdown, alarm = [], [], []
        for i in range(self.data.size):
            Mi = W.mean()
            Ni = self.data[i] - Mi
            if Ni > self.extreme_quantile["up"]:
                if with_alarm:
                    alarm.append(i)
                else:
                    self._peak("up", Ni - self.init_threshold["up"])
                    W = np.append(W[1:], self.data[i])
            elif Ni > self.init_threshold["up"]:
                self._peak("up", Ni - self.init_threshold["up"])
                W = np.append(W[1:], self.data[i])
            elif Ni < self.extreme_quantile["down"]:
                if with_alarm:
                    alarm.append(i)
                else:
                    self._peak("down", -(Ni - self.init_threshold["down"]))
                    W = np.append(W[1:], self.data[i])
            elif Ni < self.init_threshold["down"]:
                self._peak("down", -(Ni - self.init_threshold["down"]))
                W = np.append(W[1:], self.data[i])
            else:
                self.n += 1
                W = np.append(W[1:], self.data[i])
            thup.append(self.extreme_quantile["up"] + Mi)
            thdown.append(self.extreme_quantile["down"] + Mi)
        return {"upper_thresholds": thup, "lower_thresholds": thdown, "alarms": alarm}
