"""Time replays (thresholding.replay_eval: C configurations of the live detectors over one recorded series, side by side)
against the one-at-a-time route: C thresholding.SpotStream constructions and whole-series pushes, each followed by the
host evaluation (the restated eval_methods.py adjust_predicts(pred=alarms) + calc_point2point, oracle/).

1. SMD-sized: 28 479 training and 28 479 test scores, C = 1, 16 and 128 configurations.
2. SMAP-sized test length: 135 183 training and 427 617 test scores, replays of C = 1, 128 and 256 (the one-at-a-time
   route for C = 1 only), and the peak device memory of each replay.
3. The restated spot.py SPOT.run (oracle/pot_oracle.py, scipy's fit) on the host for two SMD-sized configurations.
The configurations cycle through SPOT, dSPOT (depths 16 and 129), biSPOT and bidSPOT (depth 16), levels 0.99, 0.995
and 0.999 (the reference's SMD range) with q = 1e-3 and both with_alarm.  The scores are synthetic: gamma-distributed
with a slow ramp and planted bursts, labels over the bursts.  A timing ends in a device synchronise (the replay reads
back anyway).  Prints the card's name and power limit, read in the same run, then one JSON line per measurement.
    python scripts/replay_speed.py [--smd 1,16,128] [--smap 1,128,256]"""
import argparse
import json
import os
import sys
import time

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from scripts.eval_speed import card  # noqa: E402
from scripts.fleet_speed import timed  # noqa: E402

RULES = [dict(), dict(depth=16), dict(depth=129), dict(bidirectional=True), dict(bidirectional=True, depth=16)]
LEVELS = (0.99, 0.995, 0.999)


def configs(C):
    return [dict(RULES[c % len(RULES)], q=1e-3, level=LEVELS[(c // len(RULES)) % len(LEVELS)],
                 with_alarm=bool((c // (len(RULES) * len(LEVELS))) % 2 == 0)) for c in range(C)]


def series(rng, n_init, m):
    x = (rng.gamma(2.0, 1.0, n_init + m) + np.linspace(0, 1, n_init + m)).astype(np.float32)
    lab = np.zeros(m, np.float32)
    for s in rng.integers(0, m - 200, max(m // 4000, 3)):
        x[n_init + s:n_init + s + 50] += 8.0
        lab[s:s + 100] = 1
    return x[:n_init], x[n_init:], lab


def one_at_a_time(th, ev, tr, s, lab, cfgs):
    out = []
    for cfg in cfgs:
        sp = th.SpotStream(tr, cfg["q"], cfg["level"], cfg["with_alarm"], depth=cfg.get("depth"),
                           bidirectional=cfg.get("bidirectional", False))
        alarms = sp.push(s)[-1].cpu().numpy() != 0
        p, lat = ev.adjust_predicts(None, lab, 0.0, pred=alarms, calc_latency=True)
        out.append(ev.calc_point2point(p, lab)[0])
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--smd", default="1,16,128")
    ap.add_argument("--smap", default="1,128,256")
    args = ap.parse_args()
    assert torch.cuda.is_available(), "replay_speed.py measures on a GPU"
    from mtad_gat_pytorch_b200 import thresholding as th
    from oracle import evaluation_oracle as ev
    from oracle import pot_oracle as po
    print(card(), flush=True)
    rng = np.random.default_rng(0)
    for name, (n_init, m), Cs, base in (("SMD", (28479, 28479), args.smd, True),
                                        ("SMAP", (135183, 427617), args.smap, False)):
        init, data, lab = series(rng, n_init, m)
        tr, s = torch.from_numpy(init).cuda(), torch.from_numpy(data).cuda()
        th.replay_eval(tr, s[:5000], lab[:5000], configs(5))                   # warm-up
        for C in (int(c) for c in Cs.split(",") if c):
            cfgs = configs(C)
            torch.cuda.synchronize()
            torch.cuda.reset_peak_memory_stats()
            before = torch.cuda.memory_allocated()
            res = []
            t_rep = timed(lambda: res.append(th.replay_eval(tr, s, lab, cfgs)))
            peak = torch.cuda.max_memory_allocated() - before
            rec = {"what": "replay_eval", "series": name, "n_init": n_init, "m": m, "C": C,
                   "replay_ms": round(t_rep, 1), "peak_mib": round(peak / 2 ** 20, 1),
                   "refits": int(sum(r["refits"] for r in res[0])), "alarms": int(sum(r["alarms"] for r in res[0])),
                   "flagged": int(sum(r["flags"] != 0 for r in res[0]))}
            if base or C == 1:
                t0 = time.perf_counter()
                f1 = one_at_a_time(th, ev, tr, s, lab, cfgs)
                torch.cuda.synchronize()
                t_one = (time.perf_counter() - t0) * 1e3
                assert f1 == [r["f1"] for r in res[0]]
                rec.update(one_at_a_time_ms=round(t_one, 1), speedup=round(t_one / t_rep, 1))
            print(json.dumps(rec), flush=True)
    # the restated spot.py on the host, SMD-sized
    init, data, lab = series(np.random.default_rng(1), 28479, 28479)
    for level in (0.99, 0.995):
        sp = po.SPOT(1e-3)
        sp.fit(init, data)
        sp.initialize(level=level)
        t0 = time.perf_counter()
        r = sp.run(with_alarm=True, dynamic=True)
        host_ms = (time.perf_counter() - t0) * 1e3
        dev = th.replay_eval(torch.from_numpy(init).cuda(), torch.from_numpy(data).cuda(), lab,
                             [dict(level=level, q=1e-3)])[0]
        print(json.dumps({"what": "spot.py SPOT.run on the host", "level": level, "points": data.size,
                          "host_run_ms": round(host_ms, 1), "alarms_host": len(r["alarms"]),
                          "alarms_device": dev["alarms"]}), flush=True)


if __name__ == "__main__":
    main()
