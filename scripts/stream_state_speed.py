"""Time exporting and importing the live state of a fleet's streams: FleetDetector.state_dict (one launch, one
device-to-host copy) and FleetDetector.import_streams (one host-to-device copy, one launch) against the same record
built from per-stream torch copies.

C2 model (k = 38, n = 100, three forecasting layers, random weights), S = 1, 8, 55 and 256 streams, every stream past
its first window.  SPOT is initialised on synthetic scores whose lengths give each stream between 300 and 10 000 peaks
(log-uniform, level 0.9), so the peaks dominate the record at the large end.  Arms, alternated in one process:
  - export: fleet.state_dict() against, per stream, the ring un-rotated by torch indexing, the last forecast, the state
            words and the peaks each copied to the host (4 copies per stream), then stacked;
  - import: fleet.import_streams(record) against new device tensors filled per stream from the record (ring rows
            scattered to g % n, last forecast, state words re-pointed at a new peak array, peaks: 4 copies per stream).
The imported streams are removed again after each call (not timed).  A timing ends in a device synchronise.  Median and
range over --reps calls after one warm-up, and the library's kernel launches per call (mtadgat_launch_count).  The
torch arm's export is checked to equal the kernel's bit for bit.  Prints the card's name and power limit, read in the
same run, then one JSON line per measurement.
    python scripts/stream_state_speed.py [--reps 20] [--streams 1,8,55,256]"""
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


def timed(fn):
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    fn()
    torch.cuda.synchronize()
    return (time.perf_counter() - t0) * 1e3


def stats(ts):
    return {"median_ms": round(float(np.median(ts)), 3), "min_ms": round(float(np.min(ts)), 3),
            "max_ms": round(float(np.max(ts)), 3)}


def torch_export(fleet):
    """The record's state tensors from per-stream torch copies."""
    from mtad_gat_pytorch_b200.scoring import history_rows
    sc, sp = fleet.scorer, fleet.spots
    hist, last, words, peaks = [], [], [], []
    for s in range(fleet.n_streams):
        rows = int(sc.rows[s])
        h = torch.zeros(sc.n, sc.k)
        pos = history_rows(rows, sc.n)
        h[:pos.size] = sc._hist[s][torch.from_numpy(pos).to(sc.device)].cpu()
        hist.append(h)
        last.append(sc._last_pred[s].cpu() if rows >= sc.n else torch.zeros(sc.out))
        w = sp.state[s].cpu()
        w[5:7] = 0
        words.append(w)
        peaks.append(sp._peaks[s][:int(sp._host[s, 2])].cpu())
    return torch.stack(words), torch.stack(hist), torch.stack(last), torch.cat(peaks)


def torch_import(fleet, rec):
    """The record's streams written into new device tensors with per-stream torch copies (not attached)."""
    from mtad_gat_pytorch_b200.scoring import history_rows
    sc, dev = fleet.scorer, fleet.scorer.device
    B = rec["rows"].numel()
    hist = torch.zeros(B, sc.n, sc.k, device=dev)
    last = torch.empty(B, sc.out, device=dev)
    words = torch.empty(B, 24, dtype=torch.int64, device=dev)
    off = rec["peak_offsets"].tolist()
    peaks = []
    for b in range(B):
        rows = int(rec["rows"][b])
        pos = history_rows(rows, sc.n)
        hist[b][torch.from_numpy(pos).to(dev)] = rec["hist"][b][:pos.size].to(dev)
        last[b] = rec["last_pred"][b].to(dev)
        p = torch.empty(max(2 * (off[b + 1] - off[b]), 16), device=dev)
        w = rec["spot"][b].clone()
        w[5], w[6] = p.data_ptr(), p.numel()
        words[b] = w.to(dev)
        p[:off[b + 1] - off[b]] = rec["peaks"][off[b]:off[b + 1]].to(dev)
        peaks.append(p)
    return hist, last, words, peaks


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=20)
    ap.add_argument("--streams", default="1,8,55,256")
    args = ap.parse_args()
    assert torch.cuda.is_available(), "stream_state_speed.py measures on a GPU"
    import mtad_gat_pytorch_b200 as mg
    from mtad_gat_pytorch_b200 import prediction
    from mtad_gat_pytorch_b200 import thresholding as th
    print(f"[stream_state_speed] card: {card()}", flush=True)

    torch.manual_seed(0)
    k, n = 38, 100
    model = mg.MTAD_GAT(n_features=k, window_size=n, out_dim=k, forecast_n_layers=3, dropout=0.3).cuda().eval()
    rng = np.random.default_rng(0)

    for S in (int(v) for v in args.streams.split(",")):
        fleet = prediction.FleetDetector(model, [torch.from_numpy(rng.random((n + 200, k)).astype(np.float32))
                                                 for _ in range(S)], level=0.9)
        want = np.exp(rng.uniform(np.log(300), np.log(10000), S)).astype(np.int64)
        scores = [torch.from_numpy(rng.pareto(3.0, 10 * int(m)).astype(np.float32)).cuda() for m in want]
        fleet.spots = th.SpotStreams(scores, q=1e-3, level=0.9)
        fleet.train_scores = scores
        extra = rng.integers(1, 40, S)
        fleet.push(torch.from_numpy(rng.random((int(S * n + extra.sum()), k)).astype(np.float32)),
                   np.repeat(np.arange(S), n + extra))
        rec = fleet.state_dict()
        ref = torch_export(fleet)
        same = all(torch.equal(a.view(torch.int32) if a.dtype == torch.float32 else a,
                               b.view(torch.int32) if b.dtype == torch.float32 else b)
                   for a, b in zip(ref, (rec["spot"], rec["hist"], rec["last_pred"], rec["peaks"])))
        nbytes = sum(t.numel() * t.element_size() for t in rec.values() if isinstance(t, torch.Tensor))

        def drop():
            fleet.remove_streams(list(range(S, fleet.n_streams)))
        arms = {"export": (lambda: fleet.state_dict(), lambda: torch_export(fleet), None),
                "import": (lambda: fleet.import_streams(rec), lambda: torch_import(fleet, rec), drop)}
        for what, (kernel, separate, undo) in arms.items():
            t_k, t_s, launches = [], [], {}
            for rep in range(args.reps + 1):
                for name, fn, ts in (("kernel", kernel, t_k), ("torch", separate, t_s)):
                    mg.reset_launch_count()
                    t = timed(fn)
                    launches[name] = mg.launch_count()
                    if undo is not None and fleet.n_streams > S:
                        undo()
                    if rep:                                             # the first call of each arm is a warm-up
                        ts.append(t)
            a, b = stats(t_k), stats(t_s)
            print(json.dumps({"what": what, "model": "C2", "streams": S, "peaks_total": int(rec["peaks"].numel()),
                              "peaks_min": int(np.diff(rec["peak_offsets"].numpy()).min()),
                              "peaks_max": int(np.diff(rec["peak_offsets"].numpy()).max()),
                              "record_mb": round(nbytes / 2 ** 20, 2), "kernel": a, "torch_per_stream": b,
                              "speedup": round(b["median_ms"] / a["median_ms"], 2),
                              "launches_kernel": launches["kernel"], "bitwise_equal_export": same,
                              "calls": args.reps}), flush=True)
        del fleet
        torch.cuda.empty_cache()


if __name__ == "__main__":
    main()
