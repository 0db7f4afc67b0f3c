"""Timeline of one CUDA-graph replay of the C2 training step (CUPTI activity records via torch.profiler).

Writes every kernel / memset / memcpy of the last replay (start offset, duration, stream, name) to a csv next to the
trace and prints: the span, the all-idle time (no kernel, memset or memcpy running on any stream), per-stream busy
time, the 20 largest same-stream gaps with the kernels on either side, and every memset / memcpy event.

usage: timeline.py [gru_split] [trace.json] [pipelines]"""
import sys, os, json
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import torch
import mtad_gat_pytorch_b200 as mg
from mtad_gat_pytorch_b200 import training as mgt
from torch.profiler import profile, ProfilerActivity
split = int(sys.argv[1]) if len(sys.argv) > 1 else 0
if split: mg.set_gru_split(split)
pipes = int(sys.argv[3]) if len(sys.argv) > 3 else 1
B = 256
torch.manual_seed(0)
m = mg.MTAD_GAT(38, 100, 38, forecast_n_layers=3, dropout=0.3).cuda().train()
opt = mgt.FusedAdam(m.parameters(), lr=1e-3)        # the optimizer bench.py times
step = mgt.TrainStep(m, opt, batch=B, use_graph=True, world_size=1, pipeline=pipes)
x = torch.rand(B, 100, 38, device="cuda"); y = torch.rand(B, 1, 38, device="cuda")
for _ in range(5): step.run_device(x, y)
torch.cuda.synchronize()
with profile(activities=[ProfilerActivity.CUDA, ProfilerActivity.CPU]) as prof:
    for _ in range(3):
        step.run_device(x, y)
        torch.cuda.synchronize()
out = sys.argv[2] if len(sys.argv) > 2 else "gpurun_out/timeline.json"
os.makedirs(os.path.dirname(os.path.abspath(out)), exist_ok=True)
prof.export_chrome_trace(out)
trace = json.load(open(out))["traceEvents"]
os.remove(out)
# the device records of the last graph replay share the correlation id of its cudaGraphLaunch
launches = sorted((e for e in trace if e.get("cat") == "cuda_runtime" and e.get("name", "").startswith("cudaGraphLaunch")),
                  key=lambda e: e["ts"])
corr = launches[-1]["args"]["correlation"]
GPU_CATS = ("kernel", "gpu_memset", "gpu_memcpy")
last = sorted((e for e in trace if e.get("cat") in GPU_CATS and e.get("args", {}).get("correlation") == corr),
              key=lambda e: e["ts"])
if not last:            # a trace without per-launch correlation: everything on the device after the last launch call
    last = sorted((e for e in trace if e.get("cat") in GPU_CATS and e["ts"] >= launches[-1]["ts"]), key=lambda e: e["ts"])
t0 = last[0]["ts"]


def kind(e):
    # the driver runs some graph memset / memcpy nodes as kernels of its own (memset32, memcpy32_post, ...)
    if e["cat"] == "kernel" and e["name"].startswith(("memset", "memcpy")):
        return "gpu_memcpy" if e["name"].startswith("memcpy") else "gpu_memset"
    return e["cat"]


rows = [(e["ts"] - t0, e["dur"], e["args"].get("stream"), kind(e), e["name"][:90]) for e in last]
with open(out.replace(".json", ".csv"), "w") as f:
    f.write("start_us,dur_us,stream,cat,name\n")
    for r in rows: f.write("%.1f,%.1f,%s,%s,%s\n" % r)
end = max(r[0] + r[1] for r in rows)
# all-idle = span minus the union of every record's interval
busy, cur_s, cur_e = 0.0, None, None
for s, d, *_ in sorted(rows):
    if cur_e is None or s > cur_e:
        if cur_e is not None: busy += cur_e - cur_s
        cur_s, cur_e = s, s + d
    else:
        cur_e = max(cur_e, s + d)
busy += cur_e - cur_s
copies = [r for r in rows if r[3] != "kernel"]
main = rows[0][2]               # the capture stream: the step's first node runs there
main_copy_us = sum(r[1] for r in copies if r[2] == main)
print("records", len(rows), "kernels", len(rows) - len(copies), "memset_memcpy", len(copies), "span_us", round(end, 1),
      "all_idle_us", round(end - busy, 1))
print("main stream", main, "memset_memcpy_us", round(main_copy_us, 1), "all_idle + main memset_memcpy us",
      round(end - busy + main_copy_us, 1))
bys = {}
for r in rows: bys.setdefault(r[2], []).append(r)
gaps = []
for s, rs in sorted(bys.items(), key=lambda kv: -len(kv[1])):
    cp = [r for r in rs if r[3] != "kernel"]
    print("stream", s, "n", len(rs), "busy_us", round(sum(r[1] for r in rs), 1), "memset_memcpy_us",
          round(sum(r[1] for r in cp), 1), "first", round(rs[0][0], 1), "last_end", round(max(r[0] + r[1] for r in rs), 1))
    for a, b in zip(rs, rs[1:]):
        gaps.append((b[0] - (a[0] + a[1]), s, a[4], b[4]))
print("largest same-stream gaps (us, stream, before -> after):")
for g, s, a, b in sorted(gaps, reverse=True)[:20]:
    print("  %7.1f  %s  %s -> %s" % (g, s, a[:60], b[:60]))
print("memset / memcpy records (start_us, dur_us, stream, name):")
for r in copies:
    print("  %8.1f %6.1f  %s  %s" % (r[0], r[1], r[2], r[4]))
