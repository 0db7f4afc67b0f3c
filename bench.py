#!/usr/bin/env python
"""bench.py -- windows/sec of the MTAD-GAT hot path on one or more H100s, next to the reference's own PyTorch path.

    python bench.py [--gpus N] [--steps K] [--warmup W] [--impl ours|reference] [--config c2|c3|c4|c5]
                    [--scaling weak|strong] [--gatv1] [--batch B] [--no-graph] [--skip-cpu] [--skip-ref-cuda]
                    [--dump-outputs DIR]

Default workload ("C2"): MTAD_GAT(k=38, n=100, out=38, forecast_n_layers=3, dropout=0.3) in
train mode, 256 windows per GPU of synthetic uniform[0,1) data; one step = zero_grad, forward, sqrt(mse)+sqrt(mse)
loss, backward, Adam (the reference's training.py:109-127).  Other configs: --config c3 (k=55, out=1,
forward-only scoring, batch 4096), c4 (k=512, batch 1024 GLOBAL, strong scaling), c5 (n=512, batch 512 global).

JSON line (driver contract): value = device-resident inputs, per-step CUDA events, L2 flushed between steps;
e2e = pinned host batch -> H2D -> step -> D2H result inside the timed region; roofline = the dominant single kernel,
timed live, against its algorithmic bytes; cpu_baseline = the UNMODIFIED reference (baseline/_ref, staged by
__graft_entry__.build() from a reference checkout) on the host cores; reference_cuda = the same reference model run eagerly
on this GPU (cuBLAS/cuDNN: what a user of the reference gets today; informative).
`--impl reference` runs only that reference on the host CPU at the same config (same batch for C2).
`--dump-outputs DIR` writes what the last timed step computed (see dump_outputs) so two builds can be compared.
"""
import argparse
import csv
import glob
import importlib
import json
import os
import subprocess
import sys
import threading
import time

import numpy as np

ROOT = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, ROOT)
REF_DIR = os.path.join(ROOT, "baseline", "_ref")

# name -> model kwargs, mode, batch, whether that batch is global, reference micro-batch
CONFIGS = {
    "c2": dict(kw=dict(n_features=38, window_size=100, out_dim=38, forecast_n_layers=3, dropout=0.3), train=True,
               batch=256, batch_is_global=False, ref_batch=256,
               label="SMD-shape (k=38,n=100) MTAD_GAT train step fwd+bwd+Adam, batch 256/GPU, fp32"),
    "c3": dict(kw=dict(n_features=55, window_size=100, out_dim=1, forecast_n_layers=3, dropout=0.3), train=False,
               batch=4096, batch_is_global=False, ref_batch=256,
               label="MSL-shape (k=55,n=100,out=1) MTAD_GAT forward-only scoring, batch 4096/GPU, fp32"),
    "c4": dict(kw=dict(n_features=512, window_size=100, out_dim=512, forecast_n_layers=3, dropout=0.3), train=True,
               batch=1024, batch_is_global=True, ref_batch=4,
               label="wide-feature (k=512,n=100) MTAD_GAT train step, global batch 1024, fp32"),
    "c5": dict(kw=dict(n_features=38, window_size=512, out_dim=38, forecast_n_layers=3, dropout=0.3), train=True,
               batch=512, batch_is_global=True, ref_batch=8,
               label="long-window (k=38,n=512) MTAD_GAT train step, global batch 512, fp32"),
}
METRIC = "windows/sec MTAD-GAT fwd+bwd (k=38,n=100)"


def metric_name(cfgname):
    c = CONFIGS[cfgname]
    k, n = c["kw"]["n_features"], c["kw"]["window_size"]
    return METRIC if cfgname == "c2" else f"windows/sec MTAD-GAT {'fwd+bwd' if c['train'] else 'fwd'} (k={k},n={n})"


def load_peaks():
    p = os.path.join(ROOT, "MEASURED_PEAKS.json")
    if os.path.exists(p):
        d = json.load(open(p))
        return {"hbm_gbs": d["hbm_gbs"], "bf16_tflops": d["bf16_tflops"],
                "bf16_tflops_sustained": d.get("bf16_tflops_sustained", d["bf16_tflops"]), "src": "MEASURED_PEAKS.json"}
    # fallback: NVIDIA's H100 SXM data sheet (3.35 TB/s HBM3, 989 TFLOP/s dense BF16 at up to 700 W); not measured
    return {"hbm_gbs": 3350.0, "bf16_tflops": 989.0, "bf16_tflops_sustained": 989.0, "src": "H100 SXM data sheet"}


def ncu_traffic(kernel_substr):
    """dram__bytes_read.sum + dram__bytes_write.sum per launch of the named kernel, from the newest
    profiles/*traffic*.csv, which scripts/ncu_traffic.py writes from an `ncu --set full` capture of this command (none
    are committed; the directory exists only where someone has made such a capture).
    None when no capture names the kernel: the number is never a constant in this file."""
    best = None
    for path in sorted(glob.glob(os.path.join(ROOT, "profiles", "*traffic*.csv"))):
        try:
            for row in csv.DictReader(open(path)):
                if kernel_substr in row.get("kernel", ""):
                    best = {"bytes": float(row["dram_read_bytes"]) + float(row["dram_write_bytes"]),
                            "src": os.path.relpath(path, ROOT), "batch": int(row.get("batch", 0) or 0)}
        except Exception:
            continue
    return best


# ----------------------------------------------------------------------------------------------------------
# the reference itself (unmodified modules.py / mtad_gat.py staged under baseline/_ref)
# ----------------------------------------------------------------------------------------------------------
def load_reference():
    """Import MTAD_GAT from baseline/_ref (never from the package under test).  None when it was not staged."""
    if not os.path.exists(os.path.join(REF_DIR, "mtad_gat.py")):
        return None
    for name in ("modules", "mtad_gat"):
        sys.modules.pop(name, None)
    sys.path.insert(0, REF_DIR)
    try:
        mod = importlib.import_module("mtad_gat")
    finally:
        sys.path.remove(REF_DIR)
    assert os.path.samefile(os.path.dirname(mod.__file__), REF_DIR)
    return mod.MTAD_GAT


def calibrate_threads(cfgname, gatv1=False):
    """The reference's CPU path at this shape is dominated by page-faulting multi-GB temporaries: on a 128-thread host it
    runs several times SLOWER with all threads than with a few.  The baseline should be the reference at its best, so
    one short step at a reduced batch is timed per candidate thread count and the fastest is used (reported as `cores`)."""
    import torch
    n_all = os.cpu_count() or 1
    cands = sorted({c for c in (4, 8, 16, 32, 64) if c <= n_all} | ({n_all} if n_all <= 64 else set()))
    rb = max(2, min(16, CONFIGS[cfgname]["ref_batch"]))
    best = (None, 0.0)
    tried = {}
    torch.set_num_threads(cands[0])
    reference_rate(cfgname, rb, 1, 0, "cpu", gatv1, budget_s=20.0)          # lazy initialisation, untimed
    for c in cands:
        torch.set_num_threads(c)
        res = reference_rate(cfgname, rb, 2, 0, "cpu", gatv1, budget_s=15.0)
        if res is None:
            return n_all, {}
        tried[c] = round(res[1], 1)
        if res[1] > best[1]:
            best = (c, res[1])
    torch.set_num_threads(best[0])
    return best[0], tried


def reference_rate(cfgname, batch, steps, warmup, device, gatv1=False, budget_s=150.0):
    """windows/s of the reference's own step (training.py:109-127: zero_grad, forward, sqrt-MSE losses, backward,
    Adam.step) or no_grad forward (prediction.py:50-55), fp32, on `device`.  Returns (mean_rate, best_rate, times_s)."""
    import torch
    RefModel = load_reference()
    if RefModel is None:
        return None
    c = CONFIGS[cfgname]
    kw = dict(c["kw"])
    if gatv1:
        kw["use_gatv2"] = False
    torch.manual_seed(0)
    model = RefModel(**kw).to(device)
    k, n = kw["n_features"], kw["window_size"]
    x = torch.rand(batch, n, k).to(device)
    y = torch.rand(batch, 1, k).to(device)
    td = [0] if kw["out_dim"] == 1 else None
    crit = torch.nn.MSELoss()
    times = []
    if c["train"]:
        model.train()
        opt = torch.optim.Adam(model.parameters(), lr=1e-3)

        def one():
            opt.zero_grad()
            preds, recons = model(x)
            xx, yy = x, y
            if td is not None:
                xx = x[:, :, td]; yy = y[:, :, td].squeeze(-1)
            if preds.ndim == 3:
                preds = preds.squeeze(1)
            if yy.ndim == 3:
                yy = yy.squeeze(1)
            loss = torch.sqrt(crit(yy, preds)) + torch.sqrt(crit(xx, recons))
            loss.backward()
            opt.step()
            return loss
    else:
        model.eval()

        def one():
            with torch.no_grad():
                return model(x)[0]
    cuda = str(device).startswith("cuda")
    t_begin = time.perf_counter()
    for i in range(warmup + steps):
        if len(times) >= 2 and time.perf_counter() - t_begin > budget_s:
            break                                    # bounded sample: the run must end within a few minutes
        if cuda:
            torch.cuda.synchronize()
        t0 = time.perf_counter()
        r = one()
        if cuda:
            torch.cuda.synchronize()
        else:
            float(r.detach().sum())
        if i >= warmup:
            times.append(time.perf_counter() - t0)
    mean = batch / (sum(times) / len(times))
    return mean, batch / min(times), times


def cpu_model_name():
    try:
        for l in open("/proc/cpuinfo"):
            if l.startswith("model name"):
                return l.split(":", 1)[1].strip()
    except Exception:
        pass
    return "unknown"


def oracle_port_rate(cfgname, sample_b, reps):
    """Fallback when baseline/_ref is absent: the numpy port of the reference path (oracle/), forward + backward."""
    from oracle import mtad_gat_oracle as orc
    kw = CONFIGS[cfgname]["kw"]
    cfg = orc.Config(**kw)
    params = orc.make_params(cfg, seed=0, dtype=np.float32)
    rng = np.random.default_rng(0)
    x = rng.random((sample_b, cfg.n, cfg.k)).astype(np.float32)
    y = rng.random((sample_b, 1, cfg.k)).astype(np.float32)
    orc.loss_fwd_bwd(x, y, params, cfg)
    times = []
    for _ in range(reps):
        t0 = time.perf_counter()
        orc.loss_fwd_bwd(x, y, params, cfg)
        times.append(time.perf_counter() - t0)
    return sample_b / (sum(times) / len(times)), sample_b / min(times), times


def run_reference(args):
    """The reference arm: the UNMODIFIED reference (baseline/_ref) on this box's host cores, same config; each step is
    one full reference step at the reference batch (C2: the same 256-window batch as our arm)."""
    rank = int(os.environ.get("RANK", "0"))
    if rank != 0:
        return
    import torch
    cores, tried = calibrate_threads(args.config, args.gatv1)
    c = CONFIGS[args.config]
    rb = c["ref_batch"]
    res = reference_rate(args.config, rb, args.steps, max(1, min(args.warmup, 2)), "cpu", args.gatv1,
                         budget_s=float("inf"))                       # exactly --steps timed steps
    kind = "reference"
    if res is None:
        kind = "port"
        rb = 16
        res = oracle_port_rate(args.config, rb, args.steps)
    mean, best, times = res
    ms = 1e3 * sum(times) / len(times)
    sample = (f"{len(times)} timed steps of the unmodified reference (baseline/_ref mtad_gat.py + modules.py, torch "
              f"{torch.__version__} CPU, fp32) at batch {rb} with {cores} of {os.cpu_count()} host threads -- the fastest of "
              f"the calibrated counts {tried} (windows/s at a reduced batch)" if kind == "reference" else
              f"{len(times)} timed {rb}-window fwd+bwd passes of the numpy port (oracle/): baseline/_ref was not staged")
    line = {
        "impl": "reference", "metric": metric_name(args.config), "value": mean, "unit": "windows/s",
        "n_gpus": args.gpus, "steps": len(times), "warmup": args.warmup, "ms_per_step": ms,
        "higher_is_better": True, "scaling": args.scaling, "vs_baseline": None, "dtype": "fp32", "data": "synthetic",
        "config": {"workload": c["label"], "reference_batch": rb, "same_config": rb == c["batch"] and kind == "reference",
                   "gat": "v1" if args.gatv1 else "v2", "cpu": cpu_model_name()},
        "cpu_baseline": {"value": mean, "unit": "windows/s", "cores": cores, "kind": kind, "sample": sample,
                         "best": best},
        "e2e": {"value": mean, "unit": "windows/s", "h2d_bytes_per_step": 0, "d2h_bytes_per_step": 0},
    }
    print(json.dumps(line), flush=True)


# ----------------------------------------------------------------------------------------------------------
class ClockSampler:
    """SM clock and throttle reasons sampled DURING the timed region: NVML (the library behind nvidia-smi; ~1 ms per
    sample) when importable, else the `nvidia-smi --query-gpu=clocks.sm,...` line of the profiling recipe."""
    FIELDS = ("clocks.sm,clocks.max.sm,power.draw,clocks_event_reasons.hw_slowdown,"
              "clocks_event_reasons.hw_thermal_slowdown,clocks_event_reasons.sw_thermal_slowdown,"
              "clocks_event_reasons.sw_power_cap")
    NAMES = ["hw_slowdown", "hw_thermal_slowdown", "sw_thermal_slowdown", "sw_power_cap"]

    def __init__(self, gpu_index):
        self.idx = gpu_index
        self.samples = []          # (sm_mhz, [reason flags], power_w)
        self.sm_max = None
        self.source = None
        self.stop = threading.Event()
        self.th = None
        self.nv = None
        try:
            import pynvml
            pynvml.nvmlInit()
            vis = os.environ.get("CUDA_VISIBLE_DEVICES")
            phys = int(vis.split(",")[gpu_index]) if vis and all(v.strip().isdigit() for v in vis.split(",")) else gpu_index
            self.h = pynvml.nvmlDeviceGetHandleByIndex(phys)
            self.sm_max = float(pynvml.nvmlDeviceGetMaxClockInfo(self.h, pynvml.NVML_CLOCK_SM))
            self.nv = pynvml
            self.source = "nvml"
        except Exception:
            self.nv = None
            self.source = "nvidia-smi"

    def _sample_nvml(self):
        nv = self.nv
        sm = float(nv.nvmlDeviceGetClockInfo(self.h, nv.NVML_CLOCK_SM))
        r = nv.nvmlDeviceGetCurrentClocksEventReasons(self.h)
        flags = [bool(r & nv.nvmlClocksEventReasonHwSlowdown), bool(r & nv.nvmlClocksEventReasonHwThermalSlowdown),
                 bool(r & nv.nvmlClocksEventReasonSwThermalSlowdown), bool(r & nv.nvmlClocksEventReasonSwPowerCap)]
        try:
            pw = nv.nvmlDeviceGetPowerUsage(self.h) / 1000.0
        except Exception:
            pw = None
        self.samples.append((sm, flags, pw))

    def _sample_smi(self):
        out = subprocess.run(["nvidia-smi", "-i", str(self.idx), f"--query-gpu={self.FIELDS}",
                              "--format=csv,noheader,nounits"], capture_output=True, text=True, timeout=5).stdout
        parts = [p.strip() for p in out.strip().split(",")]
        if len(parts) >= 7 and parts[0].replace(".", "").isdigit():
            self.sm_max = float(parts[1])
            try:
                pw = float(parts[2])
            except ValueError:
                pw = None
            self.samples.append((float(parts[0]), [parts[3 + i].lower().startswith("active") for i in range(4)], pw))

    def _run(self):
        while not self.stop.is_set():
            try:
                if self.nv is not None:
                    self._sample_nvml()
                else:
                    self._sample_smi()
            except Exception:
                pass
            self.stop.wait(0.005 if self.nv is not None else 0.05)

    def __enter__(self):
        self.th = threading.Thread(target=self._run, daemon=True)
        self.th.start()
        return self

    def __exit__(self, *a):
        self.stop.set()
        self.th.join(timeout=6)

    def summary(self):
        if not self.samples:
            return {"sm_mhz": None, "sm_max_mhz": self.sm_max, "reasons": ["clock sampling unavailable"], "samples": 0}
        sm = sorted(s[0] for s in self.samples)
        reasons = [n for i, n in enumerate(self.NAMES) if any(s[1][i] for s in self.samples)]
        pws = [s[2] for s in self.samples if s[2] is not None]
        return {"sm_mhz": sm[len(sm) // 2], "sm_max_mhz": self.sm_max, "reasons": reasons, "samples": len(self.samples),
                "power_w_max": max(pws) if pws else None, "source": self.source}


class ForwardStep:
    """Forward-only scoring step (C3): one no_grad forward of a static batch, optionally replayed from a CUDA graph,
    with the same host-input pipeline interface as training.TrainStep."""

    def __init__(self, model, batch, use_graph=True):
        import torch
        p0 = next(model.parameters())
        n, k = model.temporal_gat.window_size, model.temporal_gat.n_features
        self.model, self.use_graph = model, use_graph
        self.x = torch.zeros(batch, n, k, device=p0.device)
        self.preds = self.recons = None
        self.g = None
        self.launches_per_step = 0
        self._stage = [torch.zeros_like(self.x) for _ in range(2)]
        self._copy_stream = torch.cuda.Stream(device=p0.device)
        self._ev = [None, None]
        self._put = self._get = 0
        self._host = None

    def _fwd(self):
        import torch
        with torch.no_grad():
            self.preds, self.recons = self.model(self.x)

    def _run(self):
        import torch
        import mtad_gat_pytorch_b200 as mg
        if not self.use_graph:
            self._fwd()
            return
        if self.g is None:
            s = torch.cuda.Stream()
            s.wait_stream(torch.cuda.current_stream())
            with torch.cuda.stream(s):
                for _ in range(2):
                    self._fwd()
            torch.cuda.current_stream().wait_stream(s)
            torch.cuda.synchronize()
            mg.reset_launch_count()
            self.g = torch.cuda.CUDAGraph()
            with torch.cuda.graph(self.g, stream=s):
                self._fwd()
            self.launches_per_step = mg.launch_count()
        self.g.replay()

    def run_device(self, x, y=None):
        self.x.copy_(x)
        self._run()

    def prefetch_host(self, x_host, y_host=None):
        import torch
        slot = self._put & 1
        cs = self._copy_stream
        cs.wait_stream(torch.cuda.current_stream())
        with torch.cuda.stream(cs):
            self._stage[slot].copy_(x_host, non_blocking=True)
            ev = torch.cuda.Event(); ev.record(cs)
        self._ev[slot] = ev
        self._put += 1

    def launch_prefetched(self):
        import torch
        slot = self._get & 1
        self._get += 1
        torch.cuda.current_stream().wait_event(self._ev[slot])
        self.x.copy_(self._stage[slot])
        self._run()
        if self._host is None:
            self._host = [(torch.zeros_like(self.preds, device="cpu").pin_memory(),
                           torch.zeros_like(self.recons, device="cpu").pin_memory()) for _ in range(2)]
            self._hev = [None, None]
            self._hput = self._hget = 0
        k = self._hput & 1
        self._hput += 1
        self._host[k][0].copy_(self.preds, non_blocking=True)
        self._host[k][1].copy_(self.recons, non_blocking=True)
        ev = torch.cuda.Event(); ev.record()
        self._hev[k] = ev

    def collect(self):
        k = self._hget & 1
        self._hget += 1
        self._hev[k].synchronize()
        return float(self._host[k][0].sum())

    def d2h_bytes(self):
        return int(self.preds.numel() * 4 + self.recons.numel() * 4)


DUMP_MAX_ELEMS = 1 << 20          # per array; larger outputs are dumped as a fixed, seeded sample
DUMP_MAX_BYTES = 64 << 20         # all arrays together


def dump_outputs(out_dir, step, model, train):
    """What the last timed step handed its caller, as DIR/<name>.npy (float32): the two loss terms, every gradient and
    every updated parameter of a training step, or the predictions and reconstructions of a forward step.  Arrays
    above their share of the budget (DUMP_MAX_ELEMS, and never more than what is left of DUMP_MAX_BYTES) are replaced by
    the elements at that many sorted flat indices drawn from a fixed seed (name suffix `.sample`), so two builds compare
    output for output within 64 MB."""
    import numpy as np
    import torch
    torch.cuda.synchronize()
    arrays = {}
    if train:
        arrays["loss_terms"] = step.losses
        for name, p in model.named_parameters():
            arrays["param." + name] = p.detach()
            if p.grad is not None:
                arrays["grad." + name] = p.grad
    else:
        arrays["preds"] = step.preds
        arrays["recons"] = step.recons
    os.makedirs(out_dir, exist_ok=True)
    left = DUMP_MAX_BYTES // 4 - 32 * len(arrays)        # elements; 128 B of .npy header per file
    for i, (name, t) in enumerate(arrays.items()):
        a = t.detach().float().cpu().numpy()
        cap = min(DUMP_MAX_ELEMS, left // (len(arrays) - i))          # the rest of the budget shared fairly
        if a.size > cap:
            idx = np.sort(np.random.default_rng(0).choice(a.size, cap, replace=False))
            a, name = a.reshape(-1)[idx], name + ".sample"
        left -= a.size
        np.save(os.path.join(out_dir, name + ".npy"), np.ascontiguousarray(a, dtype=np.float32))


def run_ours(args):
    import torch
    import torch.distributed as dist
    import mtad_gat_pytorch_b200 as mg
    from mtad_gat_pytorch_b200 import training as mgt

    world = int(os.environ.get("WORLD_SIZE", "1"))
    rank = int(os.environ.get("RANK", "0"))
    local = int(os.environ.get("LOCAL_RANK", "0"))
    torch.cuda.set_device(local)
    dev = torch.device("cuda", local)
    if world > 1:
        dist.init_process_group("nccl", device_id=dev)
    c = CONFIGS[args.config]
    kw = dict(c["kw"])
    if args.gatv1:
        kw["use_gatv2"] = False
    k, n = kw["n_features"], kw["window_size"]
    base_b = args.batch or c["batch"]
    if args.scaling == "strong":
        lo, hi = mgt.shard_batch(base_b, world, rank)
        B, global_b = hi - lo, base_b
    else:
        B, global_b = base_b, base_b * world
    if args.gru_split:
        mg.set_gru_split(args.gru_split)
    torch.manual_seed(0)
    model = mg.MTAD_GAT(**kw).to(dev)
    model.train(c["train"])
    if c["train"]:
        if args.torch_adam:
            opt = torch.optim.Adam(model.parameters(), lr=1e-3, capturable=not args.no_graph, fused=True)
        else:
            opt = mgt.FusedAdam(model.parameters(), lr=1e-3)       # torch.optim.Adam semantics, one launch (mtadgat_adam_step)
        step = mgt.TrainStep(model, opt, batch=B, use_graph=not args.no_graph, world_size=world,
                             target_dims=[0] if kw["out_dim"] == 1 else None, capture_comm=args.capture_comm,
                             overlap_comm=args.overlap_comm, pipeline=args.pipeline)
    else:
        step = ForwardStep(model, B, use_graph=not args.no_graph)

    g = torch.Generator(device="cpu").manual_seed(1234 + rank)
    n_host = 4 if B * n * k * 4 > (64 << 20) else 8
    xs_host = [torch.rand(B, n, k, generator=g).pin_memory() for _ in range(n_host)]
    ys_host = [torch.rand(B, 1, k, generator=g).pin_memory() for _ in range(n_host)]
    xs_dev = [t.to(dev) for t in xs_host]
    ys_dev = [t.to(dev) for t in ys_host]
    flush = torch.empty(256 * 1024 * 1024 // 4, dtype=torch.float32, device=dev)   # > 50 MB L2

    def barrier():
        if world > 1:
            dist.barrier()
        torch.cuda.synchronize()

    # ---- warm-up (also captures the CUDA graph) ----
    W = max(args.warmup, 3)
    for i in range(W):
        step.run_device(xs_dev[i % n_host], ys_dev[i % n_host])
    barrier()

    # ---- timed region: device-resident inputs, per-step CUDA events, L2 flushed between steps ----
    mg.reset_launch_count()
    evs = [(torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)) for _ in range(args.steps)]
    with ClockSampler(local) as clocks:
        barrier()
        t_wall0 = time.perf_counter()
        for i in range(args.steps):
            flush.zero_()
            evs[i][0].record()
            step.run_device(xs_dev[i % n_host], ys_dev[i % n_host])
            evs[i][1].record()
        barrier()
        t_wall = time.perf_counter() - t_wall0
        ms_dev = sum(a.elapsed_time(b) for a, b in evs) / args.steps
        launches = step.launches_per_step * args.steps if step.launches_per_step else mg.launch_count()
        if args.dump_outputs and rank == 0:
            dump_outputs(args.dump_outputs, step, model, c["train"])

        # ---- e2e: host pinned inputs -> H2D -> step -> D2H result, wall clock over K steps ----
        barrier()
        t0 = time.perf_counter()
        last = None
        # software pipeline of the caller's loop: H2D of batch i+1 (copy stream) and the host-side enqueue of step
        # i+1 overlap step i; every step still copies its batch in and its result out (the result of step i is read on
        # the host after step i+1 has been enqueued)
        step.prefetch_host(xs_host[0], ys_host[0])
        for i in range(args.steps):
            if i + 1 < args.steps:
                step.prefetch_host(xs_host[(i + 1) % n_host], ys_host[(i + 1) % n_host])
            step.launch_prefetched()
            if i > 0:
                last = step.collect()
        last = step.collect()
        torch.cuda.synchronize()
        e2e_s = (time.perf_counter() - t0) / args.steps     # local wall time; MAX over ranks below (the closing
        barrier()                                           # collective barrier itself is not part of the K steps)

        # ---- sustained: the same device-resident loop for ~2 s without the per-step flush bookkeeping (burst vs
        #      sustained clocks; reported next to `value`, never instead of it) ----
        sustained = None
        if args.sustain_s > 0:
            n_s = max(args.steps, int(args.sustain_s / (ms_dev * 1e-3)))
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            barrier()
            e0.record()
            for i in range(n_s):
                flush.zero_()
                step.run_device(xs_dev[i % n_host], ys_dev[i % n_host])
            e1.record()
            barrier()
            sustained = {"steps": n_s, "ms_per_step_incl_flush": e0.elapsed_time(e1) / n_s}
    t_ms = torch.tensor([ms_dev, e2e_s * 1e3], dtype=torch.float64, device=dev)
    if world > 1:
        dist.all_reduce(t_ms, op=dist.ReduceOp.MAX)
    ms_dev, e2e_ms = float(t_ms[0]), float(t_ms[1])

    if rank == 0:
        peaks = load_peaks()
        from mtad_gat_pytorch_b200 import kernel_bench
        pipes = getattr(step, "pipeline", 1)
        rec_b = B if pipes == 1 else (B // pipes + 15) // 16 * 16
        kern = kernel_bench.stage_rooflines(model, B, peaks, dev, train=c["train"], rec_batch=rec_b)
        # dominant single kernel = the slowest single launch of the step among the persistent recurrences and the GAT
        # score kernels; the other rows are whole stages (several launches)
        single = [r for r in kern if r.get("single_kernel")]
        dominant = max(single or kern, key=lambda r: r["ms"])
        tr = ncu_traffic(dominant.get("ncu_name", dominant["kernel"]))
        roof = {k_: dominant[k_] for k_ in ("bound", "achieved", "peak", "unit", "frac")}
        roof.update({"traffic": tr["bytes"] if tr and tr["batch"] in (0, rec_b) else None,
                     "traffic_src": tr["src"] if tr and tr["batch"] in (0, rec_b) else None, "windows_per_launch": rec_b,
                     "kernel": dominant["kernel"], "ms": dominant["ms"], "alg_bytes": dominant["alg_bytes"],
                     "alg_bytes_def": dominant.get("alg_bytes_def"), "operand_bytes": dominant.get("operand_bytes"),
                     "frac_operand_bytes": dominant.get("frac_operand_bytes"), "frac_tensor": dominant.get("frac_tensor"),
                     "peak_src": peaks["src"]})
        cpu = None
        ref_cuda = None
        if world == 1 and not args.skip_cpu:
            cores, tried = calibrate_threads(args.config, args.gatv1)
            res = reference_rate(args.config, c["ref_batch"], 3 if c["ref_batch"] >= 64 else 2, 1, "cpu", args.gatv1, budget_s=60.0)
            if res is not None:
                mean, best, times = res
                cpu = {"value": mean, "best": best, "unit": "windows/s", "cores": cores, "kind": "reference",
                       "cpu": cpu_model_name(), "host_threads": os.cpu_count(), "threads_calibration": tried,
                       "sample": f"{len(times)} timed steps (after 1 warm-up) of the unmodified reference (baseline/_ref, torch CPU "
                                 f"fp32, {cores} threads = fastest calibrated count) at batch {c['ref_batch']} ({sum(times):.1f} s)"}
            else:
                mean, best, times = oracle_port_rate(args.config, 16, 3)
                cpu = {"value": mean, "unit": "windows/s", "cores": os.cpu_count(), "kind": "port",
                       "sample": f"3 timed 16-window fwd+bwd passes of the numpy port (oracle/); baseline/_ref not staged ({sum(times):.1f} s)"}
        if world == 1 and not args.skip_ref_cuda:
            try:
                rb = c["ref_batch"]
                res = reference_rate(args.config, rb, 10, 3, dev, args.gatv1)
                if res is not None:
                    ref_cuda = {"value": res[0], "best": res[1], "unit": "windows/s", "batch": rb,
                                "what": "the unmodified reference model on this GPU, eager PyTorch (cuBLAS/cuDNN kernels), "
                                        "wall clock with synchronize per step; informative"}
            except Exception as e:                                   # e.g. out of memory at the larger shapes
                ref_cuda = {"unavailable": f"{type(e).__name__}: {str(e)[:120]}"}
            torch.cuda.empty_cache()
        scoring_blk = None
        if not c["train"] and world == 1:
            # the caller-level inference loop (prediction.py:36-94) through this package's single-pass scorer: a pinned
            # host (N,k) series in, per-timestamp anomaly scores out; every scored timestamp costs ONE window forward
            # (the reference runs two) and the H2D traffic is the series itself, not n overlapping copies of it
            from mtad_gat_pytorch_b200 import scoring
            n_chunks = 4
            Ns = n + n_chunks * B
            series = torch.rand(Ns, k, generator=g).pin_memory()
            scorer = scoring.SeriesScorer(model, batch=B, use_graph=not args.no_graph)
            td = [0] if kw["out_dim"] == 1 else None
            scorer.score(series, 1.0, td)                    # warm-up + graph capture
            torch.cuda.synchronize()
            ts = []
            for _ in range(3):
                t0 = time.perf_counter()
                res = scorer.score(series, 1.0, td)
                ag = res["a_global"].cpu()
                ts.append(time.perf_counter() - t0)
            ts.sort()
            scoring_blk = {"timestamps_per_s": (Ns - n) / ts[1], "windows_forwarded": Ns - n + 1, "series_rows": Ns,
                           "h2d_bytes": Ns * k * 4, "d2h_bytes": int(ag.numel() * 4), "median_s": ts[1],
                           "what": "SeriesScorer.score on a pinned host series: H2D of the series, one forward per distinct "
                                   "window read in place, device score epilogue, D2H of A_Score_Global (wall clock, median of 3)",
                           "reference_equivalent_forwards": 2 * (Ns - n)}
        h2d = int(xs_host[0].numel() * 4 + (ys_host[0].numel() * 4 if c["train"] else 0))
        d2h = 8 if c["train"] else step.d2h_bytes()
        line = {
            "metric": metric_name(args.config), "value": global_b / (ms_dev * 1e-3), "unit": "windows/s",
            "n_gpus": world, "steps": args.steps, "warmup": W, "ms_per_step": ms_dev,
            "higher_is_better": True, "scaling": args.scaling, "vs_baseline": None, "dtype": "fp32", "data": "synthetic",
            "config": {"workload": c["label"], "global_batch": global_b, "per_gpu_batch": B, "parallelism": f"dp{world}",
                       "gat": "v1" if args.gatv1 else "v2",
                       "arithmetic": "fp32 storage/accumulate; GEMMs bf16x3 on wgmma, recurrences fp16 operands on wgmma",
                       "e2e_loop": "pinned host batches, H2D of batch i+1 and enqueue of step i+1 overlap step i, result of every step copied back",
                       "cuda_graph": not args.no_graph, "l2": "256 MiB buffer zeroed between timed steps",
                       "optimizer": (("torch.optim.Adam(fused)" if args.torch_adam else "Adam in one launch (mtadgat_adam_step, torch.optim.Adam semantics)") + " inside the step") if c["train"] else None,
                       "comm": None if world == 1 else ("NCCL all-reduce of the gradient bucket in place, " + ("captured in the step graph" if args.capture_comm else "eager between the fwd/bwd graph and the Adam graph")),
                       "pipeline": getattr(step, "pipeline", 1)},
            "e2e": {"value": global_b / (e2e_ms * 1e-3), "unit": "windows/s", "h2d_bytes_per_step": h2d,
                    "d2h_bytes_per_step": d2h, "ms_per_step": e2e_ms},
            "gpu_launches": int(launches), "roofline": roof, "kernels": kern, "cpu_baseline": cpu,
            "reference_cuda": ref_cuda, "sustained": sustained, "single_pass_scoring": scoring_blk,
            "clocks": clocks.summary(), "wall_s_timed": t_wall, "result": last,
        }
        print(json.dumps(line), flush=True)
    if world > 1:
        # orderly teardown, but never hang on it: the result line is out; a watchdog ends the process if the collective
        # teardown does not return (graphs that captured collectives, a peer that already left, ...)
        t = threading.Timer(20.0, lambda: os._exit(0))
        t.daemon = True
        t.start()
        if hasattr(step, "release"):
            step.release()
        torch.cuda.synchronize()
        try:
            dist.destroy_process_group()
        except Exception:
            pass
        sys.stdout.flush()
        os._exit(0)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--gpus", type=int, default=1)
    ap.add_argument("--steps", type=int, default=None, help="timed steps (default 200; 5 with --impl reference)")
    ap.add_argument("--warmup", type=int, default=5)
    ap.add_argument("--impl", default="ours", choices=["ours", "reference"])
    ap.add_argument("--config", default="c2", choices=sorted(CONFIGS))
    ap.add_argument("--scaling", default=None, choices=["weak", "strong"])
    ap.add_argument("--gatv1", action="store_true", help="use_gatv2=False (the HBM-bound GAT variant)")
    ap.add_argument("--batch", type=int, default=0, help="override the config's batch")
    ap.add_argument("--no-graph", action="store_true")
    ap.add_argument("--capture-comm", action="store_true", help="capture the gradient all-reduce into the step graph")
    ap.add_argument("--overlap-comm", action="store_true", help="with --capture-comm: reduce the early bucket half during backward")
    ap.add_argument("--pipeline", type=int, default=-1, help="micro-batch pipelines inside the step (-1 = auto)")
    ap.add_argument("--torch-adam", action="store_true", help="use torch.optim.Adam(fused) instead of the library's one-launch Adam")
    ap.add_argument("--skip-cpu", action="store_true")
    ap.add_argument("--skip-ref-cuda", action="store_true")
    ap.add_argument("--sustain-s", type=float, default=2.0)
    ap.add_argument("--gru-split", type=int, default=0, help="clusters per 16-window tile in the recurrence (0 = auto)")
    ap.add_argument("--dump-outputs", default=None, metavar="DIR",
                    help="after the timed steps, write what the last timed step computed to DIR/<name>.npy")
    args = ap.parse_args()
    if args.steps is None:
        args.steps = 5 if args.impl == "reference" else 200
    if args.steps < 1:
        ap.error("--steps must be at least 1")
    if args.scaling is None:
        args.scaling = "strong" if CONFIGS[args.config]["batch_is_global"] else "weak"
    if args.impl == "reference":
        run_reference(args)
    else:
        run_ours(args)


if __name__ == "__main__":
    main()
