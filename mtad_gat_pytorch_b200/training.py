"""Training-step driver for the H100 path: the reference's step (training.py:106-127: zero_grad, forward,
sqrt-MSE losses, backward, Adam) with static device buffers, optionally captured once in a CUDA graph and
replayed (the step is launch-bound at batch 256), and with a flat-bucket NCCL gradient all-reduce when
world_size > 1 (one process per GPU; windows shard over the batch, parameters are replicated)."""
import torch
import torch.distributed as dist

from . import functional as F


def rmse_losses(x, y, preds, recons, target_dims=None):
    """training.py:113-124.  CUDA tensors of matching element counts take the fused two-launch kernel
    (mtadgat_rmse_pair_fwd / _bwd); CPU tensors (host-side tests) use the plain expression."""
    if target_dims is not None:
        x = x[:, :, target_dims]
        y = y[:, :, target_dims].squeeze(-1)
    if preds.ndim == 3:
        preds = preds.squeeze(1)
    if y.ndim == 3:
        y = y.squeeze(1)
    if preds.is_cuda and preds.shape == y.shape and recons.shape == x.shape and preds.dtype == torch.float32:
        return F.RmsePairFn.apply(preds, y, recons, x)
    fl = torch.sqrt(torch.mean((y - preds) ** 2))
    rl = torch.sqrt(torch.mean((x - recons) ** 2))
    return fl, rl


def allreduce_gradients(params, world_size):
    """Average the gradients of `params` across ranks with ONE flat-bucket all-reduce (1.6 MB at SMD shape).
    Backend-agnostic (NCCL on the GPUs, gloo in the CPU tests).  Generic path: flatten, reduce, copy back; TrainStep
    avoids both copies by having the backward kernels write straight into a GradBucket."""
    if world_size == 1:
        return
    grads = [p.grad for p in params]
    flat = torch._utils._flatten_dense_tensors(grads)
    if dist.get_backend() == "nccl":
        dist.all_reduce(flat, op=dist.ReduceOp.AVG)        # the average is formed inside the collective
    else:
        dist.all_reduce(flat)
        flat.div_(world_size)
    torch._foreach_copy_(grads, torch._utils._unflatten_dense_tensors(flat, grads))


class GradBucket:
    """One flat fp32 buffer that the weight-gradient kernels write into directly (functional._grad_out hands every
    backward a view of it instead of a fresh tensor, and autograd adopts that view as `.grad`): the all-reduce runs on
    the buffer in place -- no flatten before, no copy back after.

    Parameters are laid out in two contiguous groups, in the order backpropagation finishes them:
      early = heads + decoder + encoder GRU (1.03 MB at SMD shape; complete when the encoder BPTT has been issued),
      late  = conv + the two GAT layers (complete at the end of backward).
    The early group is reduced on a communication stream while the GAT/conv backward still runs."""

    def __init__(self, model):
        early, late = [], []
        for name, p in model.named_parameters():
            if not p.requires_grad:
                continue
            (late if name.startswith(("conv.", "feature_gat.", "temporal_gat.")) else early).append(p)
        self.params = early + late
        ALIGN = 64                         # floats: every slot starts on a 256-byte boundary (vectorised stores in the
        offs, off = [], 0                  # weight-gradient kernels); the zero padding rides along in the all-reduce
        for p in self.params:
            offs.append(off)
            off += (p.numel() + ALIGN - 1) // ALIGN * ALIGN
        total = off
        n_early = offs[len(early)] if late else total
        self.flat = torch.zeros(total, dtype=torch.float32, device=self.params[0].device)
        self.early = self.flat.narrow(0, 0, n_early)
        self.late = self.flat.narrow(0, n_early, total - n_early)
        self.sinks = {id(p): (self.flat, o) for p, o in zip(self.params, offs)}

    def adopted(self):
        """True when every parameter's .grad aliases its slot of the bucket (autograd adopted the views)."""
        return all(p.grad is not None and p.grad.data_ptr() == self.flat.data_ptr() + 4 * off
                   for p in self.params for (_, off) in [self.sinks[id(p)]])


class FusedAdam:
    """torch.optim.Adam(lr, betas, eps) semantics (no weight decay, no amsgrad -- train.py:92 uses neither) for CUDA
    fp32 parameters, as ONE kernel launch over all tensors (`mtadgat_adam_step`): torch's multi-tensor Adam takes 38 us
    for this model's 28 small tensors at the tail of every step, this one ~5 us.  Graph-capturable (the step counter lives
    on the device; lr / betas / eps are kernel arguments, so a captured graph keeps the values it was captured with --
    re-capture after changing them; the reference's loop never does, training.py:106-127).  Exposes
    `.state[p] = {step, exp_avg, exp_avg_sq}`, `.param_groups`, `.zero_grad`, `.step`."""

    def __init__(self, params, lr=1e-3, betas=(0.9, 0.999), eps=1e-8):
        self.params = [p for p in params if p.requires_grad]
        assert self.params and all(p.is_cuda and p.dtype == torch.float32 and p.is_contiguous() for p in self.params)
        dev = self.params[0].device
        self.lr, self.betas, self.eps = float(lr), (float(betas[0]), float(betas[1])), float(eps)
        self.param_groups = [{"params": self.params, "lr": self.lr, "betas": self.betas, "eps": self.eps}]
        self._step = torch.zeros(1, dtype=torch.float32, device=dev)
        self.state = {p: {"step": self._step, "exp_avg": torch.zeros_like(p), "exp_avg_sq": torch.zeros_like(p)}
                      for p in self.params}
        self._table = None
        self._table_key = None
        self._max = max(p.numel() for p in self.params)

    def zero_grad(self, set_to_none=True):
        for p in self.params:
            if set_to_none:
                p.grad = None
            elif p.grad is not None:
                p.grad.zero_()

    def step(self):
        from ._lib import lib, check
        grads = [p.grad for p in self.params]
        assert all(g is not None and g.is_contiguous() for g in grads), "FusedAdam.step: every parameter needs a gradient"
        key = tuple(g.data_ptr() for g in grads)
        if key != self._table_key:            # gradient buffers are static under graph replay / GradBucket; rebuilt when they move
            rows = [[p.data_ptr(), g.data_ptr(), self.state[p]["exp_avg"].data_ptr(), self.state[p]["exp_avg_sq"].data_ptr(),
                     p.numel()] for p, g in zip(self.params, grads)]
            if torch.cuda.is_current_stream_capturing():
                raise RuntimeError("FusedAdam: gradient buffers moved during CUDA-graph capture; run one eager step with the "
                                   "same gradient buffers first (TrainStep keeps them in a GradBucket)")
            self._table = torch.tensor(rows, dtype=torch.int64).to(self.params[0].device, non_blocking=False)
            self._table_key = key
        with torch.cuda.device(self.params[0].device):
            check(lib.mtadgat_adam_step(self._table.data_ptr(), len(self.params), self._max, self.lr, self.betas[0],
                                        self.betas[1], self.eps, self._step.data_ptr(),
                                        torch.cuda.current_stream().cuda_stream))


def shard_batch(global_batch, world_size, rank):
    """Windows shard over the batch: contiguous [lo, hi) slice of the global batch owned by `rank`."""
    base, rem = divmod(global_batch, world_size)
    lo = rank * base + min(rank, rem)
    return lo, lo + base + (1 if rank < rem else 0)


class TrainStep:
    """training.py:106-127 of the reference as one replayable unit.

    world_size > 1 (one process per GPU, NCCL): the weight-gradient kernels write straight into a GradBucket, which is
    all-reduced in place (no flatten / copy-back).  Default: the collective runs eagerly between the forward/backward
    graph and the Adam graph.  Opt-in: `capture_comm=True` captures it INTO the step graph (one replay per step) and
    `overlap_comm=True` reduces the early half of the bucket on a communication stream as soon as the encoder BPTT has
    been issued.  At C2 the gradient bucket is 1.6 MB: the collective costs about NCCL's latency floor whichever way it
    is issued, so the simplest variant is the default."""

    def __init__(self, model, optimizer, batch, use_graph=True, world_size=1, target_dims=None, capture_comm=False,
                 overlap_comm=False, pipeline=-1):
        p0 = next(model.parameters())
        self.model, self.opt, self.world = model, optimizer, world_size
        self.target_dims = target_dims
        n, k = model.temporal_gat.window_size, model.temporal_gat.n_features
        self.x = torch.zeros(batch, n, k, device=p0.device)
        self.y = torch.zeros(batch, 1, k, device=p0.device)
        self.losses = torch.zeros(2, device=p0.device)
        self.params = [p for p in model.parameters() if p.requires_grad]
        self.use_graph = use_graph
        # micro-batch pipelines: the step's critical path is four strictly serial 100-step recurrences (latency-, not
        # throughput-bound: 64 SMs run them as fast as 128), so the batch is split into `pipeline` contiguous slices that
        # run forward and backward on their own streams -- one slice's recurrences overlap the other's GAT / GEMM work.
        # The loss is still the reference's sqrt(MSE) over the WHOLE batch (the slices join at the loss), and the
        # slices' parameter gradients are summed, so the step computes exactly what the unsplit step does.
        # At C2 (batch 256) every kernel of the step is latency-bound, so halving its batch does not halve its time and
        # the two slices contend for SMs.
        # The mechanism stays (tested, opt-in); auto = unsplit.
        if pipeline < 0:
            pipeline = 1
        self.pipeline = max(1, pipeline)
        self._pipe_streams = [torch.cuda.Stream(device=p0.device) for _ in range(self.pipeline)] if self.pipeline > 1 else []
        # slice i > 0 runs the model on ALIASES of the parameters (same storage, separate autograd leaves): each slice
        # then owns its gradient tensors and no accumulation kernel races with the parameter-gradient side streams
        self._names = [nm for nm, p in model.named_parameters() if p.requires_grad]
        self._alias = [{nm: p.detach().requires_grad_() for nm, p in model.named_parameters() if p.requires_grad}
                       for _ in range(self.pipeline - 1)]
        self.bucket = None
        self.capture_comm = capture_comm
        self.overlap_comm = overlap_comm
        self._comm_stream = None
        self._early_work = None
        if p0.is_cuda and (world_size == 1 or dist.get_backend() == "nccl"):
            # also on one GPU: gradients at fixed addresses (views of one flat buffer) -- what the one-launch FusedAdam's
            # pointer table and a data-parallel all-reduce both want
            self.bucket = GradBucket(model)
            if world_size > 1:
                self._comm_stream = torch.cuda.Stream(device=p0.device)
        # host-input pipeline: two device staging buffers filled by a copy stream, so the H2D copy of batch i+1
        # overlaps the step on batch i (every batch is still copied inside the timed region)
        self._stage = [(torch.zeros_like(self.x), torch.zeros_like(self.y)) for _ in range(2)]
        self._copy_stream = torch.cuda.Stream(device=p0.device)
        self._staged = [None, None]
        self._put = self._get = 0
        self.g_fb = self.g_opt = None
        self.launches_per_step = 0
        self._warm = 0

    # -- pieces ------------------------------------------------------------------------------------------
    def _reduce_early(self):
        """Called by the encoder GRU's backward bridge once its parameter-gradient kernels have been issued: every
        gradient of the early group is now in flight on the parameter side streams."""
        dev = self.x.device
        cs = self._comm_stream
        cs.wait_stream(torch.cuda.current_stream(dev))
        for st in F._param_stream_list(dev):
            cs.wait_stream(st)
        with torch.cuda.stream(cs):
            dist.all_reduce(self.bucket.early, op=dist.ReduceOp.AVG)
        self._early_work = cs

    def _fwd_bwd(self):
        self.opt.zero_grad(set_to_none=True)
        dev = self.x.device
        hooked = self.bucket is not None
        if hooked:
            F._grad_sinks[dev] = self.bucket.sinks
            if self.overlap_comm and self.capture_comm and self.pipeline == 1:
                F._after_encoder_bwd[dev] = self._reduce_early
        self._early_work = None
        try:
            if self.pipeline == 1:
                preds, recons = self.model(self.x)
            else:
                preds, recons = self._forward_pipelined()
            fl, rl = rmse_losses(self.x, self.y, preds, recons, self.target_dims)
            (fl + rl).backward()
            if self.pipeline > 1:
                main = [p.grad for p in self.params]
                for al in self._alias:
                    torch._foreach_add_(main, [al[nm].grad for nm in self._names])
        finally:
            if hooked:
                F._grad_sinks.pop(dev, None)
                F._after_encoder_bwd.pop(dev, None)
        self.losses[0].copy_(fl.detach())
        self.losses[1].copy_(rl.detach())

    def _forward_pipelined(self):
        cur = torch.cuda.current_stream(self.x.device)
        B = self.x.shape[0]
        per = (B // self.pipeline + 15) // 16 * 16
        outs = []
        for i, st in enumerate(self._pipe_streams):
            lo, hi = i * per, (B if i == self.pipeline - 1 else (i + 1) * per)
            st.wait_stream(cur)
            with torch.cuda.stream(st):
                xi = self.x[lo:hi]
                if i == 0:
                    o = self.model(xi)
                else:
                    for a in self._alias[i - 1].values():
                        a.grad = None
                    o = torch.func.functional_call(self.model, self._alias[i - 1], (xi,))
            outs.append(o)
        for st, o in zip(self._pipe_streams, outs):
            cur.wait_stream(st)
            o[0].record_stream(cur); o[1].record_stream(cur)
        return torch.cat([o[0] for o in outs]), torch.cat([o[1] for o in outs])

    def _allreduce(self):
        if self.world == 1:
            return
        if self.bucket is not None and getattr(self, "_adopted", None) is None:
            self._adopted = self.bucket.adopted()                 # checked once: the gradient plumbing is static
        if self.bucket is None or not self._adopted:
            allreduce_gradients(self.params, self.world)          # generic path (gloo, or views not adopted)
            if self._early_work is not None:
                torch.cuda.current_stream().wait_stream(self._early_work)
            return
        if self._early_work is None:
            dist.all_reduce(self.bucket.flat, op=dist.ReduceOp.AVG)
        else:
            dist.all_reduce(self.bucket.late, op=dist.ReduceOp.AVG)
            torch.cuda.current_stream().wait_stream(self._early_work)

    def _snapshot(self):
        seed = F.seed_state(self.x.device)
        return ([p.detach().clone() for p in self.params],
                {id(p): {k: (v.clone() if torch.is_tensor(v) else v) for k, v in self.opt.state.get(p, {}).items()}
                 for p in self.params},
                None if seed is None else seed.clone())

    def _restore(self, snap):
        """Undo the warm-up steps IN PLACE (a capture holds the addresses of parameters, optimizer state and seed)."""
        ps, st, seed = snap
        with torch.no_grad():
            for p, q in zip(self.params, ps):
                p.copy_(q)
            for p in self.params:
                cur, old = self.opt.state.get(p, {}), st[id(p)]
                for k, v in cur.items():
                    if torch.is_tensor(v):
                        if k in old:
                            v.copy_(old[k])
                        else:
                            v.zero_()                     # state created by the warm-up: back to its initial value
            now = F.seed_state(self.x.device)
            if now is not None:
                if seed is not None:
                    now.copy_(seed)
                elif self._seed0 is not None:
                    now.fill_(self._seed0)

    def _capture(self):
        # warm-up and capture on the SAME stream: the library's GEMM pack workspaces are per stream and cannot grow
        # during capture (include/mtadgat.h: mtadgat_workspace_reserve).  The warm-up steps are undone afterwards:
        # the first run_* call performs exactly one optimisation step.
        self._seed0 = torch.initial_seed() & 0x7FFFFFFFFFFFFFFF
        snap = self._snapshot()
        s = torch.cuda.Stream()
        s.wait_stream(torch.cuda.current_stream())
        with torch.cuda.stream(s):
            for _ in range(3):
                self._fwd_bwd(); self._allreduce(); self.opt.step()
        torch.cuda.current_stream().wait_stream(s)
        torch.cuda.synchronize()
        self._restore(snap)
        torch.cuda.synchronize()
        F.reset_launch_count()
        one_graph = self.world == 1 or (self.capture_comm and self.bucket is not None)
        if one_graph:
            self.g_fb = torch.cuda.CUDAGraph()
            with torch.cuda.graph(self.g_fb, stream=s):
                self._fwd_bwd()
                self._allreduce()
                self.opt.step()
        else:
            self.g_fb = torch.cuda.CUDAGraph()
            with torch.cuda.graph(self.g_fb, stream=s):
                self._fwd_bwd()
            self.g_opt = torch.cuda.CUDAGraph()
            with torch.cuda.graph(self.g_opt, stream=s):
                self.opt.step()
        self.launches_per_step = F.launch_count()

    def release(self):
        """Drop the captured graphs (call before torch.distributed.destroy_process_group: a graph that captured a
        collective keeps communicator resources alive)."""
        self.g_fb = self.g_opt = None

    def _run(self):
        if not self.use_graph:
            self._fwd_bwd(); self._allreduce(); self.opt.step()
            return
        if self.g_fb is None:
            self._capture()
        self.g_fb.replay()
        if self.g_opt is not None:
            self._allreduce()
            self.g_opt.replay()

    # -- public ------------------------------------------------------------------------------------------
    def run_device(self, x, y):
        """x (B,n,k), y (B,1,k) already on the device."""
        self.x.copy_(x); self.y.copy_(y)
        self._run()

    def prefetch_host(self, x_host, y_host):
        """Start the H2D copy of a pinned host batch on the copy stream (call before run_prefetched)."""
        slot = self._put & 1
        sx, sy = self._stage[slot]
        cs = self._copy_stream
        cs.wait_stream(torch.cuda.current_stream())      # the step that last read this slot has been enqueued
        with torch.cuda.stream(cs):
            sx.copy_(x_host, non_blocking=True); sy.copy_(y_host, non_blocking=True)
            ev = torch.cuda.Event(); ev.record(cs)
        self._staged[slot] = ev
        self._put += 1

    def run_prefetched(self):
        """Run the step on the oldest prefetched batch; returns the scalar loss (D2H)."""
        slot = self._get & 1
        self._get += 1
        torch.cuda.current_stream().wait_event(self._staged[slot])
        sx, sy = self._stage[slot]
        self.x.copy_(sx); self.y.copy_(sy)
        self._run()
        fl, rl = self.losses.tolist()
        return fl + rl

    def launch_prefetched(self):
        """Enqueue the step on the oldest prefetched batch plus an asynchronous D2H copy of its two loss terms into
        pinned host memory, without waiting: the host can enqueue step i+1 while step i runs.  collect() returns the
        losses in launch order."""
        slot = self._get & 1
        self._get += 1
        torch.cuda.current_stream().wait_event(self._staged[slot])
        sx, sy = self._stage[slot]
        self.x.copy_(sx); self.y.copy_(sy)
        self._run()
        if not hasattr(self, "_loss_host"):
            self._loss_host = [torch.zeros(2, dtype=torch.float32).pin_memory() for _ in range(2)]
            self._loss_ev = [None, None]
            self._lput = self._lget = 0
        k = self._lput & 1
        self._lput += 1
        self._loss_host[k].copy_(self.losses, non_blocking=True)
        ev = torch.cuda.Event(); ev.record()
        self._loss_ev[k] = ev

    def collect(self):
        """Scalar loss of the oldest launched-but-uncollected step (waits for that step only)."""
        k = self._lget & 1
        self._lget += 1
        self._loss_ev[k].synchronize()
        v = self._loss_host[k]
        return float(v[0]) + float(v[1])

    def run_host(self, x_host, y_host):
        """Pinned host batch in, scalar loss out (H2D + step + D2H)."""
        self.x.copy_(x_host, non_blocking=True); self.y.copy_(y_host, non_blocking=True)
        self._run()
        fl, rl = self.losses.tolist()
        return fl + rl
