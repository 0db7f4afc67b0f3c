"""2-rank NCCL test of the REAL model: windows
shard over the batch, the backward kernels write into the flat GradBucket, one all-reduce averages it in place, and the
result equals the mean of the per-shard oracle gradients; the graph step (fwd/bwd graph, eager collective, Adam graph)
keeps the replicas bit-identical and agrees with the eager step.  Needs 2 GPUs (gpurun --gpus 2); skipped otherwise."""
import os

import numpy as np
import pytest
import torch
import torch.distributed as dist
import torch.multiprocessing as mp

pytestmark = pytest.mark.gpu

KW = dict(n_features=38, window_size=100, out_dim=38, forecast_n_layers=3, dropout=0.0)


def _worker(rank, world, port, ret):
    os.environ.update(MASTER_ADDR="127.0.0.1", MASTER_PORT=str(port), RANK=str(rank), WORLD_SIZE=str(world),
                      LOCAL_RANK=str(rank))
    torch.cuda.set_device(rank)
    dev = torch.device("cuda", rank)
    dist.init_process_group("nccl", rank=rank, world_size=world, device_id=dev)
    import mtad_gat_pytorch_b200 as mg
    from mtad_gat_pytorch_b200 import training as mgt
    from oracle import mtad_gat_oracle as orc
    cfg = orc.Config(**KW)
    params = orc.make_params(cfg, seed=80, dtype=np.float64)
    Bg = 16
    rng = np.random.default_rng(80)
    X, Y = rng.random((Bg, cfg.n, cfg.k)), rng.random((Bg, 1, cfg.k))
    lo, hi = mgt.shard_batch(Bg, world, rank)
    xd = torch.from_numpy(X[lo:hi].astype(np.float32)).to(dev)
    yd = torch.from_numpy(Y[lo:hi].astype(np.float32)).to(dev)

    def fresh():
        m = mg.MTAD_GAT(**KW)
        m.load_state_dict({k: torch.from_numpy(v.astype(np.float32)) for k, v in params.items()})
        return m.to(dev).train()

    out = {}
    # (1) eager: gradients after the bucket all-reduce == mean over ranks of the per-shard oracle gradients (fp32 kernels:
    #     this checks the data-parallel plumbing, not the tensor-core arithmetic)
    mg.set_mode("fp32")
    m = fresh()
    opt = torch.optim.Adam(m.parameters(), lr=1e-3, capturable=True, fused=True)
    step = mgt.TrainStep(m, opt, batch=hi - lo, use_graph=False, world_size=world)
    step.x.copy_(xd); step.y.copy_(yd)
    step._fwd_bwd(); step._allreduce()
    torch.cuda.synchronize()
    out["adopted"] = bool(step.bucket.adopted())
    g_mean = None
    for r in range(world):
        a, b = mgt.shard_batch(Bg, world, r)
        g = orc.loss_fwd_bwd(X[a:b], Y[a:b], params, cfg)[6]
        g_mean = g if g_mean is None else {k: g_mean[k] + g[k] for k in g}
    errs = {}
    for name, p in m.named_parameters():
        ref = g_mean[name] / world
        errs[name] = float(np.abs(p.grad.cpu().numpy() - ref).max() / max(np.abs(ref).max(), 1e-9))
    out["grad_err"] = max(errs.values())
    mg.set_mode("tc")
    # (2) three optimisation steps: graph step vs eager step
    finals = {}
    variants = [("graph", dict(use_graph=True)), ("eager", dict(use_graph=False))]
    if os.environ.get("MTADGAT_TEST_CAPTURED_COMM"):       # opt-in: collectives captured into the step graph
        variants.append(("graph_captured", dict(use_graph=True, capture_comm=True)))
    for tag, kw in variants:
        m = fresh()
        opt = torch.optim.Adam(m.parameters(), lr=1e-3, capturable=True, fused=True)
        step = mgt.TrainStep(m, opt, batch=hi - lo, world_size=world, **kw)
        for _ in range(3):
            step.run_device(xd, yd)
        torch.cuda.synchronize()
        flat = torch.cat([p.detach().reshape(-1) for p in m.parameters()])
        others = [torch.empty_like(flat) for _ in range(world)]
        dist.all_gather(others, flat)
        out[tag + "_replicas_equal"] = all(torch.equal(o, others[0]) for o in others)
        finals[tag] = flat
        if tag == "graph":
            out["two_graphs"] = step.g_opt is not None and step.g_fb is not None
        step.release()
    upd = float((finals["eager"] - torch.cat([torch.from_numpy(params[k].astype(np.float32)).reshape(-1)
                                               for k, _ in m.named_parameters()]).to(dev)).norm())
    out["graph_vs_eager"] = float((finals["graph"] - finals["eager"]).norm()) / upd
    if "graph_captured" in finals:
        out["captured_vs_eager"] = float((finals["graph_captured"] - finals["eager"]).norm()) / upd
    ret[rank] = out
    torch.cuda.synchronize()
    os._exit(0)            # results are with the parent; skip communicator teardown (it can block on exit ordering)


def test_two_rank_nccl_model_gradients_and_one_graph_step():
    if not torch.cuda.is_available() or torch.cuda.device_count() < 2:
        pytest.skip("needs 2 GPUs")
    mgr = mp.Manager()
    ret = mgr.dict()
    port = 29500 + os.getpid() % 400
    ctx = mp.spawn(_worker, args=(2, port, ret), nprocs=2, join=False)
    import time
    t0 = time.time()
    while not ctx.join(timeout=5):
        if time.time() - t0 > 240:
            for p in ctx.processes:
                p.kill()
            pytest.fail(f"workers did not finish in 240 s; partial results {dict(ret)}")
    assert len(ret) == 2
    for rank, out in ret.items():
        print(f"[nccl rank {rank}] {out}")
        assert out["adopted"], "gradient views were not adopted by autograd: the bucket path is not in use"
        assert out["grad_err"] < 1e-3, out
        assert out["two_graphs"]
        assert out["graph_replicas_equal"] and out["eager_replicas_equal"]
        assert out["graph_vs_eager"] < 0.05 and out.get("captured_vs_eager", 0.0) < 0.05, out
