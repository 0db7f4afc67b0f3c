"""Batches of more than 65 535 windows.  CUDA stops gridDim.y and gridDim.z at 65 535, and several launches put the window
index there: the tiled GAT score kernel and gat_bwd1_kernel (y), the two-pass gat_bwd2_kernel and the batched GEMMs of
the GAT projection and dV products (z).  They launch the windows in chunks of at most 65 535 (DESIGN §4).  Here
B = 65 573, so a chunk boundary falls inside the batch, and windows 65 534 .. 65 536 and B - 1 sit on either side of it.

* GAT entry points (mtadgat_gat_fwd / _bwd) against the float64 reference of tests/gat_reference.py on the kernel's own
  LeakyReLU branches, with the gates of tests/test_gpu_gat.py, at every batch-dependent launch: win and tiled forward,
  bwd1<4> and bwd1<2>, bwd2_win and two-pass bwd2, tensor-core and SIMT projection and dV GEMMs, GATv1 and GATv2,
  training with dropout and inference.  Outputs, `saved` and `scratch` start as NaN.  The sampled windows run alone
  give bitwise the same out and dx.  Parameter gradients (sums over all windows) against float64 over the whole batch.
* The model (MTAD_GAT) at B = 65 573, one config on the whole-window GAT kernels and one with a tiled feature layer:
  eval forward and dx against the float64 oracle (oracle/mtad_gat_oracle.py); the parameter gradients equal the sum of
  those of windows [0, 65 535) and [65 535, B) run as two batches.
* SeriesScorer with 65 573-window chunks equals 4 096-window chunks bit for bit.
* Dispatch: torch.profiler's launches and grids against the launch counts gat_reference.expected_paths and
  gemm_reference.expected_paths state.

The K = 129 / 130 cases repeat their windows with period 1 000, which keeps their float64 reference affordable: every
window still runs through the kernels, the layer's parameter-gradient reference over the whole batch is that of the
first 1 000 windows weighted by how often each occurs (the gradients are linear in the upstream gradient), and the
layer's outputs must repeat bitwise with the same period.  65 535 is not a
multiple of 1 000, so a launch that read the wrong chunk of windows would not reproduce the pattern."""
import copy
import os
import re
import subprocess
import sys

import numpy as np
import pytest
import torch

from oracle import mtad_gat_oracle as orc
from tests import gat_reference as gr
from tests import gemm_reference as gm
from tests import oracle_tools as ot
from tests.test_gpu_gat import FWD_GATE, GATE, SLOPE_GATE, Layer, _np

pytestmark = pytest.mark.gpu
MODES = ["tc", "fp32"]
LIMIT = 65535                     # CUDA's gridDim.y / gridDim.z limit
B = LIMIT + 38                    # 65 573
TOL = 1e-3                        # the model-level parity gate (tests/test_gpu_parity.py)
CHUNK = 4096                      # windows per float64 reference call


@pytest.fixture(autouse=True)
def _default_mode():
    import mtad_gat_pytorch_b200 as mg
    mg.set_mode("tc")
    yield
    mg.set_mode("tc")
    torch.cuda.empty_cache()


def sample_windows(seed):
    """0, the windows around the chunk boundary, the last one and a random sample"""
    rng = np.random.default_rng(seed)
    return sorted({0, LIMIT - 1, LIMIT, LIMIT + 1, B - 1} | set(rng.choice(B, 6, replace=False).tolist()))


def repeat_index(period):
    return np.arange(B) % period


def weights(period):
    """how often each of the first `period` windows occurs in a batch of B windows that repeats with that period"""
    return np.bincount(repeat_index(period), minlength=period).astype(np.float64)


# ---- GAT entry points -----------------------------------------------------------------------------------------------
# (layer, v2, n, k, E, p, period)
GAT_CASES = [
    ("temporal", True, 16, 32, 8, 0.3, None),   # win, bwd1<2>, bwd2_win; tensor-core projection, dV and parameter GEMMs
                                                # under tc; training with dropout
    ("feature", False, 8, 12, 8, 0.0, None),    # GATv1, win; K = 12 < 16: SIMT projection and dV GEMMs
    ("feature", True, 4, 130, 1, 0.0, 1000),    # K = 130: tiled forward (rows split), bwd1<4>, two-pass bwd2; D = 4: SIMT
]


def gat_id(c):
    return f"{c[0][:4]}-v{2 if c[1] else 1}-n{c[2]}-k{c[3]}-E{c[4]}-p{c[5]}"


def make_layer(case, seed):
    layer, v2, n, k, E, p, period = case
    L = Layer(layer, v2, n, k, E, B, seed, p=p)
    if period:
        rep = torch.from_numpy(repeat_index(period)).cuda()
        L.x, L.gout = L.x[:period][rep].contiguous(), L.gout[:period][rep].contiguous()
    return L


def saved_parts(L, saved):
    """meta (host int32), pqt (B,NC,Kp) and att (B,K,Kp) views of a device `saved` buffer"""
    lay = gr.saved_layout(L.B, L.n, L.k, L.E, L.feature, L.v2)
    meta = _np(saved[lay["meta"]:lay["meta"] + 2 * L.E + 4]).view(np.int32)
    pqt = saved[lay["pqt"]:lay["att"]].view(L.B, L.NC, L.Kp)
    att = saved[lay["att"]:lay["total"]].view(L.B, L.K, L.Kp)
    return meta, pqt, att


def gat_reference(L, meta, pqt, windows, period):
    """float64 forward and backward on the kernel's slope decisions, CHUNK windows at a time: the reference's out, att
    and dx at `windows`, the parameter gradients summed over the whole batch, and the largest slope disagreement."""
    q = {key: None if v is None else v.astype(np.float64) for key, v in L.np.items() if key != "x"}
    mask = L.mask()
    rows = period or L.B
    wt = weights(period) if period else None
    at = {w: (w % period if period else w) for w in windows}
    ref = {"out": {}, "att": {}, "dx": {}}
    sums = {}
    worst = 0.0
    for lo in range(0, rows, CHUNK):
        hi = min(rows, lo + CHUNK)
        x = L.np["x"][lo:hi].astype(np.float64)
        slope, stats = gr.align_slopes(_np(pqt[lo:hi]), meta, x, q["lin_w"], q["lin_b"], q["a"], L.feature, L.v2)
        worst = max(worst, float(stats["worst_rel_z"].max()))
        out, cache = gr.gat_fwd(x, q["lin_w"], q["lin_b"], q["a"], q["bias"], L.alpha, L.feature, L.v2,
                                mask=None if mask is None else mask[lo:hi], slope=slope)
        gout = _np(L.gout[lo:hi]).astype(np.float64)
        res = gr.gat_bwd(gout, cache)
        dx = res[0]
        if wt is not None:                  # the weighted upstream gradient gives the whole batch's parameter sums
            res = gr.gat_bwd(gout * wt[lo:hi, None, None], cache)
        _, dlin_w, dlin_b, da, dbias = res
        for name, v in (("dlin_w", dlin_w), ("dlin_b", dlin_b), ("da", da.reshape(-1, 1)), ("dbias", dbias)):
            if v is not None:
                sums[name] = sums.get(name, 0.0) + v
        for w, r in at.items():
            if lo <= r < hi:
                ref["out"][w], ref["att"][w], ref["dx"][w] = out[r - lo], cache["att"][r - lo], dx[r - lo]
    return {key: np.stack([v[w] for w in windows]) for key, v in ref.items()}, sums, worst


@pytest.mark.parametrize("mode", MODES)
@pytest.mark.parametrize("case", GAT_CASES, ids=gat_id)
def test_gat_layer_past_65535_windows(case, mode):
    import mtad_gat_pytorch_b200 as mg
    mg.set_mode(mode)
    layer, v2, n, k, E, p, period = case
    L = make_layer(case, seed=n + k)
    windows = sample_windows(n + k)
    out, saved = L.fwd()
    g = L.bwd(out, saved)
    assert bool(torch.isfinite(out).all()) and bool(torch.isfinite(g["dx"]).all()), "unwritten outputs"
    meta, pqt, att = saved_parts(L, saved)
    if period:
        rep = torch.from_numpy(repeat_index(period)).cuda()
        for name, t in (("pqt", pqt[:, :, :L.K]), ("out", out), ("dx", g["dx"])):
            assert torch.equal(t, t[:period][rep]), f"{name} does not repeat with the windows"
    ref, sums, worst = gat_reference(L, meta, pqt, windows, period)
    got = {"out": _np(out[windows]), "att": _np(att[windows])[:, :, :L.K], "dx": _np(g["dx"][windows])}
    bad, line = [], []
    for name, gate in (("out", FWD_GATE), ("att", FWD_GATE), ("dx", GATE[mode])):
        e = ot.window_errors(got[name], ref[name])
        line.append(f"{name} {np.max(e):.1e}")
        if not np.all(e < gate):
            bad.append((name, windows[int(np.argmax(np.where(np.isfinite(e), e, np.inf)))], float(np.max(e))))
    for name, r in sums.items():
        # lin.bias is the bias column of the affine map [lin.weight | lin.bias]: its error is measured on the map's
        # scale.  Alone it is a sum over B * K * K terms whose softmax-gradient rows add to zero, which cancels to
        # ~1e-3 of that scale at B = 65 573
        scale = max(np.abs(r).max(), np.abs(sums["dlin_w"]).max() if name == "dlin_b" else 0.0, 1e-300)
        e = float(np.abs(_np(g[name]).astype(np.float64) - r).max() / scale)
        line.append(f"{name} {e:.1e}")
        if not e < GATE[mode]:
            bad.append((name, e))
    print(f"[{mode} {gat_id(case)} B={B}] worst per window over {windows}: " + ", ".join(line) +
          f" | worst slope disagreement |z| {worst:.1e} of the window max")
    if not worst <= SLOPE_GATE:
        bad.append(("slope", worst))
    # the sampled windows alone: inference forward, and (without dropout) the training forward and backward
    unequal = []
    out0 = L.fwd(training=0)[0] if p > 0 else out
    for w in windows:
        one = copy.copy(L)
        one.B, one.x, one.gout = 1, L.x[w:w + 1].clone(), L.gout[w:w + 1].clone()
        if not torch.equal(one.fwd(training=0)[0][0], out0[w]):
            unequal.append(("inference out", w))
        if p == 0:
            o1, s1 = one.fwd()
            if not torch.equal(o1[0], out[w]):
                unequal.append(("out", w))
            if not torch.equal(one.bwd(o1, s1)["dx"][0], g["dx"][w]):
                unequal.append(("dx", w))
    assert not bad and not unequal, (bad, unequal)


# ---- the model --------------------------------------------------------------------------------------------------------
SMALL = dict(gru_hid_dim=16, forecast_hid_dim=16, recon_hid_dim=16)
# name -> (MTAD_GAT arguments, period of the windows or None)
MODEL_CFGS = {
    "win": (dict(n_features=5, window_size=8, out_dim=5, **SMALL), None),
    # feature layer K = 129 nodes: tiled score kernel with its rows split over two CTAs, two-pass bwd2
    "tiled": (dict(n_features=129, window_size=4, out_dim=129, feat_gat_embed_dim=1, time_gat_embed_dim=1, **SMALL),
              1000),
}
_ORACLE = {}


def model_case(name):
    """(params, x, upstream gradients of preds and recons, sampled windows, float64 reference), the reference computed
    once for both modes: preds, recons and dx at the sampled windows."""
    if name in _ORACLE:
        return _ORACLE[name]
    kwargs, period = MODEL_CFGS[name]
    cfg = orc.Config(**kwargs)
    params = orc.make_params(cfg, seed=70, dtype=np.float32)
    p64 = {key: v.astype(np.float64) for key, v in params.items()}
    windows = sample_windows(72)
    at = {w: (w % period if period else w) for w in windows}
    rows = period or max(at.values()) + 1
    rng = np.random.default_rng(71)
    x = rng.random((rows, cfg.n, cfg.k)).astype(np.float32)
    gp = rng.standard_normal((rows, cfg.out_dim)).astype(np.float32)
    grc = rng.standard_normal((rows, cfg.n, cfg.out_dim)).astype(np.float32)
    if not period:                                  # independent windows: the rest of the batch
        x = np.concatenate([x, rng.random((B - rows, cfg.n, cfg.k)).astype(np.float32)])
        gp = np.concatenate([gp, rng.standard_normal((B - rows, cfg.out_dim)).astype(np.float32)])
        grc = np.concatenate([grc, rng.standard_normal((B - rows, cfg.n, cfg.out_dim)).astype(np.float32)])
    idx = np.array(sorted(set(at.values())))
    preds, recons, cache = orc.model_fwd(x[idx].astype(np.float64), p64, cfg)
    dx, _ = orc.model_bwd(gp[idx].astype(np.float64), grc[idx].astype(np.float64), cache, p64, cfg)
    pos = {r: i for i, r in enumerate(idx)}
    ref = {key: np.stack([v[pos[at[w]]] for w in windows]) for key, v in (("preds", preds), ("recons", recons),
                                                                            ("dx", dx))}
    if period:
        rep = repeat_index(period)
        x, gp, grc = x[rep], gp[rep], grc[rep]
    _ORACLE[name] = (kwargs, params, x, gp, grc, windows, ref)
    return _ORACLE[name]


def build(kwargs, params):
    import mtad_gat_pytorch_b200 as mg
    m = mg.MTAD_GAT(**kwargs)
    m.load_state_dict({key: torch.from_numpy(np.asarray(v, dtype=np.float32)) for key, v in params.items()}, strict=True)
    return m.cuda().eval()


@pytest.mark.parametrize("mode", MODES)
@pytest.mark.parametrize("cfg", list(MODEL_CFGS))
def test_model_past_65535_windows(cfg, mode):
    """Eval forward: preds and recons of the sampled windows against float64 and bitwise equal to the window run alone.
    Backward with fixed upstream gradients: dx of the sampled windows against float64, and every parameter gradient
    equal to the sum of those of the two batches [0, 65 535) and [65 535, B).  A float64 sum over the whole batch is no
    measure here: with random-sign upstream gradients the sums cancel to ~sqrt(B) of one window's contribution, so one
    ReLU / LeakyReLU branch that the kernels take differently from float64 moves them by ~1/sqrt(B) = 4e-3 (the layer
    tests compare such sums on the kernel's own branches).  dx is not compared with the window run alone: the fp16 BPTT
    scale comes from the whole batch's gradient maximum, as it does for the two batches (hence the tc gate)."""
    import mtad_gat_pytorch_b200 as mg
    mg.set_mode(mode)
    kwargs, params, x, gp, grc, windows, ref = model_case(cfg)
    m = build(kwargs, params)
    xt = torch.from_numpy(x).cuda()
    with torch.no_grad():
        preds, recons = m(xt)
        alone = [m(xt[w:w + 1].contiguous()) for w in windows]
    assert bool(torch.isfinite(preds).all()) and bool(torch.isfinite(recons).all()), "unwritten outputs"
    unequal = [w for w, (p1, r1) in zip(windows, alone) if not (torch.equal(p1[0], preds[w]) and
                                                               torch.equal(r1[0], recons[w]))]
    errs = {"preds": float(np.max(ot.window_errors(_np(preds[windows]), ref["preds"]))),
            "recons": float(np.max(ot.window_errors(_np(recons[windows]), ref["recons"])))}
    gpt, grt = torch.from_numpy(gp).cuda(), torch.from_numpy(grc).cuda()

    def grads(sl):
        m.zero_grad(set_to_none=True)
        xs = xt[sl].clone().requires_grad_(True)
        p, r = m(xs)
        torch.autograd.backward([p, r], [gpt[sl].contiguous(), grt[sl].contiguous()])
        return {name: prm.grad.clone() for name, prm in m.named_parameters()}, xs.grad
    full, dx = grads(slice(0, B))
    assert bool(torch.isfinite(dx).all()), "unwritten dx"
    errs["dx"] = float(np.max(ot.window_errors(_np(dx[windows]), ref["dx"])))
    del dx
    ga, gb = grads(slice(0, LIMIT))[0], grads(slice(LIMIT, B))[0]
    perr = {}
    for name, f in full.items():
        a_, b_ = _np(ga[name]).astype(np.float64), _np(gb[name]).astype(np.float64)
        # on the scale of the two summands, and a GAT lin.bias on that of its affine map's lin.weight (as in
        # test_gat_layer_past_65535_windows): its per-window terms cancel, so the sum is far below its terms
        w = name.replace("lin.bias", "lin.weight")
        scale = max(np.abs(a_ + b_).max(), (np.abs(a_) + np.abs(b_)).max(), 1e-300,
                    np.abs(_np(ga[w]).astype(np.float64) + _np(gb[w])).max() if w != name else 0.0)
        perr["grad." + name] = float(np.abs(_np(f) - (a_ + b_)).max() / scale)
    worst = max(perr, key=perr.get)
    print(f"[model {cfg} {mode} B={B}] windows {windows}: preds {errs['preds']:.1e} recons {errs['recons']:.1e} "
          f"dx {errs['dx']:.1e}; parameter gradients against the two batches: worst {worst} {perr[worst]:.1e}")
    split_gate = TOL if mode == "tc" else 1e-4      # fp32: tests/test_gpu_parity.py's split-batch gate
    bad = {key: e for key, e in errs.items() if not e < TOL}
    bad.update({key: e for key, e in perr.items() if not e < split_gate})
    assert not bad and not unequal, (bad, unequal)


# ---- scoring ----------------------------------------------------------------------------------------------------------
def test_series_scorer_past_65535_windows():
    """A 70 000-row series scored in chunks of 65 573 windows (CUDA graph and eager) and of 4 096: forecast, recon,
    a_score and a_global bitwise equal (no forward reduction order depends on the window count)."""
    from mtad_gat_pytorch_b200.scoring import SeriesScorer
    kwargs = MODEL_CFGS["win"][0]
    m = build(kwargs, orc.make_params(orc.Config(**kwargs), seed=73, dtype=np.float32))
    g = torch.Generator(device="cuda").manual_seed(73)
    series = torch.rand(70000, kwargs["n_features"], generator=g, device="cuda")
    want = SeriesScorer(m, batch=4096).score(series)
    keys = ("forecast", "recon", "a_score", "a_global")
    for use_graph in (True, False):
        got = SeriesScorer(m, batch=B, use_graph=use_graph).score(series)
        unequal = [key for key in keys if not torch.equal(got[key], want[key])]
        assert not unequal, (use_graph, unequal)
    assert bool(torch.isfinite(want["a_score"]).all())


# ---- dispatch, measured -----------------------------------------------------------------------------------------------
def _launch_key(name):
    """(key of gat_reference.expected_paths()["launches"], grid axis holding the windows) of a kernel, None otherwise"""
    if "gat_score_win_kernel" in name:
        return "fwd", 0
    if "gat_score_fwd_kernel" in name:
        return "fwd", 1
    if "gat_bwd1_kernel" in name:
        return "bwd1", 1
    if "gat_bwd2_win_kernel" in name:
        return "bwd2", 0
    if "gat_bwd2_kernel" in name:
        return "bwd2", 2
    if "gemm2_kernel<" in name or re.search(r"(?<![\w])gemm_kernel<", name):
        if "StPQt" in name:
            return "proj", 2
        if "StNodeAcc" in name or "StNodeT" in name:
            return "dv", 2
    return None


def measure_launches(L, mode, case):
    """One profiled forward + backward of layer L: the list of disagreements with the stated launches (empty = all
    agree).  Printed one line per measurement."""
    from tests.test_gpu_gemm_stages import traced
    layer, v2, n, k, E, p, _ = case
    bad, counts, cover, first = [], {}, {}, {}
    for name, grid, cat in traced(lambda: L.bwd(*L.fwd())):
        key = _launch_key(name) if cat == "kernel" else None
        if key is None:
            continue
        key, axis = key
        counts[key] = counts.get(key, 0) + 1
        cover[key] = cover.get(key, 0) + grid[axis]
        first.setdefault(key, grid)
        if axis > 0 and grid[axis] > LIMIT:
            bad.append((mode, gat_id(case), key, grid))
    exp = gr.expected_paths(layer, v2, n, k, E, mode, B)
    el = dict(exp["launches"])
    el["dv"] = el.pop("dv1") + el.pop("dv2")
    passes = {"bwd2": 1 if exp["bwd2"] == "bwd2_win" else 2, "dv": 2}
    want_cover = {key: B * passes.get(key, 1) for key in el}
    K, D, _, NC, _ = gr.dims(n, k, E, layer == "feature", v2)
    proj = gm.expected_paths("precise", NC, K, D, mode, B)
    print(f"[dispatch {mode} {gat_id(case)} B={B}] launches {counts} windows covered {cover} "
          f"projection first grid {first.get('proj')}")
    if counts != el or cover != want_cover:
        bad.append((mode, gat_id(case), counts, el, cover, want_cover))
    if tuple(first.get("proj", ())) != proj["grid"] or counts.get("proj") != proj["launches"]:
        bad.append((mode, gat_id(case), "proj", first.get("proj"), proj["grid"], proj["launches"]))
    return bad


def dispatch_past_limit():
    """The batch-dependent launches of a GAT forward + backward at B = 65 573 (torch.profiler): launch counts against
    gat_reference.expected_paths, the projection GEMM's first grid against gemm_reference.expected_paths, no launch
    with more than 65 535 windows on its axis, and every window covered once per pass.  A case that disagrees is
    measured again, up to three times in all: the launches are a deterministic function of the shapes, so a wrong
    dispatch disagrees every time, while a profiler session on a shared GPU can drop events (tests/test_gpu_gemm_stages.py
    `traced`)."""
    import mtad_gat_pytorch_b200 as mg
    bad = []
    for mode in MODES:
        mg.set_mode(mode)
        for case in (GAT_CASES[0], GAT_CASES[2]):
            L = make_layer(case, seed=1)
            for _ in range(3):
                got = measure_launches(L, mode, case)
                if not got:
                    break
            bad += got
            del L
            torch.cuda.empty_cache()
    assert not bad, bad


def test_dispatch_past_65535_windows():
    """dispatch_past_limit() in a child process, as tests/test_gpu_gat.py::test_dispatch_table"""
    root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    code = "from tests.test_gpu_batch_limits import dispatch_past_limit; dispatch_past_limit()"
    r = subprocess.run([sys.executable, "-c", code], cwd=root, capture_output=True, text=True, timeout=900)
    print(r.stdout)
    assert r.returncode == 0, r.stdout[-3000:] + r.stderr[-3000:]
