"""The GAT layer entry points (mtadgat_gat_fwd / mtadgat_gat_bwd, csrc/gat.cu) called directly, against the factored
float64 reference of tests/gat_reference.py, at every dispatch path of the forward, the backward and the GEMMs they
issue, under `set_mode("tc")` and `set_mode("fp32")`.

* `saved`, `scratch`, `out` and `dx` are filled with NaN before every call, so a kernel that reads a padding column or
  slot it never wrote gives a non-finite result.
* LeakyReLU slopes: the backward recomputes the branch of each of the K*K*E pre-activations from the saved fp32 P + Q.
  The reference is evaluated on those branches (gat_reference.align_slopes) and the disagreement with its own z > 0 is
  bounded separately: every differing decision has |z| <= 1e-5 of its window's max |z|.
* Errors are per window (max |err| / max |ref| of the window, oracle_tools.window_errors): forward output and saved
  attention 2e-4 in both modes (fp32 arithmetic, three-term projection operands), dx 1e-3 under `tc` (two-term dV
  products) and 2e-4 under `fp32`.  Parameter gradients (lin.weight, lin.bias, a, bias) are sums over windows: the
  same two gates, tensor-wide.
* Bitwise: training=0 == training=1 at p=0; a window's forward in a batch of 17 == that window alone; the split
  backward (parts 9, then 2 on a second stream, then 4) == parts=3; two backward runs are equal."""
import re

import numpy as np
import pytest
import torch

from tests import gat_reference as gr
from tests import oracle_tools as ot

pytestmark = pytest.mark.gpu
MODES = ["tc", "fp32"]
FWD_GATE = 2e-4
GATE = {"tc": 1e-3, "fp32": 2e-4}
SLOPE_GATE = 1e-5

# (layer, use_gatv2, n, k, E, B): together they reach every path of gat_reference.expected_paths (test_dispatch_table)
CASES = [
    ("temporal", True, 100, 38, 76, 3),     # C2 temporal: win<4,10>, bwd1<4>, bwd2_win, tensor-core split-K
    ("feature", True, 100, 38, 200, 17),    # C2 feature: win<2,4>, bwd1<2>, transposed dV
    ("feature", True, 100, 55, 48, 3),      # win<4,4>
    ("feature", True, 100, 5, 200, 17),     # win<2,2>; K < 16: SIMT projection and dV GEMMs under tc
    ("feature", True, 100, 13, 24, 1),      # K < 16, non-default E
    ("temporal", True, 99, 55, 110, 3),     # tiled<4,4> at K <= 128 (over the window budget), two-pass bwd2
    ("temporal", True, 97, 25, 50, 17),     # D < 32: SIMT split-K weight gradient + dpq_colsum
    ("temporal", True, 97, 5, 10, 3),       # D < 16: SIMT projection and dV GEMMs under tc
    ("temporal", False, 97, 38, 38, 3),     # GATv1 temporal
    ("feature", False, 100, 38, 100, 17),   # GATv1 feature
    ("feature", True, 100, 129, 200, 1),    # K = 129: rows split over CTAs
    ("feature", True, 100, 64, 200, 3),     # tiled<2,4>, transposed dV at K = 64
    ("feature", True, 100, 65, 200, 3),     # K = 65: untransposed dV
    ("temporal", True, 512, 38, 76, 2),     # C5 temporal: tiled<2,4>, JT < K, DT < E
    ("feature", True, 100, 512, 200, 2),    # C4 feature: tiled<4,4>, JT < K, DT < E
    ("temporal", True, 100, 512, 48, 2),    # tiled<2,2>; bwd1 column tile shrunk to 16
]


def case_id(c):
    return f"{c[0][:4]}-v{2 if c[1] else 1}-n{c[2]}-k{c[3]}-E{c[4]}-B{c[5]}"


@pytest.fixture(autouse=True)
def _default_mode():
    import mtad_gat_pytorch_b200 as mg
    mg.set_mode("tc")
    yield
    mg.set_mode("tc")


def _cu(a):
    return None if a is None else torch.from_numpy(np.ascontiguousarray(a, dtype=np.float32)).cuda()


def _np(t):
    return t.detach().cpu().numpy()


def _ptr(t):
    return None if t is None else t.data_ptr()


def _nan(*shape):
    return torch.full(shape, float("nan"), device="cuda")


_SIDE = []


def _side_stream():
    """one second stream for every split backward (the library keeps one workspace per stream)"""
    if not _SIDE:
        _SIDE.append(torch.cuda.Stream())
    return _SIDE[0]


# ---- the entry points -----------------------------------------------------------------------------------------------
class Layer:
    """One GAT layer problem: fp32 inputs on the device and the ABI arguments."""

    def __init__(self, layer, v2, n, k, E, B, seed, a_kind="mixed", alpha=0.2, bias=True, p=0.0, scale0=None):
        self.feature, self.v2, self.n, self.k, self.E, self.B = layer == "feature", v2, n, k, E, B
        self.alpha, self.p = alpha, p
        self.K, self.D, _, self.NC, self.Kp = gr.dims(n, k, E, self.feature, v2)
        rng = np.random.default_rng(seed)
        x = rng.standard_normal((B, n, k)).astype(np.float32)
        if scale0:
            x[0] *= scale0
        D, K = self.D, self.K
        lin_w = (rng.standard_normal((E, 2 * D if v2 else D)) / np.sqrt(D)).astype(np.float32)
        lin_b = (rng.standard_normal(E) * 0.1).astype(np.float32)
        a = rng.standard_normal((E if v2 else 2 * E, 1)) * (2.0 / np.sqrt(E))
        if a_kind == "pos":
            a = np.abs(a)
        elif a_kind == "neg":
            a = -np.abs(a)
        elif a_kind == "zero":
            a[::3] = 0.0
        a = a.astype(np.float32)
        b = (rng.standard_normal((K, K)) * 0.1).astype(np.float32) if bias else None
        self.np = dict(x=x, lin_w=lin_w, lin_b=lin_b, a=a, bias=b)
        self.x, self.lin_w, self.lin_b, self.a, self.bias = (_cu(v) for v in (x, lin_w, lin_b, a, b))
        self.gout = _cu(rng.uniform(-1, 1, (B, n, k)))
        self.seed = torch.tensor([1234 + seed], dtype=torch.int64, device="cuda")

    def fwd(self, training=1, p=None, x=None):
        from mtad_gat_pytorch_b200._lib import lib, check
        p = self.p if p is None else p
        x = self.x if x is None else x
        B = x.shape[0]
        saved = _nan(max(1, lib.mtadgat_gat_saved_floats(B, self.n, self.k, self.E, int(self.feature), int(self.v2),
                                                        training)))
        out = _nan(B, self.n, self.k)
        check(lib.mtadgat_gat_fwd(x.data_ptr(), self.lin_w.data_ptr(), self.lin_b.data_ptr(), self.a.data_ptr(),
                                  _ptr(self.bias), out.data_ptr(), saved.data_ptr(), B, self.n, self.k, self.E,
                                  int(self.feature), int(self.v2), float(self.alpha), training, float(p),
                                  self.seed.data_ptr(), torch.cuda.current_stream().cuda_stream))
        torch.cuda.synchronize()
        return out, saved

    def bwd(self, out, saved, split=False, dx0=None):
        """parts=3 on the current stream, or (split) parts 9, then 2 on a second stream, then 4, as _run_bwd issues."""
        from mtad_gat_pytorch_b200._lib import lib, check
        B = self.B
        scratch = _nan(lib.mtadgat_gat_bwd_scratch_floats(B, self.n, self.k, self.E, int(self.feature), int(self.v2)))
        dx = dx0.clone() if dx0 is not None else _nan(B, self.n, self.k)
        g = {"dlin_w": _nan(*self.lin_w.shape), "dlin_b": _nan(*self.lin_b.shape), "da": _nan(*self.a.shape),
             "dbias": _nan(self.K, self.K) if self.bias is not None else None}

        def call(parts, stream):
            check(lib.mtadgat_gat_bwd(self.x.data_ptr(), self.lin_w.data_ptr(), self.lin_b.data_ptr(), self.a.data_ptr(),
                                      out.data_ptr(), self.gout.data_ptr(), saved.data_ptr(), scratch.data_ptr(),
                                      dx.data_ptr(), int(dx0 is not None), g["dlin_w"].data_ptr(),
                                      g["dlin_b"].data_ptr(), g["da"].data_ptr(), _ptr(g["dbias"]), B, self.n, self.k,
                                      self.E, int(self.feature), int(self.v2), float(self.alpha), float(self.p),
                                      self.seed.data_ptr(), parts, stream.cuda_stream))
        cur = torch.cuda.current_stream()
        if split:
            side = _side_stream()
            call(9, cur)
            side.wait_stream(cur)
            call(2, side)
            call(4, cur)
            cur.wait_stream(side)
        else:
            call(3, cur)
        torch.cuda.synchronize()
        g["dx"] = dx
        return g

    def mask(self):
        from mtad_gat_pytorch_b200 import functional as F
        if self.p == 0.0:
            return None
        m = F.dropout_multipliers(self.B * self.K * self.K, self.p, self.seed,
                                  F.RNG_FEATURE if self.feature else F.RNG_TEMPORAL)
        return _np(m).astype(np.float64).reshape(self.B, self.K, self.K)


def reference(L, saved, dx0=None):
    """float64 forward/backward on the kernel's slope decisions; returns (refs, slope stats)."""
    q = {k: None if v is None else v.astype(np.float64) for k, v in L.np.items()}
    views = gr.saved_views(_np(saved), L.B, L.n, L.k, L.E, L.feature, L.v2)
    slope, stats = gr.align_slopes(views["pqt"], views["meta"], q["x"], q["lin_w"], q["lin_b"], q["a"], L.feature,
                                   L.v2)
    out, cache = gr.gat_fwd(q["x"], q["lin_w"], q["lin_b"], q["a"], q["bias"], L.alpha, L.feature, L.v2,
                            mask=L.mask(), slope=slope)
    dx, dlin_w, dlin_b, da, dbias = gr.gat_bwd(_np(L.gout).astype(np.float64), cache)
    if dx0 is not None:
        dx = dx + _np(dx0)
    ref = {"out": out, "att": cache["att"], "dx": dx, "dlin_w": dlin_w, "dlin_b": dlin_b, "da": da.reshape(-1, 1),
           "dbias": dbias}
    return ref, stats, views


def compare(tag, L, mode, out, views, g, ref, stats):
    """Prints per-window and tensor-wide errors; returns the list of failed gates."""
    bad = []
    got = {"out": _np(out), "att": views["att"][:, :, :L.K], "dx": _np(g["dx"])}
    line = []
    for name, gate in (("out", FWD_GATE), ("att", FWD_GATE), ("dx", GATE[mode])):
        e = ot.window_errors(got[name], ref[name])
        tw = float(np.abs(got[name].astype(np.float64) - ref[name]).max() / max(np.abs(ref[name]).max(), 1e-300))
        line.append(f"{name} {np.nanmax(np.where(np.isfinite(e), e, np.inf)):.1e}/{tw:.1e}")
        if not np.all(e < gate):
            bad.append((name, int(np.argmax(np.where(np.isfinite(e), e, np.inf))), float(np.max(e))))
    for name in ("dlin_w", "dlin_b", "da", "dbias"):
        if ref[name] is None:
            continue
        a, r = _np(g[name]).astype(np.float64), ref[name]
        e = float(np.abs(a - r).max() / max(np.abs(r).max(), 1e-300))
        line.append(f"{name} {e:.1e}")
        if not e < GATE[mode]:
            bad.append((name, e))
    print(f"[{tag}] per-window/tensor-wide: " + ", ".join(line) +
          f" | slope disagreements {int(stats['disagree'].sum())} (per window {stats['disagree'].tolist()[:4]}), "
          f"worst |z| {float(stats['worst_rel_z'].max()):.1e} of the window max")
    if not np.all(stats["worst_rel_z"] <= SLOPE_GATE):
        bad.append(("slope", float(stats["worst_rel_z"].max())))
    return bad


def run_case(mode, case, seed, dx_acc=False, **kw):
    import mtad_gat_pytorch_b200 as mg
    mg.set_mode(mode)
    layer, v2, n, k, E, B = case
    L = Layer(layer, v2, n, k, E, B, seed, **kw)
    out, saved = L.fwd()
    dx0 = _cu(np.random.default_rng(seed + 1).uniform(-1, 1, (B, n, k))) if dx_acc else None
    g = L.bwd(out, saved, dx0=dx0)
    # bitwise: a second run, and the split issued by _run_bwd
    g2 = L.bwd(out, saved, dx0=dx0)
    g3 = L.bwd(out, saved, split=True, dx0=dx0)
    unequal = [(what, name) for name, t in g.items() if t is not None
               for what, o in (("repeat", g2), ("split", g3)) if not torch.equal(t, o[name])]
    ref, stats, views = reference(L, saved, dx0)
    return L, out, views, g, ref, stats, unequal


@pytest.mark.parametrize("mode", MODES)
@pytest.mark.parametrize("case", CASES, ids=case_id)
def test_gat_layer_vs_fp64(case, mode):
    L, out, views, g, ref, stats, unequal = run_case(mode, case, seed=sum(case[2:]))
    bad = compare(f"{mode} {case_id(case)}", L, mode, out, views, g, ref, stats)
    assert not bad and not unequal, (bad, unequal)


EDGES = {
    "a_all_pos": dict(a_kind="pos"),                 # npos = E
    "a_all_neg": dict(a_kind="neg"),                 # npos = 0
    "a_some_zero": dict(a_kind="zero"),              # a_e == 0 exactly: da_e = sum de lrelu(z_e) still
    "alpha_0.05": dict(alpha=0.05),
    "no_bias": dict(bias=False),
    "dropout_0.3": dict(p=0.3),
    "one_hot": dict(scale0=6.0),                     # window 0 scaled: its softmax rows are nearly one-hot
    "dx_accumulate": dict(dx_acc=True),
}


@pytest.mark.parametrize("mode", MODES)
@pytest.mark.parametrize("edge", list(EDGES))
@pytest.mark.parametrize("case", [("temporal", True, 97, 25, 50, 3), ("feature", True, 100, 38, 200, 3),
                                  ("temporal", False, 97, 38, 38, 3)], ids=case_id)
def test_gat_edges_vs_fp64(case, edge, mode):
    kw = EDGES[edge]
    if case[1] is False and "a_kind" in kw and kw["a_kind"] != "zero":
        pytest.skip("GATv1 has no sign-sorted channels")
    L, out, views, g, ref, stats, unequal = run_case(mode, case, seed=7 + sum(case[2:]), **kw)
    if L.v2:
        npos = int(views["meta"][0])
        want = {"pos": L.E, "neg": 0}.get(kw.get("a_kind"), int((L.np["a"] > 0).sum()))
        assert npos == want, (npos, want)
    if edge == "one_hot":
        print(f"[one_hot] window 0 mean row max of the attention {ref['att'][0].max(axis=-1).mean():.3f}, other windows "
              f"{ref['att'][1:].max(axis=-1).mean():.3f}")
    bad = compare(f"{mode} {edge} {case_id(case)}", L, mode, out, views, g, ref, stats)
    assert not bad and not unequal, (bad, unequal)


# ---- bitwise forward properties -------------------------------------------------------------------------------------
FWD_PATHS = [("temporal", True, 100, 38, 76), ("feature", True, 100, 55, 48), ("feature", True, 100, 38, 200),
             ("feature", True, 100, 5, 200), ("feature", True, 100, 129, 200), ("feature", True, 100, 64, 200),
             ("temporal", True, 100, 512, 48), ("temporal", False, 97, 38, 38)]


@pytest.mark.parametrize("mode", MODES)
@pytest.mark.parametrize("shape", FWD_PATHS, ids=lambda s: case_id(s + (17,)))
def test_forward_window_is_batch_independent(shape, mode):
    """One shape per forward path: a window's output is bitwise the same in a batch of 17 as alone, and the inference
    forward (training=0, what the stream scorers run) equals the training forward at p = 0."""
    import mtad_gat_pytorch_b200 as mg
    mg.set_mode(mode)
    layer, v2, n, k, E = shape
    L = Layer(layer, v2, n, k, E, 17, seed=n + k)
    print(f"[{mode} {case_id(shape + (17,))}] {gr.expected_paths(layer, v2, n, k, E, mode, 17)['fwd']}")
    out1, _ = L.fwd(training=1, p=0.0)
    out0, _ = L.fwd(training=0)
    assert torch.equal(out0, out1)
    for w in (0, 9, 16):
        alone, _ = L.fwd(training=0, x=L.x[w:w + 1].clone())
        assert torch.equal(alone[0], out0[w]), w


# ---- dispatch, measured ---------------------------------------------------------------------------------------------
def measured_paths(names):
    r = {}

    def put(key, val):
        r.setdefault(key, set()).add(val)
    for nm in names:
        kind = "tc" if "pack_kernel<" in nm else ("simt" if re.search(r"(?<![\w])gemm_kernel<", nm) else None)
        m = re.search(r"gat_score_win_kernel<(\d+), (\d+)>", nm)
        if m:
            put("fwd", f"win<{m[1]},{m[2]}>")
        m = re.search(r"gat_score_fwd_kernel<(\d+), (\d+)>", nm)
        if m:
            put("fwd", f"tiled<{m[1]},{m[2]}>")
        m = re.search(r"gat_bwd1_kernel<(\d+)>", nm)
        if m:
            put("bwd1", f"bwd1<{m[1]}>")
        if "gat_bwd2_win_kernel" in nm:
            put("bwd2", "bwd2_win")
        elif "gat_bwd2_kernel" in nm:
            put("bwd2", "bwd2")
        if "dpq_colsum_kernel" in nm:
            put("colsum", True)
        if "splitk_reduce_kernel" in nm and "StAtomic2" in nm:
            put("param_reduce", True)
        if kind:
            if "WpT" in nm:
                put("proj", kind)
            if "NodeAT" in nm:
                put("param", kind)
            if "DsTA" in nm or "WpA2" in nm:
                put("dv", "T")
            if "AttTA" in nm or "DpqA" in nm:
                put("dv", "N")
            if "AttTA" in nm or "DsTA" in nm:
                put("dv1", kind)
            if "DpqA" in nm or "WpA2" in nm:
                put("dv2", kind)
    return {k: (next(iter(v)) if len(v) == 1 else tuple(sorted(map(str, v)))) for k, v in r.items()}


KEYS = ("fwd", "proj", "bwd1", "bwd2", "param", "param_reduce", "colsum", "dv", "dv1", "dv2")


def dispatch_table():
    """Every case of the matrix in both modes: the kernels torch.profiler records against expected_paths, one line per
    case; and the union of the cases reaches every path of the GAT dispatch."""
    import mtad_gat_pytorch_b200 as mg
    bad, reached = [], {m: set() for m in MODES}
    for mode in MODES:
        mg.set_mode(mode)
        for case in CASES:
            layer, v2, n, k, E, B = case
            L = Layer(layer, v2, n, k, E, B, seed=1)
            with torch.profiler.profile(activities=[torch.profiler.ProfilerActivity.CUDA]) as prof:
                out, saved = L.fwd()
                L.bwd(out, saved)
                torch.cuda.synchronize()
            got = measured_paths({e.name for e in prof.events()})
            exp = gr.expected_paths(layer, v2, n, k, E, mode, B)
            want = {key: exp[key] for key in KEYS if exp[key] not in (False, None)}
            print(f"[dispatch {mode} {case_id(case)}] " + " ".join(f"{key}={got.get(key, '-')}" for key in KEYS) +
                  f" split={'+'.join(exp['split']) or '-'} bwd1_split={'+'.join(exp['bwd1_split']) or '-'}")
            if got != want:
                bad.append((mode, case, got, want))
            reached[mode] |= {f"{key}={got.get(key)}" for key in KEYS} | {f"split:{s}" for s in exp["split"]} | \
                {f"bwd1_split:{s}" for s in exp["bwd1_split"]} | {f"{got.get('param')}:v{2 if v2 else 1}"}
    need = {f"fwd={p}" for p in ("win<4,10>", "win<4,4>", "win<2,4>", "win<2,2>", "tiled<4,4>", "tiled<2,4>",
                                  "tiled<2,2>")} | {"bwd1=bwd1<4>", "bwd1=bwd1<2>", "bwd2=bwd2_win", "bwd2=bwd2",
                                                    "dv=T", "dv=N", "proj=simt", "dv1=simt", "dv2=simt",
                                                    "param=simt", "colsum=True", "param_reduce=True", "simt:v1",
                                                    "split:rows", "split:JT<K", "split:DT<E", "bwd1_split:JT<K"}
    for mode in MODES:
        missing = need - reached[mode]
        if mode == "tc":
            missing |= {"proj=tc", "param=tc", "dv1=tc", "dv2=tc"} - reached[mode]
        assert not missing, (mode, sorted(missing))
    assert not bad, bad


def test_dispatch_table():
    """dispatch_table() in a child process, so that its profiler sessions do not share a process with the rest of the
    suite: with them in the same process, torch.profiler sessions of later tests recorded no kernels."""
    import os
    import subprocess
    import sys
    root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    r = subprocess.run([sys.executable, "-c", "from tests.test_gpu_gat import dispatch_table; dispatch_table()"],
                       cwd=root, capture_output=True, text=True, timeout=900)
    print(r.stdout)
    assert r.returncode == 0, r.stdout[-3000:] + r.stderr[-3000:]


def test_envelope_refusal():
    """A tiled layer with D > 1024 (feature layer, n = 1100, k = 200) is outside the score kernels' envelope: the call
    raises MtadGatLibraryError with the envelope message, and nothing after the weight folding is launched."""
    import mtad_gat_pytorch_b200 as mg
    from mtad_gat_pytorch_b200._lib import MtadGatLibraryError
    L = Layer("feature", True, 1100, 200, 16, 1, seed=3)
    mg.reset_launch_count()
    with pytest.raises(MtadGatLibraryError, match="outside the kernel envelope"):
        L.fwd()
    assert mg.launch_count() == 2           # the two weight-folding kernels; no projection GEMM, no score kernel
