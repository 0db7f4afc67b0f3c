"""Test-side helpers around the numpy oracle (oracle/mtad_gat_oracle.py): chunked evaluation at the benchmark's
batch size, the Philox masks the kernels draw, and a numpy Adam.  Test infrastructure only."""
import numpy as np
import torch

from oracle import mtad_gat_oracle as orc

SEED_STEP = 0x9E3779B97F4A7C15          # seed_advance_kernel (csrc/api.cu): one splitmix64 increment per forward
MASK64 = (1 << 64) - 1


def _slice_masks(masks, lo, hi):
    if not masks:
        return None
    out = {}
    for key, v in masks.items():
        out[key] = [m[lo:hi] for m in v] if isinstance(v, list) else v[lo:hi]
    return out


def loss_fwd_bwd_chunked(x, y, params, cfg, masks=None, target_dims=None, chunk=32):
    """orc.loss_fwd_bwd for batches whose materialised (B,K,K,2D) tensors do not fit at once: windows are independent
    up to the two global sqrt(MSE) normalisers, so forward in chunks, form the losses, then forward+backward in chunks
    with the chunk's slice of dL/dpreds, dL/drecons and sum the parameter gradients.
    Returns (loss, lf, lr, preds, recons, dx, grads) like orc.loss_fwd_bwd."""
    B = x.shape[0]
    preds, recons, pres = [], [], []
    for lo in range(0, B, chunk):
        p, r, cache = orc.model_fwd(x[lo:lo + chunk], params, cfg, _slice_masks(masks, lo, lo + chunk))
        preds.append(p); recons.append(r); pres.append(cache[4][4])
    preds, recons = np.concatenate(preds), np.concatenate(recons)
    loss_fwd_bwd_chunked.last_mlp_pre = [np.concatenate([c[i] for c in pres]) for i in range(len(pres[0]))]
    xt = x if target_dims is None else x[:, :, target_dims]
    yt = y if target_dims is None else y[:, :, target_dims]
    yt = yt.reshape(B, -1)
    lf, lr = np.sqrt(((yt - preds) ** 2).mean()), np.sqrt(((xt - recons) ** 2).mean())
    dpreds = (preds - yt) / (preds.size * lf)
    drecons = (recons - xt) / (recons.size * lr)
    dx = np.zeros_like(x)
    grads = None
    for lo in range(0, B, chunk):
        hi = min(B, lo + chunk)
        _, _, cache = orc.model_fwd(x[lo:hi], params, cfg, _slice_masks(masks, lo, hi))
        dxi, gi = orc.model_bwd(dpreds[lo:hi], drecons[lo:hi], cache, params, cfg)
        dx[lo:hi] = dxi
        if grads is None:
            grads = {k: v.copy() for k, v in gi.items()}
        else:
            for k, v in gi.items():
                grads[k] += v
    direct = (xt - recons) / (recons.size * lr)            # x is also the reconstruction target
    if target_dims is None:
        dx += direct
    else:
        dx[:, :, target_dims] += direct
    return lf + lr, lf, lr, preds, recons, dx, grads


def tile(x, fill=0.0):
    """(B,n,C) -> the window-tiled layout of the recurrence kernels, T[b//16][t][c][b%16] with B rounded up to 16
    (csrc/gru_common.cuh); the padded windows b >= B hold `fill`.  numpy arrays or torch tensors."""
    B, n, C = x.shape
    T = (B + 15) // 16
    if torch.is_tensor(x):
        xp = torch.full((T * 16, n, C), fill, dtype=x.dtype, device=x.device)
        xp[:B] = x
        return xp.view(T, 16, n, C).permute(0, 2, 3, 1).contiguous()
    xp = np.full((T * 16, n, C), fill, dtype=x.dtype)
    xp[:B] = x
    return np.ascontiguousarray(xp.reshape(T, 16, n, C).transpose(0, 2, 3, 1))


def untile(t, B):
    """Inverse of tile(): (T,n,C,16) -> (B,n,C), dropping the padded windows."""
    T, n, C, _ = t.shape
    if torch.is_tensor(t):
        return t.permute(0, 3, 1, 2).reshape(T * 16, n, C)[:B]
    return t.transpose(0, 3, 1, 2).reshape(T * 16, n, C)[:B]


def window_errors(a, ref):
    """Per window (leading axis): max |a - ref| / max |ref| over the window's elements, in float64.  A NaN or inf in
    `a` gives a NaN or inf error, which fails any `<` gate."""
    a = np.asarray(a, dtype=np.float64).reshape(len(ref), -1)
    r = np.asarray(ref, dtype=np.float64).reshape(len(ref), -1)
    return np.abs(a - r).max(axis=1) / np.maximum(np.abs(r).max(axis=1), np.finfo(np.float64).tiny)


def seed_after(seed0, n_forwards):
    """Value of the device seed after `n_forwards` training-mode forwards starting from manual_seed(seed0)."""
    return (int(seed0) + n_forwards * SEED_STEP) & MASK64


def masks_for_seed(seed_value, cfg, B, p, device="cuda"):
    """The dropout multipliers MTAD_GAT.forward applies under the given per-step seed, via mtadgat_dropout_mask
    (same Philox stream ids as the kernels), as float64 numpy arrays in the oracle's mask format."""
    from mtad_gat_pytorch_b200 import functional as F
    v = seed_value & MASK64
    if v >= 1 << 63:
        v -= 1 << 64
    st = torch.tensor([v], dtype=torch.int64, device=device)

    def m(numel, stream, shape):
        return F.dropout_multipliers(numel, p, st, stream).view(*shape).cpu().numpy().astype(np.float64)
    return {"feat": m(B * cfg.k * cfg.k, F.RNG_FEATURE, (B, cfg.k, cfg.k)),
            "temp": m(B * cfg.n * cfg.n, F.RNG_TEMPORAL, (B, cfg.n, cfg.n)),
            "mlp": [m(B * cfg.forecast_hid_dim, F.RNG_MLP0 + i, (B, cfg.forecast_hid_dim))
                    for i in range(cfg.forecast_n_layers)]}


class NumpyAdam:
    """torch.optim.Adam(lr, betas=(0.9, 0.999), eps=1e-8, weight_decay=0) on a dict of numpy arrays."""

    def __init__(self, params, lr=1e-3, b1=0.9, b2=0.999, eps=1e-8):
        self.p, self.lr, self.b1, self.b2, self.eps, self.t = params, lr, b1, b2, eps, 0
        self.m = {k: np.zeros_like(v) for k, v in params.items()}
        self.v = {k: np.zeros_like(v) for k, v in params.items()}

    def step(self, grads):
        self.t += 1
        c1, c2 = 1 - self.b1 ** self.t, 1 - self.b2 ** self.t
        for k, g in grads.items():
            self.m[k] = self.b1 * self.m[k] + (1 - self.b1) * g
            self.v[k] = self.b2 * self.v[k] + (1 - self.b2) * g * g
            self.p[k] = self.p[k] - (self.lr / c1) * self.m[k] / (np.sqrt(self.v[k]) / np.sqrt(c2) + self.eps)


def align_mlp_gates(gpu_gates, masks, x, params, cfg, tol=1e-3):
    """ReLU-branch bookkeeping for the forecasting head (see orc.forecast_fwd): `gpu_gates` = the implementation's
    (activation > 0) per hidden layer.  Returns (masks + 'mlp_gates', stats) where the gate of every KEPT activation is
    the implementation's, and stats bounds the disagreement with the oracle's own branch choice: how many kept
    activations disagree, out of how many, and the largest |pre-activation| (relative to the layer's max) among them --
    a disagreement is legitimate only right at the kink."""
    B = x.shape[0]
    pres = []
    for lo in range(0, B, 32):
        _, _, cache = orc.model_fwd(x[lo:lo + 32], params, cfg, _slice_masks(masks, lo, lo + 32))
        pres.append(cache[4][4])
    pres = [np.concatenate([c[i] for c in pres]) for i in range(len(pres[0]))]
    out = dict(masks or {})
    gates, n_dis, n_tot, worst = [], 0, 0, 0.0
    for i, (z, g) in enumerate(zip(pres, gpu_gates)):
        kept = (masks["mlp"][i] > 0) if masks and masks.get("mlp") is not None else np.ones_like(z, dtype=bool)
        nat = z > 0
        dis = kept & (nat != g)
        n_dis += int(dis.sum()); n_tot += int(kept.sum())
        if dis.any():
            worst = max(worst, float(np.abs(z[dis]).max() / np.abs(z).max()))
        gates.append(np.where(kept, g, nat))
        # the aligned gates only move the branch of later layers' inputs by O(tol): later layers' natural gates are
        # taken from the unaligned pass, which is what the implementation is compared against anyway
    out["mlp_gates"] = gates
    return out, {"disagree": n_dis, "kept": n_tot, "worst_rel_preact": worst}


def align_conv_gates(gpu_xc, masks, x, params, cfg):
    """Same bookkeeping for the ConvLayer's ReLU (orc.conv_fwd `gates`): gpu_xc = the implementation's conv output
    (B,n,k).  Returns (masks + 'conv_gates', stats)."""
    pre = orc.conv_fwd(x, params["conv.conv.weight"], params["conv.conv.bias"])[1][1]
    g = np.asarray(gpu_xc) > 0
    nat = pre > 0
    dis = nat != g
    out = dict(masks or {})
    out["conv_gates"] = g
    worst = float(np.abs(pre[dis]).max() / np.abs(pre).max()) if dis.any() else 0.0
    return out, {"disagree": int(dis.sum()), "kept": int(pre.size), "worst_rel_preact": worst}
