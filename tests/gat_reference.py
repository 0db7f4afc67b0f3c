"""Test-side restatements for the GAT layer kernels (csrc/gat.cu): the `saved` buffer layout, a float64 reference in the
factored form of gat.cu's header comment, the LeakyReLU slope alignment, and the host dispatch of mtadgat_gat_fwd /
mtadgat_gat_bwd and the GEMMs they issue (gemm.cuh, tc_gemm2.cuh).  Test infrastructure only.

Factored form: lin([v_i || v_j]) = W1 v_i + W2 v_j + b, so z_ij = P_i + Q_j with P = V W1^T, Q = V W2^T + b (GATv2), and
the score of GATv1 is lrelu(s_i + t_j) with s = (V W^T + b) a1, t = (V W^T + b) a2.  No (B,K,K,2D) tensor is formed; the
(B,K,K,E) pre-activations are built `rows` rows i at a time."""
import numpy as np


def cdiv(a, b):
    return -(-a // b)


# ---- shapes and the saved-buffer layout -----------------------------------------------------------------------------
def dims(n, k, E, feature, v2):
    """(K, D, E', NC, Kp) of make_dims: nodes, node length, P/Q block width (0 for v1), channels, K rounded up to 4."""
    K, D = (k, n) if feature else (n, k)
    Ew = E if v2 else 0
    return K, D, Ew, 2 * Ew + 2, (K + 3) & ~3


def saved_layout(B, n, k, E, feature, v2, training=1):
    """Offsets (floats) of saved_layout(): wp (D,NC), bp (NC), meta (ints, 4-aligned), pqt (B,NC,Kp), att (B,K,Kp)."""
    K, D, _, NC, Kp = dims(n, k, E, feature, v2)
    L, o = {}, 0
    L["wp"] = o; o += D * NC
    L["bp"] = o; o += NC
    o = (o + 3) & ~3
    L["meta"] = o; o += 2 * E + 4
    o = (o + 3) & ~3
    L["pqt"] = o; o += B * NC * Kp
    L["att"] = o
    if training:
        o += B * K * Kp
    L["total"] = o
    return L


def saved_views(saved, B, n, k, E, feature, v2):
    """numpy views of a float32 `saved` buffer: meta (int32), pqt (B,NC,Kp), att (B,K,Kp)."""
    K, D, _, NC, Kp = dims(n, k, E, feature, v2)
    L = saved_layout(B, n, k, E, feature, v2)
    s = np.asarray(saved, dtype=np.float32)
    return {"meta": s[L["meta"]:L["meta"] + 2 * E + 4].view(np.int32),
            "pqt": s[L["pqt"]:L["pqt"] + B * NC * Kp].reshape(B, NC, Kp),
            "att": s[L["att"]:L["att"] + B * K * Kp].reshape(B, K, Kp)}


def nodes(x, feature):
    """(B,n,k) window -> V (B,K,D)"""
    return x.transpose(0, 2, 1) if feature else x


# ---- the float64 reference ------------------------------------------------------------------------------------------
def _proj(v, lin_w, lin_b, v2):
    D = v.shape[2]
    if v2:
        return v @ lin_w[:, :D].T, v @ lin_w[:, D:].T + lin_b
    wx = v @ lin_w.T + lin_b
    return wx, None


def _pre(P, Q, a, v2, i0, i1):
    """pre-activation rows i0..i1: (B,r,K,E) z for v2, (B,r,K) s_i + t_j for v1"""
    if v2:
        return P[:, i0:i1, None, :] + Q[:, None, :, :]
    E = P.shape[2]
    s, t = P @ a[:E], P @ a[E:]
    return s[:, i0:i1, None] + t[:, None, :]


def gat_fwd(x, lin_w, lin_b, a, bias, alpha, feature, v2, mask=None, slope=None, rows=16):
    """out (B,n,k) and a cache for gat_bwd.  mask: (B,K,K) dropout multipliers; slope: boolean (B,K,K,E) (v2) or (B,K,K)
    (v1) branch of every pre-activation (None = the reference's own z > 0)."""
    a = np.asarray(a, dtype=np.float64).reshape(-1)
    v = nodes(x, feature)
    B, K, D = v.shape
    P, Q = _proj(v, lin_w, lin_b, v2)
    e = np.empty((B, K, K))
    for i0 in range(0, K, rows):
        i1 = min(K, i0 + rows)
        z = _pre(P, Q, a, v2, i0, i1)
        g = (z > 0) if slope is None else slope[:, i0:i1]
        l = np.where(g, z, alpha * z)
        e[:, i0:i1] = l @ a if v2 else l
    if bias is not None:
        e = e + bias
    m = e.max(axis=-1, keepdims=True)
    att = np.exp(e - m)
    att /= att.sum(axis=-1, keepdims=True)
    att_d = att if mask is None else att * mask
    s = att_d @ v
    h = 1.0 / (1.0 + np.exp(-s))
    out = h.transpose(0, 2, 1) if feature else h
    return out, dict(v=v, P=P, Q=Q, att=att, att_d=att_d, h=h, lin_w=lin_w, a=a, alpha=alpha, feature=feature, v2=v2,
                     mask=mask, slope=slope, bias=bias is not None, rows=rows)


def gat_bwd(dout, c):
    """dx, dlin_w, dlin_b, da (flat), dbias (None without bias)"""
    v, P, Q, att, a, alpha, v2 = c["v"], c["P"], c["Q"], c["att"], c["a"], c["alpha"], c["v2"]
    B, K, D = v.shape
    h = c["h"]
    dh = dout.transpose(0, 2, 1) if c["feature"] else dout
    ds = dh * h * (1.0 - h)
    datt = ds @ v.transpose(0, 2, 1)
    dv = c["att_d"].transpose(0, 2, 1) @ ds
    if c["mask"] is not None:
        datt = datt * c["mask"]
    de = att * (datt - (att * datt).sum(axis=-1, keepdims=True))
    dbias = de.sum(axis=0) if c["bias"] else None
    lin_w = c["lin_w"]
    if v2:
        E = P.shape[2]
        da = np.zeros(E)
        dP, dQ = np.zeros((B, K, E)), np.zeros((B, K, E))
        for i0 in range(0, K, c["rows"]):
            i1 = min(K, i0 + c["rows"])
            z = _pre(P, Q, a, True, i0, i1)
            g = (z > 0) if c["slope"] is None else c["slope"][:, i0:i1]
            dei = de[:, i0:i1, :, None]
            da += (dei * np.where(g, z, alpha * z)).sum(axis=(0, 1, 2))
            dz = dei * a * np.where(g, 1.0, alpha)
            dP[:, i0:i1] = dz.sum(axis=2)
            dQ += dz.sum(axis=1)
        Vf = v.reshape(-1, D)
        dlin_w = np.concatenate([dP.reshape(-1, E).T @ Vf, dQ.reshape(-1, E).T @ Vf], axis=1)
        dlin_b = dQ.sum(axis=(0, 1))
        dv = dv + dP @ lin_w[:, :D] + dQ @ lin_w[:, D:]
    else:
        wx = P
        E = wx.shape[2]
        z = _pre(P, None, a, False, 0, K)
        g = (z > 0) if c["slope"] is None else c["slope"]
        dpre = de * np.where(g, 1.0, alpha)
        r, cl = dpre.sum(axis=2), dpre.sum(axis=1)            # (B,K): sum over j of row i, sum over i of column j
        da = np.concatenate([(r[..., None] * wx).sum(axis=(0, 1)), (cl[..., None] * wx).sum(axis=(0, 1))])
        dwx = r[..., None] * a[:E] + cl[..., None] * a[E:]
        dlin_w = dwx.reshape(-1, E).T @ v.reshape(-1, D)
        dlin_b = dwx.sum(axis=(0, 1))
        dv = dv + dwx @ lin_w
    dx = dv.transpose(0, 2, 1) if c["feature"] else dv
    return dx, dlin_w, dlin_b, da, dbias


# ---- slope alignment ------------------------------------------------------------------------------------------------
def align_slopes(pqt, meta, x, lin_w, lin_b, a, feature, v2, rows=16):
    """The branch the kernels' backward takes for every pre-activation, from the saved fp32 projections: P_id + Q_jd > 0
    with the sign-sorted channels put back in original order through meta (GATv2), p_i + q_j > 0 (GATv1).  Returns the
    boolean slope array and, per window, how many of those decisions differ from the float64 reference's own z > 0 and
    the largest |z| among them relative to the window's max |z|."""
    a = np.asarray(a, dtype=np.float64).reshape(-1)
    v = nodes(x, feature)
    B, K, D = v.shape
    Pr, Qr = _proj(v, lin_w, lin_b, v2)
    if v2:
        E = lin_w.shape[0]
        inv = np.asarray(meta[4 + E:4 + 2 * E])
        Pk = np.ascontiguousarray(pqt[:, inv, :K].transpose(0, 2, 1))           # (B,K,E) fp32, original column order
        Qk = np.ascontiguousarray(pqt[:, E + inv, :K].transpose(0, 2, 1))
        slope = np.empty((B, K, K, E), dtype=bool)
    else:
        E = 0
        pk, qk = pqt[:, 0, :K], pqt[:, 1, :K]
        slope = np.empty((B, K, K), dtype=bool)
    count = np.zeros(B, dtype=np.int64)
    worst, zmax = np.zeros(B), np.zeros(B)
    for i0 in range(0, K, rows):
        i1 = min(K, i0 + rows)
        if v2:
            g = (Pk[:, i0:i1, None, :] + Qk[:, None, :, :]) > 0                  # float32 add, as the kernels
        else:
            g = (pk[:, i0:i1, None] + qk[:, None, :]) > 0
        slope[:, i0:i1] = g
        z = _pre(Pr, Qr, a, v2, i0, i1)
        dis = g != (z > 0)
        az = np.abs(z).reshape(B, -1)
        zmax = np.maximum(zmax, az.max(axis=1))
        count += dis.reshape(B, -1).sum(axis=1)
        worst = np.maximum(worst, np.where(dis.reshape(B, -1), az, 0.0).max(axis=1))
    return slope, {"disagree": count, "worst_rel_z": worst / np.maximum(zmax, np.finfo(np.float64).tiny)}


# ---- dispatch ---------------------------------------------------------------------------------------------------------
def _score_win_smem(K, D, NC, Kp):
    Dp = (D + 3) & ~3
    pq = max(NC * Kp + 16, K * Dp)
    pq = (pq + 3) & ~3
    return 4 * (pq + K * Kp) + 16


def _bwd2_win_smem(K, E, Kp):
    NCp = 2 * ((E + 3) & ~3)
    return 4 * (K * (NCp + 16) + K * (Kp + 1) + 2 * Kp)


def _pick_score_tiles(K, D, E, Kp):
    ntd = (D + 3) // 4
    if ntd > 256:
        return None
    RB = min(K, 4 * (256 // ntd))
    if K > 128:
        RB = min(RB, (K + 1) // 2)
    JT, DT = K, (E if E > 0 else 1)
    while True:
        RBp, JTp = (RB + 3) & ~3, (JT + 3) & ~3
        smem = 4 * (RB * Kp + max(DT * RBp + DT * JTp, JT * (D + 1)))
        if smem <= 200 * 1024:
            return RB, JT, DT
        if DT > 32:
            DT = (DT + 1) // 2
        elif JT > 32:
            JT = (JT + 1) // 2
        elif RB > 4:
            RB = (RB + 1) // 2
        else:
            return None


def _splitk_reduces(M, N, Kd, mode):
    """True when launch_gemm_splitk (mode 'tc' packed path, else SIMT) splits K into more than one slice"""
    if mode == "tc":
        bn = 64 if N <= 64 else 128
        tiles = cdiv(N, bn) * cdiv(M, 128)
        splits = max(1, min(cdiv(Kd, 128), cdiv(264, tiles)))
        KT = cdiv(Kd, 32)
        splits = max(1, min(KT, splits))
        return cdiv(KT, cdiv(KT, splits)) > 1
    tiles = cdiv(N, 64) * cdiv(M, 64)
    splits = max(1, min(cdiv(Kd, 64), cdiv(528, tiles)))
    klen = cdiv(cdiv(Kd, splits), 16) * 16
    return cdiv(Kd, klen) > 1


MAX_GRID_YZ = 65535                 # CUDA's gridDim.y / gridDim.z limit


def expected_paths(layer, v2, n, k, E, mode, B=1):
    """The kernels one forward + backward of a GAT layer runs, as the host code of mtadgat_gat_fwd / mtadgat_gat_bwd and
    the GEMM launchers choose them.  layer: 'feature' or 'temporal'; mode: 'tc' or 'fp32' (set_mode).  Returns a dict:
      fwd   'win<MI,MJ>' (gat_score_win_kernel) or 'tiled<MI,MJ>' (gat_score_fwd_kernel), None outside the envelope
      split (tiled only) 'rows' when K > 128 splits a window over CTAs, 'JT<K' / 'DT<E' when the column / channel tiles
            are smaller than the window
      proj  'tc' (gemm2_kernel) or 'simt' (gemm_kernel) for the projection GEMM
      bwd1  'bwd1<4>' / 'bwd1<2>', and 'JT<K' in bwd1_split when its column tile shrank below min(K, 64)
      bwd2  'bwd2_win' (gat_bwd2_win_kernel) or 'bwd2' (two-pass gat_bwd2_kernel)
      param 'tc' or 'simt' for the weight-gradient split-K; param_reduce True when splitk_reduce_kernel follows it;
            colsum True when dpq_colsum_kernel makes the bias-channel sums (the SIMT path)
      dv    'T' for the transposed products (feature layer, K <= 64), else 'N'; dv1 / dv2 'tc' or 'simt' for the
            att~-product and the projection product
      launches  {fwd, bwd1, bwd2, proj, dv1, dv2}: kernel launches per call.  The window kernels put the windows on
            gridDim.x (one launch); gat_score_fwd_kernel and gat_bwd1_kernel put them on gridDim.y, gat_bwd2_kernel (per
            pass) and the batched GEMMs on gridDim.z, each launched in chunks of at most 65 535 windows"""
    feature = layer == "feature"
    K, D, Ew, NC, Kp = dims(n, k, E, feature, v2)
    tc = mode == "tc"
    chunks = cdiv(B, MAX_GRID_YZ)
    r = {"launches": {}}
    win = K <= 128 and _score_win_smem(K, D, NC, Kp) <= 112 * 1024
    if win:
        best, best_cost = None, None
        for mi, mj in ((4, 10), (4, 4), (2, 4), (2, 2)):
            cost = cdiv(cdiv(K, mi) * cdiv(K, mj), 256) * mi * mj
            if best_cost is None or cost < best_cost:
                best, best_cost = (mi, mj), cost
        r["fwd"], r["split"] = f"win<{best[0]},{best[1]}>", ()
        r["launches"]["fwd"] = 1
    else:
        t = _pick_score_tiles(K, D, Ew, Kp)
        if t is None:
            r["fwd"] = None
            return r
        RB, JT, DT = t
        jt = min(JT, K)
        if cdiv(RB, 4) * cdiv(jt, 4) >= 200:
            r["fwd"] = "tiled<4,4>"
        elif cdiv(RB, 2) * cdiv(jt, 4) >= 160:
            r["fwd"] = "tiled<2,4>"
        else:
            r["fwd"] = "tiled<2,2>"
        r["split"] = tuple(s for s, on in (("rows", RB < K), ("JT<K", JT < K), ("DT<E", DT < max(Ew, 1))) if on)
        r["launches"]["fwd"] = chunks
    r["proj"] = "tc" if tc and K >= 16 and D >= 16 else "simt"
    RB, JT = min(K, 64), min(K, 64)
    while True:
        Dp = 4 * (((D + 3) >> 2) | 1)
        if 4 * (RB * Kp + RB * Dp + JT * Dp) <= 200 * 1024:
            break
        if JT > 8:
            JT = (JT + 1) // 2
        elif RB > 1:
            RB = (RB + 1) // 2
        else:
            r["bwd1"] = None
            return r
    r["bwd1"] = "bwd1<4>" if cdiv(RB, 4) * cdiv(JT, 4) >= 200 else "bwd1<2>"
    r["bwd1_split"] = ("JT<K",) if JT < min(K, 64) else ()
    r["bwd2"] = "bwd2_win" if K <= 128 and _bwd2_win_smem(K, Ew, Kp) <= 112 * 1024 else "bwd2"
    r["launches"].update(bwd1=chunks, bwd2=1 if r["bwd2"] == "bwd2_win" else 2 * chunks)
    ptc = tc and D >= 32 and NC >= 16
    r["param"] = "tc" if ptc else "simt"
    r["param_reduce"] = _splitk_reduces(D, NC, B * K, "tc" if ptc else "simt")
    r["colsum"] = not ptc
    if feature and K <= 64:
        r["dv"] = "T"
        dims1, dims2 = (D, K, K), (D, K, NC)
    else:
        r["dv"] = "N"
        dims1, dims2 = (K, D, K), (K, D, NC)
    r["dv1"] = "tc" if tc and dims1[1] >= 16 and dims1[2] >= 16 else "simt"
    r["dv2"] = "tc" if tc and dims2[1] >= 16 and dims2[2] >= 16 else "simt"
    # the GEMMs' M (NC, K or D rows) stays far below 65 535 tiles: one launch per chunk of windows
    r["launches"].update(proj=chunks, dv1=chunks, dv2=chunks)
    return r
