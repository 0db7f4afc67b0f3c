"""Host restatement of the per-feature layout (csrc/fleet.cu mtadgat_feature_gather / _scatter): feature i of stream s
is SPOT stream s*out + i, and stream s's rows offsets[s] .. offsets[s+1]-1 of a push's (M, out) scores become out
contiguous runs of m_s scores each, one per feature."""
import numpy as np


def feature_map(offsets, out):
    """(dst, feature_offsets) for streams delimited by `offsets` (S + 1, non-decreasing from 0 to M): entry r*out + i of
    the row-major (M, out) scores goes to position dst[r*out + i] of the feature-major scores, and feature stream j's
    run is feature_offsets[j] .. feature_offsets[j+1] - 1."""
    off = np.asarray(offsets, np.int64)
    m = np.diff(off)
    stream = np.repeat(np.arange(m.size), m)
    o, ms = off[stream], m[stream]
    r = np.arange(off[-1], dtype=np.int64)
    dst = (out * o[:, None] + np.arange(out)[None, :] * ms[:, None] + (r - o)[:, None]).reshape(-1)
    foff = np.append((out * off[:-1, None] + np.arange(out)[None, :] * m[:, None]).reshape(-1), out * off[-1])
    return dst, foff


def gather(a_score, offsets):
    """mtadgat_feature_gather on the host: (feature-major scores, feature offsets)."""
    a = np.asarray(a_score)
    dst, foff = feature_map(offsets, a.shape[1])
    fm = np.empty(a.size, a.dtype)
    fm[dst] = a.reshape(-1)
    return fm, foff


def scatter(values, offsets, out):
    """mtadgat_feature_scatter on the host: the feature-major `values` back to (M, out)."""
    dst, _ = feature_map(offsets, out)
    return np.asarray(values)[dst].reshape(-1, out)
