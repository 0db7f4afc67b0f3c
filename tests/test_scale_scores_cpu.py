"""CPU tests: the host restatement of `scale_scores=True` (prediction.py:82-86) that the device kernels (csrc/scale.cu)
follow, pinned bit for bit against numpy.

For each column `sc` (float32): q75, q25 = np.percentile(sc, [75, 25]) (np.float64), m = np.median(sc) (np.float32),
A_Score_i = (sc - m) / (1 + (q75 - q25)) (float64), and A_Score_Global = np.mean(scores, 1) over the float32 matrix the
columns are rounded into."""
import numpy as np
import pytest


def order_keys(x):
    """Unsigned keys whose order is the float order (-0.0 before +0.0), as csrc/select.cuh forms them."""
    u = np.ascontiguousarray(x, dtype=np.float32).view(np.uint32)
    return np.where(u & 0x80000000, ~u, u | 0x80000000).astype(np.uint32)


def scale_ranks(n):
    """The six order-statistic ranks the median and both quartiles read: median low / high, q25 a / b, q75 a / b."""
    i25, i75 = (n - 1) // 4, 3 * (n - 1) // 4
    return [(n - 1) // 2, n // 2, i25, min(i25 + 1, n - 1), i75, min(i75 + 1, n - 1)]


def percentile(a, b, t):
    """numpy's 'linear' method between the order statistics a <= b at weight t (numpy's _lerp)."""
    d = np.float32(b - a)
    return float(b) - float(d) * (1.0 - t) if t >= 0.5 else float(a) + float(d) * t


def column_stats(sc):
    """(median as np.float32, q25, q75 as np.float64) of one float32 column."""
    n = sc.size
    if np.isnan(sc).any():
        return np.float32(np.nan), np.nan, np.nan
    s = sc[np.argsort(order_keys(sc), kind="stable")]
    r = scale_ranks(n)
    med = np.float32(0) + s[r[0]]                                  # np.mean of the middle one or two, from 0
    if n % 2 == 0:
        med = np.float32(med + s[r[1]])
    med = np.float32(med / np.float32(2 if n % 2 == 0 else 1))
    q25 = percentile(s[r[2]], s[r[3]], ((n - 1) % 4) / 4)
    q75 = percentile(s[r[4]], s[r[5]], (3 * (n - 1) % 4) / 4)
    return med, q25, q75


def pairwise_rows(x):
    """numpy's float32 pairwise sum along each contiguous row of x (N, n): 8 partial sums from 8 values, recursive
    halves (rounded down to a multiple of 8) above 128."""
    n = x.shape[1]
    if n < 8:
        res = np.zeros(x.shape[0], np.float32)
        for i in range(n):
            res = res + x[:, i]
        return res
    if n <= 128:
        r = [x[:, j].copy() for j in range(8)]
        i = 8
        while i < n - n % 8:
            for j in range(8):
                r[j] = r[j] + x[:, i + j]
            i += 8
        res = ((r[0] + r[1]) + (r[2] + r[3])) + ((r[4] + r[5]) + (r[6] + r[7]))
        for i in range(i, n):
            res = res + x[:, i]
        return res
    n2 = n // 2
    n2 -= n2 % 8
    return pairwise_rows(x[:, :n2]) + pairwise_rows(x[:, n2:])


def host_scale(a):
    """a: (N, C) float32 -> (stats (C, 3) float64: median, q25, q75; scaled (N, C) float64; global (N,) float32)."""
    N, C = a.shape
    stats = np.empty((C, 3), np.float64)
    scaled = np.empty((N, C), np.float64)
    for c in range(C):
        med, q25, q75 = column_stats(a[:, c])
        stats[c] = (med, q25, q75)
        scaled[:, c] = (a[:, c] - med).astype(np.float64) / (1.0 + (q75 - q25))    # float32 difference, float64 quotient
    g = (np.float32(0) + pairwise_rows(scaled.astype(np.float32))) / np.float32(C)
    return stats, scaled, g.astype(np.float32)


def numpy_scale(a):
    """The reference's numpy loop for scale_scores=True (prediction.py:82-86, get_score's global mean): the spec."""
    N, C = a.shape
    stats = np.empty((C, 3), np.float64)
    scaled = np.empty((N, C), np.float64)
    scores = np.zeros_like(a)
    for i in range(C):
        sc = a[:, i]
        q75, q25 = np.percentile(sc, [75, 25])
        m = np.median(sc)
        stats[i] = (m, q25, q75)
        sc = (sc - m) / (1 + (q75 - q25))
        scaled[:, i] = sc
        scores[:, i] = sc
    return stats, scaled, np.mean(scores, 1)


def bits(x):
    x = np.asarray(x)
    return x.view(np.uint64 if x.dtype == np.float64 else np.uint32)


def assert_same(got, want):
    """Bitwise equal, NaNs of either sign being equal."""
    got, want = np.asarray(got), np.asarray(want)
    assert got.dtype == want.dtype and got.shape == want.shape
    nan = np.isnan(want)
    assert np.array_equal(np.isnan(got), nan)
    assert np.array_equal(bits(got)[~nan], bits(want)[~nan])


def assert_same_stats(got, want):
    """Medians bitwise; a quartile that is zero may carry either sign (numpy's partition leaves the order of -0.0 and
    +0.0 open), otherwise bitwise.  The scaled values do not depend on that sign: 1 + (q75 - q25) is the same."""
    assert_same(got[:, 0], want[:, 0])
    q_got, q_want = got[:, 1:].copy(), want[:, 1:].copy()
    z = (q_got == 0) & (q_want == 0)
    q_got[z] = q_want[z] = 0.0
    assert_same(q_got, q_want)


def scale_matrix(rng, N, C, kind="wide"):
    """Scores with ties, negative values, both zeros and a wide range of magnitudes (so that any other summation order
    shows in the last bits)."""
    a = rng.standard_normal((N, C)).astype(np.float32)
    if kind == "wide":
        a *= np.float32(10.0) ** rng.uniform(-6, 6, (N, C)).astype(np.float32)
    elif kind == "ties":
        a = np.round(a * 2).astype(np.float32)
    elif kind == "zeros":
        z = np.where(rng.random((N, C)) < 0.5, np.float32(0.0), np.float32(-0.0))
        a = np.where(rng.random((N, C)) < 0.3, np.round(a), z)
    return np.ascontiguousarray(a, dtype=np.float32)


def test_percentile_restatement_equals_numpy():
    """np.percentile's linear method at 25 / 75 through the order statistics, on random float32 arrays of many
    lengths."""
    rng = np.random.default_rng(0)
    for it in range(160):
        n = int(rng.integers(1, 28480)) if it >= 20 else it + 1
        x = (rng.standard_normal(n) * 10.0 ** rng.uniform(-4, 4)).astype(np.float32)
        if it % 3 == 0:
            x = np.round(x).astype(np.float32)
        med, q25, q75 = column_stats(x)
        w75, w25 = np.percentile(x, [75, 25])
        assert bits(np.float64(q25)) == bits(w25) or q25 == w25 == 0
        assert bits(np.float64(q75)) == bits(w75) or q75 == w75 == 0
        assert bits(med) == bits(np.median(x))


@pytest.mark.parametrize("N", [1, 2, 3, 4, 5, 8, 1001])
@pytest.mark.parametrize("kind", ["wide", "ties", "zeros"])
def test_column_statistics_and_scaled_columns_equal_numpy(N, kind):
    rng = np.random.default_rng(N * 7 + len(kind))
    a = scale_matrix(rng, N, 9, kind)
    stats, scaled, g = host_scale(a)
    want_stats, want_scaled, want_g = numpy_scale(a)
    assert_same_stats(stats, want_stats)
    assert_same(scaled, want_scaled)
    assert scaled.dtype == np.float64 and g.dtype == np.float32
    assert_same(g, want_g)


@pytest.mark.parametrize("C", [1, 7, 8, 9, 38, 55, 128, 129, 300])
@pytest.mark.parametrize("N", [1, 2, 3, 4, 5, 8, 1001])
def test_global_mean_equals_numpy(N, C):
    rng = np.random.default_rng(1000 * N + C)
    a = scale_matrix(rng, N, C, "wide")
    _, scaled, g = host_scale(a)
    _, want_scaled, want_g = numpy_scale(a)
    assert_same(scaled, want_scaled)
    assert_same(g, want_g)
    x = scaled.astype(np.float32)
    assert_same(g, np.mean(x, 1))


def test_nan_column_and_constant_column():
    rng = np.random.default_rng(3)
    a = scale_matrix(rng, 1001, 5, "wide")
    a[17, 1] = np.nan
    a[:, 3] = np.float32(2.5)                                       # IQR 0: divisor 1
    with np.errstate(invalid="ignore"):
        stats, scaled, g = host_scale(a)
        want_stats, want_scaled, want_g = numpy_scale(a)
    assert np.isnan(stats[1]).all() and np.isnan(scaled[:, 1]).all() and np.isnan(g).all()
    assert stats[3].tolist() == [2.5, 2.5, 2.5] and (scaled[:, 3] == 0).all()
    assert_same_stats(stats, want_stats)
    assert_same(scaled, want_scaled)
    assert_same(g, want_g)


def test_signed_zero_median_and_first_partial_sum():
    """np.mean of the middle values starts from +0.0, so an all -0.0 column has the median +0.0 and its scaled values
    are -0.0 - +0.0 = -0.0; a row of -0.0 sums to +0.0."""
    a = np.full((4, 3), -0.0, np.float32)
    stats, scaled, g = host_scale(a)
    want_stats, want_scaled, want_g = numpy_scale(a)
    assert bits(np.float32(stats[0, 0])) == 0
    assert_same_stats(stats, want_stats)
    assert_same(scaled, want_scaled)
    assert_same(g, want_g)
