"""Host references for the small SIMT kernels of the training and scoring path: the Philox4x32-10 dropout stream
(csrc/common.cuh, csrc/api.cu), the RMSE loss pair, Adam and the score epilogue (csrc/loss.cu), and the window and ring
movement of csrc/fleet.cu and csrc/series.cu.  Test infrastructure only: tests/test_gpu_simt_stages.py compares the
kernels with these, tests/test_simt_reference_cpu.py pins these without a GPU (Philox to the published Random123
known-answer vectors, Adam to torch.optim.Adam, the loss to torch autograd, the fleet tables to a per-stream model).

Philox is restated in numpy uint64 arithmetic on uint32 words; the arithmetic references are float64; the data-movement
references move float32 words and are compared bit for bit."""
import numpy as np

M32 = np.uint64(0xFFFFFFFF)
PHILOX_M0, PHILOX_M1 = np.uint64(0xD2511F53), np.uint64(0xCD9E8D57)
PHILOX_W0, PHILOX_W1 = 0x9E3779B9, 0xBB67AE85
SEED_STEP = 0x9E3779B97F4A7C15
MASK64 = (1 << 64) - 1


# ---- Philox4x32-10 and the dropout multipliers ----------------------------------------------------------------------
def philox4x32_10(ctr, key):
    """Random123's philox4x32_10: ctr = four uint32 words (scalars or equal-shape arrays), key = two.  Returns the four
    output words as uint32 arrays.  One round: (hi, lo) = M0 * c0 and M1 * c2 as 64-bit products, then
    c = (hi1 ^ c1 ^ k0, lo1, hi0 ^ c3 ^ k1, lo0); the key is bumped by the Weyl constants between rounds."""
    c = [np.asarray(w, dtype=np.uint64) & M32 for w in ctr]
    c = list(np.broadcast_arrays(*c))
    k0, k1 = int(key[0]) & 0xFFFFFFFF, int(key[1]) & 0xFFFFFFFF
    for _ in range(10):
        p0, p1 = PHILOX_M0 * c[0], PHILOX_M1 * c[2]
        hi0, lo0, hi1, lo1 = p0 >> np.uint64(32), p0 & M32, p1 >> np.uint64(32), p1 & M32
        c = [hi1 ^ c[1] ^ np.uint64(k0), lo1, hi0 ^ c[3] ^ np.uint64(k1), lo0]
        k0, k1 = (k0 + PHILOX_W0) & 0xFFFFFFFF, (k1 + PHILOX_W1) & 0xFFFFFFFF
    return [w.astype(np.uint32) for w in c]


def philox_uniform(seed, stream, numel):
    """The uniforms of elements 0 .. numel-1 of dropout stream `stream` under `seed` (float32): element idx takes word
    idx & 3 of the block with counter (idx >> 2, idx >> 34, stream, 0x9E3779B9) and key (seed low, seed high), and
    maps it to (word >> 8) * 2^-24."""
    seed = int(seed) & MASK64
    blocks = (int(numel) + 3) // 4
    b = np.arange(blocks, dtype=np.uint64)
    words = philox4x32_10((b & M32, b >> np.uint64(32), np.full(blocks, stream, dtype=np.uint64),
                           np.full(blocks, 0x9E3779B9, dtype=np.uint64)), (seed & 0xFFFFFFFF, seed >> 32))
    w = np.stack(words, axis=1).reshape(-1)[:int(numel)]
    return (w >> np.uint32(8)).astype(np.float32) * np.float32(2.0 ** -24)


def philox_uniform_at(seed, stream, idx):
    """philox_uniform at arbitrary element indices idx (uint64), one Philox block per element"""
    seed = int(seed) & MASK64
    idx = np.asarray(idx, dtype=np.uint64)
    c = idx >> np.uint64(2)
    words = philox4x32_10((c & M32, c >> np.uint64(32), np.full(idx.shape, stream, dtype=np.uint64),
                           np.full(idx.shape, 0x9E3779B9, dtype=np.uint64)), (seed & 0xFFFFFFFF, seed >> 32))
    w = np.choose((idx & np.uint64(3)).astype(np.int64), words)
    return (w >> np.uint32(8)).astype(np.float32) * np.float32(2.0 ** -24)


def dropout_mask(u, p):
    """The multipliers for uniforms u at drop probability p: u >= p keeps with 1/(1-p), else 0 (float32, as the entry
    point takes p)."""
    p = np.float32(p)
    return np.where(u >= p, np.float32(1.0) / (np.float32(1.0) - p), np.float32(0.0)).astype(np.float32)


def keep_probability(p):
    """P(u >= p) for u uniform on the 2^24-point grid of philox_uniform"""
    return 1.0 - np.ceil(float(np.float32(p)) * 2.0 ** 24) / 2.0 ** 24


def seed_advance(seed):
    return (int(seed) + SEED_STEP) & MASK64


# ---- RMSE pair --------------------------------------------------------------------------------------------------------
def rmse_sum(a, b):
    """sum over i of float32 (a_i - b_i)^2, the products as the kernel forms them, added in float64"""
    d = (np.asarray(a, dtype=np.float32) - np.asarray(b, dtype=np.float32)).astype(np.float32)
    return float(np.sum((d * d).astype(np.float64)))


def rmse_exact(a, b):
    """sqrt(mean((a - b)^2)) in float64"""
    d = np.asarray(a, dtype=np.float64) - np.asarray(b, dtype=np.float64)
    return float(np.sqrt(np.mean(d * d)))


def rmse_grad(a, b, loss, g):
    """d loss / d a times the upstream gradient g: g (a - b) / (n loss), float64, for the float32 `loss`"""
    a, b = np.asarray(a, dtype=np.float64), np.asarray(b, dtype=np.float64)
    return float(g) * (a - b) / (a.size * float(loss))


def ulp32(x):
    """the spacing of float32 at |x| (elementwise, float64)"""
    return np.spacing(np.abs(np.asarray(x, dtype=np.float64)).astype(np.float32)).astype(np.float64)


# ---- Adam -------------------------------------------------------------------------------------------------------------
def bias_corrections_f32(beta1, beta2, t):
    """(1 - b1^t, 1 - b2^t) as torch.optim.Adam(capturable=True) forms them for a CUDA graph: the step counter is a
    float32 device tensor, so b^t is a float32 power (correctly rounded) and 1 - b^t a float32 subtraction"""
    one = np.float32(1.0)
    return tuple(float(one - np.float32(float(np.float32(b)) ** float(np.float32(t)))) for b in (beta1, beta2))


def adam_step(p, g, m, v, step, lr, beta1, beta2, eps, capturable=False):
    """One torch.optim.Adam step (no weight decay, no amsgrad) in float64 after `step` steps taken:
    m = b1 m + (1-b1) g, v = b2 v + (1-b2) g^2, p -= lr / (1 - b1^t) * m / (sqrt(v) / sqrt(1 - b2^t) + eps), t = step+1.
    capturable: the two bias corrections 1 - b^t as the graph-capturable step forms them (bias_corrections_f32), the rest
    in float64; otherwise all of it in float64, as the eager step does.  Returns (p, m, v) as float64."""
    p, g, m, v = (np.asarray(a, dtype=np.float64) for a in (p, g, m, v))
    m = beta1 * m + (1.0 - beta1) * g
    v = beta2 * v + (1.0 - beta2) * g * g
    return p - adam_update_per_m(v, step, lr, beta1, beta2, eps, capturable) * m, m, v


def adam_update_per_m(v, step, lr, beta1, beta2, eps, capturable=False):
    """d(update)/dm of adam_step for the new second moment v: lr / (1 - b1^t) / (sqrt(v) / sqrt(1 - b2^t) + eps)"""
    t = float(step) + 1.0
    bc1, bc2 = bias_corrections_f32(beta1, beta2, t) if capturable else (1.0 - beta1 ** t, 1.0 - beta2 ** t)
    return (lr / bc1) / (np.sqrt(np.asarray(v, dtype=np.float64)) / np.sqrt(bc2) + eps)


# ---- score epilogues --------------------------------------------------------------------------------------------------
def score_f32(p, r, actual, gamma):
    """prediction.py's per-feature score in float32 numpy: sqrt((p - a)^2) + gamma * sqrt((r - a)^2)"""
    p, r, a = (np.asarray(x, dtype=np.float32) for x in (p, r, actual))
    g = np.float32(gamma)
    with np.errstate(over="ignore", invalid="ignore"):
        return (np.sqrt((p - a) ** 2) + g * np.sqrt((r - a) ** 2)).astype(np.float32)


def epilogue_actual(series, target, n, n_windows):
    """actual[i][c] = series[n + i][target[c]] (target None: c)"""
    rows = np.asarray(series)[n:n + n_windows]
    return rows if target is None else rows[:, np.asarray(target)]


def indexed_operands(preds, last_preds, recons, rows, tab, m, target):
    """(forecast, recon, actual) of mtadgat_score_epilogue_indexed for tab = (f, r, a) rows: forecast = preds[f] for
    f >= 0, last_preds[-1 - f] otherwise; recon = recons[r]; actual = rows[a][target]"""
    f, r, a = (np.asarray(t[:m], dtype=np.int64) for t in tab)
    fc = np.where((f >= 0)[:, None], preds[np.maximum(f, 0)], last_preds[np.maximum(-1 - f, 0)])
    act = rows[a] if target is None else rows[a][:, np.asarray(target)]
    return fc, recons[r], act


def row_mean64(a):
    with np.errstate(over="ignore", invalid="ignore"):
        return np.asarray(a, dtype=np.float64).mean(axis=1)


# ---- window and ring movement -----------------------------------------------------------------------------------------
class FleetPush:
    """One push of new rows to S live streams, stated per stream: stream s has data[s] (its whole history, rows
    0 .. before[s] + new[s] - 1), its ring holds rows before[s] - n .. before[s] - 1 at hist[s][g % n], and the push
    brings rows before[s] .. of every stream interleaved in arrival order `rows`.

    Windows: every window of n consecutive rows of a stream that ends at one of its new rows, plus the window that ends
    at its last ring row (entirely in the ring), in a shuffled order.  The tables are the ones the kernels take:
    perm (sorted position -> pushed row), win (4, ld) = {s, first, n_old, xpos}, row_tab (2, R) = {pushed row, ring row
    s*n + g%n or -1 when the row is not among its stream's last n}."""

    def __init__(self, S, n, k, new, before, rng, pad=3):
        self.S, self.n, self.k = S, n, k
        self.new, self.before = np.asarray(new, dtype=np.int64), np.asarray(before, dtype=np.int64)
        self.data = [rng.standard_normal((int(b + c), k)).astype(np.float32) for b, c in zip(self.before, self.new)]
        self.hist = rng.standard_normal((S, n, k)).astype(np.float32)          # slots of streams with < n rows: junk
        for s in range(S):
            for g in range(max(0, int(self.before[s]) - n), int(self.before[s])):
                self.hist[s, g % n] = self.data[s][g]
        arrivals = np.concatenate([np.full(c, s) for s, c in enumerate(self.new)]).astype(np.int64)
        rng.shuffle(arrivals)                                    # interleaved arrival, each stream's rows in order
        R = arrivals.size
        self.rows = np.empty((R, k), dtype=np.float32)
        seen = np.zeros(S, dtype=np.int64)
        self.row_stream, self.row_g = np.empty(R, dtype=np.int64), np.empty(R, dtype=np.int64)
        for r, s in enumerate(arrivals):
            g = self.before[s] + seen[s]
            self.rows[r] = self.data[s][g]
            self.row_stream[r], self.row_g[r] = s, g
            seen[s] += 1
        self.perm = np.lexsort((np.arange(R), arrivals)).astype(np.int64)           # grouped by stream, arrival order
        group = np.concatenate([[0], np.cumsum(self.new)])
        wins = []
        for s in range(self.S):
            b = int(self.before[s])
            for end in range(b - 1, b + int(self.new[s])):
                first = end - n + 1
                if first < 0:
                    continue
                wins.append((s, first, max(0, b - first), group[s] + max(0, first - b)))
        wins = np.asarray(wins, dtype=np.int64).reshape(-1, 4)
        rng.shuffle(wins)
        self.count = len(wins)
        self.ld = self.count + pad
        self.win = np.full((4, self.ld), -7, dtype=np.int64)       # the columns past count are never read
        self.win[:, :self.count] = wins.T
        dst = np.full(R, -1, dtype=np.int64)
        for p in range(R):
            r = self.perm[p]
            s, g = self.row_stream[r], self.row_g[r]
            if g >= self.before[s] + self.new[s] - n:
                dst[p] = s * n + g % n
        self.row_tab = np.stack([self.perm, dst])

    def windows(self):
        """(count, n, k): window b = rows first .. first + n - 1 of its stream"""
        return np.stack([self.data[s][f:f + self.n] for s, f in self.win[:2, :self.count].T]) if self.count else \
            np.zeros((0, self.n, self.k), dtype=np.float32)

    def hist_after(self):
        """the rings once every stream has taken its new rows"""
        h = self.hist.copy()
        for s in range(self.S):
            end = int(self.before[s] + self.new[s])
            for g in range(max(int(self.before[s]), end - self.n), end):
                h[s, g % self.n] = self.data[s][g]
        return h


def gather_windows(series, idx, counter, count, n):
    """x[b] = series[i : i + n], y[b] = series[i + n] with i = idx[counter][b]"""
    starts = np.asarray(idx)[int(counter), :count]
    x = np.stack([series[i:i + n] for i in starts])
    y = np.stack([series[i + n:i + n + 1] for i in starts])
    return x, y
