"""Host-side index arithmetic of the fleet scorer (scoring.fleet_tables): window tables, completed-timestamp indices and
offsets against a plain per-stream restatement of scoring.StreamScorer.push's arithmetic, over random push schedules."""
import numpy as np
import pytest


@pytest.fixture(scope="module")
def scoring():
    import __graft_entry__ as ge
    ge.build()
    from mtad_gat_pytorch_b200 import scoring as sc
    return sc


def restated(streams, rows_before, n):
    """Per stream, StreamScorer.push's arithmetic, with every row named by (stream, stream-local row index)."""
    S = len(rows_before)
    windows, stamps, last, offsets = [], [], [], [0]
    ring = {}
    for s in range(S):
        mine = [p for p, q in enumerate(streams) if q == s]             # pushed rows of s, in arrival order
        R0, R1 = rows_before[s], rows_before[s] + len(mine)
        for j, p in enumerate(mine):
            if R0 + j >= R1 - n:
                ring[p] = s * n + (R0 + j) % n
        a = max(0, R0 - n)
        m_out = max(0, R1 - n - a)
        w0 = max(0, R0 - n + 1)
        c = R1 - n - w0 + 1 if R1 >= n and mine else 0
        base = len(windows)
        for w in range(w0, w0 + c):
            rows = [("ring", s * n + g % n) if g < R0 else ("new", mine[g - R0]) for g in range(w, w + n)]
            windows.append((s, w, rows))
        for i in range(a, a + m_out):
            f = ("last", s) if i < w0 else ("win", base + i - w0)
            stamps.append((s, i, f, base + i + 1 - w0, mine[i + n - R0]))
        if c:
            last.append((base + c - 1, s))
        offsets.append(len(stamps))
    return windows, stamps, last, offsets, ring


@pytest.mark.parametrize("seed", range(6))
def test_fleet_tables_against_per_stream_restatement(scoring, seed):
    rng = np.random.default_rng(seed)
    S, n = int(rng.integers(1, 7)), int(rng.integers(2, 9))
    rows_before = np.zeros(S, np.int64)
    for _ in range(25):
        counts = rng.choice([0, 0, 1, 1, 2, 3, n, n + 3], S)
        streams = rng.permutation(np.repeat(np.arange(S), counts))
        t = scoring.fleet_tables(streams, rows_before, n)
        windows, stamps, last, offsets, ring = restated(streams.tolist(), rows_before.tolist(), n)
        R = streams.size
        assert sorted(t["perm"].tolist()) == list(range(R))
        assert np.all(np.diff(streams[t["perm"]]) >= 0)
        for s in range(S):                                              # arrival order kept inside a stream
            assert np.all(np.diff(t["perm"][streams[t["perm"]] == s]) > 0)
        assert {int(t["perm"][p]): int(d) for p, d in enumerate(t["hist_dst"]) if d >= 0} == ring
        assert t["win"].shape == (4, len(windows))
        for b, (s, w, rows) in enumerate(windows):
            ws, wf, n_old, xpos = (int(v) for v in t["win"][:, b])
            assert (ws, wf) == (s, w)
            got = [("ring", s * n + (wf + j) % n) if j < n_old else ("new", int(t["perm"][xpos + j - n_old]))
                   for j in range(n)]
            assert got == rows
            assert all(streams[p] == s for kind, p in rows if kind == "new")      # never another stream's rows
        assert t["ts"].shape == (3, len(stamps))
        for e, (s, i, f, r, arow) in enumerate(stamps):
            fs, rs, ar = (int(v) for v in t["ts"][:, e])
            assert (int(t["ts_stream"][e]), int(t["ts_index"][e])) == (s, i)
            assert (("last", -1 - fs) if fs < 0 else ("win", fs)) == f
            assert (rs, ar) == (r, arow)
        assert t["offsets"].tolist() == offsets
        assert [tuple(int(v) for v in col) for col in t["last"].T] == last
        rows_before = rows_before + np.bincount(streams, minlength=S)


def test_fleet_tables_empty_push(scoring):
    t = scoring.fleet_tables(np.zeros(0, np.int64), np.array([3, 0]), 4)
    assert t["win"].shape == (4, 0) and t["ts"].shape == (3, 0) and t["offsets"].tolist() == [0, 0, 0]
    assert all(v.dtype == np.int64 for v in t.values())
