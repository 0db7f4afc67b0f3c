"""CPU tests for per-feature SPOT on live streams (the detectors' per_feature=True): the per-feature record keys and
each refusal of check_state_record, the argument checks, and the host restatement of the gather / scatter index maps
(tests/feature_reference.py) on ragged offsets with streams that have no rows."""
import copy

import numpy as np
import pytest
import torch

from tests import feature_reference as fr
from tests.test_stream_state_cpu import EXPECT, N, OUT, WORDS, NT_WORD, _record

N_WORD, DEPTH = 1, 4


def _side(rng, B, n_words=None):
    nt = rng.integers(0, 7, B)
    spot = torch.from_numpy(rng.integers(0, 1 << 40, (B, WORDS)).astype(np.int64))
    spot[:, NT_WORD] = torch.from_numpy(nt)
    if n_words is not None:
        spot[:, N_WORD] = n_words
    return [spot, torch.from_numpy(np.concatenate([[0], np.cumsum(nt)]).astype(np.int64)),
            torch.from_numpy(rng.random(int(nt.sum())).astype(np.float32))]


def _feature_record(B=3, depth=None, bidirectional=False, seed=1):
    """A per-feature record: `_record`'s plus the B * OUT feature streams' keys for the rule."""
    rng = np.random.default_rng(seed)
    rec = _record(B, seed)
    rec["per_feature"] = True
    keys = ("feature_spot", "feature_peak_offsets", "feature_peaks")
    rec.update(zip(keys, _side(rng, B * OUT)))
    if depth is not None:
        rec["depth"], rec["window"] = depth, torch.from_numpy(rng.random((B, depth)).astype(np.float32))
        rec["feature_window"] = torch.from_numpy(rng.random((B * OUT, depth)).astype(np.float32))
    if bidirectional:
        rec["bidirectional"] = True
        lower = _side(rng, B, rec["spot"][:, N_WORD])
        rec.update(zip(("spot_lower", "peak_offsets_lower", "peaks_lower"), lower))
        rec.update(zip(("feature_spot_lower", "feature_peak_offsets_lower", "feature_peaks_lower"),
                       _side(rng, B * OUT, rec["feature_spot"][:, N_WORD])))
    return rec


def _check(rec, expect=None):
    from mtad_gat_pytorch_b200 import prediction
    return prediction.check_state_record(rec, dict(EXPECT, per_feature=True) if expect is None else expect,
                                         lambda: "abc", "import")


@pytest.mark.parametrize("depth,bidirectional", [(None, False), (DEPTH, False), (None, True), (DEPTH, True)])
def test_a_valid_feature_record_is_accepted_and_survives_torch_save(depth, bidirectional, tmp_path):
    rec = _feature_record(depth=depth, bidirectional=bidirectional)
    torch.save(rec, tmp_path / "state.pt")
    got = _check(torch.load(tmp_path / "state.pt", weights_only=True),
                 dict(EXPECT, per_feature=True, depth=depth, bidirectional=bidirectional))
    assert got["per_feature"] is True and got["B"] == 3
    assert torch.equal(got["feature_spot"], rec["feature_spot"])
    assert got["feature_peak_offsets"].tolist() == rec["feature_peak_offsets"].tolist()
    assert (got.get("feature_window") is not None) == (depth is not None)
    assert ("feature_spot_lower" in got) == bidirectional


def test_records_without_features_keep_their_keys():
    from mtad_gat_pytorch_b200 import prediction
    cfg = {"n": N, "k": 3, "out": OUT, "gamma": 0.5, "target_dims": None, "with_alarm": True, "depth": None,
           "bidirectional": False, "per_feature": False}
    rec = prediction._record(cfg, 0.9, "abc", [1], {})
    assert "per_feature" not in rec and "depth" not in rec and "bidirectional" not in rec
    assert prediction._record(dict(cfg, per_feature=True), 0.9, "abc", [1], {})["per_feature"] is True
    assert prediction.STATE_VERSION == 1
    assert _check(_record(), dict(EXPECT, per_feature=False))["per_feature"] is False


def _mutations():
    def tensor(key, fn):
        def f(r):
            r[key] = fn(r[key])
        return f

    def nt_word(key):
        def f(r):
            r[key][4, NT_WORD] += 1
        return f

    def offsets_down(r):
        off = r["feature_peak_offsets"].clone()
        off[1] = int(off[2]) + 1
        r["feature_peak_offsets"] = off

    def lower_n(r):
        r["feature_spot_lower"][2, N_WORD] += 1
    return {
        "per_feature not True": (lambda r: r.update(per_feature=1), "per_feature must be True"),
        "per_feature False": (lambda r: r.update(per_feature=False), "must be True"),
        "feature keys without per_feature": (lambda r: r.pop("per_feature"), "no per-feature state"),
        "missing feature_peaks": (lambda r: r.pop("feature_peaks"), r"lacks \['feature_peaks'\]"),
        "feature_window without depth": (lambda r: r.update(feature_window=torch.zeros(3 * OUT, 2)), "no use"),
        "lower half on a one-sided record": (lambda r: r.update(feature_spot_lower=r["feature_spot"]), "no use"),
        "feature_spot rows": (tensor("feature_spot", lambda t: t[:-1]), "feature_spot must be"),
        "feature_spot dtype": (tensor("feature_spot", lambda t: t.int()), "feature_spot must be"),
        "feature_spot words": (tensor("feature_spot", lambda t: t[:, :-1]), "feature_spot must be"),
        "feature offsets length": (tensor("feature_peak_offsets", lambda t: t[:-1]), "feature_peak_offsets must be"),
        "feature offsets dtype": (tensor("feature_peak_offsets", lambda t: t.int()), "feature_peak_offsets must be"),
        "feature peaks dtype": (tensor("feature_peaks", lambda t: t.double()), "feature_peaks must be"),
        "feature offsets start": (tensor("feature_peak_offsets", lambda t: t + 1), "must rise"),
        "feature offsets end": (tensor("feature_peaks", lambda t: torch.cat([t, t[:1]])), "must rise"),
        "feature offsets order": (offsets_down, "must rise"),
        "feature Nt word": (nt_word("feature_spot"), r"feature Nt word of stream\(s\) \[4\]"),
    }, {
        "feature_window missing": (lambda r: r.pop("feature_window"), r"lacks \['feature_window'\]"),
        "feature_window shape": (tensor("feature_window", lambda t: t[:, :-1]), "feature_window must be"),
        "feature_window dtype": (tensor("feature_window", lambda t: t.double()), "feature_window must be"),
        "lower half missing": (lambda r: r.pop("feature_peaks_lower"), r"lacks \['feature_peaks_lower'\]"),
        "lower rows": (tensor("feature_spot_lower", lambda t: t[:-1]), "feature_spot_lower must be"),
        "lower offsets order": (tensor("feature_peak_offsets_lower", lambda t: t.flip(0)), "must rise"),
        "lower Nt word": (nt_word("feature_spot_lower"), r"feature lower Nt word of stream\(s\) \[4\]"),
        "lower N word": (lower_n, r"feature lower N word of stream\(s\) \[2\] differs"),
    }


@pytest.mark.parametrize("case", list(_mutations()[0]))
def test_bad_feature_records_are_refused(case):
    rec = copy.deepcopy(_feature_record())
    fn, msg = _mutations()[0][case]
    fn(rec)
    with pytest.raises(ValueError, match="^import: .*" + msg):
        _check(rec, dict(EXPECT, depth=None, bidirectional=False))


@pytest.mark.parametrize("case", list(_mutations()[1]))
def test_bad_two_sided_drift_feature_records_are_refused(case):
    rec = copy.deepcopy(_feature_record(depth=DEPTH, bidirectional=True))
    fn, msg = _mutations()[1][case]
    fn(rec)
    with pytest.raises(ValueError, match="^import: .*" + msg):
        _check(rec, dict(EXPECT, depth=DEPTH, bidirectional=True))


def test_records_do_not_cross_between_detectors_with_and_without_features():
    with pytest.raises(ValueError, match="a per-feature record does not enter a detector without features"):
        _check(_feature_record(), dict(EXPECT, per_feature=False))
    with pytest.raises(ValueError, match="a record without features does not enter a per-feature detector"):
        _check(_record(), dict(EXPECT, per_feature=True))
    assert _check(_feature_record(), dict(EXPECT))["per_feature"] is True      # per_feature left out: accepted


def test_per_feature_must_be_a_bool():
    from mtad_gat_pytorch_b200 import prediction
    for bad in (1, "yes", None, np.bool_(True)):
        with pytest.raises(ValueError, match="StreamDetector: per_feature must be True or False"):
            prediction.StreamDetector(None, None, per_feature=bad)
        with pytest.raises(ValueError, match="FleetDetector: per_feature must be True or False"):
            prediction.FleetDetector(None, [None], per_feature=bad)


def test_entry_points_refuse_bad_arguments():
    """The library's argument checks return before anything is launched, so they run without a GPU."""
    from mtad_gat_pytorch_b200._lib import lib
    p = 1 << 20                                                        # never dereferenced
    gather = lib.mtadgat_feature_gather
    assert gather(None, 4, 2, None, None, 1, p, p, None) != 0
    assert b"null pointer" in lib.mtadgat_last_error()
    assert gather(p, 0, 2, None, None, 1, p, p, None) != 0               # no rows
    assert gather(p, 4, 0, None, None, 1, p, p, None) != 0               # no feature
    assert gather(p, 4, 2, p, None, 1, p, p, None) != 0                  # streams without offsets
    assert gather(p, 4, 2, None, None, 3, p, p, None) != 0               # several streams without offsets
    scatter = lib.mtadgat_feature_scatter
    assert scatter(p, None, None, 4, 2, None, None, p, None, p, None) != 0
    assert scatter(p, p, p, 4, 2, None, None, p, None, p, None) != 0      # lower thresholds without their output
    assert scatter(p, None, p, 4, 2, None, p, p, None, p, None) != 0      # offsets without streams
    assert scatter(p, None, p, -1, 2, None, None, p, None, p, None) != 0


def _restated(offsets, out):
    """The layout written out stream by stream and feature by feature, as a loop."""
    dst, foff, pos = {}, [], 0
    for s in range(len(offsets) - 1):
        for i in range(out):
            foff.append(pos)
            for r in range(offsets[s], offsets[s + 1]):
                dst[r * out + i] = pos
                pos += 1
    return np.array([dst[e] for e in range(len(dst))], np.int64), np.array(foff + [pos], np.int64)


@pytest.mark.parametrize("offsets,out", [([0, 3, 3, 7, 8, 8], 3), ([0, 0, 5], 2), ([0, 6], 4), ([0, 1, 2, 3], 1),
                                         ([0, 0, 0], 3)])
def test_gather_and_scatter_maps_restate_the_layout(offsets, out):
    dst, foff = fr.feature_map(offsets, out)
    want_dst, want_foff = _restated(offsets, out)
    assert dst.tolist() == want_dst.tolist() and foff.tolist() == want_foff.tolist()
    M = offsets[-1]
    assert sorted(dst.tolist()) == list(range(M * out))               # a permutation
    a = np.arange(M * out, dtype=np.float32).reshape(M, out) + 0.5
    fm, foff = fr.gather(a, offsets)
    for s in range(len(offsets) - 1):
        for i in range(out):
            j = s * out + i
            assert fm[foff[j]:foff[j + 1]].tolist() == a[offsets[s]:offsets[s + 1], i].tolist()
    assert np.array_equal(fr.scatter(fm, offsets, out), a)
    one_fm, one_foff = fr.gather(a, [0, M])                            # null tables: all rows are one stream
    assert np.array_equal(one_fm, a.T.reshape(-1)) and one_foff.tolist() == [M * i for i in range(out + 1)]
