"""CPU tests for per-stream detector configurations: normalisation and defaults of thresholding.stream_configs, and the
checks of per-stream stream state records (prediction.check_state_record): configs, ragged window offsets, the lower
half for every stream, and a per-stream record refused by a detector with one configuration for all streams."""
import numpy as np
import pytest
import torch

from tests.test_stream_state_cpu import K, N, OUT, WORDS, _record

NT_WORD, Q_WORD = 2, 7
DEFAULTS = {"q": 1e-3, "level": 0.99, "depth": None, "bidirectional": False, "with_alarm": True}
CFGS = [{"q": 1e-3, "level": 0.98, "depth": None, "bidirectional": False, "with_alarm": True},
        {"q": 1e-4, "level": 0.99, "depth": 4, "bidirectional": True, "with_alarm": False},
        {"q": 1e-3, "level": 0.995, "depth": 2, "bidirectional": False, "with_alarm": True}]


def test_configs_take_the_defaults_and_normalise():
    from mtad_gat_pytorch_b200 import thresholding as th
    got = th.stream_configs([{}, {"depth": 0, "q": 1e-4}, {"bidirectional": 1, "depth": np.int64(3)}], [10, 10, 10],
                            dict(DEFAULTS, level=0.98, with_alarm=False), "SpotStreams")
    assert got[0] == dict(DEFAULTS, level=0.98, with_alarm=False)
    assert got[1]["depth"] is None and got[1]["q"] == 1e-4
    assert got[2]["bidirectional"] is True and got[2]["depth"] == 3 and type(got[2]["depth"]) is int
    assert all(set(c) == set(th._REPLAY_KEYS) for c in got)


@pytest.mark.parametrize("cfg, match", [
    ({"depht": 3}, "stream 1: a mapping"),
    ({"depth": 10}, "stream 1: 10 training scores"),
    ({"depth": -1}, "stream 1: depth"),
    ({"bidirectional": True, "level": 0.5}, "stream 1: a two-sided stream needs level"),
    ({"level": 1.0}, "stream 1: level"),
    ({"q": 0}, "stream 1: q"),
    ("depth", "stream 1: a mapping"),
])
def test_bad_configs_name_the_stream(cfg, match):
    from mtad_gat_pytorch_b200 import thresholding as th
    with pytest.raises(ValueError, match=match):
        th.stream_configs([{}, cfg], [20, 10], DEFAULTS, "SpotStreams")


def test_config_count_must_match_the_streams():
    from mtad_gat_pytorch_b200 import thresholding as th
    with pytest.raises(ValueError, match="2 streams but 1 configurations"):
        th.stream_configs([{}], [20, 10], DEFAULTS, "SpotStreams")


def _per_stream_record():
    rec = _record(3)
    for key in ("with_alarm", "level"):
        del rec[key]
    rec["configs"] = [dict(c) for c in CFGS]
    rec["spot"][:, Q_WORD] = torch.from_numpy(np.array([c["q"] for c in CFGS]).view(np.int64))
    lower = torch.zeros(3, WORDS, dtype=torch.int64)
    lower[1] = torch.arange(WORDS)
    lower[1, NT_WORD] = 2
    lower[1, 1] = rec["spot"][1, 1]                                    # the N word, shared with the upper block
    rec.update(spot_lower=lower, peak_offsets_lower=torch.tensor([0, 0, 2, 2]), peaks_lower=torch.ones(2),
               window=torch.arange(6, dtype=torch.float32), window_offsets=torch.tensor([0, 0, 4, 6]))
    return rec


EXPECT = {"n": N, "k": K, "out": OUT, "gamma": 0.5, "target_dims": None}


def _check(rec, expect):
    from mtad_gat_pytorch_b200 import prediction
    return prediction.check_state_record(rec, expect, lambda: "abc", "import")


def test_a_valid_per_stream_record_is_accepted():
    rec = _check(_per_stream_record(), dict(EXPECT, per_stream=True))
    assert rec["configs"] == CFGS and rec["window_offsets"].tolist() == [0, 0, 4, 6]
    assert rec["spot_lower"].shape == (3, WORDS)


def test_a_uniform_record_takes_the_per_stream_form():
    uni = _record(2)
    uni["spot"][:, Q_WORD] = torch.from_numpy(np.array([1e-3, 1e-4]).view(np.int64))
    rec = _check(uni, dict(EXPECT, per_stream=True))
    assert [c["q"] for c in rec["configs"]] == [1e-3, 1e-4]
    assert all(c["level"] == 0.9 and c["depth"] is None and not c["bidirectional"] for c in rec["configs"])
    assert not rec["spot_lower"].any() and rec["window"].numel() == 0


def test_a_detector_with_one_configuration_refuses_a_per_stream_record():
    with pytest.raises(ValueError, match="per-stream record \\(configs\\)"):
        _check(_per_stream_record(), dict(EXPECT, with_alarm=True, per_stream=False))


def _mutations():
    def cfg(b, key, value):
        def f(r):
            r["configs"][b][key] = value
        return f

    def drop_cfg_key(r):
        del r["configs"][0]["q"]

    def q_word(r):
        r["spot"][0, Q_WORD] = torch.tensor([1e-2], dtype=torch.float64).view(torch.int64)[0]

    def one_sided_lower(r):
        r["spot_lower"][0, 3] = 1

    def lower_n(r):
        r["spot_lower"][1, 1] += 1

    def lower_shape(r):
        r["spot_lower"] = r["spot_lower"][:2]

    def window_offsets(r):
        r["window_offsets"] = torch.tensor([0, 1, 4, 6])

    def window_length(r):
        r["window"] = r["window"][:5]

    def uniform_key(r):
        r["depth"] = 4

    def missing(r):
        del r["window_offsets"]

    def not_a_list(r):
        r["configs"] = tuple(r["configs"])

    return [("configs", not_a_list), ("configs", drop_cfg_key),
            ("stream 1: a two-sided stream needs level", cfg(1, "level", 0.4)),
            ("bools", cfg(0, "with_alarm", 1)), ("depth", cfg(2, "depth", 5000)), ("q of configs", q_word),
            ("lower block of a one-sided", one_sided_lower), ("lower N word", lower_n), ("spot_lower", lower_shape),
            ("window_offsets", window_offsets), ("window", window_length), ("has no", uniform_key),
            ("lacks", missing)]


@pytest.mark.parametrize("match, mutate", _mutations())
def test_bad_per_stream_records_are_refused(match, mutate):
    rec = _per_stream_record()
    mutate(rec)
    with pytest.raises(ValueError, match=match):
        _check(rec, dict(EXPECT, per_stream=True))
