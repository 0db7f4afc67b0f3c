"""CPU tests for stream state records: record validation (prediction.check_state_record), the model digest, and the
history positions of the ring and linear layouts (scoring.history_rows) against a plain restatement."""
import copy

import numpy as np
import pytest
import torch

N, K, OUT, WORDS, NT_WORD = 6, 3, 2, 24, 2


def _record(B=3, seed=0):
    from mtad_gat_pytorch_b200 import prediction
    rng = np.random.default_rng(seed)
    nt = rng.integers(0, 9, B)
    spot = torch.from_numpy(rng.integers(0, 1 << 40, (B, WORDS)).astype(np.int64))
    spot[:, NT_WORD] = torch.from_numpy(nt)
    return {"format": prediction.STATE_FORMAT, "version": 1, "n": N, "k": K, "out": OUT, "gamma": 0.5,
            "target_dims": None, "with_alarm": True, "level": 0.9, "model_digest": "abc",
            "rows": torch.tensor([0, N, 3 * N + 1][:B], dtype=torch.int64),
            "hist": torch.from_numpy(rng.random((B, N, K)).astype(np.float32)),
            "last_pred": torch.zeros(B, OUT), "spot": spot,
            "peak_offsets": torch.from_numpy(np.concatenate([[0], np.cumsum(nt)]).astype(np.int64)),
            "peaks": torch.from_numpy(rng.random(int(nt.sum())).astype(np.float32)), "errors": "flag"}


EXPECT = {"n": N, "k": K, "out": OUT, "gamma": 0.5, "target_dims": None, "with_alarm": True}


def _check(rec, expect=EXPECT, digest="abc"):
    from mtad_gat_pytorch_b200 import prediction
    return prediction.check_state_record(rec, expect, lambda: digest, "import")


def test_a_valid_record_is_accepted_and_survives_torch_save(tmp_path):
    rec = _record()
    torch.save(rec, tmp_path / "state.pt")
    loaded = torch.load(tmp_path / "state.pt", weights_only=True)
    got = _check(loaded)
    assert got["B"] == 3 and got["rows"].tolist() == rec["rows"].tolist()
    assert torch.equal(got["peaks"], rec["peaks"]) and got["peak_offsets"].tolist() == rec["peak_offsets"].tolist()
    assert _check(rec, {"n": N})["B"] == 3                              # a key left out of expect is only type-checked


def _mutations():
    def setter(key, value):
        def f(r):
            r[key] = value
        return f

    def tensor(key, fn):
        def f(r):
            r[key] = fn(r[key])
        return f

    def nt_word(r):
        r["spot"][1, NT_WORD] += 1

    def offsets_down(r):
        off = r["peak_offsets"].clone()
        off[1], off[2] = off[2] + 1, off[1]
        r["peak_offsets"] = off
    return {
        "not a dict": lambda r: r.clear(),
        "format": setter("format", "other"), "version 2": setter("version", 2), "version bool": setter("version", True),
        "missing peaks": lambda r: r.pop("peaks"),
        "n": setter("n", N + 1), "k": setter("k", K - 1), "out": setter("out", OUT + 1), "gamma": setter("gamma", 0.25),
        "target_dims": setter("target_dims", [0, 1]), "with_alarm": setter("with_alarm", False),
        "with_alarm int": setter("with_alarm", 1), "level": setter("level", "0.9"), "digest type": setter("model_digest", 3),
        "hist shape": tensor("hist", lambda t: t[:, :-1]), "hist dtype": tensor("hist", lambda t: t.double()),
        "last_pred shape": tensor("last_pred", lambda t: t[:2]), "spot dtype": tensor("spot", lambda t: t.int()),
        "rows 2-D": tensor("rows", lambda t: t[None]), "rows dtype": tensor("rows", lambda t: t.int()),
        "rows numpy": tensor("rows", lambda t: t.numpy()), "peaks dtype": tensor("peaks", lambda t: t.half()),
        "offsets length": tensor("peak_offsets", lambda t: t[:-1]),
        "offsets start": tensor("peak_offsets", lambda t: t + 1),
        "offsets end": tensor("peaks", lambda t: torch.cat([t, t[:1]])),
        "offsets order": offsets_down, "Nt word": nt_word,
        "rows < 0": tensor("rows", lambda t: t - 1),
        "no stream": lambda r: r.update(rows=r["rows"][:0], hist=r["hist"][:0], last_pred=r["last_pred"][:0],
                                        spot=r["spot"][:0], peak_offsets=r["peak_offsets"][:1], peaks=r["peaks"][:0]),
    }


@pytest.mark.parametrize("case", list(_mutations()))
def test_bad_records_are_refused(case):
    rec = copy.deepcopy(_record())
    _mutations()[case](rec)
    with pytest.raises(ValueError, match="^import: "):
        _check(rec)


def test_digest_mismatch_is_refused_after_the_other_checks():
    calls = []

    def digest():
        calls.append(1)
        return "other"
    from mtad_gat_pytorch_b200 import prediction
    with pytest.raises(ValueError, match="model_digest"):
        prediction.check_state_record(_record(), EXPECT, digest, "import")
    rec = _record()
    rec["n"] = 99
    with pytest.raises(ValueError, match="n 99"):
        prediction.check_state_record(rec, EXPECT, digest, "import")
    assert calls == [1]                                                 # the weights are not read for a refused shape


def _cpu_model():
    import mtad_gat_pytorch_b200 as mg
    torch.manual_seed(0)
    return mg.MTAD_GAT(5, 20, 5, kernel_size=3, gru_hid_dim=16, forecast_hid_dim=12, recon_hid_dim=10)


def test_digest_follows_the_weights_only():
    from mtad_gat_pytorch_b200 import prediction
    a = _cpu_model()
    b = copy.deepcopy(a)
    d = prediction.model_digest(a)
    assert len(d) == 64 and d == prediction.model_digest(b) == prediction.model_digest(a.eval())
    c = _cpu_model()
    c.load_state_dict({k: v.clone() for k, v in a.state_dict().items()})
    assert prediction.model_digest(c) == d
    name, p = next(iter(b.state_dict().items()))
    with torch.no_grad():
        flat = p.view(-1)
        flat[3] = torch.nextafter(flat[3], torch.tensor(np.inf))        # one ulp
    assert prediction.model_digest(b) != d
    assert name in dict(a.named_parameters()) or name in dict(a.named_buffers())


def test_history_rows_restate_the_ring_and_linear_layouts():
    from mtad_gat_pytorch_b200.scoring import history_rows
    for n in (1, 4, 7):
        for rows in range(0, 4 * n + 3):
            h = min(rows, n)
            ring = [g % n for g in range(rows - h, rows)]                # a ring keeps row g at g % n
            assert history_rows(rows, n).tolist() == ring
            assert history_rows(rows, n, ring=False).tolist() == list(range(h))
            assert sorted(ring) == list(range(h))                       # distinct positions, 0 .. h-1 before a wrap
