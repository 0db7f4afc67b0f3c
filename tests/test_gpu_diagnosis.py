"""Anomaly diagnosis on the device (thresholding.rank_features / diagnosis_eval, csrc/diagnose.cu): the ranking equals
np.argsort(-a, kind="stable") with ties, signed zeros, infinities and NaN; HitRate@P% and NDCG@P% against TranAD's
literal hit_att / ndcg on the host copy (Hit bitwise, NDCG to 1e-12), on tie-free and tied scores, float32 and float64,
strided views, several P, every label dtype, row masks and replay alarms; a model's scores through SeriesScorer; run to
run bitwise; the errors; one read-back per call and the stated launch counts."""
import numpy as np
import pytest
import torch

from tests import diagnosis_reference as ref

pytestmark = pytest.mark.gpu
PS = [100, 150, 250, 137.5]


def _tied(rng, m, out, dtype=np.float32, specials=True):
    """Scores from a few values (ties in every row), with signed zeros, infinities and NaN."""
    a = rng.integers(-3, 4, (m, out)).astype(dtype) / 2
    if specials:
        u = rng.random((m, out))
        a[u < 0.08] = -0.0
        a[(u >= 0.08) & (u < 0.12)] = np.inf
        a[(u >= 0.12) & (u < 0.15)] = -np.inf
        a[(u >= 0.15) & (u < 0.18)] = np.nan
    return a


def _tie_free(rng, m, out, dtype=np.float32):
    a = np.stack([rng.permutation(out) for _ in range(m)]).astype(np.float64) + rng.random((m, 1))
    return (a / out).astype(dtype)


def _labels(rng, m, out):
    lab = (rng.random((m, out)) < rng.uniform(0.03, 0.3, (m, 1))).astype(np.float32)
    lab[::5] = 0                                                       # rows with no labelled feature
    return lab


def _close(got, want, tied=False):
    """diagnosis_eval's dict against the literal one: Hit bitwise, NDCG to 1e-12 relative."""
    assert set(got) == set(want) | {"rows"}
    for key, v in want.items():
        if key.startswith("Hit"):
            assert got[key] == v, key
        else:
            assert got[key] == pytest.approx(v, rel=1e-12, abs=0), key


def _bits(d):
    return {k: (np.float64(v).view(np.int64) if isinstance(v, float) else v) for k, v in d.items()}


# ---------------------------------------------------------------------------------------------------------------------
# rank_features

@pytest.mark.parametrize("dtype", [np.float32, np.float64])
@pytest.mark.parametrize("out", [2, 31, 33, 38, 1024])
@pytest.mark.parametrize("strided", [False, True])
def test_rank_features_is_stable_argsort(dtype, out, strided):
    from mtad_gat_pytorch_b200 import thresholding as th
    rng = np.random.default_rng(out + strided)
    for m in (1, 257):
        a = _tied(rng, m, out, dtype)
        if strided:
            big = torch.from_numpy(_tied(rng, m, out + 7, dtype)).cuda()
            big[:, 3:3 + out] = torch.from_numpy(a).cuda()
            x = big[:, 3:3 + out]
            assert x.stride(0) == out + 7
        else:
            x = torch.from_numpy(a).cuda()
        got = th.rank_features(x)
        assert got.dtype == torch.int32 and got.shape == (m, out) and got.is_cuda
        assert np.array_equal(got.cpu().numpy(), np.argsort(-a, axis=1, kind="stable"))


@pytest.mark.parametrize("dtype", [np.float32, np.float64])
@pytest.mark.parametrize("out", [2, 38])
def test_rank_features_past_65535_rows(dtype, out):
    from mtad_gat_pytorch_b200 import thresholding as th
    a = _tied(np.random.default_rng(out), 70001, out, dtype)
    got = th.rank_features(torch.from_numpy(a).cuda())
    assert np.array_equal(got.cpu().numpy(), np.argsort(-a, axis=1, kind="stable"))


def test_rank_features_signed_zeros_infinities_nan():
    from mtad_gat_pytorch_b200 import thresholding as th
    a = np.array([[0.0, np.nan, -0.0, 2.0, np.inf, 2.0, -np.inf, np.nan]], np.float32)
    assert th.rank_features(torch.from_numpy(a).cuda()).cpu().tolist() == [[4, 3, 5, 0, 2, 6, 1, 7]]


# ---------------------------------------------------------------------------------------------------------------------
# diagnosis_eval against TranAD's code

@pytest.mark.parametrize("dtype", [np.float32, np.float64])
@pytest.mark.parametrize("out", [2, 38, 300])
def test_tie_free_scores_equal_literal_code(dtype, out):
    from mtad_gat_pytorch_b200 import thresholding as th
    rng = np.random.default_rng(out)
    m = 1500 if out < 300 else 200
    a, lab = _tie_free(rng, m, out, dtype), _labels(rng, m, out)
    got = th.diagnosis_eval(torch.from_numpy(a).cuda(), lab, ps=PS)
    _close(got, ref.literal(a, lab, PS))
    assert got["rows"] == int(lab.any(1).sum())


@pytest.mark.parametrize("dtype", [np.float32, np.float64])
def test_tied_scores_hit_by_the_rule_ndcg_by_sklearn(dtype):
    from mtad_gat_pytorch_b200 import thresholding as th
    rng = np.random.default_rng(5)
    a, lab = _tied(rng, 1200, 38, dtype, specials=False), _labels(rng, 1200, 38)
    a[rng.random(a.shape) < 0.1] = -0.0
    got = th.diagnosis_eval(torch.from_numpy(a).cuda(), lab, ps=PS)
    want = ref.restated(a, lab, PS)
    sk = ref.ndcg(a, lab.astype(np.float64), PS)
    for p in PS:
        assert got[f"Hit@{p}%"] == want[f"Hit@{p}%"]
        assert got[f"NDCG@{p}%"] == pytest.approx(sk[f"NDCG@{p}%"], rel=1e-12, abs=0)
        assert got[f"NDCG@{p}%"] == pytest.approx(want[f"NDCG@{p}%"], rel=1e-12, abs=0)
    assert got["rows"] == want["rows"]


def test_infinite_scores_rank_as_values():
    """sklearn refuses infinite scores; the device ranks them as ordinary values, as the stated rule does."""
    from mtad_gat_pytorch_b200 import thresholding as th
    rng = np.random.default_rng(6)
    a, lab = _tied(rng, 600, 38), _labels(rng, 600, 38)
    a[np.isnan(a)] = 1.25
    got, want = th.diagnosis_eval(torch.from_numpy(a).cuda(), lab, ps=PS), ref.restated(a, lab, PS)
    for key in want:
        assert got[key] == want[key] if key.startswith(("Hit", "rows")) else \
            got[key] == pytest.approx(want[key], rel=1e-12, abs=0)


def test_strided_view_is_read_in_place_and_runs_repeat():
    from mtad_gat_pytorch_b200 import thresholding as th
    rng = np.random.default_rng(7)
    a, lab = _tie_free(rng, 900, 38, np.float64), _labels(rng, 900, 38)
    big = torch.zeros(900, 50, dtype=torch.float64, device="cuda")
    big[:, 5:43] = torch.from_numpy(a).cuda()
    x = big[:, 5:43]
    one = th.diagnosis_eval(x, lab, ps=PS)
    assert _bits(one) == _bits(th.diagnosis_eval(torch.from_numpy(a).cuda(), lab, ps=PS))
    assert _bits(one) == _bits(th.diagnosis_eval(x, lab, ps=PS))


def test_label_dtypes_numpy_and_cuda():
    from mtad_gat_pytorch_b200 import thresholding as th
    rng = np.random.default_rng(8)
    a, lab = _tie_free(rng, 800, 38), _labels(rng, 800, 38)
    x = torch.from_numpy(a).cuda()
    want = th.diagnosis_eval(x, lab, ps=PS)
    _close(want, ref.literal(a, lab, PS))
    for dt, tdt in ((np.float32, torch.float32), (np.int64, torch.int64), (np.bool_, torch.bool)):
        host = lab.astype(dt)
        assert _bits(th.diagnosis_eval(x, host, ps=PS)) == _bits(want)
        assert _bits(th.diagnosis_eval(x, torch.from_numpy(host).cuda(), ps=PS)) == _bits(want)
        assert _bits(th.diagnosis_eval(x, torch.from_numpy(host), ps=PS)) == _bits(want)


def test_rows_without_labels_are_skipped():
    from mtad_gat_pytorch_b200 import thresholding as th
    rng = np.random.default_rng(9)
    a, lab = _tie_free(rng, 700, 38), _labels(rng, 700, 38)
    lab[:100] = 0
    a2 = np.concatenate([a, _tie_free(rng, 300, 38)])
    lab2 = np.concatenate([lab, np.zeros((300, 38), np.float32)])
    one = th.diagnosis_eval(torch.from_numpy(a).cuda(), lab, ps=PS)
    assert _bits(th.diagnosis_eval(torch.from_numpy(a2).cuda(), lab2, ps=PS)) == _bits(one)
    assert one["rows"] == int(lab.any(1).sum())
    nothing = th.diagnosis_eval(torch.from_numpy(a).cuda(), np.zeros_like(lab), ps=PS)
    assert nothing["rows"] == 0 and all(np.isnan(v) for k, v in nothing.items() if k != "rows")


# ---------------------------------------------------------------------------------------------------------------------
# row masks

def test_masks_equal_single_calls_and_the_rule():
    from mtad_gat_pytorch_b200 import thresholding as th
    rng = np.random.default_rng(10)
    m = 1100
    a, lab = _tie_free(rng, m, 38), _labels(rng, m, 38)
    x = torch.from_numpy(a).cuda()
    masks = (rng.random((6, m)) < np.array([0.5, 0.1, 0.9, 0.0, 1.0, 0.02])[:, None]).astype(np.uint8)
    masks[1] *= 2                                                      # biSPOT's lower alarm code selects too
    many = th.diagnosis_eval(x, lab, ps=PS, rows=torch.from_numpy(masks).cuda())
    assert isinstance(many, list) and len(many) == 6
    for r in range(6):
        single = th.diagnosis_eval(x, lab, ps=PS, rows=masks[r])
        assert _bits(many[r]) == _bits(single)
        assert _bits(th.diagnosis_eval(x, lab, ps=PS, rows=torch.from_numpy(masks[r] != 0).cuda())) == _bits(single)
    assert many[3]["rows"] == 0 and all(np.isnan(v) for k, v in many[3].items() if k != "rows")
    assert _bits(many[4]) == _bits(th.diagnosis_eval(x, lab, ps=PS))
    want = ref.restated(a, lab, PS, rows=masks[0] != 0)
    assert many[0]["rows"] == want["rows"]
    for p in PS:
        assert many[0][f"Hit@{p}%"] == want[f"Hit@{p}%"]
        assert many[0][f"NDCG@{p}%"] == pytest.approx(want[f"NDCG@{p}%"], rel=1e-12, abs=0)


def test_replay_alarms_as_rows():
    from mtad_gat_pytorch_b200 import thresholding as th
    from tests.test_gpu_replay import _grid, _series
    m = 2500
    tr, s = _series(11, 1500, m)
    grid = _grid()
    alarms = th.replay(tr, s, grid)["alarms"]
    assert (alarms == 2).any() and (alarms == 1).any()
    rng = np.random.default_rng(12)
    a, lab = _tie_free(rng, m, 38), _labels(rng, m, 38)
    x = torch.from_numpy(a).cuda()
    res = th.diagnosis_eval(x, lab, ps=PS, rows=alarms)
    assert len(res) == len(grid)
    for c in range(len(grid)):
        assert _bits(res[c]) == _bits(th.diagnosis_eval(x, lab, ps=PS, rows=alarms[c]))
    c = int(torch.argmax((alarms == 2).sum(1)))
    sel = alarms[c].cpu().numpy() != 0
    _close(res[c], ref.literal(a[sel], lab[sel], PS))


# ---------------------------------------------------------------------------------------------------------------------
# a model's scores

@pytest.mark.parametrize("scale", [False, True])
def test_series_scorer_a_score(scale):
    import mtad_gat_pytorch_b200 as mg
    from mtad_gat_pytorch_b200 import scoring, thresholding as th
    torch.manual_seed(0)
    model = mg.MTAD_GAT(6, 20, 6, kernel_size=3, gru_hid_dim=16, forecast_hid_dim=12, recon_hid_dim=10).cuda().eval()
    rng = np.random.default_rng(13)
    series = rng.random((900, 6)).astype(np.float32)
    res = scoring.SeriesScorer(model, batch=256).score(torch.from_numpy(series), scale_scores=scale)
    a_score = res["a_score"]
    assert a_score.dtype == (torch.float64 if scale else torch.float32)
    a = a_score.cpu().numpy()
    lab = _labels(rng, a.shape[0], 6)
    got = th.diagnosis_eval(a_score, lab, ps=PS)
    tie_free = all(len(set(r.tolist())) == r.size for r in a)
    want = ref.literal(a, lab, PS) if tie_free else ref.restated(a, lab, PS)
    for p in PS:
        assert got[f"Hit@{p}%"] == want[f"Hit@{p}%"]
    _close({k: v for k, v in got.items() if not k.startswith("Hit")},
           {k: v for k, v in ref.ndcg(a, lab.astype(np.float64), PS).items()})
    assert np.array_equal(th.rank_features(a_score).cpu().numpy(), np.argsort(-a, axis=1, kind="stable"))


# ---------------------------------------------------------------------------------------------------------------------
# errors, read-backs, launches

def test_nan_scores_and_bad_cuda_labels_raise():
    from mtad_gat_pytorch_b200 import thresholding as th
    rng = np.random.default_rng(14)
    a, lab = _tie_free(rng, 300, 38), _labels(rng, 300, 38)
    lab[7] = 0
    lab[8, 3] = 1
    a[8, 5] = np.nan
    x = torch.from_numpy(a).cuda()
    with pytest.raises(ValueError, match="NaN"):
        th.diagnosis_eval(x, lab)
    a[8, 5] = 0.5
    a[7, 5] = np.nan                                                   # a row with no labelled feature is not evaluated
    th.diagnosis_eval(torch.from_numpy(a).cuda(), lab)
    a[8, 5] = np.nan
    keep = np.ones(300, bool)
    keep[8] = False
    th.diagnosis_eval(torch.from_numpy(a).cuda(), lab, rows=keep)    # nor a row no mask selects
    a[8, 5] = 0.5
    x = torch.from_numpy(a).cuda()
    for bad in (torch.from_numpy(lab).cuda() * 0.5, torch.from_numpy(lab).cuda().long() * 2,
                torch.from_numpy(lab).cuda().to(torch.uint8) * 3):
        with pytest.raises(ValueError, match="0 or 1"):
            th.diagnosis_eval(x, bad)


def test_one_read_back_and_the_stated_launch_counts(monkeypatch):
    import mtad_gat_pytorch_b200 as mg
    from mtad_gat_pytorch_b200 import thresholding as th
    rng = np.random.default_rng(15)
    a, lab = _tie_free(rng, 1000, 38), _labels(rng, 1000, 38)
    x = torch.from_numpy(a).cuda()
    lab_d = torch.from_numpy(lab).cuda()
    masks = torch.from_numpy((rng.random((40, 1000)) < 0.3).astype(np.uint8)).cuda()
    th.diagnosis_eval(x, lab_d, ps=PS, rows=masks)                     # warm-up
    torch.cuda.synchronize()
    calls = []
    real_cpu = torch.Tensor.cpu

    def counting_cpu(self, *args, **kw):
        calls.append(self.device.type)
        return real_cpu(self, *args, **kw)

    def refuse(fn):
        def wrapped(self, *args, **kw):
            assert not self.is_cuda, f"{fn.__name__} on a CUDA tensor"
            return fn(self, *args, **kw)
        return wrapped
    for name in ("item", "tolist", "numpy"):
        monkeypatch.setattr(torch.Tensor, name, refuse(getattr(torch.Tensor, name)))
    monkeypatch.setattr(torch.Tensor, "cpu", counting_cpu)
    for rows, R in ((None, 1), (masks, 40), (masks[:1], 1)):
        calls.clear()
        mg.reset_launch_count()
        res = th.diagnosis_eval(x, lab_d, ps=PS, rows=rows)
        assert calls == ["cuda"]
        assert mg.launch_count() == 3
        assert (len(res) if isinstance(res, list) else 1) == R
    calls.clear()
    mg.reset_launch_count()
    th.rank_features(x)
    assert calls == [] and mg.launch_count() == 1
