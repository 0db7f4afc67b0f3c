"""GPU tests of predict_anomalies on the device: the SMAP / MSL channel adjustment (csrc/channels.cu), numpy's row mean
(mtadgat_row_mean), the float64 per-feature epsilons, and `prediction.SeriesPredictor` end to end against the restated
predict_anomalies tail (oracle/prediction_oracle.py) run at the device's thresholds."""
import json
import os
import shutil

import numpy as np
import pandas as pd
import pytest
import torch

from oracle import pot_oracle
from oracle import prediction_oracle as po
from oracle import thresholding_oracle as tho
from tests.test_prediction_cpu import write_metadata
from tests.test_scale_scores_cpu import assert_same, scale_matrix

pytestmark = pytest.mark.gpu


def assert_adjusted(got, want):
    """Bitwise, NaN equal to NaN and a zero equal to a zero of either sign."""
    got, want = np.asarray(got), np.asarray(want)
    assert got.dtype == want.dtype == np.float32 and got.shape == want.shape
    nan = np.isnan(want)
    assert np.array_equal(np.isnan(got), nan)
    zero = (want == 0) & (got == 0)
    keep = ~nan & ~zero
    assert np.array_equal(got.view(np.uint32)[keep], want.view(np.uint32)[keep]), np.flatnonzero(
        got.view(np.uint32)[keep] != want.view(np.uint32)[keep])[:5]


def channel_case(rng, m, N, lookback=100, short=False):
    """(zero_idx, bounds) of m channels whose cumulative lengths end at N + lookback, as channel_bounds forms them."""
    if short:
        sizes = rng.integers(1, 4, m)
        sizes[0] = lookback + 1
    else:
        w = rng.random(m) + 0.05
        sizes = np.maximum(np.round(w / w.sum() * (N + lookback)).astype(np.int64), 2)
        sizes[0] = max(sizes[0], lookback + 1)
    sizes[-1] += N + lookback - sizes.sum()
    assert sizes[-1] > 0
    sep = np.cumsum(sizes) - lookback
    bounds = np.concatenate([[0], sep]).astype(np.int64)
    z = np.concatenate([(sep[:-1, None] + np.arange(1, 20)).ravel(), (sep[:-1, None] - np.arange(1, 20)).ravel()])
    return np.unique(z[(z >= 0) & (z < N)]).astype(np.int64), bounds


def device_adjust(x, zero, bounds, alias=False):
    from mtad_gat_pytorch_b200._lib import lib, check
    n = x.size
    s = torch.from_numpy(x).cuda()
    out = s if alias else torch.full_like(s, 7.0)
    z = torch.from_numpy(zero).cuda()
    b = torch.from_numpy(bounds).cuda()
    scratch = torch.empty((int(lib.mtadgat_channel_adjust_scratch_bytes(n, b.numel())) + 7) // 8, dtype=torch.int64,
                          device="cuda")
    check(lib.mtadgat_channel_adjust(s.data_ptr(), n, z.data_ptr() if z.numel() else None, z.numel(), b.data_ptr(),
                                     b.numel(), out.data_ptr(), scratch.data_ptr(),
                                     torch.cuda.current_stream().cuda_stream))
    return out.cpu().numpy()


@pytest.mark.parametrize("N,m", [(427617, 54), (135183, 27), (28479, 54), (300, 3)])
@pytest.mark.parametrize("kind", ["random", "nan", "constant", "short", "alias"])
def test_channel_adjust_equals_restatement(N, m, kind):
    rng = np.random.default_rng(N + m + len(kind))
    zero, bounds = channel_case(rng, m, N, short=(kind == "short"))
    N = int(bounds[-1])
    x = (rng.random(N) * 10.0 ** rng.uniform(-3, 3, N)).astype(np.float32)
    if kind == "nan":
        x[rng.integers(bounds[m // 2] + 1, bounds[m // 2 + 1])] = np.nan
    if kind == "constant":                       # the last segment's interior equals the value its head arrives with
        j = m - 1
        zero = zero[zero <= bounds[j]]
        with np.errstate(invalid="ignore", divide="ignore"):
            head = po.normalise_segments(x, zero, bounds[:j + 1])[bounds[j]]
        x[bounds[j] + 1:] = head
    with np.errstate(invalid="ignore", divide="ignore"):
        want = po.normalise_segments(x, zero, bounds)
    got = device_adjust(x, zero, bounds, alias=(kind == "alias"))
    assert_adjusted(got, want)
    if kind in ("nan", "constant"):
        assert np.isnan(want).any()


def test_channel_adjust_from_metadata(tmp_path, monkeypatch):
    """adjust_anomaly_scores (the host metadata + the device) equals the statement-by-statement restatement."""
    from mtad_gat_pytorch_b200 import prediction
    monkeypatch.chdir(tmp_path)
    rng = np.random.default_rng(4)
    write_metadata(str(tmp_path), "SMAP", list(rng.integers(300, 9000, 54)), list(rng.integers(300, 9000, 54)))
    for is_train in (True, False):
        md = pd.read_csv("datasets/data/smap_train_md.csv" if is_train else "datasets/data/labeled_anomalies.csv")
        md = md[md["chan_id"] != "P-2"]
        if not is_train:
            md = md[md["spacecraft"] == "SMAP"]
        x = rng.random(int(md["num_values"].sum()) - 100).astype(np.float32)
        d = torch.from_numpy(x).cuda()
        got = prediction.adjust_anomaly_scores(d, "SMAP", is_train, 100)
        assert_adjusted(got.cpu().numpy(), po.adjust_anomaly_scores(x, "SMAP", is_train, 100))
        assert prediction.adjust_anomaly_scores(d, "SMAP", is_train, 100, out=d) is d
        assert_adjusted(d.cpu().numpy(), got.cpu().numpy())
        assert prediction.adjust_anomaly_scores(d, "SMD", is_train, 100) is d


def test_channel_adjust_graph_replay_on_new_data():
    from mtad_gat_pytorch_b200._lib import lib, check
    rng = np.random.default_rng(9)
    zero, bounds = channel_case(rng, 54, 427617)
    n = int(bounds[-1])
    x = torch.zeros(n, device="cuda")
    out = torch.zeros(n, device="cuda")
    z, b = torch.from_numpy(zero).cuda(), torch.from_numpy(bounds).cuda()
    scratch = torch.empty((int(lib.mtadgat_channel_adjust_scratch_bytes(n, b.numel())) + 7) // 8, dtype=torch.int64,
                          device="cuda")
    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    g = torch.cuda.CUDAGraph()
    with torch.cuda.stream(s), torch.cuda.graph(g, stream=s):
        check(lib.mtadgat_channel_adjust(x.data_ptr(), n, z.data_ptr(), z.numel(), b.data_ptr(), b.numel(),
                                         out.data_ptr(), scratch.data_ptr(), s.cuda_stream))
    for seed in (10, 11):
        h = np.random.default_rng(seed).random(n).astype(np.float32)
        x.copy_(torch.from_numpy(h))
        out.zero_()
        g.replay()
        torch.cuda.synchronize()
        assert_adjusted(out.cpu().numpy(), po.normalise_segments(h, zero, bounds))


@pytest.mark.parametrize("C", [1, 7, 8, 38, 55, 129, 300])
def test_row_mean_equals_numpy(C):
    from mtad_gat_pytorch_b200 import scoring
    rng = np.random.default_rng(C)
    for N in (1, 1001, 28479 if C <= 55 else 3001):
        a = scale_matrix(rng, N, C, "wide")
        wide = torch.full((N, C + 5), 3.0, device="cuda")
        wide[:, 2:2 + C] = torch.from_numpy(a).cuda()
        got = scoring.row_mean(wide[:, 2:2 + C])
        assert_same(got.cpu().numpy(), np.mean(a, 1))
        assert_same(scoring.row_mean(torch.from_numpy(a).cuda()).cpu().numpy(), np.mean(a, 1))


def _oracle_z(e, eps):
    """The z of find_epsilon's winning candidate (-1 when it returned max(e))."""
    if eps == np.max(e):
        return -1.0
    return float(np.round((eps - np.mean(e)) / np.std(e) * 2) / 2)


def test_float64_column_epsilons():
    from mtad_gat_pytorch_b200._lib import lib, check
    from mtad_gat_pytorch_b200 import scoring
    from tests.test_oracle_golden import _score_series
    n, C = 5000, 9
    raw = np.stack([_score_series(c, n) for c in range(C)], 1)
    raw[:, 4] = 0.5                                                       # no candidate qualifies: max
    scaled, _, _ = scoring.robust_scale(torch.from_numpy(raw).cuda())
    wide = torch.zeros((n, C + 3), dtype=torch.float64, device="cuda")
    wide[:, 1:1 + C] = scaled
    x = wide[:, 1:1 + C]
    xh = scaled.cpu().numpy()
    out = torch.empty(3 * C, dtype=torch.float64, device="cuda")
    scratch = torch.empty(int(lib.mtadgat_find_epsilon_columns_scratch_doubles(n, C)), dtype=torch.float64,
                          device="cuda")
    stream = torch.cuda.current_stream().cuda_stream
    check(lib.mtadgat_find_epsilon_columns_f64(x.data_ptr(), n, C, x.stride(0), 2, out.data_ptr(), scratch.data_ptr(),
                                               stream))
    o = out.cpu().numpy()
    for c in range(C):
        ref = float(tho.find_epsilon(xh[:, c], 2))
        assert abs(o[c] - ref) <= 2e-6 * max(1.0, abs(ref)), c
        assert o[C + c] == _oracle_z(xh[:, c], ref), c
    assert o[C + 4] == -1 and o[4] == xh[:, 4].max()
    pred = torch.empty((n, C), dtype=torch.bool, device="cuda")
    check(lib.mtadgat_compare_columns_f64(x.data_ptr(), n, C, x.stride(0), out.data_ptr(), 1, pred.data_ptr(), stream))
    assert np.array_equal(pred.cpu().numpy(), xh >= o[None, :C])


# ---------------------------------------------------------------------------------------------------------------------
# SeriesPredictor end to end

WINDOW = 20


def _model_and_series():
    import mtad_gat_pytorch_b200 as mg
    torch.manual_seed(0)
    m = mg.MTAD_GAT(5, WINDOW, 5, kernel_size=3, gru_hid_dim=16, forecast_hid_dim=12, recon_hid_dim=10).cuda().eval()
    rng = np.random.default_rng(0)
    train = rng.random((3020, 5)).astype(np.float32)
    test = rng.random((1520, 5)).astype(np.float32)
    test[700:720] += 2.0
    test[1100:1104] += 1.0
    labels = np.zeros(1500, np.float32)
    labels[675:705] = 1
    labels[1075:1090] = 1
    return m, train, test, labels


def _pred_args(dataset, scale, dynamic, save_path):
    return dict(dataset=dataset, target_dims=None, scale_scores=scale, q=1e-3, level=0.95, dynamic_pot=dynamic,
                use_mov_av=False, gamma=1, reg_level=1, save_path=save_path)


def _read(d):
    with open(os.path.join(d, "summary.txt")) as f:
        summary = json.load(f)
    return summary, [pd.read_pickle(os.path.join(d, f"{k}_output.pkl")) for k in ("train", "test")]


def _oracle_at_device_thresholds(pred_args, labels, frames, summary, dev_frames, load_scores=False):
    """The restated tail with the device's epsilons and POT threshold injected (and bf_search / the threshold
    evaluations in closed form)."""
    eps_iter = iter([dev_frames[0][f"Thresh_{i}"].iloc[0] for i in range(5)])

    def find_epsilon(e, reg_level):
        return next(eps_iter)

    def epsilon_eval(tr, te, lab, reg_level=1):
        t = np.float64(summary["epsilon_result"]["threshold"])
        if lab is None:
            return {"threshold": t, "reg_level": reg_level}
        r = po.fast_threshold_eval(te, lab, t)
        r["reg_level"] = reg_level
        return r

    def pot_eval(tr, te, lab, q=1e-3, level=0.99, dynamic=False):
        t = np.float64(summary["pot_result"]["threshold"])
        return {"threshold": t} if lab is None else po.fast_threshold_eval(te, lab, t)

    return po.predict_tail(pred_args, WINDOW, 5, labels, *(frames or (None, None)), load_scores=load_scores,
                           find_epsilon=find_epsilon, epsilon_eval=epsilon_eval, pot_eval=pot_eval,
                           bf_search=po.fast_bf_search)


CASES = [(dataset, scale, labelled, False) for dataset in ("SMD", "SMAP") for scale in (False, True)
         for labelled in (True, False)] + [("SMAP", scale, True, True) for scale in (False, True)]


@pytest.mark.parametrize("dataset,scale,labelled,dynamic", CASES)
def test_predict_anomalies_end_to_end(tmp_path, monkeypatch, dataset, scale, labelled, dynamic):
    from mtad_gat_pytorch_b200 import prediction, scoring
    monkeypatch.chdir(tmp_path)
    write_metadata(str(tmp_path), "SMAP", [1000, 1200, 820], [500, 600, 420])
    m, train, test, labels = _model_and_series()
    lab = labels if labelled else None
    dev_dir, orc_dir = str(tmp_path / "device"), str(tmp_path / "oracle")
    os.makedirs(dev_dir)
    os.makedirs(orc_dir)
    p = prediction.SeriesPredictor(m, WINDOW, 5, _pred_args(dataset, scale, dynamic, dev_dir))
    returned = p.predict_anomalies(train, test, lab)
    summary, dev_frames = _read(dev_dir)
    assert returned == summary

    frames = [scoring.score_dataframe(m, torch.from_numpy(x), scale_scores=scale) for x in (train, test)]
    with np.errstate(invalid="ignore", divide="ignore"):
        tr_adj = po.adjust_anomaly_scores(frames[0]["A_Score_Global"].values, dataset, True, WINDOW)
        te_adj = po.adjust_anomaly_scores(frames[1]["A_Score_Global"].values, dataset, False, WINDOW)
        s_orc, f_tr, f_te = _oracle_at_device_thresholds(_pred_args(dataset, scale, dynamic, orc_dir), lab,
                                                         frames, summary, dev_frames)
    for got, want in zip(dev_frames, (f_tr, f_te)):
        pd.testing.assert_frame_equal(got, want, check_exact=True)
    assert summary.keys() == s_orc.keys()
    for key in summary:
        assert summary[key] == s_orc[key], key

    # the thresholds themselves against the oracle's
    eps = float(tho.find_epsilon(tr_adj, 1))
    assert abs(summary["epsilon_result"]["threshold"] - eps) <= 2e-6 * max(1.0, abs(eps))
    for i in range(5):
        col = frames[0][f"A_Score_{i}"].values
        ref = float(tho.find_epsilon(col, 2))
        assert abs(dev_frames[0][f"Thresh_{i}"].iloc[0] - ref) <= 2e-6 * max(1.0, abs(ref)), i
    model = pot_oracle.pot_model(tr_adj, te_adj, q=1e-3, level=0.95, dynamic=dynamic)
    assert abs(summary["pot_result"]["threshold"] - model["pot_th"]) <= 1e-12 * max(1.0, abs(model["pot_th"]))
    if not labelled:
        assert summary["bf_result"] == {} and set(summary["pot_result"]) == {"threshold"}
        assert set(summary["epsilon_result"]) == {"threshold", "reg_level"}
        assert dev_frames[1]["A_True_Global"].isna().all()

    # load_scores: the saved pickles again, with the reference's second adjustment of the saved global score
    if labelled and not dynamic:
        for name in ("train_output.pkl", "test_output.pkl"):
            shutil.copyfile(os.path.join(dev_dir, name), os.path.join(orc_dir, name))
        again = p.predict_anomalies(None, None, lab, load_scores=True)
        summary2, dev_frames2 = _read(dev_dir)
        assert again == summary2
        with np.errstate(invalid="ignore", divide="ignore"):
            s_orc2, f_tr2, f_te2 = _oracle_at_device_thresholds(_pred_args(dataset, scale, dynamic, orc_dir), lab,
                                                                None, summary2, dev_frames2, load_scores=True)
        for got, want in zip(dev_frames2, (f_tr2, f_te2)):
            pd.testing.assert_frame_equal(got, want, check_exact=True)
        assert summary2 == s_orc2
        if dataset == "SMD":
            assert summary2 == summary
        eps2 = float(tho.find_epsilon(f_tr2["A_Score_Global"].values, 1))
        assert abs(summary2["epsilon_result"]["threshold"] - eps2) <= 2e-6 * max(1.0, abs(eps2))


def test_evaluate_reads_back_once(tmp_path, monkeypatch):
    """SeriesPredictor.evaluate at SMAP size: one device-to-host copy."""
    from mtad_gat_pytorch_b200 import prediction
    monkeypatch.chdir(tmp_path)
    rng = np.random.default_rng(6)
    tr_sizes, te_sizes = rng.integers(1000, 4000, 54), rng.integers(3000, 12000, 54)
    write_metadata(str(tmp_path), "SMAP", list(tr_sizes), list(te_sizes))
    n_tr, n_te = int(tr_sizes.sum()) - 100, int(te_sizes.sum()) - 100
    scores = []
    for n in (n_tr, n_te):
        a = torch.from_numpy(rng.random((n, 1)).astype(np.float32)).cuda()
        scores.append({"a_score": a, "a_global": a[:, 0].clone()})
    labels = np.zeros(n_te, np.float32)
    labels[5000:5200] = 1
    labels[90000:90500] = 1
    m = torch.nn.Linear(1, 1).cuda()
    p = prediction.SeriesPredictor(m, 100, 1, _pred_args("SMAP", False, False, str(tmp_path)))
    p.evaluate(*scores, labels)                                          # warm-up
    torch.cuda.synchronize()
    calls = []
    real_cpu = torch.Tensor.cpu

    def counting_cpu(self, *a, **k):
        calls.append(self.device)
        return real_cpu(self, *a, **k)
    for name in ("item", "tolist", "numpy"):
        monkeypatch.setattr(torch.Tensor, name, _refuse_on_device(getattr(torch.Tensor, name)))
    monkeypatch.setattr(torch.Tensor, "cpu", counting_cpu)
    tensors, summary = p.evaluate(*scores, labels)
    assert [d.type for d in calls] == ["cuda"]
    assert set(summary) == {"epsilon_result", "pot_result", "bf_result"} and summary["bf_result"]
    assert tensors["test_pred_global"].shape == (n_te,) and tensors["train_pred"].shape == (n_tr, 1)


def _refuse_on_device(fn):
    def wrapped(self, *a, **k):
        assert not self.is_cuda, f"{fn.__name__} on a CUDA tensor"
        return fn(self, *a, **k)
    return wrapped


def test_use_mov_av_raises(tmp_path):
    from mtad_gat_pytorch_b200 import prediction
    m, train, test, labels = _model_and_series()
    args = _pred_args("SMD", False, False, str(tmp_path))
    args["use_mov_av"] = True
    p = prediction.SeriesPredictor(m, WINDOW, 5, args)
    with pytest.raises(NotImplementedError):
        p.predict_anomalies(train, test, labels)
    assert not os.listdir(tmp_path)
