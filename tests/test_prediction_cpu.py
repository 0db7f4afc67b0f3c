"""CPU tests of predict_anomalies' host pieces: the restatement of utils.py adjust_anomaly_scores (hand-computed cases
and, when the reference is staged, the reference's own function), `prediction.channel_bounds`, and the restated
predict_anomalies tail against the reference's Predictor(load_scores=True)."""
import os
import sys
import types

import numpy as np
import pandas as pd
import pytest

from oracle import prediction_oracle as po

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
REF_DIR = os.path.join(ROOT, "baseline", "_ref")


def write_metadata(directory, dataset, train_sizes, test_sizes, other=(("MSL", "M-1", 77),)):
    """Synthetic channel metadata in the reference's layout under directory/datasets/data: `{dataset}_train_md.csv`
    (chan_id, num_values) and `labeled_anomalies.csv` (chan_id, spacecraft, num_values) with rows of another
    spacecraft, a P-2 row and shuffled channel order."""
    d = os.path.join(directory, "datasets", "data")
    os.makedirs(d, exist_ok=True)
    rng = np.random.default_rng(len(train_sizes))
    names = [f"{chr(65 + i % 26)}-{i // 26 + 1}" for i in range(len(train_sizes))]
    order = rng.permutation(len(names))
    pd.DataFrame({"chan_id": [names[i] for i in order] + ["P-2"],
                  "num_values": [train_sizes[i] for i in order] + [5000]}).to_csv(
        os.path.join(d, f"{dataset.lower()}_train_md.csv"), index=False)
    rows = [(names[i], dataset.upper(), test_sizes[i]) for i in order] + [("P-2", dataset.upper(), 4000)] + list(
        (c, sc, nv) for sc, c, nv in other)
    pd.DataFrame(rows, columns=["chan_id", "spacecraft", "num_values"]).to_csv(
        os.path.join(d, "labeled_anomalies.csv"), index=False)
    return names


def test_shared_endpoint_is_normalised_twice_and_can_become_the_next_minimum():
    # segments [0..3] and [3..6]: element 3 (raw 5) becomes (5-1)/(9-1) = 0.5 in segment 0, which is below every raw
    # value of segment 1, so it is segment 1's minimum: (0.5 - 0.5) / (8 - 0.5) = 0
    x = np.array([1, 9, 3, 5, 2, 8, 4], np.float32)
    got = po.normalise_segments(x, [], [0, 3, 6])
    f = np.float32
    s0 = [(f(1) - f(1)) / f(8), (f(9) - f(1)) / f(8), (f(3) - f(1)) / f(8)]
    mid = (f(5) - f(1)) / f(8)
    lo, hi = mid, f(8)
    want = np.array(s0 + [(mid - lo) / (hi - lo)] + [(f(v) - lo) / (hi - lo) for v in (2, 8, 4)], np.float32)
    assert np.array_equal(got, want) and got[3] == 0


def test_zeroed_indices_are_clipped_and_the_last_slice_by_n(tmp_path, monkeypatch):
    from mtad_gat_pytorch_b200 import prediction
    monkeypatch.chdir(tmp_path)
    write_metadata(str(tmp_path), "SMAP", [30, 50, 40], [25, 60, 45])
    lookback = 10
    n = 60 + 25 + 45 - lookback                                          # the test scores: sep[-1] == n
    zero, bounds = prediction.channel_bounds("SMAP", False, lookback, n)
    # sorted chan_ids A-1, B-1, C-1: 25, 60, 45 values
    assert bounds.tolist() == [0, 15, 75, 120]
    want = np.unique(np.concatenate([15 + np.arange(-19, 20), 75 + np.arange(-19, 20)]))
    want = want[(want >= 0) & (want < n) & ~np.isin(want, [15, 75])]
    assert zero.tolist() == want.tolist()                                  # 15-19 < 0 clipped, the boundary kept
    x = np.random.default_rng(0).random(n).astype(np.float32) + 1
    with np.errstate(invalid="ignore"):
        got = po.adjust_anomaly_scores(x, "SMAP", False, lookback)
    assert np.array_equal(got, po.normalise_segments(x, zero, bounds))
    assert got[15] != 0 and got[14] == got[16] == 0 and got[75] != 0
    assert got.dtype == np.float32 and np.nanmax(got) <= 1 and np.nanmin(got) == 0
    # the last slice [75, 121) is clipped to n = 120 and normalised over what is there
    assert got[75:].min() == 0 and got[75:].max() == 1
    # another dataset: unchanged, the same object
    assert po.adjust_anomaly_scores(x, "SMD", False, lookback) is x
    assert prediction.channel_bounds("SMD", False, lookback, n) is None


def test_constant_and_nan_segments():
    x = np.array([3, 3, 3, 1, 2, 4, 0, 5, 6], np.float32)
    with np.errstate(invalid="ignore"):
        got = po.normalise_segments(x, [], [0, 2, 5, 8])
    # segment [0..2] is constant 3: 0 / 0 everywhere, so the shared element 2 is NaN and poisons segment [2..5]
    assert np.isnan(got[:6]).all()
    assert np.isnan(got[5:]).all()                                       # ... and through element 5 the next one
    y = np.array([1, 2, 3, np.nan, 5, 6, 7, 8, 9], np.float32)
    with np.errstate(invalid="ignore"):
        got = po.normalise_segments(y, [], [0, 5, 8])
    assert np.isnan(got[:6]).all() and np.isnan(got[5:]).all()
    z = np.array([1, 2, 3, 4, 5, 6, 7, 8, 9], np.float32)
    z[7] = np.nan
    got = po.normalise_segments(z, [], [0, 4, 6])                          # NaN after the last segment: left alone
    assert not np.isnan(got[:7]).any() and np.isnan(got[7]) and got[8] == 9


def test_channel_bounds_filters_sorts_and_drops_p2(tmp_path):
    from mtad_gat_pytorch_b200 import prediction
    names = write_metadata(str(tmp_path), "MSL", [300, 500, 400, 350], [250, 600, 450, 380],
                           other=(("SMAP", "B-2", 77),))
    d = str(tmp_path / "datasets" / "data")
    order = np.argsort(names)
    for is_train, sizes in ((True, [300, 500, 400, 350]), (False, [250, 600, 450, 380])):
        zero, bounds = prediction.channel_bounds("msl", is_train, 100, data_dir=d)
        sep = np.cumsum(np.array(sizes)[order]) - 100
        assert bounds.tolist() == [0] + sep.tolist() and bounds.dtype == np.int64 and zero.dtype == np.int64
        assert np.array_equal(zero, np.unique(np.concatenate([(sep[:-1, None] + np.arange(1, 20)).ravel(),
                                                               (sep[:-1, None] - np.arange(1, 20)).ravel()])))
    assert prediction.channel_bounds("SMD", True, 100, data_dir=d) is None


def test_channel_bounds_raises_on_an_empty_segment(tmp_path):
    from mtad_gat_pytorch_b200 import prediction
    write_metadata(str(tmp_path), "SMAP", [300, 500, 400], [250, 600, 450])
    d = str(tmp_path / "datasets" / "data")
    # sorted by chan_id: 300, 500, 400 values; the last segment starts at 800 - 100
    with pytest.raises(ValueError):
        prediction.channel_bounds("SMAP", True, 100, n=700, data_dir=d)
    prediction.channel_bounds("SMAP", True, 100, n=701, data_dir=d)
    with pytest.raises(ValueError):                                      # a channel shorter than the lookback
        prediction.channel_bounds("SMAP", True, 301, data_dir=d)


# ---------------------------------------------------------------------------------------------------------------------
# against the staged reference

def _import_reference():
    if not os.path.exists(os.path.join(REF_DIR, "prediction.py")):
        pytest.skip("reference not present")
    saved = dict(sys.modules)
    mit = types.ModuleType("more_itertools")
    mit.consecutive_groups = lambda it: iter([])
    stubs = {"more_itertools": mit}
    for name in ("matplotlib", "matplotlib.pyplot", "tqdm", "sklearn", "sklearn.preprocessing"):
        try:
            __import__(name)
        except ImportError:
            stubs[name] = types.ModuleType(name)
    if "tqdm" in stubs:
        stubs["tqdm"].tqdm = lambda x, *a, **k: x
    if "sklearn.preprocessing" in stubs:
        stubs["sklearn.preprocessing"].MinMaxScaler = object
    sys.modules.update(stubs)
    if "matplotlib" in stubs:
        sys.modules["matplotlib"].pyplot = sys.modules["matplotlib.pyplot"]
    sys.path.insert(0, REF_DIR)
    import prediction as ref_prediction
    import utils as ref_utils
    return saved, ref_prediction, ref_utils


def _release_reference(saved):
    sys.path.remove(REF_DIR)
    for name in list(sys.modules):
        if name not in saved:
            sys.modules.pop(name, None)


def test_adjust_restatement_equals_reference(tmp_path, monkeypatch):
    saved, _, ref_utils = _import_reference()
    try:
        monkeypatch.chdir(tmp_path)
        rng = np.random.default_rng(1)
        write_metadata(str(tmp_path), "SMAP", list(rng.integers(120, 900, 54)), list(rng.integers(120, 900, 54)))
        md = pd.read_csv("datasets/data/smap_train_md.csv")
        for is_train in (True, False):
            md = pd.read_csv("datasets/data/smap_train_md.csv" if is_train else "datasets/data/labeled_anomalies.csv")
            total = int(md[(md["chan_id"] != "P-2") & (md.get("spacecraft", "SMAP") == "SMAP")]["num_values"].sum())
            x = rng.random(total - 100).astype(np.float32)
            x[rng.integers(0, x.size, 5)] = 0
            with np.errstate(invalid="ignore"):
                a = po.adjust_anomaly_scores(x, "SMAP", is_train, 100)
                b = ref_utils.adjust_anomaly_scores(x, "SMAP", is_train, 100)
            assert a.dtype == b.dtype and np.array_equal(a, b, equal_nan=True)
    finally:
        _release_reference(saved)


@pytest.mark.parametrize("dataset", ["SMD", "SMAP"])
@pytest.mark.parametrize("labelled", [True, False])
def test_predict_tail_equals_reference_on_saved_scores(tmp_path, monkeypatch, dataset, labelled):
    saved, ref_prediction, _ = _import_reference()
    try:
        monkeypatch.chdir(tmp_path)
        rng = np.random.default_rng(2)
        write_metadata(str(tmp_path), "SMAP", [400, 700, 500], [450, 600, 550])
        lookback, C = 100, 3
        frames = {}
        for key, n in (("train", 1600 - lookback), ("test", 1600 - lookback)):
            a = np.abs(rng.standard_normal((n, C))).astype(np.float32)
            a[700:720] += 3
            cols = {}
            for i in range(C):
                cols[f"A_Score_{i}"] = a[:, i]
            cols["A_Score_Global"] = np.mean(a, 1)
            frames[key] = pd.DataFrame(cols)
        labels = np.zeros(1500, np.float32)
        labels[690:730] = 1
        pred_args = dict(dataset=dataset, target_dims=None, scale_scores=False, q=1e-3, level=0.9, dynamic_pot=False,
                         use_mov_av=False, gamma=1, reg_level=1)
        dirs = {}
        for arm in ("ref", "oracle"):
            dirs[arm] = str(tmp_path / arm)
            os.makedirs(dirs[arm])
            for key in frames:
                frames[key].to_pickle(os.path.join(dirs[arm], f"{key}_output.pkl"))
        lab = labels if labelled else None
        with np.errstate(invalid="ignore", divide="ignore"):
            ref = ref_prediction.Predictor(None, lookback, C, dict(pred_args, save_path=dirs["ref"]))
            ref.predict_anomalies(None, None, lab, load_scores=True)
            po.predict_tail(dict(pred_args, save_path=dirs["oracle"]), lookback, C, lab, load_scores=True)
        import json
        with open(os.path.join(dirs["ref"], "summary.txt")) as f:
            s_ref = json.load(f)
        with open(os.path.join(dirs["oracle"], "summary.txt")) as f:
            s_orc = json.load(f)
        assert s_ref == s_orc
        for key in frames:
            pd.testing.assert_frame_equal(pd.read_pickle(os.path.join(dirs["oracle"], f"{key}_output.pkl")),
                                          pd.read_pickle(os.path.join(dirs["ref"], f"{key}_output.pkl")),
                                          check_exact=True)
    finally:
        _release_reference(saved)
