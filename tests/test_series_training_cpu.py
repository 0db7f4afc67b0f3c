"""CPU tests of the series-training host side: `loader_batches` reproduces a reference DataLoader's batches and its
use of the global RNG, and `index_table` rejects bad index batches before anything reaches the device."""
import numpy as np
import pytest
import torch
from torch.utils.data import DataLoader

from tests import reference_loop as ref


@pytest.fixture(scope="module")
def mgt():
    import __graft_entry__ as ge
    ge.build()
    from mtad_gat_pytorch_b200 import training
    return training


def _series(N=431, k=5):
    return torch.from_numpy(np.random.default_rng(3).random((N, k)).astype(np.float32))


def _gather(series, idx, n):
    idx = idx.tolist()
    return (torch.stack([series[i:i + n] for i in idx]), torch.stack([series[i + n:i + n + 1] for i in idx]))


def _check_same_batches(mgt, make_loaders, series, n, epochs=3):
    """Iterating the loaders and iterating loader_batches from the same global RNG state yield the same windows and
    leave the same RNG state."""
    loaders = make_loaders()
    torch.manual_seed(11)
    real = [[(x.clone(), y.clone()) for x, y in ld] for _ in range(epochs) for ld in loaders]
    state_real = torch.get_rng_state()
    torch.manual_seed(11)
    mine = [list(mgt.loader_batches(ld)) for _ in range(epochs) for ld in loaders]
    assert torch.equal(torch.get_rng_state(), state_real)
    assert len(real) == len(mine) == epochs * len(loaders)
    for r_ep, m_ep in zip(real, mine):
        assert len(r_ep) == len(m_ep)
        for (x, y), idx in zip(r_ep, m_ep):
            assert idx.dtype == torch.int64 and idx.ndim == 1
            gx, gy = _gather(series, idx, n)
            assert torch.equal(gx, x) and torch.equal(gy, y)
    return mine


def test_loader_batches_shuffle(mgt):
    series, n = _series(), 20
    ds = ref.SlidingWindowDataset(series, n)
    batches = _check_same_batches(mgt, lambda: [DataLoader(ds, batch_size=64, shuffle=True)], series, n)
    assert [len(b) for b in batches[0]] == [64] * 6 + [27]
    assert sorted(torch.cat(batches[0]).tolist()) == list(range(len(ds)))
    assert not torch.equal(torch.cat(batches[0]), torch.cat(batches[1]))        # reshuffled every epoch


def test_loader_batches_create_data_loaders_split(mgt):
    series, n = _series(), 20
    ds = ref.SlidingWindowDataset(series, n)
    np.random.seed(5)
    train_loader, val_loader = ref.create_data_loaders(ds, 64, 0.1, True)
    batches = _check_same_batches(mgt, lambda: [train_loader, val_loader], series, n)
    assert [len(b) for b in batches[0]] == [64] * 5 + [50] and [len(b) for b in batches[1]] == [41]
    tr, va = set(torch.cat(batches[0]).tolist()), set(torch.cat(batches[1]).tolist())
    assert not tr & va and len(tr | va) == len(ds)


def test_index_table_layout(mgt):
    table, counts = mgt.index_table([np.arange(4), torch.tensor([7, 0, 9, 3]), [9, 1]], 4, 10)
    assert counts == [4, 4, 2] and table.dtype == np.int64
    assert table.tolist() == [[0, 1, 2, 3], [7, 0, 9, 3], [9, 1, 0, 0]]


@pytest.mark.parametrize("batches,message", [
    ([np.arange(4), np.array([1, 10])], "batch 1: window index 10 outside"),
    ([np.arange(4), np.array([-1, 2])], "batch 1: window index -1 outside"),
    ([np.arange(3), np.arange(4)], "batch 0 of 2: 3 indices"),
    ([np.arange(4), np.arange(5)], "batch 1 of 2: 5 indices"),
    ([np.arange(4), np.array([], dtype=np.int64)], "batch 1 of 2: 0 indices"),
    ([np.arange(4), np.array([1.0, 2.0])], "batch 1: a 1-D integer index array expected"),
    ([np.array([True, False, True, True])], "batch 0: a 1-D integer index array expected"),
    ([np.arange(4).reshape(2, 2)], "batch 0: a 1-D integer index array expected"),
    ([], "no batches"),
])
def test_index_table_rejects(mgt, batches, message):
    with pytest.raises(ValueError, match=message):
        mgt.index_table(batches, 4, 10)


def test_host_series_is_refused(mgt):
    import mtad_gat_pytorch_b200 as mg
    m = mg.MTAD_GAT(5, 12, 5)
    with pytest.raises(ValueError, match="reference's Trainer"):
        mgt.SeriesTrainer(m, torch.optim.Adam(m.parameters()), torch.rand(40, 5))
