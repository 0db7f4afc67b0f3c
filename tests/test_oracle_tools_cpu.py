"""CPU checks of the test-side oracle helpers: the chunked evaluation used at batch 256 equals the one-shot oracle,
and the numpy Adam equals torch.optim.Adam."""
import numpy as np
import torch

from oracle import mtad_gat_oracle as orc
from tests import oracle_tools as ot


def test_chunked_oracle_equals_one_shot():
    kw = dict(n_features=5, window_size=12, out_dim=5, kernel_size=3, gru_hid_dim=8, forecast_n_layers=2,
              forecast_hid_dim=6, recon_hid_dim=7, dropout=0.3)
    cfg = orc.Config(**kw)
    params = orc.make_params(cfg, seed=1, dtype=np.float64)
    rng = np.random.default_rng(0)
    B = 7
    x, y = rng.random((B, cfg.n, cfg.k)), rng.random((B, 1, cfg.k))
    keep = lambda *s: (rng.random(s) >= 0.3) / 0.7
    masks = {"feat": keep(B, cfg.k, cfg.k), "temp": keep(B, cfg.n, cfg.n),
             "mlp": [keep(B, cfg.forecast_hid_dim) for _ in range(cfg.forecast_n_layers)]}
    a = orc.loss_fwd_bwd(x, y, params, cfg, masks=masks)
    b = ot.loss_fwd_bwd_chunked(x, y, params, cfg, masks=masks, chunk=3)
    assert abs(a[0] - b[0]) < 1e-12
    for i in (3, 4, 5):
        assert np.allclose(a[i], b[i], atol=1e-12)
    for k in a[6]:
        assert np.allclose(a[6][k], b[6][k], atol=1e-12), k


def test_numpy_adam_equals_torch_adam():
    rng = np.random.default_rng(1)
    p = {"w": rng.standard_normal((4, 3)), "b": rng.standard_normal(3)}
    tp = {k: torch.nn.Parameter(torch.from_numpy(v.copy())) for k, v in p.items()}
    opt = torch.optim.Adam(tp.values(), lr=1e-3)
    adam = ot.NumpyAdam({k: v.copy() for k, v in p.items()})
    for _ in range(4):
        g = {k: rng.standard_normal(v.shape) for k, v in p.items()}
        for k in tp:
            tp[k].grad = torch.from_numpy(g[k].copy())
        opt.step()
        adam.step(g)
    for k in p:
        assert np.allclose(adam.p[k], tp[k].detach().numpy(), atol=1e-12)


def test_window_tiling_round_trip_and_layout():
    """tile() puts x[b,t,c] at T[b//16][t][c][b%16] (the layout of the recurrence kernels' gi_t / gates_t / dgi_t),
    pads B up to a multiple of 16 with the fill value, and untile() inverts it -- for numpy arrays and torch tensors."""
    rng = np.random.default_rng(2)
    for B, n, C in [(1, 1, 3), (16, 2, 5), (17, 3, 4), (40, 2, 7)]:
        x = rng.standard_normal((B, n, C))
        T = ot.tile(x, fill=7.5)
        assert T.shape == ((B + 15) // 16, n, C, 16)
        for b in (0, B // 2, B - 1):
            for t in range(n):
                assert np.array_equal(T[b // 16, t, :, b % 16], x[b, t])
        pad = T.transpose(0, 3, 1, 2).reshape(-1, n, C)[B:]
        assert pad.size == ((-B) % 16) * n * C and np.all(pad == 7.5)
        assert np.array_equal(ot.untile(T, B), x)
        Tt = ot.tile(torch.from_numpy(x), fill=7.5)
        assert Tt.is_contiguous() and np.array_equal(Tt.numpy(), T)
        assert np.array_equal(ot.untile(Tt, B).numpy(), x)


def test_window_errors_are_per_window():
    ref = np.array([[1.0, -2.0], [1e-6, 0.0], [0.0, 0.0]])
    a = ref + np.array([[1e-3, 0.0], [1e-9, 0.0], [0.0, 0.0]])
    e = ot.window_errors(a, ref)
    assert np.allclose(e, [5e-4, 1e-3, 0.0])
    a[0, 0] = np.nan
    assert not ot.window_errors(a, ref)[0] < 1.0


def test_seed_arithmetic_wraps_like_uint64():
    assert ot.seed_after(5, 0) == 5
    assert ot.seed_after((1 << 64) - 1, 1) == ot.SEED_STEP - 1
