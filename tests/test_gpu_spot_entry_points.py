"""Which SPOT-family library entry points a push calls, for SPOT, dSPOT, biSPOT and bidSPOT on thresholding.SpotStream,
SpotStreams, prediction.StreamDetector and FleetDetector: exactly the rule's push entry point (one stream: the
one-stream entry point, or the batched one without device offsets), after any peak-array grows, and nothing else; and
a SpotStream push uploads nothing."""
import numpy as np
import pytest
import torch

from tests.test_gpu_fleet import _model
from tests.test_stream_cpu import gpd

pytestmark = pytest.mark.gpu
K, N = 5, 20
RULES = {"spot": {}, "dspot": {"depth": 8}, "bispot": {"bidirectional": True},
         "bidspot": {"depth": 8, "bidirectional": True}}
GROW = "mtadgat_spot_stream_grow"


def _entry(rule, one):
    """The push entry point of `rule`, and where a one-stream push passes offsets=None (then m)."""
    if rule == "spot":
        return ("mtadgat_spot_stream_push", None) if one else ("mtadgat_spot_stream_push_batched", None)
    return ("mtadgat_dspot_push_batched", 5) if rule == "dspot" else ("mtadgat_bispot_push_batched", 6)


def _spy(monkeypatch):
    """Wraps every SPOT-family entry point of the library; returns the list of (name, args) calls."""
    from mtad_gat_pytorch_b200._lib import SIGNATURES, lib
    calls = []

    def wrap(name, fn):
        def wrapped(*args):
            calls.append((name, args))
            return fn(*args)
        return wrapped
    for name in SIGNATURES:
        if "spot" in name:
            monkeypatch.setattr(lib, name, wrap(name, getattr(lib, name)))
    return calls


def _count_uploads(monkeypatch):
    """Counts host-to-device copies through Tensor.to, Tensor.cuda and Tensor.copy_."""
    uploads = []

    def counting(method):
        real = getattr(torch.Tensor, method)

        def wrapped(self, *a, **kw):
            out = real(self, *a, **kw)
            src = a[0] if method == "copy_" else self
            dst = self if method == "copy_" else out
            if isinstance(src, torch.Tensor) and src.device.type == "cpu" and dst.device.type == "cuda":
                uploads.append(method)
            return out
        return wrapped
    for method in ("to", "cuda", "copy_"):
        monkeypatch.setattr(torch.Tensor, method, counting(method))
    return uploads


def _check(calls, rule, one, m):
    name, off_arg = _entry(rule, one)
    names = [c[0] for c in calls]
    assert names.count(name) == 1 and set(names) <= {name, GROW} and names[-1] == name, names
    args = calls[-1][1]
    if off_arg is not None and one:
        assert args[off_arg] is None and args[off_arg + 1] == m
    return names.count(GROW)


@pytest.mark.parametrize("rule", RULES)
def test_stream_sets(rule, monkeypatch):
    from mtad_gat_pytorch_b200 import thresholding as th
    rng = np.random.default_rng(3)
    inits = [torch.from_numpy(gpd(rng, 300 + 50 * s) - 0.05).float().cuda() for s in range(3)]
    data = [torch.from_numpy(gpd(rng, 400) - 0.05).float().cuda() for _ in range(2)]
    kw = dict(q=1e-3, level=0.9, **RULES[rule])
    one = th.SpotStream(inits[0], **kw)
    many = th.SpotStreams(inits, **kw)
    torch.cuda.synchronize()
    grows = []
    for x in data:                                      # the first push grows the peak arrays, the second need not
        with monkeypatch.context() as mp:
            calls, uploads = _spy(mp), _count_uploads(mp)
            one.push(x)
            assert uploads == []
            grows.append(_check(calls, rule, True, x.numel()))
        with monkeypatch.context() as mp:
            calls = _spy(mp)
            many.push(torch.cat([x] * 3), [0, x.numel(), 2 * x.numel(), 3 * x.numel()])
            grows.append(_check(calls, rule, False, None))
    assert grows[0] >= (2 if "bi" in rule else 1) and grows[1] >= 3 * (2 if "bi" in rule else 1)


@pytest.mark.parametrize("rule", RULES)
def test_detectors(rule, monkeypatch):
    from mtad_gat_pytorch_b200 import prediction
    model = _model(K, N)
    rng = np.random.default_rng(4)
    train = [torch.from_numpy(rng.random((300, K)).astype(np.float32)) for _ in range(2)]
    kw = dict(q=1e-3, level=0.9, **RULES[rule])
    det = prediction.StreamDetector(model, train[0], **kw)
    fleet = prediction.FleetDetector(model, train, **kw)
    for m in (N + 40, 3):
        rows = torch.from_numpy(rng.random((m, K)).astype(np.float32))
        with monkeypatch.context() as mp:
            calls = _spy(mp)
            res = det.push(rows)
            _check(calls, rule, True, res["a_global"].numel())
        with monkeypatch.context() as mp:
            calls = _spy(mp)
            fleet.push(torch.cat([rows, rows]), np.repeat(np.arange(2), m))
            _check(calls, rule, False, None)
