"""Host-side mirror of the reference's `modules.py` classes for the H100 hot path.

Device dispatch: CUDA tensors run the sm_90a kernels (functional.py); host tensors run the library's own CPU backend
(cpu_backend.py -> `mtadgat_cpu_*`), as the reference's callers expect (training.py:60).  Never one for the other.

Same class names, constructor signatures, parameter names/shapes (hence the same state-dict and, because the
parameter containers are constructed in the same order with the same torch initialisers, the same values
under the same torch seed) and forward signatures as the reference.  The `nn.Conv1d`,
`nn.Linear` and `nn.GRU` members are used ONLY as parameter containers -- their forwards are never called;
every forward/backward runs in libmtadgat.so through `functional.py`.  CUDA only: CPU tensors raise.
"""
import torch
import torch.nn as nn

from . import functional as F
from . import cpu_backend as C


class _SeedMixin:
    """Dropout seed plumbing: MTAD_GAT hands one per-step seed to its children; a layer used on its own
    draws a fresh one per call."""
    _step_seed = None

    def _seed(self, device, p):
        if not (self.training and p > 0.0):
            return None
        return self._step_seed if self._step_seed is not None else F.fresh_seed(device)


class ConvLayer(nn.Module):
    """1-D convolution over time + ReLU (reference modules.py:5-22).  (B,n,k) -> (B,n,k)."""

    def __init__(self, n_features, kernel_size=7):
        super().__init__()
        if kernel_size % 2 == 0:
            raise ValueError("kernel_size must be odd: an even size changes the window length in the reference")
        self.conv = nn.Conv1d(in_channels=n_features, out_channels=n_features, kernel_size=kernel_size)

    def forward(self, x):
        if not x.is_cuda:
            return C.ConvReluFn.apply(x, self.conv.weight, self.conv.bias)
        return F.ConvReluFn.apply(x, self.conv.weight, self.conv.bias)

    def forward_fanout(self, x, fanout):
        """The same output `fanout` times (aliases), one per consumer: their gradients are summed inside the
        backward kernels (used by MTAD_GAT.forward, whose conv output feeds both GAT layers and the GRU)."""
        return F.ConvReluFn.apply(x, self.conv.weight, self.conv.bias, fanout)


class _GraphAttention(nn.Module, _SeedMixin):
    """Shared body of the feature- and time-oriented GAT layers (reference modules.py:25-217)."""
    _feature = None

    def __init__(self, n_features, window_size, dropout, alpha, embed_dim=None, use_gatv2=True, use_bias=True):
        super().__init__()
        self.n_features = n_features
        self.window_size = window_size
        self.dropout = dropout
        self.alpha = alpha
        self.use_gatv2 = use_gatv2
        self.use_bias = use_bias
        node_dim = window_size if self._feature else n_features     # length of one node's vector
        self.num_nodes = n_features if self._feature else window_size
        self.embed_dim = embed_dim if embed_dim is not None else node_dim
        if use_gatv2:                       # linear map applied to the concatenated pair (modules.py:46-49)
            self.embed_dim *= 2
            lin_in, a_in = 2 * node_dim, self.embed_dim
        else:
            lin_in, a_in = node_dim, 2 * self.embed_dim
        self.lin = nn.Linear(lin_in, self.embed_dim)
        self.a = nn.Parameter(torch.empty((a_in, 1)))
        nn.init.xavier_uniform_(self.a.data, gain=1.414)
        if use_bias:
            self.bias = nn.Parameter(torch.zeros(self.num_nodes, self.num_nodes))

    def forward(self, x):
        p = self.dropout if self.training else 0.0
        if not x.is_cuda:
            return C.GatFn.apply(x, self.lin.weight, self.lin.bias, self.a, self.bias if self.use_bias else None,
                                 self._feature, self.use_gatv2, self.alpha, p, self._seed(x.device, p))
        return F.GatFn.apply(x, self.lin.weight, self.lin.bias, self.a, self.bias if self.use_bias else None,
                             self._feature, self.use_gatv2, self.alpha, p, self._seed(x.device, p))


class FeatureAttentionLayer(_GraphAttention):
    """Nodes = the k features, node vector = its n values (reference modules.py:25-122)."""
    _feature = True


class TemporalAttentionLayer(_GraphAttention):
    """Nodes = the n timestamps, node vector = its k feature values (reference modules.py:125-217)."""
    _feature = False


def _gru_stack(rnn, layer0, n_layers, p_between, training, seed_fn, rng_base):
    """Layers 1.. of an nn.GRU parameter container on top of `layer0`'s per-step outputs.  `rng_base` is the Philox
    stream id of the inter-layer dropout: the encoder and the decoder receive the same per-step seed, so they need
    distinct stream ids to draw independent masks (as the reference's two nn.GRU modules do)."""
    out, h_last = layer0
    for l in range(1, n_layers):
        if training and p_between > 0.0:     # nn.GRU inter-layer dropout (modules.py:231-233)
            m = F.dropout_multipliers(out.numel(), p_between, seed_fn(), rng_base + l).view_as(out)
            out = out * m
        out, h_last = F.GruFn.apply(out, None, None, getattr(rnn, f"weight_ih_l{l}"), getattr(rnn, f"weight_hh_l{l}"),
                                    getattr(rnn, f"bias_ih_l{l}"), getattr(rnn, f"bias_hh_l{l}"), True)
    return out, h_last


class GRULayer(nn.Module, _SeedMixin):
    """Encoder GRU (reference modules.py:220-238)."""

    def __init__(self, in_dim, hid_dim, n_layers, dropout):
        super().__init__()
        self.hid_dim = hid_dim
        self.n_layers = n_layers
        self.dropout = 0.0 if n_layers == 1 else dropout
        self.gru = nn.GRU(in_dim, hid_dim, num_layers=n_layers, batch_first=True, dropout=self.dropout)

    def _run(self, slices, need_out):
        g = self.gru
        if not slices[0].is_cuda:
            x = slices[0] if len(slices) == 1 else torch.cat(list(slices), dim=2)      # mtad_gat.py:71
            out = C.gru_layers(g, x, self.n_layers, self.dropout, self.training,
                               lambda: self._step_seed if self._step_seed is not None else F.fresh_seed(x.device), F.RNG_GRU0)
            return out, out[:, -1, :]
        xs = list(slices) + [None] * (3 - len(slices))
        multi = self.n_layers > 1
        layer0 = F.GruFn.apply(xs[0], xs[1], xs[2], g.weight_ih_l0, g.weight_hh_l0, g.bias_ih_l0, g.bias_hh_l0,
                               need_out or multi)
        if multi:
            dev = xs[0].device
            return _gru_stack(g, layer0, self.n_layers, self.dropout, self.training,
                              lambda: self._step_seed if self._step_seed is not None else F.fresh_seed(dev), F.RNG_GRU0)
        return layer0

    def forward_slices(self, slices):
        """h_n[-1] (B,H) of the GRU run over torch.cat(slices, dim=2) without materialising the cat
        (what MTAD_GAT.forward consumes, mtad_gat.py:71-74)."""
        return self._run(slices, need_out=False)[1]

    def forward(self, x):
        out, h = self._run([x], need_out=True)
        return out[-1, :, :], h               # the reference returns out[-1]: the last *batch element* (modules.py:237)


class RNNDecoder(nn.Module, _SeedMixin):
    """Decoder GRU (reference modules.py:241-257): all n outputs."""

    def __init__(self, in_dim, hid_dim, n_layers, dropout):
        super().__init__()
        self.in_dim = in_dim
        self.n_layers = n_layers
        self.dropout = 0.0 if n_layers == 1 else dropout
        self.rnn = nn.GRU(in_dim, hid_dim, n_layers, batch_first=True, dropout=self.dropout)

    def _finish(self, out, dev):
        if self.n_layers == 1:
            return out
        return _gru_stack(self.rnn, (out, None), self.n_layers, self.dropout, self.training,
                          lambda: self._step_seed if self._step_seed is not None else F.fresh_seed(dev), F.RNG_DEC0)[0]

    def forward_repeat(self, h_end, window_size):
        """Decoder over the reference's scrambled repeat of h_end (modules.py:279) without building it."""
        r = self.rnn
        if not h_end.is_cuda:
            rep = h_end.repeat_interleave(int(window_size), dim=1).view(h_end.size(0), int(window_size), -1)   # modules.py:279
            return self.forward(rep)
        out = F.GruRepFn.apply(h_end, r.weight_ih_l0, r.weight_hh_l0, r.bias_ih_l0, r.bias_hh_l0, int(window_size))
        return self._finish(out, h_end.device)

    def forward(self, x):
        r = self.rnn
        if not x.is_cuda:
            return C.gru_layers(r, x, self.n_layers, self.dropout, self.training,
                                lambda: self._step_seed if self._step_seed is not None else F.fresh_seed(x.device), F.RNG_DEC0)
        out, _ = F.GruFn.apply(x, None, None, r.weight_ih_l0, r.weight_hh_l0, r.bias_ih_l0, r.bias_hh_l0, True)
        return self._finish(out, x.device)


class ReconstructionModel(nn.Module):
    """GRU decoder + Linear (reference modules.py:260-283)."""

    def __init__(self, window_size, in_dim, hid_dim, out_dim, n_layers, dropout):
        super().__init__()
        self.window_size = window_size
        self.decoder = RNNDecoder(in_dim, hid_dim, n_layers, dropout)
        self.fc = nn.Linear(hid_dim, out_dim)

    def forward(self, x):
        dec = self.decoder.forward_repeat(x, self.window_size)
        if not x.is_cuda:
            return C.LinearFn.apply(dec, self.fc.weight, self.fc.bias, 0, 0.0, None, 0)
        return F.LinearFn.apply(dec, self.fc.weight, self.fc.bias, 0, 0.0, None, 0)


class Forecasting_Model(nn.Module, _SeedMixin):
    """n_layers+1 Linear layers, ReLU+Dropout after all but the last (reference modules.py:286-311)."""

    def __init__(self, in_dim, hid_dim, out_dim, n_layers, dropout):
        super().__init__()
        layers = [nn.Linear(in_dim, hid_dim)]
        for _ in range(n_layers - 1):
            layers.append(nn.Linear(hid_dim, hid_dim))
        layers.append(nn.Linear(hid_dim, out_dim))
        self.layers = nn.ModuleList(layers)
        self.dropout = nn.Dropout(dropout)

    def forward(self, x):
        p = self.dropout.p if self.training else 0.0
        seed = self._seed(x.device, p)
        rec = getattr(self, "_gate_record", None)       # tests: a list collects (activation > 0) per hidden layer
        Lin = F.LinearFn if x.is_cuda else C.LinearFn
        for i in range(len(self.layers) - 1):
            x = Lin.apply(x, self.layers[i].weight, self.layers[i].bias, 1, p, seed, F.RNG_MLP0 + i)
            if rec is not None:
                rec.append(x.detach() > 0)
        return Lin.apply(x, self.layers[-1].weight, self.layers[-1].bias, 0, 0.0, None, 0)
