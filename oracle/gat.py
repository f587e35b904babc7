"""Oracle: torch_geometric 2.6.1 ``GATv2Conv`` [3P-memory] in the configuration GATStack builds
(hydragnn/models/GATStack.py:175-190: add_self_loops=True, fill_value="mean", bias=True, share_weights=False, residual=False),
and the GAT stack on ``oracle.base.StackOracle``.  Test infrastructure only.

PyG is absent here, so ``GATv2Conv`` is written from the published algorithm:
  * ``lin_l`` / ``lin_r`` = Linear(in, heads c) with bias and ``lin_edge`` = Linear(edge_dim, heads c, bias=False) (only with an
    edge_dim), all PyG Linears with glorot weights and uniform(1 / sqrt(in)) biases; ``att`` [1, heads, c]; ``bias`` [heads c]
    (concat) or [c].  Construction draws the Linears once, ``reset_parameters`` draws lin_l, lin_r, lin_edge again, then
    glorot(att) and zeros(bias);
  * ``forward``: x_l = lin_l(x), x_r = lin_r(x) as [N, heads, c]; remove_self_loops, then add_self_loops with
    fill_value="mean" (the loop attribute of node i is the mean of its remaining in-edges' attributes, index edge_index[1], 0
    without any; the loops are appended after the edges);
  * ``edge_update``: z = x_r[i] + x_l[j] (+ lin_edge(a) when edge_attr is given: an AssertionError without lin_edge),
    s = (leaky_relu(z) * att).sum(-1), alpha = softmax(s, i) with the max detached and 1e-16 added to the denominator, then
    dropout on alpha;
  * out[i] = sum alpha x_l[j], viewed [N, heads c] (concat) or averaged over the heads, + bias.
tests/golden/make_gat_golden.py plugs this class into the reference's own GATStack.py + Base.py + gps.py, so models_gat.pt pins
everything except this class; test_oracle_gat.py pins this class by hand-computed cases.

``GATStackOracle`` states what GATStack overrides: ``_init_conv`` (concat convs with head-multiplied widths, BatchNorm(hidden
heads) after them and BatchNorm(hidden) after the head-averaging last one), the ``out_lin`` after the concat convs under GPS, and
the head-multiplied widths of its conv-type node heads, whose convs have no edge input.  Its convs run without attention
dropout.
"""
import math

import torch
import torch.nn.functional as F
from torch import nn

from .base import StackOracle, _Conv
from .gps import PyGBatchNorm


def _glorot(w):
    a = math.sqrt(6.0 / (w.size(-2) + w.size(-1)))
    with torch.no_grad():
        w.uniform_(-a, a)


def _reset_linear(lin):
    _glorot(lin.weight)
    if lin.bias is not None:
        b = 1.0 / math.sqrt(lin.in_features)
        with torch.no_grad():
            lin.bias.uniform_(-b, b)


class GATv2Conv(nn.Module):
    def __init__(self, in_channels, out_channels, heads=1, concat=True, negative_slope=0.2, dropout=0.0, add_self_loops=True,
                 edge_dim=None, fill_value="mean", bias=True, share_weights=False, residual=False, **kwargs):
        assert add_self_loops and fill_value == "mean" and bias and not share_weights and not residual, "GATStack's configuration"
        super().__init__()
        self.in_channels, self.out_channels, self.heads, self.concat = in_channels, out_channels, heads, concat
        self.negative_slope, self.dropout, self.edge_dim = negative_slope, dropout, edge_dim
        self.lin_l = nn.Linear(in_channels, heads * out_channels)
        self.lin_r = nn.Linear(in_channels, heads * out_channels)
        self.att = nn.Parameter(torch.empty(1, heads, out_channels))
        self.lin_edge = nn.Linear(edge_dim, heads * out_channels, bias=False) if edge_dim is not None else None
        self.bias = nn.Parameter(torch.empty(heads * out_channels if concat else out_channels))
        self.reset_parameters()

    def reset_parameters(self):
        _reset_linear(self.lin_l)
        _reset_linear(self.lin_r)
        if self.lin_edge is not None:
            _reset_linear(self.lin_edge)
        _glorot(self.att)
        with torch.no_grad():
            self.bias.zero_()

    def forward(self, x, edge_index, edge_attr=None):
        H, C, N = self.heads, self.out_channels, x.shape[0]
        xl = self.lin_l(x).view(N, H, C)
        xr = self.lin_r(x).view(N, H, C)
        keep = edge_index[0] != edge_index[1]                                        # remove_self_loops
        src, dst = edge_index[0][keep], edge_index[1][keep]
        loops = torch.arange(N, dtype=src.dtype)
        if edge_attr is not None:
            if edge_attr.dim() == 1:
                edge_attr = edge_attr.view(-1, 1)
            ea = edge_attr[keep]
            cnt = torch.zeros(N, dtype=ea.dtype).index_add_(0, dst, torch.ones_like(dst, dtype=ea.dtype)).clamp(min=1)
            fill = torch.zeros(N, ea.shape[1], dtype=ea.dtype).index_add_(0, dst, ea) / cnt[:, None]
            ea = torch.cat([ea, fill], 0)
        src, dst = torch.cat([src, loops]), torch.cat([dst, loops])
        z = xr[dst] + xl[src]
        if edge_attr is not None:
            assert self.lin_edge is not None
            z = z + self.lin_edge(ea).view(-1, H, C)
        s = (F.leaky_relu(z, self.negative_slope) * self.att).sum(-1)                # [E', H]
        smax = torch.full((N, H), float("-inf"), dtype=s.dtype).scatter_reduce(0, dst[:, None].expand_as(s), s.detach(), "amax")
        ex = (s - smax[dst]).exp()
        den = torch.zeros(N, H, dtype=s.dtype).index_add_(0, dst, ex) + 1e-16
        alpha = ex / den[dst]
        alpha = F.dropout(alpha, p=self.dropout, training=self.training)
        out = torch.zeros(N, H, C, dtype=xl.dtype).index_add_(0, dst, alpha[:, :, None] * xl[src])
        out = out.reshape(N, H * C) if self.concat else out.mean(dim=1)
        return out + self.bias


class GATStackOracle(StackOracle):
    def __init__(self, input_dim, hidden_dim, output_dim, output_type, output_heads, edge_dim=None, heads=6, negative_slope=0.05,
                 **kw):
        self.heads, self.negative_slope, self.edge_dim = heads, negative_slope, edge_dim
        super().__init__(input_dim, hidden_dim, output_dim, output_type, output_heads, **kw)

    def _get_conv(self, fin, fout, last, edge_dim=None):
        """GATStack.get_conv: the conv is ``module_0``, out_lin ``module_1``; every conv but a last one concatenates its heads."""
        concat = not last
        out_lin = nn.Linear(self.hidden_dim * self.heads, self.hidden_dim) if (self.use_global_attn and concat) else nn.Identity()
        return _Conv([GATv2Conv(fin, fout, heads=self.heads, concat=concat, negative_slope=self.negative_slope, edge_dim=edge_dim),
                      out_lin])

    def _conv_width(self, fout, last):
        return fout if last else fout * self.heads

    def _init_conv(self):
        """GATStack._init_conv (:39-111): a first and a last conv whatever num_conv_layers is; under GPS out_lin brings the
        concat convs back to hidden_dim."""
        h, gps = self.hidden_dim, self.use_global_attn
        mid_in = h if gps else self._conv_width(h, False)
        for fin, last in [(self.embed_dim, False)] + [(mid_in, False)] * (self.num_conv_layers - 2) + [(mid_in, True)]:
            self.graph_convs.append(self._wrap(self._get_conv(fin, h, last, edge_dim=self.edge_embed_dim)))
            self.feature_layers.append(PyGBatchNorm(h if gps else self._conv_width(h, last)))

    def _run_conv(self, conv, x, equiv, ctx):
        return conv.module_1(conv.module_0(x, ctx["edge_index"], ctx["edge_attr"])), equiv
