"""Oracle: torch_geometric 2.6.1 ``SAGEConv`` and ``MFConv`` [3P-memory] in the configurations SAGEStack and MFCStack build
(hydragnn/models/SAGEStack.py, hydragnn/models/MFCStack.py), and both stacks on ``oracle.base.StackOracle``.  Test
infrastructure only.

PyG is absent here, so both convs are written from the published algorithm (flow source_to_target: the target is
i = edge_index[1], the source j = edge_index[0]):
  * ``SAGEConv(in, out)``: aggr "mean", root_weight=True, normalize=False, project=False.  ``lin_l = Linear(in, out)`` with a
    bias and ``lin_r = Linear(in, out, bias=False)``, drawn at construction and again by ``reset_parameters`` (lin_l, then
    lin_r).  out_i = lin_l(mean_j x_j) + lin_r(x_i); a node without in-edges has a mean of 0 (sum / clamp(count, 1)).
  * ``MFConv(in, out, max_degree)``: aggr "add".  ``lins_l`` = max_degree + 1 Linears with a bias, ``lins_r`` = max_degree + 1
    without, drawn at construction and again by ``reset_parameters`` (every lins_l, then every lins_r).  deg_i = min(count of
    i in edge_index[1], max_degree) (duplicates and self-loops count); h_i = sum_j x_j; out_i = lins_l[deg_i](h_i) +
    lins_r[deg_i](x_i).  Every degree's Linears are applied (to an empty selection when no node has that degree), so their
    gradients are zeros, not None.
The draw order of ``reset_parameters`` is restated from memory of the PyG source and cannot be checked against PyG here.
tests/golden/make_sage_mfc_golden.py plugs these classes into the reference's own SAGEStack.py / MFCStack.py + Base.py + gps.py,
so models_sage.pt and models_mfc.pt pin everything except these classes; test_oracle_sage_mfc.py pins them by hand-computed cases.
"""
import torch
from torch import nn

from .base import StackOracle, _Conv
from .gps import PyGBatchNorm


def _aggregate(x, edge_index, mean):
    src, dst = edge_index[0], edge_index[1]
    h = torch.zeros(x.shape[0], x.shape[1], dtype=x.dtype).index_add_(0, dst, x[src])
    if mean:
        cnt = torch.zeros(x.shape[0], dtype=x.dtype).index_add_(0, dst, torch.ones(dst.shape[0], dtype=x.dtype))
        h = h / cnt.clamp(min=1)[:, None]
    return h


class SAGEConv(nn.Module):
    def __init__(self, in_channels, out_channels, **kwargs):
        super().__init__()
        self.in_channels, self.out_channels = in_channels, out_channels
        self.lin_l = nn.Linear(in_channels, out_channels, bias=True)
        self.lin_r = nn.Linear(in_channels, out_channels, bias=False)
        self.reset_parameters()

    def reset_parameters(self):
        self.lin_l.reset_parameters()
        self.lin_r.reset_parameters()

    def forward(self, x, edge_index):
        return self.lin_l(_aggregate(x, edge_index, True)) + self.lin_r(x)


class MFConv(nn.Module):
    def __init__(self, in_channels, out_channels, max_degree=10, bias=True, **kwargs):
        super().__init__()
        self.in_channels, self.out_channels, self.max_degree = in_channels, out_channels, max_degree
        self.lins_l = nn.ModuleList([nn.Linear(in_channels, out_channels, bias=bias) for _ in range(max_degree + 1)])
        self.lins_r = nn.ModuleList([nn.Linear(in_channels, out_channels, bias=False) for _ in range(max_degree + 1)])
        self.reset_parameters()

    def reset_parameters(self):
        for lin in self.lins_l:
            lin.reset_parameters()
        for lin in self.lins_r:
            lin.reset_parameters()

    def forward(self, x, edge_index):
        dst = edge_index[1]
        deg = torch.zeros(x.shape[0], dtype=torch.long).index_add_(0, dst, torch.ones_like(dst)).clamp(max=self.max_degree)
        h = _aggregate(x, edge_index, False)
        out = x.new_zeros(x.shape[0], self.out_channels)
        for i, (lin_l, lin_r) in enumerate(zip(self.lins_l, self.lins_r)):
            idx = (deg == i).nonzero().view(-1)
            r = lin_l(h.index_select(0, idx)) + lin_r(x.index_select(0, idx))
            out = out.index_copy(0, idx, r)
        return out


class _NbrStackOracle(StackOracle):
    """``Base._init_conv`` (a PyG BatchNorm after every conv) and the default ``Base._init_node_conv``; no edge features."""

    def __init__(self, input_dim, hidden_dim, output_dim, output_type, output_heads, **kw):
        self.edge_dim = None
        kw.pop("edge_dim", None)
        super().__init__(input_dim, hidden_dim, output_dim, output_type, output_heads, **kw)
        if self.use_global_attn:
            del self.rel_pos_emb                                      # is_edge_model = False: no edge embedding under GPS

    def _feature_layer(self, width):
        return PyGBatchNorm(width)

    def _embedding(self, data):
        x = data.x
        if self.use_global_attn:                                      # Base._embedding (:477-491), node part only
            x = self.pos_emb(data.pe)
            if self.input_dim:
                x = self.node_lin(torch.cat((self.node_emb(data.x.to(x.dtype)), x), 1))
        return x, None, {"edge_index": data.edge_index}

    def _run_conv(self, conv, x, equiv, ctx):
        return conv.module_0(x, ctx["edge_index"]), equiv


class SAGEStackOracle(_NbrStackOracle):
    def _get_conv(self, fin, fout, last, edge_dim=None):
        return _Conv([SAGEConv(fin, fout)])


class MFCStackOracle(_NbrStackOracle):
    def __init__(self, *args, max_neighbours=None, **kw):
        self.max_degree = max_neighbours
        super().__init__(*args, **kw)

    def _get_conv(self, fin, fout, last, edge_dim=None):
        return _Conv([MFConv(fin, fout, max_degree=self.max_degree)])
