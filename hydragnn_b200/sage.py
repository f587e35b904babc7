"""SAGE and MFC stacks on libhgb.so.

Host-side mirrors of ``hydragnn/models/SAGEStack.py`` with torch_geometric 2.6.1 ``SAGEConv(in, out)`` (aggr "mean",
root_weight, no normalisation, no projection) and ``hydragnn/models/MFCStack.py`` with ``MFConv(in, out, max_degree)`` (aggr
"add"), each on the default ``Base._init_conv`` (hydragnn/models/Base.py:446-463): a PyG ``BatchNorm(hidden_dim)`` after every
conv, GPS-wrapped when global attention is on.  Module and parameter names are the reference's
(``graph_convs.<i>.module_0.{lin_l, lin_r}``, ``...module_0.{lins_l, lins_r}.<d>``, under GPS ``graph_convs.<i>.conv.module_0``),
so reference checkpoints load.

Both layers are out_i = lin_l,g(h_i) + lin_r,g(x_i), h_i aggregated over the in-edges j -> i (i = edge_index[1]).  SAGE takes the
mean and one weight pair; MFC takes the sum and the pair of the node's clamped in-degree g = min(deg_i, max_degree), counting
every entry of edge_index[1].  First-order passes run ``ops.NbrLinearFn``: the neighbour rows are gathered straight into the
A operand of one degree-grouped wgmma Linear.  Higher-order passes and shapes ``ops.nbr_linear_supported`` refuses run
``ops.nbr_linear_composed``.  Neither stack is an edge model: edge attributes never reach the conv.
"""
import torch
from torch import nn

from . import ops
from .gps import PyGBatchNorm
from .stacks import DEGREE_PLAN, Base, SingleConv, cached, remember


def _nbr_layer(x, plan, dp, wl, bl, wr, mean, higher_order):
    if not higher_order and x.is_cuda and ops.nbr_linear_supported(x.shape[1], wl.shape[1], dp.groups):
        if x.shape[0] == 0:
            return x.new_zeros(0, wl.shape[1])
        return ops.NbrLinearFn.apply(x, wl, bl, wr, dp, plan, mean)
    return ops.nbr_linear_composed(x, wl, bl, wr, dp, plan, mean, higher_order)


class SAGEConv(nn.Module):
    """torch_geometric 2.6.1 ``SAGEConv(in, out)``: ``lin_l = Linear(in, out)`` (bias) and ``lin_r = Linear(in, out,
    bias=False)``, drawn at construction and again by ``reset_parameters`` (lin_l, then lin_r)."""

    def __init__(self, in_channels, out_channels):
        super().__init__()
        self.in_channels, self.out_channels = in_channels, out_channels
        self.lin_l = nn.Linear(in_channels, out_channels)
        self.lin_r = nn.Linear(in_channels, out_channels, bias=False)
        self.reset_parameters()

    def reset_parameters(self):
        self.lin_l.reset_parameters()
        self.lin_r.reset_parameters()

    def forward(self, x, plan, degree_plan, higher_order=False):
        return _nbr_layer(x, plan, degree_plan, self.lin_l.weight[None], self.lin_l.bias[None], self.lin_r.weight[None], True,
                          higher_order)


class MFConv(nn.Module):
    """torch_geometric 2.6.1 ``MFConv(in, out, max_degree)``: ``lins_l`` = max_degree + 1 ``Linear(in, out)`` (bias) and
    ``lins_r`` = max_degree + 1 ``Linear(in, out, bias=False)``, drawn at construction and again by ``reset_parameters``
    (every lins_l, then every lins_r).  Every degree's Linears take part in each pass, so degrees no node has get zero
    gradients."""

    def __init__(self, in_channels, out_channels, max_degree=10):
        super().__init__()
        self.in_channels, self.out_channels, self.max_degree = in_channels, out_channels, max_degree
        self.lins_l = nn.ModuleList([nn.Linear(in_channels, out_channels) for _ in range(max_degree + 1)])
        self.lins_r = nn.ModuleList([nn.Linear(in_channels, out_channels, bias=False) for _ in range(max_degree + 1)])
        self.reset_parameters()

    def reset_parameters(self):
        for lin in self.lins_l:
            lin.reset_parameters()
        for lin in self.lins_r:
            lin.reset_parameters()

    def forward(self, x, plan, degree_plan, higher_order=False):
        wl = torch.stack([lin.weight for lin in self.lins_l])
        bl = torch.stack([lin.bias for lin in self.lins_l])
        wr = torch.stack([lin.weight for lin in self.lins_r])
        return _nbr_layer(x, plan, degree_plan, wl, bl, wr, False, higher_order)


class NbrStack(Base):
    """What SAGE and MFC share: no edge input, a BatchNorm after every conv, and the conv arguments of ``_embedding``."""
    is_edge_model = False

    def _feature_layer(self, width):
        return PyGBatchNorm(width)

    def _embedding(self, data, plan, higher):
        """The input features (the GPS node embedding under global attention) and the in-degree grouping of the batch, built
        once per batch and cached on it."""
        x = self._gps_embed(data, higher)[0] if self.use_global_attn else data.x
        hit = cached(data, DEGREE_PLAN)
        if hit is None or hit[0] is not plan or hit[1].groups != self.weight_groups:
            hit = remember(data, DEGREE_PLAN, (plan, ops.degree_plan(plan, self.weight_groups)))
        return x, data.pos, {"degree_plan": hit[1]}


class SAGEStack(NbrStack):
    weight_groups = 1

    def get_conv(self, input_dim, output_dim, last_layer=False, edge_dim=None):
        return SingleConv(SAGEConv(input_dim, output_dim))

    def __str__(self):
        return "SAGEStack"


class MFCStack(NbrStack):
    def __init__(self, max_degree, *args, **kwargs):
        self.max_degree = max_degree
        self.weight_groups = max_degree + 1
        super().__init__(*args, **kwargs)

    def get_conv(self, input_dim, output_dim, last_layer=False, edge_dim=None):
        return SingleConv(MFConv(input_dim, output_dim, max_degree=self.max_degree))

    def __str__(self):
        return "MFCStack"
