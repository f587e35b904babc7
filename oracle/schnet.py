"""Oracle: SchNet's pieces in plain torch (any dtype, fp64 in the tests), and the SchNet stack on ``oracle.base.StackOracle``.
Test infrastructure only.

torch_geometric 2.6.1 [3P-memory], absent here, written from the published code:
  * ``GaussianSmearing(start, stop, G)``: offset = linspace(start, stop, G), coeff = -0.5 / (offset[1] - offset[0])^2 (a Python
    float), forward exp(coeff (d - offset)^2);
  * ``ShiftedSoftplus``: softplus(x) - log(2), the shift read back from an fp32 tensor.
tests/golden/make_schnet_golden.py plugs these into the reference's own SCFStack.py, so models_schnet.pt pins everything else.

``cfconv`` is CFConv.forward (hydragnn/models/SCFStack.py:267-298) as one function of plain tensors; the GPU tests compare the
fused kernels against it in fp64.

``SCFStackOracle`` states what SCFStack overrides: without edge attributes and GPS every conv builds its own radius graph
(``oracle.radius_graph`` on the positions rounded to fp32, as the reference's fp32 model builds them) inside a Sequential
(interaction_graph, distance_expansion, conv); its feature layers are Identity.
"""
import math

import torch
import torch.nn.functional as F
from torch import nn

from .base import StackOracle, _Conv
from .radius_graph import radius_graph


class GaussianSmearing(nn.Module):
    def __init__(self, start=0.0, stop=5.0, num_gaussians=50):
        super().__init__()
        offset = torch.linspace(start, stop, num_gaussians)
        self.coeff = -0.5 / (offset[1] - offset[0]).item() ** 2
        self.register_buffer("offset", offset)

    def forward(self, dist):
        dist = dist.view(-1, 1) - self.offset.view(1, -1)
        return torch.exp(self.coeff * torch.pow(dist, 2))


class ShiftedSoftplus(nn.Module):
    def __init__(self):
        super().__init__()
        self.shift = torch.log(torch.tensor(2.0)).item()

    def forward(self, x):
        return F.softplus(x) - self.shift


def cfconv(x, pos, edge_index, w_lin1, w1, b1, w2, b2, w_lin2, b_lin2, offset, coeff, cutoff, edge_attr=None):
    """CFConv.forward without the coordinate update: returns (out, W)."""
    row, col = edge_index
    d = (pos[col] - pos[row]).norm(dim=-1)
    c = 0.5 * (torch.cos(d * math.pi / cutoff) + 1.0)
    rbf = torch.exp(coeff * (d.view(-1, 1) - offset.view(1, -1)) ** 2)
    inp = rbf if edge_attr is None else torch.cat([rbf, edge_attr], dim=-1)
    w = (F.linear(F.softplus(F.linear(inp, w1, b1)) - math.log(2.0), w2, b2)) * c.view(-1, 1)
    xl = x @ w_lin1.t()
    agg = torch.zeros_like(xl[:, :1].expand(-1, w.shape[1])).clone().index_add_(0, col, xl[row] * w)
    return agg @ w_lin2.t() + b_lin2, w


def coord_update(pos, edge_index, w, coord_mlp):
    """CFConv.coord_model (SCFStack.py:252-260): pos + mean over the SOURCE index of clamp(coord_diff * coord_mlp(W))."""
    row, col = edge_index
    vec = pos[col] - pos[row]
    coord_diff = vec / (vec.norm(dim=-1, keepdim=True) + 1.0)
    trans = torch.clamp(coord_diff * coord_mlp(w), min=-100, max=100)
    s = torch.zeros_like(pos).index_add_(0, row, trans)
    cnt = torch.bincount(row, minlength=pos.shape[0]).clamp(min=1).to(pos.dtype)
    return pos + s / cnt[:, None]


class _NoState(nn.Module):
    """The stateless ``interaction_graph`` child (``module_0`` of the in-layer Sequential)."""


class CFConv(nn.Module):
    def __init__(self, fin, fout, num_filters, mlp_in, equivariant):
        super().__init__()
        self.lin1 = nn.Linear(fin, num_filters, bias=False)
        self.lin2 = nn.Linear(num_filters, fout)
        self.nn = nn.Sequential(nn.Linear(mlp_in, num_filters), ShiftedSoftplus(), nn.Linear(num_filters, num_filters))
        self.equivariant = equivariant
        if equivariant:
            self.coord_mlp = nn.Sequential(nn.Linear(num_filters, num_filters), nn.ReLU(), nn.Linear(num_filters, 1, bias=False))

    def forward(self, x, pos, edge_index, smearing, cutoff, edge_attr=None):
        out, w = cfconv(x, pos, edge_index, self.lin1.weight, self.nn[0].weight, self.nn[0].bias, self.nn[2].weight, self.nn[2].bias,
                        self.lin2.weight, self.lin2.bias, smearing.offset, smearing.coeff, cutoff, edge_attr)
        if self.equivariant:
            pos = coord_update(pos, edge_index, w, self.coord_mlp)
        return out, pos


class SCFStackOracle(StackOracle):
    def __init__(self, input_dim, hidden_dim, output_dim, output_type, output_heads, num_filters, num_gaussians, radius,
                 max_neighbours=None, edge_dim=None, **kw):
        self.num_filters, self.num_gaussians, self.radius, self.max_neighbours = num_filters, num_gaussians, radius, max_neighbours
        self.edge_dim = edge_dim
        super().__init__(input_dim, hidden_dim, output_dim, output_type, output_heads, **kw)

    def _init_conv(self):
        self.in_layer = not (self.use_edge_attr or self.use_global_attn)     # SCFStack.py:128-161
        self.distance_expansion = GaussianSmearing(0.0, self.radius, self.num_gaussians)
        super()._init_conv()

    def _get_conv(self, fin, fout, last, edge_dim=None):
        conv = CFConv(fin, fout, self.num_filters, self.num_gaussians + (edge_dim or 0), self.equivariance and not last)
        return _Conv([_NoState(), self.distance_expansion, conv] if self.in_layer else [conv])

    def _embedding(self, data):
        x, eattr = self._node_edge_features(data)
        return x, data.pos, {"edge_index": None if self.in_layer else data.edge_index, "edge_attr": eattr, "batch": data.batch}

    def _run_conv(self, conv, x, pos, ctx):
        edge_index = ctx["edge_index"]
        if self.in_layer:
            edge_index = radius_graph(pos.detach().float(), self.radius, ctx["batch"], max_num_neighbors=self.max_neighbours).to(pos.device)
        c = conv.module_2 if self.in_layer else conv.module_0
        # the head convs are built without an edge input (get_conv's edge_dim None) and are handed no edge attributes
        edge_attr = ctx["edge_attr"] if c.nn[0].in_features > self.num_gaussians else None
        return c(x, pos, edge_index, self.distance_expansion, self.radius, edge_attr)
