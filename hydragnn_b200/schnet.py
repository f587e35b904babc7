"""SchNet stack on libhgb.so.

Host-side mirror of ``hydragnn/models/SCFStack.py`` with torch_geometric 2.6.1's ``GaussianSmearing``, ``ShiftedSoftplus`` and
``RadiusInteractionGraph``.  Module and parameter names are the reference's, so reference checkpoints load:

* without edge attributes and without GPS, every layer builds its radius graph from the current positions (``SCFStack.py``
  :128-161): ``graph_convs.<i>.module_0`` is the interaction graph, ``module_1`` the shared ``GaussianSmearing`` (its ``offset``
  buffer appears under every layer and as ``distance_expansion.offset``), ``module_2`` the ``CFConv``;
* with ``edge_dim > 0`` or GPS the convolution runs on ``data.edge_index`` with the PBC shifts ignored (:166-193):
  ``graph_convs.<i>.module_0`` is the ``CFConv`` (under GPS: ``graph_convs.<i>.conv.module_0``).

The fused path (first-order passes on CUDA, at most ``FUSED_MAX_FILTERS`` filters, shapes ``ops.cfconv_supported`` takes) runs the whole filter network, the envelope,
the message and the sum in ``ops.CfConvFn``.  The edge block of the filter's first Linear acts on a raw per-edge input r_e of at
most 16 columns through a folded matrix Mt: without GPS r_e is ``edge_attr`` and Mt = W1e^T; under GPS r_e = [edge_attr |
rel_pe] and Mt = (W1e L)^T with L the product of the bias-free edge-embedding Linears, so the [E, hidden] embedding is never
formed.  Higher-order passes (force training) and other shapes compose the same math from GatherRows / SegmentSum / Linear /
EdgeLenFn and ATen elementwise ops.
"""
import math

import torch
import torch.nn.functional as F
from torch import nn

from . import ops, radius
from .ops import GatherRows, SegmentSum
from .stacks import Base, edge_geometry, run_mlp


FUSED_MAX_FILTERS = 64


class GaussianSmearing(nn.Module):
    """torch_geometric.nn.models.schnet.GaussianSmearing."""

    def __init__(self, start=0.0, stop=5.0, num_gaussians=50):
        super().__init__()
        offset = torch.linspace(start, stop, num_gaussians)
        self.coeff = -0.5 / (offset[1] - offset[0]).item() ** 2
        self.register_buffer("offset", offset)

    def forward(self, dist):
        dist = dist.view(-1, 1) - self.offset.view(1, -1)
        return torch.exp(self.coeff * torch.pow(dist, 2))


class ShiftedSoftplus(nn.Module):
    """torch_geometric.nn.models.schnet.ShiftedSoftplus: softplus(x) - log 2 (softplus with PyTorch's threshold 20)."""

    def __init__(self):
        super().__init__()
        self.shift = torch.log(torch.tensor(2.0)).item()

    def forward(self, x):
        return F.softplus(x) - self.shift


class RadiusInteractionGraph(nn.Module):
    """torch_geometric.nn.models.schnet.RadiusInteractionGraph on the engine's radius graph (targets ascending, torch_cluster's
    nearest-first truncation to ``max_num_neighbors`` per target, no self loops).  Returns an ``EdgePlan`` whose by-target view
    needs no sort.  ``cache`` holds the plan of the last positions seen, so layers that do not move the atoms share it."""

    def __init__(self, cutoff, max_num_neighbors):
        super().__init__()
        self.cutoff, self.max_num_neighbors = cutoff, max_num_neighbors

    def forward(self, pos, graph_ptr, num_graphs, cache):
        if cache.get("pos") is pos and cache.get("version") == pos._version:
            return cache["plan"]
        ei, rowptr = radius.radius_graph(pos.detach(), self.cutoff, graph_ptr, num_graphs, False, self.max_num_neighbors)
        plan = ops.EdgePlan(ei, pos.shape[0], col_rowptr=rowptr, graph_ptr=graph_ptr)
        cache.update(pos=pos, version=pos._version, plan=plan)
        return plan


class CFConv(nn.Module):
    """``CFConv`` (SCFStack.py:222-301).  Construction order = the reference's: lin1, lin2, then (equivariant) the coordinate
    MLP's last Linear (xavier, gain 0.001) before its first, then ``reset_parameters`` re-draws lin1 and lin2."""

    def __init__(self, in_channels, out_channels, num_filters, nn_, cutoff, equivariant):
        super().__init__()
        self.lin1 = nn.Linear(in_channels, num_filters, bias=False)
        self.lin2 = nn.Linear(num_filters, out_channels)
        self.nn = nn_
        self.cutoff = cutoff
        self.equivariant = equivariant
        if self.equivariant:
            layer = nn.Linear(num_filters, 1, bias=False)
            torch.nn.init.xavier_uniform_(layer.weight, gain=0.001)
            self.coord_mlp = nn.Sequential(nn.Linear(num_filters, num_filters), nn.ReLU(), layer)
        self.reset_parameters()

    def reset_parameters(self):
        torch.nn.init.xavier_uniform_(self.lin1.weight)
        torch.nn.init.xavier_uniform_(self.lin2.weight)
        self.lin2.bias.data.fill_(0)

    def fused_ok(self, x, g, d):
        # above 64 filters the fused backward (an NF x NF parameter-gradient tile summed in shared memory per 8 edges) is slower
        # than the composed path: ci_schnet (NF 126) 3.2 ms vs 2.1 ms per layer, qm9_schnet (NF 8) 1.2 vs 2.0 ms (DESIGN.md)
        nf = self.lin1.out_features
        return x.is_cuda and nf <= FUSED_MAX_FILTERS and ops.cfconv_supported(g, nf, d)

    def forward(self, x, pos, plan, smearing, edge_raw=None, higher_order=False):
        """``edge_raw`` = (r, L): the edge input of the filter network is r L^T (L None: r itself), or None without one."""
        r, emb = edge_raw if edge_raw is not None else (None, None)
        g = smearing.offset.numel()
        w1 = self.nn[0].weight
        lin = ops.linear_any_order if higher_order else ops.linear_act
        xl = lin(x, self.lin1.weight, None)
        if not higher_order and self.fused_ok(x, g, 0 if r is None else r.shape[1]):
            a1t = w1[:, :g].t()
            if r is not None:
                mt = w1[:, g:].t() if emb is None else ops.MatMul.apply(emb, w1[:, g:], True, True)      # (W1e L)^T  [d, nf]
                a1t = torch.cat([a1t, mt], dim=0)
            agg, w = ops.CfConvFn.apply(xl, pos, r, a1t.contiguous(), self.nn[0].bias, self.nn[2].weight, self.nn[2].bias,
                                        smearing.offset, smearing.coeff, self.cutoff, plan, self.equivariant)
        else:
            dist = ops.EdgeLenFn.apply(pos, None, plan)
            c = 0.5 * (torch.cos(dist * math.pi / self.cutoff) + 1.0)
            inp = smearing(dist)
            if r is not None:
                inp = torch.cat([inp, r if emb is None else lin(r, emb, None)], dim=-1)
            w = run_mlp(self.nn, inp, higher_order) * c.view(-1, 1)
            agg = SegmentSum.apply(GatherRows.apply(xl, plan.by_row) * w, plan.by_col)     # message x_j * W, aggr "add" at i
        if self.equivariant:                                                                 # coord_model (:252-260)
            _, coord_diff = edge_geometry(pos, None, plan, 1.0, higher_order)
            trans = torch.clamp(coord_diff * run_mlp(self.coord_mlp, w, higher_order), min=-100, max=100)
            cnt = (plan.by_row.rowptr[1:] - plan.by_row.rowptr[:-1]).clamp(min=1).to(trans.dtype)
            pos = pos + SegmentSum.apply(trans, plan.by_row) / cnt[:, None]                  # mean over the source index
        return lin(agg, self.lin2.weight, self.lin2.bias), pos


class CFConvEdgeSequential(nn.Module):
    """The PyG ``Sequential`` of get_conv's ``data.edge_index`` branch (SCFStack.py:114-127): the conv is ``module_0``."""

    def __init__(self, conv):
        super().__init__()
        self.module_0 = conv

    def forward(self, inv_node_feat, equiv_node_feat, plan, higher_order=False, smearing=None, edge_raw=None, **kwargs):
        x, _ = self.module_0(inv_node_feat, equiv_node_feat, plan, smearing, edge_raw, higher_order)
        return x, equiv_node_feat


class CFConvGraphSequential(nn.Module):
    """The PyG ``Sequential`` of get_conv's in-layer branches (SCFStack.py:128-161): ``module_0`` builds the radius graph on the
    current positions, ``module_1`` is the shared Gaussian expansion, ``module_2`` the conv."""

    def __init__(self, graph, smearing, conv):
        super().__init__()
        self.module_0, self.module_1, self.module_2 = graph, smearing, conv

    def forward(self, inv_node_feat, equiv_node_feat, plan=None, higher_order=False, graph_ptr=None, num_graphs=None, cache=None,
                **kwargs):
        plan = self.module_0(equiv_node_feat, graph_ptr, num_graphs, cache)
        return self.module_2(inv_node_feat, equiv_node_feat, plan, self.module_1, None, higher_order)


class SCFStack(Base):
    is_edge_model = True

    def __init__(self, num_filters, edge_dim, num_gaussians, radius, *args, max_neighbours=None, **kwargs):
        self.radius, self.max_neighbours = radius, max_neighbours
        self.num_filters, self.edge_dim, self.num_gaussians = num_filters, edge_dim, num_gaussians
        super().__init__(*args, **kwargs)

    @property
    def graph_in_layer(self):
        """True when every layer builds its own radius graph (no edge attributes, no GPS: SCFStack.py:128-161)."""
        return not (self.use_edge_attr or self.use_global_attn)

    def _init_conv(self):
        self.distance_expansion = GaussianSmearing(0.0, self.radius, self.num_gaussians)
        self.interaction_graph = RadiusInteractionGraph(self.radius, self.max_neighbours)
        super()._init_conv()

    def get_conv(self, input_dim, output_dim, last_layer=False, edge_dim=None):
        mlp_edge_dim = self.num_gaussians + edge_dim if edge_dim else self.num_gaussians
        mlp = nn.Sequential(nn.Linear(mlp_edge_dim, self.num_filters), ShiftedSoftplus(), nn.Linear(self.num_filters, self.num_filters))
        conv = CFConv(input_dim, output_dim, self.num_filters, mlp, self.radius, self.equivariance and not last_layer)
        if self.use_edge_attr or self.use_global_attn:
            return CFConvEdgeSequential(conv)
        return CFConvGraphSequential(self.interaction_graph, self.distance_expansion, conv)

    def _edge_plan(self, data):
        return None if self.graph_in_layer else self.plan_for(data)

    def _embedding(self, data, plan, higher):
        if not self.graph_in_layer and self.equivariance:
            raise ValueError("For SchNet if using edge attributes or edge encodings for gps, then E(3)-equivariance cannot be "
                             "ensured. Please disable equivariance or edge attributes.")
        if self.graph_in_layer:
            if self.max_neighbours is None:
                # RadiusInteractionGraph hands max_num_neighbors to radius_graph as given: what None means there is not set
                # by the reference's code, so it is not guessed here
                raise ValueError("SchNet builds its radius graph in every layer and needs max_neighbours (got None)")
            gptr, g = radius._graph_ptr(data, data.pos.shape[0], data.pos.device)
            return data.x, data.pos, {"graph_ptr": gptr, "num_graphs": g, "cache": {}}
        x, edge_raw = self._raw_edge_input(data, higher)          # SCFStack.py:199-214, the edge embedding folded (see module doc)
        return x, data.pos, {"smearing": self.distance_expansion, "edge_raw": edge_raw}

    def __str__(self):
        return "SCFStack"
