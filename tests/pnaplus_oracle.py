"""CPU restatement of the torch_geometric 2.6.1 pieces PNAPlusStack.py imports [3P-memory], and of the whole PNAPlus stack
without GPS.  Test infrastructure only.

* ``Envelope`` / ``BesselBasisLayer`` (torch_geometric.nn.models.dimenet): rbf_k(d) = env(d / cutoff) sin(freq_k d / cutoff),
  env(x) = (1/x + a x^(p-1) + b x^p + c x^(p+1)) [x < 1], p = exponent + 1, a = -(p+1)(p+2)/2, b = p(p+2), c = -p(p+1)/2;
  ``freq`` is a parameter initialised to pi (1..R).  test_oracle_pnaplus.py pins both by hand-computed values.
* ``MessagePassing``: the part of PyG's base class the reference's PNAConv uses -- ``aggr_module`` registered first,
  ``propagate`` gathering x_i = x[edge_index[1]] (target) and x_j = x[edge_index[0]] and aggregating ``message`` at the targets.
* ``DegreeScalerAggregation``: oracle.pnaeq's restatement, taking PyG's [E, towers, F] messages.

tests/golden/make_pnaplus_golden.py plugs these into the reference's own PNAPlusStack.py, Base.py and gps.py.
``PNAPlusStackOracle`` assembles the stack (graph and ``mlp`` node heads, no GPS) from plain torch with the reference's parameter
names, so reference and engine state dicts load into it strictly.
"""
import math

import torch
from torch import nn

from oracle.pnaeq import DegreeScalerAggregation as _DSA
from pna_oracle import PNAStackOracle


class Envelope(nn.Module):
    def __init__(self, exponent):
        super().__init__()
        self.p = exponent + 1
        self.a = -(self.p + 1) * (self.p + 2) / 2
        self.b = self.p * (self.p + 2)
        self.c = -self.p * (self.p + 1) / 2

    def forward(self, x):
        p, a, b, c = self.p, self.a, self.b, self.c
        x_pow_p0 = x.pow(p - 1)
        x_pow_p1 = x_pow_p0 * x
        x_pow_p2 = x_pow_p1 * x
        return (1.0 / x + a * x_pow_p0 + b * x_pow_p1 + c * x_pow_p2) * (x < 1.0).to(x.dtype)


class BesselBasisLayer(nn.Module):
    def __init__(self, num_radial, cutoff=5.0, envelope_exponent=5):
        super().__init__()
        self.cutoff = cutoff
        self.envelope = Envelope(envelope_exponent)
        self.freq = nn.Parameter(torch.empty(num_radial))
        self.reset_parameters()

    def reset_parameters(self):
        with torch.no_grad():
            torch.arange(1, self.freq.numel() + 1, out=self.freq).mul_(math.pi)
        self.freq.requires_grad_()

    def forward(self, dist):
        dist = dist.unsqueeze(-1) / self.cutoff
        return self.envelope(dist) * (self.freq * dist).sin()


class DegreeScalerAggregation(_DSA):
    def __init__(self, aggr, scaler, deg, train_norm=False):
        assert not train_norm, "PNAConv's default train_norm=False only"
        super().__init__(aggr, scaler, deg)

    def forward(self, x, index=None, dim_size=None, **kw):
        out = super().forward(x.reshape(x.shape[0], -1), index, dim_size)
        return out.view(out.shape[0], 1, -1)


class MessagePassing(nn.Module):
    def __init__(self, aggr=None, node_dim=0, **kw):
        super().__init__()
        self.aggr_module = aggr

    def reset_parameters(self):
        pass

    def propagate(self, edge_index, size=None, x=None, edge_attr=None, rbf=None):
        src, dst = edge_index[0], edge_index[1]
        m = self.message(x[dst], x[src], rbf=rbf, edge_attr=edge_attr)
        return self.aggr_module(m, dst, x.shape[0])


def reset(value):
    """torch_geometric.nn.inits.reset."""
    if hasattr(value, "reset_parameters"):
        value.reset_parameters()
    else:
        for child in value.children() if hasattr(value, "children") else []:
            reset(child)


class PNAPlusConv(nn.Module):
    """The reference's PNAConv message / forward (PNAPlusStack.py:233-263) on plain tensors, towers = 1."""

    def __init__(self, fin, fout, deg, edge_dim, num_radial):
        super().__init__()
        aggr, scal = ["mean", "min", "max", "std"], ["identity", "amplification", "attenuation", "linear"]
        self.aggr_module = _DSA(aggr, scal, deg)
        self.pre_nns = nn.ModuleList([nn.Sequential(nn.Linear(3 * fin, fin))])
        self.post_nns = nn.ModuleList([nn.Sequential(nn.Linear(17 * fin, fout))])
        self.lin = nn.Linear(fout, fout)
        self.rbf_lin = nn.Linear(num_radial, fin, bias=False)
        self.rbf_emb = nn.Sequential(nn.Linear(num_radial, fin), nn.ReLU())
        if edge_dim is not None:
            self.edge_encoder = nn.Linear(fin + edge_dim, fin)

    def forward(self, x, edge_index, rbf, edge_attr=None):
        src, dst = edge_index[0], edge_index[1]
        et = self.rbf_emb(rbf)
        if edge_attr is not None:
            et = self.edge_encoder(torch.cat([edge_attr, et], dim=-1))
        h = self.pre_nns[0](torch.cat([x[dst], x[src], et], dim=-1)) * self.rbf_lin(rbf)
        out = self.aggr_module(h, dst, x.shape[0])
        return self.lin(self.post_nns[0](torch.cat([x, out], dim=-1)))


class PNAPlusStackOracle(PNAStackOracle):
    def __init__(self, input_dim, hidden_dim, output_dim, output_type, output_heads, pna_deg, edge_dim=None, num_conv_layers=2,
                 num_radial=5, radius=5.0, envelope_exponent=5, **kw):
        super().__init__(input_dim, hidden_dim, output_dim, output_type, output_heads, pna_deg, edge_dim=None,
                         num_conv_layers=num_conv_layers, **kw)
        self.use_edge_attr = edge_dim is not None and edge_dim > 0
        deg = torch.Tensor(pna_deg)
        for i, seq in enumerate(self.graph_convs):
            seq.module_0 = PNAPlusConv(input_dim if i == 0 else hidden_dim, hidden_dim, deg, edge_dim, num_radial)
        self.rbf = BesselBasisLayer(num_radial, radius, envelope_exponent)

    def forward(self, data):
        x, ei = data.x, data.edge_index
        ea = data.edge_attr if self.use_edge_attr else None
        shifts = data.edge_shifts if getattr(data, "edge_shifts", None) is not None else torch.zeros(ei.shape[1], 3, dtype=x.dtype)
        dist = (data.pos[ei[1]] - data.pos[ei[0]] + shifts).norm(dim=-1)            # get_edge_vectors_and_lengths
        rbf = self.rbf(dist)
        for conv, bn in zip(self.graph_convs, self.feature_layers):
            x = self.act(bn.module(conv.module_0(x, ei, rbf, ea)))
        from oracle.geometry import graph_pool
        g = int(data.batch.max()) + 1
        xg = graph_pool(x, data.batch, g, self.graph_pooling)
        out = []
        for dim, kind, head in zip(self.head_dims, self.head_type, self.heads_NN):
            if kind == "graph":
                out.append(head["branch-0"](self.graph_shared["branch-0"](xg))[:, :dim])
            else:
                out.append(head["branch-0"](x)[:, :dim])
        return out
