"""Oracle: the torch_geometric 2.6.1 pieces PNAPlusStack.py imports [3P-memory], and the PNAPlus stack on
``oracle.base.StackOracle``.  Test infrastructure only.

* ``Envelope`` / ``BesselBasisLayer`` (torch_geometric.nn.models.dimenet): rbf_k(d) = env(d / cutoff) sin(freq_k d / cutoff),
  env(x) = (1/x + a x^(p-1) + b x^p + c x^(p+1)) [x < 1], p = exponent + 1, a = -(p+1)(p+2)/2, b = p(p+2), c = -p(p+1)/2;
  ``freq`` is a parameter initialised to pi (1..R).  test_oracle_pnaplus.py pins both by hand-computed values.
* ``PNAPlusConv``: the reference's own PNAConv message / forward (PNAPlusStack.py:233-263) on plain tensors, towers = 1.

tests/golden/make_pnaplus_golden.py plugs the basis into the reference's own PNAPlusStack.py, Base.py and gps.py.
``PNAPlusStackOracle`` is the PNA stack with the Bessel basis of the edge lengths handed to every conv, and the reference's
parameter names, so reference and engine state dicts load into it strictly.
"""
import math

import torch
from torch import nn

from .base import _Conv
from .pna import PNAStackOracle
from .pnaeq import DegreeScalerAggregation as _DSA


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
    def __init__(self, input_dim, hidden_dim, output_dim, output_type, output_heads, pna_deg, edge_dim=None, num_radial=5,
                 radius=5.0, envelope_exponent=5, **kw):
        self.num_radial = num_radial
        super().__init__(input_dim, hidden_dim, output_dim, output_type, output_heads, pna_deg, edge_dim=edge_dim, **kw)
        self.rbf = BesselBasisLayer(num_radial, radius, envelope_exponent)      # registered last, as in PNAPlusStack.__init__

    def _get_conv(self, fin, fout, last, edge_dim=None):
        return _Conv([PNAPlusConv(fin, fout, self.deg, edge_dim, self.num_radial)])

    def _embedding(self, data):
        x, _, ctx = super()._embedding(data)
        ei = data.edge_index
        shifts = data.edge_shifts if getattr(data, "edge_shifts", None) is not None else torch.zeros(ei.shape[1], 3, dtype=x.dtype)
        dist = (data.pos[ei[1]] - data.pos[ei[0]] + shifts).norm(dim=-1)            # get_edge_vectors_and_lengths
        ctx["rbf"] = self.rbf(dist)
        return x, None, ctx

    def _run_conv(self, conv, x, equiv, ctx):
        return conv.module_0(x, ctx["edge_index"], ctx["rbf"], ctx["edge_attr"]), equiv
