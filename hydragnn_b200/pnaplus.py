"""PNAPlus stack on libhgb.so.

Host-side mirror of ``hydragnn/models/PNAPlusStack.py``: its own ``PNAConv`` (PyG 2.6.1 PNAConv with a Bessel-gated message;
towers = pre_layers = post_layers = 1, ``act="relu"``) and PyG 2.6.1 ``BesselBasisLayer`` / ``Envelope``.  Every conv is
followed by a PyG BatchNorm feature layer (``PNAStack._feature_layer``).  Module and parameter names are the reference's
(``graph_convs.<i>.module_0.{aggr_module, pre_nns.0.0, post_nns.0.0, lin, rbf_lin, rbf_emb.0, edge_encoder}``,
``feature_layers.<i>.module``, ``rbf.freq`` last), so reference checkpoints load.

With i = edge_index[1] the target, j the source, rbf_e the Bessel basis of the edge length and u_e = relu(W_r rbf_e + b_r),
the pre_nn Linear is affine in its blocks: h_e = P[i] + Q[j] + M_r u_e + M_a a_e + c, M_r = W_c (or W_c W_enc[:, D:] with an
encoder), M_a = W_c W_enc[:, :D], c = b_pre + W_c b_enc.  The message is m_e = h_e * (W_l rbf_e).  The fused path hands the
per-node [P | Q] and the folded weights to ``ops.PnaPlusConvFn``, which reads the edge lengths only and reduces m_e straight into
[mean | min | max | std]; the degree scalers are folded into the post Linear (``pnaeq.post_linear_scaled``).  Higher-order passes
(MLIP training), edge inputs wider than 16 (GPS) and shapes ``ops.pnaplus_conv_supported`` refuses run the same math composed
from EdgeLenFn, ATen elementwise ops, GatherRows, Linear and DegreeScalerAggregation.
"""
import math

import torch
from torch import nn

from . import ops
from .ops import GatherRows
from .pna import AGGREGATORS, SCALERS, PNAStack
from .pnaeq import DegreeScalerAggregation, post_linear_scaled
from .stacks import SingleConv, run_mlp

# Above this width the fused kernel's per-edge F x F product is not measured to beat the composed path (DESIGN.md, a6d).
FUSED_MAX_F = 64


class Envelope(nn.Module):
    """torch_geometric.nn.models.dimenet.Envelope: (1/x + a x^(p-1) + b x^p + c x^(p+1)) [x < 1], p = exponent + 1."""

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
    """torch_geometric.nn.models.dimenet.BesselBasisLayer: rbf_k(d) = env(d / cutoff) sin(freq_k d / cutoff), with the trainable
    ``freq`` initialised to pi (1..R) without drawing from the generator."""

    def __init__(self, num_radial, cutoff=5.0, envelope_exponent=5):
        super().__init__()
        self.cutoff = cutoff
        self.envelope_exponent = envelope_exponent
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


class PNAConv(nn.Module):
    """PNAPlusStack.py's ``PNAConv(in, out, aggregators, scalers, deg, edge_dim, num_radial, pre_layers=1, post_layers=1,
    divide_input=False)``.  Construction order: pre_nns, post_nns, lin, rbf_lin, rbf_emb, edge_encoder (built whenever edge_dim
    is not None, also for 0); then ``reset_parameters`` draws edge_encoder, pre_nns, post_nns and lin again, not rbf_lin or
    rbf_emb.  pre_nn is always 3 F_in wide."""

    def __init__(self, in_channels, out_channels, aggregators, scalers, deg, edge_dim=None, num_radial=5):
        super().__init__()
        self.in_channels, self.out_channels, self.edge_dim = in_channels, out_channels, edge_dim
        self.towers, self.divide_input = 1, False
        self.F_in, self.F_out = in_channels, out_channels
        self.aggr_module = DegreeScalerAggregation(aggregators, scalers, deg)
        self.pre_nns = nn.ModuleList([nn.Sequential(nn.Linear(3 * in_channels, in_channels))])
        self.post_nns = nn.ModuleList([nn.Sequential(nn.Linear((len(aggregators) * len(scalers) + 1) * in_channels, out_channels))])
        self.lin = nn.Linear(out_channels, out_channels)
        self.rbf_lin = nn.Linear(num_radial, in_channels, bias=False)
        self.rbf_emb = nn.Sequential(nn.Linear(num_radial, in_channels), nn.ReLU())
        if edge_dim is not None:
            self.edge_encoder = nn.Linear(in_channels + edge_dim, in_channels)
        self.reset_parameters()

    def reset_parameters(self):
        if self.edge_dim is not None:
            self.edge_encoder.reset_parameters()
        self.pre_nns[0][0].reset_parameters()
        self.post_nns[0][0].reset_parameters()
        self.lin.reset_parameters()

    def fused_ok(self, x, r, edge_attr):
        d = 0 if edge_attr is None else edge_attr.shape[1]
        return x.is_cuda and self.F_in <= FUSED_MAX_F and ops.pnaplus_conv_supported(self.F_in, r, d)

    def forward(self, x, plan, bessel, edge_attr=None, higher_order=False):
        """``bessel``: the stack's per-forward dict {"basis": BesselBasisLayer, "dist": [E], "rbf": [E, R] or None}; the composed
        path fills "rbf" once and every later layer reuses it."""
        if edge_attr is not None and self.edge_dim is None:
            # the reference's message would call the missing edge_encoder (AttributeError in PNAPlusStack.py:243)
            raise ValueError("PNAPlus conv built without edge_dim cannot take edge attributes")
        fin = self.F_in
        pre = self.pre_nns[0][0]
        w = pre.weight
        wc = w[:, 2 * fin:]
        basis, dist = bessel["basis"], bessel["dist"]
        tgt = plan.by_col                                                # flow source_to_target: aggregate at i = edge_index[1]
        wr, br = self.rbf_emb[0].weight, self.rbf_emb[0].bias
        if not higher_order and self.fused_ok(x, basis.freq.numel(), edge_attr):
            pq = ops.linear_act(x, torch.cat([w[:, :fin], w[:, fin:2 * fin]], dim=0), None)      # [N, 2F] = [x W_a^T | x W_b^T]
            mr, mat, cvec = wc, None, pre.bias
            if edge_attr is not None:
                enc, d = self.edge_encoder, edge_attr.shape[1]
                mr = ops.MatMul.apply(wc, enc.weight[:, d:], False, False)                        # W_c W_enc[:, D:]   [F, F]
                mat = ops.MatMul.apply(enc.weight[:, :d], wc, True, True)                         # (W_c W_enc[:, :D])^T  [D, F]
                cvec = ops.MatMul.apply(enc.bias[None, :], wc, False, True)[0] + pre.bias         # W_c b_enc + b_pre
            agg4 = ops.PnaPlusConvFn.apply(pq, dist, edge_attr, basis.freq, wr, br, self.rbf_lin.weight, mr, mat, cvec,
                                           basis.cutoff, basis.envelope_exponent, plan)
            out = post_linear_scaled(self.post_nns[0][0], x, agg4, self.aggr_module, tgt)
        else:
            lin = ops.linear_any_order if higher_order else ops.linear_act
            if bessel["rbf"] is None:
                bessel["rbf"] = basis(dist)
            rbf = bessel["rbf"]
            et = torch.relu(lin(rbf, wr, br))                                                     # rbf_emb
            if edge_attr is not None:
                et = lin(torch.cat([edge_attr, et], dim=-1), self.edge_encoder.weight, self.edge_encoder.bias)
            h = GatherRows.apply(lin(x, w[:, :fin], None), tgt) + GatherRows.apply(lin(x, w[:, fin:2 * fin], None), plan.by_row)
            h = h + lin(et, wc, pre.bias)
            m = h * lin(rbf, self.rbf_lin.weight, None)
            agg = self.aggr_module(m, tgt)                                                        # [N, 16F]
            out = run_mlp(self.post_nns[0], torch.cat([x, agg], dim=-1), higher_order)
        return (ops.linear_any_order if higher_order else ops.linear_act)(out, self.lin.weight, self.lin.bias)


class PNAPlusStack(PNAStack):
    def __init__(self, deg, edge_dim, envelope_exponent, num_radial, radius, *args, **kwargs):
        self.envelope_exponent, self.num_radial, self.radius = envelope_exponent, num_radial, radius
        super().__init__(deg, edge_dim, *args, **kwargs)
        self.rbf = BesselBasisLayer(self.num_radial, self.radius, self.envelope_exponent)

    def get_conv(self, input_dim, output_dim, last_layer=False, edge_dim=None):
        # the reference's get_conv takes no last_layer; Base._init_conv passes it and it is ignored here
        return SingleConv(PNAConv(input_dim, output_dim, self.aggregators, self.scalers, self.deg, edge_dim=edge_dim,
                                  num_radial=self.num_radial))

    def _forward(self, data, higher):
        if self.use_edge_attr and any(isinstance(m, nn.ModuleList) for h in self.heads_NN for m in h.values()):
            # conv-type node heads are built with edge_dim=None (Base._init_node_conv) but receive edge_attr: the reference
            # fails there, so no kernel is launched here
            raise ValueError("PNAPlus: conv-type node heads cannot run with edge attributes (their convs have no edge_encoder)")
        return super()._forward(data, higher)

    def _embedding(self, data, plan, higher):
        assert data.pos is not None, "PNA+ requires node positions (data.pos) to be set."
        x, eattr = data.x, (data.edge_attr if self.use_edge_attr else None)
        if self.use_edge_attr:
            assert eattr is not None, "Data must have edge attributes if use_edge_attributes is set."
        dist = ops.EdgeLenFn.apply(data.pos, data.edge_shifts, plan)                # get_edge_vectors_and_lengths
        if self.use_global_attn:
            x, eattr = self._gps_embed(data, higher)
        return x, data.pos, {"edge_attr": eattr, "bessel": {"basis": self.rbf, "dist": dist, "rbf": None}}
