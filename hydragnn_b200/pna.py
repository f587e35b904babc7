"""PNA stack on libhgb.so.

Host-side mirror of ``hydragnn/models/PNAStack.py`` with torch_geometric 2.6.1 ``PNAConv`` (towers = 1, pre_layers =
post_layers = 1, divide_input = False) and the default ``Base._init_conv`` (hydragnn/models/Base.py:446-463): every conv
is followed by a PyG ``BatchNorm(hidden_dim)`` feature layer.  Module and parameter names are the reference's
(``graph_convs.<i>.module_0.{aggr_module, edge_encoder, pre_nns.0.0, post_nns.0.0, lin}``, ``feature_layers.<i>.module``),
so reference checkpoints load.

PNAConv's message is affine in its inputs (pre_layers = 1): with i = edge_index[1] the target and j = edge_index[0] the
source, h_e = W_a x_i + W_b x_j + W_c edge_encoder(a_e) + b.  The fused path multiplies [W_a; W_b] per NODE and hands
the per-node products to ``hgb_pna_conv_fwd``, which forms h_e in registers and reduces it straight into
[mean | min | max | std]; the degree scalers are folded into the post Linear (``pnaeq.post_linear_scaled``).  Neither the
[E, 3F] concatenation nor the [E, F] message is ever written.  Higher-order passes and edge attributes wider than 16 run
the same math composed from the closed primitives (GatherRows / Linear / DegreeScalerAggregation).
"""
import torch
from torch import nn

from . import ops
from .gps import PyGBatchNorm
from .ops import GatherRows
from .pnaeq import DegreeScalerAggregation, post_linear_scaled
from .stacks import Base, SingleConv, run_mlp

AGGREGATORS = ["mean", "min", "max", "std"]
SCALERS = ["identity", "amplification", "attenuation", "linear"]          # PNAStack.py:30-36: no inverse_linear


class PNAConv(nn.Module):
    """torch_geometric 2.6.1 ``PNAConv(in, out, aggregators, scalers, deg, edge_dim, towers=1, pre_layers=1, post_layers=1,
    divide_input=False)``.  Construction draws every Linear once and ``reset_parameters`` draws them again in the order
    edge_encoder, pre_nns, post_nns, lin, as PyG does: the second draw fixes the seeded values of every later module."""

    def __init__(self, in_channels, out_channels, aggregators, scalers, deg, edge_dim=None):
        super().__init__()
        self.in_channels, self.out_channels, self.edge_dim = in_channels, out_channels, edge_dim
        self.towers, self.divide_input = 1, False
        self.F_in, self.F_out = in_channels, out_channels
        self.aggr_module = DegreeScalerAggregation(aggregators, scalers, deg)
        if edge_dim is not None:
            self.edge_encoder = nn.Linear(edge_dim, in_channels)
        self.pre_nns = nn.ModuleList([nn.Sequential(nn.Linear((3 if edge_dim else 2) * in_channels, in_channels))])
        self.post_nns = nn.ModuleList([nn.Sequential(nn.Linear((len(aggregators) * len(scalers) + 1) * in_channels, out_channels))])
        self.lin = nn.Linear(out_channels, out_channels)
        self.reset_parameters()

    def reset_parameters(self):
        if self.edge_dim is not None:
            self.edge_encoder.reset_parameters()
        self.pre_nns[0][0].reset_parameters()
        self.post_nns[0][0].reset_parameters()
        self.lin.reset_parameters()

    def fused_ok(self, x, edge_attr):
        return x.is_cuda and (edge_attr is None or edge_attr.shape[1] <= ops.PNA_CONV_MAX_EDGE_DIM)

    def forward(self, x, plan, edge_attr=None, higher_order=False):
        fin = self.F_in
        pre = self.pre_nns[0][0]
        w = pre.weight
        if self.edge_dim and edge_attr is None:
            # PyG would hand the 2F-wide [x_i | x_j] to the 3F-wide pre_nn and fail; dropping the W_c columns would run another model
            raise ValueError("PNAConv was built with edge_dim=%d but called without edge_attr" % self.edge_dim)
        ea = edge_attr if self.edge_dim is not None else None       # PNAConv.message reads edge_attr only with an encoder
        tgt = plan.by_col                                          # flow source_to_target: aggregate at i = edge_index[1]
        if not higher_order and self.fused_ok(x, ea):
            pq = ops.linear_act(x, torch.cat([w[:, :fin], w[:, fin:2 * fin]], dim=0), None)      # [N, 2F] = [x W_a^T | x W_b^T]
            mt = None
            cvec = pre.bias
            if ea is not None:
                enc, wc = self.edge_encoder, w[:, 2 * fin:]
                mt = ops.MatMul.apply(enc.weight, wc, True, True)                           # (W_c W_enc)^T  [d, F]
                cvec = ops.MatMul.apply(enc.bias[None, :], wc, False, True)[0] + pre.bias      # W_c b_enc + b_pre
            agg4 = ops.PnaConvFn.apply(pq, ea, mt, cvec, plan)                            # [N, 4F]
            out = post_linear_scaled(self.post_nns[0][0], x, agg4, self.aggr_module, tgt)
        else:
            lin = ops.linear_any_order if higher_order else ops.linear_act
            h = GatherRows.apply(lin(x, w[:, :fin], None), tgt) + GatherRows.apply(lin(x, w[:, fin:2 * fin], None), plan.by_row)
            if ea is not None:
                enc = self.edge_encoder
                h = h + lin(lin(ea, enc.weight, enc.bias), w[:, 2 * fin:], None)
            h = h + pre.bias
            agg = self.aggr_module(h, tgt)                                                 # [N, 16F]
            out = run_mlp(self.post_nns[0], torch.cat([x, agg], dim=-1), higher_order)
        return (ops.linear_any_order if higher_order else ops.linear_act)(out, self.lin.weight, self.lin.bias)


class PNAStack(Base):
    is_edge_model = True

    def __init__(self, deg, edge_dim, *args, **kwargs):
        self.aggregators, self.scalers = list(AGGREGATORS), list(SCALERS)
        self.deg = torch.Tensor(deg)                   # PNAStack.py:37: taken as given (PNAEq sanitises, PNA does not)
        self.edge_dim = edge_dim
        super().__init__(*args, **kwargs)

    def get_conv(self, input_dim, output_dim, last_layer=False, edge_dim=None):
        return SingleConv(PNAConv(input_dim, output_dim, self.aggregators, self.scalers, self.deg, edge_dim=edge_dim))

    def _feature_layer(self, width):
        return PyGBatchNorm(width)

    def _embedding(self, data, plan, higher):
        eattr = data.edge_attr if self.use_edge_attr else None
        x = data.x
        if self.use_global_attn:
            x, eattr = self._gps_embed(data, higher)
        return x, data.pos, {"edge_attr": eattr}

    def __str__(self):
        return "PNAStack"
