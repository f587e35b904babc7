"""Oracle: torch_geometric 2.6.1 ``PNAConv`` [3P-memory] in the configuration PNAStack builds
(hydragnn/models/PNAStack.py:42-53: towers = 1, pre_layers = post_layers = 1, divide_input = False), and the PNA stack on
``oracle.base.StackOracle``.  Test infrastructure only.

PyG is absent here, so this class is written from the published algorithm; the reference's own modified copy
(hydragnn/models/PNAPlusStack.py:144-279) is in-repo evidence for its structure:
  * ``edge_encoder = Linear(edge_dim, F_in)``, ``pre_nns[0] = Sequential(Linear((3 if edge_dim else 2) F_in, F_in))``,
    ``post_nns[0] = Sequential(Linear((|aggregators| |scalers| + 1) F_in, F_out))``, ``lin = Linear(F_out, F_out)``;
  * every Linear draws at construction, then ``reset_parameters`` draws edge_encoder, pre_nns, post_nns, lin again;
  * ``message(x_i, x_j, edge_attr) = pre_nn(cat[x_i, x_j, edge_encoder(edge_attr)])`` with x_i the TARGET
    (edge_index[1], flow source_to_target) and x_j the source;
  * ``forward = lin(post_nn(cat[x, DegreeScalerAggregation(messages at the targets)]))``.
The aggregation is ``oracle.pnaeq.DegreeScalerAggregation``.  tests/golden/make_pna_golden.py plugs this class into the
reference's own PNAStack.py + Base.py, so models_pna.pt pins everything except this class; test_oracle_pna.py pins this class
by hand-computed cases.

``PNAStackOracle`` is the default ``Base._init_conv`` (a PyG BatchNorm after every conv, hydragnn/models/Base.py:446-463) with
PNAStack.get_conv.  Its parameter and buffer names are the reference's, so a state dict of either the reference or the engine
loads into it strictly.
"""
import torch
from torch import nn

from .base import StackOracle, _Conv
from .gps import PyGBatchNorm
from .pnaeq import DegreeScalerAggregation

AGGREGATORS = ["mean", "min", "max", "std"]
SCALERS = ["identity", "amplification", "attenuation", "linear"]


class PNAConv(nn.Module):
    def __init__(self, in_channels, out_channels, aggregators, scalers, deg, edge_dim=None, towers=1, pre_layers=1,
                 post_layers=1, divide_input=False, **kwargs):
        assert towers == 1 and pre_layers == 1 and post_layers == 1 and not divide_input, "only PNAStack's configuration"
        super().__init__()
        self.in_channels, self.out_channels, self.edge_dim = in_channels, out_channels, edge_dim
        self.towers, self.divide_input = towers, divide_input
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
        for seq in (self.pre_nns[0], self.post_nns[0]):
            for m in seq:
                m.reset_parameters()
        self.lin.reset_parameters()

    def message(self, x_i, x_j, edge_attr):
        if edge_attr is not None:
            h = torch.cat([x_i, x_j, self.edge_encoder(edge_attr)], dim=-1)
        else:
            h = torch.cat([x_i, x_j], dim=-1)
        return self.pre_nns[0](h)

    def forward(self, x, edge_index, edge_attr=None):
        src, dst = edge_index[0], edge_index[1]
        m = self.message(x[dst], x[src], edge_attr)
        out = self.aggr_module(m, dst, x.shape[0])
        return self.lin(self.post_nns[0](torch.cat([x, out], dim=-1)))


class PNAStackOracle(StackOracle):
    def __init__(self, input_dim, hidden_dim, output_dim, output_type, output_heads, pna_deg, edge_dim=None, **kw):
        self.deg = torch.Tensor(pna_deg)                         # PNAStack.py:37: taken as given
        self.edge_dim = edge_dim
        super().__init__(input_dim, hidden_dim, output_dim, output_type, output_heads, **kw)

    def _get_conv(self, fin, fout, last, edge_dim=None):
        return _Conv([PNAConv(fin, fout, AGGREGATORS, SCALERS, self.deg, edge_dim=edge_dim)])

    def _feature_layer(self, width):
        return PyGBatchNorm(width)

    def _run_conv(self, conv, x, equiv, ctx):
        return conv.module_0(x, ctx["edge_index"], ctx["edge_attr"]), equiv
