"""Oracle: torch_geometric 2.6.1 ``CGConv`` [3P-memory] in the configuration CGCNNStack builds
(hydragnn/models/CGCNNStack.py:60-80: aggr "add", batch_norm=False, bias=True), and the CGCNN stack on
``oracle.base.StackOracle``.  Test infrastructure only.

PyG is absent here, so ``CGConv`` is written from the published algorithm:
  * ``lin_f = Linear(2 channels + dim, channels)`` and ``lin_s`` alike, drawn at construction and again by
    ``reset_parameters`` (lin_f, then lin_s); with ``batch_norm=False`` there is no ``bn`` module;
  * ``message(x_i, x_j, edge_attr)``: z = cat[x_i, x_j] (cat[x_i, x_j, edge_attr] with edge attributes), x_i the TARGET
    (edge_index[1], flow source_to_target), m = sigmoid(lin_f(z)) * softplus(lin_s(z));
  * ``forward``: out = sum of m at the targets (aggr "add", a scatter-add in edge order) + x.
tests/golden/make_cgcnn_golden.py plugs this class into the reference's own CGCNNStack.py + Base.py + gps.py, so
models_cgcnn.pt pins everything except this class; test_oracle_cgcnn.py pins this class by hand-computed cases.

``CGCNNStackOracle``: ``Base._init_conv`` (a PyG BatchNorm after every conv), CGConv keeping its width, and no conv-type node
heads.
"""
import torch
import torch.nn.functional as F
from torch import nn

from .base import StackOracle, _Conv
from .gps import PyGBatchNorm


class CGConv(nn.Module):
    def __init__(self, channels, dim=0, aggr="add", batch_norm=False, bias=True, **kwargs):
        assert aggr == "add" and not batch_norm, "only CGCNNStack's configuration"
        super().__init__()
        if isinstance(channels, int):
            channels = (channels, channels)
        self.channels, self.dim = channels, dim
        self.lin_f = nn.Linear(sum(channels) + dim, channels[1], bias=bias)
        self.lin_s = nn.Linear(sum(channels) + dim, channels[1], bias=bias)
        self.bn = None
        self.reset_parameters()

    def reset_parameters(self):
        self.lin_f.reset_parameters()
        self.lin_s.reset_parameters()

    def message(self, x_i, x_j, edge_attr):
        z = torch.cat([x_i, x_j] if edge_attr is None else [x_i, x_j, edge_attr], dim=-1)
        return self.lin_f(z).sigmoid() * F.softplus(self.lin_s(z))

    def forward(self, x, edge_index, edge_attr=None):
        src, dst = edge_index[0], edge_index[1]
        m = self.message(x[dst], x[src], edge_attr)
        out = torch.zeros(x.shape[0], m.shape[1], dtype=m.dtype).index_add_(0, dst, m)
        return out + x


class CGCNNStackOracle(StackOracle):
    def __init__(self, input_dim, hidden_dim, output_dim, output_type, output_heads, edge_dim=0, **kw):
        self.edge_dim = edge_dim
        super().__init__(input_dim, hidden_dim, output_dim, output_type, output_heads, **kw)

    def _get_conv(self, fin, fout, last, edge_dim=None):
        return _Conv([CGConv(fin, edge_dim)])                # CGConv keeps its width: output_dim is not read

    def _feature_layer(self, width):
        return PyGBatchNorm(width)

    def _init_node_conv(self):
        assert all(br["architecture"]["type"] != "conv" for br in self.config_heads["node"]), "CGCNN builds no conv-type node heads"

    def _run_conv(self, conv, x, equiv, ctx):
        return conv.module_0(x, ctx["edge_index"], ctx["edge_attr"]), equiv
