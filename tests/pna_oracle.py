"""CPU restatement of torch_geometric 2.6.1 ``PNAConv`` [3P-memory] in the configuration PNAStack builds
(hydragnn/models/PNAStack.py:42-53: towers = 1, pre_layers = post_layers = 1, divide_input = False).  Test infrastructure only.

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

``PNAStackOracle`` assembles the whole stack without GPS in plain torch on the CPU: the default ``Base._init_conv`` (a PyG
BatchNorm after every conv, hydragnn/models/Base.py:446-463), ``Base.forward``'s layer loop (:707-726), graph pooling, the graph
and ``mlp`` node heads and ``loss_hpweighted``.  Its parameter and buffer names are the reference's, so a state dict of either
the reference or the engine loads into it strictly.  test_oracle_pna.py checks it against models_pna.pt; the GPU tests use it
as the independent reference at the benchmark shapes.
"""
import torch
from torch import nn

from oracle.base import activation, normalize_heads
from oracle.geometry import graph_pool
from oracle.gps import PyGBatchNorm
from oracle.pnaeq import DegreeScalerAggregation


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


class _Sequential(nn.Module):
    """PNAStack.get_conv's PyG Sequential: the conv is its child ``module_0``."""

    def __init__(self, conv):
        super().__init__()
        self.module_0 = conv


class _MLPNode(nn.Module):
    """``MLPNode`` with node_type 'mlp' (Base.py:912-979): one shared MLP under ``mlp.0``."""

    def __init__(self, input_dim, output_dim, hidden, act):
        super().__init__()
        dims = [input_dim] + list(hidden)
        layers = []
        for a, b in zip(dims[:-1], dims[1:]):
            layers += [nn.Linear(a, b), act]
        self.mlp = nn.ModuleList([nn.Sequential(*layers, nn.Linear(dims[-1], output_dim))])

    def forward(self, x):
        return self.mlp[0](x)


class PNAStackOracle(nn.Module):
    def __init__(self, input_dim, hidden_dim, output_dim, output_type, output_heads, pna_deg, edge_dim=None, num_conv_layers=2,
                 activation_function="relu", task_weights=None, graph_pooling="mean", **_unused):
        super().__init__()
        self.act = activation(activation_function)
        self.head_dims, self.head_type = list(output_dim), list(output_type)
        w = list(task_weights if task_weights is not None else [1.0] * len(self.head_dims))
        self.loss_weights = [t / sum(abs(v) for v in w) for t in w]
        self.graph_pooling = "add" if graph_pooling.lower() == "sum" else graph_pooling.lower()
        self.use_edge_attr = edge_dim is not None and edge_dim > 0
        deg = torch.Tensor(pna_deg)
        aggr, scal = ["mean", "min", "max", "std"], ["identity", "amplification", "attenuation", "linear"]
        self.graph_convs, self.feature_layers = nn.ModuleList(), nn.ModuleList()
        for i in range(num_conv_layers):
            conv = PNAConv(input_dim if i == 0 else hidden_dim, hidden_dim, aggr, scal, deg, edge_dim=edge_dim)
            self.graph_convs.append(_Sequential(conv))
            self.feature_layers.append(PyGBatchNorm(hidden_dim))
        heads = normalize_heads(output_heads)
        self.heads_NN, self.graph_shared = nn.ModuleList(), nn.ModuleDict()
        if "graph" in heads:
            a = heads["graph"][0]["architecture"]
            layers = [nn.Linear(hidden_dim, a["dim_sharedlayers"]), self.act]
            for _ in range(a["num_sharedlayers"] - 1):
                layers += [nn.Linear(a["dim_sharedlayers"], a["dim_sharedlayers"]), self.act]
            self.graph_shared["branch-0"] = nn.Sequential(*layers)
        for dim, kind in zip(self.head_dims, self.head_type):
            head = nn.ModuleDict()
            a = heads[kind][0]["architecture"]
            if kind == "graph":
                hid = list(a["dim_headlayers"])
                layers = [nn.Linear(a["dim_sharedlayers"], hid[0]), self.act]
                for j in range(a["num_headlayers"] - 1):
                    layers += [nn.Linear(hid[j], hid[j + 1]), self.act]
                head["branch-0"] = nn.Sequential(*layers, nn.Linear(hid[-1], dim))
            else:
                assert a["type"] == "mlp", "the oracle restates 'mlp' node heads only"
                head["branch-0"] = _MLPNode(hidden_dim, dim, a["dim_headlayers"], self.act)
            self.heads_NN.append(head)

    def forward(self, data):
        x, ei = data.x, data.edge_index
        ea = data.edge_attr if self.use_edge_attr else None
        for conv, bn in zip(self.graph_convs, self.feature_layers):
            x = self.act(bn.module(conv.module_0(x, ei, ea)))
        g = int(data.batch.max()) + 1
        xg = graph_pool(x, data.batch, g, self.graph_pooling)
        out = []
        for dim, kind, head in zip(self.head_dims, self.head_type, self.heads_NN):
            if kind == "graph":
                out.append(head["branch-0"](self.graph_shared["branch-0"](xg))[:, :dim])
            else:
                out.append(head["branch-0"](x)[:, :dim])
        return out

    def loss(self, pred, value, head_index):
        tot = 0
        for w, p, idx in zip(self.loss_weights, pred, head_index):
            tot = tot + torch.nn.functional.mse_loss(p, value[idx].reshape(p.shape).to(p.dtype)) * w
        return tot


def _round_tf32(t):
    """fp32 -> the nearest value with a 10-bit mantissa (TF32), kept in fp32."""
    i = t.contiguous().view(torch.int32)
    return ((i + 0x1000) & ~0x1FFF).view(torch.float32)


class _RoundTF32(torch.autograd.Function):
    @staticmethod
    def forward(ctx, x):
        return _round_tf32(x)

    @staticmethod
    def backward(ctx, g):
        return _round_tf32(g)


class tf32_linears:
    """Context manager: every ``nn.Linear`` of an fp32 oracle rounds its input, its weight and the incoming gradient to TF32
    before the product, as the engine's tensor-core Linears do under precision "bf16".  The rest stays fp32."""

    def __enter__(self):
        self.orig = nn.Linear.forward
        nn.Linear.forward = lambda m, x: torch.nn.functional.linear(_RoundTF32.apply(x), _RoundTF32.apply(m.weight), m.bias)
        return self

    def __exit__(self, *exc):
        nn.Linear.forward = self.orig
        return False
