"""CPU restatement of torch_geometric 2.6.1 ``CGConv`` [3P-memory] in the configuration CGCNNStack builds
(hydragnn/models/CGCNNStack.py:60-80: aggr "add", batch_norm=False, bias=True), and of the whole stack.  Test infrastructure only.

PyG is absent here, so ``CGConv`` is written from the published algorithm:
  * ``lin_f = Linear(2 channels + dim, channels)`` and ``lin_s`` alike, drawn at construction and again by
    ``reset_parameters`` (lin_f, then lin_s); with ``batch_norm=False`` there is no ``bn`` module;
  * ``message(x_i, x_j, edge_attr)``: z = cat[x_i, x_j] (cat[x_i, x_j, edge_attr] with edge attributes), x_i the TARGET
    (edge_index[1], flow source_to_target), m = sigmoid(lin_f(z)) * softplus(lin_s(z));
  * ``forward``: out = sum of m at the targets (aggr "add", a scatter-add in edge order) + x.
tests/golden/make_cgcnn_golden.py plugs this class into the reference's own CGCNNStack.py + Base.py + gps.py, so
models_cgcnn.pt pins everything except this class; test_oracle_cgcnn.py pins this class by hand-computed cases.

``CGCNNStackOracle`` assembles the stack in plain torch: ``Base._init_conv`` (a PyG BatchNorm after every conv), GPS
(``oracle.gps.GPSConv`` with the reference's node and edge embeddings), the layer loop, graph pooling, the graph, ``mlp`` and
``mlp_per_node`` heads and ``loss_hpweighted`` with mse.  Its parameter and buffer names are the reference's, so a state dict of
either the reference or the engine loads into it strictly.
"""
import torch
import torch.nn.functional as F
from torch import nn

from oracle.base import _MLPNode, activation, normalize_heads
from oracle.geometry import graph_pool
from oracle.gps import GPSConv, PyGBatchNorm


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


class _Sequential(nn.Module):
    """CGCNNStack.get_conv's PyG Sequential: the conv is its child ``module_0``."""

    def __init__(self, conv):
        super().__init__()
        self.module_0 = conv


class CGCNNStackOracle(nn.Module):
    def __init__(self, input_dim, hidden_dim, output_dim, output_type, output_heads, edge_dim=0, num_conv_layers=2,
                 activation_function="relu", task_weights=None, graph_pooling="mean", num_nodes=None, global_attn_engine=None,
                 global_attn_heads=0, pe_dim=0, **_unused):
        super().__init__()
        self.act = activation(activation_function)
        self.head_dims, self.head_type = list(output_dim), list(output_type)
        w = list(task_weights if task_weights is not None else [1.0] * len(self.head_dims))
        self.loss_weights = [t / sum(abs(v) for v in w) for t in w]
        self.graph_pooling = "add" if graph_pooling.lower() == "sum" else graph_pooling.lower()
        self.input_dim = input_dim
        self.use_edge_attr = edge_dim is not None and edge_dim > 0
        self.gps = bool(global_attn_engine)
        if self.gps:
            self.pos_emb = nn.Linear(pe_dim, hidden_dim, bias=False)
            if input_dim:
                self.node_emb = nn.Linear(input_dim, hidden_dim, bias=False)
                self.node_lin = nn.Linear(2 * hidden_dim, hidden_dim, bias=False)
            self.rel_pos_emb = nn.Linear(pe_dim, hidden_dim, bias=False)
            if self.use_edge_attr:
                self.edge_emb = nn.Linear(edge_dim, hidden_dim, bias=False)
                self.edge_lin = nn.Linear(2 * hidden_dim, hidden_dim, bias=False)
        width, dim = (hidden_dim, hidden_dim) if self.gps else (input_dim, edge_dim)
        self.graph_convs, self.feature_layers = nn.ModuleList(), nn.ModuleList()
        for _ in range(num_conv_layers):
            conv = _Sequential(CGConv(width, dim))
            self.graph_convs.append(GPSConv(hidden_dim, conv, heads=global_attn_heads) if self.gps else conv)
            self.feature_layers.append(PyGBatchNorm(hidden_dim))
        heads = normalize_heads(output_heads)
        self.graph_shared, self.heads_NN = nn.ModuleDict(), nn.ModuleList()
        if "graph" in heads:
            a = heads["graph"][0]["architecture"]
            layers = [nn.Linear(hidden_dim, a["dim_sharedlayers"]), self.act]
            for _ in range(a["num_sharedlayers"] - 1):
                layers += [nn.Linear(a["dim_sharedlayers"], a["dim_sharedlayers"]), self.act]
            self.graph_shared["branch-0"] = nn.Sequential(*layers)
        for d, kind in zip(self.head_dims, self.head_type):
            head = nn.ModuleDict()
            a = heads[kind][0]["architecture"]
            if kind == "graph":
                hid = list(a["dim_headlayers"])
                layers = [nn.Linear(a["dim_sharedlayers"], hid[0]), self.act]
                for j in range(a["num_headlayers"] - 1):
                    layers += [nn.Linear(hid[j], hid[j + 1]), self.act]
                head["branch-0"] = nn.Sequential(*layers, nn.Linear(hid[-1], d))
            else:
                per_node = a["type"] == "mlp_per_node"
                assert per_node or a["type"] == "mlp", "CGCNN builds no conv-type node heads"
                head["branch-0"] = _MLPNode(hidden_dim, d, a["dim_headlayers"], self.act, num_mlp=num_nodes if per_node else 1,
                                            num_nodes=num_nodes if per_node else None)
            self.heads_NN.append(head)

    def forward(self, data):
        x, ei, batch = data.x, data.edge_index, data.batch
        e = data.edge_attr if self.use_edge_attr else None
        if self.gps:
            x = self.pos_emb(data.pe)
            if self.input_dim:
                x = self.node_lin(torch.cat((self.node_emb(data.x), x), 1))
            e = self.rel_pos_emb(data.rel_pe)
            if self.use_edge_attr:
                e = self.edge_lin(torch.cat((self.edge_emb(data.edge_attr), e), 1))
        for conv, bn in zip(self.graph_convs, self.feature_layers):
            if self.gps:
                x, _ = conv(x, None, lambda h, eq, conv=conv: (conv.conv.module_0(h, ei, e), eq))
            else:
                x = conv.module_0(x, ei, e)
            x = self.act(bn(x))
        g = int(batch.max()) + 1
        out = []
        for d, kind, head in zip(self.head_dims, self.head_type, self.heads_NN):
            if kind == "graph":
                out.append(head["branch-0"](self.graph_shared["branch-0"](graph_pool(x, batch, g, self.graph_pooling)))[:, :d])
            else:
                out.append(head["branch-0"](x)[:, :d])
        return out

    def loss(self, pred, value, head_index):
        tot = 0
        for w, p, idx in zip(self.loss_weights, pred, head_index):
            tot = tot + F.mse_loss(p, value[idx].reshape(p.shape).to(p.dtype)) * w
        return tot


def oracle_from_case(case, dtype=torch.float64):
    """The oracle stack of a models_cgcnn.pt case with its state loaded, in ``dtype``."""
    cfg = dict(case["cfg"])
    if cfg.pop("gps"):
        cfg.update(global_attn_engine="GPS", global_attn_heads=4, pe_dim=4)
    m = CGCNNStackOracle(**cfg, task_weights=[1.0] * len(cfg["output_type"]))
    m.load_state_dict(case["state"], strict=True)
    return m.to(dtype)
