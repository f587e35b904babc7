"""CPU restatement of torch_geometric 2.6.1 ``GATv2Conv`` [3P-memory] in the configuration GATStack builds
(hydragnn/models/GATStack.py:175-190: add_self_loops=True, fill_value="mean", bias=True, share_weights=False, residual=False),
and of the whole stack.  Test infrastructure only.

PyG is absent here, so ``GATv2Conv`` is written from the published algorithm:
  * ``lin_l`` / ``lin_r`` = Linear(in, heads c) with bias and ``lin_edge`` = Linear(edge_dim, heads c, bias=False) (only with an
    edge_dim), all PyG Linears with glorot weights and uniform(1 / sqrt(in)) biases; ``att`` [1, heads, c]; ``bias`` [heads c]
    (concat) or [c].  Construction draws the Linears once, ``reset_parameters`` draws lin_l, lin_r, lin_edge again, then
    glorot(att) and zeros(bias);
  * ``forward``: x_l = lin_l(x), x_r = lin_r(x) as [N, heads, c]; remove_self_loops, then add_self_loops with
    fill_value="mean" (the loop attribute of node i is the mean of its remaining in-edges' attributes, index edge_index[1], 0
    without any; the loops are appended after the edges);
  * ``edge_update``: z = x_r[i] + x_l[j] (+ lin_edge(a) when edge_attr is given: an AssertionError without lin_edge),
    s = (leaky_relu(z) * att).sum(-1), alpha = softmax(s, i) with the max detached and 1e-16 added to the denominator, then
    dropout on alpha;
  * out[i] = sum alpha x_l[j], viewed [N, heads c] (concat) or averaged over the heads, + bias.
tests/golden/make_gat_golden.py plugs this class into the reference's own GATStack.py + Base.py + gps.py, so models_gat.pt pins
everything except this class; test_oracle_gat.py pins this class by hand-computed cases.

``GATStackOracle`` assembles the stack in plain torch: GAT's ``_init_conv`` (BatchNorm(hidden heads) after the concat convs,
BatchNorm(hidden) after the last), GPS (``oracle.gps.GPSConv`` with the reference's node and edge embeddings, out_lin after the
concat convs), the layer loop, graph pooling, the graph, ``mlp`` and ``conv`` heads and ``loss_hpweighted`` with mse.  Its
parameter and buffer names are the reference's, so a state dict of either the reference or the engine loads into it strictly.
"""
import hashlib
import math

import torch
import torch.nn.functional as F
from torch import nn

from oracle.base import _MLPNode, activation, normalize_heads
from oracle.geometry import graph_pool
from oracle.gps import GPSConv, PyGBatchNorm


def _glorot(w):
    a = math.sqrt(6.0 / (w.size(-2) + w.size(-1)))
    with torch.no_grad():
        w.uniform_(-a, a)


def _reset_linear(lin):
    _glorot(lin.weight)
    if lin.bias is not None:
        b = 1.0 / math.sqrt(lin.in_features)
        with torch.no_grad():
            lin.bias.uniform_(-b, b)


class GATv2Conv(nn.Module):
    def __init__(self, in_channels, out_channels, heads=1, concat=True, negative_slope=0.2, dropout=0.0, add_self_loops=True,
                 edge_dim=None, fill_value="mean", bias=True, share_weights=False, residual=False, **kwargs):
        assert add_self_loops and fill_value == "mean" and bias and not share_weights and not residual, "GATStack's configuration"
        super().__init__()
        self.in_channels, self.out_channels, self.heads, self.concat = in_channels, out_channels, heads, concat
        self.negative_slope, self.dropout, self.edge_dim = negative_slope, dropout, edge_dim
        self.lin_l = nn.Linear(in_channels, heads * out_channels)
        self.lin_r = nn.Linear(in_channels, heads * out_channels)
        self.att = nn.Parameter(torch.empty(1, heads, out_channels))
        self.lin_edge = nn.Linear(edge_dim, heads * out_channels, bias=False) if edge_dim is not None else None
        self.bias = nn.Parameter(torch.empty(heads * out_channels if concat else out_channels))
        self.reset_parameters()

    def reset_parameters(self):
        _reset_linear(self.lin_l)
        _reset_linear(self.lin_r)
        if self.lin_edge is not None:
            _reset_linear(self.lin_edge)
        _glorot(self.att)
        with torch.no_grad():
            self.bias.zero_()

    def forward(self, x, edge_index, edge_attr=None):
        H, C, N = self.heads, self.out_channels, x.shape[0]
        xl = self.lin_l(x).view(N, H, C)
        xr = self.lin_r(x).view(N, H, C)
        keep = edge_index[0] != edge_index[1]                                        # remove_self_loops
        src, dst = edge_index[0][keep], edge_index[1][keep]
        loops = torch.arange(N, dtype=src.dtype)
        if edge_attr is not None:
            if edge_attr.dim() == 1:
                edge_attr = edge_attr.view(-1, 1)
            ea = edge_attr[keep]
            cnt = torch.zeros(N, dtype=ea.dtype).index_add_(0, dst, torch.ones_like(dst, dtype=ea.dtype)).clamp(min=1)
            fill = torch.zeros(N, ea.shape[1], dtype=ea.dtype).index_add_(0, dst, ea) / cnt[:, None]
            ea = torch.cat([ea, fill], 0)
        src, dst = torch.cat([src, loops]), torch.cat([dst, loops])
        z = xr[dst] + xl[src]
        if edge_attr is not None:
            assert self.lin_edge is not None
            z = z + self.lin_edge(ea).view(-1, H, C)
        s = (F.leaky_relu(z, self.negative_slope) * self.att).sum(-1)                # [E', H]
        smax = torch.full((N, H), float("-inf"), dtype=s.dtype).scatter_reduce(0, dst[:, None].expand_as(s), s.detach(), "amax")
        ex = (s - smax[dst]).exp()
        den = torch.zeros(N, H, dtype=s.dtype).index_add_(0, dst, ex) + 1e-16
        alpha = ex / den[dst]
        alpha = F.dropout(alpha, p=self.dropout, training=self.training)
        out = torch.zeros(N, H, C, dtype=xl.dtype).index_add_(0, dst, alpha[:, :, None] * xl[src])
        out = out.reshape(N, H * C) if self.concat else out.mean(dim=1)
        return out + self.bias


class _Sequential(nn.Module):
    """GATStack.get_conv's PyG Sequential: the conv is ``module_0``, out_lin ``module_1``."""

    def __init__(self, conv, out_lin):
        super().__init__()
        self.module_0, self.module_1 = conv, out_lin

    def run(self, x, ei, e):
        return self.module_1(self.module_0(x, ei, e))


class GATStackOracle(nn.Module):
    def __init__(self, input_dim, hidden_dim, output_dim, output_type, output_heads, edge_dim=None, num_conv_layers=2,
                 activation_function="relu", task_weights=None, graph_pooling="mean", num_nodes=None, global_attn_engine=None,
                 global_attn_heads=0, pe_dim=0, heads=6, negative_slope=0.05, **_unused):
        super().__init__()
        self.act = activation(activation_function)
        self.head_dims, self.head_type = list(output_dim), list(output_type)
        w = list(task_weights if task_weights is not None else [1.0] * len(self.head_dims))
        self.loss_weights = [t / sum(abs(v) for v in w) for t in w]
        self.graph_pooling = "add" if graph_pooling.lower() == "sum" else graph_pooling.lower()
        self.input_dim = input_dim
        self.use_edge_attr = edge_dim is not None and edge_dim > 0
        self.gps = bool(global_attn_engine)
        k = heads
        if self.gps:
            self.pos_emb = nn.Linear(pe_dim, hidden_dim, bias=False)
            if input_dim:
                self.node_emb = nn.Linear(input_dim, hidden_dim, bias=False)
                self.node_lin = nn.Linear(2 * hidden_dim, hidden_dim, bias=False)
            self.rel_pos_emb = nn.Linear(pe_dim, hidden_dim, bias=False)
            if self.use_edge_attr:
                self.edge_emb = nn.Linear(edge_dim, hidden_dim, bias=False)
                self.edge_lin = nn.Linear(2 * hidden_dim, hidden_dim, bias=False)

        def conv(i, o, concat, ed):
            lin = nn.Linear(hidden_dim * k, hidden_dim) if (self.gps and concat) else nn.Identity()
            return _Sequential(GATv2Conv(i, o, heads=k, concat=concat, negative_slope=negative_slope, edge_dim=ed), lin)

        ed = hidden_dim if self.gps else edge_dim
        widths = [(input_dim if not self.gps else hidden_dim, True)] + [(hidden_dim if self.gps else hidden_dim * k, True)] * (
            num_conv_layers - 2) + [(hidden_dim if self.gps else hidden_dim * k, False)]
        self.graph_convs, self.feature_layers = nn.ModuleList(), nn.ModuleList()
        for i, concat in widths:
            c = conv(i, hidden_dim, concat, ed)
            self.graph_convs.append(GPSConv(hidden_dim, c, heads=global_attn_heads) if self.gps else c)
            self.feature_layers.append(PyGBatchNorm(hidden_dim * k if (concat and not self.gps) else hidden_dim))
        heads_cfg = normalize_heads(output_heads)
        self.graph_shared, self.heads_NN = nn.ModuleDict(), nn.ModuleList()
        if "graph" in heads_cfg:
            a = heads_cfg["graph"][0]["architecture"]
            layers = [nn.Linear(hidden_dim, a["dim_sharedlayers"]), self.act]
            for _ in range(a["num_sharedlayers"] - 1):
                layers += [nn.Linear(a["dim_sharedlayers"], a["dim_sharedlayers"]), self.act]
            self.graph_shared["branch-0"] = nn.Sequential(*layers)
        self.conv_head = None
        self.convs_node_hidden, self.batch_norms_node_hidden = nn.ModuleDict(), nn.ModuleDict()
        self.convs_node_output, self.batch_norms_node_output = nn.ModuleDict(), nn.ModuleDict()
        if "node" in heads_cfg and heads_cfg["node"][0]["architecture"]["type"] == "conv":
            a = heads_cfg["node"][0]["architecture"]
            hid = a["dim_headlayers"]
            hidden_convs = [conv(hidden_dim, hid[0], True, None), PyGBatchNorm(hid[0] * k)]
            for i in range(a["num_headlayers"] - 1):
                hidden_convs += [conv(hid[i] * k, hid[i + 1], True, None), PyGBatchNorm(hid[i + 1] * k)]
            self.conv_head = (hidden_convs, hid, k)
        for d, kind in zip(self.head_dims, self.head_type):
            head = nn.ModuleDict()
            a = heads_cfg[kind][0]["architecture"]
            if kind == "graph":
                hid = list(a["dim_headlayers"])
                layers = [nn.Linear(a["dim_sharedlayers"], hid[0]), self.act]
                for j in range(a["num_headlayers"] - 1):
                    layers += [nn.Linear(hid[j], hid[j + 1]), self.act]
                head["branch-0"] = nn.Sequential(*layers, nn.Linear(hid[-1], d))
            elif a["type"] == "conv":
                hidden_convs, hid, k = self.conv_head
                outc, outb = conv(hid[-1] * k, d, False, None), PyGBatchNorm(d)
                head["branch-0"] = nn.ModuleList(hidden_convs + [outc, outb])
                if "branch-0" not in self.convs_node_hidden:          # Base.py:88-91: the same modules listed again
                    self.convs_node_hidden["branch-0"] = nn.ModuleList(hidden_convs[0::2])
                    self.batch_norms_node_hidden["branch-0"] = nn.ModuleList(hidden_convs[1::2])
                    self.convs_node_output["branch-0"] = nn.ModuleList()
                    self.batch_norms_node_output["branch-0"] = nn.ModuleList()
                self.convs_node_output["branch-0"].append(outc)
                self.batch_norms_node_output["branch-0"].append(outb)
            else:
                per_node = a["type"] == "mlp_per_node"
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
                x, _ = conv(x, None, lambda h, eq, conv=conv: (conv.conv.run(h, ei, e), eq))
            else:
                x = conv.run(x, ei, e)
            x = self.act(bn(x))
        g = int(batch.max()) + 1
        out = []
        for d, kind, head in zip(self.head_dims, self.head_type, self.heads_NN):
            if kind == "graph":
                out.append(head["branch-0"](self.graph_shared["branch-0"](graph_pool(x, batch, g, self.graph_pooling)))[:, :d])
            elif isinstance(head["branch-0"], nn.ModuleList):
                a = x
                mods = head["branch-0"]
                for conv, bn in zip(mods[0::2], mods[1::2]):
                    a = self.act(bn(conv.run(a, ei, e)))
                out.append(a[:, :d])
            else:
                out.append(head["branch-0"](x)[:, :d])
        return out

    def loss(self, pred, value, head_index):
        tot = 0
        for w, p, idx in zip(self.loss_weights, pred, head_index):
            tot = tot + F.mse_loss(p, value[idx].reshape(p.shape).to(p.dtype)) * w
        return tot


def state_digest(t):
    """SHA-256 of a tensor's dtype, shape and bytes: models_gat.pt pins the reference's seeded state dict entry by entry this way."""
    h = hashlib.sha256(repr((str(t.dtype), tuple(t.shape))).encode())
    h.update(t.detach().contiguous().cpu().numpy().tobytes())
    return h.hexdigest()


def engine_kwargs(case):
    """create_model keyword arguments of a models_gat.pt case (the reference's create.py fixes heads = 6, slope = 0.05)."""
    cfg = dict(case["cfg"])
    if cfg.pop("gps"):
        cfg.update(pe_dim=4, global_attn_engine="GPS", global_attn_type="multihead", global_attn_heads=4)
    return dict(mpnn_type="GAT", task_weights=[1.0] * len(cfg["output_type"]), **cfg)


def seeded_state(case):
    """The reference's seeded state dict of a models_gat.pt case.  The file holds it as names in order with one SHA-256 per entry;
    the engine's own seeded construction (create_model on the CPU) reproduces it, and is checked against every digest here."""
    import hydragnn_b200 as hb
    sd = hb.create_model(**engine_kwargs(case), use_gpu=False).state_dict()
    want = case["state_sha256"]
    assert list(sd.keys()) == list(want.keys()), "state-dict names or order differ from the reference's"
    bad = [k for k, v in sd.items() if state_digest(v) != want[k]]
    assert not bad, "seeded values differ from the reference's: %s" % bad[:5]
    return {k: v.clone() for k, v in sd.items()}


def check_grads(case, named_grads, check):
    """Calls ``check(name, grad, reference)`` for every gradient the case stores.  The conv-head case stores the gradients of its
    head modules only (its 120-wide stack convs are covered by the other cases); every other case stores all of them."""
    names = [n for n, _ in named_grads]
    stored = case["grads"]
    assert set(stored) <= set(names)
    if case.get("grads_scope", "all") == "all":
        assert set(stored) == set(names)
    for n, g in named_grads:
        if n in stored:
            check(n, g, stored[n])


def oracle_from_case(case, dtype=torch.float64):
    """The oracle stack of a models_gat.pt case with the reference's seeded state loaded, in ``dtype``."""
    cfg = dict(case["cfg"])
    if cfg.pop("gps"):
        cfg.update(global_attn_engine="GPS", global_attn_heads=4, pe_dim=4)
    m = GATStackOracle(**cfg, task_weights=[1.0] * len(cfg["output_type"]))
    m.load_state_dict(seeded_state(case), strict=True)
    return m.to(dtype)
