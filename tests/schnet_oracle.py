"""Plain-torch restatement of SchNet's pieces for tests (any dtype, fp64 in the tests).

torch_geometric 2.6.1 [3P-memory], absent here, written from the published code:
  * ``GaussianSmearing(start, stop, G)``: offset = linspace(start, stop, G), coeff = -0.5 / (offset[1] - offset[0])^2 (a Python
    float), forward exp(coeff (d - offset)^2);
  * ``ShiftedSoftplus``: softplus(x) - log(2), the shift read back from an fp32 tensor;
  * ``RadiusInteractionGraph(cutoff, max_num_neighbors)``: edge_index = radius_graph(pos, cutoff, batch, max_num_neighbors)
    (torch_cluster's ordering and truncation, ``oracle.radius_graph``), edge_weight = |pos[row] - pos[col]|;
  * ``MessagePassing`` with aggr "add" and flow source_to_target: x_j = x[edge_index[0]], summed at edge_index[1].
tests/golden/make_schnet_golden.py plugs these into the reference's own SCFStack.py, so models_schnet.pt pins everything else.

``cfconv`` is CFConv.forward (hydragnn/models/SCFStack.py:267-298) as one function of plain tensors; the GPU tests compare the
fused kernels against it in fp64.
"""
import math

import torch
import torch.nn.functional as F
from torch import nn

from oracle.radius_graph import radius_graph


class GaussianSmearing(nn.Module):
    def __init__(self, start=0.0, stop=5.0, num_gaussians=50):
        super().__init__()
        offset = torch.linspace(start, stop, num_gaussians)
        self.coeff = -0.5 / (offset[1] - offset[0]).item() ** 2
        self.register_buffer("offset", offset)

    def forward(self, dist):
        dist = dist.view(-1, 1) - self.offset.view(1, -1)
        return torch.exp(self.coeff * torch.pow(dist, 2))


class ShiftedSoftplus(nn.Module):
    def __init__(self):
        super().__init__()
        self.shift = torch.log(torch.tensor(2.0)).item()

    def forward(self, x):
        return F.softplus(x) - self.shift


class RadiusInteractionGraph(nn.Module):
    def __init__(self, cutoff=10.0, max_num_neighbors=32):
        super().__init__()
        self.cutoff, self.max_num_neighbors = cutoff, max_num_neighbors

    def forward(self, pos, batch):
        edge_index = radius_graph(pos, r=self.cutoff, batch=batch, max_num_neighbors=self.max_num_neighbors).to(pos.device)
        row, col = edge_index
        return edge_index, (pos[row] - pos[col]).norm(dim=-1)


class MessagePassing(nn.Module):
    """aggr "add", flow source_to_target; ``propagate(edge_index, **kw)`` lifts every ``*_j`` argument of ``message`` to
    the sources and sums the messages at the targets."""

    def __init__(self, aggr="add", **kw):
        super().__init__()
        assert aggr == "add"

    def propagate(self, edge_index, x, W):
        m = self.message(x[edge_index[0]], W)
        return m.new_zeros((x.shape[0],) + tuple(m.shape[1:])).index_add_(0, edge_index[1], m)


def cfconv(x, pos, edge_index, w_lin1, w1, b1, w2, b2, w_lin2, b_lin2, offset, coeff, cutoff, edge_attr=None):
    """CFConv.forward without the coordinate update: returns (out, W)."""
    row, col = edge_index
    d = (pos[col] - pos[row]).norm(dim=-1)
    c = 0.5 * (torch.cos(d * math.pi / cutoff) + 1.0)
    rbf = torch.exp(coeff * (d.view(-1, 1) - offset.view(1, -1)) ** 2)
    inp = rbf if edge_attr is None else torch.cat([rbf, edge_attr], dim=-1)
    w = (F.linear(F.softplus(F.linear(inp, w1, b1)) - math.log(2.0), w2, b2)) * c.view(-1, 1)
    xl = x @ w_lin1.t()
    agg = torch.zeros_like(xl[:, :1].expand(-1, w.shape[1])).clone().index_add_(0, col, xl[row] * w)
    return agg @ w_lin2.t() + b_lin2, w


def coord_update(pos, edge_index, w, coord_mlp):
    """CFConv.coord_model (SCFStack.py:252-260): pos + mean over the SOURCE index of clamp(coord_diff * coord_mlp(W))."""
    row, col = edge_index
    vec = pos[col] - pos[row]
    coord_diff = vec / (vec.norm(dim=-1, keepdim=True) + 1.0)
    trans = torch.clamp(coord_diff * coord_mlp(w), min=-100, max=100)
    s = torch.zeros_like(pos).index_add_(0, row, trans)
    cnt = torch.bincount(row, minlength=pos.shape[0]).clamp(min=1).to(pos.dtype)
    return pos + s / cnt[:, None]


# ---- the whole stack (hydragnn/models/SCFStack.py + the parts of Base.py it runs) ----------------------------------------------
class _NoState(nn.Module):
    """The stateless ``interaction_graph`` child (``module_0`` of the in-layer Sequential)."""


class CFConv(nn.Module):
    def __init__(self, fin, fout, num_filters, mlp_in, equivariant):
        super().__init__()
        self.lin1 = nn.Linear(fin, num_filters, bias=False)
        self.lin2 = nn.Linear(num_filters, fout)
        self.nn = nn.Sequential(nn.Linear(mlp_in, num_filters), ShiftedSoftplus(), nn.Linear(num_filters, num_filters))
        self.equivariant = equivariant
        if equivariant:
            self.coord_mlp = nn.Sequential(nn.Linear(num_filters, num_filters), nn.ReLU(), nn.Linear(num_filters, 1, bias=False))

    def forward(self, x, pos, edge_index, smearing, cutoff, edge_attr=None):
        out, w = cfconv(x, pos, edge_index, self.lin1.weight, self.nn[0].weight, self.nn[0].bias, self.nn[2].weight, self.nn[2].bias,
                        self.lin2.weight, self.lin2.bias, smearing.offset, smearing.coeff, cutoff, edge_attr)
        if self.equivariant:
            pos = coord_update(pos, edge_index, w, self.coord_mlp)
        return out, pos


class _Seq(nn.Module):
    def __init__(self, conv, in_layer, smearing):
        super().__init__()
        if in_layer:
            self.module_0, self.module_1, self.module_2 = _NoState(), smearing, conv
        else:
            self.module_0 = conv
        self.in_layer = in_layer

    @property
    def conv(self):
        return self.module_2 if self.in_layer else self.module_0


class _MLP(nn.Module):
    def __init__(self, fin, fout, hidden, act):
        super().__init__()
        dims = [fin] + list(hidden)
        layers = []
        for a, b in zip(dims[:-1], dims[1:]):
            layers += [nn.Linear(a, b), act]
        self.mlp = nn.ModuleList([nn.Sequential(*layers, nn.Linear(dims[-1], fout))])

    def forward(self, x):
        return self.mlp[0](x)


class SCFStackOracle(nn.Module):
    """SCFStack with Base's encoder loop (Identity feature layers, activation after every conv), GPS (``oracle.gps.GPSConv``),
    graph pooling, graph / ``mlp`` / ``conv`` node heads and ``loss_hpweighted`` with mse.  Parameter and buffer names are the
    reference's, so its state dicts (and the engine's) load strictly.  Radius graphs are built on the positions rounded to fp32,
    as the reference's fp32 model builds them."""

    def __init__(self, input_dim, hidden_dim, output_dim, output_type, output_heads, num_filters, num_gaussians, radius,
                 max_neighbours=None, edge_dim=None, num_conv_layers=2, activation_function="relu", task_weights=None,
                 graph_pooling="mean", equivariance=False, global_attn_engine=None, global_attn_heads=0, pe_dim=0, **_unused):
        super().__init__()
        from oracle.base import activation, normalize_heads
        from oracle.gps import GPSConv, PyGBatchNorm
        self.act = activation(activation_function)
        self.head_dims, self.head_type = list(output_dim), list(output_type)
        w = list(task_weights if task_weights is not None else [1.0] * len(self.head_dims))
        self.loss_weights = [t / sum(abs(v) for v in w) for t in w]
        self.graph_pooling = "add" if graph_pooling.lower() == "sum" else graph_pooling.lower()
        self.radius, self.max_neighbours, self.input_dim = radius, max_neighbours, input_dim
        self.use_edge_attr = edge_dim is not None and edge_dim > 0
        self.gps = bool(global_attn_engine)
        self.in_layer = not (self.use_edge_attr or self.gps)
        self.distance_expansion = GaussianSmearing(0.0, radius, num_gaussians)
        edge_in = hidden_dim if self.gps else (edge_dim or 0)
        if self.gps:
            self.pos_emb = nn.Linear(pe_dim, hidden_dim, bias=False)
            if input_dim:
                self.node_emb = nn.Linear(input_dim, hidden_dim, bias=False)
                self.node_lin = nn.Linear(2 * hidden_dim, hidden_dim, bias=False)
            self.rel_pos_emb = nn.Linear(pe_dim, hidden_dim, bias=False)
            if self.use_edge_attr:
                self.edge_emb = nn.Linear(edge_dim, hidden_dim, bias=False)
                self.edge_lin = nn.Linear(2 * hidden_dim, hidden_dim, bias=False)

        def seq(fin, fout, last, e_in=edge_in):
            conv = CFConv(fin, fout, num_filters, num_gaussians + e_in, equivariance and not last)
            return _Seq(conv, self.in_layer, self.distance_expansion)

        self.graph_convs = nn.ModuleList()
        for i in range(num_conv_layers):
            s = seq(hidden_dim if (i > 0 or self.gps) else input_dim, hidden_dim, i == num_conv_layers - 1)
            self.graph_convs.append(GPSConv(hidden_dim, s, heads=global_attn_heads) if self.gps else s)
        heads = normalize_heads(output_heads)
        self.graph_shared, self.heads_NN = nn.ModuleDict(), nn.ModuleList()
        if "graph" in heads:
            a = heads["graph"][0]["architecture"]
            layers = [nn.Linear(hidden_dim, a["dim_sharedlayers"]), self.act]
            for _ in range(a["num_sharedlayers"] - 1):
                layers += [nn.Linear(a["dim_sharedlayers"], a["dim_sharedlayers"]), self.act]
            self.graph_shared["branch-0"] = nn.Sequential(*layers)
        node_conv = "node" in heads and heads["node"][0]["architecture"]["type"] == "conv"
        if node_conv:
            a = heads["node"][0]["architecture"]
            hid = a["dim_headlayers"]
            ch = nn.ModuleList([seq(hidden_dim, hid[0], False, 0)] + [seq(hid[k], hid[k + 1], False, 0) for k in range(len(hid) - 1)])
            bh = nn.ModuleList([PyGBatchNorm(h) for h in hid])
            co = nn.ModuleList([seq(hid[-1], d, True, 0) for d, t in zip(self.head_dims, self.head_type) if t == "node"])
            bo = nn.ModuleList([PyGBatchNorm(d) for d, t in zip(self.head_dims, self.head_type) if t == "node"])
            self.convs_node_hidden, self.batch_norms_node_hidden = nn.ModuleDict({"branch-0": ch}), nn.ModuleDict({"branch-0": bh})
            self.convs_node_output, self.batch_norms_node_output = nn.ModuleDict({"branch-0": co}), nn.ModuleDict({"branch-0": bo})
        inode = 0
        for dim, kind in zip(self.head_dims, self.head_type):
            head = nn.ModuleDict()
            a = heads[kind][0]["architecture"]
            if kind == "graph":
                hid = list(a["dim_headlayers"])
                layers = [nn.Linear(a["dim_sharedlayers"], hid[0]), self.act]
                for j in range(a["num_headlayers"] - 1):
                    layers += [nn.Linear(hid[j], hid[j + 1]), self.act]
                head["branch-0"] = nn.Sequential(*layers, nn.Linear(hid[-1], dim))
            elif node_conv:
                mods = nn.ModuleList()
                for c, b in zip(ch, bh):
                    mods.append(c)
                    mods.append(b)
                mods.append(co[inode])
                mods.append(bo[inode])
                inode += 1
                head["branch-0"] = mods
            else:
                head["branch-0"] = _MLP(hidden_dim, dim, a["dim_headlayers"], self.act)
            self.heads_NN.append(head)

    def _run(self, s, x, pos, batch, edge_index, edge_attr):
        if s.in_layer:
            edge_index = radius_graph(pos.detach().float(), self.radius, batch, max_num_neighbors=self.max_neighbours).to(pos.device)
        return s.conv(x, pos, edge_index, self.distance_expansion, self.radius, edge_attr)

    def forward(self, data):
        from oracle.geometry import graph_pool
        x, pos, batch = data.x, data.pos, data.batch
        ei = None if self.in_layer else data.edge_index
        e = data.edge_attr if self.use_edge_attr else None
        if self.gps:
            x = self.pos_emb(data.pe)
            if self.input_dim:
                x = self.node_lin(torch.cat((self.node_emb(data.x), x), 1))
            e = self.rel_pos_emb(data.rel_pe)
            if self.use_edge_attr:
                e = self.edge_lin(torch.cat((self.edge_emb(data.edge_attr), e), 1))
        for conv in self.graph_convs:
            if self.gps:
                x, pos = conv(x, pos, lambda h, p, conv=conv: self._run(conv.conv, h, p, batch, ei, e))
            else:
                x, pos = self._run(conv, x, pos, batch, ei, e)
            x = self.act(x)
        g = int(batch.max()) + 1
        out = []
        for dim, kind, head in zip(self.head_dims, self.head_type, self.heads_NN):
            if kind == "graph":
                out.append(head["branch-0"](self.graph_shared["branch-0"](graph_pool(x, batch, g, self.graph_pooling)))[:, :dim])
            elif isinstance(head["branch-0"], nn.ModuleList):
                a, p = x, pos
                mods = head["branch-0"]
                for c, bn in zip(mods[0::2], mods[1::2]):
                    a, p = self._run(c, a, p, batch, ei, None)
                    a = self.act(bn(a))
                out.append(a[:, :dim])
            else:
                out.append(head["branch-0"](x)[:, :dim])
        return out

    def loss(self, pred, value, head_index):
        tot = 0
        for w, p, idx in zip(self.loss_weights, pred, head_index):
            tot = tot + F.mse_loss(p, value[idx].reshape(p.shape).to(p.dtype)) * w
        return tot


def oracle_from_case(case, dtype=torch.float64):
    """The oracle stack of a models_schnet.pt case with its state loaded, in ``dtype``."""
    cfg = dict(case["cfg"])
    if cfg.pop("gps"):
        cfg.update(global_attn_engine="GPS", global_attn_heads=4, pe_dim=4)
    m = SCFStackOracle(**cfg, task_weights=[1.0])
    m.load_state_dict(case["state"], strict=True)
    return m.to(dtype)
