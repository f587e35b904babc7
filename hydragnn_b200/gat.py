"""GAT stack on libhgb.so.

Host-side mirror of ``hydragnn/models/GATStack.py`` with torch_geometric 2.6.1 ``GATv2Conv(in, c, heads, concat,
negative_slope, dropout, add_self_loops=True, edge_dim, fill_value="mean", bias=True, share_weights=False, residual=False)``
and GAT's own ``_init_conv`` / ``_init_node_conv``: the concat convs are followed by ``BatchNorm(hidden heads)``, the last
(head-averaging) conv by ``BatchNorm(hidden)``; under GPS every conv runs at hidden_dim and a concat conv is followed by
``out_lin = Linear(hidden heads, hidden)`` inside its PyG ``Sequential`` (``module_1``).  Module and parameter names and the
order of construction are the reference's, so reference checkpoints load strictly.

``lin_l`` and ``lin_r`` run as one [n, 2 heads c] Linear on the engine's dispatch; ``ops.GatConvFn`` then forms, per edge
j -> i, z = x_r[i] + x_l[j] + lin_edge(a), the scores, the softmax over the in-edges of i and its self-loop, the attention
dropout and the weighted sum in one pass over the by-target CSR.  Under GPS the conv's edge input is linear in the raw
r_e = [edge_attr | rel_pe] (or rel_pe alone), so the kernel takes mt = (W_edge L)^T with L built from the bias-free embedding
weights (``Base._raw_edge_input``), and the [E, hidden] edge embedding is never formed.  Higher-order passes
and shapes ``ops.gat_supported`` refuses run the same math composed from GatherRows, SegmentSum, Linear and ATen elementwise
ops, with the dropout mask of ``hgb_gat_dropout_keep`` under the same seed.
"""
import math

import torch
import torch.nn.functional as F
from torch import nn

from . import _lib, ops
from .gps import PyGBatchNorm
from .ops import GatherRows, SegmentSum
from .stacks import Base


def _glorot(w):
    a = math.sqrt(6.0 / (w.size(-2) + w.size(-1)))
    with torch.no_grad():
        w.uniform_(-a, a)


def _pyg_linear_reset(lin):
    """torch_geometric Linear.reset_parameters with weight_initializer="glorot" and the default bias initializer."""
    _glorot(lin.weight)
    if lin.bias is not None:
        bound = 1.0 / math.sqrt(lin.in_features)
        with torch.no_grad():
            lin.bias.uniform_(-bound, bound)


def _segment_max_detached(s, csr):
    """max over the segments of ``csr`` of s [E, H], -inf for an empty segment; no gradient (PyG's softmax detaches it)."""
    s = s.detach().contiguous()
    n, h = csr.n, s.shape[1]
    amin = torch.empty(n, h, dtype=torch.int64, device=s.device)
    amax = torch.empty(n, h, dtype=torch.int64, device=s.device)
    if n:
        _lib.call("hgb_segment_argminmax", ops._p(s), ops._p(csr.rowptr), ops._p(csr.perm), n, h, ops._p(amin), ops._p(amax),
                  ops._stream())
    if s.shape[0] == 0:
        return s.new_full((n, h), float("-inf"))
    vals = torch.gather(s, 0, amax.clamp(min=0))
    return torch.where(amax >= 0, vals, torch.full_like(vals, float("-inf")))


def gat_composed(xlr, r, mt, att, bias, plan, heads, c, concat, slope, keep=None, p=0.0, higher_order=False):
    """The math of ``ops.GatConvFn`` from GatherRows / SegmentSum / Linear and ATen elementwise ops (any order of
    differentiation).  ``keep`` uint8 [e + n, heads] from ``ops.raw_gat_dropout_keep`` (None: no dropout)."""
    n, hc = xlr.shape[0], heads * c
    lin = ops.linear_any_order if higher_order else ops.linear_act
    xl, xr = xlr[:, :hc].contiguous(), xlr[:, hc:].contiguous()
    z = GatherRows.apply(xr, plan.by_col) + GatherRows.apply(xl, plan.by_row)       # [E, hc]: x_r[i] + x_l[j]
    zl = xr + xl                                                                    # the self-loops
    other = plan.row != plan.col                                                   # remove_self_loops
    if r is not None:
        w = other.to(r.dtype)[:, None]
        cnt = SegmentSum.apply(w, plan.by_col).clamp(min=1)
        mean = SegmentSum.apply(r * w, plan.by_col) / cnt                           # fill_value "mean" over the remaining in-edges
        wt = mt.t()
        z = z + lin(r, wt, None)
        zl = zl + lin(mean, wt, None)
    a = att.reshape(1, heads, c)
    s = (F.leaky_relu(z, slope).view(-1, heads, c) * a).sum(-1)
    sl = (F.leaky_relu(zl, slope).view(n, heads, c) * a).sum(-1)
    s = torch.where(other[:, None], s, torch.full_like(s, float("-inf")))
    m = torch.maximum(_segment_max_detached(s, plan.by_col), sl.detach())
    ex = torch.exp(s - GatherRows.apply(m, plan.by_col))
    exl = torch.exp(sl - m)
    den = SegmentSum.apply(ex, plan.by_col) + exl + 1e-16
    al = ex / GatherRows.apply(den, plan.by_col)
    all_ = exl / den
    if keep is not None:
        e = al.shape[0]
        kf = keep.to(al.dtype) / (1.0 - p)
        al, all_ = al * kf[:e], all_ * kf[e:]
    msg = al[:, :, None] * GatherRows.apply(xl, plan.by_row).view(-1, heads, c)
    out = SegmentSum.apply(msg, plan.by_col) + all_[:, :, None] * xl.view(n, heads, c)
    out = out.reshape(n, hc) if concat else out.mean(dim=1)
    return out + bias


class GATv2Conv(nn.Module):
    """torch_geometric 2.6.1 ``GATv2Conv`` in GATStack's configuration.  Construction draws lin_l, lin_r and lin_edge once and
    ``reset_parameters`` draws them again (glorot weights, uniform biases), then glorot(att) and zeros(bias), as PyG does: the
    second draw fixes the seeded values."""

    def __init__(self, in_channels, out_channels, heads=1, concat=True, negative_slope=0.2, dropout=0.0, edge_dim=None):
        super().__init__()
        if edge_dim is not None and edge_dim <= 0:
            raise ValueError("GATv2Conv needs edge_dim None (no edge features) or > 0, got %r" % (edge_dim,))
        self.in_channels, self.out_channels, self.heads, self.concat = in_channels, out_channels, heads, concat
        self.negative_slope, self.dropout, self.edge_dim = negative_slope, dropout, edge_dim
        hc = heads * out_channels
        self.lin_l = nn.Linear(in_channels, hc)
        self.lin_r = nn.Linear(in_channels, hc)
        self.att = nn.Parameter(torch.empty(1, heads, out_channels))
        self.lin_edge = nn.Linear(edge_dim, hc, bias=False) if edge_dim is not None else None
        self.bias = nn.Parameter(torch.empty(hc if concat else out_channels))
        self.reset_parameters()

    def reset_parameters(self):
        _pyg_linear_reset(self.lin_l)
        _pyg_linear_reset(self.lin_r)
        if self.lin_edge is not None:
            _pyg_linear_reset(self.lin_edge)
        _glorot(self.att)
        with torch.no_grad():
            self.bias.zero_()

    def forward(self, x, plan, edge_raw=None, higher_order=False):
        """``edge_raw`` = (r, L): the conv's edge input is r L^T (L None: r itself), or None without one."""
        r, emb = edge_raw if edge_raw is not None else (None, None)
        if r is not None and self.lin_edge is None:
            # PyG's GATv2Conv.edge_update asserts lin_edge is not None when it is handed edge attributes
            raise AssertionError("GATv2Conv was built with edge_dim=None but called with edge_attr")
        if self.lin_edge is None:
            r = None
        heads, c = self.heads, self.out_channels
        w = torch.cat([self.lin_l.weight, self.lin_r.weight], dim=0)
        b = torch.cat([self.lin_l.bias, self.lin_r.bias])
        lin = ops.linear_any_order if higher_order else ops.linear_act
        xlr = lin(x, w, b)                                                           # [N, 2 heads c] = [x_l | x_r]
        mt = None
        if r is not None:
            we = self.lin_edge.weight
            mt = we.t() if emb is None else ops.MatMul.apply(emb, we, True, True)    # (W_edge L)^T  [d, heads c]
        p = float(self.dropout) if self.training else 0.0
        seed = ops.gat_dropout_seed(x.device) if p > 0 else None
        d = 0 if r is None else r.shape[1]
        if not higher_order and x.is_cuda and ops.gat_supported(heads, c, d):
            return ops.GatConvFn.apply(xlr, r, mt, self.att.reshape(-1), self.bias, plan, heads, c, self.concat,
                                       self.negative_slope, p, seed)
        keep = ops.raw_gat_dropout_keep(x.shape[0], plan.num_edges, heads, p, seed) if p > 0 else None
        return gat_composed(xlr, r, mt, self.att, self.bias, plan, heads, c, self.concat, self.negative_slope, keep, p,
                            higher_order)


class GATSequential(nn.Module):
    """The PyG ``Sequential`` of GATStack.get_conv (:192-205): the conv is ``module_0``, ``out_lin`` (a Linear under GPS after a
    concat conv, else Identity) ``module_1``; the lambda step that passes ``equiv_node_feat`` through has no parameters."""

    def __init__(self, conv, out_lin):
        super().__init__()
        self.module_0 = conv
        self.module_1 = out_lin

    def forward(self, inv_node_feat, equiv_node_feat, plan, edge_raw=None, higher_order=False, **kwargs):
        h = self.module_0(inv_node_feat, plan, edge_raw, higher_order)
        lin = self.module_1
        if isinstance(lin, nn.Linear):
            h = (ops.linear_any_order if higher_order else ops.linear_act)(h, lin.weight, lin.bias)
        return h, equiv_node_feat


class GATStack(Base):
    is_edge_model = True

    def __init__(self, heads, negative_slope, edge_dim, *args, **kwargs):
        # self.heads is GATv2Conv's number of attention heads, not the number of output heads
        self.heads = heads
        self.negative_slope = negative_slope
        self.edge_dim = edge_dim
        super().__init__(*args, **kwargs)

    def _init_conv(self):
        """GATStack._init_conv (:39-111): concat convs with head-multiplied widths, a head-averaging last conv."""
        h, k = self.hidden_dim, self.heads
        gps = self.use_global_attn
        mid_in = h if gps else h * k
        self.graph_convs.append(self._wrap(self.get_conv(self.embed_dim, h, concat=True, edge_dim=self.edge_embed_dim)))
        self.feature_layers.append(PyGBatchNorm(h if gps else h * k))
        for _ in range(self.num_conv_layers - 2):
            self.graph_convs.append(self._wrap(self.get_conv(mid_in, h, concat=True, edge_dim=self.edge_embed_dim)))
            self.feature_layers.append(PyGBatchNorm(h if gps else h * k))
        self.graph_convs.append(self._wrap(self.get_conv(mid_in, h, concat=False, edge_dim=self.edge_embed_dim)))
        self.feature_layers.append(PyGBatchNorm(h))

    def _init_node_conv(self):
        """GATStack._init_node_conv (:113-173): conv-type node heads, hidden convs concat with BatchNorm(dim heads), one
        head-averaging output conv per node head; these convs have no edge input (edge_dim=None)."""
        cfgs = self.config_heads["node"]
        assert self.num_branches == len(cfgs), "asumming node head has the same branches as graph head, if any"
        if any(br["architecture"]["type"] != "conv" for br in cfgs):
            return
        node_heads = [i for i, t in enumerate(self.head_type) if t == "node"]
        if not node_heads:
            return
        if self.use_global_attn or len(cfgs) > 1:
            raise ValueError("b200 engine: conv-type node heads are implemented for one branch and without global attention")
        if self.var_output:
            # GATStack._init_node_conv keeps the output convs at head_dim, so the reference's variance is [N, 0] and its
            # GaussianNLLLoss raises
            raise ValueError("b200 engine: GAT conv-type node heads have no variance outputs; GaussianNLLLoss is not supported")
        k = self.heads
        for br in cfgs:
            a = br["architecture"]
            hid = a["dim_headlayers"]
            ch, bh, co, bo = nn.ModuleList(), nn.ModuleList(), nn.ModuleList(), nn.ModuleList()
            ch.append(self.get_conv(self.hidden_dim, hid[0], True))
            bh.append(PyGBatchNorm(hid[0] * k))
            for i in range(a["num_headlayers"] - 1):
                ch.append(self.get_conv(hid[i] * k, hid[i + 1], True))
                bh.append(PyGBatchNorm(hid[i + 1] * k))
            for ih in node_heads:
                co.append(self.get_conv(hid[-1] * k, self.head_dims[ih], False))
                bo.append(PyGBatchNorm(self.head_dims[ih]))
            key = br["type"]
            self.convs_node_hidden[key], self.batch_norms_node_hidden[key] = ch, bh
            self.convs_node_output[key], self.batch_norms_node_output[key] = co, bo

    def get_conv(self, input_dim, output_dim, concat, edge_dim=None):
        gat = GATv2Conv(input_dim, output_dim, heads=self.heads, concat=concat, negative_slope=self.negative_slope,
                        dropout=self.dropout, edge_dim=edge_dim)
        # the reference assigns out_lin on the stack as well; the last call is always a head-averaging conv, so what stays
        # there is an Identity without parameters
        self.out_lin = nn.Linear(self.hidden_dim * self.heads, self.hidden_dim) if (self.use_global_attn and concat) else nn.Identity()
        return GATSequential(gat, self.out_lin)

    def _forward(self, data, higher):
        if self.use_edge_attr and len(self.convs_node_hidden):
            # the reference's head convs are built with edge_dim=None and PyG's GATv2Conv asserts when they are handed the
            # edge attributes: raised here before any kernel is launched
            raise AssertionError("GAT conv-type node heads have no edge input (edge_dim=None) but the model uses edge features")
        return super()._forward(data, higher)

    def _embedding(self, data, plan, higher):
        x, edge_raw = self._raw_edge_input(data, higher)
        return x, data.pos, {"edge_raw": edge_raw}

    def __str__(self):
        return "GATStack"
