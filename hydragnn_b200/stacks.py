"""EGNN and PaiNN stacks + the shared encoder / multi-head decoder, executing on libhgb.so.

Host-side mirror of the reference's plugin surface for this path:
``hydragnn/models/Base.py`` (encoder loop :697-727, pooling :733-738, heads :742-846, losses :848-906),
``hydragnn/models/EGCLStack.py`` and ``hydragnn/models/PAINNStack.py``.  Module / parameter names are the
reference's (``graph_convs.<i>.module_<k>...``, ``graph_shared.branch-0...``, ``heads_NN.<i>.branch-0...``)
so reference checkpoints load (SURVEY 8f-2); class names ``E_GCL`` / ``PainnMessage`` / ``PainnUpdate`` are
kept because reference tests locate the modules by class (tests/test_forces_equivariant.py:93-114).

Every conv has two execution modes, selected per forward call:
* fused (default): hand-written forward + first-order backward kernels;
* any-order (``higher_order=True``; chosen automatically for MLIP *training*, where the force loss is
  differentiated again -- hydragnn/models/create.py:718-724 with ``create_graph=True``): the same math
  composed from the closed primitives GatherRows / SegmentSum / MatMul, with ATen only for elementwise glue.
"""
import os

import torch
import torch.nn.functional as F
from torch import nn

from . import ops
from .ops import GatherRows, LinearAct, MatMul, SegmentSum  # noqa: F401


# ------------------------------------------------------------------------------------------------
# activation / loss selection  (hydragnn/utils/model/model.py:30-62)
# ------------------------------------------------------------------------------------------------
def activation_function_selection(name):
    table = {"relu": nn.ReLU, "selu": nn.SELU, "elu": nn.ELU, "sigmoid": nn.Sigmoid,
             "lrelu_01": lambda: nn.LeakyReLU(0.1), "lrelu_025": lambda: nn.LeakyReLU(0.25),
             "lrelu_05": lambda: nn.LeakyReLU(0.5)}
    if name == "prelu":
        raise ValueError("activation 'prelu' (a learnable slope) is not supported by the b200 engine")
    if name not in table:
        raise ValueError("Unknown activation function: " + str(name))
    return table[name]()


def _act_code(mod):
    """(kernel activation name, parameter) of an nn activation module, or None if it is not one."""
    if isinstance(mod, nn.ReLU):
        return "relu", 0.0
    if isinstance(mod, nn.SiLU):
        return "silu", 0.0
    if isinstance(mod, nn.Tanh):
        return "tanh", 0.0
    if isinstance(mod, nn.Sigmoid):
        return "sigmoid", 0.0
    if isinstance(mod, nn.LeakyReLU):
        return "lrelu", float(mod.negative_slope)
    if isinstance(mod, nn.ELU) and mod.alpha == 1.0:
        return "elu", 0.0
    if isinstance(mod, nn.SELU):
        return "selu", 0.0
    return None


def loss_function_selection(name):
    if name == "mse":
        return _Loss(0, False)
    if name == "mae":
        return _Loss(1, False)
    if name == "rmse":
        return _Loss(0, True)
    raise ValueError("loss_function_type %r is not supported by the b200 engine (mse / mae / rmse)" % (name,))


class _Loss:
    """mse / mae / rmse.  Uses the fused value+gradient kernel when only first derivatives can be asked
    for, plain tensor arithmetic (any-order differentiable) when the prediction carries a graph that
    will itself be differentiated (forces)."""

    def __init__(self, mode, sqrt):
        self.mode, self.sqrt = mode, sqrt

    def __call__(self, pred, target, any_order=False):
        target = target.to(pred.dtype)
        if any_order or not pred.is_cuda:
            d = pred - target
            val = (d * d).mean() if self.mode == 0 else d.abs().mean()
        else:
            val = ops.LossFn.apply(pred.reshape(-1), target.reshape(-1), self.mode)
        return torch.sqrt(val) if self.sqrt else val

    def masked(self, pred, target, valid_rows, row_width):
        """Mean over the first ``valid_rows[0]`` rows only (capacity-padded batches, hydragnn_b200/padded.py)."""
        val = ops.LossFn.apply(pred.reshape(-1), target.to(pred.dtype).reshape(-1), self.mode, valid_rows, row_width)
        return torch.sqrt(val) if self.sqrt else val

    def masked_any_order(self, pred, target, mask, count):
        """Any-order differentiable masked mean: ``mask`` is 0/1 per element, ``count`` the (device) number of real elements."""
        d = (pred - target.to(pred.dtype)) * mask
        val = ((d * d).sum() if self.mode == 0 else d.abs().sum()) / count
        return torch.sqrt(val) if self.sqrt else val


PAD_MLP = os.environ.get("HGB_PAD_MLP", "1") == "1"
PAD_MLP_MIN_ROWS = 32768      # below this the chain is launch-bound and the extra pad / slice kernels cost more than the GEMMs save


def _round32(v):
    return (int(v) + 31) // 32 * 32


def _padded_chain(mods, x):
    """Head MLPs carry the reference's widths (60, 20, 1 / 50, 25 / 200: examples/*.json) that the tensor-core Linear cannot take
    (multiples of 32).  On many rows the chain is run with every width rounded up to a multiple of 32: weights / biases are
    zero-padded (tiny, differentiable ``F.pad``), the activations between the layers stay padded, the result is sliced once at the
    end.  Exact: the padded weight columns are zero, so whatever the activation makes of the padded columns meets a zero weight,
    and the gradient of the padding is dropped by ``F.pad``'s own backward.  Returns [(weight, bias)] per Linear, or None."""
    if not (PAD_MLP and x.is_cuda and (ops._TC["enabled"] or ops.EXACT_TC)):
        return None
    k0 = x.shape[-1]
    rows = x.numel() // max(k0, 1)
    lins = [m for m in mods if isinstance(m, nn.Linear)]
    if rows < PAD_MLP_MIN_ROWS or not lins or k0 % 32 or not 32 <= k0 <= 1024 or lins[0].in_features != k0:
        return None
    if any((not isinstance(m, nn.Linear)) and _act_code(m) is None for m in mods):
        return None
    if all(l.out_features % 32 == 0 for l in lins) or any(l.out_features > 1024 for l in lins):
        return None
    out, kin = [], k0
    for l in lins:
        if l.in_features > kin or _round32(l.in_features) != kin:
            return None                                   # not a plain chain
        nout = _round32(l.out_features)
        w = F.pad(l.weight, (0, kin - l.in_features, 0, nout - l.out_features))
        b = F.pad(l.bias, (0, nout - l.out_features)) if l.bias is not None else None
        out.append((w, b))
        kin = nout
    return out


def run_mlp(seq, x, higher_order=False):
    """Execute an ``nn.Sequential`` of Linear / activation modules on the engine: every Linear (with the
    activation that follows it) is one fused kernel; in any-order mode it is MatMul + ATen glue."""
    mods = list(seq)
    padded = _padded_chain(mods, x)
    params = iter(padded) if padded is not None else None

    def wb(lin):
        return next(params) if params is not None else (lin.weight, lin.bias)

    i = 0
    while i < len(mods):
        m = mods[i]
        if isinstance(m, nn.Linear):
            code = _act_code(mods[i + 1]) if i + 1 < len(mods) else None
            w, b = wb(m)
            if (not higher_order and code is not None and i + 2 < len(mods) and isinstance(mods[i + 2], nn.Linear)):
                # Linear - act - Linear (- act): one autograd node, activation gradient folded into a GEMM epilogue
                w2, b2 = wb(mods[i + 2])
                code2 = _act_code(mods[i + 3]) if i + 3 < len(mods) else None
                x = ops.mlp2(x, w, b, code[0], code[1], w2, b2, code2[0] if code2 else None, code2[1] if code2 else 0.0)
                i += 4 if code2 is not None else 3
                continue
            if higher_order:
                x = ops.linear_any_order(x, w, b)
            elif code is not None:
                x = ops.linear_act(x, w, b, code[0], code[1])
                i += 1
            else:
                x = ops.linear_act(x, w, b)
        else:
            x = m(x)
        i += 1
    if padded is not None:
        x = x[..., :[m for m in mods if isinstance(m, nn.Linear)][-1].out_features]
    return x


# ------------------------------------------------------------------------------------------------
# EGNN  (hydragnn/models/EGCLStack.py:180-300)
# ------------------------------------------------------------------------------------------------
class E_GCL(nn.Module):
    def __init__(self, input_channels, output_channels, hidden_channels, edge_attr_dim=0, equivariant=False):
        super().__init__()
        ed = edge_attr_dim or 0
        self.equivariant = bool(equivariant)
        self.edge_attr_dim = ed
        self.edge_mlp = nn.Sequential(nn.Linear(2 * input_channels + 1 + ed, hidden_channels), nn.ReLU(),
                                      nn.Linear(hidden_channels, hidden_channels), nn.ReLU())
        self.node_mlp = nn.Sequential(nn.Linear(hidden_channels + input_channels, hidden_channels), nn.ReLU(),
                                      nn.Linear(hidden_channels, output_channels))
        if self.equivariant:
            last = nn.Linear(hidden_channels, 1, bias=False)
            nn.init.xavier_uniform_(last.weight, gain=0.001)
            self.coord_mlp = nn.Sequential(nn.Linear(hidden_channels, hidden_channels), nn.ReLU(), last, nn.Tanh())

    def _fused_ok(self, x, edge_attr):
        hid = self.edge_mlp[2].weight.shape[0]
        return (ops.FUSED_EGNN and not self.equivariant and edge_attr is None and x.is_cuda and ops.egnn_edge_supported(hid)
                and self.edge_mlp[2].weight.shape[1] == hid)

    def _forward_fused(self, x, coord, plan, edge_shifts, higher_order, cache):
        """edge model + scatter in ONE kernel (csrc/hgb_egnn.cu), any order of differentiation the MLIP loss needs; the node
        model stays a Linear-ReLU-Linear chain (fused first-order block, or closed primitives in any-order mode)."""
        lin0, fin = self.edge_mlp[0], x.shape[1]
        w0 = lin0.weight
        key = (coord.data_ptr(), coord._version, id(plan))
        if cache is not None and cache.get("key") == key:
            radial = cache["radial"]                         # the geometry of a non-equivariant stack is the same in every layer
        else:
            radial = ops.EdgeLenFn.apply(coord, edge_shifts, plan)
            if cache is not None:
                cache["key"], cache["radial"] = key, radial
        lin = ops.linear_any_order if higher_order else ops.linear_act
        pq = lin(x, torch.cat([w0[:, :fin], w0[:, fin:2 * fin]], dim=0), None)          # [N, 2H] = [x W0a^T | x W0b^T]
        agg = ops.EgnnEdgeFn.apply(pq, radial, w0[:, 2 * fin], lin0.bias, self.edge_mlp[2].weight, self.edge_mlp[2].bias, plan)
        out = run_mlp(self.node_mlp, torch.cat([x, agg], dim=1), higher_order)       # :262-263
        return out, coord

    def forward(self, x, coord, plan, edge_attr=None, edge_shifts=None, higher_order=False, cache=None):
        n = x.shape[0]
        if self._fused_ok(x, edge_attr):
            return self._forward_fused(x, coord, plan, edge_shifts, higher_order, cache)
        # geometry with eps = 1.0 (quirk Q3, EGCLStack.py:280-282); "radial" is the length
        if higher_order:
            vec = GatherRows.apply(coord, plan.by_col) - GatherRows.apply(coord, plan.by_row)
            if edge_shifts is not None:
                vec = vec + edge_shifts
            radial = torch.linalg.norm(vec, dim=-1, keepdim=True)
            coord_diff = vec / (radial + 1.0)
        else:
            _, radial, coord_diff = ops.EdgeGeomFn.apply(coord, edge_shifts, plan, 1.0)
        # edge_mlp (:245-250).  Its first Linear acts on [x_row | x_col | radial | edge_attr]; it is linear in the blocks,
        # so the two node blocks are multiplied per NODE (N rows instead of E) and gathered per edge afterwards.
        lin0, fin = self.edge_mlp[0], x.shape[1]
        w0 = lin0.weight
        lin = ops.linear_any_order if higher_order else ops.linear_act
        h = GatherRows.apply(lin(x, w0[:, :fin], None), plan.by_row) + GatherRows.apply(lin(x, w0[:, fin:2 * fin], None), plan.by_col)
        h = h + radial * w0[:, 2 * fin] + lin0.bias
        if edge_attr is not None:
            h = h + lin(edge_attr, w0[:, 2 * fin + 1:], None)
        m = run_mlp(self.edge_mlp[2:], self.edge_mlp[1](h), higher_order)
        if self.equivariant:                                                         # :268-276
            trans = torch.clamp(coord_diff * run_mlp(self.coord_mlp, m, higher_order), min=-100, max=100)
            cnt = (plan.by_row.rowptr[1:] - plan.by_row.rowptr[:-1]).clamp(min=1).to(trans.dtype)
            coord = coord + SegmentSum.apply(trans, plan.by_row) / cnt[:, None]
        agg = SegmentSum.apply(m, plan.by_row)                                       # :257-258
        out = run_mlp(self.node_mlp, torch.cat([x, agg], dim=1), higher_order)       # :262-263
        return out, coord


# ------------------------------------------------------------------------------------------------
# PaiNN  (hydragnn/models/PAINNStack.py:194-328)
# ------------------------------------------------------------------------------------------------
class PainnMessage(nn.Module):
    def __init__(self, node_size, num_radial, cutoff, edge_dim=None):
        super().__init__()
        self.node_size, self.num_radial, self.cutoff, self.edge_dim = node_size, num_radial, cutoff, edge_dim
        self.scalar_message_mlp = nn.Sequential(nn.Linear(node_size, node_size), nn.SiLU(),
                                                nn.Linear(node_size, node_size * 3))
        self.filter_layer = nn.Linear(num_radial, node_size * 3)
        if edge_dim is not None:
            self.edge_filter = nn.Sequential(nn.Linear(edge_dim, node_size), nn.SiLU(),
                                             nn.Linear(node_size, node_size * 3))

    def forward(self, s, v, plan, geom, edge_attr=None, higher_order=False):
        f = self.node_size
        if higher_order:
            diff, dist = geom["unit"], geom["len"]
            n = torch.arange(1, self.num_radial + 1, device=dist.device)
            rbf = torch.sin(dist * n * torch.pi / self.cutoff) / dist
            fcut = torch.where(dist < self.cutoff, 0.5 * (torch.cos(torch.pi * dist / self.cutoff) + 1.0),
                               torch.zeros_like(dist))
            w = ops.linear_any_order(rbf, self.filter_layer.weight, self.filter_layer.bias) * fcut
            if edge_attr is not None:
                w = w * run_mlp(self.edge_filter, edge_attr, True)
            phi = run_mlp(self.scalar_message_mlp, s, True)
            fo = w * GatherRows.apply(phi, plan.by_col)
            g_v, g_e, m_s = torch.split(fo, f, dim=1)
            m_v = GatherRows.apply(v, plan.by_col) * g_v.unsqueeze(1) + g_e.unsqueeze(1) * (diff / dist).unsqueeze(-1)
            return s + SegmentSum.apply(m_s, plan.by_row), v + SegmentSum.apply(m_v, plan.by_row)
        phi = run_mlp(self.scalar_message_mlp, s)
        efilt = run_mlp(self.edge_filter, edge_attr) if edge_attr is not None else None
        if "rec_row" not in geom and self.node_size % 64 == 0:      # built once per batch, reused by every layer
            geom["rec_row"] = ops.painn_edge_records(geom["epack"], plan, "row")
        return ops.PainnMessageFn.apply(phi, s, v, geom["epack"], self.filter_layer.weight, self.filter_layer.bias, efilt, plan,
                                        geom.get("rec_row"))


class PainnUpdate(nn.Module):
    def __init__(self, node_size, last_layer=False):
        super().__init__()
        self.update_U = nn.Linear(node_size, node_size)
        self.update_V = nn.Linear(node_size, node_size)
        self.last_layer = last_layer
        self.update_mlp = nn.Sequential(nn.Linear(node_size * 2, node_size), nn.SiLU(),
                                        nn.Linear(node_size, node_size * (2 if last_layer else 3)))

    def forward(self, s, v, higher_order=False):
        f = v.shape[-1]
        if higher_order:
            uv = ops.linear_any_order(v, self.update_U.weight, self.update_U.bias)
            vv = ops.linear_any_order(v, self.update_V.weight, self.update_V.bias)
            a = run_mlp(self.update_mlp, torch.cat([torch.linalg.norm(vv, dim=1), s], dim=1), True)
            inner = (uv * vv).sum(dim=1)
            if self.last_layer:
                a_sv, a_ss = torch.split(a, f, dim=1)
                return s + a_sv * inner + a_ss, None
            a_vv, a_sv, a_ss = torch.split(a, f, dim=1)
            return s + a_sv * inner + a_ss, v + a_vv.unsqueeze(1) * uv
        fn = ops.PainnUpdateScalarFn if (f == 1 and ops.SCALAR_UPDATE) else ops.PainnUpdateFn   # width-1 layer (quirk Q4)
        s_out, v_out = fn.apply(s, v, self.update_U.weight, self.update_U.bias, self.update_V.weight,
                                               self.update_V.bias, self.update_mlp[0].weight, self.update_mlp[0].bias,
                                               self.update_mlp[2].weight, self.update_mlp[2].bias, self.last_layer)
        return s_out, (None if self.last_layer else v_out)


# ------------------------------------------------------------------------------------------------
# conv containers: children are named module_<i> like the PyG Sequential the reference builds
# ------------------------------------------------------------------------------------------------
class EGNNConv(nn.Module):
    def __init__(self, egcl):
        super().__init__()
        self.module_0 = egcl

    def forward(self, inv_node_feat, equiv_node_feat, plan, edge_attr=None, edge_shifts=None, geom=None, higher_order=False):
        x, pos = self.module_0(inv_node_feat, equiv_node_feat, plan, edge_attr, edge_shifts, higher_order, cache=geom)
        return x, pos


class PainnConv(nn.Module):
    def __init__(self, msg, upd, node_embed_out, vec_embed_out):
        super().__init__()
        self.module_0, self.module_1, self.module_2 = msg, upd, node_embed_out
        if vec_embed_out is not None:
            self.module_3 = vec_embed_out
        self.last = vec_embed_out is None

    def forward(self, inv_node_feat, equiv_node_feat, plan, edge_attr=None, edge_shifts=None, geom=None, higher_order=False):
        s, v = self.module_0(inv_node_feat, equiv_node_feat, plan, geom, edge_attr, higher_order)
        s, v_new = self.module_1(s, v, higher_order)
        s = run_mlp(self.module_2, s, higher_order)
        if self.last:
            return s, v          # PAINNStack.py:124-147: v passes through unchanged in the last layer
        lin = self.module_3
        v_new = ops.linear_any_order(v_new, lin.weight, lin.bias) if higher_order else ops.linear_act(v_new, lin.weight, lin.bias)
        return s, v_new


class MLPNode(nn.Module):
    """Node-level MLP head (hydragnn/models/Base.py:912-979): one shared MLP (``node_type == 'mlp'``) or one MLP per node
    position (``'mlp_per_node'``: graphs of exactly ``num_nodes`` atoms, node i of every graph goes through ``mlp[i]``)."""

    def __init__(self, input_dim, output_dim, hidden_dim_node, activation, num_mlp=1, num_nodes=None):
        super().__init__()
        self.num_nodes, self.output_dim = num_nodes, output_dim
        self.mlp = nn.ModuleList()
        for _ in range(num_mlp):
            dims = [input_dim] + list(hidden_dim_node)
            layers = []
            for d0, d1 in zip(dims[:-1], dims[1:]):
                layers += [nn.Linear(d0, d1), activation]
            layers.append(nn.Linear(dims[-1], output_dim))
            self.mlp.append(nn.Sequential(*layers))

    def forward(self, x, higher_order=False):
        if self.num_nodes is None:
            return run_mlp(self.mlp[0], x, higher_order)
        k = self.num_nodes
        if x.shape[0] % k:
            raise ValueError("mlp_per_node needs graphs of exactly num_nodes = %d atoms" % k)
        xs = x.reshape(-1, k, x.shape[1])
        return torch.stack([run_mlp(self.mlp[i], xs[:, i, :].contiguous(), higher_order) for i in range(k)], dim=1).reshape(x.shape[0], -1)


# ------------------------------------------------------------------------------------------------
# Base: encoder loop + pooling + multi-head decoder
# ------------------------------------------------------------------------------------------------
class Base(nn.Module):
    def __init__(self, input_dim, hidden_dim, output_dim, output_type, config_heads, activation_function_type,
                 loss_function_type, equivariance=False, loss_weights=None, freeze_conv=False, initial_bias=None,
                 num_conv_layers=16, num_nodes=None, graph_pooling="mean", pe_dim=0, global_attn_engine=None,
                 global_attn_type=None, global_attn_heads=0, dropout=0.25):
        super().__init__()
        self.pe_dim, self.global_attn_engine, self.global_attn_type = pe_dim, global_attn_engine, global_attn_type
        self.global_attn_heads, self.dropout, self.global_attn_dropout = global_attn_heads, dropout, dropout
        self.input_dim, self.hidden_dim = input_dim, hidden_dim
        self.num_conv_layers, self.num_nodes = num_conv_layers, num_nodes
        self.head_dims, self.head_type = list(output_dim), list(output_type)
        self.num_heads = len(self.head_dims)
        self.config_heads = config_heads
        self.equivariance = bool(equivariance)
        self.activation_function = activation_function_selection(activation_function_type)
        self.var_output = 0
        if loss_function_type == "GaussianNLLLoss":
            raise ValueError("GaussianNLLLoss is not supported by the b200 engine")
        self.loss_function_type = loss_function_type
        self.loss_function = loss_function_selection(loss_function_type)
        self.ilossweights_hyperp, self.ilossweights_nll = 1, 0
        loss_weights = list(loss_weights if loss_weights is not None else [1.0] * self.num_heads)
        if len(loss_weights) != self.num_heads:
            raise ValueError("Inconsistent number of loss weights and tasks: " + str(len(loss_weights)) + " VS " + str(self.num_heads))
        tot = sum(abs(w) for w in loss_weights)
        self.loss_weights = [w / tot for w in loss_weights]
        self.use_edge_attr = getattr(self, "edge_dim", None) is not None and self.edge_dim > 0
        mode = graph_pooling.lower()
        mode = "add" if mode == "sum" else mode
        if mode not in ("mean", "add", "max"):
            raise ValueError("Unsupported graph_pooling: " + graph_pooling)
        self.graph_pooling = mode
        self.freeze_conv, self.initial_bias = freeze_conv, initial_bias
        self.force_higher_order = False   # tests can force the any-order path
        self.graph_convs = nn.ModuleList()
        self.feature_layers = nn.ModuleList()
        self.heads_NN = nn.ModuleList()
        self.convs_node_hidden, self.batch_norms_node_hidden = nn.ModuleDict(), nn.ModuleDict()      # Base.py:88-91
        self.convs_node_output, self.batch_norms_node_output = nn.ModuleDict(), nn.ModuleDict()
        # global attention: every conv runs at hidden_dim and is wrapped in a GPS layer (Base.py:177-215)
        if self.global_attn_engine:
            if self.global_attn_engine != "GPS":
                raise ValueError("Unsupported global_attn_engine: " + str(self.global_attn_engine))
            self.use_global_attn = True
            self.embed_dim = self.edge_embed_dim = hidden_dim
            self.pos_emb = nn.Linear(self.pe_dim, hidden_dim, bias=False)
            if self.input_dim:
                self.node_emb = nn.Linear(self.input_dim, hidden_dim, bias=False)
                self.node_lin = nn.Linear(2 * hidden_dim, hidden_dim, bias=False)
            if self.is_edge_model:
                self.rel_pos_emb = nn.Linear(self.pe_dim, hidden_dim, bias=False)
                if self.use_edge_attr:
                    self.edge_emb = nn.Linear(self.edge_dim, hidden_dim, bias=False)
                    self.edge_lin = nn.Linear(2 * hidden_dim, hidden_dim, bias=False)
        else:
            self.use_global_attn = False
            self.embed_dim = input_dim
            self.edge_embed_dim = getattr(self, "edge_dim", None)
        self._init_conv()
        if freeze_conv:
            for p in self.graph_convs.parameters():
                p.requires_grad = False
        self._multihead()
        if initial_bias is not None:
            for head, kind in zip(self.heads_NN, self.head_type):
                if kind == "graph":
                    for br in head.values():
                        br[-1].bias.data.fill_(initial_bias)

    # first layer at width input_dim (quirk Q4), last layer flagged (EGCLStack.py:45-70, PAINNStack.py:49-74)
    def _init_conv(self):
        for i in range(self.num_conv_layers):
            last = i == self.num_conv_layers - 1
            conv = self.get_conv(self.embed_dim if i == 0 else self.hidden_dim, self.hidden_dim, last, edge_dim=self.edge_embed_dim)
            if self.use_global_attn:                                           # Base._apply_global_attn :234-247
                from .gps import GPSConv
                conv = GPSConv(self.hidden_dim, conv, heads=self.global_attn_heads, dropout=self.global_attn_dropout,
                               attn_type=self.global_attn_type)
            self.graph_convs.append(conv)
            self.feature_layers.append(nn.Identity())

    def _multihead(self):                                                  # Base.py:590-691
        act = self.activation_function
        self.graph_shared = nn.ModuleDict()
        self.num_branches = 1
        if "graph" in self.config_heads:
            self.num_branches = len(self.config_heads["graph"])
            for br in self.config_heads["graph"]:
                a = br["architecture"]
                layers = [nn.Linear(self.hidden_dim, a["dim_sharedlayers"]), act]
                for _ in range(a["num_sharedlayers"] - 1):
                    layers += [nn.Linear(a["dim_sharedlayers"], a["dim_sharedlayers"]), act]
                self.graph_shared[br["type"]] = nn.Sequential(*layers)
        if "node" in self.config_heads:
            self._init_node_conv()
        inode = 0
        for ih in range(self.num_heads):
            head = nn.ModuleDict()
            if self.head_type[ih] == "graph":
                for br in self.config_heads["graph"]:
                    a = br["architecture"]
                    hid = list(a["dim_headlayers"])
                    layers = [nn.Linear(a["dim_sharedlayers"], hid[0]), act]
                    for j in range(a["num_headlayers"] - 1):
                        layers += [nn.Linear(hid[j], hid[j + 1]), act]
                    layers.append(nn.Linear(hid[-1], self.head_dims[ih]))
                    head[br["type"]] = nn.Sequential(*layers)
            elif self.head_type[ih] == "node":
                for br in self.config_heads["node"]:
                    a = br["architecture"]
                    if a["type"] in ("mlp", "mlp_per_node"):                            # Base.py:648-664
                        per_node = a["type"] == "mlp_per_node"
                        if per_node:
                            assert self.num_nodes is not None, "num_nodes must be provided for mlp_per_node; use 'mlp' for variable-size graphs"
                        head[br["type"]] = MLPNode(self.hidden_dim, self.head_dims[ih], a["dim_headlayers"], act,
                                                   num_mlp=self.num_nodes if per_node else 1, num_nodes=self.num_nodes if per_node else None)
                    elif a["type"] == "conv":                                            # :665-680, the same modules listed again
                        key, mods = br["type"], nn.ModuleList()
                        for conv, bn in zip(self.convs_node_hidden[key], self.batch_norms_node_hidden[key]):
                            mods.append(conv)
                            mods.append(bn)
                        mods.append(self.convs_node_output[key][inode])
                        mods.append(self.batch_norms_node_output[key][inode])
                        head[key] = mods
                        inode += 1
                    else:
                        raise ValueError("Unknown head NN structure for node features" + str(a["type"]) +
                                         "; currently only support 'mlp', 'mlp_per_node' or 'conv'")
            else:
                raise ValueError("Unknown head type" + str(self.head_type[ih]) + "; currently only support 'graph' or 'node'")
            self.heads_NN.append(head)

    def _init_node_conv(self):
        """Base._init_node_conv (:508-588): conv-type node heads; the hidden convolutions are shared between the heads."""
        from .gps import PyGBatchNorm
        cfgs = self.config_heads["node"]
        if any(br["architecture"]["type"] != "conv" for br in cfgs):
            return
        node_heads = [i for i, t in enumerate(self.head_type) if t == "node"]
        if not node_heads:
            return
        if self.use_global_attn or len(cfgs) > 1:
            raise ValueError("b200 engine: conv-type node heads are implemented for one branch and without global attention")
        for br in cfgs:
            a = br["architecture"]
            hid = a["dim_headlayers"]
            ch, bh, co, bo = nn.ModuleList(), nn.ModuleList(), nn.ModuleList(), nn.ModuleList()
            ch.append(self.get_conv(self.hidden_dim, hid[0], last_layer=False))
            bh.append(PyGBatchNorm(hid[0]))
            for k in range(a["num_headlayers"] - 1):
                ch.append(self.get_conv(hid[k], hid[k + 1], last_layer=False))
                bh.append(PyGBatchNorm(hid[k + 1]))
            for ih in node_heads:
                co.append(self.get_conv(hid[-1], self.head_dims[ih], last_layer=True))
                bo.append(PyGBatchNorm(self.head_dims[ih]))
            key = br["type"]
            self.convs_node_hidden[key], self.batch_norms_node_hidden[key] = ch, bh
            self.convs_node_output[key], self.batch_norms_node_output[key] = co, bo

    # -- per-batch preparation -----------------------------------------------------------------------
    @staticmethod
    def plan_for(data):
        plan = data.__dict__.get("_hgb_plan") if hasattr(data, "__dict__") else None
        ei = data.edge_index
        if plan is None or plan.num_edges != ei.shape[1] or plan.row.device != ei.device or plan._src is not ei:
            hint = data.__dict__.get("_hgb_col_sorted") if hasattr(data, "__dict__") else None     # (edge_index, rowptr[, graph_ptr])
            ok = ops.COL_HINT and hint is not None and hint[0] is ei
            plan = ops.EdgePlan(ei, data.pos.shape[0] if data.pos is not None else data.x.shape[0],
                                col_rowptr=hint[1] if ok else None, graph_ptr=hint[2] if (ok and len(hint) > 2) else None)
            plan._src = ei
            try:
                data._hgb_plan = plan
            except Exception:
                pass
        return plan

    def _gps_embed(self, data, higher):
        """Node / edge embeddings used when global attention is on (Base.py:477-491): returns (x, edge_attr)."""
        lin = (lambda m, t: ops.linear_any_order(t, m.weight, None)) if higher else (lambda m, t: ops.linear_act(t, m.weight, None))
        x = lin(self.pos_emb, data.pe)
        if self.input_dim:
            x = lin(self.node_lin, torch.cat((lin(self.node_emb, data.x.float()), x), 1))
        e = None
        if self.is_edge_model:
            e = lin(self.rel_pos_emb, data.rel_pe)
            if self.use_edge_attr:
                e = lin(self.edge_lin, torch.cat((lin(self.edge_emb, data.edge_attr), e), 1))
        return x, e

    def _higher_order(self, data):
        pos = data.pos
        return bool(self.force_higher_order or
                    (self.training and torch.is_grad_enabled() and pos is not None and pos.requires_grad))

    def forward(self, data):
        x = data.x
        if x.dtype != torch.float32:
            raise RuntimeError("b200 engine kernels are fp32 (bf16 via autocast-style GEMMs); got " + str(x.dtype))
        higher = self._higher_order(data)
        if getattr(self, "precision", "fp32") == "bf16" and not ops._TC["enabled"]:
            with ops.tensor_cores(True):       # large-M Linears on wgmma (TF32 in, fp32 accumulate)
                return self.forward(data)
        plan = self.plan_for(data)
        inv, equiv, conv_args = self._embedding(data, plan, higher)
        for conv, feat in zip(self.graph_convs, self.feature_layers):
            inv, equiv = conv(inv_node_feat=inv, equiv_node_feat=equiv, plan=plan, higher_order=higher, **conv_args)
            inv = self.activation_function(feat(inv))                        # Base.py:726
        x = inv
        batch = data.batch
        if batch is None:
            batch = torch.zeros(x.shape[0], dtype=torch.long, device=x.device)
        num_graphs = data.__dict__.get("_num_graphs") if hasattr(data, "__dict__") else None
        if num_graphs is None:
            num_graphs = int(batch.max()) + 1
        gcsr = data.__dict__.get("_hgb_gcsr") if hasattr(data, "__dict__") else None
        if gcsr is None or gcsr.n != num_graphs or gcsr.idx.numel() != batch.numel():
            gcsr = ops.graph_ptr_from_batch(batch, num_graphs)
            try:
                data._hgb_gcsr = gcsr
            except Exception:
                pass
        x_graph = self.pool(x, gcsr, higher)                                  # Base.py:733-738
        ds = getattr(data, "dataset_name", None)
        outputs = []
        for hd, head, kind in zip(self.head_dims, self.heads_NN, self.head_type):
            if self.num_branches == 1:
                if kind == "graph":
                    h = run_mlp(self.graph_shared["branch-0"], x_graph, higher)
                    outputs.append(run_mlp(head["branch-0"], h, higher)[:, :hd])
                elif isinstance(head["branch-0"], nn.ModuleList):                 # conv-type node head (Base.py:800-810)
                    a, b = x, equiv
                    mods = head["branch-0"]
                    for conv, bn in zip(mods[0::2], mods[1::2]):
                        a, b = conv(inv_node_feat=a, equiv_node_feat=b, plan=plan, higher_order=higher, **conv_args)
                        a = self.activation_function(bn(a))
                    outputs.append(a[:, :hd])
                else:
                    outputs.append(head["branch-0"](x, higher)[:, :hd])
                continue
            ids = ds[:, 0]                                                   # Base.py:770-780, 816-840
            out = None if higher else self._grouped_decode(kind, head, ids, x, x_graph, batch, hd, num_graphs)
            if out is not None:
                outputs.append(out)
                continue
            if kind == "graph":
                out = x.new_zeros(num_graphs, hd)
                for b in ids.unique():
                    msk = ids == b
                    key = "branch-%d" % int(b)
                    out[msk] = run_mlp(head[key], run_mlp(self.graph_shared[key], x_graph[msk], higher), higher)[:, :hd]
            else:
                out = x.new_zeros(x.shape[0], hd)
                for b in ids.unique():
                    msk = (ids == b)[batch]
                    out[msk] = head["branch-%d" % int(b)](x[msk], higher)[:, :hd]
            outputs.append(out)
        return outputs

    def _grouped_decode(self, kind, head, ids, x, x_graph, batch, hd, num_graphs):
        """Branch decoding as grouped GEMMs (SURVEY 8f-4): rows are sorted by dataset branch on the device (CSR over the branch
        ids), each layer of the per-branch MLPs is one ``hgb_grouped_linear`` launch, the result is scattered back -- no
        ``unique()``, no boolean masks, no host synchronisation.  None if the branches differ in architecture."""
        keys = ["branch-%d" % b for b in range(self.num_branches)]
        if any(k not in head for k in keys):
            return None
        if kind == "graph":
            rows_ids, feats = ids, x_graph
            seqs = [nn.Sequential(*list(self.graph_shared[k]), *list(head[k])) for k in keys]
        else:
            if not all(isinstance(head[k], MLPNode) and head[k].num_nodes is None for k in keys):
                return None
            rows_ids, feats = ids[batch], x
            seqs = [head[k].mlp[0] for k in keys]
        bcsr = ops.csr_build(rows_ids.to(torch.int64).contiguous(), self.num_branches)     # rows grouped by branch (stable)
        pcsr = ops.csr_build(bcsr.perm.to(torch.int64), feats.shape[0])                     # the permutation as a gather / scatter pair
        xs = GatherRows.apply(feats, pcsr)
        ys = ops.grouped_mlp(seqs, xs, bcsr.rowptr)
        if ys is None:
            return None
        return SegmentSum.apply(ys, pcsr)[:, :hd]

    def pool(self, x, gcsr, higher_order=False):
        if higher_order and self.graph_pooling != "max":
            out = SegmentSum.apply(x, ops.Csr(gcsr.idx, gcsr.rowptr, None, gcsr.n))
            if self.graph_pooling == "mean":
                cnt = (gcsr.rowptr[1:] - gcsr.rowptr[:-1]).clamp(min=1).to(x.dtype)
                out = out / cnt[:, None]
            return out
        return ops.PoolFn.apply(x, gcsr, self.graph_pooling)

    def loss(self, pred, value, head_index):
        """``loss_hpweighted`` (hydragnn/models/Base.py:879-906)."""
        tot_loss = 0
        tasks_loss = []
        for ihead in range(self.num_heads):
            head_pre = pred[ihead]
            head_val = value[head_index[ihead]].reshape(head_pre.shape)
            li = self.loss_function(head_pre, head_val)
            tot_loss = tot_loss + li * self.loss_weights[ihead]
            tasks_loss.append(li)
        return tot_loss, tasks_loss

    def __str__(self):
        return "Base"


class EGCLStack(Base):
    def __init__(self, edge_attr_dim, *args, max_neighbours=None, **kwargs):
        self.edge_dim = 0 if edge_attr_dim is None else edge_attr_dim       # EGCLStack.py:33-35
        self.is_edge_model = True
        super().__init__(*args, **kwargs)

    def get_conv(self, input_dim, output_dim, last_layer=False, edge_dim=None):
        return EGNNConv(E_GCL(input_dim, output_dim, self.hidden_dim, edge_attr_dim=edge_dim or self.edge_dim,
                              equivariant=self.equivariance and not last_layer))

    def _embedding(self, data, plan, higher):
        shifts = data.edge_shifts                                            # zeros if absent (EGCLStack.py:114-118)
        if self.use_global_attn:
            x, e = self._gps_embed(data, higher)
            return x, data.pos, {"edge_attr": e, "edge_shifts": shifts, "geom": {}}
        return data.x, data.pos, {"edge_attr": data.edge_attr if self.use_edge_attr else None, "edge_shifts": shifts, "geom": {}}

    def __str__(self):
        return "EGCLStack"


class PAINNStack(Base):
    def __init__(self, edge_dim, num_radial, radius, *args, **kwargs):
        self.edge_dim, self.num_radial, self.radius = edge_dim, num_radial, radius
        self.is_edge_model = True
        super().__init__(*args, **kwargs)

    def get_conv(self, input_dim, output_dim, last_layer=False, edge_dim=None):
        hidden = output_dim if input_dim == 1 else input_dim
        assert hidden > 1, "PainnNet requires more than one hidden dimension between input_dim and output_dim."
        msg = PainnMessage(node_size=input_dim, num_radial=self.num_radial, cutoff=self.radius,
                           edge_dim=edge_dim if edge_dim is not None else self.edge_dim)
        upd = PainnUpdate(node_size=input_dim, last_layer=last_layer)
        node_embed_out = nn.Sequential(nn.Linear(input_dim, output_dim), nn.Tanh(), nn.Linear(output_dim, output_dim))
        vec_embed_out = nn.Linear(input_dim, output_dim) if not last_layer else None
        return PainnConv(msg, upd, node_embed_out, vec_embed_out)

    def _embedding(self, data, plan, higher):
        assert data.pos is not None, "PAINN requires node positions (data.pos) to be set."
        x, pos, shifts = data.x, data.pos, data.edge_shifts
        if higher:
            vec = GatherRows.apply(pos, plan.by_col) - GatherRows.apply(pos, plan.by_row)
            if shifts is not None:
                vec = vec + shifts
            ln = torch.linalg.norm(vec, dim=-1, keepdim=True)
            geom = {"unit": vec / (ln + 1e-9), "len": ln}
        else:
            _, ln, unit = ops.EdgeGeomFn.apply(pos, shifts, plan, 1e-9)      # PAINNStack.py:157-159
            geom = {"epack": ops.PainnEdgeEmbedFn.apply(unit, ln, self.num_radial, self.radius)}
        eattr = data.edge_attr if self.use_edge_attr else None
        if self.use_global_attn:
            x, eattr = self._gps_embed(data, higher)
        v = torch.zeros(x.shape[0], 3, x.shape[1], dtype=x.dtype, device=x.device)   # PAINNStack.py:190
        return x, v, {"edge_attr": eattr, "geom": geom}

    def __str__(self):
        return "Base"       # quirk Q10: the reference class defines no __str__, so the model calls itself "Base" (Base.py:908)
