"""MACE on the engine (``mpnn_type="MACE"``; hydragnn/models/MACEStack.py:70-498 and mace_utils/modules/blocks.py).

Parameter names, shapes and creation order are the reference's (e3nn flat ``weight`` vectors, ``weights_max`` /
``weights.k`` of the symmetric contraction, ``conv_tp_weights.layer<i>.weight``), so state dicts interchange with
the oracle.  What differs is the device layout: a feature with irreps ``F x 0e + F x 1o + ...`` is a LIST of tensors
``[N, 2l+1, F]`` (channels contiguous), never e3nn's mul-major rows; an equivariant Linear is then one GEMM per degree
on a ``[(N (2l+1)), F_in]`` view, and the tensor product / scatter work on whole channel rows.

First-order path (ordinary training, inference, first-order forces): ``conv_tp`` + the receiver scatter and the
correlation-2 symmetric contraction are the fused kernels of hgb_mace.cu (``ops.MaceTpScatterFn``,
``ops.MaceSymContractFn``), the radial MLP and every equivariant Linear run on the wgmma / SIMT Linear kernels, the
spherical harmonics and the radial basis are ATen elementwise glue on [E, 9]-sized tensors.  Any-order path (MLIP double
backward), correlation 3 and channel counts that are not a multiple of 32: the per-path coupling and the contraction are
composed from gathers / segment sums / MatMuls plus ATen einsum glue.
"""
import math
import os

import torch
from torch import nn

from . import e3, ops
from .stacks import (_act_code, activation_function_selection, loss_function_selection, run_mlp)

NUM_ELEMENTS = 118
EDGE_EMBED_KERNEL = os.environ.get("HGB_MACE_EDGE_EMBED", "1") == "1"   # 0: spherical harmonics / radial basis as ATen glue


def _lin(x, w_t, higher, act=None):
    """x [..., k] times w_t^T with w_t [n, k] (no bias)."""
    if higher:
        y = ops.linear_any_order(x, w_t, None)
        return torch.nn.functional.silu(y) if act == "silu" else y
    return ops.linear_act(x, w_t, None, act)


class E3Linear(nn.Module):
    """o3.Linear without biases on per-degree channel-last features.  `irreps_in` / `irreps_out`: [(mul, l, p)]."""

    def __init__(self, irreps_in, irreps_out):
        super().__init__()
        self.irreps_in, self.irreps_out = list(irreps_in), list(irreps_out)
        self.paths = [(i, o) for i, (_, li, pi) in enumerate(self.irreps_in) for o, (_, lo, po) in enumerate(self.irreps_out)
                      if (li, pi) == (lo, po)]
        fan = {}
        for i, o in self.paths:
            fan[o] = fan.get(o, 0) + self.irreps_in[i][0]
        self.alpha = [1.0 / math.sqrt(fan[o]) for _, o in self.paths]
        self.weight_numel = sum(self.irreps_in[i][0] * self.irreps_out[o][0] for i, o in self.paths)
        self.weight = nn.Parameter(torch.randn(self.weight_numel))

    def forward(self, xs, higher=False):
        """xs: list aligned with irreps_in of [N, 2l+1, mul_in]; returns list aligned with irreps_out."""
        outs = [None] * len(self.irreps_out)
        off = 0
        for (i, o), a in zip(self.paths, self.alpha):
            mi, mo = self.irreps_in[i][0], self.irreps_out[o][0]
            w_t = (self.weight[off:off + mi * mo].reshape(mi, mo) * a).t()
            off += mi * mo
            y = _lin(xs[i], w_t, higher)
            outs[o] = y if outs[o] is None else outs[o] + y
        n = xs[0].shape[0]
        return [y if y is not None else xs[0].new_zeros(n, 2 * l + 1, m) for y, (m, l, _) in zip(outs, self.irreps_out)]


class RadialMLP(nn.Module):
    """nn.FullyConnectedNet(hs, silu) of e3nn (blocks.py:344-349): W/sqrt(fan_in), SiLU rescaled to unit second moment.
    The rescaling constant is folded into the next layer's weights, so every layer is one fused Linear+SiLU kernel."""

    def __init__(self, hs):
        super().__init__()
        self.hs = list(hs)
        for i, (a, b) in enumerate(zip(hs, hs[1:])):
            layer = nn.Module()
            layer.weight = nn.Parameter(torch.randn(a, b))
            self.add_module("layer%d" % i, layer)

    def forward_split(self, radial, down, plan, higher=False):
        """Same network on the input [radial | down[sender] | down[receiver]] without building it: the first layer is
        linear in the three blocks, so the two node blocks are multiplied per NODE and gathered per edge afterwards."""
        r, f = radial.shape[1], down.shape[1]
        w0 = self.layer0.weight / math.sqrt(self.hs[0])
        h = _lin(radial, w0[:r].t(), higher)
        h = h + ops.GatherRows.apply(_lin(down, w0[r:r + f].t(), higher), plan.by_row)
        h = h + ops.GatherRows.apply(_lin(down, w0[r + f:].t(), higher), plan.by_col)
        return self.forward(torch.nn.functional.silu(h), higher, first=1)

    def forward(self, x, higher=False, first=0):
        cst = e3.silu_second_moment_constant()
        nl = len(self.hs) - 1
        for i in range(first, nl):
            w = getattr(self, "layer%d" % i).weight
            scale = (cst if i > 0 else 1.0) / math.sqrt(self.hs[i])
            x = _lin(x, (w * scale).t(), higher, "silu" if i < nl - 1 else None)
        return x


class Interaction(nn.Module):
    """RealAgnosticAttResidualInteractionBlock (blocks.py:297-402)."""

    def __init__(self, channels, lmax_in, lmax_sh, lmax_hidden, num_radial, avg_num_neighbors):
        super().__init__()
        f = channels
        self.f, self.lmax_in, self.lmax_sh, self.avg = f, lmax_in, lmax_sh, avg_num_neighbors
        feats = e3.hidden_irreps(f, lmax_in)
        target = e3.hidden_irreps(f, lmax_sh)
        hidden = e3.hidden_irreps(f, lmax_hidden)
        self.paths = e3.tp_paths(lmax_in, lmax_sh, lmax_sh)
        self.linear_up = E3Linear(feats, feats)
        self.linear_down = E3Linear(feats, [(f, 0, 1)])
        self.conv_tp_weights = RadialMLP([num_radial + 2 * f] + 3 * [f] + [len(self.paths) * f])
        n_paths = [sum(1 for p in self.paths if p[2] == l) for l in range(lmax_sh + 1)]
        self.linear = E3Linear([(n_paths[l] * f, l, (-1) ** l) for l in range(lmax_sh + 1) if n_paths[l]], target)
        self.skip_linear = E3Linear(feats, hidden)
        # coupling constants c * C[m1, m2, m3] with c = sqrt(2 l3 + 1) (component normalisation, one path per output slot)
        for k, (l1, l2, l3) in enumerate(self.paths):
            self.register_buffer("_cg%d" % k, (e3.w3j(l1, l2, l3) * math.sqrt(2 * l3 + 1)).float(), persistent=False)

    def forward(self, xs, sh, radial, plan, higher=False):
        f = self.f
        sc = self.skip_linear(xs, higher)
        up = self.linear_up(xs, higher)
        down = self.linear_down(xs, higher)[0].reshape(-1, f)
        gather = ops.GatherRows.apply
        tpw = self.conv_tp_weights.forward_split(radial, down, plan, higher)         # [E, n_paths * F]
        e = tpw.shape[0]
        if not higher and ops.mace_tp_supported(self.lmax_in, self.lmax_sh, f):
            # fused: coupling, path weights and the scatter over receivers in one kernel; mji [E, F (L+1)^2] never exists
            packed = ops.MaceTpScatterFn.apply(torch.cat(up, dim=1), sh, tpw, plan, self.lmax_in, self.lmax_sh)
            n, msgs, off = up[0].shape[0], [], 0
            for l3 in range(self.lmax_sh + 1):
                n_p = sum(1 for p in self.paths if p[2] == l3)
                if n_p:
                    size = n * (2 * l3 + 1) * n_p * f
                    msgs.append(packed.narrow(0, off, size).view(n, 2 * l3 + 1, n_p * f))
                    off += size
            out = self.linear(msgs, higher)
            return [o / self.avg for o in out], sc
        # any-order / general-shape path: per-edge sender rows (GatherRows) and one closed TpOut primitive per path
        # (csrc/hgb_mace_any.cu) -- no einsum; every derivative of any order is again a libhgb kernel
        up_s = [gather(u.reshape(u.shape[0], -1), plan.by_row).reshape(e, u.shape[1], f) for u in up]
        per_l = [[] for _ in range(self.lmax_sh + 1)]
        for k, (l1, l2, l3) in enumerate(self.paths):
            y = sh[:, l2 * l2:(l2 + 1) ** 2]
            per_l[l3].append(ops.TpOut.apply(up_s[l1], y, tpw[:, k * f:(k + 1) * f], getattr(self, "_cg%d" % k)))   # [E, 2l3+1, F]
        msgs = []
        for l3, parts in enumerate(per_l):
            if parts:
                mji = torch.cat(parts, dim=2)                                         # [E, 2l3+1, n_p F]
                agg = ops.SegmentSum.apply(mji.reshape(e, -1), plan.by_col)
                msgs.append(agg.reshape(-1, 2 * l3 + 1, mji.shape[2]))
        out = self.linear(msgs, higher)
        return [o / self.avg for o in out], sc


ALPHABET = ["w", "x", "v", "n", "z", "r", "t", "y", "u", "o", "p", "s"]


class Contraction(nn.Module):
    """symmetric_contraction.py:92-242 for one output irrep; `x` is channel-last [N, S, F].  The reference draws
    example inputs for opt_einsum_fx from the global RNG before each weight (:150-158, :195-214); the same draws are
    made here so that seeded initialisation lines up."""

    def __init__(self, channels, lmax_in, l_out, correlation):
        super().__init__()
        self.f, self.l_out, self.correlation = channels, l_out, correlation
        for nu in range(1, correlation + 1):
            self.register_buffer("U_matrix_%d" % nu, e3.u_matrix(lmax_in, l_out, nu).to(torch.get_default_dtype()))
        self.weights = nn.ParameterList([])
        d_out = 2 * l_out + 1
        for i in range(correlation, 0, -1):
            u = getattr(self, "U_matrix_%d" % i)
            num_params, num_ell = u.shape[-1], u.shape[-2]
            shapes = [[d_out] + [num_ell] * i + [num_params], (NUM_ELEMENTS, num_params, channels)]
            if i == correlation:
                shapes += [(10, channels, num_ell), (10, NUM_ELEMENTS)]
            else:
                shapes += [(10, NUM_ELEMENTS), [10, channels, d_out] + [num_ell] * i, (10, channels, num_ell)]
            for shape in shapes:
                torch.randn(*shape)
            w = nn.Parameter(torch.randn(NUM_ELEMENTS, num_params, channels) / num_params)
            if i == correlation:
                self.weights_max = w
            else:
                self.weights.append(w)

    def forward(self, x, zcsr):
        c, e = self.correlation, min(self.l_out, 1)
        n, f = x.shape[0], self.f
        # weights picked by element, rows = (node, channel), columns = k:  [N F, K]  (closed GatherRows + a layout copy)
        pick = lambda w: ops.GatherRows.apply(w.reshape(NUM_ELEMENTS, -1), zcsr).reshape(n, w.shape[1], f).transpose(1, 2).reshape(n * f, -1)
        # symmetric_contraction.py:217-239 without einsum: every "U x weights" product is a closed MatMul, every contraction with
        # x a closed ChanCL step (csrc/hgb_mace_any.cu)
        u = getattr(self, "U_matrix_%d" % c)                                          # [lead..., i, k]
        ni, nk = u.shape[-2], u.shape[-1]
        t = ops.MatMul.apply(pick(self.weights_max), u.reshape(-1, nk), False, True)  # [N F, P i]
        out = ops.ChanCL.apply(t.reshape(n, f, -1, ni), x)                            # [N, F, P]
        for k, weight in enumerate(self.weights):
            i = c - k - 1
            u = getattr(self, "U_matrix_%d" % i)
            ct = ops.MatMul.apply(pick(weight), u.reshape(-1, u.shape[-1]), False, True).reshape(n, f, -1) + out
            out = ops.ChanCL.apply(ct.reshape(n, f, -1, ni), x)
        return out.reshape(n, f, -1).transpose(1, 2)                                  # [N, 2 l_out + 1, F]


class SymmetricContraction(nn.Module):
    def __init__(self, channels, lmax_in, lmax_out, correlation):
        super().__init__()
        self.contractions = nn.ModuleList([Contraction(channels, lmax_in, l, correlation) for l in range(lmax_out + 1)])

    def forward(self, x, zcsr):
        return [c(x, zcsr) for c in self.contractions]


class Product(nn.Module):
    """EquivariantProductBasisBlock (blocks.py:181-216)."""

    def __init__(self, channels, lmax_in, lmax_out, correlation):
        super().__init__()
        target = e3.hidden_irreps(channels, lmax_out)
        self.symmetric_contractions = SymmetricContraction(channels, lmax_in, lmax_out, correlation)
        self.linear = E3Linear(target, target)

    def forward(self, msgs, sc, zcsr, higher=False):
        x = torch.cat(msgs, dim=1)
        cons = self.symmetric_contractions.contractions
        lin, lout = int(round(math.sqrt(x.shape[1]))) - 1, len(cons) - 1
        if not higher and ops.mace_sc_supported(lin, lout, cons[0].correlation):
            wall = torch.cat([w for c in cons for w in (c.weights_max, c.weights[0])], dim=1)       # [118, KTOT, F]
            y = ops.MaceSymContractFn.apply(x, wall, zcsr, lin, lout)
            contracted = [y[:, l * l:(l + 1) ** 2, :] for l in range(lout + 1)]
        else:
            contracted = self.symmetric_contractions(x, zcsr)
        out = self.linear(contracted, higher)
        return [a + b for a, b in zip(out, sc)]


class MaceConv(nn.Module):
    """The PyG Sequential of MACEStack.get_conv (MACEStack.py:349-377): module_1 interaction, module_2 product,
    module_3 sizing Linear (module_0 / 4 / 5 are parameter-free combine / split glue)."""

    def __init__(self, inter, prod, sizing):
        super().__init__()
        self.module_1, self.module_2, self.module_3 = inter, prod, sizing

    def forward(self, xs, sh, radial, plan, zcsr, higher=False):
        msgs, sc = self.module_1(xs, sh, radial, plan, higher)
        return self.module_3(self.module_2(msgs, sc, zcsr, higher), higher)


class _NodeMLP(nn.Module):
    """LinearMLPNode / NonLinearMLPNode, node_type 'mlp' (blocks.py:824-960): an o3.Linear to scalars (only the 0e block
    of the input connects), then ordinary Linear layers."""

    def __init__(self, in_scalars, output_dim, hidden, act):
        super().__init__()
        first = E3Linear([(in_scalars, 0, 1)], [(output_dim if hidden is None else hidden[0], 0, 1)])
        layers = [first]
        if hidden is not None:
            layers.append(act)
            for a, b in zip(hidden[:-1], hidden[1:]):
                layers += [nn.Linear(a, b), act]
            layers.append(nn.Linear(hidden[-1], output_dim))
        self.mlp = nn.ModuleList([nn.Sequential(*layers)])

    def forward(self, x, higher=False):
        seq = self.mlp[0]
        h = seq[0]([x[:, None, :]], higher)[0][:, 0, :]
        if len(seq) == 1:
            return h
        h = seq[1](h)
        return run_mlp(nn.Sequential(*list(seq)[2:]), h, higher)


class MultiheadDecoder(nn.Module):
    """LinearMultiheadDecoderBlock (blocks.py:432-601) / NonLinearMultiheadDecoderBlock (:604-821): graph heads read
    the pooled scalar block, node heads start with an o3.Linear to scalars."""

    def __init__(self, nonlinear, in_scalars, config_heads, head_dims, head_type, act, graph_pooling, num_nodes=None):
        super().__init__()
        self.nonlinear, self.head_dims, self.head_type, self.graph_pooling = nonlinear, head_dims, head_type, graph_pooling
        self.graph_shared = nn.ModuleDict({})
        self.heads_NN = nn.ModuleList()
        if nonlinear and "graph" in config_heads:
            for br in config_heads["graph"]:
                a = br["architecture"]
                dim = a["dim_sharedlayers"]
                layers = [nn.Linear(in_scalars, dim), act]
                for _ in range(a["num_sharedlayers"] - 1):
                    layers += [nn.Linear(dim, dim), act]
                self.graph_shared[br["type"]] = nn.Sequential(*layers)
        for ih in range(len(head_dims)):
            head = nn.ModuleDict({})
            if head_type[ih] == "graph":
                for br in config_heads["graph"]:
                    a = br["architecture"]
                    if nonlinear:
                        dims = a["dim_headlayers"]
                        layers = [nn.Linear(a["dim_sharedlayers"], dims[0]), act]
                        for k in range(a["num_headlayers"] - 1):
                            layers += [nn.Linear(dims[k], dims[k + 1]), act]
                        layers.append(nn.Linear(dims[-1], head_dims[ih]))
                    else:
                        layers = [nn.Linear(in_scalars, head_dims[ih])]
                    head[br["type"]] = nn.Sequential(*layers)
            elif head_type[ih] == "node":
                for br in config_heads["node"]:
                    a = br["architecture"]
                    if a["type"] == "conv":
                        raise ValueError("Node-level convolutional layers are not supported in MACE")
                    if a["type"] != "mlp":
                        raise ValueError("b200 engine: MACE node heads of type %r are not supported (use 'mlp')" % (a["type"],))
                    assert num_nodes is not None, "num_nodes must be positive integer for MLP"          # blocks.py:499-502
                    head[br["type"]] = _NodeMLP(in_scalars, head_dims[ih], a["dim_headlayers"] if nonlinear else None, act)
            else:
                raise ValueError("Unknown head type" + str(head_type[ih]) + "; currently only support 'graph' or 'node'")
            self.heads_NN.append(head)

    def forward(self, scalars, pooled, batch, num_graphs, dataset_name, higher=False):
        ids = None if dataset_name is None else dataset_name[:, 0]
        outs = []
        for hd, head, kind in zip(self.head_dims, self.heads_NN, self.head_type):
            if kind == "graph":
                if len(head) == 1:
                    z = run_mlp(self.graph_shared["branch-0"], pooled, higher) if self.nonlinear else pooled
                    out = run_mlp(head["branch-0"], z, higher)[:, :hd]
                else:
                    out = pooled.new_zeros(num_graphs, hd)
                    for b in ids.unique():
                        m, key = ids == b, "branch-%d" % int(b)
                        z = run_mlp(self.graph_shared[key], pooled[m], higher) if self.nonlinear else pooled[m]
                        out[m] = run_mlp(head[key], z, higher)[:, :hd]
            else:
                if len(head) == 1:
                    out = head["branch-0"](scalars, higher)[:, :hd]
                else:
                    out = scalars.new_zeros(scalars.shape[0], hd)
                    for b in ids.unique():
                        m = (ids == b)[batch]
                        out[m] = head["branch-%d" % int(b)](scalars[m], higher)[:, :hd]
            outs.append(out)
        return outs


class MACEStack(nn.Module):
    """hydragnn/models/MACEStack.py:70-498 (no GPS wrapping, no graph-attr conditioning, no edge_attr)."""

    def __init__(self, r_max, radial_type, distance_transform, num_bessel, edge_dim, max_ell, node_max_ell, avg_num_neighbors,
                 num_polynomial_cutoff, correlation, input_dim, hidden_dim, output_dim, output_type, config_heads,
                 activation_function_type, loss_function_type, loss_weights=None, freeze_conv=False, initial_bias=None,
                 num_conv_layers=2, num_nodes=None, graph_pooling="mean", global_attn_engine=None):
        super().__init__()
        if global_attn_engine:
            raise ValueError("b200 engine: MACE inside GPS is not implemented")
        if edge_dim:
            raise ValueError("b200 engine: MACE with edge_attr is not implemented")
        if distance_transform in ("Agnesi", "Soft"):
            raise ValueError("b200 engine: MACE distance transforms need ase covalent radii and are not implemented")
        if max_ell > 3:
            raise ValueError("b200 engine: MACE max_ell <= 3")
        self.input_dim, self.hidden_dim, self.num_conv_layers, self.num_nodes = input_dim, hidden_dim, num_conv_layers, num_nodes
        self.max_ell, self.node_max_ell, self.avg_num_neighbors = max_ell, node_max_ell, avg_num_neighbors
        self.head_dims, self.head_type = list(output_dim), list(output_type)
        self.num_heads, self.config_heads = len(self.head_dims), config_heads
        self.activation_function = activation_function_selection(activation_function_type)
        self.var_output = 0
        if loss_function_type == "GaussianNLLLoss":
            raise ValueError("GaussianNLLLoss is not supported by the b200 engine")
        self.loss_function_type, self.loss_function = loss_function_type, loss_function_selection(loss_function_type)
        self.ilossweights_hyperp, self.ilossweights_nll = 1, 0
        loss_weights = list(loss_weights if loss_weights is not None else [1.0] * self.num_heads)
        if len(loss_weights) != self.num_heads:
            raise ValueError("Inconsistent number of loss weights and tasks: " + str(len(loss_weights)) + " VS " + str(self.num_heads))
        tot = sum(abs(w) for w in loss_weights)
        self.loss_weights = [w / tot for w in loss_weights]
        mode = graph_pooling.lower()
        mode = "add" if mode == "sum" else mode
        if mode not in ("mean", "add", "max"):
            raise ValueError("Unsupported graph_pooling: " + graph_pooling)
        self.graph_pooling = mode
        self.freeze_conv, self.initial_bias, self.force_higher_order = freeze_conv, initial_bias, False
        p_cut = 5 if num_polynomial_cutoff is None else num_polynomial_cutoff
        if correlation is None:
            self.correlation = [2] * num_conv_layers
        elif isinstance(correlation, int):
            self.correlation = [correlation] * num_conv_layers
        elif isinstance(correlation, (list, tuple)):
            self.correlation = list(correlation) * (num_conv_layers if len(correlation) == 1 else 1)
        else:
            raise TypeError("correlation must be int, list, tuple, or None")
        self.radial_type = "bessel" if radial_type is None else radial_type
        if self.radial_type not in ("bessel", "gaussian", "chebyshev"):
            raise ValueError("unknown radial_type " + str(radial_type))
        self.num_bessel, self.radius, self.p_cut = num_bessel, float(r_max), float(p_cut)
        # ---- decoders and convolutions interleaved, as MACEStack._init_conv creates them (:190-275)
        self.graph_convs, self.multihead_decoders = nn.ModuleList(), nn.ModuleList()
        f = hidden_dim
        last = num_conv_layers == 1
        self.multihead_decoders.append(self._decoder(last, NUM_ELEMENTS))
        self.graph_convs.append(self._get_conv(0, last))
        self.multihead_decoders.append(self._decoder(last, f))
        for i in range(num_conv_layers - 1):
            last = i == num_conv_layers - 2
            self.graph_convs.append(self._get_conv(node_max_ell, last))
            self.multihead_decoders.append(self._decoder(last, f))
        if freeze_conv:
            for p in self.graph_convs.parameters():
                p.requires_grad = False
        # ---- post-inheritance part of MACEStack.__init__ (:154-187)
        self.register_buffer("atomic_numbers", torch.arange(1, NUM_ELEMENTS + 1, dtype=torch.int64))
        self.register_buffer("r_max", torch.tensor(float(r_max)))
        self.register_buffer("num_interactions", torch.tensor(num_conv_layers, dtype=torch.int64))
        self.radial_embedding = nn.Module()
        self.radial_embedding.bessel_fn, self.radial_embedding.cutoff_fn = nn.Module(), nn.Module()
        bf = self.radial_embedding.bessel_fn
        if self.radial_type == "bessel":
            bf.register_buffer("bessel_weights", math.pi / r_max * torch.linspace(1.0, num_bessel, num_bessel))
            bf.register_buffer("r_max", torch.tensor(float(r_max)))
            bf.register_buffer("prefactor", torch.tensor(math.sqrt(2.0 / r_max)))
        elif self.radial_type == "gaussian":
            bf.register_buffer("gaussian_weights", torch.linspace(0.0, r_max, num_bessel))
        else:
            bf.register_buffer("n", torch.arange(1, num_bessel + 1, dtype=torch.get_default_dtype()).unsqueeze(0))
        self.radial_embedding.cutoff_fn.register_buffer("p", torch.tensor(float(p_cut)))
        self.radial_embedding.cutoff_fn.register_buffer("r_max", torch.tensor(float(r_max)))
        self.node_embedding = nn.Module()
        self.node_embedding.linear = E3Linear([(NUM_ELEMENTS, 0, 1)], [(f, 0, 1)])

    def _decoder(self, nonlinear, in_scalars):
        return MultiheadDecoder(nonlinear, in_scalars, self.config_heads, self.head_dims, self.head_type, self.activation_function,
                                self.graph_pooling, self.num_nodes)

    def _get_conv(self, lmax_in, last_layer):
        f = self.hidden_dim
        lmax_hidden = 0 if last_layer else self.node_max_ell
        inter = Interaction(f, lmax_in, self.max_ell, lmax_hidden, self.num_bessel, self.avg_num_neighbors)
        prod = Product(f, self.max_ell, lmax_hidden, self.correlation[0])
        hid = e3.hidden_irreps(f, lmax_hidden)
        return MaceConv(inter, prod, E3Linear(hid, hid))

    # ---- embeddings (ATen elementwise glue on [E]-sized vectors) ---------------------------------------------------------
    def _radial(self, d):
        """RadialEmbeddingBlock (blocks.py:164-177): basis(d) * polynomial cutoff(d), d [E, 1]."""
        p, rc = self.p_cut, self.radius
        x = d / rc
        env = 1.0 - ((p + 1.0) * (p + 2.0) / 2.0) * x.pow(p) + p * (p + 2.0) * x.pow(p + 1) - (p * (p + 1.0) / 2) * x.pow(p + 2)
        cutoff = env * (d < rc)
        bf = self.radial_embedding.bessel_fn
        if self.radial_type == "bessel":
            radial = bf.prefactor * (torch.sin(bf.bessel_weights * d) / d)
        elif self.radial_type == "gaussian":
            radial = torch.exp((-0.5 / (rc / (self.num_bessel - 1)) ** 2) * (d - bf.gaussian_weights).pow(2))
        else:
            radial = torch.special.chebyshev_polynomial_t(d.repeat(1, self.num_bessel), bf.n.repeat(len(d), 1))
        return radial * cutoff

    def _higher_order(self, data):
        pos = data.pos
        return bool(self.force_higher_order or (self.training and torch.is_grad_enabled() and pos is not None and pos.requires_grad))

    def forward(self, data):
        from .stacks import Base
        if data.x.dtype != torch.float32:
            raise RuntimeError("b200 engine kernels are fp32 (bf16 via autocast-style GEMMs); got " + str(data.x.dtype))
        assert data.pos is not None, "MACE requires node positions (data.pos) to be set."
        higher = self._higher_order(data)
        if getattr(self, "precision", "fp32") == "bf16" and not ops._TC["enabled"]:
            with ops.tensor_cores(True):
                return self.forward(data)
        plan = Base.plan_for(data)
        pos, batch = data.pos, data.batch
        n = pos.shape[0]
        if batch is None:
            batch = torch.zeros(n, dtype=torch.long, device=pos.device)
        num_graphs = data.__dict__.get("_num_graphs") if hasattr(data, "__dict__") else None
        if num_graphs is None:
            num_graphs = int(batch.max()) + 1
        gcsr = data.__dict__.get("_hgb_gcsr") if hasattr(data, "__dict__") else None
        if gcsr is None or gcsr.n != num_graphs or gcsr.idx.numel() != n:
            gcsr = ops.graph_ptr_from_batch(batch, num_graphs)
            try:
                data._hgb_gcsr = gcsr
            except Exception:
                pass
        # centre every graph (MACEStack.py:438-443); deterministic segmented mean + gather back
        cnt = (gcsr.rowptr[1:] - gcsr.rowptr[:-1]).clamp(min=1).to(pos.dtype)
        gsum = ops.SegmentSum.apply(pos, ops.Csr(gcsr.idx, gcsr.rowptr, None, gcsr.n))
        pos = pos - ops.GatherRows.apply(gsum / cnt[:, None], gcsr)
        shifts = getattr(data, "edge_shifts", None)
        if not higher and self.radial_type == "bessel" and EDGE_EMBED_KERNEL:
            # first-order path: geometry, spherical harmonics and Bessel x cutoff of every edge in ONE kernel (SURVEY K2)
            sh, radial = ops.MaceEdgeEmbedFn.apply(pos, shifts, plan, self.max_ell, self.num_bessel, self.radius, self.p_cut)
        else:
            vec = ops.GatherRows.apply(pos, plan.by_col) - ops.GatherRows.apply(pos, plan.by_row)
            if shifts is not None:
                vec = vec + shifts
            dist = vec.pow(2).sum(-1, keepdim=True).sqrt()
            sh = e3.spherical_harmonics_cl(self.max_ell, vec / dist.clamp(min=1e-12))
            radial = self._radial(dist)
        # node attributes (process_node_attributes, MACEStack.py:501-535): element index instead of a one-hot matrix
        z = data.x.squeeze()
        assert z.dim() == 1, "MACE only supports raw atomic numbers as node_attributes."
        z = (z.clamp(min=1, max=NUM_ELEMENTS) - 1).long()
        zcsr = data.__dict__.get("_hgb_zcsr") if hasattr(data, "__dict__") else None
        if zcsr is None or zcsr.idx.numel() != n:
            zcsr = ops.csr_build(z, NUM_ELEMENTS)
            try:
                data._hgb_zcsr = zcsr
            except Exception:
                pass
        emb = self.node_embedding.linear
        table = emb.weight.reshape(NUM_ELEMENTS, self.hidden_dim) * emb.alpha[0]      # one-hot @ W == row gather
        xs = [ops.GatherRows.apply(table, zcsr)[:, None, :]]
        ds = getattr(data, "dataset_name", None)
        onehot = torch.nn.functional.one_hot(z, NUM_ELEMENTS).to(pos.dtype)
        outputs = self.multihead_decoders[0](onehot, self._pool(onehot, gcsr, higher), batch, num_graphs, ds, higher)
        for conv, readout in zip(self.graph_convs, self.multihead_decoders[1:]):
            xs = conv(xs, sh, radial, plan, zcsr, higher)
            scalars = xs[0][:, 0, :]
            out = readout(scalars, self._pool(scalars, gcsr, higher), batch, num_graphs, ds, higher)
            outputs = [a + b for a, b in zip(outputs, out)]
        return outputs

    def _pool(self, x, gcsr, higher):
        if higher and self.graph_pooling != "max":
            out = ops.SegmentSum.apply(x, ops.Csr(gcsr.idx, gcsr.rowptr, None, gcsr.n))
            if self.graph_pooling == "mean":
                out = out / (gcsr.rowptr[1:] - gcsr.rowptr[:-1]).clamp(min=1).to(x.dtype)[:, None]
            return out
        return ops.PoolFn.apply(x.contiguous(), gcsr, self.graph_pooling)

    def loss(self, pred, value, head_index):
        """``loss_hpweighted`` (hydragnn/models/Base.py:879-906)."""
        tot_loss, tasks_loss = 0, []
        for ihead in range(self.num_heads):
            head_pre = pred[ihead]
            head_val = value[head_index[ihead]].reshape(head_pre.shape)
            li = self.loss_function(head_pre, head_val)
            tot_loss = tot_loss + li * self.loss_weights[ihead]
            tasks_loss.append(li)
        return tot_loss, tasks_loss

    def __str__(self):
        return "MACEStack"
