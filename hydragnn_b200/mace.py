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

Distance transforms (``distance_transform`` "Agnesi" / "Soft", radial.py:151-245): the radial basis reads T(d, r0) of the
covalent radii of the edge's two elements, the cutoff the raw d.  First order with Bessel radials: inside the fused edge
embedding (``ops.MaceEdgeEmbedDtFn``); otherwise ``ops.DistTransformFn`` (T, with T' and T'' as its closed derivatives).
"""
import math

import torch
from torch import nn

from . import e3, ops
from .covalent_radii import covalent_radii_tensor
from .stacks import (ELEMENT_CSR, Base, _linear_layers, apply_act, cached, decode_branches, decode_plan, graph_head_mlp,
                     graph_shared_mlp, graph_sum, grouped_decode, remember, run_mlp)

NUM_ELEMENTS = 118


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

    def __init__(self, channels, lmax_in, lmax_sh, lmax_hidden, num_radial, avg_num_neighbors, edge_dim=0):
        super().__init__()
        f = channels
        self.f, self.lmax_in, self.lmax_sh, self.avg, self.edge_dim = f, lmax_in, lmax_sh, avg_num_neighbors, edge_dim
        feats = e3.hidden_irreps(f, lmax_in)
        target = e3.hidden_irreps(f, lmax_sh)
        hidden = e3.hidden_irreps(f, lmax_hidden)
        self.paths = e3.tp_paths(lmax_in, lmax_sh, lmax_sh)
        # edge irreps (D+1)x0e + 1x1o + ... (MACEStack.py:198-203): a path whose edge irrep is 0e has a [F, D+1] weight block
        # (u-major) in tpw, every other path F weights; _wcol[k] = first tpw column of path k
        self._wcol, col = [], 0
        for (_, l2, _) in self.paths:
            self._wcol.append(col)
            col += f * (edge_dim + 1 if l2 == 0 else 1)
        self.linear_up = E3Linear(feats, feats)
        self.linear_down = E3Linear(feats, [(f, 0, 1)])
        self.conv_tp_weights = RadialMLP([num_radial + 2 * f] + 3 * [f] + [col])
        n_paths = [sum(1 for p in self.paths if p[2] == l) for l in range(lmax_sh + 1)]
        self.linear = E3Linear([(n_paths[l] * f, l, (-1) ** l) for l in range(lmax_sh + 1) if n_paths[l]], target)
        self.skip_linear = E3Linear(feats, hidden)
        # coupling constants c * C[m1, m2, m3] with c = sqrt(2 l3 + 1) (component normalisation, one path per output slot)
        for k, (l1, l2, l3) in enumerate(self.paths):
            self.register_buffer("_cg%d" % k, (e3.w3j(l1, l2, l3) * math.sqrt(2 * l3 + 1)).float(), persistent=False)

    def forward(self, xs, sh, radial, plan, higher=False, eattr=None):
        f, d = self.f, self.edge_dim
        sc = self.skip_linear(xs, higher)
        up = self.linear_up(xs, higher)
        down = self.linear_down(xs, higher)[0].reshape(-1, f)
        gather = ops.GatherRows.apply
        tpw = self.conv_tp_weights.forward_split(radial, down, plan, higher)         # [E, n_paths * F]
        e = tpw.shape[0]
        if not higher and ops.mace_tp_supported(self.lmax_in, self.lmax_sh, f, d):
            # fused: coupling, path weights (mixed with the edge attributes) and the scatter over receivers in one kernel;
            # mji [E, F (L+1)^2] never exists
            packed = ops.MaceTpScatterFn.apply(torch.cat(up, dim=1), sh, tpw, plan, self.lmax_in, self.lmax_sh, eattr)
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
            c0 = self._wcol[k]
            if l2 == 0 and d:
                # c = sqrt((2 l3 + 1) / (D + 1)): the 1/sqrt(D + 1) goes with the mixing, sqrt(2 l3 + 1) stays in _cg
                w = ops.EdgeMix.apply(tpw[:, c0:c0 + f * (d + 1)], eattr, 1.0 / math.sqrt(d + 1))
            else:
                w = tpw[:, c0:c0 + f]
            per_l[l3].append(ops.TpOut.apply(up_s[l1], y, w, getattr(self, "_cg%d" % k)))   # [E, 2l3+1, F]
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

    def forward(self, xs, sh, radial, plan, zcsr, higher=False, eattr=None):
        msgs, sc = self.module_1(xs, sh, radial, plan, higher, eattr)
        return self.module_3(self.module_2(msgs, sc, zcsr, higher), higher)


class _NodeMLP(nn.Module):
    """LinearMLPNode / NonLinearMLPNode, node_type 'mlp' (blocks.py:824-960): an o3.Linear to scalars (only the 0e block
    of the input connects), then ordinary Linear layers."""

    def __init__(self, in_scalars, output_dim, hidden, act):
        super().__init__()
        if isinstance(act, nn.PReLU):
            self.activation_function = act          # blocks.py: the decoders keep the shared slope under their own name too
        first = E3Linear([(in_scalars, 0, 1)], [(output_dim if hidden is None else hidden[0], 0, 1)])
        layers = [first]
        if hidden is not None:
            layers.append(act)
            for a, b in zip(hidden[:-1], hidden[1:]):
                layers += [nn.Linear(a, b), act]
            layers.append(nn.Linear(hidden[-1], output_dim))
        self.mlp = nn.ModuleList([nn.Sequential(*layers)])

    def grouped_layers(self):
        """The MLP as ``ops.grouped_mlp`` takes it: the o3.Linear on scalars is a Linear without bias whose weight is
        ``weight.reshape(mi, mo) * alpha``, transposed."""
        seq = self.mlp[0]
        e = seq[0]
        mi, mo = e.irreps_in[0][0], e.irreps_out[0][0]
        return [((e.weight.reshape(mi, mo) * e.alpha[0]).t(), None)] + _linear_layers(list(seq)[1:])

    def forward(self, x, higher=False):
        seq = self.mlp[0]
        h = seq[0]([x[:, None, :]], higher)[0][:, 0, :]
        if len(seq) == 1:
            return h
        h = apply_act(seq[1], h, higher)
        return run_mlp(nn.Sequential(*list(seq)[2:]), h, higher)


class MultiheadDecoder(nn.Module):
    """LinearMultiheadDecoderBlock (blocks.py:432-601) / NonLinearMultiheadDecoderBlock (:604-821): graph heads read
    the pooled scalar block, node heads start with an o3.Linear to scalars."""

    def __init__(self, nonlinear, in_scalars, config_heads, head_dims, head_type, act, graph_pooling, num_nodes=None):
        super().__init__()
        self.nonlinear, self.head_dims, self.head_type, self.graph_pooling = nonlinear, head_dims, head_type, graph_pooling
        if isinstance(act, nn.PReLU):
            self.activation_function = act
        self.graph_shared = nn.ModuleDict({})
        self.heads_NN = nn.ModuleList()
        if nonlinear and "graph" in config_heads:
            for br in config_heads["graph"]:
                self.graph_shared[br["type"]] = graph_shared_mlp(in_scalars, br["architecture"], act)
        for ih in range(len(head_dims)):
            head = nn.ModuleDict({})
            if head_type[ih] == "graph":
                for br in config_heads["graph"]:
                    head[br["type"]] = (graph_head_mlp(br["architecture"], head_dims[ih], act) if nonlinear
                                        else nn.Sequential(nn.Linear(in_scalars, head_dims[ih])))
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

    def forward(self, scalars, pooled, batch, num_graphs, branches, higher=False):
        """``branches``: the batch's ``BranchPlan`` (None with one branch)."""
        outs = []
        for hd, head, kind in zip(self.head_dims, self.heads_NN, self.head_type):
            if len(head) > 1:
                out = grouped_decode(kind, head, self.graph_shared, branches, scalars, pooled, hd, higher)
                if out is None:
                    out = decode_branches(kind, head, self.graph_shared, branches.ds[:, 0], scalars, pooled, batch, hd, num_graphs,
                                          higher)
                outs.append(out)
            elif kind == "graph":
                z = run_mlp(self.graph_shared["branch-0"], pooled, higher) if self.nonlinear else pooled
                outs.append(run_mlp(head["branch-0"], z, higher)[:, :hd])
            else:
                outs.append(head["branch-0"](scalars, higher)[:, :hd])
        return outs


CONDITIONING_MODES = ("film", "concat_node", "fuse_pool")


class MACEStack(Base):
    """hydragnn/models/MACEStack.py:70-498 (no GPS wrapping).  With edge_dim = D > 0 every convolution reads ``data.edge_attr``
    [E, D] as D extra 0e edge irreps in front of the spherical harmonics.

    Graph-attribute conditioning (``use_graph_attr_conditioning``; hydragnn/models/Base.py:97-106, 217-223, 249-391) changes the
    scalar block once after the embedding and after every convolution but the last, after that layer's readout -- the reference
    also conditions the last layer's output, which nothing reads.  Its modules (``graph_conditioner`` for "film",
    ``graph_concat_projector`` for "concat_node") are created at the first forward on the CPU generator and then moved, as the
    reference does; "fuse_pool" checks ``graph_attr`` and changes nothing, because MACEStack.forward never pools with it."""

    def __init__(self, r_max, radial_type, distance_transform, num_bessel, edge_dim, max_ell, node_max_ell, avg_num_neighbors,
                 num_polynomial_cutoff, correlation, *args, use_graph_attr_conditioning=False, graph_attr_conditioning_mode="fuse_pool",
                 **kwargs):
        # refused before Base.__init__, which would build the GPS embeddings first
        if kwargs.get("global_attn_engine"):
            raise ValueError("b200 engine: MACE inside GPS is not implemented")
        if max_ell > 3:
            raise ValueError("b200 engine: MACE max_ell <= 3")
        if kwargs.get("loss_function_type") == "GaussianNLLLoss":
            # the reference's MACE decoders keep their width and Base.loss then unpacks the output list as (pred, var)
            raise ValueError("b200 engine: MACE has no mean-and-variance heads; GaussianNLLLoss is not supported")
        # ---- prior to inheritance (:111-150): Base.__init__ calls _init_conv, which reads these
        num_conv_layers = kwargs["num_conv_layers"]
        self.edge_dim = int(edge_dim or 0)
        self.max_ell, self.node_max_ell, self.avg_num_neighbors = max_ell, node_max_ell, avg_num_neighbors
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
        self.use_graph_attr_conditioning = bool(use_graph_attr_conditioning)
        self.graph_attr_conditioning_mode = graph_attr_conditioning_mode.lower()
        if self.graph_attr_conditioning_mode not in CONDITIONING_MODES:
            raise ValueError("graph_attr_conditioning_mode must be one of: 'film', 'concat_node', 'fuse_pool'.")
        self.graph_conditioner = None
        self.graph_concat_projector = None
        self.graph_concat_projector_in_dim = None
        super().__init__(*args, **kwargs)
        # ---- post inheritance (:154-187)
        self.register_buffer("atomic_numbers", torch.arange(1, NUM_ELEMENTS + 1, dtype=torch.int64))
        self.register_buffer("r_max", torch.tensor(float(r_max)))
        self.register_buffer("num_interactions", torch.tensor(num_conv_layers, dtype=torch.int64))
        self.radial_embedding = nn.Module()
        self.radial_embedding.bessel_fn = nn.Module()
        bf = self.radial_embedding.bessel_fn
        if self.radial_type == "bessel":
            bf.register_buffer("bessel_weights", math.pi / r_max * torch.linspace(1.0, num_bessel, num_bessel))
            bf.register_buffer("r_max", torch.tensor(float(r_max)))
            bf.register_buffer("prefactor", torch.tensor(math.sqrt(2.0 / r_max)))
        elif self.radial_type == "gaussian":
            bf.register_buffer("gaussian_weights", torch.linspace(0.0, r_max, num_bessel))
        else:
            bf.register_buffer("n", torch.arange(1, num_bessel + 1, dtype=torch.get_default_dtype()).unsqueeze(0))
        # AgnesiTransform / SoftTransform (radial.py:151-245) for the exact strings only, registered between the basis and the
        # cutoff as RadialEmbeddingBlock does (blocks.py:154-159); any other value means no transform.  Buffers, never trained.
        self.distance_transform = distance_transform if distance_transform in ops.DIST_TRANSFORMS else None
        if self.distance_transform is not None:
            dt, fp = nn.Module(), torch.get_default_dtype()
            if self.distance_transform == "Agnesi":
                dt.register_buffer("q", torch.tensor(0.9183, dtype=fp))
                dt.register_buffer("p", torch.tensor(4.5791, dtype=fp))
                dt.register_buffer("a", torch.tensor(1.0805, dtype=fp))
                dt.register_buffer("covalent_radii", covalent_radii_tensor())
            else:
                dt.register_buffer("covalent_radii", covalent_radii_tensor())
                dt.register_buffer("a", torch.tensor(0.2))
                dt.register_buffer("b", torch.tensor(3.0))
            self.radial_embedding.distance_transform = dt
        self.radial_embedding.cutoff_fn = nn.Module()
        self.radial_embedding.cutoff_fn.register_buffer("p", torch.tensor(float(p_cut)))
        self.radial_embedding.cutoff_fn.register_buffer("r_max", torch.tensor(float(r_max)))
        self.node_embedding = nn.Module()
        self.node_embedding.linear = E3Linear([(NUM_ELEMENTS, 0, 1)], [(self.hidden_dim, 0, 1)])

    @property
    def device(self):
        """Where the parameters live: the device ``load_existing_model`` creates missing conditioning modules on."""
        return next(self.parameters()).device

    # ---- graph-attribute conditioning (Base.py:249-391) -------------------------------------------------------------------
    def _new_module_outside_capture(self):
        if torch.cuda.is_available() and torch.cuda.is_current_stream_capturing():
            raise RuntimeError("MACE graph-attribute conditioning creates its modules at the first forward; run one forward (or "
                               "load the checkpoint) before capturing a step")

    def _ensure_graph_conditioner(self, graph_attr_dim, device):
        """FiLM's ``Sequential(Linear(G, max(H, G)), act, Linear(max(H, G), 2H))``, created on the CPU, moved to ``device``."""
        if self.graph_conditioner is None:
            self._new_module_outside_capture()
            hidden = max(self.hidden_dim, graph_attr_dim)
            self.graph_conditioner = nn.Sequential(nn.Linear(graph_attr_dim, hidden), self.activation_function,
                                                   nn.Linear(hidden, 2 * self.hidden_dim))
        if self.graph_conditioner[0].weight.device != device:
            self.graph_conditioner = self.graph_conditioner.to(device)

    def _ensure_graph_concat_projector(self, graph_attr_dim, channel_dim, device, dtype=None):
        """concat_node's ``Linear(channel_dim + G, channel_dim)``, created on the CPU, moved to ``device`` / ``dtype``."""
        in_dim = channel_dim + graph_attr_dim
        if self.graph_concat_projector is None or self.graph_concat_projector_in_dim != in_dim:
            self._new_module_outside_capture()
            self.graph_concat_projector = nn.Linear(in_dim, channel_dim)
            self.graph_concat_projector_in_dim = in_dim
        w = self.graph_concat_projector.weight
        if w.device != device or (dtype is not None and w.dtype != dtype):
            self.graph_concat_projector = self.graph_concat_projector.to(device=device, dtype=dtype)

    def graph_attr_modules_missing(self):
        """True while a conditioned model has not created its conditioning modules (no forward, no checkpoint load yet)."""
        if not self.use_graph_attr_conditioning:
            return False
        mode = self.graph_attr_conditioning_mode
        return ((mode == "film" and self.graph_conditioner is None) or
                (mode == "concat_node" and self.graph_concat_projector is None))

    def _graph_attr(self, data, num_graphs, like):
        """``data.graph_attr`` as [num_graphs, G] with ``like``'s device and dtype; the reference's checks and messages."""
        ga = getattr(data, "graph_attr", None)
        if ga is None:
            raise ValueError("use_graph_attr_conditioning=True but data.graph_attr is missing.")
        ga = ga.to(device=like.device, dtype=like.dtype)
        if ga.dim() == 1:
            if ga.numel() % num_graphs == 0:
                return ga.view(num_graphs, ga.numel() // num_graphs)
            raise ValueError(f"One-dimensional graph_attr with numel={ga.numel()} is not divisible by num_graphs={num_graphs}.")
        if ga.dim() == 2:
            if ga.size(0) != num_graphs:
                raise ValueError(f"graph_attr first dim {ga.size(0)} does not match num_graphs={num_graphs}.")
            return ga
        raise ValueError(f"Unsupported graph_attr ndim={ga.dim()}; expected 1/2.")

    def _conditioning(self, ga, gcsr, higher):
        """The map h [N, H] -> conditioned h for this batch (None for fuse_pool); the per-graph terms are computed once."""
        mode, hd = self.graph_attr_conditioning_mode, self.hidden_dim
        gather = ops.GatherRows.apply
        if mode == "film":
            self._ensure_graph_conditioner(ga.shape[1], ga.device)
            st = run_mlp(self.graph_conditioner, ga, higher)                              # [B, 2H] = [s | t]
            if higher:
                scale = 1 + torch.tanh(gather(st[:, :hd].contiguous(), gcsr))
                shift = gather(st[:, hd:].contiguous(), gcsr)
                return lambda h: h * scale + shift
            return lambda h: ops.FilmFn.apply(h, st, gcsr)
        if mode == "concat_node":
            self._ensure_graph_concat_projector(graph_attr_dim=ga.shape[1], channel_dim=hd, device=ga.device, dtype=ga.dtype)
            proj = self.graph_concat_projector
            w_h, w_g = proj.weight[:, :hd], proj.weight[:, hd:]
            if higher:
                c = gather(ops.linear_any_order(ga, w_g, proj.bias), gcsr)
                return lambda h: ops.linear_any_order(h, w_h) + c
            c = ops.linear_act(ga, w_g.contiguous(), proj.bias)                           # [B, H] = graph_attr W_g^T + b
            return lambda h: ops.GraphAddLinearFn.apply(h, w_h, c, gcsr)
        return None

    def _init_conv(self):
        """Decoders and convolutions interleaved, in the order MACEStack._init_conv creates them (:190-275)."""
        self.multihead_decoders = nn.ModuleList([self._decoder(self.num_conv_layers == 1, NUM_ELEMENTS)])
        for i in range(self.num_conv_layers):
            last = i == self.num_conv_layers - 1
            self.graph_convs.append(self._get_conv(self.node_max_ell if i else 0, last))
            self.multihead_decoders.append(self._decoder(last, self.hidden_dim))

    def _multihead(self):
        """Nothing (:500): every decoder is one of ``multihead_decoders``."""
        self.num_branches = max(len(v) for v in self.config_heads.values())

    def _decoder(self, nonlinear, in_scalars):
        return MultiheadDecoder(nonlinear, in_scalars, self.config_heads, self.head_dims, self.head_type, self.activation_function,
                                self.graph_pooling, self.num_nodes)

    def _get_conv(self, lmax_in, last_layer):
        f = self.hidden_dim
        lmax_hidden = 0 if last_layer else self.node_max_ell
        inter = Interaction(f, lmax_in, self.max_ell, lmax_hidden, self.num_bessel, self.avg_num_neighbors, self.edge_dim)
        prod = Product(f, self.max_ell, lmax_hidden, self.correlation[0])
        hid = e3.hidden_irreps(f, lmax_hidden)
        return MaceConv(inter, prod, E3Linear(hid, hid))

    # ---- embeddings (ATen elementwise glue on [E]-sized vectors) ---------------------------------------------------------
    def _radial(self, d, t=None):
        """RadialEmbeddingBlock (blocks.py:164-177): basis(t) * polynomial cutoff(d), d [E, 1]; t is the transformed length
        (``DistTransformFn``) under a distance transform, else d itself."""
        p, rc = self.p_cut, self.radius
        x = d / rc
        env = 1.0 - ((p + 1.0) * (p + 2.0) / 2.0) * x.pow(p) + p * (p + 2.0) * x.pow(p + 1) - (p * (p + 1.0) / 2) * x.pow(p + 2)
        cutoff = env * (d < rc)
        d = d if t is None else t
        bf = self.radial_embedding.bessel_fn
        if self.radial_type == "bessel":
            radial = bf.prefactor * (torch.sin(bf.bessel_weights * d) / d)
        elif self.radial_type == "gaussian":
            radial = torch.exp((-0.5 / (rc / (self.num_bessel - 1)) ** 2) * (d - bf.gaussian_weights).pow(2))
        else:
            radial = torch.special.chebyshev_polynomial_t(d.repeat(1, self.num_bessel), bf.n.repeat(len(d), 1))
        return radial * cutoff

    def distance_transform_operands(self, z):
        """(kind, z, radii, c0, c1, c2) of ``ops.MaceEdgeEmbedDtFn`` / ``ops.DistTransformFn``: the element indices z [N] and the
        transform's buffers themselves, so the kernels read their current device values (after ``load_state_dict`` too)."""
        dt = self.radial_embedding.distance_transform
        if self.distance_transform == "Agnesi":
            return ops.DIST_TRANSFORMS["Agnesi"], z, dt.covalent_radii, dt.q, dt.p, dt.a
        return ops.DIST_TRANSFORMS["Soft"], z, dt.covalent_radii, dt.a, dt.b, None

    def _forward(self, data, higher):
        """MACEStack.forward (:375-421): a readout before the convolutions and after each, outputs summed."""
        assert data.pos is not None, "MACE requires node positions (data.pos) to be set."
        ga = None
        if self.use_graph_attr_conditioning:      # checked before any kernel; the graph count is kept for graph_index
            num_graphs = cached(data, "_num_graphs")
            if num_graphs is None:
                num_graphs = 1 if data.batch is None else int(data.batch.max()) + 1
                remember(data, "_num_graphs", num_graphs)
            ga = self._graph_attr(data, num_graphs, data.pos)
        plan = self.plan_for(data)
        batch, num_graphs, gcsr = self.graph_index(data)
        pos, n = data.pos, data.pos.shape[0]
        # centre every graph (MACEStack.py:438-443); deterministic segmented mean + gather back
        cnt = (gcsr.rowptr[1:] - gcsr.rowptr[:-1]).clamp(min=1).to(pos.dtype)
        pos = pos - ops.GatherRows.apply(graph_sum(pos, gcsr) / cnt[:, None], gcsr)
        shifts = getattr(data, "edge_shifts", None)
        eattr = self._edge_attr(data, plan.num_edges) if self.use_edge_attr else None
        # node attributes (process_node_attributes, MACEStack.py:501-535): element index instead of a one-hot matrix
        z = data.x.squeeze()
        assert z.dim() == 1, "MACE only supports raw atomic numbers as node_attributes."
        z = (z.clamp(min=1, max=NUM_ELEMENTS) - 1).long()
        dt = None if self.distance_transform is None else self.distance_transform_operands(z)
        if not higher and self.radial_type == "bessel":
            # first-order path: geometry, spherical harmonics and Bessel x cutoff of every edge in ONE kernel (SURVEY K2)
            if dt is None:
                sh, radial = ops.MaceEdgeEmbedFn.apply(pos, shifts, plan, self.max_ell, self.num_bessel, self.radius, self.p_cut)
            else:
                sh, radial = ops.MaceEdgeEmbedDtFn.apply(pos, shifts, plan, dt, self.max_ell, self.num_bessel, self.radius, self.p_cut)
        else:
            vec = ops.GatherRows.apply(pos, plan.by_col) - ops.GatherRows.apply(pos, plan.by_row)
            if shifts is not None:
                vec = vec + shifts
            dist = vec.pow(2).sum(-1, keepdim=True).sqrt()
            sh = e3.spherical_harmonics_cl(self.max_ell, vec / dist.clamp(min=1e-12))
            radial = self._radial(dist, None if dt is None else ops.DistTransformFn.apply(dist, plan, dt))
        zcsr = cached(data, ELEMENT_CSR)
        if zcsr is None or zcsr.idx.numel() != n:
            zcsr = remember(data, ELEMENT_CSR, ops.csr_build(z, NUM_ELEMENTS))
        emb = self.node_embedding.linear
        table = emb.weight.reshape(NUM_ELEMENTS, self.hidden_dim) * emb.alpha[0]      # one-hot @ W == row gather
        xs = [ops.GatherRows.apply(table, zcsr)[:, None, :]]
        cond = None if ga is None else self._conditioning(ga, gcsr, higher)
        if cond is not None:
            xs = [cond(xs[0].reshape(n, -1))[:, None, :]]
        ds = decode_plan(data, batch, num_graphs, self.num_branches)
        onehot = torch.nn.functional.one_hot(z, NUM_ELEMENTS).to(pos.dtype)
        outputs = self.multihead_decoders[0](onehot, self.pool(onehot, gcsr, higher), batch, num_graphs, ds, higher)
        for i, (conv, readout) in enumerate(zip(self.graph_convs, self.multihead_decoders[1:])):
            xs = conv(xs, sh, radial, plan, zcsr, higher, eattr)
            scalars = xs[0][:, 0, :]
            out = readout(scalars, self.pool(scalars, gcsr, higher), batch, num_graphs, ds, higher)
            outputs = [a + b for a, b in zip(outputs, out)]
            if cond is not None and i + 1 < len(self.graph_convs):     # the readout above saw the unconditioned scalars
                xs = [cond(xs[0].reshape(n, -1))[:, None, :]] + xs[1:]
        return outputs

    def _edge_attr(self, data, num_edges):
        """data.edge_attr as read by MACEStack.py:459-461.  Edge attributes are data, as every preprocessing produces them."""
        ea = getattr(data, "edge_attr", None)
        if ea is None:
            raise ValueError("MACE with edge_dim=%d needs data.edge_attr [E, %d]" % (self.edge_dim, self.edge_dim))
        if ea.dim() != 2 or tuple(ea.shape) != (num_edges, self.edge_dim) or ea.dtype != torch.float32:
            raise ValueError("MACE edge_attr must be a float32 [E, edge_dim] = [%d, %d] tensor, got %s %s"
                             % (num_edges, self.edge_dim, ea.dtype, tuple(ea.shape)))
        if ea.requires_grad:
            raise ValueError("MACE edge_attr must not require grad: edge attributes are data (detach them)")
        return ea.contiguous()

    def __str__(self):
        return "MACEStack"
