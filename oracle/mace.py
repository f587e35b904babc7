"""ORACLE (test infrastructure only): CPU restatement of the reference's MACE path.

Follows, line by line:
  MACEStack                         hydragnn/models/MACEStack.py:70-576
  RadialEmbeddingBlock & bases      hydragnn/utils/model/mace_utils/modules/blocks.py:141-177, radial.py:22-143
  RealAgnosticAttResidualInteractionBlock                blocks.py:297-402
  EquivariantProductBasisBlock      blocks.py:181-216
  SymmetricContraction/Contraction  mace_utils/modules/symmetric_contraction.py:29-242
  U_matrix_real / _wigner_nj        mace_utils/tools/cg.py:22-136
  tp_out_irreps_with_instructions, reshape_irreps        hydragnn/utils/model/irreps_tools.py:15-86
  Linear / NonLinear multihead decoders, LinearMLPNode, NonLinearMLPNode      blocks.py:432-960

Pinning: tests/golden/models_mace.pt was produced by running the reference's OWN files listed above with only e3nn replaced
(by oracle/e3.py), opt_einsum_fx by the identity and torch_scatter.scatter by index_add_ (tests/golden/make_golden.py);
this restatement reproduces those outputs, forces, parameter gradients, state-dict keys and seeded initial values.  What
stays unpinned is e3nn itself (oracle/e3.py, see its header), checked through properties (rotation / translation /
permutation invariance of the energy, equivariance of the forces, identities of the coupling tensors).
Edge attributes (MACEStack.py:198-203, 459-461) are pinned by tests/golden/models_mace_edge.pt and graph-attribute
conditioning (Base.py:97-106, 249-391; MACEStack.py:375-421) by tests/golden/models_mace_cond.pt, both made the same way
(tests/golden/make_mace_{edge,cond}_golden.py).
Distance transforms (Agnesi / Soft, radial.py:146-248) need ase.data.covalent_radii, which is not in this image:
they raise NotImplementedError.
"""
import math

import numpy as np
import torch
from torch import nn

from . import e3
from .base import activation, loss_function, normalize_heads
from .geometry import edge_vectors_and_lengths, graph_pool, segment_sum


# ---------------------------------------------------------------------------------------------------------------
# irreps tools (irreps_tools.py)
# ---------------------------------------------------------------------------------------------------------------
def tp_out_irreps_with_instructions(irreps1, irreps2, target_irreps):
    """irreps_tools.py:15-44."""
    out_list, instructions = [], []
    for i, (mul, ir_in) in enumerate(irreps1):
        for j, (_, ir_edge) in enumerate(irreps2):
            for ir_out in ir_in * ir_edge:
                if ir_out in target_irreps:
                    k = len(out_list)
                    out_list.append((mul, ir_out))
                    instructions.append((i, j, k, "uvu", True))
    irreps_out, permut, _ = e3.Irreps(out_list).sort()
    instructions = [(i1, i2, permut[io], mode, train) for i1, i2, io, mode, train in instructions]
    return irreps_out, sorted(instructions, key=lambda x: x[2])


def reshape_irreps(irreps, tensor):
    """irreps_tools.py:66-86: [N, sum mul*d] -> [N, mul, sum d] (all muls equal)."""
    out, ix = [], 0
    for mul, ir in irreps:
        out.append(tensor[:, ix:ix + mul * ir.dim].reshape(tensor.shape[0], mul, ir.dim))
        ix += mul * ir.dim
    return torch.cat(out, dim=-1)


# ---------------------------------------------------------------------------------------------------------------
# generalised Clebsch-Gordan (cg.py)
# ---------------------------------------------------------------------------------------------------------------
def _wigner_nj(irrepss, dtype):
    """cg.py:22-91 with normalization='component', filter_ir_mid=None.  Returns sorted [(ir, C)]."""
    irrepss = [e3.Irreps(x) for x in irrepss]
    if len(irrepss) == 1:
        (irreps,) = irrepss
        ret, eye, i = [], torch.eye(irreps.dim, dtype=dtype), 0
        for mul, ir in irreps:
            for _ in range(mul):
                ret.append((ir, eye[i:i + ir.dim]))
                i += ir.dim
        return ret
    *left, right = irrepss
    ret = []
    for ir_left, c_left in _wigner_nj(left, dtype):
        i = 0
        for mul, ir in right:
            for ir_out in ir_left * ir:
                c = e3.wigner_3j(ir_out.l, ir_left.l, ir.l, dtype=dtype) * ir_out.dim ** 0.5
                c = torch.einsum("jk,ijl->ikl", c_left.flatten(1), c)
                c = c.reshape(ir_out.dim, *(x.dim for x in left), ir.dim)
                for u in range(mul):
                    full = torch.zeros(ir_out.dim, *(x.dim for x in left), right.dim, dtype=dtype)
                    full[..., i + u * ir.dim:i + (u + 1) * ir.dim] = c
                    ret.append((ir_out, full))
            i += mul * ir.dim
    return sorted(ret, key=lambda x: x[0])          # stable: ties keep generation order


def u_matrix_real(irreps_in, irrep_out, correlation, dtype=torch.float64):
    """cg.py:94-136, last stacked tensor for `irrep_out`: [(2L+1)] + [dim_in]*correlation + [num_params], squeezed."""
    assert correlation <= 3, "oracle restates correlation <= 3 (correlation 4 adds a filter, cg.py:104-118)"
    irrep_out = e3.Irrep(irrep_out)
    stack = [c.squeeze().unsqueeze(-1) for ir, c in _wigner_nj([e3.Irreps(irreps_in)] * correlation, dtype) if ir == irrep_out]
    return torch.cat(stack, dim=-1)


# ---------------------------------------------------------------------------------------------------------------
# radial embedding
# ---------------------------------------------------------------------------------------------------------------
class RadialEmbedding(nn.Module):
    """blocks.py:141-177 with radial.py bases.  Buffers are named as in the reference."""

    def __init__(self, r_max, num_bessel, num_polynomial_cutoff, radial_type="bessel", distance_transform=None):
        super().__init__()
        if distance_transform in ("Agnesi", "Soft"):
            raise NotImplementedError("distance_transform needs ase.data.covalent_radii (not available here)")
        self.radial_type, self.num_basis, self.r_max_f = radial_type, num_bessel, float(r_max)
        self.bessel_fn, self.cutoff_fn = nn.Module(), nn.Module()
        if radial_type == "bessel":
            self.bessel_fn.register_buffer("bessel_weights", np.pi / r_max * torch.linspace(1.0, num_bessel, num_bessel))
            self.bessel_fn.register_buffer("r_max", torch.tensor(float(r_max)))
            self.bessel_fn.register_buffer("prefactor", torch.tensor(float(np.sqrt(2.0 / r_max))))
        elif radial_type == "gaussian":
            self.bessel_fn.register_buffer("gaussian_weights", torch.linspace(0.0, r_max, num_bessel))
            self.coeff = -0.5 / (r_max / (num_bessel - 1)) ** 2
        elif radial_type == "chebyshev":
            self.bessel_fn.register_buffer("n", torch.arange(1, num_bessel + 1, dtype=torch.get_default_dtype()).unsqueeze(0))
        else:
            raise ValueError("unknown radial_type " + str(radial_type))
        self.cutoff_fn.register_buffer("p", torch.tensor(float(num_polynomial_cutoff)))
        self.cutoff_fn.register_buffer("r_max", torch.tensor(float(r_max)))

    def forward(self, d):
        p, rc = self.cutoff_fn.p.to(d.dtype), self.cutoff_fn.r_max.to(d.dtype)
        env = (1.0 - ((p + 1.0) * (p + 2.0) / 2.0) * torch.pow(d / rc, p) + p * (p + 2.0) * torch.pow(d / rc, p + 1)
               - (p * (p + 1.0) / 2) * torch.pow(d / rc, p + 2))
        cutoff = env * (d < rc)
        if self.radial_type == "bessel":
            radial = self.bessel_fn.prefactor.to(d.dtype) * (torch.sin(self.bessel_fn.bessel_weights.to(d.dtype) * d) / d)
        elif self.radial_type == "gaussian":
            radial = torch.exp(self.coeff * torch.pow(d - self.bessel_fn.gaussian_weights.to(d.dtype), 2))
        else:
            radial = torch.special.chebyshev_polynomial_t(d.repeat(1, self.num_basis), self.bessel_fn.n.to(d.dtype).repeat(len(d), 1))
        return radial * cutoff


# ---------------------------------------------------------------------------------------------------------------
# interaction + product
# ---------------------------------------------------------------------------------------------------------------
class Interaction(nn.Module):
    """RealAgnosticAttResidualInteractionBlock (blocks.py:297-402).  Child order = creation order of the reference."""

    def __init__(self, node_feats_irreps, edge_attrs_irreps, edge_feats_irreps, target_irreps, hidden_irreps, avg_num_neighbors,
                 radial_mlp):
        super().__init__()
        self.target_irreps, self.avg_num_neighbors = target_irreps, avg_num_neighbors
        n_scalar = hidden_irreps.count("0e")
        down_irreps = e3.Irreps([(n_scalar, (0, 1))])
        self.linear_up = e3.Linear(node_feats_irreps, node_feats_irreps)
        irreps_mid, instructions = tp_out_irreps_with_instructions(node_feats_irreps, edge_attrs_irreps, target_irreps)
        self.conv_tp = e3.TensorProductUVU(node_feats_irreps, edge_attrs_irreps, irreps_mid, instructions)
        self.linear_down = e3.Linear(node_feats_irreps, down_irreps)
        input_dim = edge_feats_irreps.num_irreps + 2 * down_irreps.num_irreps
        self.conv_tp_weights = e3.FullyConnectedNet([input_dim] + 3 * [n_scalar] + [self.conv_tp.weight_numel],
                                                    torch.nn.functional.silu)
        self.linear = e3.Linear(irreps_mid.simplify(), target_irreps)
        self.skip_linear = e3.Linear(node_feats_irreps, hidden_irreps)
        del radial_mlp      # computed by the reference (MACEStack.py:277-281) but never read by this block (blocks.py:344-349)

    def forward(self, node_feats, edge_attrs, edge_feats, edge_index):
        sender, receiver = edge_index[0], edge_index[1]
        sc = self.skip_linear(node_feats)
        up = self.linear_up(node_feats)
        down = self.linear_down(node_feats)
        w = self.conv_tp_weights(torch.cat([edge_feats, down[sender], down[receiver]], dim=-1))
        mji = self.conv_tp(up[sender], edge_attrs, w)
        message = segment_sum(mji, receiver, node_feats.shape[0])
        message = self.linear(message) / self.avg_num_neighbors
        return reshape_irreps(self.target_irreps, message), sc


ALPHABET = ["w", "x", "v", "n", "z", "r", "t", "y", "u", "o", "p", "s"]


class Contraction(nn.Module):
    """symmetric_contraction.py:92-242.  The example inputs handed to opt_einsum_fx are drawn from the global RNG in the
    reference (:150-158, :195-214); the same draws are made here so that seeded initialisation stays aligned."""

    def __init__(self, irreps_in, irrep_out, correlation, num_elements):
        super().__init__()
        irrep_out = e3.Irrep(irrep_out)
        self.num_features = irreps_in.count("0e")
        coupling = e3.Irreps([ir for _, ir in irreps_in])
        self.correlation, self.lmax_out = correlation, irrep_out.l
        dtype = torch.get_default_dtype()
        for nu in range(1, correlation + 1):
            self.register_buffer("U_matrix_%d" % nu, u_matrix_real(coupling, irrep_out, nu, dtype=dtype))   # default dtype, as :107-116
        self.weights = nn.ParameterList([])
        num_equivariance = 2 * irrep_out.l + 1
        for i in range(correlation, 0, -1):
            u = getattr(self, "U_matrix_%d" % i)
            num_params, num_ell = u.shape[-1], u.shape[-2]
            if i == correlation:
                for shape in ([num_equivariance] + [num_ell] * i + [num_params], (num_elements, num_params, self.num_features),
                              (10, self.num_features, num_ell), (10, num_elements)):
                    torch.randn(*shape)
                self.weights_max = nn.Parameter(torch.randn(num_elements, num_params, self.num_features) / num_params)
            else:
                for shape in ([num_equivariance] + [num_ell] * i + [num_params], (num_elements, num_params, self.num_features),
                              (10, num_elements), [10, self.num_features, num_equivariance] + [num_ell] * i,
                              (10, self.num_features, num_ell)):
                    torch.randn(*shape)
                self.weights.append(nn.Parameter(torch.randn(num_elements, num_params, self.num_features) / num_params))

    def forward(self, x, y):
        """x [N, F, dim_in], y [N, num_elements] one-hot."""
        c, e = self.correlation, min(self.lmax_out, 1)
        lead = "".join(ALPHABET[:c + e - 1])
        out = torch.einsum(lead + "ik,ekc,bci,be->bc" + lead, getattr(self, "U_matrix_%d" % c).to(x.dtype), self.weights_max, x, y)
        for k, weight in enumerate(self.weights):
            i = c - k - 1
            lead_w = "".join(ALPHABET[:i + e])
            c_tensor = torch.einsum(lead_w + "k,ekc,be->bc" + lead_w, getattr(self, "U_matrix_%d" % i).to(x.dtype), weight, y)
            c_tensor = c_tensor + out
            lead_f = "".join(ALPHABET[:i - 1 + e])
            out = torch.einsum("bc" + lead_f + "i,bci->bc" + lead_f, c_tensor, x)
        return out.reshape(out.shape[0], -1)


class SymmetricContraction(nn.Module):
    def __init__(self, irreps_in, irreps_out, correlation, num_elements):
        super().__init__()
        self.contractions = nn.ModuleList([Contraction(irreps_in, ir, correlation, num_elements) for _, ir in irreps_out])

    def forward(self, x, y):
        return torch.cat([c(x, y) for c in self.contractions], dim=-1)


class Product(nn.Module):
    """EquivariantProductBasisBlock (blocks.py:181-216)."""

    def __init__(self, node_feats_irreps, target_irreps, correlation, num_elements, use_sc):
        super().__init__()
        self.use_sc = use_sc
        self.symmetric_contractions = SymmetricContraction(node_feats_irreps, target_irreps, correlation, num_elements)
        self.linear = e3.Linear(target_irreps, target_irreps)

    def forward(self, node_feats, sc, node_attrs):
        out = self.linear(self.symmetric_contractions(node_feats, node_attrs))
        return out + sc if (self.use_sc and sc is not None) else out


class _MaceConv(nn.Module):
    """The PyG Sequential of MACEStack.get_conv (MACEStack.py:349-377): module_1 = interaction, module_2 = product,
    module_3 = sizing linear (module_0 / 4 / 5 hold no parameters)."""

    def __init__(self, inter, prod, sizing, n_scalar_out):
        super().__init__()
        self.module_1, self.module_2, self.module_3 = inter, prod, sizing
        self.n_scalar_out = n_scalar_out

    def forward(self, inv, equiv, node_attrs, edge_attrs, edge_feats, edge_index):
        x = torch.cat([inv, equiv], dim=1)
        x, sc = self.module_1(x, edge_attrs, edge_feats, edge_index)
        x = self.module_2(x, sc, node_attrs)
        x = self.module_3(x)
        return x[:, :self.n_scalar_out], x[:, self.n_scalar_out:]


# ---------------------------------------------------------------------------------------------------------------
# decoders
# ---------------------------------------------------------------------------------------------------------------
class _MLPNodeIrreps(nn.Module):
    """LinearMLPNode / NonLinearMLPNode with node_type == 'mlp' (blocks.py:824-960)."""

    def __init__(self, input_irreps, output_dim, hidden, act):
        super().__init__()
        if hidden is None:
            layers = [e3.Linear(input_irreps, e3.create_irreps_string(output_dim, 0))]
        else:
            layers = [e3.Linear(input_irreps, e3.create_irreps_string(hidden[0], 0)), act]
            for a, b in zip(hidden[:-1], hidden[1:]):
                layers += [nn.Linear(a, b), act]
            layers.append(nn.Linear(hidden[-1], output_dim))
        self.mlp = nn.ModuleList([nn.Sequential(*layers)])

    def forward(self, x):
        return self.mlp[0](x)


class MultiheadDecoder(nn.Module):
    """LinearMultiheadDecoderBlock (blocks.py:432-601) / NonLinearMultiheadDecoderBlock (:604-821)."""

    def __init__(self, nonlinear, input_irreps, config_heads, head_dims, head_type, act, graph_pooling, num_nodes=None):
        super().__init__()
        self.nonlinear, self.head_dims, self.head_type, self.graph_pooling = nonlinear, head_dims, head_type, graph_pooling
        self.input_scalar_dim = input_irreps.count("0e")
        self.graph_shared = nn.ModuleDict({})
        self.heads_NN = nn.ModuleList()
        if nonlinear and "graph" in config_heads:
            for branch in config_heads["graph"]:
                arch = branch["architecture"]
                dim = arch["dim_sharedlayers"]
                layers = [nn.Linear(self.input_scalar_dim, dim), act]
                for _ in range(arch["num_sharedlayers"] - 1):
                    layers += [nn.Linear(dim, dim), act]
                self.graph_shared[branch["type"]] = nn.Sequential(*layers)
        for ih in range(len(head_dims)):
            head = nn.ModuleDict({})
            if head_type[ih] == "graph":
                for branch in config_heads["graph"]:
                    arch = branch["architecture"]
                    if nonlinear:
                        dims = arch["dim_headlayers"]
                        layers = [nn.Linear(arch["dim_sharedlayers"], dims[0]), act]
                        for k in range(arch["num_headlayers"] - 1):
                            layers += [nn.Linear(dims[k], dims[k + 1]), act]
                        layers.append(nn.Linear(dims[-1], head_dims[ih]))
                    else:
                        layers = [nn.Linear(self.input_scalar_dim, head_dims[ih])]
                    head[branch["type"]] = nn.Sequential(*layers)
            elif head_type[ih] == "node":
                for branch in config_heads["node"]:
                    arch = branch["architecture"]
                    if arch["type"] == "conv":
                        raise ValueError("Node-level convolutional layers are not supported in MACE")
                    if arch["type"] != "mlp":
                        raise ValueError("oracle restates node heads of type 'mlp' only, got " + arch["type"])
                    assert num_nodes is not None, "num_nodes must be positive integer for MLP"      # blocks.py:499-502
                    head[branch["type"]] = _MLPNodeIrreps(input_irreps, head_dims[ih], arch["dim_headlayers"] if nonlinear else None, act)
            else:
                raise ValueError("Unknown head type" + head_type[ih])
            self.heads_NN.append(head)

    def forward(self, node_features, batch, num_graphs, dataset_name=None):
        xg = graph_pool(node_features[:, :self.input_scalar_dim], batch, num_graphs, self.graph_pooling)
        ids = None if dataset_name is None else dataset_name[:, 0]
        outs = []
        for hd, head, kind in zip(self.head_dims, self.heads_NN, self.head_type):
            if kind == "graph":
                if len(head) == 1:
                    z = self.graph_shared["branch-0"](xg) if self.nonlinear else xg
                    out = head["branch-0"](z)[:, :hd]
                else:
                    out = xg.new_zeros(num_graphs, hd)
                    for b in ids.unique():
                        m, key = ids == b, "branch-%d" % int(b)
                        z = self.graph_shared[key](xg[m]) if self.nonlinear else xg[m]
                        out[m] = head[key](z)[:, :hd]
            else:
                if len(head) == 1:
                    out = head["branch-0"](node_features)[:, :hd]
                else:
                    out = node_features.new_zeros(node_features.shape[0], hd)
                    for b in ids.unique():
                        m = (ids == b)[batch]
                        out[m] = head["branch-%d" % int(b)](node_features[m])[:, :hd]
            outs.append(out)
        return outs


# ---------------------------------------------------------------------------------------------------------------
# the stack
# ---------------------------------------------------------------------------------------------------------------
class MACEOracle(nn.Module):
    """MACEStack (MACEStack.py:70-498) for use_global_attn = False.

    With ``edge_dim`` D > 0 the edge irreps are (D x 0e + sh).simplify() = (D+1)x0e + 1x1o + ... and every interaction reads
    cat([edge_attr, sh]): the "uvu" tensor product (oracle/e3.py) takes the multiplicity D+1 on its second input, with the path
    constant sqrt((2 l3 + 1) / (D+1)) on the 0e paths, and the radial MLP's last layer grows to the new weight_numel.

    With ``use_graph_attr_conditioning`` the invariant channels are conditioned on ``data.graph_attr`` after the embedding and
    after each convolution once that layer's readout has run.  The conditioning modules are created at the first forward (on
    the CPU generator), so they come after every other state-dict entry.  "fuse_pool" only checks graph_attr: MACEStack never
    pools with it.

    ``edge_dim``, ``use_graph_attr_conditioning`` and ``graph_attr_conditioning_mode`` come from the arguments or, where these
    are not given, from a subclass that set them before calling this constructor, as StackOracle's stacks set ``edge_dim``.
    """

    num_elements = 118

    def __init__(self, input_dim, hidden_dim, output_dim, output_type, output_heads, activation_function="relu",
                 loss_function_type="mse", task_weights=None, num_conv_layers=2, num_nodes=None, edge_dim=None, num_radial=None,
                 radius=None, radial_type=None, distance_transform=None, max_ell=None, node_max_ell=None, avg_num_neighbors=None,
                 envelope_exponent=None, correlation=None, graph_pooling="mean", global_attn_engine=None,
                 use_graph_attr_conditioning=False, graph_attr_conditioning_mode=None, **_unused):
        super().__init__()
        preset = vars(self)
        self.edge_dim = int(edge_dim or preset.get("edge_dim") or 0)
        self.use_graph_attr_conditioning = bool(use_graph_attr_conditioning or preset.get("use_graph_attr_conditioning"))
        mode = graph_attr_conditioning_mode or preset.get("graph_attr_conditioning_mode") or "concat_node"
        self.graph_attr_conditioning_mode = mode.lower()                             # Base.py:97-106
        if self.graph_attr_conditioning_mode not in ("film", "concat_node", "fuse_pool"):
            raise ValueError("graph_attr_conditioning_mode must be one of: 'film', 'concat_node', 'fuse_pool'.")
        assert radius is not None, "MACE requires radius input."
        assert num_radial is not None, "MACE requires num_radial input."
        assert max_ell is not None, "MACE requires max_ell input."
        assert node_max_ell is not None, "MACE requires node_max_ell input."
        assert max_ell >= 1, "MACE requires max_ell >= 1."
        assert node_max_ell >= 1, "MACE requires node_max_ell >= 1."
        if global_attn_engine:
            raise ValueError("oracle MACE: GPS wrapping is not restated")
        self.mpnn_type, self.hidden_dim, self.input_dim, self.num_nodes = "MACE", hidden_dim, input_dim, num_nodes
        self.max_ell, self.node_max_ell, self.avg_num_neighbors = max_ell, node_max_ell, avg_num_neighbors
        self.head_dims, self.head_type = list(output_dim), list(output_type)
        self.num_heads, self.num_conv_layers = len(self.head_dims), num_conv_layers
        pool = graph_pooling.lower()
        pool = "add" if pool == "sum" else pool
        if pool not in ("mean", "add", "max"):
            raise ValueError("Unsupported graph_pooling: " + graph_pooling)
        self.graph_pooling = pool
        p_cut = 5 if envelope_exponent is None else envelope_exponent
        if correlation is None:
            self.correlation = [2] * num_conv_layers
        elif isinstance(correlation, int):
            self.correlation = [correlation] * num_conv_layers
        elif isinstance(correlation, (list, tuple)):
            self.correlation = list(correlation) * (num_conv_layers if len(correlation) == 1 else 1)
        else:
            raise TypeError("correlation must be int, list, tuple, or None")
        radial_type = "bessel" if radial_type is None else radial_type
        self.activation_function = activation(activation_function)
        self.loss_function = loss_function(loss_function_type)
        weights = [1.0] * self.num_heads if task_weights is None else list(task_weights)
        if len(weights) != self.num_heads:
            raise ValueError("Inconsistent number of loss weights and tasks: %d VS %d" % (len(weights), self.num_heads))
        tot = sum(abs(w) for w in weights)
        self.loss_weights = [w / tot for w in weights]
        self.config_heads = normalize_heads(output_heads)

        self.edge_feats_irreps = e3.Irreps("%dx0e" % num_radial)
        self.node_attr_irreps = e3.Irreps([(self.num_elements, (0, 1))])
        self.sh_irreps = e3.Irreps.spherical_harmonics(max_ell)
        if self.edge_dim:                                                              # MACEStack.py:198-203
            self.edge_attrs_irreps = (e3.Irreps("%dx0e" % self.edge_dim) + self.sh_irreps).simplify()
        else:
            self.edge_attrs_irreps = self.sh_irreps
        # ---- Base.__init__ -> _init_conv (MACEStack.py:190-275): decoders and convolutions, interleaved
        self.graph_convs = nn.ModuleList()
        self.multihead_decoders = nn.ModuleList()
        hidden_irreps = e3.Irreps(e3.create_irreps_string(hidden_dim, node_max_ell))
        final_irreps = e3.Irreps(e3.create_irreps_string(hidden_dim, 0))
        last = num_conv_layers == 1
        self.multihead_decoders.append(self._decoder(last, self.node_attr_irreps))
        self.graph_convs.append(self._get_conv(hidden_dim, hidden_dim, first_layer=True, last_layer=last))
        self.multihead_decoders.append(self._decoder(last, final_irreps if last else hidden_irreps))
        for i in range(num_conv_layers - 1):
            last = i == num_conv_layers - 2
            self.graph_convs.append(self._get_conv(hidden_dim, hidden_dim, last_layer=last))
            self.multihead_decoders.append(self._decoder(last, final_irreps if last else hidden_irreps))
        # ---- post-inheritance (MACEStack.py:154-187)
        self.register_buffer("atomic_numbers", torch.arange(1, 119, dtype=torch.int64))
        self.register_buffer("r_max", torch.tensor(float(radius)))
        self.register_buffer("num_interactions", torch.tensor(num_conv_layers, dtype=torch.int64))
        self.radial_embedding = RadialEmbedding(radius, num_radial, p_cut, radial_type, distance_transform)
        self.node_embedding = nn.Module()
        self.node_embedding.linear = e3.Linear(self.node_attr_irreps, e3.create_irreps_string(hidden_dim, 0))
        self.graph_conditioner = self.graph_concat_projector = self.graph_concat_projector_in_dim = None
        self.device = torch.device("cpu")          # Base.py:66; read by load_existing_model

    def _decoder(self, nonlinear, irreps):
        return MultiheadDecoder(nonlinear, irreps, self.config_heads, self.head_dims, self.head_type, self.activation_function,
                                self.graph_pooling, self.num_nodes)

    def _get_conv(self, input_dim, output_dim, first_layer=False, last_layer=False):
        """MACEStack.py:277-377."""
        hidden_dim = output_dim if input_dim == 1 else input_dim
        mlp_dim = math.ceil(float(hidden_dim) / 3)
        node_feats_irreps = e3.Irreps(e3.create_irreps_string(input_dim, 0 if first_layer else self.node_max_ell))
        hidden_irreps = e3.Irreps(e3.create_irreps_string(hidden_dim, self.node_max_ell))
        interaction_irreps = (self.sh_irreps * hidden_dim).sort()[0].simplify()
        output_irreps = e3.Irreps(e3.create_irreps_string(output_dim, self.node_max_ell))
        if last_layer:
            hidden_irreps, output_irreps = hidden_irreps[:1], output_irreps[:1]
        inter = Interaction(node_feats_irreps, self.edge_attrs_irreps, self.edge_feats_irreps, interaction_irreps, hidden_irreps,
                            self.avg_num_neighbors, [mlp_dim] * 3)
        prod = Product(interaction_irreps, hidden_irreps, self.correlation[0], self.num_elements, use_sc=True)
        sizing = e3.Linear(hidden_irreps, output_irreps)
        return _MaceConv(inter, prod, sizing, output_irreps.count("0e"))

    def node_attributes(self, x):
        """process_node_attributes (MACEStack.py:501-535)."""
        z = x.squeeze()
        assert z.dim() == 1, "MACE only supports raw atomic numbers as node_attributes."
        if not torch.all((z >= 1) & (z <= self.num_elements)):
            z = torch.clamp(z, min=1, max=118)
        return torch.nn.functional.one_hot((z - 1).long(), num_classes=self.num_elements).float()

    def forward(self, data):
        pos, batch = data.pos, data.batch
        num_graphs = int(data.num_graphs)
        dtype = self.node_embedding.linear.weight.dtype
        mean_pos = segment_sum(pos, batch, num_graphs) / segment_sum(torch.ones_like(pos[:, :1]), batch, num_graphs).clamp(min=1)
        pos = pos - mean_pos[batch]
        shifts = getattr(data, "edge_shifts", None)
        vec, dist = edge_vectors_and_lengths(pos, data.edge_index, shifts)
        attrs = self.node_attributes(data.x).to(dtype)
        feats = self.node_embedding.linear(attrs)
        edge_attrs = e3.spherical_harmonics(self.max_ell, vec, normalize=True, normalization="component")
        if self.edge_dim:                                                              # MACEStack.py:459-461
            edge_attrs = torch.cat([data.edge_attr.to(edge_attrs.dtype), edge_attrs], dim=1)
        edge_feats = self.radial_embedding(dist)
        inv, equiv = feats[:, :self.hidden_dim], feats[:, self.hidden_dim:]
        inv = self.condition(inv, batch, data, num_graphs)
        ds = getattr(data, "dataset_name", None)
        outputs = self.multihead_decoders[0](attrs, batch, num_graphs, ds)
        for conv, readout in zip(self.graph_convs, self.multihead_decoders[1:]):
            inv, equiv = conv(inv, equiv, attrs, edge_attrs, edge_feats, data.edge_index)
            out = readout(torch.cat([inv, equiv], dim=1), batch, num_graphs, ds)
            inv = self.condition(inv, batch, data, num_graphs)
            outputs = [a + b for a, b in zip(outputs, out)]
        return outputs

    def _ensure_graph_conditioner(self, graph_attr_dim, device):
        """Base.py:249-259."""
        if self.graph_conditioner is None:
            hidden = max(self.hidden_dim, graph_attr_dim)
            self.graph_conditioner = nn.Sequential(nn.Linear(graph_attr_dim, hidden), self.activation_function,
                                                   nn.Linear(hidden, 2 * self.hidden_dim))
        self.graph_conditioner = self.graph_conditioner.to(device=device, dtype=self.node_embedding.linear.weight.dtype)

    def _ensure_graph_concat_projector(self, graph_attr_dim, channel_dim, device, dtype=None):
        """Base.py:261-276."""
        in_dim = channel_dim + graph_attr_dim
        if self.graph_concat_projector is None or self.graph_concat_projector_in_dim != in_dim:
            self.graph_concat_projector = nn.Linear(in_dim, channel_dim)
            self.graph_concat_projector_in_dim = in_dim
        self.graph_concat_projector = self.graph_concat_projector.to(device=device,
                                                                     dtype=dtype or self.node_embedding.linear.weight.dtype)

    def condition(self, inv, batch, data, num_graphs):
        """_apply_graph_conditioning (Base.py:299-391) on the invariant channels."""
        if not self.use_graph_attr_conditioning:
            return inv
        ga = getattr(data, "graph_attr", None)
        if ga is None:
            raise ValueError("use_graph_attr_conditioning=True but data.graph_attr is missing.")
        ga = ga.to(device=inv.device, dtype=inv.dtype)
        if ga.dim() == 1:
            if ga.numel() % num_graphs:
                raise ValueError(f"One-dimensional graph_attr with numel={ga.numel()} is not divisible by num_graphs={num_graphs}.")
            ga = ga.view(num_graphs, ga.numel() // num_graphs)
        elif ga.dim() == 2:
            if ga.size(0) != num_graphs:
                raise ValueError(f"graph_attr first dim {ga.size(0)} does not match num_graphs={num_graphs}.")
        else:
            raise ValueError(f"Unsupported graph_attr ndim={ga.dim()}; expected 1/2.")
        mode = self.graph_attr_conditioning_mode
        if mode == "film":
            self._ensure_graph_conditioner(ga.size(-1), inv.device)
            scale, shift = self.graph_conditioner(ga).split(self.hidden_dim, dim=-1)
            return inv * (1 + torch.tanh(scale)[batch]) + shift[batch]
        if mode == "concat_node":
            self._ensure_graph_concat_projector(ga.size(-1), inv.size(-1), inv.device, inv.dtype)
            return self.graph_concat_projector(torch.cat([inv, ga[batch]], dim=-1))
        return inv

    def loss(self, pred, value, head_index):
        tot, tasks = 0, []
        for ih in range(self.num_heads):
            tgt = value[head_index[ih]].reshape(pred[ih].shape)
            li = self.loss_function(pred[ih], tgt)
            tot = tot + li * self.loss_weights[ih]
            tasks.append(li)
        return tot, tasks

    def __str__(self):
        return "MACEStack"
