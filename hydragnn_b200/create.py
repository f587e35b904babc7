"""``create_model`` / ``create_model_config`` -- the ``mpnn_type`` plugin entry point of the engine.

Same keyword surface, error behaviour and return contract as ``hydragnn.models.create``
(hydragnn/models/create.py:41-161): ``torch.manual_seed(0)`` before construction (:164), unknown
``mpnn_type`` -> ``ValueError`` (:584), MLIP wrapping with ``energy_force_loss`` (:586-756), model moved to
the rank's device (:766).  INTEGRATION.md shows the three-line dispatch a maintainer adds to the reference.
"""
import os

import torch
from torch import nn

from . import ops
from .stacks import EGCLStack, PAINNStack, cached, graph_sum

SUPPORTED = ("EGNN", "PAINN", "PNA", "PNAPlus", "PNAEq", "MACE", "SchNet", "CGCNN", "GAT", "SAGE", "MFC")


def get_device(use_gpu=True):
    if use_gpu and torch.cuda.is_available():
        return torch.device("cuda", int(os.environ.get("LOCAL_RANK", "0")) % torch.cuda.device_count())
    return torch.device("cpu")


def update_multibranch_heads(output_heads):
    """Legacy single-branch dicts -> list-of-branches (hydragnn/utils/model/model.py:314-349)."""
    out = dict(output_heads)
    for name, val in output_heads.items():
        if isinstance(val, list):
            for br in val:
                if not (isinstance(br, dict) and "type" in br and "architecture" in br):
                    raise ValueError("output_heads['%s'] does not contain proper branch config, %s." % (name, val))
        elif isinstance(val, dict):
            out[name] = [{"type": "branch-0", "architecture": val}]
        else:
            raise ValueError("Unknown output_heads config!")
    return out


def create_model_config(config, verbosity=0, use_gpu=True):
    """``config`` is ``config["NeuralNetwork"]`` after ``update_config`` (hydragnn/models/create.py:41-108)."""
    arch, training = config["Architecture"], config["Training"]
    g = arch.get
    model = create_model(
        mpnn_type=arch["mpnn_type"], input_dim=arch["input_dim"], hidden_dim=arch["hidden_dim"],
        output_dim=arch["output_dim"], pe_dim=g("pe_dim", 0), global_attn_engine=g("global_attn_engine"),
        global_attn_type=g("global_attn_type"), global_attn_heads=g("global_attn_heads", 0),
        output_type=arch["output_type"], output_heads=arch["output_heads"],
        activation_function=g("activation_function", "relu"), loss_function_type=training.get("loss_function_type", "mse"),
        task_weights=arch["task_weights"], num_conv_layers=arch["num_conv_layers"],
        freeze_conv=g("freeze_conv_layers", False), initial_bias=g("initial_bias"), num_nodes=g("num_nodes"),
        max_neighbours=g("max_neighbours"), edge_dim=g("edge_dim"), pna_deg=g("pna_deg"), num_radial=g("num_radial"),
        num_gaussians=g("num_gaussians"), num_filters=g("num_filters"), envelope_exponent=g("envelope_exponent"),
        radial_type=g("radial_type"), distance_transform=g("distance_transform"), radius=g("radius"),
        equivariance=g("equivariance"), correlation=g("correlation"), max_ell=g("max_ell"), node_max_ell=g("node_max_ell"),
        avg_num_neighbors=g("avg_num_neighbors"), conv_checkpointing=training.get("conv_checkpointing", False),
        enable_interatomic_potential=g("enable_interatomic_potential", False), energy_weight=g("energy_weight", 0.0),
        energy_peratom_weight=g("energy_peratom_weight", 0.0), force_weight=g("force_weight", 0.0),
        use_graph_attr_conditioning=g("use_graph_attr_conditioning", False),
        graph_attr_conditioning_mode=g("graph_attr_conditioning_mode", "concat_node"),
        graph_pooling=g("graph_pooling", "mean"), verbosity=verbosity, use_gpu=use_gpu)
    prec = str(training.get("precision", "fp32")).lower()
    if prec in ("fp64", "float64", "double"):
        raise ValueError("the b200 engine computes in fp32 (bf16 tensor-core GEMMs under precision='bf16'); fp64 is not supported")
    return set_precision(model, "bf16" if prec in ("bf16", "bfloat16") else "fp32")


def set_precision(model, precision):
    """'fp32': exact fp32 kernels everywhere.  'bf16': the large-M Linear layers run on the wgmma tensor-core
    kernels (TF32 products, fp32 accumulation; parameters and activations stay fp32 like the reference's
    autocast mode, hydragnn/train/train_validate_test.py:43-49)."""
    if precision not in ("fp32", "bf16"):
        raise ValueError("Unsupported precision %s" % (precision,))
    model.precision = precision
    for m in model.modules():
        m.precision = precision
    return model


def create_model(mpnn_type, input_dim, hidden_dim, output_dim, pe_dim=0, global_attn_engine=None, global_attn_type=None,
                 global_attn_heads=0, output_type=None, output_heads=None, activation_function="relu",
                 loss_function_type="mse", task_weights=None, num_conv_layers=2, freeze_conv=False, initial_bias=None,
                 num_nodes=None, max_neighbours=None, edge_dim=None, pna_deg=None, num_before_skip=None, num_after_skip=None,
                 num_radial=None, radial_type=None, distance_transform=None, basis_emb_size=None, int_emb_size=None,
                 out_emb_size=None, envelope_exponent=None, num_spherical=None, num_gaussians=None, num_filters=None,
                 radius=None, equivariance=False, correlation=None, max_ell=None, node_max_ell=None, avg_num_neighbors=None,
                 conv_checkpointing=False, enable_interatomic_potential=False, energy_weight=0.0, energy_peratom_weight=0.0,
                 force_weight=0.0, use_graph_attr_conditioning=False, graph_attr_conditioning_mode="fuse_pool",
                 graph_pooling="mean", verbosity=0, use_gpu=True):
    torch.manual_seed(0)
    if global_attn_engine and (global_attn_engine != "GPS" or global_attn_type != "multihead"):
        raise ValueError("b200 engine: only global_attn_engine='GPS' with global_attn_type='multihead' is implemented")
    if use_graph_attr_conditioning and mpnn_type != "MACE":
        raise ValueError("b200 engine: graph_attr conditioning is not implemented yet")
    heads = update_multibranch_heads(output_heads)
    common = dict(input_dim=input_dim, hidden_dim=hidden_dim, output_dim=output_dim, output_type=output_type,
                  config_heads=heads, activation_function_type=activation_function, loss_function_type=loss_function_type,
                  equivariance=equivariance, loss_weights=task_weights, freeze_conv=freeze_conv, initial_bias=initial_bias,
                  num_conv_layers=num_conv_layers, num_nodes=num_nodes, graph_pooling=graph_pooling, pe_dim=pe_dim,
                  global_attn_engine=global_attn_engine, global_attn_type=global_attn_type, global_attn_heads=global_attn_heads)
    if mpnn_type == "EGNN":
        model = EGCLStack(edge_dim, max_neighbours=max_neighbours, **common)
    elif mpnn_type == "PAINN":
        model = PAINNStack(edge_dim, num_radial, radius, **common)
    elif mpnn_type == "PNA":
        assert pna_deg is not None, "PNA requires degree input."
        from .pna import PNAStack
        model = PNAStack(pna_deg, edge_dim, **common)
    elif mpnn_type == "PNAPlus":
        assert pna_deg is not None, "PNAPlus requires degree input."
        assert envelope_exponent is not None, "PNAPlus requires envelope_exponent input."
        assert num_radial is not None, "PNAPlus requires num_radial input."
        assert radius is not None, "PNAPlus requires radius input."
        from .pnaplus import PNAPlusStack
        model = PNAPlusStack(pna_deg, edge_dim, envelope_exponent, num_radial, radius, **common)
    elif mpnn_type == "PNAEq":
        assert pna_deg is not None, "PNAEq requires degree input."
        from .pnaeq import PNAEqStack
        model = PNAEqStack(pna_deg, edge_dim, num_radial, radius, **common)
    elif mpnn_type == "MACE":
        assert radius is not None, "MACE requires radius input."
        assert num_radial is not None, "MACE requires num_radial input."
        assert max_ell is not None, "MACE requires max_ell input."
        assert node_max_ell is not None, "MACE requires node_max_ell input."
        assert max_ell >= 1, "MACE requires max_ell >= 1."
        assert node_max_ell >= 1, "MACE requires node_max_ell >= 1."
        from .mace import MACEStack
        model = MACEStack(radius, radial_type, distance_transform, num_radial, edge_dim, max_ell, node_max_ell, avg_num_neighbors,
                          envelope_exponent, correlation, use_graph_attr_conditioning=use_graph_attr_conditioning,
                          graph_attr_conditioning_mode=graph_attr_conditioning_mode, **common)
    elif mpnn_type == "SchNet":
        assert num_gaussians is not None, "SchNet requires num_guassians input."
        assert num_filters is not None, "SchNet requires num_filters input."
        assert radius is not None, "SchNet requires radius input."
        from .schnet import SCFStack
        model = SCFStack(num_filters, edge_dim, num_gaussians, radius, max_neighbours=max_neighbours, **common)
    elif mpnn_type == "CGCNN":
        from .cgcnn import CGCNNStack
        model = CGCNNStack(edge_dim, **common)
    elif mpnn_type == "GAT":
        # hydragnn/models/create.py:261-264: the attention heads and the slope are fixed there, and so here
        heads = 6
        negative_slope = 0.05
        from .gat import GATStack
        model = GATStack(heads, negative_slope, edge_dim, **common)
    elif mpnn_type == "SAGE":
        # hydragnn/models/create.py:348-370 does not pass initial_bias to SAGEStack
        from .sage import SAGEStack
        model = SAGEStack(**dict(common, initial_bias=None))
    elif mpnn_type == "MFC":
        assert max_neighbours is not None, "MFC requires max_neighbours input."
        from .sage import MFCStack
        model = MFCStack(max_neighbours, **common)
    else:
        raise ValueError("Unknown mpnn_type: {0}".format(mpnn_type))
    if enable_interatomic_potential:
        model = EnhancedModelWrapper(model, energy_weight, energy_peratom_weight, force_weight)
    return model.to(get_device(use_gpu))


class EnhancedModelWrapper(nn.Module):
    """MLIP wrapper: E_graph = sum of node energies (or an add-pooled graph head); losses on E, E/atom and
    F = -dE/dpos (hydragnn/models/create.py:590-738)."""

    def __init__(self, original_model, energy_weight, energy_peratom_weight, force_weight):
        if getattr(original_model, "var_output", 0):
            # the reference's energy_force_loss reads pred[0] as the energy tensor, which a (outputs, outputs_var) pair is not
            raise ValueError("b200 engine: interatomic potentials have no mean-and-variance heads; GaussianNLLLoss is not supported")
        super().__init__()
        self.model = original_model
        self.energy_weight, self.energy_peratom_weight, self.force_weight = energy_weight, energy_peratom_weight, force_weight

    def __getattr__(self, name):
        try:
            return super().__getattr__(name)
        except AttributeError:
            return getattr(super().__getattr__("model"), name)

    def forward(self, data):
        return self.model(data)

    def energy_force_loss(self, pred, data, create_graph=True):
        assert data.pos is not None and data.energy is not None and data.forces is not None, \
            "data.pos, data.energy, data.forces must be provided for energy-force loss. Check your dataset creation and naming."
        assert data.pos.requires_grad, \
            "data.pos does not have grad, so force predictions cannot be computed. Check that data.pos has grad set to true before prediction."
        assert self.num_heads == 1, "Force predictions require exactly one head."
        lf = self.loss_function
        gcsr = self.graph_index(data)[2]
        if self.head_type[0] == "node":
            graph_energy_pred = graph_sum(pred[0], gcsr).squeeze().float()
        elif self.head_type[0] == "graph":
            if getattr(self.model, "graph_pooling", "mean") not in ["add"]:
                raise ValueError("Graph head force loss requires sum pooling (graph_pooling='add').")
            graph_energy_pred = pred[0].squeeze().float()
        else:
            raise ValueError("Force predictions are only supported for node or graph energy heads.")
        graph_energy_true = data.energy.squeeze().float()
        valid = cached(data, "_hgb_valid")
        if valid is not None:
            # capacity-padded batch (hydragnn_b200/padded.py): means run over the real graphs / atoms only; the counts live
            # on the device, nothing is read back
            gmask = (torch.arange(gcsr.n, device=valid.device) < valid[0]).to(graph_energy_pred.dtype)
            nmask = (torch.arange(data.pos.shape[0], device=valid.device) < valid[1]).to(graph_energy_pred.dtype)
            gcount = valid[0].to(graph_energy_pred.dtype).clamp(min=1)
            ncount = (valid[1].to(graph_energy_pred.dtype) * 3).clamp(min=1)
            energy_loss = lambda a, b: lf.masked_any_order(a, b, gmask, gcount)                      # noqa: E731
            force_loss_fn = lambda a, b: lf.masked_any_order(a, b, nmask[:, None], ncount)           # noqa: E731
        else:
            energy_loss = force_loss_fn = lambda a, b: lf(a, b, True)                                # noqa: E731
        tasks_loss = [energy_loss(graph_energy_pred, graph_energy_true)]
        ew, epw, fw = self.energy_weight, self.energy_peratom_weight, self.force_weight
        if ew <= 0 and epw <= 0 and fw <= 0:
            raise ValueError("All interatomic potential loss weights are zero; set at least one of energy_weight, "
                             "energy_peratom_weight, or force_weight to a positive value.")
        tot_loss = 0
        if ew > 0:
            tot_loss = tot_loss + tasks_loss[0] * ew
        natoms = (gcsr.rowptr[1:] - gcsr.rowptr[:-1]).to(graph_energy_pred.dtype)
        peratom = energy_loss(graph_energy_pred / natoms, graph_energy_true / natoms)
        tasks_loss.append(peratom)
        if epw > 0:
            tot_loss = tot_loss + peratom * epw
        with ops.only_data_grads():      # the force pass needs d/dpos only: fused blocks skip their parameter gradients
            forces_pred = -torch.autograd.grad(graph_energy_pred, data.pos, grad_outputs=torch.ones_like(graph_energy_pred),
                                               retain_graph=graph_energy_pred.requires_grad, create_graph=create_graph)[0].float()
        force_loss = force_loss_fn(forces_pred, data.forces.float())
        tasks_loss.append(force_loss)
        if fw > 0:
            tot_loss = tot_loss + force_loss * fw
        return tot_loss, tasks_loss
