"""Branch-weighted energies and forces of a multi-branch interatomic potential in one pass.

The reference evaluates such a potential with examples/multidataset_hpo_sc26/inference_fused.py: every dataset branch on every
structure, the branch energies mixed with per-graph weights (``weights = softmax(mlp(composition))``, :1215, the caller's
code here), forces as -dE/dpos.  Without encoder reuse it runs one full forward per branch (``_predict_branch_energy_forces``
:429-451), then ``_weighted_average`` (:547-563), or one fused backward (``_fused_energy_forces`` :508-544).  Here the encoder
runs once, every branch is decoded in one grouped launch per head layer (``stacks.all_branches``), the weighted sum is one
kernel (``ops.BranchMixFn``) and the forces one backward.

With E_gb the energy branch b predicts for graph g (``dataset_name`` := b) and w [G, B] the caller's weights:

    E_g = sum_b w_gb E_gb                   (ascending b, fp32)
    F_i = -d(sum_g E_g)/dpos_i              (one backward)
    branch_energy [G, B] = E_gb

In eval mode E_gb depends on the atoms of graph g only, so F_i = sum_b w_{g(i)b} F_{b,i}: the reference's ``_weighted_average``
of the per-branch forces, and ``_fused_energy_forces`` with every branch live.
"""
import torch

from . import ops
from .create import EnhancedModelWrapper
from .padded import PaddedBatch, _branches_grouped, supported
from .stacks import Base, all_branches, cached


def _inner(model):
    """The wrapped stack of an MLIP model in eval mode with one energy head that the all-branch decoding serves."""
    m = getattr(model, "module", model)
    if not isinstance(m, EnhancedModelWrapper):
        raise ValueError("branch-weighted prediction needs an interatomic potential (enable_interatomic_potential=True)")
    if m.training:
        raise ValueError("branch-weighted prediction runs in eval mode: call model.eval() first")
    inner = m.model
    if getattr(inner, "var_output", 0):
        raise ValueError("branch-weighted prediction does not take mean-and-variance heads")
    if inner.num_heads != 1 or inner.head_dims[0] != 1:
        raise ValueError("branch-weighted prediction needs one energy head of width 1")
    if inner.head_type[0] == "graph" and inner.graph_pooling != "add":
        raise ValueError("a graph energy head needs sum pooling (graph_pooling='add')")
    if getattr(inner, "num_branches", 1) > 1 and not _branches_grouped(inner):
        raise ValueError("branch-weighted prediction needs branches that share one architecture")
    return inner


def _num_graphs(data):
    g = cached(data, "_num_graphs")
    return int(g) if g is not None else int(data.batch.max()) + 1


def _check_weights(model, inner, data, weights):
    dev = next(model.parameters()).device
    g, b = _num_graphs(data), getattr(inner, "num_branches", 1)
    if not torch.is_tensor(weights) or weights.dtype != torch.float32 or tuple(weights.shape) != (g, b) or weights.device != dev:
        raise ValueError("weights must be a float32 [graphs, branches] = [%d, %d] tensor on %s, got %s" % (
            g, b, dev, "%s %s on %s" % (weights.dtype, tuple(weights.shape), weights.device) if torch.is_tensor(weights)
            else type(weights).__name__))
    if weights.requires_grad:
        raise ValueError("weights are data: they must not require grad (detach them)")


def _mix(model, inner, data, weights):
    """The body shared by the eager call and the captured step: one forward with every branch decoded, the mix and one
    force backward.  Returns detached (energy [G], forces [N, 3], branch_energy [G, B])."""
    if not data.pos.requires_grad:
        data.pos.requires_grad_(True)
    with torch.enable_grad():
        with all_branches():
            e = model(data)[0]
        gcsr = Base.graph_index(data)[2] if inner.head_type[0] == "node" else None
        energy, branch_energy = ops.branch_mix(e, weights, gcsr)
        with ops.only_data_grads():
            grad, = torch.autograd.grad(energy, data.pos, grad_outputs=torch.ones_like(energy))
    return energy.detach(), -grad, branch_energy


def branch_weighted_energy_forces(model, data, weights):
    """(energy [G], forces [N, 3], branch_energy [G, B]) of an interatomic potential with B dataset branches, every branch
    evaluated on every graph of ``data`` and mixed with the per-graph ``weights`` [G, B] (float32, on the model's device):
    energy_g = sum_b weights_gb branch_energy_gb and forces = -d(sum_g energy_g)/dpos.  Because each graph's energy depends on
    its own atoms only, the forces equal the weighted average of the per-branch forces (the reference's ``_weighted_average``)
    and the single fused backward of ``_fused_energy_forces``.

    One encoder pass, one all-branch decode, one mix kernel and one backward under ``ops.only_data_grads``; no parameter's
    ``.grad`` changes.  ``data.pos`` is marked as requiring grad, as the reference's loop does.  Refused: training mode, a
    model without the MLIP wrapper, mean-and-variance heads, more than one head, branches of differing architectures and
    weights of another shape, dtype or device."""
    inner = _inner(model)
    _check_weights(model, inner, data, weights)
    return _mix(model, inner, data, weights)


class PaddedPredictStep(PaddedBatch):
    """``branch_weighted_energy_forces`` captured as one CUDA graph that serves batches of every size: the capacities and
    filler graphs of ``PaddedGraphStep`` (the same staging, recapture and neighbour build), no loss and no optimizer.  Filler
    graphs get weight rows of zero.

        step = PaddedPredictStep(model, first_batch)
        step.load(batch, weights)
        energy, forces, branch_energy = step.run()

    ``run`` returns views of the real graphs and atoms in the step's own buffers: the next ``run`` overwrites them."""

    def __init__(self, model, first_batch, neighbour_build=None, node_cap=None, edge_cap=None, graph_cap=None, slack=1.12,
                 warmup=2):
        self.inner = _inner(model)
        if not supported(model):
            raise ValueError("PaddedPredictStep: this model (global attention / BatchNorm feature layers) needs the eager "
                             "branch_weighted_energy_forces")
        self.graph = None
        b = getattr(self.inner, "num_branches", 1)
        super().__init__(model, first_batch, neighbour_build, node_cap, edge_cap, graph_cap, slack, warmup, targets=False,
                         extra={"branch_weights": ((b,), torch.float32)})

    def load(self, batch, weights):
        """Pad ``batch`` and its weights [G, B] (float32) into the static buffers; returns the number of graphs."""
        b = self._widths["branch_weights"][0][0]
        g = int(batch.num_graphs)
        if not torch.is_tensor(weights) or weights.dtype != torch.float32 or tuple(weights.shape) != (g, b):
            raise ValueError("weights must be a float32 [graphs, branches] = [%d, %d] tensor" % (g, b))
        return super().load(batch, branch_weights=weights.detach())

    def _body(self):
        self._prologue()
        self.out = _mix(self.model, self.inner, self.data, self.data.branch_weights)

    def _do_capture(self):
        side = torch.cuda.Stream()
        side.wait_stream(torch.cuda.current_stream())
        with torch.cuda.stream(side):
            for _ in range(self.warmup):
                self._body()
        torch.cuda.current_stream().wait_stream(side)
        torch.cuda.synchronize()
        self.graph = torch.cuda.CUDAGraph()
        with ops.capture_graph(self.graph):
            self._body()
        self._captured = True

    def run(self):
        """(energy [g], forces [n, 3], branch_energy [g, B]) of the batch last loaded."""
        self.graph.replay()
        g, n = self.real
        energy, forces, branch_energy = self.out
        return energy[:g], forces[:n], branch_energy[:g]
