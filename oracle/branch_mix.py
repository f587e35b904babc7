"""Oracle: branch-weighted energies and forces of a multi-branch interatomic potential.  Test infrastructure only.

Restates examples/multidataset_hpo_sc26/inference_fused.py's path without encoder reuse: for every branch b, ``dataset_name``
:= b (``_build_dataset_name`` :408-416), one forward and -dE_b/dpos (``_predict_branch_energy_forces`` :429-451), then the
weighted average of energies and forces (``_weighted_average`` :547-563); and the single backward of the weighted energy
(``_fused_energy_forces`` :508-544, every branch live).  A node head's energies are summed per graph first, as
``energy_force_loss`` does (hydragnn/models/create.py:651-657).
"""
import torch

from .geometry import segment_sum


def _graph_energy(model, data, branch, num_graphs):
    data.dataset_name = torch.full((num_graphs, 1), branch, dtype=torch.long)
    pred = model(data)[0]
    if model.head_type[0] == "node":
        pred = segment_sum(pred, data.batch, num_graphs)
    return pred.squeeze(-1)


def per_branch(model, data, num_branches):
    """(energy [B, G], forces [B, N, 3]) of every branch on every graph (``_predict_branch_energy_forces``)."""
    g = int(data.batch.max()) + 1
    energies, forces = [], []
    for b in range(num_branches):
        e = _graph_energy(model, data, b, g)
        forces.append(-torch.autograd.grad(e, data.pos, grad_outputs=torch.ones_like(e))[0])
        energies.append(e.detach())
    return torch.stack(energies), torch.stack(forces)


def weighted_average(energies, forces, weights, batch):
    """``_weighted_average``: energies [B, G], forces [B, N, 3], weights [G, B] -> (energy [G], forces [N, 3])."""
    energy = torch.sum(weights * energies.transpose(0, 1), dim=1)
    counts = torch.bincount(batch)
    out = torch.zeros_like(forces[0])
    for b in range(energies.shape[0]):
        out = out + torch.repeat_interleave(weights[:, b], counts).unsqueeze(-1) * forces[b]
    return energy, out


def fused(model, data, weights):
    """``_fused_energy_forces`` with every branch live: sum_b w_b E_b, then one backward for the forces."""
    g = int(data.batch.max()) + 1
    energy = torch.zeros(g, dtype=data.pos.dtype)
    for b in range(weights.shape[1]):
        energy = energy + weights[:, b] * _graph_energy(model, data, b, g)
    forces = -torch.autograd.grad(energy, data.pos, grad_outputs=torch.ones_like(energy))[0]
    return energy.detach(), forces
