"""Golden vectors of the branch-weighted prediction of multi-branch interatomic potentials, recorded by running the REFERENCE's
own code (the checkout record.REF names); the tests never read it.

    python tests/golden/make_branch_mix_golden.py      # writes tests/golden/models_branch_mix.pt

Each case is one of make_multibranch_golden.py's 3-branch EGNN and PaiNN stacks (the reference's Base.py, EGCLStack.py /
PAINNStack.py, loaded with make_golden's stubs), in eval mode, with a graph energy head (add pooling) or an ``mlp`` node
energy head.  For every branch b, ``dataset_name`` := b for every graph, one forward and -dE_b/dpos, as
examples/multidataset_hpo_sc26/inference_fused.py's ``_predict_branch_energy_forces`` (:429-451) does (a node head's energies
summed per graph first, as ``energy_force_loss`` does).  Then the reference's own ``_weighted_average`` (:547-563) of those and
``_fused_energy_forces`` (:508-544) with every branch live, both AST-extracted from inference_fused.py, for fixed weights.
"""
import sys
import typing

import torch

import make_golden as mg
import make_multibranch_golden as mb
from record import HERE, REF, save, t2d


def main():
    egcl, painn = mg.install_stubs()
    scatter_add = sys.modules["torch_scatter"].scatter_add
    glb = {"torch": torch, "Tuple": typing.Tuple}
    mg._extract(REF + "/examples/multidataset_hpo_sc26/inference_fused.py", ["_weighted_average", "_fused_energy_forces"], glb)
    gen = torch.Generator().manual_seed(20261019)
    out = {}
    for stack in ("egnn", "painn"):
        for kind in ("graph", "node"):
            b = mg.toy_batch(gen, [6, 5, 8, 3, 7], 4.0, input_dim=1)
            g = int(b.batch.max()) + 1
            weights = torch.softmax(torch.randn(g, mb.BRANCHES, generator=gen), dim=-1)
            m = mb.build(egcl, painn, stack, kind)
            m.eval()
            state = {k: v.clone() for k, v in m.state_dict().items()}
            inp = t2d(b)
            b.pos.requires_grad_(True)

            def energy(branch):
                b.dataset_name = torch.full((g, 1), branch, dtype=torch.long)
                pred = m(b)[0]
                return pred.squeeze(-1) if kind == "graph" else scatter_add(pred, b.batch, dim=0).squeeze(-1)

            energies, forces, live = [], [], []
            for branch in range(mb.BRANCHES):
                e = energy(branch)
                forces.append(-torch.autograd.grad(e, b.pos, grad_outputs=torch.ones_like(e))[0])
                energies.append(e.detach())
                live.append(energy(branch))
            e_avg, f_avg = glb["_weighted_average"](torch.stack(energies), torch.stack(forces), weights, b.batch)
            e_fused, f_fused = glb["_fused_energy_forces"](live, [weights[:, k] for k in range(mb.BRANCHES)], [], [], b.pos, b.batch)
            out["%s_%s" % (stack, kind)] = {
                "state": state, "inputs": inp, "weights": weights,
                "branch_energy": torch.stack(energies, dim=1), "branch_forces": torch.stack(forces).detach(),
                "avg_energy": e_avg.detach(), "avg_forces": f_avg.detach(),
                "fused_energy": e_fused.detach(), "fused_forces": f_fused.detach(),
                "cfg": dict(mpnn_type="EGNN" if stack == "egnn" else "PAINN", input_dim=1, hidden_dim=16, num_conv_layers=2,
                            output_dim=[1], output_type=[kind], output_heads=mb.heads(kind), task_weights=[1.0],
                            activation_function="relu", loss_function_type="mse",
                            graph_pooling="add" if kind == "graph" else "mean", num_radial=5, radius=7.0)}
    save(out, HERE + "/models_branch_mix.pt")


if __name__ == "__main__":
    main()
