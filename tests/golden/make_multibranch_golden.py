"""Golden vectors of multi-branch interatomic potentials, recorded by running the REFERENCE's own code (the checkout record.REF
names); the tests never read it.

    python tests/golden/make_multibranch_golden.py      # writes tests/golden/models_multibranch.pt

Each case is an EGNN or PaiNN stack (the reference's Base.py, EGCLStack.py / PAINNStack.py, loaded with make_golden's stubs) with
three dataset branches per head, trained as make_golden.py records ``egnn_mlip``: the reference's own
``EnhancedModelWrapper.energy_force_loss`` (AST-extracted from hydragnn/models/create.py) with create_graph=True, then the
gradient of that loss for every parameter.  ``dataset_name`` sends the graphs of the batch to branches 0 and 2 only, so
branch 1 receives no graph and its gradients are exactly zero.

* ``egnn_graph`` / ``painn_graph``: one graph energy head, add pooling (the reference's force loss needs sum pooling);
* ``egnn_node`` / ``painn_node``: one ``mlp`` node energy head; the config carries three graph branches too, which is what makes
  Base count three branches (Base.py:599-601).
"""
import sys
import types

import torch

import make_golden as mg
from record import HERE, REF, save, t2d

GRAPH = {"num_sharedlayers": 2, "dim_sharedlayers": 6, "num_headlayers": 2, "dim_headlayers": [10, 7]}
NODE = {"num_headlayers": 2, "dim_headlayers": [12, 6], "type": "mlp"}
BRANCHES = 3


def heads(kind):
    hd = {"graph": [{"type": "branch-%d" % b, "architecture": dict(GRAPH)} for b in range(BRANCHES)]}
    if kind == "node":
        hd["node"] = [{"type": "branch-%d" % b, "architecture": dict(NODE)} for b in range(BRANCHES)]
    return hd


def build(egcl, painn, stack, kind):
    pool = "add" if kind == "graph" else "mean"
    torch.manual_seed(0)
    if stack == "egnn":
        return egcl.EGCLStack("inv_node_feat, equiv_node_feat, edge_index, edge_attr, edge_shifts", "", None,
                              1, 16, [1], 0, "", "", 0, [kind], heads(kind), "relu", "mse", False,
                              max_neighbours=None, loss_weights=[1.0], freeze_conv=False, initial_bias=None,
                              num_conv_layers=2, num_nodes=None, graph_pooling=pool)
    return painn.PAINNStack("inv_node_feat, equiv_node_feat, edge_index, diff, dist",
                            "inv_node_feat, equiv_node_feat, edge_index, diff, dist", None, 5, 7.0,
                            1, 16, [1], 0, "", "", 0, [kind], heads(kind), "relu", "mse", False,
                            loss_weights=[1.0], freeze_conv=False, num_conv_layers=2, num_nodes=None, graph_pooling=pool)


def main():
    egcl, painn = mg.install_stubs()
    glb = {"torch": torch, "torch_scatter": sys.modules["torch_scatter"]}
    mg._extract(REF + "/hydragnn/models/create.py", ["energy_force_loss"], glb)
    gen = torch.Generator().manual_seed(20261018)
    out = {}
    for stack in ("egnn", "painn"):
        for kind in ("graph", "node"):
            b = mg.toy_batch(gen, [6, 5, 8, 3, 7], 4.0, input_dim=1)
            b.dataset_name = torch.tensor([[2], [0], [2], [0], [0]])
            m = build(egcl, painn, stack, kind)
            m.train()
            state = {k: v.clone() for k, v in m.state_dict().items()}
            inp = t2d(b)
            b.pos.requires_grad_(True)
            pred = m(b)
            fake = types.SimpleNamespace(num_heads=1, head_type=[kind], model=m, loss_function=m.loss_function,
                                         energy_weight=1.0, energy_peratom_weight=1.0, force_weight=1.0)
            tot, tasks = glb["energy_force_loss"](fake, pred, b, create_graph=True)
            energy = pred[0].sum() if kind == "graph" else sys.modules["torch_scatter"].scatter_add(pred[0], b.batch, dim=0).sum()
            forces = -torch.autograd.grad(energy, b.pos, retain_graph=True)[0]
            grads = torch.autograd.grad(tot, list(m.parameters()), allow_unused=True)
            out["%s_%s" % (stack, kind)] = {
                "state": state, "inputs": inp, "pred": [p.detach() for p in pred], "loss": tot.detach(),
                "tasks": [t.detach() for t in tasks], "forces": forces.detach(),
                "grads": {n: (g.detach() if g is not None else None) for (n, _), g in zip(m.named_parameters(), grads)},
                "cfg": dict(mpnn_type="EGNN" if stack == "egnn" else "PAINN", input_dim=1, hidden_dim=16, num_conv_layers=2,
                            output_dim=[1], output_type=[kind], output_heads=heads(kind), task_weights=[1.0],
                            activation_function="relu", loss_function_type="mse",
                            graph_pooling="add" if kind == "graph" else "mean", num_radial=5, radius=7.0)}
    save(out, HERE + "/models_multibranch.pt")


if __name__ == "__main__":
    main()
