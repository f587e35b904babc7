"""Generate tests/golden/models_mace_edge.pt by running the REFERENCE's own MACEStack with edge attributes (edge_dim > 0),
on the same stubs as make_golden.py (e3nn restated by oracle/e3.py, opt_einsum_fx the identity, torch_scatter.scatter
index_add_).  Run where the reference checkout is (record.REF); the tests never read it.

    python tests/golden/make_mace_edge_golden.py       # writes tests/golden/models_mace_edge.pt, nothing else

With edge_dim = D the reference's edge irreps are (Dx0e + sh).simplify() and the edge attributes cat([edge_attr, sh])
(MACEStack.py:198-203, 459-461).  edge_dim 1 takes the edge lengths, as the reference's own CI does
(tests/test_graphs.py: pytest_train_mace_model_lengths); edge_dim 3 takes random features.
"""
import torch

import make_golden as mg
from record import HERE, save, t2d

CONFIGS = {   # name: (edge_dim, max_ell, node_max_ell, correlation, num_conv_layers, hidden_dim)
    "mace_edge_d1_one_layer": (1, 2, 1, 2, 1, 8),
    "mace_edge_d3_l3": (3, 3, 2, 2, 2, 4),
}


def main():
    mg.install_stubs()
    mace = mg.install_mace_stubs()
    gen = torch.Generator().manual_seed(424242)
    heads = {"graph": [{"type": "branch-0", "architecture": {"num_sharedlayers": 2, "dim_sharedlayers": 5, "num_headlayers": 2,
                                                              "dim_headlayers": [10, 6]}}],
             "node": [{"type": "branch-0", "architecture": {"num_headlayers": 2, "dim_headlayers": [12, 12], "type": "mlp"}}]}
    out = {}
    for name, (edge_dim, max_ell, node_max_ell, corr, layers, hidden) in CONFIGS.items():
        b = mg.toy_batch(gen, [7, 9, 5], 3.5, input_dim=1)
        b.y = torch.randn(b.x.shape[0], 1, generator=gen)
        if edge_dim == 1:
            vec = b.pos[b.edge_index[1]] - b.pos[b.edge_index[0]]
            b.edge_attr = vec.norm(dim=1, keepdim=True)
        else:
            b.edge_attr = torch.randn(b.edge_index.shape[1], edge_dim, generator=gen)
        torch.manual_seed(0)
        m = mace.MACEStack("node_attributes, equiv_node_feat, inv_node_feat, edge_attributes, edge_features, edge_index",
                           "node_attributes, edge_attributes, edge_features, edge_index", 6.0, "bessel", None, 8, edge_dim,
                           max_ell, node_max_ell, 10.0, 5, corr, 1, hidden, [1, 3], 0, "", "", 0, ["graph", "node"], heads,
                           "relu", "mae", None, loss_weights=[1.0, 1.0], freeze_conv=False, initial_bias=None,
                           num_conv_layers=layers, num_nodes=9, graph_pooling="mean")
        m.eval()
        state = {k: v.clone() for k, v in m.state_dict().items()}
        inp = t2d(b)
        pos0 = b.pos.clone().requires_grad_(True)
        b.pos = pos0
        pred = m(b)
        obj = pred[0].sum() + pred[1].pow(2).sum()
        forces = torch.autograd.grad(obj, pos0, retain_graph=True)[0]
        grads = torch.autograd.grad(obj, list(m.parameters()), allow_unused=True)
        out[name] = {"state": state, "inputs": inp, "pred": [p.detach() for p in pred], "dobj_dpos": forces.detach(),
                     "grads": {n: (g.detach() if g is not None else None) for (n, _), g in zip(m.named_parameters(), grads)},
                     "cfg": dict(edge_dim=edge_dim, max_ell=max_ell, node_max_ell=node_max_ell, correlation=corr,
                                 num_conv_layers=layers, hidden_dim=hidden)}
    save(out, HERE + "/models_mace_edge.pt")


if __name__ == "__main__":
    main()
