"""Generate tests/golden/models_mace_cond.pt by running the REFERENCE's own MACEStack with graph-attribute conditioning, on the
stubs make_mace_edge_golden.py uses (make_golden.install_stubs / install_mace_stubs).  Run where the reference checkout is
(record.REF); the tests never read it.

    python tests/golden/make_mace_cond_golden.py       # writes tests/golden/models_mace_cond.pt, nothing else

Cases: every mode ("film", "concat_node", "fuse_pool") with edge_dim 0 and 1, graph_attr given as [num_graphs, 2] and as the
flat [2 num_graphs] vector.  The conditioning modules are created at the first forward (hydragnn/models/Base.py:249-297), so a
case's state is the state dict after a seeded forward; the refusals are the reference's own exceptions.

What every case shares is stored once, to keep the file small:
* "batches" / "base_state": per edge_dim, the batch without graph_attr and the state dict without the conditioning modules
  (the seeded stack is the same for every mode and form);
* per case: graph_attr, the conditioning modules' entries ("cond_state", which the reference appends after every other entry
  of the state dict), the predictions, the
  position gradient of the objective, and parameter gradients: every one for FiLM with the [num_graphs, 2] form at edge_dim 0,
  otherwise those of the conditioning modules and of the radial MLPs that read the edge attributes (the flat form differs from
  the 2-D one only by a reshape, which the predictions and position gradients pin).
"""
import torch

import make_golden as mg
from record import HERE, refusal, save, t2d

COND = ("graph_conditioner.", "graph_concat_projector.")


def full_grads(edge_dim, mode, form):
    return edge_dim == 0 and form == "2d" and mode == "film"

MODES = ("film", "concat_node", "fuse_pool")
HEADS = {"graph": [{"type": "branch-0", "architecture": {"num_sharedlayers": 2, "dim_sharedlayers": 5, "num_headlayers": 2,
                                                          "dim_headlayers": [10, 6]}}],
         "node": [{"type": "branch-0", "architecture": {"num_headlayers": 2, "dim_headlayers": [12, 12], "type": "mlp"}}]}


def build(mace, edge_dim, mode, layers=2, hidden=8):
    torch.manual_seed(0)
    return mace.MACEStack("node_attributes, equiv_node_feat, inv_node_feat, edge_attributes, edge_features, edge_index",
                          "node_attributes, edge_attributes, edge_features, edge_index", 6.0, "bessel", None, 8, edge_dim,
                          2, 1, 10.0, 5, 2, 1, hidden, [1, 3], 0, "", "", 0, ["graph", "node"], HEADS,
                          "relu", "mae", None, loss_weights=[1.0, 1.0], freeze_conv=False, initial_bias=None,
                          num_conv_layers=layers, num_nodes=9, graph_pooling="mean", use_graph_attr_conditioning=True,
                          graph_attr_conditioning_mode=mode)


def main():
    mg.install_stubs()
    mace = mg.install_mace_stubs()
    gen = torch.Generator().manual_seed(515151)
    out = {"batches": {}, "base_state": {}, "cases": {}}
    for edge_dim in (0, 1):
        b = mg.toy_batch(gen, [7, 9, 5], 3.5, input_dim=1)
        if edge_dim:
            b.edge_attr = (b.pos[b.edge_index[1]] - b.pos[b.edge_index[0]]).norm(dim=1, keepdim=True)
        ga = torch.randn(3, 2, generator=gen)
        out["batches"][edge_dim] = t2d(b)
        for mode in MODES:
            for form in ("2d", "1d"):
                b.graph_attr = ga if form == "2d" else ga.reshape(-1)
                m = build(mace, edge_dim, mode)
                m.eval()
                inp = t2d(b)
                pos0 = b.pos.clone().requires_grad_(True)
                b.pos = pos0
                torch.manual_seed(1234)                     # the lazy modules draw from this state at the first forward
                pred = m(b)
                b.pos = inp["pos"]
                obj = pred[0].sum() + pred[1].pow(2).sum()
                forces = torch.autograd.grad(obj, pos0, retain_graph=True)[0]
                grads = torch.autograd.grad(obj, list(m.parameters()), allow_unused=True)
                state = m.state_dict()
                out["base_state"][edge_dim] = {k: v.clone() for k, v in state.items() if not k.startswith(COND)}
                cond_keys = [k for k in state if k.startswith(COND)]
                assert list(state) == list(out["base_state"][edge_dim]) + cond_keys
                keep = full_grads(edge_dim, mode, form)
                out["cases"]["%s_d%d_%s" % (mode, edge_dim, form)] = {
                    "graph_attr": inp["graph_attr"],
                    "cond_state": {k: v.clone() for k, v in state.items() if k.startswith(COND)},
                    "pred": [p.detach() for p in pred], "dobj_dpos": forces.detach(),
                    "grads": {n: (g.detach() if g is not None else None) for (n, _), g in zip(m.named_parameters(), grads)
                              if keep or n.startswith(COND) or "conv_tp_weights" in n},
                    "cfg": dict(edge_dim=edge_dim, use_graph_attr_conditioning=True, graph_attr_conditioning_mode=mode)}
    # refusals: a bad mode at construction, graph_attr missing / of the wrong size / of the wrong rank at the first forward
    b = mg.toy_batch(gen, [7, 9, 5], 3.5, input_dim=1)
    refusals = {"bad_mode": refusal(lambda: build(mace, 0, "sum"))}
    for name, ga in (("missing", None), ("1d_not_divisible", torch.randn(4)), ("2d_wrong_rows", torch.randn(2, 2)),
                     ("3d", torch.randn(3, 1, 2))):
        b.graph_attr = ga
        refusals[name] = refusal(lambda: build(mace, 0, "concat_node")(b), graph_attr=ga)
    out["refusals"] = refusals
    save(out, HERE + "/models_mace_cond.pt")


if __name__ == "__main__":
    main()
