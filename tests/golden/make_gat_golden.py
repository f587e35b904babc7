"""Generate tests/golden/models_gat.pt and tests/golden/dropin_gat.pt by running the REFERENCE's own GATStack.py + Base.py (and
gps.py for the GPS cases) on the stubs of make_golden.py.  Run in the build container only; the reference tree does not exist on
the GPU machines.

    python tests/golden/make_gat_golden.py      # writes models_gat.pt and dropin_gat.pt, nothing else

What the golden pins: everything in GATStack.py / Base.py / gps.py that runs -- GAT's own _init_conv (head-multiplied BatchNorm
widths, the two-conv quirk at num_conv_layers = 1, out_lin under GPS) and _init_node_conv, the GPS embedding and wrapper,
pooling, heads, losses -- EXCEPT PyG's ``GATv2Conv`` itself, which is the restatement in oracle/gat.py [3P-memory];
test_oracle_gat.py pins it by hand-computed cases.

Each case of models_gat.pt stores the seeded state dict as its names in order with one SHA-256 per entry (stack_support.state_digest;
the engine's own seeded construction reproduces the values, stack_support.seeded_state checks it), the inputs, the eval-mode
predictions, and one train-mode step (batch statistics, every dropout off, the attention dropout of the convs included):
predictions, the reference's own loss, every parameter gradient (the conv-head case: those of its head modules) and the BatchNorm
running statistics afterwards.  "errors" stores what the reference raises for a conv-type
node head on a model with edge features.  dropin_gat.pt stores what the reference's own ``create_model_config`` (with the
INTEGRATION.md dispatch) builds for GAT configurations after update_config (edge_dim None without edge features).
"""
import sys

import torch

import make_golden as mg
from record import (GPS, HEAD_GRAPH, HEAD_NODE, HERE, REF, dropin_config, add_edge_and_pe, pna_batch, record_case, record_dropin,
                    reference_create, refusal, save, targets)
from stack_support import state_digest

CONV_HEAD = {"node": [{"type": "branch-0", "architecture": {"num_headlayers": 2, "dim_headlayers": [20, 10], "type": "conv"}}]}

# name: (input_dim, hidden, layers, output_type, output_dim, edge_dim, edge attribute kind, pooling, gps, heads, graph sizes)
CASES = {
    "gat_graph_noedge": (3, 8, 3, ["graph"], [1], None, None, "mean", False, HEAD_GRAPH, [7, 5, 9, 6]),
    "gat_node_edge_len": (4, 5, 3, ["node"], [1], 1, "length", "mean", False, HEAD_NODE, [7, 5, 9, 6]),
    "gat_multihead": (5, 4, 2, ["graph", "node", "node"], [1, 1, 1], None, None, "mean", False, None, [7, 5, 9, 6]),
    "gat_add_pool_edge3": (2, 4, 2, ["graph"], [1], 3, "random", "add", False, HEAD_GRAPH, [7, 5, 9, 6]),
    "gat_one_layer": (3, 4, 1, ["graph"], [1], None, None, "mean", False, HEAD_GRAPH, [7, 5, 9, 6]),
    "gat_input_ne_hidden": (7, 3, 2, ["node"], [1], None, None, "mean", False, HEAD_NODE, [7, 5, 9, 6]),
    "gat_conv_head": (1, 20, 2, ["node"], [1], None, None, "mean", False, CONV_HEAD, [7, 5, 9, 6]),
    "gat_gps": (2, 8, 3, ["graph"], [1], None, None, "mean", True, HEAD_GRAPH, [7, 5, 9, 6]),
    "gat_gps_edge2": (2, 8, 2, ["graph"], [1], 2, "random", "mean", True, HEAD_GRAPH, [7, 5, 9, 6]),
    "gat_loops_dups_isolated": (3, 4, 2, ["node"], [1], 2, "random", "mean", False, HEAD_NODE, [7, 5, 9, 6]),
}


def install_gat_stubs():
    from oracle.gat import GATv2Conv
    from oracle.gps import PyGBatchNorm
    mg.install_stubs()
    tg = sys.modules["torch_geometric.nn"]
    tg.GATv2Conv, tg.BatchNorm = GATv2Conv, PyGBatchNorm
    sys.modules["hydragnn.models.Base"].BatchNorm = PyGBatchNorm
    mg.install_gps_stubs()
    return mg._load("hydragnn.models.GATStack", REF + "/hydragnn/models/GATStack.py")


def build(mod, input_dim, hidden, layers, otype, odim, edge_dim, pool, use_gps, heads, num_nodes=None):
    torch.manual_seed(0)
    return mod.GATStack("inv_node_feat, equiv_node_feat, edge_index", "inv_node_feat, edge_index", 6, 0.05, edge_dim,  # create.py:261-290
                        input_dim, hidden, odim, 4 if use_gps else 0, "GPS" if use_gps else None, "multihead" if use_gps else None,
                        4 if use_gps else 0, otype, heads, "relu", "mse", False, loss_weights=[1.0] * len(otype), freeze_conv=False,
                        initial_bias=None, num_conv_layers=layers, num_nodes=num_nodes, graph_pooling=pool)


def loops_dups_isolated(b):
    """An input self-loop on two nodes, a duplicate of the first edge, and node 6 of graph 0 left without any edge."""
    ei = b.edge_index
    ei = ei[:, (ei[0] != 6) & (ei[1] != 6)]
    extra = torch.tensor([[0, 9], [0, 9]]).long()
    b.edge_index = torch.cat([ei, extra, ei[:, :1]], dim=1)
    b.edge_shifts = torch.zeros(b.edge_index.shape[1], 3)
    return b


def make_models(mod):
    gen = torch.Generator().manual_seed(20261018)
    out = {}
    for name, (input_dim, hidden, layers, otype, odim, edge_dim, ekind, pool, use_gps, heads, sizes) in CASES.items():
        b = pna_batch(gen, sizes, input_dim)
        if name == "gat_loops_dups_isolated":
            b = loops_dups_isolated(b)
        add_edge_and_pe(b, gen, ekind, edge_dim, use_gps)
        if heads is None:
            heads = dict(HEAD_GRAPH, **HEAD_NODE)
        m = build(mod, input_dim, hidden, layers, otype, odim, edge_dim, pool, use_gps, heads)
        rec = record_case(m, b, *targets(b, otype, gen),
                          cfg=dict(input_dim=input_dim, hidden_dim=hidden, num_conv_layers=layers, output_type=otype, output_dim=odim,
                                   edge_dim=edge_dim, graph_pooling=pool, gps=use_gps, output_heads=heads))
        rec.update(state_sha256={k: state_digest(v) for k, v in rec["state"].items()}, grads_scope="all",
                   top_level=sorted(n for n, _ in m.named_children()))
        if name == "gat_conv_head":
            # the head modules are listed first under heads_NN (and again under convs_node_* / batch_norms_node_*)
            rec.update(grads_scope="conv_heads", grads={n: g for n, g in rec["grads"].items() if n.startswith("heads_NN.")})
            assert rec["grads"]
        out[name] = {k: rec[k] for k in ("state_sha256", "grads_scope", "inputs", "pred_eval", "pred_train", "value", "head_index",
                                         "loss", "str", "state_after", "grads", "top_level", "cfg")}
    # a conv-type node head on a model with edge features: the head convs are built with edge_dim=None and handed edge_attr
    gen = torch.Generator().manual_seed(7)
    b = pna_batch(gen, [5, 6], 1)
    b.edge_attr = torch.rand(b.edge_index.shape[1], 1, generator=gen)
    m = build(mod, 1, 4, 2, ["node"], [1], 1, "mean", False, CONV_HEAD)
    out["errors"] = {"conv_head_edge_attr": refusal(lambda: m(b))}
    return out


DROPIN_CASES = {"GAT-edge1-node": (1, "node", False), "GAT-noedge-graph": (None, "graph", False),
                "GAT-gps-noedge-graph": (None, "graph", True)}


def make_dropin():
    create_model_config, _ = reference_create()
    create_model_config.__globals__["GATStack"] = install_gat_stubs().GATStack
    out = {}
    for key, (edge_dim, otype, use_gps) in DROPIN_CASES.items():
        arch = dict(edge_dim=edge_dim, input_dim=1, hidden_dim=8, num_conv_layers=3, **(GPS if use_gps else {}))
        out[key] = record_dropin(create_model_config, dropin_config("GAT", otype, **arch))[0]
    return out


def main():
    save(make_models(install_gat_stubs()), HERE + "/models_gat.pt")
    save(make_dropin(), HERE + "/dropin_gat.pt")


if __name__ == "__main__":
    main()
