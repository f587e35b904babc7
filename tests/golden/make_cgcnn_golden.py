"""Generate tests/golden/models_cgcnn.pt and tests/golden/dropin_cgcnn.pt by running the REFERENCE's own CGCNNStack.py + Base.py
(and gps.py for the GPS cases) on the stubs of make_golden.py.  Run in the build container only; the reference tree does not exist
on the GPU machines.

    python tests/golden/make_cgcnn_golden.py      # writes models_cgcnn.pt and dropin_cgcnn.pt, nothing else

What the golden pins: everything in CGCNNStack.py / Base.py / gps.py that runs -- the layer loop with its BatchNorm feature
layers, the GPS embedding and wrapper, pooling, heads, losses, the conv-head refusals -- EXCEPT PyG's ``CGConv`` itself, which is
the restatement in oracle/cgcnn.py [3P-memory]; test_oracle_cgcnn.py pins it by hand-computed cases.

Each case of models_cgcnn.pt stores the state dict, the inputs, the eval-mode predictions, and one train-mode step (batch
statistics, dropout off): predictions, the reference's own loss, every parameter gradient and the BatchNorm running statistics
afterwards.  "errors" stores what the reference raises (type and message) when it builds a stack with conv-type node heads.
dropin_cgcnn.pt stores what the reference's own ``create_model_config`` (with the INTEGRATION.md dispatch) builds for CGCNN
configurations that already carry update_config's two CGCNN rules (hidden_dim = input_dim without GPS, edge_dim = 0 without
edge features).
"""
import sys

import torch

import make_golden as mg
from record import (GPS, HEAD_GRAPH, HEAD_NODE, HERE, REF, add_edge_and_pe, dropin_config, pna_batch, record_case, record_dropin,
                    reference_create, refusal, save, targets)

# defined here, not in record.py: the pickled goldens hold one "branch-0" string object per module that spells it
HEAD_PER_NODE = {"node": [{"type": "branch-0", "architecture": {"num_headlayers": 2, "dim_headlayers": [7, 4], "type": "mlp_per_node"}}]}

# name: (input_dim, hidden, layers, output_type, output_dim, edge_dim, edge attribute kind, pooling, gps, heads, graph sizes)
CASES = {
    "cgcnn_graph_edge0": (3, 3, 3, ["graph"], [1], 0, None, "mean", False, HEAD_GRAPH, [7, 5, 9, 6]),
    "cgcnn_node_edge_len": (4, 4, 3, ["node"], [1], 1, "length", "mean", False, HEAD_NODE, [7, 5, 9, 6]),
    "cgcnn_add_pool_edge3": (2, 2, 2, ["graph"], [1], 3, "random", "add", False, HEAD_GRAPH, [7, 5, 9, 6]),
    "cgcnn_multihead": (5, 5, 2, ["graph", "node", "node"], [1, 1, 1], 0, None, "mean", False, None, [7, 5, 9, 6]),
    "cgcnn_mlp_per_node": (3, 3, 2, ["node"], [1], 0, None, "mean", False, HEAD_PER_NODE, [6, 6, 6, 6]),
    "cgcnn_gps": (2, 16, 2, ["graph"], [1], 0, None, "mean", True, HEAD_GRAPH, [7, 5, 9, 6]),
    "cgcnn_gps_edge2": (2, 8, 2, ["graph"], [1], 2, "random", "mean", True, HEAD_GRAPH, [7, 5, 9, 6]),
    "cgcnn_ci_width1": (1, 1, 3, ["graph"], [1], 1, "length", "mean", False, HEAD_GRAPH, [7, 5, 9, 6]),
}

CONV_HEAD = {"num_headlayers": 2, "dim_headlayers": [6, 5], "type": "conv"}
# conv-type node heads: a branch whose own "type" is "conv" (the reference's ValueError), and the legacy single-branch form
# that update_multibranch_heads turns into "branch-0" (the reference fails reading num_headlayers from the branch)
ERROR_CASES = {
    "conv_branch": {"node": [dict(CONV_HEAD, architecture=CONV_HEAD)]},
    "conv_legacy": {"node": [{"type": "branch-0", "architecture": CONV_HEAD}]},
}


def install_cgcnn_stubs():
    from oracle.cgcnn import CGConv
    from oracle.gps import PyGBatchNorm
    mg.install_stubs()
    tg = sys.modules["torch_geometric.nn"]
    tg.CGConv, tg.BatchNorm = CGConv, PyGBatchNorm
    sys.modules["hydragnn.models.Base"].BatchNorm = PyGBatchNorm
    mg.install_gps_stubs()
    return mg._load("hydragnn.models.CGCNNStack", REF + "/hydragnn/models/CGCNNStack.py")


def build(mod, input_dim, hidden, layers, otype, odim, edge_dim, pool, use_gps, heads, num_nodes=None):
    torch.manual_seed(0)
    return mod.CGCNNStack("inv_node_feat, equiv_node_feat, edge_index", "inv_node_feat, edge_index", edge_dim,   # create.py:321-324
                          input_dim, hidden, odim, 4 if use_gps else 0, "GPS" if use_gps else None, "multihead" if use_gps else None,
                          4 if use_gps else 0, otype, heads, "relu", "mse", False, loss_weights=[1.0] * len(otype), freeze_conv=False,
                          initial_bias=None, num_conv_layers=layers, num_nodes=num_nodes, graph_pooling=pool)


def make_models(mod):
    gen = torch.Generator().manual_seed(20261017)
    out = {}
    for name, (input_dim, hidden, layers, otype, odim, edge_dim, ekind, pool, use_gps, heads, sizes) in CASES.items():
        b = add_edge_and_pe(pna_batch(gen, sizes, input_dim), gen, ekind, edge_dim, use_gps)
        if heads is None:
            heads = dict(HEAD_GRAPH, **HEAD_NODE)
        num_nodes = sizes[0] if heads is HEAD_PER_NODE else None
        m = build(mod, input_dim, hidden, layers, otype, odim, edge_dim, pool, use_gps, heads, num_nodes)
        out[name] = record_case(m, b, *targets(b, otype, gen),
                                cfg=dict(input_dim=input_dim, hidden_dim=hidden, num_conv_layers=layers, output_type=otype,
                                         output_dim=odim, edge_dim=edge_dim, graph_pooling=pool, gps=use_gps, output_heads=heads,
                                         num_nodes=num_nodes))
    out["errors"] = {name: refusal(lambda: build(mod, 3, 3, 2, ["node"], [1], 0, "mean", False, heads), heads=heads)
                     for name, heads in ERROR_CASES.items()}
    return out


DROPIN_CASES = {"CGCNN-edge1-node": (1, "node", False), "CGCNN-edge0-graph": (0, "graph", False),
                "CGCNN-gps-edge0-graph": (0, "graph", True)}


def make_dropin():
    create_model_config, _ = reference_create()
    create_model_config.__globals__["CGCNNStack"] = install_cgcnn_stubs().CGCNNStack
    out = {}
    for key, (edge_dim, otype, use_gps) in DROPIN_CASES.items():
        arch = dict(edge_dim=edge_dim, input_dim=1, hidden_dim=1, num_conv_layers=3)
        if use_gps:
            arch.update(GPS, hidden_dim=8)
        out[key] = record_dropin(create_model_config, dropin_config("CGCNN", otype, **arch))[0]
    return out


def main():
    save(make_models(install_cgcnn_stubs()), HERE + "/models_cgcnn.pt")
    save(make_dropin(), HERE + "/dropin_cgcnn.pt")


if __name__ == "__main__":
    main()
