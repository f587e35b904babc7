"""Generate tests/golden/models_pna.pt and tests/golden/dropin_pna.pt by running the REFERENCE's own PNAStack.py + Base.py
(and gps.py for the GPS case) on the stubs of make_golden.py.  Run in the build container only; the reference tree does not
exist on the GPU machines.

    python tests/golden/make_pna_golden.py      # writes models_pna.pt and dropin_pna.pt, nothing else

What the golden pins: everything in PNAStack.py / Base.py / gps.py that runs -- the layer loop with its BatchNorm feature
layers, the GPS embedding and wrapper, pooling, heads, losses -- EXCEPT PyG's ``PNAConv`` itself.  That class is third-party
and absent here, so the generator uses the restatement in oracle/pna.py [3P-memory]; test_oracle_pna.py pins it by
hand-computed cases instead.  PyG's ``BatchNorm`` is ``PyGBatchNorm`` (a module holding ``.module = BatchNorm1d``), as in
make_golden.py.

Each case of models_pna.pt stores the state dict, the inputs, the eval-mode predictions, and one train-mode step (batch
statistics, dropout off): predictions, the reference's own loss, every parameter gradient and the BatchNorm running statistics
afterwards.  dropin_pna.pt stores what the reference's own ``create_model_config`` (with the INTEGRATION.md dispatch) builds
for PNA configurations, for tests/test_cpu_dropin_pna.py.
"""
import sys

import torch

import make_golden as mg
from record import (HEAD_GRAPH, HEAD_NODE, HERE, REF, add_edge_and_pe, degree_histogram, dropin_config, pna_batch, record_case,
                    record_dropin, reference_create, save, targets)

# name: (input_dim, hidden, layers, output_type, output_dim, edge_dim, edge attribute kind, pooling, gps)
CASES = {
    "pna_graph_noedge": (3, 11, 3, ["graph"], [1], None, None, "mean", False),                       # ogb-like
    "pna_node_edge_len": (1, 10, 3, ["node"], [1], 1, "length", "mean", False),                      # EAM-like
    "pna_multihead_h5": (1, 5, 2, ["graph", "node", "node"], [1, 1, 1], None, None, "mean", False),  # lsms-like
    "pna_gps": (2, 16, 2, ["graph"], [1], None, None, "mean", True),
    "pna_add_pool_edge3": (2, 8, 2, ["graph"], [1], 3, "random", "add", False),
}


def install_pna_stubs():
    """PNAStack.py imports PNAConv / BatchNorm / Sequential from torch_geometric.nn: PNAConv is the restatement, BatchNorm the PyG
    wrapper; gps.py for the GPS case."""
    from oracle.gps import PyGBatchNorm
    from oracle.pna import PNAConv
    mg.install_stubs()
    tg = sys.modules["torch_geometric.nn"]
    tg.PNAConv, tg.BatchNorm = PNAConv, PyGBatchNorm
    sys.modules["hydragnn.models.Base"].BatchNorm = PyGBatchNorm
    mg.install_gps_stubs()
    return mg._load("hydragnn.models.PNAStack", REF + "/hydragnn/models/PNAStack.py")


def make_models(pna):
    gen = torch.Generator().manual_seed(8675309)
    out = {}
    for name, (input_dim, hidden, layers, otype, odim, edge_dim, ekind, pool, use_gps) in CASES.items():
        b = add_edge_and_pe(pna_batch(gen, [7, 5, 9, 6], input_dim), gen, ekind, edge_dim, use_gps)
        heads = {}
        if "graph" in otype:
            heads.update(HEAD_GRAPH)
        if "node" in otype:
            heads.update(HEAD_NODE)
        deg = degree_histogram(b)
        torch.manual_seed(0)
        m = pna.PNAStack("inv_node_feat, equiv_node_feat, edge_index", "inv_node_feat, edge_index", deg, edge_dim,
                         input_dim, hidden, odim, 4 if use_gps else 0, "GPS" if use_gps else None, "multihead" if use_gps else None,
                         4 if use_gps else 0, otype, heads, "relu", "mse", False, loss_weights=[1.0] * len(otype),
                         freeze_conv=False, initial_bias=None, num_conv_layers=layers, num_nodes=None, graph_pooling=pool)
        rec = record_case(m, b, *targets(b, otype, gen),
                          cfg=dict(input_dim=input_dim, hidden_dim=hidden, num_conv_layers=layers, output_type=otype, output_dim=odim,
                                   edge_dim=edge_dim, graph_pooling=pool, gps=use_gps, output_heads=heads))
        rec["deg"] = deg
        out[name] = {k: rec[k] for k in ("state", "inputs", "deg", "pred_eval", "pred_train", "value", "head_index", "loss",
                                         "state_after", "grads", "cfg")}
    return out


DROPIN_CASES = {"PNA-edge1-node": (1, "node"), "PNA-noedge-graph": (None, "graph")}


def make_dropin():
    create_model_config, _ = reference_create()
    create_model_config.__globals__["PNAStack"] = install_pna_stubs().PNAStack
    return {key: record_dropin(create_model_config, dropin_config("PNA", otype, edge_dim=edge_dim, pna_deg=[0, 4, 10, 7, 3, 1],
                                                                  hidden_dim=20, num_conv_layers=3))[0]
            for key, (edge_dim, otype) in DROPIN_CASES.items()}


def main():
    save(make_models(install_pna_stubs()), HERE + "/models_pna.pt", compact=False)
    save(make_dropin(), HERE + "/dropin_pna.pt", compact=False)


if __name__ == "__main__":
    main()
