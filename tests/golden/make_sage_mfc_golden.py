"""Generate tests/golden/models_sage.pt, models_mfc.pt and dropin_sage_mfc.pt by running the REFERENCE's own SAGEStack.py /
MFCStack.py + Base.py (and gps.py for the GPS cases, create.py for the drop-in cases) on the stubs of make_golden.py.  Run in the
build container only; the reference tree does not exist on the GPU machines.

    python tests/golden/make_sage_mfc_golden.py      # writes models_sage.pt, models_mfc.pt and dropin_sage_mfc.pt, nothing else

What the goldens pin: everything in those files that runs -- the layer loop with its BatchNorm feature layers, the GPS embedding
and wrapper, pooling, heads (conv-type node heads included), losses, ``initial_bias``, the MFC assertion -- EXCEPT PyG's
``SAGEConv`` and ``MFConv`` themselves, which are the restatements in oracle/sage.py [3P-memory]; test_oracle_sage_mfc.py pins
them by hand-computed cases.

Each model case stores the state dict, the inputs, the eval-mode predictions, and one train-mode step (batch statistics,
dropout off): predictions, the reference's own loss, every parameter gradient and the BatchNorm running statistics afterwards.
The graphs have isolated nodes, self-loops, duplicate edges and a hub whose in-degree exceeds every max_degree below 20.
"errors" stores what the reference's create_model raises; "interatomic" what its MLIP wrapper does with these position-free
stacks.
"""
import sys

import torch

import make_golden as mg
from record import (GPS, HEAD_GRAPH, HEAD_NODE, HERE, REF, dropin_config, pna_batch, record_case, record_dropin, reference_create,
                    refusal, save, targets)

# defined here, not in record.py: the pickled goldens hold one "branch-0" string object per module that spells it
HEAD_PER_NODE = {"node": [{"type": "branch-0", "architecture": {"num_headlayers": 2, "dim_headlayers": [7, 4], "type": "mlp_per_node"}}]}
HEAD_CONV = {"node": [{"type": "branch-0", "architecture": {"num_headlayers": 2, "dim_headlayers": [6, 5], "type": "conv"}}]}
SIZES = [7, 5, 9, 6]

# name: (input_dim, hidden, layers, output_type, output_dim, pooling, gps, heads, max_degree, initial_bias, graph sizes)
SAGE_CASES = {
    "sage_graph": (3, 8, 3, ["graph"], [1], "mean", False, HEAD_GRAPH, None, None, SIZES),
    "sage_node": (4, 6, 2, ["node"], [1], "mean", False, HEAD_NODE, None, None, SIZES),
    "sage_multihead": (2, 5, 2, ["graph", "node", "node"], [1, 1, 1], "add", False, None, None, None, SIZES),
    "sage_mlp_per_node": (3, 4, 2, ["node"], [1], "mean", False, HEAD_PER_NODE, None, None, [6, 6, 6, 6]),
    "sage_conv_head": (3, 6, 2, ["node"], [1], "mean", False, HEAD_CONV, None, None, SIZES),
    "sage_max_pool_in1": (1, 8, 3, ["graph"], [1], "max", False, HEAD_GRAPH, None, None, SIZES),
    "sage_gps": (2, 16, 2, ["graph"], [1], "mean", True, HEAD_GRAPH, None, None, SIZES),
    "sage_initial_bias": (3, 8, 2, ["graph"], [1], "mean", False, HEAD_GRAPH, None, 0.75, SIZES),
    "sage_initial_bias_node": (3, 8, 2, ["node"], [1], "mean", False, HEAD_NODE, None, 0.75, SIZES),
}
MFC_CASES = {
    "mfc_graph_deg5": (3, 8, 3, ["graph"], [1], "mean", False, HEAD_GRAPH, 5, None, SIZES),
    "mfc_node_deg1": (4, 6, 2, ["node"], [1], "mean", False, HEAD_NODE, 1, None, SIZES),
    "mfc_multihead_deg100": (2, 5, 2, ["graph", "node", "node"], [1, 1, 1], "add", False, None, 100, None, SIZES),
    "mfc_mlp_per_node": (3, 4, 2, ["node"], [1], "mean", False, HEAD_PER_NODE, 5, None, [6, 6, 6, 6]),
    "mfc_conv_head": (3, 6, 2, ["node"], [1], "mean", False, HEAD_CONV, 5, None, SIZES),
    "mfc_max_pool_in1": (1, 8, 3, ["graph"], [1], "max", False, HEAD_GRAPH, 5, None, SIZES),
    "mfc_gps": (2, 16, 2, ["graph"], [1], "mean", True, HEAD_GRAPH, 5, None, SIZES),
    "mfc_initial_bias_node": (3, 8, 2, ["node"], [1], "mean", False, HEAD_NODE, 5, 0.75, SIZES),
}


def batch(gen, sizes, input_dim):
    """pna_batch (isolated nodes, duplicate pairs) plus a self-loop on node 0, a duplicated self-loop on node 2 and a hub: node 1
    receives 20 more edges from the other nodes of the first graph."""
    b = pna_batch(gen, sizes, input_dim)
    n0 = sizes[0]
    hub_src = torch.randint(2, n0, (20,), generator=gen)
    extra = torch.stack([torch.cat([torch.tensor([0, 2, 2]), hub_src]), torch.cat([torch.tensor([0, 2, 2]), torch.ones(20, dtype=torch.long)])])
    b.edge_index = torch.cat([b.edge_index, extra], dim=1)
    b.edge_shifts = torch.zeros(b.edge_index.shape[1], 3)
    return b


def install_sage_mfc_stubs():
    from oracle.gps import PyGBatchNorm
    from oracle.sage import MFConv, SAGEConv
    mg.install_stubs()
    tg = sys.modules["torch_geometric.nn"]
    tg.SAGEConv, tg.MFConv, tg.BatchNorm = SAGEConv, MFConv, PyGBatchNorm
    tg.global_mean_pool = None
    sys.modules["hydragnn.models.Base"].BatchNorm = PyGBatchNorm
    mg.install_gps_stubs()
    sage = mg._load("hydragnn.models.SAGEStack", REF + "/hydragnn/models/SAGEStack.py")
    mfc = mg._load("hydragnn.models.MFCStack", REF + "/hydragnn/models/MFCStack.py")
    return sage, mfc


ARGS = ("inv_node_feat, equiv_node_feat, edge_index", "inv_node_feat, edge_index")     # create.py:296-297, 350-351


def build(kind, mods, input_dim, hidden, layers, otype, odim, pool, use_gps, heads, max_degree, initial_bias, num_nodes=None):
    """The stack as the reference's create_model builds it: SAGE without initial_bias (create.py:348-370), MFC with it."""
    torch.manual_seed(0)
    common = (input_dim, hidden, odim, 4 if use_gps else 0, "GPS" if use_gps else None, "multihead" if use_gps else None,
              4 if use_gps else 0, otype, heads, "relu", "mse", False)
    kw = dict(loss_weights=[1.0] * len(otype), freeze_conv=False, num_conv_layers=layers, num_nodes=num_nodes, graph_pooling=pool)
    if kind == "SAGE":
        return mods[0].SAGEStack(*ARGS, *common, **kw)
    return mods[1].MFCStack(*ARGS, max_degree, *common, initial_bias=initial_bias, **kw)


def make_models(kind, cases, mods, seed):
    gen = torch.Generator().manual_seed(seed)
    out = {}
    for name, (input_dim, hidden, layers, otype, odim, pool, use_gps, heads, max_degree, ibias, sizes) in cases.items():
        b = batch(gen, sizes, input_dim)
        if use_gps:
            b.pe = torch.randn(b.x.shape[0], 4, generator=gen)
            b.rel_pe = (b.pe[b.edge_index[0]] - b.pe[b.edge_index[1]]).abs()
        if heads is None:
            heads = dict(HEAD_GRAPH, **HEAD_NODE)
        num_nodes = sizes[0] if heads is HEAD_PER_NODE else None
        m = build(kind, mods, input_dim, hidden, layers, otype, odim, pool, use_gps, heads, max_degree, ibias, num_nodes)
        cfg = dict(input_dim=input_dim, hidden_dim=hidden, num_conv_layers=layers, output_type=otype, output_dim=odim,
                   graph_pooling=pool, gps=use_gps, output_heads=heads, num_nodes=num_nodes, initial_bias=ibias)
        if kind == "MFC":
            cfg["max_neighbours"] = max_degree
        out[name] = record_case(m, b, *targets(b, otype, gen), cfg=cfg)
    return out


def _config(mpnn_type, output_type, use_gps, initial_bias=None):
    return dropin_config(mpnn_type, output_type, input_dim=1, hidden_dim=8, num_conv_layers=3, max_neighbours=20,
                         initial_bias=initial_bias, **(GPS if use_gps else {}))


DROPIN_CASES = {"SAGE-graph-bias": ("SAGE", "graph", False, 0.5), "SAGE-node": ("SAGE", "node", False, None),
                "SAGE-gps-graph": ("SAGE", "graph", True, None), "MFC-node-bias": ("MFC", "node", False, 0.5),
                "MFC-node": ("MFC", "node", False, None), "MFC-gps-graph": ("MFC", "graph", True, None)}


def make_dropin():
    create_model_config, _ = reference_create()
    sage, mfc = install_sage_mfc_stubs()
    create_model_config.__globals__.update(SAGEStack=sage.SAGEStack, MFCStack=mfc.MFCStack)
    out = {key: record_dropin(create_model_config, _config(*case))[0] for key, case in DROPIN_CASES.items()}
    # the reference's refusals: MFC without max_neighbours; initial_bias with a graph head on MFC (Base._set_bias indexes the
    # head's branch dict with -1), which SAGE never meets because create.py does not pass initial_bias to it
    no_max = _config("MFC", "graph", False)
    no_max["Architecture"]["max_neighbours"] = None
    bias_graph = _config("MFC", "graph", False, 0.5)
    out["errors"] = {key: refusal(lambda: create_model_config(cfg, verbosity=0, use_gpu=False), config=cfg)
                     for key, cfg in (("mfc_no_max_neighbours", no_max), ("mfc_initial_bias_graph", bias_graph))}
    # enable_interatomic_potential on these position-free stacks: what the reference's wrapper does with a force loss
    from hydragnn_b200.data import Batch, Data
    inter = {}
    for mpnn_type in ("SAGE", "MFC"):
        cfg = _config(mpnn_type, "node", False)
        cfg["Architecture"].update(enable_interatomic_potential=True, energy_weight=1.0, energy_peratom_weight=1.0, force_weight=1.0)
        m = create_model_config(cfg, verbosity=0, use_gpu=False)
        gen = torch.Generator().manual_seed(5)
        d = Data(x=torch.rand(4, 1, generator=gen), pos=torch.rand(4, 3, generator=gen), edge_index=torch.tensor([[0, 1, 2, 3], [1, 2, 3, 0]]),
                 energy=torch.rand(1, 1, generator=gen), forces=torch.rand(4, 3, generator=gen))
        b = Batch.from_data_list([d])
        b.pos.requires_grad_(True)
        inter[mpnn_type] = refusal(lambda: m.energy_force_loss(m(b), b), wrapped=type(m).__name__)
    out["interatomic"] = inter
    return out


def main():
    mods = install_sage_mfc_stubs()
    save(make_models("SAGE", SAGE_CASES, mods, 20261017), HERE + "/models_sage.pt")
    save(make_models("MFC", MFC_CASES, mods, 20261018), HERE + "/models_mfc.pt")
    save(make_dropin(), HERE + "/dropin_sage_mfc.pt")


if __name__ == "__main__":
    main()
