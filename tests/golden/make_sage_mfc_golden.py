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
import os
import sys

import torch

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, HERE)
sys.path.insert(0, os.path.dirname(HERE))

import make_golden as mg  # noqa: E402
import make_pna_golden as mp  # noqa: E402
from make_pnaplus_golden import _own  # noqa: E402

HEAD_PER_NODE = {"node": [{"type": "branch-0", "architecture": {"num_headlayers": 2, "dim_headlayers": [7, 4], "type": "mlp_per_node"}}]}
HEAD_CONV = {"node": [{"type": "branch-0", "architecture": {"num_headlayers": 2, "dim_headlayers": [6, 5], "type": "conv"}}]}
SIZES = [7, 5, 9, 6]

# name: (input_dim, hidden, layers, output_type, output_dim, pooling, gps, heads, max_degree, initial_bias, graph sizes)
SAGE_CASES = {
    "sage_graph": (3, 8, 3, ["graph"], [1], "mean", False, mp.HEAD_GRAPH, None, None, SIZES),
    "sage_node": (4, 6, 2, ["node"], [1], "mean", False, mp.HEAD_NODE, None, None, SIZES),
    "sage_multihead": (2, 5, 2, ["graph", "node", "node"], [1, 1, 1], "add", False, None, None, None, SIZES),
    "sage_mlp_per_node": (3, 4, 2, ["node"], [1], "mean", False, HEAD_PER_NODE, None, None, [6, 6, 6, 6]),
    "sage_conv_head": (3, 6, 2, ["node"], [1], "mean", False, HEAD_CONV, None, None, SIZES),
    "sage_max_pool_in1": (1, 8, 3, ["graph"], [1], "max", False, mp.HEAD_GRAPH, None, None, SIZES),
    "sage_gps": (2, 16, 2, ["graph"], [1], "mean", True, mp.HEAD_GRAPH, None, None, SIZES),
    "sage_initial_bias": (3, 8, 2, ["graph"], [1], "mean", False, mp.HEAD_GRAPH, None, 0.75, SIZES),
    "sage_initial_bias_node": (3, 8, 2, ["node"], [1], "mean", False, mp.HEAD_NODE, None, 0.75, SIZES),
}
MFC_CASES = {
    "mfc_graph_deg5": (3, 8, 3, ["graph"], [1], "mean", False, mp.HEAD_GRAPH, 5, None, SIZES),
    "mfc_node_deg1": (4, 6, 2, ["node"], [1], "mean", False, mp.HEAD_NODE, 1, None, SIZES),
    "mfc_multihead_deg100": (2, 5, 2, ["graph", "node", "node"], [1, 1, 1], "add", False, None, 100, None, SIZES),
    "mfc_mlp_per_node": (3, 4, 2, ["node"], [1], "mean", False, HEAD_PER_NODE, 5, None, [6, 6, 6, 6]),
    "mfc_conv_head": (3, 6, 2, ["node"], [1], "mean", False, HEAD_CONV, 5, None, SIZES),
    "mfc_max_pool_in1": (1, 8, 3, ["graph"], [1], "max", False, mp.HEAD_GRAPH, 5, None, SIZES),
    "mfc_gps": (2, 16, 2, ["graph"], [1], "mean", True, mp.HEAD_GRAPH, 5, None, SIZES),
    "mfc_initial_bias_node": (3, 8, 2, ["node"], [1], "mean", False, mp.HEAD_NODE, 5, 0.75, SIZES),
}


def batch(gen, sizes, input_dim):
    """pna_batch (isolated nodes, duplicate pairs) plus a self-loop on node 0, a duplicated self-loop on node 2 and a hub: node 1
    receives 20 more edges from the other nodes of the first graph."""
    b = mp.pna_batch(gen, sizes, input_dim)
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
    gps = mg.install_gps_stubs()
    sage = mg._load("hydragnn.models.SAGEStack", mg.REF + "/hydragnn/models/SAGEStack.py")
    mfc = mg._load("hydragnn.models.MFCStack", mg.REF + "/hydragnn/models/MFCStack.py")
    return sage, mfc, gps


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


def make_models(kind, cases, mods, gps, seed):
    gen = torch.Generator().manual_seed(seed)
    out = {}
    for name, (input_dim, hidden, layers, otype, odim, pool, use_gps, heads, max_degree, ibias, sizes) in cases.items():
        b = batch(gen, sizes, input_dim)
        if use_gps:
            b.pe = torch.randn(b.x.shape[0], 4, generator=gen)
            b.rel_pe = (b.pe[b.edge_index[0]] - b.pe[b.edge_index[1]]).abs()
        if heads is None:
            heads = dict(mp.HEAD_GRAPH, **mp.HEAD_NODE)
        num_nodes = sizes[0] if heads is HEAD_PER_NODE else None
        m = build(kind, mods, input_dim, hidden, layers, otype, odim, pool, use_gps, heads, max_degree, ibias, num_nodes)
        state = {k: v.clone() for k, v in m.state_dict().items()}
        m.eval()
        pred_eval = [p.detach() for p in m(b)]
        m.train()
        for sub in m.modules():
            if isinstance(sub, torch.nn.Dropout):
                sub.p = 0.0
            if isinstance(sub, gps.GPSConv):
                sub.dropout = 0.0
        value, head_index = mp.targets(b, otype, gen)
        pred = m(b)
        loss, _ = m.loss(pred, value, head_index)
        grads = torch.autograd.grad(loss, list(m.parameters()), allow_unused=True)
        cfg = dict(input_dim=input_dim, hidden_dim=hidden, num_conv_layers=layers, output_type=otype, output_dim=odim,
                   graph_pooling=pool, gps=use_gps, output_heads=heads, num_nodes=num_nodes, initial_bias=ibias)
        if kind == "MFC":
            cfg["max_neighbours"] = max_degree
        out[name] = {"state": state, "inputs": mg.t2d(b), "pred_eval": pred_eval, "pred_train": [p.detach() for p in pred],
                     "value": value, "head_index": head_index, "loss": loss.detach(), "str": str(m),
                     "state_after": {k: v.clone() for k, v in m.state_dict().items() if "running" in k or "num_batches" in k},
                     "grads": {n: (g.detach() if g is not None else None) for (n, _), g in zip(m.named_parameters(), grads)},
                     "cfg": cfg}
    return out


def _config(mpnn_type, output_type, use_gps, initial_bias=None):
    from test_cpu_dropin import _config as base_config
    cfg = base_config(mpnn_type, False)
    arch = cfg["Architecture"]
    arch.update(input_dim=1, hidden_dim=8, num_conv_layers=3, output_type=[output_type], max_neighbours=20, initial_bias=initial_bias)
    if use_gps:
        arch.update(pe_dim=6, global_attn_engine="GPS", global_attn_type="multihead", global_attn_heads=4)
    if output_type == "node":
        arch["output_heads"] = {"node": [{"type": "branch-0", "architecture": {"num_headlayers": 2, "dim_headlayers": [50, 25],
                                                                               "type": "mlp"}}]}
    return cfg


DROPIN_CASES = {"SAGE-graph-bias": ("SAGE", "graph", False, 0.5), "SAGE-node": ("SAGE", "node", False, None),
                "SAGE-gps-graph": ("SAGE", "graph", True, None), "MFC-node-bias": ("MFC", "node", False, 0.5),
                "MFC-node": ("MFC", "node", False, None), "MFC-gps-graph": ("MFC", "graph", True, None)}


def make_dropin():
    import make_dropin_golden as md
    import hydragnn_b200 as hb
    create_model_config, create_model = md._reference_create()
    # _reference_create re-installs the stubs: put the SAGE / MFC pieces back and hand both stacks to the reference's create_model
    sage, mfc, _ = install_sage_mfc_stubs()
    create_model_config.__globals__["SAGEStack"] = sage.SAGEStack
    create_model_config.__globals__["MFCStack"] = mfc.MFCStack
    out = {}
    for key, (mpnn_type, otype, use_gps, ibias) in DROPIN_CASES.items():
        cfg = _config(mpnn_type, otype, use_gps, ibias)
        os.environ.pop("HYDRAGNN_ENGINE", None)
        ref = create_model_config(cfg, verbosity=0, use_gpu=False)
        assert not type(ref).__module__.startswith("hydragnn_b200")
        seen = {}
        real = hb.create_model

        class Spy:
            __code__ = real.__code__

            def __call__(self, **kw):
                seen.update(kw)
                return real(**kw)

        hb.create_model = Spy()
        os.environ["HYDRAGNN_ENGINE"] = "b200"
        try:
            eng = create_model_config(cfg, verbosity=0, use_gpu=False)
        finally:
            hb.create_model = real
            os.environ.pop("HYDRAGNN_ENGINE", None)
        assert seen and type(eng).__module__.startswith("hydragnn_b200")
        out[key] = {"config": cfg, "kwargs": seen, "state_dict": {k: v.clone() for k, v in ref.state_dict().items()},
                    "attrs": {a: getattr(ref, a) for a in md.ATTRS}, "repr": str(ref)}
    # the reference's refusals: MFC without max_neighbours; initial_bias with a graph head on MFC (Base._set_bias indexes the
    # head's branch dict with -1), which SAGE never meets because create.py does not pass initial_bias to it
    errors = {}
    no_max = _config("MFC", "graph", False)
    no_max["Architecture"]["max_neighbours"] = None
    for key, cfg in (("mfc_no_max_neighbours", no_max), ("mfc_initial_bias_graph", _config("MFC", "graph", False, 0.5))):
        try:
            create_model_config(cfg, verbosity=0, use_gpu=False)
            errors[key] = None
        except Exception as e:                                        # noqa: BLE001 -- the reference's own exception is the datum
            errors[key] = {"type": type(e).__name__, "msg": str(e), "config": cfg}
    out["errors"] = errors
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
        try:
            m.energy_force_loss(m(b), b)
            inter[mpnn_type] = None
        except Exception as e:                                        # noqa: BLE001
            inter[mpnn_type] = {"type": type(e).__name__, "msg": str(e), "wrapped": type(m).__name__}
    out["interatomic"] = inter
    return out


def main():
    sage, mfc, gps = install_sage_mfc_stubs()
    torch.save(_own(make_models("SAGE", SAGE_CASES, (sage, mfc), gps, 20261017)), os.path.join(HERE, "models_sage.pt"))
    torch.save(_own(make_models("MFC", MFC_CASES, (sage, mfc), gps, 20261018)), os.path.join(HERE, "models_mfc.pt"))
    torch.save(_own(make_dropin()), os.path.join(HERE, "dropin_sage_mfc.pt"))
    print("written", *(os.path.join(HERE, f) for f in ("models_sage.pt", "models_mfc.pt", "dropin_sage_mfc.pt")))


if __name__ == "__main__":
    main()
