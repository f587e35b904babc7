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

# name: (input_dim, hidden, layers, output_type, output_dim, edge_dim, edge attribute kind, pooling, gps, heads, graph sizes)
CASES = {
    "cgcnn_graph_edge0": (3, 3, 3, ["graph"], [1], 0, None, "mean", False, mp.HEAD_GRAPH, [7, 5, 9, 6]),
    "cgcnn_node_edge_len": (4, 4, 3, ["node"], [1], 1, "length", "mean", False, mp.HEAD_NODE, [7, 5, 9, 6]),
    "cgcnn_add_pool_edge3": (2, 2, 2, ["graph"], [1], 3, "random", "add", False, mp.HEAD_GRAPH, [7, 5, 9, 6]),
    "cgcnn_multihead": (5, 5, 2, ["graph", "node", "node"], [1, 1, 1], 0, None, "mean", False, None, [7, 5, 9, 6]),
    "cgcnn_mlp_per_node": (3, 3, 2, ["node"], [1], 0, None, "mean", False, HEAD_PER_NODE, [6, 6, 6, 6]),
    "cgcnn_gps": (2, 16, 2, ["graph"], [1], 0, None, "mean", True, mp.HEAD_GRAPH, [7, 5, 9, 6]),
    "cgcnn_gps_edge2": (2, 8, 2, ["graph"], [1], 2, "random", "mean", True, mp.HEAD_GRAPH, [7, 5, 9, 6]),
    "cgcnn_ci_width1": (1, 1, 3, ["graph"], [1], 1, "length", "mean", False, mp.HEAD_GRAPH, [7, 5, 9, 6]),
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
    gps = mg.install_gps_stubs()
    mod = mg._load("hydragnn.models.CGCNNStack", mg.REF + "/hydragnn/models/CGCNNStack.py")
    return mod, gps


def build(mod, input_dim, hidden, layers, otype, odim, edge_dim, pool, use_gps, heads, num_nodes=None):
    torch.manual_seed(0)
    return mod.CGCNNStack("inv_node_feat, equiv_node_feat, edge_index", "inv_node_feat, edge_index", edge_dim,   # create.py:321-324
                          input_dim, hidden, odim, 4 if use_gps else 0, "GPS" if use_gps else None, "multihead" if use_gps else None,
                          4 if use_gps else 0, otype, heads, "relu", "mse", False, loss_weights=[1.0] * len(otype), freeze_conv=False,
                          initial_bias=None, num_conv_layers=layers, num_nodes=num_nodes, graph_pooling=pool)


def make_models(mod, gps):
    gen = torch.Generator().manual_seed(20261017)
    out = {}
    for name, (input_dim, hidden, layers, otype, odim, edge_dim, ekind, pool, use_gps, heads, sizes) in CASES.items():
        b = mp.pna_batch(gen, sizes, input_dim)
        if ekind == "length":
            b.edge_attr = (b.pos[b.edge_index[1]] - b.pos[b.edge_index[0]]).norm(dim=1, keepdim=True)
        elif ekind == "random":
            b.edge_attr = torch.randn(b.edge_index.shape[1], edge_dim, generator=gen)
        if use_gps:
            b.pe = torch.randn(b.x.shape[0], 4, generator=gen)
            b.rel_pe = (b.pe[b.edge_index[0]] - b.pe[b.edge_index[1]]).abs()
        if heads is None:
            heads = dict(mp.HEAD_GRAPH, **mp.HEAD_NODE)
        num_nodes = sizes[0] if heads is HEAD_PER_NODE else None
        m = build(mod, input_dim, hidden, layers, otype, odim, edge_dim, pool, use_gps, heads, num_nodes)
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
        out[name] = {"state": state, "inputs": mg.t2d(b), "pred_eval": pred_eval, "pred_train": [p.detach() for p in pred],
                     "value": value, "head_index": head_index, "loss": loss.detach(), "str": str(m),
                     "state_after": {k: v.clone() for k, v in m.state_dict().items() if "running" in k or "num_batches" in k},
                     "grads": {n: (g.detach() if g is not None else None) for (n, _), g in zip(m.named_parameters(), grads)},
                     "cfg": dict(input_dim=input_dim, hidden_dim=hidden, num_conv_layers=layers, output_type=otype, output_dim=odim,
                                 edge_dim=edge_dim, graph_pooling=pool, gps=use_gps, output_heads=heads, num_nodes=num_nodes)}
    errors = {}
    for name, heads in ERROR_CASES.items():
        try:
            build(mod, 3, 3, 2, ["node"], [1], 0, "mean", False, heads)
            errors[name] = None
        except Exception as e:                                       # noqa: BLE001 -- the reference's own exception is the datum
            errors[name] = {"type": type(e).__name__, "msg": str(e), "heads": heads}
    out["errors"] = errors
    return out


def _config(edge_dim, output_type, use_gps):
    from test_cpu_dropin import _config as base_config
    cfg = base_config("CGCNN", False)
    arch = cfg["Architecture"]
    arch.update(edge_dim=edge_dim, input_dim=1, hidden_dim=1, num_conv_layers=3, output_type=[output_type])
    if use_gps:
        arch.update(hidden_dim=8, pe_dim=6, global_attn_engine="GPS", global_attn_type="multihead", global_attn_heads=4)
    if output_type == "node":
        arch["output_heads"] = {"node": [{"type": "branch-0", "architecture": {"num_headlayers": 2, "dim_headlayers": [50, 25],
                                                                               "type": "mlp"}}]}
    return cfg


DROPIN_CASES = {"CGCNN-edge1-node": (1, "node", False), "CGCNN-edge0-graph": (0, "graph", False),
                "CGCNN-gps-edge0-graph": (0, "graph", True)}


def make_dropin(mod):
    import make_dropin_golden as md
    import hydragnn_b200 as hb
    create_model_config, _ = md._reference_create()
    # _reference_create re-installs the stubs: put the CGCNN pieces back and hand CGCNNStack to the reference's create_model
    mod, _ = install_cgcnn_stubs()
    create_model_config.__globals__["CGCNNStack"] = mod.CGCNNStack
    out = {}
    for key, (edge_dim, otype, use_gps) in DROPIN_CASES.items():
        cfg = _config(edge_dim, otype, use_gps)
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
    return out


def main():
    mod, gps = install_cgcnn_stubs()
    torch.save(_own(make_models(mod, gps)), os.path.join(HERE, "models_cgcnn.pt"))
    torch.save(_own(make_dropin(mod)), os.path.join(HERE, "dropin_cgcnn.pt"))
    print("written", os.path.join(HERE, "models_cgcnn.pt"), os.path.join(HERE, "dropin_cgcnn.pt"))


if __name__ == "__main__":
    main()
