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
import os
import sys

import torch

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, HERE)
sys.path.insert(0, os.path.dirname(HERE))

import make_golden as mg  # noqa: E402
from stack_support import state_digest  # noqa: E402
import make_pna_golden as mp  # noqa: E402


def _own(x, memo=None):
    """Every tensor in its own storage, except that views of one storage (the conv-head modules the reference lists twice in its
    state dict, under convs_node_* and heads_NN) stay one tensor: the file is written once per parameter, and it does not depend
    on which other tensors happened to share a storage."""
    memo = {} if memo is None else memo
    if torch.is_tensor(x):
        key = (x.untyped_storage().data_ptr(), x.storage_offset(), tuple(x.shape), tuple(x.stride()), x.dtype)
        if key not in memo:
            memo[key] = x.detach().clone()
        return memo[key]
    if isinstance(x, dict):
        return {k: _own(v, memo) for k, v in x.items()}
    if isinstance(x, (list, tuple)):
        return type(x)(_own(v, memo) for v in x)
    return x

CONV_HEAD = {"node": [{"type": "branch-0", "architecture": {"num_headlayers": 2, "dim_headlayers": [20, 10], "type": "conv"}}]}

# name: (input_dim, hidden, layers, output_type, output_dim, edge_dim, edge attribute kind, pooling, gps, heads, graph sizes)
CASES = {
    "gat_graph_noedge": (3, 8, 3, ["graph"], [1], None, None, "mean", False, mp.HEAD_GRAPH, [7, 5, 9, 6]),
    "gat_node_edge_len": (4, 5, 3, ["node"], [1], 1, "length", "mean", False, mp.HEAD_NODE, [7, 5, 9, 6]),
    "gat_multihead": (5, 4, 2, ["graph", "node", "node"], [1, 1, 1], None, None, "mean", False, None, [7, 5, 9, 6]),
    "gat_add_pool_edge3": (2, 4, 2, ["graph"], [1], 3, "random", "add", False, mp.HEAD_GRAPH, [7, 5, 9, 6]),
    "gat_one_layer": (3, 4, 1, ["graph"], [1], None, None, "mean", False, mp.HEAD_GRAPH, [7, 5, 9, 6]),
    "gat_input_ne_hidden": (7, 3, 2, ["node"], [1], None, None, "mean", False, mp.HEAD_NODE, [7, 5, 9, 6]),
    "gat_conv_head": (1, 20, 2, ["node"], [1], None, None, "mean", False, CONV_HEAD, [7, 5, 9, 6]),
    "gat_gps": (2, 8, 3, ["graph"], [1], None, None, "mean", True, mp.HEAD_GRAPH, [7, 5, 9, 6]),
    "gat_gps_edge2": (2, 8, 2, ["graph"], [1], 2, "random", "mean", True, mp.HEAD_GRAPH, [7, 5, 9, 6]),
    "gat_loops_dups_isolated": (3, 4, 2, ["node"], [1], 2, "random", "mean", False, mp.HEAD_NODE, [7, 5, 9, 6]),
}


def install_gat_stubs():
    from oracle.gat import GATv2Conv
    from oracle.gps import PyGBatchNorm
    mg.install_stubs()
    tg = sys.modules["torch_geometric.nn"]
    tg.GATv2Conv, tg.BatchNorm = GATv2Conv, PyGBatchNorm
    sys.modules["hydragnn.models.Base"].BatchNorm = PyGBatchNorm
    gps = mg.install_gps_stubs()
    mod = mg._load("hydragnn.models.GATStack", mg.REF + "/hydragnn/models/GATStack.py")
    return mod, gps


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


def make_models(mod, gps):
    gen = torch.Generator().manual_seed(20261018)
    out = {}
    for name, (input_dim, hidden, layers, otype, odim, edge_dim, ekind, pool, use_gps, heads, sizes) in CASES.items():
        b = mp.pna_batch(gen, sizes, input_dim)
        if name == "gat_loops_dups_isolated":
            b = loops_dups_isolated(b)
        if ekind == "length":
            b.edge_attr = (b.pos[b.edge_index[1]] - b.pos[b.edge_index[0]]).norm(dim=1, keepdim=True)
        elif ekind == "random":
            b.edge_attr = torch.randn(b.edge_index.shape[1], edge_dim, generator=gen)
        if use_gps:
            b.pe = torch.randn(b.x.shape[0], 4, generator=gen)
            b.rel_pe = (b.pe[b.edge_index[0]] - b.pe[b.edge_index[1]]).abs()
        if heads is None:
            heads = dict(mp.HEAD_GRAPH, **mp.HEAD_NODE)
        m = build(mod, input_dim, hidden, layers, otype, odim, edge_dim, pool, use_gps, heads)
        state = {k: state_digest(v) for k, v in m.state_dict().items()}
        m.eval()
        pred_eval = [p.detach() for p in m(b)]
        m.train()
        for sub in m.modules():
            if isinstance(sub, torch.nn.Dropout):
                sub.p = 0.0
            if isinstance(sub, gps.GPSConv):
                sub.dropout = 0.0
            if type(sub).__name__ == "GATv2Conv":
                sub.dropout = 0.0
        value, head_index = mp.targets(b, otype, gen)
        pred = m(b)
        loss, _ = m.loss(pred, value, head_index)
        grads = torch.autograd.grad(loss, list(m.parameters()), allow_unused=True)
        grads = {n: (g.detach() if g is not None else None) for (n, _), g in zip(m.named_parameters(), grads)}
        scope = "all"
        if name == "gat_conv_head":
            scope = "conv_heads"
            # the head modules are listed first under heads_NN (and again under convs_node_* / batch_norms_node_*)
            grads = {n: g for n, g in grads.items() if n.startswith("heads_NN.")}
            assert grads
        out[name] = {"state_sha256": state, "grads_scope": scope, "inputs": mg.t2d(b), "pred_eval": pred_eval, "pred_train": [p.detach() for p in pred],
                     "value": value, "head_index": head_index, "loss": loss.detach(), "str": str(m),
                     "state_after": {k: v.clone() for k, v in m.state_dict().items() if "running" in k or "num_batches" in k},
                     "grads": grads,
                     "top_level": sorted(n for n, _ in m.named_children()),
                     "cfg": dict(input_dim=input_dim, hidden_dim=hidden, num_conv_layers=layers, output_type=otype, output_dim=odim,
                                 edge_dim=edge_dim, graph_pooling=pool, gps=use_gps, output_heads=heads)}
    # a conv-type node head on a model with edge features: the head convs are built with edge_dim=None and handed edge_attr
    gen = torch.Generator().manual_seed(7)
    b = mp.pna_batch(gen, [5, 6], 1)
    b.edge_attr = torch.rand(b.edge_index.shape[1], 1, generator=gen)
    m = build(mod, 1, 4, 2, ["node"], [1], 1, "mean", False, CONV_HEAD)
    try:
        m(b)
        errors = {"conv_head_edge_attr": None}
    except Exception as e:                                           # noqa: BLE001 -- the reference's own exception is the datum
        errors = {"conv_head_edge_attr": {"type": type(e).__name__, "msg": str(e)}}
    out["errors"] = errors
    return out


def _config(edge_dim, output_type, use_gps):
    from test_cpu_dropin import _config as base_config
    cfg = base_config("GAT", False)
    arch = cfg["Architecture"]
    arch.update(edge_dim=edge_dim, input_dim=1, hidden_dim=8, num_conv_layers=3, output_type=[output_type])
    if use_gps:
        arch.update(pe_dim=6, global_attn_engine="GPS", global_attn_type="multihead", global_attn_heads=4)
    if output_type == "node":
        arch["output_heads"] = {"node": [{"type": "branch-0", "architecture": {"num_headlayers": 2, "dim_headlayers": [50, 25],
                                                                               "type": "mlp"}}]}
    return cfg


DROPIN_CASES = {"GAT-edge1-node": (1, "node", False), "GAT-noedge-graph": (None, "graph", False),
                "GAT-gps-noedge-graph": (None, "graph", True)}


def make_dropin(mod):
    import make_dropin_golden as md
    import hydragnn_b200 as hb
    create_model_config, _ = md._reference_create()
    # _reference_create re-installs the stubs: put the GAT pieces back and hand GATStack to the reference's create_model
    mod, _ = install_gat_stubs()
    create_model_config.__globals__["GATStack"] = mod.GATStack
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
    mod, gps = install_gat_stubs()
    torch.save(_own(make_models(mod, gps)), os.path.join(HERE, "models_gat.pt"))
    torch.save(_own(make_dropin(mod)), os.path.join(HERE, "dropin_gat.pt"))
    print("written", os.path.join(HERE, "models_gat.pt"), os.path.join(HERE, "dropin_gat.pt"))


if __name__ == "__main__":
    main()
