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
import os
import sys

import torch

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(HERE))
sys.path.insert(0, HERE)
sys.path.insert(0, os.path.dirname(HERE))

import make_golden as mg  # noqa: E402

HEAD_GRAPH = {"graph": [{"type": "branch-0", "architecture": {"num_sharedlayers": 2, "dim_sharedlayers": 5, "num_headlayers": 2,
                                                               "dim_headlayers": [10, 7]}}]}
HEAD_NODE = {"node": [{"type": "branch-0", "architecture": {"num_headlayers": 2, "dim_headlayers": [12, 6], "type": "mlp"}}]}

# name: (input_dim, hidden, layers, output_type, output_dim, edge_dim, edge attribute kind, pooling, gps)
CASES = {
    "pna_graph_noedge": (3, 11, 3, ["graph"], [1], None, None, "mean", False),                       # ogb-like
    "pna_node_edge_len": (1, 10, 3, ["node"], [1], 1, "length", "mean", False),                      # EAM-like
    "pna_multihead_h5": (1, 5, 2, ["graph", "node", "node"], [1, 1, 1], None, None, "mean", False),  # lsms-like
    "pna_gps": (2, 16, 2, ["graph"], [1], None, None, "mean", True),
    "pna_add_pool_edge3": (2, 8, 2, ["graph"], [1], 3, "random", "add", False),
}


def pna_batch(gen, sizes, input_dim):
    """Random directed edges inside every graph: uneven in-degrees, some nodes without incoming edges, duplicate pairs allowed."""
    from hydragnn_b200.data import Batch, Data
    samples = []
    for n in sizes:
        ne = int(torch.randint(n, 3 * n, (1,), generator=gen))
        src = torch.randint(0, n, (ne,), generator=gen)
        dst = torch.randint(0, max(n - 2, 1), (ne,), generator=gen)          # the last two nodes receive nothing
        keep = src != dst
        ei = torch.stack([src[keep], dst[keep]]).long()
        samples.append(Data(x=torch.randint(1, 9, (n, input_dim), generator=gen).float(), pos=torch.rand(n, 3, generator=gen) * 4.0,
                            edge_index=ei, edge_shifts=torch.zeros(ei.shape[1], 3), y=torch.randn(1, 1, generator=gen)))
    return Batch.from_data_list(samples)


def degree_histogram(b):
    deg = torch.bincount(b.edge_index[1], minlength=b.x.shape[0])
    return torch.bincount(deg).tolist()


def install_pna_stubs():
    """PNAStack.py imports PNAConv / BatchNorm / Sequential from torch_geometric.nn: PNAConv is the restatement, BatchNorm the PyG
    wrapper; gps.py for the GPS case."""
    from oracle.gps import PyGBatchNorm
    from oracle.pna import PNAConv
    mg.install_stubs()
    tg = sys.modules["torch_geometric.nn"]
    tg.PNAConv, tg.BatchNorm = PNAConv, PyGBatchNorm
    sys.modules["hydragnn.models.Base"].BatchNorm = PyGBatchNorm
    gps = mg.install_gps_stubs()
    pna = mg._load("hydragnn.models.PNAStack", mg.REF + "/hydragnn/models/PNAStack.py")
    return pna, gps


def targets(b, kinds, gen):
    """(value, head_index) in the layout Base.loss reads: one flat vector, one index tensor per head."""
    g, n = int(b.batch.max()) + 1, b.x.shape[0]
    vals, idx, off = [], [], 0
    for k in kinds:
        rows = g if k == "graph" else n
        vals.append(torch.randn(rows, generator=gen))
        idx.append(torch.arange(off, off + rows))
        off += rows
    return torch.cat(vals), idx


def make_models(pna, gps):
    gen = torch.Generator().manual_seed(8675309)
    out = {}
    for name, (input_dim, hidden, layers, otype, odim, edge_dim, ekind, pool, use_gps) in CASES.items():
        b = pna_batch(gen, [7, 5, 9, 6], input_dim)
        if ekind == "length":
            b.edge_attr = (b.pos[b.edge_index[1]] - b.pos[b.edge_index[0]]).norm(dim=1, keepdim=True)
        elif ekind == "random":
            b.edge_attr = torch.randn(b.edge_index.shape[1], edge_dim, generator=gen)
        if use_gps:
            b.pe = torch.randn(b.x.shape[0], 4, generator=gen)
            b.rel_pe = (b.pe[b.edge_index[0]] - b.pe[b.edge_index[1]]).abs()
        heads = {}
        if "graph" in otype:
            heads.update(HEAD_GRAPH)
        if "node" in otype:
            heads.update(HEAD_NODE)
        deg = degree_histogram(b)
        conv_args = "inv_node_feat, edge_index"
        torch.manual_seed(0)
        m = pna.PNAStack("inv_node_feat, equiv_node_feat, edge_index", conv_args, deg, edge_dim,
                         input_dim, hidden, odim, 4 if use_gps else 0, "GPS" if use_gps else None, "multihead" if use_gps else None,
                         4 if use_gps else 0, otype, heads, "relu", "mse", False, loss_weights=[1.0] * len(otype),
                         freeze_conv=False, initial_bias=None, num_conv_layers=layers, num_nodes=None, graph_pooling=pool)
        state = {k: v.clone() for k, v in m.state_dict().items()}
        m.eval()
        pred_eval = [p.detach() for p in m(b)]
        m.train()
        for mod in m.modules():
            if isinstance(mod, torch.nn.Dropout):
                mod.p = 0.0
            if isinstance(mod, gps.GPSConv):
                mod.dropout = 0.0
        value, head_index = targets(b, otype, gen)
        pred = m(b)
        loss, _ = m.loss(pred, value, head_index)
        grads = torch.autograd.grad(loss, list(m.parameters()), allow_unused=True)
        out[name] = {"state": state, "inputs": mg.t2d(b), "deg": deg, "pred_eval": pred_eval, "pred_train": [p.detach() for p in pred],
                     "value": value, "head_index": head_index, "loss": loss.detach(),
                     "state_after": {k: v.clone() for k, v in m.state_dict().items() if "running" in k or "num_batches" in k},
                     "grads": {n: (g.detach() if g is not None else None) for (n, _), g in zip(m.named_parameters(), grads)},
                     "cfg": dict(input_dim=input_dim, hidden_dim=hidden, num_conv_layers=layers, output_type=otype, output_dim=odim,
                                 edge_dim=edge_dim, graph_pooling=pool, gps=use_gps, output_heads=heads)}
    return out


def _pna_config(edge_dim, output_type):
    from test_cpu_dropin import _config
    cfg = _config("PNA", False)
    arch = cfg["Architecture"]
    arch.update(edge_dim=edge_dim, pna_deg=[0, 4, 10, 7, 3, 1], hidden_dim=20, num_conv_layers=3, output_type=[output_type])
    if output_type == "node":
        arch["output_heads"] = {"node": [{"type": "branch-0", "architecture": {"num_headlayers": 2, "dim_headlayers": [50, 25],
                                                                               "type": "mlp"}}]}
    return cfg


DROPIN_CASES = {"PNA-edge1-node": (1, "node"), "PNA-noedge-graph": (None, "graph")}


def make_dropin(pna):
    import make_dropin_golden as md
    import hydragnn_b200 as hb
    create_model_config, _ = md._reference_create()
    # _reference_create re-installs the stubs: put the PNA pieces back and hand PNAStack to the reference's create_model
    from oracle.gps import PyGBatchNorm
    from oracle.pna import PNAConv
    sys.modules["torch_geometric.nn"].PNAConv = PNAConv
    sys.modules["hydragnn.models.Base"].BatchNorm = PyGBatchNorm
    pna = mg._load("hydragnn.models.PNAStack", mg.REF + "/hydragnn/models/PNAStack.py")
    create_model_config.__globals__["PNAStack"] = pna.PNAStack
    out = {}
    for key, (edge_dim, otype) in DROPIN_CASES.items():
        cfg = _pna_config(edge_dim, otype)
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
    pna, gps = install_pna_stubs()
    torch.save(make_models(pna, gps), os.path.join(HERE, "models_pna.pt"))
    torch.save(make_dropin(pna), os.path.join(HERE, "dropin_pna.pt"))
    print("written", os.path.join(HERE, "models_pna.pt"), os.path.join(HERE, "dropin_pna.pt"))


if __name__ == "__main__":
    main()
