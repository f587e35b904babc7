"""Generate tests/golden/models_schnet.pt and tests/golden/dropin_schnet.pt by running the REFERENCE's own SCFStack.py + Base.py
(and gps.py for the GPS cases) on the stubs of make_golden.py.  Run in the build container only; the reference tree does not exist
on the GPU machines.

    python tests/golden/make_schnet_golden.py      # writes models_schnet.pt and dropin_schnet.pt, nothing else

What the golden pins: everything in SCFStack.py / Base.py / gps.py that runs -- CFConv, the three branches of get_conv, the
equivariant coordinate update, the GPS embedding, pooling, heads (including conv-type node heads), losses.  The PyG pieces
SCFStack.py imports (MessagePassing with aggr "add", GaussianSmearing, ShiftedSoftplus, RadiusInteractionGraph on
oracle/radius_graph.py, which SCFStack.py reaches as RadiusInteractionGraphCPU without CUDA) are the restatements in
oracle/schnet.py and in this file [3P-memory].

Each case of models_schnet.pt stores the state dict, the inputs, the eval-mode predictions, and one train-mode step (dropout
off): predictions, the reference's own loss and every parameter gradient, plus the radius graph of every in-layer conv.
"""
import os
import sys

import torch

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, HERE)
sys.path.insert(0, os.path.dirname(HERE))

import make_golden as mg  # noqa: E402

HEAD_GRAPH = {"graph": [{"type": "branch-0", "architecture": {"num_sharedlayers": 2, "dim_sharedlayers": 5, "num_headlayers": 2,
                                                               "dim_headlayers": [10, 7]}}]}
HEAD_CONV = {"node": [{"type": "branch-0", "architecture": {"num_headlayers": 2, "dim_headlayers": [10, 6], "type": "conv"}}]}

# name: (input_dim, hidden, layers, num_filters, num_gaussians, radius, max_neighbours, head, edge_dim, edge kind, pool, gps, equiv)
CASES = {
    "inlayer_graph": (2, 12, 2, 16, 10, 3.0, 32, "graph", None, None, "mean", False, False),
    "inlayer_truncated": (1, 8, 2, 8, 6, 3.5, 2, "graph", None, None, "mean", False, False),
    "equivariant_conv_head": (1, 10, 3, 12, 8, 3.0, 20, "conv", None, None, "mean", False, True),
    "edge_len": (1, 10, 2, 8, 10, 2.0, None, "graph", 1, "length", "mean", False, False),
    "edge3": (2, 8, 2, 12, 5, 2.5, None, "graph", 3, "random", "mean", False, False),
    "gps": (2, 16, 2, 8, 10, 3.0, None, "graph", None, None, "mean", True, False),
    "gps_edge2": (2, 16, 2, 8, 10, 3.0, None, "graph", 2, "random", "mean", True, False),
    "add_pool": (1, 12, 2, 10, 10, 3.0, 32, "graph", None, None, "add", False, False),
}


class RadiusInteractionGraph(torch.nn.Module):
    """edge_index = radius_graph(pos, cutoff, batch, max_num_neighbors) (torch_cluster's ordering and truncation,
    ``oracle.radius_graph``), edge_weight = |pos[row] - pos[col]|."""

    def __init__(self, cutoff=10.0, max_num_neighbors=32):
        super().__init__()
        self.cutoff, self.max_num_neighbors = cutoff, max_num_neighbors

    def forward(self, pos, batch):
        from oracle.radius_graph import radius_graph
        edge_index = radius_graph(pos, r=self.cutoff, batch=batch, max_num_neighbors=self.max_num_neighbors).to(pos.device)
        row, col = edge_index
        return edge_index, (pos[row] - pos[col]).norm(dim=-1)


class MessagePassing(torch.nn.Module):
    """aggr "add", flow source_to_target; ``propagate(edge_index, **kw)`` lifts every ``*_j`` argument of ``message`` to
    the sources and sums the messages at the targets."""

    def __init__(self, aggr="add", **kw):
        super().__init__()
        assert aggr == "add"

    def propagate(self, edge_index, x, W):
        m = self.message(x[edge_index[0]], W)
        return m.new_zeros((x.shape[0],) + tuple(m.shape[1:])).index_add_(0, edge_index[1], m)


def install_schnet_stubs():
    from oracle import schnet as so
    from oracle.gps import PyGBatchNorm
    mg.install_stubs()
    tg = sys.modules["torch_geometric.nn"]
    tg.MessagePassing = MessagePassing
    sys.modules["torch_geometric"].nn = tg
    mg._mod("torch_geometric.nn.models")
    mg._mod("torch_geometric.nn.models.schnet", GaussianSmearing=so.GaussianSmearing, ShiftedSoftplus=so.ShiftedSoftplus,
            RadiusInteractionGraph=RadiusInteractionGraph)
    mg._mod("hydragnn.preprocess")
    mg._mod("hydragnn.preprocess.graph_samples_checks_and_updates", RadiusInteractionGraphCPU=RadiusInteractionGraph)
    sys.modules["hydragnn.models.Base"].BatchNorm = PyGBatchNorm
    gps = mg.install_gps_stubs()
    scf = mg._load("hydragnn.models.SCFStack", mg.REF + "/hydragnn/models/SCFStack.py")
    return scf, gps


def schnet_batch(gen, sizes, input_dim, box):
    """Random molecules; ``edge_index`` (read by the edge_index branch only) holds random in-graph pairs, some longer than any
    cutoff, and nonzero ``edge_shifts`` that SchNet must ignore."""
    from hydragnn_b200.data import Batch, Data
    samples = []
    for n in sizes:
        ne = int(torch.randint(n, 3 * n, (1,), generator=gen))
        src = torch.randint(0, n, (ne,), generator=gen)
        dst = torch.randint(0, max(n - 1, 1), (ne,), generator=gen)
        keep = src != dst
        ei = torch.stack([src[keep], dst[keep]]).long()
        samples.append(Data(x=torch.randint(1, 9, (n, input_dim), generator=gen).float(), pos=torch.rand(n, 3, generator=gen) * box,
                            edge_index=ei, edge_shifts=torch.randn(ei.shape[1], 3, generator=gen),
                            energy=torch.randn(1, generator=gen), forces=torch.randn(n, 3, generator=gen),
                            y=torch.randn(1, 1, generator=gen)))
    return Batch.from_data_list(samples)


def make_models(scf, gps):
    gen = torch.Generator().manual_seed(24681357)
    out = {}
    for name, (input_dim, hidden, layers, nf, ng, rad, k, head, edge_dim, ekind, pool, use_gps, equiv) in CASES.items():
        b = schnet_batch(gen, [7, 5, 9, 6], input_dim, 4.0)
        if ekind == "length":
            b.edge_attr = (b.pos[b.edge_index[1]] - b.pos[b.edge_index[0]]).norm(dim=1, keepdim=True)
        elif ekind == "random":
            b.edge_attr = torch.randn(b.edge_index.shape[1], edge_dim, generator=gen)
        if use_gps:
            b.pe = torch.randn(b.x.shape[0], 4, generator=gen)
            b.rel_pe = (b.pe[b.edge_index[0]] - b.pe[b.edge_index[1]]).abs()
        heads = HEAD_GRAPH if head == "graph" else HEAD_CONV
        otype = ["graph"] if head == "graph" else ["node"]
        odim = [1] if head == "graph" else [2]
        if head != "graph":
            b.y = torch.randn(b.x.shape[0], 2, generator=gen)
        torch.manual_seed(0)
        m = scf.SCFStack("", "inv_node_feat, equiv_node_feat, edge_index, edge_weight, edge_rbf", nf, edge_dim, ng, rad,
                         input_dim, hidden, odim, 4 if use_gps else 0, "GPS" if use_gps else None, "multihead" if use_gps else None,
                         4 if use_gps else 0, otype, heads, "relu", "mse", equiv, max_neighbours=k, loss_weights=[1.0],
                         freeze_conv=False, initial_bias=None, num_conv_layers=layers, num_nodes=None, graph_pooling=pool)
        state = {kk: v.clone() for kk, v in m.state_dict().items()}
        graphs = []
        hooks = [mod.register_forward_hook(lambda mod_, inp, outp: graphs.append(outp[0].clone()))
                 for mod in m.modules() if isinstance(mod, sys.modules["torch_geometric.nn.models.schnet"].RadiusInteractionGraph)]
        m.eval()
        pred_eval = [p.detach() for p in m(b)]
        for h in hooks:
            h.remove()
        m.train()
        for mod in m.modules():
            if isinstance(mod, torch.nn.Dropout):
                mod.p = 0.0
            if isinstance(mod, gps.GPSConv):
                mod.dropout = 0.0
        value = b.y.reshape(-1)
        pred = m(b)
        loss, _ = m.loss(pred, value, [torch.arange(value.numel())])
        grads = torch.autograd.grad(loss, list(m.parameters()), allow_unused=True)
        out[name] = {"state": state, "inputs": mg.t2d(b), "pred_eval": pred_eval, "pred_train": [p.detach() for p in pred],
                     "value": value, "loss": loss.detach(), "graphs_eval": graphs,
                     "grads": {n: (g.detach() if g is not None else None) for (n, _), g in zip(m.named_parameters(), grads)},
                     "cfg": dict(input_dim=input_dim, hidden_dim=hidden, num_conv_layers=layers, num_filters=nf, num_gaussians=ng,
                                 radius=rad, max_neighbours=k, output_type=otype, output_dim=odim, output_heads=heads,
                                 edge_dim=edge_dim, graph_pooling=pool, gps=use_gps, equivariance=equiv)}
    return out


def _schnet_config(gps, mlip):
    from test_cpu_dropin import _config
    cfg = _config("SchNet", mlip)
    arch = cfg["Architecture"]
    arch.update(num_gaussians=10 if gps else 50, num_filters=8 if gps else 126, radius=7.0 if gps else 5.0, max_neighbours=5,
                hidden_dim=64 if gps else 32)
    if gps:
        arch.update(global_attn_engine="GPS", global_attn_type="multihead", global_attn_heads=8, pe_dim=2)
    else:
        arch.update(equivariance=True)
    return cfg


DROPIN_CASES = {"SchNet-gps-graph": (True, False), "SchNet-equivariant-mlip": (False, True)}


def make_dropin():
    import make_dropin_golden as md
    import hydragnn_b200 as hb
    create_model_config, _ = md._reference_create()
    scf, _ = install_schnet_stubs()
    create_model_config.__globals__["SCFStack"] = scf.SCFStack
    out = {}
    for key, (use_gps, mlip) in DROPIN_CASES.items():
        cfg = _schnet_config(use_gps, mlip)
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
        inner = ref.model if mlip else ref
        out[key] = {"config": cfg, "kwargs": seen, "state_dict": {k: v.clone() for k, v in ref.state_dict().items()},
                    "attrs": {a: getattr(ref, a) for a in md.ATTRS}, "repr": str(inner)}
    return out


def main():
    scf, gps = install_schnet_stubs()
    torch.save(make_models(scf, gps), os.path.join(HERE, "models_schnet.pt"))
    torch.save(make_dropin(), os.path.join(HERE, "dropin_schnet.pt"))
    print("written", os.path.join(HERE, "models_schnet.pt"), os.path.join(HERE, "dropin_schnet.pt"))


if __name__ == "__main__":
    main()
