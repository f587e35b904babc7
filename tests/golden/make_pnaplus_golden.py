"""Generate tests/golden/models_pnaplus.pt and tests/golden/dropin_pnaplus.pt by running the REFERENCE's own PNAPlusStack.py +
Base.py (and gps.py for the GPS case) on the stubs of make_golden.py / make_pna_golden.py.  Run in the build container only; the
reference tree does not exist on the GPU machines.

    python tests/golden/make_pnaplus_golden.py      # writes models_pnaplus.pt and dropin_pnaplus.pt, nothing else

What the golden pins: everything in PNAPlusStack.py (its own PNAConv included), Base.py and gps.py that runs.  The PyG pieces it
imports -- BesselBasisLayer / Envelope, MessagePassing.propagate, DegreeScalerAggregation, Linear, reset -- are the restatements
in oracle/pnaplus.py and in this file [3P-memory]; test_oracle_pnaplus.py pins the basis by hand-computed values.

Each case of models_pnaplus.pt stores the state dict, the inputs, the eval-mode predictions, and one train-mode step (batch
statistics, dropout off): predictions, the reference's own loss, every parameter gradient and the BatchNorm running statistics
afterwards.  The MLIP case stores the reference's own energy_force_loss in eval mode, the forces and the parameter gradients of
the loss (second order through the forces).  The radius is below the longest edges, so every case has edges past the cutoff.
"""
import os
import sys
import types

import torch

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, HERE)
sys.path.insert(0, os.path.dirname(HERE))

import make_golden as mg  # noqa: E402
import make_pna_golden as mp  # noqa: E402
from oracle.pnaeq import DegreeScalerAggregation as _DSA  # noqa: E402

HEAD_CONV = {"node": [{"type": "branch-0", "architecture": {"num_headlayers": 2, "dim_headlayers": [6, 5], "type": "conv"}}]}
R, EXPO, RADIUS = 5, 5, 3.0

# name: (input_dim, hidden, layers, output_type, output_dim, edge_dim, edge attribute kind, pooling, gps, heads)
CASES = {
    "pnaplus_graph_noedge": (3, 11, 3, ["graph"], [1], None, None, "mean", False, mp.HEAD_GRAPH),
    "pnaplus_node_edge_len": (1, 10, 3, ["node"], [1], 1, "length", "mean", False, mp.HEAD_NODE),
    "pnaplus_multihead_h5": (1, 5, 2, ["graph", "node", "node"], [1, 1, 1], None, None, "mean", False, None),
    "pnaplus_gps": (2, 16, 2, ["graph"], [1], None, None, "mean", True, mp.HEAD_GRAPH),
    "pnaplus_edge_dim0": (2, 8, 2, ["graph"], [1], 0, None, "mean", False, mp.HEAD_GRAPH),
    "pnaplus_add_pool_edge3": (2, 8, 2, ["graph"], [1], 3, "random", "add", False, mp.HEAD_GRAPH),
    "pnaplus_conv_head": (1, 8, 2, ["node"], [1], None, None, "mean", False, HEAD_CONV),
}


class DegreeScalerAggregation(_DSA):
    """oracle.pnaeq's restatement, taking PyG's [E, towers, F] messages."""

    def __init__(self, aggr, scaler, deg, train_norm=False):
        assert not train_norm, "PNAConv's default train_norm=False only"
        super().__init__(aggr, scaler, deg)

    def forward(self, x, index=None, dim_size=None, **kw):
        out = super().forward(x.reshape(x.shape[0], -1), index, dim_size)
        return out.view(out.shape[0], 1, -1)


class MessagePassing(torch.nn.Module):
    """The part of PyG's base class the reference's PNAConv uses: ``aggr_module`` registered first, ``propagate`` gathering
    x_i = x[edge_index[1]] (target) and x_j = x[edge_index[0]] and aggregating ``message`` at the targets."""

    def __init__(self, aggr=None, node_dim=0, **kw):
        super().__init__()
        self.aggr_module = aggr

    def reset_parameters(self):
        pass

    def propagate(self, edge_index, size=None, x=None, edge_attr=None, rbf=None):
        src, dst = edge_index[0], edge_index[1]
        m = self.message(x[dst], x[src], rbf=rbf, edge_attr=edge_attr)
        return self.aggr_module(m, dst, x.shape[0])


def reset(value):
    """torch_geometric.nn.inits.reset."""
    if hasattr(value, "reset_parameters"):
        value.reset_parameters()
    else:
        for child in value.children() if hasattr(value, "children") else []:
            reset(child)


def install_pnaplus_stubs():
    from oracle.pnaplus import BesselBasisLayer
    from oracle.gps import PyGBatchNorm
    mg.install_stubs()
    sys.modules["hydragnn.models.Base"].BatchNorm = PyGBatchNorm
    gps = mg.install_gps_stubs()
    tg = sys.modules["torch_geometric.nn"]
    tg.BatchNorm = PyGBatchNorm
    mg._mod("torch_geometric.nn.aggr", DegreeScalerAggregation=DegreeScalerAggregation)
    mg._mod("torch_geometric.nn.conv", MessagePassing=MessagePassing)
    mg._mod("torch_geometric.nn.dense")
    mg._mod("torch_geometric.nn.dense.linear", Linear=torch.nn.Linear)
    mg._mod("torch_geometric.nn.inits", reset=reset)
    sys.modules["torch_geometric.nn.resolver"].activation_resolver = lambda act, **kw: {"relu": torch.nn.ReLU}[act]()
    sys.modules["torch_geometric.typing"].Adj = object
    sys.modules["torch_geometric.utils"].degree = None
    mg._mod("torch_geometric.nn.models")
    mg._mod("torch_geometric.nn.models.dimenet", BesselBasisLayer=BesselBasisLayer)
    mod = mg._load("hydragnn.models.PNAPlusStack", mg.REF + "/hydragnn/models/PNAPlusStack.py")
    return mod, gps


def build(mod, input_dim, hidden, layers, otype, odim, edge_dim, pool, use_gps, heads, deg):
    ia, ca = "inv_node_feat, equiv_node_feat, edge_index, rbf", "inv_node_feat, edge_index, rbf"        # create.py:231-232
    torch.manual_seed(0)
    return mod.PNAPlusStack(ia, ca, deg, edge_dim, EXPO, R, RADIUS, input_dim, hidden, odim, 4 if use_gps else 0,
                            "GPS" if use_gps else None, "multihead" if use_gps else None, 4 if use_gps else 0, otype, heads,
                            "relu", "mse", False, loss_weights=[1.0] * len(otype), freeze_conv=False, initial_bias=None,
                            num_conv_layers=layers, num_nodes=None, graph_pooling=pool)


def make_models(mod, gps):
    gen = torch.Generator().manual_seed(20261016)
    out = {}
    for name, (input_dim, hidden, layers, otype, odim, edge_dim, ekind, pool, use_gps, heads) in CASES.items():
        b = mp.pna_batch(gen, [7, 5, 9, 6], input_dim)
        if ekind == "length":
            b.edge_attr = (b.pos[b.edge_index[1]] - b.pos[b.edge_index[0]]).norm(dim=1, keepdim=True)
        elif ekind == "random":
            b.edge_attr = torch.randn(b.edge_index.shape[1], edge_dim, generator=gen)
        if use_gps:
            b.pe = torch.randn(b.x.shape[0], 4, generator=gen)
            b.rel_pe = (b.pe[b.edge_index[0]] - b.pe[b.edge_index[1]]).abs()
        if heads is None:
            heads = dict(mp.HEAD_GRAPH, **mp.HEAD_NODE)
        deg = mp.degree_histogram(b)
        m = build(mod, input_dim, hidden, layers, otype, odim, edge_dim, pool, use_gps, heads, deg)
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
        out[name] = {"state": state, "inputs": mg.t2d(b), "deg": deg, "pred_eval": pred_eval, "pred_train": [p.detach() for p in pred],
                     "value": value, "head_index": head_index, "loss": loss.detach(), "str": str(m),
                     "state_after": {k: v.clone() for k, v in m.state_dict().items() if "running" in k or "num_batches" in k},
                     "grads": {n: (g.detach() if g is not None else None) for (n, _), g in zip(m.named_parameters(), grads)},
                     "cfg": dict(input_dim=input_dim, hidden_dim=hidden, num_conv_layers=layers, output_type=otype, output_dim=odim,
                                 edge_dim=edge_dim, graph_pooling=pool, gps=use_gps, output_heads=heads, num_radial=R,
                                 radius=RADIUS, envelope_exponent=EXPO)}
    # MLIP: node energy head, energy + per-atom energy + force loss (the reference's own energy_force_loss), eval mode
    b = mg.toy_batch(gen, [6, 5, 8, 3], 3.0, input_dim=1)
    deg = mp.degree_histogram(b)
    m = build(mod, 1, 8, 2, ["node"], [1], None, "mean", False, mp.HEAD_NODE, deg)
    state = {k: v.clone() for k, v in m.state_dict().items()}
    m.eval()
    inp = mg.t2d(b)
    b.pos.requires_grad_(True)
    pred = m(b)
    glb = {"torch": torch, "torch_scatter": sys.modules["torch_scatter"]}
    mg._extract(mg.REF + "/hydragnn/models/create.py", ["energy_force_loss"], glb)
    fake = types.SimpleNamespace(num_heads=1, head_type=["node"], model=m, loss_function=m.loss_function,
                                 energy_weight=1.0, energy_peratom_weight=1.0, force_weight=1.0)
    tot, tasks = glb["energy_force_loss"](fake, pred, b, create_graph=True)
    forces = -torch.autograd.grad(sys.modules["torch_scatter"].scatter_add(pred[0], b.batch, dim=0).sum(), b.pos,
                                  retain_graph=True)[0]
    grads = torch.autograd.grad(tot, list(m.parameters()), allow_unused=True)
    out["pnaplus_mlip"] = {"state": state, "inputs": inp, "deg": deg, "pred_eval": [p.detach() for p in pred], "loss": tot.detach(),
                           "tasks": [t.detach() for t in tasks], "forces": forces.detach(), "str": str(m),
                           "grads": {n: (g.detach() if g is not None else None) for (n, _), g in zip(m.named_parameters(), grads)},
                           "cfg": dict(input_dim=1, hidden_dim=8, num_conv_layers=2, output_type=["node"], output_dim=[1],
                                       edge_dim=None, graph_pooling="mean", gps=False, output_heads=mp.HEAD_NODE, num_radial=R,
                                       radius=RADIUS, envelope_exponent=EXPO)}
    return out


def _config(edge_dim, output_type):
    cfg = mp._pna_config(edge_dim, output_type)
    cfg["Architecture"].update(mpnn_type="PNAPlus", num_radial=R, radius=RADIUS, envelope_exponent=3)
    return cfg


DROPIN_CASES = {"PNAPlus-edge1-node": (1, "node"), "PNAPlus-noedge-graph": (None, "graph")}


def make_dropin(mod):
    import make_dropin_golden as md
    import hydragnn_b200 as hb
    create_model_config, _ = md._reference_create()
    # _reference_create re-installs the stubs: put the PNAPlus pieces back and hand PNAPlusStack to the reference's create_model
    mod, _ = install_pnaplus_stubs()
    create_model_config.__globals__["PNAPlusStack"] = mod.PNAPlusStack
    out = {}
    for key, (edge_dim, otype) in DROPIN_CASES.items():
        cfg = _config(edge_dim, otype)
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


def _own(x):
    """Every tensor in its own storage, so the saved file does not depend on which tensors happened to share one."""
    if torch.is_tensor(x):
        return x.detach().clone()
    if isinstance(x, dict):
        return {k: _own(v) for k, v in x.items()}
    if isinstance(x, (list, tuple)):
        return type(x)(_own(v) for v in x)
    return x


def main():
    mod, gps = install_pnaplus_stubs()
    torch.save(_own(make_models(mod, gps)), os.path.join(HERE, "models_pnaplus.pt"))
    torch.save(_own(make_dropin(mod)), os.path.join(HERE, "dropin_pnaplus.pt"))
    print("written", os.path.join(HERE, "models_pnaplus.pt"), os.path.join(HERE, "dropin_pnaplus.pt"))


if __name__ == "__main__":
    main()
