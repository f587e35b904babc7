"""Generate tests/golden/models_pnaplus.pt and tests/golden/dropin_pnaplus.pt by running the REFERENCE's own PNAPlusStack.py +
Base.py (and gps.py for the GPS case) on the stubs of make_golden.py.  Run in the build container only; the
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
import sys
import types

import torch

import make_golden as mg
from oracle.pnaeq import DegreeScalerAggregation as _DSA
from record import (HEAD_GRAPH, HEAD_NODE, HERE, REF, add_edge_and_pe, degree_histogram, dropin_config, pna_batch, record_case,
                    record_dropin, reference_create, save, t2d, targets)

HEAD_CONV = {"node": [{"type": "branch-0", "architecture": {"num_headlayers": 2, "dim_headlayers": [6, 5], "type": "conv"}}]}
R, EXPO, RADIUS = 5, 5, 3.0

# name: (input_dim, hidden, layers, output_type, output_dim, edge_dim, edge attribute kind, pooling, gps, heads)
CASES = {
    "pnaplus_graph_noedge": (3, 11, 3, ["graph"], [1], None, None, "mean", False, HEAD_GRAPH),
    "pnaplus_node_edge_len": (1, 10, 3, ["node"], [1], 1, "length", "mean", False, HEAD_NODE),
    "pnaplus_multihead_h5": (1, 5, 2, ["graph", "node", "node"], [1, 1, 1], None, None, "mean", False, None),
    "pnaplus_gps": (2, 16, 2, ["graph"], [1], None, None, "mean", True, HEAD_GRAPH),
    "pnaplus_edge_dim0": (2, 8, 2, ["graph"], [1], 0, None, "mean", False, HEAD_GRAPH),
    "pnaplus_add_pool_edge3": (2, 8, 2, ["graph"], [1], 3, "random", "add", False, HEAD_GRAPH),
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
    mg.install_gps_stubs()
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
    return mg._load("hydragnn.models.PNAPlusStack", REF + "/hydragnn/models/PNAPlusStack.py")


def build(mod, input_dim, hidden, layers, otype, odim, edge_dim, pool, use_gps, heads, deg):
    ia, ca = "inv_node_feat, equiv_node_feat, edge_index, rbf", "inv_node_feat, edge_index, rbf"        # create.py:231-232
    torch.manual_seed(0)
    return mod.PNAPlusStack(ia, ca, deg, edge_dim, EXPO, R, RADIUS, input_dim, hidden, odim, 4 if use_gps else 0,
                            "GPS" if use_gps else None, "multihead" if use_gps else None, 4 if use_gps else 0, otype, heads,
                            "relu", "mse", False, loss_weights=[1.0] * len(otype), freeze_conv=False, initial_bias=None,
                            num_conv_layers=layers, num_nodes=None, graph_pooling=pool)


def make_models(mod):
    gen = torch.Generator().manual_seed(20261016)
    out = {}
    for name, (input_dim, hidden, layers, otype, odim, edge_dim, ekind, pool, use_gps, heads) in CASES.items():
        b = add_edge_and_pe(pna_batch(gen, [7, 5, 9, 6], input_dim), gen, ekind, edge_dim, use_gps)
        if heads is None:
            heads = dict(HEAD_GRAPH, **HEAD_NODE)
        deg = degree_histogram(b)
        m = build(mod, input_dim, hidden, layers, otype, odim, edge_dim, pool, use_gps, heads, deg)
        rec = record_case(m, b, *targets(b, otype, gen),
                          cfg=dict(input_dim=input_dim, hidden_dim=hidden, num_conv_layers=layers, output_type=otype, output_dim=odim,
                                   edge_dim=edge_dim, graph_pooling=pool, gps=use_gps, output_heads=heads, num_radial=R,
                                   radius=RADIUS, envelope_exponent=EXPO))
        rec["deg"] = deg
        out[name] = {k: rec[k] for k in ("state", "inputs", "deg", "pred_eval", "pred_train", "value", "head_index", "loss", "str",
                                         "state_after", "grads", "cfg")}
    # MLIP: node energy head, energy + per-atom energy + force loss (the reference's own energy_force_loss), eval mode
    b = mg.toy_batch(gen, [6, 5, 8, 3], 3.0, input_dim=1)
    deg = degree_histogram(b)
    m = build(mod, 1, 8, 2, ["node"], [1], None, "mean", False, HEAD_NODE, deg)
    state = {k: v.clone() for k, v in m.state_dict().items()}
    m.eval()
    inp = t2d(b)
    b.pos.requires_grad_(True)
    pred = m(b)
    glb = {"torch": torch, "torch_scatter": sys.modules["torch_scatter"]}
    mg._extract(REF + "/hydragnn/models/create.py", ["energy_force_loss"], glb)
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
                                       edge_dim=None, graph_pooling="mean", gps=False, output_heads=HEAD_NODE, num_radial=R,
                                       radius=RADIUS, envelope_exponent=EXPO)}
    return out


DROPIN_CASES = {"PNAPlus-edge1-node": (1, "node"), "PNAPlus-noedge-graph": (None, "graph")}


def make_dropin():
    create_model_config, _ = reference_create()
    create_model_config.__globals__["PNAPlusStack"] = install_pnaplus_stubs().PNAPlusStack
    return {key: record_dropin(create_model_config, dropin_config("PNAPlus", otype, edge_dim=edge_dim, pna_deg=[0, 4, 10, 7, 3, 1],
                                                                  hidden_dim=20, num_conv_layers=3, num_radial=R, radius=RADIUS,
                                                                  envelope_exponent=3))[0]
            for key, (edge_dim, otype) in DROPIN_CASES.items()}


def main():
    save(make_models(install_pnaplus_stubs()), HERE + "/models_pnaplus.pt")
    save(make_dropin(), HERE + "/dropin_pnaplus.pt")


if __name__ == "__main__":
    main()
