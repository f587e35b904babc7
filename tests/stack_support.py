"""What the test modules share: the model configurations of the reference goldens, the engine model of a golden case, the
batches the GPU tests build, one training step of an oracle stack and the error summary the benchmark-shape tests bound.
A plain module on the tests' import path; no test module imports another."""
import hashlib

import torch

import hydragnn_b200 as hb
from hydragnn_b200.synthetic import ARCH, WORKLOADS, make_samples
from oracle.radius_graph import radius_graph
from oracle.workloads import add_edges_cpu

DEV = "cuda"

# ---- model configurations of tests/golden/models{,_pnaeq,_gps,_heads}.pt and of the MACE oracle ---------------------------------
HEADS_NODE = {"node": [{"type": "branch-0", "architecture": {"num_headlayers": 2, "dim_headlayers": [12, 6], "type": "mlp"}}]}
HEADS_GRAPH = {"graph": [{"type": "branch-0", "architecture": {"num_sharedlayers": 2, "dim_sharedlayers": 5,
                                                               "num_headlayers": 2, "dim_headlayers": [10, 7]}}]}

MODEL_KW = {
    "egnn_mlip": dict(mpnn_type="EGNN", input_dim=1, hidden_dim=16, output_dim=[1], output_type=["node"],
                      output_heads=HEADS_NODE, activation_function="relu", num_conv_layers=3, task_weights=[1.0]),
    "egnn_equiv_multihead": dict(mpnn_type="EGNN", input_dim=2, hidden_dim=12, output_dim=[1, 3],
                                 output_type=["graph", "node"], output_heads=dict(HEADS_GRAPH, **HEADS_NODE),
                                 activation_function="lrelu_01", num_conv_layers=3, task_weights=[1.0, 2.0],
                                 equivariance=True, graph_pooling="add"),
    "painn_graph_mean": dict(mpnn_type="PAINN", input_dim=1, hidden_dim=16, output_dim=[1], output_type=["graph"],
                             output_heads=HEADS_GRAPH, activation_function="relu", num_conv_layers=2,
                             task_weights=[1.0], num_radial=5, radius=7.0, graph_pooling="mean"),
}
MODEL_KW["painn_graph_max"] = dict(MODEL_KW["painn_graph_mean"], graph_pooling="max")

PNAEQ_KW = dict(mpnn_type="PNAEq", input_dim=1, hidden_dim=12, output_dim=[1], output_type=["graph"], output_heads=HEADS_GRAPH,
                activation_function="relu", num_conv_layers=3, task_weights=[1.0], num_radial=6, radius=5.0)

GPS_KW = {
    "gps_egnn": dict(mpnn_type="EGNN", input_dim=2, hidden_dim=16, output_dim=[1], output_type=["graph"], output_heads=HEADS_GRAPH,
                     activation_function="relu", num_conv_layers=2, task_weights=[1.0], global_attn_engine="GPS",
                     global_attn_type="multihead", global_attn_heads=4, pe_dim=4),
    "gps_painn": dict(mpnn_type="PAINN", input_dim=2, hidden_dim=16, output_dim=[1], output_type=["graph"], output_heads=HEADS_GRAPH,
                      activation_function="relu", num_conv_layers=2, task_weights=[1.0], num_radial=5, radius=7.0,
                      global_attn_engine="GPS", global_attn_type="multihead", global_attn_heads=4, pe_dim=4),
}

HEADS_PERNODE = {"node": {"num_headlayers": 2, "dim_headlayers": [7, 5], "type": "mlp_per_node"}}
HEADS_CONV = {"node": {"num_headlayers": 2, "dim_headlayers": [10, 6], "type": "conv"}}
HEAD_KW = {
    "egnn_mlp_per_node": dict(mpnn_type="EGNN", input_dim=1, hidden_dim=12, output_dim=[2], output_type=["node"], output_heads=HEADS_PERNODE,
                              activation_function="relu", num_conv_layers=2, task_weights=[1.0], num_nodes=6),
    "egnn_conv_head": dict(mpnn_type="EGNN", input_dim=1, hidden_dim=12, output_dim=[2], output_type=["node"], output_heads=HEADS_CONV,
                           activation_function="relu", num_conv_layers=2, task_weights=[1.0]),
    "painn_conv_head": dict(mpnn_type="PAINN", input_dim=1, hidden_dim=12, output_dim=[2], output_type=["node"], output_heads=HEADS_CONV,
                            activation_function="relu", num_conv_layers=2, task_weights=[1.0], num_radial=5, radius=7.0),
}

MACE_KW = dict(input_dim=1, hidden_dim=8, output_dim=[1, 3], output_type=["graph", "node"],
               output_heads={"graph": {"num_sharedlayers": 2, "dim_sharedlayers": 5, "num_headlayers": 2, "dim_headlayers": [10, 6]},
                             "node": {"num_headlayers": 2, "dim_headlayers": [12, 12], "type": "mlp"}},
               activation_function="relu", loss_function_type="mae", task_weights=[1.0, 1.0], num_conv_layers=2, num_radial=8,
               radius=6.0, max_ell=2, node_max_ell=1, avg_num_neighbors=10.0, envelope_exponent=5, correlation=2, graph_pooling="mean", num_nodes=9)


def _zero_dropout(m):
    for mod in m.modules():
        if isinstance(mod, torch.nn.Dropout):
            mod.p = 0.0
        if hasattr(mod, "dropout") and isinstance(getattr(mod, "dropout"), float):
            mod.dropout = 0.0


def random_rotation(gen):
    q = torch.randn(4, generator=gen, dtype=torch.float64)
    a, b, c, d = (q / q.norm()).tolist()
    return torch.tensor([[a * a + b * b - c * c - d * d, 2 * (b * c - a * d), 2 * (b * d + a * c)],
                         [2 * (b * c + a * d), a * a - b * b + c * c - d * d, 2 * (c * d - a * b)],
                         [2 * (b * d - a * c), 2 * (c * d + a * b), a * a - b * b - c * c + d * d]], dtype=torch.float64)


def mace_batch(gen, sizes=(7, 9), box=4.0, radius=6.0):
    pos = torch.cat([torch.rand(k, 3, generator=gen, dtype=torch.float64) * box for k in sizes])
    batch = torch.cat([torch.full((k,), i) for i, k in enumerate(sizes)])
    z = torch.randint(1, 10, (sum(sizes), 1), generator=gen).double()
    ei = radius_graph(pos.float(), radius, batch, max_num_neighbors=100)
    d = hb.Batch(x=z, pos=pos, edge_index=ei, batch=batch)
    d._num_graphs = len(sizes)
    return d


# ---- the engine model of a case of tests/golden/models_{pna,pnaplus,cgcnn,gat,schnet}.pt ---------------------------------------
def engine_kwargs(mpnn_type, case):
    """create_model keyword arguments of a golden case (the reference's create.py fixes GAT's heads = 6, slope = 0.05)."""
    cfg = dict(case["cfg"])
    if cfg.pop("gps"):
        cfg.update(pe_dim=4, global_attn_engine="GPS", global_attn_type="multihead", global_attn_heads=4)
    if "deg" in case:
        cfg["pna_deg"] = case["deg"]
    return dict(mpnn_type=mpnn_type, task_weights=[1.0] * len(cfg["output_type"]), **cfg)


def golden_engine(mpnn_type, case, state=None):
    """The engine's model of a golden case on the GPU with ``state`` (the case's own by default) loaded strictly."""
    m = hb.create_model(**engine_kwargs(mpnn_type, case))
    m.load_state_dict(case["state"] if state is None else state, strict=True)
    return m


def state_digest(t):
    """SHA-256 of a tensor's dtype, shape and bytes: models_gat.pt pins the reference's seeded state dict entry by entry this way."""
    h = hashlib.sha256(repr((str(t.dtype), tuple(t.shape))).encode())
    h.update(t.detach().contiguous().cpu().numpy().tobytes())
    return h.hexdigest()


def seeded_state(case):
    """The reference's seeded state dict of a models_gat.pt case.  The file holds it as names in order with one SHA-256 per entry;
    the engine's own seeded construction (create_model on the CPU) reproduces it, and is checked against every digest here."""
    sd = hb.create_model(**engine_kwargs("GAT", case), use_gpu=False).state_dict()
    want = case["state_sha256"]
    assert list(sd.keys()) == list(want.keys()), "state-dict names or order differ from the reference's"
    bad = [k for k, v in sd.items() if state_digest(v) != want[k]]
    assert not bad, "seeded values differ from the reference's: %s" % bad[:5]
    return {k: v.clone() for k, v in sd.items()}


def check_grads(case, named_grads, check):
    """Calls ``check(name, grad, reference)`` for every gradient the case stores.  The conv-head case stores the gradients of its
    head modules only (its 120-wide stack convs are covered by the other cases); every other case stores all of them."""
    names = [n for n, _ in named_grads]
    stored = case["grads"]
    assert set(stored) <= set(names)
    if case.get("grads_scope", "all") == "all":
        assert set(stored) == set(names)
    for n, g in named_grads:
        if n in stored:
            check(n, g, stored[n])


# ---- GPU batches -------------------------------------------------------------------------------------------------------------
def rel_l2(a, b):
    return float((a.double() - b.double()).norm() / b.double().norm().clamp(min=1e-30))


def _graph(seed=0, n=3000):
    """Nodes 0..99 and 300..399 receive nothing, node 7 receives 1000 edges, 100..199 one each, 200..299 two each, 400.. random."""
    g = torch.Generator().manual_seed(seed)
    dst = torch.cat([torch.full((1000,), 7), torch.arange(100, 200), torch.arange(200, 300).repeat(2),
                     torch.randint(400, n, (3000,), generator=g)])
    dst[:1000] = 7
    src = torch.randint(0, n, (dst.numel(),), generator=g)
    perm = torch.randperm(dst.numel(), generator=g)
    return torch.stack([src[perm], dst[perm]]).to(DEV), n


def _batch(inputs):
    d = hb.Batch(**{k: v.clone().to(DEV) for k, v in inputs.items()})
    d._num_graphs = int(inputs["batch"].max()) + 1
    return d


def _train_step(m, c):
    """One train-mode step of an engine model on a golden case's inputs, dropout off: (predictions, loss)."""
    m.train()
    _zero_dropout(m)
    m.zero_grad(set_to_none=True)
    pred = m(_batch(c["inputs"]))
    loss, _ = m.loss(pred, c["value"].to(DEV), [i.to(DEV) for i in c["head_index"]])
    loss.backward()
    return pred, loss


def _bench_batch(name, graphs):
    """A synthetic batch of the benchmark workload with the oracle's CPU radius graph, edge lengths as the edge attribute where the
    architecture reads one, per-atom targets for a node head, and the batch's in-degree histogram."""
    b = add_edges_cpu(make_samples(name, graphs), name)
    n = b.pos.shape[0]
    if ARCH[name].get("edge_dim"):
        b.edge_attr = (b.pos[b.edge_index[1]] - b.pos[b.edge_index[0]] + b.edge_shifts).norm(dim=1, keepdim=True).contiguous()
    if ARCH[name]["output_type"] == ["node"]:
        b.y = torch.randn(n, 1, generator=torch.Generator().manual_seed(11))
    deg = torch.bincount(torch.bincount(b.edge_index[1], minlength=n)).tolist()
    return b, dict(ARCH[name], pna_deg=deg)


def _gpu_batch(cpu, name, g):
    """device twin of a CPU batch with its edges built by the ENGINE's neighbour kernels"""
    w = WORKLOADS[name]
    d = make_samples(name, g).to(DEV)
    d._num_graphs = g
    if w.get("pbc") or w.get("pbc_box"):
        d = hb.get_radius_graph_pbc(w["radius"], w["max_neighbours"])(d)
    else:
        d = hb.get_radius_graph(w["radius"], w["max_neighbours"])(d)
    if w.get("pe_dim"):
        d.rel_pe = (d.pe[d.edge_index[0]] - d.pe[d.edge_index[1]]).abs()
    return d


def _loader(name, sizes, with_edges, seed0=10):
    w = WORKLOADS[name]
    out = []
    for i, g in enumerate(sizes):
        b = make_samples(name, g, seed=seed0 + i)
        if with_edges:
            d = b.clone().to(DEV)
            d._num_graphs = g
            d = (hb.get_radius_graph_pbc if w.get("pbc") else hb.get_radius_graph)(w["radius"], w["max_neighbours"])(d)
            b.edge_index = d.edge_index.cpu()
            if d.edge_shifts is not None:
                b.edge_shifts = d.edge_shifts.cpu()
        for k in ("cell", "pbc", "ptr"):
            b.__dict__.pop(k, None)
        out.append(b)
    return out


def _grad_rel(em_params, om_params):
    """rel-L2 over all parameter gradients; accepts parameter lists (same order) or modules (matched by name)."""
    if isinstance(em_params, torch.nn.Module):
        en, on = dict(em_params.named_parameters()), dict(om_params.named_parameters())
        assert set(en) == set(on)
        em_params, om_params = [en[k] for k in on], [on[k] for k in on]
    num = den = 0.0
    for p, q in zip(em_params, om_params):
        if q.grad is None:
            continue
        assert p.grad is not None
        num += float((p.grad.double().cpu() - q.grad.double()).pow(2).sum())
        den += float(q.grad.double().pow(2).sum())
    return (num / max(den, 1e-300)) ** 0.5


# ---- an oracle stack's training step against the engine's ----------------------------------------------------------------------
class _OD:
    """A batch on the CPU with its floating-point fields in ``dtype``, for an oracle stack."""

    def __init__(self, b, dtype=torch.float64):
        for k in ("x", "pos", "batch", "edge_index", "edge_shifts", "edge_attr", "pe", "rel_pe", "y", "energy", "forces"):
            v = getattr(b, k, None)
            if v is not None:
                v = v.detach().cpu()
                v = v.to(dtype) if v.is_floating_point() else v
            setattr(self, k, v)


def _oracle(cls, kw, state, dtype=torch.float64):
    m = cls(**kw)
    m.load_state_dict(state, strict=True)
    return m.to(dtype)


def _oracle_step(cls, kw, state, b, dtype):
    """One train-mode forward + loss + gradient of the oracle stack ``cls`` in ``dtype`` on the CPU, dropout off
    -> (preds, loss, {name: grad}, state)."""
    om = _oracle(cls, kw, state, dtype).train()
    _zero_dropout(om)
    od = _OD(b, dtype)
    pred = om(od)
    loss, _ = om.loss(pred, od.y, [torch.arange(od.y.shape[0])])
    grads = dict(zip([n for n, _ in om.named_parameters()], torch.autograd.grad(loss, list(om.parameters()))))
    return [p.detach() for p in pred], loss.detach(), grads, om.state_dict()


def _errors(pred, loss, grads, state, ref, bn_stats=False):
    """rel-L2 of predictions, loss and all parameter gradients together against ``ref`` (an ``_oracle_step`` result), and with
    ``bn_stats`` of the BatchNorm running statistics."""
    rpred, rloss, rgrads, rstate = ref
    names = sorted(rgrads)
    g = torch.cat([grads[n].double().cpu().reshape(-1) for n in names])
    r = torch.cat([rgrads[n].double().cpu().reshape(-1) for n in names])
    err = {"pred": max(rel_l2(p.detach().cpu(), q) for p, q in zip(pred, rpred)),
           "loss": abs(float(loss) - float(rloss)) / abs(float(rloss)),
           "grad": rel_l2(g, r)}
    if bn_stats:
        err["bn_stats"] = max(rel_l2(state[k].cpu(), rstate[k]) for k in rstate if "running" in k)
    return err
