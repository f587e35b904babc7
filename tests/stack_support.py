"""What the test modules share: the model configurations of the reference goldens, the GaussianNLLLoss and PReLU cases, the
engine model of a golden case, the checks of a model against a golden case and of the engine against a drop-in golden, the
batches the GPU tests build, one training step of an oracle stack and the error summary the benchmark-shape tests bound.  A
plain module on the tests' import path; no test module imports another, and nothing here reads tests/golden/'s makers or the
reference checkout they need."""
import hashlib
import types

import torch

import hydragnn_b200 as hb
from hydragnn_b200 import _lib
from hydragnn_b200.synthetic import ARCH, WORKLOADS, make_samples
from oracle.base import case_kwargs
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


# ---- the cases of tests/golden/models_{gnll,prelu}.pt: the reference's own code under GaussianNLLLoss and under "prelu" ----------
GNLL_CASES = ["pna_ci_multihead", "pna_conv_head", "pna_gps", "egnn_initial_bias", "egnn_two_branches", "egnn_clamped",
              "painn_mlp_per_node", "cgcnn_graph"]
PRELU_CASES = ["pna_ci_multihead", "pna_conv_head_slope", "pna_gps", "egnn_graph_node", "egnn_two_branches", "egnn_gnll",
               "painn_mlp_per_node", "sage_graph_slope"]
PRELU_MACE_CASES = ["mace", "mace_film"]


def case_mpnn_type(name):
    """The stack of a models_{gnll,prelu}.pt case, named by the first word of the case."""
    return {"pna": "PNA", "egnn": "EGNN", "painn": "PAINN", "cgcnn": "CGCNN", "sage": "SAGE", "mace": "MACE"}[name.split("_")[0]]


def named_case_kwargs(name, c):
    """create_model keyword arguments of a models_{gnll,prelu}.pt case; a MACE case's cfg holds what differs from MACE_KW."""
    t = case_mpnn_type(name)
    if t == "MACE":
        c = dict(c, cfg=dict(MACE_KW, **c["cfg"]))
    return case_kwargs(t, c)


def prelu_engine(name, c, use_gpu=False):
    """The engine model of a models_prelu.pt case with the case's slope set."""
    m = hb.create_model(**named_case_kwargs(name, c), use_gpu=use_gpu)
    if c.get("slope") is not None:
        with torch.no_grad():
            m.activation_function.weight.fill_(c["slope"])
    return m


class Flat:
    """A mean-and-variance model seen as one returning the list the golden stores: the means of every head, then their
    variances."""

    def __init__(self, m):
        self.m = m

    def __getattr__(self, name):
        return getattr(self.m, name)

    def __call__(self, data):
        mean, var = self.m(data)
        return list(mean) + list(var)

    def loss(self, pred, value, head_index):
        k = len(pred) // 2
        return self.m.loss((pred[:k], pred[k:]), value, head_index)


# ---- the engine model of a case of tests/golden/models_{pna,pnaplus,cgcnn,gat,schnet}.pt ---------------------------------------
def golden_engine(mpnn_type, case, state=None):
    """The engine's model of a golden case on the GPU with ``state`` (the case's own by default) loaded strictly."""
    m = hb.create_model(**case_kwargs(mpnn_type, case))
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
    sd = hb.create_model(**case_kwargs("GAT", case), use_gpu=False).state_dict()
    want = case["state_sha256"]
    assert list(sd.keys()) == list(want.keys()), "state-dict names or order differ from the reference's"
    bad = [k for k, v in sd.items() if state_digest(v) != want[k]]
    assert not bad, "seeded values differ from the reference's: %s" % bad[:5]
    return {k: v.clone() for k, v in sd.items()}


# ---- checks against the reference goldens ---------------------------------------------------------------------------------
def golden_data(inputs, dtype=torch.float64, device="cpu"):
    """A golden case's ``inputs`` as attributes on ``device``, the floating-point ones in ``dtype``; ``edge_attr`` is None where
    the case has none."""
    d = types.SimpleNamespace(edge_attr=None)
    for k, v in inputs.items():
        setattr(d, k, v.to(device, dtype) if v.is_floating_point() else v.to(device))
    return d


def grad_close(rtol, atol):
    """Element-wise gradient bound: |g - ref| <= atol gmax + rtol |ref|, gmax the largest reference gradient entry of the case."""
    def check(name, g, ref, gmax):
        torch.testing.assert_close(g.detach().cpu().double(), ref.double(), rtol=rtol, atol=atol * gmax,
                                   msg=lambda s: name + ": " + s)
    return check


def grad_norm(rtol, atol):
    """Norm-wise gradient bound: ||g - ref|| <= rtol ||ref|| + atol."""
    def check(name, g, ref, gmax):
        err = float((g.detach().cpu().double() - ref.double()).norm())
        assert err <= rtol * float(ref.double().norm()) + atol, (name, err)
    return check


def check_grads(case, named, grads):
    """Every gradient the golden case stores against ``named`` ({parameter name: gradient}): ``grads(name, g, ref, gmax)``
    checks one (``grad_close`` or ``grad_norm``); where the reference has none, the gradient must be None or zero.  A case whose
    ``grads_scope`` is not "all" stores the gradients of some parameters only; every other case stores all of them."""
    stored = case["grads"]
    assert set(stored) <= set(named)
    if case.get("grads_scope", "all") == "all":
        assert set(stored) == set(named)
    gmax = max(float(g.abs().max()) for g in stored.values() if g is not None)
    for n, ref in stored.items():
        g = named[n]
        if ref is None:
            assert g is None or not g.any(), n
        else:
            assert g is not None, n
            grads(n, g, ref, gmax)


def check_golden_case(m, case, data, *, pred, loss, grads, state_after=(1e-5, 1e-7), eval_kernels=()):
    """``m`` against a golden case: eval-mode predictions, then one train-mode step on the case's targets with every dropout off:
    predictions, loss, every parameter gradient the case stores and the BatchNorm running statistics afterwards.

    ``data()`` makes ``m``'s input.  Bounds: ``pred`` = (eval, train) rel-L2 of every prediction; ``loss`` = (rtol, atol);
    ``grads`` as in ``check_grads``; ``state_after`` = (rtol, atol).  ``eval_kernels`` must all run in the eval-mode forward."""
    m.eval()
    if eval_kernels:
        _lib.trace_begin()
    with torch.no_grad():
        out = m(data())
    if eval_kernels:
        calls = {t[0] for t in _lib.trace_end()}
        assert set(eval_kernels) <= calls, sorted(calls)
    assert len(out) == len(case["pred_eval"])
    for a, b in zip(out, case["pred_eval"]):
        assert rel_l2(a.cpu(), b) < pred[0]
    m.train()
    _zero_dropout(m)
    m.zero_grad(set_to_none=True)
    p0 = next(m.parameters())
    value = case["value"].to(p0.device, p0.dtype)
    head_index = [i.to(p0.device) for i in case.get("head_index", [torch.arange(value.numel())])]
    out = m(data())
    for a, b in zip(out, case["pred_train"]):
        assert rel_l2(a.detach().cpu(), b) < pred[1]
    lv, _ = m.loss(out, value, head_index)
    lv.backward()
    got, want = float(lv.detach()), float(case["loss"])
    assert abs(got - want) <= loss[1] + loss[0] * abs(want), (got, want)
    check_grads(case, {n: p.grad for n, p in m.named_parameters()}, grads)
    sd = m.state_dict()
    for k, v in case.get("state_after", {}).items():
        torch.testing.assert_close(sd[k].cpu().to(v.dtype), v, rtol=state_after[0], atol=state_after[1], msg=lambda s, k=k: k + ": " + s)


def engine_case(m, c):
    """The engine model ``m``'s own record of golden case ``c``, in the case's layout and on the CPU: eval-mode predictions, then
    one train-mode step (``_train_step``): predictions, loss, gradients (None where a parameter has none) and the BatchNorm
    statistics after."""
    m.eval()
    with torch.no_grad():
        pred_eval = [p.cpu() for p in m(_batch(c["inputs"]))]
    pred, loss = _train_step(m, c)
    return dict(c, pred_eval=pred_eval, pred_train=[p.detach().cpu() for p in pred], loss=loss.detach().cpu(),
                grads={n: (p.grad.cpu() if p.grad is not None else None) for n, p in m.named_parameters()},
                state_after={k: v.cpu() for k, v in m.state_dict().items() if "running" in k or "num_batches" in k})


def check_seeded_state(eng, state):
    """The engine's seeded state dict has the names, order, shapes and values of the reference's ``state``, and ``state`` loads
    into it strictly and comes back out unchanged."""
    se = eng.state_dict()
    assert list(se.keys()) == list(state.keys())
    for k, v in state.items():
        assert v.shape == se[k].shape and torch.equal(v, se[k]), k
    eng.load_state_dict(state, strict=True)
    assert all(torch.equal(v, state[k]) for k, v in eng.state_dict().items())


def check_dropin(g, cls, name, batch_norm=True):
    """The engine model the reference's dispatch builds from the drop-in golden entry ``g`` is interchangeable with the reference's
    own: a ``cls`` stack (inside the MLIP wrapper where there is one) whose ``str`` is ``name``, as the reference's is, with the
    reference's seeded state dict, the attributes the training loop reads, and one feature layer per conv layer: PyG's BatchNorm
    wrapper, or with ``batch_norm`` False an Identity.  Returns the engine model."""
    mpnn_type = g["kwargs"]["mpnn_type"]
    assert mpnn_type == g["config"]["Architecture"]["mpnn_type"] and mpnn_type in hb.create.SUPPORTED
    eng = hb.create_model(**g["kwargs"])
    inner = getattr(eng, "model", eng)
    assert type(inner) is cls, type(inner)
    check_seeded_state(eng, g["state_dict"])
    for attr, want in g["attrs"].items():
        assert getattr(eng, attr) == want, attr
    assert str(inner) == g["repr"] == name
    kind = torch.nn.BatchNorm1d if batch_norm else torch.nn.Identity
    assert all(type(f.module if batch_norm else f) is kind for f in inner.feature_layers)
    assert len(inner.feature_layers) == len(inner.graph_convs) == g["config"]["Architecture"]["num_conv_layers"]
    return eng


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
