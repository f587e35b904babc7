"""Multi-branch heads (one decoder branch per dataset, chosen by ``dataset_name``) in every order of differentiation.

* The closed grouped ops (``ops.GroupedMatMul``, ``ops.GroupedWgrad``, ``ops.GroupedBiasAdd``) against an fp64 ATen loop over
  the branches: outputs, first derivatives and second derivatives (``autograd.grad(create_graph=True)``), with an empty group,
  a one-row group and groups of more than one 64-row tile, at widths 1, 25, 50 and 200.  The force pass (``only_data_grads``)
  launches no grouped weight gradient.
* 3-branch EGNN and PaiNN interatomic potentials against the reference's own Base and ``energy_force_loss``
  (tests/golden/models_multibranch.pt, tests/golden/make_multibranch_golden.py), and 3-branch MACE potentials against
  oracle/mace.py: predictions, loss, tasks, forces and every parameter gradient at DESIGN §7's tolerances; the branch without
  graphs gets exactly zero gradients.
* ``hb.train``'s captured padded step against its eager path over batches whose branch mix changes: one capture serves every
  batch, which also shows that decoding reads nothing back to the host.
"""
import copy

import pytest
import torch

pytestmark = pytest.mark.gpu

import hydragnn_b200 as hb  # noqa: E402
from hydragnn_b200 import _lib, ops, padded  # noqa: E402
from hydragnn_b200.stacks import branch_groups  # noqa: E402
from hydragnn_b200.synthetic import ARCH  # noqa: E402
from oracle import mace as omace  # noqa: E402
from oracle.mlip import MLIPWrapper  # noqa: E402
from stack_support import MACE_KW, _loader, mace_batch  # noqa: E402

DEV = "cuda"
SIZES = [70, 0, 1, 130]                   # an empty group, a one-row group, groups of more than one 64-row tile


def rel_l2(a, b):
    a, b = a.detach().double().cpu(), b.detach().double().cpu()
    return float((a - b).norm() / b.norm().clamp(min=1e-30))


def _calls(fn):
    _lib.trace_begin()
    out = fn()
    return out, {c[0] for c in _lib.trace_end()}


# ---- the grouped ops against fp64 ----------------------------------------------------------------------------------------------
def _two_layers(x, w1, b1, w2, b2, lin, bias):
    """Linear - tanh - Linear per group: the grouped ops or the fp64 loop, through ``lin`` / ``bias``."""
    return bias(lin(torch.tanh(bias(lin(x, w1), b1)), w2), b2)


def _derivatives(x, params, lin, bias, c, u):
    """(y, first derivatives of <y, c> by x and every parameter, second derivatives of <d/dx, u> by the same)."""
    y = _two_layers(x, *params, lin, bias)
    leaves = [x] + list(params)
    first = torch.autograd.grad((y * c).sum(), leaves, create_graph=True)
    second = torch.autograd.grad((first[0] * u).sum(), leaves, allow_unused=True)     # d/dx does not depend on the last bias
    return y, first, [torch.zeros_like(t) if s is None else s for s, t in zip(second, leaves)]


@pytest.mark.parametrize("k,n", [(1, 25), (25, 50), (50, 200), (200, 1)])
def test_grouped_ops_match_fp64_in_every_order(k, n):
    gen = torch.Generator().manual_seed(17 + k + n)
    groups, m = len(SIZES), sum(SIZES)
    ids = torch.repeat_interleave(torch.arange(groups), torch.tensor(SIZES))[torch.randperm(m, generator=gen)]
    bg = branch_groups(ids.to(DEV), groups)
    # the grouping: rows sorted stably by branch, the branch of every sorted row
    order = torch.sort(ids, stable=True).indices
    assert torch.equal(bg.order.idx.long().cpu(), order)
    assert torch.equal(bg.rows.idx.long().cpu(), ids[order])
    assert bg.rowptr.tolist() == [0] + torch.cumsum(torch.tensor(SIZES), 0).tolist()
    h = 2 * n + 3
    x = torch.randn(m, k, generator=gen, dtype=torch.float64)[order]
    params = [torch.randn(groups, h, k, generator=gen, dtype=torch.float64) / k ** 0.5,
              torch.randn(groups, h, generator=gen, dtype=torch.float64),
              torch.randn(groups, n, h, generator=gen, dtype=torch.float64) / h ** 0.5,
              torch.randn(groups, n, generator=gen, dtype=torch.float64)]
    c = torch.randn(m, n, generator=gen, dtype=torch.float64)
    u = torch.randn(m, k, generator=gen, dtype=torch.float64)
    g_of_row = ids[order]

    def lin64(a, w):
        return torch.cat([a[g_of_row == g] @ w[g].T for g in range(groups)])

    def bias64(a, b):
        return a + b[g_of_row]

    ref = _derivatives(x.clone().requires_grad_(True), [p.clone().requires_grad_(True) for p in params], lin64, bias64, c, u)

    def lin(a, w):
        return ops.GroupedMatMul.apply(a, w, bg.rowptr, 0, True)

    def bias(a, b):
        return ops.GroupedBiasAdd.apply(a, b, bg.rows)

    f = lambda t: t.float().to(DEV).requires_grad_(True)    # noqa: E731
    out, calls = _calls(lambda: _derivatives(f(x), [f(p) for p in params], lin, bias, c.float().to(DEV), u.float().to(DEV)))
    assert {"hgb_grouped_linear", "hgb_grouped_wgrad", "hgb_gather_rows", "hgb_segment_sum"} <= calls
    y, first, second = out
    assert rel_l2(y, ref[0]) < 1e-5
    names = ["x", "w1", "b1", "w2", "b2"]
    for nm, a, b in zip(names, first, ref[1]):
        assert rel_l2(a, b) < 1e-5, ("first", nm, rel_l2(a, b))
    for nm, a, b in zip(names, second, ref[2]):
        assert rel_l2(a, b) < 1e-5, ("second", nm, rel_l2(a, b))
    for a in list(first[1:]) + list(second[1:]):
        assert float(a[1].detach().abs().max()) == 0.0          # the empty group's weights get exactly zero


def test_grouped_wgrad_closure_matches_fp64():
    """``GroupedWgrad``'s own derivatives (a third-order term of the MLIP loss): d/da = b H^T, d/db = a H."""
    gen = torch.Generator().manual_seed(3)
    groups, m, n, k = len(SIZES), sum(SIZES), 25, 50
    rowptr = torch.tensor([0] + torch.cumsum(torch.tensor(SIZES), 0).tolist(), dtype=torch.int32, device=DEV)
    g_of_row = torch.repeat_interleave(torch.arange(groups), torch.tensor(SIZES))
    a, b = torch.randn(m, n, generator=gen, dtype=torch.float64), torch.randn(m, k, generator=gen, dtype=torch.float64)
    hc = torch.randn(groups, n, k, generator=gen, dtype=torch.float64)

    def run(a, b, wgrad):
        h = wgrad(a, b)
        return (h,) + torch.autograd.grad((h * hc.to(h)).sum(), [a, b])

    def wgrad64(a, b):
        return torch.stack([a[g_of_row == g].T @ b[g_of_row == g] for g in range(groups)])

    ref = run(a.clone().requires_grad_(True), b.clone().requires_grad_(True), wgrad64)
    got = run(a.float().to(DEV).requires_grad_(True), b.float().to(DEV).requires_grad_(True),
              lambda p, q: ops.GroupedWgrad.apply(p, q, rowptr))
    for x, y in zip(got, ref):
        assert rel_l2(x, y) < 1e-5
    assert float(got[0][1].abs().max()) == 0.0


def test_force_pass_launches_no_grouped_weight_gradient():
    """Under ``only_data_grads`` (the force pass of the MLIP loss) the grouped ops differentiate by their data only; the second
    backward then still reaches every weight."""
    gen = torch.Generator().manual_seed(4)
    groups, m, k, n = len(SIZES), sum(SIZES), 50, 25
    ids = torch.repeat_interleave(torch.arange(groups), torch.tensor(SIZES))
    bg = branch_groups(ids.to(DEV), groups)
    x = torch.randn(m, k, generator=gen).to(DEV).requires_grad_(True)
    w = torch.randn(groups, n, k, generator=gen).to(DEV).requires_grad_(True)
    b = torch.randn(groups, n, generator=gen).to(DEV).requires_grad_(True)
    y = torch.tanh(ops.GroupedBiasAdd.apply(ops.GroupedMatMul.apply(x, w, bg.rowptr, 0, True), b, bg.rows))

    def force():
        with ops.only_data_grads():
            return torch.autograd.grad(y.sum(), x, create_graph=True)[0]
    gx, calls = _calls(force)
    assert "hgb_grouped_linear" in calls and "hgb_grouped_wgrad" not in calls and "hgb_segment_sum" not in calls
    gw, gb = torch.autograd.grad(gx.pow(2).sum(), [w, b])
    assert float(gw.abs().sum()) > 0 and float(gb.abs().sum()) > 0


# ---- against the reference's own code --------------------------------------------------------------------------------------------
def _check_mlip(e, d, ref_pred, ref_loss, ref_tasks, ref_forces, ref_grads, kind, rtol_grad):
    e.train()
    (pred, tot, tasks, forces), calls = _calls(lambda: _mlip_step(e, d, kind))
    assert {"hgb_grouped_linear", "hgb_grouped_wgrad"} <= calls
    assert rel_l2(pred[0], ref_pred) < 1e-5, rel_l2(pred[0], ref_pred)
    torch.testing.assert_close(tot.detach().cpu().double(), ref_loss.detach().double(), rtol=1e-5, atol=1e-6)
    for a, b in zip(tasks, ref_tasks):
        torch.testing.assert_close(a.detach().cpu().double(), b.detach().double(), rtol=1e-5, atol=1e-6)
    assert rel_l2(forces, ref_forces) < 1e-5, rel_l2(forces, ref_forces)
    pe = dict(e.model.named_parameters())
    for name, g in ref_grads.items():
        if "branch-1" in name:                                 # no graph of this batch belongs to branch 1
            assert pe[name].grad is None or float(pe[name].grad.abs().max()) == 0.0, name
        elif g is not None and float(g.abs().max()) > 0:
            assert rel_l2(pe[name].grad, g) < rtol_grad, (name, rel_l2(pe[name].grad, g))


def _mlip_step(e, d, kind):
    pred = e(d)
    energy = pred[0].sum()                                     # the sum of the graph energies (of the node energies)
    forces = -torch.autograd.grad(energy, d.pos, retain_graph=True)[0]
    tot, tasks = e.energy_force_loss(pred, d)
    tot.backward()
    return pred, tot, tasks, forces


@pytest.mark.parametrize("name", ["egnn_graph", "egnn_node", "painn_graph", "painn_node"])
def test_multibranch_mlip_matches_reference_golden(golden_dir, name):
    c = torch.load(golden_dir + "/models_multibranch.pt")[name]
    e = hb.create_model(**c["cfg"], enable_interatomic_potential=True, energy_weight=1.0, energy_peratom_weight=1.0, force_weight=1.0)
    e.model.load_state_dict(c["state"], strict=True)
    d = hb.Batch(**{k: v.clone().to(DEV) for k, v in c["inputs"].items()})
    d._num_graphs = int(c["inputs"]["batch"].max()) + 1
    d.pos.requires_grad_(True)
    _check_mlip(e, d, c["pred"][0], c["loss"], c["tasks"], c["forces"], c["grads"], c["cfg"]["output_type"][0], 1e-3)


def _branches(arch, n=3):
    return [{"type": "branch-%d" % b, "architecture": dict(arch)} for b in range(n)]


MACE_GRAPH = {"num_sharedlayers": 2, "dim_sharedlayers": 5, "num_headlayers": 2, "dim_headlayers": [10, 6]}
MACE_NODE = {"num_headlayers": 2, "dim_headlayers": [12, 12], "type": "mlp"}


@pytest.mark.parametrize("kind", ["graph", "node"])
def test_multibranch_mace_mlip_matches_oracle(kind):
    """A 3-branch MACE potential (every readout decodes by branch) against oracle/mace.py in fp64."""
    kw = dict(MACE_KW, output_dim=[1], output_type=[kind], task_weights=[1.0], loss_function_type="mse",
              output_heads={"graph": _branches(MACE_GRAPH), "node": _branches(MACE_NODE)},
              graph_pooling="add" if kind == "graph" else "mean",
              enable_interatomic_potential=True, energy_weight=1.0, energy_peratom_weight=1.0, force_weight=1.0)
    torch.manual_seed(0)
    o = omace.MACEOracle(**kw)
    with torch.no_grad():
        for p in o.parameters():                               # make every path matter, as test_gpu_mace does
            p.copy_(torch.randn_like(p) * (p.std() if p.numel() > 1 else 1.0))
    e = hb.create_model(mpnn_type="MACE", **kw)
    e.model.load_state_dict(o.state_dict(), strict=True)
    ow = MLIPWrapper(o.double(), 1.0, 1.0, 1.0)
    gen = torch.Generator().manual_seed(2)
    d = mace_batch(gen, sizes=(6, 8, 5, 7))
    d.dataset_name = torch.tensor([[2], [0], [0], [2]])
    d.energy = torch.randn(4, generator=gen, dtype=torch.float64)
    d.forces = torch.randn(26, 3, generator=gen, dtype=torch.float64)
    d.pos.requires_grad_(True)
    pred = ow(d)
    forces = -torch.autograd.grad(pred[0].sum(), d.pos, retain_graph=True)[0]
    lo, to = ow.energy_force_loss(pred, d)
    lo.backward()
    g = hb.Batch(x=d.x.float().to(DEV), pos=d.pos.detach().float().to(DEV), edge_index=d.edge_index.to(DEV), batch=d.batch.to(DEV),
                 dataset_name=d.dataset_name.to(DEV), energy=d.energy.float().to(DEV), forces=d.forces.float().to(DEV))
    g._num_graphs = 4
    g.pos.requires_grad_(True)
    _check_mlip(e, g, pred[0], lo, to, forces, {k: p.grad for k, p in o.named_parameters()}, kind, 1e-3)


# ---- the captured step against the eager path -------------------------------------------------------------------------------------
MIXES = [[0, 1, 2], [2, 0], [1], [0, 2, 2, 1], [2, 1]]      # the branch mix changes from batch to batch; one batch has one branch
GRAPH = {"num_sharedlayers": 2, "dim_sharedlayers": 5, "num_headlayers": 2, "dim_headlayers": [50, 25]}
NODE = {"num_headlayers": 2, "dim_headlayers": [60, 20], "type": "mlp"}


def _branch_loader(workload, sizes):
    loader = _loader(workload, sizes, with_edges=True)
    for b, mix in zip(loader, MIXES):
        g = int(b.batch.max()) + 1
        b.dataset_name = torch.tensor(mix)[torch.arange(g) % len(mix)].reshape(g, 1)
    return loader


def _flat(model):
    return torch.cat([p.detach().reshape(-1) for p in model.parameters()])


CASES = {
    "egnn_mlip": ("md17_egnn", True, dict(ARCH["md17_egnn"], output_heads={"graph": _branches(GRAPH), "node": _branches(NODE)})),
    "mace_mlip": ("qm9_painn", True, dict(MACE_KW, mpnn_type="MACE", hidden_dim=16, output_dim=[1], output_type=["node"],
                                          task_weights=[1.0], loss_function_type="mse",
                                          output_heads={"graph": _branches(MACE_GRAPH), "node": _branches(MACE_NODE)},
                                          enable_interatomic_potential=True, energy_weight=1.0, energy_peratom_weight=1.0,
                                          force_weight=1.0)),
    "painn_graph": ("qm9_painn", False, dict(ARCH["qm9_painn"], output_heads={"graph": _branches(GRAPH)})),
}


@pytest.mark.parametrize("case", list(CASES))
def test_captured_step_equals_eager_over_changing_branch_mixes(case):
    workload, mlip, kw = CASES[case]
    loader = _branch_loader(workload, [31, 24, 17, 24, 9])          # the largest batch first: its capacities hold every other
    m1 = hb.get_distributed_model(hb.create_model(**kw))
    m2 = copy.deepcopy(m1)
    assert padded.supported(m1)
    p0 = _flat(m1).clone()
    o1, o2 = hb.FlatAdamW(m1, lr=1e-3), hb.FlatAdamW(m2, lr=1e-3)
    fast = None
    for epoch in range(2):
        (e1, t1), calls = _calls(lambda: hb.train([b.clone() for b in loader], m1, o1, compute_grad_energy=mlip))
        e2, t2 = hb.train([b.clone() for b in loader], m2, o2, compute_grad_energy=mlip, fast=False)
        torch.testing.assert_close(e1, e2, rtol=2e-4, atol=1e-6)
        torch.testing.assert_close(t1.reshape(-1), t2.reshape(-1), rtol=2e-4, atol=1e-6)
        fast = fast or o1._hgb_fast
        assert o1._hgb_fast is fast and fast.recaptures == 0          # one capture serves every batch of both epochs
        if epoch == 0:
            assert "hgb_grouped_linear" in calls
    p1, p2 = _flat(m1), _flat(m2)
    assert rel_l2(p1, p2) < 2e-3
    assert rel_l2(p1 - p0, p2 - p0) < 2e-2                          # the distance travelled, not only where it ends


def test_differing_branch_architectures_train_eagerly():
    """Branches whose head layers differ cannot share one grouped launch: ``supported()`` refuses the captured step, ``hb.train``
    takes the eager path and decodes branch by branch."""
    graph = _branches(GRAPH)
    graph[1]["architecture"]["dim_headlayers"] = [50, 20]
    m = hb.get_distributed_model(hb.create_model(**dict(ARCH["qm9_painn"], output_heads={"graph": graph})))
    assert not padded.supported(m)
    o = hb.FlatAdamW(m, lr=1e-3)
    loader = _branch_loader("qm9_painn", [24, 17])
    p0 = _flat(m).clone()
    err, _ = hb.train([b.clone() for b in loader], m, o)
    assert getattr(o, "_hgb_fast", None) is None and bool(torch.isfinite(err).all())
    assert float((_flat(m) - p0).abs().max()) > 0
