"""SAGE and MFC on the H100: the hgb_nbr kernels against fp64 (forward, data gradient, weight gradient) over widths, group
counts, mean / sum and both precisions; determinism, the data-only backward, C-ABI refusals and empty sizes; the engine against
every golden case of the reference's own stacks, and the fused layer against the composed one."""
import pytest
import torch

import hydragnn_b200 as hb
from hydragnn_b200 import _lib, ops
from oracle.base import case_kwargs
from stack_support import check_golden_case, golden_data, grad_close

pytestmark = pytest.mark.gpu

WIDTHS = [1, 3, 8, 31, 32, 55, 64, 100, 128]


def _graph(n=3001, seed=0):
    """Isolated nodes 0..99, a hub (node 7) of in-degree 1000, self-loops, duplicate edges, n not a multiple of 64."""
    g = torch.Generator().manual_seed(seed)
    dst = torch.cat([torch.full((1000,), 7), torch.arange(100, 200), torch.arange(200, 300).repeat(2), torch.arange(300, 340),
                     torch.randint(400, n, (6000,), generator=g)])
    src = torch.randint(0, n, (dst.numel(),), generator=g)
    src[1300:1340] = torch.arange(300, 340)                  # self-loops (nodes 300..339 receive their own edge)
    ei = torch.stack([src, dst])
    ei = torch.cat([ei, ei[:, -50:]], dim=1)                 # duplicates
    return ei.cuda(), n


def _layer(k, n_out, groups, seed=1):
    g = torch.Generator().manual_seed(seed)
    wl = torch.randn(groups, n_out, k, generator=g) / k ** 0.5
    bl = torch.randn(groups, n_out, generator=g)
    wr = torch.randn(groups, n_out, k, generator=g) / k ** 0.5
    return [t.cuda().requires_grad_(True) for t in (wl, bl, wr)]


def _ref(x, ei, wl, bl, wr, mean):
    """fp64 on the CPU: out_i = W_l,g h_i + b_l,g + W_r,g x_i."""
    x, wl, bl, wr = (t.detach().double().cpu().requires_grad_(True) for t in (x, wl, bl, wr))
    ei = ei.cpu()
    n = x.shape[0]
    h = torch.zeros_like(x).index_add(0, ei[1], x[ei[0]])
    deg = torch.bincount(ei[1], minlength=n)
    if mean:
        h = h / deg.clamp(min=1).double()[:, None]
    grp = deg.clamp(max=wl.shape[0] - 1)
    out = x.new_zeros(n, wl.shape[1])
    for gi in grp.unique().tolist():
        idx = (grp == gi).nonzero().view(-1)
        out = out.index_copy(0, idx, h[idx] @ wl[gi].t() + bl[gi] + x[idx] @ wr[gi].t())
    return out, (x, wl, bl, wr)


def _run(x, ei, n, wl, bl, wr, mean):
    plan = ops.EdgePlan(ei, n)
    dp = ops.degree_plan(plan, wl.shape[0])
    return ops.NbrLinearFn.apply(x, wl, bl, wr, dp, plan, mean), plan, dp


def _rel(a, b):
    return float((a.double().cpu() - b.double()).norm() / b.double().norm().clamp(min=1e-30))


@pytest.mark.parametrize("exact", [True, False])
@pytest.mark.parametrize("groups,mean", [(1, True), (1, False), (21, False), (101, False)])
@pytest.mark.parametrize("k", WIDTHS)
def test_kernels_against_fp64(k, groups, mean, exact):
    ei, n = _graph()
    # n_out 160 and 256 reach the 5- to 8-block accumulators; k = 128 with n_out = 256 the single-buffered weight stream
    for n_out in (WIDTHS + [160, 256] if groups == 1 and exact else [max(1, 128 - k), k] + ([160, 256] if k in (1, 55, 128) else [])):
        x = torch.randn(n, k, device="cuda", requires_grad=True)
        wl, bl, wr = _layer(k, n_out, groups)
        with ops.tensor_cores(not exact):
            y, _, _ = _run(x, ei, n, wl, bl, wr, mean)
            go = torch.randn_like(y)
            grads = torch.autograd.grad(y, [x, wl, bl, wr], go)
        ref, leaves = _ref(x, ei, wl, bl, wr, mean)
        rgrads = torch.autograd.grad(ref, leaves, go.double().cpu())
        # 3xTF32 is fp32-accurate, so the bound is fp32 summation: the hub sums 1000 rows, a weight gradient 3001; TF32 keeps 10
        # mantissa bits
        tol, wtol = (2e-5, 5e-5) if exact else (5e-3, 5e-3)
        assert _rel(y, ref) < tol, (k, n_out)
        for name, a, b in zip(("x", "wl", "bl", "wr"), grads, rgrads):
            assert _rel(a, b) < (tol if name == "x" else wtol), (name, k, n_out)


def test_unused_degree_groups_get_zero_gradients_and_repeats_are_bit_identical():
    ei, n = _graph()
    x = torch.randn(n, 16, device="cuda", requires_grad=True)
    wl, bl, wr = _layer(16, 24, 101)
    deg = torch.bincount(ei[1].cpu(), minlength=n).clamp(max=100)
    unused = sorted(set(range(101)) - set(deg.tolist()))
    assert unused
    outs = []
    for _ in range(2):
        y, _, _ = _run(x, ei, n, wl, bl, wr, False)
        outs.append((y,) + torch.autograd.grad(y, [x, wl, bl, wr], torch.ones_like(y)))
    for a, b in zip(*outs):
        assert torch.equal(a, b)
    assert not outs[0][2][unused].any() and not outs[0][4][unused].any()


def test_data_only_backward_writes_no_weight_gradient():
    ei, n = _graph()
    x = torch.randn(n, 8, device="cuda", requires_grad=True)
    wl, bl, wr = _layer(8, 8, 21)
    y, _, _ = _run(x, ei, n, wl, bl, wr, False)
    with ops.only_data_grads():
        gx, gw = torch.autograd.grad(y.sum(), [x, wl], allow_unused=True)
    assert gx is not None and gw is None


def test_c_abi_refusals_happen_before_any_launch():
    L = _lib.lib()
    before = L.hgb_launch_count()
    assert not _lib.query("hgb_nbr_linear_supported", 129, 8, 1) and not _lib.query("hgb_nbr_linear_supported", 8, 257, 1)
    assert not _lib.query("hgb_nbr_linear_supported", 8, 8, 129) and not _lib.query("hgb_nbr_linear_supported", 0, 8, 1)
    for args in ((None, 10, 129), (None, -1, 8)):
        with pytest.raises(RuntimeError):
            _lib.call("hgb_nbr_linear_fwd", None, args[1], args[2], None, None, 0, 1, None, None, None, 1, None, None, 8, None, None,
                      1, None)
    with pytest.raises(RuntimeError):
        _lib.call("hgb_nbr_linear_bwd_data", None, 10, 300, None, 1, None, None, None, 1, None, 8, None, None, 1, None)
    with pytest.raises(RuntimeError):
        _lib.call("hgb_nbr_tiles", None, 0, 10, None, None)
    assert L.hgb_launch_count() == before


def test_no_nodes_and_no_edges():
    wl, bl, wr = _layer(8, 8, 3)
    # n = 0: nothing launches
    L = _lib.lib()
    before = L.hgb_launch_count()
    _lib.call("hgb_nbr_linear_fwd", None, 0, 8, None, None, 0, 1, None, None, None, 3, None, None, 8, None, None, 1, None)
    _lib.call("hgb_nbr_linear_bwd_data", None, 0, 8, None, 1, None, None, None, 3, None, 8, None, None, 1, None)
    assert L.hgb_launch_count() == before
    # e = 0: the root term alone, every node in group 0
    n = 70
    ei = torch.zeros(2, 0, dtype=torch.long, device="cuda")
    x = torch.randn(n, 8, device="cuda", requires_grad=True)
    y, _, _ = _run(x, ei, n, wl, bl, wr, True)
    torch.testing.assert_close(y, x @ wr[0].t() + bl[0], rtol=1e-5, atol=1e-5)
    gx, gwl = torch.autograd.grad(y.sum(), [x, wl])
    torch.testing.assert_close(gx, wr[0].sum(0).expand(n, 8), rtol=1e-5, atol=1e-5)
    assert not gwl.any()
    assert L.hgb_version() >= 109


# ---- engine ----------------------------------------------------------------------------------------------------------------------
def _cases(golden_dir, kind):
    return torch.load(golden_dir + "/models_%s.pt" % kind.lower())


def _engine(kind, c):
    m = hb.create_model(**case_kwargs(kind, c))
    m.load_state_dict(c["state"], strict=True)
    for sub in m.modules():
        if hasattr(sub, "dropout") and isinstance(sub.dropout, float):
            sub.dropout = 0.0
        if isinstance(sub, torch.nn.Dropout):
            sub.p = 0.0
    return m


@pytest.mark.parametrize("kind", ["SAGE", "MFC"])
def test_engine_against_every_golden_case(golden_dir, kind):
    """Eval and train-mode predictions, the loss, every parameter gradient and the BatchNorm running statistics of the
    reference's own stack (fp32 on the CPU)."""
    for name, c in _cases(golden_dir, kind).items():
        check_golden_case(_engine(kind, c), c, lambda: golden_data(c["inputs"], torch.float32, "cuda"), pred=(1e-4, 1e-4),
                          loss=(1e-4, 0), grads=grad_close(2e-3, 2e-5))


@pytest.mark.parametrize("workload", ["ogb_sage", "ogb_mfc", "ogb_sage_gps"])
@pytest.mark.parametrize("precision", ["fp32", "bf16"])
def test_fused_against_composed_at_the_workload_shapes(workload, precision):
    """One model forward + backward at the workload's shapes, the fused layers against the composed path of the same model."""
    from hydragnn_b200.synthetic import ARCH
    b = _workload_batch(workload)
    m = _no_dropout(hb.create.set_precision(hb.create_model(**ARCH[workload]), precision))
    res = []
    for composed in (False, True):
        m.force_higher_order = composed
        pred = m(b)[0]
        loss = (pred - b.y.view(pred.shape)).pow(2).mean()
        res.append((pred.detach(),) + torch.autograd.grad(loss, list(m.parameters()), allow_unused=True))
    tol = 1e-4 if precision == "fp32" else 2e-2
    assert _rel(res[0][0], res[1][0].cpu()) < tol
    # a conv bias in front of a BatchNorm has a gradient of zero up to rounding: its error is measured against the largest
    # gradient norm instead of its own
    floor = 1e-3 * max(float(c.norm()) for c in res[1][1:] if c is not None)
    for (name, _), a, c in zip(m.named_parameters(), res[0][1:], res[1][1:]):
        if c is None:
            assert a is None or not a.any(), name
            continue
        err = float((a.double() - c.double()).norm()) / max(float(c.norm()), floor)
        assert err < 10 * tol, (name, err)


@pytest.mark.parametrize("kind", ["SAGE", "MFC"])
def test_interatomic_potential_fails_as_the_reference_does(golden_dir, kind):
    """The stacks never read the positions: the reference's MLIP wrapper fails taking d energy / d pos, and so does the engine's."""
    from hydragnn_b200.data import Batch, Data
    err = torch.load(golden_dir + "/dropin_sage_mfc.pt")["interatomic"][kind]
    kw = dict(torch.load(golden_dir + "/dropin_sage_mfc.pt")[kind + "-node"]["kwargs"])
    kw.update(enable_interatomic_potential=True, energy_weight=1.0, energy_peratom_weight=1.0, force_weight=1.0, use_gpu=True)
    m = hb.create_model(**kw)
    assert type(m).__name__ == err["wrapped"]
    d = Data(x=torch.rand(4, 1), pos=torch.rand(4, 3), edge_index=torch.tensor([[0, 1, 2, 3], [1, 2, 3, 0]]), energy=torch.rand(1, 1),
             forces=torch.rand(4, 3))
    b = Batch.from_data_list([d]).to("cuda")
    b.pos.requires_grad_(True)
    with pytest.raises(Exception) as info:
        m.energy_force_loss(m(b), b)
    assert type(info.value).__name__ == err["type"] and str(info.value) == err["msg"]


@pytest.mark.parametrize("k,n_out,groups,mean,higher", [
    (130, 64, 1, True, False),          # k above the fused kernel's limit: first-order composed (linear_act)
    (16, 300, 1, False, False),         # n_out above it
    (16, 24, 150, False, False),        # more weight groups than the tile table takes: the grouped Linear, no tile table built
    (8, 12, 21, False, True),           # a higher-order pass
])
def test_composed_path_against_fp64(k, n_out, groups, mean, higher):
    from hydragnn_b200.sage import _nbr_layer
    ei, n = _graph()
    x = torch.randn(n, k, device="cuda", requires_grad=True)
    wl, bl, wr = _layer(k, n_out, groups)
    plan = ops.EdgePlan(ei, n)
    dp = ops.degree_plan(plan, groups)
    assert (dp.tiles is None) == (groups > ops.NBR_MAX_GROUPS)
    y = _nbr_layer(x, plan, dp, wl, bl, wr, mean, higher)
    go = torch.randn_like(y)
    grads = torch.autograd.grad(y, [x, wl, bl, wr], go)
    ref, leaves = _ref(x, ei, wl, bl, wr, mean)
    rgrads = torch.autograd.grad(ref, leaves, go.double().cpu())
    assert _rel(y, ref) < 2e-5
    for name, a, b in zip(("x", "wl", "bl", "wr"), grads, rgrads):
        assert _rel(a, b) < 5e-5, name


def _workload_batch(workload, graphs=64):
    from hydragnn_b200.synthetic import WORKLOADS, add_rel_pe, make_samples
    w = WORKLOADS[workload]
    b = make_samples(workload, graphs).to("cuda")
    b._num_graphs = graphs
    b = hb.get_radius_graph(w["radius"], w["max_neighbours"])(b)
    return add_rel_pe(b) if w.get("pe_dim") else b


def _no_dropout(m):
    for sub in m.modules():
        if isinstance(sub, torch.nn.Dropout):
            sub.p = 0.0
        if hasattr(sub, "dropout") and isinstance(sub.dropout, float):
            sub.dropout = 0.0
    return m


@pytest.mark.parametrize("workload,overrides", [("ogb_sage", {}), ("ogb_mfc", {}), ("ogb_sage_gps", {}),
                                                ("ogb_mfc", {"max_neighbours": 150})])
@pytest.mark.parametrize("precision", ["fp32", "bf16"])
def test_training_step_against_the_fp64_oracle(workload, overrides, precision):
    """One training step at the workload's shapes (train-mode BatchNorm, dropout off): the engine's loss and every parameter
    gradient against the oracle stack in fp64 on the CPU with the same parameters, then one SGD step on both and the loss after
    it.  max_neighbours 150 gives 151 weight groups, more than the fused kernel takes: that model runs the composed path."""
    from hydragnn_b200.synthetic import ARCH
    from oracle.sage import MFCStackOracle, SAGEStackOracle
    arch = dict(ARCH[workload], **overrides)
    b = _workload_batch(workload)
    m = _no_dropout(hb.create.set_precision(hb.create_model(**arch), precision)).train()
    cls = SAGEStackOracle if arch["mpnn_type"] == "SAGE" else MFCStackOracle
    o = cls(**{k: v for k, v in arch.items() if k != "mpnn_type"}, dropout=0.0)
    o.load_state_dict(m.state_dict(), strict=True)
    o = o.double().train()

    class _D:
        pass
    d = _D()
    for key in ("x", "pe", "batch", "edge_index"):
        v = getattr(b, key, None)
        if v is not None:
            setattr(d, key, v.detach().cpu().double() if v.is_floating_point() else v.cpu())
    value, hi = b.y.view(-1), [torch.arange(b.y.shape[0], device="cuda")]
    tol = 1e-4 if precision == "fp32" else 2e-2
    lr = 0.05

    def step(model, data, val, idx):
        loss, _ = model.loss(model(data), val, idx)
        grads = torch.autograd.grad(loss, list(model.parameters()), allow_unused=True)
        with torch.no_grad():
            for p, g in zip(model.parameters(), grads):
                if g is not None:
                    p -= lr * g
        return loss.detach(), grads

    le, ge = step(m, b, value, hi)
    lo, go = step(o, d, value.cpu().double(), [h.cpu() for h in hi])
    assert abs(float(le) - float(lo)) <= tol * abs(float(lo)), (float(le), float(lo))
    # a conv bias in front of a BatchNorm has a gradient of zero up to rounding: errors are measured against the largest norm
    floor = 1e-3 * max(float(g.norm()) for g in go if g is not None)
    by_name = {name: g for (name, _), g in zip(o.named_parameters(), go)}        # the two register some modules in another order
    for (name, _), a in zip(m.named_parameters(), ge):
        c = by_name[name]
        if c is None:
            assert a is None or not a.any(), name
            continue
        err = float((a.double().cpu() - c).norm()) / max(float(c.norm()), floor)
        assert err < 10 * tol, (name, err)
    with torch.no_grad():
        after_e, _ = m.loss(m(b), value, hi)
        after_o, _ = o.loss(o(d), value.cpu().double(), [h.cpu() for h in hi])
    assert abs(float(after_e) - float(after_o)) <= 10 * tol * abs(float(after_o)), (float(after_e), float(after_o))
