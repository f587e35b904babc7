"""PNA on the GPU: the fused PNAConv kernels (hgb_pna_conv_{fwd,bwd}) against the fp64 restatement of conv_reference.py, the raw C-ABI,
the fused path against the composed one, and the engine's PNAStack against models_pna.pt (the reference's own PNAStack.py +
Base.py + gps.py, PyG's PNAConv restated in oracle/pna.py).

Kernel cases: widths F in {1, 5, 50, 55, 64, 200} (scalar and float4 paths, widths that are not multiples of 4 or 32), edge
attribute widths D in {0, 1, 3, 16} (all three register capacities), on a graph with runs of isolated nodes, a target of
in-degree 1000, targets of in-degree 1 and 2 and shuffled edge ids.  Forward to rel-L2 1e-5, every backward output on its own.
With dyadic inputs fp32 is exact, so ties are real: the first edge in CSR order must win bit for bit, and the fused kernel must
equal hgb_pna_aggregate_fwd on the materialised messages bit for bit.

At the benchmark shapes (eam_pna: 10 layers at F = 50 with a 1-wide edge attribute; ogb_pna: 6 layers at F = 55) one training
step is checked against the CPU oracle stack of oracle/pna.py in fp64, on edges built by the oracle's own radius graph:
in fp32 and under precision "bf16" (TF32 Linears); and the captured GraphedTrainStep must reproduce the eager steps."""
import copy
import math

import pytest
import torch

pytestmark = pytest.mark.gpu

import hydragnn_b200 as hb  # noqa: E402
from hydragnn_b200 import _lib, ops  # noqa: E402
from hydragnn_b200.ops import _p, _stream  # noqa: E402
from oracle.pna import PNAStackOracle  # noqa: E402
from oracle.tf32 import tf32_linears  # noqa: E402
from conv_reference import pna_bwd as _ref_bwd, pna_fwd as _ref_fwd  # noqa: E402
from stack_support import _batch, _bench_batch, _errors, _graph, _oracle_step, _train_step, golden_engine, rel_l2  # noqa: E402

DEV = "cuda"
CASES = ["pna_graph_noedge", "pna_node_edge_len", "pna_multihead_h5", "pna_gps", "pna_add_pool_edge3"]


def _inputs(n, e, f, d, seed, dyadic=False):
    g = torch.Generator().manual_seed(seed)
    if dyadic:      # small multiples of 1/4: every sum below is exact in fp32 -> exact ties
        r = lambda *s: torch.randint(-4, 5, s, generator=g).float() * 0.25          # noqa: E731
    else:
        r = lambda *s: torch.randn(*s, generator=g)                                  # noqa: E731
    pq, c = r(n, 2 * f), r(f)
    ea, mt = (r(e, d), r(d, f) * 0.5) if d else (None, None)
    return [t.to(DEV) if t is not None else None for t in (pq, ea, mt, c)]


@pytest.mark.parametrize("d", [0, 1, 3, 16])
@pytest.mark.parametrize("f", [1, 5, 50, 55, 64, 200])
def test_pna_conv_kernels_match_fp64(f, d):
    ei, n = _graph()
    plan = ops.EdgePlan(ei, n)
    pq, ea, mt, c = _inputs(n, ei.shape[1], f, d, seed=10 * f + d)
    agg, amin, amax = ops.raw_pna_conv_fwd(pq, ea, mt, c, plan)
    ragg, ramin, ramax, h = _ref_fwd(pq, ea, mt, c, ei, n)
    err = {"agg": rel_l2(agg, ragg)}
    for k, name in enumerate(("mean", "min", "max")):
        err[name] = rel_l2(agg[:, k * f:(k + 1) * f], ragg[:, k * f:(k + 1) * f])
    # std = sqrt(E[h^2] - E[h]^2) carries an fp32 error of a few 1e-7 E[h^2] in the variance (the messages themselves are
    # rounded, up to 17 terms each, before the sums): outside a band of that width
    # around the 1e-5 clamp the mask must agree with fp64, and the value must lie within the error that formula allows
    cnt = torch.bincount(ei[1], minlength=n).double().clamp(min=1)[:, None]
    ex2 = torch.zeros(n, f, dtype=torch.float64, device=DEV).index_add_(0, ei[1], h * h) / cnt
    var = ex2 - ragg[:, :f] ** 2
    near = (var - 1e-5).abs() <= 1e-6 * (1 + ex2)
    sd, rsd = agg[:, 3 * f:].double(), ragg[:, 3 * f:]
    err["std_mask_mismatch"] = int((((sd > 0) != (rsd > 0)) & ~near).sum())
    err["std_outside_bound"] = int((((sd - rsd).abs() > 4e-6 * ex2 / rsd.clamp(min=math.sqrt(1e-5)) + 1e-5 * rsd) & ~near).sum())
    # random inputs: the extremes are unique, so the ids agree with fp64 unless the runner-up lies within fp32 rounding
    err["amin_mismatch"] = int((amin.long() != ramin).sum())
    err["amax_mismatch"] = int((amax.long() != ramax).sum())
    g = torch.randn(n, 4 * f, device=DEV)
    g_pq, g_h, g_cm = ops.raw_pna_conv_bwd(g, pq, ea, mt, c, agg, amin, amax, plan)
    gh, gp, gq, gc, gmt, gea = _ref_bwd(g, agg.double(), amin, amax, h, ea, mt, ei, n)    # the backward given the forward's agg
    err.update(g_h=rel_l2(g_h, gh), g_p=rel_l2(g_pq[:, :f], gp), g_q=rel_l2(g_pq[:, f:], gq), g_c=rel_l2(g_cm[0], gc))
    if d:
        err["g_m"] = rel_l2(g_cm[1:], gmt)
    tol = {"std_mask_mismatch": 0, "std_outside_bound": 0, "amin_mismatch": n * f // 1000, "amax_mismatch": n * f // 1000}
    bad = {k: v for k, v in err.items() if v > tol.get(k, 1e-5)}
    assert not bad, err
    assert torch.all(amin[torch.bincount(ei[1], minlength=n) == 0] == -1)
    # through the autograd node: g_eattr = g_h M^T, the parameter terms as returned
    pq_, c_ = pq.clone().requires_grad_(True), c.clone().requires_grad_(True)
    ea_ = ea.clone().requires_grad_(True) if d else None
    mt_ = mt.clone().requires_grad_(True) if d else None
    out = ops.PnaConvFn.apply(pq_, ea_, mt_, c_, plan)
    assert torch.equal(out, agg)
    out.backward(g)
    assert rel_l2(pq_.grad, torch.cat([gp, gq], dim=1)) < 1e-5 and rel_l2(c_.grad, gc) < 1e-5
    if d:
        assert rel_l2(ea_.grad, gea) < 1e-5 and rel_l2(mt_.grad, gmt) < 1e-5


@pytest.mark.parametrize("d", [0, 3])
@pytest.mark.parametrize("f", [5, 64])
def test_pna_conv_dyadic_ties_and_materialised_aggregation_bit_exact(f, d):
    ei, n = _graph(seed=1)
    plan = ops.EdgePlan(ei, n)
    pq, ea, mt, c = _inputs(n, ei.shape[1], f, d, seed=7, dyadic=True)
    agg, amin, amax = ops.raw_pna_conv_fwd(pq, ea, mt, c, plan)
    ragg, ramin, ramax, h = _ref_fwd(pq, ea, mt, c, ei, n)
    assert torch.equal(amin.long(), ramin) and torch.equal(amax.long(), ramax)          # first in CSR order wins every tie
    assert torch.equal(agg[:, f:3 * f].double(), ragg[:, f:3 * f])
    # the exact messages through the unfused aggregator: identical bits, ids included
    m = h.float().contiguous()
    assert torch.equal(m.double(), h)
    out = torch.empty(n, 4 * f, device=DEV)
    a1, a2 = torch.empty(n, f, dtype=torch.int32, device=DEV), torch.empty(n, f, dtype=torch.int32, device=DEV)
    _lib.call("hgb_pna_aggregate_fwd", _p(m), _p(plan.by_col.rowptr), _p(plan.by_col.perm), n, f, _p(out), _p(a1), _p(a2), _stream())
    assert torch.equal(out, agg) and torch.equal(a1, amin) and torch.equal(a2, amax)


def test_pna_conv_all_equal_segments_mask_std_and_its_gradient():
    ei, n = _graph(seed=2)
    plan = ops.EdgePlan(ei, n)
    f = 8
    pq, _, _, c = _inputs(n, ei.shape[1], f, 0, seed=3, dyadic=True)
    pq[:, f:] = 0.0                                    # Q = 0: every message of a segment is P[i] + c
    agg, amin, amax = ops.raw_pna_conv_fwd(pq, None, None, c, plan)
    assert torch.all(agg[:, 3 * f:] == 0)
    g = torch.randn(n, 4 * f, device=DEV)
    g_pq, g_h, _ = ops.raw_pna_conv_bwd(g, pq, None, None, c, agg, amin, amax, plan)
    _, _, _, h = _ref_fwd(pq, None, None, c, ei, n)
    gh = _ref_bwd(g, agg.double(), amin, amax, h, None, None, ei, n)[0]                 # no std term anywhere
    assert rel_l2(g_h, gh) < 1e-6


def test_pna_conv_is_deterministic():
    ei, n = _graph(seed=4)
    plan = ops.EdgePlan(ei, n)
    for f, d in ((55, 1), (64, 16)):
        pq, ea, mt, c = _inputs(n, ei.shape[1], f, d, seed=5)
        g = torch.randn(n, 4 * f, device=DEV)
        r1 = ops.raw_pna_conv_fwd(pq, ea, mt, c, plan)
        b1 = ops.raw_pna_conv_bwd(g, pq, ea, mt, c, *r1, plan)
        r2 = ops.raw_pna_conv_fwd(pq, ea, mt, c, plan)
        b2 = ops.raw_pna_conv_bwd(g, pq, ea, mt, c, *r2, plan)
        assert all(torch.equal(a, b) for a, b in zip(r1 + b1, r2 + b2))


def test_pna_conv_raw_abi_errors_and_empty_sizes():
    n, f = 10, 4
    pq = torch.randn(n, 2 * f, device=DEV)
    c = torch.zeros(f, device=DEV)
    rowptr = torch.zeros(n + 1, dtype=torch.int32, device=DEV)
    src = torch.zeros(1, dtype=torch.int32, device=DEV)
    out = torch.full((n, 4 * f), float("nan"), device=DEV)
    a1, a2 = torch.empty(n, f, dtype=torch.int32, device=DEV), torch.empty(n, f, dtype=torch.int32, device=DEV)
    ea, mt = torch.zeros(1, 17, device=DEV), torch.zeros(17, f, device=DEV)
    before = _lib.launch_count()
    for args in ((_p(pq), _p(rowptr), None, _p(src), _p(ea), 17, _p(mt), _p(c), n, f),        # d > 16
                 (_p(pq), _p(rowptr), None, _p(src), None, 0, None, _p(c), n, 0),             # f = 0
                 (None, _p(rowptr), None, _p(src), None, 0, None, _p(c), n, f),               # no pq
                 (_p(pq), _p(rowptr), None, _p(src), None, 2, None, _p(c), n, f)):            # d > 0 without attributes
        with pytest.raises(RuntimeError, match="pna_conv_fwd"):
            _lib.call("hgb_pna_conv_fwd", *args, _p(out), _p(a1), _p(a2), _stream())
    assert _lib.launch_count() == before
    assert _lib.query("hgb_pna_conv_workspace_bytes", f, 17) == -1
    # e = 0: every segment empty -> zeros and id -1; the backward gives zero gradients
    _lib.call("hgb_pna_conv_fwd", _p(pq), _p(rowptr), None, _p(src), None, 0, None, _p(c), n, f, _p(out), _p(a1), _p(a2), _stream())
    assert torch.all(out == 0) and torch.all(a1 == -1) and torch.all(a2 == -1)
    g = torch.randn(n, 4 * f, device=DEV)
    g_p = torch.full((n, f), float("nan"), device=DEV)
    g_cm = torch.full((1, f), float("nan"), device=DEV)
    ws = torch.empty(_lib.query("hgb_pna_conv_workspace_bytes", f, 0), dtype=torch.uint8, device=DEV)
    _lib.call("hgb_pna_conv_bwd", _p(g), _p(pq), _p(rowptr), None, _p(src), None, 0, None, _p(c), _p(out), _p(a1), _p(a2), n, f,
              _p(g_p), f, _p(src), _p(g_cm), _p(ws), _stream())
    assert torch.all(g_p == 0) and torch.all(g_cm == 0)
    # n = 0: nothing to do, but the parameter sums are still written (zero)
    g_cm.fill_(float("nan"))
    _lib.call("hgb_pna_conv_bwd", _p(g), _p(pq), _p(rowptr), None, _p(src), None, 0, None, _p(c), _p(out), _p(a1), _p(a2), 0, f,
              _p(g_p), f, _p(src), _p(g_cm), _p(ws), _stream())
    assert torch.all(g_cm == 0)
    torch.cuda.synchronize()


@pytest.mark.parametrize("name", CASES)
def test_pna_stack_matches_reference_golden(golden_dir, name):
    c = torch.load(golden_dir + "/models_pna.pt")[name]
    m = golden_engine("PNA", c).eval()
    _lib.trace_begin()
    with torch.no_grad():
        pred = m(_batch(c["inputs"]))
    calls = {t[0] for t in _lib.trace_end()}
    assert "hgb_pna_conv_fwd" in calls                               # the fused conv ran (edge widths here are <= 16)
    for a, b in zip(pred, c["pred_eval"]):
        assert rel_l2(a.cpu(), b) < 1e-5
    pred, loss = _train_step(m, c)
    for a, b in zip(pred, c["pred_train"]):
        assert rel_l2(a.detach().cpu(), b) < 1e-5
    torch.testing.assert_close(loss.detach().cpu(), c["loss"], rtol=1e-5, atol=1e-7)
    gmax = max(float(g.abs().max()) for g in c["grads"].values() if g is not None)
    for n, p in m.named_parameters():
        ref = c["grads"][n]
        if ref is not None:
            torch.testing.assert_close(p.grad.cpu(), ref, rtol=1e-3, atol=1e-6 * gmax, msg=lambda s, n=n: n + ": " + s)
    sd = m.state_dict()
    for k, v in c["state_after"].items():
        torch.testing.assert_close(sd[k].cpu(), v, rtol=1e-5, atol=1e-7)


@pytest.mark.parametrize("name", CASES)
def test_pna_fused_path_equals_composed_path(golden_dir, name):
    c = torch.load(golden_dir + "/models_pna.pt")[name]
    res = []
    for composed in (False, True):
        m = golden_engine("PNA", c)
        m.force_higher_order = composed
        pred, loss = _train_step(m, c)
        res.append(([p.detach() for p in pred], {n: p.grad.clone() for n, p in m.named_parameters() if p.grad is not None}))
    (pf, gf), (pc, gc) = res
    for a, b in zip(pf, pc):
        assert rel_l2(a, b) < 1e-5
    assert gf.keys() == gc.keys()
    gmax = max(float(g.abs().max()) for g in gc.values())
    for n in gf:
        torch.testing.assert_close(gf[n], gc[n], rtol=1e-3, atol=1e-6 * gmax, msg=lambda s, n=n: n + ": " + s)


@pytest.mark.parametrize("precision", ["fp32", "bf16"])
@pytest.mark.parametrize("name,graphs,hidden", [("eam_pna", 64, None), ("ogb_pna", 128, None), ("eam_pna", 64, 64)])
def test_pna_training_step_at_benchmark_shape_matches_oracle(name, graphs, hidden, precision):
    """One training step against the oracle stack in fp64.  The model is not well conditioned at these shapes: the min / max
    aggregators pick one edge per (node, channel), and where two messages lie within rounding of each other a lower-precision
    run may pick the other one, which moves the gradient of the layers below; ten layers of batch statistics amplify the rest.
    So the reference's arithmetic is also run at the engine's precision -- the oracle in fp32, and for precision "bf16" the fp32
    oracle with every Linear rounded to TF32 (``tf32_linears``) -- and measured against fp64.  The engine must be no further from
    fp64 than twice that, and never further than the fixed bounds: fp32 outputs rel-L2 1e-5, gradients 1e-4, the loss and the
    BatchNorm running statistics 1e-5; TF32 2e-2 everywhere.  (The TF32 gradient of the 10-layer eam model is about 0.3 from
    fp64 for the emulated reference as well: that is the precision mode, not the kernels.)  At the examples' widths (50, 55)
    the Linears are not tensor-core shapes, so precision "bf16" changes nothing there; the width-64 case puts the per-node
    [P | Q] Linear, the folded post Linear and the heads on the TF32 tensor cores, ahead of the std aggregator."""
    b, kw = _bench_batch(name, graphs)
    if hidden is not None:
        kw["hidden_dim"] = hidden
    em = hb.set_precision(hb.create_model(**kw), precision)
    state = {k: v.detach().cpu().clone() for k, v in em.state_dict().items()}
    ref64 = _oracle_step(PNAStackOracle, kw, state, b, torch.float64)
    if precision == "fp32":
        ref32 = _errors(*_oracle_step(PNAStackOracle, kw, state, b, torch.float32), ref64, bn_stats=True)
    else:
        with tf32_linears():
            ref32 = _errors(*_oracle_step(PNAStackOracle, kw, state, b, torch.float32), ref64, bn_stats=True)
    n_atoms, mean_deg = b.pos.shape[0], float(torch.bincount(b.edge_index[1]).float().mean())
    assert n_atoms > 2000 and mean_deg > 8                                    # thousands of atoms, realistic in-degrees
    em.train()
    d = b.clone().to(DEV)
    d._num_graphs = graphs
    _lib.trace_begin()
    pred = em(d)
    loss, _ = em.loss(pred, d.y, [torch.arange(b.y.shape[0], device=DEV)])
    loss.backward()
    calls = {t[0] for t in _lib.trace_end()}
    assert "hgb_pna_conv_fwd" in calls and "hgb_pna_conv_bwd" in calls
    if precision == "bf16" and hidden == 64:
        assert any(c.startswith("hgb_tc_linear") for c in calls), sorted(calls)
    eng = _errors([p.detach() for p in pred], loss.detach(), {n: p.grad for n, p in em.named_parameters()}, em.state_dict(), ref64, bn_stats=True)
    if precision == "fp32":
        bound = {"pred": max(1e-5, 2 * ref32["pred"]), "grad": max(1e-4, 2 * ref32["grad"]), "loss": 1e-5, "bn_stats": 1e-5}
    else:
        bound = {k: max(2e-2, 2 * v) for k, v in ref32.items()}
    assert all(eng[k] <= bound[k] for k in eng), {"engine": eng, "oracle_same_precision": ref32, "bound": bound}


def test_pna_graphed_train_step_equals_eager_steps():
    """The captured step (BatchNorm statistics updated inside the graph, fused PNA kernels, edge attributes) replays the eager
    sequence: same losses, parameters and running statistics."""
    name, graphs = "eam_pna", 64
    b, kw = _bench_batch(name, graphs)
    b = b.to(DEV)
    b._num_graphs = graphs
    model = hb.get_distributed_model(hb.create_model(**kw))
    model2 = copy.deepcopy(model)
    opt = hb.FlatAdamW(model, lr=1e-3)
    losses = [float(hb.train_step(model, opt, b)[0]) for _ in range(10)]
    assert losses[-1] < losses[0]
    opt2 = hb.FlatAdamW(model2, lr=1e-3)
    gs = hb.GraphedTrainStep(model2, opt2, b.clone(), warmup=3)
    glosses = [float(gs.run()) for _ in range(7)]
    torch.cuda.synchronize()
    assert abs(glosses[-1] - losses[-1]) <= 1e-5 * abs(losses[-1]), (glosses, losses)
    s1, s2 = model.module.state_dict(), model2.module.state_dict()
    assert int(s2["feature_layers.0.module.num_batches_tracked"]) == 10
    for k in s1:
        if s1[k].is_floating_point():
            torch.testing.assert_close(s2[k], s1[k], rtol=1e-5, atol=1e-7, msg=lambda m, k=k: k + ": " + m)
        else:
            assert torch.equal(s2[k], s1[k]), k
