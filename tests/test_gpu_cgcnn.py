"""CGCNN on the GPU: the fused kernels (hgb_cgconv_{fwd,bwd}) against an fp64 restatement written here, the raw C-ABI, the
fused path against the composed one, the engine's CGCNNStack against models_cgcnn.pt (the reference's own CGCNNStack.py +
Base.py + gps.py), and one training step at the mp_cgcnn / mp_cgcnn_gps shapes against the fp64 oracle of oracle/cgcnn.py.

Kernel graph (stack_support._graph): runs of isolated nodes, a target of in-degree 1000, targets of in-degree 1 and 2, random
sources (self loops and duplicate pairs included) and shuffled edge ids.  Some targets and sources carry pre-activations above
+20 (softplus's linear branch) and below -20 (sigmoid near 0).  Every output of the backward is checked on its own."""
import copy

import pytest
import torch

pytestmark = pytest.mark.gpu

import hydragnn_b200 as hb  # noqa: E402
from hydragnn_b200 import _lib, ops  # noqa: E402
from hydragnn_b200.ops import _p, _stream  # noqa: E402
from oracle.cgcnn import CGCNNStackOracle  # noqa: E402
from oracle.tf32 import tf32_linears  # noqa: E402
from conv_reference import cgconv as _ref  # noqa: E402
from stack_support import (_batch, _bench_batch, _errors, _graph, _oracle_step, _zero_dropout,  # noqa: E402
                           check_golden_case, engine_case, golden_engine, grad_close, rel_l2)

DEV = "cuda"
CASES = ["cgcnn_graph_edge0", "cgcnn_node_edge_len", "cgcnn_add_pool_edge3", "cgcnn_multihead", "cgcnn_mlp_per_node", "cgcnn_gps",
         "cgcnn_gps_edge2", "cgcnn_ci_width1"]


def _inputs(n, e, f, d, seed):
    g = torch.Generator().manual_seed(seed)
    pq = torch.randn(n, 4 * f, generator=g)
    hot = torch.randperm(n, generator=g)[:n // 10]
    pq[hot[: n // 20], f:2 * f] += 25.0                 # P_s: s above the softplus threshold at these targets
    pq[hot[n // 20:], 2 * f:3 * f] -= 25.0              # Q_f: f below -20 from these sources
    x = torch.randn(n, f, generator=g)
    cvec = torch.randn(2 * f, generator=g) * 0.5
    ea, mt = (torch.randn(e, d, generator=g), torch.randn(d, 2 * f, generator=g) * 0.5) if d else (None, None)
    return {k: (v.to(DEV) if v is not None else None) for k, v in dict(pq=pq, ea=ea, mt=mt, cvec=cvec, x=x).items()}


@pytest.mark.parametrize("d", [0, 1, 7, 16])
@pytest.mark.parametrize("f", [1, 2, 3, 8, 31, 32, 33, 64, 100, 128])
def test_cgconv_kernels_match_fp64(f, d):
    ei, n = _graph(seed=f * 17 + d)
    plan = ops.EdgePlan(ei, n)
    t = _inputs(n, ei.shape[1], f, d, seed=f + 100 * d)
    g_out = torch.randn(n, f, generator=torch.Generator().manual_seed(3)).to(DEV)
    out = ops.raw_cgconv_fwd(t["pq"], t["ea"], t["mt"], t["cvec"], t["x"], plan)
    g_pq, g_ea, g_par = ops.raw_cgconv_bwd(g_out, t["pq"], t["ea"], t["mt"], t["cvec"], plan)
    ref, rg = _ref(t, ei, g_out)
    assert rel_l2(out.cpu(), ref) < 1e-6
    iso = torch.cat([torch.arange(0, 7), torch.arange(8, 100), torch.arange(300, 400)])      # no incoming edge: out = x exactly
    assert torch.equal(out[iso], t["x"][iso])
    assert rel_l2(g_pq[:, :2 * f].cpu(), rg["pq"][:, :2 * f]) < 1e-5      # g_P
    assert rel_l2(g_pq[:, 2 * f:].cpu(), rg["pq"][:, 2 * f:]) < 1e-5      # g_Q: the by-source sum of g_h
    assert rel_l2(g_par[0].cpu(), rg["cvec"]) < 1e-5
    if d:
        assert rel_l2(g_ea.cpu(), rg["ea"]) < 1e-5
        assert rel_l2(g_par[1:].cpu(), rg["mt"]) < 1e-5
    else:
        assert g_ea is None and g_par.shape == (1, 2 * f)


def test_cgconv_is_deterministic_and_data_only_backward_equals_full():
    ei, n = _graph(seed=4)
    plan = ops.EdgePlan(ei, n)
    t = _inputs(n, ei.shape[1], 33, 7, seed=5)
    g = torch.randn(n, 33, device=DEV)
    args = (t["pq"], t["ea"], t["mt"], t["cvec"])
    outs = []
    for _ in range(2):
        outs.append([ops.raw_cgconv_fwd(*args, t["x"], plan)] + list(ops.raw_cgconv_bwd(g, *args, plan)))
    assert all(torch.equal(a, b) for a, b in zip(*outs))
    g_pq, g_ea, g_par = ops.raw_cgconv_bwd(g, *args, plan, need_params=False)
    assert g_par is None and torch.equal(g_pq, outs[0][1]) and torch.equal(g_ea, outs[0][2])
    # through autograd: under only_data_grads the parameter gradients are not computed
    leaves = [v.clone().requires_grad_(True) for v in (t["pq"], t["ea"], t["mt"], t["cvec"], t["x"])]
    out = ops.CgConvFn.apply(*leaves, plan)
    with ops.only_data_grads():
        gd = torch.autograd.grad(out, leaves, g, retain_graph=True, allow_unused=True)
    gf = torch.autograd.grad(out, leaves, g, allow_unused=True)
    assert gd[2] is None and gd[3] is None and gf[2] is not None and gf[3] is not None
    for a, b in zip((gd[0], gd[1], gd[4]), (gf[0], gf[1], gf[4])):
        assert torch.equal(a, b)
    assert ops.cgconv_supported(128, 16) and ops.cgconv_supported(1, 0)
    assert not ops.cgconv_supported(129, 0) and not ops.cgconv_supported(0, 0) and not ops.cgconv_supported(8, 17)
    assert _lib.query("hgb_cgconv_workspace_bytes", 129, 0) == -1


def test_cgconv_raw_abi_errors_and_empty_sizes():
    n, f, e = 10, 4, 3
    z = lambda *s: torch.zeros(*s, device=DEV)                                          # noqa: E731
    pq, cvec, x = z(n, 4 * f), z(2 * f), torch.randn(n, f, device=DEV)
    rowptr = torch.zeros(n + 1, dtype=torch.int32, device=DEV)
    src = torch.zeros(e, dtype=torch.int32, device=DEV)
    out = torch.full((n, f), float("nan"), device=DEV)
    base = [_p(pq), _p(rowptr), None, _p(src), None, 0, None, _p(cvec), _p(x), n, 0, f]
    before = _lib.launch_count()
    # f = 0, f > 128, d > 16, n < 0, e < 0, no pq, no src with edges, d > 0 without M
    for i, v in ((11, 0), (11, 129), (5, 17), (9, -1), (10, -1), (0, None), (10, e), (5, 2)):
        bad = list(base)
        bad[i] = v
        if i == 10 and v == e:
            bad[3] = None
        with pytest.raises(RuntimeError, match="cgconv_fwd"):
            _lib.call("hgb_cgconv_fwd", *bad, _p(out), _stream())
    _lib.call("hgb_cgconv_fwd", *base, _p(out), _stream())                               # e = 0: out = x, no kernel
    assert torch.equal(out, x)
    g = torch.randn(n, f, device=DEV)
    g_p = torch.full((n, 4 * f), float("nan"), device=DEV)
    gpar = torch.full((2 * f,), float("nan"), device=DEV)
    ws = torch.empty(_lib.query("hgb_cgconv_workspace_bytes", f, 0), dtype=torch.uint8, device=DEV)
    bw = [_p(g)] + base[:8] + [n, 0, f, _p(g_p), 4 * f, None, None, _p(gpar), _p(ws), _stream()]
    with pytest.raises(RuntimeError, match="ldgp"):
        _lib.call("hgb_cgconv_bwd", *(bw[:13] + [f] + bw[14:]))
    _lib.call("hgb_cgconv_bwd", *bw)
    assert torch.all(g_p[:, :2 * f] == 0) and torch.all(gpar == 0)
    gpar.fill_(float("nan"))
    bw[9] = 0                                                                            # n = 0: the parameter sums are written
    _lib.call("hgb_cgconv_bwd", *bw)
    assert torch.all(gpar == 0)
    torch.cuda.synchronize()
    assert _lib.launch_count() == before
    # the autograd wrapper without edges: out = x, zero gradients of the right shapes, no library call
    plan = ops.EdgePlan(torch.empty(2, 0, dtype=torch.long, device=DEV), n)
    leaves = [v.clone().requires_grad_(True) for v in (pq, torch.zeros(0, 2, device=DEV), z(2, 2 * f), cvec, x)]
    _lib.trace_begin()
    o = ops.CgConvFn.apply(*leaves, plan)
    gr = torch.autograd.grad(o, leaves, g)
    assert not [c for c in _lib.trace_end() if c[0].startswith("hgb_cgconv")]
    assert torch.equal(o, x) and torch.equal(gr[4], g)
    assert all(a.shape == b.shape and not a.any() for a, b in zip(gr[:4], leaves[:4]))


@pytest.mark.parametrize("name", CASES)
def test_cgcnn_stack_matches_reference_golden(golden_dir, name):
    c = torch.load(golden_dir + "/models_cgcnn.pt")[name]
    check_golden_case(golden_engine("CGCNN", c), c, lambda: _batch(c["inputs"]), pred=(1e-5, 1e-5), loss=(1e-5, 1e-7),
                      grads=grad_close(1e-3, 1e-5), eval_kernels=["hgb_cgconv_fwd"])


@pytest.mark.parametrize("name", CASES)
def test_cgcnn_fused_path_equals_composed_path(golden_dir, name):
    c = torch.load(golden_dir + "/models_cgcnn.pt")[name]
    composed = golden_engine("CGCNN", c)
    composed.force_higher_order = True
    _lib.trace_begin()
    ref = engine_case(composed, c)
    assert "hgb_cgconv_bwd" not in {t[0] for t in _lib.trace_end()}
    fused = golden_engine("CGCNN", c)
    _lib.trace_begin()
    check_golden_case(fused, ref, lambda: _batch(c["inputs"]), pred=(1e-5, 1e-5), loss=(1e-5, 0), grads=grad_close(1e-3, 1e-5))
    assert "hgb_cgconv_bwd" in {t[0] for t in _lib.trace_end()}
    assert {n for n, p in fused.named_parameters() if p.grad is not None} == {n for n, g in ref["grads"].items() if g is not None}


@pytest.mark.parametrize("precision", ["fp32", "bf16"])
@pytest.mark.parametrize("name,graphs", [("mp_cgcnn", 128), ("mp_cgcnn_gps", 64)])
def test_cgcnn_training_step_at_benchmark_shape_matches_oracle(name, graphs, precision):
    """One train-mode step against the oracle stack in fp64, with the bounds of
    test_pna_training_step_at_benchmark_shape_matches_oracle: the reference's arithmetic is also run at the engine's precision
    (fp32, or fp32 with TF32 Linears for precision "bf16") and the engine must be no further from fp64 than twice that, or than
    fixed bounds (fp32: loss 1e-5, outputs 1e-4, gradients 1e-3; TF32: 2e-2)."""
    b, kw = _bench_batch(name, graphs)
    kw = {k: v for k, v in kw.items() if k not in ("pna_deg", "radius", "max_neighbours")}
    em = hb.set_precision(hb.create_model(**kw), precision)
    state = {k: v.detach().cpu().clone() for k, v in em.state_dict().items()}
    ref64 = _oracle_step(CGCNNStackOracle, kw, state, b, torch.float64)
    if precision == "fp32":
        ref32 = _errors(*_oracle_step(CGCNNStackOracle, kw, state, b, torch.float32), ref64)
    else:
        with tf32_linears():
            ref32 = _errors(*_oracle_step(CGCNNStackOracle, kw, state, b, torch.float32), ref64)
    em.train()
    _zero_dropout(em)
    d = b.clone().to(DEV)
    d._num_graphs = graphs
    _lib.trace_begin()
    pred = em(d)
    loss, _ = em.loss(pred, d.y, [torch.arange(b.y.shape[0], device=DEV)])
    loss.backward()
    calls = {t[0] for t in _lib.trace_end()}
    assert "hgb_cgconv_fwd" in calls and "hgb_cgconv_bwd" in calls
    eng = _errors([p.detach() for p in pred], loss.detach(), {n: p.grad for n, p in em.named_parameters()}, em.state_dict(), ref64)
    if precision == "fp32":
        bound = {"pred": max(1e-4, 2 * ref32["pred"]), "grad": max(1e-3, 2 * ref32["grad"]), "loss": max(1e-5, 2 * ref32["loss"])}
    else:
        bound = {k: max(2e-2, 2 * v) for k, v in ref32.items()}
    assert all(eng[k] <= bound[k] for k in eng), {"engine": eng, "oracle_same_precision": ref32, "bound": bound}


@pytest.mark.parametrize("name", ["mp_cgcnn", "mp_cgcnn_gps"])
def test_cgcnn_graphed_train_step_equals_eager_steps(name):
    graphs = 64
    b, kw = _bench_batch(name, graphs)
    kw = {k: v for k, v in kw.items() if k != "pna_deg"}
    b = b.to(DEV)
    b._num_graphs = graphs
    model = hb.get_distributed_model(_no_dropout(hb.create_model(**kw)))
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
    for k in s1:
        if s1[k].is_floating_point():
            torch.testing.assert_close(s2[k], s1[k], rtol=1e-5, atol=1e-7, msg=lambda m, k=k: k + ": " + m)


def _no_dropout(m):
    _zero_dropout(m)
    return m
