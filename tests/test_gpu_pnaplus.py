"""PNAPlus on the GPU: the fused kernels (hgb_pnaplus_conv_{fwd,bwd}) against the fp64 restatement of conv_reference.py, the raw C-ABI,
the fused path against the composed one, the engine's PNAPlusStack against models_pnaplus.pt (the reference's own
PNAPlusStack.py + Base.py + gps.py), forces, and one training step at the lj_pnaplus / ogb_pnaplus shapes against the fp64
oracle of oracle/pnaplus.py.

Kernel graph: runs of isolated nodes, a target of in-degree 1000, targets of in-degree 1 and 2, shuffled edge ids; every
target's first edge lies past the cutoff (its message is exactly 0, the other messages are continuous, so there are no ties).
Every output of the backward is checked on its own, g_dist and g_freq included."""
import copy

import pytest
import torch

pytestmark = pytest.mark.gpu

import hydragnn_b200 as hb  # noqa: E402
from hydragnn_b200 import _lib, ops  # noqa: E402
from hydragnn_b200.ops import _p, _stream  # noqa: E402
from oracle.pnaplus import PNAPlusStackOracle  # noqa: E402
from oracle.tf32 import tf32_linears  # noqa: E402
from conv_reference import pnaplus_agg  # noqa: E402
from stack_support import (_batch, _bench_batch, _errors, _graph, _oracle_step, check_golden_case, check_grads, engine_case,  # noqa: E402
                           golden_engine, grad_close, rel_l2)

DEV = "cuda"
RADIUS, EXPO = 2.0, 5
CASES = ["pnaplus_graph_noedge", "pnaplus_node_edge_len", "pnaplus_multihead_h5", "pnaplus_gps", "pnaplus_edge_dim0",
         "pnaplus_add_pool_edge3", "pnaplus_conv_head"]


def _inputs(ei, n, f, d, r, seed):
    g = torch.Generator().manual_seed(seed)
    e = ei.shape[1]
    dist = torch.rand(e, generator=g) * 0.9 * RADIUS + 0.05 * RADIUS
    first = torch.full((n,), e, dtype=torch.long).scatter_reduce(0, ei[1].cpu(), torch.arange(e), reduce="amin")
    dist[first[first < e]] = 1.3 * RADIUS                                          # one edge per target past the cutoff
    t = dict(pq=torch.randn(n, 2 * f, generator=g), dist=dist, freq=torch.pi * torch.arange(1, r + 1) + 0.1 * torch.randn(r, generator=g),
             wr=torch.randn(f, r, generator=g) * 0.5, br=torch.randn(f, generator=g) * 0.5, wl=torch.randn(f, r, generator=g) * 0.5,
             mr=torch.randn(f, f, generator=g) / f ** 0.5, cvec=torch.randn(f, generator=g),
             eattr=torch.randn(e, d, generator=g) if d else None, mat=torch.randn(d, f, generator=g) * 0.5 if d else None)
    return t


NAMES = ["pq", "dist", "eattr", "freq", "wr", "br", "wl", "mr", "mat", "cvec"]


@pytest.mark.parametrize("f,d,r", [(1, 0, 1), (5, 1, 5), (32, 0, 5), (32, 3, 16), (55, 16, 5), (64, 0, 16), (64, 16, 1)])
def test_pnaplus_conv_kernels_match_fp64(f, d, r):
    ei, n = _graph(seed=1)
    plan = ops.EdgePlan(ei, n)
    t = _inputs(ei, n, f, d, r, seed=f * 100 + d * 10 + r)
    t64 = {k: (v.double().requires_grad_(True) if v is not None else None) for k, v in t.items()}
    ref = pnaplus_agg(t64, ei, n, RADIUS, EXPO)
    gout = torch.randn(ref.shape, generator=torch.Generator().manual_seed(3), dtype=torch.float64)
    want = torch.autograd.grad((ref * gout).sum(), [t64[k] for k in NAMES if t64[k] is not None])
    want = dict(zip([k for k in NAMES if t64[k] is not None], want))
    tg = {k: (v.to(DEV).requires_grad_(True) if v is not None else None) for k, v in t.items()}
    agg = ops.PnaPlusConvFn.apply(tg["pq"], tg["dist"], tg["eattr"], tg["freq"], tg["wr"], tg["br"], tg["wl"], tg["mr"], tg["mat"],
                                  tg["cvec"], RADIUS, EXPO, plan)
    assert rel_l2(agg.cpu(), ref.detach()) < 1e-5
    got = torch.autograd.grad((agg * gout.float().to(DEV)).sum(), [tg[k] for k in want])
    for k, g in zip(want, got):
        w = want[k]
        assert rel_l2(g.cpu(), w) < 1e-4, (k, rel_l2(g.cpu(), w))


def test_pnaplus_conv_is_deterministic_and_queries():
    ei, n = _graph(seed=4)
    plan = ops.EdgePlan(ei, n)
    t = {k: (v.to(DEV) if v is not None else None) for k, v in _inputs(ei, n, 55, 3, 5, seed=5).items()}
    args = [t[k] for k in NAMES] + [RADIUS, EXPO]
    g = torch.randn(n, 4 * 55, device=DEV)
    outs = []
    for _ in range(2):
        r1 = ops.raw_pnaplus_conv_fwd(*args, plan)
        outs.append(list(r1) + list(ops.raw_pnaplus_conv_bwd(g, *args, *r1, plan)))
    assert all(torch.equal(a, b) for a, b in zip(*outs))
    assert ops.pnaplus_conv_supported(64, 16, 16) and not ops.pnaplus_conv_supported(65, 5, 0)
    assert not ops.pnaplus_conv_supported(32, 17, 0) and not ops.pnaplus_conv_supported(32, 5, 17)
    assert _lib.query("hgb_pnaplus_conv_workspace_bytes", 65, 5, 0) == -1


def test_pnaplus_conv_raw_abi_errors_and_empty_sizes():
    n, f, r = 10, 4, 3
    z = lambda *s: torch.zeros(*s, device=DEV)                                          # noqa: E731
    pq, dist, freq, wr, br, wl, mr, c = z(n, 2 * f), z(1), z(r), z(f, r), z(f), z(f, r), z(f, f), z(f)
    rowptr = torch.zeros(n + 1, dtype=torch.int32, device=DEV)
    src = torch.zeros(1, dtype=torch.int32, device=DEV)
    out = torch.full((n, 4 * f), float("nan"), device=DEV)
    a1, a2 = torch.empty(n, f, dtype=torch.int32, device=DEV), torch.empty(n, f, dtype=torch.int32, device=DEV)
    base = [_p(pq), _p(dist), _p(rowptr), None, _p(src), None, 0, _p(freq), r, RADIUS, EXPO, _p(wr), _p(br), _p(wl), _p(mr), None,
            _p(c), n, f]
    before = _lib.launch_count()
    for i, v in ((18, 65), (8, 17), (9, 0.0), (0, None), (6, 2)):       # f > 64, r > 16, radius 0, no pq, d > 0 without attributes
        bad = list(base)
        bad[i] = v
        with pytest.raises(RuntimeError, match="pnaplus_conv_fwd"):
            _lib.call("hgb_pnaplus_conv_fwd", *bad, _p(out), _p(a1), _p(a2), _stream())
    assert _lib.launch_count() == before
    _lib.call("hgb_pnaplus_conv_fwd", *base, _p(out), _p(a1), _p(a2), _stream())         # e = 0: zeros and id -1
    assert torch.all(out == 0) and torch.all(a1 == -1) and torch.all(a2 == -1)
    g = torch.randn(n, 4 * f, device=DEV)
    g_p = torch.full((n, f), float("nan"), device=DEV)
    nparam = f + f * f + 2 * r * f + f + r
    gpar = torch.full((nparam,), float("nan"), device=DEV)
    ws = torch.empty(_lib.query("hgb_pnaplus_conv_workspace_bytes", f, r, 0), dtype=torch.uint8, device=DEV)
    bw = base[:16] + [_p(c), _p(out), _p(a1), _p(a2), n, f, _p(g_p), f, _p(pq), None, None, _p(gpar), _p(ws), _stream()]
    _lib.call("hgb_pnaplus_conv_bwd", _p(g), *bw)
    assert torch.all(g_p == 0) and torch.all(gpar == 0)
    gpar.fill_(float("nan"))
    bw[20] = 0                                                                             # n = 0: the sums are still written
    _lib.call("hgb_pnaplus_conv_bwd", _p(g), *bw)
    assert torch.all(gpar == 0)
    torch.cuda.synchronize()


def _before_batch_norm(name):
    """The biases of a conv's post Linear and last Linear shift every row alike ahead of a BatchNorm with batch statistics, which
    subtracts the mean: their gradients are 0 up to rounding in train mode (largest behind the 1-wide output of a conv head),
    so only their size is checked."""
    return name.endswith(("module_0.lin.bias", "module_0.post_nns.0.0.bias"))


def _grads(name, g, ref, gmax):
    if _before_batch_norm(name):
        assert float(g.abs().max()) <= 1e-3 * gmax and float(ref.abs().max()) <= 1e-3 * gmax, name
    else:
        grad_close(1e-3, 1e-6)(name, g, ref, gmax)


@pytest.mark.parametrize("name", CASES)
def test_pnaplus_stack_matches_reference_golden(golden_dir, name):
    c = torch.load(golden_dir + "/models_pnaplus.pt")[name]
    # every case is within the fused shapes (GPS: D = hidden = 16)
    check_golden_case(golden_engine("PNAPlus", c), c, lambda: _batch(c["inputs"]), pred=(1e-5, 1e-5), loss=(1e-5, 1e-7),
                      grads=_grads, eval_kernels=["hgb_pnaplus_conv_fwd"])


@pytest.mark.parametrize("name", CASES)
def test_pnaplus_fused_path_equals_composed_path(golden_dir, name):
    c = torch.load(golden_dir + "/models_pnaplus.pt")[name]
    composed = golden_engine("PNAPlus", c)
    composed.force_higher_order = True
    ref = engine_case(composed, c)
    fused = golden_engine("PNAPlus", c)
    check_golden_case(fused, ref, lambda: _batch(c["inputs"]), pred=(1e-5, 1e-5), loss=(1e-5, 0), grads=_grads)


def test_pnaplus_conv_head_with_edge_attributes_raises_before_any_launch(golden_dir):
    c = torch.load(golden_dir + "/models_pnaplus.pt")["pnaplus_conv_head"]
    m = hb.create_model(mpnn_type="PNAPlus", input_dim=1, hidden_dim=8, output_dim=[1], output_type=["node"],
                        output_heads=c["cfg"]["output_heads"], task_weights=[1.0], num_conv_layers=2, edge_dim=1, pna_deg=c["deg"],
                        num_radial=5, radius=3.0, envelope_exponent=5)
    d = _batch(c["inputs"])
    d.edge_attr = torch.ones(d.edge_index.shape[1], 1, device=DEV)
    before = _lib.launch_count()
    with pytest.raises(ValueError, match="conv-type node heads"):
        m(d)
    assert _lib.launch_count() == before


def test_pnaplus_mlip_matches_reference_golden_and_forces(golden_dir):
    """The MLIP case (eval mode): the loss through the composed any-order path against the reference's energy_force_loss with its
    second-order parameter gradients; the fused first-order path predicts the same forces as -autograd.grad on the composed one."""
    c = torch.load(golden_dir + "/models_pnaplus.pt")["pnaplus_mlip"]
    m = hb.create.EnhancedModelWrapper(golden_engine("PNAPlus", c), 1.0, 1.0, 1.0).eval()
    d = _batch(c["inputs"])
    d.pos.requires_grad_(True)
    m.model.force_higher_order = True
    pred = m(d)
    tot, tasks = m.energy_force_loss(pred, d)
    torch.testing.assert_close(float(tot), float(c["loss"]), rtol=1e-5, atol=0)
    grads = torch.autograd.grad(tot, list(m.model.parameters()), allow_unused=True)
    check_grads(c, {n: g for (n, _), g in zip(m.model.named_parameters(), grads)}, grad_close(1e-3, 1e-5))
    forces = {}
    for composed in (True, False):
        m.model.force_higher_order = composed
        d = _batch(c["inputs"])
        d.pos.requires_grad_(True)
        e = hb.stacks.graph_sum(m(d)[0], m.model.graph_index(d)[2])
        forces[composed] = -torch.autograd.grad(e.sum(), d.pos)[0]
    torch.testing.assert_close(forces[True].cpu(), c["forces"], rtol=1e-4, atol=1e-5)
    torch.testing.assert_close(forces[False], forces[True], rtol=1e-4, atol=1e-5)


@pytest.mark.parametrize("precision", ["fp32", "bf16"])
@pytest.mark.parametrize("name,graphs", [("lj_pnaplus", 96), ("ogb_pnaplus", 128)])
def test_pnaplus_training_step_at_benchmark_shape_matches_oracle(name, graphs, precision):
    """One train-mode step (graph or per-atom energy loss, no force term) against the oracle stack in fp64, with the bounds of
    test_pna_training_step_at_benchmark_shape_matches_oracle: the reference's arithmetic is also run at the engine's precision
    (fp32, or fp32 with TF32 Linears for precision "bf16") and the engine must be no further from fp64 than twice that, or than
    fixed bounds (fp32: loss 1e-5, outputs 1e-4, gradients 1e-3; TF32: 2e-2).  The LJ cells are jittered lattices: many messages
    of a target lie within rounding of each other, so min / max pick differently at lower precision.  The fp32 bounds are wider
    than PNA's because the engine's composed path, which runs none of the PNAPlus kernels, measured the same distance from fp64
    as the fused path on an H100 (ogb_pnaplus gradients 2.9e-4 composed, 3.0e-4 fused; lj_pnaplus outputs 3.3e-5 both), so it
    is not in the fused kernels; nor is it in the fp32 dense kernels, which tests/test_gpu_dense_kernels.py holds to their
    rounding bounds (about sqrt(k) u relative) at these widths.  Where the rest of the distance arises has not been traced."""
    b, kw = _bench_batch(name, graphs)
    kw = {k: v for k, v in kw.items() if k not in ("enable_interatomic_potential", "energy_weight", "energy_peratom_weight",
                                                   "force_weight")}
    if kw["output_type"] == ["node"]:
        b.y = torch.randn(b.pos.shape[0], 1, generator=torch.Generator().manual_seed(11))
    em = hb.set_precision(hb.create_model(**kw), precision)
    state = {k: v.detach().cpu().clone() for k, v in em.state_dict().items()}
    ref64 = _oracle_step(PNAPlusStackOracle, kw, state, b, torch.float64)
    if precision == "fp32":
        ref32 = _errors(*_oracle_step(PNAPlusStackOracle, kw, state, b, torch.float32), ref64)
    else:
        with tf32_linears():
            ref32 = _errors(*_oracle_step(PNAPlusStackOracle, kw, state, b, torch.float32), ref64)
    em.train()
    d = b.clone().to(DEV)
    d._num_graphs = graphs
    _lib.trace_begin()
    pred = em(d)
    loss, _ = em.loss(pred, d.y, [torch.arange(b.y.shape[0], device=DEV)])
    loss.backward()
    calls = {t[0] for t in _lib.trace_end()}
    assert "hgb_pnaplus_conv_fwd" in calls and "hgb_pnaplus_conv_bwd" in calls
    eng = _errors([p.detach() for p in pred], loss.detach(), {n: p.grad for n, p in em.named_parameters()}, em.state_dict(), ref64)
    if precision == "fp32":
        bound = {"pred": max(1e-4, 2 * ref32["pred"]), "grad": max(1e-3, 2 * ref32["grad"]), "loss": max(1e-5, 2 * ref32["loss"])}
    else:
        bound = {k: max(2e-2, 2 * v) for k, v in ref32.items()}
    assert all(eng[k] <= bound[k] for k in eng), {"engine": eng, "oracle_same_precision": ref32, "bound": bound}


def test_pnaplus_graphed_train_step_equals_eager_steps():
    name, graphs = "ogb_pnaplus", 64
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
    for k in s1:
        if s1[k].is_floating_point():
            torch.testing.assert_close(s2[k], s1[k], rtol=1e-5, atol=1e-7, msg=lambda m, k=k: k + ": " + m)
