"""GPU tests added in round 2 (VERDICT r1 items): engine vs ORACLE at the C4 (periodic MACE) and C5 (PNAEq + GPS, mixed
graph sizes) shapes, the tensor-core (TF32) bench precision against the oracle directly, the CUDA-graph step after a refill
with a different topology, the device-side guards of captured neighbour builds, and the radix-sort CSR build on long segments.

Tolerances: integer outputs bit-exact; fp32 engine vs fp32 oracle rel-L2 <= 1e-5 on outputs (2e-5 for the deepest models),
parameter gradients rel-L2 <= 1e-3; TF32 mode <= 2e-2 (SURVEY 8d)."""
import copy

import pytest
import torch

pytestmark = pytest.mark.gpu

import hydragnn_b200 as hb  # noqa: E402
from hydragnn_b200 import ops, radius, stacks  # noqa: E402
from hydragnn_b200.synthetic import ARCH, WORKLOADS, make_samples  # noqa: E402
import oracle  # noqa: E402
from oracle.workloads import add_edges_cpu, arch_for  # noqa: E402
from stack_support import _gpu_batch, _grad_rel, _loader  # noqa: E402

DEV = "cuda"


def rel_l2(a, b):
    return float((a.double().cpu() - b.double().cpu()).norm() / b.double().cpu().norm().clamp(min=1e-30))


def _canon(ei, sh=None):
    """canonical edge order (dst asc, then src asc, then shift) for set comparison"""
    key = ei[1].double() * 1e7 + ei[0].double()
    if sh is not None:
        key = key * 1e3 + (sh * torch.tensor([1.0, 3.0, 9.0], dtype=sh.dtype, device=sh.device)).sum(1).double() * 1e-2
    o = torch.argsort(key, stable=True)
    return o


# ---- C4: periodic MACE at the oc20 shape -------------------------------------------------------------------------------
def test_oc20_mace_shape_engine_matches_oracle_forward_loss_and_gradients():
    name, g = "oc20_mace", 3
    cpu = add_edges_cpu(make_samples(name, g), name)
    gpu = _gpu_batch(cpu, name, g)
    # a2: the batched periodic neighbour list equals the oracle's per-sample lists, bit for bit (edges AND shifts)
    assert gpu.edge_index.shape == cpu.edge_index.shape
    assert torch.equal(gpu.edge_index.cpu(), cpu.edge_index)
    assert torch.equal(gpu.edge_shifts.cpu(), cpu.edge_shifts.to(gpu.edge_shifts.dtype))
    kw = arch_for(name, cpu)
    om = oracle.base.create_model(**kw)
    em = hb.create_model(**kw)
    em.load_state_dict(om.state_dict())
    hi_c = hb.get_head_indices(om, cpu)
    hi_g = [h.to(DEV) for h in hi_c]
    po, pe = om(cpu), em(gpu)
    for a, b in zip(pe, po):
        assert rel_l2(a.detach(), b.detach()) < 2e-5
    lo, to = om.loss(po, cpu.y, hi_c)
    le, te = em.loss(pe, gpu.y, hi_g)
    torch.testing.assert_close(le.detach().cpu(), lo.detach(), rtol=2e-5, atol=1e-6)
    lo.backward()
    le.backward()
    assert _grad_rel(em, om) < 1e-3


def test_oc20_mace_shape_mlip_forces_and_double_backward_match_oracle():
    """C4 shape with the MLIP wrapper: energy from a node head, forces = -dE/dpos through the periodic shifts, and the
    gradient of the force loss (double backward through the MACE interaction / product blocks)."""
    name, g = "oc20_mace", 2
    cpu = add_edges_cpu(make_samples(name, g), name)
    gpu = _gpu_batch(cpu, name, g)
    kw = dict(arch_for(name, cpu), hidden_dim=32, output_dim=[1], output_type=["node"], task_weights=[1.0], loss_function_type="mse",
              output_heads={"node": {"num_headlayers": 2, "dim_headlayers": [32, 16], "type": "mlp"}},
              enable_interatomic_potential=True, energy_weight=1.0, energy_peratom_weight=1.0, force_weight=1.0)
    om = oracle.base.create_model(**kw)
    em = hb.create_model(**kw)
    em.model.load_state_dict(om.model.state_dict())
    om.train()
    em.train()
    cpu.pos.requires_grad_(True)
    gpu.pos.requires_grad_(True)
    lo, to = om.energy_force_loss(om(cpu), cpu)
    le, te = em.energy_force_loss(em(gpu), gpu)
    for a, b in zip(te, to):
        torch.testing.assert_close(a.detach().cpu().double(), b.detach().double(), rtol=1e-4, atol=1e-6)
    lo.backward()
    le.backward()
    assert _grad_rel(em.model, om.model) < 2e-3


# ---- C5: PNAEq + GPS on mixed graph sizes -----------------------------------------------------------------------------------
def test_gfm_pnaeq_gps_mixed_sizes_engine_matches_oracle():
    name, g = "gfm_pnaeq", 12
    cpu = add_edges_cpu(make_samples(name, g), name)
    sizes = set((cpu.ptr[1:] - cpu.ptr[:-1]).tolist())
    assert len(sizes) >= 3                                           # the batch really mixes {9, 21, 80, 200}
    gpu = _gpu_batch(cpu, name, g)
    assert torch.equal(gpu.edge_index.cpu(), cpu.edge_index)            # a1 at k = 20 on mixed sizes: bit-exact
    kw = arch_for(name, cpu)
    om = oracle.base.create_model(**kw).eval()                          # eval: dropout off, BatchNorm running stats (SURVEY 8d C5)
    em = hb.create_model(**kw).eval()
    em.load_state_dict(om.state_dict())
    hi_c = hb.get_head_indices(om, cpu)
    hi_g = [h.to(DEV) for h in hi_c]
    po, pe = om(cpu), em(gpu)
    for a, b in zip(pe, po):
        assert rel_l2(a.detach(), b.detach()) < 2e-5
    lo, _ = om.loss(po, cpu.y, hi_c)
    le, _ = em.loss(pe, gpu.y, hi_g)
    torch.testing.assert_close(le.detach().cpu(), lo.detach(), rtol=2e-5, atol=1e-6)
    lo.backward()
    le.backward()
    assert _grad_rel(em, om) < 1e-3


# ---- bench precision (TF32 tensor cores) against the ORACLE, first hand ---------------------------------------------------------
@pytest.mark.parametrize("name,g", [("qm9_painn", 512), ("oc20_mace", 2)])
def test_tensor_core_mode_against_oracle(name, g):
    cpu = add_edges_cpu(make_samples(name, g), name)
    gpu = _gpu_batch(cpu, name, g)
    kw = arch_for(name, cpu)
    om = oracle.base.create_model(**kw)
    em = hb.set_precision(hb.create_model(**kw), "bf16")
    em.load_state_dict(om.state_dict())
    hi_c = hb.get_head_indices(om, cpu)
    hi_g = [h.to(DEV) for h in hi_c]
    po, pe = om(cpu), em(gpu)
    for a, b in zip(pe, po):
        assert rel_l2(a.detach(), b.detach()) < 2e-2
    lo, _ = om.loss(po, cpu.y, hi_c)
    le, _ = em.loss(pe, gpu.y, hi_g)
    assert abs(float(le) - float(lo)) <= 2e-2 * abs(float(lo))
    lo.backward()
    le.backward()
    assert _grad_rel(em, om) < 2e-2


# ---- CUDA-graph step: refill with a different topology (ADVICE r1, train.py:203) ----------------------------------------------
def test_graphed_step_refill_with_new_topology_equals_eager():
    name, g = "qm9_painn", 128
    base = make_samples(name, g, seed=1).to(DEV)
    base._num_graphs = g
    base = hb.get_radius_graph(3.0, 5)(base)                        # r = 3: the edge pattern depends on the geometry
    e = base.edge_index.shape[1]
    # a second batch with the SAME shapes but different positions / edges: permute whole graphs (edge count is preserved)
    perm = torch.randperm(g, generator=torch.Generator().manual_seed(3))
    other = make_samples(name, g, seed=1)
    n = 9
    rows = (perm[:, None] * n + torch.arange(n)[None, :]).reshape(-1)
    other.pos, other.x, other.y = other.pos[rows].contiguous(), other.x[rows].contiguous(), other.y[perm].contiguous()
    other = other.to(DEV)
    other._num_graphs = g
    other = hb.get_radius_graph(3.0, 5)(other)
    assert other.edge_index.shape[1] == e and not torch.equal(other.edge_index, base.edge_index)
    m1 = hb.get_distributed_model(hb.create_model(**ARCH[name]))
    m2 = copy.deepcopy(m1)
    o1, o2 = hb.FlatAdamW(m1, lr=1e-3), hb.FlatAdamW(m2, lr=1e-3)
    static = base.clone()
    static._num_graphs = g
    gs = hb.GraphedTrainStep(m1, o1, static, warmup=2)              # 2 warm-up steps on `base`
    for _ in range(2):
        hb.train_step(m2, o2, base)
    l_graph = [float(gs.run())]                                     # step 3 on `base`
    l_eager = [float(hb.train_step(m2, o2, base)[0])]
    refill = hb.Batch(x=other.x, pos=other.pos, y=other.y, edge_index=other.edge_index, batch=other.batch)
    gs.refill(refill)
    l_graph.append(float(gs.run()))                                 # step 4 on `other`: new edges, same shapes
    l_eager.append(float(hb.train_step(m2, o2, other)[0]))
    for a, b in zip(l_graph, l_eager):
        assert abs(a - b) <= 1e-5 * abs(b) + 1e-7, (l_graph, l_eager)
    for p, q in zip(m1.parameters(), m2.parameters()):
        torch.testing.assert_close(p, q, rtol=1e-4, atol=1e-6)
    # the captured step follows the scheduler: lr lives on the device
    o1.param_groups[0]["lr"] = 0.0
    before = [p.detach().clone() for p in m1.parameters()]
    gs.run()
    torch.cuda.synchronize()
    for p, q in zip(m1.parameters(), before):
        torch.testing.assert_close(p, q * (1 - 0.0), rtol=0, atol=0)


# ---- device-side guards ------------------------------------------------------------------------------------------------------
def test_known_edge_count_guard_trips_on_mismatch_and_never_writes_out_of_bounds():
    name, g = "qm9_painn", 64
    b = make_samples(name, g).to(DEV)
    gptr = b.ptr.int()
    ei, rowptr = radius.radius_graph(b.pos, 7.0, gptr, g, False, 5)
    e = ei.shape[1]
    ops.check_guard(DEV)
    ei2, _ = radius.radius_graph(b.pos, 7.0, gptr, g, False, 5, known_e=e)       # the promised count is right: no trip
    torch.cuda.synchronize()
    ops.check_guard(DEV)
    assert torch.equal(ei2, ei)
    ei3, _ = radius.radius_graph(b.pos, 7.0, gptr, g, False, 5, known_e=e - 7)   # too small: guarded writes + flag
    torch.cuda.synchronize()
    with pytest.raises(RuntimeError, match="edge count"):
        ops.check_guard(DEV)
    ops.check_guard(DEV)                                                         # the flag was cleared by the raise
    # an out-of-range index handed to the CSR build is flagged too (ADVICE r1, hgb_core.cu:121)
    bad = torch.tensor([0, 1, 5, 2], dtype=torch.int64, device=DEV)
    ops.csr_build(bad, 4)
    with pytest.raises(RuntimeError, match="outside"):
        ops.check_guard(DEV)


def test_pbc_transform_refuses_cpu_samples():
    b = make_samples("lj_egnn", 2)
    with pytest.raises(RuntimeError, match="CUDA"):
        hb.get_radius_graph_pbc(5.0, 5)(b)


def test_csr_build_is_stable_on_long_segments():
    gen = torch.Generator().manual_seed(0)
    for n, e in [(1, 100000), (7, 300001), (5000, 20000), (3, 0)]:
        idx = torch.randint(0, n, (e,), generator=gen)
        c = ops.csr_build(idx.to(DEV), n)
        cnt = torch.bincount(idx, minlength=n)
        assert torch.equal(c.rowptr.cpu().long(), torch.cat([torch.zeros(1, dtype=torch.long), torch.cumsum(cnt, 0)]))
        if e:
            assert torch.equal(c.perm.cpu().long(), torch.argsort(idx, stable=True))
    ops.check_guard(DEV)


# ---- fused EGNN edge block (row a4) ---------------------------------------------------------------------------------------
def _egnn_losses(em, gpu, mlip):
    for p in em.parameters():
        p.grad = None
    d = gpu.clone()
    d._num_graphs = gpu._num_graphs
    if mlip:
        d.pos.requires_grad_(True)
        loss, tasks = em.energy_force_loss(em(d), d)
    else:
        inner = em.model if hasattr(em, "model") else em
        pred = inner(d)
        loss = sum((p_ ** 2).mean() for p_ in pred)
        tasks = []
    loss.backward()
    return loss.detach(), [t.detach() for t in tasks], [None if p.grad is None else p.grad.clone() for p in em.parameters()]


@pytest.mark.parametrize("name,g,k", [("md17_egnn", 24, 5), ("lj_egnn", 6, 5), ("md17_egnn", 5, 20), ("lj_egnn", 3, 64)])
@pytest.mark.parametrize("mlip", [True, False])
def test_fused_egnn_block_equals_composed_path_and_oracle(name, g, k, mlip, monkeypatch):
    """hgb_egnn_edge_{fwd,bwd_data,wgrad} (+ tangent mode in the double backward) against the round-1 composed path
    (gather / Linear / segment-sum closed primitives) and against the oracle: loss terms, and every parameter gradient of the
    MLIP loss (second derivatives through the fused block).  k = 20 / 64 gives denser graphs, but the tile rule
    (ops.egnn_nodes_per_tile: about 120 edges per tile) keeps every tile within one 128-edge chunk and every CTA on one tile
    at these sizes; tests/test_gpu_egnn_edge.py covers the multi-chunk and multi-tile paths kernel by kernel."""
    w = dict(WORKLOADS[name], max_neighbours=k)
    cpu = make_samples(name, g)
    gpu = make_samples(name, g).to(DEV)
    gpu._num_graphs = g
    tr = hb.get_radius_graph_pbc if w.get("pbc") else hb.get_radius_graph
    gpu = tr(w["radius"], k)(gpu)
    cpu.edge_index = gpu.edge_index.cpu()
    cpu.edge_shifts = gpu.edge_shifts.cpu() if gpu.edge_shifts is not None else torch.zeros(cpu.edge_index.shape[1], 3)
    kw = dict(ARCH[name])
    om = oracle.base.create_model(**kw).train()
    em = hb.create_model(**kw).train()
    em.model.load_state_dict(om.model.state_dict())
    assert ops.egnn_edge_supported(kw["hidden_dim"])
    launches = hb._lib.launch_count()
    l1, t1, g1 = _egnn_losses(em, gpu, mlip)
    with monkeypatch.context() as mp:
        mp.setattr(stacks.E_GCL, "_fused_ok", lambda self, x, edge_attr: False)
        l0, t0, g0 = _egnn_losses(em, gpu, mlip)
    torch.testing.assert_close(l1, l0, rtol=2e-5, atol=1e-7)
    for a, b in zip(t1, t0):
        torch.testing.assert_close(a, b, rtol=2e-5, atol=1e-7)
    num = sum(float((a - b).double().pow(2).sum()) for a, b in zip(g1, g0) if b is not None)
    den = sum(float(b.double().pow(2).sum()) for b in g0 if b is not None)
    assert (num / den) ** 0.5 < 1e-4, (num / den) ** 0.5
    if mlip:                                                     # and first hand against the oracle
        cpu.pos.requires_grad_(True)
        lo, to = om.energy_force_loss(om(cpu), cpu)
        lo.backward()
        torch.testing.assert_close(l1.cpu(), lo.detach(), rtol=1e-4, atol=1e-6)
        for a, b in zip(t1, to):
            torch.testing.assert_close(a.cpu().double(), b.detach().double(), rtol=1e-4, atol=1e-6)
        num = sum(float((a.cpu().double() - q.grad.double()).pow(2).sum()) for a, q in zip(g1, om.parameters()) if q.grad is not None)
        den = sum(float(q.grad.double().pow(2).sum()) for q in om.parameters() if q.grad is not None)
        assert (num / den) ** 0.5 < 1e-3, (num / den) ** 0.5


def test_edge_len_primitives_double_backward_matches_autograd():
    g = torch.Generator().manual_seed(0)
    n, e = 50, 400
    pos = torch.randn(n, 3, generator=g)
    ei = torch.randint(0, n, (2, e), generator=g)
    ei[1] = torch.where(ei[1] == ei[0], (ei[1] + 1) % n, ei[1])
    sh = torch.randn(e, 3, generator=g) * 0.1
    coef, tgt = torch.randn(e, generator=g), torch.randn(n, 3, generator=g)

    def run(pos_, dev):
        p = pos_.clone().to(dev).requires_grad_(True)
        if dev == "cpu":
            d = (p.double()[ei[1]] - p.double()[ei[0]] + sh.double()).norm(dim=1)
            c, t = coef.double(), tgt.double()
        else:
            plan = ops.EdgePlan(ei.to(dev), n)
            d = ops.EdgeLenFn.apply(p, sh.to(dev), plan)
            c, t = coef.to(dev), tgt.to(dev)
        en = (c * d * d).sum()
        f, = torch.autograd.grad(en, p, create_graph=True)
        loss = ((f - t) ** 2).sum() + en
        loss.backward()
        return d.detach(), f.detach(), p.grad.detach()

    d0, f0, g0 = run(pos, "cpu")
    d1, f1, g1 = run(pos, DEV)
    assert rel_l2(d1, d0) < 1e-6 and rel_l2(f1, f0) < 1e-5 and rel_l2(g1, g0) < 1e-5


# ---- tensor-core attention, head_dim 8 (row a9) ---------------------------------------------------------------------------
@pytest.mark.parametrize("n,f,heads", [(1, 8, 1), (65, 16, 2), (300, 64, 8), (1000, 64, 8), (4099, 64, 8)])
@pytest.mark.parametrize("mode", ["exact", "tf32"])
def test_tensor_core_attention_matches_fp64_reference(n, f, heads, mode, monkeypatch):
    """hgb_mha_tc_{fwd,bwd}: 3xTF32 ("exact") within the fp32 parity tolerance, plain TF32 within the bf16-config tolerance;
    the SIMT kernels are the second witness."""
    from hydragnn_b200 import gps
    g = torch.Generator().manual_seed(n + f)
    qkv = torch.randn(n, 3 * f, generator=g)
    go = torch.randn(n, f, generator=g)
    qr = qkv.double().requires_grad_(True)
    q, k, v = [t.reshape(n, heads, f // heads).transpose(0, 1) for t in qr.split(f, dim=1)]
    ref = torch.nn.functional.scaled_dot_product_attention(q, k, v).transpose(0, 1).reshape(n, f)
    gr, = torch.autograd.grad(ref, qr, go.double())
    assert hb._lib.query("hgb_mha_tc_supported", f, heads)
    qe = qkv.to(DEV).requires_grad_(True)
    with ops.tensor_cores(mode == "tf32"):
        out = gps.MhaFn.apply(qe, heads)
    ge, = torch.autograd.grad(out, qe, go.to(DEV))
    tol_o, tol_g = (2e-6, 1e-5) if mode == "exact" else (2e-3, 5e-3)
    assert rel_l2(out.detach(), ref.detach()) < tol_o
    assert rel_l2(ge, gr) < tol_g
    query = hb._lib.query
    with monkeypatch.context() as mp:                            # the library reports no tensor-core attention: SIMT kernels
        mp.setattr(hb._lib, "query", lambda name, *args: 0 if name == "hgb_mha_tc_supported" else query(name, *args))
        qs = qkv.to(DEV).requires_grad_(True)
        outs = gps.MhaFn.apply(qs, heads)
        gs, = torch.autograd.grad(outs, qs, go.to(DEV))
    assert rel_l2(out.detach(), outs.detach()) < 10 * tol_o and rel_l2(ge, gs) < 10 * tol_g


# ---- the API path IS the fast path: capacity-padded captured step behind hb.train (rows a11 / f3) -------------------------------
@pytest.mark.parametrize("name,mlip,build", [("qm9_painn", False, False), ("qm9_painn", False, True), ("md17_egnn", True, False),
                                             ("md17_egnn", True, True), ("lj_egnn", True, False)])
def test_train_fast_path_equals_eager_on_variable_batches(name, mlip, build):
    """hb.train(loader, ...) through ONE capacity-padded CUDA-graph step (filler graphs + dummy edges, masked losses) gives the
    losses and the parameters of the eager per-batch path, for batches whose graph / node / edge counts all differ."""
    w = WORKLOADS[name]
    sizes = [24, 17, 31, 24, 9]
    loader = _loader(name, sizes, with_edges=True)
    nb = (w["radius"], w["max_neighbours"]) if build else None
    m1 = hb.get_distributed_model(hb.create_model(**ARCH[name]))
    m2 = copy.deepcopy(m1)
    o1, o2 = hb.FlatAdamW(m1, lr=1e-3), hb.FlatAdamW(m2, lr=1e-3)
    launches = []
    for epoch in range(2):
        e_fast, t_fast = hb.train([b.clone() for b in loader], m1, o1, compute_grad_energy=mlip, fast=True, neighbour_build=nb)
        e_eager, t_eager = hb.train([b.clone() for b in loader], m2, o2, compute_grad_energy=mlip, fast=False)
        torch.testing.assert_close(e_fast, e_eager, rtol=2e-4, atol=1e-6)
        torch.testing.assert_close(t_fast.reshape(-1), t_eager.reshape(-1), rtol=2e-4, atol=1e-6)
    for p, q in zip(m1.parameters(), m2.parameters()):
        torch.testing.assert_close(p, q, rtol=2e-3, atol=2e-6)
    fast = o1._hgb_fast
    assert fast.recaptures <= 1                                      # one capture (plus at most one growth) served 10 steps
    # a batch that does not fit re-captures with grown capacities instead of failing
    big = _loader(name, [80], with_edges=True, seed0=77)
    hb.train(big, m1, o1, compute_grad_energy=mlip, fast=True, neighbour_build=nb)
    assert o1._hgb_fast.recaptures >= 1


def test_pna_aggregate_kernel_hand_computed_cases():
    """hgb_pna_aggregate_fwd on the hand-worked segments of tests/test_oracle_golden.py (two values, single edge, EMPTY segment,
    equal values): [mean | min | max | std] with PyG's std convention (sqrt(relu(var) + 1e-5), forced to 0 at the floor)."""
    x = torch.tensor([[1.0], [3.0], [2.0], [5.0], [5.0], [5.0]], device=DEV)
    index = torch.tensor([0, 0, 1, 3, 3, 3], device=DEV)
    csr = ops.csr_build(index, 4)
    out = ops.PnaAggregateFn.apply(x.requires_grad_(True), csr)
    want = torch.tensor([[2.0, 1.0, 3.0, 1.0], [2.0, 2.0, 2.0, 0.0], [0.0, 0.0, 0.0, 0.0], [5.0, 5.0, 5.0, 0.0]])
    torch.testing.assert_close(out.detach().cpu(), want, rtol=1e-6, atol=1e-6)
    out.sum().backward()                                           # subgradients exist everywhere (no NaN from the std floor)
    assert bool(torch.isfinite(x.grad).all())


# ---- multi-branch decoding as grouped GEMMs (row f4) ---------------------------------------------------------------------------
def test_multibranch_grouped_decoding_matches_oracle():
    """Three dataset branches, a graph head and a node head: the engine sorts rows by branch on the device and runs every head layer
    as one grouped GEMM (hgb_grouped_linear / hgb_grouped_wgrad); outputs, loss and every parameter gradient equal the oracle's
    boolean-mask loop (Base.py:770-780, 816-840).  A branch that receives no graph in this batch gets zero gradients."""
    name, g = "qm9_painn", 40
    cpu = add_edges_cpu(make_samples(name, g), name)
    gen = torch.Generator().manual_seed(5)
    ids = torch.randint(0, 3, (g, 1), generator=gen)
    ids[ids == 2] = 0                                                # branch 2 stays empty in this batch
    cpu.dataset_name = ids
    n = cpu.pos.shape[0]
    cpu.y = torch.cat([torch.randn(g, 1, generator=gen), torch.randn(g, 9 * 3, generator=gen)], dim=1).reshape(-1, 1)
    cpu.y_loc = torch.tensor([[0, 1, 28]]).expand(g, 3).contiguous()
    arch_g = {"num_sharedlayers": 2, "dim_sharedlayers": 10, "num_headlayers": 2, "dim_headlayers": [20, 10]}
    arch_n = {"num_headlayers": 2, "dim_headlayers": [24, 12], "type": "mlp"}
    kw = dict(ARCH[name], output_dim=[1, 3], output_type=["graph", "node"], task_weights=[1.0, 1.0],
              output_heads={"graph": [{"type": "branch-%d" % b, "architecture": dict(arch_g)} for b in range(3)],
                            "node": [{"type": "branch-%d" % b, "architecture": dict(arch_n)} for b in range(3)]})
    om = oracle.base.create_model(**kw)
    em = hb.create_model(**kw)
    em.load_state_dict(om.state_dict())
    gpu = cpu.clone().to(DEV)
    gpu._num_graphs = g
    hi_c = hb.get_head_indices(om, cpu)
    hi_g = [h.to(DEV) for h in hi_c]
    before = hb._lib.launch_count()
    hb._lib.trace_begin()
    po, pe = om(cpu), em(gpu)
    calls = [c[0] for c in hb._lib.trace_end()]
    assert "hgb_grouped_linear" in calls                             # the grouped path ran (not the per-branch fallback)
    for a, b in zip(pe, po):
        assert rel_l2(a.detach(), b.detach()) < 1e-5
    lo, _ = om.loss(po, cpu.y, hi_c)
    le, _ = em.loss(pe, gpu.y, hi_g)
    torch.testing.assert_close(le.detach().cpu(), lo.detach(), rtol=1e-5, atol=1e-6)
    lo.backward()
    le.backward()
    assert _grad_rel(em, om) < 1e-4
    en = dict(em.named_parameters())
    for k, q in om.named_parameters():
        if "branch-2" in k:
            assert q.grad is None or float(q.grad.abs().max()) == 0.0
            assert en[k].grad is None or float(en[k].grad.abs().max()) == 0.0


def test_grouped_csr_build_equals_radix_sort_build():
    """hgb_csr_build_grouped (one warp per graph, match_any ranking, no sort) gives the SAME rowptr / perm as the radix-sort build
    for the radius-graph output of mixed-size batches, open and periodic."""
    for name, g in (("gfm_pnaeq", 24), ("qm9_painn", 300), ("oc20_mace", 3)):
        w = WORKLOADS[name]
        d = make_samples(name, g).to(DEV)
        d._num_graphs = g
        d.ptr = d.ptr.int()
        if w.get("pbc_box"):
            cut = torch.full((g,), float(w["radius"]), dtype=torch.float64, device=DEV)
            ei, _, _, _, outptr, _ = radius.radius_graph_pbc(d.pos, d.cell, d.pbc, cut, d.ptr, g, w["max_neighbours"])
            rowptr = outptr
        else:
            ei, rowptr = radius.radius_graph(d.pos, w["radius"], d.ptr, g, False, w["max_neighbours"])
        n = d.pos.shape[0]
        a = ops.EdgePlan(ei, n, col_rowptr=rowptr, graph_ptr=d.ptr)
        b = ops.EdgePlan(ei, n)
        assert torch.equal(a.by_row.rowptr, b.by_row.rowptr) and torch.equal(a.by_row.perm, b.by_row.perm)
        assert torch.equal(a.by_row.idx, b.by_row.idx)
        assert torch.equal(a.by_col.rowptr, b.by_col.rowptr) and torch.equal(a.by_col.perm, b.by_col.perm)
    ops.check_guard(DEV)


# ---- tensor-core Linears in fp32 mode: the 3xTF32 split inside tc_linear (exact flag) -------------------------------------------
@pytest.mark.parametrize("m,n,k", [(5000, 64, 64), (4097, 192, 128), (128, 32, 32), (30000, 64, 128), (2000, 448, 64), (700, 384, 128),
                                   (1500, 576, 192), (520, 768, 256), (9001, 128, 256)])
def test_fp32_linear_runs_tc_exact_mode_and_matches_fp64(m, n, k):
    """fp32 mode routes the large-M Linears through the SAME wgmma kernel with every operand split into TF32 hi / lo pairs in
    shared memory (hi*hi + lo*hi + hi*lo per k-step): results within ~1e-6 of fp64, i.e. fp32-level -- the plain TF32 mode of the
    bf16 configs is ~1e-3."""
    g = torch.Generator().manual_seed(m + n)
    x, w, b = torch.randn(m, k, generator=g), torch.randn(n, k, generator=g) * 0.3, torch.randn(n, generator=g)
    xd, wd, bd = x.to(DEV), w.to(DEV), b.to(DEV)
    assert not ops._TC["enabled"] and ops.tc_ok(m, n, k, xd)
    hb._lib.trace_begin()
    y, z, _ = ops.linear_fwd_dispatch_ex(xd, wd, bd, ops.ACT_CODES["silu"], 0.0, want_z=True)
    calls = [c for c in hb._lib.trace_end() if c[0] == "hgb_tc_linear"]
    assert calls and all(c[1]["exact"] == 1 for c in calls)
    zr = x.double() @ w.double().t() + b.double()
    assert rel_l2(z, zr) < 2e-6, rel_l2(z, zr)
    assert rel_l2(y, torch.nn.functional.silu(zr)) < 2e-6
    gy = torch.randn(m, n, generator=g)
    add = torch.randn(m, k, generator=g)
    dx, _, _ = ops.linear_bwd_dispatch(gy.to(DEV), xd, wd, True, False, False, dx_addend=add.to(DEV))    # dgrad (+ addend epilogue)
    assert rel_l2(dx, gy.double() @ w.double() + add.double()) < 2e-6
    with ops.tensor_cores(True):                                                                       # plain TF32 for comparison
        y32, _ = ops.linear_fwd_dispatch(xd, wd, bd)
    e_tf32 = rel_l2(y32, zr)
    assert 1e-5 < e_tf32 < 5e-3                                                                        # the split is what buys the accuracy


@pytest.mark.parametrize("lmax", [1, 2, 3])
def test_mace_edge_embed_kernel_matches_aten_glue_and_oracle(lmax):
    """hgb_mace_edge_embed_{fwd,bwd} (spherical harmonics + Bessel x polynomial cutoff per edge, analytic d/dpos) against the ATen
    composition it replaces and against the oracle's e3 restatement (sympy-checked harmonics)."""
    from hydragnn_b200 import e3 as ee3
    from oracle import e3 as oe3
    g = torch.Generator().manual_seed(lmax)
    n, e = 60, 700
    pos = torch.randn(n, 3, generator=g) * 2.0
    ei = torch.randint(0, n, (2, e), generator=g)
    ei[1] = torch.where(ei[1] == ei[0], (ei[1] + 1) % n, ei[1])
    sh_w, rad_w = torch.randn(e, (lmax + 1) ** 2, generator=g), torch.randn(e, 8, generator=g)
    shifts = torch.randn(e, 3, generator=g) * 0.1
    rc, p = 6.0, 5.0
    # reference: fp64 torch
    pr = pos.double().requires_grad_(True)
    vec = pr[ei[1]] - pr[ei[0]] + shifts.double()
    d = vec.norm(dim=1, keepdim=True)
    sh_r = oe3.spherical_harmonics(lmax, vec, normalize=True, normalization="component")
    x = d / rc
    env = (1.0 - ((p + 1.0) * (p + 2.0) / 2.0) * x.pow(p) + p * (p + 2.0) * x.pow(p + 1) - (p * (p + 1.0) / 2) * x.pow(p + 2)) * (d < rc)
    w = torch.pi / rc * torch.arange(1, 9, dtype=torch.float64)
    rad_r = (2.0 / rc) ** 0.5 * torch.sin(w * d) / d * env
    ((sh_r * sh_w.double()).sum() + (rad_r * rad_w.double()).sum()).backward()
    # engine kernel
    pe = pos.to(DEV).requires_grad_(True)
    plan = ops.EdgePlan(ei.to(DEV), n)
    sh_e, rad_e = ops.MaceEdgeEmbedFn.apply(pe, shifts.to(DEV), plan, lmax, 8, rc, p)
    ((sh_e * sh_w.to(DEV)).sum() + (rad_e * rad_w.to(DEV)).sum()).backward()
    assert rel_l2(sh_e.detach(), sh_r.detach()) < 2e-6 and rel_l2(rad_e.detach(), rad_r.detach()) < 5e-6
    assert rel_l2(pe.grad, pr.grad) < 2e-5
    # and the ATen glue it replaces gives the same harmonics
    v32 = (pos[ei[1]] - pos[ei[0]] + shifts).to(DEV)
    sh_a = ee3.spherical_harmonics_cl(lmax, v32 / v32.norm(dim=1, keepdim=True))
    assert rel_l2(sh_e.detach(), sh_a) < 2e-6


# ---- weight gradients on a side stream (ops.fork_join): same bits as the single-stream order -------------------------------------
@pytest.mark.parametrize("name,g,prec", [("qm9_painn", 512, "bf16"), ("qm9_painn", 512, "fp32"), ("md17_egnn", 64, "fp32"),
                                         ("oc20_mace", 2, "fp32"), ("gfm_pnaeq", 4, "fp32")])
@pytest.mark.parametrize("deferred", [False, True])
def test_side_stream_weight_gradients_equal_single_stream(name, g, prec, deferred, monkeypatch):
    """Deferred joins (leaf parameters, inside ops.deferred_weight_gradients = FlatAdamW.backward) and immediate joins (derived
    weights, or outside that context) must both hand over finished gradients: every kernel is deterministic, so the gradients with
    and without the side stream agree bit for bit, repeatedly (5 passes, the caching allocator reusing freed blocks across streams
    and autograd accumulating residual-branch gradients in place in between)."""
    import contextlib
    cpu = add_edges_cpu(make_samples(name, g), name)
    gpu = _gpu_batch(cpu, name, g)
    kw = arch_for(name, cpu)
    em = hb.set_precision(hb.create_model(**kw).to(DEV), prec)
    hi = [h.to(DEV) for h in hb.get_head_indices(em, gpu)]
    mlip = bool(kw.get("enable_interatomic_potential"))

    def grads():
        em.zero_grad(set_to_none=True)
        torch.manual_seed(7)                                     # the GPS layers draw dropout masks (train mode): same masks every pass
        if mlip:
            gpu.pos.requires_grad_(True)
            loss, _ = em.energy_force_loss(em(gpu), gpu)
        else:
            loss, _ = em.loss(em(gpu), gpu.y, hi)
        with (ops.deferred_weight_gradients() if deferred else contextlib.nullcontext()):
            loss.backward()
        return {k: p.grad.clone() for k, p in em.named_parameters() if p.grad is not None}

    monkeypatch.setattr(ops, "WGRAD_OVERLAP", False)
    want = grads()
    monkeypatch.setattr(ops, "WGRAD_OVERLAP", True)
    for _ in range(5):
        got = grads()
        assert set(got) == set(want)
        for k in want:
            assert torch.equal(got[k], want[k]), k


# ---- fp32-accurate tensor-core weight gradient (hgb_tc_wgrad, exact = 1) ------------------------------------------------------------
@pytest.mark.parametrize("m,n,k,shift", [(130, 64, 64, 0.0), (5000, 64, 64, 0.0), (200000, 64, 128, 0.0), (200000, 128, 128, 0.5),
                                         (60000, 192, 96, 0.5), (33000, 64, 224, 0.0), (9001, 384, 64, 0.5), (400000, 32, 32, 1.0)])
def test_tc_wgrad_exact_mode_matches_fp64(m, n, k, shift):
    """fp32 mode: dW = dZ^T X (+ db) on wgmma with both operands split into TF32 hi / lo twins in shared memory.  ``shift`` gives
    the operands a non-zero mean, so every product has the same sign on average and a truncating accumulator would drift -- the
    kernel folds its register accumulators into the partial sum every 256 rows to keep the chains short.  fp32-level agreement with
    fp64 (the SIMT fp32 GEMM it replaces sits at the same level), bit-identical on repetition, pieces for wide outputs."""
    g = torch.Generator().manual_seed(m + n + k)
    dz, x = torch.randn(m, n, generator=g) + shift, torch.randn(m, k, generator=g) + shift
    dzd, xd = dz.to(DEV), x.to(DEV)
    assert not ops._TC["enabled"] and ops.tc_wgrad_ok(m, n, k, dzd, xd)
    hb._lib.trace_begin()
    dw, db = ops.raw_tc_wgrad(dzd, xd, want_bias=True)
    calls = [c for c in hb._lib.trace_end() if c[0] == "hgb_tc_wgrad"]
    assert calls and all(c[1]["exact"] == 1 for c in calls)
    ref_w, ref_b = dz.double().t() @ x.double(), dz.double().sum(0)
    e_w, e_b = rel_l2(dw, ref_w), rel_l2(db, ref_b)
    simt = ops.raw_gemm(dzd, xd, True, False)
    e_simt = rel_l2(simt, ref_w)
    assert e_w < max(5e-6, 4 * e_simt), (e_w, e_simt)
    assert e_b < 5e-6, e_b
    assert float((dw.double().cpu() - ref_w).abs().max()) <= 2e-5 * float(ref_w.abs().max())
    dw2, db2 = ops.raw_tc_wgrad(dzd, xd, want_bias=True)
    assert torch.equal(dw, dw2) and torch.equal(db, db2)
    with ops.tensor_cores(True):                                   # the plain TF32 mode of the same kernel, for scale
        dw32, _ = ops.raw_tc_wgrad(dzd, xd, want_bias=True)
    assert rel_l2(dw32, ref_w) > 3 * e_w
    # through autograd: a fused Linear's weight / bias gradients in fp32 mode come from this kernel
    w = (torch.randn(n, k, generator=g) * 0.2).to(DEV).requires_grad_(True)
    b = torch.zeros(n, device=DEV, requires_grad=True)
    hb._lib.trace_begin()
    (ops.linear_act(xd, w, b) * dzd).sum().backward()
    assert any(c[0] == "hgb_tc_wgrad" and c[1]["exact"] == 1 for c in hb._lib.trace_end())
    assert rel_l2(w.grad, ref_w) < max(5e-6, 4 * e_simt) and rel_l2(b.grad, ref_b) < 5e-6


# ---- head MLPs with the reference's odd widths on the tensor-core Linear (stacks._padded_chain) --------------------------------------
@pytest.mark.parametrize("name,g", [("md17_egnn", 256), ("lj_egnn", 256), ("qm9_painn", 4500)])
def test_zero_padded_head_mlps_equal_the_chain_below_the_row_threshold(name, g, monkeypatch):
    """Widths 60 / 20 / 1 (node heads) and 5 (shared graph layers) are rounded up to multiples of 32 with zero-padded weights so the
    chain runs on hgb_tc_linear; outputs, loss, forces and every parameter gradient (through the MLIP double backward) equal the
    unpadded SIMT chain to fp32 rounding, and the padded path really is the tensor-core one."""
    cpu = add_edges_cpu(make_samples(name, g), name)
    gpu = _gpu_batch(cpu, name, g)
    kw = arch_for(name, cpu)
    em = hb.create_model(**kw).to(DEV)
    hi = [h.to(DEV) for h in hb.get_head_indices(em, gpu)]
    mlip = bool(kw.get("enable_interatomic_potential"))

    def run(min_rows):
        monkeypatch.setattr(stacks, "PAD_MLP_MIN_ROWS", min_rows)
        em.zero_grad(set_to_none=True)
        hb._lib.trace_begin()
        if mlip:
            gpu.pos.requires_grad_(True)
            pred = em(gpu)
            loss, _ = em.energy_force_loss(pred, gpu)
        else:
            pred = em(gpu)
            loss, _ = em.loss(pred, gpu.y, hi)
        loss.backward()
        calls = hb._lib.trace_end()
        return [p.detach().clone() for p in pred], loss.detach().clone(), {k: p.grad.clone() for k, p in em.named_parameters()}, calls

    p0, l0, g0, c0 = run(gpu.pos.shape[0] + 1)                  # more rows than any head sees: the unpadded chain
    p1, l1, g1, c1 = run(1024)                                     # the production threshold is 32768 rows
    n_gemm = lambda cs: sum(1 for c in cs if c[0] == "hgb_gemm")            # noqa: E731
    n_tc = lambda cs: sum(1 for c in cs if c[0] in ("hgb_tc_linear", "hgb_tc_wgrad"))   # noqa: E731
    assert n_tc(c1) > n_tc(c0) and n_gemm(c1) < n_gemm(c0)
    for a, b in zip(p1, p0):
        assert a.shape == b.shape and rel_l2(a, b) < 2e-6
    assert abs(float(l1) - float(l0)) <= 2e-6 * abs(float(l0))
    assert set(g0) == set(g1)
    for k in g0:
        assert g1[k].shape == g0[k].shape
        assert rel_l2(g1[k], g0[k]) < 2e-5 or float((g1[k] - g0[k]).abs().max()) < 1e-9, k
