"""GPU parity tests, kernel level: every libhgb.so entry point (called through the C-ABI via
hydragnn_b200.ops / radius) against the CPU oracle or a plain torch fp32 reference on seeded inputs.

Tolerances: integer / index outputs bit-exact; fp32 kernels rtol 1e-5 (different summation association than
ATen), gradients rtol 1e-4."""
import numpy as np
import pytest
import torch

pytestmark = pytest.mark.gpu

import hydragnn_b200 as hb  # noqa: E402
from hydragnn_b200 import _lib, ops, radius  # noqa: E402
import oracle  # noqa: E402
from oracle.radius_graph import radius_graph as o_radius_graph, radius_graph_pbc as o_radius_graph_pbc  # noqa: E402

DEV = "cuda"
TOL = dict(rtol=1e-5, atol=1e-6)
GTOL = dict(rtol=1e-4, atol=1e-5)


def gen(seed=0):
    return torch.Generator().manual_seed(seed)


def test_library_loaded_and_counts_launches():
    assert _lib.lib().hgb_version() >= 100
    before = _lib.launch_count()
    ops.exclusive_scan(torch.ones(10, dtype=torch.int32, device=DEV))
    assert _lib.launch_count() > before


@pytest.mark.parametrize("n", [0, 1, 5, 1024, 1025, 300001])
def test_exclusive_scan(n):
    x = torch.randint(0, 7, (n,), generator=gen(n), dtype=torch.int32)
    out = ops.exclusive_scan(x.to(DEV)).cpu()
    ref = torch.cat([torch.zeros(1, dtype=torch.int64), torch.cumsum(x.long(), 0)]).int()
    assert torch.equal(out, ref)


@pytest.mark.parametrize("e,n", [(0, 4), (1, 1), (1000, 37), (200000, 5000)])
def test_csr_build_is_stable_counting_sort(e, n):
    idx = torch.randint(0, n, (e,), generator=gen(e))
    csr = ops.csr_build(idx.to(DEV), n)
    order = torch.sort(idx, stable=True).indices.int()
    assert torch.equal(csr.perm.cpu(), order)
    assert torch.equal(csr.idx.cpu(), idx.int())
    counts = torch.bincount(idx, minlength=n)
    assert torch.equal(csr.rowptr.cpu().long(), torch.cat([torch.zeros(1, dtype=torch.long), torch.cumsum(counts, 0)]))


@pytest.mark.parametrize("c", [1, 3, 4, 5, 64, 192, 200])
def test_gather_and_segment_sum(c):
    g = gen(c)
    n, e = 301, 2000
    x = torch.randn(n, c, generator=g)
    idx = torch.randint(0, n, (e,), generator=g)
    csr = ops.csr_build(idx.to(DEV), n)
    out = ops.raw_gather(x.to(DEV), csr.idx)
    assert torch.equal(out.cpu(), x[idx])
    m = torch.randn(e, c, generator=g)
    seg = ops.raw_segment_sum(m.to(DEV), csr.rowptr, csr.perm, n).cpu()
    ref = torch.zeros(n, c).index_add_(0, idx, m)            # sequential in edge order on CPU = CSR order
    torch.testing.assert_close(seg, ref, **TOL)
    # 3-D payload ([E,3,F] vectors) and determinism
    m3 = torch.randn(e, 3, 8, generator=g)
    a = ops.raw_segment_sum(m3.to(DEV), csr.rowptr, csr.perm, n)
    b = ops.raw_segment_sum(m3.to(DEV), csr.rowptr, csr.perm, n)
    assert torch.equal(a, b)
    torch.testing.assert_close(a.cpu(), torch.zeros(n, 3, 8).index_add_(0, idx, m3), **TOL)


def test_gather_segment_sum_any_order_autograd():
    g = gen(1)
    n, e, c = 40, 300, 6
    idx = torch.randint(0, n, (e,), generator=g)
    csr = ops.csr_build(idx.to(DEV), n)
    x = torch.randn(n, c, generator=g)
    w = torch.randn(e, c, generator=g)

    def f_ref(x):
        return (torch.zeros(n, c).index_add_(0, idx, (x[idx] * w) ** 2)).pow(2).sum()

    def f_eng(x):
        return (ops.SegmentSum.apply((ops.GatherRows.apply(x, csr) * w.to(DEV)) ** 2, csr)).pow(2).sum()

    xr = x.clone().requires_grad_(True)
    xe = x.to(DEV).requires_grad_(True)
    gr, = torch.autograd.grad(f_ref(xr), xr, create_graph=True)
    ge, = torch.autograd.grad(f_eng(xe), xe, create_graph=True)
    torch.testing.assert_close(ge.cpu(), gr, **GTOL)
    hr, = torch.autograd.grad(gr.pow(2).sum(), xr)
    he, = torch.autograd.grad(ge.pow(2).sum(), xe)
    torch.testing.assert_close(he.cpu(), hr, rtol=1e-3, atol=1e-3)


def test_matmul_any_order():
    g = gen(3)
    a, b = torch.randn(7, 5, generator=g), torch.randn(4, 5, generator=g)
    ar, br = a.clone().requires_grad_(True), b.clone().requires_grad_(True)
    ae, be = a.to(DEV).requires_grad_(True), b.to(DEV).requires_grad_(True)
    yr = (ar @ br.t()).tanh().pow(2).sum()
    ye = ops.MatMul.apply(ae, be, False, True).tanh().pow(2).sum()
    gar, gbr = torch.autograd.grad(yr, (ar, br), create_graph=True)
    gae, gbe = torch.autograd.grad(ye, (ae, be), create_graph=True)
    torch.testing.assert_close(gae.cpu(), gar, **GTOL)
    torch.testing.assert_close(gbe.cpu(), gbr, **GTOL)
    h_r = torch.autograd.grad((gar.pow(2).sum() + gbr.pow(2).sum()), (ar, br))
    h_e = torch.autograd.grad((gae.pow(2).sum() + gbe.pow(2).sum()), (ae, be))
    for x, y in zip(h_e, h_r):
        torch.testing.assert_close(x.cpu(), y, rtol=1e-3, atol=1e-4)


ACTS = {"relu": torch.relu, "silu": torch.nn.functional.silu, "tanh": torch.tanh, "sigmoid": torch.sigmoid,
        "lrelu": lambda x: torch.nn.functional.leaky_relu(x, 0.1), "elu": torch.nn.functional.elu,
        "selu": torch.selu, None: lambda x: x}


@pytest.mark.parametrize("act", list(ACTS))
@pytest.mark.parametrize("m,k,n", [(257, 64, 192), (100, 1, 3), (33, 11, 1), (5000, 1, 64), (4097, 2, 1), (3000, 8, 200), (70000, 1, 1)])
def test_linear_act_forward_backward(act, m, k, n):
    g = gen(m + k + n)
    x, w, b = torch.randn(m, k, generator=g), torch.randn(n, k, generator=g) * 0.3, torch.randn(n, generator=g)
    xr, wr, br = [t.clone().requires_grad_(True) for t in (x, w, b)]
    xe, we, be = [t.to(DEV).requires_grad_(True) for t in (x, w, b)]
    yr = ACTS[act](xr @ wr.t() + br)
    ye = ops.linear_act(xe, we, be, act, 0.1)
    torch.testing.assert_close(ye.cpu(), yr, rtol=1e-5, atol=1e-5)
    go = torch.randn(m, n, generator=g)
    gr = torch.autograd.grad(yr, (xr, wr, br), go)
    ge = torch.autograd.grad(ye, (xe, we, be), go.to(DEV))
    for a, c in zip(ge, gr):
        torch.testing.assert_close(a.cpu(), c, rtol=1e-4, atol=1e-4)


def test_linear_act_strided_weight_block_and_3d_input():
    g = gen(9)
    x = torch.randn(10, 3, 8, generator=g)
    wfull = torch.randn(5, 20, generator=g)
    ye = ops.linear_act(x.to(DEV), wfull.to(DEV)[:, 4:12], None)
    torch.testing.assert_close(ye.cpu(), x @ wfull[:, 4:12].t(), **TOL)


@pytest.mark.parametrize("mode", ["add", "mean", "max"])
def test_pool(mode):
    g = gen(5)
    sizes = [3, 1, 7, 0, 5]
    batch = torch.repeat_interleave(torch.arange(len(sizes)), torch.tensor(sizes))
    x = torch.randn(batch.numel(), 10, generator=g)
    gcsr = ops.graph_ptr_from_batch(batch.to(DEV), len(sizes))
    xe = x.to(DEV).requires_grad_(True)
    out = ops.PoolFn.apply(xe, gcsr, mode)
    xr = x.clone().requires_grad_(True)
    ref = oracle.geometry.graph_pool(xr, batch, len(sizes), mode)
    torch.testing.assert_close(out.cpu(), ref, **TOL)
    go = torch.randn(len(sizes), 10, generator=g)
    ge, = torch.autograd.grad(out, xe, go.to(DEV))
    gr, = torch.autograd.grad(ref, xr, go)
    torch.testing.assert_close(ge.cpu(), gr, **TOL)


# ---- radius graphs: bit-exact against the oracle --------------------------------------------------------
def _mols(g, sizes, box):
    pos = torch.cat([torch.rand(n, 3, generator=g) * box for n in sizes])
    batch = torch.repeat_interleave(torch.arange(len(sizes)), torch.tensor(sizes))
    return pos, batch


@pytest.mark.parametrize("k,loop", [(5, False), (5, True), (3, False), (100000, False)])
def test_radius_graph_bit_exact(k, loop):
    g = gen(k)
    pos, batch = _mols(g, [9, 21, 1, 2, 80, 9], 5.0)
    ref = o_radius_graph(pos, 4.0, batch, loop, k)
    d = hb.Batch(pos=pos.to(DEV), batch=batch.to(DEV))
    d._num_graphs = 6
    out = hb.RadiusGraph(4.0, loop, k)(d).edge_index
    assert out.dtype == torch.int64 and torch.equal(out.cpu(), ref)


def test_radius_graph_rotational_invariance_and_empty():
    g = gen(11)
    pos = 3 * torch.randn(10, 3, generator=g)
    c = pos - pos.mean(0, keepdim=True)
    _, _, v = torch.linalg.svd(c, full_matrices=False)
    rot = pos @ v.t()
    es = []
    for p in (pos, rot):
        d = hb.Data(pos=p.to(DEV))
        ei = hb.get_radius_graph_config({"radius": 7.0, "max_neighbours": 100000})(d).edge_index.cpu()
        es.append({(int(a), int(b)) for a, b in ei.t()})
    assert es[0] == es[1]
    d = hb.Data(pos=torch.zeros(0, 3, device=DEV))
    assert hb.RadiusGraph(1.0)(d).edge_index.shape == (2, 0)


def _bcc(a=3.6, reps=5, dtype=torch.float64):
    base = torch.tensor([[0.0, 0.0, 0.0], [0.5, 0.5, 0.5]], dtype=dtype) * a
    cells = torch.stack(torch.meshgrid(*[torch.arange(reps, dtype=dtype)] * 3, indexing="ij"), -1).reshape(-1, 3) * a
    return (cells[:, None, :] + base[None]).reshape(-1, 3), torch.eye(3, dtype=dtype) * a * reps


def test_pbc_known_answers():
    # the reference's own known-answer tests (tests/test_periodic_boundary_conditions.py:82-127)
    cases = [(torch.tensor([[1.0, 1.0, 1.0], [1.43, 1.43, 1.43]]), torch.eye(3) * 3.0, 0.9, 1)]
    pos, cell = _bcc()
    cases.append((pos, cell, 5.0, 14))
    for pos, cell, r, exp in cases:
        for loop in (False, True):
            d = hb.Data(pos=pos.to(DEV), cell=cell, pbc=[True, True, True], x=torch.ones(pos.shape[0], 1, device=DEV))
            d = hb.get_radius_graph_pbc_config({"radius": r, "max_neighbours": 100000}, loop=loop)(d)
            n = pos.shape[0]
            assert d.edge_index.shape[1] == (exp + int(loop)) * n
            vec = d.pos[d.edge_index[1]] - d.pos[d.edge_index[0]] + d.edge_shifts
            dist = vec.norm(dim=-1)
            assert bool(((dist <= r) & (dist >= 0)).all())


@pytest.mark.parametrize("dtype", [torch.float32, torch.float64])
@pytest.mark.parametrize("k", [4, 100000])
def test_pbc_bit_exact_vs_oracle(dtype, k):
    g = gen(17)
    L = 6.0
    pos = (torch.rand(30, 3, generator=g, dtype=torch.float64) * L).to(dtype)
    cell = torch.tensor([[L, 0, 0], [0.3, L, 0], [0.1, -0.2, L * 1.2]], dtype=torch.float64)
    for pbc in ([True, True, True], [True, True, False]):
        ref_ei, ref_sh = o_radius_graph_pbc(pos, cell, pbc, 3.5, False, k)
        d = hb.Data(pos=pos.to(DEV), cell=cell, pbc=pbc)
        d = hb.RadiusGraphPBC(3.5, False, k)(d)
        assert torch.equal(d.edge_index.cpu(), ref_ei)
        assert torch.equal(d.edge_shifts.cpu(), ref_sh)


def test_pbc_batched_equals_per_sample():
    g = gen(23)
    samples = []
    for n in (8, 27, 5):
        samples.append(hb.Data(pos=torch.rand(n, 3, generator=g) * 5.0, cell=torch.eye(3) * 5.0,
                               pbc=torch.tensor([True, True, True]), x=torch.ones(n, 1)))
    b = hb.Batch.from_data_list(samples).to(DEV)
    b = hb.RadiusGraphPBC(3.0, False, 6)(b)
    off, eis, shs = 0, [], []
    for s in samples:
        ei, sh = o_radius_graph_pbc(s.pos, s.cell, s.pbc, 3.0, False, 6)
        eis.append(ei + off)
        shs.append(sh)
        off += s.pos.shape[0]
    assert torch.equal(b.edge_index.cpu(), torch.cat(eis, 1))
    assert torch.equal(b.edge_shifts.cpu(), torch.cat(shs))


# ---- geometry / PaiNN blocks -----------------------------------------------------------------------------
def _toy_graph(g, n=50, e=400):
    pos = torch.randn(n, 3, generator=g) * 2
    ei = torch.randint(0, n, (2, e), generator=g)
    ei = ei[:, ei[0] != ei[1]]
    return pos, ei


@pytest.mark.parametrize("eps", [1e-9, 1.0])
def test_edge_geom_forward_backward(eps):
    g = gen(31)
    pos, ei = _toy_graph(g)
    sh = torch.randn(ei.shape[1], 3, generator=g) * 0.1
    plan = ops.EdgePlan(ei.to(DEV), pos.shape[0])
    pr = pos.clone().requires_grad_(True)
    pe = pos.to(DEV).requires_grad_(True)
    vr = pr[ei[1]] - pr[ei[0]] + sh
    lr = torch.linalg.norm(vr, dim=-1, keepdim=True)
    ur = vr / (lr + eps)
    ve, le, ue = ops.EdgeGeomFn.apply(pe, sh.to(DEV), plan, eps)
    for a, b in ((ve, vr), (le, lr), (ue, ur)):
        torch.testing.assert_close(a.cpu(), b, **TOL)
    w1, w2, w3 = [torch.randn(t.shape, generator=g) for t in (vr, lr, ur)]
    gr, = torch.autograd.grad((vr * w1).sum() + (lr * w2).sum() + (ur * w3).sum(), pr)
    ge, = torch.autograd.grad((ve * w1.to(DEV)).sum() + (le * w2.to(DEV)).sum() + (ue * w3.to(DEV)).sum(), pe)
    torch.testing.assert_close(ge.cpu(), gr, **GTOL)


def _painn_setup(g, f, r=5, edge_dim=None, n=60, e=500):
    pos, ei = _toy_graph(g, n, e)
    msg_o = oracle.painn.PainnMessage(f, r, 7.0, edge_dim)
    return pos, ei, msg_o


@pytest.mark.parametrize("f,edge_dim", [(1, None), (2, None), (6, None), (32, None), (33, None), (64, None), (96, None), (128, None), (16, 3), (64, 2)])
def test_painn_message_vs_oracle(f, edge_dim):
    g = gen(100 + f)
    torch.manual_seed(f)
    pos, ei, msg_o = _painn_setup(g, f, edge_dim=edge_dim)
    n, e = pos.shape[0], ei.shape[1]
    s, v = torch.randn(n, f, generator=g), torch.randn(n, 3, f, generator=g)
    ea = torch.randn(e, edge_dim, generator=g) if edge_dim else None
    from hydragnn_b200.stacks import PainnMessage
    msg_e = PainnMessage(f, 5, 7.0, edge_dim).to(DEV)
    msg_e.load_state_dict(msg_o.state_dict())
    plan = ops.EdgePlan(ei.to(DEV), n)
    # oracle
    pr, sr, vr = pos.clone().requires_grad_(True), s.clone().requires_grad_(True), v.clone().requires_grad_(True)
    diff, dist = oracle.geometry.edge_vectors_and_lengths(pr, ei, None, normalize=True)
    so, vo = msg_o(sr, vr, ei.t(), diff, dist, ea)
    # engine (fused)
    pe, se, ve = pos.to(DEV).requires_grad_(True), s.to(DEV).requires_grad_(True), v.to(DEV).requires_grad_(True)
    _, ln, unit = ops.EdgeGeomFn.apply(pe, None, plan, 1e-9)
    epack = ops.PainnEdgeEmbedFn.apply(unit, ln, 5, 7.0)
    s1, v1 = msg_e(se, ve, plan, {"epack": epack}, None if ea is None else ea.to(DEV))
    torch.testing.assert_close(s1.cpu(), so, rtol=1e-4, atol=1e-5)
    torch.testing.assert_close(v1.cpu(), vo, rtol=1e-4, atol=1e-5)
    ws, wv = torch.randn(so.shape, generator=g), torch.randn(vo.shape, generator=g)
    params_o = list(msg_o.parameters())
    params_e = list(msg_e.parameters())
    gr = torch.autograd.grad((so * ws).sum() + (vo * wv).sum(), [pr, sr, vr] + params_o)
    ge = torch.autograd.grad((s1 * ws.to(DEV)).sum() + (v1 * wv.to(DEV)).sum(), [pe, se, ve] + params_e)
    for a, b in zip(ge, gr):
        torch.testing.assert_close(a.cpu(), b, rtol=2e-4, atol=2e-4)
    # engine (any-order path) forward agrees too
    vec = ops.GatherRows.apply(pe, plan.by_col) - ops.GatherRows.apply(pe, plan.by_row)
    ln2 = torch.linalg.norm(vec, dim=-1, keepdim=True)
    s2, v2 = msg_e(se, ve, plan, {"unit": vec / (ln2 + 1e-9), "len": ln2}, None if ea is None else ea.to(DEV), higher_order=True)
    torch.testing.assert_close(s2.cpu(), so, rtol=1e-4, atol=1e-5)
    torch.testing.assert_close(v2.cpu(), vo, rtol=1e-4, atol=1e-5)


@pytest.mark.parametrize("f,n", [(64, 3000), (128, 700), (64, 257), (64, 20011), (128, 9001), (192, 1500), (256, 520)])
def test_painn_message_tiled_path_vs_oracle(f, n):
    """n >= 256 and F % 64 == 0 selects the shared-memory-tiled kernels: mostly-local edges (on-chip gathers) plus
    some long-range ones (global fallback), in a non-sorted edge order."""
    g = gen(300 + f)
    torch.manual_seed(f)
    pos = torch.randn(n, 3, generator=g) * 2
    src = torch.arange(n).repeat_interleave(6)
    dst = (src + torch.randint(-8, 9, (src.numel(),), generator=g)).clamp(0, n - 1)
    far = torch.randint(0, n, (2, n // 2), generator=g)
    ei = torch.cat([torch.stack([dst, src]), far], dim=1)
    ei = ei[:, ei[0] != ei[1]]
    ei = ei[:, torch.randperm(ei.shape[1], generator=g)]
    msg_o = oracle.painn.PainnMessage(f, 5, 7.0, None)
    from hydragnn_b200.stacks import PainnMessage
    msg_e = PainnMessage(f, 5, 7.0, None).to(DEV)
    msg_e.load_state_dict(msg_o.state_dict())
    s, v = torch.randn(n, f, generator=g), torch.randn(n, 3, f, generator=g)
    plan = ops.EdgePlan(ei.to(DEV), n)
    pr, sr, vr = pos.clone().requires_grad_(True), s.clone().requires_grad_(True), v.clone().requires_grad_(True)
    diff, dist = oracle.geometry.edge_vectors_and_lengths(pr, ei, None, normalize=True)
    so, vo = msg_o(sr, vr, ei.t(), diff, dist, None)
    pe, se, ve = pos.to(DEV).requires_grad_(True), s.to(DEV).requires_grad_(True), v.to(DEV).requires_grad_(True)
    _, ln, unit = ops.EdgeGeomFn.apply(pe, None, plan, 1e-9)
    epack = ops.PainnEdgeEmbedFn.apply(unit, ln, 5, 7.0)
    s1, v1 = msg_e(se, ve, plan, {"epack": epack}, None)
    torch.testing.assert_close(s1.cpu(), so, rtol=1e-4, atol=1e-5)
    torch.testing.assert_close(v1.cpu(), vo, rtol=1e-4, atol=1e-5)
    ws, wv = torch.randn(so.shape, generator=g), torch.randn(vo.shape, generator=g)
    gr = torch.autograd.grad((so * ws).sum() + (vo * wv).sum(), [pr, sr, vr] + list(msg_o.parameters()))
    ge = torch.autograd.grad((s1 * ws.to(DEV)).sum() + (v1 * wv.to(DEV)).sum(), [pe, se, ve] + list(msg_e.parameters()))
    for a, b in zip(ge, gr):
        torch.testing.assert_close(a.cpu(), b, rtol=5e-4, atol=5e-4)


@pytest.mark.parametrize("f,last", [(1, False), (1, True), (6, False), (64, False), (64, True), (7, True)])
def test_painn_update_vs_oracle(f, last):
    g = gen(200 + f)
    torch.manual_seed(f)
    n = 77
    upd_o = oracle.painn.PainnUpdate(f, last)
    from hydragnn_b200.stacks import PainnUpdate
    upd_e = PainnUpdate(f, last).to(DEV)
    upd_e.load_state_dict(upd_o.state_dict())
    s, v = torch.randn(n, f, generator=g), torch.randn(n, 3, f, generator=g)
    sr, vr = s.clone().requires_grad_(True), v.clone().requires_grad_(True)
    se, ve = s.to(DEV).requires_grad_(True), v.to(DEV).requires_grad_(True)
    so, vo = upd_o(sr, vr)
    s1, v1 = upd_e(se, ve)
    torch.testing.assert_close(s1.cpu(), so, rtol=1e-4, atol=1e-5)
    ws = torch.randn(so.shape, generator=g)
    lo, le = (so * ws).sum(), (s1 * ws.to(DEV)).sum()
    if not last:
        torch.testing.assert_close(v1.cpu(), vo, rtol=1e-4, atol=1e-5)
        wv = torch.randn(vo.shape, generator=g)
        lo, le = lo + (vo * wv).sum(), le + (v1 * wv.to(DEV)).sum()
    gr = torch.autograd.grad(lo, [sr, vr] + list(upd_o.parameters()))
    ge = torch.autograd.grad(le, [se, ve] + list(upd_e.parameters()))
    for a, b in zip(ge, gr):
        torch.testing.assert_close(a.cpu(), b, rtol=2e-4, atol=2e-4)


@pytest.mark.parametrize("last", [False, True])
@pytest.mark.parametrize("n", [77, 100003])
def test_painn_width_one_update_runs_one_kernel_and_matches_oracle(last, n):
    """node_size == 1 (first layer, quirk Q4): the one-kernel update block against the oracle, including the 13 parameter
    gradients that are reduced across blocks."""
    g = gen(900 + n)
    torch.manual_seed(3)
    upd_o = oracle.painn.PainnUpdate(1, last)
    from hydragnn_b200.stacks import PainnUpdate
    upd_e = PainnUpdate(1, last).to(DEV)
    upd_e.load_state_dict(upd_o.state_dict())
    s, v = torch.randn(n, 1, generator=g), torch.randn(n, 3, 1, generator=g)
    v[0] = 0.0                                              # |Vv| at the bias-only point
    sr, vr = s.double().requires_grad_(True), v.double().requires_grad_(True)
    se, ve = s.to(DEV).requires_grad_(True), v.to(DEV).requires_grad_(True)
    so, vo = upd_o.double()(sr, vr)
    before = _lib.launch_count()
    s1, v1 = upd_e(se, ve)
    assert _lib.launch_count() - before == 1               # the whole block is one launch
    torch.testing.assert_close(s1.cpu().double(), so, rtol=1e-4, atol=1e-5)
    ws = torch.randn(n, 1, generator=g)
    lo, le = (so * ws.double()).sum(), (s1 * ws.to(DEV)).sum()
    if not last:
        torch.testing.assert_close(v1.cpu().double(), vo, rtol=1e-4, atol=1e-5)
        wv = torch.randn(n, 3, 1, generator=g)
        lo, le = lo + (vo * wv.double()).sum(), le + (v1 * wv.to(DEV)).sum()
    gr = torch.autograd.grad(lo, [sr, vr] + list(upd_o.parameters()))
    ge = torch.autograd.grad(le, [se, ve] + list(upd_e.parameters()))
    for a, b in zip(ge, gr):
        scale = max(1.0, float(b.abs().max()))
        torch.testing.assert_close(a.cpu().double(), b, rtol=2e-4, atol=2e-4 * scale)


def test_loss_and_adamw_match_torch():
    g = gen(41)
    p0 = torch.randn(1000, generator=g)
    pr = p0.clone().requires_grad_(True)
    opt = torch.optim.AdamW([pr], lr=1e-2, weight_decay=0.01)
    pe, m, v = p0.to(DEV), torch.zeros(1000, device=DEV), torch.zeros(1000, device=DEV)
    step = torch.zeros(1, device=DEV)
    for it in range(5):
        tgt = torch.randn(1000, generator=g)
        opt.zero_grad()
        lr_ = torch.nn.functional.mse_loss(pr, tgt)
        lr_.backward()
        opt.step()
        pe_req = pe.clone().requires_grad_(True)
        le = ops.LossFn.apply(pe_req, tgt.to(DEV), 0)
        ge, = torch.autograd.grad(le, pe_req)
        torch.testing.assert_close(le.cpu(), lr_.detach(), **TOL)
        ops.adamw_step(pe, ge.contiguous(), m, v, step, 1e-2, 0.9, 0.999, 1e-8, 0.01, 1.0)
        torch.testing.assert_close(pe.cpu(), pr.detach(), rtol=1e-5, atol=1e-6)
    assert float(step) == 5.0
    mae = ops.LossFn.apply(pe, tgt.to(DEV), 1)
    torch.testing.assert_close(mae.cpu(), (pe.cpu() - tgt).abs().mean(), **TOL)


@pytest.mark.parametrize("n,e,c", [(50, 400, 12), (300, 5000, 64), (7, 3, 5)])
def test_pna_aggregate_kernel_vs_torch(n, e, c):
    """mean | min | max | std per segment (with empty segments) and its backward against plain torch."""
    g = gen(n + e + c)
    idx = torch.randint(0, n, (e,), generator=g)
    idx[idx == 3] = 4                                     # segment 3 stays empty
    m = torch.randn(e, c, generator=g)
    csr = ops.csr_build(idx.to(DEV), n)
    me = m.to(DEV).requires_grad_(True)
    out = ops.PnaAggregateFn.apply(me, csr)
    mr = m.double().requires_grad_(True)
    ref = torch.zeros(n, 4 * c, dtype=torch.float64)
    rows = []
    for i in range(n):
        seg = mr[idx == i]
        if seg.shape[0] == 0:
            rows.append(torch.zeros(4 * c, dtype=torch.float64))
            continue
        mean = seg.mean(0)
        var = (seg * seg).mean(0) - mean * mean
        sd = var.clamp(min=1e-5).sqrt()
        sd = sd.masked_fill(sd <= 1e-5 ** 0.5, 0.0)
        rows.append(torch.cat([mean, seg.min(0).values, seg.max(0).values, sd]))
    ref = torch.stack(rows)
    torch.testing.assert_close(out.cpu().double(), ref.detach(), rtol=1e-4, atol=1e-5)
    w = torch.randn(n, 4 * c, generator=g)
    ge, = torch.autograd.grad((out * w.to(DEV)).sum(), me)
    gr, = torch.autograd.grad((ref * w.double()).sum(), mr)
    torch.testing.assert_close(ge.cpu().double(), gr, rtol=1e-3, atol=1e-4)


def test_collate_to_device_equals_from_data_list():
    g = gen(77)
    samples = []
    for k in (5, 1, 9, 3):
        ei = torch.randint(0, k, (2, 3 * k), generator=g)
        samples.append(hb.Data(x=torch.randn(k, 2, generator=g), pos=torch.randn(k, 3, generator=g), edge_index=ei,
                               edge_attr=torch.randn(3 * k, 4, generator=g), y=torch.randn(1, 1, generator=g),
                               energy=torch.randn((), generator=g), cell=torch.randn(3, 3, generator=g),
                               pbc=torch.tensor([True, False, True])))
    ref = hb.Batch.from_data_list(samples)
    out = hb.collate_to_device(samples, DEV)
    torch.cuda.synchronize()
    for k in ("x", "pos", "edge_index", "edge_attr", "y", "energy", "cell", "pbc", "batch", "ptr"):
        assert torch.equal(out[k].cpu(), ref[k]), k
    assert out.num_graphs == 4
