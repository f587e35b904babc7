"""Kernel-level tests of the fused EGNN edge block (csrc/hgb_egnn.cu) against a plain fp64 restatement of the same operation:

    z1_e = P[row_e] + Q[col_e] + s_e w_d + b0,    z2_e = W1 relu(z1_e) + b1,    out_i = sum_{row_e = i} relu(z2_e)

Backward and weight gradients are fp64 autograd of that expression; the tangent is its JVP with the ReLU masks held fixed (the
masked block is affine in its inputs, so the JVP is the masked block of the tangent inputs without biases).  Where a ReLU argument
is within rounding of zero, fp32 and fp64 may pick different masks, so the derivative references use the kernel's own masks and
the masks are checked on their own against the fp64 signs away from zero.  With dyadic inputs fp32 is exact and everything,
masks and ReLU ties included, must equal fp64 bit for bit.

The graphs have a controlled degree profile, and `census` asserts that every case reaches the paths production batches take:
a tile of more than one 128-edge chunk, a node whose segment spans chunks, and more tiles than CTAs (each CTA loops over tiles,
carrying its weight-gradient accumulators).  Radius graphs under the production tile rule (about 120 edges per tile, at most one
tile per CTA at test sizes) reach none of them.
"""
import contextlib
import functools
import types

import pytest
import torch

pytestmark = pytest.mark.gpu

from hydragnn_b200 import _lib, ops  # noqa: E402

DEV = "cuda"
TE = 128                   # edges per chunk (hgb_egnn.cu)
GRID_MAX = 3 * 132         # CTAs per launch: min(tiles, 3 x SMs)
NPTS = (1, 3, 7, 21, 24, 32)
N_MAIN = 20011             # n % npt != 0 for every npt > 1 above (a partial last tile); ~50 tiles per CTA at npt = 1
TOL = 1e-5
PARAMS = ("pq", "s", "wd", "b0", "w1", "b1")


# ---- graphs ---------------------------------------------------------------------------------------------------------------
@functools.lru_cache(maxsize=None)
def _graph(n, seed=0):
    """edge_index [2, E] int64 on the CPU.  Degrees (edges with edge_index[0] = i) are uniform in 0..8, except for
    - runs of isolated nodes at the start, at the end and at assorted offsets (empty tiles, empty segments at tile edges);
    - nodes of degree 1, 127, 128, 129 in a row, 256 next to 301, and a hub of 1000 between two isolated runs;
    - 90 consecutive nodes of degree 20-70 (tiles of several nodes and several chunks at small npt).
    Edge ids are shuffled, so CSR order is not edge order."""
    g = torch.Generator().manual_seed(seed)
    deg = torch.randint(0, 9, (n,), generator=g)
    deg[:40] = 0
    deg[-37:] = 0
    for a in range(1000, n - 200, 1777):
        deg[a:a + 3 + a % 13] = 0
    c = n // 5
    deg[c:c + 4] = torch.tensor([1, 127, 128, 129])
    deg[n // 2:n // 2 + 2] = torch.tensor([256, 301])
    h = 4 * n // 5
    deg[h - 9:h + 10] = 0
    deg[h] = 1000
    b = 2 * n // 3
    deg[b:b + 90] = torch.randint(20, 71, (90,), generator=g)
    row = torch.repeat_interleave(torch.arange(n), deg)
    col = torch.randint(0, n, (row.numel(),), generator=g)
    order = torch.randperm(row.numel(), generator=g)
    return torch.stack([row[order], col[order]])


def census(rowptr, npt):
    """What one launch reaches with this CSR and tile size, by the kernels' tile rule: tiles of npt consecutive nodes,
    min(tiles, 3 x 132) CTAs striding over them."""
    rp = rowptr.cpu().long()
    n = rp.numel() - 1
    ntiles = (n + npt - 1) // npt
    first = torch.arange(ntiles) * npt
    tile_edges = rp[torch.clamp(first + npt, max=n)] - rp[first]
    return dict(ntiles=ntiles, ctas=min(ntiles, GRID_MAX), max_tile_edges=int(tile_edges.max()),
                max_degree=int((rp[1:] - rp[:-1]).max()))


def assert_reaches_multi_chunk_and_multi_tile(rowptr, npt):
    c = census(rowptr, npt)
    assert c["max_tile_edges"] > TE, c        # the chunk loop runs more than once: per-node sums carried across chunks
    assert c["max_degree"] > TE, c            # a node's segment spans chunks: clamped per-node ranges at the chunk edge
    assert c["ntiles"] > c["ctas"], c         # CTAs loop over tiles: per-tile resets, accumulators carried across tiles
    return c


@functools.lru_cache(maxsize=None)
def _case(h, exact):
    """The main graph, its plan, fp64 inputs on the GPU (`x`), the same values in fp32 (`x32`), and the tangent inputs with
    the biases zeroed (`xt`).  exact: dyadic values that fp32 represents and sums without rounding."""
    ei = _graph(N_MAIN)
    n, e = N_MAIN, ei.shape[1]
    g = torch.Generator().manual_seed(17 + h + 1000 * exact)
    if exact:
        # multiples of 1/4: every product the block forms is a multiple of 2^-6, so fp32 sums are exact while they stay small
        def q(lo, hi, *shape):
            return torch.randint(lo, hi + 1, shape, generator=g).double() / 4
        w1 = q(-2, 2, h, h) * (torch.rand(h, h, generator=g) < 0.4)       # sparse: z2 = 0 ties beyond column 0
        w1[0] = 0.0                                                        # z2[:, 0] = b1[0] = 0 on every edge
        w1[1] = 0.0
        w1[1, :2] = 0.25
        b1 = q(-2, 2, h)
        b1[:2] = 0.0
        x = dict(pq=q(-4, 4, n, 2 * h), s=q(0, 8, e), wd=q(-4, 4, h), b0=q(-4, 4, h), w1=w1, b1=b1,
                 g_out=q(-2, 2, n, h), pq_t=q(-4, 4, n, 2 * h), s_t=q(-4, 4, e))
    else:
        x = dict(pq=torch.randn(n, 2 * h, generator=g) * 0.5 + 0.1, s=torch.rand(e, generator=g) * 2.5 + 0.5,
                 wd=torch.randn(h, generator=g) * 0.3, b0=torch.randn(h, generator=g) * 0.1,
                 w1=torch.randn(h, h, generator=g) / h ** 0.5, b1=torch.randn(h, generator=g) * 0.1,
                 g_out=torch.randn(n, h, generator=g) + 0.3, pq_t=torch.randn(n, 2 * h, generator=g) * 0.5 + 0.1,
                 s_t=torch.randn(e, generator=g))
        x = {k: v.float().double() for k, v in x.items()}
    c = types.SimpleNamespace(n=n, e=e, h=h)
    c.ei = ei.to(DEV)
    c.row, c.col = c.ei[0], c.ei[1]
    c.plan = ops.EdgePlan(c.ei, n)
    c.x = {k: v.to(DEV) for k, v in x.items()}
    c.x32 = {k: v.float().contiguous() for k, v in c.x.items()}
    c.xt = dict(pq=c.x["pq_t"], s=c.x["s_t"], wd=c.x["wd"], b0=torch.zeros_like(c.x["b0"]), w1=c.x["w1"],
                b1=torch.zeros_like(c.x["b1"]))
    return c


# ---- fp64 reference -------------------------------------------------------------------------------------------------------
def ref_block(pq, s, wd, b0, w1, b1, row, col, n, m1=None, m2=None):
    """-> (out, z1, z2).  m1 / m2 None: the two ReLUs (torch's relu' is 0 at 0, as the kernels' z > 0); else the given 0/1
    masks (edge order) stand in for them."""
    h = w1.shape[0]
    z1 = pq[row, :h] + pq[col, h:] + s[:, None] * wd + b0
    y = torch.relu(z1) if m1 is None else z1 * m1
    z2 = y @ w1.t() + b1
    m = torch.relu(z2) if m2 is None else z2 * m2
    return torch.zeros(n, h, dtype=z2.dtype, device=z2.device).index_add_(0, row, m), z1, z2


def ref_grads(x, g_out, row, col, n, m1=None, m2=None):
    """fp64 autograd of <g_out, block(x)>: {pq, s, wd, b0, w1, b1, gz1 (= d/dz1)}"""
    leaves = [x[k].detach().clone().requires_grad_(True) for k in PARAMS]
    out, z1, _ = ref_block(*leaves, row, col, n, m1, m2)
    return dict(zip(PARAMS + ("gz1",), torch.autograd.grad(out, leaves + [z1], g_out)))


def decode(masks, perm, h):
    """kernel masks [E, 2] (CSR slot order, one bit per channel) -> edge-order 0/1 float64 [E, h] for z1 and z2, and the
    bits above h (must be clear)"""
    em = torch.empty_like(masks)
    em[perm.long()] = masks
    bits = (em.unsqueeze(2) >> torch.arange(64, device=masks.device)) & 1
    return bits[:, 0, :h].double(), bits[:, 1, :h].double(), bits[:, :, h:]


def rel(a, ref):
    return float((a.double() - ref).norm() / ref.norm())


def bits_equal(a, b):
    if a.dtype == torch.float32:
        a, b = a.view(torch.int32), b.view(torch.int32)
    return a.shape == b.shape and torch.equal(a, b)


# ---- the kernels, with an explicit tile size ------------------------------------------------------------------------------
def run_kernels(c, npt):
    x = c.x32
    masks = torch.empty(c.e, 2, dtype=torch.int64, device=DEV)
    k = dict(masks=masks)
    k["out"] = ops._raw_egnn_fwd(x["pq"], x["s"], x["wd"], x["b0"], x["w1"], x["b1"], c.plan, npt, masks, False)
    k["g_pq"], k["gz1"], k["gs"], k["g_wd"], k["g_b0"] = ops._raw_egnn_bwd_data(x["g_out"], x["s"], x["wd"], x["w1"], masks, c.plan,
                                                                                 npt, True)
    k["g_w1"], k["g_b1"] = ops._raw_egnn_wgrad(x["g_out"], x["pq"], x["s"], x["wd"], x["b0"], masks, c.plan, npt, False, True)
    k["t_out"] = ops._raw_egnn_fwd(x["pq_t"], x["s_t"], x["wd"], None, x["w1"], None, c.plan, npt, masks, True)
    k["tg_w1"], k["tg_b1"] = ops._raw_egnn_wgrad(x["g_out"], x["pq_t"], x["s_t"], x["wd"], None, masks, c.plan, npt, True, True)
    torch.cuda.synchronize()
    return k


def references(c, m1, m2):
    """fp64 references of every kernel output, the derivatives taken with the masks m1 / m2 (None: the ReLUs themselves)"""
    x, h = c.x, c.h
    out, z1, z2 = ref_block(*(x[k] for k in PARAMS), c.row, c.col, c.n)
    if m1 is None:
        m1, m2 = (z1 > 0).double(), (z2 > 0).double()
        r = ref_grads(x, x["g_out"], c.row, c.col, c.n)
    else:
        r = ref_grads(x, x["g_out"], c.row, c.col, c.n, m1, m2)
    rt = ref_grads(c.xt, x["g_out"], c.row, c.col, c.n, m1, m2)
    ref = dict(out=out, g_p=r["pq"][:, :h], g_q=r["pq"][:, h:], gz1=r["gz1"], gs=r["s"], g_wd=r["wd"], g_b0=r["b0"],
               g_w1=r["w1"], g_b1=r["b1"], t_out=ref_block(*(c.xt[k] for k in PARAMS), c.row, c.col, c.n, m1, m2)[0],
               tg_w1=rt["w1"], tg_b1=rt["b1"])
    return ref, z1, z2


def kernel_view(k, h):
    return dict(k, g_p=k["g_pq"][:, :h], g_q=k["g_pq"][:, h:])


# ---- 1. every kernel output on its own against fp64 ---------------------------------------------------------------------
@pytest.mark.parametrize("npt", NPTS)
@pytest.mark.parametrize("h", [32, 64])
def test_edge_kernels_match_fp64(h, npt):
    c = _case(h, exact=False)
    assert_reaches_multi_chunk_and_multi_tile(c.plan.by_row.rowptr, npt)
    k = kernel_view(run_kernels(c, npt), h)
    m1, m2, high = decode(k["masks"], c.plan.by_row.perm, h)
    assert not high.any()
    ref, z1, z2 = references(c, m1, m2)
    for name, m, z in (("mask1", m1, z1), ("mask2", m2, z2)):
        sure = z.abs() > 1e-4 * z.abs().max()
        assert torch.equal(m.bool()[sure], (z > 0)[sure]), name
    errs = {name: rel(k[name], ref[name]) for name in ("out", "g_p", "g_q", "gz1", "gs", "g_w1", "g_b1", "t_out", "tg_w1", "tg_b1")}
    assert max(errs.values()) <= TOL, errs
    # g_wd / g_b0 are sums over all edges that cancel heavily: elementwise against the sum of the magnitudes of their terms
    gz1 = ref["gz1"].abs()
    for name, terms in (("g_wd", (c.x["s"].abs()[:, None] * gz1).sum(0)), ("g_b0", gz1.sum(0))):
        err = (k[name].double() - ref[name]).abs()
        assert bool((err <= TOL * terms).all()), (name, float((err / terms).max()))


# ---- 2. dyadic inputs: fp32 is exact, so every output equals fp64 -------------------------------------------------------
@pytest.mark.parametrize("npt", NPTS)
@pytest.mark.parametrize("h", [32, 64])
def test_dyadic_inputs_are_exact_including_relu_ties(h, npt):
    c = _case(h, exact=True)
    k = kernel_view(run_kernels(c, npt), h)
    ref, z1, z2 = references(c, None, None)
    # the case keeps producing ReLU ties, and every partial sum stays exact in fp32: all values are multiples of 2^-6 and every
    # sum of |terms| (the same expressions of |inputs|) stays below 2^18, within fp32's 24-bit significand
    assert int((z1 == 0).sum()) > 10000 and int((z2[:, 1:] == 0).sum()) > 10000
    ax = {name: t.abs() for name, t in c.x.items()}
    m1, m2 = (z1 > 0).double(), (z2 > 0).double()
    bound = ref_grads(ax, ax["g_out"], c.row, c.col, c.n, m1, m2)
    bound["out"], bz1, bz2 = ref_block(*(ax[k] for k in PARAMS), c.row, c.col, c.n, m1, m2)
    axt = dict(ax, pq=ax["pq_t"], s=ax["s_t"])
    bound["t_out"] = ref_block(*(axt[k] for k in PARAMS), c.row, c.col, c.n, m1, m2)[0]
    bound["tg_w1"] = ref_grads(axt, ax["g_out"], c.row, c.col, c.n, m1, m2)["w1"]
    assert max(float(t.abs().max()) for t in list(bound.values()) + [bz1, bz2]) < 2 ** 18
    km1, km2, high = decode(k["masks"], c.plan.by_row.perm, h)
    assert torch.equal(km1, m1) and torch.equal(km2, m2) and not high.any()
    for name in ("out", "g_p", "g_q", "gz1", "gs", "g_wd", "g_b0", "g_w1", "g_b1", "t_out", "tg_w1", "tg_b1"):
        assert torch.equal(k[name].double(), ref[name]), (name, float((k[name].double() - ref[name]).abs().max()))


# ---- 3. the summation order is fixed by the CSR: bit-identical across tile sizes, and on a repeat ----------------------
@pytest.mark.parametrize("h", [32, 64])
def test_outputs_are_bit_identical_across_tile_sizes_and_repeats(h):
    c = _case(h, exact=False)
    base = None
    for npt in NPTS:
        k = run_kernels(c, npt)
        if base is None:
            base = k
        for name in ("out", "masks", "g_pq", "gz1", "gs", "t_out"):          # per node / per edge: independent of the tiling
            assert bits_equal(k[name], base[name]), (name, npt)
        again = run_kernels(c, npt)
        for name in ("g_w1", "g_b1", "g_wd", "g_b0", "tg_w1", "tg_b1"):      # per-CTA partials: fixed at a fixed tiling
            assert bits_equal(again[name], k[name]), (name, npt)


# ---- 4. long weight-gradient reductions ---------------------------------------------------------------------------------
@pytest.mark.parametrize("n", [180_000, 720_000])
def test_weight_gradient_long_reductions_match_fp64(n):
    """E ~ 1 M (C3's size) and ~ 4 M edges at the production tile rule (21 nodes per tile at mean degree 5.5, as in C3): each
    fp32 register accumulator chains ~E / (2 x 396) FMAs of terms with a non-zero mean (y = relu(z1) >= 0, g_out and P, Q
    biased).  The fp64 reference runs on the GPU; a plain fp32 GEMM of the same operands (TF32 off) is printed for scale."""
    h = 64
    g = torch.Generator(device=DEV).manual_seed(n)
    deg = torch.randint(4, 8, (n,), device=DEV, generator=g)
    row = torch.repeat_interleave(torch.arange(n, device=DEV), deg)
    e = row.numel()
    col = torch.randint(0, n, (e,), device=DEV, generator=g)
    order = torch.randperm(e, device=DEV, generator=g)
    ei = torch.stack([row[order], col[order]])
    row, col = ei[0], ei[1]
    plan = ops.EdgePlan(ei, n)
    npt = ops.egnn_nodes_per_tile(plan)
    cen = census(plan.by_row.rowptr, npt)
    assert npt == 21 and cen["ntiles"] > 20 * cen["ctas"], (npt, cen)
    pq = torch.randn(n, 2 * h, device=DEV, generator=g) * 0.5 + 0.2
    s = torch.rand(e, device=DEV, generator=g) * 2.5 + 0.5
    wd = torch.randn(h, device=DEV, generator=g) * 0.3
    b0 = torch.randn(h, device=DEV, generator=g) * 0.1
    w1 = torch.randn(h, h, device=DEV, generator=g) / h ** 0.5
    b1 = torch.randn(h, device=DEV, generator=g) * 0.1
    g_out = torch.randn(n, h, device=DEV, generator=g) + 0.5
    masks = torch.empty(e, 2, dtype=torch.int64, device=DEV)
    ops._raw_egnn_fwd(pq, s, wd, b0, w1, b1, plan, npt, masks, False)
    g_w1, g_b1 = ops._raw_egnn_wgrad(g_out, pq, s, wd, b0, masks, plan, npt, False, True)
    torch.cuda.synchronize()
    em = torch.empty_like(masks[:, 1])
    em[plan.by_row.perm.long()] = masks[:, 1]
    gz2 = ((em.unsqueeze(1) >> torch.arange(h, device=DEV)) & 1).double()   # the kernel's mask2: sign of z2 near 0 is its to pick
    del em
    gz2 *= g_out.double()[row]
    pq64 = pq.double()
    y = torch.relu(pq64[row, :h] + pq64[col, h:] + s.double()[:, None] * wd.double() + b0.double())
    ref_w1, ref_b1 = gz2.t() @ y, gz2.sum(0)
    prev = torch.backends.cuda.matmul.allow_tf32
    torch.backends.cuda.matmul.allow_tf32 = False
    try:
        plain = rel(gz2.float().t() @ y.float(), ref_w1)
    finally:
        torch.backends.cuda.matmul.allow_tf32 = prev
    errs = dict(g_w1=rel(g_w1, ref_w1), g_b1=rel(g_b1, ref_b1))
    print("egnn_edge_wgrad E=%d npt=%d tiles/CTA=%.1f: rel-L2 vs fp64 g_w1 %.2e g_b1 %.2e (plain fp32 GEMM %.2e)"
          % (e, npt, cen["ntiles"] / cen["ctas"], errs["g_w1"], errs["g_b1"], plain))
    assert max(errs.values()) <= TOL, (errs, plain)


# ---- 5. the autograd Functions, first and second order ------------------------------------------------------------------
@pytest.mark.parametrize("data_only", [False, True])
def test_egnn_edge_fn_double_backward_matches_fp64(data_only):
    """EgnnEdgeFn forward, a create_graph backward (under only_data_grads(): the force pass of the MLIP loss) and a second
    backward, against fp64 autograd per tensor.  The energy is quadratic in the block's output, so the second pass runs the
    tangent kernel, the tangent weight gradient and hgb_weighted_colsum; w_d is a column view of a wider weight, as
    stacks.E_GCL passes it."""
    c = _case(64, exact=False)
    h, n = c.h, c.n
    g = torch.Generator().manual_seed(5)
    w0 = (torch.randn(h, 5, generator=g) * 0.3).to(DEV)
    coef = (torch.randn(n, h, generator=g) + 0.2).to(DEV)
    quad = (torch.rand(n, h, generator=g) * 0.2).to(DEV)
    t_pq = torch.randn(n, 2 * h, generator=g).to(DEV)
    t_s = torch.randn(c.e, generator=g).to(DEV)

    def run(dtype, fused):
        leaves = [t.to(dtype).detach().clone().requires_grad_(True) for t in (c.x["pq"], c.x["s"], w0, c.x["b0"], c.x["w1"], c.x["b1"])]
        pq, s, wide, b0, w1, b1 = leaves
        wd = wide[:, 3]
        if fused:
            out = ops.EgnnEdgeFn.apply(pq, s, wd, b0, w1, b1, c.plan)
        else:
            out = ref_block(pq, s, wd, b0, w1, b1, c.row, c.col, n)[0]
        energy = (coef.to(dtype) * out).sum() + 0.5 * (quad.to(dtype) * out * out).sum()
        wrt = [pq, s] if data_only else leaves
        with ops.only_data_grads() if (fused and data_only) else contextlib.nullcontext():
            first = torch.autograd.grad(energy, wrt, create_graph=True)
        loss = (t_pq.to(dtype) * first[0]).sum() + (t_s.to(dtype) * first[1]).sum()
        second = torch.autograd.grad(loss, leaves)
        return [out] + list(first) + list(second)

    got, ref = run(torch.float32, True), run(torch.float64, False)
    names = ["out"] + ["d_" + k for k in (["pq", "s"] if data_only else ["pq", "s", "w0", "b0", "w1", "b1"])]
    names += ["dd_" + k for k in ("pq", "s", "w0", "b0", "w1", "b1")]
    errs = {name: rel(a.detach(), b.detach()) for name, a, b in zip(names, got, ref)}
    assert max(errs.values()) <= TOL, errs


# ---- 6. the raw C-ABI ---------------------------------------------------------------------------------------------------
def _bwd_data(c, npt, masks, g_p, ldp, g_wd=None, g_b0=None, ws=None, n=None, h=None):
    x = c.x32
    gz1 = torch.empty(c.e, c.h, device=DEV)
    gs = torch.empty(c.e, device=DEV)
    p = ops._p
    _lib.call("hgb_egnn_edge_bwd_data", p(x["g_out"]), p(x["s"]), p(x["wd"]), p(x["w1"]), p(masks), p(c.plan.by_row.rowptr),
              p(c.plan.by_row.perm), c.n if n is None else n, c.h if h is None else h, npt, p(g_p), ldp, p(gz1), p(gs), p(g_wd),
              p(g_b0), p(ws), ops._stream())


def test_bwd_data_honours_the_row_stride_of_g_p():
    c, npt = _case(64, exact=False), 7
    h, x = c.h, c.x32
    masks = torch.empty(c.e, 2, dtype=torch.int64, device=DEV)
    ops._raw_egnn_fwd(x["pq"], x["s"], x["wd"], x["b0"], x["w1"], x["b1"], c.plan, npt, masks, False)
    wide = torch.full((c.n, 2 * h), -1234.5, device=DEV)
    dense = torch.full((c.n, h), float("nan"), device=DEV)
    _bwd_data(c, npt, masks, wide, 2 * h)
    _bwd_data(c, npt, masks, dense, h)
    torch.cuda.synchronize()
    assert bool((wide[:, h:] == -1234.5).all())
    assert bits_equal(wide[:, :h].contiguous(), dense)
    assert not torch.isnan(dense).any()


def test_bad_arguments_are_rejected_before_any_launch():
    """Unsupported widths, tile sizes outside [1, 32] and an unpaired g_wd / g_b0: an error, and no kernel launched.  Every
    buffer is sized for h = 128, the widest h tried."""
    c = _case(64, exact=False)
    n, e, hmax = c.n, c.e, 128
    buf = {k: torch.zeros(*shape, device=DEV) for k, shape in (("pq", (n, 2 * hmax)), ("node", (n, hmax)), ("edge_h", (e, hmax)),
                                                                ("edge", (e,)), ("vec", (hmax,)), ("mat", (hmax, hmax)))}
    masks = torch.zeros(e, 2, dtype=torch.int64, device=DEV)
    ws = ops._egnn_ws(n, hmax, 1, DEV)
    rp, perm, nbr = c.plan.by_row.rowptr, c.plan.by_row.perm, c.plan.nbr("row")
    p, st = ops._p, ops._stream()

    def fwd(h, npt, tangent=0):
        _lib.call("hgb_egnn_edge_fwd", p(buf["pq"]), p(buf["edge"]), p(buf["vec"]), p(buf["vec"]), p(buf["mat"]), p(buf["vec"]),
                  p(rp), p(perm), p(nbr), n, h, npt, tangent, p(masks), p(buf["node"]), st)

    def bwd(h, npt, g_wd=True, g_b0=True, w=True):
        _lib.call("hgb_egnn_edge_bwd_data", p(buf["node"]), p(buf["edge"]), p(buf["vec"]), p(buf["mat"]), p(masks), p(rp), p(perm),
                  n, h, npt, p(buf["pq"]), 2 * h, p(buf["edge_h"]), p(buf["edge"]), p(buf["vec"]) if g_wd else None,
                  p(buf["vec"]) if g_b0 else None, p(ws) if w else None, st)

    def wgrad(h, npt, tangent=0):
        _lib.call("hgb_egnn_edge_wgrad", p(buf["node"]), p(buf["pq"]), p(buf["edge"]), p(buf["vec"]), p(buf["vec"]), p(masks), p(rp),
                  p(perm), p(nbr), n, h, npt, tangent, p(buf["mat"]), p(buf["vec"]), p(ws), st)

    calls = []
    for entry in (fwd, bwd, wgrad):
        calls += [(entry, (h, 4), "hidden width must be 32 or 64") for h in (16, 48, 128)]
        calls += [(entry, (h, npt), "bad arguments") for h in (32, 64) for npt in (0, 33)]
    calls += [(functools.partial(bwd, g_b0=False), (64, 4), "come together"),
              (functools.partial(bwd, g_wd=False), (64, 4), "come together"),
              (functools.partial(bwd, w=False), (64, 4), "need the workspace")]
    torch.cuda.synchronize()
    for fn, args, msg in calls:
        before = _lib.launch_count()
        with pytest.raises(RuntimeError, match=msg):
            fn(*args)
        assert _lib.launch_count() == before, (fn, args)
    torch.cuda.synchronize()


@pytest.mark.parametrize("h", [32, 64])
def test_nodes_without_edges_give_zeros(h):
    """e = 0, n > 0: every output is zero.  The per-edge arrays have length 0; they get small valid buffers that the kernels
    must not read."""
    n, npt = 1000, 7
    g = torch.Generator().manual_seed(h)
    pq, w1 = torch.randn(n, 2 * h, generator=g).to(DEV), torch.randn(h, h, generator=g).to(DEV)
    vec, g_out = torch.randn(h, generator=g).to(DEV), torch.randn(n, h, generator=g).to(DEV)
    rp = torch.zeros(n + 1, dtype=torch.int32, device=DEV)
    idx, edge, masks = (torch.zeros(4, dtype=torch.int32, device=DEV), torch.zeros(4, device=DEV),
                        torch.zeros(4, 2, dtype=torch.int64, device=DEV))
    ws = ops._egnn_ws(n, h, npt, DEV)
    nan = lambda *shape: torch.full(shape, float("nan"), device=DEV)  # noqa: E731
    out, t_out, g_p, g_wd, g_b0, g_w1, g_b1, tg_w1 = nan(n, h), nan(n, h), nan(n, h), nan(h), nan(h), nan(h, h), nan(h), nan(h, h)
    p, st = ops._p, ops._stream()
    _lib.call("hgb_egnn_edge_fwd", p(pq), p(edge), p(vec), p(vec), p(w1), p(vec), p(rp), p(idx), p(idx), n, h, npt, 0, p(masks), p(out), st)
    _lib.call("hgb_egnn_edge_fwd", p(pq), p(edge), p(vec), None, p(w1), None, p(rp), p(idx), p(idx), n, h, npt, 1, p(masks), p(t_out), st)
    _lib.call("hgb_egnn_edge_bwd_data", p(g_out), p(edge), p(vec), p(w1), p(masks), p(rp), p(idx), n, h, npt, p(g_p), h, p(edge), p(edge),
              p(g_wd), p(g_b0), p(ws), st)
    _lib.call("hgb_egnn_edge_wgrad", p(g_out), p(pq), p(edge), p(vec), p(vec), p(masks), p(rp), p(idx), p(idx), n, h, npt, 0, p(g_w1),
              p(g_b1), p(ws), st)
    _lib.call("hgb_egnn_edge_wgrad", p(g_out), p(pq), p(edge), p(vec), None, p(masks), p(rp), p(idx), p(idx), n, h, npt, 1, p(tg_w1),
              None, p(ws), st)
    torch.cuda.synchronize()
    for name, t in (("out", out), ("t_out", t_out), ("g_p", g_p), ("g_wd", g_wd), ("g_b0", g_b0), ("g_w1", g_w1), ("g_b1", g_b1),
                    ("tg_w1", tg_w1)):
        assert bool((t == 0).all()), name
    assert torch.equal(masks, torch.zeros_like(masks))


@pytest.mark.parametrize("h", [32, 64])
def test_no_nodes_zeroes_the_parameter_sums(h):
    """n = 0: the data backward and the weight gradient write zero parameter sums (their outputs come from torch.empty)."""
    dummy, rp = torch.zeros(64, device=DEV), torch.zeros(1, dtype=torch.int32, device=DEV)
    idx, masks = torch.zeros(4, dtype=torch.int32, device=DEV), torch.zeros(4, 2, dtype=torch.int64, device=DEV)
    ws = ops._egnn_ws(0, h, 1, DEV)
    g_wd, g_b0, g_w1, g_b1 = (torch.full(shape, float("nan"), device=DEV) for shape in ((h,), (h,), (h, h), (h,)))
    p, st = ops._p, ops._stream()
    _lib.call("hgb_egnn_edge_bwd_data", p(dummy), p(dummy), p(dummy), p(dummy), p(masks), p(rp), p(idx), 0, h, 1, p(dummy), h, p(dummy),
              p(dummy), p(g_wd), p(g_b0), p(ws), st)
    _lib.call("hgb_egnn_edge_wgrad", p(dummy), p(dummy), p(dummy), p(dummy), p(dummy), p(masks), p(rp), p(idx), p(idx), 0, h, 1, 0,
              p(g_w1), p(g_b1), p(ws), st)
    torch.cuda.synchronize()
    for name, t in (("g_wd", g_wd), ("g_b0", g_b0), ("g_w1", g_w1), ("g_b1", g_b1)):
        assert bool((t == 0).all()), name
