"""Kernel-level tests of the fused message-passing convolutions against the fp64 restatements of conv_reference.py:
hgb_pna_conv_{fwd,bwd}, hgb_pnaplus_conv_{fwd,bwd} and hgb_cgconv_{fwd,bwd} (csrc/hgb_seg.cu), hgb_gat_{fwd,bwd} and
hgb_gat_dropout_keep (csrc/hgb_gat.cu), hgb_cfconv_{fwd,bwd} (csrc/hgb_schnet.cu).

The C-ABI is called directly through the guard-row harness of kernel_harness.py: every operand is the leading block of a
NaN- or sentinel-filled buffer followed by guard rows, "unaligned" operands start one float into their buffer, and g_p of
odd widths uses a row stride of f + 3.  After each call every element in range must be written and everything else (guard
rows and the gap columns of a strided g_p included) must keep its fill bits.  Every case runs twice and must give the same
bits, and its launch count must match the restated host rule.

Accuracy is judged element by element: |x - ref| <= k L u (S + |ref|) with u = 2^-24, L the segment length plus the
per-edge operation count, k from K and, for PNAConv, S the sum of the magnitudes of the terms (Higham, Accuracy and Stability of
Numerical Algorithms, 2nd ed., 3.1): for the messages h_e = P[i] + Q[j] + c + M a_e, S sums |P[i]| + |Q[j]| + |c| +
|M| |a_e| over the segment; for the backward, the magnitudes of the terms of g_h_e, the std term weighted by the d + 4
operations of h_e it repeats.  The variance behind the std is held to its cancellation bound relative to E[S^2], and
outside that band around the 1e-5 threshold the mask must agree with fp64.  Arg-min / arg-max must name an edge whose fp64
message lies within the bound of the extremum, and with dyadic inputs, where every message is exact, the first extremum in
CSR order.  PNAPlus, CGConv, GATv2 and CFConv take S from their restatement evaluated at the absolute values of every
input, plus the largest |ref| of the tensor (see `near`).  Rel-L2 against fp64 is kept as a second witness; the GAT dropout
mask must equal a Python restatement of its Philox draw bit for bit.

`pna_plan`, `pnap_plan`, `cgc_plan`, `gat_plan` and `cf_plan` restate the host dispatch.  `test_cases_reach_every_branch`
(no GPU) asserts that the case lists reach every instantiation (PNA lane widths, vector forms, channel tiles and register
capacities; PNAPlus NC and 8 / 4 backward warps; CGConv CPT and group widths; every GAT (VEC, NV); CFConv NT) and a
grid-stride wrap, more than twice the per-pass capacity, of every forward and backward launch.
`test_launch_rules_at_their_extremes` (no GPU) pins the rules at their largest shapes and the branches no supported shape
reaches."""
import functools
import math

import numpy as np
import pytest
import torch

import conv_reference
from hydragnn_b200 import _lib
from kernel_harness import GRID_CAP, NUM_SMS, U, Buf, cdiv, grid_for, launches, stream, twice
from stack_support import _graph

H100_SMEM_OPTIN = 227 * 1024             # cudaDevAttrMaxSharedMemoryPerBlockOptin on an H100 (232,448 bytes)
BIG_N, BIG_E = 40_000, 200_000
# error constants k of |x - ref| <= k L u S, per kernel
K = dict(pna=2)


# ---- the host dispatch, restated ---------------------------------------------------------------------------------------------
def pna_plan(n, f, d, aligned, bwd):
    """pna_launch: float4 rows when f % 4 == 0 and pq (and g_h in the backward) are 16-byte aligned; `lanes` threads per
    target up to 256, blockIdx.y the channel tile; the register capacity MAXD 0 / 4 / 16"""
    v4 = f % 4 == 0 and aligned
    cv = f // 4 if v4 else f
    lanes = 1
    while lanes < cv and lanes < 256:
        lanes <<= 1
    gpb = 256 // lanes
    gx = grid_for(n, gpb, NUM_SMS * 4 if bwd else GRID_CAP)
    gy = cdiv(cv, lanes)
    maxd = 0 if d == 0 else (4 if d <= 4 else 16)
    kind = "pna_bwd" if bwd else "pna_fwd"
    cap = gx * gpb
    tags = {"%s:vec%d" % (kind, 4 if v4 else 1), "%s:lanes%d" % (kind, lanes), "%s:maxd%d" % (kind, maxd)}
    if gy > 1:
        tags.add("%s:grid_y%d" % (kind, gy))
    if n > 2 * cap:
        tags.add(kind + ":wrap")
    return dict(v4=v4, lanes=lanes, gpb=gpb, grid=(gx, gy), cap=cap, tags=tags, launches=(1 + bwd) if n else int(bwd))


def pnap_plan(n, f, r, d, grads):
    params = f * (f | 1) + 2 * r * f + d * f + 2 * f + r
    grad_smem = (f + d * f + f * f + 2 * r * f + f + r) + f * ((f | 1) - f)
    per_warp = 2 * f + (grad_smem if grads else 0)
    warps = 8 if (params + 8 * per_warp) * 4 <= 200 * 1024 else 4
    nc = 1 if f <= 32 else 2
    fwd_cap = grid_for(n, 8) * 8
    bwd_cap = grid_for(n, warps, NUM_SMS * 2) * warps
    tags = {"pnap:nc%d" % nc, "pnap_bwd:warps%d" % warps}
    if n > 2 * fwd_cap:
        tags.add("pnap_fwd:wrap")
    if n > 2 * bwd_cap:
        tags.add("pnap_bwd:wrap")
    return dict(warps=warps, tags=tags, fwd_launches=int(n > 0), bwd_launches=(1 + grads) if n else 0)


def cgc_plan(n, e, f, d, grads):
    """cgc_launch: CPT channels per lane, groups of 2^gl2 lanes per target; the backward always runs 8 warps"""
    cpt = 1 if f <= 32 else (2 if f <= 64 else 4)
    gl2 = 0
    while (1 << gl2) < f and gl2 < 5:
        gl2 += 1
    params = (d + 1) * 2 * f
    slots = (d + 1) * 2 * cpt * 32 if grads else 0
    bwd_smem = (params + 8 * slots) * 4
    fwd_cap = grid_for(n, 256 >> gl2) * (256 >> gl2)
    bwd_cap = grid_for(n, 8 * (32 >> gl2), NUM_SMS * 4) * 8 * (32 >> gl2)
    tags = {"cgc:cpt%d" % cpt, "cgc:gl2_%d" % gl2}
    live = n > 0 and e > 0
    if live and n > 2 * fwd_cap:
        tags.add("cgc_fwd:wrap")
    if live and n > 2 * bwd_cap:
        tags.add("cgc_bwd:wrap")
    return dict(bwd_smem=bwd_smem, tags=tags, fwd_launches=int(live), bwd_launches=(1 + grads) if live else 0)


def gat_bwd_warps(hc, d, gl2, grads):
    for w in (8, 4, 2):
        groups = w * (32 >> gl2)
        fl = (d + 1) * hc + groups * 2 * 16 + (groups * (d + 1) * hc if grads else 0)
        if fl * 4 <= 200 * 1024:
            return w
    return 1


def gat_plan(n, heads, c, d, aligned, grads):
    hc = heads * c
    vec = 4 if c % 4 == 0 and aligned else 1
    nvec = hc // vec
    gl2 = 0
    while (1 << gl2) < nvec and gl2 < 5:
        gl2 += 1
    need = cdiv(nvec, 1 << gl2)
    nv = need if vec == 4 else (need if need <= 2 else (4 if need <= 4 else (8 if need <= 8 else 16)))
    ok = 1 <= heads <= 8 and hc <= (512 if c % 4 == 0 else 256) and 0 <= d <= 16 and (vec == 4 or hc <= 256)
    gpw = 32 >> gl2
    warps = gat_bwd_warps(hc, d, gl2, grads)
    caps = dict(fwd=grid_for(n, 8 * gpw) * 8 * gpw, bwd_a=grid_for(n, warps * gpw, NUM_SMS * 4) * warps * gpw,
                bwd_b=grid_for(n, 256 >> gl2) * (256 >> gl2))
    tags = {"gat:vec%d_nv%d" % (vec, nv), "gat_bwd_a:warps%d" % warps}
    for kind, cap in caps.items():
        if n > 2 * cap:
            tags.add("gat_%s:wrap" % kind)
    return dict(ok=ok, vec=vec, nv=nv, warps=warps, tags=tags, fwd_launches=int(ok and n > 0),
                bwd_launches=(2 + grads) if ok and n > 0 else 0)


def cf_bwd_smem(g, nf, k1, nw):
    return 4 * (k1 * nf + nf * (nf + 1) + 2 * nf + g + nw * (k1 + 3 * nf) + k1 * nf + 2 * nf + nf * nf)


def cf_bwd_warps(g, nf, k1, limit=H100_SMEM_OPTIN):
    nw = 8
    while nw > 1 and cf_bwd_smem(g, nf, k1, nw) > limit:
        nw >>= 1
    return nw


def cf_plan(n, e, g, nf, d, grads):
    nt = cdiv(nf, 32)
    nw = cf_bwd_warps(g, nf, g + d)
    fwd_cap = grid_for(n, 8, NUM_SMS * 2) * 8
    bwd_cap = grid_for(e, nw, NUM_SMS) * nw
    tags = {"cf:nt%d" % nt, "cf_bwd:warps%d" % nw}
    if n > 2 * fwd_cap:
        tags.add("cf_fwd:wrap")
    if e > 2 * bwd_cap:
        tags.add("cf_bwd:wrap")
    return dict(nw=nw, tags=tags, fwd_launches=int(n > 0), bwd_launches=(1 + grads) if e else 1)


# ---- case lists -------------------------------------------------------------------------------------------------------------
# graphs: "small" = stack_support._graph (n 3000, a target of in-degree 1000, runs of in-degree 0, 1, 2); "big" (n 40,000,
# e 200,000, a target of in-degree 4096, runs of in-degree 0, 1, 2, duplicate edges); "sorted" = small with its edges in
# target order, passed with perm = NULL; "loops" = small plus targets whose only in-edges are input self-loops; "pairs" = 300
# targets of in-degree 2 (PNA: variances at the std mask threshold); "empty" = 50 nodes, no edges
GRAPH_N = dict(small=3000, big=BIG_N, sorted=3000, loops=3000, pairs=900, empty=50)
GRAPH_E = dict(small=4300, big=BIG_E + 3000, sorted=4300, loops=4330, pairs=600, empty=0)

# PNAConv: (graph, f, d, aligned, cvec, dyadic)
PNA_F = [1, 3, 4, 5, 64, 255, 256, 257, 1024, 1028]
PNA_CASES = ([("small", f, d, True, True, False) for f in PNA_F for d in ((0, 5) if f >= 255 else (0, 1, 4, 16))] +
             [("small", 64, 4, False, True, False), ("small", 1024, 1, False, True, False), ("small", 128, 16, True, True, False),
              ("small", 128, 1, False, True, False), ("small", 8, 0, True, False, False),
              ("small", 5, 3, True, True, True), ("small", 64, 0, True, True, True),
              ("pairs", 4, 0, True, False, False), ("pairs", 3, 0, True, False, False), ("sorted", 33, 16, True, True, False),
              ("big", 5, 1, True, True, False), ("big", 64, 0, False, True, False)])

# branches no supported shape reaches, with the arithmetic that shows it (checked in test_launch_rules_at_their_extremes)
UNREACHABLE = {
    "gat_bwd_a:warps2": "(d + 1) hc (1 + 4 groups) + 128 groups floats exceed 200 KB at 4 warps only for (d + 1) hc > 10,214; "
                        "hc <= 512 and d <= 16 give at most 8,704",
    "gat_bwd_a:warps1": "as warps2",
    "cf_bwd:warps4": "at g = 64, nf = 128, d = 16 the 8-warp backward needs 230,656 bytes, within the 232,448-byte opt-in limit",
    "cf_bwd:warps2": "as warps4",
    "cf_bwd:warps1": "as warps4",
}


def all_tags():
    """tags of every case of every list: which branches and grid-stride wraps the GPU tests reach"""
    tags = set()
    for gname, f, d, al, _, _ in PNA_CASES:
        for bwd in (False, True):
            tags |= pna_plan(GRAPH_N[gname], f, d, al, bwd)["tags"]
    for gname, f, r, d, _, grads, _, _ in PNAP_CASES:
        tags |= pnap_plan(GRAPH_N[gname], f, r, d, grads)["tags"]
    for gname, f, d, grads, _ in CGC_CASES:
        tags |= cgc_plan(GRAPH_N[gname], GRAPH_E[gname], f, d, grads)["tags"]
    for gname, h, c, d, _, al, grads, _, _ in GAT_CASES:
        tags |= gat_plan(GRAPH_N[gname], h, c, d, al, grads)["tags"]
    for gname, nf, g, d, _, _, _, grads in CF_CASES:
        tags |= cf_plan(GRAPH_N[gname], GRAPH_E[gname], g, nf, d, grads)["tags"]
    return tags


def test_cases_reach_every_branch():
    need = set()
    for kind in ("pna_fwd", "pna_bwd"):
        need |= {"%s:vec4" % kind, "%s:vec1" % kind, "%s:grid_y2" % kind, kind + ":wrap"}
        need |= {"%s:lanes%d" % (kind, 1 << k) for k in range(9)}
        need |= {"%s:maxd%d" % (kind, m) for m in (0, 4, 16)}
    need |= {"pnap:nc1", "pnap:nc2", "pnap_bwd:warps8", "pnap_bwd:warps4", "pnap_fwd:wrap", "pnap_bwd:wrap"}
    need |= {"cgc:cpt%d" % c for c in (1, 2, 4)} | {"cgc:gl2_%d" % g for g in range(6)} | {"cgc_fwd:wrap", "cgc_bwd:wrap"}
    need |= {"gat:vec4_nv%d" % v for v in (1, 2, 3, 4)} | {"gat:vec1_nv%d" % v for v in (1, 2, 4, 8)}
    need |= {"gat_bwd_a:warps8", "gat_bwd_a:warps4", "gat_fwd:wrap", "gat_bwd_a:wrap", "gat_bwd_b:wrap"}
    need |= {"cf:nt%d" % t for t in (1, 2, 3, 4)} | {"cf_bwd:warps8", "cf_fwd:wrap", "cf_bwd:wrap"}
    tags = all_tags()
    missing = need - tags
    assert not missing, "case lists miss %s" % sorted(missing)
    assert not (tags & set(UNREACHABLE)), sorted(tags & set(UNREACHABLE))
    assert all(not gat_plan(3000, h, c, 0, False, True)["ok"] for h, c in GAT_REFUSED)
    assert all(gat_plan(GRAPH_N[gname], h, c, d, al, grads)["ok"] for gname, h, c, d, _, al, grads, _, _ in GAT_CASES)
    assert pna_plan(BIG_N, 64, 0, False, True)["cap"] == 2112 and pna_plan(BIG_N, 5, 0, True, True)["cap"] == 16_896
    assert pna_plan(1, 1028, 0, True, False)["grid"] == (1, 2) and pna_plan(1, 257, 0, True, False)["grid"] == (1, 2)
    assert {"small": 4300, "big": 203_000}.items() <= GRAPH_E.items()


def test_launch_rules_at_their_extremes():
    # GAT pass A: 4 warps at heads c = 512 with d = 16 and parameter gradients, never fewer at any supported shape
    for h, c in ((1, 512), (8, 64), (4, 128)):
        assert gat_bwd_warps(h * c, 16, 5, True) == 4 and gat_bwd_warps(h * c, 16, 5, False) == 8
    plans = [gat_plan(1, 1, hc, d, al, True) for hc in range(1, 513) for d in (0, 16) for al in (False, True)]
    assert min(p["warps"] for p in plans if p["ok"]) == 4
    assert {"gat_bwd_a:warps2", "gat_bwd_a:warps1"} <= set(UNREACHABLE)
    # GAT shapes: up to 512 with whole float4 heads, 256 otherwise; above 256 unaligned operands are refused
    assert gat_plan(1, 8, 64, 16, True, True)["ok"] and not gat_plan(1, 8, 64, 16, False, True)["ok"]
    assert not gat_plan(1, 1, 257, 0, True, True)["ok"] and gat_plan(1, 1, 256, 0, False, True)["ok"]
    assert gat_plan(1, 8, 64, 0, True, False)["nv"] == 4 and gat_plan(1, 8, 32, 0, False, False)["nv"] == 8
    # CFConv: 8 backward warps at every supported shape under the H100's opt-in limit
    assert all(cf_bwd_warps(g, nf, g + d) == 8 for g in (1, 64) for nf in range(1, 129) for d in (0, 16))
    assert cf_bwd_smem(64, 128, 80, 8) == 230_656 <= H100_SMEM_OPTIN == 232_448
    assert {"cf_bwd:warps4", "cf_bwd:warps2", "cf_bwd:warps1"} <= set(UNREACHABLE)
    # CGConv: the 8-warp backward fits at the largest shape, so it needs no fallback
    assert cgc_plan(1, 1, 128, 16, True)["bwd_smem"] == 156_672 <= H100_SMEM_OPTIN
    # PNAPlus: the backward drops to 4 warps for wide rows with parameter gradients only
    assert pnap_plan(1, 64, 16, 16, True)["warps"] == 4 and pnap_plan(1, 64, 16, 16, False)["warps"] == 8
    assert pnap_plan(1, 47, 16, 16, True)["warps"] == 8


# ---- graphs -----------------------------------------------------------------------------------------------------------------
@functools.lru_cache(maxsize=None)
def graph(name):
    """(src, dst, n) as int64 numpy arrays"""
    if name in ("small", "sorted", "loops"):
        ei, n = _graph()
        src, dst = (x.cpu().numpy() for x in ei)
        if name == "sorted":
            o = np.argsort(dst, kind="stable")
            src, dst = src[o], dst[o]
        if name == "loops":                    # 50..59: only input self-loops; 60..69: a self-loop and one other edge
            src = np.concatenate([src, np.arange(50, 70), np.arange(0, 10)])
            dst = np.concatenate([dst, np.arange(50, 70), np.arange(60, 70)])
        return src.astype(np.int64), dst.astype(np.int64), n
    if name == "pairs":                        # target i < 300 receives exactly the edges 300 + 2 i -> i and 301 + 2 i -> i
        t = np.repeat(np.arange(300), 2)
        return 300 + np.arange(600), t, 900
    if name == "empty":
        return np.zeros(0, np.int64), np.zeros(0, np.int64), 50
    rng = np.random.default_rng(1)
    n = BIG_N
    fixed = np.concatenate([np.zeros(4096, np.int64), np.arange(1300, 1600), np.repeat(np.arange(1600, 1900), 2)])
    rest = rng.integers(2000, n, BIG_E - fixed.size - 3000)                     # nodes 1..1299 receive nothing
    dst = np.concatenate([fixed, rest])
    src = rng.integers(0, n, dst.size)
    dup = rng.integers(0, dst.size, 1000)                                        # duplicate edges, three copies each
    src, dst = np.concatenate([src, np.repeat(src[dup], 3)]), np.concatenate([dst, np.repeat(dst[dup], 3)])
    o = rng.permutation(dst.size)
    return src[o], dst[o], n


def csr_of(key, other, n, identity):
    """(rowptr, perm or None, other[perm]) of the CSR by `key`, stable in edge id"""
    perm = np.argsort(key, kind="stable")
    rowptr = np.concatenate([[0], np.cumsum(np.bincount(key, minlength=n))])
    if identity:
        assert np.array_equal(perm, np.arange(key.size))
    return rowptr.astype(np.int32), None if identity else perm.astype(np.int32), other[perm].astype(np.int32)


def ibuf(a):
    return Buf(len(a), dtype=torch.int32, data=torch.from_numpy(np.asarray(a, np.int32))) if a is not None else None


def fbuf(t, off=0, ld=None):
    t = torch.as_tensor(t, dtype=torch.float32)
    t2 = t if t.dim() == 2 else t.reshape(-1, 1)
    return Buf(t2.shape[0], t2.shape[1], ld=ld, off=off, data=t2)


def ptr(b):
    return b.ptr if b is not None else None


def within(what, got, ref, scale, L, k):
    """|got - ref| <= k L u (scale + |ref|) element by element (L broadcasts), and rel-L2 as a second witness"""
    got = torch.as_tensor(np.asarray(got), dtype=torch.float64)
    ref, scale = ref.detach().double().cpu(), scale.detach().double().cpu()
    L = torch.as_tensor(L, dtype=torch.float64)
    bound = k * L * U * (scale + ref.abs()) + 2.0 ** -120
    err = (got - ref).abs()
    bad = ~(err <= bound)
    if bool(bad.any()):
        i = int(torch.argmax(torch.where(bad, err / bound, torch.zeros_like(err))))
        pytest.fail("%s: %d of %d entries off their bound (k = %g); worst flat index %d: |err| %.3g, bound %.3g, ref %.8g, got %.8g"
                    % (what, int(bad.sum()), bad.numel(), k, i, err.flatten()[i], bound.flatten()[i], ref.flatten()[i],
                       got.flatten()[i]))
    den = float(ref.norm())
    if den > 0:                                # 1e-4, or the normwise form of the bound above where cancellation makes it wider
        tol = max(1e-4, float(bound.norm()) / den)
        assert float((got - ref).norm()) / den <= tol, "%s: rel-L2 %.3g > %.3g" % (what, float((got - ref).norm()) / den, tol)


def seg_len(dst, n):
    return torch.from_numpy(np.bincount(dst, minlength=n).astype(np.float64))


# ---- PNAConv ----------------------------------------------------------------------------------------------------------------
def pna_inputs(n, e, f, d, seed, dyadic, with_c):
    g = torch.Generator().manual_seed(seed)
    r = ((lambda *s: torch.randint(-4, 5, s, generator=g).double() * 0.25) if dyadic
         else (lambda *s: torch.randn(*s, generator=g, dtype=torch.float64)))
    pq = r(n, 2 * f)
    c = r(f) if with_c else None
    ea, mt = (r(e, d), r(d, f) * 0.5) if d else (None, None)
    if n == 900:                                # "pairs": target i's messages are 0 and 2 delta_i, variance delta_i^2 near 1e-5
        pq[:] = 0.0
        rel = torch.tensor([-1e-2, -1e-3, -1e-4, 0.0, 1e-4, 1e-3, 1e-2], dtype=torch.float64)
        var = 1e-5 * (1 + rel[torch.arange(300) % rel.numel()])
        pq[301 + 2 * torch.arange(300), f:] = (2 * var.sqrt())[:, None] * (1 + torch.arange(f, dtype=torch.float64) * 1e-6)
    return [x.float().double() if x is not None else None for x in (pq, ea, mt, c)]


@pytest.mark.gpu
@pytest.mark.parametrize("gname,f,d,aligned,with_c,dyadic", PNA_CASES)
def test_pna_conv(gname, f, d, aligned, with_c, dyadic):
    src, dst, n = graph(gname)
    e = src.size
    rowptr, perm, slot_src = csr_of(dst, src, n, gname == "sorted")
    pq, ea, mt, c = pna_inputs(n, e, f, d, f * 31 + d, dyadic, with_c)
    off = 0 if aligned else 1
    B = dict(pq=fbuf(pq, off), ea=fbuf(ea) if d else None, mt=fbuf(mt) if d else None, c=fbuf(c) if with_c else None,
             rowptr=ibuf(rowptr), perm=ibuf(perm), src=ibuf(slot_src))
    out, amin, amax = Buf(n, 4 * f, off=off), Buf(n, f, dtype=torch.int32), Buf(n, f, dtype=torch.int32)
    fwd = lambda: _lib.call("hgb_pna_conv_fwd", B["pq"].ptr, B["rowptr"].ptr, ptr(B["perm"]), B["src"].ptr, ptr(B["ea"]), d,
                            ptr(B["mt"]), ptr(B["c"]), n, f, out.ptr, amin.ptr, amax.ptr, stream())
    plan = pna_plan(n, f, d, B["pq"].ptr % 16 == 0, False)
    assert launches(fwd) == plan["launches"]
    for b, nm in ((out, "out"), (amin, "argmin"), (amax, "argmax")):
        b.check("pna_fwd", nm)
    twice("pna_fwd", fwd, [out, amin, amax])
    ei = torch.from_numpy(np.stack([src, dst]))
    ragg, ramin, ramax, h = (x.cpu() for x in conv_reference.pna_fwd(pq, ea, mt, c, ei, n))
    habs = pq[:, :f].abs()[dst] + pq[:, f:].abs()[src] + (c.abs() if with_c else 0) + (ea.abs() @ mt.abs() if d else 0)
    L = seg_len(dst, n)[:, None]
    cnt = L.clamp(min=1)
    k = K["pna"]
    agg = torch.from_numpy(out.np()).double()
    dt = torch.from_numpy(dst)
    sabs = torch.zeros(n, f, dtype=torch.float64).index_add_(0, dt, habs)
    mabs = torch.zeros(n, f, dtype=torch.float64).scatter_reduce(0, dt[:, None].expand(-1, f), habs, "amax")
    within("pna_fwd mean", agg[:, :f], ragg[:, :f], sabs / cnt, L + d + 3, k)
    within("pna_fwd min", agg[:, f:2 * f], ragg[:, f:2 * f], mabs, d + 3, k)
    within("pna_fwd max", agg[:, 2 * f:3 * f], ragg[:, 2 * f:3 * f], mabs, d + 3, k)
    # std: the variance carries (L + d + 4) u E[habs^2]; outside that band around the 1e-5 mask the mask agrees with fp64
    ex2 = torch.zeros(n, f, dtype=torch.float64).index_add_(0, dt, habs * habs) / cnt
    vb = k * (L + d + 5) * U * ex2 * 4
    var = torch.zeros(n, f, dtype=torch.float64).index_add_(0, dt, h * h) / cnt - ragg[:, :f] ** 2
    far = (var - 1e-5).abs() > vb
    sd, rsd = agg[:, 3 * f:], ragg[:, 3 * f:]
    assert int((((sd > 0) != (rsd > 0)) & far).sum()) == 0, "pna_fwd: std mask differs from fp64 away from the threshold"
    both = (sd > 0) & (rsd > 0) & far
    assert bool(((sd * sd - rsd * rsd).abs()[both] <= vb[both]).all()), "pna_fwd: variance outside its bound"
    # arg-min / arg-max: the kernel's edge holds the extremum within the message bound (exactly, with dyadic inputs)
    for nm, got, ref, col in (("argmin", amin, ramin, 1), ("argmax", amax, ramax, 2)):
        gi = torch.from_numpy(got.np()).long()
        assert torch.equal(gi < 0, ref < 0), "pna_fwd %s: empty segments" % nm
        own = torch.from_numpy(dst)[gi.clamp(min=0)] == torch.arange(n)[:, None]
        assert bool((own | (gi < 0)).all()), "pna_fwd %s names an edge of another target" % nm
        if dyadic:
            assert torch.equal(gi, ref), "pna_fwd %s: first extremum in CSR order" % nm
        else:
            hv = h[gi.clamp(min=0), torch.arange(f)[None, :].expand(n, -1)]
            ok = ((hv - ragg[:, col * f:(col + 1) * f]).abs() <= k * (d + 3) * U * mabs * 2) | (gi < 0)
            assert bool(ok.all()), "pna_fwd %s names an edge away from the extremum" % nm
    # backward, against fp64 given the kernel's forward
    gq = torch.randn(n, 4 * f, generator=torch.Generator().manual_seed(3), dtype=torch.float64).float().double()
    g_out = fbuf(gq, off)
    ldgp = f + 3 if f % 2 else f
    g_p, g_h = Buf(n, f, ld=ldgp), Buf(e, f, off=off)
    g_cm = Buf(d + 1, f)
    ws = Buf(cdiv(_lib.query("hgb_pna_conv_workspace_bytes", f, d), 4))
    bwd = lambda: _lib.call("hgb_pna_conv_bwd", g_out.ptr, B["pq"].ptr, B["rowptr"].ptr, ptr(B["perm"]), B["src"].ptr, ptr(B["ea"]),
                            d, ptr(B["mt"]), ptr(B["c"]), out.ptr, amin.ptr, amax.ptr, n, f, g_p.ptr, ldgp, g_h.ptr, g_cm.ptr,
                            ws.ptr, stream())
    bplan = pna_plan(n, f, d, B["pq"].ptr % 16 == 0 and g_h.ptr % 16 == 0, True)
    assert launches(bwd) == bplan["launches"]
    for b, nm in ((g_p, "g_p"), (g_h, "g_h"), (g_cm, "g_cm")):
        b.check("pna_bwd", nm)
    twice("pna_bwd", bwd, [g_p, g_h, g_cm])
    am, ax = torch.from_numpy(amin.np()).long(), torch.from_numpy(amax.np()).long()
    rgh, rgp, _, rgc, rgm, _ = (x.cpu() if x is not None else None
                                for x in conv_reference.pna_bwd(gq, agg, am, ax, h, ea, mt, ei, n))
    eid = torch.arange(e)[:, None]
    kstd = torch.where(sd > 0, gq[:, 3 * f:].abs() / (cnt * sd.clamp(min=1e-30)), torch.zeros_like(sd))
    ghabs = (gq[:, :f].abs() / cnt)[dt] + (am[dt] == eid) * gq[:, f:2 * f].abs()[dt] + (ax[dt] == eid) * gq[:, 2 * f:3 * f].abs()[dt] \
        + kstd[dt] * (habs + agg[:, :f].abs()[dt]) * (d + 4)
    within("pna_bwd g_h", g_h.np(), rgh, ghabs, d + 6, k)
    within("pna_bwd g_p", g_p.np(), rgp, torch.zeros(n, f, dtype=torch.float64).index_add_(0, dt, ghabs), L + d + 6, k)
    lpar = min(e, cdiv(n, bplan["cap"]) * int(L.max())) + bplan["gpb"] + d + 6
    gcm = torch.from_numpy(g_cm.np()).double()
    within("pna_bwd g_c", gcm[0], rgc, ghabs.sum(0), lpar, k)
    if d:
        within("pna_bwd g_M", gcm[1:], rgm, ea.abs().t() @ ghabs, lpar, k)


# ---- shared pieces of the other four kernels --------------------------------------------------------------------------------
def near(what, got, ref, absref, L, k):
    """within() with S = the restatement at |inputs| plus the largest |ref| of the tensor.  The restatement at |inputs| does
    not see the cancellation inside the Bessel envelope, the cosine cutoff and the softmax (each sums terms of both signs
    whatever the sign of the inputs), so the floor of this bound is normwise: every element within k L u max |ref|."""
    ref, absref = ref.detach().double().cpu(), absref.detach().double().cpu()
    if ref.numel() == 0:
        assert np.asarray(got).size == 0, what
        return
    within(what, got, ref, absref.abs() + ref.abs().max(), L, k)


def abs_inputs(t):
    return {k: (v.abs() if v is not None and v.is_floating_point() else v) for k, v in t.items()}


def supported(name, *args):
    return _lib.query(name, *[int(a) for a in args]) == 1


def extremum_ids(what, got, m, ref_val, dst, n, bound):
    """arg-min / arg-max ids: -1 exactly for empty targets, otherwise an edge of the row's own segment whose fp64 message
    lies within `bound` of the extremum"""
    gi = torch.from_numpy(got).long()
    deg = torch.from_numpy(np.bincount(dst, minlength=n))
    assert torch.equal(gi < 0, (deg == 0)[:, None].expand_as(gi)), "%s: empty segments" % what
    own = torch.from_numpy(dst)[gi.clamp(min=0)] == torch.arange(n)[:, None]
    assert bool((own | (gi < 0)).all()), "%s names an edge of another target" % what
    f = gi.shape[1]
    val = m[gi.clamp(min=0), torch.arange(f)[None, :].expand(n, -1)]
    assert bool((((val - ref_val).abs() <= bound) | (gi < 0)).all()), "%s names an edge away from the extremum" % what


def seg_scale(habs, dst, n, reduce):
    f = habs.shape[1]
    dt = torch.from_numpy(dst)
    if reduce == "sum":
        return torch.zeros(n, f, dtype=torch.float64).index_add_(0, dt, habs)
    return torch.zeros(n, f, dtype=torch.float64).scatter_reduce(0, dt[:, None].expand(-1, f), habs, "amax")


# ---- PNAPlus ----------------------------------------------------------------------------------------------------------------
RADIUS = 2.0
K.update(pnaplus=16, cgconv=8, gat=16, cfconv=16)

# (graph, f, r, d, expo, grads, g_dist, g_eattr)
PNAP_CASES = ([("small", f, r, d, (5, 2, 0)[(f + r) % 3], True, True, d > 0) for f in (1, 31, 32, 33, 64)
               for r, d in ((1, 0), (8, 16), (16, 16))] +
              [("small", 64, 16, 16, 5, False, True, True), ("small", 33, 8, 4, 2, True, False, False),
               ("small", 32, 16, 0, 5, False, False, False), ("sorted", 64, 8, 1, 5, True, True, True),
               ("big", 33, 8, 0, 5, True, True, False), ("big", 64, 4, 2, 5, True, False, False)])


def pnap_inputs(src, dst, n, f, r, d, seed):
    g = torch.Generator().manual_seed(seed)
    e = src.size
    dist = torch.rand(e, generator=g, dtype=torch.float64) * 0.9 * RADIUS + 0.05 * RADIUS
    edge = torch.arange(e)
    r32 = np.float32(RADIUS)
    dist[edge % 11 == 0] = 1.3 * RADIUS                                          # past the radius: rbf 0, message 0
    dist[edge % 11 == 1] = RADIUS                                                # x = 1 exactly
    dist[edge % 11 == 2] = float(np.nextafter(r32, np.float32(0)))               # x one ulp below 1
    dist[edge % 11 == 3] = 1e-3 * RADIUS                                         # near 0: env ~ 1 / x
    t = dict(pq=torch.randn(n, 2 * f, generator=g, dtype=torch.float64), dist=dist,
             freq=math.pi * torch.arange(1, r + 1, dtype=torch.float64) + 0.1 * torch.randn(r, generator=g, dtype=torch.float64),
             wr=torch.randn(f, r, generator=g, dtype=torch.float64) * 0.5, br=torch.randn(f, generator=g, dtype=torch.float64) * 0.5,
             wl=torch.randn(f, r, generator=g, dtype=torch.float64) * 0.5,
             mr=torch.randn(f, f, generator=g, dtype=torch.float64) / f ** 0.5, cvec=torch.randn(f, generator=g, dtype=torch.float64),
             eattr=torch.randn(e, d, generator=g, dtype=torch.float64) if d else None,
             mat=torch.randn(d, f, generator=g, dtype=torch.float64) * 0.5 if d else None)
    return {k: (v.float().double() if v is not None else None) for k, v in t.items()}


def pnap_backward_ref(t, ei, n, expo, g_m):
    """fp64 gradients of <m, g_m> (g_m = dL/dm per edge): g_h, g_P, g_dist, g_eattr, g_params in the kernel's layout"""
    leaves = {k: (v.clone().requires_grad_(True) if v is not None else None) for k, v in t.items()}
    leaves["hz"] = torch.zeros(ei.shape[1], t["pq"].shape[1] // 2, dtype=torch.float64, requires_grad=True)
    m = conv_reference.pnaplus_messages(leaves, ei, RADIUS, expo)
    names = ["hz", "pq", "dist", "cvec", "mr", "wr", "br", "wl", "freq"] + (["eattr", "mat"] if t["eattr"] is not None else [])
    gr = dict(zip(names, torch.autograd.grad(m, [leaves[k] for k in names], g_m)))
    f = t["pq"].shape[1] // 2
    par = [gr["cvec"]] + ([gr["mat"].reshape(-1)] if "mat" in gr else []) + [gr["mr"].reshape(-1), gr["wr"].t().reshape(-1),
                                                                             gr["br"], gr["wl"].t().reshape(-1), gr["freq"]]
    return gr["hz"], gr["pq"][:, :f], gr["dist"], gr.get("eattr"), torch.cat(par), m.detach()


@pytest.mark.gpu
@pytest.mark.parametrize("gname,f,r,d,expo,grads,gdist,geattr", PNAP_CASES)
def test_pnaplus_conv(gname, f, r, d, expo, grads, gdist, geattr):
    src, dst, n = graph(gname)
    e = src.size
    assert supported("hgb_pnaplus_conv_supported", f, r, d)
    rowptr, perm, slot_src = csr_of(dst, src, n, gname == "sorted")
    t = pnap_inputs(src, dst, n, f, r, d, f * 100 + d * 10 + r)
    B = {k: (fbuf(v) if v is not None else None) for k, v in t.items()}
    B["dist"] = fbuf(t["dist"][:, None])
    I = dict(rowptr=ibuf(rowptr), perm=ibuf(perm), src=ibuf(slot_src))
    params = lambda: [ptr(B["eattr"]), d, B["freq"].ptr, r, RADIUS, expo, B["wr"].ptr, B["br"].ptr, B["wl"].ptr, B["mr"].ptr,
                      ptr(B["mat"]), B["cvec"].ptr]
    out, amin, amax = Buf(n, 4 * f), Buf(n, f, dtype=torch.int32), Buf(n, f, dtype=torch.int32)
    fwd = lambda: _lib.call("hgb_pnaplus_conv_fwd", B["pq"].ptr, B["dist"].ptr, I["rowptr"].ptr, ptr(I["perm"]), I["src"].ptr,
                            *params(), n, f, out.ptr, amin.ptr, amax.ptr, stream())
    plan = pnap_plan(n, f, r, d, grads)
    assert launches(fwd) == plan["fwd_launches"]
    for b, nm in ((out, "out"), (amin, "argmin"), (amax, "argmax")):
        b.check("pnaplus_fwd", nm)
    twice("pnaplus_fwd", fwd, [out, amin, amax])
    ei = torch.from_numpy(np.stack([src, dst]))
    k = K["pnaplus"]
    m = conv_reference.pnaplus_messages(t, ei, RADIUS, expo)
    mabs = conv_reference.pnaplus_messages(abs_inputs(t), ei, RADIUS, expo).abs()
    L = seg_len(dst, n)[:, None]
    cnt = L.clamp(min=1)
    inner = f + r + d + 8
    ragg = conv_reference.pnaplus_agg(t, ei, n, RADIUS, expo)
    agg = torch.from_numpy(out.np()).double()
    smax = seg_scale(mabs, dst, n, "max")
    near("pnaplus_fwd mean", agg[:, :f], ragg[:, :f], seg_scale(mabs, dst, n, "sum") / cnt, L + inner, k)
    near("pnaplus_fwd min", agg[:, f:2 * f], ragg[:, f:2 * f], smax, inner, k)
    near("pnaplus_fwd max", agg[:, 2 * f:3 * f], ragg[:, 2 * f:3 * f], smax, inner, k)
    dt = torch.from_numpy(dst)
    # the variance bound takes the same normwise floor as `near`: the largest E[m^2] of the tensor
    ex2r = torch.zeros(n, f, dtype=torch.float64).index_add_(0, dt, m * m) / cnt
    ex2 = torch.zeros(n, f, dtype=torch.float64).index_add_(0, dt, mabs * mabs) / cnt + ex2r.max()
    var = ex2r - ragg[:, :f] ** 2
    far = (var - 1e-5).abs() > 4 * k * (L + inner) * U * ex2
    sd, rsd = agg[:, 3 * f:], ragg[:, 3 * f:]
    assert int((((sd > 0) != (rsd > 0)) & far).sum()) == 0, "pnaplus_fwd: std mask differs from fp64 away from the threshold"
    both = (sd > 0) & (rsd > 0) & far
    assert bool(((sd * sd - rsd * rsd).abs() <= 4 * k * (L + inner) * U * ex2)[both].all()), "pnaplus_fwd: variance"
    for nm, got, col in (("argmin", amin, 1), ("argmax", amax, 2)):
        extremum_ids("pnaplus_fwd " + nm, got.np(), m, ragg[:, col * f:(col + 1) * f], dst, n, 2 * k * inner * U * smax)
    # backward, against fp64 given the kernel's forward (its arg-min / arg-max ids and std)
    gq = torch.randn(n, 4 * f, generator=torch.Generator().manual_seed(3), dtype=torch.float64).float().double()
    g_out = fbuf(gq)
    ldgp = f + 3 if f % 2 else f
    g_p, g_h = Buf(n, f, ld=ldgp), Buf(e, f)
    g_dist = Buf(e) if gdist else None
    g_ea = Buf(e, d) if geattr else None
    npar = f + d * f + f * f + 2 * r * f + f + r
    g_par = Buf(npar) if grads else None
    ws = Buf(cdiv(_lib.query("hgb_pnaplus_conv_workspace_bytes", f, r, d), 4))
    bwd = lambda: _lib.call("hgb_pnaplus_conv_bwd", g_out.ptr, B["pq"].ptr, B["dist"].ptr, I["rowptr"].ptr, ptr(I["perm"]),
                            I["src"].ptr, *params(), out.ptr, amin.ptr, amax.ptr, n, f, g_p.ptr, ldgp, g_h.ptr, ptr(g_dist),
                            ptr(g_ea), ptr(g_par), ws.ptr, stream())
    assert launches(bwd) == plan["bwd_launches"]
    outs = [b for b in (g_p, g_h, g_dist, g_ea, g_par) if b is not None]
    for b in outs:
        b.check("pnaplus_bwd", "output")
    twice("pnaplus_bwd", bwd, outs)
    am, ax = torch.from_numpy(amin.np()).long(), torch.from_numpy(amax.np()).long()
    g_m = conv_reference.pna_bwd(gq, agg, am, ax, m, None, None, ei, n)[0]
    g_mabs = conv_reference.pna_bwd(gq.abs(), agg.abs(), am, ax, mabs, None, None, ei, n)[0].abs()
    rgh, rgp, rgd, rge, rpar, _ = pnap_backward_ref(t, ei, n, expo, g_m)
    agh, agp, agd, age, apar, _ = pnap_backward_ref(abs_inputs(t), ei, n, expo, g_mabs)
    lmax = int(L.max()) + inner
    near("pnaplus_bwd g_h", g_h.np(), rgh, agh, inner, k)
    near("pnaplus_bwd g_p", g_p.np(), rgp, agp, L + inner, k)
    if gdist:
        near("pnaplus_bwd g_dist", g_dist.np()[:, 0], rgd, agd, inner * r, k)
    if geattr:
        near("pnaplus_bwd g_eattr", g_ea.np(), rge, age, inner, k)
    if grads:
        near("pnaplus_bwd g_params", g_par.np()[:, 0], rpar, apar, lmax * max(1, cdiv(n, 2112)) + 264, k)


# ---- CGConv -----------------------------------------------------------------------------------------------------------------
CGC_F = [1, 2, 3, 16, 31, 32, 33, 64, 65, 128]
# (graph, f, d, grads, g_eattr)
CGC_CASES = ([("small", f, d, True, d > 0) for f in CGC_F for d in (0, 1, 16)] +
             [("small", 33, 16, False, False), ("small", 64, 16, False, True), ("sorted", 128, 16, True, True),
              ("big", 32, 1, True, True), ("big", 1, 0, True, False), ("empty", 7, 2, True, True), ("empty", 33, 0, False, False)])


def cgc_inputs(n, e, f, d, seed):
    g = torch.Generator().manual_seed(seed)
    r = lambda *s: torch.randn(*s, generator=g, dtype=torch.float64)              # noqa: E731
    pq, x, cvec = r(n, 4 * f), r(n, f), r(2 * f) * 0.5
    ea, mt = (r(e, d), r(d, 2 * f) * 0.5) if d else (None, None)
    if n >= 3000:
        # targets 100..199 (one in-edge each on the small graph): s = P_s exactly at the softplus threshold 20 and one ulp
        # either side (with d = 0, Q_s and the s bias zeroed); targets 200..299: f = P_f - 120, sigmoid underflows to 0
        t20 = np.float32(20.0)
        pq[100:200, f:2 * f] = torch.tensor([float(np.nextafter(t20, np.float32(0))), 20.0,
                                             float(np.nextafter(t20, np.float32(40)))], dtype=torch.float64)[torch.arange(100) % 3][:, None]
        pq[200:300, :f] -= 120.0
        if d == 0:
            pq[:, 3 * f:] = 0.0
            cvec[f:] = 0.0
    return {k: (v.float().double() if v is not None else None) for k, v in dict(pq=pq, ea=ea, mt=mt, cvec=cvec, x=x).items()}


@pytest.mark.gpu
@pytest.mark.parametrize("gname,f,d,grads,geattr", CGC_CASES)
def test_cgconv(gname, f, d, grads, geattr):
    src, dst, n = graph(gname)
    e = src.size
    assert supported("hgb_cgconv_supported", f, d)
    rowptr, perm, slot_src = csr_of(dst, src, n, gname == "sorted")
    t = cgc_inputs(n, e, f, d, f + 100 * d)
    B = {k: (fbuf(v) if v is not None else None) for k, v in t.items()}
    I = dict(rowptr=ibuf(rowptr), perm=ibuf(perm) if e else Buf(0, dtype=torch.int32), src=ibuf(slot_src))
    out = Buf(n, f)
    fwd = lambda: _lib.call("hgb_cgconv_fwd", B["pq"].ptr, I["rowptr"].ptr, ptr(I["perm"]), I["src"].ptr, ptr(B["ea"]), d,
                            ptr(B["mt"]), B["cvec"].ptr, B["x"].ptr, n, e, f, out.ptr, stream())
    plan = cgc_plan(n, e, f, d, grads)
    assert launches(fwd) == plan["fwd_launches"]
    out.check("cgconv_fwd", "out")
    twice("cgconv_fwd", fwd, [out])
    ei = torch.from_numpy(np.stack([src, dst]))
    g_out = torch.randn(n, f, generator=torch.Generator().manual_seed(3), dtype=torch.float64).float().double()
    tz = dict(t, hz=torch.zeros(e, 2 * f, dtype=torch.float64))
    ref, rg = conv_reference.cgconv(tz, ei, g_out)
    aref, ag = conv_reference.cgconv(dict(abs_inputs(t), hz=tz["hz"]), ei, g_out.abs())
    k = K["cgconv"]
    L = seg_len(dst, n)[:, None] + d + 12
    near("cgconv_fwd out", out.np(), ref, aref, L, k)
    no_edge = (seg_len(dst, n) == 0).numpy()
    assert np.array_equal(out.np()[no_edge], t["x"].float().numpy()[no_edge]), "cgconv_fwd: out = x without in-edges"
    ldgp = 2 * f + (3 if f % 2 else 0)
    g_p, g_h = Buf(n, 2 * f, ld=ldgp), Buf(e, 2 * f)
    g_ea = Buf(e, d) if geattr else None
    g_par = Buf(d + 1, 2 * f) if grads else None
    ws = Buf(cdiv(_lib.query("hgb_cgconv_workspace_bytes", f, d), 4))
    go = fbuf(g_out)
    bwd = lambda: _lib.call("hgb_cgconv_bwd", go.ptr, B["pq"].ptr, I["rowptr"].ptr, ptr(I["perm"]), I["src"].ptr, ptr(B["ea"]), d,
                            ptr(B["mt"]), B["cvec"].ptr, n, e, f, g_p.ptr, ldgp, g_h.ptr, ptr(g_ea), ptr(g_par), ws.ptr, stream())
    assert launches(bwd) == plan["bwd_launches"]
    outs = [b for b in (g_p, g_h, g_ea, g_par) if b is not None]
    for b in outs:
        b.check("cgconv_bwd", "output")                   # a strided g_p keeps its gap columns, e = 0 included
    twice("cgconv_bwd", bwd, outs)
    if e == 0:
        assert not g_p.np().any() and (g_par is None or not g_par.np().any()), "cgconv_bwd: e = 0 must give zero gradients"
        return
    near("cgconv_bwd g_h", g_h.np(), rg["hz"], ag["hz"], d + 12, k)
    near("cgconv_bwd g_p", g_p.np(), rg["pq"][:, :2 * f], ag["pq"][:, :2 * f], L, k)
    if geattr:
        near("cgconv_bwd g_eattr", g_ea.np(), rg["ea"], ag["ea"], 2 * f + d + 12, k)
    if grads:
        par = torch.cat([rg["cvec"][None]] + ([rg["mt"]] if d else []))
        apar = torch.cat([ag["cvec"][None]] + ([ag["mt"]] if d else []))
        near("cgconv_bwd g_params", g_par.np(), par, apar, int(L.max()) * max(1, cdiv(n, 4224)) + 256, k)


# ---- GATv2 ------------------------------------------------------------------------------------------------------------------
SLOPE = 0.2
# (graph, heads, c, d, concat, aligned, grads, p, hot): hot scales att so that the scores reach about 80
GAT_SHAPES = [(1, 4, True), (2, 16, True), (4, 24, True), (4, 32, True), (1, 1, True), (2, 32, False), (1, 3, True),
              (8, 4, False), (2, 9, True), (8, 16, False), (4, 128, True), (8, 64, True), (1, 201, True), (1, 200, True),
              (8, 48, True)]
GAT_CASES = ([("small", h, c, d, concat, al, True, 0.0, False) for h, c, al in GAT_SHAPES for d, concat in ((0, True), (16, False))] +
             [("small", 4, 128, 16, True, True, False, 0.0, False), ("small", 8, 64, 16, False, True, True, 0.0, True),
              ("small", 4, 16, 3, True, True, True, 0.3, False), ("small", 8, 8, 2, False, True, True, 0.5, True),
              ("loops", 2, 8, 4, True, True, True, 0.0, False), ("sorted", 2, 12, 2, False, False, True, 0.0, False),
              ("big", 1, 32, 1, True, False, True, 0.0, False)])
GAT_REFUSED = [(1, 260), (4, 128), (2, 256)]                                      # heads c 257..512 with operands unaligned


def philox_keep(seed, slots, heads, p):
    """hgb_gat_dropout_keep restated: Philox4x32-10 of (edge id, head quad, 0x47415476) under the 64-bit seed; kept where the
    top 24 bits of the draw, as a fraction of 2^24, are >= p"""
    mask = np.uint64(0xFFFFFFFF)
    eid = np.arange(slots, dtype=np.uint64)
    words = []
    for q in range(cdiv(heads, 4)):
        x0, x1 = eid & mask, eid >> np.uint64(32)
        x2, x3 = np.full_like(eid, q), np.full_like(eid, 0x47415476)
        k0, k1 = np.uint64(seed & 0xFFFFFFFF), np.uint64((seed >> 32) & 0xFFFFFFFF)
        for _ in range(10):
            p0, p1 = x0 * np.uint64(0xD2511F53), x2 * np.uint64(0xCD9E8D57)
            x0, x1, x2, x3 = (p1 >> np.uint64(32)) ^ x1 ^ k0, p1 & mask, (p0 >> np.uint64(32)) ^ x3 ^ k1, p0 & mask
            k0, k1 = (k0 + np.uint64(0x9E3779B9)) & mask, (k1 + np.uint64(0xBB67AE85)) & mask
        words += [x0, x1, x2, x3]
    u = (np.stack(words[:heads], 1) >> np.uint64(8)).astype(np.float32) * np.float32(1.0 / 16777216.0)
    return (u >= np.float32(p)).astype(np.uint8)


def gat_inputs(n, e, heads, c, d, concat, hot, seed):
    g = torch.Generator().manual_seed(seed)
    hc = heads * c
    r = lambda *s: torch.randn(*s, generator=g, dtype=torch.float64)              # noqa: E731
    t = dict(xlr=r(n, 2 * hc), ea=r(e, d) if d else None, mt=r(d, hc) * 0.5 if d else None,
             att=r(hc) * (2.0 / math.sqrt(c)) * (30.0 if hot else 1.0), bias=r(hc if concat else c) * 0.1)
    return {k: (v.float().double() if v is not None else None) for k, v in t.items()}


@pytest.mark.gpu
@pytest.mark.parametrize("gname,heads,c,d,concat,aligned,grads,p,hot", GAT_CASES)
def test_gat(gname, heads, c, d, concat, aligned, grads, p, hot):
    src, dst, n = graph(gname)
    e = src.size
    hc = heads * c
    assert supported("hgb_gat_supported", heads, c, d)
    rowptr, perm, slot_src = csr_of(dst, src, n, gname == "sorted")
    rrowptr, rperm, rdst = csr_of(src, dst, n, False)
    t = gat_inputs(n, e, heads, c, d, concat, hot, heads * 31 + c + d)
    off = 0 if aligned else 1
    B = dict(xlr=fbuf(t["xlr"], off), ea=fbuf(t["ea"]) if d else None, mt=fbuf(t["mt"]) if d else None, att=fbuf(t["att"]),
             bias=fbuf(t["bias"]))
    I = dict(rowptr=ibuf(rowptr), perm=ibuf(perm), src=ibuf(slot_src), rrowptr=ibuf(rrowptr), rperm=ibuf(rperm), rdst=ibuf(rdst))
    seed = Buf(1, dtype=torch.int64, data=torch.tensor([0x1234_5678_9ABC + heads]))
    out, lse = Buf(n, hc if concat else c, off=off), Buf(n, heads)
    fwd = lambda: _lib.call("hgb_gat_fwd", B["xlr"].ptr, I["rowptr"].ptr, ptr(I["perm"]), I["src"].ptr, ptr(B["ea"]), d, ptr(B["mt"]),
                            B["att"].ptr, B["bias"].ptr, n, e, heads, c, int(concat), SLOPE, p, seed.ptr if p > 0 else None,
                            out.ptr, lse.ptr, stream())
    plan = gat_plan(n, heads, c, d, aligned, grads)
    assert launches(fwd) == plan["fwd_launches"]
    out.check("gat_fwd", "out")
    lse.check("gat_fwd", "lse")
    twice("gat_fwd", fwd, [out, lse])
    keep = None
    if p > 0:
        kb = torch.zeros(e + n, heads, dtype=torch.uint8, device="cuda")
        assert launches(lambda: _lib.call("hgb_gat_dropout_keep", n, e, heads, p, seed.ptr, kb.data_ptr(), stream())) == 1
        keep = kb.cpu()
        assert np.array_equal(keep.numpy(), philox_keep(int(seed.np()[0, 0]), e + n, heads, p)), "gat: dropout keep mask"
    ei = torch.from_numpy(np.stack([src, dst]))
    g_out = torch.randn(n, hc if concat else c, generator=torch.Generator().manual_seed(3), dtype=torch.float64).float().double()
    ref, rg = conv_reference.gat(t, ei, heads, c, concat, g_out, SLOPE, keep, p)
    aref, ag = conv_reference.gat(abs_inputs(t), ei, heads, c, concat, g_out.abs(), SLOPE, keep, p)
    k = K["gat"]
    deg = seg_len(dst, n)[:, None]
    inner = c + d + 16
    near("gat_fwd out", out.np(), ref, aref, deg + inner, k)
    go = fbuf(g_out, off)
    g_xlr = Buf(n, 2 * hc, off=off)
    g_ea = Buf(e, d) if d else None
    g_par = Buf(d + 1, hc) if grads else None
    ws = Buf(cdiv(_lib.query("hgb_gat_workspace_bytes", n, e, heads, c, d), 4))
    bwd = lambda: _lib.call("hgb_gat_bwd", go.ptr, B["xlr"].ptr, I["rowptr"].ptr, ptr(I["perm"]), I["src"].ptr, I["rrowptr"].ptr,
                            ptr(I["rperm"]), I["rdst"].ptr, ptr(B["ea"]), d, ptr(B["mt"]), B["att"].ptr, lse.ptr, n, e, heads, c,
                            int(concat), SLOPE, p, seed.ptr if p > 0 else None, g_xlr.ptr, ptr(g_ea), ptr(g_par), ws.ptr, stream())
    assert launches(bwd) == plan["bwd_launches"]
    outs = [b for b in (g_xlr, g_ea, g_par) if b is not None]
    for b in outs:
        b.check("gat_bwd", "output")
    twice("gat_bwd", bwd, outs)
    lmax = int(max(deg.max(), np.bincount(src, minlength=n).max())) + inner
    near("gat_bwd g_xlr", g_xlr.np(), rg["xlr"], ag["xlr"], lmax, k)
    if d:
        near("gat_bwd g_eattr", g_ea.np(), rg["ea"], ag["ea"], lmax, k)
    if grads:
        par = torch.cat([rg["att"][None]] + ([rg["mt"]] if d else []))
        apar = torch.cat([ag["att"][None]] + ([ag["mt"]] if d else []))
        near("gat_bwd g_params", g_par.np(), par, apar, lmax * max(1, cdiv(n, 4224)) + 256, k)


@pytest.mark.gpu
@pytest.mark.parametrize("heads,c", GAT_REFUSED)
def test_gat_refuses_wide_unaligned_rows_before_any_launch(heads, c):
    src, dst, n = graph("small")
    e, hc = src.size, heads * c
    assert supported("hgb_gat_supported", heads, c, 0) == (c % 4 == 0)
    rowptr, perm, slot_src = csr_of(dst, src, n, False)
    I = [ibuf(rowptr), ibuf(perm), ibuf(slot_src)]
    xlr, att, bias = Buf(n, 2 * hc, off=1, data=torch.zeros(n, 2 * hc)), Buf(hc, data=torch.zeros(hc)), Buf(hc, data=torch.zeros(hc))
    out, lse = Buf(n, hc, off=1), Buf(n, heads)
    before = _lib.launch_count()
    with pytest.raises(RuntimeError, match="gat_fwd"):
        _lib.call("hgb_gat_fwd", xlr.ptr, I[0].ptr, I[1].ptr, I[2].ptr, None, 0, None, att.ptr, bias.ptr, n, e, heads, c, 1, SLOPE, 0.0,
                  None, out.ptr, lse.ptr, stream())
    ws = Buf(max(cdiv(_lib.query("hgb_gat_workspace_bytes", n, e, heads, c, 0), 4), 1))
    with pytest.raises(RuntimeError, match="gat_bwd"):
        _lib.call("hgb_gat_bwd", out.ptr, xlr.ptr, I[0].ptr, I[1].ptr, I[2].ptr, I[0].ptr, I[1].ptr, I[2].ptr, None, 0, None, att.ptr,
                  lse.ptr, n, e, heads, c, 1, SLOPE, 0.0, None, xlr.ptr, None, None, ws.ptr, stream())
    assert _lib.launch_count() == before
    out.check("gat_fwd refused", "out", written=False)


# ---- CFConv -----------------------------------------------------------------------------------------------------------------
CUTOFF = 3.0
CF_NF = [1, 32, 33, 64, 65, 96, 97, 128]
# (graph, nf, g, d, w_e and g_we, g_dist, g_r, grads)
CF_CASES = ([("small", nf, g, d, True, True, d > 0, True) for nf in CF_NF for g, d in ((1, 0), (64, 16))] +
            [("small", 64, 64, 16, False, False, False, True), ("small", 33, 8, 2, True, True, True, False),
             ("small", 97, 16, 4, False, True, False, False), ("sorted", 128, 64, 16, True, True, True, True),
             ("big", 32, 8, 1, True, True, True, True)])


@pytest.mark.gpu
@pytest.mark.parametrize("gname,nf,g,d,we,gdist,gr,grads", CF_CASES)
def test_cfconv(gname, nf, g, d, we, gdist, gr, grads):
    src, dst, n = graph(gname)
    e = src.size
    assert supported("hgb_cfconv_supported", g, nf, d)
    rowptr, perm, _ = csr_of(dst, src, n, gname == "sorted")
    gen = torch.Generator().manual_seed(nf * 7 + g + d)
    mk = lambda *s: (torch.randn(*s, generator=gen, dtype=torch.float64) * 0.5).float().double()      # noqa: E731
    pos = (torch.rand(n, 3, generator=gen, dtype=torch.float64) * 6.0).float().double()  # many edges past the cutoff
    t = dict(xl=mk(n, nf), r=mk(e, d) if d else None, a1t=mk(g + d, nf), b1=mk(nf), w2=mk(nf, nf) / math.sqrt(nf), b2=mk(nf))
    mu = torch.linspace(0, CUTOFF, g, dtype=torch.float32).double()
    coeff = float(np.float32(-0.5 / (CUTOFF / max(g - 1, 1)) ** 2))
    B = {k: (fbuf(v) if v is not None else None) for k, v in t.items()}
    P = dict(pos=fbuf(pos), mu=fbuf(mu[:, None]), row=ibuf(src), col=ibuf(dst), rowptr=ibuf(rowptr), perm=ibuf(perm))
    out = Buf(n, nf)
    w_e = Buf(e, nf) if we else None
    fwd = lambda: _lib.call("hgb_cfconv_fwd", B["xl"].ptr, P["pos"].ptr, P["row"].ptr, P["rowptr"].ptr, ptr(P["perm"]), ptr(B["r"]), d,
                            P["mu"].ptr, coeff, CUTOFF, B["a1t"].ptr, B["b1"].ptr, B["w2"].ptr, B["b2"].ptr, n, e, g, nf, out.ptr,
                            ptr(w_e), stream())
    plan = cf_plan(n, e, g, nf, d, grads)
    assert launches(fwd) == plan["fwd_launches"]
    outs = [b for b in (out, w_e) if b is not None]
    for b in outs:
        b.check("cfconv_fwd", "output")
    twice("cfconv_fwd", fwd, outs)
    row, col = torch.from_numpy(src), torch.from_numpy(dst)
    dist = (pos[col] - pos[row]).norm(dim=1)
    leaves = {k: (v.clone().requires_grad_(True) if v is not None else None) for k, v in t.items()}
    dl = dist.clone().requires_grad_(True)
    ref, rw = conv_reference.cfconv_edges(leaves, dl, row, col, n, mu, coeff, CUTOFF)
    aref, aw = conv_reference.cfconv_edges(abs_inputs(t), dist, row, col, n, mu, coeff, CUTOFF)
    k = K["cfconv"]
    inner = nf + g + d + 16
    deg = seg_len(dst, n)[:, None]
    near("cfconv_fwd out", out.np(), ref, torch.zeros(n, nf, dtype=torch.float64).index_add(0, col, t["xl"].abs()[row] * aw.abs()),
         deg + inner, k)
    if we:
        near("cfconv_fwd w_e", w_e.np(), rw, aw, inner, k)
    g_out = mk(n, nf)
    g_we = mk(e, nf)
    go, gw = fbuf(g_out), fbuf(g_we) if we else None
    g_xle = Buf(e, nf)
    g_dist = Buf(e) if gdist else None
    g_r = Buf(e, d) if gr else None
    npar = (g + d) * nf + nf + nf * nf + nf
    g_par = Buf(npar) if grads else None
    ws = Buf(cdiv(_lib.query("hgb_cfconv_workspace_bytes", g, nf, d), 4))
    bwd = lambda: _lib.call("hgb_cfconv_bwd", go.ptr, ptr(gw), B["xl"].ptr, P["pos"].ptr, P["row"].ptr, P["col"].ptr, ptr(B["r"]), d,
                            P["mu"].ptr, coeff, CUTOFF, B["a1t"].ptr, B["b1"].ptr, B["w2"].ptr, B["b2"].ptr, n, e, g, nf, g_xle.ptr,
                            ptr(g_dist), ptr(g_r), ptr(g_par), ws.ptr, stream())
    assert launches(bwd) == plan["bwd_launches"]
    outs = [b for b in (g_xle, g_dist, g_r, g_par) if b is not None]
    for b in outs:
        b.check("cfconv_bwd", "output")
    twice("cfconv_bwd", bwd, outs)
    obj = (ref * g_out).sum() + ((rw * g_we).sum() if we else 0.0)
    names = ["a1t", "b1", "w2", "b2"] + (["r"] if d else [])
    grads_ = dict(zip(names + ["dist"], torch.autograd.grad(obj, [leaves[x] for x in names] + [dl])))
    near("cfconv_bwd g_xle", g_xle.np(), g_out[col] * rw.detach(), g_out.abs()[col] * aw.abs(), inner, k)
    # magnitudes for the rest: the same gradients of the restatement at |inputs|, |g_out|, |g_we|
    al = {kk: (v.abs().clone().requires_grad_(True) if v is not None else None) for kk, v in t.items()}
    ad = dist.clone().requires_grad_(True)
    aref2, aw2 = conv_reference.cfconv_edges(al, ad, row, col, n, mu, coeff, CUTOFF)
    aobj = (aref2 * g_out.abs()).sum() + ((aw2 * g_we.abs()).sum() if we else 0.0)
    agr = dict(zip(names + ["dist"], torch.autograd.grad(aobj, [al[x] for x in names] + [ad])))
    if gdist:
        near("cfconv_bwd g_dist", g_dist.np()[:, 0], grads_["dist"], agr["dist"], inner * 2, k)
    if gr:
        near("cfconv_bwd g_r", g_r.np(), grads_["r"], agr["r"], inner, k)
    if grads:
        par = torch.cat([grads_[x].reshape(-1) for x in ("a1t", "b1", "w2", "b2")])
        apar = torch.cat([agr[x].reshape(-1) for x in ("a1t", "b1", "w2", "b2")])
        near("cfconv_bwd g_params", g_par.np()[:, 0], par, apar, cdiv(e, 132) + 8 + inner, k)
