"""Kernel-level tests of the graph plumbing every stack runs through: csrc/hgb_core.cu (prefix scan, CSR builds, int32 gather,
collate), the generic half of csrc/hgb_seg.cu (row gather, segment sum, segment arg-min/max, PNA aggregation, graph pooling),
csrc/hgb_optim.cu (loss, AdamW) and the helpers and periodic image pruning of csrc/hgb_radius.cu.  Each is checked against a
plain restatement of include/hgb.h computed on the CPU.

The C-ABI is called directly, so the test controls every pointer offset, stride, workspace and NULL argument.  Every operand is
the leading block of a buffer filled with NaN (floating point) or SENTINEL (integers), followed by GUARD rows of the same fill.
After each call every element in range must be written (finite, or not the sentinel) and every other element must keep its
fill bits: that catches unwritten elements and stores past the end of a row block, a column block or a buffer.

Exactness:
* Integer outputs (scan, CSR, arg-min/max, collate, edge lists) must match exactly.
* Gather, segment sum and pooling add in a fixed order: segment sum adds a segment in CSR order (its two loads in flight are
  still added one after the other), pooling adds a graph's rows in row order, and mean pooling divides once, its backward
  multiplying by 1.f / cnt.  So their results must equal, bit for bit, an fp32 sequential restatement (`seq_sum_f32`, never
  np.sum, which sums pairwise).  They are also held to fp64 within gamma(L) sum |m| (Higham, Accuracy and Stability of
  Numerical Algorithms, 2nd ed., eq. 3.5), L the segment length, u = 2^-24, gamma(L) = L u / (1 - L u).
* PNA aggregation: arg-min / arg-max exact (first extremum in CSR order), mean within gamma(L + 1) sum|m| / L.  The standard
  deviation sqrt(max(E[x^2] - E[x]^2, eps)) cancels: its variance is held to (gamma(L + 2) + 2 gamma(L + 1) + 3u) E[x^2], a
  bound relative to E[x^2], not to the result.  Random entries whose fp64 variance lies within that bound of eps = 1e-5f are
  left out of the masked / unmasked decision; dyadic known-answer segments pin both sides of the threshold exactly.
* Loss: per-thread sequential sums of ceil(count / 1024) terms, a 10-level tree and one scaling, plus gamma(3) per squared term.
* AdamW: each step is compared with an fp64 restatement that starts from the kernel's own fp32 state and uses the fp32-rounded
  hyper-parameters the ABI receives.  The error of the update p_new - p_old is bounded (not the error of p), with powf held
  to 4 ulp and rsqrtf to 2 ulp (CUDA C Programming Guide, Mathematical Functions).
Every case runs twice and must return the same bits: none of these kernels adds values with atomics.

`group_lanes`, `vec4_ok`, `row_plan`, `grid_for` and `scan_nb` restate the host dispatch; `test_cases_reach_every_specialisation`
(no GPU) asserts that the case lists reach every specialisation, grid-stride loop and scan-chunk path, and the GPU tests check
the number of launches each plan predicts.
"""
import math

import numpy as np
import pytest
import torch

from hydragnn_b200 import _lib, ops, radius
from kernel_harness import (DEV, NAN_BITS, SENTINEL, U, Buf, cdiv, check_bound, gamma, grid_for, launches, same_f32,
                            stream, twice, ws_buf)
from oracle.radius_graph import _neighbor_list_ijS, _shift_vectors, limit_neighbors

SCAN_B = 1024
PNA_EPS = float(np.float32(1e-5))
GUARD_BAD_INDEX = ops.GUARD_BAD_INDEX
GUARD_EDGE_COUNT = ops.GUARD_EDGE_COUNT
POOL = dict(add=0, mean=1, max=2)


# ---- the host dispatch, restated ---------------------------------------------------------------------------------------------
def group_lanes(cv):
    lanes = 1
    while lanes < cv and lanes < 32:
        lanes <<= 1
    return lanes


def vec4_ok(c, ldo, in_aligned, out_aligned):
    """gather_rows / segment_sum take float4 rows when c, ldo and both pointers allow it"""
    return c % 4 == 0 and ldo % 4 == 0 and in_aligned and out_aligned


def row_plan(kind, rows, c, ldo=None, in_aligned=True, out_aligned=True):
    """one row kernel (gather / segsum / argminmax / pna): its VEC form, lanes per row, grid and grid-stride iterations"""
    vec = 4 if kind in ("gather", "segsum") and vec4_ok(c, c if ldo is None else ldo, in_aligned, out_aligned) else 1
    cv = c // vec
    lanes = group_lanes(cv)
    rpb = 256 // lanes
    grid = grid_for(rows, rpb)
    iters = cdiv(rows, grid * rpb) if rows else 0
    tags = {"%s:vec%d" % (kind, vec), "%s:lanes%d" % (kind, lanes)}
    if cv > lanes:
        tags.add("%s:second_pass" % kind)
    if iters > 1:
        tags.add("%s:grid_stride" % kind)
    return dict(vec=vec, lanes=lanes, grid=grid, iters=iters, launches=int(rows > 0), tags=tags)


def flat_plan(kind, work, per_block=256):
    """grid-stride kernels over `work` items (pool: one warp per graph, 8 per block)"""
    grid = grid_for(work, per_block)
    iters = cdiv(work, grid * per_block) if work else 0
    return {"%s:grid_stride" % kind} if iters > 1 else set()


def scan_nb(n):
    return cdiv(n, SCAN_B)


def scan_plan(n):
    nb = scan_nb(n)
    tags = set()
    if nb > SCAN_B:
        tags.add("scan:multi_chunk")
        if nb % SCAN_B == 0:
            tags.add("scan:multi_chunk_exact")
    return dict(launches=3 if n > 0 else 0, tags=tags)


def csr_key_bits(n):
    bits = 1
    while bits < 31 and (1 << bits) < n:
        bits += 1
    return bits


def csr_plan(e, n):
    return (e > 0) + scan_plan(n)["launches"] + (e > 0)


def grouped_plan(e, n, g):
    return (e > 0) + scan_plan(n)["launches"] + (e > 0 and g > 0)


# ---- case lists -----------------------------------------------------------------------------------------------------------------
# gather: (rows, c, x_off, out_off); an offset of one float makes the pointer 16-byte misaligned
GATHER_C = [1, 2, 3, 4, 5, 8, 9, 12, 16, 17, 31, 32, 33, 64, 100, 128, 132, 200, 256, 260]
GATHER_CASES = ([(777, c, 0, 0) for c in GATHER_C] + [(501, 64, 1, 0), (501, 64, 0, 1), (300, 132, 1, 0)] +
                [(600_000, 1, 0, 0), (560_000, 4, 0, 0), (17_000, 128, 0, 0), (17_000, 132, 1, 0)])

# segment sum: (name, n, c, lens kind, perm, ldo, col_off, m_off)
SEG_CASES = [("c%d" % c, 400, c, "short", True, c, 0, 0) for c in GATHER_C] + [
    ("long_segments", 50, 64, "long", True, 64, 0, 0),
    ("long_no_perm", 50, 33, "long", False, 33, 0, 0),
    ("no_perm", 300, 16, "short", False, 16, 0, 0),
    ("ldo_wider_aligned_block", 300, 64, "short", True, 100, 4, 0),
    ("ldo_wider_misaligned_block", 300, 64, "short", True, 100, 3, 0),
    ("ldo_odd", 300, 12, "short", True, 13, 0, 0),
    ("m_misaligned", 300, 128, "short", True, 128, 0, 1),
    ("payload_E_3_F", 200, 3 * 16, "short", True, 3 * 16, 0, 0),
    ("payload_E_3_F_odd", 200, 3 * 7, "short", True, 3 * 7, 0, 0),
    ("grid_stride_lanes1", 600_000, 1, "short", True, 1, 0, 0),
    ("grid_stride_vec4_lanes1", 560_000, 4, "short", False, 4, 0, 0),
    ("grid_stride_lanes32", 17_000, 132, "short", True, 132, 0, 0),
]

# arg-min/max and PNA aggregation: (n, c, lens kind, perm)
ARG_C = [1, 2, 3, 4, 5, 9, 16, 17, 32, 33, 40, 64]
ARG_CASES = [(300, c, "short", True) for c in ARG_C] + [(40, 8, "long", True), (40, 3, "long", False),
                                                        (560_000, 1, "short", True), (17_000, 40, "short", False)]
PNA_CASES = [(300, c, "short", True) for c in ARG_C] + [(40, 8, "long", True), (40, 5, "long", False),
                                                        (560_000, 1, "short", True), (17_000, 33, "short", False)]

POOL_C = [1, 31, 32, 33, 200]
POOL_CASES = [(g, c) for c in POOL_C for g in (7, 60)] + [(17_000, 1), (17_000, 33)]

SCAN_N = [0, 1, 1023, 1024, 1025, 2 ** 20, 2 ** 20 + 1, 2 ** 21, 3 * 2 ** 20 + 5]
CSR_CASES = [(0, 4), (5, 1), (40, 2), (1000, 37), (1000, 64), (1000, 65), (3000, 1024), (3000, 1025), (200_000, 5000),
             (4000, 1)]                                           # (e, n); the last: one segment holds every edge
GROUPED_GRAPHS = ["wide", "shared_key_step", "no_edges", "no_nodes", "mixed"]
ADAMW_COUNTS = [1, 1000, 600_000, 2_200_001]
LOSS_COUNTS = [1, 7, 1024, 1025, 70_000]


def all_tags():
    tags = set()
    for rows, c, xo, oo in GATHER_CASES:
        tags |= row_plan("gather", rows, c, in_aligned=xo % 4 == 0, out_aligned=oo % 4 == 0)["tags"]
    for _, n, c, _, _, ldo, col, mo in SEG_CASES:
        tags |= row_plan("segsum", n, c, ldo, in_aligned=mo % 4 == 0, out_aligned=col % 4 == 0)["tags"]
    for n, c, _, _ in ARG_CASES:
        tags |= row_plan("argminmax", n, c)["tags"]
    for n, c, _, _ in PNA_CASES:
        tags |= row_plan("pna", n, c)["tags"]
        tags |= flat_plan("pna_bwd", n * c * 3 // 2)            # e = 1.5 n on average for "short" segments
    for g, c in POOL_CASES:
        tags |= flat_plan("pool", g, 8)
    for n in SCAN_N:
        tags |= scan_plan(n)["tags"]
    for count in ADAMW_COUNTS:
        tags |= flat_plan("adamw", cdiv(count, 4))           # aligned buffers: the float4 body, the remainder one by one
    for _, n in CSR_CASES:
        bits = csr_key_bits(n)
        if n in (1, 2):
            tags.add("key_bits:n=%d" % n)
        elif n >= 4 and n & (n - 1) == 0:
            tags.add("key_bits:pow2")
        elif n >= 5 and (n - 1) & (n - 2) == 0:
            tags.add("key_bits:pow2+1")
        assert (1 << bits) >= n
    for name in GROUPED_GRAPHS:
        tags.add("grouped:" + name)
    return tags


def test_cases_reach_every_specialisation():
    tags = all_tags()
    need = set()
    for kind in ("gather", "segsum"):
        need |= {"%s:vec4" % kind, "%s:vec1" % kind}
    for kind in ("gather", "segsum", "argminmax", "pna"):
        need |= {"%s:lanes%d" % (kind, 1 << k) for k in range(6)}
        need |= {"%s:second_pass" % kind, "%s:grid_stride" % kind}
    need |= {"pool:grid_stride", "pna_bwd:grid_stride", "adamw:grid_stride", "scan:multi_chunk", "scan:multi_chunk_exact"}
    need |= {"key_bits:n=1", "key_bits:n=2", "key_bits:pow2", "key_bits:pow2+1"}
    need |= {"grouped:wide", "grouped:shared_key_step", "grouped:no_edges"}
    missing = need - tags
    assert not missing, "case lists miss %s" % sorted(missing)
    # the restated dispatch at its edges
    assert row_plan("gather", 540_672, 1)["iters"] == 1 and row_plan("gather", 540_673, 1)["iters"] == 2
    assert row_plan("gather", 10, 132)["lanes"] == 32 and row_plan("gather", 10, 132)["vec"] == 4
    assert row_plan("segsum", 10, 64, 100, out_aligned=False)["vec"] == 1
    assert scan_nb(2 ** 20) == 1024 and scan_nb(2 ** 20 + 1) == 1025 and scan_nb(2 ** 21) == 2048
    assert [csr_key_bits(n) for n in (1, 2, 3, 4, 5, 1024, 1025)] == [1, 1, 2, 2, 3, 10, 11]
    assert flat_plan("pool", 16_896, 8) == set() and flat_plan("pool", 16_897, 8) == {"pool:grid_stride"}


# ---- CSR helpers (host) ---------------------------------------------------------------------------------------------------------
def segment_lengths(rng, n, kind):
    """"short": lengths 0..3 (empty, 1, 2 and 3 all present); "long": short ones plus segments of 1000 and 1501"""
    lens = rng.integers(0, 4, n)
    lens[:4] = [0, 1, 2, 3]
    if kind == "long":
        lens[n // 2] = 1000
        lens[-1] = 1501
    return lens


def make_csr(rng, lens, shuffle):
    """(rowptr, perm or None, target of every edge): with shuffle the edges are in random order, else in CSR order"""
    n = len(lens)
    rowptr = np.concatenate([[0], np.cumsum(lens)]).astype(np.int32)
    tgt = np.repeat(np.arange(n), lens)
    if not shuffle:
        return rowptr, None, tgt.astype(np.int32)
    tgt = tgt[rng.permutation(tgt.size)]
    perm = np.argsort(tgt, kind="stable").astype(np.int32)
    return rowptr, perm, tgt.astype(np.int32)


def csr_edges(rowptr, perm, p):
    """edge ids at CSR position p of every segment longer than p: (rows, edges)"""
    lens = np.diff(rowptr)
    rows = np.nonzero(lens > p)[0]
    pos = rowptr[rows] + p
    return rows, (perm[pos] if perm is not None else pos)


def seq_sum_f32(m, rowptr, perm):
    """fp32 sum of every segment, adding its edges one after the other in CSR order (the kernel's order)"""
    n = len(rowptr) - 1
    acc = np.zeros((n,) + m.shape[1:], np.float32)
    for p in range(int(np.diff(rowptr).max(initial=0))):
        rows, e = csr_edges(rowptr, perm, p)
        acc[rows] = acc[rows] + m[e]
    return acc


def seg_sum64(m, tgt, n):
    out = np.zeros((n,) + m.shape[1:], np.float64)
    np.add.at(out, tgt, m.astype(np.float64))
    return out


def first_extrema(m, rowptr, perm):
    """edge id of the first minimum / maximum of every (segment, channel) in CSR order, -1 for an empty segment"""
    n, c = len(rowptr) - 1, m.shape[1]
    amin, amax = np.full((n, c), -1, np.int64), np.full((n, c), -1, np.int64)
    vmin, vmax = np.zeros((n, c), np.float32), np.zeros((n, c), np.float32)
    for p in range(int(np.diff(rowptr).max(initial=0))):
        rows, e = csr_edges(rowptr, perm, p)
        v = m[e]
        for arg, val, better in ((amin, vmin, v < vmin[rows]), (amax, vmax, v > vmax[rows])):
            upd = (arg[rows] < 0) | better
            arg[rows] = np.where(upd, e[:, None], arg[rows])
            val[rows] = np.where(upd, v, val[rows])
    return amin, amax


def upload_csr(rowptr, perm):
    rp = Buf(len(rowptr), dtype=torch.int32, data=torch.from_numpy(rowptr))
    pm = Buf(len(perm), dtype=torch.int32, data=torch.from_numpy(perm)) if perm is not None else None
    return rp, pm


# ---- 2. scan, CSR, collate (hgb_core.cu) -------------------------------------------------------------------------------------------
@pytest.mark.gpu
@pytest.mark.parametrize("n", SCAN_N)
def test_exclusive_scan(n):
    rng = np.random.default_rng(n)
    x = rng.integers(0, 600, n).astype(np.int32)
    if n:
        x[-1] = 599
    inp = Buf(n, dtype=torch.int32, data=torch.from_numpy(x))
    out = Buf(n + 1, dtype=torch.int32)
    nbytes = _lib.query("hgb_exclusive_scan_workspace_bytes", n)
    assert nbytes == 4 * (scan_nb(n) + 2)
    ws = ws_buf(nbytes)
    call = lambda: _lib.call("hgb_exclusive_scan_i32", inp.ptr, out.ptr, n, ws.ptr, stream())
    assert launches(call) == scan_plan(n)["launches"]
    out.check("scan", "out")
    inp.check("scan", "in")
    ws.check("scan", "workspace", written=False)
    ref = np.concatenate([[0], np.cumsum(x.astype(np.int64))])
    assert np.array_equal(out.np()[:, 0], ref), "scan: wrong prefix sums"
    twice("scan", call, [out])


def run_csr_build(what, idx, n, guard=True):
    e = len(idx)
    ib = Buf(e, dtype=torch.int64, data=torch.from_numpy(idx))
    idx32, rowptr, perm = Buf(e, dtype=torch.int32), Buf(n + 1, dtype=torch.int32), Buf(e, dtype=torch.int32)
    flag = Buf(1, dtype=torch.int32, data=torch.zeros(1, dtype=torch.int32)) if guard else None
    ws = ws_buf(_lib.query("hgb_csr_workspace_bytes", e, n))

    def call():
        if flag is not None:
            flag.view.zero_()
        _lib.call("hgb_csr_build", ib.ptr, e, n, idx32.ptr, rowptr.ptr, perm.ptr, flag.ptr if flag else None, ws.ptr, stream())

    assert launches(call) == csr_plan(e, n)
    for b, name in ((idx32, "idx32"), (rowptr, "rowptr"), (perm, "perm"), (ib, "idx")):
        b.check(what, name)
    ws.check(what, "workspace", written=False)
    twice(what, call, [idx32, rowptr, perm])
    return idx32.np()[:, 0], rowptr.np()[:, 0], perm.np()[:, 0], (int(flag.np()[0, 0]) if flag else None)


def csr_reference(idx, n):
    key = torch.from_numpy(np.where((idx >= 0) & (idx < n), idx, 0))
    perm = torch.sort(key, stable=True).indices.numpy()
    rowptr = np.concatenate([[0], np.cumsum(np.bincount(key.numpy(), minlength=n))])
    return key.numpy(), rowptr, perm


@pytest.mark.gpu
@pytest.mark.parametrize("e,n", CSR_CASES)
def test_csr_build_matches_stable_sort(e, n):
    rng = np.random.default_rng(e + 7 * n)
    idx = rng.integers(0, n, e)
    if n > 3 and e > 100:
        idx[: e // 4] = n - 1                      # a long segment, and empty ones between
        idx[idx == 1] = 2
    idx32, rowptr, perm, flag = run_csr_build("csr[e=%d,n=%d]" % (e, n), idx, n)
    k, rp, pm = csr_reference(idx, n)
    assert flag == 0
    assert np.array_equal(idx32, k) and np.array_equal(rowptr, rp) and np.array_equal(perm, pm)


@pytest.mark.gpu
def test_csr_build_index_outside_range_sets_guard():
    rng = np.random.default_rng(3)
    n, e = 50, 2000
    idx = rng.integers(0, n, e)
    idx[[5, 77, 1999]] = [-1, n, 2 ** 40]
    idx32, rowptr, perm, flag = run_csr_build("csr_bad_index", idx, n)
    k, rp, pm = csr_reference(idx, n)
    assert flag == GUARD_BAD_INDEX
    assert np.array_equal(idx32, k) and np.array_equal(rowptr, rp) and np.array_equal(perm, pm)
    # without a guard buffer the flag goes to the workspace: the result is the same
    i2, r2, p2, _ = run_csr_build("csr_bad_index_noflag", idx, n, guard=False)
    assert np.array_equal(i2, idx32) and np.array_equal(r2, rowptr) and np.array_equal(p2, perm)


def grouped_input(rng, name):
    """radius-graph-shaped edges: (node_ptr, edge_ptr, idx).  Graph k's edges are contiguous and sorted by target, and idx (their
    sources) names only nodes of graph k.
    wide: one graph of well over 32 edges; shared_key_step: a target whose 32 in-edges all come from one source, so a whole
    32-lane step shares one key, then targets of 20 in-edges from 3 sources; no_edges: a graph with nodes and no edges;
    no_nodes: graphs without nodes, leading, interior and trailing; mixed: 300 graphs of 0..29 nodes."""
    sizes = dict(wide=[40], shared_key_step=[3, 40], no_edges=[5, 6, 7], no_nodes=[0, 4, 0, 0, 9, 0]).get(name)
    if sizes is None:
        sizes = list(rng.integers(0, 30, 300))
    node_ptr = np.concatenate([[0], np.cumsum(sizes)]).astype(np.int32)
    degs, src = [], []
    for k, s in enumerate(sizes):
        lo = int(node_ptr[k])
        for t in range(s):
            if name == "shared_key_step" and k == 1:
                d, nbr = (32, np.full(32, lo + 5)) if t == 0 else (20, lo + np.arange(20) % 3)
            else:
                d = 0 if name == "no_edges" and k == 1 else int(rng.integers(0, 12 if name == "mixed" else 6))
                nbr = rng.integers(lo, lo + s, d)
            degs.append(d)
            src.append(nbr)
    edge_ptr = np.concatenate([[0], np.cumsum(degs)]).astype(np.int32)
    idx = np.concatenate(src + [np.zeros(0, np.int64)]).astype(np.int64)
    return node_ptr, edge_ptr, idx


@pytest.mark.gpu
@pytest.mark.parametrize("name", GROUPED_GRAPHS)
def test_csr_build_grouped_equals_csr_build(name):
    rng = np.random.default_rng(len(name))
    node_ptr, edge_ptr, idx = grouped_input(rng, name)
    n, g, e = int(node_ptr[-1]), len(node_ptr) - 1, len(idx)
    assert int(edge_ptr[-1]) == e
    npb = Buf(g + 1, dtype=torch.int32, data=torch.from_numpy(node_ptr))
    epb = Buf(n + 1, dtype=torch.int32, data=torch.from_numpy(edge_ptr))
    ib = Buf(e, dtype=torch.int64, data=torch.from_numpy(idx))
    idx32, rowptr, perm = Buf(e, dtype=torch.int32), Buf(n + 1, dtype=torch.int32), Buf(e, dtype=torch.int32)
    flag = Buf(1, dtype=torch.int32, data=torch.zeros(1, dtype=torch.int32))
    ws = ws_buf(_lib.query("hgb_csr_grouped_workspace_bytes", e, n))
    call = lambda: _lib.call("hgb_csr_build_grouped", ib.ptr, e, n, npb.ptr, epb.ptr, g, idx32.ptr, rowptr.ptr, perm.ptr,
                             flag.ptr, ws.ptr, stream())
    assert launches(call) == grouped_plan(e, n, g)
    for b, nm in ((idx32, "idx32"), (rowptr, "rowptr"), (perm, "perm")):
        b.check("grouped[%s]" % name, nm)
    ws.check("grouped[%s]" % name, "workspace", written=False)
    twice("grouped[%s]" % name, call, [idx32, rowptr, perm])
    i2, r2, p2, f2 = run_csr_build("grouped_ref[%s]" % name, idx, n)
    assert int(flag.np()[0, 0]) == 0 and f2 == 0
    assert np.array_equal(idx32.np()[:, 0], i2) and np.array_equal(rowptr.np()[:, 0], r2) and np.array_equal(perm.np()[:, 0], p2)


@pytest.mark.gpu
def test_gather_i32():
    rng = np.random.default_rng(5)
    for e in (1, 1000, 600_000):
        idx = rng.integers(0, 2 ** 30, e).astype(np.int32)
        perm = rng.permutation(e).astype(np.int32)
        ib, pb = Buf(e, dtype=torch.int32, data=torch.from_numpy(idx)), Buf(e, dtype=torch.int32, data=torch.from_numpy(perm))
        out = Buf(e, dtype=torch.int32)
        call = lambda: _lib.call("hgb_gather_i32", ib.ptr, pb.ptr, e, out.ptr, stream())
        assert launches(call) == 1
        out.check("gather_i32", "out")
        assert np.array_equal(out.np()[:, 0], idx[perm])
        twice("gather_i32", call, [out])
    assert launches(lambda: _lib.call("hgb_gather_i32", None, None, 0, None, stream())) == 0


def collate_sizes(rng, g):
    nodes = rng.integers(0, 6, g)
    nodes[0], nodes[g // 2], nodes[-1] = 0, 0, 0                      # leading, interior and trailing graphs without nodes
    edges = np.where(nodes > 0, rng.integers(0, 9, g), 0)
    edges[1] = 0 if g > 2 else edges[1]                              # a graph with nodes and no edges
    return nodes, edges


@pytest.mark.gpu
@pytest.mark.parametrize("g", [3, 9, 3000])
def test_collate(g):
    rng = np.random.default_rng(g)
    nodes, edges = collate_sizes(rng, g)
    nptr = np.concatenate([[0], np.cumsum(nodes)]).astype(np.int32)
    eptr = np.concatenate([[0], np.cumsum(edges)]).astype(np.int32)
    n, e = int(nptr[-1]), int(eptr[-1])
    local = np.concatenate([rng.integers(0, max(k, 1), (2, m)) for k, m in zip(nodes, edges)] + [np.zeros((2, 0), np.int64)], 1)
    npb = Buf(g + 1, dtype=torch.int32, data=torch.from_numpy(nptr))
    epb = Buf(g + 1, dtype=torch.int32, data=torch.from_numpy(eptr))
    batch = Buf(n, dtype=torch.int64)
    lb = Buf(2 * e, dtype=torch.int64, data=torch.from_numpy(local.reshape(-1)))
    out = Buf(2 * e, dtype=torch.int64)
    cb = lambda: _lib.call("hgb_collate_batch_vector", npb.ptr, g, n, batch.ptr, stream())
    ce = lambda: _lib.call("hgb_collate_offset_edges", lb.ptr, epb.ptr, npb.ptr, g, e, out.ptr, stream())
    assert launches(cb) == int(n > 0) and launches(ce) == int(e > 0)
    batch.check("collate", "batch")
    out.check("collate", "edge_index")
    assert np.array_equal(batch.np()[:, 0], np.repeat(np.arange(g), nodes))
    off = np.repeat(nptr[:-1], edges)
    assert np.array_equal(out.np()[:, 0].reshape(2, e), local + off[None])
    twice("collate", lambda: (cb(), ce()), [batch, out])


# ---- 3. gather, segment sum, arg-min/max, PNA aggregation, pooling (hgb_seg.cu) ---------------------------------------------------
@pytest.mark.gpu
@pytest.mark.parametrize("rows,c,x_off,out_off", GATHER_CASES)
def test_gather_rows(rows, c, x_off, out_off):
    rng = np.random.default_rng(rows + c)
    nx = 1000
    x = Buf(nx, c, off=x_off, data=torch.from_numpy(rng.standard_normal((nx, c)).astype(np.float32)))
    idx = rng.integers(0, nx, rows).astype(np.int32)
    ib = Buf(rows, dtype=torch.int32, data=torch.from_numpy(idx))
    out = Buf(rows, c, off=out_off)
    plan = row_plan("gather", rows, c, in_aligned=x.ptr % 16 == 0, out_aligned=out.ptr % 16 == 0)
    call = lambda: _lib.call("hgb_gather_rows", x.ptr, ib.ptr, rows, c, out.ptr, stream())
    assert launches(call) == plan["launches"]
    out.check("gather", "out")
    x.check("gather", "x")
    same_f32("gather[%s]" % sorted(plan["tags"]), out.np(), x.np()[idx])
    twice("gather", call, [out])


def run_segment_sum(what, n, c, kind, use_perm, ldo, col_off, m_off, seed, payload3=False):
    rng = np.random.default_rng(seed)
    lens = segment_lengths(rng, n, kind)
    rowptr, perm, tgt = make_csr(rng, lens, use_perm)
    e = len(tgt)
    m = (rng.standard_normal((e, c)) * np.exp(rng.uniform(-3, 3, (e, 1)))).astype(np.float32)
    mb = Buf(e, c, off=m_off, data=torch.from_numpy(m))
    rp, pm = upload_csr(rowptr, perm)
    out = Buf(n, ldo, off=0)                 # the whole [n, ldo] matrix: the kernel writes columns [col_off, col_off + c)
    blk = out.ptr + 4 * col_off
    plan = row_plan("segsum", n, c, ldo, in_aligned=mb.ptr % 16 == 0, out_aligned=blk % 16 == 0)
    call = lambda: _lib.call("hgb_segment_sum_strided", mb.ptr, rp.ptr, pm.ptr if pm else None, n, c, blk, ldo, stream())
    assert launches(call) == plan["launches"]
    written = torch.zeros(n, ldo, dtype=torch.bool)
    written[:, col_off:col_off + c] = True
    got_all = out.view.cpu()
    assert bool(torch.isfinite(got_all[written]).all()), "%s: unwritten entries" % what
    assert bool((got_all[~written].view(torch.int32) == NAN_BITS).all()), "%s: columns outside the block were written" % what
    out.check(what, "out", written=False)
    mb.check(what, "m")
    got = got_all[:, col_off:col_off + c].numpy()
    same_f32(what + str(sorted(plan["tags"])), got, seq_sum_f32(m, rowptr, perm))
    ref = seg_sum64(m, tgt, n)
    mag = seg_sum64(np.abs(m), tgt, n)
    check_bound(what, got, ref, gamma(np.maximum(lens, 1))[:, None] * mag)
    twice(what, call, [out])
    return plan


@pytest.mark.gpu
@pytest.mark.parametrize("name,n,c,kind,use_perm,ldo,col_off,m_off", SEG_CASES)
def test_segment_sum(name, n, c, kind, use_perm, ldo, col_off, m_off):
    run_segment_sum("segment_sum[%s]" % name, n, c, kind, use_perm, ldo, col_off, m_off, seed=n + c + ldo)


@pytest.mark.gpu
def test_segment_sum_unstrided_entry_is_the_strided_one():
    rng = np.random.default_rng(11)
    rowptr, perm, tgt = make_csr(rng, segment_lengths(rng, 300, "short"), True)
    m = rng.standard_normal((len(tgt), 20)).astype(np.float32)
    mb = Buf(len(tgt), 20, data=torch.from_numpy(m))
    rp, pm = upload_csr(rowptr, perm)
    out = Buf(300, 20)
    _lib.call("hgb_segment_sum", mb.ptr, rp.ptr, pm.ptr, 300, 20, out.ptr, stream())
    out.check("segment_sum", "out")
    same_f32("segment_sum", out.np(), seq_sum_f32(m, rowptr, perm))


def special_values(rng, e, c):
    """ties, +-0.0, all-equal segments: values from a small set"""
    return rng.choice(np.array([-1.0, -0.0, 0.0, 0.5, 1.0, 2.0], np.float32), (e, c))


@pytest.mark.gpu
@pytest.mark.parametrize("n,c,kind,use_perm", ARG_CASES)
@pytest.mark.parametrize("values", ["random", "ties"])
def test_segment_argminmax(n, c, kind, use_perm, values):
    rng = np.random.default_rng(n * 3 + c)
    lens = segment_lengths(rng, n, kind)
    rowptr, perm, tgt = make_csr(rng, lens, use_perm)
    e = len(tgt)
    m = rng.standard_normal((e, c)).astype(np.float32) if values == "random" else special_values(rng, e, c)
    if values == "ties" and n > 10:
        seg = np.nonzero(lens >= 3)[0][0]                       # an all-equal segment
        m[perm[rowptr[seg]:rowptr[seg + 1]] if perm is not None else slice(rowptr[seg], rowptr[seg + 1])] = 0.5
    mb = Buf(e, c, data=torch.from_numpy(m))
    rp, pm = upload_csr(rowptr, perm)
    amin, amax = Buf(n, c, dtype=torch.int64), Buf(n, c, dtype=torch.int64)
    plan = row_plan("argminmax", n, c)
    call = lambda: _lib.call("hgb_segment_argminmax", mb.ptr, rp.ptr, pm.ptr if pm else None, n, c, amin.ptr, amax.ptr, stream())
    assert launches(call) == plan["launches"]
    amin.check("argminmax", "argmin")
    amax.check("argminmax", "argmax")
    rmin, rmax = first_extrema(m, rowptr, perm)
    assert np.array_equal(amin.np(), rmin), "argmin differs in %d entries" % int((amin.np() != rmin).sum())
    assert np.array_equal(amax.np(), rmax), "argmax differs in %d entries" % int((amax.np() != rmax).sum())
    assert (rmin[lens == 0] == -1).all()
    twice("argminmax", call, [amin, amax])


def pna_var_bound(L, sq_mean):
    """|var_fp32 - var| <= (gamma(L + 2) + 2 gamma(L + 1) + 3u) E[x^2]"""
    return (gamma(L + 2) + 2 * gamma(L + 1) + 3 * U) * sq_mean


def run_pna(what, m, rowptr, perm, tgt):
    n, (e, c) = len(rowptr) - 1, m.shape
    mb = Buf(e, c, data=torch.from_numpy(m))
    rp, pm = upload_csr(rowptr, perm)
    out = Buf(n, 4 * c)
    amin, amax = Buf(n, c, dtype=torch.int32), Buf(n, c, dtype=torch.int32)
    plan = row_plan("pna", n, c)
    call = lambda: _lib.call("hgb_pna_aggregate_fwd", mb.ptr, rp.ptr, pm.ptr if pm else None, n, c, out.ptr, amin.ptr, amax.ptr,
                             stream())
    assert launches(call) == plan["launches"]
    for b, name in ((out, "out"), (amin, "argmin"), (amax, "argmax")):
        b.check(what, name)
    twice(what, call, [out, amin, amax])
    return mb, rp, out, amin, amax


@pytest.mark.gpu
@pytest.mark.parametrize("n,c,kind,use_perm", PNA_CASES)
def test_pna_aggregate(n, c, kind, use_perm):
    what = "pna[n=%d,c=%d,%s]" % (n, c, kind)
    rng = np.random.default_rng(n + 5 * c)
    lens = segment_lengths(rng, n, kind)
    rowptr, perm, tgt = make_csr(rng, lens, use_perm)
    e = len(tgt)
    # per-edge scale and per-segment offset: variances on both sides of eps, and cancellation in E[x^2] - E[x]^2
    m = (rng.standard_normal((e, c)) * np.exp(rng.uniform(-5, 0, (e, 1))) + rng.uniform(-2, 2, (n, 1))[tgt]).astype(np.float32)
    mb, rp, out, amin, amax = run_pna(what, m, rowptr, perm, tgt)
    o = out.np()
    mean, vmin, vmax, sd = o[:, :c], o[:, c:2 * c], o[:, 2 * c:3 * c], o[:, 3 * c:]
    rmin, rmax = first_extrema(m, rowptr, perm)
    assert np.array_equal(amin.np(), rmin) and np.array_equal(amax.np(), rmax), what + ": arg-min/max"
    L = np.maximum(lens, 1)[:, None].astype(np.float64)
    has = (lens > 0)[:, None]
    assert np.array_equal(vmin[has[:, 0]], m[rmin[has[:, 0]], np.arange(c)]) if has.any() else True
    assert np.array_equal(vmax[has[:, 0]], m[rmax[has[:, 0]], np.arange(c)]) if has.any() else True
    assert (vmin[~has[:, 0]] == 0).all() and (vmax[~has[:, 0]] == 0).all() and (sd[~has[:, 0]] == 0).all()
    m64 = m.astype(np.float64)
    s1, sa, s2 = seg_sum64(m64, tgt, n), seg_sum64(np.abs(m64), tgt, n), seg_sum64(m64 * m64, tgt, n)
    check_bound(what + ": mean", mean, s1 / L, gamma(L + 1) * sa / L)
    var = s2 / L - (s1 / L) ** 2
    dvar = pna_var_bound(L, s2 / L)
    clear_hi = var > PNA_EPS + dvar + 4 * U * PNA_EPS
    clear_lo = var < PNA_EPS - dvar - 4 * U * PNA_EPS
    assert (sd[clear_lo] == 0).all(), what + ": std not masked below eps"
    assert (sd[clear_hi] > 0).all(), what + ": std masked above eps"
    sref = np.sqrt(np.maximum(var, PNA_EPS))
    check_bound(what + ": std", np.where(clear_hi, sd, 0), np.where(clear_hi, sref, 0), dvar / sref + 2 * U * sref)
    assert clear_hi.sum() > 0 and (n < 100 or clear_lo.sum() > 0), what + ": the case lacks one side of the threshold"

    # backward against fp64 autograd of the same definition, on the entries clear of the threshold
    gout = rng.standard_normal((n, 4 * c)).astype(np.float32)
    gb = Buf(n, 4 * c, data=torch.from_numpy(gout))
    ib = Buf(e, dtype=torch.int32, data=torch.from_numpy(tgt))
    gm = Buf(e, c)
    assert flat_plan("pna_bwd", e * c) <= {"pna_bwd:grid_stride"}
    call = lambda: _lib.call("hgb_pna_aggregate_bwd", gb.ptr, mb.ptr, out.ptr, ib.ptr, rp.ptr, amin.ptr, amax.ptr, e, c, gm.ptr,
                             stream())
    assert launches(call) == int(e > 0)
    gm.check(what, "g_m")
    twice(what + " bwd", call, [gm])
    mt = torch.from_numpy(m64).requires_grad_(True)
    tt = torch.from_numpy(tgt).long()
    Lt = torch.from_numpy(L)
    s1t = torch.zeros(n, c, dtype=torch.float64).index_add(0, tt, mt)
    s2t = torch.zeros(n, c, dtype=torch.float64).index_add(0, tt, mt * mt)
    meant = s1t / Lt
    vart = s2t / Lt - meant * meant
    sdt = torch.where(torch.from_numpy(clear_hi), vart.clamp_min(PNA_EPS).sqrt(), torch.zeros_like(vart))
    ar = torch.arange(c)
    amin_t, amax_t = torch.from_numpy(rmin).clamp_min(0), torch.from_numpy(rmax).clamp_min(0)
    hasm = torch.from_numpy(has).double()
    mint, maxt = mt[amin_t, ar] * hasm, mt[amax_t, ar] * hasm
    g64 = torch.from_numpy(gout.astype(np.float64))
    loss = (torch.cat([meant, mint, maxt, sdt], 1) * g64).sum()
    ref = torch.autograd.grad(loss, mt)[0].numpy()
    # bound: the kernel's roundings (8u on every term) plus the forward errors of the mean and std it reads back
    gmean, gmin, gmax, gstd = (np.abs(gout[:, k * c:(k + 1) * c].astype(np.float64)) for k in range(4))
    sdk = np.where(clear_hi, np.maximum(sref, 1e-300), np.inf)
    dmean = gamma(L + 1) * sa / L
    dsd = dvar / np.where(clear_hi, sref, 1.0) + 2 * U * sref
    dev = np.abs(m64 - (s1 / L)[tgt])
    terms = (gmean / L)[tgt] + (gmin + gmax)[tgt] + (gstd / L / sdk)[tgt] * dev
    fwd = (gstd / L / sdk)[tgt] * (dmean[tgt] + dev * (dsd / sdk)[tgt])
    keep = (clear_hi | clear_lo)[tgt]
    got = gm.np()
    check_bound(what + ": g_m", np.where(keep, got, 0), np.where(keep, ref, 0), 8 * U * terms + fwd)


@pytest.mark.gpu
def test_pna_std_threshold_known_answers():
    """segments {d, -d}: mean 0 and E[x^2] = d^2 exactly in fp32, so std is d or 0 exactly, on either side of eps = 1e-5f"""
    ds = [2.0 ** -8, 13 * 2.0 ** -12, 51 * 2.0 ** -14, 25 * 2.0 ** -13, 3 * 2.0 ** -10, 2.0 ** -9]
    m = np.array([[v] for d in ds for v in (d, -d)], np.float32)
    rowptr = np.arange(0, 2 * len(ds) + 1, 2).astype(np.int32)
    tgt = np.repeat(np.arange(len(ds)), 2).astype(np.int32)
    _, _, out, _, _ = run_pna("pna_known", m, rowptr, None, tgt)
    sd = out.np()[:, 3]
    want = np.array([d if d * d > PNA_EPS else 0.0 for d in ds], np.float32)
    assert [d * d > PNA_EPS for d in ds] == [True, True, False, False, False, False]
    assert (13 * 2.0 ** -12) ** 2 < 1.01 * PNA_EPS and (51 * 2.0 ** -14) ** 2 > 0.96 * PNA_EPS   # within 1 % and 4 % of eps
    same_f32("pna std known answers", sd, want)
    assert (out.np()[:, 0] == 0).all()


def pool_graph_sizes(rng, g):
    sizes = rng.integers(0, 5 if g > 1000 else 9, g)
    sizes[0], sizes[g // 2] = 0, 0
    if g > 2:
        sizes[1] = 1
    return sizes


def pool_reference_f32(x, gptr, mode):
    """row-order fp32 sums (mean: one division), first maximum, in the kernel's order"""
    g = len(gptr) - 1
    lens = np.diff(gptr)
    acc = seq_sum_f32(x, gptr, None)
    if mode == POOL["mean"]:
        return acc / np.maximum(lens, 1).astype(np.float32)[:, None], None
    if mode == POOL["add"]:
        return acc, None
    amin, amax = first_extrema(x, gptr, None)
    out = np.where(amax >= 0, x[np.maximum(amax, 0), np.arange(x.shape[1])], 0).astype(np.float32)
    return out, amax.astype(np.int32)


@pytest.mark.gpu
@pytest.mark.parametrize("g,c", POOL_CASES)
@pytest.mark.parametrize("mode", ["add", "mean", "max"])
def test_pool(g, c, mode):
    what = "pool_%s[g=%d,c=%d]" % (mode, g, c)
    code = POOL[mode]
    rng = np.random.default_rng(g + c + code)
    sizes = pool_graph_sizes(rng, g)
    gptr = np.concatenate([[0], np.cumsum(sizes)]).astype(np.int32)
    n = int(gptr[-1])
    x = rng.standard_normal((n, c)).astype(np.float32)
    if mode == "max":
        x[rng.random((n, c)) < 0.3] = 1.5                          # ties at the maximum
    xb = Buf(n, c, data=torch.from_numpy(x))
    gp = Buf(g + 1, dtype=torch.int32, data=torch.from_numpy(gptr))
    out = Buf(g, c)
    arg = Buf(g, c, dtype=torch.int32) if mode == "max" else None
    fwd = lambda: _lib.call("hgb_pool_fwd", xb.ptr, gp.ptr, g, c, code, out.ptr, arg.ptr if arg else None, stream())
    assert launches(fwd) == 1
    out.check(what, "out")
    if arg:
        arg.check(what, "argmax")
    twice(what, fwd, [out] + ([arg] if arg else []))
    ref, rarg = pool_reference_f32(x, gptr, code)
    same_f32(what, out.np(), ref)
    if mode == "max":
        assert np.array_equal(arg.np(), rarg)
    else:
        x64 = x.astype(np.float64)
        tgt = np.repeat(np.arange(g), sizes)
        L = np.maximum(sizes, 1)[:, None]
        div = L if mode == "mean" else 1
        check_bound(what, out.np(), seg_sum64(x64, tgt, g) / div, (gamma(L + 1) * seg_sum64(np.abs(x64), tgt, g)) / div)

    # backward, plain and (add / mean) through the ReLU mask: y with exact zeros, -0.0 and negatives
    gout = rng.standard_normal((g, c)).astype(np.float32)
    gb = Buf(g, c, data=torch.from_numpy(gout))
    scale = (np.float32(1) / np.maximum(sizes, 1).astype(np.float32)) if mode == "mean" else np.ones(g, np.float32)
    gv = (gout * scale[:, None]).astype(np.float32)
    tgt = np.repeat(np.arange(g), sizes)
    for relu in ([False, True] if mode != "max" else [False]):
        y = np.maximum(x, 0).astype(np.float32)
        y[rng.random((n, c)) < 0.1] = -0.0
        y[rng.random((n, c)) < 0.1] = -1.0
        yb = Buf(n, c, data=torch.from_numpy(y)) if relu else None
        gx = Buf(n, c)
        bwd = lambda: _lib.call("hgb_pool_bwd", gb.ptr, gp.ptr, arg.ptr if arg else None, yb.ptr if yb else None, n, g, c, code,
                                gx.ptr, stream())
        assert launches(bwd) == 1
        gx.check(what, "gx")
        twice(what + " bwd", bwd, [gx])
        want = gv[tgt]
        if mode == "max":
            want = np.where(rarg[tgt] == np.arange(n)[:, None], want, np.float32(0))
        if relu:
            want = np.where(y > 0, want, np.float32(0))
        same_f32(what + (" bwd relu" if relu else " bwd"), gx.np(), want)


@pytest.mark.gpu
@pytest.mark.parametrize("mode", ["add", "mean", "max"])
@pytest.mark.parametrize("relu", [False, True])
def test_pool_bwd_writes_rows_outside_every_graph(mode, relu):
    """Rows that no graph covers ([0, graph_ptr[0]) and [graph_ptr[g], n)) get a zero gradient: gx is a whole [n, c] tensor."""
    if relu and mode == "max":
        pytest.skip("the ReLU mask is for add / mean pooling")
    code, c = POOL[mode], 33
    gptr = np.array([2, 5, 5, 9], np.int32)
    n, g = 13, 3
    rng = np.random.default_rng(1)
    x = rng.standard_normal((n, c)).astype(np.float32)
    xb, gp = Buf(n, c, data=torch.from_numpy(x)), Buf(g + 1, dtype=torch.int32, data=torch.from_numpy(gptr))
    out = Buf(g, c)
    arg = Buf(g, c, dtype=torch.int32) if mode == "max" else None
    _lib.call("hgb_pool_fwd", xb.ptr, gp.ptr, g, c, code, out.ptr, arg.ptr if arg else None, stream())
    gb = Buf(g, c, data=torch.from_numpy(rng.standard_normal((g, c)).astype(np.float32)))
    yb = Buf(n, c, data=torch.from_numpy(np.maximum(x, 0))) if relu else None
    gx = Buf(n, c)
    _lib.call("hgb_pool_bwd", gb.ptr, gp.ptr, arg.ptr if arg else None, yb.ptr if yb else None, n, g, c, code, gx.ptr, stream())
    gx.check("pool_bwd_tail", "gx")
    got = gx.np()
    assert (got[:2] == 0).all() and (got[9:] == 0).all()
    assert not np.signbit(got[:2]).any() and not np.signbit(got[9:]).any()
    # no graph at all: every row is outside
    gx0 = Buf(4, c)
    g0 = Buf(1, dtype=torch.int32, data=torch.zeros(1, dtype=torch.int32))
    _lib.call("hgb_pool_bwd", gb.ptr, g0.ptr, arg.ptr if arg else None, yb.ptr if yb else None, 4, 0, c, code, gx0.ptr, stream())
    gx0.check("pool_bwd_no_graph", "gx")
    assert (gx0.np() == 0).all()


@pytest.mark.gpu
def test_max_pool_tie_rule():
    """The engine gives a tied maximum's whole gradient to its first row; ATen's scatter_reduce("amax") splits it evenly.
    The sums over the tied rows agree; after a ReLU whose tied output is 0 both rules give the same input gradient."""
    c = 2
    x = np.array([[1.0, -1.0], [3.0, -2.0], [3.0, -1.0], [0.5, -3.0]], np.float32)     # channel 0: tie at 3, channel 1: tie at -1
    gptr = np.array([0, 4], np.int32)
    xb, gp = Buf(4, c, data=torch.from_numpy(x)), Buf(2, dtype=torch.int32, data=torch.from_numpy(gptr))
    out, arg = Buf(1, c), Buf(1, c, dtype=torch.int32)
    _lib.call("hgb_pool_fwd", xb.ptr, gp.ptr, 1, c, POOL["max"], out.ptr, arg.ptr, stream())
    assert out.np().tolist() == [[3.0, -1.0]] and arg.np().tolist() == [[1, 0]]
    gb = Buf(1, c, data=torch.tensor([[4.0, 6.0]]))
    gx = Buf(4, c)
    _lib.call("hgb_pool_bwd", gb.ptr, gp.ptr, arg.ptr, None, 4, 1, c, POOL["max"], gx.ptr, stream())
    engine = gx.np()
    assert engine.tolist() == [[0, 6], [4, 0], [0, 0], [0, 0]]
    xt = torch.from_numpy(x).double().requires_grad_(True)
    pooled = torch.zeros(1, c, dtype=torch.float64).scatter_reduce(0, torch.zeros(4, c, dtype=torch.long), xt, "amax",
                                                                   include_self=False)
    aten = torch.autograd.grad((pooled * torch.tensor([[4.0, 6.0]], dtype=torch.float64)).sum(), xt)[0].numpy()
    assert aten.tolist() == [[0, 3], [2, 0], [2, 3], [0, 0]]
    assert np.array_equal(engine.sum(0), aten.sum(0))
    # ties produced by a ReLU at 0: the ReLU's backward (select on y > 0) zeroes every tied row under either rule
    z = np.array([[-1.0], [-2.0], [-0.5]], np.float32)
    y = np.maximum(z, 0)
    yb, gp3 = Buf(3, 1, data=torch.from_numpy(y)), Buf(2, dtype=torch.int32, data=torch.tensor([0, 3], dtype=torch.int32))
    out1, arg1, gx1 = Buf(1, 1), Buf(1, 1, dtype=torch.int32), Buf(3, 1)
    _lib.call("hgb_pool_fwd", yb.ptr, gp3.ptr, 1, 1, POOL["max"], out1.ptr, arg1.ptr, stream())
    g1 = Buf(1, 1, data=torch.tensor([[5.0]]))
    _lib.call("hgb_pool_bwd", g1.ptr, gp3.ptr, arg1.ptr, None, 3, 1, 1, POOL["max"], gx1.ptr, stream())
    assert gx1.np().ravel().tolist() == [5.0, 0.0, 0.0]                 # ATen: 5/3 to each row
    assert (np.where(y > 0, gx1.np(), 0) == 0).all() and (np.where(y > 0, np.full((3, 1), 5.0 / 3), 0) == 0).all()


# ---- 4. loss, AdamW, capacity helpers ----------------------------------------------------------------------------------------------
def run_loss(what, pred, target, mode, gscale, valid=None, row_width=1):
    count = pred.size
    pb, tb = Buf(count, data=torch.from_numpy(pred)), Buf(count, data=torch.from_numpy(target))
    loss, gp = Buf(1), Buf(count)
    vb = Buf(1, dtype=torch.int32, data=torch.tensor([valid], dtype=torch.int32)) if valid is not None else None
    call = lambda: _lib.call("hgb_loss_fwd_bwd", pb.ptr, tb.ptr, count, mode, float(gscale), loss.ptr, gp.ptr,
                             vb.ptr if vb else None, row_width, stream())
    assert launches(call) == 1
    loss.check(what, "loss")
    gp.check(what, "gpred")
    twice(what, call, [loss, gp])
    return float(loss.np()[0, 0]), gp.np()[:, 0]


def loss_reference(pred, target, mode, gscale, cnt):
    d = pred[:cnt].astype(np.float64) - target[:cnt]
    if cnt == 0:
        return 0.0, np.zeros(0), 0.0, np.zeros(0)
    gs = float(np.float32(gscale))
    L = cdiv(cnt, 1024) + 10 + 1 + 3
    if mode == 0:
        return (d * d).mean(), 2 * d / cnt * gs, gamma(L) * (d * d).mean(), gamma(4) * np.abs(2 * d / cnt * gs)
    return np.abs(d).mean(), np.sign(d) / cnt * gs, gamma(L) * np.abs(d).mean(), gamma(3) * np.abs(np.sign(d) / cnt * gs)


@pytest.mark.gpu
@pytest.mark.parametrize("count", LOSS_COUNTS)
@pytest.mark.parametrize("mode", [0, 1])
def test_loss(count, mode):
    rng = np.random.default_rng(count + mode)
    pred = rng.standard_normal(count).astype(np.float32)
    target = (pred + rng.standard_normal(count) * np.exp(rng.uniform(-4, 1, count))).astype(np.float32)
    target[: min(3, count - 1)] = pred[: min(3, count - 1)]            # d == 0: MAE's gradient is 0 there
    for gscale in (1.0, 0.37):
        what = "loss[mode=%d,count=%d,gscale=%g]" % (mode, count, gscale)
        lv, gp = run_loss(what, pred, target, mode, gscale)
        ref, gref, lb, gb = loss_reference(pred, target, mode, gscale, count)
        check_bound(what + ": loss", np.array([lv]), np.array([ref]), np.array([lb]))
        check_bound(what + ": gpred", gp, gref, gb)


@pytest.mark.gpu
@pytest.mark.parametrize("mode", [0, 1])
@pytest.mark.parametrize("valid,row_width", [(5, 3), (1, 4), (40, 3), (7, 1), (0, 3), (-2, 3)])
def test_loss_valid_rows(mode, valid, row_width):
    """Only the first valid * row_width entries are real: the mean runs over them and gpred is exactly +0 beyond.
    No real row at all (valid <= 0) gives loss 0 and an all-zero gradient."""
    rng = np.random.default_rng(valid + 10 * row_width)
    count = 30 * row_width
    pred = rng.standard_normal(count).astype(np.float32)
    target = rng.standard_normal(count).astype(np.float32)
    what = "loss_valid[mode=%d,valid=%d,w=%d]" % (mode, valid, row_width)
    lv, gp = run_loss(what, pred, target, mode, 0.5, valid=valid, row_width=row_width)
    cnt = min(max(valid, 0) * row_width, count)
    ref, gref, lb, gb = loss_reference(pred, target, mode, 0.5, cnt)
    assert np.array_equal(gp[cnt:].view(np.int32), np.zeros(count - cnt, np.int32)), what + ": gpred past the valid rows"
    if cnt == 0:
        assert np.float32(lv).view(np.int32) == 0, what + ": loss is not +0"

    else:
        check_bound(what + ": loss", np.array([lv]), np.array([ref]), np.array([lb]))
        check_bound(what + ": gpred", gp[:cnt], gref, gb)


def f32(x):
    return float(np.float32(x))


def adamw_ref_step(p, g, m, v, t, lr, b1, b2, eps, wd, gs):
    """fp64 AdamW step from the fp32 state, with the fp32-rounded hyper-parameters the ABI receives"""
    gi = g * gs
    p1 = p * (1 - lr * wd)
    M = b1 * np.abs(m) + (1 - b1) * np.abs(gi)
    m1 = b1 * m + (1 - b1) * gi
    v1 = b2 * v + (1 - b2) * gi * gi
    bc1, bc2 = 1 - b1 ** t, 1 - b2 ** t
    den = np.sqrt(v1) / math.sqrt(bc2) + eps
    upd = lr / bc1 * m1 / den
    pow_err = 4 * U                                             # powf: 4 ulp of b^t < 1
    bound = (np.abs(upd) * (pow_err / bc1 + pow_err / bc2 / 2 + 24 * U) + lr / bc1 * gamma(4) * M / den
             + 4 * U * np.abs(p) + 2 * U * np.abs(p1 - upd))
    return p1 - upd, m1, v1, p1 - upd - p, bound, gamma(4) * M, gamma(6) * v1


@pytest.mark.gpu
@pytest.mark.parametrize("count", ADAMW_COUNTS)
@pytest.mark.parametrize("form", ["by_value", "hyper_dev"])
def test_adamw(count, form):
    rng = np.random.default_rng(count)
    lr, b1, b2, eps, wd, gs = f32(3e-2), f32(0.9), f32(0.999), f32(1e-8), f32(0.05), f32(0.25)
    p0 = (rng.standard_normal(count) * lr).astype(np.float32)
    p, m, v = Buf(count, data=torch.from_numpy(p0)), Buf(count, data=torch.zeros(count)), Buf(count, data=torch.zeros(count))
    step = Buf(1, data=torch.zeros(1))
    hyper = Buf(2, data=torch.tensor([lr, gs])) if form == "hyper_dev" else None
    for t in range(1, 22):
        gnp = (rng.standard_normal(count) * np.exp(rng.uniform(-3, 2, count))).astype(np.float32)
        gnp[:3] = 0
        gb = Buf(count, data=torch.from_numpy(gnp))
        st = [x.np()[:, 0].astype(np.float64) for x in (p, m, v)]
        args_lr, args_gs = (lr, gs) if form == "by_value" else (123.0, -7.0)       # hyper_dev overrides both
        call = lambda: _lib.call("hgb_adamw_step", p.ptr, gb.ptr, m.ptr, v.ptr, count, args_lr, b1, b2, eps, wd, args_gs, step.ptr,
                                 hyper.ptr if hyper else None, stream())
        assert launches(call) == 2
        for b, name in ((p, "p"), (m, "m"), (v, "v"), (step, "step"), (gb, "g")):
            b.check("adamw", name)
        assert float(step.np()[0, 0]) == t
        pn, m1, v1, dref, bound, mb, vb = adamw_ref_step(*st[:1], gnp.astype(np.float64), st[1], st[2], t, lr, b1, b2, eps, wd, gs)
        got = [x.np()[:, 0] for x in (p, m, v)]
        what = "adamw[%s,count=%d,t=%d]" % (form, count, t)
        check_bound(what + ": update", got[0].astype(np.float64) - st[0], dref, bound)
        check_bound(what + ": m", got[1], m1, mb)
        check_bound(what + ": v", got[2], v1, vb)
    # the same step twice from the same state: the same bits
    snap = [x.base.clone() for x in (p, m, v)]
    step.view.fill_(5.0)
    call()
    first = [x.base.clone() for x in (p, m, v)]
    for x, s in zip((p, m, v), snap):
        x.base.copy_(s)
    step.view.fill_(5.0)
    call()
    torch.cuda.synchronize()
    for x, f in zip((p, m, v), first):
        assert torch.equal(x.base.view(torch.int32), f.view(torch.int32)), "adamw: two identical steps differ"


@pytest.mark.gpu
def test_adamw_count_zero_moves_only_the_step():
    p, g, m, v = (Buf(0) for _ in range(4))
    step = Buf(1, data=torch.tensor([41.0]))
    call = lambda: _lib.call("hgb_adamw_step", p.ptr, g.ptr, m.ptr, v.ptr, 0, 1e-3, 0.9, 0.999, 1e-8, 0.01, 1.0, step.ptr, None,
                             stream())
    assert launches(call) == 1
    assert float(step.np()[0, 0]) == 42.0
    for b in (p, g, m, v):
        b.check("adamw_empty", "buffer", written=False)


@pytest.mark.gpu
def test_adamw_distance_to_torch():
    """The kernel works on the fp32 betas the ABI receives: v is scaled by 1.f - 0.999f and bias-corrected by 1 - powf(0.999f, t).
    torch.optim.AdamW scales v by the double 1 - 0.999 (rounded to fp32 in the multiply) and bias-corrects in double.  The two
    updates of the same state are therefore a few 1e-6 apart (normwise, relative): about 3.4e-6 at t = 2, falling below 1e-6
    later.  That distance is a property of the float ABI, not rounding noise, and it is pinned to [1e-6, 1e-5] over 30 steps:
    a change to double bias correction or to the betas the kernel receives moves it out of that window."""
    rng = np.random.default_rng(2)
    count, lr = 4096, 1e-2
    p0 = torch.from_numpy((rng.standard_normal(count) * lr).astype(np.float32))
    pt = p0.clone().to(DEV).requires_grad_(True)
    opt = torch.optim.AdamW([pt], lr=lr, betas=(0.9, 0.999), eps=1e-8, weight_decay=0.0, foreach=False)
    p, m, v = Buf(count, data=p0), Buf(count, data=torch.zeros(count)), Buf(count, data=torch.zeros(count))
    step = Buf(1, data=torch.zeros(1))
    dist = []
    for t in range(1, 31):
        gt = torch.from_numpy((rng.standard_normal(count) * np.exp(rng.uniform(-2, 2, count))).astype(np.float32)).to(DEV)
        before = pt.detach().clone()
        gb = Buf(count, data=gt)
        _lib.call("hgb_adamw_step", p.ptr, gb.ptr, m.ptr, v.ptr, count, lr, 0.9, 0.999, 1e-8, 0.0, 1.0, step.ptr, None, stream())
        pt.grad = gt.clone()
        opt.step()
        dk = (p.view[:, 0] - before).double()
        dt = (pt.detach() - before).double()
        p.view[:, 0].copy_(pt.detach())                                   # both continue from torch's parameters
        dist.append(float((dk - dt).norm() / dt.norm()))
    assert 1e-6 <= max(dist) <= 1e-5, "kernel and torch.optim.AdamW updates %.3g apart (normwise relative)" % max(dist)


@pytest.mark.gpu
def test_clamp_and_expect_i32():
    rng = np.random.default_rng(9)
    for n, cap in ((1, 3), (1000, 7), (600_000, 0), (50, 2 ** 31 - 1)):
        x = rng.integers(-5, 20, n).astype(np.int32)
        xb, out = Buf(n, dtype=torch.int32, data=torch.from_numpy(x)), Buf(n, dtype=torch.int32)
        call = lambda: _lib.call("hgb_clamp_i32", xb.ptr, cap, n, out.ptr, stream())
        assert launches(call) == 1
        out.check("clamp", "out")
        assert np.array_equal(out.np()[:, 0], np.minimum(x, cap))
        twice("clamp", call, [out])
    for value, expected, bit, before, after in ((5, 5, 4, 0, 0), (5, 6, 4, 0, 4), (5, 6, 1, 8, 9), (-1, 7, 2, 2, 2)):
        vb = Buf(1, dtype=torch.int32, data=torch.tensor([value], dtype=torch.int32))
        fb = Buf(1, dtype=torch.int32, data=torch.tensor([before], dtype=torch.int32))
        assert launches(lambda: _lib.call("hgb_expect_i32", vb.ptr, expected, bit, fb.ptr, stream())) == 1
        fb.check("expect", "flag")
        assert int(fb.np()[0, 0]) == after


@pytest.mark.gpu
@pytest.mark.parametrize("e_real,n_real,n_cap,e_cap", [(10, 6, 10, 40), (0, 0, 5, 12), (40, 6, 10, 40), (41, 6, 10, 40),
                                                        (10, 9, 10, 40), (3, 2, 4, 600_001)])
def test_pad_edges(e_real, n_real, n_cap, e_cap):
    """slots [e_real, e_cap) get the ring n_real -> n_real + 1 -> ... -> n_cap - 1 -> n_real; guard bit 1 when e_real > e_cap or
    fewer than 2 filler nodes remain, and then nothing is written"""
    ei0 = np.arange(2 * e_cap, dtype=np.int64) + 1000                    # stands for the real edges: must stay
    eb = Buf(2 * e_cap, dtype=torch.int64, data=torch.from_numpy(ei0))
    er, nr = Buf(1, dtype=torch.int32, data=torch.tensor([e_real], dtype=torch.int32)), Buf(1, dtype=torch.int32,
                                                                                            data=torch.tensor([n_real], dtype=torch.int32))
    flag = Buf(1, dtype=torch.int32, data=torch.zeros(1, dtype=torch.int32))
    call = lambda: _lib.call("hgb_pad_edges", er.ptr, nr.ptr, n_cap, e_cap, eb.ptr, flag.ptr, stream())
    assert launches(call) == 1
    eb.check("pad_edges", "edge_index")
    fl = int(flag.np()[0, 0])
    got = eb.np()[:, 0].reshape(2, e_cap)
    p = n_cap - n_real
    want = ei0.reshape(2, e_cap).copy()
    if e_real > e_cap or p < 2:
        assert fl == GUARD_EDGE_COUNT == 1
    else:
        assert fl == 0
        k = (np.arange(e_real, e_cap) - e_real) % p
        want[0, e_real:] = n_real + k
        want[1, e_real:] = n_real + (k + 1) % p
    assert np.array_equal(got, want)
    twice("pad_edges", call, [eb])


# ---- 5. periodic image pruning (radius_pbc_kernel) ---------------------------------------------------------------------------------
def brute_force_count(pos64, cell, pbc, cutoff):
    """candidates (src, S) of an unpruned fp64 search over a generous image range, counted per target"""
    n = pos64.shape[0]
    frac = pos64 @ np.linalg.inv(cell)
    rng = []
    for a in range(3):
        if not pbc[a]:
            rng.append(np.zeros(1, np.int64))
            continue
        h = abs(np.linalg.det(cell)) / np.linalg.norm(np.cross(cell[(a + 1) % 3], cell[(a + 2) % 3]))
        na = int(np.ceil(cutoff / h + np.ptp(frac[:, a]))) + 3
        rng.append(np.arange(-na, na + 1))
    S = np.stack(np.meshgrid(*rng, indexing="ij"), -1).reshape(-1, 3).astype(np.float64)
    d = pos64[None, :, :] - pos64[:, None, :]                              # [i, j] = pos[j] - pos[i]
    cnt = np.zeros(n, np.int64)
    for s in np.array_split(S, max(1, len(S) * n * n // 2_000_000)):
        v = d[None] + (s @ cell)[:, None, None, :]
        ok = (v * v).sum(-1) < cutoff * cutoff
        zero = (s == 0).all(1)
        ok[zero] &= ~np.eye(n, dtype=bool)
        cnt += ok.sum((0, 1))
    return cnt


def pbc_case(name, rng):
    """(list of (pos [k,3] fp64, cell [3,3], pbc [3], cutoff), max_neighbours)"""
    cube = np.eye(3) * 3.0
    sheared = np.array([[4.0, 0, 0], [3.9, 1.0, 0], [0.5, 0.3, 4.0]])       # the b height is 0.25 |b|
    if name == "cutoff_longer_than_cell":
        return [(rng.random((20, 3)) @ cube, cube, [1, 1, 1], 7.5)], 10 ** 6
    if name == "strongly_sheared":
        return [(rng.random((25, 3)) @ sheared, sheared, [1, 1, 1], 3.0)], 10 ** 6
    if name == "unwrapped":
        return [(rng.uniform(-3, 4, (12, 3)) @ sheared, sheared, [1, 1, 1], 2.5)], 10 ** 6
    if name == "left_handed":
        lh = sheared[[1, 0, 2]]
        assert np.linalg.det(lh) < 0
        return [(rng.uniform(-1, 2, (20, 3)) @ lh, lh, [1, 1, 1], 3.0)], 10 ** 6
    if name == "one_periodic_axis":
        return [(rng.random((30, 3)) @ sheared, sheared, [0, 1, 0], 3.5)], 10 ** 6
    if name == "large_graph":
        big = np.diag([7.0, 6.0, 6.5])
        return [(rng.random((150, 3)) @ big, big, [1, 1, 1], 3.0)], 10 ** 6
    if name == "mixed_batch":
        tri = np.array([[5.0, 0, 0], [1.0, 4.0, 0], [-0.7, 0.4, 3.5]])
        return [(rng.random((9, 3)) @ cube, cube, [1, 1, 1], 2.8), (rng.uniform(-2, 3, (17, 3)) @ tri, tri, [1, 0, 1], 3.3),
                (rng.random((1, 3)) @ cube, cube, [1, 1, 1], 3.5), (rng.random((140, 3)) @ (tri * 1.6), tri * 1.6, [1, 1, 1], 2.5),
                (rng.random((6, 3)) @ sheared, sheared, [0, 0, 0], 3.0)], 12
    if name == "truncation_small_k":
        return [(rng.random((30, 3)) @ sheared, sheared, [1, 1, 1], 4.0)], 5
    if name == "bcc_k10":
        a = 3.0
        base = np.array([[0, 0, 0], [0.5, 0.5, 0.5]]) * a
        pos = np.concatenate([base + np.array([i, j, k]) * a for i in range(2) for j in range(2) for k in range(2)])
        return [(pos, np.eye(3) * 2 * a, [1, 1, 1], 3.2)], 10                # shells: 8 at a sqrt(3)/2, 6 at a: k = 10 cuts the 6
    raise KeyError(name)


PBC_CASES = ["cutoff_longer_than_cell", "strongly_sheared", "unwrapped", "left_handed", "one_periodic_axis", "large_graph",
             "mixed_batch", "truncation_small_k", "bcc_k10"]


@pytest.mark.gpu
@pytest.mark.parametrize("dtype", [torch.float32, torch.float64])
@pytest.mark.parametrize("name", PBC_CASES)
def test_pbc_pruning_bit_exact_vs_oracle(name, dtype):
    rng = np.random.default_rng(len(name))
    graphs, k = pbc_case(name, rng)
    pos = torch.cat([torch.from_numpy(p) for p, _, _, _ in graphs]).to(dtype)
    sizes = [p.shape[0] for p, _, _, _ in graphs]
    g = len(graphs)
    gptr = torch.tensor(np.concatenate([[0], np.cumsum(sizes)]), dtype=torch.int32, device=DEV)
    cell = torch.tensor(np.stack([c for _, c, _, _ in graphs]), dtype=torch.float64)
    pbc = torch.tensor([b for _, _, b, _ in graphs], dtype=torch.int32)
    cutoff = torch.tensor([r for _, _, _, r in graphs], dtype=torch.float64)
    run = lambda: radius.radius_graph_pbc(pos.to(DEV), cell, pbc, cutoff, gptr, g, k)
    ei, cs, sh, deg, outptr, ncand = run()
    ei2, cs2, sh2, _, _, _ = run()
    assert torch.equal(ei, ei2) and torch.equal(cs, cs2) and torch.equal(sh.view(torch.uint8), sh2.view(torch.uint8))
    off, ref_ei, ref_sh, ref_cnt, brute = 0, [], [], [], []
    for (p, c, b, r), sz in zip(graphs, sizes):
        p64 = pos[off:off + sz].double().numpy()                      # the positions the kernel reads, widened
        src, dst, S, length = _neighbor_list_ijS(p64, c, b, r)
        ref_cnt.append(np.bincount(dst, minlength=sz))
        brute.append(brute_force_count(p64, c, b, r))
        src, dst, length, S = limit_neighbors(src, dst, length, S, k)
        ref_ei.append(np.stack([src, dst]) + off)
        ref_sh.append(_shift_vectors(S, c))
        off += sz
    ref_cnt, brute = np.concatenate(ref_cnt), np.concatenate(brute)
    assert np.array_equal(ref_cnt, brute), "the oracle's image range misses candidates"
    assert ncand == int(brute.sum()), "%s: %d candidates, an unpruned fp64 search finds %d" % (name, ncand, int(brute.sum()))
    assert np.array_equal(deg.cpu().numpy(), np.minimum(brute, k))
    ref_ei = np.concatenate(ref_ei, 1)
    ref_sh = np.concatenate(ref_sh).astype(np.float32 if dtype == torch.float32 else np.float64)
    assert np.array_equal(ei.cpu().numpy(), ref_ei), "%s: edge_index differs from the oracle" % name
    assert np.array_equal(sh.cpu().numpy().view(np.uint8), ref_sh.view(np.uint8)), "%s: edge_shifts differ" % name
    if name == "bcc_k10":
        assert (brute == 14).all() and (deg.cpu().numpy() == 10).all()
