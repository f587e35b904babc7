"""Kernel-level tests of the geometry every geometric stack runs through: the open-boundary radius graph of csrc/hgb_radius.cu
(hgb_radius_graph_count / _fill), the edge vectors, lengths and units of csrc/hgb_geom.cu (hgb_edge_geom_fwd / _bwd) and the
closed edge-length primitives of csrc/hgb_egnn.cu (hgb_edge_len_bwd / _bwd2, hgb_edge_vec_scatter) that carry the position
gradient of force training, including its double backward.  Each is checked against a plain restatement computed on the CPU
from the same fp32 inputs, then the autograd wrappers are checked at workload shapes against fp64 torch autograd.

The C-ABI is called directly through tests/kernel_harness.py: every operand is the leading block of a NaN / SENTINEL-filled
buffer followed by guard rows, `Buf.check` asserts that every element in range was written and nothing else changed, every
call runs twice with identical bits, and every call launches the one kernel the host dispatch (grid_for(e, 256) over edges,
grid_for(n, 128) over nodes, capped at 132 x 16 blocks) predicts, none when there is no work.

u = 2^-24, gamma(k) = k u / (1 - k u).  nvcc contracts products into FMAs (no --fmad=false), so a result with a product gets a
bound, not bits; an FMA only removes roundings, so every bound below holds with or without contraction.  sqrtf and 1.f / x are
correctly rounded (no fast-math flags).

Exactness rules and bounds:
* Radius graph: integers, and the accept test d2 < r*r uses explicitly rounded __fmul_rn / __fadd_rn, so deg, rowptr and
  edge_index equal oracle.radius_graph.radius_graph bit for bit.  Fill slots the kernel must not write keep their SENTINEL.
* vec = (pos[col] - pos[row]) (+ shift): one or two rounded subtractions / additions, no product, so it equals the fp32
  restatement bit for bit.
* len = sqrtf(vx*vx + vy*vy + vz*vz): the sum of three non-negative squares carries a relative error theta <= gamma(3);
  sqrt halves it (|sqrt(1 + theta) - 1| <= gamma(3)/2 (1 + gamma(3))) and rounds once more:
  |len - |vec|| <= DL |vec|,  DL = gamma(3)/2 (1 + gamma(3)) (1 + u) + u.
* unit = vec * (1 / (len + eps)): len + eps is off by DL relative (eps >= 0), then one rounding each for the add, the
  reciprocal and the product: |unit_k - vec_k / (|vec| + eps)| <= (DL + 3u) |vec_k| / (|vec| + eps).
* edge_geom_bwd: g = g_in + g_unit / L + (g_len / len - <g_unit, vec> / (L^2 len)) vec, L = len + eps, from the fp32 vec and
  len it is given.  Counting the roundings on each of the four terms (at most gamma(3) + 11u on the curvature term) gives
  |err_k| <= 16u (|g_in_k| + |g_unit_k| / L + |g_len| |vec_k| / len + sum_m |g_unit_m vec_m| |vec_k| / (L^2 len)).
* edge_len_bwd: gvec_k = (gd / len) vec_k: |err_k| <= (DL + 2u) |gd vec_k| / |vec|.
* edge_len_bwd2, with h = vec / |vec|, w = ggpos[col] - ggpos[row] (one rounded subtraction: restated exactly in fp32) and
  S = sum_m |h_m w_m|: g_gd = <h, w> within (gamma(3) + DL + 2u) S, and q_k = gd (w_k - h_k <h, w>) / |vec| within
  |gd| / |vec| ((DL + 4u) |w_k| + (gamma(3) + 3 DL + 9u) |h_k| S).
* len == 0 (self-loops, coincident atoms): 1 / len := 0.  Then gvec, g_gd and q are exactly 0 and edge_geom_bwd keeps only
  g_in + g_unit / eps.  g_gd = 0 and the first-order rule are what torch.linalg.norm's backward gives
  (test_references_match_torch_autograd); torch's double backward of q is 0 * inf = NaN there, the kernel takes 0.
* edge_vec_scatter adds each node's col edges, then its row edges, one after the other in CSR order and subtracts once, so it
  equals an fp32 sequential restatement bit for bit, and fp64 within gamma(L + 1) (sum_col |g| + sum_row |g|), L the longer of
  the two segments (Higham, Accuracy and Stability of Numerical Algorithms, 2nd ed., eq. 3.5).
* Autograd wrappers at workload shapes: the fp64 reference is torch autograd of oracle.geometry.edge_vectors_and_lengths
  with the value of vec replaced by the exact fp32 vec (its derivative kept), so the bounds need not carry the rounding of
  pos[col] - pos[row] + shift, which is large next to |vec| when a periodic shift cancels a long difference.  Lengths are
  held within DL |vec| per element.  A force is a sum over a node's edges of per-edge terms t_e plus the ordered scatter:
  |F_i,k - F*_i,k| <= (C_GD + c_edge + gamma(L_i + 1)) sum_e |t_e,k|, where
  - C_GD = u + DL: the energy sum c d^2 hands back gd = 2 c d with one rounding (autograd adds the two equal halves
    exactly), from the forward's len, which is off by DL;
  - c_edge = DL + 2u for EdgeLenFn (edge_len_bwd, whose own len is off by DL again), and 16u + 3 DL for EdgeGeomFn
    (edge_geom_bwd's bound above, fed the forward's len, whose DL enters L^2 len up to three times).
  Two tolerances are estimates, not derivations: 16u + 3 DL + 8u for the ATen any-order path, whose norm, division and
  separately accumulated gradients are not restated, and rel-L2 4e-6 for the force-loss position gradient (the double
  backward chains bwd2, two scatters and the first-order backward again; each of its terms is within about 40u = 2.4e-6
  relative, and the 4e-6 assumes node sums that cancel by less than a factor of two at these shapes).  Both are tighter
  than the 1e-5 rel-L2 the wrappers were held to before.

test_cases_reach_every_form (no GPU) asserts that the case lists reach every form the issue of these kernels names, and
test_mutations_are_caught (no GPU) runs deliberately wrong fp32 restatements through the same comparison functions and case
lists and asserts that each one fails, while the faithful restatements pass.
"""
import functools
import zlib

import numpy as np
import pytest
import torch

from hydragnn_b200 import _lib, ops, radius, stacks
from hydragnn_b200.synthetic import WORKLOADS, make_samples
from kernel_harness import SENTINEL, U, Buf, cdiv, check_bound, gamma, grid_for, launches, same_f32, stream, twice
from oracle.geometry import edge_vectors_and_lengths
from oracle.radius_graph import radius_graph as oracle_radius_graph

NO_CAP = radius._NO_CAP - 1                       # what radius.radius_graph passes for "no cap"
DL = 0.5 * gamma(3) * (1 + gamma(3)) * (1 + U) + U
SLACK = 1 + 1e-5                                  # second-order terms of the first-order bounds above
C_UNIT = (DL + 3 * U) * SLACK
C_GEOM_BWD = 16 * U
C_GD = U + DL                                     # gd = 2 c d: the product's rounding and the forward's own len error
C_GEOM_EDGE = C_GEOM_BWD + 3 * DL                  # edge_geom_bwd fed the forward's len: DL enters L^2 len up to three times
C_ANY_ORDER = C_GEOM_EDGE + 8 * U                 # an estimate: ATen's norm, division and their separately rounded gradients
C_LEN_BWD = (DL + 2 * U) * SLACK
C_HW = (gamma(3) + DL + 2 * U) * SLACK
C_QW = (DL + 4 * U) * SLACK
C_QH = (gamma(3) + 3 * DL + 9 * U) * SLACK
EDGE_BLOCK, NODE_BLOCK = 256, 128


def bound(what, got, ref, b):
    """check_bound, and no NaN / inf slips through as an incomparable error"""
    got = np.asarray(got)
    if not np.isfinite(got).all():
        pytest.fail("%s: %d non-finite entries" % (what, int((~np.isfinite(got)).sum())))
    check_bound(what, got, ref, b)


def iters(work, per_block):
    """grid-stride passes of a kernel launched with grid_for(work, per_block) blocks"""
    return cdiv(work, grid_for(work, per_block) * per_block) if work else 0


def f32(x):
    return float(np.float32(x))


# ================================================================================================================================
# 1. open-boundary radius graph
# ================================================================================================================================
# (name, layout, sizes or workload graph count, box, r, max_num_neighbors, loop, fill capacity)
RADIUS_CASES = [
    ("mixed_k5", "box", [0, 9, 21, 1, 2, 80, 0, 9, 0], 5.0, 4.0, 5, False, "exact"),
    ("mixed_k5_loop", "box", [0, 9, 21, 1, 2, 80, 0, 9, 0], 5.0, 4.0, 5, True, "exact"),
    ("k1", "box", [9, 21, 1, 30], 4.0, 3.0, 1, False, "exact"),
    ("k1_loop", "box", [9, 21, 1, 30], 4.0, 3.0, 1, True, "exact"),
    ("k128_large_graphs", "box", [300, 257, 40], 6.0, 4.0, 128, False, "exact"),
    ("k128_large_graphs_loop", "box", [300, 257, 40], 6.0, 4.0, 128, True, "exact"),
    ("no_cap", "box", [0, 50, 130, 1], 6.0, 3.5, NO_CAP, False, "exact"),
    ("no_cap_loop", "box", [0, 50, 130, 1], 6.0, 3.5, NO_CAP, True, "exact"),
    ("coincident_k5", "point", [12, 7, 30], 4.0, 3.0, 5, False, "exact"),
    ("coincident_no_cap_loop", "point", [12, 7, 30], 4.0, 3.0, NO_CAP, True, "exact"),
    ("exact_r_dyadic", "dyadic", [27, 64], 0.0, 1.0, NO_CAP, False, "exact"),
    ("exact_r_dyadic_k5", "dyadic", [27, 64], 0.0, 1.0, 5, False, "exact"),
    ("r_0.1", "box", [40, 60], 0.3, 0.1, NO_CAP, False, "exact"),
    ("fill_larger_capacity", "box", [0, 9, 21, 1, 2, 80, 0, 9, 0], 5.0, 4.0, 5, False, "larger"),
    ("fill_smaller_capacity", "box", [0, 9, 21, 1, 2, 80, 0, 9, 0], 5.0, 4.0, 5, False, "smaller"),
    ("grid_stride", "many", 10_000, 0.0, 5.0, 20, False, "exact"),
    ("qm9_painn", "workload", 64, 0.0, None, None, False, "exact"),
    ("md17_egnn", "workload", 32, 0.0, None, None, False, "exact"),
    ("ogb_pna", "workload", 32, 0.0, None, None, False, "exact"),
    ("oc20_mace", "workload", 4, 0.0, None, None, False, "exact"),
]
RADIUS_BY_NAME = {c[0]: c for c in RADIUS_CASES}


@functools.lru_cache(maxsize=None)
def radius_inputs(name):
    """(pos [n, 3] fp32, graph_ptr [g + 1] int32, r, max_num_neighbors, loop, fill)"""
    _, layout, sizes, box, r, k, loop, fill = RADIUS_BY_NAME[name]
    rng = np.random.default_rng(zlib.crc32(name.encode()))
    if layout == "workload":
        w = WORKLOADS[name]
        b = make_samples(name, sizes)
        return b.pos.numpy().astype(np.float32), b.ptr.numpy().astype(np.int32), w["radius"], w["max_neighbours"], loop, fill
    if layout == "many":                          # ~30-atom graphs at 0.1 / A^3: more nodes than one grid pass covers
        sizes = list(rng.integers(25, 36, sizes))
        parts = [rng.random((s, 3)) * (s / 0.1) ** (1 / 3) for s in sizes]
    elif layout == "dyadic":                      # a cubic grid of spacing 0.5: many pairs at exactly r = 1.0
        parts = []
        for s in sizes:
            m = round(s ** (1 / 3))
            parts.append(np.stack(np.meshgrid(*[np.arange(m)] * 3, indexing="ij"), -1).reshape(-1, 3) * 0.5)
    else:
        parts = [rng.random((s, 3)) * box for s in sizes]
        if layout == "point":                     # every atom of the second graph at one point: d2 = 0, the cap alone decides
            parts[1][:] = parts[1][0]
    ptr = np.concatenate([[0], np.cumsum([len(p) for p in parts])]).astype(np.int32)
    pos = np.concatenate(parts).astype(np.float32) if parts else np.zeros((0, 3), np.float32)
    return np.ascontiguousarray(pos), ptr, r, k, loop, fill


def batch_of(ptr):
    return torch.repeat_interleave(torch.arange(len(ptr) - 1), torch.from_numpy(np.diff(ptr).astype(np.int64)))


@functools.lru_cache(maxsize=None)
def radius_reference(name):
    """oracle edge_index [2, E] int64 and in-degree [n] of a case"""
    pos, ptr, r, k, loop, _ = radius_inputs(name)
    ei = oracle_radius_graph(torch.from_numpy(pos), r, batch_of(ptr), loop, k).numpy()
    deg = np.bincount(ei[1], minlength=pos.shape[0]).astype(np.int32)
    return ei, deg


def radius_restated(pos, ptr, r, k, loop, strict=True, plus_one=True):
    """The kernel's loop, vectorised over graphs of one size: (deg [n], edge_index [2, E]).  strict / plus_one = False are
    mutations (`<=` for `<`, the cap without its + 1 when loop is False)."""
    n = pos.shape[0]
    r2 = np.float32(r) * np.float32(r)
    cap = k if (loop or not plus_one) else k + 1
    sizes = np.diff(ptr)
    accepted = []                                 # (query, neighbour) pairs
    for s in np.unique(sizes[sizes > 0]):
        lo = ptr[:-1][sizes == s]
        idx = lo[:, None] + np.arange(s)[None, :]
        q = pos[idx]                              # [G, s, 3]
        d = q[:, None, :, :] - q[:, :, None, :]   # [G, i, j] = x[j] - x[i]
        sq = d * d
        d2 = (sq[..., 0] + sq[..., 1]) + sq[..., 2]
        ok = d2 < r2 if strict else d2 <= r2
        ok &= (np.cumsum(ok, axis=2) - 1) < cap
        if not loop:
            ok &= ~np.eye(s, dtype=bool)[None]
        gi, qi, nj = np.nonzero(ok)
        accepted.append(np.stack([idx[gi, qi], idx[gi, nj]], 1))
    pairs = np.concatenate(accepted) if accepted else np.zeros((0, 2), np.int64)
    pairs = pairs[np.lexsort((pairs[:, 1], pairs[:, 0]))]
    deg = np.bincount(pairs[:, 0], minlength=n).astype(np.int32)
    return deg, np.stack([pairs[:, 1], pairs[:, 0]]).astype(np.int64)


def capacity_of(fill, count):
    return {"exact": count, "larger": count + 37, "smaller": count // 2}[fill]


def check_radius(what, name, deg, ei, cap):
    """deg [n] and the written block of edge_index [2, cap] against the oracle: slots [0, min(count, cap)) of both rows"""
    ref_ei, ref_deg = radius_reference(name)
    if not np.array_equal(deg, ref_deg):
        pytest.fail("%s: deg differs from the oracle at %d nodes" % (what, int((deg != ref_deg).sum())))
    count = ref_ei.shape[1]
    m = min(count, cap)
    if ei.shape[1] < m or not np.array_equal(ei[:, :m], ref_ei[:, :m]):
        pytest.fail("%s: edge_index differs from the oracle" % what)


def radius_tags(name):
    pos, ptr, r, k, loop, fill = radius_inputs(name)
    n = pos.shape[0]
    sizes = np.diff(ptr)
    tags = {"loop" if loop else "no_loop", "fill:" + fill}
    deg, _ = radius_restated(pos, ptr, r, k, loop)
    uncapped, _ = radius_restated(pos, ptr, r, NO_CAP, loop)
    binds = deg < uncapped                        # nodes whose neighbour list the cap cut short
    if k == NO_CAP:
        tags.add("no_cap")
    elif binds.any():
        tags.add("k%d_binds" % k)
    if RADIUS_BY_NAME[name][1] == "workload":
        tags.add("workload:" + name)
    if sizes.size and sizes[0] == 0:
        tags.add("empty_first")
    if sizes.size and sizes[-1] == 0:
        tags.add("empty_last")
    if (sizes[1:-1] == 0).any():
        tags.add("empty_middle")
    if (sizes == 1).any():
        tags.add("single_atom")
    if sizes.max(initial=0) >= 256:
        tags.add("graph_ge_256")
    if n % NODE_BLOCK:
        tags.add("n_not_multiple_of_128")
    if iters(n, NODE_BLOCK) > 1:
        tags.add("grid_stride")
    r32 = np.float32(r)
    if float(r32 * r32) != float(r32) * float(r32):
        tags.add("r2_rounds")
    for g in range(len(sizes)):
        q = pos[ptr[g]:ptr[g + 1]]
        if q.shape[0] > 1 and (q == q[0]).all():
            tags.add("coincident")
        d = q[None] - q[:, None]
        sq = d * d
        if (((sq[..., 0] + sq[..., 1]) + sq[..., 2]) == r32 * r32).any():
            tags.add("exact_r")
    if not loop and k != NO_CAP:                  # which side of the query the cap binds on
        if (binds & (deg == k + 1)).any():
            tags.add("cap_binds_before_self")
        if (binds & (deg == k)).any():
            tags.add("cap_binds_after_self")
    return tags


@pytest.mark.gpu
@pytest.mark.parametrize("name", [c[0] for c in RADIUS_CASES])
def test_radius_graph(name):
    pos, ptr, r, k, loop, fill = radius_inputs(name)
    n, g = pos.shape[0], len(ptr) - 1
    ref_ei, ref_deg = radius_reference(name)
    count = ref_ei.shape[1]
    P = Buf(n, 3, data=torch.from_numpy(pos))
    G = Buf(g + 1, dtype=torch.int32, data=torch.from_numpy(ptr))
    deg = Buf(n, dtype=torch.int32)
    count_call = lambda: _lib.call("hgb_radius_graph_count", P.ptr, G.ptr, n, g, r, k, int(loop), deg.ptr, stream())
    assert launches(count_call) == 1
    twice(name + " count", count_call, [deg])
    deg.check(name, "deg")
    rowptr = np.concatenate([[0], np.cumsum(ref_deg)]).astype(np.int32)
    R = Buf(n + 1, dtype=torch.int32, data=torch.from_numpy(rowptr))
    cap = capacity_of(fill, count)
    ei = Buf(2, cap, dtype=torch.int64)
    fill_call = lambda: _lib.call("hgb_radius_graph_fill", P.ptr, G.ptr, n, g, r, k, int(loop), R.ptr, cap, ei.ptr, stream())
    assert launches(fill_call) == 1
    twice(name + " fill", fill_call, [ei])
    written = torch.zeros(2, cap, dtype=torch.bool)
    written[:, :min(count, cap)] = True
    ei.check(name, "edge_index", mask=written)
    untouched = ei.view.cpu()[~written]           # Buf.check looks past the block only: the padded tail is checked here
    assert bool((untouched == SENTINEL).all()), "%s: %d fill slots past the count were written" % (
        name, int((untouched != SENTINEL).sum()))
    check_radius(name, name, deg.np().reshape(-1), ei.np(), cap)
    R.check(name, "rowptr (input)")
    if fill == "smaller":                         # a promised count that is too small trips the device guard
        ops.check_guard()
        radius.radius_graph(P.view, r, G.view.reshape(-1), g, loop, k, known_e=cap)
        with pytest.raises(RuntimeError, match="different edge count"):
            ops.check_guard()


@pytest.mark.gpu
def test_radius_graph_no_nodes_launches_nothing():
    G = Buf(2, dtype=torch.int32, data=torch.zeros(2, dtype=torch.int32))
    assert launches(lambda: _lib.call("hgb_radius_graph_count", None, G.ptr, 0, 1, 1.0, 5, 0, None, stream())) == 0
    assert launches(lambda: _lib.call("hgb_radius_graph_fill", None, G.ptr, 0, 1, 1.0, 5, 0, None, 0, None, stream())) == 0


# ================================================================================================================================
# 2. edge vectors, lengths, units and their backward;  3. the edge-length primitives
# ================================================================================================================================
GEOM_INPUTS = {"small": (50, 400), "zero_len": (60, 500), "grid_stride": (20_000, 600_000)}
EPS = [1e-9, 1.0]
GEOM_CASES = [(name, shifts, eps) for name in GEOM_INPUTS for shifts in (False, True) for eps in EPS]
LEN_CASES = [(name, shifts) for name in GEOM_INPUTS for shifts in (False, True)]
MASKS = list(range(8))                            # bit 0: vec / g_vec_in, bit 1: len / g_len, bit 2: unit / g_unit present


@functools.lru_cache(maxsize=None)
def geom_inputs(name, shifts):
    """pos [n, 3], row, col [e] int32 (unsorted), shifts [e, 3] or None, ggpos [n, 3], gd [e]; "zero_len" holds self-loops and
    edges between coincident atoms (zero shift on those)"""
    n, e = GEOM_INPUTS[name]
    rng = np.random.default_rng(7 + len(name) + 100 * shifts)
    pos = (rng.standard_normal((n, 3)) * 2).astype(np.float32)
    row = rng.integers(0, n, e).astype(np.int32)
    col = rng.integers(0, n, e).astype(np.int32)
    zero = np.zeros(e, bool)
    if name == "zero_len":
        pos[1] = pos[0]
        pos[5] = pos[4]
        row[:20], col[:20] = np.arange(20), np.arange(20)            # self-loops
        row[20:30], col[20:30] = 0, 1                                # coincident atoms, both directions
        row[30:40], col[30:40] = 5, 4
        zero[:40] = True
    sh = None
    if shifts:
        sh = (rng.standard_normal((e, 3)) * 0.1).astype(np.float32)
        sh[zero] = 0
    ggpos = rng.standard_normal((n, 3)).astype(np.float32)
    gd = rng.standard_normal(e).astype(np.float32)
    return pos, row, col, sh, ggpos, gd


def vec_f32(pos, row, col, sh, swap=False, shift_sign=1):
    """vec in the kernel's fp32 order (swap / shift_sign are mutations)"""
    if swap:
        row, col = col, row
    v = pos[col] - pos[row]
    if sh is not None:
        v = v + sh if shift_sign > 0 else v - sh
    return v


def emu_geom_fwd(pos, row, col, sh, eps, swap=False, shift_sign=1, unit_eps=True):
    """fp32 model of edge_geom_fwd (every operation rounded, no FMA)"""
    v = vec_f32(pos, row, col, sh, swap, shift_sign)
    ln = np.sqrt((v[:, 0] * v[:, 0] + v[:, 1] * v[:, 1]) + v[:, 2] * v[:, 2])
    with np.errstate(divide="ignore", invalid="ignore"):
        inv = np.float32(1) / ((ln + np.float32(eps)) if unit_eps else ln)
        unit = v * inv[:, None]
    return v, ln, unit


def check_geom_fwd(what, case, vec=None, ln=None, unit=None):
    name, shifts, eps = case
    pos, row, col, sh, _, _ = geom_inputs(name, shifts)
    v32 = vec_f32(pos, row, col, sh)
    v = v32.astype(np.float64)
    l = np.linalg.norm(v, axis=1)
    if vec is not None:
        same_f32(what + " vec", vec, v32)
    if ln is not None:
        bound(what + " len", np.asarray(ln).reshape(-1), l, DL * l)
    if unit is not None:
        L = l + f32(eps)
        with np.errstate(divide="ignore", invalid="ignore"):
            ref = np.where(L[:, None] > 0, v / L[:, None], 0.0)
            b = np.where(L[:, None] > 0, C_UNIT * np.abs(v) / L[:, None], 0.0)
        bound(what + " unit", unit, ref, b)


@functools.lru_cache(maxsize=None)
def geom_bwd_inputs(name, eps):
    """(vec, len) as the forward leaves them (len the correctly rounded norm), and the three incoming gradients"""
    pos, row, col, sh, _, _ = geom_inputs(name, True)
    vec = vec_f32(pos, row, col, sh)
    ln = np.linalg.norm(vec.astype(np.float64), axis=1).astype(np.float32)
    rng = np.random.default_rng(11)
    e = vec.shape[0]
    g_in = rng.standard_normal((e, 3)).astype(np.float32)
    g_len = rng.standard_normal(e).astype(np.float32)
    g_unit = rng.standard_normal((e, 3)).astype(np.float32)
    return vec, ln, g_in, g_len, g_unit


def grads_of(mask, g_in, g_len, g_unit):
    return (g_in if mask & 1 else None), (g_len if mask & 2 else None), (g_unit if mask & 4 else None)


def emu_geom_bwd(vec, ln, eps, g_in, g_len, g_unit, unit_eps=True):
    """fp32 model of edge_geom_bwd"""
    one = np.float32(1)
    with np.errstate(divide="ignore"):
        il = np.where(ln > 0, one / ln, np.float32(0)).astype(np.float32)
        iL = one / ((ln + np.float32(eps)) if unit_eps else ln)
    g = np.zeros_like(vec) if g_in is None else g_in.copy()
    radial = g_len * il if g_len is not None else np.zeros_like(ln)
    if g_unit is not None:
        g = g + g_unit * iL[:, None]
        dot = (g_unit[:, 0] * vec[:, 0] + g_unit[:, 1] * vec[:, 1]) + g_unit[:, 2] * vec[:, 2]
        with np.errstate(invalid="ignore"):
            radial = radial - dot * iL * iL * il
    return g + radial[:, None] * vec


def check_geom_bwd(what, name, eps, mask, got):
    vec32, ln32, *gs = geom_bwd_inputs(name, eps)
    g_in, g_len, g_unit = [None if x is None else x.astype(np.float64) for x in grads_of(mask, *gs)]
    v, l = vec32.astype(np.float64), ln32.astype(np.float64)
    il = np.divide(1.0, l, out=np.zeros_like(l), where=l > 0)
    L = l + f32(eps)
    ref = np.zeros_like(v)
    mag = np.zeros_like(v)
    if g_in is not None:
        ref += g_in
        mag += np.abs(g_in)
    if g_len is not None:
        ref += (g_len * il)[:, None] * v
        mag += np.abs(g_len * il)[:, None] * np.abs(v)
    if g_unit is not None:
        ref += g_unit / L[:, None] - ((g_unit * v).sum(1) * il / L ** 2)[:, None] * v
        mag += np.abs(g_unit) / L[:, None] + (np.abs(g_unit * v).sum(1) * il / L ** 2)[:, None] * np.abs(v)
    bound(what, got, ref, C_GEOM_BWD * mag)


def emu_len_bwd(pos, row, col, sh, gd):
    v = vec_f32(pos, row, col, sh)
    l = np.sqrt((v[:, 0] * v[:, 0] + v[:, 1] * v[:, 1]) + v[:, 2] * v[:, 2])
    with np.errstate(divide="ignore", invalid="ignore"):
        k = np.where(l > 0, gd / l, np.float32(0)).astype(np.float32)
    return k[:, None] * v


def emu_len_bwd2(pos, row, col, sh, gd, ggpos, curvature=True):
    v = vec_f32(pos, row, col, sh)
    l = np.sqrt((v[:, 0] * v[:, 0] + v[:, 1] * v[:, 1]) + v[:, 2] * v[:, 2])
    with np.errstate(divide="ignore"):
        il = np.where(l > 0, np.float32(1) / l, np.float32(0)).astype(np.float32)
    h = v * il[:, None]
    w = ggpos[col] - ggpos[row]
    hw = (h[:, 0] * w[:, 0] + h[:, 1] * w[:, 1]) + h[:, 2] * w[:, 2]
    k = gd * il
    q = k[:, None] * ((w - h * hw[:, None]) if curvature else w)
    return hw, q


def len_reference(name, shifts):
    pos, row, col, sh, ggpos, gd = geom_inputs(name, shifts)
    v = vec_f32(pos, row, col, sh).astype(np.float64)
    l = np.linalg.norm(v, axis=1)
    il = np.divide(1.0, l, out=np.zeros_like(l), where=l > 0)
    return v, l, il, (ggpos[col] - ggpos[row]).astype(np.float64), gd.astype(np.float64)


def check_len_bwd(what, case, gvec):
    v, l, il, _, gd = len_reference(*case)
    bound(what + " gvec", gvec, (gd * il)[:, None] * v, C_LEN_BWD * np.abs(gd * il)[:, None] * np.abs(v))


def check_len_bwd2(what, case, g_gd, q):
    v, l, il, w, gd = len_reference(*case)
    h = v * il[:, None]
    hw = (h * w).sum(1)
    S = np.abs(h * w).sum(1)
    bound(what + " g_gd", g_gd, hw, C_HW * S)
    k = np.abs(gd * il)[:, None]
    bound(what + " q", q, (gd * il)[:, None] * (w - h * hw[:, None]), k * (C_QW * np.abs(w) + C_QH * np.abs(h) * S[:, None]))
    zero = l == 0
    assert (np.asarray(g_gd)[zero] == 0).all() and (np.asarray(q)[zero] == 0).all(), what + ": g_gd, q not 0 at d = 0"


# ---- scatter -------------------------------------------------------------------------------------------------------------------
SCATTER_CASES = {"random": (300, 2000), "empty_nodes": (500, 300), "hub": (200, 3000), "grid_stride": (300_000, 900_000)}


def csr_of(idx, n):
    rowptr = np.concatenate([[0], np.cumsum(np.bincount(idx, minlength=n))]).astype(np.int32)
    return rowptr, np.argsort(idx, kind="stable").astype(np.int32)


@functools.lru_cache(maxsize=None)
def scatter_inputs(name):
    """gvec [e, 3], (col rowptr, perm), (row rowptr, perm), row, col: edges in random order"""
    n, e = SCATTER_CASES[name]
    rng = np.random.default_rng(len(name))
    hi = n // 2 if name == "empty_nodes" else n          # nodes [n/2, n) have no edges
    row, col = rng.integers(0, hi, e), rng.integers(0, hi, e)
    if name == "hub":                                    # node 7 receives 1500 edges, node 3 sends 1200
        col[rng.permutation(e)[:1500]] = 7
        row[rng.permutation(e)[:1200]] = 3
    gvec = rng.standard_normal((e, 3)).astype(np.float32)
    return gvec, csr_of(col, n), csr_of(row, n), row, col


def seq_sum_f32(m, rowptr, perm, drop=None):
    """fp32 sum of every segment, one edge after the other in CSR order (drop: a mutation leaves this edge out)"""
    lens = np.diff(rowptr)
    acc = np.zeros((len(lens),) + m.shape[1:], np.float32)
    for p in range(int(lens.max(initial=0))):
        rows = np.nonzero(lens > p)[0]
        e = perm[rowptr[rows] + p]
        if drop is not None:
            keep = e != drop
            rows, e = rows[keep], e[keep]
        acc[rows] = acc[rows] + m[e]
    return acc


def emu_scatter(gvec, ccsr, rcsr, drop=None):
    return seq_sum_f32(gvec, *ccsr, drop=drop) - seq_sum_f32(gvec, *rcsr)


def check_scatter(what, name, got):
    gvec, ccsr, rcsr, row, col = scatter_inputs(name)
    n = len(ccsr[0]) - 1
    same_f32(what, got, emu_scatter(gvec, ccsr, rcsr))
    g64 = gvec.astype(np.float64)
    ref, mag = np.zeros((n, 3)), np.zeros((n, 3))
    np.add.at(ref, col, g64)
    np.add.at(ref, row, -g64)
    np.add.at(mag, col, np.abs(g64))
    np.add.at(mag, row, np.abs(g64))
    L = np.maximum(np.diff(ccsr[0]), np.diff(rcsr[0])) + 1
    bound(what + " vs fp64", got, ref, np.array([gamma(x) for x in L])[:, None] * mag)


# ---- the tests -------------------------------------------------------------------------------------------------------------------
def upload(a, dtype=torch.float32):
    a = np.asarray(a)
    return Buf(a.shape[0], a.shape[1] if a.ndim > 1 else 1, dtype=dtype, data=torch.from_numpy(np.ascontiguousarray(a)))


def geom_bufs(name, shifts):
    pos, row, col, sh, ggpos, gd = geom_inputs(name, shifts)
    return (upload(pos), upload(row, torch.int32), upload(col, torch.int32), upload(sh) if sh is not None else None,
            upload(ggpos), upload(gd))


def ptr_of(b):
    return None if b is None else b.ptr


@pytest.mark.gpu
@pytest.mark.parametrize("name,shifts,eps", GEOM_CASES)
def test_edge_geom_fwd(name, shifts, eps):
    P, R, C, S, _, _ = geom_bufs(name, shifts)
    e = R.rows
    vec, ln, unit = Buf(e, 3), Buf(e), Buf(e, 3)
    call = lambda: _lib.call("hgb_edge_geom_fwd", P.ptr, R.ptr, C.ptr, ptr_of(S), e, eps, vec.ptr, ln.ptr, unit.ptr, stream())
    assert launches(call) == 1
    twice(name, call, [vec, ln, unit])
    for b, nm in ((vec, "vec"), (ln, "len"), (unit, "unit")):
        b.check(name, nm)
    check_geom_fwd(name, (name, shifts, eps), vec.np(), ln.np().reshape(-1), unit.np())


@pytest.mark.gpu
@pytest.mark.parametrize("mask", MASKS)
def test_edge_geom_fwd_null_outputs(mask):
    """a NULL output is never written; the others are the full-output values bit for bit"""
    case = ("zero_len", True, 1.0)
    P, R, C, S, _, _ = geom_bufs("zero_len", True)
    e = R.rows
    full = [Buf(e, 3), Buf(e), Buf(e, 3)]
    part = [Buf(e, 3), Buf(e), Buf(e, 3)]
    _lib.call("hgb_edge_geom_fwd", P.ptr, R.ptr, C.ptr, S.ptr, e, 1.0, *[b.ptr for b in full], stream())
    call = lambda: _lib.call("hgb_edge_geom_fwd", P.ptr, R.ptr, C.ptr, S.ptr, e, 1.0,
                             *[b.ptr if mask >> i & 1 else None for i, b in enumerate(part)], stream())
    assert launches(call) == 1
    for i, (f, p) in enumerate(zip(full, part)):
        p.check("mask %d" % mask, "output %d" % i, written=bool(mask >> i & 1))
        if mask >> i & 1:
            assert torch.equal(p.base.view(torch.int32), f.base.view(torch.int32))
    check_geom_fwd("mask %d" % mask, case, *[full[i].np().reshape(-1) if i == 1 else full[i].np() for i in range(3)])


@pytest.mark.gpu
@pytest.mark.parametrize("eps", EPS)
@pytest.mark.parametrize("mask", MASKS)
@pytest.mark.parametrize("name", list(GEOM_INPUTS))
def test_edge_geom_bwd(name, mask, eps):
    vec32, ln32, *gs = geom_bwd_inputs(name, eps)
    e = vec32.shape[0]
    V, Ln = upload(vec32), upload(ln32)
    G = [None if g is None else upload(g) for g in grads_of(mask, *gs)]
    out = Buf(e, 3)
    call = lambda: _lib.call("hgb_edge_geom_bwd", V.ptr, Ln.ptr, eps, *[ptr_of(g) for g in G], e, out.ptr, stream())
    assert launches(call) == 1
    twice(name, call, [out])
    out.check(name, "g_vec")
    check_geom_bwd("%s mask %d eps %g" % (name, mask, eps), name, eps, mask, out.np())


@pytest.mark.gpu
@pytest.mark.parametrize("name,shifts", LEN_CASES)
def test_edge_len_bwd_and_bwd2(name, shifts):
    P, R, C, S, GG, GD = geom_bufs(name, shifts)
    e = R.rows
    gvec, g_gd, q = Buf(e, 3), Buf(e), Buf(e, 3)
    call1 = lambda: _lib.call("hgb_edge_len_bwd", P.ptr, R.ptr, C.ptr, ptr_of(S), GD.ptr, e, gvec.ptr, stream())
    call2 = lambda: _lib.call("hgb_edge_len_bwd2", P.ptr, R.ptr, C.ptr, ptr_of(S), GD.ptr, GG.ptr, e, g_gd.ptr, q.ptr, stream())
    assert launches(call1) == 1 and launches(call2) == 1
    twice(name + " bwd", call1, [gvec])
    twice(name + " bwd2", call2, [g_gd, q])
    for b, nm in ((gvec, "gvec"), (g_gd, "g_gd"), (q, "q")):
        b.check(name, nm)
    check_len_bwd(name, (name, shifts), gvec.np())
    check_len_bwd2(name, (name, shifts), g_gd.np().reshape(-1), q.np())


@pytest.mark.gpu
@pytest.mark.parametrize("name", list(SCATTER_CASES))
def test_edge_vec_scatter(name):
    gvec, (crp, cpm), (rrp, rpm), _, _ = scatter_inputs(name)
    n = len(crp) - 1
    G, CR, CP, RR, RP = upload(gvec), *[upload(a, torch.int32) for a in (crp, cpm, rrp, rpm)]
    out = Buf(n, 3)
    call = lambda: _lib.call("hgb_edge_vec_scatter", G.ptr, CR.ptr, CP.ptr, RR.ptr, RP.ptr, n, out.ptr, stream())
    assert launches(call) == 1
    twice(name, call, [out])
    out.check(name, "g_pos")
    check_scatter(name, name, out.np())


# ================================================================================================================================
# 4. the autograd wrappers at workload shapes
# ================================================================================================================================
WRAP_WORKLOADS = [("md17_egnn", 16), ("lj_egnn", 8), ("qm9_painn", 32), ("oc20_mace", 2)]
WRAP_PATHS = ["edge_len", "edge_geom", "edge_geometry_any_order"]


@functools.lru_cache(maxsize=None)
def workload_graph(name, g):
    from oracle.workloads import add_edges_cpu
    b = add_edges_cpu(make_samples(name, g), name)
    return b.pos.float(), b.edge_index, b.edge_shifts.float()


def node_bound(t_abs, row, col, n, c_edge):
    """(C_GD + c_edge + gamma(L_i + 1)) sum over node i's edges of |t_e| (t: per-edge terms [e, 3])"""
    mag = np.zeros((n, 3))
    np.add.at(mag, col, t_abs)
    np.add.at(mag, row, t_abs)
    L = np.maximum(np.bincount(col, minlength=n), np.bincount(row, minlength=n)) + 1
    return ((C_GD + c_edge) * SLACK + np.array([gamma(x) for x in L]))[:, None] * mag


def rel_l2(a, b):
    a, b = np.asarray(a, np.float64), np.asarray(b, np.float64)
    return float(np.linalg.norm(a - b) / max(np.linalg.norm(b), 1e-300))


@pytest.mark.gpu
@pytest.mark.parametrize("path", WRAP_PATHS)
@pytest.mark.parametrize("name,g", WRAP_WORKLOADS)
def test_autograd_wrappers_at_workload_shapes(name, g, path):
    pos, ei, sh = workload_graph(name, g)
    n, e = pos.shape[0], ei.shape[1]
    rng = torch.Generator().manual_seed(e)
    coef, tgt = torch.randn(e, generator=rng), torch.randn(n, 3, generator=rng)
    a_unit = torch.randn(e, 3, generator=rng)
    eps = 1.0 if name in ("md17_egnn", "lj_egnn") else 1e-9
    plan = ops.EdgePlan(ei.cuda(), n)

    eref = ei.numpy()
    vec32 = vec_f32(pos.numpy(), eref[0], eref[1], sh.numpy())

    def energy(p, lib):
        """E = sum c d^2 (+ sum a . unit on the unit-producing paths)"""
        if not lib:
            # the oracle's vec, its value replaced by the exact fp32 vec (part 2) and its derivative kept
            vec, _ = edge_vectors_and_lengths(p, ei, sh.double())
            vec = vec - vec.detach() + torch.from_numpy(vec32).double()
            d = torch.linalg.norm(vec, dim=-1)
            unit = vec / (d[:, None] + f32(eps))
        elif path == "edge_len":
            d, unit = ops.EdgeLenFn.apply(p, sh.cuda(), plan), None
        elif path == "edge_geom":
            _, d, unit = ops.EdgeGeomFn.apply(p, sh.cuda(), plan, eps)
            d = d.reshape(-1)
        else:
            d, unit = stacks.edge_geometry(p, sh.cuda(), plan, eps, higher_order=True)
            d = d.reshape(-1)
        c = coef.to(d)
        en = (c * d * d).sum()
        if path != "edge_len":
            en = en + (a_unit.to(unit) * unit).sum()
        return en, d

    p64 = pos.double().requires_grad_(True)
    e64, d64 = energy(p64, False)
    f64, = torch.autograd.grad(e64, p64, create_graph=True)
    p32 = pos.cuda().requires_grad_(True)
    e32, d32 = energy(p32, True)
    f32_, = torch.autograd.grad(e32, p32, create_graph=path != "edge_geom")

    # lengths, per element
    bound(name + " len", d32.detach().cpu().numpy(), d64.detach().numpy(), DL * d64.detach().numpy())
    # forces, per element: the per-edge terms are 2 c d vhat (+ the unit terms)
    vec = vec32.astype(np.float64)
    d = np.linalg.norm(vec, axis=1)
    t = np.abs(2 * coef.double().numpy() * d)[:, None] * np.abs(vec / d[:, None])
    c_edge = C_LEN_BWD
    if path != "edge_len":
        L = d + f32(eps)
        a = a_unit.double().numpy()
        t = t + np.abs(a) / L[:, None] + (np.abs(a * vec).sum(1) / (L ** 2 * d))[:, None] * np.abs(vec)
        c_edge = C_GEOM_EDGE if path == "edge_geom" else C_ANY_ORDER
    bound(name + " forces", f32_.detach().cpu().numpy(), f64.detach().numpy(), node_bound(t, eref[0], eref[1], n, c_edge))
    if path == "edge_geom":                       # once-differentiable: no force loss through it
        return
    loss64 = ((f64 - tgt.double()) ** 2).sum() + e64
    g64, = torch.autograd.grad(loss64, p64)
    loss32 = ((f32_ - tgt.cuda()) ** 2).sum() + e32
    g32, = torch.autograd.grad(loss32, p32)
    err = rel_l2(g32.cpu().numpy(), g64.numpy())
    assert err < 4e-6, "%s %s: force-loss position gradient rel-L2 %.3g" % (name, path, err)


# ================================================================================================================================
# 5. edge-free batches
# ================================================================================================================================
@pytest.mark.gpu
def test_edge_free_entry_points_launch_nothing():
    """with e = 0 every edge array may be NULL: OK, and no kernel runs"""
    calls = {
        "hgb_edge_geom_fwd": (None, None, None, None, 0, 1e-9, None, None, None),
        "hgb_edge_geom_bwd": (None, None, 1.0, None, None, None, 0, None),
        "hgb_edge_len_bwd": (None, None, None, None, None, 0, None),
        "hgb_edge_len_bwd2": (None, None, None, None, None, None, 0, None, None),
        "hgb_mace_edge_embed_fwd": (None, None, None, None, 0, 2, 8, 5.0, 5.0, None, None),
        "hgb_mace_edge_embed_bwd": (None, None, None, None, None, None, 0, 2, 8, 5.0, 5.0, None),
    }
    for fn, args in calls.items():
        assert launches(lambda: _lib.call(fn, *args, stream())) == 0, fn


@pytest.mark.gpu
def test_edge_vec_scatter_without_edges_is_zero():
    n = 300
    zeros = Buf(n + 1, dtype=torch.int32, data=torch.zeros(n + 1, dtype=torch.int32))
    dummy_i, dummy_f = Buf(1, dtype=torch.int32), Buf(1, 3)                  # never read: every segment is empty
    out = Buf(n, 3)
    call = lambda: _lib.call("hgb_edge_vec_scatter", dummy_f.ptr, zeros.ptr, dummy_i.ptr, zeros.ptr, dummy_i.ptr, n, out.ptr,
                             stream())
    assert launches(call) == 1
    out.check("no edges", "g_pos")
    assert (out.np() == 0).all()


@pytest.mark.gpu
def test_autograd_wrappers_on_an_edge_free_plan():
    n = 7
    plan = ops.EdgePlan(torch.zeros(2, 0, dtype=torch.int64, device="cuda"), n)
    sh = torch.zeros(0, 3, device="cuda")
    pos = torch.randn(n, 3, device="cuda", requires_grad=True)
    zero = torch.zeros(n, 3, device="cuda")

    d = ops.EdgeLenFn.apply(pos, sh, plan)
    assert d.shape == (0,)
    f, = torch.autograd.grad(d.sum(), pos, create_graph=True)
    assert torch.equal(f, zero)
    g, = torch.autograd.grad((f * f).sum() + f.sum(), pos)        # through bwd2 and the scatter
    assert torch.equal(g, zero)
    g, = torch.autograd.grad(ops.EdgeLenFn.apply(pos, sh, plan).sum(), pos)     # first order, grad mode off inside
    assert torch.equal(g, zero)

    vec, ln, unit = ops.EdgeGeomFn.apply(pos, sh, plan, 1.0)
    assert vec.shape == (0, 3) and ln.shape == (0, 1) and unit.shape == (0, 3)
    g, = torch.autograd.grad(ln.sum() + unit.sum(), pos)
    assert torch.equal(g, zero)

    sph, rad = ops.MaceEdgeEmbedFn.apply(pos, sh, plan, 2, 8, 5.0, 5.0)
    assert sph.shape == (0, 9) and rad.shape == (0, 8)
    g, = torch.autograd.grad(sph.sum() + rad.sum(), pos)
    assert torch.equal(g, zero)


# ================================================================================================================================
# 6. no GPU: the case lists reach every form, the references agree with torch, and wrong kernels are caught
# ================================================================================================================================
def geom_tags():
    tags = set()
    for name, shifts, eps in GEOM_CASES:
        pos, row, col, sh, _, _ = geom_inputs(name, shifts)
        e = row.size
        tags |= {"fwd:shifts" if shifts else "fwd:no_shifts", "eps:%g" % eps}
        if (row == col).any():
            tags.add("zero_len:self_loop")
        if ((row != col) & (pos[row] == pos[col]).all(1)).any():
            tags.add("zero_len:coincident")
        if iters(e, EDGE_BLOCK) > 1:
            tags.add("edges:grid_stride")
        if (np.diff(col) < 0).any() and (np.diff(row) < 0).any():
            tags.add("edges:unsorted")
    tags |= {"fwd_null:%d" % m for m in MASKS}
    tags |= {"bwd_null:%d:eps%g" % (m, eps) for m in MASKS for eps in EPS}
    for name, shifts in LEN_CASES:
        v, l, _, _, _ = len_reference(name, shifts)
        tags.add("len:shifts" if shifts else "len:no_shifts")
        if (l == 0).any():
            tags.add("len:d0:shifts" if shifts else "len:d0:no_shifts")
        if iters(l.size, EDGE_BLOCK) > 1:
            tags.add("len:grid_stride")
    for name in SCATTER_CASES:
        gvec, ccsr, rcsr, row, col = scatter_inputs(name)
        n = len(ccsr[0]) - 1
        if ((np.diff(ccsr[0]) == 0) & (np.diff(rcsr[0]) == 0)).any():
            tags.add("scatter:node_without_edges")
        if np.diff(ccsr[0]).max() >= 1000:
            tags.add("scatter:hub")
        if (np.diff(col) < 0).any():
            tags.add("scatter:unsorted")
        if iters(n, NODE_BLOCK) > 1:
            tags.add("scatter:grid_stride")
    return tags


def test_cases_reach_every_form():
    tags = set()
    for c in RADIUS_CASES:
        tags |= {"radius:" + t for t in radius_tags(c[0])}
    tags |= geom_tags()
    need = {"radius:" + t for t in (
        "loop", "no_loop", "k1_binds", "k5_binds", "k128_binds", "no_cap", "cap_binds_before_self", "cap_binds_after_self", "empty_first",
        "empty_middle", "empty_last", "single_atom", "coincident", "exact_r", "r2_rounds", "graph_ge_256",
        "n_not_multiple_of_128", "grid_stride", "fill:exact", "fill:larger", "fill:smaller", "workload:qm9_painn",
        "workload:md17_egnn", "workload:ogb_pna", "workload:oc20_mace")}
    need |= {"fwd:shifts", "fwd:no_shifts", "eps:1e-09", "eps:1", "zero_len:self_loop", "zero_len:coincident",
             "edges:grid_stride", "edges:unsorted", "len:shifts", "len:no_shifts", "len:d0:shifts", "len:d0:no_shifts",
             "len:grid_stride", "scatter:node_without_edges", "scatter:hub", "scatter:unsorted", "scatter:grid_stride"}
    need |= {"fwd_null:%d" % m for m in MASKS} | {"bwd_null:%d:eps%g" % (m, eps) for m in MASKS for eps in EPS}
    missing = need - tags
    assert not missing, "case lists miss %s" % sorted(missing)
    # the restated dispatch at its edges
    assert iters(540_672, EDGE_BLOCK) == 1 and iters(540_673, EDGE_BLOCK) == 2
    assert iters(270_336, NODE_BLOCK) == 1 and iters(270_337, NODE_BLOCK) == 2


def test_radius_restatement_matches_the_oracle():
    for c in RADIUS_CASES:
        pos, ptr, r, k, loop, _ = radius_inputs(c[0])
        deg, ei = radius_restated(pos, ptr, r, k, loop)
        check_radius(c[0], c[0], deg, ei, ei.shape[1])


def test_references_match_torch_autograd():
    """the fp64 references of the backward kernels, zero-length edges included, against torch autograd of linalg.norm"""
    for eps in EPS:
        for mask in MASKS:
            vec32, ln32, *gs = geom_bwd_inputs("zero_len", eps)
            v = torch.from_numpy(vec32.astype(np.float64)).requires_grad_(True)
            ln = torch.linalg.norm(v, dim=1)
            out = [v, ln, v / (ln[:, None] + f32(eps))]
            en = sum((o * torch.from_numpy(g.astype(np.float64))).sum() for o, g in zip(out, grads_of(mask, *gs)) if g is not None)
            if not torch.is_tensor(en):
                continue
            g, = torch.autograd.grad(en, v)
            check_geom_bwd("torch eps %g mask %d" % (eps, mask), "zero_len", eps, mask, g.numpy())
    for shifts in (False, True):
        pos, row, col, sh, ggpos, gd = geom_inputs("zero_len", shifts)
        gdt = torch.from_numpy(gd.astype(np.float64)).requires_grad_(True)
        vec = torch.from_numpy(vec_f32(pos, row, col, sh).astype(np.float64)).requires_grad_(True)
        gv, = torch.autograd.grad(torch.linalg.norm(vec, dim=1), vec, gdt, create_graph=True)
        check_len_bwd("torch", ("zero_len", shifts), gv.detach().numpy())
        v, l, il, w, gd64 = len_reference("zero_len", shifts)
        q, g_gd = torch.autograd.grad((gv * torch.from_numpy(w)).sum(), [vec, gdt])
        h = v * il[:, None]
        hw = (h * w).sum(1)
        check_bound("torch g_gd", g_gd.numpy(), hw, 1e-12 * (1 + np.abs(hw)))
        assert (g_gd.numpy()[l == 0] == 0).all()
        # torch's q is NaN (0 * inf) at d = 0; elsewhere it is the reference the kernel is held to
        ref_q = (gd64 * il)[:, None] * (w - h * hw[:, None])
        check_bound("torch q", q.numpy()[l > 0], ref_q[l > 0], 1e-12 * (1 + np.abs(ref_q[l > 0])))


def mutation_runs():
    """{mutation: list of thunks, each comparing one case of a wrong fp32 restatement; None: the faithful restatements}"""
    runs = {m: [] for m in (None, "row_col_swapped", "shift_sign_flipped", "unit_without_eps", "bwd2_no_curvature",
                            "radius_le", "cap_without_plus_one", "scatter_drops_an_edge")}
    for case in GEOM_CASES:
        name, shifts, eps = case
        args = geom_inputs(name, shifts)[:4]
        for m, kw in ((None, {}), ("row_col_swapped", dict(swap=True)), ("shift_sign_flipped", dict(shift_sign=-1)),
                      ("unit_without_eps", dict(unit_eps=False))):
            runs[m].append(lambda case=case, args=args, kw=kw: check_geom_fwd(str(case), case, *emu_geom_fwd(*args, case[2], **kw)))
    for name in GEOM_INPUTS:
        for eps in EPS:
            for mask in MASKS:
                vec, ln, *gs = geom_bwd_inputs(name, eps)
                for m, kw in ((None, {}), ("unit_without_eps", dict(unit_eps=False))):
                    runs[m].append(lambda name=name, eps=eps, mask=mask, kw=kw, vec=vec, ln=ln, gs=gs: check_geom_bwd(
                        name, name, eps, mask, emu_geom_bwd(vec, ln, eps, *grads_of(mask, *gs), **kw)))
    for case in LEN_CASES:
        pos, row, col, sh, ggpos, gd = geom_inputs(*case)
        runs[None].append(lambda case=case, a=(pos, row, col, sh, gd): check_len_bwd(str(case), case, emu_len_bwd(*a)))
        for m, kw in ((None, {}), ("bwd2_no_curvature", dict(curvature=False)), ("row_col_swapped", {})):
            a = (pos, col, row) if m == "row_col_swapped" else (pos, row, col)
            runs[m].append(lambda case=case, a=a, kw=kw, sh=sh, gd=gd, gg=ggpos: check_len_bwd2(
                str(case), case, *emu_len_bwd2(*a, sh, gd, gg, **kw)))
    for c in RADIUS_CASES:
        pos, ptr, r, k, loop, _ = radius_inputs(c[0])
        for m, kw in (("radius_le", dict(strict=False)), ("cap_without_plus_one", dict(plus_one=False))):
            runs[m].append(lambda c=c, a=(pos, ptr, r, k, loop), kw=kw: check_radius(
                c[0], c[0], *radius_restated(*a, **kw), 2 ** 62))
    for name in SCATTER_CASES:
        gvec, ccsr, rcsr, _, _ = scatter_inputs(name)
        runs[None].append(lambda name=name: check_scatter(name, name, emu_scatter(*scatter_inputs(name)[:3])))
        runs["scatter_drops_an_edge"].append(lambda name=name, a=(gvec, ccsr, rcsr): check_scatter(
            name, name, emu_scatter(*a, drop=int(ccsr[1][-1]))))
    return runs


def test_mutations_are_caught():
    runs = mutation_runs()
    for thunk in runs.pop(None):                  # the faithful fp32 restatements pass every comparison
        thunk()
    for m, thunks in runs.items():
        caught = False
        for thunk in thunks:
            try:
                thunk()
            except (pytest.fail.Exception, AssertionError):
                caught = True
                break
        assert caught, "mutation %s passes every comparison" % m
