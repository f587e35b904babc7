"""Kernel-level tests of the tensor-core Linear (csrc/hgb_tc.cu: hgb_tc_linear, hgb_tc_linear_graph_add, hgb_tc_wgrad and its
reduce), the neighbour-sum Linear of SAGE / MFC (csrc/hgb_nbr.cu: hgb_nbr_tiles, hgb_nbr_linear_fwd, hgb_nbr_linear_bwd_data) and
FiLM (csrc/hgb_cond.cu: hgb_film_fwd, hgb_film_bwd and its finish kernel), each against fp64.

The C ABI is called directly through tests/kernel_harness.py.  Every operand is the leading block of a NaN-filled buffer (SENTINEL
for integers) with guard rows after it; strided operands sit in wider rows (lda > k, ldw > k forward and transposed, lddz, ldx,
lddw > k, ldg > n, ldst > 2c).  After each call every element in range is written and every other element keeps its fill bits;
the call runs twice with the same bits; it launches the kernels the restated host rule predicts; a refused shape launches nothing.

1. Host rules, restated (`tc_plan`, `wgrad_plan`, `nbr_plan`, `nbr_tiles`, `film_plan`).  `test_cases_reach_every_instantiation`
   (no GPU) asserts that the case lists below reach every kernel instantiation and every path the issue of each kernel names.

2. Exact answers.  Operands are dyadic, so every product and every partial sum is exact in fp32 whatever the order, the FMA
   contraction or the tensor cores' internal alignment: the kernel must equal fp64 bit for bit.
   * TF32 mode: values i / 8 with |i| <= 7 (3 significant bits; the tensor cores' truncation to TF32 loses nothing).
   * 3xTF32 mode: every operand is s + t with s in {+-1, +-2} and t in {0, +-2^-12}, so the splitters' RNA rounding gives hi = s and
     lo = t exactly, on both sides of the product.  The reference is fp64 of the split's own three products ah bh + ah bl + al bh
     (lo lo is dropped by design), so a missing or doubled product, a hi / lo mix-up, a misplaced column block, a wrong graph row in
     gadd or a wrong row in the nbr scatter all fail.  The weight gradient sums over rows, so it takes s in {+-1} and, above 4000
     rows, one live row per 32-row chunk (every chunk still contributes).
   * The neighbour sum: hx must equal the fp32 sequential sum in by-target CSR order followed by the root row, and in mean mode that
     sum followed by one fp32 division by max(deg, 1).  In TF32 sum mode the output is exact too.
   * FiLM: dt must equal the fp32 restatement in the kernel's order (rows within a chunk, then the tail and the heads in chunk order).
   `exact_quanta` asserts, on the actual operands of every case, that each term is a multiple of the construction's quantum and that
   the sum of the magnitudes of the terms of every output stays below 2^24 quanta.

3. Random operands: per-element bounds (u = 2^-24, gamma(L) = L u / (1 - L u)).
   * TF32 mode: gamma(K + 2) (sum |a b| + |c|) + TF32_OPERAND sum |a b| against fp64 of the TF32-rounded operands (kernel_harness).
   * 3xTF32 mode: |a - ah - al| <= 2^-22 |a|, so the split's three products are within SPLIT_OPERAND = 3 2^-22 (1 + 2^-9) |a b| of
     a b.  Round-to-nearest is not documented for the tensor cores' fp32 accumulation, so each of its additions is allowed 2u; the
     CUDA-core additions of the epilogue (bias, addend) and of the reductions u each.  A chain of T tensor-core and C CUDA-core
     additions is held to gamma(2 T + C) ((1 + 2^-9) sum |a b| + |c|) + SPLIT_OPERAND sum |a b|.
   * Epilogues: Lip(act) times the pre-activation bound plus act_eval_err; gsrc multiplies by act'(g) with grad_from_err.
   * Weight gradient: the chain is the rows per CTA between folds (3xTF32: 8 chunks), the folds, and the reduce (8 walkers over
     nparts / 8, then 8 more), plus one for accumulate.
   * nbr: the neighbour sum's gamma(deg) sum |x| enters as an operand error (divided by deg in mean mode).
   * FiLM: tanhf is within 2 ulp; ds sums over the graph's rows and chunk partials.
   On top of the worst-case bounds, the rel-L2 witness of test_gpu_dense_kernels.py: ||err|| <= 3 eps sqrt(L) ||M|| for the
   accumulation (eps = u, 2u in 3xTF32 mode) plus 3 eps_op ||sqrt(sum (a b)^2)|| for the operand conversion; it catches a systematic
   error of order 2^-13 per product that the worst-case bound at K = 128 would let through.

4. No GPU: the references against fp64 autograd, the exactness of the constructions, and deliberately wrong restatements that
   must each fail a comparison.

The module fixture prints the worst |error| / bound per section and the check that reached it.  Measured on an NVIDIA H100 80GB
HBM3 at a 700 W power limit (both read in the same run), where the whole file ran in 50 s:
  tc_linear: exact 0.9996, tf32 0.83; L2 witness 0.016 (exact), 0.15 (tf32)
  tc_wgrad:  exact 0.0040, tf32 0.056; L2 witness 0.0028 (exact), 0.15 (tf32)
  nbr:       exact 0.026, tf32 0.71; L2 witness 0.019 (exact), 0.17 (tf32)
  film:      0.90 (dh)
The two tc_linear maxima are the same kind of element: y = sigmoid(z) + addend with a dyadic z, which is exact, so the whole bound
is act_eval_err plus u |y| for the final fp32 addition.  With sigmoid(z) near 2^-30 and addend = 2^-6, the sum falls on the
half-ulp point of 2^-6, so that one rounding uses its worst case u |y| almost in full.  The FiLM maximum is dh = dy (1 + tanhf s),
where tanhf's 2 ulp and the two roundings make up the whole bound.
"""
import numpy as np
import pytest
import torch

from hydragnn_b200 import _lib
from kernel_harness import (ACT, DERIV, LIP, LIP1, LRELU_P, NUM_SMS, TF32_OPERAND, U, Buf, act64, act_eval_err, cdiv,
                            check_bound, gamma, grad_from, grad_from_err, launches, same_f32, stream, twice, ws_buf)
from oracle.tf32 import _round_tf32

SMEM_MAX = 227 * 1024
TILE_M = 64
A_STAGE = SUB_BYTES = TILE_M * 128
RELU_SELECT = 101
SPLIT_OPERAND = 3 * 2.0 ** -22 * (1 + 2.0 ** -9)
SPLIT_MAG = 1 + 2.0 ** -9            # sum |ah bh| + |ah bl| + |al bh| <= SPLIT_MAG |a b|
EXACT_Q = {"tf32": 2.0 ** -6, "exact": 2.0 ** -12}
RATIOS = {}                          # section -> (worst |err| / bound, the check that reached it)


def _note(section, ratio, what=""):
    if float(ratio) >= RATIOS.get(section, (0.0, ""))[0]:
        RATIOS[section] = (float(ratio), what)


@pytest.fixture(scope="module", autouse=True)
def _report_ratios():
    yield
    if RATIOS:
        print("\nworst |error| / bound: " + "; ".join("%s %.4g (%s)" % (k, r, w) for k, (r, w) in sorted(RATIOS.items())))


def bounded(section, what, got, ref, bnd):
    """check_bound with non-finite values failing outright; the worst ratio is noted"""
    got = np.asarray(got, np.float64)
    ref, bnd = np.asarray(ref, np.float64), np.broadcast_to(np.asarray(bnd, np.float64), got.shape)
    if not np.isfinite(got).all():
        pytest.fail("%s: %d non-finite entries" % (what, int((~np.isfinite(got)).sum())))
    err = np.abs(got - ref)
    if err.size:
        ratio = np.where(bnd > 0, err / np.maximum(bnd, 1e-300), np.where(err > 2.0 ** -126, np.inf, 0.0))
        i = int(np.argmax(ratio))
        _note(section, ratio.flat[i], "%s; |err| %.3g, bound %.3g, ref %.6g" % (what, err.flat[i], bnd.flat[i], ref.flat[i]))
    check_bound(what, got, ref, bnd)


def witness(section, what, got, ref, l2):
    err = float(np.linalg.norm(np.asarray(got, np.float64) - np.asarray(ref, np.float64)))
    _note(section + " (L2)", err / max(l2, 1e-300), what)
    assert err <= l2, "%s: L2 error %.3g exceeds the random-walk witness %.3g" % (what, err, l2)


def exact_quanta(what, mag, quantum):
    """every output's terms (sum of magnitudes `mag`, each a multiple of `quantum`) are exact in fp32"""
    worst = float(np.max(np.asarray(mag, np.float64))) / quantum if np.size(mag) else 0.0
    assert worst < 2.0 ** 24, "%s: %.3g quanta leave fp32's exact range" % (what, worst)


def is_multiple(t, q):
    t = np.asarray(t, np.float64) / q
    return bool((t == np.round(t)).all())


def d64(t):
    return t.detach().double().cpu()


# ================================================================================================================================
# the 3xTF32 split, restated: tf32_rna(x) = (bits + 0x1000) & ~0x1fff, hi = rna(x), lo = rna(x - hi)
# ================================================================================================================================
def split(x, trunc=False):
    x = x.float().contiguous()
    r = (lambda t: (t.view(torch.int32) & ~0x1FFF).view(torch.float32)) if trunc else _round_tf32
    h = r(x)
    return h, r(x - h)


def split_products(a, b, drop=None, trunc=False):
    """fp64 of ah bh^T + ah bl^T + al bh^T: the three products the split mode issues (drop: leave one out)"""
    ah, al = [t.double() for t in split(a, trunc)]
    bh, bl = [t.double() for t in split(b, trunc)]
    terms = {"hh": ah @ bh.t(), "hl": ah @ bl.t(), "lh": al @ bh.t()}
    return sum(v for k, v in terms.items() if k != drop)


def dyadic(g, shape, mode, single=False):
    """TF32: i / 8, |i| <= 7; 3xTF32: s + t, s in {+-1, +-2} ({+-1}: single), t in {0, +-2^-12}"""
    if mode == "tf32":
        return torch.randint(-7, 8, shape, generator=g).float() / 8
    s = torch.randint(1, 2 if single else 3, shape, generator=g).float() * (torch.randint(0, 2, shape, generator=g).float() * 2 - 1)
    return s + torch.randint(-1, 2, shape, generator=g).float() * 2.0 ** -12


def dyadic_small(g, shape, mode):
    """bias / addend / gadd values on the construction's quantum"""
    return torch.randint(-64, 65, shape, generator=g).float() * EXACT_Q[mode] * (16 if mode == "exact" else 1)


def tc_ref(a, b, c, mode, lt, lc):
    """fp64 value, per-element bound and L2 witness of a @ b^T + c on the tensor cores: lt tensor-core terms, lc CUDA-core additions"""
    c = torch.zeros(a.shape[0], b.shape[0], dtype=torch.float64) if c is None else c.double()
    if mode == "tf32":
        ta, tb = _round_tf32(a.float()).double(), _round_tf32(b.float()).double()
        mag = ta.abs() @ tb.abs().t()
        bnd = gamma(lt + lc) * (mag + c.abs()) + TF32_OPERAND * mag
        l2 = 3 * U * np.sqrt(lt + lc) * float((mag + c.abs()).norm()) + 3 * TF32_OPERAND * float(((ta * ta) @ (tb * tb).t()).sqrt().norm())
        return ta @ tb.t() + c, bnd, l2
    a, b = a.double(), b.double()
    mag = a.abs() @ b.abs().t()
    bnd = gamma(2 * 3 * lt + lc) * (SPLIT_MAG * mag + c.abs()) + SPLIT_OPERAND * mag
    l2 = 6 * U * np.sqrt(3 * lt + lc) * float((mag + c.abs()).norm()) + 3 * SPLIT_OPERAND * float(((a * a) @ (b * b).t()).sqrt().norm())
    return a @ b.t() + c, bnd, l2


# ================================================================================================================================
# 1. host rules, restated
# ================================================================================================================================
def tc_plan(m, n_out, k_red, exact, act=0, z=False, gsrc=False, gact=0, ga=False, addend=False):
    """tc_linear_pieces / tc_linear_piece: one kernel launch per (column piece, reduction piece)"""
    kc_max = min(k_red, 256)
    nc_max = min((64 if exact else 160) * 1024 // (4 * kc_max) // 32 * 32, 256)
    z_deriv = not gsrc and gact == DERIV
    pieces = []
    for c0 in range(0, n_out, nc_max):
        nc = min(n_out - c0, nc_max)
        for k0 in range(0, k_red, 256):
            kc = min(k_red - k0, 256)
            dup = 2 if exact else 1
            b_bytes = (kc // 32 * nc * 128 + 1023) & ~1023
            for slots in (4, 2):
                fixed = 1024 + dup * b_bytes + 2 * slots * SUB_BYTES + nc * 4 + 64
                stages = (SMEM_MAX - fixed) // (dup * A_STAGE + 24) if fixed < SMEM_MAX else 0
                stages = min(stages, 8) & ~1
                if stages >= 4:
                    break
            assert stages >= 4
            kind = {0: "NONE", 1: "RELU", 2: "SILU_ZD" if z and z_deriv else "SILU", 3: "TANH"}.get(act, "OTHER")
            pga = ga and k0 == 0
            operands = pga or gsrc or addend or k0 > 0
            nci = nc // 32
            pieces.append(dict(c0=c0, nc=nc, k0=k0, kc=kc, NC=nci, split=bool(exact), ga=pga, slots=slots, stages=stages, kind=kind,
                               timing=("early" if nci < 8 else "late") if operands else None, tiles=cdiv(m, TILE_M),
                               grid=min(cdiv(m, TILE_M), NUM_SMS), nc_max=nc_max))
    return pieces


def wgrad_plan(m, n, k, exact):
    q = k // 32
    raw = (min(n, 128) // 32 + q) * 32 * 128
    tb = (128 + k + 16) * 128 * (2 if exact else 1)
    budget = SMEM_MAX - 1024
    tbufs = 3
    while tbufs > 1 and tbufs * (tb + 16) + 2 * (raw + 16) > budget:
        tbufs -= 1
    stages = max(budget - tbufs * (tb + 16), 0) // (raw + 16)
    total = cdiv(m, 32)
    gy = cdiv(n, 128)
    gx = min(total, NUM_SMS // gy)
    cpc = cdiv(total, gx)
    gx = cdiv(total, cpc)
    return dict(Q=q, split=bool(exact), tbufs=tbufs, stages=stages, gx=gx, gy=gy, cpc=cpc, flush=8 if exact else 0,
                folds=cdiv(cpc, 8) if exact else 1, last_chunks=total - (gx - 1) * cpc, last_rows=m - 32 * (total - 1),
                reduce_grid=cdiv(n * (k + 1), 32), launches=2)


def r32(v):
    return (v + 31) // 32 * 32


def nbr_plan(direction, n, k, n_out, groups, exact):
    ka, npad = (2 * r32(k), r32(n_out)) if direction == "fwd" else (r32(n_out), 2 * r32(k))
    dup = 2 if exact else 1
    nbuf = 2 if 1024 + dup * (ka * 64 * 4 + 2 * npad * 128) + 1024 <= SMEM_MAX else 1
    return dict(NC=npad // 32, split=bool(exact), nbuf=nbuf, ka=ka, npad=npad, grid=cdiv(n, 64) + groups, launches=1 if n else 0)


def nbr_tiles(grp_ptr, groups, n):
    """hgb_nbr_tiles: (group, first row) per 64-row tile of each group, (-1, 0) for the surplus entries"""
    start, acc = [], 0
    for q in range(groups):
        start.append(acc)
        acc += cdiv(int(grp_ptr[q + 1] - grp_ptr[q]), 64)
    out = []
    for t in range(cdiv(n, 64) + groups):
        if t < acc:
            q = int(np.searchsorted(start, t, side="right")) - 1
            out.append((q, int(grp_ptr[q]) + (t - start[q]) * 64))
        else:
            out.append((-1, 0))
    return np.array(out, np.int32)


def film_threads(c):
    return 128 if c >= 128 else r32(c)


def film_finish_graphs(gptr):
    """graphs the finish kernel writes: those spanning chunks, and the empty ones"""
    return [g for g in range(len(gptr) - 1) if not (gptr[g + 1] > gptr[g] and gptr[g] // 64 == (gptr[g + 1] - 1) // 64)]


def film_launches(n, dh, dst):
    return (1 if n > 0 and (dh or dst) else 0) + (1 if dst else 0)


def graph_of(gptr, ng, rows, mut=False):
    """lin_graph_of: the last g < ng with gptr[g] <= row (mut: the off-by-one gptr[g] < row)"""
    return np.searchsorted(np.asarray(gptr[1:ng]), rows, side="left" if mut else "right")


# ================================================================================================================================
# the cases
# ================================================================================================================================
MODES = ("tf32", "exact")
# tc_linear: (mode, m, n_out, k_red, options); options: act, z, addend, gsrc (gact), trans_b, lda / ldw padding, ga (graph layout)
TC_CASES = []
for _mode in MODES:
    for _nc in range(1, 9):
        TC_CASES.append((_mode, 200, 32 * _nc, 64, dict(act="silu", z=True)))
        TC_CASES.append((_mode, 200, 32 * _nc, 64, dict(ga="edges", ldg=32 * _nc + 4)))
    TC_CASES += [
        (_mode, 1000, 96, 160, dict(act="relu", z=True, lda=4, ldw=8)),
        (_mode, 1000, 96, 96, dict(act="tanh", z=True)),
        (_mode, 777, 128, 64, dict(act="silu", z=True, gact=DERIV)),                # SILU_ZD: z = silu'(pre)
        (_mode, 500, 64, 64, dict(act="sigmoid", z=True, addend=True)),
        (_mode, 500, 64, 64, dict(act="lrelu", z=True)),
        (_mode, 500, 64, 64, dict(act="elu")),
        (_mode, 500, 64, 64, dict(act="selu", z=True)),
        (_mode, 129, 96, 128, dict(act="silu", z=True)),                            # 3 tiles: one per CTA
        (_mode, 191, 96, 128, dict(trans_b=True, addend=True, gsrc="silu", ldw=4)),
        (_mode, 64 * 264 + 1, 96, 128, dict(act="silu", z=True)),                   # 265 tiles on 132 CTAs
        (_mode, 64 * 264 + 63, 96, 128, dict(trans_b=True, addend=True, gsrc="tanh")),
        (_mode, 700, 64, 320, dict(trans_b=True, addend=True, lda=4, ldw=12)),      # reduction pieces 256 + 64 chained through y
        (_mode, 300, 256, 512, dict(trans_b=True)),                                 # NC = 8 late operands, 2 reduction pieces
        (_mode, 300, 256, 64, dict(addend=True, gsrc="deriv")),
        (_mode, 300, 256, 64, dict(trans_b=True, gsrc="relu_select")),
        (_mode, 400, 256, 64, dict(ga="edges", ldg=260)),
        (_mode, 1000, 96, 160, dict(trans_b=True, gsrc="relu")),
        (_mode, 1000, 96, 160, dict(trans_b=True, gsrc="sigmoid")),
        (_mode, 1000, 96, 160, dict(trans_b=True, addend=True, gsrc="elu")),
        (_mode, 16897, 64, 64, dict(ga="many", ldg=68)),
        (_mode, 300, 64, 64, dict(ga="one", ldg=64)),
    ]
TC_CASES += [("tf32", 1500, 224, 256, dict(act="silu", z=True)),                    # column pieces 160 + 64, slots 2
             ("exact", 1500, 480, 64, dict(act="silu", z=True)),                    # column pieces 256 + 224
             ("exact", 1200, 64, 256, dict(act="silu", z=True)),                    # 64 KB of weights per copy: slots 2
             ("exact", 1200, 224, 128, dict(ga="edges", ldg=228))]                  # column pieces 128 + 96 of a graph-add Linear
GACT = {"silu": ACT["silu"], "tanh": ACT["tanh"], "relu": ACT["relu"], "sigmoid": ACT["sigmoid"], "elu": ACT["elu"],
        "deriv": DERIV, "relu_select": RELU_SELECT}
EXACT_GACT = ("deriv", "relu_select", "relu")        # gradients that keep a dyadic result exact


def tc_id(c):
    mode, m, n, k, o = c
    return "%s-m%d-n%d-k%d-%s" % (mode, m, n, k, "-".join("%s=%s" % kv for kv in sorted(o.items())) or "plain")


def ga_sizes(layout, m, seed):
    """graph sizes: one graph; empty graphs first and last with boundaries at rows 63 / 64 of a tile and a last row of its own;
    many random graphs with empty ones among them"""
    if layout == "one":
        return [m]
    if layout == "edges":
        return [0, 0, 63, 1, 0, m - 65 - (m > 130) * 64, 0] + ([64] if m > 130 else []) + [1, 0, 0]
    g = np.random.default_rng(seed)
    sizes = []
    while sum(sizes) < m:
        sizes.append(int(g.integers(0, 90)) if g.random() > 0.1 else 0)
    sizes[-1] -= sum(sizes) - m
    return [0] + sizes + [0]


def tc_plan_of(case):
    mode, m, n, k, o = case
    return tc_plan(m, n, k, mode == "exact", ACT.get(o.get("act", "none"), 0), o.get("z", False), "gsrc" in o, o.get("gact", 0)
                   if "gsrc" not in o else GACT[o["gsrc"]], "ga" in o, o.get("addend", False))


# wgrad: (mode, m, n_out, k_out, options); every Q, the ring depths and tails of the pipeline, strides and accumulate
def m_for(chunks_per_cta, ctas, tail=0, last=7):
    """rows giving `ctas` CTAs of `chunks_per_cta` chunks, the last CTA short by `tail` chunks and its last chunk `last` rows long"""
    return 32 * (chunks_per_cta * ctas - tail - 1) + last


WG_CASES = [(mode, 3001, 192 if q <= 3 else 128, 32 * q, {}) for mode in MODES for q in range(1, 8)] + [
    ("tf32", m_for(1, 100), 64, 64, {}),
    ("tf32", m_for(2, NUM_SMS, tail=1), 64, 64, dict(accumulate=True)),
    ("tf32", m_for(24, NUM_SMS, tail=5), 128, 64, {}),
    ("tf32", m_for(13, NUM_SMS), 96, 32, dict(lddz=8, ldx=4)),
    ("tf32", m_for(7, NUM_SMS // 2, tail=4, last=1), 160, 96, dict(lddw=4)),
    ("tf32", m_for(5, NUM_SMS, tail=2, last=31), 128, 224, dict(nobias=True)),
    ("exact", m_for(3, NUM_SMS, tail=2), 64, 64, {}),
    ("exact", m_for(17, NUM_SMS, tail=9), 128, 96, dict(accumulate=True)),
    ("exact", m_for(9, NUM_SMS, last=1), 128, 160, dict(ldx=8, lddw=4)),
    ("exact", m_for(2, NUM_SMS, last=31), 96, 128, {}),
    ("exact", m_for(20, NUM_SMS, tail=3), 128, 224, dict(nobias=True)),
    ("exact", m_for(1, 40), 64, 192, {}),
    ("exact", m_for(11, 66, tail=10), 160, 64, dict(lddz=4, accumulate=True)),
]


def wg_id(c):
    mode, m, n, k, o = c
    return "%s-m%d-n%d-k%d-%s" % (mode, m, n, k, "-".join("%s=%s" % kv for kv in sorted(o.items())) or "plain")


# nbr: (mode, direction, mean, groups, k, n_out); groups = 1 runs the identity order, 7 a degree order
NBR_CASES = ([("tf32", "fwd", False, 7, 8, n) for n in (1, 40, 96, 100, 150, 192, 200, 256)]
             + [("exact", "fwd", False, 7, 24, n) for n in (32, 64, 65, 128, 129, 192, 224, 256)]
             + [("exact", "fwd", False, 7, 128, 250), ("tf32", "fwd", False, 1, 128, 256)]
             + [(mode, "fwd", True, g, 33, 64) for mode in MODES for g in (1, 7)]
             + [(mode, "fwd", False, 1, 55, 100) for mode in MODES]
             + [(mode, "bwd", mean, g, k, 70) for mode in MODES for mean in (False, True) for g in (1, 7) for k in (8, 40, 70, 128)]
             + [("exact", "bwd", False, 7, 128, 256)])
NBR_SIZES = [70, 64, 0, 130, 1, 0, 135]      # rows per degree group 0..6 (group 6: in-degree >= 6): empty groups, one of 64 rows


def nbr_id(c):
    return "%s-%s-%s-g%d-k%d-n%d" % (c[0], c[1], "mean" if c[2] else "sum", c[3], c[4], c[5])


FILM_LAYOUTS = {"one": [150], "mixed": [0, 5, 59, 0, 200, 64, 100, 3, 0]}    # see test_cases_reach_every_instantiation
FILM_C = (1, 33, 128, 200)


def test_cases_reach_every_instantiation():
    pieces = [p for c in TC_CASES for p in tc_plan_of(c)]
    assert {(p["NC"], p["split"], p["ga"]) for p in pieces} == {(nc, s, ga) for nc in range(1, 9) for s in (False, True)
                                                                for ga in (False, True)}
    assert {p["kind"] for p in pieces} == {"NONE", "RELU", "SILU", "SILU_ZD", "TANH", "OTHER"}
    assert {p["slots"] for p in pieces} == {2, 4} and {p["timing"] for p in pieces} == {"early", "late", None}
    assert any(c[3] > 256 for c in TC_CASES)                                             # reduction pieces
    assert any(len({p["c0"] for p in tc_plan_of(c)}) > 1 for c in TC_CASES)              # column split
    assert any(cdiv(c[1], 64) <= NUM_SMS for c in TC_CASES) and any(cdiv(c[1], 64) > 2 * NUM_SMS for c in TC_CASES)
    assert {(c[0], c[4].get("ga")) for c in TC_CASES if "ga" in c[4]} >= {(md, ly) for md in MODES for ly in ("one", "edges", "many")}
    plans = [wgrad_plan(m, n, k, mode == "exact") for mode, m, n, k, _ in WG_CASES]
    assert {(p["Q"], p["split"]) for p in plans} == {(q, s) for q in range(1, 8) for s in (False, True)}
    assert {p["tbufs"] for p in plans} == {1, 2, 3}
    assert any(p["split"] and p["folds"] > 2 for p in plans)                             # a CTA that folds more than once
    assert any(p["last_chunks"] < min(p["stages"], p["tbufs"]) for p in plans)
    assert {1, 31} <= {p["last_rows"] for p in plans}
    nplans = [(c, nbr_plan(c[1], sum(NBR_SIZES), c[4], c[5], c[3], c[0] == "exact")) for c in NBR_CASES]
    assert {(p["NC"], p["split"]) for _, p in nplans} == {(nc, s) for nc in range(1, 9) for s in (False, True)}
    assert {p["nbuf"] for _, p in nplans} == {1, 2}
    assert {(c[1], c[2], c[3] > 1) for c, _ in nplans} == {(d, mean, deg) for d in ("fwd", "bwd") for mean in (False, True)
                                                           for deg in (False, True)}
    gp = np.cumsum([0] + NBR_SIZES)
    tiles = nbr_tiles(gp, len(NBR_SIZES), int(gp[-1]))
    assert 0 in NBR_SIZES and 64 in NBR_SIZES and (tiles[:, 0] == -1).any()
    gptr = np.cumsum([0] + FILM_LAYOUTS["mixed"])
    spans = [(a // 64, (e - 1) // 64) for a, e in zip(gptr[:-1], gptr[1:]) if e > a]
    assert any(f == l for f, l in spans) and any(l - f >= 2 for f, l in spans)
    assert any(e % 64 == 0 and e > a for a, e in zip(gptr[:-1], gptr[1:]))
    sizes = FILM_LAYOUTS["mixed"]
    assert sizes[0] == 0 and sizes[-1] == 0 and 0 in sizes[1:-1]
    assert set(film_finish_graphs(gptr)) == {0, 3, 4, 5, 6, 8}


# ================================================================================================================================
# 2. hgb_tc_linear / hgb_tc_linear_graph_add
# ================================================================================================================================
def tc_inputs(case, data, seed):
    """CPU operands of one case: a [m, k], w [n, k] (trans_b: [k, n]), bias, addend, gsrc, gadd, gptr"""
    mode, m, n, k, o = case
    g = torch.Generator().manual_seed(seed)
    x = {}
    if data == "dyadic":
        x["a"] = dyadic(g, (m, k), mode)
        x["w"] = dyadic(g, (k, n) if o.get("trans_b") else (n, k), mode)
        small = lambda *sh: dyadic_small(g, sh, mode)  # noqa: E731
    else:
        x["a"] = torch.randn(m, k, generator=g)
        x["w"] = torch.randn(*((k, n) if o.get("trans_b") else (n, k)), generator=g) / k ** 0.5
        small = lambda *sh: torch.randn(*sh, generator=g)  # noqa: E731
    if not o.get("trans_b") and "ga" not in o:
        x["bias"] = small(n)
    if o.get("addend"):
        x["addend"] = small(m, n)
    if "gsrc" in o:
        gs = o["gsrc"]
        if data == "dyadic":
            x["gsrc"] = (torch.randint(-1, 3, (m, n), generator=g).float() * 0.5)   # {-1/2, 0, 1/2, 1}: products stay exact
        elif gs == "deriv":
            x["gsrc"] = torch.rand(m, n, generator=g) * 1.2 - 0.1
        elif gs in ("sigmoid",):
            x["gsrc"] = torch.rand(m, n, generator=g)
        elif gs == "tanh":
            x["gsrc"] = torch.rand(m, n, generator=g) * 2 - 1
        else:
            x["gsrc"] = torch.randn(m, n, generator=g) * 2
    if "ga" in o:
        sizes = ga_sizes(o["ga"], m, seed)
        x["gptr"] = torch.tensor(np.cumsum([0] + sizes), dtype=torch.int32)
        x["gadd"] = small(len(sizes), n)
    return x


def tc_bufs(case, x):
    mode, m, n, k, o = case
    b = {"a": Buf(m, k, ld=k + o.get("lda", 0), data=x["a"]),
         "w": Buf(*x["w"].shape, ld=x["w"].shape[1] + o.get("ldw", 0), data=x["w"])}
    for key in ("bias", "addend", "gsrc"):
        if key in x:
            b[key] = Buf(*(x[key].shape if x[key].dim() == 2 else (x[key].shape[0], 1)), data=x[key])
    if "ga" in o:
        b["gadd"] = Buf(x["gadd"].shape[0], n, ld=o["ldg"], data=x["gadd"])
        b["gptr"] = Buf(x["gptr"].shape[0], 1, dtype=torch.int32, data=x["gptr"])
    return b


def tc_call(case, b, y, z):
    mode, m, n, k, o = case
    ptr = lambda key: b[key].ptr if key in b else None  # noqa: E731
    exact = int(mode == "exact")
    if "ga" in o:
        return lambda: _lib.call("hgb_tc_linear_graph_add", b["a"].ptr, b["a"].ld, b["w"].ptr, b["w"].ld, m, n, k, b["gadd"].ptr,
                                 b["gadd"].ld, b["gptr"].ptr, b["gptr"].rows - 1, y.ptr, exact, stream())
    act = ACT.get(o.get("act", "none"), 0)
    gact = GACT[o["gsrc"]] if "gsrc" in o else o.get("gact", 0)
    param = LRELU_P if o.get("act") == "lrelu" else 0.0
    return lambda: _lib.call("hgb_tc_linear", b["a"].ptr, b["a"].ld, b["w"].ptr, b["w"].ld, int(bool(o.get("trans_b"))), ptr("bias"),
                             m, n, k, act, param, y.ptr, z.ptr if z is not None else None, ptr("addend"), ptr("gsrc"), gact, exact,
                             stream())


def tc_reference(case, x, data, zeta=None):
    """fp64 references and bounds of y (and z): {name: (value, bound, l2 or None, exact?)}"""
    mode, m, n, k, o = case
    a = x["a"]
    w = x["w"].t() if o.get("trans_b") else x["w"]
    c = torch.zeros(m, n, dtype=torch.float64)
    if "bias" in x:
        c = c + x["bias"].double()
    nk = cdiv(k, 256)
    act = o.get("act", "none")
    if "ga" in o:
        gp = x["gptr"].numpy()
        c = c + x["gadd"].double()[torch.from_numpy(graph_of(gp, len(gp) - 1, np.arange(m)))]
    if o.get("addend") and act == "none":
        c = c + x["addend"].double()
    lc = 2 * nk
    if data == "dyadic":
        pre = (split_products(a, w) if mode == "exact" else a.double() @ w.double().t()) + c
        bnd, l2 = torch.zeros_like(pre), None
    else:
        pre, bnd, l2 = tc_ref(a, w, c, mode, k, lc)
    out = {}
    code = ACT[act]
    if act != "none":
        zq = zeta if zeta is not None else pre
        if o.get("z"):
            if o.get("gact") == DERIV and act == "silu":
                out["z"] = (silu_d64(pre), LIP1[code] * bnd + act_eval_err(zq, code, 1), None)
            else:
                out["z"] = (pre, bnd, l2)
        yv = act64(pre, code, LRELU_P)
        yb = LIP[code] * bnd + act_eval_err(zq, code, 0, LRELU_P)
        if o.get("addend"):
            yv = yv + x["addend"].double()
            yb = yb + U * (yv.abs() + yb)
        out["y"] = (yv, yb, None)
        return out
    if "gsrc" in o:
        gs = x["gsrc"].double()
        if o["gsrc"] == "relu_select":
            out["y"] = (torch.where(gs <= 0, torch.zeros_like(pre), pre), torch.where(gs <= 0, torch.zeros_like(bnd), bnd), None)
        else:
            gc = GACT[o["gsrc"]]
            d = grad_from(gs, gs, gc)
            de = grad_from_err(gs, gs, gc)
            v = pre * d
            out["y"] = (v, d.abs() * bnd + pre.abs() * de + bnd * de + U * v.abs(), None)
        return out
    out["y"] = (pre, bnd, l2)
    return out


def silu_d64(z):
    s = torch.sigmoid(z)
    return s * (1 + z * (1 - s))


@pytest.mark.gpu
@pytest.mark.parametrize("data", ["dyadic", "random"])
@pytest.mark.parametrize("case", TC_CASES, ids=tc_id)
def test_tc_linear(case, data):
    mode, m, n, k, o = case
    what = "%s %s" % (tc_id(case), data)
    x = tc_inputs(case, data, seed=m + 3 * n + 7 * k + (data == "random"))
    if data == "dyadic" and "gsrc" in o and o["gsrc"] not in EXACT_GACT:
        x["gsrc"] = torch.randn(m, n, generator=torch.Generator().manual_seed(m))
    b = tc_bufs(case, x)
    y = Buf(m, n)
    z = Buf(m, n) if o.get("z") else None
    call = tc_call(case, b, y, z)
    plan = tc_plan_of(case)
    assert launches(call) == len(plan), what
    outs = [y] + ([z] if z is not None else [])
    twice(what, call, outs)
    for buf in list(b.values()) + outs:
        buf.check(what, "operand", written=True)
    ref = tc_reference(case, x, data, zeta=d64(z.view) if z is not None and o.get("gact") != DERIV else None)
    got = {"y": y, "z": z}
    sec = "tc_linear %s" % mode
    exact_ok = data == "dyadic" and o.get("act", "none") in ("none", "relu") and o.get("gsrc", "deriv") in EXACT_GACT
    for name, (val, bnd, l2) in ref.items():
        gv = d64(got[name].view)
        if exact_ok or (data == "dyadic" and name == "z" and o.get("gact") != DERIV):
            same_f32("%s: %s vs fp64" % (what, name), gv.numpy(), val.numpy())
            continue
        bounded(sec, "%s: %s" % (what, name), gv.numpy(), val.numpy(), bnd.numpy())
        if l2 is not None:
            witness(sec, "%s: %s" % (what, name), gv.numpy(), val.numpy(), l2)


# ================================================================================================================================
# 3. hgb_tc_wgrad
# ================================================================================================================================
def wg_inputs(case, data, seed):
    mode, m, n, k, o = case
    g = torch.Generator().manual_seed(seed)
    if data == "dyadic":
        dz, xx = dyadic(g, (m, n), mode, single=True), dyadic(g, (m, k), mode, single=True)
        if mode == "exact" and m > 4000:                  # one live row per 32-row chunk keeps the sums exact
            live = torch.zeros(m, dtype=torch.bool)
            r = torch.arange(0, m, 32)
            live[(r + (r // 32) % 32).clamp(max=m - 1)] = True
            dz[~live] = 0
            xx[~live] = 0
        dw0, db0 = dyadic_small(g, (n, k), mode), dyadic_small(g, (n,), mode)
    else:
        dz, xx = torch.randn(m, n, generator=g), torch.randn(m, k, generator=g)
        dw0, db0 = torch.randn(n, k, generator=g), torch.randn(n, generator=g)
    return dict(dz=dz, x=xx, dw0=dw0, db0=db0)


def wg_reference(case, x, data, mut=None):
    mode, m, n, k, o = case
    p = wgrad_plan(m, n, k, mode == "exact")
    acc = bool(o.get("accumulate"))
    ones = torch.ones(m, 1)
    b = torch.cat([x["x"], ones], 1)                       # the ones column: the bias gradient
    c = torch.cat([x["dw0"], x["db0"][:, None]], 1).double() if acc else None
    lt = 32 * (min(p["cpc"], 8) if p["split"] else p["cpc"])
    lc = (p["folds"] if p["split"] else 0) + cdiv(p["gx"], 8) + 2 + 8 + int(acc)
    if data == "dyadic":
        val = (split_products(x["dz"].t(), b.t()) if mode == "exact" else x["dz"].double().t() @ b.double())
        val = val + (c if c is not None else 0)
        bnd, l2 = torch.zeros_like(val), None
    else:
        val, bnd, l2 = tc_ref(x["dz"].t(), b.t(), c, mode, lt, lc)
    if mut == "bias_rows_dropped" and n > 128:
        val = val.clone()
        val[128:, k] = c[128:, k] if c is not None else 0
    return val, bnd, l2


@pytest.mark.gpu
@pytest.mark.parametrize("data", ["dyadic", "random"])
@pytest.mark.parametrize("case", WG_CASES, ids=wg_id)
def test_tc_wgrad(case, data):
    mode, m, n, k, o = case
    what = "%s %s" % (wg_id(case), data)
    x = wg_inputs(case, data, seed=m + n + k)
    p = wgrad_plan(m, n, k, mode == "exact")
    dz = Buf(m, n, ld=n + o.get("lddz", 0), data=x["dz"])
    xb = Buf(m, k, ld=k + o.get("ldx", 0), data=x["x"])
    acc = bool(o.get("accumulate"))
    want_b = not o.get("nobias")
    nbytes = _lib.query("hgb_tc_wgrad_workspace_bytes", n, k)
    assert nbytes == NUM_SMS * n * (k + 1) * 4
    ws = ws_buf(nbytes)

    def fresh():
        dw = Buf(n, k, ld=k + o.get("lddw", 0), data=x["dw0"] if acc else None)
        db = Buf(n, 1, data=x["db0"] if acc else None)
        return dw, db

    dw, db = fresh()
    call = lambda: _lib.call("hgb_tc_wgrad", dz.ptr, dz.ld, xb.ptr, xb.ld, m, n, k, dw.ptr, dw.ld, db.ptr if want_b else None,  # noqa: E731
                             int(acc), int(mode == "exact"), ws.ptr, nbytes, stream())
    assert launches(call) == p["launches"], what
    if not acc:
        twice(what, call, [dw, db])
    else:                                                  # accumulate adds into dw / db: a second call starts from fresh buffers
        first = (dw.base.clone(), db.base.clone())
        dw, db = fresh()
        call = lambda: _lib.call("hgb_tc_wgrad", dz.ptr, dz.ld, xb.ptr, xb.ld, m, n, k, dw.ptr, dw.ld, db.ptr if want_b else None,  # noqa: E731
                                 int(acc), int(mode == "exact"), ws.ptr, nbytes, stream())
        call()
        torch.cuda.synchronize()
        assert torch.equal(first[0].view(torch.int32), dw.base.view(torch.int32)), what + ": two identical calls differ"
        assert torch.equal(first[1].view(torch.int32), db.base.view(torch.int32)), what + ": two identical calls differ"
    dw.check(what, "dw")
    db.check(what, "db", written=want_b or acc)
    for buf, name in ((dz, "dz"), (xb, "x")):
        buf.check(what, name)
    ws.check(what, "workspace", written=False)
    val, bnd, l2 = wg_reference(case, x, data)
    got = torch.cat([d64(dw.view), d64(db.view)], 1)
    cols = slice(None) if want_b else slice(0, k)
    if not want_b and acc:
        same_f32(what + ": db untouched", db.np(), x["db0"][:, None].numpy())
    sec = "tc_wgrad %s" % mode
    if data == "dyadic":
        same_f32(what + ": dw, db vs fp64", got[:, cols].numpy(), val[:, cols].numpy())
    else:
        bounded(sec, what + ": dw, db", got[:, cols].numpy(), val[:, cols].numpy(), bnd[:, cols].numpy())
        witness(sec, what + ": dw, db", got[:, cols].numpy(), val[:, cols].numpy(), l2)


# ================================================================================================================================
# 4. the neighbour-sum Linear
# ================================================================================================================================
def nbr_graph(groups, seed):
    """in-degrees set group by group (NBR_SIZES rows of in-degree 0..5 and >= 6, shuffled), random sources with self-loops and
    duplicates, edges in random order; -> (n, dst, src, deg)"""
    g = np.random.default_rng(seed)
    deg = np.concatenate([np.full(s, d) if d < 6 else g.integers(6, 40, s) for d, s in enumerate(NBR_SIZES)])
    g.shuffle(deg)
    n = deg.size
    dst = np.repeat(np.arange(n), deg)
    src = g.integers(0, n, dst.size)
    perm = g.permutation(dst.size)
    return n, dst[perm], src[perm], deg


def degree_order(deg, groups):
    grp = np.minimum(deg, groups - 1)
    order = np.argsort(grp, kind="stable")
    return order.astype(np.int32), np.concatenate([[0], np.cumsum(np.bincount(grp, minlength=groups))]).astype(np.int32)


def csr_by_target(n, dst, src):
    order = np.argsort(dst, kind="stable")               # ascending edge id within each target
    return np.concatenate([[0], np.cumsum(np.bincount(dst, minlength=n))]).astype(np.int32), src[order].astype(np.int32)


def neighbour_sum_f32(x, rowptr, srcs, mean, mut=None):
    """the kernel's h: fp32 adds one after the other from +0 in CSR order, then (mean) one division by max(deg, 1)"""
    n = rowptr.size - 1
    h = np.zeros_like(x)
    for i in range(n):
        v = np.zeros(x.shape[1], np.float32)
        for e in range(rowptr[i], rowptr[i + 1]):
            v = v + x[srcs[e]]
        deg = rowptr[i + 1] - rowptr[i]
        if mean:
            with np.errstate(invalid="ignore", divide="ignore"):
                v = v / np.float32(deg if mut == "mean_by_deg" else max(deg, 1))
        h[i] = v
    return h


def nbr_inputs(case, data, seed):
    mode, direction, mean, groups, k, n_out = case
    n, dst, src, deg = nbr_graph(groups, seed)
    g = torch.Generator().manual_seed(seed)
    if data == "dyadic":
        f = lambda *sh: dyadic(g, sh, mode)  # noqa: E731
        fs = lambda *sh: dyadic_small(g, sh, mode)  # noqa: E731
    else:
        f = lambda *sh: torch.randn(*sh, generator=g)  # noqa: E731
        fs = f
    x = dict(n=n, dst=dst, src=src, deg=deg, wl=f(groups, n_out, k) / (1 if data == "dyadic" else k ** 0.5),
             wr=f(groups, n_out, k) / (1 if data == "dyadic" else k ** 0.5), bias=fs(groups, n_out),
             x=f(n, k), g_out=f(n, n_out))
    return x


def nbr_packed(x, k, n_out):
    groups = x["wl"].shape[0]
    kp = r32(k)
    w = torch.zeros(groups, r32(n_out), 2 * kp)
    w[:, :n_out, :k] = x["wl"]
    w[:, :n_out, kp:kp + k] = x["wr"]
    return w


def nbr_reference(case, x, data, h32, mut=None):
    """fp64 references: fwd out [n, n_out]; bwd g_h, g_xr [n, k]; {name: (value, bound, l2)}"""
    mode, direction, mean, groups, k, n_out = case
    n, deg = x["n"], x["deg"]
    grp = torch.from_numpy(np.minimum(deg, groups - 1))
    wl, wr = x["wl"][grp].double(), x["wr"][grp].double()      # per node [n, n_out, k]
    dd = torch.from_numpy(np.maximum(deg, 1)).double()[:, None]
    out = {}
    if direction == "fwd":
        xs = x["x"].double()
        h = torch.zeros(n, k, dtype=torch.float64).index_add_(0, torch.from_numpy(x["dst"]), xs[torch.from_numpy(x["src"])])
        habs = torch.zeros(n, k, dtype=torch.float64).index_add_(0, torch.from_numpy(x["dst"]), xs.abs()[torch.from_numpy(x["src"])])
        eh = gamma(int(max(deg.max(), 1))) * habs
        if mean:
            h, eh = h / dd, eh / dd + U * (h / dd).abs()
        a = torch.cat([h, xs], 1)                               # [n, 2k]
        wa = torch.cat([wl, wr], 2)                             # [n, n_out, 2k]
        val = torch.einsum("nk,nok->no", a, wa) + x["bias"][grp].double()
        if data == "dyadic" and mode == "tf32" and not mean:
            return {"out": (val, torch.zeros_like(val), None)}
        # the tensor-core bound on the kernel's own operands [h32 | x], group by group; the distance between h32 and the exact h
        # (gamma(deg) sum |x|, over deg in mean mode) enters as an operand error through |W_l|
        a32 = torch.cat([torch.from_numpy(h32), x["x"]], 1)
        bnd = torch.empty_like(val)
        l2sq = 0.0
        for gi in grp.unique().tolist():
            idx = (grp == gi).nonzero().view(-1)
            _, b_, l2 = tc_ref(a32[idx], torch.cat([x["wl"][gi], x["wr"][gi]], 1), x["bias"][gi].double().expand(idx.numel(), n_out),
                               mode, 2 * k, 1)
            bnd[idx] = b_
            l2sq += l2 ** 2
        eop = torch.einsum("nk,nok->no", eh, wl.abs())
        out["out"] = (val, bnd + eop, np.sqrt(l2sq) + float(eop.norm()))
        return out
    go = x["g_out"].double()
    gh = torch.einsum("no,nok->nk", go, wl)
    gx = torch.einsum("no,nok->nk", go, wr)
    if data == "dyadic" and mode == "tf32":
        b0 = torch.zeros_like(gh)
        if mean:
            inv = (np.float32(1) / np.maximum(deg, 1).astype(np.float32)).astype(np.float32)
            gh = torch.from_numpy((gh.numpy().astype(np.float32) * inv[:, None]).astype(np.float32)).double()
        if mut == "mean_on_g_xr":
            gx = gx / dd
        return {"g_h": (gh, b0, None), "g_xr": (gx, b0.clone(), None)}
    ghb = torch.empty_like(gh)
    gxb = torch.empty_like(gx)
    gh_r, gx_r = torch.empty_like(gh), torch.empty_like(gx)
    l2h = l2x = 0.0
    for gi in grp.unique().tolist():
        idx = (grp == gi).nonzero().view(-1)
        v, b_, l2 = tc_ref(x["g_out"][idx], x["wl"][gi].t(), None, mode, n_out, 0)
        gh_r[idx], ghb[idx] = v, b_
        l2h += l2 ** 2
        v, b_, l2 = tc_ref(x["g_out"][idx], x["wr"][gi].t(), None, mode, n_out, 0)
        gx_r[idx], gxb[idx] = v, b_
        l2x += l2 ** 2
    if mean:
        gh_r, ghb = gh_r / dd, ghb / dd + 3 * U * (gh_r / dd).abs()
        l2h = None
    if mut == "mean_on_g_xr":
        gx_r = gx_r / dd
    return {"g_h": (gh_r, ghb, None if l2h is None else np.sqrt(l2h)), "g_xr": (gx_r, gxb, np.sqrt(l2x))}


@pytest.mark.gpu
@pytest.mark.parametrize("data", ["dyadic", "random"])
@pytest.mark.parametrize("case", NBR_CASES, ids=nbr_id)
def test_nbr_linear(case, data):
    mode, direction, mean, groups, k, n_out = case
    what = "%s %s" % (nbr_id(case), data)
    x = nbr_inputs(case, data, seed=k + n_out + groups)
    n = x["n"]
    rowptr, srcs = csr_by_target(n, x["dst"], x["src"])
    if groups > 1:
        order, gptr = degree_order(x["deg"], groups)
    else:
        order, gptr = None, np.array([0, n], np.int32)
    exact = int(mode == "exact")
    p = nbr_plan(direction, n, k, n_out, groups, exact)
    ib = lambda a: Buf(a.size, 1, dtype=torch.int32, data=torch.from_numpy(np.ascontiguousarray(a)))  # noqa: E731
    b_rowptr, b_src, b_gptr = ib(rowptr), ib(srcs), ib(gptr)
    b_order = ib(order) if order is not None else None
    tiles = Buf(cdiv(n, 64) + groups, 2, dtype=torch.int32)
    assert launches(lambda: _lib.call("hgb_nbr_tiles", b_gptr.ptr, groups, n, tiles.ptr, stream())) == 1
    tiles.check(what, "tiles")
    assert np.array_equal(tiles.np(), nbr_tiles(gptr, groups, n)), what + ": tile table"
    w = nbr_packed(x, k, n_out)
    optr = b_order.ptr if b_order is not None else None
    rows = order if order is not None else np.arange(n)
    if direction == "fwd":
        bx = Buf(n, k, data=x["x"])
        bw = Buf(w.shape[0] * w.shape[1], w.shape[2], data=w.reshape(-1, w.shape[2]))
        bb = Buf(groups, n_out, data=x["bias"])
        out, hx = Buf(n, n_out), Buf(n, p["ka"])
        call = lambda: _lib.call("hgb_nbr_linear_fwd", bx.ptr, n, k, b_rowptr.ptr, b_src.ptr, srcs.size, int(mean), optr, b_gptr.ptr,  # noqa: E731
                                 tiles.ptr, groups, bw.ptr, bb.ptr, n_out, out.ptr, hx.ptr, exact, stream())
        outs = {"out": out, "hx": hx}
        ins = [bx, bw, bb]
    else:
        wt = w.transpose(1, 2).contiguous()
        bg = Buf(n, n_out, data=x["g_out"])
        bw = Buf(wt.shape[0] * wt.shape[1], wt.shape[2], data=wt.reshape(-1, wt.shape[2]))
        gh, gxr = Buf(n, k), Buf(n, k)
        call = lambda: _lib.call("hgb_nbr_linear_bwd_data", bg.ptr, n, n_out, b_rowptr.ptr, int(mean), optr, b_gptr.ptr, tiles.ptr,  # noqa: E731
                                 groups, bw.ptr, k, gh.ptr, gxr.ptr, exact, stream())
        outs = {"g_h": gh, "g_xr": gxr}
        ins = [bg, bw]
    assert launches(call) == p["launches"], what
    twice(what, call, list(outs.values()))
    for nm, buf in outs.items():
        buf.check(what, nm)
    for buf in ins + [b_rowptr, b_src, b_gptr, tiles] + ([b_order] if b_order is not None else []):
        buf.check(what, "input")
    h32 = None
    if direction == "fwd":
        h32 = neighbour_sum_f32(x["x"].numpy(), rowptr, srcs, mean)
        kp = r32(k)
        want = np.zeros((n, p["ka"]), np.float32)
        want[:, :k] = h32
        want[:, kp:kp + k] = x["x"].numpy()
        same_f32(what + ": hx vs the fp32 neighbour sum", hx.np(), want[rows])
        if data == "dyadic" and mode == "tf32" and not mean:
            exact_quanta(what, (np.abs(h32) + np.abs(x["x"].numpy())).sum(1) * 2 * 7 / 8 + 1, EXACT_Q["tf32"])
    ref = nbr_reference(case, x, data, h32)
    sec = "nbr %s" % mode
    for nm, (val, bnd, l2) in ref.items():
        gv = d64(outs[nm].view).numpy()
        if data == "dyadic" and mode == "tf32" and (direction == "bwd" or not mean):
            same_f32("%s: %s vs fp64" % (what, nm), gv, val.numpy())
            continue
        bounded(sec, "%s: %s" % (what, nm), gv, val.numpy(), bnd.numpy())
        if l2 is not None and data == "random":
            witness(sec, "%s: %s" % (what, nm), gv, val.numpy(), l2)


# ================================================================================================================================
# 5. FiLM
# ================================================================================================================================
def film_inputs(layout, c, seed):
    sizes = FILM_LAYOUTS[layout]
    g = torch.Generator().manual_seed(seed)
    n, ng = sum(sizes), len(sizes)
    return dict(gptr=np.cumsum([0] + sizes).astype(np.int32), h=torch.randn(n, c, generator=g), dy=torch.randn(n, c, generator=g),
                st=torch.randn(ng, 2 * c, generator=g) * 1.5)


def film_dt_f32(dy, gptr, mut=None):
    """dt in the kernel's order: a graph inside one chunk is summed by its chunk from +0; a graph spanning chunks is its first chunk's
    tail slot plus the head slots of the later chunks, in chunk order (mut "head_tail": the first chunk's head slot instead)"""
    n, c = dy.shape
    ng = len(gptr) - 1
    head = np.full((cdiv(n, 64), c), np.nan, np.float32)
    tail = np.full((cdiv(n, 64), c), np.nan, np.float32)
    dt = np.zeros((ng, c), np.float32)
    for g in range(ng):
        a, e = int(gptr[g]), int(gptr[g + 1])
        for ch in range(a // 64, (e - 1) // 64 + 1) if e > a else ():
            v = np.zeros(c, np.float32)
            for r in range(max(a, ch * 64), min(e, ch * 64 + 64)):
                v = v + dy[r]
            if a // 64 == (e - 1) // 64:
                dt[g] = v
            elif ch == a // 64:
                tail[ch] = v
            else:
                head[ch] = v
    for g in film_finish_graphs(gptr):
        a, e = int(gptr[g]), int(gptr[g + 1])
        if e <= a:
            continue
        cf, cl = a // 64, (e - 1) // 64
        v = (head if mut == "head_tail" else tail)[cf].copy()
        for ch in range(cf + 1, cl + 1):
            v = v + head[ch]
        dt[g] = v
    return dt


def film_reference(x, c):
    """fp64 y, dh, ds, dt and their bounds"""
    gptr = x["gptr"]
    ng = len(gptr) - 1
    batch = torch.from_numpy(np.repeat(np.arange(ng), np.diff(gptr)))
    h, dy, st = x["h"].double(), x["dy"].double(), x["st"].double()
    t = torch.tanh(st[:, :c])
    et = 4 * U * t.abs()                                   # tanhf: 2 ulp
    sc, esc = 1 + t, et + U * (1 + t.abs())
    y = h * sc[batch] + st[batch, c:]
    ey = h.abs() * esc[batch] + 2 * U * ((h * sc[batch]).abs() + st[batch, c:].abs())
    dh = dy * sc[batch]
    edh = dy.abs() * esc[batch] + U * dh.abs()
    s_as = torch.zeros(ng, c, dtype=torch.float64).index_add_(0, batch, dy * h)
    m_as = torch.zeros(ng, c, dtype=torch.float64).index_add_(0, batch, (dy * h).abs())
    sizes = np.diff(gptr)
    L = torch.from_numpy(sizes + sizes // 64 + 3).double()[:, None]      # rows + chunk partials
    eas = L * U / (1 - L * U) * m_as
    f = 1 - t * t
    ef = 2 * t.abs() * et + et * et + 2 * U * (1 + t * t)
    ds = s_as * f
    eds = f.abs() * eas + s_as.abs() * ef + eas * ef + U * ds.abs()
    dt = torch.zeros(ng, c, dtype=torch.float64).index_add_(0, batch, dy)
    return dict(y=(y, ey), dh=(dh, edh), ds=(ds, eds), dt=dt)


@pytest.mark.gpu
@pytest.mark.parametrize("layout", list(FILM_LAYOUTS))
@pytest.mark.parametrize("c", FILM_C)
def test_film(c, layout):
    what = "film c=%d %s" % (c, layout)
    x = film_inputs(layout, c, seed=c + len(layout))
    gptr = x["gptr"]
    n, ng = int(gptr[-1]), len(gptr) - 1
    ldst = 2 * c + 3
    bh, bdy = Buf(n, c, data=x["h"]), Buf(n, c, data=x["dy"])
    bst = Buf(ng, 2 * c, ld=ldst, data=x["st"])
    bg = Buf(ng + 1, 1, dtype=torch.int32, data=torch.from_numpy(gptr))
    y = Buf(n, c)
    fwd = lambda: _lib.call("hgb_film_fwd", bh.ptr, n, c, bst.ptr, ldst, bg.ptr, ng, y.ptr, stream())  # noqa: E731
    assert launches(fwd) == 1
    twice(what, fwd, [y])
    y.check(what, "y")
    ref = film_reference(x, c)
    sec = "film"
    bounded(sec, what + ": y", y.np(), ref["y"][0].numpy(), ref["y"][1].numpy())
    nbytes = _lib.query("hgb_film_bwd_workspace_bytes", n, c)
    assert nbytes == 2 * cdiv(n, 64) * 2 * c * 4
    for want_dh, want_dst in ((True, True), (True, False), (False, True)):
        dh, dst, ws = Buf(n, c), Buf(ng, 2 * c), ws_buf(nbytes)
        bwd = lambda: _lib.call("hgb_film_bwd", bdy.ptr, bh.ptr, n, c, bst.ptr, ldst, bg.ptr, ng, dh.ptr if want_dh else None,  # noqa: E731
                                dst.ptr if want_dst else None, ws.ptr, nbytes, stream())
        w = "%s dh=%d dst=%d" % (what, want_dh, want_dst)
        assert launches(bwd) == film_launches(n, want_dh, want_dst), w
        twice(w, bwd, [dh, dst, ws])
        dh.check(w, "dh", written=want_dh)
        dst.check(w, "dst", written=want_dst)
        ws.check(w, "workspace", written=False)
        if want_dh:
            bounded(sec, w + ": dh", dh.np(), ref["dh"][0].numpy(), ref["dh"][1].numpy())
        if want_dst:
            same_f32(w + ": dt vs the fp32 restatement", dst.np()[:, c:], film_dt_f32(x["dy"].numpy(), gptr))
            bounded(sec, w + ": ds", dst.np()[:, :c], ref["ds"][0].numpy(), ref["ds"][1].numpy())
    for buf in (bh, bdy, bst, bg):
        buf.check(what, "input")


# ================================================================================================================================
# 6. refusals: the entries' own argument checks, before anything launches
# ================================================================================================================================
@pytest.mark.gpu
def test_refused_shapes_launch_nothing():
    a, w, y = Buf(256, 64, ld=64), Buf(64, 64), Buf(256, 64)
    a_odd = Buf(256, 64, ld=66)
    a_mis = Buf(256, 64, off=1)
    gp = Buf(2, 1, dtype=torch.int32, data=torch.tensor([0, 256], dtype=torch.int32))
    gadd = Buf(1, 64)
    ws = ws_buf(_lib.query("hgb_tc_wgrad_workspace_bytes", 64, 64))
    dw = Buf(64, 64)
    st = stream()
    lin = lambda a_, m, n, k, act=0: _lib.call("hgb_tc_linear", a_.ptr, a_.ld, w.ptr, 64, 0, None, m, n, k, act, 0.0, y.ptr,  # noqa: E731
                                               None, None, None, 0, 1, st)
    refusals = [
        lambda: lin(a, 127, 64, 64), lambda: lin(a, 256, 48, 64), lambda: lin(a, 256, 64, 1056), lambda: lin(a, 256, 64, 320, 2),
        lambda: lin(a_odd, 256, 64, 64), lambda: lin(a_mis, 256, 64, 64),
        lambda: _lib.call("hgb_tc_linear_graph_add", a.ptr, 64, w.ptr, 64, 256, 64, 64, gadd.ptr, 64, gp.ptr, 0, y.ptr, 1, st),
        lambda: _lib.call("hgb_tc_linear_graph_add", a.ptr, 64, w.ptr, 64, 256, 64, 64, gadd.ptr, 66, gp.ptr, 1, y.ptr, 1, st),
        lambda: _lib.call("hgb_tc_wgrad", a.ptr, 64, a.ptr, 64, 256, 64, 256, dw.ptr, 64, None, 0, 1, ws.ptr, ws.rows * 4, st),
        lambda: _lib.call("hgb_tc_wgrad", a.ptr, 64, a.ptr, 64, 127, 64, 64, dw.ptr, 64, None, 0, 1, ws.ptr, ws.rows * 4, st),
        lambda: _lib.call("hgb_tc_wgrad", a.ptr, 64, a.ptr, 64, 256, 64, 64, dw.ptr, 64, None, 0, 1, ws.ptr, ws.rows * 4 - 4, st),
        lambda: _lib.call("hgb_tc_wgrad", a_mis.ptr, 64, a.ptr, 64, 256, 64, 64, dw.ptr, 64, None, 0, 1, ws.ptr, ws.rows * 4, st),
        lambda: _lib.call("hgb_nbr_tiles", gp.ptr, 0, 10, dw.ptr, st),
        lambda: _lib.call("hgb_nbr_tiles", gp.ptr, 129, 10, dw.ptr, st),
        lambda: _lib.call("hgb_nbr_linear_fwd", a.ptr, 10, 129, gp.ptr, gp.ptr, 0, 0, None, gp.ptr, gp.ptr, 1, w.ptr, None, 8, y.ptr,
                          None, 1, st),
        lambda: _lib.call("hgb_nbr_linear_fwd", a.ptr, -1, 8, gp.ptr, gp.ptr, 0, 0, None, gp.ptr, gp.ptr, 1, w.ptr, None, 8, y.ptr,
                          None, 1, st),
        lambda: _lib.call("hgb_nbr_linear_bwd_data", a.ptr, 10, 257, gp.ptr, 0, None, gp.ptr, gp.ptr, 1, w.ptr, 8, y.ptr, y.ptr, 1, st),
        lambda: _lib.call("hgb_film_fwd", a.ptr, 10, 8, a.ptr, 15, gp.ptr, 1, y.ptr, st),
        lambda: _lib.call("hgb_film_bwd", a.ptr, a.ptr, 10, 8, a.ptr, 16, gp.ptr, 1, y.ptr, dw.ptr, ws.ptr, 4, st),
    ]
    torch.cuda.synchronize()
    before = _lib.launch_count()
    for i, r in enumerate(refusals):
        with pytest.raises(RuntimeError):
            r()
        torch.cuda.synchronize()
        assert _lib.launch_count() == before, "refusal %d launched a kernel" % i
    for buf, nm in ((y, "y"), (dw, "dw")):
        buf.check("refusals", nm, written=False)
    # n = 0: nothing launches
    for fn in (lambda: _lib.call("hgb_nbr_linear_fwd", None, 0, 8, None, None, 0, 1, None, None, None, 3, None, None, 8, None, None, 1, st),
               lambda: _lib.call("hgb_nbr_linear_bwd_data", None, 0, 8, None, 1, None, None, None, 3, None, 8, None, None, 1, st),
               lambda: _lib.call("hgb_film_fwd", None, 0, 8, a.ptr, 16, gp.ptr, 1, None, st)):
        assert launches(fn) == 0


# ================================================================================================================================
# 7. no GPU: references, exactness of the constructions, mutations
# ================================================================================================================================
def test_references_match_fp64_autograd():
    """the nbr, graph-add and FiLM references against fp64 autograd of the layers they restate"""
    # nbr: out = [h | x] W^T + b per group; its data gradient g_h (mean: / max(deg, 1)) and g_xr through autograd
    for mean in (False, True):
        case = ("exact", "fwd", mean, 7, 5, 9)
        x = nbr_inputs(case, "random", seed=5)
        n = x["n"]
        xx = x["x"].double().requires_grad_(True)
        h = torch.zeros(n, 5, dtype=torch.float64).index_add(0, torch.from_numpy(x["dst"]), xx[torch.from_numpy(x["src"])])
        dd = torch.from_numpy(np.maximum(x["deg"], 1)).double()[:, None]
        if mean:
            h = h / dd
        grp = torch.from_numpy(np.minimum(x["deg"], 6))
        out = (torch.einsum("nk,nok->no", h, x["wl"][grp].double()) + torch.einsum("nk,nok->no", xx, x["wr"][grp].double())
               + x["bias"][grp].double())
        h32 = neighbour_sum_f32(x["x"].numpy(), *csr_by_target(n, x["dst"], x["src"]), mean)
        torch.testing.assert_close(nbr_reference(case, x, "random", h32)["out"][0], out.detach(), rtol=1e-12, atol=1e-12)
        go = x["g_out"].double()
        (gx,) = torch.autograd.grad(out, xx, go)
        r = nbr_reference(("exact", "bwd", mean, 7, 5, 9), x, "random", None)
        gh = r["g_h"][0]
        via = torch.zeros_like(gh).index_add(0, torch.from_numpy(x["src"]), gh[torch.from_numpy(x["dst"])]) + r["g_xr"][0]
        torch.testing.assert_close(via, gx, rtol=1e-12, atol=1e-12)
    # graph add: [a | graph_attr[batch]] W^T + b with gadd = graph_attr W_g^T + b
    case = ("exact", 300, 64, 64, dict(ga="edges", ldg=68))
    x = tc_inputs(case, "random", seed=1)
    ga = torch.randn(len(x["gptr"]) - 1, 3, dtype=torch.float64)
    wg = torch.randn(64, 3, dtype=torch.float64)
    bb = torch.randn(64, dtype=torch.float64)
    x["gadd"] = (ga @ wg.t() + bb).float()
    batch = torch.from_numpy(np.repeat(np.arange(len(x["gptr"]) - 1), np.diff(x["gptr"].numpy())))
    full = torch.cat([x["a"].double(), ga[batch]], 1) @ torch.cat([x["w"].double(), wg], 1).t() + bb
    torch.testing.assert_close(tc_reference(case, x, "random")["y"][0], full, rtol=1e-6, atol=1e-6)
    # FiLM: y and the gradients of fp64 autograd
    for layout in FILM_LAYOUTS:
        x = film_inputs(layout, 33, seed=2)
        gptr = x["gptr"]
        batch = torch.from_numpy(np.repeat(np.arange(len(gptr) - 1), np.diff(gptr)))
        h, st = x["h"].double().requires_grad_(True), x["st"].double().requires_grad_(True)
        y = h * (1 + torch.tanh(st[:, :33]))[batch] + st[:, 33:][batch]
        gh, gst = torch.autograd.grad(y, (h, st), x["dy"].double())
        ref = film_reference(x, 33)
        torch.testing.assert_close(ref["y"][0], y.detach(), rtol=1e-12, atol=1e-12)
        torch.testing.assert_close(ref["dh"][0], gh, rtol=1e-12, atol=1e-12)
        torch.testing.assert_close(ref["ds"][0], gst[:, :33], rtol=1e-12, atol=1e-12)
        torch.testing.assert_close(ref["dt"], gst[:, 33:], rtol=1e-12, atol=1e-12)
        bounded("film restatement", "dt f32 %s" % layout, film_dt_f32(x["dy"].numpy(), gptr), ref["dt"].numpy(),
                gamma(np.diff(gptr).max() + 8) * torch.zeros_like(ref["dt"]).index_add_(0, batch, x["dy"].double().abs()).numpy())


def test_dyadic_constructions_are_exact():
    """every term of every dyadic case is a multiple of the construction's quantum, and the magnitudes of the terms of every output
    stay below 2^24 quanta, so any summation order gives the fp64 value; the split gives hi = s, lo = t with lo != 0 on both sides"""
    g = torch.Generator().manual_seed(0)
    v = dyadic(g, (4096,), "exact")
    hi, lo = split(v)
    assert torch.equal(hi + lo, v) and bool((hi.abs() >= 1).all()) and bool((lo != 0).any())
    assert is_multiple(lo, 2.0 ** -12) and bool((hi == hi.round()).all())
    t8 = dyadic(g, (4096,), "tf32")
    assert torch.equal(_round_tf32(t8), t8) and torch.equal((t8.view(torch.int32) & ~0x1FFF).view(torch.float32), t8)
    for case in TC_CASES:
        mode, m, n, k, o = case
        x = tc_inputs(case, "dyadic", seed=m + 3 * n + 7 * k)
        a = x["a"]
        w = x["w"].t() if o.get("trans_b") else x["w"]
        q = EXACT_Q[mode]
        if mode == "exact":
            ah, al = split(a)
            wh, wl = split(w)
            mag = ah.double().abs() @ (wh.double().abs() + wl.double().abs()).t() + al.double().abs() @ wh.double().abs().t()
            for t in (ah.double()[:64] @ wl.double().t(), al.double()[:64] @ wh.double().t()):
                assert is_multiple(t, q)
        else:
            mag = a.double().abs() @ w.double().abs().t()
            assert is_multiple(a.double()[:64] @ w.double().t(), q)
        for key in ("bias", "addend", "gadd"):
            if key in x:
                assert is_multiple(x[key], q)
                mag = mag + x[key].double().abs().max()
        exact_quanta(tc_id(case), mag.max(), q)
    for case in WG_CASES:
        mode, m, n, k, o = case
        x = wg_inputs(case, "dyadic", seed=m + n + k)
        b = torch.cat([x["x"], torch.ones(m, 1)], 1)
        mag = x["dz"].double().abs().t() @ b.double().abs() * (1 + 2.0 ** -11) + x["dw0"].double().abs().max()
        exact_quanta(wg_id(case), mag.max(), EXACT_Q[mode])
    for case in NBR_CASES:
        if case[0] == "tf32":
            x = nbr_inputs(case, "dyadic", seed=case[4] + case[5] + case[3])
            rp, srcs = csr_by_target(x["n"], x["dst"], x["src"])
            h = neighbour_sum_f32(x["x"].numpy(), rp, srcs, False)
            assert np.array_equal(_round_tf32(torch.from_numpy(h)).numpy(), h), "h must be TF32-exact"
            mag = np.abs(np.concatenate([h, x["x"].numpy()], 1)).sum(1) * 7 / 8 + 1
            exact_quanta(nbr_id(case), mag, EXACT_Q["tf32"])


MUTATIONS = ("split_product_dropped", "split_truncates", "graph_row_off_by_one", "mean_by_deg", "mean_on_g_xr",
             "wgrad_bias_rows_dropped", "film_head_tail_swapped")


def mutation_checks():
    """{mutation: thunk comparing a wrong restatement with fp64 on a test case's own inputs}; None: the faithful restatements"""
    runs = {}
    case = ("exact", 300, 96, 64, {})
    x = tc_inputs(case, "dyadic", seed=7)
    ref = split_products(x["a"], x["w"])
    runs["split_product_dropped"] = lambda: same_f32("drop", split_products(x["a"], x["w"], drop="lh").numpy(), ref.numpy())
    runs["split_truncates"] = lambda: same_f32("trunc", split_products(x["a"], x["w"], trunc=True).numpy(), ref.numpy())
    gcase = ("exact", 200, 32, 64, dict(ga="edges", ldg=36))
    gx = tc_inputs(gcase, "dyadic", seed=200 + 96 + 448)
    gp = gx["gptr"].numpy()
    gref = tc_reference(gcase, gx, "dyadic")["y"][0]
    wrong = split_products(gx["a"], gx["w"]) + gx["gadd"].double()[torch.from_numpy(graph_of(gp, len(gp) - 1, np.arange(200), mut=True))]
    runs["graph_row_off_by_one"] = lambda: same_f32("graph", wrong.numpy(), gref.numpy())
    ncase = ("tf32", "fwd", True, 7, 8, 16)
    nx = nbr_inputs(ncase, "dyadic", seed=3)
    rp, srcs = csr_by_target(nx["n"], nx["dst"], nx["src"])
    h64 = torch.zeros(nx["n"], 8, dtype=torch.float64).index_add_(0, torch.from_numpy(nx["dst"]), nx["x"].double()[torch.from_numpy(nx["src"])])
    h64 = h64 / torch.from_numpy(np.maximum(nx["deg"], 1)).double()[:, None]
    runs["mean_by_deg"] = lambda: bounded("mut", "mean", neighbour_sum_f32(nx["x"].numpy(), rp, srcs, True, mut="mean_by_deg"),
                                          h64.numpy(), 4 * U * h64.abs().numpy())
    runs[None] = [lambda: bounded("mut", "mean", neighbour_sum_f32(nx["x"].numpy(), rp, srcs, True), h64.numpy(), 4 * U * h64.abs().numpy())]
    bcase = ("tf32", "bwd", True, 7, 8, 16)
    bref = nbr_reference(bcase, nx, "dyadic", None)
    bmut = nbr_reference(bcase, nx, "dyadic", None, mut="mean_on_g_xr")
    runs["mean_on_g_xr"] = lambda: same_f32("g_xr", bmut["g_xr"][0].numpy(), bref["g_xr"][0].numpy())
    wcase = ("tf32", 3001, 192, 64, {})
    wx = wg_inputs(wcase, "dyadic", seed=7)
    wref = wg_reference(wcase, wx, "dyadic")[0]
    runs["wgrad_bias_rows_dropped"] = lambda: same_f32("db", wg_reference(wcase, wx, "dyadic", mut="bias_rows_dropped")[0].numpy(),
                                                       wref.numpy())
    fx = film_inputs("mixed", 33, seed=9)
    fref = film_reference(fx, 33)["dt"]
    bnd = gamma(300) * 64
    runs["film_head_tail_swapped"] = lambda: bounded("mut", "dt", film_dt_f32(fx["dy"].numpy(), fx["gptr"], mut="head_tail"),
                                                     fref.numpy(), bnd)
    runs[None] += [lambda: same_f32("drop", split_products(x["a"], x["w"]).numpy(), ref.numpy()),
                   lambda: same_f32("graph", (split_products(gx["a"], gx["w"]) + gx["gadd"].double()[
                       torch.from_numpy(graph_of(gp, len(gp) - 1, np.arange(200)))]).numpy(), gref.numpy()),
                   lambda: bounded("mut", "dt", film_dt_f32(fx["dy"].numpy(), fx["gptr"]), fref.numpy(), bnd)]
    return runs


def test_mutations_are_caught():
    saved = dict(RATIOS)
    try:
        runs = mutation_checks()
        for thunk in runs.pop(None):
            thunk()
        assert set(runs) == set(MUTATIONS)
        for m, thunk in runs.items():
            with pytest.raises((pytest.fail.Exception, AssertionError)):
                thunk()
    finally:
        RATIOS.clear()
        RATIOS.update(saved)


def test_workspace_and_plan_restatements():
    """the restated plans on the shapes the docstrings of hgb_tc.cu name"""
    p = tc_plan(70000, 160, 256, False)
    assert [(q["nc"], q["slots"], q["stages"]) for q in p] == [(160, 2, 4)]
    p = tc_plan(70000, 64, 256, True)
    assert [(q["nc"], q["slots"], q["stages"]) for q in p] == [(64, 2, 4)]
    assert [q["nc"] for q in tc_plan(1500, 480, 64, True)] == [256, 224]
    assert [q["nc"] for q in tc_plan(1500, 224, 256, False)] == [160, 64]
    assert [(q["nc"], q["k0"]) for q in tc_plan(700, 64, 320, True)] == [(64, 0), (64, 256)]
    assert wgrad_plan(m_for(24, NUM_SMS, tail=5), 128, 64, False)["tbufs"] == 3
    assert wgrad_plan(m_for(5, NUM_SMS, tail=2), 128, 224, False)["tbufs"] == 2
    assert wgrad_plan(m_for(20, NUM_SMS, tail=3), 128, 224, True)["tbufs"] == 1
    assert nbr_plan("fwd", 100, 128, 256, 1, True)["nbuf"] == 1 and nbr_plan("fwd", 100, 128, 256, 1, False)["nbuf"] == 2
    assert [tuple(t) for t in nbr_tiles(np.array([0, 0, 64, 64, 130]), 4, 130)] == [(1, 0), (3, 64), (3, 128), (-1, 0), (-1, 0),
                                                                                     (-1, 0), (-1, 0)]
    assert film_threads(1) == 32 and film_threads(33) == 64 and film_threads(200) == 128
