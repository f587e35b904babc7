"""Kernel-level tests of the exact-fp32 dense layers (csrc/hgb_gemm.cu: the SIMT GEMM in all four forms, split-K, the long-
reduction weight gradient, the small-K Linears, the width-1 MLP, activation backward and derivatives, column sums;
csrc/hgb_grouped.cu: the multi-branch heads), each against a plain fp64 restatement of include/hgb.h computed on the CPU.

The C-ABI is called directly, so the test controls every stride, pointer offset, workspace and NULL argument.  Every operand is
the leading block of a NaN-filled buffer: strided operands sit in wider rows (ldx > k, ldc > n, lddw > k), and every input,
output and workspace is followed by GUARD rows of NaN.  After each call every element in range must be finite and every other
element must keep its NaN bits: that catches unwritten elements, stores past row m or column n, and reads of columns k..ld-1 or
rows >= m (a NaN read into a sum makes the result NaN even where its weight is 0).

Bounds, per element (u = 2^-24, gamma(L) = L u / (1 - L u)):
* A sum computed by a chain of L roundings (FMAs or adds, in any association) is off by at most gamma(L) times the sum of the
  magnitudes of its terms (Higham, Accuracy and Stability of Numerical Algorithms, 2nd ed., eq. 3.5).  So element (i, j) of a
  product is held to gamma(L) (|A| |B| + |bias| + |C_old|)_ij, L being the longest sequential chain of that kernel, read from
  the code (`gemm_plan`, `smallk_bwd_plan`, ...):
    gemm_kernel                 k, + 1 for the bias, + 1 for beta_one
    split-K                     k/splits (rounded up to 16) + ceil(splits/8) + 8 (splitk_reduce) + 1
    gemm_tn_fast_kernel         rows per slice per chunk x chunks per CTA + ceil(partials/8) + 8 + 1
    linear_smallk_fwd_*         k (the bias is the first addend)
    linear_smallk_bwd_kernel    dW, db: rows per block / 8 + 8 (walkers) + ceil(blocks/8) + 2 + 8 (reduce);  dx: NPT + 5
    linear_tiny_bwd_kernel      dW, db: rows per block / 256 + 5 + 8 + ceil(blocks/8) + 2 + 8;  dx: n
    colsum                      512/8 + 8 + blocks
    mlp2_scalar_bwd             rows per thread + 5 + 8 + blocks
    grouped rows / wgrad        k + 1 (data gradient: n) / rows of the group;  grouped colsum: rows/8 + 8
  Every bound also carries 2^-126 for the underflow term of fl(x) = x (1 + delta) + eta, |eta| <= 2^-150 per rounding
  (results in the subnormal range, such as dy sigmoid'(y) at y = sigmoid(-90)).
* Inputs of a sum that carry an error of their own add that error times the other factor: dz = dy act'(.) is off by
  E_d <= c u |dy| M(.), where M is the magnitude of the terms of the derivative formula, computed from the same rounded y (or
  z) the kernel reads: 1 + y^2 (tanh), |y| (1 + |y|) (sigmoid), 1 + |y| (ELU), |y| + s a (SELU), 1 (ReLU), |p| (leaky ReLU),
  s (1 + |z| (1 + 2 s)) (SiLU from z, s = sigmoid(z)), |z| (HGB_ACT_DERIV).  These formulas cancel (1 - y^2 near |y| = 1): the
  bound is relative to the terms, not to the result, as for ATen's own derivative of these activations.  c = 4 covers the
  roundings of each formula (at most three, plus the product with dy); the transcendental functions add their documented
  error: tanhf 2 ulp, expm1f 1 ulp, __expf 2 + 1.2 |x| ulp (CUDA C Programming Guide, Mathematical Functions), so every
  activation value or derivative is held to (12 + 2.4 |x|) u times the magnitude of its formula's terms (`act_eval_err`), plus
  2^-120 absolute where __expf overflows or underflows and the kernel returns 0 for a value of order e^-90.
* An activation applied to an fp32 pre-activation z_hat with |z_hat - z| <= E_z is held to Lip(act) E_z + act_eval_err
  (Lip: 1, except SELU 1.7581, leaky ReLU max(1, |p|), SiLU 1.0999, sigmoid 1/4); act' applied to it adds Lip(act') E_z
  (SiLU 0.5, tanh 0.77, sigmoid 0.1, ELU 1, SELU 1.7581, 0 for the piecewise-linear ones).
* On random data the relative L2 error must also stay under 3 u sqrt(L) ||M|| / ||ref|| (+ the norm of the derivative terms):
  rounding errors that behave like independent steps grow as sqrt(L), so a systematic error smaller than the worst case
  bound above (a dropped term, a wrong bias, a sum in lower precision) still fails.

Known answers are bit for bit: inputs k/8 with |k| <= 8 (at most 4 significant bits) make every product and every partial
sum of the shapes used exact in fp32, in any order, so the kernel must return the fp64 result cast to fp32.  Every case runs
twice and must return the same bits (the fixed-order reductions of split-K, tn_fast, colsum, small-K, mlp2 and the grouped
kernels).  The column-sum order is restated in fp32 on the CPU and must be reproduced bit for bit.

`gemm_plan`, `smallk_fwd_plan`, `smallk_bwd_plan`, `mlp2_plan` and `grouped_tiles` restate the host dispatch of hgb_gemm.cu
and hgb_grouped.cu; `test_cases_reach_every_specialisation` (no GPU) asserts that the case lists below reach every kernel
specialisation, and the GPU tests check the number of launches each plan predicts.

Grid limits: row tiles were indexed by gridDim.y (at most 65,535), so gemm_kernel and grouped_rows_kernel refused m above
4,194,240 rows and colsum_stage1 above 33,553,920 rows.  The kernels now stride over row tiles; `test_*_past_65535_row_*`
run one tile past each limit and check that a row's result does not depend on how many tiles the launch has.
"""
import numpy as np
import pytest
import torch

from hydragnn_b200 import _lib, ops
from kernel_harness import (ACT, DERIV, LIP, LIP1, LRELU_P, SELU_A, SELU_S, act64, act_eval_err, deriv64, deriv_terms,
                            grad_from, grad_from_err, l2_bound)

DEV = "cuda"
GUARD = 3                            # NaN rows after every buffer
NAN_BITS = 0x7FC00000                # torch.full(nan) fp32
U = 2.0 ** -24
NUM_SMS = 132                        # HGB_NUM_SMS
TNF_ROWS, TNF_THREADS = 64, 128
UNDERFLOW = 2.0 ** -126              # the underflow term eta of fl(x) = x (1 + delta) + eta, |eta| <= 2^-150, over < 2^24 roundings
CODES = list(ACT.values())


def cdiv(a, b):
    return -(-a // b)


def gamma(L):
    return L * U / (1 - L * U)


# ---- the host dispatch of hgb_gemm.cu / hgb_grouped.cu, restated ---------------------------------------------------------
def pick_splits(m, n, k):
    tiles = cdiv(m, 64) * cdiv(n, 64)
    if tiles >= NUM_SMS or k < 4096:
        return 1
    return max(1, min(cdiv(NUM_SMS * 4, tiles), cdiv(k, 64)))


def tn_fast_tps(m, n):
    """threads per slice of gemm_tn_fast_kernel, or None if the shape cannot take it"""
    if m <= 0 or n <= 0 or m % 8 or n % 8:
        return None
    tps = (m // 8) * (n // 8)
    return tps if 1 <= tps <= TNF_THREADS and TNF_THREADS % tps == 0 else None


def tn_fast_ok(m, n, k, lda, ldb, a_aligned, b_aligned):
    tps = tn_fast_tps(m, n)
    if k < 8192 or tps is None or lda % 4 or ldb % 4 or not (a_aligned and b_aligned):
        return False
    return 2 * TNF_ROWS * (m + n) * 4 <= 160 * 1024 and TNF_ROWS % (TNF_THREADS // tps) == 0


def tn_fast_grid(k):
    return min(cdiv(k, TNF_ROWS), NUM_SMS * 3)


def gemm_workspace_bytes(m, n, k, ta):
    s = pick_splits(m, n, k)
    b = s * m * n * 4 if s > 1 else 0
    tps = tn_fast_tps(m, n) if ta else None
    if tps is not None:
        b = max(b, tn_fast_grid(k) * (TNF_THREADS // tps) * m * n * 4)
    return b


def gemm_plan(m, n, k, ta, tb, lda=None, ldb=None, a_aligned=True, b_aligned=True, ws_bytes=None, beta=False, fused=False):
    """dict(tags, launches, L) of one hgb_gemm (fused: hgb_linear_fwd, bias / act / z, no workspace) call"""
    lda = (m if ta else k) if lda is None else lda
    ldb = (k if tb else n) if ldb is None else ldb
    ws_bytes = gemm_workspace_bytes(m, n, k, ta) if ws_bytes is None else ws_bytes
    if m == 0 or n == 0:
        return dict(tags={"empty"}, launches=0, L=0)
    if k == 0:
        return dict(tags={"k0"}, launches=0, L=0)
    if ta and not tb and not fused and tn_fast_ok(m, n, k, lda, ldb, a_aligned, b_aligned):
        tps = (m // 8) * (n // 8)
        nsl = TNF_THREADS // tps
        grid0 = tn_fast_grid(k)
        if ws_bytes >= grid0 * nsl * m * n * 4:
            nch = cdiv(k, TNF_ROWS)
            cpc = cdiv(nch, grid0)
            grid = cdiv(nch, cpc)
            tags = {"tn_fast[tps=%d]" % tps} | ({"tn_fast_multichunk"} if cpc > 1 else set())
            return dict(tags=tags, launches=2, L=(TNF_ROWS // nsl) * cpc + cdiv(grid * nsl, 8) + 8 + 1)
    tags = set()
    if ta and not tb and not fused and k >= 8192 and tn_fast_tps(m, n) is not None:
        tags.add("tn_fast_fallback_lda" if lda % 4 or ldb % 4 else "tn_fast_fallback_pointer" if not (a_aligned and b_aligned)
                 else "tn_fast_fallback_workspace")
    splits = 1 if fused else pick_splits(m, n, k)
    if splits > 1 and splits * m * n * 4 > ws_bytes:
        splits = 1
        tags.add("splitk_fallback")
    kps = cdiv(cdiv(k, splits), 16) * 16
    splits = max(1, cdiv(k, kps))
    tags.add("gemm<%d,%d>" % (int(ta), int(tb)) + ("+splitk" if splits > 1 else ""))
    if cdiv(m, 64) > 65535:
        tags.add("gemm_row_tiles_past_grid_y")
    if splits > 1:
        return dict(tags=tags, launches=2, L=kps + cdiv(splits, 8) + 8 + 1)
    return dict(tags=tags, launches=1, L=k + 1 + int(beta))


def smallk_fwd_plan(m, n, k, y_aligned=True, z_aligned=True):
    if m == 0:
        return dict(tags={"empty"}, launches=0, L=0)
    if n % 4 == 0 and n >= 16 and y_aligned and z_aligned:
        kt = 1 if k <= 1 else 2 if k <= 2 else 4 if k <= 4 else 8
        return dict(tags={"smallk_fwd_vec4<%d>[k=%d]" % (kt, k)}, launches=1, L=k)
    tags = {"smallk_fwd_scalar[n=%d]" % n}
    if n % 4 == 0 and n >= 16:
        tags.add("smallk_fwd_scalar_misaligned_" + ("y" if not y_aligned else "z"))
    return dict(tags=tags, launches=1, L=k)


def smallk_blocks(m):
    rpb = cdiv(m, NUM_SMS * 4)
    rpb = max(32, cdiv(rpb, 32) * 32)
    return cdiv(m, rpb), rpb


def smallk_bwd_workspace_bytes(m, n, k):
    return smallk_blocks(m)[0] * n * (k + 1) * 4


def smallk_bwd_plan(m, n, k):
    """dict(tags, launches, L_dw, L_dx): L_dw also holds for db"""
    if m == 0:
        return dict(tags={"smallk_bwd_empty"}, launches=0, L_dw=0, L_dx=0)
    nb, rpb = smallk_blocks(m)
    if n <= 8:
        rpb_t = cdiv(cdiv(m, NUM_SMS * 2), 256) * 256
        nbu = cdiv(m, rpb_t)
        return dict(tags={"tiny_bwd[k=%d]" % k}, launches=2, L_dw=cdiv(rpb_t, 256) + 5 + 8 + cdiv(nbu, 8) + 2 + 8, L_dx=n,
                    blocks=nbu)
    kt = 1 if k <= 1 else 2 if k <= 2 else 4 if k <= 4 else 8
    npt = 1 if n <= 32 else 2 if n <= 64 else 4 if n <= 128 else 8
    return dict(tags={"smallk_bwd<%d,%d>" % (kt, npt)}, launches=2, L_dw=rpb // 8 + 8 + cdiv(nb, 8) + 2 + 8, L_dx=npt + 5,
                blocks=nb)


MLP2_BLOCKS = NUM_SMS * 2


def mlp2_plan(n, out):
    if n == 0:
        return dict(tags={"mlp2_empty"}, L=0)
    nb = min(cdiv(n, 256), MLP2_BLOCKS)
    tags = {"mlp2[out=%d]" % out} | ({"mlp2_grid_stride"} if n > nb * 256 else set())
    return dict(tags=tags, L=cdiv(n, nb * 256) + 5 + 8 + nb)


def grouped_tiles(m, groups):
    """tiles of grouped_rows_kernel (the worst case: ceil(m/64) + groups; surplus tiles exit)"""
    return cdiv(m, 64) + groups


def colsum_blocks(m):
    return cdiv(m, 512)


def colsum_workspace_bytes(m, n):
    return (colsum_blocks(m) + 1) * n * 4


# ---- case lists -------------------------------------------------------------------------------------------------------------
EDGE = (1, 63, 64, 65, 129)
GEMM_FORMS = [(0, 0), (0, 1), (1, 0), (1, 1)]
GEMM_K = (0, 1, 15, 16, 17)
# (m, n, k, ta, tb): split-K (tiles < 132, k >= 4096) in all four forms
SPLITK_CASES = [(65, 63, 4096, ta, tb) for ta, tb in GEMM_FORMS] + [(3, 5, 20000, 1, 1), (130, 70, 9000, 0, 0),
                                                                     (130, 70, 9000, 1, 0)]
# (m, n) -> tps 2, 4, 16, 64, 128; r rows
TN_SHAPES = [(8, 16), (16, 16), (32, 32), (64, 64), (64, 128)]
TN_ROWS = (8192, 8193, 8255, 3 * NUM_SMS * 64 * 2 + 5)
TN_CASES = [(m, n, r) for (m, n) in TN_SHAPES for r in TN_ROWS]
TN_FALLBACK = [("pointer", 64, 64, 8200), ("lda", 64, 64, 8200), ("workspace", 32, 32, 9000)]
LINEAR_SHAPES = [(1, 1, 1), (63, 65, 15), (64, 64, 16), (65, 63, 17), (129, 129, 17), (200, 50, 50), (4097, 200, 128),
                 (20000, 24, 8), (3001, 55, 55)]      # F = 50 / 55: the PNA Linears of eam_pna / ogb_pna
SMALLK_FWD = ([(m, n, k, True, True) for k in range(1, 9) for n in (16, 64, 256) for m in (1, 31, 1000)]
              + [(m, n, k, True, True) for n in (1, 3, 5, 12, 255) for k in (1, 3, 8) for m in (1, 31, 1000)]
              + [(1000, n, k, ya, not ya) for n in (16, 64) for k in (2, 5) for ya in (False, True)])
SMALLK_BWD = ([(m, n, k) for k in range(1, 9) for n in (1, 5, 8) for m in (1, 1000)]
              + [(m, n, k) for n in (9, 32, 33, 64, 65, 128, 129, 256) for k in (1, 2, 3, 4, 5, 8) for m in (31, 1000)])
SMALLK_BWD_LARGE = [(1000000, 1, 1), (1000000, 9, 3), (1000000, 33, 8), (1000001, 5, 2)]
MLP2_N = (1, 255, 256, 257, 1000000)
COLSUM_CASES = [(m, n) for m in (1, 511, 512, 513, 1000000) for n in (1, 31, 32, 33, 200) if not (m == 1000000 and n == 200)]
GROUPED_SIZES = {"random100": None, "empty_first": [0, 70, 130], "empty_middle": [65, 0, 64], "empty_last": [129, 1, 0],
                 "edges": [1, 63, 64, 65, 130], "one_group": [300], "all_in_one": [0, 0, 257, 0]}
GROUPED_NK = [(1, 1), (50, 50), (64, 64), (65, 200), (200, 65), (1, 200)]
BIG_M = 64 * 65536 + 1               # one 64-row tile past gridDim.y = 65,535
BIG_COLSUM_M = 512 * 65536 + 1


def all_tags():
    """every specialisation the case lists reach"""
    tags = set()
    for ta, tb in GEMM_FORMS:
        for k in GEMM_K:
            for m in EDGE:
                for n in EDGE:
                    tags |= gemm_plan(m, n, k, ta, tb)["tags"]
    for m, n, k, ta, tb in SPLITK_CASES:
        tags |= gemm_plan(m, n, k, ta, tb)["tags"]
        ws = pick_splits(m, n, k) * m * n * 4
        tags |= gemm_plan(m, n, k, ta, tb, ws_bytes=ws - 4)["tags"]
    for m, n, r in TN_CASES:
        tags |= gemm_plan(m, n, r, 1, 0)["tags"]
    for how, m, n, r in TN_FALLBACK:
        tags |= gemm_plan(m, n, r, 1, 0, **_tn_fallback_args(how, m, n, r))["tags"]
    for m, n, k in LINEAR_SHAPES:
        tags |= gemm_plan(m, n, k, 0, 1, fused=True)["tags"]
    tags |= gemm_plan(BIG_M, 16, 16, 0, 1, fused=True)["tags"]
    for m, n, k, ya, za in SMALLK_FWD:
        tags |= smallk_fwd_plan(m, n, k, ya, za)["tags"]
    for m, n, k in SMALLK_BWD + SMALLK_BWD_LARGE:
        tags |= smallk_bwd_plan(m, n, k)["tags"]
    for out in range(1, 5):
        for n in MLP2_N:
            tags |= mlp2_plan(n, out)["tags"]
    if grouped_tiles(BIG_M, 3) > 65535:
        tags.add("grouped_tiles_past_grid_y")
    if colsum_blocks(BIG_COLSUM_M) > 65535:
        tags.add("colsum_blocks_past_grid_y")
    return tags


def _tn_fallback_args(how, m, n, r):
    if how == "pointer":
        return dict(a_aligned=False)
    if how == "lda":
        return dict(lda=m + 1)
    return dict(ws_bytes=gemm_workspace_bytes(m, n, r, 1) - 4)


REQUIRED = ({"gemm<%d,%d>" % f for f in GEMM_FORMS} | {"gemm<%d,%d>+splitk" % f for f in GEMM_FORMS} | {"splitk_fallback", "k0"}
            | {"tn_fast[tps=%d]" % t for t in (2, 4, 16, 64, 128)} | {"tn_fast_multichunk"}
            | {"tn_fast_fallback_%s" % h for h in ("pointer", "lda", "workspace")}
            | {"smallk_fwd_vec4<%d>[k=%d]" % (1 if k <= 1 else 2 if k <= 2 else 4 if k <= 4 else 8, k) for k in range(1, 9)}
            | {"smallk_fwd_scalar[n=%d]" % n for n in (1, 3, 5, 12, 255)}
            | {"smallk_fwd_scalar_misaligned_y", "smallk_fwd_scalar_misaligned_z"}
            | {"tiny_bwd[k=%d]" % k for k in range(1, 9)} | {"smallk_bwd<%d,%d>" % (a, b) for a in (1, 2, 4, 8) for b in (1, 2, 4, 8)}
            | {"mlp2[out=%d]" % o for o in range(1, 5)} | {"mlp2_grid_stride"}
            | {"gemm_row_tiles_past_grid_y", "grouped_tiles_past_grid_y", "colsum_blocks_past_grid_y"})


def test_cases_reach_every_specialisation():
    """the parametrised cases, run through the restated dispatch, reach every kernel specialisation of hgb_gemm.cu"""
    missing = REQUIRED - all_tags()
    assert not missing, sorted(missing)
    # every vec4 instantiation at every k it serves, every (KT, NPT) pair at more than one k where it serves several
    assert smallk_bwd_plan(1000, 9, 3)["tags"] == {"smallk_bwd<4,1>"}
    assert gemm_plan(65, 63, 4096, 0, 0)["launches"] == 2 and gemm_plan(65, 63, 4095, 0, 0)["launches"] == 1


def test_workspace_restatement_matches_library():
    """the restated workspace sizes are the library's (host-side queries: no GPU needed)"""
    for m, n, k, ta, tb in SPLITK_CASES + [(m, n, r, 1, 0) for m, n, r in TN_CASES] + [(65, 63, 17, 0, 0), (8, 8, 9000, 1, 0)]:
        assert _lib.query("hgb_gemm_workspace_bytes", m, n, k, ta) == gemm_workspace_bytes(m, n, k, ta), (m, n, k, ta)
    for m, n, k in SMALLK_BWD + SMALLK_BWD_LARGE:
        assert _lib.query("hgb_linear_smallk_bwd_workspace_bytes", m, n, k) == smallk_bwd_workspace_bytes(m, n, k)
    for m, n in COLSUM_CASES + [(0, 3), (BIG_COLSUM_M, 1)]:
        assert _lib.query("hgb_colsum_workspace_bytes", m, n) == colsum_workspace_bytes(m, n)
    assert _lib.query("hgb_mlp2_scalar_workspace_bytes") == MLP2_BLOCKS * 10 * 4


# ---- fp64 references ----------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("code", CODES)
def test_reference_activations_match_torch(code):
    """act64 against torch.nn.functional in fp64, deriv64 against fp64 autograd of it (orders 1 and 2, away from the kinks)"""
    x = torch.linspace(-25, 25, 2001, dtype=torch.float64)
    x = x[x.abs() > 1e-6].requires_grad_(True)
    F = torch.nn.functional
    plain = {0: lambda t: t, 1: F.relu, 2: F.silu, 3: torch.tanh, 4: torch.sigmoid, 5: lambda t: F.leaky_relu(t, LRELU_P),
             6: F.elu, 7: F.selu}[code]
    ref = plain(x)
    torch.testing.assert_close(act64(x.detach(), code), ref.detach(), rtol=1e-14, atol=1e-300)
    for order in (1, 2):
        ref = torch.autograd.grad(ref.sum(), x, create_graph=True)[0] if ref.requires_grad else torch.zeros_like(x)
        # atol: autograd's tanh backward is 1 - y^2 in fp64, which cancels where |y| rounds to 1
        torch.testing.assert_close(deriv64(x.detach(), code, order), ref.detach(), rtol=1e-12, atol=1e-15)
        torch.testing.assert_close(deriv_terms(x.detach(), code, order) >= ref.detach().abs() * (1 - 1e-12),
                                   torch.ones_like(x, dtype=torch.bool))
    y = act64(x.detach(), code)
    torch.testing.assert_close(grad_from(y, x.detach(), code), deriv64(x.detach(), code, 1), rtol=1e-10, atol=1e-14)


# ---- harness ------------------------------------------------------------------------------------------------------------------
class Buf:
    """rows x cols block (row stride ld, first element `off` floats into the allocation) of a NaN buffer with GUARD rows after"""

    def __init__(self, rows, cols, ld=None, off=0, data=None):
        self.rows, self.cols = rows, cols
        self.ld = max(cols, 1) if ld is None else ld
        self.off = off
        self.base = torch.full((off + (rows + GUARD) * self.ld,), float("nan"), device=DEV)
        self.view = self.base[off:off + rows * self.ld].view(rows, self.ld)[:, :cols]
        if data is not None:
            self.view.copy_(data.reshape(rows, cols))

    @property
    def ptr(self):
        return self.base.data_ptr() + 4 * self.off

    def check(self, what, name, written=True):
        """written: the block must be finite; always: everything else keeps its NaN bits"""
        mask = torch.zeros_like(self.base, dtype=torch.bool)
        mask[self.off:self.off + self.rows * self.ld].view(self.rows, self.ld)[:, :self.cols] = True
        if written:
            bad = int((~torch.isfinite(self.base[mask])).sum())
            assert bad == 0, "%s: %s has %d unwritten or non-finite entries" % (what, name, bad)
        outside = self.base[~mask].view(torch.int32)
        assert bool((outside == NAN_BITS).all()), "%s: %s written outside its block (%d entries)" % (
            what, name, int((outside != NAN_BITS).sum()))

    def cpu(self):
        return self.view.double().cpu()


def ws_buf(nbytes):
    return Buf(1, max(cdiv(int(nbytes), 4), 1))


def same_bits(a, b):
    return a.shape == b.shape and torch.equal(a.contiguous().view(torch.int32), b.contiguous().view(torch.int32))


def equal_values(a, b):
    """equal values (a known answer: +0 and -0 are the same answer)"""
    return a.shape == b.shape and bool((a == b).all())


def check_close(what, name, got, ref, bound, l2=None):
    """|got - ref| <= bound element by element; l2: bound on ||got - ref|| (absolute, same units)"""
    got = got.double().cpu() if got.is_cuda else got.double()
    err = (got - ref).abs()
    bound = bound + UNDERFLOW
    bad = err > bound
    if bool(bad.any()):
        ratio = err / bound.clamp_min(1e-300)
        i = int(ratio.argmax())
        pytest.fail("%s: %s off its bound in %d of %d entries; worst flat index %d: |err| %.3g, bound %.3g, ref %.6g, got %.6g"
                    % (what, name, int(bad.sum()), bad.numel(), i, float(err.flatten()[i]), float(bound.flatten()[i]),
                       float(ref.flatten()[i]), float(got.flatten()[i])))
    if l2 is not None:
        assert float(err.norm()) <= l2, "%s: %s: L2 error %.3g exceeds %.3g (||ref|| %.3g)" % (
            what, name, float(err.norm()), l2, float(ref.norm()))


def rand(g, *shape, scale=1.0):
    return torch.randn(*shape, generator=g, device=DEV) * scale


def coarse(g, *shape):
    """k / 8 with |k| <= 8: four significant bits"""
    return torch.randint(-8, 9, shape, generator=g, device=DEV).float() / 8.0


def launches(fn):
    torch.cuda.synchronize()
    before = _lib.launch_count()
    fn()
    torch.cuda.synchronize()
    return _lib.launch_count() - before


def twice(what, fn, outs):
    """run fn, snapshot outs, run again: the same bits"""
    fn()
    first = [o.base.clone() for o in outs]
    fn()
    torch.cuda.synchronize()
    for o, f in zip(outs, first):
        assert torch.equal(o.base.view(torch.int32), f.view(torch.int32)), "%s: two identical calls differ" % what


# ---- 1. hgb_gemm ----------------------------------------------------------------------------------------------------------------
def run_gemm(what, m, n, k, ta, tb, g, beta=False, lda=None, ldb=None, ldc=None, a_off=0, ws_bytes=None, exact=False,
             check_l2=True):
    lda = lda or max(m if ta else k, 1)
    ldb = ldb or max(k if tb else n, 1)
    ldc = ldc or max(n, 1)
    mk = (k, m) if ta else (m, k)
    kn = (n, k) if tb else (k, n)
    gen = coarse if exact else rand
    a = Buf(mk[0], mk[1], lda, off=a_off, data=gen(g, *mk))
    b = Buf(kn[0], kn[1], ldb, data=gen(g, *kn))
    c0 = gen(g, m, n)
    c = Buf(m, n, ldc, data=c0 if beta else None)
    need = _lib.query("hgb_gemm_workspace_bytes", m, n, k, int(ta))
    ws_bytes = need if ws_bytes is None else ws_bytes
    ws = ws_buf(ws_bytes)
    plan = gemm_plan(m, n, k, ta, tb, lda, ldb, (a.ptr % 16) == 0, True, ws_bytes, beta)

    def call():
        if beta:
            c.view.copy_(c0)
        _lib.call("hgb_gemm", a.ptr, b.ptr, c.ptr, m, n, k, int(ta), int(tb), lda, ldb, ldc, int(beta), ws.ptr, ws_bytes,
                  ops._stream())

    nl = launches(call)
    assert nl == plan["launches"], "%s: %d launches, the plan says %d (%s)" % (what, nl, plan["launches"], plan["tags"])
    for buf, name in ((a, "a"), (b, "b")):
        buf.check(what, name)
    c.check(what, "c", written=m * n > 0)
    ws.check(what, "workspace", written=False)
    A, B = a.cpu(), b.cpu()
    A, B = (A.t() if ta else A), (B.t() if tb else B)
    ref = A @ B + (c0.double().cpu() if beta else 0)
    mag = A.abs() @ B.abs() + (c0.double().cpu().abs() if beta else 0)
    got = c.cpu()
    if exact:
        assert equal_values(got.float(), ref.float()), "%s: not the exact answer in %d entries" % (what, int((got != ref).sum()))
    else:
        check_close(what, "c", got, ref, gamma(plan["L"]) * mag, l2_bound(plan["L"], mag) if check_l2 else None)
    twice(what, call, [c])
    return plan


@pytest.mark.gpu
@pytest.mark.parametrize("k", GEMM_K)
@pytest.mark.parametrize("ta,tb", GEMM_FORMS, ids=["%s%s" % ("T" if a else "N", "T" if b else "N") for a, b in GEMM_FORMS])
def test_gemm_forms_at_tile_edges(ta, tb, k):
    """gemm_kernel<TA,TB> at m, n in {1, 63, 64, 65, 129}: alternately accumulating (beta_one), with ld > the block (lda, ldb,
    ldc one to three columns wider, NaN-filled); k = 0 zeroes C, or leaves it alone with beta_one"""
    g = torch.Generator(device=DEV).manual_seed(10 * ta + tb + 100 * k)
    for i, (m, n) in enumerate((m, n) for m in EDGE for n in EDGE):
        beta = i % 2 == 1
        wide = i % 3 == 0
        lda = (m if ta else k) + 3 if wide else None
        ldb = (k if tb else n) + 1 if wide else None
        ldc = n + 2 if wide else None
        run_gemm("gemm ta=%d tb=%d m=%d n=%d k=%d beta=%d" % (ta, tb, m, n, k, beta), m, n, k, ta, tb, g, beta, lda, ldb, ldc)


@pytest.mark.gpu
@pytest.mark.parametrize("m,n,k,ta,tb", SPLITK_CASES)
def test_gemm_split_k(m, n, k, ta, tb):
    """split-K with beta_one and ldc > n; then the same call with a workspace 4 bytes short, which must run unsplit"""
    g = torch.Generator(device=DEV).manual_seed(m + n + k)
    p = run_gemm("split-K", m, n, k, ta, tb, g, beta=True, ldc=n + 5)
    assert any(t.endswith("+splitk") for t in p["tags"])
    need = pick_splits(m, n, k) * m * n * 4
    p = run_gemm("split-K, short workspace", m, n, k, ta, tb, g, beta=False, ws_bytes=need - 4)
    assert "splitk_fallback" in p["tags"]


@pytest.mark.gpu
@pytest.mark.parametrize("m,n,r", TN_CASES, ids=["tps%d-r%d" % ((m // 8) * (n // 8), r) for m, n, r in TN_CASES])
def test_gemm_tn_fast(m, n, r):
    """the long-reduction weight gradient C = A^T B at every threads-per-slice count, r rows with a partial last chunk and with
    several chunks per CTA; alternately accumulating into a wider C"""
    g = torch.Generator(device=DEV).manual_seed(m * n + r)
    beta = r % 2 == 1
    p = run_gemm("tn_fast m=%d n=%d r=%d" % (m, n, r), m, n, r, 1, 0, g, beta=beta, ldc=n + 4 if beta else None)
    assert any(t.startswith("tn_fast[") for t in p["tags"]), p


@pytest.mark.gpu
@pytest.mark.parametrize("how,m,n,r", TN_FALLBACK)
def test_gemm_tn_fast_fallbacks(how, m, n, r):
    """a 4-byte-offset A, lda % 4 != 0, or a workspace too short for tn_fast: gemm_kernel<true,false> (split if it fits)"""
    g = torch.Generator(device=DEV).manual_seed(r)
    kw = _tn_fallback_args(how, m, n, r)
    p = run_gemm("tn_fast fallback (%s)" % how, m, n, r, 1, 0, g, lda=kw.get("lda"), a_off=1 if how == "pointer" else 0,
                 ws_bytes=kw.get("ws_bytes"))
    assert "tn_fast_fallback_" + how in p["tags"] and not any(t.startswith("tn_fast[") for t in p["tags"]), p


@pytest.mark.gpu
@pytest.mark.parametrize("m,n,k,ta,tb", [(65, 63, 17, 0, 0), (129, 64, 16, 1, 1), (65, 63, 4096, 0, 1), (64, 64, 8255, 1, 0),
                                         (8, 16, 50693, 1, 0)])
def test_gemm_known_answers(m, n, k, ta, tb):
    """four-bit inputs: every path returns the fp64 result cast to fp32, bit for bit"""
    g = torch.Generator(device=DEV).manual_seed(m + k)
    run_gemm("gemm exact", m, n, k, ta, tb, g, beta=True, ldc=n + 1, exact=True)
    run_gemm("gemm exact", m, n, k, ta, tb, g, exact=True)


# the data gradient dZ W (NN) and a column block of a wider x accumulated into C (NT) at layer shapes
LAYER_GEMMS = [(5000, 64, 64, 0, 0, False), (4097, 128, 200, 0, 0, True), (5000, 64, 64, 0, 1, True), (3000, 192, 64, 0, 1, False)]


@pytest.mark.gpu
@pytest.mark.parametrize("m,n,k,ta,tb,beta", LAYER_GEMMS)
def test_gemm_layer_shapes(m, n, k, ta, tb, beta):
    g = torch.Generator(device=DEV).manual_seed(m + n + k)
    run_gemm("gemm layer m=%d n=%d k=%d" % (m, n, k), m, n, k, ta, tb, g, beta=beta, lda=k + 8 if beta else None)


# ---- 2. hgb_linear_fwd ----------------------------------------------------------------------------------------------------------
def check_act_output(what, name, y, zref, zmag, L, code, p=LRELU_P):
    """y = act(z_hat), |z_hat - z| <= gamma(L) zmag: Lip(act) gamma(L) zmag + act_eval_err(z)"""
    ez = gamma(L) * zmag
    check_close(what, name, y, act64(zref, code, p), LIP[code] * ez + act_eval_err(zref, code, 0, p))


def run_linear(what, m, n, k, code, bias, want_z, g, ldx=None, ldw=None, exact=False):
    gen = coarse if exact else rand
    x = Buf(m, k, ldx, data=gen(g, m, k))
    w = Buf(n, k, ldw, data=gen(g, n, k) * (1 if exact else 0.5))
    b = Buf(1, n, data=gen(g, n)) if bias else None
    y = Buf(m, n)
    z = Buf(m, n) if want_z else None
    p = 0.25 if exact else LRELU_P
    plan = gemm_plan(m, n, k, 0, 1, ldx, ldw, fused=True)

    def call():
        _lib.call("hgb_linear_fwd", x.ptr, w.ptr, b.ptr if b else None, m, n, k, x.ld, w.ld, code, p, y.ptr,
                  z.ptr if z else None, ops._stream())

    assert launches(call) == 1
    for buf, name in ((x, "x"), (w, "w"), (b, "b"), (y, "y"), (z, "z")):
        if buf is not None:
            buf.check(what, name)
    X, W = x.cpu(), w.cpu()
    B = b.cpu()[0] if b else torch.zeros(n, dtype=torch.float64)
    zref = X @ W.t() + B
    zmag = X.abs() @ W.abs().t() + B.abs()
    L = k + int(bias)
    if exact:
        assert equal_values(y.cpu().float(), act64(zref, code, p).float()), what
        if z:
            assert equal_values(z.cpu().float(), zref.float()), what
    else:
        check_act_output(what, "y", y.cpu(), zref, zmag, L, code)
        if z:
            check_close(what, "z", z.cpu(), zref, gamma(L) * zmag, l2_bound(L, zmag))
    twice(what, call, [y] + ([z] if z else []))
    return plan


@pytest.mark.gpu
@pytest.mark.parametrize("want_z", [False, True], ids=["y", "y+z"])
@pytest.mark.parametrize("bias", [False, True], ids=["nobias", "bias"])
@pytest.mark.parametrize("act", list(ACT))
def test_linear_fwd(act, bias, want_z):
    """y = act(x W^T + b) through gemm_kernel<false,true> at tile edges; x and w alternately column blocks of wider rows"""
    g = torch.Generator(device=DEV).manual_seed(ACT[act] * 4 + 2 * bias + want_z)
    for i, (m, n, k) in enumerate(LINEAR_SHAPES):
        ldx, ldw = (k + 3, k + 1) if i % 2 else (None, None)
        run_linear("linear %s m=%d n=%d k=%d" % (act, m, n, k), m, n, k, ACT[act], bias, want_z, g, ldx, ldw)


@pytest.mark.gpu
@pytest.mark.parametrize("act", ["none", "relu", "lrelu"])
def test_linear_fwd_known_answers(act):
    g = torch.Generator(device=DEV).manual_seed(ACT[act])
    for m, n, k in ((65, 63, 17), (129, 1, 40), (1, 129, 3)):
        run_linear("linear exact %s" % act, m, n, k, ACT[act], True, True, g, ldx=k + 2, exact=True)


# ---- 3. small-K Linears ---------------------------------------------------------------------------------------------------------
def run_smallk_fwd(what, m, n, k, code, bias, want_z, g, y_off=0, z_off=0, ldx=None, ldw=None, exact=False):
    gen = coarse if exact else rand
    x = Buf(m, k, ldx, data=gen(g, m, k))
    w = Buf(n, k, ldw, data=gen(g, n, k))
    b = Buf(1, n, data=gen(g, n)) if bias else None
    y = Buf(m, n, off=y_off)
    z = Buf(m, n, off=z_off) if want_z else None
    plan = smallk_fwd_plan(m, n, k, y.ptr % 16 == 0, z is None or z.ptr % 16 == 0)

    def call():
        _lib.call("hgb_linear_smallk_fwd", x.ptr, x.ld, w.ptr, w.ld, b.ptr if b else None, m, n, k, code, LRELU_P, y.ptr,
                  z.ptr if z else None, ops._stream())

    assert launches(call) == plan["launches"], what
    for buf, name in ((x, "x"), (w, "w"), (b, "b"), (y, "y"), (z, "z")):
        if buf is not None:
            buf.check(what, name, written=m > 0)
    X, W = x.cpu(), w.cpu()
    B = b.cpu()[0] if b else torch.zeros(n, dtype=torch.float64)
    zref, zmag = X @ W.t() + B, X.abs() @ W.abs().t() + B.abs()
    if exact:
        assert equal_values(y.cpu().float(), act64(zref, code).float()), what
    else:
        check_act_output(what, "y", y.cpu(), zref, zmag, plan["L"], code)
        if z:
            check_close(what, "z", z.cpu(), zref, gamma(plan["L"]) * zmag, l2_bound(plan["L"], zmag))
    twice(what, call, [y] + ([z] if z else []))
    return plan


@pytest.mark.gpu
@pytest.mark.parametrize("m,n,k,ya,za", SMALLK_FWD, ids=["m%d-n%d-k%d%s" % (m, n, k, "" if ya and za else "-y+4" if not ya
                                                                               else "-z+4") for m, n, k, ya, za in SMALLK_FWD])
def test_smallk_fwd(m, n, k, ya, za):
    """the vec4 kernel at every k (KT = 1, 2, 4, 8), the scalar kernel at n not a multiple of 4 or with y / z 4 bytes off a
    16-byte boundary; activations, bias, z and a wider x row rotate over the cases"""
    i = SMALLK_FWD.index((m, n, k, ya, za))
    code = CODES[i % len(CODES)]
    run_smallk_fwd("smallk_fwd m=%d n=%d k=%d act=%d" % (m, n, k, code), m, n, k, code, i % 3 != 0, i % 2 == 0 or not za,
                   torch.Generator(device=DEV).manual_seed(i), y_off=0 if ya else 1, z_off=0 if za else 1,
                   ldx=k + 2 if i % 4 == 1 else None, ldw=k + 1 if i % 5 == 2 else None)


@pytest.mark.gpu
@pytest.mark.parametrize("m", [0, 1, 31])
@pytest.mark.parametrize("n", [256, 255, 16])
def test_smallk_fwd_edges(m, n):
    """n = 256 (the limit), m = 0 writes nothing"""
    g = torch.Generator(device=DEV).manual_seed(m + n)
    run_smallk_fwd("smallk_fwd edge m=%d n=%d" % (m, n), m, n, 8, ACT["silu"], True, True, g)
    run_smallk_fwd("smallk_fwd exact m=%d n=%d" % (m, n), m, n, 5, ACT["relu"], True, False, g, exact=True)


def run_smallk_bwd(what, m, n, k, code, g, want=("dx", "dw", "db"), lddw=None, exact=False):
    gen = coarse if exact else rand
    p = 0.25 if exact else LRELU_P
    X = gen(g, m, k)
    Wt = gen(g, n, k)
    Z = gen(g, m, n) * (1 if exact else 2)
    Y = act64(Z.double(), code if code != DERIV else 0, p).float()
    DY = gen(g, m, n)
    x = Buf(m, k, k + 1 if m % 2 else None, data=X)
    w = Buf(n, k, k + 2 if n % 2 else None, data=Wt)
    dy = Buf(m, n, data=DY)
    uses_z = code in (ACT["silu"], DERIV)
    y = Buf(m, n, data=None if uses_z else Y)             # the one of y / z the code does not read stays NaN
    z = Buf(m, n, data=Z if uses_z else None)
    dx = Buf(m, k) if "dx" in want else None
    dw = Buf(n, k, lddw) if "dw" in want else None
    db = Buf(1, n) if "db" in want else None
    plan = smallk_bwd_plan(m, n, k)
    ws = ws_buf(_lib.query("hgb_linear_smallk_bwd_workspace_bytes", m, n, k))

    def call():
        _lib.call("hgb_linear_smallk_bwd", dy.ptr, y.ptr, z.ptr, x.ptr, x.ld, w.ptr, w.ld, m, n, k, code, p,
                  dx.ptr if dx else None, dw.ptr if dw else None, dw.ld if dw else k, db.ptr if db else None, ws.ptr,
                  ops._stream())

    assert launches(call) == plan["launches"], what
    for buf, name in ((x, "x"), (w, "w"), (dy, "dy"), (dx, "dx"), (dw, "dw"), (db, "db")):
        if buf is not None:
            buf.check(what, name, written=name in ("dw", "db") or m > 0)
    y.check(what, "y", written=not uses_z and m > 0)
    z.check(what, "z", written=uses_z and m > 0)
    ws.check(what, "workspace", written=False)
    Xd, Wd, DYd, Yd, Zd = X.double().cpu(), Wt.double().cpu(), DY.double().cpu(), Y.double().cpu(), Z.double().cpu()
    dz = DYd * grad_from(Yd, Zd, code, p)
    edz = DYd.abs() * grad_from_err(Yd, Zd, code, p) + (U * dz.abs() if code not in (ACT["none"], ACT["relu"]) else 0)
    outs = []
    if dx:
        ref, mag = dz @ Wd, dz.abs() @ Wd.abs()
        extra = edz @ Wd.abs()
        if exact:
            assert equal_values(dx.cpu().float(), ref.float()), what + " dx"
        else:
            check_close(what, "dx", dx.cpu(), ref, gamma(plan["L_dx"]) * mag + extra, l2_bound(plan["L_dx"], mag, extra))
        outs.append(dx)
    if dw:
        ref, mag, extra = dz.t() @ Xd, dz.abs().t() @ Xd.abs(), edz.t() @ Xd.abs()
        if exact:
            assert equal_values(dw.cpu().float(), ref.float()), what + " dw"
        else:
            check_close(what, "dw", dw.cpu(), ref, gamma(plan["L_dw"]) * mag + extra, l2_bound(plan["L_dw"], mag, extra))
        outs.append(dw)
    if db:
        ref, mag, extra = dz.sum(0, keepdim=True), dz.abs().sum(0, keepdim=True), edz.sum(0, keepdim=True)
        if exact:
            assert equal_values(db.cpu().float(), ref.float()), what + " db"
        else:
            check_close(what, "db", db.cpu(), ref, gamma(plan["L_dw"]) * mag + extra, l2_bound(plan["L_dw"], mag, extra))
        outs.append(db)
    twice(what, call, outs)
    return plan


BWD_CODES = CODES + [DERIV]


@pytest.mark.gpu
@pytest.mark.parametrize("m,n,k", SMALLK_BWD, ids=["m%d-n%d-k%d" % c for c in SMALLK_BWD])
def test_smallk_bwd(m, n, k):
    """linear_tiny_bwd_kernel at every k, linear_smallk_bwd_kernel at every (KT, NPT); every activation (SiLU and
    HGB_ACT_DERIV through z) rotates over the cases, as do a NULL dx / dw / db and lddw > k"""
    i = SMALLK_BWD.index((m, n, k))
    code = BWD_CODES[i % len(BWD_CODES)]
    want = [("dx", "dw", "db"), ("dw", "db"), ("dx", "db"), ("dx", "dw")][i % 4]
    run_smallk_bwd("smallk_bwd m=%d n=%d k=%d act=%d %s" % (m, n, k, code, want), m, n, k, code,
                   torch.Generator(device=DEV).manual_seed(i), want, lddw=k + 3 if i % 3 == 0 else None)


@pytest.mark.gpu
@pytest.mark.parametrize("m,n,k", SMALLK_BWD_LARGE)
def test_smallk_bwd_many_blocks(m, n, k):
    """about 520 per-block partials, the last block partial"""
    run_smallk_bwd("smallk_bwd m=%d n=%d k=%d" % (m, n, k), m, n, k, ACT["tanh"], torch.Generator(device=DEV).manual_seed(m + n))


@pytest.mark.gpu
@pytest.mark.parametrize("n,k", [(5, 3), (64, 8), (200, 1)])
def test_smallk_bwd_edges(n, k):
    """m = 0 zeroes dW (lddw > k) and db and launches nothing; four-bit inputs give the exact answer"""
    g = torch.Generator(device=DEV).manual_seed(n)
    run_smallk_bwd("smallk_bwd m=0", 0, n, k, ACT["relu"], g, lddw=k + 2)
    for code in (ACT["none"], ACT["relu"], ACT["lrelu"], DERIV):
        run_smallk_bwd("smallk_bwd exact act=%d" % code, 997, n, k, code, g, lddw=k + 1, exact=True)


# ---- 4. the width-1 MLP ---------------------------------------------------------------------------------------------------------
def mlp2_reference(x, pk, gy, out, code):
    """fp64 values and bounds of hgb_mlp2_scalar_{fwd,bwd} (module docstring)"""
    w1, b1, w2, b2 = pk[0], pk[1], pk[2:2 + out], pk[6:6 + out]
    z = w1 * x + b1
    ez = U * (abs(w1) * x.abs() + abs(b1))
    h = act64(z, code)
    eh = LIP[code] * ez + act_eval_err(z, code)
    y = h[:, None] * w2 + b2
    ey = eh[:, None] * w2.abs() + U * (h.abs()[:, None] * w2.abs() + b2.abs())
    gh = gy @ w2
    egh = gamma(4) * (gy.abs() @ w2.abs())
    d = deriv64(z, code, 1)
    ed = LIP1[code] * ez + 2 * (1 + h.abs()) * act_eval_err(z, code) + act_eval_err(z, code, 1)
    if code == ACT["none"]:
        ed = torch.zeros_like(z)
    gz = gh * d
    egz = gh.abs() * ed + d.abs() * egh + U * gz.abs()
    return dict(y=y, ey=ey, h=h, eh=eh, gz=gz, egz=egz)


def run_mlp2(what, n, out, code, g, with_gx=True):
    x = Buf(n, 1, data=rand(g, n, scale=2.0))
    pk = Buf(1, 10, data=rand(g, 10))
    gy = Buf(n, out, data=rand(g, n, out))
    y = Buf(n, out)
    gx = Buf(n, 1) if with_gx else None
    gp = Buf(1, 10)
    ws = ws_buf(_lib.query("hgb_mlp2_scalar_workspace_bytes"))
    plan = mlp2_plan(n, out)

    def call():
        _lib.call("hgb_mlp2_scalar_fwd", x.ptr, pk.ptr, n, out, code, LRELU_P, y.ptr, ops._stream())
        _lib.call("hgb_mlp2_scalar_bwd", gy.ptr, x.ptr, pk.ptr, n, out, code, LRELU_P, gx.ptr if gx else None, gp.ptr, ws.ptr,
                  ops._stream())

    assert launches(call) == (0 if n == 0 else 3), what
    for buf, name in ((x, "x"), (pk, "params"), (gy, "gy"), (y, "y"), (gx, "gx"), (gp, "gparams")):
        if buf is not None:
            buf.check(what, name, written=n > 0 or name == "gparams")
    ws.check(what, "workspace", written=False)
    X, P, GY = x.cpu()[:, 0], pk.cpu()[0], gy.cpu()
    r = mlp2_reference(X, P, GY, out, code)
    check_close(what, "y", y.cpu(), r["y"], r["ey"])
    if gx:
        check_close(what, "gx", gx.cpu()[:, 0], r["gz"] * P[0], r["egz"] * abs(P[0]) + U * (r["gz"] * P[0]).abs())
    L = plan["L"]
    terms = [(r["gz"] * X, r["egz"] * X.abs()), (r["gz"], r["egz"])]
    terms += [(GY[:, j] * r["h"], GY[:, j].abs() * r["eh"]) for j in range(out)] + [(torch.zeros(n, dtype=torch.float64),) * 2] * (4 - out)
    terms += [(GY[:, j], torch.zeros(n, dtype=torch.float64)) for j in range(out)] + [(torch.zeros(n, dtype=torch.float64),) * 2] * (4 - out)
    ref = torch.stack([t.sum() for t, _ in terms])
    bound = torch.stack([gamma(L) * t.abs().sum() + e.sum() for t, e in terms])
    check_close(what, "gparams", gp.cpu()[0], ref, bound)
    twice(what, call, [y, gp] + ([gx] if gx else []))


@pytest.mark.gpu
@pytest.mark.parametrize("out", [1, 2, 3, 4])
@pytest.mark.parametrize("act", list(ACT))
def test_mlp2_scalar(act, out):
    """Linear(1,1) - act - Linear(1,out) forward and backward at n = 1, 255, 256, 257 and 10^6 (the grid-stride loop past the
    264-block cap), gx alternately NULL; n = 0 zeroes the parameter gradient and writes nothing else"""
    g = torch.Generator(device=DEV).manual_seed(ACT[act] * 5 + out)
    for i, n in enumerate(MLP2_N + (0,)):
        run_mlp2("mlp2 %s out=%d n=%d" % (act, out, n), n, out, ACT[act], g, with_gx=(i + out) % 2 == 0)


# ---- 5. activation backward and derivatives --------------------------------------------------------------------------------------
SPECIAL_X = [0.0, -0.0, 1e-3, -1e-3, 1.0, -1.0, 4.0, -4.0, 20.0, -20.0, 90.0, -90.0]


@pytest.mark.gpu
@pytest.mark.parametrize("count", [0, 1, 1001, 300001])
@pytest.mark.parametrize("code", BWD_CODES)
def test_act_bwd(code, count):
    """dz = dy act'(.) from y (every code but SiLU, whose z buffer stays NaN) or from z (SiLU; HGB_ACT_DERIV: z holds act');
    the buffer a code does not read stays NaN"""
    g = torch.Generator(device=DEV).manual_seed(code * 7 + count)
    Z = rand(g, count, scale=3.0)
    Z[:min(count, len(SPECIAL_X))] = torch.tensor(SPECIAL_X[:min(count, len(SPECIAL_X))], device=DEV)
    Y = act64(Z.double(), code if code != DERIV else 0).float()
    DY = rand(g, count)
    uses_z = code in (ACT["silu"], DERIV)
    dy, dz = Buf(count, 1, data=DY), Buf(count, 1)
    y = Buf(count, 1, data=None if uses_z else Y)
    z = Buf(count, 1, data=Z if uses_z else None)
    what = "act_bwd code=%d count=%d" % (code, count)

    def call():
        _lib.call("hgb_act_bwd", dy.ptr, y.ptr, z.ptr, count, code, LRELU_P, dz.ptr, ops._stream())

    assert launches(call) == (1 if count else 0)
    for buf, name in ((dy, "dy"), (dz, "dz")):
        buf.check(what, name, written=count > 0)
    (z if not uses_z else y).check(what, "unread z / y", written=False)
    Yd, Zd, DYd = Y.double().cpu()[:, None], Z.double().cpu()[:, None], DY.double().cpu()[:, None]
    ref = DYd * grad_from(Yd, Zd, code)
    bound = DYd.abs() * grad_from_err(Yd, Zd, code) + (U * ref.abs() if code not in (ACT["none"], ACT["relu"]) else 0)
    check_close(what, "dz", dz.cpu(), ref, bound)
    twice(what, call, [dz])


@pytest.mark.gpu
@pytest.mark.parametrize("order", [0, 1, 2])
@pytest.mark.parametrize("act", list(ACT))
def test_act_deriv(act, order):
    """value, first and second derivative at +-0, +-1e-3, +-1, +-4, +-20, +-90 (where __expf overflows) and on N(0, 3^2);
    at x = 0 the kernel takes the left branch (x > 0 is the right one): relu'(0) = 0, leaky_relu'(0) = p, elu'(0) = 1,
    selu'(0) = s a"""
    code = ACT[act]
    g = torch.Generator(device=DEV).manual_seed(code * 3 + order)
    X = torch.cat([torch.tensor(SPECIAL_X, device=DEV), rand(g, 4001, scale=3.0), torch.linspace(-30, 30, 601, device=DEV)])
    cnt = X.numel()
    x, out = Buf(cnt, 1, data=X), Buf(cnt, 1)
    what = "act_deriv %s order=%d" % (act, order)

    def call():
        _lib.call("hgb_act_deriv", x.ptr, cnt, code, LRELU_P, order, out.ptr, ops._stream())

    assert launches(call) == 1
    x.check(what, "x")
    out.check(what, "out")
    Xd = X.double().cpu()[:, None]
    ref = deriv64(Xd, code, order)
    check_close(what, "out", out.cpu(), ref, act_eval_err(Xd, code, order) + U * ref.abs() * (code == ACT["lrelu"]))
    zero = out.cpu()[:2, 0]
    want0 = {1: (0.0, 0.0), 5: (LRELU_P, 0.0), 6: (1.0, 1.0), 7: (SELU_S * SELU_A, SELU_S * SELU_A)}
    if order in (1, 2) and code in want0:
        assert torch.allclose(zero, torch.full((2,), want0[code][order - 1], dtype=torch.float64), rtol=4 * U, atol=0), (what, zero)
    twice(what, call, [out])


# ---- 6. column sums -------------------------------------------------------------------------------------------------------------
def colsum_fp32_order(x):
    """hgb_colsum's summation order restated in fp32 (numpy: adds of two float32 round once): stage 1, per 512-row block,
    8 walkers add rows walker, walker + 8, ... from 0, then the 8 walker sums from 0; stage 2 adds the block partials in order"""
    m, n = x.shape
    nb = colsum_blocks(m)
    xp = np.zeros((nb * 512, n), dtype=np.float32)
    xp[:m] = x
    xp = xp.reshape(nb, 64, 8, n)
    acc = np.zeros((nb, 8, n), dtype=np.float32)
    for t in range(64):
        acc = acc + xp[:, t]
    part = np.zeros((nb, n), dtype=np.float32)
    for y in range(8):
        part = part + acc[:, y]
    return np.add.accumulate(np.concatenate([np.zeros((1, n), np.float32), part]), axis=0, dtype=np.float32)[-1]


def run_colsum(what, m, n, g, exact=False):
    X = (coarse if exact else rand)(g, m, n)
    x, out = Buf(m, n, data=X), Buf(1, n)
    ws = ws_buf(_lib.query("hgb_colsum_workspace_bytes", m, n))

    def call():
        _lib.call("hgb_colsum", x.ptr, m, n, out.ptr, ws.ptr, ops._stream())

    assert launches(call) == (2 if m else 0)
    x.check(what, "x")
    out.check(what, "out")
    ws.check(what, "workspace", written=False)
    Xd = X.double().cpu()
    ref = Xd.sum(0, keepdim=True)
    L = 64 + 8 + colsum_blocks(m)
    mag = Xd.abs().sum(0, keepdim=True)
    if exact:
        assert equal_values(out.cpu().float(), ref.float()), what
    else:
        check_close(what, "out", out.cpu(), ref, gamma(L) * mag, l2_bound(L, mag))
    order = torch.from_numpy(colsum_fp32_order(X.cpu().numpy()))[None, :]
    assert same_bits(out.view.cpu(), order), "%s: not the documented summation order in %d columns" % (
        what, int((out.view.cpu() != order).sum()))
    twice(what, call, [out])


@pytest.mark.gpu
@pytest.mark.parametrize("m,n", COLSUM_CASES + [(0, 5)])
def test_colsum(m, n):
    run_colsum("colsum m=%d n=%d" % (m, n), m, n, torch.Generator(device=DEV).manual_seed(m + n))


@pytest.mark.gpu
def test_colsum_known_answer():
    run_colsum("colsum exact", 100003, 33, torch.Generator(device=DEV).manual_seed(1), exact=True)


# ---- 7. grouped heads -----------------------------------------------------------------------------------------------------------
def group_sizes(name, g):
    if name == "random100":
        s = torch.randint(0, 40, (100,), generator=g).tolist()
        s[0], s[50], s[99] = 0, 0, 0
        return s
    return GROUPED_SIZES[name]


def run_grouped(what, sizes, n, k, g, code=ACT["tanh"], bias=True, want_z=True, ldx=None, exact=False):
    groups, m = len(sizes), sum(sizes)
    rowptr = torch.tensor([0] + list(np.cumsum(sizes)), dtype=torch.int32, device=DEV)
    gen = coarse if exact else rand
    gd = torch.Generator(device=DEV).manual_seed(int(torch.randint(0, 2 ** 30, (1,), generator=g)))
    x = Buf(m, k, ldx, data=gen(gd, m, k))
    w = Buf(groups * n, k, data=gen(gd, groups * n, k) * (1 if exact else 0.5))    # [groups, n, k]
    b = Buf(groups, n, data=gen(gd, groups, n)) if bias else None
    dy = Buf(m, n, data=gen(gd, m, n))
    y, z = Buf(m, n), (Buf(m, n) if want_z else None)
    gx = Buf(m, k)                     # the data gradient dy [m, n] W_g: the same w, read as [groups, k_red = n, n_out = k]
    dw, db = Buf(groups * n, k), Buf(groups, n)
    st = ops._stream()

    def call():
        _lib.call("hgb_grouped_linear", x.ptr, x.ld, w.ptr, b.ptr if b else None, rowptr.data_ptr(), groups, m, n, k, 0, code,
                  LRELU_P, y.ptr, z.ptr if z else None, st)
        _lib.call("hgb_grouped_linear", dy.ptr, n, w.ptr, None, rowptr.data_ptr(), groups, m, k, n, 1, 0, 0.0, gx.ptr, None, st)
        _lib.call("hgb_grouped_wgrad", dy.ptr, x.ptr, x.ld, rowptr.data_ptr(), groups, m, n, k, dw.ptr, db.ptr, st)

    call()
    torch.cuda.synchronize()
    for buf, name in ((x, "x"), (w, "w"), (b, "b"), (dy, "dy"), (y, "y"), (z, "z"), (gx, "gx"), (dw, "dw"),
                      (db, "db")):
        if buf is not None:
            buf.check(what, name, written=m > 0 or name in ("w", "b", "dw", "db"))
    X, W, DY = x.cpu(), w.cpu().view(groups, n, k), dy.cpu()
    B = b.cpu() if b else torch.zeros(groups, n, dtype=torch.float64)
    ofs = [0] + list(np.cumsum(sizes))
    Y, ZM, GX, GXM = (torch.zeros(m, n, dtype=torch.float64), torch.zeros(m, n, dtype=torch.float64),
                      torch.zeros(m, k, dtype=torch.float64), torch.zeros(m, k, dtype=torch.float64))
    DW, DWM, DB, DBM = (torch.zeros(groups, n, k, dtype=torch.float64), torch.zeros(groups, n, k, dtype=torch.float64),
                        torch.zeros(groups, n, dtype=torch.float64), torch.zeros(groups, n, dtype=torch.float64))
    for q in range(groups):
        r = slice(int(ofs[q]), int(ofs[q + 1]))
        Y[r] = X[r] @ W[q].t() + B[q]
        ZM[r] = X[r].abs() @ W[q].abs().t() + B[q].abs()
        GX[r] = DY[r] @ W[q]
        GXM[r] = DY[r].abs() @ W[q].abs()
        DW[q] = DY[r].t() @ X[r]
        DWM[q] = DY[r].abs().t() @ X[r].abs()
        DB[q] = DY[r].sum(0)
        DBM[q] = DY[r].abs().sum(0)
    L_rows = max(sizes) if sizes else 0
    if exact:
        for name, got, ref in (("y", y, act64(Y, code)), ("gx", gx, GX), ("dw", dw, DW.view(groups * n, k)), ("db", db, DB)):
            assert equal_values(got.cpu().float(), ref.float()), "%s: %s not exact" % (what, name)
    else:
        check_act_output(what, "y", y.cpu(), Y, ZM, k + int(bias), code)
        if z:
            check_close(what, "z", z.cpu(), Y, gamma(k + int(bias)) * ZM, l2_bound(k + 1, ZM))
        check_close(what, "gx", gx.cpu(), GX, gamma(n) * GXM, l2_bound(n, GXM))
        check_close(what, "dw", dw.cpu().view(groups, n, k), DW, gamma(L_rows) * DWM, l2_bound(L_rows, DWM))
        check_close(what, "db", db.cpu(), DB, gamma(cdiv(L_rows, 8) + 8) * DBM, l2_bound(cdiv(L_rows, 8) + 8, DBM))
    twice(what, call, [y, gx, dw, db] + ([z] if z else []))


@pytest.mark.gpu
@pytest.mark.parametrize("n,k", GROUPED_NK)
@pytest.mark.parametrize("sizes", list(GROUPED_SIZES))
def test_grouped(sizes, n, k):
    """forward (trans_w 0: bias, activation, z), data gradient (trans_w 1) and weight gradient with db per group; 100 groups of
    random sizes with empty ones, empty first / middle / last groups, groups of 1, 63, 64, 65, 130 rows, all rows in one group;
    x alternately a column block of wider rows"""
    g = torch.Generator().manual_seed(n * 1000 + k + len(sizes))
    s = group_sizes(sizes, g)
    i = list(GROUPED_SIZES).index(sizes)
    code = CODES[(i + n) % len(CODES)]
    run_grouped("grouped %s n=%d k=%d act=%d" % (sizes, n, k, code), s, n, k, g, code=code, bias=i % 2 == 0,
                want_z=i % 3 != 1, ldx=k + 3 if i % 2 else None)


@pytest.mark.gpu
def test_grouped_edges():
    """m = 0 (nothing written, the weight gradient zeroed) and four-bit inputs (the exact answer, bit for bit)"""
    g = torch.Generator().manual_seed(3)
    run_grouped("grouped m=0", [0, 0, 0], 50, 20, g)
    run_grouped("grouped exact", [1, 63, 0, 64, 65, 130], 65, 50, g, code=ACT["relu"], exact=True)


# ---- 8. past 65,535 row tiles ---------------------------------------------------------------------------------------------------
def _sample_rows(m, g, count=4096):
    picks = torch.randint(0, m, (count,), generator=g)
    return torch.unique(torch.cat([torch.arange(0, 128), torch.arange(m - 129, m), picks]))


@pytest.mark.gpu
@pytest.mark.parametrize("entry", ["linear_fwd", "gemm_nn"])
def test_gemm_past_65535_row_tiles(entry):
    """m = 64 * 65536 + 1 rows of a 16 x 16 Linear (gemm_kernel<false,true>) and of a plain NN product: the first and last
    tiles and 4,096 seeded rows against fp64, and every checked row bit-identical to the same row computed by a call over its
    own 64-row tile (a row's sum does not depend on how many tiles the launch has)"""
    m, n, k = BIG_M, 16, 16
    g = torch.Generator(device=DEV).manual_seed(5)
    X = rand(g, m, k)
    W = rand(g, n, k)
    bias = rand(g, n)
    x, y = Buf(m, k, data=X), Buf(m, n)
    wmat = W if entry == "linear_fwd" else W.t().contiguous()
    w = Buf(*wmat.shape, data=wmat)
    b = Buf(1, n, data=bias)
    st = ops._stream()

    def call(xp, rows, yp):
        if entry == "linear_fwd":
            _lib.call("hgb_linear_fwd", xp, w.ptr, b.ptr, rows, n, k, k, k, ACT["silu"], 0.0, yp, None, st)
        else:
            _lib.call("hgb_gemm", xp, w.ptr, yp, rows, n, k, 0, 0, k, n, n, 0, None, 0, st)

    assert launches(lambda: call(x.ptr, m, y.ptr)) == 1
    y.check(entry, "y")
    rows = _sample_rows(m, torch.Generator().manual_seed(6))
    Xs = X[rows.to(DEV)].double().cpu()
    Wd = W.double().cpu()
    zref = Xs @ Wd.t() + (bias.double().cpu() if entry == "linear_fwd" else 0)
    zmag = Xs.abs() @ Wd.abs().t() + (bias.double().cpu().abs() if entry == "linear_fwd" else 0)
    got = y.view[rows.to(DEV)].double().cpu()
    if entry == "linear_fwd":
        check_act_output(entry, "y", got, zref, zmag, k + 1, ACT["silu"])
    else:
        check_close(entry, "y", got, zref, gamma(k) * zmag)
    for t0 in (0, 64 * 30000, 64 * 65534, 64 * 65535, m - 1):
        rows_t = min(64, m - t0)
        one = Buf(rows_t, n)
        call(x.ptr + 4 * t0 * k, rows_t, one.ptr)
        torch.cuda.synchronize()
        assert same_bits(one.view, y.view[t0:t0 + rows_t]), "%s: tile at row %d differs from its own call" % (entry, t0)


@pytest.mark.gpu
def test_grouped_past_65535_row_tiles():
    """m = 64 * 65536 + 1 rows in 3 groups (65,539 tiles): sampled rows against fp64, and rows of the last group bit-identical
    to a call with that group alone"""
    m, n, k = BIG_M, 16, 16
    sizes = [1000, m - 1000 - 777, 777]
    g = torch.Generator(device=DEV).manual_seed(7)
    X = rand(g, m, k)
    W = rand(g, 3, n, k)
    B = rand(g, 3, n)
    x, y, w, b = Buf(m, k, data=X), Buf(m, n), Buf(3 * n, k, data=W), Buf(3, n, data=B)
    rowptr = torch.tensor([0, 1000, m - 777, m], dtype=torch.int32, device=DEV)
    st = ops._stream()
    assert launches(lambda: _lib.call("hgb_grouped_linear", x.ptr, k, w.ptr, b.ptr, rowptr.data_ptr(), 3, m, n, k, 0, 0, 0.0,
                                      y.ptr, None, st)) == 1
    y.check("grouped big", "y")
    rows = _sample_rows(m, torch.Generator().manual_seed(8))
    grp = torch.bucketize(rows, torch.tensor([1000, m - 777]), right=True)
    Xs, Wd, Bd = X[rows.to(DEV)].double().cpu(), W.double().cpu(), B.double().cpu()
    ref = torch.einsum("rk,rnk->rn", Xs, Wd[grp]) + Bd[grp]
    mag = torch.einsum("rk,rnk->rn", Xs.abs(), Wd[grp].abs()) + Bd[grp].abs()
    check_close("grouped big", "y", y.view[rows.to(DEV)].double().cpu(), ref, gamma(k + 1) * mag)
    last = Buf(777, n)
    rp = torch.tensor([0, 777], dtype=torch.int32, device=DEV)
    _lib.call("hgb_grouped_linear", x.ptr + 4 * (m - 777) * k, k, w.ptr + 4 * 2 * n * k, b.ptr + 4 * 2 * n, rp.data_ptr(), 1,
              777, n, k, 0, 0, 0.0, last.ptr, None, st)
    torch.cuda.synchronize()
    assert same_bits(last.view, y.view[m - 777:]), "grouped big: the last group differs from its own call"
    assert grouped_tiles(sum(sizes), 3) > 65535


@pytest.mark.gpu
def test_colsum_past_65535_row_blocks():
    """m = 512 * 65536 + 1 rows, n = 1 (65,537 row blocks): fp64 bound and the documented fp32 order, bit for bit"""
    run_colsum("colsum big", BIG_COLSUM_M, 1, torch.Generator(device=DEV).manual_seed(9))
