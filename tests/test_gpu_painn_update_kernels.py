"""Kernel-level tests of the PaiNN update block (hydragnn/models/PAINNStack.py:298-328), which the PaiNN and PNAEq stacks run
through three paths:

* PainnUpdateFn (any width): the U/V Linear, then the elementwise steps of csrc/hgb_painn.cu -- hgb_painn_update_pre_fwd
  (mlp_in = [|vv|, s]), hgb_painn_update_post_fwd (s_out = s + a_sv inner + a_ss, v_out = v + a_vv uv),
  hgb_painn_update_post_bwd_a (ga = [sum_d gv_out_d uv_d, gs_out inner, gs_out]) and hgb_painn_update_bwd (guv, gvv, gs and an
  optional copy gv = gv_out);
* PainnUpdateScalarFn (width 1, the first PaiNN layer): hgb_painn_update_scalar_fwd / _bwd over a 16-value parameter pack;
* PainnUpdateTcFn (width 64, TF32 mode): hgb_painn_update_tc_fwd / _post / _bwd_a / _bwd of csrc/hgb_painn_tc.cu, which recompute
  [uv | vv] on the tensor cores for every 64-node tile.

The C ABI is called directly through tests/kernel_harness.py: every output is the leading block of a NaN-filled buffer with guard
rows (`Buf.check`: everything in range written, nothing else touched), every call runs twice with identical bits, and every entry
launches the kernels its host code names, none at n = 0.

u = 2^-24, gamma(k) = k u / (1 - k u).  Nothing is built with fast-math, so sqrtf and the division are correctly rounded; nvcc
contracts products into FMAs, and an FMA only removes a rounding.

1. The elementwise steps, bit for bit.  Every input is drawn from {0, +-1/2, +-1, +-3/2, +-2}.  A product of two or three of them
   is a multiple of 1/8 below 2^4 and every sum these kernels form stays a multiple of 1/8 below 2^6, so every product and sum is
   exact in fp32 whatever the order and whatever FMA contraction nvcc applies.  The only roundings left are sqrtf (|vv|), the
   division gn / nrm, and, in gvv = g a_sv u + (gn / nrm) w, the product with that quotient and the sum after it: each a single
   correctly rounded fp32 operation, which numpy's fp32 arithmetic restates exactly.  So every output equals the numpy fp32
   restatement (`emu_steps`) bit for bit, +0 and -0 included (the restatement starts its dot products from +0 as the kernels
   do).  The restatement itself is held to fp64 (`ref_steps`): exact outputs to 0, |vv| to u |vv|, gvv to
   3u (|g a_sv u| + |gn / nrm w|).  A row with vv = 0 has nrm = 0 and must take gn_over = 0.  At f = 64 and n = 8449,
   n f > 132 x 16 x 256 threads, so the grid-stride loops run twice.

2. The width-one kernel, against fp64 autograd of oracle.painn.PainnUpdate(1, last).  The per-node bound is a running error
   analysis executed in fp64 (class R): every fp32 operation adds u times its result, errors propagate through products,
   quotients and square roots with their exact first- and second-order terms, and a fused multiply-add is counted as two
   roundings, so the bound holds with or without contraction.  hgb_sigmoid(x) = 1 / (1 + __expf(-x)); __expf is within
   2 + 1.2 |x| ulp (CUDA C Programming Guide, Mathematical Functions), the add and the reciprocal round once each and the
   sigmoid's sensitivity to a relative error of e^-x is below 1, so hgb_sigmoid is within (3 + 1.2 |x|) ulp = (3 + 1.2 |x|) 2^-23
   relative, plus its Lipschitz constant 1/4 times the error of x.  The 13 parameter gradients are sums over nodes, reduced in
   four stages (per-thread fp32 sums, the 5-step warp shuffle, the 8 warp sums added one after the other, the block partials
   in order); each is held to sum_terms err + gamma(terms per thread + 5 + 8 + blocks) sum_terms (|term| + err), sum |term| in
   fp64.  The unused slots of the
   parameter pack are NaN, so a kernel that reads them fails, and the gradient pack's unused slots must come back 0.
   n = 67585 is past the backward's 264 x 256 threads and n = 135169 past the forward's 528 x 256.

3. The tensor-core update, entry by entry, each on its own random operands: (i) bit for bit against the unfused pieces on the same
   operands (hgb_tc_linear for [uv | vv], the matching hgb_painn_update_* step, and for tc_bwd the dgrad with its addend), as the
   header of hgb_painn_tc.cu states; (ii) against fp64 with v, [U; V] and [guv | gvv] rounded to TF32 (oracle.tf32._round_tf32):
   a K-term product with its bias or addend is within gamma(K + 2) (sum |a b| + |c|) plus TF32_OPERAND sum |a b| for the
   tensor cores' own operand conversion (see its note in kernel_harness.py), then class R carries the error through the elementwise formulas.  n covers
   partial tiles (1, 63, 65, 129), the producer ring wrapping its parity, and more tiles than one persistent wave at one or two
   CTAs per SM (8449, 16897).  At n < 64 the 64-row TMA box is taller than the tensor; the hardware fills the missing rows with
   zeros, the kernels store no row >= n, and the results equal the unfused pieces bit for bit, so the entries accept any n >= 0.

Worst |error| / bound measured on an H100 (80 GB HBM3, 700 W) over this file: elementwise steps 0.76 (gvv), width-one per-node
outputs 0.92, width-one parameter gradients 0.056, tensor-core entries against fp64 1.00 (to three digits: on some element the
operand-conversion term is used almost in full); the modules' rel-L2 reached 0.62 of 5e-3 in TF32 mode.  The module fixture prints
these ratios at the end of a run.

4. The three autograd functions and PNAEq's PainnUpdate at qm9_painn / gfm_pnaeq shapes against fp64 autograd of the oracle block:
   outputs and all 10 gradients, rel-L2 5e-3 in TF32 mode (test_gpu_painn_tc.py), FP32_TOL in fp32 mode (see its note).

5. The dispatch census: which entries each module call reaches, and that together they reach every kernel instantiation.

6. No GPU: the restatements and references against torch autograd of the oracle block, and deliberately wrong restatements that
   must each fail a comparison.
"""
import functools
import math

import numpy as np
import pytest
import torch

from hydragnn_b200 import _lib, ops, pnaeq, stacks
from kernel_harness import U, Buf, cdiv, check_bound, gamma, grid_for, launches, same_f32, stream, tf32_gemm, twice, ws_buf

DEV = "cuda"
NUM_SMS = 132
F_STEP = (1, 2, 3, 7, 17, 32, 63, 64, 65, 128)
N_STEP = (0, 1, 77, 8449)
LAYOUTS = ("sep", "prod", "pad")
N_SCALAR = (0, 1, 255, 256, 257, 67585, 135169)
N_TC = (1, 63, 64, 65, 128, 129, 8449, 16897)
SCALAR_BWD_BLOCKS = 2 * NUM_SMS               # UPD_SCALAR_BLOCKS
SCALAR_FWD_BLOCKS = 4 * NUM_SMS
# rel-L2 of the fp32-mode modules against fp64, measured once on an H100 (80 GB HBM3, 700 W): worst 3.7e-6 over the outputs and
# the 10 gradients of every case in section 4; held to 2e-5
FP32_TOL = 2e-5
RATIOS = {}                                   # worst |err| / bound per section, printed at the end of the module


def _note(section, ratio):
    RATIOS[section] = max(RATIOS.get(section, 0.0), float(ratio))


@pytest.fixture(scope="module", autouse=True)
def _report_ratios():
    yield
    if RATIOS:
        print("\nworst |error| / bound: " + ", ".join("%s %.3g" % kv for kv in sorted(RATIOS.items())))


def bounded(section, what, got, ref, bnd):
    """check_bound, with NaN / inf failing outright, and the worst ratio noted"""
    got = np.asarray(got, np.float64)
    ref, bnd = np.asarray(ref, np.float64), np.broadcast_to(np.asarray(bnd, np.float64), got.shape)
    if not np.isfinite(got).all():
        pytest.fail("%s: %d non-finite entries" % (what, int((~np.isfinite(got)).sum())))
    err = np.abs(got - ref)
    if err.size:
        _note(section, np.max(np.where(bnd > 0, err / np.maximum(bnd, 1e-300), np.where(err > 2.0 ** -126, np.inf, 0.0))))
    check_bound(what, got, ref, bnd)


# ================================================================================================================================
# 1. the elementwise steps of PainnUpdateFn
# ================================================================================================================================
def exact(rng, *shape):
    return (rng.integers(-4, 5, shape) / 2).astype(np.float32)


def layout(kind, f):
    """(row stride ld, column of vv) of the [3n, ld] block holding uv at column 0; "sep": uv and vv in two buffers of stride f"""
    return {"sep": (f, None), "prod": (2 * f, f), "pad": (2 * f + 5, f + 5)}[kind]


def step_inputs(n, f, seed):
    rng = np.random.default_rng(seed)
    x = dict(uv=exact(rng, 3 * n, f), vv=exact(rng, 3 * n, f), s=exact(rng, n, f), v=exact(rng, n, 3 * f), a=exact(rng, n, 3 * f),
             gs_out=exact(rng, n, f), gv_out=exact(rng, n, 3 * f), g_mlp_in=exact(rng, n, 2 * f))
    x["vv"].reshape(n, 3, f)[::5] = 0.0                  # |vv| = 0: the gn_over = 0 rule
    return x


def image(kind, uv, vv):
    """the memory the kernels read uv and vv from: (uv flat, uv offset, vv flat, vv offset, ld)"""
    f = uv.shape[1]
    ld, col = layout(kind, f)
    if col is None:
        return uv.ravel(), 0, vv.ravel(), 0, ld
    full = np.full((uv.shape[0], ld), np.nan, np.float32)
    full[:, :f], full[:, col:col + f] = uv, vv
    return full.ravel(), 0, full.ravel(), col, ld


def gather(flat, off, ld, m, f):
    return flat[off + np.arange(m)[:, None] * ld + np.arange(f)[None, :]]


def emu_steps(x, img, n, f, last, mlp_in=None, mut=()):
    """fp32 restatement of pre_fwd, post_fwd, post_bwd_a and bwd (with the gv copy); mlp_in: bwd's operand (default: pre_fwd's
    output).  mut: deliberately wrong variants for the mutation test"""
    uf, uo, vf, vo, ld = img
    if "ld_as_f" in mut:
        ld = f
    uv, vv = gather(uf, uo, ld, 3 * n, f).reshape(n, 3, f), gather(vf, vo, ld, 3 * n, f).reshape(n, 3, f)
    na = 2 if last else 3
    a = x["a"][:, :na * f].reshape(n, na, f)
    a_sv, a_ss = a[:, na - 2], a[:, na - 1]
    if "sv_ss_swapped" in mut:
        a_sv, a_ss = a_ss, a_sv
    use_v = not last or "avv_when_last" in mut
    a_vv = a[:, 0] if use_v else np.zeros_like(a_sv)
    gvo = x["gv_out"].reshape(n, 3, f) if use_v else np.zeros((n, 3, f), np.float32)
    zero = np.float32(0.0)
    out = {}
    nrm = np.sqrt(vv[:, 0] * vv[:, 0] + vv[:, 1] * vv[:, 1] + vv[:, 2] * vv[:, 2])
    out["mlp_in"] = np.concatenate([nrm, x["s"]], axis=1)
    inner = ((zero + uv[:, 0] * vv[:, 0]) + uv[:, 1] * vv[:, 1]) + uv[:, 2] * vv[:, 2]
    out["s_out"] = (x["s"] + a_sv * inner) + a_ss
    if not last:
        out["v_out"] = (x["v"].reshape(n, 3, f) + a_vv[:, None] * uv).reshape(n, 3 * f)
    g = x["gs_out"]
    ga = np.empty((n, na, f), np.float32)
    if not last:
        gdot = ((zero + gvo[:, 0] * uv[:, 0]) + gvo[:, 1] * uv[:, 1]) + gvo[:, 2] * uv[:, 2]
        ga[:, 0] = zero if "ga_without_gv_out" in mut else gdot
    ga[:, na - 2], ga[:, na - 1] = g * inner, g
    out["ga"] = ga.reshape(n, na * f)
    mi = out["mlp_in"] if mlp_in is None else mlp_in
    gn, nin = x["g_mlp_in"][:, :f], mi[:, :f]
    with np.errstate(divide="ignore", invalid="ignore"):
        q = gn / nin if "gn_over_at_zero" in mut else np.where(nin > 0, gn / np.where(nin > 0, nin, 1), zero).astype(np.float32)
    gsv = g * a_sv
    out["guv"] = (gsv[:, None] * vv + gvo * a_vv[:, None]).reshape(3 * n, f)
    out["gvv"] = (gsv[:, None] * uv + q[:, None] * vv).reshape(3 * n, f)
    out["gs"] = g + x["g_mlp_in"][:, f:]
    out["gv"] = gvo.reshape(n, 3 * f) + zero
    return out


def ref_steps(x, n, f, last, mlp_in):
    """fp64 values of every output of the four steps from the fp32 operands, and the bound each kernel output is held to"""
    d = {k: v.astype(np.float64) for k, v in x.items()}
    uv, vv = d["uv"].reshape(n, 3, f), d["vv"].reshape(n, 3, f)
    na = 2 if last else 3
    a = d["a"][:, :na * f].reshape(n, na, f)
    a_sv, a_ss = a[:, na - 2], a[:, na - 1]
    a_vv = a[:, 0] if not last else np.zeros_like(a_sv)
    gvo = d["gv_out"].reshape(n, 3, f) if not last else np.zeros((n, 3, f))
    nrm = np.sqrt((vv * vv).sum(1))
    inner = (uv * vv).sum(1)
    g = d["gs_out"]
    ref, bnd = {}, {}
    ref["mlp_in"] = np.concatenate([nrm, d["s"]], axis=1)
    bnd["mlp_in"] = np.concatenate([U * nrm, np.zeros_like(nrm)], axis=1)
    ref["s_out"] = d["s"] + a_sv * inner + a_ss
    if not last:
        ref["v_out"] = (d["v"].reshape(n, 3, f) + a_vv[:, None] * uv).reshape(n, 3 * f)
    ga = np.empty((n, na, f))
    if not last:
        ga[:, 0] = (gvo * uv).sum(1)
    ga[:, na - 2], ga[:, na - 1] = g * inner, g
    ref["ga"] = ga.reshape(n, na * f)
    nin = mlp_in[:, :f].astype(np.float64)
    q = np.where(nin > 0, d["g_mlp_in"][:, :f] / np.where(nin > 0, nin, 1), 0.0)
    gsv = (g * a_sv)[:, None]
    ref["guv"] = (gsv * vv + gvo * a_vv[:, None]).reshape(3 * n, f)
    ref["gvv"] = (gsv * uv + q[:, None] * vv).reshape(3 * n, f)
    bnd["gvv"] = (3 * U * (1 + 4 * U) * (np.abs(gsv * uv) + np.abs(q[:, None] * vv))).reshape(3 * n, f)
    ref["gs"] = g + d["g_mlp_in"][:, f:]
    ref["gv"] = gvo.reshape(n, 3 * f)
    for k in ref:
        bnd.setdefault(k, np.zeros_like(ref[k]))
    return ref, bnd


def check_steps(what, got, ref, bnd):
    assert set(got) <= set(ref), sorted(set(got) - set(ref))
    for k in got:
        bounded("steps", "%s: %s" % (what, k), got[k], ref[k], bnd[k])


def step_case(n, f, kind, last):
    x = step_inputs(n, f, seed=7919 * n + 31 * f + 3 * LAYOUTS.index(kind) + last)
    img = image(kind, x["uv"], x["vv"])
    mlp_in = emu_steps(x, img, n, f, last)["mlp_in"]         # bwd's |vv| operand: 0 exactly on the rows with vv = 0
    return x, img, mlp_in


# ---- GPU -------------------------------------------------------------------------------------------------------------------
def uv_bufs(kind, n, f, uv=None, vv=None):
    """buffers in the given layout: (list of Bufs, uv pointer, vv pointer, ld, reader of the two [3n, f] blocks)"""
    ld, col = layout(kind, f)
    if col is None:
        bu, bv = Buf(3 * n, f, data=uv), Buf(3 * n, f, data=vv)
        return [bu, bv], bu.ptr, bv.ptr, ld, lambda: (bu.np(), bv.np())
    full = None
    if uv is not None:
        full = np.full((3 * n, ld), np.nan, np.float32)
        full[:, :f], full[:, col:col + f] = uv, vv
    b = Buf(3 * n, ld, data=full)
    return [b], b.ptr, b.ptr + 4 * col, ld, lambda: (b.np()[:, :f], b.np()[:, col:col + f])


@pytest.mark.gpu
@pytest.mark.parametrize("last", [0, 1])
@pytest.mark.parametrize("n", N_STEP)
@pytest.mark.parametrize("kind", LAYOUTS)
@pytest.mark.parametrize("f", F_STEP)
def test_update_steps_bit_for_bit(f, kind, n, last):
    """pre_fwd, post_fwd, post_bwd_a, bwd with gv NULL and non-NULL: every output the fp32 restatement's bits and within its
    fp64 bound; a last layer leaves v_out unwritten and ignores gv_out (non-NULL here); the gap columns of ld = 2f + 5 untouched"""
    x, img, mlp_in = step_case(n, f, kind, last)
    want = emu_steps(x, img, n, f, last, mlp_in)
    ref, bnd = ref_steps(x, n, f, last, mlp_in)
    na = 2 if last else 3
    ins = dict(s=Buf(n, f, data=x["s"]), v=Buf(n, 3 * f, data=x["v"]), a=Buf(n, na * f, data=np.ascontiguousarray(x["a"][:, :na * f])),
               gs_out=Buf(n, f, data=x["gs_out"]), gv_out=Buf(n, 3 * f, data=x["gv_out"]), g_mlp_in=Buf(n, 2 * f, data=x["g_mlp_in"]),
               mlp_in=Buf(n, 2 * f, data=mlp_in))
    _, uvp, vvp, ld, _ = src = uv_bufs(kind, n, f, x["uv"], x["vv"])
    for with_gv in (False, True):
        what = "f=%d %s n=%d last=%d gv=%d" % (f, kind, n, last, with_gv)
        out = dict(mlp_in=Buf(n, 2 * f), s_out=Buf(n, f), v_out=Buf(n, 3 * f), ga=Buf(n, na * f), gs=Buf(n, f), gv=Buf(n, 3 * f))
        gbufs, guvp, gvvp, _, read_g = uv_bufs(kind, n, f)

        def run():
            st = stream()
            _lib.call("hgb_painn_update_pre_fwd", vvp, ld, ins["s"].ptr, n, f, out["mlp_in"].ptr, st)
            _lib.call("hgb_painn_update_post_fwd", ins["a"].ptr, uvp, vvp, ld, ins["s"].ptr, ins["v"].ptr, n, f, last,
                      out["s_out"].ptr, out["v_out"].ptr, st)
            _lib.call("hgb_painn_update_post_bwd_a", ins["gs_out"].ptr, ins["gv_out"].ptr, uvp, vvp, ld, n, f, last, out["ga"].ptr, st)
            _lib.call("hgb_painn_update_bwd", ins["gs_out"].ptr, ins["gv_out"].ptr, ins["g_mlp_in"].ptr, ins["a"].ptr, uvp, vvp, ld,
                      ins["mlp_in"].ptr, n, f, last, guvp, gvvp, out["gs"].ptr, out["gv"].ptr if with_gv else None, st)

        assert launches(run) == (4 if n else 0), what
        twice(what, run, list(out.values()) + gbufs)
        for k in ("mlp_in", "s_out", "ga", "gs"):
            out[k].check(what, k)
        out["v_out"].check(what, "v_out", written=not last)
        out["gv"].check(what, "gv", written=with_gv)
        ld_, col = layout(kind, f)
        if col is None:
            for b, k in zip(gbufs, ("guv", "gvv")):
                b.check(what, k)
        else:
            mask = torch.zeros(3 * n, ld_, dtype=torch.bool)
            mask[:, :f] = mask[:, col:col + f] = True
            gbufs[0].check(what, "[guv | gvv]", mask=mask)
            gap = gbufs[0].np()[:, f:col]
            assert np.isnan(gap).all(), "%s: the gap between guv and gvv was written" % what
        got = {k: out[k].np() for k in ("mlp_in", "s_out", "ga", "gs")}
        got["guv"], got["gvv"] = read_g()
        if not last:
            got["v_out"] = out["v_out"].np()
        if with_gv:
            got["gv"] = out["gv"].np()
        for k, val in got.items():
            same_f32("%s: %s" % (what, k), val, want[k])
        check_steps(what, got, ref, bnd)


# ================================================================================================================================
# running error analysis (sections 2 and 3)
# ================================================================================================================================
class R:
    """a value computed in fp64 from the kernel's fp32 operands, and a bound on how far the kernel's fp32 value of it can be"""

    def __init__(self, val, err=None):
        self.val = val
        self.err = torch.zeros_like(val) if err is None else err

    @staticmethod
    def lift(b):
        return b if isinstance(b, R) else R(torch.as_tensor(b, dtype=torch.float64))

    def __add__(self, b):
        b = R.lift(b)
        v = self.val + b.val
        e = self.err + b.err
        return R(v, e + U * (v.abs() + e))

    __radd__ = __add__

    def __neg__(self):
        return R(-self.val, self.err)

    def __sub__(self, b):
        return self + (-R.lift(b))

    def __rsub__(self, b):
        return R.lift(b) - self

    def __mul__(self, b):
        b = R.lift(b)
        v = self.val * b.val
        e = self.val.abs() * b.err + b.val.abs() * self.err + self.err * b.err
        return R(v, e + U * (v.abs() + e))

    __rmul__ = __mul__

    def __truediv__(self, b):
        b = R.lift(b)
        v = self.val / b.val
        e = (self.err + v.abs() * b.err) / (b.val.abs() - b.err)
        return R(v, e + U * (v.abs() + e))

    def __getitem__(self, i):
        return R(self.val[i], self.err[i])

    def sqrt(self):
        v = self.val.clamp_min(0).sqrt()
        e = torch.minimum(self.err.sqrt(), torch.where(v > 0, self.err / v.clamp_min(1e-300), torch.full_like(v, math.inf)))
        return R(v, e + U * (v + e))

    def sigmoid(self):
        """hgb_sigmoid: within (3 + 1.2 |x|) 2^-23 relative at the kernel's x, and Lipschitz 1/4 in x"""
        v = torch.sigmoid(self.val)
        e = 0.25 * self.err
        return R(v, e + (3 + 1.2 * (self.val.abs() + self.err)) * 2.0 ** -23 * (v + e))


def where0(mask, r):
    """mask ? r : 0 (the kernel takes an exact 0 on the other branch)"""
    return R(torch.where(mask, r.val, torch.zeros_like(r.val)), torch.where(mask, r.err, torch.zeros_like(r.err)))


class F32:
    """the same formulas in plain fp32 arithmetic: the restatement of the kernels"""
    sqrt = staticmethod(torch.sqrt)
    sigmoid = staticmethod(lambda x: 1.0 / (1.0 + torch.exp(-x)))
    where0 = staticmethod(lambda mask, x: torch.where(mask, x, torch.zeros_like(x)))


class F64:
    sqrt = staticmethod(R.sqrt)
    sigmoid = staticmethod(R.sigmoid)
    where0 = staticmethod(where0)


# ================================================================================================================================
# 2. the width-one kernel
# ================================================================================================================================
def scalar_block(M, s, v, p, last, gs_out, gv_out, mut=()):
    """the update block at width 1 as painn_update_scalar_{fwd,bwd}_kernel write it: s [n], v [n, 3], p: the 16 pack values.
    M = F32 (fp32 tensors: the restatement) or F64 (R values: fp64 and the bound).  -> outputs and, per pack slot, its terms"""
    na = 2 if last else 3
    nr = 3 if "pad_read" in mut else na         # pack slots of a the restatement reads
    uv = [p[0] * v[:, k] + p[1] for k in range(3)]
    vv = [p[2] * v[:, k] + p[3] for k in range(3)]
    n2 = (vv[0] * vv[0] + vv[1] * vv[1]) + vv[2] * vv[2]
    inner = (uv[0] * vv[0] + uv[1] * vv[1]) + uv[2] * vv[2]
    nrm = M.sqrt(n2)
    z1 = p[4] * nrm + (p[5] * s + p[6])
    sg = M.sigmoid(z1)
    h = z1 * sg
    a = [p[7 + j] * h + p[10 + j] for j in range(nr)]
    a_sv, a_ss = a[nr - 2], a[nr - 1]
    out = dict(s_out=(s + a_sv * inner) + a_ss)
    if not last:
        out["v_out"] = [a[0] * uv[k] + v[:, k] for k in range(3)]
    ga = [None] * na
    ga[na - 1], ga[na - 2] = gs_out, gs_out * inner
    if not last:
        ga[0] = (gv_out[:, 0] * uv[0] + gv_out[:, 1] * uv[1]) + gv_out[:, 2] * uv[2]
    gh = ga[0] * p[7]
    for j in range(1, na):
        gh = gh + ga[j] * p[7 + j]
    gz1 = (gh * sg) * (1.0 + z1 * (1.0 - sg))
    terms = {7 + j: [ga[j] * h] for j in range(na)}
    terms.update({10 + j: [ga[j]] for j in range(na)})
    terms.update({4: [gz1 * nrm], 5: [gz1 * s], 6: [gz1]})
    out["gs"] = gs_out + gz1 * p[5]
    gn_over = M.where0(nrm.val > 0 if isinstance(nrm, R) else nrm > 0, (gz1 * p[4]) / nrm)
    g_inner = gs_out * a_sv
    gv = []
    for q in range(4):
        terms[q] = []
    for k in range(3):
        guv = g_inner * vv[k] if last else gv_out[:, k] * a[0] + g_inner * vv[k]
        gvv = g_inner * uv[k] + gn_over * vv[k]
        gv.append((guv * p[0] + (gv_out[:, k] if not last else 0.0)) + gvv * p[2])
        terms[0].append(guv * v[:, k])
        terms[1].append(guv)
        terms[2].append(gvv * v[:, k])
        terms[3].append(gvv)
    out["gv"] = gv
    return out, terms


def scalar_inputs(n, last, seed, device):
    """fp32 s [n], v [n, 3], gs_out, gv_out and the 16-value pack with NaN in its unused slots; every 11th node has v = 0 and,
    for a last layer, vb = 0, so |Vv| = 0 exactly there"""
    g = torch.Generator().manual_seed(seed)
    s, v = torch.randn(n, generator=g), torch.randn(n, 3, generator=g)
    v[::11] = 0.0
    gs, gv = torch.randn(n, generator=g), torch.randn(n, 3, generator=g)
    p = torch.randn(16, generator=g) * 0.7
    if last:
        p[3] = 0.0
        p[[9, 12]] = float("nan")
    p[13:] = float("nan")
    return [t.to(device) for t in (s, v, gs, gv, p)]


def scalar_ref(s, v, gs, gv, p, last):
    """(outputs as R, {slot: (fp64 sum, bound on the kernel's reduced sum) for the used slots}) on the inputs' device"""
    d = lambda t: R(t.double())  # noqa: E731
    pk = [R(p[q].double().reshape(1).expand(s.shape[0]).clone()) for q in range(16)]
    out, terms = scalar_block(F64, d(s), d(v), pk, last, d(gs), d(gv))
    n = s.shape[0]
    nb = grid_for(n, 256, SCALAR_BWD_BLOCKS)
    per_thread = cdiv(n, nb * 256) if n else 0
    sums = {}
    for q, ts in terms.items():
        L = per_thread * len(ts) + 5 + 8 + nb
        val = sum(t.val.sum() for t in ts)
        err = sum(t.err.sum() for t in ts)
        mag = sum((t.val.abs() + t.err).sum() for t in ts)
        sums[q] = (float(val), float(err + gamma(L) * mag))
    return out, sums


def scalar_flat(out, last):
    """outputs as fp64 tensors (R values, or fp32 tensors) in the kernel's [n] / [n, 3] layout, with their bounds (R)"""
    def stack(x):
        return R(torch.stack([t.val for t in x], 1), torch.stack([t.err for t in x], 1)) if isinstance(x[0], R) else torch.stack(x, 1)
    res = dict(s_out=out["s_out"], gs=out["gs"], gv=stack(out["gv"]))
    if not last:
        res["v_out"] = stack(out["v_out"])
    return res


def check_scalar(what, got, gp, ref, sums, last):
    """got: {name: tensor}, gp: the 16-value gradient pack (or None)"""
    for k, r in scalar_flat(ref, last).items():
        bounded("scalar per-node", "%s: %s" % (what, k), got[k].double().cpu().numpy(), r.val.cpu().numpy(), r.err.cpu().numpy())
    if gp is not None:
        gp = gp.double().cpu().numpy()
        for q in range(16):
            if q in sums:
                bounded("scalar parameter gradients", "%s: gparams16[%d]" % (what, q), gp[q:q + 1], np.array([sums[q][0]]),
                        np.array([sums[q][1]]))
            else:
                assert gp[q] == 0.0, "%s: unused gradient slot %d is %r, not 0" % (what, q, gp[q])


def scalar_emu(s, v, gs, gv, p, last, mut=()):
    """fp32 restatement: outputs and the 16 reduced parameter gradients (fp64 sums of the fp32 terms, unused slots 0)"""
    pk = [p[q] for q in range(16)]
    out, terms = scalar_block(F32, s, v, pk, last, gs, gv, mut)
    gp = torch.zeros(16, dtype=torch.float64)
    for q, ts in terms.items():
        gp[q] = sum(t.double().sum() for t in ts)
    return scalar_flat(out, last), gp


@pytest.mark.gpu
@pytest.mark.parametrize("last", [0, 1])
@pytest.mark.parametrize("n", N_SCALAR)
def test_scalar_update_vs_fp64(n, last):
    what = "scalar n=%d last=%d" % (n, last)
    s, v, gs, gv, p = scalar_inputs(n, last, seed=n + 17 * last, device=DEV)
    bs, bv, bgs, bgv, bp = Buf(n, data=s), Buf(n, 3, data=v), Buf(n, data=gs), Buf(n, 3, data=gv), Buf(16, data=p)
    out = dict(s_out=Buf(n), v_out=Buf(n, 3), gs=Buf(n), gv=Buf(n, 3), gp=Buf(16))
    ws = ws_buf(_lib.query("hgb_painn_update_scalar_workspace_bytes"))

    def fwd():
        _lib.call("hgb_painn_update_scalar_fwd", bs.ptr, bv.ptr, bp.ptr, n, last, out["s_out"].ptr, out["v_out"].ptr, stream())

    def bwd():
        _lib.call("hgb_painn_update_scalar_bwd", bgs.ptr, bgv.ptr, bs.ptr, bv.ptr, bp.ptr, n, last, out["gs"].ptr, out["gv"].ptr,
                  out["gp"].ptr, ws.ptr, stream())

    assert launches(fwd) == (1 if n else 0), what
    assert launches(bwd) == (2 if n else 0), what
    twice(what, lambda: (fwd(), bwd()), list(out.values()))
    for k in ("s_out", "gs", "gv", "gp"):
        out[k].check(what, k)
    out["v_out"].check(what, "v_out", written=not last)
    if n == 0:
        assert bool((out["gp"].view == 0).all()), "%s: gparams16 is not zeroed" % what
        return
    ref, sums = scalar_ref(s, v, gs, gv, p, last)
    got = {k: out[k].view.reshape(n, -1).squeeze(1) if k in ("s_out", "gs") else out[k].view for k in ("s_out", "v_out", "gs", "gv")}
    check_scalar(what, got, out["gp"].view.reshape(16), ref, sums, last)


# ================================================================================================================================
# 3. the tensor-core update
# ================================================================================================================================
UF = 64


def tc_inputs(n, last, seed):
    """each entry's own random operands (fp32 on the GPU); the |vv| column of mlp_in is 0 on every 9th node"""
    g = torch.Generator().manual_seed(seed)
    na = 2 if last else 3
    r = lambda *sh, sc=1.0: (torch.randn(*sh, generator=g) * sc)  # noqa: E731
    x = dict(v=r(n, 3, UF), wuv=r(2 * UF, UF, sc=0.125), buv=r(2 * UF, sc=0.1), s=r(n, UF), a=r(n, na * UF), inner=r(n, UF),
             gs_out=r(n, UF), gv_out=r(n, 3, UF), g_mlp_in=r(n, 2 * UF), mlp_in=r(n, 2 * UF))
    x["v"][::13] = 0.0
    x["mlp_in"][:, :UF] = x["mlp_in"][:, :UF].abs()
    x["mlp_in"][::9, :UF] = 0.0
    return {k: t.to(DEV) for k, t in x.items()}


def tc_bufs(x):
    return {k: Buf(t.shape[0], t[0].numel() if t.dim() > 1 else 1, data=t) for k, t in x.items()}


def tc_linear_rows(a2, w, trans_b, bias, n_out, k_red, addend=None):
    """hgb_tc_linear in TF32 mode; fewer than 128 rows are zero-padded (rows are independent) to its minimum"""
    m = a2.shape[0]
    mp = max(m, 128)
    pad = lambda t: torch.cat([t, t.new_zeros(mp - m, t.shape[1])]) if mp > m else t.contiguous()  # noqa: E731
    with ops.tensor_cores(True):
        y, _ = ops.raw_tc_linear(pad(a2), w, trans_b, bias, n_out, k_red, addend=None if addend is None else pad(addend))
    return y[:m]


def tc_unfused(x, n, last):
    """the outputs of the four entries from the unfused pieces on the same operands"""
    na = 2 if last else 3
    y = tc_linear_rows(x["v"].reshape(3 * n, UF), x["wuv"], False, x["buv"], 2 * UF, UF)           # [3n, 128] = [uv | vv]
    st = stream()
    p = lambda t: t.data_ptr()  # noqa: E731
    out = dict(mlp_in=torch.empty(n, 2 * UF, device=DEV), s_out=torch.empty(n, UF, device=DEV), v_out=torch.empty(n, 3 * UF, device=DEV),
               ga=torch.empty(n, na * UF, device=DEV), g_uv=torch.empty(3 * n, 2 * UF, device=DEV), gs=torch.empty(n, UF, device=DEV),
               inner=torch.empty(n, UF, device=DEV))
    _lib.call("hgb_painn_update_pre_fwd", p(y) + 4 * UF, 2 * UF, p(x["s"]), n, UF, p(out["mlp_in"]), st)
    # inner as post_fwd accumulates it: s = -0, a = [1 | -0] gives s_out = inner, signed zeros included
    one = torch.cat([torch.ones(n, UF, device=DEV), torch.full((n, UF), -0.0, device=DEV)], 1)
    mzero = torch.full((n, UF), -0.0, device=DEV)
    _lib.call("hgb_painn_update_post_fwd", p(one), p(y), p(y) + 4 * UF, 2 * UF, p(mzero), None, n, UF, 1, p(out["inner"]), None, st)
    if last:        # the last-layer kernels read a given inner: uv = [inner; 0; 0], vv = [1; 0; 0] makes post_fwd's inner that one
        iu = torch.zeros(n, 3, 2 * UF, device=DEV)
        iu[:, 0, :UF], iu[:, 0, UF:] = x["inner"], 1.0
        yl = iu.reshape(3 * n, 2 * UF)
        _lib.call("hgb_painn_update_post_fwd", p(x["a"]), p(yl), p(yl) + 4 * UF, 2 * UF, p(x["s"]), None, n, UF, 1, p(out["s_out"]), None, st)
        _lib.call("hgb_painn_update_post_bwd_a", p(x["gs_out"]), None, p(yl), p(yl) + 4 * UF, 2 * UF, n, UF, 1, p(out["ga"]), st)
    else:
        _lib.call("hgb_painn_update_post_fwd", p(x["a"]), p(y), p(y) + 4 * UF, 2 * UF, p(x["s"]), p(x["v"]), n, UF, 0, p(out["s_out"]),
                  p(out["v_out"]), st)
        _lib.call("hgb_painn_update_post_bwd_a", p(x["gs_out"]), p(x["gv_out"]), p(y), p(y) + 4 * UF, 2 * UF, n, UF, 0, p(out["ga"]), st)
    _lib.call("hgb_painn_update_bwd", p(x["gs_out"]), None if last else p(x["gv_out"]), p(x["g_mlp_in"]), p(x["a"]), p(y), p(y) + 4 * UF,
              2 * UF, p(x["mlp_in"]), n, UF, last, p(out["g_uv"]), p(out["g_uv"]) + 4 * UF, p(out["gs"]), None, st)
    out["gv"] = tc_linear_rows(out["g_uv"], x["wuv"], True, None, UF, 2 * UF,
                               addend=None if last else x["gv_out"].reshape(3 * n, UF)).reshape(n, 3 * UF)
    torch.cuda.synchronize()
    return out


def tc_refs(x, n, last, g_uv):
    """fp64 references of the four entries (R); g_uv: the kernel's own [guv | gvv], the dgrad's operand"""
    d = lambda t: R(t.double())  # noqa: E731
    na = 2 if last else 3
    y = R(*tf32_gemm(x["v"].reshape(3 * n, UF), x["wuv"], x["buv"].expand(3 * n, 2 * UF), UF))
    uv = [R(y.val.reshape(n, 3, 2 * UF)[:, k, :UF], y.err.reshape(n, 3, 2 * UF)[:, k, :UF]) for k in range(3)]
    vv = [R(y.val.reshape(n, 3, 2 * UF)[:, k, UF:], y.err.reshape(n, 3, 2 * UF)[:, k, UF:]) for k in range(3)]
    inner = (uv[0] * vv[0] + uv[1] * vv[1]) + uv[2] * vv[2]
    ref = dict(nrm=((vv[0] * vv[0] + vv[1] * vv[1]) + vv[2] * vv[2]).sqrt(), inner=inner)
    a = [d(x["a"][:, j * UF:(j + 1) * UF]) for j in range(na)]
    s, g = d(x["s"]), d(x["gs_out"])
    gvo = [d(x["gv_out"][:, k]) for k in range(3)]
    if last:
        ref["s_out"] = (s + a[0] * d(x["inner"])) + a[1]
        ref["ga"] = [g * d(x["inner"]), g]
    else:
        ref["s_out"] = (s + a[1] * inner) + a[2]
        ref["v_out"] = [d(x["v"][:, k]) + a[0] * uv[k] for k in range(3)]
        ref["ga"] = [(gvo[0] * uv[0] + gvo[1] * uv[1]) + gvo[2] * uv[2], g * inner, g]
    ref["gs"] = g + d(x["g_mlp_in"][:, UF:])
    nrm = x["mlp_in"][:, :UF].double()
    q = where0(nrm > 0, d(x["g_mlp_in"][:, :UF]) / R(torch.where(nrm > 0, nrm, torch.ones_like(nrm))))
    gsv = g * a[na - 2]
    ref["guv"] = [gsv * vv[k] + (0.0 if last else gvo[k] * a[0]) for k in range(3)]
    ref["gvv"] = [gsv * uv[k] + q * vv[k] for k in range(3)]
    ref["gv"] = R(*tf32_gemm(g_uv, x["wuv"].t(), None if last else x["gv_out"].reshape(3 * n, UF), 2 * UF))
    return ref


def cat3(rs):
    return R(torch.stack([r.val for r in rs], 1), torch.stack([r.err for r in rs], 1))


def tc_fused(bufs, n, last, want_inner):
    na = 2 if last else 3
    out = dict(mlp_in=Buf(n, 2 * UF), inner=Buf(n, UF), s_out=Buf(n, UF), v_out=Buf(n, 3 * UF), ga=Buf(n, na * UF),
               g_uv=Buf(3 * n, 2 * UF), gs=Buf(n, UF), gv=Buf(n, 3 * UF))
    b = bufs
    st = stream()
    calls = [
        lambda: _lib.call("hgb_painn_update_tc_fwd", b["v"].ptr, b["s"].ptr, b["wuv"].ptr, b["buv"].ptr, n, out["mlp_in"].ptr,
                          out["inner"].ptr if want_inner else None, st),
        lambda: _lib.call("hgb_painn_update_tc_post", b["v"].ptr, b["s"].ptr, b["a"].ptr, b["inner"].ptr, b["wuv"].ptr, b["buv"].ptr, n,
                          last, out["s_out"].ptr, out["v_out"].ptr, st),
        lambda: _lib.call("hgb_painn_update_tc_bwd_a", b["v"].ptr, b["gs_out"].ptr, b["gv_out"].ptr, b["inner"].ptr, b["wuv"].ptr,
                          b["buv"].ptr, n, last, out["ga"].ptr, st),
        lambda: _lib.call("hgb_painn_update_tc_bwd", b["v"].ptr, b["gs_out"].ptr, None if last else b["gv_out"].ptr, b["g_mlp_in"].ptr,
                          b["a"].ptr, b["mlp_in"].ptr, b["wuv"].ptr, b["buv"].ptr, n, last, out["g_uv"].ptr, out["gs"].ptr, out["gv"].ptr, st),
    ]
    return out, calls


@pytest.mark.gpu
@pytest.mark.parametrize("want_inner", [False, True])
@pytest.mark.parametrize("last", [0, 1])
@pytest.mark.parametrize("n", N_TC)
def test_tc_update_entries(n, last, want_inner):
    what = "tc n=%d last=%d inner=%d" % (n, last, want_inner)
    x = tc_inputs(n, last, seed=3 * n + last)
    bufs = tc_bufs(x)
    out, calls = tc_fused(bufs, n, last, want_inner)
    for c in calls:
        assert launches(c) == 1, what
    twice(what, lambda: [c() for c in calls], list(out.values()))
    for k in ("mlp_in", "s_out", "ga", "g_uv", "gs", "gv"):
        out[k].check(what, k)
    out["inner"].check(what, "inner", written=want_inner)
    out["v_out"].check(what, "v_out", written=not last)
    # (i) the unfused pieces, bit for bit
    ref = tc_unfused(x, n, last)
    names = ["mlp_in", "s_out", "ga", "g_uv", "gs", "gv"] + (["inner"] if want_inner else []) + ([] if last else ["v_out"])
    for k in names:
        same_f32("%s: %s vs the unfused pieces" % (what, k), out[k].np(), ref[k].cpu().numpy())
    # (ii) fp64 of the TF32-rounded operands
    r = tc_refs(x, n, last, out["g_uv"].view)
    sec = "tensor-core update vs fp64"
    num = lambda t: t.cpu().numpy()  # noqa: E731

    def chk(name, got, rr):
        bounded(sec, "%s: %s" % (what, name), num(got.double()), num(rr.val), num(rr.err))

    mlp = out["mlp_in"].view
    chk("|vv|", mlp[:, :UF], r["nrm"])
    same_f32("%s: mlp_in[:, 64:] = s" % what, num(mlp[:, UF:]), num(x["s"]))
    if want_inner:
        chk("inner", out["inner"].view, r["inner"])
    chk("s_out", out["s_out"].view, r["s_out"])
    if not last:
        chk("v_out", out["v_out"].view.reshape(n, 3, UF), cat3(r["v_out"]))
    chk("ga", out["ga"].view.reshape(n, -1, UF), cat3(r["ga"]))
    chk("gs", out["gs"].view, r["gs"])
    guv = out["g_uv"].view.reshape(n, 3, 2 * UF)
    chk("guv", guv[:, :, :UF], cat3(r["guv"]))
    chk("gvv", guv[:, :, UF:], cat3(r["gvv"]))
    chk("gv", out["gv"].view.reshape(3 * n, UF), r["gv"])


@pytest.mark.gpu
def test_tc_update_refuses_misaligned_and_skips_empty():
    """a v 4 bytes past a 16-byte boundary is refused by every entry before anything launches; n = 0 launches nothing"""
    n = 256
    for last in (0, 1):
        x = tc_inputs(n, last, seed=99 + last)
        bufs = tc_bufs(x)
        bufs["v"] = Buf(n, 3 * UF, off=1, data=x["v"])
        out, calls = tc_fused(bufs, n, last, True)
        torch.cuda.synchronize()
        before = _lib.launch_count()
        for c in calls:
            with pytest.raises(RuntimeError, match="16-byte aligned"):
                c()
        torch.cuda.synchronize()
        assert _lib.launch_count() == before
        for k, b in out.items():
            b.check("misaligned last=%d" % last, k, written=False)
        out, calls = tc_fused(tc_bufs(x), 0, last, True)
        for c in calls:
            assert launches(c) == 0


# ================================================================================================================================
# 4. the modules at workload shapes
# ================================================================================================================================
BATCH_GRAPHS = {"qm9_painn": 16384, "gfm_pnaeq": 128}     # bench.py's saturating batch of each workload


@functools.lru_cache(maxsize=None)
def workload_nodes(name):
    from hydragnn_b200.synthetic import WORKLOADS, make_samples
    if "n" in WORKLOADS[name]:
        return WORKLOADS[name]["n"] * BATCH_GRAPHS[name]
    return int(make_samples(name, BATCH_GRAPHS[name]).batch.numel())


def oracle_grads(mod, s, v, ws, wv, last, pnaeq_block):
    """fp64 autograd of the oracle block with the module's parameters: outputs and the 10 gradients"""
    from oracle import painn as opainn
    from oracle import pnaeq as opnaeq
    f = s.shape[1]
    ref = (opnaeq.PainnUpdate if pnaeq_block else opainn.PainnUpdate)(f, bool(last)).double().to(DEV)
    with torch.no_grad():
        for a, b in zip(ref.parameters(), mod.parameters()):
            a.copy_(b.double())
    sr, vr = s.double().requires_grad_(True), v.double().requires_grad_(True)
    so, vo = ref(sr, vr)
    loss = (so * ws.double()).sum() + (0 if last else (vo * wv.double()).sum())
    grads = torch.autograd.grad(loss, [sr, vr] + list(ref.parameters()))
    return [so.detach(), None if last else vo.detach()] + list(grads)


def module_grads(mod, s, v, ws, wv, last, tc):
    se, ve = s.clone().requires_grad_(True), v.clone().requires_grad_(True)
    with ops.tensor_cores(tc):
        so, vo = mod(se, ve)
        loss = (so * ws).sum() + (0 if last else (vo * wv).sum())
        grads = torch.autograd.grad(loss, [se, ve] + list(mod.parameters()))
    torch.cuda.synchronize()
    return [so.detach(), None if last else vo.detach()] + list(grads)


NAMES = ["s_out", "v_out", "gs", "gv", "gUw", "gUb", "gVw", "gVb", "gW1", "gb1", "gW2", "gb2"]


def rel(a, b):
    a, b = a.double(), b.double()
    den = float(b.norm())
    return float((a - b).norm()) / den if den > 0 else float((a - b).abs().max())


WORKLOAD_CASES = [("qm9_painn", "stacks", 64, tc, last) for tc in (True, False) for last in (0, 1)]
WORKLOAD_CASES += [("qm9_painn", "stacks", 1, False, last) for last in (0, 1)]
WORKLOAD_CASES += [("gfm_pnaeq", "pnaeq", f, False, last) for f in (64, 1) for last in (0, 1)]


@pytest.mark.gpu
@pytest.mark.parametrize("workload,module,f,tc,last", WORKLOAD_CASES)
def test_update_module_at_workload_shape(workload, module, f, tc, last):
    n = workload_nodes(workload)
    torch.manual_seed(n + f + last)
    mod = (stacks if module == "stacks" else pnaeq).PainnUpdate(f, bool(last)).to(DEV)
    g = torch.Generator(device=DEV).manual_seed(f + 2 * last)
    s, v, ws, wv = (torch.randn(*sh, generator=g, device=DEV) for sh in ((n, f), (n, 3, f), (n, f), (n, 3, f)))
    got = module_grads(mod, s, v, ws, wv, last, tc)
    ref = oracle_grads(mod, s, v, ws, wv, last, module == "pnaeq")
    tol = 5e-3 if tc else FP32_TOL
    for name, a, b in zip(NAMES, got, ref):
        if b is None:
            continue
        assert bool(torch.isfinite(a).all()), name
        e = rel(a, b)
        _note("modules %s" % ("TF32" if tc else "fp32"), e / tol)
        assert e <= tol, "%s n=%d f=%d tc=%d last=%d: %s rel-L2 %.3g" % (workload, n, f, tc, last, name, e)


# ================================================================================================================================
# 5. the dispatch census
# ================================================================================================================================
TC_ENTRIES = {"hgb_painn_update_tc_fwd", "hgb_painn_update_tc_post", "hgb_painn_update_tc_bwd_a", "hgb_painn_update_tc_bwd"}
UNFUSED = {"hgb_painn_update_pre_fwd", "hgb_painn_update_post_fwd", "hgb_painn_update_post_bwd_a", "hgb_painn_update_bwd"}
SCALAR = {"hgb_painn_update_scalar_fwd", "hgb_painn_update_scalar_bwd"}


def instantiations(calls):
    """the kernels of hgb_painn_update_tc_* and the scalar reduce that the traced calls launched"""
    seen = set()
    for name, args, nl in calls:
        if nl == 0:
            continue
        last = bool(args.get("last", 1))
        if name == "hgb_painn_update_tc_fwd":
            seen.add("painn_update_tc_kernel<UPD_FWD, true>")
        elif name == "hgb_painn_update_tc_post":
            seen.add("painn_update_tc_post_last_kernel" if last else "painn_update_tc_kernel<UPD_POST, false>")
        elif name == "hgb_painn_update_tc_bwd_a":
            seen.add("painn_update_tc_bwd_a_last_kernel" if last else "painn_update_tc_kernel<UPD_BWD_A, false>")
        elif name == "hgb_painn_update_tc_bwd":
            seen.add("painn_update_tc_kernel<UPD_BWD, %s>" % ("true" if last else "false"))
        elif name == "hgb_painn_update_scalar_bwd" and nl == 2:
            seen.add("painn_update_scalar_reduce_kernel")
    return seen


ALL_INSTANTIATIONS = {"painn_update_tc_kernel<UPD_FWD, true>", "painn_update_tc_kernel<UPD_POST, false>",
                      "painn_update_tc_kernel<UPD_BWD_A, false>", "painn_update_tc_kernel<UPD_BWD, true>",
                      "painn_update_tc_kernel<UPD_BWD, false>", "painn_update_tc_post_last_kernel", "painn_update_tc_bwd_a_last_kernel",
                      "painn_update_scalar_reduce_kernel"}


@pytest.mark.gpu
def test_dispatch_census():
    cases = [("stacks", 1, 300, True, False, SCALAR), ("pnaeq", 1, 300, True, False, UNFUSED),
             ("stacks", 64, 256, True, False, TC_ENTRIES), ("stacks", 64, 256, False, False, UNFUSED),
             ("stacks", 64, 127, True, False, UNFUSED), ("stacks", 64, 256, True, True, UNFUSED)]
    seen = set()
    for module, f, n, tc, offset, want in cases:
        for last in (0, 1):
            torch.manual_seed(f + n)
            mod = (stacks if module == "stacks" else pnaeq).PainnUpdate(f, bool(last)).to(DEV)
            s = torch.randn(n * f + 1, device=DEV)
            s = (s[1:] if offset else s[:-1]).view(n, f)           # offset: an s view 4 bytes past the allocation
            v = torch.randn(n, 3, f, device=DEV)
            _lib.trace_begin()
            try:
                with ops.tensor_cores(tc):
                    so, vo = mod(s.detach().requires_grad_(True), v.requires_grad_(True))
                    (so.sum() + (0 if vo is None else vo.sum())).backward()
                torch.cuda.synchronize()
            finally:
                calls = _lib.trace_end()
            used = {name for name, _, _ in calls} & (TC_ENTRIES | UNFUSED | SCALAR)
            assert used == want, (module, f, n, tc, offset, last, sorted(used))
            seen |= instantiations(calls)
    assert seen == ALL_INSTANTIATIONS, sorted(ALL_INSTANTIATIONS - seen)


# ================================================================================================================================
# 6. no GPU: references against the oracle, and mutations
# ================================================================================================================================
def _oracle_block(f, last, seed):
    from oracle.painn import PainnUpdate
    torch.manual_seed(seed)
    m = PainnUpdate(f, bool(last)).double()
    n = 41
    s, v = torch.randn(n, f, dtype=torch.float64), torch.randn(n, 3, f, dtype=torch.float64)
    v[::7] = 0.0
    with torch.no_grad():
        m.update_V.bias[: max(1, f // 2)] = 0.0                 # |vv| = 0 on the zero rows of those channels
    return m, s, v


@pytest.mark.parametrize("last", [0, 1])
@pytest.mark.parametrize("f", [1, 5])
def test_step_references_compose_to_the_oracle(f, last):
    """ref_steps (fp64) and emu_steps (fp32), chained with the U/V product, update_mlp and the U/V dgrad, give the oracle block's
    outputs and the gradients of s and v (torch autograd, fp64)"""
    m, s, v = _oracle_block(f, last, seed=f + 10 * last)
    n = s.shape[0]
    gs_out, gv_out = torch.randn(n, f, dtype=torch.float64), torch.randn(n, 3, f, dtype=torch.float64)
    sr, vr = s.clone().requires_grad_(True), v.clone().requires_grad_(True)
    so, vo = m(sr, vr)
    want = torch.autograd.grad(so, [sr, vr], gs_out, retain_graph=True) if last else \
        torch.autograd.grad((so, vo), [sr, vr], (gs_out, gv_out))
    wuv = torch.cat([m.update_U.weight, m.update_V.weight]).detach()
    buv = torch.cat([m.update_U.bias, m.update_V.bias]).detach()
    y = (v.reshape(3 * n, f) @ wuv.t() + buv).detach()
    for dt, tol in ((np.float64, 1e-12), (np.float32, 1e-4)):
        x = dict(uv=y[:, :f].numpy(), vv=y[:, f:].numpy(), s=s.numpy(), v=v.reshape(n, 3 * f).numpy(), gs_out=gs_out.numpy(),
                 gv_out=gv_out.reshape(n, 3 * f).numpy())
        x = {k: val.astype(dt) for k, val in x.items()}
        # the MLP between the steps: torch autograd on the steps' own mlp_in
        if dt == np.float64:
            mlp_in = ref_steps(dict(x, a=np.zeros((n, 3 * f)), g_mlp_in=np.zeros((n, 2 * f))), n, f, last,
                               np.ones((n, 2 * f)))[0]["mlp_in"]
        else:
            mlp_in = emu_steps(dict(x, a=np.zeros((n, 3 * f), dt), g_mlp_in=np.zeros((n, 2 * f), dt)), image("prod", x["uv"], x["vv"]),
                               n, f, last)["mlp_in"]
        mi = torch.tensor(mlp_in, dtype=torch.float64, requires_grad=True)
        a = m.update_mlp(mi)
        na = 2 if last else 3
        x["a"] = np.concatenate([a.detach().numpy(), np.zeros((n, (3 - na) * f))], 1).astype(dt)
        if dt == np.float64:
            fwd, _ = ref_steps(dict(x, g_mlp_in=np.zeros((n, 2 * f))), n, f, last, mlp_in)
        else:
            fwd = emu_steps(dict(x, g_mlp_in=np.zeros((n, 2 * f), dt)), image("pad", x["uv"], x["vv"]), n, f, last)
        np.testing.assert_allclose(fwd["s_out"], so.detach().numpy(), rtol=tol, atol=tol)
        if not last:
            np.testing.assert_allclose(fwd["v_out"], vo.detach().reshape(n, 3 * f).numpy(), rtol=tol, atol=tol)
        ga = torch.tensor(fwd["ga"], dtype=torch.float64)
        g_mlp_in, = torch.autograd.grad(a, mi, ga)
        x["g_mlp_in"] = g_mlp_in.numpy().astype(dt)
        if dt == np.float64:
            bwd, _ = ref_steps(x, n, f, last, mlp_in)
        else:
            bwd = emu_steps(x, image("sep", x["uv"], x["vv"]), n, f, last, mlp_in)
        g_uv = np.concatenate([bwd["guv"], bwd["gvv"]], 1).astype(np.float64)
        gv = (torch.tensor(g_uv) @ wuv).reshape(n, 3, f).numpy() + bwd["gv"].reshape(n, 3, f)
        np.testing.assert_allclose(bwd["gs"], want[0].numpy(), rtol=tol, atol=tol)
        np.testing.assert_allclose(gv, want[1].numpy(), rtol=tol, atol=tol)


@pytest.mark.parametrize("last", [0, 1])
def test_scalar_references_match_the_oracle(last):
    """scalar_block in fp64 (the R values) and in fp32 against torch autograd of oracle.painn.PainnUpdate(1, last)"""
    from oracle.painn import PainnUpdate
    s, v, gs, gv, p = scalar_inputs(300, last, seed=5 + last, device="cpu")
    m = PainnUpdate(1, bool(last)).double()
    na = 2 if last else 3
    pd = p.double()
    with torch.no_grad():
        for t, val in ((m.update_U.weight, pd[0:1]), (m.update_U.bias, pd[1:2]), (m.update_V.weight, pd[2:3]), (m.update_V.bias, pd[3:4]),
                       (m.update_mlp[0].weight, pd[4:6]), (m.update_mlp[0].bias, pd[6:7]), (m.update_mlp[2].weight, pd[7:7 + na]),
                       (m.update_mlp[2].bias, pd[10:10 + na])):
            t.copy_(val.reshape(t.shape))
    sr, vr = s.double().reshape(-1, 1).requires_grad_(True), v.double().reshape(-1, 3, 1).requires_grad_(True)
    so, vo = m(sr, vr)
    loss = (so.reshape(-1) * gs.double()).sum() + (0 if last else (vo.reshape(-1, 3) * gv.double()).sum())
    grads = torch.autograd.grad(loss, [sr, vr] + list(m.parameters()))
    slots = [[0], [1], [2], [3], [4, 5], [6], list(range(7, 7 + na)), list(range(10, 10 + na))]
    ref, sums = scalar_ref(s, v, gs, gv, p, last)
    flat = scalar_flat(ref, last)
    torch.testing.assert_close(flat["s_out"].val, so.detach().reshape(-1), rtol=1e-12, atol=1e-12)
    if not last:
        torch.testing.assert_close(flat["v_out"].val, vo.detach().reshape(-1, 3), rtol=1e-12, atol=1e-12)
    torch.testing.assert_close(flat["gs"].val, grads[0].reshape(-1), rtol=1e-12, atol=1e-12)
    torch.testing.assert_close(flat["gv"].val, grads[1].reshape(-1, 3), rtol=1e-12, atol=1e-12)
    for sl, gr in zip(slots, grads[2:]):
        torch.testing.assert_close(torch.tensor([sums[q][0] for q in sl], dtype=torch.float64), gr.reshape(-1), rtol=1e-10, atol=1e-10)
    emu, gp = scalar_emu(s, v, gs, gv, p, last)
    check_scalar("fp32 restatement last=%d" % last, emu, gp, ref, sums, last)


MUTATIONS = ("sv_ss_swapped", "avv_when_last", "ga_without_gv_out", "gn_over_at_zero", "ld_as_f", "pad_read")


def mutation_runs():
    """{mutation: thunks, each comparing one case of a wrong fp32 restatement with fp64; None: the faithful restatements}"""
    runs = {m: [] for m in (None,) + MUTATIONS}
    for f, kind, n, last in ((3, "pad", 77, 0), (3, "pad", 77, 1), (64, "prod", 40, 0), (64, "prod", 40, 1)):
        x, img, mlp_in = step_case(n, f, kind, last)
        ref, bnd = ref_steps(x, n, f, last, mlp_in)
        for m in (None,) + MUTATIONS[:5]:
            runs[m].append(lambda x=x, img=img, n=n, f=f, last=last, mlp_in=mlp_in, ref=ref, bnd=bnd, m=m: check_steps(
                "steps f=%d %s last=%d" % (f, kind, last), emu_steps(x, img, n, f, last, mlp_in, mut=(m,)), ref, bnd))
    for last in (0, 1):
        s, v, gs, gv, p = scalar_inputs(300, last, seed=11 + last, device="cpu")
        ref, sums = scalar_ref(s, v, gs, gv, p, last)
        for m in (None, "pad_read"):
            runs[m].append(lambda a=(s, v, gs, gv, p, last), ref=ref, sums=sums, last=last, m=m: check_scalar(
                "scalar last=%d" % last, *scalar_emu(*a, mut=(m,)), ref, sums, last))
    return runs


def test_mutations_are_caught():
    saved = dict(RATIOS)
    try:
        _mutations_are_caught()
    finally:
        RATIOS.clear()
        RATIOS.update(saved)


def _mutations_are_caught():
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
