"""The guard-row harness of the kernel tests that call the C-ABI directly (test_gpu_graph_primitives.py,
test_gpu_conv_kernels.py, test_gpu_tc_kernels.py, ...).  Every operand is the leading block of a buffer filled with NaN (floating point) or SENTINEL
(integers), followed by GUARD rows of the same fill; `Buf.check` asserts that every element in range was written and every
other element kept its fill bits.  Importing this module needs no GPU: only the harness calls touch the device.

It also holds the fp64 references and error terms more than one kernel test uses: the activations and their derivatives with
`act_eval_err` (the bound on a kernel's fp32 evaluation of them, test_gpu_dense_kernels.py's docstring), the random-walk
witness `l2_bound`, and `tf32_gemm` with TF32_OPERAND for the tensor cores' TF32 mode."""
import math

import numpy as np
import pytest
import torch

from hydragnn_b200 import _lib, ops
from oracle.tf32 import _round_tf32

DEV = "cuda"
GUARD = 3                            # fill rows after every buffer
NAN_BITS = 0x7FC00000                # torch.full(nan) fp32
SENTINEL = 0x7F7F7F7F                # integer fill
U = 2.0 ** -24
NUM_SMS = 132                        # HGB_NUM_SMS
GRID_CAP = NUM_SMS * 16              # hgb_grid_for's block cap
SELU_A, SELU_S = 1.6732632423543772848170429916717, 1.0507009873554804934193349852946
EXP_FLOOR = 2.0 ** -120
LRELU_P = float(np.float32(0.1))     # the fp32 parameter the kernels receive
ACT = dict(none=0, relu=1, silu=2, tanh=3, sigmoid=4, lrelu=5, elu=6, selu=7)
DERIV = 100
EXP_CODES = (ACT["silu"], ACT["sigmoid"], ACT["elu"], ACT["selu"])
LIP = {0: 1.0, 1: 1.0, 2: 1.0999, 3: 1.0, 4: 0.25, 5: 1.0, 6: 1.0, 7: 1.7581}        # max |act'|
LIP1 = {0: 0.0, 1: 0.0, 2: 0.5, 3: 0.77, 4: 0.1, 5: 0.0, 6: 1.0, 7: 1.7581}         # max |act''|
# The tensor cores take the leading 19 bits of an fp32 operand (truncation, test_gpu_tc.py), within one TF32 ulp (2^-10
# relative) of _round_tf32's nearest value; over both operands of a product that is 2^-9 (1 + 2^-9) of |product|.  With this term
# at 0 the worst |error| / bound of test_gpu_painn_update_kernels.py was 92 on an H100: the conversion, not the accumulation,
# dominates.
TF32_OPERAND = 2.0 ** -9 * (1 + 2.0 ** -9)


def cdiv(a, b):
    return -(-a // b)


def gamma(L):
    return L * U / (1 - L * U)


def grid_for(work, per_block, cap=GRID_CAP):
    """hgb_grid_for: enough blocks for `work` items at `per_block` each, at least 1, at most `cap`"""
    return min(max(cdiv(work, per_block), 1), cap)


def _fill_value(dtype):
    return float("nan") if dtype.is_floating_point else SENTINEL


class Buf:
    """rows x cols block (row stride ld, first element `off` elements into the allocation) of a filled buffer with GUARD rows"""

    def __init__(self, rows, cols=1, ld=None, off=0, data=None, dtype=torch.float32):
        self.rows, self.cols, self.dtype = rows, cols, dtype
        self.ld = max(cols, 1) if ld is None else ld
        self.off = off
        self.base = torch.full((off + (rows + GUARD) * self.ld,), _fill_value(dtype), dtype=dtype, device=DEV)
        self.view = self.base[off:off + rows * self.ld].view(rows, self.ld)[:, :cols]
        if data is not None:
            self.view.copy_(torch.as_tensor(data).reshape(rows, cols))

    @property
    def ptr(self):
        return self.base.data_ptr() + self.base.element_size() * self.off

    def _mask(self):
        mask = torch.zeros_like(self.base, dtype=torch.bool)
        mask[self.off:self.off + self.rows * self.ld].view(self.rows, self.ld)[:, :self.cols] = True
        return mask

    def _bits(self, t):
        return t.view(torch.int32 if t.element_size() == 4 else torch.int64)

    def check(self, what, name, written=True, mask=None):
        """written: every element of the block (or of `mask`) was written; always: everything else keeps its fill bits"""
        block = self._mask()
        fill = self._bits(torch.full((1,), _fill_value(self.dtype), dtype=self.dtype, device=DEV))
        if written:
            sel = block if mask is None else block.clone().masked_scatter_(block, mask.to(DEV).reshape(-1))
            vals = self.base[sel]
            bad = int((~torch.isfinite(vals)).sum()) if self.dtype.is_floating_point else int((self._bits(vals) == fill).sum())
            assert bad == 0, "%s: %s has %d unwritten or non-finite entries" % (what, name, bad)
        outside = self._bits(self.base[~block])
        assert bool((outside == fill).all()), "%s: %s written outside its block (%d entries)" % (what, name, int((outside != fill).sum()))

    def np(self):
        return self.view.cpu().numpy()


def ws_buf(nbytes):
    return Buf(max(cdiv(int(nbytes), 4), 1))


def launches(fn):
    torch.cuda.synchronize()
    before = _lib.launch_count()
    fn()
    torch.cuda.synchronize()
    return _lib.launch_count() - before


def twice(what, fn, outs):
    """run fn, snapshot outs, run again: the same bits"""
    first = [o.base.clone() for o in outs]
    fn()
    torch.cuda.synchronize()
    for o, f in zip(outs, first):
        assert torch.equal(o.base.view(torch.uint8), f.view(torch.uint8)), "%s: two identical calls differ" % what


def stream():
    return ops._stream()


def check_bound(what, got, ref, bound):
    err = np.abs(np.asarray(got, np.float64) - ref)
    bad = err > bound + 2.0 ** -126
    if bad.any():
        i = int(np.argmax(np.where(bad, err / np.maximum(bound, 1e-300), 0)))
        pytest.fail("%s: %d of %d entries off their bound; worst flat index %d: |err| %.3g, bound %.3g, ref %.8g, got %.8g"
                    % (what, int(bad.sum()), bad.size, i, err.flat[i], np.broadcast_to(bound, err.shape).flat[i], ref.flat[i],
                       np.asarray(got).flat[i]))


def same_f32(what, got, ref):
    got, ref = np.asarray(got, np.float32), np.asarray(ref, np.float32)
    if not np.array_equal(got.view(np.int32), ref.view(np.int32)):
        bad = got.view(np.int32) != ref.view(np.int32)
        i = int(np.argmax(bad))
        pytest.fail("%s: %d of %d entries differ from the fp32 restatement; first flat index %d: %.9g vs %.9g"
                    % (what, int(bad.sum()), bad.size, i, got.flat[i], ref.flat[i]))


# ---- fp64 references shared by the kernel tests -------------------------------------------------------------------------------
def act64(z, code, p=LRELU_P):
    if code == ACT["relu"]:
        return torch.where(z > 0, z, torch.zeros_like(z))
    if code == ACT["silu"]:
        return z * torch.sigmoid(z)
    if code == ACT["tanh"]:
        return torch.tanh(z)
    if code == ACT["sigmoid"]:
        return torch.sigmoid(z)
    if code == ACT["lrelu"]:
        return torch.where(z > 0, z, p * z)
    if code == ACT["elu"]:
        return torch.where(z > 0, z, torch.expm1(z))
    if code == ACT["selu"]:
        return SELU_S * torch.where(z > 0, z, SELU_A * torch.expm1(z))
    return z


def deriv64(x, code, order, p=LRELU_P):
    """order-th derivative at x; at the kinks x = 0 the kernel's convention: x > 0 takes the right branch, else the left"""
    if order == 0:
        return act64(x, code, p)
    one, zero = torch.ones_like(x), torch.zeros_like(x)
    pos = x > 0
    if code == ACT["relu"]:
        return torch.where(pos, one, zero) if order == 1 else zero
    if code == ACT["lrelu"]:
        return torch.where(pos, one, p * one) if order == 1 else zero
    if code == ACT["silu"]:
        s = torch.sigmoid(x)
        return s * (1 + x * (1 - s)) if order == 1 else s * (1 - s) * (2 + x * (1 - 2 * s))
    if code == ACT["tanh"]:
        t = torch.tanh(x)
        return 1 - t * t if order == 1 else -2 * t * (1 - t * t)
    if code == ACT["sigmoid"]:
        s = torch.sigmoid(x)
        return s * (1 - s) if order == 1 else s * (1 - s) * (1 - 2 * s)
    if code == ACT["elu"]:
        return torch.where(pos, one if order == 1 else zero, torch.exp(x))
    if code == ACT["selu"]:
        return torch.where(pos, SELU_S * one if order == 1 else zero, SELU_S * SELU_A * torch.exp(x))
    return one if order == 1 else zero


def deriv_terms(x, code, order, p=LRELU_P):
    """magnitude of the terms of the formula the kernel evaluates for the order-th derivative at x"""
    if order == 0:
        return act64(x, code, p).abs() + (x.abs() if code in (ACT["silu"], ACT["lrelu"]) else 0)
    a = x.abs()
    if code == ACT["silu"]:
        s = torch.sigmoid(x)
        return s * (1 + a * (1 + 2 * s)) if order == 1 else s * (1 + s) * (2 + a * (1 + 2 * s))
    if code == ACT["tanh"]:
        t = torch.tanh(x).abs()
        return 1 + t * t if order == 1 else 2 * t * (1 + t * t)
    if code == ACT["sigmoid"]:
        s = torch.sigmoid(x)
        return s * (1 + s) if order == 1 else s * (1 + s) * (1 + 2 * s)
    return deriv64(x, code, order, p).abs()


def act_eval_err(x, code, order=0, p=LRELU_P):
    """bound on the error of the kernel's fp32 evaluation of the order-th derivative at the fp32 argument x (module docstring)"""
    if code in (ACT["none"], ACT["relu"]) or (code == ACT["lrelu"] and order > 0):
        return torch.zeros_like(x)
    e = (12 + 2.4 * x.abs()) * U * deriv_terms(x, code, order, p)
    return e + (EXP_FLOOR if code in EXP_CODES else 0.0)


def grad_from(y, z, code, p=LRELU_P):
    """hgb_act_grad: act' from the activation output y (from z for SiLU; z itself for HGB_ACT_DERIV), in fp64"""
    if code == DERIV:
        return z
    if code == ACT["silu"]:
        return deriv64(z, code, 1)
    if code == ACT["relu"]:
        return (y > 0).double()
    if code == ACT["tanh"]:
        return 1 - y * y
    if code == ACT["sigmoid"]:
        return y * (1 - y)
    if code == ACT["lrelu"]:
        return torch.where(y > 0, torch.ones_like(y), p * torch.ones_like(y))
    if code == ACT["elu"]:
        return torch.where(y > 0, torch.ones_like(y), y + 1)
    if code == ACT["selu"]:
        return torch.where(y > 0, SELU_S * torch.ones_like(y), y + SELU_S * SELU_A)
    return torch.ones_like(y)


def grad_from_err(y, z, code, p=LRELU_P):
    """bound on the fp32 evaluation error of hgb_act_grad (without the product with dy)"""
    if code in (ACT["none"], ACT["relu"], ACT["lrelu"]):
        return torch.zeros_like(y)
    if code == DERIV:
        return torch.zeros_like(z)
    if code == ACT["silu"]:
        return act_eval_err(z, code, 1)
    m = {ACT["tanh"]: 1 + y * y, ACT["sigmoid"]: y.abs() * (1 + y.abs()), ACT["elu"]: 1 + y.abs(),
         ACT["selu"]: y.abs() + SELU_S * SELU_A}[code]
    return 4 * U * m


def l2_bound(L, mag, extra=None):
    """3 u sqrt(L) ||mag|| (+ ||extra||): the random-walk model of the module docstring"""
    b = 3 * U * math.sqrt(max(L, 1)) * float(mag.norm())
    return b + (float(extra.norm()) if extra is not None else 0.0)


def tf32_gemm(a, w, c, k):
    """(value, bound) of a @ w^T + c as the tensor cores' TF32 mode computes it: fp64 of the TF32-rounded operands, and the bound
    gamma(k + 2) (sum |a w| + |c|) + TF32_OPERAND sum |a w| on the kernel's distance from it"""
    ta, tw = _round_tf32(a.float()).double(), _round_tf32(w.float()).double()
    mag = ta.abs() @ tw.abs().t()
    cc = torch.zeros_like(mag) if c is None else c.double()
    return ta @ tw.t() + cc, gamma(k + 2) * (mag + cc.abs()) + TF32_OPERAND * mag
