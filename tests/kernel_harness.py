"""The guard-row harness of the kernel tests that call the C-ABI directly (test_gpu_graph_primitives.py,
test_gpu_conv_kernels.py).  Every operand is the leading block of a buffer filled with NaN (floating point) or SENTINEL
(integers), followed by GUARD rows of the same fill; `Buf.check` asserts that every element in range was written and every
other element kept its fill bits.  Importing this module needs no GPU: only the harness calls touch the device."""
import numpy as np
import pytest
import torch

from hydragnn_b200 import _lib, ops

DEV = "cuda"
GUARD = 3                            # fill rows after every buffer
NAN_BITS = 0x7FC00000                # torch.full(nan) fp32
SENTINEL = 0x7F7F7F7F                # integer fill
U = 2.0 ** -24
NUM_SMS = 132                        # HGB_NUM_SMS
GRID_CAP = NUM_SMS * 16              # hgb_grid_for's block cap


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
