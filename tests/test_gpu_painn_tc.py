"""GPU tests of the tensor-core PaiNN update block (PainnUpdateTcFn, csrc/hgb_painn_tc.cu).
It recomputes [uv | vv] from v with the products tc_linear runs and the elementwise formulas of the painn_update_* kernels, so in
TF32 mode it must give the same bits as PainnUpdateFn, its reference.  Against fp64 one TF32 GEMM stays within rel-L2 2e-3
(tests/test_gpu_tc.py); gv and the U/V weight gradient sit at the end of a chain of five (U/V, two MLP Linears, their two dgrads)
and reach 2.9e-3 in PainnUpdateFn as well, so the block is held to 5e-3."""
import pytest
import torch

pytestmark = pytest.mark.gpu

from hydragnn_b200 import _lib, ops  # noqa: E402
from hydragnn_b200.stacks import PainnUpdate  # noqa: E402

DEV = "cuda"


def rel(a, b):
    return float((a.double().cpu() - b.double().cpu()).norm() / b.double().cpu().norm())


def make_case(n, last, seed, f=64, zero_rows=0):
    g = torch.Generator().manual_seed(seed)
    torch.manual_seed(seed)
    upd = PainnUpdate(f, last).to(DEV)
    s, v = torch.randn(n, f, generator=g), torch.randn(n, 3, f, generator=g)
    if zero_rows:                                       # |vv| = 0 exactly: zero v rows and a zero V bias
        v[:zero_rows] = 0.0
        with torch.no_grad():
            upd.update_V.bias.zero_()
    ws, wv = torch.randn(n, f, generator=g), torch.randn(n, 3, f, generator=g)
    return upd, s.to(DEV), v.to(DEV), ws.to(DEV), wv.to(DEV)


def run(fn, upd, s, v, ws, wv, last):
    """(s_out, v_out, gs, gv, 8 parameter gradients) of the block through ``fn`` in TF32 mode"""
    se, ve = s.clone().requires_grad_(True), v.clone().requires_grad_(True)
    params = [upd.update_U.weight, upd.update_U.bias, upd.update_V.weight, upd.update_V.bias, upd.update_mlp[0].weight,
              upd.update_mlp[0].bias, upd.update_mlp[2].weight, upd.update_mlp[2].bias]
    with ops.tensor_cores(True):
        s1, v1 = fn.apply(se, ve, *params, last)
        loss = (s1 * ws).sum() + (0 if last else (v1 * wv).sum())
        grads = torch.autograd.grad(loss, [se, ve] + params)
    torch.cuda.synchronize()
    return [s1.detach(), None if last else v1.detach()] + list(grads)


def oracle64(upd, s, v, ws, wv, last):
    """the block in fp64 (PAINNStack.py:298-328) and its gradients"""
    p = [t.detach().double().cpu().requires_grad_(True) for t in
         (upd.update_U.weight, upd.update_U.bias, upd.update_V.weight, upd.update_V.bias, upd.update_mlp[0].weight,
          upd.update_mlp[0].bias, upd.update_mlp[2].weight, upd.update_mlp[2].bias)]
    sr, vr = s.double().cpu().requires_grad_(True), v.double().cpu().requires_grad_(True)
    uv, vv = vr @ p[0].t() + p[1], vr @ p[2].t() + p[3]
    a = torch.nn.functional.silu(torch.cat([torch.linalg.norm(vv, dim=1), sr], dim=1) @ p[4].t() + p[5]) @ p[6].t() + p[7]
    inner = (uv * vv).sum(dim=1)
    f = s.shape[1]
    if last:
        a_sv, a_ss = torch.split(a, f, dim=1)
        so, vo = sr + a_sv * inner + a_ss, None
        loss = (so * ws.double().cpu()).sum()
    else:
        a_vv, a_sv, a_ss = torch.split(a, f, dim=1)
        so, vo = sr + a_sv * inner + a_ss, vr + a_vv.unsqueeze(1) * uv
        loss = (so * ws.double().cpu()).sum() + (vo * wv.double().cpu()).sum()
    grads = torch.autograd.grad(loss, [sr, vr] + p)
    return [so.detach(), None if last else vo.detach()] + list(grads)


NAMES = ["s_out", "v_out", "gs", "gv", "gUw", "gUb", "gVw", "gVb", "gW1", "gb1", "gW2", "gb2"]


@pytest.mark.parametrize("last", [True, False])
@pytest.mark.parametrize("n,zero_rows", [(128, 0), (129, 0), (64 * 264 + 1, 0), (100003, 0), (4099, 100)])
def test_painn_update_tc_same_bits_as_unfused(n, zero_rows, last):
    """with zero_rows, |vv| = 0 exactly on those rows: the rule nrm > 0 ? gn / nrm : 0 must match too"""
    upd, s, v, ws, wv = make_case(n, last, seed=n + int(last), zero_rows=zero_rows)
    fused = run(ops.PainnUpdateTcFn, upd, s, v, ws, wv, last)
    ref = run(ops.PainnUpdateFn, upd, s, v, ws, wv, last)
    again = run(ops.PainnUpdateTcFn, upd, s, v, ws, wv, last)
    for name, x, r, y in zip(NAMES, fused, ref, again):
        if r is None:
            continue
        # bit patterns, so that +0 and -0 count as different
        assert torch.equal(x.view(torch.int32), r.view(torch.int32)), "%s differs from PainnUpdateFn: rel-L2 %.3g" % (name, rel(x, r))
        assert torch.equal(x.view(torch.int32), y.view(torch.int32)), "%s differs between two runs" % name


@pytest.mark.parametrize("last", [True, False])
@pytest.mark.parametrize("n,zero_rows", [(1000, 0), (4099, 100)])
def test_painn_update_tc_vs_fp64(n, zero_rows, last):
    """the block's TF32 tolerance against fp64; with zero_rows, |vv| = 0 exactly on those rows (the gradient rule
    nrm > 0 ? gn / nrm : 0)"""
    upd, s, v, ws, wv = make_case(n, last, seed=7 * n + zero_rows, zero_rows=zero_rows)
    fused = run(ops.PainnUpdateTcFn, upd, s, v, ws, wv, last)
    ref = oracle64(upd, s, v, ws, wv, last)
    for name, x, r in zip(NAMES, fused, ref):
        if r is None:
            continue
        assert torch.isfinite(x).all(), name
        assert rel(x, r) <= 5e-3, "%s: rel-L2 %.3g" % (name, rel(x, r))
    if zero_rows:
        assert rel(fused[3][:zero_rows], ref[3][:zero_rows]) <= 5e-3


def _entries(upd, s, v, tc):
    _lib.trace_begin()
    try:
        with ops.tensor_cores(tc):
            s1, v1 = upd(s.requires_grad_(True), v.requires_grad_(True))
            (s1.sum() + (0 if v1 is None else v1.sum())).backward()
        torch.cuda.synchronize()
    finally:
        calls = _lib.trace_end()
    return {name for name, _, _ in calls}


@pytest.mark.parametrize("last", [True, False])
def test_painn_update_dispatch(last):
    """PainnUpdate runs the tensor-core block only in TF32 mode at f = 64 with >= 128 rows; otherwise PainnUpdateFn"""
    tc_entries = {"hgb_painn_update_tc_fwd", "hgb_painn_update_tc_post", "hgb_painn_update_tc_bwd_a", "hgb_painn_update_tc_bwd"}
    for f, n, tc, fused in [(64, 256, True, True), (64, 256, False, False), (32, 256, True, False), (64, 127, True, False)]:
        upd, s, v, _, _ = make_case(n, last, seed=f + n, f=f)
        used = _entries(upd, s, v, tc)
        if fused:
            assert tc_entries <= used and "hgb_painn_update_pre_fwd" not in used
        else:
            assert not (tc_entries & used) and "hgb_painn_update_pre_fwd" in used
