"""GaussianNLLLoss on the GPU: the ``hgb_gnll_fwd_bwd`` kernel through the C-ABI against fp64 numpy (guard rows, padded prefixes,
repeat bits, launches, refusals), and the engine's mean-and-variance models against the reference goldens of
tests/golden/models_gnll.pt, against the fp64 oracle in fp32 and bf16, and through the captured training paths."""
import copy

import numpy as np
import pytest
import torch

import hydragnn_b200 as hb
from hydragnn_b200 import _lib, ops
from hydragnn_b200.synthetic import ARCH
from kernel_harness import Buf, check_bound, launches, stream, twice
from oracle.base import oracle_from_case
from stack_support import (GNLL_CASES, Flat, _batch, _loader, _zero_dropout, case_mpnn_type, check_golden_case, golden_data,
                           grad_close, named_case_kwargs, rel_l2)

pytestmark = pytest.mark.gpu
DEV = "cuda"
EPS = 1e-6


# ---- the kernel ---------------------------------------------------------------------------------------------------------------
def _inputs(count, seed):
    g = torch.Generator().manual_seed(seed)
    mean = torch.randn(count, generator=g)
    target = torch.randn(count, generator=g)
    s = torch.randn(count, generator=g)                          # negative raw outputs included
    s[::5] *= 1e-4                                                # var = s^2 < eps: clamped
    s[1::11] = 0.0
    s[2::7] *= 1e-3                                               # var = s^2 around eps, both sides
    return mean, s * s, target


def _ref(mean, var, target, n):
    m, v, t = (a.double().numpy() for a in (mean, var, target))
    d, vc = m - t, np.maximum(v, EPS)
    inv = 1.0 / max(n, 1)
    gm, gv = d / vc * inv, 0.5 * (1.0 / vc - d * d / (vc * vc)) * inv
    gm[n:] = 0.0
    gv[n:] = 0.0
    loss = 0.5 * np.sum(np.log(vc[:n]) + d[:n] ** 2 / vc[:n]) * inv if n > 0 else 0.0
    # the gradient of the variance cancels where d^2 = v_c: its bound also covers the rounding of its two terms
    scale = 0.5 * (1.0 / vc + d * d / (vc * vc)) * inv
    scale[n:] = 0.0
    return loss, gm, gv, scale


def _run(mean, var, target, valid=None, row_width=1):
    count = mean.numel()
    bufs = [Buf(count, data=t) for t in (mean, var, target)]
    loss, gm, gv = Buf(1), Buf(count), Buf(count)
    ws = Buf(max(int(_lib.query("hgb_gnll_workspace_bytes", count)) // 4, 1))
    vr = None if valid is None else torch.tensor([valid], dtype=torch.int32, device=DEV)

    def call():
        _lib.call("hgb_gnll_fwd_bwd", *(b.ptr for b in bufs), count, EPS, loss.ptr, gm.ptr, gv.ptr, ws.ptr,
                  None if vr is None else vr.data_ptr(), row_width, stream())
    return call, loss, gm, gv


@pytest.mark.parametrize("d", [1, 3, 5])
@pytest.mark.parametrize("rows", [1, 7, 1023, 1024, 1025, 65537, 1_000_003])
def test_gnll_kernel_matches_fp64(rows, d):
    count = rows * d
    mean, var, target = _inputs(count, rows * 10 + d)
    call, loss, gm, gv = _run(mean, var, target)
    assert launches(call) == 1
    for b, name in ((loss, "loss"), (gm, "gmean"), (gv, "gvar")):
        b.check("gnll", name)
    twice("gnll", call, [loss, gm, gv])
    lref, gmr, gvr, scale = _ref(mean, var, target, count)
    check_bound("gmean", gm.np().reshape(-1), gmr, 2e-6 * np.abs(gmr))
    check_bound("gvar", gv.np().reshape(-1), gvr, 2e-6 * np.abs(gvr) + 1e-12 * scale)
    assert abs(float(loss.np()[0, 0]) - lref) <= 1e-5 * abs(lref), (float(loss.np()[0, 0]), lref)


@pytest.mark.parametrize("valid", [0, 1, 700, 1025, 4000, -3])
def test_gnll_kernel_valid_rows_prefix(valid):
    """Only the first ``valid`` rows of 3 entries are real: the mean runs over them, every gradient beyond is exactly zero, and no
    real row gives a loss of 0."""
    rows, d = 1025, 3
    mean, var, target = _inputs(rows * d, 99)
    call, loss, gm, gv = _run(mean, var, target, valid, d)
    assert launches(call) == 1
    n = max(min(valid, rows), 0) * d
    lref, gmr, gvr, scale = _ref(mean, var, target, n)
    check_bound("gmean", gm.np().reshape(-1), gmr, 2e-6 * np.abs(gmr))
    check_bound("gvar", gv.np().reshape(-1), gvr, 2e-6 * np.abs(gvr) + 1e-12 * scale)
    assert not gm.np().reshape(-1)[n:].any() and not gv.np().reshape(-1)[n:].any()
    got = float(loss.np()[0, 0])
    assert (got == 0.0) if n == 0 else abs(got - lref) <= 1e-5 * abs(lref)


def test_gnll_kernel_refuses_bad_arguments():
    mean, var, target = (torch.ones(8, device=DEV) for _ in range(3))
    out = [torch.empty(8, device=DEV) for _ in range(3)]
    ws = torch.empty(int(_lib.query("hgb_gnll_workspace_bytes", 8)), dtype=torch.uint8, device=DEV)
    vr = torch.ones(1, dtype=torch.int32, device=DEV)
    p = [t.data_ptr() for t in (mean, var, target)]
    good = dict(count=8, eps=EPS, ws=ws.data_ptr(), mean=p[0], vr=None, rw=1)
    for bad in (dict(count=0), dict(count=-4), dict(mean=None), dict(ws=None), dict(eps=0.0), dict(eps=-1.0),
                dict(vr=vr.data_ptr(), rw=0), dict(vr=vr.data_ptr(), rw=-2)):
        a = dict(good, **bad)
        with pytest.raises(RuntimeError, match="gnll_fwd_bwd"):
            _lib.call("hgb_gnll_fwd_bwd", a["mean"], p[1], p[2], a["count"], a["eps"], out[0].data_ptr(), out[1].data_ptr(),
                      out[2].data_ptr(), a["ws"], a["vr"], a["rw"], stream())
    assert _lib.query("hgb_gnll_workspace_bytes", 0) == 0
    assert _lib.lib().hgb_version() >= 111


def test_gaussian_nll_fn_matches_torch_with_raw_output_gradient():
    """ops.GaussianNLLFn under var = s^2 (the heads' variance) against torch's gaussian_nll_loss on the GPU: value and the
    gradients with respect to the mean and the raw output s."""
    mean, var, target = _inputs(3 * 4099, 7)
    s = var.sqrt() * torch.where(torch.arange(var.numel()) % 2 == 0, 1.0, -1.0)
    res = []
    for fused in (True, False):
        mu = mean.to(DEV).requires_grad_(True)
        sv = s.to(DEV).requires_grad_(True)
        t = target.to(DEV)
        val = ops.GaussianNLLFn.apply(mu, sv * sv, t) if fused else torch.nn.functional.gaussian_nll_loss(mu, t, sv * sv)
        res.append([val.detach(), *torch.autograd.grad(val, (mu, sv))])
    for a, b in zip(*res):
        torch.testing.assert_close(a, b, rtol=1e-5, atol=1e-6 * float(b.abs().max()))


# ---- the engine against the reference goldens ------------------------------------------------------------------------------------
@pytest.fixture(scope="module")
def golden(golden_dir):
    return torch.load(golden_dir + "/models_gnll.pt")


def _engine(name, c):
    m = hb.create_model(**named_case_kwargs(name, c))
    m.load_state_dict(c["state"], strict=True)
    return m


@pytest.mark.parametrize("name", GNLL_CASES)
def test_engine_matches_reference_golden(golden, name):
    """Means, variances, the NLL and every gradient of the engine against the reference, at the bounds of the stacks' own golden
    tests; the fused NLL kernel runs in the train step.  The conv head and the clamped case carry (mean - target) / eps terms."""
    c = golden[name]
    atol = 1e-5 if name in ("pna_conv_head", "egnn_clamped") else 1e-6
    m = _engine(name, c)
    _lib.trace_begin()
    check_golden_case(Flat(m), c, lambda: _batch(c["inputs"]), pred=(1e-5, 1e-5), loss=(1e-5, 1e-7), grads=grad_close(1e-3, atol))
    assert "hgb_gnll_fwd_bwd" in {t[0] for t in _lib.trace_end()}


@pytest.mark.parametrize("precision", ["fp32", "bf16"])
@pytest.mark.parametrize("name", [n for n in GNLL_CASES if n != "pna_gps"])
def test_engine_training_step_matches_fp64_oracle(golden, name, precision):
    """One train-mode step of the engine, in fp32 and in bf16 (TF32 tensor-core Linears), against the oracle in fp64: rel-L2 of the
    means and variances, the NLL and all gradients together within 1e-4 (fp32) or 2e-2 (bf16)."""
    c = golden[name]
    em = hb.set_precision(_engine(name, c), precision)
    om = oracle_from_case(case_mpnn_type(name), c).train()
    _zero_dropout(om)
    value, hi = c["value"], c["head_index"]
    opred = om(golden_data(c["inputs"]))
    oloss, _ = om.loss(opred, value.double(), hi)
    ograds = torch.autograd.grad(oloss, list(om.parameters()))
    em.train()
    _zero_dropout(em)
    em.zero_grad(set_to_none=True)
    epred = em(_batch(c["inputs"]))
    eloss, _ = em.loss(epred, value.to(DEV), [i.to(DEV) for i in hi])
    eloss.backward()
    bound = 1e-4 if precision == "fp32" else 2e-2
    for a, b in zip(epred[0] + epred[1], opred[0] + opred[1]):
        assert rel_l2(a.detach().cpu(), b.detach()) < bound
    assert abs(float(eloss) - float(oloss)) <= bound * abs(float(oloss))
    names = [n for n, _ in om.named_parameters()]
    eg = dict(em.named_parameters())
    g = torch.cat([eg[n].grad.double().cpu().reshape(-1) for n in names])
    r = torch.cat([x.reshape(-1) for x in ograds])
    assert rel_l2(g, r) < bound


# ---- the training paths --------------------------------------------------------------------------------------------------------
def _qm9_gnll():
    kw = dict(ARCH["qm9_painn"], loss_function_type="GaussianNLLLoss")
    m = hb.create_model(**kw)
    _zero_dropout(m)
    return hb.get_distributed_model(m)


def test_padded_graph_step_epoch_equals_eager():
    """hb.train with the capacity-padded captured step (the masked NLL over the real graphs) against the eager epoch."""
    from hydragnn_b200 import padded
    loader = _loader("qm9_painn", [48, 40, 56, 33], with_edges=True)
    ma = _qm9_gnll()
    mb = copy.deepcopy(ma)
    assert padded.supported(ma) and ma.module.var_output == 1
    oa, ob = hb.FlatAdamW(ma, lr=1e-3), hb.FlatAdamW(mb, lr=1e-3)
    la, ta = hb.train(loader, ma, oa, fast=True)
    lb, tb = hb.train(loader, mb, ob, fast=False)
    torch.cuda.synchronize()
    assert getattr(oa, "_hgb_fast", None) is not None
    assert abs(float(la) - float(lb)) <= 1e-5 * abs(float(lb)), (float(la), float(lb))
    sa, sb = ma.module.state_dict(), mb.module.state_dict()
    for k in sa:
        if sa[k].is_floating_point():
            torch.testing.assert_close(sa[k], sb[k], rtol=1e-4, atol=1e-6, msg=lambda s, k=k: k + ": " + s)


def test_graphed_train_step_replay_equals_eager():
    b = _loader("qm9_painn", [64], with_edges=True)[0].to(DEV)
    b._num_graphs = 64
    ma = _qm9_gnll()
    mb = copy.deepcopy(ma)
    oa, ob = hb.FlatAdamW(ma, lr=1e-3), hb.FlatAdamW(mb, lr=1e-3)
    losses = [float(hb.train_step(ma, oa, b)[0]) for _ in range(6)]
    gs = hb.GraphedTrainStep(mb, ob, b.clone(), warmup=3)
    glosses = [float(gs.run()) for _ in range(3)]
    torch.cuda.synchronize()
    assert losses[-1] < losses[0]
    assert abs(glosses[-1] - losses[-1]) <= 1e-5 * abs(losses[-1]), (glosses, losses)
    sa, sb = ma.module.state_dict(), mb.module.state_dict()
    for k in sa:
        if sa[k].is_floating_point():
            torch.testing.assert_close(sb[k], sa[k], rtol=1e-5, atol=1e-7, msg=lambda s, k=k: k + ": " + s)
