"""PReLU on the GPU: ``hgb_prelu_fwd`` / ``hgb_prelu_bwd`` through the C-ABI against fp64 numpy (slopes of both signs and zero,
z exactly 0, NaN / inf, skip_slope, repeat bits, launches, refusals), a captured graph following in-place slope updates, the
engine's "prelu" models against the reference goldens of tests/golden/models_prelu.pt and the fp64 oracle, the MLIP force
training path, and the captured training paths against eager."""
import copy

import numpy as np
import pytest
import torch

import hydragnn_b200 as hb
from hydragnn_b200 import _lib, ops
from hydragnn_b200.synthetic import ARCH
from kernel_harness import Buf, check_bound, launches, stream, twice
from oracle.base import oracle_from_case
from stack_support import (MODEL_KW, PRELU_CASES, PRELU_MACE_CASES, Flat, _batch, _loader, _zero_dropout, case_mpnn_type,
                           check_golden_case, golden_data, grad_close, prelu_engine, rel_l2)

pytestmark = pytest.mark.gpu
DEV = "cuda"


# ---- the kernels --------------------------------------------------------------------------------------------------------------
def _inputs(count, seed, special=False):
    g = torch.Generator().manual_seed(seed)
    z = torch.randn(count, generator=g)
    z[::7] = 0.0                                                   # exactly 0 takes the slope branch
    z[3::11] = -0.0
    gy = torch.randn(count, generator=g)
    if special and count >= 8:
        z[1], z[2], z[4] = float("nan"), float("inf"), float("-inf")
        gy[5] = float("nan")
    return z, gy


def _ref(z, gy, a):
    z64, g64 = z.double().numpy(), gy.double().numpy()
    a32 = np.float32(a)
    pos = z.numpy() > 0
    y = np.where(pos, z.numpy(), a32 * z.numpy())                   # fp32 products, as ATen
    dz = np.where(pos, gy.numpy(), a32 * gy.numpy())
    ds = float(np.sum(np.where(pos, 0.0, z64 * g64)))
    scale = float(np.sum(np.where(pos, 0.0, np.abs(z64 * g64))))
    return y, dz, ds, scale


def _run(z, gy, a, skip=False):
    count = z.numel()
    zb, gb = Buf(count, data=z), Buf(count, data=gy)
    slope = torch.tensor([a], dtype=torch.float32, device=DEV)
    y, dz, ds = Buf(count), Buf(count), Buf(1)
    ws = Buf(max(int(_lib.query("hgb_prelu_workspace_bytes", count)) // 4, 1))

    def fwd():
        _lib.call("hgb_prelu_fwd", zb.ptr, count, slope.data_ptr(), y.ptr, stream())

    def bwd():
        _lib.call("hgb_prelu_bwd", gb.ptr, zb.ptr, count, slope.data_ptr(), dz.ptr, None if skip else ds.ptr,
                  None if skip else ws.ptr, int(skip), stream())
    return fwd, bwd, y, dz, ds


@pytest.mark.parametrize("slope", [0.25, 0.0, -0.7])
@pytest.mark.parametrize("count", [1, 7, 2047, 2048, 2049, 65537, 1_000_003, 5_000_000])
def test_prelu_kernels_match_fp64(count, slope):
    z, gy = _inputs(count, count % 1000 + 3)
    fwd, bwd, y, dz, ds = _run(z, gy, slope)
    assert launches(fwd) == 1 and launches(bwd) == 1
    y.check("prelu_fwd", "y")
    dz.check("prelu_bwd", "dz")
    ds.check("prelu_bwd", "dslope")
    twice("prelu_bwd", bwd, [dz, ds])
    yr, dzr, dsr, scale = _ref(z, gy, slope)
    assert np.array_equal(y.np().reshape(-1).view(np.int32), yr.astype(np.float32).view(np.int32))
    assert np.array_equal(dz.np().reshape(-1).view(np.int32), dzr.astype(np.float32).view(np.int32))
    check_bound("dslope", ds.np().reshape(-1), np.array([dsr]), np.array([1e-6 * scale + 2.0 ** -24 * abs(dsr)]))


def test_prelu_kernels_nan_and_inf_follow_aten():
    """NaN in z passes through y and takes the slope branch of dz; inf and -inf are ordinary values; the slope gradient of a NaN
    product is NaN, as ATen's."""
    z, gy = _inputs(4096, 9, special=True)
    fwd, bwd, y, dz, ds = _run(z, gy, 0.25)
    fwd()
    bwd()
    torch.cuda.synchronize()
    zt, wt = z.clone().to(DEV).requires_grad_(True), torch.tensor([0.25], device=DEV, requires_grad=True)
    yt = torch.nn.functional.prelu(zt, wt)
    gz, gw = torch.autograd.grad(yt, (zt, wt), gy.to(DEV))
    for got, want in ((y, yt), (dz, gz)):
        a, b = got.np().reshape(-1), want.detach().cpu().numpy()
        assert np.array_equal(np.isnan(a), np.isnan(b))
        assert np.array_equal(a[~np.isnan(a)], b[~np.isnan(b)])
    assert np.isnan(ds.np()[0, 0]) and torch.isnan(gw).all()


@pytest.mark.parametrize("count", [1, 2049, 1_000_003])
def test_prelu_bwd_skip_slope_writes_dz_only(count):
    z, gy = _inputs(count, 5)
    _, bwd, _, dz, ds = _run(z, gy, -0.4, skip=True)
    assert launches(bwd) == 1
    dz.check("prelu_bwd", "dz")
    ds.check("prelu_bwd", "dslope", written=False)
    assert np.isnan(ds.np()[0, 0])                                 # untouched
    _, dzr, _, _ = _ref(z, gy, -0.4)
    assert np.array_equal(dz.np().reshape(-1), dzr.astype(np.float32))


def test_prelu_refuses_bad_arguments():
    p = [torch.zeros(8, device=DEV) for _ in range(5)]
    slope = torch.zeros(1, device=DEV)
    ws = torch.zeros(64, device=DEV)
    for bad in (dict(count=0), dict(count=-1), dict(z=None), dict(slope=None)):
        a = dict(dict(count=8, z=p[0].data_ptr(), slope=slope.data_ptr()), **bad)
        with pytest.raises(RuntimeError, match="prelu_fwd"):
            _lib.call("hgb_prelu_fwd", a["z"], a["count"], a["slope"], p[1].data_ptr(), stream())
    good = dict(count=8, ds=p[4].data_ptr(), ws=ws.data_ptr(), skip=0, slope=slope.data_ptr())
    for bad in (dict(count=0), dict(slope=None), dict(ds=None), dict(ws=None)):
        a = dict(good, **bad)
        with pytest.raises(RuntimeError, match="prelu_bwd"):
            _lib.call("hgb_prelu_bwd", p[0].data_ptr(), p[1].data_ptr(), a["count"], a["slope"], p[2].data_ptr(), a["ds"], a["ws"],
                      a["skip"], stream())
    assert _lib.lib().hgb_version() >= 112


def test_prelu_fn_against_aten_and_data_only():
    """ops.PReluFn: y, dx and the slope gradient against ATen; under only_data_grads no slope gradient."""
    z, gy = _inputs(3 * 4099, 7)
    x = z.reshape(-1, 3).to(DEV)
    res = []
    for fused in (True, False):
        xa = x.clone().requires_grad_(True)
        w = torch.tensor([-0.3], device=DEV, requires_grad=True)
        y = ops.PReluFn.apply(xa, w) if fused else torch.nn.functional.prelu(xa, w)
        res.append([y.detach(), *torch.autograd.grad(y, (xa, w), gy.reshape(-1, 3).to(DEV))])
    for a, b in zip(*res):
        torch.testing.assert_close(a, b, rtol=1e-6, atol=1e-6 * float(b.abs().max()))
    xa = x.clone().requires_grad_(True)
    w = torch.tensor([0.2], device=DEV, requires_grad=True)
    with ops.only_data_grads():
        y = ops.PReluFn.apply(xa, w)
        y.backward(torch.ones_like(y))
    assert w.grad is None and xa.grad is not None


def test_captured_graph_follows_the_slope():
    """A captured forward + backward reads the slope when it replays: change it in place, replay, the outputs follow."""
    x = torch.randn(4096, 16, device=DEV)
    w = torch.tensor([0.25], device=DEV, requires_grad=True)
    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(s):
        for _ in range(2):
            xa = x.clone().requires_grad_(True)
            y = ops.PReluFn.apply(xa, w)
            gx, gw = torch.autograd.grad(y.sum(), (xa, w))
    torch.cuda.current_stream().wait_stream(s)
    g = torch.cuda.CUDAGraph()
    xa = x.clone().requires_grad_(True)
    with torch.cuda.graph(g):
        y = ops.PReluFn.apply(xa, w)
        gx, gw = torch.autograd.grad(y.sum(), (xa, w))
    for a in (-0.5, 0.0, 0.75):
        with torch.no_grad():
            w.fill_(a)
        g.replay()
        torch.cuda.synchronize()
        wt = torch.tensor([a], device=DEV)
        assert torch.equal(y, torch.nn.functional.prelu(x, wt))
        assert torch.equal(gx, torch.where(x > 0, 1.0, a).to(x.dtype).expand_as(x))
        torch.testing.assert_close(gw, torch.where(x > 0, 0.0, x).double().sum().float().reshape(1), rtol=1e-6, atol=1e-4)


# ---- PReLU in the Linear epilogues -------------------------------------------------------------------------------------------
def _lin_ref(x, w, b, a):
    z = x.double() @ w.double().T + (b.double() if b is not None else 0.0)
    return torch.where(z > 0, z, float(np.float32(a)) * z), z


def _lin_bound(x, w, b):
    return (x.double().abs() @ w.double().abs().T + (b.double().abs() if b is not None else 0.0)) * 2.0 ** -22 * (x.shape[1] + 2)


@pytest.mark.parametrize("slope", [0.25, -0.6])
@pytest.mark.parametrize("entry,m,n,k", [
    ("hgb_linear_fwd_prelu", 1, 1, 9), ("hgb_linear_fwd_prelu", 63, 10, 60), ("hgb_linear_fwd_prelu", 4099, 50, 25),
    ("hgb_linear_fwd_prelu", 70001, 7, 200), ("hgb_linear_smallk_fwd_prelu", 1, 3, 1), ("hgb_linear_smallk_fwd_prelu", 3001, 5, 3),
    ("hgb_linear_smallk_fwd_prelu", 3001, 64, 1), ("hgb_linear_smallk_fwd_prelu", 50003, 16, 8),
    ("hgb_linear_smallk_fwd_prelu", 777, 256, 5)])
def test_linear_prelu_epilogues_match_fp64(entry, m, n, k, slope):
    """The exact-fp32 and small-k (scalar and vec4) PReLU instances: y and z against fp64, one launch, guard rows intact, the
    slope read from device memory (a second call after an in-place change follows it)."""
    g = torch.Generator().manual_seed(m + n + k)
    x, w, b = torch.randn(m, k, generator=g), torch.randn(n, k, generator=g), torch.randn(n, generator=g)
    xb, wb, bb = Buf(m, k, data=x), Buf(n, k, data=w), Buf(n, data=b)
    y, z = Buf(m, n), Buf(m, n)
    sl = torch.tensor([slope], device=DEV)

    def call():
        if entry == "hgb_linear_fwd_prelu":
            _lib.call(entry, xb.ptr, wb.ptr, bb.ptr, m, n, k, k, k, sl.data_ptr(), y.ptr, z.ptr, stream())
        else:
            _lib.call(entry, xb.ptr, k, wb.ptr, k, bb.ptr, m, n, k, sl.data_ptr(), y.ptr, z.ptr, stream())
    for a in (slope, -slope / 3):
        sl.fill_(a)
        assert launches(call) == 1
        y.check(entry, "y")
        z.check(entry, "z")
        twice(entry, call, [y, z])
        yr, zr = _lin_ref(x, w, b, a)
        bound = _lin_bound(x, w, b)
        check_bound(entry + " z", z.np(), zr.numpy(), bound.numpy())
        check_bound(entry + " y", y.np(), yr.numpy(), (bound * max(1.0, abs(a))).numpy())
        zt = torch.from_numpy(z.np().copy())
        assert torch.equal(torch.from_numpy(y.np().copy()), torch.nn.functional.prelu(zt, torch.tensor([a])))


@pytest.mark.parametrize("counts", [[5, 0, 130, 1], [1], [0, 0, 64], [1000, 333, 2049]])
@pytest.mark.parametrize("n,k", [(10, 60), (7, 5), (64, 64)])
def test_grouped_linear_prelu_matches_fp64(counts, n, k):
    g = torch.Generator().manual_seed(sum(counts) + n)
    groups, m = len(counts), sum(counts)
    x, w, b = torch.randn(m, k, generator=g), torch.randn(groups, n, k, generator=g), torch.randn(groups, n, generator=g)
    rowptr = torch.tensor([0] + list(np.cumsum(counts)), dtype=torch.int32, device=DEV)
    xd, wd, bd = x.to(DEV), w.to(DEV), b.to(DEV)
    y, z = torch.full((m, n), float("nan"), device=DEV), torch.full((m, n), float("nan"), device=DEV)
    sl = torch.tensor([-0.35], device=DEV)

    def call():
        _lib.call("hgb_grouped_linear_prelu", xd.data_ptr(), k, wd.data_ptr(), bd.data_ptr(), rowptr.data_ptr(), groups, m, n, k,
                  sl.data_ptr(), y.data_ptr(), z.data_ptr(), stream())
    assert launches(call) == 1
    gid = torch.repeat_interleave(torch.arange(groups), torch.tensor(counts))
    zr = torch.einsum("mk,mnk->mn", x.double(), w.double()[gid]) + b.double()[gid]
    bound = (torch.einsum("mk,mnk->mn", x.double().abs(), w.double().abs()[gid]) + b.double().abs()[gid]) * 2.0 ** -22 * (k + 2)
    check_bound("grouped z", z.cpu().numpy(), zr.numpy(), bound.numpy())
    assert torch.equal(y.cpu(), torch.nn.functional.prelu(z.cpu(), sl.cpu()))


@pytest.mark.parametrize("tc", [False, True])
@pytest.mark.parametrize("m,n,k", [(4099, 50, 25), (3001, 12, 3), (40000, 64, 64), (513, 96, 128)])
def test_linear_prelu_fn_against_aten(m, n, k, tc):
    """ops.linear_act(..., "prelu", slope): y, dx, dW, db and the slope gradient against the ATen composition in fp64; the
    epilogue entry points run where the shape is not a tensor-core one (there the Linear is followed by hgb_prelu_fwd)."""
    g = torch.Generator().manual_seed(m + k)
    x = torch.randn(m, k, generator=g).to(DEV)
    lin = torch.nn.Linear(k, n).to(DEV)
    gy = torch.randn(m, n, generator=g).to(DEV)
    w = torch.tensor([-0.2], device=DEV, requires_grad=True)
    xa = x.clone().requires_grad_(True)
    _lib.trace_begin()
    with ops.tensor_cores(tc):
        on_tc = k > 8 and ops.tc_ok(m, n, k, x)
        y = ops.linear_act(xa, lin.weight, lin.bias, "prelu", w)
        got = torch.autograd.grad(y, (xa, lin.weight, lin.bias, w), gy)
    calls = {t[0] for t in _lib.trace_end()}
    if on_tc:
        # the tensor-core Linear rounds to TF32 where it runs: the reference is the engine's own Linear there, then ATen's prelu
        xr = x.clone().requires_grad_(True)
        wr, br, sr = (t.detach().clone().requires_grad_(True) for t in (lin.weight, lin.bias, w))
        with ops.tensor_cores(tc):
            yr = torch.nn.functional.prelu(ops.linear_act(xr, wr, br), sr)
            want = torch.autograd.grad(yr, (xr, wr, br, sr), gy)
    else:
        xr = x.double().requires_grad_(True)
        wr, br, sr = (t.detach().double().requires_grad_(True) for t in (lin.weight, lin.bias, w))
        yr = torch.nn.functional.prelu(xr @ wr.T + br, sr)
        want = torch.autograd.grad(yr, (xr, wr, br, sr), gy.double())
    bound = 1e-5
    assert rel_l2(y.detach().cpu(), yr.detach().cpu()) < bound
    for a, b in zip(got, want):
        assert rel_l2(a.cpu(), b.cpu()) < bound
    assert "hgb_prelu_bwd" in calls
    if not on_tc:
        assert calls & {"hgb_linear_fwd_prelu", "hgb_linear_smallk_fwd_prelu"} and "hgb_prelu_fwd" not in calls, sorted(calls)


# ---- the engine against the reference goldens ----------------------------------------------------------------------------------
@pytest.fixture(scope="module")
def golden(golden_dir):
    return torch.load(golden_dir + "/models_prelu.pt")


def _engine(name, c):
    m = prelu_engine(name, c, use_gpu=True)
    m.load_state_dict(c["state"], strict=True)
    return m


@pytest.mark.parametrize("name", PRELU_CASES)
def test_engine_matches_reference_golden(golden, name):
    """Predictions, loss and every gradient (the slope's summed over every site) of the engine against the reference; the PReLU
    kernels run in the step."""
    c = golden[name]
    m = _engine(name, c)
    if name == "egnn_gnll":
        m = Flat(m)
    # the conv head's BatchNorm cancels the gradient of the bias before it: exactly 0, rounding noise in both fp32 models.  The GPS
    # case sums attention and conv gradients in another order than the reference
    atol = {"pna_conv_head_slope": 1e-4, "pna_gps": 1e-5}.get(name, 1e-6)
    _lib.trace_begin()
    state_after = (1e-4, 1e-5) if name == "pna_gps" else (1e-5, 1e-7)       # GPS's BatchNorm sees the attention's rounding too
    check_golden_case(m, c, lambda: _batch(c["inputs"]), pred=(1e-5, 1e-5), loss=(1e-5, 1e-7), grads=grad_close(1e-3, atol),
                      state_after=state_after)
    calls = {t[0] for t in _lib.trace_end()}
    assert "hgb_prelu_bwd" in calls, sorted(calls)
    if name != "pna_conv_head_slope":                              # its PReLUs follow BatchNorms: stand-alone hgb_prelu_fwd
        assert calls & {"hgb_linear_fwd_prelu", "hgb_linear_smallk_fwd_prelu", "hgb_grouped_linear_prelu"}, sorted(calls)
    if name == "egnn_two_branches":
        assert "hgb_grouped_linear_prelu" in calls


@pytest.mark.parametrize("name", PRELU_MACE_CASES)
def test_mace_matches_reference_golden(golden, name):
    """MACE's decoders (and FiLM's conditioner) with the shared PReLU: predictions, the position gradient of the objective and
    every parameter gradient, in eval mode as the MACE goldens are recorded."""
    c = golden[name]
    m = prelu_engine(name, c, use_gpu=True)
    m.eval()
    d = _batch(c["inputs"])
    d.pos.requires_grad_(True)
    torch.manual_seed(1234)
    pred = m(d)
    m.load_state_dict(c["state"], strict=True)                  # after the first forward, which creates the conditioner
    pred = m(d)
    for p, q in zip(pred, c["pred"]):
        assert rel_l2(p.detach().cpu(), q) < 1e-5
    obj = pred[0].sum() + pred[1].pow(2).sum()
    f, = torch.autograd.grad(obj, d.pos, retain_graph=True)
    assert rel_l2(f.cpu(), c["dobj_dpos"]) < 1e-4
    grads = torch.autograd.grad(obj, list(m.parameters()), allow_unused=True)
    for (n, _), g in zip(m.named_parameters(), grads):
        ref = c["grads"][n]
        if ref is None:
            assert g is None or not g.any(), n
        else:
            assert rel_l2(g.cpu(), ref) < 1e-4, n


@pytest.mark.parametrize("precision", ["fp32", "bf16"])
@pytest.mark.parametrize("name", [n for n in PRELU_CASES if n not in ("pna_gps",)])
def test_engine_training_step_matches_fp64_oracle(golden, name, precision):
    """One train-mode step of the engine in fp32 and bf16 (TF32 tensor-core Linears) against the fp64 oracle: predictions, loss
    and all gradients together within 1e-4 (fp32) or 2e-2 (bf16)."""
    c = golden[name]
    em = hb.set_precision(_engine(name, c), precision)
    om = oracle_from_case(case_mpnn_type(name), c).train()
    _zero_dropout(om)
    nll = name == "egnn_gnll"
    if nll:
        om, em_call = Flat(om), Flat(em)
    else:
        em_call = em
    value, hi = c["value"], c["head_index"]
    opred = om(golden_data(c["inputs"]))
    oloss, _ = om.loss(opred, value.double(), hi)
    oparams = [p for _, p in (om.m if nll else om).named_parameters()]
    ograds = torch.autograd.grad(oloss, oparams)
    em.train()
    _zero_dropout(em)
    em.zero_grad(set_to_none=True)
    epred = em_call(_batch(c["inputs"]))
    eloss, _ = em_call.loss(epred, value.to(DEV), [i.to(DEV) for i in hi])
    eloss.backward()
    bound = 1e-4 if precision == "fp32" else 2e-2
    for a, b in zip(epred, opred):
        assert rel_l2(a.detach().cpu(), b.detach()) < bound
    assert abs(float(eloss) - float(oloss)) <= bound * abs(float(oloss))
    ep = dict(em.named_parameters())
    slope = em.activation_function.weight
    g, r = [], []
    for (n, _), og in zip((om.m if nll else om).named_parameters(), ograds):
        p = slope if n == "activation_function.weight" else ep[n]
        g.append(p.grad.double().cpu().reshape(-1))
        r.append(og.reshape(-1))
    assert rel_l2(torch.cat(g), torch.cat(r)) < bound
    torch.testing.assert_close(slope.grad.double().cpu(), ograds[[n for n, _ in (om.m if nll else om).named_parameters()]
                                                                 .index("activation_function.weight")],
                               rtol=bound, atol=bound * float(torch.cat(r).abs().max()))


# ---- force training and the captured paths -------------------------------------------------------------------------------------
def test_mlip_force_step_with_prelu_node_head_matches_oracle(golden_dir):
    """The force-training step (any order: ATen prelu under the double backward) of an EGNN interatomic potential with a PReLU
    node head, slope -0.2: the engine's loss and every gradient, the slope's included, against the fp64 oracle."""
    import oracle.base
    c = torch.load(golden_dir + "/models.pt")["egnn_mlip"]
    kw = dict(MODEL_KW["egnn_mlip"], activation_function="prelu", enable_interatomic_potential=True, energy_weight=1.0,
              energy_peratom_weight=1.0, force_weight=1.0)
    torch.manual_seed(0)
    em = hb.create_model(**kw)
    with torch.no_grad():
        em.model.activation_function.weight.fill_(-0.2)
    om = oracle.base.create_model(**kw)
    own = om.model.state_dict()
    om.model.load_state_dict({k: v.cpu() for k, v in em.model.state_dict().items() if k in own}, strict=True)
    om = om.double()
    res = []
    for m, dev, dt in ((em, DEV, torch.float32), (om, "cpu", torch.float64)):
        d = hb.Batch(**{k: (v.to(dt) if v.is_floating_point() else v).clone().to(dev) for k, v in c["inputs"].items()})
        d._num_graphs = int(c["inputs"]["batch"].max()) + 1
        d.pos.requires_grad_(True)
        m.train()
        tot, _ = m.energy_force_loss(m(d), d, create_graph=True)
        params = [p for _, p in m.model.named_parameters()]
        grads = torch.autograd.grad(tot, params)
        res.append((float(tot), {n: g.double().cpu() for (n, _), g in zip(m.model.named_parameters(), grads)},
                    m.model.activation_function.weight))
    (le, ge, se), (lo, go, so) = res
    assert abs(le - lo) <= 1e-5 * abs(lo), (le, lo)
    slope_e = [n for n, p in em.model.named_parameters() if p is se][0]
    names = [n for n in go if n != "activation_function.weight"]
    g = torch.cat([ge[n].reshape(-1) for n in names] + [ge[slope_e].reshape(-1)])
    r = torch.cat([go[n].reshape(-1) for n in names] + [go["activation_function.weight"].reshape(-1)])
    assert rel_l2(g, r) < 1e-4
    torch.testing.assert_close(ge[slope_e], go["activation_function.weight"], rtol=1e-4, atol=1e-6 * float(r.abs().max()))


def _qm9_prelu():
    kw = dict(ARCH["qm9_painn"], activation_function="prelu")
    m = hb.create_model(**kw)
    _zero_dropout(m)
    with torch.no_grad():
        m.activation_function.weight.fill_(-0.1)
    return hb.get_distributed_model(m)


def test_padded_graph_step_epoch_equals_eager():
    """hb.train with the capacity-padded captured step against the eager epoch: the slope trains the same way in both."""
    from hydragnn_b200 import padded
    loader = _loader("qm9_painn", [48, 40, 56, 33], with_edges=True)
    ma = _qm9_prelu()
    mb = copy.deepcopy(ma)
    assert padded.supported(ma)
    oa, ob = hb.FlatAdamW(ma, lr=1e-3), hb.FlatAdamW(mb, lr=1e-3)
    s0 = float(ma.module.activation_function.weight)
    la, _ = hb.train(loader, ma, oa, fast=True)
    lb, _ = hb.train(loader, mb, ob, fast=False)
    torch.cuda.synchronize()
    assert getattr(oa, "_hgb_fast", None) is not None
    assert abs(float(la) - float(lb)) <= 1e-5 * abs(float(lb)), (float(la), float(lb))
    sa, sb = ma.module.state_dict(), mb.module.state_dict()
    assert float(sa["activation_function.weight"]) != s0
    for k in sa:
        if sa[k].is_floating_point():
            torch.testing.assert_close(sa[k], sb[k], rtol=1e-4, atol=1e-6, msg=lambda s, k=k: k + ": " + s)


def test_graphed_train_step_replay_equals_eager():
    """GraphedTrainStep replays read the slope the optimiser updated in place: the replayed steps match eager ones."""
    b = _loader("qm9_painn", [64], with_edges=True)[0].to(DEV)
    b._num_graphs = 64
    ma = _qm9_prelu()
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
