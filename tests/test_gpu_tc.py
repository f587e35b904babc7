"""GPU parity tests of the wgmma (TF32) dense-layer kernels against fp64 references.
Tolerance: TF32 truncates operands to 10 mantissa bits -> relative L2 error <= 2e-3 (well inside the 2e-2 the
bf16 config allows, SURVEY 8d).  The fp32-accurate 3xTF32 mode ("exact", the default of the fp32 configs) is fp32-level:
<= 2e-6 for a Linear (tests/test_gpu_round2.py::test_fp32_linear_runs_tc_exact_mode_and_matches_fp64)."""
import pytest
import torch

pytestmark = pytest.mark.gpu

import hydragnn_b200 as hb  # noqa: E402
from hydragnn_b200 import ops  # noqa: E402
from hydragnn_b200.synthetic import ARCH, make_samples  # noqa: E402

DEV = "cuda"


def rel(a, b):
    return float((a.double().cpu() - b.double()).norm() / b.double().norm())


@pytest.mark.parametrize("m,k,n", [(128, 64, 64), (1000, 64, 192), (4097, 128, 64), (300, 32, 32), (20000, 192, 64), (513, 64, 128)])
@pytest.mark.parametrize("act", [None, "silu", "relu"])
def test_tc_linear_forward(m, k, n, act):
    g = torch.Generator().manual_seed(m + k + n)
    x, w, b = torch.randn(m, k, generator=g), torch.randn(n, k, generator=g) * 0.2, torch.randn(n, generator=g)
    ref_z = x.double() @ w.double().t() + b.double()
    ref = {None: lambda t: t, "silu": torch.nn.functional.silu, "relu": torch.relu}[act](ref_z)
    y, z = ops.raw_tc_linear(x.to(DEV), w.to(DEV), False, b.to(DEV), n, k, ops.ACT_CODES[act], 0.0, want_z=True)
    torch.cuda.synchronize()
    assert rel(z, ref_z) < 2e-3
    assert rel(y, ref) < 2e-3


@pytest.mark.parametrize("m,n,k", [(1000, 192, 64), (4097, 64, 128), (129, 64, 64)])
def test_tc_dgrad_and_wgrad(m, n, k):
    g = torch.Generator().manual_seed(m + n + k)
    dz, x, w = torch.randn(m, n, generator=g), torch.randn(m, k, generator=g), torch.randn(n, k, generator=g) * 0.2
    with ops.tensor_cores(True):                                  # plain TF32 (the bf16 configs)
        dx, _ = ops.raw_tc_linear(dz.to(DEV), w.to(DEV), True, None, k, n)
        assert rel(dx, dz.double() @ w.double()) < 2e-3
        dw, db = ops.raw_tc_wgrad(dz.to(DEV), x.to(DEV), want_bias=True)
        torch.cuda.synchronize()
        e = rel(dw, dz.double().t() @ x.double())
        assert 1e-5 < e < 2e-3
        assert rel(db, dz.double().sum(0)) < 2e-3
        dw2, db2 = ops.raw_tc_wgrad(dz.to(DEV), x.to(DEV), want_bias=True)
        assert torch.equal(dw, dw2) and torch.equal(db, db2)          # deterministic


@pytest.mark.parametrize("m,k,n", [(3000, 64, 448), (2000, 192, 512), (1500, 64, 288)])
def test_tc_wide_shapes_are_cut_into_pieces(m, k, n):
    """n_out > 256 -> column pieces; reduction > 256 (the dgrad of a wide layer) -> pieces accumulated through `addend`."""
    g = torch.Generator().manual_seed(m + k + n)
    x, w, b = torch.randn(m, k, generator=g), torch.randn(n, k, generator=g) * 0.2, torch.randn(n, generator=g)
    y, z = ops.raw_tc_linear(x.to(DEV), w.to(DEV), False, b.to(DEV), n, k, ops.ACT_CODES["silu"], 0.0, want_z=True)
    ref_z = x.double() @ w.double().t() + b.double()
    assert rel(z, ref_z) < 2e-3 and rel(y, torch.nn.functional.silu(ref_z)) < 2e-3
    dz = torch.randn(m, n, generator=g)
    add = torch.randn(m, k, generator=g)
    dx, _ = ops.raw_tc_linear(dz.to(DEV), w.to(DEV), True, None, k, n, addend=add.to(DEV))
    assert rel(dx, dz.double() @ w.double() + add.double()) < 2e-3
    dw, db = ops.raw_tc_wgrad(dz.to(DEV), x.to(DEV), want_bias=True)
    assert rel(dw, dz.double().t() @ x.double()) < 2e-3 and rel(db, dz.double().sum(0)) < 2e-3


def test_linear_act_autograd_on_tensor_cores():
    g = torch.Generator().manual_seed(5)
    x, w, b = torch.randn(3000, 64, generator=g), torch.randn(192, 64, generator=g) * 0.2, torch.randn(192, generator=g)
    xr, wr, br = [t.double().requires_grad_(True) for t in (x, w, b)]
    xe, we, be = [t.to(DEV).requires_grad_(True) for t in (x, w, b)]
    go = torch.randn(3000, 192, generator=g)
    yr = torch.nn.functional.silu(xr @ wr.t() + br)
    with ops.tensor_cores(True):
        ye = ops.linear_act(xe, we, be, "silu")
    gr = torch.autograd.grad(yr, (xr, wr, br), go.double())
    ge = torch.autograd.grad(ye, (xe, we, be), go.to(DEV))          # backward outside the context: flag is carried by ctx
    assert rel(ye, yr.detach()) < 2e-3
    for a, c in zip(ge, gr):
        assert rel(a, c) < 3e-3


def test_qm9_painn_bf16_mode_close_to_fp32_and_trains():
    name, G = "qm9_painn", 512
    b = make_samples(name, G).to(DEV)
    b._num_graphs = G
    b = hb.get_radius_graph(7.0, 5)(b)
    m32 = hb.create_model(**ARCH[name])
    mtc = hb.set_precision(hb.create_model(**ARCH[name]), "bf16")
    hi = [torch.arange(G, device=DEV)]
    l32, _ = m32.loss(m32(b), b.y, hi)
    ltc, _ = mtc.loss(mtc(b), b.y, hi)
    assert abs(float(ltc) - float(l32)) <= 2e-2 * abs(float(l32))
    l32.backward()
    ltc.backward()
    num = sum(float((p.grad - q.grad).double().pow(2).sum()) for p, q in zip(mtc.parameters(), m32.parameters()))
    den = sum(float(q.grad.double().pow(2).sum()) for q in m32.parameters())
    assert (num / den) ** 0.5 < 2e-2
    model = hb.get_distributed_model(mtc)
    opt = hb.FlatAdamW(model, lr=1e-3)
    losses = [float(hb.train_step(model, opt, b)[0]) for _ in range(20)]
    assert losses[-1] < losses[0]


def test_mlip_double_backward_on_tensor_cores_close_to_fp32():
    """precision="bf16" also covers the any-order (MLIP) path: MatMul and its (double) backward run on the TF32 kernels."""
    name, G = "md17_egnn", 64
    b = make_samples(name, G).to(DEV)
    b._num_graphs = G
    b = hb.get_radius_graph(7.0, 5)(b)
    m32 = hb.create_model(**ARCH[name])
    mtc = hb.set_precision(hb.create_model(**ARCH[name]), "bf16")
    out = []
    for m in (m32, mtc):
        m.train()
        d = b.clone()
        d.pos.requires_grad_(True)
        before = hb._lib.launch_count()
        loss, tasks = m.energy_force_loss(m(d), d)
        loss.backward()
        out.append((float(loss), [p.grad.clone() for p in m.parameters()]))
    assert abs(out[1][0] - out[0][0]) <= 2e-2 * abs(out[0][0])
    num = sum(float((p - q).double().pow(2).sum()) for p, q in zip(out[1][1], out[0][1]))
    den = sum(float(q.double().pow(2).sum()) for q in out[0][1])
    assert (num / den) ** 0.5 < 3e-2


@pytest.mark.parametrize("exact,k,n", [(False, 256, 160), (False, 256, 64), (True, 256, 64), (True, 224, 64), (True, 192, 96),
                                       (True, 160, 64), (True, 128, 160)])
def test_tc_linear_many_tiles_per_consumer(exact, k, n):
    """Shapes whose tiles have more k-blocks than a consumer's stage ring holds, with m large enough that each of the two consumer
    warpgroups of every CTA runs several tiles: the rings recycle their stages within a tile and across tiles.  fp64 agreement,
    and bit-identical results when a weight-gradient kernel runs concurrently on a second stream (different timing, same result)."""
    m = 70000
    g = torch.Generator().manual_seed(k + n + int(exact))
    x, w, b = torch.randn(m, k, generator=g), torch.randn(n, k, generator=g) * 0.2, torch.randn(n, generator=g)
    xd, wd, bd = x.to(DEV), w.to(DEV), b.to(DEV)
    ref_z = x.double() @ w.double().t() + b.double()
    with ops.tensor_cores(not exact):                             # exact = the fp32-accurate split mode
        y, z = ops.raw_tc_linear(xd, wd, False, bd, n, k, ops.ACT_CODES["silu"], 0.0, want_z=True)
        dz, xo = torch.randn(m, 128, device=DEV), torch.randn(m, 128, device=DEV)
        side = torch.cuda.Stream()
        side.wait_stream(torch.cuda.current_stream())
        with torch.cuda.stream(side):
            ops.raw_tc_wgrad(dz, xo, want_bias=True)
        y2, z2 = ops.raw_tc_linear(xd, wd, False, bd, n, k, ops.ACT_CODES["silu"], 0.0, want_z=True)
        torch.cuda.current_stream().wait_stream(side)
    torch.cuda.synchronize()
    tol = 2e-6 if exact else 2e-3
    assert rel(z, ref_z) < tol and rel(y, torch.nn.functional.silu(ref_z)) < tol
    assert torch.equal(y, y2) and torch.equal(z, z2)


# ==== the argument space of hgb_tc_linear / hgb_tc_wgrad against fp64 ==============================================================
TOL = {"exact": 2e-6, "tf32": 2e-3}                 # one Linear, rel-L2 against fp64 (module docstring)
MODES = ["exact", "tf32"]
ACTS = {"none": 0.0, "relu": 0.0, "silu": 0.0, "tanh": 0.0, "sigmoid": 0.0, "lrelu": 0.3, "elu": 0.0, "selu": 0.0}  # -> act_param


def mode_ctx(mode):
    """exact: the 3xTF32 split (fp32 configs, the default); tf32: plain TF32 (precision="bf16")."""
    return ops.tensor_cores(mode == "tf32")


def act64(name, z, p=0.0):
    f = torch.nn.functional
    return {"none": lambda t: t, "relu": torch.relu, "silu": f.silu, "tanh": torch.tanh, "sigmoid": torch.sigmoid,
            "lrelu": lambda t: f.leaky_relu(t, p), "elu": f.elu, "selu": f.selu}[name](z)


def dact64(name, z, p=0.0):
    """act'(z) in fp64, by autograd of the torch activation (independent of the kernels' formulas in terms of act(z))."""
    zz = z.double().detach().requires_grad_(True)
    return torch.autograd.grad(act64(name, zz, p).sum(), zz)[0]


def traced(fn, name):
    """(fn(), [(arguments, kernels launched) of every `name` call]) from the C-ABI call trace."""
    hb._lib.trace_begin()
    try:
        out = fn()
    finally:
        calls = hb._lib.trace_end()
    return out, [(c[1], c[2]) for c in calls if c[0] == name]


def wgrad_ok(dw, ref, e_simt, mode):
    """the weight-gradient bound of tests/test_gpu_round2.py::test_tc_wgrad_exact_mode_matches_fp64 (exact: within 4x of the SIMT
    fp32 GEMM, at least 5e-6) or the TF32 bound"""
    e = rel(dw, ref)
    return e < (max(5e-6, 4 * e_simt) if mode == "exact" else TOL[mode]), e


@pytest.mark.parametrize("mode", MODES)
@pytest.mark.parametrize("act", list(ACTS))
def test_tc_linear_forward_every_activation(act, mode):
    """Every epilogue activation (the __expf SiLU, tanhf, and hgb_act for sigmoid / leaky ReLU with slope 0.3 / ELU / SELU), z = the
    pre-activation.  Pre-activations have std ~2 so the saturating branches are reached."""
    assert {ops.ACT_CODES[a] for a in ACTS} == set(ops.ACT_CODES.values())
    m, k, n = 1000, 96, 160
    g = torch.Generator().manual_seed(11 + ops.ACT_CODES[act])
    x, w, b = torch.randn(m, k, generator=g), torch.randn(n, k, generator=g) * 0.2, torch.randn(n, generator=g)
    zr = x.double() @ w.double().t() + b.double()
    with mode_ctx(mode):
        (y, z), calls = traced(lambda: ops.raw_tc_linear(x.to(DEV), w.to(DEV), False, b.to(DEV), n, k, ops.ACT_CODES[act], ACTS[act],
                                                         want_z=True), "hgb_tc_linear")
    assert [c[0]["exact"] for c in calls] == [int(mode == "exact")]
    assert rel(z, zr) < TOL[mode]
    assert rel(y, act64(act, zr, ACTS[act])) < TOL[mode]


@pytest.mark.parametrize("mode", MODES)
def test_tc_linear_forward_without_bias_and_silu_derivative_in_z(mode):
    """bias = NULL; gact = HGB_ACT_DERIV with SiLU (the forward of Mlp2Fn / PainnUpdateFn under z_deriv) stores silu'(pre-activation)
    in z next to y = silu(pre-activation); with any other activation HGB_ACT_DERIV leaves z the pre-activation."""
    m, k, n = 777, 64, 128
    g = torch.Generator().manual_seed(3)
    x, w, b = torch.randn(m, k, generator=g), torch.randn(n, k, generator=g) * 0.2, torch.randn(n, generator=g)
    xd, wd, bd = x.to(DEV), w.to(DEV), b.to(DEV)
    silu, tanh = ops.ACT_CODES["silu"], ops.ACT_CODES["tanh"]
    z0 = x.double() @ w.double().t()
    zr = z0 + b.double()
    tol = TOL[mode]
    with mode_ctx(mode):
        y, z = ops.raw_tc_linear(xd, wd, False, None, n, k, silu, want_z=True)
        assert rel(z, z0) < tol and rel(y, act64("silu", z0)) < tol
        y, z = ops.raw_tc_linear(xd, wd, False, bd, n, k, silu, want_z=True, gact=ops.ACT_DERIV)
        assert rel(z, dact64("silu", zr)) < tol and rel(y, act64("silu", zr)) < tol
        y, z = ops.raw_tc_linear(xd, wd, False, bd, n, k, tanh, want_z=True, gact=ops.ACT_DERIV)
        assert rel(z, zr) < tol and rel(y, torch.tanh(zr)) < tol


@pytest.mark.parametrize("mode", MODES)
@pytest.mark.parametrize("with_addend", [False, True])
@pytest.mark.parametrize("gact", list(ACTS) + ["deriv"])
@pytest.mark.parametrize("m,n,k", [(1000, 96, 160), (700, 64, 320)])
def test_tc_dgrad_epilogue_every_gact(m, n, k, gact, with_addend, mode):
    """dX = (dZ W + addend) * act'(gsrc): the data gradient through the activation that produced the layer's input, in the dgrad
    epilogue (trans_b = 1).  gsrc is the pre-activation for SiLU, the activation output for the others, silu'(pre-activation) for
    HGB_ACT_DERIV; leaky ReLU's slope comes from act_param.  dX has k = 160 columns (one piece) or 320 (pieces 256 + 64: addend and
    gsrc are read at the piece's column offset)."""
    g = torch.Generator().manual_seed(m + k + len(gact) + 7 * with_addend)
    dz, w = torch.randn(m, n, generator=g), torch.randn(n, k, generator=g) * 0.2
    pre = torch.randn(m, k, generator=g) * 2
    add = torch.randn(m, k, generator=g) if with_addend else None
    name = "silu" if gact == "deriv" else gact
    p = ACTS[name]
    d = dact64(name, pre, p)
    gsrc = {"silu": pre, "deriv": d.float()}.get(gact)
    if gsrc is None:
        gsrc = act64(name, pre.double(), p).float()
    code = ops.ACT_DERIV if gact == "deriv" else ops.ACT_CODES[gact]
    ref = dz.double() @ w.double()
    if add is not None:
        ref = ref + add.double()
    ref = ref * d
    with mode_ctx(mode):
        dx, _ = ops.raw_tc_linear(dz.to(DEV), w.to(DEV), True, None, k, n, param=p, addend=None if add is None else add.to(DEV),
                                  gsrc=gsrc.to(DEV), gact=code)
    assert rel(dx, ref) < TOL[mode]


MLP2_CASES = [(a, mode) for mode in MODES for a in ACTS if mode == "exact" or a not in ("relu", "lrelu", "selu")]


@pytest.mark.parametrize("act1,mode", MLP2_CASES)
def test_mlp2_autograd_every_first_activation(act1, mode):
    """Mlp2Fn through autograd on the tensor-core path: the forward's choice of z (the pre-activation, or silu'(pre) under z_deriv)
    and the backward's choice of gsrc / gact must agree, for every first-layer activation; fp64 autograd of the same chain is the
    reference.  Output: the one-Linear bound.  Gradients chain two GEMMs: 5e-6 (exact, the weight-gradient bound) / 3e-3 (tf32, as
    test_linear_act_autograd_on_tensor_cores).  ReLU, leaky ReLU and SELU have a jump in act' at 0: a pre-activation closer to 0
    than the forward's error may take the other side of it, which moves a whole gradient entry.  In the exact mode that error is
    ~1e-6 absolute here (pre-activations have std ~2.2), and the rows with a pre-activation within 1e-4 of 0 get no upstream
    gradient (a handful of the 2000 rows).  In TF32 mode the band would be ~1e-2 wide and cover ~30% of the rows, so those three
    activations run in the exact mode only."""
    m, k, hdim, n = 2000, 64, 96, 64
    p1 = ACTS[act1]
    g = torch.Generator().manual_seed(40 + ops.ACT_CODES[act1])
    x, go = torch.randn(m, k, generator=g), torch.randn(m, n, generator=g)
    w1, b1 = torch.randn(hdim, k, generator=g) * 0.25, torch.randn(hdim, generator=g)
    w2, b2 = torch.randn(n, hdim, generator=g) * 0.2, torch.randn(n, generator=g)
    go[((x.double() @ w1.double().t() + b1.double()).abs() < 1e-4).any(1)] = 0
    ref_in = [t.double().requires_grad_(True) for t in (x, w1, b1, w2, b2)]
    xr, w1r, b1r, w2r, b2r = ref_in
    yr = act64(act1, xr @ w1r.t() + b1r, p1) @ w2r.t() + b2r
    gr = torch.autograd.grad(yr, ref_in, go.double())
    ins = [t.to(DEV).requires_grad_(True) for t in (x, w1, b1, w2, b2)]
    xe, w1e, b1e, w2e, b2e = ins
    with mode_ctx(mode):
        ye, calls = traced(lambda: ops.Mlp2Fn.apply(xe, w1e, b1e, act1, p1, w2e, b2e, None, 0.0), "hgb_tc_linear")
    ge, bcalls = traced(lambda: torch.autograd.grad(ye, ins, go.to(DEV)), "hgb_tc_linear")
    silu = act1 == "silu"
    assert [c[0]["gact"] for c in calls] == [ops.ACT_DERIV if silu else 0, 0]               # layer 1 stores silu'(pre) in z
    assert all(c[0]["exact"] == int(mode == "exact") for c in calls + bcalls)
    assert [c[0]["gact"] for c in bcalls if c[0]["gsrc"]] == [ops.ACT_DERIV if silu else ops.ACT_CODES[act1]]
    assert rel(ye.detach(), yr.detach()) < TOL[mode]
    tol_g = 5e-6 if mode == "exact" else 3e-3
    for name, a, b in zip(("x", "w1", "b1", "w2", "b2"), ge, gr):
        assert rel(a, b) < tol_g, (name, rel(a, b))


# (mode, n_out, k_red, piece widths): hgb_tc_linear cuts n_out into pieces of at most nc_max = (64 KB exact / 160 KB tf32) /
# (4 k_red), rounded down to a multiple of 32 and capped at 256 (hgb_tc.cu, hgb_tc_linear); a piece of width 32 NC runs
# tc_linear_kernel<NC, exact>.  k_red = 64 gives nc_max = 256 in both modes: NC = n_out / 32 for every NC = 1..8.
LINEAR_WIDTHS = [(mode, 32 * nc, 64, [32 * nc]) for mode in MODES for nc in range(1, 9)] + [
    ("exact", 224, 128, [128, 96]), ("exact", 480, 64, [256, 224]), ("tf32", 224, 256, [160, 64])]


@pytest.mark.parametrize("mode,n,k,pieces", LINEAR_WIDTHS)
def test_tc_linear_every_width_instantiation(mode, n, k, pieces):
    m = 1500
    g = torch.Generator().manual_seed(n + k)
    x, w, b = torch.randn(m, k, generator=g), torch.randn(n, k, generator=g) * 0.2, torch.randn(n, generator=g)
    zr = x.double() @ w.double().t() + b.double()
    with mode_ctx(mode):
        (y, z), calls = traced(lambda: ops.raw_tc_linear(x.to(DEV), w.to(DEV), False, b.to(DEV), n, k, ops.ACT_CODES["silu"], 0.0,
                                                         want_z=True), "hgb_tc_linear")
    assert sum(pieces) == n
    assert [(c[0]["exact"], c[1]) for c in calls] == [(int(mode == "exact"), len(pieces))]      # one kernel launch per piece
    assert rel(z, zr) < TOL[mode] and rel(y, act64("silu", zr)) < TOL[mode]


# tc_wgrad_kernel<Q = k_out / 32, exact> for every k_out the kernel takes (k_out + 16 <= 256: Q = 1..7).  raw_tc_wgrad cuts n_out
# into row pieces of 256 (k_out <= 96) or 128: n_out = 192 is one piece (two row blocks, 128 + 64 rows) for Q <= 3, and the pieces
# 128 + 64 for Q >= 4.
WGRAD_WIDTHS = [(mode, q, [192] if q <= 3 else [128, 64]) for mode in MODES for q in range(1, 8)]


@pytest.mark.parametrize("mode,q,pieces", WGRAD_WIDTHS)
def test_tc_wgrad_every_width_instantiation(mode, q, pieces):
    m, n, k = 3001, 192, 32 * q
    g = torch.Generator().manual_seed(q)
    dz, x = torch.randn(m, n, generator=g), torch.randn(m, k, generator=g)
    dzd, xd = dz.to(DEV), x.to(DEV)
    with mode_ctx(mode):
        (dw, db), calls = traced(lambda: ops.raw_tc_wgrad(dzd, xd, want_bias=True), "hgb_tc_wgrad")
    want = [(int(mode == "exact"), nc, k, 2) for nc in pieces]                                   # weight-gradient kernel + reduce
    assert [(c[0]["exact"], c[0]["n_out"], c[0]["k_out"], c[1]) for c in calls] == want
    ref_w = dz.double().t() @ x.double()
    ok, e = wgrad_ok(dw, ref_w, rel(ops.raw_gemm(dzd, xd, True, False), ref_w), mode)
    assert ok, e
    assert rel(db, dz.double().sum(0)) < (5e-6 if mode == "exact" else TOL[mode])


@pytest.mark.parametrize("mode", MODES)
@pytest.mark.parametrize("m", [128, 129, 191, 64 * 264 + 1, 64 * 264 + 63])
def test_tc_linear_tile_count_edges(m, mode):
    """m = 128..191: 2 or 3 tiles of 64 rows, one per CTA, so consumer warpgroup 1 never runs.  m = 64 * 264 + 1 / + 63: 265 =
    2 * 132 + 1 tiles on 132 CTAs, CTA 0's two consumers run 2 and 1 tiles.  m = 129, 191 and the large ones end in a tile of 1 or 63
    rows (the TMA zero-fills the rest, the epilogue masks it, also for its addend / gsrc reads).  Forward and dgrad, fp64 agreement
    and the same bits on repetition."""
    n, k = 96, 128
    g = torch.Generator().manual_seed(m)
    x, w, b = torch.randn(m, k, generator=g), torch.randn(n, k, generator=g) * 0.2, torch.randn(n, generator=g)
    dz, add, gs = torch.randn(m, n, generator=g), torch.randn(m, k, generator=g), torch.randn(m, k, generator=g)
    xd, wd, bd, dzd, addd, gsd = [t.to(DEV) for t in (x, w, b, dz, add, gs)]
    silu = ops.ACT_CODES["silu"]
    with mode_ctx(mode):
        fwd = lambda: ops.raw_tc_linear(xd, wd, False, bd, n, k, silu, 0.0, want_z=True)    # noqa: E731
        bwd = lambda: ops.raw_tc_linear(dzd, wd, True, None, k, n, addend=addd, gsrc=gsd, gact=silu)[0]    # noqa: E731
        y, z = fwd()
        dx = bwd()
        y2, z2 = fwd()
        dx2 = bwd()
    zr = x.double() @ w.double().t() + b.double()
    assert rel(z, zr) < TOL[mode] and rel(y, act64("silu", zr)) < TOL[mode]
    assert rel(dx, (dz.double() @ w.double() + add.double()) * dact64("silu", gs)) < TOL[mode]
    assert torch.equal(y, y2) and torch.equal(z, z2) and torch.equal(dx, dx2)


@pytest.mark.parametrize("mode", MODES)
@pytest.mark.parametrize("accumulate,want_bias", [(False, True), (True, True), (True, False), (False, False)])
@pytest.mark.parametrize("m,n,k,strided", [(1281, 160, 64, False), (21151, 160, 96, True), (4097, 96, 64, True), (9631, 96, 96, False)])
def test_tc_wgrad_edges(m, n, k, strided, accumulate, want_bias, mode):
    """Partial row blocks: n_out = 160 is row blocks of 128 and 32 (blockIdx.y = 1 has 32 rows: its warpgroup 1 idles and half of
    warpgroup 0's rows are zero padding), n_out = 96 one block whose warpgroup 1 has 32 padding rows.  m % 32 = 1 or 31: the last
    32-row chunk is mostly TMA zero fill; m = 21151 gives 11 chunks per CTA (the exact mode folds its accumulators after 8) and a
    last CTA with 1 chunk.  accumulate = 1 adds into prefilled dw / db, accumulate = 0 overwrites NaN; want_bias = False passes
    db = NULL.  ``strided``: x is a column block of a wider tensor (ldx = k + 8).  fp64 agreement and the same bits on repetition."""
    g = torch.Generator().manual_seed(m + n + k)
    dz, x = torch.randn(m, n, generator=g), torch.randn(m, k, generator=g)
    dw0, db0 = torch.randn(n, k, generator=g), torch.randn(n, generator=g)
    dzd = dz.to(DEV)
    xd = torch.cat([torch.randn(m, 4, generator=g), x, torch.randn(m, 4, generator=g)], 1).to(DEV)[:, 4:4 + k] if strided else x.to(DEV)
    assert xd.stride(0) == (k + 8 if strided else k)

    def run():
        init = (lambda t: t.to(DEV)) if accumulate else (lambda t: torch.full(t.shape, float("nan"), device=DEV))
        dw, db = init(dw0), (init(db0) if want_bias else None)
        with mode_ctx(mode):
            return ops.raw_tc_wgrad(dzd, xd, want_bias=want_bias, dw=dw, db=db, accumulate=accumulate)

    (dw, db), calls = traced(run, "hgb_tc_wgrad")
    assert [(c[0]["exact"], c[0]["ldx"], c[0]["accumulate"], c[0]["db"] is None) for c in calls] == \
        [(int(mode == "exact"), xd.stride(0), int(accumulate), not want_bias)]
    ref_w, ref_b = dz.double().t() @ x.double(), dz.double().sum(0)
    if accumulate:
        ref_w, ref_b = ref_w + dw0.double(), ref_b + db0.double()
    ok, e = wgrad_ok(dw, ref_w, rel(ops.raw_gemm(dzd, xd, True, False), dz.double().t() @ x.double()), mode)
    assert ok, e
    if want_bias:
        assert rel(db, ref_b) < (5e-6 if mode == "exact" else TOL[mode])
    else:
        assert db is None
    dw2, db2 = run()
    assert torch.equal(dw, dw2) and (db is None or torch.equal(db, db2))


@pytest.mark.parametrize("mode", MODES)
def test_tc_strided_operands(mode):
    """Operands that are column blocks of wider tensors: the TMA-fed A operand (lda = k + 40 > k, start 16 bytes into the row), the
    forward weight staged by plain loads (ldw = k + 7 > k at an odd column offset), the dgrad weight (trans_b = 1, ldw = k + 5 >
    n_out = k) and the weight gradient's dz / x (lddz = n + 8, ldx = k + 8)."""
    m, n, k = 1500, 96, 128
    g = torch.Generator().manual_seed(8)
    a, w, b = torch.randn(m, k, generator=g), torch.randn(n, k, generator=g) * 0.2, torch.randn(n, generator=g)
    dz, w_t = torch.randn(m, n, generator=g), torch.randn(n, k, generator=g) * 0.2

    def block(t, left, right):      # t as columns left.. of a wider device tensor
        wide = torch.cat([torch.randn(t.shape[0], left, generator=g), t, torch.randn(t.shape[0], right, generator=g)], 1).to(DEV)
        return wide[:, left:left + t.shape[1]]

    ad, wd, w_td, dzd = block(a, 4, 36), block(w, 3, 4), block(w_t, 1, 4), block(dz, 4, 4)
    assert (ad.stride(0), wd.stride(0), w_td.stride(0), dzd.stride(0)) == (k + 40, k + 7, k + 5, n + 8)
    xd = block(a, 4, 4)
    zr = a.double() @ w.double().t() + b.double()
    tol = TOL[mode]
    with mode_ctx(mode):
        y, z = ops.raw_tc_linear(ad, wd, False, b.to(DEV), n, k, ops.ACT_CODES["silu"], 0.0, want_z=True)
        assert rel(z, zr) < tol and rel(y, act64("silu", zr)) < tol
        dx, _ = ops.raw_tc_linear(dzd, w_td, True, None, k, n)
        assert rel(dx, dz.double() @ w_t.double()) < tol
        dw, db = ops.raw_tc_wgrad(dzd, xd, want_bias=True)
    ref_w = dz.double().t() @ a.double()
    ok, e = wgrad_ok(dw, ref_w, rel(ops.raw_gemm(dzd, xd, True, False), ref_w), mode)
    assert ok, e
    assert rel(db, dz.double().sum(0)) < (5e-6 if mode == "exact" else tol)


@pytest.mark.parametrize("block", ["addend", "gsrc"])
@pytest.mark.parametrize("m", [1000, 100])
def test_bwd_dispatch_column_block_epilogue_operands(m, block):
    """linear_bwd_dispatch with dx_addend or dx_gsrc handed over as a column block of a wider tensor (row stride 2k, 16-byte aligned,
    so it passes tc_ok): the tensor-core epilogue reads both with dx's row stride k and hgb_act_bwd reads gsrc as a flat array, so
    the dispatcher has to make them dense.  m = 1000 runs on hgb_tc_linear (fp32 mode: exact), m = 100 (< 128 rows) on the SIMT GEMM
    and hgb_act_bwd."""
    n, k = 64, 96
    g = torch.Generator().manual_seed(m)
    dz, x, w = torch.randn(m, n, generator=g), torch.randn(m, k, generator=g), torch.randn(n, k, generator=g) * 0.2
    add, gs = torch.randn(m, k, generator=g), torch.tanh(torch.randn(m, k, generator=g) * 2)
    addd, gsd = add.to(DEV), gs.to(DEV)
    if block == "addend":
        addd = torch.cat([torch.randn(m, k, generator=g), add], 1).to(DEV)[:, k:]
    else:
        gsd = torch.cat([torch.randn(m, k, generator=g), gs], 1).to(DEV)[:, k:]
    (dx, _, _), calls = traced(lambda: ops.linear_bwd_dispatch(dz.to(DEV), x.to(DEV), w.to(DEV), True, False, False, dx_addend=addd,
                                                               dx_gsrc=gsd, dx_gact=ops.ACT_CODES["tanh"]), "hgb_tc_linear")
    assert len(calls) == (1 if m >= 128 else 0)
    ref = (dz.double() @ w.double() + add.double()) * (1 - gs.double() ** 2)
    assert rel(dx, ref) < 2e-6
    if m >= 128:                    # the raw launcher refuses such an operand instead of reading the wrong rows
        with pytest.raises(RuntimeError, match="dense row-major"):
            ops.raw_tc_linear(dz.to(DEV), w.to(DEV), True, None, k, n, addend=addd, gsrc=gsd, gact=ops.ACT_CODES["tanh"])
