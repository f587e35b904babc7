"""GPU parity tests of the wgmma (TF32) dense-layer kernels against fp64 references.
Tolerance: TF32 truncates operands to 10 mantissa bits -> relative L2 error <= 2e-3 (well inside the 2e-2 the
bf16 config allows, SURVEY 8d)."""
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
