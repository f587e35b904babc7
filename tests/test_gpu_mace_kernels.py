"""The MACE kernels one by one against fp64: every generated specialisation of the fused tensor product + receiver scatter
(hgb_mace_tp_scatter_{fwd,bwd}) and of the correlation-2 symmetric contraction (hgb_mace_symcontract_{fwd,bwd}), the closed
any-order primitives (hgb_mace_tp_path, hgb_mace_chan_contract), the edge embedding (hgb_mace_edge_embed_{fwd,bwd}), launches
large enough for every grid-stride loop to run, and the fused path against the any-order path on the same inputs.

References are plain fp64 torch written from the mathematics.  Their coupling numbers come from oracle/e3.py and oracle/mace.py
(wigner_3j, u_matrix_real), never from hydragnn_b200/e3.py, which is what csrc/gen_mace.py reads: a wrong table in one of the
two shows up as a difference.  The CPU tests at the top check the references themselves against the oracle's modules.

Bounds: relative L2 <= 1e-5 against fp64 for values and first derivatives, <= 1e-4 for second and third derivatives and for
weight gradients reduced over 20,480 nodes; any other bound is stated where it is used."""
import math
import types

import pytest
import torch

from hydragnn_b200 import _lib, e3, mace, ops
from oracle import e3 as oe3
from oracle import mace as omace

gpu = pytest.mark.gpu
DEV = "cuda"
TP_PAIRS = [(lin, lsh) for lsh in (1, 2, 3) for lin in (0, 1, 2) if lin <= lsh]       # the 8 generated MaceTP<lin, lsh>
SC_PAIRS = [(lin, lout) for lin in (1, 2, 3) for lout in (0, 1, 2) if lout <= lin]   # the 8 generated MaceSC<lin, lout>
NUM_ELEMENTS = 118


def rel_l2(a, b):
    a, b = a.detach().double().cpu(), b.detach().double().cpu()
    assert a.shape == b.shape, (a.shape, b.shape)
    return float((a - b).norm() / b.norm().clamp(min=1e-30))


def _gen(*key):
    seed = 0
    for k in key:
        seed = seed * 1009 + int(k) + 1
    return torch.Generator().manual_seed(seed)


def _randn(gen, *shape):
    return torch.randn(*shape, generator=gen, dtype=torch.float64)


# =====================================================================================================================
# fp64 references
# =====================================================================================================================
def _paths(lin, lsh):
    """(l1, l2, l3) of every tensor-product path in the order of the per-edge weight blocks: generated l1 outer, l2 inner,
    l3 ascending, then stably sorted by the output degree."""
    gen = [(l1, l2, l3) for l1 in range(lin + 1) for l2 in range(lsh + 1) for l3 in range(abs(l1 - l2), min(l1 + l2, lsh) + 1)
           if (l1 + l2 + l3) % 2 == 0]
    return sorted(gen, key=lambda t: t[2])


def _cg(l1, l2, l3):
    """c C[m1, m2, m3] with c = sqrt(2 l3 + 1): component normalisation, one path per output slot."""
    return oe3.wigner_3j(l1, l2, l3) * math.sqrt(2 * l3 + 1)


def _tp_messages(x_e, sh, tpw, ea, lin, lsh):
    """Per-edge messages of conv_tp, per output degree l3 a [E, 2 l3 + 1, n_paths(l3) F] tensor.  x_e [E, S_in, F] are the
    sender rows.  With edge attributes ea [E, D] a path whose edge irrep is 0e reads a [F, D + 1] weight block mixed with
    [ea, 1] / sqrt(D + 1); every other path F weights."""
    f, d = x_e.shape[2], 0 if ea is None else ea.shape[1]
    a = None if d == 0 else torch.cat([ea, torch.ones_like(ea[:, :1])], dim=1)
    per_l, col = [[] for _ in range(lsh + 1)], 0
    for (l1, l2, l3) in _paths(lin, lsh):
        if l2 == 0 and d:
            w = torch.einsum("euv,ev->eu", tpw[:, col:col + f * (d + 1)].reshape(-1, f, d + 1), a) / math.sqrt(d + 1)
            col += f * (d + 1)
        else:
            w = tpw[:, col:col + f]
            col += f
        t = torch.einsum("ijk,ej->eik", _cg(l1, l2, l3), sh[:, l2 * l2:(l2 + 1) ** 2])
        per_l[l3].append(torch.einsum("eik,eif->ekf", t, x_e[:, l1 * l1:(l1 + 1) ** 2]) * w[:, None, :])
    assert col == tpw.shape[1]
    return [torch.cat(p, dim=2) for p in per_l]


def _tp_scatter_ref(up, sh, tpw, ea, ei, n, lin, lsh):
    """conv_tp + scatter-sum over receivers, packed like the kernel's output: per l3 a [n, 2 l3 + 1, n_paths F] block."""
    msgs = _tp_messages(up[ei[0]], sh, tpw, ea, lin, lsh)
    return torch.cat([m.new_zeros((n,) + m.shape[1:]).index_add_(0, ei[1], m).reshape(-1) for m in msgs])


def _tp_blocks(packed, n, f, lin, lsh):
    """views [n, 2 l3 + 1, n_paths(l3) f] of the packed buffer"""
    out, off, paths = [], 0, _paths(lin, lsh)
    for l3 in range(lsh + 1):
        width = sum(1 for q in paths if q[2] == l3) * f
        size = n * (2 * l3 + 1) * width
        out.append(packed[off:off + size].view(n, 2 * l3 + 1, width))
        off += size
    assert off == packed.numel()
    return out


def _tp_weight_cols(lin, lsh, f, d):
    return sum(f * (d + 1 if l2 == 0 else 1) for (_, l2, _) in _paths(lin, lsh))


def _sc_tables(lin, lout):
    """Per output degree l the coupling tensors of the oracle: U2 [2l+1, S, S, K2] and U1 [2l+1, S, K1]."""
    coupling = oe3.Irreps([(1, (l, (-1) ** l)) for l in range(lin + 1)])
    s, out = (lin + 1) ** 2, []
    for l in range(lout + 1):
        ir = oe3.Irrep(l, (-1) ** l)
        u2 = omace.u_matrix_real(coupling, ir, 2).reshape(2 * l + 1, s, s, -1)
        u1 = omace.u_matrix_real(coupling, ir, 1).reshape(2 * l + 1, s, -1)
        out.append((u2, u1))
    return out


def _sc_num_weights(lin, lout):
    return sum(u2.shape[-1] + u1.shape[-1] for u2, u1 in _sc_tables(lin, lout))


def _sc_ref(x, wall, z, gout, lin, lout):
    """out[b, m, c] = sum U2[m,i,j,k] W2[z_b,k,c] x[b,i,c] x[b,j,c] + sum U1[m,i,k] W1[z_b,k,c] x[b,i,c] for every output degree,
    wall [118, KTOT, F] = (W2 | W1) per output degree.  Returns (out, gx, gwall) in fp64; the work is done element by element so
    that the largest intermediate is [nodes of one element, 2l+1, S, F]."""
    tables = _sc_tables(lin, lout)
    n, _, f = x.shape
    out = x.new_zeros(n, (lout + 1) ** 2, f)
    gx, gwall = torch.zeros_like(x), torch.zeros_like(wall)
    for el in torch.unique(z).tolist():
        rows = (z == el).nonzero().squeeze(1)
        xe = x[rows].clone().requires_grad_(True)
        we = wall[el].clone().requires_grad_(True)
        parts, k = [], 0
        for (u2, u1) in tables:
            w2, w1 = we[k:k + u2.shape[-1]], we[k + u2.shape[-1]:k + u2.shape[-1] + u1.shape[-1]]
            k += u2.shape[-1] + u1.shape[-1]
            t2 = torch.einsum("mijk,kc->mijc", u2, w2)
            t1 = torch.einsum("mik,kc->mic", u1, w1)
            inner = torch.einsum("mijc,bjc->bmic", t2, xe) + t1[None]
            parts.append(torch.einsum("bmic,bic->bmc", inner, xe))
        assert k == wall.shape[1]
        o = torch.cat(parts, dim=1)
        if gout is not None:
            g1, g2 = torch.autograd.grad(o, (xe, we), gout[rows])
            gx[rows] = g1
            gwall[el] = g2
        out[rows] = o.detach()
    return out, gx, gwall


def _embed_ref(vec, lmax, nb, rc, p):
    """spherical harmonics (component normalisation) of vec / |vec| and Bessel basis x polynomial cutoff of |vec|, fp64"""
    d = vec.norm(dim=1, keepdim=True)
    sh = oe3.spherical_harmonics(lmax, vec, normalize=True, normalization="component")
    x = d / rc
    env = (1.0 - ((p + 1.0) * (p + 2.0) / 2.0) * x.pow(p) + p * (p + 2.0) * x.pow(p + 1) - (p * (p + 1.0) / 2) * x.pow(p + 2)) * (d < rc)
    w = math.pi / rc * torch.arange(1, nb + 1, dtype=torch.float64)
    return sh, math.sqrt(2.0 / rc) * torch.sin(w * d) / d * env


TP_REFS = {
    "TpOut": lambda a, y, w, c: torch.einsum("ijk,eif,ej->ekf", c, a, y) * w[:, None, :],
    "TpY": lambda a, g, w, c: torch.einsum("ijk,eif,ekf,ef->ej", c, a, g, w),
    "TpW": lambda a, y, g, c: torch.einsum("ijk,eif,ej,ekf->ef", c, a, y, g),
}
CHAN_REFS = {
    "ChanCL": lambda t, x: torch.einsum("bcpi,bic->bcp", t, x),
    "ChanOU": lambda g, x: torch.einsum("bcp,bic->bcpi", g, x),
    "ChanRP": lambda g, t: torch.einsum("bcp,bcpi->bic", g, t),
}


def _chain(fn, operands, probes):
    """[value, first derivatives, second, third]: every order differentiates sum_i <g_i, probe_i> of the previous one with
    respect to every operand (create_graph), and stops where the expression no longer depends on the operands (a map that is
    linear in each of its k operands has no derivative beyond order k)."""
    cur = [fn(*operands)]
    res = [list(cur)]
    for pr in probes:
        loss = sum((c * q.to(c)).sum() for c, q in zip(cur, pr))
        if not loss.requires_grad:
            break
        cur = list(torch.autograd.grad(loss, operands, create_graph=True, allow_unused=True, materialize_grads=True))
        res.append(cur)
    return res


def _assert_chain_close(dev, ref, what):
    assert len(dev) == len(ref), (what, len(dev), len(ref))
    for order, (ds, rs) in enumerate(zip(dev, ref)):
        for i, (a, b) in enumerate(zip(ds, rs)):
            tol = 1e-5 if order <= 1 else 1e-4
            if b.numel() < 32:
                tol *= 10         # a few sums of up to 245 cancelling terms carry the whole norm: one unlucky sum is not diluted
            assert rel_l2(a, b) < tol, (what, "order", order, "operand", i, rel_l2(a, b))


# =====================================================================================================================
# CPU: the tables agree, and the references agree with the oracle's modules
# =====================================================================================================================
def test_engine_and_oracle_coupling_tables_agree():
    """Every degree the generator uses: w3j against wigner_3j for l <= 3, u_matrix against u_matrix_real for the 8 contraction
    pairs at correlation 1 and 2; the path order against tp_out_irreps_with_instructions."""
    for l1 in range(4):
        for l2 in range(4):
            for l3 in range(abs(l1 - l2), min(l1 + l2, 3) + 1):
                assert torch.allclose(e3.w3j(l1, l2, l3), oe3.wigner_3j(l1, l2, l3), atol=1e-12, rtol=0), (l1, l2, l3)
    for lin in (1, 2, 3):
        coupling = oe3.Irreps([(1, (l, (-1) ** l)) for l in range(lin + 1)])
        for lout in range(min(lin, 2) + 1):
            for nu in (1, 2):
                a, b = e3.u_matrix(lin, lout, nu), omace.u_matrix_real(coupling, oe3.Irrep(lout, (-1) ** lout), nu)
                assert a.shape == b.shape and torch.allclose(a, b, atol=1e-12, rtol=0), (lin, lout, nu)
    for lin, lsh in TP_PAIRS:
        assert _paths(lin, lsh) == e3.tp_paths(lin, lsh, lsh)
        feats, sh = oe3.Irreps([(2, (l, (-1) ** l)) for l in range(lin + 1)]), oe3.Irreps.spherical_harmonics(lsh)
        target = oe3.Irreps([(2, (l, (-1) ** l)) for l in range(lsh + 1)])
        _, ins = omace.tp_out_irreps_with_instructions(feats, sh, target)
        mid = [(feats[i1][1].l, sh[i2][1].l) for i1, i2, _, _, _ in ins]
        assert mid == [(l1, l2) for l1, l2, _ in _paths(lin, lsh)], (lin, lsh)


@pytest.mark.parametrize("lin,lsh", TP_PAIRS)
def test_tp_reference_matches_oracle_tensor_product(lin, lsh):
    """_tp_scatter_ref (channel-last, per-degree blocks) against oracle.e3.TensorProductUVU (e3nn's mul-major rows) + index_add_"""
    gen, f, n, e = _gen(1, lin, lsh), 3, 6, 17
    ei = torch.randint(0, n, (2, e), generator=gen)
    up, sh = _randn(gen, n, (lin + 1) ** 2, f), _randn(gen, e, (lsh + 1) ** 2)
    tpw = _randn(gen, e, _tp_weight_cols(lin, lsh, f, 0))
    feats, shi = oe3.Irreps([(f, (l, (-1) ** l)) for l in range(lin + 1)]), oe3.Irreps.spherical_harmonics(lsh)
    target = oe3.Irreps([(f, (l, (-1) ** l)) for l in range(lsh + 1)])
    mid, ins = omace.tp_out_irreps_with_instructions(feats, shi, target)
    tp = oe3.TensorProductUVU(feats, shi, mid, ins)
    x1 = torch.cat([up[:, l * l:(l + 1) ** 2].transpose(1, 2).reshape(n, -1) for l in range(lin + 1)], dim=1)   # mul-major rows
    mji = tp(x1[ei[0]], sh, tpw)
    agg = torch.zeros(n, mji.shape[1], dtype=torch.float64).index_add_(0, ei[1], mji)
    mine = _tp_blocks(_tp_scatter_ref(up, sh, tpw, None, ei, n, lin, lsh), n, f, lin, lsh)
    col = 0
    for l3, blk in enumerate(mine):                               # oracle columns: per path [F, 2 l3 + 1], paths sorted by l3
        n_p = blk.shape[2] // f
        ref = agg[:, col:col + n_p * f * (2 * l3 + 1)].reshape(n, n_p, f, 2 * l3 + 1).permute(0, 3, 1, 2).reshape(n, 2 * l3 + 1, n_p * f)
        col += n_p * f * (2 * l3 + 1)
        assert torch.allclose(blk, ref, atol=1e-12), (l3, float((blk - ref).abs().max()))
    assert col == agg.shape[1]


@pytest.mark.parametrize("lin,lout", SC_PAIRS)
def test_sc_reference_matches_oracle_contraction(lin, lout):
    """_sc_ref against oracle.mace.Contraction per output degree, weights laid out as Product.forward concatenates them"""
    torch.manual_seed(10 * lin + lout)
    gen, f, n = _gen(2, lin, lout), 3, 7
    irreps_in = oe3.Irreps([(f, (l, (-1) ** l)) for l in range(lin + 1)])
    torch.set_default_dtype(torch.float64)                  # the oracle stores its U matrices in the default dtype
    try:
        cons = [omace.Contraction(irreps_in, oe3.Irrep(l, (-1) ** l), 2, NUM_ELEMENTS) for l in range(lout + 1)]
    finally:
        torch.set_default_dtype(torch.float32)
    wall = torch.cat([w.detach() for c in cons for w in (c.weights_max, c.weights[0])], dim=1)
    assert wall.shape[1] == _sc_num_weights(lin, lout)
    x = _randn(gen, n, (lin + 1) ** 2, f)
    z = torch.tensor([0, 117, 5, 5, 0, 64, 5])
    onehot = torch.nn.functional.one_hot(z, NUM_ELEMENTS).double()
    out, _, _ = _sc_ref(x, wall, z, None, lin, lout)
    for l, c in enumerate(cons):
        ref = c(x.transpose(1, 2), onehot).reshape(n, f, 2 * l + 1).transpose(1, 2)
        assert torch.allclose(out[:, l * l:(l + 1) ** 2], ref.detach(), atol=1e-12), l


def test_embed_and_primitive_references_run_on_cpu():
    gen = _gen(3)
    sh, rad = _embed_ref(_randn(gen, 9, 3) * 3, 3, 8, 6.0, 5.0)
    assert sh.shape == (9, 16) and rad.shape == (9, 8) and torch.allclose(sh.pow(2).sum(1), torch.full((9,), 16.0, dtype=torch.float64))
    c, a, y, w, g = _cg(2, 3, 3), _randn(gen, 4, 5, 2), _randn(gen, 4, 7), _randn(gen, 4, 2), _randn(gen, 4, 7, 2)
    lhs = (TP_REFS["TpOut"](a, y, w, c) * g).sum()                      # the three forms are one trilinear form
    assert torch.allclose(lhs, (TP_REFS["TpY"](a, g, w, c) * y).sum()) and torch.allclose(lhs, (TP_REFS["TpW"](a, y, g, c) * w).sum())
    t, x, q = _randn(gen, 3, 2, 5, 4), _randn(gen, 3, 4, 2), _randn(gen, 3, 2, 5)
    lhs = (CHAN_REFS["ChanCL"](t, x) * q).sum()
    assert torch.allclose(lhs, (CHAN_REFS["ChanOU"](q, x) * t).sum()) and torch.allclose(lhs, (CHAN_REFS["ChanRP"](q, t) * x).sum())


# =====================================================================================================================
# A. hgb_mace_tp_scatter_{fwd,bwd}
# =====================================================================================================================
N_EDGE_CASE = 48
NO_INCOMING = [0] + list(range(40, N_EDGE_CASE))


def _edge_case_graph(gen):
    """48 nodes holding at once: receivers with 0 (node 0, nodes 40..47), 1, 2, 128 and 300 incoming edges (nodes 1..4), senders
    that are their own receivers, duplicate edges, and an edge order that is not sorted by receiver."""
    n = N_EDGE_CASE
    rcv = [1] + [2] * 2 + [3] * 128 + [4] * 300
    snd = torch.randint(0, n, (len(rcv),), generator=gen).tolist()
    snd[5], snd[200] = 3, 4                                                     # self loops inside the long segments
    r2 = torch.randint(5, 40, (200,), generator=gen).tolist()
    s2 = torch.randint(0, n, (200,), generator=gen).tolist()
    r2, s2 = r2 + r2[:20] + [7, 9], s2 + s2[:20] + [7, 9]                       # 20 duplicates, two more self loops
    ei = torch.tensor([snd + s2, rcv + r2])
    ei = ei[:, torch.randperm(ei.shape[1], generator=gen)]
    deg = torch.bincount(ei[1], minlength=n)
    assert deg[1:5].tolist() == [1, 2, 128, 300] and int(deg[NO_INCOMING].sum()) == 0
    assert not bool((ei[1][1:] >= ei[1][:-1]).all())
    return ei, n


def _tp_inputs(gen, ei, n, lin, lsh, f, d):
    e = ei.shape[1]
    up, sh = _randn(gen, n, (lin + 1) ** 2, f), _randn(gen, e, (lsh + 1) ** 2)
    tpw = _randn(gen, e, _tp_weight_cols(lin, lsh, f, d))
    ea = _randn(gen, e, d) if d else None
    gout = _randn(gen, _lib.query("hgb_mace_tp_num_acc", lin, lsh) * n * f)
    return up, sh, tpw, ea, gout


def _tp_run(up, sh, tpw, ea, gout, plan, lin, lsh, sh_grad=True):
    leaves = [up.float().to(DEV).requires_grad_(True), sh.float().to(DEV).requires_grad_(sh_grad), tpw.float().to(DEV).requires_grad_(True)]
    out = ops.MaceTpScatterFn.apply(leaves[0], leaves[1], leaves[2], plan, lin, lsh, None if ea is None else ea.float().to(DEV))
    wanted = [t for t in leaves if t.requires_grad]
    grads = torch.autograd.grad(out, wanted, gout.float().to(DEV))
    return [out.detach()] + list(grads)


# F = 32: one pass of one channel per lane; 64, 128, 192: passes of two channels per lane where NACC allows it (forward
# NACC <= 40, backward NACC <= 24), else 2, 4, 6 passes of one; 96, 160: always one channel per lane, 3 and 5 passes.  d = 0: the
# MaceStage kernels; 3 and 16: MaceStageEdge, 16 being the bound with the 140 KB stage of (2, 2).  No case is pruned: the
# whole product is 144 launches pairs on a 48-node graph.
@gpu
@pytest.mark.parametrize("d", [0, 3, 16])
@pytest.mark.parametrize("f", [32, 64, 96, 128, 160, 192])
@pytest.mark.parametrize("lin,lsh", TP_PAIRS)
def test_tp_scatter_matches_fp64(lin, lsh, f, d):
    gen = _gen(4, lin, lsh, f, d)
    ei, n = _edge_case_graph(gen)
    up, sh, tpw, ea, gout = _tp_inputs(gen, ei, n, lin, lsh, f, d)
    for blk in _tp_blocks(gout, n, f, lin, lsh):
        blk[NO_INCOMING] = 0.0
    leaves = [t.clone().requires_grad_(True) for t in (up, sh, tpw)]
    ref = _tp_scatter_ref(*leaves, ea, ei, n, lin, lsh)
    g_ref = torch.autograd.grad(ref, leaves, gout)
    # on the device the message gradient of a node without incoming edges is NaN: a kernel that reads it poisons its output
    gout_dev = gout.clone()
    for blk in _tp_blocks(gout_dev, n, f, lin, lsh):
        blk[NO_INCOMING] = float("nan")
    plan = ops.EdgePlan(ei.to(DEV), n)
    runs = [_tp_run(up, sh, tpw, ea, gout_dev, plan, lin, lsh) for _ in range(2)]
    assert rel_l2(runs[0][0], ref) < 1e-5, rel_l2(runs[0][0], ref)
    for name, a, b in zip(("up", "sh", "tpw"), runs[0][1:], g_ref):
        assert rel_l2(a, b) < 1e-5, (name, rel_l2(a, b))
    for blk in _tp_blocks(runs[0][0], n, f, lin, lsh):                         # nodes without incoming edges: exact zeros
        assert float(blk[NO_INCOMING].abs().max()) == 0.0
    for a, b in zip(runs[0], runs[1]):                                         # summation order = CSR order: same bits, also for
        assert torch.equal(a, b)                                               # g_sh at F = 160 (five atomicAdd passes per edge)


@gpu
@pytest.mark.parametrize("d", [0, 3])
@pytest.mark.parametrize("f", [64, 96])
@pytest.mark.parametrize("lin,lsh", TP_PAIRS)
def test_tp_scatter_backward_without_harmonics_gradient(lin, lsh, f, d):
    """NEED_Y = false (every run that does not differentiate the positions): g_up and g_tpw have the bits of the NEED_Y = true run"""
    gen = _gen(5, lin, lsh, f, d)
    ei, n = _edge_case_graph(gen)
    up, sh, tpw, ea, gout = _tp_inputs(gen, ei, n, lin, lsh, f, d)
    plan = ops.EdgePlan(ei.to(DEV), n)
    with_y = _tp_run(up, sh, tpw, ea, gout, plan, lin, lsh)
    without = _tp_run(up, sh, tpw, ea, gout, plan, lin, lsh, sh_grad=False)
    assert torch.equal(with_y[0], without[0]) and torch.equal(with_y[1], without[1]) and torch.equal(with_y[3], without[2])
    leaves = [t.clone().requires_grad_(True) for t in (up, tpw)]
    ref = _tp_scatter_ref(leaves[0], sh, leaves[1], ea, ei, n, lin, lsh)
    g_ref = torch.autograd.grad(ref, leaves, gout)
    assert rel_l2(without[1], g_ref[0]) < 1e-5 and rel_l2(without[2], g_ref[1]) < 1e-5


@gpu
@pytest.mark.parametrize("lin,lsh", [(1, 2), (2, 2)])
def test_tp_scatter_at_benchmark_size(lin, lsh):
    """20,480 nodes x about 40 edges, F = 64: with 4 nodes per block and 2,112 blocks every warp strides to a third node and
    re-uses its two shared-memory stages.  (1, 2) takes two channels per lane both ways, (2, 2) two forward and one backward.
    The full fp64 reference would take minutes on the CPU, so it is evaluated on subsets: 2,000 random output rows (all their
    incoming edges), g_tpw and g_sh of 50,000 random edges, g_up of 500 random senders (all their outgoing edges)."""
    n, f, deg = 20480, 64, 40
    e = n * deg
    gen = torch.Generator(device=DEV).manual_seed(100 * lin + lsh)
    cpu_gen = _gen(6, lin, lsh)
    ei = torch.randint(0, n, (2, e), generator=gen, device=DEV)
    up = torch.randn(n, (lin + 1) ** 2, f, generator=gen, device=DEV)
    sh = torch.randn(e, (lsh + 1) ** 2, generator=gen, device=DEV)
    tpw = torch.randn(e, _tp_weight_cols(lin, lsh, f, 0), generator=gen, device=DEV)
    gout = torch.randn(_lib.query("hgb_mace_tp_num_acc", lin, lsh) * n * f, generator=gen, device=DEV)
    assert n > 2 * 4 * 2112
    plan = ops.EdgePlan(ei, n)
    leaves = [t.clone().requires_grad_(True) for t in (up, sh, tpw)]
    out = ops.MaceTpScatterFn.apply(*leaves, plan, lin, lsh, None)
    g_up, g_sh, g_tpw = torch.autograd.grad(out, leaves, gout)
    out_blocks, gout_blocks = _tp_blocks(out.detach(), n, f, lin, lsh), _tp_blocks(gout, n, f, lin, lsh)

    def edge_ref(ids):
        """fp64 messages and per-edge gradients of the edges `ids` (device index tensor)"""
        snd, rcv = ei[0][ids], ei[1][ids]
        x_e = up[snd].double().cpu().requires_grad_(True)
        sh_e, w_e = sh[ids].double().cpu().requires_grad_(True), tpw[ids].double().cpu().requires_grad_(True)
        msgs = _tp_messages(x_e, sh_e, w_e, None, lin, lsh)
        loss = sum((m * g[rcv].double().cpu()).sum() for m, g in zip(msgs, gout_blocks))
        return [m.detach() for m in msgs], torch.autograd.grad(loss, (x_e, sh_e, w_e)), snd.cpu(), rcv.cpu()

    rows = torch.randperm(n, generator=cpu_gen)[:2000].to(DEV)
    slot = torch.full((n,), -1, dtype=torch.long, device=DEV)
    slot[rows] = torch.arange(rows.numel(), device=DEV)
    ids = (slot[ei[1]] >= 0).nonzero().squeeze(1)
    msgs, _, _, rcv = edge_ref(ids)
    for m, blk in zip(msgs, out_blocks):
        ref = m.new_zeros((rows.numel(),) + m.shape[1:]).index_add_(0, slot.cpu()[rcv], m)
        assert rel_l2(blk[rows], ref) < 1e-5, rel_l2(blk[rows], ref)

    ids = torch.randperm(e, generator=cpu_gen)[:50000].to(DEV)
    _, (_, r_sh, r_tpw), _, _ = edge_ref(ids)
    assert rel_l2(g_tpw[ids], r_tpw) < 1e-5 and rel_l2(g_sh[ids], r_sh) < 1e-5, (rel_l2(g_tpw[ids], r_tpw), rel_l2(g_sh[ids], r_sh))

    senders = torch.randperm(n, generator=cpu_gen)[:500].to(DEV)
    slot.fill_(-1)
    slot[senders] = torch.arange(senders.numel(), device=DEV)
    ids = (slot[ei[0]] >= 0).nonzero().squeeze(1)
    _, (r_x, _, _), snd, _ = edge_ref(ids)
    ref = r_x.new_zeros((senders.numel(),) + r_x.shape[1:]).index_add_(0, slot.cpu()[snd], r_x)
    assert rel_l2(g_up[senders], ref) < 1e-5, rel_l2(g_up[senders], ref)


def _empty_plan(n):
    """the index plan of a graph of n nodes without edges"""
    i32 = lambda k: torch.zeros(k, dtype=torch.int32, device=DEV)  # noqa: E731
    csr = ops.Csr(i32(0), i32(n + 1), i32(0), n)
    return types.SimpleNamespace(by_row=csr, by_col=csr, num_nodes=n, num_edges=0, nbr=lambda which: i32(0))


@gpu
@pytest.mark.parametrize("n", [0, 5])
@pytest.mark.parametrize("d", [0, 3])
def test_tp_scatter_without_edges_or_nodes(n, d):
    """E = 0: the forward returns zeros of the packed shape (not torch.empty contents), the backward zeros of the operands' shapes"""
    lin, lsh, f = 1, 2, 64
    up = torch.randn(n, 4, f, device=DEV, requires_grad=True)
    sh = torch.zeros(0, 9, device=DEV, requires_grad=True)
    tpw = torch.zeros(0, _tp_weight_cols(lin, lsh, f, d), device=DEV, requires_grad=True)
    ea = torch.zeros(0, d, device=DEV) if d else None
    out = ops.MaceTpScatterFn.apply(up, sh, tpw, _empty_plan(n), lin, lsh, ea)
    assert out.shape == (21 * n * f,) and bool((out == 0).all())
    g_up, g_sh, g_tpw = torch.autograd.grad(out, (up, sh, tpw), torch.ones_like(out))
    assert g_up.shape == up.shape and bool((g_up == 0).all()) and g_sh.shape == sh.shape and g_tpw.shape == tpw.shape


class _TpRaw:
    """Operands of raw hgb_mace_tp_scatter_* calls on a random 37-node graph"""

    def __init__(self, lin, lsh, f, d, sh_cols, seed):
        gen = _gen(7, seed)
        self.n, self.e, self.f, self.lin, self.lsh, self.d = 37, 260, f, lin, lsh, d
        ei = torch.stack([torch.randint(0, self.n, (self.e,), generator=gen), torch.randint(0, self.n - 6, (self.e,), generator=gen)])
        self.plan = ops.EdgePlan(ei.to(DEV), self.n)
        dev = lambda *s: torch.randn(*s, generator=gen).to(DEV)  # noqa: E731
        self.up, self.sh, self.tpw = dev(self.n, (lin + 1) ** 2, f), dev(self.e, sh_cols), dev(self.e, _tp_weight_cols(lin, lsh, f, d))
        self.ea = dev(self.e, d) if d else None
        self.nacc = _lib.query("hgb_mace_tp_num_acc", lin, lsh)
        self.gout = dev(max(self.nacc, 1) * self.n * f)
        self.snd = self.plan.nbr("col")                     # built here: its gather is a launch of its own

    def fwd(self, sh=None, **over):
        sh = self.sh if sh is None else sh
        a = dict(lin=self.lin, lsh=self.lsh, f=self.f, d=self.d, sh_ld=sh.shape[1], ea=ops._p(self.ea), n=self.n)
        a.update(over)
        out = torch.full((max(self.nacc, 1) * self.n * self.f,), float("nan"), device=DEV)
        csr, p = self.plan.by_col, ops._p
        _lib.call("hgb_mace_tp_scatter_fwd", p(self.up), p(sh), p(self.tpw), p(csr.rowptr), p(csr.perm), p(self.snd), a["n"],
                  a["f"], a["lin"], a["lsh"], a["sh_ld"], a["ea"], a["d"], p(out), ops._stream())
        return out

    def bwd(self, sh=None, g_sh=None, **over):
        sh = self.sh if sh is None else sh
        a = dict(lin=self.lin, lsh=self.lsh, f=self.f, d=self.d, sh_ld=sh.shape[1], ea=ops._p(self.ea), n=self.n)
        a.update(over)
        g_tpw, g_up_e = torch.empty_like(self.tpw), torch.empty(self.e, (self.lin + 1) ** 2 * self.f, device=DEV)
        csr, p = self.plan.by_col, ops._p
        _lib.call("hgb_mace_tp_scatter_bwd", p(self.gout), p(self.up), p(sh), p(self.tpw), p(csr.rowptr), p(csr.perm),
                  p(self.snd), a["n"], a["f"], a["lin"], a["lsh"], a["sh_ld"], a["ea"], a["d"], p(g_tpw), p(g_up_e), p(g_sh),
                  ops._stream())
        return g_tpw, g_up_e


@gpu
def test_tp_scatter_abi_refuses_before_any_launch():
    t0, t3 = _TpRaw(1, 2, 64, 0, 9, 0), _TpRaw(1, 2, 64, 3, 9, 1)
    cases = [(t0, dict(lin=2, lsh=1), "unsupported degrees"), (t0, dict(lin=3, lsh=3), "unsupported degrees"),
             (t0, dict(lin=0, lsh=0), "unsupported degrees"), (t0, dict(f=48), "channels"), (t0, dict(f=0), "channels"),
             (t0, dict(sh_ld=8), "channels"), (t3, dict(d=17), "edge_dim"), (t3, dict(ea=None), "edge_dim"), (t0, dict(d=-1), "edge_dim")]
    torch.cuda.synchronize()
    for t, over, msg in cases:
        for fn in (t.fwd, t.bwd):
            before = _lib.launch_count()
            with pytest.raises(RuntimeError, match=msg):
                fn(**over)
            assert _lib.launch_count() == before, over
    before = _lib.launch_count()                                               # n = 0 is accepted and launches nothing
    t0.fwd(n=0)
    t0.bwd(n=0)
    assert _lib.launch_count() == before
    torch.cuda.synchronize()


@gpu
@pytest.mark.parametrize("f", [64, 96])
def test_tp_scatter_abi_accepts_wider_harmonics_rows(f):
    """sh_ld > (lmax_sh + 1)^2: harmonics of max_ell 3 (16 columns) read by the (1, 2) kernels.  Same bits as with the 9 columns
    alone, and the g_sh columns past the ninth are not written (F = 96: three atomicAdd passes into the first nine)."""
    t = _TpRaw(1, 2, f, 0, 16, f)
    tight = t.sh[:, :9].contiguous()
    assert torch.equal(t.fwd(), t.fwd(sh=tight))
    g_wide = torch.zeros(t.e, 16, device=DEV)
    g_wide[:, 9:] = 7.0
    g_tight = torch.zeros(t.e, 9, device=DEV)
    wide, narrow = t.bwd(g_sh=g_wide), t.bwd(sh=tight, g_sh=g_tight)
    assert torch.equal(wide[0], narrow[0]) and torch.equal(wide[1], narrow[1])
    assert torch.equal(g_wide[:, :9], g_tight) and bool((g_wide[:, 9:] == 7.0).all()) and float(g_tight.abs().max()) > 0


@gpu
def test_tp_scatter_abi_without_edges_writes_zeros():
    """raw E = 0, n > 0: the per-edge arrays are small valid buffers the kernels must not read; the forward zero-fills"""
    n, f = 1000, 64
    buf, idx = torch.zeros(64, device=DEV), torch.zeros(4, dtype=torch.int32, device=DEV)
    rowptr = torch.zeros(n + 1, dtype=torch.int32, device=DEV)
    up, out = torch.randn(n, 4, f, device=DEV), torch.full((21 * n * f,), float("nan"), device=DEV)
    p = ops._p
    _lib.call("hgb_mace_tp_scatter_fwd", p(up), p(buf), p(buf), p(rowptr), p(idx), p(idx), n, f, 1, 2, 9, None, 0, p(out), ops._stream())
    _lib.call("hgb_mace_tp_scatter_bwd", p(out), p(up), p(buf), p(buf), p(rowptr), p(idx), p(idx), n, f, 1, 2, 9, None, 0, p(buf), p(buf),
              None, ops._stream())
    assert bool((out == 0).all()) and bool((buf == 0).all())


# =====================================================================================================================
# B. hgb_mace_symcontract_{fwd,bwd}
# =====================================================================================================================
def _sc_run(x, wall, zcsr, gout, lin, lout):
    xd, wd = x.float().to(DEV).requires_grad_(True), wall.float().to(DEV).requires_grad_(True)
    out = ops.MaceSymContractFn.apply(xd, wd, zcsr, lin, lout)
    gx, gw = torch.autograd.grad(out, (xd, wd), gout.float().to(DEV))
    return out.detach(), gx, gw


PRESENT = [0, 5, 28, 77, 117]           # 5 of the 118 elements, both ends of the table included


def _element_batch(gen, counts):
    z = torch.cat([torch.full((c,), el) for el, c in zip(PRESENT, counts)])
    return z[torch.randperm(z.numel(), generator=gen)]


@gpu
@pytest.mark.parametrize("f", [1, 8, 50, 64, 128])
@pytest.mark.parametrize("lin,lout", SC_PAIRS)
def test_symcontract_matches_fp64(lin, lout, f):
    """Five elements with 1, 2, 37, 300 and 2,200 nodes (600 from F = 50 on, to bound the fp64 reference's [b, 2l+1, S, F]
    intermediates), 113 elements without a node; 40 nodes whose features are exactly zero and 40 with only the scalar set."""
    gen = _gen(8, lin, lout, f)
    assert _lib.query("hgb_mace_symcontract_num_weights", lin, lout) == _sc_num_weights(lin, lout)
    z = _element_batch(gen, (1, 2, 37, 300, 2200 if f <= 8 else 600))
    n, s = z.numel(), (lin + 1) ** 2
    x = _randn(gen, n, s, f)
    x[100:140] = 0.0
    x[140:180, 1:] = 0.0
    wall = _randn(gen, NUM_ELEMENTS, _sc_num_weights(lin, lout), f)
    gout = _randn(gen, n, (lout + 1) ** 2, f)
    ref, gx_ref, gw_ref = _sc_ref(x, wall, z, gout, lin, lout)
    zcsr = ops.csr_build(z.to(DEV), NUM_ELEMENTS)
    runs = [_sc_run(x, wall, zcsr, gout, lin, lout) for _ in range(2)]
    out, gx, gw = runs[0]
    assert rel_l2(out, ref) < 1e-5 and rel_l2(gx, gx_ref) < 1e-5, (rel_l2(out, ref), rel_l2(gx, gx_ref))
    # the weight gradient of each present element on its own: the element with one node must not hide behind the one with 2,200
    for el in PRESENT:
        assert rel_l2(gw[el], gw_ref[el]) < 1e-5, (el, rel_l2(gw[el], gw_ref[el]))
    absent = torch.ones(NUM_ELEMENTS, dtype=torch.bool)
    absent[PRESENT] = False
    assert float(gw[absent.to(DEV)].abs().max()) == 0.0                       # elements without a node: exactly zero
    assert float(out[100:140].abs().max()) == 0.0 and bool(torch.isfinite(gx).all())
    assert rel_l2(gx[100:180], gx_ref[100:180]) < 1e-5
    for a, b in zip(runs[0], runs[1]):
        assert torch.equal(a, b)


@gpu
@pytest.mark.parametrize("lin,lout", [(2, 1), (2, 0)])
def test_symcontract_at_benchmark_size(lin, lout):
    """20,480 nodes x F = 64 = 1.3 M (node, channel) pairs over 2,112 x 128 threads: every thread strides to a fifth pair"""
    gen, f = _gen(9, lin, lout), 64
    z = _element_batch(gen, (1, 479, 3000, 7000, 10000))
    n = z.numel()
    assert n == 20480 and n * f > 4 * 2112 * 128
    x, wall = _randn(gen, n, (lin + 1) ** 2, f), _randn(gen, NUM_ELEMENTS, _sc_num_weights(lin, lout), f)
    gout = _randn(gen, n, (lout + 1) ** 2, f)
    ref, gx_ref, gw_ref = _sc_ref(x, wall, z, gout, lin, lout)
    out, gx, gw = _sc_run(x, wall, ops.csr_build(z.to(DEV), NUM_ELEMENTS), gout, lin, lout)
    assert rel_l2(out, ref) < 1e-5 and rel_l2(gx, gx_ref) < 1e-5
    for el in PRESENT:
        assert rel_l2(gw[el], gw_ref[el]) < 1e-4, (el, rel_l2(gw[el], gw_ref[el]))


@gpu
def test_symcontract_without_nodes():
    x = torch.zeros(0, 9, 64, device=DEV, requires_grad=True)
    wall = torch.randn(NUM_ELEMENTS, _sc_num_weights(2, 1), 64, device=DEV, requires_grad=True)
    zcsr = ops.Csr(torch.zeros(0, dtype=torch.int32, device=DEV), torch.zeros(NUM_ELEMENTS + 1, dtype=torch.int32, device=DEV),
                   torch.zeros(0, dtype=torch.int32, device=DEV), NUM_ELEMENTS)
    out = ops.MaceSymContractFn.apply(x, wall, zcsr, 2, 1)
    assert out.shape == (0, 4, 64)
    gx, gw = torch.autograd.grad(out, (x, wall), torch.zeros_like(out))
    assert gx.shape == x.shape and gw.shape == wall.shape and bool((gw == 0).all())


@gpu
def test_symcontract_abi_refuses_before_any_launch():
    buf, z = torch.zeros(1 << 14, device=DEV), torch.zeros(8, dtype=torch.int32, device=DEV)
    p, st = ops._p, ops._stream()
    torch.cuda.synchronize()
    for lin, lout, f, msg in [(0, 0, 8, "unsupported degrees"), (1, 2, 8, "unsupported degrees"), (3, 3, 8, "unsupported degrees"),
                              (2, 1, 0, "bad arguments"), (2, 1, -4, "bad arguments")]:
        assert (_lib.query("hgb_mace_symcontract_num_weights", lin, lout) == -1) == (msg == "unsupported degrees")
        before = _lib.launch_count()
        with pytest.raises(RuntimeError, match=msg):
            _lib.call("hgb_mace_symcontract_fwd", p(buf), p(buf), p(z), 4, f, lin, lout, p(buf), st)
        with pytest.raises(RuntimeError, match=msg):
            _lib.call("hgb_mace_symcontract_bwd", p(buf), p(buf), p(buf), p(z), 4, f, lin, lout, p(buf), p(buf), st)
        assert _lib.launch_count() == before
    before = _lib.launch_count()
    _lib.call("hgb_mace_symcontract_fwd", p(buf), p(buf), p(z), 0, 8, 2, 1, p(buf), st)        # n = 0: accepted, nothing launched
    _lib.call("hgb_mace_symcontract_bwd", p(buf), p(buf), p(buf), p(z), 0, 8, 2, 1, p(buf), p(buf), st)
    assert _lib.launch_count() == before
    torch.cuda.synchronize()


# =====================================================================================================================
# C. closed primitives of hgb_mace_any.cu
# =====================================================================================================================
ALL_PATHS = _paths(2, 3)                                   # 17 paths, C from 1 x 1 x 1 to 5 x 7 x 7
# The kernels are not specialised by path or size (ni, nj, nk, E, F are loop bounds), so E = 5,000 runs on four C shapes and two
# widths only: E changes nothing but the number of blocks.  E = 17,000 x F = 33 is above both launch caps (2,112 blocks of 256
# (edge, channel) threads; 2,112 blocks of 8 edge warps), so all three grid-stride loops run; first order only.
TP_CASES = ([(p, f, e) for p in ALL_PATHS for f in (1, 8, 33, 64) for e in (1, 257)]
            + [(p, f, 5000) for p in [(0, 0, 0), (1, 1, 2), (2, 2, 0), (2, 3, 3)] for f in (8, 64)] + [((2, 3, 3), 33, 17000)])


def _tp_operand_shapes(name, e, f, ni, nj, nk):
    a, y, w, g = (e, ni, f), (e, nj), (e, f), (e, nk, f)
    return {"TpOut": (a, y, w), "TpY": (a, g, w), "TpW": (a, y, g)}[name]


@gpu
@pytest.mark.parametrize("path,f,e", TP_CASES, ids=lambda v: "".join(map(str, v)) if isinstance(v, tuple) else str(v))
@pytest.mark.parametrize("name", ["TpOut", "TpY", "TpW"])
def test_tp_primitive_derivatives_match_fp64(name, path, f, e):
    gen = _gen(10, *path, f, e, len(name) + ord(name[2]))
    c = _cg(*path)
    shapes = _tp_operand_shapes(name, e, f, *c.shape)
    ops64 = [_randn(gen, *s).requires_grad_(True) for s in shapes]
    out_shape = TP_REFS[name](*ops64, c).shape
    orders = 1 if e > 5000 else 3
    probes = [[_randn(gen, *out_shape)]] + [[_randn(gen, *s) for s in shapes] for _ in range(orders - 1)]
    ref = _chain(lambda *o: TP_REFS[name](*o, c), ops64, probes)
    ops32 = [t.detach().float().to(DEV).requires_grad_(True) for t in ops64]
    cd = c.float().to(DEV)
    dev = _chain(lambda *o: getattr(ops, name).apply(*o, cd), ops32, [[q.to(DEV) for q in pr] for pr in probes])
    assert len(ref) == orders + 1
    _assert_chain_close(dev, ref, (name, path, f, e))


@gpu
@pytest.mark.parametrize("path", [(1, 2, 3), (2, 3, 1), (2, 2, 2)])
def test_tp_primitives_take_a_permuted_coupling_view(path):
    """cg.permute(2, 1, 0), the non-contiguous view every backward hands on, as a direct forward argument"""
    gen, e, f = _gen(11, *path), 257, 33
    c = _cg(*path)
    ct = c.permute(2, 1, 0)
    cd = c.float().to(DEV).permute(2, 1, 0)
    assert not cd.is_contiguous()
    for name in ("TpOut", "TpY", "TpW"):
        operands = [_randn(gen, *s) for s in _tp_operand_shapes(name, e, f, *ct.shape)]
        out = getattr(ops, name).apply(*[t.float().to(DEV) for t in operands], cd)
        assert rel_l2(out, TP_REFS[name](*operands, ct)) < 1e-5, name


# (p, ni) as the contractions produce them: ni = (lmax_in + 1)^2 in {4, 9, 16}; p = 2 l + 1 after the last step, (2 l + 1) ni
# before it (correlation 2 and 3), (2 l + 1) ni ni at the first step of correlation 3
CHAN_CASES = [(p, ni, f) for ni in (4, 9, 16) for p in (1, 3, 5, ni, 3 * ni, 5 * ni, ni * ni, 5 * ni * ni) for f in (1, 4, 8, 64)
              if p * ni * f <= 5 * 16 * 16 * 16 * 8 or f == 64 and p <= 5 * ni]


@gpu
@pytest.mark.parametrize("p,ni,f", CHAN_CASES)
@pytest.mark.parametrize("name", ["ChanCL", "ChanOU", "ChanRP"])
def test_chan_primitive_derivatives_match_fp64(name, p, ni, f):
    """bilinear maps: value, first and second derivatives; the third vanishes identically and both sides must stop there"""
    n = 7 if p * ni * f > 4096 else 61
    gen = _gen(12, p, ni, f, ord(name[4]))
    t, x, g = (n, f, p, ni), (n, ni, f), (n, f, p)
    shapes = {"ChanCL": (t, x), "ChanOU": (g, x), "ChanRP": (g, t)}[name]
    ops64 = [_randn(gen, *s).requires_grad_(True) for s in shapes]
    out_shape = CHAN_REFS[name](*ops64).shape
    probes = [[_randn(gen, *out_shape)]] + [[_randn(gen, *s) for s in shapes] for _ in range(2)]
    ref = _chain(CHAN_REFS[name], ops64, probes)
    ops32 = [q.detach().float().to(DEV).requires_grad_(True) for q in ops64]
    dev = _chain(getattr(ops, name).apply, ops32, [[q.to(DEV) for q in pr] for pr in probes])
    assert len(ref) == 3
    _assert_chain_close(dev, ref, (name, p, ni, f))


@gpu
def test_chan_primitives_above_the_launch_cap():
    """n f p ni = 3,000 x 8 x 27 x 9: 5.8 M outputs of chan_ou, 648,000 of chan_cl, above the 540,672 threads of a capped launch"""
    gen, n, f, p, ni = _gen(13), 3000, 8, 27, 9
    t, x, g = _randn(gen, n, f, p, ni), _randn(gen, n, ni, f), _randn(gen, n, f, p)
    dev = lambda q: q.float().to(DEV)  # noqa: E731
    assert rel_l2(ops.ChanCL.apply(dev(t), dev(x)), CHAN_REFS["ChanCL"](t, x)) < 1e-5
    assert rel_l2(ops.ChanOU.apply(dev(g), dev(x)), CHAN_REFS["ChanOU"](g, x)) < 1e-5
    n2 = 9000                                                                  # chan_rp: n ni f = 648,000 outputs
    t2, g2 = _randn(gen, n2, f, 3, ni), _randn(gen, n2, f, 3)
    assert rel_l2(ops.ChanRP.apply(dev(g2), dev(t2)), CHAN_REFS["ChanRP"](g2, t2)) < 1e-5


@gpu
def test_closed_primitives_empty_inputs_and_refusals():
    cd = _cg(1, 1, 2).float().to(DEV)
    a, y, w, g = (torch.zeros(0, 3, 8, device=DEV), torch.zeros(0, 3, device=DEV), torch.zeros(0, 8, device=DEV), torch.zeros(0, 5, 8, device=DEV))
    assert ops.TpOut.apply(a, y, w, cd).shape == (0, 5, 8) and ops.TpY.apply(a, g, w, cd).shape == (0, 3)
    assert ops.TpW.apply(a, y, g, cd).shape == (0, 8)
    t, x, q = torch.zeros(0, 8, 5, 4, device=DEV), torch.zeros(0, 4, 8, device=DEV), torch.zeros(0, 8, 5, device=DEV)
    assert ops.ChanCL.apply(t, x).shape == (0, 8, 5) and ops.ChanOU.apply(q, x).shape == (0, 8, 5, 4) and ops.ChanRP.apply(q, t).shape == (0, 4, 8)
    buf = torch.zeros(1 << 14, device=DEV)
    p, st = ops._p, ops._stream()
    torch.cuda.synchronize()
    tp = lambda mode, p0, p1, p2, cg, e, f, ni, nj, nk: _lib.call("hgb_mace_tp_path", mode, p0, p1, p2, cg, e, f, ni, nj, nk, p(buf), st)  # noqa: E731
    ch = lambda mode, p0, p1, n, f, pp, ni: _lib.call("hgb_mace_chan_contract", mode, p0, p1, n, f, pp, ni, p(buf), st)  # noqa: E731
    b = p(buf)
    refused = [lambda: tp(0, b, b, b, b, 4, 8, 8, 3, 3), lambda: tp(0, b, b, b, b, 4, 8, 3, 8, 3), lambda: tp(0, b, b, b, b, 4, 8, 3, 3, 8),
               lambda: tp(3, b, b, b, b, 4, 8, 3, 3, 3), lambda: tp(-1, b, b, b, b, 4, 8, 3, 3, 3), lambda: tp(0, None, b, b, b, 4, 8, 3, 3, 3),
               lambda: tp(1, b, None, b, b, 4, 8, 3, 3, 3), lambda: tp(2, b, b, None, b, 4, 8, 3, 3, 3), lambda: tp(0, b, b, b, None, 4, 8, 3, 3, 3),
               lambda: tp(0, b, b, b, b, 4, 0, 3, 3, 3), lambda: tp(0, b, b, b, b, -1, 8, 3, 3, 3),
               lambda: ch(3, b, b, 4, 8, 5, 4), lambda: ch(0, None, b, 4, 8, 5, 4), lambda: ch(1, b, None, 4, 8, 5, 4),
               lambda: ch(0, b, b, 4, 0, 5, 4), lambda: ch(0, b, b, 4, 8, 0, 4), lambda: ch(0, b, b, 4, 8, 5, 0)]
    for k, call in enumerate(refused):
        before = _lib.launch_count()
        with pytest.raises(RuntimeError, match="bad"):
            call()
        assert _lib.launch_count() == before, k
    before = _lib.launch_count()
    for mode in range(3):                                                      # raw e = 0 / n = 0: accepted, nothing launched
        tp(mode, b, b, b, b, 0, 8, 3, 3, 5)
        ch(mode, b, b, 0, 8, 5, 4)
    assert _lib.launch_count() == before
    torch.cuda.synchronize()


# =====================================================================================================================
# D. the fused first-order path equals the any-order path
# =====================================================================================================================
def _leaf_grads(outs, leaves, gen_key):
    gen = _gen(14, gen_key)
    loss = sum((o * torch.randn(o.shape, generator=gen).to(o)).sum() for o in outs)
    return torch.autograd.grad(loss, leaves, allow_unused=True)


def _assert_same_grads(ga, gb, names):
    for name, a, b in zip(names, ga, gb):
        assert (a is None) == (b is None), name
        if a is not None and float(b.abs().max()) > 0:
            assert rel_l2(a, b) < 1e-5, (name, rel_l2(a, b))


@gpu
@pytest.mark.parametrize("d", [0, 3])
@pytest.mark.parametrize("lin,lsh", TP_PAIRS)
def test_interaction_fused_equals_any_order(lin, lsh, d, monkeypatch):
    """mace.Interaction.forward with higher = False (MaceTpScatterFn) and higher = True (GatherRows + TpOut per path + SegmentSum,
    EdgeMix with edge attributes): what a force-trained model predicts with and what it was trained through."""
    torch.manual_seed(100 * lin + 10 * lsh + d)
    gen, f, n, e = _gen(15, lin, lsh, d), 32, 41, 333
    block = mace.Interaction(f, lin, lsh, 1, 8, 10.0, d).to(DEV)
    calls, seen = [], []
    fused, tp_out = ops.MaceTpScatterFn.apply, ops.TpOut.apply
    monkeypatch.setattr(ops.MaceTpScatterFn, "apply", lambda *a: (calls.append("fused"), fused(*a))[1])
    monkeypatch.setattr(ops.TpOut, "apply", lambda *a: (calls.append("any"), tp_out(*a))[1])
    ei = torch.randint(0, n, (2, e), generator=gen)
    plan = ops.EdgePlan(ei.to(DEV), n)
    data = [torch.randn(n, 2 * l + 1, f, generator=gen) for l in range(lin + 1)] + [torch.randn(e, (lsh + 1) ** 2, generator=gen),
                                                                                    torch.randn(e, 8, generator=gen)]
    ea = torch.randn(e, d, generator=gen).to(DEV) if d else None
    names = ["x%d" % l for l in range(lin + 1)] + ["sh", "radial"] + [k for k, _ in block.named_parameters()]
    results = []
    for higher in (False, True):
        leaves = [t.to(DEV).requires_grad_(True) for t in data]
        msgs, sc = block(leaves[:lin + 1], leaves[-2], leaves[-1], plan, higher, ea)
        seen.append(list(calls))                            # the forward's calls (TpOut's backward is TpOut again)
        calls.clear()
        outs = list(msgs) + [s for s in sc if s.requires_grad]
        results.append(([o.detach() for o in outs], _leaf_grads(outs, leaves + list(block.parameters()), 0)))
    assert seen == [["fused"], ["any"] * len(_paths(lin, lsh))], seen
    for a, b in zip(*[r[0] for r in results]):
        assert rel_l2(a, b) < 1e-5, rel_l2(a, b)
    _assert_same_grads(results[0][1], results[1][1], names)


@gpu
@pytest.mark.parametrize("lin,lout", SC_PAIRS)
def test_product_fused_equals_any_order(lin, lout, monkeypatch):
    """mace.Product.forward with higher = False (MaceSymContractFn) and higher = True (MatMul + ChanCL per step)"""
    torch.manual_seed(10 * lin + lout)
    gen, f = _gen(16, lin, lout), 32
    block = mace.Product(f, lin, lout, 2).to(DEV)
    calls, seen = [], []
    fused, chan = ops.MaceSymContractFn.apply, ops.ChanCL.apply
    monkeypatch.setattr(ops.MaceSymContractFn, "apply", lambda *a: (calls.append("fused"), fused(*a))[1])
    monkeypatch.setattr(ops.ChanCL, "apply", lambda *a: (calls.append("any"), chan(*a))[1])
    z = _element_batch(gen, (1, 2, 7, 30, 60))
    n = z.numel()
    zcsr = ops.csr_build(z.to(DEV), NUM_ELEMENTS)
    data = [torch.randn(n, 2 * l + 1, f, generator=gen) for l in range(lin + 1)]
    sc = [torch.randn(n, 2 * l + 1, f, generator=gen).to(DEV) for l in range(lout + 1)]
    names = ["x%d" % l for l in range(lin + 1)] + [k for k, _ in block.named_parameters()]
    results = []
    for higher in (False, True):
        leaves = [t.to(DEV).requires_grad_(True) for t in data]
        outs = block(leaves, sc, zcsr, higher)
        seen.append(list(calls))
        calls.clear()
        results.append(([o.detach() for o in outs], _leaf_grads(outs, leaves + list(block.parameters()), 1)))
    assert seen == [["fused"], ["any"] * (2 * (lout + 1))], seen
    for a, b in zip(*[r[0] for r in results]):
        assert rel_l2(a, b) < 1e-5, rel_l2(a, b)
    _assert_same_grads(results[0][1], results[1][1], names)


# =====================================================================================================================
# E. edge embedding
# =====================================================================================================================
def _embed_case(gen, n, e, rc, with_shifts):
    """Random edges of lengths around r_max / 2, then by construction: edges 0..19 longer than r_max (1.0 to 3.0 times), edge 20 of
    length exactly r_max in fp32 (between (0,0,0) and (r_max,0,0), no shift), edge 21 along the polar axis."""
    pos = torch.randn(n, 3, generator=gen) * (rc / 4)
    pos[n - 2], pos[n - 1] = torch.zeros(3), torch.tensor([rc, 0.0, 0.0])
    ei = torch.randint(0, n - 2, (2, e), generator=gen)
    ei[1] = torch.where(ei[1] == ei[0], (ei[1] + 1) % (n - 2), ei[1])
    shifts = torch.randn(e, 3, generator=gen) * 0.1 if with_shifts else None
    far = torch.nn.functional.normalize(torch.randn(20, 3, generator=gen), dim=1) * rc * torch.linspace(1.0 + 1e-3, 3.0, 20)[:, None]
    ei[:, :20] = torch.stack([torch.arange(20), torch.arange(20, 40)])
    pos[20:40] = pos[:20] + far
    ei[:, 20] = torch.tensor([n - 2, n - 1])
    ei[:, 21] = torch.tensor([40, 41])
    pos[41] = pos[40] + torch.tensor([0.0, 1.5, 0.0])
    if with_shifts:
        shifts[:22] = 0.0
    return pos, ei, shifts


@gpu
@pytest.mark.parametrize("with_shifts", [True, False])
@pytest.mark.parametrize("lmax,nb,p", [(0, 8, 5.0), (1, 1, 5.0), (2, 8, 6.0), (3, 16, 5.0), (3, 8, 6.0), (2, 16, 5.0), (1, 8, 5.0), (3, 1, 6.0)])
def test_edge_embed_at_and_beyond_the_cutoff(lmax, nb, p, with_shifts):
    gen, n, e, rc = _gen(17, lmax, nb, int(p), with_shifts), 80, 900, 6.0
    pos, ei, shifts = _embed_case(gen, n, e, rc, with_shifts)
    ns = (lmax + 1) ** 2
    sh_w, rad_w = torch.randn(e, ns, generator=gen), torch.randn(e, nb, generator=gen)
    vec = (pos[ei[1]] - pos[ei[0]] + (shifts if with_shifts else 0.0)).double().requires_grad_(True)    # the fp32 edge vector, exactly
    sh_r, rad_r = _embed_ref(vec, lmax, nb, rc, p)
    g_sh_ref = torch.zeros_like(vec)                                           # lmax = 0: the constant harmonic has no gradient
    if lmax:
        g_sh_ref, = torch.autograd.grad((sh_r * sh_w.double()).sum(), vec, retain_graph=True)
    g_rad_ref, = torch.autograd.grad((rad_r * rad_w.double()).sum(), vec)
    beyond = vec.detach().norm(dim=1) >= rc
    assert int(beyond.sum()) >= 21 and bool(beyond[:21].all()) and float(vec.detach()[20].norm()) == rc
    pe = pos.to(DEV).requires_grad_(True)
    plan = ops.EdgePlan(ei.to(DEV), n)
    sd = None if shifts is None else shifts.to(DEV)
    sh_e, rad_e = ops.MaceEdgeEmbedFn.apply(pe, sd, plan, lmax, nb, rc, p)
    assert rel_l2(sh_e, sh_r) < 1e-5 and rel_l2(rad_e, rad_r) < 1e-5, (rel_l2(sh_e, sh_r), rel_l2(rad_e, rad_r))
    assert float(rad_e.detach()[beyond.to(DEV)].abs().max()) == 0.0                    # at and beyond r_max: exactly zero ...
    assert rel_l2(sh_e[:22], sh_r[:22]) < 1e-5                                 # ... and the harmonics still right
    # through autograd (both gradients given) against d/dpos of the reference
    (g_pos,) = torch.autograd.grad((sh_e * sh_w.to(DEV)).sum() + (rad_e * rad_w.to(DEV)).sum(), pe)
    g_vec_ref = g_sh_ref + g_rad_ref
    pos_ref = torch.zeros(n, 3, dtype=torch.float64).index_add_(0, ei[1], g_vec_ref).index_add_(0, ei[0], -g_vec_ref)
    assert rel_l2(g_pos, pos_ref) < 1e-5, rel_l2(g_pos, pos_ref)
    # raw backward with only one of the two gradients
    ptr, st = ops._p, ops._stream()
    for g_sh, g_rad, ref in ((sh_w.to(DEV), None, g_sh_ref), (None, rad_w.to(DEV), g_rad_ref)):
        g_vec = torch.full((e, 3), float("nan"), device=DEV)
        _lib.call("hgb_mace_edge_embed_bwd", ptr(pe.detach()), ptr(plan.row), ptr(plan.col), ptr(sd), ptr(g_sh), ptr(g_rad), e, lmax, nb, rc,
                  p, ptr(g_vec), st)
        if lmax == 0 and g_rad is None:
            assert float(g_vec.abs().max()) == 0.0                             # the constant harmonic has no gradient
        else:
            assert rel_l2(g_vec, ref) < 1e-5, (g_rad is None, rel_l2(g_vec, ref))
        if g_sh is None:
            assert float(g_vec[beyond.to(DEV)].abs().max()) == 0.0            # radial gradient at and beyond r_max: exactly zero


@gpu
def test_edge_embed_many_edges_and_widest_basis():
    """E = 600,000 > 2,112 blocks x 256 threads, so the grid strides.  num_bessel = 64 is the largest the entry point takes: the
    fp32 phase n pi d / r_max reaches 200 rad, where half an ulp is 8e-6 and the rounded frequency adds as much, so the bound
    for this basis is 1e-4 (values and gradient)."""
    gen, n, e, rc, p, lmax, nb = _gen(18), 5000, 600000, 6.0, 5.0, 3, 64
    pos = torch.randn(n, 3, generator=gen) * 1.5
    ei = torch.randint(0, n, (2, e), generator=gen)
    ei[1] = torch.where(ei[1] == ei[0], (ei[1] + 1) % n, ei[1])
    shifts = torch.randn(e, 3, generator=gen) * 0.1
    sh_w, rad_w = torch.randn(e, 16, generator=gen), torch.randn(e, nb, generator=gen)
    vec = (pos[ei[1]] - pos[ei[0]] + shifts).double().requires_grad_(True)
    sh_r, rad_r = _embed_ref(vec, lmax, nb, rc, p)
    g_ref, = torch.autograd.grad((sh_r * sh_w.double()).sum() + (rad_r * rad_w.double()).sum(), vec)
    pos_ref = torch.zeros(n, 3, dtype=torch.float64).index_add_(0, ei[1], g_ref).index_add_(0, ei[0], -g_ref)
    pe = pos.to(DEV).requires_grad_(True)
    sh_e, rad_e = ops.MaceEdgeEmbedFn.apply(pe, shifts.to(DEV), ops.EdgePlan(ei.to(DEV), n), lmax, nb, rc, p)
    assert rel_l2(sh_e, sh_r) < 1e-5 and rel_l2(rad_e[:, :16], rad_r[:, :16]) < 1e-5 and rel_l2(rad_e, rad_r) < 1e-4
    (g_pos,) = torch.autograd.grad((sh_e * sh_w.to(DEV)).sum() + (rad_e * rad_w.to(DEV)).sum(), pe)
    assert rel_l2(g_pos, pos_ref) < 1e-4, rel_l2(g_pos, pos_ref)


@gpu
def test_edge_embed_abi_refuses_before_any_launch():
    buf, idx = torch.zeros(1 << 12, device=DEV), torch.zeros(16, dtype=torch.int32, device=DEV)
    p, st = ops._p, ops._stream()
    torch.cuda.synchronize()
    for lmax, nb, rc in [(4, 8, 6.0), (-1, 8, 6.0), (2, 0, 6.0), (2, 65, 6.0), (2, 8, 0.0)]:
        before = _lib.launch_count()
        with pytest.raises(RuntimeError, match="bad arguments"):
            _lib.call("hgb_mace_edge_embed_fwd", p(buf), p(idx), p(idx), None, 4, lmax, nb, rc, 5.0, p(buf), p(buf), st)
        with pytest.raises(RuntimeError, match="bad arguments"):
            _lib.call("hgb_mace_edge_embed_bwd", p(buf), p(idx), p(idx), None, p(buf), p(buf), 4, lmax, nb, rc, 5.0, p(buf), st)
        assert _lib.launch_count() == before
    torch.cuda.synchronize()
