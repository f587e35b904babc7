"""Kernel-level tests of the GPS attention kernels (csrc/hgb_attn.cu: SIMT, head_dim 1..32; csrc/hgb_attn_tc.cu: tensor cores,
head_dim 8, plain TF32 or the 3xTF32 "exact" split), each against a plain fp64 restatement of include/hgb.h:

    head h owns columns h*d .. h*d+d-1 of each of q, k, v in qkv [n, 3f];
    S = q k^T / sqrt(d),   lse = logsumexp(S) (natural log),   out = softmax(S) v.

The C-ABI is called directly, so the test controls every argument.  Every output and the workspace carry a guard band of
extra rows filled with NaN, and so do the inputs: after each call every element of rows < n must be finite and the guard
band must still hold the same NaN bits, which catches unwritten columns, stores past row n and reads past row n (a NaN row
of V or dO read into a tile reaches the sums even where its weight is 0).

Bounds hold per (row, head), because one wrong tail row vanishes in a norm over 21 k rows.  The scale of a row is the same
sum taken over the magnitudes of its terms, with T_ij = sum_d |dO_id| |v_jd| the magnitude of the terms of dP_ij:
    out_i: max_d sum_j p_ij |v_jd|,                                dV_j: max_d sum_i p_ij |dO_id|,
    dQ_i:  max_d sum_j w_ij |k_jd| / sqrt(d),                      dK_j: max_d sum_i w_ij |q_id| / sqrt(d),
    w_ij = p_ij (T_ij + sum_l p_il T_il)                           (the terms of dS = P (dP - delta)).
dP - delta cancels when V carries a large common offset: dP, delta and their terms are all about |dO| |offset|.  An fp32
kernel forms dP and delta to a few ulp of their terms, so their difference, and dQ and dK with it, cannot be more accurate
than |dO| |V| |K| u, and that is the scale they are held to.

A score of magnitude sigma computed in fp32 carries a rounding error of order u sigma (u = 2^-24), and p = exp(s - lse) moves
by as much relative to itself: no fp32 kernel does better.  Plain fp32 ATen attention on the peaked inputs below misses a flat
1e-5 by the same margin as the kernels (1.9e-5 at head_dim 8 and 2.6e-5 at head_dim 32, with |lse| up to 300).  Each row is
therefore held to (tol + 2 cond) x scale, cond = u (|lse_i| + sigma_i) with sigma_i = max_j sum_d |q_id| |k_jd| / sqrt(d)
(a key row takes the largest cond of its head).  At the GPS scale, N(0, 1), 2 cond is about 2e-6.

Known answers must hold bit for bit (values with at most 10 mantissa bits, so the TF32 hi part is exact and lo = 0): all
keys equal gives out = mean(V); keys that are distinct +-1 sign patterns with q_i = alpha k_pi(i) give out_i = v_pi(i) and
(up to the lse round trip on the tensor cores) dV_pi(i) = dO_i, dQ = dK = 0.
"""
import math
import re

import pytest
import torch

from hydragnn_b200 import _lib, ops

DEV = "cuda"
GUARD = 5                           # extra NaN rows after every input, output and workspace
NAN_BITS = 0x7FC00000               # torch.full(nan) fp32
D_SIMT = (1, 2, 4, 8, 16, 32)
LOG2E = 1.4426950408889634
U32 = 2.0 ** -24                    # unit roundoff of fp32

# per-row bound on out, gradients and lse (lse: absolute, times 1 + |lse|); the global rel-L2 bound of the exact split
TOL = {"exact": dict(out=1e-5, grad=1e-5, lse=1e-6, l2_out=2e-6, l2_grad=1e-5),
       "tf32": dict(out=5e-3, grad=5e-3, lse=5e-3, l2_out=2e-3, l2_grad=5e-3),
       "simt": dict(out=1e-5, grad=1e-4, lse=1e-6, l2_out=None, l2_grad=None)}


# ---- fp64 references, from include/hgb.h --------------------------------------------------------------------------------
def _heads(t, heads):
    """[n, heads*d] -> [heads, n, d]"""
    return t.reshape(t.shape[0], heads, -1).transpose(0, 1)


def _unheads(t):
    """[heads, n, d] -> [n, heads*d]"""
    return t.transpose(0, 1).reshape(t.shape[1], -1)


def ref_autograd(qkv, gout, heads):
    """(out [n,f], lse [n,heads], gqkv [n,3f]) by fp64 autograd of the plain expression"""
    x = qkv.detach().clone().requires_grad_(True)
    f = x.shape[1] // 3
    q, k, v = (_heads(t, heads) for t in x.split(f, dim=1))
    s = q @ k.transpose(1, 2) / math.sqrt(f // heads)
    out = _unheads(torch.softmax(s, dim=-1) @ v)
    g, = torch.autograd.grad(out, x, gout)
    return out.detach(), torch.logsumexp(s, dim=-1).detach().t().contiguous(), g


def ref_blockwise(qkv, gout, heads, block=2048):
    """(out, lse, gqkv, scales) in fp64, one block of query rows at a time: lse first, then P, dV = P^T dO, dP = dO V^T,
    delta = rowsum(P dP) (from P, not from a kernel's out), dS = P (dP - delta), dQ = dS K / sqrt(d), dK = dS^T Q / sqrt(d).
    scales: {out, dq, dk, dv} [n, heads], the magnitude sums of the module docstring."""
    n, f = qkv.shape[0], qkv.shape[1] // 3
    d = f // heads
    c = 1.0 / math.sqrt(d)
    q, k, v = (_heads(t, heads) for t in qkv.split(f, dim=1))
    go = _heads(gout, heads)
    z = lambda *s: qkv.new_zeros(*s)  # noqa: E731
    out, dq, dk, dv = z(heads, n, d), z(heads, n, d), z(heads, n, d), z(heads, n, d)
    lse, s_out, s_dq, sigma = z(heads, n), z(heads, n), z(heads, n), z(heads, n)
    s_dk, s_dv = z(heads, n, d), z(heads, n, d)
    for h in range(heads):
        kh, vh = k[h], v[h]
        for i0 in range(0, n, block):
            i1 = min(n, i0 + block)
            qb, gb = q[h, i0:i1], go[h, i0:i1]
            s = (qb @ kh.t()) * c
            lb = torch.logsumexp(s, dim=1)
            p = torch.exp(s - lb[:, None])
            del s
            lse[h, i0:i1] = lb
            out[h, i0:i1] = p @ vh
            s_out[h, i0:i1] = (p @ vh.abs()).amax(1)
            dv[h] += p.t() @ gb
            s_dv[h] += p.t() @ gb.abs()
            sigma[h, i0:i1] = ((qb.abs() @ kh.abs().t()) * c).amax(1)
            dp = gb @ vh.t()
            delta = (p * dp).sum(1)
            ds = p * (dp - delta[:, None])
            t = gb.abs() @ vh.abs().t()                 # the magnitude of the terms of dP (and, weighted by p, of delta)
            w = p * (t + (p * t).sum(1)[:, None])
            del dp, p, t
            dq[h, i0:i1] = (ds @ kh) * c
            dk[h] += (ds.t() @ qb) * c
            s_dq[h, i0:i1] = ((w @ kh.abs()) * c).amax(1)
            s_dk[h] += (w.t() @ qb.abs()) * c
            del ds, w
    gqkv = torch.cat([_unheads(dq), _unheads(dk), _unheads(dv)], dim=1)
    cond = U32 * (lse.abs() + sigma)                     # [heads, n], per query row; a key row sees every query's
    scales = dict(out=s_out.t(), dq=s_dq.t(), dk=s_dk.amax(-1).t(), dv=s_dv.amax(-1).t(),
                  cond_q=cond.t(), cond_k=cond.amax(1)[None, :].expand(n, heads))
    return _unheads(out), lse.t().contiguous(), gqkv, scales


def ref_sdpa(qkv, gout, heads):
    x = qkv.detach().clone().requires_grad_(True)
    f = x.shape[1] // 3
    q, k, v = (_heads(t, heads) for t in x.split(f, dim=1))
    out = _unheads(torch.nn.functional.scaled_dot_product_attention(q, k, v))
    g, = torch.autograd.grad(out, x, gout)
    return out.detach(), g


# ---- CPU self-checks of the references ------------------------------------------------------------------------------------
@pytest.mark.parametrize("n,heads,d", [(1, 1, 8), (7, 2, 8), (37, 3, 4), (70, 2, 16)])
def test_blockwise_reference_matches_autograd(n, heads, d):
    """the blockwise reference, with blocks smaller than n, against fp64 autograd of the plain expression"""
    g = torch.Generator().manual_seed(n + heads + d)
    f = heads * d
    qkv = torch.randn(n, 3 * f, generator=g, dtype=torch.float64) * 2.0
    qkv[:, 2 * f:] += 3.0
    gout = torch.randn(n, f, generator=g, dtype=torch.float64)
    out_a, lse_a, g_a = ref_autograd(qkv, gout, heads)
    out_b, lse_b, g_b, scales = ref_blockwise(qkv, gout, heads, block=16)
    torch.testing.assert_close(out_b, out_a, rtol=1e-12, atol=1e-12)
    torch.testing.assert_close(lse_b, lse_a, rtol=1e-12, atol=1e-12)
    torch.testing.assert_close(g_b, g_a, rtol=1e-11, atol=1e-11)
    # each scale bounds its result: |result| <= the magnitude sum, per (row, head)
    for name, part, cols in (("out", out_a, slice(0, f)), ("dq", g_a, slice(0, f)), ("dk", g_a, slice(f, 2 * f)),
                             ("dv", g_a, slice(2 * f, 3 * f))):
        mag = part[:, cols].abs().reshape(n, heads, d).amax(-1)
        assert bool((mag <= scales[name] * (1 + 1e-12) + 1e-300).all()), name


@pytest.mark.parametrize("n,heads,d", [(1, 1, 1), (9, 2, 8), (33, 4, 2), (65, 1, 32)])
def test_references_match_sdpa(n, heads, d):
    """both references against torch.nn.functional.scaled_dot_product_attention in fp64"""
    g = torch.Generator().manual_seed(7 * n + d)
    f = heads * d
    qkv = torch.randn(n, 3 * f, generator=g, dtype=torch.float64)
    gout = torch.randn(n, f, generator=g, dtype=torch.float64)
    out_s, g_s = ref_sdpa(qkv, gout, heads)
    out_a, _, g_a = ref_autograd(qkv, gout, heads)
    out_b, _, g_b, _ = ref_blockwise(qkv, gout, heads, block=8)
    for o in (out_a, out_b):
        torch.testing.assert_close(o, out_s, rtol=1e-12, atol=1e-12)
    for gg in (g_a, g_b):
        torch.testing.assert_close(gg, g_s, rtol=1e-11, atol=1e-11)


# ---- harness ----------------------------------------------------------------------------------------------------------------
def _nan(*shape):
    return torch.full(shape, float("nan"), dtype=torch.float32, device=DEV)


def _p(t):
    return None if t is None else t.data_ptr()


def _guarded(x):
    """x [n, c] fp32 followed by GUARD rows of NaN (the kernels must read no row >= n)"""
    g = _nan(x.shape[0] + GUARD, x.shape[1])
    g[:x.shape[0]] = x
    return g


def run_fwd(path, qkv, n, f, heads, exact=1):
    out, lse = _nan(n + GUARD, f), _nan(n + GUARD, heads)
    if path == "tc":
        _lib.call("hgb_mha_tc_fwd", _p(qkv), n, f, heads, exact, _p(out), _p(lse), ops._stream())
    else:
        _lib.call("hgb_mha_fwd", _p(qkv), n, f, heads, _p(out), _p(lse), ops._stream())
    return out, lse


def run_bwd(path, qkv, out, lse, gout, n, f, heads, exact=1):
    gqkv, ws = _nan(n + GUARD, 3 * f), _nan((n + GUARD) * heads)
    if path == "tc":
        _lib.call("hgb_mha_tc_bwd", _p(qkv), _p(out), _p(lse), _p(gout), n, f, heads, exact, _p(ws), _p(gqkv), ops._stream())
    else:
        _lib.call("hgb_mha_bwd", _p(qkv), _p(out), _p(lse), _p(gout), n, f, heads, _p(gqkv), ops._stream())
    return gqkv, ws


def same_bits(a, b):
    return a.shape == b.shape and torch.equal(a.contiguous().view(torch.int32), b.contiguous().view(torch.int32))


def check_written(what, name, t, rows):
    """rows < `rows` finite, the guard band still NaN bit for bit"""
    body, guard = t[:rows], t[rows:]
    assert bool(torch.isfinite(body).all()), "%s: %s has %d unwritten or non-finite entries in rows < n" % (
        what, name, int((~torch.isfinite(body)).sum()))
    assert bool((guard.contiguous().view(torch.int32) == NAN_BITS).all()), "%s: %s written past row n" % (what, name)


def check_rows(what, name, a, ref, scale, tol, heads, cond=None):
    """per (row, head): max_d |a - ref| <= (tol + 2 cond) * scale (scale = 0 demands an exact 0); cond: the score
    conditioning term of the module docstring"""
    n = a.shape[0]
    err = (a.double() - ref).abs().reshape(n, heads, -1).amax(-1)
    lim = (tol + (0 if cond is None else 2 * cond)) * scale
    bad = err > lim
    if bool(bad.any()):
        ratio = err / lim.clamp_min(1e-300)
        i = int(ratio.argmax())
        r, h = divmod(i, heads)
        pytest.fail("%s: %s exceeds %.1e x its scale in %d of %d (row, head) pairs; worst row %d head %d: |err| %.3g, scale %.3g"
                    % (what, name, tol, int(bad.sum()), bad.numel(), r, h, float(err[r, h]), float(scale[r, h])))


def rel_l2(a, ref):
    den = ref.norm()
    return float((a.double() - ref).norm() / den) if float(den) > 0 else float((a.double() - ref).abs().max())


def inputs(n, f, dist, seed):
    """qkv [n, 3f], gout [n, f] in fp32.  normal: N(0, 1), the GPS scale; peaked: q and k x 6, so score spreads reach tens to
    hundreds of natural units and the softmax saturates; offset: V = 30 + N(0, 1); zero_gout: gout = 0."""
    g = torch.Generator(device=DEV).manual_seed(seed)
    qkv = torch.randn(n, 3 * f, generator=g, device=DEV)
    gout = torch.randn(n, f, generator=g, device=DEV)
    if dist == "peaked":
        qkv[:, :2 * f] *= 6.0
    elif dist == "offset":
        qkv[:, 2 * f:] += 30.0
    elif dist == "zero_gout":
        gout.zero_()
    else:
        assert dist == "normal", dist
    return qkv, gout


def _reference(qkv, gout, heads):
    """the blockwise reference (with its scales); for small n values from fp64 autograd"""
    out, lse, g, scales = ref_blockwise(qkv, gout, heads)
    if qkv.shape[0] <= 512:
        out, lse, g = ref_autograd(qkv, gout, heads)
    return out, lse, g, scales


def run_case(fwd_path, bwd_path, n, heads, d, mode, dist="normal", seed=0, determinism=True):
    """forward on fwd_path, backward on bwd_path ('tc' or 'simt'); mode: 'exact' or 'tf32' (the tensor-core split) or 'simt'"""
    f = heads * d
    exact = 0 if mode == "tf32" else 1
    what = "%s->%s n=%d heads=%d d=%d %s %s" % (fwd_path, bwd_path, n, heads, d, mode, dist)
    x, go = inputs(n, f, dist, seed or (n * 131 + heads * 7 + d))
    qkv, gout = _guarded(x), _guarded(go)

    def once():
        out, lse = run_fwd(fwd_path, qkv, n, f, heads, exact)
        gqkv, ws = run_bwd(bwd_path, qkv, out, lse, gout, n, f, heads, exact)
        return out, lse, gqkv, ws

    out, lse, gqkv, ws = once()
    torch.cuda.synchronize()
    check_written(what, "out", out, n)
    check_written(what, "lse", lse, n)
    check_written(what, "gqkv", gqkv, n)
    if bwd_path == "tc":
        check_written(what, "delta_ws", ws, n * heads)
    else:
        assert bool((ws.view(torch.int32) == NAN_BITS).all()), "%s: the SIMT backward wrote delta_ws" % what
    ref_out, ref_lse, ref_g, sc = _reference(x.double(), go.double(), heads)
    tol = TOL[mode]
    o, l, gq = out[:n], lse[:n], gqkv[:n]
    check_rows(what, "out", o, ref_out, sc["out"], tol["out"], heads, sc["cond_q"])
    lerr = (l.double() - ref_lse).abs()
    assert bool((lerr <= tol["lse"] * (1 + ref_lse.abs())).all()), "%s: lse off by %.3g (|lse| %.3g)" % (
        what, float(lerr.max()), float(ref_lse.abs().flatten()[int(lerr.argmax())]))
    for name, cols, cond in (("dq", slice(0, f), "cond_q"), ("dk", slice(f, 2 * f), "cond_k"),
                             ("dv", slice(2 * f, 3 * f), "cond_k")):
        check_rows(what, name, gq[:, cols], ref_g[:, cols], sc[name], tol["grad"], heads, sc[cond])
    if dist == "zero_gout":
        assert bool((gq == 0).all()), "%s: gout = 0 but gqkv is not exactly 0" % what
    if tol["l2_out"] is not None and dist == "normal":
        assert rel_l2(o, ref_out) < tol["l2_out"], (what, rel_l2(o, ref_out))
        assert rel_l2(gq, ref_g) < tol["l2_grad"], (what, rel_l2(gq, ref_g))
    if determinism:
        again = once()
        torch.cuda.synchronize()
        for name, a, b in zip(("out", "lse", "gqkv", "delta_ws"), (out, lse, gqkv, ws), again):
            assert same_bits(a, b), "%s: %s differs between two identical calls" % (what, name)


# ---- 1. tensor-core kernels -------------------------------------------------------------------------------------------------
TC_N = (1, 2, 3, 5, 15, 16, 17, 63, 64, 65, 127, 128, 129, 4095, 4096, 4097, 10600, 21504)
HEADS = (1, 2, 3, 8, 16)


def _tc_cases():
    """(n, heads): the 16-row warp tile, the 64-row CTA and the 64-key chunk on both sides of each boundary, both production
    lengths at 8 heads, every head count at n = 65"""
    cases = [(n, 8 if n >= 10000 else HEADS[i % len(HEADS)]) for i, n in enumerate(TC_N)]
    return cases + [(65, h) for h in HEADS if (65, h) not in cases]


TC_CASES = _tc_cases()


@pytest.mark.gpu
@pytest.mark.parametrize("mode", ["exact", "tf32"])
@pytest.mark.parametrize("n,heads", TC_CASES, ids=["n%d-h%d" % c for c in TC_CASES])
def test_tc_attention_matches_fp64(n, heads, mode):
    run_case("tc", "tc", n, heads, 8, mode)


@pytest.mark.gpu
def test_tc_attention_beyond_512_key_chunks():
    """33,000 keys = 516 chunks of 64, the last one partial: long sums stay in registers with round-to-nearest adds"""
    run_case("tc", "tc", 33000, 1, 8, "exact", determinism=False)


# a TF32 score of magnitude 100 is off by ~0.1, so plain TF32 is held on unsaturated scores only
TC_DISTS = [("exact", "peaked"), ("exact", "offset"), ("exact", "zero_gout"), ("tf32", "offset"), ("tf32", "zero_gout")]


@pytest.mark.gpu
@pytest.mark.parametrize("mode,dist", TC_DISTS, ids=["%s-%s" % c for c in TC_DISTS])
@pytest.mark.parametrize("n", [17, 129, 4097])
def test_tc_attention_input_distributions(n, mode, dist):
    run_case("tc", "tc", n, 8 if n > 1000 else 3, 8, mode, dist)


# ---- 2. SIMT kernels --------------------------------------------------------------------------------------------------------
SIMT_N = (1, 2, 3, 4, 5, 31, 32, 33, 63, 64, 65, 129, 4097)
SIMT_HEADS = {1: (1, 3), 2: (2, 5), 4: (1, 4), 8: (3, 1), 16: (2, 1), 32: (1, 2)}
SIMT_CASES = [(d, n, SIMT_HEADS[d][i % 2]) for d in D_SIMT for i, n in enumerate(SIMT_N)]
SIMT_CASES += [(16, 10600, 2), (32, 10600, 2)]


@pytest.mark.gpu
@pytest.mark.parametrize("d,n,heads", SIMT_CASES, ids=["d%d-n%d-h%d" % c for c in SIMT_CASES])
def test_simt_attention_matches_fp64(d, n, heads):
    run_case("simt", "simt", n, heads, d, "simt", determinism=n < 10000)


@pytest.mark.gpu
@pytest.mark.parametrize("dist", ["peaked", "offset", "zero_gout"])
@pytest.mark.parametrize("d,n,heads", [(8, 129, 2), (32, 4097, 2), (1, 65, 3)])
def test_simt_attention_input_distributions(d, n, heads, dist):
    run_case("simt", "simt", n, heads, d, "simt", dist)


# ---- 3. the shared lse / layout contract ------------------------------------------------------------------------------------
@pytest.mark.gpu
@pytest.mark.parametrize("mode", ["exact", "tf32"])
@pytest.mark.parametrize("n,heads", [(129, 2), (4097, 8)])
def test_tc_forward_feeds_simt_backward(n, heads, mode):
    """out and lse of the tensor-core forward into hgb_mha_bwd (D = 8); the tolerance is the forward's"""
    run_case("tc", "simt", n, heads, 8, mode)


@pytest.mark.gpu
@pytest.mark.parametrize("mode", ["exact", "tf32"])
@pytest.mark.parametrize("n,heads", [(129, 2), (4097, 8)])
def test_simt_forward_feeds_tc_backward(n, heads, mode):
    run_case("simt", "tc", n, heads, 8, mode)


# ---- 4. known answers, bit for bit ------------------------------------------------------------------------------------------
def _coarse(g, *shape, bits=6):
    """values k / 16 with |k| < 2^bits: at most `bits` mantissa bits, every sum of a few thousand is exact in fp32"""
    return (torch.randint(-(2 ** bits) + 1, 2 ** bits, shape, generator=g, device=DEV).float() / 16.0)


PATHS = [("tc", "exact"), ("tc", "tf32"), ("simt", "simt")]


@pytest.mark.gpu
@pytest.mark.parametrize("path,mode", PATHS, ids=[p[1] for p in PATHS])
@pytest.mark.parametrize("n", [1, 2, 16, 64, 256, 4096])
def test_uniform_keys_give_the_mean_of_v(n, path, mode):
    """all keys equal: every score of a row is the same number, p = 1 for every key, l = n, out = sum(v) / n exactly"""
    heads, d = 3, 8
    f = heads * d
    g = torch.Generator(device=DEV).manual_seed(n)
    x = torch.cat([_coarse(g, n, f), _coarse(g, 1, f).expand(n, f), _coarse(g, n, f)], dim=1)
    qkv = _guarded(x)
    out, lse = run_fwd(path, qkv, n, f, heads, 0 if mode == "tf32" else 1)
    torch.cuda.synchronize()
    check_written(mode, "out", out, n)
    check_written(mode, "lse", lse, n)
    want = x[:, 2 * f:].double().mean(0, keepdim=True).expand(n, f)
    assert torch.equal(out[:n].double(), want), "%s n=%d: out != mean(V) in %d entries" % (
        mode, n, int((out[:n].double() != want).sum()))
    s = (_heads(x[:, :f].double(), heads) * _heads(x[:1, f:2 * f].double(), heads)).sum(-1).t() / math.sqrt(d)
    lerr = (lse[:n].double() - (s + math.log(n))).abs()
    assert bool((lerr <= TOL[mode]["lse"] * (1 + s.abs() + math.log(n))).all()), float(lerr.max())


ALPHA = 148.0       # every non-winning score is 2 alpha / sqrt(8) log2(e) = 151 or more below the winner in base 2


def _permutation_case(n, heads, seed):
    """keys: n distinct +-1 sign patterns per head; q_i = ALPHA k_pi(i); v, dO with 6-bit mantissas.  (qkv, gout, pi)"""
    d = 8
    f = heads * d
    g = torch.Generator(device=DEV).manual_seed(seed)
    bits = 2 ** torch.arange(d, device=DEV)
    qs, ks, pis = [], [], []
    for _ in range(heads):
        codes = torch.randperm(256, generator=g, device=DEV)[:n]
        k = ((codes[:, None] & bits) != 0).float() * 2 - 1
        pi = torch.randperm(n, generator=g, device=DEV)
        qs.append(ALPHA * k[pi])
        ks.append(k)
        pis.append(pi)
    x = torch.cat([torch.cat(qs, 1), torch.cat(ks, 1), _coarse(g, n, f)], dim=1)
    return x, _coarse(g, n, f), pis


@pytest.mark.gpu
@pytest.mark.parametrize("path,mode", PATHS, ids=[p[1] for p in PATHS])
@pytest.mark.parametrize("n,heads", [(1, 1), (7, 3), (64, 1), (129, 2), (256, 3)])
def test_permutation_attention_is_exact(n, heads, path, mode):
    """softmax saturates on the winner: out_i = v_pi(i) bit for bit, dQ = dK = 0 (up to denormals of the losing keys),
    dV_pi(i) = dO_i bit for bit on SIMT.  The tensor-core backward rebuilds the winner's p as exp2(s log2 e - lse log2 e):
    s (base 2 about 600) reaches lse through m ln2 and back through log2 e, so p = 1 only to a few ulp of m, and
    dV_pi(i) = p dO_i is held to 8 ulp(m) ln 2 relative.  This pins the permuted fragment mapping (S accumulator -> A operand
    of P V, V loaded in the same permuted order) lane by lane."""
    d = 8
    f = heads * d
    exact = 0 if mode == "tf32" else 1
    x, go, pis = _permutation_case(n, heads, seed=n * 10 + heads)
    qkv, gout = _guarded(x), _guarded(go)
    out, lse = run_fwd(path, qkv, n, f, heads, exact)
    gqkv, _ = run_bwd(path, qkv, out, lse, gout, n, f, heads, exact)
    torch.cuda.synchronize()
    for name, t in (("out", out), ("lse", lse), ("gqkv", gqkv)):
        check_written(mode, name, t, n)
    v = _heads(x[:, 2 * f:], heads)
    gh = _heads(go, heads)
    want_out = _unheads(torch.stack([v[h][pis[h]] for h in range(heads)]))
    assert same_bits(out[:n], want_out), "%s: out != v_pi in %d entries" % (mode, int((out[:n] != want_out).sum()))
    inv = [torch.argsort(p) for p in pis]
    want_dv = _unheads(torch.stack([gh[h][inv[h]] for h in range(heads)]))
    dv = gqkv[:n, 2 * f:]
    if path == "simt":
        assert same_bits(dv, want_dv), "%s: dV != dO_pi^-1 in %d entries" % (mode, int((dv != want_dv).sum()))
    else:
        m = (lse[:n].double() * LOG2E).abs()                                 # the winner's score in base 2, [n, heads]
        ulp = torch.pow(2.0, torch.floor(torch.log2(m)) - 23)
        m_of_key = torch.stack([m[inv[h], h] for h in range(heads)], 1)      # key j wins for query pi^-1(j)
        ulp_key = torch.stack([ulp[inv[h], h] for h in range(heads)], 1)
        lim = (8 * ulp_key * math.log(2)).repeat_interleave(d, 1) * want_dv.abs().double()
        err = (dv.double() - want_dv.double()).abs()
        assert bool((err <= lim).all()), "%s: dV off by %.3g relative (m up to %.0f)" % (
            mode, float((err / want_dv.abs().double().clamp_min(1e-30)).max()), float(m_of_key.max()))
    assert bool((gqkv[:n, :2 * f].abs() <= 1e-30).all()), "%s: dQ, dK not 0: max %.3g" % (
        mode, float(gqkv[:n, :2 * f].abs().max()))


# ---- 5. which kernel each path reaches --------------------------------------------------------------------------------------
KERNEL = re.compile(r"(mha_(?:tc_)?(?:fwd|bwd_q|bwd_kv|delta)_kernel(?:<\d+>)?)")


def _launched(fn):
    from torch.profiler import ProfilerActivity, profile
    torch.cuda.synchronize()
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        fn()
        torch.cuda.synchronize()
    hits = [(e.time_range.start, KERNEL.search(e.name)) for e in prof.events() if KERNEL.search(e.name)]
    return [m.group(1) for _, m in sorted(hits, key=lambda t: t[0])]


def _mha_module(qkv, heads, gout, tf32=False):
    from hydragnn_b200 import gps
    x = qkv.detach().requires_grad_(True)
    with ops.tensor_cores(tf32):
        out = gps.MhaFn.apply(x, heads)
    g, = torch.autograd.grad(out, x, gout)
    return out.detach(), g


def _dispatch_cases():
    """(MhaFn arguments, the kernels they must launch) of every dispatch case"""
    runs, want = [], []
    for f, heads, offset in ((8, 8, False), (16, 8, False), (32, 8, False), (8, 1, False), (64, 8, False), (128, 16, False),
                             (64, 4, False), (64, 2, False), (16, 1, False), (24, 3, False), (64, 8, True)):
        d = f // heads
        for tf32 in (False, True):
            x, go = inputs(70, f, "normal", f + heads)
            runs.append((_offset_view(x) if offset else x, heads, go, tf32))
            if d == 8 and not offset:
                s = 1 if tf32 else 3
                want.append(["mha_tc_fwd_kernel<%d>" % s, "mha_tc_delta_kernel", "mha_tc_bwd_q_kernel<%d>" % s,
                             "mha_tc_bwd_kv_kernel<%d>" % s])
            else:
                want.append(["mha_fwd_kernel<%d>" % d, "mha_bwd_q_kernel<%d>" % d, "mha_bwd_kv_kernel<%d>" % d])
    return runs, want


def dispatch_names():
    """the attention kernels the dispatch cases launch, in order, from one torch.profiler session"""
    runs, _ = _dispatch_cases()
    return _launched(lambda: [_mha_module(*r) for r in runs])


@pytest.mark.gpu
def test_dispatch_reaches_every_instantiation():
    """MhaFn takes the tensor cores exactly when d = 8 and qkv is 16-byte aligned (SPLIT 3 in fp32, SPLIT 1 under
    tensor_cores()), the SIMT template <d> otherwise; together the cases launch every template of both files.  The profile
    is taken in a child process: a later torch.profiler session in the same process can miss the first kernels it should
    record, and the PaiNN dispatch test, which counts every launch of its session, lost two that way."""
    import json
    import os
    import subprocess
    import sys
    tests = os.path.dirname(os.path.abspath(__file__))
    code = ("import json, sys; sys.path[:0] = [%r, %r]; import test_gpu_attention_kernels as t; "
            "print('NAMES ' + json.dumps(t.dispatch_names()))" % (os.path.dirname(tests), tests))
    r = subprocess.run([sys.executable, "-c", code], capture_output=True, text=True, timeout=600)
    assert r.returncode == 0, r.stdout[-2000:] + r.stderr[-4000:]
    names = json.loads([ln for ln in r.stdout.splitlines() if ln.startswith("NAMES ")][-1][6:])
    runs, want = _dispatch_cases()
    assert len(names) == sum(len(w) for w in want), (len(names), sum(len(w) for w in want))
    pos = 0
    for r, w in zip(runs, want):
        assert names[pos:pos + len(w)] == w, (r[0].shape, r[1], r[3], names[pos:pos + len(w)])
        pos += len(w)
    every = {"mha_tc_delta_kernel"} | {"mha_tc_%s_kernel<%d>" % (k, s) for k in ("fwd", "bwd_q", "bwd_kv") for s in (1, 3)}
    every |= {"mha_%s_kernel<%d>" % (k, d) for k in ("fwd", "bwd_q", "bwd_kv") for d in D_SIMT}
    assert set(names) == every, sorted(every - set(names))


# ---- 6. refusals and empty inputs -------------------------------------------------------------------------------------------
def _rc(name, *args):
    return int(getattr(_lib.lib(), name)(*args))


def _abi_args(entry, qkv, out, lse, gout, gqkv, ws, n, f, heads):
    s = ops._stream()
    return {"hgb_mha_fwd": (qkv, n, f, heads, out, lse, s),
            "hgb_mha_bwd": (qkv, out, lse, gout, n, f, heads, gqkv, s),
            "hgb_mha_tc_fwd": (qkv, n, f, heads, 1, out, lse, s),
            "hgb_mha_tc_bwd": (qkv, out, lse, gout, n, f, heads, 1, ws, gqkv, s)}[entry]


ENTRIES = ("hgb_mha_fwd", "hgb_mha_bwd", "hgb_mha_tc_fwd", "hgb_mha_tc_bwd")


@pytest.mark.gpu
def test_refusals_launch_nothing():
    """every refusal returns EINVAL before any launch and leaves the outputs untouched"""
    n = 40
    buf = {k: _nan(4 * n * 3 * 128 + 64) for k in ("qkv", "out", "lse", "gout", "gqkv", "ws")}
    ptr = {k: _p(t) for k, t in buf.items()}
    torch.cuda.synchronize()
    before = _lib.launch_count()
    bad_sizes = [(n, 8, 0), (n, 8, -1), (n, 12, 8), (n, 24, 5), (-1, 8, 1), (-1, 64, 8)]
    simt_dims = [(n, 24, 8), (n, 40, 8), (n, 64, 1), (n, 48, 1), (n, 128, 2)]        # d = 3, 5, 64, 48, 64
    tc_dims = [(n, 16, 1), (n, 32, 8), (n, 64, 4), (n, 8, 8), (n, 24, 1)]            # d = 16, 4, 16, 1, 24
    cases = [(e, s, None) for e in ENTRIES for s in bad_sizes]
    cases += [(e, s, None) for e in ("hgb_mha_fwd", "hgb_mha_bwd") for s in simt_dims]
    cases += [(e, s, None) for e in ("hgb_mha_tc_fwd", "hgb_mha_tc_bwd") for s in tc_dims]
    for e in ENTRIES:
        names = [nm for nm in ("qkv", "out", "lse", "gout", "gqkv", "ws") if nm in {
            "hgb_mha_fwd": ("qkv", "out", "lse"), "hgb_mha_tc_fwd": ("qkv", "out", "lse"),
            "hgb_mha_bwd": ("qkv", "out", "lse", "gout", "gqkv"),
            "hgb_mha_tc_bwd": ("qkv", "out", "lse", "gout", "gqkv", "ws")}[e]]
        cases += [(e, (n, 64, 8), {nm: None}) for nm in names]
    # the tensor-core kernels move rows as float4 / float2
    cases += [("hgb_mha_tc_fwd", (n, 64, 8), {"qkv": ptr["qkv"] + off}) for off in (4, 8, 12)]
    cases += [("hgb_mha_tc_fwd", (n, 64, 8), {"out": ptr["out"] + 4})]
    cases += [("hgb_mha_tc_bwd", (n, 64, 8), {k: ptr[k] + off}) for k in ("qkv", "out", "gout") for off in (4, 8, 12)]
    cases += [("hgb_mha_tc_bwd", (n, 64, 8), {"gqkv": ptr["gqkv"] + 4})]
    for e, (nn, f, heads), over in cases:
        p = dict(ptr, **(over or {}))
        rc = _rc(e, *_abi_args(e, p["qkv"], p["out"], p["lse"], p["gout"], p["gqkv"], p["ws"], nn, f, heads))
        assert rc == -1, (e, nn, f, heads, over, rc)
    torch.cuda.synchronize()
    assert _lib.launch_count() == before
    for k in ("out", "lse", "gqkv", "ws"):
        assert bool((buf[k].view(torch.int32) == NAN_BITS).all()), k


@pytest.mark.gpu
@pytest.mark.parametrize("f,heads", [(8, 1), (64, 8), (64, 2)])
def test_empty_sequence_with_null_pointers(f, heads):
    """n = 0: every entry returns 0 and launches nothing, whatever the pointers (an empty tensor's address may be NULL)"""
    torch.cuda.synchronize()
    before = _lib.launch_count()
    for e in ENTRIES:
        if e.startswith("hgb_mha_tc") and f // heads != 8:
            continue
        assert _rc(e, *_abi_args(e, None, None, None, None, None, None, 0, f, heads)) == 0, e
    assert _lib.launch_count() == before


# ---- 7. module level ----------------------------------------------------------------------------------------------------------
@pytest.mark.gpu
@pytest.mark.parametrize("f,heads", [(64, 8), (64, 4)])
def test_mha_fn_on_an_empty_sequence(f, heads):
    from hydragnn_b200 import gps
    x = torch.empty(0, 3 * f, device=DEV, requires_grad=True)
    torch.cuda.synchronize()
    before = _lib.launch_count()
    out = gps.MhaFn.apply(x, heads)
    g, = torch.autograd.grad(out, x, torch.empty(0, f, device=DEV))
    assert out.shape == (0, f) and g.shape == (0, 3 * f)
    assert _lib.launch_count() == before


def _offset_view(x):
    """a contiguous copy of x whose first element sits 4 bytes past a 16-byte boundary"""
    buf = torch.empty(x.numel() + 4, device=DEV)
    v = buf[1:1 + x.numel()].view_as(x)
    v.copy_(x)
    assert v.data_ptr() % 16 == 4
    return v


@pytest.mark.gpu
@pytest.mark.parametrize("tf32", [False, True])
@pytest.mark.parametrize("which", ["qkv", "gout"])
def test_mha_fn_on_misaligned_views_takes_the_simt_kernels(which, tf32):
    """a qkv view (forward and backward) or a gout view (backward) 4 bytes off a 16-byte boundary at d = 8 runs the SIMT
    kernels, which make scalar accesses, and gives the fp64 answer to their tolerance"""
    n, f, heads = 333, 64, 8
    x, go = inputs(n, f, "normal", 5)
    if which == "qkv":
        x = _offset_view(x)
    else:
        go = _offset_view(go)
    _lib.trace_begin()
    try:
        out, g = _mha_module(x, heads, go, tf32)
    finally:
        calls = _lib.trace_end()
    want = ["hgb_mha_fwd" if which == "qkv" else "hgb_mha_tc_fwd", "hgb_mha_bwd"]
    assert [c[0] for c in calls] == want, calls
    ref_out, _, ref_g, sc = ref_blockwise(x.double(), go.double(), heads)
    tol = TOL["tf32" if (tf32 and which == "gout") else "simt"]
    check_rows(which, "out", out, ref_out, sc["out"], tol["out"], heads, sc["cond_q"])
    for name, cols, cond in (("dq", slice(0, f), "cond_q"), ("dk", slice(f, 2 * f), "cond_k"),
                             ("dv", slice(2 * f, 3 * f), "cond_k")):
        check_rows(which, name, g[:, cols], ref_g[:, cols], sc[name], tol["grad"], heads, sc[cond])


@pytest.mark.gpu
@pytest.mark.parametrize("n,f,heads", [(1, 8, 1), (9, 16, 2), (40, 64, 8), (33, 8, 2), (70, 32, 1)])
def test_any_order_attention_derivatives(n, f, heads):
    """gps.mha_any_order (MatMul + ATen softmax, the path of MLIP training through GPS): value, first derivative and a
    Hessian-vector product (create_graph=True) against fp64 autograd of the plain expression"""
    from hydragnn_b200 import gps
    g = torch.Generator().manual_seed(n + f)
    x64 = torch.randn(n, 3 * f, generator=g, dtype=torch.float64)
    go = torch.randn(n, f, generator=g, dtype=torch.float64)
    w = torch.randn(n, 3 * f, generator=g, dtype=torch.float64)

    def derivatives(fn, x, go, w):
        x = x.detach().clone().requires_grad_(True)
        out = fn(x)
        gx, = torch.autograd.grad(out, x, go, create_graph=True)
        hv, = torch.autograd.grad(gx, x, w)
        return out.detach(), gx.detach(), hv

    def plain(x):
        q, k, v = (_heads(t, heads) for t in x.split(f, dim=1))
        return _unheads(torch.softmax(q @ k.transpose(1, 2) / math.sqrt(f // heads), -1) @ v)

    r = derivatives(plain, x64, go, w)
    e = derivatives(lambda x: gps.mha_any_order(x, heads), x64.float().to(DEV), go.float().to(DEV), w.float().to(DEV))
    for name, a, b, tol in zip(("out", "grad", "hvp"), e, r, (1e-5, 1e-5, 1e-4)):
        assert rel_l2(a.cpu(), b) < tol, (name, rel_l2(a.cpu(), b))
