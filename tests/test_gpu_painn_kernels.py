"""Kernel-level tests of the PaiNN message kernels (csrc/hgb_painn.cu) and of the edge embedding and edge records they read,
each against a plain fp64 restatement of the operation include/hgb.h states:

    W_e = rb_e[:r] wf^T + bf fc_e  (* efilt_e),      (g_v, g_e, m_s) = split(W_e * phi[j_e])
    s_out = s + index_add(i, m_s),                   v_out = v + index_add(i, v[j] g_v + g_e (x) dir_e)

with i = edge_index[0] (the aggregating node) and j = edge_index[1].  The backward references are fp64 autograd of the same
expression.  The C-ABI is called directly, so the test controls every argument: the edge-record pointer (SIMT or tiled
kernel), the affine-v inputs and the alignment of the rows.

Every output buffer and the workspace start as NaN, so a row or partial a kernel leaves unwritten shows up.  With inputs drawn
from {0, +-1/2, +-1}, every term the kernels form is a multiple of 2^-6; while the sum of the magnitudes of an output's terms
stays below 2^18 (checked per output with the same expression on |inputs|), fp32 computes it exactly and the kernels must
equal fp64 bit for bit, whatever their summation order.

`census` mirrors the dispatch and tile rules of hgb_painn_message_{fwd,bwd} and asserts that each tiled case reaches what
production batches reach only at scale: more than two tiles per CTA (the double-buffer mbarrier parity comes back to 1),
segments longer than the 8 records a warp stages, neighbours outside the tile, a partial last tile.  The dispatch test checks
with torch.profiler which template each case launched.
"""
import functools
import math
import re
import types

import pytest
import torch

from hydragnn_b200 import _lib, ops

DEV = "cuda"
NSM = 132
EPK = 12
TOL, TOL_W = 1e-5, 1e-4
EXACT_UNIT = 2.0 ** -6           # every term of every output is a multiple of this in exact mode
EXACT_LIMIT = 2.0 ** 24 * EXACT_UNIT
N_CANDIDATES = (20011, 40009)    # graph sizes the census picks from (the smallest that reaches every tiled path)

F_SIMT = (1, 2, 3, 5, 16, 17, 33, 63, 64, 65, 96, 320)
F_TILED = (64, 128, 192, 256)


# ---- fp64 references, from include/hgb.h ----------------------------------------------------------------------------------
def ref_message(x, row, col, n, f, r):
    """(s_out, v_out) of hgb_painn_message_fwd; x holds phi, s, v (or v_in, v_w, v_b), epack, wf, bf, efilt (or None)"""
    v = x["v"] if x.get("v") is not None else x["v_in"][:, :, None] * x["v_w"] + x["v_b"]
    ep = x["epack"]
    w = ep[:, :r] @ x["wf"].t() + x["bf"] * ep[:, 8:9]
    if x.get("efilt") is not None:
        w = w * x["efilt"]
    g_v, g_e, m_s = (w * x["phi"][col]).split(f, dim=1)
    m_v = v[col] * g_v[:, None, :] + g_e[:, None, :] * ep[:, 9:12, None]
    s_out = x["s"] + torch.zeros_like(x["s"]).index_add_(0, row, m_s)
    v_out = v + torch.zeros(n, 3, f, dtype=v.dtype, device=v.device).index_add_(0, row, m_v)
    return s_out, v_out


GRAD_OF = dict(gphi="phi", gv="v", g_epack="epack", gwf="wf", gbf="bf", g_efilt="efilt")


def ref_all(x, gs, gv_out, row, col, n, f, r):
    """fp64 outputs and gradients; an affine v enters as the leaf v = v_in v_w + v_b (gv is the gradient of that v)"""
    x = dict(x)
    if x.get("v") is None:
        x["v"] = x["v_in"][:, :, None] * x["v_w"] + x["v_b"]
    leaves = {k: x[k].detach().clone().requires_grad_(True) for k in GRAD_OF.values() if x.get(k) is not None}
    s_out, v_out = ref_message(dict(x, **leaves), row, col, n, f, r)
    grads = torch.autograd.grad((s_out, v_out), list(leaves.values()), (gs, gv_out))
    by_leaf = dict(zip(leaves, grads))
    out = dict(s_out=s_out.detach(), v_out=v_out.detach())
    out.update({g: by_leaf[k] for g, k in GRAD_OF.items() if k in by_leaf})
    return out


def ref_embed(unit, ln, r, cutoff):
    """epack [e, 12] of hgb_painn_edge_embed_fwd: sin(n pi d / rc) / d * fcut(d) for n = 1..r (zero padded to 8), fcut, unit/d"""
    d = ln.reshape(-1, 1)
    q = torch.arange(1, r + 1, dtype=d.dtype, device=d.device)
    fc = torch.where(d < cutoff, 0.5 * (torch.cos(math.pi * d / cutoff) + 1.0), torch.zeros_like(d))
    rb = torch.sin(q * math.pi * d / cutoff) / d * fc
    return torch.cat([rb, d.new_zeros(d.shape[0], 8 - r), fc, unit / d], dim=1)


def ref_records(epack, perm, nbr):
    """rec [e, 16] of hgb_painn_edge_records: epack[perm[p]], nbr[p] and perm[p] as int bits, two zeros"""
    e = nbr.numel()
    perm = torch.arange(e, dtype=torch.int32, device=nbr.device) if perm is None else perm
    ints = torch.stack([nbr, perm, torch.zeros_like(nbr), torch.zeros_like(nbr)], dim=1)
    return torch.cat([epack[perm.long()], ints.view(torch.float32)], dim=1)


# ---- CPU self-checks of the references ------------------------------------------------------------------------------------
def test_message_reference_matches_oracle():
    """the message reference, fed the oracle's own phi, filter and embedding, gives oracle.painn.PainnMessage"""
    from oracle.geometry import cosine_cutoff, sinc_expansion
    from oracle.painn import PainnMessage
    torch.manual_seed(3)
    n, f, r, rc = 23, 6, 5, 3.0
    m = PainnMessage(f, r, rc, edge_dim=2).double()
    pos = torch.rand(n, 3, dtype=torch.float64) * 4.0
    edge = torch.randint(0, n, (80, 2))
    edge = edge[edge[:, 0] != edge[:, 1]]
    vec = pos[edge[:, 1]] - pos[edge[:, 0]]
    dist = vec.norm(dim=1, keepdim=True)
    diff = vec / dist
    s, v = torch.randn(n, f, dtype=torch.float64), torch.randn(n, 3, f, dtype=torch.float64)
    eattr = torch.randn(edge.shape[0], 2, dtype=torch.float64)
    with torch.no_grad():
        s_o, v_o = m(s, v, edge, diff, dist, eattr)
        ep = torch.cat([sinc_expansion(dist, r, rc) * cosine_cutoff(dist, rc), dist.new_zeros(dist.shape[0], 8 - r),
                        cosine_cutoff(dist, rc), diff / dist], dim=1)
        x = dict(phi=m.scalar_message_mlp(s), s=s, v=v, epack=ep, wf=m.filter_layer.weight, bf=m.filter_layer.bias,
                 efilt=m.edge_filter(eattr))
        s_r, v_r = ref_message(x, edge[:, 0], edge[:, 1], n, f, r)
    torch.testing.assert_close(s_r, s_o, rtol=1e-12, atol=1e-12)
    torch.testing.assert_close(v_r, v_o, rtol=1e-12, atol=1e-12)


def test_embed_reference_matches_oracle():
    from oracle.geometry import cosine_cutoff, sinc_expansion
    g = torch.Generator().manual_seed(5)
    d = torch.cat([torch.rand(50, 1, generator=g, dtype=torch.float64) * 4.0 + 1e-3, torch.tensor([[3.0], [3.5]])])
    unit = torch.nn.functional.normalize(torch.randn(d.shape[0], 3, generator=g, dtype=torch.float64), dim=1)
    for r in range(1, 9):
        ep = ref_embed(unit, d, r, 3.0)
        torch.testing.assert_close(ep[:, :r], sinc_expansion(d, r, 3.0) * cosine_cutoff(d, 3.0), rtol=1e-13, atol=1e-13)
        assert torch.equal(ep[:, r:8], torch.zeros_like(ep[:, r:8]))
        torch.testing.assert_close(ep[:, 8:9], cosine_cutoff(d, 3.0), rtol=1e-13, atol=1e-13)
        torch.testing.assert_close(ep[:, 9:], unit / d, rtol=1e-13, atol=1e-13)


# ---- graphs with a controlled degree profile --------------------------------------------------------------------------------
@functools.lru_cache(maxsize=None)
def _graph(n, seed=0):
    """edge_index [2, E] int64 on the CPU.  In both the by-row CSR (forward) and the by-col CSR (backward):
    - runs of isolated nodes at the start, at the end, across multiples of 480 (a multiple of every tile size) and one
      run of 130 (whole empty tiles);
    - nodes of degree 8, 9, 9, 8 in a row (the 8-record scratch of the tiled kernels) and a hub of 1000;
    - otherwise a few neighbours each, mostly within +-8 positions and 5 % anywhere in the graph (gathers from outside the tile).
    Edge ids are shuffled, so CSR order is not edge order."""
    g = torch.Generator().manual_seed(seed)
    iso = torch.zeros(n, dtype=torch.bool)
    iso[:37] = True
    iso[-41:] = True
    for a in range(480, n - 200, 480 * 7):
        iso[a - 3:a + 4 + a % 5] = True
    iso[n // 3:n // 3 + 130] = True
    special = torch.zeros(n, dtype=torch.bool)
    s8_row, s8_col = n // 5, n // 5 + 64
    hub_row, hub_col = 4 * n // 5, 3 * n // 5
    special[s8_row:s8_row + 4] = special[s8_col:s8_col + 4] = True
    special[hub_row] = special[hub_col] = True
    elig = torch.nonzero(~iso & ~special).flatten()
    pos_of = torch.searchsorted(elig, torch.arange(n))

    def neighbours(nodes):
        """one partner per entry of `nodes`: a nearby eligible node, or one anywhere (5 %)"""
        k = nodes.numel()
        near = elig[torch.clamp(pos_of[nodes] + torch.randint(-8, 9, (k,), generator=g), 0, elig.numel() - 1)]
        far = elig[torch.randint(0, elig.numel(), (k,), generator=g)]
        return torch.where(torch.rand(k, generator=g) < 0.05, far, near)

    deg_a = torch.randint(0, 6, (n,), generator=g) * (~iso & ~special)   # edges summed into node i (by-row side)
    deg_b = torch.randint(0, 4, (n,), generator=g) * (~iso & ~special)   # edges gathered from node j (by-col side)
    deg_a[s8_row:s8_row + 4] = torch.tensor([8, 9, 9, 8])
    deg_b[s8_col:s8_col + 4] = torch.tensor([9, 8, 8, 9])
    deg_a[hub_row] = 1000
    deg_b[hub_col] = 1000
    ra = torch.repeat_interleave(torch.arange(n), deg_a)
    cb = torch.repeat_interleave(torch.arange(n), deg_b)
    row = torch.cat([ra, neighbours(cb)])
    col = torch.cat([neighbours(ra), cb])
    order = torch.randperm(row.numel(), generator=g)
    return torch.stack([row[order], col[order]])


def _csr_cpu(idx, other, n):
    """(rowptr, nbr) of the CSR of `idx` (stable: ascending edge id within a segment), as hgb_csr_build / EdgePlan.nbr"""
    perm = torch.sort(idx, stable=True).indices
    rowptr = torch.zeros(n + 1, dtype=torch.int64)
    rowptr[1:] = torch.cumsum(torch.bincount(idx, minlength=n), 0)
    return rowptr, other[perm]


# ---- dispatch and tile rules of hgb_painn_message_{fwd,bwd} -----------------------------------------------------------------
def painn_group(f):
    g = 32
    if f < 32:
        g = 1
        while g < f:
            g <<= 1
    return g


def tile_size(kernel, f):
    """tn of the tiled kernels: 'fwd' (plain v), 'fwd_av' (affine v) or 'bwd'"""
    if kernel == "bwd":
        fixed = 32 + 8 * 32 * 4 + 8 * 4096
        tn = (110 * 1024 - fixed) // (2 * 4 * f * 4) // 8 * 8
        return max(min(tn, 32), 8)
    av = kernel == "fwd_av"
    fixed = 10 * 1536 + 64
    step = 20 if av else 10
    tn = (110 * 1024 - fixed) // (2 * 3 * f * 4 + 24 if av else 4 * 3 * f * 4) // step * step
    return max(tn, step)


def grid_x(kernel, n, f, ntiles=None):
    """CTAs along x: the SIMT backward's painn_bwd_grid (which sizes the workspace), or the tiled kernels' grid"""
    bwd_grid = min(max(-(-n // (8 * (32 // painn_group(f)))), 1), NSM * (2 if f < 32 else 4))
    if ntiles is None:
        return bwd_grid
    return min(ntiles, 2 * NSM, bwd_grid) if kernel == "bwd" else min(ntiles, 2 * NSM)


def census(rowptr, nbr, f, kernel):
    """What one tiled launch reaches with this CSR (rowptr [n+1], nbr [e] in CSR order), by the kernels' tile rule"""
    rp = rowptr.cpu().long()
    nb = nbr.cpu().long()
    n = rp.numel() - 1
    tn = tile_size(kernel, f)
    ntiles = -(-n // tn)
    grid = grid_x(kernel, n, f, ntiles)
    deg = rp[1:] - rp[:-1]
    owner = torch.repeat_interleave(torch.arange(n), deg)
    last_rows = n - (ntiles - 1) * tn
    return dict(n=n, tn=tn, ntiles=ntiles, grid=grid, max_degree=int(deg.max()),
                outside=int((nb // tn != owner // tn).sum()), last_rows=last_rows, last_vin_bytes=12 * last_rows)


def census_ok(c, kernel):
    return (c["ntiles"] > 2 * c["grid"]            # some CTA runs a third tile: the mbarrier parity of a buffer returns to 1
            and c["max_degree"] > 8                # records beyond the 8 staged ones are read from global memory
            and c["outside"] > 0                   # neighbour rows outside the tile are gathered from global memory
            and c["last_rows"] < c["tn"]           # a partial last tile
            and (kernel != "fwd_av" or c["last_vin_bytes"] % 16 != 0))   # the issuing thread stores the v_in tail


def assert_census(rowptr, nbr, f, kernel):
    c = census(rowptr, nbr, f, kernel)
    assert census_ok(c, kernel), (kernel, f, c)
    return c


@functools.lru_cache(maxsize=None)
def n_for(kernel, f):
    """the smallest candidate size whose graph reaches every tiled path of this kernel"""
    for n in N_CANDIDATES:
        ei = _graph(n)
        side = (ei[0], ei[1]) if kernel.startswith("fwd") else (ei[1], ei[0])
        if census_ok(census(*_csr_cpu(side[0], side[1], n), f, kernel), kernel):
            return n
    raise AssertionError("no candidate graph reaches every tiled path of %s at f = %d" % (kernel, f))


def test_census_tile_sizes():
    """the tile sizes the census assumes (hgb_painn.cu); a change of the kernels' shared-memory plan must show up here"""
    assert [tile_size("fwd", f) for f in F_TILED] == [30, 10, 10, 10]
    assert tile_size("fwd_av", 64) == 60
    assert [tile_size("bwd", f) for f in F_TILED] == [32, 16, 8, 8]


def test_census_graph_reaches_every_tiled_path():
    """the test graphs reach every path of every tiled kernel, in the by-row and the by-col CSR alike"""
    for kernel, fs in (("fwd", F_TILED), ("bwd", F_TILED), ("fwd_av", (64,))):
        for f in fs:
            n = n_for(kernel, f)
            ei = _graph(n)
            for idx, other in ((ei[0], ei[1]), (ei[1], ei[0])):
                rowptr, nbr = _csr_cpu(idx, other, n)
                deg = rowptr[1:] - rowptr[:-1]
                assert bool((deg[:37] == 0).all()) and bool((deg[-41:] == 0).all())
                assert int(deg.max()) == 1000
                pair = (deg[:-1] == 8) & (deg[1:] == 9)
                assert bool(pair.any())
                assert census_ok(census(rowptr, nbr, f, kernel), kernel)


def expected_kernels(n, f, r, ef, need_edge, rec, av, align):
    """(forward, backward) template the dispatch picks; align = largest power of two (<= 16) dividing every row address"""
    b = lambda t: "true" if t else "false"  # noqa: E731
    rt = 5 if r <= 5 else 8
    if rec and f % 64 == 0 and f <= 256 and n >= 256 and align >= 16:
        ft = 64 if f == 64 else 0
        return ("painn_message_fwd_tiled_kernel<%s, %d, %d, %s>" % (b(ef), rt, ft, b(av)),
                "painn_message_bwd_tiled_kernel<%s, %s, %d, %d, %s>" % (b(ef), b(need_edge), rt, ft, b(av)))
    cpl = 2 if (f >= 64 and f % 2 == 0 and align >= 8) else 1
    g = painn_group(f)
    return ("painn_message_fwd_kernel<%d, %s, %d, %d>" % (cpl, b(ef), g, rt),
            "painn_message_bwd_kernel<%d, %s, %s, %d, %d>" % (cpl, b(ef), b(need_edge), g, rt))


def all_instantiations():
    """every template hgb_painn_message_{fwd,bwd} can launch"""
    bs = ("false", "true")
    simt = [(1, 1), (1, 2), (1, 4), (1, 8), (1, 16), (1, 32), (2, 32)]
    tiled = [(64, "false"), (0, "false"), (64, "true")]
    out = set()
    for rt in (5, 8):
        for ef in bs:
            for cpl, g in simt:
                out.add("painn_message_fwd_kernel<%d, %s, %d, %d>" % (cpl, ef, g, rt))
                for ne in bs:
                    out.add("painn_message_bwd_kernel<%d, %s, %s, %d, %d>" % (cpl, ef, ne, g, rt))
            for ft, av in tiled:
                out.add("painn_message_fwd_tiled_kernel<%s, %d, %d, %s>" % (ef, rt, ft, av))
                for ne in bs:
                    out.add("painn_message_bwd_tiled_kernel<%s, %s, %d, %d, %s>" % (ef, ne, rt, ft, av))
    return out


# ---- cases ------------------------------------------------------------------------------------------------------------------
def _simt_cases():
    """every f at r = 5 and r = 8 with and without edge filter and edge gradient, and the other radial counts on some widths"""
    cases = [(f, r, ef, ne) for f in F_SIMT for r in (5, 8) for ef in (False, True) for ne in (False, True)]
    cases += [(f, r, (f + r) % 2 == 0, True) for f in (1, 3, 17, 64, 65) for r in (1, 3, 6)]
    return cases


def _tiled_cases():
    """(f, r, efilt, need_edge, affine v)"""
    cases = [(f, r, ef, ne, False) for f in F_TILED for r in (5, 8) for ef in (False, True) for ne in (False, True)]
    return cases + [(64, r, ef, ne, True) for r in (5, 8) for ef in (False, True) for ne in (False, True)]


def _case_id(c):
    return "-".join("%s%s" % (k, int(v) if isinstance(v, bool) else v) for k, v in zip(("f", "r", "ef", "ne", "av"), c))


SIMT_CASES = _simt_cases()
TILED_CASES = _tiled_cases()


# ---- GPU side ---------------------------------------------------------------------------------------------------------------
@functools.lru_cache(maxsize=None)
def _plan(n):
    ei = _graph(n).to(DEV)
    c = types.SimpleNamespace(n=n, e=ei.shape[1], ei=ei, row=ei[0], col=ei[1])
    c.plan = ops.EdgePlan(ei, n)
    return c


def _inputs(c, f, r, ef, exact, av=False, seed=0):
    """fp64 inputs on the GPU whose values fp32 holds exactly; epack is zero beyond column r, as hgb.h requires"""
    g = torch.Generator(device=DEV).manual_seed(1000 * f + 10 * r + 2 * ef + exact + 7 * seed)
    n, e = c.n, c.e

    def t(*shape, scale=1.0, shift=0.0):
        if exact:
            return torch.randint(-2, 3, shape, generator=g, device=DEV).double() / 2
        return (torch.randn(*shape, generator=g, device=DEV) * scale + shift).float().double()

    ep = torch.cat([t(e, r, scale=0.5), torch.zeros(e, 8 - r, dtype=torch.float64, device=DEV), t(e, 4, scale=0.7)], dim=1)
    x = dict(phi=t(n, 3 * f), s=t(n, f), epack=ep, wf=t(3 * f, r, scale=0.3), bf=t(3 * f, scale=0.3),
             efilt=t(e, 3 * f, scale=0.5, shift=0.5) if ef else None, gs=t(n, f), gv_out=t(n, 3, f))
    if av:
        x.update(v_in=t(n, 3), v_w=t(f, scale=0.5), v_b=t(f, scale=0.2))
    else:
        x["v"] = t(n, 3, f)
    return x


def _f32(x):
    return {k: (None if v is None else v.float().contiguous()) for k, v in x.items()}


def _nan(*shape):
    return torch.full(shape, float("nan"), dtype=torch.float32, device=DEV)


def _p(t):
    return None if t is None else t.data_ptr()


def run_fwd(c, x, f, r, rec=None, phi=None, nbr=None):
    """s_out, v_out of hgb_painn_message_fwd into NaN-filled buffers; x: fp32 inputs, rec: by-row records or None"""
    s_out, v_out = _nan(c.n, f), _nan(c.n, 3, f)
    agg = c.plan.by_row
    _lib.call("hgb_painn_message_fwd", _p(x["phi"] if phi is None else phi), _p(x["s"]), _p(x.get("v")), _p(x.get("v_in")),
              _p(x.get("v_w")), _p(x.get("v_b")), _p(agg.rowptr), _p(agg.perm), _p(c.plan.nbr("row") if nbr is None else nbr),
              _p(x["epack"]), _p(rec), _p(x["wf"]), _p(x["bf"]), _p(x.get("efilt")), c.n, f, r, _p(s_out), _p(v_out),
              ops._stream())
    return dict(s_out=s_out, v_out=v_out)


def run_bwd(c, x, f, r, need_edge, rec=None, phi=None, nbr=None):
    """gphi, gv, gwf, gbf (+ g_epack, g_efilt) of hgb_painn_message_bwd into NaN-filled buffers and a NaN-filled workspace
    (hgb.h: the kernels write every column of g_epack, the caller zeroes nothing); rec: by-col records or None"""
    n, e = c.n, c.e
    out = dict(gphi=_nan(n, 3 * f), gv=_nan(n, 3, f), gwf=_nan(3 * f, r), gbf=_nan(3 * f))
    if need_edge:
        out["g_epack"] = _nan(e, EPK)
    if x.get("efilt") is not None:
        out["g_efilt"] = _nan(e, 3 * f)
    nbytes = _lib.query("hgb_painn_message_bwd_workspace_bytes", n, f, r, e)
    ws = torch.full((max(nbytes, 16),), 255, dtype=torch.uint8, device=DEV)     # all-ones bytes: NaN floats
    src = c.plan.by_col
    _lib.call("hgb_painn_message_bwd", _p(x["gs"]), _p(x["gv_out"]), _p(x["phi"] if phi is None else phi), _p(x.get("v")),
              _p(x.get("v_in")), _p(x.get("v_w")), _p(x.get("v_b")), _p(src.rowptr), _p(src.perm),
              _p(c.plan.nbr("col") if nbr is None else nbr), _p(x["epack"]), _p(rec), _p(x["wf"]), _p(x["bf"]), _p(x.get("efilt")),
              n, f, r, e, _p(out["gphi"]), _p(out["gv"]), _p(out["gwf"]), _p(out["gbf"]), _p(out.get("g_epack")),
              _p(out.get("g_efilt")), _p(ws), nbytes, ops._stream())
    return out


def run_both(c, x, f, r, need_edge, tiled, phi=None):
    """forward and backward, with the edge records of both CSR views when tiled"""
    rec_row = ops.painn_edge_records(x["epack"], c.plan, "row") if tiled else None
    rec_col = ops.painn_edge_records(x["epack"], c.plan, "col") if tiled else None
    k = run_fwd(c, x, f, r, rec_row, phi)
    k.update(run_bwd(c, x, f, r, need_edge, rec_col, phi))
    return k


def rel(a, ref):
    a, ref = a.double(), ref.double()
    den = ref.norm()
    return float((a - ref).norm() / den) if float(den) > 0 else float((a - ref).abs().max())


def same_bits(a, b):
    """bitwise equality of two fp32 tensors, +0 and -0 taken as equal"""
    return a.shape == b.shape and torch.equal((a.float() + 0.0).view(torch.int32), (b.float() + 0.0).view(torch.int32))


PER_ELEMENT = ("s_out", "v_out", "gphi", "gv", "g_epack", "g_efilt")


def check(k, ref, bound, what, r):
    """k: kernel outputs; ref: fp64 references; bound: the same on |inputs| (exact mode) or None"""
    for name, a in k.items():
        ref_a = ref[name]
        assert bool(torch.isfinite(a).all()), "%s: %s has %d unwritten or non-finite entries" % (
            what, name, int((~torch.isfinite(a)).sum()))
        err = rel(a, ref_a)
        assert err <= (TOL_W if name in ("gwf", "gbf") else TOL), "%s: %s rel-L2 %.3g" % (what, name, err)
        if name == "g_epack":
            assert bool((a[:, r:8] == 0).all()), "%s: g_epack padding columns %d..7 are not 0" % (what, r)
        if bound is None:
            continue
        ok = bound[name] < EXACT_LIMIT
        if name in PER_ELEMENT:
            assert bool(ok.all()), "%s: %s leaves the exact range (max term sum %g)" % (what, name, float(bound[name].max()))
        assert same_bits(a[ok], ref_a[ok].float()), "%s: %s differs from fp64 in %d of %d exact entries" % (
            what, name, int((a[ok].double() != ref_a[ok]).sum()), int(ok.sum()))


def _bound(x, c, f, r):
    ax = {k: (None if v is None else v.abs()) for k, v in x.items()}
    return ref_all(ax, ax["gs"], ax["gv_out"], c.row, c.col, c.n, f, r)


def run_case(c, f, r, ef, need_edge, tiled, av, exact, check_determinism=True, phi_offset=False):
    what = "n=%d f=%d r=%d ef=%d ne=%d tiled=%d av=%d exact=%d" % (c.n, f, r, ef, need_edge, tiled, av, exact)
    x = _inputs(c, f, r, ef, exact, av)
    x32 = _f32(x)
    phi = None
    if phi_offset:                  # a row view 4 bytes past a 16-byte boundary: neither the tiled nor the 8-byte loads apply
        buf = torch.empty(x32["phi"].numel() + 1, device=DEV)
        phi = buf[1:].view_as(x32["phi"])
        phi.copy_(x32["phi"])
    k = run_both(c, x32, f, r, need_edge, tiled, phi)
    torch.cuda.synchronize()
    ref = ref_all(x, x["gs"], x["gv_out"], c.row, c.col, c.n, f, r)
    check(k, ref, _bound(x, c, f, r) if exact else None, what, r)
    if check_determinism:
        again = run_both(c, x32, f, r, need_edge, tiled, phi)
        for name in k:
            assert torch.equal(k[name].view(torch.int32), again[name].view(torch.int32)), \
                "%s: %s differs between two identical calls" % (what, name)


# ---- 1. SIMT kernels --------------------------------------------------------------------------------------------------------
@pytest.mark.gpu
@pytest.mark.parametrize("exact", [False, True])
@pytest.mark.parametrize("f,r,ef,ne", SIMT_CASES, ids=[_case_id(c) for c in SIMT_CASES])
def test_simt_message_matches_fp64(f, r, ef, ne, exact):
    c = _plan(N_CANDIDATES[0])
    run_case(c, f, r, ef, ne, tiled=False, av=False, exact=exact)


# ---- 2. tiled kernels -------------------------------------------------------------------------------------------------------
@pytest.mark.gpu
@pytest.mark.parametrize("exact", [False, True])
@pytest.mark.parametrize("f,r,ef,ne,av", TILED_CASES, ids=[_case_id(c) for c in TILED_CASES])
def test_tiled_message_matches_fp64(f, r, ef, ne, av, exact):
    n = max(n_for("fwd_av" if av else "fwd", f), n_for("bwd", f))
    c = _plan(n)
    assert_census(c.plan.by_row.rowptr, c.plan.nbr("row"), f, "fwd_av" if av else "fwd")
    assert_census(c.plan.by_col.rowptr, c.plan.nbr("col"), f, "bwd")
    run_case(c, f, r, ef, ne, tiled=True, av=av, exact=exact)


# ---- 3. the tiled rule failing: misaligned rows, n = 255 -------------------------------------------------------------------
@pytest.mark.gpu
@pytest.mark.parametrize("f", [64, 128])
def test_misaligned_phi_falls_back_to_simt(f):
    run_case(_plan(N_CANDIDATES[0]), f, 5, True, True, tiled=True, av=False, exact=False, phi_offset=True)


@pytest.mark.gpu
@pytest.mark.parametrize("n", [255, 256])
@pytest.mark.parametrize("exact", [False, True])
def test_small_graph_around_the_tiled_limit(n, exact):
    run_case(_plan(n), 64, 5, False, True, tiled=True, av=False, exact=exact)
    run_case(_plan(n), 128, 8, True, True, tiled=True, av=False, exact=exact)


# ---- 4. which template each case reaches ------------------------------------------------------------------------------------
@pytest.mark.gpu
def test_dispatch_reaches_every_instantiation():
    """each case launches the template the dispatch rule names, and together they launch every template"""
    from torch.profiler import ProfilerActivity, profile
    runs = []
    for f, r, ef, ne in SIMT_CASES:
        runs.append((N_CANDIDATES[0], f, r, ef, ne, False, False, False))
    for f, r, ef, ne, av in TILED_CASES:
        runs.append((max(n_for("fwd_av" if av else "fwd", f), n_for("bwd", f)), f, r, ef, ne, True, av, False))
    runs += [(N_CANDIDATES[0], 64, 5, True, True, True, False, True), (255, 64, 8, False, True, True, False, False),
             (256, 64, 8, False, True, True, False, False)]
    prepared = []
    for n, f, r, ef, ne, tiled, av, offset in runs:
        c = _plan(n)
        x32 = _f32(_inputs(c, f, r, ef, False, av))
        phi = None
        if offset:
            phi = torch.empty(x32["phi"].numel() + 1, device=DEV)[1:].view_as(x32["phi"])
            phi.copy_(x32["phi"])
        prepared.append((c, x32, phi, n, f, r, ef, ne, tiled, av))
    torch.cuda.synchronize()
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        for c, x32, phi, n, f, r, ef, ne, tiled, av in prepared:
            run_both(c, x32, f, r, ne, tiled, phi)
        torch.cuda.synchronize()
    pat = re.compile(r"(painn_message_(?:fwd|bwd)(?:_tiled)?_kernel<[^>]*>)")
    kern = [(e.time_range.start, pat.search(e.name)) for e in prof.events() if pat.search(e.name)]
    seen = [m.group(1) for _, m in sorted(kern, key=lambda t: t[0])]
    want = []
    for c, x32, phi, n, f, r, ef, ne, tiled, av in prepared:
        want += list(expected_kernels(n, f, r, ef, ne, tiled, av, 4 if phi is not None else 16))
    assert len(seen) == len(want), (len(seen), len(want))
    for i, (s, w) in enumerate(zip(seen, want)):
        assert s == w, "launch %d (%s): reached %s" % (i, prepared[i // 2][3:], s)
    missing = all_instantiations() - set(seen)
    assert not missing, sorted(missing)


# ---- 5. edge records and edge embedding -------------------------------------------------------------------------------------
@pytest.mark.gpu
@pytest.mark.parametrize("which", ["row", "col", "identity"])
def test_edge_records_match_reference_bit_for_bit(which):
    c = _plan(N_CANDIDATES[0])
    ep = _f32(_inputs(c, 1, 8, False, False))["epack"]
    if which == "identity":
        perm, nbr = None, c.plan.nbr("row")
    else:
        perm, nbr = (c.plan.by_row.perm if which == "row" else c.plan.by_col.perm), c.plan.nbr(which)
    rec = _nan(c.e, 16)
    _lib.call("hgb_painn_edge_records", _p(ep), _p(perm), _p(nbr), c.e, _p(rec), ops._stream())
    want = ref_records(ep, perm, nbr)
    assert torch.equal(rec.view(torch.int32), want.view(torch.int32))


def _embed_inputs(e, cutoff, seed):
    """len [e] (fp32) in four groups -- near 0, inside, cutoff - 1 ulp / cutoff / cutoff + 1 ulp, beyond -- and unit [e, 3]"""
    g = torch.Generator(device=DEV).manual_seed(seed)
    q = e // 4
    c32 = torch.tensor(cutoff, dtype=torch.float32)
    edge = torch.stack([torch.nextafter(c32, torch.tensor(0.0)), c32, torch.nextafter(c32, torch.tensor(2 * cutoff))]).to(DEV)
    ln = torch.cat([torch.rand(q, generator=g, device=DEV) * 1e-3 + 1e-5,
                    torch.rand(q, generator=g, device=DEV) * (cutoff - 0.01) + 0.005,
                    edge.repeat(q // 3 + 1)[:q],
                    torch.rand(e - 3 * q, generator=g, device=DEV) * cutoff + cutoff])
    unit = torch.nn.functional.normalize(torch.randn(e, 3, generator=g, device=DEV), dim=1)
    groups = torch.repeat_interleave(torch.arange(4, device=DEV), torch.tensor([q, q, q, e - 3 * q], device=DEV))
    return ln, unit, groups


EMBED_E = 600_000     # > 132 * 16 blocks of 256 threads: the grid-stride loops run a second round


@pytest.mark.gpu
@pytest.mark.parametrize("r", range(1, 9))
def test_edge_embed_matches_fp64(r):
    cutoff = 3.0
    ln, unit, grp = _embed_inputs(EMBED_E, cutoff, r)
    ep = _nan(EMBED_E, EPK)
    _lib.call("hgb_painn_edge_embed_fwd", _p(unit), _p(ln), EMBED_E, r, cutoff, _p(ep), ops._stream())
    g_ep = torch.randn(EMBED_E, EPK, device=DEV, generator=torch.Generator(device=DEV).manual_seed(r))
    g_unit, g_len = _nan(EMBED_E, 3), _nan(EMBED_E)
    _lib.call("hgb_painn_edge_embed_bwd", _p(unit), _p(ln), _p(g_ep), EMBED_E, r, cutoff, _p(g_unit), _p(g_len), ops._stream())
    torch.cuda.synchronize()
    u64 = unit.double().requires_grad_(True)
    l64 = ln.double().requires_grad_(True)
    ref = ref_embed(u64, l64, r, cutoff)
    ru, rl = torch.autograd.grad(ref, (u64, l64), g_ep.double())
    ref = ref.detach()
    assert bool(torch.isfinite(ep).all()) and bool(torch.isfinite(g_unit).all()) and bool(torch.isfinite(g_len).all())
    assert bool((ep[:, r:8] == 0).all())
    beyond = ln >= cutoff
    assert bool((ep[beyond, :9] == 0).all()), "rbf and fcut must vanish at and beyond the cutoff"
    assert bool((ep[grp <= 1, 8] > 0).all())
    for cols in (slice(0, r), slice(8, 9), slice(9, 12)):
        assert rel(ep[:, cols], ref[:, cols]) <= TOL, (cols, rel(ep[:, cols], ref[:, cols]))
    for k in range(4):                       # per distance group: the near-zero group's 1/d^2 terms would hide the others
        m = grp == k
        assert rel(g_len[m], rl[m]) <= TOL, (k, rel(g_len[m], rl[m]))
        assert rel(g_unit[m], ru[m]) <= TOL, (k, rel(g_unit[m], ru[m]))


@pytest.mark.gpu
@pytest.mark.parametrize("r", [0, 9])
def test_radial_count_out_of_range_is_an_error(r):
    """r = 0 and r > 8 are refused before anything launches (the outputs keep their NaNs)"""
    c = _plan(256)
    x = _f32(_inputs(c, 64, 5, False, False))
    x["wf"] = torch.zeros(192, max(r, 1), device=DEV)
    rec_row, rec_col = (ops.painn_edge_records(x["epack"], c.plan, w) for w in ("row", "col"))
    torch.cuda.synchronize()
    before = _lib.launch_count()
    for fn in (lambda: run_fwd(c, x, 64, r, rec_row), lambda: run_bwd(c, x, 64, r, True, rec_col),
               lambda: run_fwd(c, x, 64, r), lambda: run_bwd(c, x, 64, r, True)):
        with pytest.raises(RuntimeError, match="num_radial"):
            fn()
    ln, unit, _ = _embed_inputs(64, 3.0, 0)
    ep, gu, gl = _nan(64, EPK), _nan(64, 3), _nan(64)
    with pytest.raises(RuntimeError, match="painn_edge_embed_fwd"):
        _lib.call("hgb_painn_edge_embed_fwd", _p(unit), _p(ln), 64, r, 3.0, _p(ep), ops._stream())
    with pytest.raises(RuntimeError, match="painn_edge_embed_bwd"):
        _lib.call("hgb_painn_edge_embed_bwd", _p(unit), _p(ln), _p(ep), 64, r, 3.0, _p(gu), _p(gl), ops._stream())
    torch.cuda.synchronize()
    assert _lib.launch_count() == before
    assert bool(ep.isnan().all()) and bool(gu.isnan().all()) and bool(gl.isnan().all())


# ---- 6. graphs without edges and without nodes ------------------------------------------------------------------------------
def _empty_graph(n):
    ei = torch.empty(2, 0, dtype=torch.int64, device=DEV)
    c = types.SimpleNamespace(n=n, e=0, ei=ei, row=ei[0], col=ei[1])
    c.plan = ops.EdgePlan(ei, n)
    return c


@pytest.mark.gpu
@pytest.mark.parametrize("n,f,av", [(0, 64, False), (5, 17, False), (5, 64, False), (300, 64, False), (300, 64, True),
                                    (300, 128, False)])
def test_message_c_abi_without_edges(n, f, av):
    """no edges: s_out = s, v_out = v, gphi = 0, gv = gv_out, gwf = gbf = 0 (n = 0: nothing but gwf = gbf = 0).  nbr, epack
    and rec point at a NaN record the kernels must not read (the pointers of an empty array may be NULL; hgb.h asks for them)"""
    c = _empty_graph(n)
    r = 5
    x = _f32(_inputs(c, f, r, False, True, av))
    dummy = _nan(1, 16)
    x["epack"] = dummy
    nbr = torch.zeros(1, dtype=torch.int32, device=DEV)
    for rec in ((None, dummy) if not av else (dummy,)):
        k = run_fwd(c, x, f, r, rec, nbr=nbr)
        k.update(run_bwd(c, x, f, r, False, rec, nbr=nbr))
        torch.cuda.synchronize()
        v = x["v"] if not av else x["v_in"][:, :, None] * x["v_w"] + x["v_b"]      # exact values: no rounding
        assert same_bits(k["s_out"], x["s"]) and same_bits(k["v_out"], v)
        assert bool((k["gphi"] == 0).all()) and same_bits(k["gv"], x["gv_out"])
        assert bool((k["gwf"] == 0).all()) and bool((k["gbf"] == 0).all())


@pytest.mark.gpu
@pytest.mark.parametrize("n,f,affine", [(0, 64, False), (5, 64, False), (300, 64, True), (300, 17, False)])
def test_message_module_without_edges(n, f, affine):
    """stacks.PainnMessage over a graph without edges (from the edge geometry on): the residuals pass through, the filter
    and message-MLP gradients are zero.  n = 300 at width 64 takes the affine-v branch."""
    from hydragnn_b200 import stacks
    torch.manual_seed(n + f)
    c = _empty_graph(n)
    m = stacks.PainnMessage(f, 5, 5.0).to(DEV)
    pos = torch.randn(n, 3, device=DEV, requires_grad=True)
    s = torch.randn(n, f, device=DEV, requires_grad=True)
    if affine:
        v0 = torch.randn(n, 3, 1, device=DEV, requires_grad=True)
        lin = torch.nn.Linear(1, f).to(DEV)
        v = ops.AffineV(v0, lin.weight, lin.bias)
        v_ref = ops.linear_act(v0, lin.weight, lin.bias).detach()
    else:
        v = torch.randn(n, 3, f, device=DEV, requires_grad=True)
        v_ref = v.detach()
    _, ln, unit = ops.EdgeGeomFn.apply(pos, None, c.plan, 1e-9)
    geom = {"epack": ops.PainnEdgeEmbedFn.apply(unit, ln, 5, 5.0)}
    if n == 0:      # the message MLP's Linear refuses zero rows: the fused message is entered with its phi directly
        phi = torch.randn(0, 3 * f, device=DEV, requires_grad=True)
        s_out, v_out = ops.PainnMessageFn.apply(phi, s, v, geom["epack"], m.filter_layer.weight, m.filter_layer.bias, None,
                                                c.plan)
    else:
        s_out, v_out = m(s, v, c.plan, geom)
    if affine and n >= 256:
        assert ops.painn_affine_v_ok(v, s, geom.get("rec_row"))
    gs, gv = torch.randn_like(s_out), torch.randn_like(v_out)
    (s_out * gs).sum().add_((v_out * gv).sum()).backward()
    torch.cuda.synchronize()
    assert same_bits(s_out.detach(), s.detach()) and same_bits(v_out.detach(), v_ref)
    assert same_bits(s.grad, gs)
    if affine:
        assert rel(lin.bias.grad, gv.double().sum(dim=(0, 1))) <= TOL
    else:
        assert same_bits(v.grad, gv)
    assert bool((pos.grad == 0).all())
    for name, p in m.named_parameters():
        assert p.grad is None or bool((p.grad == 0).all()), name


@pytest.mark.gpu
def test_painn_model_on_isolated_atoms():
    """a qm9_painn-shaped model, forward and backward, on a batch whose radius graph has no edges"""
    import hydragnn_b200 as hb
    from hydragnn_b200.synthetic import ARCH, make_samples
    torch.manual_seed(0)
    m = hb.create_model(**ARCH["qm9_painn"]).to(DEV)
    b = make_samples("qm9_painn", 64).to(DEV)
    b._num_graphs = 64
    b = hb.get_radius_graph(1e-4, 5)(b)
    assert b.edge_index.shape[1] == 0
    loss, _ = m.loss(m(b), b.y, [torch.arange(64, device=DEV)])
    loss.backward()
    torch.cuda.synchronize()
    assert math.isfinite(float(loss.detach()))
    for name, p in m.named_parameters():
        if p.grad is not None:
            assert bool(torch.isfinite(p.grad).all()), name
        if "filter_layer" in name or "scalar_message_mlp" in name:
            assert p.grad is None or bool((p.grad == 0).all()), name
