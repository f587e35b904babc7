"""GPU tests of MACE with edge attributes (edge_dim = D > 0): the fused first-order kernels (hgb_mace_tp_scatter_{fwd,bwd}
with edge attributes), the closed mixing primitive of the any-order path (hgb_mace_edge_mix, ops.EdgeMix / EdgeMixT), the
engine against the fp64 restatement (oracle/mace.py), and hb.train's padded step carrying edge_attr."""
import copy
import math

import pytest
import torch

pytestmark = pytest.mark.gpu

import hydragnn_b200 as hb  # noqa: E402
from hydragnn_b200 import e3, ops  # noqa: E402
from hydragnn_b200.synthetic import ARCH, make_samples  # noqa: E402
from oracle.mace import MACEOracle  # noqa: E402
from oracle.mlip import MLIPWrapper  # noqa: E402
from oracle.workloads import add_edges_cpu, arch_for  # noqa: E402
from stack_support import MACE_KW, _gpu_batch, _grad_rel, _loader, mace_batch, random_rotation  # noqa: E402

DEV = "cuda"
PAIRS = [(lin, lsh) for lsh in (1, 2, 3) for lin in (0, 1, 2) if lin <= lsh]


def rel_l2(a, b):
    return float((a.double().cpu() - b.double().cpu()).norm() / b.double().cpu().norm().clamp(min=1e-30))


# ---- fused kernels ---------------------------------------------------------------------------------------------------
def _tp_scatter_ref(up, sh, tpw, ea, ei, n, lin, lsh):
    """fp64 conv_tp + scatter with the reference's weight layout: 0e paths read a [F, D+1] block mixed with [ea, 1]."""
    f, d = up.shape[2], ea.shape[1]
    paths = e3.tp_paths(lin, lsh, lsh)
    a = torch.cat([ea, torch.ones_like(ea[:, :1])], dim=1)
    snd, rcv = ei[0], ei[1]
    per_l, col = [[] for _ in range(lsh + 1)], 0
    for (l1, l2, l3) in paths:
        if l2 == 0:
            w = torch.einsum("euv,ev->eu", tpw[:, col:col + f * (d + 1)].reshape(-1, f, d + 1), a) / math.sqrt(d + 1)
            col += f * (d + 1)
        else:
            w = tpw[:, col:col + f]
            col += f
        cg = (e3.w3j(l1, l2, l3) * math.sqrt(2 * l3 + 1)).to(up)
        x = up[snd][:, l1 * l1:(l1 + 1) ** 2]                                  # [E, 2l1+1, F]
        y = sh[:, l2 * l2:(l2 + 1) ** 2]
        per_l[l3].append(torch.einsum("ijk,eif,ej,ef->ekf", cg, x, y, w))
    assert col == tpw.shape[1]
    out = []
    for l3, parts in enumerate(per_l):
        m = torch.cat(parts, dim=2)
        out.append(m.new_zeros((n,) + m.shape[1:]).index_add_(0, rcv, m).reshape(-1))
    return torch.cat(out)


@pytest.mark.parametrize("d", [1, 2, 5])
@pytest.mark.parametrize("f", [32, 64, 128])
@pytest.mark.parametrize("lin,lsh", PAIRS)
def test_tp_scatter_with_edge_attr_matches_fp64(lin, lsh, f, d):
    gen = torch.Generator().manual_seed(100 * lin + 10 * lsh + f + d)
    n, e = 37, 260
    snd = torch.randint(0, n, (e,), generator=gen)
    rcv = torch.randint(0, n - 6, (e,), generator=gen)                        # the last six nodes receive nothing
    ei = torch.stack([snd, rcv])
    p, p0 = len(e3.tp_paths(lin, lsh, lsh)), lin + 1
    up = torch.randn(n, (lin + 1) ** 2, f, generator=gen, dtype=torch.float64)
    sh = torch.randn(e, (lsh + 1) ** 2, generator=gen, dtype=torch.float64)
    tpw = torch.randn(e, (p + d * p0) * f, generator=gen, dtype=torch.float64)
    ea = torch.randn(e, d, generator=gen, dtype=torch.float64)
    gout = torch.randn(_lib_nacc(lin, lsh) * n * f, generator=gen, dtype=torch.float64)
    leaves = [t.clone().requires_grad_(True) for t in (up, sh, tpw)]
    ref = _tp_scatter_ref(*leaves, ea, ei, n, lin, lsh)
    g_ref = torch.autograd.grad(ref, leaves, gout)
    plan = ops.EdgePlan(ei.to(DEV), n)
    results = []
    for _ in range(2):
        dl = [t.float().to(DEV).requires_grad_(True) for t in (up, sh, tpw)]
        out = ops.MaceTpScatterFn.apply(dl[0], dl[1], dl[2], plan, lin, lsh, ea.float().to(DEV))
        grads = torch.autograd.grad(out, dl, gout.float().to(DEV))
        results.append([out] + list(grads))
    assert rel_l2(results[0][0], ref) < 1e-5
    for name, a, b in zip(("up", "sh", "tpw"), results[0][1:], g_ref):
        assert rel_l2(a, b) < 1e-5, (name, rel_l2(a, b))
    off, paths = 0, e3.tp_paths(lin, lsh, lsh)                               # nodes without incoming edges: exact zeros
    for l3 in range(lsh + 1):
        width = (2 * l3 + 1) * sum(1 for q in paths if q[2] == l3) * f
        block = results[0][0][off:off + n * width].view(n, width)
        assert float(block[n - 6:].abs().max()) == 0.0
        off += n * width
    for a, b in zip(results[0], results[1]):                                  # deterministic: same bits on a repeat
        assert torch.equal(a, b)


def _lib_nacc(lin, lsh):
    from hydragnn_b200 import _lib
    return _lib.query("hgb_mace_tp_num_acc", lin, lsh)


def test_tp_scatter_edge_dim_bound():
    assert ops.mace_tp_supported(1, 2, 64, ops.MACE_TP_MAX_EDGE_DIM)
    assert not ops.mace_tp_supported(1, 2, 64, ops.MACE_TP_MAX_EDGE_DIM + 1)


# ---- closed mixing primitive -----------------------------------------------------------------------------------------
def test_edge_mix_both_modes_and_derivatives_match_fp64():
    gen = torch.Generator().manual_seed(7)
    e, f, d = 301, 24, 3
    c = 1.0 / math.sqrt(d + 1)
    tpw = torch.randn(e, 5 * f + f * (d + 1), generator=gen, dtype=torch.float64)
    ea = torch.randn(e, d, generator=gen, dtype=torch.float64)
    a = torch.cat([ea, torch.ones(e, 1, dtype=torch.float64)], dim=1)
    col = 2 * f                                                                # a column block of a wider row
    w_ref = tpw[:, col:col + f * (d + 1)].reshape(e, f, d + 1)
    tpw_d, ea_d = tpw.float().to(DEV), ea.float().to(DEV)
    out = ops.EdgeMix.apply(tpw_d[:, col:col + f * (d + 1)], ea_d, c)
    assert rel_l2(out, c * torch.einsum("euv,ev->eu", w_ref, a)) < 1e-6
    g = torch.randn(e, f, generator=gen, dtype=torch.float64)
    out_t = ops.EdgeMixT.apply(g.float().to(DEV), ea_d, c)
    assert rel_l2(out_t, (c * g[:, :, None] * a[:, None, :]).reshape(e, -1)) < 1e-6
    # first and second derivatives through the pair, against fp64 autograd of the same expression
    w64 = tpw.clone().requires_grad_(True)
    wd = tpw_d.clone().requires_grad_(True)
    r64 = c * torch.einsum("euv,ev->eu", w64[:, col:col + f * (d + 1)].reshape(e, f, d + 1), a)
    rd = ops.EdgeMix.apply(wd[:, col:col + f * (d + 1)], ea_d, c)
    h = torch.randn(e, f, generator=gen, dtype=torch.float64)
    obj64, objd = (r64.pow(2) * h).sum(), (rd.pow(2) * h.float().to(DEV)).sum()
    g64, = torch.autograd.grad(obj64, w64, create_graph=True)
    gd, = torch.autograd.grad(objd, wd, create_graph=True)
    assert rel_l2(gd, g64) < 1e-5
    k = torch.randn_like(tpw)
    gg64, = torch.autograd.grad((g64 * k).sum(), w64)
    ggd, = torch.autograd.grad((gd * k.float().to(DEV)).sum(), wd)
    assert rel_l2(ggd, gg64) < 1e-5
    # EdgeMixT's own derivatives
    g_leaf = g.float().to(DEV).requires_grad_(True)
    g64l = g.clone().requires_grad_(True)
    q = torch.randn(e, f * (d + 1), generator=gen, dtype=torch.float64)
    t64 = ((c * g64l[:, :, None] * a[:, None, :]).reshape(e, -1).pow(2) * q).sum()
    td = (ops.EdgeMixT.apply(g_leaf, ea_d, c).pow(2) * q.float().to(DEV)).sum()
    a64, = torch.autograd.grad(t64, g64l, create_graph=True)
    ad, = torch.autograd.grad(td, g_leaf, create_graph=True)
    assert rel_l2(ad, a64) < 1e-5
    b64, = torch.autograd.grad(a64.sum(), g64l)
    bd, = torch.autograd.grad(ad.sum(), g_leaf)
    assert rel_l2(bd, b64) < 1e-5


# ---- engine against the fp64 restatement -----------------------------------------------------------------------------
def _pair(kw, seed=0):
    torch.manual_seed(seed)
    o = MACEOracle(**kw)
    with torch.no_grad():
        for p in o.parameters():
            p.copy_(torch.randn_like(p) * (p.std() if p.numel() > 1 else 1.0))
    e = hb.create_model(mpnn_type="MACE", **kw)
    e.load_state_dict(o.state_dict(), strict=True)
    return o.double(), e


def _with_edge_attr(d, dim, gen):
    if dim == 1:
        d.edge_attr = (d.pos[d.edge_index[1]] - d.pos[d.edge_index[0]]).norm(dim=1, keepdim=True).detach()
    else:
        d.edge_attr = torch.randn(d.edge_index.shape[1], dim, generator=gen, dtype=torch.float64)
    return d


def _to_dev(d, pos_grad=False):
    g = hb.Batch(x=d.x.float().to(DEV), pos=d.pos.detach().float().to(DEV), edge_index=d.edge_index.to(DEV), batch=d.batch.to(DEV),
                 edge_attr=d.edge_attr.float().to(DEV))
    g._num_graphs = d.num_graphs
    if pos_grad:
        g.pos.requires_grad_(True)
    return g


@pytest.mark.parametrize("higher", [False, True])
@pytest.mark.parametrize("d", [1, 3])
@pytest.mark.parametrize("hidden", [8, 32, 64, 128])
def test_engine_matches_oracle_with_edge_attr(hidden, d, higher, monkeypatch):
    """First order (eval mode, as inference and first-order forces run): hidden 32 / 64 / 128 take the fused kernels, hidden 8
    the general TpOut + EdgeMix path.  higher=True: the any-order path (TpOut + EdgeMix) that MLIP force training uses."""
    kw = dict(MACE_KW, hidden_dim=hidden, edge_dim=d)
    o, e = _pair(kw)
    o.eval()
    if higher:
        e.train()
        e.force_higher_order = True
    else:
        e.eval()
    calls = {"fused": 0, "mix": 0}
    fused_apply, mix_apply = ops.MaceTpScatterFn.apply, ops.EdgeMix.apply

    def count(key, fn):
        def wrapped(*args):
            calls[key] += 1
            return fn(*args)
        return wrapped
    monkeypatch.setattr(ops.MaceTpScatterFn, "apply", count("fused", fused_apply))
    monkeypatch.setattr(ops.EdgeMix, "apply", count("mix", mix_apply))
    gen = torch.Generator().manual_seed(11)
    dd = _with_edge_attr(mace_batch(gen, sizes=(7, 9, 5)), d, gen)
    dd.pos.requires_grad_(True)
    ref = o(dd)
    g = _to_dev(dd, pos_grad=True)
    out = e(g)
    fused = not higher and hidden % 32 == 0
    layers = kw["num_conv_layers"]
    assert calls == {"fused": layers if fused else 0, "mix": 0 if fused else layers * (1 + kw["node_max_ell"]) - kw["node_max_ell"]}, calls
    for a, b in zip(out, ref):
        assert a.shape == b.shape and rel_l2(a, b) < 1e-5, rel_l2(a, b)
    lo = ref[0].sum() + ref[1].pow(2).sum()
    le = out[0].sum() + out[1].pow(2).sum()
    fo, = torch.autograd.grad(lo, dd.pos, retain_graph=True)
    fe, = torch.autograd.grad(le, g.pos, retain_graph=True)
    assert rel_l2(fe, fo) < 1e-5, rel_l2(fe, fo)
    lo.backward()
    le.backward()
    po, pe = dict(o.named_parameters()), dict(e.named_parameters())
    for k, p in po.items():
        if p.grad is None or float(p.grad.abs().max()) == 0:
            continue
        assert rel_l2(pe[k].grad, p.grad) < 2e-4, (k, rel_l2(pe[k].grad, p.grad))


def test_engine_tf32_mode_with_edge_attr_within_tolerance():
    o, e = _pair(dict(MACE_KW, hidden_dim=64, edge_dim=1))
    hb.set_precision(e, "bf16")
    gen = torch.Generator().manual_seed(4)
    dd = _with_edge_attr(mace_batch(gen, sizes=(7, 9, 5)), 1, gen)
    ref = o(dd)
    out = e(_to_dev(dd))
    for a, b in zip(out, ref):
        assert rel_l2(a, b) < 1e-3, rel_l2(a, b)


def test_engine_with_lengths_is_rotation_invariant():
    _, e = _pair(dict(MACE_KW, hidden_dim=32, edge_dim=1), seed=3)
    gen = torch.Generator().manual_seed(5)
    dd = _with_edge_attr(mace_batch(gen), 1, gen)
    rot = random_rotation(gen)
    o1 = e(_to_dev(dd))
    d2 = hb.Batch(x=dd.x, pos=dd.pos @ rot.T, edge_index=dd.edge_index, batch=dd.batch)
    d2._num_graphs = dd.num_graphs
    o2 = e(_to_dev(_with_edge_attr(d2, 1, gen)))
    assert rel_l2(o2[0], o1[0]) < 1e-5 and rel_l2(o2[1], o1[1]) < 1e-4


def test_oc20_mace_shape_mlip_with_edge_lengths_matches_oracle():
    """C4 shape, MLIP wrapper, edge_dim 1 = the periodic edge lengths: losses and the double-backward parameter gradients."""
    name, g = "oc20_mace", 2
    cpu = add_edges_cpu(make_samples(name, g), name)
    gpu = _gpu_batch(cpu, name, g)
    assert torch.equal(gpu.edge_index.cpu(), cpu.edge_index)
    vec = cpu.pos[cpu.edge_index[1]] - cpu.pos[cpu.edge_index[0]] + cpu.edge_shifts.to(cpu.pos.dtype)
    cpu.edge_attr = vec.norm(dim=1, keepdim=True)
    gpu.edge_attr = cpu.edge_attr.float().to(DEV)
    kw = dict(arch_for(name, cpu), hidden_dim=32, output_dim=[1], output_type=["node"], task_weights=[1.0], loss_function_type="mse",
              output_heads={"node": {"num_headlayers": 2, "dim_headlayers": [32, 16], "type": "mlp"}},
              enable_interatomic_potential=True, energy_weight=1.0, energy_peratom_weight=1.0, force_weight=1.0, edge_dim=1)
    torch.manual_seed(0)
    om = MLIPWrapper(MACEOracle(**{k: v for k, v in kw.items() if k != "mpnn_type"}), 1.0, 1.0, 1.0)
    em = hb.create_model(**kw)
    em.model.load_state_dict(om.model.state_dict())
    om.train()
    em.train()
    cpu.pos.requires_grad_(True)
    gpu.pos.requires_grad_(True)
    lo, to = om.energy_force_loss(om(cpu), cpu)
    le, te = em.energy_force_loss(em(gpu), gpu)
    for a, b in zip(te, to):
        torch.testing.assert_close(a.detach().cpu().double(), b.detach().double(), rtol=1e-4, atol=1e-6)
    lo.backward()
    le.backward()
    assert _grad_rel(em.model, om.model) < 2e-3


# ---- hb.train's padded step carries edge_attr --------------------------------------------------------------------------
def _lengths(loader):
    for b in loader:
        vec = b.pos[b.edge_index[1]] - b.pos[b.edge_index[0]]
        if b.edge_shifts is not None:
            vec = vec + b.edge_shifts.to(vec.dtype)
        b.edge_attr = vec.norm(dim=1, keepdim=True).float()
    return loader


def test_train_fast_path_equals_eager_with_edge_attr_egnn():
    """The padded CUDA-graph step behind hb.train feeds edge_attr (zero rows for its dummy edges) to an EGNN with edge_dim 1;
    before, it dropped the field and trained without the edge features, so its losses left the eager path's."""
    loader = _lengths(_loader("md17_egnn", [5, 3, 7, 5], with_edges=True))
    m1 = hb.get_distributed_model(hb.create_model(**dict(ARCH["md17_egnn"], edge_dim=1)))
    m2 = copy.deepcopy(m1)
    o1, o2 = hb.FlatAdamW(m1, lr=1e-3), hb.FlatAdamW(m2, lr=1e-3)
    for epoch in range(2):
        e_fast, t_fast = hb.train([b.clone() for b in loader], m1, o1, compute_grad_energy=True, fast=True)
        e_eager, t_eager = hb.train([b.clone() for b in loader], m2, o2, compute_grad_energy=True, fast=False)
        torch.testing.assert_close(e_fast, e_eager, rtol=2e-4, atol=1e-6)
        torch.testing.assert_close(t_fast.reshape(-1), t_eager.reshape(-1), rtol=2e-4, atol=1e-6)


def _mace_mlip_kw(edge_dim):
    return dict(ARCH["oc20_mace"], hidden_dim=32, output_dim=[1], output_type=["node"], task_weights=[1.0], loss_function_type="mse",
                output_heads={"node": {"num_headlayers": 2, "dim_headlayers": [32, 16], "type": "mlp"}},
                enable_interatomic_potential=True, energy_weight=1.0, energy_peratom_weight=1.0, force_weight=1.0, edge_dim=edge_dim)


@pytest.mark.parametrize("edge_dim", [0, 1])
def test_train_fast_path_equals_eager_mace_mlip(edge_dim):
    """MACE force training (the route of gfm_mlip.json) through the padded step: every batch brings its own species, so the
    element CSR of the symmetric contraction is rebuilt inside the captured step like the edge plans; with edge_dim 1 the
    edge lengths ride in the [E_cap, 1] buffer and reach EdgeMix / EdgeMixT on the double-backward path."""
    loader = _loader("oc20_mace", [2, 1, 3, 2], with_edges=True)
    if edge_dim:
        loader = _lengths(loader)
    for bt in loader:
        bt.y = None                 # per-node targets of the two-head workload; the MLIP loss reads energy and forces
    m1 = hb.get_distributed_model(hb.create_model(**_mace_mlip_kw(edge_dim)))
    m2 = copy.deepcopy(m1)
    o1, o2 = hb.FlatAdamW(m1, lr=1e-3), hb.FlatAdamW(m2, lr=1e-3)
    for epoch in range(2):
        e_fast, t_fast = hb.train([b.clone() for b in loader], m1, o1, compute_grad_energy=True, fast=True)
        e_eager, t_eager = hb.train([b.clone() for b in loader], m2, o2, compute_grad_energy=True, fast=False)
        torch.testing.assert_close(e_fast, e_eager, rtol=2e-4, atol=1e-6)
        torch.testing.assert_close(t_fast.reshape(-1), t_eager.reshape(-1), rtol=2e-4, atol=1e-6)
    for p, q in zip(m1.parameters(), m2.parameters()):
        torch.testing.assert_close(p, q, rtol=2e-3, atol=2e-6)


def test_graphed_step_refill_with_new_species_equals_eager_mace():
    """GraphedTrainStep.refill with other atomic numbers: the captured MACE step picks the new elements' weights."""
    name, g = "oc20_mace", 2
    base = make_samples(name, g, seed=1).to(DEV)
    base._num_graphs = g
    base = hb.get_radius_graph_pbc(6.0, 128)(base)
    base.y = None
    other_x = base.x.flip(0).contiguous()
    assert not torch.equal(other_x, base.x)
    m1 = hb.get_distributed_model(hb.create_model(**_mace_mlip_kw(0)))
    m2 = copy.deepcopy(m1)
    o1, o2 = hb.FlatAdamW(m1, lr=1e-3), hb.FlatAdamW(m2, lr=1e-3)
    static = base.clone()
    static._num_graphs = g
    gs = hb.GraphedTrainStep(m1, o1, static, compute_grad_energy=True, warmup=2)
    for _ in range(2):
        hb.train_step(m2, o2, base, compute_grad_energy=True)
    other = base.clone()
    other._num_graphs = g
    other.x = other_x
    gs.refill(hb.Batch(x=other_x))
    l_graph = float(gs.run())
    l_eager = float(hb.train_step(m2, o2, other, compute_grad_energy=True)[0])
    assert abs(l_graph - l_eager) <= 1e-5 * abs(l_eager) + 1e-7, (l_graph, l_eager)
