"""GPU tests of MACE's distance transforms (Agnesi / Soft; radial.py:151-245, blocks.py:141-177).

* Kernels against fp64: hgb_mace_dist_transform (T, T', T'') and the fused hgb_mace_edge_embed_dt_fwd / _dt_bwd (sh, radial and
  d/dpos), over both kinds, d from 0 through 1e-30 to beyond r_max, every species 1..118 and clamped indices, periodic shifts
  and the padded step's filler atoms (H, 1.5 A apart).  The fp64 reference is the reference's own formula
  (oracle.mace_transform.transform_of_length) differentiated by autograd.
* Models against the golden of the reference's own code (tests/golden/models_mace_transform.pt): the first-order path and the
  MLIP energy / forces / force-loss gradients on the any-order path.  Outputs within rel-L2 1e-5, gradients within 1e-3.
* The transform's buffers are read on the device: a state dict loaded with other radii or another ``a`` reaches the eager
  path and a replayed GraphedTrainStep.
* hb.train's padded captured step against the eager path, and the GFM MACE architecture with "Agnesi" from
  create_model_config against the oracle."""
import copy
import types

import pytest
import torch

pytestmark = pytest.mark.gpu

import hydragnn_b200 as hb  # noqa: E402
from hydragnn_b200 import _lib, e3, ops  # noqa: E402
from hydragnn_b200.covalent_radii import covalent_radii_tensor  # noqa: E402
from hydragnn_b200.synthetic import ARCH, make_samples  # noqa: E402
from oracle.mace_transform import MACETransformOracle, transform_of_length  # noqa: E402
from oracle.mlip import MLIPWrapper  # noqa: E402
from oracle.workloads import add_edges_cpu  # noqa: E402
from mace_transform_support import load_golden  # noqa: E402
from stack_support import MACE_KW, _gpu_batch, _grad_rel, _loader  # noqa: E402

DEV = "cuda"
KINDS = ["Agnesi", "Soft"]
PARAMS = {"Agnesi": (0.9183, 4.5791, 1.0805), "Soft": (0.2, 3.0)}


def rel_l2(a, b):
    return float((a.detach().double().cpu() - b.detach().double().cpu()).norm() / b.detach().double().cpu().norm().clamp(min=1e-30))


def _dt(kind, z, params=None, radii=None):
    """Device operands (kind, z, radii, c0, c1, c2) as MACEStack.distance_transform_operands builds them."""
    params = PARAMS[kind] if params is None else params
    c = [torch.tensor(v, dtype=torch.float32, device=DEV) for v in params]
    radii = (covalent_radii_tensor() if radii is None else radii).to(DEV)
    return (ops.DIST_TRANSFORMS[kind], z.to(DEV), radii, c[0], c[1], c[2] if kind == "Agnesi" else None)


def _ref_t(kind, d, rsum, params=None):
    """fp64 T, T', T'' of the reference's formula by autograd; the d -> 0 limit of Agnesi (T = 1, T' = T'' = 0) where its
    u^(q-p) is infinite even in fp64."""
    params = [torch.tensor(v, dtype=torch.float32).double() for v in (PARAMS[kind] if params is None else params)]
    d = d.double().clone().requires_grad_(True)
    t = transform_of_length(kind, d, rsum.double(), params)
    t1, = torch.autograd.grad(t.sum(), d, create_graph=True)
    t2, = torch.autograd.grad(t1.sum(), d)
    out = [t.detach(), t1.detach(), t2.detach()]
    if kind == "Agnesi":
        zero = d.detach() == 0
        out = [torch.where(zero, torch.full_like(v, 1.0 if k == 0 else 0.0), v) for k, v in enumerate(out)]
    return out


def _close(k, r, rtol, scale_atol):
    """|k - r| <= rtol |r| + scale_atol max|r| per element, all finite."""
    k, r = k.detach().double().cpu(), r.double()
    assert torch.isfinite(k).all()
    bound = rtol * r.abs() + scale_atol * float(r.abs().max())
    worst = float(((k - r).abs() / bound.clamp(min=1e-300)).max())
    assert worst <= 1.0, worst


def _lengths_and_pairs(gen):
    """Edge lengths over the whole range the transform meets, each with a random pair of element indices 0..117 plus indices
    below and above that range (clamped by the kernel as process_node_attributes clamps Z)."""
    d = torch.cat([torch.zeros(4), torch.logspace(-30, -1, 60), torch.linspace(0.05, 12.0, 2000), torch.tensor([5.0, 6.0, 6.0001, 40.0, 1e3]),
                   torch.rand(4000, generator=gen) * 8.0]).float()
    e = d.numel()
    z = torch.cat([torch.arange(118), torch.tensor([-3, 130, 117, 0, 96, 97, 5, 25])])           # per-node indices
    row = torch.randint(0, z.numel(), (e,), generator=gen)
    col = torch.randint(0, z.numel(), (e,), generator=gen)
    row[:z.numel()] = torch.arange(z.numel())                                                     # every species appears
    return d, z, row.int(), col.int()


def _rsum(z, row, col, radii=None):
    r = (covalent_radii_tensor() if radii is None else radii).double()
    zc = z.clamp(0, 117) + 1
    return r[zc[row.long()]] + r[zc[col.long()]]


@pytest.mark.parametrize("kind", KINDS)
def test_dist_transform_kernel_matches_fp64(kind):
    gen = torch.Generator().manual_seed(7 + len(kind))
    d, z, row, col = _lengths_and_pairs(gen)
    plan = types.SimpleNamespace(row=row.to(DEV), col=col.to(DEV), num_edges=d.numel())
    dt = _dt(kind, z)
    refs = _ref_t(kind, d, _rsum(z, row, col))
    g = torch.randn(d.numel(), generator=gen)
    for order, ref in enumerate(refs):
        out = ops._dist_transform_call(order, d.to(DEV), None, plan, dt)
        _close(out, ref, 2e-5 if order < 2 else 1e-4, 1e-6)
        outg = ops._dist_transform_call(order, d.to(DEV), g.to(DEV), plan, dt)
        _close(outg, ref * g.double(), 2e-5 if order < 2 else 1e-4, 1e-6)
        again = ops._dist_transform_call(order, d.to(DEV), None, plan, dt)
        assert torch.equal(out, again)
    if kind == "Agnesi":                                  # d -> 0: T -> 1 and T' -> 0, never NaN
        t0 = ops._dist_transform_call(0, d[:4].to(DEV), None, types.SimpleNamespace(row=row[:4].to(DEV), col=col[:4].to(DEV), num_edges=4), dt)
        assert torch.equal(t0.cpu(), torch.ones(4))


@pytest.mark.parametrize("kind", KINDS)
def test_dist_transform_autograd_pair_and_third_derivative_refused(kind):
    gen = torch.Generator().manual_seed(3)
    d, z, row, col = _lengths_and_pairs(gen)
    plan = types.SimpleNamespace(row=row.to(DEV), col=col.to(DEV), num_edges=d.numel())
    dt = _dt(kind, z)
    t_ref, t1_ref, t2_ref = _ref_t(kind, d, _rsum(z, row, col))
    w = torch.randn(d.numel(), generator=gen)
    dd = d.to(DEV).requires_grad_(True)
    t = ops.DistTransformFn.apply(dd, plan, dt)
    _close(t, t_ref, 2e-5, 1e-6)
    g1, = torch.autograd.grad((t * w.to(DEV)).sum(), dd, create_graph=True)
    _close(g1, t1_ref * w.double(), 2e-5, 1e-6)
    g2, = torch.autograd.grad(g1.sum(), dd, create_graph=True)
    _close(g2, t2_ref * w.double(), 1e-4, 1e-6)
    with pytest.raises(RuntimeError, match="third derivative"):
        torch.autograd.grad(g2.sum(), dd)
    # no edges: nothing runs
    empty = types.SimpleNamespace(row=row[:0].to(DEV), col=col[:0].to(DEV), num_edges=0)
    assert ops.DistTransformFn.apply(torch.zeros(0, device=DEV), empty, dt).numel() == 0


def _geometry(kind_seed, with_shifts):
    """Positions and edges: random pairs, coincident-ish and far pairs, an edge of exactly r_max, one past it, and the filler
    chain of the padded step (H atoms 1.5 A apart on a line)."""
    gen = torch.Generator().manual_seed(kind_seed)
    n = 400
    pos = torch.rand(n, 3, generator=gen, dtype=torch.float64) * 6.0
    pos[-8:] = 0.0
    pos[-8:, 0] = 1.5 * torch.arange(8, dtype=torch.float64)            # filler atoms, off the atoms placed below
    pos[-8:, 1] = 7.0
    pos[0] = torch.tensor([0.0, 0.0, 0.0], dtype=torch.float64)
    pos[1] = torch.tensor([5.0, 0.0, 0.0], dtype=torch.float64)         # |vec| = r_max exactly
    pos[2] = torch.tensor([0.0, 5.25, 0.0], dtype=torch.float64)        # beyond r_max
    pos[3] = torch.tensor([0.0, 0.0, 0.05], dtype=torch.float64)        # a very short edge
    z = torch.randint(-2, 120, (n,), generator=gen)
    z[-8:] = 0                                                          # H
    e = 6000
    row = torch.randint(0, n, (e,), generator=gen)
    col = torch.randint(0, n, (e,), generator=gen)
    keep = row != col
    row, col = row[keep], col[keep]
    fill = torch.arange(n - 8, n - 1)
    row = torch.cat([torch.tensor([0, 0, 0, 1]), fill, fill + 1, row])
    col = torch.cat([torch.tensor([1, 2, 3, 0]), fill + 1, fill, col])
    shifts = None
    if with_shifts:
        shifts = torch.randint(-1, 2, (row.numel(), 3), generator=gen).double() * 2.0
        shifts[: 4 + 2 * fill.numel()] = 0.0
    return pos, z, row.int(), col.int(), shifts


def _edge_vec(pos, row, col, shifts):
    vec = pos[col.long()] - pos[row.long()]
    return vec if shifts is None else vec + shifts


def _ref_embed(kind, vec, z, row, col, lmax, nb, rc, p):
    """fp64 sh and Bessel(T(d)) x cutoff(d) of edge vectors vec [E, 3] (blocks.py:164-177)."""
    d = vec.norm(dim=1, keepdim=True)
    sh = e3.spherical_harmonics_cl(lmax, vec / d)
    x = d / rc
    env = 1.0 - ((p + 1.0) * (p + 2.0) / 2.0) * x.pow(p) + p * (p + 2.0) * x.pow(p + 1) - (p * (p + 1.0) / 2) * x.pow(p + 2)
    cutoff = env * (d < rc)
    params = [torch.tensor(v, dtype=torch.float32).double() for v in PARAMS[kind]]
    t = transform_of_length(kind, d, _rsum(z, row, col)[:, None], params)
    w = torch.pi / rc * torch.arange(1, nb + 1, dtype=torch.float64)
    radial = (2.0 / rc) ** 0.5 * torch.sin(w * t) / t * cutoff
    return sh, radial


@pytest.mark.parametrize("with_shifts", [False, True])
@pytest.mark.parametrize("lmax", [0, 1, 2, 3])
@pytest.mark.parametrize("kind", KINDS)
def test_fused_edge_embed_dt_kernels_match_fp64(kind, lmax, with_shifts):
    """hgb_mace_edge_embed_dt_fwd / _dt_bwd called directly: sh, radial and the per-edge g_vec = d L / d vec."""
    nb, rc, p = 8, 5.0, 5.0
    pos, z, row, col, shifts = _geometry(lmax + 10 * len(kind), with_shifts)
    e = row.numel()
    vec = _edge_vec(pos, row, col, shifts).float().double().requires_grad_(True)
    sh_ref, rad_ref = _ref_embed(kind, vec, z, row, col, lmax, nb, rc, p)
    gen = torch.Generator().manual_seed(lmax)
    gs = torch.randn(sh_ref.shape, generator=gen, dtype=torch.float64)
    gr = torch.randn(rad_ref.shape, generator=gen, dtype=torch.float64)
    gvec_ref, = torch.autograd.grad((sh_ref * gs).sum() + (rad_ref * gr).sum(), vec)
    pg, rowd, cold = pos.float().to(DEV), row.to(DEV), col.to(DEV)
    sdev = None if shifts is None else shifts.float().to(DEV)
    dt = _dt(kind, z)                                                   # kept alive: the kernels read its device memory
    kd, zp, rp, c0, c1, c2 = ops._dt_ptrs(dt)
    sh = torch.empty(e, (lmax + 1) ** 2, device=DEV)
    radial = torch.empty(e, nb, device=DEV)
    _lib.call("hgb_mace_edge_embed_dt_fwd", ops._p(pg), ops._p(rowd), ops._p(cold), ops._p(sdev), zp, e, lmax, nb, rc, p, kd, rp, c0, c1,
              c2, ops._p(sh), ops._p(radial), ops._stream())
    assert rel_l2(sh, sh_ref) < 1e-5 and rel_l2(radial, rad_ref) < 1e-5, (rel_l2(sh, sh_ref), rel_l2(radial, rad_ref))
    _close(radial, rad_ref.detach(), 1e-4, 1e-5)
    assert float(radial[[0, 1, 3]].abs().max()) == 0.0                 # d = r_max and beyond: the cutoff is zero
    gsd, grd = gs.float().to(DEV), gr.float().to(DEV)
    gvec = torch.empty(e, 3, device=DEV)
    for g_sh, g_rad, ref in [(gsd, grd, gvec_ref), (None, grd, None), (gsd, None, None)]:
        _lib.call("hgb_mace_edge_embed_dt_bwd", ops._p(pg), ops._p(rowd), ops._p(cold), ops._p(sdev), zp, ops._p(g_sh), ops._p(g_rad), e,
                  lmax, nb, rc, p, kd, rp, c0, c1, c2, ops._p(gvec), ops._stream())
        assert torch.isfinite(gvec).all()
        if ref is not None:
            assert rel_l2(gvec, ref) < 1e-4, rel_l2(gvec, ref)
    # the radial part alone, against the radial part of the reference
    _lib.call("hgb_mace_edge_embed_dt_bwd", ops._p(pg), ops._p(rowd), ops._p(cold), ops._p(sdev), zp, None, ops._p(grd), e, lmax, nb, rc, p,
              kd, rp, c0, c1, c2, ops._p(gvec), ops._stream())
    vec2 = vec.detach().clone().requires_grad_(True)
    g_rad_ref, = torch.autograd.grad((_ref_embed(kind, vec2, z, row, col, lmax, nb, rc, p)[1] * gr).sum(), vec2)
    assert rel_l2(gvec, g_rad_ref) < 1e-4, rel_l2(gvec, g_rad_ref)
    assert float(gvec[[0, 1, 3]].abs().max()) == 0.0                   # at and beyond r_max no 0 * inf: exactly zero


@pytest.mark.parametrize("kind", KINDS)
def test_fused_dt_function_forces_match_fp64(kind):
    """MaceEdgeEmbedDtFn end to end (kernel + scatter to positions) with periodic shifts."""
    nb, rc, p, lmax = 8, 5.0, 5.0, 2
    pos, z, row, col, shifts = _geometry(99, True)
    plan = ops.EdgePlan(torch.stack([row.long(), col.long()]).to(DEV), pos.shape[0])
    posd = pos.float().double().requires_grad_(True)
    sh_ref, rad_ref = _ref_embed(kind, _edge_vec(posd, row, col, shifts), z, row, col, lmax, nb, rc, p)
    pg = pos.float().to(DEV).requires_grad_(True)
    sh, radial = ops.MaceEdgeEmbedDtFn.apply(pg, shifts.float().to(DEV), plan, _dt(kind, z), lmax, nb, rc, p)
    assert rel_l2(sh, sh_ref) < 1e-5 and rel_l2(radial, rad_ref) < 1e-5
    gen = torch.Generator().manual_seed(1)
    gs, gr = torch.randn(sh_ref.shape, generator=gen, dtype=torch.float64), torch.randn(rad_ref.shape, generator=gen, dtype=torch.float64)
    f_ref, = torch.autograd.grad((sh_ref * gs).sum() + (rad_ref * gr).sum(), posd)
    f, = torch.autograd.grad((sh * gs.float().to(DEV)).sum() + (radial * gr.float().to(DEV)).sum(), pg)
    assert rel_l2(f, f_ref) < 1e-4, rel_l2(f, f_ref)


# ---- models against the reference's own code --------------------------------------------------------------------------------
def _golden(golden_dir):
    return load_golden(golden_dir)


def _dev_batch(inputs):
    d = hb.Batch(**{k: v.clone().to(DEV) for k, v in inputs.items()})
    d._num_graphs = 3
    d.pos.requires_grad_(True)
    return d


FIRST_ORDER = ["agnesi_bessel", "soft_bessel", "soft_chebyshev"]
MLIP = ["agnesi_gaussian_mlip", "soft_gaussian_mlip"]


@pytest.mark.parametrize("name", FIRST_ORDER)
def test_engine_first_order_matches_the_reference_own_code_golden(golden_dir, name):
    c = _golden(golden_dir)[name]
    e = hb.create_model(mpnn_type="MACE", **dict(MACE_KW, **c["cfg"]))
    e.load_state_dict(c["state"], strict=True)
    e.eval()
    d = _dev_batch(c["inputs"])
    _lib.trace_begin()
    pred = e(d)
    calls = {n for n, _, _ in _lib.trace_end()}
    fused = c["cfg"]["radial_type"] == "bessel"
    assert ("hgb_mace_edge_embed_dt_fwd" in calls) == fused and ("hgb_mace_dist_transform" in calls) != fused
    assert "hgb_mace_edge_embed_fwd" not in calls
    for p, q in zip(pred, c["pred"]):
        assert rel_l2(p, q) < 1e-5, (name, rel_l2(p, q))
    obj = pred[0].sum() + pred[1].pow(2).sum()
    f, = torch.autograd.grad(obj, d.pos, retain_graph=True)
    assert rel_l2(f, c["dobj_dpos"]) < 1e-3, rel_l2(f, c["dobj_dpos"])
    obj.backward()
    for n, prm in e.named_parameters():
        ref = c["grads"][n]
        if ref is None or float(ref.abs().max()) == 0:
            continue
        assert rel_l2(prm.grad, ref) < 1e-3, (name, n, rel_l2(prm.grad, ref))


@pytest.mark.parametrize("name", MLIP)
def test_engine_mlip_matches_the_reference_own_code_golden(golden_dir, name):
    """Energy, forces and the force loss's parameter gradients through DistTransformFn / DistTransformGradFn."""
    c = _golden(golden_dir)[name]
    e = hb.create_model(mpnn_type="MACE", **dict(MACE_KW, **c["cfg"], enable_interatomic_potential=True, energy_weight=1.0,
                                                 energy_peratom_weight=1.0, force_weight=1.0))
    e.model.load_state_dict(c["state"], strict=True)
    e.train()
    d = _dev_batch(c["inputs"])
    pred = e(d)
    assert rel_l2(pred[0], c["pred"][0]) < 1e-5
    f = -torch.autograd.grad(pred[0].sum(), d.pos, retain_graph=True, create_graph=True)[0]
    assert rel_l2(f, c["forces"]) < 1e-4, rel_l2(f, c["forces"])
    tot, tasks = e.energy_force_loss(pred, d)
    assert abs(float(tot) - float(c["loss"])) <= 1e-5 * abs(float(c["loss"]))
    for a, b in zip(tasks, c["tasks"]):
        assert abs(float(a) - float(b)) <= 1e-5 * max(abs(float(b)), 1e-6)
    tot.backward()
    for n, prm in e.model.named_parameters():
        ref = c["grads"][n]
        if ref is None or float(ref.abs().max()) == 0:
            continue
        assert rel_l2(prm.grad, ref) < 1e-3, (name, n, rel_l2(prm.grad, ref))


# ---- the buffers are read on the device ---------------------------------------------------------------------------------------
def _altered(state, which):
    s = {k: v.clone() for k, v in state.items()}
    if which == "covalent_radii":
        s["radial_embedding.distance_transform.covalent_radii"] *= 3.0
    else:
        s["radial_embedding.distance_transform.a"] += 1.0
    return s


@pytest.mark.parametrize("which", ["covalent_radii", "a"])
@pytest.mark.parametrize("name", ["agnesi_bessel", "soft_bessel"])
def test_loaded_buffers_reach_the_eager_path(golden_dir, name, which):
    """After load_state_dict with other radii or another ``a`` the engine follows the oracle with the same state; the change of
    the node outputs is many times the engine's distance from the oracle, so the check tells the two states apart."""
    c = _golden(golden_dir)[name]
    kw = dict(MACE_KW, **c["cfg"])
    e = hb.create_model(mpnn_type="MACE", **kw)
    e.load_state_dict(c["state"], strict=True)
    e.eval()
    before = e(_dev_batch(c["inputs"]))[-1].detach()
    state = _altered(c["state"], which)
    e.load_state_dict(state, strict=True)
    o = MACETransformOracle(**kw)
    o.load_state_dict(state, strict=True)
    ref = o.double()(_cpu_batch(c["inputs"]))
    after = e(_dev_batch(c["inputs"]))
    for p, q in zip(after, ref):
        assert rel_l2(p, q) < 1e-5, rel_l2(p, q)
    assert rel_l2(after[-1], before) > 10 * rel_l2(after[-1], ref[-1]), (rel_l2(after[-1], before), rel_l2(after[-1], ref[-1]))


def _cpu_batch(inputs):
    d = hb.Batch(**{k: (v.clone().double() if v.is_floating_point() else v.clone()) for k, v in inputs.items()})
    d._num_graphs = 3
    return d


def _mlip_kw(kind, radial="bessel"):
    return dict(ARCH["oc20_mace"], hidden_dim=32, output_dim=[1], output_type=["node"], task_weights=[1.0], loss_function_type="mse",
                output_heads={"node": {"num_headlayers": 2, "dim_headlayers": [32, 16], "type": "mlp"}},
                enable_interatomic_potential=True, energy_weight=1.0, energy_peratom_weight=1.0, force_weight=1.0,
                distance_transform=kind, radial_type=radial)


@pytest.mark.parametrize("mlip", [False, True])
@pytest.mark.parametrize("which", ["covalent_radii", "a"])
def test_loaded_buffers_reach_a_replayed_graphed_step(which, mlip):
    """Capture, then load a state dict with other transform buffers into the captured model: the replay follows it exactly as
    the eager step of a twin that loaded the same state.  First order: the fused kernels; MLIP: the any-order path."""
    name, g = "oc20_mace", 2
    base = make_samples(name, g, seed=1).to(DEV)
    base._num_graphs = g
    base = hb.get_radius_graph_pbc(6.0, 128)(base)
    if mlip:
        base.y = None
        kw = _mlip_kw("Agnesi")
    else:
        kw = dict(ARCH["oc20_mace"], hidden_dim=32, distance_transform="Agnesi")
    m1 = hb.get_distributed_model(hb.create_model(**kw))
    m2, m3 = copy.deepcopy(m1), copy.deepcopy(m1)
    o1, o2, o3 = (hb.FlatAdamW(m, lr=1e-3) for m in (m1, m2, m3))
    static = base.clone()
    static._num_graphs = g
    gs = hb.GraphedTrainStep(m1, o1, static, compute_grad_energy=mlip, warmup=2)
    for _ in range(2):
        hb.train_step(m2, o2, base, compute_grad_energy=mlip)
        hb.train_step(m3, o3, base, compute_grad_energy=mlip)
    inner = lambda m: m.module.model if mlip else m.module                                    # noqa: E731
    state = _altered(inner(m1).state_dict(), which)
    inner(m1).load_state_dict(state)
    inner(m2).load_state_dict(_altered(inner(m2).state_dict(), which))
    l_graph = float(gs.run())
    l_eager = float(hb.train_step(m2, o2, base, compute_grad_energy=mlip)[0])
    l_unaltered = float(hb.train_step(m3, o3, base, compute_grad_energy=mlip)[0])
    assert abs(l_graph - l_eager) <= 1e-5 * abs(l_eager) + 1e-7, (l_graph, l_eager)
    assert abs(l_eager - l_unaltered) > 1e-6 * abs(l_unaltered), (l_eager, l_unaltered)


# ---- hb.train: the padded captured step ---------------------------------------------------------------------------------------
@pytest.mark.parametrize("kind,radial", [("Agnesi", "bessel"), ("Soft", "gaussian")])
def test_train_fast_path_equals_eager_mace_mlip_with_transform(kind, radial):
    """Filler atoms of the padded step are H atoms 1.5 A apart: their edges go through the transform too, and must not change
    the real graphs' losses."""
    loader = _loader("oc20_mace", [2, 1, 3, 2], with_edges=True)
    for bt in loader:
        bt.y = None
    m1 = hb.get_distributed_model(hb.create_model(**_mlip_kw(kind, radial)))
    m2 = copy.deepcopy(m1)
    o1, o2 = hb.FlatAdamW(m1, lr=1e-3), hb.FlatAdamW(m2, lr=1e-3)
    for epoch in range(2):
        e_fast, t_fast = hb.train([b.clone() for b in loader], m1, o1, compute_grad_energy=True, fast=True)
        e_eager, t_eager = hb.train([b.clone() for b in loader], m2, o2, compute_grad_energy=True, fast=False)
        assert torch.isfinite(torch.as_tensor(e_fast)).all()
        torch.testing.assert_close(e_fast, e_eager, rtol=2e-4, atol=1e-6)
        torch.testing.assert_close(t_fast.reshape(-1), t_eager.reshape(-1), rtol=2e-4, atol=1e-6)


# ---- drop-in: the GFM MACE search space's draw ----------------------------------------------------------------------------------
def test_gfm_mace_config_with_agnesi_trains_and_matches_oracle():
    """create_model_config with the GFM MACE architecture (MLIP, add pooling, edge lengths as edge_dim 1, concat_node conditioning)
    plus distance_transform "Agnesi": the force-training losses and double-backward gradients against the fp64 oracle, then
    training steps."""
    name, g = "gfm_mace", 2
    cpu = add_edges_cpu(make_samples(name, g), name)
    gpu = _gpu_batch(cpu, name, g)
    assert torch.equal(gpu.edge_index.cpu(), cpu.edge_index)
    vec = cpu.pos[cpu.edge_index[1]] - cpu.pos[cpu.edge_index[0]] + cpu.edge_shifts.to(cpu.pos.dtype)
    cpu.edge_attr = vec.norm(dim=1, keepdim=True)
    gpu.edge_attr = cpu.edge_attr.float().to(DEV)
    gen = torch.Generator().manual_seed(2)
    cpu.graph_attr = torch.randn(g, 2, generator=gen, dtype=torch.float64)
    gpu.graph_attr = cpu.graph_attr.float().to(DEV)
    arch = dict(ARCH["gfm_mace"], distance_transform="Agnesi")
    loss_type = arch.pop("loss_function_type")
    torch.manual_seed(0)
    em = hb.create_model_config({"Architecture": arch, "Training": {"loss_function_type": loss_type}})
    assert em.model.distance_transform == "Agnesi"
    inner = {k: v for k, v in arch.items() if k not in ("mpnn_type", "enable_interatomic_potential", "energy_weight",
                                                         "energy_peratom_weight", "force_weight")}
    om = MLIPWrapper(MACETransformOracle(**inner, loss_function_type=loss_type), 0.0, 1.0, 10.0)
    torch.manual_seed(7)
    om.model._ensure_graph_concat_projector(2, 128, torch.device("cpu"))
    em.model._ensure_graph_concat_projector(graph_attr_dim=2, channel_dim=128, device=em.model.device)
    em.model.load_state_dict(om.model.state_dict(), strict=True)
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
    assert _grad_rel(em.model, om.model) < 1e-3
    model = hb.get_distributed_model(em)
    opt = hb.FlatAdamW(model, lr=1e-3)
    gpu.pos = gpu.pos.detach()
    losses = [float(hb.train_step(model, opt, gpu, compute_grad_energy=True)[0]) for _ in range(3)]
    assert all(torch.isfinite(torch.tensor(losses)))
