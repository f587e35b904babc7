"""Batched structure relaxation on the device (``hb.PaddedRelaxStep``, ``hgb_fire_step``, capacity-sized periodic builds).

* The FIRE kernel against oracle/relax.py's ``iteration`` on random states: structures of 1 to 5 000 atoms in one batch with a
  frozen structure and filler graphs, both vf branches, n > Nmin, the clamp both ways, every stopping rule; identical
  decisions, x and v within 1e-12 relative, the same bits on a second run, C-ABI refusals that launch nothing.
* ``radius_graph_pbc(..., capacity=)``: the head equals the exact-count build bit for bit, the tail shifts are zero, and an
  undersized candidate or edge capacity sets the guard.
* The step against the oracle's loop driven by the engine's eager ``branch_weighted_energy_forces`` one structure at a time:
  3-branch MACE with graph_attr on periodic cells, EGNN on open molecules, PaiNN and PNAEq; past Nmin so dt and a adapt.
* Captured against uncaptured (the same bits), batch independence, filler atoms that never move, the stopping semantics,
  capacity growth, weight refusals, and parameters and gradients left as they were.
"""
import numpy as np
import pytest
import torch

pytestmark = pytest.mark.gpu

import hydragnn_b200 as hb  # noqa: E402
from hydragnn_b200 import _lib, ops, radius, relax  # noqa: E402
from hydragnn_b200.synthetic import make_samples  # noqa: E402
from oracle import relax as orx  # noqa: E402

DEV = "cuda"


def _p(t):
    return None if t is None else t.data_ptr()


def _stream():
    return torch.cuda.current_stream().cuda_stream


# ---- the FIRE kernel ------------------------------------------------------------------------------------------------------------
SIZES = [1, 2, 31, 32, 33, 1000, 5000, 5000, 40, 7, 3]
# per structure: (k, direction of v relative to f, FIRE's n, force scale, what m_{k-1} makes of the rules, status)
CASES = [(0, 0, 0, 1.0, "keep", 0),          # the first step: v = 0, clamped
         (3, 1, 7, 1e-5, "keep", 0),         # downhill, n > Nmin: dt and a change; no clamp
         (2, -1, 3, 1.0, "keep", 0),         # uphill reset, clamped
         (4, 1, 2, 1.0, "keep", 0),          # downhill, n <= Nmin, clamped
         (5, 1, 6, 1e-5, "keep", 0),         # n = 6 > Nmin, no clamp
         (2, 1, 1, 1.0, "revert", 0),        # m_k > 1.05 m_{k-1}: back to x_{k-1}
         (50, 1, 4, 1.0, "keep", 0),         # k == max_steps
         (3, 1, 9, 1e-5, "keep", 0),         # 5 000 atoms, no clamp
         (2, 1, 0, 1.0, "keep", 2),          # frozen: never touched
         (1, 1, 0, 1e-9, "keep", 0),         # m_1 < fmax: converged
         (1, 1, 0, 1.0, "revert", 0)]        # k = 1: no revert test
FMAX, MAXSTEP, MAX_STEPS = 1e-7, 0.01, 50


def _random_state(seed):
    gen = torch.Generator().manual_seed(seed)
    n = sum(SIZES)
    n_cap, g, g_cap = n + 5, len(SIZES), len(SIZES) + 2
    ptr = torch.tensor([0] + np.cumsum(SIZES).tolist() + [n + 2, n_cap], dtype=torch.int32)
    x = torch.randn(n_cap, 3, generator=gen, dtype=torch.float64) * 3
    f = torch.zeros(n_cap, 3)
    v = torch.zeros(n_cap, 3, dtype=torch.float64)
    fire = torch.zeros(g_cap, 3, dtype=torch.float64)
    ist = torch.zeros(g_cap, 3, dtype=torch.int32)
    for s, (k, sign, nst, scale, rule, status) in enumerate(CASES):
        lo, hi = int(ptr[s]), int(ptr[s + 1])
        fs = (torch.randn(hi - lo, 3, generator=gen) * scale).float()
        f[lo:hi] = fs
        v[lo:hi] = sign * 0.3 * fs.double() + 0.01 * scale * torch.randn(hi - lo, 3, generator=gen, dtype=torch.float64)
        m = float(fs.double().pow(2).sum(1).max().sqrt())
        fire[s] = torch.tensor([0.05 + 0.1 * torch.rand(1, generator=gen, dtype=torch.float64).item(),
                                0.02 + 0.08 * torch.rand(1, generator=gen, dtype=torch.float64).item(),
                                m / 2 if rule == "revert" else m * 10])
        ist[s] = torch.tensor([status, k, nst])
    energy = torch.randn(g_cap, generator=gen)
    x_prev = x + 0.01 * torch.randn(n_cap, 3, generator=gen, dtype=torch.float64)
    return dict(ptr=ptr, x=x, v=v, x_prev=x_prev, fire=fire, ist=ist, f=f, energy=energy, n=n, n_cap=n_cap, g=g, g_cap=g_cap)


def _run_kernel(st, revert=True):
    t = {k: (v.to(DEV).clone() if torch.is_tensor(v) else v) for k, v in st.items()}
    t["e_hist"] = torch.full((MAX_STEPS + 1, st["g_cap"]), float("nan"), dtype=torch.float64, device=DEV)
    t["f_hist"] = torch.full_like(t["e_hist"], float("nan"))
    t["e_out"] = torch.full((st["g_cap"],), -7.0, device=DEV)
    t["f_out"] = torch.full((st["n_cap"], 3), -7.0, device=DEV)
    t["pos"] = torch.full((st["n_cap"], 3), -5.0, device=DEV)
    t["live"] = torch.full((2,), 99, dtype=torch.int32, device=DEV)
    valid = torch.tensor([st["g"], st["n"], 0], dtype=torch.int32, device=DEV)
    guard = torch.zeros(1, dtype=torch.int32, device=DEV)
    before = _lib.launch_count()
    _lib.call("hgb_fire_step", _p(valid), _p(t["ptr"]), st["g_cap"], _p(t["energy"]), _p(t["f"]), _p(t["x"]), _p(t["v"]),
              _p(t["x_prev"]), _p(t["fire"]), _p(t["ist"]), _p(t["e_hist"]), _p(t["f_hist"]), st["g_cap"], _p(t["e_out"]),
              _p(t["f_out"]), _p(t["pos"]), FMAX, MAXSTEP, MAX_STEPS, int(revert), 0.05, _p(guard), _p(t["live"]), _stream())
    assert _lib.launch_count() - before == 1
    torch.cuda.synchronize()
    return {k: (v.cpu() if torch.is_tensor(v) else v) for k, v in t.items()}


def test_fire_kernel_matches_oracle():
    st = _random_state(3)
    out = _run_kernel(st)
    ptr = st["ptr"].tolist()
    running = 0
    seen = set()
    for s, case in enumerate(CASES):
        lo, hi = ptr[s], ptr[s + 1]
        o = orx.State(st["x"][lo:hi].numpy())
        o.x_prev, o.v = st["x_prev"][lo:hi].numpy().copy(), st["v"][lo:hi].numpy().copy()
        o.dt, o.a, o.m_prev = (float(t) for t in st["fire"][s])
        o.status, o.k, o.n = (int(t) for t in st["ist"][s])
        if o.status != orx.RUNNING:                                   # frozen: nothing changes, nothing is written
            assert torch.equal(out["x"][lo:hi], st["x"][lo:hi]) and torch.equal(out["ist"][s], st["ist"][s])
            assert bool((out["pos"][lo:hi] == -5.0).all()) and bool(out["e_hist"][:, s].isnan().all())
            continue
        k0, f = o.k, st["f"][lo:hi].double().numpy()
        if k0 > 0:
            seen.add("up" if float((st["f"][lo:hi].double() * st["v"][lo:hi]).sum()) <= 0 else "down")
        e, m = orx.iteration(o, float(st["energy"][s]), f, fmax=FMAX, maxstep=MAXSTEP, max_steps=MAX_STEPS, max_force_increase=0.05)
        assert int(out["ist"][s, 0]) == o.status and int(out["ist"][s, 1]) == o.k, (s, case)
        assert float(out["f_hist"][k0, s]) == pytest.approx(m, rel=1e-14) and float(out["e_hist"][k0, s]) == e
        assert bool(out["e_hist"][k0 + 1:, s].isnan().all())
        scale = max(float(np.abs(o.x).max()), 1e-300)
        torch.testing.assert_close(out["x"][lo:hi], torch.from_numpy(o.x), rtol=0, atol=1e-12 * scale)
        if o.status in (orx.RUNNING, orx.REVERTED):                  # a structure that stops in place keeps its pos
            assert torch.equal(out["pos"][lo:hi], out["x"][lo:hi].float())
        if o.status == orx.REVERTED:
            assert torch.equal(out["x"][lo:hi], st["x_prev"][lo:hi])
            assert float(out["e_out"][s]) == -7.0 and bool((out["f_out"][lo:hi] == -7.0).all())   # E_{k-1}, F_{k-1} stay
            seen.add("revert")
            continue
        assert float(out["e_out"][s]) == float(st["energy"][s]) and torch.equal(out["f_out"][lo:hi], st["f"][lo:hi])
        if o.status != orx.RUNNING:
            seen.add(o.status)
            continue
        running += 1
        vs = max(float(np.abs(o.v).max()), 1e-300)
        torch.testing.assert_close(out["v"][lo:hi], torch.from_numpy(o.v), rtol=0, atol=1e-12 * vs)
        torch.testing.assert_close(out["x_prev"][lo:hi], st["x"][lo:hi], rtol=0, atol=0)
        assert float(out["fire"][s, 0]) == pytest.approx(o.dt, rel=1e-15) and float(out["fire"][s, 1]) == pytest.approx(o.a, rel=1e-15)
        assert int(out["ist"][s, 2]) == o.n and float(out["fire"][s, 2]) == pytest.approx(m, rel=1e-14)
        dr = np.linalg.norm(o.x - st["x"][lo:hi].numpy())
        seen.add("clamp" if dr > MAXSTEP * (1 - 1e-9) else "free")
        if o.n > 6:
            seen.add("grow")
    assert {"up", "down", "clamp", "free", "grow", "revert", orx.CONVERGED, orx.MAX_STEPS} <= seen, seen
    assert int(out["live"][0]) == running and int(out["live"][1]) == 0
    g, n = st["g"], st["n"]                                           # filler graphs and atoms: never touched
    assert torch.equal(out["x"][n:], st["x"][n:]) and torch.equal(out["v"][n:], st["v"][n:])
    assert bool((out["pos"][n:] == -5.0).all()) and torch.equal(out["ist"][g:], st["ist"][g:])
    again = _run_kernel(st)
    for key in ("x", "v", "x_prev", "fire", "ist", "e_hist", "f_hist", "e_out", "f_out", "pos", "live"):
        assert torch.equal(out[key], again[key]) or (key.endswith("hist") and torch.equal(out[key].nan_to_num(7), again[key].nan_to_num(7)))


def test_fire_kernel_refusals_launch_nothing():
    z = torch.zeros(64, dtype=torch.float64, device=DEV)
    i = torch.zeros(64, dtype=torch.int32, device=DEV)
    f = torch.zeros(64, device=DEV)
    good = [_p(i), _p(i), 2, _p(f), _p(f), _p(z), _p(z), _p(z), _p(z), _p(i), _p(z), _p(z), 2, _p(f), _p(f), _p(f), 0.02, 0.01, 5, 1,
            0.05, _p(i), _p(i)]
    bad = {0: None, 2: 0, 4: None, 5: None, 12: 1, 16: -1.0, 17: 0.0, 18: 0, 19: 2, 21: None, 22: None}
    before = _lib.launch_count()
    for pos, val in bad.items():
        args = list(good)
        args[pos] = val
        with pytest.raises(RuntimeError, match="bad arguments"):
            _lib.call("hgb_fire_step", *args, _stream())
    assert _lib.launch_count() == before


# ---- capacity-sized periodic builds ---------------------------------------------------------------------------------------------
def _cells(g=6, seed=3):
    b = make_samples("gfm_mace", g, seed=seed).to(DEV)
    gptr = b.ptr.to(torch.int32)
    return b.pos, b.cell.double(), b.pbc, torch.full((g,), 5.0, dtype=torch.float64, device=DEV), gptr, g


def test_pbc_capacity_build():
    pos, cell, pbc, cut, gptr, g = _cells()
    ei, cs, sh, deg, outptr, c = radius.radius_graph_pbc(pos, cell, pbc, cut, gptr, g, 20)
    e = ei.shape[1]
    flag = ops.guard_flag(DEV)
    flag.zero_()
    ei2, cs2, sh2, deg2, outptr2, c2 = radius.radius_graph_pbc(pos, cell, pbc, cut, gptr, g, 20, capacity=(c + 77, e + 50))
    assert ei2.shape == (2, e + 50) and sh2.shape == (e + 50, 3) and c2 == c + 77
    assert torch.equal(ei2[:, :e], ei) and torch.equal(cs2[:e], cs) and torch.equal(sh2[:e], sh)
    assert torch.equal(deg2, deg) and torch.equal(outptr2, outptr)
    assert bool((sh2[e:] == 0).all()) and bool((cs2[e:] == 0).all())
    assert int(flag) == 0
    for cap in ((c - 1, e + 50), (c // 3, e + 50), (c + 77, e - 1), (c + 77, 1)):
        radius.radius_graph_pbc(pos, cell, pbc, cut, gptr, g, 20, capacity=cap)
        torch.cuda.synchronize()
        assert int(flag) == ops.GUARD_EDGE_COUNT, cap
        flag.zero_()


# ---- models and batches ---------------------------------------------------------------------------------------------------------
GRAPH = {"num_sharedlayers": 2, "dim_sharedlayers": 5, "num_headlayers": 2, "dim_headlayers": [10, 6]}
MLIP = dict(enable_interatomic_potential=True, energy_weight=1.0, energy_peratom_weight=1.0, force_weight=1.0)


def _model(stack, branches=1, seed=0):
    torch.manual_seed(seed)
    heads = {"graph": [{"type": "branch-%d" % b, "architecture": dict(GRAPH)} for b in range(branches)]}
    kw = dict(output_dim=[1], output_type=["graph"], task_weights=[1.0], output_heads=heads, graph_pooling="add",
              activation_function="relu", loss_function_type="mse", **MLIP)
    if stack == "MACE":
        m = hb.create_model(mpnn_type="MACE", input_dim=1, hidden_dim=8, num_conv_layers=2, num_radial=6, radius=4.0, max_ell=1,
                            node_max_ell=1, avg_num_neighbors=10.0, envelope_exponent=5, correlation=2, max_neighbours=20,
                            use_graph_attr_conditioning=True, graph_attr_conditioning_mode="concat_node", **kw)
        m.model._ensure_graph_concat_projector(graph_attr_dim=2, channel_dim=m.model.hidden_dim, device=m.model.device)
    elif stack == "PNAEq":
        m = hb.create_model(mpnn_type="PNAEq", input_dim=1, hidden_dim=8, num_conv_layers=2, num_radial=5, radius=4.0,
                            pna_deg=[0, 2, 4, 6, 4, 2, 1], **kw)
    else:
        m = hb.create_model(mpnn_type=stack, input_dim=1, hidden_dim=8, num_conv_layers=2, num_radial=5, radius=4.0, **kw)
    return m.to(DEV).eval()


def _structures(periodic, sizes, seed=1):
    gen = torch.Generator().manual_seed(seed)
    out = []
    for i, n in enumerate(sizes):
        box = (n / 0.06) ** (1 / 3)
        d = hb.Batch(x=torch.randint(1, 9, (n, 1), generator=gen).float(), pos=torch.rand(n, 3, generator=gen, dtype=torch.float64) * box,
                     batch=torch.zeros(n, dtype=torch.int64))
        if periodic:
            d.cell = (torch.eye(3, dtype=torch.float64) * box)[None]
            d.pbc = torch.ones(1, 3, dtype=torch.bool)
            d.graph_attr = torch.randn(1, 2, generator=gen)
        d._num_graphs = 1
        out.append(d)
    return out


def _collate(structs):
    n = [s.pos.shape[0] for s in structs]
    b = hb.Batch(x=torch.cat([s.x for s in structs]), pos=torch.cat([s.pos for s in structs]),
                 batch=torch.repeat_interleave(torch.arange(len(n)), torch.tensor(n)))
    if structs[0].cell is not None:
        b.cell, b.pbc = torch.cat([s.cell for s in structs]), torch.cat([s.pbc for s in structs])
        b.graph_attr = torch.cat([s.graph_attr for s in structs])
    b._num_graphs = len(structs)
    return b


def _eager_forces(model, s, w, nb):
    """The engine's eager energy and forces of one structure at fp64 positions x, graph rebuilt with exact counts."""
    r, k = nb

    def forces(x):
        d = hb.Batch(x=s.x.to(DEV), pos=torch.from_numpy(x).float().to(DEV), batch=torch.zeros(x.shape[0], dtype=torch.int64, device=DEV))
        d._num_graphs = 1
        gptr = torch.tensor([0, x.shape[0]], dtype=torch.int32, device=DEV)
        if s.cell is not None:
            d.graph_attr = s.graph_attr.to(DEV)
            d.edge_index, _, d.edge_shifts, _, _, _ = radius.radius_graph_pbc(d.pos, s.cell.to(DEV), s.pbc.to(DEV),
                                                                              torch.full((1,), r, dtype=torch.float64, device=DEV), gptr, 1, k)
        else:
            d.edge_index, _ = radius.radius_graph(d.pos, r, gptr, 1, False, k)
        e, f, _ = hb.branch_weighted_energy_forces(model, d, w)
        return float(e[0]), f.detach().double().cpu().numpy()
    return forces


@pytest.mark.parametrize("stack,periodic,branches", [("MACE", True, 3), ("EGNN", False, 1), ("PAINN", False, 1), ("PNAEq", False, 1)])
def test_matches_oracle_loop(stack, periodic, branches):
    model = _model(stack, branches)
    nb = (4.0, 20)
    structs = _structures(periodic, [9, 14, 6, 11])
    gen = torch.Generator().manual_seed(4)
    w = torch.softmax(torch.randn(len(structs), branches, generator=gen), dim=-1).to(DEV)
    kw = dict(fmax=0.0, maxstep=0.01, max_steps=14, max_force_increase=None)
    step = hb.PaddedRelaxStep(model, _collate(structs), nb, **kw)
    step.load(_collate(structs), w)
    res = step.run()
    off = 0
    for i, s in enumerate(structs):
        n = s.pos.shape[0]
        ref = orx.relax(s.pos.numpy(), _eager_forces(model, s, w[i:i + 1], nb), **kw)
        assert int(res.status[i]) == ref["status"] and int(res.steps[i]) == ref["steps"]
        np.testing.assert_allclose(res.positions[off:off + n].cpu().numpy(), ref["positions"], rtol=0, atol=2e-6)
        np.testing.assert_allclose(res.fmax_history[:, i].cpu().numpy(), ref["fmax_history"], rtol=1e-4, atol=1e-6)
        np.testing.assert_allclose(res.energy_history[:, i].cpu().numpy(), ref["energy_history"], rtol=1e-5, atol=1e-5)
        np.testing.assert_allclose(res.forces[off:off + n].double().cpu().numpy(), ref["forces"], rtol=0,
                                   atol=1e-4 * max(1.0, np.abs(ref["forces"]).max()))
        off += n


def test_captured_equals_uncaptured_and_batch_independence():
    model = _model("MACE", 3)
    nb = (4.0, 20)
    structs = _structures(True, [10, 7, 13], seed=8)
    w = torch.softmax(torch.randn(3, 3, generator=torch.Generator().manual_seed(2)), dim=-1).to(DEV)
    kw = dict(fmax=0.0, max_steps=12)
    runs = []
    for capture in (True, False):
        step = hb.PaddedRelaxStep(model, _collate(structs), nb, capture=capture, **kw)
        step.load(_collate(structs), w)
        runs.append(step.run())
    for a, b in zip(*runs):
        assert torch.equal(a.nan_to_num(7), b.nan_to_num(7))
    n_real = sum(s.pos.shape[0] for s in structs)
    filler = step.data.pos.detach()[n_real:].clone()
    alone = hb.PaddedRelaxStep(model, structs[1], nb, **kw)
    alone.load(structs[1], w[1:2])
    one = alone.run()
    torch.testing.assert_close(one.positions, runs[0].positions[10:17], rtol=0, atol=1e-6)
    torch.testing.assert_close(one.energy, runs[0].energy[1:2], rtol=1e-5, atol=1e-5)
    assert torch.equal(step.data.pos.detach()[n_real:], filler)
    step.load(_collate(structs), w)                                   # a rerun: filler atoms where the staging put them
    step.run()
    assert torch.equal(step.data.pos.detach()[n_real:], filler)
    assert float(filler[1, 0] - filler[0, 0]) == 1.5


def test_stopping_semantics_and_side_effects():
    model = _model("EGNN")
    nb = (4.0, 20)
    structs = _structures(False, [8, 12, 5], seed=5)
    b = _collate(structs)
    for p in model.parameters():
        p.grad = torch.randn_like(p)
    before = [(p.detach().clone(), p.grad.clone()) for p in model.parameters()]

    def run(**kw):
        step = hb.PaddedRelaxStep(model, b, nb, **kw)
        step.load(b)
        return step.run()
    r = run(fmax=1e9)
    assert r.status.tolist() == [relax.CONVERGED] * 3 and r.steps.tolist() == [1] * 3
    assert not bool(r.fmax_history[:2].isnan().any()) and bool(r.fmax_history[2:].isnan().all())
    one = run(fmax=0.0, max_steps=1)
    assert one.status.tolist() == [relax.MAX_STEPS] * 3
    rev = run(fmax=0.0, max_force_increase=-1.0)
    assert rev.status.tolist() == [relax.REVERTED] * 3 and rev.steps.tolist() == [2] * 3
    assert torch.equal(rev.positions, one.positions) and torch.equal(rev.forces, one.forces) and torch.equal(rev.energy, one.energy)
    full = run(fmax=0.0, max_steps=17, max_force_increase=None)
    assert full.status.tolist() == [relax.MAX_STEPS] * 3 and full.steps.tolist() == [17] * 3
    assert not bool(full.fmax_history.isnan().any())
    assert not model.training
    for p, (v, g) in zip(model.parameters(), before):
        assert torch.equal(p.detach(), v) and torch.equal(p.grad, g)


def test_capacity_growth_recaptures_and_matches():
    model = _model("MACE", 3)
    nb = (4.0, 20)
    structs = _structures(True, [12, 9, 15], seed=11)
    b = _collate(structs)
    w = torch.full((3, 3), 1 / 3, device=DEV)
    kw = dict(fmax=0.0, max_steps=20)
    ample = hb.PaddedRelaxStep(model, b, nb, **kw)
    ample.load(b, w)
    ref = ample.run()
    assert ample.recaptures == 0
    tail = ample.data.edge_index[:, -1]
    assert int(tail.min()) >= sum(s.pos.shape[0] for s in structs)      # the tail holds dummy edges between filler atoms
    tiny = hb.PaddedRelaxStep(model, b, nb, candidate_cap=64, edge_cap=64, **kw)
    tiny.load(b, w)
    got = tiny.run()
    assert tiny.recaptures >= 1 and ample.e_cap > 64 and ample.cand_cap > 64
    for a, c in zip(ref, got):
        assert torch.equal(a.nan_to_num(7), c.nan_to_num(7))


def test_weight_refusals():
    model = _model("MACE", 3)
    structs = _structures(True, [6, 8])
    b = _collate(structs)
    step = hb.PaddedRelaxStep(model, b, (4.0, 20))
    before = _lib.launch_count()
    for w in (torch.full((2, 2), 0.5, device=DEV), torch.full((3, 3), 0.5, device=DEV), torch.full((2, 3), 0.5, device=DEV).double(),
              torch.full((2, 3), 0.5), None):
        with pytest.raises(ValueError, match="weights must be"):
            step.load(b, w)
    assert _lib.launch_count() == before
