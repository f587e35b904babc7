"""Structure relaxation, host side (no GPU): oracle/relax.py and the refusals of ``hb.PaddedRelaxStep``.

* Single FIRE steps against hand-computed values: the first step, the mixing branch, the uphill reset, dt growth only after
  n > Nmin and its cap at dtmax, and the maxstep clamp over the whole structure.
* The loop's rules on scripted forces: no revert test at step 1, a revert restores x_{k-1} with its energy and forces, the
  threshold is compared strictly, converged and max-steps statuses; driving ``iteration`` (the kernel's cut) gives ``relax``.
* On a harmonic well and on an LJ dimer and trimer the loop converges to the analytic minimum within fmax over the curvature.
* ``PaddedRelaxStep`` refuses what it cannot relax before any launch.
"""
import math

import numpy as np
import pytest
import torch

import hydragnn_b200 as hb
from hydragnn_b200.data import Batch
from oracle import relax as orx

F2 = np.array([[3.0, 0.0, 0.0], [0.0, 4.0, 0.0]])             # |f| = 5


def _fire(v=None, dt=0.1, a=0.1, n=0, maxstep=1.0):
    opt = orx.Fire(maxstep=maxstep)
    opt.v = None if v is None else np.array(v, dtype=np.float64)
    opt.dt, opt.a, opt.Nsteps = dt, a, n
    return opt


def test_first_step():
    opt = _fire()
    x = opt.step(np.zeros((2, 3)), F2)
    np.testing.assert_allclose(opt.v, 0.1 * F2, rtol=0, atol=1e-15)
    np.testing.assert_allclose(x, 0.01 * F2, rtol=0, atol=1e-15)          # dr = dt (dt f)
    assert (opt.dt, opt.a, opt.Nsteps) == (0.1, 0.1, 0)


def test_mixing_branch():
    opt = _fire(v=[[1.0, 0.0, 0.0], [0.0, 0.0, 0.0]])                       # <f, v> = 3 > 0, |v| = 1
    x = opt.step(np.zeros((2, 3)), F2)
    # v = 0.9 v + 0.1 f / 5 * 1 = [[0.96, 0, 0], [0, 0.08, 0]]; v += 0.1 f
    np.testing.assert_allclose(opt.v, [[1.26, 0, 0], [0, 0.48, 0]], rtol=0, atol=1e-15)
    np.testing.assert_allclose(x, [[0.126, 0, 0], [0, 0.048, 0]], rtol=0, atol=1e-15)
    assert (opt.dt, opt.a, opt.Nsteps) == (0.1, 0.1, 1)                    # n = 0 is not > Nmin: dt and a stay


def test_uphill_reset():
    opt = _fire(v=[[1.0, 0.0, 0.0], [0.0, 0.0, 0.0]], dt=0.2, a=0.05, n=9)
    f = np.array([[-3.0, 0.0, 0.0], [0.0, 4.0, 0.0]])                      # <f, v> = -3
    x = opt.step(np.ones((2, 3)), f)
    assert (opt.dt, opt.a, opt.Nsteps) == (0.1, 0.1, 0)
    np.testing.assert_allclose(opt.v, 0.1 * f, rtol=0, atol=1e-15)        # v = 0, then v += dt f
    np.testing.assert_allclose(x, 1.0 + 0.01 * f, rtol=0, atol=1e-15)


def test_dt_grows_only_after_nmin_and_caps_at_dtmax():
    v = [[1.0, 0.0, 0.0], [0.0, 0.0, 0.0]]
    opt = _fire(v=v, n=5)
    opt.step(np.zeros((2, 3)), F2)
    assert (opt.dt, opt.a, opt.Nsteps) == (0.1, 0.1, 6)                    # n = 5 is not > 5
    opt = _fire(v=v, n=6)
    opt.step(np.zeros((2, 3)), F2)
    assert opt.dt == pytest.approx(0.11, rel=1e-15) and opt.a == pytest.approx(0.099, rel=1e-15) and opt.Nsteps == 7
    opt = _fire(v=v, dt=0.95, n=6)
    opt.step(np.zeros((2, 3)), F2)
    assert opt.dt == 1.0                                                   # min(1.045, dtmax)


def test_maxstep_clamps_the_whole_structure():
    opt = _fire(maxstep=0.01)
    x = opt.step(np.zeros((2, 3)), F2)                                     # dr = 0.01 f, |dr| = 0.05
    np.testing.assert_allclose(x, 0.01 * F2 / 5.0, rtol=1e-15, atol=0)     # one norm, not per atom
    assert np.linalg.norm(x) == pytest.approx(0.01, rel=1e-15)
    opt = _fire(maxstep=0.05)
    np.testing.assert_allclose(opt.step(np.zeros((2, 3)), F2), 0.01 * F2, rtol=0, atol=1e-15)   # |dr| = maxstep: no clamp


# ---- the loop -----------------------------------------------------------------------------------------------------------------
def _scripted(ms):
    """Forces whose largest atom norm is ms[k] at the k-th evaluation (k = 0 at x_0), E_k = 10 k; they ignore x."""
    calls = []

    def forces(x):
        k = len(calls)
        calls.append(np.array(x))
        return 10.0 * k, np.array([[ms[min(k, len(ms) - 1)], 0.0, 0.0], [0.0, 0.0, 0.0]])
    return forces, calls


def test_no_revert_test_at_step_one():
    forces, _ = _scripted([1.0, 100.0, 100.0, 100.0])
    r = orx.relax(np.zeros((2, 3)), forces, fmax=0.0, max_steps=3)
    assert r["status"] == orx.MAX_STEPS and r["steps"] == 3


def test_revert_restores_previous_positions():
    forces, calls = _scripted([1.0, 1.0, 2.0])
    r = orx.relax(np.zeros((2, 3)), forces, fmax=0.0, max_steps=10)
    assert r["status"] == orx.REVERTED and r["steps"] == 2
    np.testing.assert_array_equal(r["positions"], calls[1])                # x_1
    assert r["energy"] == 10.0 and r["forces"][0, 0] == 1.0                # E_1, F_1
    np.testing.assert_array_equal(r["fmax_history"][:3], [1.0, 1.0, 2.0])  # row k = 2 is recorded before the revert
    assert np.isnan(r["fmax_history"][3:]).all()


def test_threshold_is_strict():
    forces, _ = _scripted([1.0, 1.0, 1.5, 1.5])
    assert orx.relax(np.zeros((2, 3)), forces, fmax=0.0, max_steps=3, max_force_increase=0.5)["status"] == orx.MAX_STEPS
    forces, _ = _scripted([1.0, 1.0, 1.5 + 1e-12])
    assert orx.relax(np.zeros((2, 3)), forces, fmax=0.0, max_steps=3, max_force_increase=0.5)["status"] == orx.REVERTED
    forces, _ = _scripted([1.0, 1.0, 100.0])
    assert orx.relax(np.zeros((2, 3)), forces, fmax=0.0, max_steps=3, max_force_increase=None)["status"] == orx.MAX_STEPS


def test_converged_and_max_steps():
    forces, _ = _scripted([0.001, 0.5, 0.01])               # x_0 is never tested, as in the script
    r = orx.relax(np.zeros((2, 3)), forces, fmax=0.02)
    assert r["status"] == orx.CONVERGED and r["steps"] == 2 and r["energy"] == 20.0
    forces, _ = _scripted([1.0])
    r = orx.relax(np.zeros((2, 3)), forces, fmax=0.02, max_steps=4)
    assert r["status"] == orx.MAX_STEPS and r["steps"] == 4 and not np.isnan(r["energy_history"]).any()


def _lj(x):
    """Lennard-Jones (epsilon = sigma = 1) energy and forces of a cluster."""
    x = np.asarray(x, dtype=np.float64)
    d = x[:, None, :] - x[None, :, :]
    r2 = (d ** 2).sum(-1) + np.eye(len(x))
    inv6 = 1.0 / r2 ** 3
    np.fill_diagonal(inv6, 0.0)
    e = 2.0 * float((inv6 * inv6 - inv6).sum())
    f = ((24.0 * (2.0 * inv6 * inv6 - inv6) / r2)[:, :, None] * d).sum(1)
    return e, f


@pytest.mark.parametrize("max_force_increase", [0.05, None])
def test_iteration_drives_the_loop(max_force_increase):
    """The kernel's cut of the rules (``iteration``) reproduces the script's loop bit for bit."""
    x0 = np.array([[0.0, 0.0, 0.0], [1.3, 0.0, 0.0], [0.5, 1.0, 0.1]])
    kw = dict(fmax=1e-3, maxstep=0.01, max_steps=300, max_force_increase=max_force_increase)
    ref = orx.relax(x0, _lj, **kw)
    s = orx.State(x0)
    eh, mh = [], []
    while s.status == orx.RUNNING:
        e, f = _lj(s.x)
        eh.append(e)
        mh.append(orx.iteration(s, e, f, **kw)[1])
    assert s.status == ref["status"] and s.k == ref["steps"]
    np.testing.assert_array_equal(s.x, ref["positions"])
    np.testing.assert_array_equal(np.array(mh), ref["fmax_history"][:len(mh)])
    np.testing.assert_array_equal(np.array(eh), ref["energy_history"][:len(eh)])


def test_harmonic_well_converges():
    k, fmax = 4.0, 1e-3
    xs = np.array([[0.5, -0.2, 0.1], [1.0, 1.0, 1.0], [-2.0, 0.3, 0.0]])
    x0 = xs + np.array([[0.3, 0.0, -0.1], [0.0, 0.2, 0.0], [-0.1, 0.1, 0.25]])
    r = orx.relax(x0, lambda x: (0.5 * k * float(((x - xs) ** 2).sum()), -k * (x - xs)), fmax=fmax, max_steps=2000,
                  max_force_increase=None)
    assert r["status"] == orx.CONVERGED
    assert np.linalg.norm(r["positions"] - xs, axis=1).max() < fmax / k


def _pairs(x):
    return np.array([np.linalg.norm(x[i] - x[j]) for i in range(len(x)) for j in range(i + 1, len(x))])


@pytest.mark.parametrize("x0", [[[0.0, 0.0, 0.0], [1.3, 0.0, 0.0]],
                                [[0.0, 0.0, 0.0], [1.25, 0.0, 0.0], [0.5, 1.05, 0.05]]], ids=["dimer", "trimer"])
def test_lj_clusters_converge_to_the_analytic_minimum(x0):
    fmax, rstar = 1e-4, 2.0 ** (1.0 / 6.0)
    x0 = np.array(x0)
    r = orx.relax(x0, _lj, fmax=fmax, maxstep=0.01, max_steps=5000, max_force_increase=None)
    assert r["status"] == orx.CONVERGED
    # |F| >= lambda_min |delta| on the modes that are not rigid motions, and m >= |F| / sqrt(N); a pair distance moves by at
    # most 2 |delta|.  The dimer's curvature along its bond is V''(r*) = 72 / 2^(1/3) per atom pair, the trimer's smallest
    # non-rigid eigenvalue is taken from a finite-difference Hessian at the equilateral minimum.
    n = len(x0)
    xm = np.array([[0.0, 0.0, 0.0], [rstar, 0.0, 0.0], [rstar / 2, rstar * math.sqrt(3) / 2, 0.0]])[:n]
    h = np.zeros((3 * n, 3 * n))
    for i in range(3 * n):
        dx = np.zeros(3 * n)
        dx[i] = 1e-6
        h[:, i] = -(_lj((xm.reshape(-1) + dx).reshape(n, 3))[1] - _lj((xm.reshape(-1) - dx).reshape(n, 3))[1]).reshape(-1) / 2e-6
    ev = np.linalg.eigvalsh(0.5 * (h + h.T))
    lam = ev[ev > 1e-3].min()
    assert np.abs(_pairs(r["positions"]) - rstar).max() < 2 * math.sqrt(n) * fmax / lam * 1.05


# ---- refusals -------------------------------------------------------------------------------------------------------------------
GRAPH = {"num_sharedlayers": 2, "dim_sharedlayers": 5, "num_headlayers": 2, "dim_headlayers": [10, 7]}
MLIP = dict(enable_interatomic_potential=True, energy_weight=1.0, energy_peratom_weight=1.0, force_weight=1.0)


def _model(mpnn_type="EGNN", graph=None, mlip=True, heads=None, **kw):
    heads = heads or {"graph": graph or [{"type": "branch-%d" % b, "architecture": dict(GRAPH)} for b in range(3)]}
    base = dict(mpnn_type=mpnn_type, input_dim=1, hidden_dim=8, num_conv_layers=2, num_radial=5, radius=5.0)
    base.update(kw)
    return hb.create_model(**base, output_dim=[1], output_type=["graph"], task_weights=[1.0], output_heads=heads,
                           graph_pooling="add", use_gpu=False, **(MLIP if mlip else {})).eval()


def _data(g=2):
    d = Batch(x=torch.ones(3 * g, 1), pos=torch.zeros(3 * g, 3), batch=torch.arange(g).repeat_interleave(3),
              edge_index=torch.zeros(2, 0, dtype=torch.int64))
    d._num_graphs = g
    return d


def _refused(model, match, nb=(5.0, 8), **kw):
    with pytest.raises(ValueError, match=match):
        hb.PaddedRelaxStep(model, _data(), nb, **kw)


def test_refusals():
    _refused(_model().train(), "eval mode")
    _refused(_model(mlip=False), "interatomic potential")
    m = _model()
    m.model.var_output = 1
    _refused(m, "mean-and-variance")
    differ = [{"type": "branch-%d" % b, "architecture": dict(GRAPH)} for b in range(3)]
    differ[1]["architecture"]["dim_headlayers"] = [10, 8]
    _refused(_model(graph=differ), "share one architecture")
    _refused(_model(edge_dim=1), "edge_attr")
    _refused(_model(), "neighbour_build", nb=None)
    for bad in (dict(fmax=-1.0), dict(maxstep=0.0), dict(max_steps=0)):
        _refused(_model(), "fmax >= 0", **bad)


def test_refuses_models_the_padded_batch_rejects():
    pna = _model("PNA", pna_deg=[0, 2, 4, 2], heads={"graph": [{"type": "branch-0", "architecture": dict(GRAPH)}]})
    if hb.padded.supported(pna):
        pytest.skip("this PNA configuration carries no BatchNorm feature layer")
    _refused(pna, "cannot run in a padded batch")
