"""Oracle: FIRE and the relaxation loop of examples/multidataset_hpo_sc26/structure_optimization_ASE.py, in fp64, driven by a
force callback.  Test infrastructure only.

``Fire.step`` restates ase.optimize.FIRE.step (ASE 3.26, ase/optimize/fire.py; the script builds it as
``FIRE(atoms, maxstep=1e-2)`` :268-273) with its defaults and without the downhill check, which the script leaves off.  ASE
is not installed where this was written: the step is restated from its definition, not executed against ASE.

``relax`` is the script's loop (:385-439): for k = 1 .. maxiter, one FIRE step on F(x_{k-1}), then E_k and F_k at x_k,
m_k = sqrt(max_i |F_i|^2); revert to x_{k-1} and stop when m_{k-1} > 0 and (m_k - m_{k-1}) / m_{k-1} exceeds the threshold
(never at k = 1), else stop when m_k < fmax, else stop after maxiter steps.

``iteration`` is the same rules cut where the engine's kernel (``hgb_fire_step``) cuts them: the bookkeeping of one
evaluation followed by the move to the next positions.  The CPU tests check that driving ``iteration`` gives ``relax``.
"""
import numpy as np

RUNNING, CONVERGED, REVERTED, MAX_STEPS = 0, 1, 2, 3


class Fire:
    """ASE's FIRE state of one structure: v (None before the first step), dt, a and the count n of downhill steps."""

    def __init__(self, maxstep=0.01, dt=0.1, dtmax=1.0, Nmin=5, finc=1.1, fdec=0.5, astart=0.1, fa=0.99):
        self.maxstep, self.dt, self.dtmax, self.Nmin = maxstep, dt, dtmax, Nmin
        self.finc, self.fdec, self.astart, self.fa = finc, fdec, astart, fa
        self.a, self.Nsteps, self.v = astart, 0, None

    def step(self, x, f):
        """The positions after one step from x [N, 3] with forces f [N, 3] (both fp64)."""
        f = np.asarray(f, dtype=np.float64)
        if self.v is None:
            self.v = np.zeros_like(f)
        else:
            vf = np.vdot(f, self.v)
            if vf > 0.0:
                self.v = (1.0 - self.a) * self.v + self.a * f / np.sqrt(np.vdot(f, f)) * np.sqrt(np.vdot(self.v, self.v))
                if self.Nsteps > self.Nmin:
                    self.dt = min(self.dt * self.finc, self.dtmax)
                    self.a *= self.fa
                self.Nsteps += 1
            else:
                self.v[:] *= 0.0
                self.a = self.astart
                self.dt *= self.fdec
                self.Nsteps = 0
        self.v += self.dt * f
        dr = self.dt * self.v
        normdr = np.sqrt(np.vdot(dr, dr))
        if normdr > self.maxstep:
            dr = self.maxstep * dr / normdr
        return np.asarray(x, dtype=np.float64) + dr


def max_force(f):
    """The script's m = sqrt(max_i sum_a F_ia^2) (:393)."""
    f = np.asarray(f, dtype=np.float64)
    return float(np.sqrt((f ** 2).sum(axis=1).max())) if f.size else 0.0


def relax(x0, forces, fmax=0.02, maxstep=0.01, max_steps=200, max_force_increase=0.05):
    """The script's loop on one structure.  ``forces(x)`` -> (E, F [N, 3]) at positions x [N, 3] fp64;
    ``max_force_increase`` None: no revert rule.  Returns a dict: positions, energy and forces at them, steps (the k at which
    the loop stopped), status, energy_history and fmax_history [max_steps + 1] (row 0 = x_0, NaN after the stop)."""
    x = np.array(x0, dtype=np.float64)
    opt = Fire(maxstep=maxstep)
    e, f = forces(x)
    eh, mh = [float(e)], [max_force(f)]
    prev_m = prev_x = None
    status, steps = MAX_STEPS, max_steps
    for k in range(1, max_steps + 1):
        x = opt.step(x, f)
        e_k, f_k = forces(x)
        m = max_force(f_k)
        eh.append(float(e_k))
        mh.append(m)
        if max_force_increase is not None and prev_m is not None and prev_m > 0.0:
            if (m - prev_m) / prev_m > max_force_increase:
                x, status, steps = prev_x, REVERTED, k               # E and F stay those of x_{k-1}
                break
        e, f = e_k, f_k
        if m < fmax:
            status, steps = CONVERGED, k
            break
        prev_m, prev_x = m, x.copy()
    pad = [float("nan")] * (max_steps + 1 - len(eh))
    return {"positions": x, "energy": float(e), "forces": np.asarray(f, dtype=np.float64), "steps": steps, "status": status,
            "energy_history": np.array(eh + pad), "fmax_history": np.array(mh + pad)}


class State:
    """One structure's state between kernel iterations: x, v, x_prev [N, 3], dt, a, n, m_prev, status and k."""

    def __init__(self, x0):
        self.x = np.array(x0, dtype=np.float64)
        self.x_prev = self.x.copy()
        self.v = np.zeros_like(self.x)
        self.dt, self.a, self.n, self.m_prev, self.status, self.k = 0.1, 0.1, 0, 0.0, RUNNING, 0


def iteration(s, e, f, fmax=0.02, maxstep=0.01, max_steps=200, max_force_increase=0.05):
    """One kernel iteration on a running structure ``s`` evaluated at s.x: (E_k, m_k) for row s.k of the histories; then the
    revert / converged / max-steps rules, or the FIRE move to x_{k+1}.  Returns (E_k, m_k)."""
    m = max_force(f)
    k = s.k
    if max_force_increase is not None and k >= 2 and s.m_prev > 0.0 and (m - s.m_prev) / s.m_prev > max_force_increase:
        s.status, s.x = REVERTED, s.x_prev.copy()
    elif k >= 1 and m < fmax:
        s.status = CONVERGED
    elif k >= max_steps:
        s.status = MAX_STEPS
    else:
        opt = Fire(maxstep=maxstep)
        opt.dt, opt.a, opt.Nsteps, opt.v = s.dt, s.a, s.n, (None if k == 0 else s.v)
        s.x_prev = s.x.copy()
        s.x = opt.step(s.x, f)
        s.v, s.dt, s.a, s.n, s.m_prev, s.k = opt.v, opt.dt, opt.a, opt.Nsteps, m, k + 1
    return float(e), m
