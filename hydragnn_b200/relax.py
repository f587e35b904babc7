"""Batched structure relaxation with an interatomic potential: FIRE steps, neighbour rebuilds and forces in one captured graph.

The reference relaxes one structure at a time with examples/multidataset_hpo_sc26/structure_optimization_ASE.py: an ASE
calculator around the fused prediction (``FusedHydraGNNCalculator`` :196-265) rebuilds the periodic graph from the current
positions at every evaluation (``atoms_to_graph`` :175-193, positions cast to the model dtype), and the loop (:385-439)
around ``ase.optimize.FIRE(atoms, maxstep=1e-2)`` stops a structure when its largest per-atom force falls below ``fmax``,
reverts it to its previous positions when that force grows by more than ``relative_increase_threshold``, or stops after
``maxiter`` steps.  Every step is a host round trip.

``PaddedRelaxStep`` relaxes a whole batch on the device.  One iteration is the in-step neighbour build (periodic for batches
with ``cell`` and ``pbc``, ``padded.PaddedBatch``), the branch-weighted energy and forces (``predict._mix``) and one
``hgb_fire_step`` launch, which keeps every structure's FIRE state, applies the script's stopping rules and moves the
structures still running.  ``ITERATIONS`` iterations are captured as one CUDA graph; the host replays it and reads one word
(structures still running, and the device guard) after every replay.
"""
import collections
import copy

import torch

from . import _lib, ops, radius
from .ops import _p, _stream
from .padded import PaddedBatch, _round_up, supported
from .predict import _inner, _mix

RUNNING, CONVERGED, REVERTED, MAX_STEPS = 0, 1, 2, 3

# Iterations per captured graph.  Fewer mean more host reads of the live word; more mean more iterations run after the
# last structure has stopped.  One measured fastest with profiles/relax_bench.py (DESIGN.md, "Structure relaxation").
ITERATIONS = 1

RelaxResult = collections.namedtuple("RelaxResult", "positions energy forces steps status energy_history fmax_history")


class PaddedRelaxStep(PaddedBatch):
    """Relaxes every structure of a batch to a local minimum of a (multi-branch) interatomic potential, as
    structure_optimization_ASE.py does one structure at a time with FIRE.

        step = PaddedRelaxStep(model, first_batch, neighbour_build=(radius, max_neighbours))
        step.load(batch, weights)          # weights [G, B] float32 on the model's device; B = 1 needs none
        res = step.run()

    ``res`` (a ``RelaxResult``): positions [N, 3] fp64, energy [G] and forces [N, 3] at those positions, steps [G] int32
    (the step at which each structure stopped), status [G] int32 (``CONVERGED``, ``REVERTED`` or ``MAX_STEPS``), and
    energy_history / fmax_history [max_steps + 1, G] fp64 (row 0 = the start, NaN after a structure stopped).  A reverted
    structure returns its positions before the last step, and the energy and forces there.

    ``fmax``, ``maxstep``, ``max_steps`` and ``max_force_increase`` are the script's ``--fmax``, FIRE's ``maxstep``,
    ``--maxiter`` and ``--relative_increase_threshold`` (None: no revert rule).  Positions are kept in fp64 (as ASE keeps
    them) and cast to fp32 for the neighbour build and the model, as the script casts them.  Periodic batches (with
    ``cell`` and ``pbc``) rebuild their graphs with ``radius_graph_pbc`` under candidate and edge capacities; when one is
    exceeded the last block of iterations is undone, the graph recaptured with larger capacities and the block replayed, so
    the result equals a run with ample capacities (``recaptures`` counts them).  ``capture=False`` runs the same iterations
    without a CUDA graph.  Parameters, their gradients and optimizer state are not touched; the model stays in eval mode."""

    def __init__(self, model, first_batch, neighbour_build, fmax=0.02, maxstep=0.01, max_steps=200, max_force_increase=0.05,
                 node_cap=None, edge_cap=None, graph_cap=None, candidate_cap=None, slack=1.12, warmup=2, capture=True):
        self.inner = _inner(model)
        if not supported(model):
            raise ValueError("PaddedRelaxStep: this model (global attention / BatchNorm feature layers / SchNet) cannot run "
                             "in a padded batch")
        if getattr(self.inner, "use_edge_attr", False):
            raise ValueError("PaddedRelaxStep: the model reads edge_attr, but the edges are rebuilt from the positions at "
                             "every step")
        if neighbour_build is None:
            raise ValueError("PaddedRelaxStep: neighbour_build = (radius, max_neighbours) is required: the atoms move, so "
                             "the graph is rebuilt at every step")
        if not (float(fmax) >= 0.0 and float(maxstep) > 0.0 and int(max_steps) >= 1):
            raise ValueError("PaddedRelaxStep: needs fmax >= 0, maxstep > 0 and max_steps >= 1")
        self.fmax, self.maxstep, self.max_steps = float(fmax), float(maxstep), int(max_steps)
        self.threshold = None if max_force_increase is None else float(max_force_increase)
        self.capture = capture
        self.branches = getattr(self.inner, "num_branches", 1)
        periodic = first_batch.cell is not None and first_batch.pbc is not None
        extra = {"branch_weights": ((self.branches,), torch.float32)}
        if periodic:
            extra.update(cell=((3, 3), torch.float64), pbc=((3,), torch.int32))
        self.cand_cap, self._caps = None, (candidate_cap, edge_cap)
        self.graph, self._state, self._x0 = None, None, None
        first_batch = copy.copy(first_batch)
        first_batch.pos = first_batch.pos.float()             # the model and the neighbour build read fp32 positions
        super().__init__(model, first_batch, neighbour_build, node_cap, edge_cap, graph_cap, slack, warmup, targets=False,
                         extra=extra, periodic=periodic)

    # ---- capacities ------------------------------------------------------------------------------------------------------
    def _capture(self, n_need, e_need, g_need):
        super()._capture(n_need, e_need, g_need)
        self.cand_cap = None                                 # sized on the first batch of these buffers (_size_edges)

    def _size_edges(self, grow=False):
        """Candidate and edge capacities of the periodic build: the counts at the current positions, with slack; at least
        1.5 x the last ones after an overflow.  Every target keeps at most max_neighbours edges, so n_cap x max_neighbours
        edges always fit."""
        d, k = self.data, int(self.nb[1])
        _, _, _, _, outptr, c = radius.radius_graph_pbc(d.pos.detach(), d.cell, d.pbc, self.cutoff, d.ptr, self.g_cap, k)
        c, e = _round_up(c * self.slack + 64, 64), _round_up(int(outptr[-1]) * self.slack + 64, 64)
        if grow:
            c, e = max(c, _round_up(self.cand_cap * 1.5, 64)), max(e, _round_up(self.e_cap * 1.5, 64))
        elif self._caps != (None, None):                     # the caller's capacities, for the first capture only
            c, e = self._caps[0] or c, self._caps[1] or e
            self._caps = (None, None)
        self.cand_cap, self.e_cap = c, min(e, self.n_cap * k)

    # ---- relaxation state (outside the buffers _capture reallocates) ------------------------------------------------------
    def _alloc_state(self):
        n, g, dev, f64 = self.n_cap, self.g_cap, self.dev, torch.float64
        if self._state is not None and self.x.shape[0] == n and self.e_out.shape[0] == g:
            return
        self.x, self.v, self.x_prev = (torch.zeros(n, 3, dtype=f64, device=dev) for _ in range(3))
        self.fire = torch.zeros(g, 3, dtype=f64, device=dev)                    # dt, a, m_{k-1}
        self.istate = torch.zeros(g, 3, dtype=torch.int32, device=dev)          # status, k, FIRE's n
        self.e_hist, self.f_hist = (torch.zeros(self.max_steps + 1, g, dtype=f64, device=dev) for _ in range(2))
        self.e_out, self.f_out = torch.zeros(g, device=dev), torch.zeros(n, 3, device=dev)
        self._state = [self.x, self.v, self.x_prev, self.fire, self.istate, self.e_hist, self.f_hist, self.e_out, self.f_out]
        self._snap = [torch.empty_like(t) for t in self._state]
        self.live = torch.zeros(2, dtype=torch.int32, device=dev)

    def _reset(self):
        """x = x_0 (the caller's positions, fp64), v = 0, dt = a = 0.1, n = 0, every structure running at k = 0."""
        n, pos = self.real[1], self.data.pos.detach()
        self.x.copy_(pos)
        self.x[:n] = self._x0
        self.x_prev.copy_(self.x)
        self.v.zero_()
        self.fire.zero_()
        self.fire[:, :2] = 0.1
        self.istate.zero_()
        for t in (self.e_hist, self.f_hist, self.e_out, self.f_out):
            t.fill_(float("nan"))
        pos[:n] = self._x0

    # ---- the body ---------------------------------------------------------------------------------------------------------
    def _iteration(self):
        d = self.data
        self._prologue()
        energy, forces, _ = _mix(self.model, self.inner, d, d.branch_weights)
        _lib.call("hgb_fire_step", _p(self.valid), _p(d.ptr), self.g_cap, _p(energy), _p(forces), _p(self.x), _p(self.v),
                  _p(self.x_prev), _p(self.fire), _p(self.istate), _p(self.e_hist), _p(self.f_hist), self.g_cap, _p(self.e_out),
                  _p(self.f_out), _p(d.pos), self.fmax, self.maxstep, self.max_steps, int(self.threshold is not None),
                  0.0 if self.threshold is None else self.threshold, _p(ops.guard_flag(self.dev)), _p(self.live), _stream())

    def _block(self):
        for s, t in zip(self._snap, self._state):          # the state this block starts from, restored on an overflow
            s.copy_(t)
        for _ in range(ITERATIONS):
            self._iteration()

    def _capture_block(self):
        if self.capture:
            keep = [t.clone() for t in self._state] + [self.data.pos.detach().clone()]
            side = torch.cuda.Stream()
            side.wait_stream(torch.cuda.current_stream())
            with torch.cuda.stream(side):
                for _ in range(self.warmup):
                    self._block()
            torch.cuda.current_stream().wait_stream(side)
            torch.cuda.synchronize()
            self.graph = torch.cuda.CUDAGraph()
            with ops.capture_graph(self.graph):
                self._block()
            for dst, src in zip(self._state + [self.data.pos.detach()], keep):
                dst.copy_(src)
        self._captured = True

    def _do_capture(self):
        self._alloc_state()
        self._reset()
        if self.periodic:
            self._size_edges()
        self._capture_block()

    # ---- per batch --------------------------------------------------------------------------------------------------------
    def load(self, batch, weights=None):
        """Pad ``batch`` (CPU or CUDA; positions of any float dtype, kept in fp64) and its branch weights [G, B] (float32, on
        the model's device; None for a single-branch model) into the step; every structure starts at k = 0.  Returns the
        number of structures."""
        g, b = int(batch.num_graphs), self.branches
        if weights is None and b == 1:
            weights = torch.ones(g, 1, device=self.dev)
        if not torch.is_tensor(weights) or weights.dtype != torch.float32 or tuple(weights.shape) != (g, b) \
                or weights.device != self.dev:
            raise ValueError("weights must be a float32 [graphs, branches] = [%d, %d] tensor on %s" % (g, b, self.dev))
        if self.periodic and (batch.cell is None or batch.pbc is None):
            raise ValueError("PaddedRelaxStep: the step was built for periodic batches; this batch has no cell / pbc")
        self._x0 = batch.pos.detach().to(self.dev, torch.float64)
        staged = copy.copy(batch)
        staged.pos = self._x0.float()
        extra = {"branch_weights": weights.detach()}
        if self.periodic:
            extra.update(cell=torch.as_tensor(batch.cell).reshape(g, 3, 3), pbc=torch.as_tensor(batch.pbc).reshape(g, 3))
        super().load(staged, **extra)
        self._alloc_state()
        self._reset()
        return g

    def run(self):
        """Relax the batch last loaded; returns a ``RelaxResult`` (fresh tensors)."""
        flag = ops.guard_flag(self.dev)
        while True:
            if self.capture:
                self.graph.replay()
            else:
                self._block()
            running, guard = self.live.tolist()
            if guard:
                if guard != ops.GUARD_EDGE_COUNT:
                    ops.check_guard(self.dev)                # raises: not an overflow of the neighbour build
                flag.zero_()
                saved = [s.clone() for s in self._snap]
                for t, s in zip(self._state, saved):
                    t.copy_(s)
                self.data.pos.detach()[:self.real[1]] = self.x[:self.real[1]]
                self._size_edges(grow=True)
                self._capture_block()                        # leaves the state as it found it
                self.recaptures += 1
                continue
            if running == 0:
                break
        g, n = self.real
        return RelaxResult(self.x[:n].clone(), self.e_out[:g].clone(), self.f_out[:n].clone(), self.istate[:g, 1].clone(),
                           self.istate[:g, 0].clone(), self.e_hist[:, :g].clone(), self.f_hist[:, :g].clone())
