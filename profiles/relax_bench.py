"""Structure relaxation of a 16-branch MACE potential: the reference script's one-structure loop against the batched step.

    python profiles/relax_bench.py [--graphs 16] [--steps 20] [--reps 3] [--branches 16]

The model is multibranch_step.py's ``gfm_mace_mlip`` (the architecture of the reference's
examples/multidataset_hpo_sc26/gfm_mlip.json) with its concat_node conditioning on a two-wide graph_attr, in eval mode, on
periodic cells of the gfm_mace workload (60 to 100 atoms) displaced by up to 0.1 A per coordinate, as
structure_optimization_ASE.py's ``--random_displacement`` does.  ``fmax = 0`` so that every structure runs ``--steps``
steps: fixed work on a randomly initialised potential.  Two paths over the same structures, timed alternately:

* ``loop``: structure_optimization_ASE.py's loop on the engine, one structure at a time: every step an exact-count periodic
  build, ``hb.branch_weighted_energy_forces``, the forces to the host and oracle/relax.py's FIRE there;
* ``batched``: ``hb.PaddedRelaxStep`` over all structures, once for every candidate number of iterations per captured graph.

CUDA events around each pass.  Prints one JSON line: structure-steps/s of each path (median over repetitions), the largest
position difference between the two after three steps, the card's name and its power limit.
"""
import argparse
import json
import os
import statistics
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
import torch  # noqa: E402

import hydragnn_b200 as hb  # noqa: E402
from hydragnn_b200 import radius, relax  # noqa: E402
from hydragnn_b200.synthetic import WORKLOADS, make_samples  # noqa: E402
from multibranch_step import card, gfm_mace_mlip  # noqa: E402
from oracle import relax as orx  # noqa: E402

ITERATIONS = (1, 4, 8, 16)


def structures(graphs, seed=7):
    b = make_samples("gfm_mace", graphs, seed=seed)
    gen = torch.Generator().manual_seed(seed)
    ptr = b.ptr.tolist()
    out = []
    for g in range(graphs):
        n = ptr[g + 1] - ptr[g]
        s = hb.Batch(x=b.x[ptr[g]:ptr[g + 1]], batch=torch.zeros(n, dtype=torch.int64),
                     pos=b.pos[ptr[g]:ptr[g + 1]].double() + (torch.rand(n, 3, generator=gen, dtype=torch.float64) - 0.5) * 0.2,
                     cell=b.cell[g:g + 1].double(), pbc=b.pbc[g:g + 1], graph_attr=torch.randn(1, 2, generator=gen))
        s._num_graphs = 1
        out.append(s)
    return out


def collate(structs):
    n = torch.tensor([s.pos.shape[0] for s in structs])
    b = hb.Batch(x=torch.cat([s.x for s in structs]), pos=torch.cat([s.pos for s in structs]),
                 batch=torch.repeat_interleave(torch.arange(len(structs)), n), cell=torch.cat([s.cell for s in structs]),
                 pbc=torch.cat([s.pbc for s in structs]), graph_attr=torch.cat([s.graph_attr for s in structs]))
    b._num_graphs = len(structs)
    return b


def script_loop(model, s, w, nb, steps):
    """structure_optimization_ASE.py's loop around FIRE with the engine as the calculator (:196-265, :385-439)."""
    r, k = nb
    dev = w.device
    x_, cell, pbc, ga = s.x.to(dev), s.cell.to(dev), s.pbc.to(dev), s.graph_attr.to(dev)
    gptr = torch.tensor([0, s.pos.shape[0]], dtype=torch.int32, device=dev)
    cut = torch.full((1,), r, dtype=torch.float64, device=dev)

    def forces(x):
        d = hb.Batch(x=x_, pos=torch.from_numpy(x).float().to(dev), batch=torch.zeros(x.shape[0], dtype=torch.int64, device=dev),
                     graph_attr=ga)
        d._num_graphs = 1
        d.edge_index, _, d.edge_shifts, _, _, _ = radius.radius_graph_pbc(d.pos, cell, pbc, cut, gptr, 1, k)
        e, f, _ = hb.branch_weighted_energy_forces(model, d, w)
        return float(e[0]), f.double().cpu().numpy()
    return orx.relax(s.pos.numpy(), forces, fmax=0.0, maxstep=0.01, max_steps=steps)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--graphs", type=int, default=16)
    ap.add_argument("--steps", type=int, default=20)
    ap.add_argument("--reps", type=int, default=3)
    ap.add_argument("--branches", type=int, default=16)
    a = ap.parse_args()
    w0 = WORKLOADS["gfm_mace"]
    nb = (w0["radius"], w0["max_neighbours"])
    structs = structures(a.graphs)
    batch = collate(structs)
    model = gfm_mace_mlip(a.branches, 12.0)
    model.model.use_graph_attr_conditioning, model.model.graph_attr_conditioning_mode = True, "concat_node"
    model.model._ensure_graph_concat_projector(graph_attr_dim=2, channel_dim=model.model.hidden_dim, device=model.model.device)
    model.eval()
    gen = torch.Generator().manual_seed(1)
    weights = torch.softmax(torch.randn(a.graphs, a.branches, generator=gen), dim=-1).cuda()
    steps = {it: hb.PaddedRelaxStep(model, batch, nb, fmax=0.0, max_steps=a.steps) for it in ITERATIONS}
    out = {}

    def run_loop():
        out["loop"] = [script_loop(model, s, weights[i:i + 1], nb, a.steps) for i, s in enumerate(structs)]

    def run_batched(it):
        def fn():
            relax.ITERATIONS = it
            steps[it].load(batch, weights)
            out[it] = steps[it].run()
        return fn

    def timed(fn):
        t0, t1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        t0.record()
        fn()
        t1.record()
        torch.cuda.synchronize()
        return t0.elapsed_time(t1) / 1e3

    paths = {"loop": run_loop, **{"batched_%d" % it: run_batched(it) for it in ITERATIONS}}
    for fn in paths.values():                              # warm-up: modules, allocator, the captures
        fn()
    torch.cuda.synchronize()
    secs = {k: [] for k in paths}
    for _ in range(a.reps):
        for k, fn in paths.items():
            secs[k].append(timed(fn))
    work = a.graphs * a.steps
    # the two paths after three steps, from the same start
    relax.ITERATIONS = 8
    few = hb.PaddedRelaxStep(model, batch, nb, fmax=0.0, max_steps=3)
    few.load(batch, weights)
    res = few.run()
    ref = torch.cat([torch.from_numpy(script_loop(model, s, weights[i:i + 1], nb, 3)["positions"]) for i, s in enumerate(structs)])
    full = torch.cat([torch.from_numpy(r["positions"]) for r in out["loop"]])
    name, limit = card()
    print(json.dumps({"card": name, "power_limit": limit, "graphs": a.graphs, "branches": a.branches, "steps": a.steps,
                      "atoms": int(batch.pos.shape[0]),
                      **{"%s_structure_steps_per_s" % k: work / statistics.median(v) for k, v in secs.items()},
                      "seconds_all": secs, "max_position_difference_after_3_steps": float((res.positions.cpu() - ref).abs().max()),
                      "max_position_difference_after_all_steps": float((out[8].positions.cpu() - full).abs().max()),
                      "recaptures": {it: s.recaptures for it, s in steps.items()}}))


if __name__ == "__main__":
    main()
