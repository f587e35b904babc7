"""Branch-weighted prediction of a 16-branch MACE potential: the reference's loop against the one-pass paths, in one process.

    python profiles/branch_mix_bench.py [--graphs 32] [--batches 8] [--reps 5] [--branches 16]

The model is multibranch_step.py's ``gfm_mace_mlip`` (the architecture of the reference's
examples/multidataset_hpo_sc26/gfm_mlip.json, one graph energy head per dataset branch) in eval mode, on periodic cells of the
gfm_mace workload; the weights are a softmax of random logits per graph.  Three paths, timed alternately over the same batches:

* ``loop``: examples/multidataset_hpo_sc26/inference_fused.py without encoder reuse, with ``--fused_energy_grad``, on the
  engine's model: one full forward per branch (``dataset_name`` := b), the weighted sum, one backward for the forces;
* ``eager``: ``hb.branch_weighted_energy_forces`` (one encoder pass, every branch decoded at once, the mix kernel, one backward);
* ``captured``: ``hb.PaddedPredictStep``.

CUDA events around each pass over the batches.  Prints one JSON line with structures/s of each path (median over repetitions),
the largest difference of the one-pass results from the loop's, the card's name and its power limit.
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
from hydragnn_b200 import ops  # noqa: E402
from multibranch_step import batches, card, gfm_mace_mlip  # noqa: E402


def loop(model, data, weights, branches):
    """inference_fused.py's no-reuse path with the fused backward (:1329-1365, _fused_energy_forces :508-544)."""
    data.pos.requires_grad_(True)
    g = weights.shape[0]
    energy = torch.zeros(g, device=data.pos.device)
    for b in range(branches):
        data.dataset_name = torch.full((g, 1), b, dtype=torch.long, device=data.pos.device)
        energy = energy + weights[:, b] * model(data)[0].squeeze(-1)
    with ops.only_data_grads():
        forces = -torch.autograd.grad(energy, data.pos, grad_outputs=torch.ones_like(energy))[0]
    return energy.detach(), forces


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--graphs", type=int, default=32)
    ap.add_argument("--batches", type=int, default=8)
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--branches", type=int, default=16)
    a = ap.parse_args()
    data = batches(a.batches, a.graphs, a.branches)
    for b in data:
        del b.dataset_name
    atoms = sum(b.pos.shape[0] for b in data)
    edges = sum(b.edge_index.shape[1] for b in data)
    model = gfm_mace_mlip(a.branches, edges / atoms).eval()
    gen = torch.Generator().manual_seed(0)
    weights = [torch.softmax(torch.randn(a.graphs, a.branches, generator=gen), dim=-1).cuda() for _ in data]
    step = hb.PaddedPredictStep(model, max(data, key=lambda b: b.pos.shape[0]))
    out = {}

    def run_loop():
        out["loop"] = [loop(model, b, w, a.branches) for b, w in zip(data, weights)]

    def run_eager():
        out["eager"] = [hb.branch_weighted_energy_forces(model, b, w) for b, w in zip(data, weights)]

    def run_captured():
        res = []
        for b, w in zip(data, weights):
            step.load(b, w)
            res.append(tuple(t.clone() for t in step.run()[:2]))
        out["captured"] = res

    def timed(fn):
        t0, t1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        t0.record()
        fn()
        t1.record()
        torch.cuda.synchronize()
        return t0.elapsed_time(t1) / 1e3

    paths = {"loop": run_loop, "eager": run_eager, "captured": run_captured}
    for fn in paths.values():                              # warm-up: modules, allocator, the capture itself
        fn()
    torch.cuda.synchronize()
    secs = {k: [] for k in paths}
    for _ in range(a.reps):
        for k, fn in paths.items():
            secs[k].append(timed(fn))
    step.check()
    diff = {}
    for k in ("eager", "captured"):
        de = max(float((x[0] - y[0]).abs().max() / y[0].abs().max()) for x, y in zip(out[k], out["loop"]))
        df = max(float((x[1] - y[1]).norm() / y[1].norm()) for x, y in zip(out[k], out["loop"]))
        diff[k] = {"energy_rel_max": de, "forces_rel_l2": df}
    name, limit = card()
    structures = a.graphs * len(data)
    print(json.dumps({"card": name, "power_limit": limit, "graphs_per_batch": a.graphs, "branches": a.branches,
                      "atoms_per_batch": atoms / len(data), "edges_per_batch": edges / len(data),
                      **{"%s_structures_per_s" % k: structures / statistics.median(v) for k, v in secs.items()},
                      "seconds_all": secs, "difference_from_loop": diff, "recaptures": step.recaptures}))


if __name__ == "__main__":
    main()
