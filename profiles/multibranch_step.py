"""Training-step time of a multi-branch MACE interatomic potential, eager against the captured padded step, in one process.

    python profiles/multibranch_step.py [--graphs 32] [--batches 8] [--reps 5] [--branches 16]

The model has the architecture of the reference's examples/multidataset_hpo_sc26/gfm_mlip.json: MACE, hidden 128, 4
layers, max_ell 1, 6 Bessel functions, radius 5, at most 20 neighbours, add pooling, and one graph energy head with 2 x 50
shared layers and 3 x 128 head layers, replicated once per dataset branch as gfm_mlip_all_mpnn.py does, trained on energy per
atom (weight 1) and forces (weight 10).  Left out: the config's concat_node conditioning on graph_attr and its one-wide
edge_attr.  Every batch mixes graphs of every branch (``dataset_name`` drawn per graph), so each readout of both steps decodes
through the grouped kernels.

Each repetition times every batch once eagerly (``hb.train_step``) and once through ``PaddedGraphStep``, alternating, each
with its own copy of the model and optimizer; CUDA events around each pass.  Prints one JSON line with the median ms per step
of each path, the card's name and its power limit.
"""
import argparse
import copy
import json
import os
import statistics
import subprocess
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import torch  # noqa: E402

import hydragnn_b200 as hb  # noqa: E402
from hydragnn_b200.padded import PaddedGraphStep  # noqa: E402
from hydragnn_b200.synthetic import WORKLOADS, make_samples  # noqa: E402


def gfm_mace_mlip(branches, avg_num_neighbors):
    head = {"num_sharedlayers": 2, "dim_sharedlayers": 50, "num_headlayers": 3, "dim_headlayers": [128, 128, 128]}
    return hb.create_model(mpnn_type="MACE", input_dim=1, hidden_dim=128, num_conv_layers=4, max_ell=1, node_max_ell=1,
                           num_radial=6, radius=5.0, radial_type="bessel", envelope_exponent=5, correlation=2,
                           avg_num_neighbors=avg_num_neighbors, max_neighbours=20, graph_pooling="add",
                           output_dim=[1], output_type=["graph"], task_weights=[1.0],
                           output_heads={"graph": [{"type": "branch-%d" % b, "architecture": dict(head)} for b in range(branches)]},
                           activation_function="relu", loss_function_type="mse", enable_interatomic_potential=True,
                           energy_weight=0.0, energy_peratom_weight=1.0, force_weight=10.0)


def batches(count, graphs, branches):
    w = WORKLOADS["gfm_mace"]
    out = []
    for i in range(count):
        b = make_samples("gfm_mace", graphs, seed=100 + i).to("cuda")
        b._num_graphs = graphs
        b = hb.get_radius_graph_pbc(w["radius"], w["max_neighbours"])(b)
        gen = torch.Generator().manual_seed(i)
        b.dataset_name = torch.randint(0, branches, (graphs, 1), generator=gen).to("cuda")
        for k in ("cell", "pbc", "ptr"):
            b.__dict__.pop(k, None)
        out.append(b)
    return out


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader", "-i",
                        str(torch.cuda.current_device())], capture_output=True, text=True)
    name, _, limit = q.stdout.strip().partition(", ")
    return name or torch.cuda.get_device_name(), limit or "unknown"


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--graphs", type=int, default=32)
    ap.add_argument("--batches", type=int, default=8)
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--branches", type=int, default=16)
    a = ap.parse_args()
    data = batches(a.batches, a.graphs, a.branches)
    data_c = [b.clone() for b in data]                  # the eager step marks its batches' positions as requiring grad
    atoms = sum(b.pos.shape[0] for b in data)
    edges = sum(b.edge_index.shape[1] for b in data)
    me = hb.get_distributed_model(gfm_mace_mlip(a.branches, edges / atoms))
    mc = copy.deepcopy(me)
    oe, oc = hb.FlatAdamW(me, lr=1e-4), hb.FlatAdamW(mc, lr=1e-4)
    step = PaddedGraphStep(mc, oc, max(data_c, key=lambda b: b.pos.shape[0]), compute_grad_energy=True)

    def eager():
        for b in data:
            hb.train_step(me, oe, b, compute_grad_energy=True)

    def captured():
        for b in data_c:
            step.load(b)
            step.run()

    def timed(fn):
        t0, t1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        t0.record()
        fn()
        t1.record()
        torch.cuda.synchronize()
        return t0.elapsed_time(t1) / len(data)

    eager()                                              # warm-up: modules, allocator, the capture itself
    captured()
    torch.cuda.synchronize()
    ms = {"eager": [], "captured": []}
    for _ in range(a.reps):
        ms["eager"].append(timed(eager))
        ms["captured"].append(timed(captured))
    step.check()
    name, limit = card()
    print(json.dumps({"card": name, "power_limit": limit, "graphs_per_batch": a.graphs, "branches": a.branches,
                      "atoms_per_batch": atoms / len(data), "edges_per_batch": edges / len(data),
                      "eager_ms_per_step": statistics.median(ms["eager"]), "captured_ms_per_step": statistics.median(ms["captured"]),
                      "eager_ms_all": ms["eager"], "captured_ms_all": ms["captured"], "recaptures": step.recaptures}))


if __name__ == "__main__":
    main()
