"""MACE distance-transform timing (distance_transform "Agnesi" / "Soft"; mace_utils/modules/radial.py:151-245), one GPU.

    python profiles/mace_transform_bench.py [--graphs 256] [--mlip-graphs 64] [--steps 20]

Prints one JSON line with the card name and power limit beside every number:
* the fused edge embedding, forward + backward, at the C4 (oc20_mace) shape: l <= 2 spherical harmonics and 8 Bessel functions
  per edge, hgb_mace_edge_embed_fwd / _bwd without a transform against hgb_mace_edge_embed_dt_fwd / _dt_bwd with Agnesi and
  with Soft, alternated in the same call (CUDA events, three rounds, the median), with the algorithmic bytes and their share of
  the 3.35 TB/s HBM3 bound (H100 SXM data sheet).  Per edge, with 4-byte floats and int32 indices, forward + backward:
    no transform   2 (8 + 12 + 12) + 4 (9 + 8) + 4 (9 + 8) + 12       row/col, two positions, shifts (twice); sh and radial
                                                                          written, then read as gradients; g_vec written
    transform      + 2 * 16                                               the two element indices (int64), twice
  (positions and element indices are gathered per edge; the 119-entry radii table sits in shared memory);
* eager MLIP training steps (FlatAdamW) of the gfm_mace workload with and without "Agnesi", alternated: the any-order path
  (DistTransformFn, hgb_mace_dist_transform).
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
from hydragnn_b200.synthetic import ARCH, WORKLOADS, make_samples  # noqa: E402
from pna_bench import card, timed  # noqa: E402

HBM = 3.35e12


def alternate(fns, steps):
    res = {k: [] for k in fns}
    for _ in range(3):
        for k, fn in fns.items():
            res[k] += timed(fn, steps, regions=1)
    return {k: statistics.median(v) for k, v in res.items()}


def batch(name, graphs, seed=0):
    w = WORKLOADS[name]
    d = make_samples(name, graphs, seed=seed).to("cuda")
    d._num_graphs = graphs
    return hb.get_radius_graph_pbc(w["radius"], w["max_neighbours"])(d)


def edge_embed(graphs, steps):
    name = "oc20_mace"
    a = ARCH[name]
    d = batch(name, graphs)
    n, e = d.pos.shape[0], int(d.edge_index.shape[1])
    plan = ops.EdgePlan(d.edge_index, n)
    lmax, nb, rc, p = a["max_ell"], a["num_radial"], a["radius"], float(a["envelope_exponent"])
    pos = d.pos.detach().requires_grad_(True)
    shifts = d.edge_shifts.float().contiguous()
    z = (d.x.squeeze().clamp(1, 118) - 1).long()
    models = {kind: hb.create_model(**dict(a, hidden_dim=32, distance_transform=kind)) for kind in ("Agnesi", "Soft")}
    dts = {kind: m.distance_transform_operands(z) for kind, m in models.items()}
    gen = torch.Generator(device="cuda").manual_seed(0)
    g_sh = torch.randn(e, (lmax + 1) ** 2, device="cuda", generator=gen)
    g_rad = torch.randn(e, nb, device="cuda", generator=gen)

    def run(kind):
        def fn():
            if kind == "none":
                sh, radial = ops.MaceEdgeEmbedFn.apply(pos, shifts, plan, lmax, nb, rc, p)
            else:
                sh, radial = ops.MaceEdgeEmbedDtFn.apply(pos, shifts, plan, dts[kind], lmax, nb, rc, p)
            return torch.autograd.grad((sh, radial), pos, (g_sh, g_rad))
        return fn
    fns = {k: run(k) for k in ("none", "Agnesi", "Soft")}
    for fn in fns.values():
        fn()
    torch.cuda.synchronize()
    ms = alternate(fns, steps)
    ns = (lmax + 1) ** 2
    base = e * (2 * (8 + 12 + 12) + 4 * (ns + nb) * 2 + 12)
    out = {"graphs": graphs, "atoms": n, "edges": e, "lmax": lmax, "num_bessel": nb}
    for k, v in ms.items():
        nbytes = base + (2 * 16 * e if k != "none" else 0)
        out[k] = {"ms_fwd_bwd": round(v, 4), "algorithmic_bytes": nbytes, "achieved_GBps": round(nbytes / (v * 1e-3) / 1e9, 1),
                  "frac_of_hbm_peak": round(nbytes / HBM / (v * 1e-3), 3)}
    out["overhead_vs_none"] = {k: round(ms[k] / ms["none"] - 1.0, 4) for k in ("Agnesi", "Soft")}
    return out


def mlip_steps(graphs, steps):
    name = "gfm_mace"
    d = batch(name, graphs, seed=1)
    vec = d.pos[d.edge_index[1]] - d.pos[d.edge_index[0]] + d.edge_shifts.to(d.pos.dtype)
    d.edge_attr = vec.norm(dim=1, keepdim=True).detach()
    d.graph_attr = torch.randn(graphs, 2, device="cuda", generator=torch.Generator(device="cuda").manual_seed(1))
    models = {}
    for label, kind in (("none", None), ("Agnesi", "Agnesi")):
        torch.manual_seed(0)
        m = hb.create_model(**dict(ARCH[name], distance_transform=kind))
        with torch.no_grad():
            m(d)                            # creates the concat_node projector before the optimizer flattens the parameters
        model = hb.get_distributed_model(m)
        models[label] = (model, hb.FlatAdamW(model, lr=1e-3))

    def step(label):
        model, opt = models[label]
        return lambda: hb.train_step(model, opt, d, compute_grad_energy=True)
    for label in models:
        for _ in range(2):
            step(label)()
    torch.cuda.synchronize()
    ms = alternate({k: step(k) for k in models}, steps)
    return {"graphs": graphs, "atoms": int(d.pos.shape[0]), "edges": int(d.edge_index.shape[1]),
            "step_ms": {k: round(v, 3) for k, v in ms.items()}, "overhead_vs_none": round(ms["Agnesi"] / ms["none"] - 1.0, 4)}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--graphs", type=int, default=256)
    ap.add_argument("--mlip-graphs", type=int, default=64)
    ap.add_argument("--steps", type=int, default=20)
    args = ap.parse_args()
    torch.cuda.set_device(0)
    res = {**card(), "edge_embed_oc20_mace": edge_embed(args.graphs, args.steps * 10),
           "mlip_step_gfm_mace": mlip_steps(args.mlip_graphs, args.steps)}
    print(json.dumps(res))


if __name__ == "__main__":
    main()
