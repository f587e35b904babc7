"""PNAPlus timing on the lj_pnaplus / ogb_pnaplus workloads (hydragnn_b200/synthetic.py), one GPU.

    python profiles/pnaplus_bench.py --workload lj_pnaplus [--graphs 512] [--steps 20] [--sweep]

Prints one JSON line with the card name and power limit beside every number:
* full training steps (FlatAdamW; lj_pnaplus with its energy + per-atom energy + force loss, which runs the composed any-order
  path), CUDA events: warm-up, then three timed regions of ``--steps`` steps; the median region;
* one PNAPlus conv layer (forward + backward) at the workload's hidden width, fused vs composed, alternated in the same call,
  with the rel-L2 agreement of the two layer outputs and input gradients;
* the fused kernels' algorithmic bytes and FLOPs per layer and their achieved share of the bound that applies (the larger of
  bytes / 3.35 TB/s and FLOPs / 67 TFLOP/s FP32, the H100 SXM data-sheet figures), from the layer times above:
    fwd bytes  4 (2 N F + E (D + 3) + N + 1) + N (16 F + 8 F)   [P | Q], d_e, edge input, source ids / CSR; agg and the ids
    fwd FLOPs  E (2 F^2 + 4 R F + 2 D F + 2 F + 2 F) + 20 E R    M_r u, W_r rbf / W_l rbf, M_a a, P + Q, gate; the basis
    bwd        the forward recomputed, plus 2 F^2 (g_u) + 2 F^2 (g_M_r) + 8 R F + 4 D F per edge, g_h [E, F] and g_dist written
* with ``--sweep``: the same layer comparison at widths 16, 32, 48 and 64 on the workload's graph (the fused width limit).
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
from hydragnn_b200.pnaplus import PNAConv  # noqa: E402
from hydragnn_b200.synthetic import ARCH, WORKLOADS, make_samples  # noqa: E402
from pna_bench import card, timed  # noqa: E402

HBM_BOUND, FP32_BOUND = 3.35e12, 67e12


def batch(name, graphs):
    w = WORKLOADS[name]
    b = make_samples(name, graphs).to("cuda")
    b._num_graphs = graphs
    build = hb.get_radius_graph_pbc if (w.get("pbc") or w.get("pbc_box")) else hb.get_radius_graph
    b = build(w["radius"], w["max_neighbours"])(b)
    deg = torch.bincount(torch.bincount(b.edge_index[1], minlength=b.pos.shape[0])).tolist()
    return b, deg


def layer_compare(conv, x, plan, bessel, ea, steps, warmup):
    g = torch.randn(x.shape[0], conv.F_out, device=x.device)

    def run(composed):
        y = conv(x, plan, dict(bessel, rbf=None), ea, higher_order=composed)
        (gx,) = torch.autograd.grad(y, x, g)
        return y, gx

    yf, gf = run(False)
    yc, gc = run(True)
    rel = lambda u, v: float((u.double() - v.double()).norm() / v.double().norm())                   # noqa: E731
    for _ in range(warmup):
        run(False), run(True)
    fused, composed = [], []
    for _ in range(3):
        fused += timed(lambda: run(False), steps, 1)
        composed += timed(lambda: run(True), steps, 1)
    return {"fused_ms": statistics.median(fused), "composed_ms": statistics.median(composed), "fused_ms_regions": fused,
            "composed_ms_regions": composed, "out_rel_l2": rel(yf, yc), "grad_rel_l2": rel(gf, gc)}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--workload", default="lj_pnaplus", choices=["lj_pnaplus", "ogb_pnaplus"])
    ap.add_argument("--graphs", type=int, default=512)
    ap.add_argument("--steps", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=5)
    ap.add_argument("--sweep", action="store_true")
    a = ap.parse_args()
    torch.cuda.set_device(0)
    arch = ARCH[a.workload]
    b, deg = batch(a.workload, a.graphs)
    n, e = b.pos.shape[0], b.edge_index.shape[1]
    res = {"workload": a.workload, "graphs": a.graphs, "atoms": n, "edges": e, **card()}

    model = hb.get_distributed_model(hb.create_model(**dict(arch, pna_deg=deg)))
    opt = hb.FlatAdamW(model, lr=1e-3)
    mlip = bool(arch.get("enable_interatomic_potential"))
    hi = [torch.arange(b.y.shape[0], device="cuda")]
    step = (lambda: hb.train_step(model, opt, b, compute_grad_energy=True)) if mlip else \
        (lambda: hb.train_step(model, opt, b, head_index=hi))                                        # noqa: E731
    for _ in range(a.warmup):
        step()
    torch.cuda.synchronize()
    regions = timed(step, a.steps)
    ms = statistics.median(regions)
    res.update(step_ms_regions=regions, step_ms=ms, atoms_per_s=n / ms * 1e3, step_loss="energy+forces" if mlip else "head")

    inner = getattr(model.module, "model", model.module)
    plan = inner.plan_for(b)
    dist = hb.ops.EdgeLenFn.apply(b.pos, b.edge_shifts, plan).detach()
    bessel = {"basis": inner.rbf, "dist": dist, "rbf": None}
    f, r, d = inner.hidden_dim, inner.num_radial, 0
    x = torch.randn(n, f, device="cuda", requires_grad=True)
    res["conv"] = layer_compare(inner.graph_convs[1].module_0, x, plan, bessel, None, a.steps, a.warmup)

    fwd_bytes = 4 * (2 * n * f + e * (d + 3) + n + 1) + n * 24 * f
    fwd_flops = e * (2 * f * f + 4 * r * f + 2 * d * f + 4 * f) + 20 * e * r
    bwd_bytes = fwd_bytes + 4 * n * 10 * f + 4 * e * f + 4 * n * f + 4 * e
    bwd_flops = fwd_flops + e * (4 * f * f + 8 * r * f + 4 * d * f)
    t = res["conv"]["fused_ms"] * 1e-3
    bound = max((fwd_bytes + bwd_bytes) / HBM_BOUND, (fwd_flops + bwd_flops) / FP32_BOUND)
    res["fused_layer_model"] = {"fwd_bytes": fwd_bytes, "fwd_flops": fwd_flops, "bwd_bytes": bwd_bytes, "bwd_flops": bwd_flops,
                                "bound": "fp32" if (fwd_flops + bwd_flops) / FP32_BOUND > (fwd_bytes + bwd_bytes) / HBM_BOUND else "hbm",
                                "share_of_bound": bound / t}

    if a.sweep:
        res["sweep"] = {}
        for w in (16, 32, 48, 64):
            torch.manual_seed(0)
            conv = PNAConv(w, w, inner.aggregators, inner.scalers, inner.deg, num_radial=r).cuda()
            xw = torch.randn(n, w, device="cuda", requires_grad=True)
            res["sweep"][w] = layer_compare(conv, xw, plan, bessel, None, a.steps, a.warmup)
    print(json.dumps(res))


if __name__ == "__main__":
    main()
