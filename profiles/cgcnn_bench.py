"""CGCNN timing on the mp_cgcnn / mp_cgcnn_gps workloads (hydragnn_b200/synthetic.py), one GPU.

    python profiles/cgcnn_bench.py --workload mp_cgcnn [--graphs 512] [--steps 20] [--sweep]

Prints one JSON line with the card name and power limit beside every number:
* full training steps (FlatAdamW, graph head, eager), CUDA events: warm-up, then three timed regions of ``--steps`` steps; the
  median region, and atoms/s;
* one CGConv layer (forward + backward) at the width the workload's convs run at, fused vs composed, alternated in the same
  call, with the rel-L2 agreement of the two layer outputs and input gradients;
* the fused kernels' algorithmic bytes and FLOPs per layer and their achieved share of the bound that applies (the larger of
  bytes / 3.35 TB/s and FLOPs / 67 TFLOP/s FP32, the H100 SXM data-sheet figures), from the layer times above.  With N atoms,
  E edges, F channels and D the raw edge width:
    fwd bytes  4 (4 N F + E (2 F + D + 2) + N + 1) + 4 (2 N F)      pq [N, 4F] read once, Q rows gathered per edge, a_e, source
                                                                      id and CSR slot; x read and out written
    fwd FLOPs  E F (4 D + 4 + 2 * 10)                                 both pre-activations, the gate and the sum; sigmoid and
                                                                      softplus counted as 10 each
    bwd bytes  the forward's reads + 4 (N F + 2 N F + 2 E F + E D)   g_out, g_P, g_h [E, 2F], g_eattr
    bwd FLOPs  the forward's, plus E F (10 + 8 D + 6)                 the gate's derivatives, g_eattr = g_h Mt^T, g_Mt
  The by-source segment sum of g_h and the per-node Linear are not counted (they run on their own kernels).
* with ``--sweep``: the same layer comparison at F = 1, 2, 4, 8, 16, 32, 64 and 128 on the workload's graph, with its raw edge
  width.
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
from hydragnn_b200.cgcnn import CGConv  # noqa: E402
from hydragnn_b200.synthetic import ARCH, WORKLOADS, add_rel_pe, make_samples  # noqa: E402
from pna_bench import card, timed  # noqa: E402

HBM_BOUND, FP32_BOUND = 3.35e12, 67e12


def batch(name, graphs):
    w = WORKLOADS[name]
    b = make_samples(name, graphs).to("cuda")
    b._num_graphs = graphs
    b = hb.get_radius_graph_pbc(w["radius"], w["max_neighbours"])(b)
    b.edge_attr = (b.pos[b.edge_index[1]] - b.pos[b.edge_index[0]] + b.edge_shifts).norm(dim=1, keepdim=True).contiguous()
    if w.get("pe_dim"):
        b = add_rel_pe(b)
    return b


def layer_compare(conv, x, plan, edge_raw, steps, warmup):
    g = torch.randn(x.shape[0], conv.channels, device=x.device)

    def run(composed):
        y = conv(x, plan, edge_raw, higher_order=composed)
        (gx,) = torch.autograd.grad(y, x, g)
        return y, gx

    yf, gf = (t.detach() for t in run(False))
    yc, gc = (t.detach() for t in run(True))
    rel = lambda u, v: float((u.double() - v.double()).norm() / v.double().norm())                   # noqa: E731
    for _ in range(warmup):
        run(False), run(True)
    fused, composed = [], []
    for _ in range(3):
        fused += timed(lambda: run(False), steps, 1)
        composed += timed(lambda: run(True), steps, 1)
    return {"fused_ms": statistics.median(fused), "composed_ms": statistics.median(composed), "fused_ms_regions": fused,
            "composed_ms_regions": composed, "out_rel_l2": rel(yf, yc), "grad_rel_l2": rel(gf, gc)}


def layer_model(n, e, f, d):
    fwd_bytes = 4 * (4 * n * f + e * (2 * f + d + 2) + n + 1) + 4 * 2 * n * f
    fwd_flops = e * f * (4 * d + 4 + 20)
    bwd_bytes = fwd_bytes + 4 * (n * f + 2 * n * f + 2 * e * f + e * d)
    bwd_flops = fwd_flops + e * f * (10 + 8 * d + 6)
    return fwd_bytes, fwd_flops, bwd_bytes, bwd_flops


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--workload", default="mp_cgcnn", choices=["mp_cgcnn", "mp_cgcnn_gps"])
    ap.add_argument("--graphs", type=int, default=512)
    ap.add_argument("--steps", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=5)
    ap.add_argument("--sweep", action="store_true")
    a = ap.parse_args()
    torch.cuda.set_device(0)
    arch = ARCH[a.workload]
    b = batch(a.workload, a.graphs)
    n, e = b.pos.shape[0], b.edge_index.shape[1]
    res = {"workload": a.workload, "graphs": a.graphs, "atoms": n, "edges": e, **card()}

    model = hb.get_distributed_model(hb.create_model(**arch))
    opt = hb.FlatAdamW(model, lr=1e-3)
    hi = [torch.arange(b.y.shape[0], device="cuda")]
    step = lambda: hb.train_step(model, opt, b, head_index=hi)                                       # noqa: E731
    for _ in range(a.warmup):
        step()
    torch.cuda.synchronize()
    regions = timed(step, a.steps)
    ms = statistics.median(regions)
    res.update(step_ms_regions=regions, step_ms=ms, atoms_per_s=n / ms * 1e3)

    inner = model.module
    plan = inner.plan_for(b)
    with torch.no_grad():
        _, _, conv_args = inner._embedding(b, plan, False)
    edge_raw = tuple(t.detach() if t is not None else None for t in conv_args["edge_raw"])
    conv = inner.graph_convs[-1]
    conv = getattr(conv, "conv", conv).module_0
    f, d = conv.channels, edge_raw[0].shape[1]
    x = torch.randn(n, f, device="cuda", requires_grad=True)
    res["conv"] = layer_compare(conv, x, plan, edge_raw, a.steps, a.warmup)
    fb, ff, bb, bf = layer_model(n, e, f, d)
    t = res["conv"]["fused_ms"] * 1e-3
    mem, alu = (fb + bb) / HBM_BOUND, (ff + bf) / FP32_BOUND
    res["fused_layer_model"] = {"channels": f, "raw_edge_width": d, "fwd_bytes": fb, "fwd_flops": ff, "bwd_bytes": bb,
                                "bwd_flops": bf, "bound": "fp32" if alu > mem else "hbm", "share_of_bound": max(mem, alu) / t}

    if a.sweep:
        res["sweep"] = {}
        for w in (1, 2, 4, 8, 16, 32, 64, 128):
            torch.manual_seed(0)
            cw = CGConv(w, conv.dim).cuda()
            xw = torch.randn(n, w, device="cuda", requires_grad=True)
            res["sweep"][w] = layer_compare(cw, xw, plan, edge_raw, a.steps, a.warmup)
            fb, ff, bb, bf = layer_model(n, e, w, d)
            res["sweep"][w]["share_of_bound"] = max((fb + bb) / HBM_BOUND, (ff + bf) / FP32_BOUND) / (res["sweep"][w]["fused_ms"] * 1e-3)
    print(json.dumps(res))


if __name__ == "__main__":
    main()
