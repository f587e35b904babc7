"""GAT timing on the ogb_gat / ogb_gat_gps workloads (hydragnn_b200/synthetic.py), one GPU.

    python profiles/gat_bench.py --workload ogb_gat [--graphs 512] [--steps 20] [--sweep]

Prints one JSON line with the card name and power limit beside every number:
* full training steps (FlatAdamW, graph head, eager, attention dropout on), CUDA events: warm-up, then three timed regions of
  ``--steps`` steps; the median region, and atoms/s;
* one GATv2Conv layer (the workload's middle conv: lin_l / lin_r Linear, the attention kernels, forward + backward), fused vs
  composed, alternated in the same call, with the rel-L2 agreement of the two layer outputs and input gradients; and the fused
  forward alone;
* the fused forward's algorithmic bytes and its achieved bytes/s from the forward time above.  With N atoms, E edges, H heads,
  C channels per head and D the raw edge width:
    fwd bytes  4 (2 N H C + E (H C + D + 2) + N + 1) + 4 (N H C' + N H)    x_l / x_r read once per target, one x_l row, D
                                                                            attributes, the source id and the CSR slot per edge;
                                                                            out (C' = C concat, C / H mean) and the log-sum-exp
  The lin_l / lin_r Linear is not counted (it runs on its own kernel).
* with ``--sweep``: the same layer comparison at H = 6 and C = 1, 4, 8, 16, 32, 64 on the workload's graph and raw edge width.
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
from hydragnn_b200.gat import GATv2Conv  # noqa: E402
from hydragnn_b200.synthetic import ARCH, WORKLOADS, add_rel_pe  # noqa: E402
from pna_bench import batch as pna_batch, card, timed  # noqa: E402

HBM_BOUND = 3.35e12


def batch(name, graphs):
    """The workload's open-boundary radius graphs with the edge length as the edge attribute (and rel_pe under GPS)."""
    b, _ = pna_batch(name, graphs)
    return add_rel_pe(b) if WORKLOADS[name].get("pe_dim") else b


def layer_compare(conv, x, plan, edge_raw, steps, warmup):
    out_w = conv.heads * conv.out_channels if conv.concat else conv.out_channels
    g = torch.randn(x.shape[0], out_w, device=x.device)

    def run(composed):
        y = conv(x, plan, edge_raw, higher_order=composed)
        (gx,) = torch.autograd.grad(y, x, g)
        return y, gx

    def fwd():
        with torch.no_grad():
            return conv(x, plan, edge_raw)

    yf, gf = (t.detach() for t in run(False))
    yc, gc = (t.detach() for t in run(True))
    rel = lambda u, v: float((u.double() - v.double()).norm() / v.double().norm())                   # noqa: E731
    for _ in range(warmup):
        run(False), run(True), fwd()
    fused, composed, fwd_only = [], [], []
    for _ in range(3):
        fused += timed(lambda: run(False), steps, 1)
        composed += timed(lambda: run(True), steps, 1)
        fwd_only += timed(fwd, steps, 1)
    return {"fused_ms": statistics.median(fused), "composed_ms": statistics.median(composed),
            "fused_fwd_ms": statistics.median(fwd_only), "fused_ms_regions": fused, "composed_ms_regions": composed,
            "out_rel_l2": rel(yf, yc), "grad_rel_l2": rel(gf, gc)}


def fwd_bytes(n, e, heads, c, d, concat):
    return 4 * (2 * n * heads * c + e * (heads * c + d + 2) + n + 1) + 4 * (n * (heads * c if concat else c) + n * heads)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--workload", default="ogb_gat", choices=["ogb_gat", "ogb_gat_gps"])
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
    conv = inner.graph_convs[1]
    conv = getattr(conv, "conv", conv).module_0.eval()                    # the layer comparison runs without dropout
    d = edge_raw[0].shape[1]
    x = torch.randn(n, conv.in_channels, device="cuda", requires_grad=True)
    res["conv"] = layer_compare(conv, x, plan, edge_raw, a.steps, a.warmup)
    fb = fwd_bytes(n, e, conv.heads, conv.out_channels, d, conv.concat)
    res["fused_fwd_model"] = {"heads": conv.heads, "channels": conv.out_channels, "in_channels": conv.in_channels,
                              "raw_edge_width": d, "fwd_bytes": fb,
                              "fwd_bytes_per_s": fb / (res["conv"]["fused_fwd_ms"] * 1e-3),
                              "share_of_hbm": fb / HBM_BOUND / (res["conv"]["fused_fwd_ms"] * 1e-3)}
    if a.sweep:
        res["sweep"] = {}
        for c in (1, 4, 8, 16, 32, 64):
            torch.manual_seed(0)
            cw = GATv2Conv(64, c, heads=6, concat=True, negative_slope=0.05, edge_dim=conv.edge_dim).cuda().eval()
            xw = torch.randn(n, 64, device="cuda", requires_grad=True)
            emb = edge_raw[1]
            if emb is not None and cw.edge_dim != emb.shape[0]:
                emb = None
            r = layer_compare(cw, xw, plan, (edge_raw[0], emb), a.steps, a.warmup)
            fbw = fwd_bytes(n, e, 6, c, d, True)
            r["fwd_bytes_per_s"] = fbw / (r["fused_fwd_ms"] * 1e-3)
            res["sweep"][c] = r
    print(json.dumps(res))


if __name__ == "__main__":
    main()
