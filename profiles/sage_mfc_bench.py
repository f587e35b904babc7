"""SAGE / MFC timing on the ogb_sage, ogb_mfc and ogb_sage_gps workloads (hydragnn_b200/synthetic.py), one GPU.

    python profiles/sage_mfc_bench.py --workload ogb_mfc [--graphs 512] [--steps 20] [--sweep]

Prints one JSON line with the card name and power limit beside every number:
* full training steps (FlatAdamW, graph head, eager), CUDA events: warm-up, then three timed regions of ``--steps`` steps; the
  median region, and atoms/s;
* the same step without the optimizer (model forward, loss and parameter gradients), and the parameter count: MFC keeps
  max_degree + 1 weight pairs per layer, so its optimizer and gradient buffers are that many times larger;
* one conv layer (forward + backward) at the width the workload's convs run at, fused (ops.NbrLinearFn) vs the first-order
  composed path (ops.nbr_linear_composed: GatherRows / SegmentSum, linear_act or the grouped Linear) that shapes the kernel does
  not take run, alternated in the same call, with the rel-L2 agreement of the two layer outputs and input gradients;
* the fused layer's algorithmic bytes and FLOPs and its achieved share of the bound that applies (the larger of bytes / 3.35 TB/s
  and FLOPs / 495 TFLOP/s TF32 -- a third of that in the fp32 mode's 3xTF32 -- the H100 SXM data-sheet figures), from the layer
  times above.  With N atoms, E edges, k input and n output channels, kp = k rounded up to 32:
    fwd bytes  4 (E k + E + 2 N + N k + N n + 2 N kp)   neighbour rows gathered per edge, source ids, CSR offsets, root rows,
                                                         out, the stored [h | x] operand of the weight gradient
    fwd FLOPs  E k + 4 N n kp                          the neighbour sum and the [h | x] product
    bwd bytes  4 (N n + 2 N k + E k + E + 3 N k + N n + 2 N kp)   g_out, [g_h | g_x root], the by-source gather of g_h, g_x,
                                                         and the weight gradient's reads of g_out and [h | x]
    bwd FLOPs  8 N n kp + E k                          data and weight products, the segment sum
* with ``--sweep``: the same comparison at k = n = 1, 2, 4, 8, 16, 32, 64 and 128 on the workload's graph, and (MFC) at
  max_degree 5, 20 and 100 with the time of the weight-gradient kernel alone.
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
from hydragnn_b200 import _lib  # noqa: E402
from hydragnn_b200.sage import MFConv, SAGEConv  # noqa: E402
from hydragnn_b200.synthetic import ARCH, WORKLOADS, add_rel_pe, make_samples  # noqa: E402
from pna_bench import card, timed  # noqa: E402

HBM_BOUND, TF32_BOUND = 3.35e12, 495e12


def batch(name, graphs):
    w = WORKLOADS[name]
    b = make_samples(name, graphs).to("cuda")
    b._num_graphs = graphs
    b = hb.get_radius_graph(w["radius"], w["max_neighbours"])(b)
    if w.get("pe_dim"):
        b = add_rel_pe(b)
    return b


def weights(conv):
    """(wl, bl, wr, mean) of a SAGEConv / MFConv in the layout ops.NbrLinearFn and ops.nbr_linear_composed take."""
    if isinstance(conv, SAGEConv):
        return conv.lin_l.weight[None], conv.lin_l.bias[None], conv.lin_r.weight[None], True
    return (torch.stack([lin.weight for lin in conv.lins_l]), torch.stack([lin.bias for lin in conv.lins_l]),
            torch.stack([lin.weight for lin in conv.lins_r]), False)


def layer_compare(conv, x, plan, dp, steps, warmup):
    g = torch.randn(x.shape[0], conv.out_channels, device=x.device)

    def run(composed):
        wl, bl, wr, mean = weights(conv)
        if composed:
            y = hb.ops.nbr_linear_composed(x, wl, bl, wr, dp, plan, mean, higher_order=False)
        else:
            y = hb.ops.NbrLinearFn.apply(x, wl, bl, wr, dp, plan, mean)
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


def grouped_wgrad_ms(dp, n, k, no, steps):
    """The layer's weight-gradient kernel alone (hgb_grouped_wgrad over the degree-ordered [h | x] rows): one CTA per (group,
    64 x 64 tile of dW) walks all of its group's rows, so its time follows the largest group."""
    kp = (k + 31) // 32 * 32
    dy, hx = torch.randn(n, no, device="cuda"), torch.randn(n, 2 * kp, device="cuda")
    dw = torch.empty(dp.groups, no, 2 * kp, device="cuda")
    db = torch.empty(dp.groups, no, device="cuda")
    P = hb.ops._p
    call = lambda: _lib.call("hgb_grouped_wgrad", P(dy), P(hx), 2 * kp, P(dp.grp_ptr), dp.groups, n, no, 2 * kp, P(dw), P(db),  # noqa: E731
                                hb.ops._stream())
    call()
    return statistics.median(timed(call, steps))


def layer_model(n, e, k, no):
    kp = (k + 31) // 32 * 32
    fb = 4 * (e * k + e + 2 * n + n * k + n * no + 2 * n * kp)
    ff = e * k + 4 * n * no * kp
    bb = 4 * (n * no + 2 * n * k + e * k + e + 3 * n * k + n * no + 2 * n * kp)
    bf = 8 * n * no * kp + e * k
    return fb, ff, bb, bf


def share(res, n, e, k, no, exact):
    fb, ff, bb, bf = layer_model(n, e, k, no)
    t = res["fused_ms"] * 1e-3
    mem, alu = (fb + bb) / HBM_BOUND, (ff + bf) / (TF32_BOUND / (3 if exact else 1))
    return {"fwd_bytes": fb, "fwd_flops": ff, "bwd_bytes": bb, "bwd_flops": bf, "bound": "tensor" if alu > mem else "hbm",
            "share_of_bound": max(mem, alu) / t}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--workload", default="ogb_sage", choices=["ogb_sage", "ogb_mfc", "ogb_sage_gps"])
    ap.add_argument("--graphs", type=int, default=512)
    ap.add_argument("--steps", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=5)
    ap.add_argument("--sweep", action="store_true")
    a = ap.parse_args()
    torch.cuda.set_device(0)
    arch = ARCH[a.workload]
    b = batch(a.workload, a.graphs)
    n, e = b.pos.shape[0], b.edge_index.shape[1]
    res = {"workload": a.workload, "graphs": a.graphs, "atoms": n, "edges": e, "precision": "fp32", **card()}

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
    params = list(model.parameters())
    res["parameters"] = sum(p.numel() for p in params)

    def fwd_bwd():
        loss, _ = model.module.loss(model(b), b.y.view(-1), hi)
        torch.autograd.grad(loss, params, allow_unused=True)
    for _ in range(a.warmup):
        fwd_bwd()
    fb_regions = timed(fwd_bwd, a.steps)
    res.update(fwd_bwd_ms_regions=fb_regions, fwd_bwd_ms=statistics.median(fb_regions))

    inner = model.module
    plan = inner.plan_for(b)
    with torch.no_grad():
        _, _, conv_args = inner._embedding(b, plan, False)
    dp = conv_args["degree_plan"]
    conv = inner.graph_convs[-1]
    conv = getattr(conv, "conv", conv).module_0
    k, no = conv.in_channels, conv.out_channels
    x = torch.randn(n, k, device="cuda", requires_grad=True)
    res["conv"] = layer_compare(conv, x, plan, dp, a.steps, a.warmup)
    res["fused_layer_model"] = dict(in_channels=k, out_channels=no, **share(res["conv"], n, e, k, no, True))

    if a.sweep:
        res["sweep"] = {}
        for w in (1, 2, 4, 8, 16, 32, 64, 128):
            torch.manual_seed(0)
            cw = (SAGEConv(w, w) if isinstance(conv, SAGEConv) else MFConv(w, w, conv.max_degree)).cuda()
            xw = torch.randn(n, w, device="cuda", requires_grad=True)
            r = layer_compare(cw, xw, plan, dp, a.steps, a.warmup)
            r["share_of_bound"] = share(r, n, e, w, w, True)["share_of_bound"]
            res["sweep"][w] = r
        if isinstance(conv, MFConv):
            res["max_degree_sweep"] = {}
            for md in (5, 20, 100):
                torch.manual_seed(0)
                cw = MFConv(k, no, md).cuda()
                dpm = hb.ops.degree_plan(plan, md + 1)
                res["max_degree_sweep"][md] = layer_compare(cw, x, plan, dpm, a.steps, a.warmup)
                res["max_degree_sweep"][md]["grouped_wgrad_ms"] = grouped_wgrad_ms(dpm, n, k, no, a.steps)
    print(json.dumps(res))


if __name__ == "__main__":
    main()
