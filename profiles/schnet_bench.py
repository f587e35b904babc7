"""SchNet timing on the qm9_schnet / md17_schnet / ci_schnet workloads (hydragnn_b200/synthetic.py), one GPU.

    python profiles/schnet_bench.py [--graphs 1024] [--steps 20] [--warmup 5]

Prints one JSON line per workload with the card name and power limit beside every number:
* full training steps (FlatAdamW, eager: SchNet does not take the padded captured step), CUDA events: warm-up, then three timed
  regions of ``--steps`` steps; the median region;
* one CFConv layer (forward + backward) fused vs composed, alternated in the same call;
* the fused pair alone (``ops.CfConvFn`` forward, then its backward), CUDA events, with its algorithmic bytes computed from the
  shapes and the achieved share of the 3.35 TB/s H100 SXM data-sheet bound:
    fwd  E (4 + 4 + 12 + 4 D + 4 NF) + N (4 + 12 + 4 NF)       source id, CSR slot, source position, raw edge input, xl[j];
                                                              rowptr, target position, out[i]
    bwd  E (8 + 24 + 8 D + 12 NF + 4)                         ids, both positions, r and g_r, g_out[i] / xl[j] / g_xl_e, g_d
  Each gathered row is counted once per edge (re-reads are L2 hits while xl fits in L2); the staged weights and the per-CTA
  partials are a few hundred kB and left out.
"""
import argparse
import json
import os
import statistics
import sys

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.dirname(HERE))
sys.path.insert(0, HERE)
import torch  # noqa: E402

import hydragnn_b200 as hb  # noqa: E402
from hydragnn_b200 import ops  # noqa: E402
from hydragnn_b200.synthetic import ARCH, WORKLOADS, add_rel_pe, make_samples  # noqa: E402
from pna_bench import HBM_BOUND, card, timed  # noqa: E402

WORKLOAD_NAMES = ["qm9_schnet", "md17_schnet", "ci_schnet"]


def batch(name, graphs):
    w = WORKLOADS[name]
    b = make_samples(name, graphs).to("cuda")
    b._num_graphs = graphs
    b = hb.get_radius_graph(w["radius"], w["max_neighbours"])(b)
    if ARCH[name].get("global_attn_engine"):
        add_rel_pe(b)
    return b


def layer_bench(name, b, steps):
    """First conv of the model: its CFConv forward + backward, fused and composed, alternated; then the fused pair alone."""
    m = hb.create_model(**ARCH[name]).train()
    seq = m.graph_convs[0]
    seq = getattr(seq, "conv", seq)
    conv = seq.module_2 if hasattr(seq, "module_2") else seq.module_0
    smear = m.distance_expansion
    plan = ops.EdgePlan(b.edge_index, b.pos.shape[0])
    nf, fin = conv.lin1.out_features, conv.lin1.in_features
    x = torch.randn(b.pos.shape[0], fin, device="cuda", requires_grad=True)
    d_raw = 0
    edge_raw = None
    if m.use_global_attn:
        edge_raw, d_raw = (b.rel_pe, m.rel_pos_emb.weight), b.rel_pe.shape[1]
    fused_ok = conv.fused_ok
    kernel_ok = (lambda x_, g_, d_: ops.cfconv_supported(g_, nf, d_))      # the kernels at every width they take

    def run(fused):
        conv.fused_ok = kernel_ok if fused else (lambda *a: False)
        out, _ = conv(x, b.pos, plan, smear, edge_raw)
        out.sum().backward()

    for fused in (True, False):
        run(fused)
    t_f, t_c = [], []
    for _ in range(3):
        t_f += timed(lambda: run(True), steps, 1)
        t_c += timed(lambda: run(False), steps, 1)
    conv.fused_ok = fused_ok
    # the fused pair alone
    xl = torch.randn(b.pos.shape[0], nf, device="cuda", requires_grad=True)
    g, w1 = smear.offset.numel(), conv.nn[0].weight
    a1t = w1[:, :g].t().contiguous() if d_raw == 0 else torch.cat([w1[:, :g].t(), torch.randn(d_raw, nf, device="cuda")]).contiguous()
    r = b.rel_pe.contiguous() if d_raw else None
    args = (xl, b.pos, r, a1t, conv.nn[0].bias, conv.nn[2].weight, conv.nn[2].bias, smear.offset, smear.coeff, conv.cutoff, plan,
            False)
    out, _ = ops.CfConvFn.apply(*args)
    gout = torch.randn_like(out)
    fwd = timed(lambda: ops.CfConvFn.apply(*args), steps)
    bwd_total = timed(lambda: torch.autograd.grad(ops.CfConvFn.apply(*args)[0], [xl, conv.nn[2].weight], gout), steps)
    t_fwd = statistics.median(fwd)
    t_bwd = max(statistics.median(bwd_total) - t_fwd, 1e-9)
    n, e = b.pos.shape[0], plan.num_edges
    by_fwd = e * (4 + 4 + 12 + 4 * d_raw + 4 * nf) + n * (4 + 12 + 4 * nf)
    by_bwd = e * (8 + 24 + 8 * d_raw + 12 * nf + 4)
    return {"layer_fused_ms": statistics.median(t_f), "layer_composed_ms": statistics.median(t_c),
            "cfconv_fwd_ms": t_fwd, "cfconv_bwd_ms": t_bwd,
            "bytes_per_edge_fwd": by_fwd / e, "bytes_per_node_fwd": 4 + 12 + 4 * nf, "bytes_per_edge_bwd": by_bwd / e,
            "fwd_hbm_share": by_fwd / (t_fwd * 1e-3) / HBM_BOUND, "bwd_hbm_share": by_bwd / (t_bwd * 1e-3) / HBM_BOUND,
            "num_filters": nf, "num_gaussians": g, "raw_edge_width": d_raw}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--workload", nargs="*", default=WORKLOAD_NAMES, choices=WORKLOAD_NAMES)
    ap.add_argument("--graphs", type=int, default=1024)
    ap.add_argument("--steps", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=5)
    a = ap.parse_args()
    assert torch.cuda.is_available(), "schnet_bench needs a GPU"
    c = card()
    for name in a.workload:
        b = batch(name, a.graphs)
        model = hb.get_distributed_model(hb.create_model(**ARCH[name]))
        opt = hb.FlatAdamW(model, lr=1e-4)
        for _ in range(a.warmup):
            hb.train_step(model, opt, b)
        step = timed(lambda: hb.train_step(model, opt, b), a.steps)
        ms = statistics.median(step)
        res = dict(c, workload=name, graphs=a.graphs, atoms=int(b.pos.shape[0]), edges=int(b.edge_index.shape[1]),
                   step_ms=ms, step_regions_ms=step, atoms_per_s=b.pos.shape[0] / (ms * 1e-3))
        res.update(layer_bench(name, b, a.steps))
        print(json.dumps(res))


if __name__ == "__main__":
    main()
