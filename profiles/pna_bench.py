"""PNA timing on the eam_pna / ogb_pna workloads (hydragnn_b200/synthetic.py), one GPU.

    python profiles/pna_bench.py --workload eam_pna [--graphs 512] [--steps 20] [--profile]

Prints one JSON line with the card name and power limit beside every number:
* full training steps (FlatAdamW), CUDA events: warm-up, then three timed regions of ``--steps`` steps; the median region;
* one PNAConv layer (forward + backward) fused vs composed, alternated in the same call, with the rel-L2 agreement of the two
  layer outputs and input gradients at that size;
* with ``--profile``: one profiled step (torch.profiler, a separate pass after the timing) for the kernel shares, and the two
  fused kernels' achieved bytes/s (mean call vs the mean layer's bytes) against the 3.35 TB/s H100 SXM data-sheet bound, from
  their algorithmic bytes per layer of input width F:
    fwd  4 (2 N F + E (D + 2) + N + 1) + N (16 F + 8 F)     read [P | Q] once, edge attributes, source ids / CSR;
                                                            write agg [N, 4F] and the two id arrays
    bwd  fwd + 4 N (4F + 4F + 2F) + 4 E F + 4 N F           plus g_agg, agg and the ids read; g_h and g_P written
  Q is gathered once per edge; the formula counts each row once (the re-reads are L2 hits while [N, 2F] fits in L2).
"""
import argparse
import json
import os
import statistics
import subprocess
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import torch  # noqa: E402

import hydragnn_b200 as hb  # noqa: E402
from hydragnn_b200.synthetic import ARCH, WORKLOADS, make_samples  # noqa: E402

HBM_BOUND = 3.35e12


def card():
    """Card name and power limit: NVML first, then the read-only ``nvidia-smi --query-gpu=power.limit`` query; if neither
    answers, the limit is reported as the string "not read"."""
    name, limit, source = torch.cuda.get_device_name(), None, None
    try:
        import pynvml
        pynvml.nvmlInit()
        h = pynvml.nvmlDeviceGetHandleByIndex(torch.cuda.current_device())
        limit, source = pynvml.nvmlDeviceGetPowerManagementLimit(h) / 1000.0, "NVML"
    except Exception:  # noqa: BLE001 -- fall through to nvidia-smi
        try:
            out = subprocess.run(["nvidia-smi", "--query-gpu=power.limit", "--format=csv,noheader,nounits",
                                  "-i", str(torch.cuda.current_device())], capture_output=True, text=True, timeout=30)
            limit, source = float(out.stdout.strip().splitlines()[0]), "nvidia-smi"
        except Exception:  # noqa: BLE001 -- said plainly below
            pass
    return {"gpu": name, "power_limit_w": limit if limit is not None else "not read", "power_limit_source": source}


def batch(name, graphs):
    w = WORKLOADS[name]
    b = make_samples(name, graphs).to("cuda")
    b._num_graphs = graphs
    build = hb.get_radius_graph_pbc if w.get("pbc_box") else hb.get_radius_graph
    b = build(w["radius"], w["max_neighbours"])(b)
    if ARCH[name].get("edge_dim"):
        vec = b.pos[b.edge_index[1]] - b.pos[b.edge_index[0]]
        if getattr(b, "edge_shifts", None) is not None:
            vec = vec + b.edge_shifts
        b.edge_attr = vec.norm(dim=1, keepdim=True).detach().contiguous()
    deg = torch.bincount(torch.bincount(b.edge_index[1], minlength=b.pos.shape[0])).tolist()
    return b, deg


def timed(fn, steps, regions=3):
    out = []
    for _ in range(regions):
        t0, t1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        t0.record()
        for _ in range(steps):
            fn()
        t1.record()
        torch.cuda.synchronize()
        out.append(t0.elapsed_time(t1) / steps)
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--workload", default="eam_pna", choices=["eam_pna", "ogb_pna"])
    ap.add_argument("--graphs", type=int, default=512)
    ap.add_argument("--steps", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=5)
    ap.add_argument("--profile", action="store_true")
    a = ap.parse_args()
    torch.cuda.set_device(0)
    b, deg = batch(a.workload, a.graphs)
    n, e = b.pos.shape[0], b.edge_index.shape[1]
    res = {"workload": a.workload, "graphs": a.graphs, "atoms": n, "edges": e, **card()}

    model = hb.get_distributed_model(hb.create_model(**dict(ARCH[a.workload], pna_deg=deg)))
    opt = hb.FlatAdamW(model, lr=1e-3)
    if ARCH[a.workload]["output_type"] == ["node"]:
        b.y = torch.randn(n, 1, device="cuda")                 # one per-atom target
    hi = [torch.arange(b.y.shape[0], device="cuda")]
    step = lambda: hb.train_step(model, opt, b, head_index=hi)                                      # noqa: E731
    for _ in range(a.warmup):
        step()
    torch.cuda.synchronize()
    regions = timed(step, a.steps)
    ms = statistics.median(regions)
    res.update(step_ms_regions=regions, step_ms=ms, atoms_per_s=n / ms * 1e3)

    # one conv layer at hidden width (layer 1), fused vs composed, alternated
    inner = model.module
    conv = inner.graph_convs[1].module_0
    plan = inner.plan_for(b)
    f = inner.hidden_dim
    x = torch.randn(n, f, device="cuda", requires_grad=True)
    ea = b.edge_attr if inner.use_edge_attr else None
    g = torch.randn(n, f, device="cuda")

    def layer(composed):
        y = conv(x, plan, ea, higher_order=composed)
        (gx,) = torch.autograd.grad(y, x, g)
        return y, gx

    yf, gf = layer(False)
    yc, gc = layer(True)
    rel = lambda u, v: float((u.double() - v.double()).norm() / v.double().norm())                   # noqa: E731
    fused, composed = [], []
    for _ in range(a.warmup):
        layer(False), layer(True)
    for _ in range(3):
        fused += timed(lambda: layer(False), a.steps, 1)
        composed += timed(lambda: layer(True), a.steps, 1)
    res.update(conv_fused_ms=statistics.median(fused), conv_composed_ms=statistics.median(composed),
               conv_fused_ms_regions=fused, conv_composed_ms_regions=composed,
               conv_out_rel_l2=rel(yf, yc), conv_grad_rel_l2=rel(gf, gc))

    if a.profile:
        d = ARCH[a.workload].get("edge_dim") or 0
        widths = [ARCH[a.workload]["input_dim"]] + [f] * (inner.num_conv_layers - 1)          # per-layer F_in

        def fwd_b(w):
            return 4 * (2 * n * w + e * (d + 2) + n + 1) + n * (16 * w + 8 * w)

        fwd_bytes = sum(fwd_b(w) for w in widths) / len(widths)                                 # mean over the layers
        bwd_bytes = sum(fwd_b(w) + 4 * n * (4 * w + 4 * w + 2 * w) + 4 * e * w + 4 * n * w for w in widths) / len(widths)
        with torch.profiler.profile(activities=[torch.profiler.ProfilerActivity.CUDA]) as prof:
            step()
            torch.cuda.synchronize()
        total, kern = 0.0, {}
        for ev in prof.key_averages():
            t = getattr(ev, "device_time_total", 0.0)
            total += t
            kern[ev.key] = (t, ev.count)
        top = sorted(kern.items(), key=lambda kv: -kv[1][0])[:12]
        res["kernel_shares"] = [{"kernel": k[:70], "share": t / total, "calls": c} for k, (t, c) in top]
        for kind, nbytes in (("fwd", fwd_bytes), ("bwd", bwd_bytes)):
            hits = [(t, c) for k, (t, c) in kern.items() if "pna_conv_%s_kernel" % kind in k]
            if hits:
                us = sum(t for t, _ in hits) / sum(c for _, c in hits)
                res["pna_conv_%s" % kind] = {"us_per_call": us, "algorithmic_bytes_mean_layer": nbytes,
                                             "fraction_of_3.35TB/s": nbytes / (us * 1e-6) / HBM_BOUND}
    print(json.dumps(res))


if __name__ == "__main__":
    main()
