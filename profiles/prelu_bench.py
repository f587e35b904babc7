"""PReLU timing, one GPU.

    python profiles/prelu_bench.py [--graphs 512] [--steps 20]

Prints one JSON line with the card name and power limit beside every number:
* PReLU forward + backward (slope gradient included), ``ops.PReluFn`` (hgb_prelu_fwd + hgb_prelu_bwd, one launch each) against
  ATen's ``torch.nn.functional.prelu`` and its autograd backward, at the sizes of feature layers and node heads (N x 64 and
  N x 12 for N = 1e4 .. 1e6 rows), alternated in the same call (CUDA events, the median of three regions), with their
  agreement and the fused pair's algorithmic bytes (4 B x 5 elements: z read, y written; g and z read, dz written) over its time;
* eager training steps (forward, loss, backward, FlatAdamW) of ARCH["ogb_pna"] (graph head) and of an EGNN with an ``mlp`` node
  head on the md17_egnn graphs, each under "prelu" and "relu", alternated;
* per step, the kernel time under both activations and the prelu step's share in hgb_prelu_bwd and the PReLU epilogue kernels
  (torch.profiler, in runs of their own).
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
from hydragnn_b200.synthetic import ARCH  # noqa: E402
from pna_bench import batch, card, timed  # noqa: E402

HBM = 3.35e12
NODE_HEAD = {"node": {"num_headlayers": 2, "dim_headlayers": [64, 32], "type": "mlp"}}


def rel(a, b):
    return float((a.double() - b.double()).norm() / b.double().norm().clamp(min=1e-30))


def alternate(fns, steps):
    res = {k: [] for k in fns}
    for _ in range(3):
        for k, fn in fns.items():
            res[k] += timed(fn, steps, regions=1)
    return {k: statistics.median(v) for k, v in res.items()}


def prelu_pair(rows, cols, steps):
    gen = torch.Generator(device="cuda").manual_seed(0)
    x = torch.randn(rows, cols, device="cuda", generator=gen, requires_grad=True)
    g = torch.randn(rows, cols, device="cuda", generator=gen)
    w = torch.tensor([0.25], device="cuda", requires_grad=True)

    def fused():
        return torch.autograd.grad(ops.PReluFn.apply(x, w), (x, w), g)

    def aten():
        return torch.autograd.grad(torch.nn.functional.prelu(x, w), (x, w), g)

    for fn in (fused, aten):
        fn()
    agree = max(rel(a, b) for a, b in zip(fused(), aten()))
    t = alternate({"fused": fused, "aten": aten}, steps)
    nbytes = 4 * 5 * rows * cols
    return {"rows": rows, "cols": cols, "fused_ms": t["fused"], "aten_ms": t["aten"], "speedup": t["aten"] / t["fused"],
            "grad_rel_l2": agree, "fused_gbps": nbytes / (t["fused"] * 1e-3) / 1e9,
            "fused_hbm_share": nbytes / (t["fused"] * 1e-3) / HBM}


def _models(name, graphs, extra):
    b, deg = batch(name, graphs)
    kw = dict(ARCH[name], pna_deg=deg, **extra)
    kw.pop("enable_interatomic_potential", None)
    n = b.x.shape[0]
    rows = graphs if kw["output_type"] == ["graph"] else n
    gen = torch.Generator(device="cuda").manual_seed(1)
    value = torch.randn(rows * kw["output_dim"][0], device="cuda", generator=gen)
    hi = [torch.arange(value.numel(), device="cuda")]
    steps = {}
    for act in ("prelu", "relu"):
        m = hb.create_model(**dict(kw, activation_function=act))
        m.train()
        opt = hb.FlatAdamW(m, lr=1e-4)

        def one(m=m, opt=opt):
            opt.zero_grad()
            tot, _ = m.loss(m(b), value, hi)
            opt.backward(tot)
            opt.step()
        steps[act] = one
    return b, steps


def train_steps(name, graphs, steps, warmup, extra):
    b, runs = _models(name, graphs, extra)
    for fn in runs.values():
        for _ in range(warmup):
            fn()
    t = alternate(runs, steps)
    return {"workload": name, "graphs": graphs, "atoms": int(b.x.shape[0]), "edges": int(b.edge_index.shape[1]),
            "prelu_step_ms": t["prelu"], "relu_step_ms": t["relu"], "prelu_over_relu": t["prelu"] / t["relu"], **extra}


def bwd_share(name, graphs, extra):
    """Kernel time per step (torch.profiler) under both activations, and the prelu step's share in the PReLU kernels."""
    from torch.profiler import ProfilerActivity, profile
    _, runs = _models(name, graphs, extra)
    out = {"workload": name}
    for act, one in runs.items():
        for _ in range(5):
            one()
        torch.cuda.synchronize()
        with profile(activities=[ProfilerActivity.CUDA]) as prof:
            for _ in range(10):
                one()
            torch.cuda.synchronize()
        tot, per = 0.0, {}
        for e in prof.key_averages():
            t = getattr(e, "device_time_total", None) or getattr(e, "cuda_time_total", 0.0)
            if e.key.startswith("void ") or "kernel" in e.key.lower():              # kernels only, not the host-side ops
                tot += t
                for key in ("prelu_bwd_kernel", "prelu_fwd_kernel", "gemm_prelu_kernel", "smallk_fwd_prelu", "smallk_fwd_vec4_prelu",
                            "grouped_rows_prelu"):
                    if key in e.key:
                        per[key] = per.get(key, 0.0) + t
        out[act + "_kernel_us_per_step"] = tot / 10
        if act == "prelu":
            out["prelu_kernels_us_per_step"] = {k: v / 10 for k, v in per.items()}
            out["prelu_bwd_share"] = per.get("prelu_bwd_kernel", 0.0) / tot if tot else None
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--graphs", type=int, default=512)
    ap.add_argument("--steps", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=5)
    a = ap.parse_args()
    torch.cuda.set_device(0)
    out = dict(card())
    out["prelu_pair"] = [prelu_pair(r, c, 50) for r in (10_000, 100_000, 1_000_000) for c in (12, 64)]
    egnn_node = dict(output_type=["node"], output_dim=[1], output_heads=NODE_HEAD, task_weights=[1.0])
    out["train_step"] = [train_steps("ogb_pna", a.graphs, a.steps, a.warmup, {}),
                         train_steps("md17_egnn", a.graphs, a.steps, a.warmup, egnn_node)]
    out["prelu_bwd_share"] = [bwd_share("ogb_pna", a.graphs, {}), bwd_share("md17_egnn", a.graphs, egnn_node)]
    print(json.dumps(out))


if __name__ == "__main__":
    main()
