"""GaussianNLLLoss timing, one GPU.

    python profiles/gnll_bench.py [--graphs 512] [--steps 20]

Prints one JSON line with the card name and power limit beside every number:
* the loss with both gradients, ``ops.GaussianNLLFn`` (hgb_gnll_fwd_bwd, one launch) against
  torch.nn.functional.gaussian_nll_loss and its autograd backward, at node-head sizes of 1e5 to 4e6 elements, alternated in the
  same call (CUDA events, the median of three regions), with their agreement and the kernel's algorithmic bytes
  (4 B x 5 count: mean, var and target read, the two gradients written) over its time;
* eager training steps (forward, loss, backward, FlatAdamW) of ARCH["ogb_pna"] on its synthetic graphs with the heads of the
  reference's tests/inputs/ci_multihead.json -- one graph head and three ``mlp`` node heads, task weights [20, 1, 1, 1] -- under
  GaussianNLLLoss and under mse, alternated.
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
CI_HEADS = {"graph": {"num_sharedlayers": 2, "dim_sharedlayers": 10, "num_headlayers": 2, "dim_headlayers": [10, 10]},
            "node": {"num_headlayers": 2, "dim_headlayers": [10, 10], "type": "mlp"}}


def rel(a, b):
    return float((a.double() - b.double()).norm() / b.double().norm().clamp(min=1e-30))


def alternate(fns, steps):
    res = {k: [] for k in fns}
    for _ in range(3):
        for k, fn in fns.items():
            res[k] += timed(fn, steps, regions=1)
    return {k: statistics.median(v) for k, v in res.items()}


def loss_kernel(count, steps):
    gen = torch.Generator(device="cuda").manual_seed(0)
    mean = torch.randn(count, device="cuda", generator=gen, requires_grad=True)
    target = torch.randn(count, device="cuda", generator=gen)
    var = (torch.randn(count, device="cuda", generator=gen) ** 2).requires_grad_(True)

    def fused():
        return torch.autograd.grad(ops.GaussianNLLFn.apply(mean, var, target), (mean, var))

    def aten():
        return torch.autograd.grad(torch.nn.functional.gaussian_nll_loss(mean, target, var), (mean, var))

    for fn in (fused, aten):
        fn()
    agree = max(rel(a, b) for a, b in zip(fused(), aten()))
    t = alternate({"fused": fused, "aten": aten}, steps)
    nbytes = 4 * 5 * count
    return {"count": count, "fused_ms": t["fused"], "aten_ms": t["aten"], "speedup": t["aten"] / t["fused"],
            "grad_rel_l2": agree, "fused_bytes": nbytes, "fused_gbps": nbytes / (t["fused"] * 1e-3) / 1e9,
            "fused_hbm_share": nbytes / (t["fused"] * 1e-3) / HBM}


def step(graphs, steps, warmup):
    b, deg = batch("ogb_pna", graphs)
    g, n = graphs, b.x.shape[0]
    gen = torch.Generator(device="cuda").manual_seed(1)
    value = torch.randn(g + 3 * n, device="cuda", generator=gen)
    hi = [torch.arange(g, device="cuda")] + [g + k * n + torch.arange(n, device="cuda") for k in range(3)]
    kw = dict(ARCH["ogb_pna"], pna_deg=deg, output_dim=[1, 1, 1, 1], output_type=["graph", "node", "node", "node"],
              output_heads=CI_HEADS, task_weights=[20.0, 1.0, 1.0, 1.0])
    runs = {}
    for loss in ("GaussianNLLLoss", "mse"):
        m = hb.create_model(**dict(kw, loss_function_type=loss))
        m.train()
        opt = hb.FlatAdamW(m, lr=1e-4)

        def one(m=m, opt=opt):
            opt.zero_grad()
            tot, _ = m.loss(m(b), value, hi)
            opt.backward(tot)
            opt.step()
        for _ in range(warmup):
            one()
        runs[loss] = one
    t = alternate(runs, steps)
    return {"workload": "ogb_pna", "graphs": g, "atoms": n, "edges": int(b.edge_index.shape[1]), "gnll_step_ms": t["GaussianNLLLoss"],
            "mse_step_ms": t["mse"], "gnll_over_mse": t["GaussianNLLLoss"] / t["mse"]}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--graphs", type=int, default=512)
    ap.add_argument("--steps", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=5)
    a = ap.parse_args()
    torch.cuda.set_device(0)
    out = dict(card())
    out["loss_kernel"] = [loss_kernel(c, 50) for c in (100_000, 1_000_000, 4_000_000)]
    out["train_step"] = step(a.graphs, a.steps, a.warmup)
    print(json.dumps(out))


if __name__ == "__main__":
    main()
