"""Flat optimizer step timing, one GPU.

    python profiles/optim_bench.py [--steps 20] [--sizes 1000000 10000000 100000000]

Prints one JSON line with the card name and power limit beside every number:
* for SGD, Adam, AdamW, Adamax, Adagrad, Adadelta and RMSprop (torch's defaults, Adam also with amsgrad, SGD also with
  momentum) at 1e6, 1e7 and 1e8 parameters: the flat step (one hgb_*_step kernel plus the step-count increment) against
  torch.optim with foreach=True, and with fused=True where torch has it (SGD, Adam, AdamW), alternated in the same call (CUDA
  events, the median of three regions); the bytes one update needs (4 B x (3 + 2 x states): parameter and gradient read,
  parameter written, every state read and written -- 12 B per element for plain SGD, 28 B for Adam and AdamW), the flat step's achieved bandwidth and its share of the
  H100 SXM's 3.35 TB/s, and the relative difference of the parameters from torch's after the timed steps;
* one eager training step (forward, loss, backward, optimizer) of ARCH["ogb_pna"] under FlatAdam and under FlatAdamW, alternated.
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
from hydragnn_b200.synthetic import ARCH  # noqa: E402
from pna_bench import batch, card, timed  # noqa: E402

HBM = 3.35e12
CASES = [("SGD", {}), ("SGD", {"momentum": 0.9}), ("Adam", {}), ("Adam", {"amsgrad": True}), ("AdamW", {}), ("Adamax", {}),
         ("Adagrad", {}), ("Adadelta", {}), ("RMSprop", {})]
FLAT = {"SGD": hb.FlatSGD, "Adam": hb.FlatAdam, "AdamW": hb.FlatAdamW, "Adamax": hb.FlatAdamax, "Adagrad": hb.FlatAdagrad,
        "Adadelta": hb.FlatAdadelta, "RMSprop": hb.FlatRMSprop}


def alternate(fns, steps):
    res = {k: [] for k in fns}
    for _ in range(3):
        for k, fn in fns.items():
            res[k] += timed(fn, steps, regions=1)
    return {k: statistics.median(v) for k, v in res.items()}


def rel(a, b):
    return float((a.double() - b.double()).norm() / b.double().norm().clamp(min=1e-30))


def one_size(name, hp, count, steps):
    gen = torch.Generator(device="cuda").manual_seed(0)
    p0 = torch.randn(count, device="cuda", generator=gen)
    g = torch.randn(count, device="cuda", generator=gen) * 1e-2
    flat = FLAT[name]([torch.nn.Parameter(p0.clone())], **hp)
    flat.flat_g.copy_(g)
    fns = {"flat": flat.step}
    torch_params = {}
    variants = {"foreach": {"foreach": True}}
    if name in ("SGD", "Adam", "AdamW"):
        variants["fused"] = {"fused": True}
    for label, extra in variants.items():
        q = torch.nn.Parameter(p0.clone())
        q.grad = g.clone()
        fns[label] = torch.optim.__dict__[name]([q], **hp, **extra).step
        torch_params[label] = q
    for fn in fns.values():
        fn()
    t = alternate(fns, steps)
    torch.cuda.synchronize()
    states = len(flat.state_tensors()) - 1
    nbytes = 4 * (3 + 2 * states) * count
    out = {"type": name, "options": hp, "count": count, "states": states, "bytes": nbytes, "flat_ms": t["flat"],
           "flat_gbps": nbytes / (t["flat"] * 1e-3) / 1e9, "flat_hbm_share": nbytes / (t["flat"] * 1e-3) / HBM}
    for label, q in torch_params.items():
        out[label + "_ms"] = t[label]
        out["speedup_vs_" + label] = t[label] / t["flat"]
        out["param_rel_diff_vs_" + label] = rel(flat.flat_p, q.detach())     # same number of steps on every leg
    del flat, torch_params, fns
    torch.cuda.empty_cache()
    return out


def train_step(graphs, steps, warmup):
    b, deg = batch("ogb_pna", graphs)
    kw = dict(ARCH["ogb_pna"], pna_deg=deg)
    runs = {}
    for label, cls in (("Adam", hb.FlatAdam), ("AdamW", hb.FlatAdamW)):
        torch.manual_seed(0)
        m = hb.create_model(**kw)
        m.train()
        opt = cls(m, lr=1e-4)
        hi = [torch.arange(graphs, device="cuda")]
        value = torch.randn(graphs, device="cuda", generator=torch.Generator(device="cuda").manual_seed(1))

        def one(m=m, opt=opt, value=value):
            opt.zero_grad()
            tot, _ = m.loss(m(b), value, hi)
            opt.backward(tot)
            opt.step()
        for _ in range(warmup):
            one()
        runs[label] = one
    t = alternate(runs, steps)
    return {"workload": "ogb_pna", "graphs": graphs, "adam_step_ms": t["Adam"], "adamw_step_ms": t["AdamW"],
            "adam_over_adamw": t["Adam"] / t["AdamW"]}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=5)
    ap.add_argument("--graphs", type=int, default=512)
    ap.add_argument("--sizes", type=int, nargs="+", default=[1_000_000, 10_000_000, 100_000_000])
    a = ap.parse_args()
    torch.cuda.set_device(0)
    out = dict(card())
    out["steps"] = [one_size(n, hp, c, a.steps) for n, hp in CASES for c in a.sizes]
    out["train_step"] = train_step(a.graphs, a.steps, a.warmup)
    print(json.dumps(out))


if __name__ == "__main__":
    main()
