"""MACE graph-attribute conditioning timing on the gfm_mace workload (hydragnn_b200/synthetic.py, examples/multidataset_hpo_sc26/
gfm_mlip.json), one GPU.

    python profiles/mace_cond_bench.py [--graphs 64] [--steps 10]

Prints one JSON line with the card name and power limit beside every number:
* the two conditioning kernels at the workload's N atoms, H = 128 channels, B graphs and G = 2 graph attributes, each against the
  ATen composition it replaces, alternated in the same call (CUDA events, three regions, the median):
    concat_node   ops.GraphAddLinearFn (hgb_tc_linear_graph_add)  vs  Linear(cat([h, graph_attr[batch]]))   forward + backward
    film          ops.FilmFn (hgb_film_fwd / hgb_film_bwd)         vs  h * (1 + tanh s)[batch] + t[batch] and its autograd
                                                                        backward (index_add_ per-graph sums)          forward + backward
  with the rel-L2 agreement of the outputs and gradients, and the kernels' algorithmic bytes and share of the 3.35 TB/s HBM3
  bound (H100 SXM data sheet).  Both are memory-bound; per pass, with 4-byte floats:
    concat_node fwd  4 (N H + N H + H H)           h read, y written, W_h
    concat_node bwd  4 (N H + N H + N H + N H)     dy read twice (dgrad, weight gradient), h read, dh written (+ the per-graph sum)
    film fwd         4 (2 N H)                     h read, y written (the per-graph terms stay in L2)
    film bwd         4 (3 N H)                     dy and h read, dh written
* whole MLIP training steps (FlatAdamW, eager) of the conditioned (concat_node) and the unconditioned model, alternated.
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


def rel(a, b):
    return float((a.double() - b.double()).norm() / b.double().norm().clamp(min=1e-30))


def alternate(fns, steps):
    """fns: {name: callable}; three rounds in which every fn runs one timed region in turn; median ms per call."""
    res = {k: [] for k in fns}
    for _ in range(3):
        for k, fn in fns.items():
            res[k] += timed(fn, steps, regions=1)
    return {k: statistics.median(v) for k, v in res.items()}


def kernels(n, h, b, gdim, steps, gcsr, batch):
    gen = torch.Generator(device="cuda").manual_seed(0)
    x = torch.randn(n, h, device="cuda", generator=gen, requires_grad=True)
    ga = torch.randn(b, gdim, device="cuda", generator=gen)
    w = (torch.randn(h, h + gdim, device="cuda", generator=gen) / h ** 0.5).requires_grad_(True)
    bias = torch.randn(h, device="cuda", generator=gen, requires_grad=True)
    st = torch.randn(b, 2 * h, device="cuda", generator=gen, requires_grad=True)
    dy = torch.randn(n, h, device="cuda", generator=gen)

    def concat_fused():
        c = ops.linear_act(ga, w[:, h:].contiguous(), bias)
        y = ops.GraphAddLinearFn.apply(x, w[:, :h], c, gcsr)
        return y, torch.autograd.grad(y, (x, w, bias), dy)

    def concat_aten():
        y = torch.nn.functional.linear(torch.cat([x, ga[batch]], 1), w, bias)
        return y, torch.autograd.grad(y, (x, w, bias), dy)

    def film_fused():
        y = ops.FilmFn.apply(x, st, gcsr)
        return y, torch.autograd.grad(y, (x, st), dy)

    def film_aten():
        y = x * (1 + torch.tanh(st[:, :h]))[batch] + st[:, h:][batch]
        return y, torch.autograd.grad(y, (x, st), dy)

    agree = {}
    for name, (f, a) in {"concat_node": (concat_fused, concat_aten), "film": (film_fused, film_aten)}.items():
        (yf, gf), (ya, ga_) = f(), a()
        agree[name] = {"out": rel(yf, ya), "grads": [rel(p, q) for p, q in zip(gf, ga_)]}
    ms = alternate({"concat_node_fused": concat_fused, "concat_node_aten": concat_aten, "film_fused": film_fused,
                    "film_aten": film_aten}, steps)
    nbytes = {"concat_node_fused": 4 * (2 * n * h + h * h) + 4 * (4 * n * h), "film_fused": 4 * (2 * n * h) + 4 * (3 * n * h)}
    out = {}
    for k, v in ms.items():
        out[k] = {"ms_fwd_bwd": round(v, 4)}
        if k in nbytes:
            out[k].update(algorithmic_bytes=nbytes[k], achieved_GBps=round(nbytes[k] / (v * 1e-3) / 1e9, 1),
                          frac_of_hbm_peak=round(nbytes[k] / HBM / (v * 1e-3), 3))
    return out, agree


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--graphs", type=int, default=64)
    ap.add_argument("--steps", type=int, default=10)
    args = ap.parse_args()
    torch.cuda.set_device(0)
    name, w = "gfm_mace", WORKLOADS["gfm_mace"]
    d = make_samples(name, args.graphs).to("cuda")
    d._num_graphs = args.graphs
    d = hb.get_radius_graph_pbc(w["radius"], w["max_neighbours"])(d)
    vec = d.pos[d.edge_index[1]] - d.pos[d.edge_index[0]] + d.edge_shifts.to(d.pos.dtype)
    d.edge_attr = vec.norm(dim=1, keepdim=True).detach()
    d.graph_attr = torch.randn(args.graphs, 2, device="cuda", generator=torch.Generator(device="cuda").manual_seed(1))
    n, h = d.pos.shape[0], ARCH[name]["hidden_dim"]
    batch = d.batch
    gcsr = ops.graph_ptr_from_batch(batch, args.graphs)
    res = {"workload": name, "graphs": args.graphs, "atoms": n, "edges": int(d.edge_index.shape[1]), **card()}
    with ops.tensor_cores(False):           # the fp32 configs' mode (3xTF32 in the tensor-core Linear)
        res["kernels_fp32"], res["agreement_fp32"] = kernels(n, h, args.graphs, 2, args.steps * 10, gcsr, batch)
    with ops.tensor_cores(True):
        res["kernels_tf32"], res["agreement_tf32"] = kernels(n, h, args.graphs, 2, args.steps * 10, gcsr, batch)

    models = {}
    for label, cond in (("conditioned", True), ("unconditioned", False)):
        m = hb.create_model(**dict(ARCH[name], use_graph_attr_conditioning=cond))
        if cond:
            with torch.no_grad():
                m(d)                        # creates the projector before the optimizer flattens the parameters
        model = hb.get_distributed_model(m)
        opt = hb.FlatAdamW(model, lr=1e-3)
        models[label] = (model, opt)

    def step(label):
        model, opt = models[label]
        return lambda: hb.train_step(model, opt, d, compute_grad_energy=True)
    for label in models:
        for _ in range(2):
            step(label)()
    torch.cuda.synchronize()
    res["step_ms"] = {k: round(v, 3) for k, v in alternate({k: step(k) for k in models}, args.steps).items()}
    print(json.dumps(res))


if __name__ == "__main__":
    main()
