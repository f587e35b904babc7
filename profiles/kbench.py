"""Isolated kernel timings (CUDA events, L2 flushed before every launch) on the bench shapes.
usage: python profiles/kbench.py   (needs a GPU)"""
import os, sys, json
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import torch
import hydragnn_b200 as hb
from hydragnn_b200 import ops
from hydragnn_b200.stacks import Base
from hydragnn_b200.synthetic import ARCH, make_samples

dev = torch.device("cuda")
flush = torch.empty(256 * 1024 * 1024, dtype=torch.uint8, device=dev)


def timeit(fn, iters=10, warm=3):
    ts = []
    for it in range(iters + warm):
        flush.zero_()
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        a.record(); fn(); b.record(); torch.cuda.synchronize()
        if it >= warm:
            ts.append(a.elapsed_time(b))
    return sum(ts) / len(ts)


def tc_linear_calls(n):
    """The hgb_tc_linear calls of the C2 (qm9_painn) step at n nodes, each with its real epilogue operands.
    GB/s: algorithmic bytes (bench._alg_bytes: 4 m (k_red + n_out (1 + z + addend + gsrc))) over device time."""
    silu, tanh, deriv = ops.ACT_CODES["silu"], ops.ACT_CODES["tanh"], ops.ACT_DERIV
    # name, m, k_red, n_out, trans_b, act, want_z, gact, addend, gsrc
    calls = [("fwd 64->64 silu z=silu'", n, 64, 64, False, silu, True, deriv, False, False),
             ("fwd 64->192", n, 64, 192, False, 0, False, 0, False, False),
             ("fwd 64->128 (3N rows)", 3 * n, 64, 128, False, 0, False, 0, False, False),
             ("fwd 128->64 silu z=silu'", n, 128, 64, False, silu, True, deriv, False, False),
             ("fwd 64->128", n, 64, 128, False, 0, False, 0, False, False),
             ("fwd 64->64 tanh", n, 64, 64, False, tanh, False, 0, False, False),
             ("dgrad 64->64 gsrc=silu'", n, 64, 64, True, 0, False, deriv, False, True),
             ("dgrad 64->192 gsrc=silu'", n, 192, 64, True, 0, False, deriv, False, True),
             ("dgrad 128->64 gsrc=silu'", n, 64, 128, True, 0, False, deriv, False, True),
             ("dgrad 64->64 gsrc=tanh", n, 64, 64, True, 0, False, tanh, False, True),
             ("dgrad 64->128 (3N rows) +addend", 3 * n, 128, 64, True, 0, False, 0, True, False),
             ("dgrad 64->128 plain", n, 128, 64, True, 0, False, 0, False, False)]
    res = {}
    for name, m, k, no, tb, act, want_z, gact, has_add, has_g in calls:
        a = torch.randn(m, k, device=dev)
        w = torch.randn(k, no, device=dev) if tb else torch.randn(no, k, device=dev)
        bias = None if tb else torch.randn(no, device=dev)
        add = torch.randn(m, no, device=dev) if has_add else None
        g = torch.rand(m, no, device=dev) if has_g else None
        t = timeit(lambda: ops.raw_tc_linear(a, w, tb, bias, no, k, act, 0.0, want_z, addend=add, gsrc=g, gact=gact))
        nbytes = 4 * m * (k + no * (1 + int(want_z) + int(has_add) + int(has_g)))
        res["tc_linear %s m=%d (ms | GB/s)" % (name, m)] = (round(t, 4), round(nbytes / t / 1e6, 1))
    return res


def painn_update_calls(n, f=64):
    """The F = 64 PaiNN update block of the C2 step in TF32 mode, fused (PainnUpdateTcFn) and unfused (PainnUpdateFn), forward and
    backward (weight gradients included, on one stream).  GB/s: algorithmic bytes, in units U = one [n, 64] fp32 tensor, counting
    every tensor each kernel reads and writes (DESIGN.md section 4), over device time."""
    from hydragnn_b200.stacks import PainnUpdate
    # (forward, backward) bytes in U, by last.  Fused: fwd [|vv|, s] (+ inner) 7 | 6, MLP 4 + (3 | 4), post 5 | 11; bwd ga 4 | 10,
    # dgrads 4 + 3 (5 + 3), [guv | gvv] + gv 18 | 22, weight gradients 15 | 16.  Unfused: fwd U/V 9, pre 6, MLP 4 + (3 | 4), post 10 | 17; bwd
    # post_bwd_a 9 | 13, dgrads 4 + 3 (5 + 3), update_bwd 18 | 24, U/V dgrad 9 | 12, weight gradients 15 | 16.
    units = {("fused", True): (19, 44), ("fused", False): (25, 56), ("unfused", True): (32, 58), ("unfused", False): (40, 72)}
    U = n * f * 4
    res = {}
    overlap = ops.WGRAD_OVERLAP
    ops.WGRAD_OVERLAP = False
    try:
        for last in (True, False):
            upd = PainnUpdate(f, last).to(dev)
            params = [upd.update_U.weight, upd.update_U.bias, upd.update_V.weight, upd.update_V.bias, upd.update_mlp[0].weight,
                      upd.update_mlp[0].bias, upd.update_mlp[2].weight, upd.update_mlp[2].bias]
            s = torch.randn(n, f, device=dev, requires_grad=True)
            v = torch.randn(n, 3, f, device=dev, requires_grad=True)
            for kind, fn in (("fused", ops.PainnUpdateTcFn), ("unfused", ops.PainnUpdateFn)):
                with ops.tensor_cores(True):
                    so, vo = fn.apply(s, v, *params, last)
                    outs = (so,) if last else (so, vo)
                    grads = tuple(torch.randn_like(o) for o in outs)
                    t_f = timeit(lambda: fn.apply(s, v, *params, last))
                    t_b = timeit(lambda: torch.autograd.grad(outs, [s, v] + params, grads, retain_graph=True))
                uf, ub = units[(kind, last)]
                res["painn_update %s last=%s fwd (ms | GB/s | U)" % (kind, last)] = (round(t_f, 4), round(uf * U / t_f / 1e6, 1), uf)
                res["painn_update %s last=%s bwd (ms | GB/s | U)" % (kind, last)] = (round(t_b, 4), round(ub * U / t_b / 1e6, 1), ub)
    finally:
        ops.WGRAD_OVERLAP = overlap
    return res


G = 16384
b = make_samples("qm9_painn", G).to(dev); b._num_graphs = G
if os.environ.get("KBENCH_ONLY") == "tc_linear":
    print(json.dumps(tc_linear_calls(b.pos.shape[0]), indent=1)); sys.exit(0)
if os.environ.get("KBENCH_ONLY") == "painn_update":
    print(json.dumps(painn_update_calls(b.pos.shape[0]), indent=1)); sys.exit(0)
b = hb.get_radius_graph(7.0, 5)(b)
plan = Base.plan_for(b)
n, e, f, r = plan.num_nodes, plan.num_edges, 64, 5
_, ln, unit = ops.EdgeGeomFn.apply(b.pos, None, plan, 1e-9)
epack = ops.PainnEdgeEmbedFn.apply(unit, ln, r, 7.0)
s, v, phi = torch.randn(n, f, device=dev), torch.randn(n, 3, f, device=dev), torch.randn(n, 3 * f, device=dev)
wf, bf = torch.randn(3 * f, r, device=dev), torch.randn(3 * f, device=dev)
out = {}
rec = ops.painn_edge_records(epack, plan, "row")
out["painn_message_fwd F=64 (ms)"] = timeit(lambda: ops.PainnMessageFn.apply(phi, s, v, epack, wf, bf, None, plan, rec))
out["painn_edge_records (ms)"] = timeit(lambda: ops.painn_edge_records(epack, plan, "row"))
sr, vr, pr = s.clone().requires_grad_(True), v.clone().requires_grad_(True), phi.clone().requires_grad_(True)
so, vo = ops.PainnMessageFn.apply(pr, sr, vr, epack, wf.requires_grad_(True), bf.requires_grad_(True), None, plan, rec)
gs, gv = torch.randn_like(so), torch.randn_like(vo)
out["painn_message_bwd F=64 (ms)"] = timeit(lambda: torch.autograd.grad((so, vo), (pr, sr, vr, wf, bf), (gs, gv), retain_graph=True))
so2, vo2 = ops.PainnMessageFn.apply(pr, sr, vr, epack, wf, bf, None, plan, None)
out["painn_message_bwd generic F=64 (ms)"] = timeit(lambda: torch.autograd.grad((so2, vo2), (pr, sr, vr, wf, bf), (gs, gv), retain_graph=True))
if os.environ.get("KBENCH_ONLY") == "painn":
    print(json.dumps(out, indent=1)); sys.exit(0)
alg_f = e * (6 * f * 4 + 8 + 48) + n * (8 * f * 4 + 4)
out["painn_message_fwd GB/s algorithmic"] = alg_f / out["painn_message_fwd F=64 (ms)"] / 1e6
for (m, k, nn_) in [(n, 64, 64), (n, 64, 192), (3 * n, 64, 64), (n, 128, 64), (n, 192, 64)]:
    x, w, bb = torch.randn(m, k, device=dev), torch.randn(nn_, k, device=dev), torch.randn(nn_, device=dev)
    t = timeit(lambda: ops.raw_tc_linear(x, w, False, bb, nn_, k))
    out["tc_linear m=%d k=%d n=%d (ms | GB/s)" % (m, k, nn_)] = (t, m * (k + nn_) * 4 / t / 1e6)
out.update(tc_linear_calls(n))
for (m, nn_, k) in [(n, 64, 64), (n, 192, 64), (3 * n, 64, 64)]:
    dz, x = torch.randn(m, nn_, device=dev), torch.randn(m, k, device=dev)
    t = timeit(lambda: ops.raw_tc_wgrad(dz, x))
    out["tc_wgrad m=%d n=%d k=%d (ms | GB/s)" % (m, nn_, k)] = (t, m * (k + nn_) * 4 / t / 1e6)
print(json.dumps(out, indent=1))
