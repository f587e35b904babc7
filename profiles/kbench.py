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


G = 16384
b = make_samples("qm9_painn", G).to(dev); b._num_graphs = G
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
for (m, nn_, k) in [(n, 64, 64), (n, 192, 64), (3 * n, 64, 64)]:
    dz, x = torch.randn(m, nn_, device=dev), torch.randn(m, k, device=dev)
    t = timeit(lambda: ops.raw_tc_wgrad(dz, x))
    out["tc_wgrad m=%d n=%d k=%d (ms | GB/s)" % (m, nn_, k)] = (t, m * (k + nn_) * 4 / t / 1e6)
print(json.dumps(out, indent=1))
