"""Training-step timing of the MACE path on the SURVEY C4 shape (one GPU).
usage: python profiles/mace_bench.py [graphs] [steps] [precision] [edge_dim]
edge_dim > 0: the model reads edge_attr = the built graph's edge lengths (detached), repeated edge_dim times.
MACE_BENCH_KERNELS=1 also times hgb_mace_tp_scatter_{fwd,bwd} with torch.profiler and reports their algorithmic bytes."""
import os, sys, json, time
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import torch
import hydragnn_b200 as hb
from hydragnn_b200.synthetic import ARCH, make_samples

G = int(sys.argv[1]) if len(sys.argv) > 1 else 256
steps = int(sys.argv[2]) if len(sys.argv) > 2 else 10
prec = sys.argv[3] if len(sys.argv) > 3 else "bf16"
edge_dim = int(sys.argv[4]) if len(sys.argv) > 4 else 0
dev = torch.device("cuda")
b = make_samples("oc20_mace", G).to(dev); b._num_graphs = G
b = hb.get_radius_graph_pbc(6.0, 128)(b)
n, e = b.pos.shape[0], b.edge_index.shape[1]
if edge_dim:
    vec = b.pos[b.edge_index[1]] - b.pos[b.edge_index[0]] + b.edge_shifts
    b.edge_attr = vec.norm(dim=1, keepdim=True).detach().repeat(1, edge_dim).contiguous()
kw = dict(ARCH["oc20_mace"], avg_num_neighbors=e / n, edge_dim=edge_dim)
model = hb.set_precision(hb.create_model(**kw), prec)
model = hb.get_distributed_model(model)
opt = hb.FlatAdamW(model, lr=1e-3)
hi = hb.get_head_indices(model, b)
for _ in range(3):
    loss, _ = hb.train_step(model, opt, b, head_index=hi)
torch.cuda.synchronize()
t0, t1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
t0.record()
for _ in range(steps):
    loss, _ = hb.train_step(model, opt, b, head_index=hi)
t1.record(); torch.cuda.synchronize()
ms = t0.elapsed_time(t1) / steps
res = {"workload": "oc20_mace", "graphs": G, "atoms": n, "edges": e, "precision": prec, "edge_dim": edge_dim, "ms_per_step": ms,
       "atoms_per_s": n / ms * 1e3, "loss": float(loss), "peak_mem_GB": torch.cuda.max_memory_allocated() / 2**30}
if os.environ.get("MACE_BENCH_KERNELS") == "1":
    # per-layer algorithmic bytes of the fused tensor product, E (S_in F + W + D + S_sh) 4 read + the [N, NACC F] messages written
    # (backward: the messages' gradient read instead, g_tpw and the per-edge sender gradient written)
    from hydragnn_b200 import _lib, e3
    f = kw["hidden_dim"]
    layers = []
    for lin in (0, kw["node_max_ell"]):
        lsh = kw["max_ell"]
        s_in, s_sh = (lin + 1) ** 2, (lsh + 1) ** 2
        w = (len(e3.tp_paths(lin, lsh, lsh)) + edge_dim * (lin + 1)) * f
        nacc = _lib.query("hgb_mace_tp_num_acc", lin, lsh)
        fwd = 4 * (e * (s_in * f + w + edge_dim + s_sh) + n * nacc * f)
        bwd = 4 * (e * (s_in * f + w + edge_dim + s_sh) + n * nacc * f + e * (w + s_in * f))
        layers.append({"lmax_in": lin, "fwd_bytes": fwd, "bwd_bytes": bwd})
    with torch.profiler.profile(activities=[torch.profiler.ProfilerActivity.CUDA]) as prof:
        for _ in range(steps):
            hb.train_step(model, opt, b, head_index=hi)
        torch.cuda.synchronize()
    kt = {}
    for ev in prof.key_averages():
        if "mace_tp_scatter" in ev.key:
            kind = "fwd" if "fwd" in ev.key else "bwd"
            total = getattr(ev, "device_time_total", None) or ev.cuda_time_total
            kt.setdefault(kind, []).append({"kernel": ev.key[:80], "calls": ev.count, "us_per_call": total / max(ev.count, 1)})
    res["tp_scatter_kernels"] = kt
    res["tp_scatter_bytes"] = layers
print(json.dumps(res))
