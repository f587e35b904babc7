"""Every ATen kernel in one eager C2 (qm9_painn) training step, with its device time and the op that launched it.

usage: python profiles/painn_aten_kernels.py [graphs] [precision]

The step is the bench's: radius graph on the GPU, forward, loss, backward, fused AdamW, weight gradients on the current stream
(as in bench.py's kernel-share pass).  Prints JSON: the card and power limit, the step's total kernel time, the ATen share,
every ATen kernel launched by an op with an input of at least N*64 elements (N = atoms in the batch), and every other kernel
with its device time, in launch order."""
import json
import os
import subprocess
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import torch
from torch.profiler import ProfilerActivity, profile

import hydragnn_b200 as hb
from hydragnn_b200 import ops
from hydragnn_b200.synthetic import ARCH, WORKLOADS, make_samples

G = int(sys.argv[1]) if len(sys.argv) > 1 else 16384
prec = sys.argv[2] if len(sys.argv) > 2 else "bf16"
name = "qm9_painn"
dev = torch.device("cuda")
w = WORKLOADS[name]
b = make_samples(name, G).to(dev)
b._num_graphs = G
b = hb.get_radius_graph(w["radius"], w["max_neighbours"])(b)
N, E = b.pos.shape[0], b.edge_index.shape[1]
model = hb.get_distributed_model(hb.set_precision(hb.create_model(**ARCH[name]), prec))
opt = hb.FlatAdamW(model, lr=1e-3)
hi = hb.get_head_indices(model, b)
ops.WGRAD_OVERLAP = False
run = lambda: hb.train_step(model, opt, b, head_index=hi)  # noqa: E731
for _ in range(3):
    run()
torch.cuda.synchronize()
with profile(activities=[ProfilerActivity.CPU, ProfilerActivity.CUDA], record_shapes=True) as prof:
    run()
    torch.cuda.synchronize()

is_aten = lambda n: "at::" in n or "at_cuda" in n or "cutlass" in n or "cublas" in n.lower()  # noqa: E731
evs = prof.events()
kern = [e for e in evs if getattr(e, "device_type", None) is not None and "cuda" in str(e.device_type).lower()
        and e.name and not e.name.lower().startswith(("memcpy", "memset"))]
tot_us = sum(e.time_range.elapsed_us() for e in kern)
aten_us = sum(e.time_range.elapsed_us() for e in kern if is_aten(e.name))


def numel(shape):
    n = 1
    for s in shape:
        n *= s
    return n


big = []
for e in evs:                                  # CPU ops: the kernels each one launched directly, with the op's input shapes
    ks = [k for k in (getattr(e, "kernels", None) or []) if is_aten(k.name)]
    if not ks:
        continue
    shapes = [s for s in (e.input_shapes or []) if isinstance(s, (list, tuple)) and all(isinstance(x, int) for x in s)]
    largest = max((numel(s) for s in shapes), default=0)
    if largest < N * 64:
        continue
    for k in ks:
        big.append({"op": e.name, "shapes": shapes[:3], "kernel": k.name.split("(")[0][:90], "us": round(k.duration, 1)})
big.sort(key=lambda r: -r["us"])

# every other kernel of the step in launch order (one stream): name without the parameter list, device time
ours = [[e.name.replace("(anonymous namespace)::", "").split("(")[0][:80], round(e.time_range.elapsed_us(), 1)]
        for e in sorted((e for e in kern if not is_aten(e.name)), key=lambda e: e.time_range.start)]
try:
    card = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True,
                          text=True).stdout.strip().splitlines()[0]
except Exception:                              # noqa: BLE001
    card = "unknown"
print(json.dumps({"workload": name, "graphs": G, "atoms": N, "edges": E, "precision": prec, "card": card,
                  "total_kernel_us": round(tot_us, 1), "aten_us": round(aten_us, 1), "aten_share": round(aten_us / tot_us, 4),
                  "aten_kernels_over_N64": big, "aten_over_N64_us": round(sum(r["us"] for r in big), 1),
                  "aten_over_N64_share": round(sum(r["us"] for r in big) / tot_us, 4), "other_kernels_in_order": ours}, indent=1))
