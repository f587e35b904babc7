"""Streaming rate and fixed cost of the tensor-core weight gradient (hgb_tc_wgrad) at the shapes the bench configs call it with.

usage: python profiles/wgrad_bench.py [--workloads qm9_painn:bf16,lj_egnn:fp32,md17_egnn:fp32] [--iters 40]   (needs a GPU)

The call shapes are read from one traced eager training step of each workload at its bench size (C2 qm9_painn in TF32, C1 lj_egnn
and C3 md17_egnn in the fp32-accurate mode).  Each distinct shape (m, n_out, k_out, row strides, mode) is timed at M = m/4, m/2, m
and 2m with CUDA events, once with L2 warm (back-to-back launches) and once with L2 flushed before every launch.  A least-squares
line through time against algorithmic bytes M (n_out + k_out) 4 gives the slope (the streaming rate, GB/s) and the intercept (the
fixed cost of one call: launch, pipeline fill, tail and the partial reduce).  Prints one JSON line per shape and a total over the
shapes of each workload step at M = m, with the card's name and power limit read in the same run."""
import argparse
import json
import os
import subprocess
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import torch
import hydragnn_b200 as hb
from hydragnn_b200 import _lib, ops
from hydragnn_b200.synthetic import ARCH, WORKLOADS, make_samples

GRAPHS = {"qm9_painn": 16384, "md17_egnn": 8192, "lj_egnn": 4096}      # bench.py's default sizes
dev = torch.device("cuda")


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader", "-i", str(torch.cuda.current_device())],
                       capture_output=True, text=True)
    return q.stdout.strip() if q.returncode == 0 else torch.cuda.get_device_name()


def traced_wgrad_calls(name, precision):
    """[(m, n_out, k_out, lddz, ldx, exact)] of every hgb_tc_wgrad call of one eager training step, in call order."""
    G = GRAPHS[name]
    w = WORKLOADS[name]
    b = make_samples(name, G).to(dev)
    b._num_graphs = G
    pbc = w.get("pbc") or w.get("pbc_box")
    b = (hb.get_radius_graph_pbc if pbc else hb.get_radius_graph)(w["radius"], w["max_neighbours"])(b)
    kw = dict(ARCH[name])
    mlip = bool(kw.get("enable_interatomic_potential"))
    model = hb.get_distributed_model(hb.set_precision(hb.create_model(**kw), precision))
    opt = hb.FlatAdamW(model, lr=1e-3)
    hi = None if mlip else hb.get_head_indices(model, b)
    hb.train_step(model, opt, b, compute_grad_energy=mlip, head_index=hi)
    torch.cuda.synchronize()
    _lib.trace_begin()
    hb.train_step(model, opt, b, compute_grad_energy=mlip, head_index=hi)
    torch.cuda.synchronize()
    calls = _lib.trace_end()
    del model, opt, b
    torch.cuda.empty_cache()
    return [(a["m"], a["n_out"], a["k_out"], a["lddz"], a["ldx"], a["exact"]) for e, a, _ in calls if e == "hgb_tc_wgrad"]


class Call:
    """One hgb_tc_wgrad call on seeded operands with the traced row strides (dz and x may be column slices of wider rows)."""

    def __init__(self, m, n_out, k_out, lddz, ldx, exact):
        g = torch.Generator(device=dev).manual_seed(0)
        self.dz = torch.randn(m, lddz, device=dev, generator=g)
        self.x = torch.randn(m, ldx, device=dev, generator=g)
        self.dw = torch.empty(n_out, k_out, device=dev)
        self.db = torch.empty(n_out, device=dev)
        self.nbytes = _lib.query("hgb_tc_wgrad_workspace_bytes", n_out, k_out)
        self.ws = torch.empty(self.nbytes, dtype=torch.uint8, device=dev)
        self.args = (m, n_out, k_out, lddz, ldx, exact)

    def __call__(self):
        m, n_out, k_out, lddz, ldx, exact = self.args
        _lib.call("hgb_tc_wgrad", self.dz.data_ptr(), lddz, self.x.data_ptr(), ldx, m, n_out, k_out, self.dw.data_ptr(), k_out,
                  self.db.data_ptr(), 0, exact, self.ws.data_ptr(), self.nbytes, torch.cuda.current_stream().cuda_stream)


def time_warm(fn, iters):
    for _ in range(3):
        fn()
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    a.record()
    for _ in range(iters):
        fn()
    b.record()
    torch.cuda.synchronize()
    return a.elapsed_time(b) / iters * 1e3


def time_cold(fn, iters, flush):
    ts = []
    for it in range(iters + 3):
        flush.zero_()
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        a.record()
        fn()
        b.record()
        torch.cuda.synchronize()
        if it >= 3:
            ts.append(a.elapsed_time(b) * 1e3)
    return sum(ts) / len(ts)


def fit(xs, ys):
    """least-squares y = slope x + intercept"""
    n = len(xs)
    mx, my = sum(xs) / n, sum(ys) / n
    sxx = sum((x - mx) ** 2 for x in xs)
    slope = sum((x - mx) * (y - my) for x, y in zip(xs, ys)) / sxx
    return slope, my - slope * mx


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--workloads", default="qm9_painn:bf16,lj_egnn:fp32,md17_egnn:fp32")
    ap.add_argument("--iters", type=int, default=40)
    a = ap.parse_args()
    torch.cuda.set_device(0)
    flush = torch.empty(256 * 1024 * 1024, dtype=torch.uint8, device=dev)
    print(json.dumps({"card": card(), "library": _lib.LIB_PATH}), flush=True)
    for spec in a.workloads.split(","):
        name, precision = spec.split(":")
        calls = traced_wgrad_calls(name, precision)
        shapes = {}
        for c in calls:
            shapes[c] = shapes.get(c, 0) + 1
        tot = {"warm": 0.0, "cold": 0.0}
        tot_bytes = 0
        for (m, n_out, k_out, lddz, ldx, exact), count in shapes.items():
            row = {"workload": name, "m": m, "n_out": n_out, "k_out": k_out, "lddz": lddz, "ldx": ldx, "mode": "exact" if exact else "tf32",
                   "calls_per_step": count}
            for kind in ("warm", "cold"):
                xs, ys = [], []
                for f in (0.25, 0.5, 1.0, 2.0):
                    mm = max(128, int(m * f))
                    call = Call(mm, n_out, k_out, lddz, ldx, exact)
                    t = time_warm(call, a.iters) if kind == "warm" else time_cold(call, a.iters, flush)
                    alg = mm * (n_out + k_out) * 4
                    xs.append(alg)
                    ys.append(t)
                    if f == 1.0:
                        row["%s_us_at_m" % kind] = round(t, 2)
                        row["%s_GBps_at_m" % kind] = round(alg / t * 1e-3, 1)
                        tot[kind] += t * count
                        if kind == "warm":
                            tot_bytes += alg * count
                    del call
                slope, icpt = fit(xs, ys)
                row["%s_stream_GBps" % kind] = round(1e-3 / slope, 1)
                row["%s_fixed_us" % kind] = round(icpt, 2)
            print(json.dumps(row), flush=True)
        print(json.dumps({"workload": name, "total_calls_per_step": len(calls), "alg_GB": round(tot_bytes / 1e9, 3),
                          "warm_us": round(tot["warm"], 1), "cold_us": round(tot["cold"], 1),
                          "warm_GBps": round(tot_bytes / tot["warm"] * 1e-3, 1), "cold_GBps": round(tot_bytes / tot["cold"] * 1e-3, 1),
                          "card": card()}), flush=True)


if __name__ == "__main__":
    main()
