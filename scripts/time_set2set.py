"""Time Set2Set pooling (csrc/set2set.cu) on cuda:0 against the reference composition on the existing kernels
(broadcast_nodes / softmax_nodes / reduce_nodes, the route taken above GNNB_SET2SET_MAX_D).  One JSON line per workload.

Workloads, all with n_iters = 3 (batches of equal-sized graphs; Set2Set reads no edges, so each node has one self loop):
  (a) 10 000 graphs of 23 nodes, D = 128        (molecules)
  (b) 1 024 graphs of 1 000 nodes, D = 128
  (c) one graph of 10 M nodes, D = 128           (one long row of the indicator plan: partial slots and the fix-up)
  (d) (b) at D = 512
Arms, alternated round by round in this process, each timed with CUDA events around whole calls:
  * `fused`: the layer with the fused attention;  * `composed`: the same layer with the bound patched to 0;
each as the forward alone and as forward + backward (x and every LSTM parameter require grad).  The peak memory of an arm
is torch.cuda.max_memory_allocated during one forward + backward, less what was allocated before it.
With --profile, a torch.profiler run of one forward + backward of the fused arm per workload (separate from the timed
calls) adds the device time of the attention kernels and their algorithmic rate: per iteration the forward reads x once
(N·D·4 bytes) and the backward reads x and writes dx (2·N·D·4 bytes); q, r and the statistics are graph-sized.
Each line also carries the card's name, power limit and the SM clock read after the timed calls, and the largest
normwise relative difference between the two arms' outputs.

    python scripts/time_set2set.py [--rounds 5] [--profile] [--only a,b,c,d]
"""
import argparse
import json
import os
import subprocess
import sys
import time

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import gnnb200 as gnn  # noqa: E402
from gnnb200 import readout  # noqa: E402

N_ITERS = 3


def card():
    try:
        out = subprocess.check_output(["nvidia-smi", "--id=0", "--query-gpu=name,power.limit,clocks.sm",
                                       "--format=csv,noheader,nounits"], text=True).strip().split(", ")
        return out[0], float(out[1]), float(out[2])
    except Exception:
        return torch.cuda.get_device_name(0), float("nan"), float("nan")


def event_ms(fn):
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    torch.cuda.synchronize()
    a.record()
    out = fn()
    b.record()
    torch.cuda.synchronize()
    return a.elapsed_time(b), out


def with_bound(bound, fn):
    saved = readout._SET2SET_MAX_D
    readout._SET2SET_MAX_D = bound
    try:
        return fn()
    finally:
        readout._SET2SET_MAX_D = saved


def peak_bytes(fn):
    torch.cuda.synchronize()
    base = torch.cuda.memory_allocated()
    torch.cuda.reset_peak_memory_stats()
    fn()
    torch.cuda.synchronize()
    return torch.cuda.max_memory_allocated() - base


def profile(fn):
    """device time of the attention kernels and of all device work in one call (ms)"""
    from torch.profiler import ProfilerActivity, profile as tprofile
    torch.cuda.synchronize()
    with tprofile(activities=[ProfilerActivity.CPU, ProfilerActivity.CUDA]) as prof:
        fn()
        torch.cuda.synchronize()
    fwd = bwd = dev = 0.0
    for e in prof.events():
        if getattr(e, "device_type", None) != torch.autograd.DeviceType.CUDA:
            continue
        t = e.time_range.elapsed_us() / 1e3
        dev += t
        if "set2set_fwd_kernel" in e.name:
            fwd += t
        elif "set2set_bwd_kernel" in e.name:
            bwd += t
    return fwd, bwd, dev


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rounds", type=int, default=5)
    ap.add_argument("--profile", action="store_true")
    ap.add_argument("--only", default="a,b,c,d")
    args = ap.parse_args()
    torch.cuda.set_device(0)
    workloads = [("a", 10_000, 23, 128), ("b", 1_024, 1_000, 128), ("c", 1, 10_000_000, 128), ("d", 1_024, 1_000, 512)]
    for name, G, n, D in workloads:
        if name not in args.only.split(","):
            continue
        N = G * n
        a = torch.arange(1, N + 1, device="cuda")
        gi = torch.arange(1, G + 1, device="cuda").repeat_interleave(n)
        g = gnn.GNNGraph(a, a, num_nodes=N, num_graphs=G, graph_indicator=gi if G > 1 else None)
        torch.manual_seed(0)
        l = gnn.Set2Set(D, N_ITERS, device="cuda")
        x = gnn.unrows(torch.randn(N, D, device="cuda") * 0.1).requires_grad_(True)
        params = [x] + list(l.parameters())

        def fwd():
            with torch.no_grad():
                return l(g, x)

        def fwd_bwd():
            y = l(g, x)
            return torch.autograd.grad(y.sum(), params)

        arms = {"fused": readout._SET2SET_MAX_D, "composed": 0}
        for bound in arms.values():                       # warm-up: modules, plans, algorithms
            with_bound(bound, fwd)
            with_bound(bound, fwd_bwd)
        times = {f"{arm}_{kind}": [] for arm in arms for kind in ("fwd", "fwd_bwd")}
        for _ in range(args.rounds):
            for arm, bound in arms.items():
                times[f"{arm}_fwd"].append(event_ms(lambda: with_bound(bound, fwd))[0])
                times[f"{arm}_fwd_bwd"].append(event_ms(lambda: with_bound(bound, fwd_bwd))[0])
        name_, plimit, clock = card()
        res = {"workload": name, "graphs": G, "nodes_per_graph": n, "D": D, "n_iters": N_ITERS}
        for k, v in times.items():
            res[f"{k}_ms"] = round(float(np.median(v)), 3)
            res[f"{k}_ms_all"] = [round(t, 3) for t in v]
        for arm, bound in arms.items():
            res[f"{arm}_peak_GB"] = round(peak_bytes(lambda: with_bound(bound, fwd_bwd)) / 1e9, 3)
        ya, yb = with_bound(arms["fused"], fwd), with_bound(0, fwd)
        res["rel_diff_fused_vs_composed"] = float(torch.linalg.norm(ya - yb) / torch.linalg.norm(yb))
        del ya, yb
        res.update({"gpu": name_, "power_limit_w": plimit, "sm_clock_mhz": clock})
        if args.profile:
            t0 = time.perf_counter()
            f_ms, b_ms, dev_ms = profile(lambda: with_bound(arms["fused"], fwd_bwd))
            res["profile_wall_ms"] = round((time.perf_counter() - t0) * 1e3, 3)
            res["profile_attend_fwd_ms"] = round(f_ms, 3)
            res["profile_attend_bwd_ms"] = round(b_ms, 3)
            res["profile_device_ms"] = round(dev_ms, 3)
            xb = N * D * 4
            res["attend_fwd_GBps"] = round(N_ITERS * xb / (f_ms * 1e-3) / 1e9, 1) if f_ms else None
            res["attend_bwd_GBps"] = round(N_ITERS * 2 * xb / (b_ms * 1e-3) / 1e9, 1) if b_ms else None
        print(json.dumps(res), flush=True)
        del g, l, x, params
        torch.cuda.empty_cache()


if __name__ == "__main__":
    main()
