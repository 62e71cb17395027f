"""Time global_attention_pool on cuda:0: the fused pass (gnnb_attention_pool, csrc/set2set.cu) against the composition on
the existing kernels (softmax_nodes, the D x N product α .* f, reduce_nodes), the route taken above the bound.  One JSON
line per workload.

The pooled features are given (ffeat and fgate are the identity on precomputed arrays), so what is timed is the pooling
alone:
  (a-c) 10 000 graphs of 23 nodes (molecules) at D = 64, 128 and 256
  (d)   1 024 graphs of 1 000 nodes, D = 128
  (e)   one graph of 10 M nodes, D = 128 (one long row of the indicator plan: partial slots and the fix-up)
Arms, alternated round by round in this process, each timed with CUDA events around whole calls: `fused` (the default)
and `composed` (the bound patched to 0), each as the forward alone and as forward + backward (f and the gate require
grad).  Each line carries the largest normwise relative difference between the two arms' outputs and gradients, and the
card's name, power limit and SM clock read after the timed calls.

    python scripts/time_global_attention_pool.py [--rounds 7] [--only a,b,c,d,e]
"""
import argparse
import json
import os
import subprocess
import sys

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import gnnb200 as gnn  # noqa: E402
from gnnb200 import readout  # noqa: E402


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
    saved = readout._ATTENTION_POOL_MAX_D
    readout._ATTENTION_POOL_MAX_D = bound
    try:
        return fn()
    finally:
        readout._ATTENTION_POOL_MAX_D = saved


def rel(a, b):
    return float(torch.linalg.norm(a - b) / torch.linalg.norm(b))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rounds", type=int, default=7)
    ap.add_argument("--only", default="a,b,c,d,e")
    args = ap.parse_args()
    torch.cuda.set_device(0)
    workloads = [("a", 10_000, 23, 64), ("b", 10_000, 23, 128), ("c", 10_000, 23, 256), ("d", 1_024, 1_000, 128),
                 ("e", 1, 10_000_000, 128)]
    for name, G, n, D in workloads:
        if name not in args.only.split(","):
            continue
        N = G * n
        a = torch.arange(1, N + 1, device="cuda")
        gi = torch.arange(1, G + 1, device="cuda").repeat_interleave(n)
        g = gnn.GNNGraph(a, a, num_nodes=N, num_graphs=G, graph_indicator=gi if G > 1 else None)
        torch.manual_seed(0)
        f = gnn.unrows(torch.randn(N, D, device="cuda")).requires_grad_(True)
        gate = (torch.randn(1, N, device="cuda") * 2).requires_grad_(True)
        l = gnn.GlobalAttentionPool(lambda x: gate, lambda x: f)
        cot = torch.randn(D, G, device="cuda")

        def fwd():
            with torch.no_grad():
                return l(g, f)

        def fwd_bwd():
            return torch.autograd.grad((l(g, f) * cot).sum(), [f, gate])

        arms = {"fused": readout._ATTENTION_POOL_MAX_D, "composed": 0}
        for bound in arms.values():                       # warm-up: modules, plans, algorithms
            with_bound(bound, fwd)
            with_bound(bound, fwd_bwd)
        times = {f"{arm}_{kind}": [] for arm in arms for kind in ("fwd", "fwd_bwd")}
        for _ in range(args.rounds):
            for arm, bound in arms.items():
                times[f"{arm}_fwd"].append(event_ms(lambda: with_bound(bound, fwd))[0])
                times[f"{arm}_fwd_bwd"].append(event_ms(lambda: with_bound(bound, fwd_bwd))[0])
        name_, plimit, clock = card()
        res = {"workload": name, "graphs": G, "nodes_per_graph": n, "D": D}
        for k, v in times.items():
            res[f"{k}_ms"] = round(float(np.median(v)), 3)
            res[f"{k}_ms_all"] = [round(t, 3) for t in v]
        for kind in ("fwd", "fwd_bwd"):
            res[f"speedup_{kind}"] = round(res[f"composed_{kind}_ms"] / res[f"fused_{kind}_ms"], 3)
        outs = [with_bound(b, lambda: (fwd(),) + fwd_bwd()) for b in arms.values()]
        res["rel_diff_fused_vs_composed"] = max(rel(x, y) for x, y in zip(*outs))
        del outs
        res.update({"gpu": name_, "power_limit_w": plimit, "sm_clock_mhz": clock})
        print(json.dumps(res), flush=True)
        del g, f, gate, l
        torch.cuda.empty_cache()


if __name__ == "__main__":
    main()
