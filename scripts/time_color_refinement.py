"""Time color_refinement (csrc/wl.cu) on cuda:0.  One JSON line per workload.

Workloads:
  (a) 10 000 random bidirected graphs of 23 nodes and 50 edges               (molecules)
  (b) 1 024 random directed graphs of 1 000 nodes and 5 000 edges            (config 4's batch shape)
  (c) RMAT 10 M nodes / 100 M edges
  (d) an undirected path of 10^5 nodes: about 5 * 10^4 rounds, bound by the rounds' launches and read-backs
Each line gives the plan build (timed apart, before the calls), ms per call (CUDA events around whole calls, the
plan already built), the rounds and ms per round, and the card's name, power limit and SM clock read in the same
process.  The comparison arm is the tuple-dict statement of tests/test_color_refinement.py on the host cores, at (a),
(b) and an RMAT sample of 200 000 nodes / 2 000 000 edges (the same generator), timed once.
With --profile, a torch.profiler run of one call per workload (separate from the timed calls) splits the device time
into the signature kernel (and its fix-up), the radix sort, and the relabel (heads, scans, assign, pack), and gives
the signature kernel's algorithmic bytes per second: per round 12 B per edge (col, row, the gathered colour), 16 B
per work item (counted as one per 128 edges) and 16 B per node (the two sums).

    python scripts/time_color_refinement.py [--reps 5] [--profile] [--skip d]
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
sys.path.insert(0, os.path.join(ROOT, "tests"))
import gnnb200 as gnn  # noqa: E402
from test_color_refinement import ref_color_refinement  # noqa: E402


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


def batch(G, n1, e1, bidirected, gen):
    off = (torch.arange(G, device="cuda") * n1).repeat_interleave(e1)
    s = torch.randint(0, n1, (G * e1,), device="cuda", generator=gen) + off
    t = torch.randint(0, n1, (G * e1,), device="cuda", generator=gen) + off
    if bidirected:
        s, t = torch.cat([s, t]), torch.cat([t, s])
    return s, t, G * n1


def profile(fn, E, n, n_items, rounds):
    from torch.profiler import ProfilerActivity, profile as tprofile
    torch.cuda.synchronize()
    with tprofile(activities=[ProfilerActivity.CPU, ProfilerActivity.CUDA]) as prof:
        t0 = time.perf_counter()
        fn()
        torch.cuda.synchronize()
        wall = (time.perf_counter() - t0) * 1e3
    sig = sort = relabel = other = 0.0
    host = {}
    for e in prof.events():
        if getattr(e, "device_type", None) != torch.autograd.DeviceType.CUDA:
            if e.name.startswith("cuda"):                           # runtime API calls on the host
                host[e.name] = host.get(e.name, 0.0) + e.time_range.elapsed_us() / 1e3
            continue
        t = e.time_range.elapsed_us() / 1e3
        if "wl_signature_kernel" in e.name or "wl_fixup_kernel" in e.name:
            sig += t
        elif "Radix" in e.name or "Onesweep" in e.name:
            sort += t
        elif "wl_" in e.name or "Scan" in e.name:
            relabel += t
        else:
            other += t
    sig_bytes = rounds * (12 * E + 16 * n_items + 16 * n)
    top = sorted(host.items(), key=lambda kv: -kv[1])[:4]
    return {"profile_wall_ms": round(wall, 3), "profile_host_api_ms": {k: round(v, 3) for k, v in top},
            "profile_signature_ms": round(sig, 3), "profile_sort_ms": round(sort, 3),
            "profile_relabel_ms": round(relabel, 3), "profile_other_ms": round(other, 3),
            "signature_alg_bytes": sig_bytes, "signature_gbps": round(sig_bytes / sig / 1e6, 1) if sig else None}


def host_statement(s, t, n):
    t0 = time.perf_counter()
    _, k, it = ref_color_refinement(s, t, n)
    return round((time.perf_counter() - t0) * 1e3, 1), k, it


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--profile", action="store_true")
    ap.add_argument("--skip", default="")
    args = ap.parse_args()
    torch.cuda.set_device(0)
    gen = torch.Generator(device="cuda").manual_seed(17)
    for name in "abcd":
        if name in args.skip:
            continue
        if name == "a":
            s, t, n = batch(10_000, 23, 25, True, gen)
        elif name == "b":
            s, t, n = batch(1024, 1000, 5000, False, gen)
        elif name == "c":
            g0 = gnn.rmat_graph(10 ** 7, 10 ** 8, seed=17, device="cuda")
            s, t, n = g0.s - 1, g0.t - 1, g0.num_nodes
            del g0
        else:
            n = 10 ** 5
            a = torch.arange(n - 1, device="cuda")
            s, t = torch.cat([a, a + 1]), torch.cat([a + 1, a])
        E = s.numel()
        g = gnn.GNNGraph(s + 1, t + 1, num_nodes=n)
        build_ms, _ = event_ms(lambda: g.plan())
        call = lambda: gnn.color_refinement(g)                       # noqa: E731
        t0 = time.perf_counter()                                     # warm-up: modules, items, CUB algorithms, clocks
        while True:
            call()
            torch.cuda.synchronize()
            if time.perf_counter() - t0 > 1.0 or name == "d":
                break
        times, res = [], None
        for _ in range(args.reps if name != "d" else 1):
            ms, res = event_ms(call)
            times.append(ms)
        _, k, rounds = res
        name_, plimit, clock = card()
        out = {"workload": name, "num_nodes": n, "num_edges": E, "plan_build_ms": round(build_ms, 3),
               "ms": round(float(np.median(times)), 3), "ms_all": [round(x, 3) for x in times], "rounds": rounds,
               "ms_per_round": round(float(np.median(times)) / rounds, 4), "num_colors": k,
               "gpu": name_, "power_limit_w": plimit, "sm_clock_mhz": clock}
        if name in "ab":
            out["host_statement_ms"], hk, hit = host_statement(s.cpu().numpy(), t.cpu().numpy(), n)
            out["host_statement_agrees"] = (hk, hit) == (k, rounds)
        if args.profile and name != "d":
            out.update(profile(call, E, n, -(-E // 128), rounds))      # about one work item per 128-edge chunk
        print(json.dumps(out), flush=True)
        del g, s, t
        torch.cuda.empty_cache()
    if "c" not in args.skip:
        g = gnn.rmat_graph(200_000, 2_000_000, seed=17, device="cuda")
        s, t = g.s.cpu().numpy() - 1, g.t.cpu().numpy() - 1
        ms, _ = event_ms(lambda: gnn.color_refinement(g))
        ms, (_, k, rounds) = event_ms(lambda: gnn.color_refinement(g))
        hms, hk, hit = host_statement(s, t, 200_000)
        print(json.dumps({"workload": "c_sample", "num_nodes": 200_000, "num_edges": 2_000_000, "ms": round(ms, 3),
                          "rounds": rounds, "num_colors": k, "host_statement_ms": hms,
                          "host_statement_agrees": (hk, hit) == (k, rounds)}), flush=True)


if __name__ == "__main__":
    main()
