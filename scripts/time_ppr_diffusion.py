"""Time ppr_diffusion (csrc/ppr.cu, and the dense route for graphs above the shared-memory bound) on cuda:0.
One JSON line per workload.

Workloads (batches of equal-sized random bidirected graphs with 2n edges each, no weights, alpha = 0.85; an average
in-degree of 2 keeps I - 0.15 A well away from singular):
  (a) 10 000 graphs of 23 nodes and 50 edges               (molecules)
  (b) 1 000 graphs of 150 nodes
  (c) 128 graphs at the shared-memory bound (240 nodes)
  (d) 256 graphs of 1 000 nodes                            (the dense route)
  (e) one graph of 10 000 nodes                            (the dense route)
Arms, alternated round by round in this process, each timed with CUDA events around whole calls (median of --rounds):
  * ppr_diffusion, end to end (segments, routing, the inverses, the new weights);
  * `inv`: what a user would write with torch alone — the padded per-graph dense M from the edge list (index_put),
    torch.linalg.inv of the batch, and the gather of alpha * inv[t, s];
  * `whole`: the reference's route on the device — the whole batch's dense N x N M, one torch.linalg.inv and the
    gather — where M, its inverse and the solver's workspace fit (N <= 32 768); otherwise its bytes are reported.
With --profile, a torch.profiler trace of one call per workload (a separate run of the calls) adds the device time of
the shared-memory kernel, of the dense route's matrix kernel, of all device work, and the call's wall time.
Each line also carries the card's name, power limit and the SM clock read after the timed calls, and the normwise
relative difference of the new weights between the arms.

    python scripts/time_ppr_diffusion.py [--rounds 5] [--profile] [--only a,b]
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

ALPHA = 0.85
WHOLE_MAX_NODES = 32_768


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


def make_batch(rng, G, n, pairs):
    """G random bidirected graphs of n nodes and 2 * pairs edges (no self loops), as one batched COO (0-based)"""
    a = rng.integers(0, n, (G, pairs))
    b = (a + rng.integers(1, n, (G, pairs))) % n
    off = (np.arange(G) * n)[:, None]
    s = np.concatenate([a + off, b + off], axis=1).ravel()
    t = np.concatenate([b + off, a + off], axis=1).ravel()
    return s, t


def padded_inv(s, t, G, n):
    """per-graph dense M = I + (alpha - 1) A, torch.linalg.inv of the batch, alpha * inv[t, s]"""
    a32 = float(np.float32(ALPHA))
    A = torch.zeros((G, n, n), device="cuda")
    A.index_put_((t // n, t % n, s % n), torch.ones(s.numel(), device="cuda"), accumulate=True)
    M = torch.eye(n, device="cuda") + (a32 - 1) * A
    del A
    inv = torch.linalg.inv(M)
    return a32 * inv[t // n, t % n, s % n]


def whole_inv(s, t, N):
    """the reference: the whole batch's dense M and one inverse"""
    return padded_inv(s, t, 1, N)


def profile(fn):
    from torch.profiler import ProfilerActivity, profile as tprofile
    torch.cuda.synchronize()
    with tprofile(activities=[ProfilerActivity.CPU, ProfilerActivity.CUDA]) as prof:
        t0 = time.perf_counter()
        fn()
        torch.cuda.synchronize()
        wall = (time.perf_counter() - t0) * 1e3
    smem = mat = dev = 0.0
    for e in prof.events():                                # device-side kernel and memcpy / memset records
        if getattr(e, "device_type", None) != torch.autograd.DeviceType.CUDA:
            continue
        t = e.time_range.elapsed_us() / 1e3
        dev += t
        if "ppr_matrix_kernel" in e.name:
            mat += t
        elif "ppr_kernel" in e.name:
            smem += t
    return {"profile_smem_kernel_ms": round(smem, 3), "profile_matrix_kernel_ms": round(mat, 3),
            "profile_device_ms": round(dev, 3), "profile_wall_ms": round(wall, 3)}


def rel(a, b):
    return float(torch.linalg.norm(a.double() - b.double()) / torch.linalg.norm(b.double()))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rounds", type=int, default=5)
    ap.add_argument("--profile", action="store_true")
    ap.add_argument("--only", default="a,b,c,d,e")
    args = ap.parse_args()
    torch.cuda.set_device(0)
    rng = np.random.default_rng(0)
    workloads = [("a", 10_000, 23, 25), ("b", 1_000, 150, 150), ("c", 128, 240, 240), ("d", 256, 1_000, 1_000),
                 ("e", 1, 10_000, 10_000)]
    for name, G, n, pairs in workloads:
        if name not in args.only.split(","):
            continue
        s_np, t_np = make_batch(rng, G, n, pairs)
        N = G * n
        s, t = torch.as_tensor(s_np, device="cuda"), torch.as_tensor(t_np, device="cuda")
        gi = torch.arange(1, G + 1, device="cuda").repeat_interleave(n)
        g = gnn.GNNGraph(s + 1, t + 1, num_nodes=N, num_graphs=G, graph_indicator=gi if G > 1 else None)
        g.plan()
        arms = {"ms": lambda: gnn.ppr_diffusion(g, alpha=ALPHA).w,           # noqa: E731
                "inv_ms": lambda: padded_inv(s, t, G, n)}                    # noqa: E731
        if G > 1 and N <= WHOLE_MAX_NODES:
            arms["whole_ms"] = lambda: whole_inv(s, t, N)                    # noqa: E731
        outs = {k: fn() for k, fn in arms.items()}                           # warm-up: modules, plans, algorithms
        times = {k: [] for k in arms}
        for _ in range(args.rounds):
            for k, fn in arms.items():
                times[k].append(event_ms(fn)[0])
        name_, plimit, clock = card()
        res = {"workload": name, "graphs": G, "nodes_per_graph": n, "edges_per_graph": 2 * pairs,
               "route": "smem" if n <= 240 else "dense"}
        for k, v in times.items():
            res[k] = round(float(np.median(v)), 3)
            res[k + "_all"] = [round(x, 3) for x in v]
        res["rel_diff_vs_inv"] = rel(outs["ms"], outs["inv_ms"])
        if "whole_ms" in outs:
            res["rel_diff_vs_whole"] = rel(outs["ms"], outs["whole_ms"])
        elif G == 1:
            res["whole_ms"] = res["inv_ms"]                                  # one graph: the whole batch is the inv arm
        res.update({"gpu": name_, "power_limit_w": plimit, "sm_clock_mhz": clock,
                    "gj_flops": 2 * n ** 3 * G, "whole_batch_dense_bytes": 4 * N * N})
        if args.profile:
            res.update(profile(arms["ms"]))
        print(json.dumps(res), flush=True)
        del g, outs


if __name__ == "__main__":
    main()
