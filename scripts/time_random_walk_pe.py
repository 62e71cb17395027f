"""Time random_walk_pe (csrc/rwpe.cu, and the fused propagate for graphs above the shared-memory bound) on cuda:0.
One JSON line per workload.

Workloads (batches of equal-sized random bidirected graphs, no weights):
  (a) 10 000 graphs of 23 nodes and 50 edges, K = 20       (molecules)
  (b) 1 000 graphs of 150 nodes and 300 edges, K = 16       (peptides)
  (c) 128 graphs at the shared-memory bound (896 nodes, 1 792 edges), K = 16
  (d) one graph of 20 000 nodes and 200 000 edges, K = 16   (above the bound: the propagate route)
Arms, alternated round by round in this process, each timed with CUDA events around whole calls:
  * random_walk_pe, end to end (degree, segments, the walk);
  * `bmm`: a padded per-graph dense RW from the edge list (index_put), then K - 1 torch.bmm products and their
    diagonals — the strongest simple GPU baseline (what a dense per-graph transform amounts to);
  * `scipy`: sparse powers of the block-diagonal RW on the host (scipy's sparse product runs on one thread), for
    context, where the fill-in stays small;
  * the reference's whole-batch dense route: it holds at least three N x N fp32 matrices at once (A, RW and the running
    product), reported as bytes; it is the `bmm` arm when the batch is one graph and those fit in 80 GB.
With --profile, a torch.profiler trace of one call per workload (a separate run of the calls) adds the device time of the
walk kernel, of all device work, and the call's wall time.
Each line also carries the card's name, power limit and the SM clock read after the timed calls, and the largest
normwise relative difference between random_walk_pe and the bmm arm.

    python scripts/time_random_walk_pe.py [--rounds 5] [--profile]
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


def bmm_pe(s, t, G, n, K):
    """padded per-graph dense powers: (K, G * n)"""
    A = torch.zeros((G, n, n), device="cuda")
    A.index_put_((s // n, s % n, t % n), torch.ones(s.numel(), device="cuda"), accumulate=True)
    deg = A.sum(2)
    dinv = torch.where(deg != 0, 1.0 / deg, torch.zeros_like(deg))
    RW = A * dinv[:, None, :]
    out = torch.empty((K, G, n), device="cuda")
    P = RW
    for k in range(K):
        out[k] = torch.diagonal(P, dim1=1, dim2=2)
        if k + 1 < K:
            P = torch.bmm(P, RW)
    return out.reshape(K, G * n)


def scipy_pe(s, t, N, K):
    import scipy.sparse as sp
    A = sp.csr_matrix((np.ones(len(s)), (s, t)), shape=(N, N))
    deg = np.asarray(A.sum(1)).ravel()
    RW = (A @ sp.diags(np.where(deg != 0, 1.0 / np.where(deg != 0, deg, 1), 0.0))).tocsr()
    P, out = RW, np.empty((K, N))
    for k in range(K):
        out[k] = P.diagonal()
        if k + 1 < K:
            P = P @ RW
    return out


def profile(fn):
    """device time of the walk kernel and of all device work in one call, and the call's wall time (ms)"""
    from torch.profiler import ProfilerActivity, profile as tprofile
    torch.cuda.synchronize()
    with tprofile(activities=[ProfilerActivity.CPU, ProfilerActivity.CUDA]) as prof:
        t0 = time.perf_counter()
        fn()
        torch.cuda.synchronize()
        wall = (time.perf_counter() - t0) * 1e3
    walk = dev = 0.0
    for e in prof.events():                                # device-side kernel and memcpy / memset records
        if getattr(e, "device_type", None) != torch.autograd.DeviceType.CUDA:
            continue
        t = e.time_range.elapsed_us() / 1e3
        dev += t
        if "rwpe_kernel" in e.name:
            walk += t
    return {"profile_walk_kernel_ms": round(walk, 3), "profile_device_ms": round(dev, 3),
            "profile_wall_ms": round(wall, 3)}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rounds", type=int, default=5)
    ap.add_argument("--profile", action="store_true")
    args = ap.parse_args()
    torch.cuda.set_device(0)
    rng = np.random.default_rng(0)
    workloads = [("a", 10_000, 23, 25, 20, True), ("b", 1_000, 150, 150, 16, True), ("c", 128, 896, 896, 16, False),
                 ("d", 1, 20_000, 100_000, 16, False)]
    for name, G, n, pairs, K, with_scipy in workloads:
        s_np, t_np = make_batch(rng, G, n, pairs)
        N = G * n
        s, t = torch.as_tensor(s_np, device="cuda"), torch.as_tensor(t_np, device="cuda")
        gi = torch.arange(1, G + 1, device="cuda").repeat_interleave(n)
        g = gnn.GNNGraph(s + 1, t + 1, num_nodes=N, num_graphs=G, graph_indicator=gi if G > 1 else None)
        g.plan()
        ours = lambda: gnn.random_walk_pe(g, K)                          # noqa: E731
        theirs = lambda: bmm_pe(s, t, G, n, K)                           # noqa: E731
        ours(), theirs()                                                 # warm-up: modules, plans, algorithms
        mine, base = [], []
        for _ in range(args.rounds):
            mine.append(event_ms(ours)[0])
            base.append(event_ms(theirs)[0])
        name_, plimit, clock = card()
        a, b = ours(), theirs()
        diff = float(torch.linalg.norm(a - b) / torch.linalg.norm(b))
        res = {"workload": name, "graphs": G, "nodes_per_graph": n, "edges_per_graph": 2 * pairs, "K": K,
               "route": "smem" if n <= 896 else "propagate",
               "ms": round(float(np.median(mine)), 3), "ms_all": [round(x, 3) for x in mine],
               "bmm_ms": round(float(np.median(base)), 3), "bmm_ms_all": [round(x, 3) for x in base],
               "rel_diff_vs_bmm": diff, "gpu": name_, "power_limit_w": plimit, "sm_clock_mhz": clock,
               "lane_multiply_adds": K * 2 * pairs * G * 32 * ((n + 31) // 32) if n <= 896 else None,
               "whole_batch_dense_bytes": 3 * 4 * N * N, "whole_batch_dense_fits_80GB": 3 * 4 * N * N < 80e9}
        if res["whole_batch_dense_fits_80GB"] and G == 1:
            res["whole_batch_dense_ms"] = res["bmm_ms"]                 # one graph: the batch route is the bmm arm
        if with_scipy:
            t0 = time.perf_counter()
            scipy_pe(s_np, t_np, N, K)
            res["scipy_ms"] = round((time.perf_counter() - t0) * 1e3, 1)
            res["scipy_threads"] = 1
        if args.profile:
            res.update(profile(ours))
        print(json.dumps(res), flush=True)
        del g, a, b


if __name__ == "__main__":
    main()
