"""Time rand_temporal_radius_graph / rand_temporal_hyperbolic_graph (csrc/tgen.cu + the count / fill of csrc/knn.cu) on
cuda:0.  One JSON line per workload.

Each line: ms per whole generator call (CUDA events around synchronised calls, after warm-up), the card's name, power
limit and SM clock read in the same run, pairs/s (T n² ordered pairs, each visited by the count and by the fill) and
the share of the issue bound.  Radius: the fp32 bound, 3d = 6 separately rounded instructions per pair and pass over
132 SMs x 128 fp32 lanes x the sampled SM clock.  Hyperbolic: the data sheet's 34 TFLOP/s of non-tensor FP64 (H100
SXM) counts an FMA as two flops, i.e. 17 T fp64 instructions/s; a pair costs 7 separately rounded fp64 instructions per
pass, so the bound is 2 x 7 x T n² / 17e12 s.  Beside them the reference's host algorithms: scipy's
cKDTree.query_ball_point per snapshot, and a vectorised numpy float64 statement of the hyperbolic double loop
(generate.jl:353-361, acosh of every ordered pair) on a few snapshots, reported per snapshot.

    python scripts/time_temporal_generators.py [--iters 10] [--warmup 2]
"""
import argparse
import json
import math
import os
import subprocess
import sys
import time

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import gnnb200 as gnn  # noqa: E402

FP64_INSTR_PER_S = 34e12 / 2          # data sheet, H100 SXM, non-tensor FP64, FMA counted as two flops


def card():
    try:
        out = subprocess.check_output(["nvidia-smi", "--id=0", "--query-gpu=name,power.limit,clocks.sm",
                                       "--format=csv,noheader,nounits"], text=True).strip().split(", ")
        return out[0], float(out[1]), float(out[2])
    except Exception:
        return torch.cuda.get_device_name(0), float("nan"), float("nan")


def timed(fn, iters, warmup):
    for _ in range(warmup):
        fn()
    torch.cuda.synchronize()
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    a.record()
    for _ in range(iters):
        fn()
    b.record()
    torch.cuda.synchronize()
    return a.elapsed_time(b) / iters


def host_radius(n, T, speed, r, seed, snaps):
    """cKDTree.query_ball_point on the device's own positions, per snapshot"""
    from scipy.spatial import cKDTree
    from gnnb200 import _lib
    pts = torch.empty((T * n, 2), dtype=torch.float32, device="cuda")
    _lib.check(_lib.lib.gnnb_temporal_radius_points(n, T, speed, seed, pts.data_ptr(),
                                                    torch.cuda.current_stream().cuda_stream))
    P = pts.cpu().numpy().astype(np.float64).reshape(T, n, 2)
    t0 = time.perf_counter()
    for t in range(snaps):
        cKDTree(P[t]).query_ball_point(P[t], r, workers=-1)
    return (time.perf_counter() - t0) * 1e3 / snaps


def host_hyperbolic(n, alpha, R, zeta, snaps, chunk=1000):
    """generate.jl:353-361 in vectorised numpy float64: acosh of every ordered pair, one snapshot at a time"""
    rng = np.random.default_rng(0)
    t0 = time.perf_counter()
    for _ in range(snaps):
        p = rng.random(n)
        r = (1 / alpha) * np.arccosh(1 + (math.cosh(alpha * R) - 1) * p)
        th = 2 * np.pi * rng.random(n)
        adj = np.zeros((n, n), np.float32)
        for a in range(0, n, chunk):
            A = np.cosh(zeta * r[a:a + chunk, None]) * np.cosh(zeta * r[None, :])
            B = np.sinh(zeta * r[a:a + chunk, None]) * np.sinh(zeta * r[None, :])
            c = np.cos(np.pi - np.abs(np.pi - np.abs(th[a:a + chunk, None] - th[None, :])))
            with np.errstate(invalid="ignore"):
                d = np.arccosh(A - B * c) / zeta
            adj[a:a + chunk] = d <= R
    return (time.perf_counter() - t0) * 1e3 / snaps


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--iters", type=int, default=10)
    ap.add_argument("--warmup", type=int, default=2)
    ap.add_argument("--host-snapshots", type=int, default=2)
    args = ap.parse_args()
    torch.cuda.set_device(0)
    n_big, T_big = 20000, 64
    workloads = [("radius", 30, 5, dict(speed=0.1, r=0.1)),
                 ("hyperbolic", 30, 5, dict(α=1.0, R=1.0, speed=0.1, ζ=1.0)),
                 ("radius", n_big, T_big, dict(speed=0.01, r=math.sqrt(10 / (math.pi * n_big)))),
                 ("hyperbolic", n_big, T_big, dict(α=1.0, R=2 * math.log(n_big), speed=0.01, ζ=1.0))]
    for kind, n, T, kw in workloads:
        if kind == "radius":
            fn = lambda: gnn.rand_temporal_radius_graph(n, T, kw["speed"], kw["r"], seed=1, device="cuda")
        else:
            fn = lambda: gnn.rand_temporal_hyperbolic_graph(n, T, seed=1, device="cuda", **kw)
        ms = timed(fn, args.iters, args.warmup)
        tg = fn()
        name, plimit, clock = card()
        pairs = T * n * n
        res = {"workload": kind, "n": n, "T": T, **{k: round(v, 6) for k, v in kw.items()},
               "ms": round(ms, 3), "iters": args.iters, "gpu": name, "power_limit_w": plimit, "sm_clock_mhz": clock,
               "edges": sum(tg.num_edges), "mean_degree": round(sum(tg.num_edges) / (n * T), 2),
               "pairs_per_s": pairs / (ms * 1e-3)}
        if kind == "radius":
            bound_s = 2 * pairs * 6 / (132 * 128 * clock * 1e6)
            res["bound"] = "fp32 issue: 6 instructions per pair and pass, 132 SMs x 128 lanes x sampled SM clock"
        else:
            bound_s = 2 * pairs * 7 / FP64_INSTR_PER_S
            res["bound"] = "fp64: 7 instructions per pair and pass against 34 TFLOP/s (17e12 instructions/s)"
        res["bound_share"] = round(bound_s / (ms * 1e-3), 4)
        if n == n_big:
            try:
                if kind == "radius":
                    res["host_ckdtree_ms_per_snapshot"] = round(host_radius(n, T, kw["speed"], kw["r"], 1,
                                                                            args.host_snapshots), 1)
                    res["host_cores"] = os.cpu_count()
                else:
                    res["host_numpy_ms_per_snapshot"] = round(host_hyperbolic(n, kw["α"], kw["R"], kw["ζ"],
                                                                              args.host_snapshots), 1)
                res["host_snapshots_timed"] = args.host_snapshots
            except ImportError:
                pass
        print(json.dumps(res, ensure_ascii=False), flush=True)


if __name__ == "__main__":
    main()
