"""Time knn_graph / radius_graph neighbour search (csrc/knn.cu) on cuda:0.  One JSON line per workload.

Each line: ms per call (CUDA events, after warm-up), the card's name, power limit and SM clock read in the same run,
pairs/s and the share of the fp32 issue bound (3d separately rounded instructions per pair over 132 SMs x 128 lanes x
the sampled SM clock); torch.cdist + topk beside it (GEMM expansion: a comparison point only, with the number of rows
whose neighbour set differs from the exact one) and scipy's cKDTree on the host cores when scipy imports.

    python scripts/time_knn.py [--iters 20] [--warmup 3]
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
from gnnb200 import _lib  # noqa: E402


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


def knn_entry(x, seg, k, nbr):
    n, d = x.shape
    _lib.check(_lib.lib.gnnb_knn(x.data_ptr(), n, d, None if seg is None else seg.data_ptr(),
                                 1 if seg is None else seg.numel() - 1, k, 0, nbr.data_ptr(),
                                 torch.cuda.current_stream().cuda_stream))


def radius_entries(x, r):
    import ctypes as C
    n, d = x.shape
    off = torch.empty(n + 1, dtype=torch.int64, device="cuda")
    tot = C.c_int64(0)
    s = torch.cuda.current_stream().cuda_stream
    _lib.check(_lib.lib.gnnb_radius_count(x.data_ptr(), n, d, None, 1, r, 0, off.data_ptr(), C.byref(tot), s))
    nbr = torch.empty(tot.value, dtype=torch.int32, device="cuda")
    _lib.check(_lib.lib.gnnb_radius_fill(x.data_ptr(), n, d, None, 1, r, 0, off.data_ptr(), nbr.data_ptr(),
                                         tot.value, s))
    return off, nbr


def cdist_topk(x, clouds, k, chunk=4096):
    """per cloud, torch.cdist + topk(k + 1) minus self; returns (n, k) sorted ids"""
    n, d = x.shape
    per = n // clouds
    out = torch.empty((n, k), dtype=torch.int64, device="cuda")
    if per <= chunk:
        xb = x.reshape(clouds, per, d)
        idx = torch.cdist(xb, xb).topk(k + 1, largest=False).indices[:, :, 1:]
        return (idx + (torch.arange(clouds, device="cuda") * per)[:, None, None]).reshape(n, k)
    for c in range(clouds):
        xc = x[c * per:(c + 1) * per]
        for q0 in range(0, per, chunk):
            idx = torch.cdist(xc[q0:q0 + chunk], xc).topk(k + 1, largest=False).indices[:, 1:]
            out[c * per + q0:c * per + q0 + chunk] = idx + c * per
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--iters", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=3)
    args = ap.parse_args()
    torch.cuda.set_device(0)
    rng = np.random.default_rng(0)
    try:
        from scipy.spatial import cKDTree
    except ImportError:
        cKDTree = None
    workloads = [("knn", 1024, 1024, 3, 16), ("knn", 1, 2 ** 18, 3, 16), ("knn", 64, 2048, 64, 20),
                 ("radius", 1, 2 ** 18, 3, 0.031)]
    for kind, clouds, per, d, kr in workloads:
        n = clouds * per
        P = rng.random((n, d)).astype(np.float32)
        x = torch.as_tensor(P).cuda()
        seg = None if clouds == 1 else torch.arange(clouds + 1, device="cuda", dtype=torch.int64) * per
        pairs = clouds * per * per
        res = {"workload": kind, "clouds": clouds, "points_per_cloud": per, "d": d}
        if kind == "knn":
            k = int(kr)
            res["k"] = k
            nbr = torch.empty((n, k), dtype=torch.int32, device="cuda")
            ms = timed(lambda: knn_entry(x, seg, k, nbr), args.iters, args.warmup)
            ref_ms = timed(lambda: cdist_topk(x, clouds, k), max(3, args.iters // 4), 1)
            mine = torch.sort(nbr.long(), dim=1).values
            theirs = torch.sort(cdist_topk(x, clouds, k), dim=1).values
            res["cdist_topk_ms"] = round(ref_ms, 3)
            res["cdist_topk_rows_differing"] = int((mine != theirs).any(dim=1).sum())
        else:
            r = float(kr)
            res["r"] = r
            ms = timed(lambda: radius_entries(x, r), args.iters, args.warmup)
            off, _ = radius_entries(x, r)
            res["edges"] = int(off[-1])
            res["mean_degree"] = round(int(off[-1]) / n, 2)
        name, plimit, clock = card()
        res.update({"ms": round(ms, 3), "iters": args.iters, "gpu": name, "power_limit_w": plimit,
                    "sm_clock_mhz": clock, "pairs_per_s": pairs / (ms * 1e-3)})
        passes = 2 if kind == "radius" else 1                         # count and fill each visit every pair
        bound_s = passes * pairs * 3 * d / (132 * 128 * clock * 1e6)
        res["fp32_issue_bound_share"] = round(bound_s / (ms * 1e-3), 3)
        if cKDTree is not None:
            sub = clouds if d <= 3 else min(clouds, 4)
            t0 = time.perf_counter()
            for c in range(sub):
                pc = P[c * per:(c + 1) * per]
                tree = cKDTree(pc)
                if kind == "knn":
                    tree.query(pc, int(kr) + 1, workers=-1)
                else:
                    tree.query_ball_point(pc, float(kr), workers=-1)
            res["ckdtree_ms"] = round((time.perf_counter() - t0) * 1e3, 1)
            res["ckdtree_clouds_timed"] = sub
            res["ckdtree_cores"] = os.cpu_count()
        print(json.dumps(res), flush=True)


if __name__ == "__main__":
    main()
