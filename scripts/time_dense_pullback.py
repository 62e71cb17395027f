"""Time the dense layer's pullback at config 2's shape (N = 10 M rows, 128 -> 128, relu, dx, dW and db) on cuda:0: the
fused pullback reading the relu mask bits (gnnb_linear_bwd_mask) against the same pullback reading y (gnnb_linear_bwd),
alternated in one process after a warm-up.  One JSON line: ms per call (CUDA events), algorithmic HBM bytes and GB/s,
3xTF32 tensor FLOP and TFLOP/s, and the card's name, power limit and SM clock read in the same run.  --profile adds a
second line: mean device time per kernel of each path from torch.profiler, in a run of its own after the timing.

    python scripts/time_dense_pullback.py [--n 10000000] [--rounds 5] [--iters 10] [--profile]
"""
import argparse
import json
import os
import subprocess
import sys
from collections import defaultdict

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import gnnb200 as gnn  # noqa: E402


def card():
    out = subprocess.check_output(["nvidia-smi", "--id=0", "--query-gpu=name,power.limit,clocks.sm",
                                   "--format=csv,noheader,nounits"], text=True).strip().split(", ")
    return out[0], float(out[1]), float(out[2])


def kernel_means(fn, iters):
    """mean device ms per launch of each kernel `fn` runs, over `iters` calls"""
    from torch.profiler import ProfilerActivity, profile
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        for _ in range(iters):
            fn()
        torch.cuda.synchronize()
    tot, cnt = defaultdict(float), defaultdict(int)
    for e in prof.events():
        if e.device_type == torch.autograd.DeviceType.CUDA:
            tot[e.name] += e.device_time_total / 1e3
            cnt[e.name] += 1
    return {k: round(tot[k] / cnt[k], 3) for k in sorted(tot)}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--n", type=int, default=10_000_000)
    ap.add_argument("--rounds", type=int, default=5)
    ap.add_argument("--iters", type=int, default=10)
    ap.add_argument("--profile", action="store_true")
    a = ap.parse_args()
    lib, chk = gnn._lib.lib, gnn._lib.check
    N, D = a.n, 128
    gen = torch.Generator(device="cuda").manual_seed(0)
    x = torch.randn(N, D, device="cuda", generator=gen)
    W = torch.randn(D, D, device="cuda", generator=gen) / D ** 0.5
    b = torch.randn(D, device="cuda", generator=gen)
    dy = torch.randn(N, D, device="cuda", generator=gen)
    y = torch.empty(N, D, device="cuda")
    mask = torch.empty(N, 4, dtype=torch.int32, device="cuda")
    chk(lib.gnnb_linear_relu_mask(x.data_ptr(), W.data_ptr(), b.data_ptr(), N, D, D, y.data_ptr(), mask.data_ptr(), None))
    dpre = torch.empty_like(dy); dx = torch.empty_like(x); dW = torch.empty_like(W); db = torch.empty(D, device="cuda")

    def with_mask():
        chk(lib.gnnb_linear_bwd_mask(dy.data_ptr(), mask.data_ptr(), x.data_ptr(), W.data_ptr(), N, D, D, dx.data_ptr(),
                                     dW.data_ptr(), db.data_ptr(), None))

    def with_y():
        chk(lib.gnnb_linear_bwd(dy.data_ptr(), y.data_ptr(), x.data_ptr(), W.data_ptr(), 1, N, D, D, dpre.data_ptr(),
                                dx.data_ptr(), dW.data_ptr(), db.data_ptr(), None))

    def timed(fn):
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        for _ in range(a.iters):
            fn()
        e1.record()
        e1.synchronize()
        return e0.elapsed_time(e1) / a.iters

    for fn in (with_mask, with_y, with_mask, with_y):
        fn()
    torch.cuda.synchronize()
    t_m, t_y = [], []
    for _ in range(a.rounds):
        t_m.append(timed(with_mask))
        t_y.append(timed(with_y))
    name, plim, clk = card()
    # dx pass: read dy and the mask (16 B per row) or y, write dx; dW pass: read dy, the mask or y, and x
    mbytes = 4 * N * D * 4 + 2 * N * 16
    ybytes = 6 * N * D * 4
    flop = 2 * 3 * 2 * N * D * D                # two products, three tf32 passes each
    m, yv = min(t_m), min(t_y)
    print(json.dumps({"n": N, "din": D, "dout": D, "mask_ms": round(m, 3), "y_ms": round(yv, 3),
                      "mask_ms_all": [round(v, 3) for v in t_m], "y_ms_all": [round(v, 3) for v in t_y],
                      "mask_gb": mbytes / 1e9, "y_gb": ybytes / 1e9,
                      "mask_gbps": round(mbytes / m / 1e6, 1), "y_gbps": round(ybytes / yv / 1e6, 1),
                      "tensor_tflop": flop / 1e12, "mask_tflops": round(flop / m / 1e9, 1),
                      "y_tflops": round(flop / yv / 1e9, 1), "tc_error": lib.gnnb_dense_tc_error(),
                      "card": name, "power_limit_w": plim, "sm_clock_mhz": clk}))
    if a.profile:
        print(json.dumps({"kernel_ms_mask": kernel_means(with_mask, a.iters), "kernel_ms_y": kernel_means(with_y, a.iters)}))


if __name__ == "__main__":
    main()
