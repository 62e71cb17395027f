"""Time the three 3xTF32 kernels of a GCNConv dense layer at config 2's shape (N = 10 M rows, 128 -> 128, relu) alone on
cuda:0: the forward with its relu mask (gnnb_linear_relu_mask, one kernel) and the pullback reading the mask
(gnnb_linear_bwd_mask: the dx kernel, the dW kernel and the split-K reduction), from torch.profiler's device time per
launch in a run after a CUDA-event-timed warm-up.  One JSON line: ms and algorithmic GB/s per kernel, the share of the
HBM peak (MEASURED_PEAKS.json when present, else the H100 SXM data sheet's 3.35 TB/s, said which), and the card's name,
power limit and SM clock read in the same run.

    python scripts/time_dense_ring.py [--n 10000000] [--iters 20]
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


def hbm_peak():
    path = os.path.join(ROOT, "MEASURED_PEAKS.json")
    if os.path.exists(path):
        with open(path) as f:
            return float(json.load(f)["hbm_gbs"]), "measured (MEASURED_PEAKS.json hbm_gbs)"
    return 3350.0, "H100 SXM data sheet (3.35 TB/s HBM3), not a measurement"


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--n", type=int, default=10_000_000)
    ap.add_argument("--iters", type=int, default=20)
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
    dx = torch.empty_like(x); dW = torch.empty_like(W); db = torch.empty(D, device="cuda")

    def forward():
        chk(lib.gnnb_linear_relu_mask(x.data_ptr(), W.data_ptr(), b.data_ptr(), N, D, D, y.data_ptr(), mask.data_ptr(), None))

    def pullback():
        chk(lib.gnnb_linear_bwd_mask(dy.data_ptr(), mask.data_ptr(), x.data_ptr(), W.data_ptr(), N, D, D, dx.data_ptr(),
                                     dW.data_ptr(), db.data_ptr(), None))

    calls = {}
    for name, fn in (("forward", forward), ("pullback", pullback)):
        for _ in range(3):
            fn()
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        for _ in range(a.iters):
            fn()
        e1.record()
        e1.synchronize()
        calls[name] = round(e0.elapsed_time(e1) / a.iters, 3)

    from torch.profiler import ProfilerActivity, profile
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        for _ in range(a.iters):
            forward()
            pullback()
        torch.cuda.synchronize()
    tot, cnt = defaultdict(float), defaultdict(int)
    for e in prof.events():
        if e.device_type == torch.autograd.DeviceType.CUDA:
            tot[e.name] += e.device_time_total / 1e3
            cnt[e.name] += 1
    ms = {k: tot[k] / cnt[k] for k in tot}

    def find(tag):
        hit = [k for k in ms if tag in k]
        return ms[hit[0]] if hit else None

    row_in, row_out, mask_b = 4 * D, 4 * D, 16
    kernels = {   # algorithmic HBM bytes per launch
        "linear_relu_mask_kernel": N * (row_in + row_out + mask_b),
        "linear_bwd_dx_mask_kernel": N * (row_in + mask_b + row_out),
        "linear_bwd_dw_mask_kernel": N * (row_in + mask_b + row_in),
    }
    peak, peak_src = hbm_peak()
    out = {"n": N, "call_ms": calls, "peak_gbps": peak, "peak_source": peak_src, "kernels": {}}
    for k, nbytes in kernels.items():
        t = find(k)
        if t is None:
            raise SystemExit(f"kernel {k} not found in the profile: {sorted(ms)}")
        gbps = nbytes / t / 1e6
        out["kernels"][k] = {"ms": round(t, 3), "GB": round(nbytes / 1e9, 2), "GBps": round(gbps), "of_peak": round(gbps / peak, 3)}
    red = find("dw_reduce_kernel")
    out["kernels"]["dw_reduce_kernel"] = {"ms": round(red, 3) if red is not None else None}
    name, plimit, sm = card()
    out.update(card=name, power_limit_w=plimit, sm_clock_mhz=sm)
    print(json.dumps(out))


if __name__ == "__main__":
    main()
