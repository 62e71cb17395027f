"""Time the dense layer's pullback at config 2's shape (N = 10 M rows, 128 -> 128, relu, dx, dW and db) on cuda:0: the
fused gnnb_linear_bwd against the three-pass composition it replaced (gnnb_bias_act_bwd, gnnb_linear on W^T, the dW
kernel alone), alternated in one process after a warm-up.  One JSON line: ms per call (CUDA events), algorithmic HBM
bytes and GB/s, 3xTF32 tensor FLOP and TFLOP/s, and the card's name, power limit and SM clock read in the same run.

    python scripts/time_dense_pullback.py [--n 10000000] [--rounds 5] [--iters 10]
"""
import argparse
import json
import os
import subprocess
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import gnnb200 as gnn  # noqa: E402


def card():
    out = subprocess.check_output(["nvidia-smi", "--id=0", "--query-gpu=name,power.limit,clocks.sm",
                                   "--format=csv,noheader,nounits"], text=True).strip().split(", ")
    return out[0], float(out[1]), float(out[2])


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--n", type=int, default=10_000_000)
    ap.add_argument("--rounds", type=int, default=5)
    ap.add_argument("--iters", type=int, default=10)
    a = ap.parse_args()
    lib, chk = gnn._lib.lib, gnn._lib.check
    N, D = a.n, 128
    gen = torch.Generator(device="cuda").manual_seed(0)
    x = torch.randn(N, D, device="cuda", generator=gen)
    W = torch.randn(D, D, device="cuda", generator=gen) / D ** 0.5
    dy = torch.randn(N, D, device="cuda", generator=gen)
    y = torch.randn(N, D, device="cuda", generator=gen).clamp(min=0)
    dpre = torch.empty_like(dy); dx = torch.empty_like(x); dW = torch.empty_like(W); db = torch.empty(D, device="cuda")
    Wt = torch.empty_like(W)

    def fused():
        chk(lib.gnnb_linear_bwd(dy.data_ptr(), y.data_ptr(), x.data_ptr(), W.data_ptr(), 1, N, D, D, dpre.data_ptr(),
                                dx.data_ptr(), dW.data_ptr(), db.data_ptr(), None))

    def composition():
        chk(lib.gnnb_bias_act_bwd(dy.data_ptr(), y.data_ptr(), 1, N, D, dpre.data_ptr(), db.data_ptr(), None))
        Wt.copy_(W.t())
        chk(lib.gnnb_linear(dpre.data_ptr(), Wt.data_ptr(), None, 0, N, D, D, dx.data_ptr(), None))
        chk(lib.gnnb_linear_bwd(dpre.data_ptr(), None, x.data_ptr(), W.data_ptr(), 0, N, D, D, None, None,
                                dW.data_ptr(), None, None))

    def timed(fn):
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        for _ in range(a.iters):
            fn()
        e1.record()
        e1.synchronize()
        return e0.elapsed_time(e1) / a.iters

    for fn in (fused, composition, fused, composition):
        fn()
    torch.cuda.synchronize()
    t_f, t_c = [], []
    for _ in range(a.rounds):
        t_f.append(timed(fused))
        t_c.append(timed(composition))
    name, plim, clk = card()
    fbytes = 6 * N * D * 4                      # dx pass: read dy, y, write dx; dW pass: read dy, y, x
    cbytes = 7 * N * D * 4                      # mask pass: read dy, y, write dpre; dx: read dpre, write dx; dW: read dpre, x
    flop = 2 * 3 * 2 * N * D * D                # two products, three tf32 passes each
    f, c = min(t_f), min(t_c)
    print(json.dumps({"n": N, "din": D, "dout": D, "fused_ms": round(f, 3), "composition_ms": round(c, 3),
                      "fused_ms_all": [round(v, 3) for v in t_f], "composition_ms_all": [round(v, 3) for v in t_c],
                      "fused_gb": fbytes / 1e9, "composition_gb": cbytes / 1e9,
                      "fused_gbps": round(fbytes / f / 1e6, 1), "composition_gbps": round(cbytes / c / 1e6, 1),
                      "tensor_tflop": flop / 1e12, "fused_tflops": round(flop / f / 1e9, 1),
                      "composition_tflops": round(flop / c / 1e9, 1), "tc_error": lib.gnnb_dense_tc_error(),
                      "card": name, "power_limit_w": plim, "sm_clock_mhz": clk}))


if __name__ == "__main__":
    main()
