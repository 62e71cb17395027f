"""Time the fused GCN propagate (gnnb_gcn_propagate, plan-owned normalisation, D = 128) at config 2's shape (RMAT
N = 10 M, E = 100 M + 10 M self loops, seed 17, the self-loop graph built from the planned graph as bench.py does) on
cuda:0, forward and transposed, with the L2 eviction priorities the library chooses at this size (on: the gathered rows
are 100 times the L2; DESIGN.md §4 "L2 policy").  After the timing, each direction's output is checked to be
bit-identical to the reference kernels' (variant 12, plain loads).  One JSON line: ms per pass (CUDA events, best and
all rounds), and the card's name, power limit and SM clock read in the same run.

Lines loaded evict_last would keep that priority after the kernel ends; the propagate demotes its hot rows to
evict_normal after every hinted pass.  The script checks that: it times the reference kernels (variant 12, plain loads)
before any hinted pass and again after each one, and the two must agree (without the demotion a plain pass after a hinted
one was 0.65 ms faster, DESIGN.md §4).  The library has no switch for the policy's parts or budget; the sweep that chose
them (DESIGN.md §4) is not reproducible from here.

    python scripts/time_propagate_l2.py [--n 10000000] [--e 100000000] [--rounds 5] [--iters 10]
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
    ap.add_argument("--e", type=int, default=100_000_000)
    ap.add_argument("--rounds", type=int, default=5)
    ap.add_argument("--iters", type=int, default=10)
    a = ap.parse_args()
    lib, chk = gnn._lib.lib, gnn._lib.check
    N, D = a.n, 128
    g = gnn.rmat_graph(N, a.e, 17, device="cuda")
    g.plan()                                   # as bench.py: the self-loop graph takes its edge order from this plan
    g2 = gnn.add_self_loops(g)
    h = g2.plan().h
    chk(lib.gnnb_graph_csr(h, 1, None, None, None, None))
    x = torch.randn(N, D, device="cuda", generator=torch.Generator(device="cuda").manual_seed(0))
    out = torch.empty_like(x)
    st = torch.cuda.current_stream().cuda_stream

    def run(tr):
        chk(lib.gnnb_gcn_propagate(h, tr, x.data_ptr(), None, None, D, out.data_ptr(), st))

    def timed(tr, v=0):
        chk(lib.gnnb_set_kernel_variant(v))
        try:
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record()
            for _ in range(a.iters):
                run(tr)
            e1.record()
            e1.synchronize()
            return e0.elapsed_time(e1) / a.iters
        finally:
            lib.gnnb_set_kernel_variant(0)

    # the reference kernels (variant 12: plain loads) before any hinted pass, then alternated with the hinted passes:
    # if the evict_last priority outlived a pass, the plain loads after it would find the hot rows still protected
    for tr in (0, 1):
        timed(tr, 12)
    ref_fresh = {tr: timed(tr, 12) for tr in (0, 1)}
    t = {0: [], 1: []}
    ref_after = {0: [], 1: []}
    for _ in range(a.rounds):
        for tr in (0, 1):
            t[tr].append(timed(tr))
            ref_after[tr].append(timed(tr, 12))
    same = {}
    for tr in (0, 1):
        try:
            chk(lib.gnnb_set_kernel_variant(12))
            run(tr)
            ref = out.clone()
        finally:
            lib.gnnb_set_kernel_variant(0)
        run(tr)
        same[tr] = bool(torch.equal(out.view(torch.int32), ref.view(torch.int32)))
        del ref
    torch.cuda.synchronize()
    name, plim, clk = card()
    print(json.dumps({"n": N, "e": a.e, "d": D, "bit_identical_to_reference": same[0] and same[1],
                      "forward_ms": round(min(t[0]), 3), "transposed_ms": round(min(t[1]), 3),
                      "forward_ms_all": [round(v, 3) for v in t[0]], "transposed_ms_all": [round(v, 3) for v in t[1]],
                      "reference_ms_before_hints": [round(ref_fresh[tr], 3) for tr in (0, 1)],
                      "reference_ms_after_hints": [[round(v, 3) for v in ref_after[tr]] for tr in (0, 1)],
                      "card": name, "power_limit_w": plim, "sm_clock_mhz": clk}))


if __name__ == "__main__":
    main()
