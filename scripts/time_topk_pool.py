"""Time top-k pooling (csrc/topk.cu) on cuda:0 against a torch composition.  One JSON line per workload and arm.

Workloads (D = 128, ratio 0.5 in the graph form):
  (a) 10 000 graphs of 23 nodes, graph form, forward and forward + backward
  (b) 1 024 graphs of 1 000 nodes, the same
  (c) RMAT 10 M / 100 M as one graph, the same, plus topk_index alone on 10^7 float32 keys
  (d) the reference form at N = 20 000, k = 10 000, with a dense float32 A (forward and forward + backward)
  (e) gnnb_topk_keep alone on float32 keys around the shared-memory bound: one segment of n keys and 1 024 segments of
      n keys each, for n from 1 024 to GNNB_TOPK_SMEM_MAX, on the default route (one CTA per segment) and with the bound
      forced to 0 (the multi-block passes)
Arms, alternated round by round in this process, each timed with CUDA events around whole calls:
  * `lib`: topk_pool / topk_index;
  * `torch`: y = p @ X / norm(p); one graph: torch.topk and a threshold; a batch: a stable sort by (graph, -y) and a
    per-graph threshold; x[:, idx] * sigmoid(y[idx]) by indexing; remove_nodes for the pooled graph.
The two arms' selections are compared on the same y.  Bytes are the algorithmic ones from shapes: the score reads
N·D·4 B, the gate reads and writes m·D·4 B each, the pullback reads x and dout and writes dx (2·N·D·4 + m·D·4 B).
Each line carries the card's name, power limit and SM clock read after the timed calls.

    python scripts/time_topk_pool.py [--rounds 5] [--only a,b,c,d,e]
"""
import argparse
import json
import math
import os
import re
import subprocess
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import gnnb200 as gnn  # noqa: E402
from gnnb200 import _lib, readout  # noqa: E402

with open(os.path.join(ROOT, "include", "gnnb200.h")) as f:
    BOUND = int(re.search(r"#define GNNB_TOPK_SMEM_MAX (\d+)", f.read()).group(1))
D = 128


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


def batch(G, n, dev):
    """G graphs of n nodes, each a ring with chords (4 edges per node)"""
    i = torch.arange(G * n, device=dev)
    base = (i // n) * n
    s = torch.cat([i, i]) + 1
    t = torch.cat([base + (i - base + 1) % n, base + (i - base + 7) % n]) + 1
    ind = i // n + 1
    return gnn.GNNGraph(s, t, num_nodes=G * n, num_graphs=G, graph_indicator=ind)


def torch_keep(y, ind, G, ratio):
    """stable two-key sort (graph ascending, y descending), per-graph threshold at ceil(ratio n_i)"""
    o1 = torch.sort(y, descending=True, stable=True).indices
    o = o1[torch.sort(ind[o1], stable=True).indices]
    cnt = torch.bincount(ind - 1, minlength=G)
    start = torch.cumsum(cnt, 0) - cnt
    kk = torch.ceil(ratio * cnt.double()).long()
    thr = y[o[(start + kk - 1).clamp(min=0)]]
    return ((y >= thr[ind - 1]) & (kk[ind - 1] > 0)).to(torch.uint8)


def torch_graph_pool(p, g, x, ratio, ind, G):
    y = (p @ x) / torch.linalg.norm(p)
    keep = torch_keep(y.detach(), ind, G, ratio) if G > 1 else \
        (y.detach() >= torch.topk(y.detach(), math.ceil(ratio * y.numel())).values[-1]).to(torch.uint8)
    idx = keep.nonzero().reshape(-1)
    out = x[:, idx] * torch.sigmoid(y[idx])[None, :]
    drop = (keep == 0).nonzero().reshape(-1) + 1
    return gnn.remove_nodes(g, drop), out, idx + 1


def emit(rec):
    name, plim, clk = card()
    rec.update(card=name, power_limit_w=plim, sm_clock_mhz=clk)
    print(json.dumps(rec), flush=True)


def run_graph(tag, g, ind, G, rounds):
    dev = "cuda"
    n = g.num_nodes
    torch.manual_seed(0)
    t = gnn.TopKPool(None, 0.5, D, device=dev)
    x = torch.randn(D, n, device=dev, requires_grad=True)
    p = t.p.detach().clone().requires_grad_(True)
    with torch.no_grad():                   # the torch arm's selection on the library's y
        _, _, idx_l = t(g, x)
        y = readout._topk_scores(gnn.rows(x), t.p)
        keep_t = torch_keep(y, ind, G, 0.5) if G > 1 else (y >= torch.topk(y, math.ceil(0.5 * n)).values[-1])
    same = bool(torch.equal(idx_l, keep_t.nonzero().reshape(-1) + 1))
    m = idx_l.numel()
    arms = {"lib": lambda: t(g, x), "torch": lambda: torch_graph_pool(p, g, x, 0.5, ind, G)}
    for mode in ("fwd", "fwd_bwd"):
        times = {a: [] for a in arms}
        for r in range(rounds + 1):
            for a, fn in arms.items():
                def call(fn=fn):
                    h, xp, idx = fn()
                    if mode == "fwd_bwd":
                        xp.sum().backward()
                    return idx
                ms, _ = event_ms(call)
                if r:
                    times[a].append(ms)
        for a in arms:
            bytes_ = n * D * 4 + 2 * m * D * 4 + (2 * n * D * 4 + m * D * 4 if mode == "fwd_bwd" else 0)
            best = min(times[a])
            emit(dict(workload=tag, arm=a, mode=mode, nodes=n, graphs=G, kept=m, ms_min=best,
                      ms_median=sorted(times[a])[len(times[a]) // 2], alg_bytes=bytes_,
                      alg_gbps=bytes_ / best / 1e6, same_selection=same))


def run_index(rounds):
    y = torch.randn(10 ** 7, device="cuda")
    k = 5 * 10 ** 6
    arms = {"lib": lambda: gnn.topk_index(y, k),
            "torch": lambda: (y >= torch.topk(y, k).values[-1]).nonzero().reshape(-1) + 1}
    same = bool(torch.equal(arms["lib"](), arms["torch"]()))
    times = {a: [] for a in arms}
    for r in range(rounds + 1):
        for a, fn in arms.items():
            ms, _ = event_ms(fn)
            if r:
                times[a].append(ms)
    for a in arms:
        emit(dict(workload="c_topk_index", arm=a, keys=10 ** 7, k=k, ms_min=min(times[a]),
                  ms_median=sorted(times[a])[len(times[a]) // 2], same_selection=same))


def run_reference_form(rounds):
    N, k = 20000, 10000
    torch.manual_seed(1)
    A = torch.rand(N, N, device="cuda")
    t = gnn.TopKPool(A, k, D, device="cuda")
    X = torch.randn(D, N, device="cuda", requires_grad=True)
    p = t.p.detach().clone().requires_grad_(True)
    At = torch.empty(k, k, device="cuda")

    def torch_arm():
        y = (p @ X) / torch.linalg.norm(p)
        v = torch.topk(y.detach(), k).values[-1]
        idx = (y.detach() >= v).nonzero().reshape(-1)
        At[...] = A[idx[:, None], idx[None, :]]
        return X[:, idx] * torch.sigmoid(y[idx])[None, :]
    with torch.no_grad():                   # the torch arm's selection on the library's y
        y = readout._topk_scores(gnn.rows(X), t.p)
        idx_l = gnn.topk_index(y, k)
        same = bool(torch.equal(idx_l, (y >= torch.topk(y, k).values[-1]).nonzero().reshape(-1) + 1))
    arms = {"lib": lambda: t(X), "torch": torch_arm}
    for mode in ("fwd", "fwd_bwd"):
        times = {a: [] for a in arms}
        for r in range(rounds + 1):
            for a, fn in arms.items():
                def call(fn=fn):
                    out = fn()
                    if mode == "fwd_bwd":
                        out.sum().backward()
                ms, _ = event_ms(call)
                if r:
                    times[a].append(ms)
        for a in arms:
            emit(dict(workload="d_reference_form", arm=a, mode=mode, N=N, k=k, ms_min=min(times[a]),
                      ms_median=sorted(times[a])[len(times[a]) // 2], same_selection=same))


def run_bound(rounds):
    lib = _lib.lib
    for n in (1024, 2048, 4096, BOUND):
        for segs in (1, 1024):
            y = torch.randn(n * segs, device="cuda")
            seg = torch.arange(0, n * segs + 1, n, dtype=torch.int64, device="cuda")
            keep = torch.empty(n * segs, dtype=torch.uint8, device="cuda")
            masks, times = {}, {}
            for arm, bound in (("cta", BOUND), ("multiblock", 0)):
                def call(bound=bound):
                    _lib.check(lib.gnnb_topk_set_smem_max(bound))
                    for _ in range(20):
                        _lib.check(lib.gnnb_topk_keep(y.data_ptr(), _lib.KEY_F32, y.numel(), seg.data_ptr(), segs,
                                                      n // 2, 0.0, keep.data_ptr(), None, 0))
                times[arm] = []
                for r in range(rounds + 1):
                    ms, _ = event_ms(call)
                    if r:
                        times[arm].append(ms / 20)
                masks[arm] = keep.clone()
            lib.gnnb_topk_set_smem_max(BOUND)
            for arm in times:
                emit(dict(workload="e_keep_bound", arm=arm, keys_per_segment=n, segments=segs,
                          ms_min=min(times[arm]), same_mask=bool(torch.equal(masks["cta"], masks["multiblock"]))))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rounds", type=int, default=5)
    ap.add_argument("--only", default="a,b,c,d,e")
    a = ap.parse_args()
    only = set(a.only.split(","))
    if "a" in only:
        g = batch(10000, 23, "cuda")
        run_graph("a_molecules", g, g.graph_indicator, 10000, a.rounds)
    if "b" in only:
        g = batch(1024, 1000, "cuda")
        run_graph("b_1024x1000", g, g.graph_indicator, 1024, a.rounds)
    if "c" in only:
        g = gnn.rmat_graph(10 ** 7, 10 ** 8, seed=1, device="cuda")
        g.plan()
        run_graph("c_rmat_10M_100M", g, None, 1, max(2, a.rounds // 2))
        del g
        torch.cuda.empty_cache()
        run_index(a.rounds)
    if "d" in only:
        run_reference_form(a.rounds)
    if "e" in only:
        run_bound(a.rounds)


if __name__ == "__main__":
    main()
