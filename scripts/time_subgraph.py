"""Time the graph-editing functions (csrc/plan.cu: gnnb_graph_subgraph) on cuda:0.  One JSON line per case, with the
card's name, power limit and SM clock read in the same run.

On an RMAT graph of 10 M nodes / 100 M edges whose plan has both CSRs built:
  (a) remove_edges(g, 0.2): the child's plan derived from the parent's, against the same call on a parent without a plan
      followed by the child's fresh plan and its by-source CSR (a radix sort per direction);
  (b) a DropEdge GCNConv 128 -> 128 step (remove_edges(g, 0.2), forward, backward), derived against fresh;
  (c) remove_nodes(g, 0.1), derived against fresh.
On 1 024 batched graphs shaped like config 4 (1 000 nodes, 5 000 edges each):
  (d) getgraph of 64, 256 and 512 of them, derived against fresh;
  (e) remove_edges(g, 0.2), remove_nodes(g, 0.1) and add_nodes(g, 1000) on that batch, and add_nodes on the RMAT graph;
  (f) remove_edges(g, 0.2) on a 1 M / 5 M RMAT graph and on 1 024 batched graphs of 10 000 nodes / 100 000 edges.
Then a keep-share sweep, remove_edges(g, p) and remove_nodes(g, p) over p on the same RMAT graph.  Together with (f)
these are the measurements behind transform.py's choice of route (_DERIVE_MAX_EDGES).
Derived is forced (transform._DERIVE_MAX_EDGES raised) whatever the library's choice; fresh is the same call on a parent
without a plan.  Derived and fresh alternate in one process; every call ends in a device synchronise and is timed by
the host clock, so the times include the entries' count read-back.  The median of --rounds is reported, with all
rounds beside it.  --profile DIR also writes torch.profiler tables (CUDA kernels and runtime calls, host and device
time) of one derived and one fresh remove_edges(g, 0.2) to DIR.

    python scripts/time_subgraph.py [--rounds 9] [--profile DIR]
"""
import argparse
import json
import os
import statistics
import subprocess
import sys
import time

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import gnnb200 as gnn  # noqa: E402
from gnnb200 import transform  # noqa: E402


def derive(fn):
    """run fn with the child's plan derived whenever the parent has one"""
    def run(r):
        old, transform._DERIVE_MAX_EDGES = transform._DERIVE_MAX_EDGES, 2 ** 62
        try:
            return fn(r)
        finally:
            transform._DERIVE_MAX_EDGES = old
    return run


def card():
    out = subprocess.check_output(["nvidia-smi", "--id=0", "--query-gpu=name,power.limit,clocks.sm",
                                   "--format=csv,noheader,nounits"], text=True).strip().split(", ")
    return out[0], float(out[1]), float(out[2])


def both_csr(g):
    """build the plan and its by-source CSR (no copy out)"""
    p = g.plan()
    gnn._lib.check(gnn._lib.lib.gnnb_graph_csr_device(p.h, 1, None, None, None, None))
    return g


def lazy(g):
    """the same graph value without its plan"""
    return gnn.GNNGraph(g.s, g.t, g.w, num_nodes=g.num_nodes, num_graphs=g.num_graphs,
                        graph_indicator=g.graph_indicator)


def ms(fn):
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    out = fn()
    torch.cuda.synchronize()
    return (time.perf_counter() - t0) * 1e3, out


def compare(case, derived, fresh, rounds, extra):
    derived(0), fresh(0)                                         # warm-up of both
    d, f = [], []
    for r in range(rounds):
        d.append(ms(lambda: derived(r + 1))[0])
        f.append(ms(lambda: fresh(r + 1))[0])
    name, plim, clk = card()
    print(json.dumps({"case": case, "derived_ms": round(statistics.median(d), 3),
                      "fresh_ms": round(statistics.median(f), 3), "derived_all_ms": [round(v, 3) for v in d],
                      "fresh_all_ms": [round(v, 3) for v in f], **extra, "card": name, "power_limit_w": plim,
                      "sm_clock_mhz": clk}), flush=True)


def profile(out_dir, g, g0):
    from torch.profiler import ProfilerActivity, profile as prof
    os.makedirs(out_dir, exist_ok=True)
    for name, fn in (("derived", derive(lambda r: gnn.remove_edges(g, 0.2, seed=r))),
                     ("fresh", lambda r: both_csr(gnn.remove_edges(g0, 0.2, seed=r)))):
        fn(100)
        torch.cuda.synchronize()
        with prof(activities=[ProfilerActivity.CPU, ProfilerActivity.CUDA]) as p:
            fn(101)
            torch.cuda.synchronize()
        with open(os.path.join(out_dir, f"profile_{name}.txt"), "w") as f:
            f.write(p.key_averages().table(sort_by="self_cuda_time_total", row_limit=25, max_name_column_width=60))
            f.write("\n")
            f.write(p.key_averages().table(sort_by="self_cpu_time_total", row_limit=15, max_name_column_width=60))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rounds", type=int, default=9)
    ap.add_argument("--profile", default=None)
    args = ap.parse_args()
    dev = torch.device("cuda", 0)
    torch.cuda.set_device(dev)

    n, E = 10 ** 7, 10 ** 8
    g = both_csr(gnn.rmat_graph(n, E, seed=17, device=dev))
    g0 = lazy(g)
    size = {"num_nodes": n, "num_edges": E}

    if args.profile:
        profile(args.profile, g, g0)

    compare("remove_edges(g, 0.2)", derive(lambda r: gnn.remove_edges(g, 0.2, seed=r)),
            lambda r: both_csr(gnn.remove_edges(g0, 0.2, seed=r)), args.rounds, size)

    D = 128
    layer = gnn.GCNConv(D, D, torch.relu, device=dev)
    x = gnn.unrows(torch.randn(n, D, device=dev)).requires_grad_(True)
    dy = gnn.unrows(torch.randn(n, D, device=dev))

    def step(parent, r):
        h = gnn.remove_edges(parent, 0.2, seed=r)
        layer(h, x).backward(dy)

    compare("DropEdge GCNConv 128->128 fwd+bwd", derive(lambda r: step(g, r)), lambda r: step(g0, r), args.rounds, size)
    del x, dy, layer

    compare("remove_nodes(g, 0.1)", derive(lambda r: gnn.remove_nodes(g, 0.1, seed=r)),
            lambda r: both_csr(gnn.remove_nodes(g0, 0.1, seed=r)), args.rounds, size)
    for p in (0.5, 0.7, 0.8, 0.9, 0.95, 0.99):
        compare(f"remove_edges(g, {p})", derive(lambda r: gnn.remove_edges(g, p, seed=r)),
                lambda r: both_csr(gnn.remove_edges(g0, p, seed=r)), args.rounds, size)
    for p in (0.3, 0.5, 0.7, 0.9):
        compare(f"remove_nodes(g, {p})", derive(lambda r: gnn.remove_nodes(g, p, seed=r)),
                lambda r: both_csr(gnn.remove_nodes(g0, p, seed=r)), args.rounds, size)
    compare("add_nodes(g, 1000)", derive(lambda r: gnn.add_nodes(g, 1000)),
            lambda r: both_csr(gnn.add_nodes(g0, 1000)), args.rounds, size)
    del g, g0
    torch.cuda.empty_cache()

    G, n1, e1 = 1024, 1000, 5000
    gen = torch.Generator(device=dev).manual_seed(17)
    off = (torch.arange(G, device=dev) * n1).repeat_interleave(e1)
    s = torch.randint(0, n1, (G * e1,), device=dev, generator=gen) + off + 1
    t = torch.randint(0, n1, (G * e1,), device=dev, generator=gen) + off + 1
    gi = torch.arange(1, G + 1, device=dev).repeat_interleave(n1)
    b = both_csr(gnn.GNNGraph(s, t, num_nodes=G * n1, num_graphs=G, graph_indicator=gi))
    b0 = lazy(b)
    for k in (64, 256, 512):
        pick = lambda r: torch.randperm(G, generator=torch.Generator().manual_seed(r))[:k].add(1).tolist()
        compare(f"getgraph of {k} of 1024 batched graphs", derive(lambda r: gnn.getgraph(b, pick(r))),
                lambda r: both_csr(gnn.getgraph(b0, pick(r))), args.rounds,
                {"num_nodes": G * n1, "num_edges": G * e1, "graphs": G, "picked": k})
    bsize = {"num_nodes": G * n1, "num_edges": G * e1, "graphs": G}
    compare("batched: remove_edges(g, 0.2)", derive(lambda r: gnn.remove_edges(b, 0.2, seed=r)),
            lambda r: both_csr(gnn.remove_edges(b0, 0.2, seed=r)), args.rounds, bsize)
    compare("batched: remove_nodes(g, 0.1)", derive(lambda r: gnn.remove_nodes(b, 0.1, seed=r)),
            lambda r: both_csr(gnn.remove_nodes(b0, 0.1, seed=r)), args.rounds, bsize)
    compare("batched: add_nodes(g, 1000)", derive(lambda r: gnn.add_nodes(b, 1000)),
            lambda r: both_csr(gnn.add_nodes(b0, 1000)), args.rounds, bsize)
    del b, b0
    torch.cuda.empty_cache()
    # size against edge order: a small graph in random order, and a large batch whose edges are grouped by graph
    sm = both_csr(gnn.rmat_graph(10 ** 6, 5 * 10 ** 6, seed=17, device=dev))
    sm0 = lazy(sm)
    compare("small RMAT: remove_edges(g, 0.2)", derive(lambda r: gnn.remove_edges(sm, 0.2, seed=r)),
            lambda r: both_csr(gnn.remove_edges(sm0, 0.2, seed=r)), args.rounds,
            {"num_nodes": 10 ** 6, "num_edges": 5 * 10 ** 6})
    del sm, sm0
    G, n1, e1 = 1024, 10000, 100000
    off = (torch.arange(G, device=dev) * n1).repeat_interleave(e1)
    s = torch.randint(0, n1, (G * e1,), device=dev, generator=gen) + off + 1
    t = torch.randint(0, n1, (G * e1,), device=dev, generator=gen) + off + 1
    gi = torch.arange(1, G + 1, device=dev).repeat_interleave(n1)
    b = both_csr(gnn.GNNGraph(s, t, num_nodes=G * n1, num_graphs=G, graph_indicator=gi))
    del s, t
    b0 = lazy(b)
    compare("large batch: remove_edges(g, 0.2)", derive(lambda r: gnn.remove_edges(b, 0.2, seed=r)),
            lambda r: both_csr(gnn.remove_edges(b0, 0.2, seed=r)), args.rounds,
            {"num_nodes": G * n1, "num_edges": G * e1, "graphs": G})


if __name__ == "__main__":
    main()
