"""Time the link-prediction generators (csrc/edgegen.cu) on cuda:0 at 10 M nodes / 100 M edges.  One JSON line each.

Device rows: negative_sample (directed and bidirected) on an RMAT graph, rand_graph, rand_edge_split (directed, and
bidirected on a rand_graph, which includes its three checks on the graph), in ms per call by CUDA events after a
warm-up, with the card's name and power limit read in the same run.

Host row: a numpy restatement of the reference's algorithm (GNNGraphs/src/transform.jl:897-926, directed): codes to
the host, self loops added as positives, randsubseq by geometric skips over 1:n², np.isin set difference against the
positives, the first num_neg kept, results back to the device.  It runs on a bounded number of negatives
(--host-neg, default 10 M of the 100 M) against the full positive set; the line says so.

    python scripts/time_link_prediction.py [--iters 5] [--warmup 1] [--host-neg 10000000]
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
        out = subprocess.check_output(["nvidia-smi", "--id=0", "--query-gpu=name,power.limit",
                                       "--format=csv,noheader,nounits"], text=True).strip().split(", ")
        return out[0], float(out[1])
    except Exception:
        return torch.cuda.get_device_name(0), float("nan")


def timed(fn, iters, warmup):
    for _ in range(warmup):
        fn()
    torch.cuda.synchronize()
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    a.record()
    for i in range(iters):
        fn(i)
    b.record()
    torch.cuda.synchronize()
    return a.elapsed_time(b) / iters


def host_negative_sample(g, num_neg, rng):
    """the reference's host path, directed: returns (s, t) on the device"""
    n = g.num_nodes
    s, t = g.s.cpu().numpy(), g.t.cpu().numpy()
    loops = np.arange(1, n + 1)
    idx_pos = np.unique((np.concatenate([s, loops]) - 1) * n + np.concatenate([t, loops]))
    maxid = n * n
    pneg = 1 - len(idx_pos) / (2 * maxid)
    prob = min(1.0, num_neg / (pneg * maxid) * 1.1)
    k = int(maxid * prob * 1.01) + 1000                      # randsubseq: Bernoulli(prob) over 1:maxid by geometric gaps
    rnd = np.cumsum(rng.geometric(prob, k))
    rnd = rnd[rnd <= maxid]
    neg = rnd[~np.isin(rnd, idx_pos)][:num_neg]
    return torch.as_tensor((neg - 1) // n + 1).cuda(), torch.as_tensor((neg - 1) % n + 1).cuda()


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--iters", type=int, default=5)
    ap.add_argument("--warmup", type=int, default=1)
    ap.add_argument("--nodes", type=int, default=10_000_000)
    ap.add_argument("--edges", type=int, default=100_000_000)
    ap.add_argument("--host-neg", type=int, default=10_000_000)
    args = ap.parse_args()
    torch.cuda.set_device(0)
    N, E = args.nodes, args.edges
    name, plimit = card()
    g = gnn.rmat_graph(N, E, seed=11, device="cuda")
    gb = gnn.rand_graph(N, E, seed=3, device="cuda")
    rows = [
        ("negative_sample", "rmat, directed, num_neg_edges = E",
         lambda i=0: gnn.negative_sample(g, num_neg_edges=E, bidirected=False, seed=i)),
        ("negative_sample", "rmat, bidirected, num_neg_edges = E",
         lambda i=0: gnn.negative_sample(g, num_neg_edges=E, bidirected=True, seed=i)),
        ("rand_graph", "bidirected, m = E", lambda i=0: gnn.rand_graph(N, E, seed=i, device="cuda")),
        ("rand_graph", "directed, m = E", lambda i=0: gnn.rand_graph(N, E, bidirected=False, seed=i, device="cuda")),
        ("rand_edge_split", "rmat, directed, frac = 0.9",
         lambda i=0: gnn.rand_edge_split(g, 0.9, bidirected=False, seed=i)),
        ("rand_edge_split", "rand_graph, bidirected (with its graph checks), frac = 0.9",
         lambda i=0: gnn.rand_edge_split(gb, 0.9, bidirected=True, seed=i)),
    ]
    for fn_name, case, fn in rows:
        ms = timed(fn, args.iters, args.warmup)
        print(json.dumps({"function": fn_name, "case": case, "nodes": N, "edges": E, "ms": round(ms, 2),
                          "iters": args.iters, "gpu": name, "power_limit_w": plimit}), flush=True)
        torch.cuda.empty_cache()
    rng = np.random.default_rng(0)
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    s, _ = host_negative_sample(g, args.host_neg, rng)
    torch.cuda.synchronize()
    host_ms = (time.perf_counter() - t0) * 1e3
    print(json.dumps({"function": "negative_sample (reference algorithm, numpy on the host)",
                      "case": "rmat, directed, full positive set", "nodes": N, "edges": E,
                      "num_neg_edges": args.host_neg, "negatives_returned": int(s.numel()), "ms": round(host_ms, 1),
                      "host_cores": os.cpu_count(), "gpu": name, "power_limit_w": plimit}), flush=True)
    dev_ms = timed(lambda i=0: gnn.negative_sample(g, num_neg_edges=args.host_neg, bidirected=False, seed=i),
                   args.iters, args.warmup)
    print(json.dumps({"function": "negative_sample", "case": "rmat, directed, same num_neg_edges as the host row",
                      "nodes": N, "edges": E, "num_neg_edges": args.host_neg, "ms": round(dev_ms, 2),
                      "iters": args.iters, "gpu": name, "power_limit_w": plimit}), flush=True)


if __name__ == "__main__":
    main()
