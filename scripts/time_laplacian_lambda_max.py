"""Time laplacian_lambda_max (csrc/lmax.cu, and the batched Lanczos route above the shared-memory bound) on cuda:0.
One JSON line per workload.

Workloads (random bidirected graphs plus a ring, so that no node is isolated; no weights, dir = :out):
  (a) 10 000 graphs of 23 nodes and 50 edges               (molecules)
  (b) 1 000 graphs of 150 nodes and 300 edges
  (c) 1 024 graphs of 1 000 nodes and about 5 000 edges     (config 4's shape: the Lanczos route)
  (d) RMAT 1 M nodes / 10 M edges, bidirected, plus a ring  (one graph: the Lanczos route)
Arms, alternated round by round in this process, each timed with CUDA events around whole calls (median of --rounds):
  * laplacian_lambda_max, end to end (segments, degrees, routing, the eigenvalues);
  * `eigvalsh`: batched torch.linalg.eigvalsh of the per-graph dense S, padded with -1 on the diagonal (below the
    workloads' spectra in [0, 2]), built from the edge list with index_put — (a) to (c);
  * `eigsh`: scipy's eigsh (float64, host) on the sparse S — (d), one call.
Beside them, the reference's per-graph loop restated with scipy on the host (a dense S per graph and eigvalsh) on a
sample of --sample graphs, scaled to the batch.  Each line carries the card's name, power limit and the SM clock read
after the timed calls, and the largest difference between the arms.

    python scripts/time_laplacian_lambda_max.py [--rounds 5] [--sample 200] [--only a,b]
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


def batch(G, m, e, seed):
    """G graphs of m nodes: e random edges each, both ways, plus a ring; (s, t, gi) 0-based on the device"""
    g = torch.Generator(device="cuda").manual_seed(seed)
    a = torch.randint(0, m, (G, e // 2), device="cuda", generator=g)
    b = (a + torch.randint(1, m, (G, e // 2), device="cuda", generator=g)) % m
    ring = torch.arange(m, device="cuda").expand(G, m)
    a, b = torch.cat([a, ring], 1), torch.cat([b, (ring + 1) % m], 1)
    off = (torch.arange(G, device="cuda") * m)[:, None]
    s = torch.cat([(a + off).reshape(-1), (b + off).reshape(-1)])
    t = torch.cat([(b + off).reshape(-1), (a + off).reshape(-1)])
    return s, t, torch.arange(G, device="cuda").repeat_interleave(m)


def dense_s(s, t, G, m):
    """the padded per-graph S (G, m, m), -1 on the padding's diagonal (none here: equal sizes)"""
    A = torch.zeros((G, m, m), dtype=torch.float64, device="cuda")
    A.index_put_((s // m, s % m, t % m), torch.ones_like(s, dtype=torch.float64), accumulate=True)
    c = A.sum(2).rsqrt()
    L = torch.eye(m, dtype=torch.float64, device="cuda") - c[:, :, None] * A * c[:, None, :]
    U = torch.triu(L, 1)
    return U + U.transpose(1, 2) + torch.diag_embed(torch.diagonal(L, 0, 1, 2))


def host_reference(s, t, G, m, sample):
    """the reference's loop on the host, restated: per graph a dense S and its largest eigenvalue; ms per graph"""
    s, t = s.cpu().numpy(), t.cpu().numpy()
    k = min(sample, G)
    sel = (s // m) < k
    s, t = s[sel], t[sel]
    t0 = time.perf_counter()
    for i in range(k):
        e = (s // m) == i
        A = np.zeros((m, m))
        np.add.at(A, (s[e] % m, t[e] % m), 1.0)
        c = 1 / np.sqrt(A.sum(1))
        L = np.eye(m) - c[:, None] * A * c[None, :]
        U = np.triu(L, 1)
        np.linalg.eigvalsh(U + U.T + np.diag(np.diag(L)))[-1]
    return (time.perf_counter() - t0) * 1e3 / k


def run_batch(name, G, m, e, rounds, sample):
    s, t, gi = batch(G, m, e, seed=ord(name))
    g = gnn.GNNGraph(s + 1, t + 1, num_nodes=G * m, num_graphs=G, graph_indicator=gi + 1)
    g.plan()
    ours, ref = [], []
    for r in range(rounds + 1):
        ms, lam = event_ms(lambda: gnn.laplacian_lambda_max(g))
        ours.append(ms)
        if m <= 200 or r < 2:                      # the 8 GB batch of (c): one warm-up and one timed call
            ms2, lam2 = event_ms(lambda: torch.linalg.eigvalsh(dense_s(s, t, G, m))[:, -1])
            ref.append(ms2)
    diff = float((lam - lam2).abs().max())
    per_graph = host_reference(s, t, G, m, sample)
    name_, plim, clk = card()
    return {"workload": name, "graphs": G, "nodes": m, "edges_per_graph": int(s.numel()) // G,
            "ms": float(np.median(ours[1:])), "eigvalsh_ms": float(np.median(ref[1:])) if ref else None,
            "max_abs_diff": diff, "host_reference_ms_per_graph": per_graph,
            "host_reference_ms_batch_est": per_graph * G, "card": name_, "power_limit_w": plim, "sm_clock_mhz": clk}


def run_rmat(rounds):
    import scipy.sparse as sp
    from scipy.sparse.linalg import eigsh
    n = 1_000_000
    r = gnn.rmat_graph(n, 10_000_000, seed=7, device="cuda")
    ring = torch.arange(1, n + 1, device="cuda", dtype=r.s.dtype)
    nxt = ring % n + 1
    s = torch.cat([r.s, r.t, ring, nxt])
    t = torch.cat([r.t, r.s, nxt, ring])
    g = gnn.GNNGraph(s, t, num_nodes=n)
    g.plan()
    ours = []
    for _ in range(rounds + 1):
        ms, lam = event_ms(lambda: gnn.laplacian_lambda_max(g, torch.float64))
        ours.append(ms)
    deg = gnn.degree(g, dir="out").double().cpu().numpy()
    s0, t0 = s.cpu().numpy() - 1, t.cpu().numpy() - 1
    A = sp.coo_matrix((np.ones(len(s0)), (s0, t0)), shape=(n, n)).tocsr()
    c = sp.diags(1 / np.sqrt(deg))
    L = sp.identity(n) - c @ A @ c
    S = (sp.triu(L, 1) + sp.triu(L, 1).T + sp.diags(L.diagonal())).tocsr()
    t1 = time.perf_counter()
    want = float(eigsh(S, k=1, which="LA", tol=1e-10, ncv=64, v0=np.ones(n))[0][0])
    eigsh_ms = (time.perf_counter() - t1) * 1e3
    name_, plim, clk = card()
    return {"workload": "d", "nodes": n, "edges": int(s.numel()), "ms": float(np.median(ours[1:])),
            "eigsh_host_ms": eigsh_ms, "lmax": lam, "eigsh_lmax": want, "abs_diff": abs(lam - want),
            "card": name_, "power_limit_w": plim, "sm_clock_mhz": clk}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rounds", type=int, default=5)
    ap.add_argument("--sample", type=int, default=200)
    ap.add_argument("--only", default="a,b,c,d")
    args = ap.parse_args()
    if not torch.cuda.is_available():
        sys.exit("time_laplacian_lambda_max.py needs a CUDA device")
    only = set(args.only.split(","))
    shapes = {"a": (10_000, 23, 50), "b": (1_000, 150, 300), "c": (1_024, 1_000, 4_000)}
    for k in ("a", "b", "c"):
        if k in only:
            print(json.dumps(run_batch(k, *shapes[k], args.rounds, args.sample)), flush=True)
    if "d" in only:
        print(json.dumps(run_rmat(args.rounds)), flush=True)


if __name__ == "__main__":
    main()
