"""Measurements for the other BASELINE.json configs (parity-test cases, not the bench line): config 1 (Cora-shaped 2-layer
GCN), config 3 (GATConv 8x64 on a 50 M-edge RMAT graph), config 4 (SAGEConv mean on 1024 batched graphs).
One JSON line per config: layer fwd+bwd time, the fused kernel(s) alone, algorithmic GB/s.
Usage: python scripts/bench_configs.py [1] [3] [4]"""
import json
import os
import sys
import time

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import gnnb200 as gnn

dev = torch.device("cuda", 0)
lib = gnn._lib.lib
which = [int(a) for a in sys.argv[1:]] or [1, 3, 4]


def timeit(fn, iters=10, warm=3):
    for _ in range(warm):
        fn()
    evs = [(torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)) for _ in range(iters)]
    torch.cuda.synchronize()
    for a, b in evs:
        a.record(); fn(); b.record()
    torch.cuda.synchronize()
    ts = sorted(a.elapsed_time(b) for a, b in evs)
    return ts[len(ts) // 2]


def flush_l2():
    torch.empty(64 * 1024 * 1024, dtype=torch.float32, device=dev).zero_()


if 1 in which:  # Cora-shaped: N=2708, E=10556 bidirected, X 1433 x N ~1.27 % nonzeros, GCN 1433->16->7
    n, E = 2708, 10556
    gen = torch.Generator(device=dev).manual_seed(17)
    u = torch.randint(1, n + 1, (E // 2,), device=dev, generator=gen)
    v = torch.randint(1, n + 1, (E // 2,), device=dev, generator=gen)
    g = gnn.GNNGraph(torch.cat([u, v]), torch.cat([v, u]), num_nodes=n)
    X = (torch.rand(n, 1433, device=dev, generator=gen) < 0.0127).float()
    l1 = gnn.GCNConv(1433, 16, torch.relu, device=dev)
    l2 = gnn.GCNConv(16, 7, device=dev)
    x = gnn.unrows(X)

    def step():
        for p in list(l1.parameters()) + list(l2.parameters()):
            p.grad = None
        y = l2(g, l1(g, x))
        y.sum().backward()

    ms = timeit(step, 30, 5)
    print(json.dumps({"config": 1, "workload": "2-layer GCNConv 1433->16->7 on a Cora-shaped graph (N=2708, E=10556), fwd+bwd",
                      "ms_per_step": ms, "edges_per_s": 2 * E / (ms * 1e-3), "note": "launch-latency bound"}), flush=True)

if 4 in which:  # 1024 ER graphs x (1000 nodes, 5000 edges), block-diagonal batch, SAGEConv 128->128 mean
    G, n1, e1, D = 1024, 1000, 5000, 128
    gen = torch.Generator(device=dev).manual_seed(17)
    off = (torch.arange(G, device=dev) * n1).repeat_interleave(e1)
    s = torch.randint(0, n1, (G * e1,), device=dev, generator=gen) + off + 1
    t = torch.randint(0, n1, (G * e1,), device=dev, generator=gen) + off + 1
    gi = torch.arange(1, G + 1, device=dev).repeat_interleave(n1)
    g = gnn.GNNGraph(s, t, num_nodes=G * n1, num_graphs=G, graph_indicator=gi)
    n, E = G * n1, G * e1
    layer = gnn.SAGEConv(D, D, torch.relu, device=dev)
    x = gnn.unrows(torch.randn(n, D, device=dev, generator=gen)).requires_grad_(True)
    dy = gnn.unrows(torch.randn(n, D, device=dev, generator=gen))

    def step():
        x.grad = None
        layer.weight.grad = None
        layer.bias.grad = None
        layer(g, x).backward(dy)

    ms = timeit(step)
    xr = gnn.rows(x.detach()); out = torch.empty_like(xr); p = g.plan()
    gnn._lib.check(lib.gnnb_graph_csr(p.h, 1, None, None, None, None))
    kf = timeit(lambda: (flush_l2(), gnn._lib.check(lib.gnnb_propagate(p.h, 0, 0, gnn._lib.MEAN, xr.data_ptr(), None, None, None, D, out.data_ptr(), None))))
    kfl = timeit(lambda: flush_l2())
    alg = E * (4 * D + 4) + 4 * (n + 1) + 4 * D * n
    print(json.dumps({"config": 4, "workload": f"SAGEConv {D}->{D} mean, {G} batched ER graphs ({n1} nodes, {e1} edges each): N={n} E={E}, fwd+bwd",
                      "ms_per_step": ms, "edges_per_s": E / (ms * 1e-3), "propagate_mean_kernel_ms_after_l2_flush": kf - kfl,
                      "algorithmic_GBps": alg / ((kf - kfl) * 1e-3) / 1e9, "algorithmic_bytes": alg}), flush=True)
    del g, x, dy, xr, out
    torch.cuda.empty_cache()

if 3 in which:  # GATConv 8 heads x 64, RMAT N=2M, E=50M (+2M self loops)
    n, E, H, C = 2_000_000, 50_000_000, 8, 64
    D = H * C
    g = gnn.rmat_graph(n, E, 17, device=dev)
    layer = gnn.GATConv(D, C, torch.relu, heads=H, device=dev)
    gen = torch.Generator(device=dev).manual_seed(0)
    x = gnn.unrows(torch.randn(n, D, device=dev, generator=gen)).requires_grad_(True)
    dy = gnn.unrows(torch.randn(n, D, device=dev, generator=gen))

    def step():
        x.grad = None
        for p_ in layer.parameters():
            p_.grad = None
        layer(g, x).backward(dy)

    ms = timeit(step, 5, 2)
    g2 = gnn.add_self_loops(g)
    p = g2.plan()
    Wx = torch.randn(n, H, C, device=dev, generator=gen)
    el = torch.randn(n, H, device=dev, generator=gen); er = torch.randn(n, H, device=dev, generator=gen)
    out = torch.empty_like(Wx); smax = torch.empty(n, H, device=dev); ssum = torch.empty(n, H, device=dev)
    kf = timeit(lambda: gnn._lib.check(lib.gnnb_gat_aggregate(p.h, Wx.data_ptr(), el.data_ptr(), er.data_ptr(), C, H, 0.2,
                                                              out.data_ptr(), None, smax.data_ptr(), ssum.data_ptr(), None)), 5, 2)
    dWx = torch.empty_like(Wx); del_ = torch.empty(n, H, device=dev); der = torch.empty(n, H, device=dev)
    do = torch.randn(n, H, C, device=dev, generator=gen)
    kb = timeit(lambda: gnn._lib.check(lib.gnnb_gat_aggregate_bwd(p.h, Wx.data_ptr(), el.data_ptr(), er.data_ptr(), smax.data_ptr(),
                                                                  ssum.data_ptr(), out.data_ptr(), do.data_ptr(), C, H, 0.2,
                                                                  dWx.data_ptr(), del_.data_ptr(), der.data_ptr(), None)), 5, 2)
    E2 = E + n
    alg = E2 * (4 * D + 4 + 4 * H) + 4 * (n + 1) + 4 * D * n
    print(json.dumps({"config": 3, "workload": f"GATConv {D}->{C}x{H} heads (concat, self loops) on RMAT N={n} E={E}, fwd+bwd",
                      "ms_per_step": ms, "edges_per_s": E / (ms * 1e-3), "gat_fwd_kernel_ms": kf, "gat_bwd_ms": kb,
                      "fwd_algorithmic_GBps": alg / (kf * 1e-3) / 1e9, "algorithmic_bytes_fwd": alg}), flush=True)
