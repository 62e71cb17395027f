"""dist_propagate, dist_graph_conv and dist_gin_conv on CPU with the gloo backend, world_size 2 and 3, the library
replaced by the CPU test double (tests/fake_abi.py): every aggregation, copy_xj and w_mul_xj with the graph's or an
explicit weight, forward and backward against float64 on the whole graph, and the dispatch — one max / min pullback
call per max / min backward, none for + and mean.  No GPU, no libgnnb200 compute."""
import gc
import os
import socket
import weakref

import numpy as np
import pytest
import torch
import torch.distributed as dist
import torch.multiprocessing as mp

SUM, MEAN, MAX, MIN = 0, 1, 2, 3
NAMES = {SUM: "+", MEAN: "mean", MAX: "max", MIN: "min"}


def _free_port():
    with socket.socket() as s:
        s.bind(("127.0.0.1", 0))
        return s.getsockname()[1]


def _fake_maxmin_bwd_halo(self, h, msg, aggr, x_own, dout_local, dout_halo, out_local, out_halo, n_local, w, D, dx,
                          stream):
    """gnnb_propagate_maxmin_bwd_halo's contract in numpy (include/gnnb200.h), for the CPU test double: on the backward
    shard plan (gathered = targets in [local | halo] order, reduced = owned sources j),
    dx[j] = Σ_{e: j→t} w_e dout[t] .* (float32(x[j] w_e) == out[t]), targets >= n_local from the halo buffers"""
    from fake_abi import EINVAL, OK, _arr
    self.calls.append("gnnb_propagate_maxmin_bwd_halo")
    if aggr not in (MAX, MIN):
        return self._fail(EINVAL, "max / min only")
    p = self._p(h)
    if p.nd == 0:
        return OK
    n_halo = p.ns - n_local
    both = lambda a, b: np.concatenate([_arr(a, (n_local, D)) if n_local else np.empty((0, D), np.float32),
                                        _arr(b, (n_halo, D)) if n_halo else np.empty((0, D), np.float32)])
    g, o = both(dout_local, dout_halo).astype(np.float64), both(out_local, out_halo)
    xv = _arr(x_own, (p.nd, D))
    wv = np.ones(p.E, np.float32) if msg != 1 else _arr(w, (p.E,))
    hit = (xv[p.t] * wv[:, None]) == o[p.s]                 # float32 products, as the kernel
    acc = np.zeros((p.nd, D))
    np.add.at(acc, p.t, wv.astype(np.float64)[:, None] * g[p.s] * hit)
    _arr(dx, (p.nd, D))[...] = acc
    return OK


def _f64_propagate(aggr, s0, t0, n, x, w):
    """propagate in float64 as a differentiable expression; max / min through the float32 winners' mask, so that every
    tie gets the whole gradient (NNlib's rule)"""
    m = x[s0] if w is None else x[s0] * w[:, None]
    if aggr in (SUM, MEAN):
        out = torch.zeros_like(x).index_add(0, t0, m)
        if aggr == MEAN:
            out = out / torch.bincount(t0, minlength=n).double().clamp(min=1)[:, None]
        return out
    m32 = m.detach().float()
    red = "amax" if aggr == MAX else "amin"
    init = -float("inf") if aggr == MAX else float("inf")
    out32 = torch.full((n, x.shape[1]), init).scatter_reduce(0, t0[:, None].expand(-1, x.shape[1]), m32, red,
                                                              include_self=False)
    hit = (m32 == out32[t0]).double()
    val = torch.zeros_like(x).index_add(0, t0, m * hit)
    return out32.double() + (val - val.detach())


def _worker(rank, world, port, q, ownership):
    os.environ.update(MASTER_ADDR="127.0.0.1", MASTER_PORT=str(port), GNNB_HALO="nccl", GNNB_HALO_SLICES="1")
    dist.init_process_group("gloo", rank=rank, world_size=world)
    import sys
    root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    sys.path.insert(0, root)
    sys.path.insert(0, os.path.join(root, "tests"))
    import fake_abi
    import gnnb200 as gnn
    from gnnb200 import partition as P
    from test_partition_weighted_gloo import _fake_edge_weight_grad
    # the entries this path adds to the test double's contract, in this spawned rank process only
    fake_abi.FakeLib.gnnb_propagate_maxmin_bwd_halo = _fake_maxmin_bwd_halo
    fake_abi.FakeLib.gnnb_gcn_edge_weight_grad_halo = _fake_edge_weight_grad
    n, E = 50, 400
    rng = np.random.default_rng(7)
    s = torch.as_tensor(np.minimum((rng.random(E) ** 3 * n).astype(np.int64), n - 1) + 1)
    t = torch.as_tensor(np.minimum((rng.random(E) ** 2 * n).astype(np.int64), n - 1) + 1)
    ring = torch.arange(1, n + 1)                               # every node has an in-edge: finite max / min layers
    s, t = torch.cat([s, ring % n + 1]), torch.cat([t, ring])
    E = s.numel()
    w = torch.as_tensor(rng.uniform(0.2, 2.0, E).astype(np.float32))
    results = {}
    close = lambda a, r: bool(torch.allclose(a.double(), r.double(), rtol=2e-5, atol=2e-6))
    with fake_abi.installed() as fake:
        for loops in (False, True):
            kept, orig = [], P.build_shard
            P.build_shard = lambda *a, **k: (kept.append(orig(*a, **k)) or kept[-1])
            dg = P.DistGraph(s, t, n, w=w, add_self_loops=loops, device="cpu", ownership=ownership)
            P.build_shard = orig
            for sh, d in ((dg.fwd, kept[0]), (dg.bwd, kept[1])):   # the plans csrc/shard.cu creates on a CUDA device
                sh.plan = dg._plans(d)
            ids = dg.local_nodes()
            own_t = dg.owned_by_target(t)
            s0, t0, wl = s - 1, t - 1, w.double()
            if loops:
                s0, t0 = torch.cat([s0, torch.arange(n)]), torch.cat([t0, torch.arange(n)])
            D = 5
            gen = torch.Generator().manual_seed(3)
            x_full, dout_full = torch.randn(n, D, generator=gen), torch.randn(n, D, generator=gen)
            for aggr in (SUM, MEAN, MAX, MIN):
                for mode in ("copy_xj", "w_graph", "w_explicit"):
                    fake.calls.clear()
                    f = gnn.copy_xj if mode == "copy_xj" else gnn.w_mul_xj
                    x = gnn.unrows(x_full[ids].contiguous()).requires_grad_(True)
                    ew = w[own_t].clone().requires_grad_(aggr in (SUM, MEAN)) if mode == "w_explicit" else None
                    y = P.dist_propagate(f, dg, NAMES[aggr], x, ew)
                    y.backward(gnn.unrows(dout_full[ids].contiguous()))
                    x64 = x_full.double().requires_grad_(True)
                    w64 = wl.clone().requires_grad_(True)
                    wfull = None if mode == "copy_xj" else (torch.cat([w64, torch.ones(n, dtype=torch.float64)]) if loops else w64)
                    y64 = _f64_propagate(aggr, s0, t0, n, x64, wfull)
                    y64.backward(dout_full.double())
                    tag = f"loops{loops}/{NAMES[aggr]}/{mode}"
                    results[f"{tag}/out"] = close(gnn.rows(y.detach()), y64.detach()[ids])
                    results[f"{tag}/dx"] = close(gnn.rows(x.grad), x64.grad[ids])
                    if ew is not None and ew.requires_grad:
                        dw = torch.zeros(E)
                        dw[own_t] = ew.grad                        # every edge's target is owned by exactly one rank
                        dist.all_reduce(dw)
                        results[f"{tag}/dedge_weight"] = close(dw, w64.grad)
                    n_calls = fake.calls.count("gnnb_propagate_maxmin_bwd_halo")
                    results[f"{tag}/maxmin_calls"] = n_calls == (1 if aggr in (MAX, MIN) else 0)
                    n_wgrad = fake.calls.count("gnnb_gcn_edge_weight_grad_halo")
                    results[f"{tag}/weight_grad_calls"] = n_wgrad == (1 if ew is not None and ew.requires_grad else 0)
            # the forward result is freed by reference counting once the caller drops it (no cycle through the
            # autograd context): the cyclic collector stays off while it is dropped
            gc.collect()
            gc.disable()
            try:
                for aggr in (SUM, MEAN, MAX, MIN):
                    x = gnn.unrows(x_full[ids].contiguous()).requires_grad_(True)
                    y = P.dist_propagate(gnn.w_mul_xj, dg, NAMES[aggr], x)
                    held = weakref.ref(y._base if y._base is not None else y)
                    y.backward(gnn.unrows(dout_full[ids].contiguous()))
                    del y
                    results[f"loops{loops}/{NAMES[aggr]}/result_freed_without_gc"] = held() is None
            finally:
                gc.enable()
            if not loops:
                for Din, Dout in ((6, 4), (4, 6)):
                    gen = torch.Generator().manual_seed(Din * 10 + Dout)
                    xf, dyf = torch.randn(n, Din, generator=gen), torch.randn(n, Dout, generator=gen)
                    layers = []
                    for aggr in (SUM, MEAN, MAX, MIN):
                        torch.manual_seed(0)
                        l = gnn.GraphConv(Din, Dout, torch.tanh, aggr=NAMES[aggr])
                        with torch.no_grad():
                            l.bias.copy_(torch.linspace(-0.5, 0.5, Dout))
                        layers.append((f"graph_conv/{NAMES[aggr]}", aggr, l, [l.weight1, l.weight2, l.bias], P.dist_graph_conv))
                    for aggr in (SUM, MAX):
                        torch.manual_seed(1)
                        Wn = torch.randn(Dout, Din).requires_grad_(True)
                        bn = torch.linspace(-0.5, 0.5, Dout).requires_grad_(True)
                        l = gnn.GINConv(lambda h, Wn=Wn, bn=bn: torch.tanh(Wn @ h + bn[:, None]), 0.25, aggr=NAMES[aggr])
                        layers.append((f"gin_conv/{NAMES[aggr]}", aggr, l, [Wn, bn], P.dist_gin_conv))
                    for name, aggr, l, ps, fn in layers:
                        x = gnn.unrows(xf[ids].contiguous()).requires_grad_(True)
                        y = fn(l, dg, x)
                        y.backward(gnn.unrows(dyf[ids].contiguous()))
                        for p in ps:
                            dist.all_reduce(p.grad)
                        x64 = xf.double().requires_grad_(True)
                        p64 = [p.detach().double().requires_grad_(True) for p in ps]
                        m = _f64_propagate(aggr, s0, t0, n, x64, None)
                        if name.startswith("graph"):
                            y64 = torch.tanh(x64 @ p64[0].t() + m @ p64[1].t() + p64[2])
                        else:
                            y64 = torch.tanh((1.25 * x64 + m) @ p64[0].t() + p64[1])
                        y64.backward(dyf.double())
                        tag = f"{Din}to{Dout}/{name}"
                        results[f"{tag}/y"] = close(gnn.rows(y.detach()), y64.detach()[ids])
                        results[f"{tag}/dx"] = close(gnn.rows(x.grad), x64.grad[ids])
                        for k, (p, r) in enumerate(zip(ps, p64)):
                            results[f"{tag}/dp{k}"] = close(p.grad, r.grad)
            ew = torch.ones(dg.num_owned_edges, requires_grad=True)
            x = gnn.unrows(torch.randn(dg.n_local, 5))
            bad = [lambda: P.dist_propagate(gnn.xi_sub_xj, dg, "+", x),
                   lambda: P.dist_propagate(gnn.w_mul_xj, dg, "+", x, torch.ones(dg.num_owned_edges + 1)),
                   lambda: P.dist_propagate(gnn.w_mul_xj, dg, "max", x, ew)]
            if loops:
                bad += [lambda: P.dist_graph_conv(gnn.GraphConv(5, 3), dg, x),
                        lambda: P.dist_gin_conv(gnn.GINConv(lambda h: h, 0.0), dg, x)]
            for k, f in enumerate(bad):
                fake.calls.clear()
                try:
                    f()
                    results[f"loops{loops}/value_error{k}"] = False
                except ValueError:
                    results[f"loops{loops}/value_error{k}"] = True
                results[f"loops{loops}/refused_before_any_call{k}"] = not fake.calls
    q.put((rank, all(results.values()), {k: v for k, v in results.items() if not v}))
    dist.barrier()
    dist.destroy_process_group()


@pytest.mark.parametrize("world,ownership", [(2, "contiguous"), (3, "contiguous"), (2, "cyclic"), (3, "balanced")])
def test_dist_propagate_gloo_on_the_test_double(world, ownership):
    ctx = mp.get_context("spawn")
    q = ctx.Queue()
    port = _free_port()
    procs = [ctx.Process(target=_worker, args=(r, world, port, q, ownership)) for r in range(world)]
    for p in procs:
        p.start()
    res = [q.get(timeout=300) for _ in range(world)]
    for p in procs:
        p.join(timeout=60)
        assert p.exitcode == 0
    assert all(ok for _, ok, _ in res), res
