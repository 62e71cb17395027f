"""Weighted dist_gcn_conv on CPU with the gloo backend, world_size 2 and 3, the library replaced by the CPU test double
(tests/fake_abi.py): the weights' route into both shards, the weighted degree and its halo copies, the reverse edge
exchange and the edge-weight gradient's composition — forward and backward against float64 autograd of the dense
formula on the whole graph.  No GPU, no libgnnb200 compute."""
import os
import socket

import numpy as np
import pytest
import torch
import torch.distributed as dist
import torch.multiprocessing as mp


def _free_port():
    with socket.socket() as s:
        s.bind(("127.0.0.1", 0))
        return s.getsockname()[1]


def _dense(n, s0, t0, w, x, W, b, loops):
    """relu(C Aᵀ C x Wᵀ + b) in float64, A[s, t] = Σ w over the (s, t) edges, loops of weight 1 when the layer adds them"""
    A = torch.zeros(n, n, dtype=torch.float64)
    A = A.index_put((s0, t0), w, accumulate=True)
    if loops:
        A = A + torch.eye(n, dtype=torch.float64)
    c = 1 / A.sum(0).sqrt()
    return torch.relu((c[:, None] * (A.t() @ (c[:, None] * x))) @ W.t() + b)


def _fake_edge_weight_grad(self, h, dout, h_local, h_halo, n_local, cs, ct, dd, D, dw, stream):
    """gnnb_gcn_edge_weight_grad_halo's contract in numpy float64 (include/gnnb200.h), for the CPU test double:
    dw[e] = Σ_f (dout[t,f] ct[t]) (h[s,f] cs[s]) + dd[t] over the plan's COO order, sources >= n_local from h_halo"""
    from fake_abi import OK, _arr
    self.calls.append("gnnb_gcn_edge_weight_grad_halo")
    p = self._p(h)
    if p.E == 0:
        return OK
    n_halo = p.ns - n_local
    hv = np.concatenate([_arr(h_local, (n_local, D)) if n_local else np.empty((0, D), np.float32),
                         _arr(h_halo, (n_halo, D)) if n_halo else np.empty((0, D), np.float32)]).astype(np.float64)
    g = _arr(dout, (p.nd, D)).astype(np.float64)
    csv = np.ones(p.ns) if cs is None else _arr(cs, (p.ns,)).astype(np.float64)
    ctv = np.ones(p.nd) if ct is None else _arr(ct, (p.nd,)).astype(np.float64)
    ddv = np.zeros(p.nd) if dd is None else _arr(dd, (p.nd,)).astype(np.float64)
    _arr(dw, (p.E,))[...] = ((g[p.t] * ctv[p.t, None]) * (hv[p.s] * csv[p.s, None])).sum(1) + ddv[p.t]
    return OK


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
    # the new entry on the test double, in this spawned rank process only
    fake_abi.FakeLib.gnnb_gcn_edge_weight_grad_halo = _fake_edge_weight_grad
    n, E = 50, 400
    rng = np.random.default_rng(7)
    s = torch.as_tensor(np.minimum((rng.random(E) ** 3 * n).astype(np.int64), n - 1) + 1)
    t = torch.as_tensor(np.minimum((rng.random(E) ** 2 * n).astype(np.int64), n - 1) + 1)
    w = torch.as_tensor(rng.uniform(0.2, 2.0, E).astype(np.float32))
    s0, t0 = s - 1, t - 1
    results = {}
    with fake_abi.installed() as fake:
        for loops in (True, False):
            kept, orig = [], P.build_shard
            P.build_shard = lambda *a, **k: (kept.append(orig(*a, **k)) or kept[-1])
            dg = P.DistGraph(s, t, n, w=w, add_self_loops=loops, device="cpu", ownership=ownership)
            P.build_shard = orig
            for sh, d in ((dg.fwd, kept[0]), (dg.bwd, kept[1])):   # the plans csrc/shard.cu creates on a CUDA device
                sh.plan = dg._plans(d)
            ids = dg.local_nodes()
            own_t = dg.owned_by_target(t)
            # the shards' weights are the global weights of their edges, loops last with weight 1
            extra = [torch.ones(dg.n_local)] if loops else []
            results[f"loops{loops}/w_fwd"] = torch.equal(dg.w_fwd, torch.cat([w[own_t]] + extra))
            results[f"loops{loops}/w_bwd"] = torch.equal(dg.w_bwd, torch.cat([w[dg._owned(s)]] + extra))
            results[f"loops{loops}/reverse_exchange"] = torch.equal(dg.edge_exchange_reverse(dg.w_fwd.reshape(-1, 1)).reshape(-1),
                                                                    dg.w_bwd)
            for Din, Dout in ((6, 4), (4, 6)):
                for mode in ("explicit", "graph"):
                    torch.manual_seed(0)
                    layer = gnn.GCNConv(Din, Dout, torch.relu, add_self_loops=loops, use_edge_weight=mode == "graph")
                    with torch.no_grad():
                        layer.bias.copy_(torch.linspace(-0.5, 0.5, Dout))
                    gen = torch.Generator().manual_seed(Din * 10 + Dout)
                    x_full = torch.randn(n, Din, generator=gen)
                    dy_full = torch.randn(n, Dout, generator=gen)
                    x = gnn.unrows(x_full[ids].contiguous()).requires_grad_(True)
                    ew = w[own_t].clone().requires_grad_(True) if mode == "explicit" else None
                    y = P.dist_gcn_conv(layer, dg, x, ew)
                    y.backward(gnn.unrows(dy_full[ids].contiguous()))
                    dist.all_reduce(layer.weight.grad)
                    dist.all_reduce(layer.bias.grad)
                    x64 = x_full.double().requires_grad_(True)
                    w64 = w.double().requires_grad_(True)
                    W64 = layer.weight.detach().double().requires_grad_(True)
                    b64 = layer.bias.detach().double().requires_grad_(True)
                    y64 = _dense(n, s0, t0, w64, x64, W64, b64, loops)
                    y64.backward(dy_full.double())
                    close = lambda a, r: bool(torch.allclose(a.double(), r, rtol=2e-5, atol=2e-6))
                    tag = f"loops{loops}/{Din}to{Dout}/{mode}"
                    results[f"{tag}/y"] = close(gnn.rows(y.detach()), y64.detach()[ids])
                    results[f"{tag}/dx"] = close(gnn.rows(x.grad), x64.grad[ids])
                    results[f"{tag}/dW"] = close(layer.weight.grad, W64.grad)
                    results[f"{tag}/db"] = close(layer.bias.grad, b64.grad)
                    if mode == "explicit":
                        dw = torch.zeros(E)
                        dw[own_t] = ew.grad                        # every edge's target is owned by exactly one rank
                        dist.all_reduce(dw)
                        results[f"{tag}/dedge_weight"] = close(dw, w64.grad)
            n_calls = fake.calls.count("gnnb_gcn_edge_weight_grad_halo")
            results[f"loops{loops}/kernel_calls"] = n_calls == 2    # one per explicit-weight backward, none for the graph's
            fake.calls.clear()
            for bad in (lambda: P.dist_gcn_conv(layer, dg, x, torch.ones(dg.num_owned_edges + 1)),
                        lambda: P.DistGraph(s, t, n, w=w[:-1], add_self_loops=loops, device="cpu", ownership=ownership)):
                try:
                    bad()
                    results[f"loops{loops}/value_error"] = False
                except ValueError:
                    results.setdefault(f"loops{loops}/value_error", True)
    q.put((rank, all(results.values()), {k: v for k, v in results.items() if not v}))
    dist.barrier()
    dist.destroy_process_group()


@pytest.mark.parametrize("world,ownership", [(2, "contiguous"), (3, "contiguous"), (2, "cyclic"), (3, "balanced")])
def test_weighted_dist_gcn_conv_gloo_on_the_test_double(world, ownership):
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
