"""Weighted GCNConv on the node-partitioned graph (partition.py: DistGraph(..., w=...), dist_gcn_conv(..., edge_weight))
on the GPU, with the multi-rank harness of test_partition_gpu.py: W gloo ranks share one device (or one rank per device
under NCCL), real shards, both halo routes, one and two push buffers.

Checked per rank:
- the weights land: each shard's weights equal the global weights of its edges, the edges read back through
  gnnb_graph_csr, for both constructors and for chunks that cut rows in the middle;
- the reverse edge exchange: every forward-shard edge, tagged with its global (source, target), lands on its own
  backward-shard copy;
- the weighted halo propagate, both shards: bit for bit against gnnb_propagate on the whole graph on rows of at most one
  chunk, normwise against float64 elsewhere;
- gnnb_gcn_edge_weight_grad_halo element by element against float64 at D = 1 ... 512 (rows longer than a chunk, a rank
  without nodes, a shard without halo, a misaligned operand), and the same bits from the one-base call;
- dist_gcn_conv with the graph's weights (use_edge_weight true and false) and with an explicit edge_weight, Din < Dout and
  Din > Dout: y, dx, dW, db and d edge_weight against float64 autograd of the dense formula and within 1e-5 of the
  single-GPU gcn_conv; use_edge_weight = false gives the unweighted bits;
- zero weighted in-degrees: the single-GPU NaN and Inf positions, forward and gradients;
- three steps on one DistGraph equal fresh one-step runs bit for bit;
- the argument errors."""
import ctypes as C
import datetime
import os
import sys
import traceback

import numpy as np
import pytest
import torch

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
from test_partition_gpu import (CHUNK, N_NODES, TOL_LAYER, TOL_LONG, Rank, Reference, assert_records,  # noqa: E402
                                bits_record, check_structure, make_graph, ownership_cases, rel_err,
                                require_shared_device, run_group)

pytestmark = pytest.mark.gpu

DS = (1, 5, 64, 128, 130, 256, 512)          # the generic kernel, the float4 lanes at 128 / 256 / 512
LAYERS = ((128, 256), (16, 7))               # Din < Dout (propagate at 128), Din > Dout (propagate at 7)
EPS = 2.0 ** -24


def make_weights(G, seed=3):
    """positive weights, one per global edge"""
    rng = np.random.default_rng(seed)
    return rng.uniform(0.25, 2.0, G["s"].size).astype(np.float32)


def zero_degree_weights(G, loops):
    """weights under which some nodes with in- and out-edges get a weighted in-degree of exactly 0: a node with one
    in-edge gets weight 0 on it (-1 with the loop of weight 1 appended after it)"""
    w = make_weights(G)
    indeg = np.bincount(G["t"], minlength=N_NODES)
    outdeg = np.bincount(G["s"], minlength=N_NODES)
    picked = np.nonzero((indeg == 1) & (outdeg > 0))[0][:12]
    for v in picked:
        w[G["t"] == v] = -1.0 if loops else 0.0
    return w, picked


def shard_coo(R, dg, sh, halo_nodes):
    """(gathered, reduced) global node of every edge of a shard, in the shard's COO order"""
    ids = dg.local_nodes()
    ne = sh.num_edges
    rowptr = np.zeros(sh.n_local + 1, np.int32)
    col, eid = np.zeros(max(ne, 1), np.int32), np.zeros(max(ne, 1), np.int32)
    R.gnn._lib.check(R.gnn._lib.lib.gnnb_graph_csr(sh.plan.h, 0, rowptr.ctypes.data, col.ctypes.data, eid.ctypes.data,
                                                   None))
    row = np.repeat(np.arange(sh.n_local), np.diff(rowptr))
    coo_row, coo_col = np.zeros(ne, np.int64), np.zeros(ne, np.int64)
    coo_row[eid[:ne]], coo_col[eid[:ne]] = row, col[:ne]
    space = torch.cat([ids, halo_nodes.to(ids.dtype)]).cpu().numpy()
    return space[coo_col], ids.cpu().numpy()[coo_row]


def build_weighted(R, G, w, loops, chunked, **own):
    """weighted DistGraph from int64 (s, t, w) or from ragged (s, t, w) chunks of 997 edges"""
    s1 = torch.as_tensor(G["s"] + 1, device=R.dev)
    t1 = torch.as_tensor(G["t"] + 1, device=R.dev)
    wt = torch.as_tensor(w, device=R.dev)
    n0 = len(R.requests)
    if chunked:
        s32, t32 = s1.to(torch.int32), t1.to(torch.int32)
        chunks = [(s32[i:i + 997], t32[i:i + 997], wt[i:i + 997]) for i in range(0, s32.numel(), 997)]
        dg = R.P.DistGraph.from_chunks(chunks, N_NODES, add_self_loops=loops, device=R.dev, **own)
    else:
        dg = R.P.DistGraph(s1, t1, N_NODES, w=wt, add_self_loops=loops, device=R.dev, **own)
    return dg, R.requests[n0:n0 + 2]


class WeightedFull:
    """the whole weighted graph (loops of weight 1 appended when the layer adds them) on one GPU and in float64"""

    def __init__(self, R, G, w, loops):
        gnn, n = R.gnn, N_NODES
        s, t = G["s"], G["t"]
        wl = w
        if loops:
            s, t, wl = np.concatenate([s, np.arange(n)]), np.concatenate([t, np.arange(n)]), np.concatenate([w, np.ones(n, np.float32)])
        self.s, self.t = torch.as_tensor(s, device=R.dev), torch.as_tensor(t, device=R.dev)
        self.w = torch.as_tensor(wl, device=R.dev)
        self.g0 = gnn.GNNGraph(torch.as_tensor(G["s"] + 1), torch.as_tensor(G["t"] + 1), torch.as_tensor(w),
                               num_nodes=n).cuda()
        g = gnn.add_self_loops(self.g0) if loops else self.g0
        self.plan = g.plan()
        d = torch.zeros(n, dtype=torch.float32, device=R.dev)
        R.gnn._lib.check(R.gnn._lib.lib.gnnb_degree(self.plan.h, R.gnn._lib.DIR_IN, self.w.data_ptr(), d.data_ptr(), R.stream()))
        self.c = R.gnn.layers.default_norm_fn(d)               # gcn_conv's c on the whole graph
        self.deg = (np.bincount(t, minlength=n), np.bincount(s, minlength=n))
        self.R = R

    def one_gpu(self, tr, x):
        out = torch.empty_like(x)
        lib = self.R.gnn._lib
        lib.check(lib.lib.gnnb_propagate(self.plan.h, tr, lib.W_MUL_XJ, lib.SUM, x.data_ptr(), self.w.data_ptr(),
                                         self.c.data_ptr(), self.c.data_ptr(), x.shape[1], out.data_ptr(), self.R.stream()))
        return out

    def f64(self, tr, x):
        key, other = (self.t, self.s) if tr == 0 else (self.s, self.t)
        c = self.c.double()
        out = torch.zeros(x.shape, dtype=torch.float64, device=x.device)
        out.index_add_(0, key, x.double()[other] * (c[other] * self.w.double())[:, None])
        return out * c[:, None]


# ------------------------------------------------------------------------------------------------ checks
def check_weights_land(R, tag, dg, G, w, loops, halos):
    ids = dg.local_nodes().cpu().numpy()
    mine = np.zeros(N_NODES, bool)
    mine[ids] = True
    ok_mask = np.array_equal(dg.owned_by_target(torch.as_tensor(G["t"] + 1, device=R.dev)).cpu().numpy(), mine[G["t"]])
    R.put(f"weights/{tag}/owned_by_target", ok_mask)
    for name, sh, key, other, wsh, halo in (("fwd", dg.fwd, G["t"], G["s"], dg.w_fwd, halos[0]),
                                            ("bwd", dg.bwd, G["s"], G["t"], dg.w_bwd, halos[1])):
        sel = mine[key]
        exp_key, exp_other, exp_w = key[sel], other[sel], w[sel]
        if loops:
            exp_key, exp_other = np.concatenate([exp_key, ids]), np.concatenate([exp_other, ids])
            exp_w = np.concatenate([exp_w, np.ones(ids.size, np.float32)])
        got_other, got_key = shard_coo(R, dg, sh, halo)
        ok = (np.array_equal(got_key, exp_key) and np.array_equal(got_other, exp_other)
              and np.array_equal(wsh.cpu().numpy().view(np.int32), exp_w.view(np.int32)))
        R.put(f"weights/{tag}/{name}/global_weights_of_the_shard_edges", ok)


def check_reverse_exchange(R, tag, dg, halos):
    src_f, tgt_f = shard_coo(R, dg, dg.fwd, halos[0])
    tgt_b, src_b = shard_coo(R, dg, dg.bwd, halos[1])        # bwd: gathered = target, reduced = source
    tag_f = torch.as_tensor(np.stack([src_f, tgt_f], 1), dtype=torch.float32, device=R.dev)
    want = torch.as_tensor(np.stack([src_b, tgt_b], 1), dtype=torch.float32, device=R.dev)
    R.put(f"reverse/{tag}/every_edge_onto_itself", *bits_record(dg.edge_exchange_reverse(tag_f), want))


def check_propagate(R, tag, dg, full, halos):
    ids = dg.local_nodes()
    ids_np = ids.cpu().numpy()
    c = full.c[ids]
    cf, cb = torch.cat([c, full.c[halos[0]]]), torch.cat([c, full.c[halos[1]]])
    d, cw, cwf, cwb = dg.gcn_c_weighted()
    short = torch.as_tensor(full.deg[0][ids_np] <= CHUNK, device=R.dev)
    R.put(f"propagate/{tag}/c_short_rows_bits", *bits_record(cw[short], c[short]))
    err, at = rel_err(cw, c)
    R.put(f"propagate/{tag}/c", err <= TOL_LONG, err, at)
    for D in (1, 5, 128, 256, 260, 512):
        x = torch.randn(N_NODES, D, device=R.dev, generator=torch.Generator(device=R.dev).manual_seed(200 + D))
        xl = x[ids].contiguous()
        for dd, (sh, cs, ws) in enumerate(((dg.fwd, cf, dg.w_fwd), (dg.bwd, cb, dg.w_bwd))):
            name = f"propagate/{tag}/{('fwd', 'bwd')[dd]}/D{D}"
            outs = {}
            for route, halo in (("push", "push"), ("alltoall", "nccl")):
                R.set_route(halo)
                outs[route] = dg.propagate(sh, xl, cs, c, w=ws)
            R.set_route()
            one = full.one_gpu(dd, x)[ids]
            short = torch.as_tensor(full.deg[dd][ids_np] <= CHUNK, device=R.dev)
            R.put(f"{name}/short_rows_bits_one_gpu", *bits_record(outs["push"][short], one[short]))
            err, at = rel_err(outs["push"][~short], full.f64(dd, x)[ids][~short])
            R.put(f"{name}/long_rows_f64", err <= TOL_LONG, err, at)
            R.put(f"{name}/alltoall_bits_push", *bits_record(outs["alltoall"], outs["push"]))


def ew_grad(R, plan, dout, h_local, h_halo, n_local, cs, ct, dd, D, E):
    dw = torch.full((max(E, 1),), float("nan"), device=R.dev)[:E]
    p = lambda t: None if t is None else t.data_ptr()
    R.gnn._lib.check(R.gnn._lib.lib.gnnb_gcn_edge_weight_grad_halo(plan.h, p(dout), p(h_local), p(h_halo), n_local, p(cs),
                                                                   p(ct), p(dd), D, p(dw), R.stream()))
    return dw


def check_entry(R, tag, dg, halos):
    """gnnb_gcn_edge_weight_grad_halo on the forward shard against float64, element by element: |dw - dw64| within
    (D + 4) ulp-units of the sum of the magnitudes of its terms"""
    ids = dg.local_nodes()
    sh, nl = dg.fwd, dg.n_local
    src, tgt = shard_coo(R, dg, sh, halos[0])
    pos = torch.full((N_NODES,), -1, dtype=torch.int64, device=R.dev)
    pos[ids] = torch.arange(nl, device=R.dev)
    src, tgt = torch.as_tensor(src, device=R.dev), torch.as_tensor(tgt, device=R.dev)
    d, c, cf, cb = dg.gcn_c_weighted()
    ddt = torch.randn(nl, device=R.dev, generator=torch.Generator(device=R.dev).manual_seed(9))
    space = torch.cat([ids, halos[0].to(ids.dtype)])
    for D in DS:
        gen = torch.Generator(device=R.dev).manual_seed(300 + D)
        h = torch.randn(N_NODES, D, device=R.dev, generator=gen)
        dout = torch.randn(nl, D, device=R.dev, generator=gen)
        hl, hh = h[ids].contiguous(), h[halos[0]].contiguous()
        dw = ew_grad(R, sh.plan, dout, hl, hh if sh.n_halo else None, nl, cf, c, ddt, D, sh.num_edges)
        hcat = h[space].contiguous()
        one = ew_grad(R, sh.plan, dout, hcat, None, nl + sh.n_halo, cf, c, ddt, D, sh.num_edges)
        R.put(f"entry/{tag}/D{D}/one_base_bits_halo", *bits_record(one, dw))
        r = pos[tgt]
        a = dout.double()[r] * c.double()[r, None]
        b = h.double()[src] * cf.double()[col_of(space, src)][:, None]
        prod = a * b
        ref = prod.sum(1) + ddt.double()[r]
        scale = prod.abs().sum(1) + ddt.double()[r].abs()
        # without loops, a source without in-edges has c = Inf: those edges must give float64's Inf / NaN, the others
        # (and no unwritten NaN) the bound
        got = dw.double()
        same_nf = (got == ref) | (torch.isnan(got) & torch.isnan(ref))
        within = (got - ref).abs() <= (D + 4) * EPS * scale
        bad = torch.nonzero(~torch.where(torch.isfinite(ref), within, same_nf))
        R.put(f"entry/{tag}/D{D}/f64_element_by_element", bad.numel() == 0, 0.0, int(bad[0]) if bad.numel() else -1)
    if nl and sh.num_edges:                                    # a misaligned operand: the generic kernel at D = 128
        D = 128
        h = torch.randn(N_NODES * D + 1, device=R.dev, generator=torch.Generator(device=R.dev).manual_seed(77))
        hv = h[1:].reshape(N_NODES, D)
        hl = torch.empty(nl * D + 1, device=R.dev)[1:].reshape(nl, D)
        hl.copy_(hv[ids])
        hh = hv[halos[0]].contiguous()
        dout = torch.randn(nl, D, device=R.dev, generator=torch.Generator(device=R.dev).manual_seed(78))
        mis = ew_grad(R, sh.plan, dout, hl, hh if sh.n_halo else None, nl, cf, c, ddt, D, sh.num_edges)
        ali = ew_grad(R, sh.plan, dout, hv[ids].contiguous(), hh if sh.n_halo else None, nl, cf, c, ddt, D, sh.num_edges)
        err, at = rel_err(mis, ali)
        R.put(f"entry/{tag}/misaligned_generic_vs_float4", err <= 1e-6, err, at)


def col_of(space, nodes):
    """position of every global node of `nodes` in the [local | halo] space of a shard"""
    inv = torch.full((N_NODES,), -1, dtype=torch.int64, device=space.device)
    inv[space] = torch.arange(space.numel(), device=space.device)
    return inv[nodes]


def make_layer(R, Din, Dout, loops, use_w):
    torch.manual_seed(1000 * Din + Dout)
    layer = R.gnn.GCNConv(Din, Dout, torch.relu, add_self_loops=loops, use_edge_weight=use_w, device=R.dev)
    with torch.no_grad():
        layer.bias.copy_(torch.linspace(-0.5, 0.5, Dout))
    return layer


def dist_step(R, dg, layer, x_full, dy_full, ew_global=None):
    """dist_gcn_conv forward and backward on this rank's rows: y and dx of the local rows, all-reduced dW and db, and the
    edge-weight gradient placed back in the global list and all-reduced"""
    import torch.distributed as dist
    gnn = R.gnn
    ids = dg.local_nodes()
    layer.zero_grad(set_to_none=True)
    x = gnn.unrows(x_full[ids].contiguous()).requires_grad_(True)
    ew = None
    if ew_global is not None:
        mask = dg.owned_by_target(torch.as_tensor(R.G["t"] + 1, device=R.dev))
        ew = ew_global[mask].clone().requires_grad_(True)
    y = R.P.dist_gcn_conv(layer, dg, x, ew)
    y.backward(gnn.unrows(dy_full[ids].contiguous()))
    dW, db = layer.weight.grad.clone(), layer.bias.grad.clone()
    dist.all_reduce(dW)
    dist.all_reduce(db)
    out = [gnn.rows(y.detach()).clone(), gnn.rows(x.grad).clone(), dW, db]
    if ew is not None:
        dw = torch.zeros(ew_global.numel(), device=R.dev)
        dw[mask] = ew.grad
        dist.all_reduce(dw)                                    # every edge's target has one owner
        out.append(dw)
    return out


def one_gpu_step(R, full, layer, x_full, dy_full, ew_global=None):
    gnn = R.gnn
    layer.zero_grad(set_to_none=True)
    x = gnn.unrows(x_full.clone()).requires_grad_(True)
    ew = None if ew_global is None else ew_global.clone().requires_grad_(True)
    y = layer(full.g0, x, ew)
    y.backward(gnn.unrows(dy_full.clone()))
    out = [gnn.rows(y.detach()), gnn.rows(x.grad), layer.weight.grad.clone(), layer.bias.grad.clone()]
    if ew is not None:
        out.append(ew.grad)
    return out


def f64_step(R, full, layer, x_full, dy_full, w_global, explicit, loops):
    """float64 autograd of relu(C Aᵀ C x Wᵀ + b), A[s, t] = Σ w (loops of weight 1 appended)"""
    n = N_NODES
    w64 = torch.as_tensor(w_global, device=R.dev).double().requires_grad_(explicit)
    wl = torch.cat([w64, torch.ones(n, dtype=torch.float64, device=R.dev)]) if loops else w64
    A = torch.zeros(n, n, dtype=torch.float64, device=R.dev).index_put((full.s, full.t), wl, accumulate=True)
    c = A.sum(0).rsqrt()
    x64 = x_full.double().requires_grad_(True)
    W64 = layer.weight.detach().double().requires_grad_(True)
    b64 = layer.bias.detach().double().requires_grad_(True)
    y64 = torch.relu((c[:, None] * (A.t() @ (c[:, None] * x64))) @ W64.t() + b64)
    y64.backward(dy_full.double())
    out = [y64.detach(), x64.grad, W64.grad, b64.grad]
    if explicit:
        out.append(w64.grad)
    return out


def check_layer(R, tag, dg, dg_plain, full, w, loops):
    ids = dg.local_nodes()
    names = ("y", "dx", "dW", "db", "dedge_weight")
    wt = torch.as_tensor(w, device=R.dev)
    for Din, Dout in LAYERS:
        gen = torch.Generator(device=R.dev).manual_seed(7 * Din + Dout)
        x_full = torch.randn(N_NODES, Din, device=R.dev, generator=gen)
        dy_full = torch.randn(N_NODES, Dout, device=R.dev, generator=gen)
        for mode in ("graph", "explicit"):
            name = f"layer/{tag}/{Din}to{Dout}/{mode}"
            layer = make_layer(R, Din, Dout, loops, mode == "graph")
            ew = wt if mode == "explicit" else None
            got = dist_step(R, dg, layer, x_full, dy_full, ew)
            one = one_gpu_step(R, full, layer, x_full, dy_full, ew)
            local = lambda k, v: v[ids] if k in ("y", "dx") else v
            for k, a, b in zip(names, got, one):
                err, at = rel_err(a, local(k, b))
                R.put(f"{name}/{k}/one_gpu", err <= TOL_LAYER, err, at)
            if loops:                                          # without loops: isolated targets, non-finite entries
                ref = f64_step(R, full, layer, x_full, dy_full, w, mode == "explicit", loops)
                for k, a, r in zip(names, got, ref):
                    err, at = rel_err(a, local(k, r))
                    R.put(f"{name}/{k}/f64", err <= TOL_LAYER, err, at)
        # use_edge_weight = false on the weighted graph: the unweighted path, bit for bit
        layer = make_layer(R, Din, Dout, loops, False)
        a = dist_step(R, dg, layer, x_full, dy_full)
        b = dist_step(R, dg_plain, layer, x_full, dy_full)
        for k, u, v in zip(names, a, b):
            R.put(f"layer/{tag}/{Din}to{Dout}/use_edge_weight_false_bits_unweighted/{k}", *bits_record(u, v))


def check_nonfinite(R, tag, G, loops, own):
    """weighted in-degree 0 on nodes with out-edges: c = Inf there; the single-GPU NaN / Inf positions everywhere"""
    w, picked = zero_degree_weights(G, loops)
    dg, _ = build_weighted(R, G, w, loops, False, **own)
    full = WeightedFull(R, G, w, loops)
    wt = torch.as_tensor(w, device=R.dev)
    gen = torch.Generator(device=R.dev).manual_seed(17)
    x_full, dy_full = torch.randn(N_NODES, 128, device=R.dev, generator=gen), torch.randn(N_NODES, 128, device=R.dev, generator=gen)
    ids = dg.local_nodes()
    for mode in ("graph", "explicit"):
        layer = make_layer(R, 128, 128, loops, mode == "graph")
        ew = wt if mode == "explicit" else None
        got = dist_step(R, dg, layer, x_full, dy_full, ew)
        one = one_gpu_step(R, full, layer, x_full, dy_full, ew)
        R.put(f"nonfinite/{tag}/{mode}/one_gpu_has_nonfinite", picked.size > 0 and not bool(torch.isfinite(one[0]).all()))
        for k, a, b in zip(("y", "dx", "dW", "db", "dedge_weight"), got, one):
            err, at = rel_err(a, b[ids] if k in ("y", "dx") else b)
            R.put(f"nonfinite/{tag}/{mode}/{k}", err <= TOL_LAYER, err, at)
    dg.close()


def check_steps(R, G, w, own):
    """three explicit-weight steps with different x on one DistGraph equal fresh one-step runs bit for bit, with two push
    buffers and with one"""
    wt = torch.as_tensor(w, device=R.dev)
    for nbuf in ("2", "1"):
        os.environ["GNNB_HALO_BUFFERS"] = nbuf
        layer = make_layer(R, 128, 128, True, False)
        xs = [torch.randn(N_NODES, 128, device=R.dev, generator=torch.Generator(device=R.dev).manual_seed(50 + k)) for k in range(3)]
        dy = torch.randn(N_NODES, 128, device=R.dev, generator=torch.Generator(device=R.dev).manual_seed(49))
        dg, _ = build_weighted(R, G, w, True, False, **own)
        steps = [dist_step(R, dg, layer, x, dy, wt) for x in xs]
        dg.close()
        for k, x in enumerate(xs):
            fresh, _ = build_weighted(R, G, w, True, False, **own)
            once = dist_step(R, fresh, layer, x, dy, wt)
            fresh.close()
            for name, a, b in zip(("y", "dx", "dW", "db", "dedge_weight"), steps[k], once):
                R.put(f"steps/{own['ownership']}/buffers{nbuf}/step{k}/{name}", *bits_record(a, b))
    os.environ["GNNB_HALO_BUFFERS"] = "2"


def check_errors(R, G, w, dg):
    P = R.P
    s1 = torch.as_tensor(G["s"] + 1, device=R.dev)
    t1 = torch.as_tensor(G["t"] + 1, device=R.dev)
    wt = torch.as_tensor(w, device=R.dev)
    x = R.gnn.unrows(torch.randn(dg.n_local, 8, device=R.dev))
    layer = make_layer(R, 8, 8, dg.self_loops, False)
    cases = {"edge_weight_length": lambda: P.dist_gcn_conv(layer, dg, x, torch.ones(dg.num_owned_edges + 1, device=R.dev)),
             "w_length": lambda: P.DistGraph(s1, t1, N_NODES, w=wt[:-1], device=R.dev),
             "chunk_w_length": lambda: P.DistGraph.from_chunks([(s1, t1, wt[:-1])], N_NODES, device=R.dev),
             "chunks_disagree": lambda: P.DistGraph.from_chunks([(s1[:10], t1[:10], wt[:10]), (s1[10:], t1[10:])], N_NODES,
                                                                device=R.dev)}
    for name, f in cases.items():
        try:
            f()
            ok = False
        except ValueError:
            ok = True
        R.put(f"errors/{'loops' if dg.self_loops else 'noloops'}/{name}", ok)


def run_cases(R, multi_device):
    G = dict(zip(("s", "t"), make_graph()))
    R.G = G
    w = make_weights(G)
    cases = ownership_cases(R.W) if R.W > 1 else [(o, dict(ownership=o)) for o in ("contiguous", "cyclic", "balanced")]
    for tag, own in cases:
        for loops in (True, False):
            full_tag = f"W{R.W}/{tag}/{'loops' if loops else 'noloops'}"
            full = WeightedFull(R, G, w, loops)
            dg, req = build_weighted(R, G, w, loops, False, **own)
            halos = check_structure(R, full_tag, dg, req, Reference(R, G, loops))
            check_weights_land(R, full_tag, dg, G, w, loops, halos)
            if not multi_device:
                kw = dict(own, bounds=dg.bounds) if own["ownership"] == "contiguous" else own
                dc, _ = build_weighted(R, G, w, loops, True, **kw)
                check_weights_land(R, full_tag + "/from_chunks", dc, G, w, loops, halos)
                dc.close()
            check_reverse_exchange(R, full_tag, dg, halos)
            check_propagate(R, full_tag, dg, full, halos)
            check_entry(R, full_tag, dg, halos)
            dg_plain, _ = R.build(G, loops, False, **own)
            check_layer(R, full_tag, dg, dg_plain, full, w, loops)
            dg_plain.close()
            check_errors(R, G, w, dg)
            dg.close()
            if tag in ("contiguous", "balanced"):
                check_nonfinite(R, full_tag, G, loops, own)
    if R.W > 1:
        for tag, own in ownership_cases(R.W)[1:3]:
            check_steps(R, G, w, own)


def weighted_worker(rank, W, port, q, multi_device):
    import torch.distributed as dist
    os.environ.update(MASTER_ADDR="127.0.0.1", MASTER_PORT=str(port), GNNB_HALO="push", GNNB_HALO_SLICES="1",
                      GNNB_HALO_BUFFERS="2")
    dev = torch.device("cuda", rank if multi_device else 0)
    torch.cuda.set_device(dev)
    try:
        dist.init_process_group("nccl" if multi_device else "gloo", rank=rank, world_size=W,
                                timeout=datetime.timedelta(seconds=300), device_id=dev if multi_device else None)
        R = Rank(rank, W, q, dev)
        run_cases(R, multi_device)
        torch.cuda.synchronize(dev)
        dist.barrier()
        q.put(("done", rank, True, 0.0, -1))
    except BaseException:
        q.put(("error", rank, False, 0.0, traceback.format_exc()[-4000:]))
    finally:
        if dist.is_initialized():
            dist.destroy_process_group()


FAMILIES = ["weights", "reverse", "propagate", "entry", "layer", "nonfinite", "steps", "errors"]


@pytest.mark.parametrize("W", [1, 2, 3, 4])
@pytest.mark.parametrize("check", FAMILIES)
def test_weighted_partition_on_one_device(W, check):
    """W gloo ranks on one device: `check` names the family of records"""
    require_shared_device()
    if W == 1 and check == "steps":
        pytest.skip("the repeated-steps check runs at W > 1")
    assert_records(*run_group(weighted_worker, W, False), prefix=check + "/")


def test_weighted_partition_one_rank_per_device_nccl():
    """one rank per device under NCCL, the push route over real peer mappings"""
    if not torch.cuda.is_available() or torch.cuda.device_count() < 2:
        pytest.skip("needs at least two visible CUDA devices: NCCL refuses two ranks on one device")
    W = min(torch.cuda.device_count(), 4)
    records, errors, codes = run_group(weighted_worker, W, True)
    for prefix in FAMILIES:
        assert_records(records, errors, codes, prefix + "/")


def test_edge_weight_grad_on_a_plan_without_edges():
    """an empty rank's shard plan: gnnb_gcn_edge_weight_grad_halo accepts NULL pointers, since there is nothing to write"""
    if not torch.cuda.is_available():
        pytest.skip("no CUDA device")
    sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
    import gnnb200 as gnn
    lib = gnn._lib.lib
    h = C.c_void_p()
    gnn._lib.check(lib.gnnb_graph_create(C.byref(h), None, None, 0, 0, 0, 4, 0, 1, None))
    plan = gnn.graph._Plan(h.value, torch.device("cuda", 0))
    gnn._lib.check(lib.gnnb_gcn_edge_weight_grad_halo(plan.h, None, None, None, 0, None, None, None, 8, None, None))
