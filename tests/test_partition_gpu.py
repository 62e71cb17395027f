"""The node-partitioned GCN path (partition.py) on the GPU: W rank processes share one device under gloo, or one rank per
device under NCCL when enough devices are visible, and run the real DistGraph with the real kernels — shards built by
csrc/shard.cu, the request exchange on CUDA tensors, both halo routes (the IPC push of csrc/halo.cu and pack + all-to-all),
gnnb_propagate_halo on the shard plans and dist_gcn_conv forward and backward.

Every result is checked against a float64 statement over the whole graph and against the one-GPU library on the same
graph: the shards' CSR mapped back to global ids, the request lists, propagate bits on rows of at most one chunk of edges
(a shard reduces such a row in the single-GPU order), the normwise error on longer rows, the layer's y, dx, dW and db.

A spawn group runs many cases and sends back one small record per check: (case, rank, ok, worst error, first differing
index).  The pytest functions below read those records."""
import ctypes as C
import datetime
import os
import queue as queue_mod
import socket
import sys
import time
import traceback

import numpy as np
import pytest
import torch

pytestmark = pytest.mark.gpu

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
CHUNK = 128                                  # the library's default chunk of edges per work item (gnnb_set_chunk_edges)
DS = (1, 3, 5, 128, 256, 260, 512)           # scalar and float4 push, the lean kernels at 128 / 256 / 512
TOL_LONG = 2e-6                              # rows split over several chunks, normwise against float64
TOL_LAYER = 1e-5                             # the one-GPU GCN layer tests' bar
N_NODES = 600
INNER = (560, 600)                           # nodes with only mutually internal edges
ISOLATED = (500, 520)                        # nodes without any edge
LAYERS = ((256, 256), (128, 128), (16, 7), (8, 4))


# ------------------------------------------------------------------------------------------------ graph and bounds
def make_graph(seed=11):
    """~6,000 edges over 600 nodes (0-based), low ids are hubs as in RMAT; two target hubs of ~330 in-edges (about three
    chunks) and one source hub of ~330 out-edges whose other ends are spread over the whole id range; duplicate edges and
    input self loops; isolated nodes; a block of nodes whose edges stay inside the block.  Returned in shuffled COO order."""
    rng = np.random.default_rng(seed)
    main = np.r_[0:ISOLATED[0], ISOLATED[1]:INNER[0]]
    m = main.size
    pick = lambda k, p: main[np.minimum((rng.random(k) ** p * m).astype(np.int64), m - 1)]
    s, t = [pick(4600, 3)], [pick(4600, 2)]
    for hub in (200, 301):
        s.append(main[rng.integers(0, m, 330)]); t.append(np.full(330, hub))
    s.append(np.full(330, 450)); t.append(main[rng.integers(0, m, 330)])
    s.append(rng.integers(*INNER, 250)); t.append(rng.integers(*INNER, 250))
    loops = main[rng.integers(0, m, 40)]
    s.append(loops); t.append(loops)
    s, t = np.concatenate(s), np.concatenate(t)
    dup = rng.integers(0, s.size, 150)
    s, t = np.concatenate([s, s[dup], [570]]), np.concatenate([t, t[dup], [570]])
    p = rng.permutation(s.size)
    return s[p].astype(np.int64), t[p].astype(np.int64)


def explicit_bounds(W):
    """W = 2: the last rank owns only the inner block (no halo, sends nothing); W = 3: the middle rank is empty;
    W = 4: both"""
    return {2: [0, INNER[0], N_NODES], 3: [0, 280, 280, N_NODES], 4: [0, 280, INNER[0], INNER[0], N_NODES]}[W]


def ownership_cases(W):
    return [("contiguous", dict(ownership="contiguous")),
            ("bounds", dict(ownership="contiguous", bounds=explicit_bounds(W))),
            ("cyclic", dict(ownership="cyclic")),
            ("balanced", dict(ownership="balanced"))]


# ------------------------------------------------------------------------------------------------ comparisons
def bits_diff(a, b):
    """(equal, first differing flat index or -1) of two float32 tensors, bit for bit (NaN payloads included)"""
    a, b = a.contiguous().reshape(-1), b.contiguous().reshape(-1)
    if a.numel() != b.numel():
        return False, -2
    bad = torch.nonzero(a.view(torch.int32) != b.view(torch.int32))
    return bad.numel() == 0, (int(bad[0]) if bad.numel() else -1)


def bits_record(a, b):
    """(ok, worst, first differing index) of a bit comparison, as a record's tail"""
    ok, first = bits_diff(a, b)
    return ok, 0.0, first


def rel_err(a, r):
    """normwise relative error over the finite entries of r; inf with the first index when the non-finite entries of
    a and r differ (mask or value)"""
    a, r = a.double().reshape(-1), r.double().reshape(-1)
    fa, fr = torch.isfinite(a), torch.isfinite(r)
    same_nf = (a == r) | (torch.isnan(a) & torch.isnan(r))
    bad = torch.nonzero((fa != fr) | (~fr & ~same_nf))
    if bad.numel():
        return float("inf"), int(bad[0])
    if not bool(fr.any()):
        return 0.0, -1
    d = (a - r).masked_fill(~fr, 0)
    err = float(torch.linalg.vector_norm(d) / max(float(torch.linalg.vector_norm(r[fr])), 1e-30))
    return err, int(torch.argmax(d.abs()))


def free_port():
    with socket.socket() as s:
        s.bind(("127.0.0.1", 0))
        return s.getsockname()[1]


def compute_mode(index=0):
    """the device's compute mode through the driver API (read-only; 0 = Default)"""
    cu = C.CDLL("libcuda.so.1")
    dev, mode = C.c_int(), C.c_int()
    if cu.cuInit(0) != 0 or cu.cuDeviceGet(C.byref(dev), index) != 0:
        return None
    if cu.cuDeviceGetAttribute(C.byref(mode), 20, dev) != 0:     # CU_DEVICE_ATTRIBUTE_COMPUTE_MODE
        return None
    return mode.value


# ------------------------------------------------------------------------------------------------ rank side
class Rank:
    """what every check of one rank needs: the library, the graph on the device and the record queue"""

    def __init__(self, rank, W, q, dev):
        sys.path.insert(0, ROOT)
        import gnnb200
        from gnnb200 import partition
        self.gnn, self.P, self.rank, self.W, self.q, self.dev = gnnb200, partition, rank, W, q, dev
        self.requests = []
        orig = partition.exchange_requests

        def spy(halo_local, recv_counts, group=None):            # the request list of every shard, as built
            self.requests.append((halo_local.clone(), list(recv_counts)))
            return orig(halo_local, recv_counts, group)
        partition.exchange_requests = spy

    def put(self, case, ok, worst=0.0, first=-1):
        self.q.put((case, self.rank, bool(ok), float(worst), first))

    def gather(self, obj):
        import torch.distributed as dist
        out = [None] * self.W
        dist.all_gather_object(out, obj)
        return out

    def stream(self):
        return torch.cuda.current_stream(self.dev).cuda_stream

    def set_route(self, halo="push", slices=1):
        os.environ["GNNB_HALO"] = halo
        os.environ["GNNB_HALO_SLICES"] = str(slices)

    def build(self, G, loops, chunked, **own):
        """DistGraph from int64 (s, t), or from ragged int32 chunks of 997 edges; returns it with its two request lists"""
        s1 = torch.as_tensor(G["s"] + 1, device=self.dev)
        t1 = torch.as_tensor(G["t"] + 1, device=self.dev)
        n0 = len(self.requests)
        if chunked:
            s32, t32 = s1.to(torch.int32), t1.to(torch.int32)
            chunks = [(s32[i:i + 997], t32[i:i + 997]) for i in range(0, s32.numel(), 997)]
            dg = self.P.DistGraph.from_chunks(chunks, N_NODES, add_self_loops=loops, device=self.dev, **own)
        else:
            dg = self.P.DistGraph(s1, t1, N_NODES, add_self_loops=loops, device=self.dev, **own)
        assert len(self.requests) == n0 + 2
        return dg, self.requests[n0:n0 + 2]


class Reference:
    """the full graph (with the appended loops when the layer adds them) on one GPU and in float64"""

    def __init__(self, R, G, loops):
        gnn, n = R.gnn, N_NODES
        self.R, self.n = R, n
        s, t = G["s"], G["t"]
        if loops:
            s, t = np.concatenate([s, np.arange(n)]), np.concatenate([t, np.arange(n)])
        self.s, self.t = s, t                                   # 0-based, COO order, loops last
        g = gnn.GNNGraph(torch.as_tensor(G["s"] + 1), torch.as_tensor(G["t"] + 1), num_nodes=n).cuda()
        self.g = gnn.add_self_loops(g) if loops else g
        self.plan = self.g.plan()
        self.c = gnn.layers._gcn_c(self.g)
        self.deg = (np.bincount(t, minlength=n), np.bincount(s, minlength=n))     # row lengths: forward, backward
        self.st = torch.as_tensor(s, device=R.dev), torch.as_tensor(t, device=R.dev)
        self.c64 = torch.as_tensor(self.deg[0], dtype=torch.float64, device=R.dev).rsqrt()

    def one_gpu(self, tr, x):
        out = torch.empty_like(x)
        self.R.gnn._lib.check(self.R.gnn._lib.lib.gnnb_gcn_propagate(self.plan.h, tr, x.data_ptr(), None, None, x.shape[1],
                                                                     out.data_ptr(), self.R.stream()))
        return out

    def f64(self, tr, x):
        """c .* (sum over the row's edges of c[j] x[j]) per edge, in float64 (no dense product: inf * 0 stays out)"""
        s, t = self.st
        key, other = (t, s) if tr == 0 else (s, t)
        out = torch.zeros(x.shape, dtype=torch.float64, device=x.device)
        out.index_add_(0, key, x.double()[other] * self.c64[other, None])
        return out * self.c64[:, None]


def check_structure(R, tag, dg, req, ref):
    """the shards mapped back to global ids equal the global COO per row, in COO order; the halo lists and request
    lists equal what the edges imply; send_idx of q toward p is p's request list toward q.  Returns the global node of
    every halo row, per shard."""
    W, rank, n = dg.world, dg.rank, N_NODES
    first, lo, hi = dg.first, dg.lo, dg.hi
    ids = dg.local_nodes().cpu().numpy().astype(np.int64)
    all_ids = R.gather(ids)
    node_of = np.concatenate(all_ids)                          # partition id -> node
    ok = (node_of.size == n and np.array_equal(np.sort(node_of), np.arange(n))
          and all(all_ids[q].size == first[q + 1] - first[q] for q in range(W)))
    pid_of = np.empty(n, np.int64)
    if ok:
        pid_of[node_of] = np.arange(n)
        v = np.arange(n)
        if dg.ownership == "contiguous":
            ok = np.array_equal(pid_of, v)
        elif dg.ownership == "cyclic":
            ok = np.array_equal(pid_of, np.asarray(first)[v % W] + v // W)
        else:
            ok = np.array_equal(pid_of, R.P.to_pid(torch.arange(n, device=R.dev), W, first, "balanced",
                                                   dg._relabel).cpu().numpy())
    R.put(f"structure/{tag}/ownership", ok)
    if not ok:
        raise AssertionError(f"{tag}: the ranks' local_nodes() are not the ownership rule's partition")
    halos = []
    for d, (sh, key, other) in enumerate(((dg.fwd, ref.t, ref.s), (dg.bwd, ref.s, ref.t))):
        name = ("fwd", "bwd")[d]
        halo_local, rc = req[d][0].cpu().numpy().astype(np.int64), req[d][1]
        owner = np.repeat(np.arange(W), rc)
        halo_pid = halo_local + np.asarray(first, np.int64)[owner]
        kp, op = pid_of[key], pid_of[other]
        sel = (kp >= lo) & (kp < hi)                           # COO order kept
        rows_e, other_e, other_p = kp[sel] - lo, other[sel], op[sel]
        exp_halo = np.unique(other_p[(other_p < lo) | (other_p >= hi)])
        exp_rc = np.bincount(np.searchsorted(np.asarray(first[1:]), exp_halo, side="right"), minlength=W)[:W]
        ok = (np.array_equal(halo_pid, exp_halo) and sh.n_halo == exp_halo.size and list(rc) == exp_rc.tolist()
              and sh.recv_counts == list(rc) and sh.n_local == hi - lo)
        R.put(f"structure/{tag}/{name}/halo", ok)
        halo_nodes = node_of[halo_pid] if ok else np.zeros(0, np.int64)
        halos.append(torch.as_tensor(halo_nodes, device=R.dev))
        ne = sh.num_edges
        rowptr = np.zeros(sh.n_local + 1, np.int32)
        col, eid = np.zeros(max(ne, 1), np.int32), np.zeros(max(ne, 1), np.int32)
        R.gnn._lib.check(R.gnn._lib.lib.gnnb_graph_csr(sh.plan.h, 0, rowptr.ctypes.data, col.ctypes.data, eid.ctypes.data,
                                                       None))
        col, eid = col[:ne].astype(np.int64), eid[:ne]
        order = np.argsort(rows_e, kind="stable")
        exp_rows, exp_other = rows_e[order], other_e[order]
        got_rows = np.repeat(np.arange(sh.n_local), np.diff(rowptr))
        space = np.concatenate([ids, halo_nodes])
        in_range = (col >= 0) & (col < space.size)
        got_other = np.where(in_range, space[np.clip(col, 0, max(space.size - 1, 0))] if space.size else -1, -1)
        ok = ne == exp_rows.size and got_rows.size == ne and np.array_equal(got_rows, exp_rows) and np.array_equal(got_other, exp_other)
        first_bad = -1
        if not ok and ne == exp_rows.size and got_rows.size == ne:
            bad = np.nonzero((got_rows != exp_rows) | (got_other != exp_other))[0]
            first_bad = int(bad[0]) if bad.size else -1
        R.put(f"structure/{tag}/{name}/rows_in_coo_order", ok, 0.0, first_bad)
    sends = R.gather([(sh.send_idx.cpu().numpy(), list(sh.send_counts)) for sh in (dg.fwd, dg.bwd)])
    reqs = R.gather([(r[0].cpu().numpy(), list(r[1])) for r in req])
    for d, name in enumerate(("fwd", "bwd")):
        ok = True
        for q in range(W):                                     # what I send to q == what q asked of me
            idx, counts = sends[rank][d]
            seg = np.concatenate([[0], np.cumsum(counts)])
            mine = idx[seg[q]:seg[q + 1]]
            qh, qrc = reqs[q][d]
            qseg = np.concatenate([[0], np.cumsum(qrc)])
            ok &= np.array_equal(mine, qh[qseg[rank]:qseg[rank + 1]]) and counts[q] == qrc[rank]
        R.put(f"structure/{tag}/{name}/send_idx_is_the_peers_request", ok)
    return halos


def shard_dump(dg, req):
    out = []
    for sh, r in zip((dg.fwd, dg.bwd), req):
        ne = sh.num_edges
        rowptr = np.zeros(sh.n_local + 1, np.int32)
        col, eid = np.zeros(max(ne, 1), np.int32), np.zeros(max(ne, 1), np.int32)
        import gnnb200
        gnnb200._lib.check(gnnb200._lib.lib.gnnb_graph_csr(sh.plan.h, 0, rowptr.ctypes.data, col.ctypes.data,
                                                           eid.ctypes.data, None))
        out.append((rowptr, col[:ne], eid[:ne], sh.send_idx.cpu().numpy(), list(sh.send_counts), list(sh.recv_counts),
                    r[0].cpu().numpy(), sh.n_halo))
    return out


def same_dump(a, b):
    return all(all(np.array_equal(np.asarray(u), np.asarray(v)) for u, v in zip(x, y)) for x, y in zip(a, b))


def check_propagate(R, tag, dg, ref, halos):
    c, cf, cb = dg.gcn_c()
    ids = dg.local_nodes()
    nl = dg.n_local
    ok = (bits_diff(c, ref.c[ids])[0] and bits_diff(cf[nl:], ref.c[halos[0]])[0] and bits_diff(cb[nl:], ref.c[halos[1]])[0]
          and bits_diff(cf[:nl], c)[0] and bits_diff(cb[:nl], c)[0])
    R.put(f"propagate/{tag}/c_and_its_halo_copies", ok)
    ids_np = ids.cpu().numpy()
    for D in DS:
        gen = torch.Generator(device=R.dev).manual_seed(100 + D)
        x = torch.randn(N_NODES, D, device=R.dev, generator=gen)
        xl = x[ids].contiguous()
        for d, (sh, cs) in enumerate(((dg.fwd, cf), (dg.bwd, cb))):
            name = f"propagate/{tag}/{('fwd', 'bwd')[d]}/D{D}"
            one = ref.one_gpu(d, x)[ids]
            r64 = ref.f64(d, x)[ids]
            outs = {}
            for route, halo, slices in (("push", "push", 1), ("alltoall", "nccl", 1), ("sliced", "push", 2)):
                R.set_route(halo, slices)
                outs[route] = dg.propagate(sh, xl, cs, c)
            R.set_route()
            short = torch.as_tensor(ref.deg[d][ids_np] <= CHUNK, device=R.dev)
            R.put(f"{name}/short_rows_bits_one_gpu", *bits_record(outs["push"][short], one[short]))
            err, at = rel_err(outs["push"][~short], r64[~short])
            R.put(f"{name}/long_rows_f64", err <= TOL_LONG, err, at)
            R.put(f"{name}/alltoall_bits_push", *bits_record(outs["alltoall"], outs["push"]))
            R.put(f"{name}/sliced_bits_unsliced", *bits_record(outs["sliced"], outs["push"]))


def one_step(R, dg, layer, x_full, dy_full):
    """dist_gcn_conv forward and backward on this rank's rows; y and dx of the local rows, all-reduced dW and db"""
    import torch.distributed as dist
    gnn = R.gnn
    ids = dg.local_nodes()
    layer.zero_grad(set_to_none=True)
    x = gnn.unrows(x_full[ids].contiguous()).requires_grad_(True)
    y = R.P.dist_gcn_conv(layer, dg, x)
    y.backward(gnn.unrows(dy_full[ids].contiguous()))
    dW = layer.weight.grad.clone()
    dist.all_reduce(dW)
    db = None
    if layer.bias is not None and layer.bias is not False:
        db = layer.bias.grad.clone()
        dist.all_reduce(db)
    return gnn.rows(y.detach()).clone(), gnn.rows(x.grad).clone(), dW, db


def make_layer(R, Din, Dout, bias, loops):
    torch.manual_seed(1000 * Din + Dout)
    layer = R.gnn.GCNConv(Din, Dout, torch.relu, bias=bias, add_self_loops=loops, device=R.dev)
    if bias:
        with torch.no_grad():
            layer.bias.copy_(torch.linspace(-0.5, 0.5, Dout))
    return layer


def check_layer(R, tag, dg, ref):
    gnn, n = R.gnn, N_NODES
    ids = dg.local_nodes()
    R.set_route()
    for Din, Dout in LAYERS:
        for bias in (True, False):
            name = f"layer/{tag}/{Din}to{Dout}{'' if bias else '_nobias'}"
            layer = make_layer(R, Din, Dout, bias, dg.self_loops)
            gen = torch.Generator(device=R.dev).manual_seed(7 * Din + Dout)
            x_full = torch.randn(n, Din, device=R.dev, generator=gen)
            dy_full = torch.randn(n, Dout, device=R.dev, generator=gen)
            y, dx, dW, db = one_step(R, dg, layer, x_full, dy_full)
            if dg.self_loops:                                  # float64 autograd of the dense formula
                A = torch.zeros(n, n, dtype=torch.float64, device=R.dev)
                A.index_put_(ref.st, torch.ones(ref.s.size, dtype=torch.float64, device=R.dev), accumulate=True)
                c = A.sum(0).rsqrt()
                x64 = x_full.double().requires_grad_(True)
                W64 = layer.weight.detach().double().requires_grad_(True)
                pre = (c[:, None] * (A.t() @ (c[:, None] * x64))) @ W64.t()
                b64 = None
                if bias:
                    b64 = layer.bias.detach().double().requires_grad_(True)
                    pre = pre + b64
                y64 = torch.relu(pre)
                y64.backward(dy_full.double())
                refs = {"y": (y, y64.detach()[ids]), "dx": (dx, x64.grad[ids]), "dW": (dW, W64.grad)}
                if bias:
                    refs["db"] = (db, b64.grad)
            else:                                              # isolated targets: the one-GPU layer's non-finite entries
                layer.zero_grad(set_to_none=True)
                xg = gnn.unrows(x_full.clone()).requires_grad_(True)
                yg = layer(ref.g, xg)
                yg.backward(gnn.unrows(dy_full.clone()))
                refs = {"y": (y, gnn.rows(yg.detach())[ids]), "dx": (dx, gnn.rows(xg.grad)[ids])}
            for k, (a, r) in refs.items():
                err, at = rel_err(a, r)
                R.put(f"{name}/{k}", err <= TOL_LAYER, err, at)


def check_steps(R, G, own):
    """three steps with different x on one DistGraph equal fresh one-step runs bit for bit, with two halo buffers and
    with one"""
    n = N_NODES
    R.set_route()
    for nbuf in ("2", "1"):
        os.environ["GNNB_HALO_BUFFERS"] = nbuf
        layer = make_layer(R, 128, 128, True, True)
        xs = [torch.randn(n, 128, device=R.dev, generator=torch.Generator(device=R.dev).manual_seed(50 + k)) for k in range(3)]
        dy = torch.randn(n, 128, device=R.dev, generator=torch.Generator(device=R.dev).manual_seed(49))
        dg, _ = R.build(G, True, False, **own)
        steps = [one_step(R, dg, layer, x, dy) for x in xs]
        dg.close()
        for k, x in enumerate(xs):
            fresh, _ = R.build(G, True, False, **own)
            once = one_step(R, fresh, layer, x, dy)
            fresh.close()
            for name, a, b in zip(("y", "dx", "dW", "db"), steps[k], once):
                R.put(f"steps/{own['ownership']}/buffers{nbuf}/step{k}/{name}", *bits_record(a, b))
    os.environ["GNNB_HALO_BUFFERS"] = "2"


def run_cases(R, multi_device):
    G = dict(zip(("s", "t"), make_graph()))
    refs = {}
    for tag, own in ownership_cases(R.W):
        for loops in (True, False):
            full = f"W{R.W}/{tag}/{'loops' if loops else 'noloops'}"
            ref = refs.get(loops) or refs.setdefault(loops, Reference(R, G, loops))
            dg, req = R.build(G, loops, False, **own)
            halos = check_structure(R, full, dg, req, ref)
            if not multi_device:
                kw = dict(own, bounds=dg.bounds) if own["ownership"] == "contiguous" else own
                dc, reqc = R.build(G, loops, True, **kw)
                R.put(f"structure/{full}/from_chunks_identical", same_dump(shard_dump(dg, req), shard_dump(dc, reqc)))
                dc.close()
            check_propagate(R, full, dg, ref, halos)
            check_layer(R, full, dg, ref)
            dg.close()
    for tag, own in ownership_cases(R.W)[1:3]:
        check_steps(R, G, own)


def worker(rank, W, port, q, multi_device):
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


def scale_worker(rank, W, port, q):
    """RMAT N = 1 M, E = 10 M over W ranks, 'balanced' ownership, shards from 1 M-edge chunks, D = 256 with loops"""
    import torch.distributed as dist
    os.environ.update(MASTER_ADDR="127.0.0.1", MASTER_PORT=str(port), GNNB_HALO="push", GNNB_HALO_SLICES="1",
                      GNNB_HALO_BUFFERS="2")
    dev = torch.device("cuda", 0)
    torch.cuda.set_device(dev)
    try:
        dist.init_process_group("gloo", rank=rank, world_size=W, timeout=datetime.timedelta(seconds=600))
        R = Rank(rank, W, q, dev)
        n, E, D, ce = 1_000_000, 10_000_000, 256, 1 << 20
        dg = R.P.DistGraph.from_rmat(n, E, device=dev, add_self_loops=True, ownership="balanced", chunk_edges=ce)
        pairs = [(a.clone(), b.clone()) for a, b in R.P.rmat_chunks(n, E, 17, dev, ce)]
        s = torch.cat([a for a, _ in pairs] + [torch.arange(1, n + 1, device=dev)]) - 1
        t = torch.cat([b for _, b in pairs] + [torch.arange(1, n + 1, device=dev)]) - 1
        del pairs
        g = R.gnn.add_self_loops(R.gnn.GNNGraph(s[:E] + 1, t[:E] + 1, num_nodes=n))
        plan = g.plan()
        deg = (torch.bincount(t, minlength=n), torch.bincount(s, minlength=n))
        c64 = deg[0].double().rsqrt()
        c, cf, cb = dg.gcn_c()
        ids = dg.local_nodes()
        x = torch.randn(n, D, device=dev, generator=torch.Generator(device=dev).manual_seed(5))
        xl = x[ids].contiguous()
        gen = torch.Generator(device=dev).manual_seed(6)
        sample = torch.unique(torch.cat([torch.topk(deg[0], 32).indices, torch.topk(deg[1], 32).indices,
                                         torch.randint(0, n, (4000,), device=dev, generator=gen)]))
        own_mask = torch.zeros(n, dtype=torch.bool, device=dev)
        own_mask[ids] = True
        pos = torch.full((n,), -1, dtype=torch.int64, device=dev)
        pos[ids] = torch.arange(ids.numel(), device=dev)
        mine = sample[own_mask[sample]]
        for d, (sh, cs) in enumerate(((dg.fwd, cf), (dg.bwd, cb))):
            name = f"scale/W{W}/{('fwd', 'bwd')[d]}"
            out = dg.propagate(sh, xl, cs, c)
            one = torch.empty_like(x)
            R.gnn._lib.check(R.gnn._lib.lib.gnnb_gcn_propagate(plan.h, d, x.data_ptr(), None, None, D, one.data_ptr(),
                                                               R.stream()))
            one = one[ids]
            short = deg[d][ids] <= CHUNK
            R.put(f"{name}/short_rows_bits_one_gpu", *bits_record(out[short], one[short]))
            err, at = rel_err(out, one)
            R.put(f"{name}/one_gpu_normwise", err <= TOL_LONG, err, at)
            del one
            key, other = (t, s) if d == 0 else (s, t)             # float64 over the sample's edges, torch double ops
            slot = torch.full((n,), -1, dtype=torch.int64, device=dev)
            slot[mine] = torch.arange(mine.numel(), device=dev)
            e = torch.nonzero(slot[key] >= 0).squeeze(1)
            r64 = torch.zeros(mine.numel(), D, dtype=torch.float64, device=dev)
            r64.index_add_(0, slot[key[e]], x[other[e]].double() * c64[other[e], None])
            r64 *= c64[mine, None]
            err, at = rel_err(out[pos[mine]], r64)
            R.put(f"{name}/f64_sample_{mine.numel()}_rows", err <= TOL_LONG, err, at)
            del out
        dg.close()
        torch.cuda.synchronize(dev)
        dist.barrier()
        q.put(("done", rank, True, 0.0, -1))
    except BaseException:
        q.put(("error", rank, False, 0.0, traceback.format_exc()[-4000:]))
    finally:
        if dist.is_initialized():
            dist.destroy_process_group()


# ------------------------------------------------------------------------------------------------ pytest side
_GROUPS = {}


def run_group(target, W, *extra, timeout=900):
    """spawn W daemon ranks, collect their records until every rank is done (or one fails), and leave no process
    behind"""
    key = (target.__name__, W) + extra
    if key in _GROUPS:
        return _GROUPS[key]
    import torch.multiprocessing as mp
    ctx = mp.get_context("spawn")
    q = ctx.Queue()
    port = free_port()
    procs = [ctx.Process(target=target, args=(r, W, port, q) + extra, daemon=True) for r in range(W)]
    records, done, errors = [], set(), []
    t_end = time.monotonic() + timeout
    try:
        for p in procs:
            p.start()
        while len(done) < W and not errors:
            try:
                rec = q.get(timeout=max(1.0, t_end - time.monotonic()))
            except queue_mod.Empty:
                errors.append(f"timed out after {timeout} s with ranks {sorted(done)} done")
                break
            if rec[0] == "done":
                done.add(rec[1])
            elif rec[0] == "error":
                errors.append(f"rank {rec[1]}: {rec[4]}")
            else:
                records.append(rec)
        for p in procs:
            p.join(timeout=60 if not errors else 5)
    finally:
        for p in procs:
            if p.is_alive():
                p.terminate()
        for p in procs:
            p.join()
        q.close()
    _GROUPS[key] = (records, errors, [p.exitcode for p in procs])
    return _GROUPS[key]


def require_shared_device():
    if not torch.cuda.is_available():
        pytest.skip("no CUDA device")
    mode = compute_mode(torch.cuda.current_device() if torch.cuda.is_initialized() else 0)
    if mode != 0:
        pytest.skip(f"compute mode {mode} is not Default: several rank processes cannot share the device")


def assert_records(records, errors, exitcodes, prefix):
    assert not errors, "\n".join(errors)
    assert all(c == 0 for c in exitcodes), exitcodes
    mine = [r for r in records if r[0].startswith(prefix)]
    assert mine, f"no {prefix} records"
    bad = [f"{case} rank {rank}: worst {worst:.3e} first differing index {first}"
           for case, rank, ok, worst, first in mine if not ok]
    assert not bad, f"{len(bad)} of {len(mine)} {prefix} checks failed:\n" + "\n".join(bad[:40])


def test_shard_without_targets_needs_no_output_buffer():
    """an empty rank's shard plan (no node, no edge): gnnb_gcn_norm and gnnb_propagate_halo accept the NULL data pointer
    of torch's empty CUDA tensors, since there is nothing to write"""
    if not torch.cuda.is_available():
        pytest.skip("no CUDA device")
    sys.path.insert(0, ROOT)
    import gnnb200 as gnn
    lib, dev = gnn._lib.lib, torch.device("cuda", 0)
    h = C.c_void_p()
    gnn._lib.check(lib.gnnb_graph_create(C.byref(h), None, None, 0, 0, 0, 4, 0, 1, None))
    plan = gnn.graph._Plan(h.value, dev)
    c = torch.empty(0, device=dev)
    gnn._lib.check(lib.gnnb_gcn_norm(plan.h, None, c.data_ptr(), None))
    x = torch.empty(0, 8, device=dev)
    gnn._lib.check(lib.gnnb_propagate_halo(plan.h, gnn._lib.COPY_XJ, gnn._lib.SUM, x.data_ptr(), None, 0, None,
                                           c.data_ptr(), c.data_ptr(), 8, x.data_ptr(), None))
    # the layer's pullback on the rank's zero rows: relu-masked 128 -> 128, dx empty, dW and db all-reduced afterwards
    torch.manual_seed(0)
    layer = gnn.GCNConv(128, 128, torch.relu, device=dev)
    x0 = gnn.unrows(torch.empty(0, 128, device=dev)).requires_grad_(True)
    gnn.layers._linear(layer, layer.weight, x0, True).sum().backward()
    assert x0.grad.shape == x0.shape and int(torch.count_nonzero(layer.weight.grad)) == 0


@pytest.mark.parametrize("W", [2, 3, 4])
@pytest.mark.parametrize("check", ["structure", "propagate", "layer", "steps"])
def test_partition_on_one_device(W, check):
    """W gloo ranks on one device: `check` names the family of records (shards, propagate bits, layer, repeated steps)"""
    require_shared_device()
    assert_records(*run_group(worker, W, False), prefix=check + "/")


def test_partition_at_scale_on_one_device():
    """RMAT 1 M nodes / 10 M edges, 4 ranks, balanced ownership: the multi-chunk builder, the device relabel and hub rows
    whose sources sit on every rank"""
    require_shared_device()
    assert_records(*run_group(scale_worker, 4, timeout=1200), prefix="scale/")


def test_partition_one_rank_per_device_nccl():
    """one rank per device under NCCL with the push route over real peer mappings (the transport of bench config 5)"""
    if not torch.cuda.is_available() or torch.cuda.device_count() < 2:
        pytest.skip("needs at least two visible CUDA devices: NCCL refuses two ranks on one device")
    W = min(torch.cuda.device_count(), 4)
    records, errors, codes = run_group(worker, W, True)
    for prefix in ("structure/", "propagate/", "layer/", "steps/"):
        assert_records(records, errors, codes, prefix)
