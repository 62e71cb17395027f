"""Node-partitioned message passing across the GPUs of one box (SURVEY.md §8e; the reference has no
distributed code at all — this is new work prescribed by BASELINE.json's north_star).

Layout: nodes are split into `world` contiguous ranges (cost-balanced: a node costs NODE_COST edge-equivalents
for the dense per-node work plus its in- and out-degree).  Rank p owns x[:, lo_p:hi_p], every in-edge of its
nodes (forward shard) and every out-edge of its nodes (backward shard).  One pass =

    pack the rows each peer asked for (gnnb_gather_rows)  ->  one all-to-all-v over NCCL/NVLink
    ->  ONE fused segmented-reduce kernel over the [local rows | halo rows] source space (gnnb_propagate_halo)

The halo lists are deduplicated per peer (each remote row crosses NVLink once per pass) and built once.
Both directions are "pull": the backward pass gathers dout rows of remote targets through the backward shard,
so there is no scatter-reduce across GPUs and every result stays deterministic; inside a target row the
edges keep their COO order, so a shard reproduces the single-GPU summation order.

Message passing on shards: dist_propagate (copy_xj / w_mul_xj with +, mean, max or min; max and min pull back through
gnnb_propagate_maxmin_bwd_halo, which reads the halo rows of dout and of the forward result).  Layers on shards:
dist_gcn_conv, dist_sage_conv (mean, +), dist_graph_conv, dist_gin_conv and dist_gat_conv.  GAT's pullback has one term that
crosses ranks, del of a target = the sum of its in-edges' dz, computed by the owners of their sources: the dz rows move
to the targets' owners by one all-to-all in an order both shards already share (DistGraph._edge_route).  Weighted
GCNConv keeps each shard's edge weights (an ownership mask over the global order) and moves an explicit per-rank
edge_weight to the backward shard over the same route reversed; its gradient is gnnb_gcn_edge_weight_grad_halo.

`torch.distributed` is plumbing (process group, all_to_all_single); index construction below is plain torch
ops that also run on CPU tensors with the gloo backend (tests/test_partition_gloo.py).
"""
from __future__ import annotations

import ctypes as C
import json
import os
import time
from typing import List, Optional

import torch
import torch.distributed as dist

from . import _lib
from ._lib import lib
from .graph import _Plan, _ptr, _stream, rows, unrows

NODE_COST = 12  # dense per-node work (GEMM, bias, relu, grads) in edge-equivalents, from the 1-GPU profile (1.9 ns/node vs 0.17 ns/edge)


# ---------------------------------------------------------------------------------------------------------
# index construction (device agnostic)
# ---------------------------------------------------------------------------------------------------------
def balanced_bounds(cost: torch.Tensor, world: int) -> List[int]:
    """contiguous ranges [b[p], b[p+1]) with ~equal total cost."""
    n = cost.numel()
    cs = torch.cumsum(cost.to(torch.float64), 0)
    total = float(cs[-1]) if n else 0.0
    targets = torch.tensor([total * p / world for p in range(1, world)], dtype=torch.float64, device=cost.device)
    cuts = torch.searchsorted(cs, targets).tolist() if world > 1 else []
    b = [0] + [min(max(int(c) + 1, 0), n) for c in cuts] + [n]
    for i in range(1, len(b)):
        b[i] = max(b[i], b[i - 1])
    return b


def ownership_first(num_nodes: int, world: int, ownership: str, bounds: Optional[List[int]] = None) -> List[int]:
    """Start of every rank's range in partition-id space (world + 1 entries).  'contiguous': the node ranges themselves
    (`bounds`, or equal ranges); 'cyclic': node v (0-based) belongs to rank v % world as local row v // world, so rank q
    owns ceil((N - q) / world) nodes — the hubs of a skewed id space (RMAT: the low ids) spread over all ranks."""
    if ownership == "contiguous":
        return list(bounds) if bounds is not None else [(num_nodes * q) // world for q in range(world + 1)]
    assert ownership in ("cyclic", "balanced"), ownership
    first = [0]
    for q in range(world):
        first.append(first[-1] + (num_nodes - q + world - 1) // world)
    return first


def to_pid(v0: torch.Tensor, world: int, first: List[int], ownership: str, relabel: Optional[torch.Tensor] = None) -> torch.Tensor:
    """node id (0-based) -> partition id: the bijection onto [0, N) in which every rank owns one contiguous range"""
    if ownership == "contiguous":
        return v0
    if relabel is not None:
        v0 = relabel.to(v0.dtype)[v0]
    ft = torch.tensor(first[:-1], dtype=v0.dtype, device=v0.device)
    return ft[v0 % world] + v0 // world


def degree_order(chunks, num_nodes: int, device) -> torch.Tensor:
    """nodes by decreasing in+out degree (stable: ties keep id order) — the order in which 'balanced' ownership deals
    them to the ranks; the torch restatement of gnnb_degree_accumulate + the sort of gnnb_balanced_relabel."""
    cost = torch.zeros(num_nodes, dtype=torch.int64, device=device)
    for sc, tc, *_ in chunks:
        cost += torch.bincount(sc.to(device).to(torch.int64) - 1, minlength=num_nodes)
        cost += torch.bincount(tc.to(device).to(torch.int64) - 1, minlength=num_nodes)
    return torch.sort(cost, descending=True, stable=True).indices


def build_shard(key0: torch.Tensor, other0: torch.Tensor, lo: int, hi: int, bounds: List[int],
                self_loops: bool):
    """Edges whose reduction row `key0` (0-based partition id) lies in [lo,hi), re-indexed for one GPU — the torch
    restatement of csrc/shard.cu, used for CPU tensors (gloo tests of the host logic).

    Returns dict(row: local reduction row, col: gathered node in [local | halo] space, halo: sorted partition ids of
    the remote gathered nodes, halo_local: their owner-local rows, recv_counts: rows expected from every owner)."""
    sel = (key0 >= lo) & (key0 < hi)
    k = key0[sel] - lo
    o = other0[sel]
    n_local = hi - lo
    is_local = (o >= lo) & (o < hi)
    halo = torch.unique(o[~is_local])                       # sorted => grouped by owner (ranges are contiguous)
    col = torch.where(is_local, o - lo, n_local + torch.searchsorted(halo, o))
    if self_loops:                                          # (i,i) appended after the originals (transform.jl:17-19)
        loops = torch.arange(n_local, dtype=k.dtype, device=k.device)
        k = torch.cat([k, loops])
        col = torch.cat([col, loops])
    edges = torch.tensor(bounds[1:], dtype=halo.dtype, device=halo.device)
    owner = torch.bucketize(halo, edges, right=True)
    recv_counts = torch.bincount(owner, minlength=len(bounds) - 1).tolist()
    starts = torch.tensor(bounds[:-1], dtype=halo.dtype, device=halo.device)
    halo_local = (halo - starts[owner]).to(torch.int32)
    return {"row": k, "col": col, "halo": halo, "halo_local": halo_local, "recv_counts": recv_counts, "n_local": n_local}


def exchange_requests(halo_local: torch.Tensor, recv_counts: List[int], group=None):
    """Tell every owner which of its rows (owner-local int32 indices, grouped by owner) this rank needs.  Returns
    (send_idx: int32 local row ids to pack, in peer order; send_counts)."""
    dev = halo_local.device
    rc = torch.tensor(recv_counts, dtype=torch.int64, device=dev)
    sc = torch.empty_like(rc)
    dist.all_to_all_single(sc, rc, group=group)
    send_counts = sc.tolist()
    wanted = torch.empty(int(sum(send_counts)), dtype=torch.int32, device=dev)
    dist.all_to_all_single(wanted, halo_local.to(torch.int32).contiguous(), output_split_sizes=send_counts,
                           input_split_sizes=recv_counts, group=group)
    return wanted, send_counts


# ---------------------------------------------------------------------------------------------------------
# the distributed graph
# ---------------------------------------------------------------------------------------------------------
class _DeviceRows:
    """(n, D) float32 rows at a device address the library owns (a push halo buffer), for torch.as_tensor (no copy)"""

    def __init__(self, ptr: int, n: int, D: int):
        self.__cuda_array_interface__ = {"shape": (n, D), "typestr": "<f4", "data": (int(ptr), False), "strides": None,
                                         "version": 2}


class _Shard:
    def __init__(self, n_local, n_halo, recv_counts, num_edges, send_idx, send_counts, plan):
        self.n_local = int(n_local)
        self.n_halo = int(n_halo)
        self.recv_counts = [int(v) for v in recv_counts]
        self.send_idx = send_idx
        self.send_counts = send_counts
        self.plan = plan
        self.num_edges = int(num_edges)
        self.push = None           # per-(D, purpose) state of the peer-to-peer push path (_push_state)
        self.edge_route = None     # the edge-value exchange between the two shards (DistGraph._edge_route)


def rmat_chunks(num_nodes: int, num_edges: int, seed: int, device, chunk_edges: int = 1 << 26):
    """the counter-based RMAT list of gnnb_rmat_edges as (src, dst) int64 chunks (1-based ids) generated on `device`; the two buffers are
    reused, so a chunk is valid until the next one is requested"""
    dev = torch.device(device)
    cap = min(chunk_edges, max(num_edges, 1))
    s, t = (torch.empty(cap, dtype=torch.int64, device=dev) for _ in range(2))
    for first in range(0, num_edges, chunk_edges):
        cnt = min(chunk_edges, num_edges - first)
        with torch.cuda.device(dev):
            _lib.check(lib.gnnb_rmat_edges_range(num_nodes, first, cnt, seed, s.data_ptr(), t.data_ptr(), _stream(dev)))
        yield s[:cnt], t[:cnt]


class DistGraph:
    """A GNNGraph partitioned over the ranks of `group`.

    DistGraph(s, t, num_nodes, ...): every rank passes the same global COO (1-based s, t).
    DistGraph.from_chunks(chunks, num_nodes, ...): the same from an iterable of (s, t) chunks — the global list is never
    resident (CUDA only).  DistGraph.from_rmat(...) generates the chunks of the counter-based RMAT list on the device.
    On a CUDA device the shards are built by csrc/shard.cu (stable scan-compaction of every chunk, sort + unique of the
    remote ids, renaming, plan); on CPU tensors (gloo tests) by the torch restatement above.

    ownership = 'contiguous' (node ranges, cost-balanced unless `bounds` is given), 'cyclic' (0-based node v on rank
    v % world) or 'balanced' (nodes sorted by decreasing degree and dealt to the ranks in turn: edges, nodes and served
    halo rows all balanced whatever the id space looks like — RMAT probabilities are products over id bits, so neither
    ranges nor v % world balance it; needs `chunks` to be iterable twice).  `local_nodes()` lists the owned node ids in
    local-row order.

    Edge weights: `w` aligned with the global (s, t), or (s, t, w) chunks.  Each rank keeps the weights of its forward
    shard's edges (`w_fwd`) and of its backward shard's (`w_bwd`), in shard COO order with weight 1 for every appended
    self loop; both shards are stable compactions of the global order, so each is an ownership mask over the chunk
    (`owned_by_target`), and no weight crosses ranks."""

    def __init__(self, s: Optional[torch.Tensor], t: Optional[torch.Tensor], num_nodes: int, *, w=None,
                 add_self_loops: bool = False, group=None, device=None, bounds: Optional[List[int]] = None,
                 ownership: str = "contiguous", chunks=None, chunk_edges: int = 1 << 26):
        self.group = group
        self.world = dist.get_world_size(group)
        self.rank = dist.get_rank(group)
        self.timing = {}                                     # build phases, ms (this rank)
        self.device = torch.device(device) if device is not None else s.device
        self.num_nodes = int(num_nodes)
        self.ownership = ownership
        self.self_loops = add_self_loops
        self._c = None
        self._cw = None
        self._sage_cs = None
        self._weighted = None                                # decided by the first chunk unless `w` says it
        if chunks is None:
            s = s.to(self.device)
            t = t.to(self.device)
            if w is not None:
                w = torch.as_tensor(w, device=self.device).reshape(-1)
                if w.numel() != s.numel():
                    raise ValueError(f"DistGraph: {s.numel()} edges but {w.numel()} edge weights")
                self._weighted = True
            if ownership == "contiguous" and bounds is None:
                s0, t0 = s.to(torch.int64) - 1, t.to(torch.int64) - 1
                cost = (torch.bincount(t0, minlength=num_nodes) + torch.bincount(s0, minlength=num_nodes) + NODE_COST)
                bounds = balanced_bounds(cost, self.world)
                del s0, t0, cost
            E = int(s.numel())
            chunks = [(s[i:i + chunk_edges], t[i:i + chunk_edges]) + (() if w is None else (w[i:i + chunk_edges],))
                      for i in range(0, max(E, 1), chunk_edges)] if E else []
        elif w is not None:
            raise ValueError("DistGraph: with `chunks`, pass the weights as (s, t, w) chunks")
        self._order = self._relabel = None
        if ownership == "balanced":
            if not isinstance(chunks, (list, tuple)) and not callable(chunks):
                raise ValueError("ownership='balanced' needs the chunks twice: pass a list or a callable that returns an iterator")
            W, N = self.world, self.num_nodes
            it = chunks() if callable(chunks) else chunks
            t_own = time.perf_counter()
            if self.device.type == "cuda":                   # degree histogram + stable sort + deal, on the device
                cost = torch.zeros(N, dtype=torch.int32, device=self.device)
                self._relabel = torch.empty(N, dtype=torch.int32, device=self.device)
                order = torch.empty(N, dtype=torch.int32, device=self.device)
                with torch.cuda.device(self.device):
                    for sc, tc, *_ in it:
                        sc, tc = sc.to(self.device).contiguous(), tc.to(self.device).contiguous()
                        _lib.check(lib.gnnb_degree_accumulate(sc.data_ptr(), tc.data_ptr(), sc.numel(), sc.element_size(), 1, N,
                                                              cost.data_ptr(), _stream(self.device)))
                    _lib.check(lib.gnnb_balanced_relabel(cost.data_ptr(), N, W, self._relabel.data_ptr(), order.data_ptr(),
                                                         _stream(self.device)))
                self._order = order
                del cost
            else:                                            # the same deal in torch ops (gloo tests)
                by_degree = degree_order(it, N, self.device)
                pos = torch.arange(N, device=self.device)
                r, j = pos // W, pos % W
                o = torch.where((r % 2 == 1) & (r < N // W), W - 1 - j, j)
                self._relabel = torch.empty(N, dtype=torch.int32, device=self.device)
                self._relabel[by_degree] = (r * W + o).to(torch.int32)
                self._order = torch.empty(N, dtype=torch.int64, device=self.device)      # position -> node
                self._order[self._relabel.long()] = pos
                del by_degree, pos, r, j, o
            if self.device.type == "cuda":
                torch.cuda.synchronize(self.device)
            self.timing["ownership_ms"] = (time.perf_counter() - t_own) * 1e3
        if callable(chunks):
            chunks = chunks()
        self.first = ownership_first(self.num_nodes, self.world, ownership, bounds)
        self.bounds = self.first
        self.lo, self.hi = self.first[self.rank], self.first[self.rank + 1]
        self.n_local = self.hi - self.lo
        if self.device.type == "cuda":
            self.fwd, self.bwd = self._build_native(chunks)
            torch.cuda.synchronize(self.device)
        else:
            self.fwd, self.bwd = self._build_torch(chunks)
        # the edges of the global list whose target this rank owns: the forward shard without its self loops
        self.num_owned_edges = self.fwd.num_edges - (self.n_local if self.self_loops else 0)

    @classmethod
    def from_chunks(cls, chunks, num_nodes: int, **kw):
        """chunks: (s, t) or, with edge weights, (s, t, w) tuples — every chunk the one or every chunk the other"""
        return cls(None, None, num_nodes, chunks=chunks, **kw)

    # -- ownership of edges, and the weights each shard keeps
    def _owned(self, v: torch.Tensor) -> torch.Tensor:
        """True where this rank owns node v (1-based global ids): the builder's rule (to_pid with the relabel table)"""
        pid = to_pid(v.to(self.device).to(torch.int64) - 1, self.world, self.first, self.ownership, self._relabel)
        return (pid >= self.lo) & (pid < self.hi)

    def owned_by_target(self, t: torch.Tensor) -> torch.Tensor:
        """Mask over the edges of a global list or chunk (1-based targets t): True for the edges whose target this rank
        owns, i.e. its forward shard's edges in their shard order.  `edge_weight[dg.owned_by_target(t)]` is the per-rank
        `edge_weight` of dist_gcn_conv, and the same mask places its gradient back in the global list."""
        return self._owned(t)

    def _chunk_weights(self, sc: torch.Tensor, wc) -> Optional[torch.Tensor]:
        """the float32 weights of one (s, t[, w]) chunk on the device, or None; every chunk must agree on having them"""
        w = wc[0] if wc else None
        if self._weighted is None:
            self._weighted = w is not None
        if (w is not None) != self._weighted:
            raise ValueError("DistGraph: either every chunk carries edge weights or none does")
        if w is None:
            return None
        w = torch.as_tensor(w, device=self.device).reshape(-1)
        if w.numel() != sc.numel():
            raise ValueError(f"DistGraph: a chunk of {sc.numel()} edges carries {w.numel()} edge weights")
        return w.to(torch.float32)

    def _keep_weights(self, wf: List[torch.Tensor], wb: List[torch.Tensor]) -> None:
        """w_fwd / w_bwd from the masked chunk weights, weight 1 appended for every self loop (gcn_conv's rule)"""
        self.w_fwd = self.w_bwd = None
        if not self._weighted:
            return
        loops = [torch.ones(self.n_local, dtype=torch.float32, device=self.device)] if self.self_loops else []
        empty = [torch.zeros(0, dtype=torch.float32, device=self.device)]
        self.w_fwd = torch.cat(empty + wf + loops).contiguous()
        self.w_bwd = torch.cat(empty + wb + loops).contiguous()

    @classmethod
    def from_rmat(cls, num_nodes: int, num_edges: int, seed: int = 17, *, device, chunk_edges: int = 1 << 26, **kw):
        """the RMAT list of gnnb_rmat_edges, generated (identically on every rank) and consumed chunk by chunk"""
        dev = torch.device(device)
        return cls(None, None, num_nodes, chunks=lambda: rmat_chunks(num_nodes, num_edges, seed, dev, chunk_edges), device=dev, **kw)

    def local_nodes(self) -> torch.Tensor:
        """0-based global node id of every local row, in local-row order"""
        if self.ownership == "contiguous":
            return torch.arange(self.lo, self.hi, device=self.device)
        pos = self.rank + self.world * torch.arange(self.n_local, device=self.device)
        return pos if self._order is None else self._order[pos].long()

    # -- shard construction on the device (csrc/shard.cu)
    def _build_native(self, chunks):
        dev, world = self.device, self.world
        b = C.c_void_p()
        bounds_arr = (C.c_int64 * (world + 1))(*self.first) if self.ownership == "contiguous" else None
        shards, wf, wb = [], [], []
        t_sh = time.perf_counter()
        with torch.cuda.device(dev):
            st = _stream(dev)
            _lib.check(lib.gnnb_shard_builder_create(C.byref(b), self.num_nodes, world, self.rank,
                                                     0 if self.ownership == "contiguous" else 1, bounds_arr,
                                                     None if self._relabel is None else self._relabel.data_ptr()))
            try:
                for sc, tc, *wc in chunks:
                    sc, tc = sc.to(dev).contiguous(), tc.to(dev).contiguous()
                    assert sc.dtype == tc.dtype and sc.dtype in (torch.int32, torch.int64)
                    w = self._chunk_weights(sc, wc)
                    _lib.check(lib.gnnb_shard_builder_add(b, sc.data_ptr(), tc.data_ptr(), sc.numel(), sc.element_size(), 1, st))
                    if w is not None:                        # the builder keeps each shard's edges stably: same masks
                        wf.append(w[self._owned(tc)])
                        wb.append(w[self._owned(sc)])
                for direction in (0, 1):
                    h = C.c_void_p()
                    nl, nh, ne = C.c_int64(), C.c_int64(), C.c_int64()
                    rc = (C.c_int64 * world)()
                    _lib.check(lib.gnnb_shard_builder_finish(b, direction, int(self.self_loops), C.byref(h), C.byref(nl),
                                                             C.byref(nh), C.byref(ne), rc, st))
                    halo_local = torch.empty(max(nh.value, 1), dtype=torch.int32, device=dev)[:nh.value]
                    _lib.check(lib.gnnb_shard_builder_halo(b, direction, halo_local.data_ptr() if nh.value else None, st))
                    shards.append((h, nl.value, nh.value, ne.value, list(rc), halo_local))
            finally:
                lib.gnnb_shard_builder_destroy(b)
        self._keep_weights(wf, wb)
        torch.cuda.synchronize(dev)
        self.timing["shards_ms"] = (time.perf_counter() - t_sh) * 1e3
        t_ex = time.perf_counter()
        out = []
        for h, nl, nh, ne, rc, halo_local in shards:
            send_idx, send_counts = exchange_requests(halo_local, rc, self.group)
            out.append(_Shard(nl, nh, rc, ne, send_idx, send_counts, _Plan(h.value, dev)))
        torch.cuda.synchronize(dev)
        self.timing["request_exchange_ms"] = (time.perf_counter() - t_ex) * 1e3
        return out

    def _plans(self, d):
        """plan of a torch-built shard dict over [local | halo] sources (the gloo tests call this with the CPU test double
        installed)"""
        h = C.c_void_p()
        col, row = d["col"].to(torch.int32).contiguous(), d["row"].to(torch.int32).contiguous()
        with torch.cuda.device(self.device):
            _lib.check(lib.gnnb_graph_create(C.byref(h), col.data_ptr(), row.data_ptr(), row.numel(),
                                             d["n_local"] + int(d["halo"].numel()), d["n_local"], 4, 0, 1, _stream(self.device)))
        return _Plan(h.value, self.device)

    # -- the same in torch ops, for CPU tensors (host logic under gloo)
    def _build_torch(self, chunks):
        chunks = list(chunks)
        s0 = torch.cat([c[0] for c in chunks]).to(self.device).to(torch.int64) - 1 if chunks else torch.zeros(0, dtype=torch.int64)
        t0 = torch.cat([c[1] for c in chunks]).to(self.device).to(torch.int64) - 1 if chunks else torch.zeros(0, dtype=torch.int64)
        ps = to_pid(s0, self.world, self.first, self.ownership, self._relabel)
        pt = to_pid(t0, self.world, self.first, self.ownership, self._relabel)
        ws = [self._chunk_weights(c[0], c[2:]) for c in chunks]
        if self._weighted:
            w = torch.cat([torch.zeros(0, dtype=torch.float32, device=self.device)] + ws)
            self._keep_weights([w[self._owned(t0 + 1)]], [w[self._owned(s0 + 1)]])
        else:
            self._keep_weights([], [])
        out = []
        for key0, other0 in ((pt, ps), (ps, pt)):
            d = build_shard(key0, other0, self.lo, self.hi, self.first, self.self_loops)
            send_idx, send_counts = exchange_requests(d["halo_local"], d["recv_counts"], self.group)
            out.append(_Shard(d["n_local"], d["halo"].numel(), d["recv_counts"], d["row"].numel(), send_idx, send_counts,
                              None))
        return out

    # -- halo exchange: rows (n_local, D) -> halo rows (n_halo, D)
    def halo(self, shard: _Shard, x_rows: torch.Tensor) -> torch.Tensor:
        D = x_rows.shape[1]
        n_send = int(shard.send_idx.numel())
        send = torch.empty((n_send, D), dtype=x_rows.dtype, device=x_rows.device)
        if x_rows.is_cuda:
            with torch.cuda.device(self.device):
                _lib.check(lib.gnnb_gather_rows(shard.send_idx.data_ptr(), n_send, x_rows.data_ptr(), D,
                                                send.data_ptr(), _stream(self.device)))
        else:  # gloo/CPU test path for the host logic only
            send = x_rows[shard.send_idx.long()]
        recv = torch.empty((shard.n_halo, D), dtype=x_rows.dtype, device=x_rows.device)
        dist.all_to_all_single(recv, send, output_split_sizes=shard.recv_counts,
                               input_split_sizes=shard.send_counts, group=self.group)
        return recv

    # -- halo exchange, push path: one kernel writes the requested rows into every peer's halo buffer over NVLink
    def _push_state(self, shard: _Shard, D: int, purpose: str = "x"):
        """Peer-mapped double-buffered halo buffers for rows of D floats (built once per shard, D and purpose: two
        exchanges of one pass that are read by the same kernel — GAT's Wx and er rows, both H wide at C = 1 — must not
        share a buffer).  Every rank runs the same collectives whatever happens locally; if any rank fails to allocate /
        export / map, ALL ranks fall back to the NCCL exchange (returns None)."""
        if shard.push is None:
            shard.push = {}
        key = (D, purpose)
        if key in shard.push:
            return shard.push[key]
        dev, world, rank = self.device, self.world, self.rank
        ok = 1
        all_recv = [None] * world
        dist.all_gather_object(all_recv, list(shard.recv_counts), group=self.group)
        row0 = [int(sum(all_recv[q][:rank])) for q in range(world)]   # where my rows start in every peer's halo buffer
        # double buffer: pass k+1 never overwrites what a slower rank's pass k still reads.  GNNB_HALO_BUFFERS=1 is safe when
        # passes over a shard alternate with passes over the other one (one layer, forward / backward: the other pass's
        # completion collective orders them) and halves the memory — what config 5's 1 KB rows need
        nbuf = 1 if os.environ.get("GNNB_HALO_BUFFERS", "2") == "1" else 2
        bufs, handles = [], []
        try:
            with torch.cuda.device(dev):
                for _ in range(nbuf):
                    ptr = C.c_void_p()
                    _lib.check(lib.gnnb_dev_alloc(C.byref(ptr), max(shard.n_halo, 1) * D * 4))
                    h = (C.c_ubyte * 64)()
                    _lib.check(lib.gnnb_ipc_get_handle(ptr, h))
                    bufs.append(ptr.value)
                    handles.append(bytes(h))
        except Exception:
            ok = 0
            handles = [bytes(64)] * nbuf
        all_handles = [None] * world
        dist.all_gather_object(all_handles, handles, group=self.group)
        peer_ptrs = [[0] * world for _ in range(nbuf)]
        try:
            with torch.cuda.device(dev):
                for q in range(world):
                    if q == rank or shard.send_counts[q] == 0:
                        continue
                    for b in range(nbuf):
                        pp = C.c_void_p()
                        hb = (C.c_ubyte * 64).from_buffer_copy(all_handles[q][b])
                        _lib.check(lib.gnnb_ipc_open_handle(hb, C.byref(pp)))
                        peer_ptrs[b][q] = pp.value
        except Exception:
            ok = 0
        flag = torch.tensor([ok], device=dev, dtype=torch.int32)
        dist.all_reduce(flag, op=dist.ReduceOp.MIN, group=self.group)
        if int(flag.item()) == 0:                               # NCCL for everyone: give back what this rank did set up
            self._release_push({"bufs": bufs, "peer_ptrs": peer_ptrs})
            shard.push[key] = None
            return None
        seg = [0]
        for q in range(world):
            seg.append(seg[-1] + int(shard.send_counts[q]))
        st = {"bufs": bufs, "row0": (C.c_int64 * world)(*row0), "seg": (C.c_int64 * (world + 1))(*seg),
              "peer_c": [(C.c_void_p * world)(*[C.c_void_p(v) for v in peer_ptrs[b]]) for b in range(nbuf)], "turn": 0,
              "nbuf": nbuf,
              "peer_ptrs": peer_ptrs,
              "flag": torch.zeros(1, device=dev)}
        shard.push[key] = st
        return st

    def _release_push(self, st) -> None:
        with torch.cuda.device(self.device):
            for per_buf in st["peer_ptrs"]:
                for pp in per_buf:
                    if pp:
                        lib.gnnb_ipc_close_handle(C.c_void_p(pp))
            for ptr in st["bufs"]:
                if ptr:
                    lib.gnnb_dev_free(C.c_void_p(ptr))

    def close(self) -> None:
        """unmap the peers' halo buffers and free this rank's (call on every rank once no pass is in flight)"""
        for sh in (getattr(self, "fwd", None), getattr(self, "bwd", None)):
            if sh is None or not sh.push:
                continue
            if self.device.type == "cuda":
                torch.cuda.synchronize(self.device)
            for st in sh.push.values():
                if st is not None:
                    self._release_push(st)
            sh.push = None

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass

    def halo_ptr(self, shard: _Shard, x_rows: torch.Tensor, purpose: str = "x"):
        """(device pointer of this rank's halo rows for `x_rows`, owner).  `owner` is the all-to-all receive tensor (None on
        the push route, whose buffers the shard keeps): hold it until the kernel that reads the rows is enqueued, since a
        pass may make several exchanges.  A push buffer stays valid until the next-but-one call for this shard and
        purpose (the next one under GNNB_HALO_BUFFERS=1)."""
        if self.world == 1 or os.environ.get("GNNB_HALO", "push") != "push":
            t = self.halo(shard, x_rows)
            return t.data_ptr(), t
        D = x_rows.shape[1]
        st = self._push_state(shard, D, purpose)
        if st is None:                                          # some rank could not set up peer mapping: NCCL for everyone
            t = self.halo(shard, x_rows)
            return t.data_ptr(), t
        b = st["turn"]
        st["turn"] = (b + 1) % st["nbuf"]
        with torch.cuda.device(self.device):
            _lib.check(lib.gnnb_halo_push(shard.send_idx.data_ptr(), st["seg"], st["peer_c"][b], st["row0"], self.world,
                                          x_rows.data_ptr(), D, _stream(self.device)))
        dist.all_reduce(st["flag"], group=self.group)           # every rank's push kernel precedes its part of this collective
        return st["bufs"][b], None

    def halo_rows(self, shard: _Shard, x_rows: torch.Tensor, purpose: str) -> torch.Tensor:
        """the halo rows of `x_rows` as an (n_halo, D) tensor: the receive tensor, or a view of the push buffer (valid as
        halo_ptr's pointer is)"""
        ptr, t = self.halo_ptr(shard, x_rows, purpose)
        if t is not None:
            return t
        D = x_rows.shape[1]
        if shard.n_halo == 0:
            return torch.empty((0, D), dtype=x_rows.dtype, device=x_rows.device)
        return torch.as_tensor(_DeviceRows(ptr, shard.n_halo, D), device=self.device)

    # -- the edge-value exchange (GAT's dz): backward-shard COO order -> forward-shard COO order
    def _coo_owner(self, shard: _Shard) -> torch.Tensor:
        """owner rank of the gathered node of every edge of the shard plan, in the plan's COO order (local: this rank;
        halo: found from the halo segment bounds, which are grouped by owner in rank order)"""
        E, dev = shard.num_edges, self.device
        rowptr = torch.empty(shard.n_local + 1, dtype=torch.int32, device=dev)
        col = torch.empty(max(E, 1), dtype=torch.int32, device=dev)
        eid = torch.empty(max(E, 1), dtype=torch.int32, device=dev)
        with torch.cuda.device(dev):
            _lib.check(lib.gnnb_graph_csr_device(shard.plan.h, 0, rowptr.data_ptr(), col.data_ptr(), eid.data_ptr(),
                                                 _stream(dev)))
        coo_col = torch.empty(E, dtype=torch.int64, device=dev)
        coo_col[eid[:E].long()] = col[:E].long()
        ends = torch.cumsum(torch.tensor(shard.recv_counts, dtype=torch.int64, device=dev), 0)
        halo_owner = torch.searchsorted(ends, coo_col - shard.n_local, right=True)
        return torch.where(coo_col < shard.n_local, torch.full_like(coo_col, self.rank), halo_owner)

    def _edge_route(self):
        """Built once.  Both shards are stable compactions of the same edge sequence with the self loops appended after the
        originals, so the edges of rank p's forward shard whose source rank q owns and the edges of rank q's backward
        shard whose target rank p owns are the same edges in the same order.  Send side: the backward shard's edges
        grouped by target owner (stable); receive side: the forward shard's COO position of every received row.  The
        pairwise counts are checked once."""
        if self.fwd.edge_route is None:
            W, dev = self.world, self.device
            own_b, own_f = self._coo_owner(self.bwd), self._coo_owner(self.fwd)
            send_perm = torch.sort(own_b, stable=True).indices
            recv_perm = torch.sort(own_f, stable=True).indices
            unpack = torch.empty_like(recv_perm)
            unpack[recv_perm] = torch.arange(recv_perm.numel(), device=dev)
            send_counts = torch.bincount(own_b, minlength=W)
            recv_counts = torch.bincount(own_f, minlength=W)
            peer_counts = torch.empty_like(send_counts)
            dist.all_to_all_single(peer_counts, send_counts, group=self.group)
            if not torch.equal(peer_counts, recv_counts):
                raise RuntimeError(f"rank {self.rank}: the edge exchange does not pair up: the peers' backward shards send "
                                   f"{peer_counts.tolist()} edge rows, the forward shard expects {recv_counts.tolist()}")
            unpack_b = torch.empty_like(send_perm)                 # the reverse route: backward-shard position of
            unpack_b[send_perm] = torch.arange(send_perm.numel(), device=dev)   # every row received from a target's owner
            self.fwd.edge_route = {"send_idx": send_perm.to(torch.int32), "unpack_idx": unpack.to(torch.int32),
                                   "send_counts": send_counts.tolist(), "recv_counts": recv_counts.tolist(),
                                   # one rank: pack, exchange and unpack compose into one gather
                                   "direct_idx": send_perm[unpack].to(torch.int32) if W == 1 else None,
                                   "rev_send_idx": recv_perm.to(torch.int32), "rev_unpack_idx": unpack_b.to(torch.int32),
                                   "rev_direct_idx": recv_perm[unpack_b].to(torch.int32) if W == 1 else None}
        return self.fwd.edge_route

    def edge_exchange(self, v_bwd: torch.Tensor) -> torch.Tensor:
        """(E_bwd, H) values in backward-shard COO order -> (E_fwd, H) in forward-shard COO order, every edge's row moved
        to the rank that owns its target: one pack, one all-to-all, one unpack"""
        r = self._edge_route()
        return self._move_edge_rows(v_bwd, r["send_idx"], r["send_counts"], r["recv_counts"], r["unpack_idx"], r["direct_idx"])

    def edge_exchange_reverse(self, v_fwd: torch.Tensor) -> torch.Tensor:
        """(E_fwd, H) values in forward-shard COO order -> (E_bwd, H) in backward-shard COO order, every edge's row moved
        to the rank that owns its source: edge_exchange run backwards over the same route"""
        r = self._edge_route()
        return self._move_edge_rows(v_fwd, r["rev_send_idx"], r["recv_counts"], r["send_counts"], r["rev_unpack_idx"],
                                    r["rev_direct_idx"])

    def _move_edge_rows(self, v, send_idx, send_counts, recv_counts, unpack_idx, direct_idx) -> torch.Tensor:
        H, dev = v.shape[1], self.device
        v = v.contiguous()
        n_send, n_recv = int(send_idx.numel()), int(unpack_idx.numel())
        if direct_idx is not None:
            out = torch.empty((n_recv, H), dtype=v.dtype, device=dev)
            if n_recv:
                with torch.cuda.device(dev):
                    _lib.check(lib.gnnb_gather_rows(direct_idx.data_ptr(), n_recv, v.data_ptr(), H, out.data_ptr(),
                                                    _stream(dev)))
            return out
        send = torch.empty((n_send, H), dtype=v.dtype, device=dev)
        recv = torch.empty((n_recv, H), dtype=v.dtype, device=dev)
        out = torch.empty((n_recv, H), dtype=v.dtype, device=dev)
        with torch.cuda.device(dev):
            if n_send:
                _lib.check(lib.gnnb_gather_rows(send_idx.data_ptr(), n_send, v.data_ptr(), H, send.data_ptr(),
                                                _stream(dev)))
            dist.all_to_all_single(recv, send, output_split_sizes=recv_counts, input_split_sizes=send_counts,
                                   group=self.group)
            if n_recv:
                _lib.check(lib.gnnb_gather_rows(unpack_idx.data_ptr(), n_recv, recv.data_ptr(), H, out.data_ptr(),
                                                _stream(dev)))
        return out

    def sage_cs(self):
        """1 / in-degree of the targets over the backward shard's [local | halo] space (0 for a node without in-edges, which
        no edge gathers): the scale of the mean aggregation's pullback.  Computed once."""
        if self._sage_cs is None:
            deg = torch.empty(self.n_local, dtype=torch.float32, device=self.device)
            with torch.cuda.device(self.device):
                if self.n_local:
                    _lib.check(lib.gnnb_degree(self.fwd.plan.h, _lib.DIR_IN, None, _ptr(deg), _stream(self.device)))
            inv = torch.where(deg > 0, 1.0 / deg, torch.zeros_like(deg))
            self._sage_cs = torch.cat([inv, self.halo(self.bwd, inv.reshape(-1, 1)).reshape(-1)]).contiguous()
        return self._sage_cs

    def gcn_c(self):
        """c = 1/sqrt(in-degree) of the owned nodes (exact: rowptr differences of the forward shard), plus the
        halo copies the two shards need.  Computed once."""
        if self._c is None:
            p = self.fwd.plan
            c = torch.empty(self.n_local, dtype=torch.float32, device=self.device)
            with torch.cuda.device(self.device):
                _lib.check(lib.gnnb_gcn_norm(p.h, None, c.data_ptr(), _stream(self.device)))
            cf = torch.cat([c, self.halo(self.fwd, c.reshape(-1, 1)).reshape(-1)])
            cb = torch.cat([c, self.halo(self.bwd, c.reshape(-1, 1)).reshape(-1)])
            self._c = (c, cf.contiguous(), cb.contiguous())
        return self._c

    def gcn_scales(self, w_fwd: torch.Tensor):
        """(d, c, cf, cb) of the weighted normalisation: d = weighted in-degree of the owned nodes from the forward shard's
        weights `w_fwd` (gnnb_degree, local), c = 1/sqrt(d) as gcn_conv's default norm_fn, and c's halo copies on both
        shards"""
        from .layers import default_norm_fn
        d = torch.empty(self.n_local, dtype=torch.float32, device=self.device)
        with torch.cuda.device(self.device):
            if self.n_local:
                _lib.check(lib.gnnb_degree(self.fwd.plan.h, _lib.DIR_IN, _ptr(w_fwd), _ptr(d), _stream(self.device)))
        c = default_norm_fn(d)
        cf = torch.cat([c, self.halo(self.fwd, c.reshape(-1, 1)).reshape(-1)])
        cb = torch.cat([c, self.halo(self.bwd, c.reshape(-1, 1)).reshape(-1)])
        return d, c, cf.contiguous(), cb.contiguous()

    def gcn_c_weighted(self):
        """gcn_scales of the graph's own weights (w_fwd), computed once"""
        if self._cw is None:
            self._cw = self.gcn_scales(self.w_fwd)
        return self._cw

    def _column_sliced(self, f, *cols) -> Optional[torch.Tensor]:
        """f(*cols) one block of `D / GNNB_HALO_SLICES` feature columns at a time, or None when the pass is not sliced.
        Column-sliced passes exchange and reduce a slice at a time, so that the halo buffers shrink by the slice count
        (config 5: 62 GB of halo rows per pass at D = 256 do not fit beside the features); they cost strided copies of
        the local rows and re-read the index arrays once per slice.  Every aggregation is column-wise, so the slices are
        independent."""
        slices = int(os.environ.get("GNNB_HALO_SLICES", "1"))
        if slices <= 1 or cols[0].shape[1] % slices or getattr(self, "_slicing", False):
            return None
        k = cols[0].shape[1] // slices
        out = torch.empty_like(cols[0])
        self._slicing = True
        try:
            for i in range(slices):
                out[:, i * k:(i + 1) * k] = f(*(c[:, i * k:(i + 1) * k].contiguous() for c in cols))
        finally:
            self._slicing = False
        return out

    def propagate(self, shard: _Shard, x_rows: torch.Tensor, cs, ct, aggr=_lib.SUM, w=None) -> torch.Tensor:
        """one pass over `shard`: copy_xj, or w_mul_xj with the shard's edge weights `w` (COO order)"""
        out = self._column_sliced(lambda xs: self.propagate(shard, xs, cs, ct, aggr, w), x_rows)
        if out is not None:
            return out
        D = x_rows.shape[1]
        hptr, recv = self.halo_ptr(shard, x_rows)
        out = torch.empty_like(x_rows)
        with torch.cuda.device(self.device):
            _lib.check(lib.gnnb_propagate_halo(shard.plan.h, _lib.COPY_XJ if w is None else _lib.W_MUL_XJ, aggr,
                                               x_rows.data_ptr(), hptr if shard.n_halo else None, shard.n_local, _ptr(w),
                                               _ptr(cs), _ptr(ct), D, out.data_ptr(), _stream(self.device)))
        del recv                                                # the kernel that reads it is enqueued
        return out

    def maxmin_pullback(self, dout: torch.Tensor, x_rows: torch.Tensor, out: torch.Tensor, aggr, w=None) -> torch.Tensor:
        """dx of the owned rows for max / min aggregation over the forward shard (out its result), by the backward shard:
        the halo rows of dout and of out are pulled (two purposes: one kernel reads both), then
        gnnb_propagate_maxmin_bwd_halo with the backward shard's edge weights `w` (COO order) or none"""
        dx = self._column_sliced(lambda d, x, o: self.maxmin_pullback(d, x, o, aggr, w), dout, x_rows, out)
        if dx is not None:
            return dx
        sh, D = self.bwd, x_rows.shape[1]
        d_ptr, d_recv = self.halo_ptr(sh, dout, "maxmin_dout")
        o_ptr, o_recv = self.halo_ptr(sh, out, "maxmin_out")
        dx = torch.empty_like(x_rows)
        with torch.cuda.device(self.device):
            _lib.check(lib.gnnb_propagate_maxmin_bwd_halo(sh.plan.h, _lib.COPY_XJ if w is None else _lib.W_MUL_XJ, aggr,
                                                          _ptr(x_rows), _ptr(dout), d_ptr if sh.n_halo else None,
                                                          _ptr(out), o_ptr if sh.n_halo else None, sh.n_local, _ptr(w),
                                                          D, _ptr(dx), _stream(self.device)))
        del d_recv, o_recv                                      # the kernel that reads them is enqueued
        return dx


class _DistGCNPropagateFn(torch.autograd.Function):
    @staticmethod
    def forward(ctx, x_rows, dg: DistGraph):
        c, cf, cb = dg.gcn_c()
        ctx.dg = dg
        return dg.propagate(dg.fwd, x_rows.contiguous(), cf, c)

    @staticmethod
    def backward(ctx, dout):
        dg = ctx.dg
        c, cf, cb = dg.gcn_c()
        return dg.propagate(dg.bwd, dout.contiguous(), cb, c), None


class _DistGCNWeightedFn(torch.autograd.Function):
    """y = c .* propagate(w_mul_xj, c .* h) on the forward shard, c = 1/sqrt(weighted in-degree), for the graph's weights
    (w None) or an explicit per-rank edge_weight (w: one value per original forward-shard edge).

    Pullback for h: the same pass on the backward shard with w_bwd (the graph's, or w moved there by
    edge_exchange_reverse).  Pullback for w, when it requires grad: the forward keeps the unscaled sums u (y = u .* c)
    and the backward the unscaled pullback sums dhs (dh = dhs .* c), as the single-GPU composition does; then
        dc = <dy, u> + <dhs, h>  per owned node (its target and its source role),  dd = dc through c = 1/sqrt(d),
        dw_e = <c_t dy_t, c_s h_s> + dd_t                                  (gnnb_gcn_edge_weight_grad_halo)
    over the forward shard, whose halo rows of h are exchanged again here rather than kept from the forward."""

    @staticmethod
    def forward(ctx, h_rows, w, dg: DistGraph):
        h_rows = h_rows.contiguous()
        if w is None:
            w_f = dg.w_fwd
            d, c, cf, cb = dg.gcn_c_weighted()
        else:
            w_f = w.to(dg.device, torch.float32).contiguous()
            if dg.self_loops:                                   # weight 1 for every appended loop (gcn_conv's rule)
                w_f = torch.cat([w_f, torch.ones(dg.n_local, dtype=torch.float32, device=dg.device)])
            d, c, cf, cb = dg.gcn_scales(w_f)
        ctx.dg, ctx.explicit, ctx.w_f, ctx.c, ctx.cb = dg, w is not None, w_f, c, cb
        ctx.want_w = w is not None and ctx.needs_input_grad[1]
        u = dg.propagate(dg.fwd, h_rows, cf, None, w=w_f)      # c_t applied outside, as gcn_conv: 0 * Inf = NaN for a
        if ctx.want_w:                                          # target without in-edges and d = 0
            ctx.h, ctx.u, ctx.d, ctx.cf = h_rows, u, d, cf
        return u * c[:, None]

    @staticmethod
    def backward(ctx, dy):
        dg, c, cb = ctx.dg, ctx.c, ctx.cb
        dy = dy.contiguous()
        w_b = dg.edge_exchange_reverse(ctx.w_f.reshape(-1, 1)).reshape(-1) if ctx.explicit else dg.w_bwd
        dhs = dg.propagate(dg.bwd, dy, cb, None, w=w_b)
        if not ctx.want_w:
            return dhs * c[:, None], None, None
        from .layers import default_norm_fn
        h, D = ctx.h, ctx.h.shape[1]
        dc = (dy * ctx.u).sum(1) + (dhs * h).sum(1)
        with torch.enable_grad():
            d = ctx.d.detach().requires_grad_(True)
            dd, = torch.autograd.grad(default_norm_fn(d), d, dc)
        h_halo = dg.halo_rows(dg.fwd, h, "x")
        dw = torch.empty(dg.fwd.num_edges, dtype=torch.float32, device=dg.device)
        with torch.cuda.device(dg.device):
            _lib.check(lib.gnnb_gcn_edge_weight_grad_halo(dg.fwd.plan.h, _ptr(dy), _ptr(h), _ptr(h_halo) if dg.fwd.n_halo else None,
                                                          dg.n_local, _ptr(ctx.cf), _ptr(c), _ptr(dd.contiguous()), D, _ptr(dw),
                                                          _stream(dg.device)))
        del h_halo                                              # the kernel that reads it is enqueued
        return dhs * c[:, None], dw[:dg.num_owned_edges], None  # the loops' weights are constants


def dist_gcn_conv(l, dg: DistGraph, x_local: torch.Tensor, edge_weight: Optional[torch.Tensor] = None) -> torch.Tensor:
    """gcn_conv (GNNlib/src/layers/conv.jl:14-72) on the rows this rank owns; x_local is Julia-shaped (Din, n_local).
    The graph must have been partitioned with add_self_loops = l.add_self_loops.  Weight gradients are per-rank
    partial sums: all-reduce them like any data-parallel layer.

    Edge weights follow the reference's rule: an explicit `edge_weight` is used (l.use_edge_weight is then ignored);
    otherwise the graph's weights when l.use_edge_weight is true and `dg` has them; otherwise the unweighted
    normalisation.  `edge_weight` is this rank's: one value per edge whose target it owns, in global order
    (`w[dg.owned_by_target(t)]` of a global list), and may require grad; its gradient comes back in the same order."""
    assert dg.self_loops == bool(l.add_self_loops)
    from .layers import _gcn_dense
    if edge_weight is not None:
        if edge_weight.numel() != dg.num_owned_edges:
            raise ValueError(f"Wrong number of edge weights (expected {dg.num_owned_edges}, the edges whose target rank "
                             f"{dg.rank} owns, but given {edge_weight.numel()})")
        w = edge_weight.reshape(-1)
    elif getattr(l, "use_edge_weight", False) and dg.w_fwd is not None:
        w = None
    else:
        return _gcn_dense(l, l.weight, x_local, lambda h: unrows(_DistGCNPropagateFn.apply(rows(h), dg)))
    return _gcn_dense(l, l.weight, x_local, lambda h: unrows(_DistGCNWeightedFn.apply(rows(h), w, dg)))


# ---------------------------------------------------------------------------------------------------------
# GATConv on shards: the fused attention kernels' HALO instances and the dz exchange
# ---------------------------------------------------------------------------------------------------------
def dist_gat_aggregate(dg: DistGraph, Wx: torch.Tensor, el: torch.Tensor, er: torch.Tensor, slope: float):
    """gnnb_gat_aggregate on this rank's targets: Wx (n_local, H, C) and er (n_local, H) of the owned nodes, el (n_local, H).
    One exchange of the Wx rows and one of the er rows on the forward shard, then the HALO kernel.  Returns (out, seg_max,
    seg_sum)."""
    N, H, Cc = Wx.shape
    sh, dev = dg.fwd, dg.device
    wx_ptr, wx_recv = dg.halo_ptr(sh, Wx.reshape(N, H * Cc), "gat_wx")
    er_all = torch.cat([er, dg.halo_rows(sh, er, "gat_er")]).contiguous()
    out = torch.empty_like(Wx)
    smax, ssum = torch.empty_like(el), torch.empty_like(el)
    with torch.cuda.device(dev):
        _lib.check(lib.gnnb_gat_aggregate_halo(sh.plan.h, _ptr(Wx), wx_ptr if sh.n_halo else None, N, _ptr(el), _ptr(er_all),
                                               Cc, H, slope, _ptr(out), _ptr(smax), _ptr(ssum), _stream(dev)))
    del wx_recv                                                  # the kernel that reads it is enqueued
    return out, smax, ssum


def dist_gat_aggregate_bwd(dg: DistGraph, Wx, el, er, smax, ssum, out, dout, slope: float):
    """gnnb_gat_aggregate_bwd on this rank's rows: T of the owned targets; one exchange of the packed [el | seg_max |
    seg_sum | T] rows and one of the dout rows on the backward shard; the HALO pullback kernel on the backward shard (dWx
    and der of the owned sources, dz of their out-edges); dz moved to the targets' owners (edge_exchange) and summed per
    target there.  Returns (dWx, del, der)."""
    N, H, Cc = Wx.shape
    sh, dev = dg.bwd, dg.device
    st = _stream(dev)
    T = torch.empty_like(el)
    with torch.cuda.device(dev):
        _lib.check(lib.gnnb_gat_tnode(_ptr(dout), _ptr(out), N, Cc, H, _ptr(T), st))
    packed = torch.cat([el, smax, ssum, T], dim=1)               # (n_local, 4H): one exchange for the four per-target terms
    full = torch.cat([packed, dg.halo_rows(sh, packed, "gat_stats")])
    el_a, smax_a, ssum_a, T_a = (full[:, k * H:(k + 1) * H].contiguous() for k in range(4))
    d_ptr, d_recv = dg.halo_ptr(sh, dout.reshape(N, H * Cc), "gat_dout")
    dWx, der = torch.empty_like(Wx), torch.empty_like(er)
    dz = torch.empty((sh.num_edges, H), dtype=torch.float32, device=dev)
    with torch.cuda.device(dev):
        _lib.check(lib.gnnb_gat_aggregate_bwd_halo(sh.plan.h, _ptr(Wx), _ptr(er), _ptr(dout), d_ptr if sh.n_halo else None, N,
                                                   _ptr(el_a), _ptr(smax_a), _ptr(ssum_a), _ptr(T_a), Cc, H, slope, _ptr(dWx),
                                                   _ptr(der), _ptr(dz), st))
    del d_recv
    dz_f = dg.edge_exchange(dz)                                  # del[h,i] = Σ_{k ∈ N(i)} dz_k, where i is owned
    del_ = torch.empty_like(el)
    with torch.cuda.device(dev):
        if dz_f.shape[0]:
            _lib.check(lib.gnnb_scatter(dg.fwd.plan.h, _lib.DST, _lib.SUM, _ptr(dz_f), H, _ptr(del_), st))
        else:
            del_.zero_()
    return dWx, del_, der


def dist_gat_conv(l, dg: DistGraph, x_local: torch.Tensor) -> torch.Tensor:
    """gat_conv (GNNlib/src/layers/conv.jl:112-150) on the rows this rank owns; x_local is Julia-shaped (Din, n_local).
    The graph must have been partitioned with add_self_loops = l.add_self_loops; no dropout, no edge features and a shape
    of the fused kernels (gat_fusable).  Weight gradients (dense_x, a, bias) are per-rank partial sums: all-reduce them."""
    from .layers import _attention_tail, _gat_edge_part, _jl_reshape3, gat_fusable
    _, chout = l.channel
    heads = l.heads
    if dg.self_loops != bool(l.add_self_loops):
        raise ValueError(f"dist_gat_conv: the graph was partitioned with add_self_loops={dg.self_loops}, the layer has "
                         f"add_self_loops={bool(l.add_self_loops)}")
    if getattr(l, "dense_e", None) is not None:
        raise ValueError("dist_gat_conv: edge features are not supported on a partitioned graph")
    if float(getattr(l, "dropout", 0.0) or 0.0) != 0.0:
        raise ValueError("dist_gat_conv: attention dropout is not supported on a partitioned graph")
    if not gat_fusable(chout, heads):
        raise ValueError(f"dist_gat_conv: {chout} channels x {heads} heads is not a shape of the fused GAT kernels "
                         "(C/4 a power of two <= 32, or C a power of two <= 32 with C*H <= 128)")
    Wx = _jl_reshape3(l.dense_x(x_local), chout, heads)         # (C, H, n_local)
    return _attention_tail(l, _gat_edge_part(l, Wx, None, dg, dist_gat_aggregate, dist_gat_aggregate_bwd))


# ---------------------------------------------------------------------------------------------------------
# message passing on shards: propagate(copy_xj | w_mul_xj, g, +|mean|max|min), and the layers built on it
# ---------------------------------------------------------------------------------------------------------
class _DistPropagateFn(torch.autograd.Function):
    """propagate(copy_xj | w_mul_xj, g, aggr) on the owned rows: gnnb_propagate_halo over the forward shard.  w: None
    (copy_xj), the graph's own dg.w_fwd, or explicit weights of every forward-shard edge (loops included).

    Pullback for x: + and mean run gnnb_propagate_halo over the backward shard (mean: each target's row scaled by
    1 / in-degree, sage_cs); max and min pull the halo rows of dout and of the forward result over the backward shard and
    run gnnb_propagate_maxmin_bwd_halo.  The backward shard's weights are dg.w_bwd for the graph's, or the explicit ones
    moved there by edge_exchange_reverse.  Pullback for explicit weights (+ and mean only): dw_e = <dout_t, x_s> ct[t]
    by gnnb_gcn_edge_weight_grad_halo over the forward shard (ct = 1 / in-degree for mean), whose halo rows of x are
    exchanged again here rather than kept from the forward.  The edge-weight gradient of max / min is refused by
    dist_propagate before any exchange.

    Tensors are kept with save_for_backward: the forward result kept as a ctx attribute would form the cycle
    out -> grad_fn -> ctx -> out, which only the cyclic collector frees."""

    @staticmethod
    def forward(ctx, x_rows, w, dg: DistGraph, aggr):
        ismax = aggr in (_lib.MAX, _lib.MIN)
        ctx.want_w = w is not None and ctx.needs_input_grad[1]
        x_rows = x_rows.contiguous()
        out = dg.propagate(dg.fwd, x_rows, None, None, aggr, w=w)
        ctx.dg, ctx.aggr = dg, aggr
        ctx.graph_w = w is not None and w is dg.w_fwd           # the backward shard keeps the graph's own weights
        ctx.save_for_backward(x_rows if (ismax or ctx.want_w) else None, out if ismax else None,
                              None if ctx.graph_w else w)
        return out

    @staticmethod
    def backward(ctx, dout):
        dg, aggr = ctx.dg, ctx.aggr
        x, out, w = ctx.saved_tensors
        dout = dout.contiguous()
        w_b = dg.w_bwd if ctx.graph_w else None
        if w is not None:
            w_b = dg.edge_exchange_reverse(w.detach().reshape(-1, 1)).reshape(-1)
        if aggr in (_lib.MAX, _lib.MIN):
            return dg.maxmin_pullback(dout, x, out, aggr, w_b), None, None, None
        cs = dg.sage_cs() if aggr == _lib.MEAN else None        # mean: each target's row scaled by 1 / in-degree
        dx = dg.propagate(dg.bwd, dout, cs, None, _lib.SUM, w=w_b)
        if not ctx.want_w:
            return dx, None, None, None
        D = x.shape[1]
        ct = dg.sage_cs()[:dg.n_local].contiguous() if aggr == _lib.MEAN else None
        x_halo = dg.halo_rows(dg.fwd, x, "x")
        dw = torch.empty(dg.fwd.num_edges, dtype=torch.float32, device=dg.device)
        with torch.cuda.device(dg.device):
            _lib.check(lib.gnnb_gcn_edge_weight_grad_halo(dg.fwd.plan.h, _ptr(dout), _ptr(x), _ptr(x_halo) if dg.fwd.n_halo else None,
                                                          dg.n_local, None, _ptr(ct), None, D, _ptr(dw), _stream(dg.device)))
        del x_halo                                              # the kernel that reads it is enqueued
        return dx, dw, None, None


def dist_propagate(f, dg: DistGraph, aggr, x_local: torch.Tensor, edge_weight: Optional[torch.Tensor] = None) -> torch.Tensor:
    """propagate(f, g, aggr; xj = x) (GNNlib/src/msgpass.jl:71-79) on the rows this rank owns, over the graph as
    partitioned (its self loops included); x_local and the result are Julia-shaped (D, n_local).  Differentiable in
    x_local and, for + and mean, in edge_weight.

    f is copy_xj or w_mul_xj; aggr +, mean, max or min.  w_mul_xj multiplies each message by the explicit `edge_weight`
    when given (this rank's: one value per edge whose target it owns, in global order, `w[dg.owned_by_target(t)]` of a
    global list; each self loop of the partition gets weight 1), otherwise by the graph's own weights, otherwise by
    nothing (copy_xj), as the single-GPU w_mul_xj.  The edge-weight gradient of max / min is not implemented (nor is
    it on one GPU): a weight that requires grad is refused there."""
    from .msgpass import _aggr_code, copy_xj, w_mul_xj
    if f is not copy_xj and f is not w_mul_xj:
        raise ValueError(f"dist_propagate: message function {getattr(f, '__name__', f)!r} is not supported on a "
                         "partitioned graph (copy_xj and w_mul_xj are)")
    code = _aggr_code(aggr)
    w = None
    if edge_weight is not None:
        if f is not w_mul_xj:
            raise ValueError("dist_propagate: copy_xj takes no edge weights (w_mul_xj does)")
        if edge_weight.numel() != dg.num_owned_edges:
            raise ValueError(f"Wrong number of edge weights (expected {dg.num_owned_edges}, the edges whose target rank "
                             f"{dg.rank} owns, but given {edge_weight.numel()})")
        w = edge_weight.reshape(-1).to(dg.device, torch.float32).contiguous()
        if dg.self_loops:
            w = torch.cat([w, torch.ones(dg.n_local, dtype=torch.float32, device=dg.device)])
    elif f is w_mul_xj:
        w = dg.w_fwd
    if (code in (_lib.MAX, _lib.MIN) and w is not None and w.requires_grad and torch.is_grad_enabled()):
        raise ValueError("dist_propagate: the edge-weight gradient of max / min aggregation is not implemented")
    return unrows(_DistPropagateFn.apply(rows(x_local), w, dg, code))


def _no_loops(dg: DistGraph, name: str) -> None:
    if dg.self_loops:
        raise ValueError(f"{name}: the graph was partitioned with add_self_loops=True; the layer adds no self loops")


def dist_graph_conv(l, dg: DistGraph, x_local: torch.Tensor) -> torch.Tensor:
    """graph_conv (GNNlib/src/layers/conv.jl:102-108), σ.(W1·x .+ W2·propagate(copy_xj, g, aggr, x) .+ b), on the rows
    this rank owns, for every aggregation; x_local is Julia-shaped (Din, n_local).  The graph must have been partitioned
    without self loops.  Weight gradients are per-rank partial sums: all-reduce them."""
    from .layers import _graph_conv_dense
    from .msgpass import copy_xj
    _no_loops(dg, "dist_graph_conv")
    return _graph_conv_dense(l, x_local, dist_propagate(copy_xj, dg, l.aggr, x_local))


def dist_gin_conv(l, dg: DistGraph, x_local: torch.Tensor) -> torch.Tensor:
    """gin_conv (GNNlib/src/layers/conv.jl:250-256), nn((1 + ϵ)·x .+ propagate(copy_xj, g, aggr, x)), on the rows this
    rank owns; x_local is Julia-shaped (Din, n_local).  The graph must have been partitioned without self loops.
    Gradients of nn's parameters are per-rank partial sums: all-reduce them."""
    from .layers import _gin_dense
    from .msgpass import copy_xj
    _no_loops(dg, "dist_gin_conv")
    return _gin_dense(l, x_local, dist_propagate(copy_xj, dg, l.aggr, x_local))


def dist_sage_conv(l, dg: DistGraph, x_local: torch.Tensor) -> torch.Tensor:
    """sage_conv (GNNlib/src/layers/conv.jl:277-283) on the rows this rank owns, for aggr ∈ {mean, +}; x_local is
    Julia-shaped (Din, n_local).  The graph must have been partitioned without self loops (the layer adds none).  Weight
    gradients are per-rank partial sums: all-reduce them."""
    from .layers import _sage_linear
    from .msgpass import _aggr_code
    aggr = _aggr_code(l.aggr)
    if aggr not in (_lib.SUM, _lib.MEAN):
        raise ValueError(f"dist_sage_conv: aggregation {l.aggr!r} is not supported on a partitioned graph (mean and + are)")
    if dg.self_loops:
        raise ValueError("dist_sage_conv: the graph was partitioned with add_self_loops=True; SAGEConv adds no self loops")
    r1 = rows(x_local).contiguous()
    return _sage_linear(l, r1, _DistPropagateFn.apply(r1, None, dg, aggr))


# ---------------------------------------------------------------------------------------------------------
# bench.py --gpus N>1
# ---------------------------------------------------------------------------------------------------------
def bench_multi(args, world, rank, dev, seed, ClockSampler, measured_peaks, cpu_leg=None, parity=None):
    import gnnb200 as gnn
    n, E, D = args.nodes, args.edges, args.dim
    # NCCL opens its peer-to-peer connections lazily, on the first all-to-all (seconds at 8 ranks): communicator set-up is
    # not shard construction, so it is paid (and reported) before the plan timer starts
    torch.cuda.synchronize()
    tc0 = time.perf_counter()
    warm = torch.zeros(world * 4, device=dev)
    warm_out = torch.empty_like(warm)
    dist.all_to_all_single(warm_out, warm)
    dist.all_reduce(warm)
    dist.all_gather([torch.empty_like(warm) for _ in range(world)], warm)
    torch.cuda.synchronize()
    dist.barrier()
    t_comm = time.perf_counter() - tc0
    del warm, warm_out
    t0 = time.perf_counter()
    # every rank generates the counter-based edge list chunk by chunk and keeps its shard (csrc/shard.cu); 'balanced'
    # ownership deals the nodes to the ranks by decreasing degree (one extra pass over the generated chunks)
    ownership = os.environ.get("GNNB_OWNERSHIP", "balanced")
    dg = DistGraph.from_rmat(n, E, seed, device=dev, add_self_loops=True, ownership=ownership,
                             chunk_edges=int(os.environ.get("GNNB_CHUNK_EDGES", str(1 << 26))))
    torch.cuda.synchronize()
    dg.timing["constructor_total_ms"] = (time.perf_counter() - t0) * 1e3
    tg0 = time.perf_counter()
    dg.gcn_c()
    torch.cuda.synchronize()
    dg.timing["gcn_norm_and_its_halo_ms"] = (time.perf_counter() - tg0) * 1e3
    t_plan = time.perf_counter() - t0
    torch.cuda.empty_cache()

    torch.manual_seed(0)
    layer = gnn.GCNConv(D, D, torch.relu, device=dev)   # same seed => same weights on every rank
    gen = torch.Generator(device=dev).manual_seed(1234 + rank)
    x = gnn.unrows(torch.randn(dg.n_local, D, device=dev, generator=gen)).requires_grad_(True)
    dy = gnn.unrows(torch.randn(dg.n_local, D, device=dev, generator=gen))

    def step():
        x.grad = None
        layer.weight.grad = None
        layer.bias.grad = None
        y = dist_gcn_conv(layer, dg, x)
        y.backward(dy)
        dist.all_reduce(layer.weight.grad)
        dist.all_reduce(layer.bias.grad)

    for _ in range(args.warmup):
        step()
    torch.cuda.synchronize()
    dist.barrier()
    l0 = gnn.launch_count()
    ev0, ev1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    with ClockSampler(dev.index) as clocks:
        torch.cuda.synchronize()
        dist.barrier()
        ev0.record()
        for _ in range(args.steps):
            step()
        ev1.record()
        torch.cuda.synchronize()
        dist.barrier()
    ms = torch.tensor([ev0.elapsed_time(ev1) / args.steps], device=dev)
    dist.all_reduce(ms, op=dist.ReduceOp.MAX)
    ms = float(ms)
    launches = gnn.launch_count() - l0

    # the fused kernel alone on this rank's forward shard (CUDA events on the launch stream), max over ranks
    c, cf, cb = dg.gcn_c()
    xr = gnn.rows(x.detach())
    x.grad = None
    layer.weight.grad = None
    torch.cuda.empty_cache()
    hp, hp_recv = dg.halo_ptr(dg.fwd, xr)               # the halo rows where the step's own exchange puts them
    out = torch.empty_like(xr)
    st = torch.cuda.current_stream(dev).cuda_stream

    def kern():
        _lib.check(lib.gnnb_propagate_halo(dg.fwd.plan.h, _lib.COPY_XJ, _lib.SUM, xr.data_ptr(), hp if dg.fwd.n_halo else None,
                                           dg.n_local, None, cf.data_ptr(), c.data_ptr(), D, out.data_ptr(), st))

    for _ in range(3):
        kern()
    evs = [(torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)) for _ in range(args.steps)]
    torch.cuda.synchronize()
    for a, b in evs:
        a.record(); kern(); b.record()
    torch.cuda.synchronize()
    kms = sum(a.elapsed_time(b) for a, b in evs) / len(evs)
    # halo exchange alone
    for _ in range(2):
        dg.halo_ptr(dg.fwd, xr)
    torch.cuda.synchronize(); dist.barrier()
    ev0.record()
    for _ in range(args.steps):
        dg.halo_ptr(dg.fwd, xr)
    ev1.record()
    torch.cuda.synchronize()
    hms = ev0.elapsed_time(ev1) / args.steps
    Es = dg.fwd.num_edges
    alg = Es * (4 * D + 4) + 4 * (dg.n_local + 1) + 4 * D * dg.n_local
    stats = torch.tensor([kms, hms, float(Es), float(dg.n_local), float(dg.fwd.n_halo), float(dg.bwd.n_halo), alg / (kms * 1e-3) / 1e9],
                         device=dev, dtype=torch.float64)
    allst = [torch.empty_like(stats) for _ in range(world)]
    dist.all_gather(allst, stats)
    allst = torch.stack(allst).cpu()
    peak, peak_src = measured_peaks()

    e2e = None
    if not args.no_e2e:
        xh = torch.empty(dg.n_local, D, pin_memory=True).normal_()
        dyh = torch.empty(dg.n_local, D, pin_memory=True).normal_()
        yh = torch.empty(dg.n_local, D, pin_memory=True)
        dxh = torch.empty(dg.n_local, D, pin_memory=True)

        s_in, s_out = torch.cuda.Stream(dev), torch.cuda.Stream(dev)
        main = torch.cuda.current_stream(dev)

        def step_host():
            # uploads on s_in, downloads on s_out (PCIe is full duplex), compute on the main stream
            with torch.cuda.stream(s_in):
                xd_raw = xh.to(dev, non_blocking=True)
                ev_x = torch.cuda.Event(); ev_x.record(s_in)
                dyd_raw = dyh.to(dev, non_blocking=True)
                ev_dy = torch.cuda.Event(); ev_dy.record(s_in)
            main.wait_event(ev_x)
            xd = gnn.unrows(xd_raw).requires_grad_(True)
            layer.weight.grad = None
            layer.bias.grad = None
            y = dist_gcn_conv(layer, dg, xd)
            s_out.wait_stream(main)
            with torch.cuda.stream(s_out):
                yh.copy_(gnn.rows(y.detach()), non_blocking=True)
            main.wait_event(ev_dy)
            y.backward(gnn.unrows(dyd_raw))
            s_out.wait_stream(main)
            with torch.cuda.stream(s_out):
                dxh.copy_(gnn.rows(xd.grad), non_blocking=True)
            dist.all_reduce(layer.weight.grad)
            wg = layer.weight.grad.cpu()
            main.wait_stream(s_out)
            xd_raw.record_stream(main); dyd_raw.record_stream(main)
            return wg

        ke = max(2, min(args.steps, 5))
        step_host()
        torch.cuda.synchronize(); dist.barrier()
        ev0.record()
        for _ in range(ke):
            step_host()
        ev1.record()
        torch.cuda.synchronize()
        ems = torch.tensor([ev0.elapsed_time(ev1) / ke], device=dev)
        dist.all_reduce(ems, op=dist.ReduceOp.MAX)
        ems = float(ems)
        e2e = {"value": E / (ems * 1e-3), "unit": "edges/s", "ms_per_step": ems, "steps": ke,
               "h2d_bytes_per_step": 2 * 4 * n * D, "d2h_bytes_per_step": 2 * 4 * n * D + 4 * D * D * world,
               "api": "gnnb200.partition.dist_gcn_conv on pinned host slices (all ranks; bytes are whole-job)"}

    par = None
    if parity is not None:                                   # all ranks: the checker runs collectives
        del x, dy, xr, out
        layer.weight.grad = None
        torch.cuda.empty_cache()
        par = parity(dg, layer)
    cpu = None
    if rank == 0 and cpu_leg is not None:
        cpu = cpu_leg()                                      # the oracle port on the bounded sample, host cores of rank 0
    if rank == 0:
        worst = int(torch.argmax(allst[:, 0]))
        line = {
            "metric": "edges/sec fwd+bwd GCNConv 128-dim on 100M-edge graph" if D == 128 else f"edges/sec fwd+bwd GCNConv {D}-dim (RMAT N={n} E={E})",
            "value": E / (ms * 1e-3), "unit": "edges/s", "n_gpus": world, "steps": args.steps, "warmup": args.warmup, "ms_per_step": ms, "higher_is_better": True,
            "scaling": "strong", "vs_baseline": None, "dtype": "f32", "data": "synthetic",
            "config": {"workload": f"GCNConv {D}->{D} (add_self_loops, relu, bias) fwd+bwd on RMAT N={n} E={E} seed {seed} "
                                   f"(BASELINE configs[{1 if D == 128 else 4}]), node-partitioned over {world} GPUs, halo exchange over NVLink",
                       "parallelism": f"node-partition x{world}, {ownership} ownership, shards built on the device from generated chunks",
                       "halo_exchange": os.environ.get("GNNB_HALO", "push") + (" (one kernel writes rows into peer halo buffers over NVLink, CUDA IPC)" if os.environ.get("GNNB_HALO", "push") == "push" else " (pack kernel + NCCL all_to_all_single)"),
                       "l2": "per-GPU features and halo buffers are far larger than the 50 MB L2",
                       "plan_build_ms": t_plan * 1e3, "plan_build_phases_ms_rank0": {k: round(v, 1) for k, v in dg.timing.items()},
                       "nccl_connection_setup_ms": t_comm * 1e3, "chunk_edges": 128,
                       "per_rank": {"kernel_ms": allst[:, 0].tolist(), "halo_exchange_ms": allst[:, 1].tolist(),
                                    "shard_edges": allst[:, 2].tolist(), "n_local": allst[:, 3].tolist(),
                                    "halo_rows_fwd": allst[:, 4].tolist(), "halo_rows_bwd": allst[:, 5].tolist()}},
            "clocks": clocks.summary(), "e2e": e2e, "gpu_launches": launches,
            "roofline": {"bound": "hbm", "achieved": float(allst[worst, 6]), "peak": peak, "unit": "GB/s",
                         "frac": float(allst[worst, 6]) / peak, "traffic": None,
                         "kernel": "gnnb::seg_lean_kernel (sum, per-edge scale stream, halo base) over [local|halo] rows (slowest rank)",
                         "peak_source": peak_src,
                         "halo": {"bytes_received_slowest_rank": float(allst[:, 4].max()) * D * 4,
                                  "ms": float(allst[:, 1].max()),
                                  "GBps_per_gpu": float(allst[:, 4].max()) * D * 4 / (float(allst[:, 1].max()) * 1e-3) / 1e9,
                                  "nvlink_peak_GBps": 450.0,
                                  "nvlink_peak_source": "H100 SXM data sheet (900 GB/s NVLink, both directions), not a measurement"}},
            "cpu_baseline": cpu, "parity_rel_err": par,
        }
        print(json.dumps(line), flush=True)
    dist.barrier()
    dist.destroy_process_group()
