"""GNNGraph — the COO graph value of the reference (GNNGraphs/src/gnngraph.jl:108-117) plus the handful of
GNNGraphs functions that sit on the hot path (SURVEY.md §8 a9-a11, a17):

    edge_index          GNNGraphs/src/query.jl:12-14
    degree              GNNGraphs/src/query.jl:314-369
    add_self_loops      GNNGraphs/src/transform.jl:12-28
    set_edge_weight     GNNGraphs/src/transform.jl:568-577
    batch (COO)         GNNGraphs/src/transform.jl:682-709
    graph_indicator     GNNGraphs/src/query.jl:500-512
    GNNGraph(g; ndata, edata, gdata)                     GNNGraphs/src/gnngraph.jl:187-210
    node_features / edge_features / graph_features      GNNGraphs/src/query.jl:516-544

Conventions follow the reference: node ids are 1-based Int64 (or Int32) vectors ``s`` (source) and ``t``
(target); feature arrays are Julia-shaped ``(D, num_nodes)`` / ``(K, num_edges)`` whose *memory* is
column-major (``colmajor`` below), i.e. every node owns D contiguous floats — exactly what a ``CuArray``
handed through ``ccall`` looks like to libgnnb200.

Each graph lazily owns one device *plan* (``gnnb_graph_t``: CSR by target, CSR by source on demand) that is
built once and cached — the reference rebuilds its CSC from COO on every fused call
(GNNGraphs/src/query.jl:227).
"""
from __future__ import annotations

import ctypes as C
from typing import Optional, Sequence

import numpy as np
import torch

from . import _lib
from ._lib import lib


# --------------------------------------------------------------------------------------------------
# Julia-layout helpers
# --------------------------------------------------------------------------------------------------
def colmajor(x: torch.Tensor) -> torch.Tensor:
    """Return ``x`` (any strides) as a tensor of the same shape whose memory is column-major (Julia)."""
    nd = x.dim()
    if nd <= 1:
        return x.contiguous()
    rev = tuple(range(nd - 1, -1, -1))
    return x.permute(rev).contiguous().permute(rev)


def jl_zeros(*shape, dtype=torch.float32, device=None) -> torch.Tensor:
    rev = tuple(reversed(shape))
    return torch.zeros(rev, dtype=dtype, device=device).permute(tuple(range(len(shape) - 1, -1, -1)))


def jl_randn(*shape, dtype=torch.float32, device=None, generator=None) -> torch.Tensor:
    rev = tuple(reversed(shape))
    return torch.randn(rev, dtype=dtype, device=device, generator=generator).permute(
        tuple(range(len(shape) - 1, -1, -1)))


def rows(x: torch.Tensor) -> torch.Tensor:
    """(d1,...,dk, N) Julia array -> C-contiguous (N, dk,...,d1) view (copy only if x is not column-major)."""
    nd = x.dim()
    rev = tuple(range(nd - 1, -1, -1))
    r = x.permute(rev)
    return r if r.is_contiguous() else r.contiguous()


def unrows(r: torch.Tensor) -> torch.Tensor:
    """inverse of rows(): C-contiguous (N, dk,...,d1) -> Julia-shaped (d1,...,dk,N) column-major view."""
    nd = r.dim()
    return r.permute(tuple(range(nd - 1, -1, -1)))


def _compute_device(t: torch.Tensor) -> torch.device:
    """where the library computes for data that lives with `t`: t's GPU, else the current CUDA device (host arrays are
    staged there; there is no CPU path)."""
    if t.is_cuda:
        return t.device
    return torch.device("cuda", torch.cuda.current_device() if torch.cuda.is_available() else 0)


def _stream(device) -> int:
    return int(torch.cuda.current_stream(device).cuda_stream)


def _ptr(t: Optional[torch.Tensor]) -> Optional[int]:
    return None if t is None else t.data_ptr()


class _Plan:
    """Owner of one gnnb_graph_t."""

    def __init__(self, handle: int, device: torch.device):
        self.h = C.c_void_p(handle)
        self.device = device

    def __del__(self):
        try:
            if self.h:
                lib.gnnb_graph_destroy(self.h)
                self.h = None
        except Exception:
            pass


def _as_index(v, device=None) -> torch.Tensor:
    if isinstance(v, torch.Tensor):
        t = v
    else:
        t = torch.as_tensor(np.asarray(v))
    if t.dtype not in (torch.int64, torch.int32):
        if t.is_floating_point() or t.dtype == torch.bool:
            raise ValueError("edge indices must be integers")
        t = t.to(torch.int64)
    if device is not None:
        t = t.to(device)
    return t.contiguous()


# caches a graph keeps that depend on its topology alone (never on its features): a copy with replaced data shares them
_TOPOLOGY_CACHES = ("_plan", "_gi_plan_n", "_gi_plan_e", "_lmax_cache", "_gcn_c_cache", "_cheb_op_cache", "_dconv_gt")
_KEEP = object()


def _graphdata(d, default_name: str, n: int, what: str) -> dict:
    """normalize_graphdata (GNNGraphs/src/datastore.jl): None -> empty, a bare tensor -> {default_name: it}; every array's
    last dimension must be n"""
    d = {} if d is None else ({default_name: d} if isinstance(d, torch.Tensor) else dict(d))
    for k, v in d.items():
        assert v.shape[-1] == n, f"{k} has last dimension {v.shape[-1]}; the graph has {what} = {n}"
    return d


class GNNGraph:
    """COO graph ``(s, t[, w])`` with 1-based node ids — GNNGraph{<:COO_T} (GNNGraphs/src/gnngraph.jl:108-117).

    ``GNNGraph(s, t)``, ``GNNGraph((s, t))``, ``GNNGraph((s, t, w))`` and ``GNNGraph(adjacency_matrix)`` are
    accepted (gnngraph.jl:120-199); ``num_nodes`` defaults to ``max(maximum(s), maximum(t))``
    (convert.jl:33-36).  Indices are validated once, on the device, when the plan is built
    (``1 <= idx <= num_nodes``, convert.jl:49-54 -> AssertionError).

    ``GNNGraph(g, ndata=..., edata=..., gdata=...)`` (gnngraph.jl:187-210) is ``g`` with the given stores replaced (the
    others kept): a bare tensor is named ``x`` / ``e`` / ``u`` and its last dimension must be num_nodes / num_edges /
    num_graphs.  The copy shares ``g``'s topology and the caches built from it alone (the plan, the graph-indicator
    plans, λmax), and no cache that holds features.
    """

    def __init__(self, s, t=None, w=None, *, num_nodes: Optional[int] = None, ndata=_KEEP, edata=_KEEP,
                 gdata=_KEEP, num_graphs: int = 1, graph_indicator=None, device=None):
        if isinstance(s, GNNGraph):
            assert t is None and w is None and num_nodes is None and device is None, \
                "GNNGraph(g; ndata, edata, gdata) takes the graph and the data stores only"
            self._copy(s, ndata, edata, gdata)
            return
        ndata, edata, gdata = (None if d is _KEEP else d for d in (ndata, edata, gdata))
        if t is None:
            as_edges = isinstance(s, tuple) and len(s) in (2, 3)           # (s, t) / (s, t, w): tuples
            if not as_edges and isinstance(s, list) and len(s) in (2, 3) and all(hasattr(v, "__len__") for v in s):
                # a nested list is an adjacency matrix when it is square ([[0,1],[1,0]]), a list of index vectors otherwise
                as_edges = not all(len(v) == len(s) for v in s)
            if as_edges:
                if len(s) == 3:
                    s, t, w = s
                else:
                    s, t = s
            else:  # adjacency matrix: A[i,j] != 0 <=> edge i -> j  (convert.jl:75-95, column-major findnz order)
                A = s if isinstance(s, torch.Tensor) else torch.as_tensor(np.asarray(s))
                if A.dim() != 2 or A.shape[0] != A.shape[1]:
                    raise ValueError("adjacency matrix must be square")
                nz = (A.t() != 0).nonzero()  # iterate columns first, like Julia's findnz on a dense matrix
                t, s = nz[:, 0] + 1, nz[:, 1] + 1
                if num_nodes is None:
                    num_nodes = A.shape[0]
                w = A.t()[A.t() != 0].to(torch.float32)        # v = A[nz] always travels as the edge weight (convert.jl:85)
        self.s = _as_index(s, device)
        self.t = _as_index(t, device)
        assert self.s.dim() == 1 and self.s.shape == self.t.shape, "s and t must be vectors of equal length"
        self.num_edges = int(self.s.numel())
        if num_nodes is None:
            num_nodes = int(max(int(self.s.max()), int(self.t.max()))) if self.num_edges else 0
        self.num_nodes = int(num_nodes)
        self.w = None if w is None else torch.as_tensor(w, dtype=torch.float32).to(self.s.device).contiguous()
        if self.w is not None:
            assert self.w.numel() == self.num_edges, "edge weight length must equal num_edges"  # convert.jl:47
        self.num_graphs = int(num_graphs)
        self.graph_indicator = graph_indicator
        self.ndata = dict(ndata or {}) if not isinstance(ndata, torch.Tensor) else {"x": ndata}
        self.edata = dict(edata or {}) if not isinstance(edata, torch.Tensor) else {"e": edata}
        self.gdata = dict(gdata or {}) if not isinstance(gdata, torch.Tensor) else {"u": gdata}
        for k, v in self.ndata.items():
            assert v.shape[-1] == self.num_nodes, f"ndata[{k}] last dim must be num_nodes"
        for k, v in self.edata.items():
            assert v.shape[-1] == self.num_edges, f"edata[{k}] last dim must be num_edges"
        self._plan: Optional[_Plan] = None
        self._loops: Optional["GNNGraph"] = None

    def _copy(self, g: "GNNGraph", ndata, edata, gdata) -> None:
        self.s, self.t, self.w = g.s, g.t, g.w
        self.num_edges, self.num_nodes, self.num_graphs = g.num_edges, g.num_nodes, g.num_graphs
        self.graph_indicator = g.graph_indicator
        self.ndata = _graphdata(g.ndata if ndata is _KEEP else ndata, "x", g.num_nodes, "num_nodes")
        self.edata = _graphdata(g.edata if edata is _KEEP else edata, "e", g.num_edges, "num_edges")
        self.gdata = _graphdata(g.gdata if gdata is _KEEP else gdata, "u", g.num_graphs, "num_graphs")
        self._plan = None
        self._loops = None                 # add_self_loops' result carries the features: never shared
        for k in _TOPOLOGY_CACHES:
            v = getattr(g, k, None)
            if v is not None:
                setattr(self, k, v)

    # -- conveniences mirroring g.x / g.e property access (datastore.jl getproperty)
    @property
    def x(self):
        return self.ndata["x"]

    @property
    def e(self):
        return self.edata["e"]

    @property
    def device(self) -> torch.device:
        return self.s.device

    def to(self, device) -> "GNNGraph":
        device = torch.device(device)
        g = GNNGraph(self.s.to(device), self.t.to(device), None if self.w is None else self.w.to(device),
                     num_nodes=self.num_nodes,
                     ndata={k: v.to(device) for k, v in self.ndata.items()},
                     edata={k: v.to(device) for k, v in self.edata.items()},
                     gdata={k: v.to(device) for k, v in self.gdata.items()},
                     num_graphs=self.num_graphs,
                     graph_indicator=None if self.graph_indicator is None else self.graph_indicator.to(device))
        return g

    def cuda(self) -> "GNNGraph":
        return self.to("cuda")

    def __repr__(self):
        return f"GNNGraph(num_nodes={self.num_nodes}, num_edges={self.num_edges}, num_graphs={self.num_graphs})"

    # -- the device plan ---------------------------------------------------------------------------
    def plan(self, device: Optional[torch.device] = None) -> _Plan:
        """Build (once) and return the device plan.  Raises AssertionError on out-of-range indices."""
        if self._plan is not None:
            return self._plan
        self._plan = _make_plan(self.s, self.t, self.num_edges, self.num_nodes, self.num_nodes, device)
        return self._plan


def _make_plan(s: torch.Tensor, t: torch.Tensor, num_edges: int, num_src: int, num_dst: int,
               device: Optional[torch.device] = None) -> _Plan:
    """gnnb_graph_create over 1-based (s, t): sources in [1, num_src], targets in [1, num_dst] (AssertionError
    otherwise)."""
    if device is None:
        device = _compute_device(s)
    if _lib.device_count() <= 0:
        raise _lib.GNNBError(_lib.ECUDA, "no CUDA device: the message-passing engine has no CPU fallback")
    h = C.c_void_p()
    on_dev = 1 if s.is_cuda else 0
    with torch.cuda.device(device):
        _lib.check(lib.gnnb_graph_create(C.byref(h), s.data_ptr(), t.data_ptr(), num_edges, num_src, num_dst,
                                         s.element_size(), 1, on_dev, _stream(device)))
    return _Plan(h.value, device)


def _is_hetero(g) -> bool:
    return getattr(g, "is_hetero", False)


def relation(g):
    """The one relation message passing runs over: the graph itself for a GNNGraph, the only edge type's relation
    (``s``, ``t``, ``w``, ``num_edges``, ``plan()``) for a one-relation GNNHeteroGraph (AssertionError otherwise)."""
    if _is_hetero(g):
        return g.only_relation()
    return g


def num_src_dst(g) -> tuple:
    """(num_src, num_dst) of that relation: (num_nodes, num_nodes) for a GNNGraph; the node counts of the source and
    target types for a one-relation GNNHeteroGraph.  Every array message passing makes is sized by these two."""
    if _is_hetero(g):
        r = g.only_relation()
        return r.num_src, r.num_dst
    return g.num_nodes, g.num_nodes


def homogeneous_only(g, name: str) -> None:
    """The reference types these layers for GNNGraph only: a heterograph is a TypeError naming the layer."""
    if _is_hetero(g):
        raise TypeError(f"{name} needs a GNNGraph; it has no method for a GNNHeteroGraph (use a relation-wise layer "
                        f"inside HeteroGraphConv)")


# --------------------------------------------------------------------------------------------------
# queries / transforms on the hot path
# --------------------------------------------------------------------------------------------------
def edge_index(g: GNNGraph, *args):
    """(s, t) — GNNGraphs/src/query.jl:12 (heterographs: edge_index(g[, edge_t]), gnnheterograph/query.jl:9-10)."""
    if _is_hetero(g):
        from .hetero import edge_index as f
        return f(g, *args)
    return g.s, g.t


def get_edge_weight(g: GNNGraph, *args):
    if _is_hetero(g):
        from .hetero import get_edge_weight as f
        return f(g, *args)
    return g.w


def set_edge_weight(g: GNNGraph, w: torch.Tensor) -> GNNGraph:
    """GNNGraphs/src/transform.jl:568-577."""
    assert w.numel() == g.num_edges
    h = GNNGraph(g.s, g.t, w, num_nodes=g.num_nodes, ndata=g.ndata, edata=g.edata, gdata=g.gdata,
                 num_graphs=g.num_graphs, graph_indicator=g.graph_indicator)
    h._plan = g._plan  # same topology: share the plan
    return h


def add_self_loops(g: GNNGraph, *args) -> GNNGraph:
    """s=[s;1:n], t=[t;1:n], weights padded with 1 — GNNGraphs/src/transform.jl:12-28.

    Requires empty edata (the reference asserts it).  The result (and its plan, derived on the device from
    this graph's CSR without a new sort) is cached on ``g``: graphs are immutable values.  Heterographs:
    add_self_loops(g[, edge_t]) (gnnheterograph/transform.jl:20-76)."""
    if _is_hetero(g):
        from .hetero import add_self_loops as f
        return f(g, *args)
    assert len(g.edata) == 0, "add_self_loops requires empty edata"  # transform.jl:14
    if g._loops is not None:
        return g._loops
    n = g.num_nodes
    nodes = torch.arange(1, n + 1, dtype=g.s.dtype, device=g.s.device)
    s = torch.cat([g.s, nodes])
    t = torch.cat([g.t, nodes])
    w = None if g.w is None else torch.cat([g.w, torch.ones(n, dtype=g.w.dtype, device=g.w.device)])
    h = GNNGraph(s, t, w, num_nodes=n, ndata=g.ndata, edata=g.edata, gdata=g.gdata, num_graphs=g.num_graphs,
                 graph_indicator=g.graph_indicator)
    if _lib.device_count() > 0:
        p = g.plan()
        hh = C.c_void_p()
        with torch.cuda.device(p.device):
            _lib.check(lib.gnnb_graph_add_self_loops(p.h, C.byref(hh), _stream(p.device)))
        h._plan = _Plan(hh.value, p.device)
    g._loops = h
    return h


class _WeightedDegreeFn(torch.autograd.Function):
    """Weighted degree as NNlib.scatter(+, w, idx) (GNNGraphs/src/query.jl:359-369), with scatter's pullback:
    dw = Δ[t] for dir=:in, Δ[s] for :out, and the sum of the two for :both."""

    @staticmethod
    def forward(ctx, w, plan, d, n_nodes):
        out = torch.empty(n_nodes, dtype=torch.float32, device=plan.device)
        with torch.cuda.device(plan.device):
            _lib.check(lib.gnnb_degree(plan.h, d, w.data_ptr(), out.data_ptr(), _stream(plan.device)))
        ctx.plan, ctx.d, ctx.n_edges = plan, d, w.numel()
        return out

    @staticmethod
    def backward(ctx, dout):
        plan = ctx.plan
        dout = dout.to(torch.float32).contiguous()
        which = {_lib.DIR_IN: (_lib.DST,), _lib.DIR_OUT: (_lib.SRC,), _lib.DIR_BOTH: (_lib.DST, _lib.SRC)}[ctx.d]
        dw = None
        with torch.cuda.device(plan.device):
            for k in which:
                part = torch.empty(ctx.n_edges, dtype=torch.float32, device=dout.device)
                _lib.check(lib.gnnb_gather(plan.h, k, dout.data_ptr(), 1, part.data_ptr(), _stream(plan.device)))
                dw = part if dw is None else dw + part
        return dw, None, None, None


def degree(g: GNNGraph, T=None, *args, dir: str = "out", edge_weight=True) -> torch.Tensor:
    """degree(g, T; dir, edge_weight) — GNNGraphs/src/query.jl:314-331,355-369 (note the reference default dir=:out).

    edge_weight: True -> the graph's own weights if any, False/None -> counts, tensor -> those weights.  With weights
    that require grad the result is differentiable in them (the reference's weighted degree is a scatter(+)).
    Heterographs: degree(g, edge_t, T=None; dir) (gnnheterograph/query.jl:55-68)."""
    if _is_hetero(g):
        if edge_weight is not True:
            raise TypeError("degree(g::GNNHeteroGraph, edge_t, T; dir) takes no edge_weight (its degrees are unweighted)")
        from .hetero import degree as f
        return f(g, T, *args, dir=dir)
    if args:
        raise TypeError(f"degree(g::GNNGraph, T; dir, edge_weight) takes one positional argument after g, got {1 + len(args)}")
    assert dir in ("in", "out", "both")  # query.jl:339
    if isinstance(edge_weight, torch.Tensor):
        w = edge_weight
    elif edge_weight is True:
        w = g.w
    else:
        w = None
    p = g.plan()
    if w is not None:
        assert w.numel() == g.num_edges
        w = w.to(device=p.device, dtype=torch.float32).contiguous()
    d = {"out": _lib.DIR_OUT, "in": _lib.DIR_IN, "both": _lib.DIR_BOTH}[dir]
    if w is not None and w.requires_grad and torch.is_grad_enabled():
        out = _WeightedDegreeFn.apply(w, p, d, g.num_nodes)
    else:
        out = torch.empty(g.num_nodes, dtype=torch.float32, device=p.device)
        with torch.cuda.device(p.device):
            _lib.check(lib.gnnb_degree(p.h, d, _ptr(w), out.data_ptr(), _stream(p.device)))
    if T is None:
        T = torch.float32 if w is not None else g.s.dtype
    return out.to(T)


def _only(store: dict, name: str):
    if not store:
        return None
    if len(store) > 1:
        raise ValueError(f"multiple feature arrays ({', '.join(store)}): access them through g.{name}")
    return next(iter(store.values()))


def node_features(g: GNNGraph):
    """GNNGraphs/src/query.jl:516-524: None when ndata is empty, its only array otherwise (ValueError for several)."""
    return _only(g.ndata, "ndata")


def edge_features(g: GNNGraph):
    """GNNGraphs/src/query.jl:526-534."""
    return _only(g.edata, "edata")


def graph_features(g: GNNGraph):
    """GNNGraphs/src/query.jl:536-544."""
    return _only(g.gdata, "gdata")


def graph_indicator(g: GNNGraph, edges=False) -> torch.Tensor:
    """GNNGraphs/src/query.jl:500-512 (heterographs: graph_indicator(g[, node_t]), gnnheterograph/query.jl:81-98)."""
    if _is_hetero(g):
        from .hetero import graph_indicator as f
        return f(g) if edges is False else f(g, edges)
    gi = g.graph_indicator
    if gi is None:
        gi = torch.ones(g.num_nodes, dtype=torch.int64, device=g.s.device)
    if edges:
        gi = gi[g.s.long() - 1]
    return gi


def batch(graphs: Sequence[GNNGraph]) -> GNNGraph:
    """Block-diagonal batching of COO graphs — GNNGraphs/src/transform.jl:682-709: node ids are offset by the
    cumulative node counts, graph_indicator by the cumulative graph counts; edges stay grouped per graph."""
    graphs = list(graphs)
    assert len(graphs) > 0
    if _is_hetero(graphs[0]):
        from .hetero import batch as f
        return f(graphs)
    dev = graphs[0].s.device
    nodesum = np.cumsum([0] + [g.num_nodes for g in graphs])
    graphsum = np.cumsum([0] + [g.num_graphs for g in graphs])
    s = torch.cat([g.s + int(nodesum[i]) for i, g in enumerate(graphs)])
    t = torch.cat([g.t + int(nodesum[i]) for i, g in enumerate(graphs)])
    ws = [g.w for g in graphs]
    w = None if any(x is None for x in ws) else torch.cat(ws)
    gi = torch.cat([graph_indicator(g) + int(graphsum[i]) for i, g in enumerate(graphs)]).to(dev)

    def cat(ds):
        keys = ds[0].keys()
        return {k: torch.cat([colmajor(d[k]) for d in ds], dim=-1) for k in keys}

    return GNNGraph(s, t, w, num_nodes=int(nodesum[-1]), ndata=cat([g.ndata for g in graphs]),
                    edata=cat([g.edata for g in graphs]), num_graphs=int(graphsum[-1]), graph_indicator=gi)


def rmat_graph(num_nodes: int, num_edges: int, seed: int = 17, device="cuda") -> GNNGraph:
    """Synthetic RMAT graph (ours — the reference has no RMAT generator; SURVEY.md §8d): Graph500 parameters,
    counter-based splitmix64, generated on the device; bit-identical to oracle.orc_rmat."""
    device = torch.device(device)
    s = torch.empty(num_edges, dtype=torch.int64, device=device)
    t = torch.empty(num_edges, dtype=torch.int64, device=device)
    with torch.cuda.device(device):
        _lib.check(lib.gnnb_rmat_edges(num_nodes, num_edges, seed, s.data_ptr(), t.data_ptr(), _stream(device)))
    return GNNGraph(s, t, num_nodes=num_nodes)
