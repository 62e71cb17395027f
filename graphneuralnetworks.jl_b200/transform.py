"""Edge-list transforms either side of the hot path, on the device (SURVEY.md §8f rank 3):

    sort_edge_index(u, v)            GNNGraphs/src/utils.jl:41-45   (the reference's CUDA extension round-trips through
                                     the host: GNNGraphs/ext/GNNGraphsCUDAExt.jl:24-30)
    remove_self_loops(g)             GNNGraphs/src/transform.jl:49-64
    remove_multi_edges(g; aggr=+)    GNNGraphs/src/transform.jl:157-190
    to_bidirected(g)                 GNNGraphs/src/transform.jl:495-510
    unbatch(g)                       GNNGraphs/src/transform.jl:741-778
    csr(g; transposed)               the plan's COO -> CSR conversion as an API (the reference has no CSR type)
    remove_edges(g, edges_or_p)      GNNGraphs/src/transform.jl:121-147   (DropEdge)
    remove_nodes(g, nodes_or_p)      GNNGraphs/src/transform.jl:212-276   (DropNode)
    getgraph(g, i; nmap)             GNNGraphs/src/transform.jl:825-888
    add_nodes(g, n; ndata)           GNNGraphs/src/transform.jl:553-563
    random_walk_pe(g, walk_length)   GNNGraphs/src/transform.jl:975-990   (per-graph walks, csrc/rwpe.cu)
    color_refinement(g, x0)          GNNGraphs/src/utils.jl:340-389       (1-WL colour refinement, csrc/wl.cu)
    ppr_diffusion(g; alpha)          GNNGraphs/src/transform.jl:1026-1051 (per-graph inverses, csrc/ppr.cu)

The index work (pair encoding, stable radix sort, duplicate runs) is csrc/transform.cu; the feature aggregation of
`remove_multi_edges` is the library's segmented scatter over the run ids it returns — the same kernels as
`aggregate_neighbors`.  Graphs given on the CPU are staged to the current CUDA device and the result lives there.

The four graph-editing functions share one entry, `gnnb_graph_subgraph` (csrc/plan.cu): kept nodes are renumbered in
ascending old id, which is monotone, and the plan's sort is stable, so a compaction of the parent's sorted arrays is
the child's plan — no new sort.  When g's plan exists and g has at most _DERIVE_MAX_EDGES edges, the child gets that
derived plan; otherwise the child stays lazy and its plan is a fresh sort when first needed (building the parent's plan
only to derive from it costs more than that sort, and above that size the derivation's gathers miss L2 and lose to the
sort).  Both routes give the same bits.
Random drops are `gnnb_bernoulli_keep`, keyed by a `seed` keyword or by a seed drawn from torch's default generator.

Deliberate differences from the reference:
1. The random draws are counter-based and keyed by `seed`, so they agree with the reference's `rand() < p` in
   distribution only.
2. remove_nodes slices `graph_indicator`; the reference keeps the old vector, which has the wrong length once nodes are
   gone.
3. add_nodes on a batched graph appends the new nodes to the last graph, so the indicator stays sorted and has length
   num_nodes; the reference leaves it short.
4. getgraph keeps an edge only when both of its endpoints are kept.  The reference tests only the source: on a batched
   graph the two rules agree, and on other graphs the reference throws a KeyError.
5. Ids out of range raise AssertionError instead of BoundsError.
6. random_walk_pe sums each walk step in the plan's edge order instead of forming dense matrix products, so it agrees
   with the reference to rounding; walk_length < 1 raises AssertionError (the reference throws BoundsError or
   ArgumentError).
7. color_refinement refines to the fixed point, renumbers the colours from 1 in every round and groups signatures by
   a multiset hash of its own; the reference stops after at most two rounds and carries its ids over between rounds
   (see its docstring).
8. ppr_diffusion inverts each graph of a batch on its own, by Gauss-Jordan elimination up to 240 nodes and LU above
   (LAPACK's LU of the whole batch in the reference), so the two agree to rounding; a singular M raises
   torch.linalg.LinAlgError where the reference throws SingularException.
"""
from __future__ import annotations

import ctypes as C
import numbers
import operator
from typing import List, Optional

import torch

from . import _lib
from . import graph as _graph
from . import readout as _readout
from ._lib import lib
from .graph import GNNGraph, _as_index, _Plan, _ptr, _stream, colmajor, rows, unrows
from .msgpass import mean


def _on_device(g: GNNGraph) -> GNNGraph:
    dev = _graph._compute_device(g.s)
    return g if g.s.device == dev else g.to(dev)


def _take_edges(x: torch.Tensor, idx: torch.Tensor) -> torch.Tensor:
    """getobs(x, idx) on a Julia-shaped edge array (last dimension = edges)"""
    return unrows(rows(x)[idx])


def sort_edge_index(u, v=None, *, return_perm: bool = False):
    """Lexicographic, stable sort of the pairs (u[k], v[k]) — `sort_edge_index(u, v)` / `sort_edge_index((u, v))`.
    Returns (u_sorted, v_sorted) and, with return_perm, the 0-based permutation as a third value."""
    if v is None:
        u, v = u
    u, v = _as_index(u), _as_index(v)
    assert u.dim() == 1 and u.shape == v.shape, "u and v must be vectors of equal length"
    dev = _graph._compute_device(u)
    u, v = u.to(dev), v.to(device=dev, dtype=u.dtype)
    n = int(u.numel())
    uo, vo = torch.empty_like(u), torch.empty_like(v)
    perm = torch.empty(n, dtype=torch.int64, device=dev)
    if n:
        hi = int(max(int(u.max()), int(v.max())))
        with torch.cuda.device(dev):
            _lib.check(lib.gnnb_sort_edge_index(u.data_ptr(), v.data_ptr(), n, max(hi, 0), u.element_size(),
                                                uo.data_ptr(), vo.data_ptr(), perm.data_ptr(), _stream(dev)))
    return (uo, vo, perm) if return_perm else (uo, vo)


def remove_self_loops(g: GNNGraph) -> GNNGraph:
    """Drop the edges with s == t; edge weights and features follow (transform.jl:49-64)."""
    keep = (g.s != g.t).nonzero().reshape(-1)
    return GNNGraph(g.s[keep], g.t[keep], None if g.w is None else g.w[keep], num_nodes=g.num_nodes, ndata=g.ndata,
                    edata={k: _take_edges(x, keep.to(x.device)) for k, x in g.edata.items()}, gdata=g.gdata,
                    num_graphs=g.num_graphs, graph_indicator=g.graph_indicator)


def remove_multi_edges(g: GNNGraph, aggr=operator.add) -> GNNGraph:
    """One edge per distinct (s, t), in (s, t) order; weights and edge features of the collapsed edges are reduced with
    `aggr` (+, mean, max, min) — transform.jl:157-190."""
    g = _on_device(g)
    dev, E = g.s.device, g.num_edges
    if E == 0:
        return g
    so, to = torch.empty_like(g.s), torch.empty_like(g.t)
    perm = torch.empty(E, dtype=torch.int64, device=dev)
    seg = torch.empty(E, dtype=torch.int64, device=dev)
    nu = C.c_int64(0)
    with torch.cuda.device(dev):
        _lib.check(lib.gnnb_coalesce_edges(g.s.data_ptr(), g.t.data_ptr(), E, g.num_nodes, g.s.element_size(), 1,
                                           so.data_ptr(), to.data_ptr(), perm.data_ptr(), seg.data_ptr(), C.byref(nu),
                                           _stream(dev)))
    nu = int(nu.value)
    ip = _readout._IndicatorPlan(seg, nu, dev)        # sorted edge k -> distinct pair seg[k]: `_scatter(aggr, ·, idxs)`

    def reduce(x: torch.Tensor) -> torch.Tensor:
        return _readout._reduce(aggr, ip, _take_edges(x.to(dev), perm))

    return GNNGraph(so[:nu].clone(), to[:nu].clone(), None if g.w is None else reduce(g.w), num_nodes=g.num_nodes,
                    ndata=g.ndata, edata={k: reduce(x) for k, x in g.edata.items()}, gdata=g.gdata,
                    num_graphs=g.num_graphs, graph_indicator=g.graph_indicator)


def to_bidirected(g: GNNGraph) -> GNNGraph:
    """Add the reverse of every edge, then remove_multi_edges with mean (transform.jl:495-510)."""
    both = GNNGraph(torch.cat([g.s, g.t]), torch.cat([g.t, g.s]), None if g.w is None else torch.cat([g.w, g.w]),
                    num_nodes=g.num_nodes, ndata=g.ndata,
                    edata={k: unrows(torch.cat([rows(x), rows(x)], dim=0)) for k, x in g.edata.items()},
                    gdata=g.gdata, num_graphs=g.num_graphs, graph_indicator=g.graph_indicator)
    return remove_multi_edges(both, aggr=mean)


def unbatch(g: GNNGraph) -> List[GNNGraph]:
    """Split a batched graph back into its components (transform.jl:741-778).  Node ids are shifted back, node/edge
    features are sliced; the edges must be grouped per graph (as `batch` leaves them) — asserted like the reference."""
    if g.num_graphs == 1:
        return [g]
    gi = g.graph_indicator.to(torch.int64).cpu()
    assert bool((gi[1:] >= gi[:-1]).all()), "The graph_indicator vector must be sorted."
    n_per = torch.bincount(gi - 1, minlength=g.num_graphs)
    cum = torch.cat([torch.zeros(1, dtype=torch.int64), torch.cumsum(n_per, 0)])
    ge = gi[(g.s.to(torch.int64) - 1).cpu()] - 1                       # graph of each edge (by its source)
    assert bool((ge[1:] >= ge[:-1]).all()), \
        "Error in unbatching, likely the edges are not sorted (first edges belong to the first graphs, then edges in " \
        "the second graph and so on)"
    e_per = torch.bincount(ge, minlength=g.num_graphs)
    ecum = torch.cat([torch.zeros(1, dtype=torch.int64), torch.cumsum(e_per, 0)])
    out = []
    for i in range(g.num_graphs):
        n0, n1, e0, e1 = int(cum[i]), int(cum[i + 1]), int(ecum[i]), int(ecum[i + 1])
        out.append(GNNGraph(g.s[e0:e1] - n0, g.t[e0:e1] - n0, None if g.w is None else g.w[e0:e1], num_nodes=n1 - n0,
                            ndata={k: x[..., n0:n1] for k, x in g.ndata.items()},
                            edata={k: x[..., e0:e1] for k, x in g.edata.items()},
                            gdata={k: x[..., i] for k, x in g.gdata.items()}))
    return out


def csr(g: GNNGraph, transposed: bool = False):
    """(rowptr, col, eid) of the plan as int32 device tensors: CSR by target (col = source of each sorted edge), or by
    source with transposed=True; eid[k] = 0-based COO position of sorted edge k (stable within a row)."""
    p = g.plan()
    nrows = g.num_nodes
    rowptr = torch.empty(nrows + 1, dtype=torch.int32, device=p.device)
    col = torch.empty(g.num_edges, dtype=torch.int32, device=p.device)
    eid = torch.empty(g.num_edges, dtype=torch.int32, device=p.device)
    with torch.cuda.device(p.device):
        _lib.check(lib.gnnb_graph_csr_device(p.h, int(bool(transposed)), rowptr.data_ptr(), col.data_ptr(),
                                             eid.data_ptr(), _stream(p.device)))
    return rowptr, col, eid


# ---------------------------------------------------------------------------------------------- graph editing
def _device(g: GNNGraph) -> torch.device:
    return g._plan.device if g._plan is not None else _graph._compute_device(g.s)


def _drop_mask(k: int, p, seed, dev) -> torch.Tensor:
    """keep[i] = !(u_i < p): the reference's `rand() < p` drop rule on a counter-based stream (gnnb_bernoulli_keep)"""
    from .linkpred import _seed                      # linkpred imports query, which imports this module
    keep = torch.empty(k, dtype=torch.uint8, device=dev)
    with torch.cuda.device(dev):
        _lib.check(lib.gnnb_bernoulli_keep(k, float(p), _seed(seed), _ptr(keep) if k else None, _stream(dev)))
    return keep


def _id_mask(ids, k: int, dev, what: str) -> torch.Tensor:
    """keep mask of k items without the 1-based `ids` (repeats allowed)"""
    ids = _as_index(ids).reshape(-1).to(device=dev, dtype=torch.int64)
    keep = torch.ones(k, dtype=torch.uint8, device=dev)
    if ids.numel():
        assert int(ids.min()) >= 1 and int(ids.max()) <= k, f"{what} id out of range 1:{k}"
        keep[ids - 1] = 0
    return keep


def _is_probability(x) -> bool:
    return isinstance(x, numbers.Real) or (isinstance(x, torch.Tensor) and x.dim() == 0)


def _is_integral_scalar(x) -> bool:
    return isinstance(x, numbers.Integral) or (isinstance(x, torch.Tensor) and x.dim() == 0 and
                                               not x.is_floating_point())


# The child's plan is derived from the parent's only when the parent has at most this many edges.  A derived direction
# gathers newid[eid[k]] (4 B per parent edge, in the parent's sorted order) for every parent edge; while that array fits
# in the H100's 50 MB L2 the gathers hit L2 and derivation beats a fresh sort of the child, at every keep share and for
# every function measured, and at 100 M edges in random order it loses to the sort at every keep share (DESIGN.md §7).
_DERIVE_MAX_EDGES = 1 << 23


def _subgraph(g: GNNGraph, node_keep: Optional[torch.Tensor], edge_keep: Optional[torch.Tensor], extra_nodes: int = 0):
    """The child of g that keeps the nodes of `node_keep` (uint8 mask, None = all) renumbered in ascending old id, then
    `extra_nodes` isolated nodes, and the edges of `edge_keep` (None = all) whose two endpoints are kept, in COO order.
    Returns (s, t, num_nodes, kept_eids (0-based int64), plan or None).  With g's plan built and at most _DERIVE_MAX_EDGES
    edges in g, the child's plan is derived from g's (gnnb_graph_subgraph); otherwise the child stays lazy (its plan is a fresh sort when first needed) and the same arrays come from the
    masks.  Both routes give the same bits."""
    dev = _device(g)
    n, E = g.num_nodes, g.num_edges
    s0, t0 = g.s.to(dev), g.t.to(dev)
    if g._plan is not None and E <= _DERIVE_MAX_EDGES:
        p = g._plan
        kept = torch.empty(E, dtype=torch.int64, device=dev)
        nmap = None if node_keep is None else torch.empty(n, dtype=torch.int32, device=dev)
        h, n2, e2 = C.c_void_p(), C.c_int64(0), C.c_int64(0)
        with torch.cuda.device(dev):
            _lib.check(lib.gnnb_graph_subgraph(p.h, _ptr(node_keep), _ptr(edge_keep), int(extra_nodes), C.byref(h),
                                               _ptr(nmap), _ptr(kept) if E else None, C.byref(n2), C.byref(e2),
                                               _stream(dev)))
        plan, n2, kept = _Plan(h.value, dev), int(n2.value), kept[:int(e2.value)]
    else:
        ek = torch.ones(E, dtype=torch.bool, device=dev) if edge_keep is None else edge_keep.bool()
        nmap, n2 = None, n + int(extra_nodes)
        if node_keep is not None:
            nk = node_keep.bool()
            ek = ek & nk[s0.long() - 1] & nk[t0.long() - 1]
            nmap = torch.where(nk, torch.cumsum(nk, 0, dtype=torch.int32) - 1, -1).to(torch.int32)
            n2 = int(nk.sum()) + int(extra_nodes)
        assert n2 < 2 ** 31 - 1, f"kept nodes + extra nodes = {n2} must be < 2^31-1"
        plan, kept = None, ek.nonzero().reshape(-1)
    s, t = s0[kept], t0[kept]
    if nmap is not None:
        s = (nmap[s.long() - 1] + 1).to(g.s.dtype)
        t = (nmap[t.long() - 1] + 1).to(g.s.dtype)
    return s, t, n2, kept, plan


def _with_plan(h: GNNGraph, plan: Optional[_Plan]) -> GNNGraph:
    h._plan = plan
    return h


def _take(x: Optional[torch.Tensor], idx: torch.Tensor) -> Optional[torch.Tensor]:
    """getobs along the last dimension (edges, nodes or graphs)"""
    return None if x is None else _take_edges(x, idx.to(x.device))


def remove_edges(g: GNNGraph, edges_or_p=0.5, *, seed=None) -> GNNGraph:
    """DropEdge — transform.jl:121-147.  A vector of 1-based edge ids (repeats allowed) removes those edges; a number p
    drops each edge independently with probability p (gnnb_bernoulli_keep, keyed by `seed`).  Weights and edge
    features follow the kept edges; nodes are unchanged."""
    dev = _device(g)
    if _is_probability(edges_or_p):
        keep = _drop_mask(g.num_edges, edges_or_p, seed, dev)
    else:
        keep = _id_mask(edges_or_p, g.num_edges, dev, "edge")
    s, t, n, kept, plan = _subgraph(g, None, keep)
    return _with_plan(GNNGraph(s, t, _take(g.w, kept), num_nodes=n, ndata=g.ndata,
                               edata={k: _take(x, kept) for k, x in g.edata.items()}, gdata=g.gdata,
                               num_graphs=g.num_graphs, graph_indicator=g.graph_indicator), plan)


def remove_nodes(g: GNNGraph, nodes_or_p, *, seed=None) -> GNNGraph:
    """DropNode — transform.jl:212-276.  A vector of 1-based node ids (de-duplicated) or a drop probability p per node
    (keyed by `seed`).  The edges touching a removed node go too; the kept nodes are renumbered in ascending old id.
    Node features and graph_indicator are sliced, weights and edge features follow the kept edges."""
    if _is_integral_scalar(nodes_or_p):      # the reference has remove_nodes(g, p::AbstractFloat) and a vector method
        raise TypeError("remove_nodes takes a vector of node ids or a float drop probability; to remove node i, pass [i]")
    dev = _device(g)
    if _is_probability(nodes_or_p):
        keep = _drop_mask(g.num_nodes, nodes_or_p, seed, dev)
    else:
        keep = _id_mask(nodes_or_p, g.num_nodes, dev, "node")
    return _keep_nodes(g, keep)


def _keep_nodes(g: GNNGraph, keep: torch.Tensor) -> GNNGraph:
    """remove_nodes(g, <the nodes whose uint8 `keep` is 0>) for a mask on g's device."""
    s, t, n, kept, plan = _subgraph(g, keep, None)
    nodes = keep.bool().nonzero().reshape(-1)
    return _with_plan(GNNGraph(s, t, _take(g.w, kept), num_nodes=n,
                               ndata={k: _take(x, nodes) for k, x in g.ndata.items()},
                               edata={k: _take(x, kept) for k, x in g.edata.items()}, gdata=g.gdata,
                               num_graphs=g.num_graphs, graph_indicator=_take(g.graph_indicator, nodes)), plan)


def getgraph(g: GNNGraph, i, *, nmap: bool = False):
    """The graphs `i` (1-based, an int or a vector) of a batched graph, as one graph — transform.jl:825-888.  The
    indicator is renumbered by position in `i` and gdata is sliced by `i`; with nmap=True also the 1-based old ids of
    the kept nodes.  A graph without graph_indicator is its own only component: getgraph(g, 1) is g itself."""
    ids = [int(v) for v in (i.reshape(-1).tolist() if isinstance(i, torch.Tensor) else
                            ([i] if isinstance(i, numbers.Integral) else i))]
    if g.graph_indicator is None:
        assert ids == [1], "a graph without graph_indicator has only graph 1"
        return (g, torch.arange(1, g.num_nodes + 1, device=g.s.device)) if nmap else g
    assert all(1 <= v <= g.num_graphs for v in ids), f"graph id out of range 1:{g.num_graphs}"
    dev = _device(g)
    lut = torch.zeros(g.num_graphs + 1, dtype=torch.int64)
    for pos, v in enumerate(ids):                  # the reference's Dict: a repeated id takes its last position
        lut[v] = pos + 1
    gi = lut.to(dev)[g.graph_indicator.to(dev).long()]
    keep = (gi > 0).to(torch.uint8)
    s, t, n, kept, plan = _subgraph(g, keep, None)
    nodes = keep.bool().nonzero().reshape(-1)
    gidx = torch.tensor(ids, dtype=torch.int64) - 1
    h = _with_plan(GNNGraph(s, t, _take(g.w, kept), num_nodes=n,
                            ndata={k: _take(x, nodes) for k, x in g.ndata.items()},
                            edata={k: _take(x, kept) for k, x in g.edata.items()},
                            gdata={k: _take(x, gidx) for k, x in g.gdata.items()}, num_graphs=len(ids),
                            graph_indicator=gi[nodes].to(g.graph_indicator.dtype)), plan)
    return (h, nodes + 1) if nmap else h


def add_nodes(g: GNNGraph, n: int, *, ndata=None) -> GNNGraph:
    """n isolated nodes after the existing ones — transform.jl:553-563.  `ndata` (a tensor is named x) must have the
    keys of g.ndata, with n columns each.  On a batched graph the new nodes join the last graph."""
    n = int(n)
    assert n >= 0, "the number of nodes to add must be >= 0"
    new = {} if ndata is None else ({"x": ndata} if isinstance(ndata, torch.Tensor) else dict(ndata))
    assert sorted(new) == sorted(g.ndata), "cannot concatenate feature data with different keys"
    nd = {}
    for k, x in g.ndata.items():
        y = torch.as_tensor(new[k]).to(device=x.device, dtype=x.dtype)
        assert y.shape[-1] == n, f"ndata[{k}] of the new nodes must have {n} columns"
        nd[k] = torch.cat([colmajor(x), colmajor(y)], dim=-1)
    s, t, num_nodes, kept, plan = _subgraph(g, None, None, n)
    gi = g.graph_indicator
    if gi is not None:
        gi = torch.cat([gi, torch.full((n,), g.num_graphs, dtype=gi.dtype, device=gi.device)])
    return _with_plan(GNNGraph(s, t, g.w, num_nodes=num_nodes, ndata=nd, edata=g.edata, gdata=g.gdata,
                               num_graphs=g.num_graphs, graph_indicator=gi), plan)


# ---------------------------------------------------------------------------------------------- random-walk encoding
# Segments of at most this many nodes walk in shared memory (gnnb_random_walk_pe, csrc/rwpe.cu); larger ones are composed
# from the fused propagate.  Must not exceed GNNB_RWPE_SMEM_MAX_NODES (include/gnnb200.h), whose rows the kernel leaves
# untouched; lowering it (tests do) routes more segments to the propagate route, which overwrites their rows.
_RWPE_KERNEL_MAX_NODES = 896      # GNNB_RWPE_SMEM_MAX_NODES
_RWPE_SMEM_MAX_NODES = _RWPE_KERNEL_MAX_NODES
_RWPE_BLOCK = 128          # sources per propagate pass: D = 128 is the lean kernel's row width


def _rwpe_segments(g: GNNGraph, dev) -> Optional[torch.Tensor]:
    """seg_ptr (int64, on dev) of the runs of equal graph_indicator values, or None (the whole graph is one segment)
    when there is no indicator, it is not non-decreasing, or an edge joins two graphs."""
    if g.graph_indicator is None:
        return None
    from .generate import _segments
    order, seg_ptr, _, gi = _segments(g.graph_indicator, g.num_nodes, dev)
    if order is not None or seg_ptr is None:
        return None
    gi = gi.to(device=dev, dtype=torch.int64)
    if g.num_edges and not bool((gi[g.s.long() - 1] == gi[g.t.long() - 1]).all()):
        return None
    return seg_ptr


def _rwpe_propagate(g: GNNGraph, w: Optional[torch.Tensor], dinv: torch.Tensor, K: int, out: torch.Tensor) -> None:
    """out (n, K) = the walks of g (one segment) from `walk_length` launches of the fused propagate per block of
    _RWPE_BLOCK sources: a one-hot (n, 128) state, u_k = dinv .* propagate(w_mul_xj | copy_xj, g, +; u_{k-1})."""
    p = g.plan()
    n, D = g.num_nodes, _RWPE_BLOCK
    if w is not None and w.numel() == 0:            # a segment without edges: no weights to multiply
        w = None
    x = torch.zeros((n, D), dtype=torch.float32, device=p.device)
    y = torch.empty_like(x)
    msg = _lib.W_MUL_XJ if w is not None else _lib.COPY_XJ
    for b0 in range(0, n, D):
        nb = min(D, n - b0)
        cols = torch.arange(nb, device=p.device)
        x.zero_()
        x[b0 + cols, cols] = 1.0
        for k in range(K):
            with torch.cuda.device(p.device):
                _lib.check(lib.gnnb_propagate(p.h, 0, msg, _lib.SUM, x.data_ptr(), _ptr(w), None, dinv.data_ptr(), D,
                                              y.data_ptr(), _stream(p.device)))
            out[b0:b0 + nb, k] = y[b0 + cols, cols]
            x, y = y, x


def random_walk_pe(g: GNNGraph, walk_length: int) -> torch.Tensor:
    """The random-walk structural encoding — transform.jl:975-990: a (walk_length, num_nodes) float32 matrix with
    PE[k, j] = (RW^k)[j, j], k = 1..walk_length, RW[i, j] = A[i, j] * dinv[j].  A[i, j] is the summed weight of the
    edges i -> j (g.w, or 1 without weights; multi-edges add up, self loops count), dinv = 1 / weighted out-degree with
    +-Inf set to 0: the reference's orientation, the out-degree scales the column node.  Node-major in memory (Julia's
    (K, N) matrix), on g's compute device.  Not differentiable, like the reference.

    The walk from node j is the row recurrence u_0 = e_j, u_k[t] = dinv[t] * Σ_{edges s -> t} w_e u_{k-1}[s] on the CSR
    by target (each product and sum rounded, plan order), PE[k, j] = u_k[j]: E_graph multiply-adds per step and per
    source instead of the reference's K dense N x N products (212 GB per matrix for a batch of 10 000 molecules).
    Walks never leave a graph, so a batched graph is split into segments, one per run of equal graph_indicator values,
    when the indicator is non-decreasing and no edge joins two graphs; otherwise the whole graph is one segment.
      * Segments of at most _RWPE_SMEM_MAX_NODES (896) nodes: gnnb_random_walk_pe, the walk state in shared memory
        (32 sources per warp or CTA), one launch for all segments of up to 32 nodes and one for the larger ones.
      * Larger segments, one after the other: per block of 128 sources, walk_length launches of the fused propagate at
        D = 128 on the segment's plan (derived from g's, no sort).  Memory 2 * n_seg * 128 * 4 bytes; time
        ceil(n_seg / 128) * walk_length propagates over the segment's edges — seconds for 10^5 nodes, hours for 10^7.
        No size cap.  Each propagate is followed by two small torch indexing launches, and each such segment first
        derives its plan in a pass over all of g's nodes and edges, so a batch of many graphs just above the bound costs
        (number of such graphs) x (N + E) in bookkeeping on top and is bound by launches, not by the propagates.
    Both routes give the same bits for every row of at most the plan's chunk edges (longer rows are reduced piecewise by
    the propagate).  Against the reference the only difference is the summation order, so the two agree to rounding."""
    assert isinstance(walk_length, numbers.Integral) and not isinstance(walk_length, bool) and walk_length >= 1, \
        f"walk_length = {walk_length} must be an integer >= 1"
    K = int(walk_length)
    g = _on_device(g)
    dev, n = g.s.device, g.num_nodes
    out = torch.empty((n, K), dtype=torch.float32, device=dev)
    if n == 0:
        return unrows(out)
    p = g.plan()
    w = None if g.w is None else g.w.to(device=p.device, dtype=torch.float32).contiguous()
    deg = torch.empty(n, dtype=torch.float32, device=p.device)
    with torch.cuda.device(p.device):
        _lib.check(lib.gnnb_degree(p.h, _lib.DIR_OUT, _ptr(w), deg.data_ptr(), _stream(p.device)))
    dinv = torch.reciprocal(deg)
    dinv[torch.isinf(dinv)] = 0.0
    seg_ptr = _rwpe_segments(g, p.device)
    n_seg = 1 if seg_ptr is None else int(seg_ptr.numel()) - 1
    bound = min(_RWPE_SMEM_MAX_NODES, _RWPE_KERNEL_MAX_NODES)
    if seg_ptr is None:
        big = [] if n <= bound else [0]
    else:
        big = ((seg_ptr[1:] - seg_ptr[:-1]) > bound).nonzero().reshape(-1).tolist()
    if len(big) < n_seg:
        with torch.cuda.device(p.device):
            _lib.check(lib.gnnb_random_walk_pe(p.h, _ptr(w), dinv.data_ptr(), _ptr(seg_ptr), n_seg, K, out.data_ptr(),
                                               _stream(p.device)))
    for i in big:
        if n_seg == 1:
            _rwpe_propagate(g, w, dinv, K, out)
            continue
        a, b = int(seg_ptr[i]), int(seg_ptr[i + 1])
        keep = torch.zeros(n, dtype=torch.uint8, device=p.device)
        keep[a:b] = 1
        s, t, n2, kept, plan = _subgraph(g, keep, None)
        h = _with_plan(GNNGraph(s, t, None if w is None else w[kept], num_nodes=n2), plan)
        _rwpe_propagate(h, h.w, dinv[a:b].contiguous(), K, out[a:b])
    return unrows(out)


def color_refinement(g: GNNGraph, x0=None, *, max_iters: Optional[int] = None):
    """1-WL colour refinement — utils.jl:340-389: returns (x, num_colors, niters).

    Round r maps node i to its signature (c_i, multiset{c_s : edges s -> i}): the in-neighbours, with multiplicity, a
    self loop making i its own neighbour, edge weights ignored.  Two nodes get the same new colour iff their
    signatures are equal, and the colours are numbered 1..k in order of first appearance by node id (the reference's
    `get!(hashmap, ..., length(hashmap) + 1)` within one round).  A batched graph is refined as one graph, so colours
    compare across its graphs.  x0 (an integer vector of length num_nodes) matters only through its partition; None
    starts every node in one class.  The rounds run until one leaves the number of classes unchanged — refinement only
    splits classes, so that round reproduces the previous colours — or until `max_iters` rounds (an integer >= 1; 2
    gives the reference's partition and is the h-round form of WL features).  niters counts the rounds computed,
    the last included; a capped call that has not converged returns niters == max_iters.  x is an int64 tensor on
    g's compute device; num_colors and niters are Python ints.  An empty graph gives (empty, 0, 1).

    Each round is one pass of gnnb_color_refinement's signature kernel over the in-edges and a stable radix sort of
    the exact key (c_i, S_1, S_2), S_k = Σ_{edges s -> i} splitmix64(c_s ^ salt_k) mod 2^61 - 1, with one count read
    back per round.  Deliberate differences from the reference:
      * the loop runs to the fixed point; the reference stops after at most two rounds (its x and x' alias after the
        first, so the second ends the loop), and its own test expects niters == 2;
      * colours are renumbered from 1 in every round, so nothing carries over from earlier rounds (the reference's ids
        continue across rounds: its known answer starts at 4);
      * signatures are grouped by the multiset hash above instead of Julia's `hash` of the sorted list.  Both are
        probabilistic: two different multisets with the same c_i share (S_1, S_2) with probability about 2^-122 per
        pair under a random-function model of splitmix64.  That bounds chance collisions, not inputs built to collide.
    Wrong-length x0 or a max_iters that is not an integer >= 1 raise AssertionError."""
    assert max_iters is None or (isinstance(max_iters, numbers.Integral) and not isinstance(max_iters, bool)
                                 and max_iters >= 1), f"max_iters = {max_iters} must be None or an integer >= 1"
    g = _on_device(g)
    dev, n = g.s.device, g.num_nodes
    if x0 is not None:
        x0 = torch.as_tensor(x0)
        assert x0.dim() == 1 and x0.numel() == n, f"len(x0) = {x0.numel()} must equal num_nodes = {n}"
        assert not (x0.is_floating_point() or x0.is_complex()), f"x0 must hold integers, not {x0.dtype}"
    out = torch.empty(n, dtype=torch.int64, device=dev)
    if n == 0:
        return out, 0, 1
    p = g.plan()
    x = None if x0 is None else x0.to(device=p.device, dtype=torch.int64).contiguous()
    num_colors, niters = C.c_int64(0), C.c_int64(0)
    with torch.cuda.device(p.device):
        _lib.check(lib.gnnb_color_refinement(p.h, _ptr(x), 0 if max_iters is None else int(max_iters), out.data_ptr(),
                                             C.byref(num_colors), C.byref(niters), _stream(p.device)))
    return out, int(num_colors.value), int(niters.value)


# ---------------------------------------------------------------------------------------------- PPR diffusion
# Segments of at most this many nodes are inverted in shared memory (gnnb_ppr_diffusion, csrc/ppr.cu); larger ones take
# the dense route.  Must not exceed GNNB_PPR_SMEM_MAX_NODES (include/gnnb200.h), whose larger segments the kernel skips;
# lowering it (tests do) routes more segments to the dense route.
_PPR_KERNEL_MAX_NODES = 240       # GNNB_PPR_SMEM_MAX_NODES
_PPR_SMEM_MAX_NODES = _PPR_KERNEL_MAX_NODES
_PPR_PAD = 128                    # the dense route pads a segment to a multiple of this many nodes
_PPR_BATCH_BYTES = 1 << 30        # M and its inverse of one dense batch; a single segment may exceed it


def _ppr_singular(what: str, step: int) -> torch.linalg.LinAlgError:
    return torch.linalg.LinAlgError(f"ppr_diffusion: M = I + (alpha - 1) A of {what} is singular (zero pivot at step "
                                    f"{step}); the reference's inv throws SingularException")


def _ppr_dense(p: _Plan, w: Optional[torch.Tensor], alpha: float, segs: List[tuple], s0: torch.Tensor,
               t0: torch.Tensor, eseg: torch.Tensor, out: torch.Tensor, fail) -> None:
    """The segments [(i, a, b)] above the shared-memory bound, grouped by padded size P: each batch of M blocks is built
    by gnnb_ppr_matrix into identity-padded (P, P) matrices and inverted by torch.linalg.inv_ex, and
    out[e] = fl32(alpha) * inv[t_e - a, s_e - a] is gathered for the segments' edges (eseg[e] = segment of edge e).
    Identity padding leaves the inverse of the real block unchanged and keeps a singular block singular (the pad rows
    are zero in its columns)."""
    dev = p.device
    a32 = torch.tensor(alpha, dtype=torch.float32, device=dev)
    groups = {}
    for seg in segs:
        groups.setdefault(-(-(seg[2] - seg[1]) // _PPR_PAD) * _PPR_PAD, []).append(seg)
    slot = torch.full((segs[-1][0] + 1,), -1, dtype=torch.int64, device=dev)       # segment -> matrix of the batch
    esafe = eseg.clamp(max=segs[-1][0])
    for P, members in sorted(groups.items()):
        per = max(1, _PPR_BATCH_BYTES // (2 * 4 * P * P))
        for c0 in range(0, len(members), per):
            chunk = members[c0:c0 + per]
            M = torch.eye(P, dtype=torch.float32, device=dev).repeat(len(chunk), 1, 1)
            with torch.cuda.device(dev):
                for k, (_, a, b) in enumerate(chunk):
                    _lib.check(lib.gnnb_ppr_matrix(p.h, _ptr(w), alpha, a, b, P, M[k].data_ptr(), _stream(dev)))
            inv, info = torch.linalg.inv_ex(M)
            del M
            bad = (info > 0).nonzero().reshape(-1)
            if bad.numel():
                k = int(bad[0])
                raise fail(chunk[k][0], int(info[k]))
            ids = torch.tensor([i for i, _, _ in chunk], dtype=torch.int64, device=dev)
            base = torch.tensor([a for _, a, _ in chunk], dtype=torch.int64, device=dev)
            slot[ids] = torch.arange(len(chunk), device=dev)
            e = ((eseg == esafe) & (slot[esafe] >= 0)).nonzero().reshape(-1)
            k = slot[esafe[e]]
            out[e] = a32 * inv[k, t0[e] - base[k], s0[e] - base[k]]
            slot[ids] = -1


def ppr_diffusion(g: GNNGraph, *, alpha=0.85) -> GNNGraph:
    """Personalized-PageRank diffusion of the edge weights — transform.jl:1026-1051.  Returns a graph with g's edges,
    node, edge and graph data, indicator and plan, whose weight of edge s -> t is fl32(alpha) * inv(M)[t, s] for
    M = I + (fl32(alpha) - 1) A, A[t, s] the summed weight of the edges s -> t (g.w, or 1 without weights; duplicates add
    up and all get the same new weight, self loops count).  A is not normalised: the reference's docstring mentions a
    normalisation its code does not do, and this follows the code.  Not differentiable.

    The inverse of a block-diagonal matrix is block-diagonal, so a batched graph is inverted per segment: one per run of
    equal graph_indicator values when the indicator is non-decreasing and no edge joins two graphs, otherwise the whole
    graph is one segment.
      * Segments of at most _PPR_SMEM_MAX_NODES (240) nodes: gnnb_ppr_diffusion, all in one call.  M is built and
        inverted in shared memory by Gauss-Jordan elimination with partial pivoting, one warp per segment of up to 32
        nodes and one CTA per larger one, bit for bit the float32 statement of csrc/ppr.cu.
      * Larger segments: the reference's dense inverse, per segment and on the device.  M is built by gnnb_ppr_matrix
        into identity-padded batches (a multiple of 128 nodes, about 1 GB of matrices per batch) and inverted by
        torch.linalg.inv_ex.  O(n^3) time and n^2 memory per segment: a graph too large for the card raises torch's
        out-of-memory error, as the reference would.
    A singular M on either route raises torch.linalg.LinAlgError naming the first singular graph (1-based) and the step
    of its zero pivot, where the reference throws SingularException.  Non-finite weights or alpha raise nothing."""
    g = _on_device(g)
    dev, n, E = g.s.device, g.num_nodes, g.num_edges
    w_out = torch.empty(E, dtype=torch.float32, device=dev)
    if n == 0 or E == 0:
        return _graph.set_edge_weight(g, w_out)
    alpha = float(alpha)
    p = g.plan()
    w = None if g.w is None else g.w.detach().to(device=p.device, dtype=torch.float32).contiguous()
    seg_ptr = _rwpe_segments(g, p.device)
    bounds = [0, n] if seg_ptr is None else seg_ptr.tolist()
    n_seg = len(bounds) - 1
    bound = min(_PPR_SMEM_MAX_NODES, _PPR_KERNEL_MAX_NODES)
    big = [i for i in range(n_seg) if bounds[i + 1] - bounds[i] > bound]

    def fail(i: int, step: int) -> torch.linalg.LinAlgError:
        what = "the graph" if seg_ptr is None else f"graph {int(g.graph_indicator[bounds[i]])}"
        return _ppr_singular(what, step)

    if len(big) < n_seg:
        info = torch.empty(n_seg, dtype=torch.int32, device=p.device)
        with torch.cuda.device(p.device):
            _lib.check(lib.gnnb_ppr_diffusion(p.h, _ptr(w), alpha, _ptr(seg_ptr), n_seg, w_out.data_ptr(),
                                              info.data_ptr(), _stream(p.device)))
        bad = (info > 0).nonzero().reshape(-1)
        if bad.numel():
            i = int(bad[0])
            raise fail(i, int(info[i]))
    if big:
        s0, t0 = g.s.to(p.device).long() - 1, g.t.to(p.device).long() - 1
        eseg = torch.zeros(E, dtype=torch.int64, device=p.device) if seg_ptr is None else \
            torch.searchsorted(seg_ptr, t0, right=True) - 1
        _ppr_dense(p, w, alpha, [(i, bounds[i], bounds[i + 1]) for i in big], s0, t0, eseg, w_out, fail)
    return _graph.set_edge_weight(g, w_out)
