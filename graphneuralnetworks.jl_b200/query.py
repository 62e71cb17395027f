"""Graph queries next to the hot path, answered from the device plan (GNNGraphs/src/query.jl):

    adjacency_list(g[, nodes]; dir=:out, with_eid=false)   query.jl:176-206   (the plan's CSR is that list)
    inneighbors / outneighbors(g, i)                        query.jl:109-141
    adjacency_matrix(g; dir=:out, weighted=true)           query.jl:220-231   (dense, for small graphs and tests)
    has_self_loops / has_multi_edges / is_bidirected        query.jl:553-579   (pair sort / duplicate runs on the device)
    has_isolated_nodes(g; dir=:out)                         query.jl:420-422
    laplacian_matrix / normalized_laplacian / scaled_laplacian   query.jl:424-485 (dense, for small graphs and tests)
    laplacian_lambda_max(g; add_self_loops, dir)            query.jl:598-610   (per-graph eigenvalues, csrc/lmax.cu)
"""
from __future__ import annotations

import warnings
from typing import List, Optional

import numpy as np
import torch

from . import _lib
from ._lib import lib
from .graph import GNNGraph, _as_index, _ptr, _stream, degree, homogeneous_only
from .sampling import sample_edge_ids
from .transform import _on_device, _rwpe_segments, remove_multi_edges, sort_edge_index


def adjacency_list(g: GNNGraph, nodes=None, *, dir: str = "out", with_eid: bool = False):
    """Per queried node (default: all), its out-neighbours (dir="out": targets of its out-edges) or in-neighbours, in COO
    order; with_eid also returns the 1-based edge ids.  Lists of Python lists, like the reference's Vector{Vector}."""
    assert dir in ("out", "in")
    nodes = torch.arange(1, g.num_nodes + 1) if nodes is None else _as_index(nodes).reshape(-1)
    eids, offsets = sample_edge_ids(g, nodes, -1, dir=dir)          # K = -1: every incident edge, adjacency order
    dev = eids.device
    other = (g.t if dir == "out" else g.s).to(dev)[eids - 1].tolist()
    off = offsets.tolist()
    adj = [other[off[i]:off[i + 1]] for i in range(len(off) - 1)]
    if not with_eid:
        return adj
    el = eids.tolist()
    return adj, [el[off[i]:off[i + 1]] for i in range(len(off) - 1)]


def outneighbors(g: GNNGraph, i: int) -> List[int]:
    return adjacency_list(g, [i], dir="out")[0]


def inneighbors(g: GNNGraph, i: int) -> List[int]:
    return adjacency_list(g, [i], dir="in")[0]


def adjacency_matrix(g: GNNGraph, *, dir: str = "out", weighted: bool = True) -> torch.Tensor:
    """Dense A with A[i, j] = (summed weight of the) edges i -> j for dir="out", its transpose for dir="in"."""
    assert dir in ("out", "in")
    w = g.w if (weighted and g.w is not None) else None
    A = torch.zeros(g.num_nodes, g.num_nodes, dtype=torch.float32 if w is not None else torch.int64, device=g.s.device)
    vals = w if w is not None else torch.ones(g.num_edges, dtype=torch.int64, device=g.s.device)
    A.index_put_((g.s.long() - 1, g.t.long() - 1), vals, accumulate=True)
    return A if dir == "out" else A.t()


def has_self_loops(g: GNNGraph) -> bool:
    return bool((g.s == g.t).any())


def has_multi_edges(g: GNNGraph) -> bool:
    """more edges than distinct (s, t) pairs (query.jl:575-579)"""
    if g.num_edges == 0:
        return False
    plain = GNNGraph(g.s, g.t, num_nodes=g.num_nodes)
    return remove_multi_edges(plain).num_edges < g.num_edges


def is_bidirected(g: GNNGraph) -> bool:
    """sort_edge_index(s, t) == sort_edge_index(t, s) (query.jl:553-558)"""
    s1, t1 = sort_edge_index(g.s, g.t)
    s2, t2 = sort_edge_index(g.t, g.s)
    return bool(torch.equal(s1, s2) and torch.equal(t1, t2))


# ---------------------------------------------------------------------------------------------- Laplacian queries
# Segments of at most this many nodes get their eigenvalue from the dense method in shared memory
# (gnnb_laplacian_lambda_max, csrc/lmax.cu); larger ones run together through the batched Lanczos route.  Must not
# exceed GNNB_LMAX_SMEM_MAX_NODES (include/gnnb200.h), whose larger segments the kernel skips; lowering it (tests do)
# routes more segments to the Lanczos route.
_LMAX_KERNEL_MAX_NODES = 169      # GNNB_LMAX_SMEM_MAX_NODES
_LMAX_SMEM_MAX_NODES = _LMAX_KERNEL_MAX_NODES
_LMAX_KRYLOV = 32                 # Krylov dimension of one restart cycle
_LMAX_KEEP = 16                   # Ritz vectors kept by a thick restart
_LMAX_TOL = 1e-6                  # a segment has converged when its Ritz residual |beta_k s_k| is at most this
_LMAX_MAXITER = 100               # restart cycles before giving up (KrylovKit's default maxiter)
_LMAX_DEAD = 1e-10                # a Lanczos vector of smaller norm ends its segment's Krylov space
_SEGDOT_CHUNK = 2048              # GNNB_SEGDOT_CHUNK
_ISOLATED = "Graph contains isolated nodes, cannot compute `normalized_adjacency`."


def _check_dir(dir) -> str:
    if dir not in ("out", "in", "both"):
        raise ValueError(f'dir = {dir!r} must be "out", "in" or "both"')
    return dir


def _check_float_type(T, name: str) -> None:
    if not (isinstance(T, torch.dtype) and T.is_floating_point):
        raise TypeError(f"{name}: T = {T!r} must be a floating-point torch.dtype")


def _dense_adjacency(g: GNNGraph, dir: str, dtype) -> torch.Tensor:
    """A[s, t] = summed weight (or count) of the edges s -> t, transposed for every dir but "out" (the reference's
    `dir == :out ? A : A'`)."""
    n, dev = g.num_nodes, g.s.device
    A = torch.zeros(n, n, dtype=dtype, device=dev)
    vals = torch.ones(g.num_edges, dtype=dtype, device=dev) if g.w is None else g.w.to(dtype)
    A.index_put_((g.s.long() - 1, g.t.long() - 1), vals, accumulate=True)
    return A if dir == "out" else A.t()


def laplacian_matrix(g: GNNGraph, T=None, *, dir: str = "out") -> torch.Tensor:
    """D - A (query.jl:424-428), dense (N, N), with A = adjacency_matrix(g; dir) (weighted) and D its row sums.  T
    defaults to the weights' float32, or int64 for an unweighted graph.  Dense, for small graphs and tests."""
    homogeneous_only(g, "laplacian_matrix")
    _check_dir(dir)
    if T is None:
        T = torch.float32 if g.w is not None else torch.int64
    A = _dense_adjacency(g, dir, torch.float64 if g.w is not None else torch.int64)
    return (torch.diag(A.sum(1)) - A).to(T)


def normalized_laplacian(g: GNNGraph, T=torch.float32, *, add_self_loops: bool = False,
                         dir: str = "out") -> torch.Tensor:
    """I - D^-1/2 A D^-1/2 (query.jl:443-460), dense (N, N) in T, computed in float64: A = adjacency_matrix(g; dir)
    (weighted; A' for "in" and "both"), plus I under add_self_loops, D its row sums.  A zero row sum raises the
    reference's AssertionError.  Not symmetric on a directed graph.  Dense, for small graphs and tests."""
    homogeneous_only(g, "normalized_laplacian")
    _check_dir(dir)
    _check_float_type(T, "normalized_laplacian")
    A = _dense_adjacency(g, dir, torch.float64)
    if add_self_loops:
        A = A + torch.eye(g.num_nodes, dtype=torch.float64, device=A.device)
    deg = A.sum(1)
    if bool((deg == 0).any()):
        raise AssertionError(_ISOLATED)
    c = deg.rsqrt()
    return (torch.eye(g.num_nodes, dtype=torch.float64, device=A.device) - c[:, None] * A * c[None, :]).to(T)


def scaled_laplacian(g: GNNGraph, T=torch.float32, *, dir: str = "out") -> torch.Tensor:
    """2 / lmax * L - I (query.jl:474-485) with L = normalized_laplacian(g, T), dense (N, N).  Like the reference, dir
    is accepted and not used: L is always the :out Laplacian without self loops.  lmax is the largest eigenvalue of
    Symmetric(L) (its upper triangle), which on a batch is the maximum over its graphs when the indicator is
    non-decreasing and no edge joins two graphs, and that of the whole graph otherwise."""
    homogeneous_only(g, "scaled_laplacian")
    _check_dir(dir)
    _check_float_type(T, "scaled_laplacian")
    L = normalized_laplacian(g, T)
    g = _on_device(g)
    seg_ptr = _rwpe_segments(g, g.plan().device) if g.num_graphs > 1 else None
    lmax = float(_lambda_max_segments(g, seg_ptr, "out", False).max())
    return (2 / lmax * L.double() - torch.eye(g.num_nodes, dtype=torch.float64, device=L.device)).to(T)


def has_isolated_nodes(g: GNNGraph, *, dir: str = "out") -> bool:
    """any(degree(g; dir) == 0) (query.jl:420-422), with the weighted degree."""
    homogeneous_only(g, "has_isolated_nodes")
    _check_dir(dir)
    return bool((degree(g, dir=dir) == 0).any())


def _splitmix64(x: torch.Tensor) -> torch.Tensor:
    """csrc/common.cuh's splitmix64 on int64 tensors (wrapping products; logical shifts as masked arithmetic ones)"""
    def shr(v, k):
        return (v >> k) & ((1 << (64 - k)) - 1)
    x = x + -0x61C8864680B583EB                     # 0x9E3779B97F4A7C15
    x = (x ^ shr(x, 30)) * -0x40A7B892E31B1A47      # 0xBF58476D1CE4E5B9
    x = (x ^ shr(x, 27)) * -0x6B2FB644ECCEEE15      # 0x94D049BB133111EB
    return x ^ shr(x, 31)


class _SegDots:
    """out[s, k] = sum over segment s of X[k] * y by gnnb_segment_dots: chunks counted from each segment's start, so
    the bits depend on the segment alone."""

    def __init__(self, seg_ptr: torch.Tensor, kmax: int, dev):
        sizes = seg_ptr[1:] - seg_ptr[:-1]
        chunks = (sizes + _SEGDOT_CHUNK - 1) // _SEGDOT_CHUNK
        self.chunk_ptr = torch.zeros(seg_ptr.numel(), dtype=torch.int64, device=dev)
        torch.cumsum(chunks, 0, out=self.chunk_ptr[1:])
        self.n_chunks = int(self.chunk_ptr[-1])
        self.seg_ptr, self.n_seg, self.n, self.dev = seg_ptr, seg_ptr.numel() - 1, int(seg_ptr[-1]), dev
        self.partial = torch.empty(max(self.n_chunks * kmax, 1), dtype=torch.float64, device=dev)

    def __call__(self, X: torch.Tensor, y: torch.Tensor) -> torch.Tensor:
        K = X.shape[0]
        out = torch.empty((self.n_seg, K), dtype=torch.float64, device=self.dev)
        with torch.cuda.device(self.dev):
            _lib.check(lib.gnnb_segment_dots(X.data_ptr(), K, X.stride(0), y.data_ptr(), self.n, self.seg_ptr.data_ptr(),
                                             self.chunk_ptr.data_ptr(), self.n_seg, self.n_chunks,
                                             self.partial.data_ptr(), out.data_ptr(), _stream(self.dev)))
        return out


def _lmax_lanczos(g: GNNGraph, w: Optional[torch.Tensor], deg: torch.Tensor, dir: str, self_loops: bool,
                  segs: List[tuple], out: torch.Tensor) -> None:
    """out[i] = lmax of the segments [(i, a, b)] together: thick-restart Lanczos on S through the fused propagate.
    S = diag(1 - [self_loops] c^2) - B, B the operator graph of the segments' upper-triangle edges (dir "out": s < t;
    otherwise s > t) mirrored, and their loops, each weighted c_s w c_t (float64, stored as float32), applied by one
    gnnb_propagate(W_MUL_XJ, SUM) at D = 1 on a float32 copy of the float64 Lanczos vector."""
    dev = deg.device
    n = g.num_nodes
    sizes = torch.tensor([b - a for _, a, b in segs], dtype=torch.int64, device=dev)
    seg = torch.zeros(len(segs) + 1, dtype=torch.int64, device=dev)
    torch.cumsum(sizes, 0, out=seg[1:])
    nb = int(seg[-1])
    node_seg = torch.repeat_interleave(torch.arange(len(segs), device=dev), sizes)       # operator node -> segment
    old = torch.cat([torch.arange(a, b, device=dev) for _, a, b in segs])               # operator node -> g's node
    nmap = torch.full((n,), -1, dtype=torch.int64, device=dev)
    nmap[old] = torch.arange(nb, device=dev)
    c = deg.double().rsqrt()
    s0, t0 = g.s.to(dev).long() - 1, g.t.to(dev).long() - 1
    upper = (s0 < t0) if dir == "out" else (s0 > t0)
    keep = (nmap[s0] >= 0) & (upper | (s0 == t0))
    s0, t0 = s0[keep], t0[keep]
    we = (c[s0] * (torch.ones(s0.numel(), dtype=torch.float64, device=dev) if w is None else w[keep].double())
          * c[t0]).float()
    off = s0 != t0
    S = torch.cat([nmap[s0], nmap[t0][off]]) + 1
    T = torch.cat([nmap[t0], nmap[s0][off]]) + 1
    op = GNNGraph(S, T, torch.cat([we, we[off]]), num_nodes=nb)
    p = op.plan()
    diag = 1.0 - c[old] ** 2 if self_loops else torch.ones(nb, dtype=torch.float64, device=dev)
    y32 = torch.empty(nb, dtype=torch.float32, device=dev)

    def apply(x: torch.Tensor) -> torch.Tensor:
        if op.num_edges == 0:
            return diag * x
        x32 = x.float()
        with torch.cuda.device(p.device):
            _lib.check(lib.gnnb_propagate(p.h, 0, _lib.W_MUL_XJ, _lib.SUM, x32.data_ptr(), op.w.data_ptr(), None, None,
                                          1, y32.data_ptr(), _stream(p.device)))
        return diag * x - y32.double()

    K, KEEP = _LMAX_KRYLOV, _LMAX_KEEP
    G = len(segs)
    dots = _SegDots(seg, K + 1, dev)
    V = torch.zeros((K + 1, nb), dtype=torch.float64, device=dev)
    local = torch.arange(nb, device=dev) - seg[node_seg]
    V[0] = ((_splitmix64(local) >> 11) & ((1 << 53) - 1)).double() * 2.0 ** -53 - 0.5
    V[0] /= dots(V[:1], V[0])[:, 0].sqrt()[node_seg]
    Th = np.zeros((G, K, K))                  # the projected matrix: its upper triangle, column j from step j
    theta = np.full(G, np.nan)
    done = np.zeros(G, bool)
    l = 0
    for _ in range(_LMAX_MAXITER):
        Tc = torch.zeros((G, K + 1, K), dtype=torch.float64, device=dev)    # h columns; row K holds beta_j
        for j in range(l, K):
            wv = apply(V[j])
            h = dots(V[:j + 1], wv)                                        # classical Gram-Schmidt, twice
            wv = wv - (V[:j + 1] * h[node_seg].t()).sum(0)
            h2 = dots(V[:j + 1], wv)
            wv = wv - (V[:j + 1] * h2[node_seg].t()).sum(0)
            Tc[:, :j + 1, j] = h + h2
            beta = dots(wv[None], wv)[:, 0].sqrt()
            Tc[:, K, j] = beta
            dead = ~(beta > _LMAX_DEAD)                                    # also NaN: the segment stops here
            V[j + 1] = torch.where(dead[node_seg], torch.zeros_like(wv), wv / beta[node_seg])
        Th_new = Tc.cpu().numpy()                                          # the one synchronisation of the cycle
        Th[:, :, l:] = Th_new[:, :K, l:]
        betas = Th_new[:, K, :]
        # live columns: up to and including the first dead beta of this cycle (its column is real, the next vector
        # is zero); the kept Ritz columns below l carry no beta
        dead_at = np.where(~(betas > _LMAX_DEAD) & (np.arange(K)[None, :] >= l), np.arange(K)[None, :], K)
        first = dead_at.min(1)
        L = np.minimum(first + 1, K)
        Y = np.zeros((G, K, KEEP))
        top = np.zeros((G, KEEP))                                          # the kept Ritz values, Y's columns
        resid = np.zeros(G)
        for Lg in np.unique(L):
            ids = np.nonzero(L == Lg)[0]
            M = np.triu(Th[ids][:, :Lg, :Lg])
            M = M + np.triu(M, 1).transpose(0, 2, 1)
            with np.errstate(invalid="ignore"):
                finite = np.isfinite(M).all((1, 2))
            ev = np.full((len(ids), Lg), np.nan)
            vec = np.zeros((len(ids), Lg, Lg))
            if finite.any():
                ev[finite], vec[finite] = np.linalg.eigh(M[finite])
            new = ~done[ids]
            theta[ids[new]] = ev[new, -1]
            kk = min(KEEP, Lg)
            Y[ids, :Lg, KEEP - kk:] = vec[:, :, Lg - kk:]
            top[ids, KEEP - kk:] = np.nan_to_num(ev[:, Lg - kk:])
            bl = np.where(first[ids] < K, 0.0, betas[ids, K - 1])
            resid[ids] = np.abs(bl * vec[:, Lg - 1, -1])
            resid[ids[~finite]] = 0.0                                      # NaN stays NaN: nothing to converge
        done |= resid <= _LMAX_TOL
        if done.all():
            break
        # thick restart: the KEEP largest Ritz vectors, then the residual vector; converged segments ride along
        Yd = torch.as_tensor(Y, device=dev)
        Vn = torch.zeros_like(V)
        for i in range(KEEP):
            Vn[i] = (V[:K] * Yd[:, :, i][node_seg].t()).sum(0)
        Vn[KEEP] = V[K]
        V = Vn
        Th = np.zeros((G, K, K))
        Th[:, np.arange(KEEP), np.arange(KEEP)] = top
        l = KEEP
    else:
        warnings.warn(f"laplacian_lambda_max: {int((~done).sum())} of {G} graphs did not converge to a Ritz residual "
                      f"of {_LMAX_TOL} in {_LMAX_MAXITER} restarts; their best Ritz values are returned", RuntimeWarning)
    out[[i for i, _, _ in segs]] = torch.as_tensor(theta, device=out.device)


def _lambda_max_segments(g: GNNGraph, seg_ptr: Optional[torch.Tensor], dir: str, self_loops: bool) -> torch.Tensor:
    """float64 lmax of every segment of g (seg_ptr None: the whole graph), no edge joining two segments: those of at
    most _LMAX_SMEM_MAX_NODES nodes in one call of gnnb_laplacian_lambda_max, the larger ones by _lmax_lanczos."""
    p = g.plan()
    n = g.num_nodes
    w = None if g.w is None else g.w.detach().to(device=p.device, dtype=torch.float32).contiguous()
    deg = torch.empty(n, dtype=torch.float32, device=p.device)
    d = _lib.DIR_OUT if dir == "out" else _lib.DIR_IN
    with torch.cuda.device(p.device):
        _lib.check(lib.gnnb_degree(p.h, d, _ptr(w), deg.data_ptr(), _stream(p.device)))
    if self_loops:
        deg = deg + 1
    if bool((deg == 0).any()):
        raise AssertionError(_ISOLATED)
    bounds = [0, n] if seg_ptr is None else seg_ptr.tolist()
    n_seg = len(bounds) - 1
    out = torch.full((n_seg,), float("nan"), dtype=torch.float64, device=p.device)
    bound = min(_LMAX_SMEM_MAX_NODES, _LMAX_KERNEL_MAX_NODES)
    big = [i for i in range(n_seg) if bounds[i + 1] - bounds[i] > bound]
    if len(big) < n_seg:
        info = torch.empty(n_seg, dtype=torch.int32, device=p.device)
        dcode = {"out": _lib.DIR_OUT, "in": _lib.DIR_IN, "both": _lib.DIR_BOTH}[dir]
        with torch.cuda.device(p.device):
            _lib.check(lib.gnnb_laplacian_lambda_max(p.h, _ptr(w), deg.data_ptr(), dcode, int(bool(self_loops)),
                                                     _ptr(seg_ptr), n_seg, out.data_ptr(), info.data_ptr(),
                                                     _stream(p.device)))
    if big:
        _lmax_lanczos(g, w, deg, dir, self_loops, [(i, bounds[i], bounds[i + 1]) for i in big], out)
    return out


def laplacian_lambda_max(g: GNNGraph, T=torch.float32, *, add_self_loops: bool = False, dir: str = "out"):
    """The largest eigenvalue of the normalized Laplacian — query.jl:598-610: that of Symmetric(L) (the reference's
    `_eigmax`), L = normalized_laplacian(g, T; add_self_loops, dir), whose upper triangle it reads: S[i, j] = S[j, i] =
    L[i, j] for i < j, S[i, i] = L[i, i].  On a directed graph that is not the eigenvalue of (L + L') / 2; the lower
    triangle counts only through the degrees.  dir = "out" takes A (A[s, t] the summed weight of the edges s -> t,
    self loops counted once); "in" and "both" take A', as the reference's adjacency_matrix does for every dir but :out.
    A zero degree raises the reference's AssertionError.  Not differentiable.

    One graph (num_graphs == 1): a Python float, rounded to T.  A batch: a float64 tensor of num_graphs values on g's
    device, graph i from getgraph(g, i): an edge between two graphs is dropped and does not count in either degree.
    An unsorted indicator or such an edge costs one relabelled copy of the graph (a stable sort of the nodes by graph,
    one fresh plan).  A graph without nodes raises ValueError naming it.
      * Graphs of at most _LMAX_SMEM_MAX_NODES (169) nodes: gnnb_laplacian_lambda_max, all in one call.  S is built in
        shared memory in float64 and its eigenvalue found by Householder tridiagonalisation and Sturm bisection to the
        last bit; one warp per graph of up to 32 nodes, one CTA per larger one, the same bits either way.
      * Larger graphs, all together: thick-restart Lanczos (Krylov dimension 32, 16 Ritz vectors kept) on float64
        vectors, S applied through one fused propagate at D = 1 over an operator graph of S's off-diagonal entries,
        deterministic segmented dot products, one device-to-host synchronisation per restart.  A graph has converged
        when its Ritz residual is at most 1e-6; after 100 restarts the best Ritz values are returned with one
        RuntimeWarning counting the graphs that did not converge."""
    homogeneous_only(g, "laplacian_lambda_max")
    _check_dir(dir)
    _check_float_type(T, "laplacian_lambda_max")
    g = _on_device(g)
    n, dev = g.num_nodes, g.s.device
    if g.num_graphs == 1:
        if n == 0:
            raise ValueError("laplacian_lambda_max: the graph has no nodes")
        v = float(_lambda_max_segments(g, None, dir, add_self_loops)[0])
        return float(torch.tensor(v, dtype=T))
    G = g.num_graphs
    if g.graph_indicator is None:
        raise ValueError(f"laplacian_lambda_max: a batch of {G} graphs needs a graph_indicator")
    gi = torch.as_tensor(g.graph_indicator).to(device=dev, dtype=torch.int64).reshape(-1)
    assert gi.numel() == n, f"graph_indicator has {gi.numel()} entries for {n} nodes"
    if n and (int(gi.min()) < 1 or int(gi.max()) > G):
        raise ValueError(f"laplacian_lambda_max: graph_indicator values must lie in 1:{G}")
    counts = torch.bincount(gi, minlength=G + 1)[1:]
    empty = (counts == 0).nonzero().reshape(-1)
    if empty.numel():
        raise ValueError(f"laplacian_lambda_max: graph {int(empty[0]) + 1} has no nodes (getgraph fails on it in the "
                         f"reference)")
    seg_ptr = torch.zeros(G + 1, dtype=torch.int64, device=dev)
    torch.cumsum(counts, 0, out=seg_ptr[1:])
    s0, t0 = g.s.long() - 1, g.t.long() - 1
    sorted_ = bool((gi[1:] >= gi[:-1]).all())
    crossing = (gi[s0] != gi[t0]) if g.num_edges else torch.zeros(0, dtype=torch.bool, device=dev)
    if not sorted_ or bool(crossing.any()):                    # getgraph semantics: relabel, drop crossing edges
        order = torch.sort(gi, stable=True).indices
        inv = torch.empty_like(order)
        inv[order] = torch.arange(n, device=dev)
        keep = ~crossing
        g = GNNGraph(inv[s0[keep]] + 1, inv[t0[keep]] + 1, None if g.w is None else g.w.detach()[keep], num_nodes=n)
    return _lambda_max_segments(g, seg_ptr, dir, add_self_loops)
