"""Geometric and temporal graph generators on the device:

    knn_graph(points, k; graph_indicator, self_loops=false, dir=:in, kws...)      GNNGraphs/src/generate.jl:112-145
    radius_graph(points, r; graph_indicator, self_loops=false, dir=:in, kws...)   GNNGraphs/src/generate.jl:196-222
    rand_temporal_radius_graph(n, T, speed, r; self_loops, dir, kws...)           GNNGraphs/src/generate.jl:265-284
    rand_temporal_hyperbolic_graph(n, T; α, R, speed, ζ=1, self_loop, kws...)     GNNGraphs/src/generate.jl:287-380

The neighbour search is csrc/knn.cu: brute force within each graph of the batch, exact fp32 distances
d2(i, j) = Σ_f (p_i[f] - p_j[f])² summed in ascending f with every operation rounded on its own, a NaN distance
counting as +Inf.  What stays here is device-side bookkeeping: segment offsets from `graph_indicator`, the stable sort
of an unsorted indicator and its inverse, and the COO of `to_coo(adj_list; dir)` (GNNGraphs/src/convert.jl:97-116):
edges grouped by centre i ascending, then in row order; dir="in" gives s = neighbour, t = centre, dir="out" swaps them.

Three deliberate differences from the reference:
1. Neighbour order.  The reference asks NearestNeighbors.jl for `sortres=false` and keeps each row in tree order.  Here a
   knn row is in ascending (d2, j) and a radius row in ascending j, so the output is a function of the points alone.
2. Duplicate points.  The reference takes the k + 1 nearest and then removes self loops, so a node whose duplicates hide
   itself keeps k + 1 edges.  Here the node itself is never a candidate without self loops: every node has exactly k.
3. Small graphs.  The reference asserts only that each graph has >= k nodes; a graph of exactly k nodes without self
   loops then silently gets an edge to another graph.  Here a graph needs k + 1 nodes (k with self loops), or
   AssertionError.
Graphs of a batch are separated exactly (candidates come from the point's own graph), not by the reference's dummy
coordinate, and the points are not rescaled.

The temporal generators move n nodes through T snapshots with csrc/tgen.cu (one thread per node, fp64 state, the
reference's arithmetic line by line) and then find every snapshot's edges in one count and one fill over the T
snapshots as T segments of one batch: gnnb_radius_count / _fill on the fp32 points, or gnnb_hyperbolic_count / _fill
on the fp64 records (cosh ζr, sinh ζr, cos θ, sin θ).  The draws are u(i, τ, k) = (splitmix64(K + c) >> 11) 2^-53,
K = splitmix64(seed), c = ((τ n + i) << 1) | k (include/gnnb200.h).  Deliberate differences from the reference:
1. Randomness.  The draws come from that seeded stream, not from Julia's `rand`: runs are reproducible across GPUs.
   Without a `seed` one is drawn from torch's default generator.
2. Radius precision.  The radius search runs on the fp32 rounding of the positions, with radius_graph's exact contract;
   the reference searches Float64 points.  The positions themselves evolve in fp64.
3. Hyperbolic decision.  An edge is x <= cosh(ζR) with x = C_i C_j - (S_i S_j)(c_i c_j + s_i s_j), each operation
   rounded on its own, not acosh(x)/ζ <= R.  The two differ only where x lies within rounding of the threshold.  An x
   that rounds below 1 for two close nodes is an edge here; the reference throws a DomainError from acosh there.
4. kws.  The hyperbolic generator passes kws to every snapshot's GNNGraph; the reference ignores them.
5. Row order.  Rows are in ascending node id, as in radius_graph, not in BallTree order.
"""
from __future__ import annotations

import ctypes as C
import math

import numpy as np
import torch

from . import _lib
from . import graph as _graph
from ._lib import lib
from .graph import GNNGraph, _stream, rows
from .linkpred import _seed
from .temporal import TemporalSnapshotsGNNGraph


def _points(points) -> torch.Tensor:
    """(d, n) Julia-layout points -> (n, d) contiguous fp32 rows on the compute device"""
    x = points if isinstance(points, torch.Tensor) else torch.as_tensor(np.asarray(points))
    if x.dim() != 2:
        raise ValueError("points must be a (d, n) matrix")
    dev = _graph._compute_device(x)
    return rows(x).to(device=dev, dtype=torch.float32).contiguous()


def _segments(graph_indicator, n: int, dev):
    """(order or None, seg_ptr or None, num_graphs, indicator on dev).  `order` stable-sorts the nodes by graph when the
    indicator is not already non-decreasing."""
    if graph_indicator is None:
        return None, None, 1, None
    gi = graph_indicator if isinstance(graph_indicator, torch.Tensor) else torch.as_tensor(np.asarray(graph_indicator))
    assert not gi.is_floating_point() and gi.dtype != torch.bool, "graph_indicator must hold integers"
    gi = gi.reshape(-1)
    assert gi.numel() == n, f"graph_indicator has {gi.numel()} entries for {n} points"
    g = gi.to(device=dev, dtype=torch.int64)
    if n == 0:
        return None, None, 0, gi
    order = None
    if not bool((g[1:] >= g[:-1]).all()):
        order = torch.sort(g, stable=True).indices
        g = g[order]
    _, counts = torch.unique_consecutive(g, return_counts=True)
    seg_ptr = torch.zeros(counts.numel() + 1, dtype=torch.int64, device=dev)
    torch.cumsum(counts, 0, out=seg_ptr[1:])
    return order, seg_ptr, int(g.max()), gi


def _graph_from_rows(centre: torch.Tensor, nbr: torch.Tensor, n: int, dir: str, num_graphs: int, gi, kws) -> GNNGraph:
    s, t = nbr + 1, centre + 1
    if dir == "out":
        s, t = t, s
    return GNNGraph(s, t, num_nodes=n, num_graphs=num_graphs, graph_indicator=gi, **kws)


def knn_graph(points, k: int, *, graph_indicator=None, self_loops: bool = False, dir: str = "in", **kws) -> GNNGraph:
    """GNNGraphs/src/generate.jl:112-145: node i gets an edge from each of its k nearest points of its own graph (to
    them with dir="out"), nearest first, ties broken by the smaller node id."""
    assert dir in ("in", "out"), 'dir must be "in" or "out"'
    x = _points(points)
    n, d = int(x.shape[0]), int(x.shape[1])
    dev = x.device
    order, seg_ptr, num_graphs, gi = _segments(graph_indicator, n, dev)
    k = int(k)
    if order is not None:
        x = x[order].contiguous()
    nbr = torch.empty((n, max(k, 0)), dtype=torch.int32, device=dev)
    n_seg = 1 if seg_ptr is None else int(seg_ptr.numel()) - 1
    with torch.cuda.device(dev):                                # a too-small graph: GNNB_ESIZE -> AssertionError
        _lib.check(lib.gnnb_knn(x.data_ptr(), n, d, None if seg_ptr is None else seg_ptr.data_ptr(), n_seg, k,
                                int(bool(self_loops)), nbr.data_ptr(), _stream(dev)))
    nbr = nbr.to(torch.int64)
    if order is not None:
        inv = torch.empty_like(order)
        inv[order] = torch.arange(n, device=dev)
        nbr = order[nbr[inv]]                                   # rows back in node order, ids back to node ids
    centre = torch.arange(n, device=dev).repeat_interleave(k)
    return _graph_from_rows(centre, nbr.reshape(-1), n, dir, num_graphs, gi, kws)


def radius_graph(points, r: float, *, graph_indicator=None, self_loops: bool = False, dir: str = "in",
                 **kws) -> GNNGraph:
    """GNNGraphs/src/generate.jl:196-222: node i gets an edge from every point of its own graph within distance r
    (sqrt(d2) <= r), in ascending node id."""
    assert dir in ("in", "out"), 'dir must be "in" or "out"'
    r = float(r)
    if math.isnan(r) or r < 0:
        raise ValueError(f"radius r = {r} must be >= 0 and not NaN")
    x = _points(points)
    n, d = int(x.shape[0]), int(x.shape[1])
    dev = x.device
    order, seg_ptr, num_graphs, gi = _segments(graph_indicator, n, dev)
    if order is not None:
        x = x[order].contiguous()
    n_seg = 1 if seg_ptr is None else int(seg_ptr.numel()) - 1
    sp = None if seg_ptr is None else seg_ptr.data_ptr()
    offsets = torch.zeros(n + 1, dtype=torch.int64, device=dev)
    total = C.c_int64(0)
    sl = int(bool(self_loops))
    with torch.cuda.device(dev):
        _lib.check(lib.gnnb_radius_count(x.data_ptr(), n, d, sp, n_seg, r, sl, offsets.data_ptr(), C.byref(total),
                                         _stream(dev)))
        nbr = torch.empty(int(total.value), dtype=torch.int32, device=dev)
        if total.value:
            _lib.check(lib.gnnb_radius_fill(x.data_ptr(), n, d, sp, n_seg, r, sl, offsets.data_ptr(), nbr.data_ptr(),
                                            int(total.value), _stream(dev)))
    nbr = nbr.to(torch.int64)
    counts = offsets[1:] - offsets[:-1]
    if order is None:
        centre = torch.arange(n, device=dev).repeat_interleave(counts)
        return _graph_from_rows(centre, nbr, n, dir, num_graphs, gi, kws)
    inv = torch.empty_like(order)
    inv[order] = torch.arange(n, device=dev)
    counts_out = counts[inv]                                    # row lengths in node order
    centre = torch.arange(n, device=dev).repeat_interleave(counts_out)
    start_out = torch.cumsum(counts_out, 0) - counts_out
    src = offsets[:-1][inv][centre] + (torch.arange(nbr.numel(), device=dev) - start_out[centre])
    return _graph_from_rows(centre, order[nbr[src]], n, dir, num_graphs, gi, kws)


# ---------------------------------------------------------------------------------------------- temporal generators
def _temporal_setup(n, T, device):
    """(n, T, device) after the checks shared by both generators.  T * n >= 2^31 is refused before any device work
    (the entries' GNNB_ESIZE, an AssertionError like every size limit of the library)."""
    n, T = int(n), int(T)
    if n < 0 or T < 0:
        raise ValueError(f"n = {n} and T = {T} must be >= 0")
    if n * T >= 2 ** 31:
        raise AssertionError(f"T * n = {T} * {n} must be < 2^31")
    dev = torch.device(device) if device is not None else _graph._compute_device(torch.empty(0))
    return n, T, dev


def _snapshots(offsets, nbr, n: int, T: int, dir: str, kws, weight: bool) -> TemporalSnapshotsGNNGraph:
    """Snapshot t = rows t*n .. t*n + n - 1 of the flat rows, ids shifted by t*n.  One read-back of the T + 1 snapshot
    edge offsets."""
    dev = nbr.device
    total = int(nbr.numel())
    counts = offsets[1:] - offsets[:-1]
    centre = torch.arange(n * T, device=dev).repeat_interleave(counts, output_size=total)
    nbr = nbr.to(torch.int64)
    eoff = offsets[torch.arange(T + 1, device=dev) * n].tolist()
    snaps = []
    for t in range(T):
        a, b = eoff[t], eoff[t + 1]
        kw = dict(kws)
        if weight:
            kw["w"] = torch.ones(b - a, dtype=torch.float32, device=dev)
        snaps.append(_graph_from_rows(centre[a:b] - t * n, nbr[a:b] - t * n, n, dir, 1, None, kw))
    return TemporalSnapshotsGNNGraph(snaps)


def _empty_snapshots(n: int, T: int, dev, dir: str, kws, weight: bool) -> TemporalSnapshotsGNNGraph:
    e = torch.zeros(0, dtype=torch.int64, device=dev)
    return _snapshots(torch.zeros(n * T + 1, dtype=torch.int64, device=dev), e, n, T, dir, kws, weight)


def rand_temporal_radius_graph(n: int, T: int, speed: float, r: float, *, self_loops: bool = False, dir: str = "in",
                               seed=None, device=None, **kws) -> TemporalSnapshotsGNNGraph:
    """GNNGraphs/src/generate.jl:265-284: n points start uniform in the unit square; snapshot t is radius_graph(points,
    r; self_loops, dir, kws...) of the positions after t - 1 moves.  A move displaces every point by ρ (cos θ, sin θ),
    ρ uniform in [-speed, speed), θ uniform in [0, 2π), and reflects it at the square's border (as the reference
    writes it: with speed > 1 a point can leave the square).  `seed` makes the call reproducible (see the module
    docstring for the stream)."""
    assert dir in ("in", "out"), 'dir must be "in" or "out"'
    speed, r = float(speed), float(r)
    if not math.isfinite(speed):
        raise ValueError(f"speed = {speed} must be finite")
    if math.isnan(r) or r < 0:
        raise ValueError(f"radius r = {r} must be >= 0 and not NaN")
    n, T, dev = _temporal_setup(n, T, device)
    seed = _seed(seed)
    if n * T == 0:
        return _empty_snapshots(n, T, dev, dir, kws, False)
    N = n * T
    pts = torch.empty((N, 2), dtype=torch.float32, device=dev)
    seg_ptr = torch.arange(T + 1, dtype=torch.int64, device=dev) * n
    offsets = torch.zeros(N + 1, dtype=torch.int64, device=dev)
    total = C.c_int64(0)
    sl = int(bool(self_loops))
    with torch.cuda.device(dev):
        _lib.check(lib.gnnb_temporal_radius_points(n, T, speed, seed, pts.data_ptr(), _stream(dev)))
        _lib.check(lib.gnnb_radius_count(pts.data_ptr(), N, 2, seg_ptr.data_ptr(), T, r, sl, offsets.data_ptr(),
                                         C.byref(total), _stream(dev)))
        nbr = torch.empty(int(total.value), dtype=torch.int32, device=dev)
        if total.value:
            _lib.check(lib.gnnb_radius_fill(pts.data_ptr(), N, 2, seg_ptr.data_ptr(), T, r, sl, offsets.data_ptr(),
                                            nbr.data_ptr(), int(total.value), _stream(dev)))
    return _snapshots(offsets, nbr, n, T, dir, kws, False)


def rand_temporal_hyperbolic_graph(n: int, T: int, *, α, R, speed, ζ=1, self_loop: bool = False, seed=None,
                                   device=None, **kws) -> TemporalSnapshotsGNNGraph:
    """GNNGraphs/src/generate.jl:287-297, 340-380: n nodes in a hyperbolic disk of radius R with quasi-uniform radial
    density (α), connected when their hyperbolic distance (curvature ζ) is at most R.  Between snapshots every node's
    radial probability and angle take a uniform step in [-speed, speed), the probability folded back into [0, 1] as the
    reference folds it.  Each snapshot is GNNGraph(adj) of the symmetric adjacency: edges for each centre j ascending,
    its neighbours i ascending, s = i, t = j, with a weight vector of ones (convert.jl:85).  `seed` makes the call
    reproducible (see the module docstring for the stream and for how the decision differs from acosh(x)/ζ <= R)."""
    assert int(T) > 1, "The number of snapshots must be greater than 1"
    assert α > 0, "α must be greater than 0"
    alpha, R, speed, zeta = float(α), float(R), float(speed), float(ζ)
    for name, v in (("α", alpha), ("R", R), ("speed", speed), ("ζ", zeta)):
        if not math.isfinite(v):
            raise ValueError(f"{name} = {v} must be finite")
    if zeta <= 0:
        raise ValueError(f"ζ = {zeta} must be > 0")
    if R < 0:
        raise ValueError(f"R = {R} must be >= 0")
    try:
        math.cosh(alpha * R)
        x_max = math.cosh(zeta * R)
    except OverflowError:
        raise ValueError(f"cosh(α R) = cosh({alpha * R}) or cosh(ζ R) = cosh({zeta * R}) overflows float64") from None
    n, T, dev = _temporal_setup(n, T, device)
    seed = _seed(seed)
    if n == 0:
        return _empty_snapshots(n, T, dev, "in", kws, True)
    N = n * T
    rec = torch.empty((N, 4), dtype=torch.float64, device=dev)
    seg_ptr = torch.arange(T + 1, dtype=torch.int64, device=dev) * n
    offsets = torch.zeros(N + 1, dtype=torch.int64, device=dev)
    total = C.c_int64(0)
    sl = int(bool(self_loop))
    with torch.cuda.device(dev):
        _lib.check(lib.gnnb_temporal_hyperbolic_records(n, T, alpha, R, speed, zeta, seed, rec.data_ptr(),
                                                        _stream(dev)))
        _lib.check(lib.gnnb_hyperbolic_count(rec.data_ptr(), N, seg_ptr.data_ptr(), T, x_max, sl, offsets.data_ptr(),
                                             C.byref(total), _stream(dev)))
        nbr = torch.empty(int(total.value), dtype=torch.int32, device=dev)
        if total.value:
            _lib.check(lib.gnnb_hyperbolic_fill(rec.data_ptr(), N, seg_ptr.data_ptr(), T, x_max, sl, offsets.data_ptr(),
                                                nbr.data_ptr(), int(total.value), _stream(dev)))
    return _snapshots(offsets, nbr, n, T, "in", kws, True)
