"""Geometric graph generators on the device:

    knn_graph(points, k; graph_indicator, self_loops=false, dir=:in, kws...)      GNNGraphs/src/generate.jl:112-145
    radius_graph(points, r; graph_indicator, self_loops=false, dir=:in, kws...)   GNNGraphs/src/generate.jl:196-222

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
