"""Graph-level readout on the same segment machinery (SURVEY.md §8f rank 2):

    reduce_nodes / reduce_edges        GNNlib/src/utils.jl:12-42
    softmax_nodes / softmax_edges      GNNlib/src/utils.jl:44-72
    broadcast_nodes / broadcast_edges  GNNlib/src/utils.jl:105-121
    global_pool, global_attention_pool GNNlib/src/layers/pool.jl:3-12
    set2set_pool, Set2Set              GNNlib/src/layers/pool.jl:29-43, GraphNeuralNetworks/src/layers/pool.jl:126-162

`NNlib.scatter(aggr, x, graph_indicator)` is a segmented reduce whose "edges" are the nodes and whose "targets" are the
graphs: a bipartite plan (gnnb_graph_create with num_src = #items, num_dst = #graphs) lets the library's scatter /
gather / neighbourhood-softmax kernels (and their pullbacks) do all of it.  Set2Set's attention runs on the same plan
through its own fused kernel (csrc/set2set.cu).
"""
from __future__ import annotations

import ctypes as C
import operator

import torch

from . import _lib
from . import graph as _graph
from ._lib import lib
from .graph import GNNGraph, _Plan, _stream, graph_indicator, rows, unrows
from .layers import _LSTMCell
from .msgpass import _EdgeSoftmaxFn, _GatherFn, _ScatterFn, _aggr_code, _f32


class _IndicatorPlan:
    """plan of the bipartite graph  item k -> segment indicator[k]  (1-based, like graph_indicator)"""

    def __init__(self, indicator: torch.Tensor, num_segments: int, device):
        self.n_items = int(indicator.numel())
        self.n_segments = int(num_segments)
        ind = indicator.to(device=device, dtype=torch.int64).contiguous()
        src = torch.arange(1, self.n_items + 1, dtype=torch.int64, device=device)
        h = C.c_void_p()
        with torch.cuda.device(device):
            _lib.check(lib.gnnb_graph_create(C.byref(h), src.data_ptr(), ind.data_ptr(), self.n_items, self.n_items,
                                             self.n_segments, 8, 1, 1, _stream(device)))
        self.plan = _Plan(h.value, torch.device(device))


def _indicator_plan(g: GNNGraph, edges: bool) -> _IndicatorPlan:
    key = "_gi_plan_e" if edges else "_gi_plan_n"
    p = getattr(g, key, None)
    if p is None:
        dev = g.plan().device
        p = _IndicatorPlan(graph_indicator(g, edges=edges), g.num_graphs, dev)
        setattr(g, key, p)
    return p


def _reduce(aggr, ip: _IndicatorPlan, x: torch.Tensor) -> torch.Tensor:
    assert x.shape[-1] == ip.n_items
    r = _ScatterFn.apply(_f32(rows(x), ip.plan.device), ip.plan, _lib.DST, _aggr_code(aggr), ip.n_segments)
    return unrows(r)


def _broadcast(ip: _IndicatorPlan, x: torch.Tensor) -> torch.Tensor:
    assert x.shape[-1] == ip.n_segments
    r = _GatherFn.apply(_f32(rows(x), ip.plan.device), ip.plan, _lib.DST, ip.n_items)
    return unrows(r)


def reduce_nodes(aggr, g, x: torch.Tensor) -> torch.Tensor:
    """reduce_nodes(aggr, g, x) and reduce_nodes(aggr, indicator, x) — GNNlib/src/utils.jl:12-29."""
    if isinstance(g, GNNGraph):
        assert x.shape[-1] == g.num_nodes
        return _reduce(aggr, _indicator_plan(g, False), x)
    ind = g
    dev = _graph._compute_device(x)
    return _reduce(aggr, _IndicatorPlan(ind, int(ind.max()), dev), x)


def reduce_edges(aggr, g: GNNGraph, e: torch.Tensor) -> torch.Tensor:
    """GNNlib/src/utils.jl:31-42."""
    assert e.shape[-1] == g.num_edges
    return _reduce(aggr, _indicator_plan(g, True), e)


def softmax_nodes(g: GNNGraph, x: torch.Tensor) -> torch.Tensor:
    """Graph-wise softmax of the node features — GNNlib/src/utils.jl:44-57 (fused neighbourhood-softmax kernel)."""
    assert x.shape[-1] == g.num_nodes
    ip = _indicator_plan(g, False)
    return unrows(_EdgeSoftmaxFn.apply(_f32(rows(x), ip.plan.device), ip.plan))


def softmax_edges(g: GNNGraph, e: torch.Tensor) -> torch.Tensor:
    """Graph-wise softmax of the edge features — GNNlib/src/utils.jl:59-72: the reference's own sequence, including the
    `den .+ eps(eltype(e))` it adds only here."""
    assert e.shape[-1] == g.num_edges
    ip = _indicator_plan(g, True)
    mx = _broadcast(ip, _reduce(max, ip, e))
    num = torch.exp(e - mx)
    den = _broadcast(ip, _reduce(operator.add, ip, num))
    return num / (den + torch.finfo(e.dtype).eps)


def broadcast_nodes(g: GNNGraph, x: torch.Tensor) -> torch.Tensor:
    """GNNlib/src/utils.jl:105-110."""
    assert x.shape[-1] == g.num_graphs
    return _broadcast(_indicator_plan(g, False), x)


def broadcast_edges(g: GNNGraph, x: torch.Tensor) -> torch.Tensor:
    """GNNlib/src/utils.jl:116-121."""
    assert x.shape[-1] == g.num_graphs
    return _broadcast(_indicator_plan(g, True), x)


def global_pool(l, g: GNNGraph, x: torch.Tensor) -> torch.Tensor:
    """GNNlib/src/layers/pool.jl:3-5."""
    return reduce_nodes(l.aggr, g, x)


def global_attention_pool(l, g: GNNGraph, x: torch.Tensor) -> torch.Tensor:
    """GNNlib/src/layers/pool.jl:7-12."""
    alpha = softmax_nodes(g, l.fgate(x))
    feats = alpha * l.ffeat(x)
    return reduce_nodes(operator.add, g, feats)


# Feature sizes up to this go through the fused attention (gnnb_set2set_attend, csrc/set2set.cu); larger ones through
# broadcast_nodes / softmax_nodes / reduce_nodes.  Must not exceed GNNB_SET2SET_MAX_D (include/gnnb200.h).
_SET2SET_MAX_D = 1024      # GNNB_SET2SET_MAX_D


class _Set2SetAttendFn(torch.autograd.Function):
    """r = softmax-weighted sum of the rows of x per graph, with the query q of the graph (gnnb_set2set_attend) on the
    graph-indicator plan, where edge k is node k: the per-edge dxe of the pullback is dx.  Keeps q, r and the G-sized
    softmax statistics besides x."""

    @staticmethod
    def forward(ctx, x_rows, q_rows, plan):
        G, D = q_rows.shape
        r = torch.empty((G, D), dtype=torch.float32, device=x_rows.device)
        smax = torch.empty(G, dtype=torch.float32, device=x_rows.device)
        ssum = torch.empty(G, dtype=torch.float32, device=x_rows.device)
        with torch.cuda.device(plan.device):
            _lib.check(lib.gnnb_set2set_attend(plan.h, x_rows.data_ptr(), q_rows.data_ptr(), D, r.data_ptr(),
                                               smax.data_ptr(), ssum.data_ptr(), _stream(plan.device)))
        ctx.plan = plan
        ctx.save_for_backward(x_rows, q_rows, r, smax, ssum)
        return r

    @staticmethod
    def backward(ctx, dr):
        x_rows, q_rows, r, smax, ssum = ctx.saved_tensors
        dr = dr.contiguous()
        dx = torch.empty_like(x_rows)
        dq = torch.empty_like(q_rows)
        with torch.cuda.device(ctx.plan.device):
            _lib.check(lib.gnnb_set2set_attend_bwd(ctx.plan.h, x_rows.data_ptr(), q_rows.data_ptr(), r.data_ptr(),
                                                   smax.data_ptr(), ssum.data_ptr(), dr.data_ptr(), q_rows.shape[1],
                                                   dx.data_ptr(), dq.data_ptr(), _stream(ctx.plan.device)))
        return dx, dq, None


def set2set_pool(l, g: GNNGraph, x: torch.Tensor) -> torch.Tensor:
    """GNNlib/src/layers/pool.jl:29-43: num_iters rounds of
        q, state = lstm(qstar, state);  α = softmax_nodes(g, sum(broadcast_nodes(g, q) .* x, dims = 1))
        r = reduce_nodes(+, g, x .* α);  qstar = vcat(q, r)
    starting from qstar = 0 (2·n_in, num_graphs) and zero (h, c) vectors of length n_in.  Returns qstar.
    For n_in <= _SET2SET_MAX_D the attention of a round is one fused pass over x (forward and pullback), which keeps only
    graph-sized state for the backward; a graph with no nodes gets r = 0."""
    assert x.shape[-1] == g.num_nodes, \
        f"Got {x.shape[-1]} as last dimension size instead of num_nodes={g.num_nodes}"
    n_in = x.shape[0]
    assert x.dim() == 2 and 2 * n_in == l.lstm.Wi.shape[1], \
        f"x has {n_in} rows; this Set2Set takes {l.lstm.Wi.shape[1] // 2}"
    qstar = torch.zeros((2 * n_in, g.num_graphs), dtype=x.dtype, device=x.device)
    h = torch.zeros(n_in, dtype=l.lstm.Wh.dtype, device=l.lstm.Wh.device)
    state = (h, torch.zeros_like(h))
    ip = _indicator_plan(g, False)
    fused = n_in <= _SET2SET_MAX_D
    if fused:
        x_rows = _f32(rows(x), ip.plan.device)
    for _ in range(int(l.num_iters)):
        q, state = l.lstm(qstar, state)
        if fused:
            r = unrows(_Set2SetAttendFn.apply(x_rows, _f32(rows(q), ip.plan.device), ip.plan))
        else:
            alpha = softmax_nodes(g, (broadcast_nodes(g, q) * x).sum(dim=0, keepdim=True))
            r = reduce_nodes(operator.add, g, x * alpha)
        qstar = torch.cat([q, r], dim=0)
    return qstar


class Set2Set(torch.nn.Module):
    """Set2Set(n_in, n_iters, n_layers = 1) — GraphNeuralNetworks/src/layers/pool.jl:126-162: an LSTMCell(2·n_in => n_in)
    and num_iters; forward(g, x) returns the (2·n_in, num_graphs) readout (set2set_pool)."""

    def __init__(self, n_in: int, n_iters: int, n_layers: int = 1, device=None):
        super().__init__()
        if n_layers != 1:
            raise AssertionError("multiple layers not implemented yet")
        self.lstm = _LSTMCell(2 * n_in, n_in, device=device)
        self.num_iters = int(n_iters)

    def forward(self, g: GNNGraph, x: torch.Tensor) -> torch.Tensor:
        return set2set_pool(self, g, x)
