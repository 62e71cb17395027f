"""Graph-level readout on the same segment machinery (SURVEY.md §8f rank 2):

    reduce_nodes / reduce_edges        GNNlib/src/utils.jl:12-42
    softmax_nodes / softmax_edges      GNNlib/src/utils.jl:44-72
    broadcast_nodes / broadcast_edges  GNNlib/src/utils.jl:105-121
    global_pool, global_attention_pool GNNlib/src/layers/pool.jl:3-12
    GlobalPool, GlobalAttentionPool    GraphNeuralNetworks/src/layers/pool.jl:1-99
    set2set_pool, Set2Set              GNNlib/src/layers/pool.jl:29-43, GraphNeuralNetworks/src/layers/pool.jl:126-162
    topk_index, topk_pool, TopKPool    GNNlib/src/layers/pool.jl:14-27, GraphNeuralNetworks/src/layers/pool.jl:101-123

`NNlib.scatter(aggr, x, graph_indicator)` is a segmented reduce whose "edges" are the nodes and whose "targets" are the
graphs: a bipartite plan (gnnb_graph_create with num_src = #items, num_dst = #graphs) lets the library's scatter /
gather / neighbourhood-softmax kernels (and their pullbacks) do all of it.  Set2Set's attention runs on the same plan
through its own fused kernel (csrc/set2set.cu), and so does global_attention_pool with a gate of one row (the same
kernel with the gate as the score).  Top-k pooling selects per graph by a segmented radix select and gates
the kept rows in one pass (csrc/topk.cu).
"""
from __future__ import annotations

import ctypes as C
import numbers
import operator

import torch

from . import _lib
from . import graph as _graph
from ._lib import lib
from .basic import GNNLayer
from .graph import GNNGraph, _Plan, _ptr, _stream, graph_indicator, node_features, rows, unrows
from .layers import _LSTMCell, glorot_uniform, identity
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


# Feature sizes up to this go through the fused attention (gnnb_set2set_attend, csrc/set2set.cu); larger ones through
# broadcast_nodes / softmax_nodes / reduce_nodes.  Must not exceed GNNB_SET2SET_MAX_D (include/gnnb200.h).
_SET2SET_MAX_D = 1024      # GNNB_SET2SET_MAX_D
# The same bound for global_attention_pool's fused route (gnnb_attention_pool); wider ffeat outputs compose.
_ATTENTION_POOL_MAX_D = 1024      # GNNB_SET2SET_MAX_D


class _AttentionPoolFn(torch.autograd.Function):
    """u = Σ_k softmax(gate)_k f_k per graph (gnnb_attention_pool) on the graph-indicator plan, where edge k is node k:
    the per-edge dfe and dgate_e of the pullback are df and dgate.  Keeps f, gate, u and the G-sized softmax
    statistics."""

    @staticmethod
    def forward(ctx, f_rows, gate, plan, G):
        D = f_rows.shape[1]
        u = torch.empty((G, D), dtype=torch.float32, device=f_rows.device)
        smax = torch.empty(G, dtype=torch.float32, device=f_rows.device)
        ssum = torch.empty(G, dtype=torch.float32, device=f_rows.device)
        with torch.cuda.device(plan.device):
            _lib.check(lib.gnnb_attention_pool(plan.h, f_rows.data_ptr(), gate.data_ptr(), D, u.data_ptr(),
                                               smax.data_ptr(), ssum.data_ptr(), _stream(plan.device)))
        ctx.plan = plan
        ctx.save_for_backward(f_rows, gate, u, smax, ssum)
        return u

    @staticmethod
    def backward(ctx, du):
        f_rows, gate, u, smax, ssum = ctx.saved_tensors
        du = du.contiguous()
        df = torch.empty_like(f_rows)
        dgate = torch.empty_like(gate)
        with torch.cuda.device(ctx.plan.device):
            _lib.check(lib.gnnb_attention_pool_bwd(ctx.plan.h, f_rows.data_ptr(), gate.data_ptr(), u.data_ptr(),
                                                   smax.data_ptr(), ssum.data_ptr(), du.data_ptr(), f_rows.shape[1],
                                                   df.data_ptr(), dgate.data_ptr(), _stream(ctx.plan.device)))
        return df, dgate, None, None


def global_attention_pool(l, g: GNNGraph, x: torch.Tensor) -> torch.Tensor:
    """GNNlib/src/layers/pool.jl:7-12: u = reduce_nodes(+, g, softmax_nodes(g, fgate(x)) .* ffeat(x)).
    A gate of one row and a 2-D ffeat(x) of 1 to _ATTENTION_POOL_MAX_D rows take one fused pass over ffeat(x), forward
    and pullback (a graph with no nodes gets u = 0); any other shapes (a gate per channel, wider features) compose
    softmax_nodes and reduce_nodes."""
    gate = l.fgate(x)
    feats = l.ffeat(x)
    if gate.dim() == 2 and gate.shape[0] == 1 and feats.dim() == 2 and 1 <= feats.shape[0] <= _ATTENTION_POOL_MAX_D:
        assert gate.shape[-1] == feats.shape[-1] == g.num_nodes, \
            f"fgate(x) has {gate.shape[-1]} and ffeat(x) {feats.shape[-1]} columns; the graph has {g.num_nodes} nodes"
        ip = _indicator_plan(g, False)
        dev = ip.plan.device
        u = _AttentionPoolFn.apply(_f32(rows(feats), dev), _f32(gate.reshape(-1), dev), ip.plan, ip.n_segments)
        return unrows(u)
    alpha = softmax_nodes(g, gate)
    return reduce_nodes(operator.add, g, alpha * feats)


class GlobalPool(GNNLayer):
    """GlobalPool(aggr) — GraphNeuralNetworks/src/layers/pool.jl:1-41: l(g, x) = reduce_nodes(aggr, g, x);
    l(g) = GNNGraph(g, gdata=l(g, node_features(g)))."""

    def __init__(self, aggr):
        super().__init__()
        self.aggr = aggr

    def forward(self, g: GNNGraph, x: torch.Tensor) -> torch.Tensor:
        return global_pool(self, g, x)

    def graph_forward(self, g: GNNGraph) -> GNNGraph:
        return GNNGraph(g, gdata=self(g, node_features(g)))


class GlobalAttentionPool(GNNLayer):
    """GlobalAttentionPool(fgate, ffeat=identity) — GraphNeuralNetworks/src/layers/pool.jl:43-99: l(g, x) =
    global_attention_pool; l(g) = GNNGraph(g, gdata=l(g, node_features(g))).  fgate and ffeat are registered when they
    are Modules.  Unlike the reference's struct, this is a GNNLayer, so a GNNChain passes it the graph."""

    def __init__(self, fgate, ffeat=identity):
        super().__init__()
        self.fgate = fgate
        self.ffeat = ffeat

    def forward(self, g: GNNGraph, x: torch.Tensor) -> torch.Tensor:
        return global_attention_pool(self, g, x)

    def graph_forward(self, g: GNNGraph) -> GNNGraph:
        return GNNGraph(g, gdata=self(g, node_features(g)))


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


class Set2Set(GNNLayer):
    """Set2Set(n_in, n_iters, n_layers = 1) — GraphNeuralNetworks/src/layers/pool.jl:126-162: an LSTMCell(2·n_in => n_in)
    and num_iters; forward(g, x) returns the (2·n_in, num_graphs) readout (set2set_pool); l(g) puts it in gdata."""

    def __init__(self, n_in: int, n_iters: int, n_layers: int = 1, device=None):
        super().__init__()
        if n_layers != 1:
            raise AssertionError("multiple layers not implemented yet")
        self.lstm = _LSTMCell(2 * n_in, n_in, device=device)
        self.num_iters = int(n_iters)

    def forward(self, g: GNNGraph, x: torch.Tensor) -> torch.Tensor:
        return set2set_pool(self, g, x)

    def graph_forward(self, g: GNNGraph) -> GNNGraph:
        return GNNGraph(g, gdata=self(g, node_features(g)))


# ---------------------------------------------------------------------------------------------- top-k pooling
# Key dtypes the selection entry takes as they are, and the exact casts of the narrower ones.
_KEY_CODES = {torch.float32: _lib.KEY_F32, torch.float64: _lib.KEY_F64, torch.int32: _lib.KEY_I32,
              torch.int64: _lib.KEY_I64}
_KEY_CASTS = {torch.bool: torch.int32, torch.int8: torch.int32, torch.int16: torch.int32, torch.uint8: torch.int32,
              torch.float16: torch.float32, torch.bfloat16: torch.float32}


def _keep_mask(y: torch.Tensor, dev, k: int, ratio: float, seg_ptr=None) -> torch.Tensor:
    """uint8 mask of gnnb_topk_keep over the keys y (1-D) on dev: per segment of seg_ptr (None = one), the keys >= the
    k-th largest non-NaN key (k >= 1), or the ceil(ratio * n_s)-th (k = 0)."""
    if y.dtype in _KEY_CASTS:
        y = y.to(_KEY_CASTS[y.dtype])
    if y.dtype not in _KEY_CODES:
        raise TypeError(f"top-k selection takes real or integer keys (got {y.dtype})")
    y = y.to(dev).contiguous()
    n = y.numel()
    keep = torch.empty(n, dtype=torch.uint8, device=dev)
    n_seg = 1 if seg_ptr is None else seg_ptr.numel() - 1
    with torch.cuda.device(dev):
        _lib.check(lib.gnnb_topk_keep(y.data_ptr() if n else None, _KEY_CODES[y.dtype], n, _ptr(seg_ptr), n_seg,
                                      int(k), float(ratio), keep.data_ptr() if n else None, None, _stream(dev)))
    return keep


def topk_index(y: torch.Tensor, k: int) -> torch.Tensor:
    """GNNlib/src/layers/pool.jl:24-27: the ascending 1-based ids i with y[i] >= the k-th largest value of y (all ties
    kept; every id when k exceeds the length).  y is a vector or a (1, N) row.  k < 1 is an error, as the reference's
    `v[end]` of an empty `v`.  NaN rule of this port: a NaN is never kept and does not count toward k."""
    if isinstance(k, bool) or not isinstance(k, numbers.Integral):
        raise TypeError(f"topk_index takes an integer k (got {type(k).__name__})")
    if y.dim() == 2 and y.shape[0] == 1:
        y = y.reshape(-1)
    if y.dim() != 1:
        raise ValueError(f"topk_index takes a vector or a 1 x N row (got shape {tuple(y.shape)})")
    if k < 1:
        raise ValueError(f"topk_index needs k >= 1 (got {k}): nlargest(k, y) is empty")
    if y.numel() == 0:
        raise ValueError("topk_index of an empty vector: nlargest(k, y) is empty")
    dev = _graph._compute_device(y)
    return _keep_mask(y, dev, int(k), 0.0).nonzero().reshape(-1) + 1


def _topk_scores(x_rows: torch.Tensor, p: torch.Tensor) -> torch.Tensor:
    """y = p' x / norm(p) over the node rows of x (gnnb_topk_score), outside autograd: _TopKGateFn's pullback covers it"""
    n, D = x_rows.shape
    y = torch.empty(n, dtype=torch.float32, device=x_rows.device)
    with torch.cuda.device(x_rows.device):
        _lib.check(lib.gnnb_topk_score(x_rows.data_ptr(), n, D, p.detach().data_ptr(), y.data_ptr(),
                                       _stream(x_rows.device)))
    return y


class _TopKGateFn(torch.autograd.Function):
    """out_j = x_{idx_j} σ(y[idx_j]) (gnnb_topk_gate) with y = p' x / norm(p): the pullback (gnnb_topk_gate_bwd) gives
    dx through the gather and through y, and dp through y.  idx is 0-based and ascending; the selection is not
    differentiated."""

    @staticmethod
    def forward(ctx, x_rows, p, y, idx):
        n, D = x_rows.shape
        m = idx.numel()
        out = torch.empty((m, D), dtype=torch.float32, device=x_rows.device)
        with torch.cuda.device(x_rows.device):
            _lib.check(lib.gnnb_topk_gate(x_rows.data_ptr(), n, D, y.data_ptr(), idx.data_ptr() if m else None, m,
                                          out.data_ptr() if m else None, None, _stream(x_rows.device)))
        ctx.save_for_backward(x_rows, p, y, idx)
        return out

    @staticmethod
    def backward(ctx, dout):
        x_rows, p, y, idx = ctx.saved_tensors
        n, D = x_rows.shape
        m = idx.numel()
        dout = dout.contiguous()
        dx = torch.empty_like(x_rows)
        dp = torch.empty_like(p)
        with torch.cuda.device(x_rows.device):
            _lib.check(lib.gnnb_topk_gate_bwd(x_rows.data_ptr(), n, D, y.data_ptr(), p.data_ptr(),
                                              idx.data_ptr() if m else None, m, dout.data_ptr() if m else None,
                                              dx.data_ptr(), dp.data_ptr(), None, _stream(x_rows.device)))
        return dx, dp, None, None


def _topk_x(t, x: torch.Tensor):
    if x.dim() != 2:
        raise ValueError(f"topk_pool takes a (in_channel, N) matrix (got shape {tuple(x.shape)})")
    dev = _graph._compute_device(x)
    x_rows = _f32(rows(x), dev)
    p = _f32(t.p, dev)
    if p.shape != (x_rows.shape[1],):
        raise ValueError(f"p has {tuple(p.shape)} entries; x has {x_rows.shape[1]} rows")
    return dev, x_rows, p


def topk_pool(t, *args):
    """topk_pool(t, X) — GNNlib/src/layers/pool.jl:14-22: y = p' X / norm(p), idx = topk_index(y, t.k),
    t.A_tilde .= A[idx, idx], returns X[:, idx] .* σ.(y[idx]').  Julia's broadcast of A[idx, idx] into the (k, k) A_tilde
    needs m = length(idx) == k, or m == 1 (which fills A_tilde); any other m raises.

    topk_pool(t, g, x) — the same selection applied to every graph of the batch g (t.A is not used): an int t.k keeps
    min(k, n_i) nodes of graph i plus ties, a float t.k in (0, 1] keeps ceil(k n_i).  Returns (h, x_pooled, idx): h is
    remove_nodes(g, <the nodes not kept>), x_pooled the gated kept columns, idx their ascending 1-based ids in g."""
    if len(args) == 2:
        return _topk_pool_graph(t, *args)
    (x,) = args
    if t.A is None:
        raise ValueError("this TopKPool has no adjacency matrix: call it on a graph, t(g, x)")
    if isinstance(t.k, bool) or not isinstance(t.k, numbers.Integral):
        raise TypeError(f"the matrix form of topk_pool takes an integer k (got {t.k!r}); ratios are for graphs")
    dev, x_rows, p = _topk_x(t, x)
    n = x_rows.shape[0]
    assert t.A.shape == (n, n), f"A is {tuple(t.A.shape)}; X has {n} columns"
    if t.k < 1:
        raise ValueError(f"topk_pool needs k >= 1 (got {t.k}): nlargest(k, y) is empty")
    y = _topk_scores(x_rows, p)
    idx = _keep_mask(y, dev, int(t.k), 0.0).nonzero().reshape(-1)
    m = idx.numel()
    if m != t.A_tilde.shape[0] and m != 1:
        raise ValueError(f"DimensionMismatch: cannot broadcast A[idx, idx] of size ({m}, {m}) into A_tilde of size "
                         f"{tuple(t.A_tilde.shape)}: {m} scores tie with or exceed the k-th largest, k = {t.k}")
    with torch.no_grad():
        ia = idx.to(t.A.device)
        t.A_tilde[...] = t.A[ia[:, None], ia[None, :]]
    return unrows(_TopKGateFn.apply(x_rows, p, y, idx))


def _topk_pool_graph(t, g: GNNGraph, x: torch.Tensor):
    from .generate import _segments
    from .transform import _keep_nodes
    k = t.k
    if isinstance(k, bool) or not isinstance(k, numbers.Real):
        raise TypeError(f"TopKPool's k must be an int or a float ratio (got {k!r})")
    if isinstance(k, numbers.Integral):
        if k < 1:
            raise ValueError(f"topk_pool needs k >= 1 (got {k})")
        kk, ratio = int(k), 0.0
    else:
        if not 0.0 < float(k) <= 1.0:
            raise ValueError(f"a float k is a ratio in (0, 1] (got {k})")
        kk, ratio = 0, float(k)
    assert x.shape[-1] == g.num_nodes, \
        f"Got {x.shape[-1]} as last dimension size instead of num_nodes={g.num_nodes}"
    dev, x_rows, p = _topk_x(t, x)
    n = x_rows.shape[0]
    y = _topk_scores(x_rows, p)
    order, seg_ptr = None, None
    if g.graph_indicator is not None and n > 0:
        order, seg_ptr, _, _ = _segments(g.graph_indicator, n, dev)
    if order is None:
        keep = _keep_mask(y, dev, kk, ratio, seg_ptr)
    else:                                   # select on the stably sorted keys, scatter the mask back
        keep = torch.empty(n, dtype=torch.uint8, device=dev)
        keep[order] = _keep_mask(y[order], dev, kk, ratio, seg_ptr)
    idx = keep.nonzero().reshape(-1)
    x_pooled = unrows(_TopKGateFn.apply(x_rows, p, y, idx))
    return _keep_nodes(g, keep), x_pooled, idx + 1


class TopKPool(torch.nn.Module):
    """TopKPool(adj, k, in_channel) — GraphNeuralNetworks/src/layers/pool.jl:101-123: the adjacency A, k, the float32
    projection p = glorot_uniform(in_channel) and A_tilde, a (k, k) array of A's dtype on A's device that every
    forward(X) overwrites with A[idx, idx].  forward(X) is topk_pool(t, X); forward(g, x) is the graph form.  adj may be
    None for a pool used on graphs only, and there k may be a float ratio in (0, 1]."""

    def __init__(self, adj, k, in_channel: int, device=None):
        super().__init__()
        self.A = adj
        self.k = k
        self.p = torch.nn.Parameter(glorot_uniform(int(in_channel), device=device).to(torch.float32))
        if adj is not None:
            if isinstance(k, bool) or not isinstance(k, numbers.Integral):
                raise TypeError(f"TopKPool with an adjacency takes an integer k (got {k!r})")
            self.A_tilde = torch.empty((int(k), int(k)), dtype=adj.dtype, device=adj.device)
        else:
            self.A_tilde = None

    def forward(self, *args):
        return topk_pool(self, *args)
