"""The message-passing framework of GNNlib (GNNlib/src/msgpass.jl) on libgnnb200.

Same names, argument meaning and error behaviour as the reference:

    propagate(f, g, aggr; xi, xj, e)          msgpass.jl:71-79
    apply_edges(f, g; xi, xj, e)              msgpass.jl:117-129
    aggregate_neighbors(g, aggr, m)           msgpass.jl:145-149
    copy_xj, copy_xi, xi_dot_xj, xi_sub_xj, xj_sub_xi, e_mul_xj, w_mul_xj      msgpass.jl:162-208

``propagate`` with ``copy_xj`` / ``w_mul_xj`` / ``e_mul_xj`` (vector ``e``) and ``+ | mean | max | min`` takes the
fused kernel (``gnnb_propagate``: no (D,E) intermediate) — this is the place where the reference's CUDA
extension *disables* its own fast path (GNNlib/ext/GNNlibCUDAExt.jl:13-32).  Any other message function runs
through the generic ``_gather`` -> f -> ``_scatter`` composition (GNNGraphs/src/gatherscatter.jl) on the
library's gather / segmented-scatter kernels.  Zygote's role is played by ``torch.autograd.Function``s whose
backward calls the library's pullback entries (``gnnb_propagate_bwd``, ``gnnb_scatter`` ...).

Arrays are Julia-shaped: last dimension = nodes (xi, xj) or edges (e, messages); see graph.colmajor.
"""
from __future__ import annotations

import operator
from typing import Any, Callable, Optional

import torch

from . import _lib
from ._lib import lib
from .graph import GNNGraph, _is_hetero, _ptr, _stream, num_src_dst, relation, rows, unrows

# --------------------------------------------------------------------------------------------------
# aggregation operators: `+`, mean, max, min (NNlib.scatter ops the layers use)
# --------------------------------------------------------------------------------------------------


def mean(*a, **k):  # sentinel with the reference's name (Statistics.mean)
    return torch.mean(*a, **k)


_AGGR = {
    operator.add: _lib.SUM, "+": _lib.SUM, "add": _lib.SUM, "sum": _lib.SUM, sum: _lib.SUM, torch.add: _lib.SUM,
    torch.sum: _lib.SUM,
    mean: _lib.MEAN, "mean": _lib.MEAN, torch.mean: _lib.MEAN,
    max: _lib.MAX, "max": _lib.MAX, torch.max: _lib.MAX, torch.maximum: _lib.MAX,
    min: _lib.MIN, "min": _lib.MIN, torch.min: _lib.MIN, torch.minimum: _lib.MIN,
}


def _aggr_code(aggr) -> int:
    try:
        return _AGGR[aggr]
    except (KeyError, TypeError):
        raise ValueError(f"unsupported aggregation {aggr!r}: use +, mean, max or min") from None


# --------------------------------------------------------------------------------------------------
# size checks — GNNGraphs/src/utils.jl:1-28 (AssertionError, like the reference's @assert)
# --------------------------------------------------------------------------------------------------
def check_num_nodes(g: GNNGraph, x) -> bool:
    if x is None:
        return True
    if _is_hetero(g):
        # gnnheterograph/utils.jl:1-13: a (xj, xi) pair, xj over the source type and xi over the target type
        assert isinstance(x, tuple) and len(x) == 2, "a heterograph takes the node features as a (xj, xi) pair"
        ns, nd = num_src_dst(g)
        for v, n, side in ((x[0], ns, "source"), (x[1], nd, "target")):
            if isinstance(v, torch.Tensor):
                assert v.shape[-1] == n, f"Got {v.shape[-1]} as last dimension size instead of the {side} type's {n} nodes"
        return True
    if isinstance(x, torch.Tensor):
        assert g.num_nodes == x.shape[-1], \
            f"Got {x.shape[-1]} as last dimension size instead of num_nodes={g.num_nodes}"
        return True
    if isinstance(x, dict):
        x = tuple(x.values())
    for v in x:
        check_num_nodes(g, v)
    return True


def check_num_edges(g: GNNGraph, e) -> bool:
    if e is None:
        return True
    if isinstance(e, torch.Tensor):
        E = relation(g).num_edges
        assert E == e.shape[-1], f"Got {e.shape[-1]} as last dimension size instead of num_edges={E}"
        return True
    if isinstance(e, dict):
        e = tuple(e.values())
    for v in e:
        check_num_edges(g, v)
    return True


# --------------------------------------------------------------------------------------------------
# autograd functions over the C ABI (all tensors here are C-contiguous "rows": (N, D) / (E, D))
# --------------------------------------------------------------------------------------------------
def _f32(x: torch.Tensor, device) -> torch.Tensor:
    if x.dtype != torch.float32:
        raise TypeError(f"libgnnb200 computes in float32 (got {x.dtype})")
    if x.device != device:
        x = x.to(device)
    return x.contiguous()


class _GatherFn(torch.autograd.Function):
    """NNlib.gather by s or t; pullback = scatter(+) into zeros (SURVEY.md §8 a5)."""

    @staticmethod
    def forward(ctx, x_rows, plan, which, n_edges):
        D = x_rows[0].numel() if x_rows.shape[0] else int(torch.tensor(x_rows.shape[1:]).prod())
        out = torch.empty((n_edges,) + tuple(x_rows.shape[1:]), dtype=torch.float32, device=x_rows.device)
        with torch.cuda.device(plan.device):
            _lib.check(lib.gnnb_gather(plan.h, which, x_rows.data_ptr(), D, out.data_ptr(), _stream(plan.device)))
        ctx.plan, ctx.which, ctx.D, ctx.shape = plan, which, D, x_rows.shape
        return out

    @staticmethod
    def backward(ctx, dout):
        dout = dout.contiguous()
        dx = torch.empty(ctx.shape, dtype=torch.float32, device=dout.device)
        with torch.cuda.device(ctx.plan.device):
            _lib.check(lib.gnnb_scatter(ctx.plan.h, ctx.which, _lib.SUM, dout.data_ptr(), ctx.D, dx.data_ptr(),
                                        _stream(ctx.plan.device)))
        return dx, None, None, None


class _ScatterFn(torch.autograd.Function):
    """NNlib.scatter(aggr, m, t; dstsize); pullbacks as NNlib's rrules (SURVEY.md §9)."""

    @staticmethod
    def forward(ctx, m_rows, plan, which, aggr, n_nodes):
        D = int(torch.tensor(m_rows.shape[1:]).prod()) if m_rows.dim() > 1 else 1
        out = torch.empty((n_nodes,) + tuple(m_rows.shape[1:]), dtype=torch.float32, device=m_rows.device)
        with torch.cuda.device(plan.device):
            _lib.check(lib.gnnb_scatter(plan.h, which, aggr, m_rows.data_ptr(), D, out.data_ptr(),
                                        _stream(plan.device)))
        ctx.plan, ctx.which, ctx.aggr, ctx.D = plan, which, aggr, D
        if aggr in (_lib.MAX, _lib.MIN):
            ctx.save_for_backward(m_rows, out)
        return out

    @staticmethod
    def backward(ctx, dout):
        plan, which, aggr, D = ctx.plan, ctx.which, ctx.aggr, ctx.D
        dout = dout.contiguous()
        st = _stream(plan.device)
        with torch.cuda.device(plan.device):
            if aggr == _lib.MEAN:  # gather(Δ ./ count, idx)
                deg = torch.empty(dout.shape[0], dtype=torch.float32, device=dout.device)
                _lib.check(lib.gnnb_degree(plan.h, _lib.DIR_IN if which == _lib.DST else _lib.DIR_OUT, None,
                                           deg.data_ptr(), st))
                dout = (dout / deg.clamp(min=1).reshape((-1,) + (1,) * (dout.dim() - 1))).contiguous()
            E = lib_edges(plan)
            dm = torch.empty((E,) + tuple(dout.shape[1:]), dtype=torch.float32, device=dout.device)
            _lib.check(lib.gnnb_gather(plan.h, which, dout.data_ptr(), D, dm.data_ptr(), st))
            if aggr in (_lib.MAX, _lib.MIN):  # (m .== gather(out, idx)) .* gather(Δ, idx): ties all receive Δ
                m_rows, out = ctx.saved_tensors
                og = torch.empty_like(dm)
                _lib.check(lib.gnnb_gather(plan.h, which, out.data_ptr(), D, og.data_ptr(), st))
                dm = dm * (m_rows == og)
        return dm, None, None, None, None


def lib_edges(plan) -> int:
    import ctypes as C
    e = C.c_int64()
    _lib.check(lib.gnnb_graph_info(plan.h, C.byref(e), None, None))
    return int(e.value)


class _PropagateFn(torch.autograd.Function):
    """Fused propagate(copy_xj | w_mul_xj, g, aggr): gnnb_propagate / gnnb_propagate_bwd.  x has num_src rows, the
    result num_dst (n_out)."""

    @staticmethod
    def forward(ctx, x_rows, w, plan, aggr, n_out):
        D = int(torch.tensor(x_rows.shape[1:]).prod()) if x_rows.dim() > 1 else 1
        out = torch.empty((n_out,) + tuple(x_rows.shape[1:]), dtype=torch.float32, device=x_rows.device)
        msg = _lib.COPY_XJ if w is None else _lib.W_MUL_XJ
        with torch.cuda.device(plan.device):
            _lib.check(lib.gnnb_propagate(plan.h, 0, msg, aggr, x_rows.data_ptr(), _ptr(w), None, None, D,
                                          out.data_ptr(), _stream(plan.device)))
        ctx.plan, ctx.aggr, ctx.msg, ctx.D = plan, aggr, msg, D
        ctx.save_for_backward(x_rows, w, out if aggr in (_lib.MAX, _lib.MIN) else None)
        return out

    @staticmethod
    def backward(ctx, dout):
        x_rows, w, out = ctx.saved_tensors
        plan = ctx.plan
        dout = dout.contiguous()
        need_dx, need_dw = ctx.needs_input_grad[0], (w is not None and ctx.needs_input_grad[1])
        dx = torch.empty_like(x_rows) if need_dx else None
        dw = torch.empty_like(w) if need_dw else None
        with torch.cuda.device(plan.device):
            _lib.check(lib.gnnb_propagate_bwd(plan.h, ctx.msg, ctx.aggr, dout.data_ptr(), x_rows.data_ptr(),
                                              _ptr(w), None, None, _ptr(out), ctx.D, _ptr(dx), _ptr(dw),
                                              _stream(plan.device)))
        return dx, dw, None, None, None


class _GCNPropagateFn(torch.autograd.Function):
    """c .* propagate(copy_xj, g, +, xj = x .* c') with c = 1/sqrt(in-degree): gnnb_gcn_propagate (both ways).
    c = None: the plan's own normalisation (the library keeps c and its per-edge stream with the plan)."""

    @staticmethod
    def forward(ctx, x_rows, plan, c):
        D = x_rows[0].numel() if x_rows.shape[0] else 1
        out = torch.empty_like(x_rows)
        with torch.cuda.device(plan.device):
            _lib.check(lib.gnnb_gcn_propagate(plan.h, 0, x_rows.data_ptr(), None, None if c is None else c.data_ptr(), D,
                                              out.data_ptr(), _stream(plan.device)))
        ctx.plan, ctx.D, ctx.c = plan, D, c
        return out

    @staticmethod
    def backward(ctx, dout):
        dout = dout.contiguous()
        dx = torch.empty_like(dout)
        with torch.cuda.device(ctx.plan.device):
            _lib.check(lib.gnnb_gcn_propagate(ctx.plan.h, 1, dout.data_ptr(), None,
                                              None if ctx.c is None else ctx.c.data_ptr(), ctx.D, dx.data_ptr(),
                                              _stream(ctx.plan.device)))
        return dx, None, None


class _EdgeSoftmaxFn(torch.autograd.Function):
    @staticmethod
    def forward(ctx, e_rows, plan):
        K = e_rows[0].numel() if e_rows.shape[0] else 1
        out = torch.empty_like(e_rows)
        with torch.cuda.device(plan.device):
            _lib.check(lib.gnnb_softmax_edge_neighbors(plan.h, e_rows.data_ptr(), K, out.data_ptr(),
                                                       _stream(plan.device)))
        ctx.plan, ctx.K = plan, K
        ctx.save_for_backward(out)
        return out

    @staticmethod
    def backward(ctx, dalpha):
        (alpha,) = ctx.saved_tensors
        dalpha = dalpha.contiguous()
        de = torch.empty_like(alpha)
        with torch.cuda.device(ctx.plan.device):
            _lib.check(lib.gnnb_softmax_edge_neighbors_bwd(ctx.plan.h, alpha.data_ptr(), dalpha.data_ptr(), ctx.K,
                                                           de.data_ptr(), _stream(ctx.plan.device)))
        return de, None


# --------------------------------------------------------------------------------------------------
# _gather / _scatter with the reference's structural recursion (GNNGraphs/src/gatherscatter.jl:1-18)
# --------------------------------------------------------------------------------------------------
def _map_struct(fn: Callable, x):
    if x is None:
        return None
    if isinstance(x, torch.Tensor):
        return fn(x)
    if isinstance(x, dict):
        return {k: _map_struct(fn, v) for k, v in x.items()}
    if isinstance(x, tuple) and hasattr(x, "_fields"):  # namedtuple
        return type(x)(*[_map_struct(fn, v) for v in x])
    if isinstance(x, (tuple, list)):
        return type(x)(_map_struct(fn, v) for v in x)
    raise TypeError(f"unsupported feature container {type(x)}")


def _gather(g: GNNGraph, x, which: int):
    rel = relation(g)
    plan = rel.plan()

    def one(a: torch.Tensor):
        r = _GatherFn.apply(_f32(rows(a), plan.device), plan, which, rel.num_edges)
        return unrows(r)

    return _map_struct(one, x)


def _scatter(g: GNNGraph, aggr, m, which: int = _lib.DST):
    plan = relation(g).plan()
    code = _aggr_code(aggr)
    n = num_src_dst(g)[1 if which == _lib.DST else 0]

    def one(a: torch.Tensor):
        r = _ScatterFn.apply(_f32(rows(a), plan.device), plan, which, code, n)
        return unrows(r)

    return _map_struct(one, m)


# --------------------------------------------------------------------------------------------------
# message functions — GNNlib/src/msgpass.jl:162-208
# --------------------------------------------------------------------------------------------------
def copy_xj(xi, xj, e):
    return xj


def copy_xi(xi, xj, e):
    return xi


def xi_dot_xj(xi, xj, e):
    return (xi * xj).sum(dim=0, keepdim=True)


def xi_sub_xj(xi, xj, e):
    return xi - xj


def xj_sub_xi(xi, xj, e):
    return xj - xi


def e_mul_xj(xi, xj, e):
    assert e.dim() <= xj.dim()  # msgpass.jl:193
    e = e.reshape((1,) * (xj.dim() - e.dim()) + tuple(e.shape))
    return e * xj


def w_mul_xj(xi, xj, w):
    if w is None:
        return xj  # same as copy_xj if no weights (msgpass.jl:203)
    w = w.reshape((1,) * (xj.dim() - 1) + (w.numel(),))
    return w * xj


# --------------------------------------------------------------------------------------------------
# apply_edges / aggregate_neighbors / propagate
# --------------------------------------------------------------------------------------------------
def apply_edges(f: Callable, g: GNNGraph, xi=None, xj=None, e=None):
    """msgpass.jl:117-129: gather xi on targets, xj on sources, call f(xi, xj, e); outputs keep COO order."""
    check_num_nodes(g, (xj, xi))
    check_num_edges(g, e)
    xi_e = _gather(g, xi, _lib.DST)
    xj_e = _gather(g, xj, _lib.SRC)
    return f(xi_e, xj_e, e)


def aggregate_neighbors(g: GNNGraph, aggr, m):
    """msgpass.jl:145-149: _scatter(aggr, m, t, g.num_nodes)."""
    check_num_edges(g, m)
    return _scatter(g, aggr, m, _lib.DST)


def _fusable(f, xi, xj, e, g) -> Optional[Any]:
    """Return the edge-weight tensor ('none' for unweighted) if (f, xj, e) has a fused kernel, else None."""
    if not isinstance(xj, torch.Tensor) or xj.dim() < 2:
        return None
    if f is copy_xj:
        return "none"
    if f is w_mul_xj and e is None:
        w = relation(g).w
        return "none" if w is None else w
    if f is e_mul_xj and isinstance(e, torch.Tensor) and e.dim() == 1:
        return e
    return None


def propagate(f: Callable, g: GNNGraph, aggr, xi=None, xj=None, e=None):
    """msgpass.jl:71-79.  Fused for the built-in linear messages, generic otherwise."""
    w = _fusable(f, xi, xj, e, g)
    if w is not None:
        check_num_nodes(g, (xj, xi))
        check_num_edges(g, e)
        plan = relation(g).plan()
        wt = None if isinstance(w, str) else _f32(w, plan.device)
        out = _PropagateFn.apply(_f32(rows(xj), plan.device), wt, plan, _aggr_code(aggr), num_src_dst(g)[1])
        return unrows(out)
    m = apply_edges(f, g, xi, xj, e)
    return aggregate_neighbors(g, aggr, m)


def softmax_edge_neighbors(g: GNNGraph, e: torch.Tensor) -> torch.Tensor:
    """GNNlib/src/utils.jl:84-97: softmax of the edge features over each target's in-neighbourhood."""
    rel = relation(g)
    assert e.shape[-1] == rel.num_edges
    plan = rel.plan()
    return unrows(_EdgeSoftmaxFn.apply(_f32(rows(e), plan.device), plan))


def expand_srcdst(g: GNNGraph, x):
    """GNNlib/src/utils.jl:123-125."""
    if isinstance(x, torch.Tensor) and x.dim() == 2:
        return x, x
    if isinstance(x, tuple) and len(x) == 2 and all(isinstance(v, torch.Tensor) and v.dim() == 2 for v in x):
        return x
    raise ValueError("Invalid input type, expected matrix or tuple of matrices.")


class Fix1:
    """Replacement for Base.Fix1 with several arguments — GNNlib/src/utils.jl:128-133."""

    def __init__(self, f, x):
        self.f, self.x = f, x

    def __call__(self, *y):
        return self.f(self.x, *y)
