"""Recurrent temporal graph layers — GraphNeuralNetworks/src/layers/temporalconv.jl:
    GNNRecurrence (:121-135), GConvGRUCell / GConvGRU (:200-293), GConvLSTMCell / GConvLSTM (:355-477),
    DCGRUCell / DCGRU (:537-613), EvolveGCNOCell / EvolveGCNO (:678-752), TGCNCell / TGCN (:809-884),
a minimal TemporalSnapshotsGNNGraph (GNNGraphs/src/temporalsnapshotsgnngraph.jl:56-100) with add_snapshot /
remove_snapshot (:132-145, 192-201).  The temporal graph generators are in generate.py.

Holders carry the reference's field names, so a trained model copies over parameter by parameter.  Arrays are
Julia-shaped: a static-graph sequence is x (in, T, N), one node row of T·in contiguous floats.

The reference runs every gate's operator separately at every step (`scan`, :1-8).  Here, per layer call:
  * x side, all T steps at once: the graph operator runs on the (in·T, N) view of x and each gate's weights are stacked
    into one GEMM over the (in, T·N) view, with the biases a gate sums folded in.  PX holds rows of (N, T, G·out).
  * h side, per step, shared by the gates: one basis of h for every gate that reads h, one basis of r ⊙ h for the GRU
    candidate; the gates' h-side weights stacked into one GEMM.
  * the gates: csrc/recurrent.cu, one pass over node rows (gnnb_gru_rz / gnnb_gru_out / gnnb_lstm_cell and pullbacks).
Each step reads its slice of PX through PX.unbind(1) (the backward is one stack, not a zero-filled PX per step) and the
outputs are stacked once at the end.  Every graph operator and GEMM goes through the existing autograd Functions.

Deliberate differences: σ and tanh are the accurate forms (the reference's sigmoid_fast / tanh_fast approximate); the
stacked GEMMs and folded biases sum in another order, so results agree with the reference's arithmetic to rounding;
the GRU and LSTM cells on a TemporalSnapshotsGNNGraph need one node count in every snapshot (AssertionError otherwise).
"""
from __future__ import annotations

import numbers
from types import SimpleNamespace
from typing import Optional

import torch

from . import _lib
from ._lib import lib
from .basic import GNNLayer
from .graph import GNNGraph, _stream, add_self_loops, rows, unrows
from .layers import GCNConv, _bias_act, _DenseAct, _linear, _LSTMCell, gcn_conv, glorot_uniform, relu
from .layers_more import ChebConv, Chain, DConv, cheb_basis, cheb_operator, diffusion_basis, transposed_graph
from .msgpass import _GCNPropagateFn, _f32


def _p(t):
    return None if t is None else t.data_ptr()


def lstm_dw_slots(N: int) -> int:
    """GNNB_LSTM_DW_SLOTS(N) of include/gnnb200.h: partial slots of the peephole gradient"""
    return (N + 63) // 64 if N < 65536 else 1024


# ------------------------------------------------------------------------------------------------ the gates
class _Link:
    """A GRU step's shared pullback buffers.  The out gate's backward allocates dPX_t (N, 3D), writes its n block and the
    blend's dh; the rz gate's backward (later: z and r ⊙ h feed the out gate) writes the [r | z] block, adds drh ⊙ r to
    dh and returns both.  So dPX_t is one buffer, written once per element, for the x side and the h side alike."""
    __slots__ = ("dpx", "dh")

    def __init__(self):
        self.dpx = self.dh = None


class _GRURZFn(torch.autograd.Function):
    """r = σ(px_r + ah_r), z = σ(px_z + ah_z), rh = r ⊙ h: gnnb_gru_rz / gnnb_gru_rz_bwd"""

    @staticmethod
    def forward(ctx, px, ah, h, link):
        N, D = h.shape
        r, z, rh = torch.empty_like(h), torch.empty_like(h), torch.empty_like(h)
        with torch.cuda.device(h.device):
            _lib.check(lib.gnnb_gru_rz(px.data_ptr(), _ld(px), ah.data_ptr(), h.data_ptr(), N, D, r.data_ptr(),
                                       z.data_ptr(), rh.data_ptr(), _stream(h.device)))
        ctx.save_for_backward(h, r, z)
        ctx.link = link
        ctx.mark_non_differentiable(r)
        return r, z, rh

    @staticmethod
    def backward(ctx, dr, dz, drh):
        h, r, z = ctx.saved_tensors
        N, D = h.shape
        link = ctx.link
        dpx = link.dpx if link.dpx is not None else torch.zeros((N, 3 * D), dtype=h.dtype, device=h.device)
        dh = link.dh if link.dh is not None else torch.zeros_like(h)
        link.dpx = link.dh = None
        drh, dz = drh.contiguous(), dz.contiguous()
        with torch.cuda.device(h.device):
            _lib.check(lib.gnnb_gru_rz_bwd(drh.data_ptr(), dz.data_ptr(), h.data_ptr(), r.data_ptr(), z.data_ptr(), N,
                                           D, dpx.data_ptr(), 3 * D, dh.data_ptr(), _stream(h.device)))
        return dpx, dpx[:, :2 * D], dh, None


class _GRUOutFn(torch.autograd.Function):
    """n = tanh(px_n + ah_n); h' = (1 − z) n + z h (blend 0) or (1 − z) h + z n (blend 1): gnnb_gru_out(_bwd).  Its
    gradients of px and h are completed and returned by the step's _GRURZFn (see _Link)."""

    @staticmethod
    def forward(ctx, px, ah_n, h, z, blend, link):
        N, D = h.shape
        n, hn = torch.empty_like(h), torch.empty_like(h)
        with torch.cuda.device(h.device):
            _lib.check(lib.gnnb_gru_out(px.data_ptr(), _ld(px), ah_n.data_ptr(), h.data_ptr(), z.data_ptr(), N, D,
                                        blend, n.data_ptr(), hn.data_ptr(), _stream(h.device)))
        ctx.save_for_backward(h, z, n)
        ctx.blend, ctx.link = blend, link
        return hn

    @staticmethod
    def backward(ctx, dhn):
        h, z, n = ctx.saved_tensors
        N, D = h.shape
        dhn = dhn.contiguous()
        dpx = torch.empty((N, 3 * D), dtype=h.dtype, device=h.device)
        dz, dh = torch.empty_like(h), torch.empty_like(h)
        with torch.cuda.device(h.device):
            _lib.check(lib.gnnb_gru_out_bwd(dhn.data_ptr(), h.data_ptr(), z.data_ptr(), n.data_ptr(), N, D, ctx.blend,
                                            dpx.data_ptr() + 2 * D * dpx.element_size(), 3 * D, dz.data_ptr(),
                                            dh.data_ptr(), _stream(h.device)))
        ctx.link.dpx, ctx.link.dh = dpx, dh
        return None, dpx[:, 2 * D:], None, dz, None, None


class _LSTMGateFn(torch.autograd.Function):
    """The LSTM gates with optional peepholes w (4D): gnnb_lstm_cell / gnnb_lstm_cell_bwd.  Returns (h', c')."""

    @staticmethod
    def forward(ctx, px, ah, c, w):
        N, D = c.shape
        gates = torch.empty((N, 4 * D), dtype=c.dtype, device=c.device)
        cn, hn = torch.empty_like(c), torch.empty_like(c)
        with torch.cuda.device(c.device):
            _lib.check(lib.gnnb_lstm_cell(px.data_ptr(), _ld(px), ah.data_ptr(), c.data_ptr(), _p(w), N, D,
                                          gates.data_ptr(), cn.data_ptr(), hn.data_ptr(), _stream(c.device)))
        ctx.save_for_backward(c, gates, cn, w)
        return hn, cn

    @staticmethod
    def backward(ctx, dhn, dcn):
        c, gates, cn, w = ctx.saved_tensors
        N, D = c.shape
        dhn, dcn = dhn.contiguous(), dcn.contiguous()
        dpre = torch.empty((N, 4 * D), dtype=c.dtype, device=c.device)
        dc = torch.empty_like(c)
        need_dw = w is not None and ctx.needs_input_grad[3]
        dw = torch.empty_like(w) if need_dw else None
        ws = torch.empty(lstm_dw_slots(N) * 4 * D, dtype=c.dtype, device=c.device) if need_dw else None
        with torch.cuda.device(c.device):
            _lib.check(lib.gnnb_lstm_cell_bwd(dhn.data_ptr(), dcn.data_ptr(), c.data_ptr(), gates.data_ptr(),
                                              cn.data_ptr(), _p(w), N, D, dpre.data_ptr(), dc.data_ptr(), _p(dw), _p(ws),
                                              _stream(c.device)))
        return dpre, dpre, dc, dw


# ------------------------------------------------------------------------------------------------ helpers
def _fold(*biases):
    """the sum of the biases a gate adds (None entries and `false` skipped); None when there are none"""
    bs = [b for b in biases if b is not None and b is not False]
    if not bs:
        return None
    out = bs[0].reshape(-1)
    for b in bs[1:]:
        out = out + b.reshape(-1)
    return out


def _holder(bias=None, sigma=None):
    """a parameter holder for _linear / _bias_act: σ.(W x .+ bias)"""
    h = SimpleNamespace(bias=bias)
    if sigma is not None:
        h.sigma = sigma
    return h


def _cat_bias(D: int, *gates):
    """vcat over the gates of the sum of each gate's biases (a tuple per gate; a gate with none gets zeros of width D);
    None when no gate has a bias"""
    folded = [_fold(*(b if isinstance(b, tuple) else (b,))) for b in gates]
    if all(b is None for b in folded):
        return None
    ref = next(b for b in folded if b is not None)
    return torch.cat([torch.zeros(D, dtype=ref.dtype, device=ref.device) if b is None else b for b in folded])


def _ld(px: torch.Tensor) -> int:
    """node stride of a (N, W) slice of PX (any stride is valid for a single row)"""
    return px.stride(0) if px.shape[0] > 1 else px.shape[1]


def _state_matrix(h, out: int, N: int, what: str = "state") -> torch.Tensor:
    """the reference's state rules: a vector (out,) is repeated over the nodes, a matrix must be (out, N)"""
    if h.dim() == 1:
        assert h.shape[0] == out, f"{what}: a vector state must have length {out} (got {h.shape[0]})"
        return h.reshape(out, 1).expand(out, N)
    assert h.dim() == 2 and tuple(h.shape) == (out, N), \
        f"{what}: a matrix state must be ({out}, {N}) (got {tuple(h.shape)})"
    return h


def _check_x(cell, g: GNNGraph, x: torch.Tensor) -> None:
    assert x.dim() == 3, "x must be (in, T, N)"
    assert x.shape[0] == cell.in_, f"Input feature size must match input channel size {cell.in_} (got {x.shape[0]})"
    assert x.shape[2] == g.num_nodes, f"x has {x.shape[2]} node columns, the graph {g.num_nodes} nodes"
    if x.shape[1] < 1:
        raise ValueError("a sequence needs at least one time step (T = 0)")


# Julia views of a column-major (D, T, N) array, as torch views (no copy): torch's reshape merges logical indices in
# row-major order, so the time and feature (or node) dimensions are swapped around it.
def _feat_view(x: torch.Tensor) -> torch.Tensor:
    """(D, T, N) -> the (D·T, N) view the graph operators run on (one column per node, row t·D + d)"""
    D, T, N = x.shape
    return x.transpose(0, 1).reshape(T * D, N)


def _unfeat(z: torch.Tensor, D: int, T: int) -> torch.Tensor:
    """inverse of _feat_view"""
    return z.reshape(T, D, z.shape[1]).transpose(0, 1)


def _node_view(x: torch.Tensor) -> torch.Tensor:
    """(D, T, N) -> the (D, T·N) view the GEMMs run on (column n·T + t)"""
    D, T, N = x.shape
    return x.transpose(1, 2).reshape(D, N * T)


def _unnode(y: torch.Tensor, N: int, T: int) -> torch.Tensor:
    """inverse of _node_view"""
    return y.reshape(y.shape[0], N, T).transpose(1, 2)


def _basis_nodes(z: torch.Tensor, D: int, T: int) -> torch.Tensor:
    """a (D·T, N) operator output as the (D, T·N) GEMM operand"""
    return _node_view(_unfeat(z, D, T))


def _px_rows(PX: torch.Tensor, N: int, T: int) -> torch.Tensor:
    """(G·D, T·N) (column n·T + t) -> rows (N, T, G·D)"""
    return rows(PX).reshape(N, T, PX.shape[0])


def _sum_gemms(pairs, bias=None) -> torch.Tensor:
    """Σ W_j x_j (+ bias, folded into the first GEMM) over Julia-shaped 2-D x_j"""
    out = None
    for j, (W, x) in enumerate(pairs):
        y = _linear(_holder(bias), W, x, True) if (j == 0 and bias is not None) else _linear(None, W, x, False)
        out = y if out is None else out + y
    return out


def _cheb_op(g: GNNGraph):
    """cheb_operator(g), kept on the graph: the cells call the basis several times per step"""
    op = getattr(g, "_cheb_op_cache", None)
    if op is None:
        op = cheb_operator(g)
        g._cheb_op_cache = op
    return op


def _gcn_propagate(g: GNNGraph, X: torch.Tensor) -> torch.Tensor:
    """GCNConv's normalised propagate with self loops (conv.jl:37-63, unweighted, default norm) of a (W, N) array"""
    gl = add_self_loops(g)
    plan = gl.plan()
    return unrows(_GCNPropagateFn.apply(_f32(rows(X), plan.device), plan, None))


class _GRUCellBase(torch.nn.Module):
    """A GRU-type cell: subclasses give the x side (PX for all steps), the h side of r and z, and the candidate's."""
    blend = 0

    def initialstates(self):
        return torch.zeros(self.out, dtype=self._param().dtype, device=self._param().device)

    def _sequence(self, g: GNNGraph, x: torch.Tensor, h):
        """x (in, T, N), h as the reference accepts it -> (y (out, T, N), h_T)"""
        _check_x(self, g, x)
        I, T, N = x.shape
        h = self.initialstates() if h is None else h
        hr = rows(_state_matrix(h, self.out, N))
        PX = _px_rows(self._x_side(g, x), N, T)
        ys = []
        for px in PX.unbind(1):
            link = _Link()
            ah = rows(self._h_rz(g, unrows(hr)))
            _, z, rh = _GRURZFn.apply(px, ah, hr, link)
            ahn = rows(self._h_n(g, unrows(rh)))
            hr = _GRUOutFn.apply(px, ahn, hr, z, self.blend, link)
            ys.append(hr)
        return unrows(torch.stack(ys, dim=1)), unrows(hr)

    def forward(self, g, x, state=None):
        """one step: x (in, N) -> (h', h')"""
        y, h = self._sequence(g, x.unsqueeze(1), state)
        return h, h


# ------------------------------------------------------------------------------------------------ GConvGRU
class GConvGRUCell(_GRUCellBase, GNNLayer):
    """GConvGRUCell(in => out, k; bias=true) — temporalconv.jl:200-254: six ChebConvs, fields conv_x_r … conv_h_h."""

    def __init__(self, ch_in: int, ch_out: int, k: int, *, bias: bool = True, device=None):
        super().__init__()
        if k < 2:
            raise ValueError("GConvGRUCell: k must be >= 2 (ChebConv's order)")
        for gate in ("r", "z", "h"):
            setattr(self, f"conv_x_{gate}", ChebConv(ch_in, ch_out, k, bias=bias, device=device))
            setattr(self, f"conv_h_{gate}", ChebConv(ch_out, ch_out, k, bias=bias, device=device))
        self.k, self.in_, self.out = int(k), ch_in, ch_out

    def _param(self):
        return self.conv_x_r.weight

    def _x_side(self, g, x):
        I, T, N = x.shape
        Z = cheb_basis(g, _feat_view(x), self.k, _cheb_op(g))
        W = torch.cat([self.conv_x_r.weight, self.conv_x_z.weight, self.conv_x_h.weight], 0)
        b = _cat_bias(self.out, *[(getattr(self, f"conv_x_{q}").bias, getattr(self, f"conv_h_{q}").bias)
                                  for q in ("r", "z", "h")])
        return _sum_gemms([(W[:, :, j], _basis_nodes(Z[j], I, T)) for j in range(self.k)], b)

    def _h_rz(self, g, h):
        W = torch.cat([self.conv_h_r.weight, self.conv_h_z.weight], 0)
        Z = cheb_basis(g, h, self.k, _cheb_op(g))
        return _sum_gemms([(W[:, :, j], Z[j]) for j in range(self.k)])

    def _h_n(self, g, rh):
        Z = cheb_basis(g, rh, self.k, _cheb_op(g))
        return _sum_gemms([(self.conv_h_h.weight[:, :, j], Z[j]) for j in range(self.k)])

    def __repr__(self):
        return f"GConvGRUCell({self.in_} => {self.out}, {self.k})"


# ------------------------------------------------------------------------------------------------ DCGRU
class DCGRUCell(_GRUCellBase):
    """DCGRUCell(in => out, k; bias=true) — temporalconv.jl:537-575: DConv((in+out) => out, k) dconv_u (z), dconv_r,
    dconv_c.  DConv(vcat(x, h)) is linear in the vcat: its weights split into the x and h column blocks."""

    def __init__(self, ch_in: int, ch_out: int, k: int, *, bias: bool = True, device=None):
        super().__init__()
        self.dconv_u = DConv(ch_in + ch_out, ch_out, k, bias=bias, device=device)
        self.dconv_r = DConv(ch_in + ch_out, ch_out, k, bias=bias, device=device)
        self.dconv_c = DConv(ch_in + ch_out, ch_out, k, bias=bias, device=device)
        self.k, self.in_, self.out = int(k), ch_in, ch_out

    def _param(self):
        return self.dconv_u.weights

    def _terms(self, W, terms):
        """Σ W[1, j] T_in + W[2, j] T_out over diffusion_basis terms (the two j = 0 weights summed: T_in = T_out = x)"""
        pairs = [(W[0, 0] + W[1, 0], terms[0][1])]
        for j, T_in, T_out in terms[1:]:
            pairs += [(W[0, j], T_in), (W[1, j], T_out)]
        return pairs

    def _x_side(self, g, x):
        I, T, N = x.shape
        terms = diffusion_basis(g, _feat_view(x), self.k, transposed_graph(g))
        terms = [(j, _basis_nodes(a, I, T), _basis_nodes(b, I, T)) for j, a, b in terms]
        W = torch.cat([c.weights[:, :, :, :I] for c in (self.dconv_r, self.dconv_u, self.dconv_c)], 2)
        b = _cat_bias(self.out, *[c.bias for c in (self.dconv_r, self.dconv_u, self.dconv_c)])
        return _sum_gemms(self._terms(W, terms), b)

    def _h_rz(self, g, h):
        W = torch.cat([c.weights[:, :, :, self.in_:] for c in (self.dconv_r, self.dconv_u)], 2)
        return _sum_gemms(self._terms(W, diffusion_basis(g, h, self.k, transposed_graph(g))))

    def _h_n(self, g, rh):
        W = self.dconv_c.weights[:, :, :, self.in_:]
        return _sum_gemms(self._terms(W, diffusion_basis(g, rh, self.k, transposed_graph(g))))

    def __repr__(self):
        return f"DCGRUCell({self.in_} => {self.out}, {self.k})"


# ------------------------------------------------------------------------------------------------ TGCN
class TGCNCell(_GRUCellBase, GNNLayer):
    """TGCNCell(in => out) — temporalconv.jl:809-849: conv_z / conv_r / conv_h are GNNChain(GCNConv(in => out, relu),
    GCNConv(out => out)), dense_z / dense_r Dense(2out => out, sigmoid), dense_h Dense(2out => out, tanh).  All the
    graph work is on the x side: two propagates per layer call."""
    blend = 1

    def __init__(self, ch_in: int, ch_out: int, *, bias: bool = True, device=None):
        super().__init__()
        for gate in ("z", "r", "h"):
            setattr(self, f"conv_{gate}", Chain(GCNConv(ch_in, ch_out, relu, bias=bias, device=device),
                                                GCNConv(ch_out, ch_out, bias=bias, device=device)))
            setattr(self, f"dense_{gate}", _DenseAct(2 * ch_out, ch_out, torch.tanh if gate == "h" else torch.sigmoid,
                                                     device=device))
        self.in_, self.out = ch_in, ch_out

    def _param(self):
        return self.dense_z.weight

    def _x_side(self, g, x):
        I, T, N = x.shape
        D = self.out
        chains = [self.conv_r, self.conv_z, self.conv_h]            # gate order [r | z | n]
        W1 = torch.cat([c[0].weight for c in chains], 0)             # (3D, I): layer 1 of the three chains, stacked
        b1 = _cat_bias(D, *[c[0].bias for c in chains])
        if 3 * D < I:                                                # multiply first when it is narrower (conv.jl:47)
            A = _linear(None, W1, _node_view(x), False)
            A = _gcn_propagate(g, _feat_view(_unnode(A, N, T)))
            Y1 = _bias_act(_holder(b1, relu), _basis_nodes(A, 3 * D, T))
        else:
            P = _gcn_propagate(g, _feat_view(x))
            Y1 = _linear(_holder(b1, relu), W1, _basis_nodes(P, I, T), True)
        P2 = _basis_nodes(_gcn_propagate(g, _feat_view(_unnode(Y1, N, T))), 3 * D, T)   # layer 2: one propagate
        b2 = _cat_bias(D, *[c[1].bias for c in chains])
        Y2 = _linear(_holder(b2), torch.block_diag(*[c[1].weight for c in chains]), P2, True)
        dense = [self.dense_r, self.dense_z, self.dense_h]
        bd = _cat_bias(D, *[d.bias for d in dense])
        return _linear(_holder(bd), torch.block_diag(*[d.weight[:, :D] for d in dense]), Y2, True)

    def _h_rz(self, g, h):
        return _linear(None, torch.cat([self.dense_r.weight[:, self.out:], self.dense_z.weight[:, self.out:]], 0), h,
                       False)

    def _h_n(self, g, rh):
        return _linear(None, self.dense_h.weight[:, self.out:], rh, False)

    def __repr__(self):
        return f"TGCNCell({self.in_} => {self.out})"


# ------------------------------------------------------------------------------------------------ GConvLSTM
class GConvLSTMCell(GNNLayer):
    """GConvLSTMCell(in => out, k; bias=true) — temporalconv.jl:355-437: conv_x_* / conv_h_* ChebConvs, peepholes w_*
    (out, 1) and biases b_* (out,) for the gates i, f, c, o."""

    def __init__(self, ch_in: int, ch_out: int, k: int, *, bias: bool = True, device=None):
        super().__init__()
        if k < 2:
            raise ValueError("GConvLSTMCell: k must be >= 2 (ChebConv's order)")
        for gate in ("i", "f", "c", "o"):
            setattr(self, f"conv_x_{gate}", ChebConv(ch_in, ch_out, k, bias=bias, device=device))
            setattr(self, f"conv_h_{gate}", ChebConv(ch_out, ch_out, k, bias=bias, device=device))
            setattr(self, f"w_{gate}", torch.nn.Parameter(glorot_uniform(ch_out, 1, device=device)))
            setattr(self, f"b_{gate}", torch.nn.Parameter(torch.zeros(ch_out, device=device)) if bias else None)
        self.k, self.in_, self.out = int(k), ch_in, ch_out

    def initialstates(self):
        w = self.conv_x_i.weight
        return (torch.zeros(self.out, dtype=w.dtype, device=w.device), torch.zeros(self.out, dtype=w.dtype, device=w.device))

    def _sequence(self, g: GNNGraph, x: torch.Tensor, state):
        _check_x(self, g, x)
        I, T, N = x.shape
        h, c = self.initialstates() if state is None else state
        hr = rows(_state_matrix(h, self.out, N, "h"))
        cr = rows(_state_matrix(c, self.out, N, "c"))
        gates = ("i", "f", "c", "o")
        Z = cheb_basis(g, _feat_view(x), self.k, _cheb_op(g))
        Wx = torch.cat([getattr(self, f"conv_x_{q}").weight for q in gates], 0)
        b = _cat_bias(self.out, *[(getattr(self, f"conv_x_{q}").bias, getattr(self, f"conv_h_{q}").bias,
                                   getattr(self, f"b_{q}")) for q in gates])
        PX = _px_rows(_sum_gemms([(Wx[:, :, j], _basis_nodes(Z[j], I, T)) for j in range(self.k)], b), N, T)
        Wh = torch.cat([getattr(self, f"conv_h_{q}").weight for q in gates], 0)
        w = torch.cat([getattr(self, f"w_{q}").reshape(-1) for q in gates])
        op = _cheb_op(g)
        ys = []
        for px in PX.unbind(1):
            Zh = cheb_basis(g, unrows(hr), self.k, op)
            ah = rows(_sum_gemms([(Wh[:, :, j], Zh[j]) for j in range(self.k)]))
            hr, cr = _LSTMGateFn.apply(px, ah, cr, w)
            ys.append(hr)
        return unrows(torch.stack(ys, dim=1)), (unrows(hr), unrows(cr))

    def forward(self, g, x, state=None):
        """one step: x (in, N) -> (h', (h', c'))"""
        _, (h, c) = self._sequence(g, x.unsqueeze(1), state)
        return h, (h, c)

    def __repr__(self):
        return f"GConvLSTMCell({self.in_} => {self.out}, {self.k})"


# ------------------------------------------------------------------------------------------------ EvolveGCNO
class EvolveGCNOCell(GNNLayer):
    """EvolveGCNOCell(in => out; bias=true) — temporalconv.jl:678-705: conv = GCNConv(in => out), lstm =
    LSTMCell(in·out => in·out).  The LSTM evolves the GCN weight and does not read x: per step one gate pass on a
    single row (the LSTM entry without peepholes), then the GCN with that weight."""

    def __init__(self, ch_in: int, ch_out: int, *, bias: bool = True, device=None):
        super().__init__()
        self.conv = GCNConv(ch_in, ch_out, bias=bias, device=device)
        self.lstm = _LSTMCell(ch_in * ch_out, ch_in * ch_out, device=device)
        if not bias:
            self.lstm.bias = None
        self.in_, self.out = ch_in, ch_out

    def initialstates(self):
        w = self.conv.weight
        z = torch.zeros(self.in_ * self.out, dtype=w.dtype, device=w.device)
        return SimpleNamespace(weight=w.t().reshape(-1), lstm=(z, z.clone()))   # reshape(conv.weight, :), column-major

    def _evolve(self, state):
        """the LSTM step of the weight (temporalconv.jl:702) -> (W (out, in), new state)"""
        io = self.in_ * self.out
        wv = state.weight.reshape(io, 1)
        h, c = state.lstm
        px = _linear(_holder(self.lstm.bias), self.lstm.Wi, wv, True)
        ah = _linear(None, self.lstm.Wh, h.reshape(io, 1), False)
        hn, cn = _LSTMGateFn.apply(rows(px), rows(ah), c.reshape(1, io).contiguous(), None)
        hv, cv = hn.reshape(-1), cn.reshape(-1)
        return hv.reshape(self.in_, self.out).t(), SimpleNamespace(weight=hv, lstm=(hv, cv))

    def _sequence(self, g: GNNGraph, x: torch.Tensor, state):
        assert x.dim() == 3 and x.shape[0] == self.in_, f"x must be ({self.in_}, T, N)"
        assert x.shape[2] == g.num_nodes, f"x has {x.shape[2]} node columns, the graph {g.num_nodes} nodes"
        if x.shape[1] < 1:
            raise ValueError("a sequence needs at least one time step (T = 0)")
        I, T, N = x.shape
        state = self.initialstates() if state is None else state
        P = _unfeat(_gcn_propagate(g, _feat_view(x)), I, T)               # the propagate of every step, once
        hold = _holder(self.conv.bias, getattr(self.conv, "sigma", None))
        ys = []
        for Pt in P.unbind(1):
            W, state = self._evolve(state)
            ys.append(rows(_linear(hold, W, Pt, True)))
        return unrows(torch.stack(ys, dim=1)), state

    def forward(self, g, x, state=None):
        """one step: x (in, N) -> (y, state); state has the fields weight and lstm, as the reference's"""
        state = self.initialstates() if state is None else state
        assert x.dim() == 2 and x.shape[0] == self.in_, f"x must be ({self.in_}, N)"
        W, state = self._evolve(state)
        return gcn_conv(self.conv, g, x, conv_weight=W), state

    def __repr__(self):
        return f"EvolveGCNOCell({self.in_} => {self.out})"


# ------------------------------------------------------------------------------------------------ snapshots, recurrence
class TemporalSnapshotsGNNGraph:
    """TemporalSnapshotsGNNGraph(snapshots) — GNNGraphs/src/temporalsnapshotsgnngraph.jl:56-100 (minimal): snapshots,
    num_nodes / num_edges (lists), num_snapshots; 1-based integer and vector indexing, iteration, len."""

    def __init__(self, snapshots):
        self.snapshots = list(snapshots)
        assert all(isinstance(s, GNNGraph) for s in self.snapshots), "snapshots must be GNNGraphs"

    @property
    def num_nodes(self):
        return [s.num_nodes for s in self.snapshots]

    @property
    def num_edges(self):
        return [s.num_edges for s in self.snapshots]

    @property
    def num_snapshots(self) -> int:
        return len(self.snapshots)

    def __len__(self):
        return len(self.snapshots)

    def __iter__(self):
        return iter(self.snapshots)

    def __getitem__(self, t):
        if isinstance(t, numbers.Integral):
            assert 1 <= t <= len(self.snapshots), f"snapshot index {t} out of range 1:{len(self.snapshots)}"
            return self.snapshots[t - 1]
        return TemporalSnapshotsGNNGraph([self[int(i)] for i in t])

    def __repr__(self):
        return f"TemporalSnapshotsGNNGraph(num_snapshots={self.num_snapshots})"


def add_snapshot(tg: TemporalSnapshotsGNNGraph, t: int, g: GNNGraph) -> TemporalSnapshotsGNNGraph:
    """GNNGraphs/src/temporalsnapshotsgnngraph.jl:132-145: a new temporal graph with g inserted at time index t
    (1-based; t = num_snapshots + 1 appends).  tg is not changed."""
    if tg.num_snapshots > 0:
        assert g.num_nodes == tg.num_nodes[0], "number of nodes must match"
    assert t <= tg.num_snapshots + 1, \
        f"cannot add snapshot at time {t}, the temporal graph has only {tg.num_snapshots} snapshots"
    if t < 1:
        raise IndexError(f"time index {t} out of range 1:{tg.num_snapshots + 1}")   # Julia's insert! BoundsError
    snapshots = list(tg.snapshots)
    snapshots.insert(t - 1, g)
    return TemporalSnapshotsGNNGraph(snapshots)


def remove_snapshot(tg: TemporalSnapshotsGNNGraph, t: int) -> TemporalSnapshotsGNNGraph:
    """GNNGraphs/src/temporalsnapshotsgnngraph.jl:192-201: a new temporal graph without the snapshot at time index t
    (1-based).  tg is not changed."""
    if not 1 <= t <= tg.num_snapshots:
        raise IndexError(f"time index {t} out of range 1:{tg.num_snapshots}")         # Julia's deleteat! BoundsError
    snapshots = list(tg.snapshots)
    del snapshots[t - 1]
    return TemporalSnapshotsGNNGraph(snapshots)


def initialstates(layer_or_cell):
    """Flux.initialstates of a cell or of a GNNRecurrence"""
    return layer_or_cell.initialstates()


class GNNRecurrence(GNNLayer):
    """GNNRecurrence(cell) — temporalconv.jl:121-135.  layer(g, x[, state]):
      GNNGraph: x (in, T, N) -> y (out, T, N);  TemporalSnapshotsGNNGraph: x a list of (in, N_t) -> a list."""

    def __init__(self, cell):
        super().__init__()
        self.cell = cell

    def initialstates(self):
        return self.cell.initialstates()

    def forward(self, g, x, state=None):
        if isinstance(g, TemporalSnapshotsGNNGraph):
            if len(x) != g.num_snapshots:
                raise ValueError(f"{len(x)} feature arrays for {g.num_snapshots} snapshots")
            if len(x) == 0:
                raise ValueError("a sequence needs at least one time step (T = 0)")
            if not isinstance(self.cell, EvolveGCNOCell):
                assert len(set(g.num_nodes)) == 1, \
                    f"{type(self.cell).__name__} keeps a state per node: every snapshot needs the same node count"
            ys = []
            for gt, xt in zip(g.snapshots, x):
                yt, state = self.cell(gt, xt, state)
                ys.append(yt)
            return ys
        y, _ = self.cell._sequence(g, x, state)
        return y

    def __repr__(self):
        return f"GNNRecurrence({self.cell!r})"


def GConvGRU(ch_in, ch_out, k, **kw):
    return GNNRecurrence(GConvGRUCell(ch_in, ch_out, k, **kw))


def GConvLSTM(ch_in, ch_out, k, **kw):
    return GNNRecurrence(GConvLSTMCell(ch_in, ch_out, k, **kw))


def DCGRU(ch_in, ch_out, k, **kw):
    return GNNRecurrence(DCGRUCell(ch_in, ch_out, k, **kw))


def TGCN(ch_in, ch_out, **kw):
    return GNNRecurrence(TGCNCell(ch_in, ch_out, **kw))


def EvolveGCNO(ch_in, ch_out, **kw):
    return GNNRecurrence(EvolveGCNOCell(ch_in, ch_out, **kw))
