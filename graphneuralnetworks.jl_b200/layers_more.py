"""The rest of the reference's functional layers (GNNlib/src/layers/conv.jl) — callers of the same hot path, written as
the reference writes them: dense per-node / per-edge algebra around `propagate`, `apply_edges`, `aggregate_neighbors`.

    cheb_conv              conv.jl:83-98        (X·L̃ through the fused propagate; λmax by Lanczos on the device)
                                                (its basis, cheb_basis, and DConv's, diffusion_basis, also serve temporal.py)
    edge_conv              conv.jl:237-246
    nn_conv                conv.jl:260-273
    res_gated_graph_conv   conv.jl:287-300
    cg_conv                conv.jl:304-333
    megnet_conv            conv.jl:356-368
    gmm_conv               conv.jl:372-401
    egnn_conv              conv.jl:459-495
    d_conv                 conv.jl:696-724

and their Flux-style parameter holders (GraphNeuralNetworks/src/layers/conv.jl).  `l` is duck-typed as in the reference.
Arrays are Julia-shaped (features first, nodes / edges last).
"""
from __future__ import annotations

import math
import operator
from typing import Callable, Optional

import numpy as np
import torch

from .basic import _EdgeFeatureLayer, GNNLayer
from .graph import GNNGraph, degree, edge_features, homogeneous_only, node_features, rows, unrows
from .layers import (_add_bias, _bias, _Dense, _DenseAct, _jl_reshape3, _matmul, _sigma, glorot_uniform, identity,
                     relu)
from .msgpass import (Fix1, aggregate_neighbors, apply_edges, check_num_edges, check_num_nodes, e_mul_xj,
                      expand_srcdst, mean, propagate, w_mul_xj, xi_sub_xj)


def _field(l, *names):
    """first attribute of `l` among `names` (Greek field names of the reference and their ASCII spellings)"""
    for n in names:
        if hasattr(l, n):
            return getattr(l, n)
    raise AttributeError(f"{type(l).__name__} has none of the fields {names}")


def _vcat(*xs: torch.Tensor) -> torch.Tensor:
    """Julia vcat of (d_i, M) arrays -> (Σ d_i, M), staying column-major"""
    return unrows(torch.cat([rows(x) for x in xs], dim=1))


# ------------------------------------------------------------------------------------------------ ChebConv
def _normalized_adjacency_mul(g: GNNGraph, X: torch.Tensor, c: torch.Tensor) -> torch.Tensor:
    """X * (D^-1/2 A D^-1/2) for dir = :out adjacency: column j collects the rows of its in-neighbours"""
    return propagate(w_mul_xj, g, operator.add, xj=X * c.reshape(1, -1)) * c.reshape(1, -1)


def _lambda_max(g: GNNGraph, c: torch.Tensor, steps: int = 64) -> float:
    """largest eigenvalue of L = I - D^-1/2 A D^-1/2 (the reference: KrylovKit.eigsolve(Symmetric(L), x0, 1, :LR),
    GNNGraphs/src/query.jl:482-485): Lanczos with full re-orthogonalisation; the products run on the device."""
    n = g.num_nodes
    dev = c.device
    gen = torch.Generator(device="cpu").manual_seed(17)
    v = torch.randn(n, generator=gen, dtype=torch.float64).to(dev)
    v = v / v.norm()
    V, alpha, beta = [v], [], []                               # Lanczos vectors stay in float64; the operator is fp32
    m = min(n, steps)
    for j in range(m):
        x = V[-1].float().reshape(1, -1)
        w = V[-1] - _normalized_adjacency_mul(g, x, c).reshape(-1).double()
        a = float(w @ V[-1])
        alpha.append(a)
        for _ in range(2):                                     # full re-orthogonalisation, twice
            for u in V:
                w = w - (w @ u) * u
        b = float(w.norm())
        if b < 1e-5 or j == m - 1:                             # invariant subspace reached (fp32 operator noise ~1e-7)
            break
        beta.append(b)
        V.append(w / b)
    T = np.diag(alpha) + np.diag(beta[:len(alpha) - 1], 1) + np.diag(beta[:len(alpha) - 1], -1)
    return float(np.linalg.eigvalsh(T)[-1])


def scaled_laplacian_mul(g: GNNGraph, X: torch.Tensor, c: torch.Tensor, lmax: float) -> torch.Tensor:
    """X * L̃ with L̃ = 2/λmax (I - D^-1/2 A D^-1/2) - I — scaled_laplacian, GNNGraphs/src/query.jl:474-479"""
    return (2.0 / lmax) * (X - _normalized_adjacency_mul(g, X, c)) - X


def cheb_operator(g: GNNGraph):
    """(c, λmax) of L̃ = 2/λmax (I - D^-1/2 A D^-1/2) - I: c = 1 ./ sqrt.(out-degree); λmax is cached on the graph"""
    d = degree(g, torch.float32, dir="out")
    assert bool((d != 0).all()), "Graph contains isolated nodes, cannot compute `normalized_adjacency`."
    c = 1.0 / torch.sqrt(d)
    cache = getattr(g, "_lmax_cache", None)
    if cache is None:
        cache = _lambda_max(g, c)
        g._lmax_cache = cache
    return c, cache


def cheb_basis(g: GNNGraph, X: torch.Tensor, k: int, op=None) -> list:
    """[Z_0, ..., Z_{k-1}] of cheb_conv (conv.jl:90-97), k >= 2: Z_0 = X, Z_1 = X L̃, Z_j = 2 Z_{j-1} L̃ - Z_{j-2}.
    X is (D, N): each column of the propagate is reduced on its own, so the basis of a (D·T, N) view is every time
    step's basis at once, and the basis of a vcat is the vcat of the bases.  op: cheb_operator(g), when known."""
    c, lmax = cheb_operator(g) if op is None else op
    Z_prev = X
    Z = scaled_laplacian_mul(g, X, c, lmax)
    basis = [Z_prev, Z]
    for _ in range(2, int(k)):
        Z, Z_prev = 2 * scaled_laplacian_mul(g, Z, c, lmax) - Z_prev, Z
        basis.append(Z)
    return basis


def cheb_conv(l, g: GNNGraph, X: torch.Tensor) -> torch.Tensor:
    """GNNlib/src/layers/conv.jl:83-98.  l.weight is (out, in, k), k >= 2 as in the reference."""
    homogeneous_only(g, "cheb_conv")
    check_num_nodes(g, X)
    assert X.shape[0] == l.weight.shape[1], "Input feature size must match input channel size."
    Z = cheb_basis(g, X, int(l.k))
    Y = _matmul(l.weight[:, :, 0], Z[0]) + _matmul(l.weight[:, :, 1], Z[1])
    for k in range(2, int(l.k)):
        Y = Y + _matmul(l.weight[:, :, k], Z[k])
    return _add_bias(Y, _bias(l))


# ------------------------------------------------------------------------------------------------ EdgeConv / NNConv
def edge_conv_message(l, xi, xj, e):
    return l.nn(_vcat(xi, xj - xi))


def edge_conv(l, g: GNNGraph, x: torch.Tensor) -> torch.Tensor:
    """GNNlib/src/layers/conv.jl:237-246"""
    check_num_nodes(g, x)
    xj, xi = expand_srcdst(g, x)
    return propagate(Fix1(edge_conv_message, l), g, l.aggr, xi=xi, xj=xj, e=None)


def nn_conv_message(l, xi, xj, e):
    """conv.jl:267-273: W = reshape(nn(e), (:, nin, E)); m[:, k] = W[:, :, k] * xj[:, k]"""
    nin = xj.shape[0]
    We = rows(l.nn(e))                                         # (E, out*nin), column index o + out*i
    W = We.reshape(We.shape[0], nin, -1)                       # (E, nin, out)
    return unrows(torch.einsum("kio,ki->ko", W, rows(xj)))


def nn_conv(l, g: GNNGraph, x: torch.Tensor, e: torch.Tensor) -> torch.Tensor:
    """GNNlib/src/layers/conv.jl:260-265"""
    homogeneous_only(g, "nn_conv")
    check_num_nodes(g, x)
    m = propagate(Fix1(nn_conv_message, l), g, l.aggr, xj=x, e=e)
    return _sigma(l)(_add_bias(_matmul(l.weight, x) + m, _bias(l)))


# ------------------------------------------------------------------------------------------------ ResGatedGraphConv / CGConv
def res_gated_graph_conv(l, g: GNNGraph, x: torch.Tensor) -> torch.Tensor:
    """GNNlib/src/layers/conv.jl:287-300"""
    check_num_nodes(g, x)
    xj, xi = expand_srcdst(g, x)

    def message(xi, xj, e):
        return torch.sigmoid(xi["Ax"] + xj["Bx"]) * xj["Vx"]

    m = propagate(message, g, operator.add, xi={"Ax": _matmul(l.A, xi)}, xj={"Bx": _matmul(l.B, xj), "Vx": _matmul(l.V, xj)})
    return _sigma(l)(_add_bias(_matmul(l.U, xi) + m, _bias(l)))


def cg_message(l, xi, xj, e):
    z = _vcat(xi, xj, e) if e is not None else _vcat(xi, xj)
    return l.dense_f(z) * l.dense_s(z)


def cg_conv(l, g: GNNGraph, x: torch.Tensor, e: Optional[torch.Tensor] = None) -> torch.Tensor:
    """GNNlib/src/layers/conv.jl:304-324"""
    check_num_nodes(g, x)
    xj, xi = expand_srcdst(g, x)
    if e is not None:
        check_num_edges(g, e)
    m = propagate(Fix1(cg_message, l), g, operator.add, xi=xi, xj=xj, e=e)
    if l.residual and xi.shape[0] == m.shape[0]:               # otherwise the reference only warns
        m = m + xi
    return m


# ------------------------------------------------------------------------------------------------ MEGNet / GMM / EGNN
def megnet_conv(l, g: GNNGraph, x: torch.Tensor, e: torch.Tensor):
    """GNNlib/src/layers/conv.jl:356-368: returns (x̄, ē)"""
    homogeneous_only(g, "megnet_conv")
    check_num_nodes(g, x)
    phi_e = _field(l, "\u03d5e", "\u03c6e", "phi_e")              # ϕe (Python NFKC-normalises ϕ to φ in identifiers)
    phi_v = _field(l, "\u03d5v", "\u03c6v", "phi_v")
    ebar = apply_edges(lambda xi, xj, ee: phi_e(_vcat(xi, xj, ee)), g, xi=x, xj=x, e=e)
    xe = aggregate_neighbors(g, l.aggr, ebar)
    return phi_v(_vcat(x, xe)), ebar


def gmm_conv(l, g: GNNGraph, x: torch.Tensor, e: torch.Tensor) -> torch.Tensor:
    """GNNlib/src/layers/conv.jl:372-401, statement for statement (including the sign of the exponent)."""
    homogeneous_only(g, "gmm_conv")
    (nin, ein), out = l.ch
    assert ein == e.shape[0] and g.num_edges == e.shape[1], "Pseudo-cordinate dimension is not equal to (ein,num_edge)"
    w = e.unsqueeze(1)                                         # (ein, 1, E)
    mu = l.mu.unsqueeze(-1)                                    # (ein, K, 1)
    w = ((w - mu) ** 2) / 2
    w = w * (l.sigma_inv ** 2).unsqueeze(-1)
    w = torch.exp(w.sum(dim=0, keepdim=True))                  # (1, K, E)
    xj = _jl_reshape3(l.dense_x(x), out, l.K)                  # (out, K, N)
    m = propagate(e_mul_xj, g, mean, xj=xj, e=w)
    m = m.mean(dim=1)                                          # (out, N)
    m = _sigma(l)(_add_bias(m, _bias(l)))
    if l.residual and x.shape[0] == m.shape[0]:
        m = m + x
    return m


def egnn_message(l, xi, xj, e):
    f = [xi["h"], xj["h"], e["sqnorm_xdiff"]]
    if l.num_features["edge"] > 0:
        f.append(e["e"])
    phi_e = _field(l, "\u03d5e", "\u03c6e", "phi_e")
    phi_x = _field(l, "\u03d5x", "\u03c6x", "phi_x")
    msg_h = phi_e(_vcat(*f))
    return {"x": phi_x(msg_h) * e["x_diff"], "h": msg_h}


def egnn_conv(l, g: GNNGraph, h: torch.Tensor, x: torch.Tensor, e: Optional[torch.Tensor] = None):
    """GNNlib/src/layers/conv.jl:459-483: returns (h, x)"""
    homogeneous_only(g, "egnn_conv")
    if l.num_features["edge"] > 0:
        assert e is not None, "Edge features must be provided."
    assert h.shape[0] == l.num_features["in"], "Input features must match layer input size."
    x_diff = apply_edges(xi_sub_xj, g, x, x)
    sqnorm = (x_diff ** 2).sum(dim=0, keepdim=True)
    x_diff = x_diff / (torch.sqrt(sqnorm) + 1.0e-6)
    msg = apply_edges(Fix1(egnn_message, l), g, xi={"h": h}, xj={"h": h},
                      e={"e": e, "x_diff": x_diff, "sqnorm_xdiff": sqnorm})
    h_aggr = aggregate_neighbors(g, operator.add, msg["h"])
    x_aggr = aggregate_neighbors(g, mean, msg["x"])
    phi_h = _field(l, "\u03d5h", "\u03c6h", "phi_h")
    hnew = phi_h(_vcat(h, h_aggr))
    h = h + hnew if l.residual else hnew
    return h, x + x_aggr


# ------------------------------------------------------------------------------------------------ DConv
def transposed_graph(g: GNNGraph) -> GNNGraph:
    """the reversed graph DConv diffuses on (conv.jl:697), with its plan, cached on the (immutable) graph"""
    gt = getattr(g, "_dconv_gt", None)
    if gt is None:
        gt = GNNGraph(g.t, g.s, g.w, num_nodes=g.num_nodes)
        g._dconv_gt = gt
    return gt


def diffusion_basis(g: GNNGraph, x: torch.Tensor, k: int, gt: Optional[GNNGraph] = None) -> list:
    """The terms of d_conv (conv.jl:696-724) as [(j, T_in, T_out), ...]: h = Σ W[1, j] T_in + W[2, j] T_out (Julia
    indices; j 0-based here).  The reference's recurrence keeps T0 = x and applies weights[:, 2] to both the first and
    the second diffusion step, and so does this.  x is (D, N); see cheb_basis for (D·T, N) views."""
    if gt is None:
        gt = GNNGraph(g.t, g.s, g.w, num_nodes=g.num_nodes)
    deg_out = degree(g, torch.float32, dir="out").reshape(1, -1)
    deg_in = degree(g, torch.float32, dir="in").reshape(1, -1)
    T0 = x
    terms = [(0, T0, T0)]
    if k > 1:
        T1_out = propagate(w_mul_xj, g, operator.add, xj=T0 * deg_out)
        T1_in = propagate(w_mul_xj, gt, operator.add, xj=T0 * deg_in)
        terms.append((1, T1_in, T1_out))
    for i in range(2, int(k) + 1):
        T2_in = 2 * propagate(w_mul_xj, gt, operator.add, xj=T1_in * deg_in) - T0
        T2_out = 2 * propagate(w_mul_xj, g, operator.add, xj=T1_out * deg_out) - T0
        terms.append((i - 1, T2_in, T2_out))
        T1_in, T1_out = T2_in, T2_out
    return terms


def d_conv(l, g: GNNGraph, x: torch.Tensor) -> torch.Tensor:
    """GNNlib/src/layers/conv.jl:696-724, statement for statement.  l.weights is (2, k, out, in)."""
    homogeneous_only(g, "d_conv")
    Wt = l.weights
    terms = diffusion_basis(g, x, int(l.k))
    h = _matmul(Wt[0, 0], x) + _matmul(Wt[1, 0], x)
    for j, T_in, T_out in terms[1:]:
        h = h + _matmul(Wt[0, j], T_in) + _matmul(Wt[1, j], T_out)
    return _add_bias(h, _bias(l))


# ------------------------------------------------------------------------------------------------ parameter holders
def swish(x):
    return x * torch.sigmoid(x)


class Chain(torch.nn.Sequential):
    """Flux.Chain of callables on Julia-shaped arrays"""


class ChebConv(GNNLayer):
    """ChebConv(in => out, k; bias=true) — GraphNeuralNetworks/src/layers/conv.jl:162-175"""

    def __init__(self, ch_in, ch_out, k: int, *, bias=True, device=None):
        super().__init__()
        self.weight = torch.nn.Parameter(torch.stack([glorot_uniform(ch_out, ch_in, device=device) for _ in range(k)], dim=2))
        self.bias = torch.nn.Parameter(torch.zeros(ch_out, device=device)) if bias else None
        self.k = int(k)

    def forward(self, g, x):
        return cheb_conv(self, g, x)


class EdgeConv(GNNLayer):
    """EdgeConv(nn; aggr=max) — conv.jl:575-585"""

    def __init__(self, nn: Callable, *, aggr=max):
        super().__init__()
        self.nn, self.aggr = nn, aggr

    def forward(self, g, x):
        return edge_conv(self, g, x)


class NNConv(_EdgeFeatureLayer):
    """NNConv(in => out, nn, σ=identity; aggr=+, bias=true) — conv.jl:701-717"""

    def __init__(self, ch_in, ch_out, nn: Callable, sigma: Callable = identity, *, aggr=operator.add, bias=True,
                 device=None):
        super().__init__()
        self.weight = torch.nn.Parameter(glorot_uniform(ch_out, ch_in, device=device))
        self.bias = torch.nn.Parameter(torch.zeros(ch_out, device=device)) if bias else None
        self.nn, self.sigma, self.aggr = nn, sigma, aggr

    def forward(self, g, x, e):
        return nn_conv(self, g, x, e)


class ResGatedGraphConv(GNNLayer):
    """ResGatedGraphConv(in => out, σ=identity; bias=true) — conv.jl:838-859"""

    def __init__(self, ch_in, ch_out, sigma: Callable = identity, *, bias=True, device=None):
        super().__init__()
        for name in ("A", "B", "U", "V"):
            setattr(self, name, torch.nn.Parameter(glorot_uniform(ch_out, ch_in, device=device)))
        self.bias = torch.nn.Parameter(torch.zeros(ch_out, device=device)) if bias else None
        self.sigma = sigma

    def forward(self, g, x):
        return res_gated_graph_conv(self, g, x)


class CGConv(_EdgeFeatureLayer):
    """CGConv((in, ein) => out, act=identity; bias=true, residual=false) — conv.jl:914-932"""

    def __init__(self, ch_in, ch_out, act: Callable = identity, *, residual=False, bias=True, device=None):
        super().__init__()
        nin, ein = ch_in if isinstance(ch_in, tuple) else (ch_in, 0)
        self.ch = ((nin, ein), ch_out)
        self.dense_f = _DenseAct(2 * nin + ein, ch_out, torch.sigmoid, bias=bias, device=device)
        self.dense_s = _DenseAct(2 * nin + ein, ch_out, act, bias=bias, device=device)
        self.residual = residual

    def forward(self, g, x, e=None):
        return cg_conv(self, g, x, e)


class MEGNetConv(GNNLayer):
    """MEGNetConv(ϕe, ϕv; aggr=mean) / MEGNetConv(in => out; aggr=mean) — conv.jl:1035-1055"""

    def __init__(self, a, b, *, aggr=mean, device=None):
        super().__init__()
        if isinstance(a, int):
            nin, nout = a, b
            a = Chain(_DenseAct(3 * nin, nout, relu, device=device), _Dense(nout, nout, device=device))
            b = Chain(_DenseAct(nin + nout, nout, relu, device=device), _Dense(nout, nout, device=device))
        self.phi_e, self.phi_v, self.aggr = a, b, aggr

    def forward(self, g, x, e):
        return megnet_conv(self, g, x, e)

    def graph_forward(self, g):
        """conv.jl:1056-1059: both the node and the edge features are replaced"""
        x, e = self(g, node_features(g), edge_features(g))
        return GNNGraph(g, ndata=x, edata=e)


class GMMConv(_EdgeFeatureLayer):
    """GMMConv((in, ein) => out, σ=identity; K=1, bias=true, residual=false) — conv.jl:1111-1137"""

    def __init__(self, ch_in, ch_out, sigma: Callable = identity, *, K: int = 1, bias=True, residual=False, device=None):
        super().__init__()
        nin, ein = ch_in
        self.mu = torch.nn.Parameter(glorot_uniform(ein, K, device=device))
        self.sigma_inv = torch.nn.Parameter(glorot_uniform(ein, K, device=device))
        self.bias = torch.nn.Parameter(torch.zeros(ch_out, device=device)) if bias else None
        self.sigma, self.ch, self.K, self.residual = sigma, ((nin, ein), ch_out), int(K), residual
        self.dense_x = _Dense(nin, ch_out * K, bias=False, device=device)

    def forward(self, g, x, e):
        return gmm_conv(self, g, x, e)


class EGNNConv(GNNLayer):
    """EGNNConv((in, ein) => out; hidden_size=2in, residual=false) — conv.jl:1349-1386"""

    def __init__(self, ch_in, ch_out, *, hidden_size: Optional[int] = None, residual=False, device=None):
        super().__init__()
        nin, ein = ch_in if isinstance(ch_in, tuple) else (ch_in, 0)
        hid = 2 * nin if hidden_size is None else int(hidden_size)
        self.phi_e = Chain(_DenseAct(2 * nin + ein + 1, hid, swish, device=device), _DenseAct(hid, hid, swish, device=device))
        self.phi_h = Chain(_DenseAct(nin + hid, hid, swish, device=device), _Dense(hid, ch_out, device=device))
        self.phi_x = Chain(_DenseAct(hid, hid, swish, device=device), _Dense(hid, 1, bias=False, device=device))
        self.num_features = {"in": nin, "edge": ein, "out": ch_out, "hidden": hid}
        if residual:
            assert nin == ch_out, "Residual connection only possible if in_size == out_size"
        self.residual = residual

    def forward(self, g, h, x, e=None):
        return egnn_conv(self, g, h, x, e)


class DConv(GNNLayer):
    """DConv(in => out, k; bias=true) — conv.jl:1574-1589.  weights is (2, k, out, in)."""

    def __init__(self, ch_in, ch_out, k: int, *, bias=True, device=None):
        super().__init__()
        s = math.sqrt(6.0 / (ch_in + ch_out))
        self.weights = torch.nn.Parameter((torch.rand(2, k, ch_out, ch_in, device=device) * 2 - 1) * s)
        self.bias = torch.nn.Parameter(torch.zeros(ch_out, device=device)) if bias else None
        self.k, self.ch_in, self.ch_out = int(k), ch_in, ch_out

    def forward(self, g, x):
        return d_conv(self, g, x)
