"""The remaining functional layers (graphneuralnetworks.jl_b200/layers_more.py: cheb, edge, nn, res-gated, cg, megnet,
gmm, egnn, d conv) against float64 formulas written with dense adjacency matrices / explicit per-edge loops — no code
shared with the mirror.  Forward, and the gradients of the inputs, of every parameter and of the edge weights and
features each case uses.  Back ends: the CPU test double and (under -m gpu) CUDA."""
import operator

import numpy as np
import pytest
import torch

F64 = torch.float64
CPU = torch.device("cpu")


def c64(a):
    return a.detach().to(device=CPU, dtype=F64) if isinstance(a, torch.Tensor) else torch.as_tensor(np.asarray(a), dtype=F64)


def rel(a, b):
    a, b = c64(a), c64(b)
    return float((a - b).norm() / max(float(b.norm()), 1e-30))


def setup(gnn, rng, dev, n=25, E=140, weights=False, bidirected=False, simple=False, loops=True):
    s = rng.integers(1, n + 1, E); t = rng.integers(1, n + 1, E)
    s[:n] = np.arange(1, n + 1); t[:n] = np.roll(np.arange(1, n + 1), 1)        # every node has an in- and an out-edge
    if not loops:                                                                # x_i - x_i = 0: sqrt'(0) is NaN (there too)
        t = np.where(s == t, t % n + 1, t)
    if simple:                                                                   # no repeated (s, t): no ties under max
        _, first = np.unique(s * (n + 1) + t, return_index=True)
        s, t = s[np.sort(first)], t[np.sort(first)]
    w = rng.uniform(0.5, 1.5, len(s)) if weights else None
    if bidirected:
        s, t = np.concatenate([s, t]), np.concatenate([t, s])
        w = None if w is None else np.concatenate([w, w])
    g = gnn.GNNGraph(torch.as_tensor(s).to(dev), torch.as_tensor(t).to(dev),
                     None if w is None else torch.as_tensor(w, dtype=torch.float32).to(dev), num_nodes=n)
    A = torch.zeros(n, n, dtype=F64)                                              # A[i, j] = weight of edges i -> j
    A.index_put_((torch.as_tensor(s - 1), torch.as_tensor(t - 1)),
                 torch.ones(len(s), dtype=F64) if w is None else c64(g.w), accumulate=True)
    return g, torch.as_tensor(s - 1), torch.as_tensor(t - 1), A


def jl(gnn, a, dev, grad=False):
    x = gnn.unrows(torch.as_tensor(np.ascontiguousarray(a), dtype=torch.float32).to(dev))
    return x.requires_grad_(True) if grad else x


class Twins:
    """float64 twins, requiring grad, of every parameter of the modules: P(param) is the twin the reference formula
    uses, P.pairs(*modules) the (parameter, twin) pairs of those modules (all of them by default) for grads_match."""

    def __init__(self, *modules):
        self._twin, self._all = {}, []
        for m in modules:
            for _, p in m.named_parameters():
                if id(p) not in self._twin:
                    self._twin[id(p)] = c64(p).requires_grad_(True)
                    self._all.append(p)

    def __call__(self, p):
        return self._twin[id(p)]

    def pairs(self, *modules):
        ps = [p for m in modules for _, p in m.named_parameters()] if modules else self._all
        return [(p, self._twin[id(p)]) for p in ps]


def grads_match(gnn, out, ref_out, pairs, tol):
    """the same seeded cotangent through both graphs, then the gradient of every (mirror leaf, float64 reference leaf)
    pair compared; a Julia-shaped mirror leaf (D, N) / (D, E) meets its reference in rows"""
    cot = torch.randn(ref_out.shape, dtype=F64, generator=torch.Generator().manual_seed(3))
    got = torch.autograd.grad((gnn.rows(out).double() * cot.to(out.device)).sum(), [m for m, _ in pairs],
                              retain_graph=True)
    want = torch.autograd.grad((ref_out * cot).sum(), [r for _, r in pairs], retain_graph=True)
    for i, (a, b) in enumerate(zip(got, want)):
        if a.shape != b.shape:
            a = gnn.rows(a)
        assert a.shape == b.shape
        err = rel(a, b)
        assert err < tol, f"gradient of input {i} {tuple(b.shape)}: {err:.2e}"


def dense(d, v, P):
    y = v @ P(d.weight).t()
    if d.bias is not None:
        y = y + P(d.bias)
    sig = getattr(d, "sigma", None)
    return sig(y) if sig is not None else y


def seq(chain, v, P):
    for d in chain:
        v = dense(d, v, P)
    return v


def scatter_sum(idx, m, n):
    return torch.zeros((n,) + tuple(m.shape[1:]), dtype=m.dtype).index_add(0, idx, m)


def randomise_biases(rng, module):
    with torch.no_grad():
        for name, p in module.named_parameters():
            if name.endswith("bias"):
                p.copy_(torch.as_tensor(rng.standard_normal(tuple(p.shape)), dtype=torch.float32))


@pytest.mark.parametrize("k,weights", [(2, False), (4, False), (3, True)])
def test_cheb_conv(gnn, be, k, weights):
    be, rng = be, np.random.default_rng(0)
    g, s, t, A = setup(gnn, rng, be.dev, weights=weights, bidirected=True)       # symmetric, as scaled_laplacian assumes
    n, Din, Dout = g.num_nodes, 4, 3
    layer = gnn.ChebConv(Din, Dout, k, device=be.dev)
    randomise_biases(rng, layer)
    P = Twins(layer)
    x = rng.standard_normal((n, Din))
    xt, xr = jl(gnn, x, be.dev, True), c64(x).requires_grad_(True)
    out = layer(g, xt)
    dinv = torch.diag(1 / A.sum(1).sqrt())
    L = torch.eye(n, dtype=F64) - dinv @ A @ dinv
    Lt = 2 / torch.linalg.eigvalsh((L + L.t()) / 2)[-1] * L - torch.eye(n, dtype=F64)
    W = P(layer.weight)
    Zp, Z = xr, Lt.t() @ xr                                                       # rows form of X * L̃
    Y = Zp @ W[:, :, 0].t() + Z @ W[:, :, 1].t()
    for i in range(2, k):
        Z, Zp = 2 * Lt.t() @ Z - Zp, Z
        Y = Y + Z @ W[:, :, i].t()
    ref = Y + P(layer.bias)
    assert out.shape == (Dout, n)
    assert rel(gnn.rows(out), ref) < 2e-5 * be.tol
    # x and the parameters; edge weights reach L̃ through an iterative λmax estimate (KrylovKit there, Lanczos here)
    # whose derivative neither side defines, so their gradient is not compared
    grads_match(gnn, out, ref, [(xt, xr)] + P.pairs(), 1e-4 * be.tol)
    with pytest.raises(AssertionError, match="input channel size"):
        layer(g, jl(gnn, rng.standard_normal((n, Din + 1)), be.dev))


@pytest.mark.parametrize("aggr", ["max", "+"])
def test_edge_conv(gnn, be, aggr):
    be, rng = be, np.random.default_rng(1)
    g, s, t, A = setup(gnn, rng, be.dev, simple=True)     # with repeated edges NNlib's max pullback feeds every tied
    n, Din, Dout = g.num_nodes, 4, 5                      # message, torch's amax splits the gradient: not comparable
    nn = gnn.layers._DenseAct(2 * Din, Dout, torch.tanh, device=be.dev)
    randomise_biases(rng, nn)
    P = Twins(nn)
    layer = gnn.EdgeConv(nn, aggr=max if aggr == "max" else operator.add)
    x = rng.standard_normal((n, Din))
    xt, xr = jl(gnn, x, be.dev, True), c64(x).requires_grad_(True)
    out = layer(g, xt)
    m = dense(nn, torch.cat([xr[t], xr[s] - xr[t]], dim=1), P)
    if aggr == "+":
        ref = scatter_sum(t, m, n)
    else:
        ref = torch.full((n, Dout), -float("inf"), dtype=F64).scatter_reduce(0, t[:, None].expand_as(m), m, "amax")
    assert rel(gnn.rows(out), ref) < 3e-6 * be.tol
    grads_match(gnn, out, ref, [(xt, xr)] + P.pairs(), 3e-5 * be.tol)


def test_nn_conv(gnn, be):
    be, rng = be, np.random.default_rng(2)
    g, s, t, A = setup(gnn, rng, be.dev)
    n, E, Din, Dout, De = g.num_nodes, g.num_edges, 3, 4, 2
    nn = gnn.layers._Dense(De, Dout * Din, device=be.dev)
    randomise_biases(rng, nn)
    layer = gnn.NNConv(Din, Dout, nn, torch.tanh, aggr=gnn.mean, device=be.dev)
    randomise_biases(rng, layer)
    P = Twins(layer)
    x, e = rng.standard_normal((n, Din)), rng.standard_normal((E, De))
    xt, xr = jl(gnn, x, be.dev, True), c64(x).requires_grad_(True)
    et, er = jl(gnn, e, be.dev, True), c64(e).requires_grad_(True)
    out = layer(g, xt, et)
    We = dense(nn, er, P)                                                         # (E, Dout*Din), Julia column o + Dout*i
    m = torch.stack([sum(We[:, o + Dout * i] * xr[s, i] for i in range(Din)) for o in range(Dout)], dim=1)
    cnt = torch.bincount(t, minlength=n).clamp(min=1).double()
    ref = torch.tanh(xr @ P(layer.weight).t() + scatter_sum(t, m, n) / cnt[:, None] + P(layer.bias))
    assert rel(gnn.rows(out), ref) < 3e-6 * be.tol
    assert len(P.pairs()) == 4                                                    # nn's W, b and the layer's
    grads_match(gnn, out, ref, [(xt, xr), (et, er)] + P.pairs(), 3e-5 * be.tol)


def test_res_gated_and_cg_conv(gnn, be):
    be, rng = be, np.random.default_rng(3)
    g, s, t, A = setup(gnn, rng, be.dev)
    n, E, Din, Dout, De = g.num_nodes, g.num_edges, 4, 4, 3
    x, e = rng.standard_normal((n, Din)), rng.standard_normal((E, De))
    xt, xr = jl(gnn, x, be.dev, True), c64(x).requires_grad_(True)
    layer = gnn.ResGatedGraphConv(Din, Dout, torch.relu, device=be.dev)
    randomise_biases(rng, layer)
    P = Twins(layer)
    out = layer(g, xt)
    Aw, Bw, Uw, Vw = (P(p) for p in (layer.A, layer.B, layer.U, layer.V))
    eta = torch.sigmoid((xr @ Aw.t())[t] + (xr @ Bw.t())[s])
    ref = torch.relu(xr @ Uw.t() + scatter_sum(t, eta * (xr @ Vw.t())[s], n) + P(layer.bias))
    assert rel(gnn.rows(out), ref) < 3e-6 * be.tol
    grads_match(gnn, out, ref, [(xt, xr)] + P.pairs(), 3e-5 * be.tol)
    for ein, residual in ((De, True), (0, False)):
        layer = gnn.CGConv((Din, ein), Dout, torch.tanh, residual=residual, device=be.dev)
        randomise_biases(rng, layer)
        P = Twins(layer)
        pairs = [(xt, xr)] + P.pairs()
        if ein:
            et, er = jl(gnn, e, be.dev, True), c64(e).requires_grad_(True)
            pairs.append((et, er))
        else:
            et = None
        out = layer(g, xt, et)
        z = torch.cat([xr[t], xr[s]] + ([er] if ein else []), dim=1)
        ref = scatter_sum(t, dense(layer.dense_f, z, P) * dense(layer.dense_s, z, P), n) + (xr if residual else 0)
        assert rel(gnn.rows(out), ref) < 3e-6 * be.tol
        grads_match(gnn, out, ref, pairs, 3e-5 * be.tol)
    with pytest.raises(AssertionError):
        layer(g, xt, jl(gnn, e[:-1], be.dev))


def test_megnet_conv(gnn, be):
    be, rng = be, np.random.default_rng(4)
    g, s, t, A = setup(gnn, rng, be.dev)
    n, E, Din, Dout = g.num_nodes, g.num_edges, 3, 5
    layer = gnn.MEGNetConv(Din, Dout, device=be.dev)
    randomise_biases(rng, layer)
    P = Twins(layer)
    x, e = rng.standard_normal((n, Din)), rng.standard_normal((E, Din))
    xt, xr = jl(gnn, x, be.dev, True), c64(x).requires_grad_(True)
    et, er = jl(gnn, e, be.dev, True), c64(e).requires_grad_(True)
    xbar, ebar = layer(g, xt, et)
    eb = seq(layer.phi_e, torch.cat([xr[t], xr[s], er], dim=1), P)
    cnt = torch.bincount(t, minlength=n).clamp(min=1).double()
    xb = seq(layer.phi_v, torch.cat([xr, scatter_sum(t, eb, n) / cnt[:, None]], dim=1), P)
    assert xbar.shape == (Dout, n) and ebar.shape == (Dout, E)
    assert rel(gnn.rows(ebar), eb) < 3e-6 * be.tol and rel(gnn.rows(xbar), xb) < 3e-6 * be.tol
    grads_match(gnn, xbar, xb, [(xt, xr), (et, er)] + P.pairs(), 3e-5 * be.tol)
    grads_match(gnn, ebar, eb, [(xt, xr), (et, er)] + P.pairs(layer.phi_e), 3e-5 * be.tol)


@pytest.mark.parametrize("K,residual", [(1, False), (3, True)])
def test_gmm_conv(gnn, be, K, residual):
    be, rng = be, np.random.default_rng(5)
    g, s, t, A = setup(gnn, rng, be.dev)
    n, E, Din, ein = g.num_nodes, g.num_edges, 4, 2
    Dout = Din if residual else 3
    layer = gnn.GMMConv((Din, ein), Dout, torch.tanh, K=K, residual=residual, device=be.dev)
    randomise_biases(rng, layer)
    P = Twins(layer)
    x, e = rng.standard_normal((n, Din)), rng.uniform(-1, 1, (E, ein))
    xt, xr = jl(gnn, x, be.dev, True), c64(x).requires_grad_(True)
    et, er = jl(gnn, e, be.dev, True), c64(e).requires_grad_(True)
    out = layer(g, xt, et)
    mu, si = P(layer.mu), P(layer.sigma_inv)                                      # (ein, K)
    wk = torch.exp((((er[:, :, None] - mu[None]) ** 2) / 2 * si[None] ** 2).sum(1))            # (E, K)
    xk = (xr @ P(layer.dense_x.weight).t()).reshape(n, K, Dout)                   # Julia (out, K, N) -> rows (N, K, out)
    cnt = torch.bincount(t, minlength=n).clamp(min=1).double()
    m = scatter_sum(t, wk[:, :, None] * xk[s], n) / cnt[:, None, None]
    ref = torch.tanh(m.mean(1) + P(layer.bias)) + (xr if residual else 0)
    assert out.shape == (Dout, n)
    assert rel(gnn.rows(out), ref) < 3e-6 * be.tol
    grads_match(gnn, out, ref, [(xt, xr), (et, er)] + P.pairs(), 3e-5 * be.tol)
    with pytest.raises(AssertionError, match="Pseudo-cordinate"):
        layer(g, xt, jl(gnn, rng.standard_normal((E, ein + 1)), be.dev))


@pytest.mark.parametrize("ein,residual", [(0, False), (2, True)])
def test_egnn_conv(gnn, be, ein, residual):
    be, rng = be, np.random.default_rng(6)
    g, s, t, A = setup(gnn, rng, be.dev, loops=False)
    n, E, hin, Dx = g.num_nodes, g.num_edges, 5, 3
    layer = gnn.EGNNConv((hin, ein), hin, hidden_size=6, residual=residual, device=be.dev)
    randomise_biases(rng, layer)
    P = Twins(layer)
    h, x, e = rng.standard_normal((n, hin)), rng.standard_normal((n, Dx)), rng.standard_normal((E, max(ein, 1)))
    ht, hr = jl(gnn, h, be.dev, True), c64(h).requires_grad_(True)
    xt, xr = jl(gnn, x, be.dev, True), c64(x).requires_grad_(True)
    inputs = [(ht, hr), (xt, xr)]
    if ein:
        et, er = jl(gnn, e, be.dev, True), c64(e).requires_grad_(True)
        inputs.append((et, er))
    else:
        et = None
    hnew, xnew = layer(g, ht, xt, et)
    xd = xr[t] - xr[s]
    sq = (xd ** 2).sum(1, keepdim=True)
    xd = xd / (sq.sqrt() + 1e-6)
    f = torch.cat([hr[t], hr[s], sq] + ([er] if ein else []), dim=1)
    mh = seq(layer.phi_e, f, P)
    mx = seq(layer.phi_x, mh, P) * xd
    cnt = torch.bincount(t, minlength=n).clamp(min=1).double()
    hn = seq(layer.phi_h, torch.cat([hr, scatter_sum(t, mh, n)], dim=1), P)
    href = hr + hn if residual else hn
    xref = xr + scatter_sum(t, mx, n) / cnt[:, None]
    assert hnew.shape == (hin, n) and xnew.shape == (Dx, n)
    assert rel(gnn.rows(hnew), href) < 5e-6 * be.tol and rel(gnn.rows(xnew), xref) < 5e-6 * be.tol
    grads_match(gnn, hnew, href, inputs + P.pairs(layer.phi_e, layer.phi_h), 5e-5 * be.tol)
    grads_match(gnn, xnew, xref, inputs + P.pairs(layer.phi_e, layer.phi_x), 5e-5 * be.tol)
    if ein:
        with pytest.raises(AssertionError, match="Edge features must be provided"):
            layer(g, ht, xt)


@pytest.mark.parametrize("k,weights", [(1, False), (2, True), (3, False)])
def test_d_conv(gnn, be, k, weights):
    be, rng = be, np.random.default_rng(7)
    g, s, t, A = setup(gnn, rng, be.dev, weights=weights)
    n, Din, Dout = g.num_nodes, 3, 4
    layer = gnn.DConv(Din, Dout, k, device=be.dev)
    randomise_biases(rng, layer)
    P = Twins(layer)
    x = rng.standard_normal((n, Din))
    xt, xr = jl(gnn, x, be.dev, True), c64(x).requires_grad_(True)
    pairs = [(xt, xr)] + P.pairs()
    if weights:                                                                   # GNNGraph keeps the tensor it is given
        g.w.requires_grad_(True)
        pairs.append((g.w, c64(g.w).requires_grad_(True)))
        A = torch.zeros(n, n, dtype=F64).index_put((s, t), pairs[-1][1], accumulate=True)
    out = layer(g, xt)
    W = P(layer.weights)                                                          # (2, k, out, in)
    dout, din = A.sum(1), A.sum(0)
    P_out = lambda v: A.t() @ (dout[:, None] * v)                                 # propagate(w_mul_xj, g, +; xj = v .* deg_out')
    P_in = lambda v: A @ (din[:, None] * v)                                       # the same on the reversed graph
    hsum = xr @ W[0, 0].t() + xr @ W[1, 0].t()
    T0 = xr
    if k > 1:
        T1o, T1i = P_out(T0), P_in(T0)
        hsum = hsum + T1i @ W[0, 1].t() + T1o @ W[1, 1].t()
    for i in range(2, k + 1):
        T2i, T2o = 2 * P_in(T1i) - T0, 2 * P_out(T1o) - T0
        hsum = hsum + T2i @ W[0, i - 1].t() + T2o @ W[1, i - 1].t()
        T1i, T1o = T2i, T2o
    ref = hsum + P(layer.bias)
    assert out.shape == (Dout, n)
    assert rel(gnn.rows(out), ref) < 5e-6 * be.tol
    grads_match(gnn, out, ref, pairs, 5e-5 * be.tol)
