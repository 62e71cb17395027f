"""Every layer of the mirror (graphneuralnetworks.jl_b200/layers.py, msgpass.py, readout.py), forward and gradients,
against an independent float64 formula written from the definition in the reference's docstrings with plain torch
index ops (no code shared with the mirror).  Each test runs on two back ends (fixture `be`):

  fake  — no GPU needed: tests/fake_abi.py (a numpy restatement of the C-ABI contract on host memory) is swapped in
          for libgnnb200, so what runs is every line of Python above the ABI: dispatch (fused vs generic), Julia-shape
          bookkeeping, autograd wiring, argument checks.  The fake itself is pinned on the C oracle first.  The CUDA
          kernels are NOT exercised by this variant.
  cuda  — `-m gpu`: the same bodies on the real library and kernels.
"""
import operator

import numpy as np
import pytest
import torch

F64 = torch.float64
CPU = torch.device("cpu")


def _c64(a):
    if isinstance(a, torch.Tensor):
        return a.detach().to(device=CPU, dtype=F64)
    return torch.as_tensor(np.asarray(a), dtype=F64)


def rel(a, b):
    a, b = _c64(a), _c64(b)
    return float((a - b).norm() / max(float(b.norm()), 1e-30))


def p64(param):
    """a layer parameter as a float64 CPU tensor for the reference formula"""
    return param.detach().to(device=CPU, dtype=F64)


def f32(a, dev):
    return torch.as_tensor(np.ascontiguousarray(a), dtype=torch.float32).to(dev)


# ------------------------------------------------------------------------------------------------ references
class Ref:
    """float64, row-major (N, D) restatement of the message-passing primitives with torch autograd."""

    def __init__(self, s, t, n):
        self.s = torch.as_tensor(np.asarray(s) - 1, dtype=torch.int64)
        self.t = torch.as_tensor(np.asarray(t) - 1, dtype=torch.int64)
        self.n = n

    def with_loops(self):
        loops = np.arange(1, self.n + 1)
        return Ref(np.concatenate([self.s.numpy() + 1, loops]), np.concatenate([self.t.numpy() + 1, loops]), self.n)

    def scatter_sum(self, m):
        return torch.zeros((self.n,) + tuple(m.shape[1:]), dtype=m.dtype).index_add(0, self.t, m)

    def indeg(self, w=None):
        w = torch.ones(len(self.t), dtype=F64) if w is None else w
        return torch.zeros(self.n, dtype=F64).index_add(0, self.t, w)

    def propagate(self, x, aggr="+", w=None):
        m = x[self.s]
        if w is not None:
            m = m * w.reshape((-1,) + (1,) * (m.dim() - 1))
        out = self.scatter_sum(m)
        if aggr == "mean":
            out = out / self.indeg().clamp(min=1).reshape((-1,) + (1,) * (m.dim() - 1))
        return out

    def softmax(self, e):
        idx = self.t.reshape((-1,) + (1,) * (e.dim() - 1)).expand_as(e)
        mx = torch.full((self.n,) + tuple(e.shape[1:]), -float("inf"), dtype=e.dtype).scatter_reduce(
            0, idx, e.detach(), "amax", include_self=True)
        ex = torch.exp(e - mx[self.t])
        return ex / self.scatter_sum(ex)[self.t]

    def gcn(self, x, w=None):
        c = 1.0 / torch.sqrt(self.indeg(w))
        return self.propagate(x * c[:, None], "+", w) * c[:, None]


class NT:
    def __init__(self, **kw):
        self.__dict__.update(kw)


def make_graph(gnn, rng, dev, n=40, E=260, weights=False):
    s = rng.integers(1, n + 1, E)
    t = rng.integers(1, n + 1, E)
    t[:n] = np.arange(1, n + 1)            # every node has an in-neighbour: no 1/sqrt(0) in the loop-less GCN cases
    w = f32(rng.uniform(0.5, 1.5, E), dev) if weights else None
    g = gnn.GNNGraph(torch.as_tensor(s).to(dev), torch.as_tensor(t).to(dev), w, num_nodes=n)
    return g, Ref(s, t, n), s, t


def jl(gnn, a, dev, requires_grad=False):
    """row-major numpy (N, D...) -> Julia-shaped float32 tensor on dev"""
    x = gnn.unrows(f32(a, dev))
    return x.requires_grad_(requires_grad) if requires_grad else x


def r64(a, requires_grad=False):
    x = torch.as_tensor(np.asarray(a), dtype=F64).clone()
    return x.requires_grad_(requires_grad) if requires_grad else x


class Twins:
    """float64 twins, requiring grad, of every parameter the holders own (named_parameters() of a module, the tensor
    fields of an NT that require grad).  P(param) is the twin the reference formula uses; P.pairs lists the
    (parameter, twin) pairs for grads_match."""

    def __init__(self, *holders):
        self._twin, self.pairs = {}, []
        for h in holders:
            ps = ([p for _, p in h.named_parameters()] if isinstance(h, torch.nn.Module) else
                  [v for v in vars(h).values() if isinstance(v, torch.Tensor) and v.requires_grad])
            for p in ps:
                if id(p) not in self._twin:
                    self._twin[id(p)] = p64(p).requires_grad_(True)
                    self.pairs.append((p, self._twin[id(p)]))

    def __call__(self, p):
        return self._twin[id(p)]


def grads_match(gnn, out, ref_out, pairs, tol=2e-5):
    """the same seeded cotangent through both graphs, then the gradient of every (mirror leaf, float64 reference leaf)
    pair compared.  A Julia-shaped mirror leaf (D.., N) meets its reference in rows (N, ..D); a leaf of the
    reference's own shape (a parameter, an edge-weight vector) is compared as it is.  A reference leaf None marks a
    gradient that vanishes identically (a shift the softmax cancels): its norm must stay within tol of the largest
    reference gradient's."""
    g = torch.randn(ref_out.shape, dtype=F64, generator=torch.Generator().manual_seed(7))
    got = torch.autograd.grad((gnn.rows(out).double() * g.to(out.device)).sum(), [m for m, _ in pairs],
                              retain_graph=True)
    want = torch.autograd.grad((ref_out * g).sum(), [r for _, r in pairs if r is not None], retain_graph=True)
    scale = max(float(_c64(b).norm()) for b in want)
    want = iter(want)
    for i, (a, (_, r)) in enumerate(zip(got, pairs)):
        if r is None:
            assert float(_c64(a).norm()) < tol * scale, f"gradient of input {i} should vanish"
            continue
        b = next(want)
        if a.shape != b.shape:
            a = gnn.rows(a)
        assert a.shape == b.shape
        err = rel(a, b)
        assert err < tol, f"gradient of input {i} {tuple(b.shape)}: {err:.2e}"


# ------------------------------------------------------------------------------------------------ pin the fake
def test_fake_abi_agrees_with_the_oracle(gnn, oracle, cpu_abi):
    rng = np.random.default_rng(0)
    n, E, D = 50, 400, 6
    s = rng.integers(1, n + 1, E); t = rng.integers(1, n + 1, E)
    t[t == 7] = 8                                                     # node 7 has no in-edge: neutral elements
    g = gnn.GNNGraph(torch.as_tensor(s), torch.as_tensor(t), num_nodes=n)
    x = rng.standard_normal((n, D)).astype(np.float32)
    w = rng.uniform(0.5, 2, E).astype(np.float32)
    xt = jl(gnn, x, CPU)
    for name, aggr in (("+", operator.add), ("mean", gnn.mean), ("max", max), ("min", min)):
        ref = oracle.propagate_unfused(name, s, t, n, x.astype(np.float64))
        got = gnn.rows(gnn.propagate(gnn.copy_xj, g, aggr, xj=xt)).numpy()
        assert np.array_equal(np.isinf(got), np.isinf(ref))
        fin = np.isfinite(ref)
        assert rel(got[fin], ref[fin]) < 1e-6, name
        m = rng.standard_normal((E, D)).astype(np.float32)
        ref = oracle.scatter(name, m.astype(np.float64), t, n)
        got = gnn.rows(gnn.aggregate_neighbors(g, aggr, jl(gnn, m, CPU))).numpy()
        fin = np.isfinite(ref)
        assert rel(got[fin], ref[fin]) < 1e-6
    ref = oracle.propagate_unfused("+", s, t, n, x.astype(np.float64), w.astype(np.float64))
    got = gnn.rows(gnn.propagate(gnn.e_mul_xj, g, operator.add, xj=xt, e=torch.as_tensor(w)))
    assert rel(got, ref) < 1e-6
    e = rng.standard_normal((E, 3)).astype(np.float32)
    ref = oracle.softmax_edge_neighbors(t, n, e.astype(np.float64))
    assert rel(gnn.rows(gnn.softmax_edge_neighbors(g, jl(gnn, e, CPU))), ref) < 1e-6
    assert np.array_equal(gnn.degree(g, dir="in").numpy(), np.bincount(t - 1, minlength=n).astype(np.float32))
    assert np.array_equal(gnn.degree(g, dir="out").numpy(), np.bincount(s - 1, minlength=n).astype(np.float32))
    s2, t2 = oracle.add_self_loops(s, t, n)
    ref, _ = oracle.gcn_propagate(s2, t2, n, x.astype(np.float64))
    l = NT(weight=torch.eye(D), bias=None, add_self_loops=True, use_edge_weight=False)
    assert rel(gnn.rows(gnn.gcn_conv(l, g, xt)), ref) < 1e-6
    C_, H = 4, 3
    Wx = rng.standard_normal((n, H, C_)); a = rng.standard_normal((H, 2 * C_))
    el, er = (Wx * a[:, :C_]).sum(-1), (Wx * a[:, C_:]).sum(-1)
    ref, _alpha = oracle.gat_aggregate(s2, t2, n, Wx, a, 0.2)
    out = np.empty((n, H, C_), np.float32)
    f32 = lambda a: np.ascontiguousarray(a, dtype=np.float32)
    Wx32, el32, er32 = f32(Wx), f32(el), f32(er)
    h = gnn.add_self_loops(g).plan().h
    assert cpu_abi.gnnb_gat_aggregate(h, Wx32.ctypes.data, el32.ctypes.data, er32.ctypes.data, C_, H, 0.2,
                                      out.ctypes.data, None, None, None, 0) == 0
    assert rel(out, ref) < 1e-6


def test_fake_abi_is_gone_after_the_test(gnn):
    """the fixture must restore the real library (which refuses to compute without a GPU)"""
    import ctypes
    assert isinstance(gnn._lib.lib, ctypes.CDLL) and gnn.graph.lib is gnn._lib.lib and gnn.layers.lib is gnn._lib.lib
    if gnn.device_count() == 0:
        g = gnn.GNNGraph(torch.tensor([1, 2]), torch.tensor([2, 1]))
        with pytest.raises(gnn.GNNBError):
            gnn.propagate(gnn.copy_xj, g, operator.add, xj=gnn.colmajor(torch.ones(2, 2)))


# ------------------------------------------------------------------------------------------------ gcn / sage / gat
def saw(be, name):
    """did the fake see this ABI entry?  (None on the cuda back end: nothing to assert)"""
    return None if be.calls is None else (name in be.calls)


def setp(rng, param):
    """overwrite a parameter (zeros by default) with random values, on whatever device it lives"""
    with torch.no_grad():
        param.copy_(torch.as_tensor(rng.standard_normal(tuple(param.shape)), dtype=torch.float32))


GRAPH_WEIGHTED = ("use_edge_weight", "weighted_norm_fn")      # graph weights (requiring grad) and use_edge_weight


@pytest.mark.parametrize("case", ["plain", "no_loops", "edge_weight", "use_edge_weight", "norm_fn", "weighted_norm_fn",
                                  "wide_to_narrow", "conv_weight"])
def test_gcn_conv_branches(gnn, be, case):
    """every branch of gcn_conv; gradients of x, the NT's weight and bias, and the edge weights the case uses"""
    rng = np.random.default_rng(1)
    dev = be.dev
    g, R, s, t = make_graph(gnn, rng, dev, weights=(case in GRAPH_WEIGHTED))
    Din, Dout = (12, 5) if case == "wide_to_narrow" else (5, 8)
    x = rng.standard_normal((R.n, Din))
    W = rng.standard_normal((Dout, Din)) / 3
    b = rng.standard_normal(Dout)
    l = NT(weight=f32(W, dev).requires_grad_(case != "conv_weight"), bias=f32(b, dev).requires_grad_(True),
           σ=torch.tanh, add_self_loops=case != "no_loops", use_edge_weight=case in GRAPH_WEIGHTED)
    P = Twins(l)
    xt, xr = jl(gnn, x, dev, True), r64(x, True)
    pairs = [(xt, xr)] + P.pairs
    kw, w_ref, Rl = {}, None, (R.with_loops() if l.add_self_loops else R)
    ones = torch.ones(R.n if l.add_self_loops else 0, dtype=F64)
    if case == "edge_weight":
        ew = rng.uniform(0.5, 1.5, len(s))
        kw["edge_weight"] = f32(ew, dev).requires_grad_(True)
        pairs.append((kw["edge_weight"], r64(ew, True)))
        w_ref = torch.cat([pairs[-1][1], ones])
    if case in GRAPH_WEIGHTED:                            # GNNGraph keeps the weight tensor it is given
        g.w.requires_grad_(True)
        pairs.append((g.w, p64(g.w).requires_grad_(True)))
        w_ref = torch.cat([pairs[-1][1], ones])
    Wr = P(l.weight) if case != "conv_weight" else None
    if case == "conv_weight":
        W2 = rng.standard_normal((Dout, Din)) / 3
        kw["conv_weight"] = f32(W2, dev).requires_grad_(True)
        Wr = r64(W2, True)
        pairs.append((kw["conv_weight"], Wr))
    if case in ("norm_fn", "weighted_norm_fn"):           # a custom norm on the (weighted) in-degree
        kw["norm_fn"] = lambda d: 1.0 / (1.0 + d)
        c = 1.0 / (1.0 + Rl.indeg(w_ref))
        agg = Rl.propagate(xr * c[:, None], w=w_ref) * c[:, None]
    else:
        agg = Rl.gcn(xr, w_ref)
    ref = torch.tanh(agg @ Wr.t() + P(l.bias))
    out = gnn.gcn_conv(l, g, xt, **kw)
    assert out.shape == (Dout, R.n)
    assert rel(gnn.rows(out), ref) < 2e-6 * be.tol
    n_fwd = None if be.calls is None else len(be.calls)
    grads_match(gnn, out, ref, pairs, 2e-5 * be.tol)
    if be.calls is not None:
        fwd, bwd = be.calls[:n_fwd], be.calls[n_fwd:]
        assert saw(be, "gnnb_gcn_propagate") == (case in ("plain", "no_loops", "wide_to_narrow", "conv_weight"))
        assert "gnnb_gather" not in fwd and not saw(be, "gnnb_scatter")              # never the (D,E) intermediate
        # the only gather is the weighted degree's pullback, one (1, E) row per weighted call
        assert bwd.count("gnnb_gather") == (1 if case in ("edge_weight",) + GRAPH_WEIGHTED else 0)


def test_gcn_conv_argument_errors(gnn, be):
    rng = np.random.default_rng(2)
    dev = be.dev
    g, R, s, t = make_graph(gnn, rng, dev)
    l = NT(weight=torch.zeros(4, 3, device=dev), bias=None, add_self_loops=True, use_edge_weight=False)
    x = jl(gnn, rng.standard_normal((R.n, 3)), dev)
    with pytest.raises(ValueError, match="Wrong number of edge weights"):         # conv.jl:3-10 ArgumentError
        gnn.gcn_conv(l, g, x, torch.ones(3, device=dev))
    with pytest.raises(ValueError, match="wrong size"):                           # conv.jl:22
        gnn.gcn_conv(l, g, x, conv_weight=torch.zeros(3, 3, device=dev))
    with pytest.raises(AssertionError):                                           # check_num_nodes
        gnn.gcn_conv(l, g, jl(gnn, rng.standard_normal((R.n + 1, 3)), dev))


@pytest.mark.parametrize("aggr", ["mean", "+"])
def test_sage_graph_gin_layers(gnn, be, aggr):
    rng = np.random.default_rng(3)
    dev = be.dev
    g, R, s, t = make_graph(gnn, rng, dev)
    Din, Dout = 6, 4
    x = rng.standard_normal((R.n, Din))
    op = gnn.mean if aggr == "mean" else operator.add
    xt, xr = jl(gnn, x, dev, True), r64(x, True)
    m = R.propagate(xr, aggr)
    # SAGEConv: σ(W [x_i ; aggr_j x_j] + b)
    layer = gnn.SAGEConv(Din, Dout, torch.relu, aggr=op, device=dev)
    setp(rng, layer.bias)
    P = Twins(layer)
    out = layer(g, xt)
    ref = torch.relu(torch.cat([xr, m], dim=1) @ P(layer.weight).t() + P(layer.bias))
    assert rel(gnn.rows(out), ref) < 2e-6 * be.tol
    grads_match(gnn, out, ref, [(xt, xr)] + P.pairs, 2e-5 * be.tol)
    # GraphConv: σ(W1 x_i + W2 aggr_j x_j + b)
    layer = gnn.GraphConv(Din, Dout, torch.tanh, aggr=op, device=dev)
    setp(rng, layer.bias)
    P = Twins(layer)
    out = layer(g, xt)
    ref = torch.tanh(xr @ P(layer.weight1).t() + m @ P(layer.weight2).t() + P(layer.bias))
    assert rel(gnn.rows(out), ref) < 2e-6 * be.tol
    grads_match(gnn, out, ref, [(xt, xr)] + P.pairs, 2e-5 * be.tol)
    # GINConv: nn((1 + ϵ) x_i + aggr_j x_j)
    layer = gnn.GINConv(lambda v: v ** 2, 0.3, aggr=op)
    assert not list(layer.parameters())
    out = layer(g, xt)
    ref = (1.3 * xr + m) ** 2
    assert rel(gnn.rows(out), ref) < 2e-6 * be.tol
    grads_match(gnn, out, ref, [(xt, xr)], 2e-5 * be.tol)
    if be.calls is not None:
        assert set(be.calls) <= {"gnnb_graph_create", "gnnb_propagate", "gnnb_propagate_bwd"}


def _gat_reference(R, xr, Wd, a, C_, H, slope, concat, bias):
    Wx = (xr @ Wd.t()).reshape(R.n, H, C_)
    ai, aj = a[:C_].t(), a[C_:].t()                                    # (H, C): rows 1..C pair with the target
    logit = (Wx[R.t] * ai).sum(-1) + (Wx[R.s] * aj).sum(-1)            # (E, H)
    alpha = R.softmax(torch.nn.functional.leaky_relu(logit, slope))
    out = R.scatter_sum(alpha[:, :, None] * Wx[R.s])                   # (N, H, C)
    out = out.reshape(R.n, H * C_) if concat else out.mean(dim=1)
    return out + bias


@pytest.mark.parametrize("heads,concat,fused", [(1, True, True), (3, True, True), (3, False, True), (2, True, False),
                                                (2, False, False)])
def test_gat_conv_fused_and_composed(gnn, be, heads, concat, fused):
    rng = np.random.default_rng(4)
    dev = be.dev
    g, R, s, t = make_graph(gnn, rng, dev)
    Din, C_ = 5, 4
    layer = gnn.GATConv(Din, C_, heads=heads, concat=concat, device=dev)
    setp(rng, layer.bias)
    P = Twins(layer)
    x = rng.standard_normal((R.n, Din))
    xt, xr = jl(gnn, x, dev, True), r64(x, True)
    out = layer(g, xt, fused=fused)
    Rl = R.with_loops()
    ref = _gat_reference(Rl, xr, P(layer.dense_x.weight), P(layer.a), C_, heads, 0.2, concat, P(layer.bias))
    assert out.shape == ((C_ * heads if concat else C_), R.n)
    assert rel(gnn.rows(out), ref) < 3e-6 * be.tol
    # x and every parameter (W, a, bias) through the fused pullback against autograd of the formula
    assert {id(m) for m, _ in P.pairs} == {id(layer.a), id(layer.dense_x.weight), id(layer.bias)}
    grads_match(gnn, out, ref, [(xt, xr)] + P.pairs, 2e-5 * be.tol)
    if be.calls is not None:
        assert saw(be, "gnnb_gat_aggregate") == fused
        assert saw(be, "gnnb_gather") == (not fused)


def test_gat_conv_edge_features_and_asserts(gnn, be):
    rng = np.random.default_rng(5)
    dev = be.dev
    g, R, s, t = make_graph(gnn, rng, dev)
    Din, De, C_, H = 5, 3, 4, 2
    layer = gnn.GATConv(Din, C_, heads=H, add_self_loops=False, device=dev)
    x = jl(gnn, rng.standard_normal((R.n, Din)), dev)
    e = jl(gnn, rng.standard_normal((len(s), De)), dev)
    with pytest.raises(AssertionError, match="not specified in the layer constructor"):
        layer(g, x, e)
    layer.dense_e = gnn.layers._Dense(De, C_ * H, bias=False, device=dev)
    layer.a = torch.nn.Parameter(gnn.layers.glorot_uniform(3 * C_, H, device=dev))
    with pytest.raises(AssertionError, match="Input edge features required"):
        layer(g, x)
    out = layer(g, x, e)
    xr, er = p64(gnn.rows(x)), p64(gnn.rows(e))
    Wx = (xr @ p64(layer.dense_x.weight).t()).reshape(R.n, H, C_)
    We = (er @ p64(layer.dense_e.weight).t()).reshape(len(s), H, C_)
    a = p64(layer.a)
    logit = ((Wx[R.t] * a[:C_].t()).sum(-1) + (Wx[R.s] * a[C_:2 * C_].t()).sum(-1) + (We * a[2 * C_:].t()).sum(-1))
    alpha = R.softmax(torch.nn.functional.leaky_relu(logit, 0.2))
    ref = R.scatter_sum(alpha[:, :, None] * Wx[R.s]).reshape(R.n, H * C_) + p64(layer.bias)
    assert rel(gnn.rows(out), ref) < 3e-6 * be.tol
    layer.add_self_loops = True
    with pytest.raises(AssertionError, match="not yet supported"):
        layer(g, x, e)


# ------------------------------------------------------------------------------------------------ §8f rank-1 layers
@pytest.mark.parametrize("weighted", [False, True])
def test_sg_and_tag_conv(gnn, be, weighted):
    rng = np.random.default_rng(6)
    dev = be.dev
    g, R, s, t = make_graph(gnn, rng, dev)
    Din, Dout, k = 7, 4, 3
    x = rng.standard_normal((R.n, Din))
    xt, xr = jl(gnn, x, dev, True), r64(x, True)
    ew = f32(rng.uniform(0.5, 1.5, len(s)), dev).requires_grad_(True) if weighted else None
    ew64 = p64(ew).requires_grad_(True) if weighted else None
    Rl = R.with_loops()
    w_ref = torch.cat([ew64, torch.ones(R.n, dtype=F64)]) if weighted else None
    hops = [xr]
    for _ in range(k):
        hops.append(Rl.gcn(hops[-1], w_ref))
    for cls, fn in ((gnn.SGConv, gnn.sg_conv), (gnn.TAGConv, gnn.tag_conv)):
        layer = cls(Din, Dout, k, device=dev)
        setp(rng, layer.bias)
        P = Twins(layer)
        W, b = P(layer.weight), P(layer.bias)
        out = layer(g, xt, ew)
        if cls is gnn.SGConv:
            ref = hops[k] @ W.t() + b                                     # W Â^k x + b
        else:                                                             # Σ_i W Σ_{j<=i} Â^j x + b   (conv.jl:670-682)
            run, ref = torch.zeros_like(hops[1]), 0
            for i in range(1, k + 1):
                run = run + hops[i]
                ref = ref + run @ W.t()
            ref = ref + b
        assert out.shape == (Dout, R.n)
        assert rel(gnn.rows(out), ref) < 3e-6 * be.tol
        grads_match(gnn, out, ref, [(xt, xr)] + P.pairs + ([(ew, ew64)] if weighted else []), 2e-5 * be.tol)
        assert rel(gnn.rows(fn(layer, g, xt, ew)), ref) < 3e-6 * be.tol
    if not weighted:   # sgc_conv (conv.jl:407-448) is the same function under its older name
        assert rel(gnn.sgc_conv(layer, g, xt), gnn.sg_conv(layer, g, xt)) < 1e-6
        if be.calls is not None:
            assert be.calls.count("gnnb_gcn_propagate") >= 3 * k and not saw(be, "gnnb_propagate")
    with pytest.raises(AssertionError, match="Wrong number of edge weights"):
        gnn.tag_conv(layer, g, xt, torch.ones(3, device=dev))


def test_gated_graph_conv(gnn, be):
    rng = np.random.default_rng(7)
    dev = be.dev
    g, R, s, t = make_graph(gnn, rng, dev)
    dims, L, Din = 6, 3, 4
    layer = gnn.GatedGraphConv(dims, L, aggr=gnn.mean, device=dev)
    setp(rng, layer.gru.b)
    P = Twins(layer)
    x = rng.standard_normal((R.n, Din))
    xt, xr = jl(gnn, x, dev, True), r64(x, True)
    out = layer(g, xt)
    Wi, Wh, b, Wl = (P(p) for p in (layer.gru.Wi, layer.gru.Wh, layer.gru.b, layer.weight))
    h = torch.cat([xr, torch.zeros(R.n, dims - Din, dtype=F64)], dim=1)
    for i in range(L):
        m = R.propagate(h @ Wl[:, :, i].t(), "mean")
        gx, gh = m @ Wi.t(), h @ Wh.t()
        r = torch.sigmoid(gx[:, :dims] + gh[:, :dims] + b[:dims])
        z = torch.sigmoid(gx[:, dims:2 * dims] + gh[:, dims:2 * dims] + b[dims:2 * dims])
        hc = torch.tanh(gx[:, 2 * dims:] + r * gh[:, 2 * dims:] + b[2 * dims:])
        h = (1 - z) * hc + z * h
    assert out.shape == (dims, R.n)
    assert rel(gnn.rows(out), h) < 3e-6 * be.tol
    grads_match(gnn, out, h, [(xt, xr)] + P.pairs, 2e-5 * be.tol)
    with pytest.raises(AssertionError, match="less or equal"):
        layer(g, jl(gnn, rng.standard_normal((R.n, dims + 1)), dev))


@pytest.mark.parametrize("heads,concat,ein", [(1, True, 0), (3, True, 0), (3, False, 0), (2, True, 3)])
def test_gatv2_conv(gnn, be, heads, concat, ein):
    rng = np.random.default_rng(8)
    dev = be.dev
    g, R, s, t = make_graph(gnn, rng, dev)
    Din, C_ = 5, 4
    layer = gnn.GATv2Conv((Din, ein) if ein else Din, C_, torch.tanh, heads=heads, concat=concat,
                          add_self_loops=(ein == 0), device=dev)
    setp(rng, layer.bias)
    setp(rng, layer.dense_i.bias)
    P = Twins(layer)
    x = rng.standard_normal((R.n, Din))
    xt, xr = jl(gnn, x, dev, True), r64(x, True)
    pairs = [(xt, xr)] + P.pairs
    if ein:
        ea = rng.standard_normal((len(s), ein))
        e, er = jl(gnn, ea, dev, True), r64(ea, True)
        pairs.append((e, er))
    else:
        e = None
    out = layer(g, xt, e)
    Rl = R if ein else R.with_loops()
    Wi = (xr @ P(layer.dense_i.weight).t() + P(layer.dense_i.bias)).reshape(R.n, heads, C_)
    Wj = (xr @ P(layer.dense_j.weight).t()).reshape(R.n, heads, C_)
    z = Wi[Rl.t] + Wj[Rl.s]
    if ein:
        z = z + (er @ P(layer.dense_e.weight).t()).reshape(-1, heads, C_)
    logit = (torch.nn.functional.leaky_relu(z, 0.2) * P(layer.a).t()).sum(-1)       # (E, H)
    alpha = Rl.softmax(logit)
    o = Rl.scatter_sum(alpha[:, :, None] * Wj[Rl.s])
    o = o.reshape(R.n, heads * C_) if concat else o.mean(dim=1)
    ref = torch.tanh(o + P(layer.bias))
    assert out.shape == ((C_ * heads if concat else C_), R.n)
    assert rel(gnn.rows(out), ref) < 3e-6 * be.tol
    grads_match(gnn, out, ref, pairs, 2e-5 * be.tol)
    if not ein:
        with pytest.raises(AssertionError, match="not specified in the layer constructor"):
            layer(g, xt, jl(gnn, rng.standard_normal((len(s), 2)), dev))


@pytest.mark.parametrize("cfg", [dict(), dict(heads=3), dict(heads=3, concat=False), dict(heads=2, gating=True),
                                 dict(heads=2, root_weight=False, add_self_loops=True),
                                 dict(heads=2, ein=3, skip_connection=True, ff_channels=10),
                                 dict(heads=2, batch_norm=True, ff_channels=6)])
def test_transformer_conv(gnn, be, cfg):
    rng = np.random.default_rng(9)
    dev = be.dev
    cfg = dict(cfg)
    ein = cfg.pop("ein", 0)
    heads, concat = cfg.get("heads", 1), cfg.get("concat", True)
    g, R, s, t = make_graph(gnn, rng, dev)
    C_ = 4
    Din = C_ * heads if cfg.get("skip_connection") else 5
    layer = gnn.TransformerConv((Din, ein) if ein else Din, C_, device=dev, **cfg)
    for d in (layer.W1, layer.W2, layer.W3, layer.W4, layer.W6):
        if d is not None and d.bias is not None:
            setp(rng, d.bias)
    P = Twins(layer)
    x = rng.standard_normal((R.n, Din))
    xt, xr = jl(gnn, x, dev, True), r64(x, True)
    # gradients that vanish identically: the key bias adds q_i·b to every logit of row i, which the softmax cancels;
    # a batch norm removes per-channel constants ahead of it (root and value biases before BN1 — every node has an
    # in-edge and the α of a row sum to 1 — and the last feed-forward bias before BN2)
    vanish = [layer.W4.bias]
    if layer.BN1 is not None:
        vanish += [layer.W1.bias, layer.W2.bias]
    if layer.BN2 is not None:
        vanish += [layer.FF[1].bias]
    vanish = {id(p) for p in vanish if p is not None}
    pairs = [(xt, xr)] + [(m, None if id(m) in vanish else r) for m, r in P.pairs]
    if ein:
        ea = rng.standard_normal((len(s), ein))
        e, er = jl(gnn, ea, dev, True), r64(ea, True)
        pairs.append((e, er))
    else:
        e = None
    out = layer(g, xt, e)
    Rl = R.with_loops() if cfg.get("add_self_loops") else R

    def dense(d, v):
        y = v @ P(d.weight).t()
        return y if d.bias is None else y + P(d.bias)

    q = dense(layer.W3, xr).reshape(R.n, heads, C_)
    k = dense(layer.W4, xr).reshape(R.n, heads, C_)
    v = dense(layer.W2, xr).reshape(R.n, heads, C_)
    ke, ve = k[Rl.s], v[Rl.s]
    if ein:
        ee = dense(layer.W6, er).reshape(-1, heads, C_)
        ke, ve = ke + ee, ve + ee
    alpha = Rl.softmax((q[Rl.t] * ke).sum(-1) / np.sqrt(C_))                 # (E, H)
    h = Rl.scatter_sum(alpha[:, :, None] * ve)
    h = h.reshape(R.n, heads * C_) if concat else h.mean(dim=1)
    if layer.W1 is not None:
        r = dense(layer.W1, xr)
        if layer.W5 is not None:
            beta = torch.sigmoid(torch.cat([h, r, h - r], dim=1) @ P(layer.W5.weight).t())
            h = beta * r + (1 - beta) * h
        else:
            h = h + r
    if cfg.get("skip_connection"):
        h = h + xr

    def bn(B, v):   # training-mode batch norm over nodes (γ = 1, β = 0 as initialised, but differentiated)
        return (v - v.mean(0)) / torch.sqrt(v.var(0, unbiased=False) + 1e-5) * P(B.bn.weight) + P(B.bn.bias)

    if layer.BN1 is not None:
        h = bn(layer.BN1, h)
    if layer.FF is not None:
        h1 = h
        h = dense(layer.FF[1], torch.relu(dense(layer.FF[0], h)))
        if cfg.get("skip_connection"):
            h = h + h1
        if layer.BN2 is not None:
            h = bn(layer.BN2, h)
    assert out.shape == ((C_ * heads if concat else C_), R.n)
    assert rel(gnn.rows(out), h) < 5e-6 * be.tol
    grads_match(gnn, out, h, pairs, tol=5e-5 * be.tol)


def test_agnn_conv(gnn, be):
    rng = np.random.default_rng(10)
    dev = be.dev
    g, R, s, t = make_graph(gnn, rng, dev)
    x = rng.standard_normal((R.n, 6))
    xt, xr = jl(gnn, x, dev, True), r64(x, True)
    layer = gnn.AGNNConv(init_beta=1.7, device=dev)
    P = Twins(layer)
    out = layer(g, xt)
    Rl = R.with_loops()
    xn = xr / xr.norm(dim=1, keepdim=True)
    alpha = Rl.softmax(P(layer.beta) * (xn[Rl.t] * xn[Rl.s]).sum(-1, keepdim=True))
    ref = Rl.scatter_sum(alpha * xr[Rl.s])
    assert rel(gnn.rows(out), ref) < 3e-6 * be.tol
    grads_match(gnn, out, ref, [(xt, xr)] + P.pairs, 2e-5 * be.tol)
    (gb,) = torch.autograd.grad(out.sum(), layer.beta)
    assert torch.isfinite(gb).all()


# ------------------------------------------------------------------------------------------------ generic path, readout
@pytest.mark.parametrize("sig", ["relu", "identity"])
def test_sage_conv_split_weight_path(gnn, be, sig):
    """SAGEConv 128 -> 128 on a CUDA device takes gnnb_linear2 (the CPU test double keeps the vcat formula): the two column blocks of W meet x_i and the aggregated neighbours in two
    accumulating wgmma passes instead of a (2·in, N) vcat + one GEMM (conv.jl:281); output, dx, dW, db against float64."""
    rng = np.random.default_rng(11)
    dev = be.dev
    g, R, s, t = make_graph(gnn, rng, dev)
    D = 128
    x = rng.standard_normal((R.n, D))
    xt, xr = jl(gnn, x, dev, True), r64(x, True)
    m = R.propagate(xr, "mean")
    act = torch.relu if sig == "relu" else gnn.layers.identity
    layer = gnn.SAGEConv(D, D, act, device=dev)
    setp(rng, layer.bias)
    out = layer(g, xt)
    W64, b64 = p64(layer.weight).requires_grad_(True), p64(layer.bias).requires_grad_(True)
    pre = torch.cat([xr, m], dim=1) @ W64.t() + b64
    ref = torch.relu(pre) if sig == "relu" else pre
    assert rel(gnn.rows(out), ref) < 2e-6 * be.tol
    cot = torch.randn(ref.shape, dtype=torch.float64, generator=torch.Generator().manual_seed(5))
    if sig == "relu":                                        # keep away from the kink: relu' is discontinuous at 0
        cot = cot * (pre.detach().abs() > 1e-4)
    gx, gW, gb = torch.autograd.grad((gnn.rows(out).double() * cot.to(out.device)).sum(), [xt, layer.weight, layer.bias])
    rx, rW, rb = torch.autograd.grad((ref * cot).sum(), [xr, W64, b64])
    assert rel(gnn.rows(gx), rx) < 2e-5 * be.tol and rel(gW, rW) < 2e-5 * be.tol and rel(gb, rb) < 2e-5 * be.tol


def test_generic_messages_with_structures(gnn, be):
    """apply_edges / aggregate_neighbors over dict, tuple and None containers (GNNGraphs/src/gatherscatter.jl:1-18)"""
    rng = np.random.default_rng(11)
    dev = be.dev
    g, R, s, t = make_graph(gnn, rng, dev)
    x = rng.standard_normal((R.n, 3)); y = rng.standard_normal((R.n, 2, 2)); e = rng.standard_normal((len(s), 3))
    xt, yt, et = jl(gnn, x, dev), jl(gnn, y, dev), jl(gnn, e, dev)

    def f(xi, xj, ed):
        assert xi["a"].shape == (3, len(s)) and xj["b"].shape == (2, 2, len(s)) and xj["c"] is None
        return {"u": xi["a"] * ed - xj["a"], "v": (xj["b"], xi["b"])}

    m = gnn.apply_edges(f, g, xi={"a": xt, "b": yt}, xj={"a": xt, "b": yt, "c": None}, e=et)
    assert rel(gnn.rows(m["u"]), r64(x)[R.t] * r64(e) - r64(x)[R.s]) < 1e-6
    out = gnn.aggregate_neighbors(g, operator.add, m)
    assert rel(gnn.rows(out["u"]), R.scatter_sum(r64(x)[R.t] * r64(e) - r64(x)[R.s])) < 1e-6 * be.tol
    assert rel(gnn.rows(out["v"][0]), R.scatter_sum(r64(y)[R.s])) < 1e-6 * be.tol
    assert rel(gnn.rows(out["v"][1]), R.scatter_sum(r64(y)[R.t])) < 1e-6 * be.tol
    with pytest.raises(AssertionError):
        gnn.apply_edges(f, g, xi={"a": xt[:, :-1]}, xj={"a": xt}, e=et)
    with pytest.raises(AssertionError):
        gnn.aggregate_neighbors(g, operator.add, et[:, :-1])
    with pytest.raises(ValueError, match="unsupported aggregation"):
        gnn.propagate(gnn.copy_xj, g, "prod", xj=xt)
    with pytest.raises(TypeError, match="float32"):
        gnn.propagate(gnn.copy_xj, g, operator.add, xj=xt.double())


def test_readout_on_batched_graphs(gnn, be):
    rng = np.random.default_rng(12)
    dev = be.dev
    gs = []
    for _ in range(4):
        n, E = int(rng.integers(5, 12)), int(rng.integers(10, 30))
        gs.append(gnn.GNNGraph(torch.as_tensor(rng.integers(1, n + 1, E)), torch.as_tensor(rng.integers(1, n + 1, E)),
                               num_nodes=n, ndata={"x": jl(gnn, rng.standard_normal((n, 3)), CPU)},
                               edata={"e": jl(gnn, rng.standard_normal((E, 2)), CPU)}))
    g = gnn.batch(gs).to(dev)
    x, e = g.ndata["x"], g.edata["e"]
    for aggr, fn in ((operator.add, torch.sum), (gnn.mean, torch.mean), (max, torch.amax), (min, torch.amin)):
        r = gnn.reduce_nodes(aggr, g, x).cpu()
        q = gnn.reduce_edges(aggr, g, e).cpu()
        for i, gi in enumerate(gs):
            assert torch.allclose(r[:, i], fn(gi.ndata["x"], dim=1), rtol=1e-5, atol=1e-6)
            assert torch.allclose(q[:, i], fn(gi.edata["e"], dim=1), rtol=1e-5, atol=1e-6)
    sm, se = gnn.softmax_nodes(g, x).cpu(), gnn.softmax_edges(g, e).cpu()
    no = eo = 0
    for gi in gs:
        assert torch.allclose(sm[:, no:no + gi.num_nodes], torch.softmax(gi.ndata["x"], dim=1), rtol=1e-5, atol=1e-7)
        assert torch.allclose(se[:, eo:eo + gi.num_edges], torch.softmax(gi.edata["e"], dim=1), rtol=1e-5, atol=1e-6)
        no, eo = no + gi.num_nodes, eo + gi.num_edges
    z = jl(gnn, rng.standard_normal((4, 5)), dev)
    bn = gnn.broadcast_nodes(g, z)
    assert torch.equal(bn[:, 0], z[:, 0]) and torch.equal(bn[:, -1], z[:, 3]) and bn.shape == (5, g.num_nodes)
    assert gnn.broadcast_edges(g, z).shape == (5, g.num_edges)
    xg = x.clone().requires_grad_(True)
    gnn.reduce_nodes(gnn.mean, g, gnn.softmax_nodes(g, xg) * xg).sum().backward()
    ref = x.detach().cpu().double().requires_grad_(True)
    tot, no = 0, 0
    for gi in gs:
        blk = ref[:, no:no + gi.num_nodes]
        tot = tot + (torch.softmax(blk, dim=1) * blk).mean(dim=1).sum()
        no += gi.num_nodes
    tot.backward()
    assert rel(xg.grad, ref.grad) < 2e-5 * be.tol
