"""Model composition (graphneuralnetworks.jl_b200/basic.py; GraphNeuralNetworks/src/layers/basic.jl) and the graph copy
with replaced data (GNNGraphs/src/gnngraph.jl:187-210, query.jl:516-544).

The reference's basic.jl tests, transcribed, on the `be` back ends (tests/fake_abi.py's double, and the CUDA kernels
under -m gpu).  A chain must compute exactly what its layers applied by hand compute: outputs and gradients are compared
with torch.equal.
"""
import operator

import numpy as np
import pytest
import torch


class LayerNorm(torch.nn.Module):
    """Flux.LayerNorm(d) on features-first arrays: normalise over the first dimension, then scale and shift"""

    def __init__(self, d, device=None):
        super().__init__()
        self.scale = torch.nn.Parameter(1 + 0.1 * torch.randn(d, device=device))
        self.shift = torch.nn.Parameter(0.1 * torch.randn(d, device=device))

    def forward(self, x):
        mu = x.mean(0, keepdim=True)
        var = ((x - mu) ** 2).mean(0, keepdim=True)
        shape = (-1,) + (1,) * (x.dim() - 1)
        return (x - mu) / torch.sqrt(var + 1e-5) * self.scale.view(shape) + self.shift.view(shape)


class BatchNorm(torch.nn.Module):
    """Flux.BatchNorm(d) on (d, N): batch statistics in training mode, running ones otherwise"""

    def __init__(self, d, device=None):
        super().__init__()
        self.bn = torch.nn.BatchNorm1d(d, device=device)

    def forward(self, x):
        return self.bn(x.t()).t()


class Dense(torch.nn.Module):
    """Flux.Dense(in, out, σ) on features-first arrays of any rank"""

    def __init__(self, din, dout, sigma=None, device=None):
        super().__init__()
        self.weight = torch.nn.Parameter(torch.randn(dout, din, device=device) / din ** 0.5)
        self.bias = torch.nn.Parameter(0.1 * torch.randn(dout, device=device))
        self.sigma = sigma

    def forward(self, x):
        y = torch.tensordot(self.weight, x, dims=([1], [0])) + self.bias.view((-1,) + (1,) * (x.dim() - 1))
        return y if self.sigma is None else self.sigma(y)


def regular_graph(gnn, n, dev, **kw):
    """a 4-regular graph on n nodes (i ~ i ± 1, i ± 2 mod n), both directions"""
    i = np.arange(n)
    s = np.concatenate([i, i, i, i]) + 1
    t = np.concatenate([(i + 1) % n, (i - 1) % n, (i + 2) % n, (i - 2) % n]) + 1
    return gnn.GNNGraph(torch.as_tensor(s, device=dev), torch.as_tensor(t, device=dev), num_nodes=n, **kw)


def by_hand(layers, g, x):
    """basic.jl's _applylayer spelled out: l(g, x) for a GNNLayer, l(x) otherwise"""
    for l in layers:
        x = l(g, x) if hasattr(l, "graph_forward") else l(x)
    return x


def same_grads(model, f_chain, f_hand, x):
    """f_chain() and f_hand() equal, and so are the gradients of x and of every parameter"""
    ps = [x] + list(model.parameters())
    y1 = f_chain()
    cot = torch.randn(y1.shape, generator=torch.Generator().manual_seed(7)).to(y1.device)
    g1 = torch.autograd.grad((y1 * cot).sum(), ps)
    y2 = f_hand()
    g2 = torch.autograd.grad((y2 * cot).sum(), ps)
    assert torch.equal(y1, y2)
    assert all(torch.equal(a, b) for a, b in zip(g1, g2))


N, DIN, D, DOUT = 10, 3, 4, 2


@pytest.fixture
def setup(gnn, be):
    torch.manual_seed(0)
    g = regular_graph(gnn, N, be.dev, ndata=torch.randn(DIN, N, device=be.dev))
    return SimpleSetup(gnn, be.dev, g)


class SimpleSetup:
    def __init__(self, gnn, dev, g):
        self.gnn, self.dev, self.g = gnn, dev, g

    def chain(self):
        gnn, dev = self.gnn, self.dev
        return gnn.GNNChain(gnn.GCNConv(DIN, D, device=dev), LayerNorm(D, device=dev), lambda v: torch.tanh(v),
                            gnn.GraphConv(D, D, torch.tanh, device=dev), torch.nn.Dropout(0.5),
                            Dense(D, DOUT, device=dev))


# ---------------------------------------------------------------------------------------------- basic.jl's tests
def test_chain_equals_layers_by_hand(setup):
    """basic.jl:6-22: GCNConv, LayerNorm, tanh, GraphConv, Dropout, Dense in test mode"""
    m = setup.chain()
    m.eval()
    x = setup.g.x.clone().requires_grad_(True)
    same_grads(m, lambda: m(setup.g, x), lambda: by_hand(list(m), setup.g, x), x)
    assert m(setup.g, x).shape == (DOUT, N)


def test_constructor_with_names(setup, gnn):
    """basic.jl:24-34"""
    m = gnn.GNNChain(gnn.GCNConv(DIN, D, device=setup.dev), LayerNorm(D, device=setup.dev), torch.tanh,
                     Dense(D, DOUT, device=setup.dev))
    m2 = gnn.GNNChain(enc=m, dec=gnn.DotDecoder())
    assert m2["enc"] is m and m2[0] is m
    g, x = setup.g, setup.g.x
    assert torch.equal(m2(g, x), m2["dec"](g, m2["enc"](g, x)))
    assert m2.keys() == ["enc", "dec"]
    sub = m2[[1]]
    assert isinstance(sub, gnn.GNNChain) and sub.keys() == ["dec"]


def test_constructor_with_vector(setup, gnn):
    """basic.jl:36-43"""
    m = gnn.GNNChain(gnn.GCNConv(DIN, D, device=setup.dev), LayerNorm(D, device=setup.dev), torch.tanh,
                     Dense(D, DOUT, device=setup.dev))
    m2 = gnn.GNNChain(list(m.layers))
    assert isinstance(m2.layers, list)
    assert torch.equal(m2(setup.g, setup.g.x), m(setup.g, setup.g.x))


def test_parallel_residual(setup, gnn):
    """basic.jl:45-57: Parallel(+, identity, GraphConv) inside a chain gets the graph for its GNNLayer branch; train
    mode (BatchNorm on batch statistics)"""
    dev = setup.dev
    res = gnn.GraphConv(D, D, torch.tanh, device=dev)
    m = gnn.GNNChain(gnn.GraphConv(DIN, D, torch.tanh, device=dev), LayerNorm(D, device=dev),
                     gnn.Parallel(operator.add, gnn.identity, res), BatchNorm(D, device=dev), Dense(D, DOUT, device=dev))
    m.train()
    l0, ln, _, bn, dense = list(m)
    x = setup.g.x.clone().requires_grad_(True)

    def hand():
        h = ln(l0(setup.g, x))
        return dense(bn(h + res(setup.g, h)))
    same_grads(m, lambda: m(setup.g, x), hand, x)
    assert res in list(m.modules())


def test_only_graph_input(gnn, be):
    """basic.jl:60-71: NNConv's graph-only call passes the edge features, as a chain's"""
    nin, nout = 2, 4
    torch.manual_seed(1)
    ndata, edata = torch.rand(nin, 3, device=be.dev), torch.rand(nin, 3, device=be.dev)
    g = gnn.GNNGraph([1, 1, 2], [2, 3, 3], ndata=ndata, edata=edata, device=be.dev)
    m = gnn.NNConv(nin, nout, Dense(2, nin * nout, torch.tanh, device=be.dev), device=be.dev)
    chain = gnn.GNNChain(m)
    y = m(g, g.ndata["x"], g.edata["e"])
    assert torch.equal(m(g).ndata["x"], y)
    assert torch.equal(chain(g).ndata["x"], y)
    assert torch.equal(chain(g).edata["e"], edata)


def test_with_graph(gnn, be):
    """basic.jl:74-94"""
    torch.manual_seed(2)
    x = torch.rand(2, 3, device=be.dev)
    g = gnn.GNNGraph([1, 2, 3], [2, 3, 1], ndata=x, device=be.dev)
    model = gnn.SAGEConv(2, 3, device=be.dev)
    wg = gnn.WithGraph(model, g)
    assert torch.equal(wg(x), model(g, x))
    assert [p for p in wg.parameters()] == [p for p in model.parameters()]
    g2 = gnn.GNNGraph([1, 1, 2, 3], [2, 4, 1, 1], device=be.dev)
    x2 = torch.rand(2, 4, device=be.dev)
    assert torch.equal(wg(g2, x2), model(g2, x2))
    assert len(list(gnn.WithGraph(model, g, traingraph=False).parameters())) == len(list(model.parameters()))
    g.ndata["x"].requires_grad_(True)
    wg = gnn.WithGraph(model, g, traingraph=True)
    assert len(list(wg.parameters())) == len(list(model.parameters())) + 1
    assert any(p is g.ndata["x"] for p in wg.parameters())
    assert "g.ndata.x" in dict(wg.named_parameters())


# ---------------------------------------------------------------------------------------------- the chain's interface
def test_chain_graph_call_equals_layers_by_hand(setup, gnn):
    """chain(g): l(g) on a GNNLayer, GNNGraph(g, ndata=l(node_features(g))) otherwise"""
    m = setup.chain()
    m.eval()
    h = m(setup.g)
    assert isinstance(h, gnn.GNNGraph) and h is not setup.g
    assert torch.equal(h.ndata["x"], m(setup.g, setup.g.x))
    assert h.num_nodes == N and torch.equal(h.s, setup.g.s)


def test_indexing_and_iteration(gnn, be):
    a, b, c = gnn.GraphConv(2, 3, device=be.dev), torch.nn.Tanh(), gnn.GraphConv(3, 1, device=be.dev)
    m = gnn.GNNChain(a, b, c)
    assert len(m) == 3 and list(m) == [a, b, c] and m[0] is a and m[-1] is c
    assert isinstance(m[1:], gnn.GNNChain) and list(m[1:]) == [b, c]
    assert list(m[[2, 0]]) == [c, a]
    assert m.keys() == [0, 1, 2]
    named = gnn.GNNChain(enc=a, act=b, dec=c)
    assert list(named[:2]) == [a, b] and named[:2].keys() == ["enc", "act"] and named["dec"] is c
    with pytest.raises(KeyError):
        named["nope"]
    vec = gnn.GNNChain([a, b])
    assert isinstance(vec[:1].layers, list)
    assert "GNNChain(" in repr(named) and "enc = " in repr(named)


def test_constructor_errors(gnn):
    with pytest.raises(ValueError):
        gnn.GNNChain(layers=torch.nn.Tanh())
    with pytest.raises(TypeError):
        gnn.GNNChain(torch.nn.Tanh(), act=torch.nn.Tanh())
    assert len(gnn.GNNChain()) == 0


def test_modules_reached_once(gnn):
    """parameters(), train() and eval() reach every Module member once, a repeated one included; lambdas are allowed"""
    a = gnn.GraphConv(2, 3)
    d = torch.nn.Dropout(0.5)
    m = gnn.GNNChain(a, lambda v: v * 2, d, a, gnn.GNNChain(d, gnn.GraphConv(3, 3)))
    params = list(m.parameters())
    assert len(params) == len({id(p) for p in params}) == 6
    m.eval()
    assert not d.training and not m.training
    m.train()
    assert d.training and a.training
    assert isinstance(m, gnn.GNNLayer)


def test_layers_are_gnn_layers(gnn):
    """every class the reference makes a GNNLayer; GlobalAttentionPool too (a deliberate difference: the reference's
    struct has no supertype); DCGRUCell is not one in the reference"""
    names = ["GCNConv", "GATConv", "SAGEConv", "GraphConv", "GINConv", "AGNNConv", "SGConv", "TAGConv", "GatedGraphConv",
             "GATv2Conv", "TransformerConv", "ChebConv", "EdgeConv", "NNConv", "ResGatedGraphConv", "CGConv",
             "MEGNetConv", "GMMConv", "EGNNConv", "DConv", "DotDecoder", "GlobalPool", "GlobalAttentionPool", "Set2Set",
             "GNNRecurrence", "TGCNCell", "GConvGRUCell", "GConvLSTMCell", "EvolveGCNOCell", "GNNChain"]
    for n in names:
        assert issubclass(getattr(gnn, n), gnn.GNNLayer), n
    assert not issubclass(gnn.DCGRUCell, gnn.GNNLayer)
    assert not issubclass(gnn.WithGraph, gnn.GNNLayer) and not issubclass(gnn.Parallel, gnn.GNNLayer)


def test_edge_feature_graph_calls(gnn, be):
    """GATConv and MEGNetConv: the graph-only call passes edge_features(g); MEGNetConv replaces both stores"""
    torch.manual_seed(3)
    g = gnn.GNNGraph([1, 2, 3, 1], [2, 3, 1, 3], ndata=torch.randn(3, 3, device=be.dev), device=be.dev)
    l = gnn.GATConv(3, 4, device=be.dev)
    assert torch.equal(l(g).ndata["x"], l(g, g.x))
    ge = gnn.GNNGraph(g, edata=torch.randn(3, 4, device=be.dev))
    mg = gnn.MEGNetConv(3, 4, device=be.dev)
    x, e = mg(ge, ge.x, ge.e)
    h = mg(ge)
    assert torch.equal(h.x, x) and torch.equal(h.e, e)


# ---------------------------------------------------------------------------------------------- the graph copy
def test_graph_copy_replaces_data_and_shares_the_plan(gnn, be):
    g = regular_graph(gnn, N, be.dev, ndata=torch.randn(DIN, N, device=be.dev),
                      edata=torch.randn(2, 4 * N, device=be.dev))
    p = g.plan()
    from gnnb200.readout import _indicator_plan
    ip = _indicator_plan(g, False)
    y = torch.randn(5, N, device=be.dev)
    h = gnn.GNNGraph(g, ndata=y)
    assert h.plan() is p and _indicator_plan(h, False) is ip
    assert list(h.ndata) == ["x"] and h.x is y
    assert h.edata["e"] is g.edata["e"] and h.gdata == {}
    assert g.ndata["x"] is not y                          # g itself is unchanged
    h2 = gnn.GNNGraph(g, ndata={"a": y, "b": y}, gdata=torch.zeros(3, 1, device=be.dev))
    assert set(h2.ndata) == {"a", "b"} and h2.gdata["u"].shape == (3, 1)
    assert gnn.GNNGraph(g, ndata=None).ndata == {}
    assert be.calls is None or be.calls.count("gnnb_graph_create") == 2   # g's plan and its indicator plan


def test_graph_copy_size_checks(gnn, be):
    g = regular_graph(gnn, N, be.dev)
    with pytest.raises(AssertionError):
        gnn.GNNGraph(g, ndata=torch.zeros(2, N + 1))
    with pytest.raises(AssertionError):
        gnn.GNNGraph(g, edata=torch.zeros(2, N))
    with pytest.raises(AssertionError):
        gnn.GNNGraph(g, gdata=torch.zeros(2, 2))
    with pytest.raises(AssertionError):
        gnn.GNNGraph(g, torch.zeros(2))


def test_graph_copy_no_stale_self_loops(gnn, be):
    """add_self_loops caches its result on the graph; the copy must not inherit a result carrying the old features"""
    x1, x2 = torch.randn(3, N, device=be.dev), torch.randn(3, N, device=be.dev)
    g = regular_graph(gnn, N, be.dev, ndata=x1)
    gl = gnn.add_self_loops(g)
    assert gl.x is x1
    h = gnn.GNNGraph(g, ndata=x2)
    hl = gnn.add_self_loops(h)
    assert hl.x is x2 and hl is not gl and hl.num_edges == gl.num_edges


def test_feature_queries(gnn):
    g = gnn.GNNGraph([1, 2], [2, 1])
    assert gnn.node_features(g) is None and gnn.edge_features(g) is None and gnn.graph_features(g) is None
    x = torch.zeros(3, 2)
    g = gnn.GNNGraph(g, ndata=x, edata=torch.ones(1, 2), gdata=torch.ones(4, 1))
    assert gnn.node_features(g) is x and gnn.edge_features(g).shape == (1, 2) and gnn.graph_features(g).shape == (4, 1)
    g = gnn.GNNGraph(g, ndata={"a": x, "b": x})
    with pytest.raises(ValueError):
        gnn.node_features(g)


# ---------------------------------------------------------------------------------------------- GPU
def _cuda():
    if not torch.cuda.is_available():
        pytest.skip("no CUDA device")


@pytest.mark.gpu
def test_tgcn_chain(gnn):
    """GNNChain(TGCN(3 => 5), dense) on (in, T, N) input (test/layers/temporalconv.jl:51-56)"""
    _cuda()
    torch.manual_seed(4)
    g = regular_graph(gnn, N, "cuda")
    m = gnn.GNNChain(gnn.TGCN(3, 5), Dense(5, 2, device="cuda"))
    m.cuda()
    x = torch.randn(3, 6, N, device="cuda", requires_grad=True)
    same_grads(m, lambda: m(g, x), lambda: m[1](m[0](g, x)), x)
    assert m(g, x).shape == (2, 6, N)


@pytest.mark.gpu
def test_graph_classification_model(gnn):
    """GCNConv -> GraphConv -> GlobalAttentionPool -> dense over a batch of 64 graphs: the chain's output and every
    gradient equal the layers applied by hand (the pooling on its fused route)"""
    _cuda()
    from gnnb200.layers import _Dense
    torch.manual_seed(5)
    rng = np.random.default_rng(5)
    graphs = [regular_graph(gnn, int(n), "cuda") for n in rng.integers(6, 40, 64)]
    g = gnn.batch(graphs)
    din, d = 16, 32
    pool = gnn.GlobalAttentionPool(_Dense(d, 1, device="cuda"), _Dense(d, d, device="cuda"))
    m = gnn.GNNChain(gnn.GCNConv(din, d, torch.relu, device="cuda"), gnn.GraphConv(d, d, torch.tanh, device="cuda"),
                     pool, Dense(d, 3, device="cuda"))
    x = torch.randn(din, g.num_nodes, device="cuda", requires_grad=True)
    same_grads(m, lambda: m(g, x), lambda: by_hand(list(m), g, x), x)
    assert m(g, x).shape == (3, 64)
    h = m[:3](gnn.GNNGraph(g, ndata=x.detach()))        # graph-only: the pooled readout lands in gdata
    assert torch.equal(h.gdata["u"], m[:3](g, x.detach())) and h.ndata["x"].shape == (d, g.num_nodes)
