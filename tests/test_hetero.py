"""Heterogeneous graphs (graphneuralnetworks.jl_b200/hetero.py; GNNGraphs/src/gnnheterograph/*.jl and
GraphNeuralNetworks/src/layers/heteroconv.jl), bipartite message passing and the two-sided GCN entry
(gnnb_gcn_propagate_bipartite).

Back ends: `FakeHetero`, tests/fake_abi.py's double with the new entry (and the bipartite edge-code generator) restated
in float64 on host pointers, and, under -m gpu, the CUDA library.  References are float64 restatements on
scipy.sparse matrices of shape (num_dst, num_src).
"""
import operator
import os
import sys
from types import SimpleNamespace

import numpy as np
import pytest
import scipy.sparse as sp
import torch

ROOT = os.path.dirname(os.path.abspath(os.path.dirname(__file__)))
OK, EINVAL, ESIZE = 0, 1, 2
F64 = torch.float64


def _fake_abi():
    sys.path.insert(0, os.path.join(ROOT, "tests"))
    import fake_abi
    return fake_abi


class FakeHetero:
    """gnnb_gcn_propagate_bipartite and the bipartite code generator on host pointers; the rest is the base double's"""

    def __init__(self, base):
        self.base, self.fa = base, _fake_abi()

    def __getattr__(self, name):
        return getattr(self.base, name)

    def gnnb_gcn_propagate_bipartite(self, h, transposed, x, D, out, stream):
        self.base.calls.append("gnnb_gcn_propagate_bipartite")
        p = self.base._p(h)
        dout_ = np.bincount(p.s, minlength=p.ns).astype(np.float64)
        din = np.bincount(p.t, minlength=p.nd).astype(np.float64)
        with np.errstate(divide="ignore"):
            cs, cd = 1.0 / np.sqrt(dout_), 1.0 / np.sqrt(din)
        src, dst, n_in, n_out, c_in, c_out = ((p.s, p.t, p.ns, p.nd, cs, cd) if not transposed
                                               else (p.t, p.s, p.nd, p.ns, cd, cs))
        xv = self.fa._arr(x, (n_in, D)).astype(np.float64)
        m = xv[src] * c_in[src][:, None]
        o = self.fa._segment(0, m, dst, n_out)
        has = np.bincount(dst, minlength=n_out) > 0
        o[has] *= c_out[has][:, None]                      # rows without edges stay 0
        self.fa._arr(out, (n_out, D))[...] = o
        return OK

    def gnnb_gat_logit_terms(self, Wx, a, N, Cc, H, el, er, stream):
        """one half when el or er is NULL"""
        self.base.calls.append("gnnb_gat_logit_terms")
        if el is None and er is None:
            return self.base._fail(EINVAL, "el and er are both NULL")
        W = self.fa._arr(Wx, (N, H, Cc)).astype(np.float64)
        A = self.fa._arr(a, (H, 2 * Cc)).astype(np.float64)
        if el is not None:
            self.fa._arr(el, (N, H))[...] = (W * A[None, :, :Cc]).sum(-1)
        if er is not None:
            self.fa._arr(er, (N, H))[...] = (W * A[None, :, Cc:]).sum(-1)
        return OK

    def gnnb_gat_logit_terms_bwd(self, Wx, a, del_, der, N, Cc, H, dWx, da, stream):
        """a NULL del or der contributes nothing: its half of da is 0"""
        self.base.calls.append("gnnb_gat_logit_terms_bwd")
        if del_ is None and der is None:
            return self.base._fail(EINVAL, "del and der are both NULL")
        W = self.fa._arr(Wx, (N, H, Cc)).astype(np.float64)
        A = self.fa._arr(a, (H, 2 * Cc)).astype(np.float64)
        dl = np.zeros((N, H)) if del_ is None else self.fa._arr(del_, (N, H)).astype(np.float64)
        dr = np.zeros((N, H)) if der is None else self.fa._arr(der, (N, H)).astype(np.float64)
        acc = self.fa._arr(dWx, (N, H, Cc))
        acc[...] = acc.astype(np.float64) + dl[:, :, None] * A[None, :, :Cc] + dr[:, :, None] * A[None, :, Cc:]
        out = self.fa._arr(da, (H, 2 * Cc))
        out[:, :Cc] = (dl[:, :, None] * W).sum(0)
        out[:, Cc:] = (dr[:, :, None] * W).sum(0)
        return OK

    def gnnb_sample_codes(self, M, excl, x, m, seed, out, cnt, stream):
        self.base.calls.append("gnnb_sample_codes")
        k = min(int(m), int(M))
        rng = np.random.default_rng(int(seed) & 0x7FFFFFFF)
        if k:
            self.fa._arr(out, (k,), np.int64)[...] = rng.choice(int(M), size=k, replace=False)
        self.fa._deref(cnt).value = k
        return OK

    def gnnb_edge_decode(self, space, n1, n2, codes, n, base, s, t, stream):
        self.base.calls.append("gnnb_edge_decode")
        assert space == 4                                  # GNNB_CODES_BIPARTITE: code = (s - 1) n2 + (t - 1)
        c = self.fa._arr(codes, (n,), np.int64)
        if n:
            self.fa._arr(s, (n,), np.int64)[...] = c // n2 + base
            self.fa._arr(t, (n,), np.int64)[...] = c % n2 + base
        return OK


@pytest.fixture(params=["fake", pytest.param("cuda", marks=pytest.mark.gpu)])
def hb(request, gnn):
    """back end: .dev, .calls (entries the fake saw; None on cuda)"""
    if request.param == "fake":
        from gnnb200 import _lib, graph, layers, linkpred, msgpass
        with _fake_abi().installed() as fake:
            wrap = FakeHetero(fake)
            mods = [_lib, graph, layers, linkpred, msgpass]
            saved = [(m, m.lib) for m in mods]
            for m in mods:
                m.lib = wrap
            try:
                yield SimpleNamespace(dev=torch.device("cpu"), calls=fake.calls, fake=True)
            finally:
                for m, l in saved:
                    m.lib = l
    else:
        if not torch.cuda.is_available():
            pytest.skip("no CUDA device")
        torch.cuda.set_device(0)
        yield SimpleNamespace(dev=torch.device("cuda"), calls=None, fake=False)


def jl(a, dev):
    """(N, D) float64 numpy rows -> Julia-shaped (D, N) float32 on dev"""
    return torch.as_tensor(np.ascontiguousarray(a), dtype=torch.float32, device=dev).t()


def np_rows(x):
    return x.detach().t().to(F64).cpu().numpy()


def rel(a, b):
    d = np.linalg.norm(np.asarray(a, np.float64) - b)
    n = np.linalg.norm(b)
    return d / n if n > 0 else d


def adj(s, t, ns, nd, w=None):
    """A (num_dst, num_src): A[t, s] += w"""
    w = np.ones(len(s)) if w is None else np.asarray(w, np.float64)
    return sp.csr_matrix((w, (np.asarray(t) - 1, np.asarray(s) - 1)), shape=(nd, ns))


# ---------------------------------------------------------------------------------------------- 1. reference answers
def test_empty_constructor_and_add_edges(gnn):
    """GNNGraphs/test/gnnheterograph.jl "Empty constructor" """
    g = gnn.GNNHeteroGraph()
    assert g.num_nodes == {}
    g = gnn.add_edges(g, (("user", "like", "actor"), ([1, 2, 3, 3, 3], [3, 5, 1, 9, 4])))
    assert g.num_nodes["user"] == 3 and g.num_nodes["actor"] == 9
    assert g.num_edges[("user", "like", "actor")] == 5


def test_constructor_from_pairs_and_num_nodes(gnn):
    """gnnheterograph.jl "Constructor from pairs" and "simplified constructor" """
    hg = gnn.GNNHeteroGraph((("A", "e1", "B"), ([1, 2, 3, 4], [3, 2, 1, 5])))
    assert hg.num_nodes == {"A": 4, "B": 5} and hg.num_edges == {("A", "e1", "B"): 4}
    hg = gnn.GNNHeteroGraph((("A", "e1", "B"), ([1, 2, 3], [3, 2, 1])), (("A", "e2", "C"), ([1, 2, 3], [4, 5, 6])))
    assert hg.num_nodes == {"A": 3, "B": 3, "C": 6}
    assert hg.num_edges == {("A", "e1", "B"): 3, ("A", "e2", "C"): 3}
    rng = np.random.default_rng(0)
    e1 = (rng.integers(1, 11, 20), rng.integers(1, 21, 20))
    e2 = (rng.integers(1, 21, 30), rng.integers(1, 11, 30))
    hg = gnn.GNNHeteroGraph(((("A", "rel1", "B"), e1), (("B", "rel2", "A"), e2)), num_nodes=(("A", 10), ("B", 20)))
    assert hg.num_nodes == {"A": 10, "B": 20}
    assert hg.num_edges == {("A", "rel1", "B"): 20, ("B", "rel2", "A"): 30}
    hg = gnn.GNNHeteroGraph({("A", "rel1", "B"): e1}, num_nodes={"A": 10, "B": 20})
    assert hg.num_nodes == {"A": 10, "B": 20}


def test_generation_features_and_counts(gnn, hb):
    """gnnheterograph.jl "Generation", "features", "num_edge_types / num_node_types" """
    hg = gnn.rand_heterograph({"A": 10, "B": 20}, {("A", "rel1", "B"): 30, ("B", "rel2", "A"): 10},
                              ndata={"A": torch.rand(2, 10), "B": {"x": torch.rand(3, 20), "y": torch.rand(4, 20)}},
                              edata={("A", "rel1", "B"): torch.rand(5, 30)}, gdata=1, seed=3)
    assert hg.num_nodes == {"A": 10, "B": 20}
    assert hg.num_edges == {("A", "rel1", "B"): 30, ("B", "rel2", "A"): 10}
    assert hg.graph_indicator is None and hg.num_graphs == 1
    assert sorted(hg.ntypes) == ["A", "B"] and sorted(hg.etypes) == [("A", "rel1", "B"), ("B", "rel2", "A")]
    assert hg.ndata["A"]["x"].shape == (2, 10) and hg.ndata["B"]["y"].shape == (4, 20)
    assert hg.edata[("A", "rel1", "B")]["e"].shape == (5, 30) and hg.gdata == {"u": 1}
    assert gnn.num_edge_types(hg) == 2 and gnn.num_node_types(hg) == 2
    g = gnn.GNNGraph([1, 2], [2, 1])
    assert gnn.num_edge_types(g) == 1 and gnn.num_node_types(g) == 1
    for et in hg.etypes:                                   # m distinct edges per relation, in range
        s, t = gnn.edge_index(hg, et)
        assert s.numel() == hg.num_edges[et]
        assert int(s.max()) <= hg.num_nodes[et[0]] and int(t.max()) <= hg.num_nodes[et[2]]
        assert len(set(zip(s.tolist(), t.tolist()))) == s.numel()
    bg = gnn.rand_bipartite_heterograph((5, 7), 9, seed=1)           # bidirected: the reverse is the mirror
    s1, t1 = gnn.edge_index(bg, ("A", "to", "B"))
    s2, t2 = gnn.edge_index(bg, ("B", "to", "A"))
    assert torch.equal(s1, t2) and torch.equal(t1, s2)


def test_indexing_syntax(gnn):
    """gnnheterograph.jl "indexing syntax" """
    g = gnn.GNNHeteroGraph((("user", "rate", "movie"), ([1, 1, 2, 3], [7, 13, 5, 7])))
    g["movie"]["z"] = torch.rand(64, 13)
    g[("user", "rate", "movie")]["e"] = torch.rand(64, 4)
    g["user"]["x"] = torch.rand(64, 3)
    assert g.ndata["user"]["x"].shape == (64, 3) and g.ndata["movie"]["z"].shape == (64, 13)
    assert g.edata[("user", "rate", "movie")]["e"].shape == (64, 4)


def test_add_edges_three_cases(gnn, hb):
    """gnnheterograph.jl "add_edges" """
    n = 5
    g = gnn.rand_bipartite_heterograph((n, 2 * n), 15, seed=2)
    s, t = [1, 2, 3], [3, 2, 1]
    for g1 in (gnn.add_edges(g, ("A", "rel1", "B"), s, t), gnn.add_edges(g, (("A", "rel1", "B"), (s, t)))):
        assert gnn.num_node_types(g1) == 2 and gnn.num_edge_types(g1) == 3
        assert all(gnn.has_edge(g1, ("A", "rel1", "B"), i, j) for i, j in zip(s, t))
        assert g1.num_nodes["A"] == n and g1.num_nodes["B"] == 2 * n
    ed = torch.rand(3, 3)
    g3 = gnn.add_edges(g, (("A", "rel1", "C"), (s, t)), num_nodes={"A": 1, "B": 1, "C": 10}, edata=ed)
    assert gnn.num_node_types(g3) == 3 and gnn.num_edge_types(g3) == 3
    assert all(gnn.has_edge(g3, ("A", "rel1", "C"), i, j) for i, j in zip(s, t))
    assert torch.equal(g3.edata[("A", "rel1", "C")]["e"], ed)
    assert g3.num_nodes["A"] == n and g3.num_nodes["B"] == 2 * n and g3.num_nodes["C"] == 10


def test_add_self_loops_two_cases(gnn, hb):
    """gnnheterograph.jl "add self loops" """
    g1 = gnn.GNNHeteroGraph((("A", "to", "B"), ([1, 2, 3, 4], [3, 2, 1, 5])))
    g2 = gnn.add_self_loops(g1, ("A", "to", "B"))
    assert g2.num_edges[("A", "to", "B")] == g1.num_edges[("A", "to", "B")]
    g1 = gnn.GNNHeteroGraph((("A", "to", "A"), ([1, 2, 3, 4], [3, 2, 1, 5])))
    g2 = gnn.add_self_loops(g1, ("A", "to", "A"))
    assert g2.num_edges[("A", "to", "A")] == g1.num_edges[("A", "to", "A")] + g1.num_nodes["A"]
    w = torch.tensor([2.0, 3.0, 4.0, 5.0])                               # existing weights padded with ones
    g1 = gnn.GNNHeteroGraph({("A", "to", "A"): ([1, 2, 3, 4], [3, 2, 1, 5], w)})
    assert gnn.get_edge_weight(gnn.add_self_loops(g1), ("A", "to", "A")).tolist() == [2, 3, 4, 5, 1, 1, 1, 1, 1]


def _ones_graphconv(gnn, d, dev):
    l = gnn.GraphConv(d, d, bias=False)
    with torch.no_grad():
        l.weight1.fill_(1.0)
        l.weight2.fill_(1.0)
    return l.to(dev)


def test_destination_node_aggregation(gnn, hb):
    """GraphNeuralNetworks/test/layers/heteroconv.jl "Destination node aggregation", with its expected values"""
    d, n = 3, 5
    e = ([1, 1, 2, 3], [1, 2, 2, 3])
    g = gnn.GNNHeteroGraph(((("A", "to", "B"), e), (("B", "to", "A"), e), (("C", "to", "A"), e)),
                           num_nodes={"A": n, "B": n, "C": n}, device=hb.dev)
    ets = [("A", "to", "B"), ("B", "to", "A"), ("C", "to", "A")]
    x = {k: torch.rand(d, n, device=hb.dev) for k in "ABC"}
    Wm = torch.ones(d, d, device=hb.dev)
    model = gnn.HeteroGraphConv([(et, _ones_graphconv(gnn, d, hb.dev)) for et in ets], aggr=operator.add)
    y = model(g, x)
    assert list(y) == ["B", "A"]
    close = lambda a, b: torch.allclose(a, b, rtol=1e-5, atol=1e-5)
    assert close((Wm @ x["A"][:, [0, 1]]).sum(1, keepdim=True) + Wm @ x["B"][:, [1]], y["B"][:, [1]])
    assert close(Wm @ x["B"][:, [4]], y["B"][:, [4]])
    assert close((Wm @ x["B"][:, [0]] + Wm @ x["C"][:, [0]]) + 2 * Wm @ x["A"][:, [0]], y["A"][:, [0]])
    assert close((Wm @ x["B"][:, [0, 1]] + Wm @ x["C"][:, [0, 1]]).sum(1, keepdim=True) + 2 * Wm @ x["A"][:, [1]],
                 y["A"][:, [1]])
    assert close(2 * Wm @ x["A"][:, [4]], y["A"][:, [4]])
    model2 = gnn.HeteroGraphConv([(et, _ones_graphconv(gnn, d, hb.dev)) for et in ets], aggr=operator.sub)
    y2 = model2(g, x)
    assert close(y["B"], y2["B"])
    assert close(Wm @ x["B"][:, [0]] - Wm @ x["C"][:, [0]], y2["A"][:, [0]])
    assert close((Wm @ x["B"][:, [0, 1]] - Wm @ x["C"][:, [0, 1]]).sum(1, keepdim=True), y2["A"][:, [1]])


def test_constructor_from_pairs_layer(gnn):
    """heteroconv.jl "Constructor from pairs" """
    layer = gnn.HeteroGraphConv((("A", "to", "B"), gnn.GraphConv(64, 32, torch.tanh)),
                                (("B", "to", "A"), gnn.GraphConv(64, 32, torch.tanh)))
    assert len(layer.etypes) == 2
    layer = gnn.HeteroGraphConv({("A", "to", "B"): gnn.GraphConv(4, 2)})
    assert len(layer.etypes) == 1


def _dense(gnn, i, o, sigma=None):
    from gnnb200.layers import _DenseAct, identity
    return _DenseAct(i, o, sigma or identity)


LAYERS = {
    "GraphConv": lambda gnn: gnn.GraphConv(4, 2),
    "GCNConv": lambda gnn: gnn.GCNConv(4, 2, torch.tanh),
    "GATConv": lambda gnn: gnn.GATConv(4, 2),
    "GATv2Conv": lambda gnn: gnn.GATv2Conv(4, 2),
    "SAGEConv": lambda gnn: gnn.SAGEConv(4, 2, torch.tanh, bias=False, aggr=operator.add),
    "GINConv": lambda gnn: gnn.GINConv(_dense(gnn, 4, 2), 0.4),
    "EdgeConv": lambda gnn: gnn.EdgeConv(_dense(gnn, 8, 2), aggr=operator.add),
    "CGConv": lambda gnn: gnn.CGConv(4, 2, torch.tanh),
    "ResGatedGraphConv": lambda gnn: gnn.ResGatedGraphConv(4, 2),
}


@pytest.mark.parametrize("kind", list(LAYERS))
def test_layer_output_shapes_and_gradients(gnn, hb, kind):
    """heteroconv.jl's per-layer testsets: y.A is (2, 2), y.B (2, 3); and gradients reach every input and parameter"""
    torch.manual_seed(0)
    hg = gnn.rand_bipartite_heterograph((2, 3), 6, seed=5, device=hb.dev)
    layers = gnn.HeteroGraphConv((("A", "to", "B"), LAYERS[kind](gnn)), (("B", "to", "A"), LAYERS[kind](gnn))).to(hb.dev)
    x = {"A": torch.rand(4, 2, device=hb.dev, requires_grad=True), "B": torch.rand(4, 3, device=hb.dev, requires_grad=True)}
    y = layers(hg, x)
    assert tuple(y["A"].shape) == (2, 2) and tuple(y["B"].shape) == (2, 3)
    (y["A"].sum() + (y["B"] ** 2).sum()).backward()
    assert x["A"].grad is not None and x["B"].grad is not None
    assert all(torch.isfinite(p.grad).all() for p in layers.parameters() if p.grad is not None)


# ---------------------------------------------------------------------------------------------- 2. message passing
def _bip_graph(gnn, ns, nd, E, seed, dev, long_row=0, isolated=True):
    """random relation A -> B; `long_row` extra edges into target 1 (a row longer than the plan's chunk); with
    `isolated`, the last source has no out-edge and the last target no in-edge"""
    rng = np.random.default_rng(seed)
    hi_s, hi_t = (ns - 1, nd - 1) if isolated else (ns, nd)
    s = rng.integers(1, hi_s + 1, E)
    t = rng.integers(1, hi_t + 1, E)
    if long_row:
        s = np.concatenate([s, rng.integers(1, hi_s + 1, long_row)])
        t = np.concatenate([t, np.ones(long_row, np.int64)])
    g = gnn.GNNHeteroGraph({("A", "r", "B"): (torch.as_tensor(s), torch.as_tensor(t))},
                           num_nodes={"A": ns, "B": nd}, device=dev)
    return g, s, t


def _segment_ref(A, X, aggr, s, t, nd, msgw=None):
    """float64 propagate over A (num_dst, num_src) — sum / mean / max / min of w_e x[s_e] per target"""
    if aggr in ("+", "mean"):
        out = A @ X
        if aggr == "mean":
            out = out / np.maximum(np.bincount(t - 1, minlength=nd).reshape(-1, 1), 1)
        return out
    m = X[s - 1] * (1.0 if msgw is None else msgw[:, None])
    out = np.full((nd, X.shape[1]), -np.inf if aggr == "max" else np.inf)
    (np.maximum if aggr == "max" else np.minimum).at(out, t - 1, m)
    return out


SHAPES = [(300, 7, 900, 0), (7, 300, 900, 0), (40, 30, 200, 300)]      # ns >> nd, ns << nd, a row longer than chunk


@pytest.mark.parametrize("shape", SHAPES)
@pytest.mark.parametrize("msg", ["copy_xj", "w_mul_xj", "e_mul_xj"])
@pytest.mark.parametrize("aggr", ["+", "mean", "max", "min"])
def test_propagate_bipartite(gnn, hb, shape, msg, aggr):
    ns, nd, E, lr = shape
    widths = [3, 16] if hb.fake else [3, 16, 128, 256, 512, 1000]
    g, s, t = _bip_graph(gnn, ns, nd, E, 7, hb.dev, lr)
    Et = len(s)
    rng = np.random.default_rng(1)
    w = rng.uniform(0.5, 1.5, Et)
    if msg == "w_mul_xj":
        g = gnn.GNNHeteroGraph({("A", "r", "B"): (torch.as_tensor(s), torch.as_tensor(t), torch.as_tensor(w))},
                               num_nodes={"A": ns, "B": nd}, device=hb.dev)
    A = adj(s, t, ns, nd, None if msg == "copy_xj" else w)
    f = {"copy_xj": gnn.copy_xj, "w_mul_xj": gnn.w_mul_xj, "e_mul_xj": gnn.e_mul_xj}[msg]
    ag = {"+": operator.add, "mean": gnn.mean, "max": max, "min": min}[aggr]
    for D in widths:
        X = rng.standard_normal((ns, D))
        x = jl(X, hb.dev).requires_grad_(True)
        e = torch.as_tensor(w, dtype=torch.float32, device=hb.dev) if msg == "e_mul_xj" else None
        y = gnn.propagate(f, g, ag, xj=x, e=e)
        assert tuple(y.shape) == (D, nd)
        ref = _segment_ref(A, X, aggr, s, t, nd, None if msg == "copy_xj" else w)
        got = np_rows(y)
        G = rng.standard_normal((nd, D))
        if aggr in ("max", "min"):
            empty = np.bincount(t - 1, minlength=nd) == 0
            assert np.all(np.isinf(got[empty])) and rel(got[~empty], ref[~empty]) < 2e-6
            G[empty] = 0.0                                        # the ±Inf rows take no gradient
            (y * jl(G, hb.dev)).sum().backward()
            wv = np.ones(Et) if msg == "copy_xj" else w
            m = (X[s - 1] * wv[:, None]).astype(np.float32)       # NNlib's rule: every tied extremum gets Δ
            hit = m == ref.astype(np.float32)[t - 1]
            dref = np.zeros((ns, D))
            np.add.at(dref, s - 1, hit * G[t - 1] * wv[:, None])
            assert x.grad.shape == x.shape and rel(np_rows(x.grad), dref) < 2e-6
            continue
        assert rel(got, ref) < 2e-6
        (y * jl(G, hb.dev)).sum().backward()
        if aggr == "+":
            dref = A.T @ G
        else:
            cnt = np.maximum(np.bincount(t - 1, minlength=nd), 1).reshape(-1, 1)
            dref = A.T @ (G / cnt)
        assert x.grad.shape == x.shape and rel(np_rows(x.grad), dref) < 2e-6


@pytest.mark.parametrize("D", [3, 16, 128, 256, 512, 1000])
@pytest.mark.parametrize("weighted", [False, True])
def test_propagate_bipartite_bits(gnn, hb, D, weighted):
    """rows of at most `chunk` edges: bit-equal to the float32 sequential formula (each target's in-edges in COO order,
    m = x[s] * w rounded, acc = acc + m rounded)"""
    if hb.fake:
        pytest.skip("bit equality is a property of the CUDA kernels; the double rounds once from float64")
    ns, nd = 90, 60
    g, s, t = _bip_graph(gnn, ns, nd, 700, 13, hb.dev)
    rng = np.random.default_rng(3)
    w = rng.uniform(0.5, 1.5, len(s)).astype(np.float32)
    if weighted:
        g = gnn.GNNHeteroGraph({("A", "r", "B"): (torch.as_tensor(s), torch.as_tensor(t), torch.as_tensor(w))},
                               num_nodes={"A": ns, "B": nd}, device=hb.dev)
    assert np.bincount(t - 1).max() <= 128
    X = rng.standard_normal((ns, D)).astype(np.float32)
    y = gnn.propagate(gnn.w_mul_xj if weighted else gnn.copy_xj, g, operator.add, xj=jl(X, hb.dev))
    ref = np.zeros((nd, D), np.float32)
    for e in range(len(s)):
        m = X[s[e] - 1] * w[e] if weighted else X[s[e] - 1]
        ref[t[e] - 1] = ref[t[e] - 1] + m.astype(np.float32)
    assert np.array_equal(y.detach().t().cpu().numpy(), ref)


@pytest.mark.parametrize("shape", SHAPES)
def test_apply_edges_aggregate_softmax_bipartite(gnn, hb, shape):
    ns, nd, E, lr = shape
    g, s, t = _bip_graph(gnn, ns, nd, E, 3, hb.dev, lr)
    rng = np.random.default_rng(2)
    D = 5
    Xj, Xi = rng.standard_normal((ns, D)), rng.standard_normal((nd, D))
    xj, xi = jl(Xj, hb.dev).requires_grad_(True), jl(Xi, hb.dev).requires_grad_(True)
    m = gnn.apply_edges(gnn.xi_dot_xj, g, xi=xi, xj=xj)
    ref = (Xi[t - 1] * Xj[s - 1]).sum(1, keepdims=True)
    assert rel(np_rows(m), ref) < 2e-6
    a = gnn.softmax_edge_neighbors(g, m)
    mx = np.full(nd, -np.inf)
    np.maximum.at(mx, t - 1, ref[:, 0])
    ex = np.exp(ref[:, 0] - mx[t - 1])
    den = np.zeros(nd)
    np.add.at(den, t - 1, ex)
    aref = ex / den[t - 1]
    assert rel(np_rows(a)[:, 0], aref) < 2e-6
    out = gnn.aggregate_neighbors(g, operator.add, a * gnn.apply_edges(gnn.copy_xj, g, xj=xj))
    A = sp.csr_matrix((aref, (t - 1, s - 1)), shape=(nd, ns))
    assert tuple(out.shape) == (D, nd) and rel(np_rows(out), A @ Xj) < 2e-6
    out.sum().backward()
    # float64 autograd of the same formula
    Xj_, Xi_ = torch.tensor(Xj, requires_grad=True), torch.tensor(Xi, requires_grad=True)
    st, tt = torch.as_tensor(s - 1), torch.as_tensor(t - 1)
    lg = (Xi_[tt] * Xj_[st]).sum(1)
    mxx = torch.full((nd,), -torch.inf, dtype=F64).scatter_reduce(0, tt, lg, "amax")
    ex_ = torch.exp(lg - mxx[tt])
    al = ex_ / torch.zeros(nd, dtype=F64).index_add(0, tt, ex_)[tt]
    torch.zeros(nd, D, dtype=F64).index_add(0, tt, al[:, None] * Xj_[st]).sum().backward()
    assert rel(np_rows(xj.grad), Xj_.grad.numpy()) < 2e-6 and rel(np_rows(xi.grad), Xi_.grad.numpy()) < 2e-6


# ---------------------------------------------------------------------------------------------- 3. bipartite GCN
def _gcn_ref(A, X, W, b, act):
    """conv.jl:45-69, heterograph branch, float64 torch (autograd gives dx, dW, db)"""
    dout_ = torch.as_tensor(np.asarray(A.sum(0)).ravel())
    din = torch.as_tensor(np.asarray(A.sum(1)).ravel())
    cout, cin = 1 / torch.sqrt(dout_), 1 / torch.sqrt(din)
    At = torch.as_tensor(A.toarray())
    xs = X * torch.nan_to_num(cout, posinf=0.0)[:, None]     # isolated rows: 0, not the reference's NaN
    p = (At @ xs) * torch.nan_to_num(cin, posinf=0.0)[:, None]
    return act(p @ W.t() + b)


@pytest.mark.parametrize("shape", [(300, 7, 900, 0), (7, 300, 900, 0), (40, 30, 200, 300), (20, 20, 80, 0)])
@pytest.mark.parametrize("D", [3, 16, 128, 256, 512, 1000])
def test_gcn_bipartite(gnn, hb, shape, D):
    ns, nd, E, lr = shape
    if hb.fake and D > 128:
        pytest.skip("widths past 128 select CUDA kernels; the double has one path")
    g, s, t = _bip_graph(gnn, ns, nd, E, 11, hb.dev, lr)
    A = adj(s, t, ns, nd)
    torch.manual_seed(0)
    layer = gnn.GCNConv(D, 8, torch.tanh).to(hb.dev)
    with torch.no_grad():
        layer.bias.uniform_(-1, 1)
    rng = np.random.default_rng(4)
    Xj, Xi = rng.standard_normal((ns, D)), rng.standard_normal((nd, D))
    xj = jl(Xj, hb.dev).requires_grad_(True)
    y = layer(g, (xj, jl(Xi, hb.dev)))
    if hb.fake:
        assert "gnnb_gcn_propagate_bipartite" in hb.calls
    X_ = torch.tensor(Xj, requires_grad=True)
    W_ = layer.weight.detach().to(F64).cpu().requires_grad_(True)
    b_ = layer.bias.detach().to(F64).cpu().requires_grad_(True)
    ref = _gcn_ref(A, X_, W_, b_, torch.tanh)
    assert rel(np_rows(y), ref.detach().numpy()) < 2e-6
    G = rng.standard_normal((nd, 8))
    (y * jl(G, hb.dev)).sum().backward()
    (ref * torch.as_tensor(G)).sum().backward()
    assert rel(np_rows(xj.grad), X_.grad.numpy()) < 2e-6
    assert rel(layer.weight.grad.cpu().numpy(), W_.grad.numpy()) < 2e-6
    assert rel(layer.bias.grad.cpu().numpy(), b_.grad.numpy()) < 2e-6
    no_in = np.bincount(t - 1, minlength=nd) == 0                 # isolated targets give σ(b)
    no_out = np.bincount(s - 1, minlength=ns) == 0                # isolated sources get dx = 0
    if no_in.any():
        assert np.allclose(np_rows(y)[no_in], np.tanh(layer.bias.detach().cpu().numpy())[None], atol=1e-6)
    if no_out.any():
        assert np.all(np_rows(xj.grad)[no_out] == 0)


def test_gcn_square_relation_is_two_sided_and_shares_plan(gnn, hb):
    """A -> B with |A| == |B| gets c_src / c_dst, not the symmetric scales; the same plan serves a homogeneous gcn_conv
    and a bipartite one in either order, each with its own result"""
    n, D = 30, 16
    rng = np.random.default_rng(9)
    ring = np.arange(1, n + 1)                                    # every node has an in- and an out-edge
    s = np.concatenate([ring, rng.integers(1, n + 1, 90)])
    t = np.concatenate([np.roll(ring, 1), rng.integers(1, n + 1, 90)])
    A = adj(s, t, n, n)
    X = rng.standard_normal((n, D))
    torch.manual_seed(1)
    layer = gnn.GCNConv(D, D, add_self_loops=False).to(hb.dev)
    W = layer.weight.detach().to(F64).cpu()
    b = layer.bias.detach().to(F64).cpu()
    ref_bip = _gcn_ref(A, torch.tensor(X), W, b, lambda v: v).numpy()
    d = np.asarray(A.sum(1)).ravel()
    c = np.where(d > 0, 1 / np.sqrt(np.maximum(d, 1)), 0.0)
    ref_sym = ((A @ (X * c[:, None])) * c[:, None]) @ W.numpy().T + b.numpy()
    for order in ("hom-first", "bip-first"):
        hg = gnn.GNNHeteroGraph({("A", "r", "B"): (torch.as_tensor(s), torch.as_tensor(t))},
                                num_nodes={"A": n, "B": n}, device=hb.dev)
        gg = gnn.GNNGraph(torch.as_tensor(s), torch.as_tensor(t), num_nodes=n, device=hb.dev)
        gg._plan = hg.plan()                                      # one plan for both
        x = jl(X, hb.dev)
        runs = [("hom", gg), ("bip", hg)] if order == "hom-first" else [("bip", hg), ("hom", gg)]
        for kind, g in runs:
            y = np_rows(layer(g, x if kind == "hom" else (x, x)))
            want = ref_sym if kind == "hom" else ref_bip
            assert rel(y, want) < 2e-6, (order, kind)
        assert rel(ref_bip, ref_sym) > 1e-3                       # the two normalisations differ on this graph


def test_gcn_same_type_relation_with_self_loops(gnn, hb):
    """(A, r, A) with GCNConv's self loops: the reference's degree on that subgraph fails; here the types come from et"""
    n, D = 25, 16
    rng = np.random.default_rng(12)
    s, t = rng.integers(1, n + 1, 90), rng.integers(1, n + 1, 90)
    hg = gnn.GNNHeteroGraph({("A", "r", "A"): (torch.as_tensor(s), torch.as_tensor(t))}, device=hb.dev)
    n = hg.num_nodes["A"]
    X = rng.standard_normal((n, D))
    layer = gnn.GCNConv(D, 8).to(hb.dev)
    y = layer(hg, (jl(X, hb.dev), jl(X, hb.dev)))
    sl, tl = np.concatenate([s, np.arange(1, n + 1)]), np.concatenate([t, np.arange(1, n + 1)])
    ref = _gcn_ref(adj(sl, tl, n, n), torch.tensor(X), layer.weight.detach().to(F64).cpu(),
                   layer.bias.detach().to(F64).cpu(), lambda v: v)
    assert rel(np_rows(y), ref.numpy()) < 2e-6
    d = gnn.degree(hg, ("A", "r", "A"), dir="in")
    assert d.tolist() == np.bincount(t - 1, minlength=n).tolist()


# ---------------------------------------------------------------------------------------------- 4. bipartite GAT
def _gat_ref(l, A_s, A_t, Xj, Xi, nd):
    Wd = l.dense_x.weight.detach().to(F64).cpu().requires_grad_(True)
    a = l.a.detach().to(F64).cpu().requires_grad_(True)
    Xj_, Xi_ = torch.tensor(Xj, requires_grad=True), torch.tensor(Xi, requires_grad=True)
    C, H = l.channel[1], l.heads
    Wj = (Xj_ @ Wd.t()).reshape(-1, H, C)
    Wi = (Xi_ @ Wd.t()).reshape(-1, H, C)
    st, tt = torch.as_tensor(A_s - 1), torch.as_tensor(A_t - 1)
    z = (Wi[tt] * a[:C].t()).sum(-1) + (Wj[st] * a[C:].t()).sum(-1)
    lg = torch.nn.functional.leaky_relu(z, l.negative_slope)
    mx = torch.full((nd, H), -torch.inf, dtype=F64).scatter_reduce(0, tt[:, None].expand(-1, H), lg, "amax")
    ex = torch.exp(lg - mx[tt])
    den = torch.zeros(nd, H, dtype=F64).index_add(0, tt, ex)
    al = ex / den[tt]
    out = torch.zeros(nd, H, C, dtype=F64).index_add(0, tt, al[:, :, None] * Wj[st])
    out = out.reshape(nd, H * C) if l.concat else out.mean(1)
    return out + l.bias.detach().to(F64).cpu(), (Xj_, Xi_, Wd, a)


@pytest.mark.parametrize("heads,concat,C", [(1, True, 8), (8, True, 8), (8, False, 16), (2, True, 6)])
def test_gat_bipartite(gnn, hb, heads, concat, C):
    ns, nd = 60, 35
    g, s, t = _bip_graph(gnn, ns, nd, 300, 21, hb.dev, 0, isolated=False)
    torch.manual_seed(2)
    l = gnn.GATConv(12, C, heads=heads, concat=concat).to(hb.dev)
    with torch.no_grad():
        l.bias.uniform_(-1, 1)
    rng = np.random.default_rng(5)
    Xj, Xi = rng.standard_normal((ns, 12)), rng.standard_normal((nd, 12))
    ref, leaves = _gat_ref(l, s, t, Xj, Xi, nd)
    G = rng.standard_normal(ref.shape)
    (ref * torch.as_tensor(G)).sum().backward()
    outs = []
    for fused in (True, False):
        l.zero_grad()
        xj, xi = jl(Xj, hb.dev).requires_grad_(True), jl(Xi, hb.dev).requires_grad_(True)
        n0 = len(hb.calls) if hb.fake else 0
        y = l(g, (xj, xi), fused=fused)
        if hb.fake:
            made = hb.calls[n0:]
            from gnnb200.layers import gat_fusable, gat_logit_fusable
            on_kernels = fused and gat_fusable(C, heads)          # (2, 6) is a shape outside the fused set
            assert ("gnnb_gat_aggregate" in made) == on_kernels
            if on_kernels and gat_logit_fusable(C, heads):        # the one-half logit passes, el then er
                assert made.count("gnnb_gat_logit_terms") == 2
        assert rel(np_rows(y), ref.detach().numpy()) < 2e-6
        (y * jl(G, hb.dev)).sum().backward()
        assert rel(np_rows(xj.grad), leaves[0].grad.numpy()) < 2e-6
        assert rel(np_rows(xi.grad), leaves[1].grad.numpy()) < 2e-6
        assert rel(l.dense_x.weight.grad.cpu().numpy(), leaves[2].grad.numpy()) < 2e-6
        assert rel(l.a.grad.cpu().numpy(), leaves[3].grad.numpy()) < 2e-6
        outs.append(np_rows(y))
    assert rel(outs[0], outs[1]) < 2e-6


# ---------------------------------------------------------------------------------------------- 5. HeteroGraphConv
def test_heteroconv_gradients_and_plan_reuse(gnn, hb):
    """heteroconv.jl's gradient test against a float64 restatement, and a second forward creates no plan"""
    d, n = 3, 5
    g = gnn.rand_bipartite_heterograph((n, 2 * n), 15, seed=8, device=hb.dev)
    torch.manual_seed(3)
    model = gnn.HeteroGraphConv([(("A", "to", "B"), gnn.GraphConv(d, d)), (("B", "to", "A"), gnn.GraphConv(d, d))])
    model = model.to(hb.dev)
    for p in model.parameters():
        with torch.no_grad():
            p.uniform_(-1, 1)
    rng = np.random.default_rng(6)
    X = {"A": rng.random((n, d)), "B": rng.random((2 * n, d))}
    x = {k: jl(v, hb.dev).requires_grad_(True) for k, v in X.items()}
    y = model(g, x)
    (y["B"].sum() + (y["A"] ** 2).sum()).backward()
    X_ = {k: torch.tensor(v, requires_grad=True) for k, v in X.items()}
    P_ = [[p.detach().to(F64).cpu().requires_grad_(True) for p in (l.weight1, l.weight2, l.bias)] for l in model.layers]
    outs = {}
    for (W1, W2, b), et in zip(P_, model.etypes):
        s, t = gnn.edge_index(g, et)
        A = torch.as_tensor(adj(s.cpu().numpy(), t.cpu().numpy(), g.num_nodes[et[0]], g.num_nodes[et[2]]).toarray())
        outs[et[2]] = X_[et[2]] @ W1.t() + (A @ X_[et[0]]) @ W2.t() + b
    (outs["B"].sum() + (outs["A"] ** 2).sum()).backward()
    for k in "AB":
        assert rel(np_rows(y[k]), outs[k].detach().numpy()) < 2e-6
        assert rel(np_rows(x[k].grad), X_[k].grad.numpy()) < 2e-6
    for l, ps in zip(model.layers, P_):
        for p, q in zip((l.weight1, l.weight2, l.bias), ps):
            assert rel(p.grad.cpu().numpy(), q.grad.numpy()) < 2e-6
    if hb.fake:
        n0 = hb.calls.count("gnnb_graph_create")
        model(g, x)
        assert hb.calls.count("gnnb_graph_create") == n0
    else:
        y2 = model(g, x)
        assert all(torch.equal(y[k], y2[k]) for k in y)           # run-to-run bit-identical


def test_readme_example(gnn, hb):
    g = gnn.rand_bipartite_heterograph((10, 15), 20, device=hb.dev)
    layer = gnn.HeteroGraphConv((("A", "to", "B"), gnn.GraphConv(64, 32, gnn.relu)),
                                (("B", "to", "A"), gnn.GraphConv(64, 32, gnn.relu))).to(hb.dev)
    y = layer(g, {"A": torch.rand(64, 10, device=hb.dev), "B": torch.rand(64, 15, device=hb.dev)})
    assert tuple(y["A"].shape) == (32, 10) and tuple(y["B"].shape) == (32, 15)


# ---------------------------------------------------------------------------------------------- 6. batch / subgraph
def test_batch_and_edge_type_subgraph(gnn, hb):
    g1 = gnn.GNNHeteroGraph({("A", "r", "B"): ([1, 2], [1, 3]), ("B", "q", "A"): ([3], [2])},
                            num_nodes={"A": 2, "B": 3}, ndata={"A": torch.ones(4, 2)})
    g2 = gnn.GNNHeteroGraph({("A", "r", "B"): ([1], [2])}, num_nodes={"A": 3, "B": 2}, ndata={"A": torch.zeros(4, 3)})
    b = gnn.batch([g1, g2])
    assert b.num_nodes == {"A": 5, "B": 5} and b.num_graphs == 2
    s, t = gnn.edge_index(b, ("A", "r", "B"))
    assert s.tolist() == [1, 2, 3] and t.tolist() == [1, 3, 5]
    assert gnn.graph_indicator(b, "A").tolist() == [1, 1, 2, 2, 2]
    assert gnn.graph_indicator(b, "B").tolist() == [1, 1, 1, 2, 2]
    assert b.ndata["A"]["x"].shape == (4, 5)
    sub = gnn.edge_type_subgraph(b, ("A", "r", "B"))
    assert sub.etypes == [("A", "r", "B")] and sub.ntypes == ["A", "B"]
    assert sub.relation(("A", "r", "B")) is b.relation(("A", "r", "B"))
    p = sub.plan()
    assert b.plan(("A", "r", "B")) is p                           # the subgraph's plan is the parent's


# ---------------------------------------------------------------------------------------------- 7. errors
def test_errors(gnn, hb):
    g = gnn.rand_bipartite_heterograph((4, 6), 8, seed=1, device=hb.dev)
    sub = gnn.edge_type_subgraph(g, ("A", "to", "B"))
    with pytest.raises(AssertionError):                           # wrong feature count for a type
        gnn.GraphConv(3, 2).to(hb.dev)(sub, (torch.rand(3, 5, device=hb.dev), torch.rand(3, 6, device=hb.dev)))
    with pytest.raises(AssertionError):                           # unknown edge type
        gnn.edge_type_subgraph(g, ("A", "nope", "B"))
    with pytest.raises(TypeError, match="cheb_conv"):
        gnn.ChebConv(3, 2, 2)(sub, (torch.rand(3, 4), torch.rand(3, 6)))
    with pytest.raises(TypeError, match="sgc_conv|sg_conv"):
        gnn.SGConv(3, 2)(sub, torch.rand(3, 4))
    bad = gnn.GNNHeteroGraph({("A", "r", "B"): ([1, 5], [1, 2])}, num_nodes={"A": 3, "B": 2}, device=hb.dev)
    with pytest.raises(AssertionError):                           # out-of-range index, raised when the plan is built
        bad.plan()
    with pytest.raises(TypeError):                                # arguments that do not apply are refused
        gnn.add_edges(gnn.GNNGraph([1, 2], [2, 1]), [1], [2], num_nodes=3)
    with pytest.raises(TypeError):
        gnn.degree(g, ("A", "to", "B"), edge_weight=False)
    with pytest.raises(TypeError):
        gnn.degree(gnn.GNNGraph([1, 2], [2, 1]), None, "extra")
