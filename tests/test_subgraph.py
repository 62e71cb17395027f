"""remove_edges, remove_nodes, getgraph and add_nodes (graphneuralnetworks.jl_b200/transform.py over csrc/plan.cu's
gnnb_graph_subgraph and gnnb_bernoulli_keep; GNNGraphs/src/transform.jl:121-147, 212-276, 553-563, 825-888).

The contract, stated below in numpy:
- the Bernoulli drop mask keep[i] = !(u_i < p), u_i = (splitmix64(splitmix64(seed) + i) >> 11) * 2^-53;
- the subgraph: kept nodes renumbered 0.. in ascending old id, then extra isolated nodes; the kept edges (mask and both
  endpoints kept) in parent COO order; and the child's CSR in either direction is a stable sort of the child's COO by
  row, which is what a fresh plan of the child's COO holds.

Back ends of the mirror: `FakeSub`, the two entries restated on host pointers over that statement (swapped in over
tests/fake_abi.py's double), and, under -m gpu, the CUDA kernels.  Each public function runs on both routes: a parent
without a plan (the child stays lazy) and a parent with one, with derivation forced whatever the parent's size.  On the GPU the derived plan
is compared with a fresh plan of the child's COO with torch.equal, and so are propagate and GCNConv on the two.
"""
import ctypes as C
import os
import sys

import numpy as np
import pytest
import torch
from scipy import stats

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
OK, EINVAL, ESIZE, ECUDA, ENOMEM, EUNSUPPORTED, EINDEX = range(7)
U = np.uint64
MASK = 2 ** 64 - 1


# ---------------------------------------------------------------------------------------------- the contract in numpy
def smix_int(x):
    """splitmix64's output function on a Python int"""
    x = (x + 0x9E3779B97F4A7C15) & MASK
    x = ((x ^ (x >> 30)) * 0xBF58476D1CE4E5B9) & MASK
    x = ((x ^ (x >> 27)) * 0x94D049BB133111EB) & MASK
    return x ^ (x >> 31)


def smix(x):
    """the same on a uint64 array (numpy's array arithmetic wraps mod 2^64)"""
    x = x + U(0x9E3779B97F4A7C15)
    x = (x ^ (x >> U(30))) * U(0xBF58476D1CE4E5B9)
    x = (x ^ (x >> U(27))) * U(0x94D049BB133111EB)
    return x ^ (x >> U(31))


def ref_bernoulli_keep(n, p, seed):
    u = (smix(U(smix_int(seed & MASK)) + np.arange(n, dtype=np.uint64)) >> U(11)).astype(np.float64) * 2.0 ** -53
    return (~(u < p)).astype(np.uint8)


def ref_subgraph(s, t, n, node_keep, edge_keep, extra):
    """0-based (s, t) of the child, its node count, the kept parent edge ids and the node map"""
    nk = np.ones(n, bool) if node_keep is None else node_keep != 0
    ek = np.ones(len(s), bool) if edge_keep is None else edge_keep != 0
    ek = ek & nk[s] & nk[t]
    newid = np.cumsum(nk) - 1
    kept = np.nonzero(ek)[0]
    return newid[s[kept]], newid[t[kept]], int(nk.sum()) + int(extra), kept, np.where(nk, newid, -1)


# ---------------------------------------------------------------------------------------------- the C entries in numpy
def _fake_abi():
    sys.path.insert(0, os.path.join(ROOT, "tests"))
    import fake_abi
    return fake_abi


class FakeSub:
    """gnnb_graph_subgraph and gnnb_bernoulli_keep on host pointers over the statement above; every other entry is the
    base double's (whose gnnb_graph_csr_device is the stable sort of a plan's COO)."""

    def __init__(self, base):
        self.base, self.fa = base, _fake_abi()

    def __getattr__(self, name):
        return getattr(self.base, name)

    def _fail(self, code, msg):
        self.base._err = msg.encode()
        return code

    def gnnb_graph_subgraph(self, h, node_keep, edge_keep, extra, out, node_map, kept_eids, n_out, e_out, stream):
        self.base.calls.append("gnnb_graph_subgraph")
        p = self.base._p(h)
        if p.ns != p.nd:
            return self._fail(ESIZE, "subgraph needs num_src == num_dst")
        if extra < 0:
            return self._fail(EINVAL, "extra_nodes must be >= 0")
        n, E = p.ns, p.E
        nk = None if node_keep is None else self.fa._arr(node_keep, (n,), np.uint8)
        ek = None if edge_keep is None else self.fa._arr(edge_keep, (E,), np.uint8)
        s, t, n2, kept, nmap = ref_subgraph(p.s, p.t, n, nk, ek, extra)
        if n2 >= 2 ** 31 - 1:
            return self._fail(ESIZE, "kept nodes + extra_nodes must be < 2^31-1")
        self.fa._deref(out).value = self.base._new(self.fa._Plan(s, t, n2, n2))
        if node_map is not None and n:
            self.fa._arr(node_map, (n,), np.int32)[...] = nmap
        if kept_eids is not None and len(kept):
            self.fa._arr(kept_eids, (len(kept),), np.int64)[...] = kept
        self.fa._deref(n_out).value = n2
        self.fa._deref(e_out).value = len(kept)
        return OK

    def gnnb_bernoulli_keep(self, n, p, seed, keep, stream):
        self.base.calls.append("gnnb_bernoulli_keep")
        if not 0.0 <= p <= 1.0:
            return self._fail(EINVAL, "p must lie in [0, 1]")
        if n:
            self.fa._arr(keep, (n,), np.uint8)[...] = ref_bernoulli_keep(n, p, seed)
        return OK


@pytest.fixture(params=["fake", pytest.param("cuda", marks=pytest.mark.gpu)])
def sb(request, monkeypatch, gnn):
    """back end of the mirror: the numpy entries above (host tensors) or the CUDA kernels (device tensors)"""
    if request.param == "fake":
        from gnnb200 import transform
        with _fake_abi().installed() as fake:
            monkeypatch.setattr(transform, "lib", FakeSub(fake))
            yield torch.device("cpu")
    else:
        if not torch.cuda.is_available():
            pytest.skip("no CUDA device")
        yield torch.device("cuda")


@pytest.fixture
def always_derive(monkeypatch):
    """derive the child's plan whenever the parent has one, whatever its size"""
    from gnnb200 import transform
    monkeypatch.setattr(transform, "_DERIVE_MAX_EDGES", 2 ** 62)


@pytest.fixture(params=["lazy", "derived"])
def route(request, monkeypatch):
    """prepare(g): leave the parent without a plan, or build it so that the child's plan is derived"""
    if request.param == "derived":
        from gnnb200 import transform
        monkeypatch.setattr(transform, "_DERIVE_MAX_EDGES", 2 ** 62)

    def prepare(g):
        if request.param == "derived":
            g.plan()
        return g
    prepare.derived = request.param == "derived"
    return prepare


def npy(x):
    return x.cpu().numpy()


def tl(x):
    return npy(x).tolist()


def check_child(gnn, h, derived):
    """the child has a plan exactly when its parent had one, and that plan's CSR is the stable sort of its COO"""
    assert (h._plan is not None) == derived
    s, t = npy(h.s) - 1, npy(h.t) - 1
    for tr, key, other in ((False, t, s), (True, s, t)):
        rowptr, col, eid = (npy(a) for a in gnn.csr(h, transposed=tr))
        order = np.argsort(key, kind="stable")
        assert rowptr.tolist() == [0] + np.cumsum(np.bincount(key, minlength=h.num_nodes)).tolist()
        assert col.tolist() == other[order].tolist() and eid.tolist() == order.tolist()


# ---------------------------------------------------------------------------------------------- the statement itself
def test_statement_bernoulli_is_seeded():
    a = ref_bernoulli_keep(10_000, 0.3, 7)
    assert np.array_equal(a, ref_bernoulli_keep(10_000, 0.3, 7))
    assert not np.array_equal(a, ref_bernoulli_keep(10_000, 0.3, 8))
    assert np.array_equal(ref_bernoulli_keep(5_000, 0.3, 7), a[:5_000])          # a prefix of the same stream
    assert ref_bernoulli_keep(1000, 0.0, 1).all() and not ref_bernoulli_keep(1000, 1.0, 1).any()


@pytest.mark.parametrize("p", [0.05, 0.2, 0.5, 0.9])
def test_statement_bernoulli_count_is_binomial(p):
    n = 10 ** 6
    for seed in (0, 1, 2 ** 63 + 11):
        kept = int(ref_bernoulli_keep(n, p, seed).sum())
        assert abs(kept - n * (1 - p)) < 6 * np.sqrt(n * p * (1 - p))


def test_statement_bernoulli_uniform_over_index_deciles():
    n, p = 10 ** 6, 0.3
    for seed in (3, 4):
        dropped = 1 - ref_bernoulli_keep(n, p, seed).astype(np.int64)
        obs = dropped.reshape(10, -1).sum(1)
        assert stats.chisquare(obs).pvalue > 1e-4


# ---------------------------------------------------------------------------------------------- reference tests
def test_reference_remove_edges(gnn, sb, route):
    """GNNGraphs/test/transform.jl:104-137"""
    s, t = [1, 1, 2, 3], [2, 3, 4, 5]
    w = torch.tensor([0.1, 0.2, 0.3, 0.4], device=sb)
    e = torch.tensor([10.0, 11.0, 12.0, 13.0], device=sb)         # the reference's ['a', 'b', 'c', 'd']
    mk = lambda: route(gnn.GNNGraph(torch.tensor(s, device=sb), torch.tensor(t, device=sb), w, edata=e))

    h = gnn.remove_edges(mk(), [1])
    assert h.num_edges == 3 and tl(h.s) == s[1:] and tl(h.t) == t[1:]
    check_child(gnn, h, route.derived)

    h = gnn.remove_edges(mk(), [1, 2, 4])
    assert h.num_edges == 1 and tl(h.s) == [2] and tl(h.t) == [4]
    assert tl(h.w) == [pytest.approx(0.3)] and tl(h.e) == [12.0]
    check_child(gnn, h, route.derived)

    assert gnn.remove_edges(mk(), 1.0).num_edges == 0
    h = gnn.remove_edges(mk(), 0.0)
    assert h.num_edges == 4 and tl(h.s) == s and tl(h.t) == t and h.num_nodes == 5
    check_child(gnn, h, route.derived)


def test_reference_remove_nodes(gnn, sb, route):
    """GNNGraphs/test/transform.jl:195-255"""
    w = torch.tensor([0.1, 0.2, 0.3, 0.4], device=sb)
    x = torch.tensor([1.0, 2.0, 3.0, 4.0, 5.0], device=sb)
    e = torch.tensor([10.0, 11.0, 12.0, 13.0], device=sb)
    g = route(gnn.GNNGraph(torch.tensor([1, 1, 2, 3], device=sb), torch.tensor([2, 3, 4, 5], device=sb), w, ndata=x,
                           edata=e))
    h = gnn.remove_nodes(g, [1])
    assert h.num_edges == 2 and h.num_nodes == 4
    assert tl(h.s) == [1, 2] and tl(h.t) == [3, 4]
    assert npy(h.w).tolist() == npy(w)[2:].tolist() and tl(h.x) == [2.0, 3.0, 4.0, 5.0] and tl(h.e) == [12.0, 13.0]
    check_child(gnn, h, route.derived)

    g = route(gnn.GNNGraph(torch.tensor([1, 5, 2, 3], device=sb), torch.tensor([2, 3, 4, 5], device=sb), w, ndata=x,
                           edata=e))
    h = gnn.remove_nodes(g, [1, 4])
    assert h.num_edges == 2 and h.num_nodes == 3
    assert tl(h.s) == [3, 2] and tl(h.t) == [2, 3]
    assert npy(h.w).tolist() == npy(w)[[1, 3]].tolist() and tl(h.x) == [2.0, 3.0, 5.0] and tl(h.e) == [11.0, 13.0]
    check_child(gnn, h, route.derived)
    h2 = gnn.remove_nodes(g, [4, 1, 4, 1])                       # sort(union(...)): repeats and order do not matter
    assert tl(h2.s) == tl(h.s) and tl(h2.t) == tl(h.t) and h2.num_nodes == 3


def test_reference_remove_nodes_p(gnn, sb, route):
    """GNNGraphs/test/transform.jl:257-273 (the p = 0.5 case depends on the reference's generator)"""
    mk = lambda: route(gnn.GNNGraph(torch.tensor([1, 1, 2, 3], device=sb), torch.tensor([2, 3, 4, 5], device=sb)))
    h = gnn.remove_nodes(mk(), 1.0)
    assert h.num_nodes == 0 and h.num_edges == 0
    check_child(gnn, h, route.derived)
    h = gnn.remove_nodes(mk(), 0.0)
    assert h.num_nodes == 5 and h.num_edges == 4
    check_child(gnn, h, route.derived)


def test_reference_add_nodes(gnn, sb, route):
    """GNNGraphs/test/transform.jl:275-282"""
    g = route(gnn.GNNGraph(torch.tensor([1, 2, 3, 4], device=sb), torch.tensor([2, 3, 4, 6], device=sb),
                           ndata=torch.rand(2, 6, device=sb)))
    h = gnn.add_nodes(g, 5, ndata=torch.ones(2, 5, device=sb))
    assert h.num_nodes == g.num_nodes + 5 and h.num_edges == g.num_edges and h.num_graphs == g.num_graphs
    assert bool((h.x[:, 6:11] == 1).all()) and torch.equal(h.x[:, :6], g.x)
    assert tl(h.s) == tl(g.s) and tl(h.t) == tl(g.t)
    check_child(gnn, h, route.derived)


def cycle(n, dev):
    """a 2-regular graph: the cycle 1 -> 2 -> ... -> n -> 1 and back, with 16 node features"""
    s = np.concatenate([np.arange(1, n + 1), np.roll(np.arange(1, n + 1), -1)])
    t = np.concatenate([np.roll(np.arange(1, n + 1), -1), np.arange(1, n + 1)])
    return s, t, torch.rand(16, n, device=dev)


def test_reference_getgraph(gnn, sb, route):
    """GNNGraphs/test/transform.jl:83-102, cycles in place of random_regular_graph"""
    parts = [cycle(n, sb) for n in (10, 4, 7)]
    gs = [gnn.GNNGraph(torch.tensor(s, device=sb), torch.tensor(t, device=sb), ndata=x) for s, t, x in parts]
    g = route(gnn.batch(gs))
    g2b, nodemap = gnn.getgraph(g, 2, nmap=True)
    assert tl(g2b.s) == parts[1][0].tolist() and tl(g2b.t) == parts[1][1].tolist()
    assert torch.equal(g2b.x, gs[1].x) and tl(nodemap) == list(range(11, 15))
    assert g2b.num_graphs == 1 and tl(g2b.graph_indicator) == [1] * 4
    check_child(gnn, g2b, route.derived)
    assert isinstance(gnn.getgraph(g, 2), gnn.GNNGraph)

    g1b, nodemap = gnn.getgraph(gs[0], 1, nmap=True)
    assert g1b is gs[0] and tl(nodemap) == list(range(1, 11))


# ---------------------------------------------------------------------------------------------- beyond the reference
def test_getgraph_renumbers_by_position_and_slices_gdata(gnn, sb, route):
    parts = [cycle(n, sb) for n in (3, 2, 4)]
    gs = [gnn.GNNGraph(torch.tensor(s, device=sb), torch.tensor(t, device=sb), ndata=x, gdata=torch.full((2,), 10.0 * k,
                                                                                                        device=sb))
          for k, (s, t, x) in enumerate(parts)]
    g = route(gnn.batch(gs))
    g.gdata = {"u": torch.stack([h.gdata["u"] for h in gs], dim=-1)}
    h, nodes = gnn.getgraph(g, [3, 1], nmap=True)
    assert tl(nodes) == [1, 2, 3, 6, 7, 8, 9]                          # ascending old ids
    assert tl(h.graph_indicator) == [2, 2, 2, 1, 1, 1, 1]              # renumbered by position in i
    assert h.num_graphs == 2 and tl(h.gdata["u"][0]) == [20.0, 0.0]
    s, t = np.concatenate([parts[0][0], parts[2][0] + 3]), np.concatenate([parts[0][1], parts[2][1] + 3])
    assert tl(h.s) == s.tolist() and tl(h.t) == t.tolist()
    check_child(gnn, h, route.derived)


def test_getgraph_keeps_edges_with_both_endpoints(gnn, sb, route):
    """difference 4: an edge from a kept graph into another graph is dropped"""
    g = route(gnn.GNNGraph(torch.tensor([1, 1, 3, 4], device=sb), torch.tensor([2, 3, 4, 1], device=sb), num_nodes=4,
                           num_graphs=2, graph_indicator=torch.tensor([1, 1, 2, 2], device=sb)))
    h = gnn.getgraph(g, 1)
    assert tl(h.s) == [1] and tl(h.t) == [2] and h.num_nodes == 2


def test_remove_nodes_slices_graph_indicator_and_add_nodes_extends_it(gnn, sb, route):
    """differences 2 and 3"""
    parts = [cycle(n, sb) for n in (3, 4)]
    g = route(gnn.batch([gnn.GNNGraph(torch.tensor(s, device=sb), torch.tensor(t, device=sb)) for s, t, _ in parts]))
    h = gnn.remove_nodes(g, [2, 5])
    assert tl(h.graph_indicator) == [1, 1, 2, 2, 2] and h.num_nodes == 5 and h.num_graphs == 2
    check_child(gnn, h, route.derived)
    a = gnn.add_nodes(g, 3)
    assert tl(a.graph_indicator) == [1, 1, 1, 2, 2, 2, 2, 2, 2, 2] and a.num_nodes == 10
    check_child(gnn, a, route.derived)


def test_remove_edges_repeated_ids_and_seeded_p(gnn, sb, route):
    rng = np.random.default_rng(0)
    s, t = rng.integers(1, 41, 300), rng.integers(1, 41, 300)
    mk = lambda: route(gnn.GNNGraph(torch.tensor(s, device=sb), torch.tensor(t, device=sb), num_nodes=40))
    h = gnn.remove_edges(mk(), [5, 5, 300, 1, 5])
    assert h.num_edges == 297 and tl(h.s) == np.delete(s, [0, 4, 299]).tolist()
    a, b = gnn.remove_edges(mk(), 0.4, seed=9), gnn.remove_edges(mk(), 0.4, seed=9)
    keep = ref_bernoulli_keep(300, 0.4, 9).astype(bool)
    assert tl(a.s) == tl(b.s) == s[keep].tolist() and tl(a.t) == t[keep].tolist()
    check_child(gnn, a, route.derived)
    n = gnn.remove_nodes(mk(), 0.25, seed=4)
    rs, rt, n2, _, _ = ref_subgraph(s - 1, t - 1, 40, ref_bernoulli_keep(40, 0.25, 4), None, 0)
    assert n.num_nodes == n2 and tl(n.s) == (rs + 1).tolist() and tl(n.t) == (rt + 1).tolist()
    check_child(gnn, n, route.derived)


def test_routes_agree(gnn, sb, always_derive):
    """the lazy and the derived child are the same graph with the same weights and features"""
    rng = np.random.default_rng(1)
    s, t = rng.integers(1, 61, 500), rng.integers(1, 61, 500)
    w = torch.as_tensor(rng.random(500), dtype=torch.float32, device=sb)

    def mk(derived):
        g = gnn.GNNGraph(torch.tensor(s, device=sb), torch.tensor(t, device=sb), w, num_nodes=60,
                         ndata=torch.rand(3, 60, generator=torch.Generator().manual_seed(0)).to(sb),
                         edata=torch.arange(500.0, device=sb).reshape(1, 500))
        if derived:
            g.plan()
        return g

    for f in (lambda g: gnn.remove_edges(g, 0.3, seed=2), lambda g: gnn.remove_nodes(g, 0.2, seed=3),
              lambda g: gnn.remove_nodes(g, list(range(1, 61, 3))), lambda g: gnn.add_nodes(g, 4, ndata=torch.zeros(
                  3, 4, device=sb))):
        a, b = f(mk(False)), f(mk(True))
        assert a._plan is None and b._plan is not None
        for x, y in ((a.s, b.s), (a.t, b.t), (a.w, b.w), (a.x, b.x), (a.e, b.e)):
            assert torch.equal(x.cpu(), y.cpu())
        assert a.num_nodes == b.num_nodes


def test_route_follows_the_parent_size(gnn, sb, monkeypatch):
    """with g's plan built, every function derives the child's plan while g has at most transform._DERIVE_MAX_EDGES
    edges, and leaves the child lazy above that"""
    from gnnb200 import transform
    parts = [cycle(10, sb) for _ in range(8)]
    g = gnn.batch([gnn.GNNGraph(torch.tensor(s, device=sb), torch.tensor(t, device=sb)) for s, t, _ in parts])
    g.plan()
    edits = (lambda: gnn.remove_edges(g, 0.2, seed=1), lambda: gnn.remove_nodes(g, 0.1, seed=1),
             lambda: gnn.getgraph(g, [3]), lambda: gnn.add_nodes(g, 2))
    assert g.num_edges <= transform._DERIVE_MAX_EDGES
    for f in edits:
        check_child(gnn, f(), True)
    monkeypatch.setattr(transform, "_DERIVE_MAX_EDGES", g.num_edges - 1)
    for f in edits:
        check_child(gnn, f(), False)


def test_argument_errors(gnn, sb):
    g = gnn.GNNGraph(torch.tensor([1, 2, 3], device=sb), torch.tensor([2, 3, 1], device=sb), ndata=torch.rand(2, 3,
                                                                                                             device=sb))
    for bad in ([0], [4], [1, 4]):
        with pytest.raises(AssertionError):
            gnn.remove_edges(g, bad)
        with pytest.raises(AssertionError):
            gnn.remove_nodes(g, bad)
    for p in (-0.1, 1.5, float("nan")):
        with pytest.raises(ValueError):
            gnn.remove_edges(g, p)
        with pytest.raises(ValueError):
            gnn.remove_nodes(g, p)
    for bad in (1, 0, torch.tensor(1)):                         # the reference has no remove_nodes(g, ::Integer)
        with pytest.raises(TypeError):
            gnn.remove_nodes(g, bad)
    with pytest.raises(ValueError):
        gnn.remove_edges(g, [1.0, 2.0])                          # a float vector is neither ids nor a probability
    with pytest.raises(AssertionError):
        gnn.getgraph(g, 2)                                       # no graph_indicator: graph 1 only
    b = gnn.batch([g, g])
    with pytest.raises(AssertionError):
        gnn.getgraph(b, [1, 3])
    with pytest.raises(AssertionError):
        gnn.add_nodes(g, 2)                                      # ndata keys must match
    with pytest.raises(AssertionError):
        gnn.add_nodes(g, 2, ndata={"y": torch.rand(2, 2, device=sb)})
    with pytest.raises(AssertionError):
        gnn.add_nodes(g, 2, ndata=torch.rand(2, 3, device=sb))  # one column per new node


def test_bipartite_plan_and_negative_extra_are_refused(gnn, sb):
    from gnnb200 import transform
    lib = transform.lib
    s = torch.tensor([0, 1], dtype=torch.int64, device=sb)
    h = C.c_void_p()
    gnn._lib.check(lib.gnnb_graph_create(C.byref(h), s.data_ptr(), s.data_ptr(), 2, 3, 2, 8, 0, int(s.is_cuda), None))
    out, n2, e2 = C.c_void_p(), C.c_int64(0), C.c_int64(0)
    try:
        assert lib.gnnb_graph_subgraph(h, None, None, 0, C.byref(out), None, None, C.byref(n2), C.byref(e2),
                                       None) == ESIZE
        gnn._lib.check(lib.gnnb_graph_create(C.byref(out), s.data_ptr(), s.data_ptr(), 2, 2, 2, 8, 0, int(s.is_cuda),
                                             None))
        sq = C.c_void_p(out.value)
        try:
            assert lib.gnnb_graph_subgraph(sq, None, None, -1, C.byref(out), None, None, C.byref(n2), C.byref(e2),
                                           None) == EINVAL
        finally:
            lib.gnnb_graph_destroy(sq)
    finally:
        lib.gnnb_graph_destroy(h)


# ---------------------------------------------------------------------------------------------- GPU: derived == fresh
def fresh(gnn, h, chunk=128):
    """a graph built from the child's COO alone, its plan made at `chunk`"""
    try:
        gnn._lib.check(gnn._lib.lib.gnnb_set_chunk_edges(chunk))
        f = gnn.GNNGraph(h.s, h.t, h.w, num_nodes=h.num_nodes)
        f.plan()
    finally:
        gnn._lib.lib.gnnb_set_chunk_edges(128)
    return f


def assert_same_plan(gnn, h, chunk=128):
    assert h._plan is not None
    f = fresh(gnn, h, chunk)
    for tr in (False, True):
        for a, b in zip(gnn.csr(h, transposed=tr), gnn.csr(f, transposed=tr)):
            assert torch.equal(a, b), tr
    return f


def _parity_graphs():
    sys.path.insert(0, os.path.join(ROOT, "tests"))
    import test_gpu_parity
    return test_gpu_parity


EDITS = {
    "remove_edges_p": lambda gnn, g: gnn.remove_edges(g, 0.3, seed=5),
    "remove_edges_ids": lambda gnn, g: gnn.remove_edges(g, list(range(1, g.num_edges + 1, 3))),
    "remove_nodes_p": lambda gnn, g: gnn.remove_nodes(g, 0.2, seed=6),
    "remove_nodes_ids": lambda gnn, g: gnn.remove_nodes(g, list(range(2, g.num_nodes + 1, 7))),
    "getgraph": lambda gnn, g: gnn.getgraph(g, [2, 4]),
    "add_nodes": lambda gnn, g: gnn.add_nodes(g, 7),
}
PARITY_GRAPHS = ["small", "empty_rows", "hubs", "sparse", "chunk_edges", "chunk32"]


def parity_graph(gnn, name):
    """test_gpu_parity's graph `name` with its plan built at its chunk, cut into 5 consecutive node blocks"""
    tp = _parity_graphs()
    _, s, t, n, g = tp.build_graph(gnn, name)
    g.num_graphs = 5
    g.graph_indicator = torch.as_tensor(np.minimum(np.arange(n) * 5 // n, 4) + 1, device="cuda")
    return g, tp.GRAPHS[name].get("chunk", 128)


@pytest.mark.gpu
@pytest.mark.parametrize("by_src", [False, True], ids=["by_dst_only", "both_csr"])
@pytest.mark.parametrize("edit", list(EDITS))
@pytest.mark.parametrize("name", PARITY_GRAPHS)
def test_gpu_derived_plan_equals_fresh(gnn, always_derive, name, edit, by_src):
    g, chunk = parity_graph(gnn, name)
    if by_src:
        gnn.csr(g, transposed=True)
    h = EDITS[edit](gnn, g)
    assert_same_plan(gnn, h, chunk)


@pytest.mark.gpu
@pytest.mark.parametrize("name", ["hubs", "chunk_edges", "chunk32"])
def test_gpu_derived_again_and_self_loops(gnn, always_derive, name):
    g, chunk = parity_graph(gnn, name)
    gnn.csr(g, transposed=True)
    h = gnn.remove_nodes(gnn.remove_edges(g, 0.25, seed=1), 0.1, seed=2)      # a derived plan derived again
    f = assert_same_plan(gnn, h, chunk)
    hl, fl = gnn.add_self_loops(h), gnn.add_self_loops(f)
    for tr in (False, True):
        for a, b in zip(gnn.csr(hl, transposed=tr), gnn.csr(fl, transposed=tr)):
            assert torch.equal(a, b)


@pytest.mark.gpu
@pytest.mark.parametrize("name", ["hubs", "chunk_edges", "chunk32"])
def test_gpu_same_plan_same_numbers(gnn, always_derive, name):
    """propagate (+, mean, max) and a GCNConv forward and backward on the derived child and on a fresh one: same bits"""
    g, chunk = parity_graph(gnn, name)
    gnn.csr(g, transposed=True)
    h = gnn.remove_edges(g, 0.2, seed=3)
    f = assert_same_plan(gnn, h, chunk)
    torch.manual_seed(0)
    x = gnn.unrows(torch.randn(h.num_nodes, 128, device="cuda"))
    for aggr in ("+", "mean", "max"):
        assert torch.equal(gnn.propagate(gnn.copy_xj, h, aggr, xj=x), gnn.propagate(gnn.copy_xj, f, aggr, xj=x)), aggr
    layer = gnn.GCNConv(128, 128, torch.relu, device="cuda")
    outs = []
    for gg in (h, f):
        xg = x.clone().requires_grad_(True)
        layer.zero_grad()
        y = layer(gg, xg)
        (y * y).sum().backward()
        outs.append((y.detach(), xg.grad, layer.weight.grad.clone()))
    for a, b in zip(*outs):
        assert torch.equal(a, b)


@pytest.mark.gpu
def test_gpu_bernoulli_equals_statement(gnn):
    n = 10 ** 7
    for p, seed in ((0.2, 0), (0.5, 2 ** 64 - 1), (0.0, 5), (1.0, 5), (0.999, 123456789)):
        keep = torch.empty(n, dtype=torch.uint8, device="cuda")
        gnn._lib.check(gnn._lib.lib.gnnb_bernoulli_keep(n, p, seed, keep.data_ptr(), None))
        assert np.array_equal(npy(keep), ref_bernoulli_keep(n, p, seed)), (p, seed)


@pytest.mark.gpu
def test_gpu_edge_cases(gnn, always_derive):
    dev = "cuda"
    e = torch.zeros(0, dtype=torch.int64, device=dev)
    g0 = gnn.GNNGraph(e, e, num_nodes=10)
    g0.plan()
    for h in (gnn.remove_edges(g0, 0.5, seed=1), gnn.remove_nodes(g0, [1, 2]), gnn.add_nodes(g0, 3)):
        assert h.num_edges == 0
        assert_same_plan(gnn, h)
    g, _ = parity_graph(gnn, "small")
    gnn.csr(g, transposed=True)
    h = gnn.remove_nodes(g, 1.0)                               # everything removed
    assert h.num_nodes == 0 and h.num_edges == 0
    assert_same_plan(gnn, h)
    h = gnn.remove_edges(g, 1.0)                               # every edge removed, nodes kept
    assert h.num_edges == 0 and h.num_nodes == g.num_nodes
    assert_same_plan(gnn, h)
    h = gnn.remove_edges(g, 0.0)                               # nothing removed
    assert torch.equal(h.s, g.s) and torch.equal(h.t, g.t)
    assert_same_plan(gnn, h)
    h = gnn.add_nodes(g, 1000)                                 # extra nodes on a parent with both CSRs built
    assert h.num_nodes == g.num_nodes + 1000
    assert_same_plan(gnn, h)
    nm = torch.empty(g.num_nodes, dtype=torch.int32, device=dev)
    keep = torch.zeros(g.num_nodes, dtype=torch.uint8, device=dev)
    keep[::2] = 1
    out, n2, e2 = C.c_void_p(), C.c_int64(0), C.c_int64(0)
    gnn._lib.check(gnn._lib.lib.gnnb_graph_subgraph(g.plan().h, keep.data_ptr(), None, 0, C.byref(out), nm.data_ptr(),
                                                    None, C.byref(n2), C.byref(e2), None))
    gnn._lib.lib.gnnb_graph_destroy(out)
    k = npy(keep).astype(np.int64)
    ref = np.where(k != 0, np.cumsum(k) - 1, -1)
    assert npy(nm).tolist() == ref.tolist() and n2.value == int(keep.sum())


@pytest.fixture(scope="module")
def rmat_10m(gnn):
    if not torch.cuda.is_available():
        pytest.skip("no CUDA device")
    g = gnn.rmat_graph(10 ** 7, 10 ** 8, seed=17, device="cuda")
    g.plan()
    gnn.csr(g, transposed=True)
    return g


@pytest.mark.gpu
@pytest.mark.parametrize("what,p", [("edges", 0.2), ("nodes", 0.1)])
def test_gpu_at_scale(gnn, rmat_10m, always_derive, what, p):
    g = rmat_10m
    fn = gnn.remove_edges if what == "edges" else gnn.remove_nodes
    h = fn(g, p, seed=11)
    k = g.num_edges if what == "edges" else g.num_nodes
    kept = h.num_edges if what == "edges" else h.num_nodes
    assert abs(kept - k * (1 - p)) < 6 * np.sqrt(k * p * (1 - p))
    h2 = fn(g, p, seed=11)
    assert torch.equal(h.s, h2.s) and torch.equal(h.t, h2.t)
    del h2
    f = fresh(gnn, h)
    for tr in (False, True):
        a, b = gnn.csr(h, transposed=tr), gnn.csr(f, transposed=tr)
        assert all(torch.equal(x, y) for x, y in zip(a, b)), tr
        del a, b
