"""Graph queries from the device plan (graphneuralnetworks.jl_b200/query.py): the known answers of
GNNGraphs/test/gnngraph.jl:42-170 (the symmetric 4-cycle and the directed 4-ring) and GNNGraphs/test/query.jl for
has_self_loops / has_multi_edges / is_bidirected.  CPU test double always; CUDA variants gated until they have run."""
import numpy as np
import pytest
import torch


def T(a, dev):
    return torch.tensor(a).to(dev)


def test_symmetric_graph(gnn, be):                          # gnngraph.jl:42-83
    dev = be.dev
    s, t = [1, 1, 2, 2, 3, 3, 4, 4], [2, 4, 1, 3, 2, 4, 1, 3]
    adj = [[0, 1, 0, 1], [1, 0, 1, 0], [0, 1, 0, 1], [1, 0, 1, 0]]
    g = gnn.GNNGraph(T(s, dev), T(t, dev))
    assert g.num_edges == 8 and g.num_nodes == 4
    assert sorted(gnn.outneighbors(g, 1)) == [2, 4] and sorted(gnn.inneighbors(g, 1)) == [2, 4]
    s1, t1 = gnn.sort_edge_index(gnn.edge_index(g))
    assert s1.tolist() == s and t1.tolist() == t
    lists = [[2, 4], [1, 3], [2, 4], [1, 3]]
    assert [sorted(a) for a in gnn.adjacency_list(g, dir="in")] == lists
    assert [sorted(a) for a in gnn.adjacency_list(g, dir="out")] == lists
    for d in ("out", "in"):
        assert gnn.adjacency_matrix(g, dir=d).tolist() == adj
    assert gnn.is_bidirected(g) and not gnn.has_self_loops(g) and not gnn.has_multi_edges(g)
    # a GNNGraph built from the matrix has the same edges (convert.jl:86-100)
    g2 = gnn.GNNGraph(torch.tensor(adj)).to(dev)
    a, b = gnn.sort_edge_index(gnn.edge_index(g2))
    assert a.tolist() == s and b.tolist() == t


def test_asymmetric_graph(gnn, be):                         # gnngraph.jl:128-168
    dev = be.dev
    s, t = [1, 2, 3, 4], [2, 3, 4, 1]
    g = gnn.GNNGraph(T(s, dev), T(t, dev))
    assert g.num_edges == 4 and g.num_nodes == 4
    assert gnn.outneighbors(g, 1) == [2] and gnn.inneighbors(g, 1) == [4]
    s1, t1 = gnn.sort_edge_index(gnn.edge_index(g))
    assert s1.tolist() == s and t1.tolist() == t
    assert gnn.adjacency_matrix(g).tolist() == [[0, 1, 0, 0], [0, 0, 1, 0], [0, 0, 0, 1], [1, 0, 0, 0]]
    assert gnn.adjacency_matrix(g, dir="in").tolist() == [[0, 0, 0, 1], [1, 0, 0, 0], [0, 1, 0, 0], [0, 0, 1, 0]]
    assert gnn.adjacency_list(g) == [[2], [3], [4], [1]] and gnn.adjacency_list(g, dir="out") == [[2], [3], [4], [1]]
    assert gnn.adjacency_list(g, dir="in") == [[4], [1], [2], [3]]
    assert not gnn.is_bidirected(g)


def test_adjacency_list_with_eid_and_flags(gnn, be):        # query.jl:176-198, 553-579
    dev = be.dev
    s, t = [3, 1, 3, 2, 2, 3], [1, 2, 1, 2, 3, 4]                       # a repeated edge (3 -> 1) and a self loop (2 -> 2)
    w = torch.tensor([1.0, 2.0, 3.0, 4.0, 5.0, 6.0]).to(dev)
    g = gnn.GNNGraph(T(s, dev), T(t, dev), w)
    adj, eid = gnn.adjacency_list(g, [3, 2], dir="out", with_eid=True)
    assert adj == [[1, 1, 4], [2, 3]] and eid == [[1, 3, 6], [4, 5]]    # COO order inside a node
    adj, eid = gnn.adjacency_list(g, [1, 4, 3], dir="in", with_eid=True)
    assert adj == [[3, 3], [3], [2]] and eid == [[1, 3], [6], [5]]
    assert gnn.has_self_loops(g) and gnn.has_multi_edges(g) and not gnn.is_bidirected(g)
    A = gnn.adjacency_matrix(g)
    assert float(A[2, 0]) == 4.0 and float(A[1, 1]) == 4.0 and A.dtype == torch.float32     # weights of repeats add up
    assert gnn.adjacency_matrix(g, weighted=False)[2, 0].item() == 2
    h = gnn.remove_self_loops(gnn.remove_multi_edges(g))
    assert not gnn.has_self_loops(h) and not gnn.has_multi_edges(h) and h.num_edges == 4
    assert gnn.is_bidirected(gnn.to_bidirected(h))


@pytest.mark.parametrize("dir", ["in", "out", "both"])
def test_weighted_degree_value_and_gradient(gnn, be, dir):
    """degree(g, T; dir, edge_weight=w) is scatter(+, w, t) / (w, s) / both (GNNGraphs/src/query.jl:359-369), and its
    gradient in w is scatter's pullback: Δ[t], Δ[s] or their sum — against float64 index_add and autograd"""
    dev = be.dev
    rng = np.random.default_rng(3)
    n, E = 30, 200
    s, t = rng.integers(1, n + 1, E), rng.integers(1, n - 4, E)           # the last nodes have no in-edge
    w = rng.uniform(0.5, 1.5, E)
    g = gnn.GNNGraph(T(s, dev), T(t, dev), num_nodes=n)
    wt = torch.as_tensor(w, dtype=torch.float32).to(dev).requires_grad_(True)
    w64 = torch.as_tensor(w).requires_grad_(True)

    def scatter(idx):
        return torch.zeros(n, dtype=torch.float64).index_add(0, torch.as_tensor(idx - 1), w64)

    ref = {"in": lambda: scatter(t), "out": lambda: scatter(s), "both": lambda: scatter(t) + scatter(s)}[dir]()
    d = gnn.degree(g, torch.float32, dir=dir, edge_weight=wt)
    assert d.dtype == torch.float32 and d.requires_grad
    assert torch.allclose(d.detach().cpu().double(), ref, rtol=1e-6, atol=0)
    cot = torch.randn(n, dtype=torch.float64, generator=torch.Generator().manual_seed(0))
    (gw,) = torch.autograd.grad((d.double() * cot.to(dev)).sum(), wt)
    (rw,) = torch.autograd.grad((ref * cot).sum(), w64)
    assert torch.allclose(gw.cpu().double(), rw, rtol=1e-6, atol=1e-6)
    # the graph's own weights take the same path; without grad the result has no history
    gg = gnn.GNNGraph(T(s, dev), T(t, dev), wt, num_nodes=n)
    (gw2,) = torch.autograd.grad((gnn.degree(gg, dir=dir).double() * cot.to(dev)).sum(), wt)
    assert torch.equal(gw2, gw)
    with torch.no_grad():
        assert not gnn.degree(g, dir=dir, edge_weight=wt).requires_grad
    assert not gnn.degree(g, dir=dir, edge_weight=wt.detach()).requires_grad
