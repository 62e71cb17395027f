"""random_walk_pe (graphneuralnetworks.jl_b200/transform.py over csrc/rwpe.cu's gnnb_random_walk_pe and the fused
propagate; GNNGraphs/src/transform.jl:975-990).

The contract, stated below in numpy:
- the reference: PE[k, j] = (RW^k)[j, j], RW[i, j] = A[i, j] * dinv[j], A the summed weights of the edges i -> j and
  dinv = 1 / weighted out-degree with +-Inf set to 0 (`dense_pe`, float64);
- the C entry: per segment of at most GNNB_RWPE_SMEM_MAX_NODES nodes, u_0 = e_j and
  u_k[t] = dinv[t] * Σ_{edges s -> t in plan order} w_e u_{k-1}[s], every product and sum rounded in float32, a row
  without edges 0, PE[k, j] = u_k[j]; rows of larger segments untouched (`ref_entry`).

Back ends of the mirror: `FakeRWPE`, the entry restated on host pointers over that statement (swapped in over
tests/fake_abi.py's double), and, under -m gpu, the CUDA kernels.  Each case runs on both routes: segments in shared
memory (the default) and every segment composed from the propagate (the bound patched to 0).  On the GPU the
shared-memory route must equal `ref_entry` bit for bit, and the two routes must equal each other bit for bit, on graphs
whose rows have at most the plan's chunk of edges.
"""
import os
import re
import sys
from types import SimpleNamespace

import numpy as np
import pytest
import scipy.sparse as sp
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
OK, EINVAL, ESIZE, ECUDA, ENOMEM, EUNSUPPORTED, EINDEX = range(7)
F32 = np.float32


def kernel_bound():
    with open(os.path.join(ROOT, "include", "gnnb200.h")) as f:
        return int(re.search(r"#define GNNB_RWPE_SMEM_MAX_NODES (\d+)", f.read()).group(1))


BOUND = kernel_bound()


# ---------------------------------------------------------------------------------------------- the contract in numpy
def dense_pe(s, t, n, w, K):
    """the reference statement for statement, in float64: (K, n).  s, t 0-based."""
    A = np.zeros((n, n))
    np.add.at(A, (s, t), np.ones(len(s)) if w is None else np.asarray(w, np.float64))
    deg = A.sum(1)
    with np.errstate(divide="ignore"):
        dinv = 1.0 / deg
    dinv[np.isinf(dinv)] = 0.0
    RW = A * dinv[None, :]
    out, P = np.zeros((K, n)), RW
    for k in range(K):
        out[k] = np.diag(P)
        P = P @ RW
    return out


def ref_entry(s, t, n, w, dinv, seg_ptr, K, bound=BOUND):
    """gnnb_random_walk_pe in float32: (n, K) node-major, NaN in the rows it leaves untouched; None if an edge crosses
    segments.  The plan order is a stable sort of the COO by target; every row is summed edge by edge in that order
    (vectorised over rows by the edge's rank within its row)."""
    s, t = np.asarray(s, np.int64), np.asarray(t, np.int64)
    order = np.argsort(t, kind="stable")
    ss, tt = s[order], t[order]
    ww = None if w is None else np.asarray(w, F32)[order]
    rowptr = np.concatenate([[0], np.cumsum(np.bincount(tt, minlength=n))]).astype(np.int64)
    rank = np.arange(len(tt)) - rowptr[tt]
    dinv = np.asarray(dinv, F32)
    out = np.full((n, K), np.nan, F32)
    for a, b in zip(seg_ptr[:-1], seg_ptr[1:]):
        a, b = int(a), int(b)
        m = b - a
        if m == 0 or m > bound:
            continue
        e0, e1 = rowptr[a], rowptr[b]
        sl, tl, rk = ss[e0:e1] - a, tt[e0:e1] - a, rank[e0:e1]
        if ((sl < 0) | (sl >= m)).any():
            return None
        has = rowptr[a + 1:b + 1] > rowptr[a:b]
        U = np.eye(m, dtype=F32)                              # U[node, source]: u_k of source a + c in column c
        for k in range(K):
            acc = np.zeros((m, m), F32)
            for r in range(int(rk.max()) + 1 if len(rk) else 0):
                sel = rk == r                                 # the r-th edge of every row that has one
                v = U[sl[sel]]
                if ww is not None:
                    v = v * ww[e0:e1][sel][:, None]
                acc[tl[sel]] = acc[tl[sel]] + v
            U = np.where(has[:, None], acc * dinv[a:b][:, None], F32(0))
            out[a:b, k] = np.diagonal(U)
    return out


# ---------------------------------------------------------------------------------------------- the C entry in numpy
def _fake_abi():
    sys.path.insert(0, os.path.join(ROOT, "tests"))
    import fake_abi
    return fake_abi


class FakeRWPE:
    """gnnb_random_walk_pe on host pointers over `ref_entry`, and gnnb_graph_subgraph (the node-mask case the
    propagate route uses); every other entry is the base double's."""

    def __init__(self, base):
        self.base, self.fa = base, _fake_abi()
        self.n_seg_seen = []

    def __getattr__(self, name):
        return getattr(self.base, name)

    def _fail(self, code, msg):
        self.base._err = msg.encode()
        return code

    def gnnb_random_walk_pe(self, h, w, dinv, seg_ptr, n_seg, K, out, stream):
        self.base.calls.append("gnnb_random_walk_pe")
        p = self.base._p(h)
        if p.ns != p.nd:
            return self._fail(ESIZE, "needs num_src == num_dst")
        if K < 1:
            return self._fail(EINVAL, "walk_length must be >= 1")
        n = p.nd
        sg = np.array([0, n]) if seg_ptr is None else self.fa._arr(seg_ptr, (n_seg + 1,), np.int64).copy()
        self.n_seg_seen.append(None if seg_ptr is None else int(n_seg))
        if n == 0:
            return OK
        if sg[0] != 0 or sg[-1] != n or (np.diff(sg) < 0).any():
            return self._fail(EINVAL, "seg_ptr must hold n_seg + 1 non-decreasing offsets from 0 to n")
        wv = None if w is None else self.fa._arr(w, (p.E,))
        res = ref_entry(p.s, p.t, n, wv, self.fa._arr(dinv, (n,)), sg, K)
        if res is None:
            return self._fail(EINVAL, "an edge crosses segments")
        o = self.fa._arr(out, (n, K))
        touched = ~np.isnan(res).all(1) if K else np.zeros(n, bool)
        o[touched] = res[touched]
        return OK

    def gnnb_graph_subgraph(self, h, node_keep, edge_keep, extra, out, node_map, kept_eids, n_out, e_out, stream):
        self.base.calls.append("gnnb_graph_subgraph")
        assert edge_keep is None and extra == 0
        p = self.base._p(h)
        nk = self.fa._arr(node_keep, (p.ns,), np.uint8) != 0
        newid = np.cumsum(nk) - 1
        if node_map is not None and p.ns:
            self.fa._arr(node_map, (p.ns,), np.int32)[...] = np.where(nk, newid, -1)
        kept = np.nonzero(nk[p.s] & nk[p.t])[0]
        self.fa._deref(out).value = self.base._new(self.fa._Plan(newid[p.s[kept]], newid[p.t[kept]], int(nk.sum()),
                                                                 int(nk.sum())))
        if kept_eids is not None and len(kept):
            self.fa._arr(kept_eids, (len(kept),), np.int64)[...] = kept
        self.fa._deref(n_out).value = int(nk.sum())
        self.fa._deref(e_out).value = len(kept)
        return OK


@pytest.fixture(params=["fake", pytest.param("cuda", marks=pytest.mark.gpu)])
def rb(request, gnn):
    """back end of the mirror: .dev, and .fake (the FakeRWPE in use, None on cuda)"""
    if request.param == "fake":
        from gnnb200 import transform
        with _fake_abi().installed() as fake:
            saved = transform.lib
            transform.lib = FakeRWPE(fake)
            try:
                yield SimpleNamespace(dev=torch.device("cpu"), fake=transform.lib)
            finally:
                transform.lib = saved
    else:
        if not torch.cuda.is_available():
            pytest.skip("no CUDA device")
        yield SimpleNamespace(dev=torch.device("cuda"), fake=None)


@pytest.fixture(params=["smem", "propagate"])
def route(request, monkeypatch):
    """the default routing, or every segment through the fused propagate"""
    if request.param == "propagate":
        from gnnb200 import transform
        monkeypatch.setattr(transform, "_RWPE_SMEM_MAX_NODES", 0)
    return request.param


def npy(x):
    return x.cpu().numpy()


def graph(gnn, s, t, n, dev, w=None, gi=None):
    s, t = np.asarray(s, np.int64), np.asarray(t, np.int64)
    kw = {}
    if gi is not None:
        gi = np.asarray(gi, np.int64)
        kw = dict(graph_indicator=torch.as_tensor(gi, device=dev), num_graphs=int(gi.max()) if len(gi) else 1)
    return gnn.GNNGraph(torch.as_tensor(s + 1, device=dev), torch.as_tensor(t + 1, device=dev),
                        None if w is None else torch.as_tensor(np.asarray(w, F32), device=dev), num_nodes=n, **kw)


def rel_err(got, ref):
    nr = np.linalg.norm(ref)
    if nr == 0:
        return 0.0 if not np.any(got) else np.inf
    return float(np.linalg.norm(got - ref) / nr)


def random_graph(rng, n, e, directed=True, weighted=False):
    s, t = rng.integers(0, n, e), rng.integers(0, n, e)
    if not directed:
        s, t = np.concatenate([s, t]), np.concatenate([t, s])
    w = rng.uniform(0.25, 2.0, len(s)).astype(F32) if weighted else None
    return s, t, w


def batch_of(parts):
    """(s, t, n, w or None, indicator) of the block-diagonal batch of parts [(s, t, n, w)]"""
    S, T, W, GI, off = [], [], [], [], 0
    for i, (s, t, n, w) in enumerate(parts):
        S.append(np.asarray(s, np.int64) + off)
        T.append(np.asarray(t, np.int64) + off)
        W.append(np.ones(len(s), F32) if w is None else np.asarray(w, F32))
        GI.append(np.full(n, i + 1))
        off += n
    weighted = any(p[3] is not None for p in parts)
    return (np.concatenate(S), np.concatenate(T), off, np.concatenate(W) if weighted else None, np.concatenate(GI))


def check_per_graph(got, parts, K, tol=1e-5):
    """got (K, N) against dense_pe of every part"""
    off = 0
    for s, t, n, w in parts:
        ref = dense_pe(np.asarray(s, np.int64), np.asarray(t, np.int64), n, w, K)
        err = rel_err(got[:, off:off + n], ref)
        assert err <= tol, (n, err)
        off += n


# ---------------------------------------------------------------------------------------------- the statement itself
def test_statement_entry_matches_dense_reference():
    rng = np.random.default_rng(0)
    s, t, w = random_graph(rng, 40, 120, weighted=True)
    A = np.zeros((40, 40))
    np.add.at(A, (s, t), w.astype(np.float64))
    deg = A.sum(1).astype(F32)
    with np.errstate(divide="ignore"):
        dinv = (F32(1) / deg).astype(F32)
    dinv[np.isinf(dinv)] = 0
    got = ref_entry(s, t, 40, w, dinv, np.array([0, 40]), 6)
    assert rel_err(got.T.astype(np.float64), dense_pe(s, t, 40, w, 6)) < 1e-5
    assert np.isnan(ref_entry(s, t, 40, w, dinv, np.array([0, 40]), 6, bound=39)).all()
    assert ((s < 20) != (t < 20)).any() and ref_entry(s, t, 40, w, dinv, np.array([0, 20, 40]), 6) is None


def test_header_bound_is_the_module_bound(gnn):
    from gnnb200 import transform
    assert transform._RWPE_KERNEL_MAX_NODES == BOUND == transform._RWPE_SMEM_MAX_NODES


# ---------------------------------------------------------------------------------------------- reference tests
def test_reference_known_answer(gnn, rb, route):
    """GNNGraphs/test/transform.jl:431-440"""
    g = gnn.GNNGraph(torch.tensor([1, 2, 2, 3], device=rb.dev), torch.tensor([2, 1, 3, 2], device=rb.dev),
                     ndata=torch.tensor([[-1.0, 0.0, 1.0]], device=rb.dev))
    pe = gnn.random_walk_pe(g, 3)
    assert pe.shape == (3, 3) and pe.dtype == torch.float32
    assert npy(pe).tolist() == [[0.0, 0.0, 0.0], [0.5, 1.0, 0.5], [0.0, 0.0, 0.0]]


def _cases():
    """name -> (s, t, n, w): 0-based edge lists"""
    rng = np.random.default_rng(7)
    c = {}
    c["directed"] = (*random_graph(rng, 30, 90)[:2], 30, None)
    s, t, w = random_graph(rng, 25, 60, directed=False, weighted=True)
    c["undirected_weighted"] = (s, t, 25, w)
    s, t, w = random_graph(rng, 20, 70, weighted=True)
    c["directed_weighted"] = (s, t, 20, w)
    # self loops, multi-edges, an isolated node (5), a node with in-edges and no out-edge (4)
    c["loops_multi_isolated_sink"] = ([0, 0, 0, 1, 1, 2, 3, 2, 0], [0, 1, 1, 2, 0, 2, 2, 4, 4], 6,
                                      [1.0, 2.0, 0.5, 1.5, 1.0, 3.0, 1.0, 0.25, 1.0])
    # out-degrees that sum to +0 (node 0: 1.5 - 1 - 0.5) and to -0 (node 2: a single -0.0 weight)
    c["out_degree_zero"] = ([0, 0, 0, 1, 2, 3, 1], [1, 2, 3, 0, 1, 0, 3], 4, [1.5, -1.0, -0.5, 2.0, -0.0, 1.0, 0.5])
    c["no_edges"] = ([], [], 5, None)
    return c


CASES = _cases()


# 64 powers of the signed case would measure cancellation, not the contract
@pytest.mark.parametrize("name,K", [(c, k) for c in CASES for k in (1, 3, 64) if (c, k) != ("out_degree_zero", 64)])
def test_against_dense_reference(gnn, rb, route, name, K):
    s, t, n, w = CASES[name]
    pe = npy(gnn.random_walk_pe(graph(gnn, s, t, n, rb.dev, w), K))
    assert pe.shape == (K, n)
    err = rel_err(pe.astype(np.float64), dense_pe(np.asarray(s, np.int64), np.asarray(t, np.int64), n, w, K))
    assert err <= 1e-5, err


def test_batched_cases_per_graph(gnn, rb, route):
    parts = [CASES[k] for k in CASES]
    s, t, n, w, gi = batch_of(parts)
    pe = npy(gnn.random_walk_pe(graph(gnn, s, t, n, rb.dev, w, gi), 5)).astype(np.float64)
    check_per_graph(pe, parts, 5)
    if rb.fake is not None and route == "smem":
        assert rb.fake.n_seg_seen[-1] == len(parts)


def test_empty_graph(gnn, rb):
    e = torch.zeros(0, dtype=torch.int64, device=rb.dev)
    pe = gnn.random_walk_pe(gnn.GNNGraph(e, e, num_nodes=0), 4)
    assert pe.shape == (4, 0) and pe.dtype == torch.float32


def test_bipartite_odd_steps_are_exact_zeros(gnn, rb, route):
    rng = np.random.default_rng(3)
    a, b = rng.integers(0, 12, 50), rng.integers(12, 30, 50)
    s, t = np.concatenate([a, b]), np.concatenate([b, a])
    w = rng.uniform(0.5, 2.0, len(s)).astype(F32)
    pe = npy(gnn.random_walk_pe(graph(gnn, s, t, 30, rb.dev, w), 8))
    assert (pe[0::2] == 0).all()                     # k = 1, 3, 5, 7
    assert (pe[1::2] > 0).any()
    assert rel_err(pe.astype(np.float64), dense_pe(s, t, 30, w, 8)) <= 1e-5


@pytest.mark.parametrize("bad", [0, -3])
def test_walk_length_must_be_positive(gnn, rb, bad):
    g = gnn.GNNGraph(torch.tensor([1, 2], device=rb.dev), torch.tensor([2, 1], device=rb.dev))
    with pytest.raises(AssertionError):
        gnn.random_walk_pe(g, bad)


def test_unsorted_indicator_or_crossing_edge_is_one_segment(gnn, rb):
    rng = np.random.default_rng(5)
    parts = [(*random_graph(rng, n, 3 * n, directed=False)[:2], n, None) for n in (7, 12, 9)]
    s, t, n, _, gi = batch_of(parts)
    plain = npy(gnn.random_walk_pe(graph(gnn, s, t, n, rb.dev), 6))
    seen = []
    batched = npy(gnn.random_walk_pe(graph(gnn, s, t, n, rb.dev, gi=gi), 6))
    assert np.array_equal(batched, plain)
    if rb.fake is not None:
        seen.append(rb.fake.n_seg_seen[-1])
    gi_unsorted = gi.copy()
    gi_unsorted[[0, -1]] = gi_unsorted[[-1, 0]]
    assert np.array_equal(npy(gnn.random_walk_pe(graph(gnn, s, t, n, rb.dev, gi=gi_unsorted), 6)), plain)
    if rb.fake is not None:
        seen.append(rb.fake.n_seg_seen[-1])
    s2, t2 = np.concatenate([s, [0]]), np.concatenate([t, [n - 1]])     # an edge from graph 1 to graph 3
    cross = npy(gnn.random_walk_pe(graph(gnn, s2, t2, n, rb.dev, gi=gi), 6))
    assert np.array_equal(cross, npy(gnn.random_walk_pe(graph(gnn, s2, t2, n, rb.dev), 6)))
    assert rel_err(cross.astype(np.float64), dense_pe(s2, t2, n, None, 6)) <= 1e-5
    if rb.fake is not None:
        seen.append(rb.fake.n_seg_seen[-1])
        assert seen == [3, None, None]


def test_large_segment_among_small_ones(gnn, rb, monkeypatch):
    """a bound of 10 sends the 12-node graph through the propagate on its derived subgraph plan, the rest to the entry"""
    from gnnb200 import transform
    monkeypatch.setattr(transform, "_RWPE_SMEM_MAX_NODES", 10)
    rng = np.random.default_rng(9)
    parts = []
    for n in (4, 12, 1, 9):
        s, t, w = random_graph(rng, n, 3 * n, directed=True, weighted=True)
        parts.append((s, t, n, w))
    s, t, n, w, gi = batch_of(parts)
    g = graph(gnn, s, t, n, rb.dev, w, gi)
    check_per_graph(npy(gnn.random_walk_pe(g, 7)).astype(np.float64), parts, 7)


# ---------------------------------------------------------------------------------------------- GPU: bits and scale
def gpu_dinv(gnn, g):
    deg = gnn.degree(g, torch.float32, dir="out")
    d = torch.reciprocal(deg)
    d[torch.isinf(d)] = 0
    return npy(d)


def mixed_batch(rng, sizes, weighted, deg=3):
    parts = []
    for n in sizes:
        s, t, w = random_graph(rng, n, deg * n, directed=True, weighted=weighted) if n > 1 else \
            (np.array([0]), np.array([0]), np.array([1.5], F32) if weighted else None)
        parts.append((s, t, n, w))
    return parts


@pytest.mark.gpu
@pytest.mark.parametrize("weighted", [False, True])
def test_gpu_smem_route_equals_statement_bits(gnn, weighted):
    rng = np.random.default_rng(11 + weighted)
    parts = mixed_batch(rng, [1, 2, 5, 23, 31, 32, 33, 64, 150, 300, BOUND, 17], weighted)
    s, t, n, w, gi = batch_of(parts)
    g = graph(gnn, s, t, n, "cuda", w, gi)
    assert int(np.bincount(t, minlength=n).max()) <= 128            # rows within one chunk
    pe = npy(gnn.random_walk_pe(g, 9))
    sg = np.concatenate([[0], np.cumsum([p[2] for p in parts])])
    ref = ref_entry(s, t, n, w, gpu_dinv(gnn, g), sg, 9)
    assert np.array_equal(pe, ref.T)


@pytest.mark.gpu
@pytest.mark.parametrize("weighted", [False, True])
def test_gpu_mixed_sizes_both_routes_same_bits(gnn, monkeypatch, weighted):
    from gnnb200 import transform
    rng = np.random.default_rng(21 + weighted)
    parts = mixed_batch(rng, [1, 2, 31, 32, 33, BOUND, BOUND + 1, 3, 100], weighted)
    s, t, n, w, gi = batch_of(parts)
    g = graph(gnn, s, t, n, "cuda", w, gi)
    pe = gnn.random_walk_pe(g, 12)
    check_per_graph(npy(pe).astype(np.float64), parts, 12)
    assert torch.equal(pe, gnn.random_walk_pe(g, 12))               # run to run
    monkeypatch.setattr(transform, "_RWPE_SMEM_MAX_NODES", 0)
    assert torch.equal(pe, gnn.random_walk_pe(g, 12))
    monkeypatch.setattr(transform, "_RWPE_SMEM_MAX_NODES", 32)
    assert torch.equal(pe, gnn.random_walk_pe(g, 12))


def _entry(gnn, g, dinv, seg_ptr, K, out):
    from gnnb200 import _lib
    p = g.plan()
    _lib.check(_lib.lib.gnnb_random_walk_pe(p.h, None if g.w is None else g.w.data_ptr(), dinv.data_ptr(),
                                            seg_ptr.data_ptr(), seg_ptr.numel() - 1, K, out.data_ptr(),
                                            torch.cuda.current_stream().cuda_stream))


@pytest.mark.gpu
def test_gpu_entry_rejects_foreign_segments_inside_bounds(gnn):
    """seg_ptr that an edge crosses, or that is malformed: GNNB_EINVAL, and nothing written past the output"""
    GUARD, K = 4096, 5
    rng = np.random.default_rng(4)
    parts = [(*random_graph(rng, n, 3 * n)[:2], n, None) for n in (20, 300, 40)]
    s, t, n, _, gi = batch_of(parts)
    s, t = np.concatenate([s, [5, 330]]), np.concatenate([t, [100, 2]])  # small -> medium, medium -> small
    g = graph(gnn, s, t, n, "cuda")
    dinv = torch.as_tensor(gpu_dinv(gnn, g), device="cuda")
    for seg in ([0, 20, 320, n], [0, 300, 20, n], [0, 20, 320, n + 5], [1, 20, 320, n]):
        out = torch.full((n * K + GUARD,), -7.0, device="cuda")
        with pytest.raises(ValueError):
            _entry(gnn, g, dinv, torch.tensor(seg, dtype=torch.int64, device="cuda"), K, out)
        assert bool((out[n * K:] == -7.0).all())
    out = torch.full((n * K + GUARD,), -7.0, device="cuda")        # one segment: the same call is valid
    _entry(gnn, g, dinv, torch.tensor([0, n], dtype=torch.int64, device="cuda"), K, out)
    assert bool((out[n * K:] == -7.0).all()) and not bool((out[:n * K] == -7.0).any())


@pytest.mark.gpu
def test_gpu_at_scale_molecules(gnn):
    """10 000 molecule-shaped graphs (23 nodes, about 50 edges, bidirected) against per-graph float64"""
    rng = np.random.default_rng(13)
    G, n1, K = 10_000, 23, 20
    a = rng.integers(0, n1, (G, 25))
    b = (a + rng.integers(1, n1, (G, 25))) % n1                   # no self loops
    off = (np.arange(G) * n1)[:, None]
    s = np.concatenate([(a + off).ravel(), (b + off).ravel()])
    t = np.concatenate([(b + off).ravel(), (a + off).ravel()])
    gi = np.repeat(np.arange(1, G + 1), n1)
    pe = npy(gnn.random_walk_pe(graph(gnn, s, t, G * n1, "cuda", gi=gi), K)).astype(np.float64)
    A = np.zeros((G, n1, n1))
    np.add.at(A, (s // n1, s % n1, t % n1), 1.0)
    deg = A.sum(2)
    with np.errstate(divide="ignore"):
        dinv = np.where(deg > 0, 1.0 / np.where(deg > 0, deg, 1), 0.0)
    RW = A * dinv[:, None, :]
    P = RW
    ref = np.zeros((K, G, n1))
    for k in range(K):
        ref[k] = np.diagonal(P, axis1=1, axis2=2)
        P = P @ RW
    got = pe.reshape(K, G, n1)
    err = np.linalg.norm(got - ref, axis=(0, 2)) / np.linalg.norm(ref, axis=(0, 2))
    assert err.max() <= 1e-5, err.max()


@pytest.mark.gpu
def test_gpu_at_scale_propagate_route(gnn):
    """one 20 000-node graph with 200 000 edges (above the bound: the propagate route), 512 sampled sources against
    float64 sparse mat-vecs"""
    rng = np.random.default_rng(17)
    n, E, K = 20_000, 200_000, 16
    s, t = rng.integers(0, n, E), rng.integers(0, n, E)
    w = rng.uniform(0.5, 1.5, E).astype(F32)
    pe = npy(gnn.random_walk_pe(graph(gnn, s, t, n, "cuda", w), K)).astype(np.float64)
    A = sp.csr_matrix((w.astype(np.float64), (s, t)), shape=(n, n))
    deg = np.asarray(A.sum(1)).ravel()
    dinv = np.where(deg != 0, 1.0 / np.where(deg != 0, deg, 1), 0.0)
    RWt = (A @ sp.diags(dinv)).T.tocsr()
    src = np.sort(rng.choice(n, 512, replace=False))
    R = np.zeros((n, 512))
    R[src, np.arange(512)] = 1.0                                   # column c: the row vector e_src[c]^T RW^k
    ref = np.zeros((K, 512))
    for k in range(K):
        R = RWt @ R
        ref[k] = R[src, np.arange(512)]
    assert rel_err(pe[:, src], ref) <= 1e-5
