"""laplacian_lambda_max and the Laplacian queries (graphneuralnetworks.jl_b200/query.py over csrc/lmax.cu's
gnnb_laplacian_lambda_max and gnnb_segment_dots; GNNGraphs/src/query.jl:420-485,587-610).

The contract, stated below in numpy (float64):
- `sym_s`: S of one graph, the matrix the reference's `eigsolve(Symmetric(L), ...)` sees.  A[s, t] sums the weights
  of the edges s -> t (duplicates add up, self loops count), transposed for every dir but "out"; under add_self_loops
  A + I; L = I - D^-1/2 A D^-1/2 with D the row sums; Symmetric reads the upper triangle of L.
- `ref_lmax`: its largest eigenvalue, from float64 degrees (the reference) or from the float32 degrees the entry gets.

Back ends of the mirror: `FakeLmax`, the two entries restated on host pointers (swapped in over tests/fake_abi.py's
double), and, under -m gpu, the CUDA kernels.
"""
import math
import os
import re
import sys
import warnings
from types import SimpleNamespace

import numpy as np
import pytest
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
OK, EINVAL, ESIZE, ECUDA, ENOMEM, EUNSUPPORTED, EINDEX = range(7)
F32 = np.float32


def _header_int(name):
    with open(os.path.join(ROOT, "include", "gnnb200.h")) as f:
        return int(re.search(r"#define %s (\d+)" % name, f.read()).group(1))


BOUND = _header_int("GNNB_LMAX_SMEM_MAX_NODES")
CHUNK = _header_int("GNNB_SEGDOT_CHUNK")


# ---------------------------------------------------------------------------------------------- the contract in numpy
def dense_a(s, t, n, w, dir="out"):
    A = np.zeros((n, n))
    np.add.at(A, (np.asarray(s, np.int64), np.asarray(t, np.int64)),
              np.ones(len(s)) if w is None else np.asarray(w, F32).astype(np.float64))
    return A if dir == "out" else A.T


def sym_s(s, t, n, w, dir="out", self_loops=False, deg=None):
    """S = Symmetric(L) of one graph; deg (the row sums of A, + 1 under self_loops) defaults to float64 sums"""
    A = dense_a(s, t, n, w, dir)
    if self_loops:
        A = A + np.eye(n)
    d = A.sum(1) if deg is None else np.asarray(deg, np.float64)
    c = 1 / np.sqrt(d)
    L = np.eye(n) - c[:, None] * A * c[None, :]
    U = np.triu(L, 1)
    return U + U.T + np.diag(np.diag(L))


def ref_lmax(*args, **kw):
    return float(np.linalg.eigvalsh(sym_s(*args, **kw))[-1])


def deg32(s, t, n, w, dir="out", self_loops=False):
    """the float32 degree in the reference's orientation, summed in COO order"""
    d = np.zeros(n, F32)
    idx = np.asarray(s if dir == "out" else t, np.int64)
    ww = np.ones(len(s), F32) if w is None else np.asarray(w, F32)
    for i, x in zip(idx, ww):
        d[i] = d[i] + x
    return d + F32(1) if self_loops else d


def _fake_abi():
    sys.path.insert(0, os.path.join(ROOT, "tests"))
    import fake_abi
    return fake_abi


class FakeLmax:
    """gnnb_laplacian_lambda_max and gnnb_segment_dots on host pointers over the statement; every other entry is the
    base double's."""

    def __init__(self, base):
        self.base, self.fa = base, _fake_abi()
        self.n_seg_seen = []

    def __getattr__(self, name):
        return getattr(self.base, name)

    def _fail(self, code, msg):
        self.base._err = msg.encode()
        return code

    def gnnb_laplacian_lambda_max(self, h, w, deg, dir, self_loops, seg_ptr, n_seg, lmax_out, info, stream):
        self.base.calls.append("gnnb_laplacian_lambda_max")
        p = self.base._p(h)
        n = p.nd
        sg = np.array([0, n]) if seg_ptr is None else self.fa._arr(seg_ptr, (n_seg + 1,), np.int64).copy()
        self.n_seg_seen.append(None if seg_ptr is None else int(n_seg))
        if sg[0] != 0 or sg[-1] != n or (np.diff(sg) < 0).any():
            return self._fail(EINVAL, "seg_ptr must hold n_seg + 1 non-decreasing offsets from 0 to n")
        ww = None if w is None else self.fa._arr(w, (p.E,))
        d = self.fa._arr(deg, (n,))
        out = self.fa._arr(lmax_out, (len(sg) - 1,), np.float64)
        inf = self.fa._arr(info, (len(sg) - 1,), np.int32)
        for k in range(len(sg) - 1):
            a, b = int(sg[k]), int(sg[k + 1])
            if b - a > BOUND:
                inf[k] = -1
                continue
            inf[k] = 0
            sel = ((p.s >= a) & (p.s < b)) | ((p.t >= a) & (p.t < b))
            if ((p.s[sel] < a) | (p.s[sel] >= b) | (p.t[sel] < a) | (p.t[sel] >= b)).any():
                return self._fail(EINVAL, "an edge crosses segments")
            out[k] = ref_lmax(p.s[sel] - a, p.t[sel] - a, b - a, None if ww is None else ww[sel],
                              "out" if dir == 0 else "in", bool(self_loops), deg=d[a:b]) if b > a else np.nan
        return OK

    def gnnb_segment_dots(self, X, K, ldx, y, n, seg_ptr, chunk_ptr, n_seg, n_chunks, partial, out, stream):
        self.base.calls.append("gnnb_segment_dots")
        sg = self.fa._arr(seg_ptr, (n_seg + 1,), np.int64)
        Xv = self.fa._arr(X, (K, ldx), np.float64)[:, :n]
        yv = self.fa._arr(y, (n,), np.float64)
        o = self.fa._arr(out, (n_seg, K), np.float64)
        for s in range(n_seg):
            o[s] = Xv[:, sg[s]:sg[s + 1]] @ yv[sg[s]:sg[s + 1]]
        return OK


@pytest.fixture(params=["fake", pytest.param("cuda", marks=pytest.mark.gpu)])
def pb(request, gnn):
    """back end of the mirror: .dev, and .fake (the FakeLmax in use, None on cuda)"""
    if request.param == "fake":
        from gnnb200 import query
        with _fake_abi().installed() as fake:
            saved = query.lib
            query.lib = FakeLmax(fake)
            try:
                yield SimpleNamespace(dev=torch.device("cpu"), fake=query.lib)
            finally:
                query.lib = saved
    else:
        if not torch.cuda.is_available():
            pytest.skip("no CUDA device")
        yield SimpleNamespace(dev=torch.device("cuda"), fake=None)


def npy(x):
    return x.detach().cpu().numpy()


def graph(gnn, s, t, n, dev, w=None, gi=None, **kw):
    s, t = np.asarray(s, np.int64), np.asarray(t, np.int64)
    if gi is not None:
        gi = np.asarray(gi, np.int64)
        kw.update(graph_indicator=torch.as_tensor(gi, device=dev), num_graphs=int(gi.max()) if len(gi) else 1)
    return gnn.GNNGraph(torch.as_tensor(s + 1, device=dev), torch.as_tensor(t + 1, device=dev),
                        None if w is None else torch.as_tensor(np.asarray(w, F32), device=dev), num_nodes=n, **kw)


def random_graph(rng, n, e, weighted=True):
    """directed, with duplicates and self loops, and a ring 0 -> 1 -> ... -> 0 (both ways) so that no node is
    isolated in either direction"""
    ring = np.arange(n)
    s = np.concatenate([rng.integers(0, n, e), ring, (ring + 1) % n])
    t = np.concatenate([rng.integers(0, n, e), (ring + 1) % n, ring])
    w = rng.uniform(0.1, 2.0, len(s)).astype(F32) if weighted else None
    return s, t, n, w


def batch_of(parts):
    """(s, t, n, w or None, indicator, seg_ptr) of the block-diagonal batch of parts [(s, t, n, w)]"""
    S, T, W, GI, off = [], [], [], [], 0
    for i, (s, t, n, w) in enumerate(parts):
        S.append(np.asarray(s, np.int64) + off)
        T.append(np.asarray(t, np.int64) + off)
        W.append(np.ones(len(s), F32) if w is None else np.asarray(w, F32))
        GI.append(np.full(n, i + 1))
        off += n
    weighted = any(p[3] is not None for p in parts)
    seg = np.concatenate([[0], np.cumsum([p[2] for p in parts])])
    return (np.concatenate(S), np.concatenate(T), off, np.concatenate(W) if weighted else None, np.concatenate(GI),
            seg)


CYCLE5 = ([0, 1, 2, 3, 4, 0, 1, 2, 3, 4], [1, 2, 3, 4, 0, 4, 0, 1, 2, 3], 5, None)     # GNNGraphs/test/query.jl:184-195
TRI = ([0, 1, 2], [1, 2, 0], 3, None)                                                  # 1 -> 2 -> 3 -> 1


# ---------------------------------------------------------------------------------------------- known answers
def test_statement_known_answers():
    assert abs(ref_lmax(*CYCLE5) - (1 + math.cos(math.pi / 5))) < 1e-12
    assert abs(ref_lmax(*TRI, "out") - (1 + math.sqrt(2))) < 1e-12
    sym = dense_a(*TRI, "out")
    assert abs(np.linalg.eigvalsh(np.eye(3) - (sym + sym.T) / 2)[-1] - 1.5) < 1e-12   # what a naive (A + A')/2 gives
    for d in ("in", "both"):
        assert abs(ref_lmax(*TRI, d) - 2.0) < 1e-12


def test_reference_known_answers(gnn, pb):
    """GNNGraphs/test/query.jl:184-195, and the directed 3-cycle on each dir"""
    g = graph(gnn, *CYCLE5[:3], pb.dev)
    v = gnn.laplacian_lambda_max(g)
    assert isinstance(v, float) and v == float(F32(v)) and abs(v - 1.809017) < 1e-6
    s, t, n, _, gi, _ = batch_of([CYCLE5] * 5)
    vb = gnn.laplacian_lambda_max(graph(gnn, s, t, n, pb.dev, gi=gi))
    assert vb.dtype == torch.float64 and vb.shape == (5,) and vb.device.type == pb.dev.type
    assert np.allclose(npy(vb), 1 + math.cos(math.pi / 5), rtol=0, atol=1e-12)
    for d, want in (("out", 1 + math.sqrt(2)), ("in", 2.0), ("both", 2.0)):
        assert abs(gnn.laplacian_lambda_max(graph(gnn, *TRI[:3], pb.dev), dir=d) - want) < 1e-6
        s, t, n, _, gi, _ = batch_of([TRI, CYCLE5, TRI])
        got = npy(gnn.laplacian_lambda_max(graph(gnn, s, t, n, pb.dev, gi=gi), dir=d))
        assert np.allclose(got[[0, 2]], want, rtol=0, atol=1e-12)


def _cases():
    rng = np.random.default_rng(7)
    c = {"weighted": random_graph(rng, 12, 30), "unweighted": random_graph(rng, 9, 20, weighted=False)}
    # duplicates (0 -> 1 three times), self loops on 2 and 3, a node (4) whose out-edge is only its loop
    c["duplicates_loops"] = ([0, 0, 0, 1, 2, 3, 3, 4, 1, 2, 4], [1, 1, 1, 2, 2, 3, 0, 4, 0, 4, 3], 5,
                             [1.0, 2.0, 0.5, 1.5, 3.0, 0.25, 1.0, 2.0, 0.75, 1.25, 0.5])
    return c


CASES = _cases()


@pytest.mark.parametrize("name", list(CASES))
@pytest.mark.parametrize("dir", ["out", "in", "both"])
@pytest.mark.parametrize("self_loops", [False, True])
def test_against_statement(gnn, pb, name, dir, self_loops):
    s, t, n, w = CASES[name]
    got = gnn.laplacian_lambda_max(graph(gnn, s, t, n, pb.dev, w), torch.float64, add_self_loops=self_loops, dir=dir)
    assert abs(got - ref_lmax(s, t, n, w, dir, self_loops)) <= 1e-6
    parts = [CASES[k] for k in CASES]
    S, T, N, W, gi, _ = batch_of(parts)
    got = npy(gnn.laplacian_lambda_max(graph(gnn, S, T, N, pb.dev, W, gi), add_self_loops=self_loops, dir=dir))
    want = [ref_lmax(ps, pt, pn, pw, dir, self_loops) for ps, pt, pn, pw in parts]
    assert np.allclose(got, want, rtol=0, atol=1e-6)


def test_isolated_nodes_assert(gnn, pb):
    g = graph(gnn, [0, 1], [1, 2], 3, pb.dev)                          # node 3 has no out-edge, node 1 no in-edge
    for d in ("out", "in"):
        with pytest.raises(AssertionError, match="Graph contains isolated nodes, cannot compute `normalized_adjacency`."):
            gnn.laplacian_lambda_max(g, dir=d)
        with pytest.raises(AssertionError, match="isolated"):
            gnn.normalized_laplacian(g, dir=d)
    assert gnn.laplacian_lambda_max(g, add_self_loops=True) > 0       # self loops give every node a degree


def test_unsorted_indicator_and_crossing_edges_follow_getgraph(gnn, pb):
    """graph k is getgraph(g, k): its nodes in increasing id (S reads the upper triangle, so the order matters on a
    directed graph), its edges those with both ends in it"""
    rng = np.random.default_rng(5)
    parts = [random_graph(rng, n, 2 * n) for n in (7, 12, 9)]
    s, t, n, w, gi, _ = batch_of(parts)
    perm = rng.permutation(n)                                          # shuffle the nodes: the indicator is unsorted
    inv = np.argsort(perm)
    s2, t2, gi2 = inv[s], inv[t], gi[perm]
    s2, t2 = np.concatenate([s2, [inv[0], inv[n - 1]]]), np.concatenate([t2, [inv[n - 1], inv[8]]])   # two crossing
    w2 = np.concatenate([w, [5.0, 7.0]]).astype(F32)
    for d in ("out", "in"):
        got = npy(gnn.laplacian_lambda_max(graph(gnn, s2, t2, n, pb.dev, w2, gi2), dir=d))
        for k in range(3):
            nodes = np.nonzero(gi2 == k + 1)[0]
            local = np.full(n, -1)
            local[nodes] = np.arange(len(nodes))
            e = (local[s2] >= 0) & (local[t2] >= 0)
            ps, pt, pw = local[s2[e]], local[t2[e]], w2[e]
            single = gnn.laplacian_lambda_max(graph(gnn, ps, pt, len(nodes), pb.dev, pw), torch.float64, dir=d)
            assert abs(got[k] - single) <= 1e-12 and abs(got[k] - ref_lmax(ps, pt, len(nodes), pw, d)) <= 1e-6


def test_graph_without_nodes_raises(gnn, pb):
    e = torch.zeros(0, dtype=torch.int64, device=pb.dev)
    with pytest.raises(ValueError, match="no nodes"):
        gnn.laplacian_lambda_max(gnn.GNNGraph(e, e, num_nodes=0))
    s, t, n, _, gi, _ = batch_of([CYCLE5, CYCLE5])
    gi = np.where(gi == 2, 3, gi)                                      # graph 2 of 3 has no nodes
    g = gnn.GNNGraph(torch.as_tensor(s + 1, device=pb.dev), torch.as_tensor(t + 1, device=pb.dev), num_nodes=n,
                     num_graphs=3, graph_indicator=torch.as_tensor(gi, device=pb.dev))
    with pytest.raises(ValueError, match="graph 2 has no nodes"):
        gnn.laplacian_lambda_max(g)


def test_return_types(gnn, pb):
    g = graph(gnn, *TRI[:3], pb.dev)
    v32 = gnn.laplacian_lambda_max(g)
    v64 = gnn.laplacian_lambda_max(g, torch.float64)
    assert type(v32) is float and type(v64) is float
    assert v32 == float(F32(1 + math.sqrt(2))) and abs(v64 - (1 + math.sqrt(2))) < 1e-14
    s, t, n, _, gi, _ = batch_of([TRI, CYCLE5])
    vb = gnn.laplacian_lambda_max(graph(gnn, s, t, n, pb.dev, gi=gi), torch.float16)
    assert isinstance(vb, torch.Tensor) and vb.dtype == torch.float64 and vb.shape == (2,)


def test_routing_with_the_bound_lowered(gnn, pb, monkeypatch):
    """a bound of 6 sends the graphs of 12, 30 and 90 nodes to the Lanczos route, together (90 needs restarts); the
    rest to the entry"""
    from gnnb200 import query
    monkeypatch.setattr(query, "_LMAX_SMEM_MAX_NODES", 6)
    rng = np.random.default_rng(9)
    parts = [random_graph(rng, n, 3 * n) for n in (4, 12, 1, 30, 6, 90)]
    parts[2] = ([0], [0], 1, np.array([2.0], F32))
    s, t, n, w, gi, seg = batch_of(parts)
    for d in ("out", "in"):
        got = npy(gnn.laplacian_lambda_max(graph(gnn, s, t, n, pb.dev, w, gi), dir=d))
        want = [ref_lmax(*p, d) for p in parts]
        assert np.allclose(got, want, rtol=0, atol=1e-5)
    if pb.fake is not None:
        assert pb.fake.n_seg_seen == [6, 6] and "gnnb_segment_dots" in pb.fake.calls
        assert "gnnb_propagate" in pb.fake.calls
    monkeypatch.setattr(query, "_LMAX_SMEM_MAX_NODES", 0)              # every graph on the Lanczos route
    got = npy(gnn.laplacian_lambda_max(graph(gnn, s, t, n, pb.dev, w, gi), add_self_loops=True))
    assert np.allclose(got, [ref_lmax(*p, "out", True) for p in parts], rtol=0, atol=1e-5)


def test_lanczos_gives_up_with_one_warning(gnn, pb, monkeypatch):
    from gnnb200 import query
    monkeypatch.setattr(query, "_LMAX_SMEM_MAX_NODES", 0)
    monkeypatch.setattr(query, "_LMAX_MAXITER", 1)
    monkeypatch.setattr(query, "_LMAX_TOL", 0.0)
    rng = np.random.default_rng(2)
    parts = [random_graph(rng, 80, 200), random_graph(rng, 90, 250)]
    s, t, n, w, gi, _ = batch_of(parts)
    with warnings.catch_warnings(record=True) as rec:
        warnings.simplefilter("always")
        got = npy(gnn.laplacian_lambda_max(graph(gnn, s, t, n, pb.dev, w, gi)))
    msgs = [r for r in rec if issubclass(r.category, RuntimeWarning)]
    assert len(msgs) == 1 and "2 of 2 graphs" in str(msgs[0].message)
    want = [ref_lmax(*p) for p in parts]
    assert (got <= np.array(want) + 1e-6).all() and (got > 1.0).all()  # Ritz values: from below


# ---------------------------------------------------------------------------------------------- the dense queries
def test_laplacian_matrix(gnn, pb):
    """GNNGraphs/test/query.jl:175-182: D - A with D the row sums; the element type follows the graph"""
    rng = np.random.default_rng(3)
    s, t = rng.integers(0, 10, 30), rng.integers(0, 10, 30)
    L = gnn.laplacian_matrix(graph(gnn, s, t, 10, pb.dev))
    A = dense_a(s, t, 10, None)
    assert L.dtype == torch.int64 and np.array_equal(npy(L), np.diag(A.sum(1)) - A)
    w = rng.uniform(0.1, 1.0, 30).astype(F32)
    for d in ("out", "in"):
        Lw = gnn.laplacian_matrix(graph(gnn, s, t, 10, pb.dev, w), dir=d)
        A = dense_a(s, t, 10, w, d)
        assert Lw.dtype == torch.float32 and np.allclose(npy(Lw), np.diag(A.sum(1)) - A, rtol=1e-6, atol=1e-6)


def test_normalized_and_scaled_laplacian(gnn, pb):
    s, t, n, w = CASES["duplicates_loops"]
    g = graph(gnn, s, t, n, pb.dev, w)
    for d in ("out", "in", "both"):
        for sl in (False, True):
            A = dense_a(s, t, n, w, d) + (np.eye(n) if sl else 0)
            c = 1 / np.sqrt(A.sum(1))
            L = npy(gnn.normalized_laplacian(g, add_self_loops=sl, dir=d))
            assert L.dtype == np.float32 and np.allclose(L, np.eye(n) - c[:, None] * A * c[None, :], atol=1e-6)
    L64 = npy(gnn.normalized_laplacian(g, torch.float64))
    lam = ref_lmax(s, t, n, w)
    for d in ("out", "in"):                                            # dir is not used, as in the reference
        Ls = npy(gnn.scaled_laplacian(g, torch.float64, dir=d))
        assert np.allclose(Ls, 2 / lam * L64 - np.eye(n), atol=1e-6)
    parts = [CASES["weighted"], CASES["duplicates_loops"]]
    S, T, N, W, gi, _ = batch_of(parts)
    gb = graph(gnn, S, T, N, pb.dev, W, gi)
    lam = max(ref_lmax(*p) for p in parts)
    assert np.allclose(npy(gnn.scaled_laplacian(gb, torch.float64)),
                       2 / lam * npy(gnn.normalized_laplacian(gb, torch.float64)) - np.eye(N), atol=1e-6)
    gx = graph(gnn, np.concatenate([S, [0]]), np.concatenate([T, [N - 1]]), N, pb.dev,
               np.concatenate([W, [1.0]]), gi)                         # an edge joins the graphs: the whole matrix
    lam = ref_lmax(np.concatenate([S, [0]]), np.concatenate([T, [N - 1]]), N, np.concatenate([W, [1.0]]))
    assert np.allclose(npy(gnn.scaled_laplacian(gx, torch.float64)),
                       2 / lam * npy(gnn.normalized_laplacian(gx, torch.float64)) - np.eye(N), atol=1e-6)


def test_has_isolated_nodes(gnn, pb):
    """GNNGraphs/test/query.jl:29-34"""
    g = graph(gnn, [0, 1, 2], [1, 2, 1], 3, pb.dev)
    assert gnn.has_isolated_nodes(g) is False
    assert gnn.has_isolated_nodes(g, dir="in") is True
    assert gnn.has_isolated_nodes(g, dir="both") is False


def test_argument_errors_and_heterographs(gnn, pb):
    g = graph(gnn, *TRI[:3], pb.dev)
    for f in (gnn.laplacian_lambda_max, gnn.normalized_laplacian, gnn.scaled_laplacian, gnn.laplacian_matrix,
              gnn.has_isolated_nodes):
        with pytest.raises(ValueError):
            f(g, dir="sideways")
    for f in (gnn.laplacian_lambda_max, gnn.normalized_laplacian, gnn.scaled_laplacian):
        with pytest.raises(TypeError):
            f(g, torch.int32)
    with pytest.raises(TypeError):
        gnn.laplacian_lambda_max(g, torch.float32, False)              # add_self_loops and dir are keywords
    hg = SimpleNamespace(is_hetero=True)
    for f in (gnn.laplacian_lambda_max, gnn.normalized_laplacian, gnn.scaled_laplacian, gnn.laplacian_matrix,
              gnn.has_isolated_nodes):
        with pytest.raises(TypeError, match="GNNHeteroGraph"):
            f(hg)


# ---------------------------------------------------------------------------------------------- GPU: the entry
def run_entry(gnn, g, seg, dir="out", self_loops=False, deg=None):
    """(lmax_out with -7 where untouched, info, deg) of one call of gnnb_laplacian_lambda_max"""
    from gnnb200 import _lib
    if deg is None:
        deg = gnn.degree(g, dir="out" if dir == "out" else "in").float().contiguous()
        if self_loops:
            deg = deg + 1
    out = torch.full((len(seg) - 1,), -7.0, dtype=torch.float64, device="cuda")
    info = torch.full((len(seg) - 1,), -7, dtype=torch.int32, device="cuda")
    segd = torch.as_tensor(np.asarray(seg, np.int64), device="cuda")
    dcode = {"out": 0, "in": 1, "both": 2}[dir]
    _lib.check(_lib.lib.gnnb_laplacian_lambda_max(g.plan().h, None if g.w is None else g.w.data_ptr(), deg.data_ptr(),
                                                  dcode, int(self_loops), segd.data_ptr(), len(seg) - 1,
                                                  out.data_ptr(), info.data_ptr(),
                                                  torch.cuda.current_stream().cuda_stream))
    return npy(out), npy(info), npy(deg)


def check_statement(parts, seg, got, deg, dir, self_loops, tol=1e-9):
    for k, (ps, pt, pn, pw) in enumerate(parts):
        want = ref_lmax(ps, pt, pn, pw, dir, self_loops, deg=deg[seg[k]:seg[k + 1]])
        assert abs(got[k] - want) <= tol, (pn, got[k], want)


@pytest.mark.gpu
@pytest.mark.parametrize("dir,self_loops", [("out", False), ("in", True), ("both", False)])
def test_gpu_entry_against_statement_every_size(gnn, dir, self_loops):
    rng = np.random.default_rng(11)
    parts = [random_graph(rng, n, 2 * n, weighted=n % 3 != 0) for n in range(1, BOUND + 1)]
    parts = [(s, t, n, np.ones(len(s), F32) if w is None else w) for s, t, n, w in parts]
    s, t, n, w, gi, seg = batch_of(parts)
    g = graph(gnn, s, t, n, "cuda", w, gi)
    got, info, deg = run_entry(gnn, g, seg, dir, self_loops)
    assert (info == 0).all()
    check_statement(parts, seg, got, deg, dir, self_loops)


@pytest.mark.gpu
def test_gpu_warp_and_cta_classes_same_bits(gnn):
    from gnnb200 import _lib
    rng = np.random.default_rng(23)
    parts = [random_graph(rng, n, 3 * n) for n in list(range(1, 34)) * 2]
    s, t, n, w, gi, seg = batch_of(parts)
    g = graph(gnn, s, t, n, "cuda", w, gi)
    for dir in ("out", "in"):
        a, ia, _ = run_entry(gnn, g, seg, dir)
        try:
            _lib.check(_lib.lib.gnnb_set_kernel_variant(12))
            b, ib, _ = run_entry(gnn, g, seg, dir)
        finally:
            _lib.check(_lib.lib.gnnb_set_kernel_variant(0))
        assert np.array_equal(ia, ib) and np.array_equal(a.view(np.uint64), b.view(np.uint64))


@pytest.mark.gpu
def test_gpu_same_bits_anywhere_in_a_batch_and_on_repeat(gnn):
    rng = np.random.default_rng(29)
    probe = [random_graph(rng, 20, 50), random_graph(rng, 120, 300)]
    filler = [random_graph(rng, n, 2 * n) for n in (5, 40, 3)]
    parts = filler + probe + filler[::-1] + probe
    s, t, n, w, gi, seg = batch_of(parts)
    g = graph(gnn, s, t, n, "cuda", w, gi)
    a, _, _ = run_entry(gnn, g, seg)
    assert np.array_equal(a[[3, 4]].view(np.uint64), a[[8, 9]].view(np.uint64))
    for _ in range(3):
        assert np.array_equal(run_entry(gnn, g, seg)[0].view(np.uint64), a.view(np.uint64))
    m = npy(gnn.laplacian_lambda_max(g))
    assert np.array_equal(m.view(np.uint64), a.view(np.uint64))


@pytest.mark.gpu
def test_gpu_entry_skips_large_and_rejects_bad_input(gnn):
    from gnnb200 import _lib
    rng = np.random.default_rng(4)
    parts = [random_graph(rng, n, 2 * n) for n in (20, BOUND + 1, 40)]
    s, t, n, w, gi, seg = batch_of(parts)
    g = graph(gnn, s, t, n, "cuda", w, gi)
    got, info, deg = run_entry(gnn, g, seg)
    assert info.tolist() == [0, -1, 0] and got[1] == -7.0
    check_statement(parts[:1], seg, got, deg, "out", False)
    assert abs(got[2] - ref_lmax(*parts[2], deg=deg[seg[2]:seg[3]])) <= 1e-9
    s2, t2 = np.concatenate([s, [5]]), np.concatenate([t, [int(seg[2]) + 3]])     # graph 1 -> graph 3
    g2 = graph(gnn, s2, t2, n, "cuda", np.concatenate([w, [1.0]]).astype(F32))
    with pytest.raises(ValueError, match=f"edge {len(s)} "):
        run_entry(gnn, g2, seg)
    for sg in ([0, 20, 120, n], [0, 120, 20, n], [0, 20, 120, n + 5], [1, 20, 120, n]):
        with pytest.raises(ValueError):
            run_entry(gnn, g, sg)


# ---------------------------------------------------------------------------------------------- GPU: the mirror
@pytest.mark.gpu
@pytest.mark.parametrize("n", [BOUND + 1, 1000, 5000])
def test_gpu_lanczos_route(gnn, n):
    rng = np.random.default_rng(n)
    parts = [random_graph(rng, n, 3 * n), random_graph(rng, 7, 12), random_graph(rng, n, 2 * n)]
    s, t, N, w, gi, seg = batch_of(parts)
    g = graph(gnn, s, t, N, "cuda", w, gi)
    for dir in ("out", "in"):
        got = npy(gnn.laplacian_lambda_max(g, dir=dir))
        for k, p in enumerate(parts):
            assert abs(got[k] - ref_lmax(*p, dir)) <= 1e-5, (n, k, got[k])


@pytest.mark.gpu
def test_gpu_batch_on_both_sides_of_the_bound(gnn):
    rng = np.random.default_rng(31)
    parts = [random_graph(rng, n, 3 * n) for n in (3, BOUND, 500, 17, BOUND + 1, 64, 300)]
    s, t, N, w, gi, seg = batch_of(parts)
    g = graph(gnn, s, t, N, "cuda", w, gi)
    got = npy(gnn.laplacian_lambda_max(g, add_self_loops=True))
    assert np.allclose(got, [ref_lmax(*p, "out", True) for p in parts], rtol=0, atol=1e-5)
    for k, p in enumerate(parts):                                     # one graph alone: the same value
        assert abs(gnn.laplacian_lambda_max(graph(gnn, *p[:3], "cuda", p[3]), torch.float64, add_self_loops=True)
                   - got[k]) <= 1e-6


@pytest.mark.gpu
def test_gpu_molecules(gnn):
    """10 000 molecule-shaped graphs (23 nodes, 25 bonds both ways plus a ring) against float64"""
    rng = np.random.default_rng(13)
    G, m = 10_000, 23
    a = rng.integers(0, m, (G, 25))
    b = (a + rng.integers(1, m, (G, 25))) % m
    ring = np.tile(np.arange(m), (G, 1))
    a, b = np.concatenate([a, ring], 1), np.concatenate([b, (ring + 1) % m], 1)
    off = (np.arange(G) * m)[:, None]
    s = np.concatenate([(a + off).ravel(), (b + off).ravel()])
    t = np.concatenate([(b + off).ravel(), (a + off).ravel()])
    gi = np.repeat(np.arange(1, G + 1), m)
    got = npy(gnn.laplacian_lambda_max(graph(gnn, s, t, G * m, "cuda", gi=gi)))
    A = np.zeros((G, m, m))
    np.add.at(A, (s // m, s % m, t % m), 1.0)
    c = 1 / np.sqrt(A.sum(2))
    L = np.eye(m) - c[:, :, None] * A * c[:, None, :]
    U = np.triu(L, 1)
    Sm = U + U.transpose(0, 2, 1) + np.eye(m) * np.diagonal(L, 0, 1, 2)[:, None, :]
    assert np.abs(got - np.linalg.eigvalsh(Sm)[:, -1]).max() <= 1e-9


@pytest.mark.gpu
def test_gpu_rmat_against_eigsh(gnn):
    """RMAT 200 k / 2 M, bidirected, plus a ring: the Lanczos route against scipy's eigsh in float64"""
    import scipy.sparse as sp
    from scipy.sparse.linalg import eigsh
    n = 200_000
    r = gnn.rmat_graph(n, 2_000_000, seed=5, device="cuda")
    s0, t0 = npy(r.s).astype(np.int64) - 1, npy(r.t).astype(np.int64) - 1
    ring = np.arange(n)
    s = np.concatenate([s0, t0, ring, (ring + 1) % n])
    t = np.concatenate([t0, s0, (ring + 1) % n, ring])
    g = graph(gnn, s, t, n, "cuda")
    got = gnn.laplacian_lambda_max(g, torch.float64)
    deg = npy(gnn.degree(g, dir="out")).astype(np.float64)
    A = sp.coo_matrix((np.ones(len(s)), (s, t)), shape=(n, n)).tocsr()
    c = sp.diags(1 / np.sqrt(deg))
    U = sp.triu(sp.identity(n) - c @ A @ c, 1)
    Dg = sp.diags((sp.identity(n) - c @ A @ c).diagonal())
    S = (U + U.T + Dg).tocsr()
    want = float(eigsh(S, k=1, which="LA", tol=1e-12, ncv=64, v0=np.ones(n))[0][0])
    assert abs(got - want) <= 1e-5, (got, want)


@pytest.mark.gpu
def test_gpu_nan_weight_stays_in_its_graph(gnn, monkeypatch):
    from gnnb200 import query
    rng = np.random.default_rng(17)
    parts = [random_graph(rng, n, 3 * n) for n in (10, 50, 12, 300, 400)]
    parts[1][3][4] = np.nan
    parts[3][3][7] = np.nan
    s, t, N, w, gi, _ = batch_of(parts)
    g = graph(gnn, s, t, N, "cuda", w, gi)
    for bound in (BOUND, 0):
        monkeypatch.setattr(query, "_LMAX_SMEM_MAX_NODES", bound)
        got = npy(gnn.laplacian_lambda_max(g))
        assert np.isnan(got[[1, 3]]).all()
        assert np.allclose(got[[0, 2, 4]], [ref_lmax(*parts[k]) for k in (0, 2, 4)], rtol=0, atol=1e-5)


@pytest.mark.gpu
def test_gpu_scaled_laplacian_uses_the_segment_maximum(gnn):
    rng = np.random.default_rng(19)
    parts = [random_graph(rng, n, 3 * n) for n in (30, 200, 8)]
    s, t, N, w, gi, _ = batch_of(parts)
    g = graph(gnn, s, t, N, "cuda", w, gi)
    lam = float(gnn.laplacian_lambda_max(g).max())
    assert abs(lam - max(ref_lmax(*p) for p in parts)) <= 1e-5
    L = gnn.normalized_laplacian(g, torch.float64)
    want = 2 / lam * L - torch.eye(N, dtype=torch.float64, device="cuda")
    assert torch.allclose(gnn.scaled_laplacian(g, torch.float64), want, rtol=0, atol=1e-12)
