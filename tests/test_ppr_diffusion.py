"""ppr_diffusion (graphneuralnetworks.jl_b200/transform.py over csrc/ppr.cu's gnnb_ppr_diffusion and gnnb_ppr_matrix;
GNNGraphs/src/transform.jl:1026-1051).

The contract, stated below in numpy:
- the reference: w_new[e] = alpha * inv(M)[t_e, s_e], M = I + (alpha - 1) A, A[t, s] the summed weight of the edges
  s -> t (`dense_ppr`, float64);
- the C entry, per segment of at most GNNB_PPR_SMEM_MAX_NODES nodes: M built row by row in plan order, inverted by
  Gauss-Jordan elimination with partial pivoting, every float32 operation rounded on its own (`build_m`,
  `gauss_jordan`, `ref_entry`); larger segments untouched, info = -1.

Back ends of the mirror: `FakePPR`, the two entries restated on host pointers over that statement (swapped in over
tests/fake_abi.py's double), and, under -m gpu, the CUDA kernels, which must equal `ref_entry` bit for bit.
"""
import os
import re
import sys
from types import SimpleNamespace

import numpy as np
import pytest
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
OK, EINVAL, ESIZE, ECUDA, ENOMEM, EUNSUPPORTED, EINDEX = range(7)
F32 = np.float32


def kernel_bound():
    with open(os.path.join(ROOT, "include", "gnnb200.h")) as f:
        return int(re.search(r"#define GNNB_PPR_SMEM_MAX_NODES (\d+)", f.read()).group(1))


BOUND = kernel_bound()


# ---------------------------------------------------------------------------------------------- the contract in numpy
def dense_ppr(s, t, n, w, alpha=0.85):
    """the reference statement for statement, in float64: the new weight of every edge.  s, t 0-based."""
    A = np.zeros((n, n))
    np.add.at(A, (t, s), np.ones(len(s)) if w is None else np.asarray(w, np.float64))
    M = np.eye(n) + (float(F32(alpha)) - 1) * A
    P = float(F32(alpha)) * np.linalg.inv(M)
    return P[t, s]


def build_m(s, t, w, alpha, segs):
    """M (G, m, m) float32 of the segments [(a, b)] of one size m: row i sums its in-edges' weights in plan order (a
    stable sort of the COO by target), each add rounded; M = am1 * A off the diagonal, 1 + am1 * A on it.  None if an
    edge into a segment has its source outside it."""
    s, t = np.asarray(s, np.int64), np.asarray(t, np.int64)
    m = segs[0][1] - segs[0][0]
    base = np.array([a for a, _ in segs], np.int64)
    node_seg = np.full(int(max(t.max(initial=-1), s.max(initial=-1), base.max() + m)) + 1, -1)
    for k, (a, b) in enumerate(segs):
        node_seg[a:b] = k
    order = np.argsort(t, kind="stable")
    ss, tt = s[order], t[order]
    ww = np.ones(len(s), F32) if w is None else np.asarray(w, F32)[order]
    keep = node_seg[tt] >= 0
    ss, tt, ww = ss[keep], tt[keep], ww[keep]
    gk = node_seg[tt]
    sl, tl = ss - base[gk], tt - base[gk]
    if ((sl < 0) | (sl >= m)).any():
        return None
    first = np.concatenate([[True], tt[1:] != tt[:-1]]) if len(tt) else np.zeros(0, bool)
    start = np.maximum.accumulate(np.where(first, np.arange(len(tt)), 0)) if len(tt) else np.zeros(0, np.int64)
    rank = np.arange(len(tt)) - start
    A = np.zeros((len(segs), m, m), F32)
    for r in range(int(rank.max()) + 1 if len(rank) else 0):
        sel = rank == r                                   # the r-th edge of every row that has one
        A[gk[sel], tl[sel], sl[sel]] = A[gk[sel], tl[sel], sl[sel]] + ww[sel]
    am1 = F32(alpha) - F32(1)
    M = am1 * A
    d = np.arange(m)
    M[:, d, d] = F32(1) + am1 * A[:, d, d]
    return M


def gauss_jordan(M):
    """The entry's elimination on a batch (G, n, n) float32: (inverse, info, number of row swaps).  info[g] = k + 1 for a
    zero pivot at step k (that matrix is left as it was at that step), 0 otherwise."""
    a = np.array(M, F32, copy=True)
    G, n, _ = a.shape
    info = np.zeros(G, np.int64)
    perm = np.tile(np.arange(n), (G, 1))
    live = np.ones(G, bool)
    swaps = 0
    oth = np.arange(n)
    for k in range(n):
        col = np.abs(a[:, k:, k])
        p = k + np.argmax(np.where(np.isnan(col), F32(-1), col), axis=1)    # the first largest; a NaN never wins ...
        p = np.where(np.isnan(col[:, 0]), k, p)                              # ... unless it is at row k
        piv = a[np.arange(G), p, k]
        newly = live & (piv == 0)
        info[newly] = k + 1
        live &= ~newly
        L = np.nonzero(live)[0]
        if not len(L):
            break
        sub, pl, r = a[L], p[L], np.arange(len(L))
        swaps += int((pl != k).sum())
        rk = sub[r, k].copy()
        sub[r, k] = sub[r, pl]
        sub[r, pl] = rk
        perm[L, k] = pl
        pv = sub[r, k, k].copy()
        sub[r, k, k] = 1
        sub[r, k] = sub[r, k] / pv[:, None]
        o = oth != k
        f = sub[:, :, k].copy()
        rowk = sub[:, k, :].copy()
        sub[:, o, k] = 0
        sub[:, o, :] = sub[:, o, :] - f[:, o, None] * rowk[:, None, :]
        a[L] = sub
    g = np.nonzero(info == 0)[0]
    for k in range(n - 1, -1, -1):
        q = perm[g, k]
        tmp = a[g, :, k].copy()
        a[g, :, k] = a[g, :, q]
        a[g, :, q] = tmp
    return a, info, swaps


def ref_entry(s, t, n, w, alpha, seg_ptr, bound=BOUND):
    """gnnb_ppr_diffusion in float32: (w_out with NaN where untouched, info); None if an edge crosses segments."""
    s, t = np.asarray(s, np.int64), np.asarray(t, np.int64)
    seg_ptr = np.asarray(seg_ptr, np.int64)
    out = np.full(len(s), np.nan, F32)
    info = np.zeros(len(seg_ptr) - 1, np.int64)
    sizes = np.diff(seg_ptr)
    info[sizes > bound] = -1
    eseg = np.searchsorted(seg_ptr, t, side="right") - 1
    for m in np.unique(sizes):
        if m == 0 or m > bound:
            continue
        ids = np.nonzero(sizes == m)[0]
        M = build_m(s, t, w, alpha, [(int(seg_ptr[i]), int(seg_ptr[i + 1])) for i in ids])
        if M is None:
            return None
        inv, inf, _ = gauss_jordan(M)
        info[ids] = inf
        slot = np.full(len(sizes), -1)
        slot[ids] = np.arange(len(ids))
        e = np.nonzero((slot[eseg] >= 0))[0]
        k = slot[eseg[e]]
        ok = inf[k] == 0
        e, k = e[ok], k[ok]
        out[e] = F32(alpha) * inv[k, t[e] - seg_ptr[eseg[e]], s[e] - seg_ptr[eseg[e]]]
    return out, info


# ---------------------------------------------------------------------------------------------- the C entries in numpy
def _fake_abi():
    sys.path.insert(0, os.path.join(ROOT, "tests"))
    import fake_abi
    return fake_abi


class FakePPR:
    """gnnb_ppr_diffusion and gnnb_ppr_matrix on host pointers over the statement; every other entry is the base
    double's."""

    def __init__(self, base):
        self.base, self.fa = base, _fake_abi()
        self.n_seg_seen, self.matrices = [], []

    def __getattr__(self, name):
        return getattr(self.base, name)

    def _fail(self, code, msg):
        self.base._err = msg.encode()
        return code

    def gnnb_ppr_diffusion(self, h, w, alpha, seg_ptr, n_seg, w_out, info, stream):
        self.base.calls.append("gnnb_ppr_diffusion")
        p = self.base._p(h)
        if p.ns != p.nd:
            return self._fail(ESIZE, "needs num_src == num_dst")
        n = p.nd
        sg = np.array([0, n]) if seg_ptr is None else self.fa._arr(seg_ptr, (n_seg + 1,), np.int64).copy()
        self.n_seg_seen.append(None if seg_ptr is None else int(n_seg))
        if n == 0:
            return OK
        if sg[0] != 0 or sg[-1] != n or (np.diff(sg) < 0).any():
            return self._fail(EINVAL, "seg_ptr must hold n_seg + 1 non-decreasing offsets from 0 to n")
        res = ref_entry(p.s, p.t, n, None if w is None else self.fa._arr(w, (p.E,)), F32(alpha), sg)
        if res is None:
            return self._fail(EINVAL, "an edge crosses segments")
        o, inf = res
        self.fa._arr(info, (len(sg) - 1,), np.int32)[...] = inf
        touched = ~np.isnan(o)
        self.fa._arr(w_out, (p.E,))[touched] = o[touched]
        return OK

    def gnnb_ppr_matrix(self, h, w, alpha, a, b, ld, M_out, stream):
        self.base.calls.append("gnnb_ppr_matrix")
        p = self.base._p(h)
        self.matrices.append((a, b, ld))
        if not (0 <= a <= b <= p.nd) or ld < b - a:
            return self._fail(EINVAL, "bad [a, b) or ld")
        M = build_m(p.s, p.t, None if w is None else self.fa._arr(w, (p.E,)), F32(alpha), [(a, b)])
        if M is None:
            return self._fail(EINVAL, "an edge crosses [a, b)")
        self.fa._arr(M_out, (b - a, ld))[:, :b - a] = M[0]
        return OK


@pytest.fixture(params=["fake", pytest.param("cuda", marks=pytest.mark.gpu)])
def pb(request, gnn):
    """back end of the mirror: .dev, and .fake (the FakePPR in use, None on cuda)"""
    if request.param == "fake":
        from gnnb200 import transform
        with _fake_abi().installed() as fake:
            saved = transform.lib
            transform.lib = FakePPR(fake)
            try:
                yield SimpleNamespace(dev=torch.device("cpu"), fake=transform.lib)
            finally:
                transform.lib = saved
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


def rel_err(got, ref):
    nr = np.linalg.norm(ref)
    return float(np.linalg.norm(np.asarray(got, np.float64) - ref) / nr) if nr else float(np.linalg.norm(got))


def random_graph(rng, n, e, wlo=0.1, whi=1.0, loops=True):
    """directed, with duplicates and (unless loops=False) self loops"""
    s, t = rng.integers(0, n, e), rng.integers(0, n, e)
    if not loops:
        t = np.where(s == t, (t + 1) % n, t) if n > 1 else t
    return s, t, rng.uniform(wlo, whi, e).astype(F32)


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


def check_per_graph(got, parts, alpha=0.85, tol=1e-5):
    off = 0
    for s, t, n, w in parts:
        k = len(s)
        ref = dense_ppr(np.asarray(s, np.int64), np.asarray(t, np.int64), n, w, alpha)
        assert rel_err(got[off:off + k], ref) <= tol, n
        off += k


# ---------------------------------------------------------------------------------------------- the statement itself
def test_statement_gauss_jordan_matches_float64_inverse():
    """well-conditioned matrices whose off-diagonal entries exceed the diagonal, so that pivoting swaps rows"""
    rng = np.random.default_rng(0)
    for n in (1, 2, 7, 33, 100):
        Q = np.linalg.qr(rng.standard_normal((4, n, n)))[0]
        D = rng.uniform(1.0, 3.0, (4, n))
        M = (Q * D[:, None, :]) @ np.swapaxes(Q, 1, 2)             # condition number <= 3
        M = M[:, rng.permutation(n)].astype(F32)                    # rows out of order: the pivots are off-diagonal
        inv, info, swaps = gauss_jordan(M)
        assert (info == 0).all() and (swaps > 0 or n == 1)
        ref = np.linalg.inv(M.astype(np.float64))
        assert rel_err(inv, ref) <= 1e-5


def test_statement_pivot_rules():
    # the first of two equal candidates; a NaN below row k is never chosen; a zero column is singular at that step
    _, _, swaps = gauss_jordan(np.array([[[1.0, 2.0], [-1.0, 3.0]]], F32))
    assert swaps == 0
    inv, info, swaps = gauss_jordan(np.array([[[1.0, 0.0], [np.nan, 1.0]]], F32))
    assert swaps == 0 and info[0] == 0
    _, info, _ = gauss_jordan(np.array([[[1.0, 0.0, 0.0], [0.0, 0.0, 1.0], [0.0, 0.0, 1.0]]], F32))
    assert info[0] == 2


# ---------------------------------------------------------------------------------------------- reference tests
def test_reference_known_answer(gnn, pb):
    """GNNGraphs/test/transform.jl:614-633, compared with ≈ (rtol = sqrt(eps(Float32))) as the reference does"""
    g = gnn.GNNGraph(torch.tensor([1, 1, 2, 3], device=pb.dev), torch.tensor([2, 3, 4, 5], device=pb.dev),
                     torch.tensor([0.1, 0.2, 0.3, 0.4], device=pb.dev))
    w = npy(gnn.get_edge_weight(gnn.ppr_diffusion(g)))
    expect = np.array([0.012749999, 0.025499998, 0.038249996, 0.050999995], F32)
    assert w.dtype == np.float32 and np.allclose(w, expect, rtol=np.sqrt(np.finfo(F32).eps), atol=0)


def _cases():
    """name -> (s, t, n, w): 0-based edge lists"""
    rng = np.random.default_rng(7)
    c = {}
    c["directed_unweighted"] = (*random_graph(rng, 30, 60, loops=False)[:2], 30, None)
    c["directed_weighted"] = (*random_graph(rng, 25, 80)[:2], 25, rng.uniform(0.1, 2.0, 80).astype(F32))
    # duplicates (0 -> 1 three times), self loops (2, 3), an isolated node (5), a node whose only edge is a loop (4)
    c["duplicates_loops_isolated"] = ([0, 0, 0, 1, 2, 3, 3, 4], [1, 1, 1, 2, 2, 3, 0, 4], 6,
                                      [1.0, 2.0, 0.5, 1.5, 3.0, 0.25, 1.0, 2.0])
    c["undirected_unweighted"] = ([0, 1, 1, 2, 2, 3, 3, 0], [1, 0, 2, 1, 3, 2, 0, 3], 4, None)
    return c


CASES = _cases()


@pytest.mark.parametrize("name", list(CASES))
@pytest.mark.parametrize("alpha", [0.85, 0.3])
def test_against_dense_reference(gnn, pb, name, alpha):
    s, t, n, w = CASES[name]
    h = gnn.ppr_diffusion(graph(gnn, s, t, n, pb.dev, w), alpha=alpha)
    got = npy(gnn.get_edge_weight(h))
    assert got.shape == (len(s),) and got.dtype == np.float32
    assert rel_err(got, dense_ppr(np.asarray(s), np.asarray(t), n, w, alpha)) <= 1e-5
    seg = np.array([0, n])
    assert np.array_equal(got, ref_entry(s, t, n, w, alpha, seg)[0])


def test_isolated_self_loop_is_exact(gnn, pb):
    """a node whose only edge is a self loop of weight w gets alpha * (1 / (1 + am1 * w))"""
    g = graph(gnn, [0, 1, 2], [1, 0, 2], 3, pb.dev, [0.5, 0.25, 2.0])
    got = npy(gnn.get_edge_weight(gnn.ppr_diffusion(g, alpha=0.7)))
    am1 = F32(0.7) - F32(1)
    assert got[2] == F32(0.7) * (F32(1) / (F32(1) + am1 * F32(2.0)))


def test_alpha_one_is_identity(gnn, pb):
    s, t, n, w = CASES["duplicates_loops_isolated"]
    got = npy(gnn.get_edge_weight(gnn.ppr_diffusion(graph(gnn, s, t, n, pb.dev, w), alpha=1)))
    assert np.array_equal(got, (np.asarray(s) == np.asarray(t)).astype(F32))


def test_batch_equals_whole_graph_inverse(gnn, pb):
    parts = [CASES[k] for k in CASES]
    s, t, n, w, gi, seg = batch_of(parts)
    batched = npy(gnn.get_edge_weight(gnn.ppr_diffusion(graph(gnn, s, t, n, pb.dev, w, gi))))
    whole = npy(gnn.get_edge_weight(gnn.ppr_diffusion(graph(gnn, s, t, n, pb.dev, w))))
    assert np.array_equal(batched, whole)
    assert rel_err(batched, dense_ppr(s, t, n, w)) <= 1e-5
    check_per_graph(batched, parts)
    if pb.fake is not None:
        assert pb.fake.n_seg_seen[-2:] == [len(parts), None]


# ---------------------------------------------------------------------------------------------- bookkeeping
@pytest.mark.parametrize("route", ["smem", "dense"])
def test_singular_raises_naming_the_graph(gnn, pb, monkeypatch, route):
    """alpha = 0.5 and edges 1 -> 2, 2 -> 1 of weight 2 give M = [[1, -1], [-1, 1]]"""
    from gnnb200 import transform
    if route == "dense":
        monkeypatch.setattr(transform, "_PPR_SMEM_MAX_NODES", 1)
    parts = [([0, 1], [1, 2], 3, [0.5, 0.5]), ([0, 1], [1, 0], 2, [2.0, 2.0]), ([0], [0], 1, [1.0])]
    s, t, n, w, gi, _ = batch_of(parts)
    with pytest.raises(torch.linalg.LinAlgError, match="graph 2 .*step 2"):
        gnn.ppr_diffusion(graph(gnn, s, t, n, pb.dev, w, gi), alpha=0.5)
    with pytest.raises(torch.linalg.LinAlgError, match="the graph"):
        gnn.ppr_diffusion(graph(gnn, s, t, n, pb.dev, w), alpha=0.5)


def test_large_segments_take_the_dense_route(gnn, pb, monkeypatch):
    """a bound of 10 sends the 12- and 130-node graphs to gnnb_ppr_matrix and inv_ex (two padded sizes), the rest to
    the entry in one call"""
    from gnnb200 import transform
    monkeypatch.setattr(transform, "_PPR_SMEM_MAX_NODES", 10)
    rng = np.random.default_rng(9)
    parts = [(*random_graph(rng, n, 3 * n)[:2], n, rng.uniform(0.1, 1.0, 3 * n).astype(F32))
             for n in (4, 12, 1, 130, 9)]
    s, t, n, w, gi, seg = batch_of(parts)
    got = npy(gnn.get_edge_weight(gnn.ppr_diffusion(graph(gnn, s, t, n, pb.dev, w, gi))))
    check_per_graph(got, parts)
    if pb.fake is not None:
        assert pb.fake.n_seg_seen == [5]
        assert pb.fake.matrices == [(int(seg[1]), int(seg[2]), 128), (int(seg[3]), int(seg[4]), 256)]
    monkeypatch.setattr(transform, "_PPR_SMEM_MAX_NODES", 0)      # every segment dense
    check_per_graph(npy(gnn.get_edge_weight(gnn.ppr_diffusion(graph(gnn, s, t, n, pb.dev, w, gi)))), parts)


def test_unsorted_indicator_or_crossing_edge_is_one_segment(gnn, pb):
    rng = np.random.default_rng(5)
    parts = [(*random_graph(rng, n, 3 * n)[:2], n, None) for n in (7, 12, 9)]
    s, t, n, _, gi, _ = batch_of(parts)
    plain = npy(gnn.get_edge_weight(gnn.ppr_diffusion(graph(gnn, s, t, n, pb.dev))))
    gi_unsorted = gi.copy()
    gi_unsorted[[0, -1]] = gi_unsorted[[-1, 0]]
    assert np.array_equal(npy(gnn.get_edge_weight(gnn.ppr_diffusion(graph(gnn, s, t, n, pb.dev, gi=gi_unsorted)))),
                          plain)
    s2, t2 = np.concatenate([s, [0]]), np.concatenate([t, [n - 1]])     # an edge from graph 1 to graph 3
    cross = npy(gnn.get_edge_weight(gnn.ppr_diffusion(graph(gnn, s2, t2, n, pb.dev, gi=gi))))
    assert rel_err(cross, dense_ppr(s2, t2, n, None)) <= 1e-5
    if pb.fake is not None:
        assert pb.fake.n_seg_seen == [None, None, None]


def test_empty_and_edgeless_graphs(gnn, pb):
    e = torch.zeros(0, dtype=torch.int64, device=pb.dev)
    for n in (0, 5):
        h = gnn.ppr_diffusion(gnn.GNNGraph(e, e, num_nodes=n))
        w = gnn.get_edge_weight(h)
        assert w.shape == (0,) and w.dtype == torch.float32 and h.num_nodes == n
    if pb.fake is not None:
        assert "gnnb_ppr_diffusion" not in pb.fake.calls


def test_result_keeps_data_indicator_and_plan(gnn, pb):
    parts = [CASES["directed_weighted"], CASES["undirected_unweighted"]]
    s, t, n, w, gi, _ = batch_of(parts)
    x = torch.arange(3.0 * n, device=pb.dev).reshape(3, n)
    ea = torch.arange(2.0 * len(s), device=pb.dev).reshape(2, len(s))
    g = graph(gnn, s, t, n, pb.dev, w, gi, ndata={"x": x}, edata={"e": ea}, gdata={"u": torch.ones(1, 2)})
    wg = g.w.clone().requires_grad_(True)
    g = gnn.GNNGraph(g.s, g.t, wg, num_nodes=n, ndata=g.ndata, edata=g.edata, gdata=g.gdata, num_graphs=2,
                     graph_indicator=g.graph_indicator)
    h = gnn.ppr_diffusion(g)
    assert h._plan is g._plan and torch.equal(h.s, g.s) and torch.equal(h.t, g.t)
    assert h.num_graphs == 2 and torch.equal(h.graph_indicator, g.graph_indicator)
    for k in ("x", "e", "u"):
        d, d0 = {"x": (h.ndata, g.ndata), "e": (h.edata, g.edata), "u": (h.gdata, g.gdata)}[k]
        assert torch.equal(d[k], d0[k])
    assert not h.w.requires_grad and h.w.grad_fn is None


def test_argument_errors(gnn, pb):
    g = graph(gnn, [0, 1], [1, 0], 2, pb.dev)
    with pytest.raises(TypeError):
        gnn.ppr_diffusion(g, 0.85)                                  # alpha is a keyword, as in the reference
    with pytest.raises(TypeError):
        gnn.ppr_diffusion(g, alpha=None)
    with pytest.raises(ValueError):
        gnn.ppr_diffusion(g, alpha="high")


# ---------------------------------------------------------------------------------------------- GPU: bits and scale
def _entry(g, alpha, seg_ptr, w_out, info):
    from gnnb200 import _lib
    p = g.plan()
    _lib.check(_lib.lib.gnnb_ppr_diffusion(p.h, None if g.w is None else g.w.data_ptr(), alpha,
                                           None if seg_ptr is None else seg_ptr.data_ptr(),
                                           1 if seg_ptr is None else seg_ptr.numel() - 1, w_out.data_ptr(),
                                           info.data_ptr(), torch.cuda.current_stream().cuda_stream))


def run_entry(gnn, g, seg, alpha=0.85):
    """(w_out with NaN where untouched, info) of one call of gnnb_ppr_diffusion"""
    w_out = torch.full((g.num_edges,), float("nan"), device="cuda")
    info = torch.full((len(seg) - 1,), -7, dtype=torch.int32, device="cuda")
    _entry(g, alpha, torch.as_tensor(np.asarray(seg, np.int64), device="cuda"), w_out, info)
    return npy(w_out), npy(info).astype(np.int64)


def sized_batch(rng, sizes, wlo=0.1, whi=1.0):
    return [(*random_graph(rng, n, 3 * n)[:2], n, rng.uniform(wlo, whi, 3 * n).astype(F32)) for n in sizes]


SIZES = list(range(1, 34)) + [100, BOUND - 1, BOUND]


@pytest.mark.gpu
@pytest.mark.parametrize("whi", [1.0, 20.0])
def test_gpu_entry_equals_statement_bits(gnn, whi):
    """every size 1 .. 33, 100, 239, 240, with duplicates and self loops; whi = 20 makes off-diagonal entries larger
    than the diagonal, so the pivots swap rows"""
    rng = np.random.default_rng(11 + int(whi))
    parts = sized_batch(rng, SIZES, 0.1, whi)
    s, t, n, w, gi, seg = batch_of(parts)
    g = graph(gnn, s, t, n, "cuda", w, gi)
    got, info = run_entry(gnn, g, seg)
    ref, rinfo = ref_entry(s, t, n, w, 0.85, seg)
    assert np.array_equal(info, rinfo)
    assert np.array_equal(got, ref, equal_nan=True)
    if whi > 1:
        M = build_m(s, t, w, 0.85, [(int(seg[-2]), int(seg[-1]))])
        assert gauss_jordan(M)[2] > 0
    assert (info == 0).sum() >= len(SIZES) - 3


@pytest.mark.gpu
def test_gpu_mirror_equals_statement_and_is_deterministic(gnn):
    rng = np.random.default_rng(3)
    parts = sized_batch(rng, [5, 32, 33, 64, BOUND, 2])
    s, t, n, w, gi, seg = batch_of(parts)
    g = graph(gnn, s, t, n, "cuda", w, gi)
    h = gnn.ppr_diffusion(g)
    assert np.array_equal(npy(h.w), ref_entry(s, t, n, w, 0.85, seg)[0])
    for _ in range(3):
        assert torch.equal(h.w, gnn.ppr_diffusion(g).w)
    check_per_graph(npy(h.w), parts)


@pytest.mark.gpu
@pytest.mark.parametrize("whi", [1.0, 20.0])
def test_gpu_warp_and_cta_classes_same_bits(gnn, whi):
    """gnnb_set_kernel_variant(12) sends every segment through the CTA class"""
    from gnnb200 import _lib
    rng = np.random.default_rng(23 + int(whi))
    parts = sized_batch(rng, list(range(1, 34)) * 2, 0.1, whi)
    s, t, n, w, gi, seg = batch_of(parts)
    g = graph(gnn, s, t, n, "cuda", w, gi)
    a, ia = run_entry(gnn, g, seg)
    try:
        _lib.check(_lib.lib.gnnb_set_kernel_variant(12))
        b, ib = run_entry(gnn, g, seg)
    finally:
        _lib.check(_lib.lib.gnnb_set_kernel_variant(0))
    assert np.array_equal(ia, ib) and np.array_equal(a.view(np.uint32), b.view(np.uint32))


def well_conditioned(rng, n, deg=3):
    """about three in-edges per node of weight in [0, 1): M = I - 0.15 A is diagonally dominant in most rows"""
    s, t = rng.integers(0, n, deg * n), rng.integers(0, n, deg * n)
    return s, t, n, rng.uniform(0.0, 1.0, deg * n).astype(F32)


@pytest.mark.gpu
@pytest.mark.parametrize("n", [BOUND + 1, 1000])
def test_gpu_dense_route(gnn, n):
    rng = np.random.default_rng(n)
    parts = [well_conditioned(rng, n), well_conditioned(rng, 7), well_conditioned(rng, n)]
    s, t, N, w, gi, seg = batch_of(parts)
    for ps, pt, pn, pw in parts:
        A = np.zeros((pn, pn))
        np.add.at(A, (pt, ps), pw.astype(np.float64))
        assert np.linalg.cond(np.eye(pn) - 0.15 * A) < 10
    g = graph(gnn, s, t, N, "cuda", w, gi)
    got = npy(gnn.ppr_diffusion(g).w)
    off = 0
    for ps, pt, pn, pw in parts:
        assert rel_err(got[off:off + len(ps)], dense_ppr(ps, pt, pn, pw)) <= 1e-5
        off += len(ps)
    # gnnb_ppr_matrix is the statement's M, bit for bit, and leaves the padding alone
    from gnnb200 import _lib
    ld = n + 3
    M = torch.full((n, ld), -5.0, device="cuda")
    _lib.check(_lib.lib.gnnb_ppr_matrix(g.plan().h, g.w.data_ptr(), 0.85, int(seg[2]), int(seg[3]), ld,
                                        M.data_ptr(), torch.cuda.current_stream().cuda_stream))
    Mn = npy(M)
    assert np.array_equal(Mn[:, :n], build_m(s, t, w, 0.85, [(int(seg[2]), int(seg[3]))])[0])
    assert (Mn[:, n:] == -5.0).all()


@pytest.mark.gpu
def test_gpu_at_scale_molecules(gnn):
    """10 000 molecule-shaped graphs (23 nodes, 50 edges, bidirected) against per-graph float64"""
    rng = np.random.default_rng(13)
    G, n1 = 10_000, 23
    a = rng.integers(0, n1, (G, 25))
    b = (a + rng.integers(1, n1, (G, 25))) % n1
    off = (np.arange(G) * n1)[:, None]
    s = np.concatenate([(a + off).ravel(), (b + off).ravel()])
    t = np.concatenate([(b + off).ravel(), (a + off).ravel()])
    gi = np.repeat(np.arange(1, G + 1), n1)
    got = npy(gnn.ppr_diffusion(graph(gnn, s, t, G * n1, "cuda", gi=gi)).w).astype(np.float64)
    A = np.zeros((G, n1, n1))
    np.add.at(A, (t // n1, t % n1, s % n1), 1.0)
    P = float(F32(0.85)) * np.linalg.inv(np.eye(n1) + (float(F32(0.85)) - 1) * A)
    ref = P[t // n1, t % n1, s % n1]
    gk = t // n1
    num = np.bincount(gk, (got - ref) ** 2, minlength=G)
    den = np.bincount(gk, ref ** 2, minlength=G)
    assert np.sqrt(num / den).max() <= 1e-5


@pytest.mark.gpu
def test_gpu_singular_segment_in_the_middle(gnn):
    rng = np.random.default_rng(29)
    parts = sized_batch(rng, [5, 40]) + [([0, 1], [1, 0], 2, [2.0, 2.0])] + sized_batch(rng, [3, 50])
    s, t, n, w, gi, seg = batch_of(parts)
    g = graph(gnn, s, t, n, "cuda", w, gi)
    for variant in (0, 12):
        from gnnb200 import _lib
        try:
            _lib.check(_lib.lib.gnnb_set_kernel_variant(variant))
            got, info = run_entry(gnn, g, seg, alpha=0.5)
        finally:
            _lib.check(_lib.lib.gnnb_set_kernel_variant(0))
        assert info.tolist() == [0, 0, 2, 0, 0]
        ref, rinfo = ref_entry(s, t, n, w, 0.5, seg)
        assert rinfo.tolist() == [0, 0, 2, 0, 0]
        assert np.array_equal(got, ref, equal_nan=True)
        e0 = sum(len(p[0]) for p in parts[:2])
        assert np.isnan(got[e0:e0 + 2]).all()                   # the singular segment's weights are untouched


@pytest.mark.gpu
def test_gpu_entry_rejects_crossing_edges_and_bad_segments(gnn):
    """GNNB_EINVAL, nothing written past w_out or info"""
    GUARD = 4096
    rng = np.random.default_rng(4)
    parts = sized_batch(rng, [20, 100, 40])
    s, t, n, w, gi, seg = batch_of(parts)
    s, t = np.concatenate([s, [5, 130]]), np.concatenate([t, [50, 2]])    # small -> medium, medium -> small
    w = np.concatenate([w, [1.0, 1.0]]).astype(F32)
    g = graph(gnn, s, t, n, "cuda", w)
    E = len(s)
    for sg in ([0, 20, 120, n], [0, 120, 20, n], [0, 20, 120, n + 5], [1, 20, 120, n], [0, -4, 120, n]):
        w_out = torch.full((E + GUARD,), -7.0, device="cuda")
        info = torch.full((3 + GUARD,), -7, dtype=torch.int32, device="cuda")
        with pytest.raises(ValueError):
            _entry(g, 0.85, torch.tensor(sg, dtype=torch.int64, device="cuda"), w_out, info)
        assert bool((w_out[E:] == -7.0).all()) and bool((info[3:] == -7).all())
    w_out = torch.full((E + GUARD,), -7.0, device="cuda")            # one segment: the same graph is valid
    info = torch.full((1 + GUARD,), -7, dtype=torch.int32, device="cuda")
    _entry(g, 0.85, None, w_out, info)
    assert int(info[0]) == 0 and bool((w_out[E:] == -7.0).all()) and not bool((w_out[:E] == -7.0).any())
    from gnnb200 import _lib
    M = torch.zeros((100, 100), device="cuda")
    for a, b, ld in ((20, 120, 100), (0, n + 1, n + 1), (30, 20, 100), (20, 120, 99)):
        with pytest.raises(ValueError):
            _lib.check(_lib.lib.gnnb_ppr_matrix(g.plan().h, None, 0.85, a, b, ld, M.data_ptr(),
                                                torch.cuda.current_stream().cuda_stream))


@pytest.mark.gpu
def test_gpu_nonfinite_weights_follow_the_statement(gnn):
    rng = np.random.default_rng(31)
    parts = sized_batch(rng, [3, 9, 31, 40, 64, 17])
    for k, bad in enumerate((np.nan, np.inf, -np.inf, np.nan, np.inf, -np.inf)):
        parts[k][3][k % len(parts[k][3])] = bad
    s, t, n, w, gi, seg = batch_of(parts)
    g = graph(gnn, s, t, n, "cuda", w, gi)
    for alpha in (0.85, float("nan"), float("inf")):
        got, info = run_entry(gnn, g, seg, alpha)
        with np.errstate(invalid="ignore", divide="ignore", over="ignore"):
            ref, rinfo = ref_entry(s, t, n, w, alpha, seg)
        assert np.array_equal(info, rinfo)
        assert np.array_equal(got, ref, equal_nan=True)
    with np.errstate(invalid="ignore", divide="ignore", over="ignore"):
        ref, rinfo = ref_entry(s, t, n, w, 0.85, seg)
    assert (rinfo == 0).all()
    h = gnn.ppr_diffusion(g)                                        # the mirror raises nothing on non-finite weights
    assert np.array_equal(npy(h.w), ref, equal_nan=True)
