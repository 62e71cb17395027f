"""knn_graph / radius_graph (graphneuralnetworks.jl_b200/generate.py over csrc/knn.cu; GNNGraphs/src/generate.jl:112-222).

The contract is integer-exact: d2(i, j) = Σ_f (p_i[f] - p_j[f])² in ascending f with every fp32 operation rounded on
its own (numpy's float32 ufuncs compute exactly that), a NaN distance counts as +Inf, knn rows are the k smallest
(d2, j) keys in ascending order, radius rows every j with sqrt(d2) <= r in ascending j.  `ref_knn` / `ref_radius` below
restate it in numpy and are pinned independently against scipy's KD-tree; the kernels are compared with `==`.

Back ends of the mirror: a numpy restatement of the three C entries (`FakeGen`, swapped in over tests/fake_abi.py's
double) and, under -m gpu, the CUDA kernels.
"""
import ctypes as C
import os
import sys

import numpy as np
import pytest
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
OK, EINVAL, ESIZE, ECUDA, ENOMEM, EUNSUPPORTED = range(6)


# ---------------------------------------------------------------------------------------------- the contract in numpy
def _d2(Q, Cand):
    """(len(Q), len(C)) squared distances in Q's dtype, ascending f, each op rounded on its own; NaN -> +Inf"""
    acc = np.zeros((len(Q), len(Cand)), dtype=Q.dtype)
    for f in range(Q.shape[1]):
        acc = acc + np.square(Q[:, f][:, None] - Cand[:, f][None, :])
    return np.where(np.isnan(acc), np.inf, acc).astype(Q.dtype)


def _segs(n, seg_ptr):
    return np.array([0, n], np.int64) if seg_ptr is None else np.asarray(seg_ptr, np.int64)


def ref_knn(P, k, seg_ptr=None, self_loops=False, queries=None, chunk=256):
    """rows (len(queries), k) of 0-based neighbour ids.  float32: packed uint64 keys; float64: per-row lexsort."""
    n = len(P)
    seg = _segs(n, seg_ptr)
    queries = np.arange(n) if queries is None else np.asarray(queries, np.int64)
    out = np.empty((len(queries), k), np.int64)
    sid = np.searchsorted(seg, queries, side="right") - 1
    for s in np.unique(sid):
        lo, hi = int(seg[s]), int(seg[s + 1])
        pos = np.nonzero(sid == s)[0]
        step = max(1, min(chunk, 2 ** 24 // max(hi - lo, 1)))
        for c0 in range(0, len(pos), step):
            pp = pos[c0:c0 + step]
            q = queries[pp]
            d2 = _d2(P[q], P[lo:hi])
            j = np.arange(lo, hi)
            if P.dtype == np.float32:
                key = ((d2.view(np.uint32).astype(np.uint64) + 1) << np.uint64(32)) | j.astype(np.uint64)[None, :]
                if not self_loops:
                    key[np.arange(len(q)), q - lo] = np.iinfo(np.uint64).max
                part = np.partition(key, k - 1, axis=1)[:, :k]
                out[pp] = (np.sort(part, axis=1) & np.uint64(0xFFFFFFFF)).astype(np.int64)
            else:
                for r, i in enumerate(q):
                    keep = j != i if not self_loops else np.ones(len(j), bool)
                    order = np.lexsort((j[keep], d2[r][keep]))
                    out[pp[r]] = j[keep][order[:k]]
    return out


def ref_radius(P, r, seg_ptr=None, self_loops=False, queries=None, chunk=256):
    """(offsets, flat 0-based ids) of the rows of `queries`"""
    n = len(P)
    seg = _segs(n, seg_ptr)
    queries = np.arange(n) if queries is None else np.asarray(queries, np.int64)
    rows_ = [None] * len(queries)
    sid = np.searchsorted(seg, queries, side="right") - 1
    rr = P.dtype.type(r)
    for s in np.unique(sid):
        lo, hi = int(seg[s]), int(seg[s + 1])
        pos = np.nonzero(sid == s)[0]
        step = max(1, min(chunk, 2 ** 24 // max(hi - lo, 1)))
        for c0 in range(0, len(pos), step):
            pp = pos[c0:c0 + step]
            q = queries[pp]
            hit = np.sqrt(_d2(P[q], P[lo:hi])) <= rr
            if not self_loops:
                hit[np.arange(len(q)), q - lo] = False
            for a, b in enumerate(pp):
                rows_[b] = np.nonzero(hit[a])[0] + lo
    off = np.zeros(len(queries) + 1, np.int64)
    off[1:] = np.cumsum([len(x) for x in rows_])
    flat = np.concatenate(rows_).astype(np.int64) if len(rows_) else np.empty(0, np.int64)
    return off, flat


# ---------------------------------------------------------------------------------------------- the C entries in numpy
def _fake_abi():
    sys.path.insert(0, os.path.join(ROOT, "tests"))
    import fake_abi
    return fake_abi


class FakeGen:
    """gnnb_knn / gnnb_radius_count / gnnb_radius_fill on host pointers, one query at a time with Python's sort on
    (d2, j): a second, loop-shaped statement of the contract."""

    def __init__(self, base):
        self.base, self.fa = base, _fake_abi()

    def _fail(self, code, msg):
        self.base._err = msg.encode()
        return code

    def _setup(self, points, n, d, seg_ptr, n_seg):
        if n < 0 or n >= 2 ** 31:
            return self._fail(ESIZE, "n outside [0, 2^31)"), None, None
        if d < 1:
            return self._fail(EINVAL, "d must be >= 1"), None, None
        if d > 256:
            return self._fail(EUNSUPPORTED, "d > 256"), None, None
        P = self.fa._arr(points, (n, d), np.float32)
        seg = np.array([0, n], np.int64) if seg_ptr is None else self.fa._arr(seg_ptr, (n_seg + 1,), np.int64).copy()
        if seg[0] != 0 or seg[-1] != n or (np.diff(seg) < 0).any():
            return self._fail(EINVAL, "bad seg_ptr"), None, None
        return OK, P, seg

    def _cands(self, P, seg, i, self_loops):
        s = np.searchsorted(seg, i, side="right") - 1
        j = np.arange(seg[s], seg[s + 1])
        if not self_loops:
            j = j[j != i]
        acc = np.zeros(len(j), np.float32)
        for f in range(P.shape[1]):
            acc = acc + np.square(P[j, f] - P[i, f])
        return j, acc

    def gnnb_knn(self, points, n, d, seg_ptr, n_seg, k, self_loops, nbr, stream):
        rc, P, seg = self._setup(points, n, d, seg_ptr, n_seg)
        if rc:
            return rc
        if k < 1:
            return self._fail(EINVAL, "k must be >= 1")
        if k > 64:
            return self._fail(EUNSUPPORTED, "k > 64")
        if n == 0:
            return OK
        lens = np.diff(seg)
        if ((lens > 0) & (lens < k + (0 if self_loops else 1))).any():
            return self._fail(ESIZE, "a segment has fewer than k (+1) points")
        out = self.fa._arr(nbr, (n, k), np.int32)
        for i in range(n):
            j, acc = self._cands(P, seg, i, self_loops)
            best = sorted(zip((float("inf") if np.isnan(a) else float(a) for a in acc), j.tolist()))[:k]
            out[i] = [b for _, b in best]
        return OK

    def gnnb_radius_count(self, points, n, d, seg_ptr, n_seg, r, self_loops, offsets, total, stream):
        if np.isnan(r) or r < 0:
            return self._fail(EINVAL, "bad r")
        rc, P, seg = self._setup(points, n, d, seg_ptr, n_seg)
        if rc:
            return rc
        off = self.fa._arr(offsets, (n + 1,), np.int64)
        off[0] = 0
        for i in range(n):
            j, acc = self._cands(P, seg, i, self_loops)
            off[i + 1] = off[i] + int((np.sqrt(np.where(np.isnan(acc), np.inf, acc)) <= np.float32(r)).sum())
        self.fa._deref(total).value = int(off[n])
        return OK

    def gnnb_radius_fill(self, points, n, d, seg_ptr, n_seg, r, self_loops, offsets, nbr, capacity, stream):
        if np.isnan(r) or r < 0:
            return self._fail(EINVAL, "bad r")
        rc, P, seg = self._setup(points, n, d, seg_ptr, n_seg)
        if rc:
            return rc
        off = self.fa._arr(offsets, (n + 1,), np.int64)
        if capacity < off[n]:
            return self._fail(ESIZE, "nbr too small")
        out = self.fa._arr(nbr, (int(off[n]),), np.int32)
        for i in range(n):
            j, acc = self._cands(P, seg, i, self_loops)
            out[off[i]:off[i + 1]] = j[np.sqrt(np.where(np.isnan(acc), np.inf, acc)) <= np.float32(r)]
        return OK


@pytest.fixture(params=["fake", pytest.param("cuda", marks=pytest.mark.gpu)])
def gb(request, monkeypatch, gnn):
    """back end of the mirror: the numpy entries above (host tensors) or the CUDA kernels (device tensors)"""
    if request.param == "fake":
        from gnnb200 import generate
        with _fake_abi().installed() as fake:
            monkeypatch.setattr(generate, "lib", FakeGen(fake))
            yield torch.device("cpu")
    else:
        if not torch.cuda.is_available():
            pytest.skip("no CUDA device")
        yield torch.device("cuda")


def jl(points_rows, dev):
    """(n, d) rows -> the (d, n) Julia-layout matrix the generators take"""
    return torch.as_tensor(np.ascontiguousarray(points_rows)).to(dev).t()


def st(g):
    return g.s.cpu().numpy(), g.t.cpu().numpy()


def rows_of(g, n, dir="in"):
    """centre -> list of neighbours (1-based), in edge order"""
    s, t = st(g)
    centre, nb = (t, s) if dir == "in" else (s, t)
    assert (np.diff(centre) >= 0).all(), "edges are grouped by centre"
    return {c: nb[centre == c].tolist() for c in range(1, n + 1)}


# ---------------------------------------------------------------------------------------------- reference tests
def test_reference_knn_graph(gnn, gb):
    """GNNGraphs/test/generate.jl:39-63"""
    rng = np.random.default_rng(0)
    n, k = 10, 3
    x = rng.random((n, 3))
    g = gnn.knn_graph(jl(x, gb), k)
    s, t = st(g)
    assert g.num_nodes == 10 and g.num_edges == n * k
    assert (np.bincount(t, minlength=n + 1)[1:] == k).all()
    assert not (s == t).any()
    g = gnn.knn_graph(jl(x, gb), k, dir="out", self_loops=True)
    s, t = st(g)
    assert g.num_nodes == 10 and g.num_edges == n * k
    assert (np.bincount(s, minlength=n + 1)[1:] == k).all()
    assert (s == t).any()
    gi = [1, 1, 1, 1, 1, 2, 2, 2, 2, 2]
    g = gnn.knn_graph(jl(x, gb), k, graph_indicator=gi)
    assert g.num_graphs == 2
    s, t = st(g)
    ne = n * k // 2
    assert ((1 <= s[:ne]) & (s[:ne] <= 5)).all() and ((1 <= t[:ne]) & (t[:ne] <= 5)).all()
    assert ((6 <= s[ne:]) & (s[ne:] <= 10)).all() and ((6 <= t[ne:]) & (t[ne:] <= 10)).all()


def test_reference_radius_graph(gnn, gb):
    """GNNGraphs/test/generate.jl:65-81"""
    rng = np.random.default_rng(1)
    n, r = 10, 0.5
    x = rng.random((n, 3))
    g = gnn.radius_graph(jl(x, gb), r)
    s, t = st(g)
    assert g.num_nodes == 10 and not (s == t).any()
    g = gnn.radius_graph(jl(x, gb), r, dir="out", self_loops=True)
    s, t = st(g)
    assert g.num_nodes == 10 and (s == t).any()
    g = gnn.radius_graph(jl(x, gb), r, graph_indicator=[1, 1, 1, 1, 1, 2, 2, 2, 2, 2])
    assert g.num_graphs == 2
    s, t = st(g)
    assert ((s > 5) == (t > 5)).all()


# ---------------------------------------------------------------------------------------------- known answers
def test_tie_rule_on_a_line(gnn, gb):
    x = np.arange(5, dtype=np.float32)[:, None]             # nodes 1..5 at 0..4
    rows = rows_of(gnn.knn_graph(jl(x, gb), 2), 5)
    assert rows[3] == [2, 4]                                # both at distance 1: the smaller id first
    assert rows[1] == [2, 3] and rows[5] == [4, 3]


def test_lattice(gnn, gb):
    """3x3 integer lattice, node id = 3*row + col + 1: every distance class is a tie"""
    x = np.array([(r, c) for r in range(3) for c in range(3)], dtype=np.float32)
    rows = rows_of(gnn.knn_graph(jl(x, gb), 4), 9)
    assert rows[5] == [2, 4, 6, 8]                          # centre: its four axis neighbours, by id
    assert rows[1] == [2, 4, 5, 3]                          # corner: d2 = 1, 1, 2, then 4 (3 before 7)
    assert rows[2] == [1, 3, 5, 4]                          # edge midpoint: 1, 1, 1, then 2 (4 before 6)
    rows = rows_of(gnn.knn_graph(jl(x, gb), 4, self_loops=True), 9)
    assert rows[5] == [5, 2, 4, 6]
    rad = rows_of(gnn.radius_graph(jl(x, gb), 1.0), 9)
    assert rad[5] == [2, 4, 6, 8] and rad[1] == [2, 4]


def test_duplicate_points(gnn, gb):
    x = np.array([[0.0], [0.0], [0.0], [5.0]], dtype=np.float32)
    rows = rows_of(gnn.knn_graph(jl(x, gb), 2), 4)
    assert rows == {1: [2, 3], 2: [1, 3], 3: [1, 2], 4: [1, 2]}   # exactly k each, the node itself never
    rows = rows_of(gnn.knn_graph(jl(x, gb), 2, self_loops=True), 4)
    assert rows == {1: [1, 2], 2: [1, 2], 3: [1, 2], 4: [4, 1]}
    rad = rows_of(gnn.radius_graph(jl(x, gb), 0.0), 4)
    assert rad == {1: [2, 3], 2: [1, 3], 3: [1, 2], 4: []}


def test_nan_row(gnn, gb):
    x = np.array([[0.0], [np.nan], [1.0], [3.0]], dtype=np.float32)
    rows = rows_of(gnn.knn_graph(jl(x, gb), 3), 4)
    assert rows[1] == [3, 4, 2]                             # the NaN point is the farthest of all
    assert rows[2] == [1, 3, 4]                             # from the NaN point everything is +Inf: id order
    rad = rows_of(gnn.radius_graph(jl(x, gb), 10.0), 4)
    assert rad == {1: [3, 4], 2: [], 3: [1, 4], 4: [1, 3]}


# ---------------------------------------------------------------------------------------------- the oracle, pinned
def test_oracle_against_kdtree():
    spatial = pytest.importorskip("scipy.spatial")
    rng = np.random.default_rng(2)
    P = rng.random((400, 3))
    k, r = 7, 0.12
    tree = spatial.cKDTree(P)
    _, idx = tree.query(P, k + 1)
    mine = ref_knn(P, k)
    for i in range(len(P)):
        assert idx[i, 0] == i and set(idx[i, 1:]) == set(mine[i])
    off, flat = ref_radius(P, r)
    balls = tree.query_ball_point(P, r)
    for i in range(len(P)):
        assert set(balls[i]) - {i} == set(flat[off[i]:off[i + 1]].tolist())
    # the float32 statement agrees where no near-tie can flip the rounding
    P32 = P.astype(np.float32)
    assert (ref_knn(P32, k) == mine).mean() > 0.99


def test_fake_entries_match_oracle():
    rng = np.random.default_rng(3)
    P = rng.random((150, 5)).astype(np.float32)
    P[::17] = P[1::17][: len(P[::17])]                      # duplicates
    seg = np.array([0, 40, 40, 95, 150], np.int64)
    fg = FakeGen(_fake_abi().FakeLib())
    for self_loops in (0, 1):
        for k in (1, 4, 9):
            nbr = np.empty((150, k), np.int32)
            assert fg.gnnb_knn(P.ctypes.data, 150, 5, seg.ctypes.data, 4, k, self_loops, nbr.ctypes.data, 0) == OK
            assert (nbr == ref_knn(P, k, seg, self_loops)).all()
        off = np.empty(151, np.int64)
        tot = C.c_int64(0)
        assert fg.gnnb_radius_count(P.ctypes.data, 150, 5, seg.ctypes.data, 4, 0.5, self_loops, off.ctypes.data,
                                    C.byref(tot), 0) == OK
        flat = np.empty(tot.value, np.int32)
        assert fg.gnnb_radius_fill(P.ctypes.data, 150, 5, seg.ctypes.data, 4, 0.5, self_loops, off.ctypes.data,
                                   flat.ctypes.data, tot.value, 0) == OK
        roff, rflat = ref_radius(P, 0.5, seg, self_loops)
        assert (off == roff).all() and (flat == rflat).all()


# ---------------------------------------------------------------------------------------------- mirror logic
def _coo(g):
    return np.stack(st(g))


@pytest.mark.parametrize("fn", ["knn", "radius"])
def test_unsorted_indicator(gnn, gb, fn):
    rng = np.random.default_rng(4)
    n = 60
    x = rng.random((n, 3)).astype(np.float32)
    gi = rng.integers(1, 4, n)
    gi[:3] = [3, 1, 2]
    make = (lambda pts, ind: gnn.knn_graph(pts, 4, graph_indicator=ind)) if fn == "knn" else \
        (lambda pts, ind: gnn.radius_graph(pts, 0.3, graph_indicator=ind))
    g = make(jl(x, gb), torch.as_tensor(gi))
    assert g.num_graphs == 3
    assert (np.asarray(g.graph_indicator) == gi).all()
    order = np.argsort(gi, kind="stable")                   # the sorted problem ...
    gs = make(jl(x[order], gb), torch.as_tensor(gi[order]))
    inv = np.empty(n, np.int64)
    inv[order] = np.arange(n)
    rows_u, rows_s = rows_of(g, n), rows_of(gs, n)
    for c in range(1, n + 1):                               # ... mapped back is the same graph, row by row
        assert rows_u[c] == [order[v - 1] + 1 for v in rows_s[inv[c - 1] + 1]]
    s, t = st(g)
    assert (gi[s - 1] == gi[t - 1]).all()


def test_num_graphs_and_kws(gnn, gb):
    rng = np.random.default_rng(5)
    x = rng.random((12, 2)).astype(np.float32)
    gi = np.array([1] * 4 + [2] * 4 + [4] * 4)             # graph 3 is empty: num_graphs = max(indicator)
    feat = torch.arange(12.0)[None, :]
    g = gnn.knn_graph(jl(x, gb), 2, graph_indicator=gi, ndata={"x": feat}, gdata={"u": torch.ones(1, 4)})
    assert g.num_graphs == 4 and g.ndata["x"] is feat and g.gdata["u"].shape == (1, 4)
    g = gnn.radius_graph(jl(x, gb), 0.4, edata=None, ndata=feat)
    assert g.num_graphs == 1 and g.x is feat
    g = gnn.knn_graph(jl(x, gb), 2)
    ew = torch.arange(float(g.num_edges))[None, :]
    g2 = gnn.knn_graph(jl(x, gb), 2, edata={"e": ew})
    assert g2.e is ew and (_coo(g2) == _coo(g)).all()


def test_errors(gnn, gb):
    x = jl(np.random.default_rng(6).random((6, 3)).astype(np.float32), gb)
    with pytest.raises(AssertionError):
        gnn.knn_graph(x, 6)                                 # 6 points: k + 1 = 7 needed without self loops
    gnn.knn_graph(x, 6, self_loops=True)
    with pytest.raises(AssertionError):
        gnn.knn_graph(x, 3, graph_indicator=[1, 1, 1, 2, 2, 2])     # a graph of exactly k nodes
    with pytest.raises(AssertionError):
        gnn.knn_graph(x, 2, graph_indicator=[1, 1, 2])
    with pytest.raises(AssertionError):
        gnn.radius_graph(x, 0.5, graph_indicator=[1, 1, 2])
    with pytest.raises(AssertionError):
        gnn.knn_graph(x, 2, dir="both")
    with pytest.raises(AssertionError):
        gnn.radius_graph(x, 0.5, dir="both")
    with pytest.raises(ValueError):
        gnn.knn_graph(x, 0)
    with pytest.raises(ValueError):
        gnn.knn_graph(x[:0], 1)                             # d = 0
    with pytest.raises(ValueError):
        gnn.radius_graph(x, float("nan"))
    with pytest.raises(ValueError):
        gnn.radius_graph(x, -1.0)
    with pytest.raises(gnn.GNNBError):
        gnn.knn_graph(jl(np.random.default_rng(7).random((80, 3)), gb), 65)
    with pytest.raises(gnn.GNNBError):
        gnn.knn_graph(torch.zeros(257, 4, device=gb), 1)


# ---------------------------------------------------------------------------------------------- kernels against the oracle
def dev_knn(P, k, seg=None, self_loops=False, shift=0):
    """gnnb_knn on a device copy of P that starts `shift` floats into its allocation"""
    from gnnb200 import _lib
    n, d = P.shape
    buf = torch.zeros(n * d + shift, dtype=torch.float32, device="cuda")
    buf[shift:] = torch.as_tensor(P).reshape(-1).cuda()
    x = buf[shift:]
    sp = None if seg is None else torch.as_tensor(np.asarray(seg, np.int64)).cuda()
    nbr = torch.empty((n, k), dtype=torch.int32, device="cuda")
    _lib.check(_lib.lib.gnnb_knn(x.data_ptr(), n, d, None if sp is None else sp.data_ptr(),
                                 1 if sp is None else sp.numel() - 1, k, int(self_loops), nbr.data_ptr(),
                                 torch.cuda.current_stream().cuda_stream))
    return nbr


def dev_radius(P, r, seg=None, self_loops=False):
    from gnnb200 import _lib
    x = torch.as_tensor(P).cuda().contiguous()
    n, d = x.shape
    sp = None if seg is None else torch.as_tensor(np.asarray(seg, np.int64)).cuda()
    args = (x.data_ptr(), n, d, None if sp is None else sp.data_ptr(), 1 if sp is None else sp.numel() - 1, float(r),
            int(self_loops))
    off = torch.empty(n + 1, dtype=torch.int64, device="cuda")
    tot = C.c_int64(0)
    strm = torch.cuda.current_stream().cuda_stream
    _lib.check(_lib.lib.gnnb_radius_count(*args, off.data_ptr(), C.byref(tot), strm))
    flat = torch.empty(max(tot.value, 1), dtype=torch.int32, device="cuda")
    _lib.check(_lib.lib.gnnb_radius_fill(*args, off.data_ptr(), flat.data_ptr(), tot.value, strm))
    return off, flat[:tot.value]


def check_knn(P, k, seg=None, self_loops=False):
    got = dev_knn(P, k, seg, self_loops).cpu().numpy()
    assert (got == ref_knn(P, k, seg, self_loops)).all()


def check_radius(P, r, seg=None, self_loops=False):
    off, flat = dev_radius(P, r, seg, self_loops)
    roff, rflat = ref_radius(P, r, seg, self_loops)
    assert (off.cpu().numpy() == roff).all()
    assert (flat.cpu().numpy() == rflat).all()


@pytest.mark.gpu
@pytest.mark.parametrize("d", [1, 2, 3, 4, 7, 16, 64, 129, 256])
def test_kernel_sweep(d):
    rng = np.random.default_rng(d)
    P = rng.random((230, d)).astype(np.float32)
    seg = [0, 97, 230]
    for self_loops in (False, True):
        for k in (1, 2, 8, 16, 31, 32, 33, 64):
            check_knn(P, k, seg, self_loops)
        r = np.float32(np.sqrt(d / 6.0) * 0.8)              # around the median distance of uniform points
        check_radius(P, r, seg, self_loops)


def _tiles(d):
    """query tile and candidate tile of csrc/knn.cu for dimension d"""
    return (128 if d <= 64 else 64), max(1, 4096 // d)


@pytest.mark.gpu
@pytest.mark.parametrize("d", [3, 64, 129])
def test_kernel_segment_layouts(d):
    rng = np.random.default_rng(10 + d)
    qt, ct = _tiles(d)
    sizes = [17]                                            # segments of exactly k + 1 points
    for m in (qt, ct):
        sizes += [m - 1, m, m + 1, 2 * m + 1]
    sizes += [17, 0, 40]
    seg = np.concatenate([[0], np.cumsum(sizes)])
    P = rng.random((int(seg[-1]), d)).astype(np.float32)
    check_knn(P, 16, seg, False)
    check_knn(P, 17, seg[[0, -1]], True)
    check_knn(P, 5, None, False)                            # one segment
    check_radius(P, np.float32(np.sqrt(d / 6.0) * 0.6), seg, False)
    for shift in (1, 2, 3):                                 # rows that start off the 16 B grid of the allocation
        got = dev_knn(P, 16, seg, False, shift).cpu().numpy()
        assert (got == ref_knn(P, 16, seg, False)).all()


@pytest.mark.gpu
def test_kernel_many_segments():
    rng = np.random.default_rng(11)
    P = rng.random((1024 * 1000, 3)).astype(np.float32)
    seg = np.arange(1025, dtype=np.int64) * 1000
    got = dev_knn(P, 16, seg).cpu().numpy()
    for s in rng.choice(1024, 48, replace=False):
        q = np.arange(seg[s], seg[s + 1])
        assert (got[q] == ref_knn(P, 16, seg, queries=q)).all()
    owner = np.arange(len(P)) // 1000
    assert (got // 1000 == owner[:, None]).all() and (got != np.arange(len(P))[:, None]).all()


@pytest.mark.gpu
@pytest.mark.parametrize("kind", ["uniform", "lattice", "duplicates", "nan"])
def test_kernel_point_sets(kind):
    rng = np.random.default_rng(12)
    if kind == "uniform":
        P = rng.random((600, 3))
    elif kind == "lattice":
        P = np.array([(a, b, c) for a in range(8) for b in range(8) for c in range(9)], dtype=np.float64)
    elif kind == "duplicates":
        P = rng.integers(0, 4, (600, 3)).astype(np.float64)
    else:
        P = rng.random((600, 3))
        P[[5, 77, 300]] = np.nan
        P[400, 1] = np.nan
    P = P.astype(np.float32)
    seg = [0, 250, len(P)]
    for self_loops in (False, True):
        for k in (1, 8, 27, 64):
            check_knn(P, k, seg, self_loops)
        check_radius(P, 1.5 if kind in ("lattice", "duplicates") else 0.2, seg, self_loops)


@pytest.mark.gpu
def test_kernel_at_scale_and_deterministic():
    rng = np.random.default_rng(13)
    n, k = 2 ** 18, 16
    P = rng.random((n, 3)).astype(np.float32)
    nbr = dev_knn(P, k)
    again = dev_knn(P, k)
    assert torch.equal(nbr, again)
    srt = torch.sort(nbr.long(), dim=1).values
    assert (srt[:, 1:] != srt[:, :-1]).all()                # k distinct ids
    assert (nbr.long() != torch.arange(n, device="cuda")[:, None]).all()
    assert int(nbr.min()) >= 0 and int(nbr.max()) < n
    q = rng.choice(n, 2000, replace=False)
    assert (nbr.cpu().numpy()[q] == ref_knn(P, k, queries=q)).all()


@pytest.mark.gpu
def test_radius_at_scale_symmetric():
    rng = np.random.default_rng(14)
    n = 2 ** 18
    P = rng.random((n, 3)).astype(np.float32)
    off, flat = dev_radius(P, 0.031)
    off2, flat2 = dev_radius(P, 0.031)
    assert torch.equal(off, off2) and torch.equal(flat, flat2)
    centre = torch.arange(n, device="cuda").repeat_interleave(off[1:] - off[:-1])
    nb = flat.long()
    a = torch.sort(centre * n + nb).values
    b = torch.sort(nb * n + centre).values
    assert torch.equal(a, b)
    q = rng.choice(n, 2000, replace=False)
    roff, rflat = ref_radius(P, 0.031, queries=q)
    offc, flatc = off.cpu().numpy(), flat.cpu().numpy()
    for a_, i in enumerate(q):
        assert (flatc[offc[i]:offc[i + 1]] == rflat[roff[a_]:roff[a_ + 1]]).all()


@pytest.mark.gpu
def test_edge_conv_on_device_knn_graph(gnn):
    rng = np.random.default_rng(15)
    n, din, dout, k = 3000, 6, 8, 12
    P = rng.standard_normal((n, din)).astype(np.float32)
    gi = np.repeat([1, 2, 3], [1000, 1200, 800])
    g = gnn.knn_graph(jl(P, "cuda"), k, graph_indicator=gi)
    nbr = ref_knn(P, k, np.array([0, 1000, 2200, 3000]))
    s_ref = torch.as_tensor(nbr.reshape(-1) + 1)
    t_ref = torch.arange(1, n + 1).repeat_interleave(k)
    assert torch.equal(g.s.cpu(), s_ref) and torch.equal(g.t.cpu(), t_ref)
    g_ref = gnn.GNNGraph(s_ref.cuda(), t_ref.cuda(), num_nodes=n)
    torch.manual_seed(0)
    nn = gnn.layers._DenseAct(2 * din, dout, torch.relu, device="cuda")
    layer = gnn.EdgeConv(nn, aggr=max)
    x = jl(P, "cuda")
    with torch.no_grad():
        assert torch.equal(layer(g, x), layer(g_ref, x))
