"""rand_temporal_radius_graph / rand_temporal_hyperbolic_graph (graphneuralnetworks.jl_b200/generate.py over
csrc/tgen.cu and csrc/knn.cu; GNNGraphs/src/generate.jl:265-380) and add_snapshot / remove_snapshot
(temporal.py; GNNGraphs/src/temporalsnapshotsgnngraph.jl:132-145, 192-201).

The contract is stated below in numpy:
- the stream u(i, τ, k) = (splitmix64(K + c) >> 11) 2^-53, K = splitmix64(seed), c = ((τ n + i) << 1) | k;
- the node dynamics, the reference's arithmetic in float64 (numpy rounds every operation on its own, so the positions
  differ from the kernel's only by the cos / sin / acosh / cosh / sinh implementations);
- the hyperbolic pair test x = C_i C_j - (S_i S_j)(c_i c_j + s_i s_j) <= cosh(ζR) or equal records, which numpy computes
  with the kernel's bits.  The radius rows are test_generate.py's `ref_radius`.
Edges are compared with `==` against these statements evaluated on the device's own points / records.

Back ends of the mirror: `FakeTGen`, the four new entries restated on host pointers over that statement (on top of
test_generate.py's FakeGen for the radius entries), and, under -m gpu, the CUDA kernels.
"""
import ctypes as C
import math

import numpy as np
import pytest
import torch

from test_generate import EINVAL, ESIZE, OK, FakeGen, _fake_abi, jl, ref_radius

U = np.uint64
MASK = 2 ** 64 - 1
TWO_PI = 2.0 * math.pi


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


def draws(seed, n, tau, k):
    """u(i, τ, k) for i = 0 .. n-1"""
    K = np.full(n, smix_int(seed & MASK), np.uint64)
    c = ((U(tau * n) + np.arange(n, dtype=np.uint64)) << U(1)) | U(k)
    return (smix(K + c) >> U(11)).astype(np.float64) * 2.0 ** -53


def ref_points(n, T, speed, seed):
    """(T, n, 2) float64 positions, generate.jl:274-282"""
    x, y = draws(seed, n, 0, 0), draws(seed, n, 0, 1)
    out = np.empty((T, n, 2))
    for t in range(T):
        if t > 0:
            rho = (2 * speed) * draws(seed, n, t, 0) - speed
            th = TWO_PI * draws(seed, n, t, 1)
            x = 1 - np.abs(1 - np.abs(x + rho * np.cos(th)))
            y = 1 - np.abs(1 - np.abs(y + rho * np.sin(th)))
        out[t, :, 0], out[t, :, 1] = x, y
    return out


def ref_records(n, T, alpha, R, speed, zeta, seed, quirks=None):
    """(T, n, 4) float64 records (cosh ζr, sinh ζr, cos θ, sin θ), generate.jl:360-377.  `quirks` (a dict) counts the
    folds: p > 1, p < 0, and p > 1 after both (a node outside the disk)."""
    cm1 = math.cosh(alpha * R) - 1
    p, th = draws(seed, n, 0, 0), TWO_PI * draws(seed, n, 0, 1)
    out = np.empty((T, n, 4))
    q = quirks if quirks is not None else {}
    for t in range(T):
        if t > 0:
            p = p + ((2 * speed) * draws(seed, n, t, 0) - speed)
            gt = p > 1
            p[gt] = 1 - np.fmod(p[gt], 1)
            lt = p < 0
            p[lt] = np.abs(p[lt])
            th = th + ((2 * speed) * draws(seed, n, t, 1) - speed)
            q["gt1"] = q.get("gt1", 0) + int(gt.sum())
            q["lt0"] = q.get("lt0", 0) + int(lt.sum())
            q["outside"] = q.get("outside", 0) + int((p > 1).sum())
        zr = zeta * ((1 / alpha) * np.arccosh(1 + cm1 * p))
        out[t] = np.stack([np.cosh(zr), np.sinh(zr), np.cos(th), np.sin(th)], 1)
    return out


def hyper_hits(Q, Cand, x_max):
    """(len(Q), len(Cand)) edge test of the records: x <= x_max (each operation rounded on its own) or equal records"""
    ang = Q[:, 2:3] * Cand[None, :, 2] + Q[:, 3:4] * Cand[None, :, 3]
    x = Q[:, 0:1] * Cand[None, :, 0] - (Q[:, 1:2] * Cand[None, :, 1]) * ang
    return (x <= x_max) | (Q[:, None, :] == Cand[None, :, :]).all(-1)


def ref_hyper_rows(rec, x_max, self_loop=False, queries=None, chunk=512):
    """(offsets, flat 0-based ids) of the rows of `queries` of one snapshot's records"""
    n = len(rec)
    queries = np.arange(n) if queries is None else np.asarray(queries, np.int64)
    rows_ = []
    for c0 in range(0, len(queries), chunk):
        q = queries[c0:c0 + chunk]
        hit = hyper_hits(rec[q], rec, x_max)
        if not self_loop:
            hit[np.arange(len(q)), q] = False
        rows_ += [np.nonzero(h)[0] for h in hit]
    off = np.zeros(len(queries) + 1, np.int64)
    off[1:] = np.cumsum([len(x) for x in rows_])
    return off, (np.concatenate(rows_) if rows_ else np.empty(0, np.int64)).astype(np.int64)


# ---------------------------------------------------------------------------------------------- the C entries in numpy
class FakeTGen(FakeGen):
    """The four temporal entries on host pointers, over the statement above, beside FakeGen's radius entries."""

    def _sizes(self, n, T, out):
        if n < 0 or T < 0:
            return self._fail(EINVAL, "n, T must be >= 0")
        if n * T >= 2 ** 31:
            return self._fail(ESIZE, "T * n must be < 2^31")
        return OK

    def gnnb_temporal_radius_points(self, n, T, speed, seed, pts, stream):
        rc = self._sizes(n, T, pts)
        if rc or n * T == 0:
            return rc
        if not math.isfinite(speed):
            return self._fail(EINVAL, "speed is not finite")
        self.fa._arr(pts, (T * n, 2), np.float32)[...] = ref_points(n, T, speed, seed).reshape(T * n, 2)
        return OK

    def gnnb_temporal_hyperbolic_records(self, n, T, alpha, R, speed, zeta, seed, rec, stream):
        rc = self._sizes(n, T, rec)
        if rc:
            return rc
        if not (alpha > 0 and R >= 0 and zeta > 0 and all(map(math.isfinite, (alpha, R, speed, zeta)))):
            return self._fail(EINVAL, "bad α, R, ζ or speed")
        if n * T:
            self.fa._arr(rec, (T * n, 4), np.float64)[...] = \
                ref_records(n, T, alpha, R, speed, zeta, seed).reshape(T * n, 4)
        return OK

    def _hyper(self, rec, n, seg_ptr, n_seg, x_max, self_loop):
        rc, _, seg = self._setup(rec, n, 8, seg_ptr, n_seg)
        if rc:
            return rc, None
        R = self.fa._arr(rec, (n, 4), np.float64)
        rows_ = []
        for s in range(len(seg) - 1):
            a, b = int(seg[s]), int(seg[s + 1])
            off, flat = ref_hyper_rows(R[a:b], x_max, self_loop)
            rows_ += [flat[off[i]:off[i + 1]] + a for i in range(b - a)]
        return OK, rows_

    def gnnb_hyperbolic_count(self, rec, n, seg_ptr, n_seg, x_max, self_loop, offsets, total, stream):
        if np.isnan(x_max):
            return self._fail(EINVAL, "x_max is NaN")
        rc, rows_ = self._hyper(rec, n, seg_ptr, n_seg, x_max, self_loop)
        if rc:
            return rc
        off = self.fa._arr(offsets, (n + 1,), np.int64)
        off[0] = 0
        off[1:] = np.cumsum([len(r) for r in rows_])
        self.fa._deref(total).value = int(off[n])
        return OK

    def gnnb_hyperbolic_fill(self, rec, n, seg_ptr, n_seg, x_max, self_loop, offsets, nbr, capacity, stream):
        if np.isnan(x_max):
            return self._fail(EINVAL, "x_max is NaN")
        rc, rows_ = self._hyper(rec, n, seg_ptr, n_seg, x_max, self_loop)
        if rc:
            return rc
        off = self.fa._arr(offsets, (n + 1,), np.int64)
        if capacity < off[n]:
            return self._fail(ESIZE, "nbr too small")
        out = self.fa._arr(nbr, (int(off[n]),), np.int32)
        for i, r in enumerate(rows_):
            out[off[i]:off[i + 1]] = r
        return OK


@pytest.fixture(params=["fake", pytest.param("cuda", marks=pytest.mark.gpu)])
def tb(request, monkeypatch, gnn):
    """back end: the numpy entries above (host tensors) or the CUDA kernels (device tensors)"""
    if request.param == "fake":
        from gnnb200 import generate
        with _fake_abi().installed() as fake:
            monkeypatch.setattr(generate, "lib", FakeTGen(fake))
            yield torch.device("cpu")
    else:
        if not torch.cuda.is_available():
            pytest.skip("no CUDA device")
        yield torch.device("cuda")


def _entries():
    from gnnb200 import generate
    return generate.lib


def _strm(dev):
    return torch.cuda.current_stream().cuda_stream if dev.type == "cuda" else 0


def dev_points(dev, n, T, speed, seed):
    pts = torch.empty((T * n, 2), dtype=torch.float32, device=dev)
    from gnnb200 import _lib
    _lib.check(_entries().gnnb_temporal_radius_points(n, T, speed, seed, pts.data_ptr(), _strm(dev)))
    return pts.cpu().numpy().reshape(T, n, 2)


def dev_records(dev, n, T, alpha, R, speed, zeta, seed):
    rec = torch.empty((T * n, 4), dtype=torch.float64, device=dev)
    from gnnb200 import _lib
    _lib.check(_entries().gnnb_temporal_hyperbolic_records(n, T, alpha, R, speed, zeta, seed, rec.data_ptr(),
                                                           _strm(dev)))
    return rec.cpu().numpy().reshape(T, n, 4)


def dev_hyper_rows(dev, rec, x_max, seg=None, self_loop=False):
    """gnnb_hyperbolic_count + _fill on (n, 4) records"""
    from gnnb200 import _lib
    lib = _entries()
    r = torch.as_tensor(np.ascontiguousarray(rec)).to(dev)
    n = len(rec)
    sp = None if seg is None else torch.as_tensor(np.asarray(seg, np.int64)).to(dev)
    args = (r.data_ptr(), n, None if sp is None else sp.data_ptr(), 1 if sp is None else sp.numel() - 1, float(x_max),
            int(self_loop))
    off = torch.empty(n + 1, dtype=torch.int64, device=dev)
    tot = C.c_int64(0)
    _lib.check(lib.gnnb_hyperbolic_count(*args, off.data_ptr(), C.byref(tot), _strm(dev)))
    flat = torch.empty(max(tot.value, 1), dtype=torch.int32, device=dev)
    _lib.check(lib.gnnb_hyperbolic_fill(*args, off.data_ptr(), flat.data_ptr(), tot.value, _strm(dev)))
    return off.cpu().numpy(), flat[:tot.value].cpu().numpy().astype(np.int64)


def graph_rows(g, n, dir="in"):
    """(offsets, flat 0-based neighbour ids) of a snapshot whose edges are grouped by centre"""
    s, t = g.s.cpu().numpy() - 1, g.t.cpu().numpy() - 1
    centre, nb = (t, s) if dir == "in" else (s, t)
    assert (np.diff(centre) >= 0).all(), "edges are grouped by centre"
    off = np.zeros(n + 1, np.int64)
    off[1:] = np.cumsum(np.bincount(centre, minlength=n))
    return off, nb


def bidirected(gnn, g):
    if g.s.is_cuda:
        return gnn.is_bidirected(g)
    s, t = g.s.cpu().numpy(), g.t.cpu().numpy()
    return sorted(zip(s.tolist(), t.tolist())) == sorted(zip(t.tolist(), s.tolist()))


def coo(g):
    return g.s.cpu().numpy(), g.t.cpu().numpy()


# ---------------------------------------------------------------------------------------------- 1. the stream
@pytest.mark.parametrize("speed", [0.1, 0.6, 2.5])
def test_radius_positions(tb, speed):
    n, T, seed = 700, 9, 11
    got = dev_points(tb, n, T, speed, seed)
    ref = ref_points(n, T, speed, seed)
    ref32 = ref.astype(np.float32)
    assert (np.abs(got.astype(np.float64) - ref32) <= np.spacing(np.abs(ref32))).all()     # within 1 fp32 ulp
    if speed > 1:
        assert (ref < 0).any() or (ref > 1).any()                  # the reflection as written leaves the square


@pytest.mark.parametrize("speed", [0.05, 0.4, 1.7])
def test_hyperbolic_records(tb, speed):
    n, T, seed = 700, 12, 12
    alpha, R, zeta = 0.8, 7.0, 1.3
    quirks = {}
    ref = ref_records(n, T, alpha, R, speed, zeta, seed, quirks)
    got = dev_records(tb, n, T, alpha, R, speed, zeta, seed)
    assert (np.abs(got - ref) <= 1e-13 * np.abs(ref)).all()
    if speed > 1:                                                  # generate.jl:373-374 as written: both folds, and a
        assert quirks["gt1"] > 0 and quirks["lt0"] > 0 and quirks["outside"] > 0   # p < -1 stays above 1 after |p|
        assert (got[1:, :, 0] > math.cosh(zeta * R)).any()        # those nodes lie outside the disk


# ---------------------------------------------------------------------------------------------- 2. edges, exactly
@pytest.mark.parametrize("n,T,speed,r,self_loops", [(150, 6, 0.1, 0.2, False), (97, 5, 0.7, 0.35, True),
                                                     (129, 4, 1.6, 0.3, False), (1, 3, 0.1, 0.5, True)])
def test_radius_edges_exact(gnn, tb, n, T, speed, r, self_loops):
    seed = 21
    tg = gnn.rand_temporal_radius_graph(n, T, speed, r, self_loops=self_loops, seed=seed)
    P = dev_points(tb, n, T, speed, seed)
    assert tg.num_snapshots == T and tg.num_nodes == [n] * T
    for t, g in enumerate(tg.snapshots):
        off, flat = graph_rows(g, n)
        roff, rflat = ref_radius(P[t], np.float32(r), self_loops=self_loops)
        assert (off == roff).all() and (flat == rflat).all()
        assert g.w is None


@pytest.mark.parametrize("n,T,alpha,R,speed,zeta,self_loop", [(150, 4, 1.0, 4.0, 0.1, 1.0, False),
                                                               (120, 3, 0.6, 9.0, 0.3, 1.4, True),
                                                               (129, 3, 2.0, 3.0, 1.7, 0.5, False)])
def test_hyperbolic_edges_exact(gnn, tb, n, T, alpha, R, speed, zeta, self_loop):
    seed = 22
    tg = gnn.rand_temporal_hyperbolic_graph(n, T, α=alpha, R=R, speed=speed, ζ=zeta, self_loop=self_loop, seed=seed)
    rec = dev_records(tb, n, T, alpha, R, speed, zeta, seed)
    x_max = math.cosh(zeta * R)
    assert tg.num_snapshots == T and tg.num_nodes == [n] * T
    for t, g in enumerate(tg.snapshots):
        hit = hyper_hits(rec[t], rec[t], x_max)
        if not self_loop:
            np.fill_diagonal(hit, False)
        assert (hit == hit.T).all()
        ref = gnn.GNNGraph(torch.as_tensor(hit.astype(np.float64)))          # GNNGraph(adj): the reference's order
        assert (coo(g)[0] == coo(ref)[0]).all() and (coo(g)[1] == coo(ref)[1]).all()
        assert g.w.dtype == torch.float32 and torch.equal(g.w.cpu(), ref.w)
        assert g.num_edges > 0


def _sampled_rows_match(g, n, q, roff, rflat):
    off, flat = graph_rows(g, n)
    for a, i in enumerate(q):
        assert (flat[off[i]:off[i + 1]] == rflat[roff[a]:roff[a + 1]]).all()


@pytest.mark.gpu
def test_at_scale_sampled_rows(gnn):
    n, T, seed = 20000, 64, 31
    rng = np.random.default_rng(0)
    dev = torch.device("cuda")
    r = math.sqrt(10 / (math.pi * n))                              # mean degree about 10
    tg = gnn.rand_temporal_radius_graph(n, T, 0.01, r, seed=seed)
    P = dev_points(dev, n, T, 0.01, seed)
    for t in (0, 1, 37, 63):
        q = rng.choice(n, 300, replace=False)
        roff, rflat = ref_radius(P[t], np.float32(r), queries=q)
        _sampled_rows_match(tg[t + 1], n, q, roff, rflat)
    assert all(gnn.is_bidirected(g) for g in tg.snapshots[::9])
    R = 2 * math.log(n)
    th = gnn.rand_temporal_hyperbolic_graph(n, T, α=1.0, R=R, speed=0.01, ζ=1.0, seed=seed)
    rec = dev_records(dev, n, T, 1.0, R, 0.01, 1.0, seed)
    for t in (0, 1, 37, 63):
        q = rng.choice(n, 300, replace=False)
        roff, rflat = ref_hyper_rows(rec[t], math.cosh(R), queries=q)
        _sampled_rows_match(th[t + 1], n, q, roff, rflat)
    assert all(gnn.is_bidirected(g) for g in th.snapshots[::9])


@pytest.mark.parametrize("self_loop", [False, True])
def test_hyperbolic_entries_segments(tb, self_loop):
    """the count / fill entries on their own: segments of 0, 1, 127, 128, 129 and 300 records, with duplicates"""
    sizes = [0, 1, 127, 128, 129, 300]
    seg = np.concatenate([[0], np.cumsum(sizes)])
    rec = ref_records(int(seg[-1]), 1, 1.0, 6.0, 0.1, 1.0, 5)[0]
    rec[[10, 20, 30]] = rec[[11, 21, 31]]                          # equal records in a segment
    x_max = math.cosh(6.0)
    off, flat = dev_hyper_rows(tb, rec, x_max, seg, self_loop)
    rows_ = []
    for s in range(len(sizes)):
        a, b = int(seg[s]), int(seg[s + 1])
        ro, rf = ref_hyper_rows(rec[a:b], x_max, self_loop)
        rows_ += [rf[ro[i]:ro[i + 1]] + a for i in range(b - a)]
    assert (np.diff(off) == [len(x) for x in rows_]).all()
    assert (flat == np.concatenate(rows_)).all()


# ---------------------------------------------------------------------------------------------- 3-5. batching, symmetry, seeds
def test_batching_changes_nothing(gnn, tb):
    n, T, speed, r, seed = 80, 5, 0.3, 0.25, 41
    tg = gnn.rand_temporal_radius_graph(n, T, speed, r, seed=seed)
    P = dev_points(tb, n, T, speed, seed)
    for t in range(T):
        alone = gnn.radius_graph(jl(P[t], tb), r)
        assert all((a == b).all() for a, b in zip(coo(tg[t + 1]), coo(alone)))


def test_bidirected_and_reproducible(gnn, tb):
    a = gnn.rand_temporal_radius_graph(60, 4, 0.2, 0.3, seed=7)
    b = gnn.rand_temporal_radius_graph(60, 4, 0.2, 0.3, seed=7)
    c = gnn.rand_temporal_radius_graph(60, 4, 0.2, 0.3, seed=8)
    h = gnn.rand_temporal_hyperbolic_graph(60, 4, α=1.0, R=5.0, speed=0.2, seed=7)
    h2 = gnn.rand_temporal_hyperbolic_graph(60, 4, α=1.0, R=5.0, speed=0.2, seed=7)
    h3 = gnn.rand_temporal_hyperbolic_graph(60, 4, α=1.0, R=5.0, speed=0.2, seed=8)
    for x, y in ((a, b), (h, h2)):
        for gx, gy in zip(x, y):
            assert bidirected(gnn, gx)
            assert all((p == q).all() for p, q in zip(coo(gx), coo(gy)))
    for x, y in ((a, c), (h, h3)):
        assert any(gx.num_edges != gy.num_edges or (coo(gx)[0] != coo(gy)[0]).any() for gx, gy in zip(x, y))
    for g in gnn.rand_temporal_radius_graph(60, 3, 0.2, 0.3, self_loops=True, seed=1):
        assert bidirected(gnn, g)
    for g in gnn.rand_temporal_hyperbolic_graph(60, 3, α=0.5, R=3.0, speed=0.4, self_loop=True, seed=1):
        assert bidirected(gnn, g)


def test_seed_from_torch(gnn, tb):
    torch.manual_seed(3)
    a = gnn.rand_temporal_radius_graph(40, 2, 0.2, 0.3)
    torch.manual_seed(3)
    b = gnn.rand_temporal_radius_graph(40, 2, 0.2, 0.3)
    assert all((p == q).all() for ga, gb_ in zip(a, b) for p, q in zip(coo(ga), coo(gb_)))


# ---------------------------------------------------------------------------------------------- 6. reference cases
def _mean_degree(tg):
    return np.mean([g.num_edges / g.num_nodes for g in tg])


def test_reference_radius(gnn, tb):
    """GNNGraphs/test/generate.jl:100-111 and the docstring's jldoctest"""
    n, T, r, speed = 30, 5, 0.1, 0.1
    tg = gnn.rand_temporal_radius_graph(n, T, speed, r, seed=1)
    assert tg.num_nodes == [n] * T and tg.num_snapshots == T
    tg2 = gnn.rand_temporal_radius_graph(n, T, speed, 0.95, seed=2)
    assert _mean_degree(tg) <= _mean_degree(tg2)
    tg = gnn.rand_temporal_radius_graph(10, 5, 0.1, 1.5, seed=3)  # a complete graph at each snapshot
    assert tg.num_nodes == [10] * 5 and tg.num_edges == [90] * 5


def test_reference_hyperbolic(gnn, tb):
    """GNNGraphs/test/generate.jl:113-126"""
    n, T = 30, 5
    tg = gnn.rand_temporal_hyperbolic_graph(n, T, α=1, R=1, speed=0.1, ζ=1, seed=1)
    assert tg.num_nodes == [n] * T and tg.num_snapshots == T
    tg1 = gnn.rand_temporal_hyperbolic_graph(n, T, α=1, R=10, speed=0.1, ζ=1, seed=2)
    assert _mean_degree(tg1) <= _mean_degree(tg)


def _record(r, theta, zeta=1.0):
    return np.array([math.cosh(zeta * r), math.sinh(zeta * r), math.cos(theta), math.sin(theta)])


def test_hyperbolic_distance_cases(tb):
    """_hyperbolic_distance([1,1], [1,1]) == 0 and its symmetry (GNNGraphs/test/generate.jl:114-115)"""
    A, B = _record(0.23, 0.11), _record(0.98, 0.55)
    same = np.stack([_record(1.0, 1.0), _record(1.0, 1.0)])
    off, flat = dev_hyper_rows(tb, same, 1.0)                     # R = 0: equal records are still at distance 0
    assert off.tolist() == [0, 1, 2] and flat.tolist() == [1, 0]
    off, flat = dev_hyper_rows(tb, same, 1.0, self_loop=True)
    assert off.tolist() == [0, 2, 4] and flat.tolist() == [0, 1, 0, 1]
    xab = hyper_hits(A[None], B[None], -np.inf), hyper_hits(B[None], A[None], -np.inf)
    assert xab[0] == xab[1]
    ang = A[2] * B[2] + A[3] * B[3]
    x = A[0] * B[0] - (A[1] * B[1]) * ang
    d = math.acosh(x)
    for R in (d * (1 - 1e-9), d * (1 + 1e-9)):
        off, flat = dev_hyper_rows(tb, np.stack([A, B]), math.cosh(R))
        assert off[1] - off[0] == off[2] - off[1] == int(R >= d)


# ---------------------------------------------------------------------------------------------- 7. distributions
def test_distributions(tb):
    stats = pytest.importorskip("scipy.stats")
    n, seed = 100000, 99
    P = dev_points(tb, n, 1, 0.1, seed)[0].astype(np.float64)
    assert stats.kstest(P[:, 0], "uniform").pvalue > 1e-3
    assert stats.kstest(P[:, 1], "uniform").pvalue > 1e-3
    alpha, R = 0.7, 6.0
    rec = dev_records(tb, n, 2, alpha, R, 0.1, 1.0, seed)[0]
    theta = np.mod(np.arctan2(rec[:, 3], rec[:, 2]), 2 * np.pi)
    assert stats.kstest(theta, "uniform", args=(0, 2 * np.pi)).pvalue > 1e-3
    r = np.arccosh(rec[:, 0])                                      # ζ = 1
    cdf = lambda v: (np.cosh(alpha * np.asarray(v)) - 1) / (math.cosh(alpha * R) - 1)
    assert stats.kstest(r, cdf).pvalue > 1e-3


# ---------------------------------------------------------------------------------------------- 8. edge cases
def test_small_and_still(gnn, tb):
    tg = gnn.rand_temporal_radius_graph(50, 1, 0.1, 0.2, seed=1)  # T = 1
    assert tg.num_snapshots == 1 and tg.num_nodes == [50]
    for tg in (gnn.rand_temporal_radius_graph(1, 3, 0.1, 0.2, seed=1),
               gnn.rand_temporal_hyperbolic_graph(1, 3, α=1.0, R=2.0, speed=0.1, seed=1)):
        assert tg.num_nodes == [1] * 3 and tg.num_edges == [0] * 3
    tg = gnn.rand_temporal_hyperbolic_graph(1, 2, α=1.0, R=0.0, speed=0.1, self_loop=True, seed=1)
    assert tg.num_edges == [1, 1]
    for tg in (gnn.rand_temporal_radius_graph(70, 4, 0.0, 0.2, seed=5),
               gnn.rand_temporal_hyperbolic_graph(70, 4, α=1.0, R=5.0, speed=0.0, seed=5)):
        first = coo(tg[1])
        assert tg[1].num_edges > 0
        assert all(all((a == b).all() for a, b in zip(coo(g), first)) for g in tg)


def test_dir_self_loops_kws(gnn, tb):
    n = 40
    a = gnn.rand_temporal_radius_graph(n, 3, 0.2, 0.3, seed=4)
    b = gnn.rand_temporal_radius_graph(n, 3, 0.2, 0.3, seed=4, dir="out")
    for ga, gb_ in zip(a, b):
        assert (coo(ga)[0] == coo(gb_)[1]).all() and (coo(ga)[1] == coo(gb_)[0]).all()
        assert not (coo(ga)[0] == coo(ga)[1]).any()
    for g in gnn.rand_temporal_radius_graph(n, 3, 0.2, 0.3, self_loops=True, seed=4):
        s, t = coo(g)
        assert set(range(1, n + 1)) <= set(s[s == t].tolist())
    for g in gnn.rand_temporal_hyperbolic_graph(n, 3, α=1.0, R=4.0, speed=0.2, self_loop=True, seed=4):
        s, t = coo(g)
        assert set(range(1, n + 1)) <= set(s[s == t].tolist())
    feat = torch.arange(float(n))[None, :]
    for tg in (gnn.rand_temporal_radius_graph(n, 2, 0.2, 0.3, seed=4, ndata={"x": feat}, gdata={"u": torch.ones(1)}),
               gnn.rand_temporal_hyperbolic_graph(n, 2, α=1.0, R=4.0, speed=0.2, seed=4, ndata=feat)):
        assert all(g.ndata["x"] is feat for g in tg)
    assert all(g.gdata["u"].shape == (1,) for g in gnn.rand_temporal_radius_graph(n, 2, 0.2, 0.3, seed=4,
                                                                                  gdata={"u": torch.ones(1)}))


def test_errors(gnn, tb):
    with pytest.raises(AssertionError):
        gnn.rand_temporal_radius_graph(10, 2, 0.1, 0.2, dir="both")
    for bad in (dict(speed=float("nan")), dict(speed=float("inf")), dict(r=float("nan")), dict(r=-0.1), dict(n=-1)):
        kw = dict(n=10, T=2, speed=0.1, r=0.2)
        kw.update(bad)
        with pytest.raises(ValueError):
            gnn.rand_temporal_radius_graph(kw["n"], kw["T"], kw["speed"], kw["r"])
    ok = dict(α=1.0, R=2.0, speed=0.1)
    with pytest.raises(AssertionError):
        gnn.rand_temporal_hyperbolic_graph(10, 1, **ok)          # T > 1
    for a in (0.0, -1.0):
        with pytest.raises(AssertionError):
            gnn.rand_temporal_hyperbolic_graph(10, 3, **{**ok, "α": a})
    for bad in ({"ζ": 0.0}, {"ζ": -1.0}, {"R": -1.0}, {"R": float("nan")}, {"α": float("inf")},
                {"speed": float("nan")}, {"ζ": float("inf")}, {"α": 800.0}, {"ζ": 400.0}):
        with pytest.raises(ValueError):
            gnn.rand_temporal_hyperbolic_graph(10, 3, **{**ok, **bad})


class _Called(Exception):
    pass


class _NoEntries:
    def __getattr__(self, name):
        raise _Called(name)


def test_too_large_refused_before_device_work(gnn, tb, monkeypatch):
    from gnnb200 import _lib, generate
    lib = generate.lib
    for n, T in ((2 ** 16, 2 ** 15), (2 ** 31, 1)):
        rc = lib.gnnb_temporal_radius_points(n, T, 0.1, 1, None, _strm(tb))
        assert rc == _lib.ESIZE
        rc = lib.gnnb_temporal_hyperbolic_records(n, T, 1.0, 2.0, 0.1, 1.0, 1, None, _strm(tb))
        assert rc == _lib.ESIZE
    monkeypatch.setattr(generate, "lib", _NoEntries())
    with pytest.raises(AssertionError, match="2\\^31"):
        gnn.rand_temporal_radius_graph(2 ** 16, 2 ** 15, 0.1, 0.2)
    with pytest.raises(AssertionError, match="2\\^31"):
        gnn.rand_temporal_hyperbolic_graph(2 ** 16, 2 ** 15, α=1.0, R=2.0, speed=0.1)


# ---------------------------------------------------------------------------------------------- 9. snapshot editing
def _graph(gnn, n, m, seed):
    rng = np.random.default_rng(seed)
    return gnn.GNNGraph(torch.as_tensor(rng.integers(1, n + 1, m)), torch.as_tensor(rng.integers(1, n + 1, m)),
                        num_nodes=n)


def test_add_remove_snapshot(gnn):
    """the docstrings of temporalsnapshotsgnngraph.jl:108-131 and 163-191"""
    tg = gnn.TemporalSnapshotsGNNGraph([_graph(gnn, 10, 20, k) for k in range(5)])
    assert tg.num_edges == [20] * 5
    new = gnn.add_snapshot(tg, 3, _graph(gnn, 10, 16, 9))
    assert new.num_nodes == [10] * 6 and new.num_edges == [20, 20, 16, 20, 20, 20] and new.num_snapshots == 6
    assert tg.num_edges == [20] * 5 and tg.num_snapshots == 5
    assert gnn.add_snapshot(tg, 6, _graph(gnn, 10, 3, 9)).num_edges == [20] * 5 + [3]
    with pytest.raises(AssertionError, match="number of nodes must match"):
        gnn.add_snapshot(tg, 2, _graph(gnn, 11, 16, 9))
    with pytest.raises(AssertionError, match="cannot add snapshot at time 7"):
        gnn.add_snapshot(tg, 7, _graph(gnn, 10, 16, 9))
    assert gnn.add_snapshot(gnn.TemporalSnapshotsGNNGraph([]), 1, _graph(gnn, 4, 2, 0)).num_nodes == [4]
    tg = gnn.TemporalSnapshotsGNNGraph([_graph(gnn, 10, m, m) for m in (20, 14, 22)])
    new = gnn.remove_snapshot(tg, 2)
    assert new.num_nodes == [10, 10] and new.num_edges == [20, 22] and new.num_snapshots == 2
    assert tg.num_edges == [20, 14, 22] and new[2] is tg[3]
    with pytest.raises(IndexError):
        gnn.remove_snapshot(tg, 4)


# ---------------------------------------------------------------------------------------------- 10. integration
@pytest.mark.gpu
def test_generated_graphs_through_recurrent_layers(gnn):
    n, T, din, dout = 60, 4, 3, 8
    for tg in (gnn.rand_temporal_radius_graph(n, T, 0.1, 0.25, seed=1),
               gnn.rand_temporal_hyperbolic_graph(n, T, α=1.0, R=5.0, speed=0.1, seed=1)):
        xs = [torch.randn(din, n, device="cuda") for _ in range(T)]
        for layer in (gnn.TGCN(din, dout, device="cuda"), gnn.GConvGRU(din, dout, 2, device="cuda")):
            ys = layer(tg, xs)
            assert len(ys) == T and all(tuple(y.shape) == (dout, n) and bool(torch.isfinite(y).all()) for y in ys)
