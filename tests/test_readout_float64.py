"""The graph readouts (readout.py: reduce_nodes / reduce_edges, broadcast_nodes / broadcast_edges, softmax_nodes /
softmax_edges, GlobalPool) and the unfused edge softmax (softmax_edge_neighbors: gnnb_softmax_edge_neighbors and its
_bwd, csrc/edgeops.cu) against float64, element by element, with their pullbacks.

The restatement (`Seg`, plain numpy, from GNNlib/src/utils.jl:12-121 and NNlib's scatter / gather):
  * scatter(aggr, x, ind): out[s] = AGG of the items k with ind[k] = s; a segment without items gets the neutral element
    (0 for + and mean, -Inf for max, +Inf for min); mean divides the sum by max(count, 1).
  * softmax (utils.jl:44-97): M = scatter(max, x), num = exp(x - M[ind]), S = scatter(+, num), alpha = num / S[ind];
    softmax_edges divides by S[ind] + eps(Float32) instead.
  * pullbacks: gather's is scatter(+); scatter(+)'s is gather; mean's is gather(dy ./ max(count, 1)); max / min's is
    (x .== gather(out)) .* gather(dy): EVERY tied extremum receives the full dy (torch's amax would split it among the
    ties, so torch autograd is not the reference here); softmax's is alpha (dalpha - T), T = scatter(+, alpha dalpha);
    softmax_edges adds its max path, -T eps / (S + eps), to every tied maximum.

The float32 emulation (where the kernels promise bits).  The indicator plan sorts the items stably by segment.  A segment
of at most `chunk` items is summed by one group, sequentially in item order from +0.  A longer one is cut at the
multiples of `chunk` of its plan position; each piece is summed the same way and the pieces are added in chunk order
(segwalk.cuh, seg_fixup_kernel).  max / min and every gather round nothing.  So every reduce forward, the broadcast
pullback, the degree counts and the mean / max / min pullbacks are checked bit for bit against it, long segments
included.  The softmax pullback of the library (gnnb_softmax_edge_neighbors_bwd) is emulated from the kernel's own
alpha: fl(alpha dalpha), the same chunked sum, fl(alpha fl(dalpha - T)).  softmax_edges is a torch composition: its
forward is emulated from torch.exp's own bits of fl(x - M).  expf is the one operation that is not restated.

Bounds per element (u = 2^-24, gamma_n = n u / (1 - n u)), asserted beside the bits:
  * sum:  |s^ - s| <= gamma_n sum|x_k|, n the segment's longest accumulation chain: its count when that is <= chunk,
    else chunk + its number of pieces (a piece's sequential sum, then the fix-up over the pieces).  mean: that bound
    / count, + u |mean| for the division.  The float64 reference's own error, 4 n 2^-53 sum|x_k|, is added.
  * softmax alpha: d^ = fl(x - M) is within u |d| of d, so e^(d^) is within 1.001 u |d| of e^d (relative, |d| u < 1e-3),
    and expf adds at most 2 ulp (4 u relative): num^_k = num_k (1 + e_k), |e_k| <= rho_k = 1.001 u |d_k| + 4 u.  The
    chunked sum: |S^ - S| <= E_S = sum rho_k num_k + gamma_n sum num_k.  fl(num / S) adds u, softmax_edges' + eps
    another u.  So |alpha^ - alpha| <= alpha r + 2^-140 with r = rho + E_S / S + 2 u; the 2^-140 covers an exp that
    underflows (S >= 1: the maximum contributes exp(0) = 1 exactly).
  * softmax pullback: T^ = sum fl(alpha^_j g_j) is within E_T = sum alpha_j |g_j| (r_j + u) + gamma_n A of T,
    A = sum alpha_j |g_j|; fl(g - T^) and fl(alpha^ (.)) add u each, alpha^'s own error r_i.  So
    |de^_i - de_i| <= alpha_i (|g_i| + A) (r_i + k u) + alpha_i E_T, k = 2 for the library's pullback.  softmax_edges'
    pullback is torch autograd through div, +eps, broadcast, reduce(+), exp, -, broadcast and reduce(max): the same form
    with k = 5 (the div pullback's three roundings, the accumulation of num's two gradients, the product with num), and
    at a tied maximum the max path's sum over the segment adds sum_j B_j + gamma_n sum_j alpha_j (|g_j| + A) + u |de_i|.
    Second-order terms (products of two relative errors, each < 1e-3) are covered by a factor 1.01.
  * The suite's normwise bars stay as a second assertion, 2e-6 forward and 5e-6 for the pullbacks, wherever the float32
    operation order can meet them: on every output without an emulation, and on every output whose emulation meets
    them.  Three kinds of output cannot, and are held to their bits and bounds alone: the 200 000-item sum whose terms
    cancel (sum|x| / |sum x| near 700 at D = 1), a softmax pullback that cancels to nearly 0 (one dominant alpha, so
    g - T is nearly 0), and softmax_edges' pullback at the tied maxima, where the max path's sum over the segment cancels
    to -T eps / (S + eps) (the bar covers that pullback's other elements).

Every case runs three times: the default kernels twice (no atomics on these paths: the same bits) and
gnnb_set_kernel_variant(12), which sends the 128 / 256 / 512-float rows from the lean work-item kernels back to
seg_reduce_kernel (the same bits, as segreduce.cu promises).  Features at a 4-byte offset into a larger tensor take the
scalar kernels, and must give the aligned call's bits.

Without a GPU the module checks the restatement itself against torch.scatter_reduce and torch autograd in float64, on
tie-free data, and that the exact checks see a wrong fix-up order.
"""
import contextlib
import operator
import zlib

import numpy as np
import pytest
import torch

from test_gpu_parity import GRAPHS, TOL, chunk_graph, make_graph
from test_propagate_abi import pairwise

GRAD_TOL = 5e-6            # the pullbacks' normwise bar in test_gpu_parity.py
U = 2.0 ** -24
U64 = 2.0 ** -53
EPS32 = float(np.finfo(np.float32).eps)
TINY = 2.0 ** -140
SECOND_ORDER = 1.01
AGGRS = ("+", "mean", "max", "min")
NEUTRAL = {"+": 0.0, "mean": 0.0, "max": -np.inf, "min": np.inf}


def gamma(n):
    n = np.asarray(n, np.float64)
    return n * U / (1 - n * U)


# ------------------------------------------------------------------------------------------------ restatement
class Seg:
    """An indicator plan: `ind` the 0-based segment of every item, `n_seg` segments, the plan's `chunk`.  The items in plan
    order (stable by segment), the counts, the pieces of the long segments and each segment's accumulation chain."""

    def __init__(self, ind, n_seg, chunk):
        self.ind = np.asarray(ind, np.int64)
        self.n, self.n_seg, self.chunk = len(self.ind), int(n_seg), int(chunk)
        self.order = np.argsort(self.ind, kind="stable")
        self.sorted = self.ind[self.order]
        self.deg = np.bincount(self.ind, minlength=self.n_seg)
        self.ptr = np.concatenate([[0], np.cumsum(self.deg)])
        self.long = self.deg > self.chunk
        p = np.arange(self.n)
        start = (p == self.ptr[self.sorted]) | (self.long[self.sorted] & (p % self.chunk == 0))
        self.piece = np.cumsum(start) - 1                  # piece of each plan position
        self.piece_seg = self.sorted[start]                # segment of each piece, pieces in chunk order
        pieces = np.bincount(self.piece_seg, minlength=self.n_seg)
        self.chain = np.where(self.long, self.chunk + pieces, self.deg)

    def scatter(self, aggr, x, dtype=np.float64, fixup=None):
        """NNlib.scatter(aggr, x, ind) over the rows of x (n, D).  float32: the kernels' order (pieces from +0 in plan
        order, then the pieces in chunk order; `fixup` may reorder the pieces of each segment, for the self-check)."""
        xs = np.asarray(x)[self.order].astype(dtype)
        D = xs.shape[1]
        live = self.deg > 0
        out = np.full((self.n_seg, D), NEUTRAL[aggr], dtype)
        if aggr in ("max", "min"):
            if live.any():
                out[live] = (np.maximum if aggr == "max" else np.minimum).reduceat(xs, self.ptr[:-1][live], axis=0)
            return out
        if dtype == np.float32:
            part = np.zeros((self.piece_seg.size, D), np.float32)
            np.add.at(part, self.piece, xs)                 # ufunc.at: one rounded add per item, in order
            order = np.arange(self.piece_seg.size) if fixup is None else fixup(self.piece_seg)
            out[:] = 0
            np.add.at(out, self.piece_seg[order], part[order])
        elif live.any():
            out[live] = np.add.reduceat(xs, self.ptr[:-1][live], axis=0)
        if aggr == "mean":
            out = out / np.maximum(self.deg, 1).astype(dtype)[:, None]
        return out

    def gather(self, y):
        return np.asarray(y)[self.ind]

    def scatter_pullback(self, aggr, x, out, dy, dtype=np.float64):
        """the pullback of scatter(aggr, x) at its output `out` (bits: compared in float32, as the forward formed both)"""
        dy = np.asarray(dy).astype(dtype)
        if aggr == "mean":
            dy = dy / np.maximum(self.deg, 1).astype(dtype)[:, None]
        dm = self.gather(dy)
        if aggr in ("max", "min"):
            dm = dm * (np.asarray(x) == self.gather(out)).astype(dtype)    # every tie receives the full dy
        return dm

    def sum_bound(self, x, aggr="+", ref=None):
        n = self.chain[:, None]
        b = (gamma(n) + 4 * n * U64) * self.scatter("+", np.abs(np.asarray(x, np.float64)))
        if aggr == "mean":
            b = b / np.maximum(self.deg, 1)[:, None] + U * np.abs(ref)
        return b

    def softmax(self, x, eps=0.0):
        """float64 alpha and its pieces: d = x - M[ind], num, den = S[ind] (+ eps)"""
        x = np.asarray(x, np.float64)
        d = x - self.gather(self.scatter("max", x))
        num = np.exp(d)
        den = self.gather(self.scatter("+", num)) + eps
        return num / den, d, num, den

    def softmax_bound(self, x, eps=0.0):
        """(alpha, |alpha^ - alpha| bound, relative factor r, den, d): module docstring"""
        alpha, d, num, den = self.softmax(x, eps)
        rho = 1.001 * U * np.abs(d) + 4 * U
        n = self.chain[:, None]
        es = self.scatter("+", rho * num) + gamma(n) * self.scatter("+", num)
        r = rho + self.gather(es) / den + 2 * U
        return alpha, SECOND_ORDER * alpha * r + TINY, r, den, d

    def softmax_pullback(self, alpha, g, eps=0.0, den=None, ties=None):
        """alpha (g - T); with eps, the max path -T eps / (S + eps) to every tied maximum"""
        g = np.asarray(g, np.float64)
        T = self.gather(self.scatter("+", alpha * g))
        de = alpha * (g - T)
        if eps:
            de = de - ties * T * eps / den
        return de

    def softmax_pullback_bound(self, alpha, g, r, k, ties=None, de=None):
        ag = alpha * np.abs(np.asarray(g, np.float64))
        A = self.gather(self.scatter("+", ag))
        n = self.gather(self.chain[:, None] + np.zeros((1, ag.shape[1])))
        et = self.gather(self.scatter("+", ag * (r + U))) + gamma(n) * A
        b = SECOND_ORDER * (alpha * (np.abs(g) + A) * (r + k * U) + alpha * et) + TINY * (np.abs(g) + A)
        if ties is not None:
            extra = self.scatter("+", b) + gamma(self.chain[:, None]) * self.scatter("+", alpha * (np.abs(g) + A))
            b = b + ties * (SECOND_ORDER * self.gather(extra) + U * np.abs(de))
        return b


def emulate_softmax_pullback(seg, alpha32, g32):
    """gnnb_softmax_edge_neighbors_bwd in float32 from the kernel's alpha: fl(alpha fl(g - T)), T the chunked sum"""
    T = seg.gather(seg.scatter("+", alpha32 * g32, np.float32))
    return alpha32 * (g32 - T)


# ------------------------------------------------------------------------------------------------ data
def values(kind, rng, n, D):
    """float32 rows; no -0 anywhere (fmax of +0 and -0 may return either)"""
    if kind == "randn":
        x = rng.standard_normal((n, D))
    elif kind == "levels":                      # five levels: ties for the extremum in almost every segment
        x = rng.integers(-2, 3, (n, D)) / 2
    elif kind == "relu":                        # half the entries 0: ties for the minimum
        x = np.maximum(rng.standard_normal((n, D)), 0)
    else:                                       # x30: exp spans its range, down to underflow
        x = 30 * rng.standard_normal((n, D))
    return x.astype(np.float32) + np.float32(0)


LAYOUTS = {
    # name: (graph sizes, edges per graph); node ids grouped per graph, as batch() makes them
    "tu64": lambda C: ([23] * 64, [46] * 64),                          # the TU-dataset shape
    # graphs 2 and 6 have no nodes (the indicator skips their ids), graphs 3, 4 and 8 no edges
    "empty": lambda C: ([23, 0, 17, 1, 30, 0, 9, 5], [40, 0, 0, 0, 60, 0, 12, 0]),
    "one_graph_edges": lambda C: ([10, 40, 12, 7], [0, 300, 0, 0]),   # every edge in graph 2, a long edge segment
    "chunk": lambda C: ([C, C + 1, 5, C + 1, C, 2 * C + 1, 1], [2 * C, 2 * C + 2, 10, C, C + 1, 4 * C, 2]),
    "long": lambda C: ([200_000], [60_000]),                           # ~1 560 pieces at chunk 128, 6 250 at 32
}


def layout(name, C):
    """(s, t, gi, G): 1-based edges inside their graphs, in one random order over the batch (the edges' indicator is
    unsorted), gi the nodes' graph indicator"""
    sizes, epg = LAYOUTS[name](C)
    rng = np.random.default_rng(zlib.crc32(name.encode()))
    lo = np.concatenate([[0], np.cumsum(sizes)])
    s = np.concatenate([rng.integers(lo[i] + 1, lo[i + 1] + 1, m) for i, m in enumerate(epg) if m])
    t = np.concatenate([rng.integers(lo[i] + 1, lo[i + 1] + 1, m) for i, m in enumerate(epg) if m])
    p = rng.permutation(len(s))
    gi = np.repeat(np.arange(1, len(sizes) + 1), sizes)
    return s[p], t[p], gi, len(sizes)


def gapped_indicator():
    """an explicit indicator, unsorted and with gaps: [3, 1, 3, 1, ...], segments 2 and 5 empty, segment 1 of about 350
    items (longer than the chunk)"""
    rng = np.random.default_rng(5)
    ind = rng.choice([1, 3, 4, 6], 700, p=[0.5, 0.2, 0.2, 0.1])
    ind[:4] = [3, 1, 3, 1]
    ind[-1] = 6
    return ind


def same_bits(a, b):
    a, b = np.ascontiguousarray(a, np.float32), np.ascontiguousarray(b, np.float32)
    return a.shape == b.shape and np.array_equal(a.view(np.int32), b.view(np.int32))


def normwise(a, ref, mask):
    return np.linalg.norm(a[mask] - ref[mask]) / max(np.linalg.norm(ref[mask]), 1e-30)


def check(got, ref, bound, exact=None, tol=TOL, bar=None, what=""):
    """Inf at the same places with the same signs, no NaN, |got - ref| <= bound per element, the float32 emulation's
    bits where it is given, and the normwise bar `tol` over the finite elements of `bar` (default all) where the
    operation order can meet it: always without an emulation, where the emulation meets it with one"""
    got = np.asarray(got)
    g64 = got.astype(np.float64)
    assert not np.isnan(g64).any(), f"{what}: NaN"
    inf = np.isinf(ref)
    fin = ~inf
    if inf.any():
        assert (np.isinf(g64) == inf).all() and (g64[inf] == ref[inf]).all(), f"{what}: infinities differ"
        err = np.where(fin, np.abs(g64 - np.where(fin, ref, 0)), 0)
    else:
        assert np.isfinite(g64).all(), f"{what}: infinities differ"
        err = np.abs(g64 - ref)
    ok = err <= bound
    if not ok.all():
        bad = np.argwhere(~ok)
        i = tuple(bad[0])
        raise AssertionError(f"{what}: |got - ref| = {err[i]:.3e} > bound {np.broadcast_to(bound, err.shape)[i]:.3e} "
                             f"at {list(i)} ({len(bad)} elements; got {g64[i]!r}, ref {ref[i]!r})")
    if exact is not None:
        exact = np.ascontiguousarray(exact, np.float32)
        if not np.array_equal(got.view(np.int32), exact.view(np.int32)):
            bad = np.argwhere(got.view(np.int32) != exact.view(np.int32))
            raise AssertionError(f"{what}: not the float32 emulation's bits at {bad[:4].tolist()} ({len(bad)} elements; "
                                 f"got {got[tuple(bad[0])]!r}, emulation {exact[tuple(bad[0])]!r})")
    mask = fin if bar is None else fin & bar
    if exact is None or normwise(exact.astype(np.float64), ref, mask) <= tol:
        err = normwise(g64, ref, mask)
        assert err <= tol, f"{what}: normwise {err:.3e} > {tol:.0e}"


# ------------------------------------------------------------------------------------------------ CPU: the restatement
def _torch_scatter(aggr, x, ind, n_seg):
    red = {"+": "sum", "mean": "mean", "max": "amax", "min": "amin"}[aggr]
    xt = torch.as_tensor(np.asarray(x, np.float64))
    idx = torch.as_tensor(ind).reshape(-1, 1).expand(-1, xt.shape[1])
    return torch.zeros(n_seg, xt.shape[1], dtype=torch.float64).scatter_reduce(0, idx, xt, red, include_self=False)


SELF_CHECK = [("tu64", 128), ("empty", 128), ("one_graph_edges", 128), ("chunk", 128), ("chunk", 32), ("gapped", 128),
              ("gapped", 32)]


def _self_check_segs(name, C):
    if name == "gapped":
        ind = gapped_indicator()
        return [Seg(ind - 1, ind.max(), C)]
    s, t, gi, G = layout(name, C)
    return [Seg(gi - 1, G, C), Seg(gi[s - 1] - 1, G, C)]


@pytest.mark.parametrize("name,C", SELF_CHECK)
def test_restatement_scatter_against_torch(name, C):
    """scatter in float64 == torch.scatter_reduce on the segments with items, the neutral element on the others; the
    float32 emulation within its bound; the pullbacks == torch autograd (tie-free data)"""
    rng = np.random.default_rng(C)
    for seg in _self_check_segs(name, C):
        x = rng.standard_normal((seg.n, 3))
        live = seg.deg > 0
        for aggr in AGGRS:
            ref = seg.scatter(aggr, x)
            np.testing.assert_allclose(ref[live], _torch_scatter(aggr, x, seg.ind, seg.n_seg).numpy()[live], rtol=1e-13,
                                       atol=1e-13)
            assert (ref[~live] == NEUTRAL[aggr]).all()
            x32 = x.astype(np.float32)
            ref32 = seg.scatter(aggr, x32)
            check(seg.scatter(aggr, x32, np.float32), ref32, seg.sum_bound(x32, aggr, ref32) if aggr in ("+", "mean")
                  else 0.0, what=f"float32 emulation {aggr}")
            xt = torch.as_tensor(x, dtype=torch.float64).requires_grad_(True)
            dy = rng.standard_normal((seg.n_seg, 3))
            red = {"+": "sum", "mean": "mean", "max": "amax", "min": "amin"}[aggr]
            idx = torch.as_tensor(seg.ind).reshape(-1, 1).expand(-1, 3)
            y = torch.zeros(seg.n_seg, 3, dtype=torch.float64).scatter_reduce(0, idx, xt, red, include_self=False)
            y.backward(torch.as_tensor(dy))
            np.testing.assert_allclose(seg.scatter_pullback(aggr, x, ref, dy), xt.grad.numpy(), rtol=1e-13, atol=1e-13)


@pytest.mark.parametrize("eps", [0.0, EPS32])
@pytest.mark.parametrize("name,C", SELF_CHECK)
def test_restatement_softmax_against_torch(name, C, eps):
    """softmax and its pullback (softmax_edges' max path included) == torch autograd in float64, segment by segment, on
    tie-free data; the float32 library pullback emulated from alpha within its bound"""
    rng = np.random.default_rng(7 + C)
    for seg in _self_check_segs(name, C):
        x = 3 * rng.standard_normal((seg.n, 2))
        g = rng.standard_normal((seg.n, 2))
        alpha, d, num, den = seg.softmax(x, eps)
        ties = (d == 0).astype(np.float64)
        de = seg.softmax_pullback(alpha, g, eps, den, ties)
        xt = torch.as_tensor(x).requires_grad_(True)
        out = torch.empty_like(xt)
        parts = [torch.as_tensor(np.flatnonzero(seg.ind == s)) for s in range(seg.n_seg) if seg.deg[s]]
        ys = []
        for k in parts:
            xs = xt[k]
            nm = torch.exp(xs - xs.amax(dim=0, keepdim=True))
            ys.append((k, nm / (nm.sum(dim=0, keepdim=True) + eps)))
        for k, y in ys:
            out = out.index_copy(0, k, y)
        out.backward(torch.as_tensor(g))
        np.testing.assert_allclose(alpha, out.detach().numpy(), rtol=1e-13, atol=1e-300)
        np.testing.assert_allclose(de, xt.grad.numpy(), rtol=1e-10, atol=1e-13)   # eps: the max path is ~1e-8
        if eps == 0.0:
            a32, g32 = alpha.astype(np.float32), g.astype(np.float32)
            a64 = a32.astype(np.float64)          # alpha itself exact here: r = 0
            check(emulate_softmax_pullback(seg, a32, g32), seg.softmax_pullback(a64, g32),
                  seg.softmax_pullback_bound(a64, g32, np.zeros_like(a64), 2), tol=GRAD_TOL, what="emulated pullback")


def test_tie_rule_gives_the_full_gradient():
    """NNlib's max / min pullback: both tied maxima receive dy = 5, where torch's amax gives each 2.5"""
    seg = Seg([0, 0, 0, 0], 1, 128)
    x = np.array([[1.0], [3.0], [3.0], [2.0]])
    out = seg.scatter("max", x)
    np.testing.assert_array_equal(seg.scatter_pullback("max", x, out, [[5.0]]), [[0.0], [5.0], [5.0], [0.0]])
    xt = torch.as_tensor(x).requires_grad_(True)
    xt.amax(dim=0).backward(torch.tensor([5.0], dtype=torch.float64))
    assert xt.grad.numpy().ravel().tolist() == [0.0, 2.5, 2.5, 0.0]


@pytest.mark.parametrize("C", [128, 32])
def test_emulation_sees_the_fixup_order(C):
    """On the long segments, the chunk-order emulation differs in bits from the pieces added in reverse order and from one
    sequential sum: the exact checks below would catch a fix-up that combines the pieces in another order"""
    s, t, gi, G = layout("chunk", C)
    seg = Seg(gi[s - 1] - 1, G, C)
    assert seg.long.sum() >= 3
    x = values("randn", np.random.default_rng(1), seg.n, 64)
    mine = seg.scatter("+", x, np.float32)
    rev = seg.scatter("+", x, np.float32, fixup=lambda ps: np.lexsort((-np.arange(ps.size), ps)))
    flat = np.zeros_like(mine)
    np.add.at(flat, seg.ind, x)
    for other in (rev, flat):
        assert np.array_equal(mine[~seg.long], other[~seg.long])
        assert not same_bits(mine[seg.long], other[seg.long])


# ------------------------------------------------------------------------------------------------ GPU fixtures
@contextlib.contextmanager
def chunk_set(gnn, C):
    try:
        gnn._lib.check(gnn._lib.lib.gnnb_set_chunk_edges(C))
        yield
    finally:
        gnn._lib.lib.gnnb_set_chunk_edges(128)


@pytest.fixture(scope="module")
def batches(gnn):
    """(name, chunk) -> (GNNGraph on cuda whose indicator plans were built at that chunk, Seg of its nodes, Seg of its
    edges)"""
    if not torch.cuda.is_available():
        pytest.skip("no CUDA device")
    cache = {}

    def get(name, C):
        if (name, C) not in cache:
            s, t, gi, G = layout(name, C)
            with chunk_set(gnn, C):            # the indicator plans are built lazily: build them now, at this chunk
                g = gnn.GNNGraph(torch.as_tensor(s, device="cuda"), torch.as_tensor(t, device="cuda"),
                                 num_nodes=len(gi), num_graphs=G, graph_indicator=torch.as_tensor(gi, device="cuda"))
                gnn.readout._indicator_plan(g, False)
                gnn.readout._indicator_plan(g, True)
            cache[(name, C)] = (g, Seg(gi - 1, G, C), Seg(gi[s - 1] - 1, G, C))
        return cache[(name, C)]

    yield get
    cache.clear()


@pytest.fixture
def runs(gnn):
    """runs(fn): fn() -> tensors; called with the default kernels twice and under gnnb_set_kernel_variant(12), which
    must all give the same bits; returns them as float32 numpy arrays"""
    lib = gnn._lib

    def go(fn):
        outs = []
        try:
            for v in (0, 0, 12):
                lib.check(lib.lib.gnnb_set_kernel_variant(v))
                outs.append([t.detach().contiguous().cpu().numpy() for t in fn()])
        finally:
            lib.lib.gnnb_set_kernel_variant(0)
        for k, (a, b, c) in enumerate(zip(*outs)):
            assert same_bits(a, b), f"output {k}: a second run gave other bits"
            assert same_bits(a, c), f"output {k}: gnnb_set_kernel_variant(12) gave other bits"
        return outs[0]

    yield go


def features(gnn, x, offset=0):
    """rows x (n, D) -> (leaf, Julia-shaped (D, n) view, grad getter); offset 4: the rows start 4 bytes into a larger
    allocation, so that no kernel may use 16-byte loads"""
    n, D = x.shape
    o = offset // 4
    buf = torch.zeros(x.size + 4, dtype=torch.float32, device="cuda")
    buf[o:o + x.size] = torch.from_numpy(np.ascontiguousarray(x).ravel()).cuda()
    leaf = buf.requires_grad_(True)
    view = leaf[o:o + x.size].view(n, D)
    assert (view.data_ptr() % 16 != 0) == (offset != 0)
    return leaf, gnn.unrows(view), lambda: leaf.grad[o:o + x.size].view(n, D)


def cuda_rows(x):
    return torch.from_numpy(np.ascontiguousarray(x, np.float32)).cuda()


# ------------------------------------------------------------------------------------------------ GPU: reduce, broadcast
REDUCE_AXES = dict(layout=["tu64", "empty", "one_graph_edges", "chunk", "chunk32", "gapped", "gapped32"],
                   D=[1, 3, 5, 128, 256, 260, 512], vals=["randn", "levels", "relu"], offset=[0, 4])
# the 200 000-node graph: the fix-up over ~1 560 / 6 250 pieces with the scalar kernels, the float4 chunk kernel (D = 8)
# and the lean kernel, at both chunks, aligned and not (the widths themselves are covered by the layouts above)
REDUCE_LONG = [dict(layout=lay, D=D, vals=v, offset=o) for lay, D, v, o in
               (("long", 1, "randn", 0), ("long", 8, "levels", 0), ("long", 128, "relu", 0), ("long32", 5, "levels", 4),
                ("long32", 3, "randn", 0))]
REDUCE_CASES = [pytest.param(i, *r.values(), id="-".join(f"{k}{v}" for k, v in r.items()))
                for i, r in enumerate(pairwise(REDUCE_AXES, 11) + REDUCE_LONG)]


def _split(layout_name):
    return (layout_name[:-2], 32) if layout_name.endswith("32") else (layout_name, 128)


def _aggr_fn(gnn, aggr):
    return {"+": operator.add, "mean": gnn.mean, "max": max, "min": min}[aggr]


def _check_reduce(gnn, runs, seg, x, call, offset, rng, what, ties):
    """call(aggr_fn, x_julia) -> Julia-shaped readout, for every aggregation: forward and pullback against the
    restatement, bits and bounds (`ties`: the data must give some extremum a tie); returns the forward results"""
    dy = values("randn", rng, seg.n_seg, x.shape[1])
    results = {}
    for aggr in AGGRS:
        fn = _aggr_fn(gnn, aggr)

        def once(off):
            leaf, xj, grad = features(gnn, x, off)
            y = call(fn, xj)
            y.backward(gnn.unrows(cuda_rows(dy)))
            return [gnn.rows(y), grad()]

        y, dx = runs(lambda: once(offset))
        if offset:
            y0, dx0 = runs(lambda: once(0))
            assert same_bits(y, y0) and same_bits(dx, dx0), f"{what} {aggr}: the misaligned call's bits differ"
        w = f"{what} {aggr}"
        ref = seg.scatter(aggr, x)
        bound = seg.sum_bound(x, aggr, ref) if aggr in ("+", "mean") else 0.0
        check(y, ref, bound, exact=seg.scatter(aggr, x, np.float32), what=w)
        dref = seg.scatter_pullback(aggr, x, ref, dy)
        dex = seg.scatter_pullback(aggr, x, y, dy, np.float32)
        check(dx, dref, U * np.abs(dref), exact=dex, tol=GRAD_TOL, what="d " + w)
        if aggr in ("max", "min"):
            tie = x == seg.gather(y)
            cnt = seg.scatter("+", tie.astype(np.float64))
            multi = tie & (seg.gather(cnt) > 1)
            assert multi.any() or not ties, f"{w}: no tie to check"
            assert np.array_equal(dx[multi], seg.gather(dy)[multi]), f"{w}: a tied extremum lost part of dy"
            assert not dx[~tie].any(), f"{w}: dy reached an element that is not the extremum"
        results[aggr] = y
    return results


@pytest.mark.gpu
@pytest.mark.parametrize("seed,lay,D,vals,offset", REDUCE_CASES)
def test_reduce_against_float64(gnn, batches, runs, seed, lay, D, vals, offset):
    """reduce_nodes / reduce_edges / GlobalPool (and reduce_nodes(aggr, indicator, x) on an unsorted indicator with gaps)
    with + / mean / max / min: the float32 emulation bit for bit (long segments included), the float64 bounds, the
    pullbacks bit for bit, every tie receiving the full gradient; broadcast_nodes / broadcast_edges and their pullbacks
    the same way; the degree counts behind mean exactly"""
    name, C = _split(lay)
    rng = np.random.default_rng(500 + seed)
    what = f"{lay} D={D} {vals} offset={offset}"
    if name == "gapped":
        ind = gapped_indicator()
        seg = Seg(ind - 1, ind.max(), C)
        it = torch.as_tensor(ind, device="cuda")
        x = values(vals, rng, seg.n, D)
        with chunk_set(gnn, C):              # the indicator form builds its plan on every call
            _check_reduce(gnn, runs, seg, x, lambda fn, xj: gnn.reduce_nodes(fn, it, xj), offset, rng, "indicator " + what,
                           vals == "levels")
        return
    g, nseg, eseg = batches(name, C)
    lib = gnn._lib
    for kind, seg in (("nodes", nseg), ("edges", eseg)):
        ip = gnn.readout._indicator_plan(g, kind == "edges")
        deg = torch.empty(seg.n_seg, dtype=torch.float32, device="cuda")
        lib.check(lib.lib.gnnb_degree(ip.plan.h, lib.DIR_IN, None, deg.data_ptr(), torch.cuda.current_stream().cuda_stream))
        assert same_bits(deg.cpu().numpy(), seg.deg.astype(np.float32)), f"{kind} {what}: degree counts"
        x = values(vals, rng, seg.n, D)
        red = gnn.reduce_nodes if kind == "nodes" else gnn.reduce_edges
        ys = _check_reduce(gnn, runs, seg, x, lambda fn, xj: red(fn, g, xj), offset, rng, f"{kind} {what}",
                           vals == "levels")
        if kind == "nodes":
            for aggr in AGGRS:
                pool = gnn.GlobalPool(_aggr_fn(gnn, aggr))
                assert same_bits(gnn.rows(pool(g, gnn.unrows(cuda_rows(x)))).cpu().numpy(), ys[aggr]), f"GlobalPool {aggr}"
        # broadcast: a gather forward, a scatter(+) pullback
        z = values(vals, rng, seg.n_seg, D)
        dy = values("randn", rng, seg.n, D)
        bc = gnn.broadcast_nodes if kind == "nodes" else gnn.broadcast_edges

        def once(off):
            leaf, zj, grad = features(gnn, z, off)
            y = bc(g, zj)
            y.backward(gnn.unrows(cuda_rows(dy)))
            return [gnn.rows(y), grad()]

        y, dz = runs(lambda: once(offset))
        if offset:
            y0, dz0 = runs(lambda: once(0))
            assert same_bits(y, y0) and same_bits(dz, dz0), f"broadcast {kind} {what}: the misaligned call's bits differ"
        assert same_bits(y, seg.gather(z)), f"broadcast_{kind} {what}"
        ref = seg.scatter("+", dy)
        check(dz, ref, seg.sum_bound(dy), exact=seg.scatter("+", dy, np.float32), tol=GRAD_TOL,
              what=f"d broadcast_{kind} {what}")


# ------------------------------------------------------------------------------------------------ GPU: softmax
SOFTMAX_AXES = dict(layout=["tu64", "empty", "one_graph_edges", "chunk", "chunk32"], D=[1, 3, 5, 128, 256, 260, 512],
                    vals=["randn", "levels", "x30"], offset=[0, 4])
SOFTMAX_LONG = [dict(layout=lay, D=D, vals=v, offset=o) for lay, D, v, o in
                (("long", 1, "x30", 0), ("long", 8, "randn", 0), ("long32", 5, "levels", 4), ("long32", 128, "x30", 0))]
SOFTMAX_CASES = [pytest.param(i, *r.values(), id="-".join(f"{k}{v}" for k, v in r.items()))
                 for i, r in enumerate(pairwise(SOFTMAX_AXES, 12) + SOFTMAX_LONG)]


def _check_softmax(gnn, runs, seg, x, call, offset, eps, rng, what):
    """call(x_julia) -> alpha; forward within its bound (softmax_edges: the emulation from torch.exp's bits), the
    pullback against the float64 one: the library's bit for bit from its own alpha, softmax_edges' within its bound"""
    dy = values("randn", rng, seg.n, x.shape[1])

    def once(off):
        leaf, xj, grad = features(gnn, x, off)
        y = call(xj)
        y.backward(gnn.unrows(cuda_rows(dy)))
        return [gnn.rows(y), grad()]

    a, de = runs(lambda: once(offset))
    if offset:
        a0, de0 = runs(lambda: once(0))
        assert same_bits(a, a0) and same_bits(de, de0), f"{what}: the misaligned call's bits differ"
    alpha, b_alpha, r, den, d = seg.softmax_bound(x, eps)
    exact = None
    if eps:
        m32 = seg.gather(seg.scatter("max", x, np.float32))
        num = torch.exp(cuda_rows(x - m32)).cpu().numpy()       # the one rounding not restated: torch's own exp
        exact = num / (seg.gather(seg.scatter("+", num, np.float32)) + np.float32(eps))
    check(a, alpha, b_alpha, exact=exact, what=what)
    ties = (d == 0).astype(np.float64)
    dref = seg.softmax_pullback(alpha, dy, eps, den, ties)
    if eps:
        # the max path sums the direct pullbacks of a segment, which cancel to -T eps / (S + eps): at a tied maximum
        # that sum's rounding is the error, so the normwise bar is taken over the other elements
        bound = seg.softmax_pullback_bound(alpha, dy, r, 5, ties, dref)
        check(de, dref, bound, tol=GRAD_TOL, bar=ties == 0, what="d " + what)
    else:
        bound = seg.softmax_pullback_bound(alpha, dy, r, 2)
        check(de, dref, bound, exact=emulate_softmax_pullback(seg, a, dy), tol=GRAD_TOL, what="d " + what)


@pytest.mark.gpu
@pytest.mark.parametrize("seed,lay,D,vals,offset", SOFTMAX_CASES)
def test_softmax_nodes_edges_against_float64(gnn, batches, runs, seed, lay, D, vals, offset):
    """softmax_nodes (gnnb_softmax_edge_neighbors on the indicator plan) and softmax_edges (a torch composition with
    + eps(Float32)), forward and pullback"""
    name, C = _split(lay)
    g, nseg, eseg = batches(name, C)
    rng = np.random.default_rng(700 + seed)
    for kind, seg, fn, eps in (("softmax_nodes", nseg, gnn.softmax_nodes, 0.0),
                               ("softmax_edges", eseg, gnn.softmax_edges, EPS32)):
        x = values(vals, rng, seg.n, D)
        _check_softmax(gnn, runs, seg, x, lambda xj: fn(g, xj), offset, eps, rng, f"{kind} {lay} D={D} {vals} "
                       f"offset={offset}")


@pytest.fixture(scope="module")
def neighbor_graphs(gnn):
    if not torch.cuda.is_available():
        pytest.skip("no CUDA device")
    from test_gpu_parity import fixture_plan
    cache = {}

    def get(name):
        if name not in cache:
            kw = dict(GRAPHS[name])
            rng = np.random.default_rng(list(GRAPHS).index(name))
            s, t = chunk_graph(rng, **kw) if "chunk" in kw else make_graph(rng, **kw)
            g = fixture_plan(gnn, name, s, t, kw["n"])
            cache[name] = (g, Seg(t - 1, kw["n"], kw.get("chunk", 128)))
        return cache[name]

    yield get
    cache.clear()


NEIGHBOR_AXES = dict(graph=["hubs", "chunk_edges", "chunk32", "empty_rows"], K=[1, 3, 128, 256, 260],
                     vals=["randn", "levels", "x30"])
NEIGHBOR_CASES = [pytest.param(*r.values(), id="-".join(f"{k}{v}" for k, v in r.items()))
                  for r in pairwise(NEIGHBOR_AXES, 13)]


@pytest.mark.gpu
@pytest.mark.parametrize("gname,K,vals", NEIGHBOR_CASES)
def test_softmax_edge_neighbors_against_float64(gnn, neighbor_graphs, runs, gname, K, vals):
    """softmax_edge_neighbors over every target's in-edges: hub rows far longer than the chunk, rows at the chunk
    boundaries at chunk 128 and 32, targets without in-edges"""
    g, seg = neighbor_graphs(gname)
    rng = np.random.default_rng(900 + K)
    x = values(vals, rng, seg.n, K)
    _check_softmax(gnn, runs, seg, x, lambda xj: gnn.softmax_edge_neighbors(g, xj), 4 if K == 128 else 0, 0.0, rng,
                   f"{gname} K={K} {vals}")
