"""The Set2Set and attention-pooling entries (csrc/set2set.cu: gnnb_set2set_attend, gnnb_set2set_attend_bwd,
gnnb_attention_pool, gnnb_attention_pool_bwd) against float64, element by element, on general plans and on the
graph-indicator plans the layers build.

The restatement (`Plan`, plain numpy float64, from include/gnnb200.h) over a 0-based COO (s, t) of n_src sources and
n_dst targets, the edges of a target in plan order (stable by target):
  * forward: s_k = <q_{t_k}, x_{s_k}> (Set2Set) or gate[s_k] (pooling); M_i = max_k s_k; S_i = sum_k exp(s_k - M_i);
    r_i = sum_k exp(s_k - M_i) x_{s_k} / S_i.  A target without edges: r = 0, M = -Inf, S = 0.
  * pullbacks: alpha_k = exp(s_k - M_i) / S_i; T_i = <dr_i, r_i>; g_k = <dr_i, x_{s_k}>; ds_k = alpha_k (g_k - T_i);
    Set2Set: dxe_k = alpha_k dr_i + ds_k q_i, dq_i = sum_k ds_k x_{s_k}; pooling: dfe_k = alpha_k du_i, dgate_e_k = ds_k.
    Per-edge outputs are in COO order.
Without a GPU the restatement is checked against torch autograd in float64 (tie-free data).

Bounds per element (u = 2^-24, gamma_n = n u / (1 - n u), as in test_readout_float64.py).  Write n_i for a target's
accumulation chain (`Seg.chain`: its edge count, or chunk + its number of pieces for a row longer than the chunk) and
L = ceil(D / 32) + 3, which bounds the terms one lane adds on either path (4 ceil(D / 128) float4 terms or ceil(D / 32)
scalar ones):
  * score: a per-lane fma chain of at most L terms, then a 5-level butterfly: sigma_k <= gamma_{L+5} sum_d |q_d x_d|.
    When every q and x is a multiple of a power of two g_q, g_x and sum |q x| < 2^24 g_q g_x, every partial sum is a
    float32 integer multiple of g_q g_x: sigma_k = 0.  Pooling's score is the gate itself: sigma = 0, and seg_max is
    the largest gate bit for bit.  With tau_k = sigma_k + max_i sigma, |d^_k - d_k| <= tau_k for d = s - M.
  * weights: fl(s - M) is within u |d^| of d^, and e^x moves by expm1 of its argument's error; every expf adds at most
    2 ulp (4 u), every fma or product u.  Inside a piece each edge passes at most one expf and one rounding per later
    edge (a rescale when the max moves, the sum's own fma); the fix-up adds per later piece two expf (s0, s1), a product
    and an fma.  So every weight w_k = exp(d_k) enters S and the accumulator with relative error
    eps_k = expm1(tau_k + 1.001 u (|d_k| + tau_k)) + 10 u n_i.  S: |S^ - S| <= sum_k w_k eps_k = S eps_S.
    r = fl(acc / S^): |r^ - r| <= sum_k alpha_k |x_k| eps_k + |r| (eps_S + u).
  * the pullback recomputes alpha^ = fl(expf(fl(s^ - M^)) / S^) from the forward's own M^, S^ (fed back as the layers
    do): relative error eps^a_k = expm1(tau_k + 1.001 u (|d_k| + tau_k)) + 5 u + eps_S.  T^ and g^ are dot products
    like the score: |T^ - T| <= sum |dr| b_r + gamma_{L+5} sum |dr| (|r| + b_r), |g^ - g| <= gamma_{L+5} sum |dr x|.
    ds = fl(alpha^ fl(g^ - T^)): |ds^ - ds| <= alpha (eps^a + 2 u)(|g| + |T|) + alpha (E_g + E_T), the cancellation
    magnitude |g| + |T| of test_set2set.bwd_magnitudes / test_attention_pool.dgate_magnitude.
    dxe = fma(dr, alpha^, fl(q ds^)): alpha |dr| (eps^a + u) + |q| (b_ds + 2 u |ds|).  dfe = fl(du alpha^):
    alpha |du| (eps^a + u).  dq: sum_k |x_k| b_ds,k + gamma_{n_i} sum_k |ds_k x_k|.
  Second-order terms (products of relative errors, each below 2e-3) are covered by a factor 1.01; 2^-140 per unit of
  magnitude covers an expf that underflows; 4 (D + E + 8) 2^-53 per unit of magnitude covers the float64 reference.

Exact cases (bits).  With equal scores (q = 0 for Set2Set, a constant gate per graph for pooling) every expf is of 0
and gives 1; in the fix-up s0 = expf(-FLT_MAX - M_p) = 0 on the first piece and 1 after it.  So S = count exactly,
r = fl(chunked float32 sum / count) with the chunked sum of `Seg.scatter(..., np.float32)` (pieces from +0 in plan
order, the pieces in chunk order), dfe = fl(fl(1/n) du) and Set2Set's dxe = fl(dr fl(1/n)).  Where a score lies more
than 104 below its row's max, alpha = 0 exactly, and so are dfe, dgate_e and Set2Set's dxe.  Pooling's forward and dfe
contain no dot product, so the float4 path and the scalar path (operands at 4, 8 or 12 B from a 16 B boundary) give the
same bits; for Set2Set the lane partition of the dot differs between the paths, and only the bounds are required.

Every operand sits in a `Guarded` buffer (test_propagate_abi.py): NaN around the inputs, the sentinel around and inside
the outputs; after each call no input or guard changed, no write left an output, every output element was written.

Without a GPU a float32 emulation of the kernels' operation order (the lane partition of every dot product, the online
softmax with its rescales, the fix-ups in chunk order) is checked to stay inside these bounds on the case matrix's
shapes.  np.exp stands in for expf, and fma(a, b, c) is emulated as the float64 a b + c rounded to float32 (exact
product, one float64 rounding of the sum before the float32 one), so the emulation is close to the kernels' bits but
not promised to be them.  Planted errors must fail: the pieces combined in reverse chunk order break the exact sums,
and one alpha off by 2^-10 breaks the bound.
"""
import math
import zlib

import numpy as np
import pytest
import torch

from test_propagate_abi import Guarded, raw_plan
from test_readout_float64 import SECOND_ORDER, TINY, U, U64, Seg, chunk_set, gamma

WIDTHS = [1, 4, 31, 32, 33, 64, 65, 128, 129, 132, 256, 257, 260, 512, 513, 516, 1023, 1024]
KINDS = ["randn", "sharp", "rising", "falling", "ties", "spread", "equal"]
FLT_MAX = np.float32(np.finfo(np.float32).max)
UNDERFLOW = -104.0          # below this, expf(d) is 0 in float32


def lane_terms(D):
    return -(-D // 32) + 3


def grid(a):
    """the largest power of two 2^-e (e >= 0) of which every entry of a is a multiple, 0 if none up to 2^-40"""
    a = np.asarray(a, np.float64)
    for e in range(41):
        v = a * 2.0 ** e
        if np.array_equal(v, np.round(v)):
            return 2.0 ** -e
    return 0.0


# ------------------------------------------------------------------------------------------------ restatement
class Plan:
    """0-based COO (s, t) over n_src sources and n_dst targets at `chunk`; `indicator`: edge k has source k (the
    graph-indicator plan).  The edges of every target in plan order, its pieces and its chain come from `Seg`."""

    def __init__(self, s, t, n_src, n_dst, chunk, indicator):
        self.s, self.t = np.asarray(s, np.int64), np.asarray(t, np.int64)
        self.E, self.n_src, self.n_dst, self.chunk = len(self.s), int(n_src), int(n_dst), int(chunk)
        self.indicator = indicator
        self.seg = Seg(self.t, self.n_dst, self.chunk)
        self.live = self.seg.deg > 0
        pos = np.arange(self.E) - self.seg.ptr[self.seg.sorted]      # rank of each plan position inside its row
        self.src_rank = np.zeros(self.n_src, np.int64)              # rank of each source's first edge in plan order
        self.src_rank[self.s[self.seg.order[::-1]]] = pos[::-1]

    def row(self, v):
        """per-target values -> per-edge (COO order)"""
        return np.asarray(v)[self.t]

    def sum(self, v):
        """per-edge rows (E, D) -> float64 per-target sums"""
        v = np.asarray(v, np.float64)
        return self.seg.scatter("+", v if v.ndim == 2 else v[:, None])


def scores(P, x, q=None, gate=None):
    """(s_k, sigma_k) per edge: the float64 score and the bound of the kernel's error in it"""
    if gate is not None:
        return np.asarray(gate, np.float64)[P.s], np.zeros(P.E)
    x64, q64 = np.asarray(x, np.float64), np.asarray(q, np.float64)
    D = x64.shape[1]
    sc = np.einsum("ed,ed->e", q64[P.t], x64[P.s])
    mag = np.einsum("ed,ed->e", np.abs(q64[P.t]), np.abs(x64[P.s]))
    exact = mag < 2.0 ** 24 * grid(q) * grid(x)
    return sc, np.where(exact, 0.0, gamma(lane_terms(D) + 5) * mag + 2 * D * U64 * mag)


def forward64(P, x, sc):
    """M, S, r and the per-edge d = s - M, w = exp(d), alpha"""
    x64 = np.asarray(x, np.float64)
    M = np.full(P.n_dst, -np.inf)
    np.maximum.at(M, P.t, sc)
    d = sc - P.row(M) if P.E else np.zeros(0)
    w = np.exp(d)
    S = P.sum(w)[:, 0]
    r = P.sum(w[:, None] * x64[P.s]) / np.where(S > 0, S, 1)[:, None]
    alpha = w / P.row(S) if P.E else np.zeros(0)
    return dict(M=M, S=S, r=r, d=d, w=w, alpha=alpha)


def pullback64(P, x, F, dr, q=None):
    """Set2Set (q given): dxe, dq, ds; pooling: dfe, dgate_e = ds"""
    x64, dr64 = np.asarray(x, np.float64), np.asarray(dr, np.float64)
    al = F["alpha"]
    T = np.einsum("id,id->i", dr64, F["r"])
    g = np.einsum("ed,ed->e", dr64[P.t], x64[P.s])
    ds = al * (g - P.row(T))
    de = al[:, None] * dr64[P.t]
    out = dict(T=T, g=g, ds=ds)
    if q is not None:
        out["dxe"] = de + ds[:, None] * np.asarray(q, np.float64)[P.t]
        out["dq"] = P.sum(ds[:, None] * x64[P.s])
    else:
        out["dfe"] = de
        out["dgate"] = ds
    return out


def bounds(P, x, F, sigma, dr, B, q=None):
    """per-element bounds of the kernels' outputs against forward64 / pullback64 (module docstring)"""
    x64, dr64 = np.abs(np.asarray(x, np.float64)), np.abs(np.asarray(dr, np.float64))
    D = x64.shape[1]
    ref = 4 * (D + P.E + 8) * U64
    n = P.seg.chain.astype(np.float64)
    smax = np.zeros(P.n_dst)
    if P.E:
        np.maximum.at(smax, P.t, sigma)
    tau = sigma + P.row(smax)
    d, w, al, S = F["d"], F["w"], F["alpha"], F["S"]
    shift = np.expm1(tau + 1.001 * U * (np.abs(d) + tau))
    eps = shift + 10 * U * P.row(n)
    eps_S = P.sum(w * eps)[:, 0] / np.where(S > 0, S, 1)
    xs = x64[P.s]
    ax = al[:, None] * xs
    sum_x = P.sum(xs)
    mag_r = P.sum(ax)
    b = dict(M=smax, S=SECOND_ORDER * S * eps_S + TINY * P.seg.deg + ref * S)
    absr = np.abs(F["r"])
    b["r"] = (SECOND_ORDER * (P.sum(ax * eps[:, None]) + absr * (eps_S + U)[:, None]) + TINY * sum_x
              + ref * mag_r)
    eps_a = shift + 5 * U + P.row(eps_S)
    gL = gamma(lane_terms(D) + 5)
    ET = (dr64 * b["r"]).sum(1) + gL * (dr64 * (absr + b["r"])).sum(1)
    Eg = gL * np.einsum("ed,ed->e", dr64[P.t], xs)
    mag_ds = al * (np.abs(B["g"]) + np.abs(P.row(B["T"])))
    b["ds"] = (SECOND_ORDER * (mag_ds * (eps_a + 2 * U) + al * (Eg + P.row(ET)))
               + (TINY + ref) * (np.abs(B["g"]) + np.abs(P.row(B["T"]))))
    de = al[:, None] * dr64[P.t]
    if q is None:
        b["dfe"] = SECOND_ORDER * de * (eps_a + U)[:, None] + (TINY + ref) * dr64[P.t]
        b["dgate"] = b["ds"]
    else:
        aq = np.abs(np.asarray(q, np.float64))[P.t]
        ads = np.abs(B["ds"])
        b["dxe"] = (SECOND_ORDER * (de * (eps_a + U)[:, None] + aq * (b["ds"] + 2 * U * ads)[:, None])
                    + (TINY + ref) * (dr64[P.t] + aq * ads[:, None]))
        mag_dq = P.sum(ads[:, None] * xs)
        b["dq"] = SECOND_ORDER * (P.sum(xs * b["ds"][:, None]) + gamma(n)[:, None] * mag_dq) + ref * mag_dq
    return b


# ------------------------------------------------------------------------------------------------ plans
def indicator_layout(sizes, seed=None):
    gi = np.repeat(np.arange(len(sizes)), sizes)
    if seed is not None:
        gi = np.random.default_rng(seed).permutation(gi)
    return np.arange(len(gi)), gi, len(gi), len(sizes)


def square_layout(C):
    """300 nodes: random edges, multi-edges, self loops, a hub source read by 400 targets and a hub target of 2C + 3
    in-edges"""
    rng = np.random.default_rng(31)
    n = 300
    s, t = rng.integers(0, n, 1500), rng.integers(0, n, 1500)
    k = rng.integers(0, 1500, 100)
    s = np.concatenate([s, s[k], np.arange(0, n, 6), np.full(400, 7), rng.integers(0, n, 2 * C + 3)])
    t = np.concatenate([t, t[k], np.arange(0, n, 6), rng.integers(0, n, 400), np.full(2 * C + 3, 11)])
    p = rng.permutation(len(s))
    return s[p], t[p], n, n


def bipartite_layout(n_src, n_dst, E, seed):
    rng = np.random.default_rng(seed)
    return rng.integers(0, n_src, E), rng.integers(0, n_dst, E), n_src, n_dst


def layout(name, C):
    """(s, t, n_src, n_dst, indicator) for the plan `name` at chunk C"""
    sizes = [0, 1, 2, 3, 5, 31, 32, 33, C - 1, C, C + 1, 2 * C, 2 * C + 1]
    ind = {
        "sizes": lambda: indicator_layout(sizes),
        "sizes_perm": lambda: indicator_layout(sizes, seed=C),
        # long graphs side by side: the end of one and the start of the next share a chunk (slots 2k and 2k + 1)
        "straddle": lambda: indicator_layout([C + 5, 2 * C + 7, C + 1, 2, C + 5]),
        # rows ending on lane 31 and on lane 0 of a 32-edge batch
        "lanes": lambda: indicator_layout([32, 1, 31, 32, 33, 31, 1, 64, 63, 2, 96]),
        "huge": lambda: indicator_layout([3, 10 ** 5, 17]),
        "no_nodes": lambda: indicator_layout([0, 0, 0, 0]),
    }
    gen = {
        "square": lambda: square_layout(C),
        "bip_wide": lambda: bipartite_layout(3000, 40, 2500, 41),       # n_src >> n_dst, E <= n_src
        "bip_narrow": lambda: bipartite_layout(40, 3000, 4000, 42),     # most targets empty, every source read often
        "no_edges": lambda: (np.zeros(0, np.int64), np.zeros(0, np.int64), 20, 30),
    }
    if name in ind:
        return (*ind[name](), True)
    return (*gen[name](), False)


PLANS = ["sizes", "sizes_perm", "straddle", "lanes", "no_nodes", "square", "bip_wide", "bip_narrow", "no_edges"]


def restated(name, C):
    s, t, ns, nd, indicator = layout(name, C)
    return Plan(s, t, ns, nd, C, indicator)


# ------------------------------------------------------------------------------------------------ data
def levels(rng, *shape):
    return rng.integers(-2, 3, shape) / 4


def f32(a):
    return np.asarray(a, np.float32) + np.float32(0)        # no -0


def set2set_inputs(kind, P, D, rng):
    ns, nd = P.n_src, P.n_dst
    if kind in ("randn", "sharp"):
        x = rng.standard_normal((ns, D))
        q = rng.standard_normal((nd, D)) / math.sqrt(D) * (25 if kind == "sharp" else 1)
    elif kind == "ties":
        x, q = levels(rng, ns, D), levels(rng, nd, D)
    elif kind in ("rising", "falling"):     # step > twice what the other columns can add: s rises at every edge
        q, x = levels(rng, nd, D), levels(rng, ns, D) / 4
        q[:, 0] = 1
        x[:, 0] = (D - 1) / 8 + 0.25
        x[:, 0] *= P.src_rank * (1 if kind == "rising" else -1)
    elif kind == "spread":                  # scores +-64: alpha underflows to 0 beside the max
        q = np.zeros((nd, D))
        q[:, 0] = 1
        x = levels(rng, ns, D)
        x[:, 0] = rng.choice([-64.0, 64.0], ns)
    else:                                   # equal: q = 0
        x, q = rng.standard_normal((ns, D)), np.zeros((nd, D))
    return f32(x), f32(q), f32(rng.standard_normal((nd, D)))


def pool_inputs(kind, P, D, rng):
    ns, nd = P.n_src, P.n_dst
    f = rng.standard_normal((ns, D))
    gate = {
        "randn": lambda: rng.standard_normal(ns),
        "sharp": lambda: 25 * rng.standard_normal(ns),
        "rising": lambda: 0.5 * P.src_rank,
        "falling": lambda: -0.5 * P.src_rank,
        "ties": lambda: levels(rng, ns),
        "spread": lambda: rng.choice([-64.0, 64.0], ns),
        # a constant per graph (indicator plans: source k is edge k), one constant on a general plan
        "equal": lambda: (0.25 * (P.t % 5) - 0.5) if P.indicator else np.full(ns, 0.75),
    }[kind]()
    return f32(f), f32(gate), f32(rng.standard_normal((nd, D)))


# ------------------------------------------------------------------------------------------------ checks
def within(got, ref, bound, what):
    """no NaN, +-Inf where ref has them, |got - ref| <= bound per element"""
    g64 = np.asarray(got).astype(np.float64)
    ref = np.asarray(ref, np.float64)
    assert not np.isnan(g64).any(), f"{what}: NaN at {np.argwhere(np.isnan(g64))[:4].tolist()}"
    inf = np.isinf(ref)
    assert (np.isinf(g64) == inf).all() and (g64[inf] == ref[inf]).all(), f"{what}: infinities differ"
    err = np.where(inf, 0.0, np.abs(g64 - np.where(inf, 0.0, ref)))
    ok = err <= np.broadcast_to(bound, err.shape)
    if not ok.all():
        bad = np.argwhere(~ok)
        i = tuple(bad[0])
        raise AssertionError(f"{what}: |got - ref| = {err[i]:.3e} > bound {np.broadcast_to(bound, err.shape)[i]:.3e} "
                             f"at {list(i)} ({len(bad)} elements; got {g64[i]!r}, ref {ref[i]!r})")


def bits(got, want, what, mask=None):
    got, want = np.ascontiguousarray(got, np.float32), np.ascontiguousarray(want, np.float32)
    diff = got.view(np.int32) != want.view(np.int32)
    if mask is not None:
        diff &= np.broadcast_to(mask.reshape(mask.shape + (1,) * (diff.ndim - mask.ndim)), diff.shape)
    if diff.any():
        i = tuple(np.argwhere(diff)[0])
        raise AssertionError(f"{what}: not the exact bits at {list(i)} ({int(diff.sum())} elements; got {got[i]!r}, "
                             f"want {want[i]!r})")


def check_outputs(P, entry, ins, outs, D):
    """outs (float32 arrays of the kernels or of the emulation) against the restatement: the bounds everywhere, the
    exact cases where the inputs make them so"""
    kind = ins["kind"]
    if entry == "set2set":
        x, q, dr = ins["x"], ins["q"], ins["dr"]
        sc, sigma = scores(P, x, q=q)
    else:
        x, gate, dr = ins["f"], ins["gate"], ins["du"]
        sc, sigma = scores(P, x, gate=gate)
        q = None
    F = forward64(P, x, sc)
    B = pullback64(P, x, F, dr, q)
    b = bounds(P, x, F, sigma, dr, B, q)
    w = f"{entry} {ins['what']}"
    within(outs["seg_sum"], F["S"], b["S"], w + " seg_sum")
    if entry == "pool":
        bits(outs["seg_max"], F["M"], w + " seg_max")              # the largest gate, -Inf without edges
    else:
        within(outs["seg_max"], F["M"], b["M"], w + " seg_max")
    within(outs["r"], F["r"], b["r"], w + (" r" if entry == "set2set" else " u"))
    if entry == "set2set":
        within(outs["dxe"], B["dxe"], b["dxe"], w + " dxe")
        within(outs["dq"], B["dq"], b["dq"], w + " dq")
    else:
        within(outs["dfe"], B["dfe"], b["dfe"], w + " dfe")
        within(outs["dgate"], B["dgate"], b["dgate"], w + " dgate_e")
    if kind == "equal":
        cnt = P.seg.deg.astype(np.float32)
        bits(outs["seg_sum"], cnt, w + " seg_sum = count")
        chunked = P.seg.scatter("+", x[P.s], np.float32)
        bits(outs["r"], chunked / np.maximum(cnt, 1)[:, None], w + " r = chunked sum / count", P.live)
        inv = P.row(np.float32(1) / np.maximum(cnt, 1))
        bits(outs["dxe" if entry == "set2set" else "dfe"], dr[P.t] * inv[:, None], w + " d = dr fl(1/n)")
    under = (F["d"] < UNDERFLOW) & (sigma == 0)
    if under.any():
        zero = outs["dxe" if entry == "set2set" else "dfe"][under]
        assert (zero == 0).all(), f"{w}: alpha underflows, yet d{'xe' if entry == 'set2set' else 'fe'} != 0"
        if entry == "pool":
            assert (outs["dgate"][under] == 0).all(), f"{w}: alpha underflows, yet dgate_e != 0"


# ------------------------------------------------------------------------------------------------ float32 emulation
def fma(a, b, c):
    return (np.asarray(a, np.float64) * np.asarray(b, np.float64) + np.asarray(c, np.float64)).astype(np.float32)


def dot32(a, b, vec):
    """<a, b> row by row as a warp forms it: lane l owns the slices (i 32 + l) of `vec` floats, an fma chain per lane,
    then the butterfly xor 16 .. 1"""
    m, D = a.shape
    K = -(-D // (32 * vec))
    pad = K * 32 * vec - D
    A = np.pad(a, ((0, 0), (0, pad))).reshape(m, K, 32, vec)
    Bv = np.pad(b, ((0, 0), (0, pad))).reshape(m, K, 32, vec)
    d = np.zeros((m, 32), np.float32)
    for i in range(K):
        for c in range(vec):
            d = fma(A[:, i, :, c], Bv[:, i, :, c], d)
    lane = np.arange(32)
    for o in (16, 8, 4, 2, 1):
        d = d + d[:, lane ^ o]
    return d[:, 0]


def pieces(P):
    """plan positions of each piece: (start, length) in chunk order"""
    start = np.flatnonzero(np.diff(np.concatenate([[-1], P.seg.piece])))
    return start, np.diff(np.concatenate([start, [P.E]]))


def emulate(P, entry, ins, vec, fixup_reverse=False):
    """the kernels' float32 operation order (module docstring); returns the outputs check_outputs takes"""
    seg, D = P.seg, ins["D"]
    order = seg.order
    if entry == "set2set":
        x, q, dr = ins["x"], ins["q"], ins["dr"]
        sc = dot32(q[P.t], x[P.s], vec) if P.E else np.zeros(0, np.float32)
    else:
        x, gate, dr = ins["f"], ins["gate"], ins["du"]
        sc = gate[P.s]
    st, ln = pieces(P)
    npc = len(st)
    M = np.full(npc, -np.inf, np.float32)
    S = np.zeros(npc, np.float32)
    acc = np.zeros((npc, D), np.float32)
    with np.errstate(over="ignore", invalid="ignore"):
        for j in range(int(ln.max()) if npc else 0):
            act = j < ln
            e = order[np.minimum(st + j, P.E - 1)]
            s, v = sc[e], x[P.s[e]]
            Mn = np.maximum(M, s)
            sc_ = np.exp(M - Mn)
            pp = np.exp(s - Mn)
            S = np.where(act, fma(S, sc_, pp), S)
            acc = np.where(act[:, None], fma(acc, sc_[:, None], v * pp[:, None]), acc)
            M = np.where(act, Mn, M)
        r = np.zeros((P.n_dst, D), np.float32)
        Mo = np.full(P.n_dst, -np.inf, np.float32)
        So = np.zeros(P.n_dst, np.float32)
        ps = seg.piece_seg
        whole = ~seg.long[ps]
        r[ps[whole]] = acc[whole] / S[whole][:, None]
        Mo[ps[whole]], So[ps[whole]] = M[whole], S[whole]
        rows = np.flatnonzero(seg.long)
        if rows.size:                       # gat_fwd_fixup_kernel: the slots in chunk order from M = -FLT_MAX
            lists = [np.flatnonzero(ps == i) for i in rows]
            if fixup_reverse:
                lists = [a[::-1] for a in lists]
            Mf = np.full(rows.size, -FLT_MAX, np.float32)
            Sf = np.zeros(rows.size, np.float32)
            af = np.zeros((rows.size, D), np.float32)
            for k in range(max(len(a) for a in lists)):
                act = np.array([k < len(a) for a in lists])
                p = np.array([a[min(k, len(a) - 1)] for a in lists])
                Mn = np.maximum(Mf, M[p])
                s0, s1 = np.exp(Mf - Mn), np.exp(M[p] - Mn)
                af = np.where(act[:, None], fma(af, s0[:, None], acc[p] * s1[:, None]), af)
                Sf = np.where(act, fma(Sf, s0, S[p] * s1), Sf)
                Mf = np.where(act, Mn, Mf)
            r[rows] = af / Sf[:, None]
            Mo[rows], So[rows] = Mf, Sf
        out = dict(r=r, seg_max=Mo, seg_sum=So)
        # pullback from the emulated forward
        al = (np.exp(sc - Mo[P.t]) / So[P.t]).astype(np.float32) if P.E else np.zeros(0, np.float32)
        T = dot32(dr, r, vec) if P.n_dst else np.zeros(0, np.float32)
        gd = dot32(dr[P.t], x[P.s], vec) if P.E else np.zeros(0, np.float32)
        ds = al * (gd - T[P.t])
        if entry == "pool":
            out["dfe"] = dr[P.t] * al[:, None]
            out["dgate"] = ds
            return out
        out["dxe"] = fma(dr[P.t], al[:, None], q[P.t] * ds[:, None])
        part = np.zeros((npc, D), np.float32)
        for j in range(int(ln.max()) if npc else 0):
            act = j < ln
            e = order[np.minimum(st + j, P.E - 1)]
            part = np.where(act[:, None], fma(x[P.s[e]], ds[e][:, None], part), part)
        dq = np.zeros((P.n_dst, D), np.float32)
        np.add.at(dq, ps, part)             # seg_fixup_kernel: the slots added in chunk order
        out["dq"] = dq
    return out


# ------------------------------------------------------------------------------------------------ case matrix
def _cases():
    rows = []
    i = 0
    for C in (128, 32):
        for name in PLANS:
            for kind in KINDS:
                D = WIDTHS[(i * 7) % len(WIDTHS)]
                rows.append((f"{name}@{C}", D, kind, 0))
                i += 1
    # the float4-capable widths at 4, 8 and 12 B from a 16 B boundary: the scalar path
    rows += [("sizes@128", 128, "equal", 4), ("straddle@32", 512, "rising", 8), ("square@128", 1024, "ties", 12),
             ("sizes_perm@32", 128, "spread", 12), ("bip_wide@32", 512, "equal", 4), ("lanes@128", 1024, "randn", 8),
             ("straddle@128", 128, "sharp", 8), ("square@32", 512, "randn", 12), ("bip_narrow@128", 1024, "equal", 4)]
    # one graph of 10^5 nodes between two small ones: ~780 / 3 125 pieces through the fix-ups
    rows += [("huge@32", 64, "randn", 0), ("huge@128", 33, "equal", 0), ("huge@32", 4, "ties", 4),
             ("huge@128", 1, "spread", 0), ("huge@32", 128, "equal", 0)]
    return rows


CASES = _cases()


def _split(plan):
    name, C = plan.split("@")
    return name, int(C)


def _inputs(entry, plan, D, kind, P):
    rng = np.random.default_rng(zlib.crc32(f"{entry} {plan} {D} {kind}".encode()))
    x, q, dr = (set2set_inputs if entry == "set2set" else pool_inputs)(kind, P, D, rng)
    keys = ("x", "q", "dr") if entry == "set2set" else ("f", "gate", "du")
    return dict(zip(keys, (x, q, dr)), kind=kind, D=D, what=f"{plan} D={D} {kind}")


def _id(c):
    plan, D, kind, off = c
    return f"{plan}-D{D}-{kind}" + (f"-off{off}" if off else "")


# ------------------------------------------------------------------------------------------------ CPU
AUTOGRAD_PLANS = ["square@32", "bip_wide@32", "bip_narrow@128", "sizes_perm@32", "no_edges@128"]


@pytest.mark.parametrize("plan", AUTOGRAD_PLANS)
@pytest.mark.parametrize("entry", ["set2set", "pool"])
def test_restatement_against_autograd(entry, plan):
    """forward64 == torch float64 and pullback64 == its autograd, per edge (x and the gate gathered per edge are the
    leaves, so their gradients are dxe / dfe and dgate_e), on tie-free data; empty targets give 0, -Inf and 0"""
    P = restated(*_split(plan))
    D = 5
    ins = _inputs(entry, plan, D, "randn", P)
    x, b, dr = (ins["x"], ins["q"], ins["dr"]) if entry == "set2set" else (ins["f"], ins["gate"], ins["du"])
    sc, _ = scores(P, x, **({"q": b} if entry == "set2set" else {"gate": b}))
    F = forward64(P, x, sc)
    B = pullback64(P, x, F, dr, b if entry == "set2set" else None)
    t = torch.as_tensor(P.t)
    xe = torch.as_tensor(x[P.s], dtype=torch.float64).requires_grad_(True)
    if entry == "set2set":
        lead = torch.as_tensor(b, dtype=torch.float64).requires_grad_(True)
        s = (lead[t] * xe).sum(1)
    else:
        lead = torch.as_tensor(b[P.s], dtype=torch.float64).requires_grad_(True)
        s = lead
    M = torch.full((P.n_dst,), -math.inf, dtype=torch.float64).scatter_reduce(0, t, s.detach(), "amax")
    w = torch.exp(s - M[t])
    S = torch.zeros(P.n_dst, dtype=torch.float64).index_add(0, t, w)
    r = torch.zeros(P.n_dst, D, dtype=torch.float64).index_add(0, t, w[:, None] * xe)
    r = r / torch.where(S > 0, S, torch.ones_like(S))[:, None]
    (r * torch.as_tensor(dr, dtype=torch.float64)).sum().backward()
    np.testing.assert_allclose(F["M"], M.numpy(), rtol=1e-14)
    np.testing.assert_allclose(F["S"], S.detach().numpy(), rtol=1e-13)
    np.testing.assert_allclose(F["r"], r.detach().numpy(), rtol=1e-12, atol=1e-13)
    assert (F["r"][~P.live] == 0).all() and (F["M"][~P.live] == -np.inf).all() and (F["S"][~P.live] == 0).all()
    if entry == "set2set":
        np.testing.assert_allclose(B["dxe"], xe.grad.numpy(), rtol=1e-10, atol=1e-12)
        np.testing.assert_allclose(B["dq"], lead.grad.numpy(), rtol=1e-10, atol=1e-12)
        assert (B["dq"][~P.live] == 0).all()
    else:
        np.testing.assert_allclose(B["dfe"], xe.grad.numpy(), rtol=1e-10, atol=1e-12)
        np.testing.assert_allclose(B["dgate"], lead.grad.numpy(), rtol=1e-10, atol=1e-12)


# the case matrix's shapes up to 260 floats (the emulation is a Python loop over the plan positions of a piece)
EMULATED = [c for c in CASES if c[1] <= 260 and not c[0].startswith("huge")]


@pytest.mark.parametrize("plan,D,kind,off", EMULATED, ids=[_id(c) for c in EMULATED])
@pytest.mark.parametrize("entry", ["set2set", "pool"])
def test_emulation_within_bounds(entry, plan, D, kind, off):
    """the float32 emulation of the kernels' operation order stays inside every bound, and gives the exact cases'
    bits"""
    P = restated(*_split(plan))
    ins = _inputs(entry, plan, D, kind, P)
    check_outputs(P, entry, ins, emulate(P, entry, ins, 4 if D % 4 == 0 and not off else 1), D)


@pytest.mark.parametrize("plan", ["straddle@32", "sizes@128"])
@pytest.mark.parametrize("entry", ["set2set", "pool"])
def test_planted_fixup_order_fails(entry, plan):
    """the pieces of the long rows combined in reverse chunk order: the exact sums of the equal-score case break"""
    P = restated(*_split(plan))
    assert (P.seg.chain - P.chunk >= 3).any()           # a row of three pieces or more: the order shows in the bits
    ins = _inputs(entry, plan, 64, "equal", P)
    check_outputs(P, entry, ins, emulate(P, entry, ins, 4), 64)
    with pytest.raises(AssertionError, match="chunked sum"):
        check_outputs(P, entry, ins, emulate(P, entry, ins, 4, fixup_reverse=True), 64)


@pytest.mark.parametrize("entry", ["set2set", "pool"])
def test_planted_alpha_error_fails(entry):
    """one alpha off by 2^-10 (in dxe / dfe = alpha dr + ...) breaks the bound"""
    P = restated("sizes", 128)
    ins = _inputs(entry, "sizes@128", 32, "randn", P)
    outs = emulate(P, entry, ins, 4)
    check_outputs(P, entry, ins, outs, 32)
    key, dr = ("dxe", ins["dr"]) if entry == "set2set" else ("dfe", ins["du"])
    k = int(np.flatnonzero(P.row(P.seg.deg) == 33)[5])
    outs[key][k] += dr[P.t[k]] * np.float32(2.0 ** -10)
    with pytest.raises(AssertionError, match=key):
        check_outputs(P, entry, ins, outs, 32)


# ------------------------------------------------------------------------------------------------ GPU
@pytest.fixture(scope="module")
def plans(gnn):
    """'name@chunk' -> (plan handle, Plan): indicator plans through readout._IndicatorPlan, general plans through
    gnnb_graph_create, each built at its chunk"""
    if not torch.cuda.is_available():
        pytest.skip("no CUDA device")
    lib, check = gnn._lib.lib, gnn._lib.check
    cache, raw = {}, []

    def get(plan):
        if plan not in cache:
            P = restated(*_split(plan))
            with chunk_set(gnn, P.chunk):
                if P.indicator:
                    keep = gnn.readout._IndicatorPlan(torch.as_tensor(P.t + 1), P.n_dst, torch.device("cuda"))
                    h = keep.plan.h
                else:
                    keep = h = raw_plan(lib, check, P.s + 1, P.t + 1, P.n_src, P.n_dst)
                    raw.append(h)
            cache[plan] = (h, P, keep)
        return cache[plan][:2]

    yield get
    cache.clear()
    for h in raw:
        lib.gnnb_graph_destroy(h)


def run_entry(gnn, h, P, entry, ins, off):
    """the forward, then the pullback on the forward's own outputs, every operand guarded; returns the outputs"""
    lib, check = gnn._lib.lib, gnn._lib.check
    st = torch.cuda.current_stream().cuda_stream
    D, E, nd = ins["D"], P.E, P.n_dst
    s2s = entry == "set2set"
    a, b, d = (ins["x"], ins["q"], ins["dr"]) if s2s else (ins["f"], ins["gate"], ins["du"])
    A, Bq = Guarded(a, off=off), Guarded(b, off=off)
    r, smax, ssum = (Guarded(n=nd * D, out=True, off=off), Guarded(n=nd, out=True, off=off),
                     Guarded(n=nd, out=True, off=off))
    fwd = lib.gnnb_set2set_attend if s2s else lib.gnnb_attention_pool
    check(fwd(h, A.ptr, Bq.ptr, D, r.ptr, smax.ptr, ssum.ptr, st))
    torch.cuda.synchronize()
    w = f"{entry} {ins['what']} offset={off}"
    for g, name in ((A, "x"), (Bq, "q / gate"), (r, "r / u"), (smax, "seg_max"), (smax, "seg_sum")):
        g.check(f"{w} forward {name}")
    kept = [g.raw.clone() for g in (r, smax, ssum)]
    dG = Guarded(d, off=off)
    de = Guarded(n=E * D, out=True, off=off)
    second = Guarded(n=nd * D if s2s else E, out=True, off=off)
    bwd = lib.gnnb_set2set_attend_bwd if s2s else lib.gnnb_attention_pool_bwd
    check(bwd(h, A.ptr, Bq.ptr, r.ptr, smax.ptr, ssum.ptr, dG.ptr, D, de.ptr, second.ptr, st))
    torch.cuda.synchronize()
    for g, name in ((A, "x"), (Bq, "q / gate"), (dG, "dr / du"), (de, "dxe / dfe"), (second, "dq / dgate_e")):
        g.check(f"{w} pullback {name}")
    for g, k in zip((r, smax, ssum), kept):
        assert torch.equal(g.raw, k), f"{w}: the pullback wrote into the forward's outputs"
    out = dict(r=r.get((nd, D)), seg_max=smax.get((nd,)), seg_sum=ssum.get((nd,)))
    if s2s:
        out.update(dxe=de.get((E, D)), dq=second.get((nd, D)))
    else:
        out.update(dfe=de.get((E, D)), dgate=second.get((E,)))
    return out


@pytest.mark.gpu
@pytest.mark.parametrize("plan,D,kind,off", CASES, ids=[_id(c) for c in CASES])
@pytest.mark.parametrize("entry", ["set2set", "pool"])
def test_entries_against_float64(gnn, plans, entry, plan, D, kind, off):
    """the four entries against the restatement: every element within its bound, the exact cases' bits, guards and
    coverage of every operand; pooling's forward and dfe off a 16 B boundary give the float4 path's bits"""
    h, P = plans(plan)
    ins = _inputs(entry, plan, D, kind, P)
    outs = run_entry(gnn, h, P, entry, ins, off)
    check_outputs(P, entry, ins, outs, D)
    if entry == "pool" and off and D % 4 == 0:
        ref = run_entry(gnn, h, P, entry, ins, 0)
        for k in ("r", "seg_max", "seg_sum", "dfe"):
            bits(outs[k], ref[k], f"pool {ins['what']}: {k} at offset {off} against the float4 path")
