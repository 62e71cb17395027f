"""gnnb_propagate, gnnb_propagate_bwd and their siblings called through the C ABI, against a plain float64 restatement of
include/gnnb200.h.

The Python layers pass only some of what the ABI allows; the Julia binding and the partition code pass the rest.  Here
every entry is called directly with:
  * node scales cs / ct that are absent, positive, or signed (negative entries, +0, -0, and one +Inf on a node with
    edges, compared with the IEEE rule of test_nonfinite.py: NaN masks and signed infinities exactly), in both
    directions of square and bipartite plans, forward and pullback;
  * operands at byte offsets 4, 8 and 12 from a 16 B boundary, which send every kernel of the family to its scalar
    code (the torch allocator alone never does);
  * every scale vector, weight vector, feature array and output inside a larger allocation whose guard regions hold NaN
    (inputs: a read outside the operand turns the result NaN) or a sentinel bit pattern (outputs: a write outside the
    operand changes it).  The guards are checked after every call, and so is that every output element was written.
The float64 reference is written from the header's formulas: m_e = w_e cs[s_e] x[s_e] for every edge in COO order,
out[t] = ct[t] AGG m over the in-edges of t (MEAN divides by their count first), rows without edges 0 / -Inf / +Inf.
The same code in float32 (each product, sum and quotient rounded in turn, the sums in COO order) gives the bits the
header promises for rows of at most `chunk` edges (max / min: every row).
"""
import ctypes as C
import random

import numpy as np
import pytest
import torch

from test_gpu_parity import GRAPHS, TOL, chunk_graph, fixture_plan, make_graph

pytestmark = pytest.mark.gpu

GRAD_TOL = 5e-6            # the pullbacks' bar in test_gpu_parity.py
PAD = 64                   # guard floats on either side of an operand (256 B: offset 0 stays 256 B-aligned)
NAN_BITS = 0x7FC00000
SENTINEL = 0x7FA5A5A5      # a NaN payload no kernel produces: an output element still holding it was never written
OK, EUNSUPPORTED = 0, 5
COPY_XJ, W_MUL_XJ = 0, 1
AGGR = {"sum": 0, "mean": 1, "max": 2, "min": 3}
SRC, DST = 0, 1

SQUARE = ["small", "empty_rows", "hubs", "sparse", "chunk_edges", "chunk32"]
# bipartite plans: a target hub and a source hub of 300 edges each (longer than the 128-edge chunk in both plans), the
# top fifth of the ids on either side without edges
BIPARTITE = {"bip_wide": (700, 160), "bip_narrow": (160, 700)}
GRAPH_NAMES = SQUARE + list(BIPARTITE) + ["no_edges"]


# ------------------------------------------------------------------------------------------------ graphs
class Graph:
    """0-based COO (s, t), the two node counts, the chunk and the plan handle"""

    def __init__(self, name, s, t, n_src, n_dst, chunk, h, keep=None, raw=False):
        self.name, self.s, self.t, self.n_src, self.n_dst = name, s, t, n_src, n_dst
        self.chunk, self.h, self.keep, self.raw = chunk, h, keep, raw

    def ends(self, transposed):
        """(gathered node of each edge, output row of each edge, gathered nodes, output rows)"""
        if transposed:
            return self.t, self.s, self.n_dst, self.n_src
        return self.s, self.t, self.n_src, self.n_dst


def raw_plan(lib, check, s, t, n_src, n_dst):
    """gnnb_graph_create straight from host 1-based int64 COO (num_src != num_dst allowed)"""
    h = C.c_void_p()
    s = np.ascontiguousarray(s, np.int64)
    t = np.ascontiguousarray(t, np.int64)
    check(lib.gnnb_graph_create(C.byref(h), s.ctypes.data, t.ctypes.data, len(s), n_src, n_dst, 8, 1, 0, None))
    return h.value


def bipartite_edges(rng, n_src, n_dst, E=2500, hub=300):
    hs, ht = int(n_src * 0.8), int(n_dst * 0.8)
    s = np.concatenate([rng.integers(1, hs + 1, E), rng.integers(1, hs + 1, hub), np.full(hub, 2)])
    t = np.concatenate([rng.integers(1, ht + 1, E), np.full(hub, 1), rng.integers(1, ht + 1, hub)])
    p = rng.permutation(len(s))
    return s[p].astype(np.int64), t[p].astype(np.int64)


@pytest.fixture(scope="module")
def graphs(gnn):
    if not torch.cuda.is_available():
        pytest.skip("no CUDA device")
    lib, check = gnn._lib.lib, gnn._lib.check
    cache = {}

    def get(name):
        if name in cache:
            return cache[name]
        rng = np.random.default_rng(100 + GRAPH_NAMES.index(name) if name in GRAPH_NAMES else 99)
        if name in SQUARE:
            kw = dict(GRAPHS[name])
            s, t = chunk_graph(rng, **kw) if "chunk" in kw else make_graph(rng, **kw)
            n = kw["n"]
            gg = fixture_plan(gnn, name, s, t, n)
            g = Graph(name, s - 1, t - 1, n, n, kw.get("chunk", 128), gg.plan().h, keep=gg)
        elif name == "hubs_loops":          # the hubs graph with self loops: every node has an in-edge (GCN's own c)
            gg = gnn.add_self_loops(get("hubs").keep)
            s, t = gg.s.cpu().numpy().astype(np.int64), gg.t.cpu().numpy().astype(np.int64)
            g = Graph(name, s - 1, t - 1, gg.num_nodes, gg.num_nodes, 128, gg.plan().h, keep=gg)
        elif name in BIPARTITE:
            n_src, n_dst = BIPARTITE[name]
            s, t = bipartite_edges(rng, n_src, n_dst)
            g = Graph(name, s - 1, t - 1, n_src, n_dst, 128, raw_plan(lib, check, s, t, n_src, n_dst), raw=True)
        else:                               # no_edges: 20 sources, 30 targets, E = 0
            e = np.zeros(0, np.int64)
            g = Graph(name, e, e, 20, 30, 128, raw_plan(lib, check, e, e, 20, 30), raw=True)
        cache[name] = g
        return g

    yield get
    for g in cache.values():
        if g.raw:
            lib.gnnb_graph_destroy(g.h)


@pytest.fixture
def variant(gnn):
    yield lambda v: gnn._lib.check(gnn._lib.lib.gnnb_set_kernel_variant(v))
    gnn._lib.lib.gnnb_set_kernel_variant(0)


# ------------------------------------------------------------------------------------------------ guarded operands
class Guarded:
    """an operand of `n` floats at byte offset `off` from a 256 B boundary, between two guard regions of PAD floats:
    NaN around an input, SENTINEL around (and, before the call, inside) an output"""

    def __init__(self, host=None, n=None, out=False, off=0):
        if host is not None:
            host = np.ascontiguousarray(host, np.float32)
            self.shape, n = host.shape, host.size
        else:
            self.shape = (n,)
        self.n, self.out, self.lo = n, out, PAD + off // 4
        self.raw = torch.full((2 * PAD + off // 4 + n,), SENTINEL if out else NAN_BITS, dtype=torch.int32, device="cuda")
        self.bits = self.raw[self.lo:self.lo + n]
        self.body = self.bits.view(torch.float32)
        if host is not None and not out:
            self.body.copy_(torch.from_numpy(host.ravel()))
        self.init = self.raw.cpu()

    @property
    def ptr(self):
        return self.body.data_ptr()

    def check(self, what):
        r = self.raw.cpu()
        if not self.out:
            assert torch.equal(r, self.init), f"{what}: an input (or its guard) was written"
            return
        guards = torch.cat([r[:self.lo], r[self.lo + self.n:]])
        assert (guards == SENTINEL).all(), f"{what}: a write outside the output"
        assert not (r[self.lo:self.lo + self.n] == SENTINEL).any(), f"{what}: an output element was never written"

    def untouched(self):
        return bool((self.raw.cpu() == SENTINEL).all())

    def get(self, shape):
        return self.body.cpu().numpy().reshape(shape)


def ptr(buf):
    return None if buf is None else buf.ptr


def guard(a, off=0):
    return None if a is None else Guarded(a, off=off)


# ------------------------------------------------------------------------------------------------ reference
def propagate_ref(g, transposed, msg, aggr, x, w, cs, ct, dtype=np.float64):
    """gnnb_propagate as the header states it.  float64: the reference; float32: each product, sum and quotient rounded
    in turn, the sums in COO order (np.add.at / maximum.at / minimum.at visit the edges in order)."""
    src, dst, _, n_out = g.ends(transposed)
    D = x.shape[1]
    deg = np.bincount(dst, minlength=n_out)
    live = deg > 0
    with np.errstate(all="ignore"):
        m = x.astype(dtype)[src]
        if cs is not None:
            m = m * cs.astype(dtype)[src][:, None]
        if msg == W_MUL_XJ:
            m = m * w.astype(dtype)[:, None]
        if aggr in ("sum", "mean"):
            out = np.zeros((n_out, D), dtype)
            np.add.at(out, dst, m)
            if aggr == "mean":
                out[live] = out[live] / deg[live].astype(dtype)[:, None]
        else:
            out = np.full((n_out, D), -np.inf if aggr == "max" else np.inf, dtype)
            (np.maximum if aggr == "max" else np.minimum).at(out, dst, m)
        if ct is not None:
            out[live] = out[live] * ct.astype(dtype)[live][:, None]
    return out


def pullback_ref(g, aggr, dout, x, w, cs, ct):
    """gnnb_propagate_bwd for SUM / MEAN (gnnb200.h): ct' = ct (/ in-degree for MEAN),
    dx[j] = cs[j] sum_{k: s_k = j} w_k ct'[t_k] dout[t_k] (0 for a source without out-edges),
    dw[k] = ct'[t_k] cs[s_k] <dout[t_k], x[s_k]>"""
    s, t = g.s, g.t
    E = len(s)
    deg = np.bincount(t, minlength=g.n_dst)
    ctp = np.ones(g.n_dst) if ct is None else ct.astype(np.float64)
    csv = np.ones(g.n_src) if cs is None else cs.astype(np.float64)
    wv = np.ones(E) if w is None else w.astype(np.float64)
    with np.errstate(all="ignore"):
        if aggr == "mean":
            ctp = ctp / np.maximum(deg, 1)
        d64 = dout.astype(np.float64)
        dx = np.zeros((g.n_src, dout.shape[1]))
        np.add.at(dx, s, d64[t] * (wv * ctp[t])[:, None])
        has = np.bincount(s, minlength=g.n_src) > 0
        dx[has] = dx[has] * csv[has][:, None]
        dw = ctp[t] * csv[s] * np.einsum("ed,ed->e", d64[t], x.astype(np.float64)[s])
    return dx, dw


def maxmin_pullback_ref(g, msg, dout, x, w, out_fwd):
    """NNlib's rule: every edge whose message equals its row's extremum (compared in float32, as the forward formed
    both) passes w_k dout[t_k] to x[s_k]"""
    s, t = g.s, g.t
    m = x[s] if msg == COPY_XJ else x[s] * w[:, None]
    wv = np.ones(len(s)) if msg == COPY_XJ else w.astype(np.float64)
    tie = m == out_fwd[t]
    dx = np.zeros((g.n_src, x.shape[1]))
    np.add.at(dx, s, np.where(tie, wv[:, None] * dout.astype(np.float64)[t], 0.0))
    return dx


def same(got, ref, tol, exact=None, rows=None, what=""):
    """NaN masks equal, +-Inf at the same places with the same signs, the finite entries within `tol` normwise, and equal
    to the float32 result `exact` where it is given (on the rows `rows`, default all)"""
    got = np.asarray(got)
    g64 = got.astype(np.float64)
    bad = np.argwhere(np.isnan(g64) != np.isnan(ref))
    assert bad.size == 0, f"{what}: NaN mask differs at {bad[:4].tolist()} (got {g64[tuple(bad[0])]}, ref {ref[tuple(bad[0])]})"
    inf = np.isinf(ref)
    bad = np.argwhere(np.isinf(g64) != inf)
    assert bad.size == 0, f"{what}: Inf mask differs at {bad[:4].tolist()} (got {g64[tuple(bad[0])]}, ref {ref[tuple(bad[0])]})"
    assert (g64[inf] == ref[inf]).all(), f"{what}: the sign of an infinity differs"
    fin = np.isfinite(ref)
    err = np.linalg.norm(g64[fin] - ref[fin]) / max(np.linalg.norm(ref[fin]), 1e-30)
    assert err <= tol, f"{what}: finite entries {err:.3e} > {tol:.0e}"
    if exact is not None:
        sel = fin if rows is None else fin & rows.reshape((-1,) + (1,) * (fin.ndim - 1))
        bad = np.argwhere(sel & (got != exact))
        assert bad.size == 0, f"{what}: not bit-exact at {bad[:4].tolist()} (got {got[tuple(bad[0])]!r}, " \
                              f"float32 reference {exact[tuple(bad[0])]!r})"


def scales(kind, n, deg, rng):
    """None, positive in [0.5, 1.5), or signed: both signs, +0 and -0 entries, and +Inf on the node of least positive
    degree (`deg` counts that node's edges in the role the vector plays)"""
    if kind == "none":
        return None
    v = rng.uniform(0.5, 1.5, n)
    if kind == "signed":
        v *= rng.choice([-1.0, 1.0], n)
        z = rng.random(n)
        v[z < 0.1] = 0.0
        v[(z >= 0.1) & (z < 0.2)] = -0.0
        if (deg > 0).any():
            v[np.argmin(np.where(deg > 0, deg, np.iinfo(np.int64).max))] = np.inf
    return v.astype(np.float32)


def weights(rng, E):
    """signed weights with some zeros"""
    w = rng.uniform(-1.5, 1.5, E)
    w[rng.random(E) < 0.1] = 0.0
    return w.astype(np.float32)


# ------------------------------------------------------------------------------------------------ case lists
def pairwise(axes, seed, required=()):
    """a seeded greedy covering list: every value of every axis meets every value of every other axis in some row"""
    names = list(axes)
    rnd = random.Random(seed)

    def pairs(row):
        return {(a, row[a], b, row[b]) for i, a in enumerate(names) for b in names[i + 1:]}

    todo = {(a, va, b, vb) for i, a in enumerate(names) for b in names[i + 1:] for va in axes[a] for vb in axes[b]}
    rows = []
    for r in required:
        rows.append(dict(r))
        todo -= pairs(r)
    while todo:
        cands = [{a: rnd.choice(axes[a]) for a in names} for _ in range(48)]
        best = max(cands, key=lambda r: len(pairs(r) & todo))
        if not pairs(best) & todo:
            a, va, b, vb = min(todo, key=repr)
            best[a], best[b] = va, vb
        rows.append(best)
        todo -= pairs(best)
    return rows


def case_id(r):
    return "-".join(f"{k}{v}" if k in ("D", "T") else str(v) for k, v in r.items())


FWD_AXES = dict(graph=GRAPH_NAMES, T=[0, 1], msg=["copy", "w"], aggr=list(AGGR), cs=["none", "pos", "signed"],
                ct=["none", "pos", "signed"], D=[1, 3, 4, 5, 127, 128, 129, 256, 512])
# the lean kernels serve max / min only without a gathered scale: ct of both signs there, at each of their widths
FWD_REQUIRED = [dict(graph=gname, T=tr, msg=("copy", "w")[tr], aggr=aggr, cs="none", ct="signed", D=D)
                for gname, D in (("hubs", 128), ("bip_wide", 256), ("bip_narrow", 512), ("chunk32", 128))
                for tr in (0, 1) for aggr in ("max", "min")]
FWD_CASES = [pytest.param(i, *r.values(), id=case_id(r)) for i, r in enumerate(pairwise(FWD_AXES, 1, FWD_REQUIRED))]

BWD_AXES = dict(graph=GRAPH_NAMES, aggr=["sum", "mean"], cs=["none", "pos", "signed"], ct=["none", "pos", "signed"],
                want=["dx_copy", "dx_w", "dw", "dx_dw"], D=[1, 3, 128, 129, 256, 512])
# MEAN with ct and weights: ct / deg is built in the plan's ws2 and the weights placed after it
BWD_REQUIRED = [dict(graph=gname, aggr="mean", cs=cs, ct=ct, want=want, D=D)
                for gname in ("hubs", "bip_wide", "bip_narrow")
                for cs, ct, want, D in (("none", "pos", "dx_w", 128), ("signed", "signed", "dx_dw", 3))]
BWD_CASES = [pytest.param(i, *r.values(), id=case_id(r)) for i, r in enumerate(pairwise(BWD_AXES, 2, BWD_REQUIRED))]

MAXMIN_AXES = dict(graph=GRAPH_NAMES, aggr=["max", "min"], msg=["copy", "w"], D=[1, 5, 128, 129, 256, 512])
MAXMIN_CASES = [pytest.param(i, *r.values(), id=case_id(r)) for i, r in enumerate(pairwise(MAXMIN_AXES, 3))]


# ------------------------------------------------------------------------------------------------ forward matrix
@pytest.mark.parametrize("seed,gname,transposed,msg,aggr,cs,ct,D", FWD_CASES)
def test_propagate_against_float64(graphs, gnn, variant, seed, gname, transposed, msg, aggr, cs, ct, D):
    """gnnb_propagate in either direction with node scales of every kind: the float64 reference at TOL, the float32
    sequential reference bit for bit where the header promises it, variant 0 == variant 12 bit for bit"""
    lib = gnn._lib.lib
    g = graphs(gname)
    src, dst, n_in, n_out = g.ends(transposed)
    rng = np.random.default_rng(1000 + seed)
    x = rng.standard_normal((n_in, D)).astype(np.float32)
    M = W_MUL_XJ if msg == "w" else COPY_XJ
    w = weights(rng, len(src)) if M == W_MUL_XJ else None
    csv = scales(cs, n_in, np.bincount(src, minlength=n_in), rng)      # gathered node: num_dst entries if transposed
    ctv = scales(ct, n_out, np.bincount(dst, minlength=n_out), rng)    # output row: num_src entries if transposed
    bits = {}
    for v in (12, 0):
        variant(v)
        ins = [guard(x), guard(w), guard(csv), guard(ctv)]
        out = Guarded(n=n_out * D, out=True)
        rc = lib.gnnb_propagate(g.h, transposed, M, AGGR[aggr], *map(ptr, ins), D, out.ptr, None)
        assert rc == OK, gnn._lib.lib.gnnb_last_error()
        for b in ins + [out]:
            if b is not None:
                b.check(f"variant {v}")
        bits[v] = out
    assert torch.equal(bits[0].bits, bits[12].bits), "lean kernel != seg_reduce_kernel"
    got = bits[0].get((n_out, D))
    ref = propagate_ref(g, transposed, M, aggr, x, w, csv, ctv)
    exact = propagate_ref(g, transposed, M, aggr, x, w, csv, ctv, np.float32)
    short = np.bincount(dst, minlength=n_out) <= g.chunk if aggr in ("sum", "mean") else None
    same(got, ref, TOL, exact, short, what=f"{gname} T={transposed} {msg} {aggr} cs={cs} ct={ct} D={D}")


# ------------------------------------------------------------------------------------------------ pullback matrix
@pytest.mark.parametrize("seed,gname,aggr,cs,ct,want,D", BWD_CASES)
def test_propagate_bwd_sum_mean_against_float64(graphs, gnn, seed, gname, aggr, cs, ct, want, D):
    """gnnb_propagate_bwd for SUM / MEAN with every combination of node scales: dx alone, dw alone and both"""
    lib = gnn._lib.lib
    g = graphs(gname)
    rng = np.random.default_rng(2000 + seed)
    E = len(g.s)
    x = rng.standard_normal((g.n_src, D)).astype(np.float32)
    dout = rng.standard_normal((g.n_dst, D)).astype(np.float32)
    M = COPY_XJ if want == "dx_copy" else W_MUL_XJ
    w = weights(rng, E) if M == W_MUL_XJ else None
    csv = scales(cs, g.n_src, np.bincount(g.s, minlength=g.n_src), rng)
    ctv = scales(ct, g.n_dst, np.bincount(g.t, minlength=g.n_dst), rng)
    ins = [guard(dout), guard(x), guard(w), guard(csv), guard(ctv)]
    dx = Guarded(n=g.n_src * D, out=True) if want != "dw" else None
    dw = Guarded(n=E, out=True) if want in ("dw", "dx_dw") else None
    rc = lib.gnnb_propagate_bwd(g.h, M, AGGR[aggr], *map(ptr, ins), None, D, ptr(dx), ptr(dw), None)
    assert rc == OK, lib.gnnb_last_error()
    for b in ins + [dx, dw]:
        if b is not None:
            b.check("pullback")
    dx_ref, dw_ref = pullback_ref(g, aggr, dout, x, w, csv, ctv)
    what = f"{gname} {aggr} cs={cs} ct={ct} D={D}"
    if dx is not None:
        same(dx.get((g.n_src, D)), dx_ref, GRAD_TOL, what="dx " + what)
    if dw is not None:
        same(dw.get((E,)), dw_ref, GRAD_TOL, what="dw " + what)


def tie_features(rng, n, D):
    """halves in [-3, 3]: many messages of a row are equal, so ties for the extremum are common"""
    return (rng.integers(-6, 7, (n, D)) / 2).astype(np.float32)


def tie_weights(rng, E):
    """exact binary fractions of both signs and zero: every product is exact"""
    return rng.choice(np.array([-2, -1, -0.5, 0, 0.5, 1, 2], np.float32), E)


@pytest.mark.parametrize("seed,gname,aggr,msg,D", MAXMIN_CASES)
def test_propagate_bwd_max_min_ties(graphs, gnn, seed, gname, aggr, msg, D):
    """gnnb_propagate_bwd for MAX / MIN: every tied extremum receives the gradient, with weights of both signs and zero
    and rows longer than the chunk"""
    lib = gnn._lib.lib
    g = graphs(gname)
    rng = np.random.default_rng(3000 + seed)
    x = tie_features(rng, g.n_src, D)
    M = W_MUL_XJ if msg == "w" else COPY_XJ
    w = tie_weights(rng, len(g.s)) if M == W_MUL_XJ else None
    out = Guarded(n=g.n_dst * D, out=True)
    gx, gw = guard(x), guard(w)
    assert lib.gnnb_propagate(g.h, 0, M, AGGR[aggr], gx.ptr, ptr(gw), None, None, D, out.ptr, None) == OK
    out_fwd = out.get((g.n_dst, D))
    same(out_fwd, propagate_ref(g, 0, M, aggr, x, w, None, None), 0.0, what="forward")
    dout = rng.standard_normal((g.n_dst, D)).astype(np.float32)
    ins = [guard(dout), gx, gw, guard(out_fwd)]
    dx = Guarded(n=g.n_src * D, out=True)
    rc = lib.gnnb_propagate_bwd(g.h, M, AGGR[aggr], ins[0].ptr, gx.ptr, ptr(gw), None, None, ins[3].ptr, D, dx.ptr,
                                None, None)
    assert rc == OK, lib.gnnb_last_error()
    for b in ins + [out, dx]:
        if b is not None:
            b.check("max/min pullback")
    same(dx.get((g.n_src, D)), maxmin_pullback_ref(g, M, dout, x, w, out_fwd), GRAD_TOL, what=f"dx {gname} {aggr} D={D}")


@pytest.mark.parametrize("gname", ["hubs", "bip_wide", "bip_narrow"])
@pytest.mark.parametrize("aggr", ["max", "min"])
def test_propagate_bwd_max_min_unsupported(graphs, gnn, gname, aggr):
    """dw, cs and ct with MAX / MIN: GNNB_EUNSUPPORTED, and nothing is written"""
    lib = gnn._lib.lib
    g = graphs(gname)
    D = 4
    rng = np.random.default_rng(7)
    x, dout = guard(rng.standard_normal((g.n_src, D))), guard(rng.standard_normal((g.n_dst, D)))
    of, w = guard(rng.standard_normal((g.n_dst, D))), guard(weights(rng, len(g.s)))
    cs, ct = guard(scales("pos", g.n_src, None, rng)), guard(scales("pos", g.n_dst, None, rng))
    for name, a_cs, a_ct, want_dw in (("dw", None, None, True), ("cs", cs, None, False), ("ct", None, ct, False),
                                      ("cs+ct", cs, ct, False)):
        dx = Guarded(n=g.n_src * D, out=True)
        dw = Guarded(n=len(g.s), out=True) if want_dw else None
        rc = lib.gnnb_propagate_bwd(g.h, W_MUL_XJ, AGGR[aggr], dout.ptr, x.ptr, w.ptr, ptr(a_cs), ptr(a_ct), of.ptr, D,
                                    dx.ptr, ptr(dw), None)
        assert rc == EUNSUPPORTED, (name, rc)
        torch.cuda.synchronize()
        assert dx.untouched() and (dw is None or dw.untouched()), name


# ------------------------------------------------------------------------------------------------ alignment
def scatter_ref(idx, n, aggr, m):
    out = np.zeros((n, m.shape[1])) if aggr in ("sum", "mean") else np.full((n, m.shape[1]), -np.inf if aggr == "max" else np.inf)
    m = m.astype(np.float64)
    if aggr in ("sum", "mean"):
        np.add.at(out, idx, m)
        if aggr == "mean":
            out = out / np.maximum(np.bincount(idx, minlength=n), 1)[:, None]
    else:
        (np.maximum if aggr == "max" else np.minimum).at(out, idx, m)
    return out


class Entry:
    """one C entry: its float inputs (host arrays), outputs (name -> shape), the call over pointers, the float64
    references (name -> (array, tol)) and the output rows on which a misaligned call must give the aligned call's bits"""

    def __init__(self, inputs, outputs, call, refs, same_bits=None):
        self.inputs, self.outputs, self.call, self.refs = inputs, outputs, call, refs
        self.same_bits = same_bits or {}

    def run(self, lib, offsets):
        ins = {k: Guarded(v, off=offsets.get(k, 0)) for k, v in self.inputs.items() if v is not None}
        outs = {k: Guarded(n=int(np.prod(shp)), out=True, off=offsets.get(k, 0)) for k, shp in self.outputs.items()}
        p = {k: b.ptr for k, b in {**ins, **outs}.items()}
        rc = self.call(p)
        assert rc == OK, lib.gnnb_last_error().decode()
        what = f"offsets {offsets}"
        for b in list(ins.values()) + list(outs.values()):
            b.check(what)
        return {k: outs[k].get(shp) for k, shp in self.outputs.items()}


def make_entry(lib, graphs, name, D, rng):
    g = graphs("hubs_loops" if name == "gcn_plan" else "hubs")
    s, t, n, E = g.s, g.t, g.n_src, len(g.s)
    x = rng.standard_normal((n, D)).astype(np.float32)
    w = weights(rng, E)
    cs, ct = scales("signed", n, np.bincount(s, minlength=n), rng), scales("pos", n, None, rng)
    out_rows = (n, D)
    if name.startswith("gather"):
        idx = s if name == "gather_src" else t
        which = SRC if name == "gather_src" else DST
        return Entry(dict(x=x), dict(out=(E, D)), lambda p: lib.gnnb_gather(g.h, which, p["x"], D, p["out"], None),
                     dict(out=(x[idx].astype(np.float64), 0.0)))
    if name.startswith("scatter"):
        _, end, aggr = name.split("_")
        m = rng.standard_normal((E, D)).astype(np.float32)
        idx, which = (s, SRC) if end == "src" else (t, DST)
        return Entry(dict(m=m), dict(out=out_rows),
                     lambda p: lib.gnnb_scatter(g.h, which, AGGR[aggr], p["m"], D, p["out"], None),
                     dict(out=(scatter_ref(idx, n, aggr, m), TOL)))
    if name.startswith("propagate"):
        _, aggr, *tr = name.split("_")
        T = 1 if tr else 0
        csv = cs if aggr == "sum" else None        # the lean kernels serve mean / max / min without a gathered scale
        return Entry(dict(x=x, w=w, cs=csv, ct=ct), dict(out=out_rows),
                     lambda p: lib.gnnb_propagate(g.h, T, W_MUL_XJ, AGGR[aggr], p["x"], p["w"], p.get("cs"), p["ct"], D,
                                                  p["out"], None),
                     dict(out=(propagate_ref(g, T, W_MUL_XJ, aggr, x, w, csv, ct), TOL)))
    if name.startswith("halo"):
        aggr = name.split("_")[1]
        nl = n // 3
        csv = cs if aggr == "sum" else None
        return Entry(dict(xl=x[:nl], xh=x[nl:], w=w, cs=csv, ct=ct), dict(out=out_rows),
                     lambda p: lib.gnnb_propagate_halo(g.h, W_MUL_XJ, AGGR[aggr], p["xl"], p["xh"], nl, p["w"],
                                                       p.get("cs"), p["ct"], D, p["out"], None),
                     dict(out=(propagate_ref(g, 0, W_MUL_XJ, aggr, x, w, csv, ct), TOL)))
    if name.startswith("gcn"):
        T = 1 if name == "gcn_T" else 0
        if name == "gcn_plan":      # the plan-owned c = 1 / sqrt(in-degree) and its per-edge stream
            c = (1 / np.sqrt(np.bincount(t, minlength=n))).astype(np.float32)
            return Entry(dict(x=x), dict(out=out_rows),
                         lambda p: lib.gnnb_gcn_propagate(g.h, 0, p["x"], None, None, D, p["out"], None),
                         dict(out=(propagate_ref(g, 0, COPY_XJ, "sum", x, None, c, c), TOL)))
        c = scales("pos", n, None, rng)
        return Entry(dict(x=x, w=w, c=c), dict(out=out_rows),
                     lambda p: lib.gnnb_gcn_propagate(g.h, T, p["x"], p["w"], p["c"], D, p["out"], None),
                     dict(out=(propagate_ref(g, T, W_MUL_XJ, "sum", x, w, c, c), TOL)))
    if name in ("bwd_sum", "bwd_mean"):
        aggr = name.split("_")[1]
        dout = rng.standard_normal((n, D)).astype(np.float32)
        ctv = scales("signed", n, np.bincount(t, minlength=n), rng)
        dx_ref, dw_ref = pullback_ref(g, aggr, dout, x, w, cs, ctv)
        return Entry(dict(dout=dout, x=x, w=w, cs=cs, ct=ctv), dict(dx=(n, D), dw=(E,)),
                     lambda p: lib.gnnb_propagate_bwd(g.h, W_MUL_XJ, AGGR[aggr], p["dout"], p["x"], p["w"], p["cs"],
                                                      p["ct"], None, D, p["dx"], p["dw"], None),
                     dict(dx=(dx_ref, GRAD_TOL), dw=(dw_ref, GRAD_TOL)))
    # bwd_max / bwd_min: the forward output from an aligned call; the warp-per-row fallback sums a source's out-edges
    # serially where the lean pullback sums a long row in pieces, so only rows of at most `chunk` edges keep their bits
    aggr = name.split("_")[1]
    x, w = tie_features(rng, n, D), tie_weights(rng, E)
    out = Guarded(n=n * D, out=True)
    gx, gw = Guarded(x), Guarded(w)
    assert lib.gnnb_propagate(g.h, 0, W_MUL_XJ, AGGR[aggr], gx.ptr, gw.ptr, None, None, D, out.ptr, None) == OK
    of = out.get((n, D))
    dout = rng.standard_normal((n, D)).astype(np.float32)
    return Entry(dict(dout=dout, x=x, w=w, of=of), dict(dx=(n, D)),
                 lambda p: lib.gnnb_propagate_bwd(g.h, W_MUL_XJ, AGGR[aggr], p["dout"], p["x"], p["w"], None, None,
                                                  p["of"], D, p["dx"], None, None),
                 dict(dx=(maxmin_pullback_ref(g, W_MUL_XJ, dout, x, w, of), GRAD_TOL)),
                 same_bits=dict(dx=np.bincount(s, minlength=n) <= g.chunk))


ENTRIES = ["gather_src", "gather_dst"] + [f"scatter_{e}_{a}" for e in ("src", "dst") for a in AGGR] + \
          ["propagate_sum", "propagate_sum_T", "propagate_mean", "propagate_max", "propagate_min",
           "halo_sum", "halo_max", "gcn", "gcn_T", "gcn_plan", "bwd_sum", "bwd_mean", "bwd_max", "bwd_min"]


@pytest.mark.parametrize("D", [128, 256, 512, 132])
@pytest.mark.parametrize("entry", ENTRIES)
def test_misaligned_operands(graphs, gnn, entry, D):
    """Each float operand alone, then all of them, at byte offsets 4, 8 and 12 (the scalar code of every kernel in the
    family): the aligned call's bits (rows of at most `chunk` edges for the max / min pullback, every row elsewhere: the
    fused reduce cuts long rows at the same chunk boundaries in every kernel) and the float64 reference everywhere."""
    lib = gnn._lib.lib
    e = make_entry(lib, graphs, entry, D, np.random.default_rng(D))
    base = e.run(lib, {})
    for k, (ref, tol) in e.refs.items():
        same(base[k], ref, tol, what=f"{entry} aligned {k}")
    names = [k for k, v in e.inputs.items() if v is not None] + list(e.outputs)
    for off in (4, 8, 12):
        for group in [[k] for k in names] + [names]:
            offsets = {k: off for k in group}
            got = e.run(lib, offsets)
            for k, (ref, tol) in e.refs.items():
                rows = e.same_bits.get(k)
                a, b = got[k], base[k]
                sel = np.ones(a.shape[0], bool) if rows is None else rows
                assert np.array_equal(a[sel].view(np.int32), b[sel].view(np.int32)), \
                    f"{entry} {k} at {offsets}: not the aligned call's bits"
                same(a, ref, tol, what=f"{entry} {k} at {offsets}")
