"""NaN, infinities and float32 overflow through the kernels, against the reference's IEEE results.

Reference semantics (the reference runs in Float32 with Julia's rules), written once below and evaluated in float64:
  * `max` and `min` return NaN when either argument is NaN (NNlib.scatter(max / min) and softmax's max fold with them);
  * relu(NaN) = NaN (NNlib's relu is max(0, x));
  * values that overflow Float32 (the logits el + er and <q, x>, the messages w * x, the sums of a row) are formed in
    float32 first, as the kernels and the reference's Float32 arithmetic form them; everything after that runs in
    float64, which would otherwise never overflow.
`same()` compares NaN masks and the positions and signs of the infinities exactly, then the finite entries with the bars
of test_gpu_parity.py.  Values are planted at the first, a middle and the last edge of rows, at the first edge of a
long-row piece (rows longer than the plan's chunk are reduced in pieces and merged by a fix-up) and in a row whose
logits are all -Inf, on the hubs / chunk_edges / chunk32 graphs of test_gpu_parity.py.
"""
import numpy as np
import pytest
import torch

from test_gpu_parity import GRAPHS, build_graph, jl, np_rows

F32MAX = float(np.finfo(np.float32).max)
BIG = 3e38                                  # finite; two of them overflow a float32 sum or product
PLANT_GRAPHS = ["hubs", "chunk_edges", "chunk32"]


# ------------------------------------------------------------------------------------------ reference semantics
def scatter64(aggr, m, idx, n):
    """NNlib.scatter(aggr, m, idx) on rows in float64 (idx 1-based).  np.maximum / np.minimum propagate NaN like Julia's
    max / min.  A sum beyond the float32 range becomes +-Inf, as the reference's float32 sum does (the tests plant
    overflowing values of one sign per column, so the order of the float32 sum cannot matter)."""
    m = np.asarray(m, np.float64)
    shape = (n,) + m.shape[1:]
    with np.errstate(all="ignore"):
        if aggr in ("+", "mean"):
            out = np.zeros(shape)
            np.add.at(out, idx - 1, m)
            out = np.where(np.abs(out) > F32MAX, np.sign(out) * np.inf, out)
            if aggr == "mean":
                cnt = np.maximum(np.bincount(idx - 1, minlength=n), 1).astype(np.float64)
                out = out / cnt.reshape((n,) + (1,) * (m.ndim - 1))
            return out
        out = np.full(shape, -np.inf if aggr == "max" else np.inf)
        (np.maximum if aggr == "max" else np.minimum).at(out, idx - 1, m)
        return out


def f32(a):
    """round to float32 (overflow to +-Inf) and continue in float64"""
    with np.errstate(over="ignore"):
        return np.asarray(a, np.float64).astype(np.float32).astype(np.float64)


def softmax64(u, t, n):
    """softmax_edge_neighbors: max, exp, sum, divide (GNNlib/src/utils.jl:84-97) on logits u (E, ...)"""
    with np.errstate(all="ignore"):
        ex = np.exp(u - scatter64("max", u, t, n)[t - 1])
        return ex / scatter64("+", ex, t, n)[t - 1]


def relu64(y):
    return np.maximum(y, 0.0)            # NaN stays NaN


def same(got, ref, tol=2e-6, exact=None, what=""):
    """NaN masks equal; +-Inf at the same places with the same signs; finite entries within `tol` normwise, and equal to
    `exact` (a float32 result) bit for bit where it is given"""
    got = np.asarray(got, np.float64)
    ref = np.asarray(ref, np.float64)
    assert got.shape == ref.shape, what
    bad = np.argwhere(np.isnan(got) != np.isnan(ref))
    assert bad.size == 0, f"{what}: NaN mask differs at {bad[:4].tolist()} (got {got[tuple(bad[0])]}, ref {ref[tuple(bad[0])]})"
    inf = np.isinf(ref)
    bad = np.argwhere(np.isinf(got) != inf)
    assert bad.size == 0, f"{what}: Inf mask differs at {bad[:4].tolist()} (got {got[tuple(bad[0])]}, ref {ref[tuple(bad[0])]})"
    assert (got[inf] == ref[inf]).all(), f"{what}: sign of an infinity differs"
    fin = np.isfinite(ref)
    if exact is not None:
        exact = np.asarray(exact, np.float64)
        assert (got[fin] == exact[fin]).all(), f"{what}: not bit-exact"
    err = np.linalg.norm(got[fin] - ref[fin]) / max(np.linalg.norm(ref[fin]), 1e-30)
    assert err <= tol, f"{what}: finite entries {err:.3e} > {tol:.0e}"


def bits_equal(a, b):
    """torch.equal with NaN == NaN (same bits)"""
    return torch.equal(a.contiguous().view(torch.int32), b.contiguous().view(torch.int32))


# ------------------------------------------------------------------------------------------ where to plant
def plant_sites(s, t, n, chunk):
    """COO ids of edges at the places where a kernel's running state is fresh or merged: the first, a middle and the last
    edge of three short rows (and the second edge of the first), the first edge of a long row and the first edge of one
    of its later pieces; also the edges of a long row's first piece and of a short row, all of which get the value"""
    order = np.argsort(t, kind="stable")
    deg = np.bincount(t - 1, minlength=n)
    rowptr = np.concatenate([[0], np.cumsum(deg)])
    short = [r for r in range(n) if 3 <= deg[r] <= chunk]
    long_ = [r for r in range(n) if deg[r] > chunk and (rowptr[r] // chunk + 1) * chunk < rowptr[r + 1]]
    assert len(short) >= 4 and len(long_) >= 2
    a, b, c, d = short[:4]
    L, L2 = long_[0], long_[1]
    piece = (rowptr[L] // chunk + 1) * chunk                       # a chunk boundary inside row L
    return dict(first=order[rowptr[a]], second=order[rowptr[a] + 1], middle=order[rowptr[b] + deg[b] // 2],
                last=order[rowptr[c + 1] - 1],
                long_first=order[rowptr[L]], piece=order[piece],
                piece_all=order[rowptr[L2]:(rowptr[L2] // chunk + 1) * chunk],   # the whole first piece of row L2
                row_all=order[rowptr[d]:rowptr[d + 1]], rows=dict(a=a, b=b, c=c, d=d, L=L, L2=L2))


@pytest.fixture(scope="module", params=PLANT_GRAPHS)
def pgraph(request, gnn):
    name, s, t, n, g = build_graph(gnn, request.param)
    return name, s, t, n, g, plant_sites(s, t, n, GRAPHS[name].get("chunk", 128))


# ------------------------------------------------------------------------------------------ CPU: oracle and fake ABI
def test_oracle_max_min_follow_julia_nan_rule(oracle):
    """NaN first, in the middle, last, alone, and beside +-Inf: the row is NaN wherever the NaN sits"""
    t = np.array([1, 1, 1, 2, 2, 2, 3, 3, 3, 4, 5, 5], np.int64)
    col = np.array([[np.nan, 1, 2, 3, 1, np.nan, 1, 2, np.nan, np.nan, np.inf, -np.inf]]).T
    col2 = np.array([[1, 2, 3, 3, 1, 2, np.inf, -np.inf, 0, 5, 1, np.nan]]).T
    for e in (col, col2, np.hstack([col, col2])):
        for aggr in ("max", "min"):
            for T in (np.float64, np.float32):
                got = oracle.scatter(aggr, e.astype(T), t, 6)
                same(got, scatter64(aggr, e, t, 6), tol=0, what=f"oracle {aggr} {T.__name__}")


def test_max_min_nan_rule_through_propagate(be, gnn):
    """the fused propagate with max / min on the fake ABI (numpy) and on the GPU: a NaN message makes its row NaN"""
    s = np.array([1, 2, 3, 4, 1, 2, 5, 3, 4], np.int64)
    t = np.array([2, 2, 2, 3, 3, 3, 4, 4, 4], np.int64)
    x = np.array([[np.nan, 1.0, 2.0], [1.0, np.nan, -np.inf], [3.0, 4.0, np.nan], [0.5, np.inf, 1.0],
                  [-1.0, -2.0, -3.0]], np.float32)
    g = gnn.GNNGraph(s, t, num_nodes=5).to(be.dev)
    for aggr in ("max", "min"):
        got = np_rows(gnn.propagate(gnn.copy_xj, g, aggr, xj=jl(x, be.dev)))
        same(got, scatter64(aggr, x[s - 1], t, 5), tol=0, what=aggr)


# ------------------------------------------------------------------------------------------ fused propagate
KINDS = [np.nan, np.inf, -np.inf, BIG, -BIG]         # column k of the features carries kind k (D >= 5)


def planted_features(rng, n, D, s, sites):
    x = rng.standard_normal((n, D)).astype(np.float32)
    for k, v in enumerate(KINDS):
        col = k if D >= 5 else (0, 1, 2, 1, 2)[k]          # D = 3: +-BIG share a column with the infinity of its sign
        for pos in ("first", "middle", "last", "long_first", "piece"):
            x[s[sites[pos]] - 1, col] = v
        if abs(v) == BIG:                                  # a second one in the row of the first: its sum overflows
            x[s[sites["second"]] - 1, col] = v
    x[s[sites["second"]] - 1, 0] = np.nan                  # as at every planted source: dw is NaN there, never a
    return x                                               # float32 overflow whose place depends on the order


@pytest.mark.gpu
@pytest.mark.parametrize("aggr", ["+", "mean", "max", "min"])
@pytest.mark.parametrize("D", [3, 16, 128, 256, 512])
def test_propagate_nonfinite(pgraph, oracle, gnn, aggr, D):
    """copy_xj and w_mul_xj with NaN, +-Inf and overflowing +-3e38 features; the lean kernels (variant 0) and
    seg_reduce_kernel (variant 12) give the same bits; the pullbacks"""
    name, s, t, n, g, sites = pgraph
    lib = gnn._lib.lib
    rng = np.random.default_rng(D)
    x = planted_features(rng, n, D, s, sites)
    w = (rng.random(len(s)) + 0.6).astype(np.float32)          # > 0: a product keeps its sign and may overflow
    gw = gnn.set_edge_weight(g, torch.as_tensor(w).cuda())
    try:
        outs = {}
        for v in (12, 0):
            gnn._lib.check(lib.gnnb_set_kernel_variant(v))
            outs[v] = (gnn.propagate(gnn.copy_xj, g, aggr, xj=jl(x)), gnn.propagate(gnn.w_mul_xj, gw, aggr, xj=jl(x)))
    finally:
        lib.gnnb_set_kernel_variant(0)
    for a, b in zip(outs[0], outs[12]):
        assert bits_equal(a, b), "lean kernel != seg_reduce_kernel"
    m_copy = x[s - 1].astype(np.float64)
    m_w = f32(w[:, None].astype(np.float64) * x[s - 1])           # the product is formed in float32
    for got, m, w32 in ((outs[0][0], m_copy, None), (outs[0][1], m_w, w)):
        ref = scatter64(aggr, m, t, n)
        exact = oracle.propagate_unfused(aggr, s, t, n, x, w32) if aggr in ("max", "min") else None
        same(np_rows(got), ref, exact=exact, what=f"{aggr} weighted={w32 is not None}")

    # pullbacks: + / mean weighted (dx and dw), max / min (dx; no gradient through a non-finite output, as in
    # test_gpu_parity.py)
    dout = rng.standard_normal((n, D)).astype(np.float32)
    xt = jl(x).requires_grad_(True)
    if aggr in ("+", "mean"):
        wt = torch.as_tensor(w).cuda().requires_grad_(True)
        y = gnn.propagate(gnn.e_mul_xj, g, aggr, xj=xt, e=wt)
        y.backward(jl(dout))
        cnt = np.maximum(np.bincount(t - 1, minlength=n), 1).astype(np.float64) if aggr == "mean" else np.ones(n)
        dm = dout.astype(np.float64)[t - 1] / cnt[t - 1][:, None]
        same(np_rows(xt.grad), scatter64("+", dm * w[:, None], s, n), tol=5e-6, what="dx")
        with np.errstate(all="ignore"):
            dw_ref = (dm * x[s - 1]).sum(1)
        same(wt.grad.cpu().numpy(), dw_ref, tol=5e-6, what="dw")
    else:
        y = gnn.propagate(gnn.copy_xj, g, aggr, xj=xt)
        yr = np_rows(y)
        dd = np.where(np.isfinite(yr), dout, 0).astype(np.float32)
        y.backward(jl(dd))
        with np.errstate(invalid="ignore"):
            dm = dd.astype(np.float64)[t - 1] * (m_copy == yr.astype(np.float64)[t - 1])
        same(np_rows(xt.grad), scatter64("+", dm, s, n), tol=5e-6, what="dx")


@pytest.mark.gpu
def test_aggregate_and_softmax_edge_neighbors_nonfinite(pgraph, gnn):
    """aggregate_neighbors (scatter of edge features) and softmax_edge_neighbors with NaN, +-Inf and -Inf first logits"""
    name, s, t, n, g, sites = pgraph
    rng = np.random.default_rng(1)
    E, K = len(s), 5
    e = rng.standard_normal((E, K)).astype(np.float32)
    for k, v in enumerate(KINDS):
        for pos in ("first", "middle", "last", "long_first", "piece"):
            e[sites[pos], k] = v
    for aggr in ("+", "max", "min"):
        same(np_rows(gnn.aggregate_neighbors(g, aggr, jl(e))), scatter64(aggr, e, t, n), what=aggr,
             exact=scatter64(aggr, e, t, n) if aggr != "+" else None)
    # logits: -Inf at the planted places in column 0, a row of -Inf in column 1, NaN in column 2
    z = (3 * rng.standard_normal((E, 3))).astype(np.float32)
    for pos in ("first", "middle", "last", "long_first", "piece"):
        z[sites[pos], 0] = -np.inf
    z[sites["piece_all"], 0] = -np.inf
    z[sites["row_all"], 1] = -np.inf
    z[sites["middle"], 2] = np.nan
    got = np_rows(gnn.softmax_edge_neighbors(g, jl(z)))
    same(got, softmax64(z.astype(np.float64), t, n), what="softmax_edge_neighbors")


# ------------------------------------------------------------------------------------------ GAT
GAT_CASES = [(16, 8, 0), (32, 4, 0), (64, 8, 0), (16, 8, 12), (8, 2, 0), (2, 3, 0), (4, 32, 12)]   # (C, H, variant)


def gat_logits(s, t, n, H, sites, rng):
    """el, er whose sum overflows to -Inf (both -3e38, finite) on the planted edges of every head; row d all -Inf"""
    el = rng.standard_normal((n, H)).astype(np.float32)
    er = rng.standard_normal((n, H)).astype(np.float32)
    for pos in ("first", "middle", "last", "long_first", "piece"):
        k = sites[pos]
        el[t[k] - 1] = -BIG
        er[s[k] - 1] = -BIG
    el[t[sites["piece_all"][0]] - 1] = -BIG
    er[s[sites["piece_all"]] - 1] = -BIG
    el[sites["rows"]["d"]] = -np.inf
    return el, er


@pytest.mark.gpu
@pytest.mark.parametrize("Cc,H,variant", GAT_CASES)
def test_gat_aggregate_nonfinite(pgraph, gnn, Cc, H, variant):
    """gnnb_gat_aggregate and its pullback with logits el + er that overflow to -Inf at the first, a middle and the last
    edge of rows, at a long row's first edge and piece boundary, over the whole first piece of a long row, and a row of
    -Inf logits (NaN there in the reference).  alpha (gat_alpha_kernel) and the pullback recompute α from the forward's
    seg_max and seg_sum, so those are checked through them and directly on the finite rows."""
    name, s, t, n, g, sites = pgraph
    lib = gnn._lib.lib
    rng = np.random.default_rng(Cc * 10 + H)
    Wx = rng.standard_normal((n, H, Cc)).astype(np.float32)
    dout = rng.standard_normal((n, H, Cc)).astype(np.float32)
    el, er = gat_logits(s, t, n, H, sites, rng)
    slope = 0.2
    with np.errstate(all="ignore"):
        z = f32(el[t - 1].astype(np.float32) + er[s - 1].astype(np.float32))
        u = np.where(z > 0, z, slope * z)
        M = scatter64("max", u, t, n)
        alpha = softmax64(u, t, n)
        Ssum = scatter64("+", np.exp(u - M[t - 1]), t, n)
        W64, d64 = Wx.astype(np.float64), dout.astype(np.float64)
        o_ref = scatter64("+", alpha[:, :, None] * W64[s - 1], t, n)
        dalpha = (d64[t - 1] * W64[s - 1]).sum(-1)
        T = scatter64("+", alpha * dalpha, t, n)
        dz = alpha * (dalpha - T[t - 1]) * np.where(z > 0, 1.0, slope)
        del_ref, der_ref = scatter64("+", dz, t, n), scatter64("+", dz, s, n)
        dWx_ref = scatter64("+", alpha[:, :, None] * d64[t - 1], s, n)
    dev = lambda a: torch.as_tensor(a).cuda().contiguous()
    Wx_d, el_d, er_d, do_d = dev(Wx), dev(el), dev(er), dev(dout)
    out = torch.empty_like(Wx_d); al = torch.empty(len(s), H, device="cuda")
    smax = torch.empty(n, H, device="cuda"); ssum = torch.empty(n, H, device="cuda")
    dWx = torch.empty_like(Wx_d); del_ = torch.empty(n, H, device="cuda"); der = torch.empty(n, H, device="cuda")
    p = g.plan()
    try:
        gnn._lib.check(lib.gnnb_set_kernel_variant(variant))
        gnn._lib.check(lib.gnnb_gat_aggregate(p.h, Wx_d.data_ptr(), el_d.data_ptr(), er_d.data_ptr(), Cc, H, slope,
                                              out.data_ptr(), al.data_ptr(), smax.data_ptr(), ssum.data_ptr(), None))
        gnn._lib.check(lib.gnnb_gat_aggregate_bwd(p.h, Wx_d.data_ptr(), el_d.data_ptr(), er_d.data_ptr(),
                                                  smax.data_ptr(), ssum.data_ptr(), out.data_ptr(), do_d.data_ptr(),
                                                  Cc, H, slope, dWx.data_ptr(), del_.data_ptr(), der.data_ptr(), None))
    finally:
        lib.gnnb_set_kernel_variant(0)
    same(out.cpu().numpy(), o_ref, tol=5e-6, what="out")
    same(al.cpu().numpy(), alpha, tol=5e-6, what="alpha")
    has = np.bincount(t - 1, minlength=n) > 0
    fin = has[:, None] & np.isfinite(M)
    same(smax.cpu().numpy()[fin], M[fin], tol=1e-6, what="seg_max")
    same(ssum.cpu().numpy()[fin], Ssum[fin], tol=5e-6, what="seg_sum")
    same(dWx.cpu().numpy(), dWx_ref, tol=1e-5, what="dWx")
    scale = max(np.linalg.norm(dWx_ref[np.isfinite(dWx_ref)]) / np.sqrt(dWx_ref.size) * np.sqrt(Cc), 1)
    for got, ref, what in ((del_, del_ref, "del"), (der, der_ref, "der")):
        got = got.cpu().numpy()
        same(got, ref, tol=np.inf, what=what)                       # masks; the bar below as in test_gpu_parity.py
        f = np.isfinite(ref)
        assert np.abs(got[f] - ref[f]).max() < 2e-4 * scale, what


# ------------------------------------------------------------------------------------------ Set2Set
@pytest.mark.gpu
@pytest.mark.parametrize("D", [4, 16, 130, 512])
def test_set2set_attend_nonfinite(pgraph, gnn, D):
    """gnnb_set2set_attend with <q, x> overflowing to -Inf (two -3e38 products, finite inputs) at the planted edges and
    on every edge of one row (NaN there in the reference)"""
    name, s, t, n, g, sites = pgraph
    rng = np.random.default_rng(D)
    x = (rng.standard_normal((n, D)) / np.sqrt(D)).astype(np.float32)
    q = rng.standard_normal((n, D)).astype(np.float32)
    q[:, :2] = 1.0
    for pos in ("first", "middle", "last", "long_first", "piece"):
        x[s[sites[pos]] - 1, :2] = -BIG
    x[s[sites["row_all"]] - 1, :2] = -BIG
    with np.errstate(all="ignore"):
        sc = f32((q[t - 1].astype(np.float64) * x[s - 1]).sum(1))
        alpha = softmax64(sc, t, n)
        r_ref = scatter64("+", alpha[:, None] * x[s - 1], t, n)
    xd, qd = torch.as_tensor(x).cuda(), torch.as_tensor(q).cuda()
    r = torch.empty(n, D, device="cuda"); smax = torch.empty(n, device="cuda"); ssum = torch.empty(n, device="cuda")
    gnn._lib.check(gnn._lib.lib.gnnb_set2set_attend(g.plan().h, xd.data_ptr(), qd.data_ptr(), D, r.data_ptr(),
                                                    smax.data_ptr(), ssum.data_ptr(), None))
    same(r.cpu().numpy(), r_ref, tol=5e-6, what="r")


# ------------------------------------------------------------------------------------------ dense
def no_tf32_exact(a):
    """a with every entry given a non-zero low part below the tf32 mantissa (the last bit set where it is clear).  The
    3xTF32 split multiplies x_big * w_small: for x = +-Inf and a w that tf32 represents exactly, that is Inf * 0 = NaN
    where the reference gives +-Inf (a known limit of the split, not covered here)."""
    b = np.ascontiguousarray(a, np.float32).view(np.uint32).copy()
    b[(b & 0x1FFF) == 0] |= 1
    return b.view(np.float32)


def linear_call(gnn, x, W, b, relu):
    lib = gnn._lib.lib
    N, Din = x.shape
    Dout = W.shape[0]
    xd, Wd = torch.as_tensor(x).cuda(), torch.as_tensor(W).cuda()
    bd = None if b is None else torch.as_tensor(b).cuda()
    y = torch.empty(N, Dout, device="cuda")
    gnn._lib.check(lib.gnnb_linear(xd.data_ptr(), Wd.data_ptr(), None if bd is None else bd.data_ptr(), int(relu), N, Din,
                                   Dout, y.data_ptr(), None))
    torch.cuda.synchronize()
    assert lib.gnnb_dense_tc_error() == 0
    return y.cpu().numpy()


DENSE_SHAPES = [(1000, 64, 128), (300, 128, 48), (4096, 256, 256), (500, 40, 16)]   # narrow, narrow, wide, library GEMM


@pytest.mark.gpu
@pytest.mark.parametrize("N,Din,Dout", DENSE_SHAPES)
@pytest.mark.parametrize("relu", [0, 1])
@pytest.mark.parametrize("bias", [False, True])
def test_linear_nonfinite(gnn, N, Din, Dout, relu, bias):
    """gnnb_linear with +-Inf and NaN in x and in W: rows / columns of +-Inf (and NaN where signs meet) as IEEE gives
    them, relu(NaN) = NaN"""
    rng = np.random.default_rng(Din + Dout)
    x = no_tf32_exact(rng.standard_normal((N, Din)))
    W = no_tf32_exact(rng.standard_normal((Dout, Din)) / np.sqrt(Din))
    b = rng.standard_normal(Dout).astype(np.float32) if bias else None
    x[3, 5], x[7, 6], x[11, 7] = np.inf, -np.inf, np.nan
    x[N - 1, 1] = np.inf
    W[2, 9], W[Dout - 1, 10], W[5, 11] = np.inf, -np.inf, np.nan
    with np.errstate(all="ignore"):
        ref = x.astype(np.float64) @ W.astype(np.float64).T + (0 if b is None else b.astype(np.float64))
    if relu:
        ref = relu64(ref)
    same(linear_call(gnn, x, W, b, relu), ref, tol=1e-5)


@pytest.mark.gpu
def test_bias_act_relu_mask_and_linear_bwd_nonfinite(gnn):
    """gnnb_bias_act (relu(NaN) = NaN), gnnb_linear_relu_mask (the mask bit of NaN and of 0 is 0) and gnnb_linear_bwd
    with a non-finite dy"""
    lib = gnn._lib.lib
    rng = np.random.default_rng(5)
    N, D = 257, 128
    xa = rng.standard_normal((N, D)).astype(np.float32)
    xa[0, :4] = [np.nan, np.inf, -np.inf, 0.0]
    b = rng.standard_normal(D).astype(np.float32)
    xd, bd = torch.as_tensor(xa).cuda(), torch.as_tensor(b).cuda()
    for relu in (0, 1):
        for bp in (None, bd):
            y = torch.empty_like(xd)
            gnn._lib.check(lib.gnnb_bias_act(xd.data_ptr(), None if bp is None else bp.data_ptr(), relu, N, D,
                                             y.data_ptr(), None))
            ref = (xa + (0 if bp is None else b)).astype(np.float64)          # the sum rounded to float32
            same(y.cpu().numpy(), relu64(ref) if relu else ref, tol=0, what=f"bias_act relu={relu}")

    # relu mask: NaN rows and a zero pre-activation column; bit of column n is bit 2 (n >> 3) + (n & 1) of word (n >> 1) & 3
    Din = 64
    x = no_tf32_exact(rng.standard_normal((N, Din)))
    W = no_tf32_exact(rng.standard_normal((D, Din)) / 8)
    x[4, 3] = np.nan
    W[6, :] = 0.0
    y = torch.empty(N, D, device="cuda")
    mask = torch.empty(N, 4, dtype=torch.int32, device="cuda")
    xd, Wd = torch.as_tensor(x).cuda(), torch.as_tensor(W).cuda()
    gnn._lib.check(lib.gnnb_linear_relu_mask(xd.data_ptr(), Wd.data_ptr(), None, N, Din, D, y.data_ptr(),
                                             mask.data_ptr(), None))
    torch.cuda.synchronize()
    assert lib.gnnb_dense_tc_error() == 0
    yn = y.cpu().numpy()
    same(yn, relu64(x.astype(np.float64) @ W.astype(np.float64).T), tol=1e-5, what="relu_mask y")
    m = mask.cpu().numpy().view(np.uint32)
    cols = np.arange(D)
    bits = (m[:, (cols >> 1) & 3] >> (2 * (cols >> 3) + (cols & 1))) & 1
    assert (bits == (yn > 0)).all()
    assert (bits[4] == 0).all() and np.isnan(yn[4]).all() and (bits[:, 6] == 0).all()

    # pullback with +-Inf and NaN in dy: dx = dy W, dW = dy^T x, db = column sums of dy
    for N2, Din2, Dout2 in ((1000, 64, 128), (300, 40, 16)):
        x = no_tf32_exact(rng.standard_normal((N2, Din2)))
        W = no_tf32_exact(rng.standard_normal((Dout2, Din2)) / 8)
        dy = no_tf32_exact(rng.standard_normal((N2, Dout2)))
        dy[2, 3], dy[9, 4], dy[N2 - 1, 5] = np.inf, -np.inf, np.nan
        dev = lambda a: torch.as_tensor(a).cuda()
        dyd, xd, Wd = dev(dy), dev(x), dev(W)
        dx = torch.empty(N2, Din2, device="cuda"); dW = torch.empty(Dout2, Din2, device="cuda")
        db = torch.empty(Dout2, device="cuda")
        gnn._lib.check(lib.gnnb_linear_bwd(dyd.data_ptr(), None, xd.data_ptr(), Wd.data_ptr(), 0, N2, Din2, Dout2, None,
                                           dx.data_ptr(), dW.data_ptr(), db.data_ptr(), None))
        torch.cuda.synchronize()
        assert lib.gnnb_dense_tc_error() == 0
        d64 = dy.astype(np.float64)
        with np.errstate(all="ignore"):
            same(dx.cpu().numpy(), d64 @ W.astype(np.float64), tol=1e-5, what="dx")
            same(dW.cpu().numpy(), d64.T @ x.astype(np.float64), tol=1e-5, what="dW")
            same(db.cpu().numpy(), d64.sum(0), tol=1e-5, what="db")


# ------------------------------------------------------------------------------------------ recurrent gates
@pytest.mark.gpu
@pytest.mark.parametrize("D", [8, 7])
def test_recurrent_gates_saturate_and_propagate_nan(gnn, D):
    """σ gives exactly 0 and 1 at -+Inf and at |x| = 1e4, tanh exactly -+1; NaN propagates (gnnb_gru_rz, gnnb_gru_out,
    gnnb_lstm_cell)"""
    lib = gnn._lib.lib
    vals = np.array([np.inf, -np.inf, 1e4, -1e4, 100.0, -100.0, np.nan, 0.5], np.float32)
    N = 64
    rng = np.random.default_rng(D)
    sig = lambda a: 1 / (1 + np.exp(-a))
    dev = lambda a: torch.as_tensor(np.ascontiguousarray(a, np.float32)).cuda()
    with np.errstate(all="ignore"):
        px = rng.standard_normal((N, 4 * D)).astype(np.float32)
        px[: len(vals), :] = vals[:, None]                     # row i: every gate at vals[i]
        h = rng.standard_normal((N, D)).astype(np.float32)
        p64 = px.astype(np.float64)
        # the device arrays are kept alive until the kernels have read them
        pxd, hd = dev(px), dev(h)
        zero1, zero2, zero4 = (dev(np.zeros((N, k * D))) for k in (1, 2, 4))
        # GRU: ah = 0
        r, z, rh = (torch.empty(N, D, device="cuda") for _ in range(3))
        gnn._lib.check(lib.gnnb_gru_rz(pxd.data_ptr(), 4 * D, zero2.data_ptr(), hd.data_ptr(),
                                       N, D, r.data_ptr(), z.data_ptr(), rh.data_ptr(), None))
        r_ref, z_ref = sig(p64[:, :D]), sig(p64[:, D:2 * D])
        same(r.cpu().numpy(), r_ref, tol=1e-6, what="r")
        same(z.cpu().numpy(), z_ref, tol=1e-6, what="z")
        for k, v in enumerate(vals[:4]):                       # exact saturation
            assert (r.cpu().numpy()[k] == (1.0 if v > 0 else 0.0)).all()
        nn_, hn = torch.empty(N, D, device="cuda"), torch.empty(N, D, device="cuda")
        gnn._lib.check(lib.gnnb_gru_out(pxd.data_ptr(), 4 * D, zero1.data_ptr(), hd.data_ptr(),
                                        z.data_ptr(), N, D, 0, nn_.data_ptr(), hn.data_ptr(), None))
        n_ref = np.tanh(p64[:, 2 * D:3 * D])
        same(nn_.cpu().numpy(), n_ref, tol=1e-6, what="n")
        for k, v in enumerate(vals[:4]):
            assert (nn_.cpu().numpy()[k] == np.sign(v)).all()
        zz = z.cpu().numpy().astype(np.float64)
        same(hn.cpu().numpy(), (1 - zz) * n_ref + zz * h, tol=1e-6, what="h'")
        # LSTM without peepholes: ah = 0
        c = rng.standard_normal((N, D)).astype(np.float32)
        cd = dev(c)
        gates, cn, hn = torch.empty(N, 4 * D, device="cuda"), torch.empty(N, D, device="cuda"), torch.empty(N, D, device="cuda")
        gnn._lib.check(lib.gnnb_lstm_cell(pxd.data_ptr(), 4 * D, zero4.data_ptr(), cd.data_ptr(),
                                          None, N, D, gates.data_ptr(), cn.data_ptr(), hn.data_ptr(), None))
        i_, f_, g_, o_ = sig(p64[:, :D]), sig(p64[:, D:2 * D]), np.tanh(p64[:, 2 * D:3 * D]), sig(p64[:, 3 * D:])
        c_ref = f_ * c + i_ * g_
        same(cn.cpu().numpy(), c_ref, tol=1e-6, what="c'")
        same(hn.cpu().numpy(), o_ * np.tanh(c_ref), tol=1e-6, what="h' lstm")
