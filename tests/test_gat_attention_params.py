"""The fused GAT kernels (csrc/gat.cu) across the parameters the shape sweeps of test_gpu_parity.py hold fixed, against
float64 closed forms evaluated with torch on the device:

- the negative slope over {0, 0.01, 0.2, 1, 3, -0.5}: gnnb_gat_aggregate (out, alpha, seg_max, seg_sum),
  gnnb_gat_aggregate_bwd (dWx, del, der), the halo instances, GATConv end to end (fused and generic, every gradient) and
  GATConv across two node types, on graphs whose rows sit on the chunk edges and on a 10^5-node RMAT graph;
- logits exactly on the leaky-ReLU kink (z = +0, -0 and the nearest floats either side);
- targets without in-edges and sources without out-edges on the single-GPU path, and a graph without edges;
- every outcome of gat_shape: the vector path from C = 4 to C = 128 (16 feature tiles at H = 16), the scalar path at
  C*H = 32, 64, 128 (1, 2, 4 slices per lane), operands one float off a 16 B boundary, and unsupported shapes.

Every output buffer starts as NaN, so a row a kernel skips fails the comparison.  Beside the normwise bar each result
meets a componentwise one: out[i,h,:] is a convex combination of the gathered rows Wx[s_k,h,:], so
|out - ref| <= c u max_k |Wx[s_k,h,:]| (u = 2^-24); alpha_k against alpha_k (1 + |u_k| + |M_i|), the rounding of its
exponent; dWx[j,h,:] against sum_k alpha_k (1 + |u_k| + |M_i|) max |dout[t_k,h,:]|; and the logit gradients against the
magnitudes of the terms their dz sum.  A single wrong row of a large output can pass a normwise bar; it cannot pass
these.  An empty row has bound 0: it must be exactly 0.
"""
import ctypes as C

import numpy as np
import pytest
import torch

from test_gpu_parity import build_graph

pytestmark = pytest.mark.gpu

U = 2.0 ** -24
SLOPES = [0.0, 0.01, 0.2, 1.0, 3.0, -0.5]
# c of the componentwise bars: the rounding of z = el + er and of slope * z, expf, and online-softmax and sum chains of
# at most one chunk of edges per row piece, with logits of a few units
CW = 64
# (C, H): a lean row of 128 floats, a round-1 vector shape, a scalar shape
SWEEP_SHAPES = [(32, 4), (16, 3), (2, 3)]
# leaky_relu'(z) at z == 0 that the float64 references use.  NNlib's source is not part of the reference tree, so this is
# torch's rule (aten/src/ATen/native/cpu/Activation.cpp, leaky_relu_backward: `self > 0 ? grad : grad * negval`): the
# slope, not 1, at z = +0 and at z = -0.  test_kink_rule_is_torchs checks the constant against torch.
KINK_DERIVATIVE = {0.2: 0.2, -0.5: -0.5}


def nan(*shape):
    return torch.full(shape, float("nan"), device="cuda")


def create_plan(gnn, s, t, n_src, n_dst):
    """a plan of the 0-based edge list (s, t) exactly as given: no self loops, COO order kept"""
    s, t = np.ascontiguousarray(s, np.int32), np.ascontiguousarray(t, np.int32)
    h = C.c_void_p()
    gnn._lib.check(gnn._lib.lib.gnnb_graph_create(C.byref(h), s.ctypes.data if s.size else None,
                                                  t.ctypes.data if t.size else None, s.size, n_src, n_dst, 4, 0, 0, None))
    return gnn.graph._Plan(h.value, torch.device("cuda", 0))


def rel(got, ref):
    got, ref = got.double(), ref.double()
    return float((got - ref).norm() / max(float(ref.norm()), 1e-30))


def assert_close(name, got, ref, scale, norm_tol):
    """got finite, normwise within norm_tol of ref (None: no normwise bar), and |got - ref| <= CW u scale per element
    (scale broadcasts)"""
    got = got.double()
    assert torch.isfinite(got).all(), f"{name}: {int((~torch.isfinite(got)).sum())} non-finite values (a skipped row?)"
    assert norm_tol is None or rel(got, ref) < norm_tol, f"{name}: normwise {rel(got, ref):.3e}"
    err = (got - ref).abs()
    bound = CW * U * scale.expand_as(err)
    bad = err > bound
    worst = float((err / (U * scale).clamp_min(1e-300)).max())
    assert not bad.any(), f"{name}: {int(bad.sum())} of {err.numel()} elements over {CW} u scale (worst {worst:.3g} u)"


def gat_f64(s, t, n_src, n_dst, Wx, el, er, slope, dout=None):
    """float64 closed form of the fused edge part (gat.cu header) and of its pullback, with the scales of the
    componentwise bars.  s, t: 0-based int64 device tensors.  leaky_relu'(z) is 1 for z > 0, the slope otherwise."""
    Wx, el, er = Wx.double(), el.double(), er.double()
    H = el.shape[1]
    z = el[t] + er[s]
    u = torch.where(z > 0, z, slope * z)
    tH = t[:, None].expand(-1, H)
    M = torch.full((n_dst, H), -float("inf"), dtype=torch.float64, device=z.device).scatter_reduce(0, tH, u, "amax")
    ex = torch.exp(u - M[t])
    S = torch.zeros((n_dst, H), dtype=torch.float64, device=z.device).index_add_(0, t, ex)
    al = ex / S[t]
    out = torch.zeros((n_dst,) + Wx.shape[1:], dtype=torch.float64, device=z.device).index_add_(0, t, al[:, :, None] * Wx[s])
    M = torch.where(torch.isinf(M), torch.zeros_like(M), M)          # empty rows: statistics 0 (gat.cu)
    wmax = Wx.abs().amax(-1)
    out_scale = torch.zeros((n_dst, H), dtype=torch.float64, device=z.device).scatter_reduce(0, tH, wmax[s], "amax")
    r = dict(out=out, alpha=al, seg_max=M, seg_sum=S, out_scale=out_scale[:, :, None],
             alpha_scale=al * (1 + u.abs() + M[t].abs()))
    if dout is not None:
        d = dout.double()
        da = (d[t] * Wx[s]).sum(-1)
        T = (d * out).sum(-1)
        lr = torch.where(z > 0, torch.ones_like(z), torch.full_like(z, slope))
        dz = al * (da - T[t]) * lr
        zs = lambda: torch.zeros((n_src, H), dtype=torch.float64, device=z.device)
        zd = lambda: torch.zeros((n_dst, H), dtype=torch.float64, device=z.device)
        w = al * lr.abs() * ((d[t] * Wx[s]).abs().sum(-1) + (d * out).abs().sum(-1)[t]
                             + (1 + u.abs() + M[t].abs()) * (da - T[t]).abs())
        r.update(dWx=torch.zeros(Wx.shape, dtype=torch.float64, device=z.device).index_add_(0, s, al[:, :, None] * d[t]),
                 der=zs().index_add_(0, s, dz), dl=zd().index_add_(0, t, dz), dz=dz, T=T,
                 dWx_scale=zs().index_add_(0, s, r["alpha_scale"] * d.abs().amax(-1)[t])[:, :, None],
                 der_scale=zs().index_add_(0, s, w), dl_scale=zd().index_add_(0, t, w), dz_scale=w)
    return r


def tensors(n_src, n_dst, Cc, H, seed):
    g = torch.Generator(device="cuda").manual_seed(seed)
    r = lambda *shape: torch.randn(*shape, device="cuda", generator=g)
    return r(n_src, H, Cc), r(n_dst, H), r(n_src, H), r(n_dst, H, Cc)


def run_fused(gnn, plan, n, Cc, H, slope, Wx, el, er, dout, alpha=True):
    """gnnb_gat_aggregate then gnnb_gat_aggregate_bwd on NaN-filled outputs (num_src = num_dst = n)"""
    lib = gnn._lib.lib
    E = C.c_int64()
    gnn._lib.check(lib.gnnb_graph_info(plan.h, C.byref(E), C.byref(C.c_int64()), C.byref(C.c_int64())))
    got = dict(out=nan(n, H, Cc), alpha=nan(E.value, H) if alpha else None, seg_max=nan(n, H), seg_sum=nan(n, H),
               dWx=nan(n, H, Cc), dl=nan(n, H), der=nan(n, H))
    ptr = lambda a: None if a is None else a.data_ptr()
    gnn._lib.check(lib.gnnb_gat_aggregate(plan.h, Wx.data_ptr(), el.data_ptr(), er.data_ptr(), Cc, H, slope,
                                          got["out"].data_ptr(), ptr(got["alpha"]), got["seg_max"].data_ptr(),
                                          got["seg_sum"].data_ptr(), None))
    gnn._lib.check(lib.gnnb_gat_aggregate_bwd(plan.h, Wx.data_ptr(), el.data_ptr(), er.data_ptr(), got["seg_max"].data_ptr(),
                                              got["seg_sum"].data_ptr(), got["out"].data_ptr(), dout.data_ptr(), Cc, H, slope,
                                              got["dWx"].data_ptr(), got["dl"].data_ptr(), got["der"].data_ptr(), None))
    torch.cuda.synchronize()
    return got


def check_fused(got, ref, what, slope):
    assert_close(f"out {what}", got["out"], ref["out"], ref["out_scale"], 5e-6)
    if got["alpha"] is not None:
        assert_close(f"alpha {what}", got["alpha"], ref["alpha"], ref["alpha_scale"], 5e-6)
    assert rel(got["seg_max"], ref["seg_max"]) < 5e-6, f"seg_max {what}"
    assert rel(got["seg_sum"], ref["seg_sum"]) < 5e-6, f"seg_sum {what}"
    assert_close(f"dWx {what}", got["dWx"], ref["dWx"], ref["dWx_scale"], 1e-5)
    assert_close(f"der {what}", got["der"], ref["der"], ref["der_scale"], 2e-4)
    # at slope 1 the logits are el_i + er_j: the softmax of row i cancels el_i and del vanishes identically, so only the
    # componentwise bar (rounding of the dz it sums) applies
    assert_close(f"del {what}", got["dl"], ref["dl"], ref["dl_scale"], None if slope == 1.0 else 2e-4)


# --------------------------------------------------------------------------------------------------- 1. slope sweep
@pytest.fixture(scope="module", params=["chunk_edges", "chunk32"])
def chunk_graph(request, gnn):
    """rows of c-1, c, c+1, 2c and 2c+1 edges at chunk c = 128 and 32, and nodes without edges (no self loops added)"""
    name, s, t, n, g = build_graph(gnn, request.param)
    return torch.as_tensor(s - 1, device="cuda"), torch.as_tensor(t - 1, device="cuda"), n, g


@pytest.mark.parametrize("slope", SLOPES)
@pytest.mark.parametrize("Cc,H", SWEEP_SHAPES)
def test_slope_sweep_c_abi(gnn, chunk_graph, Cc, H, slope):
    s, t, n, g = chunk_graph
    Wx, el, er, dout = tensors(n, n, Cc, H, 7 * Cc + H)
    got = run_fused(gnn, g.plan(), n, Cc, H, slope, Wx, el, er, dout)
    check_fused(got, gat_f64(s, t, n, n, Wx, el, er, slope, dout), f"C={Cc} H={H} slope={slope}", slope)


@pytest.fixture(scope="module")
def rmat(gnn):
    g = gnn.rmat_graph(100_000, 1_000_000, seed=23, device="cuda")
    return g.s.long() - 1, g.t.long() - 1, g.num_nodes, g


@pytest.mark.parametrize("slope", SLOPES)
def test_slope_sweep_at_scale(gnn, rmat, slope):
    """RMAT N = 10^5, E = 10^6 (hubs far longer than a chunk, many empty rows) on the lean kernels, C = 64, H = 4"""
    s, t, n, g = rmat
    Wx, el, er, dout = tensors(n, n, 64, 4, 11)
    got = run_fused(gnn, g.plan(), n, 64, 4, slope, Wx, el, er, dout)
    check_fused(got, gat_f64(s, t, n, n, Wx, el, er, slope, dout), f"rmat slope={slope}", slope)


@pytest.mark.parametrize("slope", SLOPES)
@pytest.mark.parametrize("Cc,H", SWEEP_SHAPES)
def test_slope_sweep_halo(gnn, chunk_graph, Cc, H, slope):
    """gnnb_gat_aggregate_halo on the plan with the gathered rows >= n/2 in a second buffer, and
    gnnb_gat_aggregate_bwd_halo on the reversed plan (rows = sources) with dout split alike: out, seg_max, seg_sum,
    dWx, der and every edge's dz against float64"""
    s, t, n, _ = chunk_graph
    lib = gnn._lib.lib
    sn, tn = s.cpu().numpy(), t.cpu().numpy()
    fwd, rev = create_plan(gnn, sn, tn, n, n), create_plan(gnn, tn, sn, n, n)
    Wx, el, er, dout = tensors(n, n, Cc, H, 13 * Cc + H)
    ref = gat_f64(s, t, n, n, Wx, el, er, slope, dout)
    split = n // 2
    out, smax, ssum = nan(n, H, Cc), nan(n, H), nan(n, H)
    x_local, x_halo = Wx[:split].clone(), Wx[split:].clone()
    gnn._lib.check(lib.gnnb_gat_aggregate_halo(fwd.h, x_local.data_ptr(), x_halo.data_ptr(), split,
                                               el.data_ptr(), er.data_ptr(), Cc, H, slope, out.data_ptr(), smax.data_ptr(),
                                               ssum.data_ptr(), None))
    T = nan(n, H)
    gnn._lib.check(lib.gnnb_gat_tnode(dout.data_ptr(), out.data_ptr(), n, Cc, H, T.data_ptr(), None))
    dWx, der, dz = nan(n, H, Cc), nan(n, H), nan(len(sn), H)
    d_local, d_halo = dout[:split].clone(), dout[split:].clone()
    gnn._lib.check(lib.gnnb_gat_aggregate_bwd_halo(rev.h, Wx.data_ptr(), er.data_ptr(), d_local.data_ptr(),
                                                   d_halo.data_ptr(), split, el.data_ptr(), smax.data_ptr(), ssum.data_ptr(),
                                                   T.data_ptr(), Cc, H, slope, dWx.data_ptr(), der.data_ptr(),
                                                   dz.data_ptr(), None))
    torch.cuda.synchronize()
    what = f"halo C={Cc} H={H} slope={slope}"
    assert_close(f"out {what}", out, ref["out"], ref["out_scale"], 5e-6)
    assert rel(smax, ref["seg_max"]) < 5e-6 and rel(ssum, ref["seg_sum"]) < 5e-6, what
    assert rel(T, ref["T"]) < 1e-5, what
    assert_close(f"dWx {what}", dWx, ref["dWx"], ref["dWx_scale"], 1e-5)
    assert_close(f"der {what}", der, ref["der"], ref["der_scale"], 2e-4)
    assert_close(f"dz {what}", dz, ref["dz"], ref["dz_scale"], 2e-4)


def gat_layer_f64(layer, s, t, n_dst, xj, xi, dy):
    """float64 autograd of gat_conv (GNNlib/src/layers/conv.jl:112-167, σ = identity, concat) over the edges (s, t):
    y and the gradients of xj, xi (None when the graph has one node type), W, a and bias"""
    Cc, H = layer.channel[1], layer.heads
    xj64 = xj.double().requires_grad_(True)
    xi64 = xj64 if xi is None else xi.double().requires_grad_(True)
    Wd, a, b = (p.detach().double().requires_grad_(True) for p in (layer.dense_x.weight, layer.a, layer.bias))
    Wj, Wi = (xj64 @ Wd.t()).reshape(-1, H, Cc), (xi64 @ Wd.t()).reshape(-1, H, Cc)
    z = (Wi[t] * a[:Cc].t()).sum(-1) + (Wj[s] * a[Cc:].t()).sum(-1)
    u = torch.nn.functional.leaky_relu(z, float(layer.negative_slope))
    M = torch.full((n_dst, H), -float("inf"), dtype=torch.float64, device=z.device)
    M = M.scatter_reduce(0, t[:, None].expand(-1, H), u.detach(), "amax")
    ex = torch.exp(u - M[t])
    al = ex / torch.zeros((n_dst, H), dtype=torch.float64, device=z.device).index_add(0, t, ex)[t]
    out = torch.zeros((n_dst, H, Cc), dtype=torch.float64, device=z.device).index_add(0, t, al[:, :, None] * Wj[s])
    y = out.reshape(n_dst, H * Cc) + b
    y.backward(dy.double())
    return y.detach(), [xj64.grad, None if xi is None else xi64.grad, Wd.grad, a.grad, b.grad]


def run_layer(gnn, layer, g, xj_rows, xi_rows, dy_rows, fused):
    """y and the gradients of xj, xi, W, a, bias of one GATConv call on Julia-shaped inputs"""
    layer.zero_grad()
    xj = gnn.unrows(xj_rows.clone()).requires_grad_(True)
    xi = None if xi_rows is None else gnn.unrows(xi_rows.clone()).requires_grad_(True)
    y = layer(g, xj if xi is None else (xj, xi), fused=fused)
    (y * gnn.unrows(dy_rows)).sum().backward()
    grads = [gnn.rows(xj.grad), None if xi is None else gnn.rows(xi.grad), layer.dense_x.weight.grad, layer.a.grad,
             layer.bias.grad]
    return gnn.rows(y.detach()), grads


def check_layer(gnn, layer, g, s, t, n_dst, xj_rows, xi_rows, what, fwd_tol=1e-5, grad_tol=1e-4, vanishing=()):
    """fused and generic GATConv against float64 autograd: y and every gradient; returns both runs.  The gradients named
    in `vanishing` are 0 in exact arithmetic: their norm is held below grad_tol times the norm of dxj."""
    torch.manual_seed(1)
    dy = torch.randn(n_dst, layer.heads * layer.channel[1], device="cuda")
    y64, g64 = gat_layer_f64(layer, s, t, n_dst, xj_rows, xi_rows, dy)
    runs = []
    for fused in (True, False):
        y, grads = run_layer(gnn, layer, g, xj_rows, xi_rows, dy, fused)
        assert torch.isfinite(y).all() and rel(y, y64) < fwd_tol, f"y fused={fused} {what}: {rel(y, y64):.3e}"
        for name, a, b in zip(("dxj", "dxi", "dW", "da", "dbias"), grads, g64):
            if b is None:
                continue
            assert torch.isfinite(a).all(), f"{name} fused={fused} {what}"
            if name in vanishing:
                assert float(a.norm()) < grad_tol * float(g64[0].norm()), f"{name} fused={fused} {what}: {float(a.norm()):.3e}"
            else:
                assert rel(a, b) < grad_tol, f"{name} fused={fused} {what}: {rel(a, b):.3e}"
        runs.append((y, grads))
    return runs


@pytest.fixture(scope="module")
def chunk_edges(gnn):
    name, s, t, n, g = build_graph(gnn, "chunk_edges")
    return s - 1, t - 1, n, g


@pytest.mark.parametrize("slope", SLOPES)
@pytest.mark.parametrize("Cc,H", SWEEP_SHAPES)
def test_slope_sweep_gat_conv(gnn, chunk_edges, Cc, H, slope):
    """GATConv(negative_slope = slope) with self loops: the lean shape through gnnb_gat_logit_terms, the vector one too,
    the scalar one with el / er from torch"""
    s, t, n, g = chunk_edges
    loops = np.arange(n)
    s2, t2 = (torch.as_tensor(np.concatenate([a, loops]), device="cuda") for a in (s, t))
    torch.manual_seed(Cc + H)
    layer = gnn.GATConv(8, Cc, heads=H, negative_slope=slope, device="cuda")
    with torch.no_grad():
        layer.bias.normal_()
    x = torch.randn(n, 8, device="cuda")
    check_layer(gnn, layer, g, s2, t2, n, x, None, f"C={Cc} H={H} slope={slope}")


@pytest.mark.parametrize("slope", SLOPES)
def test_slope_sweep_bipartite_gat_conv(gnn, slope):
    """GATConv across two node types (el from W xi over the targets, er from W xj over the sources): a target row of
    more than two chunks, a source without out-edges and a target without in-edges"""
    rng = np.random.default_rng(31)
    ns, nd = 90, 50
    s = np.concatenate([rng.integers(0, ns - 1, 400), rng.integers(0, ns - 1, 300)])
    t = np.concatenate([rng.integers(1, nd - 1, 400), np.zeros(300, np.int64)])
    g = gnn.GNNHeteroGraph({("A", "r", "B"): (torch.as_tensor(s + 1), torch.as_tensor(t + 1))},
                           num_nodes={"A": ns, "B": nd}, device="cuda")
    torch.manual_seed(5)
    layer = gnn.GATConv(12, 8, heads=8, negative_slope=slope).cuda()
    with torch.no_grad():
        layer.bias.uniform_(-1, 1)
    xj, xi = torch.randn(ns, 12, device="cuda"), torch.randn(nd, 12, device="cuda")
    # at slope 1, xi only enters through el, which the softmax of its row cancels: its gradient vanishes
    check_layer(gnn, layer, g, torch.as_tensor(s, device="cuda"), torch.as_tensor(t, device="cuda"), nd, xj, xi,
                f"bipartite slope={slope}", vanishing=("dxi",) if slope == 1.0 else ())


# ----------------------------------------------------------------------------------------------- 2. the kink, z = 0
def test_kink_rule_is_torchs():
    """KINK_DERIVATIVE is what torch's leaky_relu gives at +0 and -0, and leaky_relu(+0) carries the slope's sign"""
    for slope, d in KINK_DERIVATIVE.items():
        z = torch.tensor([0.0, -0.0], dtype=torch.float64, requires_grad=True)
        torch.nn.functional.leaky_relu(z, slope).sum().backward()
        assert z.grad.tolist() == [d, d]
    assert torch.signbit(torch.nn.functional.leaky_relu(torch.tensor(0.0), -0.5))


TINY = 2.0 ** -149                                          # the smallest subnormal: the float next to 0


def kink_logits(n, H):
    """el, er (float32, exact) whose sums z = el[t] + er[s] are exactly +0, -0, +-TINY, +-2^-24 or small integers.
    Even heads: el = 1 and er in {-1, -1 + 2^-24, -1 - 2^-23, 1, -3, -1.5} by source id mod 6, so z in {+0, 2^-24,
    -2^-23, 2, -2, -0.5}.  Odd heads: el = -0 and er in {-0, +0, TINY, -TINY, 1, -1}, so z in {-0, +0, TINY, -TINY, 1,
    -1}."""
    even = torch.tensor([-1.0, -1.0 + 2.0 ** -24, -1.0 - 2.0 ** -23, 1.0, -3.0, -1.5], dtype=torch.float32)
    odd = torch.tensor([-0.0, 0.0, TINY, -TINY, 1.0, -1.0], dtype=torch.float32)
    ids = torch.arange(n) % 6
    el = torch.empty(n, H, dtype=torch.float32)
    er = torch.empty(n, H, dtype=torch.float32)
    for h in range(H):
        el[:, h] = 1.0 if h % 2 == 0 else -0.0
        er[:, h] = (even if h % 2 == 0 else odd)[ids]
    assert TINY > 0 and torch.tensor(TINY, dtype=torch.float32).item() == TINY
    return el.cuda(), er.cuda()


@pytest.mark.parametrize("slope", list(KINK_DERIVATIVE))
@pytest.mark.parametrize("Cc,H", [(32, 4), (4, 2), (2, 2)])
def test_kink_c_abi(gnn, Cc, H, slope):
    """logits exactly on the kink through the lean, the round-1 vector and the scalar kernels.  Targets 0..119 have one
    in-edge from source i (each logit class appears alone in a row); the others 2..40 in-edges.  Forward and pullback
    against float64 with leaky_relu'(0) = KINK_DERIVATIVE[slope]; on the one-edge rows seg_max equals torch's float32
    leaky_relu of the row's logit bit for bit, sign of zero included: at z = +0 a negative slope gives -0."""
    n = 400
    rng = np.random.default_rng(3)
    deg = rng.integers(2, 41, n - 120)
    t = np.concatenate([np.arange(120), np.repeat(np.arange(120, n), deg)])
    s = np.concatenate([np.arange(120), rng.integers(0, n, deg.sum())])
    p = rng.permutation(len(s))
    s, t = s[p], t[p]
    plan = create_plan(gnn, s, t, n, n)
    el, er = kink_logits(n, H)
    Wx, _, _, dout = tensors(n, n, Cc, H, 17)
    st, tt = torch.as_tensor(s, device="cuda"), torch.as_tensor(t, device="cuda")
    z = el[tt] + er[st]
    assert (z == 0).sum() > 0.2 * z.numel() and torch.signbit(z[z == 0]).any() and (z.abs() == TINY).any()
    got = run_fused(gnn, plan, n, Cc, H, slope, Wx, el, er, dout)
    assert KINK_DERIVATIVE[slope] == slope                  # gat_f64's leaky_relu'(+-0)
    ref = gat_f64(st, tt, n, n, Wx, el, er, slope, dout)
    check_fused(got, ref, f"kink C={Cc} H={H} slope={slope}", slope)
    one = torch.arange(120, device="cuda")
    k1 = torch.nonzero(tt < 120).squeeze(1)
    u32 = torch.nn.functional.leaky_relu(z[k1], slope)
    want = torch.empty(120, H, device="cuda")
    want[tt[k1]] = u32
    assert torch.equal(got["seg_max"][one].view(torch.int32), want.view(torch.int32)), f"seg_max bits slope={slope}"


def integer_layer(gnn, Cc, H, slope):
    """GATConv whose logits are exact in float32 on the fused and the generic path: W in {-1, 0, 1}, a in {0, +-1/4,
    +-1/2} with z = (Wx_i[0] - Wx_j[0]) / 4 + (Wx_i[1] - Wx_j[1]) / 2 per head (signs vary by head), so every self loop and
    every edge between nodes of equal projections sits on the kink"""
    layer = gnn.GATConv(3, Cc, heads=H, negative_slope=slope, device="cuda")
    gen = torch.Generator().manual_seed(Cc * 10 + H)
    with torch.no_grad():
        layer.dense_x.weight.copy_(torch.randint(-1, 2, layer.dense_x.weight.shape, generator=gen).float())
        a = torch.zeros(2 * Cc, H)
        for h in range(H):
            sg = 1.0 if h % 2 == 0 else -1.0
            a[0, h], a[Cc, h] = 0.25 * sg, -0.25 * sg
            a[1, h], a[Cc + 1, h] = 0.5, -0.5
        layer.a.copy_(a)
        layer.bias.uniform_(-1, 1)
    return layer


@pytest.mark.parametrize("slope", list(KINK_DERIVATIVE))
@pytest.mark.parametrize("Cc,H", [(32, 4), (8, 2)])
def test_kink_gat_conv_fused_equals_generic(gnn, chunk_edges, Cc, H, slope):
    """GATConv with logits on the kink: fused against the generic path (torch's leaky_relu and its autograd) and both
    against float64, forward and the gradients of x, W, a and bias"""
    s, t, n, g = chunk_edges
    loops = np.arange(n)
    s2, t2 = (torch.as_tensor(np.concatenate([a, loops]), device="cuda") for a in (s, t))
    layer = integer_layer(gnn, Cc, H, slope)
    x = torch.randint(-1, 2, (n, 3), generator=torch.Generator().manual_seed(2)).float().cuda()
    Wx = (x.double() @ layer.dense_x.weight.detach().double().t()).reshape(n, H, Cc)
    a = layer.a.detach().double()
    z = (Wx[t2] * a[:Cc].t()).sum(-1) + (Wx[s2] * a[Cc:].t()).sum(-1)
    assert (z == 0).float().mean() > 0.05 and (z[-n:] == 0).all()     # every self loop and more
    (yf, gf), (yg, gg) = check_layer(gnn, layer, g, s2, t2, n, x, None, f"kink C={Cc} H={H} slope={slope}")
    assert rel(yf, yg) < 2e-6
    for a_, b_ in zip(gf, gg):
        if a_ is not None:
            assert rel(a_, b_) < 2e-5


# ---------------------------------------------------------------------------------------- 3. nodes without edges
def empty_rows_graph():
    """0-based edges without self loops over n = 600 nodes: targets 0..199 get no in-edge, sources 200..399 no
    out-edge (disjoint thirds), target 450 gets 300 in-edges and source 10 300 out-edges (rows of more than two chunks
    in both plans)"""
    rng = np.random.default_rng(41)
    n = 600
    srcs = np.concatenate([np.arange(200), np.arange(400, 600)])
    s = np.concatenate([rng.choice(srcs, 2500), rng.choice(srcs, 300), np.full(300, 10)])
    t = np.concatenate([rng.integers(200, n, 2500), np.full(300, 450), rng.integers(200, n, 300)])
    p = rng.permutation(len(s))
    return s[p], t[p], n


EMPTY_T, EMPTY_S = slice(0, 200), slice(200, 400)


@pytest.mark.parametrize("Cc,H", [(32, 4), (64, 8), (16, 3), (2, 16)])
def test_empty_rows_c_abi(gnn, Cc, H):
    """out, seg_max, seg_sum and del exactly 0 on targets without in-edges, dWx and der exactly 0 on sources without
    out-edges (gat_fill_empty_kernel on the lean shapes, the kernels' own fill on the others), the rest against float64"""
    s, t, n = empty_rows_graph()
    g = gnn.GNNGraph(torch.as_tensor(s + 1), torch.as_tensor(t + 1), num_nodes=n).cuda()
    Wx, el, er, dout = tensors(n, n, Cc, H, 19 * Cc + H)
    got = run_fused(gnn, g.plan(), n, Cc, H, 0.2, Wx, el, er, dout)
    for name in ("out", "seg_max", "seg_sum", "dl"):
        assert (got[name][EMPTY_T] == 0).all(), f"{name} on empty targets C={Cc} H={H}"
    for name in ("dWx", "der"):
        assert (got[name][EMPTY_S] == 0).all(), f"{name} on empty sources C={Cc} H={H}"
    st, tt = torch.as_tensor(s, device="cuda"), torch.as_tensor(t, device="cuda")
    check_fused(got, gat_f64(st, tt, n, n, Wx, el, er, 0.2, dout), f"empty rows C={Cc} H={H}", 0.2)


@pytest.mark.parametrize("Cc,H", [(32, 4), (16, 3), (2, 16)])
def test_no_edges_c_abi(gnn, Cc, H):
    """E = 0, n > 0: every output row is exactly 0"""
    n = 50
    plan = create_plan(gnn, np.zeros(0), np.zeros(0), n, n)
    Wx, el, er, dout = tensors(n, n, Cc, H, 5)
    got = run_fused(gnn, plan, n, Cc, H, 0.2, Wx, el, er, dout, alpha=False)
    for name, a in got.items():
        if a is not None:
            assert (a == 0).all(), name


@pytest.mark.parametrize("Cc,H", [(32, 4), (8, 2), (2, 3)])
def test_empty_rows_gat_conv_without_self_loops(gnn, Cc, H):
    """GATConv(add_self_loops = false), fused and generic, on the graph with empty rows and on a graph without edges"""
    s, t, n = empty_rows_graph()
    torch.manual_seed(Cc * H)
    layer = gnn.GATConv(8, Cc, heads=H, add_self_loops=False, device="cuda")
    with torch.no_grad():
        layer.bias.normal_()
    x = torch.randn(n, 8, device="cuda")
    g = gnn.GNNGraph(torch.as_tensor(s + 1), torch.as_tensor(t + 1), num_nodes=n).cuda()
    st, tt = torch.as_tensor(s, device="cuda"), torch.as_tensor(t, device="cuda")
    for y, grads in check_layer(gnn, layer, g, st, tt, n, x, None, f"empty rows C={Cc} H={H}"):
        assert torch.equal(y[EMPTY_T], layer.bias.detach().expand(200, -1))       # no message: the bias alone
    e0 = torch.zeros(0, dtype=torch.int64)
    g0 = gnn.GNNGraph(e0, e0, num_nodes=40).cuda()
    for y, grads in check_layer(gnn, layer, g0, e0.cuda(), e0.cuda(), 40, x[:40], None, f"E = 0 C={Cc} H={H}"):
        assert torch.equal(y, layer.bias.detach().expand(40, -1))
        assert (grads[0] == 0).all() and (grads[2] == 0).all() and (grads[3] == 0).all()


# ---------------------------------------------------------------------------------------- 4. every gat_shape outcome
@pytest.mark.parametrize("Cc,H", [(4, 1), (4, 5), (128, 1), (128, 2), (128, 16), (2, 16), (1, 64), (2, 64)],
                         ids=["vec4-C4", "vec4-C4H5", "vec4-C128-lean", "vec4-C128H2-lean", "vec4-C128H16-16tiles",
                              "scalar-kk1", "scalar-kk2", "scalar-kk4"])
def test_every_shape_c_abi(gnn, chunk_graph, Cc, H):
    s, t, n, g = chunk_graph
    Wx, el, er, dout = tensors(n, n, Cc, H, 23 * Cc + H)
    got = run_fused(gnn, g.plan(), n, Cc, H, -0.5, Wx, el, er, dout)
    check_fused(got, gat_f64(s, t, n, n, Wx, el, er, -0.5, dout), f"C={Cc} H={H}", -0.5)


def off16(shape):
    """a NaN-filled tensor whose data sits one float past a 16 B boundary"""
    buf = nan(int(np.prod(shape)) + 4)
    assert buf.data_ptr() % 16 == 0
    return buf[1:1 + int(np.prod(shape))].view(shape)


@pytest.mark.parametrize("operand", ["Wx", "out"])
def test_misaligned_vector_shape_takes_the_scalar_path(gnn, chunk_graph, operand):
    """C = 32, H = 4 (a vector shape) with Wx or out (and dWx) one float off a 16 B boundary: gat_shape drops to the
    scalar path, which returns the float64 answer.  dout or the forward's out off the boundary in the pullback, and any
    misaligned operand at C = 64 (no scalar path above C = 32), raise GNNBError (GNNB_EUNSUPPORTED) before any launch."""
    s, t, n, g = chunk_graph
    lib, Cc, H = gnn._lib.lib, 32, 4
    Wx, el, er, dout = tensors(n, n, Cc, H, 29)
    ref = gat_f64(s, t, n, n, Wx, el, er, 0.2, dout)
    if operand == "Wx":
        w = off16((n, H, Cc)); w.copy_(Wx); Wx = w
        assert Wx.data_ptr() % 16 == 4
    out = off16((n, H, Cc)) if operand == "out" else nan(n, H, Cc)
    dWx = off16((n, H, Cc))
    smax, ssum, dl, der = nan(n, H), nan(n, H), nan(n, H), nan(n, H)
    h = g.plan().h
    gnn._lib.check(lib.gnnb_gat_aggregate(h, Wx.data_ptr(), el.data_ptr(), er.data_ptr(), Cc, H, 0.2, out.data_ptr(), None,
                                          smax.data_ptr(), ssum.data_ptr(), None))
    out_a = out.clone()                                     # the pullback needs out and dout 16 B aligned
    gnn._lib.check(lib.gnnb_gat_aggregate_bwd(h, Wx.data_ptr(), el.data_ptr(), er.data_ptr(), smax.data_ptr(),
                                              ssum.data_ptr(), out_a.data_ptr(), dout.data_ptr(), Cc, H, 0.2, dWx.data_ptr(),
                                              dl.data_ptr(), der.data_ptr(), None))
    torch.cuda.synchronize()
    assert_close(f"out, {operand} off 16 B", out, ref["out"], ref["out_scale"], 5e-6)
    assert_close(f"dWx, {operand} off 16 B", dWx, ref["dWx"], ref["dWx_scale"], 1e-5)
    assert_close(f"der, {operand} off 16 B", der, ref["der"], ref["der_scale"], 2e-4)
    assert_close(f"del, {operand} off 16 B", dl, ref["dl"], ref["dl_scale"], 2e-4)
    before = gnn.launch_count()
    for bad in ("dout", "out_fwd"):
        d_ = off16((n, H, Cc)); d_.copy_(dout if bad == "dout" else out_a)
        args = (d_, dout) if bad == "out_fwd" else (out_a, d_)
        with pytest.raises(gnn.GNNBError) as e:
            gnn._lib.check(lib.gnnb_gat_aggregate_bwd(h, Wx.data_ptr(), el.data_ptr(), er.data_ptr(), smax.data_ptr(),
                                                      ssum.data_ptr(), args[0].data_ptr(), args[1].data_ptr(), Cc, H, 0.2,
                                                      dWx.data_ptr(), dl.data_ptr(), der.data_ptr(), None))
        assert e.value.status == gnn._lib.EUNSUPPORTED
    W64, o64 = off16((n, 4, 64)), off16((n, 4, 64))
    W64.normal_()
    for wp, op in ((W64, nan(n, 4, 64)), (torch.randn(n, 4, 64, device="cuda"), o64)):
        with pytest.raises(gnn.GNNBError) as e:
            gnn._lib.check(lib.gnnb_gat_aggregate(h, wp.data_ptr(), el.data_ptr(), er.data_ptr(), 64, 4, 0.2, op.data_ptr(),
                                                  None, smax.data_ptr(), ssum.data_ptr(), None))
        assert e.value.status == gnn._lib.EUNSUPPORTED
    assert gnn.launch_count() == before                      # refused before any kernel ran


@pytest.mark.parametrize("Cc,H", [(12, 2), (64, 3), (3, 4)])
def test_unsupported_shape_gat_conv_takes_the_generic_path(gnn, chunk_edges, Cc, H):
    """C = 12 and C = 3 are outside gat_shape: the C ABI raises GNNB_EUNSUPPORTED and GATConv(fused = true) takes the
    generic path, the same bits as fused = false.  (64, 3), the control, is a vector shape the C ABI accepts.  Every
    layer call matches float64 in the forward and every gradient."""
    s, t, n, g = chunk_edges
    lib = gnn._lib.lib
    Wx, el, er, _ = tensors(n, n, Cc, H, 31)
    out, smax, ssum = nan(n, H, Cc), nan(n, H), nan(n, H)
    call = lambda: gnn._lib.check(lib.gnnb_gat_aggregate(g.plan().h, Wx.data_ptr(), el.data_ptr(), er.data_ptr(), Cc, H,
                                                         0.2, out.data_ptr(), None, smax.data_ptr(), ssum.data_ptr(), None))
    fusable = gnn.layers.gat_fusable(Cc, H)
    if fusable:
        call()
    else:
        with pytest.raises(gnn.GNNBError) as e:
            call()
        assert e.value.status == gnn._lib.EUNSUPPORTED
    loops = np.arange(n)
    s2, t2 = (torch.as_tensor(np.concatenate([a, loops]), device="cuda") for a in (s, t))
    torch.manual_seed(3)
    layer = gnn.GATConv(8, Cc, heads=H, negative_slope=-0.5, device="cuda")
    with torch.no_grad():
        layer.bias.normal_()
    x = torch.randn(n, 8, device="cuda")
    (yf, gf), (yg, gg) = check_layer(gnn, layer, g, s2, t2, n, x, None, f"C={Cc} H={H}")
    if not fusable:
        assert torch.equal(yf, yg) and all(torch.equal(a, b) for a, b in zip(gf, gg) if a is not None)
