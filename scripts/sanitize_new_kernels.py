"""small calls of the hand-written dense-layer kernels, the closing line, the max pullback, the subgraph plans, the
drop mask, the random-walk encoding (both launch classes, the propagate route, a seg_ptr an edge crosses), PPR diffusion
(both launch classes, the dense route's matrix kernel, a seg_ptr an edge crosses), the largest Laplacian eigenvalue
(both launch classes, the Lanczos route, a seg_ptr an edge crosses), colour
refinement (hub rows cut into long-row pieces, a path, a batch), Set2Set (a graph with no nodes, graphs of chunk +- 1
nodes, D = 1, 3 and 1024, the composition at D = 1025) and the temporal graph generators, meant to run under `compute-sanitizer --tool memcheck`
(or racecheck / synccheck)"""
import os, sys, torch
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import gnnb200 as gnn
lib = gnn._lib.lib
torch.manual_seed(0)
# wide linear kernel (tail tile, 3 output quarters, 5 K-blocks) + its dx
N, K, Nout = 2048 + 77, 160, 384
x = torch.randn(N, K, device="cuda"); W = torch.randn(Nout, K, device="cuda") / K ** 0.5; b = torch.randn(Nout, device="cuda")
y = torch.empty(N, Nout, device="cuda")
gnn._lib.check(lib.gnnb_linear(x.data_ptr(), W.data_ptr(), b.data_ptr(), 1, N, K, Nout, y.data_ptr(), None))
ref = (x.double() @ W.double().t() + b.double()).clamp(min=0)
print("wide linear err", float((y.double() - ref).norm() / ref.norm()), "tc_error", lib.gnnb_dense_tc_error())
# narrow linear kernel (tail tile, Nout < 128) and its pullback through the fused kernels
N, K, Nout = 1000 + 13, 96, 128
x = torch.randn(N, K, device="cuda"); W = torch.randn(Nout, K, device="cuda") / K ** 0.5; b = torch.randn(Nout, device="cuda")
y = torch.empty(N, Nout, device="cuda")
gnn._lib.check(lib.gnnb_linear(x.data_ptr(), W.data_ptr(), b.data_ptr(), 1, N, K, Nout, y.data_ptr(), None))
dy = torch.randn(N, Nout, device="cuda"); ws = torch.empty_like(dy); dx = torch.empty_like(x); dW = torch.empty_like(W)
dbl = torch.empty(Nout, device="cuda")
gnn._lib.check(lib.gnnb_linear_bwd(dy.data_ptr(), y.data_ptr(), x.data_ptr(), W.data_ptr(), 1, N, K, Nout, ws.data_ptr(),
                                   dx.data_ptr(), dW.data_ptr(), dbl.data_ptr(), None))
dpre = dy.double() * (y > 0)
print("narrow linear dx err", float((dx.double() - dpre @ W.double()).norm() / (dpre @ W.double()).norm()),
      "dW err", float((dW.double() - dpre.t() @ x.double()).norm() / (dpre.t() @ x.double()).norm()),
      "tc_error", lib.gnnb_dense_tc_error())
# the fused pullback (linear_bwd_dx_kernel, linear_bwd_dw_kernel) at a ragged N: one row past a CTA's split-K range,
# no relu, no db
N, K = 132 * 32 + 1, 128
x = torch.randn(N, K, device="cuda"); W = torch.randn(Nout, K, device="cuda") / K ** 0.5
dy = torch.randn(N, Nout, device="cuda"); dx = torch.empty_like(x); dW = torch.empty_like(W)
gnn._lib.check(lib.gnnb_linear_bwd(dy.data_ptr(), None, x.data_ptr(), W.data_ptr(), 0, N, K, Nout, None, dx.data_ptr(),
                                   dW.data_ptr(), None, None))
print("fused pullback dx err", float((dx.double() - dy.double() @ W.double()).norm() / (dy.double() @ W.double()).norm()),
      "dW err", float((dW.double() - dy.double().t() @ x.double()).norm() / (dy.double().t() @ x.double()).norm()),
      "tc_error", lib.gnnb_dense_tc_error())
# closing line
D = 36
z = torch.randn(1001, D, device="cuda"); bb = torch.randn(D, device="cuda"); o = torch.empty_like(z)
gnn._lib.check(lib.gnnb_bias_act(z.data_ptr(), bb.data_ptr(), 1, 1001, D, o.data_ptr(), None))
dz = torch.empty_like(z); db = torch.empty(D, device="cuda")
gnn._lib.check(lib.gnnb_bias_act_bwd(z.data_ptr(), o.data_ptr(), 1, 1001, D, dz.data_ptr(), db.data_ptr(), None))
print("bias_act ok", bool(torch.equal(o, (z + bb).clamp(min=0))))
# max pullback on a graph with a hub in the by-source plan (long rows -> partial slots + fix-up)
n = 3000
s = torch.cat([torch.ones(1500, dtype=torch.int64), torch.randint(1, n + 1, (4000,))])
t = torch.cat([torch.randint(1, n + 1, (1500,)), torch.randint(1, n + 1, (4000,))])
g = gnn.GNNGraph(s, t, num_nodes=n).to("cuda")
for Dm in (128, 256):
    xm = gnn.unrows((torch.randn(n, Dm, device="cuda") * 2).round() / 2).requires_grad_(True)
    ym = gnn.propagate(gnn.copy_xj, g, "max", xj=xm)
    dy = torch.where(torch.isfinite(ym), torch.randn_like(ym), torch.zeros_like(ym))
    ym.backward(dy)
    print("max pullback D", Dm, float(xm.grad.abs().sum()))
# subgraph plans (gnnb_graph_subgraph) and the drop mask (gnnb_bernoulli_keep): the hub graph with both CSRs built, an
# empty graph, every edge removed, every node removed, extra nodes
gnn.csr(g, transposed=True)
e0 = torch.zeros(0, dtype=torch.int64, device="cuda")
g0 = gnn.GNNGraph(e0, e0, num_nodes=5)
g0.plan()
subs = [gnn.remove_edges(g, 0.3, seed=1), gnn.remove_nodes(g, 0.1, seed=2), gnn.remove_edges(g, 1.0),
        gnn.remove_nodes(g, 1.0), gnn.add_nodes(g, 9), gnn.remove_edges(g0, 0.5), gnn.remove_nodes(g0, [2]),
        gnn.add_nodes(g0, 3)]
for h in subs:
    f = gnn.GNNGraph(h.s, h.t, num_nodes=h.num_nodes)
    same = all(torch.equal(a, b) for tr in (False, True) for a, b in zip(gnn.csr(h, tr), gnn.csr(f, tr)))
    print("subgraph", h.num_nodes, h.num_edges, "derived == fresh", same)
keep = torch.empty(1001, dtype=torch.uint8, device="cuda")
gnn._lib.check(lib.gnnb_bernoulli_keep(1001, 0.5, 3, keep.data_ptr(), None))
print("bernoulli kept", int(keep.sum()), "of 1001")
# random_walk_pe: segments of 1, 5, 32 (small launch), 33 and 896 (medium launch) and 897 (propagate route), weighted
sizes = [1, 5, 32, 33, 896, 897]
S, T, off = [], [], 0
for m in sizes:
    S.append(torch.randint(0, m, (3 * m,), device="cuda") + off); T.append(torch.randint(0, m, (3 * m,), device="cuda") + off)
    off += m
s_, t_ = torch.cat(S), torch.cat(T)
gi = torch.repeat_interleave(torch.arange(1, len(sizes) + 1, device="cuda"), torch.tensor(sizes, device="cuda"))
gw = gnn.GNNGraph(s_ + 1, t_ + 1, torch.rand(s_.numel(), device="cuda") + 0.5, num_nodes=off, num_graphs=len(sizes),
                  graph_indicator=gi)
pe = gnn.random_walk_pe(gw, 6)
print("random_walk_pe", tuple(pe.shape), "finite", bool(torch.isfinite(pe).all()))
gx = gnn.GNNGraph(torch.cat([s_, torch.tensor([0], device="cuda")]) + 1, torch.cat([t_, torch.tensor([3], device="cuda")]) + 1,
                  num_nodes=off)                                   # an edge from the first segment into the second
deg = gnn.degree(gx, torch.float32, dir="out"); dinv = torch.where(deg != 0, 1 / deg, torch.zeros_like(deg))
seg = torch.cat([torch.zeros(1, dtype=torch.int64, device="cuda"), torch.cumsum(torch.tensor(sizes, device="cuda"), 0)])
out = torch.empty(off * 6, device="cuda")
rc = lib.gnnb_random_walk_pe(gx.plan().h, None, dinv.data_ptr(), seg.data_ptr(), len(sizes), 6, out.data_ptr(), None)
print("random_walk_pe crossing edge rejected", rc == gnn._lib.EINVAL)
# ppr_diffusion: segments of 1, 5, 32 (warp class), 33 and 240 (CTA class) and 241 (dense route: gnnb_ppr_matrix),
# weighted, then the same crossing edge, and every segment through the CTA class (variant 12)
sizes = [1, 5, 32, 33, 240, 241]
S, T, off = [], [], 0
for m in sizes:
    S.append(torch.randint(0, m, (3 * m,), device="cuda") + off); T.append(torch.randint(0, m, (3 * m,), device="cuda") + off)
    off += m
s_, t_ = torch.cat(S), torch.cat(T)
gi = torch.repeat_interleave(torch.arange(1, len(sizes) + 1, device="cuda"), torch.tensor(sizes, device="cuda"))
gw = gnn.GNNGraph(s_ + 1, t_ + 1, torch.rand(s_.numel(), device="cuda") * 0.5, num_nodes=off, num_graphs=len(sizes),
                  graph_indicator=gi)
print("ppr_diffusion", tuple(gnn.ppr_diffusion(gw).w.shape), "finite", bool(torch.isfinite(gnn.ppr_diffusion(gw).w).all()))
gnn._lib.check(lib.gnnb_set_kernel_variant(12))
print("ppr_diffusion CTA class only, finite", bool(torch.isfinite(gnn.ppr_diffusion(gw).w).all()))
gnn._lib.check(lib.gnnb_set_kernel_variant(0))
gx = gnn.GNNGraph(torch.cat([s_, torch.tensor([0], device="cuda")]) + 1, torch.cat([t_, torch.tensor([3], device="cuda")]) + 1,
                  num_nodes=off)                                   # an edge from the first segment into the second
seg = torch.cat([torch.zeros(1, dtype=torch.int64, device="cuda"), torch.cumsum(torch.tensor(sizes, device="cuda"), 0)])
w_out = torch.empty(gx.num_edges, device="cuda"); info = torch.empty(len(sizes), dtype=torch.int32, device="cuda")
rc = lib.gnnb_ppr_diffusion(gx.plan().h, None, 0.85, seg.data_ptr(), len(sizes), w_out.data_ptr(), info.data_ptr(), None)
M = torch.empty(5, 7, device="cuda")
rc2 = lib.gnnb_ppr_matrix(gx.plan().h, None, 0.85, 1, 6, 7, M.data_ptr(), None)
print("ppr_diffusion crossing edge rejected", rc == gnn._lib.EINVAL, rc2 == gnn._lib.EINVAL)
# laplacian_lambda_max: the same segments plus a ring in each (no isolated nodes), warp and CTA classes, the Lanczos
# route for the 241-node one above the bound (169), every segment through the CTA class, then the crossing edge
starts = [sum(sizes[:k]) for k in range(len(sizes))]
ring_s = torch.cat([torch.arange(m, device="cuda") + o for m, o in zip(sizes, starts)])
ring_t = torch.cat([(torch.arange(m, device="cuda") + 1) % m + o for m, o in zip(sizes, starts)])
gl = gnn.GNNGraph(torch.cat([s_, ring_s]) + 1, torch.cat([t_, ring_t]) + 1, num_nodes=off, num_graphs=len(sizes),
                  graph_indicator=gi)
print("laplacian_lambda_max", gnn.laplacian_lambda_max(gl).tolist())
gnn._lib.check(lib.gnnb_set_kernel_variant(12))
print("laplacian_lambda_max CTA class only", gnn.laplacian_lambda_max(gl).tolist())
gnn._lib.check(lib.gnnb_set_kernel_variant(0))
deg = gnn.degree(gx).float().contiguous() + 1
lm = torch.empty(len(sizes), dtype=torch.float64, device="cuda")
info = torch.empty(len(sizes), dtype=torch.int32, device="cuda")
rc = lib.gnnb_laplacian_lambda_max(gx.plan().h, None, deg.data_ptr(), 0, 1, seg.data_ptr(), len(sizes), lm.data_ptr(),
                                   info.data_ptr(), None)
print("laplacian_lambda_max crossing edge rejected", rc == gnn._lib.EINVAL)
# color_refinement: two hubs of 3 000 in-edges (pieces of 128 and the fix-up), a path of 41 nodes, a batch of small graphs
hs = torch.randint(0, 500, (6000,), device="cuda"); ht = torch.cat([torch.full((3000,), 7, device="cuda"),
                                                                   torch.full((3000,), 499, device="cuda")])
bs, bt = torch.randint(0, 500, (1500,), device="cuda"), torch.randint(0, 500, (1500,), device="cuda")
gh = gnn.GNNGraph(torch.cat([hs, bs]) + 1, torch.cat([ht, bt]) + 1, num_nodes=500)
print("color_refinement hubs", gnn.color_refinement(gh)[1:], gnn.color_refinement(gh, torch.arange(500, device="cuda") % 3)[1:])
a = torch.arange(40, device="cuda")
print("color_refinement path", gnn.color_refinement(gnn.GNNGraph(torch.cat([a, a + 1]) + 1, torch.cat([a + 1, a]) + 1,
                                                                 num_nodes=41))[1:])
ms, mt = torch.randint(0, 23, (200, 50), device="cuda"), torch.randint(0, 23, (200, 50), device="cuda")
off = (torch.arange(200, device="cuda") * 23)[:, None]
print("color_refinement batch", gnn.color_refinement(gnn.GNNGraph((ms + off).reshape(-1) + 1, (mt + off).reshape(-1) + 1,
                                                                  num_nodes=4600), max_iters=2)[1:])
# Set2Set: graphs of 127, 128, 129 nodes (chunk 128) and one without nodes, forward and backward at D = 1, 3, 1024, 1025
gi = torch.repeat_interleave(torch.tensor([1, 2, 4, 5], device="cuda"), torch.tensor([127, 128, 129, 1], device="cuda"))
a = torch.arange(1, gi.numel() + 1, device="cuda")
gs = gnn.GNNGraph(a, a, num_nodes=gi.numel(), num_graphs=5, graph_indicator=gi)
for Ds in (1, 3, 1024, 1025):
    l = gnn.Set2Set(Ds, 2, device="cuda")
    xs = torch.randn(Ds, gi.numel(), device="cuda").requires_grad_(True)
    ys = l(gs, xs)
    ys.sum().backward()
    print("set2set D", Ds, "empty graph r == 0", bool((ys[Ds:, 2] == 0).all()), "grad finite", bool(torch.isfinite(xs.grad).all()))
# attention pooling: the same graphs (127, 128, 129 nodes at chunk 128, one without nodes), forward and backward at
# D = 1, 3, 1024 (the fused entries) and 1025 (the composition)
for Da in (1, 3, 1024, 1025):
    fa = torch.randn(Da, gi.numel(), device="cuda").requires_grad_(True)
    ga = torch.randn(1, gi.numel(), device="cuda").requires_grad_(True)
    ua = gnn.GlobalAttentionPool(lambda v: ga, lambda v: fa)(gs, fa)
    ua.sum().backward()
    print("attention_pool D", Da, "empty graph u == 0", bool((ua[:, 2] == 0).all()), "grads finite",
          bool(torch.isfinite(fa.grad).all() and torch.isfinite(ga.grad).all()))
# recurrent gates: every entry at D = 1, 3, 64, 129 on a strided PX and with a 4-byte offset (the scalar path), then
# every temporal layer forward and backward on a small graph
from gnnb200._lib import lib as L, check as chk  # noqa: E402
st0 = torch.cuda.current_stream().cuda_stream
for Dr in (1, 3, 64, 129):
    for off in (0, 1):
        Nr = 300
        def rb(n):
            return torch.randn(n + off, device="cuda")[off:]
        ld3, ld4 = 3 * Dr + 4, 4 * Dr + 4
        px3, px4, ah2, ah, ah4, hr, cr, wr = (rb(Nr * ld3), rb(Nr * ld4), rb(Nr * 2 * Dr), rb(Nr * Dr), rb(Nr * 4 * Dr),
                                              rb(Nr * Dr), rb(Nr * Dr), rb(4 * Dr))
        r_, z_, rh_, n_, hn_, dz_, dh_ = (rb(Nr * Dr) for _ in range(7))
        dpx, gates, dpre = rb(Nr * 3 * Dr), rb(Nr * 4 * Dr), rb(Nr * 4 * Dr)
        dw, ws = rb(4 * Dr), rb(((Nr + 63) // 64) * 4 * Dr)
        P = lambda t: t.data_ptr()
        chk(L.gnnb_gru_rz(P(px3), ld3, P(ah2), P(hr), Nr, Dr, P(r_), P(z_), P(rh_), st0))
        for blend in (0, 1):
            chk(L.gnnb_gru_out(P(px3), ld3, P(ah), P(hr), P(z_), Nr, Dr, blend, P(n_), P(hn_), st0))
            chk(L.gnnb_gru_out_bwd(P(hn_), P(hr), P(z_), P(n_), Nr, Dr, blend, P(dpx) + 8 * Dr, 3 * Dr, P(dz_), P(dh_), st0))
            chk(L.gnnb_gru_rz_bwd(P(rh_), P(dz_), P(hr), P(r_), P(z_), Nr, Dr, P(dpx), 3 * Dr, P(dh_), st0))
        for peep in (True, False):
            chk(L.gnnb_lstm_cell(P(px4), ld4, P(ah4), P(cr), P(wr) if peep else None, Nr, Dr, P(gates), P(n_), P(hn_), st0))
            chk(L.gnnb_lstm_cell_bwd(P(hn_), P(n_), P(cr), P(gates), P(n_), P(wr) if peep else None, Nr, Dr, P(dpre),
                                     P(dz_), P(dw) if peep else None, P(ws) if peep else None, st0))
    print("recurrent gates D", Dr, "ok")
ar = torch.arange(60, device="cuda")
gr = gnn.GNNGraph(torch.cat([ar, (ar + 1) % 60]) + 1, torch.cat([(ar + 1) % 60, ar]) + 1, num_nodes=60)
for layer in (gnn.GConvGRU(3, 8, 3, device="cuda"), gnn.GConvLSTM(3, 8, 2, device="cuda"), gnn.DCGRU(3, 8, 2, device="cuda"),
              gnn.TGCN(3, 8, device="cuda"), gnn.EvolveGCNO(3, 8, device="cuda")):
    xr = gnn.colmajor(torch.randn(3, 5, 60, device="cuda")).requires_grad_(True)
    layer(gr, xr).sum().backward()
    print(repr(layer), "grad finite", bool(torch.isfinite(xr.grad).all()))
# two-sided GCN on relations: num_src >> num_dst, << num_dst, a row longer than the chunk, isolated sources and targets,
# forward and pullback at D = 3, 128, 1000
for ns_, nd_ in ((300, 7), (7, 300), (40, 30)):
    sh = torch.randint(1, ns_, (900,), device="cuda")
    th = torch.cat([torch.randint(1, nd_, (600,), device="cuda"), torch.ones(300, dtype=torch.int64, device="cuda")])
    hg = gnn.GNNHeteroGraph({("A", "r", "B"): (sh, th)}, num_nodes={"A": ns_, "B": nd_})
    for Dh in (3, 128, 1000):
        lh = gnn.GCNConv(Dh, 8, device="cuda")
        xh = torch.randn(Dh, ns_, device="cuda").requires_grad_(True)
        lh(hg, (xh, torch.randn(Dh, nd_, device="cuda"))).sum().backward()
        print("gcn bipartite", ns_, nd_, Dh, "grad finite", bool(torch.isfinite(xh.grad).all()))
    for heads_, C_ in ((1, 8), (8, 16), (3, 128)):                 # one-half logit passes, forward and pullback
        lg = gnn.GATConv(12, C_, heads=heads_, add_self_loops=False, device="cuda")
        xa = torch.randn(12, ns_, device="cuda").requires_grad_(True)
        xb = torch.randn(12, nd_, device="cuda").requires_grad_(True)
        lg(hg, (xa, xb)).sum().backward()
        print("gat bipartite", ns_, nd_, heads_, C_, "grad finite", bool(torch.isfinite(xa.grad).all() and torch.isfinite(xb.grad).all()))
# temporal generators: snapshots of 1 node, n = 127 and 129 (the query tile is 128), T = 1 for the radius generator,
# and the hyperbolic count / fill entries on records starting 8 B off the 16 B grid (head and tail of the bulk copy)
for n_, T_ in ((1, 3), (127, 4), (129, 4), (129, 1)):
    tg = gnn.rand_temporal_radius_graph(n_, T_, 0.3, 0.2, seed=n_)
    print("temporal radius", n_, T_, tg.num_edges)
    if T_ > 1:
        th = gnn.rand_temporal_hyperbolic_graph(n_, T_, α=1.0, R=4.0, speed=0.3, self_loop=n_ == 1, seed=n_)
        print("temporal hyperbolic", n_, T_, th.num_edges)
import ctypes as _C  # noqa: E402
recs = torch.empty(4 * 129 + 1, dtype=torch.float64, device="cuda")
gnn._lib.check(L.gnnb_temporal_hyperbolic_records(129, 1, 1.0, 4.0, 0.3, 1.0, 5, recs[1:].data_ptr(), st0))
offs = torch.empty(130, dtype=torch.int64, device="cuda"); tot = _C.c_int64(0)
gnn._lib.check(L.gnnb_hyperbolic_count(recs[1:].data_ptr(), 129, None, 1, 27.3, 0, offs.data_ptr(), _C.byref(tot), st0))
nb = torch.empty(max(tot.value, 1), dtype=torch.int32, device="cuda")
gnn._lib.check(L.gnnb_hyperbolic_fill(recs[1:].data_ptr(), 129, None, 1, 27.3, 0, offs.data_ptr(), nb.data_ptr(), tot.value,
                                      st0))
print("hyperbolic entries, misaligned records", tot.value)
# top-k pooling: both selection classes (a batch with empty and bound + 1 segments, the bound forced to 0), f64 keys,
# the gate and its pullback at D = 3 and 129 from a 4 B offset, and the layer in both forms
kv = torch.randn(9000, dtype=torch.float64, device="cuda")
segk = torch.tensor([0, 0, 23, 500, 500, 9000], dtype=torch.int64, device="cuda")
kp = torch.empty(9000, dtype=torch.uint8, device="cuda")
for b_ in (None, 0):
    if b_ is not None:
        gnn._lib.check(L.gnnb_topk_set_smem_max(b_))
    gnn._lib.check(L.gnnb_topk_keep(kv.data_ptr(), 1, 9000, segk.data_ptr(), 5, 0, 0.5, kp.data_ptr(), None, st0))
    print("topk keep, bound", b_, int(kp.sum()))
gnn._lib.lib.gnnb_topk_set_smem_max(8192)
gk = gnn.GNNGraph(torch.arange(1, 301, device="cuda"), torch.arange(300, 0, -1, device="cuda"), num_nodes=300,
                  num_graphs=3, graph_indicator=torch.arange(300, device="cuda") // 100 + 1)
for D_ in (3, 129):
    xb = torch.randn(300 * D_ + 1, device="cuda", requires_grad=True)
    xk = xb[1:].view(300, D_).t()
    tr = gnn.TopKPool(torch.rand(300, 300, device="cuda"), 7, D_, device="cuda")
    tr(xk).sum().backward()
    hk, xpk, _ = gnn.TopKPool(None, 0.3, D_, device="cuda")(gk, xk)
    xpk.sum().backward()
    print("topk both forms", D_, hk.num_nodes, bool(torch.isfinite(xb.grad).all()))
torch.cuda.synchronize()
print("done")
