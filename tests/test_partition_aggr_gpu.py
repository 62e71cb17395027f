"""Max / min aggregation and dist_propagate on the node-partitioned graph (partition.py: dist_propagate, dist_graph_conv,
dist_gin_conv, the max / min pullback gnnb_propagate_maxmin_bwd_halo) on the GPU.

One process, one plan (the halo split of an ordinary plan, chunks of 32 and 128 edges):
- the lean halo instances of the forward (mean, max, min, with and without weights, D = 128 / 256 / 512) give the bits
  of the reference kernel (gnnb_set_kernel_variant(12)) at every split point;
- gnnb_propagate_maxmin_bwd_halo on the reversed plan, split at every point, gives the bits of gnnb_propagate_bwd on the
  forward plan (the reversed plan's forward CSR is the forward plan's by-source CSR, row for row and chunk for chunk)
  and matches float64 element by element, at D = 1 ... 512, with ties, weights, a misaligned operand and empty rows;
- its argument errors.

With the multi-rank harness of test_partition_gpu.py (W gloo ranks on one device, or one rank per device under NCCL;
every ownership mode, with and without self loops, both halo routes, one and two push buffers), per rank:
- the shard forward of every aggregation against single-GPU gnnb_propagate: max and min bit for bit on every row, sum
  and mean on rows of at most one chunk, float64 elsewhere;
- the new entry on the real backward shard (a rank without nodes, a shard without halo) against float64 element by
  element, and against gnnb_propagate_bwd bit for bit on rows of at most one chunk;
- dist_propagate for + / mean / max / min x {copy_xj, w_mul_xj with the graph's weights, w_mul_xj with an explicit
  weight}: out, dx and d edge_weight against float64 and within 1e-5 of single-GPU propagate; GNNB_HALO_SLICES=2 gives
  the bits of 1 at D = 256 (slices of 128 floats run the same kernels: a slice narrow enough to leave the work-item
  pullback for the one-warp-per-row kernel adds long rows in another order);
- dist_graph_conv (every aggregation) and dist_gin_conv (+, max) against float64 autograd and the single-GPU layer;
- dist_sage_conv (mean, +) through the shared autograd function: single-GPU bits on short rows;
- three steps on one DistGraph equal fresh one-step runs bit for bit;
- the argument errors."""
import ctypes as C
import datetime
import os
import sys
import traceback

import numpy as np
import pytest
import torch

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
from test_partition_gpu import (CHUNK, N_NODES, ROOT, TOL_LAYER, TOL_LONG, Rank, Reference, assert_records,  # noqa: E402
                                bits_record, check_structure, make_graph, ownership_cases, rel_err,
                                require_shared_device, run_group)
from test_partition_weighted_gpu import build_weighted, make_weights  # noqa: E402

pytestmark = pytest.mark.gpu

SUM, MEAN, MAX, MIN = 0, 1, 2, 3
AGGRS = {SUM: "sum", MEAN: "mean", MAX: "max", MIN: "min"}
DS = (1, 5, 64, 128, 130, 256, 512)          # the generic kernel, the work-item kernel at 128 / 256 / 512
LAYERS = ((128, 256), (16, 7))               # Din < Dout, Din > Dout
EPS = 2.0 ** -24


def tie_features(n, D, gen, device):
    """features from a few small integers (most rows of max / min tie), some negative so that min and max differ"""
    return torch.randint(-2, 3, (n, D), generator=gen, device=device).float()


# ------------------------------------------------------------------------------------------------ float64 statements
def f64_forward(aggr, s, t, n, x, w):
    """propagate in float64 over the (s, t) edges; messages x[s] (* w)"""
    m = x.double()[s]
    if w is not None:
        m = m * w.double()[:, None]
    init = {SUM: 0.0, MEAN: 0.0, MAX: -float("inf"), MIN: float("inf")}[aggr]
    red = {SUM: "sum", MEAN: "mean", MAX: "amax", MIN: "amin"}[aggr]
    out = torch.full((n, x.shape[1]), init, dtype=torch.float64, device=x.device)
    return out.scatter_reduce(0, t[:, None].expand(-1, x.shape[1]), m, red, include_self=False)


def f64_maxmin_bwd(s, t, n_src, x, w, dout, out):
    """NNlib's rule: every tied extremum gets the gradient, each message compared as float32 (the kernel's product);
    returns (dx, the sum of the magnitudes of each dx's terms)"""
    wv = torch.ones(s.numel(), device=x.device) if w is None else w
    m32 = x[s] * wv[:, None]
    hit = (m32 == out[t]).double()
    terms = wv.double()[:, None] * dout.double()[t] * hit
    dx = torch.zeros((n_src, x.shape[1]), dtype=torch.float64, device=x.device).index_add_(0, s, terms)
    mag = torch.zeros_like(dx).index_add_(0, s, terms.abs())
    return dx, mag


def within_elementwise(got, ref, mag, nterms):
    """|got - ref| <= (nterms + 1) ulp-units of the magnitudes, per element; (ok, first bad flat index)"""
    tol = (nterms.double()[:, None] + 1) * EPS * mag
    bad = torch.nonzero(((got.double() - ref).abs() > tol).reshape(-1))
    return bad.numel() == 0, int(bad[0]) if bad.numel() else -1


# ------------------------------------------------------------------------------------------------ one process, one plan
@pytest.fixture(scope="module")
def gnn():
    if not torch.cuda.is_available():
        pytest.skip("no CUDA device")
    sys.path.insert(0, ROOT)
    import gnnb200
    return gnnb200


def plan_graph(chunk, seed=5):
    """~420 targets with rows of every special length (empty, c, c+1, 2c, 2c+1) among short ones, duplicate edges (ties
    whatever the features), COO order shuffled; sources spread over all nodes"""
    rng = np.random.default_rng(seed + chunk)
    n = 420
    lens = rng.integers(0, 7, n)
    special = rng.permutation(n)[:200]
    for k, L in enumerate((0, chunk, chunk + 1, 2 * chunk, 2 * chunk + 1)):
        lens[special[40 * k:40 * (k + 1)]] = L
    t = np.repeat(np.arange(n), lens)
    s = rng.integers(0, n, t.size)
    dup = rng.integers(0, t.size, 100)
    s, t = np.concatenate([s, s[dup]]), np.concatenate([t, t[dup]])
    p = rng.permutation(t.size)
    return s[p].astype(np.int32), t[p].astype(np.int32), n


def make_plan(gnn, src, dst, n):
    h = C.c_void_p()
    gnn._lib.check(gnn._lib.lib.gnnb_graph_create(C.byref(h), src.ctypes.data, dst.ctypes.data, src.size, n, n, 4, 0, 0,
                                                  None))
    return gnn.graph._Plan(h.value, torch.device("cuda", 0))


@pytest.fixture(scope="module", params=[32, 128], ids=["chunk32", "chunk128"])
def plans(gnn, request):
    lib = gnn._lib.lib
    gnn._lib.check(lib.gnnb_set_chunk_edges(request.param))
    try:
        s, t, n = plan_graph(request.param)
        fwd, rev = make_plan(gnn, s, t, n), make_plan(gnn, t, s, n)
    finally:
        gnn._lib.check(lib.gnnb_set_chunk_edges(128))
    dev = torch.device("cuda", 0)
    w = torch.as_tensor(np.random.default_rng(1).uniform(0.25, 2.0, s.size).astype(np.float32), device=dev)
    yield fwd, rev, torch.as_tensor(s, device=dev).long(), torch.as_tensor(t, device=dev).long(), n, w


def same(a, b):
    return a.shape == b.shape and torch.equal(a.contiguous().view(torch.int32), b.contiguous().view(torch.int32))


def halo_fwd(gnn, plan, aggr, x, w, split, D):
    out = torch.full((x.shape[0], D), float("nan"), device=x.device)
    msg = gnn._lib.COPY_XJ if w is None else gnn._lib.W_MUL_XJ
    x2 = x[split:].clone()
    gnn._lib.check(gnn._lib.lib.gnnb_propagate_halo(plan.h, msg, aggr, x.data_ptr() if split else None,
                                                    x2.data_ptr() if split < x.shape[0] else None, split,
                                                    None if w is None else w.data_ptr(), None, None, D, out.data_ptr(), None))
    torch.cuda.synchronize()
    return out


def test_lean_halo_forward_equals_reference_kernel(gnn, plans):
    """mean / max / min with a halo base at D = 128 / 256 / 512 run the lean instances: the bits of the round-1 kernel at
    every split point, with and without weights.  The plan has empty rows, which the lean path fills in a pass of its
    own and the round-1 kernel inside its one launch: a halo call makes the launches of the one-base call (split = n,
    long since on the lean kernel) and one more than the round-1 kernel."""
    fwd, rev, s, t, n, w = plans
    lib = gnn._lib.lib

    def counted(*a):
        before = gnn.launch_count()
        out = halo_fwd(gnn, *a)
        return out, gnn.launch_count() - before

    halo_fwd(gnn, fwd, MEAN, torch.zeros(n, 128, device="cuda"), None, n, 128)     # the plan's work items, built once
    for D in (128, 256, 512):
        x = torch.randn(n, D, device="cuda", generator=torch.Generator(device="cuda").manual_seed(D))
        for aggr in (MEAN, MAX, MIN):
            for wt in (None, w):
                _, one_base = counted(fwd, aggr, x, wt, n, D)
                for split in (0, 1, n // 3, n // 2, n - 1, n):
                    got, launches = counted(fwd, aggr, x, wt, split, D)
                    gnn._lib.check(lib.gnnb_set_kernel_variant(12))
                    try:
                        ref, ref_launches = counted(fwd, aggr, x, wt, split, D)
                    finally:
                        gnn._lib.check(lib.gnnb_set_kernel_variant(0))
                    name = f"{AGGRS[aggr]} w={wt is not None} D={D} split={split}"
                    assert same(got, ref), name
                    assert launches == one_base == ref_launches + 1, f"{name}: {launches} {one_base} {ref_launches} launches"


def maxmin_bwd_halo(gnn, rev, aggr, x, dout, out, w, split, D):
    dx = torch.full((x.shape[0], D), float("nan"), device=x.device)
    d2, o2 = dout[split:].clone(), out[split:].clone()
    halo = split < dout.shape[0]
    gnn._lib.check(gnn._lib.lib.gnnb_propagate_maxmin_bwd_halo(
        rev.h, gnn._lib.COPY_XJ if w is None else gnn._lib.W_MUL_XJ, aggr, x.data_ptr(),
        dout.data_ptr() if split else None, d2.data_ptr() if halo else None, out.data_ptr() if split else None,
        o2.data_ptr() if halo else None, split, None if w is None else w.data_ptr(), D, dx.data_ptr(), None))
    torch.cuda.synchronize()
    return dx


def one_gpu_bwd(gnn, fwd, aggr, x, dout, out, w, D):
    dx = torch.full_like(x, float("nan"))
    gnn._lib.check(gnn._lib.lib.gnnb_propagate_bwd(fwd.h, gnn._lib.COPY_XJ if w is None else gnn._lib.W_MUL_XJ, aggr,
                                                   dout.data_ptr(), x.data_ptr(), None if w is None else w.data_ptr(),
                                                   None, None, out.data_ptr(), D, dx.data_ptr(), None, None))
    return dx


def one_gpu_fwd(gnn, plan, aggr, x, w, D):
    out = torch.empty(x.shape[0], D, device=x.device)
    gnn._lib.check(gnn._lib.lib.gnnb_propagate(plan.h, 0, gnn._lib.COPY_XJ if w is None else gnn._lib.W_MUL_XJ, aggr,
                                               x.data_ptr(), None if w is None else w.data_ptr(), None, None, D,
                                               out.data_ptr(), None))
    return out


@pytest.mark.parametrize("D", DS)
def test_maxmin_bwd_halo_on_the_reversed_plan(gnn, plans, D):
    """the pullback on the reversed plan split at every point: gnnb_propagate_bwd's bits on the forward plan, and float64
    element by element (ties: every tied source gets the gradient; empty targets: out = -+Inf, gathered by no edge)"""
    fwd, rev, s, t, n, w = plans
    gen = torch.Generator(device="cuda").manual_seed(40 + D)
    outdeg = torch.bincount(s, minlength=n)
    for feats in ("ties", "normal"):
        x = tie_features(n, D, gen, "cuda") if feats == "ties" else torch.randn(n, D, device="cuda", generator=gen)
        dout = torch.randn(n, D, device="cuda", generator=gen)
        for aggr in (MAX, MIN):
            for wt in (None, w):
                out = one_gpu_fwd(gnn, fwd, aggr, x, wt, D)
                one = one_gpu_bwd(gnn, fwd, aggr, x, dout, out, wt, D)
                ref, mag = f64_maxmin_bwd(s, t, n, x, wt, dout, out)
                name = f"{feats} {AGGRS[aggr]} w={wt is not None} D={D}"
                if feats == "ties":
                    assert int((mag > 0).sum()) > 0, name
                for split in (0, 1, n // 2, n - 1, n):
                    dx = maxmin_bwd_halo(gnn, rev, aggr, x, dout, out, wt, split, D)
                    assert same(dx, one), f"{name} split={split}: not the bits of gnnb_propagate_bwd"
                    ok, at = within_elementwise(dx, ref, mag, outdeg)
                    assert ok, f"{name} split={split}: float64 bound fails at {at}"


def test_maxmin_bwd_halo_misaligned_operand(gnn, plans):
    """a misaligned x at D = 128: the one-warp-per-row kernel, with the bits of gnnb_propagate_bwd's (also generic)"""
    fwd, rev, s, t, n, w = plans
    D = 128
    gen = torch.Generator(device="cuda").manual_seed(3)
    x = torch.empty(n * D + 1, device="cuda")[1:].reshape(n, D)
    x.copy_(tie_features(n, D, gen, "cuda"))
    dout = torch.randn(n, D, device="cuda", generator=gen)
    for aggr in (MAX, MIN):
        out = one_gpu_fwd(gnn, fwd, aggr, x.contiguous(), w, D)
        one = one_gpu_bwd(gnn, fwd, aggr, x, dout, out, w, D)
        ref, mag = f64_maxmin_bwd(s, t, n, x, w, dout, out)
        dx = maxmin_bwd_halo(gnn, rev, aggr, x, dout, out, w, n // 2, D)
        assert same(dx, one)
        assert within_elementwise(dx, ref, mag, torch.bincount(s, minlength=n))[0]


def test_maxmin_bwd_halo_errors(gnn, plans):
    fwd, rev, s, t, n, w = plans
    lib, L = gnn._lib.lib, gnn._lib
    x = torch.randn(n, 8, device="cuda")
    p = x.data_ptr()
    call = lambda msg, aggr, xo, dl, dh, ol, oh, nl, ww, D, dx: lib.gnnb_propagate_maxmin_bwd_halo(
        rev.h, msg, aggr, xo, dl, dh, ol, oh, nl, ww, D, dx, None)
    assert call(L.COPY_XJ, L.SUM, p, p, p, p, p, n // 2, None, 8, p) == L.EINVAL
    assert call(L.COPY_XJ, L.MEAN, p, p, p, p, p, n // 2, None, 8, p) == L.EINVAL
    assert call(L.COPY_XJ, L.MAX, p, p, None, p, p, n // 2, None, 8, p) == L.EINVAL      # halo targets, no dout_halo
    assert call(L.COPY_XJ, L.MAX, p, None, p, p, p, n // 2, None, 8, p) == L.EINVAL      # local targets, no dout_local
    assert call(L.COPY_XJ, L.MAX, p, p, p, p, p, n + 1, None, 8, p) == L.ESIZE
    assert call(L.COPY_XJ, L.MAX, p, p, p, p, p, n // 2, None, 0, p) == L.ESIZE
    assert call(L.W_MUL_XJ, L.MAX, p, p, p, p, p, n // 2, None, 8, p) == L.EINVAL        # w_mul_xj without weights
    assert call(L.COPY_XJ, L.MAX, None, p, p, p, p, n // 2, None, 8, p) == L.EINVAL
    # a plan without rows (a rank that owns no node): NULL everything
    h = C.c_void_p()
    gnn._lib.check(lib.gnnb_graph_create(C.byref(h), None, None, 0, 0, 0, 4, 0, 1, None))
    empty = gnn.graph._Plan(h.value, torch.device("cuda", 0))
    gnn._lib.check(lib.gnnb_propagate_maxmin_bwd_halo(empty.h, L.COPY_XJ, L.MAX, None, None, None, None, None, 0, None, 8,
                                                      None, None))


# ------------------------------------------------------------------------------------------------ multi-rank: references
class AggrFull:
    """the whole weighted graph (loops of weight 1 appended when the partition has them) on one GPU and in float64"""

    def __init__(self, R, G, w, loops):
        gnn, n = R.gnn, N_NODES
        s, t, wl = G["s"], G["t"], w
        if loops:
            s, t, wl = np.concatenate([s, np.arange(n)]), np.concatenate([t, np.arange(n)]), np.concatenate([w, np.ones(n, np.float32)])
        self.s, self.t = torch.as_tensor(s, device=R.dev), torch.as_tensor(t, device=R.dev)
        self.w = torch.as_tensor(wl, device=R.dev)
        self.g = gnn.GNNGraph(torch.as_tensor(s + 1), torch.as_tensor(t + 1), torch.as_tensor(wl), num_nodes=n).cuda()
        self.g_plain = gnn.GNNGraph(torch.as_tensor(s + 1), torch.as_tensor(t + 1), num_nodes=n).cuda()
        self.plan = self.g.plan()
        self.indeg = torch.bincount(self.t, minlength=n)
        self.outdeg = torch.bincount(self.s, minlength=n)
        self.R = R

    def fwd(self, aggr, x, w):
        return one_gpu_fwd(self.R.gnn, self.plan, aggr, x, w, x.shape[1])

    def bwd(self, aggr, x, dout, out, w):
        return one_gpu_bwd(self.R.gnn, self.plan, aggr, x, dout, out, w, x.shape[1])


def f64_pullback(aggr, full, x, w, dout, out):
    """(dx, dw) of propagate in float64: + / mean by the linear rule, max / min by NNlib's tie rule (dw None there)"""
    s, t, n = full.s, full.t, N_NODES
    if aggr in (MAX, MIN):
        return f64_maxmin_bwd(s, t, n, x, w, dout, out)[0], None
    wv = torch.ones(s.numel(), dtype=torch.float64, device=x.device) if w is None else w.double()
    g = dout.double()[t]
    if aggr == MEAN:
        g = g / full.indeg.double().clamp(min=1)[t][:, None]
    dx = torch.zeros((n, x.shape[1]), dtype=torch.float64, device=x.device).index_add_(0, s, g * wv[:, None])
    return dx, (g * x.double()[s]).sum(1)


# ------------------------------------------------------------------------------------------------ multi-rank: checks
def check_forward(R, tag, dg, full, halos):
    """the shard forward of every aggregation against gnnb_propagate on the whole graph"""
    ids = dg.local_nodes()
    short = full.indeg[ids] <= CHUNK
    for D in (1, 5, 128, 256, 260, 512):
        x = torch.randn(N_NODES, D, device=R.dev, generator=torch.Generator(device=R.dev).manual_seed(500 + D))
        xl = x[ids].contiguous()
        for aggr in AGGRS:
            for wname, ws, wf in (("copy", None, None), ("w", dg.w_fwd, full.w)):
                name = f"forward/{tag}/{AGGRS[aggr]}/{wname}/D{D}"
                got = dg.propagate(dg.fwd, xl, None, None, aggr, w=ws)
                one = full.fwd(aggr, x, wf)[ids]
                if aggr in (MAX, MIN):
                    R.put(f"{name}/bits_one_gpu", *bits_record(got, one))
                else:
                    R.put(f"{name}/short_rows_bits_one_gpu", *bits_record(got[short], one[short]))
                    err, at = rel_err(got[~short], f64_forward(aggr, full.s, full.t, N_NODES, x, wf)[ids][~short])
                    R.put(f"{name}/long_rows_f64", err <= TOL_LONG, err, at)


def check_entry(R, tag, dg, full, halos):
    """gnnb_propagate_maxmin_bwd_halo on this rank's backward shard: float64 element by element, and the bits of
    gnnb_propagate_bwd on rows of at most one chunk"""
    ids = dg.local_nodes()
    sh, nl = dg.bwd, dg.n_local
    short = full.outdeg[ids] <= CHUNK
    for D in DS:
        gen = torch.Generator(device=R.dev).manual_seed(600 + D)
        for feats in ("ties", "normal"):
            x = tie_features(N_NODES, D, gen, R.dev) if feats == "ties" else torch.randn(N_NODES, D, device=R.dev, generator=gen)
            dout = torch.randn(N_NODES, D, device=R.dev, generator=gen)
            for aggr in (MAX, MIN):
                for wname, wb, wf in (("copy", None, None), ("w", dg.w_bwd, full.w)):
                    name = f"entry/{tag}/{feats}/{AGGRS[aggr]}/{wname}/D{D}"
                    out = full.fwd(aggr, x, wf)
                    xl, dl, ol = x[ids].contiguous(), dout[ids].contiguous(), out[ids].contiguous()
                    dh, oh = dout[halos[1]].contiguous(), out[halos[1]].contiguous()
                    dx = torch.full((nl, D), float("nan"), device=R.dev)
                    R.gnn._lib.check(R.gnn._lib.lib.gnnb_propagate_maxmin_bwd_halo(
                        sh.plan.h, R.gnn._lib.COPY_XJ if wb is None else R.gnn._lib.W_MUL_XJ, aggr, xl.data_ptr(),
                        dl.data_ptr(), dh.data_ptr() if sh.n_halo else None, ol.data_ptr(),
                        oh.data_ptr() if sh.n_halo else None, nl, None if wb is None else wb.data_ptr(), D,
                        dx.data_ptr(), R.stream()))
                    ref, mag = f64_maxmin_bwd(full.s, full.t, N_NODES, x, wf, dout, out)
                    ok, at = within_elementwise(dx, ref[ids], mag[ids], full.outdeg[ids])
                    R.put(f"{name}/f64_element_by_element", ok, 0.0, at)
                    one = full.bwd(aggr, x, dout, out, wf)[ids]
                    R.put(f"{name}/short_rows_bits_one_gpu", *bits_record(dx[short], one[short]))


def dist_prop_step(R, dg, f, aggr, x_full, dout_full, ew_global=None):
    """dist_propagate forward and backward on this rank's rows: out, dx and the edge-weight gradient placed back in the
    global list and all-reduced"""
    import torch.distributed as dist
    gnn = R.gnn
    ids = dg.local_nodes()
    x = gnn.unrows(x_full[ids].contiguous()).requires_grad_(True)
    ew, mask = None, None
    if ew_global is not None:
        mask = dg.owned_by_target(torch.as_tensor(R.G["t"] + 1, device=R.dev))
        ew = ew_global[mask].clone().requires_grad_(aggr in (SUM, MEAN))
    y = R.P.dist_propagate(f, dg, AGGRS[aggr], x, ew)
    y.backward(gnn.unrows(dout_full[ids].contiguous()))
    res = [gnn.rows(y.detach()).clone(), gnn.rows(x.grad).clone()]
    if ew is not None and ew.requires_grad:
        dw = torch.zeros(ew_global.numel(), device=R.dev)
        dw[mask] = ew.grad
        dist.all_reduce(dw)
        res.append(dw)
    return res


def check_dist_propagate(R, tag, dg, full):
    gnn = R.gnn
    ids = dg.local_nodes()
    E = R.G["s"].size
    w_glob = full.w[:E]
    for D in (7, 256):                                          # 256: two column slices of 128 keep the lean kernels
        gen = torch.Generator(device=R.dev).manual_seed(700 + D)
        x_full = torch.randn(N_NODES, D, device=R.dev, generator=gen)
        dout_full = torch.randn(N_NODES, D, device=R.dev, generator=gen)
        for aggr in AGGRS:
            for mode in ("copy_xj", "w_graph", "w_explicit"):
                name = f"propagate/{tag}/{AGGRS[aggr]}/{mode}/D{D}"
                f = gnn.copy_xj if mode == "copy_xj" else gnn.w_mul_xj
                ew = w_glob if mode == "w_explicit" else None
                got = dist_prop_step(R, dg, f, aggr, x_full, dout_full, ew)
                # single-GPU propagate on the whole graph (the explicit weight as e_mul_xj's edge vector)
                xg = gnn.unrows(x_full.clone()).requires_grad_(True)
                wg = None
                if mode == "copy_xj":
                    yg = gnn.propagate(gnn.copy_xj, full.g, AGGRS[aggr], xj=xg)
                elif mode == "w_graph":
                    yg = gnn.propagate(gnn.w_mul_xj, full.g, AGGRS[aggr], xj=xg)
                else:
                    wg = full.w.clone().requires_grad_(aggr in (SUM, MEAN))
                    yg = gnn.propagate(gnn.e_mul_xj, full.g_plain, AGGRS[aggr], xj=xg, e=wg)
                yg.backward(gnn.unrows(dout_full.clone()))
                one = [gnn.rows(yg.detach())[ids], gnn.rows(xg.grad)[ids]]
                wf = None if mode == "copy_xj" else full.w
                out64 = f64_forward(aggr, full.s, full.t, N_NODES, x_full, wf)
                out32 = full.fwd(aggr, x_full, wf)
                dx64, dw64 = f64_pullback(aggr, full, x_full, wf, dout_full, out32)
                ref = [out64[ids], dx64[ids]]
                if len(got) == 3:
                    one.append(wg.grad[:E])
                    ref.append(dw64[:E])
                for k, a, b, r in zip(("out", "dx", "dedge_weight"), got, one, ref):
                    err, at = rel_err(a, b)
                    R.put(f"{name}/{k}/one_gpu", err <= TOL_LAYER, err, at)
                    err, at = rel_err(a, r)
                    R.put(f"{name}/{k}/f64", err <= TOL_LAYER, err, at)
                if mode == "w_graph":                               # column slices: the same bits
                    R.set_route("push", 2)
                    sliced = dist_prop_step(R, dg, f, aggr, x_full, dout_full)
                    R.set_route()
                    for k, a, b in zip(("out", "dx"), sliced, got):
                        R.put(f"{name}/{k}/sliced_bits_unsliced", *bits_record(a, b))
                    R.set_route("nccl")
                    routed = dist_prop_step(R, dg, f, aggr, x_full, dout_full)
                    R.set_route()
                    for k, a, b in zip(("out", "dx"), routed, got):
                        R.put(f"{name}/{k}/alltoall_bits_push", *bits_record(a, b))


def gin_nn(R, Din, Dout):
    torch.manual_seed(31 * Din + Dout)
    W = (torch.randn(Dout, Din, device=R.dev) / Din ** 0.5).requires_grad_(True)
    b = torch.linspace(-0.5, 0.5, Dout, device=R.dev).requires_grad_(True)
    return (lambda h: torch.tanh(W @ h + b[:, None])), [W, b]


def layer_step(R, dg, fn, params, x_full, dy_full):
    import torch.distributed as dist
    gnn = R.gnn
    ids = dg.local_nodes()
    for p in params:
        p.grad = None
    x = gnn.unrows(x_full[ids].contiguous()).requires_grad_(True)
    y = fn(dg, x)
    y.backward(gnn.unrows(dy_full[ids].contiguous()))
    grads = [p.grad.clone() for p in params]
    for g in grads:
        dist.all_reduce(g)
    return [gnn.rows(y.detach()).clone(), gnn.rows(x.grad).clone()] + grads


def dense_f64(aggr, full, x64):
    """propagate(copy_xj) in float64 as a differentiable expression; max / min through a gather of the float32 winners'
    mask, so that every tie gets the whole gradient (NNlib's rule, not torch's even split)"""
    s, t = full.s, full.t
    if aggr in (SUM, MEAN):
        out = torch.zeros_like(x64).index_add(0, t, x64[s])
        if aggr == MEAN:
            out = out / full.indeg.double().clamp(min=1)[:, None]
        return out
    out32 = f64_forward(aggr, s, t, N_NODES, x64.detach(), None)
    hit = (x64.detach()[s] == out32[t]).double()
    val = torch.zeros_like(x64).index_add(0, t, x64[s] * hit)        # value path: the sum over winners
    cnt = torch.zeros_like(x64).index_add(0, t, hit)
    return torch.where(cnt > 0, out32 + (val - val.detach()), out32)


def check_layers(R, tag, dg, full):
    gnn = R.gnn
    ids = dg.local_nodes()
    names = ("y", "dx", "dp1", "dp2", "dp3")
    for Din, Dout in LAYERS:
        gen = torch.Generator(device=R.dev).manual_seed(7 * Din + Dout)
        x_full = torch.randn(N_NODES, Din, device=R.dev, generator=gen)
        dy_full = torch.randn(N_NODES, Dout, device=R.dev, generator=gen)
        cases = []
        for aggr in AGGRS:
            torch.manual_seed(1000 * Din + Dout)
            l = gnn.GraphConv(Din, Dout, torch.tanh, aggr=AGGRS[aggr], device=R.dev)
            with torch.no_grad():
                l.bias.copy_(torch.linspace(-0.5, 0.5, Dout))
            cases.append((f"graph_conv/{AGGRS[aggr]}", aggr, l, [l.weight1, l.weight2, l.bias], R.P.dist_graph_conv))
        for aggr in (SUM, MAX):
            nn, ps = gin_nn(R, Din, Dout)
            l = gnn.GINConv(nn, 0.25, aggr=AGGRS[aggr])
            cases.append((f"gin_conv/{AGGRS[aggr]}", aggr, l, ps, R.P.dist_gin_conv))
        for cname, aggr, l, ps, dist_fn in cases:
            name = f"layers/{tag}/{Din}to{Dout}/{cname}"
            got = layer_step(R, dg, lambda d, x: dist_fn(l, d, x), ps, x_full, dy_full)
            for p in ps:
                p.grad = None
            xg = gnn.unrows(x_full.clone()).requires_grad_(True)
            yg = l(full.g_plain, xg)
            yg.backward(gnn.unrows(dy_full.clone()))
            one = [gnn.rows(yg.detach())[ids], gnn.rows(xg.grad)[ids]] + [p.grad.clone() for p in ps]
            # float64 autograd of the dense formula
            x64 = x_full.double().requires_grad_(True)
            p64 = [p.detach().double().requires_grad_(True) for p in ps]
            m = dense_f64(aggr, full, x64)
            if cname.startswith("graph"):
                y64 = torch.tanh(x64 @ p64[0].t() + m @ p64[1].t() + p64[2])
            else:
                y64 = torch.tanh((1.25 * x64 + m) @ p64[0].t() + p64[1])
            y64.backward(dy_full.double())
            ref = [y64.detach()[ids], x64.grad[ids]] + [p.grad for p in p64]
            for k, a, b, r in zip(names, got, one, ref):
                err, at = rel_err(a, b)
                R.put(f"{name}/{k}/one_gpu", err <= TOL_LAYER, err, at)
                err, at = rel_err(a, r)
                R.put(f"{name}/{k}/f64", err <= TOL_LAYER, err, at)


def check_sage(R, tag, dg, full):
    """dist_sage_conv through _DistPropagateFn: the single-GPU sage_conv bits on rows of at most one chunk"""
    gnn = R.gnn
    ids = dg.local_nodes()
    short_t = full.indeg[ids] <= CHUNK
    for aggr in ("mean", "+"):
        torch.manual_seed(3)
        l = gnn.SAGEConv(128, 128, torch.relu, aggr=gnn.mean if aggr == "mean" else "+", device=R.dev)
        gen = torch.Generator(device=R.dev).manual_seed(11)
        x_full = torch.randn(N_NODES, 128, device=R.dev, generator=gen)
        dy_full = torch.randn(N_NODES, 128, device=R.dev, generator=gen)
        got = layer_step(R, dg, lambda d, x: R.P.dist_sage_conv(l, d, x), [l.weight, l.bias], x_full, dy_full)
        l.zero_grad(set_to_none=True)
        xg = gnn.unrows(x_full.clone()).requires_grad_(True)
        yg = l(full.g_plain, xg)
        yg.backward(gnn.unrows(dy_full.clone()))
        name = f"sage/{tag}/{aggr}"
        R.put(f"{name}/y_short_rows_bits_one_gpu", *bits_record(got[0][short_t], gnn.rows(yg.detach())[ids][short_t]))
        err, at = rel_err(got[1], gnn.rows(xg.grad)[ids])
        R.put(f"{name}/dx_one_gpu", err <= TOL_LAYER, err, at)


def check_steps(R, G, w, own):
    """three dist_propagate max and dist_graph_conv steps with different x on one DistGraph equal fresh one-step runs bit
    for bit, with two push buffers and with one"""
    gnn = R.gnn
    for nbuf in ("2", "1"):
        os.environ["GNNB_HALO_BUFFERS"] = nbuf
        torch.manual_seed(9)
        l = gnn.GraphConv(128, 128, torch.tanh, aggr="max", device=R.dev)
        xs = [torch.randn(N_NODES, 128, device=R.dev, generator=torch.Generator(device=R.dev).manual_seed(50 + k)) for k in range(3)]
        dy = torch.randn(N_NODES, 128, device=R.dev, generator=torch.Generator(device=R.dev).manual_seed(49))
        run = lambda d, x: (dist_prop_step(R, d, gnn.w_mul_xj, MIN, x, dy)
                            + layer_step(R, d, lambda dd, xx: R.P.dist_graph_conv(l, dd, xx), [l.weight1, l.weight2, l.bias], x, dy))
        dg, _ = build_weighted(R, G, w, False, False, **own)
        steps = [run(dg, x) for x in xs]
        dg.close()
        for k, x in enumerate(xs):
            fresh, _ = build_weighted(R, G, w, False, False, **own)
            once = run(fresh, x)
            fresh.close()
            for i, (a, b) in enumerate(zip(steps[k], once)):
                R.put(f"steps/{own['ownership']}/buffers{nbuf}/step{k}/{i}", *bits_record(a, b))
    os.environ["GNNB_HALO_BUFFERS"] = "2"


def check_errors(R, dg):
    gnn, P = R.gnn, R.P
    x = gnn.unrows(torch.randn(dg.n_local, 8, device=R.dev))
    ew = torch.ones(dg.num_owned_edges, device=R.dev, requires_grad=True)
    l = gnn.GraphConv(8, 8, device=R.dev)
    gl = gnn.GINConv(lambda h: h, 0.0)
    cases = {"message": lambda: P.dist_propagate(gnn.xi_sub_xj, dg, "+", x),
             "edge_weight_length": lambda: P.dist_propagate(gnn.w_mul_xj, dg, "+", x, torch.ones(dg.num_owned_edges + 1, device=R.dev)),
             "copy_xj_with_weight": lambda: P.dist_propagate(gnn.copy_xj, dg, "+", x, ew),
             "max_weight_grad": lambda: P.dist_propagate(gnn.w_mul_xj, dg, "max", x, ew),
             "min_weight_grad": lambda: P.dist_propagate(gnn.w_mul_xj, dg, "min", x, ew),
             "aggregation": lambda: P.dist_propagate(gnn.copy_xj, dg, "prod", x)}
    if dg.self_loops:
        cases["graph_conv_loops"] = lambda: P.dist_graph_conv(l, dg, x)
        cases["gin_conv_loops"] = lambda: P.dist_gin_conv(gl, dg, x)
    for name, f in cases.items():
        try:
            f()
            ok = False
        except ValueError:
            ok = True
        R.put(f"errors/{'loops' if dg.self_loops else 'noloops'}/{name}", ok)


def run_cases(R, multi_device):
    G = dict(zip(("s", "t"), make_graph()))
    R.G = G
    w = make_weights(G)
    ring = np.arange(N_NODES)
    GR = {"s": np.concatenate([G["s"], (ring + 1) % N_NODES]), "t": np.concatenate([G["t"], ring])}
    wr = make_weights(GR)
    cases = ownership_cases(R.W) if R.W > 1 else [(o, dict(ownership=o)) for o in ("contiguous", "cyclic", "balanced")]
    for tag, own in cases:
        for loops in (True, False):
            full_tag = f"W{R.W}/{tag}/{'loops' if loops else 'noloops'}"
            full = AggrFull(R, G, w, loops)
            dg, req = build_weighted(R, G, w, loops, False, **own)
            halos = check_structure(R, full_tag, dg, req, Reference(R, G, loops))
            check_forward(R, full_tag, dg, full, halos)
            check_entry(R, full_tag, dg, full, halos)
            check_dist_propagate(R, full_tag, dg, full)
            if not loops:
                check_sage(R, full_tag, dg, full)
                # the layers on the graph plus a ring, so that every node has an in-edge: max / min without -Inf rows,
                # whose NaN would reach every entry of W2's gradient
                dr, _ = build_weighted(R, GR, wr, False, False, **own)
                check_layers(R, full_tag, dr, AggrFull(R, GR, wr, False))
                dr.close()
            check_errors(R, dg)
            dg.close()
    if R.W > 1:
        for tag, own in ownership_cases(R.W)[1:3]:
            check_steps(R, G, w, own)


def aggr_worker(rank, W, port, q, multi_device):
    import torch.distributed as dist
    os.environ.update(MASTER_ADDR="127.0.0.1", MASTER_PORT=str(port), GNNB_HALO="push", GNNB_HALO_SLICES="1",
                      GNNB_HALO_BUFFERS="2")
    dev = torch.device("cuda", rank if multi_device else 0)
    torch.cuda.set_device(dev)
    try:
        dist.init_process_group("nccl" if multi_device else "gloo", rank=rank, world_size=W,
                                timeout=datetime.timedelta(seconds=300), device_id=dev if multi_device else None)
        R = Rank(rank, W, q, dev)
        run_cases(R, multi_device)
        torch.cuda.synchronize(dev)
        dist.barrier()
        q.put(("done", rank, True, 0.0, -1))
    except BaseException:
        q.put(("error", rank, False, 0.0, traceback.format_exc()[-4000:]))
    finally:
        if dist.is_initialized():
            dist.destroy_process_group()


FAMILIES = ["forward", "entry", "propagate", "layers", "sage", "steps", "errors"]


@pytest.mark.parametrize("W", [1, 2, 3, 4])
@pytest.mark.parametrize("check", FAMILIES)
def test_aggr_partition_on_one_device(W, check):
    """W gloo ranks on one device: `check` names the family of records"""
    require_shared_device()
    if W == 1 and check == "steps":
        pytest.skip("the repeated-steps check runs at W > 1")
    assert_records(*run_group(aggr_worker, W, False, timeout=1800), prefix=check + "/")


def test_aggr_partition_one_rank_per_device_nccl():
    """one rank per device under NCCL, the push route over real peer mappings"""
    if not torch.cuda.is_available() or torch.cuda.device_count() < 2:
        pytest.skip("needs at least two visible CUDA devices: NCCL refuses two ranks on one device")
    W = min(torch.cuda.device_count(), 4)
    records, errors, codes = run_group(aggr_worker, W, True, timeout=1800)
    for prefix in FAMILIES:
        assert_records(records, errors, codes, prefix + "/")
