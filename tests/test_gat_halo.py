"""The HALO instances of the fused GAT kernels (csrc/gat.cu) against the one-base instances, bit for bit, in one process.

Forward: gnnb_gat_aggregate_halo with the gathered rows split at `split` (the tail either at its place in Wx or in a
separately allocated copy) equals gnnb_gat_aggregate (out, seg_max, seg_sum).  Pullback: gnnb_gat_aggregate_bwd_halo on
the REVERSED plan (its forward CSR is the plan's by-source CSR) equals gnnb_gat_aggregate_bwd: dWx and der bit for bit,
and gnnb_scatter of its dz (COO order) is del bit for bit.  Every lean shape (rows of 128, 256, 512 floats), round-1
shapes (vector and scalar), both kernel variants, and graphs with empty rows and rows of c, c+1, 2c and 2c+1 edges at
chunks c = 32 and 128."""
import ctypes as C
import os
import sys

import numpy as np
import pytest
import torch

pytestmark = pytest.mark.gpu

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
SHAPES = [(32, 4), (64, 4), (64, 8), (16, 3), (8, 5), (2, 8), (1, 8)]   # (C, H): lean D = 128 / 256 / 512, then round-1
SLOPE = 0.2


@pytest.fixture(scope="module")
def gnn():
    if not torch.cuda.is_available():
        pytest.skip("no CUDA device")
    sys.path.insert(0, ROOT)
    import gnnb200
    return gnnb200


def make_graph(chunk, seed=3):
    """~40 rows of every special length (empty, c, c+1, 2c, 2c+1) among rows of 0..6 edges; sources spread over all
    nodes, COO order shuffled"""
    rng = np.random.default_rng(seed + chunk)
    n = 420
    lens = rng.integers(0, 7, n)
    special = rng.permutation(n)[:200]
    for k, L in enumerate((0, chunk, chunk + 1, 2 * chunk, 2 * chunk + 1)):
        lens[special[40 * k:40 * (k + 1)]] = L
    t = np.repeat(np.arange(n), lens)
    s = rng.integers(0, n, t.size)
    p = rng.permutation(t.size)
    return s[p].astype(np.int32), t[p].astype(np.int32), n


def plan(gnn, src, dst, n):
    h = C.c_void_p()
    gnn._lib.check(gnn._lib.lib.gnnb_graph_create(C.byref(h), src.ctypes.data, dst.ctypes.data, src.size, n, n, 4, 0, 0,
                                                  None))
    return gnn.graph._Plan(h.value, torch.device("cuda", 0))


def same(a, b):
    return a.shape == b.shape and torch.equal(a.contiguous().view(torch.int32), b.contiguous().view(torch.int32))


@pytest.fixture(scope="module", params=[(32, 0), (128, 0), (128, 12)], ids=["chunk32", "chunk128", "chunk128-variant12"])
def graphs(gnn, request):
    chunk, variant = request.param
    lib = gnn._lib.lib
    gnn._lib.check(lib.gnnb_set_chunk_edges(chunk))
    try:
        s, t, n = make_graph(chunk)
        fwd, rev = plan(gnn, s, t, n), plan(gnn, t, s, n)
    finally:
        gnn._lib.check(lib.gnnb_set_chunk_edges(128))
    gnn._lib.check(lib.gnnb_set_kernel_variant(variant))
    yield fwd, rev, n
    gnn._lib.check(lib.gnnb_set_kernel_variant(0))


def tensors(n, Cc, H, seed):
    g = torch.Generator(device="cuda").manual_seed(seed)
    r = lambda *shape: torch.randn(*shape, device="cuda", generator=g)
    return r(n, H, Cc), r(n, H), r(n, H), r(n, H, Cc)


@pytest.mark.parametrize("shape", SHAPES, ids=[f"C{c}H{h}" for c, h in SHAPES])
def test_forward_halo_equals_one_base(gnn, graphs, shape):
    fwd, _, n = graphs
    lib, Cc, H = gnn._lib.lib, *shape
    Wx, el, er, _ = tensors(n, Cc, H, 10 * Cc + H)
    D = Cc * H
    ref = [torch.empty(n, H, Cc, device="cuda"), torch.empty(n, H, device="cuda"), torch.empty(n, H, device="cuda")]
    gnn._lib.check(lib.gnnb_gat_aggregate(fwd.h, Wx.data_ptr(), el.data_ptr(), er.data_ptr(), Cc, H, SLOPE, ref[0].data_ptr(),
                                          None, ref[1].data_ptr(), ref[2].data_ptr(), None))
    for split in (0, 1, n // 2, n - 1, n):
        for tail in ("in_place", "copy"):
            x2 = Wx[split:] if tail == "in_place" else Wx[split:].clone()
            got = [torch.full_like(r, float("nan")) for r in ref]
            gnn._lib.check(lib.gnnb_gat_aggregate_halo(fwd.h, Wx.data_ptr(), x2.data_ptr() if split < n else None, split,
                                                       el.data_ptr(), er.data_ptr(), Cc, H, SLOPE, got[0].data_ptr(),
                                                       got[1].data_ptr(), got[2].data_ptr(), None))
            torch.cuda.synchronize()
            for name, a, b in zip(("out", "seg_max", "seg_sum"), got, ref):
                assert same(a, b), f"{name} split={split} {tail} D={D}"


@pytest.mark.parametrize("shape", SHAPES, ids=[f"C{c}H{h}" for c, h in SHAPES])
def test_pullback_on_reversed_plan_equals_one_base(gnn, graphs, shape):
    fwd, rev, n = graphs
    lib, Cc, H = gnn._lib.lib, *shape
    Wx, el, er, dout = tensors(n, Cc, H, 100 + 10 * Cc + H)
    out, smax, ssum = torch.empty(n, H, Cc, device="cuda"), torch.empty(n, H, device="cuda"), torch.empty(n, H, device="cuda")
    gnn._lib.check(lib.gnnb_gat_aggregate(fwd.h, Wx.data_ptr(), el.data_ptr(), er.data_ptr(), Cc, H, SLOPE, out.data_ptr(),
                                          None, smax.data_ptr(), ssum.data_ptr(), None))
    dWx, dl, dr = torch.empty_like(Wx), torch.empty_like(el), torch.empty_like(er)
    gnn._lib.check(lib.gnnb_gat_aggregate_bwd(fwd.h, Wx.data_ptr(), el.data_ptr(), er.data_ptr(), smax.data_ptr(),
                                              ssum.data_ptr(), out.data_ptr(), dout.data_ptr(), Cc, H, SLOPE, dWx.data_ptr(),
                                              dl.data_ptr(), dr.data_ptr(), None))
    T = torch.empty_like(el)
    gnn._lib.check(lib.gnnb_gat_tnode(dout.data_ptr(), out.data_ptr(), n, Cc, H, T.data_ptr(), None))
    ne, ns, nd = C.c_int64(), C.c_int64(), C.c_int64()
    gnn._lib.check(lib.gnnb_graph_info(rev.h, C.byref(ne), C.byref(ns), C.byref(nd)))
    E = ne.value
    for split in (0, 1, n // 2, n - 1, n):
        for tail in ("in_place", "copy"):
            d2 = dout[split:] if tail == "in_place" else dout[split:].clone()
            gW, gr = torch.full_like(dWx, float("nan")), torch.full_like(dr, float("nan"))
            dz = torch.full((E, H), float("nan"), device="cuda")
            gnn._lib.check(lib.gnnb_gat_aggregate_bwd_halo(rev.h, Wx.data_ptr(), er.data_ptr(), dout.data_ptr(),
                                                           d2.data_ptr() if split < n else None, split, el.data_ptr(),
                                                           smax.data_ptr(), ssum.data_ptr(), T.data_ptr(), Cc, H, SLOPE,
                                                           gW.data_ptr(), gr.data_ptr(), dz.data_ptr(), None))
            gl = torch.full_like(dl, float("nan"))
            gnn._lib.check(lib.gnnb_scatter(fwd.h, gnn._lib.DST, gnn._lib.SUM, dz.data_ptr(), H, gl.data_ptr(), None))
            torch.cuda.synchronize()
            for name, a, b in zip(("dWx", "der", "del"), (gW, gr, gl), (dWx, dr, dl)):
                assert same(a, b), f"{name} split={split} {tail} C={Cc} H={H}"


def test_empty_shard_and_missing_halo(gnn):
    """a shard without targets accepts NULL everywhere; a shard with halo sources refuses a NULL halo pointer"""
    lib = gnn._lib.lib
    h = C.c_void_p()
    gnn._lib.check(lib.gnnb_graph_create(C.byref(h), None, None, 0, 0, 0, 4, 0, 1, None))
    empty = gnn.graph._Plan(h.value, torch.device("cuda", 0))
    gnn._lib.check(lib.gnnb_gat_aggregate_halo(empty.h, None, None, 0, None, None, 64, 4, SLOPE, None, None, None, None))
    gnn._lib.check(lib.gnnb_gat_aggregate_bwd_halo(empty.h, None, None, None, None, 0, None, None, None, None, 64, 4, SLOPE,
                                                   None, None, None, None))
    gnn._lib.check(lib.gnnb_gat_tnode(None, None, 0, 64, 4, None, None))
    s, t = np.array([0, 2, 3], np.int32), np.array([1, 1, 0], np.int32)     # sources 2, 3 are halo nodes of a 2-row shard
    g = C.c_void_p()
    gnn._lib.check(lib.gnnb_graph_create(C.byref(g), s.ctypes.data, t.ctypes.data, 3, 4, 2, 4, 0, 0, None))
    shard = gnn.graph._Plan(g.value, torch.device("cuda", 0))
    Wx, el, er = torch.randn(2, 4, 64, device="cuda"), torch.randn(2, 4, device="cuda"), torch.randn(4, 4, device="cuda")
    out, sm, ss = torch.empty_like(Wx), torch.empty_like(el), torch.empty_like(el)
    with pytest.raises(ValueError):
        gnn._lib.check(lib.gnnb_gat_aggregate_halo(shard.h, Wx.data_ptr(), None, 2, el.data_ptr(), er.data_ptr(), 64, 4, SLOPE,
                                                   out.data_ptr(), sm.data_ptr(), ss.data_ptr(), None))
    halo = torch.randn(2, 4, 64, device="cuda")
    gnn._lib.check(lib.gnnb_gat_aggregate_halo(shard.h, Wx.data_ptr(), halo.data_ptr(), 2, el.data_ptr(), er.data_ptr(), 64, 4,
                                               SLOPE, out.data_ptr(), sm.data_ptr(), ss.data_ptr(), None))
    torch.cuda.synchronize()
    # row 1 gathers local source 0 and halo source 2; row 0 gathers halo source 3 alone: out = its Wx row
    assert same(out[0], halo[1])
