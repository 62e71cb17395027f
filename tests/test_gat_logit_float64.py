"""gnnb_gat_logit_terms and gnnb_gat_logit_terms_bwd (csrc/gatlogit.cu) element by element against float64 on the
device, on every shape GATConv sends them, and the gate (layers.gat_logit_fusable) GATConv chooses them by.

include/gnnb200.h promises both entries for C/4 a power of two <= 32 and C*H <= 4096.  G = C/4 lanes share a head, so a
warp covers hpp = 32/G heads per pass; the pullback runs the heads in slices of 8 passes.  H = 8 hpp is the last
one-slice shape, 8 hpp + 1 the first two-slice one, and 4096/C takes four.  Every G in 1..32 runs at
H in {1, hpp-1, hpp, hpp+1, 8 hpp, 8 hpp+1, 4096/C} and N in {1, 7, 8, 9, 4224, 4225}, plus one large N per G; 4224 =
8 x 528 is the last N at which each warp of the pullback's grid owns one node.  Each shape runs both halves together,
el only, er only, del only and der only.

Bars per element (u = 2^-24):
  el, er  |got - ref| <= 2 (4 + log2 G) u sum_c |a Wx|     a lane's four-term fma chain, then log2 G butterfly adds
  dWx     <= 4 u (|dWx0| + |del a| + |der a'|)               at most three roundings per element
  da      <= (ceil(N / (8 nblocks)) + 8 + nblocks) u sum_n |d Wx|,  nblocks = min(ceil(N / 8), 528)
                                                             a lane's chain over its warp's nodes, the 8-warp block
                                                             stage, the fixed-order sum over the blocks
and the half of da that a one-half call leaves out is exactly +0.  A zero scale is a bar of 0: a head whose half of `a`
is zero must give exactly 0.  The data are signed with magnitudes 2^-8..2^8 per row, a quarter of `a` is zero, and on
odd heads every third node's row cancels against itself exactly (a mirrored, Wx mirrored and negated).

Every operand sits inside a larger allocation, as in test_propagate_abi.py: NaN around an input, a sentinel bit pattern
around an output and inside it before the call.  After every call each output element was written, every guard holds
and every input is unchanged.  Besides the bars, the pullback's da and dWx are the same bits on a second call, and each
head's el, er, dWx and da are the bits of a one-head call on that head's columns copied out, at the same N: nblocks
depends on N alone, so the slicing of the heads must not change any head's order of operations.
"""
import math

import numpy as np
import pytest
import torch

from test_gat_attention_params import check_layer, create_plan
from test_gpu_parity import build_graph

U = 2.0 ** -24
PAD = 64                   # guard floats on either side of an operand
NAN_BITS = 0x7FC00000
SENTINEL = 0x7FA5A5A5      # a NaN payload no kernel produces: an output element still holding it was never written
OK, EUNSUPPORTED = 0, 5
NBLOCKS_MAX = 4 * 132      # the pullback's grid: 4 CTAs of 8 warps per SM of an H100 SXM
GS = (1, 2, 4, 8, 16, 32)
NS = (1, 7, 8, 9, 4224, 4225)
INVARIANCE_N = 4225        # every warp of the full grid owns a node, one owns two


def header_domain(Cc, H):
    """include/gnnb200.h: C/4 a power of two <= 32, C*H <= 4096"""
    g = Cc // 4
    return Cc % 4 == 0 and g > 0 and (g & (g - 1)) == 0 and g <= 32 and H >= 1 and Cc * H <= 4096


# every C in 1..160 and every H up to one past C*H = 4096
GRID = [(Cc, H) for Cc in range(1, 161) for H in range(1, (4096 + Cc) // Cc + 1)]


def heads_for(G):
    hpp, Cc = 32 // G, 4 * G
    return sorted({h for h in (1, hpp - 1, hpp, hpp + 1, 8 * hpp, 8 * hpp + 1, 4096 // Cc) if h >= 1})


SHAPES = [(4 * G, H) for G in GS for H in heads_for(G)]
# one large N per G: four slices at C*H = 4096, or C*H = 128 at 10^6 nodes
LARGE = [(4, 32, 1_000_000), (8, 512, 50_000), (16, 8, 1_000_000), (32, 128, 50_000), (64, 2, 1_000_000),
         (128, 32, 50_000)]


# ------------------------------------------------------------------------------------------------ gate
def test_gate_is_the_header_domain(gnn):
    """gat_logit_fusable states the domain both entries accept: neither wider (the pullback refused C*H > 1024) nor
    narrower (C = 4 with H > 16 and C = 8 with H > 32 went to torch)"""
    wrong = [(Cc, H) for Cc, H in GRID if gnn.layers.gat_logit_fusable(Cc, H) != header_domain(Cc, H)]
    assert not wrong, f"{len(wrong)} shapes disagree, e.g. {wrong[:10]}"


@pytest.mark.gpu
def test_entries_accept_exactly_the_gate(gnn):
    """over the same grid at N = 1: both logit entries return OK exactly when gat_logit_fusable holds, and
    gnnb_gat_aggregate / _bwd exactly when gat_fusable holds (one node with a self loop); every refusal is
    GNNB_EUNSUPPORTED before any launch"""
    lib = gnn._lib.lib
    F = 2 * (4096 + 160)
    Wx, a, el, er, dl, dr, dWx, da, out, smax, ssum, dout = (torch.zeros(F, device="cuda") for _ in range(12))
    plan = create_plan(gnn, np.zeros(1), np.zeros(1), 1, 1)
    p = lambda t: t.data_ptr()
    calls = {
        "logit_terms": (gnn.layers.gat_logit_fusable, lambda Cc, H: lib.gnnb_gat_logit_terms(
            p(Wx), p(a), 1, Cc, H, p(el), p(er), None)),
        "logit_terms_bwd": (gnn.layers.gat_logit_fusable, lambda Cc, H: lib.gnnb_gat_logit_terms_bwd(
            p(Wx), p(a), p(dl), p(dr), 1, Cc, H, p(dWx), p(da), None)),
        "aggregate": (gnn.layers.gat_fusable, lambda Cc, H: lib.gnnb_gat_aggregate(
            plan.h, p(Wx), p(el), p(er), Cc, H, 0.2, p(out), None, p(smax), p(ssum), None)),
        "aggregate_bwd": (gnn.layers.gat_fusable, lambda Cc, H: lib.gnnb_gat_aggregate_bwd(
            plan.h, p(Wx), p(el), p(er), p(smax), p(ssum), p(out), p(dout), Cc, H, 0.2, p(dWx), p(dl), p(dr), None)),
    }
    wrong = []
    for Cc, H in GRID:
        for name, (gate, call) in calls.items():
            before = gnn.launch_count()
            st = call(Cc, H)
            launched = gnn.launch_count() - before
            if gate(Cc, H):
                if st != OK:
                    wrong.append((name, Cc, H, f"status {st}: {gnn._lib.lib.gnnb_last_error().decode()}"))
            elif st != EUNSUPPORTED or launched:
                wrong.append((name, Cc, H, f"status {st}, {launched} launches"))
    torch.cuda.synchronize()
    assert not wrong, f"{len(wrong)} disagreements, e.g. {wrong[:10]}"


# ------------------------------------------------------------------------------------------------ guarded operands
class Buf:
    """n floats at byte offset `off` from a 256 B boundary between guards of PAD floats.  kind "in": NaN guards, the
    body holds `init`; "out": the sentinel everywhere; "inout": sentinel guards, the body holds `init`."""

    def __init__(self, n, kind, off=0, init=None):
        self.kind, self.n, self.lo = kind, n, PAD + off // 4
        self.raw = torch.full((2 * PAD + off // 4 + n,), NAN_BITS if kind == "in" else SENTINEL, dtype=torch.int32,
                              device="cuda")
        self.body = self.raw[self.lo:self.lo + n].view(torch.float32)
        if init is not None:
            self.body.copy_(init.reshape(-1))
        self.keep = self.raw.clone() if kind == "in" else None
        self.ptr = self.body.data_ptr()
        assert self.ptr % 16 == off

    def check(self, what):
        if self.kind == "in":
            assert torch.equal(self.raw, self.keep), f"{what}: an input or its guard was written"
            return
        guards = torch.cat([self.raw[:self.lo], self.raw[self.lo + self.n:]])
        assert (guards == SENTINEL).all(), f"{what}: a write outside the output"
        assert not (self.body.view(torch.int32) == SENTINEL).any(), f"{what}: an output element was never written"

    def untouched(self):
        return bool((self.raw == SENTINEL).all())


def ptr(b):
    return None if b is None else b.ptr


def within(what, got, ref, scale, k):
    """|got - ref| <= k u scale per element; NaN fails"""
    err = (got.double() - ref).abs()
    ok = err <= k * U * scale
    assert ok.all(), (f"{what}: {int((~ok).sum())} of {err.numel()} elements over {k:.4g} u scale, worst "
                      f"{float((err / (U * scale)).nan_to_num(float('inf')).max()):.4g} u scale")


def bits(x):
    return x.contiguous().view(torch.int32)


# ------------------------------------------------------------------------------------------------ data and reference
def make_inputs(N, Cc, H, seed):
    """Wx (N,H,C), a (H,2C) as the layer stores it in Julia memory order, del, der (N,H), dWx0 (N,H,C), float32"""
    g = torch.Generator(device="cuda").manual_seed(seed)
    scale = lambda *shape: torch.pow(2.0, torch.randint(-8, 9, shape, device="cuda", generator=g).float())
    Wx = torch.randn(N, H, Cc, device="cuda", generator=g) * scale(N, H, 1)
    a = torch.randn(H, 2 * Cc, device="cuda", generator=g)
    a[torch.rand(H, 2 * Cc, device="cuda", generator=g) < 0.25] = 0.0
    if H >= 2:
        a[0, Cc:] = 0.0                       # head 0: er exactly 0
        a[H - 1, :Cc] = 0.0                   # head H-1: el exactly 0
    half = Cc // 2                            # odd heads: a mirrored within each half, every third row cancels
    a[1::2, half:Cc] = a[1::2, :half]
    a[1::2, Cc + half:] = a[1::2, Cc:Cc + half]
    Wx[::3, 1::2, half:] = -Wx[::3, 1::2, :half]
    dl = torch.randn(N, H, device="cuda", generator=g) * scale(N, H)
    dr = torch.randn(N, H, device="cuda", generator=g) * scale(N, H)
    dl[torch.rand(N, H, device="cuda", generator=g) < 0.1] = 0.0
    dr[torch.rand(N, H, device="cuda", generator=g) < 0.1] = 0.0
    dW0 = torch.randn(N, H, Cc, device="cuda", generator=g)
    return Wx, a, dl, dr, dW0


def reference(Wx, a, dl, dr):
    """float64: el, er and the two halves of da with their bars' scales"""
    Cc = Wx.shape[2]
    W, A = Wx.double(), a.double()
    r = {}
    for half, Ah in (("el", A[:, :Cc]), ("er", A[:, Cc:])):
        prod = W * Ah
        r[half] = prod.sum(-1)
        r[half + "_s"] = prod.abs_().sum(-1)
        del prod
    for half, d in (("l", dl.double()), ("r", dr.double())):
        r["da_" + half] = torch.einsum("nh,nhc->hc", d, W)
        r["da_" + half + "_s"] = torch.einsum("nh,nhc->hc", d.abs(), W.abs())
    return r


def dwx_reference(dW0, a, dl, dr):
    """dWx0 + del a + der a' (a None half adds nothing) and its bar's scale, float64"""
    Cc = dW0.shape[2]
    ref, scale = dW0.double(), dW0.double().abs()
    for d, Ah in ((dl, a[:, :Cc]), (dr, a[:, Cc:])):
        if d is not None:
            t = d.double()[:, :, None] * Ah.double()
            ref, scale = ref + t, scale + t.abs()
    return ref, scale


FWD_MODES = {"both": (True, True), "el only": (True, False), "er only": (False, True)}
BWD_MODES = {"both": (True, True), "del only": (True, False), "der only": (False, True)}


def run_shape(gnn, Cc, H, N, seed, off=0):
    """every mode of both entries on guarded operands at one shape against float64; el, er, del, der and da at byte
    offset `off`.  Returns the inputs and each mode's outputs for the bitwise checks."""
    lib = gnn._lib.lib
    G = Cc // 4
    Wx, a, dl, dr, dW0 = make_inputs(N, Cc, H, seed)
    ref = reference(Wx, a, dl, dr)
    gW, ga = Buf(N * H * Cc, "in", init=Wx), Buf(2 * H * Cc, "in", init=a)
    gl, gr = Buf(N * H, "in", off, dl), Buf(N * H, "in", off, dr)
    what = f"C={Cc} H={H} N={N} off={off}"
    k_el = 2 * (4 + math.log2(G))
    got = {}
    for mode, (want_l, want_r) in FWD_MODES.items():
        el = Buf(N * H, "out", off) if want_l else None
        er = Buf(N * H, "out", off) if want_r else None
        st = lib.gnnb_gat_logit_terms(gW.ptr, ga.ptr, N, Cc, H, ptr(el), ptr(er), None)
        assert st == OK, f"forward {mode} {what}: status {st}"
        for name, b in (("el", el), ("er", er)):
            if b is not None:
                b.check(f"{name}, forward {mode} {what}")
                within(f"{name}, forward {mode} {what}", b.body.view(N, H), ref[name], ref[name + "_s"], k_el)
                got[f"fwd {mode} {name}"] = b.body.view(N, H).clone()
    nblocks = min(-(-N // 8), NBLOCKS_MAX)
    k_da = -(-N // (8 * nblocks)) + 8 + nblocks
    for mode, (use_l, use_r) in BWD_MODES.items():
        d_ref, d_scale = dwx_reference(dW0, a, dl if use_l else None, dr if use_r else None)
        runs = []
        for _ in range(2 if mode == "both" else 1):       # twice: the same bits
            dWx = Buf(N * H * Cc, "inout", init=dW0)
            da = Buf(2 * H * Cc, "out", off)
            st = lib.gnnb_gat_logit_terms_bwd(gW.ptr, ga.ptr, gl.ptr if use_l else None, gr.ptr if use_r else None, N,
                                              Cc, H, dWx.ptr, da.ptr, None)
            assert st == OK, f"pullback {mode} {what}: status {st}"
            dWx.check(f"dWx, pullback {mode} {what}")
            da.check(f"da, pullback {mode} {what}")
            runs.append((dWx.body.view(N, H, Cc).clone(), da.body.view(H, 2 * Cc).clone()))
            del dWx, da
        if len(runs) == 2:
            assert torch.equal(bits(runs[0][0]), bits(runs[1][0])), f"dWx bits differ between two calls {what}"
            assert torch.equal(bits(runs[0][1]), bits(runs[1][1])), f"da bits differ between two calls {what}"
        dWx, da = runs[0]
        within(f"dWx, pullback {mode} {what}", dWx, d_ref, d_scale, 4)
        del d_ref, d_scale
        for half, used, cols in (("l", use_l, slice(0, Cc)), ("r", use_r, slice(Cc, 2 * Cc))):
            if used:
                within(f"da_{half}, pullback {mode} {what} (nblocks {nblocks})", da[:, cols], ref["da_" + half],
                       ref["da_" + half + "_s"], k_da)
            else:
                assert (bits(da[:, cols]) == 0).all(), f"the unused half of da is not +0, pullback {mode} {what}"
        got[f"bwd {mode} dWx"], got[f"bwd {mode} da"] = dWx, da
    for b in (gW, ga, gl, gr):
        b.check(f"inputs {what}")
    return (Wx, a, dl, dr, dW0), got


def heads_first(key, v):
    """an output of run_shape with the head index first: el / er (H, N), dWx (H, N, C), da (H, 2C) as it is"""
    return v if key.endswith("da") else v.transpose(0, 1)


def check_per_head_bits(gnn, inputs, got):
    """each head alone, its columns copied out (H = 1, same N): el, er, dWx and da are the bits of the H-head calls"""
    lib = gnn._lib.lib
    Wx, a, dl, dr, dW0 = inputs
    N, H, Cc = Wx.shape
    Wh, dW0h = Wx.transpose(0, 1).contiguous(), dW0.transpose(0, 1).contiguous()       # (H, N, C)
    dlh, drh = dl.t().contiguous(), dr.t().contiguous()                                # (H, N)
    one = {k: torch.empty_like(heads_first(k, v), memory_format=torch.contiguous_format) for k, v in got.items()}
    for h in range(H):
        Wp, ap = Wh[h].data_ptr(), a[h].data_ptr()
        for mode, (want_l, want_r) in FWD_MODES.items():
            el = one[f"fwd {mode} el"][h].data_ptr() if want_l else None
            er = one[f"fwd {mode} er"][h].data_ptr() if want_r else None
            gnn._lib.check(lib.gnnb_gat_logit_terms(Wp, ap, N, Cc, 1, el, er, None))
        for mode, (use_l, use_r) in BWD_MODES.items():
            dWx = one[f"bwd {mode} dWx"][h]
            dWx.copy_(dW0h[h])
            gnn._lib.check(lib.gnnb_gat_logit_terms_bwd(Wp, ap, dlh[h].data_ptr() if use_l else None,
                                                        drh[h].data_ptr() if use_r else None, N, Cc, 1, dWx.data_ptr(),
                                                        one[f"bwd {mode} da"][h].data_ptr(), None))
    for k, v in got.items():
        same = bits(one[k]) == bits(heads_first(k, v))
        assert same.all(), f"{k}: {int((~same).sum())} elements differ from one-head calls (C={Cc} H={H} N={N})"


# ------------------------------------------------------------------------------------------------ against float64
@pytest.mark.gpu
@pytest.mark.parametrize("Cc,H", SHAPES, ids=[f"C{c}-H{h}" for c, h in SHAPES])
def test_entries_against_float64(gnn, Cc, H):
    for N in NS:
        inputs, got = run_shape(gnn, Cc, H, N, seed=Cc * 100003 + H * 101 + N)
        if N == INVARIANCE_N:
            check_per_head_bits(gnn, inputs, got)
        del inputs, got


@pytest.mark.gpu
@pytest.mark.parametrize("Cc,H,N", LARGE, ids=[f"C{c}-H{h}-N{n}" for c, h, n in LARGE])
def test_entries_against_float64_large(gnn, Cc, H, N):
    """each warp owns tens to hundreds of nodes"""
    inputs, got = run_shape(gnn, Cc, H, N, seed=Cc + H)
    check_per_head_bits(gnn, inputs, got)
    del inputs, got
    torch.cuda.empty_cache()


@pytest.mark.gpu
@pytest.mark.parametrize("off", [4, 8, 12])
@pytest.mark.parametrize("Cc,H", [(4, 33), (64, 17), (128, 9)])
def test_alignment(gnn, Cc, H, off):
    """Wx, a or dWx off a 16 B boundary: GNNB_EUNSUPPORTED before any launch, outputs and dWx untouched.  el, er, del,
    der and da there: accepted, with the float64 answer."""
    lib = gnn._lib.lib
    N = 4225
    Wx, a, dl, dr, dW0 = make_inputs(N, Cc, H, 3)
    for bad in ("Wx", "a", "dWx"):
        gW = Buf(N * H * Cc, "in", off if bad == "Wx" else 0, Wx)
        ga = Buf(2 * H * Cc, "in", off if bad == "a" else 0, a)
        gl, gr = Buf(N * H, "in", init=dl), Buf(N * H, "in", init=dr)
        before = gnn.launch_count()
        if bad != "dWx":
            el, er = Buf(N * H, "out"), Buf(N * H, "out")
            st = lib.gnnb_gat_logit_terms(gW.ptr, ga.ptr, N, Cc, H, el.ptr, er.ptr, None)
            assert st == EUNSUPPORTED, f"forward, {bad} at +{off} B: status {st}"
            assert el.untouched() and er.untouched()
        dWx, da = Buf(N * H * Cc, "inout", off if bad == "dWx" else 0, dW0), Buf(2 * H * Cc, "out")
        st = lib.gnnb_gat_logit_terms_bwd(gW.ptr, ga.ptr, gl.ptr, gr.ptr, N, Cc, H, dWx.ptr, da.ptr, None)
        assert st == EUNSUPPORTED, f"pullback, {bad} at +{off} B: status {st}"
        assert gnn.launch_count() == before, f"{bad} at +{off} B: a kernel ran before the refusal"
        assert da.untouched() and torch.equal(dWx.body.view(N, H, Cc), dW0)
        for b in (gW, ga, gl, gr):
            b.check(f"{bad} at +{off} B")
    run_shape(gnn, Cc, H, N, seed=Cc + H + off, off=off)


@pytest.mark.gpu
@pytest.mark.parametrize("Cc,H", [(64, 8), (128, 32), (4, 1024)])
def test_empty_input(gnn, Cc, H):
    """N = 0: the forward launches nothing and leaves el / er untouched; the pullback writes da as exact zeros"""
    lib = gnn._lib.lib
    gW, ga = Buf(0, "in"), Buf(2 * H * Cc, "in", init=torch.randn(H, 2 * Cc, device="cuda"))
    for mode, (want_l, want_r) in FWD_MODES.items():
        el, er = Buf(0, "out") if want_l else None, Buf(0, "out") if want_r else None
        before = gnn.launch_count()
        assert lib.gnnb_gat_logit_terms(gW.ptr, ga.ptr, 0, Cc, H, ptr(el), ptr(er), None) == OK
        assert gnn.launch_count() == before, f"forward {mode}: a launch at N = 0"
        assert all(b is None or b.untouched() for b in (el, er))
    for mode, (use_l, use_r) in BWD_MODES.items():
        gl, gr, dWx = Buf(0, "in"), Buf(0, "in"), Buf(0, "inout")
        da = Buf(2 * H * Cc, "out")
        st = lib.gnnb_gat_logit_terms_bwd(gW.ptr, ga.ptr, gl.ptr if use_l else None, gr.ptr if use_r else None, 0, Cc,
                                          H, dWx.ptr, da.ptr, None)
        assert st == OK, f"pullback {mode}: status {st}"
        da.check(f"da, pullback {mode} at N = 0")
        assert (bits(da.body) == 0).all(), f"pullback {mode} at N = 0: da is not +0"
        assert dWx.untouched()
    gW.check("Wx at N = 0")
    ga.check("a at N = 0")


# ------------------------------------------------------------------------------------------------ GATConv end to end
# refused by the pullback before it sliced the heads (C*H > 1024): six shapes; sent to torch by the old gate: three;
# config 3's 64 x 8, the control
LAYER_SHAPES = [(128, 16), (64, 17), (64, 32), (32, 33), (32, 128), (128, 32), (4, 17), (4, 1024), (8, 64), (64, 8)]


@pytest.fixture
def logit_bwd_calls(gnn, monkeypatch):
    """the calls of layers._gat_logit_terms_bwd, so that a layer test fails if the fused logit path did not run"""
    calls = []
    real = gnn.layers._gat_logit_terms_bwd

    def counted(*args):
        calls.append(tuple(args[0].shape))
        return real(*args)
    monkeypatch.setattr(gnn.layers, "_gat_logit_terms_bwd", counted)
    return calls


@pytest.fixture(scope="module")
def chunk_edges(gnn):
    """0-based edges with rows at the chunk edges, and a self loop on every node"""
    name, s, t, n, g = build_graph(gnn, "chunk_edges")
    loops = np.arange(n)
    return np.concatenate([s - 1, loops]), np.concatenate([t - 1, loops]), n


def off_the_kink(layer, xj, xi, s, t):
    """the edges whose logits sit, in every head, at least 2^-14 of their scale sum_c |a Wx| away from the leaky-ReLU
    kink.  At a logit within rounding of 0 the float32 layer may take the other branch than its float64 reference, which
    moves da by far more than its rounding error (with 10^6 logits one such edge is likely).  Logits on the kink are
    test_gat_attention_params.py's subject."""
    Cc, H = layer.channel[1], layer.heads
    W, a = layer.dense_x.weight.detach().double(), layer.a.detach().double()
    Wj = (xj.double() @ W.t()).reshape(-1, H, Cc)
    Wi = Wj if xi is None else (xi.double() @ W.t()).reshape(-1, H, Cc)
    pl, pr = Wi * a[:Cc].t(), Wj * a[Cc:].t()
    st, tt = torch.as_tensor(s, device=W.device), torch.as_tensor(t, device=W.device)
    z = pl.sum(-1)[tt] + pr.sum(-1)[st]
    scale = pl.abs().sum(-1)[tt] + pr.abs().sum(-1)[st]
    keep = (z.abs() >= 2.0 ** -14 * scale).all(1).cpu().numpy()
    assert keep.mean() > 0.85, f"{keep.mean():.3f} of the edges kept"
    return s[keep], t[keep]


@pytest.mark.gpu
@pytest.mark.parametrize("Cc,H", LAYER_SHAPES)
def test_gat_conv_one_node_type(gnn, chunk_edges, logit_bwd_calls, Cc, H):
    """GATConv on rows at the chunk edges with self loops, fused and generic, forward and every gradient against
    float64; the fused run goes through gnnb_gat_logit_terms_bwd once"""
    s, t, n = chunk_edges
    torch.manual_seed(Cc * 7 + H)
    layer = gnn.GATConv(8, Cc, heads=H, add_self_loops=False, device="cuda")     # the loops are in the edge list
    with torch.no_grad():
        layer.bias.normal_()
    x = torch.randn(n, 8, device="cuda")
    s, t = off_the_kink(layer, x, None, s, t)
    g = gnn.GNNGraph(torch.as_tensor(s + 1), torch.as_tensor(t + 1), num_nodes=n).cuda()
    check_layer(gnn, layer, g, torch.as_tensor(s, device="cuda"), torch.as_tensor(t, device="cuda"), n, x, None,
                f"C={Cc} H={H}")
    assert logit_bwd_calls == [(n, H, Cc)], logit_bwd_calls


@pytest.mark.gpu
@pytest.mark.parametrize("Cc,H", LAYER_SHAPES)
def test_gat_conv_two_node_types(gnn, logit_bwd_calls, Cc, H):
    """GATConv across two node types: the one-half entries, er over the sources and el over the targets, with a
    target row of more than two chunks, a source without out-edges and a target without in-edges"""
    rng = np.random.default_rng(31)
    ns, nd = 90, 50
    s = np.concatenate([rng.integers(0, ns - 1, 400), rng.integers(0, ns - 1, 300)])
    t = np.concatenate([rng.integers(1, nd - 1, 400), np.zeros(300, np.int64)])
    torch.manual_seed(Cc * 5 + H)
    layer = gnn.GATConv(12, Cc, heads=H).cuda()
    with torch.no_grad():
        layer.bias.uniform_(-1, 1)
    xj, xi = torch.randn(ns, 12, device="cuda"), torch.randn(nd, 12, device="cuda")
    s, t = off_the_kink(layer, xj, xi, s, t)
    g = gnn.GNNHeteroGraph({("A", "r", "B"): (torch.as_tensor(s + 1), torch.as_tensor(t + 1))},
                           num_nodes={"A": ns, "B": nd}, device="cuda")
    check_layer(gnn, layer, g, torch.as_tensor(s, device="cuda"), torch.as_tensor(t, device="cuda"), nd, xj, xi,
                f"bipartite C={Cc} H={H}")
    assert sorted(logit_bwd_calls) == sorted([(ns, H, Cc), (nd, H, Cc)]), logit_bwd_calls
