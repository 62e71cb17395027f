"""The dense layer part, σ.(W x .+ b) and its pullback, called through the C ABI on every route it dispatches to, against
float64 element by element.

Checked per element: |y - y64| <= γ (|x| |W|ᵀ + |b|) in float64 (with relu against relu(y64): relu is 1-Lipschitz), dx
against |dpre| |W|, dW against |dpre|ᵀ |x| (the reduction over the N rows), db against Σ|dpre|, with dpre formed from the
kernel's own y or relu mask.  γ depends on the route and on the length of its longest fp32 accumulation chain (`chain`).
A normwise bar only sees the large entries; this bound sees a wrong row of scale 2^-30 next to rows of scale 2^30.

The routes (`linear_route`, `bwd_plan`: a restatement of the dispatch in csrc/dense.cu and csrc/dense_tc.cu) are asserted
by the library's launch counter, or by switching the tensor-core kernels off and getting the same bits.  Every operand
sits in a `Guarded` buffer (NaN around inputs, a sentinel around and inside outputs), so a read outside an input, a write
outside an output and an output element never written all fail.  Small-integer operands make every route exact: there
the float64 result must come back bit for bit, independently of γ.

The CPU half checks the checker: the emulated 3xTF32 products (tf32_big / tf32_small of dense_tc.cu) with one cross term
dropped, 1xTF32, a 1e-3 error in rows below 2^-20, a K-block missing, or the last partial row tile shifted by a row must
each be rejected at every reduction length of the sweep, with the γ the GPU half uses.
"""
import json
import math
import os
import zlib

import numpy as np
import pytest
import torch

from test_propagate_abi import EUNSUPPORTED, OK, Guarded, pairwise

NORMWISE = 5e-6                # the normwise bar the dense entries have always met, kept on every case
U20 = 2.0 ** -20
NSM = 132                      # SMs of an H100 SXM: the split-K and column-sum partitions in `chain`
RING_NS = [1, 63, 64, 65, 127, 128, 129, 132 * 128 + 1, 1_000_037]
DATA = ["randn", "scaled", "colscaled", "pos", "poscols", "cancel", "int"]

# γ = G[route] · 2^-20 · (1 + chain / 16): the split's own error (2^-20 relative per product after the MMA reads the small
# part as tf32) plus one rounding of the partial sums per step of the accumulation chain.  G is the largest ratio
# γ / (2^-20 (1 + chain / 16)) measured on an H100 SXM over this file's cases, times a margin below 4 (the measured
# maxima are in the module's report, GNNB_DENSE_ABI_REPORT).
G = {
    "ring": 3.5, "mask": 4.0, "fused_dx": 3.5, "ring_dx": 4.0, "linear2": 2.5,
    "wide": 3.5, "wide_dx": 2.5,
    "dw": 4.0, "fused_dw": 4.5, "db": 0.3, "fused_db": 0.3,
    "lt": 2.5, "lt_dx": 2.0, "lt_dw": 1.0,
}


def chain(route, n, D=128, nsm=NSM):
    """the longest chain of fp32 accumulations behind one output element of `route` at reduction length n"""
    if route in ("ring", "mask", "fused_dx", "ring_dx", "wide", "wide_dx", "linear2"):
        return n / 8 + 3                                   # one wgmma k8 step at a time, + bias, + addend
    if route in ("dw", "fused_dw"):                        # 128-row chains, an fp32 sum per CTA, the CTA partials in order
        rpc = math.ceil(math.ceil(n / nsm) / 32) * 32
        return min(n, 128) / 8 + math.ceil(rpc / 128) + math.ceil(n / rpc)
    if route == "fused_db":                                # 8 rows per producer thread, 2 shuffles, tiles, 4 warps x CTAs
        ntiles = math.ceil(n / 128)
        grid = min(ntiles, nsm)
        return 10 + math.ceil(ntiles / grid) + 4 * grid
    if route == "db":                                      # act_bwd_kernel's rows per thread, block sum, final pass
        rpb = max(64, math.ceil(n / (nsm * 8)))
        rstep = 256 // (D // 4)
        return math.ceil(rpb / rstep) + rstep + math.ceil(n / rpb)
    # lt*: the library's own reduction order; a serial fp32 chain of n round-to-nearest adds drifts as sqrt(n)
    return math.sqrt(n)


def gamma(route, n, D=128):
    return G[route] * U20 * (1 + chain(route, n, D) / 16)


# ------------------------------------------------------------------------------------------------ the checker
REPORT = {}


def ratio(got, ref, scale):
    """max |got - ref| / scale over the elements (float64 tensors); an element whose scale is 0 must be exact"""
    if got.numel() == 0:
        return 0.0
    err = (got.double() - ref).abs()
    r = torch.where(scale > 0, err / scale.clamp_min(1e-300), torch.where(err > 0, math.inf, 0.0))
    return float(r.max())


def record(route, r, n, D=128):
    e = REPORT.setdefault(route, {"max_ratio": 0.0, "max_normalized": 0.0})
    norm = r / (U20 * (1 + chain(route, n, D) / 16))
    if norm >= e["max_normalized"]:
        e.update(max_normalized=norm, max_ratio=r, gamma=gamma(route, n, D), n=n)


def check(got, ref, scale, route, n, what, D=128, exact=False):
    """the componentwise bound, the normwise bar, and bit equality where the operands make the result exact"""
    got = got.double()
    r = ratio(got, ref, scale)
    record(route, r, n, D)
    g = gamma(route, n, D)
    assert r <= g, f"{what}: componentwise {r:.3e} > γ {g:.3e} ({route}, n = {n})"
    den = float(ref.norm())
    if den > 0:
        assert float((got - ref).norm()) / den < NORMWISE, f"{what}: normwise above {NORMWISE}"
    if exact:
        bad = torch.nonzero(got != ref)
        assert bad.numel() == 0, f"{what}: small integers not exact at {bad[:4].tolist()}"


# ------------------------------------------------------------------------------------------------ the 3xTF32 split
def tf32_big(a):
    return (a.contiguous().view(torch.int32) & np.int32(-8192)).view(torch.float32)     # low 13 mantissa bits cleared


def tf32_small(a):
    b = tf32_big(a)
    return torch.where(torch.isinf(a), torch.zeros_like(a), a - b)


def emulate(x, W, terms=("bb", "sb", "bs")):
    """x Wᵀ as the kernels form it: each operand split, the small part read as tf32 by the MMA, the products summed in
    float64 (no accumulation error of its own)"""
    xb, xs = tf32_big(x), tf32_big(tf32_small(x))
    wb, ws = tf32_big(W), tf32_big(tf32_small(W))
    pick = {"bb": (xb, wb), "sb": (xs, wb), "bs": (xb, ws)}
    return sum(a.double() @ b.double().t() for a, b in (pick[t] for t in terms))


def scaled_rows(rng, n, lo, hi, spread=False):
    e = np.linspace(lo, hi, n).round() if spread else rng.integers(lo, hi + 1, n)
    return np.exp2(e)[:, None]


def mutate(kind, x, W, xscale):
    """the product x Wᵀ with one mistake; x (M, L), W (P, L) float32"""
    if kind == "cross_term_dropped":
        return emulate(x, W, ("bb", "sb"))
    if kind == "1xTF32":
        return emulate(x, W, ("bb",))
    y = emulate(x, W)
    if kind == "tiny_rows_1e-3":
        return y * torch.where(torch.as_tensor(xscale[:, 0] < U20), 1 + 1e-3, 1.0)[:, None]     # rows of A below 2^-20
    if kind == "kblock_missing":
        L = x.shape[1]
        k0 = max(L // 32 - 1, 0) * 32                     # the last full K-block (the only, partial one below 32)
        return y - emulate(x[:, k0:k0 + 32], W[:, k0:k0 + 32])
    assert kind == "tail_tile_shifted"
    M = y.shape[0]
    t0 = ((M - 1) // 128) * 128
    z = y.clone()
    z[t0 + 1:] = y[t0:M - 1]
    if t0 > 0:
        z[t0] = y[t0 - 1]
    return z


MUTATIONS = ["cross_term_dropped", "1xTF32", "tiny_rows_1e-3", "kblock_missing", "tail_tile_shifted"]
# the reduction lengths of the routes swept below (for the library, 1xTF32 is a GEMM run in TF32 instead of fp32; for db
# the sum is the product with a row of ones)
SELF_TEST = [("ring", k) for k in (32, 64, 96, 128)] + [("mask", k) for k in (32, 64, 96, 128)] + \
            [("wide", k) for k in (160, 256, 512)] + [("ring_dx", k) for k in (32, 96, 128)] + \
            [("wide_dx", k) for k in (160, 512)] + [("fused_dx", 128), ("linear2", 256)] + \
            [("dw", n) for n in (1, 33, 132 * 32 + 1, 1_000_003)] + \
            [("fused_dw", n) for n in (1, 129, 132 * 32 + 1, 1_000_003)] + \
            [("lt", k) for k in (16, 64, 128, 1024, 1432, 2048, 2080)] + [("lt_dx", k) for k in (8, 64, 256, 2048)] + \
            [("lt_dw", n) for n in (33, 777, 5000, 400_000)] + \
            [("db", n) for n in (1, 129, 4225, 1_000_037)] + [("fused_db", n) for n in (1, 129, 4225, 1_000_037)]
# the sweep's own data classes (`operand`); cancel is randn with paired columns
SELF_TEST_DATA = ["randn", "scaled", "colscaled", "pos", "poscols", "int"]
# the rejection margin (ratio / γ, the best data class) each mutation keeps at its weakest length, printed per case
# (weakest: cross term 6.1 and 1xTF32 12.2 at the million-row dW on poscols, 1e-3 rows 11.1 in the library at K = 2080
# on scaled; a missing K-block and a shifted tail: the small integers at every length)
STATED_MARGIN = {"cross_term_dropped": 6.0, "1xTF32": 12.0, "tiny_rows_1e-3": 11.0, "kblock_missing": 1e300,
                 "tail_tile_shifted": 1e300}


def self_test_operands(route, cls, L, seed):
    """(A, B): the route's product A Bᵀ over a reduction of length L, from the sweep's generators.  Forward: A = x
    (130 rows: a full 128-row tile and a partial one), B = W; dx: A = dy, B = Wᵀ; dW: A = dyᵀ, B = xᵀ; db: A = dyᵀ,
    B = ones"""
    rng = np.random.default_rng(seed)
    big = L > 2048
    M, P = (8, 8) if big else (130, 16)
    if route in ("dw", "fused_dw", "lt_dw", "db", "fused_db"):
        A = operand(cls, rng, L, M, "dy", L).T
        B = operand(cls, rng, L, P, "x", L).T if route not in ("db", "fused_db") else np.ones((1, L), np.float32)
    elif route in ("ring_dx", "wide_dx", "fused_dx", "lt_dx"):
        A, B = operand(cls, rng, M, L, "dy", L), operand(cls, rng, L, P, "w", L).T
    else:
        A, B = operand(cls, rng, M, L, "x", L), operand(cls, rng, P, L, "w", L)
    return torch.as_tensor(np.ascontiguousarray(A)), torch.as_tensor(np.ascontiguousarray(B))


def self_test_margins(route, L):
    out = {}
    for cls in SELF_TEST_DATA:
        x, W = self_test_operands(route, cls, L, seed=L)
        xs = x.abs().amax(1, keepdim=True).numpy()             # rows of the result below 2^-20 come from these
        ref = x.double() @ W.double().t()
        scale = x.double().abs() @ W.double().abs().t()
        g = gamma(route, L)
        # the correct result: the 3xTF32 product for our kernels, the float32 rounding of float64 for the library and db
        ok = ref.float().double() if route.startswith("lt") or route.endswith("db") else emulate(x, W)
        base = ratio(ok, ref, scale)
        assert base <= g, f"{route} L={L} {cls}: the correct result itself is rejected ({base:.3e} > {g:.3e})"
        for m in MUTATIONS:
            got = mutate(m, x, W, xs)
            # small integers: the sweep asks for the float64 bits, so any difference is rejected
            out.setdefault(m, {})[cls] = (math.inf if not torch.equal(got, ref) else 0.0) if cls == "int" else \
                ratio(got, ref, scale) / g
    return out


@pytest.mark.parametrize("route,L", SELF_TEST, ids=[f"{r}-{n}" for r, n in SELF_TEST])
def test_checker_rejects_mutations(route, L):
    """each mutation is rejected by the bound, with the γ the sweep uses at this length, on one of the data classes the
    sweep runs there; the margins (ratio / γ per class, inf where small integers leave the exact bits) are printed and
    asserted against STATED_MARGIN.  A 32-row block missing from a million-row sum hides under γ with real-valued
    operands (3.2e-5 relative at most); the small-integer class, which every route must return exactly, rejects it."""
    margins = self_test_margins(route, L)
    for m, by_cls in margins.items():
        if route in ("db", "fused_db") and m == "cross_term_dropped":
            continue                                       # a plain fp32 sum: no split whose cross term could go missing
        best = max(by_cls, key=by_cls.get)
        print(f"{route} L={L} {m}: " + ", ".join(f"{c} {v:.3g}" for c, v in by_cls.items()) + f" (best: {best})")
        assert by_cls[best] > STATED_MARGIN[m], f"{route} L={L}: {m} accepted (margins {by_cls}), stated {STATED_MARGIN[m]}"


def test_checker_accepts_exact_and_rejects_wrong_zero():
    """an exact result passes with γ = 0 and an error where the bound is 0 (a zero row of x) fails at any γ"""
    x = torch.tensor([[1.0, 2.0], [0.0, 0.0]], dtype=torch.float64)
    W = torch.tensor([[3.0, -1.0]], dtype=torch.float64)
    ref, scale = x @ W.t(), x.abs() @ W.abs().t()
    assert ratio(ref.clone(), ref, scale) == 0.0
    bad = ref.clone()
    bad[1, 0] = 1e-300
    assert ratio(bad, ref, scale) == math.inf


def test_chain_model():
    """the chain lengths follow the partitions of csrc/dense_tc.cu and csrc/dense.cu at the H100's 132 SMs"""
    assert chain("ring", 128) == 19
    assert chain("dw", 1) == 1 / 8 + 1 + 1                       # one 32-row block in one CTA
    assert chain("dw", 132 * 32 + 1) == 16 + 1 + 67             # 64 rows per CTA: 67 CTAs (the last holds one row)
    assert chain("db", 1_000_037, 128) == math.ceil(948 / 8) + 8 + 1055     # 948 rows per block, 8 row sweeps


# ================================================================================================ GPU half
def dev(a):
    return torch.as_tensor(a).cuda().double()


def int_bound(L):
    """|entries| <= m with L m^2 < 2^24: every partial sum of a length-L reduction is an exact float32 integer"""
    m = 32
    while L * m * m + m >= 2 ** 24:
        m //= 2
    return m


def operand(kind, rng, rows, cols, role, L):
    """float32 host operand of the data class `kind`; role x / dy: rows (colscaled, poscols: columns) scaled over 2^±40,
    w: over 2^±20; pos, poscols all-positive"""
    if kind == "int":
        m = int_bound(L)
        return rng.integers(-m, m + 1, (rows, cols)).astype(np.float32)
    a = rng.uniform(0.5, 1.5, (rows, cols)) if kind in ("pos", "poscols") else rng.standard_normal((rows, cols))
    span = (-40, 40) if role in ("x", "dy") else (-20, 20)
    if kind == "scaled":
        a = a * scaled_rows(rng, rows, *span)
    if kind in ("colscaled", "poscols"):
        a = a * scaled_rows(rng, cols, *span).T
    return a.astype(np.float32)


def bias_for(kind, rng, n):
    if kind == "int":
        return rng.integers(-32, 33, n).astype(np.float32)
    b = rng.uniform(0.5, 1.5, n) if kind == "pos" else rng.standard_normal(n)
    return (b * (2.0 ** -70 if kind == "scaled" else 1.0)).astype(np.float32)


def cancel(a, b):
    """rows that cancel: every second row of a (M, L), from row 1, gets -(its first half) (1 + ε) as its second half,
    and b (P, L) its first half repeated, so those rows of a bᵀ are about 0 against Σ|a||b|"""
    h = a.shape[1] // 2
    if h == 0:
        return
    b[:, h:2 * h] = b[:, :h]
    a[1::2, h:2 * h] = -a[1::2, :h] * (1 + U20 * np.float32(0.5))


def lib_of(gnn):
    return gnn._lib.lib


@pytest.fixture(scope="module")
def report(gnn):
    if not torch.cuda.is_available():
        pytest.skip("no CUDA device")
    yield REPORT
    path = os.environ.get("GNNB_DENSE_ABI_REPORT")
    if path:
        with open(path, "w") as f:
            json.dump({"card": torch.cuda.get_device_name(), "G": G, "routes": REPORT}, f, indent=1, sort_keys=True)


@pytest.fixture
def switches(gnn, report):
    """set the tensor-core switch and the emulation preference for one test; both back on afterwards"""
    lib = lib_of(gnn)

    def set_(tc=1, emu=1):
        lib.gnnb_dense_set_tensor_core_kernel(tc)
        lib.gnnb_dense_set_emulation(emu)
    yield set_
    set_(1, 1)
    assert lib.gnnb_dense_tc_error() == 0


class Call:
    """one call over guarded operands: inputs (name -> host array or None), outputs (name -> element count)"""

    def __init__(self, gnn, ins, outs, offs=None, scratch=("ws",)):
        offs = offs or {}
        self.gnn, self.scratch = gnn, scratch
        self.ins = {k: Guarded(v, off=offs.get(k, 0)) for k, v in ins.items() if v is not None}
        self.outs = {k: Guarded(n=int(n), out=True, off=offs.get(k, 0)) for k, n in outs.items() if n is not None}

    def p(self, k):
        b = self.ins.get(k) or self.outs.get(k)
        return None if b is None else b.ptr

    def run(self, fn, *args, launches=None, rc=OK, written=True):
        lib = lib_of(self.gnn)
        n0 = self.gnn.launch_count()
        got = fn(*args)
        torch.cuda.synchronize()
        assert got == rc, f"rc {got}, expected {rc}: {lib.gnnb_last_error()}"
        if launches is not None and rc == OK:
            assert self.gnn.launch_count() - n0 == launches, "not the expected route"
        assert lib.gnnb_dense_tc_error() == 0
        for k, b in {**self.ins, **self.outs}.items():
            if b.out and (k in self.scratch or not (written and rc == OK)):
                r = b.raw.cpu()
                assert torch.equal(torch.cat([r[:b.lo], r[b.lo + b.n:]]), torch.cat([b.init[:b.lo], b.init[b.lo + b.n:]])), \
                    f"{k}: a write outside the output"
            else:
                b.check(k)
        return self

    def out(self, k, shape):
        return self.outs[k].body.view(shape)


# ------------------------------------------------------------------------------------------------ the dispatch
ALIGNED = frozenset()


def linear_route(N, K, Nout, tc=True, mis=ALIGNED, ldw=None):
    """gnnb_linear's route: ring / wide (the wgmma kernels of dense_tc.cu) or lt (cuBLASLt)"""
    ldw = K if ldw is None else ldw
    if not tc or mis & {"x", "W", "y"}:
        return "lt"
    if K > 128 or Nout > 128:
        ok = K % 32 == 0 and K <= 512 and Nout % 128 == 0 and Nout <= 1024 and ldw % 4 == 0 and N >= 2048
        return "wide" if ok else "lt"
    return "ring" if K % 32 == 0 and Nout % 16 == 0 else "lt"


LAUNCHES = {"ring": 1, "wide": 2, "lt": 1}


def bwd_plan(N, Din, Dout, relu, dx, dW, db, tc=True, mis=ALIGNED):
    """gnnb_linear_bwd: (launches, route of dx, route of dW, route of db), or None for GNNB_EUNSUPPORTED"""
    if tc and dx and dW and Dout == 128 and Din % 32 == 0 and Din <= 128 and \
            not mis & ({"dy", "x", "dx"} | ({"y"} if relu else set())):
        return 3, "fused_dx", "fused_dw", "fused_db"
    n = 0
    if relu or db:
        if Dout % 4 or Dout > 1024 or mis & ({"dy", "y", "ws"} if relu else {"dy"}):
            return None
        n += 1 + bool(db)
    dpre_al = not mis & ({"ws"} if relu else {"dy"})
    r_dx = r_dw = None
    if dx:
        if tc and Dout % 32 == 0 and Dout <= 128 and Din % 16 == 0 and 16 <= Din <= 128:
            r_dx = "ring_dx" if dpre_al and "dx" not in mis else "lt_dx"
            n += 1 + 1
        elif tc and (Dout > 128 or Din > 128) and Dout % 32 == 0 and Dout <= 512 and Din % 128 == 0 and Din <= 1024 \
                and N >= 2048:
            r_dx = "wide_dx" if dpre_al and "dx" not in mis else "lt_dx"
            n += 1 + (2 if r_dx == "wide_dx" else 1)
        else:
            r_dx, n = "lt_dx", n + 1
    if dW:
        ok = tc and Dout == 128 and Din % 32 == 0 and 32 <= Din <= 128 and dpre_al and not mis & {"x", "dW"}
        r_dw, n = ("dw", n + 2) if ok else ("lt_dw", n + 1)
    return n, r_dx, r_dw, "db"


# ------------------------------------------------------------------------------------------------ references
def fwd_ref(x, W, b, relu):
    x64, W64 = dev(x), dev(W)
    pre = x64 @ W64.t()
    scale = x64.abs() @ W64.abs().t()
    if b is not None:
        pre = pre + dev(b)
        scale = scale + dev(b).abs()
    return (pre.clamp(min=0) if relu else pre), scale


def check_linear(gnn, x, W, b, relu, N, K, Nout, data, what, tc=True, mis=ALIGNED, off=4, route=None):
    """one gnnb_linear over guarded operands (those named in `mis` at byte offset `off`), its route and its result"""
    lib = lib_of(gnn)
    r = route or linear_route(N, K, Nout, tc, mis)
    offs = {k: off for k in mis}
    c = Call(gnn, dict(x=x, W=W, b=b), dict(y=N * Nout), offs)
    c.run(lib.gnnb_linear, c.p("x"), c.p("W"), c.p("b"), relu, N, K, Nout, c.p("y"), None,
          launches=LAUNCHES[r] if N else 0)
    if N == 0:
        return c
    ref, scale = fwd_ref(x, W, b, relu)
    check(c.out("y", (N, Nout)), ref, scale, r, K, what, exact=data == "int")
    return c


def gen_linear(data, N, K, Nout, seed, bias=True):
    rng = np.random.default_rng(seed)
    x = operand(data, rng, N, K, "x", K)
    W = operand(data, rng, Nout, K, "w", K)
    if data == "cancel":
        cancel(x, W)
    b = bias_for(data, rng, Nout) if bias else None
    return x, W, b


ACT = ["relu+b", "relu", "b", "id"]


def act_of(a):
    return int(a.startswith("relu")), a.endswith("b")


def ids(rows):
    return ["-".join(str(v) for v in r.values()) for r in rows]


# ------------------------------------------------------------------------------------------------ forward routes
def library_bits(gnn, x, W, b, relu, N, K, Nout, data, what, mis=ALIGNED, off=4):
    """the bits of the same gnnb_linear with the tensor-core kernels off (the library GEMM), itself within its bound"""
    lib_of(gnn).gnnb_dense_set_tensor_core_kernel(0)
    try:
        return check_linear(gnn, x, W, b, relu, N, K, Nout, data, what + " library", tc=False, mis=mis,
                            off=off).outs["y"].bits
    finally:
        lib_of(gnn).gnnb_dense_set_tensor_core_kernel(1)


# every K x Nout also as a real-valued case whose bits must differ from the library's
RING = pairwise(dict(K=[32, 64, 96, 128], Nout=[16, 32, 48, 80, 96, 112, 128], N=RING_NS, data=DATA, act=ACT), 11,
                [dict(K=k, Nout=n, N=129, data="int", act="relu+b") for k in (32, 64, 96, 128)
                 for n in (16, 32, 48, 80, 96, 112, 128)] +
                [dict(K=k, Nout=n, N=129, data="randn", act="b") for k in (32, 64, 96, 128)
                 for n in (16, 32, 48, 80, 96, 112, 128)] +
                [dict(K=128, Nout=128, N=1_000_037, data="pos", act="b")])


@pytest.mark.gpu
@pytest.mark.parametrize("c", RING, ids=ids(RING))
def test_linear_ring(gnn, switches, c):
    """the forward ring kernel at every K x Nout it serves, across the row counts that end inside a tile"""
    relu, bias = act_of(c["act"])
    x, W, b = gen_linear(c["data"], c["N"], c["K"], c["Nout"], seed=zlib.crc32(str(c).encode()), bias=bias)
    assert linear_route(c["N"], c["K"], c["Nout"]) == "ring"
    y = check_linear(gnn, x, W, b, relu, c["N"], c["K"], c["Nout"], c["data"], str(c)).outs["y"].bits
    if c["data"] != "int" and c["N"] * c["Nout"] >= 1024:  # one launch either way: the library must give other bits
        assert not torch.equal(y, library_bits(gnn, x, W, b, relu, c["N"], c["K"], c["Nout"], c["data"], str(c)))


WIDE = pairwise(dict(K=[160, 256, 512], Nout=[128, 384, 1024], N=[2048, 2049, 40_000], data=DATA, act=ACT), 12,
                [dict(K=512, Nout=1024, N=2049, data="pos", act="b"), dict(K=512, Nout=384, N=40_000, data="int",
                                                                             act="relu+b")])


@pytest.mark.gpu
@pytest.mark.parametrize("c", WIDE, ids=ids(WIDE))
def test_linear_wide(gnn, switches, c):
    """the wide kernel, K up to 512 and Nout up to 1024, from the smallest row count it takes"""
    relu, bias = act_of(c["act"])
    x, W, b = gen_linear(c["data"], c["N"], c["K"], c["Nout"], seed=zlib.crc32(str(c).encode()), bias=bias)
    assert linear_route(c["N"], c["K"], c["Nout"]) == "wide"
    check_linear(gnn, x, W, b, relu, c["N"], c["K"], c["Nout"], c["data"], str(c))


# (N, K, Nout, tensor-core kernels on): shapes the wgmma kernels do not take, and every shape with them off
LT_SHAPES = {"K16": (1000, 16, 64, 1), "Nout8": (777, 64, 8, 1), "Nout136": (3000, 64, 136, 1),
             "wide_N2047": (2047, 512, 384, 1), "K1024": (4096, 1024, 384, 1), "K2048": (2049, 2048, 1024, 1),
             "K2080": (4096, 2080, 128, 1), "Nout1152": (4096, 128, 1152, 1),
             "tc_off": (5000, 128, 128, 0)}
EMULATION = {}


@pytest.mark.gpu
@pytest.mark.parametrize("data", DATA)
@pytest.mark.parametrize("emu", [1, 0])
@pytest.mark.parametrize("shape", list(LT_SHAPES))
def test_linear_cublaslt(gnn, switches, shape, emu, data):
    """the library GEMM, with the fp32-emulated compute type allowed and not; with the tensor-core kernels on, the same
    bits as with them off (so the library took the shape)"""
    N, K, Nout, tc = LT_SHAPES[shape]
    x, W, b = gen_linear(data, N, K, Nout, seed=N + K + Nout)
    assert linear_route(N, K, Nout, tc) == "lt"
    switches(tc, emu)
    c = check_linear(gnn, x, W, b, 1, N, K, Nout, data, f"{shape} emu={emu}")
    EMULATION[emu] = int(lib_of(gnn).gnnb_dense_emulation_active())
    if emu == 0:
        assert EMULATION[0] == 0, "emulation reported active while switched off"
    REPORT["emulation_active"] = {str(k): v for k, v in EMULATION.items()}
    if tc:
        switches(0, emu)
        d = check_linear(gnn, x, W, b, 1, N, K, Nout, data, f"{shape} emu={emu} tc off")
        assert torch.equal(c.outs["y"].bits, d.outs["y"].bits), "the wgmma kernels took a shape meant for the library"


MASKC = pairwise(dict(Din=[32, 64, 96, 128], N=RING_NS, data=DATA, bias=[True, False]), 13)


def mask_bits(y):
    """the relu mask words of (N, 128) y: bit 2 (n >> 3) + (n & 1) of word (n >> 1) & 3 is y[:, n] > 0"""
    n = torch.arange(128, device=y.device)
    bit = (y > 0).long() << (2 * (n >> 3) + (n & 1))
    w = torch.zeros(y.shape[0], 4, dtype=torch.long, device=y.device)
    w.index_add_(1, (n >> 1) & 3, bit)
    return w


@pytest.mark.gpu
@pytest.mark.parametrize("c", MASKC, ids=ids(MASKC))
def test_linear_relu_mask(gnn, switches, c):
    """gnnb_linear_relu_mask: y within the bound, the mask bit for bit `y > 0` of y as stored"""
    lib = lib_of(gnn)
    N, K = c["N"], c["Din"]
    x, W, b = gen_linear(c["data"], N, K, 128, seed=N + K, bias=c["bias"])
    call = Call(gnn, dict(x=x, W=W, b=b), dict(y=N * 128, mask=N * 4))
    call.run(lib.gnnb_linear_relu_mask, call.p("x"), call.p("W"), call.p("b"), N, K, 128, call.p("y"), call.p("mask"),
             None, launches=1)
    y = call.out("y", (N, 128))
    ref, scale = fwd_ref(x, W, b, 1)
    check(y, ref, scale, "mask", K, str(c), exact=c["data"] == "int")
    got = call.outs["mask"].bits.view(N, 4).long() & 0xFFFFFFFF
    assert torch.equal(got, mask_bits(y))


# ------------------------------------------------------------------------------------------------ pullbacks
def forward_y(gnn, x, W, b, relu, mask=False):
    """the forward output (and mask) the pullback reads, by the library itself on unguarded tensors"""
    lib = lib_of(gnn)
    N, K, Nout = x.shape[0], x.shape[1], W.shape[0]
    xt, Wt = torch.as_tensor(x).cuda(), torch.as_tensor(W).cuda()
    bt = None if b is None else torch.as_tensor(b).cuda()
    y = torch.empty(N, Nout, device="cuda")
    m = torch.empty(N, 4, dtype=torch.int32, device="cuda") if mask else None
    bp = None if bt is None else bt.data_ptr()
    if mask:
        gnn._lib.check(lib.gnnb_linear_relu_mask(xt.data_ptr(), Wt.data_ptr(), bp, N, K, Nout, y.data_ptr(), m.data_ptr(),
                                                 None))
    else:
        gnn._lib.check(lib.gnnb_linear(xt.data_ptr(), Wt.data_ptr(), bp, relu, N, K, Nout, y.data_ptr(), None))
    return y.cpu().numpy(), None if m is None else m.cpu().numpy()


def check_bwd(gnn, N, Din, Dout, relu, dx, dW, db, data, what, seed, tc=True, mis=ALIGNED, off=4, mask=False,
              x=None, W=None, dy=None, fwd=None, lib_only=False, distinct=False):
    """one gnnb_linear_bwd (gnnb_linear_bwd_mask when `mask`) over guarded operands: its route by launch count, dx, dW
    and db against float64 with dpre from the kernels' own forward output.  lib_only: the tensor-core kernels off for
    this call alone.  distinct: the same call with them off must give other bits in every product the plan gives to a
    wgmma kernel (the launch count alone cannot tell ring dx from the library's dx: the transpose runs either way)"""
    lib = lib_of(gnn)
    rng = np.random.default_rng(seed)
    if x is None:
        x = operand(data, rng, N, Din, "x", max(Dout, N))
        W = operand(data, rng, Dout, Din, "w", max(Dout, N))
        dy = operand(data, rng, N, Dout, "dy", max(Dout, N))
        if data == "int":                                  # dW reduces over N rows: keep N m^2 below 2^24
            m = int_bound(max(N, Dout))
            x, dy = np.clip(x, -m, m), np.clip(dy, -m, m)
        if data == "cancel":
            Wt = np.ascontiguousarray(W.T)
            cancel(dy, Wt)
            W = np.ascontiguousarray(Wt.T)
    if fwd is None:
        fwd = forward_y(gnn, x, W, bias_for(data, rng, Dout), relu, mask) if (relu or mask) and N else (None, None)
    y, m = fwd
    tc = tc and not lib_only
    plan = (3, "fused_dx", "fused_dw", "fused_db") if mask else bwd_plan(N, Din, Dout, relu, dx, dW, db, tc, mis)
    offs = {k: off for k in mis}
    c = Call(gnn, dict(dy=dy, y=None if mask else y, mask=None if m is None else m.view(np.float32), x=x, W=W),
             dict(ws=N * Dout if relu and not mask else None, dx=N * Din if dx else None, dW=Din * Dout if dW else None,
                  db=Dout if db else None), offs)
    if lib_only:
        lib.gnnb_dense_set_tensor_core_kernel(0)
    if mask:
        c.run(lib.gnnb_linear_bwd_mask, c.p("dy"), c.p("mask"), c.p("x"), c.p("W"), N, Din, Dout, c.p("dx"), c.p("dW"),
              c.p("db"), None, launches=3)
    else:
        c.run(lib.gnnb_linear_bwd, c.p("dy"), c.p("y"), c.p("x"), c.p("W"), relu, N, Din, Dout, c.p("ws"), c.p("dx"),
              c.p("dW"), c.p("db"), None, launches=(plan[0] if N else 0) if plan else None,
              rc=OK if plan or N == 0 else EUNSUPPORTED)
    if lib_only:
        lib.gnnb_dense_set_tensor_core_kernel(1)
    if N == 0:
        for k in ("dW", "db"):
            if k in c.outs:
                assert (c.outs[k].body == 0).all(), f"{what}: {k} of an empty batch is not zero"
        return c
    if plan is None:                                       # refused before any launch: no output was touched
        for k, b in c.outs.items():
            assert b.untouched(), f"{what}: {k} written by a refused call"
        return None
    exact = data == "int"
    dpre = dev(dy) * (dev(y) > 0) if (relu or mask) else dev(dy)
    if dx:
        W64 = dev(W)
        check(c.out("dx", (N, Din)), dpre @ W64, dpre.abs() @ W64.abs(), plan[1], Dout, "dx " + what, exact=exact)
    if dW:
        x64 = dev(x)
        check(c.out("dW", (Dout, Din)), dpre.t() @ x64, dpre.abs().t() @ x64.abs(), plan[2], N, "dW " + what,
              exact=exact)
    if db:
        check(c.out("db", (Dout,)), dpre.sum(0), dpre.abs().sum(0), plan[3], N, "db " + what, D=Dout, exact=exact)
    if distinct and not exact:
        d = check_bwd(gnn, N, Din, Dout, relu, dx, dW, db, data, what + " library", seed, mis=mis, off=off, x=x, W=W,
                      dy=dy, fwd=fwd, lib_only=True)
        for k, r in (("dx", plan[1]), ("dW", plan[2])):
            if k in c.outs and not r.startswith("lt"):
                assert not torch.equal(c.outs[k].bits, d.outs[k].bits), f"{what}: {k} has the library's bits ({r})"
    return c


FUSED = pairwise(dict(Din=[32, 64, 96, 128], src=["y", "mask", "none"], db=[True, False],
                      N=[1, 33, 127, 128, 129, 132 * 32 + 1, 132 * 128 + 1, 400_000], data=DATA), 14,
                 [dict(Din=128, src=s, db=True, N=1_000_037, data=d) for s in ("y", "mask") for d in ("pos", "poscols")])


@pytest.mark.gpu
@pytest.mark.parametrize("c", FUSED, ids=ids(FUSED))
def test_fused_pullback(gnn, switches, c):
    """the fused pullback (dx, dW and db in three launches), relu read from y, from the mask bits, or none"""
    check_bwd(gnn, c["N"], c["Din"], 128, int(c["src"] != "none"), True, True, c["db"], c["data"], str(c),
              seed=c["N"] + c["Din"], mask=c["src"] == "mask")


# (N, Din, Dout, dx, dW): one product per case, so the fused pullback is not taken
RING_DX = [(din, dout) for din in (16, 48, 112) for dout in (32, 96, 128)]
SPLIT = [(n, din, dout, 1, 0) for i, (din, dout) in enumerate(RING_DX) for n in (RING_NS[i], RING_NS[(i + 4) % 9])] + \
        [(n, din, dout, 1, 0) for din in (128, 1024) for dout in (160, 512) for n in (2048, 5001)] + \
        [(3000, 8, 64, 1, 0), (3000, 200, 96, 1, 0), (1000, 128, 64, 1, 0)] + \
        [(n, din, 128, 0, 1) for n in (1, 33, 132 * 32 + 1, 1_000_003) for din in (32, 96)] + \
        [(5000, 64, 64, 0, 1), (5000, 48, 128, 0, 1), (700, 128, 256, 0, 1)]
# (the relu and db pass takes Dout <= 1024: wider layers come without either)
SPLITC = [dict(N=s[0], Din=s[1], Dout=s[2], dx=s[3], dW=s[4], relu=i % 2 * (s[2] <= 1024),
               db=(i // 2) % 2 * (s[2] <= 1024), data=DATA[i % len(DATA)]) for i, s in enumerate(SPLIT)] + \
         [dict(N=1_000_003, Din=128, Dout=128, dx=0, dW=1, relu=1, db=1, data=d)
          for d in ("pos", "int", "scaled", "poscols")] + \
         [dict(N=400_000, Din=64, Dout=64, dx=0, dW=1, relu=0, db=1, data="poscols")] + \
         [dict(N=132 * 128 + 1, Din=112, Dout=128, dx=1, dW=0, relu=1, db=0, data="pos"),
          dict(N=5001, Din=1024, Dout=2048, dx=1, dW=0, relu=0, db=0, data="pos")]


@pytest.mark.gpu
@pytest.mark.parametrize("c", SPLITC, ids=ids(SPLITC))
def test_split_pullback(gnn, switches, c):
    """the non-fused pullback: ring dx (Din a multiple of 16), wide dx, library dx, dw_tf32x3 at row counts that end
    inside a 32-row block and a CTA's range, library dW"""
    plan = bwd_plan(c["N"], c["Din"], c["Dout"], c["relu"], c["dx"], c["dW"], c["db"])
    assert plan and plan[0] > 0
    check_bwd(gnn, c["N"], c["Din"], c["Dout"], c["relu"], c["dx"], c["dW"], c["db"], c["data"], str(c),
              seed=c["N"] * 3 + c["Din"], distinct=c["N"] * c["Din"] >= 1024)


def test_split_plan_routes():
    """every route of the non-fused pullback appears among the cases"""
    got = {r for c in SPLITC for r in bwd_plan(c["N"], c["Din"], c["Dout"], c["relu"], c["dx"], c["dW"], c["db"])[1:3]}
    assert {"ring_dx", "wide_dx", "lt_dx", "dw", "lt_dw"} <= got


# ------------------------------------------------------------------------------------------------ linear2
L2 = [dict(D1=d1, D2=d2, Dout=do, N=n, act=a, data=DATA[i % len(DATA)])
      for i, ((d1, d2), do, n, a) in enumerate(
          [(p, do, n, ACT[(j + k) % 4]) for j, p in enumerate([(32, 128), (128, 32), (96, 96)])
           for k, (do, n) in enumerate([(16, 129), (64, 132 * 128 + 1), (128, 1000)])] +
          [((128, 256), 128, 2048, "relu+b"), ((128, 256), 128, 40_000, "b")])]


def linear2_launches(N, D1, D2, Dout):
    return sum(LAUNCHES[linear_route(N, k, Dout, ldw=D1 + D2)] for k in (D1, D2))


@pytest.mark.gpu
@pytest.mark.parametrize("c", L2, ids=ids(L2))
def test_linear2(gnn, switches, c):
    """gnnb_linear2: two passes over the column blocks of W, the second through the wide kernel (ldw != K, the addend)
    when it is wider than 128"""
    lib = lib_of(gnn)
    N, D1, D2, Dout = c["N"], c["D1"], c["D2"], c["Dout"]
    relu, bias = act_of(c["act"])
    rng = np.random.default_rng(N + D1 + 7 * D2)
    x1 = operand(c["data"], rng, N, D1, "x", D1 + D2)
    x2 = operand(c["data"], rng, N, D2, "x", D1 + D2)
    W = operand(c["data"], rng, Dout, D1 + D2, "w", D1 + D2)
    b = bias_for(c["data"], rng, Dout) if bias else None
    call = Call(gnn, dict(x1=x1, x2=x2, W=W, b=b), dict(y=N * Dout))
    call.run(lib.gnnb_linear2, call.p("x1"), call.p("x2"), call.p("W"), call.p("b"), relu, N, D1, D2, Dout, call.p("y"),
             None, launches=linear2_launches(N, D1, D2, Dout))
    ref, scale = fwd_ref(np.concatenate([x1, x2], 1), W, b, relu)
    route = "wide" if "wide" in {linear_route(N, k, Dout, ldw=D1 + D2) for k in (D1, D2)} else "linear2"
    check(call.out("y", (N, Dout)), ref, scale, route, D1 + D2, str(c), exact=c["data"] == "int")


def check_linear2_bwd(gnn, N, D1, D2, relu, data, what, seed, want=("dx1", "dx2", "dW", "db"), mis=ALIGNED, off=4,
                      rc=OK):
    lib = lib_of(gnn)
    Dout = 128
    rng = np.random.default_rng(seed)
    x1 = operand(data, rng, N, D1, "x", max(N, Dout))
    x2 = operand(data, rng, N, D2, "x", max(N, Dout))
    W = operand(data, rng, Dout, D1 + D2, "w", Dout)
    dy = operand(data, rng, N, Dout, "dy", max(N, Dout))
    if data == "int":
        m = int_bound(max(N, Dout))
        x1, x2, dy = np.clip(x1, -m, m), np.clip(x2, -m, m), np.clip(dy, -m, m)
    x = np.concatenate([x1, x2], 1)
    y = forward_y(gnn, x, W, bias_for(data, rng, Dout), relu)[0] if relu and N else None
    outs = dict(ws=N * Dout if relu else None, dx1=N * D1, dx2=N * D2, dW=Dout * (D1 + D2), db=Dout)
    c = Call(gnn, dict(dy=dy, y=y, x1=x1, x2=x2, W=W), {k: v for k, v in outs.items() if k == "ws" or k in want},
             {k: off for k in mis})
    launches = None
    if rc == OK and N:
        launches = (1 + ("db" in want) if relu or "db" in want else 0) + \
                   sum(2 * (f"dx{i}" in want) + 3 * ("dW" in want) for i in (1, 2))
    c.run(lib.gnnb_linear2_bwd, c.p("dy"), c.p("y"), c.p("x1"), c.p("x2"), c.p("W"), relu, N, D1, D2, Dout, c.p("ws"),
          c.p("dx1"), c.p("dx2"), c.p("dW"), c.p("db"), None, launches=launches, rc=rc)
    if rc != OK:
        return c
    if N == 0:
        for k in ("dW", "db"):
            if k in c.outs:
                assert (c.outs[k].body == 0).all()
        return c
    dpre = dev(dy) * (dev(y) > 0) if relu else dev(dy)
    W64, x64 = dev(W), dev(x)
    exact = data == "int"
    for i, (lo, hi) in ((1, (0, D1)), (2, (D1, D1 + D2))):
        if f"dx{i}" in c.outs:
            check(c.out(f"dx{i}", (N, hi - lo)), dpre @ W64[:, lo:hi], dpre.abs() @ W64[:, lo:hi].abs(), "ring_dx",
                  Dout, f"dx{i} {what}", exact=exact)
    if "dW" in c.outs:
        check(c.out("dW", (Dout, D1 + D2)), dpre.t() @ x64, dpre.abs().t() @ x64.abs(), "dw", N, "dW " + what,
              exact=exact)
    if "db" in c.outs:
        check(c.out("db", (Dout,)), dpre.sum(0), dpre.abs().sum(0), "db", N, "db " + what, exact=exact)
    return c


L2B = [dict(D1=d1, D2=d2, N=n, relu=r, data=DATA[i % len(DATA)])
       for i, ((d1, d2), n, r) in enumerate([(p, n, (j + k) % 2) for j, p in enumerate([(32, 128), (128, 32), (96, 96)])
                                             for k, n in enumerate([1, 129, 132 * 32 + 1, 70_001])])]


@pytest.mark.gpu
@pytest.mark.parametrize("c", L2B, ids=ids(L2B))
def test_linear2_bwd(gnn, switches, c):
    """gnnb_linear2_bwd: dx1, dx2, dW and db against float64"""
    check_linear2_bwd(gnn, c["N"], c["D1"], c["D2"], c["relu"], c["data"], str(c), seed=c["N"] + c["D1"])


@pytest.mark.gpu
def test_linear2_bwd_wide_block_unsupported(gnn, switches):
    """a column block wider than 128 has no pullback here: GNNB_EUNSUPPORTED, and nothing is written"""
    c = check_linear2_bwd(gnn, 4096, 128, 256, 1, "randn", "(128, 256)", seed=3, rc=EUNSUPPORTED)
    for k, b in c.outs.items():
        assert b.untouched(), f"{k} written by a refused call"


@pytest.mark.gpu
@pytest.mark.parametrize("N,K,Nout,data", [(40_000, 1024, 384, "pos"), (2048, 1024, 128, "pos"),
                                           (2048, 2048, 128, "randn"), (2049, 2048, 1024, "pos")])
def test_long_k_takes_the_library(gnn, switches, N, K, Nout, data):
    """K above 512 goes to the library GEMM.  The wide wgmma kernel took K up to 2048, and at these shapes its results
    left the normwise 5e-6 of float64 on an H100 (the big*big chain of K/8 accumulations drifts); the library meets
    both bounds here, and the wide kernel still serves K = 512 with the same data"""
    x, W, b = gen_linear(data, N, K, Nout, seed=K + Nout)
    assert linear_route(N, K, Nout) == "lt"
    check_linear(gnn, x, W, b, 0, N, K, Nout, data, f"K={K}")           # one launch: not the wide kernel's two
    x, W, b = gen_linear(data, N, 512, Nout, seed=K + Nout)
    assert linear_route(N, 512, Nout) == "wide"
    check_linear(gnn, x, W, b, 0, N, 512, Nout, data, "K=512")


# ------------------------------------------------------------------------------------------------ bias_act
BA = [(70001, 512), (1, 4), (4099, 36), (129, 1024), (1000, 12)]


@pytest.mark.gpu
@pytest.mark.parametrize("relu", [0, 1])
@pytest.mark.parametrize("N,D", BA)
def test_bias_act_exact(gnn, switches, N, D, relu):
    """gnnb_bias_act and gnnb_bias_act_bwd: one rounding per element, so float32 numpy gives the same bits; db within
    its chain's bound"""
    lib = lib_of(gnn)
    rng = np.random.default_rng(N + D)
    x = rng.standard_normal((N, D)).astype(np.float32)
    x[rng.random((N, D)) < 0.05] = 0.0
    b = rng.standard_normal(D).astype(np.float32)
    c = Call(gnn, dict(x=x, b=b), dict(y=N * D))
    c.run(lib.gnnb_bias_act, c.p("x"), c.p("b"), relu, N, D, c.p("y"), None, launches=1)
    want = x + b
    want = np.maximum(want, np.float32(0)) if relu else want
    assert np.array_equal(c.outs["y"].get((N, D)).view(np.int32), want.view(np.int32))
    dy = rng.standard_normal((N, D)).astype(np.float32)
    y = c.outs["y"].get((N, D))
    d = Call(gnn, dict(dy=dy, y=y), dict(dpre=N * D if relu else None, db=D))
    d.run(lib.gnnb_bias_act_bwd, d.p("dy"), d.p("y"), relu, N, D, d.p("dpre"), d.p("db"), None, launches=2)
    dpre = np.where(y > 0, dy, np.float32(0)) if relu else dy
    if relu:
        assert np.array_equal(d.outs["dpre"].get((N, D)).view(np.int32), dpre.view(np.int32))
    check(d.out("db", (D,)), dev(dpre).sum(0), dev(dpre).abs().sum(0), "db", N, "db", D=D)


# ------------------------------------------------------------------------------------------------ empty batches
@pytest.mark.gpu
def test_empty_batch(gnn, switches):
    """N = 0: y (and the mask) untouched, dW and db zero, for every entry"""
    lib = lib_of(gnn)
    x, W, b = gen_linear("randn", 0, 64, 128, seed=0)
    c = Call(gnn, dict(x=x, W=W, b=b), dict(y=1, mask=1))
    c.run(lib.gnnb_linear, c.p("x"), c.p("W"), c.p("b"), 1, 0, 64, 128, c.p("y"), None, launches=0, written=False)
    c.run(lib.gnnb_linear_relu_mask, c.p("x"), c.p("W"), c.p("b"), 0, 64, 128, c.p("y"), c.p("mask"), None, launches=0,
          written=False)
    c.run(lib.gnnb_linear2, c.p("x"), c.p("x"), c.p("W"), c.p("b"), 1, 0, 32, 32, 128, c.p("y"), None, launches=0,
          written=False)
    c.run(lib.gnnb_bias_act, c.p("x"), c.p("b"), 1, 0, 128, c.p("y"), None, launches=0, written=False)
    assert c.outs["y"].untouched() and c.outs["mask"].untouched()
    for Din, Dout in ((64, 128), (16, 48), (1024, 2048)):
        check_bwd(gnn, 0, Din, Dout, 1, True, True, True, "randn", f"N=0 {Din}x{Dout}", seed=1,
                  x=np.zeros((0, Din), np.float32), W=np.ones((Dout, Din), np.float32),
                  dy=np.zeros((0, Dout), np.float32))
    z = Call(gnn, dict(x=np.zeros((0, 64), np.float32)), dict(dW=64 * 128, db=128))
    z.run(lib.gnnb_linear_bwd_mask, z.p("x"), None, z.p("x"), z.p("x"), 0, 64, 128, None, z.p("dW"), z.p("db"), None)
    assert (z.outs["dW"].body == 0).all() and (z.outs["db"].body == 0).all()
    check_linear2_bwd(gnn, 0, 32, 96, 1, "randn", "N=0", seed=2)
    d = Call(gnn, dict(x=np.zeros((0, 8), np.float32)), dict(db=8))
    d.run(lib.gnnb_bias_act_bwd, d.p("x"), d.p("x"), 1, 0, 8, d.p("x"), d.p("db"), None)
    assert (d.outs["db"].body == 0).all()


# ------------------------------------------------------------------------------------------------ misaligned operands
def aligned_groups(names):
    return [[k] for k in names] + [list(names)]


@pytest.mark.gpu
@pytest.mark.parametrize("off", [4, 8, 12])
@pytest.mark.parametrize("shape", [(5000, 128, 128), (4096, 256, 256), (300, 16, 8)])
def test_misaligned_linear(gnn, switches, shape, off):
    """gnnb_linear with x, W or y off a 16 B boundary: the library GEMM (the bits of the library on the same pointers),
    within the same bound; a misaligned bias keeps the wgmma route (the aligned call's bits, not the library's: the
    kernels read the bias element by element)"""
    N, K, Nout = shape
    x, W, b = gen_linear("randn", N, K, Nout, seed=off)
    base = check_linear(gnn, x, W, b, 1, N, K, Nout, "randn", f"{shape} aligned").outs["y"].bits
    if linear_route(N, K, Nout) != "lt":
        assert not torch.equal(base, library_bits(gnn, x, W, b, 1, N, K, Nout, "randn", f"{shape} aligned"))
    for group in aligned_groups(["x", "W", "b", "y"]):
        mis = frozenset(group)
        what = f"{shape} {group}@{off}"
        y = check_linear(gnn, x, W, b, 1, N, K, Nout, "randn", what, mis=mis, off=off).outs["y"].bits
        if linear_route(N, K, Nout, mis=mis) == "lt":
            assert torch.equal(y, library_bits(gnn, x, W, b, 1, N, K, Nout, "randn", what, mis=mis, off=off)), what
        else:
            assert torch.equal(y, base), f"{what}: not the aligned wgmma call's bits"


@pytest.mark.gpu
@pytest.mark.parametrize("off", [4, 8, 12])
@pytest.mark.parametrize("dims", [(5000, 64, 128), (5000, 48, 96), (4096, 128, 256)])
def test_misaligned_linear_bwd(gnn, switches, dims, off):
    """gnnb_linear_bwd: with relu or db, a misaligned dy, y or workspace is GNNB_EUNSUPPORTED; every other operand
    off its boundary sends its product to the library GEMM, within the same bound"""
    N, Din, Dout = dims
    for relu, db in ((1, 1), (0, 1), (0, 0)):
        names = ["dy", "x", "W", "dx", "dW", "db"] + (["y", "ws"] if relu else [])
        for group in aligned_groups(names):
            check_bwd(gnn, N, Din, Dout, relu, True, True, db, "randn", f"{dims} relu={relu} db={db} {group}@{off}",
                      seed=off, mis=frozenset(group), off=off)


# operands each entry needs on a 16 B boundary (GNNB_EUNSUPPORTED otherwise, include/gnnb200.h)
MUST_ALIGN = {"relu_mask": {"x", "W", "y", "mask"}, "linear2": {"x1", "x2", "W", "y"},
              "bias_act": {"x", "b", "y"}, "bias_act_bwd": {"dy", "y", "dpre"}, "bwd_mask": {"dy", "mask", "x", "dx"},
              "linear2_bwd": {"dy", "y", "ws", "x1", "x2", "dx1", "dx2"}}


@pytest.mark.gpu
@pytest.mark.parametrize("off", [4, 8, 12])
@pytest.mark.parametrize("entry", list(MUST_ALIGN))
def test_misaligned_tensor_core_only_entries(gnn, switches, entry, off):
    """the entries without a library fall-back: GNNB_EUNSUPPORTED when an operand the kernels read by vector is off
    its 16 B boundary, the float64 result when only the others are"""
    lib = lib_of(gnn)
    N, D = 1000, 128
    rng = np.random.default_rng(off)
    x, W, b = gen_linear("randn", N, 64, D, seed=off)
    dy = rng.standard_normal((N, D)).astype(np.float32)
    yf, m = forward_y(gnn, x, W, b, 1, mask=True)
    m = m.view(np.float32)
    if entry == "relu_mask":
        names = ["x", "W", "b", "y", "mask"]
        ins, outs = dict(x=x, W=W, b=b), dict(y=N * D, mask=N * 4)
        fn = lambda c: lib.gnnb_linear_relu_mask(c.p("x"), c.p("W"), c.p("b"), N, 64, D, c.p("y"), c.p("mask"), None)
    elif entry == "linear2":
        names = ["x1", "x2", "W", "b", "y"]
        ins, outs = dict(x1=x[:, :32].copy(), x2=x[:, 32:].copy(), W=W, b=b), dict(y=N * D)
        fn = lambda c: lib.gnnb_linear2(c.p("x1"), c.p("x2"), c.p("W"), c.p("b"), 1, N, 32, 32, D, c.p("y"), None)
    elif entry == "bias_act":
        names = ["x", "b", "y"]
        ins, outs = dict(x=yf, b=b), dict(y=N * D)
        fn = lambda c: lib.gnnb_bias_act(c.p("x"), c.p("b"), 1, N, D, c.p("y"), None)
    elif entry == "bias_act_bwd":
        names = ["dy", "y", "dpre", "db"]
        ins, outs = dict(dy=dy, y=yf), dict(dpre=N * D, db=D)
        fn = lambda c: lib.gnnb_bias_act_bwd(c.p("dy"), c.p("y"), 1, N, D, c.p("dpre"), c.p("db"), None)
    elif entry == "bwd_mask":
        names = ["dy", "mask", "x", "W", "dx", "dW", "db"]
        ins, outs = dict(dy=dy, mask=m, x=x, W=W), dict(dx=N * 64, dW=D * 64, db=D)
        fn = lambda c: lib.gnnb_linear_bwd_mask(c.p("dy"), c.p("mask"), c.p("x"), c.p("W"), N, 64, D, c.p("dx"),
                                                c.p("dW"), c.p("db"), None)
    else:
        for group in aligned_groups(["dy", "y", "ws", "x1", "x2", "W", "dx1", "dx2", "dW", "db"]):
            mis = frozenset(group)
            check_linear2_bwd(gnn, N, 32, 64, 1, "randn", f"{group}@{off}", seed=off, mis=mis, off=off,
                              rc=EUNSUPPORTED if mis & MUST_ALIGN[entry] else OK)
        return
    base = None
    for group in [[]] + aligned_groups(names):
        mis = frozenset(group)
        c = Call(gnn, ins, outs, {k: off for k in mis})
        rc = EUNSUPPORTED if mis & MUST_ALIGN[entry] else OK
        c.run(lambda: fn(c), rc=rc)
        if rc == OK:
            got = {k: c.outs[k].bits.clone() for k in outs}
            if base is None:
                base = got
            for k in outs:                                 # the kernels read the operand element by element: same bits
                assert torch.equal(got[k], base[k]), f"{entry} {k} at {group}@{off}: not the aligned call's bits"
    assert base is not None


# ------------------------------------------------------------------------------------------------ subnormal split parts
@pytest.mark.gpu
@pytest.mark.parametrize("route,K,Nout", [("ring", 128, 128), ("wide", 256, 256), ("lt", 128, 128)])
def test_subnormal_small_parts(gnn, switches, route, K, Nout):
    """x around 2^-115, so tf32_small(x) is subnormal: every route meets its bound (on an H100 the wgmma reads subnormal
    tf32 operands as they are: there is no flush floor)"""
    N = 4096
    rng = np.random.default_rng(K)
    x = (np.exp2(-115.0) * rng.uniform(1, 2, (N, K)) * rng.choice([-1, 1], (N, K))).astype(np.float32)
    W = rng.standard_normal((Nout, K)).astype(np.float32)
    switches(int(route != "lt"), 1)
    lib = lib_of(gnn)
    c = Call(gnn, dict(x=x, W=W), dict(y=N * Nout))
    c.run(lib.gnnb_linear, c.p("x"), c.p("W"), None, 0, N, K, Nout, c.p("y"), None, launches=LAUNCHES[route])
    ref, scale = fwd_ref(x, W, None, 0)
    r = ratio(c.out("y", (N, Nout)), ref, scale)
    REPORT.setdefault("subnormal", {})[route] = {"ratio": r, "gamma": gamma(route, K)}
    print(f"subnormal small parts, {route}: componentwise {r:.3e}, γ {gamma(route, K):.3e}")
    assert r <= gamma(route, K)


# ------------------------------------------------------------------------------------------------ the earlier shapes
LEGACY = [(1000, 128, 128), (777, 16, 8), (5000, 64, 256), (33, 1432, 16), (0, 8, 8), (4096, 64, 128),
          (130000, 128, 64), (300, 32, 16), (129, 96, 48), (1, 128, 128), (400000, 128, 128), (70001, 96, 128),
          (40000, 512, 512), (3000, 256, 256), (20001, 512, 128), (2048, 160, 384), (9000, 1024, 1024)]


@pytest.mark.gpu
@pytest.mark.parametrize("emulate", [1, 0])
@pytest.mark.parametrize("relu_flag,with_bias", [(1, True), (0, True), (1, False), (0, False)])
@pytest.mark.parametrize("N,Din,Dout", LEGACY)
def test_linear_c_abi(gnn, switches, N, Din, Dout, relu_flag, with_bias, emulate):
    """gnnb_linear and gnnb_linear_bwd on the layer shapes (GCN, GATConv's 512 -> 8 x 64, odd widths), with the
    tensor-core kernels and the emulated library GEMM (emulate = 1) or the library's fp32 sgemm alone (emulate = 0)"""
    switches(emulate, emulate)
    x, W, b = gen_linear("randn", N, Din, Dout, seed=N + Din, bias=with_bias)
    check_linear(gnn, x, W, b, relu_flag, N, Din, Dout, "randn", "forward", tc=bool(emulate))
    check_bwd(gnn, N, Din, Dout, relu_flag, True, True, True, "randn", "pullback", seed=N + Din, tc=bool(emulate))


@pytest.mark.gpu
@pytest.mark.parametrize("relu_flag,with_bias", [(1, True), (0, False)])
@pytest.mark.parametrize("N,D1,D2", [(70001, 128, 128), (5000, 96, 32), (129, 128, 64)])
def test_linear2_c_abi(gnn, switches, N, D1, D2, relu_flag, with_bias):
    """gnnb_linear2 and gnnb_linear2_bwd on sage_conv's shapes (Dout = 128)"""
    lib = lib_of(gnn)
    rng = np.random.default_rng(N + D1)
    x1, x2 = operand("randn", rng, N, D1, "x", 1), operand("randn", rng, N, D2, "x", 1)
    W = operand("randn", rng, 128, D1 + D2, "w", 1)
    b = bias_for("randn", rng, 128) if with_bias else None
    c = Call(gnn, dict(x1=x1, x2=x2, W=W, b=b), dict(y=N * 128))
    c.run(lib.gnnb_linear2, c.p("x1"), c.p("x2"), c.p("W"), c.p("b"), relu_flag, N, D1, D2, 128, c.p("y"), None,
          launches=linear2_launches(N, D1, D2, 128))
    ref, scale = fwd_ref(np.concatenate([x1, x2], 1), W, b, relu_flag)
    check(c.out("y", (N, 128)), ref, scale, "linear2", D1 + D2, "forward")
    check_linear2_bwd(gnn, N, D1, D2, relu_flag, "randn", "pullback", seed=N + D1,
                      want=("dx1", "dx2", "dW") + (("db",) if with_bias else ()))
