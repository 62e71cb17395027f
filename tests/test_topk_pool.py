"""Top-k pooling (graphneuralnetworks.jl_b200/readout.py over csrc/topk.cu's gnnb_topk_keep / gnnb_topk_score /
gnnb_topk_gate / gnnb_topk_gate_bwd; GNNlib/src/layers/pool.jl:14-27, GraphNeuralNetworks/src/layers/pool.jl:101-123).

The contract, stated below:
- the selection (`keep_ref`): per segment, keep every key >= the k_s-th largest non-NaN key, k_s = min(k, n_s) or
  ceil(ratio * n_s); NaN never kept nor counted; -0.0 == +0.0;
- score, gate and pullback (`ref_pool`): float64 torch autograd of y = p' x / norm(p), out = x[:, idx] .* σ.(y[idx]').

Back ends of the mirror: `FakeTopK`, the four entries restated on host pointers (swapped in over tests/fake_abi.py's
double), and, under -m gpu, the CUDA kernels.
"""
import ctypes as C
import gc
import math
import os
import re
import sys
from types import SimpleNamespace

import numpy as np
import pytest
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
OK, EINVAL, ESIZE, ECUDA, ENOMEM, EUNSUPPORTED, EINDEX = range(7)
F64 = torch.float64
KEY_DTYPES = [np.float32, np.float64, np.int32, np.int64]


def header_bound():
    with open(os.path.join(ROOT, "include", "gnnb200.h")) as f:
        return int(re.search(r"#define GNNB_TOPK_SMEM_MAX (\d+)", f.read()).group(1))


BOUND = header_bound()


# ---------------------------------------------------------------------------------------------- the entries in numpy
def keep_ref(keys, seg_ptr, k, ratio=0.0):
    """uint8 mask of gnnb_topk_keep"""
    keys = np.asarray(keys)
    n = len(keys)
    seg = [0, n] if seg_ptr is None else [int(v) for v in seg_ptr]
    out = np.zeros(n, np.uint8)
    flt = keys.dtype.kind == "f"
    for a, b in zip(seg[:-1], seg[1:]):
        v = keys[a:b]
        ns = b - a
        if ns == 0:
            continue
        ks = min(k, ns) if k >= 1 else min(ns, math.ceil(ratio * ns))
        ok = ~np.isnan(v) if flt else np.ones(ns, bool)
        fin = v[ok]
        r = min(ks, len(fin))
        if r == 0:
            continue
        vs = np.partition(fin, len(fin) - r)[len(fin) - r]
        out[a:b] = ok & (v >= vs)
    return out


def sigm(a):
    t = np.exp(-np.abs(a))
    return np.where(a >= 0, 1 / (1 + t), t / (1 + t))


def ref_pool(x, p, idx):
    """float64 autograd reference: x (D, n), p (D,), idx 0-based -> out (D, m) and a closure for (dx, dp)"""
    x = x.detach().to("cpu", F64).requires_grad_(True)
    p = p.detach().to("cpu", F64).requires_grad_(True)
    y = (p @ x) / torch.linalg.norm(p)
    out = x[:, idx] * torch.sigmoid(y[idx])[None, :]
    return x, p, out


def _fake_abi():
    sys.path.insert(0, os.path.join(ROOT, "tests"))
    import fake_abi
    return fake_abi


class FakeTopK:
    """the four gnnb_topk_* entries on host pointers (float64 inside); every other entry is the base double's"""

    def __init__(self, base):
        self.base, self.fa = base, _fake_abi()

    def __getattr__(self, name):
        return getattr(self.base, name)

    def _fail(self, code, msg):
        self.base._err = msg.encode()
        return code

    def gnnb_topk_keep(self, keys, kt, n, seg_ptr, n_seg, k, ratio, keep, status, stream):
        self.base.calls.append("gnnb_topk_keep")
        if kt not in range(4):
            return self._fail(EINVAL, "key_type")
        if not ((k >= 1 and ratio == 0.0) or (k == 0 and 0.0 < ratio <= 1.0)):
            return self._fail(EINVAL, "k / ratio")
        a = self.fa._arr
        ks = a(keys, (n,), KEY_DTYPES[kt]) if n else np.zeros(0, KEY_DTYPES[kt])
        seg = None if seg_ptr is None else a(seg_ptr, (n_seg + 1,), np.int64)
        if n:
            a(keep, (n,), np.uint8)[...] = keep_ref(ks, seg, k, ratio)
        return OK

    def gnnb_topk_score(self, x, n, D, p, y, stream):
        self.base.calls.append("gnnb_topk_score")
        a = self.fa._arr
        xv, pv = a(x, (n, D)).astype(np.float64), a(p, (D,)).astype(np.float64)
        a(y, (n,))[...] = xv @ pv / np.sqrt((pv * pv).sum())
        return OK

    def gnnb_topk_gate(self, x, n, D, y, idx, m, out, status, stream):
        self.base.calls.append("gnnb_topk_gate")
        if m == 0:
            return OK
        a = self.fa._arr
        ii = a(idx, (m,), np.int64)
        a(out, (m, D))[...] = a(x, (n, D)).astype(np.float64)[ii] * sigm(a(y, (n,)).astype(np.float64)[ii])[:, None]
        return OK

    def gnnb_topk_gate_bwd(self, x, n, D, y, p, idx, m, dout, dx, dp, status, stream):
        self.base.calls.append("gnnb_topk_gate_bwd")
        a = self.fa._arr
        xv, yv, pv = a(x, (n, D)).astype(np.float64), a(y, (n,)).astype(np.float64), a(p, (D,)).astype(np.float64)
        nrm = np.sqrt((pv * pv).sum())
        dxa = np.zeros((n, D))
        dpa = np.zeros(D)
        if m:
            ii = a(idx, (m,), np.int64)
            g = a(dout, (m, D)).astype(np.float64)
            s = sigm(yv[ii])
            dy = s * (1 - s) * (g * xv[ii]).sum(1)
            dxa[ii] = s[:, None] * g + dy[:, None] * pv[None, :] / nrm
            dpa = (dy[:, None] * xv[ii]).sum(0) / nrm - (dy * yv[ii]).sum() * pv / nrm ** 2
        a(dx, (n, D))[...] = dxa
        a(dp, (D,))[...] = dpa
        return OK


@pytest.fixture(params=["fake", pytest.param("cuda", marks=pytest.mark.gpu)])
def tb(request, gnn):
    """back end of the mirror: .dev, .calls (entries the fake saw, None on cuda), .tol (scale)"""
    if request.param == "fake":
        from gnnb200 import readout
        with _fake_abi().installed() as fake:
            saved = readout.lib
            readout.lib = FakeTopK(fake)
            try:
                yield SimpleNamespace(dev=torch.device("cpu"), calls=fake.calls, tol=1.0)
            finally:
                readout.lib = saved
    else:
        if not torch.cuda.is_available():
            pytest.skip("no CUDA device")
        yield SimpleNamespace(dev=torch.device("cuda"), calls=None, tol=4.0)


def close(got, ref, mag, tol):
    """|got - ref| <= tol * 2^-23 * (terms' magnitude) + tiny, elementwise"""
    got, ref, mag = (torch.as_tensor(v).detach().to("cpu", F64) for v in (got, ref, mag))
    assert got.shape == ref.shape
    bound = tol * 64 * 2.0 ** -23 * (mag + ref.abs()) + 1e-30
    bad = (got - ref).abs() > bound
    assert not bool(bad.any()), f"{int(bad.sum())} elements off; worst {float(((got - ref).abs() - bound).max()):.3e}"


# ---------------------------------------------------------------------------------------------- the reference's tests
def test_reference_topk_index(tb, gnn):
    y = torch.tensor([8, 7, 6, 5, 4, 3, 2, 1], dtype=torch.float32, device=tb.dev)
    assert gnn.topk_index(y, 4).tolist() == [1, 2, 3, 4]
    assert gnn.topk_index(y.reshape(1, 8), 4).tolist() == [1, 2, 3, 4]
    assert gnn.topk_index(y, 4).dtype == torch.int64


@pytest.mark.parametrize("adj_dtype", [torch.bool, torch.float64])
def test_reference_topkpool(tb, gnn, adj_dtype):
    N, k, C_in = 10, 4, 7
    torch.manual_seed(0)
    adj = (torch.rand(N, N) < 0.3).to(adj_dtype).to(tb.dev)
    t = gnn.TopKPool(adj, k, C_in, device=tb.dev)
    assert t.p.dtype == torch.float32 and tuple(t.p.shape) == (C_in,)
    assert t.A_tilde.dtype == adj_dtype and tuple(t.A_tilde.shape) == (k, k)
    X = torch.rand(C_in, N, device=tb.dev)
    out = t(X)
    assert tuple(out.shape) == (C_in, k)
    idx = gnn.topk_index((t.p.detach() @ X) / torch.linalg.norm(t.p.detach()), k) - 1
    assert torch.equal(t.A_tilde, adj[idx[:, None], idx[None, :]])


# ---------------------------------------------------------------------------------------------- topk_index
SPECIAL = [np.nan, -np.nan, 0.0, -0.0, np.inf, -np.inf, 1.0, -1.0, 1.0, 2.5, np.nan, -0.0]


@pytest.mark.parametrize("case", ["ties", "special", "int32", "int64", "int8", "bool", "float16", "allnan"])
def test_topk_index_statement(tb, gnn, case):
    rng = np.random.default_rng(1)
    vals = {"ties": rng.integers(0, 4, 40).astype(np.float32),
            "special": np.array(SPECIAL, np.float64),
            "int32": rng.integers(-2 ** 31, 2 ** 31, 50).astype(np.int32),
            "int64": np.concatenate([rng.integers(-2 ** 62, 2 ** 62, 50), [2 ** 63 - 1, -2 ** 63, 0, 0]]),
            "int8": rng.integers(-128, 128, 30).astype(np.int8),
            "bool": rng.integers(0, 2, 30).astype(bool),
            "float16": rng.standard_normal(30).astype(np.float16),
            "allnan": np.full(5, np.nan, np.float32)}[case]
    y = torch.as_tensor(vals).to(tb.dev)
    N = len(vals)
    keyv = vals.astype(np.int32) if vals.dtype in (np.int8, np.bool_) else \
        vals.astype(np.float32) if vals.dtype == np.float16 else vals
    for k in (1, 2, N // 2, N - 1, N, N + 1, 3 * N):
        if k < 1:
            continue
        got = gnn.topk_index(y, k).cpu().numpy()
        want = np.nonzero(keep_ref(keyv, None, k))[0] + 1
        assert np.array_equal(got, want), (case, k)


def test_topk_index_errors(tb, gnn):
    y = torch.arange(5, dtype=torch.float32, device=tb.dev)
    for k in (0, -1):
        with pytest.raises(ValueError):
            gnn.topk_index(y, k)
    with pytest.raises(TypeError):
        gnn.topk_index(y.to(torch.complex64), 2)
    with pytest.raises(TypeError):
        gnn.topk_index(y, 2.0)
    with pytest.raises(ValueError):
        gnn.topk_index(y.reshape(5, 1), 2)


def test_keep_statement_rules():
    """the statement itself on hand-worked cases"""
    assert keep_ref(np.array([1, 3, 3, 2], np.float32), None, 2).tolist() == [0, 1, 1, 0]
    assert keep_ref(np.array([1, 3, 3, 2], np.float32), None, 1).tolist() == [0, 1, 1, 0]
    assert keep_ref(np.array([np.nan, 1, np.nan], np.float32), None, 3).tolist() == [0, 1, 0]
    assert keep_ref(np.array([-0.0, 0.0, -1.0], np.float32), None, 1).tolist() == [1, 1, 0]
    assert keep_ref(np.array([5, 1, 2, 9, 9], np.int64), [0, 3, 3, 5], 0, 0.5).tolist() == [1, 0, 1, 1, 1]


# ---------------------------------------------------------------------------------------------- forward and gradients
@pytest.mark.parametrize("D,N,k", [(7, 10, 4), (1, 5, 2), (16, 40, 40), (33, 64, 1)])
def test_pool_matrix_form_grad(tb, gnn, D, N, k):
    torch.manual_seed(D * N + k)
    adj = torch.rand(N, N, device=tb.dev)
    t = gnn.TopKPool(adj, k, D, device=tb.dev)
    X = torch.randn(D, N, device=tb.dev, requires_grad=True)
    out = t(X)
    with torch.no_grad():
        y = (t.p @ X) / torch.linalg.norm(t.p)
    idx = gnn.topk_index(y, k) - 1
    xr, pr, ref = ref_pool(X, t.p, idx.cpu())
    close(out, ref, (xr.abs()[:, idx.cpu()]).detach(), tb.tol)
    g = torch.randn_like(out)
    (out * g).sum().backward()
    (ref * g.detach().to("cpu", F64)).sum().backward()
    mag = xr.abs().sum(0, keepdim=True).expand_as(xr) + 1
    close(X.grad, xr.grad, mag, tb.tol * 4)
    close(t.p.grad, pr.grad, xr.abs().sum(1) + 1, tb.tol * 4)
    assert torch.equal(X.grad[:, [i for i in range(N) if i not in set(idx.tolist())]],
                       torch.zeros(D, N - idx.numel(), device=tb.dev))


def test_a_tilde_rules(tb, gnn):
    adj = torch.arange(16, dtype=torch.float64, device=tb.dev).reshape(4, 4)
    t = gnn.TopKPool(adj, 2, 3, device=tb.dev)
    with torch.no_grad():
        t.p.copy_(torch.tensor([1.0, 0.0, 0.0]))
    X = torch.tensor([[1.0, 5.0, 5.0, 0.0], [0, 0, 0, 0], [0, 0, 0, 0]], device=tb.dev)
    t(X)                                                          # m == k: ids 2, 3
    assert torch.equal(t.A_tilde, adj[1:3, 1:3])
    X3 = torch.tensor([[5.0, 5.0, 5.0, 0.0], [0, 0, 0, 0], [0, 0, 0, 0]], device=tb.dev)
    with pytest.raises(ValueError, match="DimensionMismatch"):   # three ties for k = 2
        t(X3)
    one = gnn.TopKPool(torch.tensor([[7.0]], device=tb.dev), 3, 3, device=tb.dev)
    one(torch.ones(3, 1, device=tb.dev))                          # m == 1: fills A_tilde
    assert torch.equal(one.A_tilde, torch.full((3, 3), 7.0, dtype=torch.float32, device=tb.dev))
    with pytest.raises(TypeError):
        gnn.TopKPool(adj, 0.5, 3, device=tb.dev)
    nog = gnn.TopKPool(None, 2, 3, device=tb.dev)
    with pytest.raises(ValueError):
        nog(X)


# ---------------------------------------------------------------------------------------------- graph form
def _batch(gnn, sizes, dev, seed, perm=None):
    rng = np.random.default_rng(seed)
    gs = []
    for n in sizes:
        E = 3 * n
        s = rng.integers(1, n + 1, E) if n else np.zeros(0, np.int64)
        t = rng.integers(1, n + 1, E) if n else np.zeros(0, np.int64)
        gs.append((s, t, n))
    off, S, T, ind = 0, [], [], []
    for i, (s, t, n) in enumerate(gs):
        S.append(s + off); T.append(t + off); ind += [i + 1] * n
        off += n
    S, T, ind = np.concatenate(S), np.concatenate(T), np.array(ind, np.int64)
    if perm is not None:                                          # unsorted indicator: relabel nodes
        pm = rng.permutation(off)
        S, T, ind = pm[S - 1] + 1, pm[T - 1] + 1, np.empty_like(ind)
        ind[pm] = np.array(sum(([i + 1] * n for i, (_, _, n) in enumerate(gs)), []), np.int64)
    w = rng.random(len(S)).astype(np.float32)
    return gnn.GNNGraph(torch.as_tensor(S).to(dev), torch.as_tensor(T).to(dev), torch.as_tensor(w).to(dev),
                        num_nodes=off, num_graphs=len(sizes), graph_indicator=torch.as_tensor(ind).to(dev),
                        ndata={"f": torch.arange(off, dtype=torch.float32).reshape(1, off).to(dev)})


@pytest.mark.parametrize("k", [2, 5, 0.5, 1.0, 0.3])
@pytest.mark.parametrize("unsorted", [False, True])
def test_graph_form(tb, gnn, k, unsorted):
    sizes = [6, 0, 3, 1, 9, 0, 4]
    g = _batch(gnn, sizes, tb.dev, 7, perm=unsorted or None)
    D = 5
    torch.manual_seed(3)
    t = gnn.TopKPool(None, k, D, device=tb.dev)
    x = torch.randn(D, g.num_nodes, device=tb.dev)
    x[:, :4] = 1.0                     # equal scores in different graphs must not interact
    x.requires_grad_(True)
    h, xp, idx = t(g, x)
    with torch.no_grad():
        y = ((t.p @ x) / torch.linalg.norm(t.p)).cpu().numpy()
    ind = g.graph_indicator.cpu().numpy()
    want = np.zeros(g.num_nodes, np.uint8)
    kk, ratio = (k, 0.0) if isinstance(k, int) else (0, k)
    for gi in range(1, len(sizes) + 1):
        nodes = np.nonzero(ind == gi)[0]
        want[nodes] = keep_ref(y[nodes], None, kk, ratio)
    assert idx.cpu().tolist() == (np.nonzero(want)[0] + 1).tolist()
    xr, pr, ref = ref_pool(x, t.p, idx.cpu() - 1)
    close(xp, ref, xr.abs()[:, idx.cpu() - 1].detach(), tb.tol)
    g_out = torch.randn_like(xp)
    (xp * g_out).sum().backward()
    (ref * g_out.to("cpu", F64)).sum().backward()
    close(x.grad, xr.grad, xr.abs().sum(0, keepdim=True).expand_as(xr) + 1, tb.tol * 4)
    close(t.p.grad, pr.grad, xr.abs().sum(1) + 1, tb.tol * 4)
    drop = torch.nonzero(torch.as_tensor(want) == 0).reshape(-1).to(tb.dev) + 1
    r = gnn.remove_nodes(g, drop)
    assert h.num_nodes == r.num_nodes and h.num_graphs == r.num_graphs
    for a, b in ((h.s, r.s), (h.t, r.t), (h.w, r.w), (h.graph_indicator, r.graph_indicator),
                 (h.ndata["f"], r.ndata["f"])):
        assert torch.equal(a, b)


def test_graph_form_errors(tb, gnn):
    g = _batch(gnn, [3, 4], tb.dev, 1)
    for k in (0, -2, 1.5, 0.0):
        with pytest.raises((ValueError, TypeError)):
            gnn.TopKPool(None, k, 2, device=tb.dev)(g, torch.randn(2, 7, device=tb.dev))
    with pytest.raises(TypeError):
        gnn.TopKPool(None, 2, 2, device=tb.dev)(g, torch.randn(2, 7, device=tb.dev, dtype=F64))


# ---------------------------------------------------------------------------------------------- GPU: the entries
def _keep_dev(gnn, keys, seg=None, k=1, ratio=0.0, status=None):
    kt = {torch.float32: 0, torch.float64: 1, torch.int32: 2, torch.int64: 3}[keys.dtype]
    n = keys.numel()
    keep = torch.full((n,), 7, dtype=torch.uint8, device="cuda")
    rc = gnn._lib.lib.gnnb_topk_keep(keys.data_ptr(), kt, n, None if seg is None else seg.data_ptr(),
                                     1 if seg is None else seg.numel() - 1, k, ratio, keep.data_ptr(),
                                     None if status is None else status.data_ptr(), 0)
    return rc, keep


def _keys(dt, n, rng, distinct=None):
    if distinct is not None:
        v = rng.choice(np.array(distinct), n)
    else:
        v = rng.standard_normal(n) * 1e3 if np.dtype(dt).kind == "f" else rng.integers(-10 ** 6, 10 ** 6, n)
    return np.asarray(v).astype(dt)


@pytest.mark.gpu
@pytest.mark.parametrize("dt", KEY_DTYPES)
@pytest.mark.parametrize("n", [1, 2, 31, 32, 33, 1000, BOUND, BOUND + 1, 10 ** 6, 10 ** 7 + 1])
def test_gpu_keep_one_segment(gnn, dt, n):
    rng = np.random.default_rng(n)
    v = _keys(dt, n, rng)
    kd = torch.as_tensor(v).cuda()
    for k in sorted({1, max(1, n // 2), max(1, n - 1), n, n + 1}):
        rc, keep = _keep_dev(gnn, kd, k=k)
        assert rc == OK
        assert np.array_equal(keep.cpu().numpy(), keep_ref(v, None, k)), (dt, n, k)


@pytest.mark.gpu
@pytest.mark.parametrize("dt", KEY_DTYPES)
@pytest.mark.parametrize("mix", ["equal", "three", "zeros", "inf_nan"])
@pytest.mark.parametrize("bound", [None, 0, 64])
def test_gpu_keep_special(gnn, dt, mix, bound):
    flt = np.dtype(dt).kind == "f"
    if mix == "inf_nan" and not flt:
        pytest.skip("integers have no inf / NaN")
    distinct = {"equal": [3], "three": [-2, 5, 9], "zeros": [-0.0, 0.0, -1.0, 1.0] if flt else [0, -1, 1],
                "inf_nan": [np.inf, -np.inf, np.nan, 0.0, -0.0, 1.0]}[mix]
    rng = np.random.default_rng(5)
    try:
        if bound is not None:
            gnn._lib.check(gnn._lib.lib.gnnb_topk_set_smem_max(bound))
        for n in (5, 700, 20000):
            v = _keys(dt, n, rng, distinct)
            kd = torch.as_tensor(v).cuda()
            seg = torch.tensor([0, n // 3, n // 3, n], dtype=torch.int64, device="cuda")
            for k, ratio in ((1, 0.0), (n // 7 + 1, 0.0), (n, 0.0), (0, 0.5), (0, 1.0)):
                for sg in (None, seg):
                    rc, keep = _keep_dev(gnn, kd, sg, k, ratio)
                    assert rc == OK
                    want = keep_ref(v, None if sg is None else sg.cpu().numpy(), k, ratio)
                    assert np.array_equal(keep.cpu().numpy(), want), (mix, n, k, ratio, sg is None)
    finally:
        gnn._lib.lib.gnnb_topk_set_smem_max(BOUND)


@pytest.mark.gpu
@pytest.mark.parametrize("dt", KEY_DTYPES)
def test_gpu_keep_molecules(gnn, dt):
    rng = np.random.default_rng(11)
    sizes = rng.integers(10, 40, 10000)
    sizes[::7] = 0
    sizes[5] = BOUND + 300                                        # one large segment among them
    seg = np.concatenate([[0], np.cumsum(sizes)])
    v = _keys(dt, int(seg[-1]), rng, [1, 2, 3, 4, 5, 6, 7, 8] if dt in (np.int32, np.int64) else None)
    kd, sd = torch.as_tensor(v).cuda(), torch.as_tensor(seg).cuda()
    masks = []
    for k, ratio in ((4, 0.0), (0, 0.5)):
        want = keep_ref(v, seg, k, ratio)
        rc, keep = _keep_dev(gnn, kd, sd, k, ratio)
        assert rc == OK and np.array_equal(keep.cpu().numpy(), want)
        try:
            gnn._lib.check(gnn._lib.lib.gnnb_topk_set_smem_max(16))
            rc, keep2 = _keep_dev(gnn, kd, sd, k, ratio)
        finally:
            gnn._lib.lib.gnnb_topk_set_smem_max(BOUND)
        assert rc == OK and torch.equal(keep, keep2)
        masks.append(keep)
    rc, again = _keep_dev(gnn, kd, sd, 4)
    assert torch.equal(again, masks[0])


@pytest.mark.gpu
def test_gpu_rejected(gnn):
    lib = gnn._lib.lib
    kd = torch.randn(100, device="cuda")
    keep = torch.empty(100, dtype=torch.uint8, device="cuda")
    st = torch.full((1,), -1, dtype=torch.int32, device="cuda")
    assert lib.gnnb_topk_keep(kd.data_ptr(), 4, 100, None, 1, 2, 0.0, keep.data_ptr(), None, 0) == EINVAL
    for k, ratio in ((0, 0.0), (-1, 0.0), (0, 1.5), (0, -0.1), (2, 0.5), (0, float("nan"))):
        assert lib.gnnb_topk_keep(kd.data_ptr(), 0, 100, None, 1, k, ratio, keep.data_ptr(), None, 0) == EINVAL
    assert lib.gnnb_topk_keep(None, 0, 100, None, 1, 2, 0.0, keep.data_ptr(), None, 0) == ESIZE
    assert lib.gnnb_topk_keep(kd.data_ptr(), 0, -1, None, 1, 2, 0.0, keep.data_ptr(), None, 0) == ESIZE
    for bad in ([0, 50, 40, 100], [1, 50, 100], [0, 50, 99], [0, 101, 100]):
        sd = torch.tensor(bad, dtype=torch.int64, device="cuda")
        rc = lib.gnnb_topk_keep(kd.data_ptr(), 0, 100, sd.data_ptr(), len(bad) - 1, 2, 0.0, keep.data_ptr(),
                                st.data_ptr(), 0)
        assert rc == OK and int(st.item()) == EINVAL and int(keep.sum()) == 0, bad
    sd = torch.tensor([0, 50, 100], dtype=torch.int64, device="cuda")
    lib.gnnb_topk_keep(kd.data_ptr(), 0, 100, sd.data_ptr(), 2, 2, 0.0, keep.data_ptr(), st.data_ptr(), 0)
    assert int(st.item()) == OK and int(keep.sum()) == 4
    x = torch.randn(100, 8, device="cuda")
    y = torch.randn(100, device="cuda")
    p = torch.randn(8, device="cuda")
    out = torch.empty(3, 8, device="cuda")
    idx = torch.tensor([1, 100, 5], device="cuda")
    assert lib.gnnb_topk_gate(x.data_ptr(), 100, 8, y.data_ptr(), idx.data_ptr(), 3, out.data_ptr(), st.data_ptr(),
                              0) == OK
    assert int(st.item()) == EINDEX
    dx = torch.empty_like(x)
    dp = torch.empty_like(p)
    for ids in ([1, 5, 5], [5, 1, 7], [-1, 2, 3]):
        idx = torch.tensor(ids, device="cuda")
        assert lib.gnnb_topk_gate_bwd(x.data_ptr(), 100, 8, y.data_ptr(), p.data_ptr(), idx.data_ptr(), 3,
                                      out.data_ptr(), dx.data_ptr(), dp.data_ptr(), st.data_ptr(), 0) == OK
        assert int(st.item()) == EINDEX, ids
    assert lib.gnnb_topk_gate_bwd(x.data_ptr(), 2, 8, y.data_ptr(), p.data_ptr(), idx.data_ptr(), 3, out.data_ptr(),
                                  dx.data_ptr(), dp.data_ptr(), None, 0) == EINDEX
    assert lib.gnnb_topk_score(x.data_ptr(), 100, 0, p.data_ptr(), y.data_ptr(), 0) == ESIZE
    assert lib.gnnb_topk_score(None, 100, 8, p.data_ptr(), y.data_ptr(), 0) == ESIZE
    assert lib.gnnb_topk_set_smem_max(BOUND + 1) == EINVAL


@pytest.mark.gpu
@pytest.mark.parametrize("D", [1, 3, 4, 127, 128, 129, 512, 1500])
@pytest.mark.parametrize("offset", [0, 1])
def test_gpu_score_gate_bwd(gnn, D, offset):
    lib = gnn._lib.lib
    n, m = 3001, 1200
    torch.manual_seed(D)
    xb = torch.randn(n * D + offset, device="cuda")
    x = xb[offset:].view(n, D)                                     # offset 1: rows start 4 B past 16 B alignment
    pb = torch.randn(D + offset, device="cuda")
    p = pb[offset:]
    gb = torch.randn(m * D + offset, device="cuda")
    dout = gb[offset:].view(m, D)
    idx = torch.sort(torch.randperm(n, device="cuda")[:m]).values
    res = []
    for _ in range(2):
        y = torch.empty(n, device="cuda")
        out = torch.empty(m * D + offset, device="cuda")[offset:].view(m, D)
        dx = torch.empty(n * D + offset, device="cuda")[offset:].view(n, D)
        dp = torch.empty(D, device="cuda")
        gnn._lib.check(lib.gnnb_topk_score(x.data_ptr(), n, D, p.data_ptr(), y.data_ptr(), 0))
        gnn._lib.check(lib.gnnb_topk_gate(x.data_ptr(), n, D, y.data_ptr(), idx.data_ptr(), m, out.data_ptr(), None, 0))
        gnn._lib.check(lib.gnnb_topk_gate_bwd(x.data_ptr(), n, D, y.data_ptr(), p.data_ptr(), idx.data_ptr(), m,
                                              dout.data_ptr(), dx.data_ptr(), dp.data_ptr(), None, 0))
        res.append((y.clone(), out.clone(), dx.clone(), dp.clone()))
    for a, b in zip(*res):
        assert torch.equal(a, b)
    y, out, dx, dp = res[0]
    xd, pd, gd = x.to(F64), p.to(F64), dout.to(F64)
    nrm = torch.linalg.norm(pd)
    close(y, xd @ pd / nrm, xd.abs() @ pd.abs() / nrm, 1)
    yd = y.to(F64)                                                 # the gate and pullback from the device's own y
    s = torch.sigmoid(yd[idx])
    close(out, xd[idx] * s[:, None], xd[idx].abs(), 1)
    dy = s * (1 - s) * (gd * xd[idx]).sum(1)
    dym = s * (1 - s) * (gd * xd[idx]).abs().sum(1)
    dx_ref = torch.zeros_like(xd)
    dx_ref[idx] = s[:, None] * gd + dy[:, None] * pd[None] / nrm
    dx_mag = torch.zeros_like(xd)
    dx_mag[idx] = gd.abs() + dym[:, None] * pd.abs()[None] / nrm
    close(dx, dx_ref, dx_mag, 2)
    rest = torch.ones(n, dtype=torch.bool, device="cuda")
    rest[idx] = False
    assert torch.equal(dx[rest], torch.zeros_like(dx[rest]))
    dp_ref = (dy[:, None] * xd[idx]).sum(0) / nrm - (dy * yd[idx]).sum() * pd / nrm ** 2
    dp_mag = (dym[:, None] * xd[idx].abs()).sum(0) / nrm + (dym * yd[idx].abs()).sum() * pd.abs() / nrm ** 2
    close(dp, dp_ref, dp_mag, 8)


@pytest.mark.gpu
def test_gpu_rmat_selection_and_plan(gnn):
    """The plans are the library's own cudaMalloc allocations: blocks torch's allocator keeps cached from earlier tests
    are handed back first, and the features are dropped before the fresh plan is built."""
    n, E, D = 10 ** 7, 10 ** 8, 128
    gc.collect()
    torch.cuda.empty_cache()
    g = gnn.rmat_graph(n, E, seed=3, device="cuda")
    g.plan()
    torch.manual_seed(0)
    t = gnn.TopKPool(None, 0.5, D, device="cuda")
    x = torch.randn(D, n, device="cuda")
    with torch.no_grad():
        h, xp, idx = t(g, x)
        y = torch.empty(n, device="cuda")
        gnn._lib.check(gnn._lib.lib.gnnb_topk_score(gnn.rows(x).data_ptr(), n, D, t.p.data_ptr(), y.data_ptr(), 0))
    del x, xp
    v = torch.sort(y, descending=True).values[math.ceil(0.5 * n) - 1]
    want = torch.nonzero(y >= v).reshape(-1) + 1
    assert torch.equal(idx, want)
    del g, y, v, want
    gc.collect()
    torch.cuda.empty_cache()
    f = gnn.GNNGraph(h.s, h.t, h.w, num_nodes=h.num_nodes)
    f.plan()
    for tr in (False, True):
        for a, b in zip(gnn.csr(h, transposed=tr), gnn.csr(f, transposed=tr)):
            assert torch.equal(a, b), tr
