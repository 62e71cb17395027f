"""Attention pooling (graphneuralnetworks.jl_b200/readout.py's global_attention_pool and GlobalAttentionPool over
csrc/set2set.cu's gnnb_attention_pool / gnnb_attention_pool_bwd; GNNlib/src/layers/pool.jl:7-12,
GraphNeuralNetworks/src/layers/pool.jl:1-99), and GlobalPool.

The contract, stated below:
- the reference (`ref_pool`, float64 torch, one graph at a time): u_g = ffeat(x_g) softmax(fgate(x_g))ᵀ, u = 0 for a
  graph without nodes;
- the C entries (`entry_fwd` / `entry_bwd`, numpy float64): on a plan (s, t), the per-target softmax statistics of the
  gate, u, and the pullback dgate_e_k = α_k (<du_{t_k}, f_{s_k}> − <du_{t_k}, u_{t_k}>), dfe_k = α_k du_{t_k}.

Back ends of the mirror: `FakePool`, the entries restated on host pointers (swapped in over tests/fake_abi.py's double),
and, under -m gpu, the CUDA kernels.  The layer cases run on both routes: the fused pass (the default for a gate of one
row) and the softmax_nodes / reduce_nodes composition (the bound patched to 0).
"""
import operator
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


def header_bound():
    with open(os.path.join(ROOT, "include", "gnnb200.h")) as f:
        return int(re.search(r"#define GNNB_SET2SET_MAX_D (\d+)", f.read()).group(1))


BOUND = header_bound()


# ---------------------------------------------------------------------------------------------- the entries in numpy
def entry_fwd(s, t, nd, f, gate):
    """u (nd, D), seg_max, seg_sum of gnnb_attention_pool in float64; f (ns, D), gate (ns,)"""
    f, gate = np.asarray(f, np.float64), np.asarray(gate, np.float64)
    sc = gate[s]
    M = np.full(nd, -np.inf)
    np.maximum.at(M, t, sc)
    ex = np.exp(sc - M[t])
    S = np.zeros(nd)
    np.add.at(S, t, ex)
    u = np.zeros((nd, f.shape[1]))
    np.add.at(u, t, ex[:, None] * f[s])
    return u / np.where(S > 0, S, 1)[:, None], M, S


def entry_bwd(s, t, nd, f, gate, u, M, S, du):
    """dfe (E, D), dgate_e (E,) of gnnb_attention_pool_bwd in float64"""
    f, gate, u, du = (np.asarray(a, np.float64) for a in (f, gate, u, du))
    al = np.exp(gate[s] - M[t]) / S[t]
    T = (du * u).sum(1)
    dg = al * ((du[t] * f[s]).sum(1) - T[t])
    return al[:, None] * du[t], dg


def dgate_magnitude(s, t, f, gate, u, M, S, du):
    """the scale of dgate_e's rounding error: its terms in absolute value (<du, f> − T cancels for a sharp softmax)"""
    f, u, du = (np.abs(np.asarray(a, np.float64)) for a in (f, u, du))
    al = np.exp(np.asarray(gate, np.float64)[s] - M[t]) / S[t]
    return al * ((du[t] * f[s]).sum(1) + (du * u).sum(1)[t])


def _fake_abi():
    sys.path.insert(0, os.path.join(ROOT, "tests"))
    import fake_abi
    return fake_abi


class FakePool:
    """gnnb_attention_pool and gnnb_attention_pool_bwd on host pointers over `entry_fwd` / `entry_bwd`; every other entry
    is the base double's."""

    def __init__(self, base):
        self.base, self.fa = base, _fake_abi()

    def __getattr__(self, name):
        return getattr(self.base, name)

    def _fail(self, code, msg):
        self.base._err = msg.encode()
        return code

    def _check(self, D):
        if D < 1:
            return self._fail(ESIZE, "D must be >= 1")
        if D > BOUND:
            return self._fail(EUNSUPPORTED, "D above GNNB_SET2SET_MAX_D")
        return OK

    def gnnb_attention_pool(self, h, f, gate, D, u, smax, ssum, stream):
        self.base.calls.append("gnnb_attention_pool")
        rc = self._check(D)
        if rc != OK:
            return rc
        p, a = self.base._p(h), self.fa._arr
        uu, M, S = entry_fwd(p.s, p.t, p.nd, a(f, (p.ns, D)), a(gate, (p.ns,)))
        a(u, (p.nd, D))[...] = uu
        a(smax, (p.nd,))[...] = M
        a(ssum, (p.nd,))[...] = S
        return OK

    def gnnb_attention_pool_bwd(self, h, f, gate, u, smax, ssum, du, D, dfe, dgate, stream):
        self.base.calls.append("gnnb_attention_pool_bwd")
        rc = self._check(D)
        if rc != OK:
            return rc
        p, a = self.base._p(h), self.fa._arr
        if p.E == 0:
            return OK
        de, dg = entry_bwd(p.s, p.t, p.nd, a(f, (p.ns, D)), a(gate, (p.ns,)), a(u, (p.nd, D)), a(smax, (p.nd,)),
                           a(ssum, (p.nd,)), a(du, (p.nd, D)))
        a(dfe, (p.E, D))[...] = de
        a(dgate, (p.E,))[...] = dg
        return OK


@pytest.fixture(params=["fake", pytest.param("cuda", marks=pytest.mark.gpu)])
def sb(request, gnn):
    """back end of the mirror: .dev, .calls (entries the fake saw, None on cuda), .tol (scale)"""
    if request.param == "fake":
        from gnnb200 import readout
        with _fake_abi().installed() as fake:
            saved = readout.lib
            readout.lib = FakePool(fake)
            try:
                yield SimpleNamespace(dev=torch.device("cpu"), calls=fake.calls, tol=1.0)
            finally:
                readout.lib = saved
    else:
        if not torch.cuda.is_available():
            pytest.skip("no CUDA device")
        yield SimpleNamespace(dev=torch.device("cuda"), calls=None, tol=4.0)


@pytest.fixture(params=["fused", "composed"])
def route(request, monkeypatch):
    """the default routing, or every gate through the composition"""
    if request.param == "composed":
        from gnnb200 import readout
        monkeypatch.setattr(readout, "_ATTENTION_POOL_MAX_D", 0)
    return request.param


# ---------------------------------------------------------------------------------------------- the reference
def ref_pool(Wg, bg, Wf, bf, x, gi, G, graphs=None):
    """(chout, len(graphs)) for the graphs (0-based ids, all by default) of a batch with 1-based indicator gi: per graph
    (Wf x_g .+ bf) softmax(Wg x_g .+ bg)ᵀ"""
    graphs = range(G) if graphs is None else graphs
    cols = []
    for k in graphs:
        xg = x[:, torch.as_tensor(gi == k + 1)]
        if xg.shape[1] == 0:
            cols.append(torch.zeros(Wf.shape[0], dtype=F64))
            continue
        a = torch.softmax((Wg @ xg + bg[:, None])[0], dim=0)
        cols.append((Wf @ xg + bf[:, None]) @ a)
    return torch.stack(cols, dim=1)


def rel(a, b):
    a, b = a.detach().double().cpu(), b.detach().double().cpu()
    nb = torch.linalg.norm(b)
    return float(torch.linalg.norm(a - b) / nb) if nb > 0 else float(torch.linalg.norm(a))


def batch_graph(gnn, gi, G, dev):
    """a graph of len(gi) nodes with one self loop each and the 1-based graph indicator gi over G graphs"""
    n = len(gi)
    s = torch.arange(1, n + 1, device=dev)
    return gnn.GNNGraph(s, s.clone(), None, num_nodes=n, graph_indicator=torch.as_tensor(gi, device=dev),
                        num_graphs=G)


def indicator(sizes, rng=None):
    gi = np.concatenate([np.full(k, i + 1) for i, k in enumerate(sizes)] + [np.zeros(0)]).astype(np.int64)
    return gi if rng is None else rng.permutation(gi)


def pool_layer(gnn, chin, chout, dev, seed=0):
    from gnnb200.layers import _Dense
    torch.manual_seed(seed)
    fgate, ffeat = _Dense(chin, 1, device=dev), _Dense(chin, chout, device=dev)
    with torch.no_grad():                                # non-zero biases, so that every term is exercised
        gen = torch.Generator().manual_seed(seed)
        fgate.bias.copy_(torch.randn(1, generator=gen))
        ffeat.bias.copy_(torch.randn(chout, generator=gen) * 0.3)
    return gnn.GlobalAttentionPool(fgate, ffeat)


def params64(l):
    return [p.detach().cpu().double().requires_grad_(True)
            for p in (l.fgate.weight, l.fgate.bias, l.ffeat.weight, l.ffeat.bias)]


def run_case(gnn, sb, sizes, chin, chout, gi=None, G=None, scale=1.0, seed=0, fwd_tol=2e-5, grad_tol=1e-4):
    rng = np.random.default_rng(seed)
    gi = indicator(sizes) if gi is None else gi
    G = len(sizes) if G is None else G
    xa = (rng.standard_normal((chin, len(gi))) * scale).astype(np.float32)
    g = batch_graph(gnn, gi, G, sb.dev)
    l = pool_layer(gnn, chin, chout, sb.dev, seed)
    x = torch.as_tensor(xa, device=sb.dev).requires_grad_(True)
    y = l(g, x)
    assert y.shape == (chout, G) and y.dtype == torch.float32
    P = params64(l)
    x64 = torch.as_tensor(xa, dtype=F64).requires_grad_(True)
    ref = ref_pool(*P, x64, gi, G)
    assert rel(y, ref) < fwd_tol * sb.tol, rel(y, ref)
    cot = torch.randn(ref.shape, dtype=F64, generator=torch.Generator().manual_seed(3))
    got = torch.autograd.grad((y.double() * cot.to(y.device)).sum(),
                              [x, l.fgate.weight, l.fgate.bias, l.ffeat.weight, l.ffeat.bias])
    want = torch.autograd.grad((ref * cot).sum(), [x64] + P)
    for name, a, w in zip(("x", "Wgate", "bgate", "Wfeat", "bfeat"), got, want):
        if name == "bgate":                              # softmax is shift-invariant: 0 up to rounding
            assert abs(float(a)) < grad_tol * sb.tol * float(torch.linalg.norm(want[0])), (name, float(a))
        else:
            assert rel(a, w) < grad_tol * sb.tol, (name, rel(a, w))
    return y


# ---------------------------------------------------------------------------------------------- the statements
def test_entry_statement_matches_autograd():
    """entry_bwd is the pullback of entry_fwd's u"""
    rng = np.random.default_rng(1)
    s, t, nd, D = np.arange(12), np.array([0] * 5 + [2] * 7), 3, 4
    f, gate, du = rng.standard_normal((12, D)), rng.standard_normal(12), rng.standard_normal((nd, D))
    u, M, S = entry_fwd(s, t, nd, f, gate)
    assert (u[1] == 0).all() and M[1] == -np.inf and S[1] == 0
    dfe, dg = entry_bwd(s, t, nd, f, gate, u, M, S, du)
    ft, gt = torch.tensor(f, requires_grad=True), torch.tensor(gate, requires_grad=True)
    ut = torch.zeros(nd, D, dtype=F64)
    for i in (0, 2):
        ut = ut.index_put((torch.tensor(i),), ft[t == i].t() @ torch.softmax(gt[t == i], 0))
    gf, gg = torch.autograd.grad((ut * torch.tensor(du)).sum(), [ft, gt])
    assert np.allclose(dfe, gf.numpy()) and np.allclose(dg, gg.numpy())


def test_module_bound_is_the_header_bound(gnn):
    from gnnb200 import readout
    assert readout._ATTENTION_POOL_MAX_D == BOUND == 1024


# ---------------------------------------------------------------------------------------------- the layer
@pytest.mark.parametrize("chin,chout", [(6, 5), (3, 1), (4, 32), (8, 129)])
def test_forward_and_gradients(gnn, sb, route, chin, chout):
    """GlobalAttentionPool(Dense(chin, 1), Dense(chin, chout)): u and the gradients of x and of all four parameters
    against float64"""
    run_case(gnn, sb, [1, 7, 1, 40, 150, 3], chin, chout, seed=chin + chout)
    if sb.calls is not None:
        assert ("gnnb_attention_pool" in sb.calls) == (route == "fused")
        assert ("gnnb_attention_pool_bwd" in sb.calls) == (route == "fused")


def test_graph_without_nodes(gnn, sb, route):
    """graph 3 of 5 has no nodes, and graph 6 is beyond every id the indicator uses: their u is exactly 0"""
    gi = np.concatenate([indicator([4, 6]), np.full(5, 4), np.full(2, 5)])
    y = run_case(gnn, sb, None, 8, 4, gi=gi, G=6)
    assert (y[:, 2] == 0).all() and (y[:, 5] == 0).all()


def test_unsorted_indicator(gnn, sb, route):
    run_case(gnn, sb, None, 16, 12, gi=indicator([5, 1, 30, 9], np.random.default_rng(4)), G=4)


def test_sharp_gates(gnn, sb, route):
    """x scaled by 30: the softmax is nearly one-hot in most graphs"""
    run_case(gnn, sb, [3, 20, 64], 5, 7, scale=30.0, grad_tol=3e-4)


def test_routes_agree(gnn, sb, monkeypatch):
    """the fused pass against the composition on the same inputs, forward and every gradient"""
    from gnnb200 import readout
    rng = np.random.default_rng(5)
    gi = indicator([3, 50, 1, 200, 17], rng)
    xa = rng.standard_normal((20, len(gi))).astype(np.float32)
    outs = []
    for bound in (BOUND, 0):
        monkeypatch.setattr(readout, "_ATTENTION_POOL_MAX_D", bound)
        g = batch_graph(gnn, gi, 5, sb.dev)
        l = pool_layer(gnn, 20, 24, sb.dev, seed=9)
        x = torch.as_tensor(xa, device=sb.dev).requires_grad_(True)
        y = l(g, x)
        cot = torch.randn(y.shape, generator=torch.Generator().manual_seed(2)).to(sb.dev)
        outs.append([y] + list(torch.autograd.grad((y * cot).sum(), [x, l.fgate.weight, l.ffeat.weight, l.ffeat.bias])))
    for a, b in zip(*outs):
        assert rel(a, b) < 2e-5 * sb.tol


def test_per_channel_gate_composes(gnn, sb):
    """a gate of D rows (one softmax per channel) takes the composition, as in the reference"""
    gi = indicator([4, 9, 2])
    g = batch_graph(gnn, gi, 3, sb.dev)
    x = torch.as_tensor(np.random.default_rng(2).standard_normal((3, len(gi))).astype(np.float32), device=sb.dev)
    l = gnn.GlobalAttentionPool(lambda v: 2 * v)
    u = l(g, x)
    x64 = x.double().cpu()
    ref = torch.stack([(x64[:, gi == k + 1] * torch.softmax(2 * x64[:, gi == k + 1], dim=1)).sum(1)
                       for k in range(3)], dim=1)
    assert rel(u, ref) < 2e-6 * sb.tol
    if sb.calls is not None:
        assert "gnnb_attention_pool" not in sb.calls


def test_argument_errors(gnn, sb):
    gi = indicator([3, 4])
    g = batch_graph(gnn, gi, 2, sb.dev)
    l = pool_layer(gnn, 5, 4, sb.dev)
    with pytest.raises(AssertionError):
        l(g, torch.zeros(5, 6, device=sb.dev))           # 6 columns, 7 nodes
    x = torch.zeros(5, 7, device=sb.dev)
    with pytest.raises(AssertionError):                  # a gate with a column too many
        gnn.GlobalAttentionPool(lambda v: torch.zeros(1, 8, device=sb.dev))(g, x)


def _regular_graph(gnn, n, dev, ndata=None):
    """a 4-regular graph on n nodes (i ~ i ± 1, i ± 2 mod n), both directions"""
    i = np.arange(n)
    s = np.concatenate([i, i, i, i]) + 1
    t = np.concatenate([(i + 1) % n, (i - 1) % n, (i + 2) % n, (i - 2) % n]) + 1
    return gnn.GNNGraph(torch.as_tensor(s, device=dev), torch.as_tensor(t, device=dev), num_nodes=n, ndata=ndata)


def test_reference_global_pool(gnn, sb):
    """GraphNeuralNetworks/test/layers/pool.jl:1-24"""
    p = gnn.GlobalPool(operator.add)
    n, chin, ng = 10, 6, 3
    torch.manual_seed(0)
    X = torch.rand(6, n, device=sb.dev)
    g = _regular_graph(gnn, n, sb.dev, ndata=X)
    u = p(g, X)
    assert torch.allclose(u, X.sum(1, keepdim=True), atol=1e-6)
    g = gnn.batch([_regular_graph(gnn, n, sb.dev, ndata=torch.rand(chin, n, device=sb.dev)) for _ in range(ng)])
    u = p(g, g.x)
    assert u.shape == (chin, ng)
    assert torch.allclose(u[:, [0]], g.x[:, :n].sum(1, keepdim=True), atol=1e-6)
    assert torch.equal(p(g).gdata["u"], u)
    x = g.x.clone().requires_grad_(True)
    cot = torch.randn(chin, ng, device=sb.dev)
    (dx,) = torch.autograd.grad((p(g, x) * cot).sum(), [x])
    assert torch.equal(dx, cot[:, torch.as_tensor(gnn.graph_indicator(g), device=sb.dev) - 1])


def test_reference_global_attention_pool(gnn, sb, route):
    """GraphNeuralNetworks/test/layers/pool.jl:26-45: four trainables, a (chout, ng) readout, gradients against float64;
    and p(g).gdata["u"] is that readout"""
    n, chin, chout, ng = 10, 6, 5, 3
    p = pool_layer(gnn, chin, chout, sb.dev)
    assert len(list(p.parameters())) == 4
    torch.manual_seed(1)
    g = gnn.batch([_regular_graph(gnn, n, sb.dev, ndata=torch.rand(chin, n, device=sb.dev)) for _ in range(ng)])
    u = p(g, g.x)
    assert u.shape == (chout, ng)
    h = p(g)
    assert torch.equal(h.gdata["u"], u) and h.ndata is not None and torch.equal(h.x, g.x)
    gi = gnn.graph_indicator(g).cpu().numpy()
    P = params64(p)
    x64 = g.x.detach().cpu().double().requires_grad_(True)
    assert rel(u, ref_pool(*P, x64, gi, ng)) < 2e-6 * sb.tol
    x = g.x.clone().requires_grad_(True)
    got = torch.autograd.grad(p(g, x).sum(), [x] + list(p.parameters()))
    want = torch.autograd.grad(ref_pool(*P, x64, gi, ng).sum(), [x64] + P)
    for k, (a, w) in enumerate(zip(got, want)):
        if k == 2:                                       # the gate's bias: 0 up to rounding
            assert abs(float(a)) < 1e-5 * sb.tol * float(torch.linalg.norm(want[0]))
        else:
            assert rel(a, w) < 1e-5 * sb.tol


def test_modules_are_registered(gnn):
    from gnnb200.layers import _Dense
    p = gnn.GlobalAttentionPool(_Dense(3, 1))
    assert len(list(p.parameters())) == 2 and p.ffeat is gnn.identity
    assert isinstance(p, gnn.GNNLayer) and isinstance(gnn.GlobalPool(max), gnn.GNNLayer)
    q = gnn.GlobalAttentionPool(lambda v: v[:1], lambda v: v)
    assert len(list(q.parameters())) == 0
    p.eval()
    assert not p.fgate.training


def test_set2set_graph_call(gnn, sb, monkeypatch):
    """Set2Set's l(g) puts the readout in gdata"""
    if sb.calls is not None:                             # the double restates the composition's entries only
        from gnnb200 import readout
        monkeypatch.setattr(readout, "_SET2SET_MAX_D", 0)
    gi = indicator([4, 6])
    g = batch_graph(gnn, gi, 2, sb.dev)
    g = gnn.GNNGraph(g, ndata=torch.randn(3, len(gi), device=sb.dev))
    l = gnn.Set2Set(3, 2, device=sb.dev)
    assert torch.equal(l(g).gdata["u"], l(g, g.x))


# ---------------------------------------------------------------------------------------------- GPU: the entries
def _cuda():
    if not torch.cuda.is_available():
        pytest.skip("no CUDA device")


def plan_of(gnn, gi, G, chunk=None):
    from gnnb200 import readout
    try:
        if chunk is not None:
            gnn._lib.check(gnn._lib.lib.gnnb_set_chunk_edges(chunk))
        return readout._IndicatorPlan(torch.as_tensor(gi), G, torch.device("cuda"))
    finally:
        if chunk is not None:
            gnn._lib.lib.gnnb_set_chunk_edges(128)


def call_entries(gnn, ip, f, gate, du, offset=0):
    """the two entries on cuda arrays f (N, D), gate (N,), du (G, D); offset > 0 places every array that many floats
    into its buffer (misaligned for the scalar path)"""
    lib, chk = gnn._lib.lib, gnn._lib.check
    N, D = f.shape
    G = du.shape[0]

    def buf(shape, src=None):
        b = torch.zeros(int(np.prod(shape)) + offset, dtype=torch.float32, device="cuda")
        v = b[offset:].view(shape)
        if src is not None:
            v.copy_(src)
        return v
    f, gate, du = buf((N, D), f), buf((N,), gate), buf((G, D), du)
    u, dfe, dg = buf((G, D)), buf((N, D)), buf((N,))
    smax, ssum = buf((G,)), buf((G,))
    st = torch.cuda.current_stream().cuda_stream
    chk(lib.gnnb_attention_pool(ip.plan.h, f.data_ptr(), gate.data_ptr(), D, u.data_ptr(), smax.data_ptr(),
                                ssum.data_ptr(), st))
    chk(lib.gnnb_attention_pool_bwd(ip.plan.h, f.data_ptr(), gate.data_ptr(), u.data_ptr(), smax.data_ptr(),
                                    ssum.data_ptr(), du.data_ptr(), D, dfe.data_ptr(), dg.data_ptr(), st))
    torch.cuda.synchronize()
    return u, smax, ssum, dfe, dg


def check_entries(gnn, gi, G, D, chunk=None, scale=1.0, rising=False, offset=0, seed=0, tol=2e-5):
    rng = np.random.default_rng(seed)
    N = len(gi)
    f = rng.standard_normal((N, D)).astype(np.float32)
    gate = rng.standard_normal(N) * scale
    if rising:                                           # the gate increases along each graph: the max moves every node
        gate = np.arange(N) / max(N, 1) * 40.0
    gate = gate.astype(np.float32)
    du = rng.standard_normal((G, D)).astype(np.float32)
    ip = plan_of(gnn, gi, G, chunk)
    u, smax, ssum, dfe, dg = (a.cpu().numpy().astype(np.float64)
                              for a in call_entries(gnn, ip, torch.as_tensor(f).cuda(), torch.as_tensor(gate).cuda(),
                                                    torch.as_tensor(du).cuda(), offset))
    s, t = np.arange(N), gi - 1
    uu, M, S = entry_fwd(s, t, G, f, gate)
    de, dgr = entry_bwd(s, t, G, f, gate, uu, M, S, du)
    has = S > 0
    assert (u[~has] == 0).all() and (smax[~has] == -np.inf).all() and (ssum[~has] == 0).all()
    if has.any():
        assert rel(torch.as_tensor(u), torch.as_tensor(uu)) < tol
        assert (smax[has] == M[has]).all()               # the max of float32 gates is exact
        assert np.allclose(ssum[has], S[has], rtol=1e-4)
    if N:
        assert np.linalg.norm(dfe - de) / np.linalg.norm(de) < tol
        mag = dgate_magnitude(s, t, f, gate, uu, M, S, du)
        assert np.linalg.norm(dg - dgr) / np.linalg.norm(mag) < tol


@pytest.mark.gpu
@pytest.mark.parametrize("D", [1, 3, 4, 31, 32, 33, 128, 129, BOUND])
def test_entries_feature_sizes(gnn, D):
    _cuda()
    check_entries(gnn, indicator([1, 9, 130, 40, 300, 2], np.random.default_rng(D)), 6, D, seed=D)


@pytest.mark.gpu
@pytest.mark.parametrize("D", [3, 128])
def test_entries_misaligned(gnn, D):
    """pointers off 16 B take the scalar path"""
    _cuda()
    check_entries(gnn, indicator([1, 9, 130, 40]), 4, D, offset=1)


@pytest.mark.gpu
def test_entries_empty_and_one_node_graphs(gnn):
    """graphs without nodes among one-node graphs, a batch of one-node graphs, and a batch with no nodes at all"""
    _cuda()
    check_entries(gnn, indicator([0, 1, 1, 0, 0, 1, 0]), 7, 8)
    check_entries(gnn, indicator([1] * 1000), 1000, 4)
    check_entries(gnn, indicator([]), 3, 4)


@pytest.mark.gpu
@pytest.mark.parametrize("chunk", [32, 128])
@pytest.mark.parametrize("D", [4, 5, 128])
def test_entries_chunk_boundaries(gnn, chunk, D):
    """graphs of C, C + 1, 2C and 2C + 1 nodes, and an empty graph among them"""
    _cuda()
    C_ = chunk
    gi = indicator([C_, C_ + 1, 0, 2 * C_, 2 * C_ + 1, 1, 3])
    check_entries(gnn, gi, 7, D, chunk=chunk)
    check_entries(gnn, gi, 7, D, chunk=chunk, scale=25.0, tol=1e-4)
    check_entries(gnn, gi, 7, D, chunk=chunk, rising=True, tol=1e-4)


@pytest.mark.gpu
def test_entries_unsorted_indicator(gnn):
    _cuda()
    check_entries(gnn, indicator([5, 1, 300, 9, 0, 77], np.random.default_rng(8)), 6, 64)


@pytest.mark.gpu
def test_entries_hundred_thousand_nodes(gnn):
    """one graph of 10^5 nodes (pieces of a long row, combined by the fix-up) beside small ones"""
    _cuda()
    check_entries(gnn, indicator([3, 10 ** 5, 17]), 3, 64, scale=3.0, tol=1e-4)


@pytest.mark.gpu
def test_entries_run_to_run_and_batch_position(gnn):
    """every output bit-identical across calls, including one graph of 10^6 nodes; and a graph of up to a chunk of
    nodes gets the same bits wherever it sits in a batch"""
    _cuda()
    rng = np.random.default_rng(3)
    for gi, G, D in ((indicator([5, 500, 1, 7000, 23]), 5, 128), (np.ones(10 ** 6, np.int64), 1, 64)):
        f = torch.as_tensor(rng.standard_normal((len(gi), D)).astype(np.float32)).cuda()
        gate = torch.as_tensor(rng.standard_normal(len(gi)).astype(np.float32)).cuda()
        du = torch.as_tensor(rng.standard_normal((G, D)).astype(np.float32)).cuda()
        ip = plan_of(gnn, gi, G)
        a = call_entries(gnn, ip, f, gate, du)
        b = call_entries(gnn, ip, f, gate, du)
        assert all(torch.equal(p, q) for p, q in zip(a, b))
    D, n = 36, 100
    fg = torch.as_tensor(rng.standard_normal((n, D)).astype(np.float32)).cuda()
    gg = torch.as_tensor(rng.standard_normal(n).astype(np.float32)).cuda()
    dug = torch.as_tensor(rng.standard_normal((1, D)).astype(np.float32)).cuda()
    outs = []
    for before in (0, 3, 61, 250):
        sizes = [1] * before + [n, 7]
        N, G = sum(sizes), len(sizes)
        f = torch.cat([torch.randn(before, D, device="cuda"), fg, torch.randn(7, D, device="cuda")])
        gate = torch.cat([torch.randn(before, device="cuda"), gg, torch.randn(7, device="cuda")])
        du = torch.cat([torch.randn(before, D, device="cuda"), dug, torch.randn(1, D, device="cuda")])
        u, smax, ssum, dfe, dg = call_entries(gnn, plan_of(gnn, indicator(sizes), G), f, gate, du)
        outs.append((u[before], smax[before], ssum[before], dfe[before:before + n], dg[before:before + n]))
    for o in outs[1:]:
        assert all(torch.equal(p, q) for p, q in zip(outs[0], o))


@pytest.mark.gpu
def test_entry_errors(gnn):
    """the statuses of gnnb_set2set_attend: D out of range, NULL arrays of positive size"""
    _cuda()
    lib = gnn._lib.lib
    ip = plan_of(gnn, indicator([2]), 1)
    z = torch.zeros(2 * (BOUND + 1), device="cuda")
    p = z.data_ptr()
    assert lib.gnnb_attention_pool(ip.plan.h, p, p, BOUND + 1, p, p, p, None) == EUNSUPPORTED
    assert lib.gnnb_attention_pool(ip.plan.h, p, p, 0, p, p, p, None) == ESIZE
    assert lib.gnnb_attention_pool(ip.plan.h, p, p, 4, None, p, p, None) == ESIZE
    assert lib.gnnb_attention_pool(ip.plan.h, p, None, 4, p, p, p, None) == ESIZE
    assert lib.gnnb_attention_pool(None, p, p, 4, p, p, p, None) == EINVAL
    assert lib.gnnb_attention_pool_bwd(ip.plan.h, p, p, p, p, p, p, BOUND + 1, p, p, None) == EUNSUPPORTED
    assert lib.gnnb_attention_pool_bwd(ip.plan.h, p, p, p, p, p, p, 0, p, p, None) == ESIZE
    assert lib.gnnb_attention_pool_bwd(ip.plan.h, p, p, p, p, p, p, 4, p, None, None) == ESIZE
    assert lib.gnnb_attention_pool_bwd(ip.plan.h, p, p, p, p, p, None, 4, p, p, None) == ESIZE
    torch.cuda.synchronize()


@pytest.mark.gpu
def test_nonfinite_gates_match_the_composition(gnn, monkeypatch):
    """gates with +Inf, -Inf everywhere, NaN, and ±1e30 in separate graphs: the fused route gives the composition's IEEE
    results (NaN where it has NaN), and the gradients of the finite graphs agree"""
    _cuda()
    from gnnb200 import readout
    sizes = [6, 5, 7, 4, 8, 9]
    gi = indicator(sizes)
    rng = np.random.default_rng(12)
    D = 16
    fa = rng.standard_normal((D, len(gi))).astype(np.float32)
    ga = rng.standard_normal((1, len(gi))).astype(np.float32)
    off = np.cumsum([0] + sizes)
    ga[0, off[0] + 2] = np.inf                           # graph 1: one +Inf
    ga[0, off[1]:off[2]] = -np.inf                       # graph 2: every gate -Inf
    ga[0, off[2] + 3] = np.nan                           # graph 3: one NaN
    ga[0, off[3]:off[4]] = [1e30, -1e30, 3e38, -3e38]    # graph 4: large values
    ga[0, off[4] + 1] = -np.inf                          # graph 5: one -Inf among finite gates
    outs = []
    for bound in (BOUND, 0):
        monkeypatch.setattr(readout, "_ATTENTION_POOL_MAX_D", bound)
        g = batch_graph(gnn, gi, len(sizes), "cuda")
        f = torch.as_tensor(fa).cuda().requires_grad_(True)
        gate = torch.as_tensor(ga).cuda().requires_grad_(True)
        l = gnn.GlobalAttentionPool(lambda x: gate, lambda x: f)
        u = l(g, f)
        df, dg = torch.autograd.grad(u[:, [3, 4, 5]].sum(), [f, gate])
        outs.append((u.detach().cpu(), df.cpu(), dg.cpu()))
    (u0, df0, dg0), (u1, df1, dg1) = outs
    assert torch.equal(torch.isnan(u0), torch.isnan(u1))
    assert torch.allclose(u0, u1, rtol=1e-6, atol=1e-6, equal_nan=True)
    fin = torch.as_tensor(gi >= 4)
    assert torch.isfinite(df0[:, fin]).all() and torch.isfinite(dg0[:, fin]).all()
    assert torch.allclose(df0[:, fin], df1[:, fin], rtol=1e-5, atol=1e-6)
    assert torch.allclose(dg0[:, fin], dg1[:, fin], rtol=1e-5, atol=1e-6)


@pytest.mark.gpu
def test_molecule_batch(gnn):
    """10 000 graphs of 15-30 nodes, chin = 64, chout = 128: sampled graphs against float64, and finite gradients"""
    _cuda()
    rng = np.random.default_rng(11)
    sizes = rng.integers(15, 31, 10000)
    gi = indicator(sizes)
    g = batch_graph(gnn, gi, len(sizes), "cuda")
    l = pool_layer(gnn, 64, 128, "cuda", seed=2)
    xa = rng.standard_normal((64, len(gi))).astype(np.float32)
    x = torch.as_tensor(xa).cuda().requires_grad_(True)
    y = l(g, x)
    sample = sorted(rng.choice(len(sizes), 40, replace=False).tolist())
    ref = ref_pool(*params64(l), torch.as_tensor(xa, dtype=F64), gi, len(sizes), sample)
    assert rel(y[:, sample], ref) < 2e-5
    y.sum().backward()
    assert torch.isfinite(x.grad).all() and all(torch.isfinite(p.grad).all() for p in l.parameters())
