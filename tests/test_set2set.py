"""Set2Set pooling (graphneuralnetworks.jl_b200/readout.py over csrc/set2set.cu's gnnb_set2set_attend /
gnnb_set2set_attend_bwd; GNNlib/src/layers/pool.jl:29-43, GraphNeuralNetworks/src/layers/pool.jl:126-162).

The contract, stated below:
- the reference (`ref_graph`, float64 torch, one graph at a time with its own LSTM cell): num_iters rounds of
  q = LSTM(qstar);  α = softmax(q' x_g);  r = x_g α;  qstar = [q; r], from qstar = 0 and zero (h, c); a graph without
  nodes has r = 0.  Every column of the LSTM state depends on its own graph only, so graphs are checked one by one;
- the C entries (`entry_fwd` / `entry_bwd`, numpy float64): on a plan (s, t), s_k = <q_{t_k}, x_{s_k}>, the
  per-target softmax statistics, r, and the pullback ds_k = α_k (<dr_{t_k}, x_{s_k}> − <dr_{t_k}, r_{t_k}>),
  dxe_k = α_k dr_{t_k} + ds_k q_{t_k}, dq_i = Σ_k ds_k x_{s_k}.

Back ends of the mirror: `FakeS2S`, the entries restated on host pointers (swapped in over tests/fake_abi.py's double),
and, under -m gpu, the CUDA kernels.  The layer cases run on both routes: the fused attention (the default) and the
broadcast_nodes / softmax_nodes / reduce_nodes composition (the bound patched to 0).
"""
import ctypes as C
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
def entry_fwd(s, t, nd, x, q):
    """r (nd, D), seg_max, seg_sum of gnnb_set2set_attend in float64; x (ns, D), q (nd, D)"""
    x, q = np.asarray(x, np.float64), np.asarray(q, np.float64)
    sc = (q[t] * x[s]).sum(1)
    M = np.full(nd, -np.inf)
    np.maximum.at(M, t, sc)
    ex = np.exp(sc - M[t])
    S = np.zeros(nd)
    np.add.at(S, t, ex)
    r = np.zeros((nd, x.shape[1]))
    np.add.at(r, t, ex[:, None] * x[s])
    return r / np.where(S > 0, S, 1)[:, None], M, S


def entry_bwd(s, t, nd, x, q, r, M, S, dr):
    """dxe (E, D), dq (nd, D) of gnnb_set2set_attend_bwd in float64"""
    x, q, r, dr = (np.asarray(a, np.float64) for a in (x, q, r, dr))
    al = np.exp((q[t] * x[s]).sum(1) - M[t]) / S[t]
    T = (dr * r).sum(1)
    ds = al * ((dr[t] * x[s]).sum(1) - T[t])
    dq = np.zeros_like(q)
    np.add.at(dq, t, ds[:, None] * x[s])
    return al[:, None] * dr[t] + ds[:, None] * q[t], dq


def bwd_magnitudes(s, t, nd, x, q, r, M, S, dr):
    """entry_bwd with every term replaced by its absolute value: the scale of the rounding error of dxe and dq.  With
    sharp logits ds_k = α_k (<dr, x_k> − T) cancels, and dq can be far smaller than its terms."""
    x, q, r, dr = (np.asarray(a, np.float64) for a in (x, q, r, dr))
    al = np.exp((q[t] * x[s]).sum(1) - M[t]) / S[t]
    x, q, r, dr = (np.abs(a) for a in (x, q, r, dr))
    ds = al * ((dr[t] * x[s]).sum(1) + (dr * r).sum(1)[t])
    dq = np.zeros_like(q)
    np.add.at(dq, t, ds[:, None] * x[s])
    return al[:, None] * dr[t] + ds[:, None] * q[t], dq


def _fake_abi():
    sys.path.insert(0, os.path.join(ROOT, "tests"))
    import fake_abi
    return fake_abi


class FakeS2S:
    """gnnb_set2set_attend and gnnb_set2set_attend_bwd on host pointers over `entry_fwd` / `entry_bwd`; every other
    entry is the base double's."""

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

    def gnnb_set2set_attend(self, h, x, q, D, r, smax, ssum, stream):
        self.base.calls.append("gnnb_set2set_attend")
        rc = self._check(D)
        if rc != OK:
            return rc
        p, a = self.base._p(h), self.fa._arr
        rr, M, S = entry_fwd(p.s, p.t, p.nd, a(x, (p.ns, D)), a(q, (p.nd, D)))
        a(r, (p.nd, D))[...] = rr
        a(smax, (p.nd,))[...] = M
        a(ssum, (p.nd,))[...] = S
        return OK

    def gnnb_set2set_attend_bwd(self, h, x, q, r, smax, ssum, dr, D, dxe, dq, stream):
        self.base.calls.append("gnnb_set2set_attend_bwd")
        rc = self._check(D)
        if rc != OK:
            return rc
        p, a = self.base._p(h), self.fa._arr
        de, dqv = entry_bwd(p.s, p.t, p.nd, a(x, (p.ns, D)), a(q, (p.nd, D)), a(r, (p.nd, D)), a(smax, (p.nd,)),
                            a(ssum, (p.nd,)), a(dr, (p.nd, D)))
        a(dxe, (p.E, D))[...] = de
        a(dq, (p.nd, D))[...] = dqv
        return OK


@pytest.fixture(params=["fake", pytest.param("cuda", marks=pytest.mark.gpu)])
def sb(request, gnn):
    """back end of the mirror: .dev, .calls (entries the fake saw, None on cuda), .tol (scale)"""
    if request.param == "fake":
        from gnnb200 import readout
        with _fake_abi().installed() as fake:
            saved = readout.lib
            readout.lib = FakeS2S(fake)
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
    """the default routing, or every feature size through the composition"""
    if request.param == "composed":
        from gnnb200 import readout
        monkeypatch.setattr(readout, "_SET2SET_MAX_D", 0)
    return request.param


# ---------------------------------------------------------------------------------------------- the reference
def ref_lstm(Wi, Wh, b, x, h, c):
    n = Wh.shape[1]
    g = Wi @ x + Wh @ h + b
    i, f, cc, o = g[:n], g[n:2 * n], g[2 * n:3 * n], g[3 * n:]
    c = torch.sigmoid(f) * c + torch.sigmoid(i) * torch.tanh(cc)
    return torch.sigmoid(o) * torch.tanh(c), c


def ref_graph(Wi, Wh, b, xg, n_iters):
    """pool.jl:29-43 for one graph: xg (n_in, nodes of the graph), float64; returns qstar (2 n_in,)"""
    n = xg.shape[0]
    qstar = torch.zeros(2 * n, dtype=F64)
    h, c = torch.zeros(n, dtype=F64), torch.zeros(n, dtype=F64)
    for _ in range(n_iters):
        h, c = ref_lstm(Wi, Wh, b, qstar, h, c)
        if xg.shape[1] == 0:
            r = torch.zeros(n, dtype=F64)
        else:
            r = xg @ torch.softmax(h @ xg, dim=0)
        qstar = torch.cat([h, r])
    return qstar


def ref_pool(Wi, Wh, b, x, gi, G, n_iters, graphs=None):
    """(2 n_in, len(graphs)) for the graphs (0-based ids, all by default) of a batch with 1-based indicator gi"""
    graphs = range(G) if graphs is None else graphs
    return torch.stack([ref_graph(Wi, Wh, b, x[:, torch.as_tensor(gi == k + 1)], n_iters) for k in graphs], dim=1)


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
    gi = np.concatenate([np.full(k, i + 1) for i, k in enumerate(sizes)]).astype(np.int64)
    return gi if rng is None else rng.permutation(gi)


def layer(gnn, n_in, n_iters, dev, seed=0):
    torch.manual_seed(seed)
    l = gnn.Set2Set(n_in, n_iters, device=dev)
    with torch.no_grad():                               # non-zero biases, so that every term of the cell is exercised
        l.lstm.bias.copy_(torch.randn(4 * n_in, generator=torch.Generator().manual_seed(seed)) * 0.3)
    return l


def params64(l):
    return [p.detach().cpu().double().requires_grad_(True) for p in (l.lstm.Wi, l.lstm.Wh, l.lstm.bias)]


def run_case(gnn, sb, sizes, n_in, n_iters, gi=None, G=None, scale=1.0, seed=0, grads=True, fwd_tol=2e-5,
             grad_tol=1e-4):
    rng = np.random.default_rng(seed)
    gi = indicator(sizes) if gi is None else gi
    G = len(sizes) if G is None else G
    N = len(gi)
    xa = (rng.standard_normal((n_in, N)) * scale).astype(np.float32)
    g = batch_graph(gnn, gi, G, sb.dev)
    l = layer(gnn, n_in, n_iters, sb.dev, seed)
    x = torch.as_tensor(xa, device=sb.dev).requires_grad_(True)
    y = l(g, x)
    assert y.shape == (2 * n_in, G) and y.dtype == torch.float32
    Wi, Wh, b = params64(l)
    x64 = torch.as_tensor(xa, dtype=F64).requires_grad_(True)
    ref = ref_pool(Wi, Wh, b, x64, gi, G, n_iters)
    assert rel(y, ref) < fwd_tol * sb.tol, rel(y, ref)
    if grads:
        cot = torch.randn(ref.shape, dtype=F64, generator=torch.Generator().manual_seed(3))
        got = torch.autograd.grad((y.double() * cot.to(y.device)).sum(), [x, l.lstm.Wi, l.lstm.Wh, l.lstm.bias])
        want = torch.autograd.grad((ref * cot).sum(), [x64, Wi, Wh, b])
        for name, a, w in zip(("x", "Wi", "Wh", "bias"), got, want):
            assert rel(a, w) < grad_tol * sb.tol, (name, rel(a, w))
    return y, ref, gi


# ---------------------------------------------------------------------------------------------- the statements
def test_entry_statement_matches_autograd():
    """entry_bwd is the pullback of entry_fwd's r"""
    rng = np.random.default_rng(1)
    s, t, nd, D = np.arange(12), np.array([0] * 5 + [2] * 7), 3, 4
    x, q, dr = rng.standard_normal((12, D)), rng.standard_normal((nd, D)), rng.standard_normal((nd, D))
    r, M, S = entry_fwd(s, t, nd, x, q)
    assert (r[1] == 0).all() and M[1] == -np.inf and S[1] == 0
    dxe, dq = entry_bwd(s, t, nd, x, q, r, M, S, dr)
    xt, qt = torch.tensor(x, requires_grad=True), torch.tensor(q, requires_grad=True)
    rt = torch.zeros(nd, D, dtype=F64)
    for i in (0, 2):
        xs = xt[t == i]
        rt = rt.index_put((torch.tensor(i),), xs.t() @ torch.softmax(xs @ qt[i], 0))
    gx, gq = torch.autograd.grad((rt * torch.tensor(dr)).sum(), [xt, qt])
    assert np.allclose(dxe, gx.numpy()) and np.allclose(dq, gq.numpy())


def test_header_bound_is_the_module_bound(gnn):
    from gnnb200 import readout
    assert readout._SET2SET_MAX_D == BOUND == 1024


def test_lstm_cell_is_flux_lstmcell(gnn):
    """gate order input, forget, cell, output; vector state broadcast over the columns"""
    from gnnb200.layers import _LSTMCell
    torch.manual_seed(0)
    cell = _LSTMCell(6, 3)
    assert cell.Wi.shape == (12, 6) and cell.Wh.shape == (12, 3) and cell.bias.shape == (12,)
    assert (cell.bias == 0).all()
    x, h, c = torch.randn(6, 5), torch.randn(3), torch.randn(3)
    hn, (h2, cn) = cell(x, (h, c))
    Wi, Wh, b = params64(SimpleNamespace(lstm=cell))
    for j in range(5):
        rh, rc = ref_lstm(Wi, Wh, b, x[:, j].double(), h.double(), c.double())
        assert torch.allclose(hn[:, j].double(), rh, atol=1e-6) and torch.allclose(cn[:, j].double(), rc, atol=1e-6)
    assert hn is h2


# ---------------------------------------------------------------------------------------------- the layer
def test_reference_case(gnn, sb, route):
    """GraphNeuralNetworks/test/layers/pool.jl:73-89: 5 graphs of rand_graph(10, 40), n_in = 3, n_iters = 2"""
    y, _, _ = run_case(gnn, sb, [10] * 5, 3, 2)
    assert y.shape == (6, 5)
    if sb.calls is not None:
        n = sb.calls.count("gnnb_set2set_attend")
        assert n == (2 if route == "fused" else 0)


@pytest.mark.parametrize("n_in", [1, 3, 4, 32, 128])
@pytest.mark.parametrize("n_iters", [1, 3])
def test_forward_and_gradients(gnn, sb, route, n_in, n_iters):
    run_case(gnn, sb, [1, 7, 1, 40, 150, 3], n_in, n_iters, seed=n_in + n_iters)


def test_graph_without_nodes(gnn, sb, route):
    """graph 3 of 5 has no nodes: its r is exactly 0"""
    gi = indicator([4, 6])
    gi = np.concatenate([gi, np.full(5, 4), np.full(2, 5)])
    y, _, _ = run_case(gnn, sb, None, 8, 2, gi=gi, G=5)
    assert (y[8:, 2] == 0).all()


def test_graph_ids_beyond_the_last_node(gnn, sb, route):
    """num_graphs larger than every id the indicator uses"""
    y, _, _ = run_case(gnn, sb, None, 4, 2, gi=indicator([5, 3]), G=4)
    assert (y[4:, 2:] == 0).all()


def test_unsorted_indicator(gnn, sb, route):
    run_case(gnn, sb, None, 16, 3, gi=indicator([5, 1, 30, 9], np.random.default_rng(4)), G=4)


def test_one_graph(gnn, sb, route):
    run_case(gnn, sb, [300], 12, 2)


def test_routes_agree(gnn, sb, monkeypatch):
    """the fused attention against the composition on the same inputs, forward and every gradient"""
    from gnnb200 import readout
    rng = np.random.default_rng(5)
    gi = indicator([3, 50, 1, 200, 17], rng)
    xa = rng.standard_normal((20, len(gi))).astype(np.float32)
    outs = []
    for bound in (BOUND, 0):
        monkeypatch.setattr(readout, "_SET2SET_MAX_D", bound)
        g = batch_graph(gnn, gi, 5, sb.dev)
        l = layer(gnn, 20, 3, sb.dev, seed=9)
        x = torch.as_tensor(xa, device=sb.dev).requires_grad_(True)
        y = l(g, x)
        cot = torch.randn(y.shape, generator=torch.Generator().manual_seed(2)).to(sb.dev)
        outs.append([y] + list(torch.autograd.grad((y * cot).sum(), [x, l.lstm.Wi, l.lstm.Wh, l.lstm.bias])))
    for a, b in zip(*outs):
        assert rel(a, b) < 2e-5 * sb.tol


def test_argument_errors(gnn, sb):
    gi = indicator([3, 4])
    g = batch_graph(gnn, gi, 2, sb.dev)
    l = gnn.Set2Set(5, 2, device=sb.dev)
    with pytest.raises(AssertionError):
        l(g, torch.zeros(5, 6, device=sb.dev))           # 6 columns, 7 nodes
    with pytest.raises(AssertionError):
        l(g, torch.zeros(4, 7, device=sb.dev))           # 4 rows, n_in = 5
    with pytest.raises(AssertionError):
        gnn.Set2Set(5, 2, 2)


def test_exported(gnn):
    assert gnn.set2set_pool is gnn.readout.set2set_pool and issubclass(gnn.Set2Set, torch.nn.Module)


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


def call_entries(gnn, ip, x, q, dr, offset=0):
    """the two entries on cuda arrays x (N, D), q (G, D), dr (G, D); offset > 0 places every array that many floats into
    its buffer (misaligned for the scalar path)"""
    lib, chk = gnn._lib.lib, gnn._lib.check
    N, D = x.shape
    G = q.shape[0]

    def buf(shape, src=None):
        b = torch.zeros(int(np.prod(shape)) + offset, dtype=torch.float32, device="cuda")
        v = b[offset:].view(shape)
        if src is not None:
            v.copy_(src)
        return v
    x, q, dr = buf((N, D), x), buf((G, D), q), buf((G, D), dr)
    r, dq, dxe = buf((G, D)), buf((G, D)), buf((N, D))
    smax, ssum = buf((G,)), buf((G,))
    st = torch.cuda.current_stream().cuda_stream
    chk(lib.gnnb_set2set_attend(ip.plan.h, x.data_ptr(), q.data_ptr(), D, r.data_ptr(), smax.data_ptr(),
                                ssum.data_ptr(), st))
    chk(lib.gnnb_set2set_attend_bwd(ip.plan.h, x.data_ptr(), q.data_ptr(), r.data_ptr(), smax.data_ptr(),
                                    ssum.data_ptr(), dr.data_ptr(), D, dxe.data_ptr(), dq.data_ptr(), st))
    torch.cuda.synchronize()
    return r, smax, ssum, dxe, dq


def check_entries(gnn, gi, G, D, chunk=None, scale=1.0, rising=False, offset=0, seed=0, tol=2e-5):
    rng = np.random.default_rng(seed)
    N = len(gi)
    x = rng.standard_normal((N, D)) * scale
    q = rng.standard_normal((G, D))
    if rising:                                           # s_k increases along each graph: the max moves at every node
        q = np.abs(q)
        x = np.abs(x) * (1 + np.arange(N))[:, None] / N * 8
    x, q = x.astype(np.float32), q.astype(np.float32)
    dr = rng.standard_normal((G, D)).astype(np.float32)
    ip = plan_of(gnn, gi, G, chunk)
    r, smax, ssum, dxe, dq = (a.cpu().numpy().astype(np.float64)
                              for a in call_entries(gnn, ip, torch.as_tensor(x).cuda(), torch.as_tensor(q).cuda(),
                                                    torch.as_tensor(dr).cuda(), offset))
    s, t = np.arange(N), gi - 1
    rr, M, S = entry_fwd(s, t, G, x, q)
    de, dqr = entry_bwd(s, t, G, x, q, rr, M, S, dr)
    de_mag, dq_mag = bwd_magnitudes(s, t, G, x, q, rr, M, S, dr)
    has = S > 0
    assert (r[~has] == 0).all() and (smax[~has] == -np.inf).all() and (ssum[~has] == 0).all()
    assert (dq[~has] == 0).all()
    assert rel(torch.as_tensor(r), torch.as_tensor(rr)) < tol
    for name, a, b, mag in (("dxe", dxe, de, de_mag), ("dq", dq, dqr, dq_mag)):
        err = np.linalg.norm(a - b) / np.linalg.norm(mag)
        assert err < tol, (name, err)
    assert np.allclose(smax[has], M[has], rtol=1e-5, atol=1e-5 * np.abs(M[has]).max())
    assert np.allclose(ssum[has], S[has], rtol=1e-4)


@pytest.mark.gpu
@pytest.mark.parametrize("D", [1, 3, 4, 5, 32, 128, 132, 512, 1024])
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
def test_entries_run_to_run(gnn):
    """every output bit-identical across calls, including one graph of 10^6 nodes"""
    _cuda()
    rng = np.random.default_rng(3)
    for gi, G, D in ((indicator([5, 500, 1, 7000, 23]), 5, 128), (np.ones(10 ** 6, np.int64), 1, 64)):
        x = torch.as_tensor(rng.standard_normal((len(gi), D)).astype(np.float32)).cuda()
        q = torch.as_tensor(rng.standard_normal((G, D)).astype(np.float32)).cuda() * 0.2
        dr = torch.as_tensor(rng.standard_normal((G, D)).astype(np.float32)).cuda()
        ip = plan_of(gnn, gi, G)
        a = call_entries(gnn, ip, x, q, dr)
        b = call_entries(gnn, ip, x, q, dr)
        assert all(torch.equal(u, v) for u, v in zip(a, b))


@pytest.mark.gpu
def test_molecule_batch(gnn):
    """10 000 graphs of 15-30 nodes, D = 128: sampled graphs against float64"""
    _cuda()
    rng = np.random.default_rng(11)
    sizes = rng.integers(15, 31, 10000)
    gi = indicator(sizes)
    g = batch_graph(gnn, gi, len(sizes), "cuda")
    l = layer(gnn, 128, 3, "cuda", seed=2)
    xa = rng.standard_normal((128, len(gi))).astype(np.float32)
    x = torch.as_tensor(xa).cuda().requires_grad_(True)
    y = l(g, x)
    sample = sorted(rng.choice(len(sizes), 40, replace=False).tolist())
    Wi, Wh, b = params64(l)
    ref = ref_pool(Wi, Wh, b, torch.as_tensor(xa, dtype=F64), gi, len(sizes), 3, sample)
    assert rel(y[:, sample], ref) < 8e-5
    y.sum().backward()
    assert torch.isfinite(x.grad).all()


@pytest.mark.gpu
def test_ten_million_nodes(gnn):
    """one graph of 10^7 nodes, D = 128 (the long-row path): r against float64"""
    _cuda()
    N, D = 10 ** 7, 128
    gen = torch.Generator(device="cuda").manual_seed(0)
    x = torch.randn((N, D), device="cuda", generator=gen)
    q = torch.randn((1, D), device="cuda", generator=gen) * 0.1
    ip = plan_of(gnn, np.ones(N, np.int64), 1)
    r = torch.empty((1, D), device="cuda")
    smax, ssum = torch.empty(1, device="cuda"), torch.empty(1, device="cuda")
    gnn._lib.check(gnn._lib.lib.gnnb_set2set_attend(ip.plan.h, x.data_ptr(), q.data_ptr(), D, r.data_ptr(),
                                                    smax.data_ptr(), ssum.data_ptr(),
                                                    torch.cuda.current_stream().cuda_stream))
    s = (x.double() @ q.double().t()).squeeze(1)
    a = torch.softmax(s, 0)
    ref = (a[:, None] * x.double()).sum(0)
    assert rel(r[0], ref) < 1e-4
    assert float(smax) == float(s.max().float())


@pytest.mark.gpu
def test_above_the_bound_composes(gnn):
    """D = 1025 takes the composition and matches float64; the entry itself refuses it"""
    _cuda()
    sb = SimpleNamespace(dev=torch.device("cuda"), calls=None, tol=4.0)
    run_case(gnn, sb, [3, 40, 1], 1025, 2, grads=False)
    ip = plan_of(gnn, indicator([2]), 1)
    z = torch.zeros(1025 * 2, device="cuda")
    rc = gnn._lib.lib.gnnb_set2set_attend(ip.plan.h, z.data_ptr(), z.data_ptr(), 1025, z.data_ptr(), z.data_ptr(),
                                          z.data_ptr(), None)
    assert rc == EUNSUPPORTED
    assert gnn._lib.lib.gnnb_set2set_attend(ip.plan.h, z.data_ptr(), z.data_ptr(), 0, z.data_ptr(), z.data_ptr(),
                                            z.data_ptr(), None) == ESIZE
    assert gnn._lib.lib.gnnb_set2set_attend(ip.plan.h, z.data_ptr(), z.data_ptr(), 4, None, z.data_ptr(),
                                            z.data_ptr(), None) == ESIZE
