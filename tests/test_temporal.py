"""Recurrent temporal graph layers (graphneuralnetworks.jl_b200/temporal.py over csrc/recurrent.cu's gate entries;
GraphNeuralNetworks/src/layers/temporalconv.jl).

The contract, stated below:
- the entries (`gru_rz` … `lstm_cell_bwd`): their formulas in float64, written once for numpy and torch arrays;
- the cells (`ref_step`): the reference cells statement for statement in float64, each gate computed separately, on
  right-multiplication operators built from the graph (L̃, DConv's two diffusion operators, the self-looped GCN
  adjacency) — dense matrices on the host, sparse ones for the large GPU cases.

Back ends of the mirror: `FakeRec`, the entries restated on host pointers (swapped in over tests/fake_abi.py's double),
and, under -m gpu, the CUDA kernels.
"""
import os
import sys
from types import SimpleNamespace

import numpy as np
import pytest
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
OK, EINVAL, ESIZE, ECUDA, ENOMEM, EUNSUPPORTED, EINDEX = range(7)
F64 = torch.float64
CELLS = ["gconvgru", "gconvlstm", "dcgru", "tgcn", "evolvegcno"]


# ---------------------------------------------------------------------------------------------- the entries, float64
def _exp(a):
    return np.exp(a) if isinstance(a, np.ndarray) else torch.exp(a)


def _tanh(a):
    return np.tanh(a) if isinstance(a, np.ndarray) else torch.tanh(a)


def _sig(a):
    return 1.0 / (1.0 + _exp(-a))


def gru_rz(px, ah, h):
    """px (N, 3D) [r | z | n], ah (N, 2D), h (N, D) -> r, z, rh"""
    D = h.shape[1]
    r = _sig(px[:, :D] + ah[:, :D])
    z = _sig(px[:, D:2 * D] + ah[:, D:])
    return r, z, r * h


def gru_out(px, ah_n, h, z, blend):
    D = h.shape[1]
    n = _tanh(px[:, 2 * D:3 * D] + ah_n)
    return n, ((1 - z) * n + z * h) if blend == 0 else ((1 - z) * h + z * n)


def gru_out_bwd(dhn, h, z, n, blend):
    """-> dpre_n, dz, dh"""
    if blend == 0:
        return dhn * (1 - z) * (1 - n * n), dhn * (h - n), dhn * z
    return dhn * z * (1 - n * n), dhn * (n - h), dhn * (1 - z)


def gru_rz_bwd(drh, dz, h, r, z, dh):
    """-> dpre_rz (N, 2D), dh + drh ⊙ r"""
    cat = np.concatenate if isinstance(h, np.ndarray) else torch.cat
    return cat([drh * h * r * (1 - r), dz * z * (1 - z)], 1), dh + drh * r


def lstm_cell(px, ah, c, w):
    """px (N, 4D) [i | f | c | o], ah (N, 4D), c (N, D), w (4D,) or None -> gates [i | f | g | o], c', h'"""
    D = c.shape[1]
    a = px[:, :4 * D] + ah
    wv = [0.0] * 4 if w is None else [w[q * D:(q + 1) * D] for q in range(4)]
    i = _sig(a[:, :D] + wv[0] * c)
    f = _sig(a[:, D:2 * D] + wv[1] * c)
    g = _tanh(a[:, 2 * D:3 * D] + wv[2] * c)
    cn = f * c + i * g
    o = _sig(a[:, 3 * D:] + wv[3] * cn)
    cat = np.concatenate if isinstance(c, np.ndarray) else torch.cat
    return cat([i, f, g, o], 1), cn, o * _tanh(cn)


def lstm_cell_bwd(dhn, dcn, c, gates, cn, w):
    """-> dpre (N, 4D), dc, dw (4D,) or None"""
    D = c.shape[1]
    i, f, g, o = (gates[:, q * D:(q + 1) * D] for q in range(4))
    wv = [0.0] * 4 if w is None else [w[q * D:(q + 1) * D] for q in range(4)]
    tc = _tanh(cn)
    do = dhn * tc * o * (1 - o)
    dct = dcn + dhn * o * (1 - tc * tc) + do * wv[3]
    di = dct * g * i * (1 - i)
    df = dct * c * f * (1 - f)
    dg = dct * i * (1 - g * g)
    dc = dct * f + di * wv[0] + df * wv[1] + dg * wv[2]
    cat = np.concatenate if isinstance(c, np.ndarray) else torch.cat
    dw = None if w is None else cat([(di * c).sum(0), (df * c).sum(0), (dg * c).sum(0), (do * cn).sum(0)])
    return cat([di, df, dg, do], 1), dc, dw


# ---------------------------------------------------------------------------------------------- the entries on pointers
def _fake_abi():
    sys.path.insert(0, os.path.join(ROOT, "tests"))
    import fake_abi
    return fake_abi


def _slots(N):
    return (N + 63) // 64 if N < 65536 else 1024


class FakeRec:
    """the six gate entries on host pointers over the statements above; every other entry is the base double's"""

    def __init__(self, base):
        self.base, self.fa = base, _fake_abi()

    def __getattr__(self, name):
        return getattr(self.base, name)

    def _sizes(self, N, D, ld, G):
        if N < 0 or D < 1 or ld < G * D:
            self.base._err = b"bad sizes"
            return ESIZE
        return OK

    def _rows(self, p, N, W, ld=None):
        """(N, W) float64 copy of rows at stride ld"""
        ld = W if ld is None else ld
        if N == 0:
            return np.zeros((0, W))
        a = self.fa._arr(p, ((N - 1) * ld + W,))
        return np.lib.stride_tricks.as_strided(a, (N, W), (ld * 4, 4)).astype(np.float64)

    def _put(self, p, v, ld=None):
        N, W = v.shape
        ld = W if ld is None else ld
        if N == 0:
            return
        a = self.fa._arr(p, ((N - 1) * ld + W,))
        np.lib.stride_tricks.as_strided(a, (N, W), (ld * 4, 4))[...] = v

    def gnnb_gru_rz(self, px, ld, ah, h, N, D, r, z, rh, st):
        self.base.calls.append("gnnb_gru_rz")
        rc = self._sizes(N, D, ld, 3)
        if rc != OK or N == 0:
            return rc
        out = gru_rz(self._rows(px, N, 3 * D, ld), self._rows(ah, N, 2 * D), self._rows(h, N, D))
        for p, v in zip((r, z, rh), out):
            self._put(p, v)
        return OK

    def gnnb_gru_out(self, px, ld, ah, h, z, N, D, blend, n, hn, st):
        self.base.calls.append("gnnb_gru_out")
        rc = self._sizes(N, D, ld, 3)
        if rc != OK or N == 0:
            return rc
        nv, hv = gru_out(self._rows(px, N, 3 * D, ld), self._rows(ah, N, D), self._rows(h, N, D),
                         self._rows(z, N, D), blend)
        self._put(n, nv)
        self._put(hn, hv)
        return OK

    def gnnb_gru_out_bwd(self, dhn, h, z, n, N, D, blend, dpre, ld, dz, dh, st):
        self.base.calls.append("gnnb_gru_out_bwd")
        rc = self._sizes(N, D, ld, 1)
        if rc != OK or N == 0:
            return rc
        a, b, c = gru_out_bwd(*(self._rows(p, N, D) for p in (dhn, h, z, n)), blend)
        self._put(dpre, a, ld)
        self._put(dz, b)
        self._put(dh, c)
        return OK

    def gnnb_gru_rz_bwd(self, drh, dz, h, r, z, N, D, dpre, ld, dh, st):
        self.base.calls.append("gnnb_gru_rz_bwd")
        rc = self._sizes(N, D, ld, 2)
        if rc != OK or N == 0:
            return rc
        a, b = gru_rz_bwd(*(self._rows(p, N, D) for p in (drh, dz, h, r, z, dh)))
        self._put(dpre, a, ld)
        self._put(dh, b)
        return OK

    def gnnb_lstm_cell(self, px, ld, ah, c, w, N, D, gates, cn, hn, st):
        self.base.calls.append("gnnb_lstm_cell")
        rc = self._sizes(N, D, ld, 4)
        if rc != OK or N == 0:
            return rc
        wv = None if w is None else self.fa._arr(w, (4 * D,)).astype(np.float64)
        gv, cv, hv = lstm_cell(self._rows(px, N, 4 * D, ld), self._rows(ah, N, 4 * D), self._rows(c, N, D), wv)
        self._put(gates, gv)
        self._put(cn, cv)
        self._put(hn, hv)
        return OK

    def gnnb_lstm_cell_bwd(self, dhn, dcn, c, gates, cn, w, N, D, dpre, dc, dw, ws, st):
        self.base.calls.append("gnnb_lstm_cell_bwd")
        rc = self._sizes(N, D, D, 1)
        if rc != OK:
            return rc
        if N == 0:
            if dw is not None:
                self.fa._arr(dw, (4 * D,))[...] = 0
            return OK
        wv = None if w is None else self.fa._arr(w, (4 * D,)).astype(np.float64)
        a, b, dwv = lstm_cell_bwd(self._rows(dhn, N, D), self._rows(dcn, N, D), self._rows(c, N, D),
                                  self._rows(gates, N, 4 * D), self._rows(cn, N, D), wv)
        self._put(dpre, a)
        self._put(dc, b)
        if dw is not None:
            self.fa._arr(dw, (4 * D,))[...] = dwv
        return OK


@pytest.fixture(params=["fake", pytest.param("cuda", marks=pytest.mark.gpu)])
def tb(request, gnn):
    """back end of the mirror: .dev, .calls (entries the fake saw, None on cuda)"""
    if request.param == "fake":
        from gnnb200 import temporal
        with _fake_abi().installed() as fake:
            saved = temporal.lib
            temporal.lib = FakeRec(fake)
            try:
                yield SimpleNamespace(dev=torch.device("cpu"), calls=fake.calls)
            finally:
                temporal.lib = saved
    else:
        if not torch.cuda.is_available():
            pytest.skip("no CUDA device")
        yield SimpleNamespace(dev=torch.device("cuda"), calls=None)


# ---------------------------------------------------------------------------------------------- graphs and operators
def ring_graph(n, extra, seed):
    """a bidirected ring (every node has in- and out-edges) plus `extra` random edges; 1-based (s, t)"""
    rng = np.random.default_rng(seed)
    i = np.arange(n)
    s = np.concatenate([i, (i + 1) % n, rng.integers(0, n, extra)]) + 1
    t = np.concatenate([(i + 1) % n, i, rng.integers(0, n, extra)]) + 1
    return s, t


class Ops:
    """the right-multiplications the reference cells apply to (D, N) float64 arrays: X L̃, DConv's X·diag(d)·A and
    X·diag(d)·Aᵀ, and the self-looped GCN X Â.  Dense on the host, sparse on the device for large graphs."""

    def __init__(self, s, t, n, lmax, dev, sparse=False):
        s0, t0 = torch.as_tensor(s - 1), torch.as_tensor(t - 1)
        self.n, self.dev, self.sparse = n, dev, sparse
        ones = torch.ones(len(s0), dtype=F64)
        A = self._mat(s0, t0, ones)                               # A[s, t] = edge count
        dout = torch.zeros(n, dtype=F64).index_add_(0, s0, ones)
        din = torch.zeros(n, dtype=F64).index_add_(0, t0, ones)
        c = 1 / torch.sqrt(dout)
        self.lmax = lmax
        self.Ahat = self._mat(s0, t0, c[s0] * c[t0])              # D^-1/2 A D^-1/2 (out-degree), cheb_conv's
        self.A, self.At = A, self._mat(t0, s0, ones)
        self.dout, self.din = dout.to(dev), din.to(dev)
        loops = torch.arange(n)
        sl, tl = torch.cat([s0, loops]), torch.cat([t0, loops])
        dl = torch.zeros(n, dtype=F64).index_add_(0, tl, torch.ones(len(tl), dtype=F64))
        cg = 1 / torch.sqrt(dl)
        self.G = self._mat(sl, tl, cg[sl] * cg[tl])

    def _mat(self, r, c, v):
        M = torch.sparse_coo_tensor(torch.stack([r, c]), v, (self.n, self.n), check_invariants=True).coalesce()
        return M.to(self.dev) if self.sparse else M.to_dense().to(self.dev)

    def mul(self, X, M):
        return (M.t() @ X.t()).t() if self.sparse else X @ M

    def L(self, X):
        return (2.0 / self.lmax) * (X - self.mul(X, self.Ahat)) - X

    def dc_out(self, X):
        return self.mul(X * self.dout, self.A)

    def dc_in(self, X):
        return self.mul(X * self.din, self.At)

    def gcn(self, X):
        return self.mul(X, self.G)


# ---------------------------------------------------------------------------------------------- the reference cells
def r_cheb(P, name, ops, X):
    W, b = P[f"{name}.weight"], P.get(f"{name}.bias")
    Z = [X, ops.L(X)]
    for _ in range(2, W.shape[2]):
        Z.append(2 * ops.L(Z[-1]) - Z[-2])
    Y = sum(W[:, :, k] @ Z[k] for k in range(W.shape[2]))
    return Y if b is None else Y + b.reshape(-1, 1)


def r_dconv(P, name, ops, x):
    W, b = P[f"{name}.weights"], P.get(f"{name}.bias")
    k = W.shape[1]
    h = W[0, 0] @ x + W[1, 0] @ x
    T0 = x
    if k > 1:
        T1_out, T1_in = ops.dc_out(T0), ops.dc_in(T0)
        h = h + W[0, 1] @ T1_in + W[1, 1] @ T1_out
    for i in range(2, k + 1):
        T2_in = 2 * ops.dc_in(T1_in) - T0
        T2_out = 2 * ops.dc_out(T1_out) - T0
        h = h + W[0, i - 1] @ T2_in + W[1, i - 1] @ T2_out
        T1_in, T1_out = T2_in, T2_out
    return h if b is None else h + b.reshape(-1, 1)


def r_gcn(P, name, ops, x, act=lambda v: v, W=None):
    W = P[f"{name}.weight"] if W is None else W
    b = P.get(f"{name}.bias")
    y = W @ ops.gcn(x)
    return act(y if b is None else y + b.reshape(-1, 1))


def r_dense(P, name, x, act):
    return act(P[f"{name}.weight"] @ x + P[f"{name}.bias"].reshape(-1, 1))


def ref_step(kind, P, ops, x, state):
    """one step of the reference cell (temporalconv.jl), float64, each gate on its own -> (y, state)"""
    sg = torch.sigmoid
    if kind == "gconvgru":
        h = state
        r = sg(r_cheb(P, "conv_x_r", ops, x) + r_cheb(P, "conv_h_r", ops, h))
        z = sg(r_cheb(P, "conv_x_z", ops, x) + r_cheb(P, "conv_h_z", ops, h))
        ht = torch.tanh(r_cheb(P, "conv_x_h", ops, x) + r_cheb(P, "conv_h_h", ops, r * h))
        h = (1 - z) * ht + z * h
        return h, h
    if kind == "gconvlstm":
        h, c = state
        i = sg(r_cheb(P, "conv_x_i", ops, x) + r_cheb(P, "conv_h_i", ops, h) + P["w_i"] * c + P["b_i"].reshape(-1, 1))
        f = sg(r_cheb(P, "conv_x_f", ops, x) + r_cheb(P, "conv_h_f", ops, h) + P["w_f"] * c + P["b_f"].reshape(-1, 1))
        c = f * c + i * torch.tanh(r_cheb(P, "conv_x_c", ops, x) + r_cheb(P, "conv_h_c", ops, h) + P["w_c"] * c
                                   + P["b_c"].reshape(-1, 1))
        o = sg(r_cheb(P, "conv_x_o", ops, x) + r_cheb(P, "conv_h_o", ops, h) + P["w_o"] * c + P["b_o"].reshape(-1, 1))
        h = o * torch.tanh(c)
        return h, (h, c)
    if kind == "dcgru":
        h = state
        ht = torch.cat([x, h])
        z = sg(r_dconv(P, "dconv_u", ops, ht))
        r = sg(r_dconv(P, "dconv_r", ops, ht))
        c = torch.tanh(r_dconv(P, "dconv_c", ops, torch.cat([x, h * r])))
        h = z * h + (1 - z) * c
        return h, h
    if kind == "tgcn":
        h = state

        def chain(q):
            return r_gcn(P, f"conv_{q}.1", ops, r_gcn(P, f"conv_{q}.0", ops, x, torch.relu))
        z = r_dense(P, "dense_z", torch.cat([chain("z"), h]), sg)
        r = r_dense(P, "dense_r", torch.cat([chain("r"), h]), sg)
        ht = r_dense(P, "dense_h", torch.cat([chain("h"), r * h]), torch.tanh)
        h = (1 - z) * h + z * ht
        return h, h
    if kind == "evolvegcno":
        wv, (hl, cl) = state
        n = hl.shape[0]
        g = P["lstm.Wi"] @ wv + P["lstm.Wh"] @ hl + P["lstm.bias"]
        cl = sg(g[n:2 * n]) * cl + sg(g[:n]) * torch.tanh(g[2 * n:3 * n])
        hl = sg(g[3 * n:]) * torch.tanh(cl)
        I, O = P["conv.weight"].shape[1], P["conv.weight"].shape[0]
        W = hl.reshape(I, O).t()
        return r_gcn(P, "conv", ops, x, W=W), (hl, (hl, cl))
    raise ValueError(kind)


def ref_init(kind, P, out, N, state_kind, S):
    """the reference's initial state for state_kind in {none, vector, matrix}; S: the float64 state values"""
    if kind == "evolvegcno":
        io = P["lstm.Wh"].shape[1]
        return (P["conv.weight"].t().reshape(-1), (torch.zeros(io, dtype=F64), torch.zeros(io, dtype=F64)))

    def rep(v):
        return v.reshape(-1, 1).expand(out, N) if v.dim() == 1 else v
    if kind == "gconvlstm":
        if state_kind == "none":
            return (torch.zeros(out, N, dtype=F64), torch.zeros(out, N, dtype=F64))
        return (rep(S[0]), rep(S[1]))
    if state_kind == "none":
        return torch.zeros(out, N, dtype=F64)
    return rep(S)


# ---------------------------------------------------------------------------------------------- building the cases
def dconv_scale(s, t, k):
    """DConv diffuses with the unnormalised degree (conv.jl:705-716): each diffusion step multiplies by up to deg²,
    so its order-k term grows like deg^2k and DCGRU's recurrence has a gain of about deg^2k |W| per time step.  With
    glorot weights that is far above 1 on most graphs: the cell is chaotic and any rounding grows to O(1) within a few
    steps, in the reference as here.  The DConv weights of the DCGRU cases are scaled by 0.5 / max_degree^2k to keep
    the recurrence contractive."""
    deg = max(np.bincount(np.asarray(s)).max(), np.bincount(np.asarray(t)).max())
    return 0.5 / float(deg) ** (2 * k)


def make_layer(gnn, kind, nin, out, k, dev, seed=0, dscale=0.02):
    torch.manual_seed(seed)
    if kind == "gconvgru":
        cell = gnn.GConvGRUCell(nin, out, k, device=dev)
    elif kind == "gconvlstm":
        cell = gnn.GConvLSTMCell(nin, out, k, device=dev)
    elif kind == "dcgru":
        cell = gnn.DCGRUCell(nin, out, k, device=dev)
    elif kind == "tgcn":
        cell = gnn.TGCNCell(nin, out, device=dev)
    else:
        cell = gnn.EvolveGCNOCell(nin, out, device=dev)
    with torch.no_grad():                                     # non-zero biases, so that the folds are exercised
        for name, p in cell.named_parameters():
            if name.endswith("bias") or name.split(".")[-1].startswith("b_"):
                p.copy_(torch.randn_like(p) * 0.3)
            elif kind == "dcgru":                            # see dconv_scale
                p.mul_(dscale)
    return cell


def rel(a, b):
    a, b = a.detach().double().cpu(), b.detach().double().cpu()
    return float((a - b).norm() / max(float(b.norm()), 1e-30))


def make_state(gnn, kind, out, N, state_kind, dev, seed):
    """(the mirror's state argument with requires_grad, its float64 copies)"""
    if kind == "evolvegcno" or state_kind == "none":
        return None, None
    g = torch.Generator().manual_seed(seed)
    shape = (out,) if state_kind == "vector" else (out, N)
    mk = lambda: (torch.randn(*shape, generator=g) * 0.5)
    if kind == "gconvlstm":
        h, c = mk(), mk()
        h, c = h.double().float(), c.double().float()
        hs = gnn.colmajor(h.to(dev).clone()).requires_grad_(True)
        cs = gnn.colmajor(c.to(dev).clone()).requires_grad_(True)
        return (hs, cs), (h.double().requires_grad_(True), c.double().requires_grad_(True))
    h = mk()
    h64 = h.double().requires_grad_(True)
    hs = gnn.colmajor(h.to(dev).clone()).requires_grad_(True)
    return hs, h64


def run_case(gnn, tb, kind, nin, out, N, T, k=2, state_kind="none", seed=0, extra=None, step=False,
             fwd_tol=1e-5, grad_tol=1e-4):
    """the layer (or one cell step) against the float64 reference: y and the gradients of x, state and every parameter"""
    dev = tb.dev
    s, t = ring_graph(N, N if extra is None else extra, seed)
    g = gnn.GNNGraph(torch.as_tensor(s).to(dev), torch.as_tensor(t).to(dev), num_nodes=N)
    cell = make_layer(gnn, kind, nin, out, k, dev, seed, dconv_scale(s, t, k))
    gen = torch.Generator().manual_seed(seed + 1)
    x = torch.randn(nin, T, N, generator=gen)
    xs = gnn.colmajor(x.to(dev)).requires_grad_(True)
    st, st64 = make_state(gnn, kind, out, N, state_kind, dev, seed + 2)
    if step:
        y, _ = cell(g, xs[:, 0], st)
        y = y.unsqueeze(1)
    else:
        y = gnn.GNNRecurrence(cell)(g, xs, st)
    assert tuple(y.shape) == (out, T, N)
    R = torch.randn(out, T, N, generator=gen)
    (y * R.to(dev)).sum().backward()

    lmax = getattr(g, "_lmax_cache", None) or 1.0
    ops = Ops(s, t, N, lmax, torch.device("cpu"))
    P = {n: p.detach().double().cpu().requires_grad_(True) for n, p in cell.named_parameters()}
    x64 = x.double().requires_grad_(True)
    state = ref_init(kind, P, out, N, state_kind, st64)
    ys = []
    for tt in range(T):
        yt, state = ref_step(kind, P, ops, x64[:, tt], state)
        ys.append(yt)
    y64 = torch.stack(ys, 1)
    (y64 * R.double()).sum().backward()
    assert rel(y, y64) < fwd_tol, f"{kind} forward {rel(y, y64):.2e}"
    assert rel(xs.grad, x64.grad) < grad_tol, f"{kind} dx {rel(xs.grad, x64.grad):.2e}"
    if st is not None:
        for a, b in zip(st if isinstance(st, tuple) else (st,), st64 if isinstance(st64, tuple) else (st64,)):
            assert rel(a.grad, b.grad) < grad_tol, f"{kind} dstate {rel(a.grad, b.grad):.2e}"
    for n, p in cell.named_parameters():
        gp = P[n].grad if P[n].grad is not None else torch.zeros_like(P[n])
        got = p.grad if p.grad is not None else torch.zeros_like(p)
        if float(gp.norm()) == 0:
            assert float(got.norm()) == 0, f"{kind} d{n} should be 0"
        else:
            assert rel(got, gp) < grad_tol, f"{kind} d{n} {rel(got, gp):.2e}"
    return y, xs.grad, cell


# ---------------------------------------------------------------------------------------------- CPU: the statements
@pytest.mark.parametrize("blend", [0, 1])
def test_gru_statements_match_autograd(blend):
    rng = np.random.default_rng(0)
    N, D = 7, 5
    px, ah, h = rng.standard_normal((N, 3 * D)), rng.standard_normal((N, 2 * D)), rng.standard_normal((N, D))
    ahn, dhn = rng.standard_normal((N, D)), rng.standard_normal((N, D))
    T = [torch.tensor(a, requires_grad=True) for a in (px, ah, h, ahn)]
    r, z, rh = gru_rz(T[0], T[1], T[2])
    drh = torch.tensor(rng.standard_normal((N, D)))
    n, hn = gru_out(T[0], T[3], T[2], z, blend)
    ((hn * torch.tensor(dhn)).sum() + (rh * drh).sum()).backward()
    rn, zn, rhn = gru_rz(px, ah, h)
    nn_, hnn = gru_out(px, ahn, h, zn, blend)
    assert np.allclose(hnn, hn.detach().numpy()) and np.allclose(rhn, rh.detach().numpy())
    dpre_n, dz, dh = gru_out_bwd(dhn, h, zn, nn_, blend)
    dpre_rz, dh = gru_rz_bwd(drh.numpy(), dz, h, rn, zn, dh)
    assert np.allclose(np.concatenate([dpre_rz, dpre_n], 1), T[0].grad.numpy())
    assert np.allclose(dpre_rz, T[1].grad.numpy()) and np.allclose(dpre_n, T[3].grad.numpy())
    assert np.allclose(dh, T[2].grad.numpy())


@pytest.mark.parametrize("peep", [True, False])
def test_lstm_statements_match_autograd(peep):
    rng = np.random.default_rng(1)
    N, D = 6, 3
    px, ah, c = rng.standard_normal((N, 4 * D)), rng.standard_normal((N, 4 * D)), rng.standard_normal((N, D))
    w = rng.standard_normal(4 * D) if peep else None
    T = [torch.tensor(a, requires_grad=True) for a in (px, ah, c)]
    wt = torch.tensor(w, requires_grad=True) if peep else None
    gates, cn, hn = lstm_cell(T[0], T[1], T[2], wt)
    dhn, dcn = rng.standard_normal((N, D)), rng.standard_normal((N, D))
    ((hn * torch.tensor(dhn)).sum() + (cn * torch.tensor(dcn)).sum()).backward()
    g2, c2, h2 = lstm_cell(px, ah, c, w)
    assert np.allclose(h2, hn.detach().numpy()) and np.allclose(c2, cn.detach().numpy())
    dpre, dc, dw = lstm_cell_bwd(dhn, dcn, c, g2, c2, w)
    assert np.allclose(dpre, T[0].grad.numpy()) and np.allclose(dpre, T[1].grad.numpy())
    assert np.allclose(dc, T[2].grad.numpy())
    if peep:
        assert np.allclose(dw, wt.grad.numpy())


def test_slots_match_header():
    import re
    from gnnb200 import temporal
    with open(os.path.join(ROOT, "include", "gnnb200.h")) as f:
        m = re.search(r"#define GNNB_LSTM_DW_SLOTS\(N\) \(\(N\) < (\d+) \? \(\(N\) \+ (\d+)\) / (\d+) : (\d+)\)", f.read())
    lim, add, div, cap = (int(v) for v in m.groups())
    for N in (0, 1, 63, 64, 65, 65535, 65536, 10 ** 6):
        assert temporal.lstm_dw_slots(N) == ((N + add) // div if N < lim else cap)


def test_exported(gnn):
    for n in ("GNNRecurrence", "TemporalSnapshotsGNNGraph", "initialstates", "TGCN", "TGCNCell", "GConvGRU",
              "GConvGRUCell", "GConvLSTM", "GConvLSTMCell", "DCGRU", "DCGRUCell", "EvolveGCNO", "EvolveGCNOCell"):
        assert n in gnn.__all__


# ---------------------------------------------------------------------------------------------- cells and layers
@pytest.mark.parametrize("kind", CELLS)
@pytest.mark.parametrize("state_kind", ["none", "vector", "matrix"])
def test_cell_reference_shape(gnn, tb, kind, state_kind):
    """the reference test's shape: in 3, out 5, N 4, 8 edges, k 2; one step"""
    run_case(gnn, tb, kind, 3, 5, 4, 1, k=2, state_kind=state_kind, extra=0, step=True)


@pytest.mark.parametrize("kind", CELLS)
@pytest.mark.parametrize("k", [2, 3])
def test_cell_200_nodes(gnn, tb, kind, k):
    if k == 3 and kind in ("tgcn", "evolvegcno"):
        pytest.skip("no order parameter")
    run_case(gnn, tb, kind, 2, 16, 200, 1, k=k, state_kind="matrix", step=True)


@pytest.mark.parametrize("kind", CELLS)
@pytest.mark.parametrize("T", [5, 12])
def test_layer_sequences(gnn, tb, kind, T):
    run_case(gnn, tb, kind, 3, 8, 40, T, k=3 if kind != "dcgru" else 2, state_kind="vector")


def _count(calls):
    return sum(c in ("gnnb_propagate", "gnnb_gcn_propagate") for c in calls)


@pytest.mark.parametrize("T", [1, 5])
def test_propagate_accounting(gnn, cpu_abi, T):
    from gnnb200 import temporal
    saved = temporal.lib
    temporal.lib = FakeRec(cpu_abi)
    try:
        s, t = ring_graph(30, 30, 0)
        g = gnn.GNNGraph(torch.as_tensor(s), torch.as_tensor(t), num_nodes=30)
        x = torch.randn(2, T, 30)
        cheb = gnn.ChebConv(2, 4, 3)
        dconv = gnn.DConv(2, 4, 3)
        cheb(g, x[:, 0])                                      # λmax cached from here on
        n0 = len(cpu_abi.calls); cheb(g, x[:, 0]); c_cheb = _count(cpu_abi.calls[n0:])
        n0 = len(cpu_abi.calls); dconv(g, x[:, 0]); c_d = _count(cpu_abi.calls[n0:])
        assert c_cheb == 2 and c_d == 6
        want = {"gconvgru": (1 + 2 * T) * c_cheb, "gconvlstm": (1 + T) * c_cheb, "dcgru": (1 + 2 * T) * c_d,
                "tgcn": 2, "evolvegcno": 1}
        for kind, n in want.items():
            layer = gnn.GNNRecurrence(make_layer(gnn, kind, 2, 4, 3, None))
            n0 = len(cpu_abi.calls)
            layer(g, x)
            assert _count(cpu_abi.calls[n0:]) == n, kind
        snaps = [gnn.GNNGraph(*[torch.as_tensor(v) for v in ring_graph(30 + 5 * i, 10 * i, i)], num_nodes=30 + 5 * i)
                 for i in range(4)]
        layer = gnn.EvolveGCNO(2, 4)
        n0 = len(cpu_abi.calls)
        layer(gnn.TemporalSnapshotsGNNGraph(snaps), [torch.randn(2, sg.num_nodes) for sg in snaps])
        assert _count(cpu_abi.calls[n0:]) == 4
    finally:
        temporal.lib = saved


@pytest.mark.parametrize("kind", CELLS)
def test_snapshot_graphs(gnn, tb, kind):
    """five snapshots with different edge sets (sizes differing for EvolveGCNO) against the reference, step by step"""
    dev = tb.dev
    sizes = [20, 25, 22, 30, 20] if kind == "evolvegcno" else [20] * 5
    graphs = [ring_graph(n, 3 * i, 10 + i) for i, n in enumerate(sizes)]
    snaps = [gnn.GNNGraph(torch.as_tensor(s).to(dev), torch.as_tensor(t).to(dev), num_nodes=n)
             for (s, t), n in zip(graphs, sizes)]
    tg = gnn.TemporalSnapshotsGNNGraph(snaps)
    assert tg.num_snapshots == 5 and len(tg) == 5 and tg.num_nodes == sizes and tg[2] is snaps[1]
    assert tg[[1, 3]].snapshots == [snaps[0], snaps[2]] and list(tg) == snaps
    cell = make_layer(gnn, kind, 3, 6, 2, dev, 3)
    xs = [torch.randn(3, n) for n in sizes]
    xd = [gnn.colmajor(x.to(dev)).requires_grad_(True) for x in xs]
    ys = gnn.GNNRecurrence(cell)(tg, xd)
    loss = sum((y * (i + 1)).sum() for i, y in enumerate(ys))
    loss.backward()
    P = {n: p.detach().double().cpu().requires_grad_(True) for n, p in cell.named_parameters()}
    x64 = [x.double().requires_grad_(True) for x in xs]
    state = ref_init(kind, P, 6, sizes[0], "none", None)
    ref = []
    for i, ((s, t), n) in enumerate(zip(graphs, sizes)):
        ops = Ops(s, t, n, getattr(snaps[i], "_lmax_cache", None) or 1.0, torch.device("cpu"))
        y, state = ref_step(kind, P, ops, x64[i], state)
        ref.append(y)
    sum((y * (i + 1)).sum() for i, y in enumerate(ref)).backward()
    for a, b in zip(ys, ref):
        assert rel(a, b) < 1e-5
    for a, b in zip(xd, x64):
        assert rel(a.grad, b.grad) < 1e-4
    for n, p in cell.named_parameters():
        if P[n].grad is not None and float(P[n].grad.norm()) > 0:
            assert rel(p.grad, P[n].grad) < 1e-4, n


@pytest.mark.parametrize("kind", ["gconvgru", "gconvlstm", "dcgru", "tgcn"])
def test_snapshot_node_count_mismatch(gnn, cpu_abi, kind):
    snaps = [gnn.GNNGraph(*[torch.as_tensor(v) for v in ring_graph(n, 0, 0)], num_nodes=n) for n in (10, 12)]
    layer = gnn.GNNRecurrence(make_layer(gnn, kind, 2, 4, 2, None))
    with pytest.raises(AssertionError):
        layer(gnn.TemporalSnapshotsGNNGraph(snaps), [torch.randn(2, 10), torch.randn(2, 12)])


@pytest.mark.parametrize("kind", CELLS)
def test_argument_errors(gnn, cpu_abi, kind):
    s, t = ring_graph(10, 0, 0)
    g = gnn.GNNGraph(torch.as_tensor(s), torch.as_tensor(t), num_nodes=10)
    layer = gnn.GNNRecurrence(make_layer(gnn, kind, 2, 4, 2, None))
    with pytest.raises(AssertionError):
        layer(g, torch.randn(3, 4, 10))                       # wrong in
    with pytest.raises(ValueError):
        layer(g, torch.randn(2, 0, 10))                       # T = 0
    if kind != "evolvegcno":
        bad = torch.zeros(4, 9) if kind != "gconvlstm" else (torch.zeros(4, 9), torch.zeros(4, 9))
        with pytest.raises(AssertionError):
            layer(g, torch.randn(2, 3, 10), bad)              # wrong state shape
        bad = torch.zeros(5) if kind != "gconvlstm" else (torch.zeros(5), torch.zeros(4))
        with pytest.raises(AssertionError):
            layer(g, torch.randn(2, 3, 10), bad)


def test_chebyshev_order(gnn):
    with pytest.raises(ValueError):
        gnn.GConvGRUCell(2, 3, 1)
    with pytest.raises(ValueError):
        gnn.GConvLSTMCell(2, 3, 1)


def test_initialstates(gnn):
    for kind in ("gconvgru", "dcgru", "tgcn"):
        st = gnn.initialstates(gnn.GNNRecurrence(make_layer(gnn, kind, 2, 4, 2, None)))
        assert tuple(st.shape) == (4,) and float(st.abs().sum()) == 0
    h, c = gnn.initialstates(make_layer(gnn, "gconvlstm", 2, 4, 2, None))
    assert tuple(h.shape) == tuple(c.shape) == (4,)
    cell = make_layer(gnn, "evolvegcno", 2, 4, 2, None)
    st = gnn.initialstates(cell)
    assert torch.equal(st.weight.reshape(2, 4).t(), cell.conv.weight.detach())


# ---------------------------------------------------------------------------------------------- GPU: the entries
def _cuda():
    if not torch.cuda.is_available():
        pytest.skip("no CUDA device")
    return torch.device("cuda")


def _entry_case(gnn, N, D, ld_extra=0, offset=0, seed=0):
    """every entry on the device against the float64 statements (computed in float64 on the device)"""
    from gnnb200._lib import lib, check
    dev = _cuda()
    gen = torch.Generator(device=dev).manual_seed(seed)
    st = torch.cuda.current_stream().cuda_stream
    o = offset

    def buf(*shape):
        n = int(np.prod(shape))
        b = torch.randn(n + o, generator=gen, device=dev)
        return b[o:].view(*shape)

    def out(*shape):
        n = int(np.prod(shape))
        return torch.full((n + o,), float("nan"), device=dev)[o:].view(*shape)

    def P(t):
        return t.data_ptr()
    ld3, ld4 = 3 * D + ld_extra, 4 * D + ld_extra
    px3, px4 = buf(max(N, 1), ld3)[:N], buf(max(N, 1), ld4)[:N]
    ah2, ah1, ah4, h, c = buf(N, 2 * D), buf(N, D), buf(N, 4 * D), buf(N, D), buf(N, D)
    w = buf(4 * D)
    r, z, rh, n, hn = out(N, D), out(N, D), out(N, D), out(N, D), out(N, D)
    check(lib.gnnb_gru_rz(P(px3), ld3, P(ah2), P(h), N, D, P(r), P(z), P(rh), st))
    for blend in (0, 1):
        check(lib.gnnb_gru_out(P(px3), ld3, P(ah1), P(h), P(z), N, D, blend, P(n), P(hn), st))
        d = lambda t: t.double()
        tol = 2e-6
        if N:
            r64, z64, rh64 = gru_rz(d(px3[:, :3 * D]), d(ah2), d(h))
            n64, hn64 = gru_out(d(px3[:, :3 * D]), d(ah1), d(h), d(z), blend)
            for a, b in ((r, r64), (z, z64), (rh, rh64), (n, n64), (hn, hn64)):
                assert rel(a, b) < tol
        dhn, drh = buf(N, D), buf(N, D)
        dpx = out(N, 3 * D)
        dz, dh = out(N, D), out(N, D)
        check(lib.gnnb_gru_out_bwd(P(dhn), P(h), P(z), P(n), N, D, blend, P(dpx) + 2 * D * 4, 3 * D, P(dz), P(dh), st))
        dh0 = dh.clone()
        check(lib.gnnb_gru_rz_bwd(P(drh), P(dz), P(h), P(r), P(z), N, D, P(dpx), 3 * D, P(dh), st))
        if N:
            a, b, cc = gru_out_bwd(d(dhn), d(h), d(z), d(n), blend)
            assert rel(dpx[:, 2 * D:], a) < tol and rel(dz, b) < tol and rel(dh0, cc) < tol
            a, b = gru_rz_bwd(d(drh), d(dz), d(h), d(r), d(z), d(dh0))
            assert rel(dpx[:, :2 * D], a) < tol and rel(dh, b) < tol
    for peep in (True, False):
        gates, cn, hn2 = out(N, 4 * D), out(N, D), out(N, D)
        check(lib.gnnb_lstm_cell(P(px4), ld4, P(ah4), P(c), P(w) if peep else None, N, D, P(gates), P(cn), P(hn2), st))
        dhn, dcn = buf(N, D), buf(N, D)
        dpre, dc, dw = out(N, 4 * D), out(N, D), out(4 * D)
        ws = torch.empty(_slots(N) * 4 * D + 1, device=dev)
        check(lib.gnnb_lstm_cell_bwd(P(dhn), P(dcn), P(c), P(gates), P(cn), P(w) if peep else None, N, D, P(dpre),
                                     P(dc), P(dw) if peep else None, P(ws) if peep else None, st))
        w64 = w.double() if peep else None
        if N:
            g64, c64, h64 = lstm_cell(px4[:, :4 * D].double(), ah4.double(), c.double(), w64)
            assert rel(gates, g64) < 2e-6 and rel(cn, c64) < 2e-6 and rel(hn2, h64) < 2e-6
            a, b, dw64 = lstm_cell_bwd(dhn.double(), dcn.double(), c.double(), gates.double(), cn.double(), w64)
            assert rel(dpre, a) < 2e-6 and rel(dc, b) < 2e-6
            if peep:
                assert rel(dw, dw64) < 1e-5
        elif peep:
            assert float(dw.abs().sum()) == 0
    torch.cuda.synchronize()


@pytest.mark.gpu
@pytest.mark.parametrize("D", [1, 3, 4, 5, 64, 128, 129, 1024])
@pytest.mark.parametrize("N", [0, 1, 1000, 10 ** 6])
def test_entries(gnn, N, D):
    if N == 10 ** 6 and D > 129:
        pytest.skip("N = 10^6 at D = 1024 needs about 100 GB for the LSTM buffers and their float64 statement")
    _entry_case(gnn, N, D)


@pytest.mark.gpu
@pytest.mark.parametrize("D", [4, 64, 129])
def test_entries_strided_and_misaligned(gnn, D):
    _entry_case(gnn, 1000, D, ld_extra=8)
    _entry_case(gnn, 1000, D, offset=1)                       # 4-byte offset: the scalar path


@pytest.mark.gpu
def test_entry_status_codes(gnn):
    from gnnb200._lib import lib
    _cuda()
    x = torch.zeros(64, device="cuda")
    p = x.data_ptr()
    assert lib.gnnb_gru_rz(p, 3, p, p, -1, 1, p, p, p, None) == ESIZE
    assert lib.gnnb_gru_rz(p, 3, p, p, 1, 0, p, p, p, None) == ESIZE
    assert lib.gnnb_gru_rz(p, 2, p, p, 1, 1, p, p, p, None) == ESIZE
    assert lib.gnnb_gru_rz(None, 3, p, p, 1, 1, p, p, p, None) == ESIZE
    assert lib.gnnb_gru_rz(None, 3, None, None, 0, 1, None, None, None, None) == OK
    assert lib.gnnb_gru_out(p, 3, p, p, p, 1, 1, 2, p, p, None) == EINVAL
    assert lib.gnnb_gru_out_bwd(p, p, p, p, 1, 2, 0, p, 1, p, p, None) == ESIZE
    assert lib.gnnb_gru_rz_bwd(p, p, p, p, p, 1, 2, p, 3, p, None) == ESIZE
    assert lib.gnnb_lstm_cell(p, 3, p, p, None, 1, 1, p, p, p, None) == ESIZE
    assert lib.gnnb_lstm_cell(p, 4, p, None, None, 1, 1, p, p, p, None) == ESIZE
    assert lib.gnnb_lstm_cell_bwd(p, p, p, p, p, None, 1, 1, p, p, p, p, None) == EINVAL
    assert lib.gnnb_lstm_cell_bwd(p, p, p, p, p, p, 1, 1, p, p, p, None, None) == ESIZE
    torch.cuda.synchronize()


# ---------------------------------------------------------------------------------------------- GPU: layers
@pytest.mark.gpu
@pytest.mark.parametrize("kind", CELLS)
def test_run_to_run(gnn, kind):
    dev = _cuda()
    outs = []
    for _ in range(2):
        y, gx, cell = run_case(gnn, SimpleNamespace(dev=dev, calls=None), kind, 4, 16, 300, 6, k=3, state_kind="matrix")
        outs.append((y.detach().clone(), gx.clone(), [p.grad.clone() for p in cell.parameters() if p.grad is not None]))
    assert torch.equal(outs[0][0], outs[1][0]) and torch.equal(outs[0][1], outs[1][1])
    assert all(torch.equal(a, b) for a, b in zip(outs[0][2], outs[1][2]))


def knn_sensor_batch(gnn, windows, n=207, k=8, seed=0):
    """`windows` copies of a kNN (k = 8) graph of n points in the plane, batched: 1-based (s, t), node count"""
    rng = np.random.default_rng(seed)
    pts = rng.random((n, 2))
    d = ((pts[:, None] - pts[None]) ** 2).sum(-1)
    np.fill_diagonal(d, np.inf)
    nb = np.argsort(d, 1)[:, :k]
    s1, t1 = nb.reshape(-1), np.repeat(np.arange(n), k)          # neighbour -> node
    s = np.concatenate([s1 + w * n for w in range(windows)]) + 1
    t = np.concatenate([t1 + w * n for w in range(windows)]) + 1
    return s, t, n * windows


def big_case(gnn, kind, s, t, N, nin, out, T, k, seed=0, fwd_tol=1e-5, grad_tol=1e-4):
    """a layer on a large graph against the float64 sparse statement (on the device)"""
    dev = _cuda()
    g = gnn.GNNGraph(torch.as_tensor(s).to(dev), torch.as_tensor(t).to(dev), num_nodes=N)
    cell = make_layer(gnn, kind, nin, out, k, dev, seed, dconv_scale(s, t, k))
    gen = torch.Generator(device=dev).manual_seed(seed)
    x = torch.randn(nin, T, N, generator=gen, device=dev)
    xs = gnn.colmajor(x).requires_grad_(True)
    y = gnn.GNNRecurrence(cell)(g, xs)
    R = torch.randn(out, T, N, generator=gen, device=dev)
    (y * R).sum().backward()
    ops = Ops(s, t, N, getattr(g, "_lmax_cache", None) or 1.0, dev, sparse=True)
    P = {n: p.detach().double().requires_grad_(True) for n, p in cell.named_parameters()}
    x64 = x.double().requires_grad_(True)
    state = ref_init(kind, P, out, N, "none", None)
    if kind != "evolvegcno":
        state = (state[0].to(dev), state[1].to(dev)) if kind == "gconvlstm" else state.to(dev)
    else:
        state = (state[0], (state[1][0].to(dev), state[1][1].to(dev)))
    ys = []
    for tt in range(T):
        yt, state = ref_step(kind, P, ops, x64[:, tt], state)
        ys.append(yt)
    y64 = torch.stack(ys, 1)
    (y64 * R.double()).sum().backward()
    assert rel(y, y64) < fwd_tol, f"{kind} forward {rel(y, y64):.2e}"
    assert rel(xs.grad, x64.grad) < grad_tol, f"{kind} dx {rel(xs.grad, x64.grad):.2e}"
    for n, p in cell.named_parameters():
        if P[n].grad is not None and float(P[n].grad.norm()) > 0:
            assert rel(p.grad, P[n].grad) < grad_tol, f"{kind} d{n} {rel(p.grad, P[n].grad):.2e}"


@pytest.mark.gpu
@pytest.mark.parametrize("kind", CELLS)
def test_traffic_sized_batch(gnn, kind):
    """64 windows of a 207-node kNN sensor graph, batched, T = 12, in 2, out 64"""
    s, t, N = knn_sensor_batch(gnn, 64)
    big_case(gnn, kind, s, t, N, 2, 64, 12, 3 if kind != "dcgru" else 2)


@pytest.mark.gpu
@pytest.mark.parametrize("kind", CELLS)
def test_rmat_200k(gnn, kind):
    """RMAT 200 k nodes / 2 M edges plus a ring (no isolated nodes, as ChebConv requires), T = 12"""
    dev = _cuda()
    g0 = gnn.rmat_graph(200_000, 2_000_000, seed=17, device=dev)
    i = np.arange(200_000)
    s = np.concatenate([g0.s.cpu().numpy(), i + 1])
    t = np.concatenate([g0.t.cpu().numpy(), (i + 1) % 200_000 + 1])
    # the weight gradients sum 2.4 M node-steps of a power-law graph in fp32: 2e-4 (TGCN's first layer lands at 1.0e-4)
    big_case(gnn, kind, s, t, 200_000, 4, 16, 12, 2, grad_tol=2e-4)
