"""TEST DOUBLE of libgnnb200's C ABI on host memory — test infrastructure only, never imported by the package.

The host-side mirror (graph.py / msgpass.py / layers.py / readout.py) talks to the library through ``lib.gnnb_*`` calls
with raw pointers.  On a box without a GPU every one of those calls fails with GNNB_ECUDA (by design: no CPU
fallback), so the host logic — argument checks, Julia-shape bookkeeping, the autograd wiring of every layer — would
only ever run in the ``-m gpu`` tests.  This module restates the *contract* of each entry of include/gnnb200.h that
the mirror uses, in numpy on host pointers, and the ``cpu_abi`` fixture (conftest.py) swaps it in for the duration of
one test.  What such a test proves: the Python above the ABI composes the entries the way the reference composes
NNlib's (checked against dense torch formulas).  What it does not prove: anything about the CUDA kernels — that is
tests/test_gpu_*.py against oracle/.

Arithmetic is float64 inside, rounded once to float32 on the way out.
"""
from __future__ import annotations

import ctypes as C
from contextlib import contextmanager
from types import SimpleNamespace

import numpy as np

OK, EINVAL, ESIZE, ECUDA, ENOMEM, EUNSUPPORTED, EINDEX = range(7)
SUM, MEAN, MAX, MIN = 0, 1, 2, 3
SRC, DST = 0, 1
DIR_OUT, DIR_IN, DIR_BOTH = 0, 1, 2


def _addr(p):
    if p is None:
        return None
    if isinstance(p, C.c_void_p):
        return p.value
    return int(p)


def _arr(p, shape, dtype=np.float32):
    """numpy view (writable) of host memory at pointer p."""
    a = _addr(p)
    shape = tuple(int(v) for v in shape)
    n = int(np.prod(shape)) if shape else 1
    if a is None:
        return None
    if n == 0:
        return np.empty(shape, dtype)
    buf = (C.c_char * (n * np.dtype(dtype).itemsize)).from_address(a)
    return np.frombuffer(buf, dtype=dtype).reshape(shape)


def _deref(ref):
    """the ctypes object behind C.byref(obj) (or a pointer instance)"""
    if ref is None:
        return None
    return ref._obj if hasattr(ref, "_obj") else ref.contents


class _Plan:
    def __init__(self, s, t, ns, nd):
        self.s, self.t, self.ns, self.nd = s, t, ns, nd
        self.E = len(s)

    def idx(self, which):
        return (self.s, self.ns) if which == SRC else (self.t, self.nd)


def _segment(aggr, m, idx, n):
    """NNlib.scatter(aggr, m, idx; dstsize=n) on rows: m (E, ...) -> (n, ...), neutral element for empty segments."""
    m = m.astype(np.float64)
    shape = (n,) + m.shape[1:]
    if aggr in (SUM, MEAN):
        out = np.zeros(shape)
        np.add.at(out, idx, m)
        if aggr == MEAN:
            cnt = np.bincount(idx, minlength=n).astype(np.float64)
            out /= np.maximum(cnt, 1).reshape((n,) + (1,) * (m.ndim - 1))
        return out
    if aggr == MAX:
        out = np.full(shape, -np.inf)
        np.maximum.at(out, idx, m)
        return out
    out = np.full(shape, np.inf)
    np.minimum.at(out, idx, m)
    return out


class FakeLib:
    """Object with the ``gnnb_*`` attributes the mirror calls; every method returns a gnnb_status."""

    def __init__(self):
        self._plans = {}
        self._next = 1
        self._err = b""
        self.calls = []          # names of the entries called, in order (tests assert on the dispatch)

    # ------------------------------------------------------------------ bookkeeping
    def _fail(self, code, msg):
        self._err = msg.encode()
        return code

    def _new(self, plan):
        h = self._next
        self._next += 1
        self._plans[h] = plan
        return h

    def _p(self, h) -> _Plan:
        return self._plans[_addr(h)]

    def gnnb_last_error(self):
        return self._err

    def gnnb_version(self):
        return b"fake-abi (tests/fake_abi.py)"

    def gnnb_device_count(self):
        return 1

    def gnnb_launch_count(self):
        return 0

    # ------------------------------------------------------------------ graph
    def gnnb_graph_create(self, out, src, dst, E, ns, nd, index_bytes, index_base, on_device, stream):
        self.calls.append("gnnb_graph_create")
        if index_bytes not in (4, 8) or index_base not in (0, 1):
            return self._fail(EINVAL, "index_bytes must be 4 or 8 and index_base 0 or 1")
        if E < 0 or ns < 0 or nd < 0 or E >= 2 ** 31:
            return self._fail(ESIZE, "bad sizes")
        dt = np.int32 if index_bytes == 4 else np.int64
        s = _arr(src, (E,), dt).astype(np.int64) - index_base
        t = _arr(dst, (E,), dt).astype(np.int64) - index_base
        if E and (s.min() < 0 or s.max() >= ns or t.min() < 0 or t.max() >= nd):
            return self._fail(EINDEX, "edge index out of range")
        _deref(out).value = self._new(_Plan(s, t, int(ns), int(nd)))
        return OK

    def gnnb_graph_destroy(self, h):
        self._plans.pop(_addr(h), None)
        return OK

    def gnnb_graph_add_self_loops(self, h, out, stream):
        self.calls.append("gnnb_graph_add_self_loops")
        p = self._p(h)
        if p.ns != p.nd:
            return self._fail(ESIZE, "add_self_loops needs num_src == num_dst")
        loops = np.arange(p.ns, dtype=np.int64)
        _deref(out).value = self._new(_Plan(np.concatenate([p.s, loops]), np.concatenate([p.t, loops]), p.ns, p.nd))
        return OK

    def gnnb_graph_info(self, h, e, ns, nd):
        p = self._p(h)
        for ref, v in ((e, p.E), (ns, p.ns), (nd, p.nd)):
            if ref is not None:
                _deref(ref).value = v
        return OK

    def gnnb_degree(self, h, d, w, out, stream):
        self.calls.append("gnnb_degree")
        p = self._p(h)
        wv = np.ones(p.E) if w is None else _arr(w, (p.E,)).astype(np.float64)
        if d == DIR_BOTH and p.ns != p.nd:
            return self._fail(ESIZE, "dir=:both needs num_src == num_dst")
        n = p.nd if d != DIR_OUT else p.ns
        acc = np.zeros(n)
        if d in (DIR_IN, DIR_BOTH):
            np.add.at(acc, p.t, wv)
        if d in (DIR_OUT, DIR_BOTH):
            np.add.at(acc, p.s, wv)
        _arr(out, (n,))[...] = acc
        return OK

    # ------------------------------------------------------------------ gather / scatter
    def gnnb_gather(self, h, which, x, D, out, stream):
        self.calls.append("gnnb_gather")
        p = self._p(h)
        idx, n = p.idx(which)
        _arr(out, (p.E, D))[...] = _arr(x, (n, D))[idx]
        return OK

    def gnnb_scatter(self, h, which, aggr, m, D, out, stream):
        self.calls.append("gnnb_scatter")
        p = self._p(h)
        idx, n = p.idx(which)
        _arr(out, (n, D))[...] = _segment(aggr, _arr(m, (p.E, D)), idx, n)
        return OK

    # ------------------------------------------------------------------ propagate
    def _messages(self, p, x, w, cs, D, transposed):
        src, dst, ns, nd = (p.s, p.t, p.ns, p.nd) if not transposed else (p.t, p.s, p.nd, p.ns)
        xv = _arr(x, (ns, D)).astype(np.float64)
        if cs is not None:
            xv = xv * _arr(cs, (ns,)).astype(np.float64)[:, None]
        m = xv[src]
        if w is not None:
            m = m * _arr(w, (p.E,)).astype(np.float64)[:, None]
        return m, dst, nd

    def gnnb_propagate(self, h, transposed, msg, aggr, x, w, cs, ct, D, out, stream):
        self.calls.append("gnnb_propagate")
        p = self._p(h)
        if msg == 1 and w is None and p.E > 0:
            return self._fail(EINVAL, "w_mul_xj needs edge weights")
        m, dst, nd = self._messages(p, x, w if msg == 1 else None, cs, D, transposed)
        o = _segment(aggr, m, dst, nd)
        if ct is not None:
            o = o * _arr(ct, (nd,)).astype(np.float64)[:, None]
        _arr(out, (nd, D))[...] = o
        return OK

    def gnnb_propagate_bwd(self, h, msg, aggr, dout, x, w, cs, ct, out_fwd, D, dx, dw, stream):
        self.calls.append("gnnb_propagate_bwd")
        p = self._p(h)
        if aggr in (MAX, MIN) and dw is not None:
            return self._fail(EUNSUPPORTED, "dw for max/min")
        g = _arr(dout, (p.nd, D)).astype(np.float64)
        wv = np.ones(p.E) if (w is None or msg != 1) else _arr(w, (p.E,)).astype(np.float64)
        csv = np.ones(p.ns) if cs is None else _arr(cs, (p.ns,)).astype(np.float64)
        ctv = np.ones(p.nd) if ct is None else _arr(ct, (p.nd,)).astype(np.float64)
        xv = _arr(x, (p.ns, D)).astype(np.float64) if x is not None else None
        if aggr == MEAN:
            ctv = ctv / np.maximum(np.bincount(p.t, minlength=p.nd), 1)
        ge = g[p.t] * ctv[p.t][:, None]                               # upstream gradient per edge
        if aggr in (MAX, MIN):
            m = xv[p.s] * (csv[p.s] * wv)[:, None]
            ref = _arr(out_fwd, (p.nd, D)).astype(np.float64) / ctv[:, None]
            ge = ge * (m.astype(np.float32) == ref.astype(np.float32)[p.t])
        if dx is not None:
            acc = np.zeros((p.ns, D))
            np.add.at(acc, p.s, ge * wv[:, None])
            _arr(dx, (p.ns, D))[...] = acc * csv[:, None]
        if dw is not None:
            _arr(dw, (p.E,))[...] = (ge * xv[p.s]).sum(1) * csv[p.s]
        return OK

    # ------------------------------------------------------------------ edge softmax
    def _softmax(self, p, e):
        mx = _segment(MAX, e, p.t, p.nd)
        ex = np.exp(e.astype(np.float64) - mx[p.t])
        return ex / _segment(SUM, ex, p.t, p.nd)[p.t]

    def gnnb_softmax_edge_neighbors(self, h, e, K, out, stream):
        self.calls.append("gnnb_softmax_edge_neighbors")
        p = self._p(h)
        _arr(out, (p.E, K))[...] = self._softmax(p, _arr(e, (p.E, K)))
        return OK

    def gnnb_softmax_edge_neighbors_bwd(self, h, alpha, dalpha, K, de, stream):
        self.calls.append("gnnb_softmax_edge_neighbors_bwd")
        p = self._p(h)
        a = _arr(alpha, (p.E, K)).astype(np.float64)
        da = _arr(dalpha, (p.E, K)).astype(np.float64)
        _arr(de, (p.E, K))[...] = a * (da - _segment(SUM, a * da, p.t, p.nd)[p.t])
        return OK

    # ------------------------------------------------------------------ GCN core
    def gnnb_gcn_norm(self, h, w, c_out, stream):
        self.calls.append("gnnb_gcn_norm")
        p = self._p(h)
        wv = np.ones(p.E) if w is None else _arr(w, (p.E,)).astype(np.float64)
        d = np.zeros(p.nd)
        np.add.at(d, p.t, wv)
        with np.errstate(divide="ignore"):
            _arr(c_out, (p.nd,))[...] = 1.0 / np.sqrt(d)
        return OK

    def gnnb_gcn_propagate(self, h, transposed, x, w, c, D, out, stream):
        self.calls.append("gnnb_gcn_propagate")
        p = self._p(h)
        n = p.nd
        if c is None:                                   # the plan-owned default normalisation (unweighted only)
            assert w is None
            d = np.zeros(n)
            np.add.at(d, p.t, 1.0)
            with np.errstate(divide="ignore"):
                cv = 1.0 / np.sqrt(d)
        else:
            cv = _arr(c, (n,)).astype(np.float64)
        xv = _arr(x, (n, D)).astype(np.float64) * cv[:, None]
        src, dst = (p.s, p.t) if not transposed else (p.t, p.s)
        m = xv[src]
        if w is not None:
            m = m * _arr(w, (p.E,)).astype(np.float64)[:, None]
        _arr(out, (n, D))[...] = _segment(SUM, m, dst, n) * cv[:, None]
        return OK

    # ------------------------------------------------------------------ GAT core
    def _gat_alpha(self, p, el, er, H, slope):
        z = _arr(el, (p.nd, H)).astype(np.float64)[p.t] + _arr(er, (p.ns, H)).astype(np.float64)[p.s]
        lg = np.where(z > 0, z, slope * z)
        return z, lg

    def gnnb_gat_aggregate(self, h, Wx, el, er, Cc, H, slope, out, alpha, seg_max, seg_sum, stream):
        self.calls.append("gnnb_gat_aggregate")
        p = self._p(h)
        _, lg = self._gat_alpha(p, el, er, H, slope)
        mx = _segment(MAX, lg, p.t, p.nd)
        ex = np.exp(lg - mx[p.t])
        ssum = _segment(SUM, ex, p.t, p.nd)
        a = ex / ssum[p.t]
        W = _arr(Wx, (p.ns, H, Cc)).astype(np.float64)
        _arr(out, (p.nd, H, Cc))[...] = _segment(SUM, a[:, :, None] * W[p.s], p.t, p.nd)
        if alpha is not None:
            _arr(alpha, (p.E, H))[...] = a
        if seg_max is not None:
            _arr(seg_max, (p.nd, H))[...] = mx
        if seg_sum is not None:
            _arr(seg_sum, (p.nd, H))[...] = ssum
        return OK

    def gnnb_gat_aggregate_bwd(self, h, Wx, el, er, seg_max, seg_sum, out_fwd, dout, Cc, H, slope, dWx, del_, der,
                               stream):
        self.calls.append("gnnb_gat_aggregate_bwd")
        p = self._p(h)
        z, lg = self._gat_alpha(p, el, er, H, slope)
        mx = _arr(seg_max, (p.nd, H)).astype(np.float64)
        ss = _arr(seg_sum, (p.nd, H)).astype(np.float64)
        a = np.exp(lg - mx[p.t]) / ss[p.t]
        W = _arr(Wx, (p.ns, H, Cc)).astype(np.float64)
        g = _arr(dout, (p.nd, H, Cc)).astype(np.float64)
        o = _arr(out_fwd, (p.nd, H, Cc)).astype(np.float64)
        acc = np.zeros((p.ns, H, Cc))
        np.add.at(acc, p.s, a[:, :, None] * g[p.t])
        _arr(dWx, (p.ns, H, Cc))[...] = acc
        da = (g[p.t] * W[p.s]).sum(-1)                       # dL/dα_k
        T = (g * o).sum(-1)                                  # Σ_k α_k dα_k per target
        dlg = a * (da - T[p.t])
        dz = dlg * np.where(z > 0, 1.0, slope)
        _arr(del_, (p.nd, H))[...] = _segment(SUM, dz, p.t, p.nd)
        _arr(der, (p.ns, H))[...] = _segment(SUM, dz, p.s, p.ns)
        return OK

    def gnnb_bias_act(self, x, bias, relu, N, D, y, stream):
        self.calls.append("gnnb_bias_act")
        pre = _arr(x, (N, D)).astype(np.float64)
        if bias is not None:
            pre = pre + _arr(bias, (D,)).astype(np.float64)
        _arr(y, (N, D))[...] = np.maximum(pre, 0) if relu else pre
        return OK

    def gnnb_bias_act_bwd(self, dy, y, relu, N, D, dpre, db, stream):
        self.calls.append("gnnb_bias_act_bwd")
        d = _arr(dy, (N, D)).astype(np.float64)
        if relu:
            d = d * (_arr(y, (N, D)) > 0)
            _arr(dpre, (N, D))[...] = d
        if db is not None:
            _arr(db, (D,))[...] = d.sum(0)
        return OK

    def gnnb_linear2(self, x1, x2, W, bias, relu, N, Din1, Din2, Dout, y, stream):
        self.calls.append("gnnb_linear2")
        Wm = _arr(W, (Dout, Din1 + Din2)).astype(np.float64)
        pre = _arr(x1, (N, Din1)).astype(np.float64) @ Wm[:, :Din1].T + _arr(x2, (N, Din2)).astype(np.float64) @ Wm[:, Din1:].T
        if bias is not None:
            pre = pre + _arr(bias, (Dout,)).astype(np.float64)
        _arr(y, (N, Dout))[...] = np.maximum(pre, 0) if relu else pre
        return OK

    def gnnb_linear2_bwd(self, dy, y, x1, x2, W, relu, N, Din1, Din2, Dout, dpre_ws, dx1, dx2, dW, db, stream):
        self.calls.append("gnnb_linear2_bwd")
        Wm = _arr(W, (Dout, Din1 + Din2)).astype(np.float64)
        dpre = _arr(dy, (N, Dout)).astype(np.float64)
        if relu:
            dpre = dpre * (_arr(y, (N, Dout)) > 0)
        if dx1 is not None:
            _arr(dx1, (N, Din1))[...] = dpre @ Wm[:, :Din1]
        if dx2 is not None:
            _arr(dx2, (N, Din2))[...] = dpre @ Wm[:, Din1:]
        if dW is not None:
            out = _arr(dW, (Dout, Din1 + Din2))
            out[:, :Din1] = dpre.T @ _arr(x1, (N, Din1)).astype(np.float64)
            out[:, Din1:] = dpre.T @ _arr(x2, (N, Din2)).astype(np.float64)
        if db is not None:
            _arr(db, (Dout,))[...] = dpre.sum(0)
        return OK

    def gnnb_gat_logit_terms(self, Wx, a, N, Cc, H, el, er, stream):
        self.calls.append("gnnb_gat_logit_terms")
        W = _arr(Wx, (N, H, Cc)).astype(np.float64)
        A = _arr(a, (H, 2 * Cc)).astype(np.float64)          # Julia (2C, H) column-major memory
        _arr(el, (N, H))[...] = (W * A[None, :, :Cc]).sum(-1)
        _arr(er, (N, H))[...] = (W * A[None, :, Cc:]).sum(-1)
        return OK

    def gnnb_gat_logit_terms_bwd(self, Wx, a, del_, der, N, Cc, H, dWx, da, stream):
        self.calls.append("gnnb_gat_logit_terms_bwd")
        W = _arr(Wx, (N, H, Cc)).astype(np.float64)
        A = _arr(a, (H, 2 * Cc)).astype(np.float64)
        dl = _arr(del_, (N, H)).astype(np.float64)
        dr = _arr(der, (N, H)).astype(np.float64)
        acc = _arr(dWx, (N, H, Cc))
        acc[...] = acc.astype(np.float64) + dl[:, :, None] * A[None, :, :Cc] + dr[:, :, None] * A[None, :, Cc:]
        out = _arr(da, (H, 2 * Cc))
        out[:, :Cc] = (dl[:, :, None] * W).sum(0)
        out[:, Cc:] = (dr[:, :, None] * W).sum(0)
        return OK

    # ------------------------------------------------------------------ node-partitioned shards
    def gnnb_gather_rows(self, idx, n, x, D, out, stream):
        self.calls.append("gnnb_gather_rows")
        ii = _arr(idx, (n,), np.int32)
        nrows = int(ii.max()) + 1 if n else 0
        _arr(out, (n, D))[...] = _arr(x, (nrows, D))[ii]
        return OK

    def gnnb_propagate_halo(self, h, msg, aggr, x_local, x_halo, n_local, w, cs, ct, D, out, stream):
        self.calls.append("gnnb_propagate_halo")
        p = self._p(h)
        n_halo = p.ns - n_local
        xv = np.concatenate([_arr(x_local, (n_local, D)), _arr(x_halo, (n_halo, D)) if n_halo else
                             np.empty((0, D), np.float32)]).astype(np.float64)
        if cs is not None:
            xv = xv * _arr(cs, (p.ns,)).astype(np.float64)[:, None]
        m = xv[p.s]
        if msg == 1:
            m = m * _arr(w, (p.E,)).astype(np.float64)[:, None]
        o = _segment(aggr, m, p.t, p.nd)
        if ct is not None:
            o = o * _arr(ct, (p.nd,)).astype(np.float64)[:, None]
        _arr(out, (p.nd, D))[...] = o
        return OK

    # ------------------------------------------------------------------ neighbour sampling
    def gnnb_sample_neighbors(self, h, nodes, n, index_bytes, index_base, K, d, replace, seed, offsets, eids, capacity,
                              total, stream):
        self.calls.append("gnnb_sample_neighbors")
        p = self._p(h)
        key, nrows = (p.t, p.nd) if d == DIR_IN else (p.s, p.ns)
        _deref(total).value = 0
        off = _arr(offsets, (n + 1,), np.int64)
        off[0] = 0
        if n == 0:
            return OK
        dt = np.int32 if index_bytes == 4 else np.int64
        nd = _arr(nodes, (n,), dt).astype(np.int64) - index_base
        if nd.min() < 0 or nd.max() >= nrows:
            return self._fail(EINDEX, "node id out of range")
        order = np.argsort(key, kind="stable")
        rowptr = np.concatenate([[0], np.cumsum(np.bincount(key, minlength=nrows))])
        picks = []
        for j, r in enumerate(nd):
            row = order[rowptr[r]:rowptr[r + 1]]
            deg = len(row)
            k = 0 if deg == 0 else ((K if K > 0 else deg) if replace else (min(K, deg) if K > 0 else deg))
            rng = np.random.default_rng([int(seed) & 0x7FFFFFFF, j])
            if k == deg and not replace:
                picks.append(row)
            else:
                picks.append(rng.choice(row, size=k, replace=bool(replace)) if k else row[:0])
        cnt = np.array([len(x) for x in picks], dtype=np.int64)
        off[1:] = np.cumsum(cnt)
        tot = int(off[-1])
        _deref(total).value = tot
        if eids is None or tot == 0:
            return OK
        if capacity < tot:
            return self._fail(ESIZE, "eids buffer too small")
        _arr(eids, (tot,), np.int64)[...] = np.concatenate(picks) + index_base
        return OK

    # ------------------------------------------------------------------ edge-list transforms
    def gnnb_sort_edge_index(self, u, v, E, max_index, index_bytes, u_out, v_out, perm_out, stream):
        self.calls.append("gnnb_sort_edge_index")
        dt = np.int32 if index_bytes == 4 else np.int64
        if E == 0:
            return OK
        uu, vv = _arr(u, (E,), dt).copy(), _arr(v, (E,), dt).copy()
        if min(uu.min(), vv.min()) < 0 or max(uu.max(), vv.max()) > max_index:
            return self._fail(EINDEX, "edge index outside [0, max_index]")
        perm = np.lexsort((vv, uu))                      # stable, u major
        if u_out is not None:
            _arr(u_out, (E,), dt)[...] = uu[perm]
        if v_out is not None:
            _arr(v_out, (E,), dt)[...] = vv[perm]
        if perm_out is not None:
            _arr(perm_out, (E,), np.int64)[...] = perm
        return OK

    def gnnb_coalesce_edges(self, src, dst, E, n, index_bytes, index_base, src_out, dst_out, perm_out, seg_out,
                            num_unique, stream):
        self.calls.append("gnnb_coalesce_edges")
        dt = np.int32 if index_bytes == 4 else np.int64
        _deref(num_unique).value = 0
        if E == 0:
            return OK
        s, t = _arr(src, (E,), dt).astype(np.int64), _arr(dst, (E,), dt).astype(np.int64)
        if min(s.min(), t.min()) < index_base or max(s.max(), t.max()) >= index_base + n:
            return self._fail(EINDEX, "edge index out of range")
        perm = np.lexsort((t, s))
        ss, ts = s[perm], t[perm]
        head = np.ones(E, bool)
        head[1:] = (ss[1:] != ss[:-1]) | (ts[1:] != ts[:-1])
        seg = np.cumsum(head)
        nu = int(seg[-1])
        _arr(src_out, (E,), dt)[:nu] = ss[head]
        _arr(dst_out, (E,), dt)[:nu] = ts[head]
        _arr(perm_out, (E,), np.int64)[...] = perm
        _arr(seg_out, (E,), np.int64)[...] = seg
        _deref(num_unique).value = nu
        return OK

    def gnnb_graph_csr_device(self, h, transposed, rowptr, col, eid, stream):
        self.calls.append("gnnb_graph_csr_device")
        p = self._p(h)
        key, other, nrows = (p.t, p.s, p.nd) if not transposed else (p.s, p.t, p.ns)
        order = np.argsort(key, kind="stable")
        if rowptr is not None:
            _arr(rowptr, (nrows + 1,), np.int32)[...] = np.concatenate([[0], np.cumsum(np.bincount(key, minlength=nrows))])
        if col is not None and p.E:
            _arr(col, (p.E,), np.int32)[...] = other[order]
        if eid is not None and p.E:
            _arr(eid, (p.E,), np.int32)[...] = order
        return OK

    def __getattr__(self, name):
        if name.startswith("gnnb_"):
            raise AttributeError(f"tests/fake_abi.py does not restate {name}; the host logic under test must not need it")
        raise AttributeError(name)


class _NullDevice:
    """stand-in for torch.cuda.device(...) while the fake ABI is installed"""

    def __init__(self, *a, **k):
        pass

    def __enter__(self):
        return self

    def __exit__(self, *a):
        return False


@contextmanager
def installed():
    """Swap the fake ABI in for libgnnb200 in every module of the mirror; restore on exit."""
    import torch
    import gnnb200
    from gnnb200 import _lib, graph, layers, msgpass, partition, readout, sampling, transform

    fake = FakeLib()
    mods = [_lib, graph, layers, msgpass, readout, transform, partition, sampling]
    saved = [(m, m.lib) for m in mods]
    saved_cuda = (torch.cuda.device, torch.cuda.current_stream)
    orig_dev = graph._compute_device
    orig_init = graph._Plan.__init__
    made = []                                    # plans holding fake handles: defused before the real library returns

    def recording_init(self, handle, device):
        orig_init(self, handle, device)
        made.append(self)

    try:
        for m in mods:
            m.lib = fake
        torch.cuda.device = _NullDevice
        torch.cuda.current_stream = lambda device=None: SimpleNamespace(cuda_stream=0)
        graph._compute_device = lambda t: torch.device("cpu")
        graph._Plan.__init__ = recording_init
        yield fake
    finally:
        for pl in made:
            pl.h = None                          # _Plan.__del__ must never hand a fake handle to gnnb_graph_destroy
        graph._Plan.__init__ = orig_init
        graph._compute_device = orig_dev
        torch.cuda.device, torch.cuda.current_stream = saved_cuda
        for m, l in saved:
            m.lib = l
