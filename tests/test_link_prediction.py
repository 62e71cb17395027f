"""Link prediction: edge codes, rand_graph, negative_sample, rand_edge_split, perturb_edges, add_edges, intersect and
the dot decoder (graphneuralnetworks.jl_b200/linkpred.py over csrc/edgegen.cu; GNNGraphs/src/utils.jl:189-290,
generate.jl:51-65, transform.jl:319-418,890-968, operators.jl:7-20).

The contract is stated below in numpy and is integer-exact: the code spaces with their encode / decode (decoding by
exact integer square roots here, by a float64 estimate plus integer correction in the kernel), the Feistel
permutation π with its cycle walk, and "the first m codes of π(0), π(1), ... not in the exclusion set".  The kernels
are compared with it by `==`.

Back ends of the mirror: `FakeLink`, the five C entries restated on host pointers over that statement (swapped in
over tests/fake_abi.py's double), and, under -m gpu, the CUDA kernels.
"""
import ctypes as C
import math
import os
import re
import sys

import numpy as np
import pytest
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
OK, EINVAL, ESIZE, ECUDA, ENOMEM, EUNSUPPORTED, EINDEX = range(7)
D, DN, UD, UN, BP = range(5)           # GNNB_CODES_DIRECTED, _NOLOOP, UNDIRECTED, _NOLOOP, BIPARTITE
SPACES = (D, DN, UD, UN, BP)
U = np.uint64
MASK = 2 ** 64 - 1

with open(os.path.join(ROOT, "include", "gnnb200.h")) as _f:
    ROUNDS = int(re.search(r"#define GNNB_FEISTEL_ROUNDS (\d+)", _f.read()).group(1))


# ---------------------------------------------------------------------------------------------- the contract in numpy
def smix_int(x):
    """splitmix64's output function on a Python int"""
    x = (x + 0x9E3779B97F4A7C15) & MASK
    x = ((x ^ (x >> 30)) * 0xBF58476D1CE4E5B9) & MASK
    x = ((x ^ (x >> 27)) * 0x94D049BB133111EB) & MASK
    return x ^ (x >> 31)


def smix(x):
    """the same on a uint64 array (numpy's array arithmetic wraps mod 2^64)"""
    x = x + U(0x9E3779B97F4A7C15)
    x = (x ^ (x >> U(30))) * U(0xBF58476D1CE4E5B9)
    x = (x ^ (x >> U(27))) * U(0x94D049BB133111EB)
    return x ^ (x >> U(31))


def feistel_keys(M, seed):
    h = 1
    while h < 31 and (1 << (2 * h)) < M:
        h += 1
    k0 = smix_int(seed & MASK)
    return h, [smix_int((k0 + r) & MASK) for r in range(ROUNDS)]


def _feistel(v, h, keys, inverse=False):
    mask = U((1 << h) - 1)
    L, R = v >> U(h), v & mask
    if not inverse:
        for k in keys:
            L, R = R, L ^ (smix(R ^ U(k)) & mask)
    else:
        for k in reversed(keys):
            L, R = R ^ (smix(L ^ U(k)) & mask), L
    return (L << U(h)) | R


def ref_pi(i, M, seed, inverse=False):
    """π(i) (or π⁻¹) of the indices i < M: the network, re-applied while the value is >= M"""
    h, keys = feistel_keys(M, seed)
    out = _feistel(np.asarray(i, np.uint64).reshape(-1), h, keys, inverse)
    todo = np.nonzero(out >= U(M))[0]
    while todo.size:
        out[todo] = _feistel(out[todo], h, keys, inverse)
        todo = todo[out[todo] >= U(M)]
    return out


def _in_sorted(sorted_set, c):
    if len(sorted_set) == 0:
        return np.zeros(len(c), bool)
    pos = np.searchsorted(sorted_set, c)
    return (pos < len(sorted_set)) & (sorted_set[np.minimum(pos, len(sorted_set) - 1)] == c)


def ref_sample_codes(M, excl, m, seed, chunk=1 << 20):
    """the first min(m, M - len(excl)) codes of π(0), π(1), ... that are not in excl, in that order"""
    excl = np.asarray(excl if excl is not None else [], np.uint64)
    want = min(int(m), int(M) - len(excl))
    out, got, base = [], 0, 0
    while got < want:
        i = np.arange(base, min(M, base + chunk), dtype=np.uint64)
        c = ref_pi(i, M, seed)
        c = c[~_in_sorted(excl, c)][:want - got]
        out.append(c)
        got += len(c)
        base += len(i)
    return np.concatenate(out) if out else np.empty(0, np.uint64)


def space_size(space, n, n2=None):
    return {D: n * n, DN: n * (n - 1), UD: n * (n + 1) // 2, UN: n * (n - 1) // 2, BP: n * (n2 or 0)}[space]


def ref_encode(space, n, n2, s, t):
    """0-based codes of 0-based pairs (uint64)"""
    s, t = np.asarray(s, np.uint64), np.asarray(t, np.uint64)
    n = U(n)
    if space == D:
        return s * n + t
    if space == DN:
        assert (s != t).all()
        return s * (n - U(1)) + t - (t > s).astype(np.uint64)
    if space in (UD, UN):
        lo, hi = np.minimum(s, t), np.maximum(s, t)
        a = U(2) * n + U(1) if space == UD else U(2) * n - U(1)
        if space == UN:
            assert (lo != hi).all()
        return lo * (a - lo) // U(2) + hi - lo - U(0 if space == UD else 1)
    return s * U(n2) + t


def ref_decode(space, n, n2, codes):
    """0-based pairs of 0-based codes, exact (Python integers, integer square roots)"""
    s_out, t_out = [], []
    for c in (int(v) for v in np.asarray(codes).reshape(-1)):
        if space == D:
            s, t = divmod(c, n)
        elif space == DN:
            s, r = divmod(c, n - 1)
            t = r + (r >= s)
        elif space == BP:
            s, t = divmod(c, n2)
        else:
            a, rows = (2 * n + 1, n) if space == UD else (2 * n - 1, n - 1)
            start = lambda r: r * (a - r) // 2  # noqa: E731
            s = (a - math.isqrt(a * a - 8 * c)) // 2
            while s + 1 < rows and start(s + 1) <= c:
                s += 1
            while start(s) > c:
                s -= 1
            t = s + (c - start(s)) + (0 if space == UD else 1)
        s_out.append(s)
        t_out.append(t)
    return np.array(s_out, np.int64), np.array(t_out, np.int64)


def codes_sorted(space, n, s, t):
    """distinct codes (ascending) of the 0-based pairs the space holds"""
    s, t = np.asarray(s, np.int64), np.asarray(t, np.int64)
    if space in (DN, UN):
        keep = s != t
        s, t = s[keep], t[keep]
    return np.unique(ref_encode(space, n, n, s, t))


# the four public functions composed from the statement (1-based ids in and out)
def ref_rand_graph(n, m, bidirected, seed):
    space = UN if bidirected else DN
    k = m // 2 if bidirected else m
    s, t = ref_decode(space, n, n, ref_sample_codes(space_size(space, n), None, k, seed))
    if bidirected:
        s, t = np.concatenate([s, t]), np.concatenate([t, s])
    return s + 1, t + 1


def ref_negative_sample(s, t, n, num_neg, bidirected, seed):
    space = UN if bidirected else DN
    excl = codes_sorted(space, n, np.asarray(s) - 1, np.asarray(t) - 1)
    codes = ref_sample_codes(space_size(space, n), excl, num_neg // 2 if bidirected else num_neg, seed)
    sn, tn = ref_decode(space, n, n, codes)
    if bidirected:
        sn, tn = np.concatenate([sn, tn]), np.concatenate([tn, sn])
    return sn + 1, tn + 1


def ref_rand_edge_split(s, t, frac, bidirected, seed):
    s, t = np.asarray(s), np.asarray(t)
    if bidirected:
        keep = s < t
        s, t = s[keep], t[keep]
    ne = len(s)
    eids = ref_sample_codes(ne, None, ne, seed).astype(np.int64)
    k = round(ne * frac)
    parts = []
    for e in (eids[:k], eids[k:]):
        a, b = s[e], t[e]
        parts.append((np.concatenate([a, b]), np.concatenate([b, a])) if bidirected else (a, b))
    return parts


def ref_perturb_edges(s, t, n, ratio, seed):
    k = math.ceil(len(s) * ratio)
    sn, tn = ref_decode(DN, n, n, ref_sample_codes(n * (n - 1), None, k, seed))
    return np.concatenate([s, sn + 1]), np.concatenate([t, tn + 1])


def ref_host_negative_sample(s, t, n, num_neg, rng):
    """numpy restatement of the reference's host algorithm (transform.jl:897-926, directed): self loops added as
    positives, randsubseq over 1:n² by Bernoulli draws, setdiff! against the positives, the first num_neg kept"""
    idx_pos = np.unique((np.concatenate([s, np.arange(1, n + 1)]) - 1) * n + np.concatenate([t, np.arange(1, n + 1)]))
    maxid = n * n
    pneg = 1 - len(idx_pos) / (2 * maxid)
    prob = min(1.0, num_neg / (pneg * maxid) * 1.1)
    rnd = np.nonzero(rng.random(maxid) < prob)[0] + 1
    neg = np.setdiff1d(rnd, idx_pos, assume_unique=True)[:num_neg]
    return (neg - 1) // n + 1, (neg - 1) % n + 1


# ---------------------------------------------------------------------------------------------- the C entries in numpy
def _fake_abi():
    sys.path.insert(0, os.path.join(ROOT, "tests"))
    import fake_abi
    return fake_abi


class FakeLink:
    """gnnb_edge_encode / _decode / _codes_sorted / gnnb_codes_member / gnnb_sample_codes on host pointers over the
    statement above; every other entry is the base double's."""

    def __init__(self, base):
        self.base, self.fa = base, _fake_abi()

    def __getattr__(self, name):
        return getattr(self.base, name)

    def _fail(self, code, msg):
        self.base._err = msg.encode()
        return code

    def _pairs(self, space, n1, n2, s, t, E, base):
        s = self.fa._arr(s, (E,), np.int64) - base
        t = self.fa._arr(t, (E,), np.int64) - base
        hi2 = n2 if space == BP else n1
        if ((s < 0) | (s >= n1) | (t < 0) | (t >= hi2)).any():
            return None, None
        return s, t

    def gnnb_edge_encode(self, space, n1, n2, s, t, E, base, codes, stream):
        if E == 0:
            return OK
        s, t = self._pairs(space, n1, n2, s, t, E, base)
        if s is None:
            return self._fail(EINDEX, "edge index outside the code space")
        if space in (DN, UN) and (s == t).any():
            return self._fail(EINDEX, "a self loop has no code in a space without self loops")
        self.fa._arr(codes, (E,), np.uint64)[...] = ref_encode(space, n1, n2, s, t)
        return OK

    def gnnb_edge_decode(self, space, n1, n2, codes, E, base, s, t, stream):
        if E == 0:
            return OK
        c = self.fa._arr(codes, (E,), np.uint64)
        if (c >= U(space_size(space, n1, n2))).any():
            return self._fail(EINDEX, "code outside the space")
        a, b = ref_decode(space, n1, n2, c)
        self.fa._arr(s, (E,), np.int64)[...] = a + base
        self.fa._arr(t, (E,), np.int64)[...] = b + base
        return OK

    def gnnb_edge_codes_sorted(self, space, n1, n2, s, t, E, base, out, n_out, stream):
        self.fa._deref(n_out).value = 0
        if E == 0:
            return OK
        s, t = self._pairs(space, n1, n2, s, t, E, base)
        if s is None:
            return self._fail(EINDEX, "edge index outside the code space")
        c = codes_sorted(space, n1, s, t)
        self.fa._arr(out, (E,), np.uint64)[:len(c)] = c
        self.fa._deref(n_out).value = len(c)
        return OK

    def gnnb_codes_member(self, codes, E, set_, x, flags, stream):
        if E == 0:
            return OK
        st = self.fa._arr(set_, (x,), np.uint64) if x else np.empty(0, np.uint64)
        self.fa._arr(flags, (E,), np.uint8)[...] = _in_sorted(st, self.fa._arr(codes, (E,), np.uint64))
        return OK

    def gnnb_sample_codes(self, M, excl, x, m, seed, out, n_out, stream):
        self.fa._deref(n_out).value = 0
        ex = self.fa._arr(excl, (x,), np.uint64) if x else np.empty(0, np.uint64)
        if x > M or (x and ((np.diff(ex.astype(np.float64)) <= 0).any() or ex[-1] >= U(M))):
            return self._fail(EINVAL, "excl must be ascending, distinct and below M")
        c = ref_sample_codes(M, ex, m, seed)
        if len(c):
            self.fa._arr(out, (len(c),), np.uint64)[...] = c
        self.fa._deref(n_out).value = len(c)
        return OK


@pytest.fixture(params=["fake", pytest.param("cuda", marks=pytest.mark.gpu)])
def lb(request, monkeypatch, gnn):
    """back end of the mirror: the numpy entries above (host tensors) or the CUDA kernels (device tensors)"""
    if request.param == "fake":
        from gnnb200 import linkpred
        with _fake_abi().installed() as fake:
            monkeypatch.setattr(linkpred, "lib", FakeLink(fake))
            yield torch.device("cpu")
    else:
        if not torch.cuda.is_available():
            pytest.skip("no CUDA device")
        yield torch.device("cuda")


def npy(x):
    return x.cpu().numpy()


def st(g):
    return npy(g.s), npy(g.t)


def pairs(g):
    return set(zip(*(v.tolist() for v in st(g))))


def u64(t):
    """int64 device codes -> uint64 numpy"""
    return npy(t).astype(np.uint64)


# ---------------------------------------------------------------------------------------------- the statement itself
@pytest.mark.parametrize("M", [1, 2, 3, 4, 5, 16, 17, 100, 1000, 4097, 65536])
def test_statement_pi_is_a_permutation_and_inverts(M):
    for seed in (0, 1, 2 ** 63 + 5):
        p = ref_pi(np.arange(M), M, seed)
        assert np.array_equal(np.sort(p), np.arange(M, dtype=np.uint64))
        assert np.array_equal(ref_pi(p, M, seed, inverse=True), np.arange(M, dtype=np.uint64))


def test_statement_sample_codes_properties():
    rng = np.random.default_rng(3)
    M = 5000
    excl = np.unique(rng.integers(0, M, 700)).astype(np.uint64)
    full = ref_sample_codes(M, excl, M, 11)
    assert len(full) == M - len(excl) and len(np.unique(full)) == len(full)
    assert not _in_sorted(excl, full).any()
    assert np.all(np.diff(ref_pi(full, M, 11, inverse=True).astype(np.int64)) > 0)   # π order
    for m in (0, 1, 10, 999):                                                          # first m = prefix
        assert np.array_equal(ref_sample_codes(M, excl, m, 11), full[:m])
    assert not np.array_equal(ref_sample_codes(M, excl, 50, 12), full[:50])
    assert len(ref_sample_codes(M, np.arange(M, dtype=np.uint64), 5, 1)) == 0


@pytest.mark.parametrize("space", SPACES)
def test_statement_encode_decode_round_trip(space):
    for n in (1, 2, 3, 7, 30):
        n2 = n + 3
        M = space_size(space, n, n2)
        c = np.arange(M, dtype=np.uint64)
        s, t = ref_decode(space, n, n2, c)
        assert np.array_equal(ref_encode(space, n, n2, s, t), c)
        if space in (UD, UN):
            assert (s <= t).all() and (space == UD or (s < t).all())
        if space == DN:
            assert (s != t).all()


# ---------------------------------------------------------------------------------------------- reference tests
def test_reference_edge_encoding_decoding(gnn, lb):
    """GNNGraphs/test/utils.jl:1-94"""
    n = 5
    s = torch.tensor([1, 1, 2, 3, 3, 4, 5], device=lb)
    t = torch.tensor([1, 3, 1, 1, 2, 5, 5], device=lb)
    idx, maxid = gnn.edge_encoding(s, t, n)
    assert maxid == n ** 2 and npy(idx).tolist() == [1, 3, 6, 11, 12, 20, 25]
    sd, td = gnn.edge_decoding(idx, n)
    assert torch.equal(sd.cpu(), s.cpu()) and torch.equal(td.cpu(), t.cpu())

    idx, maxid = gnn.edge_encoding(s, t, n, directed=False)
    assert maxid == n * (n + 1) // 2 and npy(idx).tolist() == [1, 3, 2, 3, 7, 14, 15]
    sd, td = gnn.edge_decoding(idx, n, directed=False)
    assert npy(sd).tolist() == np.minimum(npy(s), npy(t)).tolist()
    assert npy(td).tolist() == np.maximum(npy(s), npy(t)).tolist()

    g = gnn.rand_graph(10, 30, seed=1, device=lb)
    idx, _ = gnn.edge_encoding(g.s, g.t, 10)
    sd, td = gnn.edge_decoding(idx, 10)
    assert torch.equal(sd, g.s) and torch.equal(td, g.t)

    edges = [(1, 2), (3, 1), (1, 4), (1, 5), (2, 3), (2, 4), (2, 5), (3, 4), (3, 5), (4, 5)]
    s = torch.tensor([e[0] for e in edges], device=lb)
    t = torch.tensor([e[1] for e in edges], device=lb)
    idx, idxmax = gnn.edge_encoding(s, t, n, directed=False, self_loops=False)
    assert idxmax == n * (n - 1) // 2 and npy(idx).tolist() == list(range(1, idxmax + 1))
    sn, tn = gnn.edge_decoding(idx, n, directed=False, self_loops=False)
    assert npy(sn).tolist() == [1, 1, 1, 1, 2, 2, 2, 3, 3, 4] and npy(tn).tolist() == [2, 3, 4, 5, 3, 4, 5, 4, 5, 5]

    idx, idxmax = gnn.edge_encoding(s, t, n, directed=True, self_loops=False)
    assert idxmax == n ** 2 - n and npy(idx).tolist() == [1, 9, 3, 4, 6, 7, 8, 11, 12, 16]
    sn, tn = gnn.edge_decoding(idx, n, directed=True, self_loops=False)
    assert torch.equal(sn.cpu(), s.cpu()) and torch.equal(tn.cpu(), t.cpu())

    sb, tb = gnn.edge_decoding(torch.tensor([1, 6, 12], device=lb), 3, 4)      # bipartite: (s - 1) n2 + t
    assert npy(sb).tolist() == [1, 2, 3] and npy(tb).tolist() == [1, 2, 4]
    ib, mb = gnn.edge_encoding(sb, tb, 3, 4)
    assert mb == 12 and npy(ib).tolist() == [1, 6, 12]


def test_reference_rand_graph(gnn, lb):
    """GNNGraphs/test/generate.jl:1-37"""
    n, m = 10, 20
    m2 = m // 2
    x = torch.rand(3, n)
    e = torch.rand(4, m2)
    g = gnn.rand_graph(n, m, ndata=x, edata=e, seed=5, device=lb)
    assert g.num_nodes == n and g.num_edges == m
    assert g.ndata["x"] is x
    s, t = st(g)
    assert (s[:m2] == t[m2:]).all() and (t[:m2] == s[m2:]).all()
    assert torch.equal(g.edata["e"][:, :m2], e) and torch.equal(g.edata["e"][:, m2:], e)
    assert not (s == t).any() and len(pairs(g)) == m

    g = gnn.rand_graph(n, m, bidirected=False, seed=17, device=lb)
    assert g.num_nodes == n and g.num_edges == m and len(pairs(g)) == m and not (npy(g.s) == npy(g.t)).any()
    g2 = gnn.rand_graph(n, m, bidirected=False, seed=17, device=lb)
    assert torch.equal(g2.s, g.s) and torch.equal(g2.t, g.t)

    ew = torch.rand(m2)
    g = gnn.rand_graph(n, m, bidirected=True, edge_weight=ew, seed=17, device=lb)
    assert torch.equal(g.w.cpu(), torch.cat([ew, ew]))
    ew = torch.rand(m)
    g = gnn.rand_graph(n, m, bidirected=False, edge_weight=ew, seed=3, device=lb)
    assert torch.equal(g.w.cpu(), ew)


def test_reference_perturb_edges(gnn, lb):
    """GNNGraphs/test/transform.jl:187-193"""
    g = gnn.GNNGraph(torch.tensor([1, 2, 3, 4, 5], device=lb), torch.tensor([2, 3, 4, 5, 1], device=lb))
    g_per = gnn.perturb_edges(g, 0.5, seed=42)
    assert g_per.num_edges == 8
    s, t = st(g_per)
    assert (s[:5] == npy(g.s)).all() and (t[:5] == npy(g.t)).all()
    assert not (s[5:] == t[5:]).any() and len(set(zip(s[5:].tolist(), t[5:].tolist()))) == 3


def test_reference_negative_sample(gnn, lb):
    """GNNGraphs/test/transform.jl:324-334"""
    n, m = 10, 30
    g = gnn.rand_graph(n, m, bidirected=True, seed=2, device=lb)
    gneg = gnn.negative_sample(g, num_neg_edges=20, seed=9)
    assert gneg.num_nodes == g.num_nodes
    assert gneg.num_edges == 20
    assert gnn.is_bidirected(gneg)
    assert gnn.intersect(g, gneg).num_edges == 0


def test_reference_rand_edge_split(gnn, lb):
    """GNNGraphs/test/transform.jl:336-363"""
    n, m = 100, 300
    g = gnn.rand_graph(n, m, bidirected=True, seed=4, device=lb)
    g1, g2 = gnn.rand_edge_split(g, 0.9, seed=1)
    assert gnn.is_bidirected(g1) and gnn.is_bidirected(g2)
    assert gnn.intersect(g1, g2).num_edges == 0
    assert g1.num_edges + g2.num_edges == g.num_edges
    assert g2.num_edges < 50

    g = gnn.rand_graph(n, m, bidirected=False, seed=4, device=lb)
    for kw in ({}, {"bidirected": False}):
        g1, g2 = gnn.rand_edge_split(g, 0.9, seed=2, **kw)
        assert not gnn.is_bidirected(g1) and not gnn.is_bidirected(g2)
        assert gnn.intersect(g1, g2).num_edges == 0
        assert g1.num_edges + g2.num_edges == g.num_edges
        assert g2.num_edges < 50


# ---------------------------------------------------------------------------------------------- mirror logic
def test_public_functions_follow_the_statement(gnn, lb):
    """each public function is its numpy composition, id for id (on the GPU: the kernels against the statement)"""
    s, t = ref_rand_graph(40, 120, True, 8)
    g = gnn.rand_graph(40, 120, seed=8, device=lb)
    assert (npy(g.s) == s).all() and (npy(g.t) == t).all()
    s, t = ref_rand_graph(40, 77, False, 8)
    g = gnn.rand_graph(40, 77, bidirected=False, seed=8, device=lb)
    assert (npy(g.s) == s).all() and (npy(g.t) == t).all()

    rs, rt = np.random.default_rng(0).integers(1, 65, 500), np.random.default_rng(1).integers(1, 65, 500)
    g = gnn.GNNGraph(torch.as_tensor(rs).to(lb), torch.as_tensor(rt).to(lb), num_nodes=64)
    for bid in (True, False):
        for num in (0, 1, 101, 5000):
            es, et = ref_negative_sample(rs, rt, 64, num, bid, 21)
            gn = gnn.negative_sample(g, num_neg_edges=num, bidirected=bid, seed=21)
            assert (npy(gn.s) == es).all() and (npy(gn.t) == et).all()
    gp = gnn.perturb_edges(g, 0.3, seed=6)
    es, et = ref_perturb_edges(rs, rt, 64, 0.3, 6)
    assert (npy(gp.s) == es).all() and (npy(gp.t) == et).all()

    gb = gnn.rand_graph(50, 400, seed=1, device=lb)
    bs, bt = st(gb)
    for bid, frac in ((True, 0.25), (False, 0.7), (False, 0.0), (True, 1.0)):
        (s1, t1), (s2, t2) = ref_rand_edge_split(bs, bt, frac, bid, 13)
        g1, g2 = gnn.rand_edge_split(gb, frac, bidirected=bid, seed=13)
        assert (npy(g1.s) == s1).all() and (npy(g1.t) == t1).all()
        assert (npy(g2.s) == s2).all() and (npy(g2.t) == t2).all()


def test_negative_sample_excludes_positives_and_counts(gnn, lb):
    g = gnn.GNNGraph(torch.tensor([1, 2, 2, 3, 4, 4], device=lb), torch.tensor([2, 1, 3, 3, 1, 1], device=lb),
                     num_nodes=4)
    pos = {(int(a), int(b)) for a, b in zip(*st(g))}
    gd = gnn.negative_sample(g, num_neg_edges=100, bidirected=False, seed=1)   # 12 ordered non-loop pairs, 4 taken
    assert sorted(pairs(gd)) == sorted({(a, b) for a in range(1, 5) for b in range(1, 5) if a != b} - pos)
    assert gd.num_edges == 8
    gu = gnn.negative_sample(g, num_neg_edges=100, bidirected=True, seed=1)    # 6 unordered pairs, {1,2},{2,3},{1,4}
    und = {(min(a, b), max(a, b)) for a, b in pos if a != b}
    assert {(a, b) for a, b in pairs(gu) if a < b} == {(a, b) for a in range(1, 5) for b in range(a + 1, 5)} - und
    assert gu.num_edges == 6
    assert gnn.negative_sample(g, num_neg_edges=3, bidirected=True, seed=1).num_edges == 2   # num_neg ÷ 2 pairs


def test_add_edges_and_intersect(gnn, lb):
    """transform.jl:319-353 (weights padded with ones on either side) and operators.jl:7-20 (g1's order, once)"""
    s, t, w = torch.tensor([1, 2, 3]), torch.tensor([2, 3, 1]), torch.tensor([0.5, 1.5, 2.5])
    g = gnn.GNNGraph(s.to(lb), t.to(lb), w.to(lb), num_nodes=3)
    g2 = gnn.add_edges(g, (torch.tensor([2, 3]), torch.tensor([4, 1]), torch.tensor([10.0, 20.0])))
    assert g2.num_nodes == 4 and g2.num_edges == 5
    assert npy(g2.w).tolist() == [0.5, 1.5, 2.5, 10.0, 20.0] and npy(g2.s).tolist() == [1, 2, 3, 2, 3]
    g3 = gnn.add_edges(g, [1, 1], [1, 2])
    assert npy(g3.w).tolist() == [0.5, 1.5, 2.5, 1.0, 1.0]
    g4 = gnn.add_edges(gnn.GNNGraph(s.to(lb), t.to(lb), num_nodes=3), (s[:1], t[:1], torch.tensor([7.0])))
    assert npy(g4.w).tolist() == [1.0, 1.0, 1.0, 7.0]
    e = torch.arange(3.0).reshape(1, 3)
    ge = gnn.GNNGraph(s.to(lb), t.to(lb), num_nodes=3, edata={"e": e.to(lb)})
    assert npy(gnn.add_edges(ge, [3], [3], edata=torch.tensor([[9.0]])).edata["e"]).tolist() == [[0, 1, 2, 9]]
    with pytest.raises(AssertionError):
        gnn.add_edges(ge, [3], [3])
    assert gnn.add_edges(g, torch.tensor([], dtype=torch.int64), torch.tensor([], dtype=torch.int64)) is g

    a = gnn.GNNGraph(torch.tensor([3, 1, 2, 1, 3], device=lb), torch.tensor([1, 2, 2, 2, 2], device=lb), num_nodes=3)
    b = gnn.GNNGraph(torch.tensor([2, 1, 3, 3], device=lb), torch.tensor([2, 2, 1, 3], device=lb), num_nodes=3)
    i = gnn.intersect(a, b)
    assert i.num_nodes == 3 and list(zip(*(x.tolist() for x in st(i)))) == [(3, 1), (1, 2), (2, 2)]
    assert gnn.intersect(a, gnn.GNNGraph(torch.tensor([], dtype=torch.int64, device=lb),
                                         torch.tensor([], dtype=torch.int64, device=lb), num_nodes=3)).num_edges == 0


def test_dot_decoder(gnn, lb):
    """GNNlib/src/layers/basic.jl:1-3 and DotDecoder (GraphNeuralNetworks/src/layers/basic.jl:187-212)"""
    g = gnn.GNNGraph(torch.tensor([1, 1, 2, 5], device=lb), torch.tensor([2, 3, 3, 4], device=lb), num_nodes=5)
    x = torch.randn(2, 5, device=lb)
    want = (x[:, g.s - 1] * x[:, g.t - 1]).sum(0, keepdim=True)
    assert torch.allclose(gnn.dot_decoder(g, x), want, rtol=1e-6, atol=1e-6)
    assert torch.allclose(gnn.DotDecoder()(g, x), want, rtol=1e-6, atol=1e-6)


def test_argument_errors(gnn, lb):
    with pytest.raises(AssertionError, match="even"):
        gnn.rand_graph(10, 7, device=lb)
    with pytest.raises(AssertionError):
        gnn.rand_graph(4, 14, device=lb)                        # 6 pairs exist, 7 asked
    with pytest.raises(AssertionError):
        gnn.rand_graph(4, 13, bidirected=False, device=lb)      # 12 ordered pairs exist
    g = gnn.rand_graph(10, 20, seed=1, device=lb)
    for bad in (-0.1, 1.5):
        with pytest.raises(AssertionError):
            gnn.rand_edge_split(g, bad)
        with pytest.raises(AssertionError):
            gnn.perturb_edges(g, bad)
    one = gnn.GNNGraph(torch.tensor([1], device=lb), torch.tensor([1], device=lb), num_nodes=1)
    with pytest.raises(AssertionError):
        gnn.negative_sample(one)
    with pytest.raises(AssertionError):
        gnn.perturb_edges(one, 1.0)
    with pytest.raises(AssertionError):
        gnn.edge_encoding(torch.tensor([1]), torch.tensor([1]), 3, self_loops=False)
    with pytest.raises(AssertionError):
        gnn.edge_encoding(torch.tensor([1]), torch.tensor([4]), 3)
    with pytest.raises(AssertionError):
        gnn.edge_decoding(torch.tensor([10]), 3)                 # maxid = 9
    loops = gnn.GNNGraph(torch.tensor([1, 2, 1], device=lb), torch.tensor([2, 1, 1], device=lb), num_nodes=2)
    with pytest.raises(AssertionError, match="self loops"):
        gnn.rand_edge_split(loops, 0.5, bidirected=True)
    from gnnb200 import linkpred
    with pytest.raises(ValueError):                              # an exclusion set that is not ascending
        linkpred.sample_codes(10, 3, exclude=torch.tensor([5, 2], device=lb), device=lb)


def test_per_code_inclusion_is_uniform(gnn, lb):
    """every available unordered pair of a 64-node graph is a bidirected negative equally often over 2 000 seeds
    (chi-square at p = 1e-6); the graph's own pairs never are"""
    from scipy.stats import chi2
    n, seeds, k = 64, 2000, 120
    rs, rt = ref_rand_graph(n, 400, True, 77)
    g = gnn.GNNGraph(torch.as_tensor(rs).to(lb), torch.as_tensor(rt).to(lb), num_nodes=n)
    M = n * (n - 1) // 2
    excl = codes_sorted(UN, n, rs - 1, rt - 1)
    counts = np.zeros(M, np.int64)
    for seed in range(seeds):
        gn = gnn.negative_sample(g, num_neg_edges=2 * k, bidirected=True, seed=seed)
        s, t = st(gn)
        np.add.at(counts, ref_encode(UN, n, n, s[:k] - 1, t[:k] - 1).astype(np.int64), 1)
    assert counts[excl.astype(np.int64)].sum() == 0
    avail = np.setdiff1d(np.arange(M), excl.astype(np.int64))
    exp = seeds * k / len(avail)
    stat = ((counts[avail] - exp) ** 2 / exp).sum()
    assert stat < chi2.isf(1e-6, len(avail) - 1), stat


def _decile_chi2(s, n, s_pos, t_pos):
    """chi-square of the negatives' source-id deciles against the exact share of directed non-loop non-edges"""
    from scipy.stats import chi2
    dec = lambda v: (np.asarray(v, np.int64) - 1) * 10 // n  # noqa: E731
    sizes = np.bincount(dec(np.arange(1, n + 1)), minlength=10)
    keep = s_pos != t_pos
    pos = np.unique((s_pos[keep] - 1) * n + (t_pos[keep] - 1))
    avail = sizes * (n - 1) - np.bincount(dec(pos // n + 1), minlength=10)
    obs = np.bincount(dec(s), minlength=10)
    exp = len(s) * avail / avail.sum()
    return ((obs - exp) ** 2 / exp).sum(), chi2.isf(1e-6, 9)


def test_source_deciles_reference_algorithm_is_biased_statement_is_not():
    """the decile test of the at-scale GPU test, on a small graph: the reference's host algorithm (truncation of an
    ascending list) fails it; the statement's sample passes"""
    rng = np.random.default_rng(5)
    n, E = 3000, 30000
    s, t = rng.integers(1, n + 1, E), rng.integers(1, n + 1, E)
    hs, _ = ref_host_negative_sample(s, t, n, E, np.random.default_rng(6))
    stat, bar = _decile_chi2(hs, n, s, t)
    assert stat > 10 * bar
    ns, _ = ref_negative_sample(s, t, n, E, False, 6)
    stat, bar = _decile_chi2(ns, n, s, t)
    assert stat < bar


# ---------------------------------------------------------------------------------------------- kernels == statement
def _dev_i64(a):
    return torch.as_tensor(np.asarray(a, np.uint64).astype(np.int64)).cuda()


@pytest.mark.gpu
@pytest.mark.parametrize("space", SPACES)
def test_gpu_encode_decode_exhaustive(gnn, space):
    from gnnb200 import linkpred
    dev = torch.device("cuda")
    for n in list(range(1, 65)):
        n2 = (n * 7) % 64 + 1
        M = space_size(space, n, n2)
        if M == 0:
            continue
        codes = torch.arange(M, dtype=torch.int64, device=dev)
        s, t = linkpred._decode(space, n, n2, codes, dev)
        es, et = ref_decode(space, n, n2, np.arange(M))
        assert (npy(s) == es + 1).all() and (npy(t) == et + 1).all(), n
        assert torch.equal(linkpred._encode(space, n, n2, s, t, dev), codes)
        if space in (UD, UN):                            # an unordered pair has one code in either orientation
            assert torch.equal(linkpred._encode(space, n, n2, t, s, dev), codes)


@pytest.mark.gpu
@pytest.mark.parametrize("space", SPACES)
def test_gpu_decode_at_n_2_31_minus_1(gnn, space):
    from gnnb200 import linkpred
    dev = torch.device("cuda")
    n = n2 = 2 ** 31 - 1
    M = space_size(space, n, n2)
    rng = np.random.default_rng(space)
    codes = [0, 1, M - 1, M - 2, M // 2] + [int(v) for v in rng.integers(0, M, 20000, dtype=np.uint64)]
    if space in (UD, UN):                                # every row start and end near the last rows and the first
        a = 2 * n + 1 if space == UD else 2 * n - 1
        for r in list(range(0, 50)) + list(range(n - 60, n - (0 if space == UD else 1))):
            st_ = r * (a - r) // 2
            codes += [st_, max(st_ - 1, 0)]
    codes = np.array(sorted(set(codes)), np.uint64)
    s, t = linkpred._decode(space, n, n2, _dev_i64(codes), dev)
    es, et = ref_decode(space, n, n2, codes)
    assert (npy(s) == es + 1).all() and (npy(t) == et + 1).all()
    assert (u64(linkpred._encode(space, n, n2, s, t, dev)) == codes).all()


def _excl_sets(M, rng):
    """name -> sorted exclusion codes (device int64) for the sample_codes sweep"""
    dev = torch.device("cuda")
    out = {"empty": None}
    k = min(M // 3, 20000)
    out["sparse"] = torch.unique(torch.as_tensor(rng.integers(0, M, k, dtype=np.int64)).cuda()) if k else None
    keep = np.unique(rng.integers(0, M, min(M, 5), dtype=np.int64))
    mask = torch.ones(M, dtype=torch.bool, device=dev)
    mask[torch.as_tensor(keep).cuda()] = False
    out["all_but_few"] = torch.nonzero(mask).reshape(-1)
    del mask
    out["all"] = torch.arange(M, dtype=torch.int64, device=dev)
    return out, keep


@pytest.mark.gpu
@pytest.mark.parametrize("M", [1, 2, 3, 4, 5, 17, 1000, 4096, 4097, 65537, 10 ** 6, 2 ** 24 + 3, 10 ** 9])
def test_gpu_sample_codes_equals_statement(gnn, M):
    from gnnb200 import linkpred
    rng = np.random.default_rng(M % 1000)
    sets, keep = _excl_sets(M, rng)
    for name, excl in sets.items():
        x = 0 if excl is None else int(excl.numel())
        for m in sorted({1, 7, min(M, 100000), M} if M <= 10 ** 6 else {1, 7, 100000}):
            seed = 1000 * M + m
            got = linkpred.sample_codes(M, m, exclude=excl, seed=seed, device="cuda")
            assert got.numel() == min(m, M - x), (name, m)
            if name in ("all_but_few", "all"):
                # exactly the remaining codes come back, in π order (the statement through π⁻¹: no 10⁹-entry set on
                # the host)
                rest = keep if name == "all_but_few" else np.empty(0, np.int64)
                want = rest[np.argsort(ref_pi(rest, M, seed, inverse=True))][:m].astype(np.uint64)
            else:
                ex = np.empty(0, np.uint64) if excl is None else u64(excl)
                want = ref_sample_codes(M, ex, m, seed)
            assert np.array_equal(u64(got), want), (name, m)
    del sets
    torch.cuda.empty_cache()


@pytest.mark.gpu
def test_gpu_codes_sorted_and_member(gnn):
    from gnnb200 import linkpred
    dev = torch.device("cuda")
    rng = np.random.default_rng(9)
    n = 1000
    s, t = rng.integers(1, n + 1, 200000), rng.integers(1, n + 1, 200000)
    s[:50] = t[:50]                                                      # self loops: skipped in the NOLOOP spaces
    S, T = torch.as_tensor(s).cuda(), torch.as_tensor(t).cuda()
    for space in (D, DN, UD, UN):
        got = linkpred._codes_sorted(space, n, S, T, dev)
        assert np.array_equal(u64(got), codes_sorted(space, n, s - 1, t - 1)), space
        probe = torch.as_tensor(rng.integers(0, space_size(space, n), 50000, dtype=np.int64)).cuda()
        flags = linkpred._member(probe, got, dev)
        assert np.array_equal(npy(flags), _in_sorted(u64(got), u64(probe)))


# ---------------------------------------------------------------------------------------------- at scale
@pytest.fixture(scope="module")
def rmat_10m(gnn):
    if not torch.cuda.is_available():
        pytest.skip("no CUDA device")
    g = gnn.rmat_graph(10_000_000, 100_000_000, seed=11, device="cuda")
    yield g
    del g
    torch.cuda.empty_cache()


def _sorted_codes_torch(a, b, n):
    return torch.unique(a.long() * n + b.long())


@pytest.mark.gpu
def test_gpu_negative_sample_at_scale(gnn, rmat_10m):
    g = rmat_10m
    n, E = g.num_nodes, g.num_edges
    gn = gnn.negative_sample(g, num_neg_edges=E, bidirected=True, seed=123)
    assert gn.num_edges == E and gn.num_nodes == n
    h = E // 2
    s, t = gn.s, gn.t
    assert torch.equal(s[:h], t[h:]) and torch.equal(t[:h], s[h:])          # bidirected symmetry
    assert not bool((s == t).any())
    pos = torch.unique(torch.cat([_sorted_codes_torch(g.s - 1, g.t - 1, n), _sorted_codes_torch(g.t - 1, g.s - 1, n)]))
    neg = (s - 1) * n + (t - 1)
    i = torch.searchsorted(pos, neg).clamp_(max=pos.numel() - 1)
    assert not bool((pos[i] == neg).any())                                    # no positive among the negatives
    assert torch.unique(neg).numel() == E                                     # all pairs distinct
    del pos, neg, i
    again = gnn.negative_sample(g, num_neg_edges=E, bidirected=True, seed=123)
    assert torch.equal(again.s, s) and torch.equal(again.t, t)
    other = gnn.negative_sample(g, num_neg_edges=E, bidirected=True, seed=124)
    assert not torch.equal(other.s, s)


@pytest.mark.gpu
def test_gpu_negative_sources_uniform_over_deciles(gnn, rmat_10m):
    """chi-square over source-id deciles at N = 10 M (the test the reference's truncation bias fails)"""
    g = rmat_10m
    n, E = g.num_nodes, g.num_edges
    gn = gnn.negative_sample(g, num_neg_edges=E, bidirected=False, seed=5)
    assert gn.num_edges == E
    dec = lambda v: torch.bincount((v.long() - 1) * 10 // n, minlength=10).double()  # noqa: E731
    sizes = dec(torch.arange(1, n + 1, device="cuda"))
    keep = g.s != g.t
    pos = _sorted_codes_torch(g.s[keep] - 1, g.t[keep] - 1, n)
    avail = sizes * (n - 1) - dec(pos // n + 1)
    exp = E * avail / avail.sum()
    stat = float((((dec(gn.s) - exp) ** 2) / exp).sum())
    from scipy.stats import chi2
    assert stat < chi2.isf(1e-6, 9), stat
