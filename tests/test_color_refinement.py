"""color_refinement (graphneuralnetworks.jl_b200/transform.py over csrc/wl.cu's gnnb_color_refinement;
GNNGraphs/src/utils.jl:340-389).

The contract, stated below in numpy (`ref_color_refinement`): round r maps node i to its signature
(c_i, tuple(sorted(c[s] for the edges s -> i))), grouped exactly as Python tuples — no hashing; colours are numbered
1..k in order of first appearance by node id, afresh every round; the rounds stop when one leaves the number of classes
unchanged, or after max_iters; niters counts the last round; an empty graph gives (empty, 0, 1).

Back ends of the mirror: `FakeWL`, the C entry restated on host pointers over that statement (swapped in over
tests/fake_abi.py's double), and, under -m gpu, the CUDA kernels, which must return exactly (==) the statement's output.
"""
import ctypes as C
import os
import sys
from types import SimpleNamespace

import numpy as np
import pytest
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
OK, EINVAL, ESIZE, ECUDA, ENOMEM, EUNSUPPORTED, EINDEX = range(7)


# ---------------------------------------------------------------------------------------------- the contract in numpy
def _first_appearance(sigs):
    ids = {}
    return np.array([ids.setdefault(x, len(ids) + 1) for x in sigs], np.int64), len(ids)


def ref_color_refinement(s, t, n, x0=None, max_iters=None):
    """(x, num_colors, niters): x 1-based int64.  s, t 0-based; the signature of i is (c_i, sorted in-neighbour
    colours) as a Python tuple."""
    s, t = np.asarray(s, np.int64), np.asarray(t, np.int64)
    if n == 0:
        return np.zeros(0, np.int64), 0, 1
    c, k = _first_appearance([0] * n if x0 is None else [int(v) for v in x0])
    rowptr = np.concatenate([[0], np.cumsum(np.bincount(t, minlength=n))])
    niters = 0
    while True:
        niters += 1
        order = np.lexsort((c[s], t))                     # by target, then by the source's colour
        cs = c[s][order].tolist()
        c2, k2 = _first_appearance([(int(c[i]), tuple(cs[rowptr[i]:rowptr[i + 1]])) for i in range(n)])
        stable = k2 == k
        c, k = c2, k2
        if stable or niters == max_iters:
            return c, k, niters


# ---------------------------------------------------------------------------------------------- the C entry in numpy
def _fake_abi():
    sys.path.insert(0, os.path.join(ROOT, "tests"))
    import fake_abi
    return fake_abi


class FakeWL:
    """gnnb_color_refinement on host pointers over `ref_color_refinement`; every other entry is the base double's"""

    def __init__(self, base):
        self.base, self.fa = base, _fake_abi()

    def __getattr__(self, name):
        return getattr(self.base, name)

    def _fail(self, code, msg):
        self.base._err = msg.encode()
        return code

    def gnnb_color_refinement(self, h, x0, max_iters, colors, num_colors, niters, stream):
        self.base.calls.append("gnnb_color_refinement")
        p = self.base._p(h)
        if p.ns != p.nd:
            return self._fail(ESIZE, "needs num_src == num_dst")
        if max_iters < 0:
            return self._fail(EINVAL, "max_iters must be >= 0")
        n = p.nd
        x = None if x0 is None or n == 0 else self.fa._arr(x0, (n,), np.int64).copy()
        c, k, it = ref_color_refinement(p.s, p.t, n, x, max_iters or None)
        if n:
            self.fa._arr(colors, (n,), np.int64)[...] = c
        self.fa._deref(num_colors).value = k
        self.fa._deref(niters).value = it
        return OK


@pytest.fixture(params=["fake", pytest.param("cuda", marks=pytest.mark.gpu)])
def wb(request, gnn):
    """back end of the mirror: .dev, and .fake (the FakeWL in use, None on cuda)"""
    if request.param == "fake":
        from gnnb200 import transform
        with _fake_abi().installed() as fake:
            saved = transform.lib
            transform.lib = FakeWL(fake)
            try:
                yield SimpleNamespace(dev=torch.device("cpu"), fake=transform.lib)
            finally:
                transform.lib = saved
    else:
        if not torch.cuda.is_available():
            pytest.skip("no CUDA device")
        yield SimpleNamespace(dev=torch.device("cuda"), fake=None)


def npy(x):
    return x.cpu().numpy()


def graph(gnn, s, t, n, dev):
    s, t = np.asarray(s, np.int64), np.asarray(t, np.int64)
    return gnn.GNNGraph(torch.as_tensor(s + 1, device=dev), torch.as_tensor(t + 1, device=dev), num_nodes=n)


def undirected(s, t):
    s, t = np.asarray(s, np.int64), np.asarray(t, np.int64)
    return np.concatenate([s, t]), np.concatenate([t, s])


def batch_of(parts):
    """(s, t, n) of the disjoint union of parts [(s, t, n)]"""
    S, T, off = [], [], 0
    for s, t, n in parts:
        S.append(np.asarray(s, np.int64) + off)
        T.append(np.asarray(t, np.int64) + off)
        off += n
    return np.concatenate(S), np.concatenate(T), off


def path(n):
    return (*undirected(np.arange(n - 1), np.arange(1, n)), n)


def cycle(n):
    return (*undirected(np.arange(n), (np.arange(n) + 1) % n), n)


def run(gnn, s, t, n, dev, x0=None, **kw):
    x, k, it = gnn.color_refinement(graph(gnn, s, t, n, dev), x0, **kw)
    assert x.dtype == torch.int64 and x.shape == (n,) and x.device.type == torch.device(dev).type
    assert isinstance(k, int) and isinstance(it, int)
    return npy(x), k, it


def assert_same(got, ref):
    assert got[1:] == ref[1:] and np.array_equal(got[0], ref[0]), (got[1:], ref[1:])


# ---------------------------------------------------------------------------------------------- known answers
def _known():
    star = (*undirected([0, 0, 0], [1, 2, 3]), 4)
    return {
        "path_P5": (path(5), [1, 2, 3, 2, 1], 3, 3),
        "directed_path_3": (([0, 1], [1, 2], 3), [1, 2, 3], 3, 3),
        "C6_with_two_C3": (batch_of([cycle(6), cycle(3), cycle(3)]), [1] * 12, 1, 1),
        "star_K13_with_P4": (batch_of([star, path(4)]), [1, 2, 2, 2, 3, 4, 4, 3], 4, 3),
    }


KNOWN = _known()


@pytest.mark.parametrize("name", list(KNOWN))
def test_statement_known_answers(name):
    (s, t, n), x, k, it = KNOWN[name]
    got = ref_color_refinement(s, t, n)
    assert got[0].tolist() == x and got[1:] == (k, it)


@pytest.mark.parametrize("name", list(KNOWN))
def test_known_answers(gnn, wb, name):
    (s, t, n), x, k, it = KNOWN[name]
    got = run(gnn, s, t, n, wb.dev)
    assert got[0].tolist() == x and got[1:] == (k, it)


def test_wl_cannot_separate_c6_from_two_c3_but_separates_star_from_p4(gnn, wb):
    (s, t, n), *_ = KNOWN["C6_with_two_C3"]
    x, _, _ = run(gnn, s, t, n, wb.dev)
    assert np.array_equal(np.bincount(x[:6]), np.bincount(x[6:]))
    (s, t, n), *_ = KNOWN["star_K13_with_P4"]
    x, _, _ = run(gnn, s, t, n, wb.dev)
    assert not np.array_equal(np.bincount(x[:4], minlength=5), np.bincount(x[4:], minlength=5))


# ---------------------------------------------------------------------------------------------- contract cases
def rand_graph(rng, n, e):
    return rng.integers(0, n, e), rng.integers(0, n, e)


def test_reference_test_shape(gnn, wb):
    """GNNGraphs/test/utils.jl:96-107: color_refinement(g) == color_refinement(g, ones)"""
    s, t = rand_graph(np.random.default_rng(1), 10, 20)
    a = run(gnn, s, t, 10, wb.dev)
    b = run(gnn, s, t, 10, wb.dev, torch.ones(10, dtype=torch.int64, device=wb.dev))
    assert_same(a, b)
    assert_same(a, ref_color_refinement(s, t, 10))


def test_x0_only_its_partition_matters(gnn, wb):
    rng = np.random.default_rng(2)
    n = 40
    s, t = rand_graph(rng, n, 90)
    x0 = rng.integers(0, 5, n)
    relabel = np.array([-(2 ** 62), -7, 3, 2 ** 40 + 1, 2 ** 62 + 5], np.int64)   # injective, negative and >= 2^40
    a = run(gnn, s, t, n, wb.dev, torch.as_tensor(x0, device=wb.dev))
    b = run(gnn, s, t, n, wb.dev, torch.as_tensor(relabel[x0], device=wb.dev))
    assert_same(a, b)
    assert_same(a, ref_color_refinement(s, t, n, x0))
    c = run(gnn, s, t, n, wb.dev, x0.tolist())                                    # a list works as well
    assert_same(a, c)


def test_multi_edges_and_self_loops_count(gnn, wb):
    # nodes 1 and 2 both hear node 0; a second 0 -> 2 edge, or a self loop on 2, sets node 2 apart
    base_s, base_t = [0, 0], [1, 2]
    x, k, _ = run(gnn, base_s, base_t, 3, wb.dev)
    assert x[1] == x[2]
    for s, t in (([0, 0, 0], [1, 2, 2]), ([0, 0, 2], [1, 2, 2])):
        got = run(gnn, s, t, 3, wb.dev)
        assert got[0][1] != got[0][2]
        assert_same(got, ref_color_refinement(s, t, 3))


@pytest.mark.parametrize("max_iters", [1, 2, 3])
def test_max_iters_against_statement(gnn, wb, max_iters):
    rng = np.random.default_rng(3)
    s, t, n = path(12)
    s2, t2 = rand_graph(rng, 30, 50)
    s, t, n = batch_of([(s, t, n), (s2, t2, 30)])
    got = run(gnn, s, t, n, wb.dev, max_iters=max_iters)
    assert_same(got, ref_color_refinement(s, t, n, None, max_iters))
    assert got[2] == max_iters                                      # a path of 12 needs more than three rounds
    full = ref_color_refinement(s, t, n)
    assert full[2] > 3


def test_empty_graph(gnn, wb):
    e = torch.zeros(0, dtype=torch.int64, device=wb.dev)
    x, k, it = gnn.color_refinement(gnn.GNNGraph(e, e, num_nodes=0))
    assert x.shape == (0,) and x.dtype == torch.int64 and (k, it) == (0, 1)


def test_graph_without_edges(gnn, wb):
    x, k, it = run(gnn, [], [], 5, wb.dev)
    assert x.tolist() == [1] * 5 and (k, it) == (1, 1)
    x, k, it = run(gnn, [], [], 5, wb.dev, torch.tensor([9, -1, 9, 4, -1], device=wb.dev))
    assert x.tolist() == [1, 2, 1, 3, 2] and (k, it) == (3, 1)


def test_permuted_copy_batched_with_original(gnn, wb):
    rng = np.random.default_rng(4)
    n = 50
    s, t = rand_graph(rng, n, 120)
    pi = rng.permutation(n)
    S, T, N = batch_of([(s, t, n), (pi[s], pi[t], n)])
    x, k, it = run(gnn, S, T, N, wb.dev)
    assert np.array_equal(x[:n], x[n:][pi])
    assert_same((x, k, it), ref_color_refinement(S, T, N))


def test_argument_errors(gnn, wb):
    g = graph(gnn, [0, 1], [1, 2], 3, wb.dev)
    for bad in (0, -1, 1.5, True, "2"):
        with pytest.raises(AssertionError):
            gnn.color_refinement(g, max_iters=bad)
    with pytest.raises(AssertionError):
        gnn.color_refinement(g, torch.ones(4, dtype=torch.int64))
    with pytest.raises(AssertionError):
        gnn.color_refinement(g, torch.ones(3))
    with pytest.raises(AssertionError):
        gnn.color_refinement(g, torch.ones(3, 1, dtype=torch.int64))


def test_fake_entry_rejects_what_the_c_entry_rejects(gnn):
    from gnnb200 import _lib
    with _fake_abi().installed() as fake:
        wl = FakeWL(fake)
        s = torch.tensor([0, 1], dtype=torch.int64)
        h = C.c_void_p()
        fake.gnnb_graph_create(C.byref(h), s.data_ptr(), s.data_ptr(), 2, 3, 2, 8, 0, 0, None)
        k, it = C.c_int64(0), C.c_int64(0)
        out = torch.empty(2, dtype=torch.int64)
        assert wl.gnnb_color_refinement(h, None, 0, out.data_ptr(), C.byref(k), C.byref(it), None) == ESIZE
        fake.gnnb_graph_create(C.byref(h), s.data_ptr(), s.data_ptr(), 2, 2, 2, 8, 0, 0, None)
        assert wl.gnnb_color_refinement(h, None, -1, out.data_ptr(), C.byref(k), C.byref(it), None) == EINVAL
    assert _lib.EINVAL == EINVAL and _lib.ESIZE == ESIZE


# ---------------------------------------------------------------------------------------------- GPU: exact and at scale
def cuda_run(gnn, g, x0=None, **kw):
    x, k, it = gnn.color_refinement(g, x0, **kw)
    return npy(x), k, it


def with_chunk(gnn, chunk, s, t, n):
    """a CUDA graph whose plan is built at `chunk` edges per work chunk"""
    try:
        gnn._lib.check(gnn._lib.lib.gnnb_set_chunk_edges(chunk))
        g = gnn.GNNGraph(torch.as_tensor(np.asarray(s, np.int64) + 1, device="cuda"),
                         torch.as_tensor(np.asarray(t, np.int64) + 1, device="cuda"), num_nodes=n)
        g.plan()
    finally:
        gnn._lib.lib.gnnb_set_chunk_edges(128)
    return g


@pytest.mark.gpu
@pytest.mark.parametrize("seed", [0, 1, 2])
def test_gpu_random_graphs_equal_statement(gnn, seed):
    rng = np.random.default_rng(100 + seed)
    n = int(rng.integers(50, 3000))
    s, t = rand_graph(rng, n, int(rng.integers(n, 6 * n)))
    if seed == 2:
        s, t = undirected(s, t)
    assert_same(run(gnn, s, t, n, "cuda"), ref_color_refinement(s, t, n))
    x0 = rng.integers(0, 3, n)
    assert_same(run(gnn, s, t, n, "cuda", torch.as_tensor(x0, device="cuda")), ref_color_refinement(s, t, n, x0))


def chunk_boundary_graph(C, seed=0):
    """configuration-model graph (random sources) whose in-degree sequence puts rows of C, C + 1, 2C and 2C + 1 edges
    on chunk boundaries of C edges: starting on one, ending on one, or both, with short rows between"""
    rng = np.random.default_rng(seed)
    long_degs = [C, C, C + 1, C - 1, 2 * C, 2 * C + 1, C - 1, 2 * C, C + 1, C - 1, 2 * C + 1, 2 * C - 1, C]
    degs = list(long_degs) + list(rng.integers(0, 6, 400))
    degs += [2 * C + 1, C + 1, 2 * C]                                 # and rows at the very end of the edge list
    n = len(degs) + 200                                               # 200 nodes without in-edges
    t = np.repeat(np.arange(len(degs)), degs)
    s = rng.integers(0, n, len(t))
    perm = rng.permutation(len(t))                                    # COO order is not plan order
    return s[perm], t[perm], n


@pytest.mark.gpu
@pytest.mark.parametrize("C", [128, 32])
def test_gpu_chunk_boundary_rows(gnn, C):
    s, t, n = chunk_boundary_graph(C)
    ref = ref_color_refinement(s, t, n)
    got = cuda_run(gnn, with_chunk(gnn, C, s, t, n))
    assert_same(got, ref)
    other = cuda_run(gnn, with_chunk(gnn, 160 - C, s, t, n))          # 32 <-> 128: the same bits
    assert_same(other, got)
    x0 = np.arange(n) % 3
    assert_same(cuda_run(gnn, with_chunk(gnn, C, s, t, n), torch.as_tensor(x0, device="cuda")),
                ref_color_refinement(s, t, n, x0))


@pytest.mark.gpu
def test_gpu_hub_rows(gnn):
    """three hubs with 10^5 in-edges each: hundreds of long-row pieces per row, combined by the fix-up"""
    rng = np.random.default_rng(7)
    n = 4000
    s, t = rand_graph(rng, n, 20000)
    hub_t = np.repeat([5, 1000, n - 1], 100_000)
    hub_s = rng.integers(0, n, len(hub_t))
    hub_s[:100_000] = rng.integers(0, 3, 100_000)                     # hub 5 hears only three nodes, many times each
    s, t = np.concatenate([s, hub_s]), np.concatenate([t, hub_t])
    ref = ref_color_refinement(s, t, n)
    assert_same(run(gnn, s, t, n, "cuda"), ref)
    for C in (32, 128):
        assert_same(cuda_run(gnn, with_chunk(gnn, C, s, t, n)), ref)


@pytest.mark.gpu
def test_gpu_long_path(gnn):
    """a 2 001-node path: about 1 000 rounds"""
    s, t, n = path(2001)
    x, k, it = run(gnn, s, t, n, "cuda")
    assert (k, it) == (1001, 1001)
    assert_same((x, k, it), ref_color_refinement(s, t, n))


def molecules(rng, G, n1=23, e1=25):
    a = rng.integers(0, n1, (G, e1))
    b = (a + rng.integers(1, n1, (G, e1))) % n1
    off = (np.arange(G) * n1)[:, None]
    return (*undirected((a + off).ravel(), (b + off).ravel()), G * n1)


@pytest.mark.gpu
def test_gpu_molecule_batch(gnn):
    s, t, n = molecules(np.random.default_rng(8), 10_000)
    assert_same(run(gnn, s, t, n, "cuda"), ref_color_refinement(s, t, n))


@pytest.fixture(scope="module")
def rmat_200k(gnn):
    if not torch.cuda.is_available():
        pytest.skip("no CUDA device")
    g = gnn.rmat_graph(200_000, 2_000_000, seed=5, device="cuda")
    return g, npy(g.s) - 1, npy(g.t) - 1


@pytest.mark.gpu
def test_gpu_rmat_200k_equals_statement(gnn, rmat_200k):
    g, s, t = rmat_200k
    n = g.num_nodes
    ref = ref_color_refinement(s, t, n)
    got = cuda_run(gnn, g)
    assert_same(got, ref)
    assert_same(cuda_run(gnn, g), got)                                # two calls
    x0 = (np.arange(n) * 7919) % 11
    assert_same(cuda_run(gnn, g, torch.as_tensor(x0, device="cuda"), max_iters=2),
                ref_color_refinement(s, t, n, x0, 2))


@pytest.mark.gpu
def test_gpu_rmat_200k_chunk_32_and_128(gnn, rmat_200k):
    g, s, t = rmat_200k
    a, ka, ia = gnn.color_refinement(with_chunk(gnn, 32, s, t, g.num_nodes))
    b, kb, ib = gnn.color_refinement(with_chunk(gnn, 128, s, t, g.num_nodes))
    assert torch.equal(a, b) and (ka, ia) == (kb, ib)


@pytest.mark.gpu
def test_gpu_entry_status_codes(gnn):
    lib = gnn._lib.lib
    s = torch.tensor([0, 1], dtype=torch.int64, device="cuda")
    out = torch.empty(3, dtype=torch.int64, device="cuda")
    k, it = C.c_int64(0), C.c_int64(0)
    for ns, nd, max_iters, code in ((3, 2, 0, ESIZE), (3, 3, -1, EINVAL)):
        h = C.c_void_p()
        gnn._lib.check(lib.gnnb_graph_create(C.byref(h), s.data_ptr(), s.data_ptr(), 2, ns, nd, 8, 0, 1, None))
        try:
            assert lib.gnnb_color_refinement(h, None, max_iters, out.data_ptr(), C.byref(k), C.byref(it), None) == code
        finally:
            lib.gnnb_graph_destroy(h)


# ---------------------------------------------------------------------------------------------- GPU: RMAT 10 M / 100 M
def check_equitable(x, s, t, n):
    """every node of a class has the same sorted multiset of in-neighbour classes as its class's first node"""
    k = int(x.max())
    key = t * (k + 1) + x[s]
    key, _ = torch.sort(key)
    tt = torch.div(key, k + 1, rounding_mode="floor")
    cs = key - tt * (k + 1)
    deg = torch.bincount(t, minlength=n)
    rowptr = torch.zeros(n + 1, dtype=torch.int64, device=x.device)
    rowptr[1:] = torch.cumsum(deg, 0)
    head = torch.full((k + 1,), n, dtype=torch.int64, device=x.device)
    head.scatter_reduce_(0, x, torch.arange(n, device=x.device), reduce="amin")
    h = head[x]                                                         # each node's class head
    assert torch.equal(deg, deg[h])
    rank = torch.arange(len(tt), device=x.device) - rowptr[tt]
    assert torch.equal(cs, cs[rowptr[h[tt]] + rank])


def check_first_appearance(x, k):
    cm = torch.cummax(x, 0).values
    assert int(x[0]) == 1 and int(cm[-1]) == k
    assert bool((x[1:] <= cm[:-1] + 1).all())


@pytest.mark.gpu
def test_gpu_rmat_10m_invariants(gnn):
    n, E = 10 ** 7, 10 ** 8
    g = gnn.rmat_graph(n, E, seed=17, device="cuda")
    x, k, it = gnn.color_refinement(g)
    assert it >= 2 and 1 < k <= n
    s, t = g.s - 1, g.t - 1
    check_first_appearance(x, k)
    check_equitable(x - 1, s, t, n)
    del g
    torch.cuda.empty_cache()
    pi = torch.randperm(n, device="cuda", generator=torch.Generator("cuda").manual_seed(3))
    gp = gnn.GNNGraph(pi[s] + 1, pi[t] + 1, num_nodes=n)
    del s, t
    xp, kp, itp = gnn.color_refinement(gp)
    assert (kp, itp) == (k, it)
    check_first_appearance(xp, kp)
    pairs = torch.unique(x * (k + 1) + xp[pi])                          # colour of v against colour of pi(v)
    assert pairs.numel() == k
