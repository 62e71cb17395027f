"""The L2 eviction priorities of the fused GCN propagate (seglean.cu, DESIGN.md §4 "L2 policy") decide where the gathered
rows are kept, never what is computed.  Forced on at every size (gnnb_set_kernel_variant(14)), the propagate with the
plan-owned normalisation, forward and transposed, and GCNConv forward and backward give the same bits as the default
(variant 0) and as the reference kernels (variant 12), on the hubs / chunk_edges / chunk32 graphs of test_gpu_parity.py
and on an RMAT graph of config 2's kind at N = 1 M, E = 10 M.  Variant 12 is the independent arm: its chunk kernel
gathers cs[col] and never reads the flagged stream.  Variant 0 runs plain loads on the small graphs, but on an H100 the
1 M graph's gathered rows (512 MB at D = 128) are more than 8 times the L2, so there variant 0 takes the hinted path
too, with a hot set that holds a small share of the nodes (both the hot and the cold load paths run).  Bits are compared
as int32, so NaN payloads count too.  The hot set itself is checked against a numpy restatement of the threshold rule
(gnnb_gcn_hot_rows), and the gate through the launch count: a hinted pass adds one launch, the demotion of its hot rows.
"""
import numpy as np
import pytest
import torch

from test_gpu_parity import build_graph

pytestmark = pytest.mark.gpu

GCN_GRAPHS = ["hubs", "chunk_edges", "chunk32"]
VARIANTS = (12, 0, 14)                      # reference kernels, default, L2 policy at every size


@pytest.fixture
def variant(gnn):
    yield lambda v: gnn._lib.check(gnn._lib.lib.gnnb_set_kernel_variant(v))
    gnn._lib.lib.gnnb_set_kernel_variant(0)


def bits(t):
    return t.contiguous().view(torch.int32)


def gcn_propagate(gnn, g2, tr, x):
    n, D = x.shape
    out = torch.empty(n, D, device="cuda")
    gnn._lib.check(gnn._lib.lib.gnnb_gcn_propagate(g2.plan().h, tr, x.data_ptr(), None, None, D, out.data_ptr(), None))
    return out


def check_same_bits(gnn, variant, g2, x):
    res = {}
    for v in VARIANTS:
        variant(v)
        res[v] = [gcn_propagate(gnn, g2, tr, x) for tr in (0, 1)]
    for v in VARIANTS[1:]:
        for tr in (0, 1):
            assert torch.equal(bits(res[v][tr]), bits(res[12][tr])), f"variant {v}, transposed {tr}"


@pytest.fixture(scope="module")
def rmat_1m(gnn):
    g = gnn.rmat_graph(1_000_000, 10_000_000, 17, device="cuda")
    return g, gnn.add_self_loops(g)


@pytest.mark.parametrize("D", [128, 256, 512])
@pytest.mark.parametrize("name", GCN_GRAPHS)
def test_gcn_propagate_same_bits_with_l2_policy(gnn, variant, name, D):
    _, s, t, n, g = build_graph(gnn, name)
    g2 = gnn.add_self_loops(g)                 # inherits the chunk of g's plan
    x = torch.randn(n, D, device="cuda", generator=torch.Generator(device="cuda").manual_seed(D))
    check_same_bits(gnn, variant, g2, x)


def test_gcn_propagate_same_bits_with_l2_policy_rmat(gnn, variant, rmat_1m):
    _, g2 = rmat_1m
    x = torch.randn(1_000_000, 128, device="cuda", generator=torch.Generator(device="cuda").manual_seed(1))
    check_same_bits(gnn, variant, g2, x)


@pytest.mark.parametrize("name", GCN_GRAPHS)
def test_gcn_propagate_nonfinite_with_l2_policy(gnn, variant, name):
    """NaN, +-Inf and values whose sums overflow float32, planted in the gathered rows: the same bits with the policy"""
    _, s, t, n, g = build_graph(gnn, name)
    g2 = gnn.add_self_loops(g)
    rng = np.random.default_rng(7)
    x = rng.standard_normal((n, 128)).astype(np.float32)
    rows = rng.choice(n, 12, replace=False)
    x[rows[:4], 5] = np.nan
    x[rows[4:8], 17] = np.inf
    x[rows[8:], 17] = -np.inf
    x[:, 64] = 3e38
    check_same_bits(gnn, variant, g2, torch.as_tensor(x).cuda())


def test_gcn_conv_same_bits_with_l2_policy(gnn, variant, rmat_1m):
    g, _ = rmat_1m
    n, D = 1_000_000, 128
    gen = torch.Generator(device="cuda").manual_seed(0)
    x0 = torch.randn(n, D, device="cuda", generator=gen)
    dy = gnn.unrows(torch.randn(n, D, device="cuda", generator=gen))
    torch.manual_seed(0)
    layer = gnn.GCNConv(D, D, torch.relu, device="cuda")
    res = {}
    for v in VARIANTS:
        variant(v)
        x = gnn.unrows(x0.clone()).requires_grad_(True)
        layer.weight.grad = None
        layer.bias.grad = None
        y = layer(g, x)
        y.backward(dy)
        res[v] = [gnn.rows(y.detach()), gnn.rows(x.grad), layer.weight.grad.clone(), layer.bias.grad.clone()]
    for v in VARIANTS[1:]:
        for i, (a, b) in enumerate(zip(res[v], res[12])):
            assert torch.equal(bits(a), bits(b)), f"variant {v}, output {('y', 'dx', 'dW', 'db')[i]}"


def hot_rule(gathered_1based, n):
    """numpy restatement: t = the smallest count whose nodes (count >= t) fit 0.56 of the L2 as 512 B rows"""
    l2 = torch.cuda.get_device_properties(0).L2_cache_size
    budget = int(l2 * 0.56) // 512
    assert gathered_1based.min() >= 1
    cnt = np.bincount(gathered_1based - 1, minlength=n)
    t = 1 if n <= budget else int(np.sort(cnt)[::-1][budget]) + 1
    return t, np.flatnonzero(cnt >= t), budget


def read_hot(gnn, g2, tr, n):
    import ctypes as C
    rows = np.empty(n, np.int32)
    nr, t = C.c_int64(), C.c_int32()
    gnn._lib.check(gnn._lib.lib.gnnb_gcn_hot_rows(g2.plan().h, tr, rows.ctypes.data, n, C.byref(nr), C.byref(t), None))
    return t.value, np.sort(rows[:nr.value])


def check_hot_set(gnn, g2, n):
    s2, t2 = g2.s.cpu().numpy(), g2.t.cpu().numpy()
    for tr, gathered in ((0, s2), (1, t2)):            # forward gathers the sources, the transposed pass the targets
        t_ref, hot_ref, budget = hot_rule(gathered, n)
        t, hot = read_hot(gnn, g2, tr, n)
        assert t == t_ref, f"transposed {tr}"
        assert np.array_equal(hot, hot_ref), f"transposed {tr}"
        assert len(hot) <= budget


@pytest.mark.parametrize("name", GCN_GRAPHS)
def test_hot_set_matches_threshold_rule(gnn, name):
    _, s, t, n, g = build_graph(gnn, name)
    check_hot_set(gnn, gnn.add_self_loops(g), n)


def test_hot_set_matches_threshold_rule_rmat(gnn, rmat_1m):
    _, g2 = rmat_1m
    check_hot_set(gnn, g2, 1_000_000)
    _, hot = read_hot(gnn, g2, 0, 1_000_000)
    assert 0 < len(hot) < 1_000_000                    # a real split into hot and cold rows


def launches(gnn, g2, x, tr=0):
    gcn_propagate(gnn, g2, tr, x)                      # the plan and its stream exist before counting
    n0 = gnn.launch_count()
    gcn_propagate(gnn, g2, tr, x)
    return gnn.launch_count() - n0


@pytest.mark.parametrize("D", [128, 256])
def test_policy_gate(gnn, variant, D):
    """small graph: hints only when forced, and only at D = 128 (wider rows never take them)"""
    _, s, t, n, g = build_graph(gnn, "hubs")
    g2 = gnn.add_self_loops(g)
    x = torch.randn(n, D, device="cuda")
    plain = [launches(gnn, g2, x, tr) for tr in (0, 1)]
    variant(14)
    for tr in (0, 1):
        assert launches(gnn, g2, x, tr) - plain[tr] == (1 if D == 128 else 0), f"transposed {tr}"


def test_policy_gate_rmat(gnn, variant, rmat_1m):
    """1 M nodes: variant 0 hints exactly when the gathered rows are at least 8 times the L2"""
    _, g2 = rmat_1m
    x = torch.randn(1_000_000, 128, device="cuda")
    on = 1_000_000 * 128 * 4 >= 8 * torch.cuda.get_device_properties(0).L2_cache_size
    variant(14)
    forced = launches(gnn, g2, x)
    variant(0)
    assert launches(gnn, g2, x) == forced - (0 if on else 1)
