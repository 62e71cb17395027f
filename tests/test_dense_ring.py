"""The 3xTF32 ring kernels (linear_tf32x3 / linear_relu_mask forward, the dx kernels of the dense pullback), which read
their A fragments from a TMA-fed ring into registers, against the same arithmetic with A read from shared memory.

The wide kernel (Dout > 128) keeps its A operand in shared memory and runs the same split, the same wgmma.m64n128k8
sequence and the same epilogue on each 128-column quarter of W, so its first quarter must equal the 128-wide kernel on
those 128 rows of W bit for bit, non-finite values included.  The dx kernels are the forward kernel run on dpre and W^T.
"""
import pytest
import torch

pytestmark = pytest.mark.gpu

DOUT = 128
NS = [1, 127, 128, 129, 2047, 2048, 1_000_037]   # 1 000 037 rows: 7 813 tiles, not a multiple of the grid
KS = [32, 64, 96, 128]


def bits(t):
    return t.contiguous().view(torch.int32)


def same_bits(a, b):
    return torch.equal(bits(a), bits(b))


def plant(t, seed):
    """NaN (quiet and one with only a low payload bit), +-Inf and subnormals at the K-block edges of rows at tile edges"""
    N, K = t.shape
    special = torch.tensor([0x7FC00000, 0x7F800001, 0x7F800000, 0xFF800000, 0x00000001, 0x80400000], dtype=torch.int64)
    special = special.to(torch.int32).view(torch.float32).to(t.device)
    rows = sorted({0, min(127, N - 1), min(128, N - 1), N - 1, N // 2})
    cols = sorted({c for kb in range(K // 32) for c in (32 * kb, 32 * kb + 31)} | {4, K - 5})
    i = seed
    for r in rows:
        for c in cols[(r % 3)::3]:
            t[r, c] = special[i % len(special)]
            i += 1
    return t


def inputs(N, K, seed, nonfinite):
    gen = torch.Generator(device="cuda").manual_seed(seed)
    x = torch.randn(N, K, device="cuda", generator=gen)
    W = torch.randn(2 * DOUT, K, device="cuda", generator=gen) / K ** 0.5
    b = torch.randn(2 * DOUT, device="cuda", generator=gen)
    if nonfinite:
        plant(x, seed)
    return x, W, b


def wide_first_quarter(gnn, x, W, b, relu):
    """y[:, :128] of the wide kernel (x padded to the 2 048 rows it takes at least; rows are independent)"""
    lib = gnn._lib.lib
    N, K = x.shape
    xp = x if N >= 2048 else torch.cat([x, torch.zeros(2048 - N, K, device="cuda")])
    y = torch.empty(xp.shape[0], 2 * DOUT, device="cuda")
    gnn._lib.check(lib.gnnb_linear(xp.data_ptr(), W.data_ptr(), b.data_ptr(), relu, xp.shape[0], K, 2 * DOUT, y.data_ptr(),
                                   None))
    return y[:N, :DOUT]


@pytest.mark.parametrize("N", NS)
@pytest.mark.parametrize("K", KS)
@pytest.mark.parametrize("nonfinite", [False, True])
def test_forward_matches_shared_memory_operand(gnn, N, K, nonfinite):
    lib = gnn._lib.lib
    x, W, b = inputs(N, K, 10 * N + K, nonfinite)
    W0, b0 = W[:DOUT].contiguous(), b[:DOUT].contiguous()
    for relu in (1, 0):
        ref = wide_first_quarter(gnn, x, W, b, relu)
        y = torch.full((N, DOUT), float("nan"), device="cuda")
        gnn._lib.check(lib.gnnb_linear(x.data_ptr(), W0.data_ptr(), b0.data_ptr(), relu, N, K, DOUT, y.data_ptr(), None))
        assert same_bits(y, ref), (relu, (bits(y) != bits(ref)).sum().item())
    y = torch.full((N, DOUT), float("nan"), device="cuda")
    mask = torch.zeros(N, 4, dtype=torch.int32, device="cuda")
    gnn._lib.check(lib.gnnb_linear_relu_mask(x.data_ptr(), W0.data_ptr(), b0.data_ptr(), N, K, DOUT, y.data_ptr(),
                                             mask.data_ptr(), None))
    assert same_bits(y, wide_first_quarter(gnn, x, W, b, 1))
    col = torch.arange(DOUT, device="cuda")
    word, bit = (col >> 1) & 3, 2 * (col >> 3) + (col & 1)
    assert torch.equal((mask[:, word] >> bit) & 1 == 1, y > 0)
    assert lib.gnnb_dense_tc_error() == 0


@pytest.mark.parametrize("N", NS)
@pytest.mark.parametrize("Din", KS)
def test_dx_is_the_forward_kernel_on_dpre(gnn, N, Din):
    """dx of both pullbacks (relu from the mask bits, relu from y) = the forward kernel on dpre and W^T, with NaN and
    +-Inf in dy at the K-block edges; both give the same db"""
    lib = gnn._lib.lib
    gen = torch.Generator(device="cuda").manual_seed(N + Din)
    x = torch.randn(N, Din, device="cuda", generator=gen)
    W = torch.randn(DOUT, Din, device="cuda", generator=gen) / Din ** 0.5
    b = torch.randn(DOUT, device="cuda", generator=gen)
    dy = plant(torch.randn(N, DOUT, device="cuda", generator=gen), N)
    y = torch.empty(N, DOUT, device="cuda")
    mask = torch.empty(N, 4, dtype=torch.int32, device="cuda")
    gnn._lib.check(lib.gnnb_linear_relu_mask(x.data_ptr(), W.data_ptr(), b.data_ptr(), N, Din, DOUT, y.data_ptr(),
                                             mask.data_ptr(), None))
    dpre = torch.where(y > 0, dy, torch.zeros_like(dy))
    Wt = W.t().contiguous()
    ref = torch.empty(N, Din, device="cuda")
    gnn._lib.check(lib.gnnb_linear(dpre.data_ptr(), Wt.data_ptr(), None, 0, N, DOUT, Din, ref.data_ptr(), None))
    out = {}
    for how in ("mask", "y"):
        dx = torch.full_like(x, float("nan")); dW = torch.empty_like(W); db = torch.empty(DOUT, device="cuda")
        if how == "mask":
            gnn._lib.check(lib.gnnb_linear_bwd_mask(dy.data_ptr(), mask.data_ptr(), x.data_ptr(), W.data_ptr(), N, Din, DOUT,
                                                    dx.data_ptr(), dW.data_ptr(), db.data_ptr(), None))
        else:
            ws = torch.empty_like(dy)
            gnn._lib.check(lib.gnnb_linear_bwd(dy.data_ptr(), y.data_ptr(), x.data_ptr(), W.data_ptr(), 1, N, Din, DOUT,
                                               ws.data_ptr(), dx.data_ptr(), dW.data_ptr(), db.data_ptr(), None))
        assert same_bits(dx, ref), (how, (bits(dx) != bits(ref)).sum().item())
        out[how] = (dW, db)
    assert same_bits(out["mask"][0], out["y"][0]) and same_bits(out["mask"][1], out["y"][1])
    assert lib.gnnb_dense_tc_error() == 0


def db_fixed_order(dpre, nsm):
    """db as the dx kernel forms it, restated with float32 adds in the same order: CTA b of min(tiles, nsm) takes tiles
    b, b + grid, ...; its producer warp w sums, per tile and column, T_q = rows 4 w + q + 16 i (i = 0..7, from 0) and adds
    (T_0 + T_1) + (T_2 + T_3) to a running sum from 0; the reduction adds the sums of (b, w) in order from 0"""
    N = dpre.shape[0]
    ntiles = -(-N // 128)
    grid = min(ntiles, nsm)
    T = -(-ntiles // grid)
    pad = torch.zeros(T * grid * 128, DOUT, device=dpre.device)
    pad[:N] = dpre
    X = pad.view(T, grid, 8, 4, 4, DOUT)                 # tile t * grid + b, row 16 i + 4 w + q
    valid = (torch.arange(T, device=dpre.device)[:, None] * grid + torch.arange(grid, device=dpre.device)) < ntiles
    cs = torch.zeros(grid, 4, DOUT, device=dpre.device)
    for t in range(T):
        s = torch.zeros(grid, 4, 4, DOUT, device=dpre.device)
        for i in range(8):
            s = s + X[t, :, i]
        cs = torch.where(valid[t][:, None, None], cs + ((s[:, :, 0] + s[:, :, 1]) + (s[:, :, 2] + s[:, :, 3])), cs)
    db = torch.zeros(DOUT, device=dpre.device)
    for row in cs.view(-1, DOUT):
        db = db + row
    return db


@pytest.mark.parametrize("N", NS)
def test_db_is_the_fixed_order_column_sum(gnn, N):
    """db of both pullbacks against the summation order restated above, with exact and negative zeros in dpre"""
    lib = gnn._lib.lib
    Din = 64
    gen = torch.Generator(device="cuda").manual_seed(3 * N + 1)
    x = torch.randn(N, Din, device="cuda", generator=gen)
    W = torch.randn(DOUT, Din, device="cuda", generator=gen) / Din ** 0.5
    b = torch.randn(DOUT, device="cuda", generator=gen)
    dy = torch.randn(N, DOUT, device="cuda", generator=gen)
    dy[: N // 3] = -0.0
    y = torch.empty(N, DOUT, device="cuda")
    mask = torch.empty(N, 4, dtype=torch.int32, device="cuda")
    gnn._lib.check(lib.gnnb_linear_relu_mask(x.data_ptr(), W.data_ptr(), b.data_ptr(), N, Din, DOUT, y.data_ptr(),
                                             mask.data_ptr(), None))
    ref = db_fixed_order(torch.where(y > 0, dy, torch.zeros_like(dy)), torch.cuda.get_device_properties(0).multi_processor_count)
    for how in ("mask", "y"):
        dx = torch.empty_like(x); dW = torch.empty_like(W); db = torch.full((DOUT,), float("nan"), device="cuda")
        if how == "mask":
            gnn._lib.check(lib.gnnb_linear_bwd_mask(dy.data_ptr(), mask.data_ptr(), x.data_ptr(), W.data_ptr(), N, Din, DOUT,
                                                    dx.data_ptr(), dW.data_ptr(), db.data_ptr(), None))
        else:
            ws = torch.empty_like(dy)
            gnn._lib.check(lib.gnnb_linear_bwd(dy.data_ptr(), y.data_ptr(), x.data_ptr(), W.data_ptr(), 1, N, Din, DOUT,
                                               ws.data_ptr(), dx.data_ptr(), dW.data_ptr(), db.data_ptr(), None))
        assert same_bits(db, ref), (how, (db - ref).abs().max().item())


def test_graph_replay_equals_eager(gnn):
    lib = gnn._lib.lib
    N, D = 300_001, 128
    gen = torch.Generator(device="cuda").manual_seed(7)
    x = plant(torch.randn(N, D, device="cuda", generator=gen), 7)
    W = torch.randn(D, D, device="cuda", generator=gen) / D ** 0.5
    b = torch.randn(D, device="cuda", generator=gen)
    dy = torch.randn(N, D, device="cuda", generator=gen)
    y = torch.empty(N, D, device="cuda"); mask = torch.empty(N, 4, dtype=torch.int32, device="cuda")
    dx = torch.empty_like(x); dW = torch.empty_like(W); db = torch.empty(D, device="cuda")
    s = torch.cuda.Stream()

    def step():
        st = s.cuda_stream
        gnn._lib.check(lib.gnnb_linear_relu_mask(x.data_ptr(), W.data_ptr(), b.data_ptr(), N, D, D, y.data_ptr(),
                                                 mask.data_ptr(), st))
        gnn._lib.check(lib.gnnb_linear_bwd_mask(dy.data_ptr(), mask.data_ptr(), x.data_ptr(), W.data_ptr(), N, D, D,
                                                dx.data_ptr(), dW.data_ptr(), db.data_ptr(), st))

    with torch.cuda.stream(s):
        step()                                   # warm-up: device state and scratch exist before capture
    s.synchronize()
    eager = [t.clone() for t in (y, mask, dx, dW, db)]
    for t in (y, dx, dW, db):
        t.fill_(float("nan"))
    mask.zero_()
    g = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g, stream=s):
        step()
    g.replay()
    torch.cuda.synchronize()
    for a, e in zip((y, mask, dx, dW, db), eager):
        assert torch.equal(bits(a), bits(e))
    assert lib.gnnb_dense_tc_error() == 0
