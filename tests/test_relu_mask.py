"""The relu mask kept as bits (gnnb_linear_relu_mask, gnnb_linear_bwd_mask): its layout restated in numpy, the bits the
forward kernel writes, and the pullback that reads them against the one that reads y, which must agree bit for bit."""
import sys

import numpy as np
import pytest
import torch

DOUT = 128
COLS = np.arange(DOUT)
# column n of a row is bit 2 (n >> 3) + (n & 1) of word (n >> 1) & 3 (stated above tc::store_tile in csrc/dense_tc.cu)
WORD = (COLS >> 1) & 3
BIT = 2 * (COLS >> 3) + (COLS & 1)


def pack(pos):
    """(N, 128) bool -> (N, 4) uint32 in the library's layout"""
    out = np.zeros((pos.shape[0], 4), dtype=np.uint32)
    for w in range(4):
        sel = WORD == w
        out[:, w] = (pos[:, sel].astype(np.uint32) << BIT[sel].astype(np.uint32)).sum(axis=1, dtype=np.uint32)
    return out


def unpack(mask):
    return ((mask[:, WORD] >> BIT.astype(np.uint32)) & 1).astype(bool)


def test_layout_round_trips():
    rng = np.random.default_rng(0)
    pos = rng.random((257, DOUT)) < 0.5
    assert (unpack(pack(pos)) == pos).all()
    assert (pack(np.ones((1, DOUT), bool)) == 0xFFFFFFFF).all() and (pack(np.zeros((1, DOUT), bool)) == 0).all()
    for n in range(DOUT):                                  # one bit per column, each (word, bit) used once
        one = np.zeros((1, DOUT), bool)
        one[0, n] = True
        m = pack(one)
        assert m.sum() == np.uint32(1) << np.uint32(BIT[n]) and m[0, WORD[n]] != 0


def test_layout_is_the_accumulator_fragment():
    # lane l of a warp holds columns 8 j + 2 (l % 4) + c (j < 16, c < 2) of its rows: they are word l % 4, bit 2 j + c
    seen = set()
    for lane in range(4):
        for j in range(16):
            for c in range(2):
                n = 8 * j + 2 * lane + c
                assert (WORD[n], BIT[n]) == (lane, 2 * j + c)
                seen.add(n)
    assert seen == set(range(DOUT))


def _layers(gnn):
    return sys.modules[gnn.GCNConv.__module__]


def _forward(gnn, x, W, b):
    lib = gnn._lib.lib
    N, Din = x.shape
    y = torch.empty(N, DOUT, device="cuda")
    mask = torch.full((N, 4), -1, dtype=torch.int32, device="cuda")
    gnn._lib.check(lib.gnnb_linear_relu_mask(x.data_ptr(), W.data_ptr(), None if b is None else b.data_ptr(), N, Din, DOUT,
                                             y.data_ptr(), mask.data_ptr(), None))
    y_ref = torch.empty_like(y)
    gnn._lib.check(lib.gnnb_linear(x.data_ptr(), W.data_ptr(), None if b is None else b.data_ptr(), 1, N, Din, DOUT,
                                   y_ref.data_ptr(), None))
    assert torch.equal(y, y_ref)
    return y, mask


@pytest.mark.gpu
@pytest.mark.parametrize("N", [1, 31, 128, 129, 4097, 10 ** 6 + 3])
def test_mask_is_y_positive(gnn, N):
    gen = torch.Generator(device="cuda").manual_seed(N)
    Din = 64
    x = torch.randn(N, Din, device="cuda", generator=gen)
    W = torch.randn(DOUT, Din, device="cuda", generator=gen) / Din ** 0.5
    zero_w = torch.zeros_like(W)
    b = torch.randn(DOUT, device="cuda", generator=gen)
    # per column: random, all negative, all positive, exactly 0, -0 (pre-activation = bias when W = 0)
    mixed = torch.tensor([0.0, -0.0, -1.0, 2.0] * (DOUT // 4), device="cuda")
    cases = [(W, b), (W, None), (W, torch.full_like(b, -1e30)), (W * 1e-6, torch.full_like(b, 1e3)),
             (zero_w, torch.zeros_like(b)), (zero_w, torch.full_like(b, -0.0)), (zero_w, mixed)]
    for Wc, bc in cases:
        y, mask = _forward(gnn, x, Wc, bc)
        got = mask.cpu().numpy().view(np.uint32)
        assert (got == pack((y > 0).cpu().numpy())).all()
    assert gnn._lib.lib.gnnb_dense_tc_error() == 0


def _pullbacks(gnn, N, Din, seed, with_db=True):
    lib = gnn._lib.lib
    gen = torch.Generator(device="cuda").manual_seed(seed)
    x = torch.randn(N, Din, device="cuda", generator=gen)
    W = torch.randn(DOUT, Din, device="cuda", generator=gen) / Din ** 0.5
    b = torch.randn(DOUT, device="cuda", generator=gen) * 0.5
    b[::7] = 0.0                                           # columns whose pre-activation is often exactly 0
    x[:, ::5] = 0.0
    dy = torch.randn(N, DOUT, device="cuda", generator=gen)
    y, mask = _forward(gnn, x, W, b)
    outs = []
    for use_mask in (True, False):
        dx = torch.full_like(x, float("nan")); dW = torch.full_like(W, float("nan"))
        db = torch.full((DOUT,), float("nan"), device="cuda") if with_db else None
        pdb = None if db is None else db.data_ptr()
        if use_mask:
            gnn._lib.check(lib.gnnb_linear_bwd_mask(dy.data_ptr(), mask.data_ptr(), x.data_ptr(), W.data_ptr(), N, Din, DOUT,
                                                    dx.data_ptr(), dW.data_ptr(), pdb, None))
        else:
            ws = torch.empty_like(dy)
            gnn._lib.check(lib.gnnb_linear_bwd(dy.data_ptr(), y.data_ptr(), x.data_ptr(), W.data_ptr(), 1, N, Din, DOUT,
                                               ws.data_ptr(), dx.data_ptr(), dW.data_ptr(), pdb, None))
        outs.append((dx, dW, db))
    return outs


@pytest.mark.gpu
@pytest.mark.parametrize("N", [1, 33, 100, 4097, 132 * 32 + 1, 1000003])
@pytest.mark.parametrize("Din", [32, 64, 96, 128])
def test_mask_pullback_matches_y_pullback(gnn, N, Din):
    (dx, dW, db), (dx_y, dW_y, db_y) = _pullbacks(gnn, N, Din, seed=N * 5 + Din)
    assert torch.equal(dx, dx_y) and torch.equal(dW, dW_y) and torch.equal(db, db_y)
    (dx2, dW2, none), _ = _pullbacks(gnn, N, Din, seed=N * 5 + Din, with_db=False)
    assert none is None and torch.equal(dx2, dx) and torch.equal(dW2, dW)
    assert gnn._lib.lib.gnnb_dense_tc_error() == 0


@pytest.mark.gpu
def test_gcn_conv_mask_path_matches_y_path(gnn, monkeypatch):
    layers, lib = _layers(gnn), gnn._lib.lib
    calls = []
    real = lib.gnnb_linear_bwd_mask

    def counted(*a):
        calls.append(1)
        return real(*a)

    monkeypatch.setattr(lib, "gnnb_linear_bwd_mask", counted)
    n, E, D = 20011, 200000, 128
    g = gnn.rmat_graph(n, E, seed=5, device="cuda:0")
    results = []
    for use_mask in (True, False):
        monkeypatch.setattr(layers, "RELU_MASK", use_mask)
        torch.manual_seed(0)
        layer = gnn.GCNConv(D, D, torch.relu, device="cuda:0")
        gen = torch.Generator(device="cuda").manual_seed(1)
        x = gnn.unrows(torch.randn(n, D, device="cuda", generator=gen)).requires_grad_(True)
        dy = gnn.unrows(torch.randn(n, D, device="cuda", generator=gen))
        before = len(calls)
        y = layer(g, x)
        y.backward(dy)
        assert len(calls) - before == (1 if use_mask else 0)
        results.append([y.detach(), x.grad, layer.weight.grad, layer.bias.grad])
    for a, b in zip(*results):
        assert torch.equal(a, b)
    assert lib.gnnb_dense_tc_error() == 0


@pytest.mark.gpu
def test_mask_entries_reject_uncovered_shapes(gnn):
    lib, EUNSUPPORTED = gnn._lib.lib, gnn._lib.EUNSUPPORTED
    N = 256
    buf = torch.zeros(N * 256 + 64, device="cuda")
    mask = torch.zeros(N * 4 + 4, dtype=torch.int32, device="cuda")
    p, m = buf.data_ptr(), mask.data_ptr()

    def fwd(Din, Dout, x=p, m_=m):
        return lib.gnnb_linear_relu_mask(x, p, None, N, Din, Dout, p, m_, None)

    def bwd(Din, Dout, x=p, m_=m):
        return lib.gnnb_linear_bwd_mask(p, m_, x, p, N, Din, Dout, p, p, None, None)

    for Din, Dout in [(64, 64), (64, 256), (48, 128), (16, 128), (160, 128), (256, 128)]:
        assert fwd(Din, Dout) == EUNSUPPORTED and bwd(Din, Dout) == EUNSUPPORTED
    assert fwd(64, 128, x=p + 4) == EUNSUPPORTED and fwd(64, 128, m_=m + 8) == EUNSUPPORTED
    assert bwd(64, 128, x=p + 4) == EUNSUPPORTED and bwd(64, 128, m_=m + 8) == EUNSUPPORTED
    lib.gnnb_dense_set_tensor_core_kernel(0)
    try:
        assert fwd(64, 128) == EUNSUPPORTED and bwd(64, 128) == EUNSUPPORTED
    finally:
        lib.gnnb_dense_set_tensor_core_kernel(1)
    assert lib.gnnb_dense_tc_error() == 0
