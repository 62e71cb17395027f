"""The fused dense pullback of gnnb_linear_bwd (Dout = 128, Din in {32, 64, 96, 128}, dx and dW requested) against the
three-pass composition it replaces, which stays reachable through the public entries:
  gnnb_bias_act_bwd -> dpre, db;   gnnb_linear(dpre, W^T) -> dx;   gnnb_linear_bwd(dpre, relu 0, dx = db = NULL) -> dW."""
import pytest
import torch

pytestmark = pytest.mark.gpu

DOUT = 128
# rows that end inside a tile, inside a 32-row block and inside a CTA's split-K range (132 * 32 + 1), and CTAs with no rows
NS = [1, 33, 127, 128, 129, 4095, 132 * 32 + 1, 400000, 1000003]


def rel(a, b):
    return float((a.double() - b.double()).norm() / b.double().norm().clamp(min=1e-300))


def inputs(N, Din, seed, zeros=False):
    gen = torch.Generator(device="cuda").manual_seed(seed)
    x = torch.randn(N, Din, device="cuda", generator=gen)
    W = torch.randn(DOUT, Din, device="cuda", generator=gen) / Din ** 0.5
    dy = torch.randn(N, DOUT, device="cuda", generator=gen)
    y = torch.randn(N, DOUT, device="cuda", generator=gen)
    if zeros:   # a relu mask with many exact zeros and negative zeros: both must mask like negatives
        pick = torch.rand(N, DOUT, device="cuda", generator=gen)
        y = torch.where(pick < 0.3, torch.zeros_like(y), y)
        y = torch.where(pick > 0.7, torch.full_like(y, -0.0), y)
    return x, W, dy, y.clamp(min=0) if not zeros else y


def fused(lib, gnn, x, W, dy, y, relu, with_db):
    N, Din = x.shape
    dx = torch.empty_like(x); dW = torch.empty_like(W)
    db = torch.empty(DOUT, device="cuda") if with_db else None
    ws = torch.full_like(dy, float("nan"))
    gnn._lib.check(lib.gnnb_linear_bwd(dy.data_ptr(), y.data_ptr(), x.data_ptr(), W.data_ptr(), relu, N, Din, DOUT,
                                       ws.data_ptr(), dx.data_ptr(), dW.data_ptr(), None if db is None else db.data_ptr(),
                                       None))
    return dx, dW, db


def composition(lib, gnn, x, W, dy, y, relu):
    N, Din = x.shape
    dpre = torch.empty_like(dy) if relu else dy
    db = torch.empty(DOUT, device="cuda")
    gnn._lib.check(lib.gnnb_bias_act_bwd(dy.data_ptr(), y.data_ptr(), relu, N, DOUT, dpre.data_ptr(), db.data_ptr(), None))
    Wt = W.t().contiguous()
    dx = torch.empty_like(x)
    gnn._lib.check(lib.gnnb_linear(dpre.data_ptr(), Wt.data_ptr(), None, 0, N, DOUT, Din, dx.data_ptr(), None))
    dW = torch.empty_like(W)
    gnn._lib.check(lib.gnnb_linear_bwd(dpre.data_ptr(), None, x.data_ptr(), W.data_ptr(), 0, N, Din, DOUT, None, None,
                                       dW.data_ptr(), None, None))
    return dpre, dx, dW, db


@pytest.mark.parametrize("N", NS)
@pytest.mark.parametrize("Din", [32, 64, 96, 128])
@pytest.mark.parametrize("relu", [1, 0])
def test_fused_pullback_matches_composition(gnn, N, Din, relu):
    lib = gnn._lib.lib
    x, W, dy, y = inputs(N, Din, seed=N * 7 + Din + relu, zeros=(N % 2 == 1))
    n0 = gnn.launch_count()
    dx, dW, db = fused(lib, gnn, x, W, dy, y, relu, with_db=True)
    assert gnn.launch_count() == n0 + 3                 # dx + column sums, dW, the final reduction
    dpre, dx_ref, dW_ref, _ = composition(lib, gnn, x, W, dy, y, relu)
    assert torch.equal(dx, dx_ref)
    assert torch.equal(dW, dW_ref)                      # same dpre, same split-K partition
    d64 = dpre.double()
    assert rel(dW, d64.t() @ x.double()) < 5e-6
    assert rel(db, d64.sum(0)) < 5e-6
    dx2, dW2, db2 = fused(lib, gnn, x, W, dy, y, relu, with_db=True)
    assert torch.equal(dx2, dx) and torch.equal(dW2, dW) and torch.equal(db2, db)
    _, dW3, none = fused(lib, gnn, x, W, dy, y, relu, with_db=False)
    assert none is None and torch.equal(dW3, dW)
    assert lib.gnnb_dense_tc_error() == 0


def test_fused_pullback_not_taken_elsewhere(gnn):
    lib = gnn._lib.lib
    N, Din = 5000, 64
    x, W, dy, y = inputs(N, Din, seed=3)
    # Dout = 64
    W64 = W[:64].contiguous(); dy64 = dy[:, :64].contiguous(); y64 = y[:, :64].contiguous()
    ws = torch.empty_like(dy64); dx = torch.empty_like(x); dW = torch.empty_like(W64); db = torch.empty(64, device="cuda")
    n0 = gnn.launch_count()
    gnn._lib.check(lib.gnnb_linear_bwd(dy64.data_ptr(), y64.data_ptr(), x.data_ptr(), W64.data_ptr(), 1, N, Din, 64,
                                       ws.data_ptr(), dx.data_ptr(), dW.data_ptr(), db.data_ptr(), None))
    assert gnn.launch_count() - n0 == 5                 # mask + column sums, their reduction, transpose, dx, library dW
    dpre = dy64.double() * (y64 > 0)
    assert rel(dx, dpre @ W64.double()) < 5e-6 and rel(dW, dpre.t() @ x.double()) < 5e-6
    # dx only
    ws = torch.empty_like(dy); db = torch.empty(DOUT, device="cuda")
    n0 = gnn.launch_count()
    gnn._lib.check(lib.gnnb_linear_bwd(dy.data_ptr(), y.data_ptr(), x.data_ptr(), W.data_ptr(), 1, N, Din, DOUT,
                                       ws.data_ptr(), dx.data_ptr(), None, db.data_ptr(), None))
    assert gnn.launch_count() - n0 == 4                 # mask + column sums, their reduction, transpose, dx
    # tensor-core kernels off: the library GEMMs
    lib.gnnb_dense_set_tensor_core_kernel(0)
    try:
        dW = torch.empty_like(W)
        n0 = gnn.launch_count()
        gnn._lib.check(lib.gnnb_linear_bwd(dy.data_ptr(), y.data_ptr(), x.data_ptr(), W.data_ptr(), 1, N, Din, DOUT,
                                           ws.data_ptr(), dx.data_ptr(), dW.data_ptr(), db.data_ptr(), None))
        assert gnn.launch_count() - n0 == 4             # mask + column sums, their reduction, two library GEMMs
    finally:
        lib.gnnb_dense_set_tensor_core_kernel(1)
    dpre = dy.double() * (y > 0)
    assert rel(dx, dpre @ W.double()) < 5e-6 and rel(dW, dpre.t() @ x.double()) < 5e-6
    assert lib.gnnb_dense_tc_error() == 0
