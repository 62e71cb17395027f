"""The library-owned device scratch (the dense and attention-logit buffers, the cuBLASLt handle, the tensor-core kernels'
setup) is per device and grows only: a warmed-up training step replays from a CUDA graph with the bits of an eager step,
and a second device in the same process gets its own state rather than the first device's."""
import pytest
import torch

pytestmark = pytest.mark.gpu

N, E, D, HEADS, C = 4096, 40960, 128, 8, 64


def make_step(gnn, dev, state=None):
    """one training step of GCNConv 128->128 relu, SAGEConv 128->128 and GATConv 8x64 on one seeded graph: forward,
    backward, and the step's outputs (y of each layer, then the gradients of x and of every parameter)"""
    gen = torch.Generator().manual_seed(5)
    s = torch.randint(1, N + 1, (E,), generator=gen)
    t = torch.randint(1, N + 1, (E,), generator=gen)
    g = gnn.GNNGraph(s.to(dev), t.to(dev), num_nodes=N)
    layers = torch.nn.ModuleList([gnn.GCNConv(D, D, torch.relu, device=dev), gnn.SAGEConv(D, D, device=dev),
                                  gnn.GATConv(D, C, heads=HEADS, device=dev)])
    if state is not None:
        layers.load_state_dict(state)
    x = gnn.unrows(torch.randn(N, D, generator=gen).to(dev)).requires_grad_(True)
    dys = [gnn.unrows(torch.randn(N, d, generator=gen).to(dev)) for d in (D, D, HEADS * C)]
    params = [x] + list(layers.parameters())

    def step():
        for p in params:
            p.grad = None
        ys = [layer(g, x) for layer in layers]
        torch.autograd.backward(ys, dys)
        return [y.detach() for y in ys] + [p.grad for p in params]

    return step, layers


def test_training_step_replays_from_a_cuda_graph(gnn):
    dev = torch.device("cuda", 0)
    step, _ = make_step(gnn, dev)
    eager = [t.clone() for t in step()]
    side = torch.cuda.Stream(dev)
    side.wait_stream(torch.cuda.current_stream(dev))
    with torch.cuda.stream(side):
        for _ in range(3):
            step()
    torch.cuda.synchronize()
    cg = torch.cuda.CUDAGraph()
    with torch.cuda.graph(cg):
        out = step()
    cg.replay()
    torch.cuda.synchronize()
    assert len(out) == len(eager)
    for a, b in zip(eager, out):
        assert torch.equal(a, b)
    assert gnn._lib.lib.gnnb_dense_tc_error() == 0


@pytest.mark.skipif(torch.cuda.device_count() < 2, reason="needs two visible CUDA devices")
def test_second_device_gets_its_own_state(gnn):
    step0, layers0 = make_step(gnn, torch.device("cuda", 0))
    first = [t.cpu() for t in step0()]
    step1, _ = make_step(gnn, torch.device("cuda", 1), state=layers0.state_dict())
    second = [t.cpu() for t in step1()]
    for a, b in zip(first, second):
        assert torch.equal(a, b)
    assert gnn._lib.lib.gnnb_dense_tc_error() == 0
