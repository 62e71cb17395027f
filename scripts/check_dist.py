"""torchrun --nproc-per-node N scripts/check_dist.py : the node-partitioned GCNConv, GATConv, SAGEConv, GraphConv and
GINConv (partition.dist_gcn_conv / dist_gat_conv / dist_sage_conv / dist_graph_conv / dist_gin_conv, halo exchange over
NCCL or the IPC push) against the single-GPU layer on the full graph: forward, dx and the all-reduced weight
gradients."""
import os
import sys

import torch
import torch.distributed as dist

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import gnnb200 as gnn
from gnnb200 import partition as P

rank, world, local = int(os.environ["RANK"]), int(os.environ["WORLD_SIZE"]), int(os.environ["LOCAL_RANK"])
torch.cuda.set_device(local)
dev = torch.device("cuda", local)
dist.init_process_group("nccl", device_id=dev)
ok = True
for (n, E, D) in ((5000, 60000, 128), (200000, 3000000, 128), (30000, 200000, 64), (150000, 2000000, 256)):
    g = gnn.rmat_graph(n, E, 17, device=dev)
    torch.manual_seed(0)
    layer = gnn.GCNConv(D, D, torch.relu, device=dev)
    with torch.no_grad():
        layer.bias.normal_()
    gen = torch.Generator(device=dev).manual_seed(1)
    x_full = torch.randn(n, D, device=dev, generator=gen)
    dy_full = torch.randn(n, D, device=dev, generator=gen)
    # single GPU reference (every rank computes it)
    xr = gnn.unrows(x_full.clone()).requires_grad_(True)
    y = layer(g, xr)
    y.backward(gnn.unrows(dy_full))
    y_ref, dx_ref = gnn.rows(y.detach()).clone(), gnn.rows(xr.grad).clone()
    dW_ref, db_ref = layer.weight.grad.clone(), layer.bias.grad.clone()
    layer.weight.grad = None; layer.bias.grad = None
    # partitioned: shards built on the device (csrc/shard.cu) from the resident COO and from generated chunks
    def rel(a, b):
        return float((a - b).norm() / b.norm().clamp(min=1e-30))

    for how, ownership in (("coo", "contiguous"), ("coo", "balanced"), ("rmat-chunks", "cyclic"), ("rmat-chunks", "balanced")):
        if how == "coo":
            dg = P.DistGraph(g.s, g.t, n, add_self_loops=True, device=dev, ownership=ownership, chunk_edges=max(E // 3, 1))
        else:
            dg = P.DistGraph.from_rmat(n, E, 17, device=dev, add_self_loops=True, ownership=ownership, chunk_edges=max(E // 5, 1))
        ids = dg.local_nodes()
        xl = gnn.unrows(x_full[ids].clone()).requires_grad_(True)
        yl = P.dist_gcn_conv(layer, dg, xl)
        yl.backward(gnn.unrows(dy_full[ids].contiguous()))
        dist.all_reduce(layer.weight.grad); dist.all_reduce(layer.bias.grad)
        errs = {"y": rel(gnn.rows(yl.detach()), y_ref[ids]), "dx": rel(gnn.rows(xl.grad), dx_ref[ids]),
                "dW": rel(layer.weight.grad, dW_ref), "db": rel(layer.bias.grad, db_ref)}
        layer.weight.grad = None; layer.bias.grad = None
        good = all(v < 2e-6 for v in errs.values())
        ok = ok and good
        print(f"rank {rank}/{world} n={n} E={E} D={D} {how}/{ownership} n_local={dg.n_local} halo_f={dg.fwd.n_halo} "
              f"halo_b={dg.bwd.n_halo} edges_f={dg.fwd.num_edges} errs={errs} {'OK' if good else 'FAIL'}", flush=True)
        del dg


def check_layer(name, layer, g, n, Din, Dout, loops, run_dist, params):
    """one layer on the full graph (every rank) against its partitioned run over the ranks, two ownership modes"""
    global ok
    gen = torch.Generator(device=dev).manual_seed(2)
    x_full = torch.randn(n, Din, device=dev, generator=gen)
    dy_full = torch.randn(n, Dout, device=dev, generator=gen)
    xr = gnn.unrows(x_full.clone()).requires_grad_(True)
    y = layer(g, xr)
    y.backward(gnn.unrows(dy_full))
    y_ref, dx_ref = gnn.rows(y.detach()).clone(), gnn.rows(xr.grad).clone()
    g_ref = [p.grad.clone() for p in params]
    for ownership in ("contiguous", "balanced"):
        for p in params:
            p.grad = None
        dg = P.DistGraph(g.s, g.t, n, add_self_loops=loops, device=dev, ownership=ownership)
        ids = dg.local_nodes()
        xl = gnn.unrows(x_full[ids].clone()).requires_grad_(True)
        yl = run_dist(layer, dg, xl)
        yl.backward(gnn.unrows(dy_full[ids].contiguous()))
        for p in params:
            dist.all_reduce(p.grad)
        rel = lambda a, b: float((a - b).norm() / b.norm().clamp(min=1e-30))
        errs = {"y": rel(gnn.rows(yl.detach()), y_ref[ids]), "dx": rel(gnn.rows(xl.grad), dx_ref[ids])}
        errs.update({f"d{i}": rel(p.grad, r) for i, (p, r) in enumerate(zip(params, g_ref))})
        good = all(v < 1e-5 for v in errs.values())
        ok = ok and good
        print(f"rank {rank}/{world} {name} n={n} {ownership} n_local={dg.n_local} halo_f={dg.fwd.n_halo} "
              f"halo_b={dg.bwd.n_halo} errs={errs} {'OK' if good else 'FAIL'}", flush=True)
        dg.close()
        del dg
    for p in params:
        p.grad = None


for (n, E) in ((5000, 60000), (200000, 3000000)):
    g = gnn.rmat_graph(n, E, 17, device=dev)
    for concat in (True, False):
        torch.manual_seed(0)
        gat = gnn.GATConv(128, 64, torch.relu, heads=8, concat=concat, device=dev)
        with torch.no_grad():
            gat.bias.normal_()
        check_layer(f"GATConv 128->8x64 concat={concat}", gat, g, n, 128, 512 if concat else 64, True, P.dist_gat_conv,
                    [gat.dense_x.weight, gat.a, gat.bias])
    for aggr in (gnn.mean, "+"):
        torch.manual_seed(0)
        sage = gnn.SAGEConv(128, 128, torch.relu, aggr=aggr, device=dev)
        with torch.no_grad():
            sage.bias.normal_()
        check_layer(f"SAGEConv 128->128 aggr={aggr if isinstance(aggr, str) else 'mean'}", sage, g, n, 128, 128, False,
                    P.dist_sage_conv, [sage.weight, sage.bias])
    # GraphConv and GINConv on the graph plus a ring, so that every node has an in-edge (max / min without -Inf rows)
    ring = torch.arange(1, n + 1, device=dev, dtype=g.s.dtype)
    gr = gnn.GNNGraph(torch.cat([g.s, ring % n + 1]), torch.cat([g.t, ring]), num_nodes=n)
    for aggr in ("+", gnn.mean, "max", "min"):
        torch.manual_seed(0)
        gc = gnn.GraphConv(128, 64, torch.tanh, aggr=aggr, device=dev)
        with torch.no_grad():
            gc.bias.normal_()
        check_layer(f"GraphConv 128->64 aggr={aggr if isinstance(aggr, str) else 'mean'}", gc, gr, n, 128, 64, False,
                    P.dist_graph_conv, [gc.weight1, gc.weight2, gc.bias])
    for aggr in ("+", "max"):
        torch.manual_seed(0)
        lin = torch.nn.Linear(128, 64, device=dev)
        gin = gnn.GINConv(lambda h, lin=lin: gnn.unrows(torch.tanh(lin(gnn.rows(h)))), 0.5, aggr=aggr)
        check_layer(f"GINConv 128->64 aggr={aggr}", gin, gr, n, 128, 64, False, P.dist_gin_conv, [lin.weight, lin.bias])
t = torch.tensor([1 if ok else 0], device=dev)
dist.all_reduce(t, op=dist.ReduceOp.MIN)
dist.barrier()
dist.destroy_process_group()
sys.exit(0 if int(t) == 1 else 1)
