"""python scripts/time_gat_halo.py : what the shard path of GATConv costs on one GPU.

1. The fused GAT kernels' HALO instances against the one-base instances at config 3's shape (RMAT N = 2 M, E = 50 M with
   self loops, 512 -> 8 heads x 64): forward gnnb_gat_aggregate_halo (gathered rows split at N/2, the tail in a separate
   buffer) against gnnb_gat_aggregate; pullback gnnb_gat_tnode + gnnb_gat_aggregate_bwd_halo on the reversed plan +
   gnnb_scatter of dz against gnnb_gat_aggregate_bwd (the same work).  Alternated, CUDA events.
2. dist_gat_conv forward + backward on a one-rank DistGraph (gloo) against gat_conv on the same graph, alternated.

Prints one JSON line with the card, its power limit and SM clock beside the numbers.  Environment: N, E, REPS."""
import ctypes as C
import json
import os
import subprocess
import sys
import tempfile

import torch
import torch.distributed as dist

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import gnnb200 as gnn  # noqa: E402
from gnnb200 import partition as P  # noqa: E402

N, E, REPS = int(os.environ.get("N", 2_000_000)), int(os.environ.get("E", 50_000_000)), int(os.environ.get("REPS", 10))
Cc, H, DIN, SLOPE = 64, 8, 512, 0.2
dev = torch.device("cuda", 0)
torch.cuda.set_device(dev)
lib, chk = gnn._lib.lib, gnn._lib.check


def card():
    q = "name,power.limit,clocks.sm,clocks.max.sm"
    out = subprocess.run(["nvidia-smi", f"--query-gpu={q}", "--format=csv,noheader", "-i", "0"], capture_output=True, text=True)
    return dict(zip(q.split(","), [v.strip() for v in out.stdout.strip().split(",")])) if out.returncode == 0 else {}


def alternate(fa, fb, reps=REPS):
    """mean ms of fa and fb, run in turns (a b a b ...) after one warm-up each"""
    fa(); fb()
    ta, tb = [], []
    for _ in range(reps):
        for f, acc in ((fa, ta), (fb, tb)):
            a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            torch.cuda.synchronize()
            a.record(); f(); b.record()
            torch.cuda.synchronize()
            acc.append(a.elapsed_time(b))
    return sum(ta) / len(ta), sum(tb) / len(tb)


res = {"gpu": card(), "shape": f"RMAT N={N} E={E} + self loops, {DIN} -> {H} x {Cc}", "reps": REPS}
g = gnn.add_self_loops(gnn.rmat_graph(N, E, 17, device=dev))
plan = g.plan()
rev = gnn.GNNGraph(g.t, g.s, num_nodes=N).plan()
st = torch.cuda.current_stream(dev).cuda_stream
gen = torch.Generator(device=dev).manual_seed(0)
Wx = torch.randn(N, H, Cc, device=dev, generator=gen)
dout = torch.randn(N, H, Cc, device=dev, generator=gen)
el, er = torch.randn(N, H, device=dev, generator=gen), torch.randn(N, H, device=dev, generator=gen)
split = N // 2
Wx_tail, dout_tail = Wx[split:].clone(), dout[split:].clone()
out, smax, ssum = torch.empty_like(Wx), torch.empty_like(el), torch.empty_like(el)
out2 = torch.empty_like(Wx)
Etot = int(g.num_edges)
dWx, dl, dr, T = torch.empty_like(Wx), torch.empty_like(el), torch.empty_like(er), torch.empty_like(el)
dz = torch.empty(Etot, H, device=dev)


def fwd_plain():
    chk(lib.gnnb_gat_aggregate(plan.h, Wx.data_ptr(), el.data_ptr(), er.data_ptr(), Cc, H, SLOPE, out.data_ptr(), None,
                               smax.data_ptr(), ssum.data_ptr(), st))


def fwd_halo():
    chk(lib.gnnb_gat_aggregate_halo(plan.h, Wx.data_ptr(), Wx_tail.data_ptr(), split, el.data_ptr(), er.data_ptr(), Cc, H,
                                    SLOPE, out2.data_ptr(), smax.data_ptr(), ssum.data_ptr(), st))


def bwd_plain():
    chk(lib.gnnb_gat_aggregate_bwd(plan.h, Wx.data_ptr(), el.data_ptr(), er.data_ptr(), smax.data_ptr(), ssum.data_ptr(),
                                   out.data_ptr(), dout.data_ptr(), Cc, H, SLOPE, dWx.data_ptr(), dl.data_ptr(), dr.data_ptr(), st))


def bwd_halo():
    chk(lib.gnnb_gat_tnode(dout.data_ptr(), out.data_ptr(), N, Cc, H, T.data_ptr(), st))
    chk(lib.gnnb_gat_aggregate_bwd_halo(rev.h, Wx.data_ptr(), er.data_ptr(), dout.data_ptr(), dout_tail.data_ptr(), split,
                                        el.data_ptr(), smax.data_ptr(), ssum.data_ptr(), T.data_ptr(), Cc, H, SLOPE,
                                        dWx.data_ptr(), dr.data_ptr(), dz.data_ptr(), st))
    chk(lib.gnnb_scatter(plan.h, gnn._lib.DST, gnn._lib.SUM, dz.data_ptr(), H, dl.data_ptr(), st))


fwd_plain()
fwd_halo()
torch.cuda.synchronize()
res["forward_bits_equal"] = bool(torch.equal(out.view(torch.int32), out2.view(torch.int32)))
a, b = alternate(fwd_plain, fwd_halo)
res["forward_ms"] = {"one_base": a, "halo_split_N/2": b}
a, b = alternate(bwd_plain, bwd_halo)
res["pullback_ms"] = {"one_base": a, "halo_split_N/2_with_tnode_and_scatter": b}
del Wx, dout, Wx_tail, dout_tail, out, out2, dWx, dz, rev
torch.cuda.empty_cache()

# 2. the layer: dist_gat_conv on one rank against gat_conv
with tempfile.TemporaryDirectory() as tmp:
    dist.init_process_group("gloo", init_method=f"file://{tmp}/store", rank=0, world_size=1)
    g0 = gnn.rmat_graph(N, E, 17, device=dev)
    dg = P.DistGraph(g0.s, g0.t, N, add_self_loops=True, device=dev)
    torch.manual_seed(0)
    layer = gnn.GATConv(DIN, Cc, torch.relu, heads=H, device=dev)
    x = gnn.unrows(torch.randn(N, DIN, device=dev, generator=gen)).requires_grad_(True)
    dy = gnn.unrows(torch.randn(N, H * Cc, device=dev, generator=gen))

    def one(run):
        def f():
            x.grad = None
            layer.zero_grad(set_to_none=True)
            run().backward(dy)
        return f

    a, b = alternate(one(lambda: layer(g0, x)), one(lambda: P.dist_gat_conv(layer, dg, x)), max(3, REPS // 2))
    res["layer_fwd_bwd_ms"] = {"gat_conv": a, "dist_gat_conv_W1": b}
    dg.close()
    dist.destroy_process_group()
print(json.dumps(res), flush=True)
