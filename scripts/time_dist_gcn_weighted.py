"""python scripts/time_dist_gcn_weighted.py : what weighted GCNConv costs on the partitioned path, on one GPU.

At config 2's shape (RMAT N = 10 M, E = 100 M, self loops, 128 -> 128, relu, random positive weights), alternated in one
process, forward + backward per call (CUDA events):
1. one-rank weighted dist_gcn_conv, with an explicit edge_weight that requires grad and with one that does not;
2. single-GPU weighted gcn_conv, the same two ways;
3. unweighted dist_gcn_conv on the same DistGraph.
Then gnnb_gcn_edge_weight_grad_halo alone on the forward shard: ms per call and its algorithmic bytes over that time.

Prints one JSON line with the card, its power limit and SM clock beside the numbers.  Environment: N, E, REPS."""
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

N, E, REPS = int(os.environ.get("N", 10_000_000)), int(os.environ.get("E", 100_000_000)), int(os.environ.get("REPS", 5))
D = 128
dev = torch.device("cuda", 0)
torch.cuda.set_device(dev)
lib, chk = gnn._lib.lib, gnn._lib.check


def card():
    q = "name,power.limit,clocks.sm,clocks.max.sm"
    out = subprocess.run(["nvidia-smi", f"--query-gpu={q}", "--format=csv,noheader", "-i", "0"], capture_output=True, text=True)
    return dict(zip(q.split(","), [v.strip() for v in out.stdout.strip().split(",")])) if out.returncode == 0 else {}


def alternate(fns, reps=REPS):
    """mean ms of every function, run in turns after one warm-up each"""
    for f in fns.values():
        f()
    acc = {k: [] for k in fns}
    for _ in range(reps):
        for k, f in fns.items():
            a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            torch.cuda.synchronize()
            a.record(); f(); b.record()
            torch.cuda.synchronize()
            acc[k].append(a.elapsed_time(b))
    return {k: sum(v) / len(v) for k, v in acc.items()}


res = {"gpu": card(), "shape": f"RMAT N={N} E={E} + self loops, GCNConv {D} -> {D} relu, weights U(0.5, 1.5)", "reps": REPS}
with tempfile.TemporaryDirectory() as tmp:
    dist.init_process_group("gloo", init_method=f"file://{tmp}/store", rank=0, world_size=1)
    g0 = gnn.rmat_graph(N, E, 17, device=dev)
    gen = torch.Generator(device=dev).manual_seed(0)
    w = torch.rand(E, device=dev, generator=gen) + 0.5
    gw = gnn.GNNGraph(g0.s, g0.t, w, num_nodes=N)
    dg = P.DistGraph(g0.s, g0.t, N, w=w, add_self_loops=True, device=dev)
    w_local = w[dg.owned_by_target(g0.t)]                       # one rank: every edge, in global order
    torch.manual_seed(0)
    layer = gnn.GCNConv(D, D, torch.relu, device=dev)
    x = gnn.unrows(torch.randn(N, D, device=dev, generator=gen)).requires_grad_(True)
    dy = gnn.unrows(torch.randn(N, D, device=dev, generator=gen))

    def step(run, ew_src, grad_w):
        def f():
            x.grad = None
            layer.zero_grad(set_to_none=True)
            ew = ew_src.detach().requires_grad_(grad_w) if ew_src is not None else None
            run(ew).backward(dy)
        return f

    arms = {"dist_weighted_with_dw": step(lambda ew: P.dist_gcn_conv(layer, dg, x, ew), w_local, True),
            "dist_weighted_no_dw": step(lambda ew: P.dist_gcn_conv(layer, dg, x, ew), w_local, False),
            "gcn_conv_weighted_with_dw": step(lambda ew: layer(gw, x, ew), w, True),
            "gcn_conv_weighted_no_dw": step(lambda ew: layer(gw, x, ew), w, False),
            "dist_unweighted": step(lambda ew: P.dist_gcn_conv(layer, dg, x), None, False)}
    res["fwd_bwd_ms"] = alternate(arms)
    res["peak_memory_GB"] = torch.cuda.max_memory_allocated() / 1e9

    # the new kernel alone on the forward shard (D = 128, float4 lanes, one base: a single rank has no halo)
    x.grad = None
    sh = dg.fwd
    d, c, cf, cb = dg.gcn_scales(torch.cat([w_local, torch.ones(dg.n_local, device=dev)]))
    h = gnn.rows(x.detach()).contiguous()
    g = gnn.rows(dy).contiguous()
    dd = torch.randn(dg.n_local, device=dev, generator=gen)
    dw = torch.empty(sh.num_edges, device=dev)
    st = torch.cuda.current_stream(dev).cuda_stream

    def kern():
        chk(lib.gnnb_gcn_edge_weight_grad_halo(sh.plan.h, g.data_ptr(), h.data_ptr(), None, dg.n_local, cf.data_ptr(),
                                               c.data_ptr(), dd.data_ptr(), D, dw.data_ptr(), st))

    ms = alternate({"kernel": kern}, reps=max(REPS, 10))["kernel"]
    Es, n = sh.num_edges, dg.n_local
    # per edge: the gathered row, col / row / eid words, the gathered scale and the output; per target: its dout row, ct, dd
    alg = Es * (4 * D + 20) + n * (4 * D + 8)
    res["edge_weight_grad_kernel"] = {"ms": ms, "edges": Es, "algorithmic_bytes": alg, "GB_per_s": alg / (ms * 1e-3) / 1e9}
    dg.close()
    dist.destroy_process_group()
print(json.dumps(res), flush=True)
