"""python scripts/time_dist_aggr.py : what max and mean aggregation cost on the partitioned path, on one GPU.

Three shapes: config 2's (RMAT N = 10 M, E = 100 M, D = 128) and RMAT N = 2 M, E = 50 M at D = 256 and 512, no self loops.
Alternated in one process, forward + backward per call (CUDA events):
1. one-rank dist_propagate(copy_xj, dg, max | mean, x);
2. single-GPU propagate(copy_xj, g, max | mean, xj = x).
A one-rank shard moves no halo rows and reduces the same rows, so the two arms do the same work.  Then
gnnb_propagate_maxmin_bwd_halo alone on the backward shard: ms per call and its algorithmic bytes E (8 D + 8) + 8 D N
(per edge the target's dout and out rows and the col / row words, per source its own row and its dx row) over that
time, against the H100 SXM data sheet's 3.35 TB/s.  The gathered target rows of a skewed graph are often served by the
L2 (RMAT's hubs are the targets of many edges), so this algorithmic rate can exceed the HBM rate.

Each shape runs in a process of its own (`python scripts/time_dist_aggr.py N,E,D` runs one), so that no allocation of
one shape limits the next.  Prints one JSON line per shape and one with the card, its power limit and SM clock beside
all the numbers.  Environment: REPS."""
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

REPS = int(os.environ.get("REPS", 5))
SHAPES = ((10_000_000, 100_000_000, 128), (2_000_000, 50_000_000, 256), (2_000_000, 50_000_000, 512))
HBM_TBPS = 3.35
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


def run_shape(N, E, D):
    with tempfile.TemporaryDirectory() as tmp:
        dist.init_process_group("gloo", init_method=f"file://{tmp}/store", rank=0, world_size=1)
        g = gnn.rmat_graph(N, E, 17, device=dev)
        dg = P.DistGraph(g.s, g.t, N, device=dev)
        gen = torch.Generator(device=dev).manual_seed(0)
        x = gnn.unrows(torch.randn(N, D, device=dev, generator=gen)).requires_grad_(True)
        dy = gnn.unrows(torch.randn(N, D, device=dev, generator=gen))

        def step(run):
            def f():
                x.grad = None
                run().backward(dy)
            return f

        arms = {}
        for name, aggr in (("max", "max"), ("mean", gnn.mean)):
            arms[f"dist_propagate_{name}"] = step(lambda a=aggr: P.dist_propagate(gnn.copy_xj, dg, a, x))
            arms[f"propagate_{name}"] = step(lambda a=aggr: gnn.propagate(gnn.copy_xj, g, a, xj=x))
        row = {"shape": f"RMAT N={N} E={E}, D={D}, copy_xj", "fwd_bwd_ms": alternate(arms)}
        # the same values both ways (max is exact; mean on one rank reduces every row in the single-GPU order)
        with torch.no_grad():
            for a in ("max", gnn.mean):
                same = torch.equal(P.dist_propagate(gnn.copy_xj, dg, a, x), gnn.propagate(gnn.copy_xj, g, a, xj=x))
                row[f"same_bits_{'max' if a == 'max' else 'mean'}"] = same
        x.grad = None

        # the new kernel alone on the backward shard (one rank: no halo rows)
        sh = dg.bwd
        xr = gnn.rows(x.detach()).contiguous()
        dout = gnn.rows(dy).contiguous()
        with torch.no_grad():
            out = gnn.rows(P.dist_propagate(gnn.copy_xj, dg, "max", x)).contiguous()
        dx = torch.empty_like(xr)
        st = torch.cuda.current_stream(dev).cuda_stream

        def kern():
            chk(lib.gnnb_propagate_maxmin_bwd_halo(sh.plan.h, gnn._lib.COPY_XJ, gnn._lib.MAX, xr.data_ptr(), dout.data_ptr(),
                                                   None, out.data_ptr(), None, dg.n_local, None, D, dx.data_ptr(), st))

        ms = alternate({"kernel": kern}, reps=max(REPS, 10))["kernel"]
        Es, n = sh.num_edges, dg.n_local
        alg = Es * (8 * D + 8) + 8 * D * n
        tbps = alg / (ms * 1e-3) / 1e12
        row["maxmin_bwd_halo_kernel"] = {"ms": ms, "edges": Es, "algorithmic_bytes": alg, "TB_per_s": tbps,
                                         "share_of_3.35_TBps": tbps / HBM_TBPS}
        dg.close()
        dist.destroy_process_group()
    return row


if len(sys.argv) > 1:
    print(json.dumps(run_shape(*(int(v) for v in sys.argv[1].split(",")))), flush=True)
else:
    res = {"gpu": card(), "reps": REPS, "shapes": []}
    for N, E, D in SHAPES:
        p = subprocess.run([sys.executable, os.path.abspath(__file__), f"{N},{E},{D}"], capture_output=True, text=True)
        if p.returncode != 0:
            sys.stderr.write(p.stderr)
            sys.exit(p.returncode)
        row = json.loads(p.stdout.strip().splitlines()[-1])
        print(json.dumps(row), flush=True)
        res["shapes"].append(row)
    print(json.dumps(res), flush=True)
