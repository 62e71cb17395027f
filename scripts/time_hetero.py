"""Time HeteroGraphConv (hetero.py) on cuda:0 against the same layers computed with torch gather/scatter per relation
(the reference's algorithm: index_select of the source rows, index_add_ / scatter_reduce into the targets).  One JSON
line per (workload, layer).

Workloads (rand_heterograph, uniform random edges, D = 128; each relation with its reverse):
  mag:  paper 736 389, author 1 134 649, institution 8 740, field 59 965 nodes;
        writes (author -> paper) 7.1 M, cites (paper -> paper) 5.4 M, has_topic (paper -> field) 7.5 M,
        affiliated (author -> institution) 1.0 M edges.  The stand-in has none of MAG's degree skew.
  mini: the same types scaled to about 50 k nodes and 500 k edges (the launch-bound side).
Layers inside HeteroGraphConv over every relation: SAGEConv(mean), GraphConv, GCNConv (no self loops), GATConv(8 x 16).
Arms, alternated round by round, timed with CUDA events around forward + backward:
  * `lib`: this library's layers;  * `torch`: a torch restatement per relation (same parameters).
With --profile, torch.profiler times the propagate kernels (seg_lean_kernel / seg_reduce_kernel) of one lib forward +
backward and sets their time against the algorithmic bytes per launch, E (4 D + 4) + 4 (N_dst + 1) + 4 D N_dst.
Each line carries the card's name, power limit and the SM clock read after the timed calls.

    python scripts/time_hetero.py [--rounds 5] [--only mag,mini] [--layers sage,graph,gcn,gat] [--profile]
"""
import argparse
import json
import operator
import os
import subprocess
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import gnnb200 as gnn  # noqa: E402

D = 128
MAG_N = {"paper": 736389, "author": 1134649, "institution": 8740, "field": 59965}
MAG_E = {("author", "writes", "paper"): 7_100_000, ("paper", "cites", "paper"): 5_400_000,
         ("paper", "has_topic", "field"): 7_500_000, ("author", "affiliated", "institution"): 1_000_000}


def card():
    try:
        out = subprocess.check_output(["nvidia-smi", "--id=0", "--query-gpu=name,power.limit,clocks.sm",
                                       "--format=csv,noheader,nounits"], text=True).strip().split(", ")
        return out[0], float(out[1]), float(out[2])
    except Exception:
        return torch.cuda.get_device_name(0), float("nan"), float("nan")


def event_ms(fn):
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    torch.cuda.synchronize()
    a.record()
    out = fn()
    b.record()
    torch.cuda.synchronize()
    return a.elapsed_time(b), out


def workload(name):
    scale = 1.0 if name == "mag" else 50_000 / sum(MAG_N.values())
    n = {k: max(2, int(v * scale)) for k, v in MAG_N.items()}
    m = {}
    for (a, r, b), e in MAG_E.items():
        k = max(1, int(e * scale))
        m[(a, r, b)] = k
        m[(b, r + "_rev", a)] = k
    g = gnn.rand_heterograph(n, m, seed=7, device="cuda")
    return g, n


def make_layer(kind):
    if kind == "sage":
        return gnn.SAGEConv(D, D, aggr=gnn.mean, device="cuda")
    if kind == "graph":
        return gnn.GraphConv(D, D, device="cuda")
    if kind == "gcn":
        return gnn.GCNConv(D, D, add_self_loops=False, device="cuda")
    return gnn.GATConv(D, 16, heads=8, add_self_loops=False, device="cuda")


# ---- the torch restatement per relation (Julia-shaped (D, N) in, rows inside) ----------------------------------------
def torch_relation(kind, l, s, t, xj, xi, nd):
    Xj, Xi = xj.t(), xi.t()
    if kind in ("sage", "graph"):
        agg = torch.zeros(nd, Xj.shape[1], device="cuda").index_add_(0, t, Xj.index_select(0, s))
        if kind == "sage":
            cnt = torch.zeros(nd, device="cuda").index_add_(0, t, torch.ones_like(t, dtype=torch.float32))
            agg = agg / cnt.clamp(min=1)[:, None]
            return (torch.cat([Xi, agg], 1) @ l.weight.t() + l.bias).t()
        return (Xi @ l.weight1.t() + agg @ l.weight2.t() + l.bias).t()
    if kind == "gcn":
        dout = torch.zeros(Xj.shape[0], device="cuda").index_add_(0, s, torch.ones_like(s, dtype=torch.float32))
        din = torch.zeros(nd, device="cuda").index_add_(0, t, torch.ones_like(t, dtype=torch.float32))
        xs = Xj * dout.rsqrt()[:, None].nan_to_num(posinf=0.0)
        p = torch.zeros(nd, Xj.shape[1], device="cuda").index_add_(0, t, xs.index_select(0, s))
        return ((p * din.rsqrt()[:, None].nan_to_num(posinf=0.0)) @ l.weight.t() + l.bias).t()
    H, C = l.heads, l.channel[1]
    Wj = (Xj @ l.dense_x.weight.t()).reshape(-1, H, C)
    Wi = (Xi @ l.dense_x.weight.t()).reshape(-1, H, C)
    el = (Wi * l.a[:C].t()).sum(-1)
    er = (Wj * l.a[C:].t()).sum(-1)
    z = torch.nn.functional.leaky_relu(el.index_select(0, t) + er.index_select(0, s), l.negative_slope)
    mx = torch.full((nd, H), -torch.inf, device="cuda").scatter_reduce(0, t[:, None].expand(-1, H), z, "amax")
    ex = torch.exp(z - mx.index_select(0, t))
    den = torch.zeros(nd, H, device="cuda").index_add_(0, t, ex)
    al = ex / den.index_select(0, t)
    out = torch.zeros(nd, H, C, device="cuda").index_add_(0, t, al[:, :, None] * Wj.index_select(0, s))
    return (out.reshape(nd, H * C) + l.bias).t()


def torch_forward(kind, model, g, x):
    out = {}
    for l, et in zip(model.layers, model.etypes):
        s, t = gnn.edge_index(g, et)
        y = torch_relation(kind, l, s.long() - 1, t.long() - 1, x[et[0]], x[et[2]], g.num_nodes[et[2]])
        out[et[2]] = y if et[2] not in out else out[et[2]] + y
    return out


def step(fwd, model, g, x):
    for p in model.parameters():
        p.grad = None
    for v in x.values():
        v.grad = None
    y = fwd(model, g, x)
    sum((v * v).sum() for v in y.values()).backward()
    return y


def profile_kernels(model, g, x):
    from torch.profiler import ProfilerActivity, profile
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        step(lambda m, gg, xx: m(gg, xx), model, g, x)
        torch.cuda.synchronize()
    ms, n = 0.0, 0
    for ev in prof.key_averages():
        if "seg_lean_kernel" in ev.key or "seg_reduce_kernel" in ev.key:
            ms += ev.device_time_total / 1e3
            n += ev.count
    return ms, n


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rounds", type=int, default=5)
    ap.add_argument("--only", default="mag,mini")
    ap.add_argument("--layers", default="sage,graph,gcn,gat")
    ap.add_argument("--profile", action="store_true")
    args = ap.parse_args()
    torch.cuda.set_device(0)
    for wname in args.only.split(","):
        g, n = workload(wname)
        gbytes = sum(g.num_edges[et] * (4 * D + 4) + 4 * (g.num_nodes[et[2]] + 1) + 4 * D * g.num_nodes[et[2]]
                     for et in g.etypes)
        for kind in args.layers.split(","):
            torch.manual_seed(0)
            model = gnn.HeteroGraphConv([(et, make_layer(kind)) for et in g.etypes], aggr=operator.add)
            x = {k: torch.randn(D, v, device="cuda").requires_grad_(True) for k, v in n.items()}
            arms = {"lib": lambda m, gg, xx: m(gg, xx), "torch": lambda m, gg, xx: torch_forward(kind, m, gg, xx)}
            times = {a: [] for a in arms}
            res = {}
            for a, f in arms.items():                 # warm-up (plans, allocator)
                try:
                    res[a] = {k: v.detach() for k, v in step(f, model, g, x).items()}
                except torch.cuda.OutOfMemoryError:
                    res[a] = None
                torch.cuda.empty_cache()
            for _ in range(args.rounds):
                for a, f in arms.items():
                    if res[a] is None:
                        continue
                    ms, _ = event_ms(lambda: step(f, model, g, x))
                    times[a].append(ms)
            agree = None
            if res["lib"] is not None and res["torch"] is not None:
                agree = max(float((res["lib"][k] - res["torch"][k]).norm() / res["torch"][k].norm()) for k in res["lib"])
            line = {"workload": wname, "layer": kind, "relations": len(g.etypes),
                    "nodes": sum(n.values()), "edges": sum(g.num_edges.values()), "D": D,
                    "ms_fwd_bwd": {a: (min(v) if v else "oom") for a, v in times.items()}, "rel_diff": agree}
            if args.profile:
                kms, launches = profile_kernels(model, g, x)
                line["propagate_kernels"] = {"ms": kms, "launches": launches,
                                             "algorithmic_bytes_per_pass_all_relations": gbytes}
            name, plimit, sm = card()
            line.update({"card": name, "power_limit_w": plimit, "sm_clock_mhz": sm})
            print(json.dumps(line), flush=True)
            del model, x, res
            torch.cuda.empty_cache()


if __name__ == "__main__":
    main()
