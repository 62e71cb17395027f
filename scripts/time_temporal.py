"""Time the recurrent temporal layers (temporal.py over csrc/recurrent.cu) on cuda:0 against the reference's schedule
composed from this library's own layers.  One JSON line per workload and layer.

Workloads (static graphs, x (in, T, N), T = 12):
  traffic  64 windows of a 207-node kNN (k = 8) sensor graph, batched; in 2, out 64; Chebyshev k = 3, DCGRU k = 2
  rmat     RMAT 1 M nodes / 10 M edges plus a ring (ChebConv needs no isolated node); in 16, out 64; same k
Arms, alternated round by round, timed with CUDA events around whole calls, forward alone and forward + backward (x and
every parameter require grad):
  * `fused`: the layer (x side once for all steps, shared h-side bases, the gate kernels);
  * `reference`: temporalconv.jl's schedule, per step and per gate, on this library's cheb_conv / d_conv / gcn_conv /
    dense calls with torch gate arithmetic (sigmoid, tanh and the broadcasts).
The peak memory of an arm is torch.cuda.max_memory_allocated during one forward + backward above what was allocated
before.  An arm that does not fit is reported as "oom".  Each line carries the card's name, power limit and the SM clock
read after the timed calls, and the normwise relative difference between the two arms' outputs.

    python scripts/time_temporal.py [--rounds 3] [--only traffic,rmat] [--layers gconvgru,...]
"""
import argparse
import gc
import json
import os
import subprocess
import sys

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import gnnb200 as gnn  # noqa: E402
from gnnb200.layers import _linear  # noqa: E402

LAYERS = ["gconvgru", "gconvlstm", "dcgru", "tgcn", "evolvegcno"]


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


def make_cell(kind, nin, out, k, g):
    torch.manual_seed(0)
    mk = {"gconvgru": lambda: gnn.GConvGRUCell(nin, out, k, device="cuda"),
          "gconvlstm": lambda: gnn.GConvLSTMCell(nin, out, k, device="cuda"),
          "dcgru": lambda: gnn.DCGRUCell(nin, out, 2, device="cuda"),
          "tgcn": lambda: gnn.TGCNCell(nin, out, device="cuda"),
          "evolvegcno": lambda: gnn.EvolveGCNOCell(nin, out, device="cuda")}[kind]
    cell = mk()
    if kind == "dcgru":
        # DConv diffuses with the unnormalised degree: with glorot weights DCGRU's recurrence (k = 2) has a gain of
        # about deg⁴ |W| per step and is chaotic; 0.5 / max_degree⁴ keeps it contractive, so the arms can be compared
        deg = max(int(torch.bincount(g.s).max()), int(torch.bincount(g.t).max()))
        with torch.no_grad():
            for p in cell.parameters():
                p.mul_(0.5 / float(deg) ** 4)
    return cell


def ref_step(kind, c, g, x, state):
    """one step of temporalconv.jl's cell on the library's layers, each gate on its own"""
    sg = torch.sigmoid
    if kind == "gconvgru":
        h = state
        r = sg(c.conv_x_r(g, x) + c.conv_h_r(g, h))
        z = sg(c.conv_x_z(g, x) + c.conv_h_z(g, h))
        ht = torch.tanh(c.conv_x_h(g, x) + c.conv_h_h(g, r * h))
        h = (1 - z) * ht + z * h
        return h, h
    if kind == "gconvlstm":
        h, cc = state
        i = sg(c.conv_x_i(g, x) + c.conv_h_i(g, h) + c.w_i * cc + c.b_i.reshape(-1, 1))
        f = sg(c.conv_x_f(g, x) + c.conv_h_f(g, h) + c.w_f * cc + c.b_f.reshape(-1, 1))
        cc = f * cc + i * torch.tanh(c.conv_x_c(g, x) + c.conv_h_c(g, h) + c.w_c * cc + c.b_c.reshape(-1, 1))
        o = sg(c.conv_x_o(g, x) + c.conv_h_o(g, h) + c.w_o * cc + c.b_o.reshape(-1, 1))
        h = o * torch.tanh(cc)
        return h, (h, cc)
    if kind == "dcgru":
        h = state
        ht = gnn.unrows(torch.cat([gnn.rows(x), gnn.rows(h)], 1))
        z = sg(c.dconv_u(g, ht))
        r = sg(c.dconv_r(g, ht))
        cc = torch.tanh(c.dconv_c(g, gnn.unrows(torch.cat([gnn.rows(x), gnn.rows(h * r)], 1))))
        h = z * h + (1 - z) * cc
        return h, h
    if kind == "tgcn":
        h = state

        def dense(d, a, b):                             # σ.(W vcat(a, b) .+ b)
            return d.sigma(_linear(d, d.weight, gnn.unrows(torch.cat([gnn.rows(a), gnn.rows(b)], 1)), False)
                           + d.bias.reshape(-1, 1))
        z = dense(c.dense_z, c.conv_z[1](g, c.conv_z[0](g, x)), h)
        r = dense(c.dense_r, c.conv_r[1](g, c.conv_r[0](g, x)), h)
        ht = dense(c.dense_h, c.conv_h[1](g, c.conv_h[0](g, x)), r * h)
        h = (1 - z) * h + z * ht
        return h, h
    w, (hl, cl) = state                                 # EvolveGCNO: Flux's LSTMCell on the weight, then GCNConv
    hl, (hl, cl) = c.lstm(w.reshape(-1, 1), (hl, cl))
    W = hl.reshape(c.in_, c.out).t()
    return c.conv(g, x, conv_weight=W), (hl.reshape(-1), (hl.reshape(-1), cl.reshape(-1)))


def ref_layer(kind, c, g, x):
    N = x.shape[2]
    z = torch.zeros(c.out, N, device="cuda")
    state = {"gconvlstm": (z, z), "evolvegcno": None}.get(kind, z)
    if kind == "evolvegcno":
        io = c.in_ * c.out
        zz = torch.zeros(io, device="cuda")
        state = (c.conv.weight.t().reshape(-1), (zz, zz))
    ys = []
    for t in range(x.shape[1]):
        y, state = ref_step(kind, c, g, x[:, t], state)
        ys.append(gnn.rows(y))
    return gnn.unrows(torch.stack(ys, 1))


def graphs(which):
    if which == "traffic":
        rng = np.random.default_rng(0)
        n, k, W = 207, 8, 64
        pts = rng.random((n, 2))
        d = ((pts[:, None] - pts[None]) ** 2).sum(-1)
        np.fill_diagonal(d, np.inf)
        nb = np.argsort(d, 1)[:, :k]
        s = np.concatenate([nb.reshape(-1) + w * n for w in range(W)]) + 1
        t = np.concatenate([np.repeat(np.arange(n), k) + w * n for w in range(W)]) + 1
        return gnn.GNNGraph(torch.as_tensor(s).cuda(), torch.as_tensor(t).cuda(), num_nodes=n * W), 2
    n = 1_000_000
    g0 = gnn.rmat_graph(n, 10_000_000, seed=17, device="cuda")
    i = torch.arange(1, n + 1, device="cuda", dtype=g0.s.dtype)
    return gnn.GNNGraph(torch.cat([g0.s, i]), torch.cat([g0.t, i % n + 1]), num_nodes=n), 16


def measure(fn, params, x):
    """(ms forward, ms forward + backward, peak GB) of one arm, or 'oom'"""
    try:
        torch.cuda.synchronize()
        base = torch.cuda.memory_allocated()
        torch.cuda.reset_peak_memory_stats()

        def fb():
            for p in params:
                p.grad = None
            x.grad = None
            y = fn()
            y.sum().backward()
            return y
        t_fb, y = event_ms(fb)
        peak = (torch.cuda.max_memory_allocated() - base) / 1e9
        with torch.no_grad():
            t_f, _ = event_ms(fn)
        return t_f, t_fb, peak, y.detach()
    except (torch.cuda.OutOfMemoryError, gnn.GNNBError) as e:
        if isinstance(e, gnn.GNNBError) and "out of memory" not in str(e):
            raise
        x.grad = None
        gc.collect()
        torch.cuda.empty_cache()
        return "oom"


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--only", default="traffic,rmat")
    ap.add_argument("--layers", default=",".join(LAYERS))
    a = ap.parse_args()
    for which in a.only.split(","):
        g, nin = graphs(which)
        N, T, out = g.num_nodes, 12, 64
        x = gnn.colmajor(torch.randn(nin, T, N, device="cuda")).requires_grad_(True)
        for kind in a.layers.split(","):
            cell = make_cell(kind, nin, out, 3, g)
            layer = gnn.GNNRecurrence(cell)
            params = list(cell.parameters())
            arms = {"fused": lambda: layer(g, x), "reference": lambda: ref_layer(kind, cell, g, x)}
            res = {k: [] for k in arms}
            for _ in range(a.rounds + 1):                # the first round warms up (λmax, plans, library handles)
                for name, fn in arms.items():
                    res[name].append(measure(fn, params, x))
            row = {"workload": which, "layer": kind, "N": N, "E": g.num_edges, "T": T, "in": nin, "out": out}
            outs = {}
            for name, rr in res.items():
                rr = rr[1:]
                if any(r == "oom" for r in rr):
                    row[name] = "oom"
                    continue
                outs[name] = rr[-1][3]
                row[name] = {"ms_fwd": float(np.median([r[0] for r in rr])),
                             "ms_fwd_bwd": float(np.median([r[1] for r in rr])),
                             "peak_gb": float(max(r[2] for r in rr))}
            if len(outs) == 2:
                row["rel_diff"] = float((outs["fused"] - outs["reference"]).norm() / outs["reference"].norm())
            row["card"], row["power_limit_w"], row["sm_clock_mhz"] = card()
            print(json.dumps(row), flush=True)
            del arms, res, outs, layer, cell, params
            x.grad = None
            gc.collect()
            torch.cuda.empty_cache()


if __name__ == "__main__":
    main()
