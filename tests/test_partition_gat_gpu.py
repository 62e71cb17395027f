"""GATConv and SAGEConv on the node-partitioned graph (partition.py: dist_gat_conv, dist_sage_conv) on the GPU, with the
multi-rank harness of test_partition_gpu.py: W gloo ranks share one device (or one rank per device under NCCL), real
shards, both halo routes, one and two push buffers.

Checked per rank against the one-GPU library on the same graph and against float64 over the whole graph:
- the GAT edge part (out, seg_max, seg_sum, dWx, der, del) bit for bit on rows whose every value is reduced in the
  single-GPU order (rows of at most one chunk of edges, and for dWx / der sources whose targets all are such rows), and
  normwise against float64 elsewhere; everything bit for bit at W = 1 in node order (balanced ownership reorders the
  rows, and with them the chunks of the long ones);
- the dz exchange: every edge value, tagged with the edge's global (source, target), lands on the same edge;
- dist_gat_conv (concat true and false, a lean shape, C = 1 and 128 x 16, whose logit pullback runs in two slices of
  heads) and dist_sage_conv (mean, +): y, dx and the all-reduced weight gradients against float64 autograd of the dense
  formula;
- three steps on one DistGraph equal fresh one-step runs bit for bit;
- the argument errors."""
import datetime
import os
import sys
import traceback

import numpy as np
import pytest
import torch

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
from test_partition_gpu import (CHUNK, N_NODES, TOL_LAYER, TOL_LONG, Rank, assert_records, bits_record,  # noqa: E402
                                Reference, check_structure, make_graph, ownership_cases, rel_err, require_shared_device,
                                run_group)

pytestmark = pytest.mark.gpu

SLOPE = 0.2
EDGE_SHAPES = ((32, 4), (1, 8), (8, 5))      # (C, H): the lean kernels at D = 128, C = 1 (Wx and er rows both H wide),
                                             # a round-1 vector shape


# ------------------------------------------------------------------------------------------------ float64 statements
class Full:
    """the whole graph (loops appended when the layer adds them), its one-GPU plan and float64 edge arithmetic"""

    def __init__(self, R, G, loops):
        gnn, n = R.gnn, N_NODES
        s, t = G["s"], G["t"]
        if loops:
            s, t = np.concatenate([s, np.arange(n)]), np.concatenate([t, np.arange(n)])
        self.s = torch.as_tensor(s, device=R.dev)
        self.t = torch.as_tensor(t, device=R.dev)
        g = gnn.GNNGraph(torch.as_tensor(G["s"] + 1), torch.as_tensor(G["t"] + 1), num_nodes=n).cuda()
        self.g = gnn.add_self_loops(g) if loops else g
        self.plan = self.g.plan()
        self.indeg = torch.bincount(self.t, minlength=n)
        self.outdeg = torch.bincount(self.s, minlength=n)

    def gat_f64(self, Wx, el, er, slope, dout=None):
        """out, seg_max, seg_sum and (with dout) dWx, der, del in float64; also sum |dz| per source and per target (the
        scale of der and del, which are sums that cancel)"""
        s, t, n = self.s, self.t, N_NODES
        Wx, el, er = Wx.double(), el.double(), er.double()
        H = el.shape[1]
        z = el[t] + er[s]
        u = torch.where(z > 0, z, slope * z)
        M = torch.full((n, H), -float("inf"), dtype=torch.float64, device=z.device)
        M = M.scatter_reduce(0, t[:, None].expand(-1, H), u, "amax")
        ex = torch.exp(u - M[t])
        S = torch.zeros((n, H), dtype=torch.float64, device=z.device).index_add_(0, t, ex)
        al = ex / S[t]
        out = torch.zeros(Wx.shape, dtype=torch.float64, device=z.device).index_add_(0, t, al[:, :, None] * Wx[s])
        M = torch.where(torch.isinf(M), torch.zeros_like(M), M)
        res = {"out": out, "seg_max": M, "seg_sum": S}
        if dout is not None:
            d = dout.double()
            da = (d[t] * Wx[s]).sum(-1)
            T = (d * out).sum(-1)
            dz = al * (da - T[t]) * torch.where(z > 0, 1.0, slope)
            z0 = torch.zeros((n, H), dtype=torch.float64, device=z.device)
            res["dWx"] = torch.zeros_like(out).index_add_(0, s, al[:, :, None] * d[t])
            res["der"] = z0.clone().index_add_(0, s, dz)
            res["del"] = z0.clone().index_add_(0, t, dz)
            res["der_scale"] = z0.clone().index_add_(0, s, dz.abs())
            res["del_scale"] = z0.clone().index_add_(0, t, dz.abs())
        return res


def gat_layer_f64(layer, full, x, dy, concat):
    """float64 autograd of gat_conv over the whole graph: y, dx and the weight gradients"""
    s, t, n = full.s, full.t, N_NODES
    Cc, H = layer.channel[1], layer.heads
    x64 = x.double().requires_grad_(True)
    Wd = layer.dense_x.weight.detach().double().requires_grad_(True)
    a = layer.a.detach().double().requires_grad_(True)
    b = layer.bias.detach().double().requires_grad_(True)
    Wx = (x64 @ Wd.t()).reshape(n, H, Cc)
    el = (Wx * a[:Cc].t()[None]).sum(-1)
    er = (Wx * a[Cc:].t()[None]).sum(-1)
    z = el[t] + er[s]
    u = torch.nn.functional.leaky_relu(z, float(layer.negative_slope))
    M = torch.full((n, H), -float("inf"), dtype=torch.float64, device=x.device)
    M = M.scatter_reduce(0, t[:, None].expand(-1, H), u.detach(), "amax")
    ex = torch.exp(u - M[t])
    S = torch.zeros((n, H), dtype=torch.float64, device=x.device).index_add(0, t, ex)
    al = ex / S[t]
    out = torch.zeros((n, H, Cc), dtype=torch.float64, device=x.device).index_add(0, t, al[:, :, None] * Wx[s])
    if not concat:
        out = out.mean(1, keepdim=True)
    y = torch.relu(out.reshape(n, -1) + b)
    y.backward(dy.double())
    return y.detach(), x64.grad, [Wd.grad, a.grad, b.grad]


def sage_layer_f64(layer, full, x, dy, mean):
    s, t, n = full.s, full.t, N_NODES
    x64 = x.double().requires_grad_(True)
    W = layer.weight.detach().double().requires_grad_(True)
    b = layer.bias.detach().double().requires_grad_(True)
    m = torch.zeros_like(x64).index_add(0, t, x64[s])
    if mean:
        m = m / full.indeg.clamp(min=1).double()[:, None]
    y = torch.relu(torch.cat([x64, m], 1) @ W.t() + b)
    y.backward(dy.double())
    return y.detach(), x64.grad, [W.grad, b.grad]


# ------------------------------------------------------------------------------------------------ rank side
def one_gpu_edge(R, full, Wx, el, er, dout):
    lib, chk, n = R.gnn._lib.lib, R.gnn._lib.check, N_NODES
    Cc, H = Wx.shape[2], Wx.shape[1]
    out, smax, ssum = torch.empty_like(Wx), torch.empty_like(el), torch.empty_like(el)
    chk(lib.gnnb_gat_aggregate(full.plan.h, Wx.data_ptr(), el.data_ptr(), er.data_ptr(), Cc, H, SLOPE, out.data_ptr(), None,
                               smax.data_ptr(), ssum.data_ptr(), R.stream()))
    dWx, dl, dr = torch.empty_like(Wx), torch.empty_like(el), torch.empty_like(er)
    chk(lib.gnnb_gat_aggregate_bwd(full.plan.h, Wx.data_ptr(), el.data_ptr(), er.data_ptr(), smax.data_ptr(), ssum.data_ptr(),
                                   out.data_ptr(), dout.data_ptr(), Cc, H, SLOPE, dWx.data_ptr(), dl.data_ptr(), dr.data_ptr(),
                                   R.stream()))
    return {"out": out, "seg_max": smax, "seg_sum": ssum, "dWx": dWx, "del": dl, "der": dr}


def check_edge_part(R, tag, dg, full):
    P, n = R.P, N_NODES
    ids = dg.local_nodes()
    short_t = full.indeg <= CHUNK
    # a source's dWx / der is in single-GPU order when its own row and every target row its edges meet are
    long_t = (~short_t).to(torch.int64)
    meets_long = torch.zeros(n, dtype=torch.int64, device=R.dev).index_add_(0, full.s, long_t[full.t]) > 0
    short_s = (full.outdeg <= CHUNK) & ~meets_long
    for Cc, H in EDGE_SHAPES:
        gen = torch.Generator(device=R.dev).manual_seed(31 * Cc + H)
        Wx, dout = (torch.randn(n, H, Cc, device=R.dev, generator=gen) for _ in range(2))
        el, er = (torch.randn(n, H, device=R.dev, generator=gen) for _ in range(2))
        one = one_gpu_edge(R, full, Wx, el, er, dout)
        f64 = full.gat_f64(Wx, el, er, SLOPE, dout)
        for route in ("push", "nccl"):
            R.set_route(route)
            name = f"edge/{tag}/C{Cc}H{H}/{route}"
            out, smax, ssum = P.dist_gat_aggregate(dg, Wx[ids].contiguous(), el[ids].contiguous(), er[ids].contiguous(), SLOPE)
            dWx, dl, dr = P.dist_gat_aggregate_bwd(dg, Wx[ids].contiguous(), el[ids].contiguous(), er[ids].contiguous(), smax,
                                                   ssum, out, dout[ids].contiguous(), SLOPE)
            got = {"out": out, "seg_max": smax, "seg_sum": ssum, "dWx": dWx, "del": dl, "der": dr}
            for k, v in got.items():
                mask = (short_s if k in ("dWx", "der") else short_t)[ids]
                if R.W == 1 and dg.ownership != "balanced":      # one shard in node order: the single-GPU chunks
                    mask = torch.ones_like(mask)
                R.put(f"{name}/{k}/bits_one_gpu", *bits_record(v[mask], one[k][ids][mask]))
                if k in ("der", "del"):                        # sums that cancel: error relative to the sum of |dz|
                    d = (v[~mask].double() - f64[k][ids][~mask]).reshape(-1)
                    sc = f64[k + "_scale"][ids][~mask].reshape(-1)
                    err = float(d.norm() / sc.norm().clamp(min=1e-30)) if d.numel() else 0.0
                    R.put(f"{name}/{k}/f64", err <= TOL_LONG, err, -1)
                else:
                    err, at = rel_err(v[~mask], f64[k][ids][~mask])
                    R.put(f"{name}/{k}/f64", err <= TOL_LONG, err, at)
    R.set_route()


def check_dz_exchange(R, tag, dg, halos):
    """tag every backward-shard edge with its global (source, target); after the exchange every forward-shard edge must
    hold its own"""
    ids = dg.local_nodes()
    coo = []
    for sh, halo in ((dg.fwd, halos[0]), (dg.bwd, halos[1])):
        ne = sh.num_edges
        rowptr = np.zeros(sh.n_local + 1, np.int32)
        col, eid = np.zeros(max(ne, 1), np.int32), np.zeros(max(ne, 1), np.int32)
        R.gnn._lib.check(R.gnn._lib.lib.gnnb_graph_csr(sh.plan.h, 0, rowptr.ctypes.data, col.ctypes.data, eid.ctypes.data,
                                                       None))
        row = np.repeat(np.arange(sh.n_local), np.diff(rowptr))
        coo_row, coo_col = np.zeros(ne, np.int64), np.zeros(ne, np.int64)
        coo_row[eid[:ne]], coo_col[eid[:ne]] = row, col[:ne]
        space = torch.cat([ids, halo.to(ids.dtype)]).cpu().numpy()
        coo.append((ids.cpu().numpy()[coo_row], space[coo_col]))
    (tgt_f, src_f), (src_b, tgt_b) = coo                     # fwd: row = target; bwd: row = source
    tag_b = torch.as_tensor(np.stack([src_b, tgt_b], 1), dtype=torch.float32, device=R.dev)
    want = torch.as_tensor(np.stack([src_f, tgt_f], 1), dtype=torch.float32, device=R.dev)
    R.put(f"dz/{tag}/every_edge_onto_itself", *bits_record(dg.edge_exchange(tag_b), want))


def gat_layer(R, Cc, H, concat, loops, Din=16):
    torch.manual_seed(7 * Cc + H + int(concat))
    layer = R.gnn.GATConv(Din, Cc, torch.relu, heads=H, concat=concat, add_self_loops=loops, device=R.dev)
    with torch.no_grad():
        layer.bias.copy_(torch.linspace(-0.5, 0.5, layer.bias.numel()))
    return layer


def dist_step(R, dg, layer, run, x_full, dy_full, params):
    import torch.distributed as dist
    gnn = R.gnn
    ids = dg.local_nodes()
    for p in params:
        p.grad = None
    x = gnn.unrows(x_full[ids].contiguous()).requires_grad_(True)
    y = run(layer, dg, x)
    y.backward(gnn.unrows(dy_full[ids].contiguous()))
    grads = [p.grad.clone() for p in params]
    for gr in grads:
        dist.all_reduce(gr)
    return [gnn.rows(y.detach()).clone(), gnn.rows(x.grad).clone()] + grads


def gat_params(layer):
    return [layer.dense_x.weight, layer.a, layer.bias]


def check_layers(R, tag, dg, full, loops):
    n = N_NODES
    ids = dg.local_nodes()
    R.set_route()
    for Cc, H in ((32, 4), (1, 8), (128, 16)):           # (128, 16): the logit pullback in two slices of heads
        for concat in (True, False):
            layer = gat_layer(R, Cc, H, concat, loops)
            gen = torch.Generator(device=R.dev).manual_seed(Cc + H)
            x_full = torch.randn(n, 16, device=R.dev, generator=gen)
            dy_full = torch.randn(n, Cc * H if concat else Cc, device=R.dev, generator=gen)
            got = dist_step(R, dg, layer, R.P.dist_gat_conv, x_full, dy_full, gat_params(layer))
            y64, dx64, g64 = gat_layer_f64(layer, full, x_full, dy_full, concat)
            for k, a, r in zip(("y", "dx", "dW", "da", "db"), got, [y64[ids], dx64[ids]] + g64):
                err, at = rel_err(a, r)
                R.put(f"layer/{tag}/gat_C{Cc}H{H}{'' if concat else '_mean'}/{k}", err <= TOL_LAYER, err, at)
    if loops:
        return
    for aggr, Din in (("mean", 128), ("+", 128), ("mean", 16)):
        torch.manual_seed(Din)
        Dout = 128 if Din == 128 else 8
        layer = R.gnn.SAGEConv(Din, Dout, torch.relu, aggr=R.gnn.mean if aggr == "mean" else "+", device=R.dev)
        with torch.no_grad():
            layer.bias.copy_(torch.linspace(-0.5, 0.5, Dout))
        gen = torch.Generator(device=R.dev).manual_seed(Din + 1)
        x_full, dy_full = torch.randn(n, Din, device=R.dev, generator=gen), torch.randn(n, Dout, device=R.dev, generator=gen)
        got = dist_step(R, dg, layer, R.P.dist_sage_conv, x_full, dy_full, [layer.weight, layer.bias])
        y64, dx64, g64 = sage_layer_f64(layer, full, x_full, dy_full, aggr == "mean")
        for k, a, r in zip(("y", "dx", "dW", "db"), got, [y64[ids], dx64[ids]] + g64):
            err, at = rel_err(a, r)
            R.put(f"layer/{tag}/sage_{aggr}_{Din}/{k}", err <= TOL_LAYER, err, at)


def check_errors(R, dg):
    P, gnn = R.P, R.gnn
    x = gnn.unrows(torch.randn(dg.n_local, 16, device=R.dev))
    cases = {"self_loops_mismatch": lambda: P.dist_gat_conv(gat_layer(R, 32, 4, True, not dg.self_loops), dg, x),
             "shape": lambda: P.dist_gat_conv(R.gnn.GATConv(16, 3, heads=2, add_self_loops=dg.self_loops, device=R.dev), dg, x),
             "dropout": lambda: P.dist_gat_conv(R.gnn.GATConv(16, 32, heads=4, add_self_loops=dg.self_loops, dropout=0.5,
                                                              device=R.dev), dg, x),
             "sage_max": lambda: P.dist_sage_conv(R.gnn.SAGEConv(16, 8, aggr=max, device=R.dev), dg, x)}
    if dg.self_loops:
        cases["sage_self_loops"] = lambda: P.dist_sage_conv(R.gnn.SAGEConv(16, 8, device=R.dev), dg, x)
    for name, f in cases.items():
        try:
            f()
            ok = False
        except ValueError:
            ok = True
        R.put(f"errors/{'loops' if dg.self_loops else 'noloops'}/{name}", ok)


def check_steps(R, G, own):
    """three steps with different x on one DistGraph equal fresh one-step runs bit for bit (GAT at C = 1, where the Wx
    and er exchanges have equal widths, and at D = 128; SAGE mean), with two push buffers and with one"""
    n = N_NODES
    R.set_route()
    runs = [("gat_C1", lambda: gat_layer(R, 1, 8, True, True), R.P.dist_gat_conv, 16, 8, True, gat_params),
            ("gat_C32", lambda: gat_layer(R, 32, 4, False, True), R.P.dist_gat_conv, 16, 32, True, gat_params),
            ("sage_mean", lambda: R.gnn.SAGEConv(128, 128, torch.relu, device=R.dev), R.P.dist_sage_conv, 128, 128, False,
             lambda l: [l.weight, l.bias])]
    for nbuf in ("2", "1"):
        os.environ["GNNB_HALO_BUFFERS"] = nbuf
        for name, make, run, Din, Dout, loops, params in runs:
            torch.manual_seed(3)
            layer = make()
            xs = [torch.randn(n, Din, device=R.dev, generator=torch.Generator(device=R.dev).manual_seed(60 + k)) for k in range(3)]
            dy = torch.randn(n, Dout, device=R.dev, generator=torch.Generator(device=R.dev).manual_seed(59))
            dg, _ = R.build(G, loops, False, **own)
            steps = [dist_step(R, dg, layer, run, x, dy, params(layer)) for x in xs]
            dg.close()
            for k, x in enumerate(xs):
                fresh, _ = R.build(G, loops, False, **own)
                once = dist_step(R, fresh, layer, run, x, dy, params(layer))
                fresh.close()
                for i, (a, b) in enumerate(zip(steps[k], once)):
                    R.put(f"steps/{own['ownership']}/buffers{nbuf}/{name}/step{k}/{i}", *bits_record(a, b))
    os.environ["GNNB_HALO_BUFFERS"] = "2"


def run_cases(R, multi_device):
    G = dict(zip(("s", "t"), make_graph()))
    fulls = {}
    cases = ownership_cases(R.W) if R.W > 1 else [(o, dict(ownership=o)) for o in ("contiguous", "cyclic", "balanced")]
    for tag, own in cases:
        for loops in (True, False):
            full_tag = f"W{R.W}/{tag}/{'loops' if loops else 'noloops'}"
            full = fulls.get(loops) or fulls.setdefault(loops, Full(R, G, loops))
            dg, req = R.build(G, loops, False, **own)
            halos = check_structure(R, full_tag, dg, req, Reference(R, G, loops))
            check_dz_exchange(R, full_tag, dg, halos)
            check_edge_part(R, full_tag, dg, full)
            check_layers(R, full_tag, dg, full, loops)
            check_errors(R, dg)
            dg.close()
    if R.W > 1:
        for tag, own in ownership_cases(R.W)[1:3]:
            check_steps(R, G, own)


def gat_worker(rank, W, port, q, multi_device):
    import torch.distributed as dist
    os.environ.update(MASTER_ADDR="127.0.0.1", MASTER_PORT=str(port), GNNB_HALO="push", GNNB_HALO_SLICES="1",
                      GNNB_HALO_BUFFERS="2")
    dev = torch.device("cuda", rank if multi_device else 0)
    torch.cuda.set_device(dev)
    try:
        dist.init_process_group("nccl" if multi_device else "gloo", rank=rank, world_size=W,
                                timeout=datetime.timedelta(seconds=300), device_id=dev if multi_device else None)
        R = Rank(rank, W, q, dev)
        run_cases(R, multi_device)
        torch.cuda.synchronize(dev)
        dist.barrier()
        q.put(("done", rank, True, 0.0, -1))
    except BaseException:
        q.put(("error", rank, False, 0.0, traceback.format_exc()[-4000:]))
    finally:
        if dist.is_initialized():
            dist.destroy_process_group()


@pytest.mark.parametrize("W", [1, 2, 3, 4])
@pytest.mark.parametrize("check", ["edge", "dz", "layer", "steps", "errors"])
def test_gat_sage_partition_on_one_device(W, check):
    """W gloo ranks on one device: `check` names the family of records"""
    require_shared_device()
    if W == 1 and check == "steps":
        pytest.skip("the repeated-steps check runs at W > 1")
    assert_records(*run_group(gat_worker, W, False), prefix=check + "/")


def test_gat_sage_partition_one_rank_per_device_nccl():
    """one rank per device under NCCL, the push route over real peer mappings"""
    if not torch.cuda.is_available() or torch.cuda.device_count() < 2:
        pytest.skip("needs at least two visible CUDA devices: NCCL refuses two ranks on one device")
    W = min(torch.cuda.device_count(), 4)
    records, errors, codes = run_group(gat_worker, W, True)
    for prefix in ("edge/", "dz/", "layer/", "steps/", "errors/"):
        assert_records(records, errors, codes, prefix)
