"""Times the fused GCN propagate (forward and transposed) at BASELINE configs[1] scale: the default kernels (variant 0,
plan-owned normalisation) against the reference kernels (variant 12, explicit normalisation) over several chunk sizes.
One JSON line per variant and chunk size, with the card's name, power limit and SM clock read in the same run.
Usage: [VARIANTS=12,0] [CHUNKS=128] python scripts/sweep_variants.py [nodes edges dim]"""
import json
import os
import subprocess
import sys

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import gnnb200 as gnn

n, E, D = (int(a) for a in sys.argv[1:4]) if len(sys.argv) >= 4 else (10_000_000, 100_000_000, 128)
lib = gnn._lib.lib


def card():
    out = subprocess.check_output(["nvidia-smi", "--id=0", "--query-gpu=name,power.limit,clocks.sm",
                                   "--format=csv,noheader,nounits"], text=True).strip().split(", ")
    return out[0], float(out[1]), float(out[2])


dev = torch.device("cuda", 0)
x = torch.randn(n, D, device=dev)
out = torch.empty_like(x)
res = []
CHUNKS = [int(c) for c in os.environ.get('CHUNKS', '128').split(',')]
VARIANTS = [int(v) for v in os.environ.get('VARIANTS', '12,0').split(',')]
for chunk in CHUNKS:
    gnn._lib.check(lib.gnnb_set_chunk_edges(chunk))
    g = gnn.rmat_graph(n, E, 17, device=dev)
    g2 = gnn.add_self_loops(g)
    gnn._lib.check(lib.gnnb_graph_csr(g2.plan().h, 1, None, None, None, None))
    c = gnn.layers._gcn_c(g2)
    ref = None
    for v in VARIANTS:
        gnn._lib.check(lib.gnnb_set_kernel_variant(v))
        row = {"chunk": chunk, "variant": v}
        for tr in (0, 1):
            for _ in range(2):
                gnn._lib.check(lib.gnnb_gcn_propagate(g2.plan().h, tr, x.data_ptr(), None, None if v == 0 else c.data_ptr(), D, out.data_ptr(), None))
            evs = [(torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)) for _ in range(5)]
            torch.cuda.synchronize()
            for a, b in evs:
                a.record()
                gnn._lib.check(lib.gnnb_gcn_propagate(g2.plan().h, tr, x.data_ptr(), None, None if v == 0 else c.data_ptr(), D, out.data_ptr(), None))
                b.record()
            torch.cuda.synchronize()
            row["fwd_ms" if tr == 0 else "bwd_ms"] = sum(a.elapsed_time(b) for a, b in evs) / 5
            if tr == 0:
                if ref is None:
                    ref = out.clone()
                else:
                    row["bit_identical_to_first"] = bool(torch.equal(out, ref))
        row["card"], row["power_limit_w"], row["sm_clock_mhz"] = card()
        print(json.dumps(row), flush=True)
        res.append(row)
    del g, g2, c
    torch.cuda.empty_cache()
gnn._lib.lib.gnnb_set_kernel_variant(0)
gnn._lib.lib.gnnb_set_chunk_edges(128)
