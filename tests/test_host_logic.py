"""Host-side mirror of the reference interface: size checks, containers, layout helpers, batching.
CPU only (no kernels run)."""
import operator

import numpy as np
import pytest
import torch


def test_colmajor_rows_roundtrip(gnn):
    x = torch.arange(12, dtype=torch.float32).reshape(3, 4)        # Julia (3, 4)
    xc = gnn.colmajor(x)
    assert xc.shape == (3, 4) and xc.stride() == (1, 3) and torch.equal(xc, x)
    r = gnn.rows(xc)
    assert r.shape == (4, 3) and r.is_contiguous() and r.data_ptr() == xc.data_ptr()   # zero copy
    assert torch.equal(gnn.unrows(r), x)
    z = gnn.jl_zeros(2, 3, 5)
    assert z.shape == (2, 3, 5) and z.stride() == (1, 2, 6)
    assert gnn.rows(z).shape == (5, 3, 2)


def test_graph_constructors(gnn):
    g = gnn.GNNGraph([1, 1, 2, 3], [2, 2, 2, 4])
    assert (g.num_nodes, g.num_edges) == (4, 4)
    g = gnn.GNNGraph(([1, 2], [2, 3], [0.5, 1.5]), num_nodes=5)
    assert g.num_nodes == 5 and g.w.tolist() == [0.5, 1.5]
    # adjacency matrix: A[i,j] != 0 <=> edge i -> j, column-major order (GNNlib/test/test_module.jl:153-178)
    adj1 = [[0, 1, 0, 1], [1, 0, 1, 0], [0, 1, 0, 1], [1, 0, 1, 0]]
    g = gnn.GNNGraph(np.array(adj1))
    s, t = gnn.edge_index(g)
    assert s.tolist() == [2, 4, 1, 3, 2, 4, 1, 3] and t.tolist() == [1, 1, 2, 2, 3, 3, 4, 4]
    with pytest.raises(AssertionError):
        gnn.GNNGraph([1, 2], [1, 2, 3])


def test_size_checks_raise_assertion_error(gnn):
    # GNNlib/test/msgpass.jl:55-66, 118-125: wrong last dimension -> AssertionError
    g = gnn.GNNGraph(np.array([[0, 1, 0, 1], [1, 0, 1, 0], [0, 1, 0, 1], [1, 0, 1, 0]]))
    x = torch.rand(3, g.num_nodes - 1)
    with pytest.raises(AssertionError):
        gnn.apply_edges(gnn.copy_xj, g, xj=x)
    with pytest.raises(AssertionError):
        gnn.apply_edges(gnn.copy_xj, g, xi=x)
    xs = {"a": torch.rand(3, g.num_nodes), "b": torch.rand(3, g.num_nodes + 1)}
    with pytest.raises(AssertionError):
        gnn.apply_edges(gnn.copy_xj, g, xj=xs)
    e = torch.rand(3, g.num_edges - 1)
    with pytest.raises(AssertionError):
        gnn.apply_edges(gnn.copy_xj, g, e=e)
    with pytest.raises(AssertionError):
        gnn.aggregate_neighbors(g, operator.add, torch.rand(2, g.num_edges - 1))
    with pytest.raises(AssertionError):
        gnn.aggregate_neighbors(g, operator.add, (torch.rand(2, g.num_edges + 1), None))
    with pytest.raises(AssertionError):
        gnn.propagate(gnn.copy_xj, g, operator.add, xj=x)


def test_aggr_codes(gnn):
    from gnnb200.msgpass import _aggr_code
    L = gnn._lib
    assert _aggr_code(operator.add) == L.SUM == _aggr_code("+")
    assert _aggr_code(gnn.mean) == L.MEAN and _aggr_code(max) == L.MAX and _aggr_code(min) == L.MIN
    with pytest.raises(ValueError):
        _aggr_code(operator.mul)


def test_message_functions(gnn):
    xi, xj = torch.rand(3, 5), torch.rand(3, 5)
    e = torch.rand(5)
    assert gnn.copy_xj(xi, xj, e) is xj and gnn.copy_xi(xi, xj, e) is xi
    assert torch.allclose(gnn.xi_dot_xj(xi, xj, None), (xi * xj).sum(0, keepdim=True))
    assert torch.equal(gnn.xi_sub_xj(xi, xj, None), xi - xj) and torch.equal(gnn.xj_sub_xi(xi, xj, None), xj - xi)
    assert torch.equal(gnn.e_mul_xj(xi, xj, e), e.reshape(1, 5) * xj)
    assert torch.equal(gnn.w_mul_xj(xi, xj, e), e.reshape(1, 5) * xj)
    assert gnn.w_mul_xj(xi, xj, None) is xj
    x3 = torch.rand(2, 3, 5)
    assert gnn.w_mul_xj(None, x3, e).shape == (2, 3, 5)
    assert gnn.Fix1(lambda a, b, c: (a, b, c), 1)(2, 3) == (1, 2, 3)
    with pytest.raises(ValueError):
        gnn.expand_srcdst(None, torch.rand(3))


def test_batch_offsets(gnn):
    # GNNGraphs/test/transform.jl:19-54: ids offset by cumulative node counts; graph_indicator 1,1,..,2,..
    rng = np.random.default_rng(0)

    def ring(n):
        s = np.arange(1, n + 1)
        return gnn.GNNGraph(s, np.roll(s, -1), ndata={"x": gnn.colmajor(torch.rand(16, n))})

    g1, g2, g3 = ring(10), ring(4), ring(7)
    g123 = gnn.batch([g1, g2, g3])
    assert g123.graph_indicator.tolist() == [1] * 10 + [2] * 4 + [3] * 7
    s, t = gnn.edge_index(g123)
    assert s.tolist() == g1.s.tolist() + (10 + g2.s).tolist() + (14 + g3.s).tolist()
    assert t.tolist() == g1.t.tolist() + (10 + g2.t).tolist() + (14 + g3.t).tolist()
    assert torch.equal(g123.ndata["x"][:, 10:14], g2.ndata["x"])
    g6 = gnn.batch([g123, g123])
    assert g6.num_graphs == 6
    assert g6.graph_indicator.tolist() == [1] * 10 + [2] * 4 + [3] * 7 + [4] * 10 + [5] * 4 + [6] * 7


def test_layer_argument_errors(gnn):
    # GNNlib/src/layers/conv.jl:3-10,22 -> ArgumentError (ValueError here), raised before any kernel runs
    l = gnn.GCNConv(3, 5)
    g = gnn.GNNGraph([1, 2, 3], [2, 3, 1])
    x = gnn.colmajor(torch.rand(3, 3))
    with pytest.raises(ValueError):
        l(g, x, torch.rand(2))
    with pytest.raises(ValueError):
        l(g, x, conv_weight=torch.zeros(5, 4))


def test_reference_arm_prints_the_contract_line():
    """bench.py --impl reference (the oracle port of the reference's CPU path) on a tiny bounded sample: one JSON line
    with the contract's keys; rank != 0 prints nothing."""
    import json
    import os
    import subprocess
    import sys
    root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    cmd = [sys.executable, os.path.join(root, "bench.py"), "--impl", "reference", "--steps", "1", "--warmup", "1",
           "--cpu-nodes", "20000", "--cpu-edges", "100000", "--ref-sample"]
    out = subprocess.check_output(cmd, text=True, timeout=300)
    line = json.loads([l for l in out.splitlines() if l.startswith("{")][-1])
    assert line["impl"] == "reference" and line["unit"] == "edges/s" and line["value"] > 0
    for key in ("metric", "n_gpus", "steps", "warmup", "ms_per_step", "higher_is_better", "config", "cpu_baseline", "e2e"):
        assert key in line
    assert line["e2e"]["h2d_bytes_per_step"] == 0 and line["cpu_baseline"]["kind"] == "port"
    env = dict(os.environ, RANK="1", WORLD_SIZE="2")
    assert subprocess.check_output(cmd, text=True, timeout=300, env=env).strip() == ""


def _bench_module():
    import importlib.util
    import os
    root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    spec = importlib.util.spec_from_file_location("bench_under_test", os.path.join(root, "bench.py"))
    mod = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(mod)
    return mod


def test_bench_argument_surface():
    """the flags the driver and the scripts rely on"""
    import sys
    b = _bench_module()
    old = sys.argv
    try:
        sys.argv = ["bench.py", "--gpus", "8", "--steps", "4", "--warmup", "3", "--config", "5", "--no-parity", "--no-cpu", "--no-e2e"]
        a = b.parse()
    finally:
        sys.argv = old
    assert (a.gpus, a.steps, a.warmup, a.config) == (8, 4, 3, 5)
    assert a.no_parity and a.no_cpu and a.no_e2e and a.impl != "reference"
    assert (a.nodes, a.edges, a.dim) == (25_000_000, 1_000_000_000, 256)      # config 5 = BASELINE configs[4]


def test_bench_dump_outputs_samples_rows_and_caps_size(tmp_path, monkeypatch):
    """--dump-outputs: float32 files; node-indexed arrays above the per-array size share one fixed seeded row sample
    (stored as sample_rows.npy and sized by the widest array); small arrays whole; over the total cap nothing is written"""
    import os
    from types import SimpleNamespace
    import numpy as np
    b = _bench_module()
    n = 40000
    y = torch.arange(n * 128, dtype=torch.float64).reshape(n, 128)         # 20.5 MB as float32: sampled
    dx = -torch.arange(n * 160, dtype=torch.float64).reshape(n, 160)       # wider: sets the sample size
    dW = torch.rand(128, 128)
    arrays = lambda: {"y": y, "dx": dx, "dW": dW}
    b.dump_outputs(SimpleNamespace(dump_outputs=None), torch, lambda: 1 / 0)   # no flag: not even evaluated
    out = tmp_path / "d"
    b.dump_outputs(SimpleNamespace(dump_outputs=str(out)), torch, arrays)
    got = {f[:-4]: np.load(out / f) for f in os.listdir(out)}
    assert sorted(got) == ["dW", "dx", "sample_rows", "y"]
    assert all(a.dtype == np.float32 for k, a in got.items() if k != "sample_rows")
    rows = got["sample_rows"].astype(np.int64)
    assert got["sample_rows"].dtype == np.float64 and np.all(np.diff(rows) > 0) and rows[-1] < n
    assert len(rows) == b.DUMP_ARRAY_BYTES // (4 * 160)
    assert np.array_equal(got["y"], y.numpy()[rows].astype(np.float32))
    assert np.array_equal(got["dx"], dx.numpy()[rows].astype(np.float32))
    assert got["dx"].nbytes <= b.DUMP_ARRAY_BYTES and np.array_equal(got["dW"], dW.numpy())
    assert sum(a.nbytes for a in got.values()) <= b.DUMP_TOTAL_BYTES
    again = tmp_path / "again"
    b.dump_outputs(SimpleNamespace(dump_outputs=str(again)), torch, arrays)
    assert np.array_equal(np.load(again / "sample_rows.npy"), got["sample_rows"])       # seeded: same rows every run
    monkeypatch.setattr(b, "DUMP_TOTAL_BYTES", 1 << 20)
    with pytest.raises(ValueError):
        b.dump_outputs(SimpleNamespace(dump_outputs=str(tmp_path / "over")), torch, arrays)
    assert not (tmp_path / "over").exists()
