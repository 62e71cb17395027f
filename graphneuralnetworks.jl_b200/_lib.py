"""ctypes binding of libgnnb200.so (include/gnnb200.h).

The library is built in-tree by ``__graft_entry__.build()`` (csrc/Makefile) and must exist: there is no
Python/CPU fallback for any compute entry — a missing or stale library raises ImportError here, and a
missing GPU makes every compute call raise ``GNNBError`` (status GNNB_ECUDA).
"""
from __future__ import annotations

import ctypes as C
import os
import re

_HERE = os.path.dirname(os.path.abspath(__file__))
LIB_PATH = os.path.join(_HERE, "lib", "libgnnb200.so")
HEADER_PATH = os.path.join(os.path.dirname(_HERE), "include", "gnnb200.h")

# status codes (gnnb_status)
OK, EINVAL, ESIZE, ECUDA, ENOMEM, EUNSUPPORTED, EINDEX = range(7)
# enums
COPY_XJ, W_MUL_XJ = 0, 1
SUM, MEAN, MAX, MIN = 0, 1, 2, 3
SRC, DST = 0, 1
DIR_OUT, DIR_IN, DIR_BOTH = 0, 1, 2
CODES_DIRECTED, CODES_DIRECTED_NOLOOP, CODES_UNDIRECTED, CODES_UNDIRECTED_NOLOOP, CODES_BIPARTITE = range(5)
KEY_F32, KEY_F64, KEY_I32, KEY_I64 = range(4)


class GNNBError(RuntimeError):
    """CUDA / allocation / unsupported errors from libgnnb200."""

    def __init__(self, status: int, msg: str):
        super().__init__(f"libgnnb200 status {status}: {msg}")
        self.status = status


def _raise(status: int) -> None:
    msg = lib.gnnb_last_error().decode("utf-8", "replace")
    if status in (ESIZE, EINDEX):
        # the reference's `@assert` failures (GNNGraphs/src/utils.jl:1-28, convert.jl:49-54)
        raise AssertionError(msg)
    if status == EINVAL:
        # the reference's ArgumentError (GNNlib/src/layers/conv.jl:3-10,22)
        raise ValueError(msg)
    raise GNNBError(status, msg)


def check(status: int) -> None:
    if status != OK:
        _raise(status)


def declared_symbols() -> list[str]:
    """Every function name include/gnnb200.h declares (used by the export test)."""
    with open(HEADER_PATH) as f:
        text = f.read()
    text = re.sub(r"/\*.*?\*/", "", text, flags=re.S)
    return sorted(set(re.findall(r"\b(gnnb_[a-z0-9_]+)\s*\(", text)))


if not os.path.exists(LIB_PATH):
    raise ImportError(
        f"{LIB_PATH} is missing: run `python -c 'import __graft_entry__ as g; g.build()'` "
        "(there is no CPU fallback for the message-passing kernels)")

lib = C.CDLL(LIB_PATH)

_vp, _i64, _i32, _f32p, _int = C.c_void_p, C.c_int64, C.c_int32, C.c_void_p, C.c_int

_SIGS = {
    "gnnb_last_error": (C.c_char_p, []),
    "gnnb_version": (C.c_char_p, []),
    "gnnb_device_count": (_int, []),
    "gnnb_launch_count": (_i64, []),
    "gnnb_graph_create": (_int, [C.POINTER(_vp), _vp, _vp, _i64, _i64, _i64, _int, _int, _int, _vp]),
    "gnnb_graph_destroy": (_int, [_vp]),
    "gnnb_graph_add_self_loops": (_int, [_vp, C.POINTER(_vp), _vp]),
    "gnnb_graph_subgraph": (_int, [_vp, _vp, _vp, _i64, C.POINTER(_vp), _vp, _vp, C.POINTER(_i64), C.POINTER(_i64),
                                   _vp]),
    "gnnb_bernoulli_keep": (_int, [_i64, C.c_double, C.c_uint64, _vp, _vp]),
    "gnnb_graph_info": (_int, [_vp, C.POINTER(_i64), C.POINTER(_i64), C.POINTER(_i64)]),
    "gnnb_graph_csr": (_int, [_vp, _int, _vp, _vp, _vp, _vp]),
    "gnnb_degree": (_int, [_vp, _int, _f32p, _f32p, _vp]),
    "gnnb_gather": (_int, [_vp, _int, _f32p, _i64, _f32p, _vp]),
    "gnnb_scatter": (_int, [_vp, _int, _int, _f32p, _i64, _f32p, _vp]),
    "gnnb_propagate": (_int, [_vp, _int, _int, _int, _f32p, _f32p, _f32p, _f32p, _i64, _f32p, _vp]),
    "gnnb_propagate_bwd": (_int, [_vp, _int, _int, _f32p, _f32p, _f32p, _f32p, _f32p, _f32p, _i64, _f32p,
                                  _f32p, _vp]),
    "gnnb_softmax_edge_neighbors": (_int, [_vp, _f32p, _i64, _f32p, _vp]),
    "gnnb_softmax_edge_neighbors_bwd": (_int, [_vp, _f32p, _f32p, _i64, _f32p, _vp]),
    "gnnb_gcn_norm": (_int, [_vp, _f32p, _f32p, _vp]),
    "gnnb_gcn_propagate": (_int, [_vp, _int, _f32p, _f32p, _f32p, _i64, _f32p, _vp]),
    "gnnb_gcn_propagate_bipartite": (_int, [_vp, _int, _f32p, _i64, _f32p, _vp]),
    "gnnb_gat_aggregate": (_int, [_vp, _f32p, _f32p, _f32p, _i64, _i64, C.c_float, _f32p, _f32p, _f32p,
                                  _f32p, _vp]),
    "gnnb_gat_aggregate_bwd": (_int, [_vp, _f32p, _f32p, _f32p, _f32p, _f32p, _f32p, _f32p, _i64, _i64, C.c_float,
                                      _f32p, _f32p, _f32p, _vp]),
    "gnnb_linear": (_int, [_f32p, _f32p, _f32p, _int, _i64, _i64, _i64, _f32p, _vp]),
    "gnnb_bias_act": (_int, [_f32p, _f32p, _int, _i64, _i64, _f32p, _vp]),
    "gnnb_bias_act_bwd": (_int, [_f32p, _f32p, _int, _i64, _i64, _f32p, _f32p, _vp]),
    "gnnb_linear_bwd": (_int, [_f32p, _f32p, _f32p, _f32p, _int, _i64, _i64, _i64, _f32p, _f32p, _f32p, _f32p, _vp]),
    "gnnb_linear_relu_mask": (_int, [_f32p, _f32p, _f32p, _i64, _i64, _i64, _f32p, _vp, _vp]),
    "gnnb_linear_bwd_mask": (_int, [_f32p, _vp, _f32p, _f32p, _i64, _i64, _i64, _f32p, _f32p, _f32p, _vp]),
    "gnnb_dense_set_emulation": (_int, [_int]),
    "gnnb_dense_set_tensor_core_kernel": (_int, [_int]),
    "gnnb_dense_tc_error": (_int, []),
    "gnnb_dense_emulation_active": (_int, []),
    "gnnb_gather_rows": (_int, [_vp, _i64, _f32p, _i64, _f32p, _vp]),
    "gnnb_propagate_halo": (_int, [_vp, _int, _int, _f32p, _f32p, _i64, _f32p, _f32p, _f32p, _i64, _f32p, _vp]),
    "gnnb_propagate_maxmin_bwd_halo": (_int, [_vp, _int, _int, _f32p, _f32p, _f32p, _f32p, _f32p, _i64, _f32p, _i64, _f32p,
                                              _vp]),
    "gnnb_gat_aggregate_halo": (_int, [_vp, _f32p, _f32p, _i64, _f32p, _f32p, _i64, _i64, C.c_float, _f32p, _f32p, _f32p,
                                       _vp]),
    "gnnb_gat_aggregate_bwd_halo": (_int, [_vp, _f32p, _f32p, _f32p, _f32p, _i64, _f32p, _f32p, _f32p, _f32p, _i64, _i64,
                                           C.c_float, _f32p, _f32p, _f32p, _vp]),
    "gnnb_gat_tnode": (_int, [_f32p, _f32p, _i64, _i64, _i64, _f32p, _vp]),
    "gnnb_gcn_edge_weight_grad_halo": (_int, [_vp, _f32p, _f32p, _f32p, _i64, _f32p, _f32p, _f32p, _i64, _f32p, _vp]),
    "gnnb_dev_alloc": (_int, [C.POINTER(_vp), _i64]),
    "gnnb_dev_free": (_int, [_vp]),
    "gnnb_ipc_get_handle": (_int, [_vp, _vp]),
    "gnnb_ipc_open_handle": (_int, [_vp, C.POINTER(_vp)]),
    "gnnb_ipc_close_handle": (_int, [_vp]),
    "gnnb_halo_push": (_int, [_vp, _vp, _vp, _vp, _int, _f32p, _i64, _vp]),
    "gnnb_sort_edge_index": (_int, [_vp, _vp, _i64, _i64, _int, _vp, _vp, _vp, _vp]),
    "gnnb_coalesce_edges": (_int, [_vp, _vp, _i64, _i64, _int, _int, _vp, _vp, _vp, _vp, C.POINTER(_i64), _vp]),
    "gnnb_graph_csr_device": (_int, [_vp, _int, _vp, _vp, _vp, _vp]),
    "gnnb_sample_neighbors": (_int, [_vp, _vp, _i64, _int, _int, _i64, _int, _int, C.c_uint64, _vp, _vp, _i64,
                                     C.POINTER(_i64), _vp]),
    "gnnb_knn": (_int, [_f32p, _i64, _int, _vp, _i64, _int, _int, _vp, _vp]),
    "gnnb_radius_count": (_int, [_f32p, _i64, _int, _vp, _i64, C.c_float, _int, _vp, C.POINTER(_i64), _vp]),
    "gnnb_radius_fill": (_int, [_f32p, _i64, _int, _vp, _i64, C.c_float, _int, _vp, _vp, _i64, _vp]),
    "gnnb_temporal_radius_points": (_int, [_i64, _i64, C.c_double, C.c_uint64, _f32p, _vp]),
    "gnnb_temporal_hyperbolic_records": (_int, [_i64, _i64, C.c_double, C.c_double, C.c_double, C.c_double, C.c_uint64,
                                                _vp, _vp]),
    "gnnb_hyperbolic_count": (_int, [_vp, _i64, _vp, _i64, C.c_double, _int, _vp, C.POINTER(_i64), _vp]),
    "gnnb_hyperbolic_fill": (_int, [_vp, _i64, _vp, _i64, C.c_double, _int, _vp, _vp, _i64, _vp]),
    "gnnb_random_walk_pe": (_int, [_vp, _f32p, _f32p, _vp, _i64, _int, _f32p, _vp]),
    "gnnb_ppr_diffusion": (_int, [_vp, _f32p, C.c_float, _vp, _i64, _f32p, _vp, _vp]),
    "gnnb_ppr_matrix": (_int, [_vp, _f32p, C.c_float, _i64, _i64, _i64, _f32p, _vp]),
    "gnnb_laplacian_lambda_max": (_int, [_vp, _f32p, _f32p, _int, _int, _vp, _i64, _vp, _vp, _vp]),
    "gnnb_segment_dots": (_int, [_vp, _i64, _i64, _vp, _i64, _vp, _vp, _i64, _i64, _vp, _vp, _vp]),
    "gnnb_color_refinement": (_int, [_vp, _vp, _i64, _vp, C.POINTER(_i64), C.POINTER(_i64), _vp]),
    "gnnb_set2set_attend": (_int, [_vp, _f32p, _f32p, _i64, _f32p, _f32p, _f32p, _vp]),
    "gnnb_set2set_attend_bwd": (_int, [_vp, _f32p, _f32p, _f32p, _f32p, _f32p, _f32p, _i64, _f32p, _f32p, _vp]),
    "gnnb_attention_pool": (_int, [_vp, _f32p, _f32p, _i64, _f32p, _f32p, _f32p, _vp]),
    "gnnb_attention_pool_bwd": (_int, [_vp, _f32p, _f32p, _f32p, _f32p, _f32p, _f32p, _i64, _f32p, _f32p, _vp]),
    "gnnb_topk_keep": (_int, [_vp, _int, _i64, _vp, _i64, _i64, C.c_double, _vp, _vp, _vp]),
    "gnnb_topk_score": (_int, [_f32p, _i64, _i64, _f32p, _f32p, _vp]),
    "gnnb_topk_gate": (_int, [_f32p, _i64, _i64, _f32p, _vp, _i64, _f32p, _vp, _vp]),
    "gnnb_topk_gate_bwd": (_int, [_f32p, _i64, _i64, _f32p, _f32p, _vp, _i64, _f32p, _f32p, _f32p, _vp, _vp]),
    "gnnb_topk_set_smem_max": (_int, [_i64]),
    "gnnb_gru_rz": (_int,[_f32p, _i64, _f32p, _f32p, _i64, _i64, _f32p, _f32p, _f32p, _vp]),
    "gnnb_gru_out": (_int, [_f32p, _i64, _f32p, _f32p, _f32p, _i64, _i64, _int, _f32p, _f32p, _vp]),
    "gnnb_gru_out_bwd": (_int, [_f32p, _f32p, _f32p, _f32p, _i64, _i64, _int, _f32p, _i64, _f32p, _f32p, _vp]),
    "gnnb_gru_rz_bwd": (_int, [_f32p, _f32p, _f32p, _f32p, _f32p, _i64, _i64, _f32p, _i64, _f32p, _vp]),
    "gnnb_lstm_cell": (_int, [_f32p, _i64, _f32p, _f32p, _f32p, _i64, _i64, _f32p, _f32p, _f32p, _vp]),
    "gnnb_lstm_cell_bwd": (_int, [_f32p, _f32p, _f32p, _f32p, _f32p, _f32p, _i64, _i64, _f32p, _f32p, _f32p, _f32p,
                                  _vp]),
    "gnnb_edge_encode":(_int, [_int, _i64, _i64, _vp, _vp, _i64, _int, _vp, _vp]),
    "gnnb_edge_decode": (_int, [_int, _i64, _i64, _vp, _i64, _int, _vp, _vp, _vp]),
    "gnnb_edge_codes_sorted": (_int, [_int, _i64, _i64, _vp, _vp, _i64, _int, _vp, C.POINTER(_i64), _vp]),
    "gnnb_codes_member": (_int, [_vp, _i64, _vp, _i64, _vp, _vp]),
    "gnnb_sample_codes": (_int, [C.c_uint64, _vp, _i64, _i64, C.c_uint64, _vp, C.POINTER(_i64), _vp]),
    "gnnb_sample_positions_host": (_int, [_i32, _i64, _int, C.c_uint64, C.c_uint64, _vp, _i64, C.POINTER(_i64)]),
    "gnnb_propagate_host": (_int, [_vp, _int, _int, _int, _f32p, _f32p, _i64, _f32p]),
    "gnnb_gcn_propagate_host": (_int, [_vp, _int, _f32p, _f32p, _i64, _f32p]),
    "gnnb_linear2": (_int, [_f32p, _f32p, _f32p, _f32p, _int, _i64, _i64, _i64, _i64, _f32p, _vp]),
    "gnnb_linear2_bwd": (_int, [_f32p, _f32p, _f32p, _f32p, _f32p, _int, _i64, _i64, _i64, _i64, _f32p, _f32p, _f32p, _f32p, _f32p, _vp]),
    "gnnb_gat_logit_terms": (_int, [_f32p, _f32p, _i64, _i64, _i64, _f32p, _f32p, _vp]),
    "gnnb_gat_logit_terms_bwd": (_int, [_f32p, _f32p, _f32p, _f32p, _i64, _i64, _i64, _f32p, _f32p, _vp]),
    "gnnb_gcn_conv_step_host": (_int, [_vp, _vp, _vp, _vp, _int, _i64, _i64, _vp, _vp, _vp, _vp, _vp]),
    "gnnb_rmat_edges": (_int, [_i64, _i64, C.c_uint64, _vp, _vp, _vp]),
    "gnnb_rmat_edges_range": (_int, [_i64, _i64, _i64, C.c_uint64, _vp, _vp, _vp]),
    "gnnb_shard_builder_create": (_int, [C.POINTER(_vp), _i64, _int, _int, _int, C.POINTER(_i64), _vp]),
    "gnnb_shard_builder_add": (_int, [_vp, _vp, _vp, _i64, _int, _int, _vp]),
    "gnnb_shard_builder_finish": (_int, [_vp, _int, _int, C.POINTER(_vp), C.POINTER(_i64), C.POINTER(_i64), C.POINTER(_i64),
                                         C.POINTER(_i64), _vp]),
    "gnnb_degree_accumulate": (_int, [_vp, _vp, _i64, _int, _int, _i64, _vp, _vp]),
    "gnnb_balanced_relabel": (_int, [_vp, _i64, _int, _vp, _vp, _vp]),
    "gnnb_shard_builder_halo": (_int, [_vp, _int, _vp, _vp]),
    "gnnb_shard_builder_destroy": (_int, [_vp]),
    "gnnb_set_chunk_edges": (_int, [_int]),
    "gnnb_set_kernel_variant": (_int, [_int]),
    "gnnb_gcn_hot_rows": (_int, [_vp, _int, _vp, _i64, C.POINTER(_i64), C.POINTER(C.c_int32), _vp]),
}

for _name, (_res, _args) in _SIGS.items():
    _fn = getattr(lib, _name)  # AttributeError here = stale library: fail loudly
    _fn.restype = _res
    _fn.argtypes = _args


if os.environ.get("GNNB_KERNEL_VARIANT"):          # the whole test-suite on the reference kernels (12)
    check(lib.gnnb_set_kernel_variant(int(os.environ["GNNB_KERNEL_VARIANT"])))


def device_count() -> int:
    return int(lib.gnnb_device_count())


def launch_count() -> int:
    return int(lib.gnnb_launch_count())


def version() -> str:
    return lib.gnnb_version().decode()
