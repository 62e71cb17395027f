"""graphneuralnetworks.jl_b200 — H100-native (sm_90a) message-passing engine behind GNNlib.jl's
`propagate` / `apply_edges` / `aggregate_neighbors` API (see DESIGN.md, INTEGRATION.md).

Import name: ``gnnb200`` (the directory name contains a dot, so the repo-root shim ``gnnb200.py`` loads this
package under that name).  Product code = csrc/ (CUDA kernels + C ABI, built into lib/libgnnb200.so) and the
host-side mirror of the reference interface in this package.  Nothing here imports ``oracle/``.
"""
from . import _lib
from ._lib import GNNBError, device_count, launch_count, version
from .graph import (GNNGraph, add_self_loops, batch, colmajor, degree, edge_features, edge_index, get_edge_weight,
                    graph_features, graph_indicator, jl_randn, jl_zeros, node_features, rmat_graph, rows,
                    set_edge_weight, unrows)
from .basic import GNNChain, GNNLayer, Parallel, WithGraph
from .msgpass import (Fix1, aggregate_neighbors, apply_edges, check_num_edges, check_num_nodes, copy_xi, copy_xj,
                      e_mul_xj, expand_srcdst, mean, propagate, softmax_edge_neighbors, w_mul_xj, xi_dot_xj,
                      xi_sub_xj, xj_sub_xi)
from .layers import (AGNNConv, GATConv, GATv2Conv, GCNConv, GINConv, GatedGraphConv, GraphConv, SAGEConv, SGConv,
                     TAGConv, TransformerConv, agnn_conv, gat_conv, gat_message, gated_graph_conv, gatv2_conv,
                     gatv2_message, gcn_conv, gin_conv, graph_conv, identity, relu, sage_conv, sg_conv, sgc_conv,
                     tag_conv, transformer_conv)
from .layers_more import (CGConv, ChebConv, DConv, EdgeConv, EGNNConv, GMMConv, MEGNetConv, NNConv,
                          ResGatedGraphConv, cg_conv, cheb_conv, d_conv, edge_conv, egnn_conv, gmm_conv, megnet_conv,
                          nn_conv, res_gated_graph_conv)
from .readout import (GlobalAttentionPool, GlobalPool, Set2Set, TopKPool, broadcast_edges, broadcast_nodes,
                      global_attention_pool, global_pool, reduce_edges, reduce_nodes, set2set_pool, softmax_edges,
                      softmax_nodes, topk_index, topk_pool)
from .transform import (add_nodes, color_refinement, csr, getgraph, ppr_diffusion, random_walk_pe, remove_edges,
                        remove_multi_edges, remove_nodes, remove_self_loops, sort_edge_index, to_bidirected, unbatch)
from .temporal import (DCGRU, DCGRUCell, EvolveGCNO, EvolveGCNOCell, GConvGRU, GConvGRUCell, GConvLSTM, GConvLSTMCell,
                       GNNRecurrence, TemporalSnapshotsGNNGraph, TGCN, TGCNCell, add_snapshot, initialstates,
                       remove_snapshot)
from .generate import knn_graph, radius_graph, rand_temporal_hyperbolic_graph, rand_temporal_radius_graph
from .linkpred import (DotDecoder, add_edges, dot_decoder, edge_decoding, edge_encoding, intersect, negative_sample,
                       perturb_edges, rand_edge_split, rand_graph)
from .sampling import NeighborLoader, induced_subgraph, sample_edge_ids, sample_neighbors
from .query import (adjacency_list, adjacency_matrix, has_isolated_nodes, has_multi_edges, has_self_loops, inneighbors,
                    is_bidirected, laplacian_lambda_max, laplacian_matrix, normalized_laplacian, outneighbors,
                    scaled_laplacian)
from .hetero import (GNNHeteroGraph, HeteroGraphConv, add_edges, edge_type_subgraph, has_edge, num_edge_types,
                     num_node_types, rand_bipartite_heterograph, rand_heterograph)

__all__ = [n for n in dir() if not n.startswith("_")]
