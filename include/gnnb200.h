/*
 * gnnb200.h — C ABI of libgnnb200.so, the H100-native (sm_90a) message-passing engine that sits
 * behind GNNlib.jl's `propagate` / `apply_edges` / `aggregate_neighbors` hot path.
 *
 * Every entry point below replaces one reference interface; the citation after "replaces:" is
 * file:line under the reference tree (CarloLucibello/GraphNeuralNetworks.jl @ e46d1b04).  The Julia
 * binding a maintainer would add (`ccall`s from a package extension that mirrors
 * GNNlib/ext/GNNlibCUDAExt.jl:13-32) is shown in INTEGRATION.md and julia/GNNlibB200Ext.jl.
 *
 * Conventions
 *   - plain C: pointers + sizes only, no torch / CUDA types (`stream` is a cudaStream_t passed as
 *     void*; NULL = the legacy default stream).
 *   - every function returns a gnnb_status; 0 = ok.  gnnb_last_error() gives the thread-local text.
 *     The host shim maps GNNB_ESIZE -> AssertionError (GNNGraphs/src/utils.jl:1-28) and
 *     GNNB_EINVAL -> ArgumentError (GNNlib/src/layers/conv.jl:3-10,22).
 *   - feature arrays are Julia column-major (D, N): node n owns D contiguous floats at x + n*D.
 *     Edge arrays (K, E) likewise, in the COO order of the graph the handle was created from.
 *   - "device" entry points take device pointers, are asynchronous on `stream`, never allocate
 *     caller-visible memory and never free caller memory.  The only library-owned object is the
 *     opaque graph plan.  "_host" entry points take HOST pointers and do the H2D/D2H themselves.
 *   - there is no CPU fallback: without a CUDA device every compute entry returns GNNB_ECUDA.
 *   - concurrency: scratch the library owns is per device (a plan's workspaces; the dense and
 *     attention-logit buffers, the cuBLASLt handle and the tensor-core watchdog flag of each device,
 *     which grow only).  Calls on one device must therefore be stream-ordered with respect to each
 *     other.  Once warm, the dense, propagate and attention entries neither allocate nor
 *     synchronise, so a step of them can be captured in a CUDA graph.
 */
#ifndef GNNB200_H
#define GNNB200_H

#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

typedef enum {
    GNNB_OK = 0,
    GNNB_EINVAL = 1,       /* bad argument value        -> ArgumentError  */
    GNNB_ESIZE = 2,        /* size mismatch             -> AssertionError */
    GNNB_ECUDA = 3,        /* CUDA runtime error / no device              */
    GNNB_ENOMEM = 4,       /* device allocation failed                    */
    GNNB_EUNSUPPORTED = 5, /* valid in the reference, not in this build   */
    GNNB_EINDEX = 6        /* node index out of [base, base+N) -> AssertionError (convert.jl:49-54) */
} gnnb_status;

/* message functions with a fused path (GNNlib/src/msgpass.jl:162-208) */
typedef enum {
    GNNB_COPY_XJ = 0,  /* copy_xj(xi,xj,e) = xj                 msgpass.jl:165 */
    GNNB_W_MUL_XJ = 1  /* w_mul_xj / e_mul_xj with a vector e   msgpass.jl:191-208 */
} gnnb_msg;

/* aggregations NNlib.scatter supports that the layers use (SURVEY.md §8 a3/a5) */
typedef enum { GNNB_SUM = 0, GNNB_MEAN = 1, GNNB_MAX = 2, GNNB_MIN = 3 } gnnb_aggr;

/* which end of an edge */
typedef enum { GNNB_SRC = 0, GNNB_DST = 1 } gnnb_end;

/* degree direction (GNNGraphs/src/query.jl:314-369 `dir`) */
typedef enum { GNNB_DIR_OUT = 0, GNNB_DIR_IN = 1, GNNB_DIR_BOTH = 2 } gnnb_dir;

typedef struct gnnb_graph* gnnb_graph_t;

/* ---------------------------------------------------------------- library */

/* thread-local text of the last failure on this thread ("" if none) */
const char* gnnb_last_error(void);
/* library version string, e.g. "gnnb200 0.1 sm_90a" */
const char* gnnb_version(void);
/* number of CUDA devices visible (0 when there is none; never fails) */
int gnnb_device_count(void);
/* kernels launched by this library on the calling process since load (bench.py `gpu_launches`) */
int64_t gnnb_launch_count(void);

/* ------------------------------------------------------------------ graph
 * replaces: the COO GNNGraph value `(s, t)` that `edge_index(g)` hands to the hot path
 *           (GNNGraphs/src/query.jl:12-14, GNNGraphs/src/gnngraph.jl:108-117) plus the range
 *           validation of `to_coo` (GNNGraphs/src/convert.jl:49-54).
 * Builds the device plan: int32 0-based COO copy, CSR-by-target (stable in COO order: rowptr, col,
 * sorted targets, edge-id permutation) and, lazily on first backward/transposed use, CSR-by-source.
 *   src,dst      : E indices, `index_bytes` = 4 (Int32) or 8 (Int64), `index_base` = 1 (Julia) or 0
 *   num_src/dst  : node counts of the two ends (equal for a GNNGraph; they differ for the
 *                  [local|halo] source space of a node-partitioned shard)
 *   on_device    : 0 = src/dst are host pointers, 1 = device pointers
 * Errors: GNNB_EINDEX if any index is outside [base, base+num); GNNB_ESIZE if E or N is negative or
 *         E >= 2^31 (per-GPU shards are int32-indexed), GNNB_EINVAL for bad index_bytes/base. */
int gnnb_graph_create(gnnb_graph_t* out, const void* src, const void* dst, int64_t num_edges,
                      int64_t num_src, int64_t num_dst, int index_bytes, int index_base,
                      int on_device, void* stream);
int gnnb_graph_destroy(gnnb_graph_t g);

/* replaces: add_self_loops(g::GNNGraph{<:COO_T}) (GNNGraphs/src/transform.jl:12-28): a NEW plan
 * whose COO is [s; 1:n], [t; 1:n] (loops appended after the originals, existing loops kept).
 * Requires num_src == num_dst (GNNB_ESIZE otherwise). */
int gnnb_graph_add_self_loops(gnnb_graph_t g, gnnb_graph_t* out, void* stream);

/* replaces: the index work of remove_edges, remove_nodes, getgraph and add_nodes (GNNGraphs/src/transform.jl:121-147,
 *           212-276, 553-563, 825-888): a NEW plan for the subgraph of a square plan (num_src == num_dst, else
 *           GNNB_ESIZE), derived from the parent's CSR without a sort.
 * node_keep: n DEVICE bytes or NULL (keep all).  Kept nodes are renumbered 0.. in ascending old id, and extra_nodes >= 0
 *            (GNNB_EINVAL otherwise) isolated nodes are appended after them (add_nodes).
 * edge_keep: E DEVICE bytes, COO order, or NULL (keep all).  Edge e is kept iff edge_keep[e] != 0 and both of its
 *            endpoints are kept.
 * The child's COO is the kept edges in parent COO order, renumbered.  Its CSR-by-target is derived from the parent's,
 * and so is its CSR-by-source when the parent has built one.  Both are bit-identical to what gnnb_graph_create builds
 * from the child's COO at the same chunk size.  The child inherits the parent's chunk.
 * node_map (n int32, DEVICE, or NULL): new 0-based id, or -1 if the node was removed.
 * kept_eids (E int64, DEVICE, or NULL): 0-based parent COO ids of the kept edges, ascending.  Capacity is the parent's
 *            E, so no count-then-fill round trip is needed.
 * num_nodes_out, num_edges_out: HOST (NULL = skip).  Kept nodes + extra_nodes must be < 2^31-1 (GNNB_ESIZE).
 * One count read-back; synchronises like gnnb_graph_add_self_loops. */
int gnnb_graph_subgraph(gnnb_graph_t g, const uint8_t* node_keep, const uint8_t* edge_keep, int64_t extra_nodes,
                        gnnb_graph_t* out, int32_t* node_map, int64_t* kept_eids,
                        int64_t* num_nodes_out, int64_t* num_edges_out, void* stream);

/* keep[i] = !(u_i < p), u_i = (splitmix64(splitmix64(seed) + i) >> 11) * 2^-53, for i < n (DEVICE bytes).
 * replaces: the reference's `rand() < p` drop rule of remove_edges(g, p) / remove_nodes(g, p)
 *           (transform.jl:143-147, 273-276), drawn from a counter-based stream.
 * p must lie in [0, 1] (GNNB_EINVAL otherwise); n < 2^31-1 (GNNB_ESIZE).  Does not synchronise. */
int gnnb_bernoulli_keep(int64_t n, double p, uint64_t seed, uint8_t* keep, void* stream);

/* num_edges, num_src, num_dst of a plan */
int gnnb_graph_info(gnnb_graph_t g, int64_t* num_edges, int64_t* num_src, int64_t* num_dst);

/* Copy the plan's index arrays to HOST buffers (NULL = skip) for bit-exact checks:
 *   transposed=0: CSR by target  (rowptr[num_dst+1], col = source of each sorted edge)
 *   transposed=1: CSR by source  (rowptr[num_src+1], col = target of each sorted edge)
 *   eid[k] = 0-based COO position of sorted edge k (stable: ascending within a row).
 * replaces nothing in the reference (it has no CSR type, SURVEY.md §0.4); rowptr differences must
 * equal degree(g; dir=:in / :out) exactly (GNNGraphs/test/query.jl:49-58). */
int gnnb_graph_csr(gnnb_graph_t g, int transposed, int32_t* rowptr, int32_t* col, int32_t* eid,
                   void* stream);

/* replaces: degree(g, Float32; dir, edge_weight) -> _degree (GNNGraphs/src/query.jl:314-331,355-369)
 * w = NULL -> counts (exact integers stored as float), else sum of w (COO order, length E).
 * out has num_dst (IN), num_src (OUT) entries; BOTH requires num_src == num_dst. */
int gnnb_degree(gnnb_graph_t g, int dir, const float* w, float* out, void* stream);

/* ------------------------------------------------------- gather / scatter
 * replaces: GNNGraphs._gather -> NNlib.gather (GNNGraphs/src/gatherscatter.jl:1-5):
 *           out[:,k] = x[:, idx[k]], idx = s (GNNB_SRC) or t (GNNB_DST), COO order. (D,N)->(D,E) */
int gnnb_gather(gnnb_graph_t g, int which, const float* x, int64_t D, float* out, void* stream);

/* replaces: GNNGraphs._scatter -> NNlib.scatter(aggr, m, t; dstsize=(D,n))
 *           (GNNGraphs/src/gatherscatter.jl:12-18; called from aggregate_neighbors, msgpass.jl:145-149)
 * m is (D,E) in COO order, out (D, num_dst).  Empty targets get the op's neutral element:
 * 0 for SUM/MEAN, -Inf for MAX, +Inf for MIN (NNlib semantics, SURVEY.md §8 a5).
 * which = GNNB_DST scatters by target (aggregate_neighbors); GNNB_SRC scatters by source into
 * (D, num_src) (the pullback of gather by s). */
int gnnb_scatter(gnnb_graph_t g, int which, int aggr, const float* m, int64_t D, float* out,
                 void* stream);

/* ------------------------------------------------------------- propagate
 * replaces: propagate(copy_xj | w_mul_xj | e_mul_xj(vector e), g, + | mean | max | min; xj)
 *           = aggregate_neighbors(g, aggr, apply_edges(f, g, xi, xj, e))   (msgpass.jl:71-79),
 *           its CPU SpMM specialisations (msgpass.jl:215-238) and the CUDA-ext re-routing
 *           (GNNlib/ext/GNNlibCUDAExt.jl:13-32) — fused: no (D,E) intermediate.
 *   out[:,i] = ct[i] * AGG_{k in N(i)} ( w[k] * cs[s_k] * x[:, s_k] )
 *   x  (D, num_src), out (D, num_dst); w NULL or E floats in COO order (required for W_MUL_XJ when E > 0);
 *   cs NULL or num_src floats, ct NULL or num_dst floats: optional per-node scales fused into the
 *   load / store (GCN's 1/sqrt(d), conv.jl:57-67).  MEAN divides by the in-degree (0 for isolated).
 *   transposed != 0 runs the same reduction on the reversed graph (x is (D,num_dst), out (D,num_src)):
 *   that is the pullback of the SUM/MEAN forward w.r.t. xj (SURVEY.md §9).  cs still scales the
 *   gathered node and ct the output row, so there cs has num_dst entries and ct num_src, and MEAN
 *   divides by the out-degree. */
int gnnb_propagate(gnnb_graph_t g, int transposed, int msg, int aggr, const float* x,
                   const float* w, const float* cs, const float* ct, int64_t D, float* out,
                   void* stream);

/* Pullbacks of gnnb_propagate (what Zygote computes today through NNlib's rrules, SURVEY.md §9).
 *   dout (D,num_dst).  dx (D,num_src) or NULL.  dw (E, COO order) or NULL (W_MUL_XJ only).
 *   SUM/MEAN: dx[:,j] = cs[j] * sum_{k: s_k=j} w_k * ct'[t_k] * dout[:,t_k]   (ct' = ct/deg for MEAN)
 *             dw[k]   = ct'[t_k] * cs[s_k] * <dout[:,t_k], x[:,s_k]>
 *   MAX/MIN : needs x and the forward output `out_fwd`; every tied arg-extremum receives the
 *             gradient (NNlib rule): dx[:,j] += w_k cs[j] ct[t_k] dout[:,t_k] .* (m_k .== out_fwd[:,t_k]/ct[t_k])
 *             (dw unsupported for MAX/MIN: GNNB_EUNSUPPORTED). */
int gnnb_propagate_bwd(gnnb_graph_t g, int msg, int aggr, const float* dout, const float* x,
                       const float* w, const float* cs, const float* ct, const float* out_fwd,
                       int64_t D, float* dx, float* dw, void* stream);

/* ------------------------------------------------------------ edge softmax
 * replaces: softmax_edge_neighbors(g, e) (GNNlib/src/utils.jl:84-97): for every leading index,
 *           a softmax over the edges that share a target.  e, out are (K,E) in COO order. */
int gnnb_softmax_edge_neighbors(gnnb_graph_t g, const float* e, int64_t K, float* out, void* stream);
/* pullback: de_k = a_k (da_k - sum_{k' in N(i)} a_k' da_k'), a = forward output. */
int gnnb_softmax_edge_neighbors_bwd(gnnb_graph_t g, const float* alpha, const float* dalpha,
                                    int64_t K, float* de, void* stream);

/* --------------------------------------------------------------- GCN core
 * replaces: the message-passing core of gcn_conv (GNNlib/src/layers/conv.jl:52-67):
 *     d = degree(g, T; dir=:in, edge_weight); c = 1 ./ sqrt.(d)       (default norm_fn, conv.jl:99)
 *     out = (propagate(copy_xj | e_mul_xj, g, +, xj = x .* c')) .* c'
 * `g` must already carry the self loops if the layer adds them (gnnb_graph_add_self_loops).
 * w NULL or E floats (COO order of g, loop weights included).  c_out (num_dst floats) receives c
 * (kept by the caller for the backward).  transposed=1 computes the pullback w.r.t. x given dout
 * and the forward's c:  dx = c .* (A^T-propagate(dout .* c)).
 * c == NULL (w must be NULL too): the plan's own c = 1 ./ sqrt.(in-degree), computed once and kept with the plan
 * together with its per-edge stream c[s_k] in plan order, which spares the kernel one dependent gather per edge. */
int gnnb_gcn_norm(gnnb_graph_t g, const float* w, float* c_out, void* stream);
int gnnb_gcn_propagate(gnnb_graph_t g, int transposed, const float* x, const float* w,
                       const float* c, int64_t D, float* out, void* stream);
/* The hot set behind the plan-owned normalisation's L2 policy (built with that stream if it is not yet): the nodes
 * gathered at least `threshold` times in one direction, `threshold` the smallest count whose nodes fit 0.56 of the
 * device's L2 as rows of 128 floats.  Writes the threshold and the number of hot nodes, and up to `capacity` of the
 * nodes (0-based, unordered) to the HOST array rows_host (may be NULL). */
int gnnb_gcn_hot_rows(gnnb_graph_t g, int transposed, int32_t* rows_host, int64_t capacity, int64_t* num_rows,
                      int32_t* threshold, void* stream);
/* The two-sided normalisation of gcn_conv on a one-relation heterograph (GNNlib/src/layers/conv.jl:45-50,58-66):
 *     c_src = 1 ./ sqrt.(out-degree)   (num_src floats)      c_dst = 1 ./ sqrt.(in-degree)   (num_dst floats)
 *     out = (propagate(copy_xj, g, +, xj = x .* c_src')) .* c_dst'          (x: num_src rows, out: num_dst rows)
 * transposed=1 is the pullback: dx (num_src rows) = c_src .* (A^T-propagate(dout .* c_dst)), dout num_dst rows.
 * Unweighted degrees, as the reference's heterograph branch.  Both scale vectors and their per-edge streams (c_src[s_k]
 * in the by-target plan order, c_dst[t_k] in the by-source order) are built once and kept with the plan, apart from the
 * symmetric scales of gnnb_gcn_propagate: a square plan may be asked for both normalisations.  Any num_src / num_dst
 * (num_src == num_dst included).  A target without in-edges gets a zero row, a source without out-edges a zero
 * gradient (the reference's 0 * 1/sqrt(0) is NaN there). */
int gnnb_gcn_propagate_bipartite(gnnb_graph_t g, int transposed, const float* x, int64_t D, float* out, void* stream);

/* --------------------------------------------------------------- GAT core
 * replaces: the edge part of gat_conv + gat_message (GNNlib/src/layers/conv.jl:136-141,152-167):
 *     logα_k[h] = leakyrelu(el[h,t_k] + er[h,s_k], slope)          (a·[Wx_i;Wx_j], SURVEY.md §3.2)
 *     α = softmax_edge_neighbors(g, logα);  out[:,h,i] = Σ_k α_k[h] Wx[:,h,s_k]
 * Wx (C,H,num_src), el (H,num_dst), er (H,num_src), out (C,H,num_dst).
 * Optional outputs (NULL = skip): alpha (H,E) in COO order; seg_max, seg_sum (H,num_dst) — the
 * per-target softmax statistics the backward recomputes α from. */
int gnnb_gat_aggregate(gnnb_graph_t g, const float* Wx, const float* el, const float* er,
                       int64_t C, int64_t H, float slope, float* out, float* alpha,
                       float* seg_max, float* seg_sum, void* stream);
/* pullback: given dout (C,H,num_dst), the forward output and the forward statistics, produce
 *   dWx (C,H,num_src) = Σ_{k: s_k=j} α_k dout[:,:,t_k]        (attention-weighted transposed pull, α recomputed)
 *   del (H,num_dst), der (H,num_src): gradients of the two per-node logit terms
 * (the el/er -> a, Wx chain is dense per-node work left to the caller's AD). */
int gnnb_gat_aggregate_bwd(gnnb_graph_t g, const float* Wx, const float* el, const float* er,
                           const float* seg_max, const float* seg_sum, const float* out_fwd,
                           const float* dout, int64_t C, int64_t H, float slope, float* dWx, float* del,
                           float* der, void* stream);

/* The per-node halves of the attention logits (csrc/gatlogit.cu) — replaces `sum(l.a .* vcat(Wxi, Wxj), dims = 1)` of
 * gat_message (GNNlib/src/layers/conv.jl:157-163), which splits into a target and a source term:
 *     el[h,i] = sum_c a[c,h] Wx[c,h,i]          er[h,j] = sum_c a[C+c,h] Wx[c,h,j]
 * Wx (C,H,N), a (2C,H) column-major as the layer stores it, el / er (H,N).  One pass over Wx.
 * Pullback: dWx_accum (C,H,N) += del[h,n] a[c,h] + der[h,n] a[C+c,h]  IN PLACE (it already holds the dWx of
 * gnnb_gat_aggregate_bwd), da (2C,H) = [sum_n del Wx ; sum_n der Wx] — deterministic (fixed-order reduction).
 * Shapes: C/4 a power of two <= 32, C*H <= 4096 (GNNB_EUNSUPPORTED otherwise).
 * One half per call (GAT across two node types, where el comes from W xi over the targets and er from W xj over the
 * sources): el or er may be NULL (not both), and the pass computes the other half alone; del or der may be NULL (not
 * both) in the pullback, which then adds that half's chain into dWx_accum and writes da with zeros in the other half. */
int gnnb_gat_logit_terms(const float* Wx, const float* a, int64_t N, int64_t C, int64_t H, float* el, float* er, void* stream);
int gnnb_gat_logit_terms_bwd(const float* Wx, const float* a, const float* del, const float* der, int64_t N, int64_t C,
                             int64_t H, float* dWx_accum, float* da, void* stream);

/* ------------------------------------------------------- dense layer part
 * replaces: l.σ.(weight * x .+ l.bias) of the conv layers (GNNlib/src/layers/conv.jl:39,69-71; :281) and its pullback.
 * Din, Dout <= 128: hand-written wgmma kernels (csrc/dense_tc.cu: 3xTF32 split, register accumulators, bias/relu
 * epilogue, W resident in shared memory); Din % 32 == 0 <= 512 and Dout % 128 == 0 <= 1024 with at
 * least 2048 nodes: the wide wgmma kernel of the same file (both operands streamed, W through cp.async.bulk; forward and
 * dx); every other shape: a library GEMM like the reference's, issued through cuBLASLt 12.9
 * with the fp32-emulated compute type where the library offers it (bf16 x9, fp32 accumulate), else the fp32 sgemm, bias (+relu) in the epilogue.  x (Din,N), W (Dout,Din) row-major as the layer stores it, bias NULL or Dout floats, y (Dout,N).
 * relu: 0 = identity, 1 = relu.  x, W or y off a 16 B boundary: the library GEMM; bias may sit anywhere.  The tensor-core
 * routes keep subnormal split parts (x around 2^-115 met the same bound as normal operands on an H100): no flush floor. */
int gnnb_linear(const float* x, const float* W, const float* bias, int relu, int64_t N, int64_t Din,
                int64_t Dout, float* y, void* stream);
/* pullback: dy (Dout,N); y = forward output (relu only); dpre_ws = (Dout,N) workspace (relu only);
 * outputs (each may be NULL): dx (Din,N), dW (Dout,Din), db (Dout).  The relu mask x upstream gradient and the bias
 * gradient are one hand-written pass (deterministic two-stage column sum): with relu or db it needs Dout % 4 == 0 <= 1024
 * and dy (relu: also y, dpre_ws) 16 B aligned, GNNB_EUNSUPPORTED otherwise; any other operand off its boundary sends its
 * product to the library GEMM. */
int gnnb_linear_bwd(const float* dy, const float* y, const float* x, const float* W, int relu, int64_t N,
                    int64_t Din, int64_t Dout, float* dpre_ws, float* dx, float* dW, float* db, void* stream);
/* The relu layer with its mask kept as bits: gnnb_linear (relu = 1) that also writes mask (N x 4 words, 16 B aligned), bit
 * by bit `y > 0` of y as stored, in a layout private to the library; gnnb_linear_bwd_mask is gnnb_linear_bwd (relu = 1)
 * reading that mask instead of y, 16 B instead of 512 per node, with the same bits in dx, dW and db.  dx and dW are both
 * required there, db may be NULL.  Both serve Dout = 128, Din in {32, 64, 96, 128} with the tensor-core kernels on
 * (gnnb_dense_set_tensor_core_kernel) and 16 B-aligned x, W, y, mask (forward) or dy, mask, x, dx (pullback; W, dW and db
 * may sit anywhere); GNNB_EUNSUPPORTED otherwise (use the y entries). */
int gnnb_linear_relu_mask(const float* x, const float* W, const float* bias, int64_t N, int64_t Din, int64_t Dout, float* y,
                          uint32_t* mask, void* stream);
int gnnb_linear_bwd_mask(const float* dy, const uint32_t* mask, const float* x, const float* W, int64_t N, int64_t Din,
                         int64_t Dout, float* dx, float* dW, float* db, void* stream);
/* σ.(W * vcat(x1, x2) .+ b) — sage_conv's dense part (GNNlib/src/layers/conv.jl:281) — without the (Din1+Din2, N) vcat
 * temporary: the two column blocks of W (Dout, Din1+Din2, row-major as the layer stores it) meet x1 (Din1,N) and x2 (Din2,N)
 * in two passes of the wgmma kernel, the second adding the first's result before bias / activation.  Pullback: dx1, dx2,
 * dW (Dout, Din1+Din2), db, each may be NULL.  Shapes: Din1, Din2 multiples of 32 <= 128, Dout = 128 (forward also Dout a
 * multiple of 16 <= 128; a second block of 128 < Din2 <= 512 with at least 2048 nodes takes the wide kernel).  16 B-aligned
 * x1, x2, W, y (forward); dy, y, dpre_ws, and x1, x2, dx1, dx2 where requested (pullback; W, dW, db anywhere);
 * GNNB_EUNSUPPORTED otherwise (callers concatenate and use gnnb_linear). */
int gnnb_linear2(const float* x1, const float* x2, const float* W, const float* bias, int relu, int64_t N, int64_t Din1,
                 int64_t Din2, int64_t Dout, float* y, void* stream);
int gnnb_linear2_bwd(const float* dy, const float* y, const float* x1, const float* x2, const float* W, int relu, int64_t N,
                     int64_t Din1, int64_t Din2, int64_t Dout, float* dpre_ws, float* dx1, float* dx2, float* dW, float* db,
                     void* stream);
/* y = act(x .+ bias) on (D,N) features and its pullback, for layers whose closing `σ.(x .+ bias)` follows an aggregation
 * rather than a GEMM (GATConv: GNNlib/src/layers/conv.jl:149): one pass each instead of the broadcast-add, the
 * activation, the mask product and the column reduction.  bias NULL or D floats; relu 0/1; y may alias x.
 * bwd: dpre = dy .* (y > 0) (relu only; dpre may alias dy), db = sum over nodes of dpre (NULL to skip; deterministic).
 * D % 4 == 0 (bwd: <= 1024) and x, y, bias (bwd: dy, y, dpre) 16 B aligned; GNNB_EUNSUPPORTED otherwise. */
int gnnb_bias_act(const float* x, const float* bias, int relu, int64_t N, int64_t D, float* y, void* stream);
int gnnb_bias_act_bwd(const float* dy, const float* y, int relu, int64_t N, int64_t D, float* dpre, float* db, void* stream);
/* 1 (default) = try the fp32-emulated tensor-core GEMM; 0 = force the SIMT sgemm.  *_active: -1 not yet used,
 * 0 unavailable / off, 1 in use (1 on an H100 with cuBLASLt 12.9). */
int gnnb_dense_set_emulation(int on);
/* The hand-written wgmma kernels (csrc/dense_tc.cu: 3xTF32 split, register accumulators, bias/relu epilogue) serve
 * Din, Dout <= 128 (Din % 32 == 0, Dout % 16 == 0) and the wide shapes named above for gnnb_linear and the dx part of
 * gnnb_linear_bwd (dW: Dout == 128 only); 0 switches them off (cuBLASLt everywhere).  gnnb_dense_tc_error() != 0 means one of its bounded pipeline waits expired. */
int gnnb_dense_set_tensor_core_kernel(int on);
int gnnb_dense_tc_error(void);
int gnnb_dense_emulation_active(void);

/* ------------------------------------------------- node-partitioned shards
 * (no reference counterpart: the reference has no distributed code, SURVEY.md §5/§8e.)
 * A shard is an ordinary plan whose targets are the nodes one GPU owns (num_dst = n_local) and whose
 * source ids live in the space [local rows | halo rows] (num_src = n_local + n_halo): created with
 * gnnb_graph_create(..., num_src, num_dst, ...).  The halo rows arrive through one all-to-all-v per pass
 * (NCCL, driven by the host side: graphneuralnetworks.jl_b200/partition.py).
 *
 * gnnb_gather_rows: out[k,:] = x[idx[k],:] for an explicit int32 0-based DEVICE index list — packs the rows
 * a peer requested into the send buffer. */
int gnnb_gather_rows(const int32_t* idx_dev, int64_t n, const float* x, int64_t D, float* out,
                     void* stream);
/* gnnb_propagate_halo: gnnb_propagate (forward direction of the shard plan) with the gathered rows split
 * over two buffers: node ids < n_local read x_local, the others read x_halo + (id - n_local)*D.
 * cs (optional) has num_src entries ([local | halo] order), ct num_dst.  A shard without targets (num_dst = 0, a rank
 * that owns no node) has nothing to write: out may be NULL then, and so may gnnb_gcn_norm's c_out. */
int gnnb_propagate_halo(gnnb_graph_t g, int msg, int aggr, const float* x_local, const float* x_halo,
                        int64_t n_local, const float* w, const float* cs, const float* ct, int64_t D,
                        float* out, void* stream);
/* gnnb_propagate_maxmin_bwd_halo: the MAX/MIN pullback of gnnb_propagate_halo, on the FORWARD CSR of a backward shard
 * plan (rows = owned sources j, num_dst of the plan; gathered = targets in [local | halo] order, num_src):
 *     dx[j,:] = Σ_{e: j→t, shard COO order} w_e · dout[t,:] .* (x_own[j,:]·w_e == out_fwd[t,:])     (NNlib's every-tie rule)
 * dout / out_fwd of targets < n_local read *_local, the others *_halo + (t - n_local)*D.  w: the backward shard's edge
 * weights in its COO order, or NULL (copy_xj).  A plan without rows accepts NULL outputs; a shard without halo rows
 * accepts NULL halo pointers.  SUM and MEAN are refused (GNNB_EINVAL): they pull back through gnnb_propagate_halo on the
 * backward shard.  Rows of 128 / 256 / 512 floats with 16 B-aligned operands run the work-item kernel, long rows in
 * pieces added in chunk order; other widths one warp per row.  No atomics: deterministic. */
int gnnb_propagate_maxmin_bwd_halo(gnnb_graph_t g, int msg, int aggr, const float* x_own, const float* dout_local,
                                   const float* dout_halo, const float* out_local, const float* out_halo, int64_t n_local,
                                   const float* w, int64_t D, float* dx, void* stream);
/* The fused GAT core on shards (csrc/gat.cu, the HALO instances of the same kernels; same shapes as gnnb_gat_aggregate).
 * gnnb_gat_aggregate_halo: gnnb_gat_aggregate on a forward shard plan, over its forward CSR: gathered sources < n_local
 *   read Wx_local, the others Wx_halo + (id - n_local)*C*H.  el (H, num_dst); er (H, num_src) in [local | halo] order.
 * gnnb_gat_aggregate_bwd_halo: the pullback kernel on the FORWARD CSR of a backward shard plan, whose rows are the owned
 *   sources j and whose gathered nodes are the targets in [local | halo]: dout_local / dout_halo split as above;
 *   el, seg_max, seg_sum and T (H, num_src of the shard) in [local | halo] order; Wx_own (C,H,num_dst), er_own
 *   (H,num_dst).  Writes dWx (C,H,num_dst), der (H,num_dst) and dz (H, E) in the shard plan's COO order, unscattered:
 *   del of a target is the sum of the dz of its in-edges, which live on the ranks that own their sources.
 * gnnb_gat_tnode: T[h,i] = <dout[:,h,i], out[:,h,i]> over n nodes, the per-target term gnnb_gat_aggregate_bwd computes.
 * A shard without targets (num_dst = 0) accepts NULL outputs; a shard without halo rows accepts a NULL halo pointer. */
int gnnb_gat_aggregate_halo(gnnb_graph_t g, const float* Wx_local, const float* Wx_halo, int64_t n_local, const float* el,
                            const float* er, int64_t C, int64_t H, float slope, float* out, float* seg_max, float* seg_sum,
                            void* stream);
int gnnb_gat_aggregate_bwd_halo(gnnb_graph_t g, const float* Wx_own, const float* er_own, const float* dout_local,
                                const float* dout_halo, int64_t n_local, const float* el, const float* seg_max,
                                const float* seg_sum, const float* T, int64_t C, int64_t H, float slope, float* dWx,
                                float* der, float* dz, void* stream);
int gnnb_gat_tnode(const float* dout, const float* out_fwd, int64_t n, int64_t C, int64_t H, float* T, void* stream);
/* gnnb_gcn_edge_weight_grad_halo: the edge-weight gradient of the weighted GCN propagate y_t = ct[t] Σ_{e: s→t} w_e cs[s]
 * h_s on the forward CSR of a (shard) plan:
 *     dw[e] = Σ_f (dout[t,f] * ct[t]) * (h[s,f] * cs[s]) + dd[t]        for every edge e = (s → t), COO order,
 * each product rounded as written (an infinite scale gives the IEEE results of the scaled rows).  dout (num_dst, D);
 * gathered sources < n_local read h_local, the others h_halo + (id - n_local)*D; cs (num_src, [local | halo] order), ct
 * and dd (num_dst) are optional (NULL: 1, 1, 0).  dd is the caller's degree term -½ d^{-3/2} dc of c = d^{-1/2}.  One warp
 * per work item of the plan, every value written once without atomics (deterministic).  h_halo NULL with n_local =
 * num_src is the one-base pass over an ordinary plan.  A plan without edges accepts NULL pointers. */
int gnnb_gcn_edge_weight_grad_halo(gnnb_graph_t g, const float* dout, const float* h_local, const float* h_halo,
                                   int64_t n_local, const float* cs, const float* ct, const float* dd, int64_t D,
                                   float* dw, void* stream);

/* Building one rank's shards on its GPU from chunks of the global edge list (csrc/shard.cu).
 *   ownership mode 0: contiguous ranges, bounds_host[q] <= v < bounds_host[q+1] (world + 1 entries; NULL = equal ranges);
 *   mode 1: cyclic — node v (0-based) belongs to rank v % world as its local row v / world, which spreads the hubs of a
 *   skewed id space over all ranks.  relabel_dev (mode 1, optional, DEVICE int32[num_nodes], alive until destroy):
 *   a permutation node -> position; the cyclic rule is applied to the position.  With positions = rank of the node by
 *   decreasing degree, the nodes are dealt to the ranks like cards: edge counts, node counts and the rows every rank must
 *   serve to its peers are all balanced, whatever the id space looks like (RMAT probabilities are products over id
 *   bits, so neither id ranges nor id % world balance it).
 * add(): a chunk of the global COO (DEVICE arrays, index_bytes 4|8, index_base 0|1; GNNB_EINDEX if out of range); keeps,
 *   stably, the edges whose target this rank owns (forward shard, direction 0) and those whose source it owns (backward
 *   shard, direction 1).  Synchronises the stream.
 * finish(direction): deduplicated sorted halo list, gathered nodes renamed into [local | halo], optional self loops
 *   (i, i) appended after the originals, plan created (*plan_out: an ordinary gnnb_graph_t, num_dst = n_local,
 *   num_src = n_local + n_halo; the caller destroys it).  recv_counts_host[q] (world entries) = halo rows owned by rank q.
 * halo(direction): the owner-local row index (int32, 0-based) of every halo entry, grouped by owner in rank order — what
 *   this rank asks each owner to send (n_halo entries, DEVICE). */
typedef struct gnnb_shard_builder* gnnb_shard_builder_t;
int gnnb_shard_builder_create(gnnb_shard_builder_t* out, int64_t num_nodes, int world, int rank, int mode,
                              const int64_t* bounds_host, const int32_t* relabel_dev);
int gnnb_shard_builder_add(gnnb_shard_builder_t b, const void* src, const void* dst, int64_t n, int index_bytes,
                           int index_base, void* stream);
int gnnb_shard_builder_finish(gnnb_shard_builder_t b, int direction, int add_self_loops, gnnb_graph_t* plan_out,
                              int64_t* n_local_out, int64_t* n_halo_out, int64_t* num_edges_out, int64_t* recv_counts_host,
                              void* stream);
int gnnb_shard_builder_halo(gnnb_shard_builder_t b, int direction, int32_t* halo_local_dev, void* stream);
int gnnb_shard_builder_destroy(gnnb_shard_builder_t b);
/* The relabel table of the degree-balanced deal: cost_dev (int32[num_nodes], zeroed by the caller) accumulates in + out
 * degree over chunks of the edge list; gnnb_balanced_relabel sorts the nodes by decreasing cost (stable) and deals them to
 * the ranks in turn, reversing direction every round: relabel_dev[node] = position (what gnnb_shard_builder_create takes),
 * order_dev[position] = node (rank q's local row k is node order_dev[k * world + q]). */
int gnnb_degree_accumulate(const void* src, const void* dst, int64_t n, int index_bytes, int index_base, int64_t num_nodes,
                           int32_t* cost_dev, void* stream);
int gnnb_balanced_relabel(const int32_t* cost_dev, int64_t num_nodes, int world, int32_t* relabel_dev, int32_t* order_dev,
                          void* stream);

/* Halo exchange without a staging copy: every rank writes the rows a peer asked for straight into that peer's halo
 * buffer over NVLink (peer-mapped memory).  gnnb_dev_alloc / gnnb_ipc_* manage exportable device buffers (plain
 * cudaMalloc + CUDA IPC handles, 64 bytes each, exchanged by the host side); gnnb_halo_push launches ONE kernel:
 * row k of the send list (grouped by peer: rows [seg_start[p], seg_start[p+1]) go to peer p) is copied from
 * x[send_idx[k],:] to peer_base[p] + (peer_row0[p] + k - seg_start[p])*D.  seg_start (world+1), peer_base (world),
 * peer_row0 (world) are HOST arrays.  Completion on the peers is published by a collective the caller issues on the
 * same stream afterwards. */
int gnnb_dev_alloc(void** p, int64_t bytes);
int gnnb_dev_free(void* p);
int gnnb_ipc_get_handle(void* p, unsigned char* handle64);
int gnnb_ipc_open_handle(const unsigned char* handle64, void** p);
int gnnb_ipc_close_handle(void* p);
int gnnb_halo_push(const int32_t* send_idx_dev, const int64_t* seg_start_host, const void* const* peer_base_host,
                   const int64_t* peer_row0_host, int world, const float* x, int64_t D, void* stream);

/* ------------------------------------------------- edge-list transforms (SURVEY.md §8f rank 3)
 * replaces: sort_edge_index(u, v) (GNNGraphs/src/utils.jl:41-45: sortperm of the zipped pairs, lexicographic and
 *           stable) — for CuArrays the reference's CUDA extension copies both arrays to the host, sorts there and copies
 *           back (GNNGraphs/ext/GNNGraphsCUDAExt.jl:24-30).  Here: one 64-bit key per pair, stable device radix sort.
 * u, v, u_out, v_out: E DEVICE integers of `index_bytes` (4|8) with values in [0, max_index] (0- or 1-based ids alike;
 * GNNB_EINDEX otherwise); outputs may alias the inputs or be NULL.  perm_out (NULL or E int64, 0-based): sorted
 * position k holds input pair perm_out[k].  Synchronises the stream. */
int gnnb_sort_edge_index(const void* u, const void* v, int64_t num_edges, int64_t max_index, int index_bytes,
                         void* u_out, void* v_out, int64_t* perm_out, void* stream);
/* replaces: the index half of remove_multi_edges(g; aggr) (GNNGraphs/src/transform.jl:157-190: edge_encoding, sortperm,
 *           first-occurrence mask, running segment id) and with it to_bidirected (transform.jl:495-510).
 * src, dst: E DEVICE indices in [index_base, index_base + num_nodes) (GNNB_EINDEX otherwise).  Outputs (DEVICE,
 * caller-allocated with E entries each): src_out/dst_out — the distinct pairs in (src, dst) order, first *num_unique
 * entries valid, same width and base as the input; perm_out (int64, 0-based) — the stable sort permutation; seg_out
 * (int64, 1-based) — which distinct pair sorted edge k collapsed into, i.e. the `idxs` the reference hands to
 * `_scatter(aggr, w[perm], idxs)`; that scatter is gnnb_scatter on a plan built from (1:E, seg_out).
 * num_unique is a HOST int64.  Synchronises the stream. */
int gnnb_coalesce_edges(const void* src, const void* dst, int64_t num_edges, int64_t num_nodes, int index_bytes,
                        int index_base, void* src_out, void* dst_out, int64_t* perm_out, int64_t* seg_out,
                        int64_t* num_unique, void* stream);
/* gnnb_graph_csr with DEVICE destinations (no synchronisation): the COO -> CSR conversion as an API, for callers that
 * keep working on the device (the reference has no CSR type, SURVEY.md §0.4). */
int gnnb_graph_csr_device(gnnb_graph_t g, int transposed, int32_t* rowptr_dev, int32_t* col_dev, int32_t* eid_dev,
                          void* stream);

/* ------------------------------------------------- neighbour sampling (SURVEY.md §8f rank 4)
 * replaces: the edge selection of sample_neighbors(g, nodes, K; dir, replace) (GNNGraphs/src/sampling.jl:68-83), i.e.
 *           adjacency_list(g, nodes; dir, with_eid = true) — a scan of every edge through a Dict on the CPU
 *           (GNNGraphs/src/query.jl:176-198) — plus StatsBase.sample(eidlist[i], k; replace) per node.  The plan's CSR
 *           is that adjacency list, so only the queried rows are touched.
 * nodes: n_nodes DEVICE ids (index_bytes 4|8, index_base 0|1; GNNB_EINDEX if out of range; repeated ids are sampled
 *        independently).  dir = GNNB_DIR_IN samples among the in-edges of each node, GNNB_DIR_OUT among the out-edges.
 * Node j contributes k_j = deg_j (K <= 0), min(K, deg_j) (replace = 0) or K (replace = 1; 0 when deg_j = 0) edges.
 * offsets_dev (n_nodes + 1 int64): running sums of k_j.  eids_dev (NULL = only count): COO positions (index_base-based)
 * of the chosen edges, node after node; capacity = entries available (GNNB_ESIZE if too small).  *total_host = Σ k_j.
 * Draws are counter-based on (seed, j, draw): reproducible per call; without replacement every k-subset of a row is
 * equally likely.  Synchronises the stream. */
int gnnb_sample_neighbors(gnnb_graph_t g, const void* nodes, int64_t n_nodes, int index_bytes, int index_base,
                          int64_t K, int dir, int replace, uint64_t seed, int64_t* offsets_dev, int64_t* eids_dev,
                          int64_t capacity, int64_t* total_host, void* stream);
/* The sampler of ONE query, run on the HOST (no GPU needed): the very function the device kernel calls (compiled for
 * both sides), so that its validity and uniformity can be tested anywhere.  Writes k = k_j positions in [0, deg) to
 * out (capacity entries available) for the counter (seed, j); *k_out = k. */
int gnnb_sample_positions_host(int32_t deg, int64_t K, int replace, uint64_t seed, uint64_t j, int64_t* out,
                               int64_t capacity, int64_t* k_out);

/* --------------------------------------------------------- geometric graphs (csrc/knn.cu)
 * replaces: knn_graph(points, k; graph_indicator, self_loops) (GNNGraphs/src/generate.jl:112-145) and
 *           radius_graph(points, r; graph_indicator, self_loops) (generate.jl:196-222): a KDTree / BallTree of
 *           NearestNeighbors.jl on the CPU, graphs of a batch kept apart by a dummy coordinate.  Brute force here, exact.
 * points: n rows of d contiguous DEVICE floats (Julia's (d, n) matrix).  d2(i,j) = Σ_{f=0..d-1} (p_i[f] - p_j[f])² in
 * ascending f, every sub / mul / add rounded on its own (no FMA); a NaN d2 counts as +Inf.
 * seg_ptr: NULL (one segment) or n_seg + 1 non-decreasing DEVICE offsets from 0 to n, validated on the device
 * (GNNB_EINVAL).  A point's candidates are the points of its own segment.  n < 2^31.
 * gnnb_knn: nbr (n*k int32, 0-based, row-major) row i = the k candidates j (j == i excluded unless self_loops) with the
 *   smallest (d2, j), in ascending (d2, j).  k >= 1 and d >= 1 (GNNB_EINVAL); k > 64 or d > 256: GNNB_EUNSUPPORTED.  A
 *   non-empty segment with fewer than k (+ 1 without self loops) points: GNNB_ESIZE.
 * gnnb_radius_count: offsets (n + 1 int64) = running counts of the rows {j : sqrt_rn(d2) <= r} (j == i excluded unless
 *   self_loops); *total_host = offsets[n].  r NaN or negative: GNNB_EINVAL.
 * gnnb_radius_fill: the rows themselves, row i at nbr[offsets[i] .. offsets[i+1]) in ascending j (0-based int32);
 *   capacity < offsets[n]: GNNB_ESIZE.  offsets must come from gnnb_radius_count with the same points, r, self_loops
 *   and segments; a row whose hits differ from offsets[i+1] - offsets[i] gives GNNB_EINVAL.  A row never writes
 *   outside its own range nor outside [0, capacity).
 * All three synchronise the stream. */
int gnnb_knn(const float* points, int64_t n, int d, const int64_t* seg_ptr, int64_t n_seg, int k, int self_loops,
             int32_t* nbr, void* stream);
int gnnb_radius_count(const float* points, int64_t n, int d, const int64_t* seg_ptr, int64_t n_seg, float r,
                      int self_loops, int64_t* offsets, int64_t* total_host, void* stream);
int gnnb_radius_fill(const float* points, int64_t n, int d, const int64_t* seg_ptr, int64_t n_seg, float r,
                     int self_loops, const int64_t* offsets, int32_t* nbr, int64_t capacity, void* stream);

/* --------------------------------------------------------- temporal graph generators (csrc/tgen.cu, csrc/knn.cu)
 * replaces: rand_temporal_radius_graph(n, T, speed, r) (GNNGraphs/src/generate.jl:265-284: a BallTree per snapshot)
 *           and rand_temporal_hyperbolic_graph(n, T; α, R, speed, ζ) (generate.jl:287-297, 340-380: a dense n x n
 *           Float64 adjacency per snapshot, acosh of every ordered pair).
 * The random stream: every draw is u(i, τ, k) = (splitmix64(K + c) >> 11) * 2^-53, a double in [0, 1), with
 *   K = splitmix64(seed), c = ((τ*n + i) << 1) | k; node i, k in {0, 1} its two draws at step τ; τ = 0 is the initial
 *   placement and τ = t (1 <= t < T) the move that follows snapshot t (1-based), i.e. the one that makes row block t.
 * Both node-dynamics entries run one thread per node with fp64 state and write snapshot t's rows at t*n .. t*n + n - 1
 * of one (T*n)-row DEVICE array.  Every fp64 mul / add / sub below is rounded on its own (no FMA); 2π = 2 * 3.14159...
 * gnnb_temporal_radius_points: pts (T*n, 2) fp32, the round-to-nearest of the state (x, y).  Start x = u(i,0,0),
 *   y = u(i,0,1).  Move t: ρ = (2 speed) u(i,t,0) - speed, θ = 2π u(i,t,1), x = 1 - |1 - |x + ρ cos θ||, y likewise
 *   with sin θ (the reference's reflection as written: with speed > 1 a point can leave [0, 1]).
 * gnnb_temporal_hyperbolic_records: rec (T*n, 4) fp64 records (cosh ζr, sinh ζr, cos θ, sin θ).  Start p = u(i,0,0),
 *   θ = 2π u(i,0,1).  Move t: p += (2 speed) u(i,t,0) - speed; then p > 1 -> 1 - fmod(p, 1); then p < 0 -> |p|;
 *   θ += (2 speed) u(i,t,1) - speed (unbounded).  r = (1/α) acosh(1 + (cosh(αR) - 1) p), cosh(αR) on the host.
 *   α > 0, R >= 0, ζ > 0 and speed finite, cosh(αR) finite, else GNNB_EINVAL.
 * Both: n, T >= 0 (GNNB_EINVAL); T*n >= 2^31: GNNB_ESIZE before anything is allocated or launched.
 * gnnb_hyperbolic_count / gnnb_hyperbolic_fill: the contract of gnnb_radius_count / gnnb_radius_fill (the same
 *   segments, offsets, *total_host, rows in ascending j, recount check) on n records, with the pair test
 *   x(i, j) = C_i C_j - (S_i S_j)(c_i c_j + s_i s_j), each operation rounded on its own in that order, so that
 *   x(i, j) == x(j, i) bit for bit: j is in row i when (j != i or self_loop) and (the records are equal or
 *   x <= x_max).  A NaN x is no edge.  x_max = cosh(ζR) makes this acosh(x)/ζ <= R without an acosh per pair.
 *   records 8 B aligned, x_max not NaN (GNNB_EINVAL).
 * All four synchronise the stream. */
int gnnb_temporal_radius_points(int64_t n, int64_t T, double speed, uint64_t seed, float* pts, void* stream);
int gnnb_temporal_hyperbolic_records(int64_t n, int64_t T, double alpha, double R, double speed, double zeta,
                                     uint64_t seed, double* rec, void* stream);
int gnnb_hyperbolic_count(const double* records, int64_t n, const int64_t* seg_ptr, int64_t n_seg, double x_max,
                          int self_loop, int64_t* offsets, int64_t* total_host, void* stream);
int gnnb_hyperbolic_fill(const double* records, int64_t n, const int64_t* seg_ptr, int64_t n_seg, double x_max,
                         int self_loop, const int64_t* offsets, int32_t* nbr, int64_t capacity, void* stream);

/* --------------------------------------------------------- random-walk structural encoding (csrc/rwpe.cu)
 * replaces: random_walk_pe(g, walk_length) (GNNGraphs/src/transform.jl:975-990): K products of the dense N x N matrix
 *           RW = A * Diagonal(deg_inv), whose diagonals are kept.  Here the walk of each segment runs in shared memory.
 * PE[k, j] = (RW^k)[j, j] for k = 1..K, RW[i, j] = A[i, j] * dinv[j], A[i, j] = summed weight of the edges i -> j.
 * Row formulation on the plan's CSR by target: u_0 = e_j, u_k[t] = dinv[t] * Σ_{edges s -> t, plan order} w_e u_{k-1}[s],
 * each product and sum rounded on its own, a row without edges 0; PE[k, j] = u_k[j].  For rows of at most the plan's
 * chunk edges that is gnnb_propagate(W_MUL_XJ | COPY_XJ, SUM, ct = dinv) bit for bit.
 * g: a square plan (GNNB_ESIZE otherwise).  w: E DEVICE floats in COO order, or NULL (every weight 1).  dinv: n DEVICE
 * floats, 1 / weighted out-degree (gnnb_degree(GNNB_DIR_OUT, w)) with +-Inf replaced by 0 — the caller computes it.
 * seg_ptr: NULL (one segment) or n_seg + 1 non-decreasing DEVICE offsets from 0 to n, validated on the device
 * (GNNB_EINVAL).  The walks of a segment never leave it: an edge into a segment this entry walks whose source lies
 * outside that segment gives GNNB_EINVAL, and nothing is read or written outside a segment.  Edges into the segments
 * it leaves untouched (below) are not looked at.
 * out: n x walk_length DEVICE floats, node-major (row j holds PE[1..K, j]).  Rows of segments with more than
 * GNNB_RWPE_SMEM_MAX_NODES nodes are left untouched: the caller composes those walks from gnnb_propagate.
 * walk_length >= 1 (GNNB_EINVAL).  Synchronises the stream. */
#define GNNB_RWPE_SMEM_MAX_NODES 896
int gnnb_random_walk_pe(gnnb_graph_t g, const float* w, const float* dinv, const int64_t* seg_ptr, int64_t n_seg,
                        int walk_length, float* out, void* stream);

/* --------------------------------------------------------- personalized-PageRank diffusion (csrc/ppr.cu)
 * replaces: ppr_diffusion(g; alpha) (GNNGraphs/src/transform.jl:1026-1051): the dense N x N matrix of the whole batch,
 *           M = I + (alpha - 1) A with A[t, s] the summed weight of the edges s -> t, and `inv` of it; the new weight of
 *           edge s -> t is alpha * inv(M)[t, s].  Here each segment (graph of a batch) is inverted on its own.
 * gnnb_ppr_diffusion: per segment [base, base + n) of at most GNNB_PPR_SMEM_MAX_NODES nodes, row i of A sums its
 *   in-edges' weights in plan order (each add rounded), am1 = alpha - 1 (rounded once), M[i][j] = am1 * A[i][j] for
 *   j != i and M[i][i] = 1 + am1 * A[i][i]; Gauss-Jordan elimination with partial pivoting (the first largest |a[i][k]|,
 *   i >= k, a NaN never chosen over a number) in shared memory, every product, difference and quotient rounded on its
 *   own; w_out[e] = alpha * inv(M)[t_e - base][s_e - base] in COO order.  The bits do not depend on the launch class.
 *   g: a square plan (GNNB_ESIZE otherwise).  w: E DEVICE floats in COO order, or NULL (every weight 1).  seg_ptr: NULL
 *   (one segment) or n_seg + 1 non-decreasing DEVICE offsets from 0 to n, validated on the device (GNNB_EINVAL; w_out
 *   is then untouched and info unspecified).  An edge into a segment this entry inverts whose source lies outside that
 *   segment gives GNNB_EINVAL, and nothing is read or written outside a segment.
 *   info: n_seg (1 without seg_ptr) DEVICE int32s: 0 = inverted, k >= 1 = zero pivot at step k (M is singular; the
 *   segment's w_out is untouched), -1 = the segment has more than GNNB_PPR_SMEM_MAX_NODES nodes and was skipped (its
 *   w_out is untouched: the caller inverts it with gnnb_ppr_matrix and a dense solver).  Synchronises the stream.
 * gnnb_ppr_matrix: M of the nodes [a, b) (the same construction) into M_out, row-major with leading dimension
 *   ld >= b - a (the caller's padding is not touched).  0 <= a <= b <= n (GNNB_EINVAL).  An edge into [a, b) whose
 *   source lies outside it gives GNNB_EINVAL.  Synchronises the stream.
 * GNNB_PPR_SMEM_MAX_NODES is the largest n whose matrix (odd leading dimension >= n + 1), pivot list and reduction
 * slots fit the 227 KB of one H100 CTA; gnnb_ppr_diffusion checks the device's opt-in limit (GNNB_EUNSUPPORTED). */
#define GNNB_PPR_SMEM_MAX_NODES 240
int gnnb_ppr_diffusion(gnnb_graph_t g, const float* w, float alpha, const int64_t* seg_ptr, int64_t n_seg,
                       float* w_out, int32_t* info, void* stream);
int gnnb_ppr_matrix(gnnb_graph_t g, const float* w, float alpha, int64_t a, int64_t b, int64_t ld, float* M_out,
                    void* stream);

/* --------------------------------------------------------- largest Laplacian eigenvalue (csrc/lmax.cu)
 * replaces: laplacian_lambda_max(g; add_self_loops, dir) (GNNGraphs/src/query.jl:598-610): for every getgraph(g, i) a
 *           dense normalized_laplacian and KrylovKit's eigsolve(Symmetric(L), x0, 1, :LR) on the host.  Symmetric reads
 *           the upper triangle, so the value is the largest eigenvalue of S, S[i][j] = S[j][i] = L[i][j] for i < j.
 * gnnb_laplacian_lambda_max: per segment [base, base + n) of at most GNNB_LMAX_SMEM_MAX_NODES nodes, with
 *   c[i] = 1 / sqrt(deg[base + i]) in double, row i of S in shared memory (double): for dir = GNNB_DIR_OUT the weights
 *   of the out-edges i -> t, t >= i, and of the in-edges s -> i, s < i, added at the other end's column in plan order;
 *   for GNNB_DIR_IN and GNNB_DIR_BOTH (the reference's A' for every dir but :out) the out-edges with t <= i and the
 *   in-edges with s > i; a self loop is read once.  S[i][j] = -(c[i] a[i][j]) c[j], S[i][i] = 1 - (c[i] (a[i][i] +
 *   [add_self_loops])) c[i].  Householder tridiagonalisation and Sturm-count multisection to the last bit; lmax_out[s]
 *   = the upper end of the final bracket (NaN if the tridiagonal matrix is not finite, or the segment has no nodes).
 *   The bits do not depend on the launch class nor on the segment's position.
 *   g: a square plan (GNNB_ESIZE otherwise).  w: E DEVICE floats in COO order, or NULL (every weight 1).  deg: n DEVICE
 *   floats, the caller's row sums of A (dir = out) or A' (gnnb_degree with GNNB_DIR_OUT or GNNB_DIR_IN), plus 1 under
 *   add_self_loops; the caller rejects zeros (the reference's isolated-node assertion).  seg_ptr: NULL (one segment)
 *   or n_seg + 1 non-decreasing DEVICE offsets from 0 to n, validated on the device (GNNB_EINVAL).  An edge with one
 *   end in a segment this entry computes and the other outside it gives GNNB_EINVAL naming the edge.
 *   lmax_out: n_seg DEVICE doubles.  info: n_seg DEVICE int32s: 0 = computed, -1 = the segment has more than
 *   GNNB_LMAX_SMEM_MAX_NODES nodes and was skipped (its lmax_out is untouched: the caller runs the Lanczos route).
 *   Synchronises the stream.
 * GNNB_LMAX_SMEM_MAX_NODES is the largest n whose n x n doubles and two working vectors fit the 227 KB of one H100
 * CTA; the entry checks the device's opt-in limit (GNNB_EUNSUPPORTED).
 * gnnb_segment_dots: out[s][k] = sum over the nodes i of segment s of X[k][i] * y[i] (k < K; X row-major with leading
 *   dimension ldx >= n, y n doubles; all DEVICE).  The sum runs over chunks of GNNB_SEGDOT_CHUNK nodes counted from
 *   the segment's start, each added in a fixed order, and the chunk sums in order: deterministic, and the same bits
 *   wherever the segment lies.  chunk_ptr: n_seg + 1 DEVICE int64 running counts of ceil(len_s / GNNB_SEGDOT_CHUNK),
 *   n_chunks its last entry; partial: n_chunks * K DEVICE doubles of scratch; seg_ptr as above (not validated: the
 *   chunk ranges are clamped to [0, n)).  Does not synchronise. */
#define GNNB_LMAX_SMEM_MAX_NODES 169
#define GNNB_SEGDOT_CHUNK 2048
int gnnb_laplacian_lambda_max(gnnb_graph_t g, const float* w, const float* deg, int dir, int add_self_loops,
                              const int64_t* seg_ptr, int64_t n_seg, double* lmax_out, int32_t* info, void* stream);
int gnnb_segment_dots(const double* X, int64_t K, int64_t ldx, const double* y, int64_t n, const int64_t* seg_ptr,
                      const int64_t* chunk_ptr, int64_t n_seg, int64_t n_chunks, double* partial, double* out,
                      void* stream);

/* --------------------------------------------------------- 1-WL colour refinement (csrc/wl.cu)
 * replaces: color_refinement(g, x0) (GNNGraphs/src/utils.jl:340-389): a host loop hashing (x_i, sort(x[in-neighbours]))
 *           into a Dict once per node per round.
 * Round r maps node i to its signature (c_i, multiset{c_s : edges s -> i}) (in-neighbours with multiplicity, a self loop
 * counts, weights ignored); two nodes get the same new colour iff their signatures are equal.  Colours are numbered
 * 1..k in order of first appearance by node id, afresh every round.  The rounds stop when a round leaves the number of
 * classes unchanged (refinement only splits classes, so that round reproduces the previous colours) or after max_iters
 * rounds.  Signatures are grouped by the exact key (c_i, S_1, S_2), S_k = Σ_edges splitmix64(c_s ^ salt_k) mod 2^61 - 1:
 * two different multisets of the same c_i share it with probability about 2^-122 under a random-function model (chance
 * collisions only, not inputs built to collide).
 * g: a square plan (GNNB_ESIZE otherwise).  x0: n DEVICE int64s (any values; only their partition matters), or NULL
 * for one starting class.  max_iters: 0 = until stable, >= 1 caps the rounds, < 0 is GNNB_EINVAL.
 * colors: n DEVICE int64s, 1-based.  num_colors, niters: HOST outputs (niters counts the last round; n == 0 gives
 * num_colors = 0, niters = 1).  Scratch: one allocation of about 92 B per node per call, plus the plan's workspace for
 * rows of more than the plan's chunk of edges.  Synchronises the stream. */
int gnnb_color_refinement(gnnb_graph_t g, const int64_t* x0, int64_t max_iters, int64_t* colors, int64_t* num_colors,
                          int64_t* niters, void* stream);

/* --------------------------------------------------------- Set2Set attention (csrc/set2set.cu)
 * replaces the per-node part of set2set_pool (GNNlib/src/layers/pool.jl:37-39): broadcast_nodes(g, q), sum(qn .* x),
 *           softmax_nodes and reduce_nodes(+, g, x .* α), about six passes over D x N floats, in one pass over x:
 *   s_k = <q[:, t_k], x[:, s_k]>;  M_i = max_k s_k;  S_i = Σ_k exp(s_k − M_i)
 *   r[:, i] = Σ_k exp(s_k − M_i) x[:, s_k] / S_i          (k over the in-edges of target i, in plan order)
 * x (D, num_src), q (D, num_dst), r (D, num_dst): DEVICE floats, column i contiguous.  seg_max, seg_sum (num_dst) are
 * kept for the pullback.  A target with no edges: r = 0 (reduce_nodes' neutral element), seg_max = −Inf, seg_sum = 0.
 * On the graph-indicator plan (edge k = node k -> its graph) the targets are the graphs of a batch.
 * 1 <= D (GNNB_ESIZE) <= GNNB_SET2SET_MAX_D (GNNB_EUNSUPPORTED: compose the three readout calls).  A NULL array of
 * positive size: GNNB_ESIZE.  Rows of more than the plan's chunk of edges are reduced in pieces and combined in a fixed
 * order: the results are run-to-run bit-identical.  Does not synchronise. */
#define GNNB_SET2SET_MAX_D 1024
int gnnb_set2set_attend(gnnb_graph_t g, const float* x, const float* q, int64_t D,
                        float* r, float* seg_max, float* seg_sum, void* stream);
/* pullback given dr (D, num_dst): α_k recomputed from seg_max / seg_sum (s_k with the forward's instructions, so α is
 * the forward's bit for bit), T_i = <dr_i, r_i>,
 *   ds_k = α_k (<dr[:, t_k], x[:, s_k]> − T_i)
 *   dxe[:, k] = α_k dr[:, t_k] + ds_k q[:, t_k]      per edge, in COO order: every column written exactly once
 *   dq[:, i]  = Σ_k ds_k x[:, s_k]                  (0 for a target with no edges)
 * On the graph-indicator plan dxe is dx.  Same bounds and errors as the forward. */
int gnnb_set2set_attend_bwd(gnnb_graph_t g, const float* x, const float* q, const float* r,
                            const float* seg_max, const float* seg_sum, const float* dr, int64_t D,
                            float* dxe, float* dq, void* stream);

/* --------------------------------------------------------- attention pooling (csrc/set2set.cu)
 * replaces the composition of global_attention_pool (GNNlib/src/layers/pool.jl:7-12) for a gate of one row:
 *           softmax_nodes(g, gate), the D x N product α .* f and reduce_nodes(+, g, ·), in one pass over f.  The Set2Set
 *           attention with a given score per source instead of <q, x>:
 *   M_i = max_k gate[s_k];  S_i = Σ_k exp(gate[s_k] − M_i)
 *   u[:, i] = Σ_k exp(gate[s_k] − M_i) f[:, s_k] / S_i    (k over the in-edges of target i, in plan order)
 * f (D, num_src), u (D, num_dst): DEVICE floats, column i contiguous; gate (num_src): DEVICE floats.  seg_max, seg_sum
 * (num_dst) are kept for the pullback.  A target with no edges: u = 0, seg_max = −Inf, seg_sum = 0.  On the
 * graph-indicator plan (edge k = node k -> its graph) the targets are the graphs of a batch.
 * Bounds, errors and determinism as gnnb_set2set_attend: 1 <= D (GNNB_ESIZE) <= GNNB_SET2SET_MAX_D
 * (GNNB_EUNSUPPORTED), a NULL array of positive size is GNNB_ESIZE, no atomics, results run-to-run bit-identical.
 * Does not synchronise. */
int gnnb_attention_pool(gnnb_graph_t g, const float* f, const float* gate, int64_t D,
                        float* u, float* seg_max, float* seg_sum, void* stream);
/* pullback given du (D, num_dst): α_k = exp(gate[s_k] − M_i) / S_i from seg_max / seg_sum (the forward's bits),
 * T_i = <du_i, u_i>,
 *   dgate_e[k] = α_k (<du[:, t_k], f[:, s_k]> − T_i)
 *   dfe[:, k]  = α_k du[:, t_k]                     per edge, in COO order: every entry written exactly once
 * On the graph-indicator plan dfe is df and dgate_e is dgate.  Same bounds and errors as the forward. */
int gnnb_attention_pool_bwd(gnnb_graph_t g, const float* f, const float* gate, const float* u,
                            const float* seg_max, const float* seg_sum, const float* du, int64_t D,
                            float* dfe, float* dgate_e, void* stream);

/* --------------------------------------------------------- top-k pooling (csrc/topk.cu)
 * replaces: topk_index(y, k) = collect(1:length(y))[y .>= nlargest(k, y)[end]] and the score and gate of
 *           topk_pool(t, X) = view(X, :, idx) .* σ.(view(y, idx)'), y = t.p' * X / norm(t.p)
 *           (GNNlib/src/layers/pool.jl:14-27), per graph of a batch.
 * All arrays are DEVICE arrays.  No entry synchronises, and every result is run-to-run bit-identical (no float atomics).
 * Inputs that only the device can check are reported through dev_status (a DEVICE int32, may be NULL): the entry sets it
 * to GNNB_OK or to the status of what it found, in stream order; the host-checked errors are returned as usual.
 *
 * gnnb_topk_keep: keep[i] (uint8) = 1 iff keys[i] >= v_s, v_s the k_s-th largest non-NaN key of i's segment, else 0.
 *   k_s = min(k, n_s) for k >= 1 (ratio must be 0), or ceil(ratio * n_s) in double for k = 0 and 0 < ratio <= 1; any
 *   other (k, ratio) is GNNB_EINVAL.  n_s counts the segment's keys, NaNs included.  A NaN key is never kept and does
 *   not count toward k_s: with fewer than k_s non-NaN keys every non-NaN key is kept, with none nothing is.  -0.0 and
 *   +0.0 are equal (ties).  Every key equal to v_s is kept, so a segment can keep more than k_s.
 *   key_type: GNNB_KEY_F32 | F64 | I32 | I64 (GNNB_EINVAL otherwise).  n in [0, 2^31) (GNNB_ESIZE).
 *   seg_ptr: NULL (one segment) or n_seg + 1 non-decreasing offsets from 0 to n, n_seg in [1, 2^31) (GNNB_ESIZE),
 *   validated on the device: a malformed seg_ptr sets dev_status to GNNB_EINVAL and keep to 0 everywhere.
 *   Segments of up to GNNB_TOPK_SMEM_MAX keys are selected by one CTA each in shared memory, larger ones by multi-block
 *   histogram passes; the masks are the same.  Scratch: the library's grow-only workspace of the device.
 * gnnb_topk_score: y[j] = <p, x_j> / sqrt(Σ_d p_d²) for the n node rows x_j (x (D, n) column-major, row j at x + j*D).
 * gnnb_topk_gate: out_j = x_{idx_j} σ(y[idx_j]) for j < m (out (D, m) column-major), idx 0-based int64;
 *   σ(a) = 1 / (1 + t) for a >= 0, t / (1 + t) otherwise, t = exp(-|a|) (NNlib's sigmoid).  An idx_j outside [0, n)
 *   sets dev_status to GNNB_EINDEX and out_j to NaN.
 * gnnb_topk_gate_bwd: the pullback of y -> gate(x, y) with y = score(x, p), given dout (D, m); s_j = σ(y[idx_j]),
 *   dy_j = s_j (1 - s_j) <dout_j, x_{idx_j}>:
 *     dx_{idx_j} = s_j dout_j + dy_j p / ‖p‖, every other row of dx exactly 0;
 *     dp = (Σ_j dy_j x_{idx_j}) / ‖p‖ - (Σ_j dy_j y[idx_j]) p / ‖p‖²   (per-block partials, then the blocks in order).
 *   idx must be strictly ascending in [0, n): m > n is GNNB_EINDEX, any other violation sets dev_status to GNNB_EINDEX
 *   and leaves that row's dx and dp terms out.  Scratch: GNNB_TOPK_DP_SLOTS(m) * (D + 1) floats of the workspace.
 * Row loads are float4 when D % 4 == 0 and the arrays are 16 B aligned, scalar otherwise.  n, m >= 0 and D >= 1
 * (GNNB_ESIZE), a NULL array of positive size: GNNB_ESIZE. */
typedef enum { GNNB_KEY_F32 = 0, GNNB_KEY_F64 = 1, GNNB_KEY_I32 = 2, GNNB_KEY_I64 = 3 } gnnb_key_type;
#define GNNB_TOPK_SMEM_MAX 8192
#define GNNB_TOPK_DP_SLOTS(m) ((m) < 65536 ? ((m) + 63) / 64 : 1024)
int gnnb_topk_keep(const void* keys, int key_type, int64_t n, const int64_t* seg_ptr, int64_t n_seg, int64_t k,
                   double ratio, uint8_t* keep, int32_t* dev_status, void* stream);
int gnnb_topk_score(const float* x, int64_t n, int64_t D, const float* p, float* y, void* stream);
int gnnb_topk_gate(const float* x, int64_t n, int64_t D, const float* y, const int64_t* idx, int64_t m, float* out,
                   int32_t* dev_status, void* stream);
int gnnb_topk_gate_bwd(const float* x, int64_t n, int64_t D, const float* y, const float* p, const int64_t* idx,
                       int64_t m, const float* dout, float* dx, float* dp, int32_t* dev_status, void* stream);
/* tuning knob for tests and timing: segments of more than `bound` keys take the multi-block class of gnnb_topk_keep
 * (0 <= bound <= GNNB_TOPK_SMEM_MAX, GNNB_EINVAL otherwise; default GNNB_TOPK_SMEM_MAX). */
int gnnb_topk_set_smem_max(int64_t bound);

/* --------------------------------------------------------- recurrent gates (csrc/recurrent.cu)
 * The gate arithmetic of the recurrent temporal cells (GraphNeuralNetworks/src/layers/temporalconv.jl), one pass over
 * node rows per entry instead of about ten broadcasts with their own (out, N) temporaries.  Arrays are DEVICE floats in
 * node rows (row n of an (N, W) array at n * W), except the x-side pre-activations:
 *   px: step t's slice of PX, the x-side operator of every gate for all steps at once.  Row n at px + n * ld_px, gate g's
 *       D floats at column g * D;  ld_px >= G * D (G = 3 for the GRU cells, 4 for the LSTM), so that a (N, T, G·D)
 *       array is read in place at px = PX + t * G·D, ld_px = T·G·D.
 * σ(a) = 1 / (1 + expf(−a)) and tanhf: the accurate forms (the reference's sigmoid_fast / tanh_fast approximate).  The
 * rows are vectorised by float4 when D % 4 == 0 and every row start is 16 B aligned, scalar otherwise; each output float
 * is written once and no atomics are used, so results are run-to-run bit-identical.
 * Errors: N < 0, D < 1, ld_px < G * D, or a NULL array of positive size: GNNB_ESIZE.  N == 0 is a no-op (except that
 * gnnb_lstm_cell_bwd writes dw = 0).  None of the entries synchronises. */
/* GRU, first half (gate order in px: [r | z | n]); ah (N, 2D) = [ah_r | ah_z], the h-side operators of r and z:
 *   r = σ(px_r + ah_r);  z = σ(px_z + ah_z);  rh = r ⊙ h
 * replaces temporalconv.jl:244-249 (GConvGRUCell), :566-569 (DCGRUCell, z = dconv_u), :842-846 (TGCNCell, the r .* h
 * input of dense_h).  r and z are kept for the pullback; rh is the input of the candidate's h-side operator. */
int gnnb_gru_rz(const float* px, int64_t ld_px, const float* ah, const float* h, int64_t N, int64_t D, float* r,
                float* z, float* rh, void* stream);
/* GRU, second half; ah_n (N, D) the candidate's h-side operator (of rh):
 *   n = tanh(px_n + ah_n)
 *   blend 0: h' = (1 − z) ⊙ n + z ⊙ h      GConvGRUCell (temporalconv.jl:250-252), DCGRUCell (:570-573)
 *   blend 1: h' = (1 − z) ⊙ h + z ⊙ n      TGCNCell (:846-847)
 * n is kept for the pullback.  blend other than 0 / 1: GNNB_EINVAL. */
int gnnb_gru_out(const float* px, int64_t ld_px, const float* ah_n, const float* h, const float* z, int64_t N,
                 int64_t D, int blend, float* n, float* h_new, void* stream);
/* pullback of gnnb_gru_out given dh' (N, D):
 *   dn = dh' ⊙ (1 − z) [blend 0] | dh' ⊙ z [blend 1];  dpre_n = dn ⊙ (1 − n²)
 *   dz = dh' ⊙ (h − n) [blend 0] | dh' ⊙ (n − h) [blend 1];  dh = dh' ⊙ z [blend 0] | dh' ⊙ (1 − z) [blend 1]
 * dpre_n: row n at dpre_n + n * ld_dpre (>= D: it may be the n block of an (N, 3D) array); dz, dh (N, D). */
int gnnb_gru_out_bwd(const float* dh_new, const float* h, const float* z, const float* n, int64_t N, int64_t D,
                     int blend, float* dpre_n, int64_t ld_dpre, float* dz, float* dh, void* stream);
/* pullback of gnnb_gru_rz given drh (the candidate operator's pullback) and dz:
 *   dpre_r = drh ⊙ h ⊙ r (1 − r);  dpre_z = dz ⊙ z (1 − z);  dh += drh ⊙ r
 * dpre_rz: row n at dpre_rz + n * ld_dpre (>= 2D), [dpre_r | dpre_z].  dh (N, D) is read and written. */
int gnnb_gru_rz_bwd(const float* drh, const float* dz, const float* h, const float* r, const float* z, int64_t N,
                    int64_t D, float* dpre_rz, int64_t ld_dpre, float* dh, void* stream);
/* LSTM with peepholes (GConvLSTMCell, temporalconv.jl:425-435), gate order [i | f | c | o]; ah (N, 4D), c (N, D):
 *   i = σ(px_i + ah_i + w_i ⊙ c);  f = σ(px_f + ah_f + w_f ⊙ c);  g = tanh(px_c + ah_c + w_c ⊙ c)
 *   c' = f ⊙ c + i ⊙ g;  o = σ(px_o + ah_o + w_o ⊙ c')   (the new c, :431-433);  h' = o ⊙ tanh(c')
 * w: 4·D floats [w_i | w_f | w_c | w_o], or NULL for no peepholes (Flux's LSTMCell).  gates (N, 4D) = [i | f | g | o]
 * is kept for the pullback. */
int gnnb_lstm_cell(const float* px, int64_t ld_px, const float* ah, const float* c, const float* w, int64_t N,
                   int64_t D, float* gates, float* c_new, float* h_new, void* stream);
/* pullback given dh', dc' (N, D) and the forward's c, gates, c':
 *   dpre_o = dh' ⊙ tanh(c') ⊙ o (1 − o);  dc'' = dc' + dh' ⊙ o ⊙ (1 − tanh²(c')) + dpre_o ⊙ w_o
 *   dpre_i = dc'' ⊙ g ⊙ i (1 − i);  dpre_f = dc'' ⊙ c ⊙ f (1 − f);  dpre_c = dc'' ⊙ i ⊙ (1 − g²)
 *   dc = dc'' ⊙ f + dpre_i ⊙ w_i + dpre_f ⊙ w_f + dpre_c ⊙ w_c
 *   dw = Σ_n [dpre_i ⊙ c | dpre_f ⊙ c | dpre_c ⊙ c | dpre_o ⊙ c']       (when w and dw are given)
 * dpre (N, 4D) serves the x side and the h side alike.  dw is a deterministic two-stage column sum (per-block partials,
 * then dense.cu's fixed-order final pass): ws holds GNNB_LSTM_DW_SLOTS(N) * 4 * D floats (NULL when dw is NULL). */
#define GNNB_LSTM_DW_SLOTS(N) ((N) < 65536 ? ((N) + 63) / 64 : 1024)
int gnnb_lstm_cell_bwd(const float* dh_new, const float* dc_new, const float* c, const float* gates,
                       const float* c_new, const float* w, int64_t N, int64_t D, float* dpre, float* dc, float* dw,
                       float* ws, void* stream);

/* ------------------------------------------------- edge codes and random edges (csrc/edgegen.cu)
 * Code spaces of edge_encoding / edge_decoding (GNNGraphs/src/utils.jl:189-268, bipartite :263-268), 0-based here (the
 * reference's idx - 1), node ids 0-based (s, t < n; bipartite s < n1, t < n2), n1, n2 in [0, 2^31):
 *   DIRECTED             M = n^2         c = s n + t
 *   DIRECTED_NOLOOP      M = n(n-1)      c = s (n-1) + t - (t > s)                       (s != t)
 *   UNDIRECTED           M = n(n+1)/2    c = start(s) + t - s,      start(s) = s(2n+1-s)/2  (s <= t after swapping)
 *   UNDIRECTED_NOLOOP    M = n(n-1)/2    c = start(s) + t - s - 1,  start(s) = s(2n-1-s)/2  (s < t after swapping)
 *   BIPARTITE            M = n1 n2       c = s n2 + t
 * Decoding is integer-exact: the undirected row comes from a float64 sqrt of the exact uint64 discriminant and is then
 * corrected with integer arithmetic.  n2 is read only for BIPARTITE. */
typedef enum {
    GNNB_CODES_DIRECTED = 0,
    GNNB_CODES_DIRECTED_NOLOOP = 1,
    GNNB_CODES_UNDIRECTED = 2,
    GNNB_CODES_UNDIRECTED_NOLOOP = 3,
    GNNB_CODES_BIPARTITE = 4
} gnnb_code_space;

/* Rounds of the Feistel network behind gnnb_sample_codes (part of its output contract: changing it changes every
 * sample). */
#define GNNB_FEISTEL_ROUNDS 8

/* replaces: edge_encoding(s, t, n; directed, self_loops) (utils.jl:189-227).  s, t: E DEVICE int64 ids with base
 * index_base (0|1); codes: E DEVICE uint64.  An id out of range, or a self loop in a NOLOOP space: GNNB_EINDEX (the
 * reference's `@assert all(s .!= t)`).  Synchronises the stream. */
int gnnb_edge_encode(int space, int64_t n1, int64_t n2, const int64_t* s, const int64_t* t, int64_t num_edges,
                     int index_base, uint64_t* codes, void* stream);
/* replaces: edge_decoding(idx, n; directed, self_loops) and edge_decoding(idx, n1, n2) (utils.jl:229-268).  Writes
 * int64 ids with base index_base; a code >= M: GNNB_EINDEX.  Undirected codes decode to s <= t (s < t).  Synchronises. */
int gnnb_edge_decode(int space, int64_t n1, int64_t n2, const uint64_t* codes, int64_t num_edges, int index_base,
                     int64_t* s, int64_t* t, void* stream);
/* The sorted set of distinct codes of an edge list: encode, device radix sort, one code per run of equal codes.
 * replaces: the host-side `edge_encoding` + `setdiff!` bookkeeping of negative_sample (GNNGraphs/src/transform.jl:
 * 899-917) and `intersect(idx1, idx2)` of intersect(g1, g2) (GNNGraphs/src/operators.jl:13-15).  Pairs the space does
 * not hold (self loops in a NOLOOP space) are skipped; ids out of range: GNNB_EINDEX.  codes_out: DEVICE uint64 with
 * num_edges entries; *n_out (HOST) = distinct codes written, ascending.  num_edges < 2^31.  Synchronises. */
int gnnb_edge_codes_sorted(int space, int64_t n1, int64_t n2, const int64_t* s, const int64_t* t, int64_t num_edges,
                           int index_base, uint64_t* codes_out, int64_t* n_out, void* stream);
/* flags[k] = 1 if codes[k] is in `set` (x ascending distinct DEVICE uint64), else 0: one binary search per code.
 * replaces: the membership half of `intersect(idx1, idx2)` (operators.jl:15).  num_codes < 2^31.  Does not
 * synchronise. */
int gnnb_codes_member(const uint64_t* codes, int64_t num_codes, const uint64_t* set, int64_t x, uint8_t* flags,
                      void* stream);
/* The first m codes of the seeded permutation π of [0, M) that are not in `excl`, in π order.
 * replaces: the sampling of negative_sample (transform.jl:904-922: randsubseq over all codes, setdiff! against the
 *           positives, truncation to the first num_neg of an ascending list) and of rand_graph (generate.jl:51-65 via
 *           _rand_edges, utils.jl:270-284: StatsBase.sample without replacement), and randperm in rand_edge_split
 *           (transform.jl:948).
 * π(i): a balanced Feistel network of GNNB_FEISTEL_ROUNDS rounds over [0, 4^h), 4^h the smallest power of four >= M
 * (h >= 1), cycle-walked until the value is < M.  Round r maps (L, R) -> (R, L ^ (splitmix64(R ^ k_r) & (2^h - 1))),
 * k_r = splitmix64(splitmix64(seed) + r), value = L 2^h + R.  excl: x ascending distinct DEVICE codes < M (GNNB_EINVAL
 * otherwise).  out: DEVICE uint64, m entries; writes min(m, M - x) codes and sets *n_out (HOST) to that number.
 * The output is distinct by construction and a pure function of (M, excl, m, seed).  M < 2^62.  Synchronises. */
int gnnb_sample_codes(uint64_t M, const uint64_t* excl, int64_t x, int64_t m, uint64_t seed, uint64_t* out,
                      int64_t* n_out, void* stream);

/* ------------------------------------------------------ host-buffer entries
 * The reference-facing call with HOST arrays (what a CPU-array caller of `propagate` has): copies
 * x (and w) to the device, runs the fused pass, copies `out` back; synchronous.  Used for the
 * end-to-end number (bench.py `e2e`).  Same semantics as gnnb_propagate / gnnb_gcn_propagate. */
int gnnb_propagate_host(gnnb_graph_t g, int transposed, int msg, int aggr, const float* x_host,
                        const float* w_host, int64_t D, float* out_host);
int gnnb_gcn_propagate_host(gnnb_graph_t g, int transposed, const float* x_host,
                            const float* w_host, int64_t D, float* out_host);

/* One GCNConv forward (+ backward when dy_host != NULL) on HOST arrays — the call a CPU-array user of the layer makes
 * (bench.py `e2e`): replaces  y = l.σ.(l.weight * (c .* propagate(copy_xj, g', +, xj = x .* c')) .+ l.bias)  and Zygote's
 * pullback (GNNlib/src/layers/conv.jl:14-72 on the `Dout >= Din` branch, default norm_fn, no edge weights).
 * `g` already carries the self loops if the layer adds them.  x_host (Din,N), W_host (Dout,Din) row-major, b_host NULL or
 * Dout, relu 0|1, dy_host (Dout,N) or NULL; outputs y_host (Dout,N), dx_host (Din,N), dW_host (Dout,Din), db_host (Dout or
 * NULL).  Uploads, kernels and downloads run on three streams (x and dy up while y comes down); the device staging lives
 * with the plan.  Pinned host memory makes the copies asynchronous; pageable memory works (staged by the driver).
 * GNNB_EUNSUPPORTED for Dout < Din (use the device entries). */
int gnnb_gcn_conv_step_host(gnnb_graph_t g, const float* x_host, const float* W_host, const float* b_host, int relu,
                            int64_t Din, int64_t Dout, const float* dy_host, float* y_host, float* dx_host,
                            float* dW_host, float* db_host);

/* ------------------------------------------------------------- generators
 * RMAT edge list (ours; the reference has none, SURVEY.md §8d): Graph500 a,b,c,d = .57,.19,.19,.05,
 * counter-based splitmix64 keyed on (seed, edge id, retry); edges with an endpoint >= N are redrawn;
 * duplicates and self loops kept; generation order.  Writes int64 1-based src/dst DEVICE arrays.
 * The oracle has the bit-identical CPU generator (oracle/gnn_oracle.c: orc_rmat). */
int gnnb_rmat_edges(int64_t num_nodes, int64_t num_edges, uint64_t seed, int64_t* src_dev,
                    int64_t* dst_dev, void* stream);
/* edges [first_edge, first_edge + count) of the same list (the generator is counter-based): a 1 B-edge graph is produced
 * and consumed chunk by chunk (gnnb_shard_builder_add) without ever being resident. */
int gnnb_rmat_edges_range(int64_t num_nodes, int64_t first_edge, int64_t count, uint64_t seed, int64_t* src_dev,
                          int64_t* dst_dev, void* stream);

/* tuning knob for experiments: edges per work chunk of the segmented-reduce kernels (default 128;
 * power of two in [32, 4096]); affects plans created afterwards. */
int gnnb_set_chunk_edges(int chunk);
/* kernels of the fused segmented reduce and of the fused GAT passes (results are bit-identical):
 * 0 = default: the lean work-item kernels (csrc/seglean.cu, csrc/gat.cu) for rows of 128/256/512 floats, the round-1
 * chunk kernels for every other shape;  12 = the round-1 chunk kernels (seg_reduce_kernel, gat_fwd_kernel,
 * gat_bwd_kernel) for every shape: the reference the lean kernels are tested against;  14 = the default kernels with the
 * fused GCN propagate's L2 eviction priorities at every size (by default only when the gathered rows are at least 8 times
 * the L2), so that tests reach them on small graphs.  Any other value: GNNB_EINVAL. */
int gnnb_set_kernel_variant(int v);

#ifdef __cplusplus
}
#endif
#endif /* GNNB200_H */
