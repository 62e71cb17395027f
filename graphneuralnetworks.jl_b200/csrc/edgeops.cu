// edgeops.cu — the unfused primitives of the reference API (gather, scatter, degree, edge softmax)
// and the per-edge pullback pieces (edge dot products, max/min pullback).  These exist so that an
// ARBITRARY message function keeps working through apply_edges / aggregate_neighbors
// (GNNlib/src/msgpass.jl:121-129,145-149); the fused kernels of segreduce.cu / gat.cu are the fast path.
#include "common.cuh"
#include <math_constants.h>

namespace gnnb {

// out[k,:] = x[idx[k],:]  (NNlib.gather, GNNGraphs/src/gatherscatter.jl:4)
template <int VEC>
__global__ void gather_rows_kernel(const int32_t* __restrict__ idx, int64_t E, const float* __restrict__ x,
                                   int64_t D, float* __restrict__ out) {
    const int64_t nvec = D / VEC;
    const int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= E * nvec) return;
    const int64_t e = i / nvec, f = (i % nvec) * VEC;
    const int64_t n = idx[e];
    if (VEC == 4)
        *reinterpret_cast<float4*>(out + e * D + f) = __ldg(reinterpret_cast<const float4*>(x + n * D + f));
    else
        out[e * D + f] = __ldg(x + n * D + f);
}

// num = exp(e - M[t]) and out = num / S[t] steps of softmax_edge_neighbors (GNNlib/src/utils.jl:93-96)
__global__ void sm_exp_kernel(const int32_t* __restrict__ t, int64_t E, int64_t K, const float* __restrict__ e,
                              const float* __restrict__ M, float* __restrict__ out) {
    int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= E * K) return;
    int64_t k = i / K, h = i % K;
    out[i] = expf(e[i] - __ldg(M + (int64_t)t[k] * K + h));
}
__global__ void sm_div_kernel(const int32_t* __restrict__ t, int64_t E, int64_t K, const float* __restrict__ S,
                              float* __restrict__ out) {
    int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= E * K) return;
    int64_t k = i / K, h = i % K;
    out[i] = __fdiv_rn(out[i], __ldg(S + (int64_t)t[k] * K + h));
}
__global__ void mul_kernel(const float* __restrict__ a, const float* __restrict__ b, int64_t n, float* __restrict__ out) {
    int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i < n) out[i] = a[i] * b[i];
}
// de = alpha * (dalpha - T[t])
__global__ void sm_bwd_kernel(const int32_t* __restrict__ t, int64_t E, int64_t K, const float* __restrict__ alpha,
                              const float* __restrict__ dalpha, const float* __restrict__ T, float* __restrict__ de) {
    int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= E * K) return;
    int64_t k = i / K, h = i % K;
    de[i] = alpha[i] * (dalpha[i] - __ldg(T + (int64_t)t[k] * K + h));
}

__global__ void deg_from_rowptr_kernel(const int32_t* __restrict__ rowptr, int32_t n, float* __restrict__ out, int accumulate) {
    int64_t r = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (r >= n) return;
    float d = (float)(rowptr[r + 1] - rowptr[r]);
    out[r] = accumulate ? out[r] + d : d;
}
__global__ void add_kernel(float* __restrict__ a, const float* __restrict__ b, int64_t n) {
    int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i < n) a[i] += b[i];
}

// c = 1 / sqrt(d)  — the default norm_fn of GCNConv (GraphNeuralNetworks/src/layers/conv.jl:99), IEEE-exact ops
__global__ void rsqrt_exact_kernel(float* __restrict__ d, int64_t n) {
    int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i < n) d[i] = __fdiv_rn(1.0f, __fsqrt_rn(d[i]));
}
int rsqrt_exact(float* d, int64_t n, cudaStream_t st) {
    if (n <= 0) return GNNB_OK;
    rsqrt_exact_kernel<<<(unsigned)ceil_div(n, 256), 256, 0, st>>>(d, n);
    GNNB_LAUNCHED();
    return GNNB_OK;
}

// dw_plan[e] = scale * <dout[row[e],:], x[col[e],:]>   (pullback of w_mul_xj w.r.t. the edge weight)
template <int TPR>
__global__ void edge_dot_kernel(const int32_t* __restrict__ row, const int32_t* __restrict__ col,
                                const int32_t* __restrict__ eid, int64_t E, const float* __restrict__ dout,
                                const float* __restrict__ x, const float* __restrict__ cs,
                                const float* __restrict__ ct, int64_t D, float* __restrict__ dw_coo) {
    const int lig = threadIdx.x % TPR;
    const int64_t e = ((int64_t)blockIdx.x * blockDim.x + threadIdx.x) / TPR;
    float acc = 0.f;
    int r = 0, c = 0;
    if (e < E) {
        r = row[e];
        c = col[e];
        const float* a = dout + (int64_t)r * D;
        const float* b = x + (int64_t)c * D;
        for (int64_t f = lig; f < D; f += TPR) acc += __ldg(a + f) * __ldg(b + f);
    }
#pragma unroll
    for (int o = TPR / 2; o > 0; o >>= 1) acc += __shfl_xor_sync(0xffffffffu, acc, o, TPR);
    if (e < E && lig == 0) {
        if (cs) acc *= cs[c];
        if (ct) acc *= ct[r];
        dw_coo[eid[e]] = acc;
    }
}

// pullback of MAX/MIN aggregation w.r.t. x (every tied extremum receives the gradient: NNlib rule)
//   dx[j,:] = sum_{e in out-edges of j} w_e * dout[t_e,:] .* ( x[j,:]*w_e == out_fwd[t_e,:] )
// HALO 1 (the forward CSR of a backward shard plan): targets >= split read dout2 / of2 + (t - split)*D
template <int HALO>
__global__ void maxmin_bwd_kernel(const int32_t* __restrict__ rowptr, const int32_t* __restrict__ col,
                                  const float* __restrict__ w_plan, int32_t nrows, const float* __restrict__ x,
                                  const float* __restrict__ dout, const float* __restrict__ out_fwd,
                                  int64_t D, float* __restrict__ dx, const float* __restrict__ dout2,
                                  const float* __restrict__ of2, int32_t split) {
    const int lane = threadIdx.x & 31;
    const int64_t j = ((int64_t)blockIdx.x * blockDim.x + threadIdx.x) >> 5;
    if (j >= nrows) return;
    const int rs = rowptr[j], re = rowptr[j + 1];
    for (int64_t f = lane; f < D; f += 32) {
        const float xv = x[j * D + f];
        float acc = 0.f;
        for (int e = rs; e < re; ++e) {
            const int64_t t = col[e];
            const bool second = HALO != 0 && t >= split;
            const int64_t tr = second ? t - split : t;
            const float w = w_plan ? w_plan[e] : 1.f;
            const float m = __fmul_rn(xv, w);
            if (m == __ldg((second ? of2 : out_fwd) + tr * D + f)) acc += w * __ldg((second ? dout2 : dout) + tr * D + f);
        }
        dx[j * D + f] = acc;
    }
}

}  // namespace gnnb

using namespace gnnb;

static inline unsigned nblk(int64_t n) { return (unsigned)ceil_div(n, 256); }

extern "C" {

int gnnb_gather(gnnb_graph_t g, int which, const float* x, int64_t D, float* out, void* stream) {
    if (!g) GNNB_FAIL(GNNB_EINVAL, "graph handle is NULL");
    if (D <= 0) GNNB_FAIL(GNNB_ESIZE, "D must be positive");
    if (which != GNNB_SRC && which != GNNB_DST) GNNB_FAIL(GNNB_EINVAL, "which must be GNNB_SRC or GNNB_DST");
    cudaStream_t st = (cudaStream_t)stream;
    if (g->E == 0) return GNNB_OK;
    const int32_t* idx = which == GNNB_SRC ? g->coo_src : g->coo_dst;
    const bool v4 = D % 4 == 0 && !((uintptr_t)x & 15) && !((uintptr_t)out & 15);
    if (v4) gather_rows_kernel<4><<<nblk(g->E * (D / 4)), 256, 0, st>>>(idx, g->E, x, D, out);
    else gather_rows_kernel<1><<<nblk(g->E * D), 256, 0, st>>>(idx, g->E, x, D, out);
    GNNB_LAUNCHED();
    return GNNB_OK;
}

int gnnb_gather_rows(const int32_t* idx_dev, int64_t n, const float* x, int64_t D, float* out, void* stream) {
    if (n < 0 || D <= 0) GNNB_FAIL(GNNB_ESIZE, "gather_rows: bad sizes");
    if (n == 0) return GNNB_OK;
    if (!idx_dev || !x || !out) GNNB_FAIL(GNNB_EINVAL, "gather_rows: NULL argument");
    cudaStream_t st = (cudaStream_t)stream;
    const bool v4 = D % 4 == 0 && !((uintptr_t)x & 15) && !((uintptr_t)out & 15);
    if (v4) gather_rows_kernel<4><<<nblk(n * (D / 4)), 256, 0, st>>>(idx_dev, n, x, D, out);
    else gather_rows_kernel<1><<<nblk(n * D), 256, 0, st>>>(idx_dev, n, x, D, out);
    GNNB_LAUNCHED();
    return GNNB_OK;
}

int gnnb_scatter(gnnb_graph_t g, int which, int aggr, const float* m, int64_t D, float* out, void* stream) {
    if (!g) GNNB_FAIL(GNNB_EINVAL, "graph handle is NULL");
    if (aggr < GNNB_SUM || aggr > GNNB_MIN) GNNB_FAIL(GNNB_EINVAL, "unknown aggregation %d", aggr);
    if (which != GNNB_SRC && which != GNNB_DST) GNNB_FAIL(GNNB_EINVAL, "which must be GNNB_SRC or GNNB_DST");
    cudaStream_t st = (cudaStream_t)stream;
    GNNB_TRY(ensure_csr(g, which == GNNB_SRC, st));
    Csr view = which == GNNB_SRC ? g->by_src : g->by_dst;
    view.col = view.eid;  // "gather" the edge's own message row: m[:, eid]
    SegArgs a;
    a.x = m; a.out = out; a.D = D; a.aggr = aggr;
    return seg_reduce(g, view, a, st);
}

int gnnb_degree(gnnb_graph_t g, int dir, const float* w, float* out, void* stream) {
    if (!g) GNNB_FAIL(GNNB_EINVAL, "graph handle is NULL");
    if (dir < GNNB_DIR_OUT || dir > GNNB_DIR_BOTH) GNNB_FAIL(GNNB_EINVAL, "dir must be out/in/both");
    if (dir == GNNB_DIR_BOTH && g->n_src != g->n_dst) GNNB_FAIL(GNNB_ESIZE, "dir=both needs num_src == num_dst");
    cudaStream_t st = (cudaStream_t)stream;
    const bool want_in = dir != GNNB_DIR_OUT, want_out = dir != GNNB_DIR_IN;
    if (want_out) GNNB_TRY(ensure_csr(g, true, st));
    if (!w) {
        // order as the reference: out first, then in (GNNGraphs/src/query.jl:362-367)
        if (want_out && g->n_src > 0) {
            deg_from_rowptr_kernel<<<nblk(g->n_src), 256, 0, st>>>(g->by_src.rowptr, g->n_src, out, 0);
            GNNB_LAUNCHED();
        }
        if (want_in && g->n_dst > 0) {
            deg_from_rowptr_kernel<<<nblk(g->n_dst), 256, 0, st>>>(g->by_dst.rowptr, g->n_dst, out, want_out ? 1 : 0);
            GNNB_LAUNCHED();
        }
        return GNNB_OK;
    }
    if (dir == GNNB_DIR_BOTH) {
        GNNB_TRY(grow_buffer(&g->ws2, &g->ws2_bytes, sizeof(float) * (size_t)g->n_dst));
        GNNB_TRY(gnnb_scatter(g, GNNB_SRC, GNNB_SUM, w, 1, out, stream));
        GNNB_TRY(gnnb_scatter(g, GNNB_DST, GNNB_SUM, w, 1, g->ws2, stream));
        if (g->n_dst > 0) { add_kernel<<<nblk(g->n_dst), 256, 0, st>>>(out, g->ws2, g->n_dst); GNNB_LAUNCHED(); }
        return GNNB_OK;
    }
    return gnnb_scatter(g, want_out ? GNNB_SRC : GNNB_DST, GNNB_SUM, w, 1, out, stream);
}

int gnnb_gcn_norm(gnnb_graph_t g, const float* w, float* c_out, void* stream) {
    if (!g) GNNB_FAIL(GNNB_EINVAL, "NULL argument");
    if (g->n_dst == 0) return GNNB_OK;   // no targets (an empty rank's shard): nothing to write, c_out may be NULL
    if (!c_out) GNNB_FAIL(GNNB_EINVAL, "NULL argument");
    cudaStream_t st = (cudaStream_t)stream;
    GNNB_TRY(gnnb_degree(g, GNNB_DIR_IN, w, c_out, stream));
    if (g->n_dst > 0) { rsqrt_exact_kernel<<<nblk(g->n_dst), 256, 0, st>>>(c_out, g->n_dst); GNNB_LAUNCHED(); }
    return GNNB_OK;
}

int gnnb_softmax_edge_neighbors(gnnb_graph_t g, const float* e, int64_t K, float* out, void* stream) {
    if (!g) GNNB_FAIL(GNNB_EINVAL, "graph handle is NULL");
    if (K <= 0) GNNB_FAIL(GNNB_ESIZE, "K must be positive");
    cudaStream_t st = (cudaStream_t)stream;
    if (g->E == 0) return GNNB_OK;
    const int64_t n = g->E * K;
    GNNB_TRY(grow_buffer(&g->ws2, &g->ws2_bytes, sizeof(float) * (size_t)g->n_dst * K));
    float* stat = g->ws2;
    GNNB_TRY(gnnb_scatter(g, GNNB_DST, GNNB_MAX, e, K, stat, stream));            // max_ = scatter(max, e, t)
    sm_exp_kernel<<<nblk(n), 256, 0, st>>>(g->coo_dst, g->E, K, e, stat, out);     // num = exp.(e .- gather(max_, t))
    GNNB_LAUNCHED();
    GNNB_TRY(gnnb_scatter(g, GNNB_DST, GNNB_SUM, out, K, stat, stream));          // den = scatter(+, num, t)
    sm_div_kernel<<<nblk(n), 256, 0, st>>>(g->coo_dst, g->E, K, stat, out);        // num ./ gather(den, t)
    GNNB_LAUNCHED();
    return GNNB_OK;
}

int gnnb_softmax_edge_neighbors_bwd(gnnb_graph_t g, const float* alpha, const float* dalpha, int64_t K,
                                    float* de, void* stream) {
    if (!g) GNNB_FAIL(GNNB_EINVAL, "graph handle is NULL");
    if (K <= 0) GNNB_FAIL(GNNB_ESIZE, "K must be positive");
    cudaStream_t st = (cudaStream_t)stream;
    if (g->E == 0) return GNNB_OK;
    const int64_t n = g->E * K;
    GNNB_TRY(grow_buffer(&g->ws2, &g->ws2_bytes, sizeof(float) * (size_t)g->n_dst * K));
    float* T = g->ws2;
    mul_kernel<<<nblk(n), 256, 0, st>>>(alpha, dalpha, n, de);
    GNNB_LAUNCHED();
    GNNB_TRY(gnnb_scatter(g, GNNB_DST, GNNB_SUM, de, K, T, stream));
    sm_bwd_kernel<<<nblk(n), 256, 0, st>>>(g->coo_dst, g->E, K, alpha, dalpha, T, de);
    GNNB_LAUNCHED();
    return GNNB_OK;
}

}  // extern "C"

namespace gnnb {

int edge_dot(gnnb_graph* g, const float* dout, const float* x, const float* cs, const float* ct, int64_t D,
             float* dw_coo, cudaStream_t st) {
    if (g->E == 0) return GNNB_OK;
    const Csr& c = g->by_dst;
    if (D >= 32) edge_dot_kernel<32><<<nblk(g->E * 32), 256, 0, st>>>(c.row, c.col, c.eid, g->E, dout, x, cs, ct, D, dw_coo);
    else if (D >= 8) edge_dot_kernel<8><<<nblk(g->E * 8), 256, 0, st>>>(c.row, c.col, c.eid, g->E, dout, x, cs, ct, D, dw_coo);
    else edge_dot_kernel<2><<<nblk(g->E * 2), 256, 0, st>>>(c.row, c.col, c.eid, g->E, dout, x, cs, ct, D, dw_coo);
    GNNB_LAUNCHED();
    return GNNB_OK;
}

int maxmin_bwd_lean(gnnb_graph* g, const Csr& c, const float* w_plan, const float* x, const float* dout,
                    const float* out_fwd, bool halo, const float* dout2, const float* of2, int32_t split, int64_t D,
                    float* dx, cudaStream_t st);   // seglean.cu
// the max / min pullback over `c`, whose rows are the sources j and whose gathered nodes the targets t (weights in c's
// plan order): the by-source plan of a graph (halo = false), or the forward CSR of a backward shard plan whose targets
// >= split read dout2 / of2 (halo = true)
static int maxmin_bwd_rows(gnnb_graph* g, const Csr& c, const float* w_plan, const float* x, const float* dout,
                           const float* out_fwd, bool halo, const float* dout2, const float* of2, int32_t split,
                           int64_t D, float* dx, cudaStream_t st) {
    if (c.nrows == 0) return GNNB_OK;
    {   // rows of 128 / 256 / 512 floats: the work-item kernel (seglean.cu); other widths: one warp per source row
        const int rc = maxmin_bwd_lean(g, c, w_plan, x, dout, out_fwd, halo, dout2, of2, split, D, dx, st);
        if (rc != GNNB_EUNSUPPORTED) return rc;
    }
    if (halo)
        maxmin_bwd_kernel<1><<<nblk((int64_t)c.nrows * 32), 256, 0, st>>>(c.rowptr, c.col, w_plan, c.nrows, x, dout,
                                                                          out_fwd, D, dx, dout2, of2, split);
    else
        maxmin_bwd_kernel<0><<<nblk((int64_t)c.nrows * 32), 256, 0, st>>>(c.rowptr, c.col, w_plan, c.nrows, x, dout,
                                                                          out_fwd, D, dx, nullptr, nullptr, 0);
    GNNB_LAUNCHED();
    return GNNB_OK;
}
int maxmin_bwd(gnnb_graph* g, const float* w_plan_src, const float* x, const float* dout, const float* out_fwd,
               int64_t D, float* dx, cudaStream_t st) {
    return maxmin_bwd_rows(g, g->by_src, w_plan_src, x, dout, out_fwd, false, nullptr, nullptr, 0, D, dx, st);
}
int maxmin_bwd_halo(gnnb_graph* g, const float* w_plan_dst, const float* x_own, const float* dout_local,
                    const float* dout_halo, const float* out_local, const float* out_halo, int32_t n_local, int64_t D,
                    float* dx, cudaStream_t st) {
    return maxmin_bwd_rows(g, g->by_dst, w_plan_dst, x_own, dout_local, out_local, true, dout_halo, out_halo, n_local, D,
                           dx, st);
}

}  // namespace gnnb
