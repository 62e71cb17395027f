// set2set.cu — the per-node part of Set2Set pooling (set2set_pool, GNNlib/src/layers/pool.jl:29-43).
//
// Each of the reference's iterations broadcasts the query to every node (qn, D x N), forms sum(qn .* x, dims = 1), a
// graph-wise softmax, x .* α and a segmented sum: about six passes over D x N floats and three D x N temporaries.  It is
// one attention with a single query per target, so on the CSR by target (the graph-indicator plan: target = graph, its
// in-edges = its nodes) it is one pass with an online softmax in registers:
//   forward:  s_k = <q_i, x_{s_k}>;  M_i = max_k s_k;  S_i = Σ_k exp(s_k − M_i);  r_i = Σ_k exp(s_k − M_i) x_{s_k} / S_i
//   backward: α_k = exp(s_k − M_i) / S_i, s_k recomputed with the forward's instructions;  T_i = <dr_i, r_i>
//             ds_k = α_k (<dr_i, x_{s_k}> − T_i);  dxe_k = α_k dr_i + ds_k q_i;  dq_i = Σ_k ds_k x_{s_k}
// One warp per work item of the plan (seglean.cu); lane l owns the slices (i·32 + l) of the D-float row, float4 or
// scalar, and each gathered x row serves the dot products and the weighted sum from the same registers.  Pieces of long
// rows go to partial slots: [acc: D][M][S] in the layout of gat.cu's forward fix-up with one head, and plain D-float
// sums in the layout of segreduce.cu's fix-up for dq.  Both fix-ups combine the slots in chunk order, so every output is
// run-to-run bit-identical.  No atomics.
//
// Attention pooling (global_attention_pool, GNNlib/src/layers/pool.jl:7-12) is the same attention with a given score per
// source, s_k = gate[s_k], instead of <q_i, x_{s_k}>: the kernels take the score as a policy (GATE), so the forward
// shares the loop, the online softmax, the lanes and gat.cu's fix-up.  Its pullback has no per-target sum (dgate_e and
// dfe are per edge), so the pieces of a long row need no slots there:
//   backward: α_k = exp(gate[s_k] − M_i) / S_i;  T_i = <du_i, u_i>;  dgate_e_k = α_k (<du_i, f_{s_k}> − T_i);  dfe_k = α_k du_i
#include "common.cuh"
#include <math_constants.h>

namespace gnnb {

int gat_fwd_fixup_one_head(const Csr& c, int64_t E, int chunk, int64_t D, bool vec4, float* ws, float* out,
                           float* seg_max, float* seg_sum, cudaStream_t st);                              // gat.cu
int seg_fixup_sum(const Csr& c, int64_t E, int chunk, int64_t D, float* ws, float* out, cudaStream_t st);  // segreduce.cu

namespace {

struct S2SParams {
    const int4* __restrict__ items;   // the plan's work items {e_begin, e_end, slot, 0} (seglean.cu)
    const int32_t* __restrict__ col;  // source of each edge, plan order
    const int32_t* __restrict__ row;  // target of each edge
    const int32_t* __restrict__ eid;  // COO position of each edge
    const float* __restrict__ x;      // [num_src][D]
    const float* __restrict__ q;      // [num_dst][D]; attention pooling: the gate [num_src]
    const float* __restrict__ r;      // bwd: the forward's r      [num_dst][D]
    const float* __restrict__ smax;   // bwd: the forward's seg_max, seg_sum
    const float* __restrict__ ssum;
    const float* __restrict__ dr;     // bwd                        [num_dst][D]
    float* __restrict__ out;          // fwd: r; bwd: dq            [num_dst][D]; attention pooling bwd: dgate_e [E]
    float* __restrict__ out_max;      // fwd: seg_max, seg_sum      [num_dst]
    float* __restrict__ out_sum;
    float* __restrict__ dxe;          // bwd                        [E][D]
    float* __restrict__ ws;           // partial slots of the long rows
    int64_t D;
    int64_t slot;                     // floats per partial slot
    int32_t n_items;
};

constexpr unsigned FULL = 0xffffffffu;

template <int VEC> struct SV;
template <> struct SV<4> { using T = float4; };
template <> struct SV<1> { using T = float; };

template <typename V> __device__ __forceinline__ V s2s_zero();
template <> __device__ __forceinline__ float4 s2s_zero<float4>() { return make_float4(0.f, 0.f, 0.f, 0.f); }
template <> __device__ __forceinline__ float s2s_zero<float>() { return 0.f; }
__device__ __forceinline__ void s2s_ld(const float* p, float4& v) { v = __ldg(reinterpret_cast<const float4*>(p)); }
__device__ __forceinline__ void s2s_ld(const float* p, float& v) { v = __ldg(p); }
__device__ __forceinline__ void s2s_st(float* p, float4 v) { *reinterpret_cast<float4*>(p) = v; }
__device__ __forceinline__ void s2s_st(float* p, float v) { *p = v; }
// d + <a, b> as a fixed chain of fmas: the forward and the backward evaluate s_k with the same instructions
__device__ __forceinline__ float s2s_dot(float4 a, float4 b, float d) {
    d = fmaf(a.x, b.x, d); d = fmaf(a.y, b.y, d); d = fmaf(a.z, b.z, d);
    return fmaf(a.w, b.w, d);
}
__device__ __forceinline__ float s2s_dot(float a, float b, float d) { return fmaf(a, b, d); }
// a*s + b*t
__device__ __forceinline__ float4 s2s_lin(float4 a, float s, float4 b, float t) {
    return make_float4(fmaf(a.x, s, b.x * t), fmaf(a.y, s, b.y * t), fmaf(a.z, s, b.z * t), fmaf(a.w, s, b.w * t));
}
__device__ __forceinline__ float s2s_lin(float a, float s, float b, float t) { return fmaf(a, s, b * t); }
// acc + a*s
__device__ __forceinline__ float4 s2s_axpy(float4 acc, float4 a, float s) {
    return make_float4(fmaf(a.x, s, acc.x), fmaf(a.y, s, acc.y), fmaf(a.z, s, acc.z), fmaf(a.w, s, acc.w));
}
__device__ __forceinline__ float s2s_axpy(float acc, float a, float s) { return fmaf(a, s, acc); }
__device__ __forceinline__ float4 s2s_scale(float4 a, float s) { return make_float4(a.x * s, a.y * s, a.z * s, a.w * s); }
__device__ __forceinline__ float s2s_scale(float a, float s) { return a * s; }
__device__ __forceinline__ float4 s2s_div(float4 a, float s) {
    return make_float4(__fdiv_rn(a.x, s), __fdiv_rn(a.y, s), __fdiv_rn(a.z, s), __fdiv_rn(a.w, s));
}
__device__ __forceinline__ float s2s_div(float a, float s) { return __fdiv_rn(a, s); }
// butterfly: a + b == b + a, so every lane ends with the same bits
__device__ __forceinline__ float warp_sum(float v) {
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(FULL, v, o);
    return v;
}

// gathered rows a warp keeps in flight: 16 floats per lane
template <int F> struct InFlight { static constexpr int U = F <= 4 ? 4 : (F <= 8 ? 2 : 1); };

// index words of the edge e0 + lane
__device__ __forceinline__ void load_edge(const S2SParams& p, int my, int e_end, int& c, int& r, int& id, bool& last) {
    c = 0; r = 0; id = 0; last = false;
    if (my < e_end) {
        c = __ldg(p.col + my);
        r = __ldg(p.row + my);
        id = __ldg(p.eid + my);
        last = (my + 1 == e_end) || (__ldg(p.row + my + 1) != r);
    }
}

// ------------------------------------------------------------------------------------------------ forward
// GATE = false: s_k = <q_i, x_{s_k}> (Set2Set).  GATE = true: s_k = gate[s_k], a given score per source in p.q
// (attention pooling); q is not read.
template <bool GATE, int VEC, int K>
__device__ __forceinline__ void attend_fwd(const S2SParams& p) {
    using V = typename SV<VEC>::T;
    constexpr int U = InFlight<VEC * K>::U;
    const int lane = threadIdx.x & 31;
    const int item = blockIdx.x * 8 + (threadIdx.x >> 5);
    if (item >= p.n_items) return;
    const int4 it = __ldg(p.items + item);
    const int e_end = it.y;
    const bool partial = it.z >= 0;                    // the same item on every lane: warp-uniform
    int64_t f[K]; bool act[K];
#pragma unroll
    for (int i = 0; i < K; ++i) { f[i] = (int64_t)(i * 32 + lane) * VEC; act[i] = f[i] < p.D; }
    V qv[K], acc[K];
#pragma unroll
    for (int i = 0; i < K; ++i) { qv[i] = s2s_zero<V>(); acc[i] = s2s_zero<V>(); }
    float M = -CUDART_INF_F, S = 0.f;
    bool fresh = true;                                 // the next edge starts a row

    for (int e = it.x; e < e_end; e += 32) {
        int c_l, r_l, id_l; bool last_l;
        load_edge(p, e + lane, e_end, c_l, r_l, id_l, last_l);
        float g_l = 0.f;
        if constexpr (GATE) { if (e + lane < e_end) g_l = __ldg(p.q + c_l); }
        const int nb = min(32, e_end - e);
        const unsigned bmask = partial ? 0u : __ballot_sync(FULL, last_l);
#pragma unroll 1
        for (int j0 = 0; j0 < nb; j0 += U) {
            V v[U][K];
#pragma unroll
            for (int u = 0; u < U; ++u) {
                const int cj = __shfl_sync(FULL, c_l, (j0 + u) & 31);
                const bool ok = j0 + u < nb;
#pragma unroll
                for (int i = 0; i < K; ++i) {
                    v[u][i] = s2s_zero<V>();
                    if (ok && act[i]) s2s_ld(p.x + (int64_t)cj * p.D + f[i], v[u][i]);
                }
            }
#pragma unroll
            for (int u = 0; u < U; ++u) {
                const int j = j0 + u;
                if (j < nb) {                          // warp-uniform
                    if (fresh) {
                        const int rj = __shfl_sync(FULL, r_l, j);
#pragma unroll
                        for (int i = 0; i < K; ++i) {
                            if constexpr (!GATE) {
                                qv[i] = s2s_zero<V>();
                                if (act[i]) s2s_ld(p.q + (int64_t)rj * p.D + f[i], qv[i]);
                            }
                            acc[i] = s2s_zero<V>();
                        }
                        M = -CUDART_INF_F; S = 0.f;
                        fresh = false;
                    }
                    float s = 0.f;
                    if constexpr (GATE) {
                        s = __shfl_sync(FULL, g_l, j);
                    } else {
#pragma unroll
                        for (int i = 0; i < K; ++i) s = s2s_dot(qv[i], v[u][i], s);
                        s = warp_sum(s);
                    }
                    const float Mn = fmaxf(M, s);
                    const float Ms = softmax_shift(Mn);
                    const float sc = expf(M - Ms);     // exp(-inf) = 0 on the first edge of a row
                    const float pp = expf(s - Ms);
                    S = fmaf(S, sc, pp);
#pragma unroll
                    for (int i = 0; i < K; ++i) acc[i] = s2s_lin(acc[i], sc, v[u][i], pp);
                    M = Mn;
                    if ((bmask >> j) & 1u) {           // row end: normalise and store, exactly once
                        const int rj = __shfl_sync(FULL, r_l, j);
#pragma unroll
                        for (int i = 0; i < K; ++i)
                            if (act[i]) s2s_st(p.out + (int64_t)rj * p.D + f[i], s2s_div(acc[i], S));
                        if (lane == 0) { p.out_max[rj] = M; p.out_sum[rj] = S; }
                        fresh = true;
                    }
                }
            }
        }
    }
    if (partial) {
        float* base = p.ws + (int64_t)it.z * p.slot;
#pragma unroll
        for (int i = 0; i < K; ++i)
            if (act[i]) s2s_st(base + f[i], acc[i]);
        if (lane == 0) { base[p.D] = M; base[p.D + 1] = S; }
    }
}

// ------------------------------------------------------------------------------------------------ backward
// GATE = true: the score is the given gate (p.q), so there is no dq; out receives dgate_e[k] = ds_k per edge (COO
// order), dxe the per-edge α_k dr_i, and a long row's pieces are independent: no partial slots.
template <bool GATE, int VEC, int K>
__device__ __forceinline__ void attend_bwd(const S2SParams& p) {
    using V = typename SV<VEC>::T;
    constexpr int U = InFlight<VEC * K>::U;
    const int lane = threadIdx.x & 31;
    const int item = blockIdx.x * 8 + (threadIdx.x >> 5);
    if (item >= p.n_items) return;
    const int4 it = __ldg(p.items + item);
    const int e_end = it.y;
    const bool partial = it.z >= 0;
    int64_t f[K]; bool act[K];
#pragma unroll
    for (int i = 0; i < K; ++i) { f[i] = (int64_t)(i * 32 + lane) * VEC; act[i] = f[i] < p.D; }
    V qv[K], dv[K], acc[K];
#pragma unroll
    for (int i = 0; i < K; ++i) { qv[i] = s2s_zero<V>(); dv[i] = s2s_zero<V>(); acc[i] = s2s_zero<V>(); }
    float M = 0.f, S = 1.f, T = 0.f;
    bool fresh = true;

    for (int e = it.x; e < e_end; e += 32) {
        int c_l, r_l, id_l; bool last_l;
        load_edge(p, e + lane, e_end, c_l, r_l, id_l, last_l);
        float g_l = 0.f;
        if constexpr (GATE) { if (e + lane < e_end) g_l = __ldg(p.q + c_l); }
        const int nb = min(32, e_end - e);
        const unsigned bmask = partial ? 0u : __ballot_sync(FULL, last_l);
#pragma unroll 1
        for (int j0 = 0; j0 < nb; j0 += U) {
            V v[U][K];
#pragma unroll
            for (int u = 0; u < U; ++u) {
                const int cj = __shfl_sync(FULL, c_l, (j0 + u) & 31);
                const bool ok = j0 + u < nb;
#pragma unroll
                for (int i = 0; i < K; ++i) {
                    v[u][i] = s2s_zero<V>();
                    if (ok && act[i]) s2s_ld(p.x + (int64_t)cj * p.D + f[i], v[u][i]);
                }
            }
#pragma unroll
            for (int u = 0; u < U; ++u) {
                const int j = j0 + u;
                if (j < nb) {                          // warp-uniform
                    if (fresh) {                       // the row's q, dr, statistics and T = <dr, r>
                        const int rj = __shfl_sync(FULL, r_l, j);
                        float t = 0.f;
#pragma unroll
                        for (int i = 0; i < K; ++i) {
                            V rv = s2s_zero<V>();
                            if constexpr (!GATE) qv[i] = s2s_zero<V>();
                            dv[i] = s2s_zero<V>();
                            if (act[i]) {
                                const int64_t o = (int64_t)rj * p.D + f[i];
                                if constexpr (!GATE) s2s_ld(p.q + o, qv[i]);
                                s2s_ld(p.dr + o, dv[i]); s2s_ld(p.r + o, rv);
                            }
                            t = s2s_dot(dv[i], rv, t);
                            if constexpr (!GATE) acc[i] = s2s_zero<V>();
                        }
                        T = warp_sum(t);
                        M = __ldg(p.smax + rj); S = __ldg(p.ssum + rj);
                        fresh = false;
                    }
                    float s = 0.f, gd = 0.f;
                    if constexpr (GATE) {
                        s = __shfl_sync(FULL, g_l, j);
#pragma unroll
                        for (int i = 0; i < K; ++i) gd = s2s_dot(dv[i], v[u][i], gd);
                    } else {
#pragma unroll
                        for (int i = 0; i < K; ++i) {
                            s = s2s_dot(qv[i], v[u][i], s); gd = s2s_dot(dv[i], v[u][i], gd);
                        }
                        s = warp_sum(s);
                    }
                    gd = warp_sum(gd);
                    const float al = __fdiv_rn(expf(s - M), S);
                    const float ds = al * (gd - T);
                    const int ek = __shfl_sync(FULL, id_l, j);
                    if constexpr (GATE) {
#pragma unroll
                        for (int i = 0; i < K; ++i)
                            if (act[i]) s2s_st(p.dxe + (int64_t)ek * p.D + f[i], s2s_scale(dv[i], al));
                        if (lane == 0) p.out[ek] = ds;
                    } else {
#pragma unroll
                        for (int i = 0; i < K; ++i) {
                            if (act[i]) s2s_st(p.dxe + (int64_t)ek * p.D + f[i], s2s_lin(dv[i], al, qv[i], ds));
                            acc[i] = s2s_axpy(acc[i], v[u][i], ds);
                        }
                    }
                    if ((bmask >> j) & 1u) {           // row end: dq, exactly once
                        if constexpr (!GATE) {
                            const int rj = __shfl_sync(FULL, r_l, j);
#pragma unroll
                            for (int i = 0; i < K; ++i)
                                if (act[i]) s2s_st(p.out + (int64_t)rj * p.D + f[i], acc[i]);
                        }
                        fresh = true;
                    }
                }
            }
        }
    }
    if (!GATE && partial) {
        float* base = p.ws + (int64_t)it.z * p.D;
#pragma unroll
        for (int i = 0; i < K; ++i)
            if (act[i]) s2s_st(base + f[i], acc[i]);
    }
}

template <int VEC, int K>
__global__ void __launch_bounds__(256) set2set_fwd_kernel(const S2SParams p) { attend_fwd<false, VEC, K>(p); }
template <int VEC, int K>
__global__ void __launch_bounds__(256) set2set_bwd_kernel(const S2SParams p) { attend_bwd<false, VEC, K>(p); }
template <int VEC, int K>
__global__ void __launch_bounds__(256) attention_pool_fwd_kernel(const S2SParams p) { attend_fwd<true, VEC, K>(p); }
// min blocks 1: without it ptxas trades a few spills (K = 2 and 32) for occupancy the gather-bound loop does not need
template <int VEC, int K>
__global__ void __launch_bounds__(256, 1) attention_pool_bwd_kernel(const S2SParams p) { attend_bwd<true, VEC, K>(p); }

// targets without edges (every target when rowptr is NULL): out = 0 and, when smax is given, seg_max = -Inf and
// seg_sum = 0.  One warp per target.
__global__ void __launch_bounds__(256) set2set_fill_empty_kernel(const int32_t* __restrict__ rowptr, int32_t nrows,
                                                                 float* __restrict__ out, int64_t D,
                                                                 float* __restrict__ smax, float* __restrict__ ssum) {
    const int lane = threadIdx.x & 31;
    const int64_t rr = ((int64_t)blockIdx.x * blockDim.x + threadIdx.x) >> 5;
    if (rr >= nrows) return;
    if (rowptr && __ldg(rowptr + rr) != __ldg(rowptr + rr + 1)) return;
    for (int64_t d = lane; d < D; d += 32) out[rr * D + d] = 0.f;
    if (lane == 0 && smax) { smax[rr] = -CUDART_INF_F; ssum[rr] = 0.f; }
}

int fill_empty(const int32_t* rowptr, int32_t nrows, float* out, int64_t D, float* smax, float* ssum, cudaStream_t st) {
    set2set_fill_empty_kernel<<<(unsigned)ceil_div(nrows, 8), 256, 0, st>>>(rowptr, nrows, out, D, smax, ssum);
    GNNB_LAUNCHED();
    return GNNB_OK;
}

template <bool GATE, int VEC, int K>
int launch2(bool bwd, const S2SParams& p, cudaStream_t st) {
    const unsigned blocks = (unsigned)ceil_div(p.n_items, 8);
    if constexpr (GATE) {
        if (bwd) attention_pool_bwd_kernel<VEC, K><<<blocks, 256, 0, st>>>(p);
        else attention_pool_fwd_kernel<VEC, K><<<blocks, 256, 0, st>>>(p);
    } else {
        if (bwd) set2set_bwd_kernel<VEC, K><<<blocks, 256, 0, st>>>(p);
        else set2set_fwd_kernel<VEC, K><<<blocks, 256, 0, st>>>(p);
    }
    GNNB_LAUNCHED();
    return GNNB_OK;
}
// K = slices per lane, the power of two that covers D (D <= GNNB_SET2SET_MAX_D = 32 floats per lane)
template <bool GATE>
int launch(bool bwd, bool vec4, const S2SParams& p, cudaStream_t st) {
    if (p.n_items == 0) return GNNB_OK;
    const int64_t k = ceil_div(p.D, vec4 ? 128 : 32);
    if (vec4) {
        if (k <= 1) return launch2<GATE, 4, 1>(bwd, p, st);
        if (k <= 2) return launch2<GATE, 4, 2>(bwd, p, st);
        if (k <= 4) return launch2<GATE, 4, 4>(bwd, p, st);
        return launch2<GATE, 4, 8>(bwd, p, st);
    }
    if (k <= 1) return launch2<GATE, 1, 1>(bwd, p, st);
    if (k <= 2) return launch2<GATE, 1, 2>(bwd, p, st);
    if (k <= 4) return launch2<GATE, 1, 4>(bwd, p, st);
    if (k <= 8) return launch2<GATE, 1, 8>(bwd, p, st);
    if (k <= 16) return launch2<GATE, 1, 16>(bwd, p, st);
    return launch2<GATE, 1, 32>(bwd, p, st);
}

bool aligned16(const void* a) { return (reinterpret_cast<uintptr_t>(a) & 15) == 0; }

}  // namespace
}  // namespace gnnb

using namespace gnnb;

extern "C" {

int gnnb_set2set_attend(gnnb_graph_t g, const float* x, const float* q, int64_t D, float* r, float* seg_max,
                        float* seg_sum, void* stream) {
    if (!g) GNNB_FAIL(GNNB_EINVAL, "graph handle is NULL");
    if (D < 1) GNNB_FAIL(GNNB_ESIZE, "set2set_attend: D must be >= 1 (got %lld)", (long long)D);
    if (D > GNNB_SET2SET_MAX_D)
        GNNB_FAIL(GNNB_EUNSUPPORTED, "set2set_attend: D = %lld is above GNNB_SET2SET_MAX_D = %d; compose "
                  "broadcast_nodes / softmax_nodes / reduce_nodes", (long long)D, GNNB_SET2SET_MAX_D);
    const int32_t nd = g->n_dst;
    if ((nd > 0 && (!q || !r || !seg_max || !seg_sum)) || (g->E > 0 && !x))
        GNNB_FAIL(GNNB_ESIZE, "set2set_attend: NULL array of positive size");
    if (nd == 0) return GNNB_OK;
    cudaStream_t st = (cudaStream_t)stream;
    GNNB_TRY(ensure_csr(g, false, st));
    const Csr& c = g->by_dst;
    if (g->E == 0) return fill_empty(nullptr, nd, r, D, seg_max, seg_sum, st);
    GNNB_TRY(ensure_items(g, c, st));
    if (c.n_empty > 0) GNNB_TRY(fill_empty(c.rowptr, nd, r, D, seg_max, seg_sum, st));
    const bool vec4 = D % 4 == 0 && aligned16(x) && aligned16(q) && aligned16(r);
    S2SParams p = {};
    p.items = reinterpret_cast<const int4*>(c.items); p.n_items = c.n_items;
    p.col = c.col; p.row = c.row; p.eid = c.eid;
    p.x = x; p.q = q; p.out = r; p.out_max = seg_max; p.out_sum = seg_sum;
    p.D = D; p.slot = (D + 2 + 3) & ~(int64_t)3;       // gat_fwd_fixup_kernel's slot with H = 1
    if (c.n_long > 0) {
        GNNB_TRY(grow_buffer(&g->ws, &g->ws_bytes, sizeof(float) * (size_t)2 * ceil_div(g->E, g->chunk) * p.slot));
        p.ws = g->ws;
    }
    GNNB_TRY(launch<false>(false, vec4, p, st));
    return gat_fwd_fixup_one_head(c, g->E, g->chunk, D, vec4, p.ws, r, seg_max, seg_sum, st);
}

int gnnb_set2set_attend_bwd(gnnb_graph_t g, const float* x, const float* q, const float* r, const float* seg_max,
                            const float* seg_sum, const float* dr, int64_t D, float* dxe, float* dq, void* stream) {
    if (!g) GNNB_FAIL(GNNB_EINVAL, "graph handle is NULL");
    if (D < 1) GNNB_FAIL(GNNB_ESIZE, "set2set_attend_bwd: D must be >= 1 (got %lld)", (long long)D);
    if (D > GNNB_SET2SET_MAX_D)
        GNNB_FAIL(GNNB_EUNSUPPORTED, "set2set_attend_bwd: D = %lld is above GNNB_SET2SET_MAX_D = %d", (long long)D,
                  GNNB_SET2SET_MAX_D);
    const int32_t nd = g->n_dst;
    if ((nd > 0 && !dq) || (g->E > 0 && (!x || !q || !r || !seg_max || !seg_sum || !dr || !dxe)))
        GNNB_FAIL(GNNB_ESIZE, "set2set_attend_bwd: NULL array of positive size");
    if (nd == 0) return GNNB_OK;
    cudaStream_t st = (cudaStream_t)stream;
    GNNB_TRY(ensure_csr(g, false, st));
    const Csr& c = g->by_dst;
    if (g->E == 0) return fill_empty(nullptr, nd, dq, D, nullptr, nullptr, st);
    GNNB_TRY(ensure_items(g, c, st));
    if (c.n_empty > 0) GNNB_TRY(fill_empty(c.rowptr, nd, dq, D, nullptr, nullptr, st));
    const bool vec4 = D % 4 == 0 && aligned16(x) && aligned16(q) && aligned16(r) && aligned16(dr) && aligned16(dxe) &&
                      aligned16(dq);
    S2SParams p = {};
    p.items = reinterpret_cast<const int4*>(c.items); p.n_items = c.n_items;
    p.col = c.col; p.row = c.row; p.eid = c.eid;
    p.x = x; p.q = q; p.r = r; p.smax = seg_max; p.ssum = seg_sum; p.dr = dr; p.out = dq; p.dxe = dxe;
    p.D = D; p.slot = D;                               // seg_fixup_kernel's slot
    if (c.n_long > 0) {
        GNNB_TRY(grow_buffer(&g->ws, &g->ws_bytes, sizeof(float) * (size_t)2 * ceil_div(g->E, g->chunk) * D));
        p.ws = g->ws;
    }
    GNNB_TRY(launch<false>(true, vec4, p, st));
    return seg_fixup_sum(c, g->E, g->chunk, D, p.ws, dq, st);
}

int gnnb_attention_pool(gnnb_graph_t g, const float* f, const float* gate, int64_t D, float* u, float* seg_max,
                        float* seg_sum, void* stream) {
    if (!g) GNNB_FAIL(GNNB_EINVAL, "graph handle is NULL");
    if (D < 1) GNNB_FAIL(GNNB_ESIZE, "attention_pool: D must be >= 1 (got %lld)", (long long)D);
    if (D > GNNB_SET2SET_MAX_D)
        GNNB_FAIL(GNNB_EUNSUPPORTED, "attention_pool: D = %lld is above GNNB_SET2SET_MAX_D = %d; compose "
                  "softmax_nodes / reduce_nodes", (long long)D, GNNB_SET2SET_MAX_D);
    const int32_t nd = g->n_dst;
    if ((nd > 0 && (!u || !seg_max || !seg_sum)) || (g->E > 0 && (!f || !gate)))
        GNNB_FAIL(GNNB_ESIZE, "attention_pool: NULL array of positive size");
    if (nd == 0) return GNNB_OK;
    cudaStream_t st = (cudaStream_t)stream;
    GNNB_TRY(ensure_csr(g, false, st));
    const Csr& c = g->by_dst;
    if (g->E == 0) return fill_empty(nullptr, nd, u, D, seg_max, seg_sum, st);
    GNNB_TRY(ensure_items(g, c, st));
    if (c.n_empty > 0) GNNB_TRY(fill_empty(c.rowptr, nd, u, D, seg_max, seg_sum, st));
    const bool vec4 = D % 4 == 0 && aligned16(f) && aligned16(u);
    S2SParams p = {};
    p.items = reinterpret_cast<const int4*>(c.items); p.n_items = c.n_items;
    p.col = c.col; p.row = c.row; p.eid = c.eid;
    p.x = f; p.q = gate; p.out = u; p.out_max = seg_max; p.out_sum = seg_sum;
    p.D = D; p.slot = (D + 2 + 3) & ~(int64_t)3;       // gat_fwd_fixup_kernel's slot with H = 1
    if (c.n_long > 0) {
        GNNB_TRY(grow_buffer(&g->ws, &g->ws_bytes, sizeof(float) * (size_t)2 * ceil_div(g->E, g->chunk) * p.slot));
        p.ws = g->ws;
    }
    GNNB_TRY(launch<true>(false, vec4, p, st));
    return gat_fwd_fixup_one_head(c, g->E, g->chunk, D, vec4, p.ws, u, seg_max, seg_sum, st);
}

int gnnb_attention_pool_bwd(gnnb_graph_t g, const float* f, const float* gate, const float* u, const float* seg_max,
                            const float* seg_sum, const float* du, int64_t D, float* dfe, float* dgate_e, void* stream) {
    if (!g) GNNB_FAIL(GNNB_EINVAL, "graph handle is NULL");
    if (D < 1) GNNB_FAIL(GNNB_ESIZE, "attention_pool_bwd: D must be >= 1 (got %lld)", (long long)D);
    if (D > GNNB_SET2SET_MAX_D)
        GNNB_FAIL(GNNB_EUNSUPPORTED, "attention_pool_bwd: D = %lld is above GNNB_SET2SET_MAX_D = %d", (long long)D,
                  GNNB_SET2SET_MAX_D);
    if (g->E > 0 && (!f || !gate || !u || !seg_max || !seg_sum || !du || !dfe || !dgate_e))
        GNNB_FAIL(GNNB_ESIZE, "attention_pool_bwd: NULL array of positive size");
    if (g->E == 0) return GNNB_OK;                     // every output is per edge
    cudaStream_t st = (cudaStream_t)stream;
    GNNB_TRY(ensure_csr(g, false, st));
    const Csr& c = g->by_dst;
    GNNB_TRY(ensure_items(g, c, st));
    const bool vec4 = D % 4 == 0 && aligned16(f) && aligned16(u) && aligned16(du) && aligned16(dfe);
    S2SParams p = {};
    p.items = reinterpret_cast<const int4*>(c.items); p.n_items = c.n_items;
    p.col = c.col; p.row = c.row; p.eid = c.eid;
    p.x = f; p.q = gate; p.r = u; p.smax = seg_max; p.ssum = seg_sum; p.dr = du; p.out = dgate_e; p.dxe = dfe;
    p.D = D;
    return launch<true>(true, vec4, p, st);
}

}  // extern "C"
