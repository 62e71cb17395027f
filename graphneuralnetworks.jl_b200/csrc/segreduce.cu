// segreduce.cu — the fused gather -> edge message -> segmented reduce kernel family.
//
// Replaces the reference's three-kernel sequence  NNlib.gather -> broadcast message -> NNlib.scatter
// (GNNlib/src/msgpass.jl:75-79,121-129,145-149; GNNGraphs/src/gatherscatter.jl:4,17) with ONE
// edge-parallel pass over a CSR-sorted edge list:
//
//     out[r,:] = ct[r] * AGG_{e in row r} ( w[e] * cs[col[e]] * x[col[e],:] )
//
// Work decomposition (load balance is independent of the degree distribution — RMAT hubs included):
//   * the sorted edge list is cut into fixed chunks of C edges; one *group* of TPR lanes owns a chunk,
//     every lane of the group owns VEC*K features of the row (TPR=32, VEC=4, K=1 for D=128: one warp
//     reads one whole 512 B feature row with a single coalesced LDG.128 per edge);
//   * a row that starts inside a chunk and has <= C edges is finished by that chunk (it may overrun
//     into the next chunk, which then skips those edges) and stored directly, scaled, exactly once;
//   * a row with > C edges ("long") is reduced piecewise: each chunk writes its raw partial to a
//     workspace slot (2 slots per chunk) and `seg_fixup_kernel` combines the slots in chunk order —
//     no atomics anywhere, results are run-to-run deterministic;
//   * rows without edges receive the neutral element (0, or -/+Inf for max/min: NNlib semantics) from
//     the group that processes the first edge of the next non-empty row.
// Inside a row the edges are visited in COO order (the plan's sort is stable), i.e. the same order
// as NNlib's sequential CPU scatter; products are rounded before the add (no FMA contraction) so a
// short row reproduces the reference's fp32 result bit for bit.
#include "common.cuh"
#include "segwalk.cuh"
#include "segparams.cuh"
#include <math_constants.h>
#include <math.h>

namespace gnnb {

// SegParams: segparams.cuh

// Reference mode (gnnb_set_kernel_variant(12)): by default (variant 0) rows of 128 / 256 / 512 floats take the lean
// work-item kernels (seglean.cu, and their GAT counterparts in gat.cu) and every other shape takes seg_reduce_kernel below
// and the round-1 GAT kernels.  Variant 12 sends every shape to the round-1 kernels.  It stays because it is the
// reference the tests hold the lean kernels to, bit for bit.  Round 1's LDGSTS rings, round 2's index-prefetch variants,
// the TMA-staged rings, the lean kernel gathering cs[col] instead of the per-edge scale stream and the uncapped build
// below were measured no faster than the default and removed (DESIGN.md §4, §7).
bool g_reference_kernels = false;

template <int VEC> struct VecT;
template <> struct VecT<4> { using T = float4; };
template <> struct VecT<1> { using T = float; };

__device__ __forceinline__ float4 vld(const float4* p) { return __ldg(p); }
__device__ __forceinline__ float vld(const float* p) { return __ldg(p); }
__device__ __forceinline__ void vst(float4* p, float4 v) { *p = v; }
__device__ __forceinline__ void vst(float* p, float v) { *p = v; }
__device__ __forceinline__ float4 vsplat4(float v) { return make_float4(v, v, v, v); }

template <bool ISMAX> __device__ __forceinline__ float comb1(float acc, float v, float s1, float s2) {
    // (x * cs) * w, each product rounded, then the reduction: matches  w .* (x .* c')  then  +
    float m = __fmul_rn(__fmul_rn(v, s1), s2);
    if (ISMAX) return fmax_nan(acc, m);     // a NaN message makes the row NaN, as Julia's max does
    return __fadd_rn(acc, m);
}
template <bool ISMAX> __device__ __forceinline__ float4 comb(float4 a, float4 v, float s1, float s2) {
    return make_float4(comb1<ISMAX>(a.x, v.x, s1, s2), comb1<ISMAX>(a.y, v.y, s1, s2),
                       comb1<ISMAX>(a.z, v.z, s1, s2), comb1<ISMAX>(a.w, v.w, s1, s2));
}
template <bool ISMAX> __device__ __forceinline__ float comb(float a, float v, float s1, float s2) {
    return comb1<ISMAX>(a, v, s1, s2);
}
__device__ __forceinline__ float4 vmulf(float4 a, float s) {
    return make_float4(a.x * s, a.y * s, a.z * s, a.w * s);
}
__device__ __forceinline__ float vmulf(float a, float s) { return a * s; }
__device__ __forceinline__ float4 vdivf(float4 a, float s) {
    return make_float4(__fdiv_rn(a.x, s), __fdiv_rn(a.y, s), __fdiv_rn(a.z, s), __fdiv_rn(a.w, s));
}
__device__ __forceinline__ float vdivf(float a, float s) { return __fdiv_rn(a, s); }
template <typename V> __device__ __forceinline__ V vsplat(float v);
template <> __device__ __forceinline__ float4 vsplat<float4>(float v) { return vsplat4(v); }
template <> __device__ __forceinline__ float vsplat<float>(float v) { return v; }

// final scaling of a finished row: mean divide (true division as NNlib), ct scale, sign restore
template <typename V>
__device__ __forceinline__ V finish_row(V acc, const SegParams& p, int r) {
    if (p.mean) {
        int deg = __ldg(p.rowptr + r + 1) - __ldg(p.rowptr + r);
        acc = vdivf(acc, (float)(deg > 0 ? deg : 1));
    }
    if (p.ct) acc = vmulf(acc, __ldg(p.ct + r));
    if (p.sign < 0.f) acc = vmulf(acc, -1.f);
    return acc;
}

// UU = row loads a group keeps in flight (0 = default 8/K); MINB = resident CTAs the register allocation must allow
template <int VEC, int TPR, int K, bool ISMAX, int UU = 0, int MINB = 1>
__global__ void __launch_bounds__(256, MINB) seg_reduce_kernel(const SegParams p) {
    using V = typename VecT<VEC>::T;
    constexpr int U = UU > 0 ? UU : ((VEC == 4) ? ((8 / K) < TPR ? (8 / K) : TPR) : (8 < TPR ? 8 : TPR));
    constexpr unsigned FULL = 0xffffffffu;
    const int lig = threadIdx.x % TPR;                                     // lane in group
    const int64_t k = ((int64_t)blockIdx.x * blockDim.x + threadIdx.x) / TPR;  // chunk id
    const int64_t d0 = (int64_t)blockIdx.y * (VEC * TPR * K);              // feature tile base
    const float neutral = ISMAX ? -CUDART_INF_F : 0.f;
    const float fillv = ISMAX ? (p.sign < 0.f ? CUDART_INF_F : -CUDART_INF_F) : 0.f;
    const int C = p.chunk;

    int64_t foff[K];
    bool fact[K];
#pragma unroll
    for (int i = 0; i < K; ++i) {
        foff[i] = d0 + (int64_t)(i * TPR + lig) * VEC;
        fact[i] = foff[i] < p.D;
    }

    const ChunkBounds cb = chunk_bounds(p.rowptr, p.row, k, C, p.E, p.nchunks);   // segwalk.cuh
    const int e_begin = cb.e_begin, e_end = cb.e_end, prev_row = cb.prev_row;
    const bool head_partial = cb.head_partial, tail_partial = cb.tail_partial;
    const bool has_work = e_begin < e_end;

    V acc[K];
#pragma unroll
    for (int i = 0; i < K; ++i) acc[i] = vsplat<V>(neutral);
    int r = -1;            // current row (none yet)
    bool first_flush = true;

    // store a finished (or partial) row
    auto flush = [&](int rr, bool last) {
        float* base;
        bool raw;
        if (first_flush && head_partial) {
            base = p.ws + (size_t)(2 * k + 0) * p.D;
            raw = true;
        } else if (last && tail_partial) {
            base = p.ws + (size_t)(2 * k + 1) * p.D;
            raw = true;
        } else {
            base = p.out + (size_t)rr * p.D;
            raw = false;
        }
        first_flush = false;
#pragma unroll
        for (int i = 0; i < K; ++i) {
            if (fact[i]) {
                V v = raw ? acc[i] : finish_row<V>(acc[i], p, rr);
                vst(reinterpret_cast<V*>(base + foff[i]), v);
            }
        }
    };
    // neutral element for the empty rows in (lo, hi)
    auto fill_gap = [&](int lo, int hi) {
        if (!p.fill) return;
        for (int q = lo + 1; q < hi; ++q) {
#pragma unroll
            for (int i = 0; i < K; ++i)
                if (fact[i]) vst(reinterpret_cast<V*>(p.out + (size_t)q * p.D + foff[i]), vsplat<V>(fillv));
        }
    };

    int e = e_begin;
    while (__any_sync(FULL, e < e_end)) {
        const int my_e = e + lig;
        const bool mine = my_e < e_end;
        int c_l = 0, d_l = -1;
        float s1_l = 1.f, s2_l = 1.f;
        if (mine) {
            c_l = __ldg(p.col + my_e);
            d_l = __ldg(p.row + my_e);
            if (p.cs) s1_l = __ldg(p.cs + c_l);
            if (p.w) s2_l = __ldg(p.w + my_e);
            if (p.sign < 0.f) s2_l = -s2_l;
        }
        const int nb = e_end - e;  // edges left for this group (may be <= 0 or > TPR)
#pragma unroll 1
        for (int j0 = 0; j0 < TPR; j0 += U) {
            if (!__any_sync(FULL, j0 < nb)) break;
            V v[U][K];
#pragma unroll
            for (int u = 0; u < U; ++u) {
                const int cj = __shfl_sync(FULL, c_l, j0 + u, TPR);
                const bool valid = (j0 + u) < nb;
                const float* xr = (p.x2 != nullptr && cj >= p.split) ? p.x2 + (size_t)(cj - p.split) * p.D
                                                                     : p.x + (size_t)cj * p.D;
#pragma unroll
                for (int i = 0; i < K; ++i)
                    v[u][i] = (valid && fact[i]) ? vld(reinterpret_cast<const V*>(xr + foff[i]))
                                                 : vsplat<V>(0.f);
            }
#pragma unroll
            for (int u = 0; u < U; ++u) {
                const int dj = __shfl_sync(FULL, d_l, j0 + u, TPR);
                const float s1 = __shfl_sync(FULL, s1_l, j0 + u, TPR);
                const float s2 = __shfl_sync(FULL, s2_l, j0 + u, TPR);
                if ((j0 + u) < nb) {
                    if (dj != r) {
                        if (r >= 0) {
                            flush(r, false);
                            fill_gap(r, dj);
                        } else if (!head_partial) {
                            fill_gap(prev_row, dj);
                        }
                        r = dj;
#pragma unroll
                        for (int i = 0; i < K; ++i) acc[i] = vsplat<V>(neutral);
                    }
#pragma unroll
                    for (int i = 0; i < K; ++i) acc[i] = comb<ISMAX>(acc[i], v[u][i], s1, s2);
                }
            }
        }
        e += TPR;
    }
    if (has_work) {
        flush(r, true);
        if (e_end == p.E) fill_gap(r, p.nrows);  // trailing empty rows
    }
}

// combine the partial slots of the long rows, in chunk order (deterministic)
template <int VEC, bool ISMAX>
__global__ void __launch_bounds__(256) seg_fixup_kernel(const SegParams p, const int32_t* __restrict__ long_rows,
                                                        int n_long) {
    using V = typename VecT<VEC>::T;
    const int64_t nvec = (p.D + VEC - 1) / VEC;
    const int64_t tid = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    const int64_t li = tid / nvec;
    if (li >= n_long) return;
    const int64_t f = (tid % nvec) * VEC;
    const int r = long_rows[li];
    const int rs = p.rowptr[r], re = p.rowptr[r + 1];
    const int k0 = rs / p.chunk, k1 = (re - 1) / p.chunk;
    V acc = *reinterpret_cast<const V*>(p.ws + (size_t)(2 * (int64_t)k0 + 1) * p.D + f);
    for (int kk = k0 + 1; kk <= k1; ++kk) {
        V v = *reinterpret_cast<const V*>(p.ws + (size_t)(2 * (int64_t)kk) * p.D + f);
        acc = comb<ISMAX>(acc, v, 1.f, 1.f);
    }
    acc = finish_row<V>(acc, p, r);
    vst(reinterpret_cast<V*>(p.out + (size_t)r * p.D + f), acc);
}

__global__ void fill_rows_kernel(float* out, int64_t n, float v) {
    int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i < n) out[i] = v;
}
// very sparse graphs (rows >> edges): fill the empty rows row-parallel instead of inside seg_reduce
__global__ void fill_empty_rows_kernel(const int32_t* __restrict__ rowptr, float* out, int64_t nrows,
                                       int64_t D, float v) {
    int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= nrows * D) return;
    int64_t r = i / D;
    if (rowptr[r] == rowptr[r + 1]) out[i] = v;
}

template <int VEC, int TPR, int K, bool ISMAX>
static int launch_seg(const SegParams& p, cudaStream_t st) {
    const int gpb = 256 / TPR;  // groups per block
    dim3 grid((unsigned)ceil_div(p.nchunks, gpb), (unsigned)ceil_div(p.D, (int64_t)VEC * TPR * K));
    // One warp per 512 B row (D = 128 fp32): capped at 64 registers => 4 CTAs x 8 warps per SM (uncapped it takes 77
    // registers, 24 warps).  On an H100 at 700 W the uncapped build was 1 % faster in the GCN propagate at 10 M / 100 M
    // (17.84 against 18.02 ms, DESIGN.md §7); the lean kernel, which serves that shape by default, takes 16.5 ms.
    constexpr bool ROW512 = VEC == 4 && TPR == 32 && K == 1;
    seg_reduce_kernel<VEC, TPR, K, ISMAX, ROW512 ? 8 : 0, ROW512 ? 4 : 1><<<grid, 256, 0, st>>>(p);
    GNNB_LAUNCHED();
    return GNNB_OK;
}

template <int VEC, bool ISMAX>
static int dispatch_seg(const SegParams& p, int tpr, int k, cudaStream_t st) {
#define GNNB_CASE(T, KK) \
    if (tpr == T && k == KK) return launch_seg<VEC, T, KK, ISMAX>(p, st);
    GNNB_CASE(1, 1) GNNB_CASE(2, 1) GNNB_CASE(4, 1) GNNB_CASE(8, 1) GNNB_CASE(16, 1) GNNB_CASE(32, 1)
    GNNB_CASE(32, 2) GNNB_CASE(32, 4)
    if (VEC == 1) { GNNB_CASE(32, 8) }
#undef GNNB_CASE
    GNNB_FAIL(GNNB_EINVAL, "seg_reduce: no kernel for tpr=%d k=%d", tpr, k);
}

static int pow2ceil(int64_t v) {
    int p = 1;
    while (p < v) p <<= 1;
    return p;
}

int seg_reduce_lean(gnnb_graph* g, const Csr& c, const SegArgs& a, float* ws, cudaStream_t st);   // seglean.cu

int seg_reduce(gnnb_graph* g, const Csr& c, const SegArgs& a, cudaStream_t st) {
    if (a.D <= 0) GNNB_FAIL(GNNB_ESIZE, "feature dimension must be positive (got %lld)", (long long)a.D);
    if (c.nrows == 0) return GNNB_OK;
    const bool ismax = (a.aggr == GNNB_MAX || a.aggr == GNNB_MIN);
    if (g->E == 0) {  // every row is empty
        float v = a.aggr == GNNB_MAX ? -HUGE_VALF : (a.aggr == GNNB_MIN ? HUGE_VALF : 0.f);
        int64_t n = (int64_t)c.nrows * a.D;
        fill_rows_kernel<<<(unsigned)ceil_div(n, 256), 256, 0, st>>>(a.out, n, v);
        GNNB_LAUNCHED();
        return GNNB_OK;
    }
    SegParams p;
    p.rowptr = c.rowptr; p.col = c.col; p.row = c.row;
    p.x = a.x; p.x2 = a.x2; p.split = a.split; p.w = a.w; p.cs = a.cs; p.ct = a.ct; p.out = a.out;
    p.D = a.D; p.E = (int32_t)g->E; p.nrows = c.nrows; p.chunk = g->chunk;
    p.nchunks = (int32_t)ceil_div(g->E, g->chunk);
    p.mean = (a.aggr == GNNB_MEAN);
    p.sign = (a.aggr == GNNB_MIN) ? -1.f : 1.f;
    p.fill = 1;
    p.ws = nullptr;
    if (c.n_long > 0) {
        GNNB_TRY(grow_buffer(&g->ws, &g->ws_bytes, (size_t)2 * p.nchunks * a.D * sizeof(float)));
        p.ws = g->ws;
    }
    // the lean work-item kernel (seglean.cu) for rows of 128 / 256 / 512 floats
    int lean_rc = GNNB_EUNSUPPORTED;
    if (!g_reference_kernels) {
        lean_rc = seg_reduce_lean(g, c, a, p.ws, st);
        if (lean_rc != GNNB_OK && lean_rc != GNNB_EUNSUPPORTED) return lean_rc;
    }
    if (lean_rc != GNNB_OK && (int64_t)c.nrows > 4 * g->E) {
        p.fill = 0;
        float v = a.aggr == GNNB_MAX ? -HUGE_VALF : (a.aggr == GNNB_MIN ? HUGE_VALF : 0.f);
        int64_t n = (int64_t)c.nrows * a.D;
        fill_empty_rows_kernel<<<(unsigned)ceil_div(n, 256), 256, 0, st>>>(c.rowptr, a.out, c.nrows, a.D, v);
        GNNB_LAUNCHED();
    }
    const bool vec4 = (a.D % 4 == 0) && ((reinterpret_cast<uintptr_t>(a.x) & 15) == 0) &&
                      ((reinterpret_cast<uintptr_t>(a.x2) & 15) == 0) &&
                      ((reinterpret_cast<uintptr_t>(a.out) & 15) == 0);
    int tpr, k;
    if (lean_rc == GNNB_OK) {
        // done by the lean kernel
    } else if (vec4) {
        int64_t nv = a.D / 4;
        tpr = (int)(nv >= 32 ? 32 : pow2ceil(nv));
        k = (int)ceil_div(nv, tpr);
        k = k >= 4 ? 4 : pow2ceil(k);
        GNNB_TRY(ismax ? (dispatch_seg<4, true>(p, tpr, k, st)) : (dispatch_seg<4, false>(p, tpr, k, st)));
    } else {
        tpr = (int)(a.D >= 32 ? 32 : pow2ceil(a.D));
        k = (int)ceil_div(a.D, tpr);
        k = k >= 8 ? 8 : pow2ceil(k);
        GNNB_TRY(ismax ? (dispatch_seg<1, true>(p, tpr, k, st)) : (dispatch_seg<1, false>(p, tpr, k, st)));
    }
    if (c.n_long > 0) {
        const int vec = vec4 ? 4 : 1;
        int64_t threads = (int64_t)c.n_long * ceil_div(a.D, vec);
        unsigned blocks = (unsigned)ceil_div(threads, 256);
        if (vec4) {
            if (ismax) seg_fixup_kernel<4, true><<<blocks, 256, 0, st>>>(p, c.long_rows, c.n_long);
            else seg_fixup_kernel<4, false><<<blocks, 256, 0, st>>>(p, c.long_rows, c.n_long);
        } else {
            if (ismax) seg_fixup_kernel<1, true><<<blocks, 256, 0, st>>>(p, c.long_rows, c.n_long);
            else seg_fixup_kernel<1, false><<<blocks, 256, 0, st>>>(p, c.long_rows, c.n_long);
        }
        GNNB_LAUNCHED();
    }
    return GNNB_OK;
}

// the partial slots of the long rows of `c`, added in chunk order into out (plain sums: no scale, no mean); float4 when D
// is a multiple of 4 and out, ws are 16 B aligned, scalar otherwise
int seg_fixup_sum(const Csr& c, int64_t E, int chunk, int64_t D, float* ws, float* out, cudaStream_t st) {
    if (c.n_long == 0) return GNNB_OK;
    SegParams p;
    p.rowptr = c.rowptr; p.col = c.col; p.row = c.row;
    p.x = nullptr; p.x2 = nullptr; p.split = 0; p.w = nullptr; p.cs = nullptr; p.ct = nullptr; p.out = out;
    p.D = D; p.E = (int32_t)E; p.nrows = c.nrows; p.chunk = chunk;
    p.nchunks = (int32_t)ceil_div(E, chunk);
    p.mean = 0; p.sign = 1.f; p.fill = 0; p.ws = ws;
    const bool vec4 = D % 4 == 0 && (reinterpret_cast<uintptr_t>(out) & 15) == 0 && (reinterpret_cast<uintptr_t>(ws) & 15) == 0;
    const int64_t threads = (int64_t)c.n_long * (vec4 ? D / 4 : D);
    if (vec4) seg_fixup_kernel<4, false><<<(unsigned)ceil_div(threads, 256), 256, 0, st>>>(p, c.long_rows, c.n_long);
    else seg_fixup_kernel<1, false><<<(unsigned)ceil_div(threads, 256), 256, 0, st>>>(p, c.long_rows, c.n_long);
    GNNB_LAUNCHED();
    return GNNB_OK;
}

// ---- COO <-> plan order for per-edge values ------------------------------------------------------
__global__ void permute_kernel(const int32_t* __restrict__ eid, int64_t E, const float* __restrict__ in,
                               int64_t K, float* __restrict__ out, int to_plan) {
    int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= E * K) return;
    int64_t e = i / K, kk = i % K;
    int64_t src = (int64_t)eid[e] * K + kk;
    if (to_plan) out[i] = __ldg(in + src);
    else out[src] = in[i];
}

int permute_edge_values(const Csr& c, int64_t E, const float* coo_vals, int64_t K, float* plan_vals,
                        cudaStream_t st) {
    if (E * K == 0) return GNNB_OK;
    permute_kernel<<<(unsigned)ceil_div(E * K, 256), 256, 0, st>>>(c.eid, E, coo_vals, K, plan_vals, 1);
    GNNB_LAUNCHED();
    return GNNB_OK;
}
int unpermute_edge_values(const Csr& c, int64_t E, const float* plan_vals, int64_t K,
                          float* coo_vals, cudaStream_t st) {
    if (E * K == 0) return GNNB_OK;
    permute_kernel<<<(unsigned)ceil_div(E * K, 256), 256, 0, st>>>(c.eid, E, plan_vals, K, coo_vals, 0);
    GNNB_LAUNCHED();
    return GNNB_OK;
}

}  // namespace gnnb
