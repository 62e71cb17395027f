// gat.cu — fused GAT edge kernels (the edge part of gat_conv + gat_message, GNNlib/src/layers/conv.jl:136-141,
// 152-167; softmax_edge_neighbors, GNNlib/src/utils.jl:84-97).
//
// The reference materialises Wxi[:,:,t], Wxj[:,:,s], their vcat, the logits, and runs 2 scatters + 2 gathers for the
// softmax plus one more gather/scatter pair for the weighted sum (config 3: >200 GB of temporaries).  Because
// `a` is (2C, H), a·[Wx_i; Wx_j] = el[h,i] + er[h,j] with two per-node scalars per head, so the whole edge part is:
//
//   forward  (one pass over the CSR-by-target edge list, online softmax in registers):
//       u_k = leakyrelu(el[h,i] + er[h,s_k]);  M_i = max_k u_k;  S_i = Σ_k exp(u_k − M_i)
//       out[:,h,i] = ( Σ_k exp(u_k − M_i) · Wx[:,h,s_k] ) / S_i          (M_i, S_i kept for the pullback)
//   backward (one pass over the CSR-by-source edge list; α recomputed from M, S — no (H,E) tensor is read):
//       α_k = exp(u_k − M_i)/S_i;  dα_k = <dout[:,h,i], Wx[:,h,j]>;  T_i = Σ_k α_k dα_k = <dout[:,h,i], out[:,h,i]>
//       dz_k = α_k (dα_k − T_i) · leakyrelu'(z_k)
//       dWx[:,h,j] = Σ_{k: s_k=j} α_k dout[:,h,t_k];   der[h,j] = Σ_{k: s_k=j} dz_k;   del[h,i] = Σ_{k∈N(i)} dz_k
//
// Both passes use the chunk decomposition of segwalk.cuh (load balance independent of the degree distribution,
// long rows through partial slots + a deterministic fix-up; no atomics).  One warp owns a chunk; lane l owns the
// float4 (or scalar) slices (i·32 + l) of the C·H-float row, i < K.
#include "common.cuh"
#include "segwalk.cuh"
#include <math_constants.h>

namespace gnnb {

extern bool g_reference_kernels;   // segreduce.cu: the round-1 chunk kernels for every shape

struct GatParams {
    const int32_t* __restrict__ rowptr;
    const int32_t* __restrict__ col;
    const int32_t* __restrict__ row;
    const int32_t* __restrict__ eid;
    const float* __restrict__ Wx;     // fwd: gathered rows; bwd: own rows        [n_src][D]
    const float* __restrict__ el;     // [n_dst][H]
    const float* __restrict__ er;     // [n_src][H]
    const float* __restrict__ smax;   // [n_dst][H]  (bwd input)
    const float* __restrict__ ssum;   // [n_dst][H]
    const float* __restrict__ tnode;  // [n_dst][H]  T_i (bwd)
    const float* __restrict__ dout;   // [n_dst][D]  (bwd: gathered rows)
    float* __restrict__ out;          // fwd: out [n_dst][D]; bwd: dWx [n_src][D]
    float* __restrict__ stat_a;       // fwd: seg_max; bwd: der [n_src][H]
    float* __restrict__ stat_b;       // fwd: seg_sum
    float* __restrict__ dz;           // bwd: dz in COO order [E][H]
    float* __restrict__ ws;           // partial slots
    int64_t D;                        // C*H
    int32_t C, H;
    int32_t E, nrows, chunk, nchunks;
    int32_t fill;
    float slope;
    const int4* __restrict__ items;   // lean kernels: the plan's work items {e_begin, e_end, slot, 0} (seglean.cu)
    int32_t n_items;
    // HALO instances (a node-partitioned shard): gathered nodes >= split read their row from x2 + (id - split)*D instead
    // of the one base (fwd: Wx, bwd: dout).  Appended last, so the HALO = 0 instances see the fields above where they were.
    int32_t split;
    const float* __restrict__ x2;
};

template <int VEC> struct GV;
template <> struct GV<4> { using T = float4; };
template <> struct GV<1> { using T = float; };
__device__ __forceinline__ float4 gld(const float4* p) { return __ldg(p); }
__device__ __forceinline__ float gld(const float* p) { return __ldg(p); }
__device__ __forceinline__ float4 gzero4() { return make_float4(0.f, 0.f, 0.f, 0.f); }
template <typename V> __device__ __forceinline__ V gzero();
template <> __device__ __forceinline__ float4 gzero<float4>() { return gzero4(); }
template <> __device__ __forceinline__ float gzero<float>() { return 0.f; }
__device__ __forceinline__ float4 gfma(float4 a, float s, float4 v, float p) {  // a*s + v*p
    return make_float4(fmaf(a.x, s, v.x * p), fmaf(a.y, s, v.y * p), fmaf(a.z, s, v.z * p), fmaf(a.w, s, v.w * p));
}
__device__ __forceinline__ float gfma(float a, float s, float v, float p) { return fmaf(a, s, v * p); }
__device__ __forceinline__ float4 gscale(float4 a, float s) { return make_float4(a.x * s, a.y * s, a.z * s, a.w * s); }
__device__ __forceinline__ float gscale(float a, float s) { return a * s; }
__device__ __forceinline__ float4 gdiv(float4 a, float s) {
    return make_float4(__fdiv_rn(a.x, s), __fdiv_rn(a.y, s), __fdiv_rn(a.z, s), __fdiv_rn(a.w, s));
}
__device__ __forceinline__ float gdiv(float a, float s) { return __fdiv_rn(a, s); }
__device__ __forceinline__ float gdot(float4 a, float4 b) { return a.x * b.x + a.y * b.y + a.z * b.z + a.w * b.w; }
__device__ __forceinline__ float gdot(float a, float b) { return a * b; }
__device__ __forceinline__ void gst(float4* p, float4 v) { *p = v; }
__device__ __forceinline__ void gst(float* p, float v) { *p = v; }

// ------------------------------------------------------------------------------------------------ forward
// partial slot layout (floats): [acc: D][M: H][S: H].  HALO: see GatParams::x2 (er stays one array over [local | halo]).
template <int VEC, int K, int HALO>
__global__ void __launch_bounds__(128, (K == 1 ? 8 : 1)) gat_fwd_kernel(const GatParams p) {
    using V = typename GV<VEC>::T;
    constexpr int U = (K >= 4) ? 2 : 4;
    constexpr unsigned FULL = 0xffffffffu;
    const int lane = threadIdx.x & 31;
    const int64_t k = ((int64_t)blockIdx.x * blockDim.x + threadIdx.x) >> 5;
    const int64_t slot = (p.D + 2 * (int64_t)p.H + 3) & ~(int64_t)3;   // keep float4 slots 16 B aligned
    const int64_t d0 = (int64_t)blockIdx.y * (32 * VEC * K);           // feature tile (whole heads per tile)

    int64_t foff[K]; bool fact[K]; int head[K]; bool lead[K];
#pragma unroll
    for (int i = 0; i < K; ++i) {
        foff[i] = d0 + (int64_t)(i * 32 + lane) * VEC;
        fact[i] = foff[i] < p.D;
        head[i] = fact[i] ? (int)(foff[i] / p.C) : 0;
        lead[i] = fact[i] && (foff[i] % p.C == 0);
    }
    const ChunkBounds b = chunk_bounds(p.rowptr, p.row, k, p.chunk, p.E, p.nchunks);
    const bool has_work = b.e_begin < b.e_end;
    const float* const x2s = HALO ? p.x2 - (int64_t)p.split * p.D : nullptr;   // halo base shifted: row id indexes it

    V acc[K]; float M[K], S[K], eli[K];
#pragma unroll
    for (int i = 0; i < K; ++i) { acc[i] = gzero<V>(); M[i] = -CUDART_INF_F; S[i] = 0.f; eli[i] = 0.f; }
    int r = -1;
    bool first_flush = true;

    auto flush = [&](int rr, bool last) {
        const bool to_head = first_flush && b.head_partial;
        const bool to_tail = !to_head && last && b.tail_partial;
        first_flush = false;
        if (to_head || to_tail) {
            float* base = p.ws + (size_t)(2 * k + (to_tail ? 1 : 0)) * slot;
#pragma unroll
            for (int i = 0; i < K; ++i) {
                if (fact[i]) gst(reinterpret_cast<V*>(base + foff[i]), acc[i]);
                if (lead[i]) { base[p.D + head[i]] = M[i]; base[p.D + p.H + head[i]] = S[i]; }
            }
        } else {
#pragma unroll
            for (int i = 0; i < K; ++i) {
                if (fact[i]) gst(reinterpret_cast<V*>(p.out + (size_t)rr * p.D + foff[i]), gdiv(acc[i], S[i]));
                if (lead[i]) {
                    p.stat_a[(size_t)rr * p.H + head[i]] = M[i];
                    p.stat_b[(size_t)rr * p.H + head[i]] = S[i];
                }
            }
        }
    };
    auto fill_gap = [&](int lo, int hi) {
        if (!p.fill) return;
        for (int q = lo + 1; q < hi; ++q) {
#pragma unroll
            for (int i = 0; i < K; ++i) {
                if (fact[i]) gst(reinterpret_cast<V*>(p.out + (size_t)q * p.D + foff[i]), gzero<V>());
                if (lead[i]) { p.stat_a[(size_t)q * p.H + head[i]] = 0.f; p.stat_b[(size_t)q * p.H + head[i]] = 0.f; }
            }
        }
    };

    for (int e = b.e_begin; e < b.e_end; e += 32) {   // warp-uniform bounds
        const int my_e = e + lane;
        int c_l = 0, d_l = -1;
        if (my_e < b.e_end) { c_l = __ldg(p.col + my_e); d_l = __ldg(p.row + my_e); }
        const int nb = min(32, b.e_end - e);
#pragma unroll 1
        for (int j0 = 0; j0 < nb; j0 += U) {
            V v[U][K]; float ev[U][K];
#pragma unroll
            for (int u = 0; u < U; ++u) {
                const int cj = __shfl_sync(FULL, c_l, (j0 + u) & 31);
                const bool valid = (j0 + u) < nb;
                const bool second = HALO != 0 && cj >= p.split;
#pragma unroll
                for (int i = 0; i < K; ++i) {
                    const bool ok = valid && fact[i];
                    if constexpr (HALO == 0) {
                        v[u][i] = ok ? gld(reinterpret_cast<const V*>(p.Wx + (size_t)cj * p.D + foff[i])) : gzero<V>();
                    } else {
                        v[u][i] = ok ? gld(reinterpret_cast<const V*>((second ? x2s : p.Wx) + (size_t)cj * p.D + foff[i])) : gzero<V>();
                    }
                    ev[u][i] = ok ? __ldg(p.er + (size_t)cj * p.H + head[i]) : 0.f;
                }
            }
#pragma unroll
            for (int u = 0; u < U; ++u) {
                const int dj = __shfl_sync(FULL, d_l, (j0 + u) & 31);
                if ((j0 + u) < nb) {
                    if (dj != r) {
                        if (r >= 0) { flush(r, false); fill_gap(r, dj); }
                        else if (!b.head_partial) fill_gap(b.prev_row, dj);
                        r = dj;
#pragma unroll
                        for (int i = 0; i < K; ++i) {
                            acc[i] = gzero<V>(); M[i] = -CUDART_INF_F; S[i] = 0.f;
                            eli[i] = fact[i] ? __ldg(p.el + (size_t)r * p.H + head[i]) : 0.f;
                        }
                    }
#pragma unroll
                    for (int i = 0; i < K; ++i) {
                        const float z = eli[i] + ev[u][i];
                        const float uu = z > 0.f ? z : p.slope * z;
                        const float Mn = fmaxf(M[i], uu);
                        const float Ms = softmax_shift(Mn);
                        const float sc = expf(M[i] - Ms);     // exp(-inf) = 0 on the first edge
                        const float pp = expf(uu - Ms);
                        S[i] = fmaf(S[i], sc, pp);
                        acc[i] = gfma(acc[i], sc, v[u][i], pp);
                        M[i] = Mn;
                    }
                }
            }
        }
    }
    if (has_work) {
        flush(r, true);
        if (b.e_end == p.E) fill_gap(r, p.nrows);
    }
}

// ------------------------------------------------------------------------------------------------ forward, lean
// The same pass on the plan's work-item list (seglean.cu): an item is a run of whole rows or one piece of a long row, so
// the flush path has no case analysis, a warp starts with one 16 B load, row ends are one ballot per 32 edges and all
// control flow is warp-uniform.  The logits of a batch of 32 edges are computed ONCE, lane = edge (H values each, from
// el[target] and er[source]), parked in shared memory and read back by head — the old kernel recomputed every logit on
// every lane of the head and re-read the index arrays for each 128-float tile of the row.  One warp covers the whole
// row of KV*128 floats.  Partial slots keep the layout [acc: D][M: H][S: H], so gat_fwd_fixup_kernel is shared.
// HALO 1: gathered nodes >= split read x2 (seg_lean_kernel's two-base load).
template <int KV, int HALO>
__global__ void __launch_bounds__(256, 2) gat_fwd_lean_kernel(const GatParams p) {
    constexpr unsigned FULL = 0xffffffffu;
    constexpr int U = 8 / KV;
    constexpr int64_t STRIDE = (int64_t)KV * 128;
    extern __shared__ float su[];                      // [warp][edge of the batch][head]
    const int lane = threadIdx.x & 31;
    const int item = blockIdx.x * 8 + (threadIdx.x >> 5);
    if (item >= p.n_items) return;
    const int H = p.H;
    float* myu = su + (threadIdx.x >> 5) * 32 * H;
    const int4 it = __ldg(p.items + item);
    const int e_end = it.y;
    const bool partial = __any_sync(FULL, it.z >= 0);
    int hd[KV]; bool lead[KV];
#pragma unroll
    for (int i = 0; i < KV; ++i) {
        const int f = i * 128 + lane * 4;
        hd[i] = f / p.C;
        lead[i] = (f % p.C) == 0;
    }
    const float* const xl = p.Wx + lane * 4;
    const float* const x2l = HALO ? p.x2 + lane * 4 - (int64_t)p.split * STRIDE : nullptr;
    float4 acc[KV]; float M[KV], S[KV];
#pragma unroll
    for (int i = 0; i < KV; ++i) { acc[i] = gzero4(); M[i] = -CUDART_INF_F; S[i] = 0.f; }

    auto load_lane = [&](int e0, int& c, int& r, bool& last) {
        const int my = e0 + lane;
        c = 0; r = 0; last = false;
        if (my < e_end) {
            c = __ldg(p.col + my);
            r = __ldg(p.row + my);
            last = (my + 1 == e_end) || (__ldg(p.row + my + 1) != r);
        }
    };
    int e = it.x;
    int c_n, r_n; bool last_n;
    load_lane(e, c_n, r_n, last_n);
    bool more = true;
    while (more) {
        const int c_l = c_n, r_l = r_n;
        const bool mine = e + lane < e_end;
        const unsigned vmask = __ballot_sync(FULL, mine);
        const unsigned bmask = partial ? 0u : __ballot_sync(FULL, last_n);
        more = __any_sync(FULL, e + 32 < e_end);
        if (more) load_lane(e + 32, c_n, r_n, last_n);
        if (mine) {                                    // this edge's logits, all heads
            const float* elr = p.el + (int64_t)r_l * H;
            const float* erc = p.er + (int64_t)c_l * H;
            for (int h = 0; h < H; ++h) {
                const float z = __ldg(elr + h) + __ldg(erc + h);
                myu[lane * H + h] = z > 0.f ? z : p.slope * z;
            }
        }
        __syncwarp();
#pragma unroll 1
        for (int j0 = 0; j0 < 32 && (vmask >> j0) != 0u; j0 += U) {
            float4 v[U][KV];
#pragma unroll
            for (int u = 0; u < U; ++u) {
                const int cj = __shfl_sync(FULL, c_l, j0 + u);
                const bool second = HALO != 0 && cj >= p.split;
                const float* xr = (second ? x2l : xl) + (int64_t)cj * STRIDE;
                if ((vmask >> (j0 + u)) & 1u) {
#pragma unroll
                    for (int i = 0; i < KV; ++i) v[u][i] = __ldg(reinterpret_cast<const float4*>(xr + i * 128));
                }
            }
#pragma unroll
            for (int u = 0; u < U; ++u) {
                if ((vmask >> (j0 + u)) & 1u) {
#pragma unroll
                    for (int i = 0; i < KV; ++i) {
                        const float uu = myu[(j0 + u) * H + hd[i]];
                        const float Mn = fmaxf(M[i], uu);
                        const float Ms = softmax_shift(Mn);
                        const float sc = __expf(M[i] - Ms);          // exp(-inf) = 0 on the first edge of a row
                        const float pp = __expf(uu - Ms);
                        S[i] = fmaf(S[i], sc, pp);
                        acc[i] = gfma(acc[i], sc, v[u][i], pp);
                        M[i] = Mn;
                    }
                }
                if ((bmask >> (j0 + u)) & 1u) {                      // row end: normalise and store, exactly once
                    const int rj = __shfl_sync(FULL, r_l, j0 + u);
                    float* o = p.out + (int64_t)rj * STRIDE + lane * 4;
#pragma unroll
                    for (int i = 0; i < KV; ++i) {
                        *reinterpret_cast<float4*>(o + i * 128) = gdiv(acc[i], S[i]);
                        if (lead[i]) {
                            p.stat_a[(int64_t)rj * H + hd[i]] = M[i];
                            p.stat_b[(int64_t)rj * H + hd[i]] = S[i];
                        }
                        acc[i] = gzero4(); M[i] = -CUDART_INF_F; S[i] = 0.f;
                    }
                }
            }
        }
        __syncwarp();                                  // the next batch overwrites the logits
        e += 32;
    }
    if (partial) {
        const int64_t slot = (p.D + 2 * (int64_t)H + 3) & ~(int64_t)3;
        float* base = p.ws + (int64_t)it.z * slot;
#pragma unroll
        for (int i = 0; i < KV; ++i) {
            *reinterpret_cast<float4*>(base + i * 128 + lane * 4) = acc[i];
            if (lead[i]) { base[p.D + hd[i]] = M[i]; base[p.D + H + hd[i]] = S[i]; }
        }
    }
}

// rows without edges: out = 0, statistics = 0 (what the old kernel's fill_gap wrote); one warp per 32 rows
__global__ void __launch_bounds__(256) gat_fill_empty_kernel(const int32_t* __restrict__ rowptr, int32_t nrows,
                                                             float* __restrict__ out, int64_t D, float* __restrict__ sa,
                                                             float* __restrict__ sb, int H) {
    const int lane = threadIdx.x & 31;
    const int64_t r0 = ((int64_t)blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5)) * 32;
    const int64_t r = r0 + lane;
    const bool empty = r < nrows && __ldg(rowptr + r) == __ldg(rowptr + r + 1);
    unsigned m = __ballot_sync(0xffffffffu, empty);
    while (m) {
        const int j = __ffs(m) - 1;
        m &= m - 1;
        float* base = out + (size_t)(r0 + j) * D;
        for (int64_t f = (int64_t)lane * 4; f < D; f += 128) *reinterpret_cast<float4*>(base + f) = gzero4();
        for (int h = lane; h < H; h += 32) { sa[(r0 + j) * H + h] = 0.f; if (sb) sb[(r0 + j) * H + h] = 0.f; }
    }
}

template <int VEC>
__global__ void __launch_bounds__(256) gat_fwd_fixup_kernel(const GatParams p, const int32_t* __restrict__ long_rows,
                                                            int n_long) {
    using V = typename GV<VEC>::T;
    const int64_t nvec = p.D / VEC;
    const int64_t tid = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    const int64_t li = tid / nvec;
    if (li >= n_long) return;
    const int64_t f = (tid % nvec) * VEC;
    const int h = (int)(f / p.C);
    const int64_t slot = (p.D + 2 * (int64_t)p.H + 3) & ~(int64_t)3;   // keep float4 slots 16 B aligned
    const int r = long_rows[li];
    const int rs = p.rowptr[r], re = p.rowptr[r + 1];
    const int k0 = rs / p.chunk, k1 = (re - 1) / p.chunk;
    // M starts at -FLT_MAX, not -Inf: a piece whose logits are all -Inf (M = -Inf, S = 0, acc = 0) then merges as
    // exp(-Inf + FLT_MAX) = 0 instead of exp(-Inf + Inf) = NaN.  On finite pieces the result has the same bits, and the
    // serial chain over the pieces of a long row gets no extra instruction.
    V acc = gzero<V>(); float M = -__int_as_float(0x7f7fffff), S = 0.f;
    for (int kk = k0; kk <= k1; ++kk) {
        const float* base = p.ws + (size_t)(2 * (int64_t)kk + (kk == k0 ? 1 : 0)) * slot;
        const V a = *reinterpret_cast<const V*>(base + f);
        const float Mp = base[p.D + h], Sp = base[p.D + p.H + h];
        const float Mn = fmaxf(M, Mp);
        const float s0 = expf(M - Mn), s1 = expf(Mp - Mn);
        acc = gfma(acc, s0, a, s1);
        S = fmaf(S, s0, Sp * s1);
        M = Mn;
    }
    gst(reinterpret_cast<V*>(p.out + (size_t)r * p.D + f), gdiv(acc, S));
    if (f % p.C == 0) { p.stat_a[(size_t)r * p.H + h] = M; p.stat_b[(size_t)r * p.H + h] = S; }
}

// alpha (H,E) in COO order from the per-target statistics
__global__ void gat_alpha_kernel(const int32_t* __restrict__ s, const int32_t* __restrict__ t, int64_t E, int H,
                                 const float* __restrict__ el, const float* __restrict__ er,
                                 const float* __restrict__ smax, const float* __restrict__ ssum, float slope,
                                 float* __restrict__ alpha) {
    int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= E * H) return;
    int64_t k = i / H; int h = (int)(i % H);
    int64_t ti = t[k], sj = s[k];
    float z = el[ti * H + h] + er[sj * H + h];
    float u = z > 0.f ? z : slope * z;
    alpha[i] = __fdiv_rn(expf(u - smax[ti * H + h]), ssum[ti * H + h]);
}

// T[i,h] = <dout[i,h,:], out[i,h,:]>   (= Σ_k α_k dα_k)
template <int VEC>
__global__ void __launch_bounds__(256) gat_tnode_kernel(const float* __restrict__ dout, const float* __restrict__ outf,
                                                        int64_t n, int64_t D, int C, int H, float* __restrict__ T) {
    using V = typename GV<VEC>::T;
    const int lane = threadIdx.x & 31;
    const int64_t i = ((int64_t)blockIdx.x * blockDim.x + threadIdx.x) >> 5;
    if (i >= n) return;
    const int L = C / VEC;
    const int nslice = (int)((D / VEC + 31) / 32);
    for (int q = 0; q < nslice; ++q) {
        const int64_t f = (int64_t)(q * 32 + lane) * VEC;
        float d = 0.f;
        if (f < D) d = gdot(gld(reinterpret_cast<const V*>(dout + i * D + f)), gld(reinterpret_cast<const V*>(outf + i * D + f)));
        for (int o = L >> 1; o > 0; o >>= 1) d += __shfl_xor_sync(0xffffffffu, d, o);
        if (f < D && (f % C) == 0) T[i * H + f / C] = d;
    }
}

// ----------------------------------------------------------------------------------------------- backward
// CSR-by-source: row j = source node; col = target i.  partial slot layout: [acc: D][der: H]
// (on a shard: the forward CSR of the backward shard, whose rows are the owned sources and whose gathered nodes are the
// targets in [local | halo]; HALO 1 reads the dout rows of targets >= split from x2, el / M / S / T stay one array each)
template <int VEC, int K, int HALO>
__global__ void __launch_bounds__(128, (K == 1 ? 5 : 1)) gat_bwd_kernel(const GatParams p) {
    using V = typename GV<VEC>::T;
    constexpr int U = (K >= 4) ? 2 : 4;
    constexpr unsigned FULL = 0xffffffffu;
    const int lane = threadIdx.x & 31;
    const int64_t k = ((int64_t)blockIdx.x * blockDim.x + threadIdx.x) >> 5;
    const int64_t slot = (p.D + (int64_t)p.H + 3) & ~(int64_t)3;
    const int L = p.C / VEC;   // lanes per head (power of two <= 32)
    const int64_t d0 = (int64_t)blockIdx.y * (32 * VEC * K);

    int64_t foff[K]; bool fact[K]; int head[K]; bool lead[K];
#pragma unroll
    for (int i = 0; i < K; ++i) {
        foff[i] = d0 + (int64_t)(i * 32 + lane) * VEC;
        fact[i] = foff[i] < p.D;
        head[i] = fact[i] ? (int)(foff[i] / p.C) : 0;
        lead[i] = fact[i] && (foff[i] % p.C == 0);
    }
    const ChunkBounds b = chunk_bounds(p.rowptr, p.row, k, p.chunk, p.E, p.nchunks);
    const bool has_work = b.e_begin < b.e_end;
    const float* const x2s = HALO ? p.x2 - (int64_t)p.split * p.D : nullptr;   // halo base shifted: row id indexes it

    V acc[K], wxj[K]; float dacc[K], erj[K];
#pragma unroll
    for (int i = 0; i < K; ++i) { acc[i] = gzero<V>(); wxj[i] = gzero<V>(); dacc[i] = 0.f; erj[i] = 0.f; }
    int r = -1;
    bool first_flush = true;

    auto flush = [&](int rr, bool last) {
        const bool to_head = first_flush && b.head_partial;
        const bool to_tail = !to_head && last && b.tail_partial;
        first_flush = false;
        float* base; float* dbase;
        if (to_head || to_tail) {
            base = p.ws + (size_t)(2 * k + (to_tail ? 1 : 0)) * slot;
            dbase = base + p.D;
        } else {
            base = p.out + (size_t)rr * p.D;
            dbase = p.stat_a + (size_t)rr * p.H;
        }
#pragma unroll
        for (int i = 0; i < K; ++i) {
            if (fact[i]) gst(reinterpret_cast<V*>(base + foff[i]), acc[i]);
            if (lead[i]) dbase[head[i]] = dacc[i];
        }
    };
    auto fill_gap = [&](int lo, int hi) {
        if (!p.fill) return;
        for (int q = lo + 1; q < hi; ++q) {
#pragma unroll
            for (int i = 0; i < K; ++i) {
                if (fact[i]) gst(reinterpret_cast<V*>(p.out + (size_t)q * p.D + foff[i]), gzero<V>());
                if (lead[i]) p.stat_a[(size_t)q * p.H + head[i]] = 0.f;
            }
        }
    };

    for (int e = b.e_begin; e < b.e_end; e += 32) {
        const int my_e = e + lane;
        int c_l = 0, d_l = -1, id_l = 0;
        if (my_e < b.e_end) { c_l = __ldg(p.col + my_e); d_l = __ldg(p.row + my_e); id_l = __ldg(p.eid + my_e); }
        const int nb = min(32, b.e_end - e);
#pragma unroll 1
        for (int j0 = 0; j0 < nb; j0 += U) {
            V v[U][K]; float eli[U][K], Mi[U][K], Si[U][K], Ti[U][K];
#pragma unroll
            for (int u = 0; u < U; ++u) {
                const int ci = __shfl_sync(FULL, c_l, (j0 + u) & 31);
                const bool valid = (j0 + u) < nb;
                const bool second = HALO != 0 && ci >= p.split;
#pragma unroll
                for (int i = 0; i < K; ++i) {
                    const bool ok = valid && fact[i];
                    const size_t hq = (size_t)ci * p.H + head[i];
                    if constexpr (HALO == 0) {
                        v[u][i] = ok ? gld(reinterpret_cast<const V*>(p.dout + (size_t)ci * p.D + foff[i])) : gzero<V>();
                    } else {
                        v[u][i] = ok ? gld(reinterpret_cast<const V*>((second ? x2s : p.dout) + (size_t)ci * p.D + foff[i])) : gzero<V>();
                    }
                    eli[u][i] = ok ? __ldg(p.el + hq) : 0.f;
                    Mi[u][i] = ok ? __ldg(p.smax + hq) : 0.f;
                    Si[u][i] = ok ? __ldg(p.ssum + hq) : 1.f;
                    Ti[u][i] = ok ? __ldg(p.tnode + hq) : 0.f;
                }
            }
#pragma unroll
            for (int u = 0; u < U; ++u) {
                const int dj = __shfl_sync(FULL, d_l, (j0 + u) & 31);
                const int ek = __shfl_sync(FULL, id_l, (j0 + u) & 31);
                if ((j0 + u) < nb) {      // warp-uniform
                    if (dj != r) {
                        if (r >= 0) { flush(r, false); fill_gap(r, dj); }
                        else if (!b.head_partial) fill_gap(b.prev_row, dj);
                        r = dj;
#pragma unroll
                        for (int i = 0; i < K; ++i) {
                            acc[i] = gzero<V>(); dacc[i] = 0.f;
                            wxj[i] = fact[i] ? gld(reinterpret_cast<const V*>(p.Wx + (size_t)r * p.D + foff[i])) : gzero<V>();
                            erj[i] = fact[i] ? __ldg(p.er + (size_t)r * p.H + head[i]) : 0.f;
                        }
                    }
#pragma unroll
                    for (int i = 0; i < K; ++i) {
                        float da = gdot(v[u][i], wxj[i]);
                        for (int o = L >> 1; o > 0; o >>= 1) da += __shfl_xor_sync(FULL, da, o);
                        const float z = eli[u][i] + erj[i];
                        const float uu = z > 0.f ? z : p.slope * z;
                        const float al = __fdiv_rn(expf(uu - Mi[u][i]), Si[u][i]);
                        const float dzv = al * (da - Ti[u][i]) * (z > 0.f ? 1.f : p.slope);
                        acc[i] = gfma(acc[i], 1.f, v[u][i], al);
                        dacc[i] += dzv;
                        if (lead[i]) p.dz[(size_t)ek * p.H + head[i]] = dzv;
                    }
                }
            }
        }
    }
    if (has_work) {
        flush(r, true);
        if (b.e_end == p.E) fill_gap(r, p.nrows);
    }
}

// ----------------------------------------------------------------------------------------------- backward, lean
// The same pass on the work-item list of the CSR-by-source plan.  Per batch of 32 edges the per-edge-per-head scalars are
// computed ONCE, lane = edge: α (from el, er and the forward's M, S), α·leakyrelu'(z) and T of the target — parked in shared
// memory; the old kernel gathered el / M / S / T and re-evaluated exp on every lane of the head, per 128-float tile.
// The source's own Wx row is read beside every gathered dout row (an L1 hit after the row's first edge) instead of being
// loaded at the row change, where the in-order warp sat out a full memory latency every ~11 edges.
// Partial slots keep the layout [acc: D][der: H] of gat_bwd_fixup_kernel.  C <= 128 (a head never spans two slices).
// HALO 1: the dout rows of gathered targets >= split come from x2.
template <int KV, int HALO>
__global__ void __launch_bounds__(256, 2) gat_bwd_lean_kernel(const GatParams p) {
    constexpr unsigned FULL = 0xffffffffu;
    constexpr int U = (KV >= 4) ? 2 : (KV == 2 ? 2 : 4);
    constexpr int64_t STRIDE = (int64_t)KV * 128;
    extern __shared__ float su[];                      // [warp][3][edge of the batch][head]: α, α·lrelu', T
    const int lane = threadIdx.x & 31;
    const int item = blockIdx.x * 8 + (threadIdx.x >> 5);
    if (item >= p.n_items) return;
    const int H = p.H;
    float* sa = su + (threadIdx.x >> 5) * 3 * 32 * H;
    float* sb = sa + 32 * H;
    float* st_ = sb + 32 * H;
    const int4 it = __ldg(p.items + item);
    const int e_end = it.y;
    const bool partial = __any_sync(FULL, it.z >= 0);
    const int L = p.C >> 2;                            // lanes per head (power of two <= 32)
    int hd[KV]; bool lead[KV];
#pragma unroll
    for (int i = 0; i < KV; ++i) {
        const int f = i * 128 + lane * 4;
        hd[i] = f / p.C;
        lead[i] = (f % p.C) == 0;
    }
    const float* const dl = p.dout + lane * 4;
    const float* const d2l = HALO ? p.x2 + lane * 4 - (int64_t)p.split * STRIDE : nullptr;
    const float* const wl = p.Wx + lane * 4;
    float4 acc[KV]; float dacc[KV];
#pragma unroll
    for (int i = 0; i < KV; ++i) { acc[i] = gzero4(); dacc[i] = 0.f; }

    auto load_lane = [&](int e0, int& c, int& r, int& id, bool& last) {
        const int my = e0 + lane;
        c = 0; r = 0; id = 0; last = false;
        if (my < e_end) {
            c = __ldg(p.col + my);
            r = __ldg(p.row + my);
            id = __ldg(p.eid + my);
            last = (my + 1 == e_end) || (__ldg(p.row + my + 1) != r);
        }
    };
    int e = it.x;
    int c_n, r_n, id_n; bool last_n;
    load_lane(e, c_n, r_n, id_n, last_n);
    bool more = true;
    while (more) {
        const int c_l = c_n, r_l = r_n, id_l = id_n;
        const bool mine = e + lane < e_end;
        const unsigned vmask = __ballot_sync(FULL, mine);
        const unsigned bmask = partial ? 0u : __ballot_sync(FULL, last_n);
        more = __any_sync(FULL, e + 32 < e_end);
        if (more) load_lane(e + 32, c_n, r_n, id_n, last_n);
        if (mine) {                                    // this edge's attention scalars, all heads
            const int64_t ti = (int64_t)c_l * H, sj = (int64_t)r_l * H;
            for (int h = 0; h < H; ++h) {
                const float z = __ldg(p.el + ti + h) + __ldg(p.er + sj + h);
                const float uu = z > 0.f ? z : p.slope * z;
                const float al = __fdiv_rn(__expf(uu - __ldg(p.smax + ti + h)), __ldg(p.ssum + ti + h));
                sa[lane * H + h] = al;
                sb[lane * H + h] = al * (z > 0.f ? 1.f : p.slope);
                st_[lane * H + h] = __ldg(p.tnode + ti + h);
            }
        }
        __syncwarp();
#pragma unroll 1
        for (int j0 = 0; j0 < 32 && (vmask >> j0) != 0u; j0 += U) {
            float4 v[U][KV], w[U][KV];
#pragma unroll
            for (int u = 0; u < U; ++u) {
                const int ci = __shfl_sync(FULL, c_l, j0 + u);
                const int rj = __shfl_sync(FULL, r_l, j0 + u);
                const bool second = HALO != 0 && ci >= p.split;
                const float* dr = (second ? d2l : dl) + (int64_t)ci * STRIDE;
                const float* wr = wl + (int64_t)rj * STRIDE;
                if ((vmask >> (j0 + u)) & 1u) {
#pragma unroll
                    for (int i = 0; i < KV; ++i) {
                        v[u][i] = __ldg(reinterpret_cast<const float4*>(dr + i * 128));
                        w[u][i] = __ldg(reinterpret_cast<const float4*>(wr + i * 128));
                    }
                }
            }
#pragma unroll
            for (int u = 0; u < U; ++u) {
                const int ek = __shfl_sync(FULL, id_l, j0 + u);
                if ((vmask >> (j0 + u)) & 1u) {
#pragma unroll
                    for (int i = 0; i < KV; ++i) {
                        float da = gdot(v[u][i], w[u][i]);
                        for (int o = L >> 1; o > 0; o >>= 1) da += __shfl_xor_sync(FULL, da, o);
                        const int q = (j0 + u) * H + hd[i];
                        const float dzv = sb[q] * (da - st_[q]);
                        acc[i] = gfma(acc[i], 1.f, v[u][i], sa[q]);
                        dacc[i] += dzv;
                        if (lead[i]) p.dz[(int64_t)ek * H + hd[i]] = dzv;
                    }
                }
                if ((bmask >> (j0 + u)) & 1u) {                      // row end: dWx row and der, exactly once
                    const int rj = __shfl_sync(FULL, r_l, j0 + u);
                    float* o = p.out + (int64_t)rj * STRIDE + lane * 4;
#pragma unroll
                    for (int i = 0; i < KV; ++i) {
                        *reinterpret_cast<float4*>(o + i * 128) = acc[i];
                        if (lead[i]) p.stat_a[(int64_t)rj * H + hd[i]] = dacc[i];
                        acc[i] = gzero4(); dacc[i] = 0.f;
                    }
                }
            }
        }
        __syncwarp();
        e += 32;
    }
    if (partial) {
        const int64_t slot = (p.D + (int64_t)H + 3) & ~(int64_t)3;
        float* base = p.ws + (int64_t)it.z * slot;
#pragma unroll
        for (int i = 0; i < KV; ++i) {
            *reinterpret_cast<float4*>(base + i * 128 + lane * 4) = acc[i];
            if (lead[i]) base[p.D + hd[i]] = dacc[i];
        }
    }
}

template <int VEC>
__global__ void __launch_bounds__(256) gat_bwd_fixup_kernel(const GatParams p, const int32_t* __restrict__ long_rows,
                                                            int n_long) {
    using V = typename GV<VEC>::T;
    const int64_t nvec = p.D / VEC;
    const int64_t tid = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    const int64_t li = tid / nvec;
    if (li >= n_long) return;
    const int64_t f = (tid % nvec) * VEC;
    const int h = (int)(f / p.C);
    const int64_t slot = (p.D + (int64_t)p.H + 3) & ~(int64_t)3;
    const int r = long_rows[li];
    const int rs = p.rowptr[r], re = p.rowptr[r + 1];
    const int k0 = rs / p.chunk, k1 = (re - 1) / p.chunk;
    V acc = gzero<V>(); float d = 0.f;
    for (int kk = k0; kk <= k1; ++kk) {
        const float* base = p.ws + (size_t)(2 * (int64_t)kk + (kk == k0 ? 1 : 0)) * slot;
        acc = gfma(acc, 1.f, *reinterpret_cast<const V*>(base + f), 1.f);
        d += base[p.D + h];
    }
    gst(reinterpret_cast<V*>(p.out + (size_t)r * p.D + f), acc);
    if (f % p.C == 0) p.stat_a[(size_t)r * p.H + h] = d;
}

__global__ void gat_zero_kernel(float* a, int64_t n) {
    int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i < n) a[i] = 0.f;
}

// shapes the fused kernels cover: vec4: C/4 a power of two <= 32 (C | 128, so a 128-float tile holds whole heads; any H,
// grid.y tiles the row); scalar: C a power of two <= 32 with C*H <= 128
static bool gat_shape(int64_t C, int64_t H, const void* a, const void* b, int* vec, int* kk) {
    const int64_t D = C * H;
    auto pow2 = [](int64_t v) { return v > 0 && (v & (v - 1)) == 0; };
    const bool aligned = !((uintptr_t)a & 15) && !((uintptr_t)b & 15);
    if (C % 4 == 0 && aligned && pow2(C / 4) && C / 4 <= 32) {
        *vec = 4; *kk = 1;
        return true;
    }
    if (pow2(C) && C <= 32 && D <= 128) {
        *vec = 1; int k = (int)ceil_div(D, 32); *kk = k <= 1 ? 1 : (k == 2 ? 2 : 4);
        return true;
    }
    return false;
}

}  // namespace gnnb

using namespace gnnb;
static inline unsigned nblk(int64_t n) { return (unsigned)ceil_div(n, 256); }

#define GAT_DISPATCH(KERNEL, HALO, vec, kk, grid, st, p)                                      \
    do {                                                                                      \
        if (vec == 4) KERNEL<4, 1, HALO><<<grid, 128, 0, st>>>(p);                            \
        else if (kk == 1) KERNEL<1, 1, HALO><<<grid, 128, 0, st>>>(p);                        \
        else if (kk == 2) KERNEL<1, 2, HALO><<<grid, 128, 0, st>>>(p);                        \
        else KERNEL<1, 4, HALO><<<grid, 128, 0, st>>>(p);                                     \
    } while (0)

namespace {

template <int HALO>
int gat_fwd_lean(const GatParams& p, int64_t D, size_t smem, cudaStream_t st) {
    const unsigned blocks = (unsigned)ceil_div(p.n_items, 8);
    if (smem > 48 * 1024) {
        GNNB_CUDA(cudaFuncSetAttribute(gat_fwd_lean_kernel<1, HALO>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
        GNNB_CUDA(cudaFuncSetAttribute(gat_fwd_lean_kernel<2, HALO>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
        GNNB_CUDA(cudaFuncSetAttribute(gat_fwd_lean_kernel<4, HALO>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
    }
    if (D == 128) gat_fwd_lean_kernel<1, HALO><<<blocks, 256, smem, st>>>(p);
    else if (D == 256) gat_fwd_lean_kernel<2, HALO><<<blocks, 256, smem, st>>>(p);
    else gat_fwd_lean_kernel<4, HALO><<<blocks, 256, smem, st>>>(p);
    GNNB_LAUNCHED();
    return GNNB_OK;
}

template <int HALO>
int gat_bwd_lean(const GatParams& p, int64_t D, size_t smem, cudaStream_t st) {
    const unsigned blocks = (unsigned)ceil_div(p.n_items, 8);
    if (smem > 48 * 1024) {
        GNNB_CUDA(cudaFuncSetAttribute(gat_bwd_lean_kernel<1, HALO>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
        GNNB_CUDA(cudaFuncSetAttribute(gat_bwd_lean_kernel<2, HALO>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
        GNNB_CUDA(cudaFuncSetAttribute(gat_bwd_lean_kernel<4, HALO>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
    }
    if (D == 128) gat_bwd_lean_kernel<1, HALO><<<blocks, 256, smem, st>>>(p);
    else if (D == 256) gat_bwd_lean_kernel<2, HALO><<<blocks, 256, smem, st>>>(p);
    else gat_bwd_lean_kernel<4, HALO><<<blocks, 256, smem, st>>>(p);
    GNNB_LAUNCHED();
    return GNNB_OK;
}

// The forward pass over g's by-target CSR, the one launch path of gnnb_gat_aggregate (x2 = NULL) and of
// gnnb_gat_aggregate_halo (gathered nodes >= split read x2): out, seg_max, seg_sum over the CSR's rows.
int gat_forward(gnnb_graph* g, const float* Wx, const float* x2, int64_t split, const float* el, const float* er, int64_t C,
                int64_t H, float slope, float* out, float* seg_max, float* seg_sum, int vec, int kk, cudaStream_t st) {
    GNNB_TRY(ensure_csr(g, false, st));
    const Csr& c = g->by_dst;
    const int64_t D = C * H;
    if (c.nrows == 0) return GNNB_OK;
    if (g->E == 0) {
        gat_zero_kernel<<<nblk((int64_t)c.nrows * D), 256, 0, st>>>(out, (int64_t)c.nrows * D); GNNB_LAUNCHED();
        gat_zero_kernel<<<nblk((int64_t)c.nrows * H), 256, 0, st>>>(seg_max, (int64_t)c.nrows * H); GNNB_LAUNCHED();
        gat_zero_kernel<<<nblk((int64_t)c.nrows * H), 256, 0, st>>>(seg_sum, (int64_t)c.nrows * H); GNNB_LAUNCHED();
        return GNNB_OK;
    }
    GatParams p = {};
    p.rowptr = c.rowptr; p.col = c.col; p.row = c.row; p.eid = c.eid;
    p.Wx = Wx; p.el = el; p.er = er; p.out = out; p.stat_a = seg_max; p.stat_b = seg_sum;
    p.D = D; p.C = (int32_t)C; p.H = (int32_t)H; p.E = (int32_t)g->E; p.nrows = c.nrows; p.chunk = g->chunk;
    p.nchunks = (int32_t)ceil_div(g->E, g->chunk); p.fill = 1; p.slope = slope;
    p.x2 = x2; p.split = (int32_t)split;
    const bool halo = x2 != nullptr;
    if (c.n_long > 0) {
        GNNB_TRY(grow_buffer(&g->ws, &g->ws_bytes, sizeof(float) * (size_t)2 * p.nchunks * (D + 2 * H + 4)));
        p.ws = g->ws;
    }
    const bool lean = !g_reference_kernels && vec == 4 && (D == 128 || D == 256 || D == 512) && (C & (C - 1)) == 0 && H <= 64;
    if (lean) {                                    // the work-item kernel (one warp per whole row, logits once per edge)
        GNNB_TRY(ensure_items(g, c, st));
        p.items = reinterpret_cast<const int4*>(c.items); p.n_items = c.n_items;
        if (c.n_empty > 0) {
            gat_fill_empty_kernel<<<(unsigned)ceil_div((int64_t)c.nrows, 256), 256, 0, st>>>(c.rowptr, c.nrows, out, D, seg_max, seg_sum, (int)H);
            GNNB_LAUNCHED();
        }
        const size_t smem = sizeof(float) * 8 * 32 * (size_t)H;
        GNNB_TRY(halo ? gat_fwd_lean<1>(p, D, smem, st) : gat_fwd_lean<0>(p, D, smem, st));
    } else {
        const dim3 grid((unsigned)ceil_div(p.nchunks, 4), (unsigned)ceil_div(D, (int64_t)32 * vec * kk));
        if (halo) GAT_DISPATCH(gat_fwd_kernel, 1, vec, kk, grid, st, p);
        else GAT_DISPATCH(gat_fwd_kernel, 0, vec, kk, grid, st, p);
        GNNB_LAUNCHED();
    }
    if (c.n_long > 0) {
        const unsigned fb = nblk((int64_t)c.n_long * (D / vec));
        if (vec == 4) gat_fwd_fixup_kernel<4><<<fb, 256, 0, st>>>(p, c.long_rows, c.n_long);
        else gat_fwd_fixup_kernel<1><<<fb, 256, 0, st>>>(p, c.long_rows, c.n_long);
        GNNB_LAUNCHED();
    }
    return GNNB_OK;
}

// The pullback pass over a CSR `c` of g whose rows are the sources j and whose gathered nodes are the targets i: the
// by-source CSR of a graph (gnnb_gat_aggregate_bwd, x2 = NULL) or the by-target CSR of a backward shard
// (gnnb_gat_aggregate_bwd_halo).  Needs E > 0.  Writes dWx and der over c's rows, dz (E, H) in g's COO order.
int gat_backward(gnnb_graph* g, const Csr& c, const float* Wx, const float* er, const float* dout, const float* x2,
                 int64_t split, const float* el, const float* seg_max, const float* seg_sum, const float* T, int64_t C,
                 int64_t H, float slope, float* dWx, float* der, float* dz, int vec, int kk, cudaStream_t st) {
    const int64_t D = C * H;
    GatParams p = {};
    p.rowptr = c.rowptr; p.col = c.col; p.row = c.row; p.eid = c.eid;
    p.Wx = Wx; p.el = el; p.er = er; p.smax = seg_max; p.ssum = seg_sum; p.tnode = T; p.dout = dout;
    p.out = dWx; p.stat_a = der; p.dz = dz;
    p.D = D; p.C = (int32_t)C; p.H = (int32_t)H; p.E = (int32_t)g->E; p.nrows = c.nrows; p.chunk = g->chunk;
    p.nchunks = (int32_t)ceil_div(g->E, g->chunk); p.fill = 1; p.slope = slope;
    p.x2 = x2; p.split = (int32_t)split;
    const bool halo = x2 != nullptr;
    if (c.n_long > 0) {
        GNNB_TRY(grow_buffer(&g->ws, &g->ws_bytes, sizeof(float) * (size_t)2 * p.nchunks * (D + H + 4)));
        p.ws = g->ws;
    }
    const bool lean = !g_reference_kernels && vec == 4 && (D == 128 || D == 256 || D == 512) && (C & (C - 1)) == 0 && C <= 128 && H <= 64;
    if (lean) {
        GNNB_TRY(ensure_items(g, c, st));
        p.items = reinterpret_cast<const int4*>(c.items); p.n_items = c.n_items;
        if (c.n_empty > 0) {
            gat_fill_empty_kernel<<<(unsigned)ceil_div((int64_t)c.nrows, 256), 256, 0, st>>>(c.rowptr, c.nrows, dWx, D, der, nullptr, (int)H);
            GNNB_LAUNCHED();
        }
        const size_t smem = sizeof(float) * 8 * 3 * 32 * (size_t)H;
        GNNB_TRY(halo ? gat_bwd_lean<1>(p, D, smem, st) : gat_bwd_lean<0>(p, D, smem, st));
    } else {
        const dim3 grid((unsigned)ceil_div(p.nchunks, 4), (unsigned)ceil_div(D, (int64_t)32 * vec * kk));
        if (halo) GAT_DISPATCH(gat_bwd_kernel, 1, vec, kk, grid, st, p);
        else GAT_DISPATCH(gat_bwd_kernel, 0, vec, kk, grid, st, p);
        GNNB_LAUNCHED();
    }
    if (c.n_long > 0) {
        const unsigned fb = nblk((int64_t)c.n_long * (D / vec));
        if (vec == 4) gat_bwd_fixup_kernel<4><<<fb, 256, 0, st>>>(p, c.long_rows, c.n_long);
        else gat_bwd_fixup_kernel<1><<<fb, 256, 0, st>>>(p, c.long_rows, c.n_long);
        GNNB_LAUNCHED();
    }
    return GNNB_OK;
}

int gat_tnode(const float* dout, const float* out_fwd, int64_t n, int64_t C, int64_t H, int vec, float* T, cudaStream_t st) {
    const unsigned tb = nblk(n * 32);
    if (vec == 4) gat_tnode_kernel<4><<<tb, 256, 0, st>>>(dout, out_fwd, n, C * H, (int)C, (int)H, T);
    else gat_tnode_kernel<1><<<tb, 256, 0, st>>>(dout, out_fwd, n, C * H, (int)C, (int)H, T);
    GNNB_LAUNCHED();
    return GNNB_OK;
}

// the two gathered bases of a halo entry: the local one, and the halo one only when some gathered node lives there
// (a shard without halo rows takes the HALO = 0 instances); no local rows at all: the halo base alone, split 0
void gat_bases(const float* local, const float* halo, int64_t n_local, int64_t n_src, const float** x, const float** x2) {
    *x = local;
    *x2 = n_local < n_src ? halo : nullptr;
    if (!local) { *x = halo; *x2 = nullptr; }
}

}  // namespace

extern "C" {

int gnnb_gat_aggregate(gnnb_graph_t g, const float* Wx, const float* el, const float* er, int64_t C, int64_t H,
                       float slope, float* out, float* alpha, float* seg_max, float* seg_sum, void* stream) {
    if (!g) GNNB_FAIL(GNNB_EINVAL, "graph handle is NULL");
    if (C <= 0 || H <= 0) GNNB_FAIL(GNNB_ESIZE, "C and H must be positive");
    if (!Wx || !el || !er || !out || !seg_max || !seg_sum) GNNB_FAIL(GNNB_EINVAL, "NULL argument");
    int vec, kk;
    if (!gat_shape(C, H, Wx, out, &vec, &kk))
        GNNB_FAIL(GNNB_EUNSUPPORTED, "fused GAT needs C/4 a power of two <= 32 with 16 B-aligned Wx / out (any number of heads), or C a "
                                     "power of two <= 32 with C*H <= 128; use the generic apply_edges/softmax_edge_neighbors/"
                                     "aggregate_neighbors composition");
    cudaStream_t st = (cudaStream_t)stream;
    GNNB_TRY(gat_forward(g, Wx, nullptr, 0, el, er, C, H, slope, out, seg_max, seg_sum, vec, kk, st));
    if (alpha && g->by_dst.nrows > 0 && g->E > 0) {
        gat_alpha_kernel<<<nblk(g->E * H), 256, 0, st>>>(g->coo_src, g->coo_dst, g->E, (int)H, el, er, seg_max, seg_sum,
                                                          slope, alpha);
        GNNB_LAUNCHED();
    }
    return GNNB_OK;
}

int gnnb_gat_aggregate_halo(gnnb_graph_t g, const float* Wx_local, const float* Wx_halo, int64_t n_local, const float* el,
                            const float* er, int64_t C, int64_t H, float slope, float* out, float* seg_max, float* seg_sum,
                            void* stream) {
    if (!g) GNNB_FAIL(GNNB_EINVAL, "graph handle is NULL");
    if (C <= 0 || H <= 0) GNNB_FAIL(GNNB_ESIZE, "C and H must be positive");
    if (n_local < 0 || n_local > g->n_src) GNNB_FAIL(GNNB_ESIZE, "n_local must be in [0, num_src]");
    if (g->n_dst == 0) return GNNB_OK;   // a rank that owns no node: no row to write, the outputs may be NULL
    if (!el || !out || !seg_max || !seg_sum || (g->E > 0 && !er)) GNNB_FAIL(GNNB_EINVAL, "NULL argument");
    if (n_local > 0 && !Wx_local) GNNB_FAIL(GNNB_EINVAL, "Wx_local is NULL");
    if (n_local < g->n_src && !Wx_halo) GNNB_FAIL(GNNB_EINVAL, "Wx_halo is NULL but the shard has halo sources");
    const float *x, *x2;
    gat_bases(Wx_local, Wx_halo, n_local, g->n_src, &x, &x2);
    int vec, kk;
    const void* both = reinterpret_cast<const void*>(reinterpret_cast<uintptr_t>(x) | reinterpret_cast<uintptr_t>(x2));
    if (!gat_shape(C, H, both, out, &vec, &kk))     // `both`: the vector path needs each gathered base 16 B-aligned
        GNNB_FAIL(GNNB_EUNSUPPORTED, "fused GAT needs C/4 a power of two <= 32 with 16 B-aligned Wx_local / Wx_halo / out, or C a "
                                     "power of two <= 32 with C*H <= 128");
    return gat_forward(g, x, x2, n_local, el, er, C, H, slope, out, seg_max, seg_sum, vec, kk, (cudaStream_t)stream);
}

int gnnb_gat_aggregate_bwd(gnnb_graph_t g, const float* Wx, const float* el, const float* er, const float* seg_max,
                           const float* seg_sum, const float* out_fwd, const float* dout, int64_t C, int64_t H,
                           float slope, float* dWx, float* del, float* der, void* stream) {
    if (!g) GNNB_FAIL(GNNB_EINVAL, "graph handle is NULL");
    if (C <= 0 || H <= 0) GNNB_FAIL(GNNB_ESIZE, "C and H must be positive");
    if (!Wx || !el || !er || !seg_max || !seg_sum || !out_fwd || !dout || !dWx || !del || !der)
        GNNB_FAIL(GNNB_EINVAL, "NULL argument");
    int vec, kk;
    if (!gat_shape(C, H, Wx, dWx, &vec, &kk) || ((uintptr_t)dout & 15) || ((uintptr_t)out_fwd & 15))
        GNNB_FAIL(GNNB_EUNSUPPORTED, "fused GAT pullback: unsupported (C,H) or unaligned pointers");
    cudaStream_t st = (cudaStream_t)stream;
    GNNB_TRY(ensure_csr(g, true, st));
    const int64_t D = C * H;
    const int64_t n_dst = g->n_dst, n_src = g->n_src;
    if (n_src > 0 && g->E == 0) {
        gat_zero_kernel<<<nblk(n_src * D), 256, 0, st>>>(dWx, n_src * D); GNNB_LAUNCHED();
        gat_zero_kernel<<<nblk(n_src * H), 256, 0, st>>>(der, n_src * H); GNNB_LAUNCHED();
    }
    if (g->E == 0) {
        if (n_dst > 0) { gat_zero_kernel<<<nblk(n_dst * H), 256, 0, st>>>(del, n_dst * H); GNNB_LAUNCHED(); }
        return GNNB_OK;
    }
    // ws2: [T: n_dst*H][dz: E*H]
    GNNB_TRY(grow_buffer(&g->ws2, &g->ws2_bytes, sizeof(float) * ((size_t)n_dst * H + (size_t)g->E * H)));
    float* T = g->ws2;
    float* dz = g->ws2 + (size_t)n_dst * H;
    GNNB_TRY(gat_tnode(dout, out_fwd, n_dst, C, H, vec, T, st));
    GNNB_TRY(gat_backward(g, g->by_src, Wx, er, dout, nullptr, 0, el, seg_max, seg_sum, T, C, H, slope, dWx, der, dz, vec,
                          kk, st));
    // del[h,i] = Σ_{k in N(i)} dz_k : the library's own deterministic segmented scatter over the (H,E) buffer
    return gnnb_scatter(g, GNNB_DST, GNNB_SUM, dz, H, del, stream);
}

int gnnb_gat_aggregate_bwd_halo(gnnb_graph_t g, const float* Wx_own, const float* er_own, const float* dout_local,
                                const float* dout_halo, int64_t n_local, const float* el, const float* seg_max,
                                const float* seg_sum, const float* T, int64_t C, int64_t H, float slope, float* dWx,
                                float* der, float* dz, void* stream) {
    if (!g) GNNB_FAIL(GNNB_EINVAL, "graph handle is NULL");
    if (C <= 0 || H <= 0) GNNB_FAIL(GNNB_ESIZE, "C and H must be positive");
    if (n_local < 0 || n_local > g->n_src) GNNB_FAIL(GNNB_ESIZE, "n_local must be in [0, num_src]");
    if (g->n_dst == 0) return GNNB_OK;   // a rank that owns no node owns no source either: nothing to write
    if (!Wx_own || !er_own || !dWx || !der) GNNB_FAIL(GNNB_EINVAL, "NULL argument");
    if (g->E > 0 && (!el || !seg_max || !seg_sum || !T || !dz)) GNNB_FAIL(GNNB_EINVAL, "NULL argument");
    if (n_local > 0 && !dout_local) GNNB_FAIL(GNNB_EINVAL, "dout_local is NULL");
    if (n_local < g->n_src && !dout_halo) GNNB_FAIL(GNNB_EINVAL, "dout_halo is NULL but the shard has halo targets");
    const float *d, *d2;
    gat_bases(dout_local, dout_halo, n_local, g->n_src, &d, &d2);
    int vec, kk;
    if (!gat_shape(C, H, Wx_own, dWx, &vec, &kk) || ((uintptr_t)d & 15) || ((uintptr_t)d2 & 15))
        GNNB_FAIL(GNNB_EUNSUPPORTED, "fused GAT pullback: unsupported (C,H) or unaligned pointers");
    cudaStream_t st = (cudaStream_t)stream;
    GNNB_TRY(ensure_csr(g, false, st));
    const int64_t D = C * H, n_own = g->n_dst;
    if (g->E == 0) {
        gat_zero_kernel<<<nblk(n_own * D), 256, 0, st>>>(dWx, n_own * D); GNNB_LAUNCHED();
        gat_zero_kernel<<<nblk(n_own * H), 256, 0, st>>>(der, n_own * H); GNNB_LAUNCHED();
        return GNNB_OK;
    }
    return gat_backward(g, g->by_dst, Wx_own, er_own, d, d2, n_local, el, seg_max, seg_sum, T, C, H, slope, dWx, der, dz,
                        vec, kk, st);
}

int gnnb_gat_tnode(const float* dout, const float* out_fwd, int64_t n, int64_t C, int64_t H, float* T, void* stream) {
    if (C <= 0 || H <= 0 || n < 0) GNNB_FAIL(GNNB_ESIZE, "C and H must be positive, n non-negative");
    if (n == 0) return GNNB_OK;
    if (!dout || !out_fwd || !T) GNNB_FAIL(GNNB_EINVAL, "NULL argument");
    int vec, kk;
    if (!gat_shape(C, H, dout, out_fwd, &vec, &kk))
        GNNB_FAIL(GNNB_EUNSUPPORTED, "gat_tnode: unsupported (C,H) or unaligned pointers");
    return gat_tnode(dout, out_fwd, n, C, H, vec, T, (cudaStream_t)stream);
}

}  // extern "C"

namespace gnnb {

// the forward fix-up with one head (C = D): the long rows' partial slots [acc: D][M][S] combined in chunk order into
// out = acc / S, seg_max = M, seg_sum = S.  set2set.cu's attention writes its slots in this layout.
int gat_fwd_fixup_one_head(const Csr& c, int64_t E, int chunk, int64_t D, bool vec4, float* ws, float* out,
                           float* seg_max, float* seg_sum, cudaStream_t st) {
    if (c.n_long == 0) return GNNB_OK;
    GatParams p = {};
    p.rowptr = c.rowptr; p.ws = ws; p.out = out; p.stat_a = seg_max; p.stat_b = seg_sum;
    p.D = D; p.C = (int32_t)D; p.H = 1; p.E = (int32_t)E; p.nrows = c.nrows; p.chunk = chunk;
    p.nchunks = (int32_t)ceil_div(E, chunk);
    const unsigned fb = nblk((int64_t)c.n_long * (vec4 ? D / 4 : D));
    if (vec4) gat_fwd_fixup_kernel<4><<<fb, 256, 0, st>>>(p, c.long_rows, c.n_long);
    else gat_fwd_fixup_kernel<1><<<fb, 256, 0, st>>>(p, c.long_rows, c.n_long);
    GNNB_LAUNCHED();
    return GNNB_OK;
}

}  // namespace gnnb
