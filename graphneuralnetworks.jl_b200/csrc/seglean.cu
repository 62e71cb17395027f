// seglean.cu — the fused gather -> edge message -> segmented reduce for rows of 128 / 256 / 512 floats, lean edition.
//
// Same decomposition, same arithmetic in the same order as seg_reduce_kernel (segreduce.cu) — results are bit-identical
// and the long-row partial slots are numbered the same, so seg_fixup_kernel is shared — but the per-edge instruction
// stream is a quarter of it (ncu of the round-1 kernel: 64 warp instructions per edge, issue slots 68 % busy, 0.74
// no-instruction stalls per issue from a 55 KB loop body: it was bound by instruction issue, not by memory).  What moved
// out of the inner loop:
//   * the chunk decomposition (segwalk.cuh) is evaluated once per plan into a compact list of work items
//     {e_begin, e_end, slot}: an item is either a run of WHOLE rows (stored at every row end) or ONE piece of a long row
//     (one raw store into its workspace slot at the end).  The head / tail / first-flush case analysis of the old
//     flush path does not exist any more; a warp's prologue is one 16 B load instead of six dependent ones;
//   * row ends are one ballot per 32 edges; the per-row scale ct[row] (and the degree for MEAN) is fetched by the lanes
//     together with the index words, so a row store never waits on a dependent load;
//   * the index words of the next 32 edges are requested before the current 32 rows are reduced;
//   * empty rows are filled by a separate pass over rowptr, and only when the plan has any (none with self loops);
//   * the gathered-node scale can come as a per-edge stream es[e] = cs[col[e]] (plan order, built once per plan for the
//     plan-owned GCN normalisation): no dependent random 4 B gather per edge, no 4·N bytes of scales competing for L2.
// Reference semantics: NNlib.gather -> message -> NNlib.scatter (GNNlib/src/msgpass.jl:75-79,121-129,145-149).
#include "common.cuh"
#include "segwalk.cuh"
#include <cub/cub.cuh>
#include <math_constants.h>

namespace gnnb {

struct LeanParams {
    const int4* __restrict__ items;
    const int32_t* __restrict__ col;     // gathered node of each edge ([x | x2] index space)
    const int32_t* __restrict__ row;
    const int32_t* __restrict__ rowptr;
    const float* __restrict__ es;   // SMODE 1: per-edge scale stream
    const float* __restrict__ cs;   // SMODE 2: per gathered-node scale
    const float* __restrict__ w;    // per-edge weights, plan order
    const float* __restrict__ ct;   // per output-row scale or nullptr
    const float* __restrict__ x;
    const float* __restrict__ x2;   // rows of gathered nodes >= split (halo buffer)
    float* __restrict__ out;
    float* __restrict__ ws;
    int32_t n_items;
    int32_t split;
    int32_t mean;
    float sign;
    int32_t l2hint;   // SMODE 1: L2 eviction priorities of the row loads (L2_* bits), 0 = plain loads
};

namespace {

// ---- plan side: work items -------------------------------------------------------------------------------------------
// the (up to three) items of chunk k: [piece of a long row begun earlier] [whole rows] [first piece of a long row]
__device__ __forceinline__ int chunk_items(const int32_t* __restrict__ rowptr, const int32_t* __restrict__ row, int64_t k,
                                           int C, int E, int nchunks, int4 out[3]) {
    const ChunkBounds b = chunk_bounds(rowptr, row, k, C, E, nchunks);
    if (b.e_begin >= b.e_end) return 0;
    int n = 0;
    int mb = b.e_begin, me = b.e_end;
    if (b.head_partial) {
        const int r0 = __ldg(row + b.e_begin);
        const int re0 = __ldg(rowptr + r0 + 1);
        const int hb = re0 < b.e_end ? re0 : b.e_end;
        out[n++] = make_int4(b.e_begin, hb, (int)(2 * k), 0);
        mb = hb;
    }
    int4 tail = make_int4(0, 0, -1, 0);
    if (mb < b.e_end && b.tail_partial) {
        const int r1 = __ldg(row + b.e_end - 1);
        const int rs1 = __ldg(rowptr + r1);
        const int tb = rs1 > mb ? rs1 : mb;
        me = tb;
        tail = make_int4(tb, b.e_end, (int)(2 * k + 1), 0);
    }
    if (mb < me) out[n++] = make_int4(mb, me, -1, 0);
    if (tail.x < tail.y) out[n++] = tail;
    return n;
}

__global__ void item_count_kernel(const int32_t* __restrict__ rowptr, const int32_t* __restrict__ row, int C, int E,
                                  int nchunks, int32_t* __restrict__ counts) {
    const int64_t k = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (k >= nchunks) return;
    int4 tmp[3];
    counts[k] = chunk_items(rowptr, row, k, C, E, nchunks, tmp);
}
__global__ void item_emit_kernel(const int32_t* __restrict__ rowptr, const int32_t* __restrict__ row, int C, int E,
                                 int nchunks, const int32_t* __restrict__ offs, int4* __restrict__ items) {
    const int64_t k = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (k >= nchunks) return;
    int4 tmp[3];
    const int n = chunk_items(rowptr, row, k, C, E, nchunks, tmp);
    for (int i = 0; i < n; ++i) items[offs[k] + i] = tmp[i];
}

__global__ void count_empty_rows_kernel(const int32_t* __restrict__ rowptr, int32_t nrows, int32_t* __restrict__ count) {
    const int64_t r = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    const bool empty = r < nrows && rowptr[r] == rowptr[r + 1];
    const unsigned m = __ballot_sync(0xffffffffu, empty);
    if ((threadIdx.x & 31) == 0 && m) atomicAdd(count, __popc(m));
}

// one warp per 32 rows: the lanes read rowptr once, then the warp writes every empty row as whole float4 lines
__global__ void __launch_bounds__(256) fill_empty_rows_warp_kernel(const int32_t* __restrict__ rowptr, int32_t nrows,
                                                                   float* __restrict__ out, int64_t D, float v) {
    const int lane = threadIdx.x & 31;
    const int64_t r0 = ((int64_t)blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5)) * 32;
    const int64_t r = r0 + lane;
    const bool empty = r < nrows && __ldg(rowptr + r) == __ldg(rowptr + r + 1);
    unsigned m = __ballot_sync(0xffffffffu, empty);
    const float4 v4 = make_float4(v, v, v, v);
    while (m) {
        const int j = __ffs(m) - 1;
        m &= m - 1;
        float* base = out + (size_t)(r0 + j) * D;
        if ((D & 3) == 0 && (reinterpret_cast<uintptr_t>(base) & 15) == 0) {
            for (int64_t f = (int64_t)lane * 4; f < D; f += 128) *reinterpret_cast<float4*>(base + f) = v4;
        } else {
            for (int64_t f = lane; f < D; f += 32) base[f] = v;
        }
    }
}

__global__ void gather_scale_kernel(const int32_t* __restrict__ col, int64_t E, const float* __restrict__ c,
                                    float* __restrict__ es) {
    const int64_t e = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (e < E) es[e] = __ldg(c + __ldg(col + e));
}

// ---- plan side: the hot rows of the plan-owned GCN stream -------------------------------------------------------------
__global__ void count_gathers_kernel(const int32_t* __restrict__ col, int64_t E, int32_t* __restrict__ cnt) {
    const int64_t e = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (e < E) atomicAdd(cnt + __ldg(col + e), 1);
}
// es[e] = 1/sqrt(d) is >= 0 or +Inf, never NaN, so its sign bit is free: set, it marks an edge whose gathered node is hot
__global__ void flag_hot_kernel(const int32_t* __restrict__ col, int64_t E, const int32_t* __restrict__ cnt, int32_t t,
                                float* __restrict__ es) {
    const int64_t e = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (e < E && __ldg(cnt + __ldg(col + e)) >= t) es[e] = __uint_as_float(__float_as_uint(es[e]) | 0x80000000u);
}
// the hot nodes as a list (order irrelevant: it only says which rows to demote)
__global__ void list_hot_kernel(const int32_t* __restrict__ cnt, int32_t n, int32_t t, int32_t* __restrict__ rows,
                                int32_t* __restrict__ n_rows) {
    const int64_t j = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (j < n && cnt[j] >= t) rows[atomicAdd(n_rows, 1)] = (int32_t)j;
}
// after a hinted pass: every 128 B line of a hot row of x back to evict_normal, so that the evict_last priority of the
// pass does not outlive it (a line no longer in L2 is left alone)
__global__ void demote_rows_kernel(const int32_t* __restrict__ rows, int32_t n_rows, const float* __restrict__ x) {
    const int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;      // 4 lines per 512 B row
    if (i >= (int64_t)n_rows * 4) return;
    const float* line = x + (int64_t)__ldg(rows + (i >> 2)) * 128 + (i & 3) * 32;
    asm volatile("applypriority.global.L2::evict_normal [%0], 128;" :: "l"(line) : "memory");
}

// ---- the kernel ------------------------------------------------------------------------------------------------------
__device__ __forceinline__ float4 f4(float v) { return make_float4(v, v, v, v); }

// aggregation of a kernel instance
constexpr int AG_SUM = 0, AG_MEAN = 1, AG_MAX = 2;   // AG_MAX serves MIN too: min(m) = -max(-m)

// L2 eviction priorities of the SMODE-1 instances (LeanParams::l2hint): hot rows evict_last, cold rows evict_first,
// output rows evict_first
constexpr int L2_HOT_LAST = 1, L2_COLD_FIRST = 2, L2_OUT_FIRST = 4;

__device__ __forceinline__ uint64_t policy_evict_last() {
    uint64_t pol;
    asm("createpolicy.fractional.L2::evict_last.b64 %0, 1.0;" : "=l"(pol));
    return pol;
}
__device__ __forceinline__ uint64_t policy_evict_first() {
    uint64_t pol;
    asm("createpolicy.fractional.L2::evict_first.b64 %0, 1.0;" : "=l"(pol));
    return pol;
}
__device__ __forceinline__ uint64_t policy_evict_normal() {
    uint64_t pol;
    asm("createpolicy.fractional.L2::evict_normal.b64 %0, 1.0;" : "=l"(pol));
    return pol;
}
__device__ __forceinline__ float4 ldg_policy(const float* ptr, uint64_t pol) {
    float4 v;
    asm("ld.global.nc.L2::cache_hint.v4.f32 {%0, %1, %2, %3}, [%4], %5;"
        : "=f"(v.x), "=f"(v.y), "=f"(v.z), "=f"(v.w) : "l"(ptr), "l"(pol));
    return v;
}
__device__ __forceinline__ void st_policy(float* ptr, float4 v, uint64_t pol) {
    asm volatile("st.global.L2::cache_hint.v4.f32 [%0], {%1, %2, %3, %4}, %5;"
                 :: "l"(ptr), "f"(v.x), "f"(v.y), "f"(v.z), "f"(v.w), "l"(pol) : "memory");
}

// message of one edge folded into the accumulator: ((x * s1) * s2) with each product rounded, then + / max
template <int SMODE, bool HAS_W, int AGG>
__device__ __forceinline__ float lcomb1(float acc, float v, float s1, float s2, float sign) {
    float m = v;
    if (SMODE != 0) m = __fmul_rn(m, s1);
    if (HAS_W) m = __fmul_rn(m, s2);
    if (AGG == AG_MAX) return fmax_nan(acc, __fmul_rn(m, sign));  // the product with +-1 is exact
    return __fadd_rn(acc, m);
}
template <int SMODE, bool HAS_W, int AGG>
__device__ __forceinline__ float4 lcomb(float4 a, float4 v, float s1, float s2, float sign) {
    return make_float4(lcomb1<SMODE, HAS_W, AGG>(a.x, v.x, s1, s2, sign), lcomb1<SMODE, HAS_W, AGG>(a.y, v.y, s1, s2, sign),
                       lcomb1<SMODE, HAS_W, AGG>(a.z, v.z, s1, s2, sign), lcomb1<SMODE, HAS_W, AGG>(a.w, v.w, s1, s2, sign));
}

// KV float4 per lane: one warp covers a row of KV*128 floats.  SMODE 0: no gathered-node scale, 1: per-edge stream es,
// 2: gather cs[col].  HALO 0: one source base; 1: nodes >= split live in x2 (the halo rows of a shard).
// L2 policy (SMODE 1 at D = 128, the plan-owned GCN stream whose sign bits flag the hot rows): hot rows are loaded
// evict_last, cold rows evict_first, output rows stored evict_first.  On an H100 at 700 W this took the config-2 pass from
// 16.6 to 15.0 ms; evict_last alone gave 16.1 ms, so the hot set pays only beside evict_first on everything else.  The
// evict_last priority would outlive the kernel; seg_reduce_lean demotes the hot rows after each hinted pass.  (A hot
// set staged in a persisting-L2 window, which takes its set-aside from the normal L2, was measured slower on a B200.  So
// was staging every row in shared memory by TMA, one 2-D tensor-map tile load per row: on an H100 at 700 W the forward
// GCN propagate took 19.3 / 35.8 / 28.3 ms against 16.5 / 35.4 / 27.9 ms here at D = 128 / 256 / 512; DESIGN.md §4.)
// Everything that steers control flow is made warp-uniform through a vote (ballot / any), so that the
// compiler keeps the loop free of divergence handling; shuffles are never executed under a lane-dependent condition.
// The halo instances of MEAN and MAX/MIN (shards: dist_propagate, dist_sage_conv) are built for 2 CTAs per SM, which lets
// them keep their registers (for 4 they spill up to 168 bytes per thread at 512 floats, for 3 up to 60).
template <int KV, int SMODE, bool HAS_W, int HALO, int AGG>
__global__ void __launch_bounds__(256, (HALO != 0 && AGG != AG_SUM) ? 2 : 4) seg_lean_kernel(const LeanParams p) {
    constexpr unsigned FULL = 0xffffffffu;
    constexpr int U = 8 / KV;                 // row loads a warp keeps in flight (4 KB)
    constexpr int64_t STRIDE = (int64_t)KV * 128;
    const int lane = threadIdx.x & 31;
    const int item = blockIdx.x * 8 + (threadIdx.x >> 5);
    if (item >= p.n_items) return;
    const int4 it = __ldg(p.items + item);
    const int e_end = it.y;
    const bool partial = __any_sync(FULL, it.z >= 0);
    const float neutral = (AGG == AG_MAX) ? -CUDART_INF_F : 0.f;
    const float* const xl = p.x + lane * 4;
    const float* const x2l = HALO ? p.x2 + lane * 4 - (int64_t)p.split * STRIDE : nullptr;

    // index words of the 32 edges starting at e0, one edge per lane (no shuffles in here: the loads are predicated)
    auto load_lane = [&](int e0, int& c, int& r, float& s1, float& s2, bool& last) {
        const int my = e0 + lane;
        c = 0; r = 0; s1 = 1.f; s2 = 1.f; last = false;
        if (my < e_end) {
            c = __ldg(p.col + my);
            r = __ldg(p.row + my);
            if (SMODE == 1) s1 = __ldg(p.es + my);
            if (HAS_W) s2 = __ldg(p.w + my);
            last = (my + 1 == e_end) || (__ldg(p.row + my + 1) != r);
            if (SMODE == 2) s1 = __ldg(p.cs + c);
        }
    };

    float4 acc[KV];
#pragma unroll
    for (int i = 0; i < KV; ++i) acc[i] = f4(neutral);
    // the hot set is classified for rows of 128 floats, and a halo base never comes with the plan-owned stream
    constexpr bool HINTS = SMODE == 1 && KV == 1 && HALO == 0;
    uint64_t pol_hot = 0, pol_cold = 0;
    if (HINTS && p.l2hint) {
        pol_hot = (p.l2hint & L2_HOT_LAST) ? policy_evict_last() : policy_evict_normal();
        pol_cold = (p.l2hint & L2_COLD_FIRST) ? policy_evict_first() : policy_evict_normal();
    }

    int e = it.x;
    int c_n, r_n;
    float s1_n, s2_n;
    bool last_n;
    load_lane(e, c_n, r_n, s1_n, s2_n, last_n);
    bool more = true;
    while (more) {
        const int c_l = c_n, r_l = r_n;
        const float s1_l = s1_n, s2_l = s2_n;
        const unsigned vmask = __ballot_sync(FULL, e + lane < e_end);            // edges of this batch
        const unsigned bmask = partial ? 0u : __ballot_sync(FULL, last_n);       // row ends among them
        const unsigned hmask = HINTS ? __ballot_sync(FULL, __float_as_int(s1_l) < 0) : 0u;   // hot gathered rows
        float sc_l = 1.f, dg_l = 1.f;                 // scale (and edge count) of the row each lane's edge belongs to:
        if (!partial && e + lane < e_end) {           // needed at the first row end, long after these loads went out
            if (p.ct) sc_l = __ldg(p.ct + r_l);
            if (AGG == AG_MEAN) dg_l = (float)(__ldg(p.rowptr + r_l + 1) - __ldg(p.rowptr + r_l));
        }
        if (AGG == AG_MAX) sc_l *= p.sign;
        more = __any_sync(FULL, e + 32 < e_end);
        if (more) load_lane(e + 32, c_n, r_n, s1_n, s2_n, last_n);               // in flight while this batch is reduced
#pragma unroll 1
        for (int j0 = 0; j0 < 32 && (vmask >> j0) != 0u; j0 += U) {
            float4 v[U][KV];
#pragma unroll
            for (int u = 0; u < U; ++u) {
                const int cj = __shfl_sync(FULL, c_l, j0 + u);
                const bool second = HALO != 0 && cj >= p.split;
                const float* xr = (second ? x2l : xl) + (int64_t)cj * STRIDE;
                if ((vmask >> (j0 + u)) & 1u) {
                    if (HINTS && p.l2hint) {
                        const uint64_t pol = ((hmask >> (j0 + u)) & 1u) ? pol_hot : pol_cold;
#pragma unroll
                        for (int i = 0; i < KV; ++i) v[u][i] = ldg_policy(xr + i * 128, pol);
                    } else {
#pragma unroll
                        for (int i = 0; i < KV; ++i) v[u][i] = __ldg(reinterpret_cast<const float4*>(xr + i * 128));
                    }
                }
            }
#pragma unroll
            for (int u = 0; u < U; ++u) {
                // SMODE 1: the sign bit of es marks a hot row; the scale is the value without it (an exact AND)
                const float s1 = SMODE == 1 ? __int_as_float(__shfl_sync(FULL, __float_as_int(s1_l), j0 + u) & 0x7fffffff)
                                            : (SMODE != 0) ? __shfl_sync(FULL, s1_l, j0 + u) : 1.f;
                const float s2 = HAS_W ? __shfl_sync(FULL, s2_l, j0 + u) : 1.f;
                if ((vmask >> (j0 + u)) & 1u) {
#pragma unroll
                    for (int i = 0; i < KV; ++i) acc[i] = lcomb<SMODE, HAS_W, AGG>(acc[i], v[u][i], s1, s2, p.sign);
                }
                if ((bmask >> (j0 + u)) & 1u) {            // row end: scale and store, exactly once
                    const int rj = __shfl_sync(FULL, r_l, j0 + u);
                    const float sc = __shfl_sync(FULL, sc_l, j0 + u);
                    float* o = p.out + (int64_t)rj * STRIDE + lane * 4;
                    if (AGG == AG_MEAN) {
                        const float dg = __shfl_sync(FULL, dg_l, j0 + u);
#pragma unroll
                        for (int i = 0; i < KV; ++i)
                            acc[i] = make_float4(__fdiv_rn(acc[i].x, dg), __fdiv_rn(acc[i].y, dg),
                                                 __fdiv_rn(acc[i].z, dg), __fdiv_rn(acc[i].w, dg));
                    }
#pragma unroll
                    for (int i = 0; i < KV; ++i) {
                        const float4 res = make_float4(acc[i].x * sc, acc[i].y * sc, acc[i].z * sc, acc[i].w * sc);
                        if (HINTS && (p.l2hint & L2_OUT_FIRST)) st_policy(o + i * 128, res, policy_evict_first());
                        else *reinterpret_cast<float4*>(o + i * 128) = res;
                        acc[i] = f4(neutral);
                    }
                }
            }
        }
        e += 32;
    }
    if (partial) {
        float* o = p.ws + (int64_t)it.z * STRIDE + lane * 4;
#pragma unroll
        for (int i = 0; i < KV; ++i) *reinterpret_cast<float4*>(o + i * 128) = acc[i];
    }
}

// ---- pullback of max / min aggregation on the work-item list of the by-source plan -----------------------------------------
//   dx[j,:] = sum over out-edges e = (j -> t) of w_e * dout[t,:] .* (x[j,:] * w_e == out_fwd[t,:])      (NNlib's rule: every
// tied extremum receives the gradient).  Two gathered rows per edge (out_fwd[t], dout[t]) plus the source's own row (an L1
// hit after its first edge).  The kernel this replaces walked a source's out-edges with ONE warp, serially: a 1 M-edge RMAT
// hub took 67 ms at N = 2 M / E = 20 M (ncu: 117 GB/s).  Here a hub is cut into 128-edge pieces like every long row.
struct MaxBwdParams {
    const int4* __restrict__ items;
    const int32_t* __restrict__ col;
    const int32_t* __restrict__ row;
    const float* __restrict__ w;
    const float* __restrict__ x;
    const float* __restrict__ dout;
    const float* __restrict__ of;
    float* __restrict__ dx;
    float* __restrict__ ws;
    int32_t n_items;
    // HALO 1 (the forward CSR of a backward shard plan): targets >= split read dout2 / of2 + (t - split)*D
    int32_t split;
    const float* __restrict__ dout2;
    const float* __restrict__ of2;
};

template <int KV, bool HAS_W, int HALO>
__global__ void __launch_bounds__(256, 2) maxmin_bwd_lean_kernel(const MaxBwdParams p) {
    constexpr unsigned FULL = 0xffffffffu;
    constexpr int U = KV == 1 ? 4 : (KV == 2 ? 2 : 1);      // edges in flight per warp (three rows each)
    constexpr int64_t STRIDE = (int64_t)KV * 128;
    const int lane = threadIdx.x & 31;
    const int item = blockIdx.x * 8 + (threadIdx.x >> 5);
    if (item >= p.n_items) return;
    const int4 it = __ldg(p.items + item);
    const int e_end = it.y;
    const bool partial = __any_sync(FULL, it.z >= 0);

    auto load_lane = [&](int e0, int& c, int& r, float& wv, bool& last) {
        const int my = e0 + lane;
        c = 0; r = 0; wv = 1.f; last = false;
        if (my < e_end) {
            c = __ldg(p.col + my);
            r = __ldg(p.row + my);
            if (HAS_W) wv = __ldg(p.w + my);
            last = (my + 1 == e_end) || (__ldg(p.row + my + 1) != r);
        }
    };
    float4 acc[KV];
#pragma unroll
    for (int i = 0; i < KV; ++i) acc[i] = f4(0.f);
    int e = it.x;
    int c_n, r_n;
    float w_n;
    bool last_n;
    load_lane(e, c_n, r_n, w_n, last_n);
    bool more = true;
    while (more) {
        const int c_l = c_n, r_l = r_n;
        const float w_l = w_n;
        const unsigned vmask = __ballot_sync(FULL, e + lane < e_end);
        const unsigned bmask = partial ? 0u : __ballot_sync(FULL, last_n);
        more = __any_sync(FULL, e + 32 < e_end);
        if (more) load_lane(e + 32, c_n, r_n, w_n, last_n);
#pragma unroll 1
        for (int j0 = 0; j0 < 32 && (vmask >> j0) != 0u; j0 += U) {
            float4 vo[U][KV], vd[U][KV], vx[U][KV];
#pragma unroll
            for (int u = 0; u < U; ++u) {
                const int cj = __shfl_sync(FULL, c_l, j0 + u);
                const int rj = __shfl_sync(FULL, r_l, j0 + u);
                if ((vmask >> (j0 + u)) & 1u) {
                    const bool second = HALO != 0 && cj >= p.split;
                    const int64_t to = (int64_t)(second ? cj - p.split : cj) * STRIDE + lane * 4,
                                  xo = (int64_t)rj * STRIDE + lane * 4;
                    const float* const of = second ? p.of2 : p.of;
                    const float* const dout = second ? p.dout2 : p.dout;
#pragma unroll
                    for (int i = 0; i < KV; ++i) {
                        vo[u][i] = __ldg(reinterpret_cast<const float4*>(of + to + i * 128));
                        vd[u][i] = __ldg(reinterpret_cast<const float4*>(dout + to + i * 128));
                        vx[u][i] = __ldg(reinterpret_cast<const float4*>(p.x + xo + i * 128));
                    }
                }
            }
#pragma unroll
            for (int u = 0; u < U; ++u) {
                const float wv = HAS_W ? __shfl_sync(FULL, w_l, j0 + u) : 1.f;
                if ((vmask >> (j0 + u)) & 1u) {
#pragma unroll
                    for (int i = 0; i < KV; ++i) {
                        if (__fmul_rn(vx[u][i].x, wv) == vo[u][i].x) acc[i].x += wv * vd[u][i].x;
                        if (__fmul_rn(vx[u][i].y, wv) == vo[u][i].y) acc[i].y += wv * vd[u][i].y;
                        if (__fmul_rn(vx[u][i].z, wv) == vo[u][i].z) acc[i].z += wv * vd[u][i].z;
                        if (__fmul_rn(vx[u][i].w, wv) == vo[u][i].w) acc[i].w += wv * vd[u][i].w;
                    }
                }
                if ((bmask >> (j0 + u)) & 1u) {
                    const int rj = __shfl_sync(FULL, r_l, j0 + u);
                    float* o = p.dx + (int64_t)rj * STRIDE + lane * 4;
#pragma unroll
                    for (int i = 0; i < KV; ++i) {
                        *reinterpret_cast<float4*>(o + i * 128) = acc[i];
                        acc[i] = f4(0.f);
                    }
                }
            }
        }
        e += 32;
    }
    if (partial) {
        float* o = p.ws + (int64_t)it.z * STRIDE + lane * 4;
#pragma unroll
        for (int i = 0; i < KV; ++i) *reinterpret_cast<float4*>(o + i * 128) = acc[i];
    }
}

template <int KV, int SMODE, bool HAS_W, int HALO, int AGG>
int launch_lean3(const LeanParams& p, cudaStream_t st) {
    const unsigned blocks = (unsigned)ceil_div(p.n_items, 8);
    seg_lean_kernel<KV, SMODE, HAS_W, HALO, AGG><<<blocks, 256, 0, st>>>(p);
    GNNB_LAUNCHED();
    return GNNB_OK;
}
// instances: SUM with every scale source, with and without a halo base; MEAN and MAX/MIN for the plain messages
// (copy_xj, w_mul_xj), with and without a halo base — the shapes the layers use; anything else stays with
// seg_reduce_kernel
template <int KV>
int launch_lean1(const LeanParams& p, int smode, bool has_w, int halo, int agg, cudaStream_t st) {
#define GNNB_LEAN(S, W, H, A) if (smode == S && has_w == W && halo == H && agg == A) return launch_lean3<KV, S, W, H, A>(p, st);
    GNNB_LEAN(0, false, 0, AG_SUM) GNNB_LEAN(0, true, 0, AG_SUM) GNNB_LEAN(1, false, 0, AG_SUM)
    GNNB_LEAN(1, true, 0, AG_SUM) GNNB_LEAN(2, false, 0, AG_SUM) GNNB_LEAN(2, true, 0, AG_SUM)
    GNNB_LEAN(0, false, 1, AG_SUM) GNNB_LEAN(0, true, 1, AG_SUM) GNNB_LEAN(1, false, 1, AG_SUM)
    GNNB_LEAN(1, true, 1, AG_SUM) GNNB_LEAN(2, false, 1, AG_SUM) GNNB_LEAN(2, true, 1, AG_SUM)
    GNNB_LEAN(0, false, 0, AG_MEAN) GNNB_LEAN(0, true, 0, AG_MEAN)
    GNNB_LEAN(0, false, 0, AG_MAX) GNNB_LEAN(0, true, 0, AG_MAX)
    GNNB_LEAN(0, false, 1, AG_MEAN) GNNB_LEAN(0, true, 1, AG_MEAN)
    GNNB_LEAN(0, false, 1, AG_MAX) GNNB_LEAN(0, true, 1, AG_MAX)
#undef GNNB_LEAN
    return GNNB_EUNSUPPORTED;
}

}  // namespace

// ---- plan side, host --------------------------------------------------------------------------------------------------
int ensure_items(gnnb_graph* g, const Csr& c, cudaStream_t st) {
    Csr& mc = const_cast<Csr&>(c);          // c is g->by_dst or g->by_src, both owned (mutably) by the plan
    if (mc.items != nullptr || g->E == 0) return GNNB_OK;
    std::lock_guard<std::mutex> lock(g->mu);
    if (mc.items != nullptr) return GNNB_OK;
    const int32_t nchunks = (int32_t)ceil_div(g->E, g->chunk);
    DeviceScratch sc;
    int32_t *counts = nullptr, *offs = nullptr, *d_empty = nullptr;
    void* tmp = nullptr;
    int4* items = nullptr;
    GNNB_TRY(sc.alloc(&counts, (size_t)nchunks + 1));
    GNNB_TRY(sc.alloc(&offs, (size_t)nchunks + 1));
    GNNB_TRY(sc.alloc(&d_empty, 1));
    GNNB_CUDA(cudaMemsetAsync(counts, 0, sizeof(int32_t) * ((size_t)nchunks + 1), st));
    GNNB_CUDA(cudaMemsetAsync(d_empty, 0, sizeof(int32_t), st));
    item_count_kernel<<<(unsigned)ceil_div(nchunks, 256), 256, 0, st>>>(c.rowptr, c.row, g->chunk, (int)g->E, nchunks, counts);
    size_t tmp_bytes = 0;
    GNNB_CUDA(cub::DeviceScan::ExclusiveSum(nullptr, tmp_bytes, counts, offs, nchunks + 1, st));
    GNNB_TRY(sc.alloc(&tmp, tmp_bytes ? tmp_bytes : 1));
    GNNB_CUDA(cub::DeviceScan::ExclusiveSum(tmp, tmp_bytes, counts, offs, nchunks + 1, st));
    count_empty_rows_kernel<<<(unsigned)ceil_div((int64_t)c.nrows, 256), 256, 0, st>>>(c.rowptr, c.nrows, d_empty);
    int32_t n_items = 0, n_empty = 0;
    GNNB_CUDA(cudaMemcpyAsync(&n_items, offs + nchunks, sizeof(int32_t), cudaMemcpyDeviceToHost, st));
    GNNB_CUDA(cudaMemcpyAsync(&n_empty, d_empty, sizeof(int32_t), cudaMemcpyDeviceToHost, st));
    GNNB_CUDA(cudaStreamSynchronize(st));
    GNNB_TRY(sc.alloc(&items, (size_t)(n_items > 0 ? n_items : 1)));
    item_emit_kernel<<<(unsigned)ceil_div(nchunks, 256), 256, 0, st>>>(c.rowptr, c.row, g->chunk, (int)g->E, nchunks, offs, items);
    GNNB_CUDA(cudaGetLastError());
    GNNB_CUDA(cudaStreamSynchronize(st));
    g_launches.fetch_add(4, std::memory_order_relaxed);
    mc.n_items = n_items;
    mc.n_empty = n_empty;
    mc.items = reinterpret_cast<int32_t*>(sc.release(items));
    return GNNB_OK;
}

bool g_l2_policy_forced = false;   // gnnb_set_kernel_variant(14): the L2 policy at every size

// L2 policy of the fused GCN propagate (DESIGN.md §4 "L2 policy").  The hot set of a direction: the nodes gathered at
// least t times, t the smallest count whose nodes fit kHotL2Fraction of the L2 as rows of 128 floats.  The policy runs
// at D = 128 when the gathered rows are at least kL2PolicyMinRatio times the L2: when they nearly fit, plain loads
// already hit.  Wider rows keep plain loads (their hot set would pin 2 or 4 times the bytes).  A hinted pass is followed
// by demote_rows_kernel over the plan's hot nodes, so that no line keeps the evict_last priority once the pass is done.
constexpr double kHotL2Fraction = 0.56;
constexpr int64_t kL2PolicyMinRatio = 8;
constexpr int kL2Hints = L2_HOT_LAST | L2_COLD_FIRST | L2_OUT_FIRST;

static int l2_bytes(const gnnb_graph* g, int64_t* bytes) {
    int v = 0;
    GNNB_CUDA(cudaDeviceGetAttribute(&v, cudaDevAttrL2CacheSize, g->device));
    *bytes = v;
    return GNNB_OK;
}

// count the gathers of each of the n gathered nodes of c, choose t, flag the hot edges in es (plan order of c); the list
// of hot nodes is allocated in the caller's `keep`
static int flag_hot_rows(gnnb_graph* g, Csr& c, int32_t n, float* es, DeviceScratch& keep, int32_t* t_out,
                         int32_t** rows_out, int32_t* n_rows_out, cudaStream_t st) {
    int64_t l2 = 0;
    GNNB_TRY(l2_bytes(g, &l2));
    int64_t budget = (int64_t)((double)l2 * kHotL2Fraction) / 512;           // rows of 128 floats
    DeviceScratch sc;
    int32_t *cnt = nullptr, *sorted = nullptr, *rows = nullptr, *d_nrows = nullptr;
    void* tmp = nullptr;
    GNNB_TRY(sc.alloc(&cnt, (size_t)n));
    GNNB_CUDA(cudaMemsetAsync(cnt, 0, sizeof(int32_t) * (size_t)n, st));
    count_gathers_kernel<<<(unsigned)ceil_div(g->E, 256), 256, 0, st>>>(c.col, g->E, cnt);
    GNNB_CUDA(cudaGetLastError());
    int32_t t = 1;                          // every gathered node fits
    if (n > budget) {                       // t = (budget+1)-th largest count + 1: at most `budget` nodes reach it
        size_t tmp_bytes = 0;
        GNNB_TRY(sc.alloc(&sorted, (size_t)n));
        GNNB_CUDA(cub::DeviceRadixSort::SortKeysDescending(nullptr, tmp_bytes, cnt, sorted, n, 0, 32, st));
        GNNB_TRY(sc.alloc(&tmp, tmp_bytes ? tmp_bytes : 1));
        GNNB_CUDA(cub::DeviceRadixSort::SortKeysDescending(tmp, tmp_bytes, cnt, sorted, n, 0, 32, st));
        int32_t kth = 0;
        GNNB_CUDA(cudaMemcpyAsync(&kth, sorted + budget, sizeof(int32_t), cudaMemcpyDeviceToHost, st));
        GNNB_CUDA(cudaStreamSynchronize(st));
        t = kth + 1;
    }
    flag_hot_kernel<<<(unsigned)ceil_div(g->E, 256), 256, 0, st>>>(c.col, g->E, cnt, t, es);
    GNNB_CUDA(cudaGetLastError());
    GNNB_TRY(keep.alloc(&rows, (size_t)(n < budget ? n : budget)));
    GNNB_TRY(sc.alloc(&d_nrows, 1));
    GNNB_CUDA(cudaMemsetAsync(d_nrows, 0, sizeof(int32_t), st));
    list_hot_kernel<<<(unsigned)ceil_div(n, 256), 256, 0, st>>>(cnt, n, t, rows, d_nrows);
    GNNB_CUDA(cudaGetLastError());
    int32_t n_rows = 0;
    GNNB_CUDA(cudaMemcpyAsync(&n_rows, d_nrows, sizeof(int32_t), cudaMemcpyDeviceToHost, st));
    GNNB_CUDA(cudaStreamSynchronize(st));
    g_launches.fetch_add(n > budget ? 4 : 3, std::memory_order_relaxed);
    *t_out = t;
    *rows_out = rows;
    *n_rows_out = n_rows;
    return GNNB_OK;
}

// g->gcn_c = 1/sqrt(in-degree) (IEEE-exact, as gnnb_gcn_norm) and, for one direction, es[e] = gcn_c[col[e]] with the
// hot edges flagged in the sign bit
int ensure_gcn_scale(gnnb_graph* g, bool transposed, cudaStream_t st) {
    Csr& c = transposed ? g->by_src : g->by_dst;
    if (g->gcn_c != nullptr && (c.es != nullptr || g->E == 0)) return GNNB_OK;
    DeviceScratch sc;   // what another thread's call installed first is freed here
    if (g->gcn_c == nullptr) {
        float* buf = nullptr;
        GNNB_TRY(sc.alloc(&buf, (size_t)(g->n_dst > 0 ? g->n_dst : 1)));
        GNNB_TRY(gnnb_gcn_norm(g, nullptr, buf, st));
        GNNB_CUDA(cudaStreamSynchronize(st));
        std::lock_guard<std::mutex> lock(g->mu);
        if (g->gcn_c == nullptr) g->gcn_c = sc.release(buf);
    }
    if (c.es == nullptr && g->E > 0) {
        float* es = nullptr;
        GNNB_TRY(sc.alloc(&es, (size_t)g->E));
        gather_scale_kernel<<<(unsigned)ceil_div(g->E, 256), 256, 0, st>>>(c.col, g->E, g->gcn_c, es);
        GNNB_LAUNCHED();
        int32_t t = 0, n_hot = 0;
        int32_t* hot = nullptr;
        GNNB_TRY(flag_hot_rows(g, c, transposed ? g->n_dst : g->n_src, es, sc, &t, &hot, &n_hot, st));
        std::lock_guard<std::mutex> lock(g->mu);
        if (c.es == nullptr) { c.es = sc.release(es); c.hot_min = t; c.hot_rows = sc.release(hot); c.n_hot = n_hot; }
    }
    return GNNB_OK;
}

// the hot set of one direction, for inspection: threshold, size and (up to `capacity`) the nodes, unordered, to host
int gcn_hot_rows(gnnb_graph* g, bool transposed, int32_t* rows_host, int64_t capacity, int64_t* num_rows,
                 int32_t* threshold, cudaStream_t st) {
    GNNB_TRY(ensure_csr(g, transposed, st));
    GNNB_TRY(ensure_gcn_scale(g, transposed, st));
    const Csr& c = transposed ? g->by_src : g->by_dst;
    if (num_rows) *num_rows = c.n_hot;
    if (threshold) *threshold = c.hot_min;
    const int64_t n = capacity < c.n_hot ? capacity : c.n_hot;
    if (rows_host && n > 0) GNNB_CUDA(cudaMemcpy(rows_host, c.hot_rows, sizeof(int32_t) * (size_t)n, cudaMemcpyDeviceToHost));
    return GNNB_OK;
}

// the two-sided scales of a relation (heterograph gcn_conv, conv.jl:45-50): c_src = 1/sqrt(out-degree), c_dst =
// 1/sqrt(in-degree), both IEEE-exact as gnnb_gcn_norm, and for one direction the per-edge stream of the gathered side's
// scale: forward (by_dst) es[e] = c_src[col[e]], pullback (by_src) es[e] = c_dst[col[e]]
int ensure_bipartite_gcn_scale(gnnb_graph* g, bool transposed, cudaStream_t st) {
    float*& es_slot = transposed ? g->bip_es_src : g->bip_es_dst;
    if (g->bip_c_src != nullptr && g->bip_c_dst != nullptr && (es_slot != nullptr || g->E == 0)) return GNNB_OK;
    GNNB_TRY(ensure_csr(g, true, st));                   // out-degrees come from the by-source rowptr
    DeviceScratch sc;   // what another thread's call installed first is freed here
    if (g->bip_c_src == nullptr || g->bip_c_dst == nullptr) {
        float *cs = nullptr, *cd = nullptr;
        GNNB_TRY(sc.alloc(&cs, (size_t)(g->n_src > 0 ? g->n_src : 1)));
        GNNB_TRY(sc.alloc(&cd, (size_t)(g->n_dst > 0 ? g->n_dst : 1)));
        GNNB_TRY(gnnb_degree(g, GNNB_DIR_OUT, nullptr, cs, st));
        GNNB_TRY(gnnb_degree(g, GNNB_DIR_IN, nullptr, cd, st));
        GNNB_TRY(rsqrt_exact(cs, g->n_src, st));
        GNNB_TRY(rsqrt_exact(cd, g->n_dst, st));
        GNNB_CUDA(cudaStreamSynchronize(st));
        std::lock_guard<std::mutex> lock(g->mu);
        if (g->bip_c_src == nullptr) { g->bip_c_src = sc.release(cs); g->bip_c_dst = sc.release(cd); }
    }
    if (es_slot == nullptr && g->E > 0) {
        const Csr& c = transposed ? g->by_src : g->by_dst;
        float* es = nullptr;
        GNNB_TRY(sc.alloc(&es, (size_t)g->E));
        gather_scale_kernel<<<(unsigned)ceil_div(g->E, 256), 256, 0, st>>>(c.col, g->E, transposed ? g->bip_c_dst : g->bip_c_src, es);
        GNNB_LAUNCHED();
        GNNB_CUDA(cudaStreamSynchronize(st));
        std::lock_guard<std::mutex> lock(g->mu);
        if (es_slot == nullptr) es_slot = sc.release(es);
    }
    return GNNB_OK;
}

// the lean path: D in {128, 256, 512}, 16 B-aligned operands.  GNNB_EUNSUPPORTED = not this kernel's shape (the caller
// falls back to seg_reduce_kernel).
int seg_reduce_lean(gnnb_graph* g, const Csr& c, const SegArgs& a, float* ws, cudaStream_t st) {
    if (a.D != 128 && a.D != 256 && a.D != 512) return GNNB_EUNSUPPORTED;
    if ((reinterpret_cast<uintptr_t>(a.x) & 15) || (reinterpret_cast<uintptr_t>(a.x2) & 15) ||
        (reinterpret_cast<uintptr_t>(a.out) & 15))
        return GNNB_EUNSUPPORTED;
    const bool ismax = (a.aggr == GNNB_MAX || a.aggr == GNNB_MIN);
    const int agg = ismax ? AG_MAX : (a.aggr == GNNB_MEAN ? AG_MEAN : AG_SUM);
    const int smode = (a.cs == nullptr) ? 0 : (a.es != nullptr ? 1 : 2);
    const bool halo = a.x2 != nullptr;
    if (agg != AG_SUM && smode != 0) return GNNB_EUNSUPPORTED;
    GNNB_TRY(ensure_items(g, c, st));
    if (c.n_empty > 0) {
        const float v = a.aggr == GNNB_MAX ? -HUGE_VALF : (a.aggr == GNNB_MIN ? HUGE_VALF : 0.f);
        fill_empty_rows_warp_kernel<<<(unsigned)ceil_div((int64_t)c.nrows, 256), 256, 0, st>>>(c.rowptr, c.nrows, a.out, a.D, v);
        GNNB_LAUNCHED();
    }
    LeanParams p;
    p.items = reinterpret_cast<const int4*>(c.items);
    p.n_items = c.n_items;
    p.col = c.col; p.row = c.row; p.rowptr = c.rowptr;
    p.es = a.es; p.cs = a.cs; p.w = a.w; p.ct = a.ct;
    p.x = a.x; p.x2 = a.x2; p.split = a.split; p.out = a.out; p.ws = ws;
    p.mean = (a.aggr == GNNB_MEAN);
    p.sign = (a.aggr == GNNB_MIN) ? -1.f : 1.f;
    p.l2hint = 0;
    if (smode == 1 && a.es == c.es && c.hot_min > 0 && a.D == 128 && !halo) {   // the plan-owned GCN stream, flagged
        int64_t l2 = 0;
        GNNB_TRY(l2_bytes(g, &l2));
        if (g_l2_policy_forced || (int64_t)g->n_src * a.D * 4 >= kL2PolicyMinRatio * l2) p.l2hint = kL2Hints;
    }
    if (p.n_items == 0) return GNNB_OK;
    const int use_halo = halo ? 1 : 0;
    int rc;
    if (a.D == 128) rc = launch_lean1<1>(p, smode, a.w != nullptr, use_halo, agg, st);
    else if (a.D == 256) rc = launch_lean1<2>(p, smode, a.w != nullptr, use_halo, agg, st);
    else rc = launch_lean1<4>(p, smode, a.w != nullptr, use_halo, agg, st);
    if (rc == GNNB_OK && (p.l2hint & L2_HOT_LAST) && c.n_hot > 0) {        // the evict_last priority ends with the pass
        demote_rows_kernel<<<(unsigned)ceil_div((int64_t)c.n_hot * 4, 256), 256, 0, st>>>(c.hot_rows, c.n_hot, a.x);
        GNNB_LAUNCHED();
    }
    return rc;
}

// max / min pullback through the work items of `c`, whose rows are the sources j and whose gathered nodes the targets t:
// the by-source plan of a graph, or the forward CSR of a backward shard plan with the targets >= split read from dout2 /
// of2 (halo = true); GNNB_EUNSUPPORTED = not this kernel's shape
int seg_fixup_sum(const Csr& c, int64_t E, int chunk, int64_t D, float* ws, float* out, cudaStream_t st);   // segreduce.cu
int maxmin_bwd_lean(gnnb_graph* g, const Csr& c, const float* w_plan, const float* x, const float* dout,
                    const float* out_fwd, bool halo, const float* dout2, const float* of2, int32_t split, int64_t D,
                    float* dx, cudaStream_t st) {
    if (D != 128 && D != 256 && D != 512) return GNNB_EUNSUPPORTED;
    if ((reinterpret_cast<uintptr_t>(x) & 15) || (reinterpret_cast<uintptr_t>(dout) & 15) ||
        (reinterpret_cast<uintptr_t>(out_fwd) & 15) || (reinterpret_cast<uintptr_t>(dx) & 15) ||
        (reinterpret_cast<uintptr_t>(dout2) & 15) || (reinterpret_cast<uintptr_t>(of2) & 15))
        return GNNB_EUNSUPPORTED;
    if (g->E == 0) return GNNB_EUNSUPPORTED;
    GNNB_TRY(ensure_items(g, c, st));
    if (c.n_empty > 0) {
        fill_empty_rows_warp_kernel<<<(unsigned)ceil_div((int64_t)c.nrows, 256), 256, 0, st>>>(c.rowptr, c.nrows, dx, D, 0.f);
        GNNB_LAUNCHED();
    }
    MaxBwdParams p;
    p.items = reinterpret_cast<const int4*>(c.items);
    p.n_items = c.n_items;
    p.col = c.col; p.row = c.row; p.w = w_plan; p.x = x; p.dout = dout; p.of = out_fwd; p.dx = dx; p.ws = nullptr;
    p.split = split; p.dout2 = dout2; p.of2 = of2;
    if (c.n_long > 0) {
        GNNB_TRY(grow_buffer(&g->ws, &g->ws_bytes, (size_t)2 * ceil_div(g->E, g->chunk) * D * sizeof(float)));
        p.ws = g->ws;
    }
    if (p.n_items > 0) {
        const unsigned blocks = (unsigned)ceil_div(p.n_items, 8);
        const bool hw = w_plan != nullptr;
#define GNNB_MAXBWD(KV, H) \
        { if (hw) maxmin_bwd_lean_kernel<KV, true, H><<<blocks, 256, 0, st>>>(p); else maxmin_bwd_lean_kernel<KV, false, H><<<blocks, 256, 0, st>>>(p); }
        if (halo) {
            if (D == 128) GNNB_MAXBWD(1, 1) else if (D == 256) GNNB_MAXBWD(2, 1) else GNNB_MAXBWD(4, 1)
        } else {
            if (D == 128) GNNB_MAXBWD(1, 0) else if (D == 256) GNNB_MAXBWD(2, 0) else GNNB_MAXBWD(4, 0)
        }
#undef GNNB_MAXBWD
        GNNB_LAUNCHED();
    }
    if (c.n_long > 0) GNNB_TRY(seg_fixup_sum(c, g->E, g->chunk, D, p.ws, dx, st));
    return GNNB_OK;
}

}  // namespace gnnb
