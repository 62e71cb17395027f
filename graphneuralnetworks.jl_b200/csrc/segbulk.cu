// segbulk.cu — the TMA-staged variant of the fused gather -> message -> segmented-reduce kernel.
//
// Same decomposition and arithmetic as segreduce.cu (chunks of C CSR-sorted edges, one warp per chunk, rows
// reduced in COO order, long rows through partial slots + fix-up), but the gathered feature rows do not travel
// through registers: every lane issues ONE `cp.async.bulk` (1-D TMA bulk copy, SASS UBLKCP) that moves the whole
// D*4-byte row of its edge from HBM/L2 into the warp's shared-memory ring, completion is tracked by an mbarrier
// per stage (complete_tx::bytes), and the warp consumes a stage of 32 rows with conflict-free LDS.128 while the
// next stages are in flight.  Bytes in flight per SM are bounded by shared memory (~190 KB) instead of by the
// register file, which bounds the register-staged kernel; here an edge costs one LDS.128 + 8 FP32 ops + a ballot-mask
// test.
//
// Used for fp32 rows of 128, 256, 384 or 512 floats (the configurations of BASELINE.json); everything else takes
// the register-staged kernel.  Results are bit-identical to it (same order of additions).
#include "common.cuh"
#include "segwalk.cuh"
#include <math_constants.h>

namespace gnnb {

struct BulkParams {
    const int32_t* __restrict__ rowptr;
    const int32_t* __restrict__ col;
    const int32_t* __restrict__ row;
    const float* __restrict__ x;
    const float* __restrict__ x2;
    const float* __restrict__ w;
    const float* __restrict__ cs;
    const float* __restrict__ ct;
    float* __restrict__ out;
    float* __restrict__ ws;
    int64_t D;
    int32_t E, nrows, chunk, nchunks, mean, fill, split;
    float sign;
};

__device__ __forceinline__ uint32_t smem_u32(const void* p) { return (uint32_t)__cvta_generic_to_shared(p); }
__device__ __forceinline__ void mbar_init(uint32_t bar, uint32_t count) {
    asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(bar), "r"(count) : "memory");
}
__device__ __forceinline__ void mbar_expect_tx(uint32_t bar, uint32_t bytes) {
    asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(bar), "r"(bytes) : "memory");
}
__device__ __forceinline__ bool mbar_try_wait(uint32_t bar, uint32_t parity) {
    uint32_t ok;
    asm volatile(
        "{\n\t.reg .pred p;\n\t"
        "mbarrier.try_wait.parity.shared::cta.b64 p, [%1], %2;\n\t"
        "selp.u32 %0, 1, 0, p;\n\t}"
        : "=r"(ok)
        : "r"(bar), "r"(parity)
        : "memory");
    return ok != 0;
}
__device__ __forceinline__ void bulk_g2s(uint32_t dst, const void* src, uint32_t bytes, uint32_t bar) {
    asm volatile("cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];" ::"r"(dst),
                 "l"(src), "r"(bytes), "r"(bar)
                 : "memory");
}
__device__ __forceinline__ void fence_proxy_async() { asm volatile("fence.proxy.async.shared::cta;" ::: "memory"); }
__device__ __forceinline__ void fence_mbar_init() { asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory"); }

template <bool ISMAX> __device__ __forceinline__ float bcomb1(float acc, float v, float s) {
    const float m = __fmul_rn(v, s);
    if (ISMAX) return fmaxf(acc, m);
    return __fadd_rn(acc, m);
}
template <bool ISMAX> __device__ __forceinline__ float4 bcomb(float4 a, float4 v, float s) {
    return make_float4(bcomb1<ISMAX>(a.x, v.x, s), bcomb1<ISMAX>(a.y, v.y, s), bcomb1<ISMAX>(a.z, v.z, s),
                       bcomb1<ISMAX>(a.w, v.w, s));
}
__device__ __forceinline__ float4 bfinish(float4 acc, const BulkParams& p, int r) {
    if (p.mean) {
        const int deg = __ldg(p.rowptr + r + 1) - __ldg(p.rowptr + r);
        const float d = (float)(deg > 0 ? deg : 1);
        acc = make_float4(__fdiv_rn(acc.x, d), __fdiv_rn(acc.y, d), __fdiv_rn(acc.z, d), __fdiv_rn(acc.w, d));
    }
    if (p.ct) { const float c = __ldg(p.ct + r); acc = make_float4(acc.x * c, acc.y * c, acc.z * c, acc.w * c); }
    if (p.sign < 0.f) acc = make_float4(-acc.x, -acc.y, -acc.z, -acc.w);
    return acc;
}

// K = D/128 float4 slices per lane; S ring stages of 32 rows; WARPS warps per CTA
template <int K, int S, int WARPS, bool ISMAX>
__global__ void __launch_bounds__(32 * WARPS) seg_reduce_bulk_kernel(const BulkParams p) {
    extern __shared__ __align__(128) unsigned char smem_raw[];
    constexpr unsigned FULL = 0xffffffffu;
    constexpr int RB = K * 512;                       // bytes per feature row
    constexpr int STAGE_BYTES = 32 * RB;
    constexpr int WARP_BYTES = (S * STAGE_BYTES + S * 32 * 8 + S * 8 + 127) & ~127;   // keep every ring 128 B aligned
    const int lane = threadIdx.x & 31;
    const int wid = threadIdx.x >> 5;
    const int64_t k = (int64_t)blockIdx.x * WARPS + wid;   // chunk id
    unsigned char* wbase = smem_raw + (size_t)wid * WARP_BYTES;
    float* sm_rows = reinterpret_cast<float*>(wbase);
    int32_t* sm_d = reinterpret_cast<int32_t*>(wbase + S * STAGE_BYTES);
    float* sm_s = reinterpret_cast<float*>(wbase + S * STAGE_BYTES + S * 32 * 4);
    const uint32_t bar0 = smem_u32(wbase + S * STAGE_BYTES + S * 32 * 8);
    const uint32_t rows0 = smem_u32(sm_rows);
    const float neutral = ISMAX ? -CUDART_INF_F : 0.f;
    const float fillv = ISMAX ? (p.sign < 0.f ? CUDART_INF_F : -CUDART_INF_F) : 0.f;

    if (lane == 0) {
#pragma unroll
        for (int s = 0; s < S; ++s) mbar_init(bar0 + 8 * s, 1);
        fence_mbar_init();
    }
    __syncwarp();

    const ChunkBounds cb = chunk_bounds(p.rowptr, p.row, k, p.chunk, p.E, p.nchunks);
    const int e_begin = cb.e_begin, e_end = cb.e_end;
    const int nE = e_end - e_begin;
    if (nE <= 0) return;                               // warp-uniform
    const int nbatch = (nE + 31) >> 5;

    float4 acc[K];
#pragma unroll
    for (int i = 0; i < K; ++i) acc[i] = make_float4(neutral, neutral, neutral, neutral);
    int r = -1;
    bool first_flush = true;

    auto flush = [&](int rr, bool last) {
        float* base;
        bool raw;
        if (first_flush && cb.head_partial) { base = p.ws + (size_t)(2 * k + 0) * p.D; raw = true; }
        else if (last && cb.tail_partial) { base = p.ws + (size_t)(2 * k + 1) * p.D; raw = true; }
        else { base = p.out + (size_t)rr * p.D; raw = false; }
        first_flush = false;
#pragma unroll
        for (int i = 0; i < K; ++i) {
            const float4 v = raw ? acc[i] : bfinish(acc[i], p, rr);
            *reinterpret_cast<float4*>(base + i * 128 + lane * 4) = v;
        }
    };
    auto fill_gap = [&](int lo, int hi) {
        if (!p.fill) return;
        for (int q = lo + 1; q < hi; ++q)
#pragma unroll
            for (int i = 0; i < K; ++i)
                *reinterpret_cast<float4*>(p.out + (size_t)q * p.D + i * 128 + lane * 4) =
                    make_float4(fillv, fillv, fillv, fillv);
    };

    // index prefetch for batch b (plain loads, consumed one full batch later) ...
    int n_c = 0, n_d = -1;
    float n_s = 1.f;
    bool n_valid = false;
    auto prefetch = [&](int b) {
        const int my_e = e_begin + b * 32 + lane;
        n_valid = my_e < e_end;
        n_c = 0; n_d = -1; n_s = 1.f;
        if (n_valid) {
            n_c = __ldg(p.col + my_e);
            n_d = __ldg(p.row + my_e);
            if (p.cs) n_s = __ldg(p.cs + n_c);
            if (p.w) n_s = __fmul_rn(n_s, __ldg(p.w + my_e));
            if (p.sign < 0.f) n_s = -n_s;
        }
    };
    // ... and the issue: every valid lane bulk-copies the feature row of its edge into stage b % S
    auto issue = [&](int b) {
        const int stage = b % S;
        sm_d[stage * 32 + lane] = n_d;
        sm_s[stage * 32 + lane] = n_s;
        const int nv = min(32, nE - b * 32);
        if (lane == 0) {
            fence_proxy_async();   // the stage's previous contents were read through the generic proxy
            mbar_expect_tx(bar0 + 8 * stage, (uint32_t)(nv * RB));
        }
        __syncwarp();
        if (n_valid) {
            const float* src = (p.x2 != nullptr && n_c >= p.split) ? p.x2 + (size_t)(n_c - p.split) * p.D
                                                                    : p.x + (size_t)n_c * p.D;
            bulk_g2s(rows0 + (uint32_t)(stage * STAGE_BYTES + lane * RB), src, RB, bar0 + 8 * stage);
        }
    };

    const int npro = nbatch < S ? nbatch : S;
    for (int b = 0; b < npro; ++b) { prefetch(b); issue(b); }

    int d_prev = -2;   // row of the edge before this batch (none yet)
    for (int b = 0; b < nbatch; ++b) {
        const int stage = b % S;
        const uint32_t parity = (uint32_t)((b / S) & 1);
        if (b + S < nbatch) prefetch(b + S);           // latency hidden behind this batch's wait + consume
        while (!mbar_try_wait(bar0 + 8 * stage, parity)) {}
        const int nb = min(32, nE - b * 32);
        const int d_l = sm_d[stage * 32 + lane];
        const float s_l = sm_s[stage * 32 + lane];
        int d_up = __shfl_up_sync(FULL, d_l, 1);
        if (lane == 0) d_up = d_prev;
        const unsigned starts = __ballot_sync(FULL, (lane < nb) && (d_l != d_up));
        d_prev = __shfl_sync(FULL, d_l, nb - 1);
        const float* srow = sm_rows + (size_t)stage * (STAGE_BYTES / 4);
#pragma unroll 4
        for (int j = 0; j < nb; ++j) {
            if ((starts >> j) & 1u) {                 // warp-uniform: a new row starts at this edge
                const int dj = __shfl_sync(FULL, d_l, j);
                if (r >= 0) { flush(r, false); fill_gap(r, dj); }
                else if (!cb.head_partial) fill_gap(cb.prev_row, dj);
                r = dj;
#pragma unroll
                for (int i = 0; i < K; ++i) acc[i] = make_float4(neutral, neutral, neutral, neutral);
            }
            const float sj = __shfl_sync(FULL, s_l, j);
#pragma unroll
            for (int i = 0; i < K; ++i) {
                const float4 v = *reinterpret_cast<const float4*>(srow + j * (RB / 4) + i * 128 + lane * 4);
                acc[i] = bcomb<ISMAX>(acc[i], v, sj);
            }
        }
        __syncwarp();                                  // every lane is done reading the stage
        if (b + S < nbatch) issue(b + S);
    }
    flush(r, true);
    if (e_end == p.E) fill_gap(r, p.nrows);
}

template <int K, int S, int WARPS, bool ISMAX>
static int launch_bulk(const BulkParams& p, cudaStream_t st) {
    constexpr int RB = K * 512;
    constexpr size_t smem = (size_t)WARPS * ((S * 32 * RB + S * 32 * 8 + S * 8 + 127) & ~127);
    static bool configured = false;
    if (!configured) {
        GNNB_CUDA(cudaFuncSetAttribute(seg_reduce_bulk_kernel<K, S, WARPS, ISMAX>,
                                       cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
        configured = true;
    }
    const unsigned grid = (unsigned)ceil_div(p.nchunks, WARPS);
    seg_reduce_bulk_kernel<K, S, WARPS, ISMAX><<<grid, 32 * WARPS, smem, st>>>(p);
    GNNB_LAUNCHED();
    return GNNB_OK;
}

// returns GNNB_EUNSUPPORTED (without setting the error text) when the shape is not covered.
// (the cp.async / LDGSTS ring variants of round 1 measured slower and are gone)
int seg_reduce_bulk(const Csr& c, const SegArgs& a, int64_t E, int chunk, float* ws, int fill, int cfg,
                    cudaStream_t st) {
    if (a.D % 128 != 0 || a.D > 512 || a.D == 384) return GNNB_EUNSUPPORTED;
    BulkParams p;
    p.rowptr = c.rowptr; p.col = c.col; p.row = c.row;
    p.x = a.x; p.x2 = a.x2; p.split = a.split; p.w = a.w; p.cs = a.cs; p.ct = a.ct; p.out = a.out; p.ws = ws;
    p.D = a.D; p.E = (int32_t)E; p.nrows = c.nrows; p.chunk = chunk; p.nchunks = (int32_t)ceil_div(E, chunk);
    p.mean = (a.aggr == GNNB_MEAN); p.fill = fill; p.sign = (a.aggr == GNNB_MIN) ? -1.f : 1.f;
    const bool ismax = (a.aggr == GNNB_MAX || a.aggr == GNNB_MIN);
    const int K = (int)(a.D / 128);
#define BULK_CASE(KK, SS, WW) \
    return ismax ? launch_bulk<KK, SS, WW, true>(p, st) : launch_bulk<KK, SS, WW, false>(p, st);
    (void)cfg;
    if (K == 1) { BULK_CASE(1, 2, 3) }
    if (K == 2) { BULK_CASE(2, 3, 1) }
    BULK_CASE(4, 2, 1)
#undef BULK_CASE
}

}  // namespace gnnb
