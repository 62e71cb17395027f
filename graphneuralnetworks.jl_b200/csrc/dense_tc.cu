// dense_tc.cu — hand-written wgmma kernels for the per-layer dense contraction  Y = act(X * W^T + b)
// (GNNlib/src/layers/conv.jl:69-71 `l.σ.(weight * x .+ l.bias)`; X is (N rows, K), W is (Nout, K) row-major).
//
// fp32 in, fp32 out, fp32-level accuracy on the TF32 tensor cores by the 3xTF32 split:
//     x = x_big + x_small,  x_big = x with the low 13 mantissa bits cleared (what the tf32 MMA reads anyway),
//     x_small = x - x_big (exact in fp32);   x*w ~= x_big*w_big + x_big*w_small + x_small*w_big
// (the dropped x_small*w_small term is 2^-22 relative).  The big*big products accumulate in one register accumulator
// and the two cross terms (2^-11 smaller) in a second one; the epilogue adds the two.
//
// Shape: one persistent CTA per SM, 384 threads.  W (<= 128 x 128) is split once into two K-major 128B-swizzled
// shared-memory images (w_big, w_small).  Row tiles of 128 rows of X stream through a 3-stage ring, one 32-float K-block
// per stage:
//   warps 0-3    producers : coalesced LDG.128 of the K-block, split in registers, st.shared into the canonical K-major
//                            SWIZZLE_128B layout (x_big, x_small), fence.proxy.async, arrive on full[stage]
//   warps 4-11   consumers : two warpgroups, 64 rows of the tile each: 12 wgmma.m64n128k8.tf32 per K-block from shared
//                            memory into registers, then + bias, relu, stores straight from the accumulator fragment
// The kernel is HBM-bound by design (2 x 4 x K bytes per row against 6 K^2 flops on the TF32 tensor cores).
// Every mbarrier wait is bounded: a broken pipeline makes the kernel flag an error and drain instead of hanging.
#include "common.cuh"

namespace gnnb {

namespace tc {
constexpr int BM = 128;           // rows per tile (two warpgroups x wgmma M = 64)
constexpr int BK = 32;            // floats per K-block = one 128 B swizzle row
constexpr int BN = 128;           // wgmma N: W images hold 128 rows, zero beyond Nout
constexpr int NSTAGE = 3;
constexpr int PRODUCERS = 128;    // warps 0-3
constexpr int CONSUMER_WARPS = 8; // warps 4-11 = warpgroups 1 and 2
constexpr int THREADS = PRODUCERS + CONSUMER_WARPS * 32;
constexpr int KBLK_BYTES = BM * 128;          // one operand image of a K-block: 128 rows x 128 B = 16 KB
constexpr int W_BYTES = 4 * KBLK_BYTES;       // up to K = 128: 64 KB per image
constexpr int SMEM_W_BIG = 0;
constexpr int SMEM_W_SMALL = W_BYTES;
constexpr int SMEM_A = 2 * W_BYTES;           // stages: [big 16 KB][small 16 KB]
constexpr int SMEM_BIAS = SMEM_A + NSTAGE * 2 * KBLK_BYTES;
constexpr int SMEM_BAR = SMEM_BIAS + 512;
constexpr int SMEM_TOTAL = SMEM_BAR + 64;

__device__ __forceinline__ uint32_t s_u32(const void* p) { return (uint32_t)__cvta_generic_to_shared(p); }
__device__ __forceinline__ void bar_init(uint32_t bar, uint32_t count) {
    asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(bar), "r"(count) : "memory");
}
__device__ __forceinline__ void bar_arrive(uint32_t bar) {
    asm volatile("mbarrier.arrive.shared::cta.b64 _, [%0];" ::"r"(bar) : "memory");
}
__device__ __forceinline__ bool bar_try(uint32_t bar, uint32_t parity) {
    uint32_t ok;
    asm volatile("{\n\t.reg .pred p;\n\tmbarrier.try_wait.parity.shared::cta.b64 p, [%1], %2;\n\tselp.u32 %0, 1, 0, p;\n\t}"
                 : "=r"(ok) : "r"(bar), "r"(parity) : "memory");
    return ok != 0;
}
// bounded wait: returns false (and raises *err) if the barrier never flips
__device__ __forceinline__ bool bar_wait(uint32_t bar, uint32_t parity, int* err) {
    for (uint32_t spin = 0; spin < (1u << 26); ++spin) {
        if (bar_try(bar, parity)) return true;
        if ((spin & 1023) == 1023 && *(volatile int*)err) return false;
    }
    atomicExch(err, 1);
    return false;
}
__device__ __forceinline__ float tf32_big(float x) { return __uint_as_float(__float_as_uint(x) & 0xffffe000u); }
// x - tf32_big(x): exact for finite x; 0 for x = +-Inf, whose big part already is x (Inf - Inf would put a NaN in the
// cross terms).  A NaN stays NaN.
__device__ __forceinline__ float tf32_small(float x, float b) { return isinf(x) ? 0.f : x - b; }
__device__ __forceinline__ float4 tf32_small(float4 v, float4 b) {
    return make_float4(tf32_small(v.x, b.x), tf32_small(v.y, b.y), tf32_small(v.z, b.z), tf32_small(v.w, b.w));
}
__device__ __forceinline__ void fence_proxy_async() { asm volatile("fence.proxy.async.shared::cta;" ::: "memory"); }
// asks L2 to fetch `bytes` (a multiple of 16) at the 16 B aligned `p` ahead of the register loads that will read them
__device__ __forceinline__ void prefetch_l2(const void* p, uint32_t bytes) {
    asm volatile("cp.async.bulk.prefetch.L2.global [%0], %1;" ::"l"(p), "r"(bytes) : "memory");
}

// wgmma shared-memory descriptor: K-major, SWIZZLE_128B, 8-row groups 1024 B apart (stride byte offset), leading byte
// offset unused by this layout.  A step of K = 8 tf32 inside the 128 B swizzle row advances the start address by 32 B.
__device__ __forceinline__ uint64_t gmma_desc(uint32_t saddr) {
    return (uint64_t)((saddr & 0x3ffffu) >> 4) | ((uint64_t)1 << 16) | ((uint64_t)(1024 >> 4) << 32) | ((uint64_t)1 << 62);
}
// D(64 x 128, fp32 registers) (+)= A(64 x 8) * B(128 x 8)^T, both operands tf32 K-major in shared memory.
// Fragment of D: register 4j + 2h + c of thread (warp w of the warpgroup, lane l) is row 16w + l/4 + 8h, column 8j + 2(l%4) + c.
__device__ __forceinline__ void wgmma_tf32(float* d, uint64_t da, uint64_t db, uint32_t accumulate) {
    asm volatile(
        "{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %66, 0;\n\t"
        "wgmma.mma_async.sync.aligned.m64n128k8.f32.tf32.tf32 "
        "{%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, %16, %17, %18, %19, %20, %21, %22, %23, "
        "%24, %25, %26, %27, %28, %29, %30, %31, %32, %33, %34, %35, %36, %37, %38, %39, %40, %41, %42, %43, %44, %45, %46, "
        "%47, %48, %49, %50, %51, %52, %53, %54, %55, %56, %57, %58, %59, %60, %61, %62, %63}, %64, %65, p, 1, 1;\n\t}"
        : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]), "+f"(d[8]),
          "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]), "+f"(d[16]),
          "+f"(d[17]), "+f"(d[18]), "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23]), "+f"(d[24]),
          "+f"(d[25]), "+f"(d[26]), "+f"(d[27]), "+f"(d[28]), "+f"(d[29]), "+f"(d[30]), "+f"(d[31]), "+f"(d[32]),
          "+f"(d[33]), "+f"(d[34]), "+f"(d[35]), "+f"(d[36]), "+f"(d[37]), "+f"(d[38]), "+f"(d[39]), "+f"(d[40]),
          "+f"(d[41]), "+f"(d[42]), "+f"(d[43]), "+f"(d[44]), "+f"(d[45]), "+f"(d[46]), "+f"(d[47]), "+f"(d[48]),
          "+f"(d[49]), "+f"(d[50]), "+f"(d[51]), "+f"(d[52]), "+f"(d[53]), "+f"(d[54]), "+f"(d[55]), "+f"(d[56]),
          "+f"(d[57]), "+f"(d[58]), "+f"(d[59]), "+f"(d[60]), "+f"(d[61]), "+f"(d[62]), "+f"(d[63])
        : "l"(da), "l"(db), "r"(accumulate));
}
// keeps the compiler from moving accumulator reads / writes across the asynchronous MMA
__device__ __forceinline__ void fence_acc(float* d) {
#pragma unroll
    for (int i = 0; i < 64; ++i) asm volatile("" : "+f"(d[i])::"memory");
}
__device__ __forceinline__ void wgmma_fence() { asm volatile("wgmma.fence.sync.aligned;" ::: "memory"); }
__device__ __forceinline__ void wgmma_commit() { asm volatile("wgmma.commit_group.sync.aligned;" ::: "memory"); }
__device__ __forceinline__ void wgmma_wait_all() { asm volatile("wgmma.wait_group.sync.aligned 0;" ::: "memory"); }

// one 32-wide K-block of the 3xTF32 product: cross terms into dc, big*big into dm (dc == dm: one accumulator);
// the images are K-major SWIZZLE_128B, A starting at this warpgroup's 64 rows
__device__ __forceinline__ void mma_kblock(float* dm, float* dc, uint32_t a_big, uint32_t a_small, uint32_t b_big,
                                           uint32_t b_small, bool first) {
    wgmma_fence();
    fence_acc(dm);
    fence_acc(dc);
#pragma unroll
    for (int j = 0; j < 4; ++j) {                      // 4 x (K = 8 tf32 = 32 B) per K-block, small terms first
        const uint32_t o = j * 32;
        const uint32_t acc = (first && j == 0) ? 0u : 1u;
        wgmma_tf32(dc, gmma_desc(a_small + o), gmma_desc(b_big + o), acc);
        wgmma_tf32(dc, gmma_desc(a_big + o), gmma_desc(b_small + o), 1u);
        wgmma_tf32(dm, gmma_desc(a_big + o), gmma_desc(b_big + o), dm == dc ? 1u : acc);
    }
    wgmma_commit();
    wgmma_wait_all();
    fence_acc(dm);
    fence_acc(dc);
}

struct Params {
    const float* __restrict__ x;     // [M][K]
    const float* __restrict__ w;     // [Nout][ldw]: row n holds its K coefficients at w + n*ldw
    const float* __restrict__ bias;  // [Nout] or null
    const float* __restrict__ addend;  // [M][Nout] or null: y = act(x W^T + bias + addend) (may alias y)
    float* __restrict__ y;           // [M][Nout]
    int64_t M;
    int K, Nout, relu, ldw;
    int* err;
    const float* __restrict__ wimg;  // wide kernel only: W split and swizzled per (quarter, K-block), see tcx::w_image_kernel
    const float* __restrict__ act;   // linear_bwd_dx_kernel only: forward output for the relu mask, or null (no mask)
    float* __restrict__ colsum;      // linear_bwd_dx_kernel only: [grid][4 producer warps][128] column sums of dpre, or null
    uint32_t* __restrict__ mask;     // linear_relu_mask_kernel: [M][4] relu mask words written beside y;
                                     // linear_bwd_dx_mask_kernel: read in place of act
};

// The relu mask of a 128-wide layer output, 4 words (16 B) per row: bit 2j + c of word w of row r is (y[r][8j + 2w + c] > 0)
// for j < 16, c < 2; equivalently column n is bit 2 (n >> 3) + (n & 1) of word (n >> 1) & 3.  This is the accumulator
// fragment's own order (register 4j + 2h + c of lane l is column 8j + 2(l%4) + c), so lane l of the epilogue owns word l%4
// of each of its rows whole, and a warp's stores for one h are 8 rows x 16 B, contiguous.  The bit is taken from the value
// y holds after the relu, so it agrees with `y > 0` on y as stored (-0 and NaN inputs give 0).

// epilogue of one 64 x 128 accumulator pair: columns col_base + [0, 128) of rows row0 + [0, 64), `ncols` of them valid.
// MASK: also the relu mask words of the rows (relu on, col_base 0, ncols = Nout = 128)
template <bool MASK = false>
__device__ __forceinline__ void store_tile(const Params& p, const float* dm, const float* dc, const float* sbias, int64_t row0,
                                           int col_base, int ncols) {
    const int lane = threadIdx.x & 31, w4 = (threadIdx.x >> 5) & 3;
    const int64_t r0 = row0 + w4 * 16 + (lane >> 2);
    uint32_t mw[2] = {0u, 0u};
#pragma unroll
    for (int j = 0; j < BN / 8; ++j) {
        const int c = 8 * j + 2 * (lane & 3);
        if (c >= ncols) continue;
        const float b0 = sbias[col_base + c], b1 = sbias[col_base + c + 1];
#pragma unroll
        for (int h = 0; h < 2; ++h) {
            const int64_t row = r0 + 8 * h;
            if (row >= p.M) continue;
            float2 o = make_float2((dm[4 * j + 2 * h] + dc[4 * j + 2 * h]) + b0, (dm[4 * j + 2 * h + 1] + dc[4 * j + 2 * h + 1]) + b1);
            const size_t at = (size_t)row * p.Nout + col_base + c;
            if (p.addend) {
                const float2 a = *reinterpret_cast<const float2*>(p.addend + at);
                o.x += a.x; o.y += a.y;
            }
            if (p.relu) { o.x = fmax_nan(o.x, 0.f); o.y = fmax_nan(o.y, 0.f); }   // relu(NaN) = NaN
            *reinterpret_cast<float2*>(p.y + at) = o;
            if (MASK) mw[h] |= ((uint32_t)(o.x > 0.f) << (2 * j)) | ((uint32_t)(o.y > 0.f) << (2 * j + 1));
        }
    }
    if (MASK) {
#pragma unroll
        for (int h = 0; h < 2; ++h) {
            const int64_t row = r0 + 8 * h;
            if (row < p.M) p.mask[(size_t)row * 4 + (lane & 3)] = mw[h];
        }
    }
}

// consumer warpgroups of the ring kernels: warpgroup wg owns rows 64 wg .. 64 wg + 63 of every tile of this CTA
template <bool MASK = false>
__device__ __forceinline__ void consume_tiles(const Params& p, uint32_t sbase, const float* sbias, int KB, int64_t ntiles) {
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    const uint32_t bar_full = sbase + SMEM_BAR, bar_empty = bar_full + 8 * NSTAGE;
    const int wg = (warp - PRODUCERS / 32) >> 2;
    float dm[64] = {}, dc[64] = {};
    uint32_t it = 0;
    bool alive = true;
    for (int64_t tile = blockIdx.x; alive && tile < ntiles; tile += gridDim.x) {
        for (int kb = 0; kb < KB; ++kb, ++it) {
            const int stage = it % NSTAGE;
            if (!bar_wait(bar_full + 8 * stage, (it / NSTAGE) & 1, p.err)) { alive = false; break; }
            const uint32_t a_big = sbase + SMEM_A + stage * 2 * KBLK_BYTES + wg * 64 * 128, a_small = a_big + KBLK_BYTES;
            const uint32_t w_big = sbase + SMEM_W_BIG + kb * KBLK_BYTES, w_small = sbase + SMEM_W_SMALL + kb * KBLK_BYTES;
            mma_kblock(dm, dc, a_big, a_small, w_big, w_small, kb == 0);
            if (lane == 0) bar_arrive(bar_empty + 8 * stage);   // this warp's reads of the stage are complete
        }
        if (alive) store_tile<MASK>(p, dm, dc, sbias, tile * BM + wg * 64, 0, p.Nout);
    }
}

// MASK: linear_relu_mask_kernel, which also writes the relu mask of y (Nout = 128, relu on)
template <bool MASK>
__device__ __forceinline__ void linear_body(const Params& p) {
    extern __shared__ __align__(1024) unsigned char smem[];
    const int tid = threadIdx.x, warp = tid >> 5;
    const int KB = p.K / BK;                                   // K-blocks per tile (<= 4)
    const int64_t ntiles = (p.M + BM - 1) / BM;
    const uint32_t sbase = s_u32(smem);
    const uint32_t bar_full = sbase + SMEM_BAR;                // [NSTAGE]
    const uint32_t bar_empty = bar_full + 8 * NSTAGE;          // [NSTAGE]
    float* sbias = reinterpret_cast<float*>(smem + SMEM_BIAS);

    // ---- one-time setup: barriers, bias, W split into the two swizzled K-major images (rows >= Nout zero)
    if (tid == 0) {
        for (int s = 0; s < NSTAGE; ++s) { bar_init(bar_full + 8 * s, PRODUCERS); bar_init(bar_empty + 8 * s, CONSUMER_WARPS); }
        asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
    }
    for (int i = tid; i < BN; i += THREADS) sbias[i] = (p.bias && i < p.Nout) ? p.bias[i] : 0.f;
    {
        const int kv = p.K >> 2;                               // float4 per row of W
        for (int idx = tid; idx < BN * kv; idx += THREADS) {
            const int n = idx / kv, c4 = idx - n * kv, kb = c4 >> 3, c = c4 & 7;
            const float4 v = n < p.Nout ? __ldg(reinterpret_cast<const float4*>(p.w + (size_t)n * p.ldw) + c4)
                                        : make_float4(0.f, 0.f, 0.f, 0.f);
            const float4 b = make_float4(tf32_big(v.x), tf32_big(v.y), tf32_big(v.z), tf32_big(v.w));
            const float4 s = tf32_small(v, b);
            const int off = kb * KBLK_BYTES + (n >> 3) * 1024 + (n & 7) * 128 + ((c ^ (n & 7)) << 4);
            *reinterpret_cast<float4*>(smem + SMEM_W_BIG + off) = b;
            *reinterpret_cast<float4*>(smem + SMEM_W_SMALL + off) = s;
        }
    }
    fence_proxy_async();                                       // W images are read by the tensor core (async proxy)
    __syncthreads();

    if (warp < PRODUCERS / 32) {
        // ================= producers =================
        const int c = tid & 7, r16 = tid >> 3, rr = r16 & 7;
        // flattened (tile, K-block) sequence of this CTA; the next item is prefetched into registers while the current
        // one waits for its shared-memory slot
        const int64_t my_tiles = (ntiles > (int64_t)blockIdx.x) ? (ntiles - blockIdx.x + gridDim.x - 1) / gridDim.x : 0;
        const int64_t total = my_tiles * KB;
        auto fetch = [&](int64_t item, float4* v) {
            const int64_t tile = blockIdx.x + (item / KB) * gridDim.x;
            const int kb = (int)(item % KB);
#pragma unroll
            for (int i = 0; i < 8; ++i) {
                const int64_t row = tile * BM + r16 + 16 * i;
                v[i] = (item < total && row < p.M)
                           ? __ldg(reinterpret_cast<const float4*>(p.x + (size_t)row * p.K + kb * BK) + c)
                           : make_float4(0.f, 0.f, 0.f, 0.f);
            }
        };
        float4 v[8], vn[8];
        fetch(0, v);
        for (int64_t it = 0; it < total; ++it) {
            fetch(it + 1, vn);
            const int stage = (int)(it % NSTAGE);
            if (!bar_wait(bar_empty + 8 * stage, (uint32_t)(((it / NSTAGE) & 1) ^ 1), p.err)) break;
            unsigned char* abig = smem + SMEM_A + stage * 2 * KBLK_BYTES;
#pragma unroll
            for (int i = 0; i < 8; ++i) {
                const float4 b = make_float4(tf32_big(v[i].x), tf32_big(v[i].y), tf32_big(v[i].z), tf32_big(v[i].w));
                const float4 s = tf32_small(v[i], b);
                const int off = ((r16 >> 3) + 2 * i) * 1024 + rr * 128 + ((c ^ rr) << 4);
                *reinterpret_cast<float4*>(abig + off) = b;
                *reinterpret_cast<float4*>(abig + KBLK_BYTES + off) = s;
            }
            fence_proxy_async();
            bar_arrive(bar_full + 8 * stage);
#pragma unroll
            for (int i = 0; i < 8; ++i) v[i] = vn[i];
        }
    } else {
        consume_tiles<MASK>(p, sbase, sbias, KB, ntiles);
    }
}

__global__ void __launch_bounds__(THREADS, 1) linear_tf32x3_kernel(const Params p) { linear_body<false>(p); }
__global__ void __launch_bounds__(THREADS, 1) linear_relu_mask_kernel(const Params p) { linear_body<true>(p); }

// dx = dpre * W for dpre = relu ? (y > 0 ? dy : 0) : dy, Dout = 128 rows of W and Din = Nout <= 128 columns.  The producers
// form dpre from dy and the forward output y (p.act) in registers, so dpre is never stored, and add it into per-thread
// column sums for db.  Tiles, images and the MMA sequence are those of linear_tf32x3_kernel run on a transposed copy of W
// with a zero bias, so dx has the same bits as that composition; W is read transposed straight into the images instead.
// MASK: linear_bwd_dx_mask_kernel, which reads the relu mask bits (p.mask, always on) in place of y: the same dpre, from
// 16 B per row instead of 512.
template <bool MASK>
__device__ __forceinline__ void bwd_dx_body(const Params& p) {
    extern __shared__ __align__(1024) unsigned char smem[];
    const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
    const int64_t ntiles = (p.M + BM - 1) / BM;
    const uint32_t sbase = s_u32(smem);
    const uint32_t bar_full = sbase + SMEM_BAR;                // [NSTAGE]
    const uint32_t bar_empty = bar_full + 8 * NSTAGE;          // [NSTAGE]
    float* sbias = reinterpret_cast<float*>(smem + SMEM_BIAS);

    if (tid == 0) {
        for (int s = 0; s < NSTAGE; ++s) { bar_init(bar_full + 8 * s, PRODUCERS); bar_init(bar_empty + 8 * s, CONSUMER_WARPS); }
        asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
    }
    for (int i = tid; i < BN; i += THREADS) sbias[i] = 0.f;    // (dm + dc) + 0: a -0 sum stores as +0, as in the composition
    // image row n = column n of W (n < Din), K = the 128 rows of W
    for (int idx = tid; idx < BN * 32; idx += THREADS) {
        const int n = idx >> 5, c4 = idx & 31, kb = c4 >> 3, c = c4 & 7;
        float4 v = make_float4(0.f, 0.f, 0.f, 0.f);
        if (n < p.Nout) {
            const float* col = p.w + (size_t)(4 * c4) * p.Nout + n;
            v = make_float4(__ldg(col), __ldg(col + p.Nout), __ldg(col + 2 * p.Nout), __ldg(col + 3 * p.Nout));
        }
        const float4 b = make_float4(tf32_big(v.x), tf32_big(v.y), tf32_big(v.z), tf32_big(v.w));
        const float4 s = tf32_small(v, b);
        const int off = kb * KBLK_BYTES + (n >> 3) * 1024 + (n & 7) * 128 + ((c ^ (n & 7)) << 4);
        *reinterpret_cast<float4*>(smem + SMEM_W_BIG + off) = b;
        *reinterpret_cast<float4*>(smem + SMEM_W_SMALL + off) = s;
    }
    fence_proxy_async();
    __syncthreads();

    if (warp < PRODUCERS / 32) {
        // ================= producers: K = 128, so a tile is 4 K-blocks.  The next item is prefetched into registers, the
        // next tile into L2.
        const int c = tid & 7, r16 = tid >> 3, rr = r16 & 7;
        const float4 zero = make_float4(0.f, 0.f, 0.f, 0.f);
        // flattened (tile, K-block) sequence of this CTA, as in linear_tf32x3_kernel
        const int64_t my_tiles = (ntiles > (int64_t)blockIdx.x) ? (ntiles - blockIdx.x + gridDim.x - 1) / gridDim.x : 0;
        const int64_t total = my_tiles * 4;
        // the relu mask of the 4 columns 32 kb + 4 c .. + 3 a thread loads: MASK, words 2 (c & 1) and 2 (c & 1) + 1 of the
        // row's mask (bits 8 kb + 2 (c >> 1) and the next of each); otherwise the 4 floats of y
        using MaskReg = typename std::conditional<MASK, uint2, float4>::type;
        auto fetch = [&](int64_t item, float4* g, MaskReg* m) {
            const int64_t tile = blockIdx.x + (item >> 2) * gridDim.x;
            const int kb = (int)(item & 3);
#pragma unroll
            for (int i = 0; i < 8; ++i) {
                const int64_t row = tile * BM + r16 + 16 * i;
                const bool in = item < total && row < p.M;
                const size_t at = (size_t)row * 128 + kb * BK;
                g[i] = in ? __ldg(reinterpret_cast<const float4*>(p.x + at) + c) : zero;
                if constexpr (MASK) m[i] = in ? __ldg(reinterpret_cast<const uint2*>(p.mask + (size_t)row * 4) + (c & 1)) : make_uint2(0u, 0u);
                else m[i] = (in && p.act) ? __ldg(reinterpret_cast<const float4*>(p.act + at) + c) : zero;
            }
        };
        // dpre = act ? (act > 0 ? g : 0) : g, applied when the prefetched registers are promoted: holding the mask of the
        // current item as well would not fit beside the next item's loads.  kb: the K-block of the item in g
        auto masked = [&](float4* g, const MaskReg* m, int kb) {
            if constexpr (MASK) {
                const int s = 8 * kb + 2 * (c >> 1);
#pragma unroll
                for (int i = 0; i < 8; ++i) {
                    g[i].x = (m[i].x >> s) & 1u ? g[i].x : 0.f; g[i].y = (m[i].x >> (s + 1)) & 1u ? g[i].y : 0.f;
                    g[i].z = (m[i].y >> s) & 1u ? g[i].z : 0.f; g[i].w = (m[i].y >> (s + 1)) & 1u ? g[i].w : 0.f;
                }
            } else {
                if (!p.act) return;
#pragma unroll
                for (int i = 0; i < 8; ++i) {
                    g[i].x = m[i].x > 0.f ? g[i].x : 0.f; g[i].y = m[i].y > 0.f ? g[i].y : 0.f;
                    g[i].z = m[i].z > 0.f ? g[i].z : 0.f; g[i].w = m[i].w > 0.f ? g[i].w : 0.f;
                }
            }
        };
        // column sums of dpre: after each item the 4 threads of a warp that share a column group add theirs in a fixed
        // order, and lanes 8 kb .. 8 kb + 7 keep the sums of K-block kb (columns 32 kb + 4 c .. + 3)
        float4 cs = zero;
        float4 g[8], gn[8];
        MaskReg mn[8];
        fetch(0, g, mn);
        masked(g, mn, 0);
        for (int64_t it = 0; it < total; ++it) {
            const int kb = (int)(it & 3);
            if (tid == 0 && kb == 0 && it + 4 < total) {       // the next tile of this CTA into L2
                const int64_t r0 = (blockIdx.x + ((it >> 2) + 1) * gridDim.x) * BM, nr = (p.M - r0 < BM) ? p.M - r0 : BM;
                prefetch_l2(p.x + (size_t)r0 * 128, (uint32_t)(nr * 512));
                if (!MASK && p.act) prefetch_l2(p.act + (size_t)r0 * 128, (uint32_t)(nr * 512));
            }
            fetch(it + 1, gn, mn);
            if (p.colsum) {
                float4 t = zero;
#pragma unroll
                for (int i = 0; i < 8; ++i) { t.x += g[i].x; t.y += g[i].y; t.z += g[i].z; t.w += g[i].w; }
#pragma unroll
                for (int o = 8; o <= 16; o <<= 1) {
                    t.x += __shfl_xor_sync(0xffffffffu, t.x, o); t.y += __shfl_xor_sync(0xffffffffu, t.y, o);
                    t.z += __shfl_xor_sync(0xffffffffu, t.z, o); t.w += __shfl_xor_sync(0xffffffffu, t.w, o);
                }
                if ((lane >> 3) == kb) { cs.x += t.x; cs.y += t.y; cs.z += t.z; cs.w += t.w; }
            }
            const int stage = (int)(it % NSTAGE);
            if (!bar_wait(bar_empty + 8 * stage, (uint32_t)(((it / NSTAGE) & 1) ^ 1), p.err)) break;
            unsigned char* abig = smem + SMEM_A + stage * 2 * KBLK_BYTES;
#pragma unroll
            for (int i = 0; i < 8; ++i) {
                const float4 b = make_float4(tf32_big(g[i].x), tf32_big(g[i].y), tf32_big(g[i].z), tf32_big(g[i].w));
                const float4 s = tf32_small(g[i], b);
                const int off = ((r16 >> 3) + 2 * i) * 1024 + rr * 128 + ((c ^ rr) << 4);
                *reinterpret_cast<float4*>(abig + off) = b;
                *reinterpret_cast<float4*>(abig + KBLK_BYTES + off) = s;
            }
            fence_proxy_async();
            bar_arrive(bar_full + 8 * stage);
#pragma unroll
            for (int i = 0; i < 8; ++i) g[i] = gn[i];
            masked(g, mn, (kb + 1) & 3);
        }
        if (p.colsum) reinterpret_cast<float4*>(p.colsum + ((size_t)blockIdx.x * 4 + warp) * 128 + (lane >> 3) * BK)[c] = cs;
    } else {
        consume_tiles(p, sbase, sbias, 128 / BK, ntiles);
    }
}

__global__ void __launch_bounds__(THREADS, 1) linear_bwd_dx_kernel(const Params p) { bwd_dx_body<false>(p); }
__global__ void __launch_bounds__(THREADS, 1) linear_bwd_dx_mask_kernel(const Params p) { bwd_dx_body<true>(p); }
}  // namespace tc

// =====================================================================================================================
// dW = dPre^T * X  (the weight pullback of the dense layer):  dW[i][j] = sum_r dPre[r][i] * X[r][j],  r over all N rows.
// Both operands are "MN-major" in memory (the reduction index r is the slow one); tf32 wgmma reads K-major shared memory
// only, so the producers transpose 32 rows of each operand into the same K-major SWIZZLE_128B images the forward kernel
// uses: A = dPre^T (128 rows i), B = X^T (Din rows j, zero up to 128).  A lane covers 8 rows r x 4 float4 columns, which
// keeps both the global loads (64 B runs) and the transposing shared-memory stores (2-way) cheap.
// Split-K: every CTA reduces a contiguous range of rows into its own register accumulators and writes a (128 x Din)
// partial; a second kernel adds the partials in CTA order (deterministic).
// The accumulation chain is cut every FLUSH row blocks and each short chain is added into an fp32 register sum with
// ordinary round-to-nearest adds, so the length of the tensor core's accumulation chain does not grow with N.
// =====================================================================================================================
namespace tcw {
using namespace tc;
constexpr int WSTAGE = 3;
constexpr int FLUSH = 4;                      // row blocks (of 32 rows) per accumulation chain
constexpr int STAGE_BYTES = 4 * KBLK_BYTES;   // dPre big/small, X big/small
constexpr int SMEM_BARW = WSTAGE * STAGE_BYTES;
constexpr int SMEM_TOTALW = SMEM_BARW + 64;

struct ParamsW {
    const float* __restrict__ dpre;   // [M][128] (dy in the fused pullback)
    const float* __restrict__ x;      // [M][Din]
    float* __restrict__ partial;      // [grid][128][Din]
    int64_t M, rows_per_cta;
    int Din;
    int* err;
    const float* __restrict__ act;    // linear_bwd_dw_kernel only: forward output y, dpre = y > 0 ? dy : 0; null: dpre = dy
    const uint32_t* __restrict__ mask;  // linear_bwd_dw_mask_kernel only: [M][4] relu mask of y (layout: above tc::store_tile)
};
constexpr int L2_AHEAD = 3;           // linear_bwd_dw_kernel: row blocks prefetched into L2 ahead of the register loads

// byte offset of element (row n, k) of a K-major SWIZZLE_128B image, k < 32
__device__ __forceinline__ int kmajor_off(int n, int k) {
    return (n >> 3) * 1024 + (n & 7) * 128 + ((((k >> 2) ^ (n & 7))) << 4) + (k & 3) * 4;
}

// FUSED: the fused pullback's variant, which forms dpre from dy and the relu mask of p.act in the producers and prefetches
// the rows L2_AHEAD blocks ahead into L2; otherwise p.dpre is read as it is.  MASK (with FUSED): the relu mask comes from
// the bits of p.mask instead of y.
template <bool FUSED, bool MASK = false>
__device__ __forceinline__ void dw_body(const ParamsW& p) {
    extern __shared__ __align__(1024) unsigned char smem[];
    const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
    const uint32_t sbase = s_u32(smem);
    const uint32_t bar_full = sbase + SMEM_BARW, bar_empty = bar_full + 8 * WSTAGE;
    const int nfB = p.Din >> 2;                   // float4 per row of X
    const int64_t r_begin = (int64_t)blockIdx.x * p.rows_per_cta;
    const int64_t r_end = (r_begin + p.rows_per_cta < p.M) ? r_begin + p.rows_per_cta : p.M;
    const int64_t nblk = (r_end > r_begin) ? (r_end - r_begin + 31) / 32 : 0;

    if (tid == 0) {
        for (int s = 0; s < WSTAGE; ++s) { bar_init(bar_full + 8 * s, PRODUCERS); bar_init(bar_empty + 8 * s, CONSUMER_WARPS); }
        asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
    }
    // rows j >= Din of the X^T images are never written: zero them once
    for (int i = tid; i < SMEM_BARW / 16; i += THREADS) reinterpret_cast<float4*>(smem)[i] = make_float4(0.f, 0.f, 0.f, 0.f);
    fence_proxy_async();
    __syncthreads();

    if (warp < PRODUCERS / 32) {
        // ---- producers: 32 rows of dPre (128 floats) and of X (Din floats) per stage, transposed + split + swizzled
        const int rl = lane >> 2, fl = lane & 3;
        // the 8 float4 this thread covers in row block blk of src (row stride ld floats, nf float4 per row)
        auto load = [&](const float* src, int ld, int nf, int64_t blk, float4* v) {
#pragma unroll
            for (int q = 0; q < 8; ++q) {
                const int64_t r = r_begin + blk * 32 + rl + 8 * (q & 3);
                const int f = 4 * (warp + 4 * (q >> 2)) + fl;
                v[q] = (blk < nblk && r < r_end && f < nf) ? __ldg(reinterpret_cast<const float4*>(src + (size_t)r * ld) + f)
                                                           : make_float4(0.f, 0.f, 0.f, 0.f);
            }
        };
        auto put1 = [&](unsigned char* big, int n, int k, float e) {
            const int off = kmajor_off(n, k);
            const float b = tf32_big(e);
            *reinterpret_cast<float*>(big + off) = b;
            *reinterpret_cast<float*>(big + KBLK_BYTES + off) = tf32_small(e, b);
        };
        auto put = [&](unsigned char* big, int n0, int k, float4 v) {
            put1(big, n0, k, v.x); put1(big, n0 + 1, k, v.y); put1(big, n0 + 2, k, v.z); put1(big, n0 + 3, k, v.w);
        };
        auto stage_in = [&](int64_t blk, const float4* va, const float4* vb) {
            const int stage = (int)(blk % WSTAGE);
            if (!bar_wait(bar_empty + 8 * stage, (uint32_t)(((blk / WSTAGE) & 1) ^ 1), p.err)) return false;
            unsigned char* st = smem + stage * STAGE_BYTES;
#pragma unroll
            for (int q = 0; q < 8; ++q) {
                const int k = rl + 8 * (q & 3);
                const int f = 4 * (warp + 4 * (q >> 2)) + fl;
                put(st, 4 * f, k, va[q]);
                if (f < nfB) put(st + 2 * KBLK_BYTES, 4 * f, k, vb[q]);
            }
            fence_proxy_async();
            bar_arrive(bar_full + 8 * stage);
            return true;
        };
        if constexpr (!FUSED) {
            float4 va[8], vb[8], na[8], nb[8];
            load(p.dpre, 128, 32, 0, va);
            load(p.x, p.Din, nfB, 0, vb);
            for (int64_t blk = 0; blk < nblk; ++blk) {
                load(p.dpre, 128, 32, blk + 1, na);
                load(p.x, p.Din, nfB, blk + 1, nb);
                if (!stage_in(blk, va, vb)) break;
#pragma unroll
                for (int q = 0; q < 8; ++q) { va[q] = na[q]; vb[q] = nb[q]; }
            }
        } else if constexpr (MASK) {
            // as below with the mask bits in place of y: the 4 columns 4 f .. 4 f + 3 of a thread's float4 f are bits
            // 2 (f >> 1) and the next of words 2 (fl & 1) and 2 (fl & 1) + 1 of the row's mask (f & 1 == fl & 1), so
            // the two float4 of one row (q and q + 4) share one 8 B load
            float4 va[8], vb[8], na[8];
            uint2 nm[4];
            auto load_mask = [&](int64_t blk) {
#pragma unroll
                for (int q = 0; q < 4; ++q) {
                    const int64_t r = r_begin + blk * 32 + rl + 8 * q;
                    nm[q] = (blk < nblk && r < r_end) ? __ldg(reinterpret_cast<const uint2*>(p.mask + (size_t)r * 4) + (fl & 1))
                                                      : make_uint2(0u, 0u);
                }
            };
            auto promote = [&]() {
#pragma unroll
                for (int q = 0; q < 8; ++q) {
                    const uint2 m = nm[q & 3];
                    const int s = 4 * (warp + 4 * (q >> 2)) + 2 * (fl >> 1);
                    va[q].x = (m.x >> s) & 1u ? na[q].x : 0.f; va[q].y = (m.x >> (s + 1)) & 1u ? na[q].y : 0.f;
                    va[q].z = (m.y >> s) & 1u ? na[q].z : 0.f; va[q].w = (m.y >> (s + 1)) & 1u ? na[q].w : 0.f;
                }
            };
            load(p.dpre, 128, 32, 0, na);
            load_mask(0);
            promote();
            for (int64_t blk = 0; blk < nblk; ++blk) {
                if (tid == 0 && blk + L2_AHEAD < nblk) {
                    const int64_t ra = r_begin + 32 * (blk + L2_AHEAD), nr = (r_end - ra < 32) ? r_end - ra : 32;
                    prefetch_l2(p.dpre + (size_t)ra * 128, (uint32_t)(nr * 512));
                    prefetch_l2(p.x + (size_t)ra * p.Din, (uint32_t)(nr * p.Din * 4));
                }
                load(p.dpre, 128, 32, blk + 1, na);
                load_mask(blk + 1);
                load(p.x, p.Din, nfB, blk, vb);
                if (!stage_in(blk, va, vb)) break;
                promote();
            }
        } else {
            // dy and y are loaded one block ahead into registers and the mask is applied when they are promoted; x is
            // loaded when its block is staged, from L2, where it was prefetched L2_AHEAD blocks ahead (dy, y and x all one
            // block ahead would not fit the registers)
            float4 va[8], vb[8], na[8], nm[8];
            auto promote = [&]() {
#pragma unroll
                for (int q = 0; q < 8; ++q) {
                    va[q] = na[q];
                    if (p.act) {
                        va[q].x = nm[q].x > 0.f ? va[q].x : 0.f; va[q].y = nm[q].y > 0.f ? va[q].y : 0.f;
                        va[q].z = nm[q].z > 0.f ? va[q].z : 0.f; va[q].w = nm[q].w > 0.f ? va[q].w : 0.f;
                    }
                }
            };
            load(p.dpre, 128, 32, 0, na);
            if (p.act) load(p.act, 128, 32, 0, nm);
            promote();
            for (int64_t blk = 0; blk < nblk; ++blk) {
                if (tid == 0 && blk + L2_AHEAD < nblk) {
                    const int64_t ra = r_begin + 32 * (blk + L2_AHEAD), nr = (r_end - ra < 32) ? r_end - ra : 32;
                    prefetch_l2(p.dpre + (size_t)ra * 128, (uint32_t)(nr * 512));
                    if (p.act) prefetch_l2(p.act + (size_t)ra * 128, (uint32_t)(nr * 512));
                    prefetch_l2(p.x + (size_t)ra * p.Din, (uint32_t)(nr * p.Din * 4));
                }
                load(p.dpre, 128, 32, blk + 1, na);
                if (p.act) load(p.act, 128, 32, blk + 1, nm);
                load(p.x, p.Din, nfB, blk, vb);
                if (!stage_in(blk, va, vb)) break;
                promote();
            }
        }
    } else {
        // ---- consumers: warpgroup wg owns rows 64 wg .. 64 wg + 63 of dW (M = 128), N = Din (padded to 128)
        const int wg = (warp - PRODUCERS / 32) >> 2;
        float acc[64] = {}, sum[64];
#pragma unroll
        for (int i = 0; i < 64; ++i) sum[i] = 0.f;
        for (int64_t blk = 0; blk < nblk; ++blk) {
            const int stage = (int)(blk % WSTAGE);
            if (!bar_wait(bar_full + 8 * stage, (uint32_t)((blk / WSTAGE) & 1), p.err)) break;
            const uint32_t a_big = sbase + stage * STAGE_BYTES + wg * 64 * 128, a_small = a_big + KBLK_BYTES;
            const uint32_t b_big = sbase + stage * STAGE_BYTES + 2 * KBLK_BYTES, b_small = b_big + KBLK_BYTES;
            mma_kblock(acc, acc, a_big, a_small, b_big, b_small, (blk % FLUSH) == 0);
            if (lane == 0) bar_arrive(bar_empty + 8 * stage);
            if ((blk % FLUSH) == FLUSH - 1 || blk == nblk - 1) {
#pragma unroll
                for (int i = 0; i < 64; ++i) sum[i] += acc[i];
            }
        }
        const int w4 = warp & 3;
        const int i0 = wg * 64 + w4 * 16 + (lane >> 2);
#pragma unroll
        for (int j = 0; j < BN / 8; ++j) {
            const int c = 8 * j + 2 * (lane & 3);
            if (c >= p.Din) continue;
#pragma unroll
            for (int h = 0; h < 2; ++h) {
                float* prow = p.partial + ((size_t)blockIdx.x * 128 + i0 + 8 * h) * p.Din;
                *reinterpret_cast<float2*>(prow + c) = make_float2(sum[4 * j + 2 * h], sum[4 * j + 2 * h + 1]);
            }
        }
    }
}

__global__ void __launch_bounds__(THREADS, 1) dw_tf32x3_kernel(const ParamsW p) { dw_body<false>(p); }
__global__ void __launch_bounds__(THREADS, 1) linear_bwd_dw_kernel(const ParamsW p) { dw_body<true>(p); }
__global__ void __launch_bounds__(THREADS, 1) linear_bwd_dw_mask_kernel(const ParamsW p) { dw_body<true, true>(p); }

// dW[i] = sum of the n-float partials; with db: threads n .. n + 127 add the 128-float column-sum partials into db
__global__ void dw_reduce_kernel(const float* __restrict__ partial, int nparts, int n, float* __restrict__ dW,
                                 const float* __restrict__ colsum = nullptr, int ncolsum = 0, float* __restrict__ db = nullptr) {
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i < n) {
        float acc = 0.f;
        for (int b = 0; b < nparts; ++b) acc += partial[(size_t)b * n + i];     // fixed order: deterministic
        dW[i] = acc;
    } else if (db && i < n + 128) {
        float acc = 0.f;
        for (int b = 0; b < ncolsum; ++b) acc += colsum[(size_t)b * 128 + i - n];
        db[i - n] = acc;
    }
}
}  // namespace tcw

// =====================================================================================================================
// Wide shapes (K and/or Nout above 128: GATConv's 512 -> 8 x 64 projection, 256 -> 256 layers).  W no longer fits beside
// the ring, so every stage carries one K-block of BOTH operands: 128 rows of X, split big/small by the producer warps, and
// 128 rows of W (one column quarter of the output), which a small pre-pass has already split and swizzled in global
// memory so that ONE cp.async.bulk (32 KB, mbarrier complete_tx) drops it into the stage.  Item order per CTA: row tile ->
// output quarter -> K-block; the X tile is re-read from L2 for every quarter (HBM sees it once), the W image (2 x the size
// of W, <= 2 MB at 512 x 512) lives in L2.  The big*big products and the cross terms accumulate in separate register
// accumulators, so the chain that carries the full-magnitude sum is K/8 accumulations long.
// =====================================================================================================================
namespace tcx {
using namespace tc;
constexpr int XSTAGE = 3;
constexpr int XSTAGE_BYTES = 4 * KBLK_BYTES;                    // X big, X small, W big, W small: 64 KB
constexpr int SMEM_BIAS_X = XSTAGE * XSTAGE_BYTES;
constexpr int MAX_NOUT = 1024;
constexpr int SMEM_BAR_X = SMEM_BIAS_X + MAX_NOUT * 4;
constexpr int SMEM_TOTAL_X = SMEM_BAR_X + 64;

// W (Nout x K, row stride ldw) -> the shared-memory images the MMA reads, laid out in global memory block by block:
// block (quarter nq, K-block kb) = [big 16 KB][small 16 KB], each already in the K-major SWIZZLE_128B order.  One
// cp.async.bulk of 32 KB then fills the W half of a stage: no producer thread touches W.
__global__ void w_image_kernel(const float* __restrict__ w, int ldw, int K, int Nout, float* __restrict__ wimg) {
    const int kv = K >> 2, KB = K / BK;
    const int idx = blockIdx.x * blockDim.x + threadIdx.x;
    if (idx >= Nout * kv) return;
    const int n = idx / kv, c4 = idx - n * kv, kb = c4 >> 3, c = c4 & 7;
    const int nq = n >> 7, nl = n & 127;
    const float4 v = __ldg(reinterpret_cast<const float4*>(w + (size_t)n * ldw) + c4);
    const float4 b = make_float4(tf32_big(v.x), tf32_big(v.y), tf32_big(v.z), tf32_big(v.w));
    const float4 sm = tf32_small(v, b);
    unsigned char* blk = reinterpret_cast<unsigned char*>(wimg) + (size_t)(nq * KB + kb) * (2 * KBLK_BYTES);
    const int off = (nl >> 3) * 1024 + (nl & 7) * 128 + ((c ^ (nl & 7)) << 4);
    *reinterpret_cast<float4*>(blk + off) = b;
    *reinterpret_cast<float4*>(blk + KBLK_BYTES + off) = sm;
}

__device__ __forceinline__ void bulk_g2s(uint32_t dst, const void* src, uint32_t bytes, uint32_t bar) {
    asm volatile("cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];"
                 ::"r"(dst), "l"(src), "r"(bytes), "r"(bar) : "memory");
}
__device__ __forceinline__ void bar_expect_tx(uint32_t bar, uint32_t bytes) {
    asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(bar), "r"(bytes) : "memory");
}

__global__ void __launch_bounds__(THREADS, 1) linear_wide_tf32x3_kernel(const Params p) {
    extern __shared__ __align__(1024) unsigned char smem[];
    const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
    const int KB = p.K / BK;                                   // K-blocks per (tile, quarter)
    const int NQ = p.Nout / 128;                               // output quarters of 128 columns
    const int64_t ntiles = (p.M + BM - 1) / BM;
    const int64_t my_tiles = (ntiles > (int64_t)blockIdx.x) ? (ntiles - blockIdx.x + gridDim.x - 1) / gridDim.x : 0;
    const uint32_t sbase = s_u32(smem);
    const uint32_t bar_full = sbase + SMEM_BAR_X;              // [XSTAGE]
    const uint32_t bar_empty = bar_full + 8 * XSTAGE;          // [XSTAGE]
    float* sbias = reinterpret_cast<float*>(smem + SMEM_BIAS_X);

    if (tid == 0) {
        // a stage is full when the 128 producer threads have stored X and the bulk copy of the W block has landed
        for (int s = 0; s < XSTAGE; ++s) { bar_init(bar_full + 8 * s, PRODUCERS + 1); bar_init(bar_empty + 8 * s, CONSUMER_WARPS); }
        asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
    }
    for (int i = tid; i < p.Nout; i += THREADS) sbias[i] = p.bias ? p.bias[i] : 0.f;
    __syncthreads();

    if (warp < PRODUCERS / 32) {
        // ================= producers: X only (8 float4 per thread and stage), two stages ahead in registers =================
        const int c = tid & 7, r16 = tid >> 3, rr = r16 & 7;
        const int64_t total = my_tiles * NQ * KB;
        // (tile, quarter, K-block) of the next item to fetch, advanced without divisions
        int64_t f_tile = blockIdx.x;
        int f_nq = 0, f_kb = 0;
        auto fetch = [&](int64_t item, float4* va) {
#pragma unroll
            for (int i = 0; i < 8; ++i) {
                const int64_t row = f_tile * BM + r16 + 16 * i;
                va[i] = (item < total && row < p.M)
                            ? __ldg(reinterpret_cast<const float4*>(p.x + (size_t)row * p.K + f_kb * BK) + c)
                            : make_float4(0.f, 0.f, 0.f, 0.f);
            }
            if (++f_kb == KB) { f_kb = 0; if (++f_nq == NQ) { f_nq = 0; f_tile += gridDim.x; } }
        };
        float4 va[8], na[8], na2[8];
        fetch(0, va);
        fetch(1, na);
        int w_blk = 0;                                          // (quarter, K-block) of the current item: index of its W block
        const int w_blocks = NQ * KB;
        for (int64_t it = 0; it < total; ++it) {
            fetch(it + 2, na2);
            const int stage = (int)(it % XSTAGE);
            if (!bar_wait(bar_empty + 8 * stage, (uint32_t)(((it / XSTAGE) & 1) ^ 1), p.err)) break;
            unsigned char* sa = smem + stage * XSTAGE_BYTES;
            if (tid == 0) {
                bar_expect_tx(bar_full + 8 * stage, 2 * KBLK_BYTES);
                bulk_g2s(sbase + stage * XSTAGE_BYTES + 2 * KBLK_BYTES,
                         reinterpret_cast<const unsigned char*>(p.wimg) + (size_t)w_blk * (2 * KBLK_BYTES), 2 * KBLK_BYTES,
                         bar_full + 8 * stage);
            }
            if (++w_blk == w_blocks) w_blk = 0;
#pragma unroll
            for (int i = 0; i < 8; ++i) {
                const int off = ((r16 >> 3) + 2 * i) * 1024 + rr * 128 + ((c ^ rr) << 4);
                const float4 b = make_float4(tf32_big(va[i].x), tf32_big(va[i].y), tf32_big(va[i].z), tf32_big(va[i].w));
                *reinterpret_cast<float4*>(sa + off) = b;
                *reinterpret_cast<float4*>(sa + KBLK_BYTES + off) = tf32_small(va[i], b);
            }
            fence_proxy_async();
            bar_arrive(bar_full + 8 * stage);
#pragma unroll
            for (int i = 0; i < 8; ++i) { va[i] = na[i]; na[i] = na2[i]; }
        }
    } else {
        // ================= consumers: M = 64 rows per warpgroup, N = 128 columns of one output quarter =================
        const int wg = (warp - PRODUCERS / 32) >> 2;
        float dm[64] = {}, dc[64] = {};
        uint32_t it = 0;
        for (int64_t t = 0; t < my_tiles; ++t) {
            const int64_t tile = blockIdx.x + t * gridDim.x;
            for (int nq = 0; nq < NQ; ++nq) {
                for (int kb = 0; kb < KB; ++kb, ++it) {
                    const int stage = it % XSTAGE;
                    if (!bar_wait(bar_full + 8 * stage, (it / XSTAGE) & 1, p.err)) return;
                    const uint32_t a_big = sbase + stage * XSTAGE_BYTES + wg * 64 * 128, a_small = a_big + KBLK_BYTES;
                    const uint32_t w_big = sbase + stage * XSTAGE_BYTES + 2 * KBLK_BYTES, w_small = w_big + KBLK_BYTES;
                    mma_kblock(dm, dc, a_big, a_small, w_big, w_small, kb == 0);
                    if (lane == 0) bar_arrive(bar_empty + 8 * stage);
                }
                store_tile(p, dm, dc, sbias, tile * BM + wg * 64, nq * 128, 128);
            }
        }
    }
}
}  // namespace tcx

static int* g_tc_err = nullptr;
int g_tc_enabled = 1;

// returns GNNB_EUNSUPPORTED (no error text) when the shape is not covered by the tensor-core kernel
int linear_tf32x3_ex(const float* x, const float* W, int64_t ldw, const float* bias, const float* addend, int relu, int64_t M,
                     int64_t K, int64_t Nout, float* y, cudaStream_t st);
int linear_tf32x3(const float* x, const float* W, const float* bias, int relu, int64_t M, int64_t K, int64_t Nout, float* y,
                  cudaStream_t st) {
    return linear_tf32x3_ex(x, W, K, bias, nullptr, relu, M, K, Nout, y, st);
}
static int linear_launch(const float* x, const float* W, int64_t ldw, const float* bias, const float* addend, int relu,
                         int64_t M, int64_t K, int64_t Nout, float* y, uint32_t* mask, cudaStream_t st);
// W rows `ldw` floats apart (a column block of a wider matrix); addend (M, Nout) added before the activation
int linear_tf32x3_ex(const float* x, const float* W, int64_t ldw, const float* bias, const float* addend, int relu, int64_t M,
                     int64_t K, int64_t Nout, float* y, cudaStream_t st) {
    return linear_launch(x, W, ldw, bias, addend, relu, M, K, Nout, y, nullptr, st);
}
// y = relu(x W^T + bias) and its relu mask (M, 4 words; layout above tc::store_tile) for Nout = 128, K in {32, 64, 96, 128}
int linear_relu_mask_tf32x3(const float* x, const float* W, const float* bias, int64_t M, int64_t K, float* y, uint32_t* mask,
                            cudaStream_t st) {
    if (K % 32 != 0 || K < 32 || K > 128 || ((uintptr_t)mask & 15)) return GNNB_EUNSUPPORTED;
    return linear_launch(x, W, K, bias, nullptr, 1, M, K, 128, y, mask, st);
}
static int linear_launch(const float* x, const float* W, int64_t ldw, const float* bias, const float* addend, int relu,
                         int64_t M, int64_t K, int64_t Nout, float* y, uint32_t* mask, cudaStream_t st) {
    if (!g_tc_enabled) return GNNB_EUNSUPPORTED;
    const bool wide = K > 128 || Nout > 128;
    if (wide) {
        // (a handful of row tiles cannot fill the machine: the library GEMM takes those)
        if (K % 32 != 0 || K > 2048 || Nout % 128 != 0 || Nout > tcx::MAX_NOUT || ldw % 4 != 0 || ldw < K || M < 2048) return GNNB_EUNSUPPORTED;
    } else if (K % 32 != 0 || Nout % 16 != 0 || Nout < 16 || ldw % 4 != 0 || ldw < K) {
        return GNNB_EUNSUPPORTED;
    }
    if (((uintptr_t)x & 15) || ((uintptr_t)W & 15) || ((uintptr_t)y & 15) || ((uintptr_t)addend & 15)) return GNNB_EUNSUPPORTED;
    if (M == 0) return GNNB_OK;
    static bool configured = false;
    static int nsm = 0;
    if (!configured) {
        GNNB_CUDA(cudaFuncSetAttribute(tc::linear_tf32x3_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, tc::SMEM_TOTAL));
        GNNB_CUDA(cudaFuncSetAttribute(tc::linear_relu_mask_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, tc::SMEM_TOTAL));
        GNNB_CUDA(cudaFuncSetAttribute(tcx::linear_wide_tf32x3_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, tcx::SMEM_TOTAL_X));
        int dev = 0;
        GNNB_CUDA(cudaGetDevice(&dev));
        GNNB_CUDA(cudaDeviceGetAttribute(&nsm, cudaDevAttrMultiProcessorCount, dev));
        GNNB_CUDA(cudaMalloc(&g_tc_err, sizeof(int)));
        GNNB_CUDA(cudaMemset(g_tc_err, 0, sizeof(int)));
        configured = true;
    }
    tc::Params p;
    p.x = x; p.w = W; p.bias = bias; p.addend = addend; p.y = y; p.M = M; p.K = (int)K; p.Nout = (int)Nout; p.relu = relu;
    p.ldw = (int)ldw; p.err = g_tc_err; p.wimg = nullptr; p.act = nullptr; p.colsum = nullptr; p.mask = mask;
    if (wide) {
        // the split, swizzled image of W (2 x its size), rebuilt per call: W changes between training steps
        static float* wimg = nullptr; static size_t wimg_elems = 0;
        const size_t need = (size_t)2 * K * Nout;
        if (wimg_elems < need) {
            if (wimg) { cudaDeviceSynchronize(); cudaFree(wimg); wimg = nullptr; wimg_elems = 0; }
            GNNB_CUDA(cudaMalloc(&wimg, sizeof(float) * need));
            wimg_elems = need;
        }
        tcx::w_image_kernel<<<(unsigned)ceil_div(Nout * (K / 4), 256), 256, 0, st>>>(W, (int)ldw, (int)K, (int)Nout, wimg);
        GNNB_LAUNCHED();
        p.wimg = wimg;
    }
    const int64_t ntiles = ceil_div(M, tc::BM);
    const unsigned grid = (unsigned)(ntiles < nsm ? ntiles : nsm);
    if (wide) tcx::linear_wide_tf32x3_kernel<<<grid, tc::THREADS, tcx::SMEM_TOTAL_X, st>>>(p);
    else if (mask) tc::linear_relu_mask_kernel<<<grid, tc::THREADS, tc::SMEM_TOTAL, st>>>(p);
    else tc::linear_tf32x3_kernel<<<grid, tc::THREADS, tc::SMEM_TOTAL, st>>>(p);
    GNNB_LAUNCHED();
    return GNNB_OK;
}

// dW (Dout = 128, Din in {32, 64, 96, 128}); GNNB_EUNSUPPORTED for anything else
int dw_tf32x3(const float* dpre, const float* x, int64_t M, int64_t Din, int64_t Dout, float* dW, cudaStream_t st) {
    if (!g_tc_enabled) return GNNB_EUNSUPPORTED;
    if (Dout != 128 || Din % 32 != 0 || Din > 128 || Din < 32) return GNNB_EUNSUPPORTED;
    if (((uintptr_t)dpre & 15) || ((uintptr_t)x & 15) || ((uintptr_t)dW & 15)) return GNNB_EUNSUPPORTED;
    static bool configured = false;
    static int nsm = 0;
    static float* partial = nullptr;
    if (!configured) {
        GNNB_CUDA(cudaFuncSetAttribute(tcw::dw_tf32x3_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, tcw::SMEM_TOTALW));
        int dev = 0;
        GNNB_CUDA(cudaGetDevice(&dev));
        GNNB_CUDA(cudaDeviceGetAttribute(&nsm, cudaDevAttrMultiProcessorCount, dev));
        GNNB_CUDA(cudaMalloc(&partial, sizeof(float) * (size_t)nsm * 128 * 128));
        if (!g_tc_err) { GNNB_CUDA(cudaMalloc(&g_tc_err, sizeof(int))); GNNB_CUDA(cudaMemset(g_tc_err, 0, sizeof(int))); }
        configured = true;
    }
    if (M == 0) { GNNB_CUDA(cudaMemsetAsync(dW, 0, sizeof(float) * (size_t)(Dout * Din), st)); return GNNB_OK; }
    tcw::ParamsW p;
    p.dpre = dpre; p.x = x; p.partial = partial; p.M = M; p.Din = (int)Din; p.err = g_tc_err; p.act = nullptr; p.mask = nullptr;
    int64_t rpc = ceil_div(M, nsm);
    rpc = ceil_div(rpc, 32) * 32;
    p.rows_per_cta = rpc;
    const int grid = (int)ceil_div(M, rpc);
    tcw::dw_tf32x3_kernel<<<grid, tc::THREADS, tcw::SMEM_TOTALW, st>>>(p);
    GNNB_LAUNCHED();
    const int n = (int)(128 * Din);
    tcw::dw_reduce_kernel<<<(unsigned)ceil_div(n, 256), 256, 0, st>>>(partial, grid, n, dW);
    GNNB_LAUNCHED();
    return GNNB_OK;
}

// The dense layer's whole pullback for Dout = 128, Din in {32, 64, 96, 128}: dpre = y > 0 ? dy : 0 (y non-null, relu) or
// dy, dx = dpre W, dW = dpre^T x and db = column sums of dpre (db may be null), in three launches that read dy, y and x
// once each per product and never store dpre.  dx has the bits of linear_tf32x3 on dpre and W^T, dW those of dw_tf32x3
// on dpre; GNNB_EUNSUPPORTED for anything else.  mask (non-null, y null): the relu mask linear_relu_mask_tf32x3 wrote beside
// y, read in place of y by the *_mask_kernel variants, with the same bits in every output.
int linear_bwd_tf32x3(const float* dy, const float* y, const uint32_t* mask, const float* x, const float* W, int64_t M,
                      int64_t Din, float* dx, float* dW, float* db, cudaStream_t st) {
    if (!g_tc_enabled) return GNNB_EUNSUPPORTED;
    if (Din % 32 != 0 || Din > 128 || Din < 32 || M <= 0) return GNNB_EUNSUPPORTED;
    if (((uintptr_t)dy & 15) || ((uintptr_t)y & 15) || ((uintptr_t)x & 15) || ((uintptr_t)dx & 15) || ((uintptr_t)mask & 15))
        return GNNB_EUNSUPPORTED;
    static bool configured = false;
    static int nsm = 0;
    static float *partial = nullptr, *colsum = nullptr;
    if (!configured) {
        GNNB_CUDA(cudaFuncSetAttribute(tc::linear_bwd_dx_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, tc::SMEM_TOTAL));
        GNNB_CUDA(cudaFuncSetAttribute(tcw::linear_bwd_dw_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, tcw::SMEM_TOTALW));
        GNNB_CUDA(cudaFuncSetAttribute(tc::linear_bwd_dx_mask_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, tc::SMEM_TOTAL));
        GNNB_CUDA(cudaFuncSetAttribute(tcw::linear_bwd_dw_mask_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, tcw::SMEM_TOTALW));
        int dev = 0;
        GNNB_CUDA(cudaGetDevice(&dev));
        GNNB_CUDA(cudaDeviceGetAttribute(&nsm, cudaDevAttrMultiProcessorCount, dev));
        GNNB_CUDA(cudaMalloc(&partial, sizeof(float) * (size_t)nsm * 128 * 128));
        GNNB_CUDA(cudaMalloc(&colsum, sizeof(float) * (size_t)nsm * 4 * 128));
        if (!g_tc_err) { GNNB_CUDA(cudaMalloc(&g_tc_err, sizeof(int))); GNNB_CUDA(cudaMemset(g_tc_err, 0, sizeof(int))); }
        configured = true;
    }
    // dx and the column sums of dpre: one CTA per SM over 128-row tiles
    tc::Params p;
    p.x = dy; p.w = W; p.bias = nullptr; p.addend = nullptr; p.y = dx; p.M = M; p.K = 128; p.Nout = (int)Din; p.relu = 0;
    p.ldw = 128; p.err = g_tc_err; p.wimg = nullptr; p.act = y; p.colsum = db ? colsum : nullptr;
    p.mask = const_cast<uint32_t*>(mask);
    const int64_t ntiles = ceil_div(M, tc::BM);
    const int grid_dx = (int)(ntiles < nsm ? ntiles : nsm);
    if (mask) tc::linear_bwd_dx_mask_kernel<<<grid_dx, tc::THREADS, tc::SMEM_TOTAL, st>>>(p);
    else tc::linear_bwd_dx_kernel<<<grid_dx, tc::THREADS, tc::SMEM_TOTAL, st>>>(p);
    GNNB_LAUNCHED();
    // dW: the split-K partition of dw_tf32x3
    tcw::ParamsW pw;
    pw.dpre = dy; pw.x = x; pw.partial = partial; pw.M = M; pw.Din = (int)Din; pw.err = g_tc_err; pw.act = y; pw.mask = mask;
    const int64_t rpc = ceil_div(ceil_div(M, nsm), 32) * 32;
    pw.rows_per_cta = rpc;
    const int grid_dw = (int)ceil_div(M, rpc);
    if (mask) tcw::linear_bwd_dw_mask_kernel<<<grid_dw, tc::THREADS, tcw::SMEM_TOTALW, st>>>(pw);
    else tcw::linear_bwd_dw_kernel<<<grid_dw, tc::THREADS, tcw::SMEM_TOTALW, st>>>(pw);
    GNNB_LAUNCHED();
    const int n = (int)(128 * Din);
    tcw::dw_reduce_kernel<<<(unsigned)ceil_div(n + 128, 256), 256, 0, st>>>(partial, grid_dw, n, dW, colsum, grid_dx * 4, db);
    GNNB_LAUNCHED();
    return GNNB_OK;
}

// pipeline watchdog: non-zero if a bounded mbarrier wait expired in any launch so far (then results are invalid)
int linear_tf32x3_error() {
    if (!g_tc_err) return 0;
    int e = 0;
    cudaMemcpy(&e, g_tc_err, sizeof(int), cudaMemcpyDeviceToHost);
    return e;
}

}  // namespace gnnb
