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
// shared-memory images (w_big, w_small).  Row tiles of 128 rows of X stream through a TMA ring, one 32-float K-block
// (a 32 x 128 box, SWIZZLE_128B: the raw fp32 values in the canonical K-major layout) per stage:
//   warp 0, lane 0 : cp.async.bulk.tensor.2d of each box into its stage, completed on full[stage] by complete_tx;
//                    the fused pullback's producer warps also read every stage for the column sums of db
//   warps 4-11     : two warpgroups, 64 rows of the tile each: ld.shared of the thread's A fragments, split into big and
//                    small in registers, 12 wgmma.m64n128k8.tf32 per K-block with A from registers and W from shared
//                    memory, one wgmma group kept in flight; then + bias, relu, stores straight from the accumulator
// The ring holds raw tiles only (the small image never goes to shared memory), so it is RING_BYTES = 96 KB deep: 6
// stages of 16 KB in the forward (5 of 18 KB, 3 of 32 KB in the pullback), up to 80-96 KB per SM in flight from HBM.  The producer warpgroup gives its registers to the consumers
// (setmaxnreg), which hold two accumulators and two K-blocks of A fragments.
// The kernel is HBM-bound by design (2 x 4 x K bytes per row against 6 K^2 flops on the TF32 tensor cores).
// Every mbarrier wait is bounded: a broken pipeline makes the kernel flag an error and drain instead of hanging, and the
// thread that issues the TMA copies waits (bounded) for its last ones to land before it exits (ring_drain).
#include "common.cuh"
#include "tma.cuh"
#include <cudaTypedefs.h>
#include <map>

namespace gnnb {

namespace tc {
constexpr int BM = 128;           // rows per tile (two warpgroups x wgmma M = 64)
constexpr int BK = 32;            // floats per K-block = one 128 B swizzle row
constexpr int BN = 128;           // wgmma N: W images hold 128 rows, zero beyond Nout
constexpr int PRODUCERS = 128;    // warps 0-3
constexpr int CONSUMER_WARPS = 8; // warps 4-11 = warpgroups 1 and 2
constexpr int THREADS = PRODUCERS + CONSUMER_WARPS * 32;
constexpr int KBLK_BYTES = BM * 128;          // one operand image of a K-block: 128 rows x 128 B = 16 KB
constexpr int W_BYTES = 4 * KBLK_BYTES;       // up to K = 128: 64 KB per image
constexpr int SMEM_W_BIG = 0;
constexpr int SMEM_W_SMALL = W_BYTES;
constexpr int SMEM_A = 2 * W_BYTES;           // the TMA ring: stages of raw boxes (see ring_stage_bytes)
constexpr int RING_BYTES = 6 * KBLK_BYTES;
constexpr int MAX_STAGES = 6;
constexpr int MASK_BYTES = BM * 16;           // the relu mask words of a tile, beside its dy box (linear_bwd_dx_mask_kernel)
constexpr int SMEM_BIAS = SMEM_A + RING_BYTES;
constexpr int SMEM_BAR = SMEM_BIAS + 512;
constexpr int SMEM_TOTAL = SMEM_BAR + 16 * MAX_STAGES;
constexpr int PRODUCER_REGS = 56;             // setmaxnreg: 128 x 56 + 256 x 224 <= 64 K registers
constexpr int CONSUMER_REGS = 224;
static_assert(SMEM_TOTAL <= 227 * 1024, "shared memory of the ring kernels");
static_assert(PRODUCERS * PRODUCER_REGS + CONSUMER_WARPS * 32 * CONSUMER_REGS <= 65536, "register split");

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

// as wgmma_tf32 with A (64 x 8) from registers: a[e] of thread (warp w of the warpgroup, lane l) is row 16w + l/4 + 8(e&1),
// column l%4 + 4(e>>1)
__device__ __forceinline__ void wgmma_tf32_rs(float* d, const uint32_t* a, uint64_t db, uint32_t accumulate) {
    asm volatile(
        "{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %69, 0;\n\t"
        "wgmma.mma_async.sync.aligned.m64n128k8.f32.tf32.tf32 "
        "{%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, %16, %17, %18, %19, %20, %21, %22, %23, "
        "%24, %25, %26, %27, %28, %29, %30, %31, %32, %33, %34, %35, %36, %37, %38, %39, %40, %41, %42, %43, %44, %45, %46, "
        "%47, %48, %49, %50, %51, %52, %53, %54, %55, %56, %57, %58, %59, %60, %61, %62, %63}, {%64, %65, %66, %67}, %68, p, 1, 1;\n\t}"
        : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]), "+f"(d[8]),
          "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]), "+f"(d[16]),
          "+f"(d[17]), "+f"(d[18]), "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23]), "+f"(d[24]),
          "+f"(d[25]), "+f"(d[26]), "+f"(d[27]), "+f"(d[28]), "+f"(d[29]), "+f"(d[30]), "+f"(d[31]), "+f"(d[32]),
          "+f"(d[33]), "+f"(d[34]), "+f"(d[35]), "+f"(d[36]), "+f"(d[37]), "+f"(d[38]), "+f"(d[39]), "+f"(d[40]),
          "+f"(d[41]), "+f"(d[42]), "+f"(d[43]), "+f"(d[44]), "+f"(d[45]), "+f"(d[46]), "+f"(d[47]), "+f"(d[48]),
          "+f"(d[49]), "+f"(d[50]), "+f"(d[51]), "+f"(d[52]), "+f"(d[53]), "+f"(d[54]), "+f"(d[55]), "+f"(d[56]),
          "+f"(d[57]), "+f"(d[58]), "+f"(d[59]), "+f"(d[60]), "+f"(d[61]), "+f"(d[62]), "+f"(d[63])
        : "r"(a[0]), "r"(a[1]), "r"(a[2]), "r"(a[3]), "l"(db), "r"(accumulate));
}
__device__ __forceinline__ void wgmma_wait_1() { asm volatile("wgmma.wait_group.sync.aligned 1;" ::: "memory"); }

// mma_kblock with the A fragments of the K-block in registers (ab / as: big / small, 4 per K = 8 step; dc == dm: one
// accumulator), committed as one group and not waited for: the same 12 instructions in the same order on the same operand values
__device__ __forceinline__ void mma_kblock_rs(float* dm, float* dc, const uint32_t* ab, const uint32_t* as, uint32_t b_big,
                                              uint32_t b_small, bool first) {
    wgmma_fence();
#pragma unroll
    for (int j = 0; j < 4; ++j) {
        const uint32_t o = j * 32;
        const uint32_t acc = (first && j == 0) ? 0u : 1u;
        wgmma_tf32_rs(dc, as + 4 * j, gmma_desc(b_big + o), acc);
        wgmma_tf32_rs(dc, ab + 4 * j, gmma_desc(b_small + o), 1u);
        wgmma_tf32_rs(dm, ab + 4 * j, gmma_desc(b_big + o), dm == dc ? 1u : acc);
    }
    wgmma_commit();
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

// The ring: stage s of the CTA's flattened (tile, K-block) sequence holds the K-block's raw boxes, 1024 B aligned as
// SWIZZLE_128B wants: [x or dy 16 KB] and, in the pullback, [y 16 KB] (relu from y) or [the tile's mask words 2 KB] (relu
// from the mask bits).  full[s] completes on the TMA transaction bytes, empty[s] when every warp reading it has arrived.
__host__ __device__ constexpr int ring_stage_bytes(int boxes, bool mask) { return boxes * KBLK_BYTES + (mask ? MASK_BYTES : 0); }
__host__ __device__ constexpr int ring_stages(int stage_bytes) {
    return RING_BYTES / stage_bytes < MAX_STAGES ? RING_BYTES / stage_bytes : MAX_STAGES;
}

// consumer warpgroups of the ring kernels: warpgroup wg owns rows 64 wg .. 64 wg + 63 of every tile of this CTA.  Each
// thread reads its A fragments of a K-block from the stage (rows r0, r0 + 8, columns 8 j + t, 8 j + t + 4, conflict-free
// in the swizzled layout), releases the stage, splits them into big and small and issues the K-block's 12 wgmma; the
// group of K-block i runs while the fragments of K-block i + 1 are read, so the two fragment sets alternate.
// DPRE (the dense pullback): A = dpre, from the dy box and the mask words beside it (1) or the y box (2, when p.act).
template <bool MASK_OUT, int DPRE>
__device__ __forceinline__ void consume_ring(const Params& p, unsigned char* smem, const float* sbias, int KB, int64_t ntiles,
                                             int ns, int stage_bytes) {
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    const int wg = (warp - PRODUCERS / 32) >> 2, g = lane >> 2, t = lane & 3;
    const int r0 = wg * 64 + (warp & 3) * 16 + g;
    const uint32_t sbase = s_u32(smem);
    const uint32_t bar_full = sbase + SMEM_BAR, bar_empty = bar_full + 8 * MAX_STAGES;
    const int64_t my_tiles = (ntiles > (int64_t)blockIdx.x) ? (ntiles - blockIdx.x + gridDim.x - 1) / gridDim.x : 0;
    const int64_t total = my_tiles * KB;
    float dm[64] = {}, dc[64] = {};
    uint32_t ab0[16], as0[16], ab1[16], as1[16];
    int stage = 0, kb = 0;
    uint32_t phase = 0;
    int64_t tile = blockIdx.x;
    bool alive = true;
    auto step = [&](uint32_t* ab, uint32_t* as) {
        if (!bar_wait(bar_full + 8 * stage, phase, p.err)) { alive = false; return; }
        const unsigned char* st = smem + SMEM_A + stage * stage_bytes;
        uint32_t mw[4];   // element e of a fragment: row r0 + 8 (e & 1), word (t >> 1) + 2 (e >> 1) of that row's mask
        if constexpr (DPRE == 1) {
            const uint32_t* m = reinterpret_cast<const uint32_t*>(st + KBLK_BYTES) + (t >> 1);
#pragma unroll
            for (int e = 0; e < 4; ++e) mw[e] = m[(r0 + 8 * (e & 1)) * 4 + 2 * (e >> 1)];
        }
#pragma unroll
        for (int j = 0; j < 4; ++j) {
#pragma unroll
            for (int e = 0; e < 4; ++e) {
                const int off = (r0 + 8 * (e & 1)) * 128 + (((2 * j + (e >> 1)) ^ g) << 4) + 4 * t;
                float v = *reinterpret_cast<const float*>(st + off);
                if constexpr (DPRE == 1) v = (mw[e] >> (8 * kb + 2 * j + (t & 1))) & 1u ? v : 0.f;
                if constexpr (DPRE == 2) {
                    if (p.act) v = *reinterpret_cast<const float*>(st + KBLK_BYTES + off) > 0.f ? v : 0.f;
                }
                const float b = tf32_big(v);
                ab[4 * j + e] = __float_as_uint(b);
                as[4 * j + e] = __float_as_uint(tf32_small(v, b));
            }
        }
        __syncwarp();
        if (lane == 0) bar_arrive(bar_empty + 8 * stage);   // this warp's reads of the stage are complete
        fence_acc(dm);
        fence_acc(dc);
        mma_kblock_rs(dm, dc, ab, as, sbase + SMEM_W_BIG + kb * KBLK_BYTES, sbase + SMEM_W_SMALL + kb * KBLK_BYTES, kb == 0);
        wgmma_wait_1();                                     // the previous K-block's group, and so its fragment set, is done
        if (++stage == ns) { stage = 0; phase ^= 1; }
        if (++kb == KB) {
            wgmma_wait_all();
            fence_acc(dm);
            fence_acc(dc);
            store_tile<MASK_OUT>(p, dm, dc, sbias, tile * BM + wg * 64, 0, p.Nout);
            kb = 0;
            tile += gridDim.x;
        }
    };
    for (int64_t it = 0; alive && it < total; it += 2) {
        step(ab0, as0);
        if (alive && it + 1 < total) step(ab1, as1);
    }
    wgmma_wait_all();
}

// the ring kernels' one-time setup: barriers (full: the TMA issue's arrive + bytes; empty: `readers` warps), bias
__device__ __forceinline__ void ring_init(unsigned char* smem, const float* bias, int nbias, int readers) {
    const int tid = threadIdx.x;
    if (tid == 0) {
        const uint32_t bar_full = s_u32(smem + SMEM_BAR), bar_empty = bar_full + 8 * MAX_STAGES;
        for (int s = 0; s < MAX_STAGES; ++s) { bar_init(bar_full + 8 * s, 1); bar_init(bar_empty + 8 * s, readers); }
        asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
    }
    float* sbias = reinterpret_cast<float*>(smem + SMEM_BIAS);
    for (int i = tid; i < BN; i += THREADS) sbias[i] = (bias && i < nbias) ? bias[i] : 0.f;
}

// the issuing thread's last act: wait, bounded but regardless of the error flag, until the copies of the last `issued`
// (at most ns) items have landed, so that no bulk copy into this CTA's shared memory outlives it when a broken pipeline
// made the readers stop early.  (stage, phase): the ring position the next item would have taken.
__device__ __forceinline__ void ring_drain(uint32_t bar_full, int ns, int stage, uint32_t phase, int64_t issued) {
    for (int k = 0; k < ns && k < issued; ++k) {
        if (--stage < 0) { stage = ns - 1; phase ^= 1; }
        for (uint32_t spin = 0; spin < (1u << 22) && !bar_try(bar_full + 8 * stage, phase); ++spin) {}
    }
}

// MASK: linear_relu_mask_kernel, which also writes the relu mask of y (Nout = 128, relu on)
template <bool MASK>
__device__ __forceinline__ void linear_body(const Params& p, const CUtensorMap* tm_x) {
    extern __shared__ __align__(1024) unsigned char smem[];
    const int tid = threadIdx.x, warp = tid >> 5;
    const int KB = p.K / BK;                                   // K-blocks per tile (<= 4)
    const int64_t ntiles = (p.M + BM - 1) / BM;
    const uint32_t sbase = s_u32(smem);
    constexpr int stage_bytes = ring_stage_bytes(1, false), ns = ring_stages(stage_bytes);

    // ---- one-time setup: barriers, bias, W split into the two swizzled K-major images (rows >= Nout zero)
    ring_init(smem, p.bias, p.Nout, CONSUMER_WARPS);
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
        asm volatile("setmaxnreg.dec.sync.aligned.u32 %0;" ::"n"(PRODUCER_REGS));
        if (tid != 0) return;
        // ================= one thread issues the CTA's (tile, K-block) boxes into the ring =================
        const uint32_t bar_full = sbase + SMEM_BAR, bar_empty = bar_full + 8 * MAX_STAGES;
        const int64_t my_tiles = (ntiles > (int64_t)blockIdx.x) ? (ntiles - blockIdx.x + gridDim.x - 1) / gridDim.x : 0;
        int stage = 0, kb = 0;
        uint32_t phase = 0;
        int64_t tile = blockIdx.x, it = 0;
        for (; it < my_tiles * KB; ++it) {
            if (!bar_wait(bar_empty + 8 * stage, phase ^ 1, p.err)) break;
            tma::mbar_expect_tx(bar_full + 8 * stage, KBLK_BYTES);
            tma::tensor_load_2d(sbase + SMEM_A + stage * stage_bytes, tm_x, kb * BK, (int)(tile * BM), bar_full + 8 * stage);
            if (++stage == ns) { stage = 0; phase ^= 1; }
            if (++kb == KB) { kb = 0; tile += gridDim.x; }
        }
        ring_drain(bar_full, ns, stage, phase, it);
    } else {
        asm volatile("setmaxnreg.inc.sync.aligned.u32 %0;" ::"n"(CONSUMER_REGS));
        consume_ring<MASK, 0>(p, smem, reinterpret_cast<float*>(smem + SMEM_BIAS), KB, ntiles, ns, stage_bytes);
    }
}

__global__ void __launch_bounds__(THREADS, 1) linear_tf32x3_kernel(const Params p, const __grid_constant__ CUtensorMap tm_x) {
    linear_body<false>(p, &tm_x);
}
__global__ void __launch_bounds__(THREADS, 1) linear_relu_mask_kernel(const Params p, const __grid_constant__ CUtensorMap tm_x) {
    linear_body<true>(p, &tm_x);
}

// dx = dpre * W for dpre = relu ? (y > 0 ? dy : 0) : dy, Dout = 128 rows of W and Din = Nout <= 128 columns.  The
// consumers form dpre from the dy box and the relu source in their stage (y, or the mask words) in registers, so dpre is
// never stored; the four producer warps read the same stages for the column sums of db.  Tiles, images and the MMA
// sequence are those of linear_tf32x3_kernel run on a transposed copy of W with a zero bias, so dx has the same bits as
// that composition; W is read transposed straight into the images instead.
// MASK: linear_bwd_dx_mask_kernel, which reads the relu mask bits (p.mask, always on) in place of y: the same dpre, from
// 16 B per row instead of 512.
template <bool MASK>
__device__ __forceinline__ void bwd_dx_body(const Params& p, const CUtensorMap* tm_dy, const CUtensorMap* tm_y) {
    extern __shared__ __align__(1024) unsigned char smem[];
    const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
    const int64_t ntiles = (p.M + BM - 1) / BM;
    const uint32_t sbase = s_u32(smem);
    const int boxes = (!MASK && p.act) ? 2 : 1;
    const int stage_bytes = ring_stage_bytes(boxes, MASK), ns = ring_stages(stage_bytes);

    ring_init(smem, nullptr, 0, CONSUMER_WARPS + PRODUCERS / 32);   // (dm + dc) + 0: a -0 sum stores as +0, as in the composition
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
        asm volatile("setmaxnreg.dec.sync.aligned.u32 %0;" ::"n"(PRODUCER_REGS));
        // ================= producers: K = 128, so a tile is 4 K-blocks.  Thread 0 issues the boxes ns - 1 items ahead of
        // the item the four warps read; each warp reads 32 rows x 128 B of every stage for the column sums.
        const uint32_t bar_full = sbase + SMEM_BAR, bar_empty = bar_full + 8 * MAX_STAGES;
        const int c = tid & 7, r16 = tid >> 3, rr = r16 & 7;
        const int64_t my_tiles = (ntiles > (int64_t)blockIdx.x) ? (ntiles - blockIdx.x + gridDim.x - 1) / gridDim.x : 0;
        const int64_t total = my_tiles * 4;
        int i_stage = 0, i_kb = 0;
        uint32_t i_phase = 0;
        int64_t i_tile = blockIdx.x;
        bool issuing = true;
        auto issue = [&]() {
            if (!issuing) return;
            if (!bar_wait(bar_empty + 8 * i_stage, i_phase ^ 1, p.err)) { issuing = false; return; }
            {
                const uint32_t dst = sbase + SMEM_A + i_stage * stage_bytes, full = bar_full + 8 * i_stage;
                const int64_t nr = (p.M - i_tile * BM < BM) ? p.M - i_tile * BM : BM;
                tma::mbar_expect_tx(full, boxes * KBLK_BYTES + (MASK ? (uint32_t)nr * 16 : 0u));
                tma::tensor_load_2d(dst, tm_dy, i_kb * BK, (int)(i_tile * BM), full);
                if (boxes == 2) tma::tensor_load_2d(dst + KBLK_BYTES, tm_y, i_kb * BK, (int)(i_tile * BM), full);
                if (MASK) tma::bulk_load(dst + KBLK_BYTES, p.mask + (size_t)i_tile * BM * 4, (uint32_t)nr * 16, full);
            }
            if (++i_stage == ns) { i_stage = 0; i_phase ^= 1; }
            if (++i_kb == 4) { i_kb = 0; i_tile += gridDim.x; }
        };
        if (tid == 0)
            for (int64_t n = 0; n < ns - 1 && n < total; ++n) issue();
        // column sums of dpre: after each item the 4 threads of a warp that share a column group add theirs in a fixed
        // order, and lanes 8 kb .. 8 kb + 7 keep the sums of K-block kb (columns 32 kb + 4 c .. + 3)
        const float4 zero = make_float4(0.f, 0.f, 0.f, 0.f);
        float4 cs = zero;
        int stage = 0;
        uint32_t phase = 0;
        for (int64_t it = 0; it < total; ++it) {
            const int kb = (int)(it & 3);
            if (tid == 0 && it + ns - 1 < total) issue();
            if (!bar_wait(bar_full + 8 * stage, phase, p.err)) break;
            if (p.colsum) {
                // the thread's 4 columns of rows r16 + 16 i; dpre = act ? (act > 0 ? dy : 0) : dy, with the relu source
                // the mask bits 8 kb + 2 (c >> 1) and the next of words 2 (c & 1) and 2 (c & 1) + 1 of the row (MASK)
                const unsigned char* st = smem + SMEM_A + stage * stage_bytes;
                float4 s = zero;
#pragma unroll
                for (int i = 0; i < 8; ++i) {
                    const int off = ((r16 >> 3) + 2 * i) * 1024 + rr * 128 + ((c ^ rr) << 4);
                    float4 g = *reinterpret_cast<const float4*>(st + off);
                    if constexpr (MASK) {
                        const uint2 m = *reinterpret_cast<const uint2*>(st + KBLK_BYTES + (r16 + 16 * i) * 16 + (c & 1) * 8);
                        const int sh = 8 * kb + 2 * (c >> 1);
                        g.x = (m.x >> sh) & 1u ? g.x : 0.f; g.y = (m.x >> (sh + 1)) & 1u ? g.y : 0.f;
                        g.z = (m.y >> sh) & 1u ? g.z : 0.f; g.w = (m.y >> (sh + 1)) & 1u ? g.w : 0.f;
                    } else if (boxes == 2) {
                        const float4 m = *reinterpret_cast<const float4*>(st + KBLK_BYTES + off);
                        g.x = m.x > 0.f ? g.x : 0.f; g.y = m.y > 0.f ? g.y : 0.f;
                        g.z = m.z > 0.f ? g.z : 0.f; g.w = m.w > 0.f ? g.w : 0.f;
                    }
                    s.x += g.x; s.y += g.y; s.z += g.z; s.w += g.w;
                }
#pragma unroll
                for (int o = 8; o <= 16; o <<= 1) {
                    s.x += __shfl_xor_sync(0xffffffffu, s.x, o); s.y += __shfl_xor_sync(0xffffffffu, s.y, o);
                    s.z += __shfl_xor_sync(0xffffffffu, s.z, o); s.w += __shfl_xor_sync(0xffffffffu, s.w, o);
                }
                if ((lane >> 3) == kb) { cs.x += s.x; cs.y += s.y; cs.z += s.z; cs.w += s.w; }
            }
            __syncwarp();
            if (lane == 0) bar_arrive(bar_empty + 8 * stage);
            if (++stage == ns) { stage = 0; phase ^= 1; }
        }
        if (tid == 0) ring_drain(bar_full, ns, i_stage, i_phase, (i_tile - blockIdx.x) / gridDim.x * 4 + i_kb);
        if (p.colsum) reinterpret_cast<float4*>(p.colsum + ((size_t)blockIdx.x * 4 + warp) * 128 + (lane >> 3) * BK)[c] = cs;
    } else {
        asm volatile("setmaxnreg.inc.sync.aligned.u32 %0;" ::"n"(CONSUMER_REGS));
        consume_ring<false, MASK ? 1 : 2>(p, smem, reinterpret_cast<float*>(smem + SMEM_BIAS), 128 / BK, ntiles, ns, stage_bytes);
    }
}

__global__ void __launch_bounds__(THREADS, 1) linear_bwd_dx_kernel(const Params p, const __grid_constant__ CUtensorMap tm_dy,
                                                                   const __grid_constant__ CUtensorMap tm_y) {
    bwd_dx_body<false>(p, &tm_dy, &tm_y);
}
__global__ void __launch_bounds__(THREADS, 1) linear_bwd_dx_mask_kernel(const Params p, const __grid_constant__ CUtensorMap tm_dy,
                                                                        const __grid_constant__ CUtensorMap tm_y) {
    bwd_dx_body<true>(p, &tm_dy, &tm_y);
}
}  // namespace tc

// =====================================================================================================================
// dW = dPre^T * X  (the weight pullback of the dense layer):  dW[i][j] = sum_r dPre[r][i] * X[r][j],  r over all N rows.
// Both operands are "MN-major" in memory (the reduction index r is the slow one) and tf32 wgmma reads K-major operands
// only.  A block of 32 rows r is a K-block.  One thread drops its row-major tiles into a TMA ring (boxes of 32 columns x
// 32 rows, SWIZZLE_128B): dy (or dpre) as 4 boxes, y as 4 more in linear_bwd_dw_kernel, X as Din / 32 boxes, and the
// rows' relu mask words (32 x 16 B, 1-D bulk copy) in linear_bwd_dw_mask_kernel.
//   A = dPre^T (128 rows i): each consumer thread reads its fragments (rows i, columns r) straight from the dy box, forms
//       dpre, splits it into big and small in registers and issues wgmma with A from registers, as the forward kernel;
//   B = X^T (Din rows j, zero up to 128): the four producer warps transpose the X boxes into a double-buffered K-major
//       SWIZZLE_128B image, big and small: lane l of a warp reads column j = 32 jb + l of 4 rows (conflict-free in the
//       swizzled box) and stores the split float4 of those 4 rows k into row j of the image (one 16 B vector per image).
// One wgmma group stays in flight; the B slot of block n - 1 is released once its group has retired.
// Split-K: every CTA reduces a contiguous range of rows into its own register accumulators and writes a (128 x Din)
// partial; a second kernel adds the partials in CTA order (deterministic).
// The accumulation chain is cut every FLUSH row blocks and each short chain is added into an fp32 register sum with
// ordinary round-to-nearest adds, so the length of the tensor core's accumulation chain does not grow with N.
// =====================================================================================================================
namespace tcw {
using namespace tc;
constexpr int FLUSH = 4;                      // row blocks (of 32 rows) per accumulation chain
constexpr int BOX_BYTES = 32 * 128;           // one box: 32 rows x 32 floats
constexpr int RINGW_BYTES = 160 * 1024;       // stages: [dy 16 KB][y 16 KB, linear_bwd_dw_kernel with y][X <= 16 KB][mask 512 B]
constexpr int MAX_WSTAGES = 4;
constexpr int SMEM_BIMG = RINGW_BYTES;        // 2 slots x [X^T big 16 KB][X^T small 16 KB]
constexpr int SMEM_BARW = SMEM_BIMG + 4 * KBLK_BYTES;
constexpr int SMEM_TOTALW = SMEM_BARW + 8 * (2 * MAX_WSTAGES + 4);
static_assert(SMEM_TOTALW <= 227 * 1024, "shared memory of the dW kernels");

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

// byte offset of element (row n, k) of a K-major SWIZZLE_128B image, k < 32
__device__ __forceinline__ int kmajor_off(int n, int k) {
    return (n >> 3) * 1024 + (n & 7) * 128 + ((((k >> 2) ^ (n & 7))) << 4) + (k & 3) * 4;
}
// byte offset of element (row r < 32, column c) of a row-major tile stored as 32-column SWIZZLE_128B boxes
__device__ __forceinline__ int box_off(int r, int c) {
    return (c >> 5) * BOX_BYTES + r * 128 + ((((c & 31) >> 2) ^ (r & 7)) << 4) + (c & 3) * 4;
}

// DPRE: 0 dpre = p.dpre as it is (dw_tf32x3_kernel); 1 dpre from dy and the mask bits (linear_bwd_dw_mask_kernel);
// 2 dpre from dy and y when p.act, else dy (linear_bwd_dw_kernel)
template <int DPRE>
__device__ __forceinline__ void dw_body(const ParamsW& p, const CUtensorMap* tm_dy, const CUtensorMap* tm_y,
                                        const CUtensorMap* tm_x) {
    extern __shared__ __align__(1024) unsigned char smem[];
    const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
    const uint32_t sbase = s_u32(smem);
    const uint32_t bar_full = sbase + SMEM_BARW, bar_empty = bar_full + 8 * MAX_WSTAGES;
    const uint32_t bar_bfull = bar_empty + 8 * MAX_WSTAGES, bar_bempty = bar_bfull + 16;
    const bool with_y = DPRE == 2 && p.act;
    const int x_at = (with_y ? 8 : 4) * BOX_BYTES, mask_at = x_at + 4 * BOX_BYTES;
    const int stage_bytes = mask_at + 1024, ns = RINGW_BYTES / stage_bytes < MAX_WSTAGES ? RINGW_BYTES / stage_bytes : MAX_WSTAGES;
    const int xboxes = p.Din >> 5;
    const int64_t r_begin = (int64_t)blockIdx.x * p.rows_per_cta;
    const int64_t r_end = (r_begin + p.rows_per_cta < p.M) ? r_begin + p.rows_per_cta : p.M;
    const int64_t nblk = (r_end > r_begin) ? (r_end - r_begin + 31) / 32 : 0;

    if (tid == 0) {
        for (int s = 0; s < MAX_WSTAGES; ++s) { bar_init(bar_full + 8 * s, 1); bar_init(bar_empty + 8 * s, CONSUMER_WARPS + 4); }
        for (int s = 0; s < 2; ++s) { bar_init(bar_bfull + 8 * s, 4); bar_init(bar_bempty + 8 * s, CONSUMER_WARPS); }
        asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
    }
    // rows j >= Din of the X^T images are never written: zero them once
    for (int i = tid; i < 4 * KBLK_BYTES / 16; i += THREADS)
        reinterpret_cast<float4*>(smem + SMEM_BIMG)[i] = make_float4(0.f, 0.f, 0.f, 0.f);
    fence_proxy_async();
    __syncthreads();

    if (warp < PRODUCERS / 32) {
        asm volatile("setmaxnreg.dec.sync.aligned.u32 %0;" ::"n"(PRODUCER_REGS));
        // ---- producers: thread 0 issues the boxes ns - 1 blocks ahead; the four warps transpose X into the B slots
        int i_stage = 0;
        uint32_t i_phase = 0;
        int64_t i_blk = 0;
        bool issuing = true;
        auto issue = [&]() {
            if (!issuing) return;
            if (!bar_wait(bar_empty + 8 * i_stage, i_phase ^ 1, p.err)) { issuing = false; return; }
            {
                const uint32_t dst = sbase + i_stage * stage_bytes, full = bar_full + 8 * i_stage;
                const int64_t r0 = r_begin + 32 * i_blk;
                const uint32_t nr = (uint32_t)((r_end - r0 < 32) ? r_end - r0 : 32);
                tma::mbar_expect_tx(full, (uint32_t)(((with_y ? 8 : 4) + xboxes) * BOX_BYTES) + (DPRE == 1 ? nr * 16 : 0u));
                for (int b = 0; b < 4; ++b) tma::tensor_load_2d(dst + b * BOX_BYTES, tm_dy, 32 * b, (int)r0, full);
                if (with_y)
                    for (int b = 0; b < 4; ++b) tma::tensor_load_2d(dst + (4 + b) * BOX_BYTES, tm_y, 32 * b, (int)r0, full);
                for (int b = 0; b < xboxes; ++b) tma::tensor_load_2d(dst + x_at + b * BOX_BYTES, tm_x, 32 * b, (int)r0, full);
                if (DPRE == 1) tma::bulk_load(dst + mask_at, p.mask + (size_t)r0 * 4, nr * 16, full);
            }
            if (++i_stage == ns) { i_stage = 0; i_phase ^= 1; }
            ++i_blk;
        };
        if (tid == 0)
            for (int64_t n = 0; n < ns - 1 && n < nblk; ++n) issue();
        int stage = 0;
        uint32_t phase = 0;
        for (int64_t blk = 0; blk < nblk; ++blk) {
            if (tid == 0 && blk + ns - 1 < nblk) issue();
            const int slot = (int)(blk & 1);
            if (!bar_wait(bar_full + 8 * stage, phase, p.err)) break;
            if (!bar_wait(bar_bempty + 8 * slot, (uint32_t)(((blk >> 1) & 1) ^ 1), p.err)) break;
            const unsigned char* sx = smem + stage * stage_bytes + x_at;
            unsigned char* big = smem + SMEM_BIMG + slot * 2 * KBLK_BYTES;
            // items (jb, q) = (32-column group of X, 4 rows k = 4 q .. 4 q + 3), spread over the warps
            for (int item = warp; item < xboxes * 8; item += 4) {
                const int j = 32 * (item >> 3) + lane, q = item & 7;
                float4 v;
                v.x = *reinterpret_cast<const float*>(sx + box_off(4 * q, j));
                v.y = *reinterpret_cast<const float*>(sx + box_off(4 * q + 1, j));
                v.z = *reinterpret_cast<const float*>(sx + box_off(4 * q + 2, j));
                v.w = *reinterpret_cast<const float*>(sx + box_off(4 * q + 3, j));
                const float4 b = make_float4(tf32_big(v.x), tf32_big(v.y), tf32_big(v.z), tf32_big(v.w));
                const int off = kmajor_off(j, 4 * q);
                *reinterpret_cast<float4*>(big + off) = b;
                *reinterpret_cast<float4*>(big + KBLK_BYTES + off) = tf32_small(v, b);
            }
            fence_proxy_async();                               // the image is read by the tensor core (async proxy)
            __syncwarp();
            if (lane == 0) { bar_arrive(bar_bfull + 8 * slot); bar_arrive(bar_empty + 8 * stage); }
            if (++stage == ns) { stage = 0; phase ^= 1; }
        }
        if (tid == 0) ring_drain(bar_full, ns, i_stage, i_phase, i_blk);
    } else {
        asm volatile("setmaxnreg.inc.sync.aligned.u32 %0;" ::"n"(CONSUMER_REGS));
        // ---- consumers: warpgroup wg owns rows 64 wg .. 64 wg + 63 of dW (M = 128), N = Din (padded to 128)
        const int wg = (warp - PRODUCERS / 32) >> 2, g = lane >> 2, t = lane & 3;
        const int i0 = wg * 64 + (warp & 3) * 16 + g;          // the thread's rows i0 and i0 + 8 of dW
        // relu mask of (r, i0 + 8 h): bit 2 (i >> 3) + (i & 1) of word (i >> 1) & 3, the same word for both rows
        const int mword = (i0 >> 1) & 3, mbit = 2 * (i0 >> 3) + (i0 & 1);
        float acc[64] = {}, sum[64];
        uint32_t ab0[16], as0[16], ab1[16], as1[16];
#pragma unroll
        for (int i = 0; i < 64; ++i) sum[i] = 0.f;
        int stage = 0;
        uint32_t phase = 0;
        int64_t blk = 0;
        bool alive = true;
        auto step = [&](uint32_t* ab, uint32_t* as) {
            const int slot = (int)(blk & 1);
            if (!bar_wait(bar_full + 8 * stage, phase, p.err)) { alive = false; return; }
            const unsigned char* st = smem + stage * stage_bytes;
#pragma unroll
            for (int j = 0; j < 4; ++j) {
#pragma unroll
                for (int kh = 0; kh < 2; ++kh) {
                    const int r = 8 * j + t + 4 * kh;
                    uint32_t m = 0;
                    if constexpr (DPRE == 1) m = *reinterpret_cast<const uint32_t*>(st + mask_at + r * 16 + mword * 4);
#pragma unroll
                    for (int h = 0; h < 2; ++h) {
                        const int e = h + 2 * kh;               // fragment element: row i0 + 8 h, column r
                        const int off = box_off(r, i0 + 8 * h);
                        float v = *reinterpret_cast<const float*>(st + off);
                        if constexpr (DPRE == 1) v = (m >> (mbit + 2 * h)) & 1u ? v : 0.f;
                        if constexpr (DPRE == 2) {
                            if (with_y) v = *reinterpret_cast<const float*>(st + 4 * BOX_BYTES + off) > 0.f ? v : 0.f;
                        }
                        const float b = tf32_big(v);
                        ab[4 * j + e] = __float_as_uint(b);
                        as[4 * j + e] = __float_as_uint(tf32_small(v, b));
                    }
                }
            }
            __syncwarp();
            if (lane == 0) bar_arrive(bar_empty + 8 * stage);
            if (!bar_wait(bar_bfull + 8 * slot, (uint32_t)((blk >> 1) & 1), p.err)) { alive = false; return; }
            const uint32_t b_big = sbase + SMEM_BIMG + slot * 2 * KBLK_BYTES;
            fence_acc(acc);
            mma_kblock_rs(acc, acc, ab, as, b_big, b_big + KBLK_BYTES, (blk % FLUSH) == 0);
            wgmma_wait_1();                                     // block blk - 1 has retired: its B slot is free
            if (lane == 0 && blk > 0) bar_arrive(bar_bempty + 8 * (slot ^ 1));
            if ((blk % FLUSH) == FLUSH - 1 || blk == nblk - 1) {
                wgmma_wait_all();
                fence_acc(acc);
#pragma unroll
                for (int i = 0; i < 64; ++i) sum[i] += acc[i];
            }
            if (++stage == ns) { stage = 0; phase ^= 1; }
            ++blk;
        };
        while (alive && blk < nblk) {
            step(ab0, as0);
            if (alive && blk < nblk) step(ab1, as1);
        }
        wgmma_wait_all();
        if (!alive) return;
        const int w4 = warp & 3;
        const int i1 = wg * 64 + w4 * 16 + (lane >> 2);
#pragma unroll
        for (int j = 0; j < BN / 8; ++j) {
            const int c = 8 * j + 2 * (lane & 3);
            if (c >= p.Din) continue;
#pragma unroll
            for (int h = 0; h < 2; ++h) {
                float* prow = p.partial + ((size_t)blockIdx.x * 128 + i1 + 8 * h) * p.Din;
                *reinterpret_cast<float2*>(prow + c) = make_float2(sum[4 * j + 2 * h], sum[4 * j + 2 * h + 1]);
            }
        }
    }
}

#define GNNB_DW_PARAMS const ParamsW p, const __grid_constant__ CUtensorMap tm_dy, const __grid_constant__ CUtensorMap tm_y, \
                       const __grid_constant__ CUtensorMap tm_x
__global__ void __launch_bounds__(THREADS, 1) dw_tf32x3_kernel(GNNB_DW_PARAMS) { dw_body<0>(p, &tm_dy, &tm_y, &tm_x); }
__global__ void __launch_bounds__(THREADS, 1) linear_bwd_dw_kernel(GNNB_DW_PARAMS) { dw_body<2>(p, &tm_dy, &tm_y, &tm_x); }
__global__ void __launch_bounds__(THREADS, 1) linear_bwd_dw_mask_kernel(GNNB_DW_PARAMS) { dw_body<1>(p, &tm_dy, &tm_y, &tm_x); }
#undef GNNB_DW_PARAMS

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
// the longest K: the big*big chain of K/8 accumulations on the tensor core's accumulator drifts with K, and at K = 1024 with
// all-positive operands (2048 with any) it left the normwise 5e-6 of float64 on an H100; longer K goes to the library GEMM
constexpr int MAX_K = 512;
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

int g_tc_enabled = 1;

static std::mutex g_states_mu;
static std::map<int, DeviceState> g_states;   // by device ordinal; never erased, so a returned pointer stays valid

int device_state(DeviceState** out) {
    int dev = 0;
    GNNB_CUDA(cudaGetDevice(&dev));
    std::lock_guard<std::mutex> lock(g_states_mu);
    auto it = g_states.find(dev);
    if (it == g_states.end()) {
        // the >48 KB dynamic shared memory of the tensor-core kernels is a per-device function attribute
        GNNB_CUDA(cudaFuncSetAttribute(tc::linear_tf32x3_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, tc::SMEM_TOTAL));
        GNNB_CUDA(cudaFuncSetAttribute(tc::linear_relu_mask_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, tc::SMEM_TOTAL));
        GNNB_CUDA(cudaFuncSetAttribute(tcx::linear_wide_tf32x3_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, tcx::SMEM_TOTAL_X));
        GNNB_CUDA(cudaFuncSetAttribute(tcw::dw_tf32x3_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, tcw::SMEM_TOTALW));
        GNNB_CUDA(cudaFuncSetAttribute(tc::linear_bwd_dx_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, tc::SMEM_TOTAL));
        GNNB_CUDA(cudaFuncSetAttribute(tcw::linear_bwd_dw_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, tcw::SMEM_TOTALW));
        GNNB_CUDA(cudaFuncSetAttribute(tc::linear_bwd_dx_mask_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, tc::SMEM_TOTAL));
        GNNB_CUDA(cudaFuncSetAttribute(tcw::linear_bwd_dw_mask_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, tcw::SMEM_TOTALW));
        DeviceState s;
        GNNB_CUDA(cudaDeviceGetAttribute(&s.nsm, cudaDevAttrMultiProcessorCount, dev));
        DeviceScratch sc;
        GNNB_TRY(sc.alloc(&s.tc_err, 1));
        GNNB_CUDA(cudaMemset(s.tc_err, 0, sizeof(int)));
        sc.release(s.tc_err);
        it = g_states.emplace(dev, s).first;
    }
    *out = &it->second;
    return GNNB_OK;
}

// returns GNNB_EUNSUPPORTED (no error text) when the shape is not covered by the tensor-core kernel
int linear_tf32x3_ex(const float* x, const float* W, int64_t ldw, const float* bias, const float* addend, int relu, int64_t M,
                     int64_t K, int64_t Nout, float* y, cudaStream_t st);
int linear_tf32x3(const float* x, const float* W, const float* bias, int relu, int64_t M, int64_t K, int64_t Nout, float* y,
                  cudaStream_t st) {
    return linear_tf32x3_ex(x, W, K, bias, nullptr, relu, M, K, Nout, y, st);
}
static int linear_launch(const float* x, const float* W, int64_t ldw, const float* bias, const float* addend, int relu,
                         int64_t M, int64_t K, int64_t Nout, float* y, uint32_t* mask, cudaStream_t st);

// the tensor map of a row-major fp32 matrix (rows x cols, rows ld floats apart) in the ring kernels' boxes: 32 columns
// (one K-block) x box_rows rows (tc::BM; 32 for the dW kernels' row blocks), SWIZZLE_128B.  Encoded per call on the host; it travels as a kernel parameter.
static int kblock_map(CUtensorMap* m, const float* base, int64_t rows, int64_t cols, int64_t ld, int box_rows = tc::BM) {
    static const PFN_cuTensorMapEncodeTiled_v12000 encode = [] {
        void* fn = nullptr;
        cudaDriverEntryPointQueryResult q;
        if (cudaGetDriverEntryPointByVersion("cuTensorMapEncodeTiled", &fn, 12000, cudaEnableDefault, &q) != cudaSuccess ||
            q != cudaDriverEntryPointSuccess)
            fn = nullptr;
        return reinterpret_cast<PFN_cuTensorMapEncodeTiled_v12000>(fn);
    }();
    if (!encode) GNNB_FAIL(GNNB_ECUDA, "the driver does not provide cuTensorMapEncodeTiled");
    // a driver call needs the device's context current in this thread (an autograd worker may not have it yet)
    int dev = 0;
    GNNB_CUDA(cudaGetDevice(&dev));
    GNNB_CUDA(cudaSetDevice(dev));
    const cuuint64_t dims[2] = {(cuuint64_t)cols, (cuuint64_t)rows};
    const cuuint64_t strides[1] = {(cuuint64_t)ld * sizeof(float)};
    const cuuint32_t box[2] = {(cuuint32_t)tc::BK, (cuuint32_t)box_rows}, estride[2] = {1, 1};
    const CUresult r = encode(m, CU_TENSOR_MAP_DATA_TYPE_FLOAT32, 2, const_cast<float*>(base), dims, strides, box, estride,
                              CU_TENSOR_MAP_INTERLEAVE_NONE, CU_TENSOR_MAP_SWIZZLE_128B, CU_TENSOR_MAP_L2_PROMOTION_L2_256B,
                              CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
    if (r != CUDA_SUCCESS) GNNB_FAIL(GNNB_ECUDA, "cuTensorMapEncodeTiled failed (CUresult %d)", (int)r);
    return GNNB_OK;
}
// the ring kernels address rows by a 32-bit box coordinate
constexpr int64_t RING_MAX_ROWS = (int64_t)INT32_MAX - tc::BM;
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
        if (K % 32 != 0 || K > tcx::MAX_K || Nout % 128 != 0 || Nout > tcx::MAX_NOUT || ldw % 4 != 0 || ldw < K || M < 2048) return GNNB_EUNSUPPORTED;
    } else if (K % 32 != 0 || Nout % 16 != 0 || Nout < 16 || ldw % 4 != 0 || ldw < K || M > RING_MAX_ROWS) {
        return GNNB_EUNSUPPORTED;
    }
    if (((uintptr_t)x & 15) || ((uintptr_t)W & 15) || ((uintptr_t)y & 15) || ((uintptr_t)addend & 15)) return GNNB_EUNSUPPORTED;
    if (M == 0) return GNNB_OK;
    DeviceState* s = nullptr;
    GNNB_TRY(device_state(&s));
    tc::Params p;
    p.x = x; p.w = W; p.bias = bias; p.addend = addend; p.y = y; p.M = M; p.K = (int)K; p.Nout = (int)Nout; p.relu = relu;
    p.ldw = (int)ldw; p.err = s->tc_err; p.wimg = nullptr; p.act = nullptr; p.colsum = nullptr; p.mask = mask;
    if (wide) {
        // the split, swizzled image of W (2 x its size), rebuilt per call: W changes between training steps
        GNNB_TRY(grow_buffer(&s->wimg, &s->wimg_bytes, sizeof(float) * (size_t)2 * K * Nout));
        tcx::w_image_kernel<<<(unsigned)ceil_div(Nout * (K / 4), 256), 256, 0, st>>>(W, (int)ldw, (int)K, (int)Nout, s->wimg);
        GNNB_LAUNCHED();
        p.wimg = s->wimg;
    }
    const int nsm = s->nsm;
    const int64_t ntiles = ceil_div(M, tc::BM);
    const unsigned grid = (unsigned)(ntiles < nsm ? ntiles : nsm);
    if (wide) {
        tcx::linear_wide_tf32x3_kernel<<<grid, tc::THREADS, tcx::SMEM_TOTAL_X, st>>>(p);
    } else {
        CUtensorMap tm_x;
        GNNB_TRY(kblock_map(&tm_x, x, M, K, K));
        if (mask) tc::linear_relu_mask_kernel<<<grid, tc::THREADS, tc::SMEM_TOTAL, st>>>(p, tm_x);
        else tc::linear_tf32x3_kernel<<<grid, tc::THREADS, tc::SMEM_TOTAL, st>>>(p, tm_x);
    }
    GNNB_LAUNCHED();
    return GNNB_OK;
}

// dW (Dout = 128, Din in {32, 64, 96, 128}); GNNB_EUNSUPPORTED for anything else
int dw_tf32x3(const float* dpre, const float* x, int64_t M, int64_t Din, int64_t Dout, float* dW, cudaStream_t st) {
    if (!g_tc_enabled) return GNNB_EUNSUPPORTED;
    if (Dout != 128 || Din % 32 != 0 || Din > 128 || Din < 32 || M > RING_MAX_ROWS) return GNNB_EUNSUPPORTED;
    if (((uintptr_t)dpre & 15) || ((uintptr_t)x & 15) || ((uintptr_t)dW & 15)) return GNNB_EUNSUPPORTED;
    DeviceState* s = nullptr;
    GNNB_TRY(device_state(&s));
    const int nsm = s->nsm;
    GNNB_TRY(grow_buffer(&s->dw_part, &s->dw_part_bytes, sizeof(float) * (size_t)nsm * 128 * 128));
    float* partial = s->dw_part;
    if (M == 0) { GNNB_CUDA(cudaMemsetAsync(dW, 0, sizeof(float) * (size_t)(Dout * Din), st)); return GNNB_OK; }
    tcw::ParamsW p;
    p.dpre = dpre; p.x = x; p.partial = partial; p.M = M; p.Din = (int)Din; p.err = s->tc_err; p.act = nullptr; p.mask = nullptr;
    int64_t rpc = ceil_div(M, nsm);
    rpc = ceil_div(rpc, 32) * 32;
    p.rows_per_cta = rpc;
    const int grid = (int)ceil_div(M, rpc);
    CUtensorMap tm_dy, tm_x;
    GNNB_TRY(kblock_map(&tm_dy, dpre, M, 128, 128, 32));
    GNNB_TRY(kblock_map(&tm_x, x, M, Din, Din, 32));
    tcw::dw_tf32x3_kernel<<<grid, tc::THREADS, tcw::SMEM_TOTALW, st>>>(p, tm_dy, tm_dy, tm_x);
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
    if (Din % 32 != 0 || Din > 128 || Din < 32 || M <= 0 || M > RING_MAX_ROWS) return GNNB_EUNSUPPORTED;
    if (((uintptr_t)dy & 15) || ((uintptr_t)y & 15) || ((uintptr_t)x & 15) || ((uintptr_t)dx & 15) || ((uintptr_t)mask & 15))
        return GNNB_EUNSUPPORTED;
    DeviceState* s = nullptr;
    GNNB_TRY(device_state(&s));
    const int nsm = s->nsm;
    GNNB_TRY(grow_buffer(&s->bwd_part, &s->bwd_part_bytes, sizeof(float) * (size_t)nsm * 128 * 128));
    GNNB_TRY(grow_buffer(&s->bwd_colsum, &s->bwd_colsum_bytes, sizeof(float) * (size_t)nsm * 4 * 128));
    float *partial = s->bwd_part, *colsum = s->bwd_colsum;
    // dx and the column sums of dpre: one CTA per SM over 128-row tiles
    tc::Params p;
    p.x = dy; p.w = W; p.bias = nullptr; p.addend = nullptr; p.y = dx; p.M = M; p.K = 128; p.Nout = (int)Din; p.relu = 0;
    p.ldw = 128; p.err = s->tc_err; p.wimg = nullptr; p.act = y; p.colsum = db ? colsum : nullptr;
    p.mask = const_cast<uint32_t*>(mask);
    const int64_t ntiles = ceil_div(M, tc::BM);
    const int grid_dx = (int)(ntiles < nsm ? ntiles : nsm);
    CUtensorMap tm_dy, tm_y;
    GNNB_TRY(kblock_map(&tm_dy, dy, M, 128, 128));
    GNNB_TRY(kblock_map(&tm_y, (y && !mask) ? y : dy, M, 128, 128));
    if (mask) tc::linear_bwd_dx_mask_kernel<<<grid_dx, tc::THREADS, tc::SMEM_TOTAL, st>>>(p, tm_dy, tm_y);
    else tc::linear_bwd_dx_kernel<<<grid_dx, tc::THREADS, tc::SMEM_TOTAL, st>>>(p, tm_dy, tm_y);
    GNNB_LAUNCHED();
    // dW: the split-K partition of dw_tf32x3
    tcw::ParamsW pw;
    pw.dpre = dy; pw.x = x; pw.partial = partial; pw.M = M; pw.Din = (int)Din; pw.err = s->tc_err; pw.act = y; pw.mask = mask;
    const int64_t rpc = ceil_div(ceil_div(M, nsm), 32) * 32;
    pw.rows_per_cta = rpc;
    const int grid_dw = (int)ceil_div(M, rpc);
    CUtensorMap tw_dy, tw_y, tw_x;
    GNNB_TRY(kblock_map(&tw_dy, dy, M, 128, 128, 32));
    GNNB_TRY(kblock_map(&tw_y, (y && !mask) ? y : dy, M, 128, 128, 32));
    GNNB_TRY(kblock_map(&tw_x, x, M, Din, Din, 32));
    if (mask) tcw::linear_bwd_dw_mask_kernel<<<grid_dw, tc::THREADS, tcw::SMEM_TOTALW, st>>>(pw, tw_dy, tw_y, tw_x);
    else tcw::linear_bwd_dw_kernel<<<grid_dw, tc::THREADS, tcw::SMEM_TOTALW, st>>>(pw, tw_dy, tw_y, tw_x);
    GNNB_LAUNCHED();
    const int n = (int)(128 * Din);
    tcw::dw_reduce_kernel<<<(unsigned)ceil_div(n + 128, 256), 256, 0, st>>>(partial, grid_dw, n, dW, colsum, grid_dx * 4, db);
    GNNB_LAUNCHED();
    return GNNB_OK;
}

// pipeline watchdog: non-zero if a bounded mbarrier wait expired in any launch so far, on any device (then results are
// invalid)
int linear_tf32x3_error() {
    std::lock_guard<std::mutex> lock(g_states_mu);
    for (const auto& kv : g_states) {
        int e = 0;
        cudaMemcpy(&e, kv.second.tc_err, sizeof(int), cudaMemcpyDeviceToHost);
        if (e) return e;
    }
    return 0;
}

}  // namespace gnnb
