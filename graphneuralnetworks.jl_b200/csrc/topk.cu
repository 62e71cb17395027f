// topk.cu — top-k pooling on the device: the per-graph selection of topk_index and the score, gate and pullback of
// topk_pool (GNNlib/src/layers/pool.jl:14-27, Graph U-Nets' gPool).
//
// Selection (gnnb_topk_keep).  keep[i] = key_i >= v_s, v_s the k_s-th largest non-NaN key of i's segment.  Keys are
// mapped to order-preserving unsigned integers (32 or 64 bits): a float's bits with the sign bit set for a positive
// number and every bit flipped for a negative one, -0.0 folded onto +0.0 first (the keep test compares values, so the
// two zeros are ties), and every NaN mapped to 0, which no number reaches (-Inf maps to 0x007fffff...).  A NaN is never
// counted nor kept: this port's own rule, the reference's NaN order lives in DataStructures' nlargest.  Integers only
// flip the sign bit.  v_s is then found by radix select on 8-bit digits from the top: per digit a 256-bin histogram of
// the keys that share the digits chosen so far, and the bin where the running count from the top reaches the rank.
// The answer is unique, so every route gives the same mask.
//   * Segments of up to the bound (GNNB_TOPK_SMEM_MAX keys): one CTA per segment with its mapped keys in shared memory,
//     one launch for all of them.
//   * Larger segments: one launch per digit over work items of CHUNK keys (a segment and a chunk of it).  The blocks of
//     a segment add their block histograms into the segment's global one (integer atomics); the next launch's blocks
//     each read it and pick the bin themselves, and the first block of the segment records (prefix, rank) for the one
//     after.  The histograms rotate over three buffers and the states over two, so no launch writes what its
//     predecessor's readers still read; a last launch of the same kernel writes the mask.
// Nothing is read back: the large-class grids are sized by the bound (at most n / (bound + 1) large segments), and a
// call whose segments are all small still issues those launches, whose blocks find no item and leave.
//
// Score, gate and pullback work on node rows (x (D, n) column-major: node j's D features are contiguous), one warp per
// row, float4 loads when D % 4 == 0 and the rows are 16 B aligned.  ‖p‖² is summed by every warp in the same order
// (warp_sumsq), so each kernel sees the same bits.  The pullback's dp is a two-stage sum: per-block partials in a fixed
// warp order, then a final pass over the blocks in order.  No float atomics anywhere: every result is run-to-run
// bit-identical.
#include "common.cuh"
#include <cub/cub.cuh>

namespace gnnb {
namespace topk {

constexpr int THREADS = 256;
constexpr int WARPS = THREADS / 32;
constexpr int CHUNK = 4096;                         // keys per large-class work item: 16 per thread
constexpr int SLICE = 1024;                         // pullback: features per block column (per-warp accumulators)
constexpr unsigned FULL = 0xffffffffu;
static_assert((size_t)GNNB_TOPK_SMEM_MAX * 8 + 4096 <= 227 * 1024, "the small class's keys must fit one CTA");

int g_bound = GNNB_TOPK_SMEM_MAX;                   // segments of more keys take the large class

// ------------------------------------------------------------------------------------------------ key transform
template <int KT> struct Key;
template <> struct Key<GNNB_KEY_F32> {
    using T = float; using U = uint32_t; static constexpr bool FLT = true;
    __device__ static U map(float f) {
        uint32_t b = __float_as_uint(f);
        if (f != f) return 0u;
        if (b == 0x80000000u) b = 0u;
        return (b & 0x80000000u) ? ~b : (b | 0x80000000u);
    }
};
template <> struct Key<GNNB_KEY_F64> {
    using T = double; using U = uint64_t; static constexpr bool FLT = true;
    __device__ static U map(double f) {
        uint64_t b = (uint64_t)__double_as_longlong(f);
        if (f != f) return 0ull;
        if (b == 0x8000000000000000ull) b = 0ull;
        return (b & 0x8000000000000000ull) ? ~b : (b | 0x8000000000000000ull);
    }
};
template <> struct Key<GNNB_KEY_I32> {
    using T = int32_t; using U = uint32_t; static constexpr bool FLT = false;
    __device__ static U map(int32_t v) { return (uint32_t)v ^ 0x80000000u; }
};
template <> struct Key<GNNB_KEY_I64> {
    using T = int64_t; using U = uint64_t; static constexpr bool FLT = false;
    __device__ static U map(int64_t v) { return (uint64_t)v ^ 0x8000000000000000ull; }
};

template <int KT> __device__ __forceinline__ bool valid(typename Key<KT>::U u) { return !Key<KT>::FLT || u != 0; }

// segment s of seg (NULL: the one segment [0, n))
__device__ __forceinline__ int64_t seg_lo(const int64_t* seg, int64_t s) { return seg ? seg[s] : 0; }
__device__ __forceinline__ int64_t seg_hi(const int64_t* seg, int64_t s, int64_t n) { return seg ? seg[s + 1] : n; }

__device__ __forceinline__ uint64_t rank_of(int64_t len, int64_t k, double ratio) {
    if (k >= 1) return (uint64_t)(k < len ? k : len);
    const double r = ceil(ratio * (double)len);
    return r >= (double)len ? (uint64_t)len : (uint64_t)r;
}

// one histogram vote per key; lanes with equal digits add once (keeps all-equal keys off one counter's queue).  Called
// by every lane of the warp; digit >= 256 abstains.
__device__ __forceinline__ void vote(uint32_t* h, unsigned digit) {
    const unsigned peers = __match_any_sync(FULL, digit);
    if (digit < 256 && (threadIdx.x & 31) == (unsigned)(__ffs(peers) - 1)) atomicAdd(h + digit, (uint32_t)__popc(peers));
}

// warp-wide: the bin where the count from the top (bin 255) first reaches rank (1 <= rank <= Σ h), and the rank within
// it.  Lane l owns bins 255 - 8l .. 248 - 8l.
struct Bin { unsigned bin; uint64_t rank; };
__device__ __forceinline__ Bin find_bin(const uint32_t* h, uint64_t rank) {
    const int lane = threadIdx.x & 31;
    uint64_t c = 0;
#pragma unroll
    for (int j = 0; j < 8; ++j) c += h[255 - 8 * lane - j];
    uint64_t S = c;
#pragma unroll
    for (int off = 1; off < 32; off <<= 1) {
        const uint64_t t = __shfl_up_sync(FULL, S, off);
        if (lane >= off) S += t;
    }
    const int L = __ffs(__ballot_sync(FULL, S >= rank)) - 1;
    unsigned b = 0;
    uint64_t r = 0;
    if (lane == L) {
        uint64_t cum = S - c;
#pragma unroll
        for (int j = 0; j < 8; ++j) {
            b = 255 - 8 * lane - j;
            if (cum + h[b] >= rank) { r = rank - cum; break; }
            cum += h[b];
        }
    }
    return Bin{__shfl_sync(FULL, b, L), __shfl_sync(FULL, r, L)};
}

// ------------------------------------------------------------------------------------------------ small class
template <int KT>
__global__ void __launch_bounds__(THREADS) small_kernel(const typename Key<KT>::T* __restrict__ keys, int64_t n,
                                                        const int64_t* __restrict__ seg, int64_t k, double ratio,
                                                        int64_t bound, const int* __restrict__ bad,
                                                        uint8_t* __restrict__ keep) {
    using U = typename Key<KT>::U;
    constexpr int NB = sizeof(U) * 8;
    extern __shared__ __align__(16) unsigned char smem_raw[];
    U* sk = reinterpret_cast<U*>(smem_raw);
    __shared__ uint32_t h[256];
    __shared__ uint32_t cnt;
    __shared__ U prefix;
    __shared__ uint64_t rank;
    if (*bad) {                                         // malformed seg_ptr: keep nothing, read no segment
        for (int64_t i = (int64_t)blockIdx.x * THREADS + threadIdx.x; i < n; i += (int64_t)gridDim.x * THREADS)
            keep[i] = 0;
        return;
    }
    const int64_t a = seg_lo(seg, blockIdx.x), len = seg_hi(seg, blockIdx.x, n) - a;
    if (len <= 0 || len > bound) return;                // block-uniform
    if (threadIdx.x == 0) cnt = 0;
    __syncthreads();
    uint32_t c = 0;
    for (int i = threadIdx.x; i < len; i += THREADS) {
        const U u = Key<KT>::map(keys[a + i]);
        sk[i] = u;
        c += valid<KT>(u);
    }
    if (c) atomicAdd(&cnt, c);
    __syncthreads();
    const uint64_t want = rank_of(len, k, ratio);
    uint64_t r = want < cnt ? want : cnt;
    U pre = 0;
    if (r > 0) {
        for (int d = 0; d < NB / 8; ++d) {
            for (int i = threadIdx.x; i < 256; i += THREADS) h[i] = 0;
            __syncthreads();
            const int sh = NB - 8 * d;                  // bits above the digit: already chosen
            for (int base = 0; base < len; base += THREADS) {
                const int i = base + threadIdx.x;
                unsigned digit = 256;
                if (i < len) {
                    const U u = sk[i];
                    if (valid<KT>(u) && (d == 0 || (u >> sh) == (pre >> sh))) digit = (unsigned)(u >> (sh - 8)) & 255u;
                }
                vote(h, digit);
            }
            __syncthreads();
            if (threadIdx.x < 32) {
                const Bin b = find_bin(h, r);
                if (threadIdx.x == 0) { prefix = pre | ((U)b.bin << (sh - 8)); rank = b.rank; }
            }
            __syncthreads();
            pre = prefix;
            r = rank;
        }
    }
    for (int i = threadIdx.x; i < len; i += THREADS) {
        const U u = sk[i];
        keep[a + i] = (r > 0 && valid<KT>(u) && u >= pre) ? 1 : 0;
    }
}

// ------------------------------------------------------------------------------------------------ large class
struct LargeArgs {
    const int64_t* seg;         // NULL: one segment
    const int64_t* item_ptr;    // [n_seg + 1]: running count of the large segments' items; slot of segment s = item_ptr[s]
    uint32_t* hist;             // [3][slots][256]
    uint64_t* state;            // [2][slots][2]: (prefix, rank) after the digits chosen so far
    const int* bad;
    uint8_t* keep;
    int64_t n, n_seg, slots, k;
    double ratio;
};

// Pass d < ND: choose digit d - 1 from the previous pass's histogram (d >= 1) and histogram digit d of this item's
// keys.  Pass ND: choose the last digit and write the item's mask.
template <int KT>
__global__ void __launch_bounds__(THREADS, 4) large_kernel(const typename Key<KT>::T* __restrict__ keys, const LargeArgs A,
                                                        int d) {
    using U = typename Key<KT>::U;
    constexpr int NB = sizeof(U) * 8, ND = NB / 8;
    __shared__ uint32_t h[256];
    __shared__ U prefix;
    __shared__ uint64_t rank;
    if (*A.bad) return;
    const int64_t item = blockIdx.x;
    if (item >= A.item_ptr[A.n_seg]) return;
    int64_t lo = 0, hi = A.n_seg;                       // item_ptr[lo] <= item < item_ptr[lo + 1]
    while (hi - lo > 1) {
        const int64_t mid = (lo + hi) >> 1;
        if (A.item_ptr[mid] <= item) lo = mid; else hi = mid;
    }
    const int64_t slot = A.item_ptr[lo], chunk = item - slot;
    const int64_t a = seg_lo(A.seg, lo), len = seg_hi(A.seg, lo, A.n) - a;
    const int64_t i0 = a + chunk * CHUNK, i1 = i0 + CHUNK < a + len ? i0 + CHUNK : a + len;
    uint32_t* const hprev = A.hist + ((size_t)((d + 2) % 3) * A.slots + slot) * 256;
    uint32_t* const hcur = A.hist + ((size_t)(d % 3) * A.slots + slot) * 256;
    uint32_t* const hnext = A.hist + ((size_t)((d + 1) % 3) * A.slots + slot) * 256;
    if (d > 0) {
        for (int i = threadIdx.x; i < 256; i += THREADS) h[i] = hprev[i];
        __syncthreads();
        if (threadIdx.x < 32) {
            U pre;
            uint64_t r;
            if (d == 1) {                               // the first histogram counts the valid keys
                uint32_t c = 0;
                for (int i = threadIdx.x; i < 256; i += 32) c += h[i];
                for (int off = 16; off; off >>= 1) c += __shfl_xor_sync(FULL, c, off);
                const uint64_t want = rank_of(len, A.k, A.ratio);
                pre = 0;
                r = want < c ? want : c;
            } else {
                const uint64_t* s = A.state + ((size_t)((d - 1) & 1) * A.slots + slot) * 2;
                pre = (U)s[0];
                r = s[1];
            }
            if (r > 0) {
                const Bin b = find_bin(h, r);
                pre |= (U)b.bin << (NB - 8 * d);
                r = b.rank;
            }
            if (threadIdx.x == 0) {
                prefix = pre;
                rank = r;
                if (chunk == 0 && d < ND) {
                    uint64_t* s = A.state + ((size_t)(d & 1) * A.slots + slot) * 2;
                    s[0] = (uint64_t)pre;
                    s[1] = r;
                }
            }
        }
        __syncthreads();
    }
    if (chunk == 0 && d < ND)                           // read two passes ago, written by the next
        for (int i = threadIdx.x; i < 256; i += THREADS) hnext[i] = 0;
    const U pre = d > 0 ? prefix : (U)0;
    const uint64_t r = d > 0 ? rank : 1;
    if (d == ND) {
        for (int64_t i = i0 + threadIdx.x; i < i1; i += THREADS) {
            const U u = Key<KT>::map(keys[i]);
            A.keep[i] = (r > 0 && valid<KT>(u) && u >= pre) ? 1 : 0;
        }
        return;
    }
    if (r == 0) return;                                 // nothing to keep (block-uniform)
    for (int i = threadIdx.x; i < 256; i += THREADS) h[i] = 0;
    __syncthreads();
    const int sh = NB - 8 * d;
    for (int64_t base = i0; base < i1; base += THREADS) {
        const int64_t i = base + threadIdx.x;
        unsigned digit = 256;
        if (i < i1) {
            const U u = Key<KT>::map(keys[i]);
            if (valid<KT>(u) && (d == 0 || (u >> sh) == (pre >> sh))) digit = (unsigned)(u >> (sh - 8)) & 255u;
        }
        vote(h, digit);
    }
    __syncthreads();
    for (int i = threadIdx.x; i < 256; i += THREADS)
        if (h[i]) atomicAdd(hcur + i, h[i]);
}

// per segment: validity of the offsets and the large-class items (ceil(len / CHUNK) for len > bound, else 0)
__global__ void classify_kernel(const int64_t* __restrict__ seg, int64_t n_seg, int64_t n, int64_t bound,
                                int64_t* __restrict__ items, int* __restrict__ bad) {
    const int64_t s = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (s >= n_seg) return;
    const int64_t a = seg_lo(seg, s), b = seg_hi(seg, s, n);
    const bool ok = !((s == 0 && a != 0) || (s == n_seg - 1 && b != n) || b < a || a < 0 || b > n);
    if (!ok) *(volatile int*)bad = GNNB_EINVAL;
    items[s] = (ok && b - a > bound) ? (b - a + CHUNK - 1) / CHUNK : 0;
}

template <int KT>
int keep_run(const void* keys, int64_t n, const int64_t* seg, int64_t n_seg, int64_t k, double ratio, uint8_t* keep,
             int32_t* dev_status, cudaStream_t st) {
    using T = typename Key<KT>::T;
    using U = typename Key<KT>::U;
    constexpr int ND = (int)sizeof(U);
    const int64_t bound = g_bound;
    const T* kp = static_cast<const T*>(keys);
    // large segments: at most n / (bound + 1); their items at most n / CHUNK + that many
    const int64_t max_large = seg ? std::min(n_seg, n / (bound + 1)) : (n > bound ? 1 : 0);
    const int64_t slots = max_large ? ceil_div(n, CHUNK) + max_large : 0;
    size_t scan_bytes = 0;
    GNNB_CUDA(cub::DeviceScan::InclusiveSum(nullptr, scan_bytes, (int64_t*)nullptr, (int64_t*)nullptr, (int)n_seg, st));
    auto al = [](size_t b) { return (b + 255) & ~(size_t)255; };
    const size_t off_ptr = al(sizeof(int64_t) * (size_t)n_seg);
    const size_t off_hist = off_ptr + al(sizeof(int64_t) * (size_t)(n_seg + 1));
    const size_t off_state = off_hist + al(sizeof(uint32_t) * 3 * 256 * (size_t)slots);
    const size_t off_flag = off_state + al(sizeof(uint64_t) * 4 * (size_t)slots);
    const size_t off_tmp = off_flag + 256;
    DeviceState* ds = nullptr;
    GNNB_TRY(device_state(&ds));
    GNNB_TRY(grow_buffer(&ds->topk_ws, &ds->topk_ws_bytes, off_tmp + scan_bytes + 1));
    char* buf = ds->topk_ws;
    int64_t* items = reinterpret_cast<int64_t*>(buf);
    int64_t* item_ptr = reinterpret_cast<int64_t*>(buf + off_ptr);
    int* bad = reinterpret_cast<int*>(buf + off_flag);
    GNNB_CUDA(cudaMemsetAsync(bad, 0, sizeof(int), st));
    GNNB_CUDA(cudaMemsetAsync(item_ptr, 0, sizeof(int64_t), st));
    classify_kernel<<<(unsigned)ceil_div(n_seg, 256), 256, 0, st>>>(seg, n_seg, n, bound, items, bad);
    GNNB_LAUNCHED();
    if (max_large) {
        GNNB_CUDA(cub::DeviceScan::InclusiveSum(buf + off_tmp, scan_bytes, items, item_ptr + 1, (int)n_seg, st));
        g_launches.fetch_add(1, std::memory_order_relaxed);
    }
    if (dev_status) GNNB_CUDA(cudaMemcpyAsync(dev_status, bad, sizeof(int32_t), cudaMemcpyDeviceToDevice, st));
    if (seg || n <= bound) {                            // some segment may be small
        const size_t smem = sizeof(U) * (size_t)std::min(n, bound);
        auto kern = small_kernel<KT>;
        GNNB_CUDA(cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
        kern<<<(unsigned)n_seg, THREADS, smem, st>>>(kp, n, seg, k, ratio, bound, bad, keep);
        GNNB_LAUNCHED();
    }
    if (max_large) {
        LargeArgs A{};
        A.seg = seg; A.item_ptr = item_ptr; A.bad = bad; A.keep = keep; A.n = n; A.n_seg = n_seg; A.slots = slots;
        A.k = k; A.ratio = ratio;
        A.hist = reinterpret_cast<uint32_t*>(buf + off_hist);
        A.state = reinterpret_cast<uint64_t*>(buf + off_state);
        GNNB_CUDA(cudaMemsetAsync(A.hist, 0, sizeof(uint32_t) * 256 * (size_t)slots, st));
        for (int d = 0; d <= ND; ++d) {
            large_kernel<KT><<<(unsigned)slots, THREADS, 0, st>>>(kp, A, d);
            GNNB_LAUNCHED();
        }
    }
    return GNNB_OK;
}

// ------------------------------------------------------------------------------------------------ score, gate, pullback
template <int VEC> __device__ __forceinline__ void ld(const float* p, float (&v)[VEC]) {
    if constexpr (VEC == 4) {
        const float4 t = __ldg(reinterpret_cast<const float4*>(p));
        v[0] = t.x; v[1] = t.y; v[2] = t.z; v[3] = t.w;
    } else {
        v[0] = __ldg(p);
    }
}
template <int VEC> __device__ __forceinline__ void st(float* p, const float (&v)[VEC]) {
    if constexpr (VEC == 4) *reinterpret_cast<float4*>(p) = make_float4(v[0], v[1], v[2], v[3]);
    else *p = v[0];
}

// Σ_d p_d², lane-strided then a butterfly: the same bits in every warp of every kernel
__device__ __forceinline__ float warp_sumsq(const float* __restrict__ p, int64_t D) {
    float s = 0.f;
    for (int64_t d = threadIdx.x & 31; d < D; d += 32) s = fmaf(__ldg(p + d), __ldg(p + d), s);
    for (int off = 16; off; off >>= 1) s += __shfl_xor_sync(FULL, s, off);
    return s;
}

template <int VEC> __device__ __forceinline__ float row_dot(const float* a, const float* b, int64_t D) {
    float acc = 0.f;
    for (int64_t d = (threadIdx.x & 31) * VEC; d < D; d += 32 * VEC) {
        float u[VEC], v[VEC];
        ld<VEC>(a + d, u); ld<VEC>(b + d, v);
#pragma unroll
        for (int q = 0; q < VEC; ++q) acc = fmaf(u[q], v[q], acc);
    }
    for (int off = 16; off; off >>= 1) acc += __shfl_xor_sync(FULL, acc, off);
    return acc;
}

// NNlib's sigmoid: t = exp(-|a|), 1 / (1 + t) for a >= 0, t / (1 + t) otherwise
__device__ __forceinline__ float sigm(float a) {
    const float t = expf(-fabsf(a));
    return a >= 0.f ? 1.f / (1.f + t) : t / (1.f + t);
}

template <int VEC>
__global__ void __launch_bounds__(THREADS) score_kernel(const float* __restrict__ x, int64_t n, int64_t D,
                                                        const float* __restrict__ p, float* __restrict__ y) {
    const float nrm = sqrtf(warp_sumsq(p, D));
    const int64_t w0 = ((int64_t)blockIdx.x * THREADS + threadIdx.x) >> 5, nw = ((int64_t)gridDim.x * THREADS) >> 5;
    for (int64_t j = w0; j < n; j += nw) {
        const float dot = row_dot<VEC>(x + j * D, p, D);
        if ((threadIdx.x & 31) == 0) y[j] = dot / nrm;
    }
}

__device__ __forceinline__ bool bad_index(const int64_t* idx, int64_t j, int64_t n, bool ascending) {
    const int64_t i = idx[j];
    return i < 0 || i >= n || (ascending && j > 0 && idx[j - 1] >= i);
}

template <int VEC>
__global__ void __launch_bounds__(THREADS) gate_kernel(const float* __restrict__ x, int64_t n, int64_t D,
                                                       const float* __restrict__ y, const int64_t* __restrict__ idx,
                                                       int64_t m, float* __restrict__ out, int32_t* status) {
    const int64_t w0 = ((int64_t)blockIdx.x * THREADS + threadIdx.x) >> 5, nw = ((int64_t)gridDim.x * THREADS) >> 5;
    for (int64_t j = w0; j < m; j += nw) {
        const int64_t i = idx[j];
        const bool bad = i < 0 || i >= n;
        if (bad && status && (threadIdx.x & 31) == 0) *(volatile int32_t*)status = GNNB_EINDEX;
        const float s = bad ? __int_as_float(0x7fc00000) : sigm(__ldg(y + i));
        for (int64_t d = (threadIdx.x & 31) * VEC; d < D; d += 32 * VEC) {
            float v[VEC];
            if (bad) {
#pragma unroll
                for (int q = 0; q < VEC; ++q) v[q] = s;
            } else {
                ld<VEC>(x + i * D + d, v);
#pragma unroll
                for (int q = 0; q < VEC; ++q) v[q] *= s;
            }
            st<VEC>(out + j * D + d, v);
        }
    }
}

// Block (bx, by): rows j of [bx * rpb, (bx + 1) * rpb), warp w taking every WARPS-th; features [by * SLICE, ...).  The dot
// <dout_j, x_i> runs over all D in every slice (the same bits); dx and the dp partials only over the slice.
template <int VEC>
__global__ void __launch_bounds__(THREADS) gate_bwd_kernel(const float* __restrict__ x, int64_t n, int64_t D,
                                                           const float* __restrict__ y, const float* __restrict__ p,
                                                           const int64_t* __restrict__ idx, int64_t m, int64_t rpb,
                                                           const float* __restrict__ dout, float* __restrict__ dx,
                                                           float* __restrict__ part, int32_t* status) {
    __shared__ __align__(16) float acc[WARPS][SLICE];
    __shared__ float yacc[WARPS];
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    const int64_t f0 = (int64_t)blockIdx.y * SLICE, f1 = f0 + SLICE < D ? f0 + SLICE : D;
    for (int64_t f = lane; f < SLICE; f += 32) acc[warp][f] = 0.f;
    const float nrm = sqrtf(warp_sumsq(p, D));
    float ys = 0.f;
    const int64_t j0 = (int64_t)blockIdx.x * rpb, j1 = j0 + rpb < m ? j0 + rpb : m;
    for (int64_t j = j0 + warp; j < j1; j += WARPS) {
        if (bad_index(idx, j, n, true)) {
            if (status && lane == 0) *(volatile int32_t*)status = GNNB_EINDEX;
            continue;
        }
        const int64_t i = idx[j];
        const float yi = __ldg(y + i), s = sigm(yi);
        const float dy = s * (1.f - s) * row_dot<VEC>(dout + j * D, x + i * D, D);
        ys = fmaf(dy, yi, ys);
        const float c = dy / nrm;
        for (int64_t d = f0 + lane * VEC; d < f1; d += 32 * VEC) {
            float g[VEC], xv[VEC], pv[VEC], o[VEC];
            ld<VEC>(dout + j * D + d, g); ld<VEC>(x + i * D + d, xv); ld<VEC>(p + d, pv);
#pragma unroll
            for (int q = 0; q < VEC; ++q) {
                o[q] = fmaf(s, g[q], c * pv[q]);
                acc[warp][d - f0 + q] = fmaf(dy, xv[q], acc[warp][d - f0 + q]);
            }
            st<VEC>(dx + i * D + d, o);
        }
    }
    if (lane == 0) yacc[warp] = ys;
    __syncthreads();
    float* out = part + (size_t)blockIdx.x * (D + 1);
    for (int64_t d = f0 + threadIdx.x; d < f1; d += THREADS) {
        float t = 0.f;
#pragma unroll
        for (int w = 0; w < WARPS; ++w) t += acc[w][d - f0];
        out[d] = t;
    }
    if (blockIdx.y == 0 && threadIdx.x == 0) {
        float t = 0.f;
#pragma unroll
        for (int w = 0; w < WARPS; ++w) t += yacc[w];
        out[D] = t;
    }
}

// dp[d] = (Σ_b part[b][d]) / ‖p‖ − (Σ_b part[b][D]) p[d] / ‖p‖², the blocks in order
__global__ void __launch_bounds__(THREADS) dp_final_kernel(const float* __restrict__ part, int64_t nblocks, int64_t D,
                                                           const float* __restrict__ p, float* __restrict__ dp) {
    const float nrm2 = warp_sumsq(p, D), nrm = sqrtf(nrm2);
    const int64_t d = (int64_t)blockIdx.x * THREADS + threadIdx.x;
    if (d >= D) return;
    float sx = 0.f, sy = 0.f;
    for (int64_t b = 0; b < nblocks; ++b) {
        sx += part[(size_t)b * (D + 1) + d];
        sy += part[(size_t)b * (D + 1) + D];
    }
    dp[d] = sx / nrm - sy * __ldg(p + d) / nrm2;
}

bool a16(const void* a) { return (reinterpret_cast<uintptr_t>(a) & 15) == 0; }
unsigned warp_grid(int64_t rows) {
    const int64_t b = ceil_div(rows, WARPS), cap = (int64_t)kNumSMs * 16;
    return (unsigned)(b < 1 ? 1 : (b < cap ? b : cap));
}

}  // namespace topk
}  // namespace gnnb

using namespace gnnb;

extern "C" {

int gnnb_topk_set_smem_max(int64_t bound) {
    if (bound < 0 || bound > GNNB_TOPK_SMEM_MAX)
        GNNB_FAIL(GNNB_EINVAL, "gnnb_topk_set_smem_max: bound = %lld must be in [0, %d]", (long long)bound,
                  GNNB_TOPK_SMEM_MAX);
    topk::g_bound = (int)bound;
    return GNNB_OK;
}

int gnnb_topk_keep(const void* keys, int key_type, int64_t n, const int64_t* seg_ptr, int64_t n_seg, int64_t k,
                   double ratio, uint8_t* keep, int32_t* dev_status, void* stream) {
    if (key_type < GNNB_KEY_F32 || key_type > GNNB_KEY_I64)
        GNNB_FAIL(GNNB_EINVAL, "gnnb_topk_keep: key_type = %d is not a GNNB_KEY_* value", key_type);
    if (!(k >= 1 && ratio == 0.0) && !(k == 0 && ratio > 0.0 && ratio <= 1.0))
        GNNB_FAIL(GNNB_EINVAL, "gnnb_topk_keep: need k >= 1 (ratio 0) or k = 0 and 0 < ratio <= 1 (got k = %lld, "
                               "ratio = %g)", (long long)k, ratio);
    if (n < 0 || n >= ((int64_t)1 << 31)) GNNB_FAIL(GNNB_ESIZE, "gnnb_topk_keep: n = %lld must be in [0, 2^31)",
                                                    (long long)n);
    if (seg_ptr && (n_seg < 1 || n_seg >= ((int64_t)1 << 31)))
        GNNB_FAIL(GNNB_ESIZE, "gnnb_topk_keep: n_seg = %lld must be in [1, 2^31)", (long long)n_seg);
    cudaStream_t st = (cudaStream_t)stream;
    if (n == 0 && !seg_ptr) {
        if (dev_status) GNNB_CUDA(cudaMemsetAsync(dev_status, 0, sizeof(int32_t), st));
        return GNNB_OK;
    }
    if ((n > 0 && (!keys || !keep)) || (!seg_ptr && n_seg != 1 && n_seg != 0))
        GNNB_FAIL(GNNB_ESIZE, "gnnb_topk_keep: NULL array of positive size, or n_seg without seg_ptr");
    const int64_t ns = seg_ptr ? n_seg : 1;
    switch (key_type) {
        case GNNB_KEY_F32: return topk::keep_run<GNNB_KEY_F32>(keys, n, seg_ptr, ns, k, ratio, keep, dev_status, st);
        case GNNB_KEY_F64: return topk::keep_run<GNNB_KEY_F64>(keys, n, seg_ptr, ns, k, ratio, keep, dev_status, st);
        case GNNB_KEY_I32: return topk::keep_run<GNNB_KEY_I32>(keys, n, seg_ptr, ns, k, ratio, keep, dev_status, st);
        default: return topk::keep_run<GNNB_KEY_I64>(keys, n, seg_ptr, ns, k, ratio, keep, dev_status, st);
    }
}

int gnnb_topk_score(const float* x, int64_t n, int64_t D, const float* p, float* y, void* stream) {
    if (n < 0 || D < 1) GNNB_FAIL(GNNB_ESIZE, "gnnb_topk_score: n must be >= 0 and D >= 1 (got n = %lld, D = %lld)",
                                  (long long)n, (long long)D);
    if (n == 0) return GNNB_OK;
    if (!x || !p || !y) GNNB_FAIL(GNNB_ESIZE, "gnnb_topk_score: NULL array of positive size");
    cudaStream_t st = (cudaStream_t)stream;
    if (D % 4 == 0 && topk::a16(x) && topk::a16(p)) topk::score_kernel<4><<<topk::warp_grid(n), topk::THREADS, 0, st>>>(x, n, D, p, y);
    else topk::score_kernel<1><<<topk::warp_grid(n), topk::THREADS, 0, st>>>(x, n, D, p, y);
    GNNB_LAUNCHED();
    return GNNB_OK;
}

int gnnb_topk_gate(const float* x, int64_t n, int64_t D, const float* y, const int64_t* idx, int64_t m, float* out,
                   int32_t* dev_status, void* stream) {
    if (n < 0 || m < 0 || D < 1)
        GNNB_FAIL(GNNB_ESIZE, "gnnb_topk_gate: n, m must be >= 0 and D >= 1 (got n = %lld, m = %lld, D = %lld)",
                  (long long)n, (long long)m, (long long)D);
    cudaStream_t st = (cudaStream_t)stream;
    if (dev_status) GNNB_CUDA(cudaMemsetAsync(dev_status, 0, sizeof(int32_t), st));
    if (m == 0) return GNNB_OK;
    if (!x || !y || !idx || !out) GNNB_FAIL(GNNB_ESIZE, "gnnb_topk_gate: NULL array of positive size");
    if (D % 4 == 0 && topk::a16(x) && topk::a16(out))
        topk::gate_kernel<4><<<topk::warp_grid(m), topk::THREADS, 0, st>>>(x, n, D, y, idx, m, out, dev_status);
    else topk::gate_kernel<1><<<topk::warp_grid(m), topk::THREADS, 0, st>>>(x, n, D, y, idx, m, out, dev_status);
    GNNB_LAUNCHED();
    return GNNB_OK;
}

int gnnb_topk_gate_bwd(const float* x, int64_t n, int64_t D, const float* y, const float* p, const int64_t* idx,
                       int64_t m, const float* dout, float* dx, float* dp, int32_t* dev_status, void* stream) {
    if (n < 0 || m < 0 || D < 1)
        GNNB_FAIL(GNNB_ESIZE, "gnnb_topk_gate_bwd: n, m must be >= 0 and D >= 1 (got n = %lld, m = %lld, D = %lld)",
                  (long long)n, (long long)m, (long long)D);
    if (m > n) GNNB_FAIL(GNNB_EINDEX, "gnnb_topk_gate_bwd: m = %lld ascending distinct ids cannot lie in [0, %lld)",
                         (long long)m, (long long)n);
    if (!p || !dp || (n > 0 && (!x || !y || !dx)) || (m > 0 && (!idx || !dout)))
        GNNB_FAIL(GNNB_ESIZE, "gnnb_topk_gate_bwd: NULL array of positive size");
    cudaStream_t st = (cudaStream_t)stream;
    if (dev_status) GNNB_CUDA(cudaMemsetAsync(dev_status, 0, sizeof(int32_t), st));
    if (n > 0) GNNB_CUDA(cudaMemsetAsync(dx, 0, sizeof(float) * (size_t)(n * D), st));
    if (m == 0) {                                       // empty sums: dp = 0
        GNNB_CUDA(cudaMemsetAsync(dp, 0, sizeof(float) * (size_t)D, st));
        return GNNB_OK;
    }
    const int64_t slots = GNNB_TOPK_DP_SLOTS(m), rpb = ceil_div(m, slots), nblocks = ceil_div(m, rpb);
    DeviceState* ds = nullptr;
    GNNB_TRY(device_state(&ds));
    GNNB_TRY(grow_buffer(&ds->topk_part, &ds->topk_part_bytes, sizeof(float) * (size_t)(nblocks * (D + 1))));
    const dim3 grid((unsigned)nblocks, (unsigned)ceil_div(D, topk::SLICE));
    if (D % 4 == 0 && topk::a16(x) && topk::a16(p) && topk::a16(dout) && topk::a16(dx))
        topk::gate_bwd_kernel<4><<<grid, topk::THREADS, 0, st>>>(x, n, D, y, p, idx, m, rpb, dout, dx, ds->topk_part,
                                                                 dev_status);
    else
        topk::gate_bwd_kernel<1><<<grid, topk::THREADS, 0, st>>>(x, n, D, y, p, idx, m, rpb, dout, dx, ds->topk_part,
                                                                 dev_status);
    GNNB_LAUNCHED();
    topk::dp_final_kernel<<<(unsigned)ceil_div(D, topk::THREADS), topk::THREADS, 0, st>>>(ds->topk_part, nblocks, D, p, dp);
    GNNB_LAUNCHED();
    return GNNB_OK;
}

}  // extern "C"
