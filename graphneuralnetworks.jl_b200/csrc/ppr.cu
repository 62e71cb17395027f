// ppr.cu — ppr_diffusion on the device: alpha * inv(I + (alpha - 1) A) of one graph of a batch (a segment) at a time,
// by Gauss-Jordan elimination in shared memory, and the dense M of one larger segment for a batched dense inverse.
//
// Reference counterpart: ppr_diffusion(g; alpha) (GNNGraphs/src/transform.jl:1026-1051), which forms the dense N x N
// matrix of the whole batch and calls `inv` on it.  The inverse of a block-diagonal matrix is block-diagonal, so the
// per-segment blocks give the same result.
//
// Contract (tests/test_ppr_diffusion.py restates it in numpy, bit for bit):
//   Row i of a segment [base, base + n) starts as zeros; its in-edges (s -> base + i) are added in plan order,
//   A[i][s - base] += w_e, each add rounded.  Then, with am1 = fl32(alpha) - 1 rounded once,
//   M[i][j] = am1 * A[i][j] (j != i) and M[i][i] = 1 + am1 * A[i][i], each product and sum rounded.
//   Gauss-Jordan with partial pivoting, every product, difference and quotient rounded on its own, no contraction:
//   for k = 0 .. n-1:
//     p = the first i >= k with the largest |a[i][k]| (scan from k, replace on a strict >: a NaN never wins over a number)
//     a[p][k] == 0: info = k + 1, the segment stops here (its outputs are not written)
//     swap rows k and p, perm[k] = p; piv = a[k][k]; a[k][k] = 1; a[k][j] = a[k][j] / piv for every j
//     for every i != k: f = a[i][k]; a[i][k] = 0; a[i][j] = a[i][j] - f * a[k][j] for every j
//   then for k = n-1 .. 0: swap columns k and perm[k].  w_out[eid] = fl32(alpha) * a[t - base][s - base].
//
// Work decomposition: thread t of the group that owns a segment owns row t (build, column swaps, outputs) and column t
// (row swap, pivot-row scaling, elimination).  The matrix is row-major with an odd leading dimension ld >= n + 1, so a
// warp reading a row or a column is free of bank conflicts; column ld - 1 holds the step's multipliers f.
//   * small segments (n <= 32): one warp per segment, eight per CTA, __syncwarp between phases;
//   * medium segments (32 < n <= GNNB_PPR_SMEM_MAX_NODES): one CTA of 256 threads per segment, a __syncthreads between
//     phases (three per step), the matrix sized by the largest medium segment of the call.
// Both classes run the same device function, so a segment gives the same bits in either; gnnb_set_kernel_variant(12)
// sends every segment through the CTA class, which the tests use to check that.  The classes are two launches, as in
// rwpe.cu: one launch sized by the largest segment would hold molecule CTAs to one per SM.
// A prep kernel validates seg_ptr and classifies the segments (CUB scan of the medium ones, two max reduces); one
// read-back sizes both grids.  An edge whose source lies outside its target's segment is never read through: it raises
// a flag (GNNB_EINVAL).
#include "common.cuh"
#include <cub/cub.cuh>

namespace gnnb {
extern bool g_reference_kernels;   // segreduce.cu: gnnb_set_kernel_variant(12)

namespace ppr {

constexpr int SMALL = 32;                    // nodes of a small segment: one lane per row and column
constexpr int WARPS = 8;
constexpr int THREADS = WARPS * 32;
constexpr int MAX_NODES = GNNB_PPR_SMEM_MAX_NODES;
static_assert(MAX_NODES < THREADS, "a CTA owns every row and column of a medium segment with one thread each");

struct Best {                                // a warp's pivot candidate: packed key and the signed value
    unsigned long long key;
    float val;
    float pad;
};

__host__ __device__ constexpr int ld_of(int n) { return (n + 1) | 1; }              // odd, >= n + 1
__host__ __device__ constexpr size_t mat_bytes(int n) {                              // one segment's shared memory
    return sizeof(float) * (size_t)n * ld_of(n) + sizeof(int) * (size_t)n;
}
constexpr size_t SMALL_SMEM = (size_t)WARPS * mat_bytes(SMALL);
__host__ __device__ constexpr size_t best_offset(int n) { return (mat_bytes(n) + 15) & ~(size_t)15; }
constexpr size_t medium_smem(int n) { return best_offset(n) + sizeof(Best) * WARPS; }
// 227 KB is the opt-in shared memory of one H100 CTA: GNNB_PPR_SMEM_MAX_NODES is the largest n that fits it.  The
// entry checks the device's own limit at run time.
static_assert(medium_smem(MAX_NODES) <= 227 * 1024 && medium_smem(MAX_NODES + 1) > 227 * 1024,
              "GNNB_PPR_SMEM_MAX_NODES must be the largest segment whose matrix fits 227 KB");

struct Params {
    const int32_t* rowptr;   // CSR by target
    const int32_t* col;      // source of each sorted edge
    const int32_t* eid;      // COO position of each sorted edge (weights and outputs are in COO order)
    const float* w;          // NULL: every weight is 1
    const int64_t* seg;      // [n_seg + 1]
    const int64_t* item_ptr; // [n_seg + 1]: running count of medium segments
    float* w_out;
    int32_t* info;
    int* crossed;            // set when an edge crosses segments
    float alpha;
    int32_t n_seg, n_small_blocks;
};

// the pivot key of row i at step k: larger wins, equal keys go to the smaller row.  A NaN at row k wins (the scan starts
// there and nothing is > NaN); a NaN below it ranks with 0, which never beats row k; rows outside [k, n) are 0.
__device__ __forceinline__ unsigned long long pivot_key(float x, int i, int k, int n) {
    if (i < k || i >= n) return 0ull;
    unsigned key = x != x ? (i == k ? 0xffffffffu : 0u) : __float_as_uint(fabsf(x));
    return ((unsigned long long)key << 32) | (0xffffffffu - (unsigned)i);
}

__device__ __forceinline__ void warp_best(unsigned long long& key, float& val) {
#pragma unroll
    for (int o = 16; o; o >>= 1) {
        const unsigned long long k2 = __shfl_xor_sync(0xffffffffu, key, o);
        const float v2 = __shfl_xor_sync(0xffffffffu, val, o);
        if (k2 > key) { key = k2; val = v2; }
    }
}

template <bool CTA>
__device__ __forceinline__ void sync_group() {
    if (CTA) __syncthreads(); else __syncwarp();
}

// The segment [base, base + n) in `a` (n x ld floats) and `perm` (n ints); `tid` = thread of the group (a warp or the
// CTA), which owns row tid and column tid.  Exits uniformly across the group.
template <bool HAS_W, bool CTA>
__device__ __forceinline__ void invert_segment(const Params& p, float* __restrict__ a, int* __restrict__ perm,
                                               Best* __restrict__ best, int s, int base, int n, int tid) {
    const int ld = ld_of(n);
    const int F = ld - 1;                     // column of the multipliers
    const float am1 = __fsub_rn(p.alpha, 1.f);
    int e0 = 0, e1 = 0;
    if (tid < n) {                            // build row tid of M
        float* row = a + (size_t)tid * ld;
        for (int j = 0; j < n; ++j) row[j] = 0.f;
        e0 = __ldg(p.rowptr + base + tid), e1 = __ldg(p.rowptr + base + tid + 1);
        for (int e = e0; e < e1; ++e) {
            const unsigned sl = (unsigned)(__ldg(p.col + e) - base);
            if (sl >= (unsigned)n) { *(volatile int*)p.crossed = 1; continue; }     // never read outside the segment
            row[sl] = __fadd_rn(row[sl], HAS_W ? __ldg(p.w + __ldg(p.eid + e)) : 1.f);
        }
        for (int j = 0; j < n; ++j) {
            const float m = __fmul_rn(am1, row[j]);
            row[j] = j == tid ? __fadd_rn(1.f, m) : m;
        }
    }
    sync_group<CTA>();
    for (int k = 0; k < n; ++k) {
        // pivot search over column k
        unsigned long long key = pivot_key(tid < n ? a[(size_t)tid * ld + k] : 0.f, tid, k, n);
        float val = tid < n ? a[(size_t)tid * ld + k] : 0.f;
        warp_best(key, val);
        if (CTA) {
            if ((threadIdx.x & 31) == 0) best[threadIdx.x >> 5] = Best{key, val, 0.f};
            __syncthreads();
            key = best[0].key; val = best[0].val;
#pragma unroll
            for (int w = 1; w < WARPS; ++w)
                if (best[w].key > key) { key = best[w].key; val = best[w].val; }
        }
        const int pr = (int)(0xffffffffu - (unsigned)(key & 0xffffffffull));
        const float piv = val;
        if (piv == 0.f) {                     // uniform: every thread holds the same key and value
            if (tid == 0) p.info[s] = k + 1;
            return;
        }
        // swap rows k and pr and scale row k (column owners); the multipliers of the other rows (row owners)
        if (tid < n) {
            const float rk = a[(size_t)k * ld + tid], rp = a[(size_t)pr * ld + tid];
            a[(size_t)k * ld + tid] = __fdiv_rn(tid == k ? 1.f : rp, piv);
            if (pr != k) a[(size_t)pr * ld + tid] = rk;
            if (tid == k && pr != k) a[(size_t)pr * ld + F] = rk;                // row pr now holds the old row k
            if (tid != k && tid != pr) a[(size_t)tid * ld + F] = a[(size_t)tid * ld + k];
            if (tid == 0) perm[k] = pr;
        }
        sync_group<CTA>();
        // eliminate column k from every other row (column owners)
        if (tid < n) {
            const float r = a[(size_t)k * ld + tid];
            for (int i = 0; i < n; ++i) {
                if (i == k) continue;
                const float f = a[(size_t)i * ld + F];
                const float x = tid == k ? 0.f : a[(size_t)i * ld + tid];
                a[(size_t)i * ld + tid] = __fsub_rn(x, __fmul_rn(f, r));
            }
        }
        sync_group<CTA>();
    }
    if (tid < n) {                            // undo the row swaps as column swaps, then write the row's edges
        float* row = a + (size_t)tid * ld;
        for (int k = n - 1; k >= 0; --k) {
            const int q = perm[k];
            if (q != k) { const float x = row[k]; row[k] = row[q]; row[q] = x; }
        }
        for (int e = e0; e < e1; ++e) {
            const unsigned sl = (unsigned)(__ldg(p.col + e) - base);
            if (sl < (unsigned)n) p.w_out[__ldg(p.eid + e)] = __fmul_rn(p.alpha, row[sl]);
        }
    }
}

template <bool HAS_W>
__global__ void __launch_bounds__(THREADS) ppr_kernel(const Params p) {
    extern __shared__ __align__(16) unsigned char smem_raw[];
    const int warp = threadIdx.x >> 5;
    if ((int)blockIdx.x < p.n_small_blocks) {               // small segments: one warp each
        const int s = blockIdx.x * WARPS + warp;
        if (s >= p.n_seg) return;
        const int a = (int)p.seg[s], m = (int)(p.seg[s + 1] - a);
        if (m <= 0 || m > SMALL) return;
        float* mat = reinterpret_cast<float*>(smem_raw + (size_t)warp * mat_bytes(SMALL));
        invert_segment<HAS_W, false>(p, mat, reinterpret_cast<int*>(mat + (size_t)SMALL * ld_of(SMALL)), nullptr, s, a,
                                     m, threadIdx.x & 31);
        return;
    }
    const int64_t item = (int64_t)blockIdx.x - p.n_small_blocks;   // medium: item_ptr[s] <= item < item_ptr[s + 1]
    int lo = 0, hi = p.n_seg;
    while (hi - lo > 1) {
        const int mid = (lo + hi) >> 1;
        if (p.item_ptr[mid] <= item) lo = mid; else hi = mid;
    }
    const int a = (int)p.seg[lo], m = (int)(p.seg[lo + 1] - a);
    if (m <= 0 || m > MAX_NODES) return;                             // block-uniform: no barrier is skipped
    float* mat = reinterpret_cast<float*>(smem_raw);
    int* perm = reinterpret_cast<int*>(mat + (size_t)m * ld_of(m));
    Best* best = reinterpret_cast<Best*>(smem_raw + best_offset(m));
    invert_segment<HAS_W, true>(p, mat, perm, best, lo, a, m, threadIdx.x);
}

// per segment: medium (1 for a segment of the CTA class), its node count if medium, whether it is small, and info =
// -1 for a segment above the bound, 0 otherwise; bad = 1 for a malformed seg_ptr (every writer stores the same value)
__global__ void classify_kernel(const int64_t* __restrict__ seg, int64_t n_seg, int64_t n, int all_medium,
                                int64_t* __restrict__ items, int32_t* __restrict__ med_nodes,
                                int32_t* __restrict__ small, int32_t* __restrict__ info, int* __restrict__ bad) {
    const int64_t s = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (s >= n_seg) return;
    const int64_t a = seg[s], b = seg[s + 1];
    const bool ok = !((s == 0 && a != 0) || (s == n_seg - 1 && b != n) || b < a || a < 0 || b > n);
    if (!ok) *(volatile int*)bad = 1;
    const int64_t m = b - a;
    const bool sm = ok && m >= 1 && m <= SMALL && !all_medium;
    const bool med = ok && m >= 1 && m <= MAX_NODES && !sm;
    items[s] = med ? 1 : 0;
    med_nodes[s] = med ? (int32_t)m : 0;
    small[s] = sm ? 1 : 0;
    if (ok) info[s] = m > MAX_NODES ? -1 : 0;
}

// M of the nodes [a, a + m) into out (row-major, leading dimension ld): one warp per row, the edges added by lane 0 in
// plan order, the rows' zeros and the scaling by the whole warp.
template <bool HAS_W>
__global__ void __launch_bounds__(THREADS) ppr_matrix_kernel(const int32_t* __restrict__ rowptr,
                                                             const int32_t* __restrict__ col,
                                                             const int32_t* __restrict__ eid,
                                                             const float* __restrict__ w, int a, int m, int64_t ld,
                                                             float alpha, float* __restrict__ out,
                                                             int* __restrict__ crossed) {
    const int i = (int)(((int64_t)blockIdx.x * THREADS + threadIdx.x) >> 5);
    const int lane = threadIdx.x & 31;
    if (i >= m) return;
    float* row = out + (size_t)i * ld;
    for (int j = lane; j < m; j += 32) row[j] = 0.f;
    __syncwarp();
    if (lane == 0) {
        const int e0 = __ldg(rowptr + a + i), e1 = __ldg(rowptr + a + i + 1);
        for (int e = e0; e < e1; ++e) {
            const unsigned sl = (unsigned)(__ldg(col + e) - a);
            if (sl >= (unsigned)m) { *(volatile int*)crossed = 1; continue; }
            row[sl] = __fadd_rn(row[sl], HAS_W ? __ldg(w + __ldg(eid + e)) : 1.f);
        }
    }
    __syncwarp();
    const float am1 = __fsub_rn(alpha, 1.f);
    for (int j = lane; j < m; j += 32) {
        const float x = __fmul_rn(am1, row[j]);
        row[j] = j == i ? __fadd_rn(1.f, x) : x;
    }
}

template <bool HAS_W>
static int launch(const Params& p, int64_t grid, size_t smem, cudaStream_t st) {
    auto kern = ppr_kernel<HAS_W>;
    GNNB_CUDA(cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
    kern<<<(unsigned)grid, THREADS, smem, st>>>(p);
    GNNB_LAUNCHED();
    return GNNB_OK;
}

static size_t align256(size_t b) { return (b + 255) & ~(size_t)255; }

static int run(gnnb_graph* g, const float* w, float alpha, const int64_t* seg_ptr, int64_t n_seg, float* w_out,
               int32_t* info, cudaStream_t st) {
    const int64_t n = g->n_dst;
    int dev = 0, optin = 0;
    GNNB_CUDA(cudaGetDevice(&dev));
    GNNB_CUDA(cudaDeviceGetAttribute(&optin, cudaDevAttrMaxSharedMemoryPerBlockOptin, dev));
    if ((size_t)optin < medium_smem(MAX_NODES))
        GNNB_FAIL(GNNB_EUNSUPPORTED, "gnnb_ppr_diffusion: a segment of %d nodes needs %zu B of shared memory per CTA, "
                                     "the device allows %d", MAX_NODES, medium_smem(MAX_NODES), optin);
    // one scratch allocation: int64 items [n_seg], item_ptr [n_seg + 1], the default segment [2]; int32 medium node
    // counts [n_seg], small flags [n_seg], their two maxima [2]; int flags [2] (bad seg_ptr, an edge crossing
    // segments); the CUB temporary storage
    size_t scan_bytes = 0, max_bytes = 0;
    GNNB_CUDA(cub::DeviceScan::InclusiveSum(nullptr, scan_bytes, (int64_t*)nullptr, (int64_t*)nullptr, (int)n_seg, st));
    GNNB_CUDA(cub::DeviceReduce::Max(nullptr, max_bytes, (int32_t*)nullptr, (int32_t*)nullptr, (int)n_seg, st));
    const size_t tmp_bytes = scan_bytes > max_bytes ? scan_bytes : max_bytes;
    const size_t off_med = align256(sizeof(int64_t) * (size_t)(2 * n_seg + 3));
    const size_t off_flags = off_med + align256(sizeof(int32_t) * (size_t)(2 * n_seg + 2));
    const size_t off_tmp = off_flags + 256;
    DeviceScratch sc(st);
    char* buf = nullptr;
    GNNB_TRY(sc.alloc(&buf, off_tmp + (tmp_bytes ? tmp_bytes : 1)));
    int64_t* items = reinterpret_cast<int64_t*>(buf);
    int64_t* item_ptr = items + n_seg;
    int32_t* med = reinterpret_cast<int32_t*>(buf + off_med);
    int32_t* small = med + n_seg;
    int32_t* red = small + n_seg;                       // [0] largest medium segment, [1] any small segment
    int* flags = reinterpret_cast<int*>(buf + off_flags);
    void* tmp = buf + off_tmp;
    GNNB_CUDA(cudaMemsetAsync(flags, 0, 2 * sizeof(int), st));
    if (!seg_ptr) {
        int64_t* dseg = item_ptr + n_seg + 1;
        const int64_t h[2] = {0, n};
        GNNB_CUDA(cudaMemcpyAsync(dseg, h, sizeof h, cudaMemcpyHostToDevice, st));
        seg_ptr = dseg;
    }
    GNNB_CUDA(cudaMemsetAsync(item_ptr, 0, sizeof(int64_t), st));
    classify_kernel<<<(unsigned)ceil_div(n_seg, 256), 256, 0, st>>>(seg_ptr, n_seg, n, g_reference_kernels ? 1 : 0,
                                                                     items, med, small, info, flags);
    GNNB_LAUNCHED();
    GNNB_CUDA(cub::DeviceScan::InclusiveSum(tmp, scan_bytes, items, item_ptr + 1, (int)n_seg, st));
    GNNB_CUDA(cub::DeviceReduce::Max(tmp, max_bytes, med, red, (int)n_seg, st));
    GNNB_CUDA(cub::DeviceReduce::Max(tmp, max_bytes, small, red + 1, (int)n_seg, st));
    g_launches.fetch_add(3, std::memory_order_relaxed);
    int64_t n_items = 0;
    int32_t hred[2] = {0, 0};
    int bad = 0;
    GNNB_CUDA(cudaMemcpyAsync(&n_items, item_ptr + n_seg, sizeof n_items, cudaMemcpyDeviceToHost, st));
    GNNB_CUDA(cudaMemcpyAsync(hred, red, sizeof hred, cudaMemcpyDeviceToHost, st));
    GNNB_CUDA(cudaMemcpyAsync(&bad, flags, sizeof bad, cudaMemcpyDeviceToHost, st));
    GNNB_CUDA(cudaStreamSynchronize(st));
    if (bad)
        GNNB_FAIL(GNNB_EINVAL, "seg_ptr must hold n_seg + 1 non-decreasing offsets from 0 to n = %lld", (long long)n);
    Params p{};
    p.rowptr = g->by_dst.rowptr; p.col = g->by_dst.col; p.eid = g->by_dst.eid;
    p.w = w; p.seg = seg_ptr; p.item_ptr = item_ptr; p.w_out = w_out; p.info = info; p.crossed = flags + 1;
    p.alpha = alpha; p.n_seg = (int32_t)n_seg;
    if (hred[1]) {                                      // small segments: every block of this launch is small
        p.n_small_blocks = (int32_t)ceil_div(n_seg, WARPS);
        if (w) GNNB_TRY(launch<true>(p, p.n_small_blocks, SMALL_SMEM, st));
        else GNNB_TRY(launch<false>(p, p.n_small_blocks, SMALL_SMEM, st));
    }
    if (n_items) {                                      // medium segments: every block of this launch is medium
        p.n_small_blocks = 0;
        const size_t smem = medium_smem(hred[0]);
        if (w) GNNB_TRY(launch<true>(p, n_items, smem, st));
        else GNNB_TRY(launch<false>(p, n_items, smem, st));
    }
    int crossed = 0;
    GNNB_CUDA(cudaMemcpyAsync(&crossed, flags + 1, sizeof crossed, cudaMemcpyDeviceToHost, st));
    GNNB_CUDA(cudaStreamSynchronize(st));
    if (crossed)
        GNNB_FAIL(GNNB_EINVAL, "gnnb_ppr_diffusion: an edge crosses segments of seg_ptr (the outputs of its segment are "
                               "not valid; nothing was read or written outside a segment)");
    return GNNB_OK;
}

}  // namespace ppr
}  // namespace gnnb

using namespace gnnb;

extern "C" {

int gnnb_ppr_diffusion(gnnb_graph_t g, const float* w, float alpha, const int64_t* seg_ptr, int64_t n_seg,
                       float* w_out, int32_t* info, void* stream) {
    if (!g) GNNB_FAIL(GNNB_EINVAL, "graph handle is NULL");
    if (g->n_src != g->n_dst) GNNB_FAIL(GNNB_ESIZE, "gnnb_ppr_diffusion needs num_src == num_dst");
    if (seg_ptr && (n_seg < 1 || n_seg >= ((int64_t)1 << 31)))
        GNNB_FAIL(GNNB_EINVAL, "gnnb_ppr_diffusion: n_seg = %lld must be in [1, 2^31)", (long long)n_seg);
    if (g->n_dst == 0) return GNNB_OK;
    if (!info || (g->E > 0 && !w_out)) GNNB_FAIL(GNNB_EINVAL, "gnnb_ppr_diffusion: w_out / info is NULL");
    cudaStream_t st = (cudaStream_t)stream;
    GNNB_TRY(ensure_csr(g, false, st));
    return ppr::run(g, w, alpha, seg_ptr, seg_ptr ? n_seg : 1, w_out, info, st);
}

int gnnb_ppr_matrix(gnnb_graph_t g, const float* w, float alpha, int64_t a, int64_t b, int64_t ld, float* M_out,
                    void* stream) {
    if (!g) GNNB_FAIL(GNNB_EINVAL, "graph handle is NULL");
    if (g->n_src != g->n_dst) GNNB_FAIL(GNNB_ESIZE, "gnnb_ppr_matrix needs num_src == num_dst");
    if (a < 0 || b < a || b > g->n_dst)
        GNNB_FAIL(GNNB_EINVAL, "gnnb_ppr_matrix: [a, b) = [%lld, %lld) must lie in [0, %d]", (long long)a, (long long)b,
                  g->n_dst);
    if (ld < b - a) GNNB_FAIL(GNNB_EINVAL, "gnnb_ppr_matrix: ld = %lld < b - a = %lld", (long long)ld, (long long)(b - a));
    if (a == b) return GNNB_OK;
    if (!M_out) GNNB_FAIL(GNNB_EINVAL, "gnnb_ppr_matrix: M_out is NULL");
    cudaStream_t st = (cudaStream_t)stream;
    GNNB_TRY(ensure_csr(g, false, st));
    DeviceScratch sc(st);
    int* crossed = nullptr;
    GNNB_TRY(sc.alloc(&crossed, 1));
    GNNB_CUDA(cudaMemsetAsync(crossed, 0, sizeof(int), st));
    const int m = (int)(b - a);
    const unsigned grid = (unsigned)ceil_div(m, ppr::WARPS);
    if (w)
        ppr::ppr_matrix_kernel<true><<<grid, ppr::THREADS, 0, st>>>(g->by_dst.rowptr, g->by_dst.col, g->by_dst.eid, w,
                                                                    (int)a, m, ld, alpha, M_out, crossed);
    else
        ppr::ppr_matrix_kernel<false><<<grid, ppr::THREADS, 0, st>>>(g->by_dst.rowptr, g->by_dst.col, g->by_dst.eid,
                                                                     nullptr, (int)a, m, ld, alpha, M_out, crossed);
    GNNB_LAUNCHED();
    int h = 0;
    GNNB_CUDA(cudaMemcpyAsync(&h, crossed, sizeof h, cudaMemcpyDeviceToHost, st));
    GNNB_CUDA(cudaStreamSynchronize(st));
    if (h)
        GNNB_FAIL(GNNB_EINVAL, "gnnb_ppr_matrix: an edge into [a, b) has its source outside it (that row of M_out is "
                               "not valid; nothing was read or written outside it)");
    return GNNB_OK;
}

}  // extern "C"
