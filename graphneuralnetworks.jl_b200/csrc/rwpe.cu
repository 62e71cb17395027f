// rwpe.cu — random_walk_pe on the device: the diagonal of the first K powers of the random-walk matrix, one graph of a
// batch (a segment) at a time, with the walk state in shared memory.
//
// Reference counterpart: random_walk_pe(g, walk_length) (GNNGraphs/src/transform.jl:975-990), which forms the dense
// N x N matrix RW = A * Diagonal(1 ./ deg_out) and multiplies it K times.
//
// Contract (tests/test_random_walk_pe.py restates it in numpy, bit for bit):
//   RW[i, j] = A[i, j] * dinv[j];  PE[k, j] = (RW^k)[j, j], k = 1..K.  Row formulation on the CSR by target:
//   u_0 = e_j,  u_k[t] = dinv[t] * Σ_{edges s -> t, plan order} w_e * u_{k-1}[s],  PE[k, j] = u_k[j].
//   Every product and sum is rounded on its own (__fmul_rn / __fadd_rn); a row without edges is 0.  That is the
//   arithmetic of gnnb_propagate(W_MUL_XJ | COPY_XJ, SUM, ct = dinv) for a row of at most `chunk` edges, so the walk of
//   a segment too large for shared memory (composed from gnnb_propagate by the caller) gives the same bits.
//
// Work decomposition (no atomics, no grid synchronisation):
//   * a work item is a segment and a block of up to 32 consecutive sources of it; lane c owns source src0 + c, so the
//     state of an item is an n x 32 fp32 array [node][lane] (lane c only touches bank c), double-buffered;
//   * small segments (n <= 32): one warp per segment, eight per CTA — a 23-node molecule does not get a CTA of its own;
//   * medium segments (32 < n <= GNNB_RWPE_SMEM_MAX_NODES): one CTA per (segment, 32-source block), the eight warps
//     striding over the segment's rows, one __syncthreads per step;
//   * the K steps of an item run inside it; the owner of row src writes u_k[src] straight to out[src][k].
// The two classes are two launches of rwpe_kernel on the stream, each only when the call has segments of its class: the
// small blocks take 64 KB of shared memory (three CTAs per SM), the medium ones 2 * 128 B per node of the largest medium
// segment of the call.  One launch sized by the largest segment would hold thousands of molecule blocks to one CTA per SM
// as soon as a single ~800-node graph joined the batch.
// A small prep kernel validates seg_ptr and classifies the segments (CUB scan of the medium items, two max reduces); one
// read-back sizes both grids.  Scratch is one allocation per call.
// An edge whose source lies outside its target's segment is never read through: it raises a flag (GNNB_EINVAL).
#include "common.cuh"
#include <cub/cub.cuh>

namespace gnnb {
namespace rwpe {

constexpr int SRC = 32;                     // sources per work item: one lane each
constexpr int WARPS = 8;
constexpr int THREADS = WARPS * 32;
constexpr int MAX_NODES = GNNB_RWPE_SMEM_MAX_NODES;
constexpr size_t SMALL_SMEM = (size_t)WARPS * 2 * SRC * SRC * sizeof(float);            // 64 KB: 8 warps x 2 x 32 x 32
static_assert((size_t)2 * MAX_NODES * SRC * sizeof(float) <= 227 * 1024, "medium state must fit the 227 KB of an SM");

struct Params {
    const int32_t* rowptr;   // CSR by target
    const int32_t* col;      // source of each sorted edge
    const int32_t* eid;      // COO position of each sorted edge (weights are in COO order)
    const float* w;          // NULL: every weight is 1 (no multiply, as COPY_XJ)
    const float* dinv;
    const int64_t* seg;      // [n_seg + 1]
    const int64_t* item_ptr; // [n_seg + 1]: running count of medium work items
    float* out;              // [n][K]
    int* crossed;            // set when an edge crosses segments
    int32_t n_seg, n_small_blocks, K;
};

// u_0 = e_src for the sources src0 .. src0 + 31 of segment [a, a + m), then K steps; warps `warp`, `warp + nwarps`, ...
// own the rows.  CTA = true: the rows of one step are shared by the whole CTA (__syncthreads), otherwise by one warp.
template <bool HAS_W, bool CTA>
__device__ __forceinline__ void walk(const Params& p, float* __restrict__ buf, int a, int m, int src0, int warp,
                                     int nwarps) {
    const int lane = threadIdx.x & 31;
    const int src = src0 + lane;
    float* const u0 = buf;
    float* const u1 = buf + (size_t)m * SRC;
    for (int t = warp; t < m; t += nwarps) u0[t * SRC + lane] = (a + t == src) ? 1.f : 0.f;
    if (CTA) __syncthreads(); else __syncwarp();
    for (int k = 0; k < p.K; ++k) {
        const float* cur = (k & 1) ? u1 : u0;
        float* nxt = (k & 1) ? u0 : u1;
        for (int t = warp; t < m; t += nwarps) {
            const int r = a + t;
            const int e0 = __ldg(p.rowptr + r), e1 = __ldg(p.rowptr + r + 1);
            float acc = 0.f;
            for (int e = e0; e < e1; ++e) {
                const unsigned sl = (unsigned)(__ldg(p.col + e) - a);       // local row of the source
                float v = 0.f;
                if (sl < (unsigned)m) v = cur[sl * SRC + lane];
                else *(volatile int*)p.crossed = 1;                         // never read outside the segment
                if (HAS_W) v = __fmul_rn(v, __ldg(p.w + __ldg(p.eid + e)));
                acc = __fadd_rn(acc, v);
            }
            const float val = e1 > e0 ? __fmul_rn(acc, __ldg(p.dinv + r)) : 0.f;
            nxt[t * SRC + lane] = val;
            if (r == src) p.out[(size_t)src * p.K + k] = val;
        }
        if (CTA) __syncthreads(); else __syncwarp();
    }
}

template <bool HAS_W>
__global__ void __launch_bounds__(THREADS) rwpe_kernel(const Params p) {
    extern __shared__ __align__(16) float smem[];
    const int warp = threadIdx.x >> 5;
    if ((int)blockIdx.x < p.n_small_blocks) {               // small segments: one warp each
        const int s = blockIdx.x * WARPS + warp;
        if (s >= p.n_seg) return;
        const int a = (int)p.seg[s], m = (int)(p.seg[s + 1] - a);
        if (m <= 0 || m > SRC) return;
        walk<HAS_W, false>(p, smem + (size_t)warp * 2 * SRC * SRC, a, m, a, 0, 1);
        return;
    }
    const int64_t item = (int64_t)blockIdx.x - p.n_small_blocks;   // medium: (segment, 32-source block)
    int lo = 0, hi = p.n_seg;                                        // item_ptr[lo] <= item < item_ptr[lo + 1]
    while (hi - lo > 1) {
        const int mid = (lo + hi) >> 1;
        if (p.item_ptr[mid] <= item) lo = mid; else hi = mid;
    }
    const int a = (int)p.seg[lo], m = (int)(p.seg[lo + 1] - a);
    if (m <= SRC || m > MAX_NODES) return;                           // block-uniform: no barrier is skipped by half a CTA
    walk<HAS_W, true>(p, smem, a, m, a + (int)(item - p.item_ptr[lo]) * SRC, warp, WARPS);
}

// per segment: medium items (ceil(n / 32) for 32 < n <= MAX_NODES, else 0), its node count if medium, and whether it is
// small (1 <= n <= 32); bad = 1 for a malformed seg_ptr (every writer stores the same value)
__global__ void classify_kernel(const int64_t* __restrict__ seg, int64_t n_seg, int64_t n, int64_t* __restrict__ items,
                                int32_t* __restrict__ med_nodes, int32_t* __restrict__ small, int* __restrict__ bad) {
    const int64_t s = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (s >= n_seg) return;
    const int64_t a = seg[s], b = seg[s + 1];
    const bool ok = !((s == 0 && a != 0) || (s == n_seg - 1 && b != n) || b < a || a < 0 || b > n);
    if (!ok) *(volatile int*)bad = 1;
    const bool med = ok && b - a > SRC && b - a <= MAX_NODES;
    items[s] = med ? (b - a + SRC - 1) / SRC : 0;
    med_nodes[s] = med ? (int32_t)(b - a) : 0;
    small[s] = (ok && b > a && b - a <= SRC) ? 1 : 0;
}

template <bool HAS_W>
static int launch(const Params& p, int64_t grid, size_t smem, cudaStream_t st) {
    auto kern = rwpe_kernel<HAS_W>;
    GNNB_CUDA(cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
    kern<<<(unsigned)grid, THREADS, smem, st>>>(p);
    GNNB_LAUNCHED();
    return GNNB_OK;
}

static size_t align256(size_t b) { return (b + 255) & ~(size_t)255; }

static int run(gnnb_graph* g, const float* w, const float* dinv, const int64_t* seg_ptr, int64_t n_seg, int K, float* out,
               cudaStream_t st) {
    const int64_t n = g->n_dst;
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
    classify_kernel<<<(unsigned)ceil_div(n_seg, 256), 256, 0, st>>>(seg_ptr, n_seg, n, items, med, small, flags);
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
    p.w = w; p.dinv = dinv; p.seg = seg_ptr; p.item_ptr = item_ptr; p.out = out; p.crossed = flags + 1;
    p.n_seg = (int32_t)n_seg; p.K = K;
    if (hred[1]) {                                      // small segments: every block of this launch is small
        p.n_small_blocks = (int32_t)ceil_div(n_seg, WARPS);
        if (w) GNNB_TRY(launch<true>(p, p.n_small_blocks, SMALL_SMEM, st));
        else GNNB_TRY(launch<false>(p, p.n_small_blocks, SMALL_SMEM, st));
    }
    if (n_items) {                                      // medium segments: every block of this launch is medium
        p.n_small_blocks = 0;
        const size_t smem = (size_t)2 * hred[0] * SRC * sizeof(float);
        if (w) GNNB_TRY(launch<true>(p, n_items, smem, st));
        else GNNB_TRY(launch<false>(p, n_items, smem, st));
    }
    int crossed = 0;
    GNNB_CUDA(cudaMemcpyAsync(&crossed, flags + 1, sizeof crossed, cudaMemcpyDeviceToHost, st));
    GNNB_CUDA(cudaStreamSynchronize(st));
    if (crossed)
        GNNB_FAIL(GNNB_EINVAL, "gnnb_random_walk_pe: an edge crosses segments of seg_ptr (the rows of its segment are "
                               "not valid; nothing was read or written outside a segment)");
    return GNNB_OK;
}

}  // namespace rwpe
}  // namespace gnnb

using namespace gnnb;

extern "C" {

int gnnb_random_walk_pe(gnnb_graph_t g, const float* w, const float* dinv, const int64_t* seg_ptr, int64_t n_seg,
                        int walk_length, float* out, void* stream) {
    if (!g) GNNB_FAIL(GNNB_EINVAL, "graph handle is NULL");
    if (g->n_src != g->n_dst) GNNB_FAIL(GNNB_ESIZE, "gnnb_random_walk_pe needs num_src == num_dst");
    if (walk_length < 1) GNNB_FAIL(GNNB_EINVAL, "gnnb_random_walk_pe: walk_length = %d must be >= 1", walk_length);
    if (seg_ptr && (n_seg < 1 || n_seg >= ((int64_t)1 << 31)))
        GNNB_FAIL(GNNB_EINVAL, "gnnb_random_walk_pe: n_seg = %lld must be in [1, 2^31)", (long long)n_seg);
    if (g->n_dst == 0) return GNNB_OK;
    if (!dinv || !out) GNNB_FAIL(GNNB_EINVAL, "gnnb_random_walk_pe: dinv / out is NULL");
    cudaStream_t st = (cudaStream_t)stream;
    GNNB_TRY(ensure_csr(g, false, st));
    return rwpe::run(g, w, dinv, seg_ptr, seg_ptr ? n_seg : 1, walk_length, out, st);
}

}  // extern "C"
