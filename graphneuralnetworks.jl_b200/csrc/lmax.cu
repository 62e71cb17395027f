// lmax.cu — laplacian_lambda_max on the device: the largest eigenvalue of each graph of a batch (a segment), from its
// dense symmetric matrix in shared memory, and the segmented dot products of the batched Lanczos route for larger ones.
//
// Reference counterpart: laplacian_lambda_max(g; add_self_loops, dir) (GNNGraphs/src/query.jl:598-610), which calls
// KrylovKit's eigsolve(Symmetric(L), x0, 1, :LR) on L = I - D^-1/2 A D^-1/2 of every getgraph(g, i) on the host.
// `Symmetric` reads the upper triangle of L, so the eigenvalue is that of S: S[i][j] = S[j][i] = L[i][j] for i < j,
// S[i][i] = L[i][i].  A lower-triangle entry of L only counts through the degrees.
//
// Contract (tests/test_laplacian.py restates it in float64):
//   c[i] = 1 / sqrt(deg[base + i]) in double (deg: the caller's float32 degree, self loops included).
//   Row i of a segment [base, base + n) starts as zeros; for dir = out its out-edges i -> t with t >= i (by_src plan
//   order) and then its in-edges s -> i with s < i (by_dst plan order) add their weight at the other end's column, in
//   double; for dir = in the out-edges with t <= i and the in-edges with s > i.  A self loop is read once, from the
//   out-edges.  Then S[i][j] = -((c[i] * a[i][j]) * c[j]) for j != i and S[i][i] = 1 - (c[i] * (a[i][i] + loops)) * c[i]
//   with loops = 1 under add_self_loops.
//   Householder tridiagonalisation (row k of the trailing matrix is its reflector's x), then the largest eigenvalue of
//   the tridiagonal matrix by Sturm-count multisection from its Gershgorin interval until no point between the
//   bracketing pair is representable; lmax_out = the upper end.  A non-finite tridiagonal entry gives NaN.
//
// Work decomposition: each dot product (a row of the trailing block times the reflector, the norms) is one warp's: lane
// l adds elements l, l + 32, ... in order with fma, then a fixed xor butterfly.  The rank-2 update is elementwise.  So a
// segment gives the same bits whichever class runs it:
//   * small segments (n <= 32): one warp per segment, eight per CTA, __syncwarp between phases;
//   * medium segments (32 < n <= GNNB_LMAX_SMEM_MAX_NODES): one CTA of 256 threads per segment, a __syncthreads between
//     phases, the matrix sized by the largest medium segment of the call.
// gnnb_set_kernel_variant(12) sends every segment through the CTA class, which the tests use to check that.  The
// classes are two launches, as in ppr.cu; a prep kernel validates seg_ptr and classifies the segments.  An edge with an
// end outside its segment is never read through: the smallest such COO id is kept and reported (GNNB_EINVAL).
#include "common.cuh"
#include <cub/cub.cuh>
#include <cfloat>

namespace gnnb {
extern bool g_reference_kernels;   // segreduce.cu: gnnb_set_kernel_variant(12)

namespace lmax {

constexpr int SMALL = 32;
constexpr int WARPS = 8;
constexpr int THREADS = WARPS * 32;
constexpr int MAX_NODES = GNNB_LMAX_SMEM_MAX_NODES;
constexpr int SCALARS = 4;                   // two broadcast slots for |x|^2 and two for K, alternating by step

__host__ __device__ constexpr size_t seg_doubles(int n) { return (size_t)n * n + 2 * (size_t)n + SCALARS; }
__host__ __device__ constexpr size_t seg_bytes(int n) { return sizeof(double) * seg_doubles(n); }
constexpr size_t SMALL_SMEM = (size_t)WARPS * seg_bytes(SMALL);
// 232 448 B (227 KB) is the opt-in shared memory of one H100 CTA: GNNB_LMAX_SMEM_MAX_NODES is the largest n whose
// matrix and two working vectors fit it.  The entry checks the device's own limit at run time.
static_assert(seg_bytes(MAX_NODES) <= 232448 && seg_bytes(MAX_NODES + 1) > 232448,
              "GNNB_LMAX_SMEM_MAX_NODES must be the largest segment whose matrix fits 227 KB");
static_assert(MAX_NODES <= THREADS, "a CTA builds every row of a medium segment in one pass");

struct Params {
    const int32_t* in_rowptr;   // CSR by target: in-edges
    const int32_t* in_col;
    const int32_t* in_eid;
    const int32_t* out_rowptr;  // CSR by source: out-edges
    const int32_t* out_col;
    const int32_t* out_eid;
    const float* w;             // NULL: every weight is 1
    const float* deg;
    const int64_t* seg;         // [n_seg + 1]
    const int64_t* item_ptr;    // [n_seg + 1]: running count of medium segments
    double* lmax;
    int* crossed;               // the smallest COO id of an edge leaving its segment (INT_MAX: none)
    int32_t n_seg, n_small_blocks;
    int dir_out, self_loops;
};

__device__ __forceinline__ double warp_sum(double a) {
#pragma unroll
    for (int o = 16; o; o >>= 1) a = __dadd_rn(a, __shfl_xor_sync(0xffffffffu, a, o));
    return a;                                // the same bits in every lane: each step adds the same two values
}

// sum_i a[i] * b[i] over i < len by one warp, in the fixed order of the contract
__device__ __forceinline__ double warp_dot(const double* a, const double* b, int len, int lane) {
    double acc = 0.0;
    for (int i = lane; i < len; i += 32) acc = __fma_rn(a[i], b[i], acc);
    return warp_sum(acc);
}

template <bool CTA>
__device__ __forceinline__ void sync_group() {
    if (CTA) __syncthreads(); else __syncwarp();
}

// the number of eigenvalues below x of the tridiagonal matrix (d = A[i][i], e = A[i][i + 1]): the signs of the LDL^T
// pivots, a pivot of magnitude <= pivmin replaced by -pivmin
__device__ __forceinline__ int sturm_count(const double* A, int n, double x, double pivmin) {
    double q = __dsub_rn(A[0], x);
    if (fabs(q) <= pivmin) q = -pivmin;
    int cnt = q < 0.0;
    for (int i = 1; i < n; ++i) {
        const double e = A[(size_t)(i - 1) * n + i];
        q = __dsub_rn(__dsub_rn(A[(size_t)i * n + i], x), __ddiv_rn(__dmul_rn(e, e), q));
        if (fabs(q) <= pivmin) q = -pivmin;
        cnt += q < 0.0;
    }
    return cnt;
}

__device__ __forceinline__ void flag_crossing(int* crossed, int eid) { atomicMin(crossed, eid); }

// The segment [base, base + n): matrix `A` (n x n), vectors v and q (n each), scalar slots sc; `tid` = thread of the
// group (a warp or the CTA), nthr its size.  Exits uniformly across the group.  The four pointers are not __restrict__:
// every phase reads what other threads of the group wrote before the barrier, which a restrict-qualified load may not
// see.
template <bool HAS_W, bool CTA>
__device__ __forceinline__ void lmax_segment(const Params& p, double* A, double* v, double* q, double* sc, int s,
                                             int base, int n, int tid, int nthr) {
    const int lane = tid & 31, warp = tid >> 5, nwarps = nthr >> 5;
    for (int i = tid; i < n; i += nthr) q[i] = __ddiv_rn(1.0, __dsqrt_rn((double)__ldg(p.deg + base + i)));
    sync_group<CTA>();
    for (int i = tid; i < n; i += nthr) {    // row i of S
        double* row = A + (size_t)i * n;
        for (int j = 0; j < n; ++j) row[j] = 0.0;
        const int o0 = __ldg(p.out_rowptr + base + i), o1 = __ldg(p.out_rowptr + base + i + 1);
        for (int e = o0; e < o1; ++e) {
            const int id = __ldg(p.out_eid + e);
            const unsigned tl = (unsigned)(__ldg(p.out_col + e) - base);
            if (tl >= (unsigned)n) { flag_crossing(p.crossed, id); continue; }
            if ((int)tl == i || (p.dir_out ? (int)tl > i : (int)tl < i))
                row[tl] = __dadd_rn(row[tl], HAS_W ? (double)__ldg(p.w + id) : 1.0);
        }
        const int i0 = __ldg(p.in_rowptr + base + i), i1 = __ldg(p.in_rowptr + base + i + 1);
        for (int e = i0; e < i1; ++e) {
            const int id = __ldg(p.in_eid + e);
            const unsigned sl = (unsigned)(__ldg(p.in_col + e) - base);
            if (sl >= (unsigned)n) { flag_crossing(p.crossed, id); continue; }
            if (p.dir_out ? (int)sl < i : (int)sl > i)
                row[sl] = __dadd_rn(row[sl], HAS_W ? (double)__ldg(p.w + id) : 1.0);
        }
        const double ci = q[i];
        for (int j = 0; j < n; ++j) {
            if (j == i) {
                const double a = p.self_loops ? __dadd_rn(row[j], 1.0) : row[j];
                row[j] = __dsub_rn(1.0, __dmul_rn(__dmul_rn(ci, a), ci));
            } else {
                row[j] = -__dmul_rn(__dmul_rn(ci, row[j]), q[j]);
            }
        }
    }
    sync_group<CTA>();
    // Householder: step k zeroes row / column k beyond k + 1 of the trailing matrix; its first off-diagonal entry
    // becomes alpha (the tridiagonal e_k, kept at A[k][k + 1])
    for (int k = 0; k + 2 < n; ++k) {
        const int m = n - k - 1;
        double* x = A + (size_t)k * n + k + 1;
        if (warp == 0) {
            const double t = warp_dot(x + 1, x + 1, m - 1, lane);
            if (lane == 0) sc[k & 1] = t;
        }
        sync_group<CTA>();
        const double sigma = sc[k & 1];
        if (sigma == 0.0) continue;                      // uniform: the column is already reduced
        const double x0 = x[0];
        const double alpha = -copysign(__dsqrt_rn(__fma_rn(x0, x0, sigma)), x0);
        const double v0 = __dsub_rn(x0, alpha);
        const double tau = __ddiv_rn(2.0, __fma_rn(v0, v0, sigma));
        for (int j = tid; j < m; j += nthr) v[j] = j == 0 ? v0 : x[j];
        sync_group<CTA>();
        for (int r = warp; r < m; r += nwarps) {         // q = tau * A22 v
            const double t = warp_dot(A + (size_t)(k + 1 + r) * n + k + 1, v, m, lane);
            if (lane == 0) q[r] = __dmul_rn(tau, t);
        }
        sync_group<CTA>();
        if (warp == 0) {                                 // K = tau / 2 * v.q
            const double t = warp_dot(v, q, m, lane);
            if (lane == 0) sc[2 + (k & 1)] = __dmul_rn(__dmul_rn(0.5, tau), t);
        }
        sync_group<CTA>();
        const double Kc = sc[2 + (k & 1)];
        for (int j = tid; j < m; j += nthr) q[j] = __fma_rn(-Kc, v[j], q[j]);   // w = q - K v
        sync_group<CTA>();
        for (int r = warp; r < m; r += nwarps) {         // A22 -= v w^T + w v^T
            double* row = A + (size_t)(k + 1 + r) * n + k + 1;
            const double vr = v[r], wr = q[r];
            for (int c = lane; c < m; c += 32)
                row[c] = __dsub_rn(row[c], __fma_rn(vr, q[c], __dmul_rn(wr, v[c])));
        }
        if (tid == 0) x[0] = alpha;
        sync_group<CTA>();
    }
    if (warp != 0) return;
    // the tridiagonal matrix: Gershgorin interval, finiteness, the pivot floor
    double lo = INFINITY, hi = -INFINITY, e2 = 0.0;
    bool finite = true;
    for (int i = lane; i < n; i += 32) {
        const double d = A[(size_t)i * n + i];
        const double el = i > 0 ? fabs(A[(size_t)(i - 1) * n + i]) : 0.0;
        const double er = i + 1 < n ? fabs(A[(size_t)i * n + i + 1]) : 0.0;
        finite = finite && isfinite(d) && isfinite(el) && isfinite(er);
        lo = fmin(lo, __dsub_rn(__dsub_rn(d, el), er));
        hi = fmax(hi, __dadd_rn(__dadd_rn(d, el), er));
        e2 = fmax(e2, __dmul_rn(er, er));
    }
#pragma unroll
    for (int o = 16; o; o >>= 1) {
        lo = fmin(lo, __shfl_xor_sync(0xffffffffu, lo, o));
        hi = fmax(hi, __shfl_xor_sync(0xffffffffu, hi, o));
        e2 = fmax(e2, __shfl_xor_sync(0xffffffffu, e2, o));
    }
    finite = __all_sync(0xffffffffu, finite) && isfinite(e2);
    if (!finite) {
        if (lane == 0) p.lmax[s] = __longlong_as_double(0x7ff8000000000000ll);
        return;
    }
    const double pivmin = DBL_MIN * fmax(1.0, e2);
    const double delta = 0x1p-40 * fmax(hi - lo, fmax(fabs(lo), fabs(hi))) + pivmin;
    lo -= delta;
    hi += delta;                                         // count(lo) < n == count(hi)
    for (int it = 0; it < 64; ++it) {                    // 33-section: about 12 rounds reach the last bit
        const double x = __fma_rn(__ddiv_rn((double)(lane + 1), 33.0), __dsub_rn(hi, lo), lo);
        const unsigned all = __ballot_sync(0xffffffffu, sturm_count(A, n, x, pivmin) == n);
        const int f = all ? __ffs(all) - 1 : 32;         // the first point above every eigenvalue
        const double xf = __shfl_sync(0xffffffffu, x, f & 31), xp = __shfl_sync(0xffffffffu, x, (f + 31) & 31);
        const double nhi = f < 32 ? xf : hi, nlo = f > 0 ? xp : lo;
        if (nhi == hi && nlo == lo) break;
        lo = nlo;
        hi = nhi;
    }
    if (lane == 0) p.lmax[s] = hi;
}

template <bool HAS_W>
__global__ void __launch_bounds__(THREADS) lmax_kernel(const Params p) {
    extern __shared__ __align__(16) unsigned char smem_raw[];
    const int warp = threadIdx.x >> 5;
    if ((int)blockIdx.x < p.n_small_blocks) {            // small segments: one warp each
        const int s = blockIdx.x * WARPS + warp;
        if (s >= p.n_seg) return;
        const int a = (int)p.seg[s], m = (int)(p.seg[s + 1] - a);
        if (m <= 0 || m > SMALL) return;
        double* A = reinterpret_cast<double*>(smem_raw) + (size_t)warp * seg_doubles(SMALL);
        lmax_segment<HAS_W, false>(p, A, A + (size_t)m * m, A + (size_t)m * m + m, A + (size_t)m * m + 2 * m, s, a, m,
                                   threadIdx.x & 31, 32);
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
    double* A = reinterpret_cast<double*>(smem_raw);
    lmax_segment<HAS_W, true>(p, A, A + (size_t)m * m, A + (size_t)m * m + m, A + (size_t)m * m + 2 * m, lo, a, m,
                              threadIdx.x, THREADS);
}

// per segment: medium (1 for a segment of the CTA class), its node count if medium, whether it is small, info = -1 for
// a segment above the bound and 0 otherwise, NaN for a segment without nodes; bad = 1 for a malformed seg_ptr
__global__ void classify_kernel(const int64_t* __restrict__ seg, int64_t n_seg, int64_t n, int all_medium,
                                int64_t* __restrict__ items, int32_t* __restrict__ med_nodes,
                                int32_t* __restrict__ small, int32_t* __restrict__ info, double* __restrict__ lmax,
                                int* __restrict__ bad) {
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
    if (ok && m == 0) lmax[s] = __longlong_as_double(0x7ff8000000000000ll);
}

template <bool HAS_W>
static int launch(const Params& p, int64_t grid, size_t smem, cudaStream_t st) {
    auto kern = lmax_kernel<HAS_W>;
    GNNB_CUDA(cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
    kern<<<(unsigned)grid, THREADS, smem, st>>>(p);
    GNNB_LAUNCHED();
    return GNNB_OK;
}

static size_t align256(size_t b) { return (b + 255) & ~(size_t)255; }

static int run(gnnb_graph* g, const float* w, const float* deg, int dir, int self_loops, const int64_t* seg_ptr,
               int64_t n_seg, double* lmax_out, int32_t* info, cudaStream_t st) {
    const int64_t n = g->n_dst;
    int dev = 0, optin = 0;
    GNNB_CUDA(cudaGetDevice(&dev));
    GNNB_CUDA(cudaDeviceGetAttribute(&optin, cudaDevAttrMaxSharedMemoryPerBlockOptin, dev));
    if ((size_t)optin < seg_bytes(MAX_NODES))
        GNNB_FAIL(GNNB_EUNSUPPORTED, "gnnb_laplacian_lambda_max: a segment of %d nodes needs %zu B of shared memory "
                                     "per CTA, the device allows %d", MAX_NODES, seg_bytes(MAX_NODES), optin);
    // one scratch allocation: int64 items [n_seg], item_ptr [n_seg + 1], the default segment [2]; int32 medium node
    // counts [n_seg], small flags [n_seg], their two maxima [2]; int flags [2] (bad seg_ptr, the crossing edge); CUB
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
    const int hflags[2] = {0, INT_MAX};
    GNNB_CUDA(cudaMemcpyAsync(flags, hflags, sizeof hflags, cudaMemcpyHostToDevice, st));
    if (!seg_ptr) {
        int64_t* dseg = item_ptr + n_seg + 1;
        const int64_t h[2] = {0, n};
        GNNB_CUDA(cudaMemcpyAsync(dseg, h, sizeof h, cudaMemcpyHostToDevice, st));
        seg_ptr = dseg;
    }
    GNNB_CUDA(cudaMemsetAsync(item_ptr, 0, sizeof(int64_t), st));
    classify_kernel<<<(unsigned)ceil_div(n_seg, 256), 256, 0, st>>>(seg_ptr, n_seg, n, g_reference_kernels ? 1 : 0,
                                                                     items, med, small, info, lmax_out, flags);
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
    p.in_rowptr = g->by_dst.rowptr; p.in_col = g->by_dst.col; p.in_eid = g->by_dst.eid;
    p.out_rowptr = g->by_src.rowptr; p.out_col = g->by_src.col; p.out_eid = g->by_src.eid;
    p.w = w; p.deg = deg; p.seg = seg_ptr; p.item_ptr = item_ptr; p.lmax = lmax_out; p.crossed = flags + 1;
    p.n_seg = (int32_t)n_seg; p.dir_out = dir == GNNB_DIR_OUT; p.self_loops = self_loops != 0;
    if (hred[1]) {                                      // small segments: every block of this launch is small
        p.n_small_blocks = (int32_t)ceil_div(n_seg, WARPS);
        if (w) GNNB_TRY(launch<true>(p, p.n_small_blocks, SMALL_SMEM, st));
        else GNNB_TRY(launch<false>(p, p.n_small_blocks, SMALL_SMEM, st));
    }
    if (n_items) {                                      // medium segments: every block of this launch is medium
        p.n_small_blocks = 0;
        const size_t smem = seg_bytes(hred[0]);
        if (w) GNNB_TRY(launch<true>(p, n_items, smem, st));
        else GNNB_TRY(launch<false>(p, n_items, smem, st));
    }
    int crossed = INT_MAX;
    GNNB_CUDA(cudaMemcpyAsync(&crossed, flags + 1, sizeof crossed, cudaMemcpyDeviceToHost, st));
    GNNB_CUDA(cudaStreamSynchronize(st));
    if (crossed != INT_MAX) {
        int32_t ends[2] = {0, 0};
        GNNB_CUDA(cudaMemcpy(ends, g->coo_src + crossed, sizeof(int32_t), cudaMemcpyDeviceToHost));
        GNNB_CUDA(cudaMemcpy(ends + 1, g->coo_dst + crossed, sizeof(int32_t), cudaMemcpyDeviceToHost));
        GNNB_FAIL(GNNB_EINVAL, "gnnb_laplacian_lambda_max: edge %d (%d -> %d, 0-based) crosses segments of seg_ptr (the "
                               "results of its segments are not valid; nothing was read or written outside a segment)",
                  crossed, ends[0], ends[1]);
    }
    return GNNB_OK;
}

// ---- segmented dot products of the Lanczos route: chunks of DOT_CHUNK nodes counted from each segment's start
constexpr int DOT_CHUNK = GNNB_SEGDOT_CHUNK;

// partial[b][k] = sum over chunk b of X[k][i] * y[i]: thread t adds nodes t, t + 256, ... in order, then a fixed tree
__global__ void __launch_bounds__(THREADS) segdot_partial_kernel(const double* __restrict__ X, int64_t ldx,
                                                                 const double* __restrict__ y,
                                                                 const int64_t* __restrict__ seg,
                                                                 const int64_t* __restrict__ chunk_ptr, int n_seg,
                                                                 int64_t n, double* __restrict__ partial) {
    __shared__ double part[WARPS];
    const int64_t b = blockIdx.x;
    const int k = blockIdx.y, K = gridDim.y;
    int lo = 0, hi = n_seg;
    while (hi - lo > 1) {
        const int mid = (lo + hi) >> 1;
        if (chunk_ptr[mid] <= b) lo = mid; else hi = mid;
    }
    int64_t a = seg[lo] + (b - chunk_ptr[lo]) * DOT_CHUNK, e = a + DOT_CHUNK;
    if (e > seg[lo + 1]) e = seg[lo + 1];
    if (a < 0) a = 0;
    if (e > n) e = n;
    const double* x = X + (size_t)k * ldx;
    double acc = 0.0;
    for (int64_t i = a + threadIdx.x; i < e; i += THREADS) acc = __fma_rn(x[i], y[i], acc);
    acc = warp_sum(acc);
    if ((threadIdx.x & 31) == 0) part[threadIdx.x >> 5] = acc;
    __syncthreads();
    if (threadIdx.x == 0) {
        double t = part[0];
#pragma unroll
        for (int w = 1; w < WARPS; ++w) t = __dadd_rn(t, part[w]);
        partial[b * K + k] = t;
    }
}

// out[s][k] = the partials of segment s's chunks added in order (0 for a segment without nodes)
__global__ void segdot_final_kernel(const double* __restrict__ partial, const int64_t* __restrict__ chunk_ptr,
                                    int64_t n_seg, int K, double* __restrict__ out) {
    const int64_t idx = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (idx >= n_seg * K) return;
    const int64_t s = idx / K, k = idx % K;
    double t = 0.0;
    for (int64_t c = chunk_ptr[s]; c < chunk_ptr[s + 1]; ++c) t = __dadd_rn(t, partial[c * K + k]);
    out[idx] = t;
}

}  // namespace lmax
}  // namespace gnnb

using namespace gnnb;

extern "C" {

int gnnb_laplacian_lambda_max(gnnb_graph_t g, const float* w, const float* deg, int dir, int add_self_loops,
                              const int64_t* seg_ptr, int64_t n_seg, double* lmax_out, int32_t* info, void* stream) {
    if (!g) GNNB_FAIL(GNNB_EINVAL, "graph handle is NULL");
    if (g->n_src != g->n_dst) GNNB_FAIL(GNNB_ESIZE, "gnnb_laplacian_lambda_max needs num_src == num_dst");
    if (dir != GNNB_DIR_OUT && dir != GNNB_DIR_IN && dir != GNNB_DIR_BOTH)
        GNNB_FAIL(GNNB_EINVAL, "gnnb_laplacian_lambda_max: dir = %d is not a gnnb_dir", dir);
    if (seg_ptr && (n_seg < 1 || n_seg >= ((int64_t)1 << 31)))
        GNNB_FAIL(GNNB_EINVAL, "gnnb_laplacian_lambda_max: n_seg = %lld must be in [1, 2^31)", (long long)n_seg);
    if (!info || !lmax_out) GNNB_FAIL(GNNB_EINVAL, "gnnb_laplacian_lambda_max: lmax_out / info is NULL");
    if (g->n_dst > 0 && !deg) GNNB_FAIL(GNNB_EINVAL, "gnnb_laplacian_lambda_max: deg is NULL");
    cudaStream_t st = (cudaStream_t)stream;
    GNNB_TRY(ensure_csr(g, false, st));
    GNNB_TRY(ensure_csr(g, true, st));
    return lmax::run(g, w, deg, dir, add_self_loops, seg_ptr, seg_ptr ? n_seg : 1, lmax_out, info, st);
}

int gnnb_segment_dots(const double* X, int64_t K, int64_t ldx, const double* y, int64_t n, const int64_t* seg_ptr,
                      const int64_t* chunk_ptr, int64_t n_seg, int64_t n_chunks, double* partial, double* out,
                      void* stream) {
    if (K < 1 || K > 65535 || ldx < n || n < 0)
        GNNB_FAIL(GNNB_EINVAL, "gnnb_segment_dots: K = %lld must be in [1, 65535] and ldx = %lld >= n = %lld >= 0",
                  (long long)K, (long long)ldx, (long long)n);
    if (n_seg < 1 || n_seg >= ((int64_t)1 << 31) || n_chunks < 0 || n_chunks >= ((int64_t)1 << 31))
        GNNB_FAIL(GNNB_EINVAL, "gnnb_segment_dots: n_seg = %lld must be in [1, 2^31), n_chunks = %lld in [0, 2^31)",
                  (long long)n_seg, (long long)n_chunks);
    if (!seg_ptr || !chunk_ptr || !out || (n_chunks > 0 && (!X || !y || !partial)))
        GNNB_FAIL(GNNB_EINVAL, "gnnb_segment_dots: a pointer is NULL");
    cudaStream_t st = (cudaStream_t)stream;
    if (n_chunks > 0) {
        lmax::segdot_partial_kernel<<<dim3((unsigned)n_chunks, (unsigned)K), lmax::THREADS, 0, st>>>(
            X, ldx, y, seg_ptr, chunk_ptr, (int)n_seg, n, partial);
        GNNB_LAUNCHED();
    }
    lmax::segdot_final_kernel<<<(unsigned)ceil_div(n_seg * K, 256), 256, 0, st>>>(partial, chunk_ptr, n_seg, (int)K,
                                                                                   out);
    GNNB_LAUNCHED();
    return GNNB_OK;
}

}  // extern "C"
