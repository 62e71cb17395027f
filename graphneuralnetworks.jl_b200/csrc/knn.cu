// knn.cu — knn_graph / radius_graph on the device: exact fp32 distances, brute force within segments (one segment per
// graph of a batch), deterministic neighbour order.
//
// Reference counterpart: knn_graph / radius_graph (GNNGraphs/src/generate.jl:112-145, 196-222), which build a KDTree /
// BallTree with NearestNeighbors.jl on the CPU and separate graphs of a batch by an extra dummy coordinate.  The same
// count / fill kernels, with the hyperbolic pair test as their policy, build rand_temporal_hyperbolic_graph's snapshots
// (generate.jl:340-380, a dense n x n adjacency per snapshot there).
//
// Contract (the oracle restates it bit for bit):
//   d2(i, j) = Σ_{f = 0..d-1} (p_i[f] - p_j[f])², ascending f, sub / mul / add each rounded on its own (no FMA);
//   a NaN d2 counts as +Inf.  The key of candidate j for query i is (d2, j), compared lexicographically; since d2 >= +0
//   the fp32 bits order like the values (bits(d2) + 1 keeps 0 free as a sentinel below every real distance).
//   knn:    the k smallest keys of the segment (j == i excluded unless self_loops), in ascending key order.
//   radius: every j of the segment with sqrt_rn(d2) <= r (j == i excluded unless self_loops), in ascending j.
//   hyperbolic: records (C, S, c, s) of 4 doubles; x(i, j) = C_i C_j - (S_i S_j)(c_i c_j + s_i s_j), every mul / add /
//   sub rounded on its own (so x(i, j) == x(j, i) bit for bit); j is in the row when the two records are equal or
//   x <= x_max (a NaN x is not), j == i excluded unless self_loops, in ascending j.
//
// Work decomposition: a work item is a query tile of QT consecutive points of one segment (one thread per query), so
// one segment of 2^18 points gives 2048 items and 1024 segments of 1000 give 8192: both fill the 132 SMs.  The tile
// offsets per segment are built on the device (count + CUB scan) and the item grid is launched at its upper bound
// n / QT + n_seg, so a call is O(1) launches with no host round trip before the main kernel.  Every item streams its
// segment's candidate points through two shared-memory buffers: one 1-D cp.async.bulk per tile (the 16 B aligned
// interior of the tile's byte range; the < 16 B head and tail are loaded by threads), completion on an mbarrier
// (complete_tx), the next-but-one tile in flight while the current one is scanned.  Each thread visits the candidates in
// ascending j and keeps its running top-k as KB sorted (distance bits, j) pairs in registers; a candidate is rejected
// against the k-th distance before any insertion work.  Because j only grows, a new candidate goes after every held
// entry of equal distance, so the 32-bit distance compare alone keeps the (d2, j) order.
//
// Query coordinates sit in registers for d <= 64 (DREG = 3 exactly, or buckets 4, 16, 64 with loops unrolled to DREG and
// cut at d); larger d
// (<= 256) keeps the query tile in shared memory (DREG = 0, QT = 64).  The work is fp32-issue bound: 3d separately
// rounded instructions per pair.
#include "common.cuh"
#include "tma.cuh"
#include <cub/cub.cuh>

namespace gnnb {
namespace knn {

enum { KNN = 0, COUNT = 1, FILL = 2 };
enum { EUCLID = 0, HYPERBOLIC = 1 };                   // the pair test of the count / fill kernels

constexpr int BUF_FLOATS = 4096;                       // candidate floats per tile
constexpr int BUF_BYTES = BUF_FLOATS * 4 + 16;         // + the 16 B alignment slack of the tile's first row
constexpr int MAX_K = 64;
constexpr int MAX_D = 256;

struct Params {
    const float* pts;        // [n][d]
    const int64_t* seg;      // [n_seg + 1]
    const int64_t* tile_ptr; // [n_seg + 1]: running count of query tiles
    int n_seg, d, k, self_loops, ct;
    float r;
    int32_t* nbr;            // KNN: [n][k];  FILL: flat, rows at offsets
    int64_t* counts;         // COUNT: [n]
    const int64_t* offsets;  // FILL: [n + 1]
    int64_t capacity;        // FILL: entries of nbr
    int* err;                // pipeline stall flag
    int* mismatch;           // FILL: a row's hits differ from offsets[i+1] - offsets[i]
    const int* bad;          // segment validation flags (the item kernel does nothing if set)
    double xmax;             // HYPERBOLIC: the largest x of an edge
};

__device__ __forceinline__ void fence_mbar_init() { asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory"); }

// bits(d2) + 1 with NaN as +Inf (fminf returns the non-NaN operand): ordered like d2, and 0 stays free as a sentinel
__device__ __forceinline__ uint32_t dist_key(float d2) { return __float_as_uint(fminf(d2, __int_as_float(0x7f800000))) + 1u; }

__device__ __forceinline__ float sq_term(float a, float b) {
    const float t = __fsub_rn(a, b);
    return __fmul_rn(t, t);
}

// x = C_q C_c - (S_q S_c)(c_q c_c + s_q s_c) <= xmax, or the records are equal.  Each operation is rounded on its own and
// IEEE products and sums commute, so the test is symmetric in q and c bit for bit.
__device__ __forceinline__ bool hyperbolic_hit(const double* q, const double* c, double xmax) {
    const double ang = __dadd_rn(__dmul_rn(q[2], c[2]), __dmul_rn(q[3], c[3]));
    const double x = __dsub_rn(__dmul_rn(q[0], c[0]), __dmul_rn(__dmul_rn(q[1], c[1]), ang));
    return x <= xmax || (q[0] == c[0] && q[1] == c[1] && q[2] == c[2] && q[3] == c[3]);
}

// Stage candidates [j0, j0 + cnt) into `buf`: the bulk copy covers the 16 B aligned interior of the byte range, threads
// 0-3 the head floats before it and threads 4-7 the tail floats after it.  Returns the buffer's float offset of j0.
__device__ __forceinline__ int stage_tile(const Params& p, int j0, int cnt, unsigned char* buf, uint32_t bar) {
    const uintptr_t lo = (uintptr_t)(p.pts + (size_t)j0 * p.d);
    const uintptr_t hi = lo + (size_t)cnt * p.d * 4;
    const uintptr_t a = lo & ~(uintptr_t)15, b16 = (lo + 15) & ~(uintptr_t)15, e16 = hi & ~(uintptr_t)15;
    const uintptr_t mid_end = e16 > b16 ? e16 : b16;
    if (threadIdx.x == 0) {
        const uint32_t bytes = e16 > b16 ? (uint32_t)(e16 - b16) : 0u;
        tma::fence_proxy_async();                       // earlier generic-proxy use of this buffer before the async write
        tma::mbar_expect_tx(bar, bytes);
        if (bytes) tma::bulk_load(tma::smem_u32(buf + (b16 - a)), (const void*)b16, bytes, bar);
    }
    const int t = threadIdx.x;
    if (t < 4) {
        const uintptr_t addr = lo + 4 * t;
        if (addr < b16 && addr < hi) *reinterpret_cast<float*>(buf + (addr - a)) = __ldg(reinterpret_cast<const float*>(addr));
    } else if (t < 8) {
        const uintptr_t addr = mid_end + 4 * (t - 4);
        if (addr >= lo && addr < hi) *reinterpret_cast<float*>(buf + (addr - a)) = __ldg(reinterpret_cast<const float*>(addr));
    }
    return (int)((lo - a) >> 2);
}

// The body of the search kernels.  PAIR == HYPERBOLIC: p.pts holds records of d = 8 floats (4 doubles, 8 B aligned),
// MODE is COUNT or FILL, DREG == 0.
template <int MODE, int KB, int DREG, int QT, int PAIR>
__device__ __forceinline__ void pair_search(const Params& p) {
    extern __shared__ __align__(128) unsigned char smem[];
    if (*(volatile const int*)p.bad) return;
    const int64_t item = blockIdx.x;
    if (item >= p.tile_ptr[p.n_seg]) return;
    int lo = 0, hi = p.n_seg;                                     // the segment s with tile_ptr[s] <= item < tile_ptr[s+1]
    while (hi - lo > 1) {
        const int mid = (lo + hi) >> 1;
        if (p.tile_ptr[mid] <= item) lo = mid; else hi = mid;
    }
    const int s0 = (int)p.seg[lo], s1 = (int)p.seg[lo + 1];
    const int q0 = s0 + (int)(item - p.tile_ptr[lo]) * QT;
    const int i = q0 + (int)threadIdx.x;
    const bool active = i < s1;
    const int d = DREG == 3 ? 3 : p.d;                            // DREG == 3: exactly three coordinates

    unsigned char* buf0 = smem;
    unsigned char* buf1 = smem + BUF_BYTES;
    const uint32_t bar0 = tma::smem_u32(smem + 2 * BUF_BYTES);
    float* qs = reinterpret_cast<float*>(smem + 2 * BUF_BYTES + 16);   // DREG == 0: the query tile, row stride d | 1
    const int qstride = d | 1;

    float q[DREG > 0 ? DREG : 1];
    double hq[4];
    if constexpr (PAIR == HYPERBOLIC) {
#pragma unroll
        for (int f = 0; f < 4; ++f) hq[f] = active ? __ldg(reinterpret_cast<const double*>(p.pts) + (size_t)i * 4 + f) : 0.0;
    } else if (DREG > 0) {
#pragma unroll
        for (int f = 0; f < (DREG > 0 ? DREG : 1); ++f) q[f] = (active && f < d) ? __ldg(p.pts + (size_t)i * d + f) : 0.f;
    } else {
        const int nq = min(QT, s1 - q0);
        for (int e = threadIdx.x; e < nq * d; e += QT) {
            const int row = e / d, f = e - row * d;
            qs[row * qstride + f] = __ldg(p.pts + (size_t)q0 * d + e);
        }
    }

    // running top-k: td = bits(d2) + 1 (NaN as +Inf), tj = j, ascending in (td, tj).  Slots below KB - k hold the low
    // sentinel 0 and never move; the others start at the high sentinel ~0u.
    uint32_t td[MODE == KNN ? KB : 1];
    int32_t tj[MODE == KNN ? KB : 1];
    if (MODE == KNN) {
#pragma unroll
        for (int m = 0; m < KB; ++m) {
            td[m] = (m < KB - p.k) ? 0u : ~0u;
            tj[m] = 0;
        }
    }
    int64_t cnt_out = 0;
    // FILL: row i owns nbr[row_begin, row_end); writes never leave it nor [0, capacity), whatever offsets holds
    int64_t wpos = 0, row_lim = 0;
    if (MODE == FILL && active) {
        wpos = p.offsets[i];
        row_lim = wpos < 0 ? wpos : min(p.offsets[i + 1], p.capacity);
    }

    if (threadIdx.x == 0) {
        tma::mbar_init(bar0, 1);
        tma::mbar_init(bar0 + 8, 1);
        fence_mbar_init();
    }
    __syncthreads();

    const int ct = p.ct;
    const int T = (s1 - s0 + ct - 1) / ct;
    int off0 = stage_tile(p, s0, min(ct, s1 - s0), buf0, bar0);
    int off1 = T > 1 ? stage_tile(p, s0 + ct, min(ct, s1 - s0 - ct), buf1, bar0 + 8) : 0;

    for (int t = 0; t < T; ++t) {
        const int b = t & 1;
        const bool ok = tma::mbar_wait_bounded(bar0 + 8 * b, (uint32_t)((t >> 1) & 1), p.err);
        if (__syncthreads_or(!ok)) return;              // also publishes the thread-loaded head / tail floats
        const int j0 = s0 + t * ct, cnt = min(ct, s1 - j0);
        const float* cand = reinterpret_cast<const float*>(b ? buf1 : buf0) + (b ? off1 : off0);
        if (active) {
            for (int jl = 0; jl < cnt; ++jl) {
                const int j = j0 + jl;
                if (!p.self_loops && j == i) continue;
                const float* c = cand + jl * d;
                if constexpr (PAIR == HYPERBOLIC) {
                    if (hyperbolic_hit(hq, reinterpret_cast<const double*>(c), p.xmax)) {
                        if (MODE == FILL) {
                            if (wpos < row_lim) p.nbr[wpos] = j;
                            ++wpos;
                        } else {
                            ++cnt_out;
                        }
                    }
                    continue;
                }
                float acc = 0.f;
                if (DREG > 0) {
#pragma unroll
                    for (int f = 0; f < (DREG > 0 ? DREG : 1); ++f) {
                        if (f >= d) break;
                        acc = __fadd_rn(acc, sq_term(q[f], c[f]));
                    }
                } else {
                    const float* qr = qs + (i - q0) * qstride;
                    for (int f = 0; f < d; ++f) acc = __fadd_rn(acc, sq_term(qr[f], c[f]));
                }
                if (MODE == KNN) {
                    // j exceeds every j already held, so the key (d2, j) goes right after the entries with td <= u:
                    // comparing td alone orders the full keys
                    const uint32_t u = dist_key(acc);
                    if (u < td[KB - 1]) {
#pragma unroll
                        for (int m = KB - 1; m > 0; --m) {
                            const bool shift = td[m - 1] > u, here = td[m] > u;
                            tj[m] = shift ? tj[m - 1] : (here ? j : tj[m]);
                            td[m] = shift ? td[m - 1] : (here ? u : td[m]);
                        }
                        if (td[0] > u) {
                            td[0] = u;
                            tj[0] = j;
                        }
                    }
                } else {
                    const float dist = (acc != acc) ? __int_as_float(0x7f800000) : __fsqrt_rn(acc);
                    if (dist <= p.r) {
                        if (MODE == FILL) {
                            if (wpos < row_lim) p.nbr[wpos] = j;
                            ++wpos;
                        } else {
                            ++cnt_out;
                        }
                    }
                }
            }
        }
        __syncthreads();                                  // every thread is done with buffer b
        if (t + 2 < T) {
            const int o = stage_tile(p, s0 + (t + 2) * ct, min(ct, s1 - s0 - (t + 2) * ct), b ? buf1 : buf0, bar0 + 8 * b);
            if (b) off1 = o; else off0 = o;
        }
    }
    if (!active) return;
    if (MODE == KNN) {
        int32_t* row = p.nbr + (size_t)i * p.k;
#pragma unroll
        for (int m = 0; m < KB; ++m)
            if (m >= KB - p.k) row[m - (KB - p.k)] = tj[m];
    } else if (MODE == COUNT) {
        p.counts[i] = cnt_out;
    } else if (wpos != p.offsets[i + 1]) {
        atomicOr(p.mismatch, 1);                          // offsets do not come from the same count
    }
}

template <int MODE, int KB, int DREG, int QT>
__global__ void __launch_bounds__(QT) knn_kernel(const Params p) { pair_search<MODE, KB, DREG, QT, EUCLID>(p); }

// A kernel of its own so that its launch bounds leave knn_kernel's register allocation alone: with __launch_bounds__(128)
// alone ptxas fits the fill into 40 registers and spills 16 B; with a minimum of 4 CTAs it takes 78 and spills nothing.
template <int MODE>
__global__ void __launch_bounds__(128, 4) hyperbolic_kernel(const Params p) {
    pair_search<MODE, 1, 0, 128, HYPERBOLIC>(p);
}

// tiles[s] = query tiles of segment s; flags bad |= 1 for a malformed seg_ptr, |= 2 for a non-empty segment with fewer
// than `need` points
__global__ void tiles_kernel(const int64_t* __restrict__ seg, int64_t n_seg, int64_t n, int need, int qt,
                             int64_t* __restrict__ tiles, int* __restrict__ bad) {
    const int64_t s = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (s >= n_seg) return;
    const int64_t a = seg[s], b = seg[s + 1];
    int flag = 0;
    if ((s == 0 && a != 0) || (s == n_seg - 1 && b != n) || b < a || a < 0 || b > n) flag |= 1;
    else if (b > a && b - a < need) flag |= 2;
    if (flag) atomicOr(bad, flag);
    tiles[s] = flag ? 0 : (b - a + qt - 1) / qt;
}

template <int MODE, int KB, int DREG, int QT, int PAIR = EUCLID>
static int launch(const Params& p, int64_t grid, cudaStream_t st) {
    const size_t smem = 2 * BUF_BYTES + 16 + (DREG == 0 && PAIR == EUCLID ? (size_t)QT * (p.d | 1) * 4 : 0);
    void (*kern)(const Params);
    if constexpr (PAIR == HYPERBOLIC) kern = hyperbolic_kernel<MODE>;
    else kern = knn_kernel<MODE, KB, DREG, QT>;
    GNNB_CUDA(cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
    kern<<<(unsigned)grid, QT, smem, st>>>(p);
    GNNB_LAUNCHED();
    return GNNB_OK;
}

template <int MODE, int KB>
static int dispatch_d(const Params& p, int64_t n, int64_t n_seg, cudaStream_t st) {
    if (p.d == 3) return launch<MODE, KB, 3, 128>(p, ceil_div(n, 128) + n_seg, st);
    if (p.d <= 4) return launch<MODE, KB, 4, 128>(p, ceil_div(n, 128) + n_seg, st);
    if (p.d <= 16) return launch<MODE, KB, 16, 128>(p, ceil_div(n, 128) + n_seg, st);
    if (p.d <= 64) return launch<MODE, KB, 64, 128>(p, ceil_div(n, 128) + n_seg, st);
    return launch<MODE, KB, 0, 64>(p, ceil_div(n, 64) + n_seg, st);
}

static int query_tile(int d) { return d <= 64 ? 128 : 64; }

// One call: validate + tile the segments, run the MODE kernel, report flags.  Synchronises the stream.  pair ==
// HYPERBOLIC: points are the records (d = 8 floats each) and xmax replaces r.
static int run(int mode, const float* points, int64_t n, int d, const int64_t* seg_ptr, int64_t n_seg, int k,
               int self_loops, float r, int32_t* nbr, int64_t* counts, const int64_t* offsets, int64_t capacity,
               cudaStream_t st, int pair = EUCLID, double xmax = 0.0) {
    DeviceScratch sc(st);
    int64_t* dseg = nullptr;
    int64_t* tiles = nullptr;   // [n_seg + 1 (+ 2 for the default segment)]: counts, then the scan into tile_ptr
    int* flags = nullptr;       // [0] bad, [1] pipeline stall, [2] fill / count mismatch
    void* tmp = nullptr;
    const int qt = query_tile(d);
    GNNB_TRY(sc.alloc(&tiles, (size_t)(2 * n_seg + 3)));
    GNNB_TRY(sc.alloc(&flags, 3));
    GNNB_CUDA(cudaMemsetAsync(flags, 0, 3 * sizeof(int), st));
    if (!seg_ptr) {
        dseg = tiles + 2 * n_seg + 1;
        const int64_t h[2] = {0, n};
        GNNB_CUDA(cudaMemcpyAsync(dseg, h, sizeof h, cudaMemcpyHostToDevice, st));
        seg_ptr = dseg;
    }
    int64_t* cnt = tiles;
    int64_t* tile_ptr = tiles + n_seg;
    GNNB_CUDA(cudaMemsetAsync(tile_ptr, 0, sizeof(int64_t), st));
    const int need = mode == KNN ? k + (self_loops ? 0 : 1) : 0;
    tiles_kernel<<<(unsigned)ceil_div(n_seg, 256), 256, 0, st>>>(seg_ptr, n_seg, n, need, qt, cnt, flags);
    GNNB_LAUNCHED();
    size_t tmp_bytes = 0;
    GNNB_CUDA(cub::DeviceScan::InclusiveSum(nullptr, tmp_bytes, cnt, tile_ptr + 1, (int)n_seg, st));
    GNNB_TRY(sc.alloc(&tmp, tmp_bytes ? tmp_bytes : 1));
    GNNB_CUDA(cub::DeviceScan::InclusiveSum(tmp, tmp_bytes, cnt, tile_ptr + 1, (int)n_seg, st));
    g_launches.fetch_add(1, std::memory_order_relaxed);
    Params p{};
    p.pts = points; p.seg = seg_ptr; p.tile_ptr = tile_ptr; p.n_seg = (int)n_seg; p.d = d; p.k = k;
    p.self_loops = self_loops ? 1 : 0; p.ct = BUF_FLOATS / d > 0 ? BUF_FLOATS / d : 1; p.r = r;
    p.nbr = nbr; p.counts = counts; p.offsets = offsets; p.capacity = capacity;
    p.err = flags + 1; p.mismatch = flags + 2; p.bad = flags; p.xmax = xmax;
    if (pair == HYPERBOLIC) {
        if (mode == COUNT) GNNB_TRY((launch<COUNT, 1, 0, 128, HYPERBOLIC>(p, ceil_div(n, 128) + n_seg, st)));
        else GNNB_TRY((launch<FILL, 1, 0, 128, HYPERBOLIC>(p, ceil_div(n, 128) + n_seg, st)));
    } else if (mode == KNN) {
        if (k <= 8) GNNB_TRY((dispatch_d<KNN, 8>(p, n, n_seg, st)));
        else if (k <= 16) GNNB_TRY((dispatch_d<KNN, 16>(p, n, n_seg, st)));
        else if (k <= 32) GNNB_TRY((dispatch_d<KNN, 32>(p, n, n_seg, st)));
        else GNNB_TRY((dispatch_d<KNN, 64>(p, n, n_seg, st)));
    } else if (mode == COUNT) {
        GNNB_TRY((dispatch_d<COUNT, 1>(p, n, n_seg, st)));
    } else {
        GNNB_TRY((dispatch_d<FILL, 1>(p, n, n_seg, st)));
    }
    int h[3] = {0, 0, 0};
    GNNB_CUDA(cudaMemcpyAsync(h, flags, sizeof h, cudaMemcpyDeviceToHost, st));
    GNNB_CUDA(cudaStreamSynchronize(st));
    if (h[0] & 1)
        GNNB_FAIL(GNNB_EINVAL, "seg_ptr must hold n_seg + 1 non-decreasing offsets from 0 to n = %lld", (long long)n);
    if (h[0] & 2)
        GNNB_FAIL(GNNB_ESIZE, "a segment has fewer than k%s = %d points", self_loops ? "" : " + 1", need);
    if (h[1]) GNNB_FAIL(GNNB_ECUDA, "knn: the candidate pipeline stalled (mbarrier wait timed out)");
    if (h[2] && pair == HYPERBOLIC)
        GNNB_FAIL(GNNB_EINVAL, "gnnb_hyperbolic_fill: offsets do not match the rows of these records, x_max, self_loop "
                               "and segments (nothing was written outside a row's own range)");
    if (h[2])
        GNNB_FAIL(GNNB_EINVAL, "gnnb_radius_fill: offsets do not match the rows of these points, r, self_loops and "
                               "segments (nothing was written outside a row's own range)");
    return GNNB_OK;
}

static int check_common(const char* who, const float* points, int64_t n, int d, const int64_t* seg_ptr, int64_t n_seg) {
    if (n < 0 || n >= ((int64_t)1 << 31)) GNNB_FAIL(GNNB_ESIZE, "%s: n = %lld outside [0, 2^31)", who, (long long)n);
    if (d < 1) GNNB_FAIL(GNNB_EINVAL, "%s: d = %d must be >= 1", who, d);
    if (d > MAX_D) GNNB_FAIL(GNNB_EUNSUPPORTED, "%s: d = %d > %d is not supported", who, d, MAX_D);
    if (seg_ptr && (n_seg < 1 || n_seg >= ((int64_t)1 << 31)))
        GNNB_FAIL(GNNB_EINVAL, "%s: n_seg = %lld must be in [1, 2^31)", who, (long long)n_seg);
    if (n > 0 && !points) GNNB_FAIL(GNNB_EINVAL, "%s: points is NULL", who);
    return GNNB_OK;
}

static int check_radius(float r) {
    if (r != r || r < 0.f) GNNB_FAIL(GNNB_EINVAL, "radius r = %g must be >= 0 and not NaN", (double)r);
    return GNNB_OK;
}

static int check_hyperbolic(const char* who, const double* records, int64_t n, const int64_t* seg_ptr, int64_t n_seg,
                            double x_max) {
    GNNB_TRY(check_common(who, reinterpret_cast<const float*>(records), n, 8, seg_ptr, n_seg));
    if (x_max != x_max) GNNB_FAIL(GNNB_EINVAL, "%s: x_max is NaN", who);
    if ((uintptr_t)records % 8) GNNB_FAIL(GNNB_EINVAL, "%s: records must be 8 B aligned", who);
    return GNNB_OK;
}

// The count entries: offsets = running row counts, *total_host = offsets[n].  Synchronises the stream.
static int count_rows(const char* who, const float* points, int64_t n, int d, const int64_t* seg_ptr, int64_t n_seg,
                      float r, int self_loops, int64_t* offsets, int64_t* total_host, cudaStream_t st, int pair,
                      double xmax) {
    if (!offsets || !total_host) GNNB_FAIL(GNNB_EINVAL, "%s: offsets / total is NULL", who);
    *total_host = 0;
    GNNB_CUDA(cudaMemsetAsync(offsets, 0, sizeof(int64_t), st));
    if (n == 0) {
        GNNB_CUDA(cudaStreamSynchronize(st));
        return GNNB_OK;
    }
    DeviceScratch sc(st);
    int64_t* counts = nullptr;
    void* tmp = nullptr;
    GNNB_TRY(sc.alloc(&counts, (size_t)n));
    GNNB_TRY(run(COUNT, points, n, d, seg_ptr, seg_ptr ? n_seg : 1, 0, self_loops, r, nullptr, counts, nullptr, 0, st,
                 pair, xmax));
    size_t tmp_bytes = 0;
    GNNB_CUDA(cub::DeviceScan::InclusiveSum(nullptr, tmp_bytes, counts, offsets + 1, (int)n, st));
    GNNB_TRY(sc.alloc(&tmp, tmp_bytes ? tmp_bytes : 1));
    GNNB_CUDA(cub::DeviceScan::InclusiveSum(tmp, tmp_bytes, counts, offsets + 1, (int)n, st));
    g_launches.fetch_add(1, std::memory_order_relaxed);
    GNNB_CUDA(cudaMemcpyAsync(total_host, offsets + n, sizeof(int64_t), cudaMemcpyDeviceToHost, st));
    GNNB_CUDA(cudaStreamSynchronize(st));
    return GNNB_OK;
}

// The fill entries: row i at nbr[offsets[i] .. offsets[i+1]).  Synchronises the stream.
static int fill_rows(const char* who, const float* points, int64_t n, int d, const int64_t* seg_ptr, int64_t n_seg,
                     float r, int self_loops, const int64_t* offsets, int32_t* nbr, int64_t capacity, cudaStream_t st,
                     int pair, double xmax) {
    if (!offsets) GNNB_FAIL(GNNB_EINVAL, "%s: offsets is NULL", who);
    if (n == 0) return GNNB_OK;
    int64_t total = 0;
    GNNB_CUDA(cudaMemcpyAsync(&total, offsets + n, sizeof(int64_t), cudaMemcpyDeviceToHost, st));
    GNNB_CUDA(cudaStreamSynchronize(st));
    if (capacity < total)
        GNNB_FAIL(GNNB_ESIZE, "nbr holds %lld entries, %lld needed", (long long)capacity, (long long)total);
    if (total == 0) return GNNB_OK;
    if (!nbr) GNNB_FAIL(GNNB_EINVAL, "%s: nbr is NULL", who);
    return run(FILL, points, n, d, seg_ptr, seg_ptr ? n_seg : 1, 0, self_loops, r, nbr, nullptr, offsets, capacity, st,
               pair, xmax);
}

}  // namespace knn
}  // namespace gnnb

using namespace gnnb;

extern "C" {

int gnnb_knn(const float* points, int64_t n, int d, const int64_t* seg_ptr, int64_t n_seg, int k, int self_loops,
             int32_t* nbr, void* stream) {
    GNNB_TRY(knn::check_common("gnnb_knn", points, n, d, seg_ptr, n_seg));
    if (k < 1) GNNB_FAIL(GNNB_EINVAL, "gnnb_knn: k = %d must be >= 1", k);
    if (k > knn::MAX_K) GNNB_FAIL(GNNB_EUNSUPPORTED, "gnnb_knn: k = %d > %d is not supported", k, knn::MAX_K);
    if (n == 0) return GNNB_OK;
    if (!nbr) GNNB_FAIL(GNNB_EINVAL, "gnnb_knn: nbr is NULL");
    return knn::run(knn::KNN, points, n, d, seg_ptr, seg_ptr ? n_seg : 1, k, self_loops, 0.f, nbr, nullptr, nullptr, 0,
                    (cudaStream_t)stream);
}

int gnnb_radius_count(const float* points, int64_t n, int d, const int64_t* seg_ptr, int64_t n_seg, float r,
                      int self_loops, int64_t* offsets, int64_t* total_host, void* stream) {
    GNNB_TRY(knn::check_common("gnnb_radius_count", points, n, d, seg_ptr, n_seg));
    GNNB_TRY(knn::check_radius(r));
    return knn::count_rows("gnnb_radius_count", points, n, d, seg_ptr, n_seg, r, self_loops, offsets, total_host,
                           (cudaStream_t)stream, knn::EUCLID, 0.0);
}

int gnnb_radius_fill(const float* points, int64_t n, int d, const int64_t* seg_ptr, int64_t n_seg, float r,
                     int self_loops, const int64_t* offsets, int32_t* nbr, int64_t capacity, void* stream) {
    GNNB_TRY(knn::check_common("gnnb_radius_fill", points, n, d, seg_ptr, n_seg));
    GNNB_TRY(knn::check_radius(r));
    return knn::fill_rows("gnnb_radius_fill", points, n, d, seg_ptr, n_seg, r, self_loops, offsets, nbr, capacity,
                          (cudaStream_t)stream, knn::EUCLID, 0.0);
}

int gnnb_hyperbolic_count(const double* records, int64_t n, const int64_t* seg_ptr, int64_t n_seg, double x_max,
                          int self_loop, int64_t* offsets, int64_t* total_host, void* stream) {
    GNNB_TRY(knn::check_hyperbolic("gnnb_hyperbolic_count", records, n, seg_ptr, n_seg, x_max));
    return knn::count_rows("gnnb_hyperbolic_count", reinterpret_cast<const float*>(records), n, 8, seg_ptr, n_seg, 0.f,
                           self_loop, offsets, total_host, (cudaStream_t)stream, knn::HYPERBOLIC, x_max);
}

int gnnb_hyperbolic_fill(const double* records, int64_t n, const int64_t* seg_ptr, int64_t n_seg, double x_max,
                         int self_loop, const int64_t* offsets, int32_t* nbr, int64_t capacity, void* stream) {
    GNNB_TRY(knn::check_hyperbolic("gnnb_hyperbolic_fill", records, n, seg_ptr, n_seg, x_max));
    return knn::fill_rows("gnnb_hyperbolic_fill", reinterpret_cast<const float*>(records), n, 8, seg_ptr, n_seg, 0.f,
                          self_loop, offsets, nbr, capacity, (cudaStream_t)stream, knn::HYPERBOLIC, x_max);
}

}  // extern "C"
