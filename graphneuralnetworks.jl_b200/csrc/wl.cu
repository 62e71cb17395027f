// wl.cu — color_refinement (1-WL colour refinement) on the device: one pass per round over the plan's in-edges, the
// classes renumbered by a stable radix sort of the exact signature key.
//
// Reference counterpart: color_refinement(g, x0) (GNNGraphs/src/utils.jl:340-389), a host loop that hashes
// (x_i, sort(x[in-neighbours of i])) into a Dict once per node per round.
//
// Contract (tests/test_color_refinement.py restates it in numpy with exact tuples):
//   round r maps node i to its signature (c_i, multiset{c_s : edges s -> i}); two nodes share a new colour iff their
//   signatures are equal; colours are numbered 0 .. k-1 in order of first appearance by node id (1-based on output);
//   the rounds stop when a round leaves the number of classes unchanged, or after max_iters rounds.
//
// Signature pass (wl_signature_kernel), over the work items {e_begin, e_end, slot} of the CSR by target (seglean.cu's
// ensure_items): one warp per item, one edge per lane, col[e] and row[e] read coalesced, the 4-byte colour c[col[e]]
// gathered.  Each edge contributes phi_k(c) = splitmix64(c ^ salt_k) mod p, p = 2^61 - 1, k = 1, 2, and a row's
// signature is S_k(i) = Σ phi_k mod p, folded after every add (a sum of raw 61-bit values would overflow 64 bits).  The
// per-row sums are a segmented warp scan on the sorted row ids plus a carry into the next 32 edges.  A piece of a long
// row stores its sum into workspace slot `slot` (2 slots per chunk, as segwalk.cuh numbers them) and wl_fixup_kernel
// adds the pieces.  Addition mod p is associative and commutative, so every chunk size gives the same bits, with no
// atomics.  Rows without in-edges keep S = (0, 0).
//   Two different multisets collide when the multiplicity differences of their colours, weighted by phi, sum to 0 mod p.
//   The differences are below 2^31 < p, so they are never 0 mod p; under a random-function model of phi two different
//   signatures with the same c_i match in both components with probability about p^-2 ~ 2^-122 per pair.  (Mod 2^64
//   a difference divisible by 2^j would cost j bits, and an RMAT hub holds one colour 10^5 times.)  This guards against
//   chance collisions, not against inputs built to collide.
//
// Relabel (the same code for round 0, which normalises x0, and for every round):
//   * a stable CUB radix sort of the exact key (c_i, S_1, S_2), packed into 122 + bits(k - 1) bits, node ids as values
//     (round 0 sorts x0 as a sign-flipped uint64, 64 bits);
//   * run heads on equal keys: the head of a run holds its smallest node id, because the sort is stable.  The head
//     nodes are flagged in node order, and an exclusive scan over n + 1 flags gives each head its rank and, at [n], the
//     class count — the one value read back per round;
//   * an inclusive max-scan of the head positions gives each sorted position its run's head; every node takes the rank
//     of its run's head.
// No atomics anywhere.  Scratch is one allocation per call, about 92 B per node; the long-row pieces use the plan's
// workspace (16 B per piece).
#include "common.cuh"
#include <cub/cub.cuh>
#include <cuda/std/tuple>
#include <algorithm>

namespace gnnb {
namespace wl {

constexpr uint64_t P61 = (1ull << 61) - 1;
constexpr uint64_t SALT1 = 0x5851F42D4C957F2Dull;
constexpr uint64_t SALT2 = 0x14057B7EF767814Full;

__device__ __forceinline__ uint64_t mod_p(uint64_t x) {          // x mod 2^61 - 1
    x = (x & P61) + (x >> 61);
    return x >= P61 ? x - P61 : x;
}
__device__ __forceinline__ uint64_t add_p(uint64_t a, uint64_t b) {   // a, b < p
    const uint64_t s = a + b;
    return s >= P61 ? s - P61 : s;
}

// the exact sort key: (c, S_1, S_2) as one 122 + bits(c) bit integer hi:mid:lo; round 0 puts the flipped x0 in lo
struct Key {
    uint64_t lo, mid;
    uint32_t hi, pad;
};
struct KeyBits {
    __host__ __device__ ::cuda::std::tuple<uint32_t&, uint64_t&, uint64_t&> operator()(Key& k) const {
        return {k.hi, k.mid, k.lo};
    }
};
struct MaxOp {
    __host__ __device__ int32_t operator()(int32_t a, int32_t b) const { return a > b ? a : b; }
};

struct SigParams {
    const int4* __restrict__ items;
    const int32_t* __restrict__ col;
    const int32_t* __restrict__ row;
    const int32_t* __restrict__ c;      // current colours, 0-based
    uint64_t* __restrict__ s1;
    uint64_t* __restrict__ s2;
    uint64_t* __restrict__ ws;          // [slot][2]: the sums of the long-row pieces
    int32_t n_items;
};

__global__ void __launch_bounds__(256) wl_signature_kernel(const SigParams p) {
    constexpr unsigned FULL = 0xffffffffu;
    const int lane = threadIdx.x & 31;
    const int item = blockIdx.x * 8 + (threadIdx.x >> 5);
    if (item >= p.n_items) return;
    const int4 it = __ldg(p.items + item);
    const bool partial = it.z >= 0;                 // one piece of a long row: a single row, summed into slot it.z
    uint64_t carry1 = 0, carry2 = 0;                // sum of the row that runs on from the previous 32 edges
    int carry_row = -1;
    for (int e0 = it.x; e0 < it.y; e0 += 32) {
        const int e = e0 + lane;
        const bool valid = e < it.y;
        int r = -1;
        uint64_t v1 = 0, v2 = 0;
        if (valid) {
            r = __ldg(p.row + e);
            const uint64_t cc = (uint32_t)__ldg(p.c + __ldg(p.col + e));
            v1 = mod_p(splitmix64(cc ^ SALT1));
            v2 = mod_p(splitmix64(cc ^ SALT2));
        }
        // segmented inclusive scan: rows are sorted, so lane - d in the same row means every lane between is too
#pragma unroll
        for (int d = 1; d < 32; d <<= 1) {
            const int ro = __shfl_up_sync(FULL, r, d);
            const uint64_t o1 = __shfl_up_sync(FULL, v1, d), o2 = __shfl_up_sync(FULL, v2, d);
            if (lane >= d && ro == r) { v1 = add_p(v1, o1); v2 = add_p(v2, o2); }
        }
        if (valid && r == carry_row) { v1 = add_p(v1, carry1); v2 = add_p(v2, carry2); }
        int rn = __shfl_down_sync(FULL, r, 1);
        if (lane == 31) rn = (!partial && e + 1 < it.y) ? __ldg(p.row + e + 1) : r;
        if (valid && (e + 1 == it.y || (!partial && rn != r))) {     // the last edge of its row in this item
            if (partial) { p.ws[2 * (int64_t)it.z] = v1; p.ws[2 * (int64_t)it.z + 1] = v2; }
            else { p.s1[r] = v1; p.s2[r] = v2; }
        }
        carry1 = __shfl_sync(FULL, v1, 31);         // a row that ended at lane 31 never matches the next rows
        carry2 = __shfl_sync(FULL, v2, 31);
        carry_row = __shfl_sync(FULL, r, 31);
    }
}

// long rows: slot 2 k0 + 1 holds the piece in the chunk where the row starts, slot 2 k for every later chunk k
__global__ void wl_fixup_kernel(const int32_t* __restrict__ long_rows, int32_t n_long, const int32_t* __restrict__ rowptr,
                                int chunk, const uint64_t* __restrict__ ws, uint64_t* __restrict__ s1,
                                uint64_t* __restrict__ s2) {
    const int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n_long) return;
    const int r = long_rows[i];
    const int k0 = rowptr[r] / chunk, k1 = (rowptr[r + 1] - 1) / chunk;
    uint64_t a1 = ws[2 * (2 * (int64_t)k0 + 1)], a2 = ws[2 * (2 * (int64_t)k0 + 1) + 1];
    for (int64_t k = k0 + 1; k <= k1; ++k) {
        a1 = add_p(a1, ws[4 * k]);
        a2 = add_p(a2, ws[4 * k + 1]);
    }
    s1[r] = a1;
    s2[r] = a2;
}

__global__ void wl_pack_kernel(const int32_t* __restrict__ c, const uint64_t* __restrict__ s1,
                               const uint64_t* __restrict__ s2, int64_t n, Key* __restrict__ keys) {
    const int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    const uint64_t ci = (uint32_t)c[i], a = s1[i], b = s2[i];
    keys[i] = Key{b | (a << 61), (a >> 3) | (ci << 58), (uint32_t)(ci >> 6), 0u};
}

__global__ void wl_pack_x0_kernel(const int64_t* __restrict__ x0, int64_t n, Key* __restrict__ keys,
                                  int32_t* __restrict__ iota) {
    const int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    keys[i] = Key{x0 ? (uint64_t)x0[i] ^ (1ull << 63) : 0ull, 0ull, 0u, 0u};
    iota[i] = (int32_t)i;
}

// sorted position k: flag its node if it heads a run of equal keys, and record the position of a head (0 otherwise)
__global__ void wl_heads_kernel(const Key* __restrict__ keys, const int32_t* __restrict__ v, int64_t n,
                                int32_t* __restrict__ flag, int32_t* __restrict__ hp) {
    const int64_t k = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (k >= n) return;
    bool h = k == 0;
    if (!h) {
        const Key a = keys[k], b = keys[k - 1];
        h = a.lo != b.lo || a.mid != b.mid || a.hi != b.hi;
    }
    flag[v[k]] = h ? 1 : 0;
    hp[k] = h ? (int32_t)k : 0;
}

// every node takes the rank (in node order) of its run's head
__global__ void wl_assign_kernel(const int32_t* __restrict__ v, const int32_t* __restrict__ headpos,
                                 const int32_t* __restrict__ rank, int64_t n, int32_t* __restrict__ c) {
    const int64_t k = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (k >= n) return;
    c[v[k]] = rank[v[headpos[k]]];
}

__global__ void wl_output_kernel(const int32_t* __restrict__ c, int64_t n, int64_t* __restrict__ out) {
    const int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i < n) out[i] = (int64_t)c[i] + 1;
}

static size_t align256(size_t b) { return (b + 255) & ~(size_t)255; }
static int bits_of(int64_t x) { int b = 0; while (x > 0) { ++b; x >>= 1; } return b; }

struct Arrays {   // the per-call arrays, carved from one allocation
    Key* keys[2];
    int32_t *iota, *v, *c, *flag, *rank, *hp, *headpos;
    uint64_t* s;           // [2][n]: S_1 then S_2
    void* tmp;
    size_t tmp_bytes;
};

// sort keys[0] (end_bit bits), renumber into sc.c by first appearance; *count = number of classes
static int relabel(const Arrays& sc, int64_t n, int end_bit, int64_t* count, cudaStream_t st) {
    const unsigned blocks = (unsigned)ceil_div(n, 256);
    size_t b = sc.tmp_bytes;
    GNNB_CUDA(cub::DeviceRadixSort::SortPairs(sc.tmp, b, sc.keys[0], sc.keys[1], sc.iota, sc.v, (int)n, KeyBits{}, 0,
                                              end_bit, st));
    g_launches.fetch_add(2, std::memory_order_relaxed);      // histogram + onesweep passes (library kernels)
    wl_heads_kernel<<<blocks, 256, 0, st>>>(sc.keys[1], sc.v, n, sc.flag, sc.hp);
    GNNB_LAUNCHED();
    b = sc.tmp_bytes;
    GNNB_CUDA(cub::DeviceScan::ExclusiveSum(sc.tmp, b, sc.flag, sc.rank, (int)(n + 1), st));
    b = sc.tmp_bytes;
    GNNB_CUDA(cub::DeviceScan::InclusiveScan(sc.tmp, b, sc.hp, sc.headpos, MaxOp{}, (int)n, st));
    g_launches.fetch_add(4, std::memory_order_relaxed);      // tile-state init + scan, twice (library kernels)
    wl_assign_kernel<<<blocks, 256, 0, st>>>(sc.v, sc.headpos, sc.rank, n, sc.c);
    GNNB_LAUNCHED();
    int32_t k = 0;
    GNNB_CUDA(cudaMemcpyAsync(&k, sc.rank + n, sizeof k, cudaMemcpyDeviceToHost, st));
    GNNB_CUDA(cudaStreamSynchronize(st));
    *count = k;
    return GNNB_OK;
}

static int run(gnnb_graph* g, const int64_t* x0, int64_t max_iters, int64_t* colors, int64_t* num_colors,
               int64_t* niters, cudaStream_t st) {
    const int64_t n = g->n_dst;
    const Csr& csr = g->by_dst;
    GNNB_TRY(ensure_items(g, csr, st));
    if (csr.n_long > 0)
        GNNB_TRY(grow_buffer(&g->ws, &g->ws_bytes, (size_t)2 * ceil_div(g->E, g->chunk) * 2 * sizeof(uint64_t)));
    uint64_t* ws = reinterpret_cast<uint64_t*>(g->ws);

    // CUB temporary storage: the sort at its widest bit range (fewer bits never need more), the two scans
    size_t sort_bytes = 0, sum_bytes = 0, max_bytes = 0;
    GNNB_CUDA(cub::DeviceRadixSort::SortPairs(nullptr, sort_bytes, (const Key*)nullptr, (Key*)nullptr,
                                              (const int32_t*)nullptr, (int32_t*)nullptr, (int)n, KeyBits{}, 0,
                                              122 + 32, st));
    GNNB_CUDA(cub::DeviceScan::ExclusiveSum(nullptr, sum_bytes, (int32_t*)nullptr, (int32_t*)nullptr, (int)(n + 1), st));
    GNNB_CUDA(cub::DeviceScan::InclusiveScan(nullptr, max_bytes, (int32_t*)nullptr, (int32_t*)nullptr, MaxOp{}, (int)n,
                                             st));
    const size_t tmp_bytes = std::max(sort_bytes, std::max(sum_bytes, max_bytes)) + 1;
    const size_t key_b = align256(sizeof(Key) * (size_t)n), s_b = align256(2 * sizeof(uint64_t) * (size_t)n);
    const size_t i_b = align256(sizeof(int32_t) * (size_t)(n + 1));
    DeviceScratch scratch(st);
    char* buf = nullptr;
    GNNB_TRY(scratch.alloc(&buf, 2 * key_b + s_b + 7 * i_b + tmp_bytes));
    Arrays sc;
    char* q = buf;
    sc.keys[0] = reinterpret_cast<Key*>(q); q += key_b;
    sc.keys[1] = reinterpret_cast<Key*>(q); q += key_b;
    sc.s = reinterpret_cast<uint64_t*>(q); q += s_b;
    int32_t** ints[7] = {&sc.iota, &sc.v, &sc.c, &sc.flag, &sc.rank, &sc.hp, &sc.headpos};
    for (int32_t** a : ints) { *a = reinterpret_cast<int32_t*>(q); q += i_b; }
    sc.tmp = q;
    sc.tmp_bytes = tmp_bytes;
    const unsigned blocks = (unsigned)ceil_div(n, 256);
    GNNB_CUDA(cudaMemsetAsync(sc.flag + n, 0, sizeof(int32_t), st));   // the scan's n + 1-th item
    // round 0: the iota values, and x0's partition (or one class)
    wl_pack_x0_kernel<<<blocks, 256, 0, st>>>(x0, n, sc.keys[0], sc.iota);
    GNNB_LAUNCHED();
    int64_t count = 1;
    if (x0) GNNB_TRY(relabel(sc, n, 64, &count, st));
    else GNNB_CUDA(cudaMemsetAsync(sc.c, 0, sizeof(int32_t) * (size_t)n, st));
    SigParams p;
    p.items = reinterpret_cast<const int4*>(csr.items);
    p.col = csr.col; p.row = csr.row; p.c = sc.c;
    p.s1 = sc.s; p.s2 = sc.s + n; p.ws = ws;
    p.n_items = csr.n_items;
    const bool zero_fill = g->E == 0 || csr.n_empty != 0;     // rows without in-edges keep S = (0, 0)
    int64_t round = 0;
    for (;;) {
        ++round;
        if (zero_fill) GNNB_CUDA(cudaMemsetAsync(sc.s, 0, 2 * sizeof(uint64_t) * (size_t)n, st));
        if (p.n_items > 0) {
            wl_signature_kernel<<<(unsigned)ceil_div(p.n_items, 8), 256, 0, st>>>(p);
            GNNB_LAUNCHED();
        }
        if (csr.n_long > 0) {
            wl_fixup_kernel<<<(unsigned)ceil_div(csr.n_long, 256), 256, 0, st>>>(
                csr.long_rows, csr.n_long, csr.rowptr, g->chunk, ws, p.s1, p.s2);
            GNNB_LAUNCHED();
        }
        wl_pack_kernel<<<blocks, 256, 0, st>>>(sc.c, p.s1, p.s2, n, sc.keys[0]);
        GNNB_LAUNCHED();
        int64_t next = 0;
        GNNB_TRY(relabel(sc, n, 122 + bits_of(count - 1), &next, st));
        const bool stable = next == count;
        count = next;
        if (stable || round == max_iters) break;
    }
    wl_output_kernel<<<blocks, 256, 0, st>>>(sc.c, n, colors);
    GNNB_LAUNCHED();
    GNNB_CUDA(cudaStreamSynchronize(st));
    *num_colors = count;
    *niters = round;
    return GNNB_OK;
}

}  // namespace wl
}  // namespace gnnb

using namespace gnnb;

extern "C" {

int gnnb_color_refinement(gnnb_graph_t g, const int64_t* x0, int64_t max_iters, int64_t* colors, int64_t* num_colors,
                          int64_t* niters, void* stream) {
    if (!g) GNNB_FAIL(GNNB_EINVAL, "graph handle is NULL");
    if (g->n_src != g->n_dst) GNNB_FAIL(GNNB_ESIZE, "gnnb_color_refinement needs num_src == num_dst");
    if (max_iters < 0)
        GNNB_FAIL(GNNB_EINVAL, "gnnb_color_refinement: max_iters = %lld must be >= 0 (0: until stable)",
                  (long long)max_iters);
    if (!num_colors || !niters) GNNB_FAIL(GNNB_EINVAL, "gnnb_color_refinement: num_colors / niters is NULL");
    if (g->n_dst == 0) {
        *num_colors = 0;
        *niters = 1;
        return GNNB_OK;
    }
    if (!colors) GNNB_FAIL(GNNB_EINVAL, "gnnb_color_refinement: colors is NULL");
    if (g->n_dst >= INT32_MAX) GNNB_FAIL(GNNB_ESIZE, "gnnb_color_refinement: n = %d must be < 2^31 - 1", g->n_dst);
    cudaStream_t st = (cudaStream_t)stream;
    GNNB_TRY(ensure_csr(g, false, st));
    return wl::run(g, x0, max_iters, colors, num_colors, niters, st);
}

}  // extern "C"
