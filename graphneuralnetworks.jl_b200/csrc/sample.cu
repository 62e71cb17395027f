// sample.cu — neighbour sampling over the CSR plan (SURVEY.md §8f rank 4): the step before the hot path for graphs
// that are trained in mini-batches.
//
// Reference counterpart: the edge selection of sample_neighbors(g, nodes, K; dir, replace)
// (GNNGraphs/src/sampling.jl:68-83): `adjacency_list(g, nodes; dir, with_eid=true)` — a Dict-driven scan of ALL edges
// on the CPU (GNNGraphs/src/query.jl:176-198) — followed by `StatsBase.sample(eidlist[i], k; replace)` per node.  Here
// the plan's CSR already is the adjacency list with edge ids (rowptr / eid), so a query touches only the rows asked for.
//
// Random numbers are counter based (splitmix64 keyed on seed, position in `nodes`, draw index): a call is reproducible
// and order independent.  The reference's draws come from Julia's task-local RNG, so parity here is distributional
// (every k-subset equally likely; with replacement: independent uniform draws), checked by the tests through
// size-independent properties.
#include "common.cuh"
#include <cub/cub.cuh>

namespace gnnb {

__host__ __device__ static inline uint64_t mulhi64(uint64_t a, uint64_t b) {
#ifdef __CUDA_ARCH__
    return __umul64hi(a, b);
#else
    return (uint64_t)(((unsigned __int128)a * b) >> 64);
#endif
}
// uniform integer in [0, m), m <= 2^31, from the (seed, j, draw) counter
__host__ __device__ static inline uint32_t rnd_below(uint64_t seed, uint64_t j, uint64_t draw, uint32_t m) {
    const uint64_t r = splitmix64(splitmix64(seed ^ (j * 0xD1342543DE82EF95ull)) + draw);
    return (uint32_t)mulhi64(r, (uint64_t)m);
}

__host__ __device__ static inline int32_t take_count(int32_t deg, int64_t K, int replace) {
    if (deg == 0) return 0;
    if (replace) return (int32_t)(K > 0 ? K : deg);
    return (int32_t)(K > 0 ? (K < deg ? K : deg) : deg);
}

// The sampler proper, for one query j over a row of `deg` edges: writes k positions in [0, deg) to out[0..k).
// With replacement: k independent uniform draws.  Without: everything (k == deg), Floyd's subset algorithm (k small
// against deg: O(k^2), the picks double as the membership list), or selection sampling (Knuth's algorithm S, O(deg),
// keeps adjacency order).  All three give every k-subset the same probability.  Host + device: the tests run this very
// code on the CPU through gnnb_sample_positions_host.
__host__ __device__ static inline void sample_positions(int32_t deg, int32_t k, int replace, uint64_t seed, uint64_t j,
                                                        int64_t* out) {
    if (replace) {
        for (int32_t i = 0; i < k; ++i) out[i] = (int64_t)rnd_below(seed, j, (uint64_t)i, (uint32_t)deg);
        return;
    }
    if (k == deg) {
        for (int32_t i = 0; i < k; ++i) out[i] = i;
        return;
    }
    if ((int64_t)k * k <= 4 * (int64_t)deg) {  // Floyd: for i = deg-k .. deg-1: t = U[0, i]; take t unless taken already, then i
        int32_t cnt = 0;
        for (int32_t i = deg - k; i < deg; ++i) {
            const int64_t t = (int64_t)rnd_below(seed, j, (uint64_t)i, (uint32_t)(i + 1));
            bool dup = false;
            for (int32_t q = 0; q < cnt; ++q) dup |= (out[q] == t);
            out[cnt++] = dup ? (int64_t)i : t;
        }
        return;
    }
    int32_t chosen = 0;  // algorithm S: take position pos with probability (k - chosen) / (deg - pos)
    for (int32_t pos = 0; pos < deg && chosen < k; ++pos) {
        const uint32_t u = rnd_below(seed, j, (uint64_t)pos, (uint32_t)(deg - pos));
        if (u < (uint32_t)(k - chosen)) out[chosen++] = pos;
    }
}

template <typename T>
__device__ __forceinline__ int64_t load_node(const void* nodes, int64_t j) {
    return (int64_t)reinterpret_cast<const T*>(nodes)[j];
}

// counts[j] = number of edges node j contributes (scanned into offsets by the caller)
__global__ void sample_count_kernel(const void* nodes, int64_t n, int index_bytes, int64_t index_base,
                                    const int32_t* __restrict__ rowptr, int32_t nrows, int64_t K, int replace,
                                    int64_t* __restrict__ counts, int* __restrict__ bad) {
    int64_t j = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (j >= n) return;
    int64_t r = (index_bytes == 8 ? load_node<int64_t>(nodes, j) : load_node<int32_t>(nodes, j)) - index_base;
    if (r < 0 || r >= nrows) {
        atomicExch(bad, 1);
        counts[j] = 0;
        return;
    }
    counts[j] = take_count(rowptr[r + 1] - rowptr[r], K, replace);
}

// one thread per queried node: positions from sample_positions, then position -> COO edge id
__global__ void sample_fill_kernel(const void* nodes, int64_t n, int index_bytes, int64_t index_base,
                                   const int32_t* __restrict__ rowptr, const int32_t* __restrict__ eid,
                                   const int64_t* __restrict__ offsets, int replace, uint64_t seed,
                                   int64_t* __restrict__ eids_out) {
    int64_t j = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (j >= n) return;
    const int64_t r = (index_bytes == 8 ? load_node<int64_t>(nodes, j) : load_node<int32_t>(nodes, j)) - index_base;
    const int64_t base = offsets[j];
    const int32_t k = (int32_t)(offsets[j + 1] - base);
    if (k == 0) return;
    const int32_t start = rowptr[r], deg = rowptr[r + 1] - start;
    int64_t* out = eids_out + base;
    sample_positions(deg, k, replace, seed, (uint64_t)j, out);
    for (int32_t q = 0; q < k; ++q) out[q] = (int64_t)eid[start + (int32_t)out[q]] + index_base;
}

}  // namespace gnnb

using namespace gnnb;

extern "C" {

int gnnb_sample_positions_host(int32_t deg, int64_t K, int replace, uint64_t seed, uint64_t j, int64_t* out,
                               int64_t capacity, int64_t* k_out) {
    if (deg < 0 || !out || !k_out) GNNB_FAIL(GNNB_EINVAL, "gnnb_sample_positions_host: bad arguments");
    const int32_t k = take_count(deg, K, replace);
    *k_out = k;
    if (k > capacity) GNNB_FAIL(GNNB_ESIZE, "out holds %lld entries, %d needed", (long long)capacity, k);
    sample_positions(deg, k, replace, seed, j, out);
    return GNNB_OK;
}

int gnnb_sample_neighbors(gnnb_graph_t g, const void* nodes, int64_t n_nodes, int index_bytes, int index_base,
                          int64_t K, int dir, int replace, uint64_t seed, int64_t* offsets_dev, int64_t* eids_dev,
                          int64_t capacity, int64_t* total_host, void* stream) {
    if (!g) GNNB_FAIL(GNNB_EINVAL, "gnnb_sample_neighbors: NULL graph");
    if (index_bytes != 4 && index_bytes != 8) GNNB_FAIL(GNNB_EINVAL, "index_bytes must be 4 or 8 (got %d)", index_bytes);
    if (index_base != 0 && index_base != 1) GNNB_FAIL(GNNB_EINVAL, "index_base must be 0 or 1 (got %d)", index_base);
    if (dir != GNNB_DIR_IN && dir != GNNB_DIR_OUT) GNNB_FAIL(GNNB_EINVAL, "dir must be GNNB_DIR_IN or GNNB_DIR_OUT");
    if (n_nodes < 0 || n_nodes >= ((int64_t)1 << 31)) GNNB_FAIL(GNNB_ESIZE, "n_nodes %lld outside [0, 2^31)", (long long)n_nodes);
    if (!offsets_dev || !total_host) GNNB_FAIL(GNNB_EINVAL, "gnnb_sample_neighbors: offsets / total is NULL");
    if (replace && K > 0 && K >= ((int64_t)1 << 31)) GNNB_FAIL(GNNB_ESIZE, "K too large");
    cudaStream_t st = (cudaStream_t)stream;
    *total_host = 0;
    const bool transposed = (dir == GNNB_DIR_OUT);
    GNNB_TRY(ensure_csr(g, transposed, st));
    const Csr& c = transposed ? g->by_src : g->by_dst;
    GNNB_CUDA(cudaMemsetAsync(offsets_dev, 0, sizeof(int64_t), st));
    if (n_nodes == 0) {
        GNNB_CUDA(cudaStreamSynchronize(st));
        return GNNB_OK;
    }
    if (!nodes) GNNB_FAIL(GNNB_EINVAL, "gnnb_sample_neighbors: nodes is NULL");
    DeviceScratch sc(st);
    int* bad = nullptr;
    int64_t* counts = nullptr;
    void* tmp = nullptr;
    const unsigned blocks = (unsigned)ceil_div(n_nodes, 128);
    GNNB_TRY(sc.alloc(&bad, 1));
    GNNB_TRY(sc.alloc(&counts, (size_t)n_nodes));
    GNNB_CUDA(cudaMemsetAsync(bad, 0, sizeof(int), st));
    sample_count_kernel<<<blocks, 128, 0, st>>>(nodes, n_nodes, index_bytes, index_base, c.rowptr, c.nrows, K, replace,
                                                counts, bad);
    GNNB_LAUNCHED();
    size_t tmp_bytes = 0;
    GNNB_CUDA(cub::DeviceScan::InclusiveSum(nullptr, tmp_bytes, counts, offsets_dev + 1, (int)n_nodes, st));
    GNNB_TRY(sc.alloc(&tmp, tmp_bytes ? tmp_bytes : 1));
    GNNB_CUDA(cub::DeviceScan::InclusiveSum(tmp, tmp_bytes, counts, offsets_dev + 1, (int)n_nodes, st));
    g_launches.fetch_add(1, std::memory_order_relaxed);
    int hbad = 0;
    int64_t total = 0;
    GNNB_CUDA(cudaMemcpyAsync(&hbad, bad, sizeof(int), cudaMemcpyDeviceToHost, st));
    GNNB_CUDA(cudaMemcpyAsync(&total, offsets_dev + n_nodes, sizeof(int64_t), cudaMemcpyDeviceToHost, st));
    GNNB_CUDA(cudaStreamSynchronize(st));
    if (hbad) GNNB_FAIL(GNNB_EINDEX, "node id outside [%d, %d]", index_base, index_base + c.nrows - 1);
    *total_host = total;
    if (!eids_dev || total == 0) return GNNB_OK;
    if (capacity < total) GNNB_FAIL(GNNB_ESIZE, "eids buffer holds %lld entries, %lld needed", (long long)capacity, (long long)total);
    sample_fill_kernel<<<blocks, 128, 0, st>>>(nodes, n_nodes, index_bytes, index_base, c.rowptr, c.eid, offsets_dev,
                                               replace, seed, eids_dev);
    GNNB_LAUNCHED();
    return GNNB_OK;
}

}  // extern "C"
