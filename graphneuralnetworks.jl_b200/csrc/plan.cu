// plan.cu — the graph plan: COO (Julia 1-based Int64/Int32, host or device) -> int32 0-based device
// COO + CSR-by-target (+ lazily CSR-by-source), stable in COO order.
//
// Reference counterparts: the COO GNNGraph `(s,t)` (GNNGraphs/src/gnngraph.jl:108-117), index-range
// asserts of to_coo (GNNGraphs/src/convert.jl:49-54), add_self_loops (GNNGraphs/src/transform.jl:12-28).
// The reference has no CSR type and no GPU edge sort (GNNGraphs/ext/GNNGraphsCUDAExt.jl:24-30 sorts on
// the CPU); it rebuilds a CSC from COO on every fused CPU call (GNNGraphs/src/query.jl:227).
#include "common.cuh"
#include <cub/cub.cuh>
#include <thrust/iterator/counting_iterator.h>
#include <thrust/iterator/transform_iterator.h>

namespace gnnb {

static int g_chunk_default = 128;

// ---- kernels ------------------------------------------------------------------------------------
template <typename T>
__global__ void convert_index_kernel(const T* __restrict__ in, int64_t n, int64_t base, int64_t limit,
                                     int32_t* __restrict__ out, int* __restrict__ bad) {
    int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    int64_t v = (int64_t)in[i] - base;
    if (v < 0 || v >= limit) {
        *bad = 1;
        v = 0;
    }
    out[i] = (int32_t)v;
}

__global__ void iota_kernel(int32_t* out, int64_t n, int32_t start) {
    int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i < n) out[i] = start + (int32_t)i;
}

__global__ void gather_i32_kernel(const int32_t* __restrict__ src, const int32_t* __restrict__ idx,
                                  int64_t n, int32_t* __restrict__ out) {
    int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i < n) out[i] = src[idx[i]];
}

// rowptr from the sorted row array: rowptr[r] = first position whose row >= r
__global__ void rowptr_kernel(const int32_t* __restrict__ row, int64_t E, int32_t nrows,
                              int32_t* __restrict__ rowptr) {
    int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i > E) return;
    int32_t lo = (i == 0) ? -1 : row[i - 1];
    int32_t hi = (i == E) ? nrows : row[i];
    for (int32_t r = lo + 1; r <= hi; ++r) rowptr[r] = (int32_t)i;
}

__global__ void long_rows_kernel(const int32_t* __restrict__ rowptr, int32_t nrows, int32_t chunk,
                                 int32_t* __restrict__ list, int32_t* __restrict__ count) {
    int64_t r = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (r >= nrows) return;
    if (rowptr[r + 1] - rowptr[r] > chunk) list[atomicAdd(count, 1)] = (int32_t)r;
}

__global__ void invdeg_kernel(const int32_t* __restrict__ rowptr, int32_t nrows, float* __restrict__ out) {
    int64_t r = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (r >= nrows) return;
    int d = rowptr[r + 1] - rowptr[r];
    out[r] = 1.0f / (float)(d > 0 ? d : 1);
}

// CSR of add_self_loops(g) from the CSR of g: row r gains one trailing entry (the appended loop
// sorts last inside its row because the sort is stable and loops come after the originals).
__global__ void selfloop_edges_kernel(const int32_t* __restrict__ row, const int32_t* __restrict__ col,
                                      const int32_t* __restrict__ eid, int64_t E,
                                      int32_t* __restrict__ nrow, int32_t* __restrict__ ncol,
                                      int32_t* __restrict__ neid) {
    int64_t e = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (e >= E) return;
    int32_t r = row[e];
    int64_t pos = e + r;
    nrow[pos] = r;
    ncol[pos] = col[e];
    neid[pos] = eid[e];
}
__global__ void selfloop_rows_kernel(const int32_t* __restrict__ rowptr, int32_t n, int32_t E,
                                     int32_t* __restrict__ nrowptr, int32_t* __restrict__ nrow,
                                     int32_t* __restrict__ ncol, int32_t* __restrict__ neid) {
    int64_t r = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (r > n) return;
    nrowptr[r] = rowptr[r] + (int32_t)r;
    if (r < n) {
        int64_t pos = (int64_t)rowptr[r + 1] + r;  // last slot of the new row r
        nrow[pos] = (int32_t)r;
        ncol[pos] = (int32_t)r;
        neid[pos] = E + (int32_t)r;
    }
}

// ---- subgraph plans (remove_edges / remove_nodes / getgraph / add_nodes) ----------------------------
// A kept set of nodes renumbered in ascending old id is a monotone map, and the plan's sort is stable, so compacting
// the parent's sorted arrays (keeping their order) gives exactly the arrays a fresh stable sort of the child's COO
// gives.  Every position comes from an exclusive scan of 0/1 flags over n + 1 (or E + 1) items whose last flag is 0:
// entry [n] (or [E]) of the scan is the kept count, and item i is kept iff scan[i + 1] != scan[i].
struct NodeKeepFlag {        // node i is kept (keep == NULL keeps all)
    const uint8_t* keep;
    int64_t n;
    __host__ __device__ int32_t operator()(int64_t i) const { return (i < n && (!keep || keep[i])) ? 1 : 0; }
};
struct EdgeKeepFlag {        // COO edge e is kept: its mask (NULL keeps all) and both of its endpoints
    const uint8_t* ekeep;
    const uint8_t* nkeep;
    const int32_t* src;
    const int32_t* dst;
    int64_t E;
    __host__ __device__ int32_t operator()(int64_t e) const {
        if (e >= E || (ekeep && !ekeep[e])) return 0;
        return (!nkeep || (nkeep[src[e]] && nkeep[dst[e]])) ? 1 : 0;
    }
};
struct SortedKeepFlag {      // sorted position k of a parent CSR holds a kept edge
    const int32_t* eid;
    const int32_t* newid;    // exclusive scan of EdgeKeepFlag, E + 1 entries
    int64_t E;
    __host__ __device__ int32_t operator()(int64_t k) const {
        if (k >= E) return 0;
        const int32_t e = eid[k];
        return newid[e + 1] - newid[e];
    }
};
template <typename F>
using FlagIter = thrust::transform_iterator<F, thrust::counting_iterator<int64_t>, int32_t>;
template <typename F>
static FlagIter<F> flag_iter(F f) { return FlagIter<F>(thrust::counting_iterator<int64_t>(0), f); }

__global__ void node_map_kernel(const uint8_t* __restrict__ keep, const int32_t* __restrict__ scan, int64_t n,
                                int32_t* __restrict__ node_map) {
    int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i < n) node_map[i] = (!keep || keep[i]) ? scan[i] : -1;
}

__global__ void subgraph_coo_kernel(const int32_t* __restrict__ src, const int32_t* __restrict__ dst, int64_t E,
                                    const int32_t* __restrict__ newid, const int32_t* __restrict__ map,
                                    int32_t* __restrict__ nsrc, int32_t* __restrict__ ndst,
                                    int64_t* __restrict__ kept_eids) {
    int64_t e = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (e >= E) return;
    const int32_t p = newid[e];
    if (newid[e + 1] == p) return;
    nsrc[p] = map[src[e]];
    ndst[p] = map[dst[e]];
    if (kept_eids) kept_eids[p] = e;
}

__global__ void subgraph_csr_kernel(const int32_t* __restrict__ row, const int32_t* __restrict__ col,
                                    const int32_t* __restrict__ eid, int64_t E, const int32_t* __restrict__ pos,
                                    const int32_t* __restrict__ newid, const int32_t* __restrict__ map,
                                    int32_t* __restrict__ nrow, int32_t* __restrict__ ncol,
                                    int32_t* __restrict__ neid) {
    int64_t k = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (k >= E) return;
    const int32_t p = pos[k];
    if (pos[k + 1] == p) return;
    nrow[p] = map[row[k]];
    ncol[p] = map[col[k]];
    neid[p] = newid[eid[k]];
}

// keep[i] = !(u_i < p), u_i = (splitmix64(splitmix64(seed) + i) >> 11) * 2^-53
__global__ void bernoulli_keep_kernel(int64_t n, double p, uint64_t key, uint8_t* __restrict__ keep) {
    int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    const double u = (double)(splitmix64(key + (uint64_t)i) >> 11) * 0x1.0p-53;
    keep[i] = (u < p) ? 0 : 1;
}

// ---- helpers ------------------------------------------------------------------------------------
static void free_csr(Csr& c) {
    cudaFree(c.rowptr); cudaFree(c.col); cudaFree(c.row); cudaFree(c.eid);
    cudaFree(c.long_rows); cudaFree(c.invdeg); cudaFree(c.items); cudaFree(c.es);
    cudaFree(c.hot_rows);
    c = Csr();
}

static int alloc_csr(Csr& c, int64_t E, int32_t nrows, int32_t chunk) {
    c.nrows = nrows;
    GNNB_CUDA(cudaMalloc(&c.rowptr, sizeof(int32_t) * ((size_t)nrows + 1)));
    GNNB_CUDA(cudaMalloc(&c.col, sizeof(int32_t) * (size_t)(E > 0 ? E : 1)));
    GNNB_CUDA(cudaMalloc(&c.row, sizeof(int32_t) * (size_t)(E > 0 ? E : 1)));
    GNNB_CUDA(cudaMalloc(&c.eid, sizeof(int32_t) * (size_t)(E > 0 ? E : 1)));
    GNNB_CUDA(cudaMalloc(&c.long_rows, sizeof(int32_t) * (size_t)(E / chunk + 2)));
    return GNNB_OK;
}

static int find_long_rows(Csr& c, int32_t chunk, cudaStream_t st) {
    DeviceScratch sc;
    int32_t* d_count = nullptr;
    GNNB_TRY(sc.alloc(&d_count, 1));
    GNNB_CUDA(cudaMemsetAsync(d_count, 0, sizeof(int32_t), st));
    if (c.nrows > 0) {
        long_rows_kernel<<<(unsigned)ceil_div(c.nrows, 256), 256, 0, st>>>(c.rowptr, c.nrows, chunk,
                                                                           c.long_rows, d_count);
        GNNB_LAUNCHED();
    }
    GNNB_CUDA(cudaMemcpyAsync(&c.n_long, d_count, sizeof(int32_t), cudaMemcpyDeviceToHost, st));
    GNNB_CUDA(cudaStreamSynchronize(st));
    return GNNB_OK;
}

int ensure_csr(gnnb_graph* g, bool transposed, cudaStream_t st) {
    Csr& c = transposed ? g->by_src : g->by_dst;
    if (c.built) return GNNB_OK;
    std::lock_guard<std::mutex> lock(g->mu);
    if (c.built) return GNNB_OK;
    const int64_t E = g->E;
    const int32_t nrows = transposed ? g->n_src : g->n_dst;
    const int32_t* keys = transposed ? g->coo_src : g->coo_dst;
    const int32_t* other = transposed ? g->coo_dst : g->coo_src;
    GNNB_TRY(alloc_csr(c, E, nrows, g->chunk));
    if (E > 0) {
        DeviceScratch sc;
        int32_t* iota = nullptr;
        GNNB_TRY(sc.alloc(&iota, (size_t)E));
        iota_kernel<<<(unsigned)ceil_div(E, 256), 256, 0, st>>>(iota, E, 0);
        GNNB_LAUNCHED();
        int end_bit = 1;
        while (end_bit < 31 && ((int64_t)1 << end_bit) < (int64_t)nrows) ++end_bit;
        size_t tmp_bytes = 0;
        GNNB_CUDA(cub::DeviceRadixSort::SortPairs(nullptr, tmp_bytes, keys, c.row, iota, c.eid, (int)E, 0,
                                                  end_bit, st));
        void* tmp = nullptr;
        GNNB_TRY(sc.alloc(&tmp, tmp_bytes ? tmp_bytes : 1));
        GNNB_CUDA(cub::DeviceRadixSort::SortPairs(tmp, tmp_bytes, keys, c.row, iota, c.eid, (int)E, 0,
                                                  end_bit, st));
        g_launches.fetch_add(4, std::memory_order_relaxed);  // histogram + onesweep passes (library kernels)
        gather_i32_kernel<<<(unsigned)ceil_div(E, 256), 256, 0, st>>>(other, c.eid, E, c.col);
        GNNB_LAUNCHED();
        GNNB_CUDA(cudaStreamSynchronize(st));
    }
    rowptr_kernel<<<(unsigned)ceil_div(E + 1, 256), 256, 0, st>>>(c.row, E, nrows, c.rowptr);
    GNNB_LAUNCHED();
    GNNB_TRY(find_long_rows(c, g->chunk, st));
    c.built = true;
    return GNNB_OK;
}

int ensure_invdeg(gnnb_graph* g, Csr& c, cudaStream_t st) {
    if (c.invdeg) return GNNB_OK;
    std::lock_guard<std::mutex> lock(g->mu);
    if (c.invdeg) return GNNB_OK;
    DeviceScratch sc;
    float* p = nullptr;
    GNNB_TRY(sc.alloc(&p, (size_t)(c.nrows > 0 ? c.nrows : 1)));
    if (c.nrows > 0) {
        invdeg_kernel<<<(unsigned)ceil_div(c.nrows, 256), 256, 0, st>>>(c.rowptr, c.nrows, p);
        GNNB_LAUNCHED();
    }
    c.invdeg = sc.release(p);
    return GNNB_OK;
}

static int convert_indices(const void* p, int64_t n, int index_bytes, int index_base, int64_t limit,
                           int on_device, int32_t* out, int* d_bad, cudaStream_t st) {
    if (n == 0) return GNNB_OK;
    const void* dev = p;
    DeviceScratch sc;
    void* staged = nullptr;
    if (!on_device) {
        GNNB_TRY(sc.alloc(&staged, (size_t)n * index_bytes));
        GNNB_CUDA(cudaMemcpyAsync(staged, p, (size_t)n * index_bytes, cudaMemcpyHostToDevice, st));
        dev = staged;
    }
    unsigned blocks = (unsigned)ceil_div(n, 256);
    if (index_bytes == 8)
        convert_index_kernel<int64_t><<<blocks, 256, 0, st>>>((const int64_t*)dev, n, index_base, limit, out, d_bad);
    else
        convert_index_kernel<int32_t><<<blocks, 256, 0, st>>>((const int32_t*)dev, n, index_base, limit, out, d_bad);
    GNNB_LAUNCHED();
    if (staged) GNNB_CUDA(cudaStreamSynchronize(st));
    return GNNB_OK;
}

// the plan of a new graph g (sizes set): its COO converted and range-checked, and the forward CSR
static int build_plan(gnnb_graph* g, const void* src, const void* dst, int index_bytes, int index_base, int on_device,
                      cudaStream_t st) {
    const size_t nE = (size_t)(g->E > 0 ? g->E : 1);
    GNNB_CUDA(cudaMalloc(&g->coo_src, sizeof(int32_t) * nE));
    GNNB_CUDA(cudaMalloc(&g->coo_dst, sizeof(int32_t) * nE));
    DeviceScratch sc;
    int* d_bad = nullptr;
    GNNB_TRY(sc.alloc(&d_bad, 1));
    GNNB_CUDA(cudaMemsetAsync(d_bad, 0, sizeof(int), st));
    GNNB_TRY(convert_indices(src, g->E, index_bytes, index_base, g->n_src, on_device, g->coo_src, d_bad, st));
    GNNB_TRY(convert_indices(dst, g->E, index_bytes, index_base, g->n_dst, on_device, g->coo_dst, d_bad, st));
    int bad = 0;
    GNNB_CUDA(cudaMemcpyAsync(&bad, d_bad, sizeof(int), cudaMemcpyDeviceToHost, st));
    GNNB_CUDA(cudaStreamSynchronize(st));
    if (bad)
        GNNB_FAIL(GNNB_EINDEX, "edge index out of range: every index must lie in [%d, num_nodes%s] (convert.jl:49-54)",
                  index_base, index_base ? "" : ")");
    return ensure_csr(g, false, st);
}

}  // namespace gnnb

using namespace gnnb;

extern "C" {

int gnnb_set_chunk_edges(int chunk) {
    if (chunk < 32 || chunk > 4096 || (chunk & (chunk - 1))) GNNB_FAIL(GNNB_EINVAL, "chunk must be a power of two in [32,4096]");
    g_chunk_default = chunk;
    return GNNB_OK;
}

int gnnb_graph_create(gnnb_graph_t* out, const void* src, const void* dst, int64_t num_edges,
                      int64_t num_src, int64_t num_dst, int index_bytes, int index_base,
                      int on_device, void* stream) {
    if (!out) GNNB_FAIL(GNNB_EINVAL, "out handle is NULL");
    *out = nullptr;
    if (index_bytes != 4 && index_bytes != 8) GNNB_FAIL(GNNB_EINVAL, "index_bytes must be 4 or 8 (got %d)", index_bytes);
    if (index_base != 0 && index_base != 1) GNNB_FAIL(GNNB_EINVAL, "index_base must be 0 or 1 (got %d)", index_base);
    if (num_edges < 0 || num_src < 0 || num_dst < 0) GNNB_FAIL(GNNB_ESIZE, "negative size");
    if (num_edges >= ((int64_t)1 << 31) - 1 || num_src >= ((int64_t)1 << 31) - 1 || num_dst >= ((int64_t)1 << 31) - 1)
        GNNB_FAIL(GNNB_ESIZE, "a single plan is int32-indexed: E and N must be < 2^31-1 (partition larger graphs)");
    if (num_edges > 0 && (!src || !dst)) GNNB_FAIL(GNNB_EINVAL, "src/dst is NULL");
    if (gnnb_device_count() <= 0) GNNB_FAIL(GNNB_ECUDA, "no CUDA device: libgnnb200 has no CPU fallback");
    cudaStream_t st = (cudaStream_t)stream;
    gnnb_graph* g = new gnnb_graph();
    g->E = num_edges;
    g->n_src = (int32_t)num_src;
    g->n_dst = (int32_t)num_dst;
    g->chunk = g_chunk_default;
    cudaGetDevice(&g->device);
    const int status = build_plan(g, src, dst, index_bytes, index_base, on_device, st);
    if (status != GNNB_OK) {
        gnnb_graph_destroy(g);
        return status;
    }
    *out = g;
    return GNNB_OK;
}

int gnnb_graph_destroy(gnnb_graph_t g) {
    if (!g) return GNNB_OK;
    cudaFree(g->coo_src);
    cudaFree(g->coo_dst);
    free_csr(g->by_dst);
    free_csr(g->by_src);
    cudaFree(g->ws);
    cudaFree(g->ws2);
    cudaFree(g->gcn_c);
    cudaFree(g->bip_c_src);
    cudaFree(g->bip_c_dst);
    cudaFree(g->bip_es_dst);
    cudaFree(g->bip_es_src);
    cudaFree(g->host_ws);
    delete g;
    return GNNB_OK;
}

int gnnb_graph_info(gnnb_graph_t g, int64_t* num_edges, int64_t* num_src, int64_t* num_dst) {
    if (!g) GNNB_FAIL(GNNB_EINVAL, "graph handle is NULL");
    if (num_edges) *num_edges = g->E;
    if (num_src) *num_src = g->n_src;
    if (num_dst) *num_dst = g->n_dst;
    return GNNB_OK;
}

static int derive_self_loop_csr(const Csr& o, Csr& c, int64_t E, int32_t n, int32_t chunk, cudaStream_t st) {
    GNNB_TRY(alloc_csr(c, E + n, n, chunk));
    if (E > 0) {
        selfloop_edges_kernel<<<(unsigned)ceil_div(E, 256), 256, 0, st>>>(o.row, o.col, o.eid, E, c.row, c.col, c.eid);
        GNNB_LAUNCHED();
    }
    selfloop_rows_kernel<<<(unsigned)ceil_div((int64_t)n + 1, 256), 256, 0, st>>>(o.rowptr, n, (int32_t)E, c.rowptr,
                                                                              c.row, c.col, c.eid);
    GNNB_LAUNCHED();
    GNNB_TRY(find_long_rows(c, chunk, st));
    c.built = true;
    return GNNB_OK;
}

// h = add_self_loops(g) (sizes set): g's COO with the n loops appended, and the CSR of each direction g has built
static int self_loops_into(gnnb_graph* g, gnnb_graph* h, cudaStream_t st) {
    const int32_t n = g->n_src;
    const int64_t E = g->E;
    const size_t nE = (size_t)(h->E > 0 ? h->E : 1);
    GNNB_CUDA(cudaMalloc(&h->coo_src, sizeof(int32_t) * nE));
    GNNB_CUDA(cudaMalloc(&h->coo_dst, sizeof(int32_t) * nE));
    if (E > 0) {
        GNNB_CUDA(cudaMemcpyAsync(h->coo_src, g->coo_src, sizeof(int32_t) * E, cudaMemcpyDeviceToDevice, st));
        GNNB_CUDA(cudaMemcpyAsync(h->coo_dst, g->coo_dst, sizeof(int32_t) * E, cudaMemcpyDeviceToDevice, st));
    }
    if (n > 0) {
        iota_kernel<<<(unsigned)ceil_div(n, 256), 256, 0, st>>>(h->coo_src + E, n, 0);
        GNNB_LAUNCHED();
        iota_kernel<<<(unsigned)ceil_div(n, 256), 256, 0, st>>>(h->coo_dst + E, n, 0);
        GNNB_LAUNCHED();
    }
    GNNB_TRY(ensure_csr(g, false, st));
    GNNB_TRY(derive_self_loop_csr(g->by_dst, h->by_dst, E, n, h->chunk, st));
    if (g->by_src.built) GNNB_TRY(derive_self_loop_csr(g->by_src, h->by_src, E, n, h->chunk, st));
    GNNB_CUDA(cudaStreamSynchronize(st));
    return GNNB_OK;
}

int gnnb_graph_add_self_loops(gnnb_graph_t g, gnnb_graph_t* out, void* stream) {
    if (!g || !out) GNNB_FAIL(GNNB_EINVAL, "NULL argument");
    *out = nullptr;
    if (g->n_src != g->n_dst) GNNB_FAIL(GNNB_ESIZE, "add_self_loops needs num_src == num_dst");
    const int32_t n = g->n_src;
    const int64_t E = g->E, E2 = E + n;
    if (E2 >= ((int64_t)1 << 31) - 1) GNNB_FAIL(GNNB_ESIZE, "E + N must be < 2^31-1");
    cudaStream_t st = (cudaStream_t)stream;
    gnnb_graph* h = new gnnb_graph();
    h->E = E2; h->n_src = n; h->n_dst = n; h->chunk = g->chunk; h->device = g->device;
    const int status = self_loops_into(g, h, st);
    if (status != GNNB_OK) { gnnb_graph_destroy(h); return status; }
    *out = h;
    return GNNB_OK;
}

}  // extern "C"

namespace gnnb {

template <typename F>
static int exclusive_scan_flags(F f, int64_t items, int32_t* out, void* tmp, size_t tmp_bytes, cudaStream_t st) {
    GNNB_CUDA(cub::DeviceScan::ExclusiveSum(tmp, tmp_bytes, flag_iter(f), out, (int)items, st));
    g_launches.fetch_add(2, std::memory_order_relaxed);  // tile-state init + scan (library kernels)
    return GNNB_OK;
}

// one direction of the child: compact the parent's sorted (row, col, eid), renumbered, then rowptr and long rows
static int derive_subgraph_csr(const Csr& o, Csr& c, int64_t E, int64_t E2, int32_t nrows, const int32_t* newid,
                               const int32_t* map, int32_t* pos, void* tmp, size_t tmp_bytes, int32_t chunk,
                               cudaStream_t st) {
    GNNB_TRY(alloc_csr(c, E2, nrows, chunk));
    if (E2 > 0) {
        GNNB_TRY(exclusive_scan_flags(SortedKeepFlag{o.eid, newid, E}, E + 1, pos, tmp, tmp_bytes, st));
        subgraph_csr_kernel<<<(unsigned)ceil_div(E, 256), 256, 0, st>>>(o.row, o.col, o.eid, E, pos, newid, map, c.row,
                                                                        c.col, c.eid);
        GNNB_LAUNCHED();
    }
    rowptr_kernel<<<(unsigned)ceil_div(E2 + 1, 256), 256, 0, st>>>(c.row, E2, nrows, c.rowptr);
    GNNB_LAUNCHED();
    GNNB_TRY(find_long_rows(c, chunk, st));
    c.built = true;
    return GNNB_OK;
}

static int subgraph_into(gnnb_graph* g, const uint8_t* node_keep, const uint8_t* edge_keep, int64_t extra_nodes,
                         gnnb_graph* h, int32_t* node_map, int64_t* kept_eids, cudaStream_t st) {
    const int64_t n = g->n_src, E = g->E;
    GNNB_TRY(ensure_csr(g, false, st));
    DeviceScratch sc;
    int32_t* map = nullptr;      // exclusive scan of the node flags: new id of each kept node, count at [n]
    int32_t* newid = nullptr;    // exclusive scan of the COO edge flags: child COO id, count at [E]
    int32_t* pos = nullptr;      // exclusive scan of the flags in one parent direction's sorted order
    GNNB_TRY(sc.alloc(&map, (size_t)(n + 1)));
    GNNB_TRY(sc.alloc(&newid, (size_t)(E + 1)));
    GNNB_TRY(sc.alloc(&pos, (size_t)(E + 1)));
    const NodeKeepFlag nf{node_keep, n};
    const EdgeKeepFlag ef{edge_keep, node_keep, g->coo_src, g->coo_dst, E};
    const SortedKeepFlag sf{g->by_dst.eid, newid, E};
    size_t b0 = 0, b1 = 0, b2 = 0;
    GNNB_CUDA(cub::DeviceScan::ExclusiveSum(nullptr, b0, flag_iter(nf), map, (int)(n + 1), st));
    GNNB_CUDA(cub::DeviceScan::ExclusiveSum(nullptr, b1, flag_iter(ef), newid, (int)(E + 1), st));
    GNNB_CUDA(cub::DeviceScan::ExclusiveSum(nullptr, b2, flag_iter(sf), pos, (int)(E + 1), st));
    const size_t tmp_bytes = std::max(b0, std::max(b1, b2)) + 1;
    void* tmp = nullptr;
    GNNB_TRY(sc.alloc(&tmp, tmp_bytes));

    GNNB_TRY(exclusive_scan_flags(nf, n + 1, map, tmp, tmp_bytes, st));
    GNNB_TRY(exclusive_scan_flags(ef, E + 1, newid, tmp, tmp_bytes, st));
    int32_t counts[2] = {0, 0};
    GNNB_CUDA(cudaMemcpyAsync(&counts[0], map + n, sizeof(int32_t), cudaMemcpyDeviceToHost, st));
    GNNB_CUDA(cudaMemcpyAsync(&counts[1], newid + E, sizeof(int32_t), cudaMemcpyDeviceToHost, st));
    GNNB_CUDA(cudaStreamSynchronize(st));
    const int64_t n2 = (int64_t)counts[0] + extra_nodes, E2 = counts[1];
    if (n2 >= ((int64_t)1 << 31) - 1)
        GNNB_FAIL(GNNB_ESIZE, "kept nodes + extra_nodes = %lld must be < 2^31-1", (long long)n2);
    if (node_map && n > 0) {
        node_map_kernel<<<(unsigned)ceil_div(n, 256), 256, 0, st>>>(node_keep, map, n, node_map);
        GNNB_LAUNCHED();
    }
    h->E = E2;
    h->n_src = h->n_dst = (int32_t)n2;
    const size_t nE = (size_t)(E2 > 0 ? E2 : 1);
    GNNB_CUDA(cudaMalloc(&h->coo_src, sizeof(int32_t) * nE));
    GNNB_CUDA(cudaMalloc(&h->coo_dst, sizeof(int32_t) * nE));
    if (E > 0) {
        subgraph_coo_kernel<<<(unsigned)ceil_div(E, 256), 256, 0, st>>>(g->coo_src, g->coo_dst, E, newid, map,
                                                                        h->coo_src, h->coo_dst, kept_eids);
        GNNB_LAUNCHED();
    }
    GNNB_TRY(derive_subgraph_csr(g->by_dst, h->by_dst, E, E2, (int32_t)n2, newid, map, pos, tmp, tmp_bytes, h->chunk,
                                 st));
    if (g->by_src.built)
        GNNB_TRY(derive_subgraph_csr(g->by_src, h->by_src, E, E2, (int32_t)n2, newid, map, pos, tmp, tmp_bytes,
                                     h->chunk, st));
    GNNB_CUDA(cudaStreamSynchronize(st));
    return GNNB_OK;
}

}  // namespace gnnb

extern "C" {

int gnnb_graph_subgraph(gnnb_graph_t g, const uint8_t* node_keep, const uint8_t* edge_keep, int64_t extra_nodes,
                        gnnb_graph_t* out, int32_t* node_map, int64_t* kept_eids, int64_t* num_nodes_out,
                        int64_t* num_edges_out, void* stream) {
    if (!g || !out) GNNB_FAIL(GNNB_EINVAL, "NULL argument");
    *out = nullptr;
    if (g->n_src != g->n_dst) GNNB_FAIL(GNNB_ESIZE, "subgraph needs num_src == num_dst (no bipartite plans)");
    if (extra_nodes < 0) GNNB_FAIL(GNNB_EINVAL, "extra_nodes must be >= 0 (got %lld)", (long long)extra_nodes);
    gnnb_graph* h = new gnnb_graph();
    h->chunk = g->chunk;
    h->device = g->device;
    const int status = subgraph_into(g, node_keep, edge_keep, extra_nodes, h, node_map, kept_eids,
                                     (cudaStream_t)stream);
    if (status != GNNB_OK) {
        gnnb_graph_destroy(h);
        return status;
    }
    if (num_nodes_out) *num_nodes_out = h->n_src;
    if (num_edges_out) *num_edges_out = h->E;
    *out = h;
    return GNNB_OK;
}

int gnnb_bernoulli_keep(int64_t n, double p, uint64_t seed, uint8_t* keep, void* stream) {
    if (!(p >= 0.0 && p <= 1.0)) GNNB_FAIL(GNNB_EINVAL, "drop probability p = %g must lie in [0, 1]", p);
    if (n < 0 || n >= ((int64_t)1 << 31) - 1) GNNB_FAIL(GNNB_ESIZE, "n = %lld must lie in [0, 2^31-1)", (long long)n);
    if (n == 0) return GNNB_OK;
    if (!keep) GNNB_FAIL(GNNB_EINVAL, "keep is NULL");
    bernoulli_keep_kernel<<<(unsigned)ceil_div(n, 256), 256, 0, (cudaStream_t)stream>>>(n, p, splitmix64(seed), keep);
    GNNB_LAUNCHED();
    return GNNB_OK;
}

int gnnb_graph_csr(gnnb_graph_t g, int transposed, int32_t* rowptr, int32_t* col, int32_t* eid, void* stream) {
    if (!g) GNNB_FAIL(GNNB_EINVAL, "graph handle is NULL");
    cudaStream_t st = (cudaStream_t)stream;
    GNNB_TRY(ensure_csr(g, transposed != 0, st));
    const Csr& c = transposed ? g->by_src : g->by_dst;
    if (rowptr) GNNB_CUDA(cudaMemcpyAsync(rowptr, c.rowptr, sizeof(int32_t) * ((size_t)c.nrows + 1), cudaMemcpyDeviceToHost, st));
    if (col && g->E) GNNB_CUDA(cudaMemcpyAsync(col, c.col, sizeof(int32_t) * (size_t)g->E, cudaMemcpyDeviceToHost, st));
    if (eid && g->E) GNNB_CUDA(cudaMemcpyAsync(eid, c.eid, sizeof(int32_t) * (size_t)g->E, cudaMemcpyDeviceToHost, st));
    GNNB_CUDA(cudaStreamSynchronize(st));
    return GNNB_OK;
}

}  // extern "C"
