// transform.cu — edge-list transforms on the device (SURVEY.md §8f rank 3): the index work either side of the hot
// path that the reference does on the CPU.
//
// Reference counterparts:
//   sort_edge_index(u, v)                 GNNGraphs/src/utils.jl:41-45 (sortperm of the zipped pairs); for CuArrays the
//                                         CUDA extension copies to the host, sorts there and copies back
//                                         (GNNGraphs/ext/GNNGraphsCUDAExt.jl:24-30, "TODO proper cuda friendly
//                                         implementation") — this is that implementation.
//   remove_multi_edges(g; aggr)           GNNGraphs/src/transform.jl:157-190: edge_encoding, sortperm, first-occurrence
//                                         mask, running segment id; the feature aggregation (`_scatter(aggr, ·, idxs)`)
//                                         is the library's segmented scatter over the segment ids this returns.
//   to_bidirected(g)                      transform.jl:495-510 = concatenate both directions + the above with mean.
//
// Both are one 64-bit key per edge ((u << vbits) | v — order-isomorphic to the reference's (s-1)*n + t encoding and
// to tuple comparison), a stable CUB radix sort over just the bits in use, and one or two streaming passes.  HBM-bound
// integer work: 8 B key + 4 B payload per edge per radix pass.
#include "common.cuh"
#include <cub/cub.cuh>

namespace gnnb {

template <typename T>
__global__ void encode_pairs_kernel(const T* __restrict__ u, const T* __restrict__ v, int64_t E, int64_t lo,
                                    int64_t hi, int vbits, uint64_t* __restrict__ keys, int32_t* __restrict__ iota,
                                    int* __restrict__ bad) {
    int64_t k = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (k >= E) return;
    int64_t a = (int64_t)u[k], b = (int64_t)v[k];
    if (a < lo || a >= hi || b < lo || b >= hi) {
        atomicExch(bad, 1);
        a = lo;
        b = lo;
    }
    keys[k] = ((uint64_t)(a - lo) << vbits) | (uint64_t)(b - lo);
    iota[k] = (int32_t)k;
}

template <typename T>
__global__ void decode_pairs_kernel(const uint64_t* __restrict__ keys, const int32_t* __restrict__ perm, int64_t E,
                                    int64_t lo, int vbits, T* __restrict__ u_out, T* __restrict__ v_out,
                                    int64_t* __restrict__ perm_out) {
    int64_t k = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (k >= E) return;
    uint64_t key = keys[k];
    if (u_out) u_out[k] = (T)((int64_t)(key >> vbits) + lo);
    if (v_out) v_out[k] = (T)((int64_t)(key & ((1ull << vbits) - 1)) + lo);
    if (perm_out) perm_out[k] = (int64_t)perm[k];
}

__global__ void head_flags_kernel(const uint64_t* __restrict__ keys, int64_t E, int32_t* __restrict__ flags) {
    int64_t k = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (k >= E) return;
    flags[k] = (k == 0 || keys[k] != keys[k - 1]) ? 1 : 0;
}

// seg[k] = 1-based id of the run sorted edge k belongs to (inclusive scan of the head flags); the head of each run
// writes the run's pair.
template <typename T>
__global__ void emit_unique_kernel(const uint64_t* __restrict__ keys, const int32_t* __restrict__ flags,
                                   const int32_t* __restrict__ seg, const int32_t* __restrict__ perm, int64_t E,
                                   int64_t lo, int vbits, T* __restrict__ s_out, T* __restrict__ t_out,
                                   int64_t* __restrict__ perm_out, int64_t* __restrict__ seg_out) {
    int64_t k = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (k >= E) return;
    int32_t sg = seg[k];
    perm_out[k] = (int64_t)perm[k];
    seg_out[k] = (int64_t)sg;
    if (flags[k]) {
        uint64_t key = keys[k];
        s_out[sg - 1] = (T)((int64_t)(key >> vbits) + lo);
        t_out[sg - 1] = (T)((int64_t)(key & ((1ull << vbits) - 1)) + lo);
    }
}

static int bits_for(int64_t span) {  // bits needed for values in [0, span)
    int b = 1;
    while (b < 31 && ((int64_t)1 << b) < span) ++b;
    return b;
}

// *keys_sorted / *perm <- stable sort of the pairs by (u, v), in the caller's scratch; values must lie in [lo, hi)
static int sort_pairs(const void* u, const void* v, int64_t E, int index_bytes, int64_t lo, int64_t hi, int vbits,
                      DeviceScratch& sc, uint64_t** keys_sorted, int32_t** perm, cudaStream_t st) {
    uint64_t* keys = nullptr;
    int32_t* iota = nullptr;
    int* d_bad = nullptr;
    void* tmp = nullptr;
    GNNB_TRY(sc.alloc(&keys, (size_t)E));
    GNNB_TRY(sc.alloc(keys_sorted, (size_t)E));
    GNNB_TRY(sc.alloc(&iota, (size_t)E));
    GNNB_TRY(sc.alloc(perm, (size_t)E));
    GNNB_TRY(sc.alloc(&d_bad, 1));
    GNNB_CUDA(cudaMemsetAsync(d_bad, 0, sizeof(int), st));
    const unsigned blocks = (unsigned)ceil_div(E, 256);
    if (index_bytes == 8)
        encode_pairs_kernel<int64_t><<<blocks, 256, 0, st>>>((const int64_t*)u, (const int64_t*)v, E, lo, hi, vbits,
                                                             keys, iota, d_bad);
    else
        encode_pairs_kernel<int32_t><<<blocks, 256, 0, st>>>((const int32_t*)u, (const int32_t*)v, E, lo, hi, vbits,
                                                             keys, iota, d_bad);
    GNNB_LAUNCHED();
    size_t tmp_bytes = 0;
    GNNB_CUDA(cub::DeviceRadixSort::SortPairs(nullptr, tmp_bytes, keys, *keys_sorted, iota, *perm, (int)E, 0,
                                              2 * vbits, st));
    GNNB_TRY(sc.alloc(&tmp, tmp_bytes ? tmp_bytes : 1));
    GNNB_CUDA(cub::DeviceRadixSort::SortPairs(tmp, tmp_bytes, keys, *keys_sorted, iota, *perm, (int)E, 0,
                                              2 * vbits, st));
    g_launches.fetch_add(2, std::memory_order_relaxed);  // histogram + onesweep passes (library kernels)
    int bad = 0;
    GNNB_CUDA(cudaMemcpyAsync(&bad, d_bad, sizeof(int), cudaMemcpyDeviceToHost, st));
    GNNB_CUDA(cudaStreamSynchronize(st));
    if (bad) GNNB_FAIL(GNNB_EINDEX, "edge index outside [%lld, %lld)", (long long)lo, (long long)hi);
    return GNNB_OK;
}

int run_head_flags(const uint64_t* keys, int64_t E, int32_t* flags, cudaStream_t st) {
    if (E == 0) return GNNB_OK;
    head_flags_kernel<<<(unsigned)ceil_div(E, 256), 256, 0, st>>>(keys, E, flags);
    GNNB_LAUNCHED();
    return GNNB_OK;
}

static int check_args(int64_t E, int64_t max_index, int index_bytes) {
    if (index_bytes != 4 && index_bytes != 8) GNNB_FAIL(GNNB_EINVAL, "index_bytes must be 4 or 8 (got %d)", index_bytes);
    if (E < 0 || E >= ((int64_t)1 << 31)) GNNB_FAIL(GNNB_ESIZE, "number of edges %lld outside [0, 2^31)", (long long)E);
    if (max_index < 0 || max_index >= ((int64_t)1 << 31))
        GNNB_FAIL(GNNB_ESIZE, "index bound %lld outside [0, 2^31)", (long long)max_index);
    return GNNB_OK;
}

}  // namespace gnnb

using namespace gnnb;

extern "C" {

int gnnb_sort_edge_index(const void* u, const void* v, int64_t num_edges, int64_t max_index, int index_bytes,
                         void* u_out, void* v_out, int64_t* perm_out, void* stream) {
    GNNB_TRY(check_args(num_edges, max_index, index_bytes));
    if (num_edges == 0) return GNNB_OK;
    if (!u || !v) GNNB_FAIL(GNNB_EINVAL, "gnnb_sort_edge_index: NULL index array");
    cudaStream_t st = (cudaStream_t)stream;
    const int64_t lo = 0, hi = max_index + 1;  // values in [0, max_index]: works for 0- and 1-based ids alike
    const int vbits = bits_for(hi);
    DeviceScratch sc;
    uint64_t* keys_sorted = nullptr;
    int32_t* perm = nullptr;
    GNNB_TRY(sort_pairs(u, v, num_edges, index_bytes, lo, hi, vbits, sc, &keys_sorted, &perm, st));
    const unsigned blocks = (unsigned)ceil_div(num_edges, 256);
    if (index_bytes == 8)
        decode_pairs_kernel<int64_t><<<blocks, 256, 0, st>>>(keys_sorted, perm, num_edges, lo, vbits, (int64_t*)u_out,
                                                             (int64_t*)v_out, perm_out);
    else
        decode_pairs_kernel<int32_t><<<blocks, 256, 0, st>>>(keys_sorted, perm, num_edges, lo, vbits, (int32_t*)u_out,
                                                             (int32_t*)v_out, perm_out);
    GNNB_LAUNCHED();
    GNNB_CUDA(cudaStreamSynchronize(st));  // scratch is freed on return
    return GNNB_OK;
}

int gnnb_coalesce_edges(const void* src, const void* dst, int64_t num_edges, int64_t num_nodes, int index_bytes,
                        int index_base, void* src_out, void* dst_out, int64_t* perm_out, int64_t* seg_out,
                        int64_t* num_unique, void* stream) {
    GNNB_TRY(check_args(num_edges, num_nodes, index_bytes));
    if (index_base != 0 && index_base != 1) GNNB_FAIL(GNNB_EINVAL, "index_base must be 0 or 1 (got %d)", index_base);
    if (!num_unique) GNNB_FAIL(GNNB_EINVAL, "gnnb_coalesce_edges: num_unique is NULL");
    *num_unique = 0;
    if (num_edges == 0) return GNNB_OK;
    if (!src || !dst || !src_out || !dst_out || !perm_out || !seg_out)
        GNNB_FAIL(GNNB_EINVAL, "gnnb_coalesce_edges: NULL array");
    cudaStream_t st = (cudaStream_t)stream;
    const int64_t lo = index_base, hi = index_base + num_nodes;
    const int vbits = bits_for(num_nodes);
    DeviceScratch sc;
    uint64_t* keys_sorted = nullptr;
    int32_t *perm = nullptr, *flags = nullptr, *seg = nullptr;
    void* tmp = nullptr;
    GNNB_TRY(sort_pairs(src, dst, num_edges, index_bytes, lo, hi, vbits, sc, &keys_sorted, &perm, st));
    const unsigned blocks = (unsigned)ceil_div(num_edges, 256);
    GNNB_TRY(sc.alloc(&flags, (size_t)num_edges));
    GNNB_TRY(sc.alloc(&seg, (size_t)num_edges));
    head_flags_kernel<<<blocks, 256, 0, st>>>(keys_sorted, num_edges, flags);
    GNNB_LAUNCHED();
    size_t tmp_bytes = 0;
    GNNB_CUDA(cub::DeviceScan::InclusiveSum(nullptr, tmp_bytes, flags, seg, (int)num_edges, st));
    GNNB_TRY(sc.alloc(&tmp, tmp_bytes ? tmp_bytes : 1));
    GNNB_CUDA(cub::DeviceScan::InclusiveSum(tmp, tmp_bytes, flags, seg, (int)num_edges, st));
    g_launches.fetch_add(1, std::memory_order_relaxed);
    if (index_bytes == 8)
        emit_unique_kernel<int64_t><<<blocks, 256, 0, st>>>(keys_sorted, flags, seg, perm, num_edges, lo, vbits,
                                                            (int64_t*)src_out, (int64_t*)dst_out, perm_out, seg_out);
    else
        emit_unique_kernel<int32_t><<<blocks, 256, 0, st>>>(keys_sorted, flags, seg, perm, num_edges, lo, vbits,
                                                            (int32_t*)src_out, (int32_t*)dst_out, perm_out, seg_out);
    GNNB_LAUNCHED();
    int32_t last = 0;
    GNNB_CUDA(cudaMemcpyAsync(&last, seg + (num_edges - 1), sizeof(int32_t), cudaMemcpyDeviceToHost, st));
    GNNB_CUDA(cudaStreamSynchronize(st));
    *num_unique = last;
    return GNNB_OK;
}

int gnnb_graph_csr_device(gnnb_graph_t g, int transposed, int32_t* rowptr_dev, int32_t* col_dev, int32_t* eid_dev,
                          void* stream) {
    if (!g) GNNB_FAIL(GNNB_EINVAL, "gnnb_graph_csr_device: NULL graph");
    cudaStream_t st = (cudaStream_t)stream;
    GNNB_TRY(ensure_csr(g, transposed != 0, st));
    const Csr& c = transposed ? g->by_src : g->by_dst;
    if (rowptr_dev)
        GNNB_CUDA(cudaMemcpyAsync(rowptr_dev, c.rowptr, sizeof(int32_t) * ((size_t)c.nrows + 1), cudaMemcpyDeviceToDevice, st));
    if (col_dev && g->E)
        GNNB_CUDA(cudaMemcpyAsync(col_dev, c.col, sizeof(int32_t) * (size_t)g->E, cudaMemcpyDeviceToDevice, st));
    if (eid_dev && g->E)
        GNNB_CUDA(cudaMemcpyAsync(eid_dev, c.eid, sizeof(int32_t) * (size_t)g->E, cudaMemcpyDeviceToDevice, st));
    return GNNB_OK;
}

}  // extern "C"
