// shard.cu — building one GPU's shard of a node-partitioned graph ON that GPU, from chunks of the global edge list.
//
// (No reference counterpart: the reference has no distributed code, SURVEY.md §5/§8e.  Round 1 built shards with torch
// ops over the whole COO on every rank — 3.3-7.5 s at 100 M edges, impossible at 1 B.)
//
// Ownership of node v (0-based): mode 0 = contiguous ranges bounds[q] <= v < bounds[q+1]; mode 1 = cyclic, owner v % W,
// local index v / W (hubs of a skewed id space spread over all ranks).  Either way a node has a *partition id*
// pid(v) = first[owner] + local, a bijection onto [0, N) in which every rank owns one contiguous range — everything below
// works in pid space.  A rank keeps, for the forward shard, every edge whose target it owns (key = local target row,
// other = pid of the source) and, for the backward shard, every edge whose source it owns.  Chunks are compacted with a
// stable scan, so edges keep their COO order inside a row and a shard reproduces the single-GPU summation order.
// finish(): sorted unique remote pids = the halo list (grouped by owner because pid ranges are contiguous), gathered-node
// ids renamed into the [local | halo] space of gnnb_propagate_halo, optional self loops appended, plan created.
#include "common.cuh"
#include <cub/cub.cuh>
#include <vector>

struct gnnb_shard_builder {
    int64_t N = 0;
    int world = 1, rank = 0, mode = 0;
    std::vector<int64_t> first;      // pid range starts per owner, world + 1 entries
    int64_t* d_first = nullptr;      // device copy
    const int32_t* relabel = nullptr;   // optional (caller-owned, device): node -> position in the caller's order; the cyclic
                                        // rule is applied to that position instead of the node id
    int32_t n_local = 0;
    struct Dir {
        int32_t* key = nullptr;      // local reduction row of each kept edge
        int32_t* other = nullptr;    // pid of the gathered node
        int64_t n = 0, cap = 0;
        int32_t* halo_local = nullptr;   // after finish: owner-local row of every halo entry (grouped by owner, ascending)
        int64_t n_halo = 0;
    } dir[2];
    // per-chunk scratch
    uint64_t* flags = nullptr;
    uint64_t* offs = nullptr;
    void* scan_tmp = nullptr;
    size_t scan_bytes = 0;
    int64_t chunk_cap = 0;
    int* d_bad = nullptr;
};

namespace gnnb {
namespace {

struct Owner {
    int64_t N;
    const int64_t* first;   // world + 1
    const int32_t* relabel; // or nullptr
    int world, mode;
    __device__ __forceinline__ int64_t pid(int64_t v) const {
        if (mode == 0) return v;
        if (relabel) v = relabel[v];
        const int q = (int)(v % world);
        return first[q] + v / world;
    }
};

template <typename T>
__global__ void shard_flag_kernel(const T* __restrict__ src, const T* __restrict__ dst, int64_t n, int64_t base, Owner ow,
                                  int64_t lo, int64_t hi, uint64_t* __restrict__ flags, int* __restrict__ bad) {
    const int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    const int64_t s = (int64_t)src[i] - base, t = (int64_t)dst[i] - base;
    if (s < 0 || s >= ow.N || t < 0 || t >= ow.N) { *bad = 1; flags[i] = 0; return; }
    const int64_t ps = ow.pid(s), pt = ow.pid(t);
    const uint64_t f = (pt >= lo && pt < hi) ? 1ull : 0ull;     // forward shard keeps it (target owned)
    const uint64_t b = (ps >= lo && ps < hi) ? 1ull : 0ull;     // backward shard keeps it (source owned)
    flags[i] = f | (b << 32);
}
template <typename T>
__global__ void shard_scatter_kernel(const T* __restrict__ src, const T* __restrict__ dst, int64_t n, int64_t base, Owner ow,
                                     int64_t lo, const uint64_t* __restrict__ flags, const uint64_t* __restrict__ offs,
                                     int32_t* __restrict__ fkey, int32_t* __restrict__ fother, int64_t fbase,
                                     int32_t* __restrict__ bkey, int32_t* __restrict__ bother, int64_t bbase) {
    const int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    const uint64_t fl = flags[i];
    if (fl == 0) return;
    const int64_t ps = ow.pid((int64_t)src[i] - base), pt = ow.pid((int64_t)dst[i] - base);
    const uint64_t o = offs[i];
    if (fl & 0xffffffffull) {
        const int64_t k = fbase + (int64_t)(o & 0xffffffffull);
        fkey[k] = (int32_t)(pt - lo);
        fother[k] = (int32_t)ps;
    }
    if (fl >> 32) {
        const int64_t k = bbase + (int64_t)(o >> 32);
        bkey[k] = (int32_t)(ps - lo);
        bother[k] = (int32_t)pt;
    }
}

__global__ void remote_flag_kernel(const int32_t* __restrict__ other, int64_t n, int32_t lo, int32_t hi,
                                   int32_t* __restrict__ flags) {
    const int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i < n) { const int32_t p = other[i]; flags[i] = (p < lo || p >= hi) ? 1 : 0; }
}
__global__ void compact_kernel(const int32_t* __restrict__ in, const int32_t* __restrict__ flags,
                               const int32_t* __restrict__ offs, int64_t n, int32_t* __restrict__ out) {
    const int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i < n && flags[i]) out[offs[i]] = in[i];
}
__global__ void head_flag_kernel(const int32_t* __restrict__ sorted, int64_t n, int32_t* __restrict__ flags) {
    const int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i < n) flags[i] = (i == 0 || sorted[i] != sorted[i - 1]) ? 1 : 0;
}
// gathered node -> [local | halo] index; appends the self loops (i, i) after the originals
__global__ void rename_kernel(const int32_t* __restrict__ key, const int32_t* __restrict__ other, int64_t n, int32_t lo,
                              int32_t hi, const int32_t* __restrict__ halo, int64_t n_halo, int32_t n_local,
                              int64_t n_loops, int32_t* __restrict__ row, int32_t* __restrict__ col) {
    const int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n + n_loops) return;
    if (i >= n) { row[i] = (int32_t)(i - n); col[i] = (int32_t)(i - n); return; }
    row[i] = key[i];
    const int32_t p = other[i];
    if (p >= lo && p < hi) { col[i] = p - lo; return; }
    int64_t a = 0, b = n_halo;                       // lower_bound: p is present by construction
    while (a < b) { const int64_t m = (a + b) >> 1; if (halo[m] < p) a = m + 1; else b = m; }
    col[i] = n_local + (int32_t)a;
}
// recv_counts[q] = halo entries owned by q; halo_local = owner-local row of every entry
__global__ void halo_owner_kernel(const int32_t* __restrict__ halo, int64_t n_halo, const int64_t* __restrict__ first,
                                  int world, int32_t* __restrict__ halo_local, int64_t* __restrict__ counts) {
    const int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i < n_halo) {
        const int64_t p = halo[i];
        int q = 0;
        while (q + 1 < world && first[q + 1] <= p) ++q;         // world <= 8-16: a short scan
        halo_local[i] = (int32_t)(p - first[q]);
    }
    if (i <= world) {                                            // lower_bound(halo, first[i]) for the count differences
        const int64_t target = first[i];
        int64_t a = 0, b = n_halo;
        while (a < b) { const int64_t m = (a + b) >> 1; if ((int64_t)halo[m] < target) a = m + 1; else b = m; }
        counts[i] = a;
    }
}

template <typename T>
__global__ void degree_acc_kernel(const T* __restrict__ src, const T* __restrict__ dst, int64_t n, int64_t base, int64_t N,
                                  int32_t* __restrict__ cost) {
    const int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    const int64_t s = (int64_t)src[i] - base, t = (int64_t)dst[i] - base;
    if (s >= 0 && s < N) atomicAdd(cost + s, 1);
    if (t >= 0 && t < N) atomicAdd(cost + t, 1);
}
__global__ void iota32_kernel(int32_t* __restrict__ out, int32_t n) {
    const int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i < n) out[i] = (int32_t)i;
}
// deal like cards, reversing direction every round (0..W-1, W-1..0, ...) so that no rank always gets the larger node of a
// round; the last, partial round goes forward to stay inside [0, N).  relabel: node -> position; order: position -> node
__global__ void deal_kernel(const int32_t* __restrict__ by_degree, int32_t n, int world, int32_t* __restrict__ relabel,
                            int32_t* __restrict__ order) {
    const int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    const int32_t r = (int32_t)(i / world), j = (int32_t)(i % world);
    const int32_t o = ((r & 1) && r < n / world) ? world - 1 - j : j;
    const int32_t pos = r * world + o;
    const int32_t v = by_degree[i];
    relabel[v] = pos;
    order[pos] = v;
}

int grow(gnnb_shard_builder::Dir& d, int64_t need, cudaStream_t st) {
    if (need <= d.cap) return GNNB_OK;
    int64_t cap = d.cap + d.cap / 2;
    if (cap < need) cap = need;
    if (cap < (1 << 20)) cap = 1 << 20;
    int32_t *k = nullptr, *o = nullptr;
    GNNB_CUDA(cudaMalloc(&k, sizeof(int32_t) * (size_t)cap));
    GNNB_CUDA(cudaMalloc(&o, sizeof(int32_t) * (size_t)cap));
    if (d.n > 0) {
        GNNB_CUDA(cudaMemcpyAsync(k, d.key, sizeof(int32_t) * (size_t)d.n, cudaMemcpyDeviceToDevice, st));
        GNNB_CUDA(cudaMemcpyAsync(o, d.other, sizeof(int32_t) * (size_t)d.n, cudaMemcpyDeviceToDevice, st));
        GNNB_CUDA(cudaStreamSynchronize(st));
    }
    cudaFree(d.key); cudaFree(d.other);
    d.key = k; d.other = o; d.cap = cap;
    return GNNB_OK;
}

}  // namespace
}  // namespace gnnb

using namespace gnnb;

extern "C" {

int gnnb_shard_builder_create(gnnb_shard_builder_t* out, int64_t num_nodes, int world, int rank, int mode,
                              const int64_t* bounds_host, const int32_t* relabel_dev) {
    if (!out) GNNB_FAIL(GNNB_EINVAL, "out is NULL");
    *out = nullptr;
    if (num_nodes < 0 || num_nodes >= ((int64_t)1 << 31) - 1) GNNB_FAIL(GNNB_ESIZE, "num_nodes must be in [0, 2^31-1)");
    if (world < 1 || world > 64 || rank < 0 || rank >= world) GNNB_FAIL(GNNB_EINVAL, "bad world/rank");
    if (mode != 0 && mode != 1) GNNB_FAIL(GNNB_EINVAL, "ownership mode must be 0 (contiguous) or 1 (cyclic)");
    if (gnnb_device_count() <= 0) GNNB_FAIL(GNNB_ECUDA, "no CUDA device: libgnnb200 has no CPU fallback");
    gnnb_shard_builder* b = new gnnb_shard_builder();
    b->N = num_nodes; b->world = world; b->rank = rank; b->mode = mode;
    b->relabel = mode == 1 ? relabel_dev : nullptr;
    b->first.resize(world + 1);
    if (mode == 0) {
        for (int q = 0; q <= world; ++q)
            b->first[q] = bounds_host ? bounds_host[q] : (num_nodes * q) / world;
        if (b->first[0] != 0 || b->first[world] != num_nodes) { delete b; GNNB_FAIL(GNNB_EINVAL, "bounds must run from 0 to num_nodes"); }
        for (int q = 0; q < world; ++q)
            if (b->first[q + 1] < b->first[q]) { delete b; GNNB_FAIL(GNNB_EINVAL, "bounds must be non-decreasing"); }
    } else {
        b->first[0] = 0;
        for (int q = 0; q < world; ++q) b->first[q + 1] = b->first[q] + (num_nodes - q + world - 1) / world;
    }
    b->n_local = (int32_t)(b->first[rank + 1] - b->first[rank]);
    if (cudaMalloc(&b->d_first, sizeof(int64_t) * (world + 1)) != cudaSuccess || cudaMalloc(&b->d_bad, sizeof(int)) != cudaSuccess) {
        gnnb_shard_builder_destroy(b);
        GNNB_FAIL(GNNB_ENOMEM, "shard builder: cudaMalloc failed");
    }
    cudaMemcpy(b->d_first, b->first.data(), sizeof(int64_t) * (world + 1), cudaMemcpyHostToDevice);
    cudaMemset(b->d_bad, 0, sizeof(int));
    *out = b;
    return GNNB_OK;
}

int gnnb_shard_builder_destroy(gnnb_shard_builder_t b) {
    if (!b) return GNNB_OK;
    for (int d = 0; d < 2; ++d) { cudaFree(b->dir[d].key); cudaFree(b->dir[d].other); cudaFree(b->dir[d].halo_local); }
    cudaFree(b->flags); cudaFree(b->offs); cudaFree(b->scan_tmp); cudaFree(b->d_first); cudaFree(b->d_bad);
    delete b;
    return GNNB_OK;
}

int gnnb_shard_builder_add(gnnb_shard_builder_t b, const void* src, const void* dst, int64_t n, int index_bytes,
                           int index_base, void* stream) {
    if (!b) GNNB_FAIL(GNNB_EINVAL, "builder is NULL");
    if (n < 0 || n >= ((int64_t)1 << 31)) GNNB_FAIL(GNNB_ESIZE, "chunk size must be in [0, 2^31)");
    if (n == 0) return GNNB_OK;
    if (!src || !dst) GNNB_FAIL(GNNB_EINVAL, "src/dst is NULL");
    if (index_bytes != 4 && index_bytes != 8) GNNB_FAIL(GNNB_EINVAL, "index_bytes must be 4 or 8");
    cudaStream_t st = (cudaStream_t)stream;
    if (n > b->chunk_cap) {
        cudaFree(b->flags); cudaFree(b->offs); cudaFree(b->scan_tmp);
        b->flags = nullptr; b->offs = nullptr; b->scan_tmp = nullptr; b->chunk_cap = 0;
        GNNB_CUDA(cudaMalloc(&b->flags, sizeof(uint64_t) * (size_t)n));
        GNNB_CUDA(cudaMalloc(&b->offs, sizeof(uint64_t) * (size_t)n));
        size_t bytes = 0;
        GNNB_CUDA(cub::DeviceScan::ExclusiveSum(nullptr, bytes, b->flags, b->offs, (int)n, st));
        GNNB_CUDA(cudaMalloc(&b->scan_tmp, bytes ? bytes : 1));
        b->scan_bytes = bytes;
        b->chunk_cap = n;
    }
    Owner ow{b->N, b->d_first, b->relabel, b->world, b->mode};
    const int64_t lo = b->first[b->rank], hi = b->first[b->rank + 1];
    const unsigned blocks = (unsigned)ceil_div(n, 256);
    if (index_bytes == 8)
        shard_flag_kernel<int64_t><<<blocks, 256, 0, st>>>((const int64_t*)src, (const int64_t*)dst, n, index_base, ow, lo, hi, b->flags, b->d_bad);
    else
        shard_flag_kernel<int32_t><<<blocks, 256, 0, st>>>((const int32_t*)src, (const int32_t*)dst, n, index_base, ow, lo, hi, b->flags, b->d_bad);
    GNNB_LAUNCHED();
    size_t bytes = b->scan_bytes;
    GNNB_CUDA(cub::DeviceScan::ExclusiveSum(b->scan_tmp, bytes, b->flags, b->offs, (int)n, st));
    g_launches.fetch_add(1, std::memory_order_relaxed);
    uint64_t last_f = 0, last_o = 0;
    int bad = 0;
    GNNB_CUDA(cudaMemcpyAsync(&last_f, b->flags + (n - 1), sizeof(uint64_t), cudaMemcpyDeviceToHost, st));
    GNNB_CUDA(cudaMemcpyAsync(&last_o, b->offs + (n - 1), sizeof(uint64_t), cudaMemcpyDeviceToHost, st));
    GNNB_CUDA(cudaMemcpyAsync(&bad, b->d_bad, sizeof(int), cudaMemcpyDeviceToHost, st));
    GNNB_CUDA(cudaStreamSynchronize(st));
    if (bad) GNNB_FAIL(GNNB_EINDEX, "edge index out of range: every index must lie in [%d, num_nodes%s] (convert.jl:49-54)",
                       index_base, index_base ? "" : ")");
    const uint64_t tot = last_f + last_o;
    const int64_t nf = (int64_t)(tot & 0xffffffffull), nb = (int64_t)(tot >> 32);
    if (b->dir[0].n + nf >= ((int64_t)1 << 31) - 1 - b->n_local || b->dir[1].n + nb >= ((int64_t)1 << 31) - 1 - b->n_local)
        GNNB_FAIL(GNNB_ESIZE, "a shard is int32-indexed: more than 2^31 edges on one rank (use more ranks)");
    GNNB_TRY(grow(b->dir[0], b->dir[0].n + nf, st));
    GNNB_TRY(grow(b->dir[1], b->dir[1].n + nb, st));
    if (index_bytes == 8)
        shard_scatter_kernel<int64_t><<<blocks, 256, 0, st>>>((const int64_t*)src, (const int64_t*)dst, n, index_base, ow, lo, b->flags, b->offs,
                                                              b->dir[0].key, b->dir[0].other, b->dir[0].n, b->dir[1].key, b->dir[1].other, b->dir[1].n);
    else
        shard_scatter_kernel<int32_t><<<blocks, 256, 0, st>>>((const int32_t*)src, (const int32_t*)dst, n, index_base, ow, lo, b->flags, b->offs,
                                                              b->dir[0].key, b->dir[0].other, b->dir[0].n, b->dir[1].key, b->dir[1].other, b->dir[1].n);
    GNNB_LAUNCHED();
    b->dir[0].n += nf;
    b->dir[1].n += nb;
    return GNNB_OK;
}

int gnnb_shard_builder_finish(gnnb_shard_builder_t b, int direction, int add_self_loops, gnnb_graph_t* plan_out,
                              int64_t* n_local_out, int64_t* n_halo_out, int64_t* num_edges_out, int64_t* recv_counts_host,
                              void* stream) {
    if (!b || !plan_out) GNNB_FAIL(GNNB_EINVAL, "NULL argument");
    if (direction != 0 && direction != 1) GNNB_FAIL(GNNB_EINVAL, "direction must be 0 (forward shard) or 1 (backward shard)");
    *plan_out = nullptr;
    cudaStream_t st = (cudaStream_t)stream;
    gnnb_shard_builder::Dir& d = b->dir[direction];
    const int64_t n = d.n;
    const int32_t lo = (int32_t)b->first[b->rank], hi = (int32_t)b->first[b->rank + 1];
    const int32_t n_local = b->n_local;
    const int64_t n_loops = add_self_loops ? n_local : 0;
    const int64_t ne = n + n_loops;
    DeviceScratch sc;                 // the halo, the renamed edges and the receive counts: until the plan is built
    int32_t *halo = nullptr, *row = nullptr, *col = nullptr;
    int64_t* counts = nullptr;
    int64_t n_halo = 0;
    {
        DeviceScratch edge_sc;        // the remote-source flags, their scan and the sorted remote sources
        if (n > 0) {
            int32_t *flags = nullptr, *offs = nullptr, *rem = nullptr, *rem_s = nullptr;
            void* tmp = nullptr;
            GNNB_TRY(edge_sc.alloc(&flags, (size_t)n));
            GNNB_TRY(edge_sc.alloc(&offs, (size_t)n));
            remote_flag_kernel<<<(unsigned)ceil_div(n, 256), 256, 0, st>>>(d.other, n, lo, hi, flags);
            size_t bytes = 0;
            GNNB_CUDA(cub::DeviceScan::ExclusiveSum(nullptr, bytes, flags, offs, (int)n, st));
            GNNB_TRY(edge_sc.alloc(&tmp, bytes ? bytes : 1));
            GNNB_CUDA(cub::DeviceScan::ExclusiveSum(tmp, bytes, flags, offs, (int)n, st));
            int32_t lf = 0, lo_ = 0;
            GNNB_CUDA(cudaMemcpyAsync(&lf, flags + (n - 1), sizeof(int32_t), cudaMemcpyDeviceToHost, st));
            GNNB_CUDA(cudaMemcpyAsync(&lo_, offs + (n - 1), sizeof(int32_t), cudaMemcpyDeviceToHost, st));
            GNNB_CUDA(cudaStreamSynchronize(st));
            const int64_t n_rem = (int64_t)lf + lo_;
            if (n_rem > 0) {
                GNNB_TRY(edge_sc.alloc(&rem, (size_t)n_rem));
                GNNB_TRY(edge_sc.alloc(&rem_s, (size_t)n_rem));
                compact_kernel<<<(unsigned)ceil_div(n, 256), 256, 0, st>>>(d.other, flags, offs, n, rem);
                int end_bit = 1;
                while (end_bit < 31 && ((int64_t)1 << end_bit) < b->N) ++end_bit;
                GNNB_CUDA(cub::DeviceRadixSort::SortKeys(nullptr, bytes, rem, rem_s, (int)n_rem, 0, end_bit, st));
                GNNB_TRY(edge_sc.alloc(&tmp, bytes ? bytes : 1));
                GNNB_CUDA(cub::DeviceRadixSort::SortKeys(tmp, bytes, rem, rem_s, (int)n_rem, 0, end_bit, st));
                // unique: head flags -> scan -> compact (flags / offs are reused: n_rem <= n)
                head_flag_kernel<<<(unsigned)ceil_div(n_rem, 256), 256, 0, st>>>(rem_s, n_rem, flags);
                GNNB_CUDA(cub::DeviceScan::ExclusiveSum(nullptr, bytes, flags, offs, (int)n_rem, st));
                GNNB_TRY(edge_sc.alloc(&tmp, bytes ? bytes : 1));
                GNNB_CUDA(cub::DeviceScan::ExclusiveSum(tmp, bytes, flags, offs, (int)n_rem, st));
                GNNB_CUDA(cudaMemcpyAsync(&lf, flags + (n_rem - 1), sizeof(int32_t), cudaMemcpyDeviceToHost, st));
                GNNB_CUDA(cudaMemcpyAsync(&lo_, offs + (n_rem - 1), sizeof(int32_t), cudaMemcpyDeviceToHost, st));
                GNNB_CUDA(cudaStreamSynchronize(st));
                n_halo = (int64_t)lf + lo_;
                GNNB_TRY(sc.alloc(&halo, (size_t)n_halo));
                compact_kernel<<<(unsigned)ceil_div(n_rem, 256), 256, 0, st>>>(rem_s, flags, offs, n_rem, halo);
            }
            g_launches.fetch_add(8, std::memory_order_relaxed);
        }
        GNNB_TRY(sc.alloc(&row, (size_t)(ne > 0 ? ne : 1)));
        GNNB_TRY(sc.alloc(&col, (size_t)(ne > 0 ? ne : 1)));
        if (ne > 0) {
            rename_kernel<<<(unsigned)ceil_div(ne, 256), 256, 0, st>>>(d.key, d.other, n, lo, hi, halo, n_halo, n_local, n_loops, row, col);
            g_launches.fetch_add(1, std::memory_order_relaxed);
        }
        GNNB_TRY(sc.alloc(&counts, (size_t)(b->world + 1)));
        cudaFree(d.halo_local); d.halo_local = nullptr;
        GNNB_CUDA(cudaMalloc(&d.halo_local, sizeof(int32_t) * (size_t)(n_halo > 0 ? n_halo : 1)));
        {
            const int64_t threads = n_halo > b->world + 1 ? n_halo : b->world + 1;
            halo_owner_kernel<<<(unsigned)ceil_div(threads, 256), 256, 0, st>>>(halo, n_halo, b->d_first, b->world, d.halo_local, counts);
            g_launches.fetch_add(1, std::memory_order_relaxed);
        }
        std::vector<int64_t> hc(b->world + 1);
        GNNB_CUDA(cudaMemcpyAsync(hc.data(), counts, sizeof(int64_t) * (size_t)(b->world + 1), cudaMemcpyDeviceToHost, st));
        GNNB_CUDA(cudaGetLastError());
        GNNB_CUDA(cudaStreamSynchronize(st));
        if (recv_counts_host) for (int q = 0; q < b->world; ++q) recv_counts_host[q] = hc[q + 1] - hc[q];
        d.n_halo = n_halo;
        // the edge arrays of this direction are no longer needed: the plan keeps its own copies
        cudaFree(d.key); cudaFree(d.other); d.key = nullptr; d.other = nullptr; d.cap = 0; d.n = 0;
    }
    GNNB_TRY(gnnb_graph_create(plan_out, col, row, ne, (int64_t)n_local + n_halo, n_local, 4, 0, 1, stream));
    if (n_local_out) *n_local_out = n_local;
    if (n_halo_out) *n_halo_out = n_halo;
    if (num_edges_out) *num_edges_out = ne;
    return GNNB_OK;
}

// ---- 'balanced' ownership: degree histogram over the chunks, then the nodes dealt to the ranks by decreasing degree ------
int gnnb_degree_accumulate(const void* src, const void* dst, int64_t n, int index_bytes, int index_base, int64_t num_nodes,
                           int32_t* cost_dev, void* stream) {
    if (n < 0 || num_nodes < 0) GNNB_FAIL(GNNB_ESIZE, "negative size");
    if (n == 0) return GNNB_OK;
    if (!src || !dst || !cost_dev) GNNB_FAIL(GNNB_EINVAL, "NULL argument");
    if (index_bytes != 4 && index_bytes != 8) GNNB_FAIL(GNNB_EINVAL, "index_bytes must be 4 or 8");
    cudaStream_t st = (cudaStream_t)stream;
    if (index_bytes == 8) degree_acc_kernel<int64_t><<<(unsigned)ceil_div(n, 256), 256, 0, st>>>((const int64_t*)src, (const int64_t*)dst, n, index_base, num_nodes, cost_dev);
    else degree_acc_kernel<int32_t><<<(unsigned)ceil_div(n, 256), 256, 0, st>>>((const int32_t*)src, (const int32_t*)dst, n, index_base, num_nodes, cost_dev);
    GNNB_LAUNCHED();
    return GNNB_OK;
}

int gnnb_balanced_relabel(const int32_t* cost_dev, int64_t num_nodes, int world, int32_t* relabel_dev, int32_t* order_dev,
                          void* stream) {
    if (num_nodes < 0 || num_nodes >= ((int64_t)1 << 31) - 1 || world < 1) GNNB_FAIL(GNNB_ESIZE, "bad sizes");
    if (num_nodes == 0) return GNNB_OK;
    if (!cost_dev || !relabel_dev || !order_dev) GNNB_FAIL(GNNB_EINVAL, "NULL argument");
    cudaStream_t st = (cudaStream_t)stream;
    const int n = (int)num_nodes;
    DeviceScratch sc;
    int32_t *ids = nullptr, *cost_s = nullptr, *by_degree = nullptr;
    void* tmp = nullptr;
    GNNB_TRY(sc.alloc(&ids, (size_t)n));
    GNNB_TRY(sc.alloc(&cost_s, (size_t)n));
    GNNB_TRY(sc.alloc(&by_degree, (size_t)n));
    iota32_kernel<<<(unsigned)ceil_div((int64_t)n, 256), 256, 0, st>>>(ids, n);
    size_t bytes = 0;                                        // stable: ties keep id order, identical on every rank
    GNNB_CUDA(cub::DeviceRadixSort::SortPairsDescending(nullptr, bytes, cost_dev, cost_s, ids, by_degree, n, 0, 32, st));
    GNNB_TRY(sc.alloc(&tmp, bytes ? bytes : 1));
    GNNB_CUDA(cub::DeviceRadixSort::SortPairsDescending(tmp, bytes, cost_dev, cost_s, ids, by_degree, n, 0, 32, st));
    deal_kernel<<<(unsigned)ceil_div((int64_t)n, 256), 256, 0, st>>>(by_degree, n, world, relabel_dev, order_dev);
    GNNB_CUDA(cudaGetLastError());
    GNNB_CUDA(cudaStreamSynchronize(st));
    g_launches.fetch_add(4, std::memory_order_relaxed);
    return GNNB_OK;
}

int gnnb_shard_builder_halo(gnnb_shard_builder_t b, int direction, int32_t* halo_local_dev, void* stream) {
    if (!b || (direction != 0 && direction != 1)) GNNB_FAIL(GNNB_EINVAL, "bad argument");
    const gnnb_shard_builder::Dir& d = b->dir[direction];
    if (d.n_halo > 0) {
        if (!halo_local_dev) GNNB_FAIL(GNNB_EINVAL, "halo_local_dev is NULL");
        GNNB_CUDA(cudaMemcpyAsync(halo_local_dev, d.halo_local, sizeof(int32_t) * (size_t)d.n_halo, cudaMemcpyDeviceToDevice,
                                  (cudaStream_t)stream));
    }
    return GNNB_OK;
}

}  // extern "C"
