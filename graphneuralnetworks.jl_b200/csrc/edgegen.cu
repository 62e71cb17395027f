// edgegen.cu — edge codes and random edges on the device: the primitive behind rand_graph, negative_sample,
// rand_edge_split and perturb_edges (link prediction), plus the encode / decode / sorted-set / membership helpers.
//
// Reference counterparts (all on the host there):
//   edge_encoding / edge_decoding      GNNGraphs/src/utils.jl:189-268
//   _rand_edges (StatsBase.sample)     GNNGraphs/src/utils.jl:270-290, used by rand_graph (generate.jl:51-65)
//   negative_sample                    GNNGraphs/src/transform.jl:890-929: copies the graph to the CPU, randsubseq over
//                                      all codes, setdiff! against the positives, keeps the smallest num_neg codes
//   randperm in rand_edge_split        GNNGraphs/src/transform.jl:945-968
//
// One primitive: the first m codes of a seeded permutation π of [0, M) that are not in a sorted exclusion set.  π is a
// Feistel network over the smallest power of four >= M, cycle-walked into [0, M) (a walk from i < M ends because the
// network is a bijection: the orbit of i returns to i).  A batch of consecutive indices is permuted and tested
// against the exclusion set by binary search, a CUB scan numbers the survivors, and an order-preserving scatter keeps
// the first ones.  The host sizes batches from the exact number of available codes M - x, so one batch usually
// suffices; each batch reads back one count.
#include "common.cuh"
#include <cub/cub.cuh>
#include <math.h>
#include <algorithm>

namespace gnnb {

// ---- code spaces ------------------------------------------------------------------------------------------------
struct Space {
    int kind;
    uint64_t n1, n2;  // n2 only for BIPARTITE (else == n1)
    uint64_t M;
};

static int make_space(int kind, int64_t n1, int64_t n2, Space* sp) {
    if (kind < GNNB_CODES_DIRECTED || kind > GNNB_CODES_BIPARTITE) GNNB_FAIL(GNNB_EINVAL, "unknown code space %d", kind);
    if (n1 < 0 || n1 >= ((int64_t)1 << 31)) GNNB_FAIL(GNNB_ESIZE, "n = %lld outside [0, 2^31)", (long long)n1);
    if (kind == GNNB_CODES_BIPARTITE && (n2 < 0 || n2 >= ((int64_t)1 << 31)))
        GNNB_FAIL(GNNB_ESIZE, "n2 = %lld outside [0, 2^31)", (long long)n2);
    const uint64_t n = (uint64_t)n1;
    sp->kind = kind;
    sp->n1 = n;
    sp->n2 = kind == GNNB_CODES_BIPARTITE ? (uint64_t)n2 : n;
    switch (kind) {
        case GNNB_CODES_DIRECTED: sp->M = n * n; break;
        case GNNB_CODES_DIRECTED_NOLOOP: sp->M = n ? n * (n - 1) : 0; break;
        case GNNB_CODES_UNDIRECTED: sp->M = n * (n + 1) / 2; break;
        case GNNB_CODES_UNDIRECTED_NOLOOP: sp->M = n ? n * (n - 1) / 2 : 0; break;
        default: sp->M = n * sp->n2; break;
    }
    return GNNB_OK;
}

// first code of row s in the undirected spaces: s (a - s) / 2 with a = 2n + 1 (loops) or 2n - 1 (no loops)
__host__ __device__ static inline uint64_t tri_start(uint64_t a, uint64_t s) { return s * (a - s) / 2; }

// 0 = encoded; 1 = id out of range; 2 = a self loop in a NOLOOP space
__host__ __device__ static inline int encode_pair(const Space& sp, int64_t a, int64_t b, uint64_t* code) {
    if (a < 0 || b < 0 || (uint64_t)a >= sp.n1 || (uint64_t)b >= sp.n2) return 1;
    uint64_t s = (uint64_t)a, t = (uint64_t)b;
    const uint64_t n = sp.n1;
    switch (sp.kind) {
        case GNNB_CODES_DIRECTED: *code = s * n + t; return 0;
        case GNNB_CODES_DIRECTED_NOLOOP:
            if (s == t) return 2;
            *code = s * (n - 1) + t - (t > s ? 1 : 0);
            return 0;
        case GNNB_CODES_UNDIRECTED:
        case GNNB_CODES_UNDIRECTED_NOLOOP: {
            if (s > t) { const uint64_t z = s; s = t; t = z; }
            const bool loops = sp.kind == GNNB_CODES_UNDIRECTED;
            if (!loops && s == t) return 2;
            *code = tri_start(loops ? 2 * n + 1 : 2 * n - 1, s) + (t - s) - (loops ? 0 : 1);
            return 0;
        }
        default: *code = s * sp.n2 + t; return 0;
    }
}

// c < sp.M
__host__ __device__ static inline void decode_code(const Space& sp, uint64_t c, uint64_t* s_out, uint64_t* t_out) {
    const uint64_t n = sp.n1;
    switch (sp.kind) {
        case GNNB_CODES_DIRECTED: *s_out = c / n; *t_out = c % n; return;
        case GNNB_CODES_DIRECTED_NOLOOP: {
            const uint64_t s = c / (n - 1), r = c % (n - 1);
            *s_out = s;
            *t_out = r + (r >= s ? 1 : 0);
            return;
        }
        case GNNB_CODES_UNDIRECTED:
        case GNNB_CODES_UNDIRECTED_NOLOOP: {
            const bool loops = sp.kind == GNNB_CODES_UNDIRECTED;
            const uint64_t a = loops ? 2 * n + 1 : 2 * n - 1;   // a < 2^32, so a² and 8c < a² fit in uint64
            const uint64_t rows = loops ? n : n - 1;
            const uint64_t disc = a * a - 8 * c;                 // row s = floor((a - sqrt(disc)) / 2), exact integer
            double est = floor(((double)a - sqrt((double)disc)) * 0.5);
            uint64_t s = est <= 0.0 ? 0 : (uint64_t)est;
            if (s > rows - 1) s = rows - 1;
            while (s > 0 && tri_start(a, s) > c) --s;           // the float estimate is within one row: correct it
            while (s + 1 < rows && tri_start(a, s + 1) <= c) ++s;
            *s_out = s;
            *t_out = s + (c - tri_start(a, s)) + (loops ? 0 : 1);
            return;
        }
        default: *s_out = c / sp.n2; *t_out = c % sp.n2; return;
    }
}

// mode 0 (encode): every pair must be in the space.  mode 1 (set): pairs outside the space become the sentinel M.
__global__ void encode_kernel(Space sp, const int64_t* __restrict__ s, const int64_t* __restrict__ t, int64_t E,
                              int64_t base, int mode, uint64_t* __restrict__ codes, int* __restrict__ bad) {
    const int64_t k = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (k >= E) return;
    uint64_t c = sp.M;
    const int rc = encode_pair(sp, s[k] - base, t[k] - base, &c);
    if (rc == 1 || (rc == 2 && mode == 0)) atomicExch(bad, rc);
    codes[k] = rc == 0 ? c : sp.M;
}

__global__ void decode_kernel(Space sp, const uint64_t* __restrict__ codes, int64_t E, int64_t base,
                              int64_t* __restrict__ s, int64_t* __restrict__ t, int* __restrict__ bad) {
    const int64_t k = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (k >= E) return;
    const uint64_t c = codes[k];
    uint64_t a = 0, b = 0;
    if (c >= sp.M) atomicExch(bad, 1);
    else decode_code(sp, c, &a, &b);
    s[k] = (int64_t)a + base;
    t[k] = (int64_t)b + base;
}

__device__ __forceinline__ bool in_sorted(const uint64_t* __restrict__ set, int64_t x, uint64_t c) {
    int64_t lo = 0, hi = x;  // lower bound of c
    while (lo < hi) {
        const int64_t mid = lo + ((hi - lo) >> 1);
        if (set[mid] < c) lo = mid + 1;
        else hi = mid;
    }
    return lo < x && set[lo] == c;
}

__global__ void member_kernel(const uint64_t* __restrict__ codes, int64_t E, const uint64_t* __restrict__ set,
                              int64_t x, uint8_t* __restrict__ flags) {
    const int64_t k = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (k >= E) return;
    flags[k] = in_sorted(set, x, codes[k]) ? 1 : 0;
}

// excl must be strictly ascending and below M
__global__ void check_set_kernel(const uint64_t* __restrict__ set, int64_t x, uint64_t M, int* __restrict__ bad) {
    const int64_t k = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (k >= x) return;
    if (set[k] >= M || (k > 0 && set[k - 1] >= set[k])) atomicExch(bad, 1);
}

// out[off + pos[i] - 1] = codes[i] for the flagged i with code < bound and rank pos[i] <= limit (pos = inclusive scan
// of the flags): an order-preserving compaction of the first `limit` flagged codes
__global__ void compact_kernel(const uint64_t* __restrict__ codes, const int32_t* __restrict__ flags,
                               const int32_t* __restrict__ pos, int64_t B, uint64_t bound, int64_t limit,
                               uint64_t* __restrict__ out) {
    const int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= B) return;
    if (flags[i] && codes[i] < bound && pos[i] <= limit) out[pos[i] - 1] = codes[i];
}

// ---- the permutation --------------------------------------------------------------------------------------------
struct Feistel {
    int h;          // bits per half
    uint64_t mask;  // 2^h - 1
    uint64_t key[GNNB_FEISTEL_ROUNDS];
};

static Feistel make_feistel(uint64_t M, uint64_t seed) {
    Feistel f;
    f.h = 1;
    while (f.h < 31 && ((uint64_t)1 << (2 * f.h)) < M) ++f.h;
    f.mask = ((uint64_t)1 << f.h) - 1;
    const uint64_t k0 = splitmix64(seed);
    for (int r = 0; r < GNNB_FEISTEL_ROUNDS; ++r) f.key[r] = splitmix64(k0 + (uint64_t)r);
    return f;
}

__host__ __device__ static inline uint64_t feistel(const Feistel& f, uint64_t v) {
    uint64_t L = v >> f.h, R = v & f.mask;
#pragma unroll
    for (int r = 0; r < GNNB_FEISTEL_ROUNDS; ++r) {
        const uint64_t nl = R;
        R = L ^ (splitmix64(R ^ f.key[r]) & f.mask);
        L = nl;
    }
    return (L << f.h) | R;
}

// π(i) for i < M: cycle-walk the network into [0, M)
__host__ __device__ static inline uint64_t permute(const Feistel& f, uint64_t M, uint64_t i) {
    uint64_t v = feistel(f, i);
    while (v >= M) v = feistel(f, v);
    return v;
}

// codes[i] = π(base + i), flags[i] = codes[i] is not excluded
__global__ void perm_batch_kernel(Feistel f, uint64_t M, uint64_t base, int64_t B, const uint64_t* __restrict__ excl,
                                  int64_t x, uint64_t* __restrict__ codes, int32_t* __restrict__ flags) {
    const int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= B) return;
    const uint64_t c = permute(f, M, base + (uint64_t)i);
    codes[i] = c;
    flags[i] = in_sorted(excl, x, c) ? 0 : 1;
}

// largest batch of permuted indices held at once (2 GB of codes + 1 GB of flags and 1 GB of ranks)
constexpr int64_t kMaxBatch = (int64_t)1 << 28;

static int check_edges(int64_t E, int index_base) {
    if (E < 0 || E >= ((int64_t)1 << 31)) GNNB_FAIL(GNNB_ESIZE, "number of edges %lld outside [0, 2^31)", (long long)E);
    if (index_base != 0 && index_base != 1) GNNB_FAIL(GNNB_EINVAL, "index_base must be 0 or 1 (got %d)", index_base);
    return GNNB_OK;
}

static int read_bad(const int* bad_dev, cudaStream_t st, int* bad) {
    GNNB_CUDA(cudaMemcpyAsync(bad, bad_dev, sizeof(int), cudaMemcpyDeviceToHost, st));
    GNNB_CUDA(cudaStreamSynchronize(st));
    return GNNB_OK;
}

}  // namespace gnnb

using namespace gnnb;

extern "C" {

int gnnb_edge_encode(int space, int64_t n1, int64_t n2, const int64_t* s, const int64_t* t, int64_t num_edges,
                     int index_base, uint64_t* codes, void* stream) {
    Space sp;
    GNNB_TRY(make_space(space, n1, n2, &sp));
    GNNB_TRY(check_edges(num_edges, index_base));
    if (num_edges == 0) return GNNB_OK;
    if (!s || !t || !codes) GNNB_FAIL(GNNB_EINVAL, "gnnb_edge_encode: NULL array");
    cudaStream_t st = (cudaStream_t)stream;
    DeviceScratch sc;
    int* bad_dev = nullptr;
    GNNB_TRY(sc.alloc(&bad_dev, 1));
    GNNB_CUDA(cudaMemsetAsync(bad_dev, 0, sizeof(int), st));
    encode_kernel<<<(unsigned)ceil_div(num_edges, 256), 256, 0, st>>>(sp, s, t, num_edges, index_base, 0, codes, bad_dev);
    GNNB_LAUNCHED();
    int bad = 0;
    GNNB_TRY(read_bad(bad_dev, st, &bad));
    if (bad == 1) GNNB_FAIL(GNNB_EINDEX, "edge index outside the %lld x %lld code space", (long long)sp.n1, (long long)sp.n2);
    if (bad == 2) GNNB_FAIL(GNNB_EINDEX, "a self loop has no code in a space without self loops");
    return GNNB_OK;
}

int gnnb_edge_decode(int space, int64_t n1, int64_t n2, const uint64_t* codes, int64_t num_edges, int index_base,
                     int64_t* s, int64_t* t, void* stream) {
    Space sp;
    GNNB_TRY(make_space(space, n1, n2, &sp));
    GNNB_TRY(check_edges(num_edges, index_base));
    if (num_edges == 0) return GNNB_OK;
    if (!s || !t || !codes) GNNB_FAIL(GNNB_EINVAL, "gnnb_edge_decode: NULL array");
    cudaStream_t st = (cudaStream_t)stream;
    DeviceScratch sc;
    int* bad_dev = nullptr;
    GNNB_TRY(sc.alloc(&bad_dev, 1));
    GNNB_CUDA(cudaMemsetAsync(bad_dev, 0, sizeof(int), st));
    decode_kernel<<<(unsigned)ceil_div(num_edges, 256), 256, 0, st>>>(sp, codes, num_edges, index_base, s, t, bad_dev);
    GNNB_LAUNCHED();
    int bad = 0;
    GNNB_TRY(read_bad(bad_dev, st, &bad));
    if (bad) GNNB_FAIL(GNNB_EINDEX, "code outside [0, %llu)", (unsigned long long)sp.M);
    return GNNB_OK;
}

int gnnb_edge_codes_sorted(int space, int64_t n1, int64_t n2, const int64_t* s, const int64_t* t, int64_t num_edges,
                           int index_base, uint64_t* codes_out, int64_t* n_out, void* stream) {
    Space sp;
    GNNB_TRY(make_space(space, n1, n2, &sp));
    GNNB_TRY(check_edges(num_edges, index_base));
    if (!n_out) GNNB_FAIL(GNNB_EINVAL, "gnnb_edge_codes_sorted: n_out is NULL");
    *n_out = 0;
    if (num_edges == 0) return GNNB_OK;
    if (!s || !t || !codes_out) GNNB_FAIL(GNNB_EINVAL, "gnnb_edge_codes_sorted: NULL array");
    cudaStream_t st = (cudaStream_t)stream;
    const int64_t E = num_edges;
    const unsigned blocks = (unsigned)ceil_div(E, 256);
    int end_bit = 1;                     // codes and the sentinel M fit in end_bit bits
    while (end_bit < 64 && (sp.M >> end_bit) != 0) ++end_bit;
    DeviceScratch sc;
    // one allocation for the codes, the sorted codes, the run heads and their ranks
    const size_t nb = (size_t)E;
    void* buf = nullptr;
    GNNB_TRY(sc.alloc(&buf, nb * (8 + 8 + 4 + 4) + 16));
    uint64_t* codes = (uint64_t*)buf;

    uint64_t* sorted = codes + nb;
    int32_t* heads = (int32_t*)(sorted + nb);
    int32_t* pos = heads + nb;
    int* bad_dev = (int*)(pos + nb);
    GNNB_CUDA(cudaMemsetAsync(bad_dev, 0, sizeof(int), st));
    encode_kernel<<<blocks, 256, 0, st>>>(sp, s, t, E, index_base, 1, codes, bad_dev);
    GNNB_LAUNCHED();
    size_t sort_bytes = 0, scan_bytes = 0;
    GNNB_CUDA(cub::DeviceRadixSort::SortKeys(nullptr, sort_bytes, codes, sorted, (int)E, 0, end_bit, st));
    GNNB_CUDA(cub::DeviceScan::InclusiveSum(nullptr, scan_bytes, heads, pos, (int)E, st));
    void* tmp = nullptr;
    GNNB_TRY(sc.alloc(&tmp, std::max(sort_bytes, scan_bytes) + 1));
    GNNB_CUDA(cub::DeviceRadixSort::SortKeys(tmp, sort_bytes, codes, sorted, (int)E, 0, end_bit, st));
    g_launches.fetch_add(2, std::memory_order_relaxed);
    GNNB_TRY(run_head_flags(sorted, E, heads, st));
    GNNB_CUDA(cub::DeviceScan::InclusiveSum(tmp, scan_bytes, heads, pos, (int)E, st));
    g_launches.fetch_add(1, std::memory_order_relaxed);
    compact_kernel<<<blocks, 256, 0, st>>>(sorted, heads, pos, E, sp.M, E, codes_out);  // the sentinel run is skipped
    GNNB_LAUNCHED();
    int bad = 0;
    int32_t runs = 0;
    uint64_t last = 0;
    GNNB_CUDA(cudaMemcpyAsync(&runs, pos + (E - 1), sizeof(int32_t), cudaMemcpyDeviceToHost, st));
    GNNB_CUDA(cudaMemcpyAsync(&last, sorted + (E - 1), sizeof(uint64_t), cudaMemcpyDeviceToHost, st));
    GNNB_TRY(read_bad(bad_dev, st, &bad));
    if (bad) GNNB_FAIL(GNNB_EINDEX, "edge index outside the %lld x %lld code space", (long long)sp.n1, (long long)sp.n2);
    *n_out = (int64_t)runs - (last == sp.M ? 1 : 0);
    return GNNB_OK;
}

int gnnb_codes_member(const uint64_t* codes, int64_t num_codes, const uint64_t* set, int64_t x, uint8_t* flags,
                      void* stream) {
    if (num_codes < 0 || num_codes >= ((int64_t)1 << 31))
        GNNB_FAIL(GNNB_ESIZE, "number of codes %lld outside [0, 2^31)", (long long)num_codes);
    if (x < 0) GNNB_FAIL(GNNB_ESIZE, "set size %lld is negative", (long long)x);
    if (num_codes == 0) return GNNB_OK;
    if (!codes || !flags || (x > 0 && !set)) GNNB_FAIL(GNNB_EINVAL, "gnnb_codes_member: NULL array");
    member_kernel<<<(unsigned)ceil_div(num_codes, 256), 256, 0, (cudaStream_t)stream>>>(codes, num_codes, set, x, flags);
    GNNB_LAUNCHED();
    return GNNB_OK;
}

int gnnb_sample_codes(uint64_t M, const uint64_t* excl, int64_t x, int64_t m, uint64_t seed, uint64_t* out,
                      int64_t* n_out, void* stream) {
    if (!n_out) GNNB_FAIL(GNNB_EINVAL, "gnnb_sample_codes: n_out is NULL");
    *n_out = 0;
    if (M >= ((uint64_t)1 << 62)) GNNB_FAIL(GNNB_ESIZE, "code space of %llu codes: must be below 2^62", (unsigned long long)M);
    if (x < 0 || (uint64_t)x > M) GNNB_FAIL(GNNB_EINVAL, "exclusion set of %lld codes in a space of %llu", (long long)x,
                                            (unsigned long long)M);
    if (m < 0) GNNB_FAIL(GNNB_EINVAL, "m = %lld is negative", (long long)m);
    if (x > 0 && !excl) GNNB_FAIL(GNNB_EINVAL, "gnnb_sample_codes: excl is NULL");
    cudaStream_t st = (cudaStream_t)stream;
    DeviceScratch sc;
    int* bad_dev = nullptr;
    GNNB_TRY(sc.alloc(&bad_dev, 1));
    if (x > 0) {                         // the batch sizes below count on excl being a set of codes < M
        GNNB_CUDA(cudaMemsetAsync(bad_dev, 0, sizeof(int), st));
        check_set_kernel<<<(unsigned)ceil_div(x, 256), 256, 0, st>>>(excl, x, M, bad_dev);
        GNNB_LAUNCHED();
        int bad = 0;
        GNNB_TRY(read_bad(bad_dev, st, &bad));
        if (bad) GNNB_FAIL(GNNB_EINVAL, "excl must be ascending, distinct and below M = %llu", (unsigned long long)M);
    }
    const uint64_t avail = M - (uint64_t)x;
    const int64_t want = (uint64_t)m < avail ? m : (int64_t)avail;
    if (want == 0) return GNNB_OK;
    if (!out) GNNB_FAIL(GNNB_EINVAL, "gnnb_sample_codes: out is NULL");
    const Feistel f = make_feistel(M, seed);
    int64_t written = 0, cap = 0;
    uint64_t base = 0, left = avail;     // left: available codes among the indices not yet permuted
    uint64_t* codes = nullptr;
    int32_t *flags = nullptr, *pos = nullptr;
    void* tmp = nullptr;
    size_t scan_bytes = 0;
    while (written < want) {             // left > 0 here, so base < M: every pass permutes >= 1 new index
        const double need = (double)(want - written);
        const double rest = (double)(M - base);
        // expected survivors of a batch of B: B left / rest; ask for 4 standard deviations and a little more
        const double est = ceil((need + 4.0 * sqrt(need) + 32.0) * rest / (double)left);
        int64_t B = est >= (double)kMaxBatch ? kMaxBatch : (int64_t)est;
        if ((uint64_t)B > M - base) B = (int64_t)(M - base);
        if (cap == 0) {                  // buffers sized by the first batch; later batches reuse them
            cap = B;
            void* buf = nullptr;
            GNNB_TRY(sc.alloc(&buf, (size_t)cap * (8 + 4 + 4)));
            codes = (uint64_t*)buf;
            flags = (int32_t*)(codes + cap);
            pos = flags + cap;
            GNNB_CUDA(cub::DeviceScan::InclusiveSum(nullptr, scan_bytes, flags, pos, (int)cap, st));
            GNNB_TRY(sc.alloc(&tmp, scan_bytes + 1));
        }
        if (B > cap) B = cap;
        const unsigned blocks = (unsigned)ceil_div(B, 256);
        perm_batch_kernel<<<blocks, 256, 0, st>>>(f, M, base, B, excl, x, codes, flags);
        GNNB_LAUNCHED();
        GNNB_CUDA(cub::DeviceScan::InclusiveSum(tmp, scan_bytes, flags, pos, (int)B, st));
        g_launches.fetch_add(1, std::memory_order_relaxed);
        compact_kernel<<<blocks, 256, 0, st>>>(codes, flags, pos, B, M, want - written, out + written);
        GNNB_LAUNCHED();
        int32_t got = 0;
        GNNB_CUDA(cudaMemcpyAsync(&got, pos + (B - 1), sizeof(int32_t), cudaMemcpyDeviceToHost, st));
        GNNB_CUDA(cudaStreamSynchronize(st));
        written += std::min<int64_t>(got, want - written);
        left -= (uint64_t)got;
        base += (uint64_t)B;
    }
    *n_out = written;
    return GNNB_OK;
}

}  // extern "C"
