// common.cuh — shared host/device helpers for libgnnb200 (sm_90a only).
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>
#include <stdio.h>
#include <stdarg.h>
#include <atomic>
#include <mutex>
#include "../../include/gnnb200.h"

namespace gnnb {

// ---- error plumbing -------------------------------------------------------------------------
void set_error(const char* fmt, ...);
extern std::atomic<int64_t> g_launches;

#define GNNB_CUDA(expr)                                                                   \
    do {                                                                                  \
        cudaError_t _e = (expr);                                                          \
        if (_e != cudaSuccess) {                                                          \
            ::gnnb::set_error("%s failed: %s (%s:%d)", #expr, cudaGetErrorString(_e),     \
                              __FILE__, __LINE__);                                        \
            return (_e == cudaErrorMemoryAllocation) ? GNNB_ENOMEM : GNNB_ECUDA;          \
        }                                                                                 \
    } while (0)

#define GNNB_TRY(expr)                 \
    do {                               \
        int _s = (expr);               \
        if (_s != GNNB_OK) return _s;  \
    } while (0)

#define GNNB_FAIL(code, ...)             \
    do {                                 \
        ::gnnb::set_error(__VA_ARGS__);  \
        return (code);                   \
    } while (0)

// count a launch and check it
#define GNNB_LAUNCHED()                                         \
    do {                                                        \
        ::gnnb::g_launches.fetch_add(1, std::memory_order_relaxed); \
        GNNB_CUDA(cudaGetLastError());                          \
    } while (0)

static inline int64_t ceil_div(int64_t a, int64_t b) { return (a + b - 1) / b; }

// splitmix64's output function: the mixer of every counter-based random stream in the library (RMAT, neighbour
// sampling, the edge-code permutation)
__host__ __device__ static inline uint64_t splitmix64(uint64_t x) {
    x += 0x9E3779B97F4A7C15ull;
    x = (x ^ (x >> 30)) * 0xBF58476D1CE4E5B9ull;
    x = (x ^ (x >> 27)) * 0x94D049BB133111EBull;
    return x ^ (x >> 31);
}

// SMs of the H100 SXM: the block-count caps of the grid-stride and two-stage reduction kernels are multiples of it
constexpr int kNumSMs = 132;

// ---- one direction of a plan: CSR over `nrows` reduction rows ---------------------------------
struct Csr {
    int32_t* rowptr = nullptr;  // [nrows+1]
    int32_t* col = nullptr;     // [E] gathered node of each sorted edge
    int32_t* row = nullptr;     // [E] reduction row of each sorted edge (sorted, non-decreasing)
    int32_t* eid = nullptr;     // [E] COO position of each sorted edge (stable)
    int32_t* long_rows = nullptr;  // rows with more than `chunk` edges (unordered)
    int32_t n_long = 0;
    int32_t nrows = 0;  // reduction rows (targets; sources when transposed)
    float* invdeg = nullptr;  // lazily: 1/max(deg,1) per row (for MEAN)
    // lazily (seglean.cu): the chunk decomposition as a compact list of work items {e_begin, e_end, slot, 0}: slot < 0 = whole
    // rows (stored at every row end), slot >= 0 = one piece of a long row (raw partial into workspace slot `slot`)
    int32_t* items = nullptr;
    int32_t n_items = 0;
    int32_t n_empty = -1;     // rows without edges (-1 = not counted yet)
    float* es = nullptr;      // lazily: es[e] = node_scale[col[e]] in plan order (the plan-owned GCN normalisation)
    bool built = false;
};

#ifdef __CUDACC__
// max(a, b) that returns NaN when either operand is NaN (max.NaN.f32): Julia's `max`, which NNlib's scatter(max) and
// relu fold with.  fmaxf returns the other operand instead.  Same bits as fmaxf whenever neither operand is NaN.
__device__ __forceinline__ float fmax_nan(float a, float b) {
    float d;
    asm("max.NaN.f32 %0, %1, %2;" : "=f"(d) : "f"(a), "f"(b));
    return d;
}
// the shift of an online softmax step whose new running max is Mn: Mn itself, or 0 while every logit seen so far is
// -Inf, so that exp(M - shift) and exp(u - shift) give 0 there instead of exp(-Inf + Inf) = NaN
__device__ __forceinline__ float softmax_shift(float Mn) { return Mn == -__int_as_float(0x7f800000) ? 0.f : Mn; }
#endif

}  // namespace gnnb

struct gnnb_graph {
    int64_t E = 0;
    int32_t n_src = 0, n_dst = 0;
    int32_t chunk = 128;     // edges per work chunk (segmented reduce)
    int device = 0;
    int32_t* coo_src = nullptr;  // [E] 0-based
    int32_t* coo_dst = nullptr;  // [E]
    gnnb::Csr by_dst;            // forward plan (reduce over in-edges of each target)
    gnnb::Csr by_src;            // transposed plan (reduce over out-edges of each source)
    // per-plan workspace for long-row partials and permuted edge values (grown on demand)
    float* ws = nullptr;
    size_t ws_bytes = 0;
    float* ws2 = nullptr;
    size_t ws2_bytes = 0;
    float* gcn_c = nullptr;      // lazily: 1/sqrt(in-degree), the default symmetric normalisation (unweighted), plan-owned
    // lazily: the two-sided (heterograph) GCN normalisation, kept apart from gcn_c / Csr::es so a square plan can serve both
    float* bip_c_src = nullptr;  // [n_src] 1/sqrt(out-degree)
    float* bip_c_dst = nullptr;  // [n_dst] 1/sqrt(in-degree)
    float* bip_es_dst = nullptr; // [E] bip_c_src[col[e]] in by_dst plan order (forward)
    float* bip_es_src = nullptr; // [E] bip_c_dst[col[e]] in by_src plan order (pullback)
    void* host_ws = nullptr;     // device staging of the *_host entries (grown on demand, freed with the plan)
    size_t host_ws_bytes = 0;
    std::mutex mu;
};

namespace gnnb {
int ensure_ws(gnnb_graph* g, size_t bytes);
int ensure_ws2(gnnb_graph* g, size_t bytes);
int ensure_csr(gnnb_graph* g, bool transposed, cudaStream_t st);
int ensure_invdeg(gnnb_graph* g, Csr& c, cudaStream_t st);
int ensure_items(gnnb_graph* g, const Csr& c, cudaStream_t st);            // seglean.cu
int ensure_gcn_scale(gnnb_graph* g, bool transposed, cudaStream_t st);     // seglean.cu: g->gcn_c and the Csr's es stream
int ensure_bipartite_gcn_scale(gnnb_graph* g, bool transposed, cudaStream_t st);   // seglean.cu: g->bip_* for one direction
int rsqrt_exact(float* d, int64_t n, cudaStream_t st);                     // edgeops.cu: d = 1/sqrt(d) in place
// transform.cu: flags[k] = 1 where sorted key k starts a run of equal keys (k == 0 or keys[k] != keys[k-1])
int run_head_flags(const uint64_t* keys, int64_t E, int32_t* flags, cudaStream_t st);

// segreduce.cu
struct SegArgs {
    const float* x = nullptr;   // gathered rows, [gathered nodes][D]
    const float* x2 = nullptr;  // optional second base for gathered nodes >= split (halo rows)
    int32_t split = 0;
    const float* w = nullptr;   // per-edge weight in PLAN order or nullptr
    const float* cs = nullptr;  // per gathered-node scale or nullptr
    const float* es = nullptr;  // the same scale already gathered per edge (plan order): es[e] == cs[col[e]]; needs cs too
    const float* ct = nullptr;  // per output-row scale or nullptr
    float* out = nullptr;       // [nrows][D]
    int64_t D = 0;
    int aggr = GNNB_SUM;
};
int seg_reduce(gnnb_graph* g, const Csr& c, const SegArgs& a, cudaStream_t st);
// permute K floats per edge COO order -> plan order of `c`
int permute_edge_values(const Csr& c, int64_t E, const float* coo_vals, int64_t K, float* plan_vals,
                        cudaStream_t st);
int unpermute_edge_values(const Csr& c, int64_t E, const float* plan_vals, int64_t K,
                          float* coo_vals, cudaStream_t st);
}  // namespace gnnb
