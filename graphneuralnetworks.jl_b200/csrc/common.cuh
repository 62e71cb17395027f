// common.cuh — shared host/device helpers for libgnnb200 (sm_90a only).
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>
#include <stdio.h>
#include <stdarg.h>
#include <atomic>
#include <mutex>
#include <type_traits>
#include <vector>
#include "../../include/gnnb200.h"

struct cublasLtContext;  // cublasLtHandle_t points to it

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

// ---- device memory ----------------------------------------------------------------------------
// Scoped device temporaries: every buffer alloc() hands out is freed when the scratch goes out of scope, on every return
// path, unless release() has handed it to a longer-lived owner (a plan) first.  Constructed with a stream, it
// synchronises that stream before freeing, so that launches an early error return left queued finish first.
class DeviceScratch {
  public:
    DeviceScratch() = default;
    explicit DeviceScratch(cudaStream_t sync_on_exit) : st_(sync_on_exit), sync_(true) {}
    DeviceScratch(const DeviceScratch&) = delete;
    DeviceScratch& operator=(const DeviceScratch&) = delete;
    ~DeviceScratch() {
        if (sync_) cudaStreamSynchronize(st_);
        for (void* q : bufs_) cudaFree(q);
    }
    // *p = `count` elements of T (bytes for void); the status and error text of GNNB_CUDA when cudaMalloc fails
    template <typename T>
    int alloc(T** p, size_t count) {
        using Elem = typename std::conditional<std::is_void<T>::value, char, T>::type;
        void* q = nullptr;
        *p = nullptr;
        GNNB_CUDA(cudaMalloc(&q, sizeof(Elem) * count));
        bufs_.push_back(q);
        *p = static_cast<T*>(q);
        return GNNB_OK;
    }
    template <typename T>
    T* release(T* p) {
        for (void*& q : bufs_)
            if (q == p) q = nullptr;
        return p;
    }

  private:
    std::vector<void*> bufs_;
    cudaStream_t st_ = nullptr;
    bool sync_ = false;
};

// Grow-only device buffer *p of *cap bytes: reallocated only when `bytes` exceeds *cap, after a device-wide synchronise
// so that no launch still reads the old one.  Once large enough it neither allocates nor synchronises, which keeps a
// warmed-up call legal inside CUDA-graph capture.
template <typename T>
int grow_buffer(T** p, size_t* cap, size_t bytes) {
    if (*cap >= bytes) return GNNB_OK;
    if (*p) {
        cudaDeviceSynchronize();
        cudaFree(*p);
        *p = nullptr;
        *cap = 0;
    }
    GNNB_CUDA(cudaMalloc(p, bytes));
    *cap = bytes;
    return GNNB_OK;
}

// Library-owned state of one device (dense.cu, dense_tc.cu, gatlogit.cu), built on the first call that needs it on that
// device.  Every call on the device shares it, so calls on one device must be stream-ordered with respect to each other.
struct DeviceState {
    int nsm = 0;                      // SMs: the persistent grid of the tensor-core kernels (their attributes are set)
    int* tc_err = nullptr;            // dense_tc.cu's pipeline watchdog: a bounded mbarrier wait expired
    cublasLtContext* lt = nullptr;    // cuBLASLt handle and its workspace (lazily, on the first library GEMM)
    void* lt_ws = nullptr;
    // grow-only scratch (grow_buffer): pointer and bytes
    float* w_blk = nullptr; size_t w_blk_bytes = 0;             // gnnb_linear2_bwd: a 128x128 block of W^T / dW
    float* wt = nullptr; size_t wt_bytes = 0;                   // gnnb_linear_bwd: W^T (<= 128x128) for the wgmma dx
    float* wt_wide = nullptr; size_t wt_wide_bytes = 0;         // gnnb_linear_bwd: W^T for the wide wgmma dx
    float* act_part = nullptr; size_t act_part_bytes = 0;       // act_bwd_kernel: per-block column sums
    float* wimg = nullptr; size_t wimg_bytes = 0;               // the wide kernel's split, swizzled image of W
    float* dw_part = nullptr; size_t dw_part_bytes = 0;         // dw_tf32x3: split-K partials
    float* bwd_part = nullptr; size_t bwd_part_bytes = 0;       // linear_bwd_tf32x3: split-K partials of dW
    float* bwd_colsum = nullptr; size_t bwd_colsum_bytes = 0;   // linear_bwd_tf32x3: column-sum partials of db
    float* gat_part = nullptr; size_t gat_part_bytes = 0;       // gnnb_gat_logit_terms_bwd: per-block partials of da
    char* topk_ws = nullptr; size_t topk_ws_bytes = 0;          // gnnb_topk_keep: segment items, histograms, states
    float* topk_part = nullptr; size_t topk_part_bytes = 0;     // gnnb_topk_gate_bwd: per-block partials of dp
};
// the current device's state, created (tensor-core kernels configured, watchdog flag allocated) on first use
int device_state(DeviceState** out);

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
    int32_t hot_min = 0;      // with es: edges whose gathered node is gathered >= hot_min times carry es's sign bit
    int32_t* hot_rows = nullptr;  // with es: those gathered nodes (unordered), whose rows the propagate demotes after use
    int32_t n_hot = 0;
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
int ensure_csr(gnnb_graph* g, bool transposed, cudaStream_t st);
int ensure_invdeg(gnnb_graph* g, Csr& c, cudaStream_t st);
int ensure_items(gnnb_graph* g, const Csr& c, cudaStream_t st);            // seglean.cu
int ensure_gcn_scale(gnnb_graph* g, bool transposed, cudaStream_t st);     // seglean.cu: g->gcn_c and the Csr's es stream
int gcn_hot_rows(gnnb_graph* g, bool transposed, int32_t* rows_host, int64_t capacity, int64_t* num_rows,
                 int32_t* threshold, cudaStream_t st);                      // seglean.cu: the hot set of es, read back
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
