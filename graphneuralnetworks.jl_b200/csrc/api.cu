// api.cu — C-ABI glue: error state, propagate / pullbacks / GCN core / host-buffer entries / RMAT.
#include "common.cuh"
#include <string.h>
#include <math_constants.h>

namespace gnnb {

static thread_local char t_err[512] = "";
std::atomic<int64_t> g_launches{0};

void set_error(const char* fmt, ...) {
    va_list ap;
    va_start(ap, fmt);
    vsnprintf(t_err, sizeof(t_err), fmt, ap);
    va_end(ap);
}

extern bool g_reference_kernels;   // segreduce.cu
extern bool g_l2_policy_forced;    // seglean.cu
int edge_dot(gnnb_graph* g, const float* dout, const float* x, const float* cs, const float* ct, int64_t D,
             float* dw_coo, cudaStream_t st);
int maxmin_bwd(gnnb_graph* g, const float* w_plan_src, const float* x, const float* dout, const float* out_fwd,
               int64_t D, float* dx, cudaStream_t st);
int maxmin_bwd_halo(gnnb_graph* g, const float* w_plan_dst, const float* x_own, const float* dout_local,
                    const float* dout_halo, const float* out_local, const float* out_halo, int32_t n_local, int64_t D,
                    float* dx, cudaStream_t st);

__global__ void mul_vec_kernel(const float* __restrict__ a, const float* __restrict__ b, int64_t n, float* __restrict__ o) {
    int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i < n) o[i] = a[i] * b[i];
}

// ---- RMAT (Graph500 a,b,c,d = .57,.19,.19,.05), counter-based, integer thresholds ------------------
__global__ void rmat_kernel(int64_t N, int64_t first, int64_t count, uint64_t seed, int scale, int64_t* __restrict__ src,
                            int64_t* __restrict__ dst) {
    const int64_t k = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (k >= count) return;
    const int64_t id = first + k;                    // the edge's global counter: a chunk equals the same slice of the whole list
    const uint32_t TA = 9563013u, TB = 12750684u, TC = 15938355u;  // floor(.57, .76, .95 * 2^24)
    uint64_t s = 0, d = 0;
    for (uint64_t retry = 0;; ++retry) {
        uint64_t state = splitmix64(seed ^ splitmix64((uint64_t)id * 0x100000001B3ull + retry));
        s = 0; d = 0;
        for (int l = 0; l < scale; ++l) {
            state = splitmix64(state);
            const uint32_t u = (uint32_t)(state >> 40);
            const uint64_t sb = (u >= TB) ? 1 : 0;                       // quadrants c,d set the source bit
            const uint64_t db = (u >= TA && u < TB) || (u >= TC) ? 1 : 0;  // quadrants b,d set the target bit
            s = (s << 1) | sb;
            d = (d << 1) | db;
        }
        if ((int64_t)s < N && (int64_t)d < N) break;
        if (retry >= 63) { s %= (uint64_t)N; d %= (uint64_t)N; break; }
    }
    src[k] = (int64_t)s + 1;
    dst[k] = (int64_t)d + 1;
}

}  // namespace gnnb

using namespace gnnb;
static inline unsigned nblk(int64_t n) { return (unsigned)ceil_div(n, 256); }

static int check_common(gnnb_graph_t g, int msg, int aggr, int64_t D, const float* w) {
    if (!g) GNNB_FAIL(GNNB_EINVAL, "graph handle is NULL");
    if (msg != GNNB_COPY_XJ && msg != GNNB_W_MUL_XJ) GNNB_FAIL(GNNB_EINVAL, "unknown message function %d", msg);
    if (aggr < GNNB_SUM || aggr > GNNB_MIN) GNNB_FAIL(GNNB_EINVAL, "unknown aggregation %d", aggr);
    if (D <= 0) GNNB_FAIL(GNNB_ESIZE, "feature dimension must be positive (got %lld)", (long long)D);
    // an edgeless plan's weight vector is empty, and an empty array's pointer may be NULL (torch, CUDA.jl)
    if (msg == GNNB_W_MUL_XJ && !w && g->E > 0) GNNB_FAIL(GNNB_EINVAL, "w_mul_xj/e_mul_xj needs the edge weights");
    return GNNB_OK;
}

// weights in COO order -> plan order of `c` (into ws2); returns nullptr when there are none
static int plan_weights(gnnb_graph* g, const Csr& c, int msg, const float* w, size_t ws2_off_floats, const float** out,
                        cudaStream_t st) {
    *out = nullptr;
    if (msg != GNNB_W_MUL_XJ || !w || g->E == 0) return GNNB_OK;
    GNNB_TRY(grow_buffer(&g->ws2, &g->ws2_bytes, sizeof(float) * ((size_t)g->E + ws2_off_floats)));
    float* p = g->ws2 + ws2_off_floats;
    GNNB_TRY(permute_edge_values(c, g->E, w, 1, p, st));
    *out = p;
    return GNNB_OK;
}

extern "C" {

const char* gnnb_last_error(void) { return t_err; }
const char* gnnb_version(void) { return "gnnb200 0.1 sm_90a"; }
int gnnb_device_count(void) {
    int n = 0;
    if (cudaGetDeviceCount(&n) != cudaSuccess) { cudaGetLastError(); return 0; }
    return n;
}
int64_t gnnb_launch_count(void) { return g_launches.load(); }
int gnnb_set_kernel_variant(int v) {
    if (v != 0 && v != 12 && v != 14)
        GNNB_FAIL(GNNB_EINVAL, "kernel variant must be 0 (default), 12 (reference kernels) or 14 (L2 policy at every size), got %d", v);
    gnnb::g_reference_kernels = v == 12;
    gnnb::g_l2_policy_forced = v == 14;
    return GNNB_OK;
}

int gnnb_propagate(gnnb_graph_t g, int transposed, int msg, int aggr, const float* x, const float* w,
                   const float* cs, const float* ct, int64_t D, float* out, void* stream) {
    GNNB_TRY(check_common(g, msg, aggr, D, w));
    if (!x || !out) GNNB_FAIL(GNNB_EINVAL, "x/out is NULL");
    cudaStream_t st = (cudaStream_t)stream;
    GNNB_TRY(ensure_csr(g, transposed != 0, st));
    const Csr& c = transposed ? g->by_src : g->by_dst;
    SegArgs a;
    a.x = x; a.cs = cs; a.ct = ct; a.out = out; a.D = D; a.aggr = aggr;
    GNNB_TRY(plan_weights(g, c, msg, w, 0, &a.w, st));
    return seg_reduce(g, c, a, st);
}

int gnnb_propagate_bwd(gnnb_graph_t g, int msg, int aggr, const float* dout, const float* x, const float* w,
                       const float* cs, const float* ct, const float* out_fwd, int64_t D, float* dx, float* dw,
                       void* stream) {
    GNNB_TRY(check_common(g, msg, aggr, D, w));
    if (!dout) GNNB_FAIL(GNNB_EINVAL, "dout is NULL");
    cudaStream_t st = (cudaStream_t)stream;
    const bool ismax = aggr == GNNB_MAX || aggr == GNNB_MIN;
    if (ismax) {
        if (dw) GNNB_FAIL(GNNB_EUNSUPPORTED, "dw for max/min aggregation is not implemented");
        if (cs || ct) GNNB_FAIL(GNNB_EUNSUPPORTED, "max/min pullback with node scales is not implemented");
        if (!x || !out_fwd) GNNB_FAIL(GNNB_EINVAL, "max/min pullback needs x and the forward output");
        if (!dx) return GNNB_OK;
        GNNB_TRY(ensure_csr(g, true, st));
        const float* wp = nullptr;
        GNNB_TRY(plan_weights(g, g->by_src, msg, w, 0, &wp, st));
        return maxmin_bwd(g, wp, x, dout, out_fwd, D, dx, st);
    }
    // scale of the gathered dout row: ct (SUM) or ct/deg (MEAN)
    const float* gscale = ct;
    size_t off = 0;
    if (aggr == GNNB_MEAN) {
        GNNB_TRY(ensure_invdeg(g, g->by_dst, st));
        if (ct) {
            GNNB_TRY(grow_buffer(&g->ws2, &g->ws2_bytes, sizeof(float) * ((size_t)g->n_dst + (size_t)g->E)));
            if (g->n_dst > 0) {
                mul_vec_kernel<<<nblk(g->n_dst), 256, 0, st>>>(ct, g->by_dst.invdeg, g->n_dst, g->ws2);
                GNNB_LAUNCHED();
            }
            gscale = g->ws2;
            off = (size_t)g->n_dst;
        } else {
            gscale = g->by_dst.invdeg;
        }
    }
    if (dx) {
        GNNB_TRY(ensure_csr(g, true, st));
        SegArgs a;
        a.x = dout; a.cs = gscale; a.ct = cs; a.out = dx; a.D = D; a.aggr = GNNB_SUM;
        GNNB_TRY(plan_weights(g, g->by_src, msg, w, off, &a.w, st));
        GNNB_TRY(seg_reduce(g, g->by_src, a, st));
    }
    if (dw) {
        if (msg != GNNB_W_MUL_XJ) GNNB_FAIL(GNNB_EINVAL, "dw requested for a message without weights");
        if (!x) GNNB_FAIL(GNNB_EINVAL, "dw needs x");
        GNNB_TRY(edge_dot(g, dout, x, cs, gscale, D, dw, st));
    }
    return GNNB_OK;
}

int gnnb_gcn_propagate(gnnb_graph_t g, int transposed, const float* x, const float* w, const float* c,
                       int64_t D, float* out, void* stream) {
    if (!g) GNNB_FAIL(GNNB_EINVAL, "graph handle is NULL");
    if (g->n_src != g->n_dst) GNNB_FAIL(GNNB_ESIZE, "gcn_propagate needs num_src == num_dst");
    if (!c) {
        // the plan's own default normalisation c = 1/sqrt(in-degree) (unweighted): plan-owned, immutable, and with it the
        // per-edge stream es[e] = c[col[e]] that spares the kernel a dependent 4 B gather per edge
        if (w) GNNB_FAIL(GNNB_EINVAL, "c is NULL: the plan-owned normalisation exists for unweighted graphs only");
        if (!x || !out) GNNB_FAIL(GNNB_EINVAL, "x/out is NULL");
        if (D <= 0) GNNB_FAIL(GNNB_ESIZE, "feature dimension must be positive (got %lld)", (long long)D);
        cudaStream_t st = (cudaStream_t)stream;
        GNNB_TRY(ensure_csr(g, transposed != 0, st));
        GNNB_TRY(ensure_gcn_scale(g, transposed != 0, st));
        const Csr& cc = transposed ? g->by_src : g->by_dst;
        SegArgs a;
        a.x = x; a.cs = g->gcn_c; a.es = cc.es; a.ct = g->gcn_c; a.out = out; a.D = D; a.aggr = GNNB_SUM;
        return seg_reduce(g, cc, a, st);
    }
    return gnnb_propagate(g, transposed, w ? GNNB_W_MUL_XJ : GNNB_COPY_XJ, GNNB_SUM, x, w, c, c, D, out, stream);
}

int gnnb_gcn_hot_rows(gnnb_graph_t g, int transposed, int32_t* rows_host, int64_t capacity, int64_t* num_rows,
                      int32_t* threshold, void* stream) {
    if (!g) GNNB_FAIL(GNNB_EINVAL, "graph handle is NULL");
    if (g->n_src != g->n_dst) GNNB_FAIL(GNNB_ESIZE, "gcn_hot_rows needs num_src == num_dst");
    if (capacity < 0) GNNB_FAIL(GNNB_ESIZE, "capacity must be >= 0");
    return gcn_hot_rows(g, transposed != 0, rows_host, capacity, num_rows, threshold, (cudaStream_t)stream);
}

int gnnb_gcn_propagate_bipartite(gnnb_graph_t g, int transposed, const float* x, int64_t D, float* out, void* stream) {
    if (!g) GNNB_FAIL(GNNB_EINVAL, "graph handle is NULL");
    if (!x || !out) GNNB_FAIL(GNNB_EINVAL, "x/out is NULL");
    if (D <= 0) GNNB_FAIL(GNNB_ESIZE, "feature dimension must be positive (got %lld)", (long long)D);
    cudaStream_t st = (cudaStream_t)stream;
    GNNB_TRY(ensure_csr(g, transposed != 0, st));
    GNNB_TRY(ensure_bipartite_gcn_scale(g, transposed != 0, st));
    const Csr& cc = transposed ? g->by_src : g->by_dst;
    SegArgs a;
    // forward: gathered sources scaled by c_src (as the per-edge stream), target rows by c_dst; the pullback swaps them
    a.x = x; a.out = out; a.D = D; a.aggr = GNNB_SUM;
    a.cs = transposed ? g->bip_c_dst : g->bip_c_src;
    a.es = transposed ? g->bip_es_src : g->bip_es_dst;
    a.ct = transposed ? g->bip_c_src : g->bip_c_dst;
    return seg_reduce(g, cc, a, st);
}

// ---- node-partitioned shards ---------------------------------------------------------------------
int gnnb_propagate_halo(gnnb_graph_t g, int msg, int aggr, const float* x_local, const float* x_halo,
                        int64_t n_local, const float* w, const float* cs, const float* ct, int64_t D, float* out,
                        void* stream) {
    GNNB_TRY(check_common(g, msg, aggr, D, w));
    if (n_local < 0 || n_local > g->n_src) GNNB_FAIL(GNNB_ESIZE, "n_local must be in [0, num_src]");
    if (g->n_dst == 0) return GNNB_OK;   // a rank that owns no node: no row to reduce, out may be NULL
    if (!out) GNNB_FAIL(GNNB_EINVAL, "out is NULL");
    if (n_local > 0 && !x_local) GNNB_FAIL(GNNB_EINVAL, "x_local is NULL");
    if (n_local < g->n_src && !x_halo) GNNB_FAIL(GNNB_EINVAL, "x_halo is NULL but the shard has halo sources");
    cudaStream_t st = (cudaStream_t)stream;
    GNNB_TRY(ensure_csr(g, false, st));
    const Csr& c = g->by_dst;
    SegArgs a;
    a.x = x_local; a.x2 = x_halo; a.split = (int32_t)n_local;
    if (!x_local) { a.x = x_halo; a.x2 = nullptr; }   // no local rows at all
    a.cs = cs; a.ct = ct; a.out = out; a.D = D; a.aggr = aggr;
    GNNB_TRY(plan_weights(g, c, msg, w, 0, &a.w, st));
    return seg_reduce(g, c, a, st);
}

int gnnb_propagate_maxmin_bwd_halo(gnnb_graph_t g, int msg, int aggr, const float* x_own, const float* dout_local,
                                   const float* dout_halo, const float* out_local, const float* out_halo, int64_t n_local,
                                   const float* w, int64_t D, float* dx, void* stream) {
    GNNB_TRY(check_common(g, msg, aggr, D, w));
    if (aggr != GNNB_MAX && aggr != GNNB_MIN)
        GNNB_FAIL(GNNB_EINVAL, "maxmin_bwd_halo serves max and min (sum and mean pull back through gnnb_propagate_halo)");
    if (n_local < 0 || n_local > g->n_src) GNNB_FAIL(GNNB_ESIZE, "n_local must be in [0, num_src]");
    if (g->n_dst == 0) return GNNB_OK;   // a rank that owns no node: no source row to write, dx may be NULL
    if (!x_own || !dx) GNNB_FAIL(GNNB_EINVAL, "x_own/dx is NULL");
    if (n_local > 0 && (!dout_local || !out_local)) GNNB_FAIL(GNNB_EINVAL, "dout_local/out_local is NULL");
    if (n_local < g->n_src && (!dout_halo || !out_halo))
        GNNB_FAIL(GNNB_EINVAL, "dout_halo/out_halo is NULL but the shard has halo targets");
    cudaStream_t st = (cudaStream_t)stream;
    GNNB_TRY(ensure_csr(g, false, st));
    const float* wp = nullptr;
    GNNB_TRY(plan_weights(g, g->by_dst, msg, w, 0, &wp, st));
    return maxmin_bwd_halo(g, wp, x_own, dout_local, dout_halo, out_local, out_halo, (int32_t)n_local, D, dx, st);
}

// ---- host-buffer entries ------------------------------------------------------------------------
// The streams and events of one *_host call, destroyed on every return path.  A return before `finished` is set (an
// error) first waits for the device, so that no copy into the caller's host buffers is still in flight.
struct HostCall {
    cudaStream_t st[3] = {nullptr, nullptr, nullptr};
    cudaEvent_t ev[4] = {nullptr, nullptr, nullptr, nullptr};
    bool finished = false;
    HostCall() = default;
    HostCall(const HostCall&) = delete;
    HostCall& operator=(const HostCall&) = delete;
    ~HostCall() {
        if (!finished) cudaDeviceSynchronize();
        for (cudaEvent_t e : ev)
            if (e) cudaEventDestroy(e);
        for (cudaStream_t q : st)
            if (q) cudaStreamDestroy(q);
    }
};

static int host_pass(gnnb_graph_t g, int transposed, int msg, int aggr, int gcn, const float* x_host,
                     const float* w_host, int64_t D, float* out_host) {
    if (!g) GNNB_FAIL(GNNB_EINVAL, "graph handle is NULL");
    if (!x_host || !out_host) GNNB_FAIL(GNNB_EINVAL, "host buffer is NULL");
    if (D <= 0) GNNB_FAIL(GNNB_ESIZE, "feature dimension must be positive");
    const int64_t n_in = transposed ? g->n_dst : g->n_src, n_out = transposed ? g->n_src : g->n_dst;
    DeviceScratch sc;
    HostCall hc;
    GNNB_CUDA(cudaStreamCreateWithFlags(&hc.st[0], cudaStreamNonBlocking));
    cudaStream_t st = hc.st[0];
    float *dx = nullptr, *dout = nullptr, *dw = nullptr, *dc = nullptr;
    GNNB_TRY(sc.alloc(&dx, (size_t)(n_in * D > 0 ? n_in * D : 1)));
    GNNB_TRY(sc.alloc(&dout, (size_t)(n_out * D > 0 ? n_out * D : 1)));
    GNNB_CUDA(cudaMemcpyAsync(dx, x_host, sizeof(float) * (size_t)(n_in * D), cudaMemcpyHostToDevice, st));
    if (w_host && g->E > 0) {
        GNNB_TRY(sc.alloc(&dw, (size_t)g->E));
        GNNB_CUDA(cudaMemcpyAsync(dw, w_host, sizeof(float) * (size_t)g->E, cudaMemcpyHostToDevice, st));
    }
    if (gcn) {
        GNNB_TRY(sc.alloc(&dc, (size_t)(g->n_dst > 0 ? g->n_dst : 1)));
        GNNB_TRY(gnnb_gcn_norm(g, dw, dc, st));
        GNNB_TRY(gnnb_gcn_propagate(g, transposed, dx, dw, dc, D, dout, st));
    } else {
        GNNB_TRY(gnnb_propagate(g, transposed, msg, aggr, dx, dw, nullptr, nullptr, D, dout, st));
    }
    GNNB_CUDA(cudaMemcpyAsync(out_host, dout, sizeof(float) * (size_t)(n_out * D), cudaMemcpyDeviceToHost, st));
    GNNB_CUDA(cudaStreamSynchronize(st));
    hc.finished = true;
    return GNNB_OK;
}

int gnnb_propagate_host(gnnb_graph_t g, int transposed, int msg, int aggr, const float* x_host,
                        const float* w_host, int64_t D, float* out_host) {
    GNNB_TRY(check_common(g, msg, aggr, D, w_host));
    return host_pass(g, transposed, msg, aggr, 0, x_host, w_host, D, out_host);
}
int gnnb_gcn_propagate_host(gnnb_graph_t g, int transposed, const float* x_host, const float* w_host,
                            int64_t D, float* out_host) {
    return host_pass(g, transposed, GNNB_COPY_XJ, GNNB_SUM, 1, x_host, w_host, D, out_host);
}

// ---- one GCNConv forward + backward on host arrays ----------------------------------------------------------------
int gnnb_gcn_conv_step_host(gnnb_graph_t g, const float* x_host, const float* W_host, const float* b_host, int relu,
                            int64_t Din, int64_t Dout, const float* dy_host, float* y_host, float* dx_host,
                            float* dW_host, float* db_host) {
    if (!g) GNNB_FAIL(GNNB_EINVAL, "graph handle is NULL");
    if (g->n_src != g->n_dst) GNNB_FAIL(GNNB_ESIZE, "gcn_conv needs num_src == num_dst");
    if (Din <= 0 || Dout <= 0) GNNB_FAIL(GNNB_ESIZE, "feature dimensions must be positive");
    if (!x_host || !W_host || !y_host) GNNB_FAIL(GNNB_EINVAL, "host buffer is NULL");
    const bool bwd = dy_host != nullptr;
    if (bwd && (!dx_host || !dW_host)) GNNB_FAIL(GNNB_EINVAL, "the backward half needs dx_host and dW_host");
    const int64_t N = g->n_dst;
    if (Dout < Din)                                        // conv.jl:36-40 multiplies before the convolution then
        GNNB_FAIL(GNNB_EUNSUPPORTED, "gcn_conv_step_host serves the Dout >= Din branch (propagate, then GEMM with bias/activation)");
    const int64_t Dp = Din;                                // width at which the graph is traversed
    // device staging, carved from one plan-owned allocation: x, p (propagated / pre-propagated), y, dy, dpre, dp, dx, W, b, dW, db
    const size_t nx = (size_t)N * Din, np_ = (size_t)N * Dp, ny = (size_t)N * Dout;
    const size_t words = nx + np_ + ny + (bwd ? (ny + ny + np_ + nx + (size_t)N * 4) : 0) + 2 * (size_t)(Dout * Din) + 2 * (size_t)Dout + 64;
    GNNB_TRY(grow_buffer(&g->host_ws, &g->host_ws_bytes, words * sizeof(float)));
    float* q = (float*)g->host_ws;
    auto take = [&](size_t n) { float* r = q; q += (n + 3) & ~(size_t)3; return r; };
    float *x = take(nx), *p = take(np_), *y = take(ny);
    float *dy = bwd ? take(ny) : nullptr, *dpre = bwd ? take(ny) : nullptr, *dp = bwd ? take(np_) : nullptr, *dx = bwd ? take(nx) : nullptr;
    float *W = take((size_t)(Dout * Din)), *b = take((size_t)Dout), *dW = take((size_t)(Dout * Din)), *db = take((size_t)Dout);
    // the relu mask of y (N x 4 words, 16 B aligned like every carve): the pullback reads it instead of y where it can
    uint32_t* mask = bwd ? reinterpret_cast<uint32_t*>(take((size_t)N * 4)) : nullptr;
    bool masked = false;
    HostCall hc;
    for (cudaStream_t& q : hc.st) GNNB_CUDA(cudaStreamCreateWithFlags(&q, cudaStreamNonBlocking));
    for (cudaEvent_t& e : hc.ev) GNNB_CUDA(cudaEventCreateWithFlags(&e, cudaEventDisableTiming));
    cudaStream_t s_main = hc.st[0], s_in = hc.st[1], s_out = hc.st[2];
    cudaEvent_t ev_x = hc.ev[0], ev_dy = hc.ev[1], ev_y = hc.ev[2], ev_dx = hc.ev[3];
    // uploads ride s_in, downloads s_out (PCIe is full duplex), kernels s_main
    GNNB_CUDA(cudaMemcpyAsync(W, W_host, sizeof(float) * (size_t)(Dout * Din), cudaMemcpyHostToDevice, s_in));
    if (b_host) GNNB_CUDA(cudaMemcpyAsync(b, b_host, sizeof(float) * (size_t)Dout, cudaMemcpyHostToDevice, s_in));
    GNNB_CUDA(cudaMemcpyAsync(x, x_host, sizeof(float) * nx, cudaMemcpyHostToDevice, s_in));
    GNNB_CUDA(cudaEventRecord(ev_x, s_in));
    if (bwd) {
        GNNB_CUDA(cudaMemcpyAsync(dy, dy_host, sizeof(float) * ny, cudaMemcpyHostToDevice, s_in));
        GNNB_CUDA(cudaEventRecord(ev_dy, s_in));
    }
    GNNB_CUDA(cudaStreamWaitEvent(s_main, ev_x, 0));
    GNNB_TRY(gnnb_gcn_propagate(g, 0, x, nullptr, nullptr, Dp, p, s_main));                     // p = Â x
    if (bwd && relu && Dout == 128) {                                                     // y = relu(W p + b) + mask
        const int rc = gnnb_linear_relu_mask(p, W, b_host ? b : nullptr, N, Din, Dout, y, mask, s_main);
        if (rc != GNNB_OK && rc != GNNB_EUNSUPPORTED) return rc;
        masked = rc == GNNB_OK;
    }
    if (!masked) GNNB_TRY(gnnb_linear(p, W, b_host ? b : nullptr, relu, N, Din, Dout, y, s_main));  // y = act(W p + b)
    GNNB_CUDA(cudaEventRecord(ev_y, s_main));
    GNNB_CUDA(cudaStreamWaitEvent(s_out, ev_y, 0));
    GNNB_CUDA(cudaMemcpyAsync(y_host, y, sizeof(float) * ny, cudaMemcpyDeviceToHost, s_out));
    if (bwd) {
        GNNB_CUDA(cudaStreamWaitEvent(s_main, ev_dy, 0));
        if (masked) {
            GNNB_TRY(gnnb_linear_bwd_mask(dy, mask, p, W, N, Din, Dout, dp, dW, (b_host && db_host) ? db : nullptr, s_main));
        } else {
            GNNB_TRY(gnnb_linear_bwd(dy, y, p, W, relu, N, Din, Dout, dpre, dp, dW, (b_host && db_host) ? db : nullptr, s_main));
        }
        GNNB_TRY(gnnb_gcn_propagate(g, 1, dp, nullptr, nullptr, Dp, dx, s_main));               // dx = Â' dp
        GNNB_CUDA(cudaEventRecord(ev_dx, s_main));
        GNNB_CUDA(cudaStreamWaitEvent(s_out, ev_dx, 0));
        GNNB_CUDA(cudaMemcpyAsync(dx_host, dx, sizeof(float) * nx, cudaMemcpyDeviceToHost, s_out));
        GNNB_CUDA(cudaMemcpyAsync(dW_host, dW, sizeof(float) * (size_t)(Dout * Din), cudaMemcpyDeviceToHost, s_out));
        if (b_host && db_host) GNNB_CUDA(cudaMemcpyAsync(db_host, db, sizeof(float) * (size_t)Dout, cudaMemcpyDeviceToHost, s_out));
    }
    GNNB_CUDA(cudaStreamSynchronize(s_out));
    GNNB_CUDA(cudaStreamSynchronize(s_main));
    hc.finished = true;
    return GNNB_OK;
}

int gnnb_rmat_edges_range(int64_t num_nodes, int64_t first_edge, int64_t count, uint64_t seed, int64_t* src_dev,
                          int64_t* dst_dev, void* stream) {
    if (num_nodes <= 0 || count < 0 || first_edge < 0) GNNB_FAIL(GNNB_ESIZE, "rmat: bad sizes");
    if (count > 0 && (!src_dev || !dst_dev)) GNNB_FAIL(GNNB_EINVAL, "rmat: NULL output");
    if (gnnb_device_count() <= 0) GNNB_FAIL(GNNB_ECUDA, "no CUDA device");
    int scale = 0;
    while (((int64_t)1 << scale) < num_nodes) ++scale;
    if (count == 0) return GNNB_OK;
    rmat_kernel<<<nblk(count), 256, 0, (cudaStream_t)stream>>>(num_nodes, first_edge, count, seed, scale, src_dev, dst_dev);
    GNNB_LAUNCHED();
    return GNNB_OK;
}
int gnnb_rmat_edges(int64_t num_nodes, int64_t num_edges, uint64_t seed, int64_t* src_dev, int64_t* dst_dev,
                    void* stream) {
    return gnnb_rmat_edges_range(num_nodes, 0, num_edges, seed, src_dev, dst_dev, stream);
}

}  // extern "C"
