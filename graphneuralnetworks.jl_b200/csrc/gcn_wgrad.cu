// gcn_wgrad.cu — the edge-weight gradient of the weighted GCN propagate on a shard's forward plan.
//
// The layer computes y_t = c_t Σ_{e: s→t} w_e c_s h_s with c = d^{-1/2}, d_t = Σ_{e→t} w_e.  Its gradient with respect to
// the weight of edge e = (s → t) is
//     dw_e = <c_t dy_t, c_s h_s> + dd_t,
// where dd_t = -½ d_t^{-3/2} dc_t is the degree term the caller forms from node-sized dots.  One warp walks one work item
// of the plan's target CSR (seglean.cu's items: a run of whole rows or one piece of a long row) and writes every edge's
// value once, at its COO position: no atomics, so the result is the same bits run after run.  The gathered source row
// comes from the local base or the halo base (ids >= split), as in seg_lean_kernel's HALO instance.  The products are
// rounded as the single-GPU composition rounds them, (dy * c_t) * (h * c_s) per element, so that an infinite scale (a
// weighted in-degree of 0) gives the same Inf and NaN entries.  No reference counterpart: the reference differentiates
// the composition of degree, scaling and propagate (GNNlib/src/layers/conv.jl:14-72).
#include "common.cuh"

namespace gnnb {

struct EwGradParams {
    const int4* __restrict__ items;
    const int32_t* __restrict__ col;     // gathered node of each edge ([local | halo] index space)
    const int32_t* __restrict__ row;
    const int32_t* __restrict__ eid;
    const float* __restrict__ dout;      // [num_dst][D]
    const float* __restrict__ x;         // gathered rows < split
    const float* __restrict__ x2;        // gathered rows >= split (halo rows), or nullptr
    const float* __restrict__ cs;        // per gathered-node scale or nullptr
    const float* __restrict__ ct;        // per target scale or nullptr
    const float* __restrict__ dd;        // per target additive term or nullptr
    float* __restrict__ dw;              // [E], COO order
    int64_t D;
    int32_t n_items;
    int32_t split;
};

namespace {

// the index words and per-node terms of the 32 edges starting at e0, one edge per lane
struct EdgeWords {
    int c = 0, r = 0, id = 0;
    float s = 1.f, t = 1.f, a = 0.f;
};
__device__ __forceinline__ EdgeWords load_words(const EwGradParams& p, int my, int e_end) {
    EdgeWords w;
    if (my < e_end) {
        w.c = __ldg(p.col + my);
        w.r = __ldg(p.row + my);
        w.id = __ldg(p.eid + my);
        if (p.cs) w.s = __ldg(p.cs + w.c);
        if (p.ct) w.t = __ldg(p.ct + w.r);
        if (p.dd) w.a = __ldg(p.dd + w.r);
    }
    return w;
}

__device__ __forceinline__ float warp_sum(float v) {
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
    return v;   // the same bits in every lane: each step adds the same two operands, in either order
}

__device__ __forceinline__ float dot4(float acc, float4 g, float4 h, float t, float s) {
    acc = __fmaf_rn(__fmul_rn(g.x, t), __fmul_rn(h.x, s), acc);
    acc = __fmaf_rn(__fmul_rn(g.y, t), __fmul_rn(h.y, s), acc);
    acc = __fmaf_rn(__fmul_rn(g.z, t), __fmul_rn(h.z, s), acc);
    return __fmaf_rn(__fmul_rn(g.w, t), __fmul_rn(h.w, s), acc);
}

// rows of KV*128 floats, 16 B-aligned: lane l holds floats [4l, 4l+4) of every 128-float slice.  U edges in flight, each
// with its gathered row and its target's dout row (an L1 hit after the first edge of the row), so that no load waits on a
// row change.  Every branch that guards a shuffle is warp-uniform.
template <int KV, int HALO>
__global__ void __launch_bounds__(256, 3) gcn_ew_grad_kernel(const EwGradParams p) {
    constexpr unsigned FULL = 0xffffffffu;
    constexpr int U = 4 / KV > 0 ? 4 / KV : 1;   // edges in flight: two rows each
    constexpr int64_t STRIDE = (int64_t)KV * 128;
    const int lane = threadIdx.x & 31;
    const int item = blockIdx.x * 8 + (threadIdx.x >> 5);
    if (item >= p.n_items) return;
    const int4 it = __ldg(p.items + item);
    const int e_end = it.y;
    const float* const xl = p.x + lane * 4;
    const float* const x2l = HALO ? p.x2 + lane * 4 - (int64_t)p.split * STRIDE : nullptr;
    const float* const gl = p.dout + lane * 4;
    for (int e0 = it.x; e0 < e_end; e0 += 32) {
        const EdgeWords w = load_words(p, e0 + lane, e_end);
        const int n = e_end - e0 < 32 ? e_end - e0 : 32;
#pragma unroll 1
        for (int j0 = 0; j0 < n; j0 += U) {
            float4 v[U][KV], g[U][KV];
#pragma unroll
            for (int u = 0; u < U; ++u) {
                const int cj = __shfl_sync(FULL, w.c, j0 + u);
                const int rj = __shfl_sync(FULL, w.r, j0 + u);
                if (j0 + u < n) {
                    const float* xr = (HALO && cj >= p.split ? x2l : xl) + (int64_t)cj * STRIDE;
                    const float* gr = gl + (int64_t)rj * STRIDE;
#pragma unroll
                    for (int i = 0; i < KV; ++i) {
                        v[u][i] = __ldg(reinterpret_cast<const float4*>(xr + i * 128));
                        g[u][i] = __ldg(reinterpret_cast<const float4*>(gr + i * 128));
                    }
                }
            }
#pragma unroll
            for (int u = 0; u < U; ++u) {
                const float sj = __shfl_sync(FULL, w.s, j0 + u);
                const float tj = __shfl_sync(FULL, w.t, j0 + u);
                if (j0 + u < n) {
                    float acc = 0.f;
#pragma unroll
                    for (int i = 0; i < KV; ++i) acc = dot4(acc, g[u][i], v[u][i], tj, sj);
                    acc = warp_sum(acc);
                    if (lane == j0 + u) p.dw[w.id] = __fadd_rn(acc, w.a);
                }
            }
        }
    }
}

// any width and alignment: the lanes stride over the features of one edge at a time
template <int HALO>
__global__ void __launch_bounds__(256) gcn_ew_grad_generic_kernel(const EwGradParams p) {
    constexpr unsigned FULL = 0xffffffffu;
    const int lane = threadIdx.x & 31;
    const int item = blockIdx.x * 8 + (threadIdx.x >> 5);
    if (item >= p.n_items) return;
    const int4 it = __ldg(p.items + item);
    const int e_end = it.y;
    const int64_t D = p.D;
    for (int e0 = it.x; e0 < e_end; e0 += 32) {
        const EdgeWords w = load_words(p, e0 + lane, e_end);
        const int n = e_end - e0 < 32 ? e_end - e0 : 32;
#pragma unroll 1
        for (int j = 0; j < n; ++j) {
            const int cj = __shfl_sync(FULL, w.c, j);
            const int rj = __shfl_sync(FULL, w.r, j);
            const float sj = __shfl_sync(FULL, w.s, j);
            const float tj = __shfl_sync(FULL, w.t, j);
            const float* xr = HALO && cj >= p.split ? p.x2 + (int64_t)(cj - p.split) * D : p.x + (int64_t)cj * D;
            const float* gr = p.dout + (int64_t)rj * D;
            float acc = 0.f;
            for (int64_t f = lane; f < D; f += 32)
                acc = __fmaf_rn(__fmul_rn(__ldg(gr + f), tj), __fmul_rn(__ldg(xr + f), sj), acc);
            acc = warp_sum(acc);
            if (lane == j) p.dw[w.id] = __fadd_rn(acc, w.a);
        }
    }
}

}  // namespace
}  // namespace gnnb

using namespace gnnb;

extern "C" {

int gnnb_gcn_edge_weight_grad_halo(gnnb_graph_t g, const float* dout, const float* h_local, const float* h_halo,
                                   int64_t n_local, const float* cs, const float* ct, const float* dd, int64_t D,
                                   float* dw, void* stream) {
    if (!g) GNNB_FAIL(GNNB_EINVAL, "graph handle is NULL");
    if (D <= 0) GNNB_FAIL(GNNB_ESIZE, "feature dimension must be positive (got %lld)", (long long)D);
    if (n_local < 0 || n_local > g->n_src) GNNB_FAIL(GNNB_ESIZE, "n_local must be in [0, num_src]");
    if (g->E == 0) return GNNB_OK;   // no edge (a rank that owns no node, or none with in-edges): nothing to write
    if (!dout || !dw) GNNB_FAIL(GNNB_EINVAL, "dout/dw is NULL");
    if (n_local > 0 && !h_local) GNNB_FAIL(GNNB_EINVAL, "h_local is NULL");
    if (n_local < g->n_src && !h_halo) GNNB_FAIL(GNNB_EINVAL, "h_halo is NULL but the plan has sources >= n_local");
    cudaStream_t st = (cudaStream_t)stream;
    GNNB_TRY(ensure_csr(g, false, st));
    const Csr& c = g->by_dst;
    GNNB_TRY(ensure_items(g, c, st));
    EwGradParams p;
    p.items = reinterpret_cast<const int4*>(c.items);
    p.n_items = c.n_items;
    p.col = c.col; p.row = c.row; p.eid = c.eid;
    p.dout = dout; p.x = h_local; p.x2 = h_halo; p.split = (int32_t)n_local;
    if (!h_local) { p.x = h_halo; p.x2 = nullptr; p.split = 0; }   // no local rows at all: one base
    p.cs = cs; p.ct = ct; p.dd = dd; p.dw = dw; p.D = D;
    if (p.n_items == 0) return GNNB_OK;
    const int halo = p.x2 != nullptr;
    const unsigned blocks = (unsigned)ceil_div(p.n_items, 8);
    const bool aligned = !(reinterpret_cast<uintptr_t>(p.x) & 15) && !(reinterpret_cast<uintptr_t>(p.x2) & 15) &&
                         !(reinterpret_cast<uintptr_t>(dout) & 15);
    if (aligned && D == 128) {
        if (halo) gcn_ew_grad_kernel<1, 1><<<blocks, 256, 0, st>>>(p); else gcn_ew_grad_kernel<1, 0><<<blocks, 256, 0, st>>>(p);
    } else if (aligned && D == 256) {
        if (halo) gcn_ew_grad_kernel<2, 1><<<blocks, 256, 0, st>>>(p); else gcn_ew_grad_kernel<2, 0><<<blocks, 256, 0, st>>>(p);
    } else if (aligned && D == 512) {
        if (halo) gcn_ew_grad_kernel<4, 1><<<blocks, 256, 0, st>>>(p); else gcn_ew_grad_kernel<4, 0><<<blocks, 256, 0, st>>>(p);
    } else {
        if (halo) gcn_ew_grad_generic_kernel<1><<<blocks, 256, 0, st>>>(p); else gcn_ew_grad_generic_kernel<0><<<blocks, 256, 0, st>>>(p);
    }
    GNNB_LAUNCHED();
    return GNNB_OK;
}

}  // extern "C"
