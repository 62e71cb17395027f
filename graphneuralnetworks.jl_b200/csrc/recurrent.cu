// recurrent.cu — the gate arithmetic of the recurrent temporal cells (GraphNeuralNetworks/src/layers/temporalconv.jl):
// GConvGRUCell, DCGRUCell and TGCNCell share the GRU gates, GConvLSTMCell (and Flux's LSTMCell, without peepholes) the
// LSTM gates.  The reference evaluates each gate as a chain of broadcasts, each with its own (out, N) temporary; here a
// step's gates are one pass over node rows.  The graph operators and GEMMs around the gates stay where they are
// (the fused propagate, dense.cu); these kernels only see their outputs:
//   px  the x-side pre-activations of every gate, a (N, G·D) slice of the whole sequence's PX read in place (ld_px);
//   ah  the step's h-side GEMM output, contiguous.
// Each thread owns a float4 or a float of one row: float4 when D % 4 == 0 and every row start is 16 B aligned.  Every
// output is written once, with no atomics; the peephole gradient of the LSTM is a two-stage column sum (per-block
// partials in a fixed order, then dense.cu's colsum_final_kernel), so every result is run-to-run bit-identical.
#include "common.cuh"

namespace gnnb {

int colsum_final(const float* partial, int nblocks, int64_t D, float* out, cudaStream_t st);   // dense.cu

namespace {

template <int VEC> __device__ __forceinline__ void ldv(const float* p, float (&v)[VEC]) {
    if constexpr (VEC == 4) {
        const float4 t = __ldg(reinterpret_cast<const float4*>(p));
        v[0] = t.x; v[1] = t.y; v[2] = t.z; v[3] = t.w;
    } else {
        v[0] = __ldg(p);
    }
}
template <int VEC> __device__ __forceinline__ void stv(float* p, const float (&v)[VEC]) {
    if constexpr (VEC == 4) *reinterpret_cast<float4*>(p) = make_float4(v[0], v[1], v[2], v[3]);
    else *p = v[0];
}
__device__ __forceinline__ float sigm(float a) { return 1.f / (1.f + expf(-a)); }

struct GruParams {
    const float* px; int64_t ld_px;
    const float* ah;                  // rz: (N, 2D); out: (N, D)
    const float* h;
    const float* z;                   // out
    float* r; float* zo; float* rh;   // rz outputs
    float* n; float* h_new;           // out outputs
    int64_t N, D;
    int blend;
};

template <int VEC>
__global__ void __launch_bounds__(256) gru_rz_kernel(const GruParams p) {
    const int64_t nv = p.D / VEC, total = p.N * nv;
    for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (int64_t)gridDim.x * blockDim.x) {
        const int64_t row = i / nv, col = (i - row * nv) * VEC;
        float xr[VEC], xz[VEC], ar[VEC], az[VEC], hv[VEC], r[VEC], z[VEC], rh[VEC];
        const float* pxr = p.px + row * p.ld_px + col;
        ldv<VEC>(pxr, xr); ldv<VEC>(pxr + p.D, xz);
        ldv<VEC>(p.ah + row * 2 * p.D + col, ar); ldv<VEC>(p.ah + row * 2 * p.D + p.D + col, az);
        ldv<VEC>(p.h + row * p.D + col, hv);
#pragma unroll
        for (int k = 0; k < VEC; ++k) {
            r[k] = sigm(xr[k] + ar[k]);
            z[k] = sigm(xz[k] + az[k]);
            rh[k] = r[k] * hv[k];
        }
        stv<VEC>(p.r + row * p.D + col, r); stv<VEC>(p.zo + row * p.D + col, z); stv<VEC>(p.rh + row * p.D + col, rh);
    }
}

template <int VEC>
__global__ void __launch_bounds__(256) gru_out_kernel(const GruParams p) {
    const int64_t nv = p.D / VEC, total = p.N * nv;
    for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (int64_t)gridDim.x * blockDim.x) {
        const int64_t row = i / nv, col = (i - row * nv) * VEC, o = row * p.D + col;
        float xn[VEC], an[VEC], hv[VEC], z[VEC], n[VEC], hn[VEC];
        ldv<VEC>(p.px + row * p.ld_px + 2 * p.D + col, xn); ldv<VEC>(p.ah + o, an);
        ldv<VEC>(p.h + o, hv); ldv<VEC>(p.z + o, z);
#pragma unroll
        for (int k = 0; k < VEC; ++k) {
            n[k] = tanhf(xn[k] + an[k]);
            hn[k] = p.blend == 0 ? (1.f - z[k]) * n[k] + z[k] * hv[k] : (1.f - z[k]) * hv[k] + z[k] * n[k];
        }
        stv<VEC>(p.n + o, n); stv<VEC>(p.h_new + o, hn);
    }
}

struct GruBwdParams {
    const float* dh_new; const float* drh; const float* dz_in;
    const float* h; const float* r; const float* z; const float* n;
    float* dpre; int64_t ld_dpre;     // out_bwd: the n block; rz_bwd: [r | z]
    float* dz; float* dh;
    int64_t N, D;
    int blend;
};

template <int VEC>
__global__ void __launch_bounds__(256) gru_out_bwd_kernel(const GruBwdParams p) {
    const int64_t nv = p.D / VEC, total = p.N * nv;
    for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (int64_t)gridDim.x * blockDim.x) {
        const int64_t row = i / nv, col = (i - row * nv) * VEC, o = row * p.D + col;
        float dy[VEC], hv[VEC], z[VEC], n[VEC], dn[VEC], dz[VEC], dh[VEC];
        ldv<VEC>(p.dh_new + o, dy); ldv<VEC>(p.h + o, hv); ldv<VEC>(p.z + o, z); ldv<VEC>(p.n + o, n);
#pragma unroll
        for (int k = 0; k < VEC; ++k) {
            const float a = p.blend == 0 ? 1.f - z[k] : z[k];          // the weight of n in h'
            dn[k] = dy[k] * a * (1.f - n[k] * n[k]);
            dz[k] = p.blend == 0 ? dy[k] * (hv[k] - n[k]) : dy[k] * (n[k] - hv[k]);
            dh[k] = dy[k] * (p.blend == 0 ? z[k] : 1.f - z[k]);
        }
        stv<VEC>(p.dpre + row * p.ld_dpre + col, dn); stv<VEC>(p.dz + o, dz); stv<VEC>(p.dh + o, dh);
    }
}

template <int VEC>
__global__ void __launch_bounds__(256) gru_rz_bwd_kernel(const GruBwdParams p) {
    const int64_t nv = p.D / VEC, total = p.N * nv;
    for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (int64_t)gridDim.x * blockDim.x) {
        const int64_t row = i / nv, col = (i - row * nv) * VEC, o = row * p.D + col;
        float drh[VEC], dzv[VEC], hv[VEC], r[VEC], z[VEC], dh[VEC], dr[VEC], dzz[VEC];
        ldv<VEC>(p.drh + o, drh); ldv<VEC>(p.dz_in + o, dzv); ldv<VEC>(p.h + o, hv); ldv<VEC>(p.r + o, r);
        ldv<VEC>(p.z + o, z); ldv<VEC>(p.dh + o, dh);
#pragma unroll
        for (int k = 0; k < VEC; ++k) {
            dr[k] = drh[k] * hv[k] * (r[k] * (1.f - r[k]));
            dzz[k] = dzv[k] * (z[k] * (1.f - z[k]));
            dh[k] = fmaf(drh[k], r[k], dh[k]);
        }
        float* d = p.dpre + row * p.ld_dpre + col;
        stv<VEC>(d, dr); stv<VEC>(d + p.D, dzz); stv<VEC>(p.dh + o, dh);
    }
}

struct LstmParams {
    const float* px; int64_t ld_px;
    const float* ah; const float* c; const float* w;
    float* gates; float* c_new; float* h_new;
    const float* dh_new; const float* dc_new; const float* gates_in; const float* cn_in;   // bwd
    float* dpre; float* dc; float* partial;
    int64_t N, D;
    int rows_per_block, tile_w;
};

template <int VEC>
__global__ void __launch_bounds__(256) lstm_fwd_kernel(const LstmParams p) {
    const int64_t nv = p.D / VEC, total = p.N * nv, D = p.D;
    for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (int64_t)gridDim.x * blockDim.x) {
        const int64_t row = i / nv, col = (i - row * nv) * VEC, o = row * D + col;
        float pre[4][VEC], a[VEC], c[VEC], w[4][VEC], cn[VEC], hn[VEC];
        ldv<VEC>(p.c + o, c);
#pragma unroll
        for (int g = 0; g < 4; ++g) {
            ldv<VEC>(p.px + row * p.ld_px + g * D + col, pre[g]);
            ldv<VEC>(p.ah + row * 4 * D + g * D + col, a);
#pragma unroll
            for (int k = 0; k < VEC; ++k) { pre[g][k] += a[k]; w[g][k] = 0.f; }
            if (p.w) ldv<VEC>(p.w + g * D + col, w[g]);
        }
#pragma unroll
        for (int k = 0; k < VEC; ++k) {
            const float ig = sigm(fmaf(w[0][k], c[k], pre[0][k]));
            const float fg = sigm(fmaf(w[1][k], c[k], pre[1][k]));
            const float gg = tanhf(fmaf(w[2][k], c[k], pre[2][k]));
            cn[k] = fmaf(fg, c[k], ig * gg);
            const float og = sigm(fmaf(w[3][k], cn[k], pre[3][k]));
            hn[k] = og * tanhf(cn[k]);
            pre[0][k] = ig; pre[1][k] = fg; pre[2][k] = gg; pre[3][k] = og;
        }
#pragma unroll
        for (int g = 0; g < 4; ++g) stv<VEC>(p.gates + row * 4 * D + g * D + col, pre[g]);
        stv<VEC>(p.c_new + o, cn); stv<VEC>(p.h_new + o, hn);
    }
}

// Block (bx, by): rows [bx·rows_per_block, ...) of the column groups [by·tile_w, (by+1)·tile_w).  With fewer than 256
// column groups, 256 / tile_w threads walk interleaved rows of the same group and their peephole partials are added in
// thread order; the block's sums go to partial[bx][4D].  (dense.cu's act_bwd_kernel has the same layout.)
template <int VEC, bool PEEP>
__global__ void __launch_bounds__(256) lstm_bwd_kernel(const LstmParams p) {
    const int64_t nv = p.D / VEC, D = p.D;
    const int tw = p.tile_w, cgl = threadIdx.x % tw, rsub = threadIdx.x / tw, rstep = 256 / tw;
    const int64_t cg = (int64_t)blockIdx.y * tw + cgl, col = cg * VEC;
    const bool active = rsub < rstep && cg < nv;
    const int64_t r0 = (int64_t)blockIdx.x * p.rows_per_block;
    const int64_t r1 = r0 + p.rows_per_block < p.N ? r0 + p.rows_per_block : p.N;
    float acc[4][VEC];
#pragma unroll
    for (int g = 0; g < 4; ++g)
#pragma unroll
        for (int k = 0; k < VEC; ++k) acc[g][k] = 0.f;
    float w[4][VEC];
#pragma unroll
    for (int g = 0; g < 4; ++g) {
#pragma unroll
        for (int k = 0; k < VEC; ++k) w[g][k] = 0.f;
        if (PEEP && active) ldv<VEC>(p.w + g * D + col, w[g]);
    }
    if (active) {
        for (int64_t row = r0 + rsub; row < r1; row += rstep) {
            const int64_t o = row * D + col;
            float gt[4][VEC], dy[VEC], dcn[VEC], c[VEC], cn[VEC], d[4][VEC], dc[VEC];
#pragma unroll
            for (int g = 0; g < 4; ++g) ldv<VEC>(p.gates_in + row * 4 * D + g * D + col, gt[g]);
            ldv<VEC>(p.dh_new + o, dy); ldv<VEC>(p.dc_new + o, dcn); ldv<VEC>(p.c + o, c); ldv<VEC>(p.cn_in + o, cn);
#pragma unroll
            for (int k = 0; k < VEC; ++k) {
                const float ig = gt[0][k], fg = gt[1][k], gg = gt[2][k], og = gt[3][k];
                const float tc = tanhf(cn[k]);
                d[3][k] = dy[k] * tc * (og * (1.f - og));
                float dct = dcn[k] + dy[k] * og * (1.f - tc * tc);
                if (PEEP) dct = fmaf(d[3][k], w[3][k], dct);
                d[0][k] = dct * gg * (ig * (1.f - ig));
                d[1][k] = dct * c[k] * (fg * (1.f - fg));
                d[2][k] = dct * ig * (1.f - gg * gg);
                dc[k] = dct * fg;
                if (PEEP) {
                    dc[k] = fmaf(d[0][k], w[0][k], dc[k]);
                    dc[k] = fmaf(d[1][k], w[1][k], dc[k]);
                    dc[k] = fmaf(d[2][k], w[2][k], dc[k]);
                    acc[0][k] = fmaf(d[0][k], c[k], acc[0][k]);
                    acc[1][k] = fmaf(d[1][k], c[k], acc[1][k]);
                    acc[2][k] = fmaf(d[2][k], c[k], acc[2][k]);
                    acc[3][k] = fmaf(d[3][k], cn[k], acc[3][k]);
                }
            }
#pragma unroll
            for (int g = 0; g < 4; ++g) stv<VEC>(p.dpre + row * 4 * D + g * D + col, d[g]);
            stv<VEC>(p.dc + o, dc);
        }
    }
    if constexpr (PEEP) {
        if (!p.partial) return;                        // block-uniform
        __shared__ float sm[4 * VEC][256];
#pragma unroll
        for (int g = 0; g < 4; ++g)
#pragma unroll
            for (int k = 0; k < VEC; ++k) sm[g * VEC + k][threadIdx.x] = acc[g][k];
        __syncthreads();
        if (rsub == 0 && cg < nv) {
            for (int q = 1; q < rstep; ++q)
#pragma unroll
                for (int g = 0; g < 4; ++g)
#pragma unroll
                    for (int k = 0; k < VEC; ++k) acc[g][k] += sm[g * VEC + k][q * tw + cgl];
            float* out = p.partial + (int64_t)blockIdx.x * 4 * D;
#pragma unroll
            for (int g = 0; g < 4; ++g)
#pragma unroll
                for (int k = 0; k < VEC; ++k) out[g * D + col + k] = acc[g][k];
        }
    }
}

bool a16(const void* a) { return (reinterpret_cast<uintptr_t>(a) & 15) == 0; }
unsigned grid_for(int64_t work) {
    const int64_t b = ceil_div(work, 256), cap = (int64_t)kNumSMs * 16;
    return (unsigned)(b < cap ? b : cap);
}
#define GNNB_GRID(vec, N, D) grid_for((N) * ((D) / (vec)))

}  // namespace
}  // namespace gnnb

using namespace gnnb;

#define REC_SIZES(name, G, ld)                                                                                       \
    if (N < 0 || D < 1) GNNB_FAIL(GNNB_ESIZE, name ": N must be >= 0 and D >= 1 (got N = %lld, D = %lld)",          \
                                  (long long)N, (long long)D);                                                       \
    if ((ld) < (G) * D) GNNB_FAIL(GNNB_ESIZE, name ": row stride %lld is below %d * D = %lld", (long long)(ld),    \
                                  (int)(G), (long long)((G) * D));

extern "C" {

int gnnb_gru_rz(const float* px, int64_t ld_px, const float* ah, const float* h, int64_t N, int64_t D, float* r,
                float* z, float* rh, void* stream) {
    REC_SIZES("gru_rz", 3, ld_px)
    if (N == 0) return GNNB_OK;
    if (!px || !ah || !h || !r || !z || !rh) GNNB_FAIL(GNNB_ESIZE, "gru_rz: NULL array of positive size");
    GruParams p = {};
    p.px = px; p.ld_px = ld_px; p.ah = ah; p.h = h; p.r = r; p.zo = z; p.rh = rh; p.N = N; p.D = D;
    const bool v4 = D % 4 == 0 && ld_px % 4 == 0 && a16(px) && a16(ah) && a16(h) && a16(r) && a16(z) && a16(rh);
    cudaStream_t st = (cudaStream_t)stream;
    if (v4) gru_rz_kernel<4><<<GNNB_GRID(4, N, D), 256, 0, st>>>(p);
    else gru_rz_kernel<1><<<GNNB_GRID(1, N, D), 256, 0, st>>>(p);
    GNNB_LAUNCHED();
    return GNNB_OK;
}

int gnnb_gru_out(const float* px, int64_t ld_px, const float* ah_n, const float* h, const float* z, int64_t N,
                 int64_t D, int blend, float* n, float* h_new, void* stream) {
    REC_SIZES("gru_out", 3, ld_px)
    if (blend != 0 && blend != 1) GNNB_FAIL(GNNB_EINVAL, "gru_out: blend must be 0 or 1 (got %d)", blend);
    if (N == 0) return GNNB_OK;
    if (!px || !ah_n || !h || !z || !n || !h_new) GNNB_FAIL(GNNB_ESIZE, "gru_out: NULL array of positive size");
    GruParams p = {};
    p.px = px; p.ld_px = ld_px; p.ah = ah_n; p.h = h; p.z = z; p.n = n; p.h_new = h_new; p.N = N; p.D = D;
    p.blend = blend;
    const bool v4 = D % 4 == 0 && ld_px % 4 == 0 && a16(px) && a16(ah_n) && a16(h) && a16(z) && a16(n) && a16(h_new);
    cudaStream_t st = (cudaStream_t)stream;
    if (v4) gru_out_kernel<4><<<GNNB_GRID(4, N, D), 256, 0, st>>>(p);
    else gru_out_kernel<1><<<GNNB_GRID(1, N, D), 256, 0, st>>>(p);
    GNNB_LAUNCHED();
    return GNNB_OK;
}

int gnnb_gru_out_bwd(const float* dh_new, const float* h, const float* z, const float* n, int64_t N, int64_t D,
                     int blend, float* dpre_n, int64_t ld_dpre, float* dz, float* dh, void* stream) {
    REC_SIZES("gru_out_bwd", 1, ld_dpre)
    if (blend != 0 && blend != 1) GNNB_FAIL(GNNB_EINVAL, "gru_out_bwd: blend must be 0 or 1 (got %d)", blend);
    if (N == 0) return GNNB_OK;
    if (!dh_new || !h || !z || !n || !dpre_n || !dz || !dh)
        GNNB_FAIL(GNNB_ESIZE, "gru_out_bwd: NULL array of positive size");
    GruBwdParams p = {};
    p.dh_new = dh_new; p.h = h; p.z = z; p.n = n; p.dpre = dpre_n; p.ld_dpre = ld_dpre; p.dz = dz; p.dh = dh;
    p.N = N; p.D = D; p.blend = blend;
    const bool v4 = D % 4 == 0 && ld_dpre % 4 == 0 && a16(dh_new) && a16(h) && a16(z) && a16(n) && a16(dpre_n) &&
                    a16(dz) && a16(dh);
    cudaStream_t st = (cudaStream_t)stream;
    if (v4) gru_out_bwd_kernel<4><<<GNNB_GRID(4, N, D), 256, 0, st>>>(p);
    else gru_out_bwd_kernel<1><<<GNNB_GRID(1, N, D), 256, 0, st>>>(p);
    GNNB_LAUNCHED();
    return GNNB_OK;
}

int gnnb_gru_rz_bwd(const float* drh, const float* dz, const float* h, const float* r, const float* z, int64_t N,
                    int64_t D, float* dpre_rz, int64_t ld_dpre, float* dh, void* stream) {
    REC_SIZES("gru_rz_bwd", 2, ld_dpre)
    if (N == 0) return GNNB_OK;
    if (!drh || !dz || !h || !r || !z || !dpre_rz || !dh) GNNB_FAIL(GNNB_ESIZE, "gru_rz_bwd: NULL array of positive size");
    GruBwdParams p = {};
    p.drh = drh; p.dz_in = dz; p.h = h; p.r = r; p.z = z; p.dpre = dpre_rz; p.ld_dpre = ld_dpre; p.dh = dh;
    p.N = N; p.D = D;
    const bool v4 = D % 4 == 0 && ld_dpre % 4 == 0 && a16(drh) && a16(dz) && a16(h) && a16(r) && a16(z) &&
                    a16(dpre_rz) && a16(dh);
    cudaStream_t st = (cudaStream_t)stream;
    if (v4) gru_rz_bwd_kernel<4><<<GNNB_GRID(4, N, D), 256, 0, st>>>(p);
    else gru_rz_bwd_kernel<1><<<GNNB_GRID(1, N, D), 256, 0, st>>>(p);
    GNNB_LAUNCHED();
    return GNNB_OK;
}

int gnnb_lstm_cell(const float* px, int64_t ld_px, const float* ah, const float* c, const float* w, int64_t N,
                   int64_t D, float* gates, float* c_new, float* h_new, void* stream) {
    REC_SIZES("lstm_cell", 4, ld_px)
    if (N == 0) return GNNB_OK;
    if (!px || !ah || !c || !gates || !c_new || !h_new) GNNB_FAIL(GNNB_ESIZE, "lstm_cell: NULL array of positive size");
    LstmParams p = {};
    p.px = px; p.ld_px = ld_px; p.ah = ah; p.c = c; p.w = w; p.gates = gates; p.c_new = c_new; p.h_new = h_new;
    p.N = N; p.D = D;
    const bool v4 = D % 4 == 0 && ld_px % 4 == 0 && a16(px) && a16(ah) && a16(c) && (!w || a16(w)) && a16(gates) &&
                    a16(c_new) && a16(h_new);
    cudaStream_t st = (cudaStream_t)stream;
    if (v4) lstm_fwd_kernel<4><<<GNNB_GRID(4, N, D), 256, 0, st>>>(p);
    else lstm_fwd_kernel<1><<<GNNB_GRID(1, N, D), 256, 0, st>>>(p);
    GNNB_LAUNCHED();
    return GNNB_OK;
}

int gnnb_lstm_cell_bwd(const float* dh_new, const float* dc_new, const float* c, const float* gates,
                       const float* c_new, const float* w, int64_t N, int64_t D, float* dpre, float* dc, float* dw,
                       float* ws, void* stream) {
    REC_SIZES("lstm_cell_bwd", 1, D)
    if (dw && !w) GNNB_FAIL(GNNB_EINVAL, "lstm_cell_bwd: dw asks for the peephole gradient, but w is NULL");
    if (dw && !ws) GNNB_FAIL(GNNB_ESIZE, "lstm_cell_bwd: NULL array of positive size (ws)");
    cudaStream_t st = (cudaStream_t)stream;
    if (N == 0) {                                      // an empty sum: dw = 0
        if (dw) GNNB_CUDA(cudaMemsetAsync(dw, 0, sizeof(float) * (size_t)(4 * D), st));
        return GNNB_OK;
    }
    if (!dh_new || !dc_new || !c || !gates || !c_new || !dpre || !dc)
        GNNB_FAIL(GNNB_ESIZE, "lstm_cell_bwd: NULL array of positive size");
    const bool v4 = D % 4 == 0 && a16(dh_new) && a16(dc_new) && a16(c) && a16(gates) && a16(c_new) && (!w || a16(w)) &&
                    a16(dpre) && a16(dc);
    const int vec = v4 ? 4 : 1;
    const int64_t nv = D / vec;
    const int64_t slots = GNNB_LSTM_DW_SLOTS(N);
    LstmParams p = {};
    p.dh_new = dh_new; p.dc_new = dc_new; p.c = c; p.gates_in = gates; p.cn_in = c_new; p.w = w; p.dpre = dpre; p.dc = dc;
    p.partial = dw ? ws : nullptr; p.N = N; p.D = D;
    p.rows_per_block = (int)ceil_div(N, slots);
    p.tile_w = (int)(nv < 256 ? nv : 256);
    const dim3 grid((unsigned)ceil_div(N, p.rows_per_block), (unsigned)ceil_div(nv, p.tile_w));
    if (v4) {
        if (w) lstm_bwd_kernel<4, true><<<grid, 256, 0, st>>>(p);
        else lstm_bwd_kernel<4, false><<<grid, 256, 0, st>>>(p);
    } else {
        if (w) lstm_bwd_kernel<1, true><<<grid, 256, 0, st>>>(p);
        else lstm_bwd_kernel<1, false><<<grid, 256, 0, st>>>(p);
    }
    GNNB_LAUNCHED();
    if (dw) return colsum_final(ws, (int)grid.x, 4 * D, dw, st);
    return GNNB_OK;
}

}  // extern "C"
