// gatlogit.cu — the per-node halves of GAT's attention logits and their pullback.
//
// gat_message (GNNlib/src/layers/conv.jl:152-167) computes  aWW = sum(l.a .* vcat(Wxi, Wxj), dims = 1)  on (2C, H, E) edge
// tensors; the sum splits into a target term and a source term that only depend on the node:
//     el[h, i] = sum_c a[c, h]     * Wx[c, h, i]        (rows 1..C of `a` pair with the target, conv.jl:157)
//     er[h, j] = sum_c a[C + c, h] * Wx[c, h, j]        (rows C+1..2C with the source)
// Forward: ONE pass over Wx (the round-1 host code did it with two broadcast-multiply-reduce expressions in eager PyTorch:
// two (C,H,N) temporaries, ~60 GB of traffic at config 3 with their autograd).  Pullback, given del (H,N), der (H,N):
//     dWx[c,h,n] += del[h,n] a[c,h] + der[h,n] a[C+c,h]            (accumulated IN PLACE into the dWx of gnnb_gat_aggregate_bwd)
//     da[c,h] = sum_n del[h,n] Wx[c,h,n],   da[C+c,h] = sum_n der[h,n] Wx[c,h,n]
// da is reduced deterministically: per-lane partial sums over a fixed node assignment, fixed-order block and grid stages.
// Layouts are the Julia arrays' memory: Wx (C,H,N) = node-major rows of H*C floats, a (2C,H) column-major = a[h*2C + c].
#include "common.cuh"

namespace gnnb {
namespace {

constexpr int LOGIT_WARPS = 8;                 // warps per CTA

// G lanes share a head (G = C/4, a power of two <= 32); a warp covers 32/G heads per pass
template <int G>
__global__ void __launch_bounds__(LOGIT_WARPS * 32) gat_logit_fwd_kernel(const float* __restrict__ Wx, const float* __restrict__ a,
                                                                         int64_t N, int C, int H, float* __restrict__ el,
                                                                         float* __restrict__ er) {
    constexpr int HPP = 32 / G;                // heads per pass
    const int lane = threadIdx.x & 31;
    const int64_t n = (int64_t)blockIdx.x * LOGIT_WARPS + (threadIdx.x >> 5);
    if (n >= N) return;
    const int sub = lane / G, c4 = (lane % G) * 4;
    const float* row = Wx + n * (int64_t)H * C;
    for (int h0 = 0; h0 < H; h0 += HPP) {
        const int h = h0 + sub;
        float pl = 0.f, pr = 0.f;
        if (h < H) {
            const float4 w = __ldg(reinterpret_cast<const float4*>(row + h * C + c4));
            const float4 ai = __ldg(reinterpret_cast<const float4*>(a + (int64_t)h * 2 * C + c4));
            const float4 aj = __ldg(reinterpret_cast<const float4*>(a + (int64_t)h * 2 * C + C + c4));
            pl = ai.x * w.x + ai.y * w.y + ai.z * w.z + ai.w * w.w;
            pr = aj.x * w.x + aj.y * w.y + aj.z * w.z + aj.w * w.w;
        }
#pragma unroll
        for (int o = G / 2; o > 0; o >>= 1) {
            pl += __shfl_xor_sync(0xffffffffu, pl, o);
            pr += __shfl_xor_sync(0xffffffffu, pr, o);
        }
        if (h < H && (lane % G) == 0) { el[n * H + h] = pl; er[n * H + h] = pr; }
    }
}

// persistent: warp w of the grid owns nodes w, w + W, ...; per-lane da partials stay in registers across its nodes.
// One slice of H heads: Wx, a, del, der and dWx point at the slice's first head, ldh is the heads per node of the whole
// arrays (row strides ldh * C and ldh), partial holds the slice's [h][2C] block.
template <int G, int PASSES>
__global__ void __launch_bounds__(LOGIT_WARPS * 32) gat_logit_bwd_kernel(const float* __restrict__ Wx, const float* __restrict__ a,
                                                                         const float* __restrict__ del, const float* __restrict__ der,
                                                                         int64_t N, int C, int H, int ldh, float* __restrict__ dWx,
                                                                         float* __restrict__ partial) {
    constexpr int HPP = 32 / G;
    extern __shared__ float sm[];              // [LOGIT_WARPS][2 * H * C]
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    const int sub = lane / G, c4 = (lane % G) * 4;
    const int64_t W = (int64_t)gridDim.x * LOGIT_WARPS;
    float4 acci[PASSES], accj[PASSES], ai[PASSES], aj[PASSES];
#pragma unroll
    for (int p = 0; p < PASSES; ++p) {
        acci[p] = make_float4(0.f, 0.f, 0.f, 0.f);
        accj[p] = make_float4(0.f, 0.f, 0.f, 0.f);
        const int h = p * HPP + sub;
        ai[p] = aj[p] = make_float4(0.f, 0.f, 0.f, 0.f);
        if (h < H) {
            ai[p] = __ldg(reinterpret_cast<const float4*>(a + (int64_t)h * 2 * C + c4));
            aj[p] = __ldg(reinterpret_cast<const float4*>(a + (int64_t)h * 2 * C + C + c4));
        }
    }
    for (int64_t n = (int64_t)blockIdx.x * LOGIT_WARPS + warp; n < N; n += W) {
        const float* row = Wx + n * (int64_t)ldh * C;
        float* drow = dWx + n * (int64_t)ldh * C;
#pragma unroll
        for (int p = 0; p < PASSES; ++p) {
            const int h = p * HPP + sub;
            if (h < H) {
                const float dl = __ldg(del + n * ldh + h), dr = __ldg(der + n * ldh + h);
                const float4 w = __ldg(reinterpret_cast<const float4*>(row + h * C + c4));
                float4 d = *reinterpret_cast<const float4*>(drow + h * C + c4);
                d.x += dl * ai[p].x + dr * aj[p].x; d.y += dl * ai[p].y + dr * aj[p].y;
                d.z += dl * ai[p].z + dr * aj[p].z; d.w += dl * ai[p].w + dr * aj[p].w;
                *reinterpret_cast<float4*>(drow + h * C + c4) = d;
                acci[p].x += dl * w.x; acci[p].y += dl * w.y; acci[p].z += dl * w.z; acci[p].w += dl * w.w;
                accj[p].x += dr * w.x; accj[p].y += dr * w.y; accj[p].z += dr * w.z; accj[p].w += dr * w.w;
            }
        }
    }
    // block stage: every warp's partial (laid out as da: [h][2C]) into shared memory, summed in warp order
    const int A = 2 * H * C;
    float* mine = sm + warp * A;
#pragma unroll
    for (int p = 0; p < PASSES; ++p) {
        const int h = p * HPP + sub;
        if (h < H) {
            *reinterpret_cast<float4*>(mine + h * 2 * C + c4) = acci[p];
            *reinterpret_cast<float4*>(mine + h * 2 * C + C + c4) = accj[p];
        }
    }
    __syncthreads();
    for (int i = threadIdx.x; i < A; i += blockDim.x) {
        float s = 0.f;
        for (int w = 0; w < LOGIT_WARPS; ++w) s += sm[w * A + i];
        partial[(int64_t)blockIdx.x * A + i] = s;
    }
}

// one half per pass (a relation between two node types: el over the targets' W xi, er over the sources' W xj):
// out[n, h] = sum_c a[off + c, h] Wx[c, h, n], off = 0 (el) or C (er)
template <int G>
__global__ void __launch_bounds__(LOGIT_WARPS * 32) gat_logit_half_fwd_kernel(const float* __restrict__ Wx, const float* __restrict__ a,
                                                                              int64_t N, int C, int H, int off, float* __restrict__ out) {
    constexpr int HPP = 32 / G;
    const int lane = threadIdx.x & 31;
    const int64_t n = (int64_t)blockIdx.x * LOGIT_WARPS + (threadIdx.x >> 5);
    if (n >= N) return;
    const int sub = lane / G, c4 = (lane % G) * 4;
    const float* row = Wx + n * (int64_t)H * C;
    for (int h0 = 0; h0 < H; h0 += HPP) {
        const int h = h0 + sub;
        float p = 0.f;
        if (h < H) {
            const float4 w = __ldg(reinterpret_cast<const float4*>(row + h * C + c4));
            const float4 ah = __ldg(reinterpret_cast<const float4*>(a + (int64_t)h * 2 * C + off + c4));
            p = ah.x * w.x + ah.y * w.y + ah.z * w.z + ah.w * w.w;
        }
#pragma unroll
        for (int o = G / 2; o > 0; o >>= 1) p += __shfl_xor_sync(0xffffffffu, p, o);
        if (h < H && (lane % G) == 0) out[n * H + h] = p;
    }
}

// pullback of one half: dWx[c,h,n] += d[h,n] a[off+c,h]; the da partial holds sum_n d Wx in its half and 0 in the other.
// One slice of H heads with row stride ldh, as gat_logit_bwd_kernel.
template <int G, int PASSES>
__global__ void __launch_bounds__(LOGIT_WARPS * 32) gat_logit_half_bwd_kernel(const float* __restrict__ Wx, const float* __restrict__ a,
                                                                              const float* __restrict__ dh, int64_t N, int C, int H, int ldh,
                                                                              int off, float* __restrict__ dWx, float* __restrict__ partial) {
    constexpr int HPP = 32 / G;
    extern __shared__ float sm[];              // [LOGIT_WARPS][2 * H * C]
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    const int sub = lane / G, c4 = (lane % G) * 4;
    const int64_t W = (int64_t)gridDim.x * LOGIT_WARPS;
    float4 acc[PASSES], ah[PASSES];
#pragma unroll
    for (int p = 0; p < PASSES; ++p) {
        acc[p] = make_float4(0.f, 0.f, 0.f, 0.f);
        const int h = p * HPP + sub;
        ah[p] = make_float4(0.f, 0.f, 0.f, 0.f);
        if (h < H) ah[p] = __ldg(reinterpret_cast<const float4*>(a + (int64_t)h * 2 * C + off + c4));
    }
    for (int64_t n = (int64_t)blockIdx.x * LOGIT_WARPS + warp; n < N; n += W) {
        const float* row = Wx + n * (int64_t)ldh * C;
        float* drow = dWx + n * (int64_t)ldh * C;
#pragma unroll
        for (int p = 0; p < PASSES; ++p) {
            const int h = p * HPP + sub;
            if (h < H) {
                const float d = __ldg(dh + n * ldh + h);
                const float4 w = __ldg(reinterpret_cast<const float4*>(row + h * C + c4));
                float4 v = *reinterpret_cast<const float4*>(drow + h * C + c4);
                v.x += d * ah[p].x; v.y += d * ah[p].y; v.z += d * ah[p].z; v.w += d * ah[p].w;
                *reinterpret_cast<float4*>(drow + h * C + c4) = v;
                acc[p].x += d * w.x; acc[p].y += d * w.y; acc[p].z += d * w.z; acc[p].w += d * w.w;
            }
        }
    }
    const int A = 2 * H * C;
    float* mine = sm + warp * A;
#pragma unroll
    for (int p = 0; p < PASSES; ++p) {
        const int h = p * HPP + sub;
        if (h < H) {
            *reinterpret_cast<float4*>(mine + h * 2 * C + off + c4) = acc[p];
            *reinterpret_cast<float4*>(mine + h * 2 * C + (C - off) + c4) = make_float4(0.f, 0.f, 0.f, 0.f);
        }
    }
    __syncthreads();
    for (int i = threadIdx.x; i < A; i += blockDim.x) {
        float s = 0.f;
        for (int w = 0; w < LOGIT_WARPS; ++w) s += sm[w * A + i];
        partial[(int64_t)blockIdx.x * A + i] = s;
    }
}

__global__ void gat_logit_final_kernel(const float* __restrict__ partial, int nblocks, int A, float* __restrict__ da) {
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= A) return;
    float s = 0.f;
    for (int b = 0; b < nblocks; ++b) s += partial[(int64_t)b * A + i];      // fixed order: deterministic
    da[i] = s;
}

bool logit_shape(int64_t C, int64_t H, int* g) {
    if (C < 4 || C % 4 != 0) return false;
    const int64_t G = C / 4;
    if (G > 32 || (G & (G - 1))) return false;
    if (H < 1 || H * C > 4096) return false;
    *g = (int)G;
    return true;
}

}  // namespace
}  // namespace gnnb

using namespace gnnb;

extern "C" {

int gnnb_gat_logit_terms(const float* Wx, const float* a, int64_t N, int64_t C, int64_t H, float* el, float* er, void* stream) {
    if (N < 0 || C <= 0 || H <= 0) GNNB_FAIL(GNNB_ESIZE, "bad sizes");
    if (N == 0) return GNNB_OK;
    if (!Wx || !a || (!el && !er)) GNNB_FAIL(GNNB_EINVAL, "NULL argument");
    int G = 0;
    if (!logit_shape(C, H, &G) || ((uintptr_t)Wx & 15) || ((uintptr_t)a & 15))
        GNNB_FAIL(GNNB_EUNSUPPORTED, "gat_logit_terms: C/4 must be a power of two <= 32, C*H <= 4096, 16 B-aligned operands");
    cudaStream_t st = (cudaStream_t)stream;
    const unsigned blocks = (unsigned)ceil_div(N, LOGIT_WARPS);
    if (!el || !er) {                          // one half: el (rows 1..C of a) or er (rows C+1..2C)
        float* out = el ? el : er;
        const int off = el ? 0 : (int)C;
#define GNNB_LH(GG) case GG: gat_logit_half_fwd_kernel<GG><<<blocks, LOGIT_WARPS * 32, 0, st>>>(Wx, a, N, (int)C, (int)H, off, out); break;
        switch (G) { GNNB_LH(1) GNNB_LH(2) GNNB_LH(4) GNNB_LH(8) GNNB_LH(16) GNNB_LH(32) }
#undef GNNB_LH
        GNNB_LAUNCHED();
        return GNNB_OK;
    }
#define GNNB_LG(GG) case GG: gat_logit_fwd_kernel<GG><<<blocks, LOGIT_WARPS * 32, 0, st>>>(Wx, a, N, (int)C, (int)H, el, er); break;
    switch (G) { GNNB_LG(1) GNNB_LG(2) GNNB_LG(4) GNNB_LG(8) GNNB_LG(16) GNNB_LG(32) }
#undef GNNB_LG
    GNNB_LAUNCHED();
    return GNNB_OK;
}

int gnnb_gat_logit_terms_bwd(const float* Wx, const float* a, const float* del, const float* der, int64_t N, int64_t C,
                             int64_t H, float* dWx_accum, float* da, void* stream) {
    if (N < 0 || C <= 0 || H <= 0) GNNB_FAIL(GNNB_ESIZE, "bad sizes");
    if (!da) GNNB_FAIL(GNNB_EINVAL, "da is NULL");
    cudaStream_t st = (cudaStream_t)stream;
    if (N == 0) { GNNB_CUDA(cudaMemsetAsync(da, 0, sizeof(float) * (size_t)(2 * H * C), st)); return GNNB_OK; }
    if (!Wx || !a || (!del && !der) || !dWx_accum) GNNB_FAIL(GNNB_EINVAL, "NULL argument");
    int G = 0;
    if (!logit_shape(C, H, &G) || ((uintptr_t)Wx & 15) || ((uintptr_t)a & 15) || ((uintptr_t)dWx_accum & 15))
        GNNB_FAIL(GNNB_EUNSUPPORTED, "gat_logit_terms_bwd: C/4 must be a power of two <= 32, C*H <= 4096, 16 B-aligned operands");
    // heads in slices of 8 passes of 32/G heads (C * heads <= 1024 per slice): a slice's block stage needs at most
    // 8 warps x 2 x 1024 floats = 64 KB of shared memory.  nblocks depends on N alone, so each head's da is summed in the
    // same order whatever H and the slice; the slices run in order on one stream and reuse one partial buffer.
    const int hpp = 32 / G;
    const int64_t slice = 8 * hpp;
    const int64_t want = ceil_div(N, LOGIT_WARPS);
    const int nblocks = (int)(want < kNumSMs * 4 ? want : kNumSMs * 4);
    DeviceState* s = nullptr;
    GNNB_TRY(device_state(&s));
    GNNB_TRY(grow_buffer(&s->gat_part, &s->gat_part_bytes, sizeof(float) * (size_t)nblocks * 2 * (H < slice ? H : slice) * C));
    float* part_buf = s->gat_part;
    const int ldh = (int)H;
    for (int64_t h0 = 0; h0 < H; h0 += slice) {
        const int hs = (int)(H - h0 < slice ? H - h0 : slice);
        const int passes = (int)ceil_div(hs, hpp);
        const int A = 2 * hs * (int)C;
        const size_t smem = sizeof(float) * (size_t)LOGIT_WARPS * A;
        const float* Wxs = Wx + h0 * C;
        const float* as = a + h0 * 2 * C;
        float* dWxs = dWx_accum + h0 * C;
        if (!del || !der) {                    // one half: del (target half of da) or der (source half)
            const float* dh = (del ? del : der) + h0;
            const int off = del ? 0 : (int)C;
#define GNNB_LHB(GG, PP) { auto k = gat_logit_half_bwd_kernel<GG, PP>; \
            if (smem > 48 * 1024) GNNB_CUDA(cudaFuncSetAttribute(k, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem)); \
            k<<<nblocks, LOGIT_WARPS * 32, smem, st>>>(Wxs, as, dh, N, (int)C, hs, ldh, off, dWxs, part_buf); }
#define GNNB_LHBP(GG) switch (passes) { case 1: GNNB_LHB(GG, 1) break; case 2: GNNB_LHB(GG, 2) break; case 3: case 4: GNNB_LHB(GG, 4) break; default: GNNB_LHB(GG, 8) break; }
            switch (G) {
                case 1: GNNB_LHBP(1) break; case 2: GNNB_LHBP(2) break; case 4: GNNB_LHBP(4) break;
                case 8: GNNB_LHBP(8) break; case 16: GNNB_LHBP(16) break; default: GNNB_LHBP(32) break;
            }
#undef GNNB_LHBP
#undef GNNB_LHB
        } else {
            const float *dl = del + h0, *dr = der + h0;
#define GNNB_LB(GG, PP) { auto k = gat_logit_bwd_kernel<GG, PP>; \
            if (smem > 48 * 1024) GNNB_CUDA(cudaFuncSetAttribute(k, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem)); \
            k<<<nblocks, LOGIT_WARPS * 32, smem, st>>>(Wxs, as, dl, dr, N, (int)C, hs, ldh, dWxs, part_buf); }
#define GNNB_LBP(GG) switch (passes) { case 1: GNNB_LB(GG, 1) break; case 2: GNNB_LB(GG, 2) break; case 3: case 4: GNNB_LB(GG, 4) break; default: GNNB_LB(GG, 8) break; }
            switch (G) {
                case 1: GNNB_LBP(1) break; case 2: GNNB_LBP(2) break; case 4: GNNB_LBP(4) break;
                case 8: GNNB_LBP(8) break; case 16: GNNB_LBP(16) break; default: GNNB_LBP(32) break;
            }
#undef GNNB_LBP
#undef GNNB_LB
        }
        GNNB_LAUNCHED();
        gat_logit_final_kernel<<<(unsigned)ceil_div((int64_t)A, 128), 128, 0, st>>>(part_buf, nblocks, A, da + h0 * 2 * C);
        GNNB_LAUNCHED();
    }
    return GNNB_OK;
}

}  // extern "C"
