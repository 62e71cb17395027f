// dense.cu — the per-layer dense contraction of the conv layers:  σ.(W * x .+ b)  and its pullback
// (GNNlib/src/layers/conv.jl:39,69-71 for gcn_conv; :281 for sage_conv).
//
// This is the only true dense contraction on the hot path.  The shapes the layers use most go to the hand-written
// 3xTF32 wgmma kernels of dense_tc.cu; every other shape is a plain library GEMM, as in the reference (BLAS/cuBLAS
// sgemm), through cuBLASLt from the CUDA 12.9 toolkit with
//   * compute type CUBLAS_COMPUTE_32F_EMULATED_16BFX9 where the library offers it (fp32 in/out, each operand split into
//     three bf16 terms), else CUBLAS_COMPUTE_32F, the fp32 sgemm;
//   * the bias and relu fused into the GEMM epilogue (CUBLASLT_EPILOGUE_[RELU_]BIAS);
// and hand-written kernels for the elementwise pullback pieces (relu mask × upstream gradient + bias gradient in one
// pass).  cuBLASLt 12.9 is dlopen'ed by absolute path so that it does not collide with the older cuBLAS a host
// framework may have loaded under the same SONAME.
#include "common.cuh"
#include <cublasLt.h>
#include <dlfcn.h>
#include <stdlib.h>

namespace gnnb {

namespace lt {
#define LT_FN(name) static decltype(&::name) name = nullptr;
LT_FN(cublasLtCreate) LT_FN(cublasLtMatmulDescCreate) LT_FN(cublasLtMatmulDescDestroy) LT_FN(cublasLtMatmulDescSetAttribute)
LT_FN(cublasLtMatrixLayoutCreate) LT_FN(cublasLtMatrixLayoutDestroy) LT_FN(cublasLtMatmulPreferenceCreate)
LT_FN(cublasLtMatmulPreferenceDestroy) LT_FN(cublasLtMatmulPreferenceSetAttribute) LT_FN(cublasLtMatmulAlgoGetHeuristic)
LT_FN(cublasLtMatmul) LT_FN(cublasLtGetVersion)
#undef LT_FN
static void* handle_lib = nullptr;
static bool loaded = false;   // every symbol above resolved (process-wide: the library is loaded once)
static const size_t workspace_bytes = (size_t)256 << 20;
static int emulation = -1;   // -1 unknown, 0 unavailable, 1 in use
static int want_emulation = 1;
static std::mutex mu;

static int load_symbols() {
    if (loaded) return GNNB_OK;
    const char* env = getenv("GNNB_CUBLASLT");
    const char* cands[] = {env, "/usr/local/cuda/lib64/libcublasLt.so.12", "/usr/local/cuda/lib64/libcublasLt.so",
                           "libcublasLt.so.12"};
    for (const char* c : cands) {
        if (!c) continue;
        handle_lib = dlopen(c, RTLD_NOW | RTLD_LOCAL);
        if (handle_lib) break;
    }
    if (!handle_lib) GNNB_FAIL(GNNB_ECUDA, "cannot dlopen cuBLASLt: %s", dlerror());
#define LT_LOAD(name)                                                        \
    name = (decltype(name))dlsym(handle_lib, #name);                         \
    if (!name) GNNB_FAIL(GNNB_ECUDA, "cuBLASLt symbol %s not found", #name);
    LT_LOAD(cublasLtCreate) LT_LOAD(cublasLtMatmulDescCreate) LT_LOAD(cublasLtMatmulDescDestroy)
    LT_LOAD(cublasLtMatmulDescSetAttribute) LT_LOAD(cublasLtMatrixLayoutCreate) LT_LOAD(cublasLtMatrixLayoutDestroy)
    LT_LOAD(cublasLtMatmulPreferenceCreate) LT_LOAD(cublasLtMatmulPreferenceDestroy)
    LT_LOAD(cublasLtMatmulPreferenceSetAttribute) LT_LOAD(cublasLtMatmulAlgoGetHeuristic) LT_LOAD(cublasLtMatmul)
    LT_LOAD(cublasLtGetVersion)
#undef LT_LOAD
    loaded = true;
    return GNNB_OK;
}

// the library and the current device's handle and workspace (s->lt, s->lt_ws), loaded on first use
static int load(DeviceState* s) {
    std::lock_guard<std::mutex> lock(mu);
    if (s->lt) return GNNB_OK;
    GNNB_TRY(load_symbols());
    cublasLtHandle_t h = nullptr;
    if (cublasLtCreate(&h) != CUBLAS_STATUS_SUCCESS) GNNB_FAIL(GNNB_ECUDA, "cublasLtCreate failed");
    GNNB_CUDA(cudaMalloc(&s->lt_ws, workspace_bytes));
    s->lt = h;
    return GNNB_OK;
}

// C(m x n, ldc) = op(A)(m x k) * op(B)(k x n) [+ bias(m)] [relu], all column-major fp32
static int matmul(cublasOperation_t ta, cublasOperation_t tb, int64_t m, int64_t n, int64_t k, const float* A, int64_t lda,
                  const float* B, int64_t ldb, float* C, int64_t ldc, const float* bias, int relu, cudaStream_t st) {
    DeviceState* ds = nullptr;
    GNNB_TRY(device_state(&ds));
    GNNB_TRY(load(ds));
    cublasLtHandle_t handle = ds->lt;
    void* workspace = ds->lt_ws;
    if (m == 0 || n == 0) return GNNB_OK;
    if (k == 0 && ldc == m && !bias) { GNNB_CUDA(cudaMemsetAsync(C, 0, sizeof(float) * (size_t)(m * n), st)); return GNNB_OK; }
    const bool try_emu = want_emulation && emulation != 0;
    for (int pass = try_emu ? 0 : 1; pass < 2; ++pass) {
        const bool emu = (pass == 0);
        cublasLtMatmulDesc_t desc = nullptr;
        cublasLtMatrixLayout_t la = nullptr, lb = nullptr, lc = nullptr;
        cublasLtMatmulPreference_t pref = nullptr;
        cublasStatus_t s = cublasLtMatmulDescCreate(&desc, emu ? CUBLAS_COMPUTE_32F_EMULATED_16BFX9 : CUBLAS_COMPUTE_32F, CUDA_R_32F);
        bool ok = (s == CUBLAS_STATUS_SUCCESS);
        cublasLtEpilogue_t epi = bias ? (relu ? CUBLASLT_EPILOGUE_RELU_BIAS : CUBLASLT_EPILOGUE_BIAS)
                                      : (relu ? CUBLASLT_EPILOGUE_RELU : CUBLASLT_EPILOGUE_DEFAULT);
        if (ok) ok = cublasLtMatmulDescSetAttribute(desc, CUBLASLT_MATMUL_DESC_TRANSA, &ta, sizeof(ta)) == CUBLAS_STATUS_SUCCESS;
        if (ok) ok = cublasLtMatmulDescSetAttribute(desc, CUBLASLT_MATMUL_DESC_TRANSB, &tb, sizeof(tb)) == CUBLAS_STATUS_SUCCESS;
        if (ok) ok = cublasLtMatmulDescSetAttribute(desc, CUBLASLT_MATMUL_DESC_EPILOGUE, &epi, sizeof(epi)) == CUBLAS_STATUS_SUCCESS;
        if (ok && bias) ok = cublasLtMatmulDescSetAttribute(desc, CUBLASLT_MATMUL_DESC_BIAS_POINTER, &bias, sizeof(bias)) == CUBLAS_STATUS_SUCCESS;
        if (ok) ok = cublasLtMatrixLayoutCreate(&la, CUDA_R_32F, ta == CUBLAS_OP_N ? m : k, ta == CUBLAS_OP_N ? k : m, lda) == CUBLAS_STATUS_SUCCESS;
        if (ok) ok = cublasLtMatrixLayoutCreate(&lb, CUDA_R_32F, tb == CUBLAS_OP_N ? k : n, tb == CUBLAS_OP_N ? n : k, ldb) == CUBLAS_STATUS_SUCCESS;
        if (ok) ok = cublasLtMatrixLayoutCreate(&lc, CUDA_R_32F, m, n, ldc) == CUBLAS_STATUS_SUCCESS;
        if (ok) ok = cublasLtMatmulPreferenceCreate(&pref) == CUBLAS_STATUS_SUCCESS;
        if (ok) ok = cublasLtMatmulPreferenceSetAttribute(pref, CUBLASLT_MATMUL_PREF_MAX_WORKSPACE_BYTES, &workspace_bytes, sizeof(workspace_bytes)) == CUBLAS_STATUS_SUCCESS;
        cublasLtMatmulHeuristicResult_t heur;
        int found = 0;
        if (ok) ok = cublasLtMatmulAlgoGetHeuristic(handle, desc, la, lb, lc, lc, pref, 1, &heur, &found) == CUBLAS_STATUS_SUCCESS && found > 0;
        const float one = 1.f, zero = 0.f;
        if (ok) {
            s = cublasLtMatmul(handle, desc, &one, A, la, B, lb, &zero, C, lc, C, lc, &heur.algo, workspace, workspace_bytes, st);
            ok = (s == CUBLAS_STATUS_SUCCESS);
        }
        if (pref) cublasLtMatmulPreferenceDestroy(pref);
        if (la) cublasLtMatrixLayoutDestroy(la);
        if (lb) cublasLtMatrixLayoutDestroy(lb);
        if (lc) cublasLtMatrixLayoutDestroy(lc);
        if (desc) cublasLtMatmulDescDestroy(desc);
        if (ok) {
            if (emu) emulation = 1;
            g_launches.fetch_add(1, std::memory_order_relaxed);
            return GNNB_OK;
        }
        if (emu) { emulation = 0; continue; }       // retry once with the plain fp32 compute type
        GNNB_FAIL(GNNB_ECUDA, "cublasLtMatmul failed (m=%lld n=%lld k=%lld, status %d)", (long long)m, (long long)n, (long long)k, (int)s);
    }
    GNNB_FAIL(GNNB_ECUDA, "cublasLtMatmul: no usable algorithm");
}
}  // namespace lt

int linear_tf32x3(const float* x, const float* W, const float* bias, int relu, int64_t M, int64_t K, int64_t Nout, float* y,
                  cudaStream_t st);   // dense_tc.cu
int linear_tf32x3_ex(const float* x, const float* W, int64_t ldw, const float* bias, const float* addend, int relu, int64_t M,
                     int64_t K, int64_t Nout, float* y, cudaStream_t st);
int linear_tf32x3_error();
int dw_tf32x3(const float* dpre, const float* x, int64_t M, int64_t Din, int64_t Dout, float* dW, cudaStream_t st);
int linear_relu_mask_tf32x3(const float* x, const float* W, const float* bias, int64_t M, int64_t K, float* y, uint32_t* mask,
                            cudaStream_t st);
int linear_bwd_tf32x3(const float* dy, const float* y, const uint32_t* mask, const float* x, const float* W, int64_t M,
                      int64_t Din, float* dx, float* dW, float* db, cudaStream_t st);
extern int g_tc_enabled;

__global__ void transpose_small_kernel(const float* __restrict__ w, int rows, int cols, float* __restrict__ wt) {
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i < rows * cols) { const int r = i / cols, c = i % cols; wt[(size_t)c * rows + r] = w[i]; }
}
// the same for a column block of a wider matrix (row stride ld), and the inverse copy of a block into such a matrix
__global__ void transpose_block_kernel(const float* __restrict__ w, int rows, int cols, int ld, float* __restrict__ wt) {
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i < rows * cols) { const int r = i / cols, c = i % cols; wt[(size_t)c * rows + r] = w[(size_t)r * ld + c]; }
}
__global__ void place_block_kernel(const float* __restrict__ blk, int rows, int cols, int ld, float* __restrict__ out) {
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i < rows * cols) { const int r = i / cols, c = i % cols; out[(size_t)r * ld + c] = blk[i]; }
}

// y = act(x + bias): the layers' closing `σ.(x .+ bias)` when no GEMM epilogue can carry it (GATConv, conv.jl:149)
template <int RELU>
__global__ void __launch_bounds__(256) bias_act_kernel(const float* __restrict__ x, const float* __restrict__ bias, int64_t nvec,
                                                       int nv, float* __restrict__ y) {
    const int64_t stride = (int64_t)gridDim.x * blockDim.x;
    for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < nvec; i += stride) {
        float4 v = __ldcs(reinterpret_cast<const float4*>(x) + i);
        if (bias) {
            const float4 b = __ldg(reinterpret_cast<const float4*>(bias) + (int)(i % nv));
            v.x += b.x; v.y += b.y; v.z += b.z; v.w += b.w;
        }
        if (RELU) { v.x = fmax_nan(v.x, 0.f); v.y = fmax_nan(v.y, 0.f); v.z = fmax_nan(v.z, 0.f); v.w = fmax_nan(v.w, 0.f); }
        reinterpret_cast<float4*>(y)[i] = v;
    }
}

// dpre = dy * (y > 0) (relu pullback, y = forward output) or dpre = dy; partial column sums per block for db
template <int RELU>
__global__ void __launch_bounds__(256) act_bwd_kernel(const float* __restrict__ dy, const float* __restrict__ y, int64_t n,
                                                      int D, float* __restrict__ dpre, float* __restrict__ partial,
                                                      int rows_per_block) {
    // thread t owns float4 column group (t % (D/4)); D/4 threads cover a row; 256/(D/4) rows per sweep
    const int nv = D >> 2;
    const int cg = threadIdx.x % nv;
    const int rsub = threadIdx.x / nv;
    const int rstep = blockDim.x / nv;
    const int64_t r0 = (int64_t)blockIdx.x * rows_per_block;
    const int64_t r1 = (r0 + rows_per_block < n) ? r0 + rows_per_block : n;
    float4 acc = make_float4(0.f, 0.f, 0.f, 0.f);
    if (rsub < rstep) {
        for (int64_t r = r0 + rsub; r < r1; r += rstep) {
            const float4 g = __ldg(reinterpret_cast<const float4*>(dy + r * D) + cg);
            float4 o = g;
            if (RELU) {
                const float4 v = __ldg(reinterpret_cast<const float4*>(y + r * D) + cg);
                o.x = v.x > 0.f ? g.x : 0.f; o.y = v.y > 0.f ? g.y : 0.f;
                o.z = v.z > 0.f ? g.z : 0.f; o.w = v.w > 0.f ? g.w : 0.f;
                reinterpret_cast<float4*>(dpre + r * D)[cg] = o;
            }
            acc.x += o.x; acc.y += o.y; acc.z += o.z; acc.w += o.w;
        }
    }
    __shared__ float4 sm[256];
    sm[threadIdx.x] = acc;
    __syncthreads();
    if (rsub == 0) {
        for (int q = 1; q < rstep; ++q) {
            const float4 o = sm[q * nv + cg];
            acc.x += o.x; acc.y += o.y; acc.z += o.z; acc.w += o.w;
        }
        if (partial) reinterpret_cast<float4*>(partial + (size_t)blockIdx.x * D)[cg] = acc;
    }
}
__global__ void colsum_final_kernel(const float* __restrict__ partial, int nblocks, int D, float* __restrict__ db) {
    const int c = blockIdx.x * blockDim.x + threadIdx.x;
    if (c >= D) return;
    float acc = 0.f;
    for (int b = 0; b < nblocks; ++b) acc += partial[(size_t)b * D + c];   // fixed order: deterministic
    db[c] = acc;
}

// the final pass of the two-stage column sum over partials written by other kernels (recurrent.cu's peephole gradient)
int colsum_final(const float* partial, int nblocks, int64_t D, float* out, cudaStream_t st) {
    colsum_final_kernel<<<(unsigned)ceil_div(D, 128), 128, 0, st>>>(partial, nblocks, (int)D, out);
    GNNB_LAUNCHED();
    return GNNB_OK;
}

}  // namespace gnnb

using namespace gnnb;

extern "C" {

int gnnb_dense_set_tensor_core_kernel(int on) { g_tc_enabled = on ? 1 : 0; return GNNB_OK; }
int gnnb_dense_tc_error(void) { return linear_tf32x3_error(); }
int gnnb_dense_set_emulation(int on) { lt::want_emulation = on ? 1 : 0; if (on && lt::emulation == 0) lt::emulation = -1; return GNNB_OK; }
int gnnb_dense_emulation_active(void) { return lt::want_emulation ? lt::emulation : 0; }

int gnnb_linear(const float* x, const float* W, const float* bias, int relu, int64_t N, int64_t Din, int64_t Dout,
                float* y, void* stream) {
    if (N < 0 || Din <= 0 || Dout <= 0) GNNB_FAIL(GNNB_ESIZE, "bad sizes");
    if (N == 0) return GNNB_OK;
    if (!x || !W || !y) GNNB_FAIL(GNNB_EINVAL, "NULL argument");
    {   // hand-written wgmma 3xTF32 kernels (dense_tc.cu) for the shapes they cover; cuBLASLt for every other shape
        const int rc = linear_tf32x3(x, W, bias, relu, N, Din, Dout, y, (cudaStream_t)stream);
        if (rc != GNNB_EUNSUPPORTED) return rc;
    }
    // column-major: Y(Dout x N) = W(Dout x Din) X(Din x N); W is stored (Dout, Din) row-major = col-major (Din x Dout)
    return lt::matmul(CUBLAS_OP_T, CUBLAS_OP_N, Dout, N, Din, W, Din, x, Din, y, Dout, bias, relu, (cudaStream_t)stream);
}

// σ.(W * vcat(x1, x2) .+ b) without the vcat: the two column blocks of W hit x1 and x2 in two accumulating passes of the
// wgmma kernel (the second adds the first's result before the activation).  sage_conv, conv.jl:281.
int gnnb_linear2(const float* x1, const float* x2, const float* W, const float* bias, int relu, int64_t N, int64_t Din1,
                 int64_t Din2, int64_t Dout, float* y, void* stream) {
    if (N < 0 || Din1 <= 0 || Din2 <= 0 || Dout <= 0) GNNB_FAIL(GNNB_ESIZE, "bad sizes");
    if (N == 0) return GNNB_OK;
    if (!x1 || !x2 || !W || !y) GNNB_FAIL(GNNB_EINVAL, "NULL argument");
    cudaStream_t st = (cudaStream_t)stream;
    const int64_t ld = Din1 + Din2;
    int rc = linear_tf32x3_ex(x1, W, ld, nullptr, nullptr, 0, N, Din1, Dout, y, st);
    if (rc == GNNB_EUNSUPPORTED) GNNB_FAIL(GNNB_EUNSUPPORTED, "linear2: both input widths must be multiples of 32 <= 128, Dout a multiple of 16 <= 128, 16 B-aligned operands");
    if (rc != GNNB_OK) return rc;
    rc = linear_tf32x3_ex(x2, W + Din1, ld, bias, y, relu, N, Din2, Dout, y, st);
    if (rc == GNNB_EUNSUPPORTED) GNNB_FAIL(GNNB_EUNSUPPORTED, "linear2: unsupported second block");
    return rc;
}

int gnnb_linear2_bwd(const float* dy, const float* y, const float* x1, const float* x2, const float* W, int relu, int64_t N,
                     int64_t Din1, int64_t Din2, int64_t Dout, float* dpre_ws, float* dx1, float* dx2, float* dW, float* db,
                     void* stream) {
    if (N < 0 || Din1 <= 0 || Din2 <= 0 || Dout <= 0) GNNB_FAIL(GNNB_ESIZE, "bad sizes");
    cudaStream_t st = (cudaStream_t)stream;
    const int64_t ld = Din1 + Din2;
    if (N == 0) {
        if (dW) GNNB_CUDA(cudaMemsetAsync(dW, 0, sizeof(float) * (size_t)(ld * Dout), st));
        if (db) GNNB_CUDA(cudaMemsetAsync(db, 0, sizeof(float) * (size_t)Dout, st));
        return GNNB_OK;
    }
    if (!dy || !W || !x1 || !x2) GNNB_FAIL(GNNB_EINVAL, "NULL argument");
    if (relu && (!y || !dpre_ws)) GNNB_FAIL(GNNB_EINVAL, "relu pullback needs the forward output and a (N,Dout) workspace");
    if (Dout != 128 || Din1 % 32 || Din2 % 32 || Din1 > 128 || Din2 > 128)
        GNNB_FAIL(GNNB_EUNSUPPORTED, "linear2_bwd: Dout must be 128 and both input widths multiples of 32 <= 128");
    // dpre = dy .* (y > 0), db: one pass (gnnb_linear_bwd's own, with no GEMM outputs requested)
    const float* dpre = dy;
    if (relu || db) {
        GNNB_TRY(gnnb_linear_bwd(dy, y, nullptr, W, relu, N, Din1, Dout, dpre_ws, nullptr, nullptr, db, stream));
        if (relu) dpre = dpre_ws;
    }
    DeviceState* s = nullptr;
    GNNB_TRY(device_state(&s));
    GNNB_TRY(grow_buffer(&s->w_blk, &s->w_blk_bytes, sizeof(float) * 128 * 128));
    float* tmp = s->w_blk;                             // 128x128 transposed block / dW block
    for (int blk = 0; blk < 2; ++blk) {
        const int64_t Din = blk ? Din2 : Din1;
        const float* Wb = W + (blk ? Din1 : 0);
        float* dx = blk ? dx2 : dx1;
        if (dx) {                                      // dx = dpre * W_block
            transpose_block_kernel<<<(unsigned)ceil_div(Dout * Din, 256), 256, 0, st>>>(Wb, (int)Dout, (int)Din, (int)ld, tmp);
            GNNB_LAUNCHED();
            const int rc = linear_tf32x3(dpre, tmp, nullptr, 0, N, Dout, Din, dx, st);
            if (rc != GNNB_OK) { if (rc == GNNB_EUNSUPPORTED) GNNB_FAIL(GNNB_EUNSUPPORTED, "linear2_bwd: dx shape not covered"); return rc; }
        }
        if (dW) {                                      // dW_block = dpre' * x_block, placed into its columns of dW
            const int rc = dw_tf32x3(dpre, blk ? x2 : x1, N, Din, Dout, tmp, st);
            if (rc != GNNB_OK) { if (rc == GNNB_EUNSUPPORTED) GNNB_FAIL(GNNB_EUNSUPPORTED, "linear2_bwd: dW shape not covered"); return rc; }
            place_block_kernel<<<(unsigned)ceil_div(Dout * Din, 256), 256, 0, st>>>(tmp, (int)Dout, (int)Din, (int)ld, dW + (blk ? Din1 : 0));
            GNNB_LAUNCHED();
        }
    }
    return GNNB_OK;
}

// the relu mask x upstream gradient and the deterministic two-stage bias gradient, one pass over dy (and y)
static int act_bwd_launch(const float* dy, const float* y, int relu, int64_t N, int64_t D, float* dpre, float* db, cudaStream_t st) {
    // about 8 CTAs per SM worth of blocks: long row runs per block keep the deterministic final pass short
    int64_t rpb = ceil_div(N, kNumSMs * 8);
    const int rows_per_block = (int)(rpb < 64 ? 64 : rpb);
    const int nblocks = (int)ceil_div(N, rows_per_block);
    float* partial = nullptr;
    if (db) {
        DeviceState* s = nullptr;
        GNNB_TRY(device_state(&s));
        GNNB_TRY(grow_buffer(&s->act_part, &s->act_part_bytes, sizeof(float) * (size_t)nblocks * D));
        partial = s->act_part;
    }
    if (relu) act_bwd_kernel<1><<<nblocks, 256, 0, st>>>(dy, y, N, (int)D, dpre, partial, rows_per_block);
    else act_bwd_kernel<0><<<nblocks, 256, 0, st>>>(dy, y, N, (int)D, nullptr, partial, rows_per_block);
    GNNB_LAUNCHED();
    if (db) { colsum_final_kernel<<<(unsigned)ceil_div(D, 128), 128, 0, st>>>(partial, nblocks, (int)D, db); GNNB_LAUNCHED(); }
    return GNNB_OK;
}

int gnnb_bias_act(const float* x, const float* bias, int relu, int64_t N, int64_t D, float* y, void* stream) {
    if (N < 0 || D <= 0) GNNB_FAIL(GNNB_ESIZE, "bad sizes");
    if (N == 0) return GNNB_OK;
    if (!x || !y) GNNB_FAIL(GNNB_EINVAL, "NULL argument");
    if (D % 4 != 0 || ((uintptr_t)x & 15) || ((uintptr_t)y & 15) || (bias && ((uintptr_t)bias & 15)))
        GNNB_FAIL(GNNB_EUNSUPPORTED, "bias_act: D must be a multiple of 4 and pointers 16 B aligned");
    cudaStream_t st = (cudaStream_t)stream;
    const int64_t nvec = N * (D / 4);
    const unsigned grid = (unsigned)(ceil_div(nvec, 256) < kNumSMs * 16 ? ceil_div(nvec, 256) : kNumSMs * 16);
    if (relu) bias_act_kernel<1><<<grid, 256, 0, st>>>(x, bias, nvec, (int)(D / 4), y);
    else bias_act_kernel<0><<<grid, 256, 0, st>>>(x, bias, nvec, (int)(D / 4), y);
    GNNB_LAUNCHED();
    return GNNB_OK;
}

int gnnb_bias_act_bwd(const float* dy, const float* y, int relu, int64_t N, int64_t D, float* dpre, float* db, void* stream) {
    if (N < 0 || D <= 0) GNNB_FAIL(GNNB_ESIZE, "bad sizes");
    cudaStream_t st = (cudaStream_t)stream;
    if (N == 0) { if (db) GNNB_CUDA(cudaMemsetAsync(db, 0, sizeof(float) * (size_t)D, st)); return GNNB_OK; }
    if (!dy || (relu && (!y || !dpre))) GNNB_FAIL(GNNB_EINVAL, "NULL argument");
    if (!relu && !db) return GNNB_OK;
    if (D % 4 != 0 || D > 1024 || ((uintptr_t)dy & 15) || (relu && (((uintptr_t)y & 15) || ((uintptr_t)dpre & 15))))
        GNNB_FAIL(GNNB_EUNSUPPORTED, "bias_act_bwd: D must be a multiple of 4 (<= 1024) and pointers 16 B aligned");
    return act_bwd_launch(dy, y, relu, N, D, dpre, db, st);
}

int gnnb_linear_bwd(const float* dy, const float* y, const float* x, const float* W, int relu, int64_t N, int64_t Din,
                    int64_t Dout, float* dpre_ws, float* dx, float* dW, float* db, void* stream) {
    if (N < 0 || Din <= 0 || Dout <= 0) GNNB_FAIL(GNNB_ESIZE, "bad sizes");
    cudaStream_t st = (cudaStream_t)stream;
    if (N == 0) {   // empty batch: zero parameter gradients, nothing else to do
        if (dW) GNNB_CUDA(cudaMemsetAsync(dW, 0, sizeof(float) * (size_t)(Din * Dout), st));
        if (db) GNNB_CUDA(cudaMemsetAsync(db, 0, sizeof(float) * (size_t)Dout, st));
        return GNNB_OK;
    }
    if (!dy || !W) GNNB_FAIL(GNNB_EINVAL, "NULL argument");
    if (relu && (!y || !dpre_ws)) GNNB_FAIL(GNNB_EINVAL, "relu pullback needs the forward output and a (N,Dout) workspace");
    if (dx && dW && x && Dout == 128) {   // the fused pullback: dpre stays on chip, dpre_ws is not touched
        const int rc = linear_bwd_tf32x3(dy, relu ? y : nullptr, nullptr, x, W, N, Din, dx, dW, db, st);
        if (rc != GNNB_EUNSUPPORTED) return rc;
    }
    const float* dpre = dy;
    if ((relu || db) && N > 0) {
        if (Dout % 4 != 0 || Dout > 1024 || ((uintptr_t)dy & 15) || (relu && (((uintptr_t)y & 15) || ((uintptr_t)dpre_ws & 15))))
            GNNB_FAIL(GNNB_EUNSUPPORTED, "linear_bwd: Dout must be a multiple of 4 (<= 1024) and pointers 16 B aligned");
        GNNB_TRY(act_bwd_launch(dy, y, relu, N, Dout, dpre_ws, db, st));
        if (relu) dpre = dpre_ws;
    } else if (db && N == 0) {
        GNNB_CUDA(cudaMemsetAsync(db, 0, sizeof(float) * Dout, st));
    }
    // dX = dPre * W : rows of dPre (K = Dout) against W^T stored K-major => the same wgmma kernel on a transposed copy of W
    if (dx && g_tc_enabled && Dout % 32 == 0 && Dout <= 128 && Din % 16 == 0 && Din <= 128 && Din >= 16) {
        DeviceState* s = nullptr;
        GNNB_TRY(device_state(&s));
        GNNB_TRY(grow_buffer(&s->wt, &s->wt_bytes, sizeof(float) * 128 * 128));
        transpose_small_kernel<<<(unsigned)ceil_div(Dout * Din, 256), 256, 0, st>>>(W, (int)Dout, (int)Din, s->wt);
        GNNB_LAUNCHED();
        const int rc = linear_tf32x3(dpre, s->wt, nullptr, 0, N, Dout, Din, dx, st);
        if (rc == GNNB_OK) dx = nullptr;
        else if (rc != GNNB_EUNSUPPORTED) return rc;
    } else if (dx && g_tc_enabled && (Dout > 128 || Din > 128) && Dout % 32 == 0 && Dout <= 512 && Din % 128 == 0 && Din <= 1024 &&
               N >= 2048) {
        // wide shapes: the same product through the wide wgmma kernel on a transposed copy of W (<= 8 MB, kept)
        DeviceState* s = nullptr;
        GNNB_TRY(device_state(&s));
        GNNB_TRY(grow_buffer(&s->wt_wide, &s->wt_wide_bytes, sizeof(float) * (size_t)(Dout * Din)));
        transpose_small_kernel<<<(unsigned)ceil_div(Dout * Din, 256), 256, 0, st>>>(W, (int)Dout, (int)Din, s->wt_wide);
        GNNB_LAUNCHED();
        const int rc = linear_tf32x3(dpre, s->wt_wide, nullptr, 0, N, Dout, Din, dx, st);
        if (rc == GNNB_OK) dx = nullptr;
        else if (rc != GNNB_EUNSUPPORTED) return rc;
    }
    // dX(Din x N) = W^T-as-stored(Din x Dout) dPre(Dout x N)
    if (dx) GNNB_TRY(lt::matmul(CUBLAS_OP_N, CUBLAS_OP_N, Din, N, Dout, W, Din, dpre, Dout, dx, Din, nullptr, 0, st));
    // dW row-major (Dout, Din) = col-major (Din x Dout) = X(Din x N) dPre^T(N x Dout)
    if (dW) {
        if (!x) GNNB_FAIL(GNNB_EINVAL, "dW needs x");
        const int rc = dw_tf32x3(dpre, x, N, Din, Dout, dW, st);      // wgmma, transposing producers, split-K
        if (rc == GNNB_OK) return GNNB_OK;
        if (rc != GNNB_EUNSUPPORTED) return rc;
        GNNB_TRY(lt::matmul(CUBLAS_OP_N, CUBLAS_OP_T, Din, Dout, N, x, Din, dpre, Dout, dW, Din, nullptr, 0, st));
    }
    return GNNB_OK;
}

int gnnb_linear_relu_mask(const float* x, const float* W, const float* bias, int64_t N, int64_t Din, int64_t Dout, float* y,
                          uint32_t* mask, void* stream) {
    if (N < 0 || Din <= 0 || Dout <= 0) GNNB_FAIL(GNNB_ESIZE, "bad sizes");
    if (Dout != 128) GNNB_FAIL(GNNB_EUNSUPPORTED, "linear_relu_mask: Dout must be 128");
    if (N > 0 && (!x || !W || !y || !mask)) GNNB_FAIL(GNNB_EINVAL, "NULL argument");
    const int rc = linear_relu_mask_tf32x3(x, W, bias, N, Din, y, mask, (cudaStream_t)stream);
    if (rc == GNNB_EUNSUPPORTED)
        GNNB_FAIL(GNNB_EUNSUPPORTED, "linear_relu_mask: Din must be 32, 64, 96 or 128, operands 16 B aligned, tensor-core kernels on");
    return rc;
}

int gnnb_linear_bwd_mask(const float* dy, const uint32_t* mask, const float* x, const float* W, int64_t N, int64_t Din,
                         int64_t Dout, float* dx, float* dW, float* db, void* stream) {
    if (N < 0 || Din <= 0 || Dout <= 0) GNNB_FAIL(GNNB_ESIZE, "bad sizes");
    if (Dout != 128 || Din % 32 != 0 || Din > 128 || !g_tc_enabled)
        GNNB_FAIL(GNNB_EUNSUPPORTED, "linear_bwd_mask: Dout must be 128, Din 32, 64, 96 or 128, tensor-core kernels on");
    // dx of an empty batch has no element (torch hands over NULL for it: a rank that owns no node)
    if ((!dx && N > 0) || !dW) GNNB_FAIL(GNNB_EINVAL, "linear_bwd_mask computes dx and dW together: both are required");
    cudaStream_t st = (cudaStream_t)stream;
    if (N == 0) {
        GNNB_CUDA(cudaMemsetAsync(dW, 0, sizeof(float) * (size_t)(Din * Dout), st));
        if (db) GNNB_CUDA(cudaMemsetAsync(db, 0, sizeof(float) * (size_t)Dout, st));
        return GNNB_OK;
    }
    if (!dy || !mask || !x || !W) GNNB_FAIL(GNNB_EINVAL, "NULL argument");
    const int rc = linear_bwd_tf32x3(dy, nullptr, mask, x, W, N, Din, dx, dW, db, st);
    if (rc == GNNB_EUNSUPPORTED) GNNB_FAIL(GNNB_EUNSUPPORTED, "linear_bwd_mask: operands must be 16 B aligned");
    return rc;
}

}  // extern "C"
