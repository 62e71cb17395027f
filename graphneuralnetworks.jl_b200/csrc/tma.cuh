// tma.cuh — tensor maps (cuTensorMapEncodeTiled through the runtime's driver-entry-point query: no link against libcuda)
// and the device-side wrappers of the TMA instructions this library issues: mbarrier transaction counting and
// cp.async.bulk.tensor.2d ... tile (one box of a 2-D tensor per request).
#pragma once
#include <cuda.h>
#include <cuda_runtime.h>
#include <stdint.h>

namespace gnnb {
namespace tma {

typedef CUresult (*EncodeTiledFn)(CUtensorMap*, CUtensorMapDataType, cuuint32_t, void*, const cuuint64_t*, const cuuint64_t*,
                                  const cuuint32_t*, const cuuint32_t*, CUtensorMapInterleave, CUtensorMapSwizzle,
                                  CUtensorMapL2promotion, CUtensorMapFloatOOBfill);

inline EncodeTiledFn encode_fn() {
    static EncodeTiledFn fn = [] {
        void* p = nullptr;
        cudaDriverEntryPointQueryResult q;
        if (cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &p, cudaEnableDefault, &q) != cudaSuccess ||
            q != cudaDriverEntryPointSuccess)
            p = nullptr;
        return (EncodeTiledFn)p;
    }();
    return fn;
}

// fp32 row-major matrix [rows][cols] (row stride in bytes, a multiple of 16), box = box_cols x box_rows elements, no swizzle.
// Returns 0 on success.
inline int make_map_2d_f32(CUtensorMap* m, const void* base, uint64_t rows, uint64_t cols, uint64_t row_stride_bytes,
                           uint32_t box_cols, uint32_t box_rows) {
    EncodeTiledFn fn = encode_fn();
    if (!fn) return -1;
    const cuuint64_t dims[2] = {cols, rows};
    const cuuint64_t strides[1] = {row_stride_bytes};
    const cuuint32_t box[2] = {box_cols, box_rows};
    const cuuint32_t estr[2] = {1, 1};
    const CUresult r = fn(m, CU_TENSOR_MAP_DATA_TYPE_FLOAT32, 2, const_cast<void*>(base), dims, strides, box, estr,
                          CU_TENSOR_MAP_INTERLEAVE_NONE, CU_TENSOR_MAP_SWIZZLE_NONE, CU_TENSOR_MAP_L2_PROMOTION_L2_128B,
                          CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
    return r == CUDA_SUCCESS ? 0 : (int)r;
}

__device__ __forceinline__ uint32_t smem_u32(const void* p) { return (uint32_t)__cvta_generic_to_shared(p); }
__device__ __forceinline__ void mbar_init(uint32_t bar, uint32_t count) {
    asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(bar), "r"(count) : "memory");
}
__device__ __forceinline__ void mbar_expect_tx(uint32_t bar, uint32_t bytes) {
    asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(bar), "r"(bytes) : "memory");
}
__device__ __forceinline__ bool mbar_try(uint32_t bar, uint32_t parity) {
    uint32_t ok;
    asm volatile("{\n\t.reg .pred p;\n\tmbarrier.try_wait.parity.shared::cta.b64 p, [%1], %2;\n\tselp.u32 %0, 1, 0, p;\n\t}"
                 : "=r"(ok) : "r"(bar), "r"(parity) : "memory");
    return ok != 0;
}
// bounded wait on phase `parity`: false if it never completes (then *err is raised) or if another thread already raised
// *err; a broken pipeline reports a status instead of hanging the kernel
__device__ __forceinline__ bool mbar_wait_bounded(uint32_t bar, uint32_t parity, int* err) {
    for (uint32_t spin = 0; spin < (1u << 26); ++spin) {
        if (mbar_try(bar, parity)) return true;
        if ((spin & 1023) == 1023 && *(volatile int*)err) return false;
    }
    atomicExch(err, 1);
    return false;
}
// columns [col, col + box_cols) of row `row` of the 2-D tensor behind `map` (box_rows = 1) into dst
__device__ __forceinline__ void load_row(uint32_t dst, const CUtensorMap* map, int col, int row, uint32_t bar) {
    asm volatile("cp.async.bulk.tensor.2d.shared::cluster.global.tile.mbarrier::complete_tx::bytes [%0], [%1, {%2, %3}], [%4];"
                 ::"r"(dst), "l"(map), "r"(col), "r"(row), "r"(bar) : "memory");
}
__device__ __forceinline__ void fence_proxy_async() { asm volatile("fence.proxy.async.shared::cta;" ::: "memory"); }
// 1-D bulk copy (cp.async.bulk, no tensor map) of `bytes` from global `src` into shared `dst`, completion counted on `bar`.
// src and dst 16 B aligned, bytes a non-zero multiple of 16.
__device__ __forceinline__ void bulk_load(uint32_t dst, const void* src, uint32_t bytes, uint32_t bar) {
    asm volatile("cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];"
                 ::"r"(dst), "l"(src), "r"(bytes), "r"(bar) : "memory");
}

}  // namespace tma
}  // namespace gnnb
