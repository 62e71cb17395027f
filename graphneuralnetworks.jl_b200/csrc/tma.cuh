// tma.cuh — device-side wrappers of the TMA instructions this library issues: mbarrier transaction counting, the 1-D
// bulk copy cp.async.bulk (no tensor map) and the 2-D tiled copy cp.async.bulk.tensor (host-encoded tensor map) from
// global into shared memory.
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>

namespace gnnb {
namespace tma {

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
__device__ __forceinline__ void fence_proxy_async() { asm volatile("fence.proxy.async.shared::cta;" ::: "memory"); }
// 1-D bulk copy (cp.async.bulk, no tensor map) of `bytes` from global `src` into shared `dst`, completion counted on `bar`.
// src and dst 16 B aligned, bytes a non-zero multiple of 16.
__device__ __forceinline__ void bulk_load(uint32_t dst, const void* src, uint32_t bytes, uint32_t bar) {
    asm volatile("cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];"
                 ::"r"(dst), "l"(src), "r"(bytes), "r"(bar) : "memory");
}
// 2-D tiled copy (cp.async.bulk.tensor) of the box at element coordinates (x0 inner, x1 outer) of the tensor map `map`
// (a __grid_constant__ kernel parameter) into shared `dst`, completion counted on `bar`.  Elements outside the tensor
// arrive as zeros and the whole box counts towards the transaction bytes.
__device__ __forceinline__ void tensor_load_2d(uint32_t dst, const void* map, int x0, int x1, uint32_t bar) {
    asm volatile("cp.async.bulk.tensor.2d.shared::cluster.global.tile.mbarrier::complete_tx::bytes [%0], [%1, {%2, %3}], [%4];"
                 ::"r"(dst), "l"(map), "r"(x0), "r"(x1), "r"(bar) : "memory");
}

}  // namespace tma
}  // namespace gnnb
