// mbarrier / TMA (cp.async.bulk.tensor) / tensor-map helpers shared by the sm_90a kernels.
#pragma once
#include "common.cuh"
#include <cuda.h>

namespace tma {

__device__ __forceinline__ uint32_t smem_u32(const void* p) { return (uint32_t)__cvta_generic_to_shared(p); }

__device__ __forceinline__ void mbar_init(uint64_t* bar, uint32_t count) {
    asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(smem_u32(bar)), "r"(count));
}
__device__ __forceinline__ void fence_barrier_init() { asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory"); }
__device__ __forceinline__ void fence_proxy_async() { asm volatile("fence.proxy.async.shared::cta;" ::: "memory"); }
__device__ __forceinline__ void mbar_expect_tx(uint64_t* bar, uint32_t bytes) {
    asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(smem_u32(bar)), "r"(bytes) : "memory");
}
__device__ __forceinline__ void mbar_arrive(uint64_t* bar) {
    asm volatile("mbarrier.arrive.shared::cta.b64 _, [%0];" ::"r"(smem_u32(bar)) : "memory");
}
__device__ __forceinline__ void mbar_wait(uint64_t* bar, uint32_t parity) {
    const uint32_t addr = smem_u32(bar);
    uint32_t done;
    uint32_t spins = 0;
    do {
        // a lost TMA / MMA completion must surface as a launch failure, never as a hung GPU
        if (++spins > (1u << 26)) __trap();
        asm volatile(
            "{\n\t.reg .pred p;\n\t"
            "mbarrier.try_wait.parity.shared::cta.b64 p, [%1], %2;\n\t"
            "selp.u32 %0, 1, 0, p;\n\t}"
            : "=r"(done)
            : "r"(addr), "r"(parity)
            : "memory");
    } while (!done);
}
__device__ __forceinline__ bool elect_one() {
    uint32_t pred;
    asm volatile(
        "{\n\t.reg .pred p;\n\t"
        "elect.sync _|p, 0xffffffff;\n\t"
        "selp.u32 %0, 1, 0, p;\n\t}"
        : "=r"(pred));
    return pred != 0;
}
__device__ __forceinline__ void prefetch_map(const CUtensorMap* m) {
    asm volatile("prefetch.tensormap [%0];" ::"l"(m) : "memory");
}
__device__ __forceinline__ void load_2d(void* smem_dst, const CUtensorMap* map, uint64_t* bar, int c0, int c1) {
    asm volatile(
        "cp.async.bulk.tensor.2d.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1, {%3, %4}], [%2];"
        ::"r"(smem_u32(smem_dst)), "l"(map), "r"(smem_u32(bar)), "r"(c0), "r"(c1)
        : "memory");
}
// L2 eviction-priority hint for bulk tensor loads (the encoding createpolicy.fractional.L2::evict_first produces with fraction 1.0):
// KV-cache streams are read once per step. hint == 0 keeps the default policy, which the weight tiles use.
constexpr uint64_t kL2EvictFirst = 0x12F0000000000000ull;
__device__ __forceinline__ void load_2d_hint(void* smem_dst, const CUtensorMap* map, uint64_t* bar, int c0, int c1, uint64_t hint) {
    if (hint == 0) {
        load_2d(smem_dst, map, bar, c0, c1);
    } else {
        asm volatile(
            "cp.async.bulk.tensor.2d.shared::cluster.global.mbarrier::complete_tx::bytes.L2::cache_hint [%0], [%1, {%3, %4}], [%2], %5;"
            ::"r"(smem_u32(smem_dst)), "l"(map), "r"(smem_u32(bar)), "r"(c0), "r"(c1), "l"(hint)
            : "memory");
    }
}
__device__ __forceinline__ void load_4d(void* smem_dst, const CUtensorMap* map, uint64_t* bar, int c0, int c1, int c2, int c3) {
    asm volatile(
        "cp.async.bulk.tensor.4d.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1, {%3, %4, %5, %6}], [%2];"
        ::"r"(smem_u32(smem_dst)), "l"(map), "r"(smem_u32(bar)), "r"(c0), "r"(c1), "r"(c2), "r"(c3)
        : "memory");
}

// host: 2-D row-major [rows, cols] of a 16-bit LG_DTYPE_* (bf16 or fp16; cols contiguous, `ld_elems` between rows); box
// [box_rows, box_cols]; 128-byte swizzle (box_cols * 2 bytes must be <= 128); out-of-bounds elements read as zero.
int make_map_2d(CUtensorMap* m, const void* base, uint64_t rows, uint64_t cols, uint64_t ld_elems, uint32_t box_rows,
                uint32_t box_cols, int dtype = LG_DTYPE_BF16);
// host: 4-D bf16 NHWC activation [B, H, W, C]; box [1, box_h, box_w, box_c]; 128-byte swizzle; OOB -> zero
// (signed start coordinates give the conv's zero padding for free).
int make_map_nhwc(CUtensorMap* m, const void* base, uint64_t B, uint64_t H, uint64_t W, uint64_t C, uint32_t box_h,
                  uint32_t box_w, uint32_t box_c, uint32_t pixel_stride = 1);

}  // namespace tma
