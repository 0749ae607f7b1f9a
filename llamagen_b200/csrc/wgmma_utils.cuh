// wgmma (Hopper warpgroup MMA) helpers shared by the tensor-core kernels (gemm_tc.cu, conv_tc.cu).
//
// Both operands are K-major bf16 (or fp16) tiles in shared memory written by TMA with the 128-byte swizzle: rows of 64 elements
// (128 B), 8-row groups 1024 B apart, tile bases 1024-aligned. One warpgroup (128 threads) computes a 64 x N fp32
// accumulator held in registers; thread t of the warpgroup owns, for register i of Wgmma<N>,
//   row = 16 * (warp % 4) + lane / 4 + 8 * ((i >> 1) & 1),   col = 8 * (i >> 2) + 2 * (lane % 4) + (i & 1).
#pragma once
#include "tma_utils.cuh"
#include <type_traits>

namespace wg {
using tma::smem_u32;

// GMMA shared-memory descriptor: start >> 4 [0,14), LBO >> 4 [16,30) (unused for swizzled K-major), SBO >> 4 [32,46) = 1024 B,
// layout type [62,64) = 1 (128-byte swizzle).
__device__ __forceinline__ uint64_t make_desc_sw128(uint32_t smem_addr) {
    return (uint64_t)((smem_addr >> 4) & 0x3FFF) | (1ull << 16) | (64ull << 32) | (1ull << 62);
}
__device__ __forceinline__ void fence() { asm volatile("wgmma.fence.sync.aligned;" ::: "memory"); }
__device__ __forceinline__ void commit() { asm volatile("wgmma.commit_group.sync.aligned;" ::: "memory"); }
template <int Pending>
__device__ __forceinline__ void wait() { asm volatile("wgmma.wait_group.sync.aligned %0;" ::"n"(Pending) : "memory"); }
// keeps the compiler from moving accumulator accesses across the asynchronous MMAs
template <int R>
__device__ __forceinline__ void fence_regs(float* d) {
#pragma unroll
    for (int i = 0; i < R; ++i) asm volatile("" : "+f"(d[i])::"memory");
}

// D[64 x N] += A[64 x 16] * B[N x 16]^T, both operands from shared memory; T (bf16 or f16) selects the instruction's operand
// type, everything else (layouts, swizzle, descriptors, accumulator fragments) is the same for both.
#define LG_WG_R8(o) "+f"(d[o]), "+f"(d[o + 1]), "+f"(d[o + 2]), "+f"(d[o + 3]), "+f"(d[o + 4]), "+f"(d[o + 5]), "+f"(d[o + 6]), "+f"(d[o + 7])
template <int N, typename T = bf16>
struct Wgmma;

#define LG_WG_ASM16(TY) \
    "{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %10, 0;\n\t" \
    "wgmma.mma_async.sync.aligned.m64n16k16.f32." TY "." TY " {" \
    "%0,%1,%2,%3,%4,%5,%6,%7" \
    "}, %8, %9, p, 1, 1, 0, 0;\n\t}"
template <typename T>
struct Wgmma<16, T> {
    static __device__ __forceinline__ void mma(float* d, uint64_t adesc, uint64_t bdesc) {
        if constexpr (std::is_same<T, f16>::value)
            asm volatile(LG_WG_ASM16("f16") : LG_WG_R8(0) : "l"(adesc), "l"(bdesc), "r"(1));
        else
            asm volatile(LG_WG_ASM16("bf16") : LG_WG_R8(0) : "l"(adesc), "l"(bdesc), "r"(1));
    }
};

#define LG_WG_ASM32(TY) \
    "{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %18, 0;\n\t" \
    "wgmma.mma_async.sync.aligned.m64n32k16.f32." TY "." TY " {" \
    "%0,%1,%2,%3,%4,%5,%6,%7,%8,%9,%10,%11,%12,%13,%14,%15" \
    "}, %16, %17, p, 1, 1, 0, 0;\n\t}"
template <typename T>
struct Wgmma<32, T> {
    static __device__ __forceinline__ void mma(float* d, uint64_t adesc, uint64_t bdesc) {
        if constexpr (std::is_same<T, f16>::value)
            asm volatile(LG_WG_ASM32("f16") : LG_WG_R8(0), LG_WG_R8(8) : "l"(adesc), "l"(bdesc), "r"(1));
        else
            asm volatile(LG_WG_ASM32("bf16") : LG_WG_R8(0), LG_WG_R8(8) : "l"(adesc), "l"(bdesc), "r"(1));
    }
};

#define LG_WG_ASM64(TY) \
    "{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %34, 0;\n\t" \
    "wgmma.mma_async.sync.aligned.m64n64k16.f32." TY "." TY " {" \
    "%0,%1,%2,%3,%4,%5,%6,%7,%8,%9,%10,%11,%12,%13,%14,%15,%16,%17,%18,%19,%20,%21,%22,%23,%24,%25,%26,%27,%28,%29,%30,%31" \
    "}, %32, %33, p, 1, 1, 0, 0;\n\t}"
template <typename T>
struct Wgmma<64, T> {
    static __device__ __forceinline__ void mma(float* d, uint64_t adesc, uint64_t bdesc) {
        if constexpr (std::is_same<T, f16>::value)
            asm volatile(LG_WG_ASM64("f16") : LG_WG_R8(0), LG_WG_R8(8), LG_WG_R8(16), LG_WG_R8(24) : "l"(adesc), "l"(bdesc), "r"(1));
        else
            asm volatile(LG_WG_ASM64("bf16") : LG_WG_R8(0), LG_WG_R8(8), LG_WG_R8(16), LG_WG_R8(24) : "l"(adesc), "l"(bdesc), "r"(1));
    }
};

#define LG_WG_ASM128(TY) \
    "{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %66, 0;\n\t" \
    "wgmma.mma_async.sync.aligned.m64n128k16.f32." TY "." TY " {" \
    "%0,%1,%2,%3,%4,%5,%6,%7,%8,%9,%10,%11,%12,%13,%14,%15,%16,%17,%18,%19,%20,%21,%22,%23,%24,%25,%26,%27,%28,%29,%30,%31,%32,%33,%34,%35,%36,%37,%38,%39,%40,%41,%42,%43,%44,%45,%46,%47,%48,%49,%50,%51,%52,%53,%54,%55,%56,%57,%58,%59,%60,%61,%62,%63" \
    "}, %64, %65, p, 1, 1, 0, 0;\n\t}"
template <typename T>
struct Wgmma<128, T> {
    static __device__ __forceinline__ void mma(float* d, uint64_t adesc, uint64_t bdesc) {
        if constexpr (std::is_same<T, f16>::value)
            asm volatile(LG_WG_ASM128("f16") : LG_WG_R8(0), LG_WG_R8(8), LG_WG_R8(16), LG_WG_R8(24), LG_WG_R8(32), LG_WG_R8(40), LG_WG_R8(48), LG_WG_R8(56) : "l"(adesc), "l"(bdesc), "r"(1));
        else
            asm volatile(LG_WG_ASM128("bf16") : LG_WG_R8(0), LG_WG_R8(8), LG_WG_R8(16), LG_WG_R8(24), LG_WG_R8(32), LG_WG_R8(40), LG_WG_R8(48), LG_WG_R8(56) : "l"(adesc), "l"(bdesc), "r"(1));
    }
};

#define LG_WG_ASM256(TY) \
    "{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %130, 0;\n\t" \
    "wgmma.mma_async.sync.aligned.m64n256k16.f32." TY "." TY " {" \
    "%0,%1,%2,%3,%4,%5,%6,%7,%8,%9,%10,%11,%12,%13,%14,%15,%16,%17,%18,%19,%20,%21,%22,%23,%24,%25,%26,%27,%28,%29,%30,%31,%32,%33,%34,%35,%36,%37,%38,%39,%40,%41,%42,%43,%44,%45,%46,%47,%48,%49,%50,%51,%52,%53,%54,%55,%56,%57,%58,%59,%60,%61,%62,%63,%64,%65,%66,%67,%68,%69,%70,%71,%72,%73,%74,%75,%76,%77,%78,%79,%80,%81,%82,%83,%84,%85,%86,%87,%88,%89,%90,%91,%92,%93,%94,%95,%96,%97,%98,%99,%100,%101,%102,%103,%104,%105,%106,%107,%108,%109,%110,%111,%112,%113,%114,%115,%116,%117,%118,%119,%120,%121,%122,%123,%124,%125,%126,%127" \
    "}, %128, %129, p, 1, 1, 0, 0;\n\t}"
template <typename T>
struct Wgmma<256, T> {
    static __device__ __forceinline__ void mma(float* d, uint64_t adesc, uint64_t bdesc) {
        if constexpr (std::is_same<T, f16>::value)
            asm volatile(LG_WG_ASM256("f16") : LG_WG_R8(0), LG_WG_R8(8), LG_WG_R8(16), LG_WG_R8(24), LG_WG_R8(32), LG_WG_R8(40), LG_WG_R8(48), LG_WG_R8(56), LG_WG_R8(64), LG_WG_R8(72), LG_WG_R8(80), LG_WG_R8(88), LG_WG_R8(96), LG_WG_R8(104), LG_WG_R8(112), LG_WG_R8(120) : "l"(adesc), "l"(bdesc), "r"(1));
        else
            asm volatile(LG_WG_ASM256("bf16") : LG_WG_R8(0), LG_WG_R8(8), LG_WG_R8(16), LG_WG_R8(24), LG_WG_R8(32), LG_WG_R8(40), LG_WG_R8(48), LG_WG_R8(56), LG_WG_R8(64), LG_WG_R8(72), LG_WG_R8(80), LG_WG_R8(88), LG_WG_R8(96), LG_WG_R8(104), LG_WG_R8(112), LG_WG_R8(120) : "l"(adesc), "l"(bdesc), "r"(1));
    }
};

// one 64-wide k-block: A = 64 rows at a_addr, B = N rows at b_addr; four K = 16 steps advance 32 bytes inside the
// swizzle span (+2 in the address field). Issue only: the caller commits and waits.
template <int N, typename T = bf16>
__device__ __forceinline__ void mma_kblock(float* d, uint32_t a_addr, uint32_t b_addr) {
    const uint64_t ad = make_desc_sw128(a_addr), bd = make_desc_sw128(b_addr);
#pragma unroll
    for (int k = 0; k < 4; ++k) Wgmma<N, T>::mma(d, ad + (uint64_t)(2 * k), bd + (uint64_t)(2 * k));
}

__device__ __forceinline__ int frag_row(int i) { return 16 * (((int)threadIdx.x >> 5) & 3) + (((int)threadIdx.x & 31) >> 2) + 8 * ((i >> 1) & 1); }
__device__ __forceinline__ int frag_col(int i) { return 8 * (i >> 2) + 2 * ((int)threadIdx.x & 3) + (i & 1); }

// named barrier over the two consumer warpgroups (threads 0..255) that leaves the producer warp out
__device__ __forceinline__ void consumer_sync() { asm volatile("bar.sync 1, 256;" ::: "memory"); }

}  // namespace wg
