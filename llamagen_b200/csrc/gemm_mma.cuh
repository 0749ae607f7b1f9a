// bf16 / fp16 tensor-core GEMM main loop, C[M,N] = A[M,K] * B[N,K]^T, fp32 accumulate (round-1 workhorse:
// mma.sync m16n8k16 fed by a multi-stage cp.async pipeline; BK = 64 so every shared-memory row is one
// 128-byte line, XOR-swizzled by (row & 7) -> conflict-free cp.async stores and ldmatrix loads).
//
// The A operand comes through a loader functor so the same loop serves
//   * dense activations (transformer GEMMs, VQ attention batched GEMMs), and
//   * implicit-GEMM convolution over NHWC activations (zero padding and the nearest-2x upsample of
//     vq_model.py:374-378 are folded into the address computation, nothing is materialised).
// The epilogue is a functor called with two adjacent output columns (n, n+1) of one row.
// T (bf16 by default, f16 for fp16 transformers) only selects the MMA operand type: loads move raw 16-bit elements, so the
// loaders address fp16 tensors through the same bf16-typed pointers.
#pragma once
#include "common.cuh"

namespace mma {

constexpr int BK = 64;          // bf16 elements per k-tile = 128 bytes
constexpr int kThreads = 256;

__device__ __forceinline__ uint32_t smem_u32(const void* p) { return (uint32_t)__cvta_generic_to_shared(p); }

__device__ __forceinline__ void cp_async16(uint32_t dst, const void* src, bool valid) {
    const int sz = valid ? 16 : 0;
    asm volatile("cp.async.cg.shared.global [%0], [%1], 16, %2;\n" ::"r"(dst), "l"(src), "r"(sz));
}
__device__ __forceinline__ void cp_async_commit() { asm volatile("cp.async.commit_group;\n" ::); }
template <int N> __device__ __forceinline__ void cp_async_wait() { asm volatile("cp.async.wait_group %0;\n" ::"n"(N)); }

__device__ __forceinline__ void ldmatrix_x4(uint32_t addr, uint32_t& r0, uint32_t& r1, uint32_t& r2, uint32_t& r3) {
    asm volatile("ldmatrix.sync.aligned.m8n8.x4.shared.b16 {%0,%1,%2,%3}, [%4];\n"
                 : "=r"(r0), "=r"(r1), "=r"(r2), "=r"(r3) : "r"(addr));
}

// byte offset of 16-byte chunk `c` (0..7) of row `r` inside a [rows][128 B] swizzled tile
__device__ __forceinline__ uint32_t swz(int r, int c) { return (uint32_t)(r * 128 + ((c ^ (r & 7)) << 4)); }

// ---------------------------------------------------------------- A loaders
struct DenseA {
    const bf16* X;
    long long ldx;           // elements between rows
    long long batch_stride;  // elements between batches (0 = shared)
    int M;
    struct Row { const bf16* p; };
    __device__ __forceinline__ Row row(int m, int bz) const {
        Row r;
        r.p = m < M ? X + (long long)bz * batch_stride + (long long)m * ldx : nullptr;
        return r;
    }
    __device__ __forceinline__ const bf16* ptr(const Row& r, int k) const { return r.p ? r.p + k : nullptr; }
};

struct ConvA {               // NHWC input [B, Hin, Win, Cin]; output pixel grid Hout x Wout
    const bf16* in;
    int Hin, Win, Cin, Hout, Wout;
    int ksize;               // 1 or 3 (pad = ksize/2, stride 1)
    int up;                  // 1: input is nearest-upsampled x2 on the fly (Hout = 2*Hin)
                             // 2: Downsample (vq_model.py:389-397): zero pad right/bottom by one, 3x3 stride 2, Hout = Hin/2
    int M;                   // B*Hout*Wout
    struct Row { int b, y, x; };
    __device__ __forceinline__ Row row(int m, int) const {
        Row r;
        if (m < M) {
            const int hw = Hout * Wout;
            r.b = m / hw;
            const int rem = m - r.b * hw;
            r.y = rem / Wout;
            r.x = rem - r.y * Wout;
        } else {
            r.b = -1; r.y = 0; r.x = 0;
        }
        return r;
    }
    __device__ __forceinline__ const bf16* ptr(const Row& r, int k) const {
        if (r.b < 0) return nullptr;
        const int tap = k / Cin, c = k - tap * Cin;
        int yy = r.y, xx = r.x;
        if (up == 2) {
            const int ty = tap / 3;
            yy = 2 * yy + ty;
            xx = 2 * xx + tap - ty * 3;
            if (yy >= Hin || xx >= Win) return nullptr;
            return in + (((long long)r.b * Hin + yy) * Win + xx) * Cin + c;
        }
        if (ksize == 3) {
            const int ty = tap / 3;
            yy += ty - 1;
            xx += tap - ty * 3 - 1;
            if ((unsigned)yy >= (unsigned)Hout || (unsigned)xx >= (unsigned)Wout) return nullptr;
        }
        if (up) { yy >>= 1; xx >>= 1; }
        return in + (((long long)r.b * Hin + yy) * Win + xx) * Cin + c;
    }
};

// B operand: rows n < n_split come from Wa, the rest from Wb (w1 | w3 without a repacked copy)
struct BRows {
    const bf16* Wa; const bf16* Wb;
    int n_split; long long ldw; long long batch_stride; int N;
    __device__ __forceinline__ const bf16* row(int n, int bz) const {
        if (n >= N) return nullptr;
        const bf16* base = n < n_split ? Wa + (long long)n * ldw : Wb + (long long)(n - n_split) * ldw;
        return base + (long long)bz * batch_stride;
    }
};

struct EpiPartial {          // fp32 slabs [z][M][N]
    float* out; int M, N;
    __device__ __forceinline__ void operator()(int m, int n, float v0, float v1, int z) const {
        float* p = out + ((size_t)z * M + m) * N + n;
        if (n + 1 < N) *reinterpret_cast<float2*>(p) = make_float2(v0, v1);
        else p[0] = v0;
    }
};

template <int BM, int BN, int WARPS_M, int WARPS_N, int STAGES, class AL, class Epi, typename T = bf16>
__global__ void __launch_bounds__(kThreads) gemm_mma_kernel(AL al, BRows bw, int M, int N, int K, int kper,
                                                            int ksplit, Epi epi) {
    lg_pdl_sync();
    static_assert(WARPS_M * WARPS_N == 8, "8 warps");
    constexpr int WTM = BM / WARPS_M, WTN = BN / WARPS_N;
    constexpr int MT = WTM / 16, NT = WTN / 8;
    static_assert(WTM % 16 == 0 && WTN % 16 == 0, "warp tile");
    constexpr int A_ITERS = (BM + 31) / 32, B_ITERS = (BN + 31) / 32;
    constexpr int STAGE_BYTES = (BM + BN) * 128;

    extern __shared__ __align__(1024) unsigned char smem_raw[];
    const uint32_t smem_base = smem_u32(smem_raw);

    const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
    const int wm = warp / WARPS_N, wn = warp % WARPS_N;
    const int m0 = blockIdx.x * BM, n0 = blockIdx.y * BN;
    const int bz = blockIdx.z / ksplit, ks = blockIdx.z - bz * ksplit;
    const int kbeg = ks * kper, kend = min(K, kbeg + kper);
    const int KT = (kend - kbeg + BK - 1) / BK;

    const int lrow = tid >> 3, lchunk = tid & 7;
    typename AL::Row arow[A_ITERS];
    const bf16* brow[B_ITERS];
#pragma unroll
    for (int i = 0; i < A_ITERS; ++i) arow[i] = al.row(m0 + lrow + i * 32, bz);
#pragma unroll
    for (int i = 0; i < B_ITERS; ++i) brow[i] = bw.row(n0 + lrow + i * 32, bz);

    auto load_tile = [&](int stage, int kt) {
        const int k = kbeg + kt * BK + lchunk * 8;
        const bool kin = k < kend;
        const uint32_t sa = smem_base + stage * STAGE_BYTES, sb = sa + BM * 128;
#pragma unroll
        for (int i = 0; i < A_ITERS; ++i) {
            const int r = lrow + i * 32;
            if (BM % 32 == 0 || r < BM) {
                const bf16* p = kin ? al.ptr(arow[i], k) : nullptr;
                cp_async16(sa + swz(r, lchunk), p ? (const void*)p : (const void*)bw.Wa, p != nullptr);
            }
        }
#pragma unroll
        for (int i = 0; i < B_ITERS; ++i) {
            const int r = lrow + i * 32;
            if (BN % 32 == 0 || r < BN) {
                const bf16* p = (kin && brow[i]) ? brow[i] + k : nullptr;
                cp_async16(sb + swz(r, lchunk), p ? (const void*)p : (const void*)bw.Wa, p != nullptr);
            }
        }
    };

    float acc[MT][NT][4];
#pragma unroll
    for (int i = 0; i < MT; ++i)
#pragma unroll
        for (int j = 0; j < NT; ++j)
#pragma unroll
            for (int c = 0; c < 4; ++c) acc[i][j][c] = 0.f;

#pragma unroll
    for (int s = 0; s < STAGES - 1; ++s) {
        if (s < KT) load_tile(s, s);
        cp_async_commit();
    }

    for (int kt = 0; kt < KT; ++kt) {
        cp_async_wait<STAGES - 2>();
        __syncthreads();
        {
            const int nk = kt + STAGES - 1;
            if (nk < KT) load_tile(nk % STAGES, nk);
            cp_async_commit();
        }
        const uint32_t sa = smem_base + (kt % STAGES) * STAGE_BYTES, sb = sa + BM * 128;
#pragma unroll
        for (int kk = 0; kk < BK / 16; ++kk) {
            uint32_t af[MT][4];
#pragma unroll
            for (int mt = 0; mt < MT; ++mt) {
                const int r = wm * WTM + mt * 16 + (lane & 15);
                ldmatrix_x4(sa + swz(r, kk * 2 + (lane >> 4)), af[mt][0], af[mt][1], af[mt][2], af[mt][3]);
            }
#pragma unroll
            for (int np = 0; np < NT / 2; ++np) {
                uint32_t b0, b1, b2, b3;
                const int r = wn * WTN + np * 16 + (lane & 7) + ((lane >> 4) << 3);
                ldmatrix_x4(sb + swz(r, kk * 2 + ((lane >> 3) & 1)), b0, b1, b2, b3);
#pragma unroll
                for (int mt = 0; mt < MT; ++mt) {
                    mma_m16n8k16<T>(acc[mt][2 * np], af[mt][0], af[mt][1], af[mt][2], af[mt][3], b0, b1);
                    mma_m16n8k16<T>(acc[mt][2 * np + 1], af[mt][0], af[mt][1], af[mt][2], af[mt][3], b2, b3);
                }
            }
        }
    }
    cp_async_wait<0>();

    const int g = lane >> 2, tg = lane & 3;
#pragma unroll
    for (int mt = 0; mt < MT; ++mt) {
#pragma unroll
        for (int nt = 0; nt < NT; ++nt) {
            const int n = n0 + wn * WTN + nt * 8 + tg * 2;
            if (n >= N) continue;
            const int ma = m0 + wm * WTM + mt * 16 + g;
            if (ma < M) epi(ma, n, acc[mt][nt][0], acc[mt][nt][1], (int)blockIdx.z);
            if (ma + 8 < M) epi(ma + 8, n, acc[mt][nt][2], acc[mt][nt][3], (int)blockIdx.z);
        }
    }
}

template <int BM, int BN, int WARPS_M, int WARPS_N, int STAGES, typename T = bf16, class AL, class Epi>
int launch_gemm_mma(const AL& al, const BRows& bw, int M, int N, int K, int ksplit, int nbatch, const Epi& epi,
                    cudaStream_t st, bool pdl = true) {
    auto kern = gemm_mma_kernel<BM, BN, WARPS_M, WARPS_N, STAGES, AL, Epi, T>;
    constexpr int smem = STAGES * (BM + BN) * 128;
    static DevOnce attr_set;
    if (lg_first_on_device(attr_set)) {
        LG_CUDA_OK(cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, smem));
    }
    LG_REQUIRE(K % 8 == 0, "gemm: K=%d must be a multiple of 8", K);
    const int kt_total = (K + BK - 1) / BK;
    const int kper = ((kt_total + ksplit - 1) / ksplit) * BK;
    dim3 grid((M + BM - 1) / BM, (N + BN - 1) / BN, nbatch * ksplit);
    LG_REQUIRE(grid.y <= 65535 && grid.z <= 65535, "gemm: grid too large (%u, %u)", grid.y, grid.z);
    (void)lg_launch_pdl(pdl, kern, grid, dim3(kThreads), smem, st, al, bw, M, N, K, kper, ksplit, epi);
    LG_LAUNCH_CHECK();
    return 0;
}

}  // namespace mma
