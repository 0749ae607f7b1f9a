// Dense transformer GEMMs: y[M,N] = x[M,K] * W[N,K]^T (nn.Linear without bias, gpt.py:161-163,199-200,287).
// Two kernels, both produce fp32 split-K slabs consumed by the row-wise epilogues in xf_kernels.cu:
//   * gemm_skinny_kernel : M <= 8 rows per tile on CUDA cores, 128-bit weight streaming. Used for the
//     batch-1 latency path (HBM-bound GEMV regime) and for the fp32 "exact" mode at any M.
//   * mma::gemm_mma_kernel: bf16 / fp16 tensor-core tiles for M > 8 (the fallback of the wgmma kernel, gemm_tc.cu).
// bf16 and fp16 take the same path for every shape; only the MMA operand type differs.
#include "kernels.cuh"
#include "gemm_mma.cuh"
#include <algorithm>

namespace {

constexpr int kSkinnyRT = 8;      // rows per tile held in registers
constexpr int kSkinnyKC = 2048;   // K elements staged in shared memory per chunk
constexpr int kSkinnyWarps = 8;

template <typename T>
__global__ void __launch_bounds__(kSkinnyWarps * 32) gemm_skinny_kernel(const T* __restrict__ X, long long ldx,
                                                                        const T* __restrict__ Wa,
                                                                        const T* __restrict__ Wb, int n_split,
                                                                        int M, int N, int K, int kper,
                                                                        float* __restrict__ partial) {
    lg_pdl_sync();
    constexpr int VEC = 16 / sizeof(T);
    constexpr int RT = kSkinnyRT, KC = kSkinnyKC;
    extern __shared__ __align__(16) unsigned char sraw[];
    T* xs = reinterpret_cast<T*>(sraw);  // [RT][KC]

    const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
    const int ks = blockIdx.z, kbeg = ks * kper, kend = min(K, kbeg + kper);
    const int m0 = blockIdx.y * RT;
    const int n = (blockIdx.x * kSkinnyWarps + warp) * 2;
    const bool nvalid = n < N;
    const T* w0 = nullptr;
    const T* w1 = nullptr;
    if (nvalid) {
        w0 = n < n_split ? Wa + (long long)n * K : Wb + (long long)(n - n_split) * K;
        w1 = (n + 1) < n_split ? Wa + (long long)(n + 1) * K : Wb + (long long)(n + 1 - n_split) * K;
    }

    float acc0[RT], acc1[RT];
#pragma unroll
    for (int r = 0; r < RT; ++r) { acc0[r] = 0.f; acc1[r] = 0.f; }

    for (int kc0 = kbeg; kc0 < kend; kc0 += KC) {
        const int kc = min(KC, kend - kc0);
        const int cpr = kc / VEC;  // 16-byte chunks per row
        for (int idx = tid; idx < RT * cpr; idx += kSkinnyWarps * 32) {
            const int r = idx / cpr, c = idx - r * cpr;
            uint4 v = make_uint4(0, 0, 0, 0);
            if (m0 + r < M) v = *reinterpret_cast<const uint4*>(X + (long long)(m0 + r) * ldx + kc0 + c * VEC);
            *reinterpret_cast<uint4*>(xs + r * KC + c * VEC) = v;
        }
        __syncthreads();
        if (nvalid) {
#pragma unroll 2
            for (int kk = lane * VEC; kk < kc; kk += 32 * VEC) {
                float a[VEC], b[VEC];
                VecLoad<T, VEC>::load(w0 + kc0 + kk, a);
                VecLoad<T, VEC>::load(w1 + kc0 + kk, b);
#pragma unroll
                for (int r = 0; r < RT; ++r) {
                    float xv[VEC];
                    VecLoad<T, VEC>::load(xs + r * KC + kk, xv);
#pragma unroll
                    for (int i = 0; i < VEC; ++i) {
                        acc0[r] = fmaf(a[i], xv[i], acc0[r]);
                        acc1[r] = fmaf(b[i], xv[i], acc1[r]);
                    }
                }
            }
        }
        __syncthreads();
    }
    if (!nvalid) return;
#pragma unroll
    for (int r = 0; r < RT; ++r) {
        acc0[r] = warp_sum(acc0[r]);
        acc1[r] = warp_sum(acc1[r]);
    }
#pragma unroll
    for (int r = 0; r < RT; ++r) {
        if (lane == r && m0 + r < M) {
            float* p = partial + ((size_t)ks * M + (m0 + r)) * N + n;
            *reinterpret_cast<float2*>(p) = make_float2(acc0[r], acc1[r]);
        }
    }
}

struct Plan {
    bool skinny;
    bool tc;      // wgmma / TMA kernel (gemm_tc.cu)
    int bm;       // mma tile rows
    int ksplit;
};

Plan make_plan(int M, int N, int K, int dtype) {
    Plan p;
    p.tc = false;
    // bf16 / fp16: the wgmma kernel is used for every row count (a batch-1 step pads its 2 rows to the minimum N = 16); the CUDA-core
    // skinny kernel stays for the fp32 exact mode.
    const bool tc_ok = lg_env_flag("LG_GEMM_TC", 1) && gemm_tc_supported(M, N, K, dtype) && N % 128 == 0;
    p.skinny = (dtype == LG_DTYPE_F32) || (M <= kSkinnyRT && !tc_ok);
    if (!p.skinny && tc_ok) {
        p.tc = true;
        p.bm = 0;
        p.ksplit = gemm_tc_ksplit(M, N, K);
        return p;
    }
    if (p.skinny) {
        p.bm = kSkinnyRT;
        const long long ctas = (long long)cdiv(N, 2 * kSkinnyWarps) * cdiv(M, kSkinnyRT);
        int ks = (int)std::max<long long>(1, 264 / std::max<long long>(ctas, 1));
        ks = std::min(ks, std::max(1, K / 512));
        p.ksplit = std::min(ks, 16);
    } else {
        p.bm = M <= 32 ? 32 : (M <= 64 ? 64 : 128);
        const long long tiles = (long long)cdiv(M, p.bm) * cdiv(N, 128);
        int ks = (int)std::max<long long>(1, 132 / std::max<long long>(tiles, 1));
        ks = std::min(ks, std::max(1, (K / mma::BK) / 4));
        p.ksplit = std::min(ks, 16);
    }
    return p;
}

}  // namespace

size_t gemm_partial_floats(int M, int N, int K, int dtype) {
    const Plan p = make_plan(M, N, K, dtype);
    return (size_t)p.ksplit * M * N;
}

int gemm_partial(const void* X, int ldx, const void* Wa, const void* Wb, int n_split, int M, int N, int K, int dtype,
                 float* partial, GemmPlan* plan, cudaStream_t st, const GemmNext* next) {
    LG_REQUIRE(M > 0 && N > 0 && K > 0, "gemm: bad shape %d %d %d", M, N, K);
    LG_REQUIRE(N % 2 == 0 && K % 8 == 0, "gemm: N=%d must be even and K=%d a multiple of 8", N, K);
    if (Wb == nullptr) { Wb = Wa; n_split = N; }
    const Plan p = make_plan(M, N, K, dtype);
    if (plan) plan->ksplit = p.ksplit;
    if (p.skinny) {
        // kper: multiple of 256 elements so every lane's 16-byte vector stays inside the slab
        int kper = cdiv(cdiv(K, p.ksplit), 256) * 256;
        dim3 grid(cdiv(N, 2 * kSkinnyWarps), cdiv(M, kSkinnyRT), p.ksplit);
        LG_REQUIRE(grid.y <= 65535, "gemm: too many rows for the skinny path (%d)", M);
        if (dtype == LG_DTYPE_F32) {
            const size_t smem = (size_t)kSkinnyRT * kSkinnyKC * sizeof(float);
            static DevOnce attr;
            if (lg_first_on_device(attr)) {
                LG_CUDA_OK(cudaFuncSetAttribute(gemm_skinny_kernel<float>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
            }
            (void)lg_launch(gemm_skinny_kernel<float>, dim3(grid), dim3(kSkinnyWarps * 32), smem, st, 
                (const float*)X, ldx, (const float*)Wa, (const float*)Wb, n_split, M, N, K, kper, partial);
        } else if (dtype == LG_DTYPE_F16) {
            const size_t smem = (size_t)kSkinnyRT * kSkinnyKC * sizeof(f16);
            (void)lg_launch(gemm_skinny_kernel<f16>, dim3(grid), dim3(kSkinnyWarps * 32), smem, st,
                (const f16*)X, ldx, (const f16*)Wa, (const f16*)Wb, n_split, M, N, K, kper, partial);
        } else {
            const size_t smem = (size_t)kSkinnyRT * kSkinnyKC * sizeof(bf16);
            (void)lg_launch(gemm_skinny_kernel<bf16>, dim3(grid), dim3(kSkinnyWarps * 32), smem, st, 
                (const bf16*)X, ldx, (const bf16*)Wa, (const bf16*)Wb, n_split, M, N, K, kper, partial);
        }
        LG_LAUNCH_CHECK();
        return 0;
    }
    if (p.tc) {
        if (n_split % 128 != 0 && n_split != N) return lg_fail("gemm: weight segment boundary %d not tile aligned", n_split);
        return gemm_tc_partial(X, ldx, Wa, Wb, n_split, M, N, K, dtype, partial, nullptr, st, next);
    }
    LG_REQUIRE(lg_dtype_is16(dtype), "gemm: unsupported dtype %d", dtype);
    mma::DenseA al{(const bf16*)X, ldx, 0, M};   // raw 16-bit elements: the same loaders serve fp16
    mma::BRows bw{(const bf16*)Wa, (const bf16*)Wb, n_split, K, 0, N};
    mma::EpiPartial epi{partial, M, N};
    if (dtype == LG_DTYPE_F16) {
        if (p.bm == 32) return mma::launch_gemm_mma<32, 128, 1, 8, 4, f16>(al, bw, M, N, K, p.ksplit, 1, epi, st);
        if (p.bm == 64) return mma::launch_gemm_mma<64, 128, 2, 4, 4, f16>(al, bw, M, N, K, p.ksplit, 1, epi, st);
        return mma::launch_gemm_mma<128, 128, 2, 4, 3, f16>(al, bw, M, N, K, p.ksplit, 1, epi, st);
    }
    if (p.bm == 32) return mma::launch_gemm_mma<32, 128, 1, 8, 4>(al, bw, M, N, K, p.ksplit, 1, epi, st);
    if (p.bm == 64) return mma::launch_gemm_mma<64, 128, 2, 4, 4>(al, bw, M, N, K, p.ksplit, 1, epi, st);
    return mma::launch_gemm_mma<128, 128, 2, 4, 3>(al, bw, M, N, K, p.ksplit, 1, epi, st);
}
