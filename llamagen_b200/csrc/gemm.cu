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

}  // namespace

GemmPlan gemm_plan(int M, int N, int K, int n_split, int dtype, bool w8) {
    GemmPlan p;
    if (M <= 0 || N <= 0 || K <= 0) {
        snprintf(p.error, sizeof(p.error), "gemm: bad shape %d %d %d", M, N, K);
        return p;
    }
    if (N % 2 != 0 || K % 8 != 0) {
        snprintf(p.error, sizeof(p.error), "gemm: N=%d must be even and K=%d a multiple of 8", N, K);
        return p;
    }
    if (dtype != LG_DTYPE_F32 && !lg_dtype_is16(dtype)) {
        snprintf(p.error, sizeof(p.error), "gemm: unsupported dtype %d", dtype);
        return p;
    }
    if (n_split < 0 || n_split > N) {
        snprintf(p.error, sizeof(p.error), "gemm: weight segment boundary %d outside [0, %d]", n_split, N);
        return p;
    }
    // bf16 / fp16: the wgmma kernel is used for every row count (a batch-1 step pads its 2 rows to the minimum N = 16); the CUDA-core
    // skinny kernel stays for the fp32 exact mode. A wgmma CTA streams one 128-row weight tile from one segment, so the w1 | w3
    // boundary must fall on a tile edge; any other boundary (ffn_dim % 128 != 0) goes to the row-wise loaders of the other kernels.
    const bool one_segment = n_split == 0 || n_split == N;
    if (w8) {
        // fp8 weights exist only as e4m3 codes: the wgmma kernel is their one batched kernel, and a call it cannot take is an error
        if (!lg_dtype_is16(dtype))
            snprintf(p.error, sizeof(p.error), "gemm: fp8 weights need a bf16 or fp16 model (dtype %d)", dtype);
        else if (N % 128 != 0 || !(one_segment || n_split % 128 == 0))
            snprintf(p.error, sizeof(p.error), "gemm: fp8 weights need N=%d and the segment boundary %d on 128-row tiles", N, n_split);
        else if (K % 64 != 0)
            snprintf(p.error, sizeof(p.error), "gemm: fp8 weights need K=%d a multiple of 64", K);
        else if (!lg_env_flag("LG_GEMM_TC", 1))
            snprintf(p.error, sizeof(p.error), "gemm: fp8 weights run on the wgmma kernel only (LG_GEMM_TC=0)");
        if (p.error[0]) return p;
    }
    const bool tc_ok = lg_env_flag("LG_GEMM_TC", 1) && lg_dtype_is16(dtype) && N % 128 == 0 && (one_segment || n_split % 128 == 0);
    if (tc_ok) {
        const int rblk = std::min(M, 256);
        p.kernel = 2;
        p.tile = 16;
        while (p.tile < rblk) p.tile *= 2;
        p.row_blocks = cdiv(M, rblk);
        p.ksplit = gemm_tc_ksplit(M, N, K);
        return p;
    }
    if (dtype == LG_DTYPE_F32 || M <= kSkinnyRT) {
        p.kernel = 0;
        p.tile = kSkinnyRT;
        const long long ctas = (long long)cdiv(N, 2 * kSkinnyWarps) * cdiv(M, kSkinnyRT);
        int ks = (int)std::max<long long>(1, 264 / std::max<long long>(ctas, 1));
        ks = std::min(ks, std::max(1, K / 512));
        p.ksplit = std::min(ks, 16);
    } else {
        p.kernel = 1;
        p.tile = M <= 32 ? 32 : (M <= 64 ? 64 : 128);
        const long long tiles = (long long)cdiv(M, p.tile) * cdiv(N, 128);
        int ks = (int)std::max<long long>(1, 132 / std::max<long long>(tiles, 1));
        ks = std::min(ks, std::max(1, (K / mma::BK) / 4));
        p.ksplit = std::min(ks, 16);
    }
    p.row_blocks = cdiv(M, p.tile);
    return p;
}

size_t gemm_partial_floats(int M, int N, int K, int n_split, int dtype, bool w8) {
    const GemmPlan p = gemm_plan(M, N, K, n_split, dtype, w8);
    return p.kernel < 0 ? 0 : (size_t)p.ksplit * M * N;
}

int gemm_partial(const void* X, int ldx, const GemmWeight& wa, const GemmWeight& wb_in, int n_split, int M, int N, int K, int dtype,
                 float* partial, GemmPlan* plan, cudaStream_t st, const GemmNext* next, bool pdl) {
    GemmWeight wb = wb_in;
    if (wb.p == nullptr || n_split == 0) { wb = wa; n_split = N; }
    LG_REQUIRE((wa.scale != nullptr) == (wb.scale != nullptr), "gemm: both weight segments must be fp8 or both 16-bit");
    const GemmPlan p = gemm_plan(M, N, K, n_split, dtype, wa.scale != nullptr);
    if (plan) *plan = p;
    if (p.kernel < 0) return lg_fail("%s", p.error);
    const void *Wa = wa.p, *Wb = wb.p;
    if (p.kernel == 0) {
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
            (void)lg_launch_pdl(pdl, gemm_skinny_kernel<float>, dim3(grid), dim3(kSkinnyWarps * 32), smem, st, 
                (const float*)X, ldx, (const float*)Wa, (const float*)Wb, n_split, M, N, K, kper, partial);
        } else if (dtype == LG_DTYPE_F16) {
            const size_t smem = (size_t)kSkinnyRT * kSkinnyKC * sizeof(f16);
            (void)lg_launch_pdl(pdl, gemm_skinny_kernel<f16>, dim3(grid), dim3(kSkinnyWarps * 32), smem, st,
                (const f16*)X, ldx, (const f16*)Wa, (const f16*)Wb, n_split, M, N, K, kper, partial);
        } else {
            const size_t smem = (size_t)kSkinnyRT * kSkinnyKC * sizeof(bf16);
            (void)lg_launch_pdl(pdl, gemm_skinny_kernel<bf16>, dim3(grid), dim3(kSkinnyWarps * 32), smem, st, 
                (const bf16*)X, ldx, (const bf16*)Wa, (const bf16*)Wb, n_split, M, N, K, kper, partial);
        }
        LG_LAUNCH_CHECK();
        return 0;
    }
    if (p.kernel == 2) return gemm_tc_partial(X, ldx, wa, wb, n_split, M, N, K, dtype, p, partial, st, next, pdl);
    mma::DenseA al{(const bf16*)X, ldx, 0, M};   // raw 16-bit elements: the same loaders serve fp16
    mma::BRows bw{(const bf16*)Wa, (const bf16*)Wb, n_split, K, 0, N};
    mma::EpiPartial epi{partial, M, N};
    if (dtype == LG_DTYPE_F16) {
        if (p.tile == 32) return mma::launch_gemm_mma<32, 128, 1, 8, 4, f16>(al, bw, M, N, K, p.ksplit, 1, epi, st, pdl);
        if (p.tile == 64) return mma::launch_gemm_mma<64, 128, 2, 4, 4, f16>(al, bw, M, N, K, p.ksplit, 1, epi, st, pdl);
        return mma::launch_gemm_mma<128, 128, 2, 4, 3, f16>(al, bw, M, N, K, p.ksplit, 1, epi, st, pdl);
    }
    if (p.tile == 32) return mma::launch_gemm_mma<32, 128, 1, 8, 4>(al, bw, M, N, K, p.ksplit, 1, epi, st, pdl);
    if (p.tile == 64) return mma::launch_gemm_mma<64, 128, 2, 4, 4>(al, bw, M, N, K, p.ksplit, 1, epi, st, pdl);
    return mma::launch_gemm_mma<128, 128, 2, 4, 3>(al, bw, M, N, K, p.ksplit, 1, epi, st, pdl);
}
