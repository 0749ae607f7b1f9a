// fp8 (e4m3) GEMM weights: the quantiser that defines the stored byte, and the host-side checks of what enters the engine.
//
// A weight W [N][K] of a bf16 / fp16 model becomes code [N][K] (uint8) + scale [N] (fp32), include/llamagen_b200.h:
//   scale[n] = 2^e with max_k |W[n,k]| / 2^e in (224, 448] (e4m3's top binade), e clamped to the model dtype's range, 1 for a zero row;
//   code of (n, k) = e4m3_satfinite_rne(float(W[n,k]) / scale[n]) (the KV writers' conversion, e4m3x2_pack);
//   the code of column k sits at byte w8_stored_index(k) of its row: inside every 64-wide k-block the order is that of the
//   tensor-core A fragments, so a thread of gemm_tc_kernel / gemv_small_kernel fetches the fragments of a k-block with one 16-byte load.
#include "kernels.cuh"
#include <cmath>
#include <vector>

namespace {

// byte position inside a 64-wide k-block of the code of column k = 16 s + 8 h + 2 q + b: piece q (16 bytes) holds, for each K = 16 step s,
// the columns 2q, 2q + 1 (h = 0) and 8 + 2q, 8 + 2q + 1 (h = 1) that lane q of a quad feeds to the MMA
__host__ __device__ inline int stored_index(int k) {
    const int kb = k & ~63, s = (k >> 4) & 3, h = (k >> 3) & 1, q = (k >> 1) & 3, b = k & 1;
    return kb + 16 * q + 4 * s + 2 * h + b;
}

template <typename T>
__global__ void __launch_bounds__(256) quantize_rows_e4m3_kernel(const T* __restrict__ w, int K, int emin, int emax,
                                                                 uint8_t* __restrict__ codes, float* __restrict__ scales) {
    __shared__ float red[33];
    lg_pdl_sync();
    const T* row = w + (size_t)blockIdx.x * K;
    uint8_t* out = codes + (size_t)blockIdx.x * K;
    float amax = 0.f;
    for (int k = threadIdx.x * 8; k < K; k += 256 * 8) {
        float v[8];
        VecLoad<T, 8>::load(row + k, v);
#pragma unroll
        for (int i = 0; i < 8; ++i) amax = fmaxf(amax, fabsf(v[i]));
    }
    amax = block_max(amax, red);
    int e = 0;
    if (amax > 0.f) {
        int ex;
        const float m = frexpf(amax, &ex);              // amax = m * 2^ex, m in [0.5, 1); 448 = 0.875 * 2^9
        e = min(max(m <= 0.875f ? ex - 9 : ex - 8, emin), emax);
    }
    const float inv = ldexpf(1.0f, -e);                 // the division by a power of two is this exact product
    if (threadIdx.x == 0) scales[blockIdx.x] = ldexpf(1.0f, e);
    for (int k = threadIdx.x * 8; k < K; k += 256 * 8) {
        float v[8];
        VecLoad<T, 8>::load(row + k, v);
#pragma unroll
        for (int i = 0; i < 4; ++i)                     // columns k + 2i, k + 2i + 1 stay adjacent in the stored order
            *reinterpret_cast<uint16_t*>(out + stored_index(k + 2 * i)) = (uint16_t)e4m3x2_pack(v[2 * i] * inv, v[2 * i + 1] * inv);
    }
}

}  // namespace

int w8_stored_index(int k) { return stored_index(k); }

void w8_scale_exponents(int dtype, int* emin, int* emax) {
    // fp16: the smallest e4m3 subnormal 2^-9 times 2^-15 is fp16's smallest subnormal, and 448 * 2^7 < 65504. bf16 has fp32's exponent
    // range; +-64 keeps every code * scale and every 1 / scale a normal number with room to spare.
    *emin = dtype == LG_DTYPE_F16 ? -15 : -64;
    *emax = dtype == LG_DTYPE_F16 ? 7 : 64;
}

int launch_quantize_rows_e4m3(const void* w, int N, int K, int dtype, uint8_t* codes, float* scales, cudaStream_t st) {
    LG_REQUIRE(w && codes && scales && N > 0 && K > 0, "quantize_rows_e4m3: null argument or bad shape %d x %d", N, K);
    LG_REQUIRE(lg_dtype_is16(dtype), "quantize_rows_e4m3: fp8 weights need a bf16 or fp16 source (dtype %d)", dtype);
    LG_REQUIRE(K % 64 == 0, "quantize_rows_e4m3: K=%d must be a multiple of 64 (the stored order permutes 64-wide k-blocks)", K);
    LG_REQUIRE(((uintptr_t)w & 15) == 0 && ((uintptr_t)codes & 15) == 0, "quantize_rows_e4m3: operands must be 16-byte aligned");
    int emin, emax;
    w8_scale_exponents(dtype, &emin, &emax);
    if (dtype == LG_DTYPE_F16)
        (void)lg_launch(quantize_rows_e4m3_kernel<f16>, dim3(N), dim3(256), 0, st, (const f16*)w, K, emin, emax, codes, scales);
    else
        (void)lg_launch(quantize_rows_e4m3_kernel<bf16>, dim3(N), dim3(256), 0, st, (const bf16*)w, K, emin, emax, codes, scales);
    LG_LAUNCH_CHECK();
    return 0;
}

int w8_check_scales(const char* name, const float* dev_scales, int N, int dtype) {
    std::vector<float> h((size_t)N);
    LG_CUDA_OK(cudaMemcpy(h.data(), dev_scales, (size_t)N * sizeof(float), cudaMemcpyDeviceToHost));
    int emin, emax;
    w8_scale_exponents(dtype, &emin, &emax);
    for (int n = 0; n < N; ++n) {
        int ex = 0;
        const float s = h[n];
        const bool ok = std::isfinite(s) && s > 0.f && std::frexp(s, &ex) == 0.5f && ex - 1 >= emin && ex - 1 <= emax;
        LG_REQUIRE(ok, "'%s' row %d is %g; fp8 weight scales must be powers of two in [2^%d, 2^%d]", name, n, (double)s, emin, emax);
    }
    return 0;
}
