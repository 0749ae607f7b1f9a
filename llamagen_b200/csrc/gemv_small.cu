// Decode GEMMs for R <= 8 activation rows (the batch-1 latency path; R = 2 with classifier-free guidance).
//
// At R <= 8 a 16-wide wgmma N tile is >= 50 % padding and the split-K slabs + row-epilogue kernels of the batched path
// dominate the token time (8 dependent kernels per layer). Here every CTA OWNS a few output columns over the full K, so
// there is no split-K, no slab and no separate epilogue kernel: RMSNorm moves into the prologue, residual add /
// SwiGLU gate / fp32 store into the epilogue, and a layer is 5 dependent kernels
//     qkv' (norm prologue) -> attention (fused RoPE + KV write, attn_tma.cu) -> wo' (+residual) -> w13' (norm, SwiGLU) -> w2' (+residual).
//
// Math: mma.sync m16n8k16 (bf16 x bf16 or fp16 x fp16 -> fp32), weights as the M operand (16 weight rows), activations as the N operand
// (8 rows). Both operands are fetched with 128-bit loads: lane (g, t) loads 8 consecutive k of weight rows g / g+8 from
// HBM and of activation row g from shared memory, and feeds registers {0,1} to one MMA and {2,3} to the next — the k
// permutation this implies is the same on both operands, so the dot products are exact. The 8 warps of a CTA interleave
// 32-wide k chunks (adjacent warps read adjacent 64-byte segments of the same weight rows) and combine through shared
// memory in a fixed order. Weight loads do not depend on the previous kernel: the first PF chunks are requested before
// the programmatic-dependency wait.
//
// Rounding points are those of the batched path (xf_kernels.cu: residual_norm_kernel, silu_mul_kernel), i.e. of the
// reference's bf16 / fp16 tensors (gpt.py:143-148,167,255-256).
#include "kernels.cuh"

namespace {

constexpr int kWarps = 8, kThreads = 256;

// 16-bit tensors of element type T (bf16 or f16)
template <typename T>
struct GemvArgs {
    const T* Wa;           // [N][K]
    const T* Wb;           // paired form (SwiGLU): second matrix [N][K], else null
    int N, K, R;
    int pro;               // 0: x = in    1: x = rmsnorm(in) * normw
    const T* in;           // [R][K]
    const T* normw;        // [K]
    float eps;
    int epi;               // 0: out_f32[r][n] = acc   1: h[r][n] = T(h + T(acc))   2: ff[r][n] = T(T(silu(T(a))) * T(b))
    float* out_f32;
    T* h;
    T* ff;
};

// ROWS weight rows per CTA: 8 (upper half of one m16 tile), 16 (one tile) or 32 (two tiles; in the paired form tile 0 comes
// from Wa and tile 1 from the same rows of Wb). PF = chunks of 32 k kept in flight per warp.
template <int ROWS, int PF, typename T>
__global__ void __launch_bounds__(kThreads) gemv_small_kernel(GemvArgs<T> a) {
    using TR = ElemTraits<T>;
    constexpr int MT = ROWS == 32 ? 2 : 1;          // m16 tiles
    constexpr int HALVES = ROWS == 8 ? 1 : 2;       // row halves (g, g+8) loaded per tile
    extern __shared__ __align__(16) uint8_t smem[];
    const int K = a.K, R = a.R;
    const int xstride = K * 2 + 16;                 // bytes; +16 staggers the rows over the banks
    float* red = reinterpret_cast<float*>(smem);    // [kWarps][MT][16][8]
    float* rowsum = red + kWarps * MT * 16 * 8;     // [8 rows][8 warps]
    uint8_t* xs = reinterpret_cast<uint8_t*>(rowsum + 64);

    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31, g = lane >> 2, t = lane & 3;
    const int n0 = blockIdx.x * (a.Wb ? 16 : ROWS);
    const int nchunks = K / 32;
    const int my_chunks = (nchunks - warp + kWarps - 1) / kWarps;     // chunks warp, warp+8, ...

    const T* wrow[MT][HALVES];
#pragma unroll
    for (int mt = 0; mt < MT; ++mt)
#pragma unroll
        for (int hh = 0; hh < HALVES; ++hh) {
            const T* base = (a.Wb && mt == 1) ? a.Wb : a.Wa;
            const int row = n0 + ((a.Wb || mt == 0) ? 0 : 16) + g + 8 * hh;
            wrow[mt][hh] = base + (size_t)row * K + t * 8;
        }

    uint4 wbuf[PF][MT][HALVES];
    auto load_chunk = [&](int slot, int it) {
        const int c = warp + it * kWarps;
#pragma unroll
        for (int mt = 0; mt < MT; ++mt)
#pragma unroll
            for (int hh = 0; hh < HALVES; ++hh)
                wbuf[slot][mt][hh] = it < my_chunks ? __ldg(reinterpret_cast<const uint4*>(wrow[mt][hh] + (size_t)c * 32))
                                                    : make_uint4(0u, 0u, 0u, 0u);
    };
    lg_pdl_launch_dependents();
#pragma unroll
    for (int s = 0; s < PF; ++s) load_chunk(s, s);
    int rp = 1;
    while (rp < R) rp <<= 1;                        // rows padded to a power of two: 256 / rp threads per row
    const int tpr = kThreads / rp, row = threadIdx.x / tpr, j = threadIdx.x % tpr;
    const int pieces = K / 8;
    constexpr int NPW = 4;                          // norm-weight pieces per thread requested ahead of the dependency wait
    uint4 nwbuf[NPW];
    if (a.pro == 1) {
#pragma unroll
        for (int q = 0; q < NPW; ++q)
            nwbuf[q] = (row < R && j + q * tpr < pieces) ? __ldg(reinterpret_cast<const uint4*>(a.normw) + j + q * tpr) : make_uint4(0u, 0u, 0u, 0u);
    }
    lg_pdl_wait();
    // residual epilogue: request this thread's h element now, it is only needed after the main loop
    const int ei = threadIdx.x >> 3, er = threadIdx.x & 7;
    float h_old = 0.f;
    if (a.epi == 1 && er < R && ei < ROWS) h_old = TR::to_f(a.h[(size_t)er * a.N + n0 + ei]);

    // ---------------------------------------------------------------- prologue: activations -> shared memory
    {
        float ss = 0.f;
        if (row < R) {
            const uint4* src = reinterpret_cast<const uint4*>(a.in + (size_t)row * K);
            for (int p = j; p < pieces; p += tpr) {
                const uint4 v = src[p];
                *reinterpret_cast<uint4*>(xs + (size_t)row * xstride + (size_t)p * 16) = v;
                if (a.pro == 1) {
                    const uint32_t w[4] = {v.x, v.y, v.z, v.w};
#pragma unroll
                    for (int q = 0; q < 4; ++q) {
                        const float lo = TR::lo(w[q]), hi = TR::hi(w[q]);
                        ss = fmaf(lo, lo, ss);
                        ss = fmaf(hi, hi, ss);
                    }
                }
            }
        }
        if (a.pro == 1) {
            ss = warp_sum(ss);
            if (lane == 0) rowsum[warp] = ss;       // warps of one row are contiguous: row = warp / (tpr / 32)
            __syncthreads();
            if (row < R) {
                const int wpr = tpr / 32;
                float tot = 0.f;
                for (int w = 0; w < wpr; ++w) tot += rowsum[row * wpr + w];
                const float rinv = 1.0f / sqrtf(tot / (float)K + a.eps);
                int q0 = 0;
                for (int p = j; p < pieces; p += tpr, ++q0) {
                    uint4* px = reinterpret_cast<uint4*>(xs + (size_t)row * xstride + (size_t)p * 16);
                    const uint4 v = *px;
                    uint4 nw;
                    if (q0 == 0) nw = nwbuf[0];
                    else if (q0 == 1) nw = nwbuf[1];
                    else if (q0 == 2) nw = nwbuf[2];
                    else if (q0 == 3) nw = nwbuf[3];
                    else nw = __ldg(reinterpret_cast<const uint4*>(a.normw) + p);
                    const uint32_t w[4] = {v.x, v.y, v.z, v.w}, n[4] = {nw.x, nw.y, nw.z, nw.w};
                    uint32_t o[4];
#pragma unroll
                    for (int q = 0; q < 4; ++q) {
                        // (x.float() * rsqrt(mean(x^2) + eps)).type_as(x) * weight   (gpt.py:143-148)
                        const float lo = TR::round(TR::lo(w[q]) * rinv) * TR::lo(n[q]);
                        const float hi = TR::round(TR::hi(w[q]) * rinv) * TR::hi(n[q]);
                        o[q] = TR::pack2(lo, hi);
                    }
                    *px = make_uint4(o[0], o[1], o[2], o[3]);
                }
            }
        }
        __syncthreads();
    }

    // ---------------------------------------------------------------- main loop
    float acc[MT][4];
#pragma unroll
    for (int mt = 0; mt < MT; ++mt)
#pragma unroll
        for (int q = 0; q < 4; ++q) acc[mt][q] = 0.f;
    const uint8_t* xrow = xs + (size_t)min(g, R - 1) * xstride + t * 16;   // lanes of padding rows re-read a real row (columns are independent)
    for (int it0 = 0; it0 < my_chunks; it0 += PF) {
#pragma unroll
        for (int s = 0; s < PF; ++s) {
            const int it = it0 + s;
            if (it < my_chunks) {
                const int c = warp + it * kWarps;
                const uint4 xb = *reinterpret_cast<const uint4*>(xrow + (size_t)c * 64);
#pragma unroll
                for (int mt = 0; mt < MT; ++mt) {
                    const uint4 w0 = wbuf[s][mt][0];
                    const uint4 w1 = HALVES == 2 ? wbuf[s][mt][HALVES - 1] : make_uint4(0u, 0u, 0u, 0u);
                    mma_m16n8k16<T>(acc[mt], w0.x, w1.x, w0.y, w1.y, xb.x, xb.y);
                    mma_m16n8k16<T>(acc[mt], w0.z, w1.z, w0.w, w1.w, xb.z, xb.w);
                }
            }
            load_chunk(s, it + PF);
        }
    }

    // ---------------------------------------------------------------- combine the 8 k-slices, epilogue
#pragma unroll
    for (int mt = 0; mt < MT; ++mt) {
        float* rw = red + ((warp * MT + mt) * 16) * 8;
        *reinterpret_cast<float2*>(rw + g * 8 + 2 * t) = make_float2(acc[mt][0], acc[mt][1]);
        *reinterpret_cast<float2*>(rw + (g + 8) * 8 + 2 * t) = make_float2(acc[mt][2], acc[mt][3]);
    }
    __syncthreads();
    const int i = ei, r = er;                                // output (row i of the CTA, activation row r)
    if (r >= R) return;
    if (a.Wb) {                                              // paired: i < 16, tile 0 = w1 row, tile 1 = w3 row
        if (i >= 16) return;
        float av = 0.f, bv = 0.f;
#pragma unroll
        for (int w = 0; w < kWarps; ++w) {
            av += red[((w * MT + 0) * 16 + i) * 8 + r];
            bv += red[((w * MT + (MT - 1)) * 16 + i) * 8 + r];
        }
        av = TR::round(av);
        bv = TR::round(bv);
        const float sv = TR::round(av / (1.0f + expf(-av)));  // F.silu(w1 x) * w3 x in T tensors (gpt.py:167)
        a.ff[(size_t)r * a.N + n0 + i] = TR::from_f(sv * bv);
        return;
    }
    if (i >= ROWS) return;
    const int mt = i >> 4, ii = i & 15;
    float v = 0.f;
#pragma unroll
    for (int w = 0; w < kWarps; ++w) v += red[((w * MT + mt) * 16 + ii) * 8 + r];
    const size_t o = (size_t)r * a.N + n0 + i;
    if (a.epi == 0) {
        a.out_f32[o] = v;
    } else {                                                 // h = x + f(x), both T tensors (gpt.py:255-256)
        a.h[o] = TR::from_f(h_old + TR::round(v));
    }
}

template <int ROWS, int PF, typename T>
int launch_t(const GemvArgs<T>& a, cudaStream_t st) {
    constexpr int MT = ROWS == 32 ? 2 : 1;
    const size_t smem = (size_t)(kWarps * MT * 16 * 8 + 64) * sizeof(float) + (size_t)a.R * (a.K * 2 + 16);
    static DevOnce attr;
    if (lg_first_on_device(attr)) {
        LG_CUDA_OK(cudaFuncSetAttribute(gemv_small_kernel<ROWS, PF, T>, cudaFuncAttributeMaxDynamicSharedMemorySize, 100 * 1024));
    }
    LG_REQUIRE(smem <= 100 * 1024, "gemv_small: %zu bytes of shared memory (R=%d K=%d)", smem, a.R, a.K);
    const int rows_per_cta = a.Wb ? 16 : ROWS;
    (void)lg_launch(gemv_small_kernel<ROWS, PF, T>, dim3(a.N / rows_per_cta), dim3(kThreads), smem, st, a);
    LG_LAUNCH_CHECK();
    return 0;
}

template <typename T>
int launch_typed(const GemvSmall& g, cudaStream_t st) {
    GemvArgs<T> a;
    a.Wa = (const T*)g.Wa; a.Wb = (const T*)g.Wb; a.N = g.N; a.K = g.K; a.R = g.R;
    a.pro = g.normw ? 1 : 0; a.in = (const T*)g.in; a.normw = (const T*)g.normw; a.eps = g.eps;
    a.epi = g.Wb ? 2 : (g.out_f32 ? 0 : 1); a.out_f32 = g.out_f32; a.h = (T*)g.h; a.ff = (T*)g.ff;
    if (g.Wb) return launch_t<32, 4>(a, st);
    // Row granularity: enough CTAs to pull the matrix from all SMs (8 rows/CTA below ~2.4k outputs), fatter CTAs for the head
    if (g.N <= 2048) return launch_t<8, 12>(a, st);
    if (g.N <= 8192) return launch_t<16, 4>(a, st);
    return launch_t<32, 4>(a, st);
}

}  // namespace

bool gemv_small_supported(int R, int N, int K, int dtype, bool paired) {
    if (!lg_dtype_is16(dtype) || R < 1 || R > 8 || K % 32 != 0 || K < 256) return false;
    if ((size_t)R * (K * 2 + 16) > 90 * 1024) return false;
    return N % (paired ? 16 : 32) == 0;      // every row granularity used below divides N
}

int launch_gemv_small(const GemvSmall& g, cudaStream_t st) {
    LG_REQUIRE(gemv_small_supported(g.R, g.N, g.K, g.dtype, g.Wb != nullptr), "gemv_small: unsupported shape R=%d N=%d K=%d dtype %d",
               g.R, g.N, g.K, g.dtype);
    return g.dtype == LG_DTYPE_F16 ? launch_typed<f16>(g, st) : launch_typed<bf16>(g, st);
}
