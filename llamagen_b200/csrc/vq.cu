// VQ tokenizer decode path + codebook argmin on sm_90a (see include/llamagen_b200.h).
//
// Replaces tokenizer/tokenizer_image/vq_model.py:
//   decode_code :52-55 = get_codebook_entry :261-276 -> post_quant_conv :48 -> Decoder.forward :173-194
//   ResnetBlock :298-314, AttnBlock :327-351, Upsample :374-378, GroupNorm(32, eps 1e-6) :359-362, swish :354-356
//   VectorQuantizer.forward index path :215-233 (argmin-L2 over the L2-normalised codebook)
// Data layout: activations are bf16 NHWC in HBM (channels contiguous -> every implicit-GEMM k-chunk is one
// 16-byte load), conv weights are repacked once to bf16 [Cout][ky][kx][Cin]; GroupNorm statistics and all
// accumulation are fp32; the final conv writes fp32 NCHW like the reference.
#include "kernels.cuh"
#include "gemm_mma.cuh"
#include <algorithm>
#include <string>
#include <unordered_map>
#include <vector>

namespace {

// ------------------------------------------------------------------------------------------------ epilogue
struct EpiVq {
    const float* bias;       // nullable
    int bias_by_row;         // bias[m] instead of bias[n]
    const bf16* residual;    // nullable, [M, ldr]
    long long ldr;
    bf16* out_bf;            // one of out_bf / out_f32
    float* out_f32;
    long long ldo;
    long long out_batch_stride;  // elements per z (batched GEMMs)
    float scale;
    int N;
    int nchw;                // out_f32 as NCHW: m = b*hw + pix -> out[(b*N + n)*hw + pix]
    int hw;
    __device__ __forceinline__ void one(int m, int n, float v, int z) const {
        v *= scale;
        if (bias) v += bias_by_row ? bias[m] : bias[n];
        if (residual) v += __bfloat162float(residual[(long long)m * ldr + n]);
        if (nchw) {
            const int b = m / hw, pix = m - b * hw;
            out_f32[((long long)b * N + n) * hw + pix] = v;
        } else if (out_f32) {
            out_f32[(long long)z * out_batch_stride + (long long)m * ldo + n] = v;
        } else {
            out_bf[(long long)z * out_batch_stride + (long long)m * ldo + n] = __float2bfloat16_rn(v);
        }
    }
    __device__ __forceinline__ void operator()(int m, int n, float v0, float v1, int z) const {
        if (!nchw && !out_f32 && !residual && n + 1 < N && ((ldo | out_batch_stride) & 1) == 0) {
            v0 *= scale; v1 *= scale;
            if (bias) {
                if (bias_by_row) { v0 += bias[m]; v1 += bias[m]; }
                else { v0 += bias[n]; v1 += bias[n + 1]; }
            }
            __nv_bfloat162 p = __floats2bfloat162_rn(v0, v1);
            *reinterpret_cast<__nv_bfloat162*>(out_bf + (long long)z * out_batch_stride + (long long)m * ldo + n) = p;
            return;
        }
        one(m, n, v0, z);
        if (n + 1 < N) one(m, n + 1, v1, z);
    }
};

template <class AL>
int launch_vq_gemm(const AL& al, const mma::BRows& bw, int M, int N, int K, int nbatch, const EpiVq& epi, cudaStream_t st) {
    if (N >= 128) return mma::launch_gemm_mma<128, 128, 2, 4, 3>(al, bw, M, N, K, 1, nbatch, epi, st);
    return mma::launch_gemm_mma<128, 64, 4, 2, 4>(al, bw, M, N, K, 1, nbatch, epi, st);
}

// ------------------------------------------------------------------------------------------------ small kernels
__global__ void repack_conv_kernel(const float* __restrict__ src, bf16* __restrict__ dst, int cout, int cin, int kk) {
    const size_t total = (size_t)cout * cin * kk;
    for (size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (size_t)gridDim.x * blockDim.x) {
        const int ci = (int)(i % cin);
        const int t = (int)((i / cin) % kk);
        const int co = (int)(i / ((size_t)cin * kk));
        dst[i] = __float2bfloat16_rn(src[((size_t)co * cin + ci) * kk + t]);
    }
}

__global__ void copy_f32_kernel(const float* __restrict__ src, float* __restrict__ dst, size_t n) {
    for (size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (size_t)gridDim.x * blockDim.x) dst[i] = src[i];
}

// F.normalize(e, p=2, dim=-1) (vq_model.py:264): e / max(||e||, 1e-12); also the row's squared norm.
__global__ void normalize_codebook_kernel(const float* __restrict__ e, float* __restrict__ out, float* __restrict__ sq,
                                          int n, int d, int l2) {
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    float ss = 0.f;
    for (int j = 0; j < d; ++j) ss += e[(size_t)i * d + j] * e[(size_t)i * d + j];
    const float inv = l2 ? 1.0f / fmaxf(sqrtf(ss), 1e-12f) : 1.0f;
    float s2 = 0.f;
    for (int j = 0; j < d; ++j) {
        const float v = l2 ? e[(size_t)i * d + j] / fmaxf(sqrtf(ss), 1e-12f) : e[(size_t)i * d + j];
        (void)inv;
        out[(size_t)i * d + j] = v;
        s2 += v * v;
    }
    sq[i] = s2;
}

// get_codebook_entry + post_quant_conv (1x1, e_dim -> z_channels) fused; out bf16 NHWC [B*g*g, Z]
__global__ void lookup_postquant_kernel(const int32_t* __restrict__ codes, const float* __restrict__ cb, int n_e, int ed,
                                        const float* __restrict__ w /*[Z][ed]*/, const float* __restrict__ bias, int Z,
                                        bf16* __restrict__ out) {
    const int pix = blockIdx.x;
    int code = codes[pix];
    code = min(max(code, 0), n_e - 1);
    const float* e = cb + (size_t)code * ed;
    for (int c = threadIdx.x; c < Z; c += blockDim.x) {
        float acc = bias[c];
        for (int d = 0; d < ed; ++d) acc = fmaf(e[d], w[(size_t)c * ed + d], acc);
        out[(size_t)pix * Z + c] = __float2bfloat16_rn(acc);
    }
}

// GroupNorm(32) statistics, pass 1: per (image, pixel-chunk) partial sum / sum-of-squares per group.
// grid (splits, B), 256 threads; thread -> 8 contiguous channels (one 16-byte load per pixel).
__global__ void __launch_bounds__(256) gn_stats_kernel(const bf16* __restrict__ x, int HW, int C, float* __restrict__ partial) {
    // deterministic: per-thread partials go to shared memory and are combined in a fixed order (no atomics),
    // so decode_code is bit-reproducible and batch-invariant.
    __shared__ float part[256][17];   // [thread][8 sums + 8 squares], padded
    __shared__ float chs[512 * 2];
    const int b = blockIdx.y, split = blockIdx.x, splits = gridDim.x;
    const int tpp = C / 8;                       // threads per pixel (divides 256, checked on the host)
    const int ppi = 256 / tpp;                   // pixels per iteration
    const int col = threadIdx.x % tpp, prow = threadIdx.x / tpp;
    const int per = (HW + splits - 1) / splits;
    const int p0 = split * per, p1 = min(HW, p0 + per);
    float s[8], q[8];
#pragma unroll
    for (int i = 0; i < 8; ++i) { s[i] = 0.f; q[i] = 0.f; }
#pragma unroll 4
    for (int p = p0 + prow; p < p1; p += ppi) {
        float v[8];
        VecLoad<bf16, 8>::load(x + ((size_t)b * HW + p) * C + col * 8, v);
#pragma unroll
        for (int i = 0; i < 8; ++i) { s[i] += v[i]; q[i] = fmaf(v[i], v[i], q[i]); }
    }
#pragma unroll
    for (int i = 0; i < 8; ++i) { part[threadIdx.x][i] = s[i]; part[threadIdx.x][8 + i] = q[i]; }
    __syncthreads();
    for (int c = threadIdx.x; c < C; c += 256) {
        const int cc = c / 8, ci = c % 8;
        float cs = 0.f, cq = 0.f;
        for (int pr = 0; pr < ppi; ++pr) { cs += part[pr * tpp + cc][ci]; cq += part[pr * tpp + cc][8 + ci]; }
        chs[c * 2] = cs;
        chs[c * 2 + 1] = cq;
    }
    __syncthreads();
    if (threadIdx.x < 32) {
        const int cpg = C / 32, g = threadIdx.x;
        float gs = 0.f, gq = 0.f;
        for (int c = g * cpg; c < (g + 1) * cpg; ++c) { gs += chs[c * 2]; gq += chs[c * 2 + 1]; }
        float* o = partial + (((size_t)b * splits + split) * 32 + g) * 2;
        o[0] = gs;
        o[1] = gq;
    }
}

// pass 2: y = GN(x) [* sigmoid] -> bf16.  grid (chunks, B)
__global__ void __launch_bounds__(256) gn_apply_kernel(const bf16* __restrict__ x, const float* __restrict__ partial, int splits,
                                                       const float* __restrict__ gamma, const float* __restrict__ beta,
                                                       bf16* __restrict__ y, int HW, int C, int swish) {
    __shared__ float mean[32], rstd[32], var_s[32];
    __shared__ float red[8][32][2];
    const int b = blockIdx.y;
    const size_t img = (size_t)b * HW * C;
    {   // combine the per-split partials: 8 interleaved subsets in parallel, then a fixed-order sum (deterministic)
        const int g = threadIdx.x & 31, sub = threadIdx.x >> 5;
        float gs = 0.f, gq = 0.f;
        for (int sp = sub; sp < splits; sp += 8) {
            const float2 o = *reinterpret_cast<const float2*>(partial + (((size_t)b * splits + sp) * 32 + g) * 2);
            gs += o.x;
            gq += o.y;
        }
        red[sub][g][0] = gs;
        red[sub][g][1] = gq;
    }
    __syncthreads();
    if (threadIdx.x < 32) {
        float gs = 0.f, gq = 0.f;
#pragma unroll
        for (int sub = 0; sub < 8; ++sub) { gs += red[sub][threadIdx.x][0]; gq += red[sub][threadIdx.x][1]; }
        const float cnt = (float)HW * (float)(C / 32);
        const float mu = gs / cnt;
        const float var = fmaxf(gq / cnt - mu * mu, 0.f);
        mean[threadIdx.x] = mu;
        var_s[threadIdx.x] = var;
        rstd[threadIdx.x] = 1.0f / sqrtf(var + 1e-6f);
    }
    __syncthreads();
    // E[x^2] - mean^2 from fp32 sums cancels catastrophically once |mean| >> std (at |mean| / std = 100 the variance is off by
    // several percent). Such groups are recomputed here by a corrected two-pass sum around the first-pass mean over the whole
    // image: every block of the image does the same arithmetic, so the result stays deterministic, and well-conditioned groups keep
    // the one-pass statistics untouched.
    const int cpg = C / 32;
    for (int g = 0; g < 32; ++g) {
        const float mu0 = mean[g];
        if (!(mu0 * mu0 > 64.f * var_s[g])) continue;                 // |mean| / std <= 8: the one-pass variance is accurate
        const int n = HW * cpg;
        float s1 = 0.f, s2 = 0.f;
        for (int i = threadIdx.x; i < n; i += 256) {
            const int p = i / cpg;
            const float d = __bfloat162float(x[img + (size_t)p * C + g * cpg + (i - p * cpg)]) - mu0;
            s1 += d;
            s2 = fmaf(d, d, s2);
        }
        s1 = block_sum(s1, &red[0][0][0]);
        s2 = block_sum(s2, &red[0][0][0]);
        if (threadIdx.x == 0) {
            const float dm = s1 / (float)n;
            mean[g] = mu0 + dm;
            rstd[g] = 1.0f / sqrtf(fmaxf(s2 / (float)n - dm * dm, 0.f) + 1e-6f);
        }
        __syncthreads();
    }
    // Each thread owns one 8-channel column for the whole kernel: 256 threads step over the image in multiples of
    // C/8 vectors, so the per-channel scale/shift (rstd*gamma, beta - mean*rstd*gamma) is computed ONCE and the
    // inner loop is one FMA + swish per element (the first version recomputed channel/group indices with integer
    // divisions per element and ran at 19 % of HBM bandwidth).
    const int vpp = C / 8;                               // vectors per pixel; divides 256 (checked on the host)
    const int vec_per_img = HW * vpp;
    int per = (vec_per_img + gridDim.x - 1) / gridDim.x;
    per = (per + 255) / 256 * 256;                       // keep every block's start a multiple of 256 (hence of vpp)
    const int v0 = blockIdx.x * per, v1 = min(vec_per_img, v0 + per);
    const int c0 = (threadIdx.x % vpp) * 8;
    float sa[8], sb[8];
#pragma unroll
    for (int j = 0; j < 8; ++j) {
        const int c = c0 + j, g = c / cpg;
        sa[j] = rstd[g] * gamma[c];
        sb[j] = beta[c] - mean[g] * sa[j];
    }
#pragma unroll 4
    for (int i = v0 + threadIdx.x; i < v1; i += 256) {
        float v[8];
        const size_t off = img + (size_t)i * 8;
        VecLoad<bf16, 8>::load(x + off, v);
        uint32_t packed[4];
#pragma unroll
        for (int j = 0; j < 8; j += 2) {
            float t0 = fmaf(v[j], sa[j], sb[j]), t1 = fmaf(v[j + 1], sa[j + 1], sb[j + 1]);
            if (swish) {
                t0 = __fdividef(t0, 1.0f + __expf(-t0));
                t1 = __fdividef(t1, 1.0f + __expf(-t1));
            }
            __nv_bfloat162 p = __floats2bfloat162_rn(t0, t1);
            packed[j / 2] = *reinterpret_cast<uint32_t*>(&p);
        }
        *reinterpret_cast<uint4*>(y + off) = make_uint4(packed[0], packed[1], packed[2], packed[3]);
    }
}

// row softmax fp32 [rows, n] -> bf16 probabilities (AttnBlock, vq_model.py:341)
__global__ void __launch_bounds__(256) softmax_rows_kernel(const float* __restrict__ s, bf16* __restrict__ p, int n) {
    __shared__ float red[33];
    const float* row = s + (size_t)blockIdx.x * n;
    bf16* out = p + (size_t)blockIdx.x * n;
    float m = -INFINITY;
    for (int i = threadIdx.x; i < n; i += 256) m = fmaxf(m, row[i]);
    m = block_max(m, red);
    float z = 0.f;
    for (int i = threadIdx.x; i < n; i += 256) z += __expf(row[i] - m);
    z = block_sum(z, red);
    const float inv = 1.0f / z;
    for (int i = threadIdx.x; i < n; i += 256) out[i] = __float2bfloat16_rn(__expf(row[i] - m) * inv);
}

// argmin-L2 (vq_model.py:215-233): one thread per latent vector, codebook staged through shared memory in
// tiles; running (min, idx) in registers; d = (|z|^2 + |e|^2) - 2 z.e in fp32 like the reference.
constexpr int kArgminTile = 2048;
template <int ED>
__global__ void __launch_bounds__(128) argmin_kernel(const float* __restrict__ z_nchw, int B, int g, const float* __restrict__ cb,
                                                     const float* __restrict__ cbsq, int n_e, int l2, int64_t* __restrict__ out) {
    extern __shared__ float sm[];  // [tile][ED] + [tile]
    float* se = sm;
    float* sq = sm + kArgminTile * ED;
    const int hw = g * g, nz = B * hw;
    const int i = blockIdx.x * 128 + threadIdx.x;
    float z[ED], zz = 0.f;
    if (i < nz) {
        const int b = i / hw, pix = i - b * hw;
        float ss = 0.f;
#pragma unroll
        for (int d = 0; d < ED; ++d) { z[d] = z_nchw[((size_t)b * ED + d) * hw + pix]; ss += z[d] * z[d]; }
        if (l2) {
            const float nrm = fmaxf(sqrtf(ss), 1e-12f);
#pragma unroll
            for (int d = 0; d < ED; ++d) z[d] = z[d] / nrm;
        }
#pragma unroll
        for (int d = 0; d < ED; ++d) zz += z[d] * z[d];
    } else {
#pragma unroll
        for (int d = 0; d < ED; ++d) z[d] = 0.f;
    }
    float best = INFINITY;
    int besti = 0;
    for (int t0 = 0; t0 < n_e; t0 += kArgminTile) {
        const int tn = min(kArgminTile, n_e - t0);
        __syncthreads();
        for (int k = threadIdx.x; k < tn * ED; k += 128) se[k] = cb[(size_t)t0 * ED + k];
        for (int k = threadIdx.x; k < tn; k += 128) sq[k] = cbsq[t0 + k];
        __syncthreads();
        for (int j = 0; j < tn; ++j) {
            float dot = 0.f;
#pragma unroll
            for (int d = 0; d < ED; ++d) dot = fmaf(z[d], se[j * ED + d], dot);
            const float dist = (zz + sq[j]) - 2.0f * dot;
            if (dist < best) { best = dist; besti = t0 + j; }
        }
    }
    if (i < nz) out[i] = besti;
}


// ------------------------------------------------------------------------------------------------ encoder front / pixel back
// Encoder.conv_in (vq_model.py:70,101): 3x3 pad 1, 3 -> ch, evaluated in fp32 straight from the fp32 NCHW image
// (K = 27 is far too thin for a tensor-core tile); writes the bf16 NHWC activation the rest of the encoder consumes.
// One work item = 4 adjacent pixels of a row x 8 output channels (each weight read from shared memory feeds 4 pixels,
// each input value 3 taps); the grid is persistent so the transposed weights ([tap][ch]) are staged once per CTA.
__global__ void __launch_bounds__(256) conv_in_rgb_kernel(const float* __restrict__ x, const float* __restrict__ w,
                                                          const float* __restrict__ bias, bf16* __restrict__ out, int B, int H,
                                                          int W, int ch) {
    extern __shared__ float ws[];   // [27][ch] then bias [ch]
    for (int i = threadIdx.x; i < 27 * ch; i += blockDim.x) {
        const int c = i / 27, t = i - c * 27;               // source layout [ch][cin=3][ky][kx] -> t = cin*9 + ky*3 + kx
        ws[t * ch + c] = w[i];
    }
    for (int i = threadIdx.x; i < ch; i += blockDim.x) ws[27 * ch + i] = bias[i];
    __syncthreads();
    const int oct = ch / 8, xg = W / 4;
    const long long total = (long long)B * H * xg * oct;
    for (long long item = (long long)blockIdx.x * blockDim.x + threadIdx.x; item < total; item += (long long)gridDim.x * blockDim.x) {
        const int o = (int)(item % oct);
        long long rest = item / oct;
        const int x0 = (int)(rest % xg) * 4;
        rest /= xg;
        const int yy = (int)(rest % H);
        const int b = (int)(rest / H);
        float acc[4][8];
#pragma unroll
        for (int p = 0; p < 4; ++p)
#pragma unroll
            for (int j = 0; j < 8; ++j) acc[p][j] = ws[27 * ch + o * 8 + j];
#pragma unroll
        for (int ci = 0; ci < 3; ++ci) {
            const float* plane = x + ((long long)b * 3 + ci) * H * W;
#pragma unroll
            for (int ky = 0; ky < 3; ++ky) {
                const int y2 = yy + ky - 1;
                float v[6];
                const bool yok = (unsigned)y2 < (unsigned)H;
#pragma unroll
                for (int i = 0; i < 6; ++i) {
                    const int x2 = x0 + i - 1;
                    v[i] = (yok && (unsigned)x2 < (unsigned)W) ? plane[(long long)y2 * W + x2] : 0.f;
                }
#pragma unroll
                for (int kx = 0; kx < 3; ++kx) {
                    const float4* wr = reinterpret_cast<const float4*>(ws + (ci * 9 + ky * 3 + kx) * ch + o * 8);
                    const float4 w0 = wr[0], w1 = wr[1];
                    const float wv[8] = {w0.x, w0.y, w0.z, w0.w, w1.x, w1.y, w1.z, w1.w};
#pragma unroll
                    for (int p = 0; p < 4; ++p)
#pragma unroll
                        for (int j = 0; j < 8; ++j) acc[p][j] = fmaf(v[p + kx], wv[j], acc[p][j]);
                }
            }
        }
#pragma unroll
        for (int p = 0; p < 4; ++p) {
            uint4 pk;
            __nv_bfloat162* p2 = reinterpret_cast<__nv_bfloat162*>(&pk);
#pragma unroll
            for (int j = 0; j < 4; ++j) p2[j] = __floats2bfloat162_rn(acc[p][2 * j], acc[p][2 * j + 1]);
            *reinterpret_cast<uint4*>(out + (((long long)b * H + yy) * W + x0 + p) * ch + o * 8) = pk;
        }
    }
}

// VectorQuantizer.forward's returned tensor (vq_model.py:233,252-255): z_q = z + (e[idx] - z) with z L2-normalised
// when codebook_l2_norm; NCHW in, NCHW out. One thread per latent position.
__global__ void quant_out_kernel(const float* __restrict__ z, const int64_t* __restrict__ idx, const float* __restrict__ cb,
                                 int B, int hw, int ed, int l2norm, float* __restrict__ out) {
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= B * hw) return;
    const int b = i / hw, p = i - b * hw;
    const float* zp = z + (long long)b * ed * hw + p;
    float inv = 1.f;
    if (l2norm) {
        float ss = 0.f;
        for (int c = 0; c < ed; ++c) ss = __fadd_rn(ss, __fmul_rn(zp[(long long)c * hw], zp[(long long)c * hw]));
        inv = fmaxf(sqrtf(ss), 1e-12f);                     // F.normalize: x / max(||x||, eps)
    }
    const float* e = cb + idx[i] * ed;
    for (int c = 0; c < ed; ++c) {
        const float zn = l2norm ? __fdiv_rn(zp[(long long)c * hw], inv) : zp[(long long)c * hw];
        out[((long long)b * ed + c) * hw + p] = __fadd_rn(zn, __fsub_rn(e[c], zn));
    }
}

// Pixel finishing of the DDP sampler (sample_c2i_ddp.py:141-143) in one pass: optional bicubic resize
// (F.interpolate(mode='bicubic'), align_corners=False, A = -0.75, border-clamped taps, no antialias), then
// clamp(127.5 x + 128, 0, 255) -> uint8 (truncation) in NHWC. fp32 NCHW in. One thread per output pixel, all C channels.
__device__ __forceinline__ void cubic_coeffs(float t, float* c) {
    const float A = -0.75f;
    const float x0 = t + 1.f, x3 = 2.f - t, x2 = 1.f - t;
    c[0] = ((A * x0 - 5.f * A) * x0 + 8.f * A) * x0 - 4.f * A;
    c[1] = ((A + 2.f) * t - (A + 3.f)) * t * t + 1.f;
    c[2] = ((A + 2.f) * x2 - (A + 3.f)) * x2 * x2 + 1.f;
    c[3] = ((A * x3 - 5.f * A) * x3 + 8.f * A) * x3 - 4.f * A;
}

// One output value: tap sums in the association order of ATen's CUDA kernel (x taps first, then y).
__device__ __forceinline__ float pixel_value(const float* __restrict__ plane, int H, int W, bool resize, int oy, int ox, int iy, int ix,
                                             const float* cy, const float* cx) {
    float v;
    if (!resize) {
        v = plane[(long long)oy * W + ox];
    } else {
        v = 0.f;
#pragma unroll
        for (int i = 0; i < 4; ++i) {
            const int yy = min(max(iy - 1 + i, 0), H - 1);
            float r = 0.f;
#pragma unroll
            for (int j = 0; j < 4; ++j) {
                const int xx = min(max(ix - 1 + j, 0), W - 1);
                r += plane[(long long)yy * W + xx] * cx[j];
            }
            v += r * cy[i];
        }
    }
    v = __fadd_rn(__fmul_rn(127.5f, v), 128.0f);
    return fminf(fmaxf(v, 0.f), 255.f);
}

// PX output pixels per thread along x. PX = 4 with C = 3 packs the 12 output bytes into three 32-bit stores and, without
// a resize, reads each plane with one 128-bit load; PX = 1 is the general fallback (any C, any width).
template <int PX>
__global__ void __launch_bounds__(256) pixels_to_u8_kernel(const float* __restrict__ in, int B, int C, int H, int W, int OH, int OW,
                                                           uint8_t* __restrict__ out) {
    const long long gid = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    const int groups = OW / PX;
    if (gid >= (long long)B * OH * groups) return;
    const int ox0 = (int)(gid % groups) * PX;
    const int oy = (int)((gid / groups) % OH);
    const int b = (int)(gid / ((long long)groups * OH));
    const bool resize = OH != H || OW != W;
    float cy[4] = {0.f, 0.f, 0.f, 0.f};
    int iy = oy;
    const float sy = (float)H / (float)OH, sx = (float)W / (float)OW;
    if (resize) {
        const float fy = sy * ((float)oy + 0.5f) - 0.5f;
        iy = (int)floorf(fy);
        cubic_coeffs(fy - (float)iy, cy);
    }
    if (PX == 4) {
        uint8_t bytes[12];
        if (!resize) {
#pragma unroll
            for (int c = 0; c < 3; ++c) {
                const float4 v = *reinterpret_cast<const float4*>(in + (((long long)b * 3 + c) * H + oy) * W + ox0);
                const float f[4] = {v.x, v.y, v.z, v.w};
#pragma unroll
                for (int p = 0; p < 4; ++p)
                    bytes[p * 3 + c] = (uint8_t)fminf(fmaxf(__fadd_rn(__fmul_rn(127.5f, f[p]), 128.0f), 0.f), 255.f);
            }
        } else {
#pragma unroll
            for (int p = 0; p < 4; ++p) {
                const float fx = sx * ((float)(ox0 + p) + 0.5f) - 0.5f;
                const int ix = (int)floorf(fx);
                float cx[4];
                cubic_coeffs(fx - (float)ix, cx);
#pragma unroll
                for (int c = 0; c < 3; ++c)
                    bytes[p * 3 + c] = (uint8_t)pixel_value(in + ((long long)b * 3 + c) * H * W, H, W, true, oy, ox0 + p, iy, ix, cy, cx);
            }
        }
        uint32_t* dst = reinterpret_cast<uint32_t*>(out + (((long long)b * OH + oy) * OW + ox0) * 3);
#pragma unroll
        for (int w = 0; w < 3; ++w)
            dst[w] = (uint32_t)bytes[4 * w] | ((uint32_t)bytes[4 * w + 1] << 8) | ((uint32_t)bytes[4 * w + 2] << 16) |
                     ((uint32_t)bytes[4 * w + 3] << 24);
    } else {
        float cx[4] = {0.f, 0.f, 0.f, 0.f};
        int ix = ox0;
        if (resize) {
            const float fx = sx * ((float)ox0 + 0.5f) - 0.5f;
            ix = (int)floorf(fx);
            cubic_coeffs(fx - (float)ix, cx);
        }
        for (int c = 0; c < C; ++c)   // truncation toward zero, like Tensor.to(torch.uint8)
            out[(((long long)b * OH + oy) * OW + ox0) * C + c] =
                (uint8_t)pixel_value(in + ((long long)b * C + c) * H * W, H, W, resize, oy, ox0, iy, ix, cy, cx);
    }
}

// ------------------------------------------------------------------------------------------------ model structs
struct HostTensor { const float* p = nullptr; int64_t shape[4] = {0, 0, 0, 0}; int ndim = 0; };
struct ConvW { bf16* w = nullptr; bf16* w_phase = nullptr; const float* bias = nullptr; int cout = 0, cin = 0, k = 0; };
struct NormW { const float* gamma = nullptr; const float* beta = nullptr; int c = 0; };
struct ResW { NormW n1, n2; ConvW c1, c2, nin; bool has_nin = false; int cin = 0, cout = 0; };
struct AttnW { NormW norm; ConvW qk, v, proj; float* qk_bias = nullptr; int c = 0; };
struct LevelW { std::vector<ResW> res; std::vector<AttnW> attn; bool up = false; ConvW upconv; };   // upconv: up- or downsample conv

}  // namespace

struct lg_vq {
    lg_vq_cfg cfg;
    int device = 0;
    std::unordered_map<std::string, HostTensor> t;
    std::vector<void*> owned;   // cudaMalloc'ed repacked weights
    bool finalized = false;
    ConvW conv_in, conv_out;
    ResW mid0, mid2;
    AttnW mid1;
    std::vector<LevelW> levels;
    NormW norm_out;
    float* codebook = nullptr;  // normalised [n_e, e_dim]
    float* codebook_sq = nullptr;
    const float* pq_w = nullptr;
    const float* pq_b = nullptr;
    // encoder (optional: built when encoder.* and quant_conv.* are bound)
    bool has_encoder = false;
    const float* enc_in_w = nullptr;   // fp32 [ch,3,3,3], applied in fp32 by conv_in_rgb_kernel
    const float* enc_in_b = nullptr;
    std::vector<LevelW> enc_levels;
    ResW enc_mid0, enc_mid2;
    AttnW enc_mid1;
    NormW enc_norm_out;
    ConvW enc_conv_out, quant_conv;

    ~lg_vq() { for (void* p : owned) cudaFree(p); }
};

namespace {

int get(lg_vq* v, const std::string& name, std::initializer_list<int64_t> shape, const float** out) {
    auto it = v->t.find(name);
    LG_REQUIRE(it != v->t.end(), "missing weight '%s'", name.c_str());
    const HostTensor& h = it->second;
    LG_REQUIRE(h.ndim == (int)shape.size(), "weight '%s': %d dims, expected %d", name.c_str(), h.ndim, (int)shape.size());
    int i = 0;
    for (int64_t s : shape) {
        LG_REQUIRE(h.shape[i] == s, "weight '%s' dim %d is %lld, expected %lld", name.c_str(), i, (long long)h.shape[i], (long long)s);
        ++i;
    }
    *out = h.p;
    return 0;
}

template <typename T> int dev_alloc(lg_vq* v, size_t n, T** out) {
    void* p = nullptr;
    LG_CUDA_OK(cudaMalloc(&p, n * sizeof(T)));
    v->owned.push_back(p);
    *out = (T*)p;
    return 0;
}

int make_conv(lg_vq* v, const std::string& name, int cout, int cin, int k, ConvW* cw, cudaStream_t st) {
    const float* w = nullptr;
    const float* b = nullptr;
    LG_TRY(get(v, name + ".weight", {cout, cin, k, k}, &w));
    LG_TRY(get(v, name + ".bias", {cout}, &b));
    LG_REQUIRE(cin % 8 == 0, "conv '%s': Cin=%d must be a multiple of 8", name.c_str(), cin);
    bf16* d = nullptr;
    LG_TRY(dev_alloc(v, (size_t)cout * cin * k * k, &d));
    repack_conv_kernel<<<132 * 4, 256, 0, st>>>(w, d, cout, cin, k * k);
    LG_LAUNCH_CHECK();
    cw->w = d; cw->bias = b; cw->cout = cout; cw->cin = cin; cw->k = k;
    return 0;
}

int make_norm(lg_vq* v, const std::string& name, int c, NormW* nw) {
    LG_REQUIRE(c % 32 == 0 && c % 8 == 0 && c <= 512 && (256 % (c / 8)) == 0, "GroupNorm '%s': unsupported channel count %d", name.c_str(), c);
    LG_TRY(get(v, name + ".weight", {c}, &nw->gamma));
    LG_TRY(get(v, name + ".bias", {c}, &nw->beta));
    nw->c = c;
    return 0;
}

int make_res(lg_vq* v, const std::string& p, int cin, int cout, ResW* r, cudaStream_t st) {
    r->cin = cin; r->cout = cout;
    LG_TRY(make_norm(v, p + ".norm1", cin, &r->n1));
    LG_TRY(make_conv(v, p + ".conv1", cout, cin, 3, &r->c1, st));
    LG_TRY(make_norm(v, p + ".norm2", cout, &r->n2));
    LG_TRY(make_conv(v, p + ".conv2", cout, cout, 3, &r->c2, st));
    r->has_nin = cin != cout;
    if (r->has_nin) LG_TRY(make_conv(v, p + ".nin_shortcut", cout, cin, 1, &r->nin, st));
    return 0;
}

int make_attn(lg_vq* v, const std::string& p, int c, AttnW* a, cudaStream_t st) {
    a->c = c;
    LG_TRY(make_norm(v, p + ".norm", c, &a->norm));
    ConvW q, k;
    LG_TRY(make_conv(v, p + ".q", c, c, 1, &q, st));
    LG_TRY(make_conv(v, p + ".k", c, c, 1, &k, st));
    LG_TRY(make_conv(v, p + ".v", c, c, 1, &a->v, st));
    LG_TRY(make_conv(v, p + ".proj_out", c, c, 1, &a->proj, st));
    // q | k as one [2C, C] GEMM operand
    bf16* qk = nullptr;
    LG_TRY(dev_alloc(v, (size_t)2 * c * c, &qk));
    LG_CUDA_OK(cudaMemcpyAsync(qk, q.w, (size_t)c * c * sizeof(bf16), cudaMemcpyDeviceToDevice, st));
    LG_CUDA_OK(cudaMemcpyAsync(qk + (size_t)c * c, k.w, (size_t)c * c * sizeof(bf16), cudaMemcpyDeviceToDevice, st));
    LG_TRY(dev_alloc(v, (size_t)2 * c, &a->qk_bias));
    copy_f32_kernel<<<1, 256, 0, st>>>(q.bias, a->qk_bias, c);
    LG_LAUNCH_CHECK();
    copy_f32_kernel<<<1, 256, 0, st>>>(k.bias, a->qk_bias + c, c);
    LG_LAUNCH_CHECK();
    a->qk.w = qk; a->qk.bias = a->qk_bias; a->qk.cout = 2 * c; a->qk.cin = c; a->qk.k = 1;
    return 0;
}

// workspace carve (per chunk of Bc images)
struct VqWs {
    bf16 *X, *T, *U, *VT, *P;
    float *S, *gn, *Z;
    size_t bytes;
    int attn_bc;   // images per attention chunk
    size_t gn_floats = 0;            // capacity of gn
    // GroupNorm statistics produced by the drain of the conv that wrote `gn_src` (conv_tcw_kernel): run_gn skips its statistics pass
    // when it is asked to normalise exactly that tensor
    const bf16* gn_src = nullptr;
    int gn_splits = 0;
};

size_t a256(size_t v) { return (v + 255) / 256 * 256; }

VqWs carve_vq(const lg_vq* v, char* base, int Bc, int g) {
    const lg_vq_cfg& c = v->cfg;
    size_t maxact = 0;
    int res = g;
    for (int i = c.n_mult - 1; i >= 0; --i) {
        const size_t ch = (size_t)c.ch * c.ch_mult[i];
        // a level runs at `res`; its upsample conv writes [2res, 2res, ch]
        maxact = std::max(maxact, (size_t)Bc * res * res * ch);
        if (i != 0) { maxact = std::max(maxact, (size_t)Bc * 4 * res * res * ch); res *= 2; }
    }
    const size_t Cd = (size_t)c.ch * c.ch_mult[c.n_mult - 1];
    const size_t N = (size_t)g * g;
    maxact = std::max(maxact, (size_t)Bc * N * std::max((size_t)c.z_channels, 2 * Cd));
    // attention scores: chunk images so S (fp32) stays <= 256 MiB
    int abc = (int)std::max<size_t>(1, std::min<size_t>(Bc, (256ull << 20) / (N * N * 4)));
    VqWs w;
    size_t off = 0;
    auto take = [&](size_t b) { char* p = base ? base + off : nullptr; off += a256(b); return p; };
    w.X = (bf16*)take(maxact * 2);
    w.T = (bf16*)take(maxact * 2);
    w.U = (bf16*)take(maxact * 2);
    w.VT = (bf16*)take((size_t)Bc * N * Cd * 2);
    w.S = (float*)take((size_t)abc * N * N * 4);
    w.P = (bf16*)take((size_t)abc * N * N * 2);
    // statistics partials: gn_stats_kernel uses <= 64 splits per image, the conv drains one per 16x16-pixel tile of the largest output
    {
        int rmax = g;
        for (int i = 0; i + 1 < c.n_mult; ++i) rmax *= 2;
        const size_t splits = std::max<size_t>(64, (size_t)((rmax + 15) / 16) * ((rmax + 15) / 16) * 4);
        w.gn_floats = (size_t)Bc * splits * 32 * 2;
        w.gn = (float*)take(w.gn_floats * 4);
    }
    w.Z = (float*)take((size_t)Bc * N * c.codebook_embed_dim * 4);   // encoder output z (fp32 NCHW) ahead of the argmin
    w.bytes = off;
    w.attn_bc = abc;
    return w;
}

size_t per_image_bytes(const lg_vq* v, int g) { return carve_vq(v, nullptr, 1, g).bytes; }

int chunk_images(const lg_vq* v, int B, int g) {
    const size_t cap = 6ull << 30;
    const size_t per = per_image_bytes(v, g);
    return (int)std::max<size_t>(1, std::min<size_t>(B, cap / std::max<size_t>(per, 1)));
}

// ---- layer launchers --------------------------------------------------------------------------------
// up: 0 = same resolution, 1 = nearest-2x upsample folded in, 2 = Downsample (pad right/bottom, stride 2)
// *path (optional): 0 = mma.sync gather kernel, 1 = conv_tc_kernel, 2 = conv_tcw_kernel
int run_conv(const ConvW& cw, const bf16* in, int B, int Hin, int Win, int up, const bf16* residual, bf16* out_bf,
             float* out_nchw, cudaStream_t st, uint8_t* out_u8 = nullptr, VqWs* ws = nullptr, int* path = nullptr) {
    if (ws && out_bf && ws->gn_src == out_bf) ws->gn_src = nullptr;          // the tensor the statistics described is being overwritten
    if (lg_env_flag("LG_CONV_TC", 1) && conv_tc_supported(Hin, Win, cw.cin, cw.cout, cw.k, up, out_nchw != nullptr || out_u8 != nullptr) &&
        (up != 1 || cw.w_phase)) {
        int splits = 0;
        LG_PROF(PC_VQ_CONV, st, launch_conv_tc(in, B, Hin, Win, cw.cin, up == 1 ? cw.w_phase : cw.w, cw.bias, cw.cout, cw.k, up, residual,
                                               out_bf, out_nchw, st, out_u8, ws ? ws->gn : nullptr, ws ? ws->gn_floats : 0, ws ? &splits : nullptr,
                                               path));
        if (ws && splits > 0) { ws->gn_src = out_bf; ws->gn_splits = splits; }
        return 0;
    }
    LG_REQUIRE(!out_u8, "uint8 output needs the wgmma conv path (Cin %% 64 == 0, LG_CONV_TC=1)");
    if (path) *path = 0;
    const int Hout = up == 1 ? 2 * Hin : (up == 2 ? Hin / 2 : Hin), Wout = up == 1 ? 2 * Win : (up == 2 ? Win / 2 : Win);
    const int M = B * Hout * Wout, K = cw.k * cw.k * cw.cin;
    mma::ConvA al{in, Hin, Win, cw.cin, Hout, Wout, cw.k, up, M};
    mma::BRows bw{cw.w, cw.w, cw.cout, K, 0, cw.cout};
    EpiVq e{};
    e.bias = cw.bias; e.residual = residual; e.ldr = cw.cout; e.out_bf = out_bf; e.ldo = cw.cout; e.scale = 1.f;
    e.N = cw.cout;
    if (out_nchw) { e.out_f32 = out_nchw; e.nchw = 1; e.hw = Hout * Wout; e.out_bf = nullptr; }
    LG_PROF(PC_VQ_CONV, st, launch_vq_gemm(al, bw, M, cw.cout, K, 1, e, st));
    return 0;
}

int run_gn(const NormW& nw, const bf16* x, bf16* y, int B, int HW, int swish, float* gnbuf, cudaStream_t st, VqWs* ws = nullptr) {
    int splits = (int)std::min<long long>(64, std::max<long long>(1, (long long)HW * nw.c / 8 / 2048));
    if (ws && ws->gn_src == x && ws->gn_splits > 0) {
        splits = ws->gn_splits;                  // the producing conv's drain already wrote the partial statistics of x
    } else {
        prof_begin(PC_VQ_GN_STATS, st);
        gn_stats_kernel<<<dim3(splits, B), 256, 0, st>>>(x, HW, nw.c, gnbuf);
        prof_end(st);
        LG_LAUNCH_CHECK();
    }
    if (ws) ws->gn_src = nullptr;                // gnbuf is consumed below; y (and any later writer of x) invalidates it anyway
    int chunks = (int)std::min<long long>(256, std::max<long long>(1, (long long)HW * (nw.c / 8) / 1024));
    prof_begin(PC_VQ_GN_APPLY, st);
    gn_apply_kernel<<<dim3(chunks, B), 256, 0, st>>>(x, gnbuf, splits, nw.gamma, nw.beta, y, HW, nw.c, swish);
    prof_end(st);
    LG_LAUNCH_CHECK();
    return 0;
}

// ResnetBlock (vq_model.py:298-314). x lives in w.X and the result is left in w.X.
int run_res(const ResW& r, VqWs& w, int B, int H, int W, cudaStream_t st) {
    const int HW = H * W;
    LG_TRY(run_gn(r.n1, w.X, w.T, B, HW, 1, w.gn, st, &w));
    LG_TRY(run_conv(r.c1, w.T, B, H, W, 0, nullptr, w.U, nullptr, st, nullptr, &w));
    LG_TRY(run_gn(r.n2, w.U, w.T, B, HW, 1, w.gn, st, &w));
    if (r.has_nin) {
        LG_TRY(run_conv(r.nin, w.X, B, H, W, 0, nullptr, w.U, nullptr, st));     // shortcut -> U
        LG_TRY(run_conv(r.c2, w.T, B, H, W, 0, w.U, w.X, nullptr, st, nullptr, &w));  // X = conv2 + shortcut
    } else {
        LG_TRY(run_conv(r.c2, w.T, B, H, W, 0, w.X, w.X, nullptr, st, nullptr, &w));  // in-place residual
    }
    return 0;
}

// AttnBlock (vq_model.py:327-351), single head over N = H*W tokens, C channels. In/out: w.X.
int run_attn(const AttnW& a, VqWs& w, int B, int H, int W, cudaStream_t st) {
    const int N = H * W, C = a.c;
    LG_REQUIRE(N % 8 == 0, "attention block: token count %d must be a multiple of 8", N);
    LG_TRY(run_gn(a.norm, w.X, w.T, B, N, 0, w.gn, st, &w));                      // hn -> T  [B*N, C]
    {   // q | k  -> U [B*N, 2C]
        mma::DenseA al{w.T, C, 0, B * N};
        mma::BRows bw{a.qk.w, a.qk.w, 2 * C, C, 0, 2 * C};
        EpiVq e{}; e.bias = a.qk.bias; e.out_bf = w.U; e.ldo = 2 * C; e.scale = 1.f; e.N = 2 * C;
        LG_PROF(PC_VQ_ATTN, st, launch_vq_gemm(al, bw, B * N, 2 * C, C, 1, e, st));
    }
    {   // V^T[b] = Wv * hn[b]^T + bv  -> VT [B][C][N]   (A = Wv shared, "weights" = hn[b])
        mma::DenseA al{a.v.w, C, 0, C};
        mma::BRows bw{w.T, w.T, N, C, (long long)N * C, N};
        EpiVq e{}; e.bias = a.v.bias; e.bias_by_row = 1; e.out_bf = w.VT; e.ldo = N; e.out_batch_stride = (long long)C * N;
        e.scale = 1.f; e.N = N;
        LG_PROF(PC_VQ_ATTN, st, launch_vq_gemm(al, bw, C, N, C, B, e, st));
    }
    const float scale = 1.0f / sqrtf((float)C);                                   // int(c)**(-0.5), :338
    for (int b0 = 0; b0 < B; b0 += w.attn_bc) {
        const int bc = std::min(w.attn_bc, B - b0);
        {   // S[b] = scale * q[b] k[b]^T  (fp32)
            mma::DenseA al{w.U + (size_t)b0 * N * 2 * C, 2 * C, (long long)N * 2 * C, N};
            mma::BRows bw{w.U + (size_t)b0 * N * 2 * C + C, nullptr, N, 2 * C, (long long)N * 2 * C, N};
            bw.Wb = bw.Wa;
            EpiVq e{}; e.out_f32 = w.S; e.ldo = N; e.out_batch_stride = (long long)N * N; e.scale = scale; e.N = N;
            LG_PROF(PC_VQ_ATTN, st, launch_vq_gemm(al, bw, N, N, C, bc, e, st));
        }
        prof_begin(PC_VQ_ATTN, st);
        softmax_rows_kernel<<<bc * N, 256, 0, st>>>(w.S, w.P, N);
        prof_end(st);
        LG_LAUNCH_CHECK();
        {   // O[b] = P[b] V[b]  -> T [B*N, C]
            mma::DenseA al{w.P, N, (long long)N * N, N};
            mma::BRows bw{w.VT + (size_t)b0 * C * N, nullptr, C, N, (long long)C * N, C};
            bw.Wb = bw.Wa;
            EpiVq e{}; e.out_bf = w.T + (size_t)b0 * N * C; e.ldo = C; e.out_batch_stride = (long long)N * C; e.scale = 1.f; e.N = C;
            LG_PROF(PC_VQ_ATTN, st, launch_vq_gemm(al, bw, N, C, N, bc, e, st));
        }
    }
    // x = x + proj_out(O)
    return run_conv(a.proj, w.T, B, H, W, 0, w.X, w.X, nullptr, st, nullptr, &w);
}

}  // namespace

extern "C" {

int lg_vq_create(const lg_vq_cfg* cfg, int device, lg_vq** out) {
    LG_REQUIRE(cfg && out, "lg_vq_create: null argument");
    LG_REQUIRE(cfg->n_mult >= 1 && cfg->n_mult <= 8, "bad ch_mult length %d", cfg->n_mult);
    LG_REQUIRE(cfg->codebook_embed_dim == 8 || cfg->codebook_embed_dim == 4 || cfg->codebook_embed_dim == 16 ||
                   cfg->codebook_embed_dim == 32, "codebook_embed_dim %d unsupported (4, 8, 16, 32)", cfg->codebook_embed_dim);
    LG_REQUIRE(cfg->num_res_blocks >= 1, "bad num_res_blocks");
    lg_vq* v = new lg_vq();
    v->cfg = *cfg;
    v->device = device;
    *out = v;
    return 0;
}

void lg_vq_destroy(lg_vq* v) {
    if (!v) return;
    DeviceGuard guard(v->device);
    delete v;
}

int lg_vq_bind_weight(lg_vq* v, const char* name, const void* dev_ptr, const int64_t* shape, int ndim) {
    LG_REQUIRE(v && name && dev_ptr && shape && ndim >= 1 && ndim <= 4, "lg_vq_bind_weight: bad argument");
    HostTensor h;
    h.p = (const float*)dev_ptr;
    h.ndim = ndim;
    for (int i = 0; i < ndim; ++i) h.shape[i] = shape[i];
    v->t[name] = h;
    v->finalized = false;
    return 0;
}

int lg_vq_finalize(lg_vq* v, void* stream) {
    cudaStream_t st = (cudaStream_t)stream;
    LG_REQUIRE(v, "null vq");
    DeviceGuard guard(v->device);
    for (void* p : v->owned) cudaFree(p);
    v->owned.clear();
    v->levels.clear();
    const lg_vq_cfg& c = v->cfg;
    const int n = c.n_mult, nrb = c.num_res_blocks;
    int block_in = c.ch * c.ch_mult[n - 1];
    const float* e = nullptr;
    LG_TRY(get(v, "quantize.embedding.weight", {c.codebook_size, c.codebook_embed_dim}, &e));
    LG_TRY(dev_alloc(v, (size_t)c.codebook_size * c.codebook_embed_dim, &v->codebook));
    LG_TRY(dev_alloc(v, (size_t)c.codebook_size, &v->codebook_sq));
    normalize_codebook_kernel<<<cdiv(c.codebook_size, 256), 256, 0, st>>>(e, v->codebook, v->codebook_sq, c.codebook_size,
                                                                           c.codebook_embed_dim, c.l2_norm);
    LG_LAUNCH_CHECK();
    LG_TRY(get(v, "post_quant_conv.weight", {c.z_channels, c.codebook_embed_dim, 1, 1}, &v->pq_w));
    LG_TRY(get(v, "post_quant_conv.bias", {c.z_channels}, &v->pq_b));
    LG_TRY(make_conv(v, "decoder.conv_in", block_in, c.z_channels, 3, &v->conv_in, st));
    LG_TRY(make_res(v, "decoder.mid.0", block_in, block_in, &v->mid0, st));
    LG_TRY(make_attn(v, "decoder.mid.1", block_in, &v->mid1, st));
    LG_TRY(make_res(v, "decoder.mid.2", block_in, block_in, &v->mid2, st));
    for (int bi = 0; bi < n; ++bi) {
        const int i_level = n - 1 - bi;
        const int block_out = c.ch * c.ch_mult[i_level];
        LevelW lv;
        for (int j = 0; j < nrb + 1; ++j) {
            const std::string p = "decoder.conv_blocks." + std::to_string(bi);
            ResW r;
            LG_TRY(make_res(v, p + ".res." + std::to_string(j), block_in, block_out, &r, st));
            lv.res.push_back(r);
            block_in = block_out;
            if (i_level == n - 1) {
                AttnW a;
                LG_TRY(make_attn(v, p + ".attn." + std::to_string(j), block_in, &a, st));
                lv.attn.push_back(a);
            }
        }
        lv.up = i_level != 0;
        if (lv.up) {
            const std::string un = "decoder.conv_blocks." + std::to_string(bi) + ".upsample.conv";
            LG_TRY(make_conv(v, un, block_in, block_in, 3, &lv.upconv, st));
            if (block_in % 64 == 0) {   // pre-summed 2x2 phase weights for the wgmma upsample path (conv_tc.cu)
                const float* wf = nullptr;
                LG_TRY(get(v, un + ".weight", {block_in, block_in, 3, 3}, &wf));
                LG_TRY(dev_alloc(v, (size_t)16 * block_in * block_in, &lv.upconv.w_phase));
                LG_TRY(conv_tc_make_phase_weights(wf, lv.upconv.w_phase, block_in, block_in, st));
            }
        }
        v->levels.push_back(lv);
    }
    LG_TRY(make_norm(v, "decoder.norm_out", block_in, &v->norm_out));
    LG_TRY(make_conv(v, "decoder.conv_out", 3, block_in, 3, &v->conv_out, st));
    // ---- encoder (vq_model.py:64-97) + quant_conv (:35): only when the caller bound those tensors
    v->enc_levels.clear();
    v->has_encoder = v->t.count("encoder.conv_in.weight") && v->t.count("quant_conv.weight");
    if (v->has_encoder) {
        LG_REQUIRE(c.ch % 8 == 0, "encoder: ch=%d must be a multiple of 8", c.ch);
        LG_TRY(get(v, "encoder.conv_in.weight", {c.ch, 3, 3, 3}, &v->enc_in_w));
        LG_TRY(get(v, "encoder.conv_in.bias", {c.ch}, &v->enc_in_b));
        int bin = c.ch;
        for (int i_level = 0; i_level < n; ++i_level) {
            const int bout = c.ch * c.ch_mult[i_level];
            const std::string p = "encoder.conv_blocks." + std::to_string(i_level);
            LevelW lv;
            for (int j = 0; j < nrb; ++j) {
                ResW r;
                LG_TRY(make_res(v, p + ".res." + std::to_string(j), bin, bout, &r, st));
                lv.res.push_back(r);
                bin = bout;
                if (i_level == n - 1) {
                    AttnW a;
                    LG_TRY(make_attn(v, p + ".attn." + std::to_string(j), bin, &a, st));
                    lv.attn.push_back(a);
                }
            }
            lv.up = i_level != n - 1;   // here: has a Downsample conv
            if (lv.up) LG_TRY(make_conv(v, p + ".downsample.conv", bin, bin, 3, &lv.upconv, st));
            v->enc_levels.push_back(lv);
        }
        LG_TRY(make_res(v, "encoder.mid.0", bin, bin, &v->enc_mid0, st));
        LG_TRY(make_attn(v, "encoder.mid.1", bin, &v->enc_mid1, st));
        LG_TRY(make_res(v, "encoder.mid.2", bin, bin, &v->enc_mid2, st));
        LG_TRY(make_norm(v, "encoder.norm_out", bin, &v->enc_norm_out));
        LG_TRY(make_conv(v, "encoder.conv_out", c.z_channels, bin, 3, &v->enc_conv_out, st));
        LG_TRY(make_conv(v, "quant_conv", c.codebook_embed_dim, c.z_channels, 1, &v->quant_conv, st));
    }
    LG_CUDA_OK(cudaStreamSynchronize(st));
    v->finalized = true;
    return 0;
}

int lg_vq_workspace_bytes(lg_vq* v, int B, int grid, size_t* bytes) {
    LG_REQUIRE(v && bytes && B > 0 && grid > 0, "lg_vq_workspace_bytes: bad argument");
    const int Bc = chunk_images(v, B, grid);
    *bytes = carve_vq(v, nullptr, Bc, grid).bytes;
    return 0;
}

static int vq_decode_impl(lg_vq* v, const int32_t* codes, int B, int grid, void* dev_ws, size_t ws_bytes, float* out_nchw, uint8_t* out_u8,
                          void* stream) {
    cudaStream_t st = (cudaStream_t)stream;
    LG_REQUIRE(v && v->finalized, "vq engine not finalized");
    DeviceGuard guard(v->device);
    LG_REQUIRE(codes && dev_ws && (out_nchw || out_u8) && B > 0 && grid > 0, "lg_vq_decode: bad argument");
    LG_REQUIRE(((uintptr_t)dev_ws & 255) == 0, "workspace must be 256-byte aligned");
    const lg_vq_cfg& c = v->cfg;
    const int Bc = chunk_images(v, B, grid);
    VqWs w = carve_vq(v, (char*)dev_ws, Bc, grid);
    LG_REQUIRE(ws_bytes >= w.bytes, "vq workspace too small: %zu < %zu", ws_bytes, w.bytes);
    const int up_total = 1 << (c.n_mult - 1);
    const size_t out_per_img = (size_t)3 * grid * up_total * grid * up_total;
    for (int b0 = 0; b0 < B; b0 += Bc) {
        const int bc = std::min(Bc, B - b0);
        int H = grid, W = grid;
        lookup_postquant_kernel<<<bc * grid * grid, 256, 0, st>>>(codes + (size_t)b0 * grid * grid, v->codebook, c.codebook_size,
                                                                  c.codebook_embed_dim, v->pq_w, v->pq_b, c.z_channels, w.T);
        LG_LAUNCH_CHECK();
        w.gn_src = nullptr;
        LG_TRY(run_conv(v->conv_in, w.T, bc, H, W, 0, nullptr, w.X, nullptr, st, nullptr, &w));
        LG_TRY(run_res(v->mid0, w, bc, H, W, st));
        LG_TRY(run_attn(v->mid1, w, bc, H, W, st));
        LG_TRY(run_res(v->mid2, w, bc, H, W, st));
        for (size_t li = 0; li < v->levels.size(); ++li) {
            const LevelW& lv = v->levels[li];
            for (size_t j = 0; j < lv.res.size(); ++j) {
                LG_TRY(run_res(lv.res[j], w, bc, H, W, st));
                if (!lv.attn.empty()) LG_TRY(run_attn(lv.attn[j], w, bc, H, W, st));
            }
            if (lv.up) {  // nearest x2 folded into the conv's gather; result -> T, then swap
                LG_TRY(run_conv(lv.upconv, w.X, bc, H, W, 1, nullptr, w.T, nullptr, st, nullptr, &w));
                std::swap(w.X, w.T);
                H *= 2; W *= 2;
            }
        }
        LG_TRY(run_gn(v->norm_out, w.X, w.T, bc, H * W, 1, w.gn, st, &w));
        LG_TRY(run_conv(v->conv_out, w.T, bc, H, W, 0, nullptr, nullptr, out_nchw ? out_nchw + (size_t)b0 * out_per_img : nullptr, st,
                        out_u8 ? out_u8 + (size_t)b0 * out_per_img : nullptr));
    }
    return 0;
}

int lg_vq_decode(lg_vq* v, const int32_t* codes, int B, int grid, void* dev_ws, size_t ws_bytes, float* out_nchw, void* stream) {
    return vq_decode_impl(v, codes, B, grid, dev_ws, ws_bytes, out_nchw, nullptr, stream);
}

int lg_vq_decode_u8(lg_vq* v, const int32_t* codes, int B, int grid, void* dev_ws, size_t ws_bytes, uint8_t* out_nhwc, void* stream) {
    return vq_decode_impl(v, codes, B, grid, dev_ws, ws_bytes, nullptr, out_nhwc, stream);
}

int lg_vq_argmin(lg_vq* v, const float* z_nchw, int B, int grid, int64_t* out_idx, void* stream) {
    cudaStream_t st = (cudaStream_t)stream;
    LG_REQUIRE(v && v->finalized, "vq engine not finalized");
    DeviceGuard guard(v->device);
    LG_REQUIRE(z_nchw && out_idx && B > 0 && grid > 0, "lg_vq_argmin: bad argument");
    const lg_vq_cfg& c = v->cfg;
    const int nz = B * grid * grid, ed = c.codebook_embed_dim;
    const size_t smem = (size_t)kArgminTile * (ed + 1) * sizeof(float);
#define LG_ARGMIN(ED)                                                                                              \
    do {                                                                                                           \
        static DevOnce attr;                                                                                  \
        if (lg_first_on_device(attr)) { LG_CUDA_OK(cudaFuncSetAttribute(argmin_kernel<ED>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)((size_t)kArgminTile * (ED + 1) * 4))); } \
        argmin_kernel<ED><<<cdiv(nz, 128), 128, smem, st>>>(z_nchw, B, grid, v->codebook, v->codebook_sq, c.codebook_size, c.l2_norm, out_idx); \
    } while (0)
    if (ed == 8) LG_ARGMIN(8);
    else if (ed == 4) LG_ARGMIN(4);
    else if (ed == 16) LG_ARGMIN(16);
    else LG_ARGMIN(32);
#undef LG_ARGMIN
    LG_LAUNCH_CHECK();
    return 0;
}

int lg_vq_encode(lg_vq* v, const float* x_nchw, int B, int H, int W, void* dev_ws, size_t ws_bytes, int64_t* out_idx,
                 float* out_quant_nchw, float* out_z_nchw, void* stream) {
    cudaStream_t st = (cudaStream_t)stream;
    LG_REQUIRE(v && v->finalized, "vq engine not finalized");
    DeviceGuard guard(v->device);
    LG_REQUIRE(v->has_encoder, "lg_vq_encode: encoder.* / quant_conv.* weights were not bound");
    LG_REQUIRE(x_nchw && dev_ws && out_idx && B > 0, "lg_vq_encode: bad argument");
    LG_REQUIRE(((uintptr_t)dev_ws & 255) == 0, "workspace must be 256-byte aligned");
    const lg_vq_cfg& c = v->cfg;
    const int down = 1 << (c.n_mult - 1);
    LG_REQUIRE(H == W && H > 0 && H % down == 0 && W % 4 == 0, "lg_vq_encode: image %dx%d must be square and a multiple of %d (and of 4)", H, W, down);
    const int grid = H / down, N = grid * grid, ed = c.codebook_embed_dim;
    const int Bc = chunk_images(v, B, grid);
    VqWs w = carve_vq(v, (char*)dev_ws, Bc, grid);
    LG_REQUIRE(ws_bytes >= w.bytes, "vq workspace too small: %zu < %zu", ws_bytes, w.bytes);
    for (int b0 = 0; b0 < B; b0 += Bc) {
        const int bc = std::min(Bc, B - b0);
        int h = H, wd = W;
        {
            const long long items = (long long)bc * h * (wd / 4) * (c.ch / 8);
            const size_t smem = (size_t)28 * c.ch * sizeof(float);
            prof_begin(PC_VQ_CONV, st);
            conv_in_rgb_kernel<<<(unsigned)std::min<long long>(cdiv(items, 256), 132 * 8), 256, smem, st>>>(x_nchw + (size_t)b0 * 3 * H * W, v->enc_in_w,
                                                                                v->enc_in_b, w.X, bc, h, wd, c.ch);
            prof_end(st);
            LG_LAUNCH_CHECK();
        }
        for (size_t li = 0; li < v->enc_levels.size(); ++li) {
            const LevelW& lv = v->enc_levels[li];
            for (size_t j = 0; j < lv.res.size(); ++j) {
                LG_TRY(run_res(lv.res[j], w, bc, h, wd, st));
                if (!lv.attn.empty()) LG_TRY(run_attn(lv.attn[j], w, bc, h, wd, st));
            }
            if (lv.up) {
                LG_TRY(run_conv(lv.upconv, w.X, bc, h, wd, 2, nullptr, w.T, nullptr, st, nullptr, &w));
                std::swap(w.X, w.T);
                h /= 2; wd /= 2;
            }
        }
        LG_TRY(run_res(v->enc_mid0, w, bc, h, wd, st));
        LG_TRY(run_attn(v->enc_mid1, w, bc, h, wd, st));
        LG_TRY(run_res(v->enc_mid2, w, bc, h, wd, st));
        LG_TRY(run_gn(v->enc_norm_out, w.X, w.T, bc, h * wd, 1, w.gn, st, &w));
        LG_TRY(run_conv(v->enc_conv_out, w.T, bc, h, wd, 0, nullptr, w.U, nullptr, st));
        float* z = out_z_nchw ? out_z_nchw + (size_t)b0 * ed * N : w.Z;
        LG_TRY(run_conv(v->quant_conv, w.U, bc, h, wd, 0, nullptr, nullptr, z, st));
        LG_TRY(lg_vq_argmin(v, z, bc, grid, out_idx + (size_t)b0 * N, stream));
        if (out_quant_nchw) {
            quant_out_kernel<<<cdiv(bc * N, 256), 256, 0, st>>>(z, out_idx + (size_t)b0 * N, v->codebook, bc, N, ed, c.l2_norm,
                                                               out_quant_nchw + (size_t)b0 * ed * N);
            LG_LAUNCH_CHECK();
        }
    }
    return 0;
}

int lg_pixels_to_u8(const float* in_nchw, int B, int C, int H, int W, int out_h, int out_w, uint8_t* out_nhwc, void* stream) {
    cudaStream_t st = (cudaStream_t)stream;
    LG_REQUIRE(in_nchw && out_nhwc && B > 0 && C > 0 && H > 0 && W > 0 && out_h > 0 && out_w > 0, "lg_pixels_to_u8: bad argument");
    const long long n = (long long)B * out_h * out_w;
    const bool vec = C == 3 && out_w % 4 == 0 && (out_w != W || out_h != H || (W % 4 == 0 && ((uintptr_t)in_nchw & 15) == 0)) &&
                     ((uintptr_t)out_nhwc & 3) == 0;
    if (vec) pixels_to_u8_kernel<4><<<(unsigned)cdiv(n / 4, 256), 256, 0, st>>>(in_nchw, B, C, H, W, out_h, out_w, out_nhwc);
    else pixels_to_u8_kernel<1><<<(unsigned)cdiv(n, 256), 256, 0, st>>>(in_nchw, B, C, H, W, out_h, out_w, out_nhwc);
    LG_LAUNCH_CHECK();
    return 0;
}

int lg_test_vq_conv(const void* x, int B, int Hin, int Win, int Cin, const float* w, const float* bias, int Cout, int ksize, int up,
                    const void* residual, void* out_bf, float* out_nchw, uint8_t* out_u8, const float* gn_gamma, const float* gn_beta,
                    int gn_swish, void* gn_out, float* gn_partial, size_t gn_partial_floats, void* dev_scratch, size_t scratch_bytes,
                    int* path, int* gn_splits, void* stream) {
    cudaStream_t st = (cudaStream_t)stream;
    LG_REQUIRE(x && w && bias && dev_scratch && path && gn_splits && B > 0 && Hin > 0 && Win > 0 && Cout > 0,
               "lg_test_vq_conv: bad argument");
    LG_REQUIRE((out_bf != nullptr) + (out_nchw != nullptr) + (out_u8 != nullptr) == 1, "lg_test_vq_conv: exactly one output");
    LG_REQUIRE(ksize == 3 || (ksize == 1 && up == 0), "lg_test_vq_conv: ksize %d with up %d", ksize, up);
    LG_REQUIRE(up >= 0 && up <= 2 && (up != 2 || (Hin % 2 == 0 && Win % 2 == 0)), "lg_test_vq_conv: bad up %d for %dx%d", up, Hin, Win);
    LG_REQUIRE(Cin % 8 == 0, "lg_test_vq_conv: Cin=%d must be a multiple of 8", Cin);
    LG_REQUIRE(((uintptr_t)dev_scratch & 255) == 0, "lg_test_vq_conv: scratch must be 256-byte aligned");
    const bool gn = gn_gamma != nullptr;
    LG_REQUIRE(!gn || (gn_beta && gn_out && out_bf && Cout % 32 == 0 && Cout <= 512 && 256 % (Cout / 8) == 0),
               "lg_test_vq_conv: GroupNorm needs gamma, beta, gn_out, a bf16 output and a supported channel count (%d)", Cout);
    const int Hout = up == 1 ? 2 * Hin : (up == 2 ? Hin / 2 : Hin), Wout = up == 1 ? 2 * Win : (up == 2 ? Win / 2 : Win);
    // scratch: repacked weights, phase weights, GroupNorm partials (64 stand-alone splits or one per 16x16 tile and phase)
    const bool phase = up == 1 && Cin % 64 == 0;
    const size_t wq_bytes = a256((size_t)Cout * Cin * ksize * ksize * sizeof(bf16));
    const size_t wp_bytes = phase ? a256((size_t)16 * Cout * Cin * sizeof(bf16)) : 0;
    const size_t gn_floats = (size_t)B * std::max(64, cdiv(Hin, 16) * cdiv(Win, 16) * 4) * 64;
    const size_t need = wq_bytes + wp_bytes + gn_floats * sizeof(float);
    LG_REQUIRE(scratch_bytes >= need, "lg_test_vq_conv: scratch %zu < %zu", scratch_bytes, need);
    char* s = (char*)dev_scratch;
    ConvW cw;
    cw.w = (bf16*)s; cw.bias = bias; cw.cout = Cout; cw.cin = Cin; cw.k = ksize;
    repack_conv_kernel<<<132 * 4, 256, 0, st>>>(w, cw.w, Cout, Cin, ksize * ksize);
    LG_LAUNCH_CHECK();
    if (phase) {
        cw.w_phase = (bf16*)(s + wq_bytes);
        LG_TRY(conv_tc_make_phase_weights(w, cw.w_phase, Cout, Cin, st));
    }
    VqWs ws{};
    ws.gn = (float*)(s + wq_bytes + wp_bytes);
    ws.gn_floats = gn_floats;
    LG_TRY(run_conv(cw, (const bf16*)x, B, Hin, Win, up, (const bf16*)residual, (bf16*)out_bf, out_nchw, st, out_u8, &ws, path));
    *gn_splits = ws.gn_src == out_bf && out_bf ? ws.gn_splits : 0;
    if (gn_partial && *gn_splits > 0) {
        const size_t n = (size_t)B * *gn_splits * 64;
        LG_REQUIRE(gn_partial_floats >= n, "lg_test_vq_conv: gn_partial %zu < %zu floats", gn_partial_floats, n);
        LG_CUDA_OK(cudaMemcpyAsync(gn_partial, ws.gn, n * sizeof(float), cudaMemcpyDeviceToDevice, st));
    }
    if (gn) {
        const NormW nw{gn_gamma, gn_beta, Cout};
        LG_TRY(run_gn(nw, (const bf16*)out_bf, (bf16*)gn_out, B, Hout * Wout, gn_swish, ws.gn, st, &ws));
    }
    return 0;
}

int lg_test_group_norm(const void* x, int B, int HW, int C, const float* gamma, const float* beta, int swish, void* y,
                       void* dev_scratch, size_t scratch_bytes, void* stream) {
    LG_REQUIRE(x && gamma && beta && y && dev_scratch && B > 0 && HW > 0, "lg_test_group_norm: bad argument");
    LG_REQUIRE(C % 32 == 0 && C <= 512 && 256 % (C / 8) == 0, "lg_test_group_norm: unsupported channel count %d", C);
    const size_t need = (size_t)B * 64 * 64 * sizeof(float);       // gn_stats_kernel: at most 64 splits x 32 groups x (sum, sum sq)
    LG_REQUIRE(scratch_bytes >= need, "lg_test_group_norm: scratch %zu < %zu", scratch_bytes, need);
    const NormW nw{gamma, beta, C};
    return run_gn(nw, (const bf16*)x, (bf16*)y, B, HW, swish, (float*)dev_scratch, (cudaStream_t)stream);
}

}  // extern "C"
