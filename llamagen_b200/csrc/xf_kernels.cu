// Transformer glue kernels: embedding gathers, RMSNorm, the row-wise GEMM epilogues (RoPE + KV-cache
// write, residual + next-norm, SiLU*mul, GELU) and the KV-cached attention kernel.
//
// Reference: autoregressive/models/gpt.py — RMSNorm :137-148, Attention.forward :207-241,
// apply_rotary_emb :420-430, KVCache.update :177-185, FeedForward.forward :166-167, MLP :127-131,
// TransformerBlock.forward :253-257.  Every value the reference materialises as a tensor in the
// model dtype T is rounded to T at the same point here (ElemTraits<T>::round).
#include "kernels.cuh"
#include <algorithm>
#include <type_traits>

namespace {

template <typename T> using TR = ElemTraits<T>;

__device__ __forceinline__ int load_pos(const PosArg& p, int r) { return p.rows ? p.rows[r] : (p.dev ? *p.dev : 0) + p.value; }

__device__ __forceinline__ float sum_partials(const float* __restrict__ p, size_t idx, int ks, size_t slab) {
    float s = p[idx];
    for (int k = 1; k < ks; ++k) s += p[idx + (size_t)k * slab];
    return s;
}

// ---------------------------------------------------------------- embedding gathers
template <typename T>
__global__ void embed_kernel(const T* __restrict__ table, const int32_t* __restrict__ src, int B, int null_idx,
                             int D, T* __restrict__ out) {
    lg_pdl_sync();
    const int r = blockIdx.x;
    const int idx = r < B ? src[r] : (null_idx >= 0 ? null_idx : src[r - B]);
    const T* s = table + (size_t)idx * D;
    T* d = out + (size_t)r * D;
    for (int i = threadIdx.x; i < D; i += blockDim.x) d[i] = s[i];
}

// continuous batching (c2i): per-row choice between the class table (position 0) and the token table
template <typename T>
__global__ void embed_rows_kernel(const T* __restrict__ cls_table, const T* __restrict__ tok_table, const int32_t* __restrict__ src,
                                  const int* __restrict__ pos_rows, int B, int null_idx, int D, T* __restrict__ out) {
    lg_pdl_sync();
    const int r = blockIdx.x, b = r < B ? r : r - B;
    // a class id outside [0, null_idx] (e.g. a stale token left in a free serving slot) reads the null class instead of running past the table
    const int cls = (r < B && (unsigned)src[b] <= (unsigned)null_idx) ? src[b] : null_idx;
    const T* s = pos_rows[r] == 0 ? cls_table + (size_t)cls * D : tok_table + (size_t)src[b] * D;
    T* d = out + (size_t)r * D;
    for (int i = threadIdx.x; i < D; i += blockDim.x) d[i] = s[i];
}

template <typename T>
__global__ void caption_rows_kernel(const T* __restrict__ cond, const T* __restrict__ uncond, size_t ustride, int B, int T_,
                                    int C, T* __restrict__ out) {
    lg_pdl_sync();
    const int row = blockIdx.x, r = row / T_, t = row % T_;
    const T* s = r < B ? cond + ((size_t)r * T_ + t) * C : uncond + (size_t)(r - B) * ustride + (size_t)t * C;
    T* d = out + (size_t)row * C;
    for (int i = threadIdx.x; i < C; i += blockDim.x) d[i] = s[i];
}

template <typename T>
__global__ void gather_last_kernel(const T* __restrict__ in, int T_, int D, T* __restrict__ out) {
    lg_pdl_sync();
    const int r = blockIdx.x;
    const T* s = in + ((size_t)r * T_ + (T_ - 1)) * D;
    T* d = out + (size_t)r * D;
    for (int i = threadIdx.x; i < D; i += blockDim.x) d[i] = s[i];
}

// ---------------------------------------------------------------- RMSNorm (gpt.py:143-148)
template <typename T>
__global__ void __launch_bounds__(256) rmsnorm_kernel(const T* __restrict__ x, const T* __restrict__ w,
                                                      T* __restrict__ xn, int D, float eps) {
    lg_pdl_sync();
    __shared__ float red[33];
    const size_t row = (size_t)blockIdx.x * D;
    float ss = 0.f;
    for (int i = threadIdx.x; i < D; i += blockDim.x) {      // 256 threads: the sample kernel's fused tail reduces in the same order
        const float v = TR<T>::to_f(x[row + i]);
        ss = fmaf(v, v, ss);
    }
    ss = block_sum(ss, red);
    const float r = 1.0f / sqrtf(ss / (float)D + eps);
    for (int i = threadIdx.x; i < D; i += blockDim.x) {
        const float v = TR<T>::round(TR<T>::to_f(x[row + i]) * r);
        xn[row + i] = TR<T>::from_f(v * TR<T>::to_f(w[i]));
    }
}

// ---------------------------------------------------------------- QKV epilogue: RoPE + cache write
__device__ __forceinline__ float4 sum_partials4(const float* __restrict__ p, size_t idx, int ks, size_t slab) {
    float4 s = *reinterpret_cast<const float4*>(p + idx);
    for (int k = 1; k < ks; ++k) {
        const float4 t = *reinterpret_cast<const float4*>(p + idx + (size_t)k * slab);
        s.x += t.x; s.y += t.y; s.z += t.z; s.w += t.w;
    }
    return s;
}
template <typename T> __device__ __forceinline__ void store4(T* p, float a, float b, float c, float d);
template <> __device__ __forceinline__ void store4<float>(float* p, float a, float b, float c, float d) {
    *reinterpret_cast<float4*>(p) = make_float4(a, b, c, d);
}
template <> __device__ __forceinline__ void store4<bf16>(bf16* p, float a, float b, float c, float d) {
    __nv_bfloat162 lo = __floats2bfloat162_rn(a, b), hi = __floats2bfloat162_rn(c, d);
    uint2 u;
    u.x = *reinterpret_cast<uint32_t*>(&lo);
    u.y = *reinterpret_cast<uint32_t*>(&hi);
    *reinterpret_cast<uint2*>(p) = u;
}
template <> __device__ __forceinline__ void store4<f16>(f16* p, float a, float b, float c, float d) {
    uint2 u;
    u.x = ElemTraits<f16>::pack2(a, b);
    u.y = ElemTraits<f16>::pack2(c, d);
    *reinterpret_cast<uint2*>(p) = u;
}
template <typename T> __device__ __forceinline__ void load4(const T* p, float* o) { VecLoad<T, 4>::load(p, o); }
__device__ __forceinline__ void store4_e4m3(e4m3* p, float a, float b, float c, float d) {
    *reinterpret_cast<uint32_t*>(p) = e4m3x2_pack(a, b) | (e4m3x2_pack(c, d) << 16);
}

// One CTA per row, one thread per 4 consecutive output features (two RoPE pairs), all loads up front.
// F8: the K / V rows go to an fp8 cache as e4m3(x * inv), x the model-dtype value the 16-bit cache would hold.
template <typename T, bool F8 = false>
__global__ void __launch_bounds__(1024) qkv_epilogue_kernel(QkvEpiArgs a) {
    lg_pdl_sync();
    const int m = blockIdx.x, r = m / a.Tq, t = m % a.Tq;
    const int p = load_pos(a.pos, r) + t;
    const int D = a.D, hd = a.hd, half = hd >> 1, N = 3 * D;
    const int hdp = a.hdp ? a.hdp : hd;                 // cache row stride
    const size_t slab = (size_t)a.M * N;
    const float* fr = a.freqs + (size_t)p * half * 2;
    T* q = reinterpret_cast<T*>(a.q);
    T* kc = reinterpret_cast<T*>(a.kcache);
    T* vc = reinterpret_cast<T*>(a.vcache);
    for (int n = threadIdx.x * 4; n < N; n += blockDim.x * 4) {
        const float4 sv = sum_partials4(a.partial, (size_t)m * N + n, a.ksplit, slab);
        // the GEMM output is a T tensor in the reference; RoPE then runs in fp32 (gpt.py:423)
        const float x0 = TR<T>::round(sv.x), x1 = TR<T>::round(sv.y), x2 = TR<T>::round(sv.z), x3 = TR<T>::round(sv.w);
        const int sec = n / D, within = n - sec * D, head = within / hd, e = within - head * hd;   // hd % 4 == 0
        if (sec == 2) {
            if constexpr (F8) {
                const float s = a.v_inv;
                store4_e4m3(reinterpret_cast<e4m3*>(a.vcache) + (((size_t)r * a.H + head) * a.maxS + p) * hdp + e, x0 * s, x1 * s, x2 * s, x3 * s);
            } else {
                store4<T>(vc + (((size_t)r * a.H + head) * a.maxS + p) * hdp + e, x0, x1, x2, x3);
            }
        } else {
            const float4 cs = *reinterpret_cast<const float4*>(fr + (e >> 1) * 2);   // (cos, sin) of two pairs
            const float y0 = __fsub_rn(__fmul_rn(x0, cs.x), __fmul_rn(x1, cs.y));
            const float y1 = __fadd_rn(__fmul_rn(x1, cs.x), __fmul_rn(x0, cs.y));
            const float y2 = __fsub_rn(__fmul_rn(x2, cs.z), __fmul_rn(x3, cs.w));
            const float y3 = __fadd_rn(__fmul_rn(x3, cs.z), __fmul_rn(x2, cs.w));
            if constexpr (F8) {
                if (sec == 1) {   // the key is rounded to T after RoPE (as the 16-bit cache stores it), then quantised
                    const float s = a.k_inv;
                    store4_e4m3(reinterpret_cast<e4m3*>(a.kcache) + (((size_t)r * a.H + head) * a.maxS + p) * hdp + e,
                                TR<T>::round(y0) * s, TR<T>::round(y1) * s, TR<T>::round(y2) * s, TR<T>::round(y3) * s);
                    continue;
                }
            }
            T* dst = sec == 0 ? q + (size_t)m * D + within : kc + (((size_t)r * a.H + head) * a.maxS + p) * hdp + e;
            store4<T>(dst, y0, y1, y2, y3);
        }
    }
}

// ---------------------------------------------------------------- residual add (+ next RMSNorm)
// One CTA per row, D/4 threads, everything in registers between the two phases (D <= 4096).
template <typename T>
__global__ void __launch_bounds__(1024) residual_norm_kernel(const float* __restrict__ partial, int ks, int M,
                                                             int D, T* __restrict__ h, const T* __restrict__ nw,
                                                             T* __restrict__ xn, float eps) {
    lg_pdl_sync();
    __shared__ float red[33];
    const int m = blockIdx.x, i = threadIdx.x * 4;
    const size_t slab = (size_t)M * D, row = (size_t)m * D;
    float v[4] = {0.f, 0.f, 0.f, 0.f}, w[4] = {0.f, 0.f, 0.f, 0.f};
    const bool act = i < D;
    if (act) {
        const float4 o = sum_partials4(partial, row + i, ks, slab);
        float hv[4];
        load4<T>(h + row + i, hv);
        if (xn) load4<T>(nw + i, w);
        // h = x + f(x) in dtype T (gpt.py:255-256): the branch output is a T tensor, the sum is rounded again
        v[0] = TR<T>::round(hv[0] + TR<T>::round(o.x));
        v[1] = TR<T>::round(hv[1] + TR<T>::round(o.y));
        v[2] = TR<T>::round(hv[2] + TR<T>::round(o.z));
        v[3] = TR<T>::round(hv[3] + TR<T>::round(o.w));
        store4<T>(h + row + i, v[0], v[1], v[2], v[3]);
    }
    if (xn == nullptr) return;
    float ss = v[0] * v[0] + v[1] * v[1] + v[2] * v[2] + v[3] * v[3];
    ss = block_sum(ss, red);
    const float r = 1.0f / sqrtf(ss / (float)D + eps);
    if (act)
        store4<T>(xn + row + i, TR<T>::round(v[0] * r) * w[0], TR<T>::round(v[1] * r) * w[1],
                  TR<T>::round(v[2] * r) * w[2], TR<T>::round(v[3] * r) * w[3]);
}

// ---------------------------------------------------------------- SwiGLU gate (gpt.py:167)
template <typename T>
__global__ void silu_mul_kernel(const float* __restrict__ partial, int ks, int M, int F, T* __restrict__ out) {
    lg_pdl_sync();
    const size_t total4 = (size_t)M * F / 4, slab = (size_t)M * 2 * F;
    const int f4 = F / 4;
    for (size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x; i < total4; i += (size_t)gridDim.x * blockDim.x) {
        const size_t m = i / f4, j = (i - m * f4) * 4;
        const float4 a4 = sum_partials4(partial, m * 2 * F + j, ks, slab);
        const float4 b4 = sum_partials4(partial, m * 2 * F + F + j, ks, slab);
        const float a[4] = {a4.x, a4.y, a4.z, a4.w}, b[4] = {b4.x, b4.y, b4.z, b4.w};
        float o[4];
#pragma unroll
        for (int k = 0; k < 4; ++k) {
            const float av = TR<T>::round(a[k]), bv = TR<T>::round(b[k]);
            const float sv = TR<T>::round(av / (1.0f + expf(-av)));
            o[k] = sv * bv;
        }
        store4<T>(out + m * F + j, o[0], o[1], o[2], o[3]);
    }
}

__device__ __forceinline__ float gelu_tanh(float v) {   // nn.GELU(approximate='tanh'), gpt.py:122; T5's NewGELUActivation
    const float kBeta = 0.7978845608028654f, kKappa = 0.044715f;
    const float inner = kBeta * (v + kKappa * v * v * v);
    return 0.5f * v * (1.0f + tanhf(inner));
}

// ---------------------------------------------------------------- gated-GELU (T5DenseGatedActDense: gelu_new(wi_0 x) * wi_1 x)
// The rounding points of silu_mul_kernel: each GEMM output is a T tensor, so is the activation, and the product is rounded on store.
template <typename T>
__global__ void gelu_mul_kernel(const float* __restrict__ partial, int ks, int M, int F, T* __restrict__ out) {
    lg_pdl_sync();
    const size_t total4 = (size_t)M * F / 4, slab = (size_t)M * 2 * F;
    const int f4 = F / 4;
    for (size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x; i < total4; i += (size_t)gridDim.x * blockDim.x) {
        const size_t m = i / f4, j = (i - m * f4) * 4;
        const float4 a4 = sum_partials4(partial, m * 2 * F + j, ks, slab);
        const float4 b4 = sum_partials4(partial, m * 2 * F + F + j, ks, slab);
        const float a[4] = {a4.x, a4.y, a4.z, a4.w}, b[4] = {b4.x, b4.y, b4.z, b4.w};
        float o[4];
#pragma unroll
        for (int k = 0; k < 4; ++k) o[k] = TR<T>::round(gelu_tanh(TR<T>::round(a[k]))) * TR<T>::round(b[k]);
        store4<T>(out + m * F + j, o[0], o[1], o[2], o[3]);
    }
}

template <typename T>
__global__ void store_act_kernel(const float* __restrict__ partial, int ks, size_t total, int gelu,
                                 T* __restrict__ out) {
    lg_pdl_sync();
    for (size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (size_t)gridDim.x * blockDim.x) {
        float v = TR<T>::round(sum_partials(partial, i, ks, total));
        if (gelu) v = gelu_tanh(v);
        out[i] = TR<T>::from_f(v);
    }
}

__global__ void reduce_f32_kernel(const float* __restrict__ partial, int ks, size_t total, float* __restrict__ out) {
    lg_pdl_sync();
    for (size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (size_t)gridDim.x * blockDim.x)
        out[i] = sum_partials(partial, i, ks, total);
}

// ---------------------------------------------------------------- KV-cached attention
// One CTA per (query row m = r*Tq + t, head h). A key is owned by a group of LPK lanes, each holding VEC
// contiguous head elements (128-bit loads for hd=64 bf16); every lane group runs an independent online
// softmax over its keys; groups merge by shuffles, warps merge through shared memory.
// Mask (gpt.py:354 + generate.py:154-163): key j visible iff j <= qpos and (j >= Tc or mask[r%B, j] != 0 or j == qpos), mask the
// emb_mask of the row's half (attn_mask_row).
// KV = e4m3 (fp8 cache): K and V are read as their e4m3 codes; a.scale carries the K scale and the output is multiplied by a.v_scale.
template <typename T, int HD, int VEC, int LPK, int HDP = HD, typename KV = T>
__global__ void __launch_bounds__(256) attention_kernel(AttnArgs a) {
    lg_pdl_sync();
    constexpr int KPW = 32 / LPK;  // keys per warp per iteration
    constexpr int UNROLL = 4;
    extern __shared__ float smem[];  // [nwarps][HD + 2]
    const int h = blockIdx.x, m = blockIdx.y;
    const int r = m / a.Tq, t = m - r * a.Tq;
    const int qpos = load_pos(a.pos, r) + t;
    const int nkeys = qpos + 1;
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5, nwarps = blockDim.x >> 5;
    const int g = lane / LPK, li = lane - g * LPK;
    const bool active = li * VEC < HD;
    const int D = a.H * HD;
    constexpr int hdp = HDP;                            // cache row stride (compile-time: the address math sits in the inner loop)

    const T* qp = reinterpret_cast<const T*>(a.q) + (size_t)m * D + (size_t)h * HD;
    const KV* kbase = reinterpret_cast<const KV*>(a.kcache) + ((size_t)r * a.H + h) * (size_t)a.maxS * hdp;
    const KV* vbase = reinterpret_cast<const KV*>(a.vcache) + ((size_t)r * a.H + h) * (size_t)a.maxS * hdp;
    const float* mrow = attn_mask_row(a, r);

    float qv[VEC];
#pragma unroll
    for (int i = 0; i < VEC; ++i) qv[i] = 0.f;
    if (active) VecLoad<T, VEC>::load(qp + li * VEC, qv);
#pragma unroll
    for (int i = 0; i < VEC; ++i) qv[i] *= a.scale;

    float mx = -INFINITY, l = 0.f, acc[VEC];
#pragma unroll
    for (int i = 0; i < VEC; ++i) acc[i] = 0.f;

    const int stride = nwarps * KPW;
    // the trip count must be warp-uniform: the full-mask shuffles below need all 32 lanes
    for (int jb = warp * KPW; jb < nkeys; jb += stride * UNROLL) {
        const int j0 = jb + g;
        float kv[UNROLL][VEC], vv[UNROLL][VEC];
#pragma unroll
        for (int u = 0; u < UNROLL; ++u) {
            const int j = j0 + u * stride;
#pragma unroll
            for (int i = 0; i < VEC; ++i) { kv[u][i] = 0.f; vv[u][i] = 0.f; }
            if (j < nkeys && active) {
                VecLoad<KV, VEC>::load(kbase + (size_t)j * hdp + li * VEC, kv[u]);
                VecLoad<KV, VEC>::load(vbase + (size_t)j * hdp + li * VEC, vv[u]);
            }
        }
#pragma unroll
        for (int u = 0; u < UNROLL; ++u) {
            const int j = j0 + u * stride;
            float s = 0.f;
#pragma unroll
            for (int i = 0; i < VEC; ++i) s = fmaf(qv[i], kv[u][i], s);
#pragma unroll
            for (int o = LPK / 2; o > 0; o >>= 1) s += __shfl_xor_sync(0xffffffffu, s, o);
            bool vis = j < nkeys;
            if (vis && mrow && j < a.Tc && j != qpos) vis = mrow[j] != 0.f;
            if (vis) {
                const float mn = fmaxf(mx, s);
                const float corr = __expf(mx - mn);  // exp(-inf) = 0 on the first visible key
                const float pw = __expf(s - mn);
                l = l * corr + pw;
#pragma unroll
                for (int i = 0; i < VEC; ++i) acc[i] = acc[i] * corr + pw * vv[u][i];
                mx = mn;
            }
        }
    }

    // merge the KPW lane groups of this warp
#pragma unroll
    for (int o = LPK; o < 32; o <<= 1) {
        const float mo = __shfl_xor_sync(0xffffffffu, mx, o);
        const float lo = __shfl_xor_sync(0xffffffffu, l, o);
        const float mn = fmaxf(mx, mo);
        const float ca = mx == -INFINITY ? 0.f : __expf(mx - mn);
        const float cb = mo == -INFINITY ? 0.f : __expf(mo - mn);
        l = l * ca + lo * cb;
#pragma unroll
        for (int i = 0; i < VEC; ++i) {
            const float ao = __shfl_xor_sync(0xffffffffu, acc[i], o);
            acc[i] = acc[i] * ca + ao * cb;
        }
        mx = mn;
    }
    float* wrow = smem + (size_t)warp * (HD + 2);
    if (g == 0 && active) {
#pragma unroll
        for (int i = 0; i < VEC; ++i) wrow[li * VEC + i] = acc[i];
    }
    if (lane == 0) { wrow[HD] = mx; wrow[HD + 1] = l; }
    __syncthreads();
    T* op = reinterpret_cast<T*>(a.out) + (size_t)m * D + (size_t)h * HD;
    for (int e = threadIdx.x; e < HD; e += blockDim.x) {
        float M_ = -INFINITY;
        for (int w = 0; w < nwarps; ++w) M_ = fmaxf(M_, smem[(size_t)w * (HD + 2) + HD]);
        float L = 0.f, O = 0.f;
        for (int w = 0; w < nwarps; ++w) {
            const float mw = smem[(size_t)w * (HD + 2) + HD];
            const float c = mw == -INFINITY ? 0.f : __expf(mw - M_);
            L += smem[(size_t)w * (HD + 2) + HD + 1] * c;
            O += smem[(size_t)w * (HD + 2) + e] * c;
        }
        if constexpr (std::is_same<KV, e4m3>::value) op[e] = TR<T>::from_f(O / L * a.v_scale);
        else op[e] = TR<T>::from_f(O / L);
    }
}

// ---------------------------------------------------------------- teacher-forced scoring (lg_score)
// h[r, t] = t < T ? the condition embedding cond[r, t] ([R * T, D]) : tok_emb[idx[r % B, t - T]]  (gpt.py:342-344, CFG twins share idx)
template <typename T>
__global__ void embed_seq_kernel(const T* __restrict__ cond, const T* __restrict__ table, const int32_t* __restrict__ idx, int B, int T_,
                                 int seq, int D, T* __restrict__ out) {
    lg_pdl_sync();
    const int row = blockIdx.x, r = row / seq, t = row - r * seq;
    const T* s = t < T_ ? cond + ((size_t)r * T_ + t) * D : table + (size_t)idx[(size_t)(r % B) * (seq - T_) + (t - T_)] * D;
    T* d = out + (size_t)row * D;
    for (int i = threadIdx.x; i < D; i += blockDim.x) d[i] = s[i];
}

// out row (b * S + s) * nh + half = in row (b + half * B) * seq + T - 1 + s: the scored positions, CFG twins adjacent
template <typename T>
__global__ void gather_scored_kernel(const T* __restrict__ in, int B, int nh, int seq, int T_, int S, int D, T* __restrict__ out) {
    lg_pdl_sync();
    const int o = blockIdx.x, half = o % nh, p = o / nh, b = p / S, s = p - b * S;
    const T* src = in + ((size_t)(b + half * B) * seq + T_ - 1 + s) * D;
    T* d = out + (size_t)o * D;
    for (int i = threadIdx.x; i < D; i += blockDim.x) d[i] = src[i];
}

constexpr int kScoreThreads = 512;
// One CTA per scored position p (head rows p * nh .. p * nh + nh - 1 of the split-K slabs): the logit the reference materialises
// (rounded to T like round_logits_inplace), CFG-mixed as generate.py:79-82 / sampling.cu mix it when nh == 2, written to logits
// when asked, then nll = logsumexp - logit[target] in fp32 (F.cross_entropy, gpt.py:378).
template <typename T>
__global__ void __launch_bounds__(kScoreThreads) score_head_kernel(const float* __restrict__ partial, int ks, int Mh, int V, int nh,
                                                                   float cfg_scale, const int32_t* __restrict__ targets,
                                                                   float* __restrict__ logits, float* __restrict__ nll) {
    lg_pdl_sync();
    __shared__ float red[33];
    const int p = blockIdx.x;
    const size_t slab = (size_t)Mh * V;
    const float* pc = partial + (size_t)p * nh * V;
    auto logit = [&](int v) {
        const float c = TR<T>::round(sum_partials(pc, v, ks, slab));
        if (nh == 1) return c;
        const float u = TR<T>::round(sum_partials(pc + V, v, ks, slab));
        return __fadd_rn(u, __fmul_rn(__fsub_rn(c, u), cfg_scale));
    };
    float* lrow = logits ? logits + (size_t)p * V : nullptr;
    float m = -INFINITY, sum = 0.f;
    for (int v = threadIdx.x; v < V; v += kScoreThreads) {
        const float x = logit(v);
        if (lrow) lrow[v] = x;
        if (x > m) { sum = sum * expf(m - x) + 1.f; m = x; }
        else if (x != -INFINITY) sum += expf(x - m);
    }
    if (!nll) return;
    // merge the threads' (max, sum) pairs: block max first, then the rescaled sums
    const float M_ = block_max(m, red);
    const float total = block_sum(m == -INFINITY ? 0.f : sum * expf(m - M_), red);
    if (threadIdx.x == 0) {
        const int tg = targets[p];
        nll[p] = (tg >= 0 && tg < V) ? M_ + logf(total) - logit(tg) : __int_as_float(0x7fc00000);
    }
}

__global__ void advance_kernel(int* pos, int* step) {
    lg_pdl_sync();
    if (pos) *pos += 1;
    if (step) *step += 1;
}
__global__ void set_counters_kernel(int* pos, int pv, int* step, int sv) {
    lg_pdl_sync();
    if (pos) *pos = pv;
    if (step) *step = sv;
}

// One CTA column per (layer, K | V, half, head) segment: positions [0, len) of the source row, read once in W-wide words and written
// to every destination row; blockIdx.y strides over the segment
template <typename W>
__global__ void __launch_bounds__(256) copy_slot_kv_kernel(KvCopyArgs a) {
    lg_pdl_sync();
    int seg = blockIdx.x;
    const int head = seg % a.H;
    seg /= a.H;
    const int half = seg % a.nh;
    seg /= a.nh;
    char* base = (seg & 1) ? a.vcache : a.kcache;
    const int layer = seg >> 1;
    const size_t seg_bytes = (size_t)a.max_seq * a.row_bytes, n = (size_t)a.len * a.row_bytes / sizeof(W);
    const size_t row0 = (size_t)layer * a.rows + (size_t)half * a.B;
    const W* src = reinterpret_cast<const W*>(base + ((row0 + a.src) * a.H + head) * seg_bytes);
    for (size_t i = (size_t)blockIdx.y * blockDim.x + threadIdx.x; i < n; i += (size_t)gridDim.y * blockDim.x) {
        const W v = src[i];
        for (int d = 0; d < a.n_dst; ++d)
            reinterpret_cast<W*>(base + ((row0 + a.dst[d]) * a.H + head) * seg_bytes)[i] = v;
    }
}

// f is called with a value of the element type: f(T{}) for T = float, bf16 or f16
template <typename F>
int dispatch_dtype(int dtype, F f) {
    if (dtype == LG_DTYPE_F32) return f(float{});
    if (dtype == LG_DTYPE_BF16) return f(bf16{});
    if (dtype == LG_DTYPE_F16) return f(f16{});
    return lg_fail("unsupported dtype %d", dtype);
}

}  // namespace

int launch_embed(const void* table, const int32_t* src, int B, int R, int null_idx, int D, int dtype, void* out,
                 cudaStream_t st, bool pdl) {
    return dispatch_dtype(
        dtype, [&](auto z) {
            using E = decltype(z);
            (void)lg_launch_pdl(pdl, embed_kernel<E>, dim3(R), dim3(128), 0, st, (const E*)table, src, B, null_idx, D, (E*)out);
            LG_LAUNCH_CHECK();
            return 0;
        });
}

int launch_embed_rows(const void* cls_table, const void* tok_table, const int32_t* src, const int* pos_rows, int B, int R, int null_idx,
                      int D, int dtype, void* out, cudaStream_t st) {
    return dispatch_dtype(
        dtype, [&](auto z) {
            using E = decltype(z);
            (void)lg_launch(embed_rows_kernel<E>, dim3(R), dim3(128), 0, st, (const E*)cls_table, (const E*)tok_table, src, pos_rows, B, null_idx, D, (E*)out);
            LG_LAUNCH_CHECK();
            return 0;
        });
}

int launch_build_caption_rows(const void* cond, const void* uncond, size_t uncond_stride, int B, int R, int T, int C, int dtype, void* out,
                              cudaStream_t st) {
    return dispatch_dtype(
        dtype, [&](auto z) {
            using E = decltype(z);
            (void)lg_launch(caption_rows_kernel<E>, dim3(R * T), dim3(128), 0, st, (const E*)cond, (const E*)uncond, uncond_stride, B, T, C,
                            (E*)out);
            LG_LAUNCH_CHECK();
            return 0;
        });
}

int launch_gather_last(const void* in, int R, int T, int D, int dtype, void* out, cudaStream_t st) {
    return dispatch_dtype(
        dtype, [&](auto z) {
            using E = decltype(z);
            (void)lg_launch(gather_last_kernel<E>, dim3(R), dim3(128), 0, st, (const E*)in, T, D, (E*)out);
            LG_LAUNCH_CHECK();
            return 0;
        });
}

int launch_rmsnorm(const void* x, const void* w, void* xn, int M, int D, float eps, int dtype, cudaStream_t st, bool pdl) {
    return dispatch_dtype(
        dtype, [&](auto z) {
            using E = decltype(z);
            (void)lg_launch_pdl(pdl, rmsnorm_kernel<E>, dim3(M), dim3(256), 0, st, (const E*)x, (const E*)w, (E*)xn, D, eps);
            LG_LAUNCH_CHECK();
            return 0;
        });
}

int launch_qkv_epilogue(const QkvEpiArgs& a, cudaStream_t st) {
    LG_REQUIRE(a.hd % 4 == 0 && a.D % 4 == 0, "head_dim %d / dim %d must be multiples of 4", a.hd, a.D);
    const int threads = std::min(1024, ((3 * a.D / 4 + 31) / 32) * 32);
    if (a.kv_f8) {
        LG_REQUIRE(lg_dtype_is16(a.dtype), "qkv epilogue: an fp8 KV cache needs a bf16 or fp16 model (dtype %d)", a.dtype);
        (void)lg_launch(a.dtype == LG_DTYPE_F16 ? qkv_epilogue_kernel<f16, true> : qkv_epilogue_kernel<bf16, true>, dim3(a.M), dim3(threads), 0,
                        st, a);
        LG_LAUNCH_CHECK();
        return 0;
    }
    return dispatch_dtype(
        a.dtype, [&](auto z) {
            using E = decltype(z);
            (void)lg_launch(qkv_epilogue_kernel<E>, dim3(a.M), dim3(threads), 0, st, a);
            LG_LAUNCH_CHECK();
            return 0;
        });
}

int launch_residual_norm(const float* partial, int ksplit, int M, int D, void* h, const void* norm_w, void* xn,
                         float eps, int dtype, cudaStream_t st) {
    LG_REQUIRE(D % 4 == 0 && D <= 4096, "dim %d must be a multiple of 4 and <= 4096", D);
    const int threads = ((D / 4 + 31) / 32) * 32;
    return dispatch_dtype(
        dtype, [&](auto z) {
            using E = decltype(z);
            (void)lg_launch(residual_norm_kernel<E>, dim3(M), dim3(threads), 0, st, partial, ksplit, M, D, (E*)h, (const E*)norm_w, (E*)xn, eps);
            LG_LAUNCH_CHECK();
            return 0;
        });
}

int launch_silu_mul(const float* partial, int ksplit, int M, int F, void* out, int dtype, cudaStream_t st) {
    LG_REQUIRE(F % 4 == 0, "ffn dim %d must be a multiple of 4", F);
    const int blocks = (int)std::min<long long>(((long long)M * F / 4 + 255) / 256, 132 * 16);
    return dispatch_dtype(
        dtype, [&](auto z) {
            using E = decltype(z);
            (void)lg_launch(silu_mul_kernel<E>, dim3(blocks), dim3(256), 0, st, partial, ksplit, M, F, (E*)out);
            LG_LAUNCH_CHECK();
            return 0;
        });
}

int launch_gelu_mul(const float* partial, int ksplit, int M, int F, void* out, int dtype, cudaStream_t st) {
    LG_REQUIRE(F % 4 == 0, "ffn dim %d must be a multiple of 4", F);
    const int blocks = (int)std::min<long long>(((long long)M * F / 4 + 255) / 256, 132 * 16);
    return dispatch_dtype(
        dtype, [&](auto z) {
            using E = decltype(z);
            (void)lg_launch(gelu_mul_kernel<E>, dim3(blocks), dim3(256), 0, st, partial, ksplit, M, F, (E*)out);
            LG_LAUNCH_CHECK();
            return 0;
        });
}

int launch_store_act(const float* partial, int ksplit, int M, int N, void* out, int gelu, int dtype, cudaStream_t st) {
    const size_t total = (size_t)M * N;
    const int blocks = (int)std::min<size_t>((total + 255) / 256, 132 * 16);
    return dispatch_dtype(
        dtype, [&](auto z) {
            using E = decltype(z);
            (void)lg_launch(store_act_kernel<E>, dim3(blocks), dim3(256), 0, st, partial, ksplit, total, gelu, (E*)out);
            LG_LAUNCH_CHECK();
            return 0;
        });
}

int launch_reduce_f32(const float* partial, int ksplit, int M, int N, float* out, cudaStream_t st) {
    const size_t total = (size_t)M * N;
    const int blocks = (int)std::min<size_t>((total + 255) / 256, 132 * 16);
    (void)lg_launch(reduce_f32_kernel, dim3(blocks), dim3(256), 0, st, partial, ksplit, total, out);
    LG_LAUNCH_CHECK();
    return 0;
}

template <typename T, int HD, int VEC, int LPK, int HDP = HD, typename KV = T>
static int launch_attention_t(const AttnArgs& a, cudaStream_t st) {
    const long long ctas = (long long)a.R * a.Tq * a.H;
    const int nwarps = ctas >= 592 ? 4 : 8;
    const size_t smem = (size_t)nwarps * (HD + 2) * sizeof(float);
    dim3 grid(a.H, a.R * a.Tq);
    (void)lg_launch(attention_kernel<T, HD, VEC, LPK, HDP, KV>, dim3(grid), dim3(nwarps * 32), smem, st, a);
    LG_LAUNCH_CHECK();
    return 0;
}

int launch_attention(const AttnArgs& a, cudaStream_t st, int* path) {
    const AttnPlan p = attn_plan(a);
    if (path) { path[0] = p.kernel; path[1] = p.stages; path[2] = p.fused; }
    LG_REQUIRE(p.kernel >= 0, "%s", p.error);
    if (p.kernel > 0) return launch_attention_tma(a, p, st);
    if (a.kv_f8) {   // fp8 cache of a 16-bit model
        if (a.dtype == LG_DTYPE_BF16) {
            if (a.hd == 64) return launch_attention_t<bf16, 64, 8, 8, 64, e4m3>(a, st);
            if (a.hd == 128) return launch_attention_t<bf16, 128, 8, 16, 128, e4m3>(a, st);
            if (a.hd == 100) return launch_attention_t<bf16, 100, 4, 32, 112, e4m3>(a, st);
        } else if (a.dtype == LG_DTYPE_F16) {
            if (a.hd == 64) return launch_attention_t<f16, 64, 8, 8, 64, e4m3>(a, st);
            if (a.hd == 128) return launch_attention_t<f16, 128, 8, 16, 128, e4m3>(a, st);
            if (a.hd == 100) return launch_attention_t<f16, 100, 4, 32, 112, e4m3>(a, st);
        }
        return lg_fail("attention: no fp8 KV-cache kernel for head_dim %d / dtype %d", a.hd, a.dtype);
    }
    if (a.dtype == LG_DTYPE_BF16) {
        if (a.hd == 64) return launch_attention_t<bf16, 64, 8, 8>(a, st);
        if (a.hd == 128) return launch_attention_t<bf16, 128, 8, 16>(a, st);
        if (a.hd == 100) return launch_attention_t<bf16, 100, 4, 32, 112>(a, st);
    } else if (a.dtype == LG_DTYPE_F16) {
        if (a.hd == 64) return launch_attention_t<f16, 64, 8, 8>(a, st);
        if (a.hd == 128) return launch_attention_t<f16, 128, 8, 16>(a, st);
        if (a.hd == 100) return launch_attention_t<f16, 100, 4, 32, 112>(a, st);
    } else if (a.dtype == LG_DTYPE_F32) {
        if (a.hd == 64) return launch_attention_t<float, 64, 8, 8>(a, st);
        if (a.hd == 128) return launch_attention_t<float, 128, 8, 16>(a, st);
        if (a.hd == 100) return launch_attention_t<float, 100, 4, 32>(a, st);
    }
    return lg_fail("attention: unsupported head_dim %d / dtype %d (supported: 64, 100, 128)", a.hd, a.dtype);
}

int launch_embed_seq(const void* cond_rows, const void* table, const int32_t* idx, int B, int R, int T, int seq, int D, int dtype, void* out,
                     cudaStream_t st) {
    return dispatch_dtype(
        dtype, [&](auto z) {
            using E = decltype(z);
            (void)lg_launch(embed_seq_kernel<E>, dim3(R * seq), dim3(128), 0, st, (const E*)cond_rows, (const E*)table, idx, B, T, seq, D,
                            (E*)out);
            LG_LAUNCH_CHECK();
            return 0;
        });
}

int launch_gather_scored(const void* in, int B, int nh, int seq, int T, int S, int D, int dtype, void* out, cudaStream_t st) {
    return dispatch_dtype(
        dtype, [&](auto z) {
            using E = decltype(z);
            (void)lg_launch(gather_scored_kernel<E>, dim3(B * S * nh), dim3(128), 0, st, (const E*)in, B, nh, seq, T, S, D, (E*)out);
            LG_LAUNCH_CHECK();
            return 0;
        });
}

int launch_score_head(const float* partial, int ksplit, int P, int V, int nh, float cfg_scale, int dtype, const int32_t* targets,
                      float* logits, float* nll, cudaStream_t st) {
    return dispatch_dtype(
        dtype, [&](auto z) {
            using E = decltype(z);
            (void)lg_launch(score_head_kernel<E>, dim3(P), dim3(kScoreThreads), 0, st, partial, ksplit, P * nh, V, nh, cfg_scale, targets,
                            logits, nll);
            LG_LAUNCH_CHECK();
            return 0;
        });
}

int launch_advance(int* pos, int* step, cudaStream_t st) {
    (void)lg_launch(advance_kernel, dim3(1), dim3(1), 0, st, pos, step);
    LG_LAUNCH_CHECK();
    return 0;
}
int launch_set_counters(int* pos, int pos_v, int* step, int step_v, cudaStream_t st) {
    (void)lg_launch(set_counters_kernel, dim3(1), dim3(1), 0, st, pos, pos_v, step, step_v);
    LG_LAUNCH_CHECK();
    return 0;
}

int launch_copy_slot_kv(const KvCopyArgs& a, cudaStream_t st) {
    LG_REQUIRE(a.n_dst >= 0 && a.n_dst <= kKvCopyMaxDst && a.len >= 0 && a.len <= a.max_seq && a.row_bytes > 0,
               "copy_slot_kv: bad shape (n_dst=%d len=%d max_seq=%d)", a.n_dst, a.len, a.max_seq);
    if (a.n_dst == 0 || a.len == 0) return 0;
    const size_t segs = (size_t)a.layers * 2 * a.nh * a.H, words16 = (size_t)a.len * a.row_bytes / 16;
    LG_REQUIRE(segs <= 0x7fffffffu, "copy_slot_kv: %zu segments", segs);
    // 16-byte words when every segment's start and length allow them (hdp-wide rows are 16-byte multiples in every cache the engine
    // stores), else 4-byte or single-byte words
    const size_t seg_bytes = (size_t)a.max_seq * a.row_bytes, len_bytes = (size_t)a.len * a.row_bytes;
    const uintptr_t al = (uintptr_t)a.kcache | (uintptr_t)a.vcache | seg_bytes | len_bytes;
    const dim3 block(256), grid((unsigned)segs, (unsigned)std::max<size_t>(1, std::min<size_t>(8, words16 / (4 * 256))));
    if ((al & 15) == 0) (void)lg_launch(copy_slot_kv_kernel<uint4>, grid, block, 0, st, a);
    else if ((al & 3) == 0) (void)lg_launch(copy_slot_kv_kernel<uint32_t>, grid, block, 0, st, a);
    else (void)lg_launch(copy_slot_kv_kernel<uint8_t>, grid, block, 0, st, a);
    LG_LAUNCH_CHECK();
    return 0;
}
