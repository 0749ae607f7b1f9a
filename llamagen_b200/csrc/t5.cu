// T5 text encoder (transformers T5EncoderModel, as the reference's language/t5.py runs it for Flan-T5 / T5 v1.1): the caption
// features every text-to-image path starts from.
//   layer i: xn = RMSNorm(h) -> QKV GEMM -> self-attention (relative-position bias, key-padding mask, no 1/sqrt(d)) -> O GEMM,
//            h += T(o), xn = RMSNorm(h) -> wi_0 | wi_1 GEMM -> T(gelu_tanh(T(a))) * T(b) -> wo GEMM, h += T(y), next norm
//   output: final_layer_norm(h), fused into the last residual as its "next norm".
// The GEMMs, the residual + RMSNorm and the embedding are the transformer's own kernels; the attention kernels below are T5's.
#include "kernels.cuh"
#include <map>
#include <string>
#include <vector>

namespace {

constexpr int kT5Hd = 64;          // d_kv: the only head size the attention kernels take
constexpr int kT5MaxT = 512;       // longest caption (the K / V of one (caption, head) stay in shared memory)
constexpr int kT5RowChunk = 256;   // rows of every encoder GEMM call (one wgmma row block): plans never depend on B * T
constexpr int kKs = kT5Hd + 8;     // shared-memory row stride of K / V (elements): conflict-free fragment reads

__device__ __forceinline__ int t5_bucket(const int32_t* buckets, int d, int nb) { return min(max(buckets[d], 0), nb - 1); }

// ---------------------------------------------------------------- tensor-core attention (bf16)
// One CTA (4 warps) per (64-query block, head, caption). The caption's whole K and V for the head (T <= 512 rows) are staged in
// shared memory once, with the head's bias row by relative offset and the additive key mask; each warp then runs 16 query rows
// over 64-key blocks: mma.sync q.K^T, fp32 online softmax, P rounded to T for the mma.sync P.V, one division by the row sum at the
// end. A masked key weighs exactly 0 (-inf score); a row with no valid key writes zeros.
template <typename T>
__global__ void __launch_bounds__(128) t5_attn_tc_kernel(const T* __restrict__ q, int ldq, const T* __restrict__ kv,
                                                          int ldkv, const int32_t* __restrict__ mask,
                                                          const int32_t* __restrict__ buckets, const T* __restrict__ bias, int nb,
                                                          int T_, int H, T* __restrict__ out) {
    lg_pdl_sync();
    extern __shared__ __align__(16) unsigned char sraw[];
    const int nkb = (T_ + 63) / 64;   // 64-key blocks
    T* Ks = reinterpret_cast<T*>(sraw);
    T* Vs = Ks + (size_t)nkb * 64 * kKs;
    float* relb = reinterpret_cast<float*>(Vs + (size_t)nkb * 64 * kKs);   // [2T - 1]
    float* kadd = relb + 2 * nkb * 64;                                    // [nkb * 64]
    const int b = blockIdx.z, h = blockIdx.y, tid = threadIdx.x;
    const int I = H * kT5Hd;
    const T* qb = q + (size_t)b * T_ * ldq + h * kT5Hd;
    const T* kb_ = kv + (size_t)b * T_ * ldkv + h * kT5Hd;   // V of the head sits I elements further
    for (int idx = tid; idx < nkb * 64 * 8; idx += blockDim.x) {
        const int j = idx >> 3, c = (idx & 7) * 8;
        uint4 kx = make_uint4(0, 0, 0, 0), vx = make_uint4(0, 0, 0, 0);
        if (j < T_) {
            kx = *reinterpret_cast<const uint4*>(kb_ + (size_t)j * ldkv + c);
            vx = *reinterpret_cast<const uint4*>(kb_ + (size_t)j * ldkv + I + c);
        }
        *reinterpret_cast<uint4*>(Ks + j * kKs + c) = kx;
        *reinterpret_cast<uint4*>(Vs + j * kKs + c) = vx;
    }
    for (int d = tid; d < 2 * T_ - 1; d += blockDim.x) relb[d] = ElemTraits<T>::to_f(bias[t5_bucket(buckets, d, nb) * H + h]);
    for (int j = tid; j < nkb * 64; j += blockDim.x) kadd[j] = (j < T_ && mask[(size_t)b * T_ + j] != 0) ? 0.f : -INFINITY;
    __syncthreads();

    const int warp = tid >> 5, lane = tid & 31, g = lane >> 2, c = lane & 3;
    const int r0 = blockIdx.x * 64 + warp * 16 + g, r1 = r0 + 8;
    uint32_t qa[4][4];
#pragma unroll
    for (int kc = 0; kc < 4; ++kc) {
        const int e = kc * 16 + 2 * c;
        qa[kc][0] = r0 < T_ ? *reinterpret_cast<const uint32_t*>(qb + (size_t)r0 * ldq + e) : 0u;
        qa[kc][1] = r1 < T_ ? *reinterpret_cast<const uint32_t*>(qb + (size_t)r1 * ldq + e) : 0u;
        qa[kc][2] = r0 < T_ ? *reinterpret_cast<const uint32_t*>(qb + (size_t)r0 * ldq + e + 8) : 0u;
        qa[kc][3] = r1 < T_ ? *reinterpret_cast<const uint32_t*>(qb + (size_t)r1 * ldq + e + 8) : 0u;
    }
    float m[2] = {-INFINITY, -INFINITY}, l[2] = {0.f, 0.f};
    float o[8][4];
#pragma unroll
    for (int nd = 0; nd < 8; ++nd) o[nd][0] = o[nd][1] = o[nd][2] = o[nd][3] = 0.f;
    const int dmax = 2 * T_ - 2;
    for (int kb = 0; kb < nkb; ++kb) {
        float s[8][4];
#pragma unroll
        for (int nt = 0; nt < 8; ++nt) {
            s[nt][0] = s[nt][1] = s[nt][2] = s[nt][3] = 0.f;
            const T* kr = Ks + (kb * 64 + nt * 8 + g) * kKs + 2 * c;
#pragma unroll
            for (int kc = 0; kc < 4; ++kc)
                mma_m16n8k16<T>(s[nt], qa[kc][0], qa[kc][1], qa[kc][2], qa[kc][3], *reinterpret_cast<const uint32_t*>(kr + kc * 16),
                                *reinterpret_cast<const uint32_t*>(kr + kc * 16 + 8));
        }
        float mx[2] = {-INFINITY, -INFINITY};
#pragma unroll
        for (int nt = 0; nt < 8; ++nt) {
#pragma unroll
            for (int e = 0; e < 4; ++e) {
                const int j = kb * 64 + nt * 8 + 2 * c + (e & 1), i = (e < 2 ? r0 : r1);
                const int d = min(max(j - i + T_ - 1, 0), dmax);
                s[nt][e] = s[nt][e] + relb[d] + kadd[j];
                mx[e >> 1] = fmaxf(mx[e >> 1], s[nt][e]);
            }
        }
        float alpha[2], ms[2];
#pragma unroll
        for (int r = 0; r < 2; ++r) {
            mx[r] = fmaxf(mx[r], __shfl_xor_sync(0xffffffffu, mx[r], 1));
            mx[r] = fmaxf(mx[r], __shfl_xor_sync(0xffffffffu, mx[r], 2));
            const float mn = fmaxf(m[r], mx[r]);
            ms[r] = mn == -INFINITY ? 0.f : mn;   // every key so far masked: p = 0, nothing to rescale
            alpha[r] = __expf(m[r] - ms[r]);
            m[r] = mn;
            l[r] *= alpha[r];
        }
#pragma unroll
        for (int nd = 0; nd < 8; ++nd) {
            o[nd][0] *= alpha[0]; o[nd][1] *= alpha[0];
            o[nd][2] *= alpha[1]; o[nd][3] *= alpha[1];
        }
        uint32_t pa[8][2];   // P rounded to T, packed in the A-fragment order of the P.V mma
#pragma unroll
        for (int nt = 0; nt < 8; ++nt) {
            const float p0 = ElemTraits<T>::round(__expf(s[nt][0] - ms[0])), p1 = ElemTraits<T>::round(__expf(s[nt][1] - ms[0]));
            const float p2 = ElemTraits<T>::round(__expf(s[nt][2] - ms[1])), p3 = ElemTraits<T>::round(__expf(s[nt][3] - ms[1]));
            l[0] += p0 + p1;
            l[1] += p2 + p3;
            pa[nt][0] = ElemTraits<T>::pack2(p0, p1);
            pa[nt][1] = ElemTraits<T>::pack2(p2, p3);
        }
#pragma unroll
        for (int kk = 0; kk < 4; ++kk) {
            const int key = kb * 64 + kk * 16 + (lane & 7) + ((lane >> 3) & 1) * 8;
#pragma unroll
            for (int nd = 0; nd < 8; nd += 2) {
                const uint32_t addr = (uint32_t)__cvta_generic_to_shared(Vs + key * kKs + nd * 8 + (lane >> 4) * 8);
                uint32_t b0, b1, b2, b3;
                asm volatile("ldmatrix.sync.aligned.m8n8.x4.trans.shared.b16 {%0,%1,%2,%3}, [%4];\n"
                             : "=r"(b0), "=r"(b1), "=r"(b2), "=r"(b3) : "r"(addr));
                mma_m16n8k16<T>(o[nd], pa[2 * kk][0], pa[2 * kk][1], pa[2 * kk + 1][0], pa[2 * kk + 1][1], b0, b1);
                mma_m16n8k16<T>(o[nd + 1], pa[2 * kk][0], pa[2 * kk][1], pa[2 * kk + 1][0], pa[2 * kk + 1][1], b2, b3);
            }
        }
    }
#pragma unroll
    for (int r = 0; r < 2; ++r) {
        l[r] += __shfl_xor_sync(0xffffffffu, l[r], 1);
        l[r] += __shfl_xor_sync(0xffffffffu, l[r], 2);
    }
    const float inv0 = l[0] > 0.f ? 1.f / l[0] : 0.f, inv1 = l[1] > 0.f ? 1.f / l[1] : 0.f;
    T* ob = out + (size_t)b * T_ * I + h * kT5Hd;
#pragma unroll
    for (int nd = 0; nd < 8; ++nd) {
        const int e = nd * 8 + 2 * c;
        if (r0 < T_) *reinterpret_cast<uint32_t*>(ob + (size_t)r0 * I + e) = ElemTraits<T>::pack2(o[nd][0] * inv0, o[nd][1] * inv0);
        if (r1 < T_) *reinterpret_cast<uint32_t*>(ob + (size_t)r1 * I + e) = ElemTraits<T>::pack2(o[nd][2] * inv1, o[nd][3] * inv1);
    }
}

// ---------------------------------------------------------------- CUDA-core attention (fp32 exact mode)
// One CTA of 64 threads per (query row, head, caption): scores in shared memory, block max and sum, thread d accumulates dim d over
// the keys in order. Same semantics as t5_attn_tc_kernel, fp32 throughout.
template <typename T>
__global__ void __launch_bounds__(64) t5_attn_kernel(const T* __restrict__ q, int ldq, const T* __restrict__ kv, int ldkv,
                                                     const int32_t* __restrict__ mask,
                                                     const int32_t* __restrict__ buckets, const T* __restrict__ bias, int nb, int T_,
                                                     int H, T* __restrict__ out) {
    lg_pdl_sync();
    extern __shared__ float sc[];   // [T]
    __shared__ float qs[kT5Hd];
    __shared__ float red[33];
    const int i = blockIdx.x, h = blockIdx.y, b = blockIdx.z, tid = threadIdx.x;
    const int I = H * kT5Hd;
    const T* kb_ = kv + (size_t)b * T_ * ldkv + h * kT5Hd;   // V of the head sits I elements further
    qs[tid] = ElemTraits<T>::to_f(q[((size_t)b * T_ + i) * ldq + h * kT5Hd + tid]);
    __syncthreads();
    float mx = -INFINITY;
    for (int j = tid; j < T_; j += blockDim.x) {
        float s = -INFINITY;
        if (mask[(size_t)b * T_ + j] != 0) {
            const T* kr = kb_ + (size_t)j * ldkv;
            float acc = 0.f;
#pragma unroll 8
            for (int d = 0; d < kT5Hd; ++d) acc = fmaf(qs[d], ElemTraits<T>::to_f(kr[d]), acc);
            s = acc + ElemTraits<T>::to_f(bias[t5_bucket(buckets, j - i + T_ - 1, nb) * H + h]);
        }
        sc[j] = s;
        mx = fmaxf(mx, s);
    }
    mx = block_max(mx, red);
    const float ms = mx == -INFINITY ? 0.f : mx;
    float sum = 0.f;
    for (int j = tid; j < T_; j += blockDim.x) {
        const float p = expf(sc[j] - ms);
        sc[j] = p;
        sum += p;
    }
    sum = block_sum(sum, red);   // its barriers also publish sc
    float acc = 0.f;
    const T* vr = kb_ + I + tid;
    for (int j = 0; j < T_; ++j) acc = fmaf(sc[j], ElemTraits<T>::to_f(vr[(size_t)j * ldkv]), acc);
    out[((size_t)b * T_ + i) * I + h * kT5Hd + tid] = ElemTraits<T>::from_f(sum > 0.f ? acc / sum : 0.f);
}

size_t tc_smem_bytes(int T) {
    const size_t Tp = (size_t)cdiv(T, 64) * 64;
    return 2 * Tp * kKs * sizeof(bf16) + 3 * Tp * sizeof(float);
}

int t5_attention_args(const char* fn, int dtype, int B, int T, int H, int nb) {
    LG_REQUIRE(dtype == LG_DTYPE_BF16 || dtype == LG_DTYPE_F32, "%s: dtype %d (the T5 attention runs bf16 and fp32)", fn, dtype);
    LG_REQUIRE(B >= 1 && B <= 65535 && H >= 1 && H <= 65535, "%s: B=%d and H=%d must lie in [1, 65535]", fn, B, H);
    LG_REQUIRE(T >= 1 && T <= kT5MaxT, "%s: T=%d outside [1, %d]", fn, T, kT5MaxT);
    LG_REQUIRE(nb >= 1, "%s: num_buckets %d < 1", fn, nb);
    return 0;
}

// q: [B * T] rows of ldq elements, head h at column h * 64; kv: [B * T] rows of ldkv elements, K of head h at column h * 64 and its
// V at I + h * 64 (I = H * 64); out [B * T][I]
int launch_t5_attention(int dtype, int B, int T, int H, const void* q, int ldq, const void* kv, int ldkv, const int32_t* mask,
                        const int32_t* buckets, const void* bias, int nb, void* out, cudaStream_t st) {
    if (dtype == LG_DTYPE_BF16) {
        const size_t smem = tc_smem_bytes(T);
        static DevOnce attr;
        if (lg_first_on_device(attr))
            LG_CUDA_OK(cudaFuncSetAttribute(t5_attn_tc_kernel<bf16>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)tc_smem_bytes(kT5MaxT)));
        (void)lg_launch(t5_attn_tc_kernel<bf16>, dim3(cdiv(T, 64), H, B), dim3(128), smem, st, (const bf16*)q, ldq, (const bf16*)kv,
                        ldkv, mask, buckets, (const bf16*)bias, nb, T, H, (bf16*)out);
    } else {
        (void)lg_launch(t5_attn_kernel<float>, dim3(T, H, B), dim3(64), (size_t)T * sizeof(float), st, (const float*)q, ldq,
                        (const float*)kv, ldkv, mask, buckets, (const float*)bias, nb, T, H, (float*)out);
    }
    LG_LAUNCH_CHECK();
    return 0;
}

size_t t5_align(size_t v) { return (v + 255) / 256 * 256; }

struct T5Tensor {
    const void* p = nullptr;
    int64_t shape[4] = {0, 0, 0, 0};
    int ndim = 0;
    int dtype = 0;
};

// Every weight is the caller's tensor, borrowed: the encoder holds no copy, so an in-place write to a parameter is seen by the
// next call. q is one GEMM; k | v are the two segments of another (no concatenated copy of q | k | v exists).
struct T5Layer {
    const void *ln0, *ln1, *wq, *wk, *wv, *wo, *wi0, *wi1, *wff;
};

// The encoder's GEMMs: {N, K, n_split} of q, k | v, o, wi_0 | wi_1, wo
constexpr int kT5Gemms = 5;
struct T5Gemms {
    int n[kT5Gemms], k[kT5Gemms], split[kT5Gemms];
};

}  // namespace

struct lg_t5 {
    lg_t5_cfg cfg;
    int device = 0;
    size_t esz = 2;
    std::map<std::string, T5Tensor> w;
    std::vector<T5Layer> layers;
    const void* embed = nullptr;
    const void* relbias = nullptr;
    const void* final_norm = nullptr;
    bool finalized = false;
    T5Gemms gemms() const {
        const int D = cfg.d_model, I = cfg.n_head * kT5Hd, F = cfg.d_ff;
        return {{I, 2 * I, D, 2 * F, D}, {D, D, I, D, F}, {0, I, 0, F, 0}};
    }
};

namespace {

struct T5Ws {
    void *h, *xn, *q, *kv, *attn, *ff;
    float* slab;
    size_t bytes;
};

// Workspace views for B captions of T tokens (rows padded to whole GEMM chunks); base may be null to measure
int t5_carve(const lg_t5* t, int B, int T, char* base, T5Ws* v) {
    const lg_t5_cfg& c = t->cfg;
    const size_t Mp = (size_t)cdiv((long long)B * T, kT5RowChunk) * kT5RowChunk;
    const int D = c.d_model, I = c.n_head * kT5Hd, F = c.d_ff;
    const T5Gemms g = t->gemms();
    size_t slab = 0;
    for (int i = 0; i < kT5Gemms; ++i) {
        const size_t f = gemm_partial_floats(kT5RowChunk, g.n[i], g.k[i], g.split[i], c.dtype);
        LG_REQUIRE(f > 0, "lg_t5: GEMM [%d x %d] has no kernel: %s", g.n[i], g.k[i],
                   gemm_plan(kT5RowChunk, g.n[i], g.k[i], g.split[i], c.dtype).error);
        slab = std::max(slab, f);
    }
    size_t off = 0;
    auto take = [&](size_t bytes) { char* p = base ? base + off : nullptr; off += t5_align(bytes); return (void*)p; };
    v->h = take(Mp * D * t->esz);
    v->xn = take(Mp * D * t->esz);
    v->q = take(Mp * I * t->esz);
    v->kv = take(Mp * 2 * I * t->esz);
    v->attn = take(Mp * I * t->esz);
    v->ff = take(Mp * F * t->esz);
    v->slab = (float*)take(slab * sizeof(float));
    v->bytes = off;
    return 0;
}

int t5_need(lg_t5* t, const std::string& name, std::initializer_list<int64_t> shape, const void** out) {
    auto it = t->w.find(name);
    LG_REQUIRE(it != t->w.end(), "lg_t5_finalize: missing weight '%s'", name.c_str());
    const T5Tensor& x = it->second;
    LG_REQUIRE(x.dtype == t->cfg.dtype, "lg_t5_finalize: weight '%s' has dtype %d, expected %d", name.c_str(), x.dtype, t->cfg.dtype);
    LG_REQUIRE(x.ndim == (int)shape.size(), "lg_t5_finalize: weight '%s' has %d dims, expected %d", name.c_str(), x.ndim, (int)shape.size());
    int i = 0;
    for (int64_t s : shape) {
        LG_REQUIRE(x.shape[i] == s, "lg_t5_finalize: weight '%s' dim %d is %lld, expected %lld", name.c_str(), i, (long long)x.shape[i],
                   (long long)s);
        ++i;
    }
    LG_REQUIRE(((uintptr_t)x.p & 15) == 0, "lg_t5_finalize: weight '%s' is not 16-byte aligned", name.c_str());
    *out = x.p;
    return 0;
}

}  // namespace

extern "C" {

int lg_t5_create(const lg_t5_cfg* cfg, int device, lg_t5** out) {
    LG_REQUIRE(cfg && out, "lg_t5_create: null argument");
    LG_REQUIRE(cfg->dtype != LG_DTYPE_F16,
               "lg_t5_create: fp16 is not supported: T5 activations overflow fp16 (transformers only runs it with inf clamps and an fp32 wo)");
    LG_REQUIRE(cfg->dtype == LG_DTYPE_BF16 || cfg->dtype == LG_DTYPE_F32, "lg_t5_create: unsupported dtype %d (fp32 and bf16 only)", cfg->dtype);
    LG_REQUIRE(cfg->d_kv == kT5Hd, "lg_t5_create: d_kv %d is not supported (64 only)", cfg->d_kv);
    LG_REQUIRE(cfg->gated_gelu == 1, "lg_t5_create: only the gated-gelu feed-forward is supported");
    LG_REQUIRE(cfg->n_layer > 0 && cfg->n_head > 0 && cfg->vocab_size > 0 && cfg->num_buckets > 0, "lg_t5_create: bad model dims");
    LG_REQUIRE(cfg->d_model > 0 && cfg->d_model % 128 == 0 && cfg->d_model <= 4096,
               "lg_t5_create: d_model %d must be a positive multiple of 128, at most 4096", cfg->d_model);
    LG_REQUIRE(cfg->d_ff > 0 && cfg->d_ff % 128 == 0, "lg_t5_create: d_ff %d must be a positive multiple of 128", cfg->d_ff);
    LG_REQUIRE(cfg->n_head * kT5Hd % 128 == 0, "lg_t5_create: n_head * d_kv = %d must be a multiple of 128", cfg->n_head * kT5Hd);
    lg_t5* t = new lg_t5();
    t->cfg = *cfg;
    t->device = device;
    t->esz = (size_t)lg_dtype_info(cfg->dtype).esz;
    *out = t;
    return 0;
}

void lg_t5_destroy(lg_t5* t) {
    if (!t) return;
    delete t;
}

int lg_t5_bind_weight(lg_t5* t, const char* name, const void* dev_ptr, const int64_t* shape, int ndim, int dtype) {
    LG_REQUIRE(t && name && dev_ptr && shape && ndim >= 1 && ndim <= 4, "lg_t5_bind_weight: bad argument");
    T5Tensor x;
    x.p = dev_ptr;
    x.ndim = ndim;
    x.dtype = dtype;
    for (int i = 0; i < ndim; ++i) x.shape[i] = shape[i];
    t->w[name] = x;
    t->finalized = false;
    return 0;
}

int lg_t5_finalize(lg_t5* t) {
    LG_REQUIRE(t, "lg_t5_finalize: null encoder");
    const lg_t5_cfg& c = t->cfg;
    const int64_t D = c.d_model, I = c.n_head * kT5Hd, F = c.d_ff;
    t->finalized = false;
    LG_TRY(t5_need(t, "shared.weight", {c.vocab_size, D}, &t->embed));
    LG_TRY(t5_need(t, "encoder.block.0.layer.0.SelfAttention.relative_attention_bias.weight", {c.num_buckets, c.n_head}, &t->relbias));
    LG_TRY(t5_need(t, "encoder.final_layer_norm.weight", {D}, &t->final_norm));
    std::vector<T5Layer> layers(c.n_layer);
    for (int i = 0; i < c.n_layer; ++i) {
        const std::string p = "encoder.block." + std::to_string(i) + ".layer.";
        T5Layer& l = layers[i];
        LG_TRY(t5_need(t, p + "0.SelfAttention.q.weight", {I, D}, &l.wq));
        LG_TRY(t5_need(t, p + "0.SelfAttention.k.weight", {I, D}, &l.wk));
        LG_TRY(t5_need(t, p + "0.SelfAttention.v.weight", {I, D}, &l.wv));
        LG_TRY(t5_need(t, p + "0.SelfAttention.o.weight", {D, I}, &l.wo));
        LG_TRY(t5_need(t, p + "0.layer_norm.weight", {D}, &l.ln0));
        LG_TRY(t5_need(t, p + "1.layer_norm.weight", {D}, &l.ln1));
        LG_TRY(t5_need(t, p + "1.DenseReluDense.wi_0.weight", {F, D}, &l.wi0));
        LG_TRY(t5_need(t, p + "1.DenseReluDense.wi_1.weight", {F, D}, &l.wi1));
        LG_TRY(t5_need(t, p + "1.DenseReluDense.wo.weight", {D, F}, &l.wff));
    }
    t->layers = layers;
    t->finalized = true;
    return 0;
}

int lg_t5_workspace_bytes(lg_t5* t, int B, int T, size_t* bytes) {
    LG_REQUIRE(t && bytes, "lg_t5_workspace_bytes: null argument");
    LG_REQUIRE(B >= 1 && T >= 1 && T <= kT5MaxT, "lg_t5_workspace_bytes: B=%d must be >= 1 and T=%d in [1, %d]", B, T, kT5MaxT);
    T5Ws v;
    LG_TRY(t5_carve(t, B, T, nullptr, &v));
    *bytes = v.bytes;
    return 0;
}

int lg_t5_encode(lg_t5* t, const int32_t* ids, const int32_t* mask, const int32_t* buckets, int B, int T, void* ws, size_t ws_bytes,
                 void* out, void* stream) {
    LG_REQUIRE(t, "lg_t5_encode: null encoder");
    LG_REQUIRE(t->finalized, "lg_t5_encode: call lg_t5_finalize first");
    LG_REQUIRE(ids && mask && buckets && ws && out, "lg_t5_encode: null argument");
    const lg_t5_cfg& c = t->cfg;
    LG_TRY(t5_attention_args("lg_t5_encode", c.dtype, B, T, c.n_head, c.num_buckets));
    LG_REQUIRE(((uintptr_t)ws & 255) == 0, "lg_t5_encode: workspace is not 256-byte aligned");
    T5Ws v;
    LG_TRY(t5_carve(t, B, T, (char*)ws, &v));
    LG_REQUIRE(ws_bytes >= v.bytes, "lg_t5_encode: workspace %zu < %zu bytes", ws_bytes, v.bytes);
    DeviceGuard guard(t->device);
    cudaStream_t st = (cudaStream_t)stream;
    const int M = B * T, Mp = cdiv(M, kT5RowChunk) * kT5RowChunk, nchunk = Mp / kT5RowChunk, C = kT5RowChunk;
    const int D = c.d_model, I = c.n_head * kT5Hd, F = c.d_ff, dt = c.dtype;
    const size_t es = t->esz;
    const T5Gemms g = t->gemms();
    char *h = (char*)v.h, *xn = (char*)v.xn, *q = (char*)v.q, *kv = (char*)v.kv, *attn = (char*)v.attn, *ff = (char*)v.ff;
    // rows past B * T are padding of the last GEMM chunk: zeroed so they stay finite, never read by the attention
    if (Mp > M) {
        LG_CUDA_OK(cudaMemsetAsync(h + (size_t)M * D * es, 0, (size_t)(Mp - M) * D * es, st));
        LG_CUDA_OK(cudaMemsetAsync(attn + (size_t)M * I * es, 0, (size_t)(Mp - M) * I * es, st));
    }
    LG_TRY(launch_embed(t->embed, ids, M, M, -1, D, dt, h, st));   // T5 does not scale its embeddings
    LG_TRY(launch_rmsnorm(h, t->layers[0].ln0, xn, Mp, D, c.eps, dt, st));
    for (int li = 0; li < c.n_layer; ++li) {
        const T5Layer& l = t->layers[li];
        const void* next_norm = li + 1 < c.n_layer ? t->layers[li + 1].ln0 : t->final_norm;
        GemmPlan p;
        for (int k = 0; k < nchunk; ++k) {
            const size_t r = (size_t)k * C;
            LG_TRY(gemm_partial(xn + r * D * es, D, GemmWeight(l.wq), GemmWeight(), 0, C, g.n[0], g.k[0], dt, v.slab, &p, st));
            LG_TRY(launch_store_act(v.slab, p.ksplit, C, I, q + r * I * es, 0, dt, st));
            LG_TRY(gemm_partial(xn + r * D * es, D, GemmWeight(l.wk), GemmWeight(l.wv), I, C, g.n[1], g.k[1], dt, v.slab, &p, st));
            LG_TRY(launch_store_act(v.slab, p.ksplit, C, 2 * I, kv + r * 2 * I * es, 0, dt, st));
        }
        LG_TRY(launch_t5_attention(dt, B, T, c.n_head, q, I, kv, 2 * I, mask, buckets, t->relbias, c.num_buckets, attn, st));
        for (int k = 0; k < nchunk; ++k) {
            const size_t r = (size_t)k * C;
            LG_TRY(gemm_partial(attn + r * I * es, I, GemmWeight(l.wo), GemmWeight(), 0, C, g.n[2], g.k[2], dt, v.slab, &p, st));
            LG_TRY(launch_residual_norm(v.slab, p.ksplit, C, D, h + r * D * es, l.ln1, xn + r * D * es, c.eps, dt, st));
            LG_TRY(gemm_partial(xn + r * D * es, D, GemmWeight(l.wi0), GemmWeight(l.wi1), F, C, g.n[3], g.k[3], dt, v.slab, &p, st));
            LG_TRY(launch_gelu_mul(v.slab, p.ksplit, C, F, ff + r * F * es, dt, st));
            LG_TRY(gemm_partial(ff + r * F * es, F, GemmWeight(l.wff), GemmWeight(), 0, C, g.n[4], g.k[4], dt, v.slab, &p, st));
            LG_TRY(launch_residual_norm(v.slab, p.ksplit, C, D, h + r * D * es, next_norm, xn + r * D * es, c.eps, dt, st));
        }
    }
    LG_CUDA_OK(cudaMemcpyAsync(out, xn, (size_t)M * D * es, cudaMemcpyDeviceToDevice, st));
    return 0;
}

int lg_test_t5_attention(int dtype, int B, int T, int H, const void* qkv, const int32_t* mask, const int32_t* buckets, const void* bias,
                         int num_buckets, void* out, int* path, void* stream) {
    LG_TRY(t5_attention_args("lg_test_t5_attention", dtype, B, T, H, num_buckets));
    LG_REQUIRE(qkv && mask && buckets && bias && out, "lg_test_t5_attention: null argument");
    LG_REQUIRE(((uintptr_t)qkv & 15) == 0 && ((uintptr_t)out & 15) == 0, "lg_test_t5_attention: qkv / out not 16-byte aligned");
    if (path) *path = dtype == LG_DTYPE_BF16 ? 1 : 0;
    const int I = H * kT5Hd, es = dtype == LG_DTYPE_BF16 ? 2 : 4;
    return launch_t5_attention(dtype, B, T, H, qkv, 3 * I, (const char*)qkv + (size_t)I * es, 3 * I, mask, buckets, bias, num_buckets, out,
                               (cudaStream_t)stream);
}

}  // extern "C"
