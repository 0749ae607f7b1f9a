// Fused CFG-mix + temperature + top-k + top-p + softmax + (argmax | multinomial) — one CTA per image.
//
// Reference semantics (autoregressive/models/generate.py):
//   :95-97   logits = uncond + (cond - uncond) * cfg_scale           (fp32, three separate roundings)
//   :58      logits / max(temperature, 1e-5)
//   :33-36   top-k: remove logits < (k-th largest value)  -> ties with the k-th value are KEPT
//   :38-53   top-p: sort desc, softmax, cumsum; token j is kept iff the cumulative probability of the
//            tokens ranked before it is <= top_p (so the first token crossing the threshold is kept)
//   :61      softmax;  :63 multinomial(1)  or  :65 topk(k=1)
// The whole row (V floats) is staged once in shared memory; k-th value / nucleus threshold are found
// with 4x8-bit radix selects over an order-preserving integer key (no sort), reductions are warp shuffles.
#include "kernels.cuh"

namespace {

constexpr int kSampleThreads = 1024;
constexpr int kNB = 2048;            // linear buckets of the fast top-k select

__device__ __forceinline__ uint32_t fkey(float x) {
    uint32_t u = __float_as_uint(x);
    return (u & 0x80000000u) ? ~u : (u | 0x80000000u);
}
__device__ __forceinline__ float fkey_inv(uint32_t k) {
    uint32_t u = (k & 0x80000000u) ? (k & 0x7fffffffu) : ~k;
    return __uint_as_float(u);
}
__device__ __forceinline__ uint64_t splitmix64(uint64_t x) {
    x += 0x9E3779B97F4A7C15ull;
    x = (x ^ (x >> 30)) * 0xBF58476D1CE4E5B9ull;
    x = (x ^ (x >> 27)) * 0x94D049BB133111EBull;
    return x ^ (x >> 31);
}

// E: the 16-bit type of the rounding (a.round_dtype != LG_DTYPE_F32) and of the fused tail's rows
template <typename E>
__global__ void __launch_bounds__(kSampleThreads) sample_kernel(SampleArgs a) {
    using TR = ElemTraits<E>;
    lg_pdl_sync();
    extern __shared__ float sh[];  // V floats: the working logits row, later exp() values
    __shared__ float red[33];
    __shared__ uint32_t hist[256];
    __shared__ float mhist[256];
    __shared__ uint32_t s_prefix, s_remaining;
    __shared__ float s_acc;
    __shared__ int s_pick;
    __shared__ float s_wtot[32];

    const int b = blockIdx.x, tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
    const int V = a.V, B = a.B;
    const uint64_t step = a.step_rows ? (uint64_t)a.step_rows[b] : (a.step_dev ? (uint64_t)(*a.step_dev) : a.step);

    bool mix = a.mix_cfg != 0;
    // generate.py:113-114 — decode iteration i = step-1; once i > cfg_interval the mix is dropped.
    if (mix && a.cfg_interval > -1 && step >= 1 && (long long)(step - 1) > (long long)a.cfg_interval) mix = false;

    const float* lc = a.logits + (size_t)b * V;
    const float* lu = a.logits + (size_t)(B + b) * V;
    const float tdiv = fmaxf(a.temperature, 1e-5f);
    const int dbgB = a.dbg_batch > 0 ? a.dbg_batch : B;
    float* dbg = a.dbg_logits ? a.dbg_logits + ((size_t)step * dbgB + a.row_offset + b) * V : nullptr;

    auto mix1 = [&](float c, float u) -> float {
        if (a.round_dtype) c = TR::round(c);
        if (!mix) return c;
        if (a.round_dtype) u = TR::round(u);
        return __fadd_rn(u, __fmul_rn(__fsub_rn(c, u), a.cfg_scale));
    };
    if ((V & 3) == 0) {
        // 128-bit loads, several requests of a thread in flight before the first use (the scalar loop was
        // latency-bound: 16 dependent L2 round trips per thread)
        const float4* lc4 = reinterpret_cast<const float4*>(lc);
        const float4* lu4 = reinterpret_cast<const float4*>(lu);
        const int V4 = V >> 2;
#pragma unroll 4
        for (int v4 = tid; v4 < V4; v4 += kSampleThreads) {
            const float4 c = lc4[v4];
            float4 u = c;
            if (mix) u = lu4[v4];
            float4 x;
            x.x = mix1(c.x, u.x); x.y = mix1(c.y, u.y); x.z = mix1(c.z, u.z); x.w = mix1(c.w, u.w);
            if (dbg) reinterpret_cast<float4*>(dbg)[v4] = x;
            x.x = __fdiv_rn(x.x, tdiv); x.y = __fdiv_rn(x.y, tdiv); x.z = __fdiv_rn(x.z, tdiv); x.w = __fdiv_rn(x.w, tdiv);
            reinterpret_cast<float4*>(sh)[v4] = x;
        }
    } else {
        for (int v = tid; v < V; v += kSampleThreads) {
            const float x = mix1(lc[v], mix ? lu[v] : 0.f);
            if (dbg) dbg[v] = x;
            sh[v] = __fdiv_rn(x, tdiv);
        }
    }
    __syncthreads();

    // ---------------- top-k: value of the k-th largest, ties kept (generate.py:33-36) -----------------------------
    // Fast path: ONE histogram over 2048 linear buckets of [min, max] (logits are roughly Gaussian, so the fullest bucket holds a
    // few dozen of the 16384 values and the shared-memory atomics barely collide), a block-wide suffix scan to find the bucket
    // holding the k-th largest, then an exact rank count among that bucket's few members. The bucket map is monotone in x, so
    // the selected VALUE is exact. The 4-pass 8-bit radix select below stays as the fallback for degenerate rows (its first
    // pass hashes sign+exponent: ~6 live buckets -> 16384 colliding atomics, measured 26.5 us per row).
    if (a.top_k > 0) {
        const int k = min(max(a.top_k, 1), V);
        if (k < V) {
            __shared__ uint32_t hist2[kNB];
            __shared__ float cand[kSampleThreads];
            __shared__ uint32_t s_warp_tot[32];
            __shared__ uint32_t s_cnt, s_bsel, s_rank;
            __shared__ float s_thr;
            __shared__ int s_ok;
            float lmn = INFINITY, lmx = -INFINITY;
            for (int v = tid; v < V; v += kSampleThreads) { const float x = sh[v]; lmn = fminf(lmn, x); lmx = fmaxf(lmx, x); }
            const float mx = block_max(lmx, red);
            const float mn = -block_max(-lmn, red);
            bool fast = mx > mn && mn > -INFINITY && mx < INFINITY;      // NaNs fail the comparisons too
            float thr = mn;
            if (fast) {
                const float scale = (float)kNB / (mx - mn);
                auto bucket = [&](float x) -> uint32_t { return min((uint32_t)(kNB - 1), (uint32_t)((x - mn) * scale)); };
                for (int i = tid; i < kNB; i += kSampleThreads) hist2[i] = 0;
                if (tid == 0) { s_cnt = 0; s_ok = 0; }
                __syncthreads();
                for (int v = tid; v < V; v += kSampleThreads) atomicAdd(&hist2[bucket(sh[v])], 1u);
                __syncthreads();
                // thread t owns buckets 2t (lower values) and 2t+1; suffix sums over the threads above it
                static_assert(kNB == 2 * kSampleThreads, "two buckets per thread");
                const uint32_t h0 = hist2[2 * tid], h1 = hist2[2 * tid + 1], own = h0 + h1;
                uint32_t suf = own;                                        // inclusive suffix within the warp
#pragma unroll
                for (int o = 1; o < 32; o <<= 1) {
                    const uint32_t tv = __shfl_down_sync(0xffffffffu, suf, o);
                    if (lane + o < 32) suf += tv;
                }
                if (lane == 0) s_warp_tot[warp] = suf;
                __syncthreads();
                uint32_t above_w = 0;
                for (int w = warp + 1; w < kSampleThreads / 32; ++w) above_w += s_warp_tot[w];
                const uint32_t above = above_w + suf - own;                // members of all buckets above 2t+1
                const uint32_t kk = (uint32_t)k;
                if (above < kk && kk <= above + h1) { s_bsel = 2 * tid + 1; s_rank = kk - above; }
                else if (above + h1 < kk && kk <= above + own) { s_bsel = 2 * tid; s_rank = kk - above - h1; }
                __syncthreads();
                const uint32_t bsel = s_bsel, rank = s_rank;
                for (int v = tid; v < V; v += kSampleThreads) {
                    const float x = sh[v];
                    if (bucket(x) == bsel) {
                        const uint32_t i = atomicAdd(&s_cnt, 1u);
                        if (i < (uint32_t)kSampleThreads) cand[i] = x;
                    }
                }
                __syncthreads();
                const uint32_t n = s_cnt;
                if (n <= (uint32_t)kSampleThreads) {
                    if (tid < (int)n) {
                        const float x = cand[tid];
                        uint32_t gt = 0, ge = 0;
                        for (uint32_t j = 0; j < n; ++j) { const float y = cand[j]; gt += y > x; ge += y >= x; }
                        if (gt < rank && rank <= ge) { s_thr = x; s_ok = 1; }   // every tie of the k-th value writes the same number
                    }
                    __syncthreads();
                    fast = s_ok != 0;
                    thr = s_thr;
                } else {
                    fast = false;
                }
            }
            if (!fast) {
                uint32_t prefix = 0, remaining = (uint32_t)k;
                for (int pass = 0; pass < 4; ++pass) {
                    const int shift = 24 - 8 * pass;
                    if (tid < 256) hist[tid] = 0;
                    __syncthreads();
                    for (int v = tid; v < V; v += kSampleThreads) {
                        const uint32_t key = fkey(sh[v]);
                        if (pass == 0 || (key >> (shift + 8)) == prefix) atomicAdd(&hist[(key >> shift) & 255u], 1u);
                    }
                    __syncthreads();
                    if (warp == 0) {
                        uint32_t c[8], lsum = 0;
#pragma unroll
                        for (int j = 0; j < 8; ++j) { c[j] = hist[255 - 8 * lane - j]; lsum += c[j]; }
                        uint32_t incl = lsum;
#pragma unroll
                        for (int o = 1; o < 32; o <<= 1) {
                            uint32_t tv = __shfl_up_sync(0xffffffffu, incl, o);
                            if (lane >= o) incl += tv;
                        }
                        uint32_t cum = incl - lsum;
#pragma unroll
                        for (int j = 0; j < 8; ++j) {
                            if (cum < remaining && cum + c[j] >= remaining) {
                                s_prefix = (prefix << 8) | (uint32_t)(255 - 8 * lane - j);
                                s_remaining = remaining - cum;
                            }
                            cum += c[j];
                        }
                    }
                    __syncthreads();
                    prefix = s_prefix;
                    remaining = s_remaining;
                }
                thr = fkey_inv(prefix);
            }
            for (int v = tid; v < V; v += kSampleThreads)
                if (sh[v] < thr) sh[v] = -INFINITY;
            __syncthreads();
        }
    }

    // ---------------- top-p (nucleus) ---------------------------------------------------------------
    if (a.top_p < 1.0f) {
        float lm = -INFINITY;
        for (int v = tid; v < V; v += kSampleThreads) lm = fmaxf(lm, sh[v]);
        const float m = block_max(lm, red);
        float ls = 0.f;
        for (int v = tid; v < V; v += kSampleThreads) ls += expf(sh[v] - m);
        const float Z = block_sum(ls, red);

        uint32_t prefix = 0;
        float acc = 0.f;  // probability mass of values strictly above the current prefix range
        for (int pass = 0; pass < 4; ++pass) {
            const int shift = 24 - 8 * pass;
            if (tid < 256) { hist[tid] = 0; mhist[tid] = 0.f; }
            __syncthreads();
            for (int v = tid; v < V; v += kSampleThreads) {
                const float x = sh[v];
                if (x == -INFINITY) continue;
                const uint32_t key = fkey(x);
                if (pass == 0 || (key >> (shift + 8)) == prefix) {
                    const uint32_t bk = (key >> shift) & 255u;
                    atomicAdd(&hist[bk], 1u);
                    atomicAdd(&mhist[bk], expf(x - m) / Z);
                }
            }
            __syncthreads();
            if (warp == 0) {
                float ms[8], lsum = 0.f;
                uint32_t c[8];
#pragma unroll
                for (int j = 0; j < 8; ++j) {
                    c[j] = hist[255 - 8 * lane - j];
                    ms[j] = mhist[255 - 8 * lane - j];
                    lsum += ms[j];
                }
                float incl = lsum;
#pragma unroll
                for (int o = 1; o < 32; o <<= 1) {
                    float t = __shfl_up_sync(0xffffffffu, incl, o);
                    if (lane >= o) incl += t;
                }
                float G = acc + (incl - lsum);
                int cand = -1, first_nonempty = -1;
                float candG = 0.f, firstG = 0.f;
#pragma unroll
                for (int j = 0; j < 8; ++j) {
                    if (c[j] > 0) {
                        if (first_nonempty < 0) { first_nonempty = 255 - 8 * lane - j; firstG = G; }
                        if (G <= a.top_p) { cand = 255 - 8 * lane - j; candG = G; }
                    }
                    G += ms[j];
                }
                // lowest qualifying bucket lives in the highest lane that has one
                unsigned has = __ballot_sync(0xffffffffu, cand >= 0);
                int src;
                if (has) {
                    src = 31 - __clz(has);
                } else {  // degenerate top_p < 0: keep only the maximum
                    unsigned ne = __ballot_sync(0xffffffffu, first_nonempty >= 0);
                    src = __ffs(ne) - 1;
                    cand = first_nonempty;
                    candG = firstG;
                }
                const int bsel = __shfl_sync(0xffffffffu, cand, src);
                const float gsel = __shfl_sync(0xffffffffu, candG, src);
                if (lane == 0) { s_prefix = (prefix << 8) | (uint32_t)bsel; s_acc = gsel; }
            }
            __syncthreads();
            prefix = s_prefix;
            acc = s_acc;
        }
        const float vstar = fkey_inv(prefix);
        // ties at v*: the j-th tie (ascending index) is kept iff acc + j*p* <= top_p
        const float pstar = expf(vstar - m) / Z;
        int lt = 0;
        for (int v = tid; v < V; v += kSampleThreads) {
            const float x = sh[v];
            if (x < vstar) sh[v] = -INFINITY;
            else if (x == vstar) ++lt;
        }
        const int nties = (int)(block_sum((float)lt, red) + 0.5f);
        if (nties > 1) {
            int nkeep = 1;
            while (nkeep < nties && acc + (float)nkeep * pstar <= a.top_p) ++nkeep;
            if (nkeep < nties && tid == 0) {
                int seen = 0;
                for (int v = 0; v < V; ++v)
                    if (sh[v] == vstar) { if (seen >= nkeep) sh[v] = -INFINITY; ++seen; }
            }
        }
        __syncthreads();
    }

    // ---------------- final softmax -------------------------------------------------------------------
    float lm = -INFINITY;
    for (int v = tid; v < V; v += kSampleThreads) lm = fmaxf(lm, sh[v]);
    const float m = block_max(lm, red);
    float ls = 0.f;
    for (int v = tid; v < V; v += kSampleThreads) {
        const float e = expf(sh[v] - m);
        sh[v] = e;
        ls += e;
    }
    const float Z = block_sum(ls, red);
    if (a.out_probs) {
        float* op = a.out_probs + (size_t)b * V;
        for (int v = tid; v < V; v += kSampleThreads) op[v] = sh[v] / Z;
    }

    if (tid == 0) s_pick = -1;
    __syncthreads();

    if (a.greedy) {
        // torch.topk(probs, 1): arg-max of the probabilities; lowest index wins ties.
        float bv = -1.f;
        int bi = 0x7fffffff;
        for (int v = tid; v < V; v += kSampleThreads) {
            const float p = sh[v] / Z;
            if (p > bv) { bv = p; bi = v; }
        }
#pragma unroll
        for (int o = 16; o > 0; o >>= 1) {
            const float ov = __shfl_xor_sync(0xffffffffu, bv, o);
            const int oi = __shfl_xor_sync(0xffffffffu, bi, o);
            if (ov > bv || (ov == bv && oi < bi)) { bv = ov; bi = oi; }
        }
        __shared__ float s_bv[32];
        __shared__ int s_bi[32];
        if (lane == 0) { s_bv[warp] = bv; s_bi[warp] = bi; }
        __syncthreads();
        if (warp == 0) {
            bv = s_bv[lane];
            bi = s_bi[lane];
#pragma unroll
            for (int o = 16; o > 0; o >>= 1) {
                const float ov = __shfl_xor_sync(0xffffffffu, bv, o);
                const int oi = __shfl_xor_sync(0xffffffffu, bi, o);
                if (ov > bv || (ov == bv && oi < bi)) { bv = ov; bi = oi; }
            }
            if (lane == 0) s_pick = bi;
        }
        __syncthreads();
    } else {
        // inverse-CDF draw over the unnormalised weights e_v (same distribution as torch.multinomial).
        const int seg = (V + kSampleThreads - 1) / kSampleThreads;
        const int v0 = min(tid * seg, V), v1 = min(v0 + seg, V);
        float local = 0.f;
        for (int v = v0; v < v1; ++v) local += sh[v];
        float incl = local;
#pragma unroll
        for (int o = 1; o < 32; o <<= 1) {
            float t = __shfl_up_sync(0xffffffffu, incl, o);
            if (lane >= o) incl += t;
        }
        if (lane == 31) s_wtot[warp] = incl;
        __syncthreads();
        if (warp == 0) {
            float w = s_wtot[lane], wi = w;
#pragma unroll
            for (int o = 1; o < 32; o <<= 1) {
                float t = __shfl_up_sync(0xffffffffu, wi, o);
                if (lane >= o) wi += t;
            }
            s_wtot[lane] = wi - w;  // exclusive warp offsets
            if (lane == 31) red[32] = wi;
        }
        __syncthreads();
        const float total = red[32];
        const float excl = s_wtot[warp] + (incl - local);
        // per-request streams (seed_rows): every image draws exactly what a batch-of-one generate() with its seed would draw
        const uint64_t seed = a.seed_rows ? a.seed_rows[b] : a.seed;
        const uint64_t rrow = a.seed_rows ? 1ull : (uint64_t)(b + 1 + a.row_offset);
        const uint64_t r = splitmix64(splitmix64(seed ^ (0xA0761D6478BD642Full * (step + 1))) ^ (0xE7037ED1A0B428DBull * rrow));
        const float u = (float)(r >> 40) * (1.0f / 16777216.0f);
        const float target = u * total;
        if (local > 0.f && target >= excl && target < excl + local) {
            float c = excl;
            int pick = -1, lastnz = -1;
            for (int v = v0; v < v1; ++v) {
                const float e = sh[v];
                if (e > 0.f) lastnz = v;
                c += e;
                if (c > target && e > 0.f) { pick = v; break; }
            }
            s_pick = pick >= 0 ? pick : lastnz;
        }
        __syncthreads();
        if (s_pick < 0) {  // rounding pushed the target past the total: take the last non-zero weight
            int cand = -1;
            for (int v = tid; v < V; v += kSampleThreads)
                if (sh[v] > 0.f) cand = max(cand, v);
            cand = (int)block_max((float)cand, red);
            if (tid == 0) s_pick = cand;
            __syncthreads();
        }
    }

    __shared__ int s_next;
    if (tid == 0) {
        const int pick = s_pick;
        if (a.out_idx) a.out_idx[b] = pick;
        if (a.out_seq) a.out_seq[(size_t)b * a.seq_stride + step] = pick;
        const int nxt = a.teacher ? a.teacher[(size_t)b * a.seq_stride + step] : pick;
        if (a.next_tokens) a.next_tokens[b] = nxt;
        s_next = nxt;
    }
    // ---------------- fused tail: next step's input rows (embedding lookup + layer-0 RMSNorm) and the counter advance ----------
    if (a.emb_table) {
        __syncthreads();
        const int D = a.emb_D;
        const E* src = reinterpret_cast<const E*>(a.emb_table) + (size_t)s_next * D;
        // thread -> 2 consecutive elements per pass (D even); the same token feeds the cond and the uncond row (generate.py:91)
        for (int i = tid * 2; i < D; i += kSampleThreads * 2) {
            const uint32_t w = *reinterpret_cast<const uint32_t*>(src + i);
            for (int row = b; row < a.emb_rows; row += B)
                *reinterpret_cast<uint32_t*>(reinterpret_cast<E*>(a.emb_h) + (size_t)row * D + i) = w;
        }
        if (a.emb_xn) {
            // sum of squares in rmsnorm_kernel's order (256 threads striding the row, then the same block reduction tree: the other
            // 24 warps contribute zeros) so that this path and the stand-alone kernels produce bit-identical activations
            float ss = 0.f;
            if (tid < 256)
                for (int i = tid; i < D; i += 256) {
                    const float v = TR::to_f(src[i]);
                    ss = fmaf(v, v, ss);
                }
            const float tot = block_sum(ss, red);
            const float rinv = 1.0f / sqrtf(tot / (float)D + a.emb_eps);
            const E* nw = reinterpret_cast<const E*>(a.emb_norm_w);
            for (int i = tid * 2; i < D; i += kSampleThreads * 2) {
                const uint32_t w = *reinterpret_cast<const uint32_t*>(src + i);
                const uint32_t g2 = *reinterpret_cast<const uint32_t*>(nw + i);
                // norm(x.float()).type_as(x) * weight: two E roundings, as rmsnorm_kernel / residual_norm_kernel
                const float lo = TR::round(TR::lo(w) * rinv) * TR::lo(g2);
                const float hi = TR::round(TR::hi(w) * rinv) * TR::hi(g2);
                const uint32_t pk = TR::pack2(lo, hi);
                for (int row = b; row < a.emb_rows; row += B)
                    *reinterpret_cast<uint32_t*>(reinterpret_cast<E*>(a.emb_xn) + (size_t)row * D + i) = pk;
            }
        }
    }
    if (a.adv_ticket) {
        // every CTA has read `step` (and the logits) by now; the last one to arrive moves the loop counters for the next step
        __syncthreads();
        if (tid == 0) {
            __threadfence();
            const unsigned int old = atomicAdd(a.adv_ticket, 1u);
            if (old == gridDim.x - 1) {
                if (a.adv_pos) *a.adv_pos += 1;
                if (a.adv_step) *a.adv_step += 1;
                *a.adv_ticket = 0u;
            }
        }
    }
}

}  // namespace

int launch_sample(const SampleArgs& a, cudaStream_t st) {
    LG_REQUIRE(a.B > 0 && a.V > 0, "lg_sample: bad shape B=%d V=%d", a.B, a.V);
    const size_t smem = (size_t)a.V * sizeof(float);
    LG_REQUIRE(smem <= 200 * 1024, "lg_sample: vocab %d too large for the shared-memory row stage", a.V);
    LG_REQUIRE(a.round_dtype == LG_DTYPE_F32 || lg_dtype_is16(a.round_dtype), "lg_sample: unsupported round dtype %d", a.round_dtype);
    LG_REQUIRE(!a.emb_table || a.round_dtype != LG_DTYPE_F32, "lg_sample: the fused tail needs a 16-bit round dtype");
    const bool half = a.round_dtype == LG_DTYPE_F16;
    auto kern = half ? sample_kernel<f16> : sample_kernel<bf16>;
    static DevOnce attr_set[2];
    if (lg_first_on_device(attr_set[half])) {
        LG_CUDA_OK(cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, 200 * 1024));
    }
    (void)lg_launch(kern, dim3(a.B), dim3(kSampleThreads), smem, st, a);
    LG_LAUNCH_CHECK();
    return 0;
}
