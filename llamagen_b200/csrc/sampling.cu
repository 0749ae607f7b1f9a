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

// Highest thread index of the block (kThreads threads) for which pred holds, -1 if none; returned to every thread. s_w: 32 ints.
template <int kThreads>
__device__ __forceinline__ int block_last_true(bool pred, int* s_w) {
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    const unsigned bal = __ballot_sync(0xffffffffu, pred);
    if (lane == 0) s_w[warp] = bal ? warp * 32 + 31 - __clz((int)bal) : -1;
    __syncthreads();
    int r = lane < kThreads / 32 ? s_w[lane] : -1;
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) r = max(r, __shfl_xor_sync(0xffffffffu, r, o));
    __syncthreads();   // s_w may be reused
    return r;
}

// Dynamic shared memory of the logprob instantiation: the working row, a copy of the processed row x (the exp pass overwrites the
// working row), then every warp's top-N candidates (x, id)
__host__ __device__ constexpr size_t sample_lp_smem(int V) {
    return (size_t)2 * V * sizeof(float) + (size_t)(kSampleThreads / 32) * kMaxTopLogprobs * (sizeof(float) + sizeof(int));
}

// Logprob, rank and top-N of the row x (xs, V floats) the draw took `pick` from; m, Z: the final softmax's max and sum, so that
// exp(logprob) is the kernel's own probability. o: the output element (out_seq's index). Called by every thread after the draw.
__device__ void sample_logprobs(const SampleArgs& a, const float* xs, float* cx, int* ci, int V, float m, float Z, int pick, size_t o) {
    __shared__ int s_gt[kSampleThreads / 32];
    const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
    const float lz = logf(Z);
    const float xp = pick >= 0 ? xs[pick] : __int_as_float(0x7fffffff);
    if (a.rank_out) {   // on x, not on exp values: distinct logits can round to the same expf
        int gt = 0;
        for (int v = tid; v < V; v += kSampleThreads) gt += xs[v] > xp;
        gt = __reduce_add_sync(0xffffffffu, gt);
        if (lane == 0) s_gt[warp] = gt;
        __syncthreads();
        if (tid == 0) {
            int r = 1;
            for (int w = 0; w < kSampleThreads / 32; ++w) r += s_gt[w];
            a.rank_out[o] = r;
        }
    }
    if (tid == 0 && a.lp_out) a.lp_out[o] = (xp - m) - lz;
    const int N = a.top_n;
    if (N <= 0) return;
    // order (x desc, id asc); (bx, bi) is better than (x, i); kept tokens only, so an empty slot (-inf, INT_MAX) loses to all of them
    auto better = [](float x, int i, float bx, int bi) { return x > bx || (x == bx && i < bi); };
    auto warp_best = [&](float& bx, int& bi) {
#pragma unroll
        for (int s = 16; s > 0; s >>= 1) {
            const float ox = __shfl_xor_sync(0xffffffffu, bx, s);
            const int oi = __shfl_xor_sync(0xffffffffu, bi, s);
            if (better(ox, oi, bx, bi)) { bx = ox; bi = oi; }
        }
    };
    // each lane: the best kept entry of its columns (v = 32 warp + lane + 1024 j) strictly after (lx, li) in the order
    auto scan = [&](float lx, int li, float& bx, int& bi) {
        bx = -INFINITY; bi = 0x7fffffff;
        for (int v = warp * 32 + lane; v < V; v += kSampleThreads) {
            const float x = xs[v];
            if ((x < lx || (x == lx && v > li)) && x > -INFINITY && better(x, v, bx, bi)) { bx = x; bi = v; }
        }
    };
    // each warp: its N best in N shuffle-argmax rounds; the other lanes' candidates stay valid, so only the winner's lane rescans
    float bx, wx;
    int bi, wi;
    scan(INFINITY, -1, bx, bi);
    for (int r = 0; r < N; ++r) {
        wx = bx; wi = bi;
        warp_best(wx, wi);
        if (lane == 0) { cx[warp * N + r] = wx; ci[warp * N + r] = wi; }
        if (wi != 0x7fffffff && bi == wi) scan(wx, wi, bx, bi);
    }
    __syncthreads();
    // warp 0 merges the 32 sorted lists: lane w holds the head of warp w's, and the winner's lane advances
    static_assert(kSampleThreads / 32 == 32, "one list per lane");
    if (warp == 0) {
        int p = 0;
        for (int r = 0; r < N; ++r) {
            const float x = p < N ? cx[lane * N + p] : -INFINITY;
            const int id = p < N ? ci[lane * N + p] : 0x7fffffff;
            wx = x; wi = id;
            warp_best(wx, wi);
            if (lane == 0) {
                const bool kept = wi != 0x7fffffff;
                a.top_ids[o * N + r] = kept ? wi : -1;
                a.top_lp[o * N + r] = kept ? (wx - m) - lz : -INFINITY;
            }
            if (wi != 0x7fffffff && id == wi) ++p;
        }
    }
}

// E: the 16-bit type of the rounding (a.round_dtype != LG_DTYPE_F32) and of the fused tail's rows. kLogprobs: also write the token
// log-probabilities (SampleArgs.lp_out ...); the draw is the same. kGroups: composable guidance (SampleArgs.mix_groups = K): CTA b is
// image b, which reads its K conditional rows b K .. b K + K - 1 and the unconditional row B + b K and mixes them with its weights;
// every per-image output, input and key is image b's, and its token feeds all 2K of its rows
template <typename E, bool kLogprobs, bool kGroups>
__global__ void __launch_bounds__(kSampleThreads) sample_kernel(SampleArgs a) {
    using TR = ElemTraits<E>;
    lg_pdl_sync();
    extern __shared__ float sh[];  // V floats: the working logits row, later exp() values
    __shared__ float red[33];
    __shared__ uint32_t hist[256];
    __shared__ float mhist[256];
    __shared__ uint32_t s_prefix, s_remaining;
    __shared__ float s_acc;
    __shared__ int s_pick, s_end;
    __shared__ float s_wtot[32];
    __shared__ int s_own[32];

    const int b = blockIdx.x, tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
    const int V = a.V, B = a.B;
    const uint64_t step = a.step_rows ? (uint64_t)a.step_rows[b] : (a.step_dev ? (uint64_t)(*a.step_dev) : a.step);

    // a gather table (mix_rows, grouped instantiation only): row b's role, -2 condition row, -1 plain row, u >= 0 lead row mixing
    // unconditional row u; without one, -1
    const int32_t* mr = kGroups && a.mix_rows ? a.mix_rows + (size_t)b * (1 + kMaxMixGroups) : nullptr;
    const int role = mr ? mr[0] : -1;
    if (role == -2) return;   // a condition row: its logits are read by its lead's CTA

    const float cfg_scale = a.cfg_rows ? a.cfg_rows[b] : a.cfg_scale;
    const int cfg_interval = a.interval_rows ? a.interval_rows[b] : a.cfg_interval;
    // a row with its own scale mixes only above 1 (generate.py:79 `if cfg_scale > 1.0`; a NaN scale does not mix either): it then
    // reads only its conditional row. A lead row always mixes (its weights are the scales)
    bool mix = a.mix_cfg != 0 && (role >= 0 || !a.cfg_rows || cfg_scale > 1.0f);
    // generate.py:113-114 — decode iteration i = step-1; once i > cfg_interval the mix is dropped.
    if (mix && cfg_interval > -1 && step >= 1 && (long long)(step - 1) > (long long)cfg_interval) mix = false;

    const int G = kGroups ? (mr ? 1 : a.mix_groups) : 1;   // rows per image and half (a gather table: one row per CTA)
    const float* lc = a.logits + (size_t)b * G * V;
    const float* lu = a.logits + (size_t)(role >= 0 ? role : B + b * G) * V;
    // the image's filters: its entry of the row arrays, or the call's scalars
    const int fr = b / a.param_div;
    const float tdiv = fmaxf(a.temp_rows ? a.temp_rows[fr] : a.temperature, 1e-5f);
    const int top_k = a.topk_rows ? a.topk_rows[fr] : a.top_k;
    const float top_p = a.topp_rows ? a.topp_rows[fr] : a.top_p;
    const bool greedy = a.greedy_rows ? a.greedy_rows[fr] != 0 : a.greedy != 0;
    const int dbgB = a.dbg_batch > 0 ? a.dbg_batch : B;
    float* dbg = a.dbg_logits ? a.dbg_logits + ((size_t)step * dbgB + a.row_offset + b) * V : nullptr;

    auto mix1 = [&](float c, float u) -> float {
        if (a.round_dtype) c = TR::round(c);
        if (!mix) return c;
        if (a.round_dtype) u = TR::round(u);
        return __fadd_rn(u, __fmul_rn(__fsub_rn(c, u), cfg_scale));
    };
    if constexpr (kGroups) {
        // x = u + d, d = w_1 (c_1 - u) + ... + w_K (c_K - u) accumulated left to right, every row rounded first; K = 1 is mix1 with
        // cfg_scale = w_1 exactly. Without the mix (cfg_interval passed, K = 1 only) x = c_1, as mix1. With a gather table a lead row
        // mixes the nc conditional rows its entries name, and a plain row is one condition at its own scale (mix1 bit for bit)
        int nc = G;
        if (role >= 0) {
            nc = 0;
            while (nc < kMaxMixGroups && mr[1 + nc] >= 0) ++nc;
        }
        int crow[kMaxMixGroups];   // the conditional rows
        float w[kMaxMixGroups];
#pragma unroll
        for (int i = 0; i < kMaxMixGroups; ++i) {
            crow[i] = role >= 0 ? mr[1 + min(i, nc - 1)] : b * G + i;
            w[i] = i >= nc ? 0.f : !mr ? a.mix_weights[(size_t)b * G + i] : role >= 0 ? a.mix_weights[(size_t)b * kMaxMixGroups + i] : cfg_scale;
        }
        auto crow_ptr = [&](int i) { return a.logits + (size_t)crow[i] * V; };
        auto rd = [&](float x) -> float { return a.round_dtype ? TR::round(x) : x; };
        auto mixg = [&](int v) -> float {
            const float c1 = rd(crow_ptr(0)[v]);
            if (!mix) return c1;
            const float u = rd(lu[v]);
            float d = __fmul_rn(__fsub_rn(c1, u), w[0]);
#pragma unroll
            for (int i = 1; i < kMaxMixGroups; ++i)
                if (i < nc) d = __fadd_rn(d, __fmul_rn(__fsub_rn(rd(crow_ptr(i)[v]), u), w[i]));
            return __fadd_rn(u, d);
        };
        if (sample_vec_loads(a)) {   // 128-bit loads, as below
            const float4* lu4 = reinterpret_cast<const float4*>(lu);
            const int V4 = V >> 2;
            auto row4 = [&](int i) { return reinterpret_cast<const float4*>(crow_ptr(i)); };
            auto rd4 = [&](float4 x) -> float4 { return make_float4(rd(x.x), rd(x.y), rd(x.z), rd(x.w)); };
            auto term = [](float c, float u, float wi) { return __fmul_rn(__fsub_rn(c, u), wi); };
#pragma unroll 2
            for (int v4 = tid; v4 < V4; v4 += kSampleThreads) {
                float4 x = rd4(row4(0)[v4]);
                if (mix) {
                    const float4 u = rd4(lu4[v4]);
                    float4 d = make_float4(term(x.x, u.x, w[0]), term(x.y, u.y, w[0]), term(x.z, u.z, w[0]), term(x.w, u.w, w[0]));
#pragma unroll
                    for (int i = 1; i < kMaxMixGroups; ++i)
                        if (i < nc) {
                            const float4 c = rd4(row4(i)[v4]);
                            d.x = __fadd_rn(d.x, term(c.x, u.x, w[i])); d.y = __fadd_rn(d.y, term(c.y, u.y, w[i]));
                            d.z = __fadd_rn(d.z, term(c.z, u.z, w[i])); d.w = __fadd_rn(d.w, term(c.w, u.w, w[i]));
                        }
                    x = make_float4(__fadd_rn(u.x, d.x), __fadd_rn(u.y, d.y), __fadd_rn(u.z, d.z), __fadd_rn(u.w, d.w));
                }
                x.x = __fdiv_rn(x.x, tdiv); x.y = __fdiv_rn(x.y, tdiv); x.z = __fdiv_rn(x.z, tdiv); x.w = __fdiv_rn(x.w, tdiv);
                reinterpret_cast<float4*>(sh)[v4] = x;
            }
        } else {
            for (int v = tid; v < V; v += kSampleThreads) sh[v] = __fdiv_rn(mixg(v), tdiv);
        }
    } else if (sample_vec_loads(a)) {
        // 128-bit loads, several requests of a thread in flight before the first use (the scalar loop was
        // latency-bound: 16 dependent L2 round trips per thread); a caller's row that is not 16-byte aligned takes the scalar loop
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
    int path_topk = 0, path_trim = 0;   // dbg_path (lg_test_sample); the draw ending is s_end
    if (top_k > 0) {
        const int k = min(max(top_k, 1), V);
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
            path_topk = fast ? 1 : 2;
            for (int v = tid; v < V; v += kSampleThreads)
                if (sh[v] < thr) sh[v] = -INFINITY;
            __syncthreads();
        }
    }

    // ---------------- top-p (nucleus) ---------------------------------------------------------------
    if (top_p < 1.0f) {
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
                        if (G <= top_p) { cand = 255 - 8 * lane - j; candG = G; }
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
            while (nkeep < nties && acc + (float)nkeep * pstar <= top_p) ++nkeep;
            path_trim = nkeep < nties;
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
        if constexpr (kLogprobs) sh[V + v] = sh[v];
        const float e = expf(sh[v] - m);
        sh[v] = e;
        ls += e;
    }
    const float Z = block_sum(ls, red);
    if (a.out_probs) {
        float* op = a.out_probs + (size_t)b * V;
        for (int v = tid; v < V; v += kSampleThreads) op[v] = sh[v] / Z;
    }

    if (tid == 0) { s_pick = -1; s_end = 0; }
    __syncthreads();

    if (greedy) {
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
        // per-request streams (seed_rows): every image draws exactly what a batch-of-one generate() with its seed would draw, or, with
        // img_rows, what image img_rows[b] of a generate() with its seed draws
        const uint64_t seed = a.seed_rows ? a.seed_rows[b] : a.seed;
        const uint64_t rrow = a.seed_rows ? (a.img_rows ? (uint64_t)a.img_rows[b] + 1 : 1ull)
                                          : (uint64_t)(b + 1 + (kGroups ? a.row_offset / G : a.row_offset));
        const uint64_t r = splitmix64(splitmix64(seed ^ (0xA0761D6478BD642Full * (step + 1))) ^ (0xE7037ED1A0B428DBull * rrow));
        const float u = (float)(r >> 40) * (1.0f / 16777216.0f);
        const float target = u * total;
        // The fp32 prefixes are not additive across threads (excl + local, rounded, need not equal the next thread's excl), so
        // "excl <= target < excl + local" would give some targets to no thread and others to two. The target belongs instead to the
        // highest thread with a non-zero segment that starts at or below it: exactly one owner for every target.
        const int owner = block_last_true<kSampleThreads>(local > 0.f && excl <= target, s_own);
        const int lastseg = a.dbg_path ? block_last_true<kSampleThreads>(local > 0.f, s_own) : -1;
        if (tid == owner) {
            float c = excl;
            int pick = -1, lastnz = -1;
            for (int v = v0; v < v1; ++v) {
                const float e = sh[v];
                if (e > 0.f) lastnz = v;
                c += e;
                if (c > target && e > 0.f) { pick = v; break; }
            }
            // a walk that never passes the target (the target past the total, or in the rounding gap before the next segment's
            // start) takes the segment's last non-zero weight
            s_pick = pick >= 0 ? pick : lastnz;
            s_end = pick < 0 && tid == lastseg ? 2 : 1;
        }
        __syncthreads();
        if (s_pick < 0) {  // no owner (no segment with a positive sum: a NaN row): the last non-zero weight, if any
            if (tid == 0) s_end = 2;
            int cand = -1;
            for (int v = tid; v < V; v += kSampleThreads)
                if (sh[v] > 0.f) cand = max(cand, v);
            cand = (int)block_max((float)cand, red);
            if (tid == 0) s_pick = cand;
            __syncthreads();
        }
    }

    if constexpr (kLogprobs) {
        float* cx = sh + 2 * (size_t)V;
        sample_logprobs(a, sh + V, cx, reinterpret_cast<int*>(cx + (kSampleThreads / 32) * kMaxTopLogprobs), V, m, Z, s_pick,
                        (size_t)b * a.seq_stride + step);
    }
    __shared__ int s_next;
    if (tid == 0) {
        int pick = s_pick;
        if (a.given) {   // a given token of an inpainting call replaces the draw
            const int g = a.given[(size_t)b * G * a.seq_stride + step];
            if (g >= 0) pick = g;
        }
        if (a.out_idx) a.out_idx[b] = pick;
        if (a.out_seq) a.out_seq[(size_t)b * a.seq_stride + step] = pick;
        const int nxt = a.teacher ? a.teacher[(size_t)b * a.seq_stride + step] : pick;
        if (a.next_tokens) {
            if constexpr (kGroups) {
                for (int i = 0; i < G; ++i) a.next_tokens[b * G + i] = nxt;
            } else {
                a.next_tokens[b] = nxt;
            }
        }
        s_next = nxt;
        if (a.dbg_path) {
            a.dbg_path[3 * b] = path_topk;
            a.dbg_path[3 * b + 1] = path_trim;
            a.dbg_path[3 * b + 2] = s_end;
        }
    }
    // ---------------- fused tail: next step's input rows (embedding lookup + layer-0 RMSNorm) and the counter advance ----------
    if (a.emb_table) {
        __syncthreads();
        const int D = a.emb_D;
        const E* src = reinterpret_cast<const E*>(a.emb_table) + (size_t)s_next * D;
        // thread -> 2 consecutive elements per pass (D even); the same token feeds the cond and the uncond row (generate.py:91)
        for (int i = tid * 2; i < D; i += kSampleThreads * 2) {
            const uint32_t w = *reinterpret_cast<const uint32_t*>(src + i);
            for (int row = b * G; row < a.emb_rows; row += B)
                for (int j = 0; j < G; ++j)   // G = 1 without kGroups
                    *reinterpret_cast<uint32_t*>(reinterpret_cast<E*>(a.emb_h) + (size_t)(row + j) * D + i) = w;
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
                for (int row = b * G; row < a.emb_rows; row += B)
                    for (int j = 0; j < G; ++j)
                        *reinterpret_cast<uint32_t*>(reinterpret_cast<E*>(a.emb_xn) + (size_t)(row + j) * D + i) = pk;
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
    LG_REQUIRE(a.B > 0 && a.V > 0 && a.param_div >= 1, "lg_sample: bad shape B=%d V=%d param_div=%d", a.B, a.V, a.param_div);
    const bool lp = sample_wants_logprobs(a);
    const size_t smem = lp ? sample_lp_smem(a.V) : (size_t)a.V * sizeof(float);
    LG_REQUIRE(smem <= 200 * 1024, "lg_sample: vocab %d too large for the shared-memory row stage%s", a.V, lp ? " with logprobs" : "");
    LG_REQUIRE(a.round_dtype == LG_DTYPE_F32 || lg_dtype_is16(a.round_dtype), "lg_sample: unsupported round dtype %d", a.round_dtype);
    LG_REQUIRE(!a.emb_table || a.round_dtype != LG_DTYPE_F32, "lg_sample: the fused tail needs a 16-bit round dtype");
    LG_REQUIRE(a.top_n >= 0 && a.top_n <= kMaxTopLogprobs && (a.top_n == 0) == (!a.top_ids && !a.top_lp) &&
                   (a.top_n == 0 || (a.top_ids && a.top_lp)),
               "lg_sample: top_n=%d outside [0, %d], or top_ids / top_logprob not both given exactly when top_n > 0", a.top_n,
               kMaxTopLogprobs);
    const bool table = a.mix_rows != nullptr;
    const bool grp = a.mix_groups > 0 || table;
    if (table) {
        LG_REQUIRE(a.mix_groups == 0 && a.mix_cfg && a.mix_weights && a.seed_rows,
                   "lg_sample: a gather table (mix_rows) needs mix_groups 0, mix_cfg, per-row weights and seed_rows");
        LG_REQUIRE(!a.emb_table && !a.adv_pos && !a.adv_step && !a.dbg_logits,
                   "lg_sample: a gather table (mix_rows) takes no fused tail or dbg_logits");
    } else if (grp) {
        LG_REQUIRE(a.mix_groups <= kMaxMixGroups && a.B % a.mix_groups == 0 && a.mix_cfg && a.mix_weights,
                   "lg_sample: composable guidance needs 1 <= K=%d <= %d dividing B=%d rows, mix_cfg and weights", a.mix_groups,
                   kMaxMixGroups, a.B);
        LG_REQUIRE(!a.cfg_rows && !a.interval_rows && !a.dbg_logits,
                   "lg_sample: composable guidance takes no per-row guidance or dbg_logits");
        LG_REQUIRE(!a.emb_table || a.emb_rows == a.B || a.emb_rows == 2 * a.B, "lg_sample: the fused tail of groups needs emb_rows B or 2B");
    }
    const bool half = a.round_dtype == LG_DTYPE_F16;
    auto kern = grp ? (lp ? (half ? sample_kernel<f16, true, true> : sample_kernel<bf16, true, true>)
                          : (half ? sample_kernel<f16, false, true> : sample_kernel<bf16, false, true>))
                    : lp ? (half ? sample_kernel<f16, true, false> : sample_kernel<bf16, true, false>)
                         : (half ? sample_kernel<f16, false, false> : sample_kernel<bf16, false, false>);
    static DevOnce attr_set[8];
    if (lg_first_on_device(attr_set[4 * grp + 2 * lp + half])) {
        LG_CUDA_OK(cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, 200 * 1024));
    }
    (void)lg_launch(kern, dim3(grp && !table ? a.B / a.mix_groups : a.B), dim3(kSampleThreads), smem, st, a);
    LG_LAUNCH_CHECK();
    return 0;
}

namespace {
__global__ void given_logprobs_kernel(float* lp, int32_t* rank, int32_t* top_ids, float* top_lp, int top_n, int S, int P) {
    lg_pdl_sync();
    const int b = blockIdx.x;
    for (int k = threadIdx.x; k < P; k += blockDim.x) {
        const size_t o = (size_t)b * S + k;
        if (lp) lp[o] = 0.f;
        if (rank) rank[o] = 0;
        for (int j = 0; j < top_n; ++j) {
            if (top_ids) top_ids[o * top_n + j] = -1;
            if (top_lp) top_lp[o * top_n + j] = -INFINITY;
        }
    }
}
}  // namespace

int launch_given_logprobs(float* lp, int32_t* rank, int32_t* top_ids, float* top_lp, int top_n, int B, int S, int P, cudaStream_t st) {
    LG_REQUIRE(B > 0 && P >= 0 && P <= S && top_n >= 0, "given logprobs: bad shape B=%d S=%d P=%d top_n=%d", B, S, P, top_n);
    if (P == 0) return 0;
    (void)lg_launch(given_logprobs_kernel, dim3(B), dim3(128), 0, st, lp, rank, top_ids, top_lp, top_n, S, P);
    LG_LAUNCH_CHECK();
    return 0;
}

namespace {
__global__ void given_window_kernel(const int32_t* tokens, const int32_t* given, int B, int nh, int S, int j0, int n, int from_tokens,
                                    int pos0, int32_t* win, int32_t* pos_rows) {
    lg_pdl_sync();
    const int b = blockIdx.x;
    for (int i = threadIdx.x; i < n; i += blockDim.x)
        win[(size_t)b * n + i] = i == 0 && from_tokens ? tokens[b] : given[(size_t)b * S + j0 + i];
    if (threadIdx.x == 0)
        for (int h = 0; h < nh; ++h) pos_rows[h * B + b] = pos0;
}
}  // namespace

int launch_given_window(const int32_t* tokens, const int32_t* given, int B, int nh, int S, int j0, int n, int from_tokens, int pos0,
                        int32_t* win, int32_t* pos_rows, cudaStream_t st) {
    LG_REQUIRE(B > 0 && (nh == 1 || nh == 2) && n >= 1 && j0 >= 0 && j0 + n <= S, "given window: bad shape B=%d nh=%d S=%d j0=%d n=%d", B,
               nh, S, j0, n);
    (void)lg_launch(given_window_kernel, dim3(B), dim3(64), 0, st, tokens, given, B, nh, S, j0, n, from_tokens, pos0, win, pos_rows);
    LG_LAUNCH_CHECK();
    return 0;
}

// ---------------------------------------------------------------------------------------------------
// Speculative Jacobi decoding (lg_generate_sjd): acceptance and the next window. One pass of the loop feeds image b's window of L
// tokens (slot i holds token s_b + i - 1, s_b = start[b]) through the model; the sample kernel then writes p_{s_b + i} for every slot
// (out_probs) and a draw x_i from it (argmax in greedy mode). The uniforms (sjd_uniform, mirrored by tests/sjd_oracle.py) are keyed
// by (seed, image, token index, purpose); the redraw x_i is the sample kernel's own draw with seed_rows = sjd_pass_seed(seed, b, pass)
// and step_rows = the token index, so no uniform is used twice.
namespace {

enum SjdPurpose : uint64_t { kSjdAccept = 1, kSjdResidual = 2, kSjdInit = 3 };

__device__ __forceinline__ float sjd_uniform(uint64_t seed, int b, int k, uint64_t purpose) {
    const uint64_t r = splitmix64(splitmix64(splitmix64(seed ^ (0xA0761D6478BD642Full * (uint64_t)(k + 1))) ^
                                             (0xE7037ED1A0B428DBull * (uint64_t)(b + 1))) ^
                                  (0x8EBC6AF09C88C6E3ull * purpose));
    return (float)(r >> 40) * (1.0f / 16777216.0f);
}
__device__ __forceinline__ uint64_t sjd_pass_seed(uint64_t seed, int b, int pass) {
    return splitmix64(splitmix64(seed ^ (0x9E6C63D0676A9A99ull * (uint64_t)(b + 1))) ^ (0xD6E8FEB86659FD93ull * (uint64_t)(pass + 1)));
}

constexpr int kSjdThreads = 512;

// One CTA per image: accept a prefix of the drafts, draw the token that ends it, advance the image's window
__global__ void __launch_bounds__(kSjdThreads) sjd_verify_kernel(SjdArgs a) {
    lg_pdl_sync();
    __shared__ float red[33];
    __shared__ float s_wtot[32];
    __shared__ int s_i, s_pick, s_own[32];
    const int b = blockIdx.x, tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
    const int L = a.L, V = a.V, S = a.S;
    const int n = a.nfin[b], s = a.start[b];
    const bool active = n < S;
    const uint64_t seed = a.seed_slots ? a.seed_slots[b] : a.seed;   // per-slot mode: the slot's seed and image index
    const bool greedy = a.greedy_rows ? a.greedy_rows[b] != 0 : a.greedy != 0;
    const int img = a.seed_slots ? (a.img_slots ? a.img_slots[b] : 0) : b + a.row_offset;
    if (active) {
        const size_t row0 = (size_t)b * L;
        if (tid == 0) {
            int i = n - s;
            for (; i <= L - 2; ++i) {   // the draft for token s + i is fed in slot i + 1 and checked against p_{s + i} (slot i)
                const int d = a.win[row0 + i + 1], k = s + i;
                bool acc;
                if (greedy) {
                    acc = d == a.x[row0 + i];
                } else {
                    const float pd = a.p[(row0 + i) * V + d];
                    const float qd = a.qflag[row0 + i] ? 1.0f / (float)V : a.q[(row0 + i) * V + d];
                    acc = sjd_uniform(seed, img, k, kSjdAccept) * qd < pd;
                }
                if (!acc) break;
                a.out[(size_t)b * S + k] = d;
            }
            s_i = i;
            s_pick = a.x[row0 + min(i, L - 1)];   // bonus token, greedy correction, or the fallback of an empty residual
        }
        __syncthreads();
        const int i = s_i;
        if (i <= L - 2 && !greedy) {
            // residual draw: normalize(max(0, p - q)), inverse CDF over contiguous per-thread segments
            const float* pr = a.p + (row0 + i) * V;
            const float* qr = a.q + (row0 + i) * V;
            const bool uni = a.qflag[row0 + i] != 0;
            const float qu = 1.0f / (float)V;
            const int seg = (V + kSjdThreads - 1) / kSjdThreads;
            const int v0 = min(tid * seg, V), v1 = min(v0 + seg, V);
            float local = 0.f;
            for (int v = v0; v < v1; ++v) local += fmaxf(0.f, pr[v] - (uni ? qu : qr[v]));
            float incl = local;
#pragma unroll
            for (int o = 1; o < 32; o <<= 1) {
                const float t = __shfl_up_sync(0xffffffffu, incl, o);
                if (lane >= o) incl += t;
            }
            if (lane == 31) s_wtot[warp] = incl;
            __syncthreads();
            if (warp == 0) {
                const float w = lane < kSjdThreads / 32 ? s_wtot[lane] : 0.f;
                float wi = w;
#pragma unroll
                for (int o = 1; o < 32; o <<= 1) {
                    const float t = __shfl_up_sync(0xffffffffu, wi, o);
                    if (lane >= o) wi += t;
                }
                if (lane < kSjdThreads / 32) s_wtot[lane] = wi - w;
                if (lane == 31) red[32] = wi;
            }
            __syncthreads();
            const float total = red[32];
            if (total > 0.f) {
                const float target = sjd_uniform(seed, img, s + i, kSjdResidual) * total;
                const float excl = s_wtot[warp] + (incl - local);
                // one owner for every target, as in sample_kernel: the highest thread with a positive segment starting at or below
                // it; a walk that never passes the target takes the segment's last positive weight
                const int owner = block_last_true<kSjdThreads>(local > 0.f && excl <= target, s_own);
                if (tid == owner) {
                    float c = excl;
                    int pick = -1, lastnz = -1;
                    for (int v = v0; v < v1; ++v) {
                        const float e = fmaxf(0.f, pr[v] - (uni ? qu : qr[v]));
                        if (e > 0.f) lastnz = v;
                        c += e;
                        if (c > target && e > 0.f) { pick = v; break; }
                    }
                    s_pick = pick >= 0 ? pick : lastnz;
                }
            }
            __syncthreads();
        }
        if (tid == 0) {
            const int k = s + i, n2 = k + 1, s2 = min(n2, S - L);
            a.out[(size_t)b * S + k] = s_pick;
            a.nfin[b] = n2;
            a.start[b] = s2;
            a.shift[b] = s2 - s;
            for (int hh = 0; hh < a.nh; ++hh) a.pos_rows[hh * a.B + b] = a.T + s2 - 1;
            if (a.pass_slots) a.pass_slots[b] += 1;
            atomicAdd(&a.state[kSjdActive], 1);
            if (n2 >= S) atomicAdd(&a.state[kSjdFinished], 1);
        }
    }
    if (tid == 0) {
        __threadfence();
        if (atomicAdd(reinterpret_cast<unsigned int*>(&a.state[kSjdTicket]), 1u) == gridDim.x - 1) {
            const int act = atomicExch(&a.state[kSjdActive], 0);
            a.state[kSjdLive] = act > 0;
            if (act > 0) a.state[kSjdIters] += 1;
            if (atomicAdd(&a.state[kSjdFinished], 0) >= a.B) a.state[kSjdDone] = a.done_token;
            a.state[kSjdTicket] = 0;
        }
    }
}

// grid (B, L), or (1, L) for image `slot` >= 0: slot i of image b's next window. first = 1 sets up the window after the prefill (token
// 0 final, all drafts new); in per-slot mode it also sets the slot's seed, pass counter, image index and window rows' guidance.
__global__ void __launch_bounds__(256) sjd_refresh_kernel(SjdArgs a, int first, int only) {
    lg_pdl_sync();
    const int b = only >= 0 ? only : blockIdx.x, i = blockIdx.y, L = a.L, V = a.V, S = a.S;
    const size_t slot = (size_t)b * L + i;
    if (!first && !a.state[kSjdLive]) return;   // a pass after every image finished changes nothing
    // index of the next pass: the call's, or the slot's own (0 at its start)
    const int pass = a.pass_slots ? (first ? 0 : a.pass_slots[b]) : a.state[kSjdIters];
    const uint64_t seed = a.seed_slots && !first ? a.seed_slots[b] : a.seed;
    const int img = !a.seed_slots ? b + a.row_offset : first ? a.start_img : a.img_slots ? a.img_slots[b] : 0;
    if (!first && a.dbg) {
        float* d = a.dbg + ((size_t)(pass - 1) * a.B * L + slot) * V;
        for (int v = threadIdx.x; v < V; v += blockDim.x) d[v] = a.p[slot * V + v];
    }
    int n, s, shift;
    if (first) {
        n = 1; s = 1; shift = 1 << 20;
        if (i == 0 && threadIdx.x == 0) {
            a.nfin[b] = 1; a.start[b] = 1;
            for (int hh = 0; hh < a.nh; ++hh) a.pos_rows[hh * a.B + b] = a.T;
            if (a.seed_slots) { a.seed_slots[b] = a.seed; a.pass_slots[b] = 0; }
            if (a.img_slots) a.img_slots[b] = a.start_img;
        }
        if (a.cfg_rows && threadIdx.x == 0) { a.cfg_rows[slot] = a.start_cfg; a.interval_rows[slot] = a.start_interval; }
    } else {
        n = a.nfin[b]; s = a.start[b]; shift = a.shift[b];
        if (n >= S) return;                      // finished: its rows keep running on the old window, their outputs unused
    }
    const int k = s + i - 1;                     // the token this slot feeds
    if (threadIdx.x == 0) {
        a.seed_rows[slot] = sjd_pass_seed(seed, img, pass);
        a.step_rows[slot] = s + i;
    }
    if (k < n) {
        if (threadIdx.x == 0) a.win[slot] = a.out[(size_t)b * S + k];
        return;
    }
    const int j = k - (s - shift);               // the slot of the pass just run that computed p_k
    const size_t qs = slot - 1;                  // q of the draft for token k sits at slot k - s
    if (j <= L - 1) {                            // Jacobi update: redraw from p_k, which becomes its q
        const float* src = a.p + ((size_t)b * L + j) * V;
        float* dst = a.q + qs * V;
        for (int v = threadIdx.x; v < V; v += blockDim.x) dst[v] = src[v];
        if (threadIdx.x == 0) { a.win[slot] = a.x[(size_t)b * L + j]; a.qflag[qs] = 0; }
    } else if (threadIdx.x == 0) {               // a new index: uniform over the vocabulary, q = 1 / V
        const int t = (int)(sjd_uniform(seed, img, k, kSjdInit) * (float)V);
        a.win[slot] = min(t, V - 1);
        a.qflag[qs] = 1;
    }
}

}  // namespace

int launch_sjd_verify(const SjdArgs& a, cudaStream_t st) {
    LG_REQUIRE(a.B > 0 && a.L >= 1 && a.L <= 64 && a.S > a.L && a.V > 0, "sjd: bad shape B=%d L=%d S=%d V=%d", a.B, a.L, a.S, a.V);
    (void)lg_launch(sjd_verify_kernel, dim3(a.B), dim3(kSjdThreads), 0, st, a);
    LG_LAUNCH_CHECK();
    return 0;
}

int launch_sjd_refresh(const SjdArgs& a, int first, cudaStream_t st, int slot) {
    LG_REQUIRE(a.B > 0 && a.L >= 1 && a.L <= 64 && a.S > a.L && a.V > 0, "sjd: bad shape B=%d L=%d S=%d V=%d", a.B, a.L, a.S, a.V);
    LG_REQUIRE(slot < a.B && (slot < 0 || first), "sjd: a refresh of one slot (%d of B=%d) is a start (first = 1)", slot, a.B);
    (void)lg_launch(sjd_refresh_kernel, dim3(slot >= 0 ? 1 : a.B, a.L), dim3(256), 0, st, a, first, slot);
    LG_LAUNCH_CHECK();
    return 0;
}
