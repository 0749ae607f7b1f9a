// Persistent decode step for R <= 8 activation rows (the batch-1 latency path; R = 2 with classifier-free guidance).
//
// One cooperative launch runs ONE WHOLE TOKEN (all layers + the head) of gpt.py:243-257,341-368 on every SM:
//   per layer  P1  xn = RMSNorm(h); q,k,v = xn Wqkv^T; RoPE(q,k); K/V row -> cache         (gpt.py:143-148,214-230)
//              P2  split-context attention over the cached prefix + the new key             (gpt.py:232-236)
//              P3  h += merge(P2) Wo^T                                                      (gpt.py:239,255)
//              P4  xn = RMSNorm(h); ff = silu(xn W1^T) * (xn W3^T)                          (gpt.py:167)
//              P5  h += ff W2^T                                                             (gpt.py:256)
//   then       PH  logits = RMSNorm(h) Wout^T                                               (gpt.py:367-368)
// Phases are separated by a grid barrier (one L2 atomic + an acquire spin per CTA, ~0.5 us) instead of a kernel boundary
// (~3.3 us measured per dependent kernel on the 5-kernel/layer path this replaces: 122 kernels/token = 411 us).
//
// The point of being persistent: WEIGHTS AND OLD KV ROWS DO NOT DEPEND ON ACTIVATIONS. A dedicated producer warp per CTA
// walks the CTA's static tile list of the whole token (every phase, every layer) and streams it with cp.async.bulk into a
// shared-memory ring (11 x 16.5 KB), throttled only by the ring's empty barriers — so the HBM stream never stops at a phase
// boundary, and when a grid barrier releases, the tiles of the next phase are already on chip.
//
// Work split: a phase's output features are cut into groups of 8 (one n8 MMA tile); group gi belongs to CTA
// (gi + rot) mod G with a per-phase rotation `rot`, so the byte load per CTA is balanced over a layer. Inside a CTA the 8
// compute warps split K (each owns a k-range of every tile), accumulate with mma.sync m16n8k16 (activations = M operand,
// rows >= R are zero; the 8 weight rows = N operand, fetched from the ring with ldmatrix) and combine through shared memory
// in a fixed order — no atomics on any data path, results are bit-reproducible.
//
// Rounding points are those of the batched path and of the reference's bf16 tensors (see gemv_small.cu / xf_kernels.cu).
#include "kernels.cuh"
#include "tma_utils.cuh"
#include <algorithm>

namespace {

using namespace tma;

constexpr int kCW = 8;                            // compute warps
constexpr int kCT = kCW * 32;                     // compute threads
constexpr int kThreadsPd = kCT + 32;              // + one producer warp
constexpr int kKc = 1024;                         // k elements of one weight tile (8 rows x kKc)
constexpr int kSlot = 8 * (kKc * 2 + 16);         // 16512 B: 8 rows, each padded by 16 B (conflict-free ldmatrix)
constexpr int kHalf = kSlot / 2;                  // KV tile: K rows in the first half, V rows in the second
constexpr int kGB = 8;                            // feature groups combined per epilogue round
constexpr int kMaxSlots = 12;

struct PdArgs {
    int L, D, F, V, H, hd, R, B, Tc, maxS, nslots, nsplit;
    float eps, scale;
    const PdLayerW* layers;      // device array [L]
    const bf16 *final_norm, *output, *tok_emb;
    const float* freqs;          // [P, hd/2, 2]
    bf16 *kcache, *vcache;       // layer 0 of the (sub-)workspace: [rows, H, maxS, hd]
    size_t layer_elems;          // elements between layers
    bf16 *h, *q, *ff;            // [R][D], [R][D], [R][F]
    float* part;                 // [R*H*nsplit][hd + 2] attention partials (o[hd], m, l)
    float* logits;               // [R][V]
    const int32_t* tokens;       // [B] token fed to this step
    const int* pos_dev; int pos_value;
    const float* emb_mask;       // [B][Tc] or null
    unsigned int* bar;           // [0] grid-barrier counter, [1] exit counter (both zero between launches)
    int xs_bytes;                // bytes of the activation stage
    unsigned long long* trace;   // debug: %globaltimer stamps [2 CTAs][L + 1][16] (nullable), see tools/persist_probe.py
};

__device__ __forceinline__ void bulk_g2s(void* dst, const void* src, uint32_t bytes, uint64_t* bar) {
    asm volatile("cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];"
                 ::"r"(smem_u32(dst)), "l"(src), "r"(bytes), "r"(smem_u32(bar)) : "memory");
}
__device__ __forceinline__ void ldsm_x4(uint32_t addr, uint32_t& r0, uint32_t& r1, uint32_t& r2, uint32_t& r3) {
    asm volatile("ldmatrix.sync.aligned.m8n8.x4.shared.b16 {%0,%1,%2,%3}, [%4];\n" : "=r"(r0), "=r"(r1), "=r"(r2), "=r"(r3) : "r"(addr));
}
__device__ __forceinline__ void mma16816(float* c, uint32_t a0, uint32_t a2, uint32_t b0, uint32_t b1) {
    // rows 8..15 of the A tile (a1, a3) are zero: at most 8 activation rows
    asm volatile("mma.sync.aligned.m16n8k16.row.col.f32.bf16.bf16.f32 {%0,%1,%2,%3}, {%4,%5,%6,%7}, {%8,%9}, {%0,%1,%2,%3};\n"
                 : "+f"(c[0]), "+f"(c[1]), "+f"(c[2]), "+f"(c[3]) : "r"(a0), "r"(0u), "r"(a2), "r"(0u), "r"(b0), "r"(b1));
}
__device__ __forceinline__ void cbar() { asm volatile("bar.sync 1, %0;" ::"n"(kCT) : "memory"); }   // compute warps only
__device__ __forceinline__ float bfr(float v) { return __bfloat162float(__float2bfloat16_rn(v)); }
__device__ __forceinline__ uint32_t pack2(float a, float b) {
    __nv_bfloat162 p = __floats2bfloat162_rn(a, b);
    return *reinterpret_cast<uint32_t*>(&p);
}
__device__ __forceinline__ float lo_f(uint32_t w) { return __uint_as_float(w << 16); }
__device__ __forceinline__ float hi_f(uint32_t w) { return __uint_as_float(w & 0xffff0000u); }

// One GEMM phase: y[r, n] = sum_k x[r, k] W[n, k]; paired: two matrices with the same row range (w1 | w3).
struct Gemm {
    const bf16* Wa; const bf16* Wb;   // Wb != null: paired
    int N, K, rot;
};
__device__ __forceinline__ int first_group(const Gemm& gm, int cta, int G) {
    int f = (cta - gm.rot) % G;
    return f < 0 ? f + G : f;
}
__device__ __forceinline__ int owned_groups(const Gemm& gm, int cta, int G) {
    const int ng = gm.N / 8, f = first_group(gm, cta, G);
    return f < ng ? (ng - f + G - 1) / G : 0;
}
__device__ __forceinline__ int phase_rot(int layer, int phase, int G) { return (int)(((unsigned)(layer * 6 + phase) * 53u) % (unsigned)G); }

// Attention work unit u = ((r * H) + head) * nsplit + s : keys [jb, je) of the context c = qpos + 1; the old keys [jb, oe) come
// from the cache through the ring in tiles of kt keys, the new key (index qpos) from global memory after the barrier.
struct Unit { int r, head, jb, je, oe, ntiles; bool has_new; };
__device__ __forceinline__ Unit make_unit(int u, int H, int nsplit, int qpos, int kt) {
    Unit x;
    const int item = u / nsplit, s = u - item * nsplit;
    x.r = item / H; x.head = item - x.r * H;
    const int c = qpos + 1, cq = (c + nsplit - 1) / nsplit;
    x.jb = min(c, s * cq); x.je = min(c, x.jb + cq);
    x.oe = min(x.je, qpos);
    x.has_new = x.jb <= qpos && qpos < x.je;
    x.ntiles = x.oe > x.jb ? (x.oe - x.jb + kt - 1) / kt : 0;
    return x;
}

__global__ void __launch_bounds__(kThreadsPd, 1) decode_small_persistent_kernel(PdArgs a) {
    extern __shared__ __align__(128) uint8_t smem[];
    // layout: [ring nslots * kSlot][full bars][empty bars][xs activation stage][red][misc]
    uint8_t* ring = smem;
    uint64_t* full = reinterpret_cast<uint64_t*>(ring + (size_t)a.nslots * kSlot);
    uint64_t* empty = full + kMaxSlots;
    uint8_t* xs = reinterpret_cast<uint8_t*>(empty + kMaxSlots);
    float* red = reinterpret_cast<float*>(xs + a.xs_bytes);          // [kCW][kGB slots][8 rows][8 feats]
    float* misc = red + kCW * kGB * 64;                               // 512 floats: row sums, attention scratch
    const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
    const int cta = blockIdx.x, G = gridDim.x;
    const int ns = a.nslots;
    const int D = a.D, F = a.F, H = a.H, hd = a.hd, R = a.R;
    const int kt = kHalf / (hd * 2);                                  // keys per KV tile

    if (tid == 0) {
        for (int s = 0; s < ns; ++s) { mbar_init(&full[s], 1); mbar_init(&empty[s], kCW); }
        fence_barrier_init();
    }
    __syncthreads();
    const int qpos = (a.pos_dev ? *a.pos_dev : 0) + a.pos_value;
    const int nunits = R * H * a.nsplit;

    // ======================================================================================== producer warp
    if (warp == kCW) {
        if (lane == 0) {
            uint32_t seq = 0;
            auto acquire = [&](uint32_t bytes) -> uint8_t* {
                const int s = (int)(seq % (uint32_t)ns);
                mbar_wait(&empty[s], ((seq / (uint32_t)ns) & 1u) ^ 1u);
                mbar_expect_tx(&full[s], bytes);
                return ring + (size_t)s * kSlot;
            };
            auto gemm_tiles = [&](const Gemm& gm) {
                const int cnt = owned_groups(gm, cta, G), f0 = first_group(gm, cta, G);
                const int nmat = gm.Wb ? 2 : 1, nkc = (gm.K + kKc - 1) / kKc;
                for (int m = 0; m < cnt; ++m) {
                    const size_t row0 = (size_t)(f0 + m * G) * 8;
                    for (int mat = 0; mat < nmat; ++mat) {
                        const bf16* W = (mat ? gm.Wb : gm.Wa) + row0 * gm.K;
                        for (int kc = 0; kc < nkc; ++kc) {
                            const int k0 = kc * kKc, kl = min(kKc, gm.K - k0);
                            uint8_t* dst = acquire((uint32_t)(8 * kl * 2));
                            const int s = (int)(seq % (uint32_t)ns);
#pragma unroll
                            for (int r = 0; r < 8; ++r)
                                bulk_g2s(dst + (size_t)r * (kl * 2 + 16), W + (size_t)r * gm.K + k0, (uint32_t)(kl * 2), &full[s]);
                            ++seq;
                        }
                    }
                }
            };
            for (int l = 0; l < a.L; ++l) {
                const PdLayerW& ly = a.layers[l];
                gemm_tiles(Gemm{ly.wqkv, nullptr, 3 * D, D, phase_rot(l, 0, G)});
                // old K/V rows of this CTA's attention units (rows written in EARLIER steps only)
                for (int u = cta; u < nunits; u += G) {
                    const Unit x = make_unit(u, H, a.nsplit, qpos, kt);
                    const size_t base = (size_t)l * a.layer_elems + ((size_t)(x.r * H + x.head) * a.maxS) * hd;
                    for (int t = 0; t < x.ntiles; ++t) {
                        const int j0 = x.jb + t * kt, nk = min(kt, x.oe - j0);
                        const uint32_t bytes = (uint32_t)(nk * hd * 2);
                        uint8_t* dst = acquire(2 * bytes);
                        const int s = (int)(seq % (uint32_t)ns);
                        bulk_g2s(dst, a.kcache + base + (size_t)j0 * hd, bytes, &full[s]);
                        bulk_g2s(dst + kHalf, a.vcache + base + (size_t)j0 * hd, bytes, &full[s]);
                        ++seq;
                    }
                }
                gemm_tiles(Gemm{ly.wo, nullptr, D, D, phase_rot(l, 2, G)});
                gemm_tiles(Gemm{ly.w1, ly.w3, F, D, phase_rot(l, 3, G)});
                gemm_tiles(Gemm{ly.w2, nullptr, D, F, phase_rot(l, 4, G)});
            }
            gemm_tiles(Gemm{a.output, nullptr, a.V, D, phase_rot(a.L, 0, G)});
        }
        return;      // the producer warp takes no part in the compute-side barriers (bar.sync 1, kCT)
    }

    // ======================================================================================== compute warps
    const int g = lane >> 2, t = lane & 3;
    const int tcta = cta == 0 ? 0 : (cta == G - 1 ? 1 : -1);
    auto stamp = [&](int l, int k) {
        if (a.trace && tcta >= 0 && tid == 0) {
            unsigned long long tm;
            asm volatile("mov.u64 %0, %%globaltimer;" : "=l"(tm));
            a.trace[((size_t)tcta * (a.L + 1) + l) * 16 + k] = tm;
        }
    };
    uint32_t seq = 0;                      // same tile sequence as the producer
    unsigned int bar_target = 0;
    auto grid_barrier = [&]() {
        cbar();
        if (tid == 0) {
            __threadfence();
            atomicAdd(a.bar, 1u);
            bar_target += (unsigned)G;
            unsigned int v;
            unsigned long long spins = 0;
            do {
                asm volatile("ld.acquire.gpu.global.u32 %0, [%1];" : "=r"(v) : "l"(a.bar) : "memory");
                if (++spins > (1ull << 27)) __trap();      // a lost CTA must surface as a launch failure, never as a hung GPU
            } while (v < bar_target);
        }
        cbar();
    };

    // token rows of this step (decode: cond and uncond rows carry the same token, generate.py:91)
    auto h_row = [&](int l, int r) -> const bf16* {
        return l == 0 ? a.tok_emb + (size_t)a.tokens[r % a.B] * D : a.h + (size_t)r * D;
    };

    int rp = 1;
    while (rp < R) rp <<= 1;
    const int tpr = kCT / rp, srow = tid / tpr, sj = tid % tpr;       // activation staging: tpr threads per row

    // xs <- rows [R][K] (bf16) given by src(r); optional RMSNorm * normw (gpt.py:143-148)
    auto stage_rows = [&](auto src, int K, const bf16* normw) {
        const int stride = K * 2 + 16, pieces = K / 8;
        float ss = 0.f;
        if (srow < R) {
            const uint4* sp = reinterpret_cast<const uint4*>(src(srow));
            for (int p = sj; p < pieces; p += tpr) {
                const uint4 v = __ldcg(sp + p);
                *reinterpret_cast<uint4*>(xs + (size_t)srow * stride + (size_t)p * 16) = v;
                if (normw) {
                    const uint32_t w[4] = {v.x, v.y, v.z, v.w};
#pragma unroll
                    for (int q = 0; q < 4; ++q) { ss = fmaf(lo_f(w[q]), lo_f(w[q]), ss); ss = fmaf(hi_f(w[q]), hi_f(w[q]), ss); }
                }
            }
        }
        if (normw) {
            ss = warp_sum(ss);
            if (lane == 0) misc[warp] = ss;                 // warps of one row are contiguous
            cbar();
            if (srow < R) {
                const int wpr = tpr / 32;
                float tot = 0.f;
                for (int w = 0; w < wpr; ++w) tot += misc[srow * wpr + w];
                const float rinv = 1.0f / sqrtf(tot / (float)K + a.eps);
                for (int p = sj; p < pieces; p += tpr) {
                    uint4* px = reinterpret_cast<uint4*>(xs + (size_t)srow * stride + (size_t)p * 16);
                    const uint4 v = *px, nw = __ldg(reinterpret_cast<const uint4*>(normw) + p);
                    const uint32_t w[4] = {v.x, v.y, v.z, v.w}, n[4] = {nw.x, nw.y, nw.z, nw.w};
                    uint32_t o[4];
#pragma unroll
                    for (int q = 0; q < 4; ++q)
                        o[q] = pack2(bfr(lo_f(w[q]) * rinv) * lo_f(n[q]), bfr(hi_f(w[q]) * rinv) * hi_f(n[q]));
                    *px = make_uint4(o[0], o[1], o[2], o[3]);
                }
            }
        }
        cbar();
    };

    // Runs the CTA's tiles of one GEMM phase against xs; epi(m0, nb) is called after every batch of nb <= kGB / nmat groups
    // (first group index m0) with red[w][slot][row][feat] holding the 8 warps' partial sums (slot = (m - m0) * nmat + mat).
    auto run_gemm = [&](const Gemm& gm, auto epi) {
        const int cnt = owned_groups(gm, cta, G);
        const int nmat = gm.Wb ? 2 : 1, nkc = (gm.K + kKc - 1) / kKc;
        const int xstride = gm.K * 2 + 16;
        const int gcap = kGB / nmat;                         // groups per batch (paired: 2 slots per group)
        const uint8_t* xrow = xs + (size_t)min(g, R - 1) * xstride;
        const bool live = g < R;
        for (int m0 = 0; m0 < cnt; m0 += gcap) {
            const int nb = min(gcap, cnt - m0);
            for (int m = 0; m < nb; ++m) {
                for (int mat = 0; mat < nmat; ++mat) {
                    float acc[4] = {0.f, 0.f, 0.f, 0.f};
                    for (int kc = 0; kc < nkc; ++kc) {
                        const int k0 = kc * kKc, kl = min(kKc, gm.K - k0);
                        const int s = (int)(seq % (uint32_t)ns);
                        mbar_wait(&full[s], (seq / (uint32_t)ns) & 1u);
                        const int np = kl / 32;              // pairs of k16 steps
                        const int p0 = warp * np / kCW, p1 = (warp + 1) * np / kCW;
                        const uint32_t tb = smem_u32(ring + (size_t)s * kSlot) + (uint32_t)((lane & 7) * (kl * 2 + 16) + (lane >> 3) * 16);
                        for (int p = p0; p < p1; ++p) {
                            uint32_t b0, b1, b2, b3;
                            ldsm_x4(tb + (uint32_t)(p * 64), b0, b1, b2, b3);
                            const uint8_t* xa = xrow + (size_t)(k0 + p * 32 + 2 * t) * 2;
                            uint32_t a0 = *reinterpret_cast<const uint32_t*>(xa), a2 = *reinterpret_cast<const uint32_t*>(xa + 16);
                            uint32_t c0 = *reinterpret_cast<const uint32_t*>(xa + 32), c2 = *reinterpret_cast<const uint32_t*>(xa + 48);
                            if (!live) { a0 = 0u; a2 = 0u; c0 = 0u; c2 = 0u; }
                            mma16816(acc, a0, a2, b0, b1);
                            mma16816(acc, c0, c2, b2, b3);
                        }
                        __syncwarp();
                        if (lane == 0) mbar_arrive(&empty[s]);
                        ++seq;
                    }
                    float* rw = red + ((size_t)(warp * kGB + m * nmat + mat) * 8 + g) * 8 + 2 * t;
                    *reinterpret_cast<float2*>(rw) = make_float2(acc[0], acc[1]);
                }
            }
            cbar();
            epi(m0, nb);
            cbar();
        }
    };
    // sum of the 8 warps' partials for (slot, row, feat) in warp order (deterministic)
    auto red_sum = [&](int slot, int row, int feat) -> float {
        float v = 0.f;
#pragma unroll
        for (int w = 0; w < kCW; ++w) v += red[((size_t)(w * kGB + slot) * 8 + row) * 8 + feat];
        return v;
    };

    for (int l = 0; l < a.L; ++l) {
        const PdLayerW& ly = a.layers[l];
        // ------------------------------------------------------------------------------------------------ P1: QKV
        {
            const Gemm gm{ly.wqkv, nullptr, 3 * D, D, phase_rot(l, 0, G)};
            stamp(l, 0);
            stage_rows([&](int r) { return h_row(l, r); }, D, ly.attn_norm);
            stamp(l, 1);
            const int f0 = first_group(gm, cta, G);
            run_gemm(gm, [&](int m0, int nb) {
                // thread -> (group slot, feature pair, row): RoPE needs the (2j, 2j+1) pair (gpt.py:420-430)
                for (int i = tid; i < nb * 4 * 8; i += kCT) {
                    const int row = i & 7, fp = (i >> 3) & 3, sl = i >> 5;
                    if (row >= R) continue;
                    const int n = (f0 + (m0 + sl) * G) * 8 + 2 * fp;               // feature index in [0, 3D)
                    float x0 = bfr(red_sum(sl, row, 2 * fp)), x1 = bfr(red_sum(sl, row, 2 * fp + 1));
                    const int sec = n / D, nn = n - sec * D, head = nn / hd, d = nn - head * hd;
                    if (sec < 2) {
                        const float2 cs = *reinterpret_cast<const float2*>(a.freqs + ((size_t)qpos * (hd / 2) + (d >> 1)) * 2);
                        const float y0 = __fsub_rn(__fmul_rn(x0, cs.x), __fmul_rn(x1, cs.y));
                        const float y1 = __fadd_rn(__fmul_rn(x1, cs.x), __fmul_rn(x0, cs.y));
                        x0 = y0; x1 = y1;
                    }
                    const uint32_t pk = pack2(x0, x1);
                    if (sec == 0) {
                        *reinterpret_cast<uint32_t*>(a.q + (size_t)row * D + nn) = pk;
                    } else {
                        bf16* cache = (sec == 1 ? a.kcache : a.vcache) + (size_t)l * a.layer_elems;
                        *reinterpret_cast<uint32_t*>(cache + (((size_t)row * H + head) * a.maxS + qpos) * hd + d) = pk;
                    }
                }
            });
        }
        stamp(l, 2);
        grid_barrier();
        stamp(l, 3);
        // ------------------------------------------------------------------------------------------------ P2: attention
        {
            float* qs = misc;                       // [hd] query (fp32)
            float* sc = misc + 128;                 // [kt + 1] scores / probabilities
            float* opart = misc + 256;              // [kCT / hd][hd] partial outputs  (<= 256 floats)
            float* st = misc + 200;                 // [0] running max, [1] running sum, [2] correction of this tile
            uint8_t* newkv = reinterpret_cast<uint8_t*>(xs);          // the new K row then the new V row (hd bf16 each)
            const int nkg = kCT / hd;               // key groups of the P.V pass (4 at hd 64, 2 at hd 128)
            for (int u = cta; u < nunits; u += G) {
                const Unit x = make_unit(u, H, a.nsplit, qpos, kt);
                const size_t cbase = (size_t)l * a.layer_elems + ((size_t)(x.r * H + x.head) * a.maxS) * hd;
                if (tid < hd)
                    qs[tid] = __bfloat162float(__ushort_as_bfloat16(__ldcg(reinterpret_cast<const unsigned short*>(a.q) + (size_t)x.r * D + x.head * hd + tid)));
                if (x.has_new && tid < hd / 4) {    // 8-byte pieces of the two new rows
                    const uint2 kv = __ldcg(reinterpret_cast<const uint2*>(a.kcache + cbase + (size_t)qpos * hd) + tid);
                    const uint2 vv = __ldcg(reinterpret_cast<const uint2*>(a.vcache + cbase + (size_t)qpos * hd) + tid);
                    reinterpret_cast<uint2*>(newkv)[tid] = kv;
                    reinterpret_cast<uint2*>(newkv + hd * 2)[tid] = vv;
                }
                if (tid == 0) { st[0] = -INFINITY; st[1] = 0.f; }
                float oacc = 0.f;                   // output dim `tid` (threads < hd)
                cbar();
                const float* mrow = a.emb_mask ? a.emb_mask + (size_t)(x.r % a.B) * a.Tc : nullptr;
                const int nsteps = x.ntiles + (x.has_new ? 1 : 0);
                for (int stp = 0; stp < nsteps; ++stp) {
                    const bool is_new = stp == x.ntiles;
                    const uint8_t *kp, *vp;
                    int nk, jbase, s = 0;
                    if (is_new) {
                        kp = newkv; vp = newkv + hd * 2; nk = 1; jbase = qpos;
                    } else {
                        s = (int)(seq % (uint32_t)ns);
                        mbar_wait(&full[s], (seq / (uint32_t)ns) & 1u);
                        kp = ring + (size_t)s * kSlot; vp = kp + kHalf;
                        jbase = x.jb + stp * kt; nk = min(kt, x.oe - jbase);
                    }
                    // (1) scores: 4 lanes per key, each hd/4 dims
                    {
                        const int kk = tid >> 2, part = tid & 3, dl = hd / 4;
                        float dot = 0.f;
                        if (kk < nk) {
                            const uint4* kr = reinterpret_cast<const uint4*>(kp + (size_t)kk * hd * 2 + (size_t)part * dl * 2);
                            const float* qq = qs + part * dl;
                            for (int i = 0; i < dl / 8; ++i) {
                                const uint4 v = kr[i];
                                const uint32_t w[4] = {v.x, v.y, v.z, v.w};
#pragma unroll
                                for (int e = 0; e < 4; ++e) {
                                    dot = fmaf(lo_f(w[e]), qq[i * 8 + 2 * e], dot);
                                    dot = fmaf(hi_f(w[e]), qq[i * 8 + 2 * e + 1], dot);
                                }
                            }
                        }
                        dot += __shfl_xor_sync(0xffffffffu, dot, 1);
                        dot += __shfl_xor_sync(0xffffffffu, dot, 2);
                        if (part == 0 && kk <= kt) {
                            const int j = jbase + kk;
                            bool vis = kk < nk;
                            if (vis && mrow && j < a.Tc && j != qpos) vis = mrow[j] != 0.f;       // generate.py:154-163
                            sc[kk] = vis ? dot * a.scale : -INFINITY;
                        }
                    }
                    cbar();
                    // (2) online softmax bookkeeping by warp 0
                    if (warp == 0) {
                        float mx = -INFINITY;
                        for (int j = lane; j < nk; j += 32) mx = fmaxf(mx, sc[j]);
                        mx = warp_max(mx);
                        const float mo = st[0], mn = fmaxf(mo, mx);
                        float ls = 0.f;
                        for (int j = lane; j < nk; j += 32) {
                            const float p = mn == -INFINITY ? 0.f : __expf(sc[j] - mn);
                            sc[j] = p;
                            ls += p;
                        }
                        ls = warp_sum(ls);
                        if (lane == 0) {
                            const float corr = mn == -INFINITY ? 1.f : __expf(mo - mn);
                            st[0] = mn; st[1] = st[1] * corr + ls; st[2] = corr;
                        }
                    }
                    cbar();
                    // (3) P.V: thread -> (key group, dim)
                    {
                        const int d = tid % hd, kg = tid / hd;
                        float acc = 0.f;
                        if (kg < nkg)
                            for (int j = kg; j < nk; j += nkg)
                                acc = fmaf(sc[j], __bfloat162float(reinterpret_cast<const bf16*>(vp)[(size_t)j * hd + d]), acc);
                        if (kg < nkg) opart[kg * hd + d] = acc;
                    }
                    cbar();
                    if (tid < hd) {
                        float sum = 0.f;
                        for (int kg = 0; kg < nkg; ++kg) sum += opart[kg * hd + tid];
                        oacc = oacc * st[2] + sum;
                    }
                    if (!is_new) {
                        __syncwarp();
                        if (lane == 0) mbar_arrive(&empty[s]);
                        ++seq;
                    }
                    cbar();
                }
                float* pu = a.part + (size_t)u * (hd + 2);
                if (tid < hd) pu[tid] = oacc;
                if (tid == 0) { pu[hd] = st[0]; pu[hd + 1] = st[1]; }
                cbar();
            }
        }
        stamp(l, 4);
        grid_barrier();
        stamp(l, 5);
        // ------------------------------------------------------------------------------------------------ P3: wo + residual
        {
            const Gemm gm{ly.wo, nullptr, D, D, phase_rot(l, 2, G)};
            // xs <- merged attention output (bf16 [R][D]): combine the nsplit partials of every (row, head)
            {
                const int stride = D * 2 + 16;
                for (int i = tid; i < R * D / 2; i += kCT) {
                    const int r = (2 * i) / D, n = 2 * i - r * D, head = n / hd, d = n - head * hd;
                    const float* p0 = a.part + (size_t)((r * H + head) * a.nsplit) * (hd + 2);
                    float M = -INFINITY;
                    for (int s = 0; s < a.nsplit; ++s) M = fmaxf(M, __ldcg(p0 + (size_t)s * (hd + 2) + hd));
                    float Lw = 0.f, o0 = 0.f, o1 = 0.f;
                    for (int s = 0; s < a.nsplit; ++s) {
                        const float* ps = p0 + (size_t)s * (hd + 2);
                        const float ms = __ldcg(ps + hd);
                        const float w = ms == -INFINITY ? 0.f : __expf(ms - M);
                        Lw += __ldcg(ps + hd + 1) * w;
                        const float2 ov = __ldcg(reinterpret_cast<const float2*>(ps + d));
                        o0 += ov.x * w; o1 += ov.y * w;
                    }
                    *reinterpret_cast<uint32_t*>(xs + (size_t)r * stride + (size_t)n * 2) = pack2(o0 / Lw, o1 / Lw);
                }
                cbar();
            }
            stamp(l, 6);
            const int f0 = first_group(gm, cta, G);
            run_gemm(gm, [&](int m0, int nb) {
                for (int i = tid; i < nb * 4 * 8; i += kCT) {
                    const int row = i & 7, fp = (i >> 3) & 3, sl = i >> 5;
                    if (row >= R) continue;
                    const int n = (f0 + (m0 + sl) * G) * 8 + 2 * fp;
                    const uint32_t ho = __ldcg(reinterpret_cast<const uint32_t*>(h_row(l, row) + n));
                    // h = x + f(x), both bf16 tensors (gpt.py:255)
                    *reinterpret_cast<uint32_t*>(a.h + (size_t)row * D + n) =
                        pack2(lo_f(ho) + bfr(red_sum(sl, row, 2 * fp)), hi_f(ho) + bfr(red_sum(sl, row, 2 * fp + 1)));
                }
            });
        }
        stamp(l, 7);
        grid_barrier();
        stamp(l, 8);
        // ------------------------------------------------------------------------------------------------ P4: w1 | w3 + SwiGLU
        {
            const Gemm gm{ly.w1, ly.w3, F, D, phase_rot(l, 3, G)};
            stage_rows([&](int r) { return (const bf16*)(a.h + (size_t)r * D); }, D, ly.ffn_norm);
            stamp(l, 9);
            const int f0 = first_group(gm, cta, G);
            run_gemm(gm, [&](int m0, int nb) {
                for (int i = tid; i < nb * 4 * 8; i += kCT) {
                    const int row = i & 7, fp = (i >> 3) & 3, sl = i >> 5;
                    if (row >= R) continue;
                    const int n = (f0 + (m0 + sl) * G) * 8 + 2 * fp;
                    float o[2];
#pragma unroll
                    for (int e = 0; e < 2; ++e) {           // silu(w1 x) * (w3 x) in bf16 tensors (gpt.py:167)
                        const float av = bfr(red_sum(2 * sl, row, 2 * fp + e)), bv = bfr(red_sum(2 * sl + 1, row, 2 * fp + e));
                        o[e] = bfr(av / (1.0f + expf(-av))) * bv;
                    }
                    *reinterpret_cast<uint32_t*>(a.ff + (size_t)row * F + n) = pack2(o[0], o[1]);
                }
            });
        }
        stamp(l, 10);
        grid_barrier();
        stamp(l, 11);
        // ------------------------------------------------------------------------------------------------ P5: w2 + residual
        {
            const Gemm gm{ly.w2, nullptr, D, F, phase_rot(l, 4, G)};
            stage_rows([&](int r) { return (const bf16*)(a.ff + (size_t)r * F); }, F, nullptr);
            stamp(l, 12);
            const int f0 = first_group(gm, cta, G);
            run_gemm(gm, [&](int m0, int nb) {
                for (int i = tid; i < nb * 4 * 8; i += kCT) {
                    const int row = i & 7, fp = (i >> 3) & 3, sl = i >> 5;
                    if (row >= R) continue;
                    const int n = (f0 + (m0 + sl) * G) * 8 + 2 * fp;
                    const uint32_t ho = __ldcg(reinterpret_cast<const uint32_t*>(a.h + (size_t)row * D + n));
                    *reinterpret_cast<uint32_t*>(a.h + (size_t)row * D + n) =       // gpt.py:256
                        pack2(lo_f(ho) + bfr(red_sum(sl, row, 2 * fp)), hi_f(ho) + bfr(red_sum(sl, row, 2 * fp + 1)));
                }
            });
        }
        stamp(l, 13);
        grid_barrier();
        stamp(l, 14);
    }
    // ---------------------------------------------------------------------------------------------------- PH: final norm + head
    {
        const Gemm gm{a.output, nullptr, a.V, D, phase_rot(a.L, 0, G)};
        stamp(a.L, 0);
        stage_rows([&](int r) { return (const bf16*)(a.h + (size_t)r * D); }, D, a.final_norm);
        stamp(a.L, 1);
        const int f0 = first_group(gm, cta, G);
        run_gemm(gm, [&](int m0, int nb) {
            for (int i = tid; i < nb * 4 * 8; i += kCT) {
                const int row = i & 7, fp = (i >> 3) & 3, sl = i >> 5;
                if (row >= R) continue;
                const int n = (f0 + (m0 + sl) * G) * 8 + 2 * fp;
                *reinterpret_cast<float2*>(a.logits + (size_t)row * a.V + n) = make_float2(red_sum(sl, row, 2 * fp), red_sum(sl, row, 2 * fp + 1));
            }
        });
    }
    stamp(a.L, 2);
    // leave both counters at zero for the next launch: the last CTA to get here resets them (every CTA has passed all barriers)
    if (tid == 0) {
        __threadfence();
        const unsigned int old = atomicAdd(a.bar + 1, 1u);
        if (old == (unsigned)G - 1u) {
            a.bar[0] = 0u;
            a.bar[1] = 0u;
            __threadfence();
        }
    }
}

}  // namespace

bool decode_persist_supported(int R, int D, int F, int V, int H, int hd, int dtype) {
    if (dtype != LG_DTYPE_BF16 || R < 1 || R > 8) return false;
    if (hd != 64 && hd != 128) return false;                  // 16-byte aligned cache rows, hd/4 a multiple of 8
    if (D % 64 || F % 64 || V % 8 || (3 * D) % 8) return false;
    if (D != H * hd) return false;
    const size_t xs = (size_t)R * (std::max(D, F) * 2 + 16);
    return xs <= 96 * 1024;
}

static unsigned long long* g_pd_trace = nullptr;
extern "C" void lg_debug_set_pd_trace(unsigned long long* dev_buf) { g_pd_trace = dev_buf; }

static int pd_sm_count() {
    static int sms[32] = {0};
    int dev = 0;
    cudaGetDevice(&dev);
    if (!sms[dev & 31]) cudaDeviceGetAttribute(&sms[dev & 31], cudaDevAttrMultiProcessorCount, dev);
    return sms[dev & 31] > 0 ? sms[dev & 31] : 132;
}
static int pd_nsplit(int R, int H) {
    const int forced = lg_env_flag("LG_PD_NSPLIT", 0);            // test hook: force the number of context slices (1..8)
    if (forced >= 1 && forced <= 8) return forced;
    return std::max(1, std::min(8, pd_sm_count() / std::max(1, R * H)));
}
size_t decode_persist_part_floats(int R, int H, int hd) { return (size_t)R * H * pd_nsplit(R, H) * (hd + 2); }

int launch_decode_persist(const PdLaunch& p, cudaStream_t st) {
    LG_REQUIRE(decode_persist_supported(p.R, p.D, p.F, p.V, p.H, p.hd, LG_DTYPE_BF16), "decode_persist: unsupported shape");
    static DevOnce once;
    if (lg_first_on_device(once)) {
        LG_CUDA_OK(cudaFuncSetAttribute(decode_small_persistent_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, 227 * 1024));
    }
    const int G = pd_sm_count();
    PdArgs a{};
    a.L = p.L; a.D = p.D; a.F = p.F; a.V = p.V; a.H = p.H; a.hd = p.hd; a.R = p.R; a.B = p.B; a.Tc = p.Tc; a.maxS = p.maxS;
    a.eps = p.eps; a.scale = p.scale;
    a.layers = p.layers; a.final_norm = (const bf16*)p.final_norm; a.output = (const bf16*)p.output; a.tok_emb = (const bf16*)p.tok_emb;
    a.freqs = p.freqs; a.kcache = (bf16*)p.kcache; a.vcache = (bf16*)p.vcache; a.layer_elems = p.layer_elems;
    a.h = (bf16*)p.h; a.q = (bf16*)p.q; a.ff = (bf16*)p.ff; a.part = p.part; a.logits = p.logits;
    a.tokens = p.tokens; a.pos_dev = p.pos_dev; a.pos_value = p.pos_value; a.emb_mask = p.emb_mask; a.bar = p.bar;
    // attention split: as many (row, head, context-slice) units as there are CTAs, at most 8 slices
    a.nsplit = pd_nsplit(p.R, p.H);
    a.trace = g_pd_trace;
    LG_REQUIRE((size_t)p.R * p.H * a.nsplit * (p.hd + 2) <= p.part_floats, "decode_persist: attention partial buffer too small");
    a.xs_bytes = (int)(((size_t)p.R * (std::max(p.D, p.F) * 2 + 16) + 127) / 128 * 128);
    const size_t fixed = 2 * kMaxSlots * sizeof(uint64_t) + (size_t)a.xs_bytes + (size_t)(kCW * kGB * 64 + 512) * sizeof(float);
    a.nslots = (int)std::min<size_t>(kMaxSlots, (227 * 1024 - fixed) / kSlot);
    LG_REQUIRE(a.nslots >= 3, "decode_persist: not enough shared memory for the tile ring (%d slots)", a.nslots);
    const size_t smem = (size_t)a.nslots * kSlot + fixed;
    cudaLaunchConfig_t cfg = {};
    cfg.gridDim = dim3(G); cfg.blockDim = dim3(kThreadsPd); cfg.dynamicSmemBytes = smem; cfg.stream = st;
    cudaLaunchAttribute at[1];
    at[0].id = cudaLaunchAttributeCooperative;       // all CTAs co-resident (the grid barrier needs it), also inside a captured graph
    at[0].val.cooperative = lg_env_flag("LG_PD_COOP", 1) ? 1 : 0;
    cfg.attrs = at; cfg.numAttrs = 1;
    LG_CUDA_OK(cudaLaunchKernelEx(&cfg, decode_small_persistent_kernel, a));
    LG_LAUNCH_CHECK();
    return 0;
}
