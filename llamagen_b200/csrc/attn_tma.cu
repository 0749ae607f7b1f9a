// Decode attention (one query per sequence row) for bf16 or fp16 KV caches: the K and V prefixes of one (row, head)
// are contiguous [c, hd] streams in HBM, so they are pulled by TMA (cp.async.bulk.tensor, 128-byte swizzle)
// through a 3-stage mbarrier ring — no registers are spent on loads in flight — and the two tiny matrix
// products (q.K^T and P.V, M = 1 query padded to the m16 MMA shape) run on the tensor cores with ldmatrix
// operands; softmax stays fp32 in registers (FlashAttention-2 style register reuse of P).
//
// Replaces, for Tq == 1, gpt.py:229-236 (repeat_interleave copies + masked SDPA over all max_seq slots):
// only the valid prefix [0, pos] is read. Mask rule: generate.py:154-163 (emb_masks on the condition keys).
#include "kernels.cuh"
#include "tma_utils.cuh"

namespace {

using namespace tma;

constexpr int kKC = 32;           // keys per stage: 32 keys / 2 warps per CTA leave shared memory for the other chain's GEMM CTAs
constexpr int kStagesA = 2;       // 2 stages of K+V per CTA; contexts here are <= 1144 keys
constexpr int kWarps = kKC / 16;  // each warp owns 16 keys of a stage
constexpr int kDeepStages = 8;    // few-item (batch-1) variant: a whole context of up to 256 keys is requested before the dependency wait
constexpr int kCtasPerSm64 = 12;  // launch bound of the sequential hd-64 kernels (5 for hd 128)

__device__ __forceinline__ void ldsm_x4(uint32_t addr, uint32_t& r0, uint32_t& r1, uint32_t& r2, uint32_t& r3) {
    asm volatile("ldmatrix.sync.aligned.m8n8.x4.shared.b16 {%0,%1,%2,%3}, [%4];\n"
                 : "=r"(r0), "=r"(r1), "=r"(r2), "=r"(r3) : "r"(addr));
}
__device__ __forceinline__ void ldsm_x4_t(uint32_t addr, uint32_t& r0, uint32_t& r1, uint32_t& r2, uint32_t& r3) {
    asm volatile("ldmatrix.sync.aligned.m8n8.x4.trans.shared.b16 {%0,%1,%2,%3}, [%4];\n"
                 : "=r"(r0), "=r"(r1), "=r"(r2), "=r"(r3) : "r"(addr));
}
// T = bf16 or f16: the operand type of the MMA and the storage type of q, the KV cache and the output
template <typename T = bf16>
__device__ __forceinline__ void mma16816(float* c, uint32_t a0, uint32_t a1, uint32_t a2, uint32_t a3, uint32_t b0, uint32_t b1) {
    mma_m16n8k16<T>(c, a0, a1, a2, a3, b0, b1);
}
__device__ __forceinline__ uint32_t swz(int r, int c) { return (uint32_t)(r * 128 + ((c ^ (r & 7)) << 4)); }
template <typename T = bf16>
__device__ __forceinline__ uint32_t pack16(float a, float b) { return ElemTraits<T>::pack2(a, b); }
// fp8 tiles: byte offset of 16-byte chunk c of row r. 64-byte rows (hd 64) come in with the 64-byte swizzle (address bits 4-5 ^= 7-8),
// 128-byte rows (hd 128, 100-in-112) with the 128-byte swizzle (bits 4-6 ^= 7-9).
template <int RB>
__device__ __forceinline__ uint32_t swz8(int r, int c) {
    return RB == 64 ? (uint32_t)(r * 64 + ((c ^ ((r >> 1) & 3)) << 4)) : (uint32_t)(r * 128 + ((c ^ (r & 7)) << 4));
}
// fp8 q.K^T: a lane reads whole 16-byte chunks of its key row, so the head dims are visited in a permuted order that q follows too.
// Chunk of lane quad index tg in 64-dim block j (16 dims = 4 k16 steps of 4 dims: 2 for b0, 2 for b1); 128-byte rows interleave the
// chunks of the two blocks so that the two rows of a quarter warp fall on distinct banks.
template <int HD>
__device__ __forceinline__ int f8_kchunk(int tg, int j) { return HD == 64 ? tg : 2 * tg + j; }
// first head dim of the q pairs that k16 step kk of lane quad index tg multiplies (a0 = dims d, d + 1; a2 = dims d + 2, d + 3)
template <int HD>
__device__ __forceinline__ int f8_qdim(int tg, int kk) { return f8_kchunk<HD>(tg, kk / 4) * 16 + (kk % 4) * 4; }

struct AttnTmaArgs {   // the 16-bit tensors are bf16 or fp16 (the kernel's T); declared bf16 for their 2-byte element arithmetic
    const bf16* q;     // [R, D] (unfused path)
    bf16* out;         // [R, D]
    int R, H, maxS;
    const int* pos_dev; int pos_value;
    const int* pos_rows;         // per-row positions [R] or null (continuous batching)
    long long row_base;          // first cache row of this layer inside the tensor maps
    const float* emb_mask; int B, Tc;
    const float* emb_mask_uncond;   // the mask rows r >= B read, or null (attn_mask_row)
    float scale;
    // fused QKV epilogue (FUSED kernels): split-K slabs of the QKV GEMM, RoPE table, this layer's cache bases
    const float* partial; int ksplit;
    const float* freqs;
    bf16* kcache; bf16* vcache;
    unsigned long long kvhint;   // L2 eviction hint of the K/V stream (0: default policy)
    int hd;                      // real head dim (<= HD): GPT-3B's hd = 100 runs the HD = 128 kernel over zero-padded tiles
    int hdp;                     // elements between consecutive cache rows (112 for hd = 100: the tensor map zero-fills 112..127)
};
// fp8 cache (F8 kernels; a separate last argument, so the argument layout of the other kernels that take AttnTmaArgs stays put):
// kcache / vcache hold e4m3 codes, AttnTmaArgs::scale includes the K scale, the output is multiplied by v_scale, the writer stores
// e4m3(k * k_inv) and e4m3(v * v_inv)
struct KvScales {
    float k_inv, v_inv, v_scale;
};

// FUSED = true: the kernel also IS the QKV epilogue of gpt.py:214-230 for its (row, head): it reduces the split-K
// slabs of the QKV GEMM for its 3*hd columns, applies RoPE to q and k, writes the new K/V row into the cache
// (for future steps) and attends to it straight from shared memory. Every TMA load then only touches rows written
// in EARLIER steps, so the whole KV stream is requested before the programmatic-dependency wait and overlaps the
// QKV GEMM; one dependent kernel per layer disappears.
//
// F8 = true: fp8 e4m3 cache. A stage holds [kKC keys][hdp bytes] boxes (64-byte rows for hd 64, 128-byte rows otherwise), and the
// B operands are decoded from shared memory in registers instead of ldmatrix: for q.K^T a lane's B fragment is 4 consecutive bytes
// of its key row (the head dims are permuted consistently in q), for P.V a lane gathers one 4-byte word from each of its 4 key rows
// and transposes bytes with prmt (the output dims come out permuted and are put back in the merge). The fused writer stores
// e4m3(x * inv) and the step attends to those codes too; the K scale is in a.scale and the V scale multiplies O / L.
template <typename T, int HD, bool FUSED, int NST, bool PAR_ = (NST > 2), bool F8 = false>
__global__ void __launch_bounds__(kWarps * 32 * (PAR_ ? NST : 1), PAR_ ? 1 : (HD == 64 ? (NST > 2 ? 4 : kCtasPerSm64) : 5)) attn_tma_kernel(const __grid_constant__ CUtensorMap kmap,
                                                               const __grid_constant__ CUtensorMap vmap,
                                                               const __grid_constant__ CUtensorMap kmap16,
                                                               const __grid_constant__ CUtensorMap vmap16, AttnTmaArgs a,
                                                               KvScales f8s) {
    constexpr int RB = F8 ? (HD == 64 ? 64 : 128) : 128;   // bytes per tile row of one box
    constexpr int NSUB = F8 ? 1 : HD / 64;        // 128-byte-wide sub-tiles per row (fp8: one box covers the whole row)
    constexpr int SUB_BYTES = kKC * RB;           // one [kKC keys][64 dims] bf16 sub-tile
    constexpr int TILE_BYTES = NSUB * SUB_BYTES;  // K (or V) of one stage
    // NST > 2 (few work items, batch-1 latency path): one warp group per ring stage, so the chunks of a context are processed
    // concurrently instead of one after the other; a stage is private to its group (named barrier, no CTA-wide sync per chunk)
    constexpr bool PAR = PAR_;
    constexpr int NW = PAR ? NST * kWarps : kWarps;
    constexpr int NSLOT = NW + (FUSED ? 1 : 0);
    extern __shared__ __align__(1024) uint8_t smem_raw[];
    uint8_t* tiles = reinterpret_cast<uint8_t*>(((uintptr_t)smem_raw + 1023) & ~(uintptr_t)1023);
    uint64_t* full_bar = reinterpret_cast<uint64_t*>(tiles + NST * 2 * TILE_BYTES);
    float* merge = reinterpret_cast<float*>(full_bar + NST);            // [NSLOT][HD + 2]
    T* qbuf = reinterpret_cast<T*>(merge + NSLOT * (HD + 2));                  // [3][HD]: q, k_new, v_new (FUSED)

    const int h = blockIdx.x, r = blockIdx.y;
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31, g = lane >> 2, tg = lane & 3;
    const int grp = PAR ? warp / kWarps : 0, wk = PAR ? warp % kWarps : warp;   // ring stage owned / 16-key slice inside a chunk
    const long long row0 = a.row_base + ((long long)r * a.H + h) * a.maxS;
    const int hdr = a.hd;                      // real head dim; q / slabs / out are [.., H * hdr]
    const int D = a.H * hdr;

    if (threadIdx.x == 0) {
        prefetch_map(&kmap);
        prefetch_map(&vmap);
        prefetch_map(&kmap16);
        prefetch_map(&vmap16);
        for (int s = 0; s < NST; ++s) mbar_init(&full_bar[s], 1);
        fence_barrier_init();
    }
    __syncthreads();
    // Read before the dependency wait: the position (counter or per-row array) and every key row of EARLIER steps. Precondition:
    // each must be complete when the predecessor (the QKV GEMM, which lets this kernel start before its own wait) STARTS. The
    // engine guarantees it by launching an eager decode step's first kernel without PDL, after the sample kernel or set_counters
    // that wrote the counter has completed; graph replay orders the step the same way (DESIGN §4, "Reads before the dependency wait").
    const int qpos = a.pos_rows ? a.pos_rows[r] : (a.pos_dev ? *a.pos_dev : 0) + a.pos_value;
    const int nkeys = FUSED ? qpos : qpos + 1;      // keys streamed from the cache (FUSED: the new key stays on chip)
    const int nchunks = (nkeys + kKC - 1) / kKC;

    auto issue = [&](int ci) {
        const int s = ci % NST;
        uint8_t* kt = tiles + s * 2 * TILE_BYTES;
        uint8_t* vt = kt + TILE_BYTES;
        const int row = (int)(row0 + (long long)ci * kKC);
        const int valid = nkeys - ci * kKC;            // keys of this chunk that exist
        if (valid >= kKC) {
            mbar_expect_tx(&full_bar[s], 2 * TILE_BYTES);
#pragma unroll
            for (int sub = 0; sub < NSUB; ++sub) {
                load_2d_hint(kt + sub * SUB_BYTES, &kmap, &full_bar[s], sub * 64, row, a.kvhint);
                load_2d_hint(vt + sub * SUB_BYTES, &vmap, &full_bar[s], sub * 64, row, a.kvhint);
            }
        } else {
            // tail chunk: 16-row boxes (one per warp's key group) so at most 15 rows beyond the context are read;
            // groups that are not loaded are never touched by the MMA loop (it skips j0 >= nkeys).
            const int n16 = (valid + 15) / 16;
            mbar_expect_tx(&full_bar[s], (uint32_t)(n16 * 2 * NSUB * 16 * RB));
            for (int i = 0; i < n16; ++i) {
#pragma unroll
                for (int sub = 0; sub < NSUB; ++sub) {
                    load_2d_hint(kt + sub * SUB_BYTES + i * 16 * RB, &kmap16, &full_bar[s], sub * 64, row + 16 * i, a.kvhint);
                    load_2d_hint(vt + sub * SUB_BYTES + i * 16 * RB, &vmap16, &full_bar[s], sub * 64, row + 16 * i, a.kvhint);
                }
            }
        }
    };
    const int npro = min(NST, nchunks);
    if (threadIdx.x == 0)
        for (int ci = 0; ci < npro; ++ci)
            if (FUSED || ci != nchunks - 1) issue(ci);
    // RoPE angles of this step's position: a table lookup that does not depend on the producer kernel -> issued before the wait
    float4 cs_pre = make_float4(1.f, 0.f, 1.f, 0.f);
    if (FUSED && threadIdx.x < 2 * HD / 4) {
        const int e = (threadIdx.x % (HD / 4)) * 4;
        if (e < hdr) cs_pre = __ldg(reinterpret_cast<const float4*>(a.freqs + ((size_t)qpos * (hdr / 2) + (e >> 1)) * 2));
    }
    lg_pdl_sync();
    if (!FUSED && threadIdx.x == 0 && nchunks - 1 < npro && nchunks > 0) issue(nchunks - 1);

    uint32_t qa[HD / 16][2];
    if (FUSED) {
        // ---- QKV epilogue for this (row, head): slab reduce -> dtype rounding -> RoPE -> cache write / smem
        for (int it = threadIdx.x; it < 3 * HD / 4; it += blockDim.x) {     // 48 / 96 items; a CTA may have only 64 threads (32-key stages)
            const int sec = it / (HD / 4), e = (it % (HD / 4)) * 4;
            const bool live = e < hdr;                 // dims [hdr, HD) are zero padding (hdr % 4 == 0)
            const size_t N3 = (size_t)3 * D, slab = (size_t)a.R * N3;
            const float* p = a.partial + (size_t)r * N3 + (size_t)sec * D + (size_t)h * hdr + e;
            float4 sv = make_float4(0.f, 0.f, 0.f, 0.f);
            if (live) {
                sv = *reinterpret_cast<const float4*>(p);
                for (int k = 1; k < a.ksplit; ++k) {
                    const float4 t = *reinterpret_cast<const float4*>(p + (size_t)k * slab);
                    sv.x += t.x; sv.y += t.y; sv.z += t.z; sv.w += t.w;
                }
            }
            float x0 = ElemTraits<T>::round(sv.x), x1 = ElemTraits<T>::round(sv.y), x2 = ElemTraits<T>::round(sv.z),
                  x3 = ElemTraits<T>::round(sv.w);
            if (sec < 2 && live) {   // apply_rotary_emb (gpt.py:420-430): adjacent pairs, fp32, separate roundings
                // first pass: the angles were fetched before the dependency wait; a second pass (HD = 128 on 64 threads) loads its own
                const float4 cs = it == (int)threadIdx.x ? cs_pre
                                                         : __ldg(reinterpret_cast<const float4*>(a.freqs + ((size_t)qpos * (hdr / 2) + (e >> 1)) * 2));
                const float y0 = __fsub_rn(__fmul_rn(x0, cs.x), __fmul_rn(x1, cs.y));
                const float y1 = __fadd_rn(__fmul_rn(x1, cs.x), __fmul_rn(x0, cs.y));
                const float y2 = __fsub_rn(__fmul_rn(x2, cs.z), __fmul_rn(x3, cs.w));
                const float y3 = __fadd_rn(__fmul_rn(x3, cs.z), __fmul_rn(x2, cs.w));
                x0 = y0; x1 = y1; x2 = y2; x3 = y3;
            }
            uint2 pk;
            if constexpr (F8) {
                if (sec > 0) {
                    // the cache gets e4m3(T(x) * inv); qbuf keeps the decoded codes, so the new key and value are attended to as stored
                    const float inv = sec == 1 ? f8s.k_inv : f8s.v_inv;
                    const uint32_t c01 = e4m3x2_pack(ElemTraits<T>::round(x0) * inv, ElemTraits<T>::round(x1) * inv);
                    const uint32_t c23 = e4m3x2_pack(ElemTraits<T>::round(x2) * inv, ElemTraits<T>::round(x3) * inv);
                    pk.x = e4m3x2_to<T>(c01);
                    pk.y = e4m3x2_to<T>(c23);
                    if (live)
                        *reinterpret_cast<uint32_t*>(reinterpret_cast<uint8_t*>(sec == 1 ? a.kcache : a.vcache) +
                                                     (((size_t)r * a.H + h) * a.maxS + qpos) * a.hdp + e) = c01 | (c23 << 16);
                } else {
                    pk.x = pack16<T>(x0, x1);
                    pk.y = pack16<T>(x2, x3);
                }
                *reinterpret_cast<uint2*>(qbuf + sec * HD + e) = pk;
            } else {
                pk.x = pack16<T>(x0, x1);
                pk.y = pack16<T>(x2, x3);
                *reinterpret_cast<uint2*>(qbuf + sec * HD + e) = pk;
                if (sec > 0 && live) {
                    bf16* cache = sec == 1 ? a.kcache : a.vcache;
                    *reinterpret_cast<uint2*>(cache + (((size_t)r * a.H + h) * a.maxS + qpos) * a.hdp + e) = pk;
                }
            }
        }
        __syncthreads();
#pragma unroll
        for (int kk = 0; kk < HD / 16; ++kk) {
            qa[kk][0] = 0; qa[kk][1] = 0;
            if (g == 0) {
                if constexpr (F8) {
                    const int d = f8_qdim<HD>(tg, kk);
                    qa[kk][0] = *reinterpret_cast<const uint32_t*>(qbuf + d);
                    qa[kk][1] = *reinterpret_cast<const uint32_t*>(qbuf + d + 2);
                } else {
                    qa[kk][0] = *reinterpret_cast<const uint32_t*>(qbuf + kk * 16 + tg * 2);
                    qa[kk][1] = *reinterpret_cast<const uint32_t*>(qbuf + kk * 16 + 8 + tg * 2);
                }
            }
        }
    } else {
        // q as the A operand of m16n8k16: only MMA row 0 (lanes with g == 0) is real, the other 15 rows are zero
        const bf16* qp = a.q + (size_t)r * D + (size_t)h * hdr;
#pragma unroll
        for (int kk = 0; kk < HD / 16; ++kk) {
            qa[kk][0] = 0; qa[kk][1] = 0;
            if (g == 0) {
                if constexpr (F8) {
                    const int d = f8_qdim<HD>(tg, kk);   // hdr % 4 == 0: the 4 dims are all real or all padding
                    if (d < hdr) {
                        qa[kk][0] = *reinterpret_cast<const uint32_t*>(qp + d);
                        qa[kk][1] = *reinterpret_cast<const uint32_t*>(qp + d + 2);
                    }
                } else {
                    if (kk * 16 + tg * 2 < hdr) qa[kk][0] = *reinterpret_cast<const uint32_t*>(qp + kk * 16 + tg * 2);
                    if (kk * 16 + 8 + tg * 2 < hdr) qa[kk][1] = *reinterpret_cast<const uint32_t*>(qp + kk * 16 + 8 + tg * 2);
                }
            }
        }
    }
    const float* mrow = attn_mask_row(a, r);

    float o[HD / 8][4];
#pragma unroll
    for (int i = 0; i < HD / 8; ++i) { o[i][0] = 0.f; o[i][1] = 0.f; o[i][2] = 0.f; o[i][3] = 0.f; }
    float mx = -INFINITY, l = 0.f;

    for (int ci = grp; ci < nchunks; ci += PAR ? NST : 1) {
        const int s = ci % NST;
        mbar_wait(&full_bar[s], (uint32_t)((ci / NST) & 1));
        const uint32_t kt = smem_u32(tiles + s * 2 * TILE_BYTES);
        const uint32_t vt = kt + TILE_BYTES;
        const int j0 = ci * kKC + wk * 16;            // this warp's 16 keys
        if (j0 < nkeys) {                              // warp-uniform
            // ---- S = q K^T for 16 keys (two n8 tiles)
            float sc[2][4] = {{0.f, 0.f, 0.f, 0.f}, {0.f, 0.f, 0.f, 0.f}};
            if constexpr (F8) {
                const uint8_t* ktp = tiles + s * 2 * TILE_BYTES;
#pragma unroll
                for (int j = 0; j < HD / 64; ++j) {
                    uint4 kw[2];                            // 16 dims of key g of each n8 tile
#pragma unroll
                    for (int nt = 0; nt < 2; ++nt)
                        kw[nt] = *reinterpret_cast<const uint4*>(ktp + swz8<RB>(wk * 16 + nt * 8 + g, f8_kchunk<HD>(tg, j)));
#pragma unroll
                    for (int i = 0; i < 4; ++i) {
                        const int kk = j * 4 + i;
#pragma unroll
                        for (int nt = 0; nt < 2; ++nt) {
                            const uint32_t w = i == 0 ? kw[nt].x : i == 1 ? kw[nt].y : i == 2 ? kw[nt].z : kw[nt].w;
                            mma16816<T>(sc[nt], qa[kk][0], 0u, qa[kk][1], 0u, e4m3x2_to<T>(w), e4m3x2_to<T>(w >> 16));
                        }
                    }
                }
            } else {
#pragma unroll
                for (int kk = 0; kk < HD / 16; ++kk) {
                    uint32_t b0, b1, b2, b3;
                    const int row = wk * 16 + (lane & 7) + ((lane >> 4) << 3);
                    const int chunk = (kk * 2 + ((lane >> 3) & 1)) & 7;
                    ldsm_x4(kt + (kk / 4) * SUB_BYTES + swz(row, chunk), b0, b1, b2, b3);
                    mma16816<T>(sc[0], qa[kk][0], 0u, qa[kk][1], 0u, b0, b1);
                    mma16816<T>(sc[1], qa[kk][0], 0u, qa[kk][1], 0u, b2, b3);
                }
            }
            // ---- online softmax on MMA row 0 (held by the quad g == 0; other quads carry zero rows)
            float pv[4];
            float lmax = -INFINITY;
#pragma unroll
            for (int i = 0; i < 4; ++i) {
                const int j = j0 + (i >> 1) * 8 + tg * 2 + (i & 1);
                bool vis = j < nkeys;
                if (vis && mrow && j < a.Tc && j != qpos) vis = mrow[j] != 0.f;
                pv[i] = vis ? sc[i >> 1][i & 1] * a.scale : -INFINITY;
                lmax = fmaxf(lmax, pv[i]);
            }
            lmax = fmaxf(lmax, __shfl_xor_sync(0xffffffffu, lmax, 1));
            lmax = fmaxf(lmax, __shfl_xor_sync(0xffffffffu, lmax, 2));
            const float mn = fmaxf(mx, lmax);
            float corr = 1.f, lsum = 0.f;
            if (mn != -INFINITY) {
                corr = __expf(mx - mn);
#pragma unroll
                for (int i = 0; i < 4; ++i) { pv[i] = __expf(pv[i] - mn); lsum += pv[i]; }
            } else {
#pragma unroll
                for (int i = 0; i < 4; ++i) pv[i] = 0.f;
            }
            lsum += __shfl_xor_sync(0xffffffffu, lsum, 1);
            lsum += __shfl_xor_sync(0xffffffffu, lsum, 2);
            l = l * corr + lsum;
            mx = mn;
#pragma unroll
            for (int i = 0; i < HD / 8; ++i) { o[i][0] *= corr; o[i][1] *= corr; }
            // ---- O += P V : P (packed to T) is already in A-fragment layout (C layout of S == A layout of P)
            const uint32_t pa0 = pack16<T>(pv[0], pv[1]);   // keys tg*2, +1
            const uint32_t pa2 = pack16<T>(pv[2], pv[3]);   // keys 8 + tg*2, +1
            if constexpr (F8) {
                // B fragment of n8 tile t: V[keys 2tg, 2tg+1 | 2tg+8, 2tg+9][dim DPT*g + t]. The lane reads DPT bytes (dims DPT*g ..)
                // of each of its 4 key rows; odd tg take the two rows of a pair in swapped order so a half warp hits distinct banks.
                constexpr int DPT = HD / 8, NWD = DPT / 4;
                const uint8_t* vtp = tiles + s * 2 * TILE_BYTES + TILE_BYTES;
                const int sw = tg & 1, rb = wk * 16 + 2 * tg;
                uint32_t w[4][NWD];                         // rows rb + sw, rb + 1 - sw, rb + 8 + sw, rb + 9 - sw
#pragma unroll
                for (int q = 0; q < 4; ++q) {
                    const int row = rb + (q >> 1) * 8 + ((q & 1) ^ sw);
                    if constexpr (RB == 64) {
                        const uint2 u = *reinterpret_cast<const uint2*>(vtp + swz8<RB>(row, g >> 1) + (g & 1) * 8);
                        w[q][0] = u.x; w[q][NWD - 1] = u.y;
                    } else {
                        const uint4 u = *reinterpret_cast<const uint4*>(vtp + swz8<RB>(row, g));
                        w[q][0] = u.x; w[q][1 % NWD] = u.y; w[q][2 % NWD] = u.z; w[q][3 % NWD] = u.w;
                    }
                }
                // prmt: interleave the bytes of (key 2tg, key 2tg + 1) -> e4m3x2 pairs of dims 0|1 (lo) and 2|3 (hi) of a word
                const uint32_t sel_lo = sw ? 0x1504u : 0x5140u, sel_hi = sw ? 0x3726u : 0x7362u;
#pragma unroll
                for (int wd = 0; wd < NWD; ++wd) {
                    const uint32_t x01 = __byte_perm(w[0][wd], w[1][wd], sel_lo), x23 = __byte_perm(w[0][wd], w[1][wd], sel_hi);
                    const uint32_t y01 = __byte_perm(w[2][wd], w[3][wd], sel_lo), y23 = __byte_perm(w[2][wd], w[3][wd], sel_hi);
                    mma16816<T>(o[4 * wd + 0], pa0, 0u, pa2, 0u, e4m3x2_to<T>(x01), e4m3x2_to<T>(y01));
                    mma16816<T>(o[4 * wd + 1], pa0, 0u, pa2, 0u, e4m3x2_to<T>(x01 >> 16), e4m3x2_to<T>(y01 >> 16));
                    mma16816<T>(o[4 * wd + 2], pa0, 0u, pa2, 0u, e4m3x2_to<T>(x23), e4m3x2_to<T>(y23));
                    mma16816<T>(o[4 * wd + 3], pa0, 0u, pa2, 0u, e4m3x2_to<T>(x23 >> 16), e4m3x2_to<T>(y23 >> 16));
                }
            } else {
#pragma unroll
                for (int np = 0; np < HD / 16; ++np) {
                    uint32_t b0, b1, b2, b3;
                    const int row = wk * 16 + (lane & 7) + (((lane >> 3) & 1) << 3);
                    const int chunk = (np * 2 + (lane >> 4)) & 7;
                    ldsm_x4_t(vt + (np / 4) * SUB_BYTES + swz(row, chunk), b0, b1, b2, b3);
                    mma16816<T>(o[2 * np], pa0, 0u, pa2, 0u, b0, b1);
                    mma16816<T>(o[2 * np + 1], pa0, 0u, pa2, 0u, b2, b3);
                }
            }
        }
        if (PAR) {
            if (ci + NST < nchunks) {                   // uniform within the group: refill this group's stage
                asm volatile("bar.sync %0, %1;" ::"r"(grp + 1), "r"(kWarps * 32) : "memory");
                if (wk == 0 && lane == 0) issue(ci + NST);
            }
        } else {
            __syncthreads();                            // every warp is done with stage s
            if (threadIdx.x == 0 && ci + NST < nchunks) issue(ci + NST);
        }
    }

    // ---- merge the warps (each saw a disjoint key subset) and, when FUSED, the new key held in shared memory
    float* wrow = merge + warp * (HD + 2);
    if (g == 0) {
#pragma unroll
        for (int i = 0; i < HD / 8; ++i) {
            if constexpr (F8) {                        // n8 tile i, column n <-> head dim (HD / 8) * n + i
                wrow[(HD / 8) * (2 * tg) + i] = o[i][0];
                wrow[(HD / 8) * (2 * tg + 1) + i] = o[i][1];
            } else {
                wrow[i * 8 + tg * 2] = o[i][0];
                wrow[i * 8 + tg * 2 + 1] = o[i][1];
            }
        }
        if (tg == 0) { wrow[HD] = mx; wrow[HD + 1] = l; }
    }
    if (FUSED && warp == 0) {
        float dot = 0.f;
#pragma unroll
        for (int i = 0; i < HD / 32; ++i) {
            const int e = lane * (HD / 32) + i;
            dot = fmaf(ElemTraits<T>::to_f(qbuf[e]), ElemTraits<T>::to_f(qbuf[HD + e]), dot);
        }
        dot = warp_sum(dot);
        float* crow = merge + NW * (HD + 2);
#pragma unroll
        for (int i = 0; i < HD / 32; ++i) {
            const int e = lane * (HD / 32) + i;
            crow[e] = ElemTraits<T>::to_f(qbuf[2 * HD + e]);
        }
        if (lane == 0) { crow[HD] = dot * a.scale; crow[HD + 1] = 1.f; }
    }
    __syncthreads();
    T* op = reinterpret_cast<T*>(a.out) + (size_t)r * D + (size_t)h * hdr;
    for (int e = threadIdx.x; e < hdr; e += blockDim.x) {
        float M_ = -INFINITY;
#pragma unroll
        for (int w = 0; w < NSLOT; ++w) M_ = fmaxf(M_, merge[w * (HD + 2) + HD]);
        float L = 0.f, O = 0.f;
#pragma unroll
        for (int w = 0; w < NSLOT; ++w) {
            const float mw = merge[w * (HD + 2) + HD];
            const float c = mw == -INFINITY ? 0.f : __expf(mw - M_);
            L += merge[w * (HD + 2) + HD + 1] * c;
            O += merge[w * (HD + 2) + e] * c;
        }
        if constexpr (F8) op[e] = ElemTraits<T>::from_f(O / L * f8s.v_scale);
        else op[e] = ElemTraits<T>::from_f(O / L);
    }
}

// The AttnTmaArgs of a call (kernels 1-4)
AttnTmaArgs tma_args(const AttnArgs& a) {
    AttnTmaArgs t{};
    t.q = (const bf16*)a.q; t.out = (bf16*)a.out; t.R = a.R; t.H = a.H; t.maxS = a.maxS;
    t.pos_dev = a.pos.dev; t.pos_value = a.pos.value; t.pos_rows = a.pos.rows; t.row_base = a.cache_row_base;
    t.emb_mask = a.emb_mask; t.B = a.B; t.Tc = a.Tc; t.emb_mask_uncond = a.emb_mask_uncond; t.scale = a.scale;
    t.partial = a.qkv_partial; t.ksplit = a.qkv_ksplit; t.freqs = a.freqs;
    t.kcache = (bf16*)const_cast<void*>(a.kcache); t.vcache = (bf16*)const_cast<void*>(a.vcache);
    t.hd = a.hd; t.hdp = a.hdp ? a.hdp : a.hd;
    return t;
}

template <typename T, int HD, bool FUSED, int NST, bool PAR, bool F8>
int launch_t(const AttnArgs& a, cudaStream_t st) {
    constexpr int TILE_BYTES = F8 ? kKC * (HD == 64 ? 64 : 128) : (HD / 64) * kKC * 128;
    constexpr int NW = PAR ? NST * kWarps : kWarps;
    const size_t smem = 1024 + (size_t)NST * 2 * TILE_BYTES + NST * sizeof(uint64_t) +
                        (NW + 1) * (HD + 2) * sizeof(float) + 3 * HD * sizeof(T) + 16;
    static DevOnce attr;
    if (lg_first_on_device(attr)) {
        LG_CUDA_OK(cudaFuncSetAttribute(attn_tma_kernel<T, HD, FUSED, NST, PAR, F8>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
    }
    AttnTmaArgs t = tma_args(a);
    t.kvhint = tma::kL2EvictFirst;   // each K/V byte is read once per step
    auto map = [](const void* m) -> const CUtensorMap& { return *reinterpret_cast<const CUtensorMap*>(m); };
    dim3 grid(a.H, a.R);
    (void)lg_launch(attn_tma_kernel<T, HD, FUSED, NST, PAR, F8>, dim3(grid), dim3(NW * 32), smem, st, map(a.kmap), map(a.vmap),
                    map(a.kmap16), map(a.vmap16), t, KvScales{a.k_inv, a.v_inv, a.v_scale});
    LG_LAUNCH_CHECK();
    return 0;
}

}  // namespace

// ---------------------------------------------------------------------------------------------------
// Prefill attention for the t2i condition (Tq = T <= 128 query positions per row, gpt.py:232-236 with the causal mask of
// gpt.py:354 and the emb_masks of generate.py:154-163): one CTA per (row, head). Q (post-RoPE, [R*T, D]) and the T freshly
// written K/V rows arrive by TMA (one box for Q, kKC-row boxes of the cache maps for K and V), S = Q K^T and O = P V run on
// mma.sync m16n8k16 with ldmatrix operands (each warp owns 16 query rows and skips the key blocks above its causal diagonal),
// softmax in fp32 registers, P reused from the score fragments. Replaces one CUDA-core CTA per (query, head).
// ---------------------------------------------------------------------------------------------------
constexpr int kPfRows = 128;                                   // query / key rows staged per (row, head)
constexpr int kPfBoxes = (kPfRows + kKC - 1) / kKC;            // K (or V) boxes of kKC rows

// F8 = true: fp8 e4m3 cache. The K / V boxes are [kKC keys][64 bytes] (64-byte swizzle) and are decoded in registers like the decode
// kernel's: q.K^T visits the head dims in the permuted order of f8_qdim (the Q fragments are read from shared memory in that order
// instead of by ldmatrix), P.V transposes key bytes with prmt and yields 16 contiguous output dims per lane and row.
template <typename T, bool F8 = false>
__global__ void __launch_bounds__(256, 2) attn_prefill_tc_kernel(const __grid_constant__ CUtensorMap qmap,
                                                                 const __grid_constant__ CUtensorMap kmap,
                                                                 const __grid_constant__ CUtensorMap vmap, AttnTmaArgs a, int Tq,
                                                                 KvScales f8s) {
    constexpr int HD = 64;
    constexpr int RB = F8 ? 64 : 128;                // bytes per K / V tile row
    extern __shared__ __align__(1024) uint8_t smem_raw[];
    uint8_t* qs = reinterpret_cast<uint8_t*>(((uintptr_t)smem_raw + 1023) & ~(uintptr_t)1023);   // [128][64] T, swizzle-128B
    uint8_t* ks = qs + kPfRows * 128;                                                              // [kPfBoxes * kKC][64]
    uint8_t* vs = ks + kPfBoxes * kKC * RB;
    uint64_t* bar = reinterpret_cast<uint64_t*>(vs + kPfBoxes * kKC * RB);
    const int h = blockIdx.x, r = blockIdx.y;
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31, g = lane >> 2, tg = lane & 3;
    const long long row0 = a.row_base + ((long long)r * a.H + h) * a.maxS;
    const int D = a.H * HD;
    if (threadIdx.x == 0) {
        prefetch_map(&qmap);
        prefetch_map(&kmap);
        prefetch_map(&vmap);
        mbar_init(bar, 1);
        fence_barrier_init();
    }
    __syncthreads();
    lg_pdl_sync();                                   // q and the K/V rows were written by the QKV epilogue just before
    if (threadIdx.x == 0) {
        mbar_expect_tx(bar, (uint32_t)(kPfRows * 128 + 2 * kPfBoxes * kKC * RB));
        load_2d(qs, &qmap, bar, h * HD, r * Tq);
        for (int i = 0; i < kPfBoxes; ++i) {
            load_2d(ks + i * kKC * RB, &kmap, bar, 0, (int)(row0 + (long long)i * kKC));
            load_2d(vs + i * kKC * RB, &vmap, bar, 0, (int)(row0 + (long long)i * kKC));
        }
    }
    mbar_wait(bar, 0);
    const int q0 = warp * 16;                        // this warp's query rows [q0, q0 + 16)
    if (q0 >= Tq) return;
    const uint32_t qb = smem_u32(qs), kb = smem_u32(ks), vb = smem_u32(vs);
    const int nkb = warp + 1;                        // 16-key blocks at or below the causal diagonal of these rows

    float sc[16][4];
#pragma unroll
    for (int i = 0; i < 16; ++i) { sc[i][0] = 0.f; sc[i][1] = 0.f; sc[i][2] = 0.f; sc[i][3] = 0.f; }
    if constexpr (F8) {
        // A fragments of rows q0 + g and q0 + g + 8 for the 4 k16 steps, dims in f8_qdim order (4 consecutive dims of one chunk)
        uint32_t qf[HD / 16][4];
#pragma unroll
        for (int kk = 0; kk < HD / 16; ++kk) {
            const int d = f8_qdim<HD>(tg, kk);
#pragma unroll
            for (int hh = 0; hh < 2; ++hh) {
                const uint8_t* p = qs + swz(q0 + g + 8 * hh, d >> 3) + (d & 7) * 2;
                qf[kk][hh] = *reinterpret_cast<const uint32_t*>(p);           // a0 / a1: dims d, d + 1
                qf[kk][2 + hh] = *reinterpret_cast<const uint32_t*>(p + 4);   // a2 / a3: dims d + 2, d + 3
            }
        }
#pragma unroll
        for (int kb16 = 0; kb16 < 8; ++kb16) {
            if (kb16 < nkb) {
#pragma unroll
                for (int nt = 0; nt < 2; ++nt) {
                    const uint4 kw = *reinterpret_cast<const uint4*>(ks + swz8<RB>(kb16 * 16 + nt * 8 + g, f8_kchunk<HD>(tg, 0)));
                    const uint32_t w[4] = {kw.x, kw.y, kw.z, kw.w};
#pragma unroll
                    for (int kk = 0; kk < HD / 16; ++kk)
                        mma16816<T>(sc[2 * kb16 + nt], qf[kk][0], qf[kk][1], qf[kk][2], qf[kk][3], e4m3x2_to<T>(w[kk]),
                                    e4m3x2_to<T>(w[kk] >> 16));
                }
            }
        }
    } else {
#pragma unroll
        for (int kk = 0; kk < HD / 16; ++kk) {
            uint32_t a0, a1, a2, a3;
            ldsm_x4(qb + swz(q0 + (lane & 15), (kk * 2 + (lane >> 4)) & 7), a0, a1, a2, a3);
#pragma unroll
            for (int kb16 = 0; kb16 < 8; ++kb16) {
                if (kb16 < nkb) {
                    uint32_t b0, b1, b2, b3;
                    const int row = kb16 * 16 + (lane & 7) + ((lane >> 4) << 3);
                    ldsm_x4(kb + swz(row, (kk * 2 + ((lane >> 3) & 1)) & 7), b0, b1, b2, b3);
                    mma16816<T>(sc[2 * kb16], a0, a1, a2, a3, b0, b1);
                    mma16816<T>(sc[2 * kb16 + 1], a0, a1, a2, a3, b2, b3);
                }
            }
        }
    }
    // ---- mask + softmax; this thread holds rows t0 = q0 + g (values [..][0..1]) and t1 = t0 + 8 (values [..][2..3])
    const float* mrow = attn_mask_row(a, r);
    float mx[2] = {-INFINITY, -INFINITY};
#pragma unroll
    for (int nt = 0; nt < 16; ++nt) {
#pragma unroll
        for (int e = 0; e < 4; ++e) {
            const int t = q0 + g + ((e >> 1) << 3), j = nt * 8 + tg * 2 + (e & 1);
            bool vis = j <= t && nt < 2 * nkb;
            if (vis && mrow && j < a.Tc && j != t) vis = mrow[j] != 0.f;
            const float x = vis ? sc[nt][e] * a.scale : -INFINITY;
            sc[nt][e] = x;
            mx[e >> 1] = fmaxf(mx[e >> 1], x);
        }
    }
    float l[2] = {0.f, 0.f};
#pragma unroll
    for (int hh = 0; hh < 2; ++hh) {
        mx[hh] = fmaxf(mx[hh], __shfl_xor_sync(0xffffffffu, mx[hh], 1));
        mx[hh] = fmaxf(mx[hh], __shfl_xor_sync(0xffffffffu, mx[hh], 2));
    }
#pragma unroll
    for (int nt = 0; nt < 16; ++nt) {
#pragma unroll
        for (int e = 0; e < 4; ++e) {
            const float pv = __expf(sc[nt][e] - mx[e >> 1]);      // the diagonal key is always visible: mx is finite
            sc[nt][e] = pv;
            l[e >> 1] += pv;
        }
    }
#pragma unroll
    for (int hh = 0; hh < 2; ++hh) {
        l[hh] += __shfl_xor_sync(0xffffffffu, l[hh], 1);
        l[hh] += __shfl_xor_sync(0xffffffffu, l[hh], 2);
    }
    // ---- O = P V
    float o[HD / 8][4];
#pragma unroll
    for (int i = 0; i < HD / 8; ++i) { o[i][0] = 0.f; o[i][1] = 0.f; o[i][2] = 0.f; o[i][3] = 0.f; }
#pragma unroll
    for (int kb16 = 0; kb16 < 8; ++kb16) {
        if (kb16 < nkb) {
            const uint32_t pa0 = pack16<T>(sc[2 * kb16][0], sc[2 * kb16][1]), pa1 = pack16<T>(sc[2 * kb16][2], sc[2 * kb16][3]);
            const uint32_t pa2 = pack16<T>(sc[2 * kb16 + 1][0], sc[2 * kb16 + 1][1]), pa3 = pack16<T>(sc[2 * kb16 + 1][2], sc[2 * kb16 + 1][3]);
            if constexpr (F8) {
                // n8 tile t, column n <-> head dim 8n + t; the lane reads 8 bytes (dims 8g .. 8g + 7) of keys 2tg, 2tg + 1, +8, +9
                const int sw = tg & 1, rb = kb16 * 16 + 2 * tg;
                uint32_t w[4][2];
#pragma unroll
                for (int q = 0; q < 4; ++q) {
                    const uint2 u = *reinterpret_cast<const uint2*>(vs + swz8<RB>(rb + (q >> 1) * 8 + ((q & 1) ^ sw), g >> 1) + (g & 1) * 8);
                    w[q][0] = u.x; w[q][1] = u.y;
                }
                const uint32_t sel_lo = sw ? 0x1504u : 0x5140u, sel_hi = sw ? 0x3726u : 0x7362u;
#pragma unroll
                for (int wd = 0; wd < 2; ++wd) {
                    const uint32_t x01 = __byte_perm(w[0][wd], w[1][wd], sel_lo), x23 = __byte_perm(w[0][wd], w[1][wd], sel_hi);
                    const uint32_t y01 = __byte_perm(w[2][wd], w[3][wd], sel_lo), y23 = __byte_perm(w[2][wd], w[3][wd], sel_hi);
                    mma16816<T>(o[4 * wd + 0], pa0, pa1, pa2, pa3, e4m3x2_to<T>(x01), e4m3x2_to<T>(y01));
                    mma16816<T>(o[4 * wd + 1], pa0, pa1, pa2, pa3, e4m3x2_to<T>(x01 >> 16), e4m3x2_to<T>(y01 >> 16));
                    mma16816<T>(o[4 * wd + 2], pa0, pa1, pa2, pa3, e4m3x2_to<T>(x23), e4m3x2_to<T>(y23));
                    mma16816<T>(o[4 * wd + 3], pa0, pa1, pa2, pa3, e4m3x2_to<T>(x23 >> 16), e4m3x2_to<T>(y23 >> 16));
                }
            } else {
#pragma unroll
                for (int np = 0; np < HD / 16; ++np) {
                    uint32_t b0, b1, b2, b3;
                    const int row = kb16 * 16 + (lane & 7) + (((lane >> 3) & 1) << 3);
                    ldsm_x4_t(vb + swz(row, (np * 2 + (lane >> 4)) & 7), b0, b1, b2, b3);
                    mma16816<T>(o[2 * np], pa0, pa1, pa2, pa3, b0, b1);
                    mma16816<T>(o[2 * np + 1], pa0, pa1, pa2, pa3, b2, b3);
                }
            }
        }
    }
#pragma unroll
    for (int hh = 0; hh < 2; ++hh) {
        const int t = q0 + g + hh * 8;
        if (t < Tq) {
            const float inv = 1.0f / l[hh];
            T* op = reinterpret_cast<T*>(a.out) + ((size_t)r * Tq + t) * D + (size_t)h * HD;
            if constexpr (F8) {   // o[i][2hh] -> dim 16tg + i, o[i][2hh + 1] -> dim 16tg + 8 + i: 16 contiguous dims (O / L * v_scale)
                uint32_t pk[8];
#pragma unroll
                for (int i = 0; i < 4; ++i) {
                    pk[i] = pack16<T>(o[2 * i][2 * hh] * inv * f8s.v_scale, o[2 * i + 1][2 * hh] * inv * f8s.v_scale);
                    pk[4 + i] = pack16<T>(o[2 * i][2 * hh + 1] * inv * f8s.v_scale, o[2 * i + 1][2 * hh + 1] * inv * f8s.v_scale);
                }
                *reinterpret_cast<uint4*>(op + 16 * tg) = make_uint4(pk[0], pk[1], pk[2], pk[3]);
                *reinterpret_cast<uint4*>(op + 16 * tg + 8) = make_uint4(pk[4], pk[5], pk[6], pk[7]);
            } else {
#pragma unroll
                for (int i = 0; i < HD / 8; ++i)
                    *reinterpret_cast<uint32_t*>(op + i * 8 + tg * 2) = pack16<T>(o[i][2 * hh] * inv, o[i][2 * hh + 1] * inv);
            }
        }
    }
}

// ---------------------------------------------------------------------------------------------------
// Long causal attention (Tq > 128 query positions per row, from position 0: the teacher-forced sequence of lg_score, gpt.py:341-368
// in eval mode): one CTA per (head, row, block of kCqRows queries), 4 warps of 16 query rows each. The key blocks at or below the
// block's causal diagonal stream through a kCqStages-deep TMA / mbarrier ring in kCqKeys-key blocks (kKC-row boxes of the KV maps);
// S = Q K^T and O += P V run on mma.sync m16n8k16 with ldmatrix operands, the softmax is online in fp32 registers and P is reused
// from the score fragments (FlashAttention-2). Q comes straight from global memory into A fragments (rows of 64, 128 or the 100
// dims of GPT-3B, whose K / V rows are 112 wide: the maps read dims 112..127 as zeros). No R * Tq grid limit.
//
// F8 = true: fp8 e4m3 cache (kernel 2 only: attn_causal_tc_f8_kernel). A stage holds [kCqKeys keys][64 or 128 bytes] (one box covers
// a whole row, 64-byte swizzle for hd 64, 128-byte otherwise) and the B operands are decoded in registers as in attn_tma_kernel<..,
// F8>: q.K^T visits the head dims in the f8_qdim order (Q's A fragments are read in that order), P.V transposes key bytes with prmt
// and leaves the output dims permuted (put back in the store). The K scale is in a.scale, the V scale multiplies O / L.
// ---------------------------------------------------------------------------------------------------
constexpr int kCqRows = 64;       // query rows per CTA
constexpr int kCqKeys = 64;       // keys per ring stage
constexpr int kCqStages = 2;

//
// The speculative (Jacobi) decoding window runs the same body with a per-row start (attn_window_tc_kernel): row r's Tq <= kCqRows
// queries sit at positions a.pos_rows[r] + t and attend keys [0, a.pos_rows[r] + t]; q and out stay [R * Tq, D].
template <typename T, int HD, bool WINDOW, bool F8 = false>
__device__ __forceinline__ void causal_tc_body(const CUtensorMap& kmap, const CUtensorMap& vmap, const AttnTmaArgs& a, int Tq,
                                               KvScales f8s = KvScales{1.f, 1.f, 1.f}) {
    constexpr int RB = F8 ? (HD == 64 ? 64 : 128) : 128;   // bytes per tile row of one box
    constexpr int NSUB = F8 ? 1 : HD / 64;        // 64-dim sub-tiles per row (fp8: one box covers the whole row)
    constexpr int SUB_BYTES = kCqKeys * RB;       // [kCqKeys keys][64 dims] 16-bit, 128-byte swizzle (fp8: [kCqKeys][RB bytes])
    constexpr int TILE_BYTES = NSUB * SUB_BYTES;
    constexpr int NT = kCqKeys / 8;               // n8 score tiles per stage
    extern __shared__ __align__(1024) uint8_t smem_raw[];
    uint8_t* tiles = reinterpret_cast<uint8_t*>(((uintptr_t)smem_raw + 1023) & ~(uintptr_t)1023);
    uint64_t* full_bar = reinterpret_cast<uint64_t*>(tiles + kCqStages * 2 * TILE_BYTES);

    const int h = blockIdx.x, r = blockIdx.y;
    const int q0 = (gridDim.z - 1 - blockIdx.z) * kCqRows;   // the longest blocks start first
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31, g = lane >> 2, tg = lane & 3;
    const long long row0 = a.row_base + ((long long)r * a.H + h) * a.maxS;
    const int hdr = a.hd, D = a.H * hdr;

    if (threadIdx.x == 0) {
        prefetch_map(&kmap);
        prefetch_map(&vmap);
        for (int s = 0; s < kCqStages; ++s) mbar_init(&full_bar[s], 1);
        fence_barrier_init();
    }
    __syncthreads();
    lg_pdl_sync();                                   // q and the K / V rows were written by the QKV epilogue just before
    // absolute position of query 0: read after the dependency wait, since the previous iteration's last kernel moves the positions
    const int p0 = WINDOW ? a.pos_rows[r] : 0;
    const int nkeys = p0 + min(q0 + kCqRows, Tq);
    const int nblk = (nkeys + kCqKeys - 1) / kCqKeys;
    auto issue = [&](int kb) {
        const int s = kb % kCqStages;
        uint8_t* kt = tiles + s * 2 * TILE_BYTES;
        uint8_t* vt = kt + TILE_BYTES;
        mbar_expect_tx(&full_bar[s], 2 * TILE_BYTES);
#pragma unroll
        for (int sub = 0; sub < NSUB; ++sub)
#pragma unroll
            for (int i = 0; i < kCqKeys / kKC; ++i) {
                const int row = (int)(row0 + (long long)kb * kCqKeys + i * kKC);
                load_2d(kt + sub * SUB_BYTES + i * kKC * RB, &kmap, &full_bar[s], sub * 64, row);
                load_2d(vt + sub * SUB_BYTES + i * kKC * RB, &vmap, &full_bar[s], sub * 64, row);
            }
    };
    if (threadIdx.x == 0)
        for (int kb = 0; kb < min(kCqStages, nblk); ++kb) issue(kb);

    // Q rows t0 = q0 + 16 warp + g and t1 = t0 + 8 as m16n8k16 A fragments (pairs of dims; hdr % 4 == 0, so a pair is all real
    // or all padding)
    const int t0 = q0 + warp * 16 + g, t1 = t0 + 8;
    uint32_t qa[HD / 16][4];
    {
        const T* qp = reinterpret_cast<const T*>(a.q) + (size_t)h * hdr;
        const T* r0p = qp + ((size_t)r * Tq + t0) * D;
        const T* r1p = qp + ((size_t)r * Tq + t1) * D;
#pragma unroll
        for (int kk = 0; kk < HD / 16; ++kk) {
            // fp8: the k16 step's pairs are dims d, d + 1 (a0 / a1) and d + 2, d + 3 (a2 / a3) of f8_qdim, all real or all padding
            const int d0 = F8 ? f8_qdim<HD>(tg, kk) : kk * 16 + tg * 2, d1 = F8 ? d0 + 2 : d0 + 8;
            qa[kk][0] = (t0 < Tq && d0 < hdr) ? *reinterpret_cast<const uint32_t*>(r0p + d0) : 0u;
            qa[kk][1] = (t1 < Tq && d0 < hdr) ? *reinterpret_cast<const uint32_t*>(r1p + d0) : 0u;
            qa[kk][2] = (t0 < Tq && d1 < hdr) ? *reinterpret_cast<const uint32_t*>(r0p + d1) : 0u;
            qa[kk][3] = (t1 < Tq && d1 < hdr) ? *reinterpret_cast<const uint32_t*>(r1p + d1) : 0u;
        }
    }
    const float* mrow = attn_mask_row(a, r);
    float o[HD / 8][4];
#pragma unroll
    for (int i = 0; i < HD / 8; ++i) { o[i][0] = 0.f; o[i][1] = 0.f; o[i][2] = 0.f; o[i][3] = 0.f; }
    float mx[2] = {-INFINITY, -INFINITY}, l[2] = {0.f, 0.f};   // running max (quad-uniform) and this lane's share of the sum

    for (int kb = 0; kb < nblk; ++kb) {
        const int s = kb % kCqStages;
        mbar_wait(&full_bar[s], (uint32_t)((kb / kCqStages) & 1));
        const int j0 = kb * kCqKeys;
        if (j0 <= p0 + q0 + warp * 16 + 15) {        // warp-uniform: some key of the block is at or below this warp's diagonal
            const uint32_t kt = smem_u32(tiles + s * 2 * TILE_BYTES);
            const uint32_t vt = kt + TILE_BYTES;
            float sc[NT][4];
#pragma unroll
            for (int i = 0; i < NT; ++i) { sc[i][0] = 0.f; sc[i][1] = 0.f; sc[i][2] = 0.f; sc[i][3] = 0.f; }
            if constexpr (F8) {
                // key nt * 8 + g of n8 tile nt: 16 dims (4 k16 steps) per 16-byte chunk f8_kchunk of each 64-dim block
                const uint8_t* ktp = tiles + s * 2 * TILE_BYTES;
#pragma unroll
                for (int nt = 0; nt < NT; ++nt) {
#pragma unroll
                    for (int j = 0; j < HD / 64; ++j) {
                        const uint4 kw = *reinterpret_cast<const uint4*>(ktp + swz8<RB>(nt * 8 + g, f8_kchunk<HD>(tg, j)));
                        const uint32_t w[4] = {kw.x, kw.y, kw.z, kw.w};
#pragma unroll
                        for (int i = 0; i < 4; ++i) {
                            const int kk = j * 4 + i;
                            mma16816<T>(sc[nt], qa[kk][0], qa[kk][1], qa[kk][2], qa[kk][3], e4m3x2_to<T>(w[i]), e4m3x2_to<T>(w[i] >> 16));
                        }
                    }
                }
            } else {
#pragma unroll
                for (int kk = 0; kk < HD / 16; ++kk) {
#pragma unroll
                    for (int np = 0; np < NT / 2; ++np) {
                        uint32_t b0, b1, b2, b3;
                        const int row = np * 16 + (lane & 7) + ((lane >> 4) << 3);
                        ldsm_x4(kt + (kk / 4) * SUB_BYTES + swz(row, (kk * 2 + ((lane >> 3) & 1)) & 7), b0, b1, b2, b3);
                        mma16816<T>(sc[2 * np], qa[kk][0], qa[kk][1], qa[kk][2], qa[kk][3], b0, b1);
                        mma16816<T>(sc[2 * np + 1], qa[kk][0], qa[kk][1], qa[kk][2], qa[kk][3], b2, b3);
                    }
                }
            }
            // ---- mask + online softmax; values [..][0..1] belong to row t0, [..][2..3] to row t1
            float bmax[2] = {-INFINITY, -INFINITY};
#pragma unroll
            for (int nt = 0; nt < NT; ++nt) {
#pragma unroll
                for (int e = 0; e < 4; ++e) {
                    const int t = p0 + ((e >> 1) ? t1 : t0), j = j0 + nt * 8 + tg * 2 + (e & 1);
                    bool vis = j <= t;
                    if (vis && mrow && j < a.Tc && j != t) vis = mrow[j] != 0.f;
                    const float x = vis ? sc[nt][e] * a.scale : -INFINITY;
                    sc[nt][e] = x;
                    bmax[e >> 1] = fmaxf(bmax[e >> 1], x);
                }
            }
            float corr[2];
#pragma unroll
            for (int hh = 0; hh < 2; ++hh) {
                bmax[hh] = fmaxf(bmax[hh], __shfl_xor_sync(0xffffffffu, bmax[hh], 1));
                bmax[hh] = fmaxf(bmax[hh], __shfl_xor_sync(0xffffffffu, bmax[hh], 2));
                const float mn = fmaxf(mx[hh], bmax[hh]);
                corr[hh] = mn == -INFINITY ? 1.f : __expf(mx[hh] - mn);   // exp(-inf) = 0 when the row saw no visible key yet
                mx[hh] = mn;
                l[hh] *= corr[hh];
            }
#pragma unroll
            for (int nt = 0; nt < NT; ++nt) {
#pragma unroll
                for (int e = 0; e < 4; ++e) {
                    const float m = mx[e >> 1];
                    const float pv = m == -INFINITY ? 0.f : __expf(sc[nt][e] - m);
                    sc[nt][e] = pv;
                    l[e >> 1] += pv;
                }
            }
#pragma unroll
            for (int i = 0; i < HD / 8; ++i) { o[i][0] *= corr[0]; o[i][1] *= corr[0]; o[i][2] *= corr[1]; o[i][3] *= corr[1]; }
            // ---- O += P V, P packed to T from the score fragments (C layout of S == A layout of P)
#pragma unroll
            for (int kb16 = 0; kb16 < kCqKeys / 16; ++kb16) {
                const uint32_t pa0 = pack16<T>(sc[2 * kb16][0], sc[2 * kb16][1]), pa1 = pack16<T>(sc[2 * kb16][2], sc[2 * kb16][3]);
                const uint32_t pa2 = pack16<T>(sc[2 * kb16 + 1][0], sc[2 * kb16 + 1][1]);
                const uint32_t pa3 = pack16<T>(sc[2 * kb16 + 1][2], sc[2 * kb16 + 1][3]);
                if constexpr (F8) {
                    // n8 tile i, column n <-> head dim DPT * n + i; the lane reads DPT bytes (dims DPT * g ..) of keys 2tg, 2tg + 1,
                    // + 8, + 9 (odd tg swap the rows of a pair so a half warp hits distinct banks), prmt pairs the keys' bytes
                    constexpr int DPT = HD / 8, NWD = DPT / 4;
                    const uint8_t* vtp = tiles + s * 2 * TILE_BYTES + TILE_BYTES;
                    const int sw = tg & 1, rb = kb16 * 16 + 2 * tg;
                    uint32_t w[4][NWD];
#pragma unroll
                    for (int q = 0; q < 4; ++q) {
                        const int row = rb + (q >> 1) * 8 + ((q & 1) ^ sw);
                        if constexpr (RB == 64) {
                            const uint2 u = *reinterpret_cast<const uint2*>(vtp + swz8<RB>(row, g >> 1) + (g & 1) * 8);
                            w[q][0] = u.x; w[q][NWD - 1] = u.y;
                        } else {
                            const uint4 u = *reinterpret_cast<const uint4*>(vtp + swz8<RB>(row, g));
                            w[q][0] = u.x; w[q][1 % NWD] = u.y; w[q][2 % NWD] = u.z; w[q][3 % NWD] = u.w;
                        }
                    }
                    const uint32_t sel_lo = sw ? 0x1504u : 0x5140u, sel_hi = sw ? 0x3726u : 0x7362u;
#pragma unroll
                    for (int wd = 0; wd < NWD; ++wd) {
                        const uint32_t x01 = __byte_perm(w[0][wd], w[1][wd], sel_lo), x23 = __byte_perm(w[0][wd], w[1][wd], sel_hi);
                        const uint32_t y01 = __byte_perm(w[2][wd], w[3][wd], sel_lo), y23 = __byte_perm(w[2][wd], w[3][wd], sel_hi);
                        mma16816<T>(o[4 * wd + 0], pa0, pa1, pa2, pa3, e4m3x2_to<T>(x01), e4m3x2_to<T>(y01));
                        mma16816<T>(o[4 * wd + 1], pa0, pa1, pa2, pa3, e4m3x2_to<T>(x01 >> 16), e4m3x2_to<T>(y01 >> 16));
                        mma16816<T>(o[4 * wd + 2], pa0, pa1, pa2, pa3, e4m3x2_to<T>(x23), e4m3x2_to<T>(y23));
                        mma16816<T>(o[4 * wd + 3], pa0, pa1, pa2, pa3, e4m3x2_to<T>(x23 >> 16), e4m3x2_to<T>(y23 >> 16));
                    }
                } else {
#pragma unroll
                    for (int np = 0; np < HD / 16; ++np) {
                        uint32_t b0, b1, b2, b3;
                        const int row = kb16 * 16 + (lane & 7) + (((lane >> 3) & 1) << 3);
                        ldsm_x4_t(vt + (np / 4) * SUB_BYTES + swz(row, (np * 2 + (lane >> 4)) & 7), b0, b1, b2, b3);
                        mma16816<T>(o[2 * np], pa0, pa1, pa2, pa3, b0, b1);
                        mma16816<T>(o[2 * np + 1], pa0, pa1, pa2, pa3, b2, b3);
                    }
                }
            }
        }
        __syncthreads();                             // every warp is done with stage s
        if (threadIdx.x == 0 && kb + kCqStages < nblk) issue(kb + kCqStages);
    }
#pragma unroll
    for (int hh = 0; hh < 2; ++hh) {
        l[hh] += __shfl_xor_sync(0xffffffffu, l[hh], 1);
        l[hh] += __shfl_xor_sync(0xffffffffu, l[hh], 2);
    }
#pragma unroll
    for (int hh = 0; hh < 2; ++hh) {
        const int t = hh ? t1 : t0;
        if (t < Tq) {
            const float inv = 1.0f / l[hh];          // the diagonal key is always visible: l > 0
            T* op = reinterpret_cast<T*>(a.out) + ((size_t)r * Tq + t) * D + (size_t)h * hdr;
            if constexpr (F8) {   // o[i][2hh] -> dim DPT * 2tg + i, o[i][2hh + 1] -> dim DPT * (2tg + 1) + i (O / L * v_scale)
                constexpr int DPT = HD / 8;
                const float f = inv * f8s.v_scale;
#pragma unroll
                for (int i = 0; i < DPT; i += 2)
#pragma unroll
                    for (int c = 0; c < 2; ++c) {
                        const int d = DPT * (2 * tg + c) + i;
                        if (d < hdr) *reinterpret_cast<uint32_t*>(op + d) = pack16<T>(o[i][2 * hh + c] * f, o[i + 1][2 * hh + c] * f);
                    }
            } else {
#pragma unroll
                for (int i = 0; i < HD / 8; ++i)
                    if (i * 8 + tg * 2 < hdr) *reinterpret_cast<uint32_t*>(op + i * 8 + tg * 2) = pack16<T>(o[i][2 * hh] * inv, o[i][2 * hh + 1] * inv);
            }
        }
    }
}

template <typename T, int HD>
__global__ void __launch_bounds__(128) attn_causal_tc_kernel(const __grid_constant__ CUtensorMap kmap,
                                                             const __grid_constant__ CUtensorMap vmap, AttnTmaArgs a, int Tq) {
    causal_tc_body<T, HD, false>(kmap, vmap, a, Tq);
}

// kernel 2 over an fp8 cache: the same body with F8 = true; the scales are a separate last argument so that the 16-bit kernel above
// keeps its argument layout and its code
template <typename T, int HD>
__global__ void __launch_bounds__(128) attn_causal_tc_f8_kernel(const __grid_constant__ CUtensorMap kmap,
                                                                const __grid_constant__ CUtensorMap vmap, AttnTmaArgs a, int Tq,
                                                                KvScales f8s) {
    causal_tc_body<T, HD, false, true>(kmap, vmap, a, Tq, f8s);
}

template <typename T, int HD>
__global__ void __launch_bounds__(128) attn_window_tc_kernel(const __grid_constant__ CUtensorMap kmap,
                                                             const __grid_constant__ CUtensorMap vmap, AttnTmaArgs a, int Tq) {
    causal_tc_body<T, HD, true>(kmap, vmap, a, Tq);
}

// KV-cache tensor maps: the whole K (or V) region of the workspace as one [rows, hd] bf16 / fp16 matrix, or (dtype LG_DTYPE_E4M3)
// one [rows, hdp] byte matrix read in boxes of 64 bytes (hd 64) or 128 bytes (hdp 128 or 112; bytes 112..127 read as zeros)
int attn_tma_make_map(void* map_out, const void* cache_base, long long total_rows, int hdp, int dtype, int tail16) {
    // hdp = cache row width in elements (64, 128, or 112 for head_dim 100: the second 64-wide box then reads 112..127 as zeros)
    return tma::make_map_2d(reinterpret_cast<CUtensorMap*>(map_out), cache_base, (uint64_t)total_rows, (uint64_t)hdp, (uint64_t)hdp,
                            tail16 ? 16 : kKC, dtype == LG_DTYPE_E4M3 ? (hdp == 64 ? 64 : 128) : 64, dtype);
}

// Head shapes of the TMA kernels: hd 64 or 128, or hd 100 in 112-wide rows (the maps read 112..127 as zeros)
static bool tma_head_shape(int hd, int hdp) { return hd == 64 || hd == 128 || (hd == 100 && hdp == 112); }

bool attn_tma_maps_usable(int dtype, int hd, int hdp, long long total_rows) {
    return lg_dtype_is16(dtype) && tma_head_shape(hd, hdp) && total_rows < (1ll << 31);
}

AttnPlan attn_plan(const AttnArgs& a) {
    AttnPlan p;
    auto plan = [&](int kernel, int stages) { p.kernel = kernel; p.stages = stages; return p; };
    const bool fused = a.qkv_partial != nullptr;
    const bool from0 = a.pos.dev == nullptr && a.pos.rows == nullptr && a.pos.value == 0;   // query t sits at position t
    // kernels 1-4: a 16-bit model whose cache the maps cover, one grid row per sequence row
    const bool tma = lg_env_flag("LG_ATTN_TMA", 1) && lg_dtype_is16(a.dtype) && tma_head_shape(a.hd, a.hdp) && a.kmap && a.vmap &&
                     a.R <= 65535;
    if (tma && a.Tq == 1 && a.kmap16 && a.vmap16) {
        p.fused = fused;
        // few (row, head) items (batch-1 latency path): an 8-stage ring (kKC = 32) holds a whole 256-key context, so every K/V byte
        // is requested before the dependency wait instead of two stages at a time
        if (fused && a.hd == 64 && a.R * a.H <= 2 * 132 && lg_env_flag("LG_ATTN_DEEP", 1)) return plan(1, kDeepStages);
        // deeper sequential ring (A/B switch): more keys requested before the dependency wait, fewer refill round trips
        if (fused && a.hd == 64 && lg_env_flag("LG_ATTN_NST", 2) == 3) return plan(1, 3);
        return plan(1, kStagesA);
    }
    if (tma && !fused && a.hd == 64 && (a.hdp == 0 || a.hdp == 64) && a.Tq > 1 && a.Tq <= kPfRows && from0 && a.maxS >= kPfBoxes * kKC &&
        lg_env_flag("LG_ATTN_PREFILL_TC", 1))
        return plan(3, 1);
    if (tma && !fused && a.Tq > kPfRows && from0 && a.maxS >= a.Tq) return plan(2, kCqStages);   // kernel 2 reads fp8 caches too
    const bool tc16 = tma && !fused && !a.kv_f8;   // kernel 4: a 16-bit cache in the model dtype
    if (tc16 && a.Tq >= 2 && a.Tq <= kCqRows && a.pos.rows) return plan(4, kCqStages);
    if (fused) snprintf(p.error, sizeof(p.error), "attention: fused QKV epilogue requested on a path that does not support it");
    else if ((long long)a.R * a.Tq > 65535) snprintf(p.error, sizeof(p.error), "attention: too many query rows (%d x %d)", a.R, a.Tq);
    else if ((a.hdp ? a.hdp : a.hd) != attn_kv_row_width(a.dtype, a.hd))
        snprintf(p.error, sizeof(p.error), "attention: KV row width %d for head_dim %d", a.hdp, a.hd);
    else p.kernel = 0;
    return p;
}

// attn_tma_kernel at the plan's head dim, fusion and ring depth
template <typename T, bool F8>
static int launch_decode(const AttnArgs& a, const AttnPlan& p, cudaStream_t st) {
    const bool hd64 = a.hd == 64;
    if (!p.fused) return hd64 ? launch_t<T, 64, false, kStagesA, false, F8>(a, st) : launch_t<T, 128, false, kStagesA, false, F8>(a, st);
    if (p.stages == kDeepStages) return launch_t<T, 64, true, kDeepStages, true, F8>(a, st);
    if (p.stages == 3) return launch_t<T, 64, true, 3, false, F8>(a, st);
    return hd64 ? launch_t<T, 64, true, kStagesA, false, F8>(a, st) : launch_t<T, 128, true, kStagesA, false, F8>(a, st);
}

static int launch_prefill_tc(const AttnArgs& a, cudaStream_t st) {
    CUtensorMap qmap;
    LG_TRY(tma::make_map_2d(&qmap, a.q, (uint64_t)a.R * a.Tq, (uint64_t)a.H * a.hd, (uint64_t)a.H * a.hd, kPfRows, 64, a.dtype));
    const size_t smem = 1024 + (size_t)kPfRows * 128 + 2 * (size_t)kPfBoxes * kKC * (a.kv_f8 ? 64 : 128) + 16;
    const bool half = a.dtype == LG_DTYPE_F16;
    const int which = (half ? 1 : 0) + (a.kv_f8 ? 2 : 0);
    auto kern = a.kv_f8 ? (half ? attn_prefill_tc_kernel<f16, true> : attn_prefill_tc_kernel<bf16, true>)
                        : (half ? attn_prefill_tc_kernel<f16> : attn_prefill_tc_kernel<bf16>);
    static DevOnce attr[4];
    if (lg_first_on_device(attr[which])) {
        LG_CUDA_OK(cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
    }
    dim3 grid(a.H, a.R);
    (void)lg_launch(kern, dim3(grid), dim3(256), smem, st, qmap, *reinterpret_cast<const CUtensorMap*>(a.kmap),
                    *reinterpret_cast<const CUtensorMap*>(a.vmap), tma_args(a), a.Tq, KvScales{a.k_inv, a.v_inv, a.v_scale});
    LG_LAUNCH_CHECK();
    return 0;
}

// attn_window_tc_kernel (one query block per row, at the row's own position; caches in the model dtype)
static int launch_window_tc(const AttnArgs& a, cudaStream_t st) {
    const bool half = a.dtype == LG_DTYPE_F16, wide = a.hd != 64;
    auto kern = wide ? (half ? attn_window_tc_kernel<f16, 128> : attn_window_tc_kernel<bf16, 128>)
                     : (half ? attn_window_tc_kernel<f16, 64> : attn_window_tc_kernel<bf16, 64>);
    const size_t smem = 1024 + (size_t)kCqStages * 2 * (wide ? 2 : 1) * kCqKeys * 128 + kCqStages * sizeof(uint64_t);
    static DevOnce attr[4];
    if (lg_first_on_device(attr[(half ? 1 : 0) + (wide ? 2 : 0)])) {
        LG_CUDA_OK(cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
    }
    dim3 grid(a.H, a.R, (a.Tq + kCqRows - 1) / kCqRows);
    (void)lg_launch(kern, dim3(grid), dim3(128), smem, st, *reinterpret_cast<const CUtensorMap*>(a.kmap),
                    *reinterpret_cast<const CUtensorMap*>(a.vmap), tma_args(a), a.Tq);
    LG_LAUNCH_CHECK();
    return 0;
}

// attn_causal_tc_kernel (attn_causal_tc_f8_kernel for an fp8 cache) at the call's dtype and head dim
template <typename T, int HD, bool F8>
static int launch_causal_t(const AttnArgs& a, cudaStream_t st) {
    constexpr int TILE_BYTES = F8 ? kCqKeys * (HD == 64 ? 64 : 128) : (HD / 64) * kCqKeys * 128;
    const size_t smem = 1024 + (size_t)kCqStages * 2 * TILE_BYTES + kCqStages * sizeof(uint64_t);
    static DevOnce attr;
    const auto& kmap = *reinterpret_cast<const CUtensorMap*>(a.kmap);
    const auto& vmap = *reinterpret_cast<const CUtensorMap*>(a.vmap);
    dim3 grid(a.H, a.R, (a.Tq + kCqRows - 1) / kCqRows);
    if constexpr (F8) {
        if (lg_first_on_device(attr))
            LG_CUDA_OK(cudaFuncSetAttribute(attn_causal_tc_f8_kernel<T, HD>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
        (void)lg_launch(attn_causal_tc_f8_kernel<T, HD>, dim3(grid), dim3(128), smem, st, kmap, vmap, tma_args(a), a.Tq,
                        KvScales{a.k_inv, a.v_inv, a.v_scale});
    } else {
        if (lg_first_on_device(attr))
            LG_CUDA_OK(cudaFuncSetAttribute(attn_causal_tc_kernel<T, HD>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
        (void)lg_launch(attn_causal_tc_kernel<T, HD>, dim3(grid), dim3(128), smem, st, kmap, vmap, tma_args(a), a.Tq);
    }
    LG_LAUNCH_CHECK();
    return 0;
}

template <typename T>
static int launch_causal_tc(const AttnArgs& a, cudaStream_t st) {
    if (a.hd == 64) return a.kv_f8 ? launch_causal_t<T, 64, true>(a, st) : launch_causal_t<T, 64, false>(a, st);
    return a.kv_f8 ? launch_causal_t<T, 128, true>(a, st) : launch_causal_t<T, 128, false>(a, st);
}

int launch_attention_tma(const AttnArgs& a, const AttnPlan& p, cudaStream_t st) {
    const bool half = a.dtype == LG_DTYPE_F16;
    switch (p.kernel) {
        case 1:
            if (a.kv_f8) return half ? launch_decode<f16, true>(a, p, st) : launch_decode<bf16, true>(a, p, st);
            return half ? launch_decode<f16, false>(a, p, st) : launch_decode<bf16, false>(a, p, st);
        case 2: return half ? launch_causal_tc<f16>(a, st) : launch_causal_tc<bf16>(a, st);
        case 3: return launch_prefill_tc(a, st);
        case 4: return launch_window_tc(a, st);
    }
    return lg_fail("attention: kernel %d is not one of the TMA kernels", p.kernel);
}
