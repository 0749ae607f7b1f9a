// "Direct" wgmma GEMM for the decode step: one CTA = (128-feature weight tile) x (row block) over the FULL reduction, so
// there is no split-K slab and no separate row-epilogue kernel — the consumer of gpt.py's op is fused on both sides:
//
//   prologue (optional)  x_hat = RMSNorm(x) * w          gpt.py:143-148   (the CTA holds its rows over all of K in shared memory)
//   y[r, n] = sum_k x_hat[r, k] W[n, k]                   gpt.py:161-163,199-200
//   epilogue DX_RESID    h[r, n] = bf16(h[r, n] + bf16(y))                gpt.py:255-256 (in place)
//            DX_SWIGLU   ff[r, f] = bf16(bf16(silu(bf16(y1))) * bf16(y3)) gpt.py:167     (tile = 64 rows of w1 | the same 64 of w3)
//            DX_F32      y as fp32 (tests)
//
// A decode layer then is  QKV (split-K slabs) -> attention (reduces them) -> WO' [DX_RESID] -> W13' [norm + DX_SWIGLU] ->
// W2 (slabs) -> residual_norm : 6 dependent kernels instead of 8 (at decode sizes a kernel's dependent latency outweighs its
// bytes or flops).
//
// Data path: weights are the wgmma A operand (128 features = two warpgroups of M = 64) streamed by TMA through an mbarrier
// ring that is filled BEFORE the programmatic-dependency wait (weights never depend on activations); the activation rows of
// the CTA are the B operand (N = 16/32/64 rows), resident in shared memory for all of K as nkb swizzle-128B tiles. With a
// norm prologue the eight consumer warps rewrite those tiles in place (row sum of squares, then bf16(bf16(x * rstd) * w),
// the reference's rounding points) and hand them to the async proxy with fence.proxy.async before the first MMA. The
// accumulator lives in registers (feature = fragment row, activation row = fragment column).
#include "kernels.cuh"
#include "tma_utils.cuh"
#include "wgmma_utils.cuh"
#include <algorithm>

namespace {

using namespace tma;

constexpr int kTileN = 128;                      // weight rows per CTA; paired: 64 of Wa followed by 64 of Wb
constexpr int kBK = 64;                          // bf16 elements per k-block = one 128-byte swizzle row
constexpr int kWBytes = kTileN * kBK * 2;        // 16 KB weight stage
constexpr int kMaxSt = 12;
constexpr int kThreadsDx = 288;                  // warps 0-7: two consumer warpgroups, warp 8: TMA producer
constexpr int kConsumers = 256;
constexpr size_t kMaxXBytes = 128 * 1024;        // resident activation rows of one CTA (leaves >= 5 weight stages)
constexpr int kMiscBytes = 2 * kMaxSt * 8 + 8 + 64 * 4 + kConsumers * 4;   // barriers, rstd[64], red[256]

struct DxArgs {
    int M, N, K;          // activation rows, output features (paired: F), reduction
    int nkb;              // k-blocks of 64
    int stages;           // weight ring depth
    int mode, paired;
    const bf16* normw; float eps;
    float* out_f32; bf16* h; bf16* ff;
    const char* pf0; unsigned long long pfb0;   // next GEMM's weights to pull into L2 (see GemmNext)
    const char* pf1; unsigned long long pfb1;
    unsigned long long* trace;   // debug: [cta][12] %globaltimer stamps (nullable), see tools/dx_probe.py
};

__device__ __forceinline__ unsigned long long dx_gtime() {
    unsigned long long t;
    asm volatile("mov.u64 %0, %%globaltimer;" : "=l"(t));
    return t;
}
#define DX_TRACE(slot)                                                                                       \
    do {                                                                                                     \
        if (a.trace) a.trace[(size_t)(blockIdx.y * gridDim.x + blockIdx.x) * 12 + (slot)] = dx_gtime();      \
    } while (0)

__device__ __forceinline__ uint32_t pack_rn(float lo, float hi) {
    __nv_bfloat162 p = __floats2bfloat162_rn(lo, hi);
    return *reinterpret_cast<uint32_t*>(&p);
}
__device__ __forceinline__ uint32_t mul_bf16x2(uint32_t a, uint32_t b) {
    __nv_bfloat162 r = __hmul2(*reinterpret_cast<__nv_bfloat162*>(&a), *reinterpret_cast<__nv_bfloat162*>(&b));
    return *reinterpret_cast<uint32_t*>(&r);
}

// RB: rows per CTA = wgmma N (16, 32 or 64)
template <int RB>
__global__ void __launch_bounds__(kThreadsDx, 1) gemm_dx_kernel(const __grid_constant__ CUtensorMap map_wa,
                                                                const __grid_constant__ CUtensorMap map_wb,
                                                                const __grid_constant__ CUtensorMap map_x, DxArgs a) {
    extern __shared__ __align__(1024) uint8_t smem_raw[];
    uint8_t* base = reinterpret_cast<uint8_t*>(((uintptr_t)smem_raw + 1023) & ~(uintptr_t)1023);
    constexpr int xtile = RB * 128;                                  // one [RB rows][64 k] bf16 tile (2/4/8 KB)
    uint8_t* xres = base;                                            // nkb resident activation tiles
    uint8_t* ring = xres + (size_t)a.nkb * xtile;                    // weight stages (1024-aligned: xtile is a multiple of 2 KB)
    uint64_t* full = reinterpret_cast<uint64_t*>(ring + (size_t)a.stages * kWBytes);
    uint64_t* empty = full + kMaxSt;
    uint64_t* xfull = empty + kMaxSt;
    float* rstd_s = reinterpret_cast<float*>(xfull + 1);             // [64]
    float* red = rstd_s + 64;                                        // [256]
    bf16* gbuf = reinterpret_cast<bf16*>(((uintptr_t)(red + kConsumers) + 15) & ~(uintptr_t)15);   // [nkb * 64] norm weights (zero beyond K), read as uint4

    const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
    const int nt = blockIdx.x;
    const int row0 = (int)blockIdx.y * RB;
    const int Mb = min(RB, a.M - row0);
    const bool norm = a.normw != nullptr;
    if (tid == 0) DX_TRACE(0);

    if (warp == 8 && lane == 0) {
        prefetch_map(&map_wa);
        prefetch_map(&map_wb);
        prefetch_map(&map_x);
        for (int s = 0; s < a.stages; ++s) { mbar_init(&full[s], 1); mbar_init(&empty[s], 2); }
        mbar_init(xfull, 1);
        fence_barrier_init();
    }
    if (norm && warp < 8) {
        // the norm weight is a parameter: staged before the dependency wait
        const int n8 = a.nkb * 8, k8 = a.K / 8;
        for (int i = tid; i < n8; i += kConsumers)
            reinterpret_cast<uint4*>(gbuf)[i] = i < k8 ? __ldg(reinterpret_cast<const uint4*>(a.normw) + i) : make_uint4(0u, 0u, 0u, 0u);
    }
    __syncthreads();
    if (tid == 0) DX_TRACE(1);
    lg_pdl_launch_dependents();
    if (warp != 8) lg_pdl_wait();     // the producer waits after it has requested the first weight tiles

    if (warp == 8) {
        // ------------------------------------------------------------------ TMA producer
        if (elect_one()) {
            auto load_w = [&](int i, int s) {
                uint8_t* dst = ring + (size_t)s * kWBytes;
                mbar_expect_tx(&full[s], (uint32_t)kWBytes);
                if (!a.paired) {
                    load_2d(dst, &map_wa, &full[s], i * kBK, nt * kTileN);
                } else {
                    load_2d(dst, &map_wa, &full[s], i * kBK, nt * (kTileN / 2));
                    load_2d(dst + kWBytes / 2, &map_wb, &full[s], i * kBK, nt * (kTileN / 2));
                }
            };
            const int npre = min(a.nkb, a.stages);
            for (int i = 0; i < npre; ++i) load_w(i, i);
            DX_TRACE(2);
            lg_pdl_wait();
            DX_TRACE(3);
            mbar_expect_tx(xfull, (uint32_t)(a.nkb * xtile));
            for (int kb = 0; kb < a.nkb; ++kb) load_2d(xres + (size_t)kb * xtile, &map_x, xfull, kb * kBK, row0);
            for (int i = npre; i < a.nkb; ++i) {
                const int s = i % a.stages;
                mbar_wait(&empty[s], (uint32_t)(((i / a.stages) & 1) ^ 1));
                load_w(i, s);
            }
            DX_TRACE(4);
            // ask L2 for this CTA's share of the next GEMM's weights
            const unsigned long long cta = (unsigned long long)blockIdx.y * gridDim.x + blockIdx.x;
            const unsigned long long ncta = (unsigned long long)gridDim.x * gridDim.y;
            const char* pp[2] = {a.pf0, a.pf1};
            const unsigned long long bb[2] = {a.pfb0, a.pfb1};
#pragma unroll
            for (int t = 0; t < 2; ++t) {
                if (!bb[t]) continue;
                const unsigned long long per = ((bb[t] + ncta - 1) / ncta + 4095ull) & ~4095ull;
                unsigned long long off = cta * per;
                const unsigned long long end = off + per < bb[t] ? off + per : bb[t];
                for (; off < end; off += 16384ull) {
                    const unsigned long long len = end - off < 16384ull ? end - off : 16384ull;
                    asm volatile("cp.async.bulk.prefetch.L2.global [%0], %1;" ::"l"(pp[t] + off), "r"((uint32_t)(len & ~15ull)) : "memory");
                }
            }
        }
        __syncwarp();
        return;
    }

    mbar_wait(xfull, 0);
    if (norm) {
        // ------------------------------------------------------------------ RMSNorm prologue on the resident rows
        // thread -> (row, group); a group walks the (k-block, 16-byte chunk) pairs g, g + G, ...  Lanes of a warp hold
        // consecutive rows of the same chunk: with the 128-byte swizzle that is the conflict-free pattern for 128-bit accesses.
        const int row = tid % RB, grp = tid / RB, G = kConsumers / RB;
        const int npairs = a.nkb * 8;
        if (tid == 0) DX_TRACE(5);
        float ss = 0.f;
        for (int j = grp; j < npairs; j += G) {
            const int kb = j >> 3, c = j & 7;
            const uint4 v = *reinterpret_cast<const uint4*>(xres + (size_t)kb * xtile + row * 128 + ((c ^ (row & 7)) << 4));
            const uint32_t w[4] = {v.x, v.y, v.z, v.w};
#pragma unroll
            for (int e = 0; e < 4; ++e) {
                const float lo = __uint_as_float(w[e] << 16), hi = __uint_as_float(w[e] & 0xffff0000u);
                ss = fmaf(lo, lo, ss);
                ss = fmaf(hi, hi, ss);
            }
        }
        red[grp * RB + row] = ss;
        wg::consumer_sync();
        if (tid < RB) {
            float tot = 0.f;
            for (int g2 = 0; g2 < G; ++g2) tot += red[g2 * RB + tid];      // fixed order: deterministic
            rstd_s[tid] = 1.0f / sqrtf(tot / (float)a.K + a.eps);
        }
        wg::consumer_sync();
        const float rs = rstd_s[row];
        for (int j = grp; j < npairs; j += G) {
            const int kb = j >> 3, c = j & 7;
            uint4* px = reinterpret_cast<uint4*>(xres + (size_t)kb * xtile + row * 128 + ((c ^ (row & 7)) << 4));
            const uint4 v = *px;
            const uint4 gw = *reinterpret_cast<const uint4*>(gbuf + kb * kBK + c * 8);
            const uint32_t w[4] = {v.x, v.y, v.z, v.w}, gq[4] = {gw.x, gw.y, gw.z, gw.w};
            uint32_t o[4];
#pragma unroll
            for (int e = 0; e < 4; ++e) {
                // output = norm(x.float()).type_as(x) * weight: two bf16 roundings (gpt.py:147-148)
                const float lo = __uint_as_float(w[e] << 16) * rs, hi = __uint_as_float(w[e] & 0xffff0000u) * rs;
                o[e] = mul_bf16x2(pack_rn(lo, hi), gq[e]);
            }
            *px = make_uint4(o[0], o[1], o[2], o[3]);
        }
        fence_proxy_async();          // generic-proxy writes -> visible to the tensor core's async-proxy reads
        wg::consumer_sync();
    }

    // ---------------------------------------------------------------------- MMA: warpgroup g owns features [64 g, 64 g + 64)
    if (tid == 0) DX_TRACE(6);
    const int g = warp >> 2;
    float acc[RB / 2];
#pragma unroll
    for (int i = 0; i < RB / 2; ++i) acc[i] = 0.f;
    for (int i = 0; i < a.nkb; ++i) {
        const int s = i % a.stages;
        mbar_wait(&full[s], (uint32_t)((i / a.stages) & 1));
        if (i == a.nkb - 1 && tid == 0) DX_TRACE(7);
        wg::fence_regs<RB / 2>(acc);
        wg::fence();
        wg::mma_kblock<RB>(acc, smem_u32(ring + (size_t)s * kWBytes) + g * (kWBytes / 2), smem_u32(xres + (size_t)i * xtile));
        wg::commit();
        wg::wait<1>();
        wg::fence_regs<RB / 2>(acc);
        if (i > 0 && (tid & 127) == 0) mbar_arrive(&empty[(i - 1) % a.stages]);
    }
    wg::wait<0>();
    wg::fence_regs<RB / 2>(acc);
    if (tid == 0) DX_TRACE(8);

    // ---------------------------------------------------------------------- epilogue from registers
    if (a.mode == DX_SWIGLU) {
        float* stash = reinterpret_cast<float*>(ring);               // [RB][64] fp32, free once both warpgroups' MMAs retired
        wg::consumer_sync();
        if (g == 1) {
#pragma unroll
            for (int i = 0; i < RB / 2; ++i) stash[wg::frag_col(i) * 64 + wg::frag_row(i)] = round_bf16(acc[i]);
        }
        wg::consumer_sync();
        if (g == 0) {
#pragma unroll
            for (int i = 0; i < RB / 2; ++i) {
                const int c = wg::frag_col(i), nl = wg::frag_row(i);
                if (c < Mb) {
                    const float av = round_bf16(acc[i]), bv = stash[c * 64 + nl];
                    const float sv = round_bf16(av / (1.0f + expf(-av)));
                    a.ff[(size_t)(row0 + c) * a.N + (size_t)nt * 64 + nl] = __float2bfloat16_rn(sv * bv);
                }
            }
        }
    } else {
#pragma unroll
        for (int i = 0; i < RB / 2; ++i) {
            const int c = wg::frag_col(i);
            const size_t n = (size_t)nt * kTileN + 64 * g + wg::frag_row(i);
            if (c >= Mb) continue;
            const size_t o = (size_t)(row0 + c) * a.N + n;
            if (a.mode == DX_RESID) a.h[o] = __float2bfloat16_rn(__bfloat162float(a.h[o]) + round_bf16(acc[i]));
            else a.out_f32[o] = acc[i];
        }
    }
    if (tid == 0) DX_TRACE(9);
}

int pick_rblk(int M, int K) {
    const int nkb = cdiv(K, kBK);
    int r = lg_env_flag("LG_DX_RBLK", 32);
    r = r >= 64 ? 64 : (r >= 32 ? 32 : 16);
    while (r > 16 && (r / 2 >= M || (size_t)r * 128 * nkb > kMaxXBytes)) r >>= 1;
    return r;
}

}  // namespace

static unsigned long long* g_dx_trace = nullptr;
extern "C" void lg_debug_set_dx_trace(unsigned long long* dev_buf) { g_dx_trace = dev_buf; }

bool gemm_dx_supported(int M, int N, int K, int dtype, int mode, bool norm) {
    if (dtype != LG_DTYPE_BF16 || M < 1 || K % 8 != 0 || K > 8192) return false;
    if (mode == DX_SWIGLU ? (N % 64 != 0) : (N % kTileN != 0)) return false;
    const int nkb = cdiv(K, kBK);
    if ((size_t)16 * 128 * nkb > kMaxXBytes) return false;             // the row block must stay resident over all of K
    (void)norm;
    return true;
}

template <int RB>
static int launch_dx_t(const CUtensorMap& mwa, const CUtensorMap& mwb, const CUtensorMap& mx, const DxArgs& a, dim3 grid,
                       size_t smem, cudaStream_t st) {
    static DevOnce attr;
    if (lg_first_on_device(attr)) {
        LG_CUDA_OK(cudaFuncSetAttribute(gemm_dx_kernel<RB>, cudaFuncAttributeMaxDynamicSharedMemorySize, 227 * 1024));
    }
    (void)lg_launch(gemm_dx_kernel<RB>, grid, dim3(kThreadsDx), smem, st, mwa, mwb, mx, a);
    LG_LAUNCH_CHECK();
    return 0;
}

int launch_gemm_dx(const GemmDx& g, cudaStream_t st, const GemmNext* next) {
    const bool norm = g.normw != nullptr;
    LG_REQUIRE(gemm_dx_supported(g.M, g.N, g.K, LG_DTYPE_BF16, g.mode, norm), "gemm_dx: unsupported shape %d %d %d mode %d", g.M, g.N, g.K, g.mode);
    const bool paired = g.mode == DX_SWIGLU;
    LG_REQUIRE(!paired || g.Wb, "gemm_dx: the SwiGLU form needs two weight matrices");
    LG_REQUIRE(((uintptr_t)g.X & 15) == 0 && ((uintptr_t)g.Wa & 15) == 0 && (!g.Wb || ((uintptr_t)g.Wb & 15) == 0) && g.ldx % 8 == 0,
               "gemm_dx: operands must be 16-byte aligned");
    LG_REQUIRE((g.mode == DX_F32 && g.out_f32) || (g.mode == DX_RESID && g.h) || (g.mode == DX_SWIGLU && g.ff), "gemm_dx: missing output");
    DxArgs a{};
    a.M = g.M; a.N = g.N; a.K = g.K;
    const int rblk = pick_rblk(g.M, g.K);
    a.nkb = cdiv(g.K, kBK);
    a.mode = g.mode; a.paired = paired ? 1 : 0;
    a.normw = (const bf16*)g.normw; a.eps = g.eps;
    a.out_f32 = g.out_f32; a.h = (bf16*)g.h; a.ff = (bf16*)g.ff;
    const size_t xbytes = (size_t)a.nkb * rblk * 128;
    const size_t fixed = 1024 + xbytes + kMiscBytes + (norm ? (size_t)a.nkb * kBK * 2 : 0) + 64;
    int stages = (int)std::min<size_t>(kMaxSt, (227 * 1024 - fixed) / kWBytes);
    stages = std::min(stages, std::max(2, lg_env_flag("LG_DX_STAGES", kMaxSt)));
    stages = std::min(stages, std::max(2, a.nkb));
    LG_REQUIRE(stages >= 2, "gemm_dx: no room for a 2-stage weight ring (K = %d)", g.K);
    a.stages = stages;
    const bool pf = next && lg_env_flag("LG_L2_PREFETCH", 1);
    a.pf0 = pf ? (const char*)next->p0 : nullptr; a.pfb0 = pf ? next->b0 : 0;
    a.pf1 = pf ? (const char*)next->p1 : nullptr; a.pfb1 = pf ? next->b1 : 0;
    a.trace = g_dx_trace;

    CUtensorMap mwa, mwb, mx;
    const int wbox = paired ? kTileN / 2 : kTileN;
    LG_TRY(tma::make_map_2d(&mwa, g.Wa, (uint64_t)g.N, (uint64_t)g.K, (uint64_t)g.K, wbox, kBK));
    LG_TRY(tma::make_map_2d(&mwb, paired ? g.Wb : g.Wa, (uint64_t)g.N, (uint64_t)g.K, (uint64_t)g.K, wbox, kBK));
    LG_TRY(tma::make_map_2d(&mx, g.X, (uint64_t)g.M, (uint64_t)g.K, (uint64_t)g.ldx, (uint32_t)rblk, kBK));   // rows >= M read as zero

    const size_t smem = fixed + (size_t)stages * kWBytes;
    LG_REQUIRE(smem <= 227 * 1024, "gemm_dx: shared memory %zu too large", smem);
    dim3 grid(paired ? g.N / 64 : g.N / kTileN, cdiv(g.M, rblk));
    LG_REQUIRE(grid.y <= 65535, "gemm_dx: too many row blocks");
    if (rblk == 16) return launch_dx_t<16>(mwa, mwb, mx, a, grid, smem, st);
    if (rblk == 32) return launch_dx_t<32>(mwa, mwb, mx, a, grid, smem, st);
    return launch_dx_t<64>(mwa, mwb, mx, a, grid, smem, st);
}
