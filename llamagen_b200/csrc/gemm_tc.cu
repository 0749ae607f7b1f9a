// Hopper weight-streaming GEMM: wgmma with the accumulator in registers, operands staged in shared memory by TMA
// (cp.async.bulk.tensor) through an mbarrier full/empty ring.
//
//   y[r, n] = sum_k x[r, k] * W[n, k]        (nn.Linear without bias, gpt.py:161-163,199-200,287)
//
// "Swap-AB" orientation for decode: the WEIGHT tile is the MMA A operand (128 output features = two warpgroups of
// M = 64), the activations are the B operand (N = rows padded to a power of two in [16, 256]), so a skinny batch never
// wastes the 64-row MMA shape and each CTA streams a [128 x Kslice] weight slab from HBM exactly once. One CTA = one
// (n-tile, k-slice); split-K slabs (fp32) are reduced by the row-wise epilogue kernels in xf_kernels.cu, exactly like the
// mma.sync path (gemm.cu).
//
// Warp roles (288 threads): warps 0-7 = two consumer warpgroups (features [0, 64) and [64, 128) of the tile), warp 8 = TMA
// producer (one elected lane). Each consumer warpgroup stores its accumulator straight from registers into the fp32 slab.
//
// fp8 weights (W8 instantiations, LG_DTYPE_E4M3 codes + one fp32 power-of-two scale per weight row, see the layout in
// include/llamagen_b200.h): the weight stage is a [128 x 64] byte tile written by TMA with the 64-byte swizzle, half the bytes of the
// 16-bit tile. The consumers do not hand it to the MMA through a descriptor: each thread reads the two 16-byte pieces that hold
// its A fragments of the whole k-block (the stored K order makes them contiguous), widens them exactly to T (e4m3x2_to<T>) and
// issues the k-block's four wgmma with A from registers as one group, which it waits for before it widens the next k-block (the
// next k-block's bytes are fetched from shared memory while the group runs); B (activations) and everything else are as in the
// 16-bit kernel. The drain multiplies
// accumulator row n by scale[n] before the slab store, so the slabs hold what a 16-bit GEMM on the dequantised weight would.
#include "kernels.cuh"
#include "tma_utils.cuh"
#include "wgmma_utils.cuh"
#include <mutex>
#include <unordered_map>

namespace {

constexpr int kBlockN = 128;    // weight rows per CTA (two warpgroups of M = 64)
constexpr int kBlockK = 64;     // bf16 elements per k-block = 128 B = one swizzle-128B row
constexpr int kMaxStages = 8;   // barrier slots in shared memory
constexpr int kRingStages = 4;  // stages the host launches with (fewer when a CTA owns fewer k-blocks)
constexpr int kTargetCtas = 92; // split-K CTA target per GEMM (~0.7 per SM of an H100)
constexpr int kThreads = 288;   // 2 consumer warpgroups + 1 producer warp
constexpr int kATileBytes = kBlockN * kBlockK * 2;   // 16 KB
constexpr int kATileBytesW8 = kBlockN * kBlockK;     // 8 KB of e4m3 codes
constexpr int kMaxRowsPerCta = 256;                  // wgmma N <= 256

using namespace tma;

struct TcArgs {
    int M, N, K;          // activations rows, weight rows, reduction
    int n_split;          // weight rows [0, n_split) come from map_wa, the rest from map_wb
    int rblk;             // rows per row block (== M when gridDim.z == 1); M > 256 is cut into gridDim.z blocks of rblk rows
    int kblocks_per_split;
    int stages;           // smem ring depth (<= kMaxStages)
    float* partial;       // [ksplit][M][N]
    const char* pf0; unsigned long long pfb0;   // next GEMM's weights to pull into L2 (see GemmNext)
    const char* pf1; unsigned long long pfb1;
    unsigned long long whint;    // L2 eviction hint of the weight tiles (0: default policy)
    const float* sca; const float* scb;   // fp8 weights: the row scales of the two weight segments
};

// RP: rows of one row block padded to a power of two (wgmma N); the activation box has RP rows, rows >= M read as zero.
// T: operand type (bf16 or f16), only the wgmma instruction depends on it. W8: the weight maps are e4m3 code maps.
template <int RP, typename T, bool W8>
__global__ void __launch_bounds__(kThreads, 1) gemm_tc_kernel(const __grid_constant__ CUtensorMap map_wa,
                                                              const __grid_constant__ CUtensorMap map_wb,
                                                              const __grid_constant__ CUtensorMap map_x, TcArgs a) {
    extern __shared__ __align__(1024) uint8_t smem_raw[];
    constexpr int b_tile_bytes = RP * kBlockK * 2;
    constexpr int a_tile_bytes = W8 ? kATileBytesW8 : kATileBytes;
    constexpr int stage_bytes = a_tile_bytes + ((b_tile_bytes + 1023) / 1024) * 1024;
    uint8_t* tiles = reinterpret_cast<uint8_t*>(((uintptr_t)smem_raw + 1023) & ~(uintptr_t)1023);
    const int kStages = a.stages;
    uint64_t* full_bar = reinterpret_cast<uint64_t*>(tiles + kStages * stage_bytes);
    uint64_t* empty_bar = full_bar + kMaxStages;

    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    const int n0 = blockIdx.x * kBlockN;
    const int ks = blockIdx.y;
    const int row0 = (int)blockIdx.z * a.rblk;               // first activation row of this CTA's row block (t2i prefill: M = R*120)
    const int Mb = min(a.rblk, a.M - row0);                  // valid rows in the block
    const int total_kb = (a.K + kBlockK - 1) / kBlockK;
    const int kb0 = ks * a.kblocks_per_split;
    const int nkb = max(0, min(a.kblocks_per_split, total_kb - kb0));

    if (warp == 8 && lane == 0) {
        prefetch_map(&map_wa);
        prefetch_map(&map_wb);
        prefetch_map(&map_x);
        for (int s = 0; s < kStages; ++s) { mbar_init(&full_bar[s], 1); mbar_init(&empty_bar[s], 2); }
        fence_barrier_init();
    }
    __syncthreads();
    lg_pdl_launch_dependents();
    if (warp != 8) lg_pdl_wait();   // the producer waits after it has requested the first weight tiles

    if (warp == 8) {
        // ------------------------------------------------------------------ TMA producer
        if (elect_one()) {
            const bool second = n0 >= a.n_split;
            const CUtensorMap* wmap = second ? &map_wb : &map_wa;
            const int wrow = second ? n0 - a.n_split : n0;
            const uint32_t tx = (uint32_t)(a_tile_bytes + b_tile_bytes);
            // Weights do not depend on the previous kernel: the first ring of weight tiles is requested BEFORE
            // the programmatic-dependency wait, so the HBM stream of this GEMM overlaps the tail of its producer.
            const int npre = min(nkb, kStages);
            for (int i = 0; i < npre; ++i) {
                mbar_expect_tx(&full_bar[i], tx);
                load_2d_hint(tiles + i * stage_bytes, wmap, &full_bar[i], (kb0 + i) * kBlockK, wrow, a.whint);
            }
            lg_pdl_wait();
            for (int i = 0; i < npre; ++i)
                load_2d(tiles + i * stage_bytes + a_tile_bytes, &map_x, &full_bar[i], (kb0 + i) * kBlockK, row0);
            for (int i = npre; i < nkb; ++i) {
                const int s = i % kStages;
                const uint32_t ph = (uint32_t)((i / kStages) & 1);
                mbar_wait(&empty_bar[s], ph ^ 1);
                mbar_expect_tx(&full_bar[s], tx);
                uint8_t* sa = tiles + s * stage_bytes;
                load_2d_hint(sa, wmap, &full_bar[s], (kb0 + i) * kBlockK, wrow, a.whint);
                load_2d(sa + a_tile_bytes, &map_x, &full_bar[s], (kb0 + i) * kBlockK, row0);
            }
            // ask L2 for this CTA's share of the next GEMM's weights (static chain: qkv -> wo -> w1|w3 -> w2 -> next qkv)
            {
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
        }
        __syncwarp();
        return;
    }
    // ---------------------------------------------------------------------- consumers: warpgroup g owns features [64 g, 64 g + 64)
    const int g = warp >> 2;
    float acc[RP / 2];
#pragma unroll
    for (int i = 0; i < RP / 2; ++i) acc[i] = 0.f;
    float sc[2] = {1.f, 1.f};   // fp8: the scales of accumulator rows frag_row(i), one per value of (i >> 1) & 1
    if constexpr (W8) {
        const bool second = n0 >= a.n_split;
        const float* sp = (second ? a.scb + (n0 - a.n_split) : a.sca + n0) + 64 * g + wg::frag_row(0);
        sc[0] = __ldg(sp);
        sc[1] = __ldg(sp + 8);
        // This thread's A fragments of one k-block: rows r and r + 8 of the warpgroup's half tile, 16-byte piece q = lane % 4 of the 64-byte row
        // (TMA's 64-byte swizzle XORs the piece index with bits 7-8 of the address, the same for both rows).
        const int r = 64 * g + wg::frag_row(0), q = lane & 3;
        const uint32_t aoff = (uint32_t)(r * kBlockK + ((q ^ ((r >> 1) & 3)) << 4));
        // One k-block: widen the raw pieces into the A registers, issue its four MMAs as one group, fetch the next k-block's raw pieces from
        // shared memory while they run, then wait for the group. The A registers are written only while no wgmma is in flight (ptxas
        // serialises every wgmma of a pipeline stage in which another instruction defines one of its input registers); the raw pieces
        // are ordinary registers, so the full-barrier wait and the shared-memory latency of k-block i + 1 overlap the MMAs of k-block i.
        auto fetch = [&](int i, uint4& lo, uint4& hi) {
            const int s = i % kStages;
            mbar_wait(&full_bar[s], (uint32_t)((i / kStages) & 1));
            const uint8_t* wt = tiles + s * stage_bytes;
            lo = *reinterpret_cast<const uint4*>(wt + aoff);
            hi = *reinterpret_cast<const uint4*>(wt + aoff + 8 * kBlockK);
        };
        uint4 lo = make_uint4(0u, 0u, 0u, 0u), hi = lo;
        if (nkb > 0) fetch(0, lo, hi);
        for (int i = 0; i < nkb; ++i) {
            const uint32_t wl[4] = {lo.x, lo.y, lo.z, lo.w}, wh[4] = {hi.x, hi.y, hi.z, hi.w};
            const int s = i % kStages;
            const uint64_t bd = wg::make_desc_sw128(smem_u32(tiles + s * stage_bytes + a_tile_bytes));
            // MMAs per group: the whole k-block, but two for the 256-row tile, whose 128 accumulators leave room for 8 A registers
            // under the 168-register ceiling of a 288-thread CTA (with 16, ptxas serialises every wgmma for lack of registers)
            constexpr int G = RP == 256 ? 2 : 4;
#pragma unroll
            for (int k0 = 0; k0 < 4; k0 += G) {
                uint32_t af[4 * G];
#pragma unroll
                for (int k = 0; k < G; ++k) {   // word k: codes of k = 16k + 2q, +1 (low half) and 16k + 8 + 2q, +1 (high half)
                    af[4 * k + 0] = e4m3x2_to<T>(wl[k0 + k]);
                    af[4 * k + 1] = e4m3x2_to<T>(wh[k0 + k]);
                    af[4 * k + 2] = e4m3x2_to<T>(wl[k0 + k] >> 16);
                    af[4 * k + 3] = e4m3x2_to<T>(wh[k0 + k] >> 16);
                }
                wg::fence_regs<RP / 2>(acc);
                wg::fence();
#pragma unroll
                for (int k = 0; k < G; ++k) wg::WgmmaRS<RP, T>::mma(acc, af + 4 * k, bd + (uint64_t)(2 * (k0 + k)));
                wg::commit();
                if (k0 + G < 4) {
                    wg::wait<0>();
                    wg::fence_regs<RP / 2>(acc);
                }
            }
            // the 256-row tile has no registers to spare for raw pieces beside 128 accumulators (ptxas would serialise its wgmma):
            // it fetches after the wait
            if (RP < 256 && i + 1 < nkb) fetch(i + 1, lo, hi);
            wg::wait<0>();                              // this k-block's MMAs have retired (its weight bytes left the stage before them)
            wg::fence_regs<RP / 2>(acc);
            if (RP == 256 && i + 1 < nkb) fetch(i + 1, lo, hi);
            if ((threadIdx.x & 127) == 0) mbar_arrive(&empty_bar[s]);
        }
    } else {
        for (int i = 0; i < nkb; ++i) {
            const int s = i % kStages;
            const uint32_t ph = (uint32_t)((i / kStages) & 1);
            mbar_wait(&full_bar[s], ph);
            const uint32_t sa = smem_u32(tiles + s * stage_bytes);
            wg::fence_regs<RP / 2>(acc);
            wg::fence();
            wg::mma_kblock<RP, T>(acc, sa + g * (kATileBytes / 2), sa + kATileBytes);
            wg::commit();
            wg::wait<1>();                                  // the previous k-block's MMAs have retired: release its stage
            wg::fence_regs<RP / 2>(acc);
            if (i > 0 && (threadIdx.x & 127) == 0) mbar_arrive(&empty_bar[(i - 1) % kStages]);
        }
    }
    wg::wait<0>();
    wg::fence_regs<RP / 2>(acc);
    // ---------------------------------------------------------------------- drain: registers -> fp32 slab [row][feature]
    float* out = a.partial + (size_t)ks * a.M * a.N + (size_t)row0 * a.N;
#pragma unroll
    for (int i = 0; i < RP / 2; ++i) {
        const int n = n0 + 64 * g + wg::frag_row(i), r = wg::frag_col(i);
        if (n < a.N && r < Mb) out[(size_t)r * a.N + n] = W8 ? acc[i] * sc[(i >> 1) & 1] : acc[i];
    }
}

// ---------------------------------------------------------------------------------------------- host side
}  // namespace

namespace tma {
typedef CUresult (*EncodeTiledFn)(CUtensorMap*, CUtensorMapDataType, cuuint32_t, void*, const cuuint64_t*, const cuuint64_t*,
                                  const cuuint32_t*, const cuuint32_t*, CUtensorMapInterleave, CUtensorMapSwizzle,
                                  CUtensorMapL2promotion, CUtensorMapFloatOOBfill);
static EncodeTiledFn get_encode() {
    static EncodeTiledFn fn = nullptr;
    static std::once_flag once;
    std::call_once(once, [] {
        void* p = nullptr;
        cudaDriverEntryPointQueryResult q;
        if (cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &p, cudaEnableDefault, &q) == cudaSuccess &&
            q == cudaDriverEntryPointSuccess)
            fn = (EncodeTiledFn)p;
    });
    return fn;
}
int make_map_2d(CUtensorMap* m, const void* base, uint64_t rows, uint64_t cols, uint64_t ld_elems, uint32_t box_rows,
                uint32_t box_cols, int dtype) {
    EncodeTiledFn enc = get_encode();
    LG_REQUIRE(enc, "cuTensorMapEncodeTiled is not available from the driver");
    LG_REQUIRE(lg_dtype_is16(dtype) || dtype == LG_DTYPE_E4M3, "make_map_2d: dtype %d has no tensor map", dtype);
    const DtypeInfo di = lg_dtype_info(dtype);
    cuuint64_t dims[2] = {cols, rows};
    cuuint64_t strides[1] = {ld_elems * (cuuint64_t)di.esz};
    cuuint32_t box[2] = {box_cols, box_rows};
    cuuint32_t estr[2] = {1, 1};
    // 128-byte swizzle; fp8 KV boxes of 64 bytes use the 64-byte swizzle
    const CUtensorMapSwizzle swz = box_cols * di.esz == 64 && dtype == LG_DTYPE_E4M3 ? CU_TENSOR_MAP_SWIZZLE_64B : CU_TENSOR_MAP_SWIZZLE_128B;
    CUresult r = enc(m, di.tma, 2, const_cast<void*>(base), dims, strides, box, estr,
                     CU_TENSOR_MAP_INTERLEAVE_NONE, swz, CU_TENSOR_MAP_L2_PROMOTION_L2_256B,
                     CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
    LG_REQUIRE(r == CUDA_SUCCESS, "cuTensorMapEncodeTiled(2d) failed (%d) rows=%llu cols=%llu ld=%llu box=%ux%u", (int)r,
               (unsigned long long)rows, (unsigned long long)cols, (unsigned long long)ld_elems, box_rows, box_cols);
    return 0;
}
int make_map_nhwc(CUtensorMap* m, const void* base, uint64_t B, uint64_t H, uint64_t W, uint64_t C, uint32_t box_h,
                  uint32_t box_w, uint32_t box_c, uint32_t pixel_stride) {
    EncodeTiledFn enc = get_encode();
    LG_REQUIRE(enc, "cuTensorMapEncodeTiled is not available from the driver");
    cuuint64_t dims[4] = {C, W, H, B};
    cuuint64_t strides[3] = {C * 2, W * C * 2, H * W * C * 2};
    // pixel_stride s > 1: the box traverses s*box_w x s*box_h input pixels and keeps every s-th one (a strided conv's taps)
    cuuint32_t box[4] = {box_c, box_w * pixel_stride, box_h * pixel_stride, 1};
    cuuint32_t estr[4] = {1, pixel_stride, pixel_stride, 1};
    CUresult r = enc(m, CU_TENSOR_MAP_DATA_TYPE_BFLOAT16, 4, const_cast<void*>(base), dims, strides, box, estr,
                     CU_TENSOR_MAP_INTERLEAVE_NONE, CU_TENSOR_MAP_SWIZZLE_128B, CU_TENSOR_MAP_L2_PROMOTION_L2_256B,
                     CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
    LG_REQUIRE(r == CUDA_SUCCESS, "cuTensorMapEncodeTiled(4d) failed (%d) B=%llu H=%llu W=%llu C=%llu box=%ux%ux%u", (int)r,
               (unsigned long long)B, (unsigned long long)H, (unsigned long long)W, (unsigned long long)C, box_h, box_w, box_c);
    return 0;
}
}  // namespace tma

// Plan: number of k-slices so that (N/128) * ksplit is about kTargetCtas CTAs (fewer, fatter slices than one per SM halve the
// fp32 slab traffic), >= 2 k-blocks per slice.
int gemm_tc_ksplit(int M, int N, int K) {
    // row blocks (M > 256: t2i prefill) already multiply the CTA count
    const int tiles = cdiv(N, kBlockN) * cdiv(M, kMaxRowsPerCta), kb = cdiv(K, kBlockK);
    int ks = std::max(1, kTargetCtas / std::max(tiles, 1));
    ks = std::min(ks, std::max(1, kb / 2));
    return std::min(ks, 16);
}

template <int RP, typename T, bool W8>
static int gemm_tc_launch_t(const CUtensorMap& mwa, const CUtensorMap& mwb, const CUtensorMap& mx, TcArgs& a, dim3 grid,
                            bool pdl, cudaStream_t st) {
    constexpr int b_tile_bytes = RP * kBlockK * 2;
    constexpr int stage_bytes = (W8 ? kATileBytesW8 : kATileBytes) + ((b_tile_bytes + 1023) / 1024) * 1024;
    // 4 stages instead of filling shared memory: a CTA never owns more than ~8 k-blocks, and the smaller footprint lets the
    // PDL-launched next kernel become resident next to this one.
    static_assert(1024 + kRingStages * stage_bytes + 2 * kMaxStages * sizeof(uint64_t) <= 227 * 1024, "gemm_tc: ring too large");
    a.stages = std::min(kRingStages, std::max(2, a.kblocks_per_split));   // never more stages than k-blocks
    const size_t smem = 1024 + (size_t)a.stages * stage_bytes + 2 * kMaxStages * sizeof(uint64_t);
    static DevOnce attr;
    if (lg_first_on_device(attr)) {
        LG_CUDA_OK(cudaFuncSetAttribute(gemm_tc_kernel<RP, T, W8>, cudaFuncAttributeMaxDynamicSharedMemorySize, 227 * 1024));
    }
    (void)lg_launch_pdl(pdl, gemm_tc_kernel<RP, T, W8>, grid, dim3(kThreads), smem, st, mwa, mwb, mx, a);
    LG_LAUNCH_CHECK();
    return 0;
}

template <typename T, bool W8>
static int gemm_tc_launch(const void* X, int ldx, const void* Wa, const void* Wb, int n_split, int M, int N, int K,
                          const float* sca, const float* scb, const GemmPlan& p, float* partial, cudaStream_t st, const GemmNext* next,
                          bool pdl) {
    constexpr int dt = ElemTraits<T>::dtype, wdt = W8 ? LG_DTYPE_E4M3 : dt;
    if (Wb == nullptr) { Wb = Wa; scb = sca; n_split = N; }
    LG_REQUIRE(!W8 || (sca && scb && K % kBlockK == 0 && N % kBlockN == 0), "gemm_tc: fp8 weights need row scales, K %% 64 == 0 and N %% 128 == 0");
    LG_REQUIRE(p.kernel == 2, "gemm_tc: the call is planned on kernel %d", p.kernel);
    LG_REQUIRE(((uintptr_t)X & 15) == 0 && ((uintptr_t)Wa & 15) == 0 && ((uintptr_t)Wb & 15) == 0 && ldx % 8 == 0,
               "gemm_tc: operands must be 16-byte aligned");
    TcArgs a;
    a.M = M; a.N = N; a.K = K; a.n_split = n_split;
    a.rblk = M <= kMaxRowsPerCta ? M : kMaxRowsPerCta;
    const int zblocks = p.row_blocks;
    LG_REQUIRE(zblocks <= 65535, "gemm_tc: %d row blocks not launchable", zblocks);
    const int rpad = p.tile;
    const int ks = p.ksplit;
    const int kb = cdiv(K, kBlockK);
    a.kblocks_per_split = cdiv(kb, ks);
    a.partial = partial;

    CUtensorMap mwa, mwb, mx;
    LG_TRY(tma::make_map_2d(&mwa, Wa, (uint64_t)std::min(n_split, N), (uint64_t)K, (uint64_t)K, kBlockN, kBlockK, wdt));
    LG_TRY(tma::make_map_2d(&mwb, Wb, (uint64_t)std::max(N - n_split, Wb == Wa ? N : 1), (uint64_t)K, (uint64_t)K, kBlockN, kBlockK, wdt));
    LG_TRY(tma::make_map_2d(&mx, X, (uint64_t)M, (uint64_t)K, (uint64_t)ldx, (uint32_t)rpad, kBlockK, dt));   // rows >= M read as zero

    a.whint = 0ull;   // the weight tiles take the default L2 policy
    a.sca = sca; a.scb = scb;
    a.pf0 = next ? (const char*)next->p0 : nullptr; a.pfb0 = next ? next->b0 : 0;
    a.pf1 = next ? (const char*)next->p1 : nullptr; a.pfb1 = next ? next->b1 : 0;
    const dim3 grid(cdiv(N, kBlockN), ks, zblocks);
    switch (rpad) {
        case 16: return gemm_tc_launch_t<16, T, W8>(mwa, mwb, mx, a, grid, pdl, st);
        case 32: return gemm_tc_launch_t<32, T, W8>(mwa, mwb, mx, a, grid, pdl, st);
        case 64: return gemm_tc_launch_t<64, T, W8>(mwa, mwb, mx, a, grid, pdl, st);
        case 128: return gemm_tc_launch_t<128, T, W8>(mwa, mwb, mx, a, grid, pdl, st);
        default: return gemm_tc_launch_t<256, T, W8>(mwa, mwb, mx, a, grid, pdl, st);
    }
}

int gemm_tc_partial(const void* X, int ldx, const GemmWeight& wa, const GemmWeight& wb, int n_split, int M, int N, int K, int dtype,
                    const GemmPlan& p, float* partial, cudaStream_t st, const GemmNext* next, bool pdl) {
    LG_REQUIRE(lg_dtype_is16(dtype), "gemm_tc: unsupported dtype %d", dtype);
    if (wa.scale) {
        if (dtype == LG_DTYPE_F16) return gemm_tc_launch<f16, true>(X, ldx, wa.p, wb.p, n_split, M, N, K, wa.scale, wb.scale, p, partial, st, next, pdl);
        return gemm_tc_launch<bf16, true>(X, ldx, wa.p, wb.p, n_split, M, N, K, wa.scale, wb.scale, p, partial, st, next, pdl);
    }
    if (dtype == LG_DTYPE_F16) return gemm_tc_launch<f16, false>(X, ldx, wa.p, wb.p, n_split, M, N, K, nullptr, nullptr, p, partial, st, next, pdl);
    return gemm_tc_launch<bf16, false>(X, ldx, wa.p, wb.p, n_split, M, N, K, nullptr, nullptr, p, partial, st, next, pdl);
}
