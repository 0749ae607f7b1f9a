// Hopper implicit-GEMM convolution for the VQ decoder (vq_model.py:128-194):
//   out[pixel, co] = bias[co] + sum_{tap, ci} in[pixel + tap][ci] * W[co][tap][ci]  (+ residual)
// on wgmma tensor cores with the accumulator in registers.
//
//  * A operand (128 pixels = two warpgroups of M = 64): an 8x16-pixel patch x 64 channels of the bf16 NHWC activation,
//    fetched by ONE 4-D TMA box per (tap, channel chunk). The tap offset is just a signed shift of the box origin and the
//    3x3 zero padding is TMA's out-of-bounds fill — no im2col buffer, no address arithmetic on the SM.
//  * B operand (N = Cout tile, a power of two <= 128): the weight slab [Cout][tap*Cin + ci] (bf16, K-major), 2-D TMA.
//  * nearest-2x upsample + 3x3 conv (Upsample, vq_model.py:374-378) is evaluated as four 2x2 "phase" convolutions
//    on the low-resolution input with pre-summed weights: 16 tap-GEMMs instead of 36 (2.25x fewer FLOPs) and the
//    upsampled tensor never exists.
//  * epilogue: the consumer warpgroups add bias (+ residual) to their registers and write bf16 NHWC (or fp32 NCHW / uint8
//    for conv_out).
// Warp roles (288 threads): warps 0-7 = two consumer warpgroups, warp 8 = TMA producer.
#include "kernels.cuh"
#include "tma_utils.cuh"
#include "wgmma_utils.cuh"
#include <algorithm>

namespace {

using namespace tma;

constexpr int kPix = 128;          // pixels per tile (two warpgroups of M = 64)
constexpr int kCk = 64;            // channels per k-block (128 B)
constexpr int kConvThreads = 288;  // 2 consumer warpgroups + 1 producer warp
constexpr int kConvStages = 3;     // 3 x 32 KB -> two CTAs per SM overlap prologue / drain with the other's main loop
constexpr int kATile = kPix * kCk * 2;

struct ConvTcArgs {
    int B, Hin, Win, Cin, Hout, Wout, Cout;
    int mode;            // 0: 3x3 pad 1   1: 1x1   2: nearest-2x + 3x3 as 2x2 phase convs
                         // 3: Downsample (vq_model.py:389-397): 3x3 stride 2 over the input zero-padded right/bottom by one
    int Ht, Wt;          // extent of the pixel grid the patches tile: the input for modes 0-2, the output for mode 3
    int bh, bw;          // pixel patch, bh*bw == 128
    int tiles_x, tiles_y;
    int bn;              // Cout tile (power of two in [16, 128])
    int kchunks;         // Cin / 64
    int ntaps;           // 9, 1 or 4
    const float* bias;
    const bf16* residual;
    bf16* out_bf;
    float* out_nchw;
    uint8_t* out_u8;     // conv_out with the samplers' pixel finishing in the drain: uint8 NHWC [B][H][W][3] (sample_c2i_ddp.py:141-143)
    int gx, gy, gz;      // logical tile grid (pixel patches, Cout tiles, upsample phases); the launch grid is min(gx*gy*gz, CTA budget)
    float* gn_partial;   // conv_tcw_kernel: per (image, tile, group) sum / sum of squares of the bf16 OUTPUT for the following
    int gn_cpg;          // GroupNorm(32) (vq_model.py:279-314): [B][gn_splits][32][2], channels per group, tiles per image
    int gn_splits;
};

// TMA shift of the activation box for k-block i of a tile (tap = i / kchunks)
__device__ __forceinline__ void conv_tap_offset(const ConvTcArgs& a, int tap, int y0, int x0, int py, int px, int& dy, int& dx) {
    dy = 0; dx = 0;
    if (a.mode == 0) { dy = tap / 3 - 1; dx = tap % 3 - 1; }
    else if (a.mode == 2) { const int ta = tap >> 1, tb = tap & 1; dy = py == 0 ? ta - 1 : ta; dx = px == 0 ? tb - 1 : tb; }
    // mode 3: the map steps two input pixels per box element, so tap (ky, kx) of output patch (y0, x0) is the box
    // at input origin (2*y0 + ky, 2*x0 + kx); the right/bottom padding is TMA's out-of-bounds zero fill
    else if (a.mode == 3) { dy = y0 + tap / 3; dx = x0 + tap % 3; }
}

template <int BN>
__global__ void __launch_bounds__(kConvThreads, 2) conv_tc_kernel(const __grid_constant__ CUtensorMap amap,
                                                                  const __grid_constant__ CUtensorMap wmap, ConvTcArgs a) {
    extern __shared__ __align__(1024) uint8_t smem_raw[];
    constexpr int b_tile_bytes = BN * kCk * 2;
    constexpr int stage_bytes = kATile + ((b_tile_bytes + 1023) / 1024) * 1024;
    uint8_t* tiles = reinterpret_cast<uint8_t*>(((uintptr_t)smem_raw + 1023) & ~(uintptr_t)1023);
    uint64_t* full_bar = reinterpret_cast<uint64_t*>(tiles + kConvStages * stage_bytes);
    uint64_t* empty_bar = full_bar + kConvStages;

    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    const int tiles_per_img = a.tiles_x * a.tiles_y;
    const int nkb = a.ntaps * a.kchunks;
    const int total_tiles = a.gx * a.gy * a.gz;

    if (warp == 8 && lane == 0) {
        prefetch_map(&amap);
        prefetch_map(&wmap);
        for (int s = 0; s < kConvStages; ++s) { mbar_init(&full_bar[s], 1); mbar_init(&empty_bar[s], 2); }
        fence_barrier_init();
    }
    __syncthreads();

    // Persistent tile loop: CTA c processes tiles c, c + gridDim.x, ...  (tile = ((phase * gy) + cout_tile) * gx + pixel_patch).
    // With gridDim.x == total_tiles this is the one-tile-per-CTA kernel; a smaller grid caps how many SMs the decoder may occupy,
    // which is what lets the AR sampling of the next batch keep its latency while this batch is decoded (pipeline.py).
    uint32_t it0 = 0;                      // k-blocks issued / consumed before the current tile (ring position carries across tiles)
    for (int tile = blockIdx.x; tile < total_tiles; tile += gridDim.x, it0 += (uint32_t)nkb) {
    const int bxi = tile % a.gx, byz = tile / a.gx;
    const int b = bxi / tiles_per_img;
    const int trem = bxi - b * tiles_per_img;
    const int y0 = (trem / a.tiles_x) * a.bh, x0 = (trem % a.tiles_x) * a.bw;
    const int n0 = (byz % a.gy) * BN;
    const int phase = byz / a.gy, py = phase >> 1, px = phase & 1;

    if (warp == 8) {
        if (elect_one()) {
            const uint32_t tx = (uint32_t)(kATile + b_tile_bytes);
            for (int i = 0; i < nkb; ++i) {
                const uint32_t it = it0 + (uint32_t)i;
                const int s = (int)(it % kConvStages);
                const uint32_t ph = (it / kConvStages) & 1u;
                const int tap = i / a.kchunks, cc = i - tap * a.kchunks;
                int dy, dx;
                conv_tap_offset(a, tap, y0, x0, py, px, dy, dx);
                mbar_wait(&empty_bar[s], ph ^ 1);
                mbar_expect_tx(&full_bar[s], tx);
                uint8_t* sa = tiles + s * stage_bytes;
                load_4d(sa, &amap, &full_bar[s], cc * kCk, x0 + dx, y0 + dy, b);
                load_2d(sa + kATile, &wmap, &full_bar[s], tap * a.Cin + cc * kCk, phase * a.Cout + n0);
            }
        }
        __syncwarp();
        continue;
    }

    // ---------------------------------------------------------------------- consumers: warpgroup g owns pixels [64 g, 64 g + 64)
    const int g = warp >> 2;
    float acc[BN / 2];
#pragma unroll
    for (int i = 0; i < BN / 2; ++i) acc[i] = 0.f;
    for (int i = 0; i < nkb; ++i) {
        const uint32_t it = it0 + (uint32_t)i;
        const int s = (int)(it % kConvStages);
        mbar_wait(&full_bar[s], (it / kConvStages) & 1u);
        const uint32_t sa = smem_u32(tiles + s * stage_bytes);
        wg::fence_regs<BN / 2>(acc);
        wg::fence();
        wg::mma_kblock<BN>(acc, sa + g * (kATile / 2), sa + kATile);
        wg::commit();
        wg::wait<1>();
        wg::fence_regs<BN / 2>(acc);
        if (i > 0 && (threadIdx.x & 127) == 0) mbar_arrive(&empty_bar[(it - 1) % kConvStages]);
    }
    wg::wait<0>();
    wg::fence_regs<BN / 2>(acc);
    if (nkb > 0 && (threadIdx.x & 127) == 0) mbar_arrive(&empty_bar[(it0 + (uint32_t)nkb - 1) % kConvStages]);

    // ---------------------------------------------------------------------- epilogue: fragment row = pixel of the patch
#pragma unroll
    for (int i = 0; i < BN / 2; i += 2) {
        const int pix = 64 * g + wg::frag_row(i);
        const int iy = pix / a.bw, ix = pix - iy * a.bw;
        int oy = y0 + iy, ox = x0 + ix;
        if (oy >= a.Ht || ox >= a.Wt) continue;        // patches may overhang the image (TMA zero-filled the reads)
        if (a.mode == 2) { oy = 2 * oy + py; ox = 2 * ox + px; }
        const int n = n0 + wg::frag_col(i);            // even; (n, n + 1) are this thread's pair
        if (n >= a.Cout) continue;
        const bool two = n + 1 < a.Cout;
        const float f0 = acc[i] + a.bias[n], f1 = two ? acc[i + 1] + a.bias[n + 1] : 0.f;
        const size_t opix = ((size_t)b * a.Hout + oy) * a.Wout + ox;
        if (a.out_u8) {         // conv_out -> clamp(127.5*x + 128, 0, 255) -> uint8 NHWC, same two roundings as torch's mul then add
            a.out_u8[opix * a.Cout + n] = (uint8_t)fminf(fmaxf(__fadd_rn(__fmul_rn(127.5f, f0), 128.0f), 0.f), 255.f);
            if (two) a.out_u8[opix * a.Cout + n + 1] = (uint8_t)fminf(fmaxf(__fadd_rn(__fmul_rn(127.5f, f1), 128.0f), 0.f), 255.f);
            continue;
        }
        if (a.out_nchw) {       // conv_out: fp32 NCHW, Cout = 3
            a.out_nchw[(((size_t)b * a.Cout + n) * a.Hout + oy) * a.Wout + ox] = f0;
            if (two) a.out_nchw[(((size_t)b * a.Cout + n + 1) * a.Hout + oy) * a.Wout + ox] = f1;
            continue;
        }
        // bf16 NHWC: Cout % 16 == 0, so the pair is complete and 4-byte aligned
        float v0 = f0, v1 = f1;
        if (a.residual) {
            const uint32_t r = *reinterpret_cast<const uint32_t*>(a.residual + opix * a.Cout + n);
            v0 += __uint_as_float(r << 16);
            v1 += __uint_as_float(r & 0xffff0000u);
        }
        *reinterpret_cast<__nv_bfloat162*>(a.out_bf + opix * a.Cout + n) = __floats2bfloat162_rn(v0, v1);
    }
    }   // tile loop
}

// ---------------------------------------------------------------------------------------------------
// Weights-as-A variant for Cout % 128 == 0 (every ResnetBlock / Upsample / Downsample conv of the VQ models).
//
// A = the 128-row weight slab (two warpgroups of 64 output channels) and B = a 16x16-pixel patch (two 4-D TMA boxes =
// 256 pixels), so every wgmma is m64n256k16, the largest shape: the 64 x 16 A slice fetched from shared memory is reused
// across 256 pixels instead of 128.
//
// The drain goes through shared memory 64 pixels at a time (fp32 [64][128] in a retired B stage) so that global traffic
// stays 16-byte vectors along the NHWC channel axis and acc + bias + residual is rounded to bf16 once, as in the kernel above.
// ---------------------------------------------------------------------------------------------------
constexpr int kWStages = 2;                      // 2 x 48 KB
constexpr int kWATile = 128 * kCk * 2;           // weights: 128 couts x 64 ch = 16 KB
constexpr int kWBTile = 256 * kCk * 2;           // pixels: 256 x 64 ch = 32 KB (two 8x16 boxes)
constexpr int kWStage = kWATile + kWBTile;
// drain staging row stride (floats): 132 instead of 128 moves the 4 lanes that share a fragment row (columns 2 apart) to different
// banks; 64 rows x 132 floats = 33 KB spill 1 KB past stage 0's B tile into stage 1's A tile, which is also held during the drain
constexpr int kStgLd = 132;

__global__ void __launch_bounds__(kConvThreads, 1) conv_tcw_kernel(const __grid_constant__ CUtensorMap amap,
                                                                   const __grid_constant__ CUtensorMap wmap, ConvTcArgs a) {
    extern __shared__ __align__(1024) uint8_t smem_raw[];
    uint8_t* tiles = reinterpret_cast<uint8_t*>(((uintptr_t)smem_raw + 1023) & ~(uintptr_t)1023);
    uint64_t* full_bar = reinterpret_cast<uint64_t*>(tiles + kWStages * kWStage);
    uint64_t* empty_bar = full_bar + kWStages;
    float* bias_s = reinterpret_cast<float*>(empty_bar + kWStages);     // [128]

    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    const int tiles_per_img = a.tiles_x * a.tiles_y;
    const int nkb = a.ntaps * a.kchunks;
    const int total_tiles = a.gx * a.gy * a.gz;

    if (warp == 8 && lane == 0) {
        prefetch_map(&amap);
        prefetch_map(&wmap);
        for (int s = 0; s < kWStages; ++s) { mbar_init(&full_bar[s], 1); mbar_init(&empty_bar[s], 2); }
        fence_barrier_init();
    }
    __syncthreads();

    uint32_t it0 = 0;
    for (int tile = blockIdx.x; tile < total_tiles; tile += gridDim.x, it0 += (uint32_t)nkb) {
        const int bxi = tile % a.gx, byz = tile / a.gx;
        const int b = bxi / tiles_per_img;
        const int trem = bxi - b * tiles_per_img;
        const int y0 = (trem / a.tiles_x) * 16, x0 = (trem % a.tiles_x) * 16;      // 16x16-pixel patch
        const int n0 = (byz % a.gy) * 128;
        const int phase = byz / a.gy, py = phase >> 1, px = phase & 1;

        if (warp == 8) {
            if (elect_one()) {
                for (int i = 0; i < nkb; ++i) {
                    const uint32_t it = it0 + (uint32_t)i;
                    const int s = (int)(it % kWStages);
                    const uint32_t ph = (it / kWStages) & 1u;
                    const int tap = i / a.kchunks, cc = i - tap * a.kchunks;
                    int dy, dx;
                    conv_tap_offset(a, tap, y0, x0, py, px, dy, dx);
                    const int ys = a.mode == 3 ? 16 : 8;      // stride-2 map: coordinates are input pixels
                    mbar_wait(&empty_bar[s], ph ^ 1);
                    mbar_expect_tx(&full_bar[s], (uint32_t)kWStage);
                    uint8_t* sa = tiles + s * kWStage;
                    load_2d(sa, &wmap, &full_bar[s], tap * a.Cin + cc * kCk, phase * a.Cout + n0);
                    load_4d(sa + kWATile, &amap, &full_bar[s], cc * kCk, x0 + dx, y0 + dy, b);
                    load_4d(sa + kWATile + kWBTile / 2, &amap, &full_bar[s], cc * kCk, x0 + dx, y0 + dy + ys, b);
                }
            }
            __syncwarp();
            continue;
        }

        // ------------------------------------------------------------------ consumers: warpgroup g owns couts [64 g, 64 g + 64)
        const int g = warp >> 2;
        float acc[128];
#pragma unroll
        for (int i = 0; i < 128; ++i) acc[i] = 0.f;
        for (int i = 0; i < nkb; ++i) {
            const uint32_t it = it0 + (uint32_t)i;
            const int s = (int)(it % kWStages);
            mbar_wait(&full_bar[s], (it / kWStages) & 1u);
            const uint32_t sa = smem_u32(tiles + s * kWStage);
            wg::fence_regs<128>(acc);
            wg::fence();
            wg::mma_kblock<256>(acc, sa + g * (kWATile / 2), sa + kWATile);
            wg::commit();
            wg::wait<1>();
            wg::fence_regs<128>(acc);
            // the last two k-blocks do not release their stages through the ring: the drain reuses stage memory, so the
            // producer may only refill after both warpgroups have left the drain
            if (i > 0 && i - 1 < nkb - kWStages && (threadIdx.x & 127) == 0) mbar_arrive(&empty_bar[(it - 1) % kWStages]);
        }
        wg::wait<0>();
        wg::fence_regs<128>(acc);
        if (threadIdx.x < 128) bias_s[threadIdx.x] = n0 + (int)threadIdx.x < a.Cout ? a.bias[n0 + threadIdx.x] : 0.f;
        // both warpgroups' MMAs have retired and neither stage has been released (nkb >= kWStages), so all stage memory is idle:
        // staging buffer = the B half of stage 0 (+ 1 KB of stage 1)
        wg::consumer_sync();

        // ------------------------------------------------------------------ drain: 4 rounds of 64 pixels through shared memory
        float* stg = reinterpret_cast<float*>(tiles + kWATile);            // [64 pixels][kStgLd] fp32
        float gs[8], gq[8];                                                // GroupNorm statistics of this thread's 8 channels
#pragma unroll
        for (int j = 0; j < 8; ++j) { gs[j] = 0.f; gq[j] = 0.f; }
#pragma unroll
        for (int rnd = 0; rnd < 4; ++rnd) {
            // registers -> staging: the fragment columns [64 rnd, 64 rnd + 64) are registers [32 rnd, 32 rnd + 32)
#pragma unroll
            for (int j = 0; j < 32; ++j) {
                const int i = rnd * 32 + j;
                stg[(wg::frag_col(i) - rnd * 64) * kStgLd + 64 * g + wg::frag_row(i)] = acc[i];
            }
            wg::consumer_sync();
            // staging -> global: 64 pixels x 16 chunks of 8 channels; thread -> 4 chunks
#pragma unroll
            for (int u = 0; u < 4; ++u) {
                const int idx = u * 256 + (int)threadIdx.x;               // [0, 1024)
                const int pl = idx >> 4, c8 = (idx & 15) * 8;             // pixel inside the round, first of 8 channels
                const int n = rnd * 64 + pl;                               // pixel column of the tile: box = n / 128, row-major 8x16 inside
                const int iy = (n >> 7) * 8 + ((n & 127) >> 4), ix = n & 15;
                int oy = y0 + iy, ox = x0 + ix;
                if (oy >= a.Ht || ox >= a.Wt) continue;                   // the patch may overhang the image
                if (a.mode == 2) { oy = 2 * oy + py; ox = 2 * ox + px; }
                const size_t off = (((size_t)b * a.Hout + oy) * a.Wout + ox) * a.Cout + n0 + c8;
                const float4 f0 = *reinterpret_cast<const float4*>(stg + pl * kStgLd + c8);
                const float4 f1 = *reinterpret_cast<const float4*>(stg + pl * kStgLd + c8 + 4);
                float f[8] = {f0.x, f0.y, f0.z, f0.w, f1.x, f1.y, f1.z, f1.w};
#pragma unroll
                for (int j = 0; j < 8; ++j) f[j] += bias_s[c8 + j];
                if (a.residual) {
                    const uint4 r = *reinterpret_cast<const uint4*>(a.residual + off);
                    const uint32_t w[4] = {r.x, r.y, r.z, r.w};
#pragma unroll
                    for (int j = 0; j < 4; ++j) {
                        f[2 * j] += __uint_as_float(w[j] << 16);
                        f[2 * j + 1] += __uint_as_float(w[j] & 0xffff0000u);
                    }
                }
                uint32_t pk[4];
#pragma unroll
                for (int j = 0; j < 4; ++j) {
                    __nv_bfloat162 t = __floats2bfloat162_rn(f[2 * j], f[2 * j + 1]);
                    pk[j] = *reinterpret_cast<uint32_t*>(&t);
                }
                *reinterpret_cast<uint4*>(a.out_bf + off) = make_uint4(pk[0], pk[1], pk[2], pk[3]);
                if (a.gn_partial) {          // statistics of the values as stored (bf16), like gn_stats_kernel reading them back
#pragma unroll
                    for (int j = 0; j < 4; ++j) {
                        const float lo = __uint_as_float(pk[j] << 16), hi = __uint_as_float(pk[j] & 0xffff0000u);
                        gs[2 * j] += lo; gq[2 * j] = fmaf(lo, lo, gq[2 * j]);
                        gs[2 * j + 1] += hi; gq[2 * j + 1] = fmaf(hi, hi, gq[2 * j + 1]);
                    }
                }
            }
            wg::consumer_sync();
        }
        if (a.gn_partial) {
            // thread t owns channels (t & 15) * 8 .. +7 of the tile for 16 of its pixels: combine the 16 threads of a channel column
            // and the channels of a group in a fixed order (no atomics: decode_code stays bit-reproducible)
            float* part = stg;                                             // [256 threads][16]
#pragma unroll
            for (int j = 0; j < 8; ++j) { part[threadIdx.x * 16 + j] = gs[j]; part[threadIdx.x * 16 + 8 + j] = gq[j]; }
            wg::consumer_sync();
            const int ngrp = 128 / a.gn_cpg;
            if ((int)threadIdx.x < ngrp) {
                float ts = 0.f, tq = 0.f;
                for (int c = (int)threadIdx.x * a.gn_cpg; c < ((int)threadIdx.x + 1) * a.gn_cpg; ++c) {
                    const int col = c >> 3, ci = c & 7;
                    for (int j = 0; j < 16; ++j) { ts += part[(col + 16 * j) * 16 + ci]; tq += part[(col + 16 * j) * 16 + 8 + ci]; }
                }
                const int split = phase * tiles_per_img + trem;
                float* o = a.gn_partial + (((size_t)b * a.gn_splits + split) * 32 + (n0 / a.gn_cpg + (int)threadIdx.x)) * 2;
                o[0] = ts;
                o[1] = tq;
            }
            wg::consumer_sync();
        }
        // hand the stage memory back: the producer waits on the stage-empty barriers released here
        if ((threadIdx.x & 127) == 0) {
            const int nrel = nkb < kWStages ? nkb : kWStages;
            for (int i = nkb - nrel; i < nkb; ++i) mbar_arrive(&empty_bar[(it0 + (uint32_t)i) % kWStages]);
        }
    }
}

// W'[phase][co][a*2+b][ci] = sum of the 3x3 taps that land on input offset (a, b) for output parity (py, px)
__global__ void upsample_phase_weights_kernel(const float* __restrict__ w /*[Cout][Cin][3][3]*/, bf16* __restrict__ out,
                                              int cout, int cin) {
    const size_t total = (size_t)4 * cout * 4 * cin;
    for (size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (size_t)gridDim.x * blockDim.x) {
        const int ci = (int)(i % cin);
        const int t = (int)((i / cin) % 4);
        const int co = (int)((i / ((size_t)cin * 4)) % cout);
        const int p = (int)(i / ((size_t)cin * 4 * cout));
        const int py = p >> 1, px = p & 1, ta = t >> 1, tb = t & 1;
        // rows: py==0: a=0 -> ky {0}, a=1 -> ky {1,2};  py==1: a=0 -> ky {0,1}, a=1 -> ky {2}   (same for columns)
        const int ky0 = py == 0 ? (ta == 0 ? 0 : 1) : (ta == 0 ? 0 : 2), ky1 = py == 0 ? (ta == 0 ? 0 : 2) : (ta == 0 ? 1 : 2);
        const int kx0 = px == 0 ? (tb == 0 ? 0 : 1) : (tb == 0 ? 0 : 2), kx1 = px == 0 ? (tb == 0 ? 0 : 2) : (tb == 0 ? 1 : 2);
        float s = 0.f;
        for (int ky = ky0; ky <= ky1; ++ky)
            for (int kx = kx0; kx <= kx1; ++kx) s += w[(((size_t)co * cin + ci) * 3 + ky) * 3 + kx];
        out[i] = __float2bfloat16_rn(s);
    }
}

}  // namespace

int conv_tc_make_phase_weights(const float* w_f32, bf16* out, int cout, int cin, cudaStream_t st) {
    upsample_phase_weights_kernel<<<132 * 4, 256, 0, st>>>(w_f32, out, cout, cin);
    LG_LAUNCH_CHECK();
    return 0;
}

static int g_conv_cta_budget = 0;
void conv_tc_set_cta_budget(int ctas) { g_conv_cta_budget = ctas; }

bool conv_tc_supported(int Hin, int Win, int Cin, int Cout, int ksize, int up, bool nchw_out) {
    if (Cin % 64 != 0) return false;
    if (Win < 8 || Hin < 8) return false;
    if (!nchw_out && Cout % 16 != 0) return false;
    if (up && ksize != 3) return false;
    if (up == 2 && (Hin % 2 || Win % 2 || Win < 16 || Hin < 16)) return false;
    return ksize == 1 || ksize == 3;
}

template <int BN>
static int launch_conv_tc_t(const CUtensorMap& amap, const CUtensorMap& wmap, const ConvTcArgs& a, dim3 grid, cudaStream_t st) {
    constexpr int b_tile_bytes = BN * kCk * 2;
    constexpr int stage_bytes = kATile + ((b_tile_bytes + 1023) / 1024) * 1024;
    const size_t smem = 1024 + (size_t)kConvStages * stage_bytes + 2 * kConvStages * sizeof(uint64_t);
    static DevOnce attr;
    if (lg_first_on_device(attr)) {
        LG_CUDA_OK(cudaFuncSetAttribute(conv_tc_kernel<BN>, cudaFuncAttributeMaxDynamicSharedMemorySize, 110 * 1024));
    }
    LG_REQUIRE(smem <= 110 * 1024, "conv_tc: shared memory %zu too large", smem);
    conv_tc_kernel<BN><<<grid, kConvThreads, smem, st>>>(amap, wmap, a);
    LG_LAUNCH_CHECK();
    return 0;
}

// weights: up == 0 or 2 (stride-2 Downsample) -> [Cout][k*k][Cin] bf16 ; up == 1 -> phase weights [4][Cout][4][Cin] bf16
int launch_conv_tc(const bf16* in, int B, int Hin, int Win, int Cin, const bf16* weights, const float* bias, int Cout,
                   int ksize, int up, const bf16* residual, bf16* out_bf, float* out_nchw, cudaStream_t st, uint8_t* out_u8,
                   float* gn_partial, size_t gn_floats, int* gn_splits, int* path) {
    if (gn_splits) *gn_splits = 0;
    if (path) *path = 1;
    ConvTcArgs a;
    a.gn_partial = nullptr; a.gn_cpg = 0; a.gn_splits = 0;
    a.B = B; a.Hin = Hin; a.Win = Win; a.Cin = Cin; a.Cout = Cout;
    const bool down = up == 2;
    up = up == 1;
    a.Hout = up ? 2 * Hin : (down ? Hin / 2 : Hin); a.Wout = up ? 2 * Win : (down ? Win / 2 : Win);
    a.mode = up ? 2 : (down ? 3 : (ksize == 1 ? 1 : 0));
    a.ntaps = up ? 4 : ksize * ksize;
    a.Ht = down ? a.Hout : Hin; a.Wt = down ? a.Wout : Win;
    a.bw = a.Wt >= 16 ? 16 : 8;
    a.bh = kPix / a.bw;
    a.tiles_x = cdiv(a.Wt, a.bw);
    a.tiles_y = cdiv(a.Ht, a.bh);
    a.bn = 16;
    while (a.bn < 128 && a.bn < Cout) a.bn *= 2;
    a.kchunks = Cin / kCk;
    a.bias = bias; a.residual = residual; a.out_bf = out_bf; a.out_nchw = out_nchw; a.out_u8 = out_u8;

    CUtensorMap amap, wmap;
    LG_TRY(tma::make_map_nhwc(&amap, in, (uint64_t)B, (uint64_t)Hin, (uint64_t)Win, (uint64_t)Cin, (uint32_t)a.bh, (uint32_t)a.bw, kCk,
                              down ? 2u : 1u));
    const uint64_t wrows = (uint64_t)(up ? 4 : 1) * Cout, wcols = (uint64_t)a.ntaps * Cin;
    LG_TRY(tma::make_map_2d(&wmap, weights, wrows, wcols, wcols, (uint32_t)a.bn, kCk));

    // CTA budget: 0 = one CTA per tile; > 0 = persistent CTAs (lg_vq_set_cta_budget), e.g. 64 while the next batch samples
    const int budget = g_conv_cta_budget;
    // the weights-as-A kernel drains through its stage memory, which needs every stage held by the tile (>= kWStages k-blocks)
    if (Cout % 128 == 0 && a.Ht >= 16 && a.Wt >= 16 && out_bf && !out_nchw && !out_u8 && a.ntaps * a.kchunks >= kWStages &&
        lg_env_flag("LG_CONV_SWAP", 1)) {
        // weights-as-A kernel: 128 couts x a 16x16-pixel patch (two 8x16 boxes) per tile
        ConvTcArgs w = a;
        w.bw = 16; w.bh = 8;
        w.tiles_x = cdiv(a.Wt, 16); w.tiles_y = cdiv(a.Ht, 16);
        w.bn = 128;
        w.gx = B * w.tiles_x * w.tiles_y; w.gy = Cout / 128; w.gz = up ? 4 : 1;
        // GroupNorm(32) statistics of the output in the drain: every (image, tile, group) slot is written by exactly one CTA
        const int splits = w.tiles_x * w.tiles_y * w.gz, cpg = Cout / 32;
        if (gn_partial && gn_splits && Cout % 32 == 0 && 128 % cpg == 0 && (size_t)B * splits * 64 <= gn_floats && lg_env_flag("LG_GN_FUSE", 1)) {
            w.gn_partial = gn_partial; w.gn_cpg = cpg; w.gn_splits = splits;
            *gn_splits = splits;
        }
        CUtensorMap amap2, wmap2;
        LG_TRY(tma::make_map_nhwc(&amap2, in, (uint64_t)B, (uint64_t)Hin, (uint64_t)Win, (uint64_t)Cin, 8u, 16u, kCk, down ? 2u : 1u));
        const uint64_t wrows2 = (uint64_t)(up ? 4 : 1) * Cout, wcols2 = (uint64_t)a.ntaps * Cin;
        LG_TRY(tma::make_map_2d(&wmap2, weights, wrows2, wcols2, wcols2, 128u, kCk));
        const size_t smem2 = 1024 + (size_t)kWStages * kWStage + 2 * kWStages * sizeof(uint64_t) + 128 * sizeof(float);
        static DevOnce attr2;
        if (lg_first_on_device(attr2)) {
            LG_CUDA_OK(cudaFuncSetAttribute(conv_tcw_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, 110 * 1024));
        }
        LG_REQUIRE(smem2 <= 110 * 1024, "conv_tcw: shared memory %zu too large", smem2);
        const long long total2 = (long long)w.gx * w.gy * w.gz;
        LG_REQUIRE(total2 < (1ll << 31), "conv_tcw: too many tiles");
        dim3 grid2((unsigned)(budget > 0 ? std::min<long long>(total2, budget) : total2));
        conv_tcw_kernel<<<grid2, kConvThreads, smem2, st>>>(amap2, wmap2, w);
        LG_LAUNCH_CHECK();
        if (path) *path = 2;
        return 0;
    }
    a.gx = B * a.tiles_x * a.tiles_y; a.gy = cdiv(Cout, a.bn); a.gz = up ? 4 : 1;
    const long long total = (long long)a.gx * a.gy * a.gz;
    LG_REQUIRE(total < (1ll << 31), "conv_tc: too many tiles");
    dim3 grid((unsigned)(budget > 0 ? std::min<long long>(total, budget) : total));
    switch (a.bn) {
        case 16: return launch_conv_tc_t<16>(amap, wmap, a, grid, st);
        case 32: return launch_conv_tc_t<32>(amap, wmap, a, grid, st);
        case 64: return launch_conv_tc_t<64>(amap, wmap, a, grid, st);
        default: return launch_conv_tc_t<128>(amap, wmap, a, grid, st);
    }
}
