// Shared device/host helpers for the llamagen_b200 CUDA library (sm_90a only).
#pragma once
#include <cuda_runtime.h>
#include <cuda_bf16.h>
#include <cuda_fp16.h>
#include <cuda_fp8.h>
#include <cuda.h>
#include <stdint.h>
#include <string>
#include <cstdio>
#include <atomic>

#include "../../include/llamagen_b200.h"

typedef __nv_bfloat16 bf16;
typedef __half f16;

// The one place an LG_DTYPE_* becomes a storage format: element size in bytes and the TMA data type of the 16-bit tensor
// kernels (LG_DTYPE_F32 has no TMA path; its format is reported for completeness).
struct DtypeInfo {
    int esz;
    CUtensorMapDataType tma;
};
inline DtypeInfo lg_dtype_info(int dtype) {
    if (dtype == LG_DTYPE_F16) return {2, CU_TENSOR_MAP_DATA_TYPE_FLOAT16};
    if (dtype == LG_DTYPE_BF16) return {2, CU_TENSOR_MAP_DATA_TYPE_BFLOAT16};
    if (dtype == LG_DTYPE_E4M3) return {1, CU_TENSOR_MAP_DATA_TYPE_UINT8};   // fp8 KV cache: raw bytes, decoded in registers
    return {4, CU_TENSOR_MAP_DATA_TYPE_FLOAT32};
}
// bf16 and fp16 share every tensor-core kernel (same shared-memory layouts and MMA rates on sm_90a)
inline bool lg_dtype_is16(int dtype) { return dtype == LG_DTYPE_BF16 || dtype == LG_DTYPE_F16; }

// ---------------------------------------------------------------------------------------------
// host-side error plumbing: every extern "C" entry point returns <0 and records a message.
// ---------------------------------------------------------------------------------------------
std::string& lg_err_slot();
int lg_fail(const char* fmt, ...);
extern std::atomic<uint64_t> g_lg_launches;

#define LG_CUDA_OK(expr)                                                                         \
    do {                                                                                         \
        cudaError_t _e = (expr);                                                                 \
        if (_e != cudaSuccess) {                                                                 \
            (void)cudaGetLastError(); /* do not leave it behind for the next launch check */     \
            return lg_fail("%s:%d CUDA error %s: %s", __FILE__, __LINE__, #expr,                 \
                           cudaGetErrorString(_e));                                              \
        }                                                                                        \
    } while (0)

// LG_DEBUG_SYNC=1 synchronises after every launch and logs the launch site (hang / fault localisation).
bool lg_debug_sync();
#define LG_LAUNCH_CHECK()                                                                        \
    do {                                                                                         \
        g_lg_launches.fetch_add(1, std::memory_order_relaxed);                                   \
        cudaError_t _e = cudaGetLastError();                                                     \
        if (_e != cudaSuccess)                                                                   \
            return lg_fail("%s:%d kernel launch failed: %s", __FILE__, __LINE__,                 \
                           cudaGetErrorString(_e));                                              \
        if (lg_debug_sync()) {                                                                   \
            fprintf(stderr, "[lg] launched %s:%d ...", __FILE__, __LINE__);                      \
            fflush(stderr);                                                                      \
            _e = cudaDeviceSynchronize();                                                        \
            fprintf(stderr, " %s\n", cudaGetErrorString(_e));                                    \
            fflush(stderr);                                                                      \
            if (_e != cudaSuccess)                                                               \
                return lg_fail("%s:%d kernel failed: %s", __FILE__, __LINE__,                    \
                               cudaGetErrorString(_e));                                          \
        }                                                                                        \
    } while (0)

#define LG_TRY(expr)                                                                             \
    do {                                                                                         \
        int _r = (expr);                                                                         \
        if (_r < 0) return _r;                                                                   \
    } while (0)

#define LG_REQUIRE(cond, ...)                                                                    \
    do {                                                                                         \
        if (!(cond)) return lg_fail(__VA_ARGS__);                                                \
    } while (0)

static inline int cdiv(long long a, long long b) { return (int)((a + b - 1) / b); }

// Function attributes (dynamic shared memory opt-in, cluster size) are per device: one bit per device ordinal.
struct DevOnce { std::atomic<uint32_t> mask{0}; };
inline bool lg_first_on_device(DevOnce& o) {
    int d = 0;
    cudaGetDevice(&d);
    const uint32_t bit = 1u << (d & 31);
    return (o.mask.fetch_or(bit) & bit) == 0;
}
// Every extern "C" entry point that launches, allocates or records events runs on the engine's own device, whatever the
// caller's current device is (one process may hold engines on several GPUs).
struct DeviceGuard {
    int prev = -1;
    explicit DeviceGuard(int dev) {
        if (cudaGetDevice(&prev) != cudaSuccess) prev = -1;
        if (prev != dev) cudaSetDevice(dev); else prev = -1;
    }
    ~DeviceGuard() { if (prev >= 0) cudaSetDevice(prev); }
    DeviceGuard(const DeviceGuard&) = delete;
    DeviceGuard& operator=(const DeviceGuard&) = delete;
};

// ---------------------------------------------------------------------------------------------
// Programmatic dependent launch (PDL): every kernel of the decode step is launched with
// programmaticStreamSerializationAllowed so its CTAs are scheduled (and run their prologue) while the
// previous kernel drains; lg_pdl_sync() at the top of the kernel blocks until the producer grid's memory
// is visible. Inside the captured CUDA graph these become programmatic dependency edges.
// ---------------------------------------------------------------------------------------------
int lg_env_flag(const char* name, int dflt);
extern int g_lg_pdl;     // -1: read LG_PDL from the environment on first use
inline bool lg_pdl_enabled() {
    if (g_lg_pdl < 0) g_lg_pdl = lg_env_flag("LG_PDL", 1) ? 1 : 0;
    return g_lg_pdl == 1;
}
template <typename... KArgs, typename... Args>
inline cudaError_t lg_launch(void (*kern)(KArgs...), dim3 grid, dim3 block, size_t smem, cudaStream_t st, Args&&... args) {
    cudaLaunchConfig_t cfg = {};
    cfg.gridDim = grid;
    cfg.blockDim = block;
    cfg.dynamicSmemBytes = smem;
    cfg.stream = st;
    cudaLaunchAttribute attr[1];
    attr[0].id = cudaLaunchAttributeProgrammaticStreamSerialization;
    attr[0].val.programmaticStreamSerializationAllowed = lg_pdl_enabled() ? 1 : 0;
    cfg.attrs = attr;
    cfg.numAttrs = 1;
    return cudaLaunchKernelEx(&cfg, kern, KArgs(args)...);
}
#ifdef __CUDACC__
__device__ __forceinline__ void lg_pdl_wait() { asm volatile("griddepcontrol.wait;" ::: "memory"); }
__device__ __forceinline__ void lg_pdl_launch_dependents() { asm volatile("griddepcontrol.launch_dependents;" ::: "memory"); }
__device__ __forceinline__ void lg_pdl_sync() { lg_pdl_wait(); lg_pdl_launch_dependents(); }
#endif

// ---------------------------------------------------------------------------------------------
// element conversion. The reference keeps activations in the weight dtype, so every op output is
// rounded to T (bf16 RNE) exactly where torch would materialise a tensor.
// ---------------------------------------------------------------------------------------------
template <typename T> struct ElemTraits;
template <> struct ElemTraits<float> {
    static constexpr int dtype = LG_DTYPE_F32;
    __device__ __forceinline__ static float to_f(float v) { return v; }
    __device__ __forceinline__ static float from_f(float v) { return v; }
    __device__ __forceinline__ static float round(float v) { return v; }
};
template <> struct ElemTraits<bf16> {
    static constexpr int dtype = LG_DTYPE_BF16;
    __device__ __forceinline__ static float to_f(bf16 v) { return __bfloat162float(v); }
    __device__ __forceinline__ static bf16 from_f(float v) { return __float2bfloat16_rn(v); }
    __device__ __forceinline__ static float round(float v) { return __bfloat162float(__float2bfloat16_rn(v)); }
    // two packed elements <-> floats (element 0 in the low half)
    __device__ __forceinline__ static float lo(uint32_t w) { return __uint_as_float(w << 16); }
    __device__ __forceinline__ static float hi(uint32_t w) { return __uint_as_float(w & 0xffff0000u); }
    __device__ __forceinline__ static uint32_t pack2(float a, float b) {
        __nv_bfloat162 p = __floats2bfloat162_rn(a, b);
        return *reinterpret_cast<uint32_t*>(&p);
    }
};
// IEEE half: round-to-nearest-even, overflow to +-inf like torch (no saturation)
template <> struct ElemTraits<f16> {
    static constexpr int dtype = LG_DTYPE_F16;
    __device__ __forceinline__ static float to_f(f16 v) { return __half2float(v); }
    __device__ __forceinline__ static f16 from_f(float v) { return __float2half_rn(v); }
    __device__ __forceinline__ static float round(float v) { return __half2float(__float2half_rn(v)); }
    __device__ __forceinline__ static float lo(uint32_t w) { return __half2float(__ushort_as_half((unsigned short)(w & 0xffffu))); }
    __device__ __forceinline__ static float hi(uint32_t w) { return __half2float(__ushort_as_half((unsigned short)(w >> 16))); }
    __device__ __forceinline__ static uint32_t pack2(float a, float b) {
        __half2 p = __floats2half2_rn(a, b);
        return *reinterpret_cast<uint32_t*>(&p);
    }
};

__device__ __forceinline__ float round_bf16(float v) { return __bfloat162float(__float2bfloat16_rn(v)); }

// ---------------------------------------------------------------------------------------------
// fp8 e4m3 KV cache (LG_DTYPE_E4M3): one instruction each way on sm_90a. Every e4m3 value is exact in fp16 and in bf16.
// ---------------------------------------------------------------------------------------------
typedef __nv_fp8_e4m3 e4m3;   // storage tag of the fp8 cache (1 byte)
// (a, b) -> two e4m3 bytes, a in the low byte: clamp to +-448 (inf too), round to nearest even
__device__ __forceinline__ uint32_t e4m3x2_pack(float a, float b) {
    uint16_t r;
    asm("cvt.rn.satfinite.e4m3x2.f32 %0, %1, %2;" : "=h"(r) : "f"(b), "f"(a));
    return r;
}
// two e4m3 bytes (low 16 bits of v) -> f16x2, the low byte in the low half
__device__ __forceinline__ uint32_t e4m3x2_to_f16x2(uint32_t v) {
    uint32_t r;
    asm("cvt.rn.f16x2.e4m3x2 %0, %1;" : "=r"(r) : "h"((uint16_t)v));
    return r;
}
// two e4m3 bytes -> a packed pair of T (bf16 widens through fp32, exactly)
template <typename T> __device__ __forceinline__ uint32_t e4m3x2_to(uint32_t v);
template <> __device__ __forceinline__ uint32_t e4m3x2_to<f16>(uint32_t v) { return e4m3x2_to_f16x2(v); }
template <> __device__ __forceinline__ uint32_t e4m3x2_to<bf16>(uint32_t v) {
    const uint32_t h = e4m3x2_to_f16x2(v);
    return ElemTraits<bf16>::pack2(ElemTraits<f16>::lo(h), ElemTraits<f16>::hi(h));
}

#ifdef __CUDACC__
// mma.sync m16n8k16 with fp32 accumulators; T selects the .bf16 or .f16 operand type (register layouts are identical)
template <typename T>
__device__ __forceinline__ void mma_m16n8k16(float* c, uint32_t a0, uint32_t a1, uint32_t a2, uint32_t a3, uint32_t b0, uint32_t b1);
template <>
__device__ __forceinline__ void mma_m16n8k16<bf16>(float* c, uint32_t a0, uint32_t a1, uint32_t a2, uint32_t a3, uint32_t b0, uint32_t b1) {
    asm volatile("mma.sync.aligned.m16n8k16.row.col.f32.bf16.bf16.f32 {%0,%1,%2,%3}, {%4,%5,%6,%7}, {%8,%9}, {%0,%1,%2,%3};\n"
                 : "+f"(c[0]), "+f"(c[1]), "+f"(c[2]), "+f"(c[3])
                 : "r"(a0), "r"(a1), "r"(a2), "r"(a3), "r"(b0), "r"(b1));
}
template <>
__device__ __forceinline__ void mma_m16n8k16<f16>(float* c, uint32_t a0, uint32_t a1, uint32_t a2, uint32_t a3, uint32_t b0, uint32_t b1) {
    asm volatile("mma.sync.aligned.m16n8k16.row.col.f32.f16.f16.f32 {%0,%1,%2,%3}, {%4,%5,%6,%7}, {%8,%9}, {%0,%1,%2,%3};\n"
                 : "+f"(c[0]), "+f"(c[1]), "+f"(c[2]), "+f"(c[3])
                 : "r"(a0), "r"(a1), "r"(a2), "r"(a3), "r"(b0), "r"(b1));
}
#endif

// Load VEC contiguous elements of T as floats (VEC*sizeof(T) is 8, 16 or 32 bytes, pointer aligned to
// min(16, VEC*sizeof(T))).
template <typename T, int VEC> struct VecLoad;
template <> struct VecLoad<bf16, 8> {
    __device__ __forceinline__ static void load(const bf16* p, float* o) {
        uint4 u = *reinterpret_cast<const uint4*>(p);
        const uint32_t w[4] = {u.x, u.y, u.z, u.w};
#pragma unroll
        for (int i = 0; i < 4; ++i) {
            o[2 * i] = __uint_as_float(w[i] << 16);
            o[2 * i + 1] = __uint_as_float(w[i] & 0xffff0000u);
        }
    }
};
template <> struct VecLoad<bf16, 4> {
    __device__ __forceinline__ static void load(const bf16* p, float* o) {
        uint2 u = *reinterpret_cast<const uint2*>(p);
        o[0] = __uint_as_float(u.x << 16);
        o[1] = __uint_as_float(u.x & 0xffff0000u);
        o[2] = __uint_as_float(u.y << 16);
        o[3] = __uint_as_float(u.y & 0xffff0000u);
    }
};
template <> struct VecLoad<f16, 8> {
    __device__ __forceinline__ static void load(const f16* p, float* o) {
        uint4 u = *reinterpret_cast<const uint4*>(p);
        const uint32_t w[4] = {u.x, u.y, u.z, u.w};
#pragma unroll
        for (int i = 0; i < 4; ++i) {
            o[2 * i] = ElemTraits<f16>::lo(w[i]);
            o[2 * i + 1] = ElemTraits<f16>::hi(w[i]);
        }
    }
};
template <> struct VecLoad<f16, 4> {
    __device__ __forceinline__ static void load(const f16* p, float* o) {
        uint2 u = *reinterpret_cast<const uint2*>(p);
        o[0] = ElemTraits<f16>::lo(u.x);
        o[1] = ElemTraits<f16>::hi(u.x);
        o[2] = ElemTraits<f16>::lo(u.y);
        o[3] = ElemTraits<f16>::hi(u.y);
    }
};
template <> struct VecLoad<e4m3, 8> {   // fp8 cache: the undecoded e4m3 values (the scale is folded in by the caller)
    __device__ __forceinline__ static void load(const e4m3* p, float* o) {
        uint2 u = *reinterpret_cast<const uint2*>(p);
        const uint32_t w[2] = {u.x, u.y};
#pragma unroll
        for (int i = 0; i < 2; ++i) {
            const uint32_t lo = e4m3x2_to_f16x2(w[i]), hi = e4m3x2_to_f16x2(w[i] >> 16);
            o[4 * i] = ElemTraits<f16>::lo(lo);
            o[4 * i + 1] = ElemTraits<f16>::hi(lo);
            o[4 * i + 2] = ElemTraits<f16>::lo(hi);
            o[4 * i + 3] = ElemTraits<f16>::hi(hi);
        }
    }
};
template <> struct VecLoad<e4m3, 4> {
    __device__ __forceinline__ static void load(const e4m3* p, float* o) {
        const uint32_t w = *reinterpret_cast<const uint32_t*>(p);
        const uint32_t lo = e4m3x2_to_f16x2(w), hi = e4m3x2_to_f16x2(w >> 16);
        o[0] = ElemTraits<f16>::lo(lo);
        o[1] = ElemTraits<f16>::hi(lo);
        o[2] = ElemTraits<f16>::lo(hi);
        o[3] = ElemTraits<f16>::hi(hi);
    }
};
template <> struct VecLoad<float, 8> {
    __device__ __forceinline__ static void load(const float* p, float* o) {
        float4 a = *reinterpret_cast<const float4*>(p);
        float4 b = *reinterpret_cast<const float4*>(p + 4);
        o[0] = a.x; o[1] = a.y; o[2] = a.z; o[3] = a.w;
        o[4] = b.x; o[5] = b.y; o[6] = b.z; o[7] = b.w;
    }
};
template <> struct VecLoad<float, 4> {
    __device__ __forceinline__ static void load(const float* p, float* o) {
        float4 a = *reinterpret_cast<const float4*>(p);
        o[0] = a.x; o[1] = a.y; o[2] = a.z; o[3] = a.w;
    }
};

__device__ __forceinline__ float warp_sum(float v) {
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
    return v;
}
__device__ __forceinline__ float warp_max(float v) {
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) v = fmaxf(v, __shfl_xor_sync(0xffffffffu, v, o));
    return v;
}

// Block-wide sum/max via one smem round (blockDim.x multiple of 32, <= 1024). `red` holds >= 33 floats.
__device__ __forceinline__ float block_sum(float v, float* red) {
    const int lane = threadIdx.x & 31, w = threadIdx.x >> 5, nw = blockDim.x >> 5;
    v = warp_sum(v);
    __syncthreads();
    if (lane == 0) red[w] = v;
    __syncthreads();
    if (w == 0) {
        float t = lane < nw ? red[lane] : 0.f;
        t = warp_sum(t);
        if (lane == 0) red[32] = t;
    }
    __syncthreads();
    return red[32];
}
__device__ __forceinline__ float block_max(float v, float* red) {
    const int lane = threadIdx.x & 31, w = threadIdx.x >> 5, nw = blockDim.x >> 5;
    v = warp_max(v);
    __syncthreads();
    if (lane == 0) red[w] = v;
    __syncthreads();
    if (w == 0) {
        float t = lane < nw ? red[lane] : -INFINITY;
        t = warp_max(t);
        if (lane == 0) red[32] = t;
    }
    __syncthreads();
    return red[32];
}
