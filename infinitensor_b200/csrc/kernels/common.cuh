// common.cuh -- shared device/host helpers for the sm_90a kernels.
#pragma once
#include <cuda_bf16.h>
#include <cuda_fp16.h>
#include <cuda_runtime.h>
#include <stdint.h>
#include <stdio.h>

#include <utility>

#include "it_b200.h"

namespace itb {

// ---- error reporting (the C spelling of infini::Exception) -------------------------------
void set_error(const char *fmt, ...);

#define ITB_FAIL(...)                                                                          \
    do {                                                                                       \
        itb::set_error(__VA_ARGS__);                                                           \
        return 1;                                                                              \
    } while (0)

#define ITB_CHECK(cond, ...)                                                                   \
    do {                                                                                       \
        if (!(cond)) ITB_FAIL(__VA_ARGS__);                                                    \
    } while (0)

constexpr int kNumSMs = 132;  // H100 SXM

// ---- programmatic dependent launch (PDL) -----------------------------------------------------
// Every kernel is launched with cudaLaunchAttributeProgrammaticStreamSerialization, and every kernel begins with
// pdl_trigger() (lets the NEXT kernel in the stream start its launch + prologue now) and executes pdl_wait() before
// its first read of an activation or its first global write (blocks until the PREVIOUS kernel has fully completed
// and flushed).  In a decode step of ~450 short kernels this hides the launch gap, and the GEMM kernels prefetch
// their weight tiles -- which no kernel in the step writes -- ahead of pdl_wait().
__device__ __forceinline__ void pdl_trigger() { asm volatile("griddepcontrol.launch_dependents;" ::: "memory"); }
__device__ __forceinline__ void pdl_wait() { asm volatile("griddepcontrol.wait;" ::: "memory"); }
bool pdl_enabled();  // false when ITB_NO_PDL=1
// zero-initialised, self-cleaning int tickets private to (device, stream); nullptr if n exceeds the pool (65536)
int *stream_tickets(cudaStream_t st, int n);

// ---- the one kernel launch path ------------------------------------------------------------
struct LaunchCfg {
    dim3 grid, block;
    int smem;  // dynamic shared memory, bytes
    cudaStream_t stream;
    dim3 cluster = dim3(0, 0, 0);  // x == 0: no cluster attribute
};
// raises `kernel`'s dynamic shared-memory limit on the current device to `smem` unless it already allows that much;
// 0, or 1 with the error set
int opt_in_smem(const char *what, const void *kernel, int smem);
// the result of one cudaLaunchKernelEx: counts the launch (0), or sets "<what>: <CUDA error>" (1)
int launched(const char *what, cudaError_t e);

// Every kernel goes through here: its shared memory opted in, the cluster attribute when given, PDL unless ITB_NO_PDL=1,
// and one count in it_b200_launch_count() per kernel launched.  0, or 1 with the error set.
template <typename... KArgs, typename... Args>
inline int launch(const char *what, void (*kernel)(KArgs...), const LaunchCfg &c, Args &&...args) {
    if (c.smem > 0 && opt_in_smem(what, reinterpret_cast<const void *>(kernel), c.smem)) return 1;
    cudaLaunchConfig_t cfg{};
    cfg.gridDim = c.grid;
    cfg.blockDim = c.block;
    cfg.dynamicSmemBytes = (size_t)c.smem;
    cfg.stream = c.stream;
    cudaLaunchAttribute attr[2];
    unsigned n = 0;
    if (c.cluster.x) {
        attr[n].id = cudaLaunchAttributeClusterDimension;
        attr[n].val.clusterDim.x = c.cluster.x;
        attr[n].val.clusterDim.y = c.cluster.y;
        attr[n].val.clusterDim.z = c.cluster.z;
        ++n;
    }
    if (pdl_enabled()) {
        attr[n].id = cudaLaunchAttributeProgrammaticStreamSerialization;
        attr[n].val.programmaticStreamSerializationAllowed = 1;
        ++n;
    }
    cfg.attrs = attr;
    cfg.numAttrs = n;
    return launched(what, cudaLaunchKernelEx(&cfg, kernel, std::forward<Args>(args)...));
}

inline int dtype_size(int dt) {
    switch (dt) {
    case ITB_F32: case ITB_I32: case ITB_U32: return 4;
    case ITB_F16: case ITB_BF16: return 2;
    case ITB_I64: return 8;
    case ITB_U8: case ITB_I8: case ITB_BOOL: return 1;
    default: return 0;
    }
}

// ---- dtype traits --------------------------------------------------------------------------
template <typename T> struct TypeOps;
template <> struct TypeOps<float> {
    static __device__ __forceinline__ float to_f(float v) { return v; }
    static __device__ __forceinline__ float from_f(float v) { return v; }
};
template <> struct TypeOps<__half> {
    static __device__ __forceinline__ float to_f(__half v) { return __half2float(v); }
    static __device__ __forceinline__ __half from_f(float v) { return __float2half_rn(v); }
};
template <> struct TypeOps<__nv_bfloat16> {
    static __device__ __forceinline__ float to_f(__nv_bfloat16 v) { return __bfloat162float(v); }
    static __device__ __forceinline__ __nv_bfloat16 from_f(float v) { return __float2bfloat16_rn(v); }
};
template <typename T> __device__ __forceinline__ float to_f(T v) { return TypeOps<T>::to_f(v); }
template <typename T> __device__ __forceinline__ T from_f(float v) { return TypeOps<T>::from_f(v); }
// round a float to T and back (the reference's "(T)(expr)" points)
template <typename T> __device__ __forceinline__ float round_t(float v) { return to_f<T>(from_f<T>(v)); }

// inference BatchNorm arithmetic, spelled with intrinsics so the stand-alone kernel and the conv epilogue round alike:
//   y = scale * (x - mean) * rs + bias,  rs = 1 / sqrt(var + eps)      (reference batch_norm.cc:9-69 via cuDNN)
//   rs as the hardware reciprocal square root (what cudnnBatchNormalizationForwardInference evaluates): the reference's own
//   golden vector (test_cuda_batch_norm.cc:49-52: (8 - 9) / sqrt(9) expected "-0.333333" within its relative 1e-6) holds for
//   rsqrt(9) = 0.33333331 and NOT for the correctly rounded 1 / sqrt(9) = 0.33333334
__device__ __forceinline__ float bn_rs(float var, float eps) { return rsqrtf(var + eps); }
__device__ __forceinline__ float bn_apply(float x, float mean, float rs, float scale, float bias) {
    return __fmaf_rn(__fmul_rn(scale, __fsub_rn(x, mean)), rs, bias);
}

// 16-byte vector of T
template <typename T> struct Vec16 {
    static constexpr int N = 16 / sizeof(T);
    T v[N];
};
template <typename T> __device__ __forceinline__ Vec16<T> ld16(const T *p) {
    Vec16<T> r;
    *reinterpret_cast<uint4 *>(r.v) = *reinterpret_cast<const uint4 *>(p);
    return r;
}
template <typename T> __device__ __forceinline__ Vec16<T> ld16_stream(const T *p) {
    Vec16<T> r;
    uint4 u;
    asm volatile("ld.global.nc.L1::no_allocate.v4.u32 {%0,%1,%2,%3}, [%4];"
                 : "=r"(u.x), "=r"(u.y), "=r"(u.z), "=r"(u.w) : "l"(p));
    *reinterpret_cast<uint4 *>(r.v) = u;
    return r;
}
template <typename T> __device__ __forceinline__ void st16(T *p, const Vec16<T> &r) {
    *reinterpret_cast<uint4 *>(p) = *reinterpret_cast<const uint4 *>(r.v);
}

// two FP8 E4M3 codes (low byte = first element) -> two values of the activation type, exactly (every E4M3 value is
// representable in f16 and in bf16)
template <typename T> __device__ __forceinline__ uint32_t e4m3x2_to(uint32_t pair16);
template <> __device__ __forceinline__ uint32_t e4m3x2_to<__half>(uint32_t pair16) {
    uint32_t r;
    asm("cvt.rn.f16x2.e4m3x2 %0, %1;" : "=r"(r) : "h"((unsigned short)pair16));
    return r;
}
template <> __device__ __forceinline__ uint32_t e4m3x2_to<__nv_bfloat16>(uint32_t pair16) {
    const uint32_t h2 = e4m3x2_to<__half>(pair16);
    const float2 f = __half22float2(*reinterpret_cast<const __half2 *>(&h2));
    const __nv_bfloat162 b = __floats2bfloat162_rn(f.x, f.y);
    return *reinterpret_cast<const uint32_t *>(&b);
}
// two fp32 values -> two FP8 E4M3 codes (low byte = lo): round to nearest even, saturated to +-448, NaN kept
__device__ __forceinline__ uint32_t f32x2_to_e4m3x2(float lo, float hi) {
    unsigned short r;
    asm("cvt.rn.satfinite.e4m3x2.f32 %0, %1, %2;" : "=h"(r) : "f"(hi), "f"(lo));
    return r;
}

inline bool aligned16(const void *p) { return (reinterpret_cast<uintptr_t>(p) & 15) == 0; }

// ---- rolling KV cache (ITB_POS_RING): the one place that maps a position to its cache row ----------------------------
// A ring of Smax rows holds position p in row p mod Smax; a linear cache, in row p.  Ring positions are clamped to
// [0, ring_pos_max(Smax)], so that every position a step forms (below p + Smax) stays inside int
__host__ __device__ constexpr int ring_pos_max(int Smax) { return 0x7fffffff - Smax; }
__device__ __forceinline__ int cache_row(int p, int Smax, bool ring) { return ring ? p % Smax : p; }
// the ring's shape rule, before any launch (S: tokens per step): 0, or 1 with the error set
inline int check_ring(const char *what, int window, int Smax, int S) {
    ITB_CHECK(window >= 1, "%s: a rolling cache (ITB_POS_RING) needs a window >= 1", what);
    ITB_CHECK(Smax >= window, "%s: a rolling cache of %d rows is shorter than the window of %d", what, Smax, window);
    ITB_CHECK(Smax % 64 == 0, "%s: a rolling cache's length %d is not a multiple of 64", what, Smax);
    ITB_CHECK(S <= 1 || Smax >= (int64_t)window + S - 1,
              "%s: a chunk of %d tokens needs a rolling cache of window + %d = %lld rows or more, not %d (split the prompt)", what,
              S, S - 1, (long long)window + S - 1, Smax);
    return 0;
}

// ---- reductions -----------------------------------------------------------------------------
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
// block-wide sum; `red` is >= 32 floats of shared memory; all threads get the result
__device__ __forceinline__ float block_sum(float v, float *red) {
    int lane = threadIdx.x & 31, wid = threadIdx.x >> 5, nw = (blockDim.x + 31) >> 5;
    v = warp_sum(v);
    __syncthreads();
    if (lane == 0) red[wid] = v;
    __syncthreads();
    float r = lane < nw ? red[lane] : 0.f;
    return warp_sum(r);
}
__device__ __forceinline__ float block_max(float v, float *red) {
    int lane = threadIdx.x & 31, wid = threadIdx.x >> 5, nw = (blockDim.x + 31) >> 5;
    v = warp_max(v);
    __syncthreads();
    if (lane == 0) red[wid] = v;
    __syncthreads();
    float r = lane < nw ? red[lane] : -INFINITY;
    return warp_max(r);
}

// grid sizing for HBM-bound grid-stride kernels: a few waves of 132 SMs
inline int grid_for(int64_t work_items, int threads, int max_ctas_per_sm = 8) {
    int64_t need = (work_items + threads - 1) / threads;
    int64_t cap = (int64_t)kNumSMs * max_ctas_per_sm;
    if (need < 1) need = 1;
    return (int)(need < cap ? need : cap);
}

struct Dims8 {
    int64_t v[ITB_MAX_RANK];
};

#define ITB_DISPATCH_FLOAT(dt, NAME, ...)                                                      \
    switch (dt) {                                                                              \
    case ITB_F32: { using T = float; __VA_ARGS__; } break;                                     \
    case ITB_F16: { using T = __half; __VA_ARGS__; } break;                                    \
    case ITB_BF16: { using T = __nv_bfloat16; __VA_ARGS__; } break;                            \
    default: ITB_FAIL("%s: unsupported dtype %d", NAME, dt);                                   \
    }

}  // namespace itb
