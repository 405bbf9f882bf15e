// elementwise.cu -- HBM-bound elementwise family for sm_90a: unary, binary (numpy broadcast),
// cast, where, expand.  128-bit coalesced accesses on the contiguous fast paths, grid sized in
// multiples of the 132 SMs, fp32 arithmetic with one rounding to the storage dtype.
//
// Replaces (reference, relative to /root/reference):
//   unary.cu:31-143 + ActivationCudnn unary.cc:70-122      -> it_b200_unary
//   ElementWiseCudnn element_wise.cc:8-121, element_wise.cu:9-131 -> it_b200_binary
//   _cast_kernel unary.cu:145-154                           -> it_b200_cast
//   _whereKernel where.cu:20-41                             -> it_b200_where
//   _expandKernel/_expandRowKernel expand.cu:10-49,154-170  -> it_b200_expand
#include "common.cuh"

namespace itb {

__device__ __forceinline__ float apply_unary(int op, float v, float alpha = 0.f) {
    switch (op) {
    case ITB_RELU: return v > 0.f ? v : 0.f;
    case ITB_SIGMOID: return 1.f / (1.f + expf(-v));
    case ITB_TANH: return tanhf(v);
    case ITB_GELU: return 0.5f * v * (1.f + erff(v * 0.70710678118654752440f));  // unary.cu:113 (erf form)
    case ITB_SILU: return v / (1.f + expf(-v));                                  // unary.cu:123
    case ITB_ERF: return erff(v);
    case ITB_NEG: return -v;
    case ITB_ABS: return fabsf(v);
    case ITB_SQRT: return sqrtf(v);
    case ITB_HARDSIGMOID: return fmaxf(0.f, fminf(1.f, 0.2f * v + 0.5f));
    case ITB_HARDSWISH: return v * fmaxf(0.f, fminf(1.f, (1.f / 6.f) * v + 0.5f));
    case ITB_EXP: return expf(v);
    case ITB_LEAKYRELU: return v > 0.f ? v : alpha * v;              // unary.cu:157-165
    case ITB_ELU: return v >= 0.f ? v : alpha * (expf(v) - 1.f);     // unary.cu:97-106
    }
    return v;
}

template <typename T>
__global__ void __launch_bounds__(256) unary_kernel(int op, const T *__restrict__ x, T *__restrict__ y,
                                                    int64_t n, bool vec, float alpha) {
    pdl_trigger();
    pdl_wait();
    constexpr int V = Vec16<T>::N;
    int64_t tid = blockIdx.x * (int64_t)blockDim.x + threadIdx.x;
    int64_t nthreads = (int64_t)gridDim.x * blockDim.x;
    if (vec) {
        int64_t nv = n / V;
        for (int64_t i = tid; i < nv; i += nthreads) {
            Vec16<T> a = ld16_stream(x + i * V), r;
#pragma unroll
            for (int j = 0; j < V; ++j) r.v[j] = from_f<T>(apply_unary(op, to_f(a.v[j]), alpha));
            st16(y + i * V, r);
        }
        for (int64_t i = nv * V + tid; i < n; i += nthreads) y[i] = from_f<T>(apply_unary(op, to_f(x[i]), alpha));
    } else {
        for (int64_t i = tid; i < n; i += nthreads) y[i] = from_f<T>(apply_unary(op, to_f(x[i]), alpha));
    }
}

__device__ __forceinline__ float apply_binary(int op, float a, float b) {
    switch (op) {
    case ITB_ADD: return a + b;
    case ITB_SUB: return a - b;
    case ITB_MUL: return a * b;
    case ITB_DIV: return a / b;
    case ITB_POW: return powf(a, b);
    case ITB_MIN: return fminf(a, b);
    case ITB_MAX: return fmaxf(a, b);
    case ITB_LESS: return a < b ? 1.f : 0.f;
    case ITB_EQUAL: return a == b ? 1.f : 0.f;
    case ITB_GREATER: return a > b ? 1.f : 0.f;
    }
    return 0.f;
}

// same-shape contiguous (sa = sb = 1) or one scalar operand (stride 0): vectorised
template <typename T>
__global__ void __launch_bounds__(256) binary_flat_kernel(int op, const T *__restrict__ a,
                                                          const T *__restrict__ b, T *__restrict__ c,
                                                          int64_t n, int sa, int sb, bool vec) {
    pdl_trigger();
    pdl_wait();
    constexpr int V = Vec16<T>::N;
    int64_t tid = blockIdx.x * (int64_t)blockDim.x + threadIdx.x;
    int64_t nthreads = (int64_t)gridDim.x * blockDim.x;
    float a0 = sa ? 0.f : to_f(a[0]), b0 = sb ? 0.f : to_f(b[0]);
    int64_t done = 0;
    if (vec) {
        int64_t nv = n / V;
        for (int64_t i = tid; i < nv; i += nthreads) {
            Vec16<T> va, vb, r;
            if (sa) va = ld16_stream(a + i * V);
            if (sb) vb = ld16_stream(b + i * V);
#pragma unroll
            for (int j = 0; j < V; ++j)
                r.v[j] = from_f<T>(apply_binary(op, sa ? to_f(va.v[j]) : a0, sb ? to_f(vb.v[j]) : b0));
            st16(c + i * V, r);
        }
        done = nv * V;
    }
    for (int64_t i = done + tid; i < n; i += nthreads)
        c[i] = from_f<T>(apply_binary(op, sa ? to_f(a[i]) : a0, sb ? to_f(b[i]) : b0));
}

// general broadcast; OUT is T (arithmetic) or uint8_t (comparison)
template <typename T, typename OUT>
__global__ void __launch_bounds__(256) binary_general_kernel(int op, const T *__restrict__ a,
                                                             const T *__restrict__ b, OUT *__restrict__ c,
                                                             int64_t n, int rank, Dims8 dims, Dims8 sa,
                                                             Dims8 sb) {
    pdl_trigger();
    pdl_wait();
    int64_t nthreads = (int64_t)gridDim.x * blockDim.x;
    for (int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; i < n; i += nthreads) {
        int64_t rem = i, oa = 0, ob = 0;
        for (int d = rank - 1; d >= 0; --d) {
            int64_t q = rem / dims.v[d], ci = rem - q * dims.v[d];
            rem = q;
            oa += ci * sa.v[d];
            ob += ci * sb.v[d];
        }
        float r = apply_binary(op, to_f(a[oa]), to_f(b[ob]));
        if constexpr (sizeof(OUT) == 1 && !std::is_same<OUT, T>::value)
            c[i] = (OUT)(r != 0.f);
        else
            c[i] = from_f<T>(r);
    }
}

// out = T( T(silu(g)) * u )  -- the Silu -> Mul pair of the Llama MLP in one pass
template <typename T>
__global__ void __launch_bounds__(256) silu_mul_kernel(const T *__restrict__ g, const T *__restrict__ u,
                                                       T *__restrict__ o, int64_t n, bool vec) {
    pdl_trigger();
    pdl_wait();
    constexpr int V = Vec16<T>::N;
    int64_t tid = blockIdx.x * (int64_t)blockDim.x + threadIdx.x;
    int64_t nthreads = (int64_t)gridDim.x * blockDim.x;
    int64_t done = 0;
    if (vec) {
        int64_t nv = n / V;
        for (int64_t i = tid; i < nv; i += nthreads) {
            Vec16<T> a = ld16_stream(g + i * V), b = ld16_stream(u + i * V), r;
#pragma unroll
            for (int j = 0; j < V; ++j)
                r.v[j] = from_f<T>(round_t<T>(apply_unary(ITB_SILU, to_f(a.v[j]))) * to_f(b.v[j]));
            st16(o + i * V, r);
        }
        done = nv * V;
    }
    for (int64_t i = done + tid; i < n; i += nthreads)
        o[i] = from_f<T>(round_t<T>(apply_unary(ITB_SILU, to_f(g[i]))) * to_f(u[i]));
}

// collapse adjacent dims whose strides chain for every operand
static int collapse(int rank, const int64_t *dims, const int64_t *const *strides, int nops, Dims8 &od,
                    Dims8 *os) {
    int r = 0;
    for (int d = 0; d < rank; ++d) {
        if (dims[d] == 1) continue;
        bool merge = r > 0;
        if (merge)
            for (int o = 0; o < nops; ++o)
                if (os[o].v[r - 1] != strides[o][d] * dims[d]) merge = false;
        if (merge) {
            od.v[r - 1] *= dims[d];
            for (int o = 0; o < nops; ++o) os[o].v[r - 1] = strides[o][d];
        } else {
            od.v[r] = dims[d];
            for (int o = 0; o < nops; ++o) os[o].v[r] = strides[o][d];
            ++r;
        }
    }
    if (r == 0) {
        od.v[0] = 1;
        for (int o = 0; o < nops; ++o) os[o].v[0] = 0;
        r = 1;
    }
    return r;
}

template <typename SRC, typename DST> __device__ __forceinline__ DST cast_one(SRC v) {
    if constexpr (std::is_same<SRC, __half>::value || std::is_same<SRC, __nv_bfloat16>::value) {
        float f = to_f(v);
        if constexpr (std::is_same<DST, __half>::value || std::is_same<DST, __nv_bfloat16>::value)
            return from_f<DST>(f);
        else
            return (DST)f;
    } else if constexpr (std::is_same<DST, __half>::value || std::is_same<DST, __nv_bfloat16>::value) {
        return from_f<DST>((float)v);
    } else {
        return (DST)v;  // static_cast semantics == cub::CastOp (unary.cu:150)
    }
}

template <typename SRC, typename DST>
__global__ void __launch_bounds__(256) cast_kernel(const SRC *__restrict__ x, DST *__restrict__ y, int64_t n) {
    pdl_trigger();
    pdl_wait();
    int64_t nthreads = (int64_t)gridDim.x * blockDim.x;
    for (int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; i < n; i += nthreads)
        y[i] = cast_one<SRC, DST>(x[i]);
}

template <typename E>
__global__ void __launch_bounds__(256) where_kernel(const uint8_t *__restrict__ cond, const E *__restrict__ x,
                                                    const E *__restrict__ y, E *__restrict__ out, int64_t n,
                                                    int rank, Dims8 dims, Dims8 sc, Dims8 sx, Dims8 sy) {
    pdl_trigger();
    pdl_wait();
    int64_t nthreads = (int64_t)gridDim.x * blockDim.x;
    for (int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; i < n; i += nthreads) {
        int64_t rem = i, oc = 0, ox = 0, oy = 0;
        for (int d = rank - 1; d >= 0; --d) {
            int64_t q = rem / dims.v[d], ci = rem - q * dims.v[d];
            rem = q;
            oc += ci * sc.v[d];
            ox += ci * sx.v[d];
            oy += ci * sy.v[d];
        }
        out[i] = cond[oc] ? x[ox] : y[oy];
    }
}

template <typename E>
__global__ void __launch_bounds__(256) expand_kernel(const E *__restrict__ x, E *__restrict__ y, int64_t n,
                                                     int rank, Dims8 dims, Dims8 sx) {
    pdl_trigger();
    pdl_wait();
    int64_t nthreads = (int64_t)gridDim.x * blockDim.x;
    for (int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; i < n; i += nthreads) {
        int64_t rem = i, ox = 0;
        for (int d = rank - 1; d >= 0; --d) {
            int64_t q = rem / dims.v[d], ci = rem - q * dims.v[d];
            rem = q;
            ox += ci * sx.v[d];
        }
        y[i] = x[ox];
    }
}

// DequantizeLinear for FP8 E4M3 codes with a per-column scale: y[r][c] = T(e4m3(xq[r][c]) * scale[c])
__device__ __forceinline__ float e4m3_to_f(uint8_t c) {
    const unsigned short pair = c;
    uint32_t h2;
    asm("cvt.rn.f16x2.e4m3x2 %0, %1;" : "=r"(h2) : "h"(pair));
    return __half2float(__ushort_as_half((unsigned short)(h2 & 0xffffu)));
}
template <typename T>
__global__ void __launch_bounds__(256) dequant_fp8_kernel(const uint8_t *__restrict__ xq, const float *__restrict__ scale,
                                                          T *__restrict__ y, int64_t n, int64_t cols) {
    pdl_trigger();
    pdl_wait();
    for (int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; i < n; i += (int64_t)gridDim.x * blockDim.x)
        y[i] = from_f<T>(e4m3_to_f(xq[i]) * scale[i % cols]);
}

}  // namespace itb

using namespace itb;

extern "C" int it_b200_dequantize_fp8(int dtype_out, const void *xq, const float *scale, void *y, int64_t rows, int64_t cols,
                                      void *stream) {
    const int64_t n = rows * cols;
    if (n == 0) return 0;
    ITB_DISPATCH_FLOAT(dtype_out, "dequantize_fp8", {
        return launch("dequantize_fp8", dequant_fp8_kernel<T>, {dim3(grid_for(n, 256)), dim3(256), 0, (cudaStream_t)stream},
                      (const uint8_t *)xq, scale, (T *)y, n, cols);
    });
    return 0;
}

extern "C" int it_b200_unary_alpha(int op, int dtype, const void *x, void *y, int64_t n, float alpha, void *stream) {
    ITB_CHECK(op >= ITB_RELU && op <= ITB_ELU, "unary: bad op %d", op);
    if (n == 0) return 0;
    auto st = (cudaStream_t)stream;
    ITB_DISPATCH_FLOAT(dtype, "unary", {
        bool vec = aligned16(x) && aligned16(y);
        int64_t items = vec ? (n + Vec16<T>::N - 1) / Vec16<T>::N : n;
        return launch("unary", unary_kernel<T>, {dim3(grid_for(items, 256)), dim3(256), 0, st}, op, (const T *)x, (T *)y, n, vec,
                      alpha);
    });
    return 0;
}
extern "C" int it_b200_unary(int op, int dtype, const void *x, void *y, int64_t n, void *stream) {
    ITB_CHECK(op >= ITB_RELU && op <= ITB_EXP, "unary: bad op %d", op);
    return it_b200_unary_alpha(op, dtype, x, y, n, 0.f, stream);
}

extern "C" int it_b200_silu_mul(int dtype, const void *gate, const void *up, void *out, int64_t n, void *stream) {
    if (n == 0) return 0;
    ITB_DISPATCH_FLOAT(dtype, "silu_mul", {
        bool vec = aligned16(gate) && aligned16(up) && aligned16(out);
        int64_t items = vec ? (n + Vec16<T>::N - 1) / Vec16<T>::N : n;
        return launch("silu_mul", silu_mul_kernel<T>, {dim3(grid_for(items, 256)), dim3(256), 0, (cudaStream_t)stream},
                      (const T *)gate, (const T *)up, (T *)out, n, vec);
    });
    return 0;
}

extern "C" int it_b200_binary(int op, int dtype, const void *a, const void *b, void *c, int rank,
                              const int64_t *dims, const int64_t *stride_a, const int64_t *stride_b,
                              void *stream) {
    ITB_CHECK(op >= ITB_ADD && op <= ITB_GREATER, "binary: bad op %d", op);
    ITB_CHECK(rank >= 0 && rank <= ITB_MAX_RANK, "binary: rank %d > %d", rank, ITB_MAX_RANK);
    auto st = (cudaStream_t)stream;
    int64_t n = 1;
    for (int i = 0; i < rank; ++i) n *= dims[i];
    if (n == 0) return 0;
    Dims8 cd{}, cs[2]{};
    const int64_t *strides[2] = {stride_a, stride_b};
    int cr = collapse(rank, dims, strides, 2, cd, cs);
    bool cmp = op >= ITB_LESS;
    bool flat = !cmp && cr == 1 && (cs[0].v[0] == 0 || cs[0].v[0] == 1) && (cs[1].v[0] == 0 || cs[1].v[0] == 1);
    ITB_DISPATCH_FLOAT(dtype, "binary", {
        if (flat) {
            bool vec = aligned16(a) && aligned16(b) && aligned16(c);
            int64_t items = vec ? (n + Vec16<T>::N - 1) / Vec16<T>::N : n;
            return launch("binary", binary_flat_kernel<T>, {dim3(grid_for(items, 256)), dim3(256), 0, st}, op, (const T *)a, (const T *)b, (T *)c, n, (int)cs[0].v[0], (int)cs[1].v[0], vec);
        }
        const LaunchCfg cfg{dim3(grid_for(n, 256)), dim3(256), 0, st};
        if (cmp)
            return launch("binary", binary_general_kernel<T, uint8_t>, cfg, op, (const T *)a, (const T *)b, (uint8_t *)c, n, cr, cd, cs[0], cs[1]);
        return launch("binary", binary_general_kernel<T, T>, cfg, op, (const T *)a, (const T *)b, (T *)c, n, cr, cd, cs[0], cs[1]);
    });
    return 0;
}

#define CAST_CASE(FROM, TO, SRC, DST)                                                          \
    if (from == FROM && to == TO) return launch("cast", cast_kernel<SRC, DST>, {dim3(g), dim3(256), 0, st}, (const SRC *)x, (DST *)y, n);

extern "C" int it_b200_cast(int from, int to, const void *x, void *y, int64_t n, void *stream) {
    if (n == 0) return 0;
    auto st = (cudaStream_t)stream;
    int g = grid_for(n, 256);
    // reference set (unary.cc:30-68): f32<->f16, f32->i32, f32<->i8; plus the bf16 / i64 pairs the
    // bf16 decode graph needs.
    CAST_CASE(ITB_F32, ITB_F16, float, __half)
    CAST_CASE(ITB_F16, ITB_F32, __half, float)
    CAST_CASE(ITB_F32, ITB_BF16, float, __nv_bfloat16)
    CAST_CASE(ITB_BF16, ITB_F32, __nv_bfloat16, float)
    CAST_CASE(ITB_F16, ITB_BF16, __half, __nv_bfloat16)
    CAST_CASE(ITB_BF16, ITB_F16, __nv_bfloat16, __half)
    CAST_CASE(ITB_F32, ITB_I32, float, int32_t)
    CAST_CASE(ITB_I32, ITB_F32, int32_t, float)
    CAST_CASE(ITB_F32, ITB_I8, float, int8_t)
    CAST_CASE(ITB_I8, ITB_F32, int8_t, float)
    CAST_CASE(ITB_I64, ITB_F32, int64_t, float)
    CAST_CASE(ITB_F32, ITB_I64, float, int64_t)
    CAST_CASE(ITB_I64, ITB_I32, int64_t, int32_t)
    CAST_CASE(ITB_I32, ITB_I64, int32_t, int64_t)
    CAST_CASE(ITB_F32, ITB_F32, float, float)
    ITB_FAIL("cast: unsupported pair %d -> %d", from, to);
}

#define ELEM_DISPATCH(es, NAME, ...)                                                           \
    switch (es) {                                                                              \
    case 1: { using E = uint8_t; __VA_ARGS__; } break;                                         \
    case 2: { using E = uint16_t; __VA_ARGS__; } break;                                        \
    case 4: { using E = uint32_t; __VA_ARGS__; } break;                                        \
    case 8: { using E = uint64_t; __VA_ARGS__; } break;                                        \
    default: ITB_FAIL("%s: unsupported element size %d", NAME, es);                            \
    }

extern "C" int it_b200_where(int elem_size, const void *cond, const void *x, const void *y, void *out,
                             int rank, const int64_t *dims, const int64_t *stride_c,
                             const int64_t *stride_x, const int64_t *stride_y, void *stream) {
    ITB_CHECK(rank >= 0 && rank <= ITB_MAX_RANK, "where: rank %d > %d", rank, ITB_MAX_RANK);
    auto st = (cudaStream_t)stream;
    int64_t n = 1;
    for (int i = 0; i < rank; ++i) n *= dims[i];
    if (n == 0) return 0;
    Dims8 cd{}, cs[3]{};
    const int64_t *strides[3] = {stride_c, stride_x, stride_y};
    int cr = collapse(rank, dims, strides, 3, cd, cs);
    ELEM_DISPATCH(elem_size, "where", {
        return launch("where", where_kernel<E>, {dim3(grid_for(n, 256)), dim3(256), 0, st}, (const uint8_t *)cond, (const E *)x,
                      (const E *)y, (E *)out, n, cr, cd, cs[0], cs[1], cs[2]);
    });
    return 0;
}

extern "C" int it_b200_expand(int elem_size, const void *x, void *y, int rank, const int64_t *dims,
                              const int64_t *stride_x, void *stream) {
    ITB_CHECK(rank >= 0 && rank <= ITB_MAX_RANK, "expand: rank %d > %d", rank, ITB_MAX_RANK);
    auto st = (cudaStream_t)stream;
    int64_t n = 1;
    for (int i = 0; i < rank; ++i) n *= dims[i];
    if (n == 0) return 0;
    Dims8 cd{}, cs[1]{};
    const int64_t *strides[1] = {stride_x};
    int cr = collapse(rank, dims, strides, 1, cd, cs);
    ELEM_DISPATCH(elem_size, "expand", {
        return launch("expand", expand_kernel<E>, {dim3(grid_for(n, 256)), dim3(256), 0, st}, (const E *)x, (E *)y, n, cr, cd, cs[0]);
    });
    return 0;
}
