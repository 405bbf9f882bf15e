// norm.cu -- Softmax, LayerNormalization, RMSNorm, RoPE for sm_90a.
// HBM-bound row reductions: one read + one write of the tensor, fp32 accumulation, warp-shuffle
// reductions; rows cached in registers (warp-per-row) or shared memory (block-per-row).
//
// Replaces (reference): softmax.cu:18-404, layer_norm.cu:4-557, rms_norm.cu:36-110, rope.cu:7-88.
#include <type_traits>

#include "common.cuh"

namespace itb {

// ------------------------------------------------------------------ last-axis, warp per row
// MODE 0 softmax, 1 layernorm
template <typename T, int ITEMS, int MODE>
__global__ void __launch_bounds__(256) row_warp_kernel(const T *__restrict__ x, T *__restrict__ y,
                                                       const T *__restrict__ scale, const T *__restrict__ bias,
                                                       int64_t rows, int dim, int scale_size, int bias_size,
                                                       float eps) {
    pdl_trigger();
    pdl_wait();
    int lane = threadIdx.x & 31;
    int64_t row = (blockIdx.x * (int64_t)blockDim.x + threadIdx.x) >> 5;
    if (row >= rows) return;
    const T *px = x + row * dim;
    T *py = y + row * dim;
    float v[ITEMS];
#pragma unroll
    for (int i = 0; i < ITEMS; ++i) {
        int d = lane + i * 32;
        v[i] = d < dim ? to_f(px[d]) : (MODE == 0 ? -INFINITY : 0.f);
    }
    if (MODE == 0) {
        float mx = -INFINITY;
#pragma unroll
        for (int i = 0; i < ITEMS; ++i) mx = fmaxf(mx, v[i]);
        mx = warp_max(mx);
        float s = 0.f;
#pragma unroll
        for (int i = 0; i < ITEMS; ++i) {
            v[i] = (lane + i * 32 < dim) ? expf(v[i] - mx) : 0.f;
            s += v[i];
        }
        s = warp_sum(s);
#pragma unroll
        for (int i = 0; i < ITEMS; ++i) {
            int d = lane + i * 32;
            if (d < dim) py[d] = from_f<T>(v[i] / s);
        }
    } else {
        float s = 0.f;
#pragma unroll
        for (int i = 0; i < ITEMS; ++i) s += v[i];
        float mu = warp_sum(s) / (float)dim;
        float q = 0.f;
#pragma unroll
        for (int i = 0; i < ITEMS; ++i) {
            float t = (lane + i * 32 < dim) ? v[i] - mu : 0.f;
            q += t * t;
        }
        float rs = rsqrtf(warp_sum(q) / (float)dim + eps);
#pragma unroll
        for (int i = 0; i < ITEMS; ++i) {
            int d = lane + i * 32;
            if (d < dim) {
                float sc = to_f(scale[scale_size == dim ? d : 0]);
                float bi = bias ? to_f(bias[bias_size == dim ? d : 0]) : 0.f;
                py[d] = from_f<T>(sc * (v[i] - mu) * rs + bi);
            }
        }
    }
}

// the same for 2-byte types with dim % 8 == 0 (<= 1024): a lane owns 16-byte chunks lane, lane + 32, ... of the row -- three 16-byte
// loads instead of 24 scalar ones for a 768-wide row (the scalar kernel runs a chain of
// ~100 dependent 2-byte loads / stores per lane on GPT-2's [128, 768] LayerNorms)
template <typename T, int CHUNKS, int MODE>
__global__ void __launch_bounds__(256) row_warp_vec_kernel(const T *__restrict__ x, T *__restrict__ y, const T *__restrict__ scale,
                                                           const T *__restrict__ bias, int64_t rows, int dim, int scale_size,
                                                           int bias_size, float eps) {
    pdl_trigger();
    pdl_wait();
    constexpr int V = 8;
    const int lane = threadIdx.x & 31;
    const int64_t row = (blockIdx.x * (int64_t)blockDim.x + threadIdx.x) >> 5;
    if (row >= rows) return;
    const T *px = x + row * dim;
    T *py = y + row * dim;
    const int nch = dim / V;
    float v[CHUNKS][V];
#pragma unroll
    for (int i = 0; i < CHUNKS; ++i) {
        const int c = lane + i * 32;
        if (c < nch) {
            const Vec16<T> a = ld16(px + c * V);
#pragma unroll
            for (int j = 0; j < V; ++j) v[i][j] = to_f(a.v[j]);
        } else {
#pragma unroll
            for (int j = 0; j < V; ++j) v[i][j] = MODE == 0 ? -INFINITY : 0.f;
        }
    }
    if (MODE == 0) {
        float mx = -INFINITY;
#pragma unroll
        for (int i = 0; i < CHUNKS; ++i)
#pragma unroll
            for (int j = 0; j < V; ++j) mx = fmaxf(mx, v[i][j]);
        mx = warp_max(mx);
        float s = 0.f;
#pragma unroll
        for (int i = 0; i < CHUNKS; ++i)
#pragma unroll
            for (int j = 0; j < V; ++j) {
                v[i][j] = (lane + i * 32 < nch) ? expf(v[i][j] - mx) : 0.f;
                s += v[i][j];
            }
        s = warp_sum(s);
#pragma unroll
        for (int i = 0; i < CHUNKS; ++i) {
            const int c = lane + i * 32;
            if (c < nch) {
                Vec16<T> o;
#pragma unroll
                for (int j = 0; j < V; ++j) o.v[j] = from_f<T>(v[i][j] / s);
                st16(py + c * V, o);
            }
        }
    } else {
        float s = 0.f;
#pragma unroll
        for (int i = 0; i < CHUNKS; ++i)
#pragma unroll
            for (int j = 0; j < V; ++j) s += v[i][j];
        const float mu = warp_sum(s) / (float)dim;
        float q = 0.f;
#pragma unroll
        for (int i = 0; i < CHUNKS; ++i)
#pragma unroll
            for (int j = 0; j < V; ++j) {
                const float t = (lane + i * 32 < nch) ? v[i][j] - mu : 0.f;
                q += t * t;
            }
        const float rs = rsqrtf(warp_sum(q) / (float)dim + eps);
#pragma unroll
        for (int i = 0; i < CHUNKS; ++i) {
            const int c = lane + i * 32;
            if (c < nch) {
                Vec16<T> sc, bi, o;
                if (scale_size == dim) sc = ld16(scale + c * V);
                if (bias && bias_size == dim) bi = ld16(bias + c * V);
#pragma unroll
                for (int j = 0; j < V; ++j) {
                    const float scf = scale_size == dim ? to_f(sc.v[j]) : to_f(scale[0]);
                    const float bif = bias ? (bias_size == dim ? to_f(bi.v[j]) : to_f(bias[0])) : 0.f;
                    o.v[j] = from_f<T>(scf * (v[i][j] - mu) * rs + bif);
                }
                st16(py + c * V, o);
            }
        }
    }
}

// ------------------------------------------------------------------ last-axis, block per row
template <typename T, int MODE>
__global__ void __launch_bounds__(1024) row_block_kernel(const T *__restrict__ x, T *__restrict__ y,
                                                         const T *__restrict__ scale, const T *__restrict__ bias,
                                                         int dim, int scale_size, int bias_size, float eps,
                                                         int cache_in_smem) {
    pdl_trigger();
    pdl_wait();
    extern __shared__ float srow[];
    __shared__ float red[32];
    const T *px = x + blockIdx.x * (int64_t)dim;
    T *py = y + blockIdx.x * (int64_t)dim;
    auto ld = [&](int d) { return cache_in_smem ? srow[d] : to_f(px[d]); };
    if (cache_in_smem) {
        for (int d = threadIdx.x; d < dim; d += blockDim.x) srow[d] = to_f(px[d]);
        __syncthreads();
    }
    if (MODE == 0) {
        float mx = -INFINITY;
        for (int d = threadIdx.x; d < dim; d += blockDim.x) mx = fmaxf(mx, ld(d));
        mx = block_max(mx, red);
        float s = 0.f;
        for (int d = threadIdx.x; d < dim; d += blockDim.x) s += expf(ld(d) - mx);
        s = block_sum(s, red);
        for (int d = threadIdx.x; d < dim; d += blockDim.x) py[d] = from_f<T>(expf(ld(d) - mx) / s);
    } else {
        float s = 0.f;
        for (int d = threadIdx.x; d < dim; d += blockDim.x) s += ld(d);
        float mu = block_sum(s, red) / (float)dim;
        float q = 0.f;
        for (int d = threadIdx.x; d < dim; d += blockDim.x) {
            float t = ld(d) - mu;
            q += t * t;
        }
        float rs = rsqrtf(block_sum(q, red) / (float)dim + eps);
        for (int d = threadIdx.x; d < dim; d += blockDim.x) {
            float sc = to_f(scale[scale_size == dim ? d : 0]);
            float bi = bias ? to_f(bias[bias_size == dim ? d : 0]) : 0.f;
            py[d] = from_f<T>(sc * (ld(d) - mu) * rs + bi);
        }
    }
}

// ------------------------------------------------------------------ strided axis: thread per (outer, inner)
template <typename T, int MODE>
__global__ void __launch_bounds__(256) strided_kernel(const T *__restrict__ x, T *__restrict__ y,
                                                      const T *__restrict__ scale, const T *__restrict__ bias,
                                                      int64_t outer, int dim, int64_t inner, int scale_size,
                                                      int bias_size, float eps) {
    pdl_trigger();
    pdl_wait();
    int64_t idx = blockIdx.x * (int64_t)blockDim.x + threadIdx.x;
    if (idx >= outer * inner) return;
    int64_t o = idx / inner, i = idx - o * inner;
    const T *px = x + o * dim * inner + i;
    T *py = y + o * dim * inner + i;
    if (MODE == 0) {
        float mx = -INFINITY;
        for (int d = 0; d < dim; ++d) mx = fmaxf(mx, to_f(px[d * inner]));
        float s = 0.f;
        for (int d = 0; d < dim; ++d) s += expf(to_f(px[d * inner]) - mx);
        for (int d = 0; d < dim; ++d) py[d * inner] = from_f<T>(expf(to_f(px[d * inner]) - mx) / s);
    } else {
        float s = 0.f;
        for (int d = 0; d < dim; ++d) s += to_f(px[d * inner]);
        float mu = s / (float)dim, q = 0.f;
        for (int d = 0; d < dim; ++d) {
            float t = to_f(px[d * inner]) - mu;
            q += t * t;
        }
        float rs = rsqrtf(q / (float)dim + eps);
        for (int d = 0; d < dim; ++d) {
            float sc = to_f(scale[scale_size == dim ? d : 0]);
            float bi = bias ? to_f(bias[bias_size == dim ? d : 0]) : 0.f;
            py[d * inner] = from_f<T>(sc * (to_f(px[d * inner]) - mu) * rs + bi);
        }
    }
}

template <typename T, int MODE>
static int launch_rowop(const char *name, const T *x, T *y, const T *scale, const T *bias, int64_t outer,
                        int dim, int64_t inner, int scale_size, int bias_size, float eps, cudaStream_t st) {
    if (outer * inner == 0 || dim == 0) return 0;
    if (inner != 1) {
        int64_t n = outer * inner;
        return launch(name, strided_kernel<T, MODE>, {dim3((unsigned)((n + 255) / 256)), dim3(256), 0, st}, x, y, scale, bias,
                      outer, dim, inner, scale_size, bias_size, eps);
    }
    if (dim <= 1024) {
        int64_t rows = outer;
        const LaunchCfg c{dim3((unsigned)((rows * 32 + 255) / 256)), dim3(256), 0, st};
#define RW(I) return launch(name, row_warp_kernel<T, I, MODE>, c, x, y, scale, bias, rows, dim, scale_size, bias_size, eps)
#define RWV(I) return launch(name, row_warp_vec_kernel<T, I, MODE>, c, x, y, scale, bias, rows, dim, scale_size, bias_size, eps)
        bool vec_ok = false;
        if constexpr (sizeof(T) == 2)
            vec_ok = dim % 8 == 0 && dim >= 64 && aligned16(x) && aligned16(y) && (!scale || scale_size != dim || aligned16(scale)) &&
                     (!bias || bias_size != dim || aligned16(bias));
        if (vec_ok) {
            if constexpr (sizeof(T) == 2) {
                if (dim <= 256) RWV(1);
                else if (dim <= 512) RWV(2);
                else if (dim <= 768) RWV(3);
                else RWV(4);
            }
        } else
        if (dim <= 32) RW(1);
        else if (dim <= 64) RW(2);
        else if (dim <= 128) RW(4);
        else if (dim <= 256) RW(8);
        else if (dim <= 512) RW(16);
        else RW(32);
#undef RW
#undef RWV
    }
    // a cached row of up to 12288 floats fills the 48 KB a block gets without opting in, and the kernel's static reduction
    // buffer comes on top: the launch raises the dynamic limit to the row
    int cache = dim <= 12288;
    int threads = dim >= 8192 ? 1024 : 512;
    const int smem = cache ? dim * (int)sizeof(float) : 0;
    return launch(name, row_block_kernel<T, MODE>, {dim3((unsigned)outer), dim3(threads), smem, st}, x, y, scale, bias, dim,
                  scale_size, bias_size, eps, cache);
}

// ------------------------------------------------------------------ RMSNorm
// y = T( T(x * rsqrt(mean(x^2) + 1e-5)) * w )   (rms_norm.cu:46,52 -- round before weight)
// ONE = the row fits one 16-byte vector per thread (hidden <= 8 * blockDim for 2-byte types): the row stays in registers
// between the two passes.  WCONST = the weight is a graph constant: it is fetched ahead of griddepcontrol.wait.
template <typename T, bool ONE, bool WCONST>
__global__ void __launch_bounds__(512) rmsnorm_kernel(const T *__restrict__ x, const T *__restrict__ w,
                                                      T *__restrict__ y, int hidden, bool vec) {
    pdl_trigger();
    constexpr int V = Vec16<T>::N;
    __shared__ float red[32];
    const T *px = x + blockIdx.x * (int64_t)hidden;
    T *py = y + blockIdx.x * (int64_t)hidden;
    if (ONE) {
        const int i = threadIdx.x, nv = hidden / V;
        Vec16<T> a, ww, o;
        if (WCONST && i < nv) ww = ld16(w + i * V);
        pdl_wait();
        float ss = 0.f;
        if (i < nv) {
            a = ld16(px + i * V);
            if (!WCONST) ww = ld16(w + i * V);
#pragma unroll
            for (int j = 0; j < V; ++j) {
                float f = to_f(a.v[j]);
                ss += f * f;
            }
        }
        const float r = rsqrtf(block_sum(ss, red) / (float)hidden + 0.00001f);
        if (i < nv) {
#pragma unroll
            for (int j = 0; j < V; ++j) o.v[j] = from_f<T>(round_t<T>(to_f(a.v[j]) * r) * to_f(ww.v[j]));
            st16(py + i * V, o);
        }
        return;
    }
    pdl_wait();
    float ss = 0.f;
    if (vec) {
        int nv = hidden / V;
        for (int i = threadIdx.x; i < nv; i += blockDim.x) {
            Vec16<T> a = ld16(px + i * V);
#pragma unroll
            for (int j = 0; j < V; ++j) {
                float f = to_f(a.v[j]);
                ss += f * f;
            }
        }
    } else {
        for (int i = threadIdx.x; i < hidden; i += blockDim.x) {
            float f = to_f(px[i]);
            ss += f * f;
        }
    }
    float r = rsqrtf(block_sum(ss, red) / (float)hidden + 0.00001f);
    if (vec) {
        int nv = hidden / V;
        for (int i = threadIdx.x; i < nv; i += blockDim.x) {
            Vec16<T> a = ld16(px + i * V), ww = ld16(w + i * V), o;
#pragma unroll
            for (int j = 0; j < V; ++j) o.v[j] = from_f<T>(round_t<T>(to_f(a.v[j]) * r) * to_f(ww.v[j]));
            st16(py + i * V, o);
        }
    } else {
        for (int i = threadIdx.x; i < hidden; i += blockDim.x)
            py[i] = from_f<T>(round_t<T>(to_f(px[i]) * r) * to_f(w[i]));
    }
}

// ------------------------------------------------------------------ RoPE (rotate-half)
// column pair c of a head rotates by p x 10000^(-2c / dim_head), or with an inv_freq table (TABLE) by fp32(p x inv_freq[c])
template <typename T, typename P, bool TABLE>
__device__ __forceinline__ void rope_body(const P *__restrict__ pos, const T *__restrict__ x, T *__restrict__ y, int64_t rows,
                                          int dim_model, int dim_head, const float *__restrict__ inv_freq) {
    pdl_trigger();
    pdl_wait();
    int half = dim_head >> 1;
    int pairs_per_row = dim_model >> 1;
    int64_t total = rows * pairs_per_row;
    for (int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; i < total;
         i += (int64_t)gridDim.x * blockDim.x) {
        int64_t row = i / pairs_per_row;
        int pr = (int)(i - row * pairs_per_row);
        int head = pr / half, c = pr - head * half;
        int lo = head * dim_head + c, hi = lo + half;
        float p = (float)(int)pos[row];
        float freq = TABLE ? __fmul_rn(p, inv_freq[c]) : p * powf(10000.f, -(float)(c * 2) / (float)dim_head);
        float cs = round_t<T>(cosf(freq)), sn = round_t<T>(sinf(freq));
        float xl = to_f(x[row * dim_model + lo]), xh = to_f(x[row * dim_model + hi]);
        // arithmetic in T exactly as rope.cu:21-29: each product and the sum rounded to T (__fmul_rn: for fp32 the compiler must
        // not fuse a product into the sum -- the RoPE folded into attention has to give the same bits)
        float ol = round_t<T>(__fmul_rn(xl, cs)) - round_t<T>(__fmul_rn(xh, sn));
        float oh = round_t<T>(__fmul_rn(xh, cs)) + round_t<T>(__fmul_rn(xl, sn));
        y[row * dim_model + lo] = from_f<T>(ol);
        y[row * dim_model + hi] = from_f<T>(oh);
    }
}
template <typename T, typename P>
__global__ void __launch_bounds__(256) rope_kernel(const P *__restrict__ pos, const T *__restrict__ x,
                                                   T *__restrict__ y, int64_t rows, int dim_model,
                                                   int dim_head) {
    rope_body<T, P, false>(pos, x, y, rows, dim_model, dim_head, nullptr);  // (pdl_trigger / pdl_wait inside)
}
template <typename T, typename P>
__global__ void __launch_bounds__(256) rope_freq_kernel(const P *__restrict__ pos, const T *__restrict__ x, T *__restrict__ y,
                                                        int64_t rows, int dim_model, int dim_head,
                                                        const float *__restrict__ inv_freq) {
    rope_body<T, P, true>(pos, x, y, rows, dim_model, dim_head, inv_freq);  // (pdl_trigger / pdl_wait inside)
}

// dim_model not a multiple of dim_head (the reference's own golden test runs dim_model = 32 against its hard-coded 128-wide
// heads, test_cuda_rope.cc:17-35 / rope.cc:25): one thread per column; a rotation partner beyond the row counts as 0 (the
// reference reads out of bounds there, quirk q2 -- its expected values are the cosines, i.e. partner = 0)
template <typename T, typename P>
__global__ void __launch_bounds__(256) rope_ragged_kernel(const P *__restrict__ pos, const T *__restrict__ x,
                                                          T *__restrict__ y, int64_t rows, int dim_model, int dim_head) {
    pdl_trigger();
    pdl_wait();
    const int half = dim_head >> 1;
    const int64_t total = rows * dim_model;
    for (int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; i < total; i += (int64_t)gridDim.x * blockDim.x) {
        const int64_t row = i / dim_model;
        const int col = (int)(i - row * dim_model);
        const int j = col % dim_head, c = j % half;
        const bool lo = j < half;
        const int pcol = lo ? col + half : col - half;
        const float p = (float)(int)pos[row];
        const float freq = p * powf(10000.f, -(float)(c * 2) / (float)dim_head);
        const float cs = round_t<T>(cosf(freq)), sn = round_t<T>(sinf(freq));
        const float xv = to_f(x[row * dim_model + col]), xp = pcol < dim_model ? to_f(x[row * dim_model + pcol]) : 0.f;
        const float a = round_t<T>(__fmul_rn(xv, cs)), b = round_t<T>(__fmul_rn(xp, sn));
        const float o = lo ? a - b : a + b;
        y[row * dim_model + col] = from_f<T>(o);
    }
}

}  // namespace itb

using namespace itb;

extern "C" int it_b200_softmax(int dtype, const void *x, void *y, int64_t outer, int dim, int64_t inner,
                               void *stream) {
    ITB_DISPATCH_FLOAT(dtype, "softmax", {
        return launch_rowop<T, 0>("softmax", (const T *)x, (T *)y, nullptr, nullptr, outer, dim, inner, 0, 0, 0.f,
                                  (cudaStream_t)stream);
    });
    return 0;
}

extern "C" int it_b200_layernorm(int dtype, const void *x, const void *scale, const void *bias, void *y,
                                 int64_t outer, int dim, int64_t inner, int scale_size, int bias_size,
                                 float eps, void *stream) {
    ITB_CHECK(scale_size == dim || scale_size == 1, "layernorm: scale size %d must be %d or 1", scale_size, dim);
    ITB_CHECK(!bias || bias_size == dim || bias_size == 1, "layernorm: bias size %d must be %d or 1", bias_size,
              dim);
    ITB_DISPATCH_FLOAT(dtype, "layernorm", {
        return launch_rowop<T, 1>("layernorm", (const T *)x, (T *)y, (const T *)scale, (const T *)bias, outer, dim,
                                  inner, scale_size, bias_size, eps, (cudaStream_t)stream);
    });
    return 0;
}

static int rmsnorm_impl(int dtype, const void *x, const void *w, void *y, int64_t tokens, int hidden, bool w_const,
                        void *stream) {
    if (tokens == 0 || hidden == 0) return 0;
    ITB_DISPATCH_FLOAT(dtype, "rmsnorm", {
        bool vec = aligned16(x) && aligned16(w) && aligned16(y) && hidden % Vec16<T>::N == 0;
        int threads = hidden >= 4096 ? 512 : (hidden >= 1024 ? 256 : 128);
        const bool one = vec && hidden / Vec16<T>::N <= threads;
        auto go = [&](auto kern) {
            return launch("rmsnorm", kern, {dim3((unsigned)tokens), dim3(threads), 0, (cudaStream_t)stream}, (const T *)x,
                          (const T *)w, (T *)y, hidden, vec);
        };
        if (one && w_const) return go(rmsnorm_kernel<T, true, true>);
        if (one) return go(rmsnorm_kernel<T, true, false>);
        return go(rmsnorm_kernel<T, false, false>);
    });
    return 0;
}

extern "C" int it_b200_rmsnorm(int dtype, const void *x, const void *w, void *y, int64_t tokens, int hidden,
                               void *stream) {
    return rmsnorm_impl(dtype, x, w, y, tokens, hidden, false, stream);
}

extern "C" int it_b200_rmsnorm_constw(int dtype, const void *x, const void *w, void *y, int64_t tokens, int hidden,
                                      void *stream) {
    return rmsnorm_impl(dtype, x, w, y, tokens, hidden, true, stream);
}

static int rope_impl(int dtype, const void *pos, int pos_dtype, const void *x, void *y, int B, int S, int dim_model,
                     int dim_head, const float *inv_freq, void *stream) {
    ITB_CHECK(dim_head > 0 && dim_head % 2 == 0, "rope: dim_head %d must be even", dim_head);
    int64_t rows = (int64_t)B * S;
    if (rows == 0) return 0;
    int64_t total = rows * (dim_model / 2);
    auto st = (cudaStream_t)stream;
    if (dim_model % dim_head != 0) {
        ITB_CHECK(!inv_freq, "rope: an inv_freq table needs dim_model (%d) to be a multiple of dim_head (%d)", dim_model, dim_head);
        ITB_CHECK(pos_dtype == ITB_I64 || pos_dtype == ITB_I32 || pos_dtype == ITB_U32, "rope: unsupported position dtype %d", pos_dtype);
        ITB_DISPATCH_FLOAT(dtype, "rope", {
            const LaunchCfg c{dim3(grid_for(rows * dim_model, 256)), dim3(256), 0, st};
            if (pos_dtype == ITB_I64)
                return launch("rope", rope_ragged_kernel<T, int64_t>, c, (const int64_t *)pos, (const T *)x, (T *)y, rows, dim_model, dim_head);
            return launch("rope", rope_ragged_kernel<T, int32_t>, c, (const int32_t *)pos, (const T *)x, (T *)y, rows, dim_model, dim_head);
        });
        return 0;
    }
    ITB_DISPATCH_FLOAT(dtype, "rope", {
        const LaunchCfg c{dim3(grid_for(total, 256)), dim3(256), 0, st};
        const bool p64 = pos_dtype == ITB_I64;
        if (!p64 && pos_dtype != ITB_I32 && pos_dtype != ITB_U32) ITB_FAIL("rope: unsupported position dtype %d", pos_dtype);
        if (inv_freq) {
            if (p64) return launch("rope", rope_freq_kernel<T, int64_t>, c, (const int64_t *)pos, (const T *)x, (T *)y, rows, dim_model, dim_head, inv_freq);
            return launch("rope", rope_freq_kernel<T, int32_t>, c, (const int32_t *)pos, (const T *)x, (T *)y, rows, dim_model, dim_head, inv_freq);
        }
        if (p64)
            return launch("rope", rope_kernel<T, int64_t>, c, (const int64_t *)pos, (const T *)x, (T *)y, rows, dim_model, dim_head);
        return launch("rope", rope_kernel<T, int32_t>, c, (const int32_t *)pos, (const T *)x, (T *)y, rows, dim_model, dim_head);
    });
    return 0;
}

extern "C" int it_b200_rope(int dtype, const void *pos, int pos_dtype, const void *x, void *y, int B, int S,
                            int dim_model, int dim_head, void *stream) {
    return rope_impl(dtype, pos, pos_dtype, x, y, B, S, dim_model, dim_head, nullptr, stream);
}

extern "C" int it_b200_rope_freq(int dtype, const void *pos, int pos_dtype, const void *x, void *y, int B, int S,
                                 int dim_model, int dim_head, const void *inv_freq, int freq_dtype, int64_t freq_len,
                                 void *stream) {
    ITB_CHECK(inv_freq, "rope: inv_freq table missing");
    ITB_CHECK(freq_dtype == ITB_F32, "rope: inv_freq must be f32 (dtype %d)", freq_dtype);
    ITB_CHECK(dim_head > 0 && freq_len >= dim_head / 2, "rope: inv_freq has %lld entries, dim_head %d needs %d",
              (long long)freq_len, dim_head, dim_head / 2);
    ITB_CHECK((reinterpret_cast<uintptr_t>(inv_freq) & 3) == 0, "rope: inv_freq must be 4-byte aligned");
    return rope_impl(dtype, pos, pos_dtype, x, y, B, S, dim_model, dim_head, (const float *)inv_freq, stream);
}
