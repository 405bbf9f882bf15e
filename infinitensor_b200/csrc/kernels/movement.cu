// movement.cu -- bit-exact data-movement kernels for sm_90a: Transpose, Concat/Split, Gather,
// Reshape-copy, Pad/Slice, Reduce, Pool2d, BatchNorm.  All are HBM-bound byte movers: the widest
// unit (up to 16 B) that divides every row length / offset / alignment is chosen on the host so
// accesses are 128-bit wherever the shapes allow; transposes go through a padded shared-memory tile
// so both the read and the write side stay coalesced.
//
// Replaces (reference): transpose.cu:10-78, split_concat.cu:28-84, gather.cu:31-55,
// reshape.cc:4-21, pad_slice.cu:6-47, reduce.cc:7-125, pooling.cc:8-95, batch_norm.cc:9-69.
#include <algorithm>
#include <initializer_list>
#include <type_traits>

#include "common.cuh"

namespace itb {

struct alignas(16) U16 { uint32_t a, b, c, d; };

static int pick_unit(int elem_size, std::initializer_list<int64_t> byte_counts,
                     std::initializer_list<const void *> ptrs) {
    for (int u = 16; u > elem_size; u >>= 1) {
        bool ok = true;
        for (int64_t b : byte_counts) ok = ok && (b % u == 0);
        for (const void *p : ptrs) ok = ok && ((reinterpret_cast<uintptr_t>(p) % u) == 0);
        if (ok) return u;
    }
    return elem_size;
}

#define UNIT_DISPATCH(u, NAME, ...)                                                            \
    switch (u) {                                                                               \
    case 1: { using E = uint8_t; __VA_ARGS__; } break;                                         \
    case 2: { using E = uint16_t; __VA_ARGS__; } break;                                        \
    case 4: { using E = uint32_t; __VA_ARGS__; } break;                                        \
    case 8: { using E = uint64_t; __VA_ARGS__; } break;                                        \
    case 16: { using E = U16; __VA_ARGS__; } break;                                            \
    default: ITB_FAIL("%s: unsupported unit size %d", NAME, u);                                \
    }

template <typename E>
__global__ void __launch_bounds__(256) copy_kernel(const E *__restrict__ x, E *__restrict__ y, int64_t n) {
    pdl_trigger();
    pdl_wait();
    for (int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; i < n; i += (int64_t)gridDim.x * blockDim.x)
        y[i] = x[i];
}

// ---------------------------------------------------------------- transpose
// rows contiguous on both sides: out_row[r] (len L units) = in + sum(coord * in_stride)
template <typename E>
__global__ void __launch_bounds__(256) permute_rows_kernel(const E *__restrict__ x, E *__restrict__ y,
                                                           int64_t n_units, int64_t L, int rank, Dims8 odims,
                                                           Dims8 istr) {
    pdl_trigger();
    pdl_wait();
    // odims/istr describe the OUTER dims (units of E for strides); innermost run of L units is contiguous
    for (int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; i < n_units;
         i += (int64_t)gridDim.x * blockDim.x) {
        int64_t row = i / L, c = i - row * L;
        int64_t rem = row, off = 0;
        for (int d = rank - 1; d >= 0; --d) {
            int64_t q = rem / odims.v[d], ci = rem - q * odims.v[d];
            rem = q;
            off += ci * istr.v[d];
        }
        y[i] = x[off + c];
    }
}

// general case: tile 32x32 over (output-last dim j, the output dim q whose input stride is 1)
template <typename E>
__global__ void __launch_bounds__(256) permute_tiled_kernel(const E *__restrict__ x, E *__restrict__ y, int rank,
                                                            Dims8 odims, Dims8 istr, Dims8 ostr, int q,
                                                            int64_t tiles_j, int64_t tiles_i) {
    pdl_trigger();
    pdl_wait();
    __shared__ E tile[32][33];
    int64_t b = blockIdx.x;
    int64_t tj = b % tiles_j;
    b /= tiles_j;
    int64_t ti = b % tiles_i;
    b /= tiles_i;
    // remaining dims (all but q and rank-1) decode `b`
    int64_t in_base = 0, out_base = 0;
    for (int d = rank - 2; d >= 0; --d) {
        if (d == q) continue;
        int64_t qq = b / odims.v[d], ci = b - qq * odims.v[d];
        b = qq;
        in_base += ci * istr.v[d];
        out_base += ci * ostr.v[d];
    }
    int64_t J = odims.v[rank - 1], I = odims.v[q];
    int64_t S = istr.v[rank - 1], OQ = ostr.v[q];
    int tx = threadIdx.x & 31, ty = threadIdx.x >> 5;
    for (int r = ty; r < 32; r += 8) {
        int64_t j = tj * 32 + r, i = ti * 32 + tx;
        if (j < J && i < I) tile[r][tx] = x[in_base + j * S + i];
    }
    __syncthreads();
    for (int r = ty; r < 32; r += 8) {
        int64_t i = ti * 32 + r, j = tj * 32 + tx;
        if (j < J && i < I) y[out_base + i * OQ + j] = tile[tx][r];
    }
}

// ---------------------------------------------------------------- concat / split
struct Parts {
    const void *ptr[32];
    int64_t len[32];  // row length of each part, in units
    int64_t off[32];  // column offset inside the joined row, in units
};

template <typename E, bool SPLIT>
__global__ void __launch_bounds__(256) concat_split_kernel(Parts parts, E *joined, int64_t outer, int64_t Ltot) {
    pdl_trigger();
    pdl_wait();
    int p = blockIdx.y;
    int64_t L = parts.len[p], off = parts.off[p];
    E *part = (E *)parts.ptr[p];
    int64_t n = outer * L;
    for (int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; i < n; i += (int64_t)gridDim.x * blockDim.x) {
        int64_t o = i / L, c = i - o * L;
        if (SPLIT)
            part[i] = joined[o * Ltot + off + c];
        else
            joined[o * Ltot + off + c] = part[i];
    }
}

// ---------------------------------------------------------------- gather
template <typename E, typename I>
__global__ void __launch_bounds__(256) gather_kernel(const E *__restrict__ data, const I *__restrict__ idx,
                                                     E *__restrict__ out, int64_t outer, int64_t axis_len,
                                                     int64_t inner, int64_t n_idx) {
    pdl_trigger();
    pdl_wait();
    int64_t n = outer * n_idx * inner;
    for (int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; i < n; i += (int64_t)gridDim.x * blockDim.x) {
        int64_t c = i % inner, t = i / inner;
        int64_t j = t % n_idx, o = t / n_idx;
        int64_t g = (int64_t)idx[j];
        if (g < 0) g += axis_len;
        out[i] = data[(o * axis_len + g) * inner + c];
    }
}

// ---------------------------------------------------------------- pad / slice (strided window)
template <typename E>
__global__ void __launch_bounds__(256) pad_slice_kernel(const E *__restrict__ in, E *__restrict__ out, int64_t n,
                                                        int rank, Dims8 din, Dims8 dout, Dims8 start, Dims8 step) {
    pdl_trigger();
    pdl_wait();
    for (int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; i < n; i += (int64_t)gridDim.x * blockDim.x) {
        int64_t rem = i, off = 0, mul = 1;
        bool inside = true;
        for (int d = rank - 1; d >= 0; --d) {
            int64_t q = rem / dout.v[d], ci = rem - q * dout.v[d];
            rem = q;
            int64_t src = start.v[d] + ci * step.v[d];
            inside = inside && src >= 0 && src < din.v[d];
            off += src * mul;
            mul *= din.v[d];
        }
        E zero{};
        out[i] = inside ? in[off] : zero;
    }
}

// ---------------------------------------------------------------- reduce (warp per output)
template <typename T>
__global__ void __launch_bounds__(256) reduce_kernel(const T *__restrict__ x, T *__restrict__ y, int64_t n_out,
                                                     int64_t R, int krank, Dims8 kdims, Dims8 kstr, int rrank,
                                                     Dims8 rdims, Dims8 rstr, float scale) {
    pdl_trigger();
    pdl_wait();
    int lane = threadIdx.x & 31;
    int64_t o = (blockIdx.x * (int64_t)blockDim.x + threadIdx.x) >> 5;
    if (o >= n_out) return;
    int64_t rem = o, base = 0;
    for (int d = krank - 1; d >= 0; --d) {
        int64_t q = rem / kdims.v[d], ci = rem - q * kdims.v[d];
        rem = q;
        base += ci * kstr.v[d];
    }
    float acc = 0.f;
    for (int64_t r = lane; r < R; r += 32) {
        int64_t rr = r, off = base;
        for (int d = rrank - 1; d >= 0; --d) {
            int64_t q = rr / rdims.v[d], ci = rr - q * rdims.v[d];
            rr = q;
            off += ci * rstr.v[d];
        }
        acc += to_f(x[off]);
    }
    acc = warp_sum(acc);
    if (lane == 0) y[o] = from_f<T>(acc * scale);
}

// ---------------------------------------------------------------- pooling / batchnorm
template <typename T>
__global__ void __launch_bounds__(256) pool2d_kernel(int is_max, const T *__restrict__ x, T *__restrict__ y,
                                                     int64_t NC, int H, int W, int kh, int kw, int dh, int dw,
                                                     int ph, int pw, int sh, int sw, int OH, int OW) {
    pdl_trigger();
    pdl_wait();
    int64_t n = NC * OH * OW;
    for (int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; i < n; i += (int64_t)gridDim.x * blockDim.x) {
        int ow = (int)(i % OW);
        int64_t t = i / OW;
        int oh = (int)(t % OH);
        int64_t nc = t / OH;
        const T *px = x + nc * H * W;
        float acc = is_max ? -INFINITY : 0.f;
        for (int r = 0; r < kh; ++r) {
            int ih = oh * sh - ph + r * dh;
            if (ih < 0 || ih >= H) continue;
            for (int s = 0; s < kw; ++s) {
                int iw = ow * sw - pw + s * dw;
                if (iw < 0 || iw >= W) continue;
                float v = to_f(px[ih * W + iw]);
                acc = is_max ? fmaxf(acc, v) : acc + v;
            }
        }
        if (!is_max) acc /= (float)(kh * kw);  // count-include-pad (pooling.cc:88)
        y[i] = from_f<T>(acc);
    }
}

// the same pooling over NHWC activations ([N, H, W, C], C % 8 == 0; 2-byte types): one thread = 8 channels (16 bytes) of one output
// pixel, so every tap is one coalesced 16-byte load along C.  Same arithmetic as pool2d_kernel (fp32 max / sum, count-include-pad).
template <typename T>
__global__ void __launch_bounds__(256) pool2d_nhwc_kernel(int is_max, const T *__restrict__ x, T *__restrict__ y, int64_t total,
                                                          int C8, int H, int W, int kh, int kw, int dh, int dw, int ph, int pw,
                                                          int sh, int sw, int OH, int OW) {
    pdl_trigger();
    pdl_wait();
    constexpr int V = 8;
    for (int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; i < total; i += (int64_t)gridDim.x * blockDim.x) {
        const int c8 = (int)(i % C8);
        int64_t t = i / C8;
        const int ow = (int)(t % OW);
        t /= OW;
        const int oh = (int)(t % OH);
        const int64_t n = t / OH;
        float acc[V];
#pragma unroll
        for (int e = 0; e < V; ++e) acc[e] = is_max ? -INFINITY : 0.f;
        for (int r = 0; r < kh; ++r) {
            const int ih = oh * sh - ph + r * dh;
            if (ih < 0 || ih >= H) continue;
            for (int s = 0; s < kw; ++s) {
                const int iw = ow * sw - pw + s * dw;
                if (iw < 0 || iw >= W) continue;
                const Vec16<T> v = ld16(x + (((n * H + ih) * W + iw) * C8 + c8) * V);
#pragma unroll
                for (int e = 0; e < V; ++e) {
                    const float f = to_f(v.v[e]);
                    acc[e] = is_max ? fmaxf(acc[e], f) : acc[e] + f;
                }
            }
        }
        Vec16<T> o;
#pragma unroll
        for (int e = 0; e < V; ++e) o.v[e] = from_f<T>(is_max ? acc[e] : acc[e] / (float)(kh * kw));
        st16(y + i * V, o);
    }
}

// 3x3 windows (the ResNet max pool) with the nine taps unrolled: all loads of a thread are issued before the first use (clamped
// addresses, validity applied afterwards) -- the generic kernel above, one dependent load at a time behind its bounds checks, is
// latency-bound there
template <typename T>
__global__ void __launch_bounds__(256) pool2d_nhwc3x3_kernel(int is_max, const T *__restrict__ x, T *__restrict__ y, int64_t total,
                                                             int C8, int H, int W, int ph, int pw, int sh, int sw, int OH, int OW) {
    pdl_trigger();
    pdl_wait();
    constexpr int V = 8;
    for (int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; i < total; i += (int64_t)gridDim.x * blockDim.x) {
        const int c8 = (int)(i % C8);
        int64_t t = i / C8;
        const int ow = (int)(t % OW);
        t /= OW;
        const int oh = (int)(t % OH);
        const int64_t n = t / OH;
        Vec16<T> v[9];
        bool ok[9];
#pragma unroll
        for (int r = 0; r < 3; ++r)
#pragma unroll
            for (int s = 0; s < 3; ++s) {
                const int ih = oh * sh - ph + r, iw = ow * sw - pw + s;
                ok[r * 3 + s] = ih >= 0 && ih < H && iw >= 0 && iw < W;
                const int ihc = min(max(ih, 0), H - 1), iwc = min(max(iw, 0), W - 1);
                v[r * 3 + s] = ld16(x + (((n * H + ihc) * W + iwc) * C8 + c8) * V);
            }
        Vec16<T> o;
#pragma unroll
        for (int e = 0; e < V; ++e) {
            float acc = is_max ? -INFINITY : 0.f;
#pragma unroll
            for (int k = 0; k < 9; ++k) {
                const float f = to_f(v[k].v[e]);
                if (ok[k]) acc = is_max ? fmaxf(acc, f) : acc + f;
            }
            o.v[e] = from_f<T>(is_max ? acc : acc / 9.f);
        }
        st16(y + i * V, o);
    }
}

// global average pool ([N, H, W, C] -> [N, 1, 1, C]): block = 32 channel chunks x 8 pixel groups, shared-memory reduction over the groups
// (the windowed kernel walks the H*W taps of one output serially)
template <typename T>
__global__ void __launch_bounds__(256) global_avgpool_nhwc_kernel(const T *__restrict__ x, T *__restrict__ y, int C8, int HW) {
    pdl_trigger();
    pdl_wait();
    constexpr int V = 8;
    __shared__ float part[8][32][V + 1];
    const int cx = threadIdx.x & 31, pg = threadIdx.x >> 5;
    const int c8 = blockIdx.x * 32 + cx;
    const int64_t n = blockIdx.y;
    float acc[V];
#pragma unroll
    for (int e = 0; e < V; ++e) acc[e] = 0.f;
    if (c8 < C8)
        for (int p = pg; p < HW; p += 8) {
            const Vec16<T> v = ld16(x + ((n * HW + p) * C8 + c8) * V);
#pragma unroll
            for (int e = 0; e < V; ++e) acc[e] += to_f(v.v[e]);
        }
#pragma unroll
    for (int e = 0; e < V; ++e) part[pg][cx][e] = acc[e];
    __syncthreads();
    if (pg == 0 && c8 < C8) {
        Vec16<T> o;
#pragma unroll
        for (int e = 0; e < V; ++e) {
            float s = 0.f;
#pragma unroll
            for (int g = 0; g < 8; ++g) s += part[g][cx][e];
            o.v[e] = from_f<T>(s / (float)HW);
        }
        st16(y + (n * C8 + c8) * V, o);
    }
}

// y = scale[c] * (x - mean[c]) / sqrt(var[c] + eps) + bias[c] over NCHW (batch_norm.cc:9-69 semantics; fp32 parameters).
// VEC: one thread = one 16-byte vector inside a single (n, c) plane (HW % V == 0), one channel lookup per vector.
template <typename T, bool VEC>
__global__ void __launch_bounds__(256) batchnorm_kernel(const T *__restrict__ x, const float *__restrict__ mean,
                                                        const float *__restrict__ var,
                                                        const float *__restrict__ scale,
                                                        const float *__restrict__ bias, T *__restrict__ y,
                                                        int64_t n, int C, int64_t HW, float eps, int relu) {
    pdl_trigger();
    pdl_wait();
    constexpr int V = VEC ? Vec16<T>::N : 1;
    const int64_t nv = n / V;
    for (int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; i < nv; i += (int64_t)gridDim.x * blockDim.x) {
        const int c = (int)(((i * V) / HW) % C);
        const float rs = bn_rs(var[c], eps), sc = scale[c], mu = mean[c], bi = bias[c];
        if (VEC) {
            const Vec16<T> in = ld16(x + i * V);
            Vec16<T> out;
#pragma unroll
            for (int j = 0; j < V; ++j) {
                float v = bn_apply(to_f(in.v[j]), mu, rs, sc, bi);
                if (relu) v = round_t<T>(v) > 0.f ? v : 0.f;
                out.v[j] = from_f<T>(v);
            }
            st16(y + i * V, out);
        } else {
            float v = bn_apply(to_f(x[i]), mu, rs, sc, bi);
            if (relu) v = round_t<T>(v) > 0.f ? v : 0.f;
            y[i] = from_f<T>(v);
        }
    }
}

}  // namespace itb

using namespace itb;

extern "C" int it_b200_copy(const void *src, void *dst, int64_t bytes, void *stream) {
    if (bytes == 0 || src == dst) return 0;
    // a kernel (not cudaMemcpyAsync) so the copy stays inside the PDL chain of the step
    int u = pick_unit(1, {bytes}, {src, dst});
    int64_t n = bytes / u;
    UNIT_DISPATCH(u, "copy", {
        return launch("copy", copy_kernel<E>, {dim3(grid_for(n, 256)), dim3(256), 0, (cudaStream_t)stream}, (const E *)src,
                      (E *)dst, n);
    });
    return 0;
}

extern "C" int it_b200_transpose(int elem_size, const void *x, void *y, int rank, const int64_t *dims_in,
                                 const int *perm, void *stream) {
    ITB_CHECK(rank >= 1 && rank <= ITB_MAX_RANK, "transpose: rank %d out of range", rank);
    auto st = (cudaStream_t)stream;
    int64_t in_str[ITB_MAX_RANK], n = 1;
    for (int d = rank - 1; d >= 0; --d) {
        in_str[d] = n;
        n *= dims_in[d];
    }
    if (n == 0) return 0;
    // output-ordered dims with their input strides; drop size-1 dims; merge runs adjacent in both
    int64_t od[ITB_MAX_RANK], is[ITB_MAX_RANK];
    int r = 0;
    for (int k = 0; k < rank; ++k) {
        ITB_CHECK(perm[k] >= 0 && perm[k] < rank, "transpose: bad perm[%d]=%d", k, perm[k]);
        int64_t d = dims_in[perm[k]], s = in_str[perm[k]];
        if (d == 1) continue;
        if (r > 0 && is[r - 1] == s * d) {
            od[r - 1] *= d;
            is[r - 1] = s;
        } else {
            od[r] = d;
            is[r] = s;
            ++r;
        }
    }
    if (r == 0 || (r == 1 && is[0] == 1)) return it_b200_copy(x, y, n * elem_size, stream);
    if (is[r - 1] == 1) {
        // innermost run contiguous on both sides: vectorised row copy
        int64_t Lb = od[r - 1] * elem_size;
        int64_t min_stride_b = Lb;
        for (int k = 0; k < r - 1; ++k) min_stride_b = std::min<int64_t>(min_stride_b, is[k] * elem_size);
        int u = elem_size;
        for (int cand = 16; cand > elem_size; cand >>= 1) {
            bool ok = Lb % cand == 0 && (uintptr_t)x % cand == 0 && (uintptr_t)y % cand == 0;
            for (int k = 0; k < r - 1; ++k) ok = ok && (is[k] * elem_size) % cand == 0;
            if (ok) { u = cand; break; }
        }
        Dims8 odims{}, istr{};
        for (int k = 0; k < r - 1; ++k) {
            odims.v[k] = od[k];
            istr.v[k] = is[k] * elem_size / u;
        }
        int64_t L = Lb / u, units = n * elem_size / u;
        UNIT_DISPATCH(u, "transpose", {
            return launch("transpose", permute_rows_kernel<E>, {dim3(grid_for(units, 256)), dim3(256), 0, st}, (const E *)x, (E *)y,
                          units, L, r - 1, odims, istr);
        });
        return 0;
    }
    // general: find q with input stride 1
    int q = -1;
    for (int k = 0; k < r - 1; ++k)
        if (is[k] == 1) q = k;
    ITB_CHECK(q >= 0, "transpose: internal: no unit-stride dim");
    Dims8 odims{}, istr{}, ostr{};
    int64_t acc = 1;
    for (int k = r - 1; k >= 0; --k) {
        odims.v[k] = od[k];
        istr.v[k] = is[k];
        ostr.v[k] = acc;
        acc *= od[k];
    }
    int64_t tiles_j = (od[r - 1] + 31) / 32, tiles_i = (od[q] + 31) / 32;
    int64_t batch = n / (od[r - 1] * od[q]);
    int64_t blocks = tiles_j * tiles_i * batch;
    ITB_CHECK(blocks < (1ll << 31), "transpose: grid too large");
    const LaunchCfg c{dim3((unsigned)blocks), dim3(256), 0, st};
    switch (elem_size) {
    case 1: return launch("transpose", permute_tiled_kernel<uint8_t>, c, (const uint8_t *)x, (uint8_t *)y, r, odims, istr, ostr, q, tiles_j, tiles_i);
    case 2: return launch("transpose", permute_tiled_kernel<uint16_t>, c, (const uint16_t *)x, (uint16_t *)y, r, odims, istr, ostr, q, tiles_j, tiles_i);
    case 4: return launch("transpose", permute_tiled_kernel<uint32_t>, c, (const uint32_t *)x, (uint32_t *)y, r, odims, istr, ostr, q, tiles_j, tiles_i);
    case 8: return launch("transpose", permute_tiled_kernel<uint64_t>, c, (const uint64_t *)x, (uint64_t *)y, r, odims, istr, ostr, q, tiles_j, tiles_i);
    default: ITB_FAIL("transpose: unsupported element size %d", elem_size);
    }
}

template <bool SPLIT>
static int concat_split_impl(const char *name, int elem_size, int n_parts, const void *const *parts,
                             const int64_t *axis_len, void *joined, int64_t outer, int64_t inner,
                             cudaStream_t st) {
    ITB_CHECK(n_parts >= 1, "%s: no parts", name);
    int64_t tot = 0;
    for (int p = 0; p < n_parts; ++p) tot += axis_len[p];
    if (outer * tot * inner == 0) return 0;
    // widest unit dividing every row length / offset and every pointer
    int u = 16;
    for (; u > elem_size; u >>= 1) {
        bool ok = (uintptr_t)joined % u == 0 && (tot * inner * elem_size) % u == 0;
        int64_t off = 0;
        for (int p = 0; p < n_parts && ok; ++p) {
            ok = ok && (uintptr_t)parts[p] % u == 0 && (axis_len[p] * inner * elem_size) % u == 0 &&
                 (off * inner * elem_size) % u == 0;
            off += axis_len[p];
        }
        if (ok) break;
    }
    int64_t Ltot = tot * inner * elem_size / u, off = 0;
    for (int p0 = 0; p0 < n_parts; p0 += 32) {
        Parts ps{};
        int cnt = std::min(32, n_parts - p0);
        int64_t max_n = 0;
        for (int p = 0; p < cnt; ++p) {
            ps.ptr[p] = parts[p0 + p];
            ps.len[p] = axis_len[p0 + p] * inner * elem_size / u;
            ps.off[p] = off;
            off += ps.len[p];
            max_n = std::max(max_n, ps.len[p] * outer);
        }
        if (max_n == 0) continue;
        dim3 grid(grid_for(max_n, 256, 4), cnt);
        UNIT_DISPATCH(u, name, {
            if (launch(name, concat_split_kernel<E, SPLIT>, {grid, dim3(256), 0, st}, ps, (E *)joined, outer, Ltot)) return 1;
        });
    }
    return 0;
}

extern "C" int it_b200_concat(int elem_size, int n_parts, const void *const *parts, const int64_t *axis_len,
                              void *out, int64_t outer, int64_t inner, void *stream) {
    return concat_split_impl<false>("concat", elem_size, n_parts, parts, axis_len, out, outer, inner,
                                    (cudaStream_t)stream);
}

extern "C" int it_b200_split(int elem_size, int n_parts, void *const *parts, const int64_t *axis_len,
                             const void *in, int64_t outer, int64_t inner, void *stream) {
    return concat_split_impl<true>("split", elem_size, n_parts, (const void *const *)parts, axis_len, (void *)in,
                                   outer, inner, (cudaStream_t)stream);
}

extern "C" int it_b200_gather(int elem_size, int idx_dtype, const void *data, const void *idx, void *out,
                              int64_t outer, int64_t axis_len, int64_t inner, int64_t n_idx, void *stream) {
    ITB_CHECK(idx_dtype == ITB_I32 || idx_dtype == ITB_I64 || idx_dtype == ITB_U32,
              "gather: index dtype %d must be int32/int64", idx_dtype);
    if (outer * n_idx * inner == 0) return 0;
    auto st = (cudaStream_t)stream;
    int u = pick_unit(elem_size, {inner * elem_size}, {data, out});
    int64_t inner_u = inner * elem_size / u;
    int64_t n = outer * n_idx * inner_u;
    const LaunchCfg c{dim3(grid_for(n, 256)), dim3(256), 0, st};
    UNIT_DISPATCH(u, "gather", {
        if (idx_dtype == ITB_I64)
            return launch("gather", gather_kernel<E, int64_t>, c, (const E *)data, (const int64_t *)idx, (E *)out, outer, axis_len,
                          inner_u, n_idx);
        return launch("gather", gather_kernel<E, int32_t>, c, (const E *)data, (const int32_t *)idx, (E *)out, outer, axis_len,
                      inner_u, n_idx);
    });
    return 0;
}

extern "C" int it_b200_pad_slice(int elem_size, const void *in, void *out, int rank, const int64_t *dims_in,
                                 const int64_t *dims_out, const int64_t *start, const int64_t *step,
                                 void *stream) {
    ITB_CHECK(rank >= 1 && rank <= ITB_MAX_RANK, "pad_slice: rank %d out of range", rank);
    Dims8 din{}, dout{}, s{}, t{};
    int64_t n = 1;
    for (int d = 0; d < rank; ++d) {
        din.v[d] = dims_in[d];
        dout.v[d] = dims_out[d];
        s.v[d] = start[d];
        t.v[d] = step[d];
        n *= dims_out[d];
    }
    if (n == 0) return 0;
    auto st = (cudaStream_t)stream;
    const LaunchCfg c{dim3(grid_for(n, 256)), dim3(256), 0, st};
    switch (elem_size) {
    case 1: return launch("pad_slice", pad_slice_kernel<uint8_t>, c, (const uint8_t *)in, (uint8_t *)out, n, rank, din, dout, s, t);
    case 2: return launch("pad_slice", pad_slice_kernel<uint16_t>, c, (const uint16_t *)in, (uint16_t *)out, n, rank, din, dout, s, t);
    case 4: return launch("pad_slice", pad_slice_kernel<uint32_t>, c, (const uint32_t *)in, (uint32_t *)out, n, rank, din, dout, s, t);
    case 8: return launch("pad_slice", pad_slice_kernel<uint64_t>, c, (const uint64_t *)in, (uint64_t *)out, n, rank, din, dout, s, t);
    default: ITB_FAIL("pad_slice: unsupported element size %d", elem_size);
    }
}

extern "C" int it_b200_reduce(int dtype, int is_mean, const void *x, void *y, int rank, const int64_t *dims,
                              const int *reduce_mask, void *stream) {
    ITB_CHECK(rank >= 1 && rank <= ITB_MAX_RANK, "reduce: rank %d out of range", rank);
    Dims8 kd{}, ks{}, rd{}, rs{};
    int kr = 0, rr = 0;
    int64_t str = 1, n_out = 1, R = 1;
    int64_t strides[ITB_MAX_RANK];
    for (int d = rank - 1; d >= 0; --d) {
        strides[d] = str;
        str *= dims[d];
    }
    for (int d = 0; d < rank; ++d) {
        if (reduce_mask[d]) {
            rd.v[rr] = dims[d];
            rs.v[rr++] = strides[d];
            R *= dims[d];
        } else {
            kd.v[kr] = dims[d];
            ks.v[kr++] = strides[d];
            n_out *= dims[d];
        }
    }
    if (n_out == 0) return 0;
    float scale = is_mean ? 1.0f / (float)R : 1.0f;
    auto st = (cudaStream_t)stream;
    unsigned grid = (unsigned)((n_out * 32 + 255) / 256);
    ITB_DISPATCH_FLOAT(dtype, "reduce", {
        return launch("reduce", reduce_kernel<T>, {dim3(grid), dim3(256), 0, st}, (const T *)x, (T *)y, n_out, R, kr, kd, ks, rr, rd,
                      rs, scale);
    });
    return 0;
}

extern "C" int it_b200_pool2d(int dtype, int is_max, const void *x, void *y, int N, int C, int H, int W, int kh,
                              int kw, int dh, int dw, int ph, int pw, int sh, int sw, int OH, int OW,
                              void *stream) {
    int64_t n = (int64_t)N * C * OH * OW;
    if (n == 0) return 0;
    ITB_DISPATCH_FLOAT(dtype, "pool2d", {
        return launch("pool2d", pool2d_kernel<T>, {dim3(grid_for(n, 256)), dim3(256), 0, (cudaStream_t)stream}, is_max, (const T *)x,
                      (T *)y, (int64_t)N * C, H, W, kh, kw, dh, dw, ph, pw, sh, sw, OH, OW);
    });
    return 0;
}

extern "C" int it_b200_pool2d_nhwc(int dtype, int is_max, const void *x, void *y, int N, int C, int H, int W, int kh, int kw,
                                   int dh, int dw, int ph, int pw, int sh, int sw, int OH, int OW, void *stream) {
    ITB_CHECK((dtype == ITB_F16 || dtype == ITB_BF16) && C % 8 == 0 && aligned16(x) && aligned16(y),
              "pool2d(nhwc): f16 / bf16 with C %% 8 == 0 (C = %d)", C);
    const int64_t total = (int64_t)N * OH * OW * (C / 8);
    if (total == 0) return 0;
    auto st = (cudaStream_t)stream;
    if (!is_max && kh == H && kw == W && ph == 0 && pw == 0 && OH == 1 && OW == 1 && dh == 1 && dw == 1 && N <= 65535) {
        const LaunchCfg c{dim3((unsigned)((C / 8 + 31) / 32), (unsigned)N), dim3(256), 0, st};
        if (dtype == ITB_F16)
            return launch("pool2d(nhwc, global average)", global_avgpool_nhwc_kernel<__half>, c, (const __half *)x, (__half *)y, C / 8,
                          H * W);
        return launch("pool2d(nhwc, global average)", global_avgpool_nhwc_kernel<__nv_bfloat16>, c, (const __nv_bfloat16 *)x,
                      (__nv_bfloat16 *)y, C / 8, H * W);
    }
    const LaunchCfg c{dim3(grid_for(total, 256)), dim3(256), 0, st};
    if (kh == 3 && kw == 3 && dh == 1 && dw == 1) {
        if (dtype == ITB_F16)
            return launch("pool2d(nhwc, 3x3)", pool2d_nhwc3x3_kernel<__half>, c, is_max, (const __half *)x, (__half *)y, total, C / 8, H,
                          W, ph, pw, sh, sw, OH, OW);
        return launch("pool2d(nhwc, 3x3)", pool2d_nhwc3x3_kernel<__nv_bfloat16>, c, is_max, (const __nv_bfloat16 *)x,
                      (__nv_bfloat16 *)y, total, C / 8, H, W, ph, pw, sh, sw, OH, OW);
    }
    if (dtype == ITB_F16)
        return launch("pool2d(nhwc)", pool2d_nhwc_kernel<__half>, c, is_max, (const __half *)x, (__half *)y, total, C / 8, H, W, kh,
                      kw, dh, dw, ph, pw, sh, sw, OH, OW);
    return launch("pool2d(nhwc)", pool2d_nhwc_kernel<__nv_bfloat16>, c, is_max, (const __nv_bfloat16 *)x, (__nv_bfloat16 *)y, total,
                  C / 8, H, W, kh, kw, dh, dw, ph, pw, sh, sw, OH, OW);
}

static int batchnorm_impl(int dtype, const void *x, const float *mean, const float *var, const float *scale,
                          const float *bias, void *y, int N, int C, int64_t HW, float eps, int relu, void *stream) {
    int64_t n = (int64_t)N * C * HW;
    if (n == 0) return 0;
    ITB_DISPATCH_FLOAT(dtype, "batchnorm", {
        constexpr int V = Vec16<T>::N;
        if (HW % V == 0 && aligned16(x) && aligned16(y))
            return launch("batchnorm", batchnorm_kernel<T, true>, {dim3(grid_for(n / V, 256)), dim3(256), 0, (cudaStream_t)stream},
                          (const T *)x, mean, var, scale, bias, (T *)y, n, C, HW, eps, relu);
        return launch("batchnorm", batchnorm_kernel<T, false>, {dim3(grid_for(n, 256)), dim3(256), 0, (cudaStream_t)stream},
                      (const T *)x, mean, var, scale, bias, (T *)y, n, C, HW, eps, relu);
    });
    return 0;
}

extern "C" int it_b200_batchnorm(int dtype, const void *x, const float *mean, const float *var,
                                 const float *scale, const float *bias, void *y, int N, int C, int64_t HW,
                                 float eps, void *stream) {
    return batchnorm_impl(dtype, x, mean, var, scale, bias, y, N, C, HW, eps, 0, stream);
}

extern "C" int it_b200_batchnorm_relu(int dtype, const void *x, const float *mean, const float *var,
                                      const float *scale, const float *bias, void *y, int N, int C, int64_t HW,
                                      float eps, void *stream) {
    return batchnorm_impl(dtype, x, mean, var, scale, bias, y, N, C, HW, eps, 1, stream);
}
