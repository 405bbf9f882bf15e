// gemm.cu -- MatMul / Conv entry points: shape dispatch + TMA descriptor helper + im2col.
//
// it_b200_matmul replaces matmulCublas (reference src/kernels/cuda/matmul.cc:66-211):
//   M <= 64, bf16/fp16, [K,N] weights  -> gemm_skinny.cu  (TMA + mbarrier + cluster split-K, HBM-bound)
//   large aligned bf16/fp16             -> gemm_tc.cu      (wgmma + TMEM + TMA)
//   fp32 (exact, no TF32) and the rest  -> gemm_simt.cu
// it_b200_conv2d replaces convCudnn (conv.cc:36-265): im2col into the workspace, then the same GEMMs
// (the "conv/im2col-GEMM path" BASELINE.json names for ResNet-50).
#include <cudaTypedefs.h>

#include <mutex>

#include "conv_shapes.h"
#include "gemm.cuh"

namespace itb {

static PFN_cuTensorMapEncodeTiled_v12000 get_encode_fn() {
    static PFN_cuTensorMapEncodeTiled_v12000 fn = nullptr;
    static std::once_flag once;
    std::call_once(once, [] {
        void *p = nullptr;
        cudaDriverEntryPointQueryResult q;
        if (cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &p, cudaEnableDefault, &q) == cudaSuccess &&
            q == cudaDriverEntryPointSuccess)
            fn = reinterpret_cast<PFN_cuTensorMapEncodeTiled_v12000>(p);
    });
    return fn;
}

bool make_tma_2d_b16(CUtensorMap *map, const void *base, uint64_t rows, uint64_t cols,
                     uint64_t row_stride_elems, uint32_t box_rows, uint32_t box_cols, int swizzle_bytes) {
    auto fn = get_encode_fn();
    if (!fn) return false;
    cuuint64_t gdim[2] = {cols, rows};
    cuuint64_t gstride[1] = {row_stride_elems * 2};
    cuuint32_t box[2] = {box_cols, box_rows};
    cuuint32_t estr[2] = {1, 1};
    CUtensorMapSwizzle sw = swizzle_bytes == 128 ? CU_TENSOR_MAP_SWIZZLE_128B
                            : swizzle_bytes == 64 ? CU_TENSOR_MAP_SWIZZLE_64B
                            : swizzle_bytes == 32 ? CU_TENSOR_MAP_SWIZZLE_32B
                                                  : CU_TENSOR_MAP_SWIZZLE_NONE;
    CUresult r = fn(map, CU_TENSOR_MAP_DATA_TYPE_BFLOAT16, 2, const_cast<void *>(base), gdim, gstride, box, estr,
                    CU_TENSOR_MAP_INTERLEAVE_NONE, sw, CU_TENSOR_MAP_L2_PROMOTION_L2_256B,
                    CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
    return r == CUDA_SUCCESS;
}

bool make_tma_2d_u8(CUtensorMap *map, const void *base, uint64_t rows, uint64_t cols, uint64_t row_stride_bytes,
                    uint32_t box_rows, uint32_t box_cols) {
    auto fn = get_encode_fn();
    if (!fn) return false;
    cuuint64_t gdim[2] = {cols, rows};
    cuuint64_t gstride[1] = {row_stride_bytes};
    cuuint32_t box[2] = {box_cols, box_rows};
    cuuint32_t estr[2] = {1, 1};
    CUresult r = fn(map, CU_TENSOR_MAP_DATA_TYPE_UINT8, 2, const_cast<void *>(base), gdim, gstride, box, estr,
                    CU_TENSOR_MAP_INTERLEAVE_NONE, CU_TENSOR_MAP_SWIZZLE_NONE, CU_TENSOR_MAP_L2_PROMOTION_L2_256B,
                    CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
    return r == CUDA_SUCCESS;
}

// the same over bytes with 128B swizzle (box_cols = 128: the 4-bit codes of gemm_w4.cu, one 128-byte row per output column)
bool make_tma_2d_u8_sw128(CUtensorMap *map, const void *base, uint64_t rows, uint64_t cols, uint64_t row_stride_bytes,
                          uint32_t box_rows, uint32_t box_cols) {
    auto fn = get_encode_fn();
    if (!fn) return false;
    cuuint64_t gdim[2] = {cols, rows};
    cuuint64_t gstride[1] = {row_stride_bytes};
    cuuint32_t box[2] = {box_cols, box_rows};
    cuuint32_t estr[2] = {1, 1};
    CUresult r = fn(map, CU_TENSOR_MAP_DATA_TYPE_UINT8, 2, const_cast<void *>(base), gdim, gstride, box, estr,
                    CU_TENSOR_MAP_INTERLEAVE_NONE, CU_TENSOR_MAP_SWIZZLE_128B, CU_TENSOR_MAP_L2_PROMOTION_L2_256B,
                    CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
    return r == CUDA_SUCCESS;
}

// 3-D tensor [batch][rows][cols] of 2-byte elements (batch stride in elements), box [1, box_rows, box_cols], 128B swizzle
bool make_tma_3d_b16(CUtensorMap *map, const void *base, uint64_t batch, uint64_t rows, uint64_t cols,
                     uint64_t row_stride_elems, uint64_t batch_stride_elems, uint32_t box_rows, uint32_t box_cols) {
    auto fn = get_encode_fn();
    if (!fn) return false;
    if (batch <= 1) {
        batch = 1;
        batch_stride_elems = rows * row_stride_elems;  // unused dimension; must still be a legal stride
    }
    cuuint64_t gdim[3] = {cols, rows, batch};
    cuuint64_t gstride[2] = {row_stride_elems * 2, batch_stride_elems * 2};
    cuuint32_t box[3] = {box_cols, box_rows, 1};
    cuuint32_t estr[3] = {1, 1, 1};
    CUresult r = fn(map, CU_TENSOR_MAP_DATA_TYPE_BFLOAT16, 3, const_cast<void *>(base), gdim, gstride, box, estr,
                    CU_TENSOR_MAP_INTERLEAVE_NONE, CU_TENSOR_MAP_SWIZZLE_128B, CU_TENSOR_MAP_L2_PROMOTION_L2_256B,
                    CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
    return r == CUDA_SUCCESS;
}

// 4-D tensor of 2-byte elements, dimensions d0 (contiguous) .. d3 with strides s1..s3 in elements (ascending), 128B swizzle
bool make_tma_4d_b16(CUtensorMap *map, const void *base, uint64_t d0, uint64_t d1, uint64_t d2, uint64_t d3, uint64_t s1, uint64_t s2,
                     uint64_t s3, uint32_t b0, uint32_t b1, uint32_t b2, uint32_t b3) {
    auto fn = get_encode_fn();
    if (!fn) return false;
    cuuint64_t gdim[4] = {d0, d1, d2, d3};
    cuuint64_t gstride[3] = {s1 * 2, s2 * 2, s3 * 2};
    cuuint32_t box[4] = {b0, b1, b2, b3};
    cuuint32_t estr[4] = {1, 1, 1, 1};
    CUresult r = fn(map, CU_TENSOR_MAP_DATA_TYPE_BFLOAT16, 4, const_cast<void *>(base), gdim, gstride, box, estr,
                    CU_TENSOR_MAP_INTERLEAVE_NONE, CU_TENSOR_MAP_SWIZZLE_128B, CU_TENSOR_MAP_L2_PROMOTION_L2_256B,
                    CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
    return r == CUDA_SUCCESS;
}

// ---------------------------------------------------------------- im2col (NCHW -> [N][C*R*S, OH*OW])
// FOLD = false: col[n][kc][p] (one [Kc, P] matrix per image);  FOLD = true: col[kc][n * P + p] (the batch folded into
// the GEMM columns -- one [Kc, N*P] matrix, legal for TMA whenever N*P % 8 == 0 even if P is odd, e.g. 7x7 / 14x14 maps).
// kc = (c*R + r)*S + s, p = oh*OW + ow.  VEC: one thread produces 8 consecutive elements of one col row (row length % 8
// == 0) with one 16-byte store and incremental (ow, oh, n) stepping -- one div/mod set per 8 elements, 32-bit math.
template <typename T, bool FOLD, bool VEC>
__global__ void __launch_bounds__(256) im2col_kernel(const T *__restrict__ x, T *__restrict__ col, int64_t total,
                                                     int NB, int C, int H, int W, int R, int S, int OH, int OW, int ph,
                                                     int pw, int sh, int sw, int dh, int dw) {
    // (FOLD: `total` may cover more than C*R*S rows -- the extra rows, c >= C, are the zero padding of K to a multiple of 8)
    pdl_trigger();
    pdl_wait();
    const int P = OH * OW, Kc = C * R * S;
    if (VEC) {
        constexpr int V = 8;
        static_assert(sizeof(T) == 2 || !VEC, "vector im2col is for 2-byte types");
        const int rowlen = FOLD ? NB * P : P, row8 = rowlen / V;
        for (int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; i < total / V;
             i += (int64_t)gridDim.x * blockDim.x) {
            const int64_t rowid = i / row8;  // FOLD: kc;  else n * Kc + kc
            const int j0 = (int)(i - rowid * row8) * V;
            const int kc = FOLD ? (int)rowid : (int)(rowid % Kc);
            int n = FOLD ? j0 / P : (int)(rowid / Kc);
            const int p0 = FOLD ? j0 - n * P : j0;
            const int s = kc % S, r = (kc / S) % R, c = kc / (R * S);
            int oh = p0 / OW, ow = p0 - oh * OW;
            T out[V];
#pragma unroll
            for (int e = 0; e < V; ++e) {
                const int ih = oh * sh - ph + r * dh, iw = ow * sw - pw + s * dw;
                T v = from_f<T>(0.f);
                if (c < C && ih >= 0 && ih < H && iw >= 0 && iw < W) v = x[(((int64_t)n * C + c) * H + ih) * W + iw];
                out[e] = v;
                if (++ow == OW) {
                    ow = 0;
                    if (++oh == OH) {
                        oh = 0;
                        ++n;
                    }
                }
            }
            *reinterpret_cast<uint4 *>(col + rowid * rowlen + j0) = *reinterpret_cast<const uint4 *>(out);
        }
    } else {
        for (int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; i < total;
             i += (int64_t)gridDim.x * blockDim.x) {
            int64_t p = i % P, t = i / P;
            int64_t kc = FOLD ? t / NB : t % Kc, n = FOLD ? t % NB : t / Kc;
            int s = (int)(kc % S), r = (int)((kc / S) % R), c = (int)(kc / ((int64_t)R * S));
            int oh = (int)(p / OW), ow = (int)(p % OW);
            int ih = oh * sh - ph + r * dh, iw = ow * sw - pw + s * dw;
            T v = from_f<T>(0.f);
            if (c < C && ih >= 0 && ih < H && iw >= 0 && iw < W) v = x[(((int64_t)n * C + c) * H + ih) * W + iw];
            col[i] = v;
        }
    }
}

// filters [F, Kc] -> [F, Kp] with zero fill (Kc not a multiple of 8, e.g. the 3x7x7 stem of ResNet)
template <typename T>
__global__ void __launch_bounds__(256) pad_rows_kernel(const T *__restrict__ w, T *__restrict__ out, int64_t total, int Kc,
                                                       int Kp) {
    pdl_trigger();
    pdl_wait();
    for (int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; i < total; i += (int64_t)gridDim.x * blockDim.x) {
        const int64_t f = i / Kp;
        const int k = (int)(i - f * Kp);
        out[i] = k < Kc ? w[f * Kc + k] : from_f<T>(0.f);
    }
}

// Kernel selection: the production order below, unless it_b200_matmul_select pinned one kernel for this thread's next calls
// (MatMul's tune() and tuned compute(), and the parity tests that must exercise each kernel)
enum { SEL_AUTO = 0, SEL_SKINNY = 1, SEL_TC = 2, SEL_SIMT = 3 };
static thread_local int g_sel_impl = SEL_AUTO;

static int run_gemm(int dtype, const GemmArgs &g, cudaStream_t st) {
    if (g.batch == 0 || g.m == 0 || g.n == 0) return 0;
    int r = -1;
    if (g_sel_impl != SEL_AUTO) {
        if (g_sel_impl == SEL_TC) r = launch_gemm_tc(dtype, g, st);
        else if (g_sel_impl == SEL_SKINNY) r = launch_gemm_skinny(dtype, g, st);
        if (r >= 0) return r;
        return launch_gemm_simt(dtype, g, st);
    }
    // decode rows with enough 128-wide column tiles to fill the SMs without split-K (logits): wgmma swap-AB
    if (g.m <= 64 && g.batch == 1 && !g.trans_a && !g.trans_b && (g.n + 127) / 128 >= TC_MIN_TILES_DECODE) {
        GemmArgs gt = g;
        gt.no_splitk = 1;
        r = launch_gemm_tc(dtype, gt, st);
        if (r >= 0) return r;
    }
    r = launch_gemm_skinny(dtype, g, st);
    if (r >= 0) return r;
    r = launch_gemm_tc(dtype, g, st);
    if (r >= 0) return r;
    return launch_gemm_simt(dtype, g, st);
}

}  // namespace itb

using namespace itb;

extern "C" int64_t it_b200_matmul_workspace(int, int64_t, int, int, int) { return 0; }

extern "C" void it_b200_tune_skinny(int nb, int splitk);
// impl: 0 production order, 1 gemm_skinny, 2 gemm_tc, 3 gemm_simt (a kernel that does not take the shape falls through to
// gemm_simt; it_b200_matmul_grouped / _fused skip the grouped or fused launch of a kernel that is not the pinned one);
// skinny_nb: 1 / 2 = 64- / 128-column tiles, 0 automatic.  Stays in force on this thread until called again.
extern "C" void it_b200_matmul_select(int impl, int skinny_nb) {
    g_sel_impl = impl >= SEL_AUTO && impl <= SEL_SIMT ? impl : SEL_AUTO;
    it_b200_tune_skinny(skinny_nb, 0);
}

extern "C" int it_b200_matmul(int dtype, const void *A, const void *B, const void *bias, void *C, int64_t b,
                              int m, int n, int k, int64_t stride_a, int64_t stride_b, int trans_a, int trans_b,
                              int64_t bias_stride_b, int64_t bias_stride_m, int64_t bias_stride_n, int act,
                              void *workspace, int64_t workspace_bytes, void *stream) {
    (void)workspace;
    (void)workspace_bytes;
    ITB_CHECK(dtype == ITB_F32 || dtype == ITB_F16 || dtype == ITB_BF16, "matmul: unsupported dtype %d", dtype);
    ITB_CHECK(m >= 0 && n >= 0 && k >= 0 && b >= 0, "matmul: negative dimension");
    ITB_CHECK((act & 0xff) <= 3 && (act & ~0x3ff) == 0, "matmul: bad act %d (Gelu / residual fusion: it_b200_matmul_fused)", act);
    GemmArgs g{A, B, bias, C, b, m, n, k, stride_a, stride_b, trans_a, trans_b,
               bias_stride_b, bias_stride_m, bias_stride_n, act};
    return run_gemm(dtype, g, (cudaStream_t)stream);
}

// MatMul (+ bias) -> [Relu | Sigmoid | Tanh | Gelu] -> [+ residual] in ONE tensor-core epilogue, every operator boundary rounded to
// the storage type like the separate kernels.  2 = shape outside the wgmma kernel (nothing launched).
extern "C" int it_b200_matmul_fused(int dtype, const void *A, const void *B, const void *bias, const void *residual, void *C,
                                    int64_t b, int m, int n, int k, int64_t stride_a, int64_t stride_b, int trans_a, int trans_b,
                                    int64_t bias_stride_b, int64_t bias_stride_m, int64_t bias_stride_n, int act, void *stream) {
    ITB_CHECK((act & 0xff) <= 4 && (act & ~0x2ff) == 0, "matmul_fused: bad act %d", act);
    ITB_CHECK(m >= 0 && n >= 0 && k >= 0 && b >= 0, "matmul_fused: negative dimension");
    if (b == 0 || m == 0 || n == 0) return 0;
    GemmArgs g{A, B, bias, C, b, m, n, k, stride_a, stride_b, trans_a, trans_b, bias_stride_b, bias_stride_m, bias_stride_n, act};
    g.residual = residual;
    g.no_splitk = 1;
    if (g_sel_impl != SEL_AUTO && g_sel_impl != SEL_TC) return 2;
    if (!aligned16(C) || (residual && !aligned16(residual)) || (g.act & 0xff) == 0 && !residual) return 2;
    const int r = launch_gemm_tc(dtype, g, (cudaStream_t)stream);
    return r < 0 ? 2 : r;
}

extern "C" int it_b200_matmul_grouped(int dtype, const void *X, int n_groups, const void *const *W, void *const *C,
                                      const int *N, int m, int k, void *stream) {
    ITB_CHECK(n_groups >= 1, "matmul_grouped: no groups");
    auto st = (cudaStream_t)stream;
    GemmArgs g{X, W[0], nullptr, C[0], 1, m, N[0], k, (int64_t)m * k, 0, 0, 0, 0, 0, 0, ITB_MATMUL_B_CONST};
    if (g_sel_impl == SEL_AUTO || g_sel_impl == SEL_TC) {
        int r = launch_gemm_tc_grouped(dtype, g, n_groups, W, C, N, st);  // only when its tiles fill the machine (gate/up)
        if (r >= 0) return r;
    }
    if (g_sel_impl == SEL_AUTO || g_sel_impl == SEL_SKINNY) {
        int r = launch_gemm_skinny_grouped(dtype, g, n_groups, W, C, N, st);
        if (r >= 0) return r;
    }
    for (int i = 0; i < n_groups; ++i) {
        GemmArgs gi = g;
        gi.B = W[i];
        gi.C = C[i];
        gi.n = N[i];
        int r = run_gemm(dtype, gi, st);
        if (r) return r;
    }
    return 0;
}

extern "C" int it_b200_matmul_fp8w(int dtype, const void *X, int n_groups, const void *const *Wq, const float *const *scale,
                                   void *const *C, const int *N, int m, int k, const void *residual, void *stream) {
    ITB_CHECK(n_groups >= 1 && n_groups <= 4, "matmul_fp8w: 1..4 weight matrices per launch");
    ITB_CHECK(!residual || n_groups == 1, "matmul_fp8w: a residual goes with a single weight matrix");
    GemmArgs g{X, Wq[0], residual, C[0], 1, m, N[0], k, (int64_t)m * k, 0, 0, 0, 0, residual ? (int64_t)N[0] : 0, residual ? 1 : 0,
               residual ? ITB_ACT_ROUND_BEFORE_BIAS : 0};
    g.w_scale = scale[0];
    int r = launch_gemm_skinny_fp8w(dtype, g, n_groups, Wq, scale, C, N, (cudaStream_t)stream);
    ITB_CHECK(r >= 0, "matmul_fp8w: shape outside the decode kernel (m = %d <= 64, K = %d %% 16, N %% 16, f16 / bf16 activations)", m, k);
    return r;
}

extern "C" int64_t it_b200_conv2d_workspace(int dtype, int N, int C, int H, int W, int F, int R, int S, int ph,
                                            int pw, int sh, int sw, int dh, int dw, int groups) {
    int OH, OW;
    conv_out_hw(H, W, R, S, ph, pw, sh, sw, dh, dw, OH, OW);
    const int64_t P = (int64_t)OH * OW, Kc = (int64_t)C * R * S;
    const bool foldable = conv_fold_ok(dtype, N, P, Kc, F, groups);
    if (conv_is_1x1_direct(R, S, ph, pw, sh, sw) && (P % 8 == 0 || !foldable)) return 0;
    const int64_t Kp = foldable ? (Kc + 7) & ~7ll : Kc;
    int64_t bytes = (int64_t)N * Kp * P * dtype_size(dtype);
    if (Kp != Kc) bytes = ((bytes + 255) & ~255ll) + (int64_t)F * Kp * dtype_size(dtype);  // + zero-padded filter copy
    return bytes;
}

struct ConvTail {
    const float *mean = nullptr, *var = nullptr, *scale = nullptr, *bias = nullptr;
    float eps = 0.f;
    const void *residual = nullptr;
    int relu = 0;
    bool any() const { return scale || residual || relu; }
};

// returns 0 done, 1 error, 2 = a fused tail was asked for but this shape does not run on the tensor-core GEMM (nothing
// was launched; the caller executes the operators one by one)
static int conv_impl(int dtype, const void *x, const void *w, void *y, int N, int C, int H, int W, int F, int R, int S,
                     int ph, int pw, int sh, int sw, int dh, int dw, int groups, const ConvTail &tail, void *workspace,
                     int64_t workspace_bytes, void *stream, int y_nhwc = 0) {
    ITB_CHECK(groups >= 1 && C % groups == 0 && F % groups == 0, "conv: bad groups %d for C=%d F=%d", groups, C, F);
    auto st = (cudaStream_t)stream;
    int OH, OW;
    conv_out_hw(H, W, R, S, ph, pw, sh, sw, dh, dw, OH, OW);
    if ((int64_t)N * F * OH * OW == 0) return 0;
    const int es = dtype_size(dtype);
    const int64_t P = (int64_t)OH * OW, Kc = (int64_t)C * R * S;
    const bool direct = conv_is_1x1_direct(R, S, ph, pw, sh, sw);
    // 1x1 s1 p0 with P % 8 == 0: the NCHW activation already is [N][C, P] -> batched GEMM, no repack.
    // otherwise fold the batch into the GEMM columns when that makes the matrix TMA-legal (tensor-core path).
    const bool direct_tc = direct && P % 8 == 0;
    const bool fold = !direct_tc && conv_fold_ok(dtype, N, P, Kc, F, groups);
    const int64_t Kp = fold ? (Kc + 7) & ~7ll : Kc;  // GEMM K (zero-padded when folded)
    auto with_tail = [&](GemmArgs &g) {
        g.bn_mean = tail.mean;
        g.bn_var = tail.var;
        g.bn_scale = tail.scale;
        g.bn_bias = tail.bias;
        g.bn_eps = tail.eps;
        g.residual = tail.residual;
        g.post_relu = tail.relu;
    };
    // NHWC output (x stays NCHW): only the folded tensor-core GEMM scatters that way
    if (y_nhwc && !(fold && F % 8 == 0 && aligned16(y) && (!tail.residual || aligned16(tail.residual)) &&
                    (Kp != Kc || aligned16(w)) && aligned16(workspace)))
        return 2;
    if (tail.any()) {
        // the tail is implemented by the wgmma epilogue: decide BEFORE launching anything
        const bool tc_batched = direct_tc && groups == 1 && (dtype == ITB_F16 || dtype == ITB_BF16) && Kc % 8 == 0 &&
                                Kc >= 64 && P >= 64 && aligned16(x) && aligned16(w) && (int64_t)N * ((F + 255) / 256) <= 65535;
        if (!fold && !tc_batched) return 2;
        if (fold && ((Kp == Kc && !aligned16(w)) || !aligned16(workspace))) return 2;
    }
    const void *col = x;
    if (!direct || fold) {
        int64_t need = it_b200_conv2d_workspace(dtype, N, C, H, W, F, R, S, ph, pw, sh, sw, dh, dw, groups);
        ITB_CHECK(workspace && workspace_bytes >= need, "conv: workspace %lld < %lld bytes",
                  (long long)workspace_bytes, (long long)need);
        int64_t total = (int64_t)N * Kp * P;
        const int64_t rowlen = fold ? (int64_t)N * P : P;
        ITB_DISPATCH_FLOAT(dtype, "conv(im2col)", {
            auto go = [&](auto kern, int64_t items) {
                return launch("conv(im2col)", kern, {dim3(grid_for(items, 256)), dim3(256), 0, st}, (const T *)x, (T *)workspace,
                              total, N, C, H, W, R, S, OH, OW, ph, pw, sh, sw, dh, dw);
            };
            int rc;
            if constexpr (sizeof(T) == 2) {
                if (rowlen % 8 == 0 && aligned16(workspace)) {
                    rc = fold ? go(im2col_kernel<T, true, true>, total / 8) : go(im2col_kernel<T, false, true>, total / 8);
                } else {
                    rc = fold ? go(im2col_kernel<T, true, false>, total) : go(im2col_kernel<T, false, false>, total);
                }
            } else {
                rc = fold ? go(im2col_kernel<T, true, false>, total) : go(im2col_kernel<T, false, false>, total);
            }
            if (rc) return 1;
        });
        col = workspace;
    }
    if (fold) {
        // y[n][f][p] = sum_kc W[f, kc] . col[kc, n*P + p]
        const void *wmat = w;
        if (Kp != Kc) {
            char *wpad = (char *)workspace + (((int64_t)N * Kp * P * es + 255) & ~255ll);
            const int64_t wt = (int64_t)F * Kp;
            ITB_DISPATCH_FLOAT(dtype, "conv(pad filters)", {
                if (launch("conv(pad filters)", pad_rows_kernel<T>, {dim3(grid_for(wt, 256)), dim3(256), 0, st}, (const T *)w,
                           (T *)wpad, wt, (int)Kc, (int)Kp))
                    return 1;
            });
            wmat = wpad;
        }
        GemmArgs g{};
        g.A = wmat;
        g.B = col;
        g.C = y;
        g.batch = 1;
        g.m = F;
        g.n = (int)(N * P);
        g.k = (int)Kp;
        g.stride_a = (int64_t)F * Kp;
        g.stride_b = Kp * N * P;
        if (y_nhwc) {
            g.c_nhwc = 1;
        } else {
            g.c_block = (int)P;
            g.c_block_stride = (int64_t)F * P;
        }
        g.no_splitk = 1;
        with_tail(g);
        int r = launch_gemm_tc(dtype, g, st);
        ITB_CHECK(r >= 0, "conv: the tensor-core GEMM refused a folded im2col matrix (F=%d Kc=%lld N*P=%lld)", F,
                  (long long)Kc, (long long)(N * P));
        return r;
    }
    // y[n][f, p] = W[f, kc] . col[n][kc, p] : A = weights (batch-broadcast), B = col
    const int Cg = C / groups, Fg = F / groups;
    const int64_t Kg = (int64_t)Cg * R * S;
    for (int gi = 0; gi < groups; ++gi) {
        GemmArgs g{};
        g.A = (const char *)w + (int64_t)gi * Fg * Kg * es;
        g.B = (const char *)col + (int64_t)gi * Kg * P * es;
        g.C = (char *)y + (int64_t)gi * Fg * P * es;
        g.bias = nullptr;
        g.batch = N;
        g.m = Fg;
        g.n = (int)P;
        g.k = (int)Kg;
        g.stride_a = 0;
        g.stride_b = Kc * P;
        g.trans_a = g.trans_b = 0;
        g.act = 0;
        g.no_splitk = 1;
        if (groups == 1 && tail.any()) {
            with_tail(g);
            int r = launch_gemm_tc(dtype, g, st);
            ITB_CHECK(r >= 0, "conv: the tensor-core GEMM refused a fused 1x1 conv (F=%d C=%d P=%lld)", F, C, (long long)P);
            if (r) return r;
        } else if (groups == 1) {
            int r = run_gemm(dtype, g, st);
            if (r) return r;
        } else {
            // grouped: C batch stride is F*P, not Fg*P -> one launch per image
            for (int n = 0; n < N; ++n) {
                GemmArgs gn = g;
                gn.batch = 1;
                gn.B = (const char *)g.B + (int64_t)n * Kc * P * es;
                gn.C = (char *)g.C + (int64_t)n * F * P * es;
                int r = run_gemm(dtype, gn, st);
                if (r) return r;
            }
        }
    }
    return 0;
}

extern "C" int it_b200_conv2d(int dtype, const void *x, const void *w, void *y, int N, int C, int H, int W, int F,
                              int R, int S, int ph, int pw, int sh, int sw, int dh, int dw, int groups,
                              void *workspace, int64_t workspace_bytes, void *stream) {
    return conv_impl(dtype, x, w, y, N, C, H, W, F, R, S, ph, pw, sh, sw, dh, dw, groups, ConvTail{}, workspace,
                     workspace_bytes, stream);
}

extern "C" int it_b200_conv2d_fused(int dtype, const void *x, const void *w, void *y, int N, int C, int H, int W,
                                    int F, int R, int S, int ph, int pw, int sh, int sw, int dh, int dw, int groups,
                                    const float *bn_mean, const float *bn_var, const float *bn_scale,
                                    const float *bn_bias, float bn_eps, const void *residual, int relu,
                                    void *workspace, int64_t workspace_bytes, void *stream) {
    ITB_CHECK((bn_scale == nullptr) == (bn_mean == nullptr) && (bn_scale == nullptr) == (bn_var == nullptr) &&
                  (bn_scale == nullptr) == (bn_bias == nullptr),
              "conv_fused: the four BatchNorm parameter vectors go together");
    ConvTail t;
    t.mean = bn_mean;
    t.var = bn_var;
    t.scale = bn_scale;
    t.bias = bn_bias;
    t.eps = bn_eps;
    t.residual = residual;
    t.relu = relu;
    return conv_impl(dtype, x, w, y, N, C, H, W, F, R, S, ph, pw, sh, sw, dh, dw, groups, t, workspace, workspace_bytes,
                     stream);
}

// Conv over an NCHW input whose consumers live in the NHWC domain (the stem of a ResNet: C = 3 cannot feed the implicit-GEMM kernel):
// the same im2col + tensor-core GEMM, the epilogue writes y (and reads `residual`) as [N, OH, OW, F].  _supported = the shape takes
// that path (otherwise the call answers 2 and launches nothing).
extern "C" int it_b200_conv2d_nchw_to_nhwc_supported(int dtype, int N, int C, int H, int W, int F, int R, int S, int ph, int pw,
                                                     int sh, int sw, int dh, int dw, int groups) {
    return conv_nchw_to_nhwc_ok(dtype, N, C, H, W, F, R, S, ph, pw, sh, sw, dh, dw, groups) ? 1 : 0;
}

extern "C" int it_b200_conv2d_fused_nhwc_out(int dtype, const void *x, const void *w, void *y, int N, int C, int H, int W,
                                             int F, int R, int S, int ph, int pw, int sh, int sw, int dh, int dw, int groups,
                                             const float *bn_mean, const float *bn_var, const float *bn_scale,
                                             const float *bn_bias, float bn_eps, const void *residual, int relu,
                                             void *workspace, int64_t workspace_bytes, void *stream) {
    ITB_CHECK((bn_scale == nullptr) == (bn_mean == nullptr) && (bn_scale == nullptr) == (bn_var == nullptr) &&
                  (bn_scale == nullptr) == (bn_bias == nullptr),
              "conv_fused: the four BatchNorm parameter vectors go together");
    ConvTail t;
    t.mean = bn_mean;
    t.var = bn_var;
    t.scale = bn_scale;
    t.bias = bn_bias;
    t.eps = bn_eps;
    t.residual = residual;
    t.relu = relu;
    return conv_impl(dtype, x, w, y, N, C, H, W, F, R, S, ph, pw, sh, sw, dh, dw, groups, t, workspace, workspace_bytes,
                     stream, 1);
}
