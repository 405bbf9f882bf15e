/*
 * it_b200.h -- C-ABI of the B200-native operator-kernel backend for InfiniTensor.
 *
 * Two groups of entry points, both plain C (pointers + sizes, no C++/torch types):
 *
 *  (1) KERNEL LAUNCHERS  it_b200_<op>(..., void *stream)
 *      One per reference CUDA kernel (SURVEY.md section 2.2 / 8a).  All pointers are
 *      DEVICE pointers, `stream` is a cudaStream_t.  Every launcher is
 *      CUDA-graph-capturable: no allocation, no synchronisation, no host read of
 *      device data (contract of reference src/cuda/cuda_runtime.cc:252-283).
 *      These are what the Kernel::compute() bodies registered through
 *      REGISTER_KERNEL (reference include/core/kernel.h:186-195) bottom out in.
 *
 *  (2) GRAPH / RUNTIME HANDLE API  itb_*  (HOST buffers in copyin/copyout)
 *      The C spelling of the reference's pybind `backend` module
 *      (reference src/ffi/ffi_infinitensor.cc:441-638): Runtime, GraphHandler,
 *      Tensor.  This is the reference-facing boundary a Python/cgo/JNI caller binds.
 *
 * dtype codes are the ONNX enum the reference uses (include/core/data_type.h:6-23):
 *   1 f32, 2 u8, 3 i8, 6 i32, 7 i64, 9 bool, 10 f16, 12 u32, 16 bf16.
 * Every function returns 0 on success; on failure it returns non-zero and
 * it_b200_last_error() describes why (the C spelling of infini::Exception,
 * reference include/core/common.h:44-55).  Nothing here ever falls back to a CPU path.
 */
#ifndef IT_B200_H
#define IT_B200_H

#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#define ITB_F32 1
#define ITB_U8 2
#define ITB_I8 3
#define ITB_I32 6
#define ITB_I64 7
#define ITB_BOOL 9
#define ITB_F16 10
#define ITB_U32 12
#define ITB_BF16 16

#define ITB_MAX_RANK 8

const char *it_b200_last_error(void);
int it_b200_version(void);
/* tuning hook for tools/gemm_sweep.py: force the decode-GEMM tile width (nb = 1: 64 columns, 2: 128) and split-K factor;
 * 0 = automatic (the default).  Not part of the reference-facing surface. */
void it_b200_tune_skinny(int nb, int splitk);

/* ---- unary family: replaces unary.cu:31-143 + ActivationCudnn (unary.cc:70-122) ---- */
enum { ITB_RELU = 0, ITB_SIGMOID, ITB_TANH, ITB_GELU, ITB_SILU, ITB_ERF, ITB_NEG, ITB_ABS,
       ITB_SQRT, ITB_HARDSIGMOID, ITB_HARDSWISH, ITB_EXP, ITB_LEAKYRELU, ITB_ELU };
int it_b200_unary(int op, int dtype, const void *x, void *y, int64_t n, void *stream);
/* LeakyRelu (x > 0 ? x : alpha x; unary.cu:157-165) and Elu (x >= 0 ? x : alpha (exp x - 1); unary.cu:97-106) carry `alpha` */
int it_b200_unary_alpha(int op, int dtype, const void *x, void *y, int64_t n, float alpha, void *stream);

/* ---- binary with full numpy broadcast (rank <= 8): replaces ElementWiseCudnn
 *      (element_wise.cc:8-121) and element_wise.cu:9-131.  strides in elements, 0 = broadcast.
 *      Comparison ops write uint8 0/1. ---- */
enum { ITB_ADD = 0, ITB_SUB, ITB_MUL, ITB_DIV, ITB_POW, ITB_MIN, ITB_MAX, ITB_LESS, ITB_EQUAL,
       ITB_GREATER };
int it_b200_binary(int op, int dtype, const void *a, const void *b, void *c, int rank,
                   const int64_t *dims, const int64_t *stride_a, const int64_t *stride_b,
                   void *stream);

/* ---- Cast: replaces _cast_kernel (unary.cu:145-154, unary.cc:30-68) ---- */
int it_b200_cast(int from, int to, const void *x, void *y, int64_t n, void *stream);

/* ---- Where: replaces _whereKernel (where.cu:20-41); cond is uint8/bool ---- */
int it_b200_where(int elem_size, const void *cond, const void *x, const void *y, void *out,
                  int rank, const int64_t *dims, const int64_t *stride_c,
                  const int64_t *stride_x, const int64_t *stride_y, void *stream);

/* ---- Expand: replaces _expandKernel/_expandRowKernel (expand.cu:10-49,154-170) ---- */
int it_b200_expand(int elem_size, const void *x, void *y, int rank, const int64_t *dims,
                   const int64_t *stride_x, void *stream);

/* ---- Softmax over one axis, tensor viewed [outer, dim, inner]: replaces softmax.cu:18-404 ---- */
int it_b200_softmax(int dtype, const void *x, void *y, int64_t outer, int dim, int64_t inner,
                    void *stream);

/* ---- LayerNormalization over one axis with stride: replaces layer_norm.cu:4-557.
 *      scale_size / bias_size are `dim` or 1 (scalar broadcast); bias may be NULL. ---- */
int it_b200_layernorm(int dtype, const void *x, const void *scale, const void *bias, void *y,
                      int64_t outer, int dim, int64_t inner, int scale_size, int bias_size,
                      float eps, void *stream);

/* ---- RMSNorm: replaces _rmsnorm_kernel (rms_norm.cu:36-54); eps 1e-5, round before weight ---- */
int it_b200_rmsnorm(int dtype, const void *x, const void *w, void *y, int64_t tokens, int hidden,
                    void *stream);
/* same, when `w` is a graph constant (written by no kernel of the step): the weight row is fetched ahead of the
 * programmatic-dependent-launch wait */
int it_b200_rmsnorm_constw(int dtype, const void *x, const void *w, void *y, int64_t tokens, int hidden,
                           void *stream);

/* ---- RoPE: replaces _rope_kernel (rope.cu:7-31); processes every (b, s) row.
 *      pos_dtype: ITB_I32 / ITB_U32 / ITB_I64. ---- */
int it_b200_rope(int dtype, const void *pos, int pos_dtype, const void *x, void *y, int B, int S,
                 int dim_model, int dim_head, void *stream);

/* ---- RoPE with a model's own frequencies: it_b200_rope, but column pair c of every head rotates by the angle
 *      fp32(p x inv_freq[c]) (HF's inv_freq @ position_ids).  inv_freq: f32 (freq_dtype ITB_F32), at least dim_head / 2
 *      entries; dim_model must be a multiple of dim_head. ---- */
int it_b200_rope_freq(int dtype, const void *pos, int pos_dtype, const void *x, void *y, int B, int S, int dim_model,
                      int dim_head, const void *inv_freq, int freq_dtype, int64_t freq_len, void *stream);

/* ---- Transpose (N-d permute): replaces _transpose_kernel (transpose.cu:10-24) ---- */
int it_b200_transpose(int elem_size, const void *x, void *y, int rank, const int64_t *dims_in,
                      const int *perm, void *stream);

/* ---- Concat / Split along one axis: replaces _split_concat_kernel (split_concat.cu:28-84).
 *      Tensors are viewed [outer, axis_len_i * inner]; `parts` are device pointers. ---- */
int it_b200_concat(int elem_size, int n_parts, const void *const *parts, const int64_t *axis_len,
                   void *out, int64_t outer, int64_t inner, void *stream);
int it_b200_split(int elem_size, int n_parts, void *const *parts, const int64_t *axis_len,
                  const void *in, int64_t outer, int64_t inner, void *stream);

/* ---- Gather along axis: replaces _gather_kernel (gather.cu:31-55). data viewed
 *      [outer, axis_len, inner]; out [outer, n_idx, inner]. idx_dtype ITB_I32 / ITB_I64. ---- */
int it_b200_gather(int elem_size, int idx_dtype, const void *data, const void *idx, void *out,
                   int64_t outer, int64_t axis_len, int64_t inner, int64_t n_idx, void *stream);

/* ---- Reshape/Flatten/Identity/Squeeze/Unsqueeze: replaces CopyCuda (reshape.cc:4-21) ---- */
int it_b200_copy(const void *src, void *dst, int64_t bytes, void *stream);

/* ---- Pad / Slice: replaces _pad_slice_kernel (pad_slice.cu:6-47).  Generic strided window:
 *      out[i] = in[start + i*step] per dim when inside [0, dims_in), else 0. ---- */
int it_b200_pad_slice(int elem_size, const void *in, void *out, int rank, const int64_t *dims_in,
                      const int64_t *dims_out, const int64_t *start, const int64_t *step,
                      void *stream);

/* ---- ReduceMean / ReduceSum: replaces ReduceCudnnBase (reduce.cc:7-125).
 *      reduce_mask[i] != 0 marks a reduced axis. ---- */
int it_b200_reduce(int dtype, int is_mean, const void *x, void *y, int rank, const int64_t *dims,
                   const int *reduce_mask, void *stream);

/* ---- MaxPool / AveragePool (count-include-pad): replaces poolingCudnn (pooling.cc:8-95) ---- */
int it_b200_pool2d(int dtype, int is_max, const void *x, void *y, int N, int C, int H, int W,
                   int kh, int kw, int dh, int dw, int ph, int pw, int sh, int sw, int OH, int OW,
                   void *stream);
/* the same pooling over NHWC activations ([N, H, W, C] -> [N, OH, OW, C]; f16 / bf16, C % 8 == 0): the layout the runtime's NHWC
 * domain keeps between Conv / Pool / Add / Relu steps (host/schedule.cc) */
int it_b200_pool2d_nhwc(int dtype, int is_max, const void *x, void *y, int N, int C, int H, int W, int kh, int kw, int dh,
                        int dw, int ph, int pw, int sh, int sw, int OH, int OW, void *stream);

/* ---- BatchNormalization inference: replaces BatchNormCudnn (batch_norm.cc:9-69).
 *      mean/var/scale/bias are f32 (as the reference requires). ---- */
int it_b200_batchnorm(int dtype, const void *x, const float *mean, const float *var,
                      const float *scale, const float *bias, void *y, int N, int C, int64_t HW,
                      float eps, void *stream);
/* BatchNorm followed by ReLU in one pass (bit-identical to the two kernels). */
int it_b200_batchnorm_relu(int dtype, const void *x, const float *mean, const float *var, const float *scale,
                           const float *bias, void *y, int N, int C, int64_t HW, float eps, void *stream);


/* ---- MatMul: replaces matmulCublas (matmul.cc:66-211).
 *      C[b,m,n] = op(A)[b,m,k] . op(B)[b,k,n] (+ bias) ; row-major; stride_a / stride_b in
 *      elements between batches (0 = broadcast, matmul.cc:124-137).  bias (may be NULL) is
 *      broadcast by bias_stride_{b,m,n} (elements; 0 = broadcast) -- the fused form of the
 *      reference's expand-into-C + beta=1 (matmul.cc:86-118).  act: 0 none (the reference
 *      ignores MatmulObj::act on CUDA, quirk q5), 1 relu, 2 sigmoid, 3 tanh (operator attr).
 *      fp32 accumulate for every dtype.  workspace: device scratch (may be NULL when
 *      it_b200_matmul_workspace() returns 0). ---- */
#define ITB_ACT_ROUND_BEFORE_BIAS 0x100 /* OR into `act`: round the product to the storage dtype before the bias
                                          add -- makes a fused MatMul -> Add bit-identical to the two separate ops */
#define ITB_MATMUL_B_CONST 0x200 /* OR into `act`: operand B is a constant (weight) that no kernel of the stream writes;
                                    lets the GEMM request its first weight tiles ahead of griddepcontrol.wait */
int64_t it_b200_matmul_workspace(int dtype, int64_t b, int m, int n, int k);
/* Kernel selection for this thread's following it_b200_matmul calls -- what MatMul's tune() records per shape in PerfEngine and its
 * compute(op, record) re-applies (reference: the cuBLAS algorithm index of MatmulCublasPerfRecordObj, matmul.cc:12-24,187-208).
 * impl: 0 production dispatch, 1 gemm_skinny (mma.sync + cluster split-K), 2 gemm_tc (wgmma), 3 gemm_simt; skinny_nb: 0 auto, 1, 2.
 * A pinned kernel that does not take a shape falls through to gemm_simt.  Also honoured by it_b200_matmul_grouped (only the pinned
 * kernel's grouped launch) and it_b200_matmul_fused (returns 2 unless impl is 0 or 2). */
void it_b200_matmul_select(int impl, int skinny_nb);
int it_b200_matmul(int dtype, const void *A, const void *B, const void *bias, void *C, int64_t b,
                   int m, int n, int k, int64_t stride_a, int64_t stride_b, int trans_a,
                   int trans_b, int64_t bias_stride_b, int64_t bias_stride_m,
                   int64_t bias_stride_n, int act, void *workspace, int64_t workspace_bytes,
                   void *stream);

/* MatMul (+ bias) -> [activation: 1 relu, 2 sigmoid, 3 tanh, 4 Gelu (erf form, unary.cu:113)] -> [+ residual laid out like C] in
 * the wgmma kernel's epilogue -- the schedule's MatMulAdd step for graphs whose Linear layers carry a bias (GPT-2: c_proj + Add,
 * c_fc + Gelu).  Every operator boundary rounds to the storage type (MatMul output, activation output) exactly as the separate
 * kernels do.  Returns 2 when the shape does not run on that kernel (f16 / bf16, K % 8 == 0, N % 8 == 0, no transA): nothing is
 * launched and the caller runs the operators one by one. */
int it_b200_matmul_fused(int dtype, const void *A, const void *B, const void *bias, const void *residual, void *C, int64_t b,
                         int m, int n, int k, int64_t stride_a, int64_t stride_b, int trans_a, int trans_b,
                         int64_t bias_stride_b, int64_t bias_stride_m, int64_t bias_stride_n, int act, void *stream);

/* ---- Grouped MatMul: up to 4 weight matrices W_i[K,N_i] sharing one activation operand X[M,K] (the q/k/v and
 *      gate/up projections of a decoder layer) in ONE launch; C_i[M,N_i] = X . W_i.  No bias / activation.
 *      Falls back to one it_b200_matmul per group when the shapes are not taken by the grouped kernel. ---- */
int it_b200_matmul_grouped(int dtype, const void *X, int n_groups, const void *const *W, void *const *C,
                           const int *N, int m, int k, void *stream);

/* ---- Weight-only FP8 (SURVEY 8(f-4); no counterpart in the reference, whose only quantised op is the int8 Cast, unary.cc:30-68).
 *      Wq_i [K, N_i]: FP8 E4M3 (OCP "FN": 1-4-3, bias 7, max 448, no inf) codes, one byte each, row-major like the 16-bit weights;
 *      scale_i [N_i] f32 per output column.  C_i[m, N_i] = X[m, K] . (Wq_i * scale_i): the codes are converted to the
 *      activation type inside the GEMM main loop (exact), the column scale multiplies the fp32 sum in the epilogue; halves the
 *      HBM bytes of a decode GEMM.  1..4 matrices sharing X per launch; residual (single matrix only, may be NULL) is added
 *      after the product has been rounded, like MatMul -> Add.  m <= 64, K % 16 == 0, N_i % 16 == 0.
 *      it_b200_dequantize_fp8 is the stand-alone DequantizeLinear (y = T(e4m3(xq) * scale[col])) of the unfused graph. ---- */
int it_b200_matmul_fp8w(int dtype, const void *X, int n_groups, const void *const *Wq, const float *const *scale,
                        void *const *C, const int *N, int m, int k, const void *residual, void *stream);
int it_b200_dequantize_fp8(int dtype_out, const void *xq, const float *scale, void *y, int64_t rows, int64_t cols,
                           void *stream);

/* ---- Weight-only 4-bit MatMul: the subset of ONNX com.microsoft MatMulNBits this project accepts (no counterpart in the reference).
 *      C_i[m, N_i] = X[m, K] . W_i,   W[k, n] = (q[n, k] - z[n, k / bs]) * s[n, k / bs],   bs = block_size in {32, 64, 128}.
 *      X, C, s and the residual: f16 or bf16, all of the same dtype (fp32 is refused).
 *      Wq_i (MatMulNBits input B): uint8 [N, K / bs, bs / 2], N-major -- column n's K codes are K / 2 contiguous bytes; element k of
 *           column n is in byte (n, k / bs, (k % bs) / 2), even k in the low nibble, odd k in the high nibble.
 *      scales_i: [N * K / bs] of the activation dtype; the scale of (n, block) is element n * (K / bs) + block.
 *      zero_points: NULL (z = 8 everywhere) or one pointer per matrix, uint8 nibble-packed: (K / bs) / 2 bytes per column, block b
 *           at byte n * (K / bs) / 2 + b / 2, low nibble for even b.  Accepted only when K / bs is even.
 *      K % bs == 0, N_i % 16 == 0; X, Wq_i, C_i and the residual 16-byte aligned.  1..4 matrices sharing X; residual (single
 *      matrix only, may be NULL) is added after the product has been rounded to the dtype, like MatMul -> Add.
 *      m <= 64: gemm_skinny_w4_kernel.  (q - z) enters the tensor core exactly in the activation type; each block's fp32 partial
 *           sum is multiplied by fp32(s) and added to the fp32 accumulator; the output is rounded once.  No workspace.
 *      m > 64: each matrix is dequantised to T((q - z) * s) [K, N] in the workspace (it_b200_matmul_nbits_workspace bytes),
 *           then multiplied by it_b200_matmul: the weights are rounded to the dtype once, unlike the decode kernel.
 *      it_b200_dequantize_w4 is that dequantiser on its own: W [K, N] row-major = T((q - z) * s), the product in fp32. ---- */
int64_t it_b200_matmul_nbits_workspace(int dtype, int m, int k, int n_groups, const int *N);
int it_b200_matmul_nbits(int dtype, const void *X, int n_groups, const void *const *Wq, const void *const *scales,
                         const void *const *zero_points, void *const *C, const int *N, int m, int k, int block_size,
                         const void *residual, void *workspace, int64_t workspace_bytes, void *stream);
int it_b200_dequantize_w4(int dtype, const void *Wq, const void *scales, const void *zero_points, void *W, int k, int n,
                          int block_size, void *stream);

/* ---- SiLU(gate) * up in one pass (the fused form of Silu -> Mul; the Silu result is rounded to the storage
 *      dtype before the multiply, exactly as the two separate kernels would). ---- */
int it_b200_silu_mul(int dtype, const void *gate, const void *up, void *out, int64_t n, void *stream);

/* ---- Conv (NCHW x FCRS, groups, symmetric pad): replaces convCudnn (conv.cc:36-265).
 *      im2col into workspace + tensor-core GEMM. ---- */
int64_t it_b200_conv2d_workspace(int dtype, int N, int C, int H, int W, int F, int R, int S,
                                 int ph, int pw, int sh, int sw, int dh, int dw, int groups);
int it_b200_conv2d(int dtype, const void *x, const void *w, void *y, int N, int C, int H, int W,
                   int F, int R, int S, int ph, int pw, int sh, int sw, int dh, int dw, int groups,
                   void *workspace, int64_t workspace_bytes, void *stream);
/* Conv with the tail of a ResNet bottleneck folded into the tensor-core GEMM epilogue: Conv -> BatchNorm (fp32
 * statistics; all four vectors or none) -> [+ residual, laid out like y] -> [ReLU].  Every stage rounds to the storage
 * dtype exactly as the separate kernels would, so the result is bit-identical to running them one by one.
 * Returns 0 = done, 1 = error, 2 = this shape does not take the tensor-core path (nothing launched: run the operators
 * separately).  Same workspace as it_b200_conv2d. */
int it_b200_conv2d_fused(int dtype, const void *x, const void *w, void *y, int N, int C, int H, int W, int F, int R,
                         int S, int ph, int pw, int sh, int sw, int dh, int dw, int groups, const float *bn_mean,
                         const float *bn_var, const float *bn_scale, const float *bn_bias, float bn_eps,
                         const void *residual, int relu, void *workspace, int64_t workspace_bytes, void *stream);

/* it_b200_conv2d_fused with x in NCHW and y (and `residual`) in NHWC ([N, OH, OW, F]): the entry into the NHWC domain for a conv the
 * implicit-GEMM kernel cannot take (the 3-channel stem).  _supported = 1 when the shape runs this way (f16 / bf16, groups 1,
 * folded im2col GEMM, F % 8 == 0); otherwise the call returns 2 and launches nothing.  Same workspace as it_b200_conv2d. */
int it_b200_conv2d_nchw_to_nhwc_supported(int dtype, int N, int C, int H, int W, int F, int R, int S, int ph, int pw, int sh,
                                          int sw, int dh, int dw, int groups);
int it_b200_conv2d_fused_nhwc_out(int dtype, const void *x, const void *w, void *y, int N, int C, int H, int W, int F, int R,
                                  int S, int ph, int pw, int sh, int sw, int dh, int dw, int groups, const float *bn_mean,
                                  const float *bn_var, const float *bn_scale, const float *bn_bias, float bn_eps,
                                  const void *residual, int relu, void *workspace, int64_t workspace_bytes, void *stream);

/* The stem of an image network (kernels/conv_stem.cu): x NCHW with C <= 4 channels, y NHWC [N, OH, OW, F], F <= 64 (F % 8 == 0),
 * filters up to 7 x 8, strides <= 2, no dilation / groups, optional BatchNorm (folded, one rounding) + ReLU.  The input patch of a
 * 16 x 16 output block is staged in shared memory and mma.sync fragments are built from it: no im2col matrix, no workspace. */
int it_b200_conv2d_stem_supported(int dtype, int C, int F, int R, int S, int ph, int pw, int sh, int sw, int dh, int dw,
                                  int groups);
int it_b200_conv2d_stem(int dtype, const void *x, const void *w, void *y, int N, int C, int H, int W, int F, int R, int S, int ph,
                        int pw, int sh, int sw, const float *bn_mean, const float *bn_var, const float *bn_scale,
                        const float *bn_bias, float bn_eps, int relu, void *stream);

/* Implicit-GEMM Conv over NHWC activations (kernels/conv_nhwc.cu): x is [N, H, W, C], w stays in the reference's [F, C, R, S]
 * order, y is [N, OH, OW, F] (y_nhwc = 1) or [N, F, OH, OW] (y_nhwc = 0, for a consumer outside the NHWC domain); `residual` is
 * laid out like y.  No im2col matrix: the TMA unit's im2col mode feeds wgmma directly.  The optional tail
 * BatchNorm (fp32 statistics, folded to y = a * conv + b) -> + residual -> ReLU is evaluated in fp32 and rounded ONCE (the NCHW
 * entry point above rounds after every stage).  f16 / bf16, groups = 1, C % 8 == 0, F % 8 == 0, strides <= 8; _supported answers
 * 1 for shapes the kernel takes.  Workspace: the filters re-ordered to [F][R*S][ceil64(C)] (0 bytes for 1x1 filters).
 * Replaces cudnnConvolutionForward (reference src/kernels/cuda/conv.cc:143-168) for the layout the runtime's NHWC domain uses
 * between Conv / Pool / Add / Relu steps (host/schedule.cc).
 * workspace_bytes < 0: `workspace` already holds the filters as it_b200_conv_repack_filters wrote them (-workspace_bytes = their
 * size) and is only read -- the runtime repacks every bank of a graph in one launch at the start of a step. */
int it_b200_conv2d_nhwc_supported(int dtype, int C, int F, int R, int S, int ph, int pw, int sh, int sw, int dh, int dw,
                                  int groups);
/* n filter banks [F_i, C_i, R_i, S_i] -> [F_i][R_i*S_i][ceil64(C_i)] (out[i]: it_b200_conv2d_nhwc_workspace bytes each), one launch per
 * 24 banks */
int it_b200_conv_repack_filters(int dtype, int n, const void *const *w, void *const *out, const int *F, const int *C, const int *R,
                                const int *S, void *stream);
int64_t it_b200_conv2d_nhwc_workspace(int dtype, int C, int F, int R, int S);
int it_b200_conv2d_nhwc(int dtype, const void *x, const void *w, void *y, int y_nhwc, int N, int C, int H, int W, int F, int R,
                        int S, int ph, int pw, int sh, int sw, int dh, int dw, const float *bn_mean, const float *bn_var,
                        const float *bn_scale, const float *bn_bias, float bn_eps, const void *residual, int relu,
                        void *workspace, int64_t workspace_bytes, void *stream);

/* ---- AttentionKVCache (decode, q-len 1): replaces _attention_kvcache_kernel_128_1/_2
 *      (attention_kvcache.cu:8-169).  Appends k,v IN PLACE into k_cache/v_cache at
 *      position_id[0]; caches [B,H,S_max,D], q/k/v/out [B,H,1,D]; D == 128 (the reference's width, scale 1/sqrt(128))
 *      or, as an extension for GPT-2 / TinyLlama-shape heads, D == 64; the scale is 1/sqrt(D).  Other D are refused.
 *      pos_dtype: ITB_I32 / ITB_U32 / ITB_I64 (element 0 is used for every row, .cu:17).
 *      Ordering contract (programmatic dependent launch): q / k / v (and the RoPE positions of the _rope variant) may come from
 *      the kernel launched just before on the same stream; `position_id` and the cache rows BELOW the position are read
 *      ahead of griddepcontrol.wait, so they must be OLDER than that -- graph inputs or the previous step's appends, as in
 *      every decode graph the frontend emits.  A caller that produces any of them with a kernel of this library in the
 *      same step ORs ITB_POS_IN_STEP into pos_dtype (the host kernels do, whenever one of those tensors has a source
 *      operator).  The workspace is always required (per-head partial slots). ---- */
#define ITB_POS_PER_ROW 0x100 /* OR into pos_dtype: batch row b uses position_id[b] (ragged batches; SURVEY 8(f-3)) instead of the
                                 reference's element 0 for every row */
#define ITB_POS_IN_STEP 0x200 /* OR into pos_dtype: position_id / the RoPE positions / cache rows below the position may be written by a
                                 kernel of the SAME step (in-graph position arithmetic, a Concat of the past): nothing is read ahead of
                                 griddepcontrol.wait */
#define ITB_POS_RING 0x400    /* OR into pos_flags: the caches are a rolling buffer (sliding-window launchers only; see
                                 it_b200_attention_kvcache_window) */
int64_t it_b200_attention_kvcache_workspace(int B, int H, int S_max, int D);
int it_b200_attention_kvcache(int dtype, void *k_cache, void *v_cache, const void *q,
                              const void *k, const void *v, const void *position_id,
                              int pos_dtype, void *out, int B, int H, int S_max, int D,
                              void *workspace, int64_t workspace_bytes, void *stream);

/* ---- One-shot all-reduce over NVLink peer memory fused with the residual Add and RMSNorm that follow it in a
 *      tensor-parallel decoder layer: replaces ncclAllReduce (all_reduce.cc:8-63) + Add + RMSNorm for messages of
 *      <= 64 rows x 16 KiB.  out = T(T(sum_r in_r) + residual); out_norm = RMSNorm(out) * norm_w (optional).
 *      peer_ws[world]: every rank's comm workspace (it_b200_allreduce_workspace_bytes(), zero-filled once) as mapped
 *      in this process (cudaIpcOpenMemHandle); peer_ws[rank] is the local one.  Every rank must issue the same
 *      sequence of calls.  Stream-ordered, CUDA-graph-capturable.  timeout_flag: device-visible int (host-mapped) set
 *      non-zero when a peer's packets never arrive -- the step then completes with garbage and the caller raises after
 *      its next synchronise; NULL = trap instead. ---- */
int64_t it_b200_allreduce_workspace_bytes(void);
int it_b200_allreduce_fused(int dtype, const void *in, const void *residual, const void *norm_w, void *out,
                            void *out_norm, int tokens, int hidden, void *const *peer_ws, int world, int rank,
                            int *timeout_flag, void *stream);

/* ---- AttentionKVCache with the layer's two RoPE ops folded in: q_pre / k_pre are the PRE-RoPE projections
 *      ([B, H*D] == [B,H,1,D], D = 128 or 64); RoPE (rotate-half over each D-wide head, i.e. it_b200_rope with dim_head = D,
 *      position rope_pos[b]) is applied on load, the rotated k is what gets appended -- bit-identical to RoPE ->
 *      AttentionKVCache (rope.cu:7-31 + attention_kvcache.cu). ---- */
int it_b200_attention_kvcache_rope(int dtype, void *k_cache, void *v_cache, const void *q_pre, const void *k_pre,
                                   const void *v, const void *position_id, int pos_dtype, const void *rope_pos,
                                   int rope_pos_dtype, void *out, int B, int H, int S_max, int D, void *workspace,
                                   int64_t workspace_bytes, void *stream);

/* ---- AttentionKVCache with grouped-query attention: caches [B,Hkv,S_max,D], k/v [B,Hkv,1,D], q/out [B,Hq,1,D],
 *      Hq = G * Hkv, G >= 1.  Query head i attends over KV head i / G (HF repeat_kv order); each K / V row is read once
 *      for every 32 query heads of its group (once in all for G <= 32).  pos_flags as for it_b200_attention_kvcache; rope_pos NULL: no RoPE, else as the _rope
 *      variant (q rotated per query head, k per KV head).  Workspace: it_b200_attention_kvcache_workspace(B, Hq, S_max, D).
 *      Hq == Hkv launches exactly what it_b200_attention_kvcache / _rope launch. ---- */
int it_b200_attention_kvcache_gqa(int dtype, void *k_cache, void *v_cache, const void *q, const void *k, const void *v,
                                  const void *position_id, int pos_flags, const void *rope_pos, int rope_pos_dtype, void *out,
                                  int B, int Hq, int Hkv, int S_max, int D, void *workspace, int64_t workspace_bytes,
                                  void *stream);

/* ---- AttentionKVCache (decode, one token per step) over an FP8 E4M3 KV cache: it_b200_attention_kvcache_gqa with caches
 *      [B,Hkv,S_max,D] of one-byte OCP E4M3 "FN" codes and k_scale / v_scale, f32 [Hkv], one scale per KV head.  A cache
 *      element's value is e4m3(code) * scale[h].  dtype (q / k / v / out) is ITB_F16 or ITB_BF16; fp32 is refused.
 *      Append: row p of KV head h is stored as code = cvt.rn.satfinite.e4m3(fp32(x) / scale[h]) -- the fp32 division correctly
 *      rounded, round to nearest even, saturated to +-448 -- with k rotated first (in the activation type) when rope_pos is
 *      given.  Attention over rows 0 .. p, the appended row read back from its codes:
 *        s_j = fp32(q . code_k,j) * scale_k[h] / sqrt(D),  stable softmax,  out = (sum_j p_j code_v,j) / l * scale_v[h] rounded
 *      once to the activation type (codes widen exactly to f16 / bf16).  Positions, pos_flags, RoPE, G = Hq / Hkv and the
 *      workspace (it_b200_attention_kvcache_workspace(B, Hq, S_max, D)) are as for it_b200_attention_kvcache_gqa. ---- */
int it_b200_attention_kvcache_fp8(int dtype, void *k_cache, void *v_cache, const void *k_scale, const void *v_scale,
                                  const void *q, const void *k, const void *v, const void *position_id, int pos_flags,
                                  const void *rope_pos, int rope_pos_dtype, void *out, int B, int Hq, int Hkv, int S_max,
                                  int D, void *workspace, int64_t workspace_bytes, void *stream);

/* ---- it_b200_attention_kvcache_gqa / _fp8 with the folded RoPE's angles from a table: fp32(rope_pos[b] x inv_freq[c]) for
 *      column pair c of every head, exactly as it_b200_rope_freq.  rope_pos is required; inv_freq is f32 (freq_dtype
 *      ITB_F32) with at least D / 2 entries, and like position_id it is read ahead of griddepcontrol.wait (a graph weight),
 *      unless pos_flags has ITB_POS_IN_STEP. ---- */
int it_b200_attention_kvcache_gqa_freq(int dtype, void *k_cache, void *v_cache, const void *q, const void *k, const void *v,
                                       const void *position_id, int pos_flags, const void *rope_pos, int rope_pos_dtype,
                                       const void *inv_freq, int freq_dtype, int64_t freq_len, void *out, int B, int Hq,
                                       int Hkv, int S_max, int D, void *workspace, int64_t workspace_bytes, void *stream);
int it_b200_attention_kvcache_fp8_freq(int dtype, void *k_cache, void *v_cache, const void *k_scale, const void *v_scale,
                                       const void *q, const void *k, const void *v, const void *position_id, int pos_flags,
                                       const void *rope_pos, int rope_pos_dtype, const void *inv_freq, int freq_dtype,
                                       int64_t freq_len, void *out, int B, int Hq, int Hkv, int S_max, int D,
                                       void *workspace, int64_t workspace_bytes, void *stream);

/* ---- AttentionKVCache over a prompt chunk of S >= 1 new tokens (attention_prefill.cu): exactly S single-token AttentionKVCache
 *      calls in order, token i of batch row b at position p_b + i.  Caches [B,Hkv,S_max,D]; q / out [B,Hq,S,D]; k / v [B,Hkv,S,D];
 *      Hq = G * Hkv.  Token i's k / v are copied into cache row p_b + i; query i of head h attends over rows 0 .. p_b + i of KV
 *      head h / G with scale 1/sqrt(D) (causal attention with an offset: also chunked prefill, p_b > 0).  p_b is element 0 of
 *      position_id, or with ITB_POS_PER_ROW element b * stride (stride = pos_flags >> ITB_POS_ROW_STRIDE_SHIFT, 0 meaning 1: a
 *      [B, S] position tensor has stride S); positions inside a row are taken to be consecutive, only the start is read.
 *      p_b is clamped to [0, S_max - S]; S > S_max is refused.  f16 / bf16 only (fp32 is refused), D = 64 or 128.  Two launches
 *      (append, then attention, PDL-chained); nothing is read before griddepcontrol.wait, so ITB_POS_IN_STEP changes nothing.
 *      No workspace. ---- */
#define ITB_POS_ROW_STRIDE_SHIFT 16
int it_b200_attention_kvcache_prompt(int dtype, void *k_cache, void *v_cache, const void *q, const void *k, const void *v,
                                     const void *position_id, int pos_flags, void *out, int B, int Hq, int Hkv, int S, int S_max,
                                     int D, void *stream);

/* ---- Sliding-window attention (Mistral-7B-v0.1 and models trained like it).  window >= 1: the query at position P reads only
 *      cache rows j with P - window < j <= P, its own row included (transformers' `kv_idx > q_idx - sliding_window`; the
 *      original Mistral code keeps one row more: pass window + 1 for that).  Positions, clamping and the append are unchanged;
 *      without ITB_POS_RING the cache is indexed by absolute position, so S_max must cover the longest position.  Rows below a query's window
 *      never reach its output, even when they hold NaN.  window 0 is no window: the same kernels as the unwindowed calls.
 *      window < 0 is refused, before any launch.
 *   _window: every decode variant in one call.  k_scale / v_scale NULL: 16-bit or fp32 caches, non-NULL: FP8 E4M3 caches
 *      (it_b200_attention_kvcache_fp8); rope_pos NULL: no RoPE; inv_freq NULL: base 10000, else the table
 *      (it_b200_attention_kvcache_gqa_freq, freq_dtype / freq_len checked alike).  A windowed head streams only the rows
 *      [max(0, P - window + 1), P): min(P + 1, window) rows per step instead of P + 1.
 *   _prompt_window: it_b200_attention_kvcache_prompt, query i of batch row b reading rows (p_b + i - window, p_b + i].
 *   Rolling cache (ITB_POS_RING in pos_flags, these two launchers only; Mistral's "rolling buffer cache"): the caches
 *      [B, Hkv, S_max, D] are a ring, position P in row P mod S_max, so S_max bounds the window, not the context.  The
 *      attention rule is the window's; the append writes row P mod S_max.  Positions are clamped to
 *      [0, INT32_MAX - S_max] instead of S_max - 1 (S_max - S for a prompt), int64 ones before they are narrowed.  A ring
 *      call is bit for bit the windowed call over a linear cache holding the same positions.  Refused before any launch:
 *      window 0, S_max < window (the window and the row being appended must be distinct rows), S_max % 64 != 0 (a prompt
 *      key tile never straddles the wrap), and a prompt chunk with S_max < window + S - 1 (its appends would overwrite
 *      rows its own earlier queries read; split the prompt into chunks of at most S_max - window + 1 tokens).  Every
 *      other AttentionKVCache launcher refuses the flag. ---- */
int it_b200_attention_kvcache_window(int dtype, void *k_cache, void *v_cache, const void *k_scale, const void *v_scale,
                                     const void *q, const void *k, const void *v, const void *rope_pos, int rope_pos_dtype,
                                     const void *inv_freq, int freq_dtype, int64_t freq_len, int window, const void *position_id,
                                     int pos_flags, void *out, int B, int Hq, int Hkv, int S_max, int D, void *workspace,
                                     int64_t workspace_bytes, void *stream);
int it_b200_attention_kvcache_prompt_window(int dtype, void *k_cache, void *v_cache, const void *q, const void *k, const void *v,
                                            const void *position_id, int pos_flags, void *out, int B, int Hq, int Hkv, int S,
                                            int S_max, int D, int window, void *stream);

/* ---- Fused prefill attention (q-len > 1) on wgmma (SURVEY 8(f-3); attention_prefill.cu):
 *      out[b,h] = softmax((q . k^T) (/ or *) scale + mask) . v, q / k / v / out [B, H, S, D] f16 / bf16, D = 64 or 128.
 *      Replaces the chain the frontend lowers multi-token attention to -- Transpose(k) -> MatMul (matmul.cc:66-211) ->
 *      Div / Mul by a scalar (element_wise.cc) -> Add(mask) -> Softmax(axis -1) (softmax.cu:242-404) -> MatMul -- and keeps
 *      its rounding points (every intermediate rounded to the storage type).  scale: device scalar or NULL; mask: additive,
 *      element (b,h,i,j) at mask[b*sb + h*sh + i*si + j*sj] (0 = broadcast) or NULL.  No causal assumption. ---- */
int it_b200_attention_prefill(int dtype, const void *q, const void *k, const void *v, void *out, int B, int H, int S_q,
                              int S_kv, int D, const void *scale, int scale_is_div, const void *mask,
                              int64_t mask_stride_b, int64_t mask_stride_h, int64_t mask_stride_i,
                              int64_t mask_stride_j, void *stream);
/* The same kernel over STRIDED views of q / k / v / out: element (b, h, i, d) at base[b*st[0] + h*st[1] + i*st[2] + d] (strides in
 * elements, multiples of 8; d contiguous).  The frontend's Split -> Reshape -> Transpose([0,2,1,3]) of a fused q/k/v projection
 * output [B, S, 3 H D] and the Transpose -> Reshape behind the attention become addressing (4-D tensor maps, strided output rows):
 * the schedule's PrefillAttention step absorbs those operators when every link has a single consumer. */
int it_b200_attention_prefill_strided(int dtype, const void *q, const void *k, const void *v, void *out, int B, int H, int S_q,
                                      int S_kv, int D, const int64_t *q_strides, const int64_t *k_strides,
                                      const int64_t *v_strides, const int64_t *out_strides, const void *scale, int scale_is_div,
                                      const void *mask, int64_t mask_stride_b, int64_t mask_stride_h, int64_t mask_stride_i,
                                      int64_t mask_stride_j, void *stream);

/* ======================================================================
 * (2) Graph / runtime handle API -- see infinitensor_b200/csrc/host/capi.cc.
 * Mirrors reference GraphHandlerObj (include/core/graph_handler.h:15-159),
 * CudaRuntimeObj (include/cuda/cuda_runtime.h:70-110) and the Tensor bindings
 * (src/ffi/ffi_infinitensor.cc:499-535).  Handles are opaque.
 * ====================================================================== */
typedef struct itb_runtime itb_runtime;
typedef struct itb_graph itb_graph;
typedef int64_t itb_tensor; /* tensor id inside one graph; -1 = null */

int itb_runtime_create(int device, int64_t cuda_graph_cache_capacity, itb_runtime **out);
int itb_runtime_destroy(itb_runtime *rt);
int itb_runtime_init_comm(itb_runtime *rt, const char *name, int world_size, int rank);
int itb_runtime_init_comm_with_id(itb_runtime *rt, const void *nccl_unique_id, int id_bytes,
                                  int world_size, int rank);
int itb_runtime_nccl_unique_id(void *out, int out_bytes);
/* NVLink peer-memory comm for the fused all-reduce: export this rank's 64-byte cudaIpc handle, then import all ranks' */
int itb_runtime_p2p_export(itb_runtime *rt, void *handle_out_64_bytes);
int itb_runtime_p2p_import(itb_runtime *rt, const void *all_handles, int world_size, int rank);
int64_t itb_runtime_cuda_graph_cache_size(itb_runtime *rt);
int64_t itb_runtime_cuda_graph_capture_count(itb_runtime *rt);
int itb_runtime_clear_cuda_graph_cache(itb_runtime *rt);
int64_t itb_runtime_kernel_launches(itb_runtime *rt); /* launches issued by our kernels so far */
void *itb_runtime_stream(itb_runtime *rt);

int itb_graph_create(itb_runtime *rt, itb_graph **out);
int itb_graph_destroy(itb_graph *g);
int itb_graph_tensor(itb_graph *g, const int *dims, int rank, int dtype, itb_tensor *out);
int itb_tensor_set_weight(itb_graph *g, itb_tensor t);
int itb_tensor_set_input(itb_graph *g, itb_tensor t);
int itb_tensor_set_output(itb_graph *g, itb_tensor t);
int itb_tensor_rank(itb_graph *g, itb_tensor t);
int itb_tensor_shape(itb_graph *g, itb_tensor t, int *dims_out);
int itb_tensor_dtype(itb_graph *g, itb_tensor t);
int64_t itb_tensor_bytes(itb_graph *g, itb_tensor t);
void *itb_tensor_device_ptr(itb_graph *g, itb_tensor t);
int itb_tensor_copyin(itb_graph *g, itb_tensor t, const void *host, int64_t bytes);
int itb_tensor_copyout(itb_graph *g, itb_tensor t, void *host, int64_t bytes);
int itb_tensor_copyin_async(itb_graph *g, itb_tensor t, const void *pinned_host, int64_t bytes);
int itb_tensor_copyout_async(itb_graph *g, itb_tensor t, void *pinned_host, int64_t bytes);

/* Generic operator insertion: op_type is the reference OpType name ("MatMul", "Conv",
 * "AttentionKVCache", ...).  inputs/outputs are tensor ids (-1 in outputs = infer + create).
 * iattrs / fattrs carry the operator's constructor attributes in the reference's argument
 * order (documented per op in INTEGRATION.md).  The created output ids are written back. */
int itb_graph_add_op(itb_graph *g, const char *op_type, const itb_tensor *inputs, int n_inputs,
                     itb_tensor *outputs, int n_outputs, const int64_t *iattrs, int n_iattrs,
                     const double *fattrs, int n_fattrs);
int itb_graph_num_ops(itb_graph *g);
int itb_graph_op_type(itb_graph *g, int index, char *buf, int buf_len);
/* the fused execution schedule derived from the graph ("Kind:Op[+Op...]" per step; see ExecStep, core.h) */
int itb_graph_num_steps(itb_graph *g);
int itb_graph_step(itb_graph *g, int index, char *buf, int buf_len);
int itb_graph_topo_sort(itb_graph *g);
int itb_graph_shape_infer(itb_graph *g);
int itb_graph_optimize(itb_graph *g);
int itb_graph_data_malloc(itb_graph *g, int use_naive_allocator, int64_t mem_pool_size);
int itb_graph_run(itb_graph *g);
int itb_graph_run_without_sync(itb_graph *g);
int itb_graph_run_with_cudagraph(itb_graph *g);
/* graph replay without the trailing stream synchronise (serving loop: copyin_async -> launch -> copyout_async -> sync) */
int itb_graph_launch_cudagraph_async(itb_graph *g);
int itb_graph_tune(itb_graph *g);
int itb_graph_sync(itb_graph *g);
double itb_graph_get_perf_time(itb_graph *g);
/* PerfEngine table (filled by itb_graph_tune) <-> JSON file, in the layout of the reference's savePerfEngineData /
 * loadPerfEngineData (src/core/perf_engine.cc:7-22): files are interchangeable; load replaces the table. */
int itb_perf_engine_save(const char *path);
int itb_perf_engine_load(const char *path);
int64_t itb_perf_engine_size(void);
void itb_perf_engine_clear(void);
int64_t itb_graph_arena_bytes(itb_graph *g, int which /*0 weights, 1 activations*/);

#ifdef __cplusplus
}
#endif
#endif /* IT_B200_H */
