// gemm.cuh -- shared GEMM argument block + Hopper PTX helpers (mbarrier, TMA, wgmma).
#pragma once
#include <cuda.h>

#include "common.cuh"

namespace itb {

struct GemmArgs {
    const void *A, *B, *bias;
    void *C;
    int64_t batch;
    int m, n, k;
    int64_t stride_a, stride_b;  // elements between batches (0 = broadcast)
    int trans_a, trans_b;
    int64_t bias_sb, bias_sm, bias_sn;  // bias strides in elements (0 = broadcast)
    int act;                            // 0 none, 1 relu, 2 sigmoid, 3 tanh
    // optional output scatter (conv with the batch folded into the GEMM columns): column gn of row m goes to
    // C[(gn / c_block) * c_block_stride + m * c_block + gn % c_block]; 0 = plain row-major C[m * n + gn].
    // Honoured by the wgmma kernel only (launch_gemm_tc is called directly for it).
    int c_block = 0;
    int64_t c_block_stride = 0;
    // conv with an NHWC consumer: element (row m = filter, column gn = pixel) goes to C[gn * m_total + m] (wgmma kernel, batch 1)
    int c_nhwc = 0;
    // optional fused conv tail (wgmma kernel only), applied per output ROW m (= conv filter) after the product has been
    // rounded to the storage dtype, each stage rounded like the separate kernel it replaces:
    //   BatchNorm (fp32 statistics, bn_scale != nullptr) -> + residual (same layout as C) -> ReLU
    const float *bn_mean = nullptr, *bn_var = nullptr, *bn_scale = nullptr, *bn_bias = nullptr;
    float bn_eps = 0.f;
    const void *residual = nullptr;
    int post_relu = 0;
    int no_splitk = 0;  // keep one CTA per output tile (conv GEMMs: same fp32 summation order with and without a tail)
    // weight-only quantisation (SURVEY 8(f-4)): B holds FP8 E4M3 codes [K, N] (one byte each); the kernel converts them to the
    // activation type on their way into the tensor core and multiplies column n of the fp32 sum by w_scale[n] in the epilogue
    const float *w_scale = nullptr;
};

__device__ __forceinline__ float gemm_act(int act, float v) {
    switch (act & 0xff) {
    case 1: return v > 0.f ? v : 0.f;
    case 2: return 1.f / (1.f + expf(-v));
    case 3: return tanhf(v);
    }
    return v;
}

int launch_gemm_simt(int dtype, const GemmArgs &g, cudaStream_t st);
// returns 0 = launched, 1 = error, -1 = shape not taken by this kernel
int launch_gemm_skinny(int dtype, const GemmArgs &g, cudaStream_t st);
int launch_gemm_skinny_grouped(int dtype, const GemmArgs &g0, int ngroups, const void *const *Ws, void *const *Cs,
                               const int *Ns, cudaStream_t st);
int launch_gemm_tc(int dtype, const GemmArgs &g, cudaStream_t st);
int launch_gemm_tc_grouped(int dtype, const GemmArgs &g0, int ngroups, const void *const *Ws, void *const *Cs, const int *Ns,
                           cudaStream_t st);
// column tiles (128 wide) from which a decode GEMM (M <= 64) runs on the wgmma kernel instead of gemm_skinny: once its tiles alone
// occupy every SM.  With fewer tiles gemm_skinny's cluster split-K spreads the weight stream over more SMs (tools/gemm_bench.py
// compares the two)
constexpr int TC_MIN_TILES_DECODE = kNumSMs;
int launch_gemm_skinny_fp8w(int dtype, const GemmArgs &g0, int ngroups, const void *const *Wq, const float *const *scales,
                            void *const *Cs, const int *Ns, cudaStream_t st);

// ---- TMA descriptor creation (driver entry point fetched at run time; no link-time libcuda) ----
// 2-D row-major tensor [rows, cols] of 2-byte elements, box [box_rows, box_cols], 128B swizzle.
bool make_tma_2d_b16(CUtensorMap *map, const void *base, uint64_t rows, uint64_t cols,
                     uint64_t row_stride_elems, uint32_t box_rows, uint32_t box_cols, int swizzle_bytes);

// 2-D row-major tensor [rows, cols] of BYTES (fp8 codes), box [box_rows, box_cols], no swizzle
bool make_tma_2d_u8(CUtensorMap *map, const void *base, uint64_t rows, uint64_t cols, uint64_t row_stride_bytes,
                    uint32_t box_rows, uint32_t box_cols);
// the same with 128B swizzle (box_cols = 128)
bool make_tma_2d_u8_sw128(CUtensorMap *map, const void *base, uint64_t rows, uint64_t cols, uint64_t row_stride_bytes,
                          uint32_t box_rows, uint32_t box_cols);

bool make_tma_3d_b16(CUtensorMap *map, const void *base, uint64_t batch, uint64_t rows, uint64_t cols,
                     uint64_t row_stride_elems, uint64_t batch_stride_elems, uint32_t box_rows, uint32_t box_cols);

bool make_tma_4d_b16(CUtensorMap *map, const void *base, uint64_t d0, uint64_t d1, uint64_t d2, uint64_t d3, uint64_t s1, uint64_t s2,
                     uint64_t s3, uint32_t b0, uint32_t b1, uint32_t b2, uint32_t b3);

// ---------------------------------------------------------------- PTX helpers
__device__ __forceinline__ uint32_t smem_u32(const void *p) { return (uint32_t)__cvta_generic_to_shared(p); }

__device__ __forceinline__ void mbar_init(uint64_t *bar, uint32_t count) {
    asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(smem_u32(bar)), "r"(count));
}
__device__ __forceinline__ void fence_mbar_init() {
    asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
}
__device__ __forceinline__ void fence_proxy_async() {
    asm volatile("fence.proxy.async.shared::cta;" ::: "memory");
}
__device__ __forceinline__ void mbar_expect_tx(uint64_t *bar, uint32_t bytes) {
    asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(smem_u32(bar)), "r"(bytes)
                 : "memory");
}
__device__ __forceinline__ void mbar_arrive_n(uint64_t *bar, uint32_t n) {
    asm volatile("mbarrier.arrive.shared::cta.b64 _, [%0], %1;" ::"r"(smem_u32(bar)), "r"(n) : "memory");
}
__device__ __forceinline__ void mbar_arrive(uint64_t *bar) {
    asm volatile("mbarrier.arrive.shared::cta.b64 _, [%0];" ::"r"(smem_u32(bar)) : "memory");
}
__device__ __forceinline__ bool mbar_try_wait(uint64_t *bar, uint32_t parity) {
    uint32_t ok;
    asm volatile(
        "{\n\t.reg .pred p;\n\t"
        "mbarrier.try_wait.parity.shared::cta.b64 p, [%1], %2;\n\t"
        "selp.u32 %0, 1, 0, p;\n\t}"
        : "=r"(ok)
        : "r"(smem_u32(bar)), "r"(parity)
        : "memory");
    return ok != 0;
}
// Bounded spin: a protocol bug must trap, not hang the GPU box.
__device__ __forceinline__ void mbar_wait(uint64_t *bar, uint32_t parity) {
    uint32_t spins = 0;
    while (!mbar_try_wait(bar, parity)) {
        if (++spins > (1u << 26)) __trap();
    }
}

__device__ __forceinline__ uint64_t l2_policy_evict_first() {
    uint64_t p;
    asm volatile("createpolicy.fractional.L2::evict_first.b64 %0, 1.0;" : "=l"(p));
    return p;
}
__device__ __forceinline__ uint64_t l2_policy_evict_last() {
    uint64_t p;
    asm volatile("createpolicy.fractional.L2::evict_last.b64 %0, 1.0;" : "=l"(p));
    return p;
}

__device__ __forceinline__ void tma_prefetch_desc(const CUtensorMap *m) {
    asm volatile("prefetch.tensormap [%0];" ::"l"(reinterpret_cast<uint64_t>(m)) : "memory");
}
// 2-D tile load: coordinates are (c0 = innermost/column index, c1 = row index)
__device__ __forceinline__ void tma_load_2d(void *smem_dst, const CUtensorMap *m, uint64_t *bar, int c0, int c1,
                                            uint64_t policy) {
    asm volatile(
        "cp.async.bulk.tensor.2d.shared::cluster.global.mbarrier::complete_tx::bytes.L2::cache_hint"
        " [%0], [%1, {%3, %4}], [%2], %5;"
        ::"r"(smem_u32(smem_dst)), "l"(reinterpret_cast<uint64_t>(m)), "r"(smem_u32(bar)), "r"(c0), "r"(c1),
          "l"(policy)
        : "memory");
}

// 3-D tile load: (c0 = column, c1 = row, c2 = batch)
__device__ __forceinline__ void tma_load_3d(void *smem_dst, const CUtensorMap *m, uint64_t *bar, int c0, int c1, int c2,
                                            uint64_t policy) {
    asm volatile(
        "cp.async.bulk.tensor.3d.shared::cluster.global.mbarrier::complete_tx::bytes.L2::cache_hint"
        " [%0], [%1, {%3, %4, %5}], [%2], %6;"
        ::"r"(smem_u32(smem_dst)), "l"(reinterpret_cast<uint64_t>(m)), "r"(smem_u32(bar)), "r"(c0), "r"(c1), "r"(c2),
          "l"(policy)
        : "memory");
}

__device__ __forceinline__ void bulk_load_1d(void *smem_dst, const void *gsrc, uint32_t bytes, uint64_t *bar,
                                             uint64_t policy) {
    asm volatile(
        "cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes.L2::cache_hint [%0], [%1], %2, [%3], %4;"
        ::"r"(smem_u32(smem_dst)), "l"(gsrc), "r"(bytes), "r"(smem_u32(bar)), "l"(policy)
        : "memory");
}
__device__ __forceinline__ void named_bar_sync(int id, int threads) {
    asm volatile("bar.sync %0, %1;" ::"r"(id), "r"(threads) : "memory");
}

// ---- wgmma (Hopper warpgroup MMA) ------------------------------------------------------------------
// D[64 x N] (+)= A[64 x 16] . B[16 x N], both operands read from shared memory through descriptors, fp32 accumulator in the
// registers of the issuing warpgroup (128 threads).  TA / TB = 1: that operand is MN-major (transposed) instead of K-major.
// Fragment layout of the accumulator: d[4j + 2i + e] holds row 16 (warp % 4) + lane / 4 + 8 i, column 8 j + 2 (lane % 4) + e.
template <typename T, int N> struct Wgmma;
template <> struct Wgmma<__half, 16> {
    template <int TA, int TB> static __device__ __forceinline__ void mma(float (&d)[8], uint64_t a, uint64_t b, uint32_t acc) {
        asm volatile("{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %10, 0;\n\t"
                     "wgmma.mma_async.sync.aligned.m64n16k16.f32.f16.f16 {%0,%1,%2,%3,%4,%5,%6,%7}, %8, %9, p, 1, 1, %11, %12;\n\t}"
                     : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7])
                     : "l"(a), "l"(b), "r"(acc), "n"(TA), "n"(TB));
    }
};
template <> struct Wgmma<__half, 32> {
    template <int TA, int TB> static __device__ __forceinline__ void mma(float (&d)[16], uint64_t a, uint64_t b, uint32_t acc) {
        asm volatile("{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %18, 0;\n\t"
                     "wgmma.mma_async.sync.aligned.m64n32k16.f32.f16.f16 {%0,%1,%2,%3,%4,%5,%6,%7,%8,%9,%10,%11,%12,%13,%14,%15}, %16, %17, p, 1, 1, %19, %20;\n\t}"
                     : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]), "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15])
                     : "l"(a), "l"(b), "r"(acc), "n"(TA), "n"(TB));
    }
};
template <> struct Wgmma<__half, 64> {
    template <int TA, int TB> static __device__ __forceinline__ void mma(float (&d)[32], uint64_t a, uint64_t b, uint32_t acc) {
        asm volatile("{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %34, 0;\n\t"
                     "wgmma.mma_async.sync.aligned.m64n64k16.f32.f16.f16 {%0,%1,%2,%3,%4,%5,%6,%7,%8,%9,%10,%11,%12,%13,%14,%15,%16,%17,%18,%19,%20,%21,%22,%23,%24,%25,%26,%27,%28,%29,%30,%31}, %32, %33, p, 1, 1, %35, %36;\n\t}"
                     : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]), "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]), "+f"(d[16]), "+f"(d[17]), "+f"(d[18]), "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23]), "+f"(d[24]), "+f"(d[25]), "+f"(d[26]), "+f"(d[27]), "+f"(d[28]), "+f"(d[29]), "+f"(d[30]), "+f"(d[31])
                     : "l"(a), "l"(b), "r"(acc), "n"(TA), "n"(TB));
    }
};
template <> struct Wgmma<__half, 128> {
    template <int TA, int TB> static __device__ __forceinline__ void mma(float (&d)[64], uint64_t a, uint64_t b, uint32_t acc) {
        asm volatile("{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %66, 0;\n\t"
                     "wgmma.mma_async.sync.aligned.m64n128k16.f32.f16.f16 {%0,%1,%2,%3,%4,%5,%6,%7,%8,%9,%10,%11,%12,%13,%14,%15,%16,%17,%18,%19,%20,%21,%22,%23,%24,%25,%26,%27,%28,%29,%30,%31,%32,%33,%34,%35,%36,%37,%38,%39,%40,%41,%42,%43,%44,%45,%46,%47,%48,%49,%50,%51,%52,%53,%54,%55,%56,%57,%58,%59,%60,%61,%62,%63}, %64, %65, p, 1, 1, %67, %68;\n\t}"
                     : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]), "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]), "+f"(d[16]), "+f"(d[17]), "+f"(d[18]), "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23]), "+f"(d[24]), "+f"(d[25]), "+f"(d[26]), "+f"(d[27]), "+f"(d[28]), "+f"(d[29]), "+f"(d[30]), "+f"(d[31]), "+f"(d[32]), "+f"(d[33]), "+f"(d[34]), "+f"(d[35]), "+f"(d[36]), "+f"(d[37]), "+f"(d[38]), "+f"(d[39]), "+f"(d[40]), "+f"(d[41]), "+f"(d[42]), "+f"(d[43]), "+f"(d[44]), "+f"(d[45]), "+f"(d[46]), "+f"(d[47]), "+f"(d[48]), "+f"(d[49]), "+f"(d[50]), "+f"(d[51]), "+f"(d[52]), "+f"(d[53]), "+f"(d[54]), "+f"(d[55]), "+f"(d[56]), "+f"(d[57]), "+f"(d[58]), "+f"(d[59]), "+f"(d[60]), "+f"(d[61]), "+f"(d[62]), "+f"(d[63])
                     : "l"(a), "l"(b), "r"(acc), "n"(TA), "n"(TB));
    }
};
template <> struct Wgmma<__nv_bfloat16, 16> {
    template <int TA, int TB> static __device__ __forceinline__ void mma(float (&d)[8], uint64_t a, uint64_t b, uint32_t acc) {
        asm volatile("{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %10, 0;\n\t"
                     "wgmma.mma_async.sync.aligned.m64n16k16.f32.bf16.bf16 {%0,%1,%2,%3,%4,%5,%6,%7}, %8, %9, p, 1, 1, %11, %12;\n\t}"
                     : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7])
                     : "l"(a), "l"(b), "r"(acc), "n"(TA), "n"(TB));
    }
};
template <> struct Wgmma<__nv_bfloat16, 32> {
    template <int TA, int TB> static __device__ __forceinline__ void mma(float (&d)[16], uint64_t a, uint64_t b, uint32_t acc) {
        asm volatile("{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %18, 0;\n\t"
                     "wgmma.mma_async.sync.aligned.m64n32k16.f32.bf16.bf16 {%0,%1,%2,%3,%4,%5,%6,%7,%8,%9,%10,%11,%12,%13,%14,%15}, %16, %17, p, 1, 1, %19, %20;\n\t}"
                     : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]), "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15])
                     : "l"(a), "l"(b), "r"(acc), "n"(TA), "n"(TB));
    }
};
template <> struct Wgmma<__nv_bfloat16, 64> {
    template <int TA, int TB> static __device__ __forceinline__ void mma(float (&d)[32], uint64_t a, uint64_t b, uint32_t acc) {
        asm volatile("{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %34, 0;\n\t"
                     "wgmma.mma_async.sync.aligned.m64n64k16.f32.bf16.bf16 {%0,%1,%2,%3,%4,%5,%6,%7,%8,%9,%10,%11,%12,%13,%14,%15,%16,%17,%18,%19,%20,%21,%22,%23,%24,%25,%26,%27,%28,%29,%30,%31}, %32, %33, p, 1, 1, %35, %36;\n\t}"
                     : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]), "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]), "+f"(d[16]), "+f"(d[17]), "+f"(d[18]), "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23]), "+f"(d[24]), "+f"(d[25]), "+f"(d[26]), "+f"(d[27]), "+f"(d[28]), "+f"(d[29]), "+f"(d[30]), "+f"(d[31])
                     : "l"(a), "l"(b), "r"(acc), "n"(TA), "n"(TB));
    }
};
template <> struct Wgmma<__nv_bfloat16, 128> {
    template <int TA, int TB> static __device__ __forceinline__ void mma(float (&d)[64], uint64_t a, uint64_t b, uint32_t acc) {
        asm volatile("{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %66, 0;\n\t"
                     "wgmma.mma_async.sync.aligned.m64n128k16.f32.bf16.bf16 {%0,%1,%2,%3,%4,%5,%6,%7,%8,%9,%10,%11,%12,%13,%14,%15,%16,%17,%18,%19,%20,%21,%22,%23,%24,%25,%26,%27,%28,%29,%30,%31,%32,%33,%34,%35,%36,%37,%38,%39,%40,%41,%42,%43,%44,%45,%46,%47,%48,%49,%50,%51,%52,%53,%54,%55,%56,%57,%58,%59,%60,%61,%62,%63}, %64, %65, p, 1, 1, %67, %68;\n\t}"
                     : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]), "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]), "+f"(d[16]), "+f"(d[17]), "+f"(d[18]), "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23]), "+f"(d[24]), "+f"(d[25]), "+f"(d[26]), "+f"(d[27]), "+f"(d[28]), "+f"(d[29]), "+f"(d[30]), "+f"(d[31]), "+f"(d[32]), "+f"(d[33]), "+f"(d[34]), "+f"(d[35]), "+f"(d[36]), "+f"(d[37]), "+f"(d[38]), "+f"(d[39]), "+f"(d[40]), "+f"(d[41]), "+f"(d[42]), "+f"(d[43]), "+f"(d[44]), "+f"(d[45]), "+f"(d[46]), "+f"(d[47]), "+f"(d[48]), "+f"(d[49]), "+f"(d[50]), "+f"(d[51]), "+f"(d[52]), "+f"(d[53]), "+f"(d[54]), "+f"(d[55]), "+f"(d[56]), "+f"(d[57]), "+f"(d[58]), "+f"(d[59]), "+f"(d[60]), "+f"(d[61]), "+f"(d[62]), "+f"(d[63])
                     : "l"(a), "l"(b), "r"(acc), "n"(TA), "n"(TB));
    }
};

__device__ __forceinline__ void wg_fence() { asm volatile("wgmma.fence.sync.aligned;" ::: "memory"); }
__device__ __forceinline__ void wg_commit() { asm volatile("wgmma.commit_group.sync.aligned;" ::: "memory"); }
template <int N> __device__ __forceinline__ void wg_wait() { asm volatile("wgmma.wait_group.sync.aligned %0;" ::"n"(N) : "memory"); }

// shared-memory matrix descriptor (GMMA): start>>4 [0,14), LBO>>4 [16,30), SBO>>4 [32,46), layout type [62,64) (1 = SWIZZLE_128B).
// 128B swizzle, K-major: 8-row groups SBO apart, LBO unused.  MN-major: 64-element MN blocks LBO apart, 8-row k groups SBO apart.
// A k16 step or a 64-row sub-tile is selected by adding (byte offset >> 4) to the descriptor.
__device__ __forceinline__ uint64_t gmma_desc_sw128(uint32_t smem_addr, uint32_t lbo_bytes, uint32_t sbo_bytes) {
    uint64_t d = 0;
    d |= (uint64_t)((smem_addr & 0x3FFFF) >> 4);
    d |= (uint64_t)((lbo_bytes >> 4) & 0x3FFF) << 16;
    d |= (uint64_t)((sbo_bytes >> 4) & 0x3FFF) << 32;
    d |= (uint64_t)1 << 62;
    return d;
}

// A 128-row accumulator tile parked in shared memory as acc[col * ACC_LD + row] (fp32): the two 64-row halves come from two
// warpgroups' wgmma fragments, and an epilogue thread that owns one row reads consecutive columns.  The padding of 4 words makes
// both the fragment stores (8 rows x 4 column pairs per instruction) and the row reads bank-conflict free.
constexpr int ACC_LD = 132;
// store this warpgroup's m64 x N fragment as rows [row0, row0 + 64) of the parked tile
template <int N>
__device__ __forceinline__ void acc_park(const float (&d)[N / 2], float *acc, int row0) {
    const int w = (threadIdx.x >> 5) & 3, l = threadIdx.x & 31;
    const int r = row0 + 16 * w + (l >> 2), c = 2 * (l & 3);
#pragma unroll
    for (int j = 0; j < N / 8; ++j)
#pragma unroll
        for (int i = 0; i < 2; ++i)
#pragma unroll
            for (int e = 0; e < 2; ++e) acc[(8 * j + c + e) * ACC_LD + r + 8 * i] = d[4 * j + 2 * i + e];
}
// columns [c0, c0 + NV) of one row of a parked tile (as raw bits, like the values of a tensor-memory load)
template <int NV>
__device__ __forceinline__ void acc_row(const float *acc, int row, int c0, uint32_t (&v)[NV]) {
#pragma unroll
    for (int j = 0; j < NV; ++j) v[j] = __float_as_uint(acc[(c0 + j) * ACC_LD + row]);
}

__device__ __forceinline__ void ldmatrix_x4(uint32_t &r0, uint32_t &r1, uint32_t &r2, uint32_t &r3, uint32_t addr) {
    asm volatile("ldmatrix.sync.aligned.m8n8.x4.shared.b16 {%0,%1,%2,%3}, [%4];"
                 : "=r"(r0), "=r"(r1), "=r"(r2), "=r"(r3) : "r"(addr));
}
__device__ __forceinline__ void ldmatrix_x4_trans(uint32_t &r0, uint32_t &r1, uint32_t &r2, uint32_t &r3,
                                                  uint32_t addr) {
    asm volatile("ldmatrix.sync.aligned.m8n8.x4.trans.shared.b16 {%0,%1,%2,%3}, [%4];"
                 : "=r"(r0), "=r"(r1), "=r"(r2), "=r"(r3) : "r"(addr));
}
template <typename T>
__device__ __forceinline__ void mma_m16n8k16(float (&d)[4], const uint32_t (&a)[4], uint32_t b0, uint32_t b1);
template <>
__device__ __forceinline__ void mma_m16n8k16<__nv_bfloat16>(float (&d)[4], const uint32_t (&a)[4], uint32_t b0,
                                                            uint32_t b1) {
    asm volatile("mma.sync.aligned.m16n8k16.row.col.f32.bf16.bf16.f32 {%0,%1,%2,%3}, {%4,%5,%6,%7}, {%8,%9}, "
                 "{%0,%1,%2,%3};"
                 : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3])
                 : "r"(a[0]), "r"(a[1]), "r"(a[2]), "r"(a[3]), "r"(b0), "r"(b1));
}
template <>
__device__ __forceinline__ void mma_m16n8k16<__half>(float (&d)[4], const uint32_t (&a)[4], uint32_t b0,
                                                     uint32_t b1) {
    asm volatile("mma.sync.aligned.m16n8k16.row.col.f32.f16.f16.f32 {%0,%1,%2,%3}, {%4,%5,%6,%7}, {%8,%9}, "
                 "{%0,%1,%2,%3};"
                 : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3])
                 : "r"(a[0]), "r"(a[1]), "r"(a[2]), "r"(a[3]), "r"(b0), "r"(b1));
}

}  // namespace itb
