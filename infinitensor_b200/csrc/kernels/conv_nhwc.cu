// conv_nhwc.cu -- Conv2d as an IMPLICIT GEMM on the wgmma tensor cores (sm_90a), activations in NHWC.
//
//   y[n, oh, ow, f] = tail( sum_{r, s, c} x[n, oh*sh - ph + r*dh, ow*sw - pw + s*dw, c] . w[f, c, r, s] )
//
// The im2col matrix is never materialised: the TMA unit's IM2COL mode (cuTensorMapEncodeIm2col) walks 128 consecutive
// output pixels of the (n, oh, ow) space -- stride, padding (zero fill) and image boundaries handled by the hardware -- and
// delivers, for one filter tap (r, s), their 64-channel slices as a K-major [128 pixels x 128 B] tile in the 128B-swizzle
// layout the wgmma descriptor reads.  The GEMM per output tile:
//     D[pixel (128 rows), f (FT = 64 columns)] += A[pixel, k64] . B[f, k64]^T ,  k = (r, s, c)
//   A = activations (im2col TMA), B = filters as [F][R*S][Cp] rows (K-major; 1x1 filters are used as stored, [F][C]).
// One PERSISTENT CTA per SM walks (pixel tile, filter tile) pairs:
//   warp 12     : TMA producer (im2col box + filter box per k-tile, mbarrier ring)
//   warps 8..11 : MMA warpgroup: wgmma for both 64-pixel halves, fp32 accumulators in registers; each finished tile is parked
//                 in shared memory, so the epilogue of tile i runs under the MMAs of tile i+1
//   warps 0..7  : epilogue: parked accumulator rows, BatchNorm (folded to one FMA) + residual + ReLU,
//                 16-byte stores along f (NHWC) or coalesced along pixels (NCHW output for consumers outside the NHWC domain)
// Replaces cudnnConvolutionForward + the separate BatchNorm / Add / Relu kernels (reference src/kernels/cuda/conv.cc:143-168,
// batch_norm.cc:9-69, element_wise.cu) for the ResNet-style Conv -> BN -> [Add] -> [Relu] chains.
#include <algorithm>
#include <mutex>

#include <cudaTypedefs.h>

#include "conv_shapes.h"
#include "gemm.cuh"

namespace itb {

constexpr int CV_BM = 128, CV_BK = 64;
constexpr int CV_A_BYTES = CV_BM * CV_BK * 2;  // 16 KB
constexpr int CV_EPI_WARPS = 8;
constexpr int CV_EPI_THREADS = CV_EPI_WARPS * 32;
constexpr int CV_WARP_MMA = 8, CV_WARP_TMA = 12;  // MMA warpgroup = warps 8..11
constexpr int CV_THREADS = (CV_WARP_TMA + 1) * 32;
// filter columns per tile: the MMA warpgroup holds two m64 x FT fp32 accumulators, FT = 128 would spill them
constexpr int CV_FT = 64;

constexpr int CV_RING = 4;                  // staging slabs per epilogue warp
constexpr int CV_SLAB_BYTES = 32 * 32 * 2;  // [32 pixels x 32 filters]

struct ConvNhwcParams {
    void *y;
    const void *residual;  // same layout as y
    const float *bn_mean, *bn_var, *bn_scale, *bn_bias;
    float bn_eps;
    int relu;
    int y_nhwc;
    int P, OW, M, F, FT, tiles_f, tiles, cchunks, Cp, RS, S, sh, sw, ph, pw, dh, dw;
    int stages, b_bytes, stg_off;
};

__device__ __forceinline__ bool mbar_try_wait_addr(uint32_t bar_addr, uint32_t parity) {
    uint32_t ok;
    asm volatile(
        "{\n\t.reg .pred p;\n\t"
        "mbarrier.try_wait.parity.shared::cta.b64 p, [%1], %2;\n\t"
        "selp.u32 %0, 1, 0, p;\n\t}"
        : "=r"(ok)
        : "r"(bar_addr), "r"(parity)
        : "memory");
    return ok != 0;
}
__device__ __forceinline__ void tma_store_2d(const CUtensorMap *m, const void *smem_src, int c0, int c1) {
    asm volatile("cp.async.bulk.tensor.2d.global.shared::cta.bulk_group [%0, {%2, %3}], [%1];" ::"l"(reinterpret_cast<uint64_t>(m)),
                 "r"(smem_u32(smem_src)), "r"(c0), "r"(c1)
                 : "memory");
}
__device__ __forceinline__ void bulk_commit() { asm volatile("cp.async.bulk.commit_group;" ::: "memory"); }
template <int N> __device__ __forceinline__ void bulk_wait_read() {
    asm volatile("cp.async.bulk.wait_group.read %0;" ::"n"(N) : "memory");
}
__device__ __forceinline__ void bulk_wait_all() { asm volatile("cp.async.bulk.wait_group 0;" ::: "memory"); }

__device__ __forceinline__ void tma_im2col_4d(void *smem_dst, const CUtensorMap *m, uint64_t *bar, int c, int w, int h, int n,
                                              uint16_t off_w, uint16_t off_h) {
    asm volatile(
        "cp.async.bulk.tensor.4d.shared::cluster.global.im2col.mbarrier::complete_tx::bytes"
        " [%0], [%1, {%3, %4, %5, %6}], [%2], {%7, %8};"
        ::"r"(smem_u32(smem_dst)), "l"(reinterpret_cast<uint64_t>(m)), "r"(smem_u32(bar)), "r"(c), "r"(w), "r"(h), "r"(n),
          "h"(off_w), "h"(off_h)
        : "memory");
}

template <typename T> struct Pack2;
template <> struct Pack2<__half> {
    static __device__ __forceinline__ uint32_t pack(float a, float b) {
        __half2 h = __floats2half2_rn(a, b);
        return *reinterpret_cast<uint32_t *>(&h);
    }
    static __device__ __forceinline__ float2 unpack(uint32_t u) { return __half22float2(*reinterpret_cast<__half2 *>(&u)); }
};
template <> struct Pack2<__nv_bfloat16> {
    static __device__ __forceinline__ uint32_t pack(float a, float b) {
        __nv_bfloat162 h = __floats2bfloat162_rn(a, b);
        return *reinterpret_cast<uint32_t *>(&h);
    }
    static __device__ __forceinline__ float2 unpack(uint32_t u) {
        return __bfloat1622float2(*reinterpret_cast<__nv_bfloat162 *>(&u));
    }
};

template <typename T, int FT>
__global__ void __launch_bounds__(CV_THREADS, 1) conv_nhwc_kernel(const __grid_constant__ CUtensorMap mapA,
                                                                  const __grid_constant__ CUtensorMap mapB,
                                                                  const __grid_constant__ CUtensorMap mapY,
                                                                  const __grid_constant__ CUtensorMap mapR,
                                                                  ConvNhwcParams p) {
    extern __shared__ uint8_t smem_raw[];
    uint8_t *smem = smem_raw + ((1024u - (smem_u32(smem_raw) & 1023u)) & 1023u);
    const int S = p.stages;
    uint8_t *a_sm = smem;
    uint8_t *b_sm = smem + S * CV_A_BYTES;
    float *acc_sm = reinterpret_cast<float *>(smem + p.stg_off + CV_EPI_WARPS * CV_RING * CV_SLAB_BYTES);  // parked tile [FT][ACC_LD]
    float2 *bn_sm = reinterpret_cast<float2 *>(acc_sm + FT * ACC_LD);  // {a, b}: y = a * conv + b
    uint64_t *full = reinterpret_cast<uint64_t *>(bn_sm + FT);
    uint64_t *empty = full + S;
    uint64_t *acc_full = empty + S;
    uint64_t *acc_empty = acc_full + 1;
    uint64_t *res_bar = acc_empty + 1;  // [CV_EPI_WARPS][CV_RING]
    // per epilogue warp: CV_RING slabs of [32 pixels x 32 filters] (2 KB, 64B swizzle) -- residual in by TMA, result out by TMA
    uint8_t *stg_sm = smem + p.stg_off;

    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    pdl_trigger();
    if (threadIdx.x == 0) {
        for (int s = 0; s < S; ++s) {
            mbar_init(&full[s], 1);
            mbar_init(&empty[s], 1);
        }
        mbar_init(acc_full, 128);  // every MMA thread after parking its fragment
        mbar_init(acc_empty, CV_EPI_WARPS);
        for (int i = 0; i < CV_EPI_WARPS * CV_RING; ++i) mbar_init(&res_bar[i], 1);
        fence_mbar_init();
    }
    if (warp == CV_WARP_TMA && lane == 0) {
        tma_prefetch_desc(&mapA);
        tma_prefetch_desc(&mapB);
    }
    __syncthreads();
    const int ktiles = p.RS * p.cchunks;

    if (warp == CV_WARP_TMA) {
        // ===== TMA producer (one thread): the loop body is kept to a few dozen instructions -- a single thread retires one
        // dependent instruction every ~5 cycles, and at ~130 instructions per k-tile (runtime divisions for the ring slot and the
        // filter tap) this loop, not the memory system, would set the pace of the whole kernel =====
        if (lane == 0) {
            const uint64_t pol_b = l2_policy_evict_last();  // the filters are re-read by every CTA
            pdl_wait();  // activations (and the repacked filters) come from the kernels before this one
            const uint32_t a_base = smem_u32(a_sm), b_base = smem_u32(b_sm), full_base = smem_u32(full), empty_base = smem_u32(empty);
            const uint32_t tx = CV_A_BYTES + p.b_bytes;
            const uint64_t mA = reinterpret_cast<uint64_t>(&mapA), mB = reinterpret_cast<uint64_t>(&mapB);
            int st = 0, fill = 0;
            uint32_t ph = 0;
            for (int t = blockIdx.x; t < p.tiles; t += gridDim.x) {
                const int ft = t % p.tiles_f, mt = t / p.tiles_f;
                const int m0 = mt * CV_BM;
                const int n0 = m0 / p.P, pp = m0 - n0 * p.P;
                const int oh0 = pp / p.OW, ow0 = pp - oh0 * p.OW;
                const int wc = ow0 * p.sw - p.pw, hc = oh0 * p.sh - p.ph;  // base pixel of the tile's first output position
                const int f0 = ft * p.FT;
                int kb = 0;  // column of the filter matrix: (r*S + s) * Cp + channel
                uint32_t off_w = 0, off_h = 0;
                int s = 0;
                for (int rs = 0; rs < p.RS; ++rs) {
                    const uint32_t offs = off_w | (off_h << 16);
                    for (int c0 = 0; c0 < p.cchunks * CV_BK; c0 += CV_BK) {
                        if (fill >= S) {
                            uint32_t spins = 0;
                            while (!mbar_try_wait_addr(empty_base + st * 8, ph ^ 1))
                                if (++spins > (1u << 26)) __trap();
                        } else {
                            ++fill;
                        }
                        const uint32_t bar = full_base + st * 8;
                        asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(bar), "r"(tx) : "memory");
                        asm volatile(
                            "{\n\t.reg .b16 ow, oh;\n\tmov.b32 {ow, oh}, %7;\n\t"
                            "cp.async.bulk.tensor.4d.shared::cluster.global.im2col.mbarrier::complete_tx::bytes"
                            " [%0], [%1, {%3, %4, %5, %6}], [%2], {ow, oh};\n\t}"
                            ::"r"(a_base + st * CV_A_BYTES), "l"(mA), "r"(bar), "r"(c0), "r"(wc), "r"(hc), "r"(n0), "r"(offs)
                            : "memory");
                        asm volatile(
                            "cp.async.bulk.tensor.2d.shared::cluster.global.mbarrier::complete_tx::bytes.L2::cache_hint"
                            " [%0], [%1, {%3, %4}], [%2], %5;"
                            ::"r"(b_base + st * p.b_bytes), "l"(mB), "r"(bar), "r"(kb + c0), "r"(f0), "l"(pol_b)
                            : "memory");
                        if (++st == S) {
                            st = 0;
                            ph ^= 1;
                        }
                    }
                    kb += p.Cp;
                    off_w += p.dw;
                    if (++s == p.S) {
                        s = 0;
                        off_w = 0;
                        off_h += p.dh;
                    }
                }
            }
        }
        __syncwarp();
    } else if (warp >= CV_WARP_MMA) {
        // ===== MMA warpgroup (same economy as the producer: running ring slot / phase, descriptors advanced by adding to the
        // address field).  Both operands K-major, 128 B rows: 8-row groups 1 KB apart (SBO), one k16 step = +32 B = +2 in the
        // (address >> 4) field; pixels 64..127 of the A tile start 8 KB in =====
        const uint32_t full_base = smem_u32(full);
        const uint64_t a_desc0 = gmma_desc_sw128(smem_u32(a_sm), 0, 1024), b_desc0 = gmma_desc_sw128(smem_u32(b_sm), 0, 1024);
        const uint32_t a_step = CV_A_BYTES >> 4, b_step = (uint32_t)p.b_bytes >> 4;
        const bool leader = (threadIdx.x & 127) == 0;
        int st = 0, it = 0;
        uint32_t ph = 0;
        for (int t = blockIdx.x; t < p.tiles; t += gridDim.x, ++it) {
            float d0[FT / 2], d1[FT / 2];
#pragma unroll
            for (int j = 0; j < FT / 2; ++j) d0[j] = d1[j] = 0.f;
            int prev = -1;
            for (int kt = 0; kt < ktiles; ++kt) {
                {
                    uint32_t spins = 0;
                    while (!mbar_try_wait_addr(full_base + st * 8, ph))
                        if (++spins > (1u << 26)) __trap();
                }
                const uint64_t a_desc = a_desc0 + (uint64_t)(st * a_step), b_desc = b_desc0 + (uint64_t)(st * b_step);
                wg_fence();
#pragma unroll
                for (int kk = 0; kk < CV_BK / 16; ++kk) {
                    Wgmma<T, FT>::template mma<0, 0>(d0, a_desc + 2 * kk, b_desc + 2 * kk, 1u);
                    Wgmma<T, FT>::template mma<0, 0>(d1, a_desc + (CV_A_BYTES / 2 >> 4) + 2 * kk, b_desc + 2 * kk, 1u);
                }
                wg_commit();
                wg_wait<1>();  // the previous stage's MMAs are done: it may be refilled
                if (prev >= 0 && leader) mbar_arrive(&empty[prev]);
                prev = st;
                if (++st == S) {
                    st = 0;
                    ph ^= 1;
                }
            }
            wg_wait<0>();
            if (prev >= 0 && leader) mbar_arrive(&empty[prev]);
            if (it >= 1) mbar_wait(acc_empty, (it - 1) & 1);  // the epilogue has drained the previous parked tile
            acc_park<FT>(d0, acc_sm, 0);
            acc_park<FT>(d1, acc_sm, 64);
            mbar_arrive(acc_full);
        }
    } else {
        // ===== epilogue: warp w owns accumulator rows [32 (w & 3), +32) = pixels; warps 0-3 / 4-7 split the filter columns =====
        pdl_wait();
        const int quad = warp & 3, half = warp >> 2;
        const int row = quad * 32 + lane;
        const int cbeg = half * (FT / 2), cend = cbeg + FT / 2;
        T *Y = (T *)p.y;
        const T *R = (const T *)p.residual;
        int cur_ft = -1, it = 0;
        uint8_t *my_stg = stg_sm + warp * (CV_RING * CV_SLAB_BYTES);
        uint64_t *my_bar = res_bar + warp * CV_RING;
        const uint64_t pol_r = l2_policy_evict_first();  // the residual is read exactly once
        uint32_t q = 0;                    // slabs this warp has processed
        int pf_t = blockIdx.x, pf_c = cbeg;  // next residual slab to request (tile, first column)
        if (p.y_nhwc && R && lane == 0) {
            for (int i = 0; i < CV_RING - 1 && pf_t < p.tiles; ++i) {
                mbar_expect_tx(&my_bar[i], CV_SLAB_BYTES);
                tma_load_2d(my_stg + i * CV_SLAB_BYTES, &mapR, &my_bar[i], (pf_t % p.tiles_f) * p.FT + pf_c,
                            (pf_t / p.tiles_f) * CV_BM + quad * 32, pol_r);
                pf_c += 32;
                if (pf_c >= cend) {
                    pf_c = cbeg;
                    pf_t += gridDim.x;
                }
            }
        }
        for (int t = blockIdx.x; t < p.tiles; t += gridDim.x, ++it) {
            const int ft = t % p.tiles_f, mt = t / p.tiles_f;
            const int f0 = ft * p.FT;
            if (ft != cur_ft) {
                named_bar_sync(1, CV_EPI_THREADS);  // nobody still reads the previous tile's parameters
                for (int i = threadIdx.x; i < p.FT; i += CV_EPI_THREADS) {
                    const int f = f0 + i;
                    float2 ab = make_float2(1.f, 0.f);
                    if (f < p.F && p.bn_scale) {
                        ab.x = p.bn_scale[f] * bn_rs(p.bn_var[f], p.bn_eps);
                        ab.y = __fmaf_rn(-p.bn_mean[f], ab.x, p.bn_bias[f]);
                    }
                    bn_sm[i] = ab;
                }
                named_bar_sync(1, CV_EPI_THREADS);
                cur_ft = ft;
            }
            mbar_wait(acc_full, it & 1);
            const int64_t gm = (int64_t)mt * CV_BM + row;
            const bool ok = gm < p.M;
            if (p.y_nhwc) {
                // slab q of this warp = 32 pixels x 32 filters through ring buffer q % CV_RING: the residual slab lands there by TMA
                // (requested CV_RING - 1 slabs ahead), the result overwrites it in place and leaves by TMA; the tensor maps clip
                // the ragged last pixel tile and filter tile
                const int m_row = mt * CV_BM + quad * 32;
                for (int c0 = cbeg; c0 < cend; c0 += 32, ++q) {
                    const int b = q & (CV_RING - 1);
                    uint8_t *slab = my_stg + b * CV_SLAB_BYTES;
                    uint32_t v[32];
                    acc_row<32>(acc_sm, row, c0, v);
                    if (R) mbar_wait(&my_bar[b], (q / CV_RING) & 1);
                    else if (lane == 0) bulk_wait_read<CV_RING - 1>();  // the store that last used this buffer has read it
                    __syncwarp();
#pragma unroll
                    for (int j8 = 0; j8 < 32; j8 += 8) {
                        uint4 *cell = reinterpret_cast<uint4 *>(slab + lane * 64 + (((j8 >> 3) ^ ((lane >> 1) & 3)) << 4));
                        uint4 rv = make_uint4(0u, 0u, 0u, 0u);
                        if (R) rv = *cell;
                        const uint32_t rw[4] = {rv.x, rv.y, rv.z, rv.w};
                        uint32_t ow[4];
#pragma unroll
                        for (int e = 0; e < 4; ++e) {
                            const float2 ab0 = bn_sm[c0 + j8 + 2 * e], ab1 = bn_sm[c0 + j8 + 2 * e + 1];
                            const float2 rr = Pack2<T>::unpack(rw[e]);
                            float x0 = __fmaf_rn(__uint_as_float(v[j8 + 2 * e]), ab0.x, ab0.y) + rr.x;
                            float x1 = __fmaf_rn(__uint_as_float(v[j8 + 2 * e + 1]), ab1.x, ab1.y) + rr.y;
                            if (p.relu) {
                                x0 = fmaxf(x0, 0.f);
                                x1 = fmaxf(x1, 0.f);
                            }
                            ow[e] = Pack2<T>::pack(x0, x1);
                        }
                        *cell = make_uint4(ow[0], ow[1], ow[2], ow[3]);
                    }
                    fence_proxy_async();
                    __syncwarp();
                    if (lane == 0) {
                        tma_store_2d(&mapY, slab, f0 + c0, m_row);
                        bulk_commit();
                        if (R) {
                            // slab q + CV_RING - 1 goes into the buffer slab q - 1 used: its store must have read the buffer
                            bulk_wait_read<1>();
                            if (pf_t < p.tiles) {
                                const int pb = (q + CV_RING - 1) & (CV_RING - 1);
                                mbar_expect_tx(&my_bar[pb], CV_SLAB_BYTES);
                                tma_load_2d(my_stg + pb * CV_SLAB_BYTES, &mapR, &my_bar[pb], (pf_t % p.tiles_f) * p.FT + pf_c,
                                            (pf_t / p.tiles_f) * CV_BM + quad * 32, pol_r);
                                pf_c += 32;
                                if (pf_c >= cend) {
                                    pf_c = cbeg;
                                    pf_t += gridDim.x;
                                }
                            }
                        }
                    }
                    __syncwarp();
                }
            } else {
                // NCHW output: element (pixel gm = n*P + pp, filter f) at y[(n*F + f)*P + pp]; lanes = consecutive pixels
                const int n = ok ? (int)(gm / p.P) : 0;
                const int64_t base = (int64_t)n * p.F * p.P + (gm - (int64_t)n * p.P);
                for (int c0 = cbeg; c0 < cend; c0 += 32) {
                    uint32_t v[32];
                    acc_row<32>(acc_sm, row, c0, v);
                    if (!ok) continue;
#pragma unroll
                    for (int j = 0; j < 32; ++j) {
                        const int f = f0 + c0 + j;
                        if (f >= p.F) break;
                        const float2 ab = bn_sm[c0 + j];
                        float x = __fmaf_rn(__uint_as_float(v[j]), ab.x, ab.y);
                        if (R) x += to_f(R[base + (int64_t)f * p.P]);
                        if (p.relu) x = fmaxf(x, 0.f);
                        Y[base + (int64_t)f * p.P] = from_f<T>(x);
                    }
                }
            }
            __syncwarp();
            if (lane == 0) mbar_arrive(acc_empty);
        }
        if (lane == 0) bulk_wait_all();  // every TMA store of this warp is complete before the CTA (and its shared memory) goes away
    }
}

// filters [F][C][R*S] -> [F][R*S][Cp] (channel-innermost rows, zero-padded to the 64-channel k-tiles)
template <typename T>
__global__ void __launch_bounds__(256) repack_filters_kernel(const T *__restrict__ w, T *__restrict__ out, int64_t total, int C,
                                                             int RS, int Cp) {
    pdl_trigger();
    pdl_wait();  // the workspace may still be read by the previous conv
    for (int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; i < total; i += (int64_t)gridDim.x * blockDim.x) {
        const int c = (int)(i % Cp);
        const int64_t t = i / Cp;
        const int rs = (int)(t % RS);
        const int64_t f = t / RS;
        out[i] = c < C ? w[(f * C + c) * RS + rs] : from_f<T>(0.f);
    }
}

// the same for RS = 9 (3x3): one thread = 8 channels of one filter = 72 contiguous input elements (nine 16-byte loads), written as
// nine 16-byte channel vectors -- both sides coalesced (the element-wise kernel above reads the filters with a stride of 9 elements)
template <typename T>
__global__ void __launch_bounds__(256) repack_filters9_kernel(const T *__restrict__ w, T *__restrict__ out, int64_t items, int C,
                                                              int Cp) {
    pdl_trigger();
    pdl_wait();
    const int cp8 = Cp / 8;
    for (int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; i < items; i += (int64_t)gridDim.x * blockDim.x) {
        const int c8 = (int)(i % cp8);
        const int64_t f = i / cp8;
        alignas(16) T in[72];
        const bool real = c8 * 8 < C;
        if (real) {
            const uint4 *src = reinterpret_cast<const uint4 *>(w + (f * C + c8 * 8) * 9);
#pragma unroll
            for (int v = 0; v < 9; ++v) reinterpret_cast<uint4 *>(in)[v] = __ldg(src + v);
        }
#pragma unroll
        for (int rs = 0; rs < 9; ++rs) {
            alignas(16) T o[8];
#pragma unroll
            for (int c = 0; c < 8; ++c) o[c] = real ? in[c * 9 + rs] : from_f<T>(0.f);
            *reinterpret_cast<uint4 *>(out + (f * 9 + rs) * Cp + c8 * 8) = *reinterpret_cast<const uint4 *>(o);
        }
    }
}

// every filter bank of a graph in ONE launch (blockIdx.y = bank): the runtime repacks at the start of each step into buffers it
// owns, so no conv waits behind its own repack kernel (16 dependent launches per ResNet-50 step otherwise)
constexpr int CV_REPACK_BATCH = 24;
struct RepackBatch {
    const void *src[CV_REPACK_BATCH];
    void *dst[CV_REPACK_BATCH];
    int F[CV_REPACK_BATCH], C[CV_REPACK_BATCH], RS[CV_REPACK_BATCH], Cp[CV_REPACK_BATCH];
};
template <typename T>
__global__ void __launch_bounds__(256) repack_filters_batch_kernel(const __grid_constant__ RepackBatch b) {
    pdl_trigger();
    pdl_wait();  // the convs of the previous step may still read the buffers
    const int e = blockIdx.y;
    const T *__restrict__ w = (const T *)b.src[e];
    T *__restrict__ out = (T *)b.dst[e];
    const int C = b.C[e], RS = b.RS[e], Cp = b.Cp[e];
    if (RS == 9) {
        const int cp8 = Cp / 8;
        const int64_t items = (int64_t)b.F[e] * cp8;
        for (int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; i < items; i += (int64_t)gridDim.x * blockDim.x) {
            const int c8 = (int)(i % cp8);
            const int64_t f = i / cp8;
            alignas(16) T in[72];
            const bool real = c8 * 8 < C;
            if (real) {
                const uint4 *src = reinterpret_cast<const uint4 *>(w + (f * C + c8 * 8) * 9);
#pragma unroll
                for (int v = 0; v < 9; ++v) reinterpret_cast<uint4 *>(in)[v] = __ldg(src + v);
            }
#pragma unroll
            for (int rs = 0; rs < 9; ++rs) {
                alignas(16) T o[8];
#pragma unroll
                for (int c = 0; c < 8; ++c) o[c] = real ? in[c * 9 + rs] : from_f<T>(0.f);
                *reinterpret_cast<uint4 *>(out + (f * 9 + rs) * Cp + c8 * 8) = *reinterpret_cast<const uint4 *>(o);
            }
        }
    } else {
        const int64_t total = (int64_t)b.F[e] * RS * Cp;
        for (int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; i < total; i += (int64_t)gridDim.x * blockDim.x) {
            const int c = (int)(i % Cp);
            const int64_t t = i / Cp;
            const int rs = (int)(t % RS);
            const int64_t f = t / RS;
            out[i] = c < C ? w[(f * C + c) * RS + rs] : from_f<T>(0.f);
        }
    }
}

static PFN_cuTensorMapEncodeIm2col_v12000 get_im2col_fn() {
    static PFN_cuTensorMapEncodeIm2col_v12000 fn = nullptr;
    static std::once_flag once;
    std::call_once(once, [] {
        void *ptr = nullptr;
        cudaDriverEntryPointQueryResult q;
        if (cudaGetDriverEntryPoint("cuTensorMapEncodeIm2col", &ptr, cudaEnableDefault, &q) == cudaSuccess &&
            q == cudaDriverEntryPointSuccess)
            fn = reinterpret_cast<PFN_cuTensorMapEncodeIm2col_v12000>(ptr);
    });
    return fn;
}


template <typename T>
static int launch_conv_nhwc_t(bool is_bf16, const void *x, const void *wk, int Cp, void *y, int y_nhwc, int N, int C, int H,
                              int W, int F, int R, int S, int OH, int OW, int ph, int pw, int sh, int sw, int dh, int dw,
                              const float *bn_mean, const float *bn_var, const float *bn_scale, const float *bn_bias,
                              float bn_eps, const void *residual, int relu, cudaStream_t st) {
    ConvNhwcParams p{};
    p.y = y;
    p.residual = residual;
    p.bn_mean = bn_mean;
    p.bn_var = bn_var;
    p.bn_scale = bn_scale;
    p.bn_bias = bn_bias;
    p.bn_eps = bn_eps;
    p.relu = relu;
    p.y_nhwc = y_nhwc;
    p.P = OH * OW;
    p.OW = OW;
    p.M = N * p.P;
    p.F = F;
    const int tiles_m = (p.M + CV_BM - 1) / CV_BM;
    p.cchunks = (C + CV_BK - 1) / CV_BK;
    p.FT = CV_FT;
    p.tiles_f = (F + p.FT - 1) / p.FT;
    p.tiles = tiles_m * p.tiles_f;
    p.Cp = Cp;
    p.RS = R * S;
    p.S = S;
    p.sh = sh;
    p.sw = sw;
    p.ph = ph;
    p.pw = pw;
    p.dh = dh;
    p.dw = dw;
    p.b_bytes = p.FT * CV_BK * 2;
    const int stage_bytes = CV_A_BYTES + p.b_bytes;
    const int stg_bytes = CV_EPI_WARPS * CV_RING * CV_SLAB_BYTES;  // 64 KB
    const int fixed = stg_bytes + p.FT * ACC_LD * 4 + p.FT * 8 + (16 * 2 + 2 + CV_EPI_WARPS * CV_RING) * 8 + 64 + 1024;
    // bytes in flight, not stage count, is what hides the L2 latency: 3 x 48 KB is as good as 4 (measured bound: L2 -> SM bandwidth)
    p.stages = std::max(2, std::min(6, (225 * 1024 - fixed) / stage_bytes));
    p.stg_off = p.stages * stage_bytes;
    const int smem = p.stages * stage_bytes + fixed;

    auto enc = get_im2col_fn();
    ITB_CHECK(enc, "conv(nhwc): cuTensorMapEncodeIm2col is not available from this driver");
    alignas(64) CUtensorMap mapA, mapB, mapY, mapR;
    {
        cuuint64_t gdim[4] = {(cuuint64_t)C, (cuuint64_t)W, (cuuint64_t)H, (cuuint64_t)N};
        cuuint64_t gstr[3] = {(cuuint64_t)C * 2, (cuuint64_t)W * C * 2, (cuuint64_t)H * W * C * 2};
        int lower[2] = {-pw, -ph};
        int upper[2] = {pw - (S - 1) * dw, ph - (R - 1) * dh};
        cuuint32_t estr[4] = {1, (cuuint32_t)sw, (cuuint32_t)sh, 1};
        CUresult r = enc(&mapA, is_bf16 ? CU_TENSOR_MAP_DATA_TYPE_BFLOAT16 : CU_TENSOR_MAP_DATA_TYPE_FLOAT16, 4,
                         const_cast<void *>(x), gdim, gstr, lower, upper, CV_BK, CV_BM, estr, CU_TENSOR_MAP_INTERLEAVE_NONE,
                         CU_TENSOR_MAP_SWIZZLE_128B, CU_TENSOR_MAP_L2_PROMOTION_L2_256B, CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
        ITB_CHECK(r == CUDA_SUCCESS, "conv(nhwc): cuTensorMapEncodeIm2col failed (%d) for N=%d H=%d W=%d C=%d R=%d S=%d", (int)r, N, H,
                  W, C, R, S);
    }
    // filters as a [F rows][R*S*Cp columns] K-major matrix; box [FT rows x 64 k]
    if (!make_tma_2d_b16(&mapB, wk, (uint64_t)F, (uint64_t)R * S * Cp, (uint64_t)R * S * Cp, (uint32_t)p.FT, CV_BK, 128))
        ITB_FAIL("conv(nhwc): cuTensorMapEncodeTiled(filters) failed");

    // y / residual as [N*OH*OW rows][F columns] matrices, box [32 pixels x 32 filters], 64B swizzle (NHWC output only)
    const void *ymat = y_nhwc ? y : wk, *rmat = (y_nhwc && residual) ? residual : ymat;
    const uint64_t yrows = y_nhwc ? (uint64_t)p.M : (uint64_t)F, ycols = y_nhwc ? (uint64_t)F : (uint64_t)R * S * Cp;
    if (!make_tma_2d_b16(&mapY, ymat, yrows, ycols, ycols, 32, 32, 64) || !make_tma_2d_b16(&mapR, rmat, yrows, ycols, ycols, 32, 32, 64))
        ITB_FAIL("conv(nhwc): cuTensorMapEncodeTiled(output) failed");

    return launch("conv(nhwc)", conv_nhwc_kernel<T, CV_FT>, {dim3(std::min(p.tiles, kNumSMs)), dim3(CV_THREADS), smem, st}, mapA,
                  mapB, mapY, mapR, p);
}

}  // namespace itb

using namespace itb;

static int nhwc_cp(int C, int R, int S) { return (R * S == 1) ? C : ((C + CV_BK - 1) / CV_BK) * CV_BK; }

extern "C" int it_b200_conv2d_nhwc_supported(int dtype, int C, int F, int R, int S, int ph, int pw, int sh, int sw, int dh,
                                             int dw, int groups) {
    return conv_nhwc_ok(dtype, C, F, R, S, ph, pw, sh, sw, dh, dw, groups) ? 1 : 0;
}

extern "C" int64_t it_b200_conv2d_nhwc_workspace(int dtype, int C, int F, int R, int S) {
    if (R * S == 1) return 0;  // [F][C] is already the K-major filter matrix
    return (int64_t)F * R * S * nhwc_cp(C, R, S) * dtype_size(dtype);
}

extern "C" int it_b200_conv2d_nhwc(int dtype, const void *x, const void *w, void *y, int y_nhwc, int N, int C, int H, int W,
                                   int F, int R, int S, int ph, int pw, int sh, int sw, int dh, int dw,
                                   const float *bn_mean, const float *bn_var, const float *bn_scale, const float *bn_bias,
                                   float bn_eps, const void *residual, int relu, void *workspace, int64_t workspace_bytes,
                                   void *stream) {
    ITB_CHECK(conv_nhwc_ok(dtype, C, F, R, S, ph, pw, sh, sw, dh, dw, 1),
              "conv(nhwc): shape outside the implicit-GEMM kernel (f16/bf16, C %% 8 == 0, F %% 8 == 0, stride <= 8): C=%d F=%d %dx%d", C,
              F, R, S);
    ITB_CHECK((bn_scale == nullptr) == (bn_mean == nullptr) && (bn_scale == nullptr) == (bn_var == nullptr) &&
                  (bn_scale == nullptr) == (bn_bias == nullptr),
              "conv(nhwc): the four BatchNorm parameter vectors go together");
    ITB_CHECK(aligned16(x) && aligned16(w) && aligned16(y) && (!residual || aligned16(residual)), "conv(nhwc): operands must be 16-byte aligned");
    auto st = (cudaStream_t)stream;
    const int OH = (H + 2 * ph - dh * (R - 1) - 1) / sh + 1, OW = (W + 2 * pw - dw * (S - 1) - 1) / sw + 1;
    if ((int64_t)N * F * OH * OW <= 0) return 0;
    ITB_CHECK((int64_t)N * OH * OW < (1ll << 31) - CV_BM, "conv(nhwc): too many output pixels");
    const int Cp = nhwc_cp(C, R, S);
    const void *wk = w;
    if (R * S > 1 && workspace_bytes < 0) {
        // filters already repacked by it_b200_conv_repack_filters (the runtime does that once per step for all convs)
        ITB_CHECK(workspace && -workspace_bytes >= it_b200_conv2d_nhwc_workspace(dtype, C, F, R, S) && aligned16(workspace),
                  "conv(nhwc): repacked filters too small");
        wk = workspace;
    } else if (R * S > 1) {
        const int64_t need = it_b200_conv2d_nhwc_workspace(dtype, C, F, R, S);
        ITB_CHECK(workspace && workspace_bytes >= need && aligned16(workspace), "conv(nhwc): workspace %lld < %lld bytes",
                  (long long)workspace_bytes, (long long)need);
        const int64_t total = (int64_t)F * R * S * Cp;
        const char *what = "conv(nhwc): filter repack";
        const int64_t items = R * S == 9 ? (int64_t)F * (Cp / 8) : total;
        const LaunchCfg c{dim3(grid_for(items, 256)), dim3(256), 0, st};
        int rc;
        if (R * S == 9)
            rc = dtype == ITB_F16 ? launch(what, repack_filters9_kernel<__half>, c, (const __half *)w, (__half *)workspace, items, C, Cp)
                                  : launch(what, repack_filters9_kernel<__nv_bfloat16>, c, (const __nv_bfloat16 *)w,
                                           (__nv_bfloat16 *)workspace, items, C, Cp);
        else
            rc = dtype == ITB_F16 ? launch(what, repack_filters_kernel<__half>, c, (const __half *)w, (__half *)workspace, total, C,
                                           R * S, Cp)
                                  : launch(what, repack_filters_kernel<__nv_bfloat16>, c, (const __nv_bfloat16 *)w,
                                           (__nv_bfloat16 *)workspace, total, C, R * S, Cp);
        if (rc) return 1;
        wk = workspace;
    }
    if (dtype == ITB_F16)
        return launch_conv_nhwc_t<__half>(false, x, wk, Cp, y, y_nhwc, N, C, H, W, F, R, S, OH, OW, ph, pw, sh, sw, dh, dw, bn_mean,
                                          bn_var, bn_scale, bn_bias, bn_eps, residual, relu, st);
    return launch_conv_nhwc_t<__nv_bfloat16>(true, x, wk, Cp, y, y_nhwc, N, C, H, W, F, R, S, OH, OW, ph, pw, sh, sw, dh, dw,
                                             bn_mean, bn_var, bn_scale, bn_bias, bn_eps, residual, relu, st);
}

extern "C" int it_b200_conv_repack_filters(int dtype, int n, const void *const *w, void *const *out, const int *F, const int *C,
                                           const int *R, const int *S, void *stream) {
    ITB_CHECK(dtype == ITB_F16 || dtype == ITB_BF16, "conv_repack_filters: f16 / bf16");
    auto st = (cudaStream_t)stream;
    for (int base = 0; base < n; base += CV_REPACK_BATCH) {
        const int cnt = std::min(CV_REPACK_BATCH, n - base);
        RepackBatch b{};
        int64_t most = 1;
        for (int i = 0; i < CV_REPACK_BATCH; ++i) {
            const int j = base + std::min(i, cnt - 1);  // unused slots repeat the last bank (never launched: gridDim.y = cnt)
            ITB_CHECK(C[j] % 8 == 0 && aligned16(w[j]) && aligned16(out[j]), "conv_repack_filters: bank %d: C %% 8 == 0, 16-byte aligned", j);
            b.src[i] = w[j];
            b.dst[i] = out[j];
            b.F[i] = F[j];
            b.C[i] = C[j];
            b.RS[i] = R[j] * S[j];
            b.Cp[i] = nhwc_cp(C[j], R[j], S[j]);
            most = std::max<int64_t>(most, (int64_t)F[j] * b.RS[i] * b.Cp[i] / (b.RS[i] == 9 ? 72 : 1));
        }
        const LaunchCfg c{dim3((unsigned)std::min<int64_t>((most + 255) / 256, 2 * kNumSMs), (unsigned)cnt), dim3(256), 0, st};
        const int rc = dtype == ITB_F16 ? launch("conv_repack_filters", repack_filters_batch_kernel<__half>, c, b)
                                        : launch("conv_repack_filters", repack_filters_batch_kernel<__nv_bfloat16>, c, b);
        if (rc) return 1;
    }
    return 0;
}
