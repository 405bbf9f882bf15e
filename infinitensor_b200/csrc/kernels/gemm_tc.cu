// gemm_tc.cu -- wgmma tensor-core GEMM for sm_90a:  C[M,N] = X[M,K] . W[K,N] (+bias, act)
//   X, W, C bf16 / fp16 row-major, fp32 accumulation in registers.
//
// The tensor core is driven "swap-AB": the streamed operand W (row-major [K,N], the layout ONNX MatMul weights and im2col
// matrices arrive in) is the wgmma A operand in MN-major form, 128 of its columns per CTA (two warpgroups x 64), and the
// <= 128-row operand X is the B operand (K-major), so
//     D[n (128 rows), m (NT columns)] += W^T[n, k16] . X^T[k16, m]
// runs as `wgmma.mma_async.m64nNTk16` per warpgroup and 16 k-values; M = 16 decode rows cost an N = 16 instruction instead of
// a padded 64-row tile.  Per CTA:
//   warp 8      : TMA producer -- cp.async.bulk.tensor, 128B swizzle, [64k x 64n] x2 weight boxes and one [NT x 64k]
//                 activation box per stage, mbarrier complete_tx
//   warps 0..7  : two consumer warpgroups -- wgmma over the stage ring (warpgroup h owns tile rows [64h, 64h + 64)), then the
//                 epilogue: the accumulator is parked in shared memory (the drained ring), optional split-K reduction over the
//                 thread-block CLUSTER through distributed shared memory, fused bias / activation / dtype conversion, stores
// Used for every MatMul with transA = 0, batch dense, N % 8 == 0, K % 8 == 0: the Llama decode GEMMs (M = 16, HBM-bound
// weight streaming, grid = N/128 x splitK clusters), GPT-2 (M = 128) and the im2col GEMMs of Conv (X = filter matrix
// [F, C*R*S], W = im2col matrix).
// Replaces the reference's cublasGemmEx dispatch (src/kernels/cuda/matmul.cc:141-168).
#include <cooperative_groups.h>

#include <type_traits>

#include "gemm.cuh"

namespace cg = cooperative_groups;

namespace itb {

constexpr int TC_BN = 128, TC_BK = 64;
constexpr int TC_W_BYTES = TC_BN * TC_BK * 2;  // 16 KB: two [64k x 64n] swizzled boxes
constexpr int TC_EPI_WARPS = 8;                      // two consumer warpgroups; in the epilogue two warps per 32-row quadrant
constexpr int TC_THREADS = (TC_EPI_WARPS + 1) * 32;  // + TMA producer warp
constexpr int TC_MAX_ROWS = 128;                     // rows of X per CTA (wgmma N): 16, 32, 64 or 128
constexpr int TC_SPLITK_MIN_KTILES = 24;             // k-tiles from which a GEMM on few CTAs is split over a cluster

// 16 consecutive values -> two 16-byte stores (registers only: an address-taken T[16] costs a stack frame and 26 registers,
// which halves the CTAs per SM of this kernel)
template <typename T> __device__ __forceinline__ uint32_t tc_pack2(float a, float b);
template <> __device__ __forceinline__ uint32_t tc_pack2<__half>(float a, float b) {
    const __half2 h = __floats2half2_rn(a, b);
    return *reinterpret_cast<const uint32_t *>(&h);
}
template <> __device__ __forceinline__ uint32_t tc_pack2<__nv_bfloat16>(float a, float b) {
    const __nv_bfloat162 h = __floats2bfloat162_rn(a, b);
    return *reinterpret_cast<const uint32_t *>(&h);
}
template <typename T> __device__ __forceinline__ void tc_store16(T *dst, const float (&f)[16]) {
    uint4 lo, hi;
    lo.x = tc_pack2<T>(f[0], f[1]);
    lo.y = tc_pack2<T>(f[2], f[3]);
    lo.z = tc_pack2<T>(f[4], f[5]);
    lo.w = tc_pack2<T>(f[6], f[7]);
    hi.x = tc_pack2<T>(f[8], f[9]);
    hi.y = tc_pack2<T>(f[10], f[11]);
    hi.z = tc_pack2<T>(f[12], f[13]);
    hi.w = tc_pack2<T>(f[14], f[15]);
    reinterpret_cast<uint4 *>(dst)[0] = lo;
    reinterpret_cast<uint4 *>(dst)[1] = hi;
}

struct TcParams {
    int mpad;        // wgmma N: rows of X rounded up to a power of two (16..128)
    int stages;
    int ring_bytes;  // stages x stage bytes, at least the parked accumulator tile
    int x_bytes;     // mpad * 128
    int red_bytes;   // split-K partial tile: mpad * 128 * 4 (0 when splitk == 1)
    int ktiles, ktiles_per_split;
    int m_chunks;    // ceil(M / mpad): grid.z = batch * m_chunks
    int a_batched;   // X has a batch dimension (stride_a != 0); otherwise it is broadcast over the batch
    int b_batched;   // same for W
    int w_kmajor;    // trans_b: W is stored [N, K] (ONNX Gemm transB): one [128 n x 64 k] K-major box per stage
};

// up to 4 weight matrices sharing the activation operand X (q/k/v, gate/up) in ONE launch: the column-tile index selects the
// group (its tensor map, output pointer and width); a plain MatMul is the 1-group case
constexpr int TC_MAX_GROUPS = 4;
struct TcGroups {
    CUtensorMap mapW[TC_MAX_GROUPS];
    void *C[TC_MAX_GROUPS];
    int n[TC_MAX_GROUPS];
    int tile_start[TC_MAX_GROUPS + 1];
    int ngroups;
};

template <typename T, int NT>
__global__ void __launch_bounds__(TC_THREADS, 2) gemm_tc_kernel(const __grid_constant__ TcGroups grp,
                                                             const __grid_constant__ CUtensorMap mapX, GemmArgs g,
                                                             TcParams p) {
    extern __shared__ uint8_t smem_raw[];
    uint8_t *smem = smem_raw + ((1024u - (smem_u32(smem_raw) & 1023u)) & 1023u);
    const int S = p.stages;
    uint8_t *w_sm = smem;
    uint8_t *x_sm = smem + S * TC_W_BYTES;
    float *acc_sm = reinterpret_cast<float *>(smem);  // the parked accumulator, once the ring is drained
    float *red = reinterpret_cast<float *>(smem + p.ring_bytes);
    uint64_t *full = reinterpret_cast<uint64_t *>(reinterpret_cast<uint8_t *>(red) + p.red_bytes);
    uint64_t *empty = full + S;
    float *bn_sm = reinterpret_cast<float *>(empty + S + 2);  // float4[mpad]: {mean, rs, scale, bias} of this row chunk (16-B aligned)

    cg::cluster_group cluster = cg::this_cluster();
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    int gi = 0;
    while (gi + 1 < grp.ngroups && (int)blockIdx.x >= grp.tile_start[gi + 1]) ++gi;
    const CUtensorMap *mapWp = &grp.mapW[gi];
    const int n0 = ((int)blockIdx.x - grp.tile_start[gi]) * TC_BN;
    const int Ng = grp.n[gi];  // columns of this group's weight matrix / output
    const int bz = (int)blockIdx.z / p.m_chunks;                  // batch index
    const int m0 = ((int)blockIdx.z % p.m_chunks) * p.mpad;      // first row of this CTA's row chunk
    const int bx = p.a_batched ? bz : 0, bw = p.b_batched ? bz : 0;
    const int split = blockIdx.y, nsplit = gridDim.y;
    const int kt_begin = split * p.ktiles_per_split;
    const int kt_end = min(p.ktiles, kt_begin + p.ktiles_per_split);
    const int my_kt = max(0, kt_end - kt_begin);

    pdl_trigger();
    if (threadIdx.x == 0) {
        for (int s = 0; s < S; ++s) {
            mbar_init(&full[s], 1);
            mbar_init(&empty[s], 2);  // one arrival per consumer warpgroup
        }
        fence_mbar_init();
    }
    if (warp == TC_EPI_WARPS && lane == 0) {
        tma_prefetch_desc(mapWp);
        tma_prefetch_desc(&mapX);
    }
    __syncthreads();

    if (warp == TC_EPI_WARPS) {
        // ===== TMA producer (one thread; running ring slot / phase instead of it % S, it / S: a lone thread retires a dependent
        // instruction every ~5 cycles, and two runtime divisions per k-tile made this loop the pace-setter of M = 128 GEMMs) =====
        if (lane == 0) {
            const uint64_t pol_w = l2_policy_evict_first();
            const uint64_t pol_x = l2_policy_evict_last();
            // PDL: weight tiles of the first ring are requested before waiting for the predecessor kernel
            const int pre = min(S, my_kt);
            if (!(g.act & ITB_MATMUL_B_CONST)) pdl_wait();  // B produced upstream: no early prefetch
            const uint32_t tx = TC_W_BYTES + p.x_bytes;
            int k0 = kt_begin * TC_BK;
            for (int it = 0; it < pre; ++it, k0 += TC_BK) {
                mbar_expect_tx(&full[it], tx);
                if (p.w_kmajor) {
                    tma_load_3d(w_sm + it * TC_W_BYTES, mapWp, &full[it], k0, n0, bw, pol_w);
                } else {
                    tma_load_3d(w_sm + it * TC_W_BYTES, mapWp, &full[it], n0, k0, bw, pol_w);
                    tma_load_3d(w_sm + it * TC_W_BYTES + TC_W_BYTES / 2, mapWp, &full[it], n0 + 64, k0, bw, pol_w);
                }
            }
            pdl_wait();
            k0 = kt_begin * TC_BK;
            for (int it = 0; it < pre; ++it, k0 += TC_BK) tma_load_3d(x_sm + it * p.x_bytes, &mapX, &full[it], k0, m0, bx, pol_x);
            int s = 0;            // pre == S whenever the loop below runs
            uint32_t ph = 0;      // parity of the `empty` phase to wait for: flips each time the ring wraps
            for (int it = pre; it < my_kt; ++it, k0 += TC_BK) {
                mbar_wait(&empty[s], ph);
                mbar_expect_tx(&full[s], tx);
                uint8_t *wdst = w_sm + s * TC_W_BYTES;
                if (p.w_kmajor) {
                    tma_load_3d(wdst, mapWp, &full[s], k0, n0, bw, pol_w);
                } else {
                    tma_load_3d(wdst, mapWp, &full[s], n0, k0, bw, pol_w);
                    tma_load_3d(wdst + TC_W_BYTES / 2, mapWp, &full[s], n0 + 64, k0, bw, pol_w);
                }
                tma_load_3d(x_sm + s * p.x_bytes, &mapX, &full[s], k0, m0, bx, pol_x);
                if (++s == S) {
                    s = 0;
                    ph ^= 1;
                }
            }
        }
        __syncwarp();
    } else {
        // ===== consumers: warpgroup h multiplies tile rows [64h, 64h + 64) (weight columns n0 + 64h ..) =====
        // A = W tile, MN-major: the [64k x 64n] box of this warpgroup, 8-row k groups 1 KB apart (SBO); one k16 step = 16 rows x
        //     128 B = 2 KB  (trans_b: the tile is [128 n rows x 128 B of k], K-major like X: rows 64h.. start 8 KB in, k16 = +32 B)
        // B = X tile, K-major: 8-row groups 1 KB apart (SBO); one k16 step = 32 B inside the 128 B row
        const int h = warp >> 2;
        const uint64_t a_desc0 = gmma_desc_sw128(smem_u32(w_sm) + h * (TC_W_BYTES / 2), TC_W_BYTES / 2, 1024);
        const uint64_t b_desc0 = gmma_desc_sw128(smem_u32(x_sm), 0, 1024);
        const uint32_t a_kk = p.w_kmajor ? 2u : 128u, a_st = TC_W_BYTES >> 4, b_st = (uint32_t)p.x_bytes >> 4;
        float d[NT / 2];
#pragma unroll
        for (int j = 0; j < NT / 2; ++j) d[j] = 0.f;
        // (the operand major-ness is an immediate of the instruction: one loop per form, no branch between the MMAs)
        auto mainloop = [&](auto ta) {
            int s = 0, prev = -1;
            uint32_t ph = 0;
            for (int it = 0; it < my_kt; ++it) {
                mbar_wait(&full[s], ph);
                const uint64_t a_desc = a_desc0 + (uint64_t)(s * a_st), b_desc = b_desc0 + (uint64_t)(s * b_st);
                wg_fence();
#pragma unroll
                for (int kk = 0; kk < TC_BK / 16; ++kk)
                    Wgmma<T, NT>::template mma<decltype(ta)::value, 0>(d, a_desc + (uint64_t)(kk * a_kk), b_desc + 2 * kk, 1u);
                wg_commit();
                wg_wait<1>();  // the previous stage's MMAs are done: it may be refilled
                if (prev >= 0 && (threadIdx.x & 127) == 0) mbar_arrive(&empty[prev]);
                prev = s;
                if (++s == S) {
                    s = 0;
                    ph ^= 1;
                }
            }
        };
        if (p.w_kmajor) mainloop(std::integral_constant<int, 0>{});
        else mainloop(std::integral_constant<int, 1>{});
        wg_wait<0>();
        named_bar_sync(1, TC_EPI_WARPS * 32);  // both warpgroups are done with the ring: it holds the accumulator from here on
        acc_park<NT>(d, acc_sm, 64 * h);
        named_bar_sync(1, TC_EPI_WARPS * 32);
    }

    // ===== epilogue: warps w and w + 4 own accumulator rows [32 (w & 3), +32) = output columns n0 + 32 (w & 3) + lane =====
    const T *bias = g.bias ? (const T *)g.bias + (int64_t)bz * g.bias_sb : nullptr;
    T *C = (T *)grp.C[gi] + (int64_t)bz * g.m * Ng;
    const bool tail = g.bn_scale != nullptr || g.residual != nullptr || g.post_relu;
    if (warp < TC_EPI_WARPS) {
        pdl_wait();
        if (g.bn_scale) {
            float4 *bn4 = reinterpret_cast<float4 *>(bn_sm);  // {mean, rs, scale, bias} of row r
            for (int r = threadIdx.x; r < p.mpad; r += TC_EPI_WARPS * 32) {
                const int m = min(m0 + r, g.m - 1);
                bn4[r] = make_float4(g.bn_mean[m], bn_rs(g.bn_var[m], g.bn_eps), g.bn_scale[m], g.bn_bias[m]);
            }
            asm volatile("bar.sync 1, %0;" ::"n"(TC_EPI_WARPS * 32) : "memory");
        }
        // warp w reads accumulator rows [32 (w & 3), +32) = output columns n0 + 32 (w & 3) + lane; warps 0-3 take the first half
        // of the 16-row groups of X (accumulator columns), warps 4-7 the second
        const int quad = warp & 3;
        const int groups16 = p.mpad / 16, g_split = (groups16 + 1) / 2;
        const int c_begin = (warp < 4 ? 0 : g_split) * 16, c_end = (warp < 4 ? g_split : groups16) * 16;
        const int nl = quad * 32 + lane;  // column inside the tile
        const int gn = n0 + nl;
        // element (m, gn) lives at C[c_off + m * c_ld] (plain row-major, or the conv scatter of GemmArgs::c_block)
        const int64_t c_ld = g.c_nhwc ? 1 : g.c_block ? g.c_block : Ng;
        const int64_t c_off = g.c_nhwc ? (int64_t)gn * g.m
                              : g.c_block ? (int64_t)(gn / g.c_block) * g.c_block_stride + gn % g.c_block : gn;
        // (a BatchNorm / ReLU tail excludes bias / act; a residual alone may follow them: MatMul + bias -> [act] -> + residual)
        const int mode = (bias || (g.act & 0xff)) ? 2 : tail ? 1 : 0;
        const float bias_col = (bias && g.bias_sm == 0 && gn < Ng) ? to_f(bias[(int64_t)gn * g.bias_sn]) : 0.f;
        for (int c0 = c_begin; c0 < c_end; c0 += 16) {
            uint32_t v[16];
            acc_row<16>(acc_sm, nl, c0, v);
            if (nsplit > 1) {
#pragma unroll
                for (int j = 0; j < 16; ++j) red[(c0 + j) * TC_BN + nl] = __uint_as_float(v[j]);
            } else if (gn < Ng) {
                // three specialisations of the per-element tail, chosen by CTA-uniform flags, so the common cases do
                // not carry the generic bias / activation code (that alone made the epilogue instruction-bound)
                const int rows = min(16, g.m - (m0 + c0));  // valid rows of this 16-row group
                T *cp = C + c_off + (int64_t)(m0 + c0) * c_ld;
                if (mode == 0) {
                    if (g.c_nhwc && rows == 16) {  // 16 consecutive filters of one pixel: two 16-byte stores
                        float fv[16];
#pragma unroll
                        for (int j = 0; j < 16; ++j) fv[j] = __uint_as_float(v[j]);
                        tc_store16<T>(cp, fv);
                    } else {
#pragma unroll
                        for (int j = 0; j < 16; ++j)
                            if (j < rows) cp[(int64_t)j * c_ld] = from_f<T>(__uint_as_float(v[j]));
                    }
                } else if (mode == 1) {
                    float resv[16];
                    if (g.residual) {  // all 16 residual loads in flight before the first (possibly aliasing) store
                        const T *rp = (const T *)g.residual + (int64_t)bz * g.m * Ng + c_off + (int64_t)(m0 + c0) * c_ld;
#pragma unroll
                        for (int j = 0; j < 16; ++j) resv[j] = j < rows ? to_f(rp[(int64_t)j * c_ld]) : 0.f;
                    }
#pragma unroll
                    for (int j = 0; j < 16; ++j) {
                        const int r = c0 + j;
                        float f = round_t<T>(__uint_as_float(v[j]));  // the Conv output as the separate kernel stores it
                        if (g.bn_scale) {
                            const float4 bp = reinterpret_cast<const float4 *>(bn_sm)[r];
                            f = round_t<T>(bn_apply(f, bp.x, bp.y, bp.z, bp.w));
                        }
                        if (g.residual) f = round_t<T>(f + resv[j]);
                        if (g.post_relu) f = fmaxf(f, 0.f);
                        resv[j] = f;
                    }
                    if (g.c_nhwc && rows == 16) {
                        tc_store16<T>(cp, resv);
                    } else {
#pragma unroll
                        for (int j = 0; j < 16; ++j)
                            if (j < rows) cp[(int64_t)j * c_ld] = from_f<T>(resv[j]);
                    }
                } else {
                    // bias / activation: the bias of a Gemm is a row vector (bias_sm == 0) -> ONE value per thread (its column), and
                    // the activation switch is taken once per 16 rows, not per element (the per-element form costs
                    // ~115 instructions per stored value)
                    const bool rb = (g.act & ITB_ACT_ROUND_BEFORE_BIAS) != 0;
                    if (bias) {
                        const bool row_const = g.bias_sm == 0;
                        const T *bp = bias + (int64_t)(m0 + c0) * g.bias_sm + (int64_t)gn * g.bias_sn;
#pragma unroll
                        for (int j = 0; j < 16; ++j) {
                            float f = __uint_as_float(v[j]);
                            if (rb) f = round_t<T>(f);
                            f += row_const ? bias_col : (j < rows ? to_f(bp[(int64_t)j * g.bias_sm]) : 0.f);
                            v[j] = __float_as_uint(f);
                        }
                    }
                    switch (g.act & 0xff) {
                    case 1:
#pragma unroll
                        for (int j = 0; j < 16; ++j) v[j] = __float_as_uint(__uint_as_float(v[j]) > 0.f ? __uint_as_float(v[j]) : 0.f);
                        break;
                    case 2:
#pragma unroll
                        for (int j = 0; j < 16; ++j) v[j] = __float_as_uint(1.f / (1.f + expf(-__uint_as_float(v[j]))));
                        break;
                    case 3:
#pragma unroll
                        for (int j = 0; j < 16; ++j) v[j] = __float_as_uint(tanhf(__uint_as_float(v[j])));
                        break;
                    case 4:  // Gelu (erf form, the unary kernel's formula) of the MatMul's ROUNDED output: MatMul -> Gelu in one epilogue
#pragma unroll
                        for (int j = 0; j < 16; ++j) {
                            const float x = round_t<T>(__uint_as_float(v[j]));
                            v[j] = __float_as_uint(0.5f * x * (1.f + erff(x * 0.70710678118654752440f)));
                        }
                        break;
                    }
                    if (g.residual) {  // -> Add(residual): the operator before it rounds first
                        const T *rp = (const T *)g.residual + (int64_t)bz * g.m * Ng + c_off + (int64_t)(m0 + c0) * c_ld;
#pragma unroll
                        for (int j = 0; j < 16; ++j)
                            v[j] = __float_as_uint(round_t<T>(__uint_as_float(v[j])) + (j < rows ? to_f(rp[(int64_t)j * c_ld]) : 0.f));
                    }
#pragma unroll
                    for (int j = 0; j < 16; ++j)
                        if (j < rows) cp[(int64_t)j * c_ld] = from_f<T>(__uint_as_float(v[j]));
                }
            }
        }
    }
    if (nsplit > 1) {
        cluster.sync();
        if (warp < TC_EPI_WARPS) {
            // reduce-scatter over distributed shared memory: rank r finishes rows [r, r + 1) * mpad / nsplit of the tile -- every CTA
            // of the cluster reads 1 / nsplit of each peer's partial (the first version had rank 0 read all of it: 8 x 64 KB at
            // M = 128, slower than the serial k walk it replaced); partials are summed in rank order -> deterministic
            const float *peers[8];
            for (int r = 0; r < nsplit; ++r) peers[r] = (const float *)cluster.map_shared_rank(red, r);
            const int rows_per = (p.mpad + nsplit - 1) / nsplit;
            const int r_begin = split * rows_per, r_end = min(p.mpad, r_begin + rows_per);
            const bool rb = (g.act & ITB_ACT_ROUND_BEFORE_BIAS) != 0;
            const int act = g.act & 0xff;
            const T *resid = g.residual ? (const T *)g.residual + (int64_t)bz * g.m * Ng : nullptr;
            for (int idx = r_begin * TC_BN + (int)threadIdx.x; idx < r_end * TC_BN; idx += TC_EPI_WARPS * 32) {
                const int m = m0 + idx / TC_BN, nl = idx % TC_BN, gn = n0 + nl;
                if (m >= g.m || gn >= Ng) continue;
                float f = 0.f;
                for (int r = 0; r < nsplit; ++r) f += peers[r][idx];
                if (bias) {
                    if (rb) f = round_t<T>(f);
                    f += to_f(bias[m * g.bias_sm + gn * g.bias_sn]);
                }
                if (act == 4) {
                    const float x = round_t<T>(f);
                    f = 0.5f * x * (1.f + erff(x * 0.70710678118654752440f));
                } else {
                    f = gemm_act(act, f);
                }
                const int64_t off = g.c_block ? (int64_t)(gn / g.c_block) * g.c_block_stride + (int64_t)m * g.c_block + gn % g.c_block
                                              : (int64_t)m * Ng + gn;
                if (resid) f = round_t<T>(f) + to_f(resid[off]);
                C[off] = from_f<T>(f);
            }
        }
        cluster.sync();
    } else {
        __syncthreads();
    }
}

template <typename T>
static int launch_tc_t(const GemmArgs &g, cudaStream_t st, bool is_bf16, int ngroups = 1, const void *const *Ws = nullptr,
                       void *const *Cs = nullptr, const int *Ns = nullptr) {
    TcParams p{};
    p.mpad = 16;
    while (p.mpad < g.m && p.mpad < TC_MAX_ROWS) p.mpad <<= 1;
    p.m_chunks = (g.m + p.mpad - 1) / p.mpad;
    p.a_batched = g.batch > 1 && g.stride_a != 0;
    p.b_batched = g.batch > 1 && g.stride_b != 0;
    p.x_bytes = p.mpad * 128;
    TcGroups grp{};
    grp.ngroups = ngroups;
    int tiles_n = 0;
    for (int i = 0; i < ngroups; ++i) {
        grp.C[i] = Cs ? Cs[i] : g.C;
        grp.n[i] = Ns ? Ns[i] : g.n;
        grp.tile_start[i] = tiles_n;
        tiles_n += (grp.n[i] + TC_BN - 1) / TC_BN;
    }
    for (int i = ngroups; i <= TC_MAX_GROUPS; ++i) grp.tile_start[i] = tiles_n;
    p.ktiles = (g.k + TC_BK - 1) / TC_BK;
    // split-K only where the partial tile is small (decode regime); clusters of <= 8 CTAs
    int splitk = 1;
    // the fused conv tail lives in the direct epilogue only (a residual after bias / activation is handled by the reduction too)
    const bool tail = g.bn_scale || g.post_relu || (g.residual && !(g.bias || (g.act & 0xff)));
    // (a split M = 128 tile reduced by rank 0 alone would pull 8 x 64 KB through one CTA's DSMEM reads; the reduce-scatter form
    //  below reads 1/8 of that per CTA)
    if (p.mpad <= 64 && g.batch == 1 && !tail && !g.no_splitk) {
        splitk = (2 * kNumSMs) / tiles_n;
        splitk = std::max(1, std::min(splitk, 8));
        splitk = std::min(splitk, std::max(1, p.ktiles / 4));
    } else if (p.mpad <= 128 && g.batch == 1 && !tail && !g.c_block && !g.c_nhwc && p.ktiles >= TC_SPLITK_MIN_KTILES &&
               tiles_n * p.m_chunks * 4 <= kNumSMs) {
        // a long serial k walk on a handful of CTAs (GPT-2's mlp c_proj: 48 k-tiles on 6 CTAs): split it over a cluster, >= 6 k-tiles each
        // (shorter walks -- the K = 768 projections -- stay unsplit: two cluster syncs and the DSMEM exchange cost about as much as the
        //  k-tiles they save)
        splitk = std::min(8, std::min(p.ktiles / 6, kNumSMs / (tiles_n * p.m_chunks)));
        splitk = std::max(1, splitk);
    }
    p.ktiles_per_split = (p.ktiles + splitk - 1) / splitk;
    splitk = (p.ktiles + p.ktiles_per_split - 1) / p.ktiles_per_split;
    p.red_bytes = splitk > 1 ? p.mpad * TC_BN * 4 : 0;
    const int stage_bytes = TC_W_BYTES + p.x_bytes;
    // a grid that cannot fill the SMs anyway (GPT-2's 6..24-tile projections) takes the whole shared memory for a deep ring:
    // one CTA per SM walking K serially is bound by bytes in flight / latency, so more stages help
    const bool small_grid = (int64_t)tiles_n * splitk * g.batch * p.m_chunks <= kNumSMs;
    // two CTAs per SM (<= 113 KB each): one CTA's epilogue overlaps the other's main loop
    const int budget = (p.mpad <= 64 ? 104 : small_grid ? 200 : 110) * 1024;
    p.stages = std::max(2, std::min(8, (budget - p.red_bytes - 2048 - 16 * p.mpad) / stage_bytes));
    p.w_kmajor = g.trans_b ? 1 : 0;
    p.ring_bytes = std::max(p.stages * stage_bytes, p.mpad * ACC_LD * 4);
    const int smem = p.ring_bytes + p.red_bytes + (2 * p.stages + 2) * 8 + 4 * p.mpad * 4 + 1024;

    CUtensorMap mapX;
    for (int i = 0; i < ngroups; ++i) {
        const void *Wi = Ws ? Ws[i] : g.B;
        const uint64_t ni = (uint64_t)grp.n[i];
        const bool w_ok = p.w_kmajor
                              ? make_tma_3d_b16(&grp.mapW[i], Wi, p.b_batched ? (uint64_t)g.batch : 1, ni, (uint64_t)g.k, (uint64_t)g.k,
                                                (uint64_t)g.stride_b, TC_BN, TC_BK)
                              : make_tma_3d_b16(&grp.mapW[i], Wi, p.b_batched ? (uint64_t)g.batch : 1, (uint64_t)g.k, ni, ni,
                                                (uint64_t)g.stride_b, TC_BK, 64);
        if (!w_ok) ITB_FAIL("matmul(wgmma): cuTensorMapEncodeTiled(W) failed");
    }
    for (int i = ngroups; i < TC_MAX_GROUPS; ++i) grp.mapW[i] = grp.mapW[0];
    if (!make_tma_3d_b16(&mapX, g.A, p.a_batched ? (uint64_t)g.batch : 1, (uint64_t)g.m, (uint64_t)g.k, (uint64_t)g.k,
                         (uint64_t)g.stride_a, (uint32_t)p.mpad, TC_BK))
        ITB_FAIL("matmul(wgmma): cuTensorMapEncodeTiled(X) failed");

    auto kern = p.mpad == 16 ? gemm_tc_kernel<T, 16> : p.mpad == 32 ? gemm_tc_kernel<T, 32> : p.mpad == 64 ? gemm_tc_kernel<T, 64>
                                                                                                : gemm_tc_kernel<T, 128>;
    return launch("matmul(wgmma)", kern,
                  {dim3(tiles_n, splitk, (unsigned)(g.batch * p.m_chunks)), dim3(TC_THREADS, 1, 1), smem, st, dim3(1, splitk, 1)},
                  grp, mapX, g, p);
}

int launch_gemm_tc(int dtype, const GemmArgs &g, cudaStream_t st) {
    if (dtype != ITB_BF16 && dtype != ITB_F16) return -1;
    if (g.batch < 1 || g.trans_a || g.m < 1) return -1;
    if (g.n % 8 != 0 || g.k % 8 != 0 || g.n < 64 || g.k < 64) return -1;
    if (!aligned16(g.A) || !aligned16(g.B)) return -1;
    if (g.batch > 1) {
        // batches must be dense [b][K][N] / [b][M][K] (or X broadcast): that is what the 3-D tensor maps describe
        if (g.stride_b != 0 && g.stride_b != (int64_t)g.k * g.n) return -1;
        if (g.stride_a != 0 && g.stride_a != (int64_t)g.m * g.k) return -1;
        if ((int64_t)g.batch * ((g.m + TC_MAX_ROWS - 1) / TC_MAX_ROWS) > 65535) return -1;
    }
    if ((g.bn_scale || g.post_relu) && (g.bias || (g.act & 0xff))) return -1;  // the conv tail excludes bias / act
    if (g.residual && (g.bias || (g.act & 0xff)) && (g.c_block || g.c_nhwc)) return -1;
    if (g.c_nhwc && (g.batch != 1 || g.m % 8 != 0 || g.bias || (g.act & 0xff) || !g.no_splitk)) return -1;
    if (dtype == ITB_BF16) return launch_tc_t<__nv_bfloat16>(g, st, true);
    return launch_tc_t<__half>(g, st, false);
}

// 2..4 weight matrices [K, N_i] sharing X (decode rows): one launch when 128-wide tiles alone fill the machine (no split-K).
// -1 = not taken (the mma.sync kernel's cluster split-K is the better shape then)
int launch_gemm_tc_grouped(int dtype, const GemmArgs &g0, int ngroups, const void *const *Ws, void *const *Cs, const int *Ns,
                           cudaStream_t st) {
    if (dtype != ITB_BF16 && dtype != ITB_F16) return -1;
    if (ngroups < 1 || ngroups > TC_MAX_GROUPS) return -1;
    if (g0.batch != 1 || g0.trans_a || g0.trans_b || g0.m < 1 || g0.m > 64 || g0.bias || (g0.act & 0xff) || g0.residual || g0.bn_scale ||
        g0.post_relu || g0.c_block || g0.c_nhwc)
        return -1;
    if (g0.k % 8 != 0 || g0.k < 64 || !aligned16(g0.A)) return -1;
    int tiles = 0;
    for (int i = 0; i < ngroups; ++i) {
        if (Ns[i] % 8 != 0 || Ns[i] < 64 || !aligned16(Ws[i]) || !aligned16(Cs[i])) return -1;
        tiles += (Ns[i] + TC_BN - 1) / TC_BN;
    }
    if (tiles < TC_MIN_TILES_DECODE) return -1;
    GemmArgs g = g0;
    g.B = Ws[0];
    g.C = Cs[0];
    g.n = Ns[0];
    g.act |= ITB_MATMUL_B_CONST;
    g.no_splitk = 1;
    if (dtype == ITB_BF16) return launch_tc_t<__nv_bfloat16>(g, st, true, ngroups, Ws, Cs, Ns);
    return launch_tc_t<__half>(g, st, false, ngroups, Ws, Cs, Ns);
}

}  // namespace itb
