// gemm_w4.cu -- 4-bit weight-only MatMul (com.microsoft MatMulNBits, bits = 4) for sm_90a.
//
//   Y[m, n] = sum_k X[m, k] . (q[n, k] - z[n, k / bs]) . s[n, k / bs]        X, Y, s: f16 / bf16
//
// B (the codes) is N-major: column n's K nibbles are K / 2 contiguous bytes, element k in byte k / 2, even k in the low nibble.
// The layout of every operand is documented with it_b200_matmul_nbits in include/it_b200.h.
//
// M <= 64: gemm_skinny_w4_kernel, the decode GEMM.  It keeps gemm_skinny_kernel's architecture -- one TMA producer lane filling
// an mbarrier ring, four mma.sync m16n8k16 consumer warps, 1..4 weight matrices sharing X in one launch, split-K over a cluster
// reduced through distributed shared memory, the residual epilogue, weight tiles requested ahead of griddepcontrol.wait, PDL:
//   * a stage carries a [64 n x 256 k] box of codes: 64 rows of 128 bytes (8 KB, the 16-bit kernel's box size), 128B swizzle,
//     and the matching four [16 MT x 64 k] boxes of X;
//   * lane (g, t) of a warp reads one 32-bit word per column and k32 chunk: the 8 nibbles k = 8t .. 8t + 7 of column g.  They
//     widen to exact (q - z) pairs (k, k + 4) in T with the magic-number LOP3 + subtract, giving the B fragments of two
//     m16n8k16 steps.  The k order inside a step is free, so X's A fragments are read in the same permuted order (PRMT of one
//     16-byte row read), as attn_gqa_kv8_kernel does for Q and K;
//   * every MMA step lies inside one quantisation block: the block's fp32 partial sum is multiplied by fp32(s) and added to the
//     fp32 accumulator (one FMA) at each block boundary, so the weight value (q - z) . s is never rounded;
//   * the output is rounded to T once; a residual is added after that rounding, as MatMul -> Add does.
// M > 64 (prompt steps): dequant_w4_kernel writes T((q - z) . s) as a [K, N] row-major matrix into the workspace and the 16-bit
// it_b200_matmul runs on it.  The weights are rounded to T once there, so that path's numerics differ from the decode kernel's.
#include <cooperative_groups.h>

#include "gemm.cuh"

namespace cg = cooperative_groups;

namespace itb {

constexpr int W4_BN = 64;                      // output columns per CTA
constexpr int W4_BK = 256;                     // k per stage
constexpr int W4_W_BYTES = W4_BN * W4_BK / 2;  // 8 KB of codes per stage
constexpr int W4_THREADS = 160;                // 4 consumer warps + 1 producer warp
constexpr int W4_MAX_GROUPS = 4;

template <int MT> struct W4Cfg {
    static constexpr int X_BOX_BYTES = MT * 16 * 64 * 2;  // one [16 MT x 64 k] box of X
    static constexpr int X_BYTES = 4 * X_BOX_BYTES;
    static constexpr int RED_BYTES = MT * 16 * W4_BN * 4;
    static constexpr int stages_for(int budget_kb) {
        int s = (budget_kb * 1024 - RED_BYTES - 1024 - 256) / (W4_W_BYTES + X_BYTES);
        return s < 2 ? 2 : (s > 16 ? 16 : s);
    }
    static constexpr int smem_for(int stages) { return stages * (W4_W_BYTES + X_BYTES) + RED_BYTES + 2 * stages * 8 + 1024; }
};
// unsplit launches: two CTAs per SM; split-K clusters: three
constexpr int kW4DeepBudgetKB = 110, kW4SplitBudgetKB = 72;
static_assert(3 * (W4Cfg<1>::smem_for(W4Cfg<1>::stages_for(kW4SplitBudgetKB)) + 1024) <= 228 * 1024, "w4: three split CTAs per SM");

struct W4Groups {
    CUtensorMap mapW[W4_MAX_GROUPS];
    void *C[W4_MAX_GROUPS];
    const void *scale[W4_MAX_GROUPS];
    const uint8_t *zp[W4_MAX_GROUPS];
    int n[W4_MAX_GROUPS];
    int tile_start[W4_MAX_GROUPS + 1];
    int ngroups;
};

__device__ __forceinline__ uint32_t lop3_and_or(uint32_t a, uint32_t b, uint32_t c) {  // (a & b) | c
    uint32_t r;
    asm("lop3.b32 %0, %1, %2, %3, 0xEA;" : "=r"(r) : "r"(a), "r"(b), "r"(c));
    return r;
}
__device__ __forceinline__ uint32_t prmt(uint32_t a, uint32_t b, uint32_t sel) {
    uint32_t r;
    asm("prmt.b32 %0, %1, %2, %3;" : "=r"(r) : "r"(a), "r"(b), "r"(sel));
    return r;
}

// 8 nibbles of one column (k = 0..7 at bits 4k) -> four pairs of exact (q - z) in T: o[0] = (k0, k4), o[1] = (k1, k5),
// o[2] = (k2, k6), o[3] = (k3, k7), the first element of each pair in the low half.
template <typename T> struct W4Widen;
template <> struct W4Widen<__half> {
    // OR-ing a nibble into the mantissa of 1024.0 (0x6400) gives 1024 + q exactly; a nibble 4 bits higher gives 1024 + 16 q
    struct Z {
        __half2 sub, fma_c;
    };
    static __device__ __forceinline__ Z zero(int z) {
        return {__half2half2(__int2half_rn(1024 + z)), __half2half2(__int2half_rn(-(64 + z)))};
    }
    static __device__ __forceinline__ void run(uint32_t w, const Z &z, uint32_t (&o)[4]) {
        const uint32_t M = 0x64006400u;
        const __half2 sixteenth = __half2half2(__float2half_rn(0.0625f));
        const uint32_t p04 = lop3_and_or(w, 0x000F000Fu, M), p15 = lop3_and_or(w, 0x00F000F0u, M);
        const uint32_t w8 = w >> 8;
        const uint32_t p26 = lop3_and_or(w8, 0x000F000Fu, M), p37 = lop3_and_or(w8, 0x00F000F0u, M);
        __half2 r0 = __hsub2(*reinterpret_cast<const __half2 *>(&p04), z.sub);
        __half2 r1 = __hfma2(*reinterpret_cast<const __half2 *>(&p15), sixteenth, z.fma_c);
        __half2 r2 = __hsub2(*reinterpret_cast<const __half2 *>(&p26), z.sub);
        __half2 r3 = __hfma2(*reinterpret_cast<const __half2 *>(&p37), sixteenth, z.fma_c);
        o[0] = *reinterpret_cast<uint32_t *>(&r0);
        o[1] = *reinterpret_cast<uint32_t *>(&r1);
        o[2] = *reinterpret_cast<uint32_t *>(&r2);
        o[3] = *reinterpret_cast<uint32_t *>(&r3);
    }
};
template <> struct W4Widen<__nv_bfloat16> {
    // 128.0 (0x4300) has 7 mantissa bits: each nibble is shifted to bits 0..3 of its half before the OR
    struct Z {
        __nv_bfloat162 sub;
    };
    static __device__ __forceinline__ Z zero(int z) { return {__bfloat162bfloat162(__int2bfloat16_rn(128 + z))}; }
    static __device__ __forceinline__ void run(uint32_t w, const Z &z, uint32_t (&o)[4]) {
        const uint32_t M = 0x43004300u;
#pragma unroll
        for (int i = 0; i < 4; ++i) {
            const uint32_t p = lop3_and_or(w >> (4 * i), 0x000F000Fu, M);
            __nv_bfloat162 r = __hsub2(*reinterpret_cast<const __nv_bfloat162 *>(&p), z.sub);
            o[i] = *reinterpret_cast<uint32_t *>(&r);
        }
    }
};

template <typename T> __device__ __forceinline__ float ldg_f(const void *p, int64_t i) {
    const unsigned short u = __ldg(reinterpret_cast<const unsigned short *>(p) + i);
    return to_f<T>(*reinterpret_cast<const T *>(&u));
}

// BS: block size; ZP: zero points present (otherwise z = 8)
template <typename T, int MT, int BS, bool ZP>
__global__ void __launch_bounds__(W4_THREADS) gemm_skinny_w4_kernel(const __grid_constant__ W4Groups grp,
                                                                    const __grid_constant__ CUtensorMap mapX, const void *residual,
                                                                    int M, int K, int ktiles, int ktiles_per_split, int S) {
    using Cfg = W4Cfg<MT>;
    constexpr int NBS = W4_BK / BS;  // quantisation blocks per stage
    constexpr int CPB = BS / 32;     // k32 chunks per block
    using Widen = W4Widen<T>;
    extern __shared__ uint8_t smem_raw[];
    uint8_t *smem = smem_raw + ((1024u - (smem_u32(smem_raw) & 1023u)) & 1023u);
    uint8_t *w_sm = smem;
    uint8_t *x_sm = smem + S * W4_W_BYTES;
    float *red = reinterpret_cast<float *>(x_sm + S * Cfg::X_BYTES);
    uint64_t *full = reinterpret_cast<uint64_t *>(reinterpret_cast<uint8_t *>(red) + Cfg::RED_BYTES);
    uint64_t *empty = full + S;

    cg::cluster_group cluster = cg::this_cluster();
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    int gi = 0;
#pragma unroll
    for (int i = 1; i < W4_MAX_GROUPS; ++i)
        if (i < grp.ngroups && (int)blockIdx.x >= grp.tile_start[i]) gi = i;
    const CUtensorMap *mapWp = &grp.mapW[gi];
    const int n0 = ((int)blockIdx.x - grp.tile_start[gi]) * W4_BN;
    const int gN = grp.n[gi];
    const int split = blockIdx.y, nsplit = gridDim.y;
    const int kt_begin = split * ktiles_per_split;
    const int kt_end = min(ktiles, kt_begin + ktiles_per_split);
    const int my_kt = max(0, kt_end - kt_begin);
    const int nblk = K / BS;

    pdl_trigger();
    if (threadIdx.x == 0) {
        for (int s = 0; s < S; ++s) {
            mbar_init(&full[s], 1);
            mbar_init(&empty[s], 4);
        }
        fence_mbar_init();
    }
    if (warp == 4 && lane == 0) {
        tma_prefetch_desc(mapWp);
        tma_prefetch_desc(&mapX);
    }
    __syncthreads();

    if (warp == 4) {
        // ===== TMA producer (one lane) =====
        if (lane == 0) {
            const uint64_t pol_w = l2_policy_evict_first();
            const uint64_t pol_x = l2_policy_evict_last();
            // the codes are constants of the step: the first ring of them is requested before waiting for the predecessor
            const int pre = min(S, my_kt);
            for (int it = 0; it < pre; ++it) {
                mbar_expect_tx(&full[it], W4_W_BYTES + Cfg::X_BYTES);
                tma_load_2d(w_sm + it * W4_W_BYTES, mapWp, &full[it], (kt_begin + it) * (W4_BK / 2), n0, pol_w);
            }
            pdl_wait();
            for (int it = 0; it < pre; ++it)
#pragma unroll
                for (int bx = 0; bx < 4; ++bx)
                    tma_load_2d(x_sm + it * Cfg::X_BYTES + bx * Cfg::X_BOX_BYTES, &mapX, &full[it], (kt_begin + it) * W4_BK + bx * 64,
                                0, pol_x);
            int s = 0;
            uint32_t ph = 0;
            for (int it = pre; it < my_kt; ++it) {
                mbar_wait(&empty[s], ph);
                mbar_expect_tx(&full[s], W4_W_BYTES + Cfg::X_BYTES);
                const int kt = kt_begin + it;
                tma_load_2d(w_sm + s * W4_W_BYTES, mapWp, &full[s], kt * (W4_BK / 2), n0, pol_w);
#pragma unroll
                for (int bx = 0; bx < 4; ++bx)
                    tma_load_2d(x_sm + s * Cfg::X_BYTES + bx * Cfg::X_BOX_BYTES, &mapX, &full[s], kt * W4_BK + bx * 64, 0, pol_x);
                if (++s == S) {
                    s = 0;
                    ph ^= 1;
                }
            }
        }
        __syncwarp();
    } else {
        // ===== consumers: warp w owns columns [16w, 16w + 16) of the tile; lane (g, t) = (lane / 4, lane % 4) =====
        const int g = lane >> 2, t = lane & 3;
        float acc[MT][2][4], part[MT][2][4];
#pragma unroll
        for (int mt = 0; mt < MT; ++mt)
#pragma unroll
            for (int nb = 0; nb < 2; ++nb)
#pragma unroll
                for (int i = 0; i < 4; ++i) acc[mt][nb][i] = part[mt][nb][i] = 0.f;
        const void *scale = grp.scale[gi];
        const uint8_t *zp = grp.zp[gi];
        int s = 0;
        uint32_t ph = 0;
        for (int it = 0; it < my_kt; ++it) {
            const int kt = kt_begin + it;
            const int b0 = kt * NBS;  // first block of the stage
            // this stage's block scales of the lane's accumulator columns 2t, 2t + 1 of both 8-column tiles, and (ZP) the zero
            // points of its B columns g -- constants, read while the stage's tiles are in flight
            float sc[2][2][NBS];
#pragma unroll
            for (int nb = 0; nb < 2; ++nb)
#pragma unroll
                for (int e = 0; e < 2; ++e) {
                    const int cn = n0 + warp * 16 + nb * 8 + 2 * t + e;
#pragma unroll
                    for (int bi = 0; bi < NBS; ++bi)
                        sc[nb][e][bi] = (cn < gN && b0 + bi < nblk) ? ldg_f<T>(scale, (int64_t)cn * nblk + b0 + bi) : 0.f;
                }
            uint32_t zb[2] = {0, 0};  // NBS nibbles of each B column, block bi at bits 4 bi
            if constexpr (ZP) {
#pragma unroll
                for (int nb = 0; nb < 2; ++nb) {
                    const int bn = n0 + warp * 16 + nb * 8 + g;
#pragma unroll
                    for (int bi = 0; bi < NBS; bi += 2)
                        if (bn < gN && b0 + bi < nblk) zb[nb] |= (uint32_t)__ldg(zp + (int64_t)bn * (nblk / 2) + (b0 + bi) / 2) << (4 * bi);
                }
            }
            mbar_wait(&full[s], ph);
            const uint8_t *ws = w_sm + s * W4_W_BYTES, *xs = x_sm + s * Cfg::X_BYTES;
            typename Widen::Z zc[2];
#pragma unroll
            for (int j = 0; j < W4_BK / 32; ++j) {
                const int bi = j / CPB;
                if (j % CPB == 0) {
#pragma unroll
                    for (int nb = 0; nb < 2; ++nb) zc[nb] = Widen::zero(ZP ? (int)((zb[nb] >> (4 * bi)) & 15u) : 8);
                }
                // A fragments of both steps: X rows g, g + 8 of each 16-row tile, k = 32 j + 8 t .. + 7 (one 16-byte read per row)
                uint32_t a[2][MT][4];
#pragma unroll
                for (int mt = 0; mt < MT; ++mt) {
                    uint4 xr[2];
#pragma unroll
                    for (int h = 0; h < 2; ++h) {
                        const int row = mt * 16 + g + 8 * h;
                        const int ch = (j & 1) * 4 + t;
                        xr[h] = *reinterpret_cast<const uint4 *>(xs + (j >> 1) * Cfg::X_BOX_BYTES + row * 128 + ((ch ^ (row & 7)) << 4));
                    }
                    a[0][mt][0] = prmt(xr[0].x, xr[0].z, 0x5410);  // (k0, k4) of row g
                    a[0][mt][1] = prmt(xr[1].x, xr[1].z, 0x5410);  // (k0, k4) of row g + 8
                    a[0][mt][2] = prmt(xr[0].x, xr[0].z, 0x7632);  // (k1, k5)
                    a[0][mt][3] = prmt(xr[1].x, xr[1].z, 0x7632);
                    a[1][mt][0] = prmt(xr[0].y, xr[0].w, 0x5410);  // (k2, k6)
                    a[1][mt][1] = prmt(xr[1].y, xr[1].w, 0x5410);
                    a[1][mt][2] = prmt(xr[0].y, xr[0].w, 0x7632);  // (k3, k7)
                    a[1][mt][3] = prmt(xr[1].y, xr[1].w, 0x7632);
                }
#pragma unroll
                for (int nb = 0; nb < 2; ++nb) {
                    const int row = warp * 16 + nb * 8 + g;  // the code row = output column of this lane's B fragment
                    const uint32_t wd = *reinterpret_cast<const uint32_t *>(ws + row * 128 + ((j ^ (row & 7)) << 4) + 4 * t);
                    uint32_t b[4];
                    Widen::run(wd, zc[nb], b);
#pragma unroll
                    for (int mt = 0; mt < MT; ++mt) {
                        mma_m16n8k16<T>(part[mt][nb], a[0][mt], b[0], b[1]);
                        mma_m16n8k16<T>(part[mt][nb], a[1][mt], b[2], b[3]);
                    }
                }
                if (j % CPB == CPB - 1) {  // end of a quantisation block: fold its partial sum with the block's scale
#pragma unroll
                    for (int mt = 0; mt < MT; ++mt)
#pragma unroll
                        for (int nb = 0; nb < 2; ++nb)
#pragma unroll
                            for (int i = 0; i < 4; ++i) {
                                acc[mt][nb][i] = __fmaf_rn(part[mt][nb][i], sc[nb][i & 1][bi], acc[mt][nb][i]);
                                part[mt][nb][i] = 0.f;
                            }
                }
            }
            __syncwarp();
            if (lane == 0) mbar_arrive(&empty[s]);
            if (++s == S) {
                s = 0;
                ph ^= 1;
            }
        }
#pragma unroll
        for (int mt = 0; mt < MT; ++mt)
#pragma unroll
            for (int nb = 0; nb < 2; ++nb) {
                const int row = mt * 16 + g;
                const int col = warp * 16 + nb * 8 + 2 * t;
                *reinterpret_cast<float2 *>(&red[row * W4_BN + col]) = make_float2(acc[mt][nb][0], acc[mt][nb][1]);
                *reinterpret_cast<float2 *>(&red[(row + 8) * W4_BN + col]) = make_float2(acc[mt][nb][2], acc[mt][nb][3]);
            }
    }

    // ===== split-K reduction through distributed shared memory + epilogue =====
    pdl_wait();  // every thread that reads the residual / writes C is ordered after the predecessor kernel
    if (nsplit > 1) cluster.sync(); else __syncthreads();
    if (split == 0) {
        const float *peers[8];
        for (int r = 0; r < nsplit; ++r) peers[r] = nsplit > 1 ? (const float *)cluster.map_shared_rank(red, r) : red;
        const T *res = (const T *)residual;
        T *C = (T *)grp.C[gi];
        for (int idx = threadIdx.x; idx < MT * 16 * (W4_BN / 2); idx += W4_THREADS) {
            const int row = idx / (W4_BN / 2), col = (idx % (W4_BN / 2)) * 2;
            const int gn = n0 + col;
            if (row >= M || gn >= gN) continue;  // (N % 16 == 0: both columns of the pair are in range)
            float2 v = make_float2(0.f, 0.f);
            for (int r = 0; r < nsplit; ++r) {
                const float2 p = *reinterpret_cast<const float2 *>(&peers[r][row * W4_BN + col]);
                v.x += p.x;
                v.y += p.y;
            }
            if (res) {  // MatMul -> Add: the product is rounded to T, then the residual added
                v.x = round_t<T>(v.x) + to_f(res[(int64_t)row * gN + gn]);
                v.y = round_t<T>(v.y) + to_f(res[(int64_t)row * gN + gn + 1]);
            }
            T *dst = C + (int64_t)row * gN + gn;
            if constexpr (std::is_same<T, __nv_bfloat16>::value)
                *reinterpret_cast<__nv_bfloat162 *>(dst) = __floats2bfloat162_rn(v.x, v.y);
            else
                *reinterpret_cast<__half2 *>(dst) = __floats2half2_rn(v.x, v.y);
        }
    }
    if (nsplit > 1) cluster.sync();  // peers' shared memory must outlive the leader's reads
}

template <typename T, int MT, int BS, bool ZP>
static int launch_w4(const void *X, int ngroups, const void *const *Wq, const void *const *scales, const void *const *zps,
                     void *const *Cs, const int *Ns, int m, int k, const void *residual, cudaStream_t st) {
    using Cfg = W4Cfg<MT>;
    W4Groups grp{};
    CUtensorMap mapX;
    grp.ngroups = ngroups;
    int tiles_n = 0;
    for (int i = 0; i < ngroups; ++i) {
        // the codes as a [N rows x K / 2 bytes] matrix, box [64 rows x 128 bytes]
        if (!make_tma_2d_u8_sw128(&grp.mapW[i], Wq[i], (uint64_t)Ns[i], (uint64_t)k / 2, (uint64_t)k / 2, W4_BN, W4_BK / 2))
            ITB_FAIL("matmul_nbits: cuTensorMapEncodeTiled(B) failed");
        grp.C[i] = Cs[i];
        grp.scale[i] = scales[i];
        grp.zp[i] = ZP ? (const uint8_t *)zps[i] : nullptr;
        grp.n[i] = Ns[i];
        grp.tile_start[i] = tiles_n;
        tiles_n += (Ns[i] + W4_BN - 1) / W4_BN;
    }
    for (int i = ngroups; i <= W4_MAX_GROUPS; ++i) grp.tile_start[i] = tiles_n;
    if (!make_tma_2d_b16(&mapX, X, (uint64_t)m, (uint64_t)k, (uint64_t)k, MT * 16, 64, 128))
        ITB_FAIL("matmul_nbits: cuTensorMapEncodeTiled(X) failed");
    const int ktiles = (k + W4_BK - 1) / W4_BK;
    // enough CTAs for two per SM, at least 2 stages of 256 k per CTA, cluster <= 8
    int splitk = std::max(1, std::min(2 * kNumSMs / tiles_n, 8));
    splitk = std::min(splitk, std::max(1, ktiles / 2));
    int per = (ktiles + splitk - 1) / splitk;
    splitk = (ktiles + per - 1) / per;  // no empty split
    constexpr int stages_deep = Cfg::stages_for(kW4DeepBudgetKB), stages_split = Cfg::stages_for(kW4SplitBudgetKB);
    const int stages = splitk > 1 ? stages_split : stages_deep;
    const int smem_bytes = Cfg::smem_for(stages);
    return launch("matmul_nbits", gemm_skinny_w4_kernel<T, MT, BS, ZP>,
                  {dim3(tiles_n, splitk, 1), dim3(W4_THREADS, 1, 1), smem_bytes, st, dim3(1, splitk, 1)}, grp, mapX, residual, m,
                  k, ktiles, per, stages);
}

template <typename T, int MT, int BS>
static int launch_w4_zp(bool zp, const void *X, int ng, const void *const *Wq, const void *const *sc, const void *const *zps,
                        void *const *C, const int *N, int m, int k, const void *res, cudaStream_t st) {
    if (zp) return launch_w4<T, MT, BS, true>(X, ng, Wq, sc, zps, C, N, m, k, res, st);
    return launch_w4<T, MT, BS, false>(X, ng, Wq, sc, zps, C, N, m, k, res, st);
}
template <typename T, int MT>
static int launch_w4_bs(int bs, bool zp, const void *X, int ng, const void *const *Wq, const void *const *sc, const void *const *zps,
                        void *const *C, const int *N, int m, int k, const void *res, cudaStream_t st) {
    if (bs == 32) return launch_w4_zp<T, MT, 32>(zp, X, ng, Wq, sc, zps, C, N, m, k, res, st);
    if (bs == 64) return launch_w4_zp<T, MT, 64>(zp, X, ng, Wq, sc, zps, C, N, m, k, res, st);
    return launch_w4_zp<T, MT, 128>(zp, X, ng, Wq, sc, zps, C, N, m, k, res, st);
}
template <typename T>
static int launch_w4_mt(int bs, bool zp, const void *X, int ng, const void *const *Wq, const void *const *sc, const void *const *zps,
                        void *const *C, const int *N, int m, int k, const void *res, cudaStream_t st) {
    const int mt = (m + 15) / 16;
    if (mt == 1) return launch_w4_bs<T, 1>(bs, zp, X, ng, Wq, sc, zps, C, N, m, k, res, st);
    if (mt == 2) return launch_w4_bs<T, 2>(bs, zp, X, ng, Wq, sc, zps, C, N, m, k, res, st);
    return launch_w4_bs<T, 4>(bs, zp, X, ng, Wq, sc, zps, C, N, m, k, res, st);
}

// W[k, n] = T((q[n, k] - z[n, k / bs]) . s[n, k / bs]) as a [K, N] row-major matrix; one thread per (byte of codes, column):
// threads of a warp take consecutive columns, so the two rows they write are coalesced
template <typename T>
__global__ void __launch_bounds__(256) dequant_w4_kernel(const uint8_t *__restrict__ q, const T *__restrict__ s,
                                                         const uint8_t *__restrict__ zp, T *__restrict__ w, int K, int N, int bs) {
    pdl_trigger();
    pdl_wait();
    const int nblk = K / bs;
    const int64_t total = (int64_t)(K / 2) * N;
    for (int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; i < total; i += (int64_t)gridDim.x * blockDim.x) {
        const int n = (int)(i % N), kb = (int)(i / N);  // code byte kb of column n: k = 2 kb, 2 kb + 1
        const int k = 2 * kb, blk = k / bs;
        const uint32_t byte = q[(int64_t)n * (K / 2) + kb];
        const int z = zp ? (zp[(int64_t)n * (nblk / 2) + blk / 2] >> (4 * (blk & 1))) & 15 : 8;
        const float sc = to_f(s[(int64_t)n * nblk + blk]);
        w[(int64_t)k * N + n] = from_f<T>((float)((int)(byte & 15u) - z) * sc);
        w[(int64_t)(k + 1) * N + n] = from_f<T>((float)((int)(byte >> 4) - z) * sc);
    }
}

static int dequant_w4(int dtype, const void *q, const void *s, const void *zp, void *w, int k, int n, int bs, cudaStream_t st) {
    const int64_t total = (int64_t)(k / 2) * n;
    if (total == 0) return 0;
    const LaunchCfg c{dim3(grid_for(total, 256)), dim3(256), 0, st};
    if (dtype == ITB_BF16)
        return launch("dequantize_w4", dequant_w4_kernel<__nv_bfloat16>, c, (const uint8_t *)q, (const __nv_bfloat16 *)s,
                      (const uint8_t *)zp, (__nv_bfloat16 *)w, k, n, bs);
    return launch("dequantize_w4", dequant_w4_kernel<__half>, c, (const uint8_t *)q, (const __half *)s, (const uint8_t *)zp,
                  (__half *)w, k, n, bs);
}

// the operator contract's rules on (dtype, K, N, block size, zero points); 0 = accepted, else the error is set
static int nbits_check(const char *who, int dtype, int k, int n, int bs, bool zp) {
    ITB_CHECK(dtype == ITB_F16 || dtype == ITB_BF16, "%s: activations / scales must be f16 or bf16 (dtype %d)", who, dtype);
    ITB_CHECK(bs == 32 || bs == 64 || bs == 128, "%s: block_size %d is not 32, 64 or 128", who, bs);
    ITB_CHECK(k > 0 && k % bs == 0, "%s: K = %d is not a positive multiple of block_size %d", who, k, bs);
    ITB_CHECK(n > 0 && n % 16 == 0, "%s: N = %d is not a positive multiple of 16", who, n);
    ITB_CHECK(!zp || (k / bs) % 2 == 0, "%s: zero points need an even number of blocks per column (K / block_size = %d)", who, k / bs);
    return 0;
}

}  // namespace itb

using namespace itb;

extern "C" int64_t it_b200_matmul_nbits_workspace(int dtype, int m, int k, int n_groups, const int *N) {
    if (m <= 64 || (dtype != ITB_F16 && dtype != ITB_BF16)) return 0;
    int64_t nmax = 0;
    for (int i = 0; i < n_groups; ++i) nmax = std::max<int64_t>(nmax, N[i]);
    return (int64_t)k * nmax * 2;
}

extern "C" int it_b200_dequantize_w4(int dtype, const void *Wq, const void *scales, const void *zero_points, void *W, int k, int n,
                                     int block_size, void *stream) {
    if (nbits_check("dequantize_w4", dtype, k, n, block_size, zero_points != nullptr)) return 1;
    return dequant_w4(dtype, Wq, scales, zero_points, W, k, n, block_size, (cudaStream_t)stream);
}

extern "C" int it_b200_matmul_nbits(int dtype, const void *X, int n_groups, const void *const *Wq, const void *const *scales,
                                    const void *const *zero_points, void *const *C, const int *N, int m, int k, int block_size,
                                    const void *residual, void *workspace, int64_t workspace_bytes, void *stream) {
    ITB_CHECK(n_groups >= 1 && n_groups <= 4, "matmul_nbits: 1..4 weight matrices per launch (%d)", n_groups);
    ITB_CHECK(!residual || n_groups == 1, "matmul_nbits: a residual goes with a single weight matrix");
    ITB_CHECK(m >= 0, "matmul_nbits: negative row count %d", m);
    const bool zp = zero_points != nullptr;
    for (int i = 0; i < n_groups; ++i) {
        if (nbits_check("matmul_nbits", dtype, k, N[i], block_size, zp)) return 1;
        ITB_CHECK(Wq[i] && scales[i] && (!zp || zero_points[i]), "matmul_nbits: matrix %d lacks its codes, scales or zero points", i);
        ITB_CHECK(aligned16(Wq[i]) && aligned16(C[i]), "matmul_nbits: codes and outputs must be 16-byte aligned");
    }
    ITB_CHECK(aligned16(X) && (!residual || aligned16(residual)), "matmul_nbits: X and the residual must be 16-byte aligned");
    if (m == 0) return 0;
    auto st = (cudaStream_t)stream;
    if (m <= 64) {
        if (dtype == ITB_BF16)
            return launch_w4_mt<__nv_bfloat16>(block_size, zp, X, n_groups, Wq, scales, zero_points, C, N, m, k, residual, st);
        return launch_w4_mt<__half>(block_size, zp, X, n_groups, Wq, scales, zero_points, C, N, m, k, residual, st);
    }
    // more rows than the decode kernel takes: each matrix dequantised into the workspace, then the 16-bit GEMM
    const int64_t need = it_b200_matmul_nbits_workspace(dtype, m, k, n_groups, N);
    ITB_CHECK(workspace && workspace_bytes >= need && aligned16(workspace), "matmul_nbits: workspace %lld < %lld bytes (or unaligned)",
              (long long)workspace_bytes, (long long)need);
    for (int i = 0; i < n_groups; ++i) {
        if (dequant_w4(dtype, Wq[i], scales[i], zp ? zero_points[i] : nullptr, workspace, k, N[i], block_size, st)) return 1;
        // (not ITB_MATMUL_B_CONST: the dequantised matrix is written by the kernel just before)
        const int act = residual ? ITB_ACT_ROUND_BEFORE_BIAS : 0;
        const int r = it_b200_matmul(dtype, X, workspace, residual, C[i], 1, m, N[i], k, (int64_t)m * k, 0, 0, 0, 0, residual ? N[i] : 0,
                                     residual ? 1 : 0, act, nullptr, 0, stream);
        if (r) return r;
    }
    return 0;
}
