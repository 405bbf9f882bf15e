// gemm_skinny.cu -- decode-regime MatMul (M <= 64) for sm_90a: pure weight streaming, HBM-bound.
//
//   C[M,N] = X[M,K] . W[K,N] (+bias, act)      X, W, C: bf16 / fp16 row-major, fp32 accumulate
//
// Replaces the reference's cublasGemmEx call for the Llama decode shapes (matmul.cc:141-168;
// SURVEY 8a row a1: q/k/v/o 16x4096x4096, gate/up 16x4096x11008, down 16x11008x4096, logits
// 16x4096x32000).  The weight matrix is read exactly once:
//   * TMA (cp.async.bulk.tensor.2d, 128B swizzle) streams 64(k) x 64(n) weight tiles and the
//     matching 16*MT x 64 activation tile into a STAGES-deep shared-memory ring, completion on
//     mbarriers; one producer lane issues, four consumer warps drain.
//   * consumers feed legacy mma.sync m16n8k16 from the swizzled tiles with ldmatrix(.trans); at
//     M = 16 the tensor pipe needs < 5 % of its rate to keep up with HBM, so the legacy path is
//     not the limiter (the wgmma swap-AB variant lives in gemm_tc.cu for M > 64).
//   * split-K across a thread-block CLUSTER (<= 8 CTAs along K): partial tiles are reduced by the
//     rank-0 CTA through distributed shared memory, so there is no global workspace, no atomics
//     and no second kernel; bias / activation / dtype conversion are fused into that store.
// Grid = ceil(N/64) x splitK CTAs: unsplit, two co-resident per SM (~105 KB smem each); split-K, three (~65 KB each).
#include <cooperative_groups.h>

#include "gemm.cuh"

namespace cg = cooperative_groups;

namespace itb {

constexpr int SK_BOX = 64, SK_BK = 64;
constexpr int SK_BOX_BYTES = SK_BOX * SK_BK * 2;  // 8 KB: one [64k x 64n] swizzled TMA box
constexpr int SK_THREADS = 160;                // 4 consumer warps + 1 producer warp

// NB = 64-column boxes per tile: NB = 1 -> 64-wide tiles (128 B per weight row), NB = 2 -> 128-wide tiles (256 B
// contiguous per row: better DRAM efficiency when there are enough column tiles to fill the machine)
// W8: the weight operand is FP8 E4M3 (one byte per element, [64k x 64n] boxes of 4 KB, unswizzled): half the bytes per stage
template <int MT, int NB, bool W8 = false> struct SkinnyCfg {
    static constexpr int BN = NB * SK_BOX;
    static constexpr int BOX_BYTES = W8 ? SK_BOX_BYTES / 2 : SK_BOX_BYTES;
    static constexpr int W_BYTES = NB * BOX_BYTES;
    static constexpr int X_BYTES = MT * 16 * SK_BK * 2;
    static constexpr int RED_BYTES = MT * 16 * BN * 4;
    static constexpr int stages_for(int budget_kb) {
        int s = (budget_kb * 1024 - RED_BYTES - 1024 - 256) / (W_BYTES + X_BYTES);
        return s < 2 ? 2 : (s > 16 ? 16 : s);
    }
    static constexpr int smem_for(int stages) { return stages * (W_BYTES + X_BYTES) + RED_BYTES + 2 * stages * 8 + 1024; }
};

// Ring budget of split-K launches (see launch_skinny_nb): three CTAs per SM.  An SM has 228 KB of shared memory and
// reserves 1 KB per resident CTA.
constexpr int kSkinnySplitBudgetKB = 66;
constexpr int kSkinnySplitSmem = SkinnyCfg<1, 1>::smem_for(SkinnyCfg<1, 1>::stages_for(kSkinnySplitBudgetKB));
static_assert(3 * (kSkinnySplitSmem + 1024) <= 228 * 1024, "split-K skinny GEMM: three CTAs must fit on one SM");

// Up to 4 weight matrices that share the activation operand X (q/k/v, gate/up) run as ONE launch: the
// N-tile index selects the group.  A plain MatMul is the 1-group case.
constexpr int SK_MAX_GROUPS = 4;
struct SkinnyGroups {
    CUtensorMap mapW[SK_MAX_GROUPS];
    void *C[SK_MAX_GROUPS];
    int n[SK_MAX_GROUPS];
    int tile_start[SK_MAX_GROUPS + 1];
    int ngroups;
    const float *w_scale[SK_MAX_GROUPS];  // W8: per-output-column scale of each group's weight matrix
};

template <typename T, int MT, int NB, bool W8>
__global__ void __launch_bounds__(SK_THREADS) gemm_skinny_kernel(const __grid_constant__ SkinnyGroups grp,
                                                                 const __grid_constant__ CUtensorMap mapX,
                                                                 GemmArgs g, int ktiles, int ktiles_per_split,
                                                                 int S) {
    using Cfg = SkinnyCfg<MT, NB, W8>;
    constexpr int SK_BN = Cfg::BN, SK_W_BYTES = Cfg::W_BYTES, BOXB = Cfg::BOX_BYTES;
    extern __shared__ uint8_t smem_raw[];
    // 128B-swizzled TMA tiles need 1024-byte alignment
    uint8_t *smem = smem_raw + ((1024u - (smem_u32(smem_raw) & 1023u)) & 1023u);
    uint8_t *w_sm = smem;
    uint8_t *x_sm = smem + S * SK_W_BYTES;
    float *red = reinterpret_cast<float *>(x_sm + S * Cfg::X_BYTES);
    uint64_t *full = reinterpret_cast<uint64_t *>(reinterpret_cast<uint8_t *>(red) + Cfg::RED_BYTES);
    uint64_t *empty = full + S;

    cg::cluster_group cluster = cg::this_cluster();
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    int gi = 0;
#pragma unroll
    for (int i = 1; i < SK_MAX_GROUPS; ++i)
        if (i < grp.ngroups && (int)blockIdx.x >= grp.tile_start[i]) gi = i;
    const CUtensorMap *mapWp = &grp.mapW[gi];
    const int n0 = ((int)blockIdx.x - grp.tile_start[gi]) * SK_BN;
    const int gN = grp.n[gi];
    const int split = blockIdx.y, nsplit = gridDim.y;
    const int kt_begin = split * ktiles_per_split;
    const int kt_end = min(ktiles, kt_begin + ktiles_per_split);
    const int my_kt = max(0, kt_end - kt_begin);

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

    float acc[MT][2 * NB][4];
#pragma unroll
    for (int mt = 0; mt < MT; ++mt)
#pragma unroll
        for (int nb = 0; nb < 2 * NB; ++nb)
#pragma unroll
            for (int i = 0; i < 4; ++i) acc[mt][nb][i] = 0.f;

    if (warp == 4) {
        // ===== TMA producer (one lane) =====
        if (lane == 0) {
            const uint64_t pol_w = l2_policy_evict_first();  // weights are read once per step
            const uint64_t pol_x = l2_policy_evict_last();   // activations are re-read by every N-tile
            // PDL: the weights are written by no kernel of the step, so the first ring of weight tiles is
            // requested BEFORE waiting for the predecessor kernel; activations only after pdl_wait()
            const int pre = min(S, my_kt);
            if (!(g.act & ITB_MATMUL_B_CONST)) pdl_wait();  // B produced upstream: no early prefetch
            for (int it = 0; it < pre; ++it) {
                mbar_expect_tx(&full[it], SK_W_BYTES + Cfg::X_BYTES);
#pragma unroll
                for (int bx = 0; bx < NB; ++bx)
                    tma_load_2d(w_sm + it * SK_W_BYTES + bx * BOXB, mapWp, &full[it], n0 + bx * SK_BOX,
                                (kt_begin + it) * SK_BK, pol_w);
            }
            pdl_wait();
            for (int it = 0; it < pre; ++it)
                tma_load_2d(x_sm + it * Cfg::X_BYTES, &mapX, &full[it], (kt_begin + it) * SK_BK, 0, pol_x);
            int s = 0;
            uint32_t ph = 0;  // parity of the `empty` completion that frees stage s for its next use
            for (int it = pre; it < my_kt; ++it) {
                mbar_wait(&empty[s], ph);
                mbar_expect_tx(&full[s], SK_W_BYTES + Cfg::X_BYTES);
                const int k0 = (kt_begin + it) * SK_BK;
#pragma unroll
                for (int bx = 0; bx < NB; ++bx)
                    tma_load_2d(w_sm + s * SK_W_BYTES + bx * BOXB, mapWp, &full[s], n0 + bx * SK_BOX, k0, pol_w);
                tma_load_2d(x_sm + s * Cfg::X_BYTES, &mapX, &full[s], k0, 0, pol_x);
                if (++s == S) {
                    s = 0;
                    ph ^= 1;
                }
            }
        }
        __syncwarp();
    } else {
        // ===== consumers: warp w owns columns [16w, 16w+16) of the tile =====
        const int mi = lane >> 3;             // which 8x8 matrix this lane addresses
        const int r8 = lane & 7;
        const uint32_t w_base = smem_u32(w_sm), x_base = smem_u32(x_sm);
        int s = 0;
        uint32_t ph = 0;
        for (int it = 0; it < my_kt; ++it) {
            mbar_wait(&full[s], ph);
            const uint32_t wb = w_base + s * SK_W_BYTES, xb = x_base + s * Cfg::X_BYTES;
#pragma unroll
            for (int kk = 0; kk < SK_BK / 16; ++kk) {
                uint32_t a[MT][4];
#pragma unroll
                for (int mt = 0; mt < MT; ++mt) {
                    const int row = mt * 16 + r8 + 8 * (mi & 1);
                    const int chunk = kk * 2 + (mi >> 1);
                    ldmatrix_x4(a[mt][0], a[mt][1], a[mt][2], a[mt][3],
                                xb + row * 128 + ((chunk ^ (row & 7)) << 4));
                }
#pragma unroll
                for (int bx = 0; bx < NB; ++bx) {  // warp w owns columns [16w, 16w+16) of every 64-column box
                    uint32_t b0, b1, b2, b3;
                    if constexpr (W8) {
                        // This mma.sync path spends ~700 warp instructions per 4 KB chunk on byte gathers and the e4m3 -> bf16
                        // conversion, so it is instruction-bound rather than HBM-bound.  It halves the weight footprint and is
                        // parity-exact; a bandwidth win needs the tensor core to consume the codes directly (FP8 wgmma with
                        // quantised activations).
                        // FP8 weights: the box is [64 k][64 n] bytes, unswizzled.  B fragment of mma.m16n8k16 (col-major): lane
                        // (g = lane / 4, t = lane % 4) holds {W[2t][g], W[2t+1][g]} and {W[2t+8][g], W[2t+9][g]} of each 8-column
                        // tile -- two byte loads per register, converted to the activation type on the way (the "dequant" of
                        // the main loop; the per-column scale is applied once, to the fp32 sum, in the epilogue)
                        const uint8_t *tile = w_sm + s * SK_W_BYTES + bx * BOXB + (kk * 16 + 2 * (lane & 3)) * 64 + warp * 16 + (lane >> 2);
                        auto frag = [&](const uint8_t *p) { return e4m3x2_to<T>((uint32_t)p[0] | ((uint32_t)p[64] << 8)); };
                        b0 = frag(tile);
                        b1 = frag(tile + 8 * 64);
                        b2 = frag(tile + 8);
                        b3 = frag(tile + 8 * 64 + 8);
                    } else {
                    const int krow = kk * 16 + r8 + 8 * (mi & 1);
                    const int nchunk = warp * 2 + (mi >> 1);
                    ldmatrix_x4_trans(b0, b1, b2, b3, wb + bx * SK_BOX_BYTES + krow * 128 + ((nchunk ^ (krow & 7)) << 4));
                    }
#pragma unroll
                    for (int mt = 0; mt < MT; ++mt) {
                        mma_m16n8k16<T>(acc[mt][bx * 2 + 0], a[mt], b0, b1);
                        mma_m16n8k16<T>(acc[mt][bx * 2 + 1], a[mt], b2, b3);
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
        // partial tile -> shared memory (fp32)
#pragma unroll
        for (int mt = 0; mt < MT; ++mt)
#pragma unroll
            for (int nb = 0; nb < 2 * NB; ++nb) {
                const int row = mt * 16 + (lane >> 2);
                const int col = (nb >> 1) * SK_BOX + warp * 16 + (nb & 1) * 8 + (lane & 3) * 2;
                *reinterpret_cast<float2 *>(&red[row * SK_BN + col]) = make_float2(acc[mt][nb][0], acc[mt][nb][1]);
                *reinterpret_cast<float2 *>(&red[(row + 8) * SK_BN + col]) =
                    make_float2(acc[mt][nb][2], acc[mt][nb][3]);
            }
    }

    // ===== split-K reduction through distributed shared memory + fused epilogue =====
    pdl_wait();  // every thread that reads bias / writes C is ordered after the predecessor kernel
    if (nsplit > 1) cluster.sync(); else __syncthreads();
    if (split == 0) {
        const float *peers[8];
        for (int r = 0; r < nsplit; ++r)
            peers[r] = nsplit > 1 ? (const float *)cluster.map_shared_rank(red, r) : red;
        const T *bias = (const T *)g.bias;
        T *C = (T *)grp.C[gi];
        const bool round_first = (g.act & ITB_ACT_ROUND_BEFORE_BIAS) != 0;
        const int act = g.act & 0xff;
        for (int idx = threadIdx.x; idx < MT * 16 * (SK_BN / 2); idx += SK_THREADS) {
            const int row = idx / (SK_BN / 2), col = (idx % (SK_BN / 2)) * 2;
            const int gn = n0 + col;
            if (row >= g.m || gn >= gN) continue;
            float2 v = make_float2(0.f, 0.f);
            for (int r = 0; r < nsplit; ++r) {
                float2 p = *reinterpret_cast<const float2 *>(&peers[r][row * SK_BN + col]);
                v.x += p.x;
                v.y += p.y;
            }
            if constexpr (W8) {  // dequantisation: column scale of the weight matrix
                const float *sc = grp.w_scale[gi];
                v.x *= sc[gn];
                if (gn + 1 < gN) v.y *= sc[gn + 1];
            }
            if (bias) {
                if (round_first) {  // MatMul -> Add fusion: reproduce the unfused graph's rounding of the MatMul output
                    v.x = round_t<T>(v.x);
                    v.y = round_t<T>(v.y);
                }
                v.x += to_f(bias[row * g.bias_sm + gn * g.bias_sn]);
                if (gn + 1 < gN) v.y += to_f(bias[row * g.bias_sm + (gn + 1) * g.bias_sn]);
            }
            v.x = gemm_act(act, v.x);
            v.y = gemm_act(act, v.y);
            T *dst = C + (int64_t)row * gN + gn;
            if (gn + 1 < gN && (gN & 1) == 0) {
                if constexpr (std::is_same<T, __nv_bfloat16>::value)
                    *reinterpret_cast<__nv_bfloat162 *>(dst) = __floats2bfloat162_rn(v.x, v.y);
                else
                    *reinterpret_cast<__half2 *>(dst) = __floats2half2_rn(v.x, v.y);
            } else {
                dst[0] = from_f<T>(v.x);
                if (gn + 1 < gN) dst[1] = from_f<T>(v.y);
            }
        }
    }
    if (nsplit > 1) cluster.sync();  // peers' shared memory must outlive the leader's reads
}

// tuning hook (tools/gemm_sweep.py): force the tile width (NB boxes of 64 columns) and the split-K factor; 0 = automatic
static int g_nb_override = 0, g_splitk_override = 0;

template <typename T, int MT, int NB, bool W8 = false>
static int launch_skinny_nb(const GemmArgs &g, int ngroups, const void *const *Ws, void *const *Cs, const int *Ns,
                            cudaStream_t st, const float *const *scales = nullptr) {
    using Cfg = SkinnyCfg<MT, NB, W8>;
    constexpr int SK_BN = Cfg::BN;
    SkinnyGroups grp{};
    CUtensorMap mapX;
    grp.ngroups = ngroups;
    int tiles_n = 0;
    for (int i = 0; i < ngroups; ++i) {
        const bool okW = W8 ? make_tma_2d_u8(&grp.mapW[i], Ws[i], (uint64_t)g.k, (uint64_t)Ns[i], (uint64_t)Ns[i], SK_BK, SK_BOX)
                            : make_tma_2d_b16(&grp.mapW[i], Ws[i], (uint64_t)g.k, (uint64_t)Ns[i], (uint64_t)Ns[i], SK_BK, SK_BOX, 128);
        if (!okW) ITB_FAIL("matmul(skinny): cuTensorMapEncodeTiled(W) failed");
        grp.w_scale[i] = scales ? scales[i] : nullptr;
        grp.C[i] = Cs[i];
        grp.n[i] = Ns[i];
        grp.tile_start[i] = tiles_n;
        tiles_n += (Ns[i] + SK_BN - 1) / SK_BN;
    }
    for (int i = ngroups; i <= SK_MAX_GROUPS; ++i) grp.tile_start[i] = tiles_n;
    if (!make_tma_2d_b16(&mapX, g.A, (uint64_t)g.m, (uint64_t)g.k, (uint64_t)g.k, MT * 16, SK_BK, 128))
        ITB_FAIL("matmul(skinny): cuTensorMapEncodeTiled(X) failed");
    const int ktiles = (g.k + SK_BK - 1) / SK_BK;
    // enough CTAs for two per SM, at least 4 k-tiles per CTA, cluster <= 8
    int splitk = 2 * kNumSMs / tiles_n;
    splitk = std::max(1, std::min(splitk, 8));
    splitk = std::min(splitk, std::max(1, ktiles / 4));
    if (g_splitk_override) splitk = std::max(1, std::min(g_splitk_override, 8));
    int per = (ktiles + splitk - 1) / splitk;
    splitk = (ktiles + per - 1) / per;  // no empty split

    // Unsplit launches: a 106 KB ring per CTA, two CTAs per SM, as many bytes in flight as the SM can hold.
    // Split-K launches run as clusters, which are placed GPC by GPC: at two 106 KB CTAs per SM the 64 four-CTA clusters of
    // a 4096-wide decode GEMM (o, down) took about twice their streaming time on H100, as a second wave of clusters would.
    // A 66 KB ring lets three CTAs share an SM, and leaves room beside two of them for a gemm_tc CTA of the next GEMM
    // (gate/up, logits), which then streams its first weight tiles under this kernel's tail (PDL).  FP8 weights keep the
    // deep ring (measured slower at 66 KB).
    constexpr int stages_deep = Cfg::stages_for(106);
    constexpr int stages_split = W8 ? stages_deep : Cfg::stages_for(kSkinnySplitBudgetKB);
    const int stages = splitk > 1 ? stages_split : stages_deep;
    const int smem_bytes = Cfg::smem_for(stages);
    return launch("matmul(skinny)", gemm_skinny_kernel<T, MT, NB, W8>,
                  {dim3(tiles_n, splitk, 1), dim3(SK_THREADS, 1, 1), smem_bytes, st, dim3(1, splitk, 1)}, grp, mapX, g, ktiles,
                  per, stages);
}

// tile width: 128 columns once 64-wide tiles would already oversubscribe the 2 x 132 CTA slots
template <typename T, int MT>
static int launch_skinny_t(const GemmArgs &g, int ngroups, const void *const *Ws, void *const *Cs, const int *Ns,
                           cudaStream_t st) {
    int tiles64 = 0;
    for (int i = 0; i < ngroups; ++i) tiles64 += (Ns[i] + 63) / 64;
    const int nb = g_nb_override ? g_nb_override : (tiles64 > 2 * kNumSMs ? 2 : 1);
    if (nb == 2) return launch_skinny_nb<T, MT, 2>(g, ngroups, Ws, Cs, Ns, st);
    return launch_skinny_nb<T, MT, 1>(g, ngroups, Ws, Cs, Ns, st);
}

static bool skinny_ok(int dtype, const GemmArgs &g) {
    if (dtype != ITB_BF16 && dtype != ITB_F16) return false;
    if (g.batch != 1 || g.trans_a || g.trans_b || g.m > 64 || g.m < 1 || g.no_splitk) return false;
    if (g.n % 8 != 0 || g.k % 8 != 0 || g.n < 64 || g.k < 64) return false;
    if (!aligned16(g.A) || !aligned16(g.B) || ((uintptr_t)g.C & 3)) return false;
    return true;
}

// FP8-weight variants (64-wide tiles below 2 x 132 x ... column tiles, 128-wide above, as for 16-bit weights)
template <typename T, int MT>
static int launch_skinny_w8_t(const GemmArgs &g, int ngroups, const void *const *Ws, void *const *Cs, const int *Ns,
                              const float *const *scales, cudaStream_t st) {
    int tiles64 = 0;
    for (int i = 0; i < ngroups; ++i) tiles64 += (Ns[i] + 63) / 64;
    const int nb = g_nb_override ? g_nb_override : (tiles64 > 2 * kNumSMs ? 2 : 1);
    if (nb == 2) return launch_skinny_nb<T, MT, 2, true>(g, ngroups, Ws, Cs, Ns, st, scales);
    return launch_skinny_nb<T, MT, 1, true>(g, ngroups, Ws, Cs, Ns, st, scales);
}

#define SK_GO(TT, ...)                                                                         \
    do {                                                                                       \
        if (mt == 1) return launch_skinny_t<TT, 1>(__VA_ARGS__);                               \
        if (mt == 2) return launch_skinny_t<TT, 2>(__VA_ARGS__);                               \
        return launch_skinny_t<TT, 4>(__VA_ARGS__);                                            \
    } while (0)

int launch_gemm_skinny(int dtype, const GemmArgs &g, cudaStream_t st) {
    if (!skinny_ok(dtype, g)) return -1;
    const int mt = (g.m + 15) / 16;
    const void *Ws[1] = {g.B};
    void *Cs[1] = {g.C};
    int Ns[1] = {g.n};
    if (dtype == ITB_BF16) SK_GO(__nv_bfloat16, g, 1, Ws, Cs, Ns, st);
    SK_GO(__half, g, 1, Ws, Cs, Ns, st);
}

// X[M,K] . {W_i[K,N_i]} -> {C_i[M,N_i]} in one launch (no bias / activation)
int launch_gemm_skinny_grouped(int dtype, const GemmArgs &g0, int ngroups, const void *const *Ws, void *const *Cs,
                               const int *Ns, cudaStream_t st) {
    if (ngroups < 1 || ngroups > SK_MAX_GROUPS) return -1;
    for (int i = 0; i < ngroups; ++i) {
        GemmArgs g = g0;
        g.B = Ws[i];
        g.C = Cs[i];
        g.n = Ns[i];
        if (!skinny_ok(dtype, g)) return -1;
    }
    const int mt = (g0.m + 15) / 16;
    GemmArgs gc = g0;
    gc.act |= ITB_MATMUL_B_CONST;  // grouped weights are constants by contract
    if (dtype == ITB_BF16) SK_GO(__nv_bfloat16, gc, ngroups, Ws, Cs, Ns, st);
    SK_GO(__half, gc, ngroups, Ws, Cs, Ns, st);
}
#undef SK_GO

// X[M,K] (f16 / bf16) . {Wq_i[K,N_i] FP8 E4M3 x scale_i[N_i]} -> {C_i[M,N_i]}: 1..4 weight matrices sharing X in one launch;
// g0 carries bias / residual / act for the single-matrix case exactly like launch_gemm_skinny.  -1 = shape not taken.
int launch_gemm_skinny_fp8w(int dtype, const GemmArgs &g0, int ngroups, const void *const *Wq, const float *const *scales,
                            void *const *Cs, const int *Ns, cudaStream_t st) {
    if (ngroups < 1 || ngroups > SK_MAX_GROUPS) return -1;
    if (dtype != ITB_BF16 && dtype != ITB_F16) return -1;
    if (g0.batch != 1 || g0.trans_a || g0.trans_b || g0.m > 64 || g0.m < 1) return -1;
    if (g0.k % 16 != 0 || g0.k < 64 || !aligned16(g0.A)) return -1;
    for (int i = 0; i < ngroups; ++i)
        if (Ns[i] % 16 != 0 || Ns[i] < 64 || !aligned16(Wq[i]) || !scales[i] || ((uintptr_t)Cs[i] & 3)) return -1;
    const int mt = (g0.m + 15) / 16;
    GemmArgs gc = g0;
    gc.act |= ITB_MATMUL_B_CONST;  // quantised weights are constants by contract
#define SK8(TT)                                                                                            \
    do {                                                                                                   \
        if (mt == 1) return launch_skinny_w8_t<TT, 1>(gc, ngroups, Wq, Cs, Ns, scales, st);                \
        if (mt == 2) return launch_skinny_w8_t<TT, 2>(gc, ngroups, Wq, Cs, Ns, scales, st);                \
        return launch_skinny_w8_t<TT, 4>(gc, ngroups, Wq, Cs, Ns, scales, st);                             \
    } while (0)
    if (dtype == ITB_BF16) SK8(__nv_bfloat16);
    SK8(__half);
#undef SK8
}

}  // namespace itb

extern "C" void it_b200_tune_skinny(int nb, int splitk) {
    itb::g_nb_override = nb == 1 || nb == 2 ? nb : 0;
    itb::g_splitk_override = splitk > 0 ? splitk : 0;
}
