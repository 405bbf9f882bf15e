// attention_prefill.cu -- fused multi-token (prefill) attention on the Hopper tensor core (wgmma), sm_90a.
//
//   out[b,h] = softmax( (q[b,h] . k[b,h]^T) (/ or *) scale  + mask ) . v[b,h]        q, k, v, out: [B, H, S, D] f16 / bf16
//
// SURVEY 8(f-3).  The reference has no such kernel: its frontend lowers attention with q-len > 1 to
// Transpose -> MatMul -> Div -> Add(mask) -> Softmax -> MatMul (examples/python + pyinfinitensor/onnx.py; config C2, GPT-2),
// five launches of matmul.cc:66-211 / element_wise.cc / softmax.cu:242-404 per head group plus the [B,H,S,S] score tensor's
// round trips through HBM.  This kernel is the whole chain for one (batch, head, 128-query tile) per CTA:
//   * Q, K, V tiles arrive by TMA (3-D tensor maps over [B*H, S, D], 128B swizzle) into shared memory;
//   * S = Q K^T runs as wgmma (M = 128 queries, N = 128 keys, K = 16 per instruction, both operands K-major): each of the four
//     warpgroups computes one [64 queries x 64 keys] quarter in registers and parks it, rounded to the storage type (the
//     MatMul output rounding, the first thing every score applies), in shared memory;
//   * 512 threads: warp w owns query rows [32 (w & 3), +32), and the four warps sharing those rows split each
//     128-key tile into 32-column parts (w >> 2) -- one warp per scheduler, as in the first version (128 threads, a whole row
//     each), left every dependent exp / round chain exposed; the parts' running
//     (max, sum) meet once in shared memory after pass A.  Each thread reads its part of S back, applies the graph's own
//     rounding points (MatMul output, Div / Mul by the scalar, Add mask -- each rounded to the storage type like the separate
//     kernels), and the softmax: pass A accumulates the row maximum / sum over all key tiles (online), pass B recomputes S,
//     writes P = exp(s - max) / sum (rounded like the Softmax kernel's output) as the K-major A operand into shared memory
//     and the tensor core accumulates O += P V (V consumed as the MN-major B operand, straight from its [S, D] layout) in
//     the registers of D / 32 warpgroups, one [64 queries x 64 head columns] block each;
//   * O leaves the registers once, rounded to the storage type, through the same shared-memory tile as S.
// Two passes over K instead of rescaling O in registers: the extra QK^T costs 2 S^2 D flops on an idle tensor pipe, and the
// result needs no correction step -- the probabilities are final when they meet V.
// No causal shortcut: the mask is whatever tensor the graph adds (broadcast strides), so every graph the frontend emits is
// reproduced, not only triangular ones.
#include <cstring>

#include "gemm.cuh"

namespace itb {

constexpr int AP_BQ = 128, AP_BK = 128;
constexpr int AP_PARTS = 4, AP_PCOLS = AP_BK / AP_PARTS, AP_THREADS = 128 * AP_PARTS;
constexpr int AP_MPAD = AP_BQ + 2;  // 65 words per key column: the transposing store hits 32 distinct banks
constexpr int AP_SLD = AP_BQ + 8;   // parked S / O tile s_sm[column * AP_SLD + query row]: fragment stores spread over the banks

// this warpgroup's m64 x 64 fragment, rounded to T, as rows [row0, +64) x columns [col0, +64) of a parked tile
template <typename T>
__device__ __forceinline__ void ap_park(const float (&d)[32], T *dst, int row0, int col0) {
    const int w = (threadIdx.x >> 5) & 3, l = threadIdx.x & 31;
    const int r = row0 + 16 * w + (l >> 2), c = col0 + 2 * (l & 3);
#pragma unroll
    for (int j = 0; j < 8; ++j)
#pragma unroll
        for (int i = 0; i < 2; ++i)
#pragma unroll
            for (int e = 0; e < 2; ++e) dst[(8 * j + c + e) * AP_SLD + r + 8 * i] = from_f<T>(d[4 * j + 2 * i + e]);
}

struct ApArgs {
    int BH, H, Sq, Skv, D;
    const void *scale;      // device scalar (nullptr: none)
    int scale_is_div;       // 1: s / scale, 0: s * scale
    const void *mask;       // additive mask (nullptr: none), element (b, h, i, j) at mask[b*mb + h*mh + i*mi + j*mj]
    int64_t mb, mh, mi, mj;
    void *out;              // element (b, h, i, d) at out[b*ob + h*oh + i*os + d]  ([B, H, S, D] dense: ob = H*S*D, oh = S*D, os = D)
    int64_t ob, oh, os;
    // q / k / v tensor maps: 0 = 3-D over a dense [B*H, S, D]; 1 = 4-D with dimensions (d, h, s, b); 2 = 4-D (d, s, h, b) -- strided
    // views of e.g. a fused q/k/v projection output [B, S, 3 H D] (it_b200_attention_prefill_strided)
    int map_mode;
};

__device__ __forceinline__ void tma_load_4d(void *smem_dst, const CUtensorMap *m, uint64_t *bar, int c0, int c1, int c2, int c3,
                                            uint64_t policy) {
    asm volatile(
        "cp.async.bulk.tensor.4d.shared::cluster.global.mbarrier::complete_tx::bytes.L2::cache_hint"
        " [%0], [%1, {%3, %4, %5, %6}], [%2], %7;"
        ::"r"(smem_u32(smem_dst)), "l"(reinterpret_cast<uint64_t>(m)), "r"(smem_u32(bar)), "r"(c0), "r"(c1), "r"(c2), "r"(c3),
          "l"(policy)
        : "memory");
}

template <typename T, int D>
__global__ void __launch_bounds__(AP_THREADS, 1) attention_prefill_kernel(const __grid_constant__ CUtensorMap mapQ,
                                                                   const __grid_constant__ CUtensorMap mapK,
                                                                   const __grid_constant__ CUtensorMap mapV, const ApArgs a) {
    constexpr int DG = D / 64;                    // 64-column groups of the head dim
    constexpr int QK_BYTES = AP_BQ * D * 2;       // one Q or K tile (DG boxes of [128 rows x 64 cols])
    constexpr int V_BYTES = AP_BK * D * 2;        // one V tile (DG x 2 boxes of [64 kv rows x 64 cols])
    constexpr int P_BYTES = AP_BQ * AP_BK * 2;    // probabilities, two k-blocks of [128 rows x 64 keys]
    constexpr int M_BYTES = AP_BK * AP_MPAD * 2;  // mask tile
    extern __shared__ uint8_t ap_smem_raw[];
    uint8_t *smem = ap_smem_raw + ((1024u - (smem_u32(ap_smem_raw) & 1023u)) & 1023u);
    uint8_t *q_sm = smem, *k_sm = q_sm + QK_BYTES, *v_sm = k_sm + QK_BYTES, *p_sm = v_sm + V_BYTES;
    // the mask tile of the running (query tile, key tile), TRANSPOSED and padded: m_sm[j * AP_MPAD + i] -- every thread reads its own
    // query row i for consecutive keys j (lanes = consecutive i: conflict-free), the cooperative fill writes with lanes = keys
    T *m_sm = reinterpret_cast<T *>(p_sm + P_BYTES);
    T *s_sm = reinterpret_cast<T *>(p_sm + P_BYTES + M_BYTES);  // [128 columns][AP_SLD]: S of the running key tile, at the end O
    __shared__ __align__(8) uint64_t bar_load;
    __shared__ float red_m[AP_PARTS][AP_BQ], red_l[AP_PARTS][AP_BQ];

    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    const int bh = blockIdx.y, q0 = blockIdx.x * AP_BQ;
    const int quad = warp & 3, part = warp >> 2;
    const int row = quad * 32 + lane;  // query row inside the tile
    const int wg = warp >> 2, qh = wg & 1, ch = wg >> 1;  // this warpgroup's MMA block: query half, key / head-column half
    const int pc0 = part * AP_PCOLS;   // this thread's columns of every key tile: [pc0, pc0 + 32)
    pdl_trigger();
    if (threadIdx.x == 0) {
        mbar_init(&bar_load, 1);
        fence_mbar_init();
        tma_prefetch_desc(&mapQ);
        tma_prefetch_desc(&mapK);
        tma_prefetch_desc(&mapV);
    }
    __syncthreads();
    pdl_wait();

    const uint64_t pol = l2_policy_evict_last();
    uint32_t ph_load = 0;
    float o_acc[32];  // O block [64 queries (qh) x 64 head columns (ch)] of the first D / 32 warpgroups
#pragma unroll
    for (int j = 0; j < 32; ++j) o_acc[j] = 0.f;
    const bool o_owner = wg < D / 32;
    const int b = bh / a.H, h = bh % a.H;
    // one [rows x 64 columns] box of q / k / v: (column, sequence row) of head (b, h), whatever the tensor map's dimension order
    auto ld = [&](void *dst, const CUtensorMap *m, int c_d, int c_s) {
        if (a.map_mode == 0) tma_load_3d(dst, m, &bar_load, c_d, c_s, bh, pol);
        else if (a.map_mode == 1) tma_load_4d(dst, m, &bar_load, c_d, h, c_s, b, pol);
        else tma_load_4d(dst, m, &bar_load, c_d, c_s, h, b, pol);
    };

    // Q tile once -- together with the first K tile (and V when there is only one key tile): one round trip instead of three
    const int ntiles = (a.Skv + AP_BK - 1) / AP_BK;
    const bool single = ntiles == 1;  // one key tile (GPT-2's S = 128): K, V and the mask tile stay in shared memory for both passes
    if (threadIdx.x == 0) {
        mbar_expect_tx(&bar_load, QK_BYTES + (ntiles > 0 ? QK_BYTES : 0) + (single ? V_BYTES : 0));
#pragma unroll
        for (int g = 0; g < DG; ++g) ld(q_sm + g * (AP_BQ * 128), &mapQ, g * 64, q0);
        if (ntiles > 0)
#pragma unroll
            for (int g = 0; g < DG; ++g) ld(k_sm + g * (AP_BK * 128), &mapK, g * 64, 0);
        if (single)
#pragma unroll
            for (int g = 0; g < DG; ++g)
#pragma unroll
                for (int hh = 0; hh < 2; ++hh)
                    ld(v_sm + g * (AP_BK * 128) + hh * (64 * 128), &mapV, g * 64, hh * 64);
    }

    float sc = 1.f;
    if (a.scale) sc = to_f(*(const T *)a.scale);
    // s / 2^k == s * 2^-k exactly (GPT-2: sqrt(64)): spares a division per score and pass
    const bool div_pow2 = a.scale && a.scale_is_div && (__float_as_uint(sc) & 0x007fffffu) == 0u && sc != 0.f && fabsf(sc) < 1e30f && fabsf(sc) > 1e-30f;
    const float sc_mul = a.scale ? (a.scale_is_div ? (div_pow2 ? 1.f / sc : 0.f) : sc) : 1.f;
    const bool use_mul = a.scale && (!a.scale_is_div || div_pow2);
    const T *mbase = a.mask ? (const T *)a.mask + b * a.mb + h * a.mh : nullptr;
    const bool mvec = mbase && a.mj == 1 && (a.mi & 7) == 0 && (((uintptr_t)mbase & 15) == 0);
    // cooperative, coalesced fill of the mask tile (rows q0.., keys j0..): 16 threads cover one row's 128 keys with 16-byte loads
    auto load_mask = [&](int j0) {
        if (!mbase) return;
        const int jc = (threadIdx.x & 15) * 8, r0 = threadIdx.x >> 4;  // 32 rows per sweep
        // all four sweeps' loads in flight before the first transposing store (the stores may alias the mask as far as the
        // compiler knows: issued row by row, the dependent L2 round trips would dominate the tile)
        {
            constexpr int NSW = AP_BQ / (AP_THREADS / 16);
            uint4 buf[NSW];
#pragma unroll
            for (int i = 0; i < NSW; ++i) {
                const int r = r0 + (AP_THREADS / 16) * i;
                const bool rok = q0 + r < a.Sq;
                const T *src = mbase + (int64_t)(q0 + r) * a.mi + (int64_t)(j0 + jc) * a.mj;
                if (rok && mvec && j0 + jc + 8 <= a.Skv && ((((int64_t)(q0 + r) * a.mi + j0 + jc) & 7) == 0)) {
                    buf[i] = __ldg(reinterpret_cast<const uint4 *>(src));
                } else {
                    T vals[8];
#pragma unroll
                    for (int e = 0; e < 8; ++e) vals[e] = (rok && j0 + jc + e < a.Skv) ? src[(int64_t)e * a.mj] : from_f<T>(0.f);
                    buf[i] = *reinterpret_cast<const uint4 *>(vals);
                }
            }
#pragma unroll
            for (int i = 0; i < NSW; ++i) {
                const int r = r0 + (AP_THREADS / 16) * i;
                const T *vals = reinterpret_cast<const T *>(&buf[i]);
#pragma unroll
                for (int e = 0; e < 8; ++e) m_sm[(jc + e) * AP_MPAD + r] = vals[e];
            }
        }
    };
    const bool row_ok = q0 + row < a.Sq;

    // score of (this row, key j0 + c) from the raw accumulator value, with the graph's rounding points
    auto score = [&](float acc, int j) -> float {
        float s = round_t<T>(acc);                                      // MatMul output
        if (a.scale) s = round_t<T>(use_mul ? s * sc_mul : s / sc);  // Div / Mul by the scalar constant
        if (mbase && row_ok) s = round_t<T>(s + to_f(m_sm[(j % AP_BK) * AP_MPAD + row]));  // Add(mask)
        return s;
    };
    auto load_k = [&](int t) {
        if (threadIdx.x == 0) {
            mbar_expect_tx(&bar_load, QK_BYTES);
#pragma unroll
            for (int g = 0; g < DG; ++g) ld(k_sm + g * (AP_BK * 128), &mapK, g * 64, t * AP_BK);
        }
    };
    auto mma_s = [&]() {  // S = Q K^T, rounded to T, into s_sm: warpgroup (qh, ch) computes queries 64 qh.. x keys 64 ch..
        const uint32_t qb = smem_u32(q_sm) + qh * (64 * 128), kb = smem_u32(k_sm) + ch * (64 * 128);
        float d[32];
#pragma unroll
        for (int j = 0; j < 32; ++j) d[j] = 0.f;
        wg_fence();
#pragma unroll
        for (int kk = 0; kk < D / 16; ++kk) {
            const uint32_t off = (kk >> 2) * (128 * 128) + (kk & 3) * 32;
            Wgmma<T, 64>::template mma<0, 0>(d, gmma_desc_sw128(qb + off, 0, 1024), gmma_desc_sw128(kb + off, 0, 1024), 1u);
        }
        wg_commit();
        wg_wait<0>();
        ap_park<T>(d, s_sm, 64 * qh, 64 * ch);
    };
    // columns [c0, c0 + 16) of this thread's row of the parked tile
    auto ld_s = [&](int c0, uint32_t (&v)[16]) {
#pragma unroll
        for (int j = 0; j < 16; ++j) v[j] = __float_as_uint(to_f(s_sm[(c0 + j) * AP_SLD + row]));
    };

    // ---------------- pass A: row maximum and sum over all keys ----------------
    float m = -INFINITY, l = 0.f;
    if (ntiles == 0) {  // no keys: only Q was requested
        mbar_wait(&bar_load, ph_load);
        ph_load ^= 1;
    }
    for (int t = 0; t < ntiles; ++t) {
        if (t > 0) load_k(t);  // (tile 0 came with Q)
        const int j0 = t * AP_BK;
        load_mask(j0);  // (the previous tile's readers are behind the __syncthreads that closed it)
        mbar_wait(&bar_load, ph_load);
        ph_load ^= 1;
        mma_s();
        __syncthreads();  // mask tile and S complete
#pragma unroll 1
        for (int c0 = pc0; c0 < pc0 + AP_PCOLS; c0 += 16) {
            uint32_t v[16];
            ld_s(c0, v);
            float sv[16], mx = m;
#pragma unroll
            for (int j = 0; j < 16; ++j) {
                sv[j] = j0 + c0 + j < a.Skv ? score(__uint_as_float(v[j]), j0 + c0 + j) : -INFINITY;
                mx = fmaxf(mx, sv[j]);
            }
            if (mx > -INFINITY) {
                float add = 0.f;
#pragma unroll
                for (int j = 0; j < 16; ++j) add += expf(sv[j] - mx);  // exp(-inf) = 0
                l = l * expf(m - mx) + add;
                m = mx;
            }
        }
        __syncthreads();  // every row has read S before the next tile's MMA overwrites it (and K is reloaded)
    }
    // the four column parts of a row meet: global maximum, sums rescaled to it (same order for every part -> identical values)
    red_m[part][row] = m;
    red_l[part][row] = l;
    __syncthreads();
    {
        float mg = -INFINITY;
#pragma unroll
        for (int pp = 0; pp < AP_PARTS; ++pp) mg = fmaxf(mg, red_m[pp][row]);
        float lg = 0.f;
#pragma unroll
        for (int pp = 0; pp < AP_PARTS; ++pp) {
            const float mp = red_m[pp][row];
            if (mp > -INFINITY) lg += red_l[pp][row] * expf(mp - mg);
        }
        m = mg;
        l = lg;
    }
    const float inv_l = l > 0.f ? 1.f / l : 0.f;

    // ---------------- pass B: P = softmax row (final), O += P V ----------------
    for (int t = 0; t < ntiles; ++t) {
        if (threadIdx.x == 0 && !single) {
            mbar_expect_tx(&bar_load, QK_BYTES + V_BYTES);
#pragma unroll
            for (int g = 0; g < DG; ++g) ld(k_sm + g * (AP_BK * 128), &mapK, g * 64, t * AP_BK);
#pragma unroll
            for (int g = 0; g < DG; ++g)
#pragma unroll
                for (int hh = 0; hh < 2; ++hh)
                    ld(v_sm + g * (AP_BK * 128) + hh * (64 * 128), &mapV, g * 64, t * AP_BK + hh * 64);
        }
        const int j0 = t * AP_BK;
        if (!single) {
            load_mask(j0);  // (every reader of the previous tile's mask passed the __syncthreads before that tile's P.V)
            mbar_wait(&bar_load, ph_load);
            ph_load ^= 1;
        }
        if (!single) {  // (one key tile: S of pass A is still in shared memory)
            mma_s();
            __syncthreads();  // mask tile and S complete
        }
#pragma unroll 1
        for (int c0 = pc0; c0 < pc0 + AP_PCOLS; c0 += 16) {
            uint32_t v[16];
            ld_s(c0, v);
            T pv[16];
#pragma unroll
            for (int j = 0; j < 16; ++j) {
                float pr = 0.f;
                if (j0 + c0 + j < a.Skv && m > -INFINITY) pr = expf(score(__uint_as_float(v[j]), j0 + c0 + j) - m) * inv_l;
                pv[j] = from_f<T>(pr);  // the Softmax kernel's output rounding
            }
            // P is the K-major A operand of the second MMA: k-block = 64 keys, rows of 128 B, 128B swizzle
            uint8_t *blk = p_sm + (c0 >> 6) * (AP_BQ * 128) + row * 128;
            const int chunk = (c0 & 63) >> 3;  // first of the two 16-byte chunks these 16 keys fill
            *reinterpret_cast<uint4 *>(blk + (((chunk) ^ (row & 7)) << 4)) = *reinterpret_cast<const uint4 *>(&pv[0]);
            *reinterpret_cast<uint4 *>(blk + (((chunk + 1) ^ (row & 7)) << 4)) = *reinterpret_cast<const uint4 *>(&pv[8]);
        }
        fence_proxy_async();
        __syncthreads();
        if (o_owner) {
            // A = P: query half qh (8 KB in), k-block (kk >> 2), 32 B per k16 step inside the 128 B row;  B = V (MN-major): the
            // [keys x 64 head columns] group ch, 8-row key groups 1 KB apart (SBO), one k16 step = 16 key rows = 2 KB
            const uint32_t pb = smem_u32(p_sm) + qh * (64 * 128), vb = smem_u32(v_sm) + ch * (AP_BK * 128);
            wg_fence();
#pragma unroll
            for (int kk = 0; kk < AP_BK / 16; ++kk) {
                const uint64_t ad = gmma_desc_sw128(pb + (kk >> 2) * (AP_BQ * 128) + (kk & 3) * 32, 0, 1024);
                const uint64_t bd = gmma_desc_sw128(vb + kk * 2048, AP_BK * 128, 1024);
                Wgmma<T, 64>::template mma<0, 1>(o_acc, ad, bd, 1u);
            }
            wg_commit();
            wg_wait<0>();
        }
        __syncthreads();  // P, K, V are free again
    }
    if (o_owner) ap_park<T>(o_acc, s_sm, 64 * qh, 64 * ch);  // (every reader of S passed the barrier above)
    __syncthreads();

    // ---------------- epilogue: O row -> out ----------------
    T *orow = (T *)a.out + (int64_t)b * a.ob + (int64_t)h * a.oh + (int64_t)(q0 + row) * a.os;
#pragma unroll 1
    for (int c0 = part * (D / AP_PARTS); c0 < (part + 1) * (D / AP_PARTS); c0 += 16) {
        T ov[16];
#pragma unroll
        for (int j = 0; j < 16; ++j) ov[j] = s_sm[(c0 + j) * AP_SLD + row];
        if (row_ok) {
            *reinterpret_cast<uint4 *>(orow + c0) = *reinterpret_cast<const uint4 *>(&ov[0]);
            *reinterpret_cast<uint4 *>(orow + c0 + 8) = *reinterpret_cast<const uint4 *>(&ov[8]);
        }
    }
    (void)lane;
}

// strides of a q / k / v view in elements: {batch, head, sequence row}; the head dimension is contiguous
struct ApStrides {
    int64_t b, h, s;
};

template <typename T, int D>
static int launch_ap(const void *q, const void *k, const void *v, ApArgs a, cudaStream_t st, const ApStrides *sq = nullptr,
                     const ApStrides *sk = nullptr, const ApStrides *sv = nullptr) {
    CUtensorMap mq, mk, mv;
    // Skv = 0 launches no K / V load (every row is written as 0), but a tensor map cannot have an empty dimension: one row
    const int skv_map = a.Skv > 0 ? a.Skv : 1;
    if (!sq) {
        a.map_mode = 0;
        if (!make_tma_3d_b16(&mq, q, (uint64_t)a.BH, (uint64_t)a.Sq, (uint64_t)D, (uint64_t)D, (uint64_t)a.Sq * D, AP_BQ, 64) ||
            !make_tma_3d_b16(&mk, k, (uint64_t)a.BH, (uint64_t)skv_map, (uint64_t)D, (uint64_t)D, (uint64_t)skv_map * D, AP_BK, 64) ||
            !make_tma_3d_b16(&mv, v, (uint64_t)a.BH, (uint64_t)skv_map, (uint64_t)D, (uint64_t)D, (uint64_t)skv_map * D, 64, 64))
            ITB_FAIL("attention_prefill: cuTensorMapEncodeTiled failed");
    } else {
        // 4-D maps, dimensions ordered by stride (TMA wants them ascending): (d, h, s, b) when heads are the inner stride (a fused
        // projection's [B, S, H D] rows), (d, s, h, b) for [B, H, S, D]
        const int B = a.BH / a.H;
        const bool h_inner = sq->h < sq->s;
        ITB_CHECK((sk->h < sk->s) == h_inner && (sv->h < sv->s) == h_inner, "attention_prefill: q / k / v views must share a dimension order");
        a.map_mode = h_inner ? 1 : 2;
        auto mk4 = [&](CUtensorMap *m, const void *base, const ApStrides &t, int S, uint32_t box_s) {
            return h_inner ? make_tma_4d_b16(m, base, (uint64_t)D, (uint64_t)a.H, (uint64_t)S, (uint64_t)B, (uint64_t)t.h, (uint64_t)t.s,
                                             (uint64_t)t.b, 64, 1, box_s, 1)
                           : make_tma_4d_b16(m, base, (uint64_t)D, (uint64_t)S, (uint64_t)a.H, (uint64_t)B, (uint64_t)t.s, (uint64_t)t.h,
                                             (uint64_t)t.b, 64, box_s, 1, 1);
        };
        if (!mk4(&mq, q, *sq, a.Sq, AP_BQ) || !mk4(&mk, k, *sk, skv_map, AP_BK) || !mk4(&mv, v, *sv, skv_map, 64))
            ITB_FAIL("attention_prefill: cuTensorMapEncodeTiled (strided views) failed");
    }
    const int smem = 2 * AP_BQ * D * 2 + AP_BK * D * 2 + AP_BQ * AP_BK * 2 + AP_BK * AP_MPAD * 2 + AP_BK * AP_SLD * 2 + 1024;
    return launch("attention_prefill", attention_prefill_kernel<T, D>,
                  {dim3((a.Sq + AP_BQ - 1) / AP_BQ, a.BH), dim3(AP_THREADS), smem, st}, mq, mk, mv, a);
}

// ------------------------------------------------------------------------------------------------------------------
// AttentionKVCache over a prompt chunk of S > 1 tokens (it_b200_attention_kvcache_prompt): S single-token AttentionKVCache
// steps in order, token i of batch row b at position p_b + i.  Two launches, the second PDL-chained behind the first:
//   kvcache_append_kernel      copies k / v [B, Hkv, S, D] into cache rows [p_b, p_b + S), bit for bit;
//   attention_kvcache_prompt_kernel  one CTA (one warpgroup) per (batch row, query head, 64-query tile): causal attention
//                                    of the tile's queries over cache rows 0 .. p_b + i of KV head h / G.
// The attention kernel reads the cache only after griddepcontrol.wait, so every row it reads, the appended ones included,
// is complete; no CTA writes what another reads.  Per 64-key tile:
//   S = Q K^T   wgmma m64n64k16 (D / 16 steps, fp32 accumulators), Q and K by TMA (128B swizzle), scaled by fp32 1/sqrt(D)
//               like the decode kernels; key j of query i is kept when j <= p_b + i (only the diagonal tiles test it; key
//               tiles wholly past the tile's last query are never loaded);
//   softmax     online over the key tiles in fp32 (row max and sum across the 4 lanes of a fragment row);
//   O += P V    P enters the tensor core as hi = P rounded to T and lo = P - hi rounded to T, two wgmma chains into the
//               same fp32 accumulator (16 / 22 significant bits per weight for bf16 / f16, as attn_gqa_kernel keeps them);
//               V is the MN-major B operand straight from its [keys, D] tile.
// The output leaves the registers once, O / l rounded to T.  Query heads of one KV head run in separate CTAs (simpler
// than packing G heads x tokens into the M rows as attn_gqa_kernel does): each K / V tile is fetched once per query head,
// the repeats mostly from L2.  K / V tiles are double-buffered.
// ------------------------------------------------------------------------------------------------------------------
constexpr int PK_BQ = 64, PK_BK = 64, PK_THREADS = 128;

struct PkArgs {
    const void *pos;
    int pos_flags;  // ITB_I32 / ITB_U32 / ITB_I64 | ITB_POS_PER_ROW, row stride in bits ITB_POS_ROW_STRIDE_SHIFT..
    void *out;      // [B, Hq, S, D]
    int Hq, Hkv, G, S, Smax;
};

// p_b: element 0 of the positions, or (ITB_POS_PER_ROW) row b's first element at flat index b * stride; clamped to
// [0, Smax - S] so that rows [p_b, p_b + S) lie in the cache, or over a ring (ITB_POS_RING) to [0, ring_pos_max(Smax)]
__device__ __forceinline__ int prompt_start(const void *pos, int flags, int b, int S, int Smax, bool ring = false) {
    const int stride = max(flags >> ITB_POS_ROW_STRIDE_SHIFT, 1);
    const int64_t i = (flags & ITB_POS_PER_ROW) ? (int64_t)b * stride : 0;
    const int64_t p = (flags & 0xff) == ITB_I64 ? ((const int64_t *)pos)[i] : (int64_t)((const int32_t *)pos)[i];
    return (int)min(max(p, (int64_t)0), (int64_t)(ring ? ring_pos_max(Smax) : Smax - S));
}

// grid (ceil(S D / 8 / 256), B Hkv): one 16-byte chunk of k and of v per thread.  RING: token i goes to row (p_b + i) mod Smax
template <typename T, bool RING>
__device__ __forceinline__ void append_body(T *__restrict__ kc, T *__restrict__ vc, const T *__restrict__ k, const T *__restrict__ v,
                                            const void *pos, int pos_flags, int Hkv, int S, int Smax, int D) {
    pdl_trigger();
    pdl_wait();
    const int bh = blockIdx.y, b = bh / Hkv;
    const int64_t n = (int64_t)S * D / 8, c = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (c >= n) return;
    const int p = prompt_start(pos, pos_flags, b, S, Smax, RING);
    const int64_t src = (int64_t)bh * S * D / 8 + c;
    int64_t dst;
    if constexpr (RING) {
        const int i = (int)(c / (D / 8));  // the chunk's token
        dst = ((int64_t)bh * Smax + cache_row(p + i, Smax, true)) * D / 8 + c % (D / 8);
    } else {
        dst = ((int64_t)bh * Smax + p) * D / 8 + c;
    }
    reinterpret_cast<uint4 *>(kc)[dst] = reinterpret_cast<const uint4 *>(k)[src];
    reinterpret_cast<uint4 *>(vc)[dst] = reinterpret_cast<const uint4 *>(v)[src];
}
template <typename T>
__global__ void __launch_bounds__(256) kvcache_append_kernel(T *__restrict__ kc, T *__restrict__ vc, const T *__restrict__ k,
                                                             const T *__restrict__ v, const void *pos, int pos_flags, int Hkv,
                                                             int S, int Smax, int D) {
    append_body<T, false>(kc, vc, k, v, pos, pos_flags, Hkv, S, Smax, D);  // (pdl_trigger / pdl_wait inside)
}
template <typename T>
__global__ void __launch_bounds__(256) kvcache_append_ring_kernel(T *__restrict__ kc, T *__restrict__ vc, const T *__restrict__ k,
                                                                  const T *__restrict__ v, const void *pos, int pos_flags, int Hkv,
                                                                  int S, int Smax, int D) {
    append_body<T, true>(kc, vc, k, v, pos, pos_flags, Hkv, S, Smax, D);  // (pdl_trigger / pdl_wait inside)
}

// WIN (window >= 1): query i attends over rows (p_b + i - window, p_b + i] only.  Key tiles wholly below the tile's first query's
// window are never loaded; the leading edge is masked per element like the causal one
template <typename T, int D, bool WIN>
__device__ __forceinline__ void prompt_body(const CUtensorMap &mapQ, const CUtensorMap &mapK, const CUtensorMap &mapV,
                                            const PkArgs &a, int window) {
    constexpr int DG = D / 64;                  // 64-column groups of the head dim
    constexpr int TILE_BYTES = PK_BQ * D * 2;   // a Q, K or V tile: DG boxes of [64 rows x 64 columns], 128B swizzle
    constexpr int P_BYTES = PK_BQ * PK_BK * 2;  // P hi or lo: [64 queries x 64 keys], K-major, 128B swizzle
    constexpr float kScale = D == 128 ? 0.08838834764831845f : 0.125f;  // fp32 1/sqrt(D), as the decode kernels
    extern __shared__ uint8_t pk_smem_raw[];
    uint8_t *smem = pk_smem_raw + ((1024u - (smem_u32(pk_smem_raw) & 1023u)) & 1023u);
    uint8_t *q_sm = smem, *kv_sm = q_sm + TILE_BYTES;  // kv_sm: stage s = { K tile, V tile } at 2 s TILE_BYTES
    uint8_t *ph_sm = kv_sm + 4 * TILE_BYTES, *pl_sm = ph_sm + P_BYTES;
    __shared__ __align__(8) uint64_t bar_q, bar_kv[2];

    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    const int qt = gridDim.x - 1 - blockIdx.x;  // the longest (last) query tiles start first
    const int bh = blockIdx.y, b = bh / a.Hq, h = bh % a.Hq;
    const int kvh = b * a.Hkv + h / a.G;
    const int i0 = qt * PK_BQ;
    pdl_trigger();
    if (threadIdx.x == 0) {
        mbar_init(&bar_q, 1);
        mbar_init(&bar_kv[0], 1);
        mbar_init(&bar_kv[1], 1);
        fence_mbar_init();
        tma_prefetch_desc(&mapQ);
        tma_prefetch_desc(&mapK);
        tma_prefetch_desc(&mapV);
    }
    __syncthreads();
    pdl_wait();  // q / k / v and every cache row >= p_b are written in this step (the append launch)

    // (WIN) ITB_POS_RING: the caches are a ring, key tile t at row cache_row(64 t), one TMA box as Smax % 64 == 0.  Every
    // mask and limit below stays in positions.  Smax >= window + S - 1 (check_ring) keeps the positions the tile's queries
    // read in distinct rows; the first tile's rows below lo0 and the last tile's rows past p + S - 1 may hold other
    // positions (the chunk's own appends among them) and are made harmless like any rows outside the windows
    const bool ring = WIN && (a.pos_flags & ITB_POS_RING) != 0;
    const int p = prompt_start(a.pos, a.pos_flags, b, a.S, a.Smax, ring);
    const int last = p + min(i0 + PK_BQ - 1, a.S - 1);  // the tile's last query attends over rows 0 .. last
    const int nkt = last / PK_BK + 1;
    const int lo0 = WIN ? max(p + i0 - window + 1, 0) : 0;  // the first row of the tile's first query's window
    const int t0 = lo0 / PK_BK;                              // the first key tile loaded; tile t uses stage (t - t0) & 1
    const uint64_t pol = l2_policy_evict_last();
    auto load_kv = [&](int t) {
        const int sg = (t - t0) & 1;
        uint8_t *ks = kv_sm + sg * 2 * TILE_BYTES, *vs = ks + TILE_BYTES;
        mbar_expect_tx(&bar_kv[sg], 2 * TILE_BYTES);
#pragma unroll
        for (int g = 0; g < DG; ++g) {
            tma_load_3d(ks + g * (PK_BK * 128), &mapK, &bar_kv[sg], g * 64, cache_row(t * PK_BK, a.Smax, ring), kvh, pol);
            tma_load_3d(vs + g * (PK_BK * 128), &mapV, &bar_kv[sg], g * 64, cache_row(t * PK_BK, a.Smax, ring), kvh, pol);
        }
    };
    if (threadIdx.x == 0) {
        mbar_expect_tx(&bar_q, TILE_BYTES);
#pragma unroll
        for (int g = 0; g < DG; ++g) tma_load_3d(q_sm + g * (PK_BQ * 128), &mapQ, &bar_q, g * 64, i0, bh, pol);
        load_kv(t0);
    }

    // accumulator fragment: d[4 j + 2 r + e] is row 16 warp + lane / 4 + 8 r, column 8 j + 2 (lane % 4) + e
    const int fr = 16 * warp + (lane >> 2), fc = 2 * (lane & 3);
    int lim[2];  // per fragment row: the last key it attends to (rows past S behave like row S - 1; they are not stored)
#pragma unroll
    for (int r = 0; r < 2; ++r) lim[r] = p + min(i0 + fr + 8 * r, a.S - 1);
    float o[DG][32];
#pragma unroll
    for (int g = 0; g < DG; ++g)
#pragma unroll
        for (int j = 0; j < 32; ++j) o[g][j] = 0.f;
    float m[2] = {-INFINITY, -INFINITY}, l[2] = {0.f, 0.f};
    mbar_wait(&bar_q, 0);

    for (int t = t0; t < nkt; ++t) {
        if (threadIdx.x == 0 && t + 1 < nkt) load_kv(t + 1);  // (stage (t + 1 - t0) & 1 was released by the barrier closing t - 1)
        const int sg = (t - t0) & 1;
        uint8_t *ks = kv_sm + sg * 2 * TILE_BYTES, *vs = ks + TILE_BYTES;
        mbar_wait(&bar_kv[sg], ((t - t0) >> 1) & 1);
        const int j0 = t * PK_BK;
        // V rows past p_b + S - 1 (the last tile only) are cache contents this step does not own, possibly non-finite: they
        // meet P = 0 in the product, so they are zeroed here
        if (j0 + PK_BK > p + a.S) {
            const int r0 = p + a.S - j0;
            for (int c = threadIdx.x; c < (PK_BK - r0) * DG * 8; c += PK_THREADS) {
                const int r = r0 + c / (DG * 8), g = (c / 8) % DG, ch = c % 8;
                *reinterpret_cast<uint4 *>(vs + g * (PK_BK * 128) + r * 128 + ch * 16) = make_uint4(0, 0, 0, 0);
            }
            fence_proxy_async();
        }
        // likewise V rows below the first query's window (the first tile only): no query of the tile attends to them
        if (WIN && j0 < lo0) {
            for (int c = threadIdx.x; c < (lo0 - j0) * DG * 8; c += PK_THREADS) {
                const int r = c / (DG * 8), g = (c / 8) % DG, ch = c % 8;
                *reinterpret_cast<uint4 *>(vs + g * (PK_BK * 128) + r * 128 + ch * 16) = make_uint4(0, 0, 0, 0);
            }
            fence_proxy_async();
        }

        float s[32];
#pragma unroll
        for (int j = 0; j < 32; ++j) s[j] = 0.f;
        wg_fence();
#pragma unroll
        for (int kk = 0; kk < D / 16; ++kk) {
            const uint32_t off = (kk >> 2) * (PK_BK * 128) + (kk & 3) * 32;
            Wgmma<T, 64>::template mma<0, 0>(s, gmma_desc_sw128(smem_u32(q_sm) + off, 0, 1024),
                                             gmma_desc_sw128(smem_u32(ks) + off, 0, 1024), 1u);
        }
        wg_commit();
        wg_wait<0>();

        const bool diag = j0 + PK_BK - 1 > p + i0;  // some key of the tile lies past the first query's limit
        const bool lead = WIN && j0 <= last - window;  // some key of the tile lies below the last query's window
#pragma unroll
        for (int r = 0; r < 2; ++r) {
            float mx = m[r];
#pragma unroll
            for (int j = 0; j < 8; ++j)
#pragma unroll
                for (int e = 0; e < 2; ++e) {
                    float &x = s[4 * j + 2 * r + e];
                    const int key = j0 + 8 * j + fc + e;
                    x = ((diag && key > lim[r]) || (lead && key <= lim[r] - window)) ? -INFINITY : x * kScale;
                    mx = fmaxf(mx, x);
                }
            mx = fmaxf(mx, __shfl_xor_sync(0xffffffffu, mx, 1));
            mx = fmaxf(mx, __shfl_xor_sync(0xffffffffu, mx, 2));  // unwindowed, finite: key 0 of tile 0 is in every row
            // windowed, a row may have met only masked keys so far (m = mx = -inf): its exponentials subtract 0 instead, so
            // that its weights and the correction stay 0 rather than exp(-inf + inf) = NaN, and m stays -inf
            const float mxe = WIN && mx == -INFINITY ? 0.f : mx;
            const int prow = fr + 8 * r;
            uint8_t *hrow = ph_sm + prow * 128, *lrow = pl_sm + prow * 128;
            float sum = 0.f;
#pragma unroll
            for (int j = 0; j < 8; ++j) {
                __align__(4) T hi[2], lo[2];
#pragma unroll
                for (int e = 0; e < 2; ++e) {
                    const float pr = expf(s[4 * j + 2 * r + e] - mxe);  // masked: exp(-inf) = 0
                    hi[e] = from_f<T>(pr);
                    lo[e] = from_f<T>(pr - to_f(hi[e]));
                    sum += pr;
                }
                // K-major A operand, 128B swizzle: key c of row prow at 16-byte chunk (c / 8) ^ (prow % 8)
                const int boff = (((j ^ (prow & 7)) << 4)) + 2 * fc;
                *reinterpret_cast<uint32_t *>(hrow + boff) = *reinterpret_cast<const uint32_t *>(hi);
                *reinterpret_cast<uint32_t *>(lrow + boff) = *reinterpret_cast<const uint32_t *>(lo);
            }
            sum += __shfl_xor_sync(0xffffffffu, sum, 1);
            sum += __shfl_xor_sync(0xffffffffu, sum, 2);
            const float corr = expf(m[r] - mxe);  // m = -inf (first tile): 0, and o, l are still 0
            l[r] = l[r] * corr + sum;
            m[r] = mx;
#pragma unroll
            for (int g = 0; g < DG; ++g)
#pragma unroll
                for (int j = 0; j < 8; ++j) {
                    o[g][4 * j + 2 * r] *= corr;
                    o[g][4 * j + 2 * r + 1] *= corr;
                }
        }
        fence_proxy_async();
        __syncthreads();  // P complete (and the zeroed V rows visible to the tensor core)
        wg_fence();
#pragma unroll
        for (int g = 0; g < DG; ++g) {
            // B = V (MN-major): the [64 keys x 64 head columns] box g, 8-key groups 1 KB apart, one k16 step = 16 keys = 2 KB
            const uint32_t vb = smem_u32(vs) + g * (PK_BK * 128);
#pragma unroll
            for (int kk = 0; kk < PK_BK / 16; ++kk)
                Wgmma<T, 64>::template mma<0, 1>(o[g], gmma_desc_sw128(smem_u32(ph_sm) + kk * 32, 0, 1024),
                                                 gmma_desc_sw128(vb + kk * 2048, PK_BK * 128, 1024), 1u);
#pragma unroll
            for (int kk = 0; kk < PK_BK / 16; ++kk)
                Wgmma<T, 64>::template mma<0, 1>(o[g], gmma_desc_sw128(smem_u32(pl_sm) + kk * 32, 0, 1024),
                                                 gmma_desc_sw128(vb + kk * 2048, PK_BK * 128, 1024), 1u);
        }
        wg_commit();
        wg_wait<0>();
        __syncthreads();  // P and this K / V stage are free again
    }

    T *obase = (T *)a.out + ((int64_t)bh * a.S + i0) * D;
#pragma unroll
    for (int r = 0; r < 2; ++r) {
        const int row = fr + 8 * r;
        if (i0 + row >= a.S) continue;
        const float inv = 1.f / l[r];
#pragma unroll
        for (int g = 0; g < DG; ++g)
#pragma unroll
            for (int j = 0; j < 8; ++j) {
                __align__(4) T ov[2] = {from_f<T>(o[g][4 * j + 2 * r] * inv), from_f<T>(o[g][4 * j + 2 * r + 1] * inv)};
                *reinterpret_cast<uint32_t *>(obase + (int64_t)row * D + g * 64 + 8 * j + fc) = *reinterpret_cast<const uint32_t *>(ov);
            }
    }
}

template <typename T, int D>
__global__ void __launch_bounds__(PK_THREADS, 1) attention_kvcache_prompt_kernel(const __grid_constant__ CUtensorMap mapQ,
                                                                                 const __grid_constant__ CUtensorMap mapK,
                                                                                 const __grid_constant__ CUtensorMap mapV,
                                                                                 const PkArgs a) {
    prompt_body<T, D, false>(mapQ, mapK, mapV, a, 0);  // (pdl_trigger / pdl_wait inside)
}
template <typename T, int D>
__global__ void __launch_bounds__(PK_THREADS, 1) attention_kvcache_prompt_win_kernel(const __grid_constant__ CUtensorMap mapQ,
                                                                                     const __grid_constant__ CUtensorMap mapK,
                                                                                     const __grid_constant__ CUtensorMap mapV,
                                                                                     const PkArgs a, int window) {
    prompt_body<T, D, true>(mapQ, mapK, mapV, a, window);  // (pdl_trigger / pdl_wait inside)
}

template <typename T, int D>
static int launch_prompt(void *kc, void *vc, const void *q, const void *k, const void *v, const PkArgs &a, int B, int window,
                         cudaStream_t st) {
    const int64_t chunks = (int64_t)a.S * D / 8;
    if (launch("AttentionKVCache prompt: append",
               (a.pos_flags & ITB_POS_RING) ? kvcache_append_ring_kernel<T> : kvcache_append_kernel<T>,
               {dim3((unsigned)((chunks + 255) / 256), B * a.Hkv), dim3(256), 0, st}, (T *)kc, (T *)vc, (const T *)k, (const T *)v,
               a.pos, a.pos_flags, a.Hkv, a.S, a.Smax, D))
        return 1;
    CUtensorMap mq, mk, mv;
    if (!make_tma_3d_b16(&mq, q, (uint64_t)B * a.Hq, (uint64_t)a.S, D, D, (uint64_t)a.S * D, PK_BQ, 64) ||
        !make_tma_3d_b16(&mk, kc, (uint64_t)B * a.Hkv, (uint64_t)a.Smax, D, D, (uint64_t)a.Smax * D, PK_BK, 64) ||
        !make_tma_3d_b16(&mv, vc, (uint64_t)B * a.Hkv, (uint64_t)a.Smax, D, D, (uint64_t)a.Smax * D, PK_BK, 64))
        ITB_FAIL("AttentionKVCache prompt: cuTensorMapEncodeTiled failed");
    const int smem = 5 * PK_BQ * D * 2 + 2 * PK_BQ * PK_BK * 2 + 1024;
    if (window > 0)
        return launch("AttentionKVCache prompt (window)", attention_kvcache_prompt_win_kernel<T, D>,
                      {dim3((a.S + PK_BQ - 1) / PK_BQ, B * a.Hq), dim3(PK_THREADS), smem, st}, mq, mk, mv, a, window);
    return launch("AttentionKVCache prompt", attention_kvcache_prompt_kernel<T, D>,
                  {dim3((a.S + PK_BQ - 1) / PK_BQ, B * a.Hq), dim3(PK_THREADS), smem, st}, mq, mk, mv, a);
}

}  // namespace itb

using namespace itb;

extern "C" int it_b200_attention_prefill(int dtype, const void *q, const void *k, const void *v, void *out, int B, int H, int S_q,
                                         int S_kv, int D, const void *scale, int scale_is_div, const void *mask,
                                         int64_t mask_stride_b, int64_t mask_stride_h, int64_t mask_stride_i,
                                         int64_t mask_stride_j, void *stream) {
    ITB_CHECK(dtype == ITB_F16 || dtype == ITB_BF16, "attention_prefill: dtype %d must be f16 / bf16", dtype);
    ITB_CHECK(D == 64 || D == 128, "attention_prefill: head dim %d must be 64 or 128", D);
    ITB_CHECK(B >= 0 && H >= 0 && S_q >= 0 && S_kv >= 0, "attention_prefill: negative dimension");
    ITB_CHECK((int64_t)B * H <= 65535, "attention_prefill: B * H beyond the grid limit");
    if ((int64_t)B * H * S_q == 0) return 0;
    ITB_CHECK(aligned16(q) && aligned16(k) && aligned16(v) && aligned16(out), "attention_prefill: tensors must be 16-byte aligned");
    ApArgs a{};
    a.BH = B * H;
    a.H = H;
    a.Sq = S_q;
    a.Skv = S_kv;
    a.D = D;
    a.scale = scale;
    a.scale_is_div = scale_is_div;
    a.mask = mask;
    a.mb = mask_stride_b;
    a.mh = mask_stride_h;
    a.mi = mask_stride_i;
    a.mj = mask_stride_j;
    a.out = out;
    a.ob = (int64_t)H * S_q * D;
    a.oh = (int64_t)S_q * D;
    a.os = D;
    auto st = (cudaStream_t)stream;
    if (dtype == ITB_BF16) return D == 64 ? launch_ap<__nv_bfloat16, 64>(q, k, v, a, st) : launch_ap<__nv_bfloat16, 128>(q, k, v, a, st);
    return D == 64 ? launch_ap<__half, 64>(q, k, v, a, st) : launch_ap<__half, 128>(q, k, v, a, st);
}

// The same attention over STRIDED views: element (b, h, i, d) of q at q[b*qs[0] + h*qs[1] + i*qs[2] + d] (likewise k, v, out) -- the
// frontend's Split -> Reshape -> Transpose([0,2,1,3]) of a fused q/k/v projection and the Transpose -> Reshape after the attention
// become addressing (4-D tensor maps, strided output rows) instead of five copy kernels per layer.
extern "C" int it_b200_attention_prefill_strided(int dtype, const void *q, const void *k, const void *v, void *out, int B, int H,
                                                 int S_q, int S_kv, int D, const int64_t *q_strides, const int64_t *k_strides,
                                                 const int64_t *v_strides, const int64_t *out_strides, const void *scale,
                                                 int scale_is_div, const void *mask, int64_t mask_stride_b, int64_t mask_stride_h,
                                                 int64_t mask_stride_i, int64_t mask_stride_j, void *stream) {
    ITB_CHECK(dtype == ITB_F16 || dtype == ITB_BF16, "attention_prefill: dtype %d must be f16 / bf16", dtype);
    ITB_CHECK(D == 64 || D == 128, "attention_prefill: head dim %d must be 64 or 128", D);
    ITB_CHECK(B >= 0 && H >= 0 && S_q >= 0 && S_kv >= 0, "attention_prefill: negative dimension");
    ITB_CHECK((int64_t)B * H <= 65535, "attention_prefill: B * H beyond the grid limit");
    if ((int64_t)B * H * S_q == 0) return 0;
    ITB_CHECK(aligned16(q) && aligned16(k) && aligned16(v) && aligned16(out), "attention_prefill: tensors must be 16-byte aligned");
    for (int i = 0; i < 3; ++i)
        ITB_CHECK(q_strides[i] % 8 == 0 && k_strides[i] % 8 == 0 && v_strides[i] % 8 == 0 && out_strides[i] % 8 == 0 && q_strides[i] > 0 &&
                      k_strides[i] > 0 && v_strides[i] > 0,
                  "attention_prefill: view strides must be positive multiples of 8 elements");
    ApArgs a{};
    a.BH = B * H;
    a.H = H;
    a.Sq = S_q;
    a.Skv = S_kv;
    a.D = D;
    a.scale = scale;
    a.scale_is_div = scale_is_div;
    a.mask = mask;
    a.mb = mask_stride_b;
    a.mh = mask_stride_h;
    a.mi = mask_stride_i;
    a.mj = mask_stride_j;
    a.out = out;
    a.ob = out_strides[0];
    a.oh = out_strides[1];
    a.os = out_strides[2];
    const ApStrides sq{q_strides[0], q_strides[1], q_strides[2]}, sk{k_strides[0], k_strides[1], k_strides[2]},
        sv{v_strides[0], v_strides[1], v_strides[2]};
    auto st = (cudaStream_t)stream;
    if (dtype == ITB_BF16)
        return D == 64 ? launch_ap<__nv_bfloat16, 64>(q, k, v, a, st, &sq, &sk, &sv) : launch_ap<__nv_bfloat16, 128>(q, k, v, a, st, &sq, &sk, &sv);
    return D == 64 ? launch_ap<__half, 64>(q, k, v, a, st, &sq, &sk, &sv) : launch_ap<__half, 128>(q, k, v, a, st, &sq, &sk, &sv);
}

// AttentionKVCache over S >= 1 new tokens per batch row (S = 1 is one decode step, served by the same two launches); window >= 1
// limits query i to rows (p_b + i - window, p_b + i]
static int prompt_impl(int dtype, void *k_cache, void *v_cache, const void *q, const void *k, const void *v, const void *position_id,
                       int pos_flags, void *out, int B, int Hq, int Hkv, int S, int S_max, int D, int window, void *stream) {
    ITB_CHECK(dtype == ITB_F16 || dtype == ITB_BF16, "AttentionKVCache prompt: dtype %d must be f16 / bf16 (no fp32 prefill)", dtype);
    ITB_CHECK(D == 64 || D == 128, "AttentionKVCache prompt: head dim %d must be 64 or 128", D);
    const int pos_dtype = pos_flags & 0xff;
    ITB_CHECK(pos_dtype == ITB_I32 || pos_dtype == ITB_U32 || pos_dtype == ITB_I64,
              "AttentionKVCache prompt: position dtype %d must be int32/uint32/int64", pos_dtype);
    ITB_CHECK(window > 0 || !(pos_flags & ITB_POS_RING),
              "AttentionKVCache prompt: a rolling cache (ITB_POS_RING) needs a window: it_b200_attention_kvcache_prompt_window");
    ITB_CHECK(B >= 0 && Hq >= 0 && S >= 1 && S <= S_max, "AttentionKVCache prompt: %d tokens do not fit a cache of %d rows", S, S_max);
    ITB_CHECK(Hkv > 0 && Hq % Hkv == 0, "AttentionKVCache prompt: %d query heads are not a multiple of %d KV heads", Hq, Hkv);
    ITB_CHECK((int64_t)B * Hq <= 65535 && (int64_t)B * Hkv <= 65535, "AttentionKVCache prompt: batch x heads beyond the grid limit");
    if ((int64_t)B * Hq == 0) return 0;
    ITB_CHECK(aligned16(k_cache) && aligned16(v_cache) && aligned16(q) && aligned16(k) && aligned16(v) && aligned16(out),
              "AttentionKVCache prompt: tensors must be 16-byte aligned");
    PkArgs a{};
    a.pos = position_id;
    a.pos_flags = pos_flags;
    a.out = out;
    a.Hq = Hq;
    a.Hkv = Hkv;
    a.G = Hq / Hkv;
    a.S = S;
    a.Smax = S_max;
    auto st = (cudaStream_t)stream;
    if (dtype == ITB_BF16)
        return D == 64 ? launch_prompt<__nv_bfloat16, 64>(k_cache, v_cache, q, k, v, a, B, window, st)
                       : launch_prompt<__nv_bfloat16, 128>(k_cache, v_cache, q, k, v, a, B, window, st);
    return D == 64 ? launch_prompt<__half, 64>(k_cache, v_cache, q, k, v, a, B, window, st)
                   : launch_prompt<__half, 128>(k_cache, v_cache, q, k, v, a, B, window, st);
}

extern "C" int it_b200_attention_kvcache_prompt(int dtype, void *k_cache, void *v_cache, const void *q, const void *k,
                                                const void *v, const void *position_id, int pos_flags, void *out, int B,
                                                int Hq, int Hkv, int S, int S_max, int D, void *stream) {
    return prompt_impl(dtype, k_cache, v_cache, q, k, v, position_id, pos_flags, out, B, Hq, Hkv, S, S_max, D, 0, stream);
}

extern "C" int it_b200_attention_kvcache_prompt_window(int dtype, void *k_cache, void *v_cache, const void *q, const void *k,
                                                       const void *v, const void *position_id, int pos_flags, void *out, int B,
                                                       int Hq, int Hkv, int S, int S_max, int D, int window, void *stream) {
    ITB_CHECK(window >= 0, "AttentionKVCache prompt: window %d is negative", window);
    if ((pos_flags & ITB_POS_RING) && check_ring("AttentionKVCache prompt", window, S_max, S)) return 1;
    return prompt_impl(dtype, k_cache, v_cache, q, k, v, position_id, pos_flags, out, B, Hq, Hkv, S, S_max, D, window, stream);
}
