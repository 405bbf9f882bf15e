// attention.cu -- AttentionKVCache decode kernel (q-len 1) for sm_90a.
//
// Replaces reference _attention_kvcache_kernel_128_1/_2 (src/kernels/cuda/attention_kvcache.cu:8-169,
// wrapper attention_kvcache.cc:8-56).  Contract kept from the reference:
//   * seq_length = position_id[0] + 1 for every batch row (.cu:17) -- unless the caller asks for PER-ROW positions
//     (ITB_POS_PER_ROW: row b attends to position_id[b] + 1 rows and appends at position_id[b]; SURVEY 8(f-3): ragged
//     batches cannot be served with the reference's element-0 rule)
//   * k, v are appended IN PLACE into the cache INPUT tensors at position_id[0] (.cu:49-53, 89-93)
//   * cache layout [B, H, S_max, D] contiguous; q/k/v/out [B, H, 1, D]; scale 1/sqrt(D) -- the reference's 1/sqrt(128)
//     (.cu:72) at D = 128, the only width it has; D = 64 (GPT-2, TinyLlama) is an extension with the same rule
// Differences by design (DESIGN.md): numerically stable online softmax instead of the reference's
// exp without max-subtraction (same mathematics; quirk q1), f16/bf16 caches in addition to fp32,
// no 2 GiB scratch round trip -- a single kernel when B*H alone fills the 132 SMs.
//
// HBM-bound: every K and V row up to position p is read exactly once with 128-bit loads; a warp
// holds RPW = 32/LPR rows per load instruction (LPR = lanes per D-wide row: D/8 for 2-byte types,
// D/4 for fp32), U independent K and V loads are issued before any arithmetic so each lane keeps
// 2*U 16-byte requests in flight.
#include <algorithm>
#include <string>
#include <type_traits>

#include "common.cuh"
#include "gemm.cuh"  // mbarrier / bulk-copy PTX helpers

namespace itb {

template <typename T, int D> struct RowCfg {
    static_assert(D == 64 || D == 128, "decode attention: head width 64 or 128");
    static constexpr int EPL = 16 / sizeof(T);  // elements per lane per row
    static constexpr int LPR = D / EPL;         // lanes per row
    static constexpr int RPW = 32 / LPR;        // rows per warp-load
};

// softmax scale 1/sqrt(D) as an fp32 constant: 1/sqrt(128) rounded to fp32, 1/8 exactly
template <int D> __host__ __device__ constexpr float attn_scale() { return D == 128 ? 0.08838834764831845f : 0.125f; }

template <typename P> __device__ __forceinline__ int read_pos(const void *p, int i) { return (int)((const P *)p)[i]; }
// a windowed body's position i: narrowed, then clamped to [0, Smax - 1] over a linear cache (the unwindowed rule); over a
// ring (ITB_POS_RING) clamped to [0, ring_pos_max(Smax)] first, so that an int64 position is never wrapped by the narrowing
__device__ __forceinline__ int win_pos(const void *position_id, int pos_dtype, int i, int Smax, bool ring) {
    int64_t p = pos_dtype == ITB_I64 ? ((const int64_t *)position_id)[i] : (int64_t)read_pos<int32_t>(position_id, i);
    if (!ring) p = (int)p;
    return (int)min(max(p, (int64_t)0), (int64_t)(ring ? ring_pos_max(Smax) : Smax - 1));
}
// a windowed body's bulk copy of `rows` K and V rows from position `p0` of cache head `head` into a ring stage (K at dst, V
// at dst + chunk_bytes), completing `bytes` = rows x D x sizeof(KT) on `bar` each.  Over a ring, a run of rows that crosses
// the ring's end is two copies into consecutive addresses of the stage: both pieces are whole rows of D x sizeof(KT) >= 64
// bytes, so they stay 16-byte aligned multiples of 16 bytes, and the stage's transaction count is unchanged
template <typename KT, int D>
__device__ __forceinline__ void win_chunk_load(unsigned char *dst, int chunk_bytes, const KT *kcache, const KT *vcache, int64_t head,
                                               int Smax, int p0, int rows, bool ring, uint64_t *bar, uint64_t policy) {
    const uint32_t bytes = (uint32_t)rows * D * (uint32_t)sizeof(KT);
    const int r0 = cache_row(p0, Smax, ring);
    const uint32_t b0 = (uint32_t)min(rows, Smax - r0) * D * (uint32_t)sizeof(KT);  // rows before the ring's end
    const int64_t off = (head * Smax + r0) * D, wrap = head * Smax * D;
    mbar_expect_tx(bar, 2 * bytes);
    bulk_load_1d(dst, kcache + off, b0, bar, policy);
    if (b0 < bytes) bulk_load_1d(dst + b0, kcache + wrap, bytes - b0, bar, policy);
    bulk_load_1d(dst + chunk_bytes, vcache + off, b0, bar, policy);
    if (b0 < bytes) bulk_load_1d(dst + chunk_bytes + b0, vcache + wrap, bytes - b0, bar, policy);
}

// ------------------------------------------------------------------------------------------------------------------
// attn_stream_kernel: the production decode kernel.  Same arithmetic per cache row as attn_decode_kernel, but
//   * the (head, 64-row chunk) work units of the whole batch are FLATTENED and dealt out in equal contiguous ranges to
//     a persistent grid of 2 x 132 CTAs -- a head count that is not a multiple of the CTA slots no longer costs a
//     partly filled last wave, as a split-per-head grid does;
//   * every chunk of K rows and of V rows is ONE contiguous 16 KiB range of the cache ([B,H,S,D] layout), so a
//     producer warp streams it HBM -> shared memory with cp.async.bulk (TMA 1-D) through a full/empty mbarrier ring;
//     bytes in flight are set by the ring depth (2 x 32 KiB per CTA), not by registers per thread;
//   * a head whose units straddle two or three CTAs is finished by the LAST of them to arrive (self-cleaning ticket per
//     head), which merges the (m, l, acc) partials in CTA order -- deterministic, no second kernel.
// The in-place append and the appended row's contribution are done by the CTA that owns the head's last chunk, from
// registers; chunk loads stop at row pos-1, so the append never races the bulk reads.
// FP8 E4M3 caches (KT = uint8_t, attn_stream_kv8_kernel): a lane holds 16 codes of a row (one 16-byte load) and widens
// them in registers before the fp32 dot products, so a 16 KiB chunk holds twice the rows of a 16-bit one and the ring's
// bytes in flight are unchanged.  K's scale folds into q with 1/sqrt(D); V's scales the normalised output once.
// ------------------------------------------------------------------------------------------------------------------
constexpr int AS_STAGES = 2;  // ring depth
constexpr int AS_CTAS_PER_SM = 2;

// rotate-half RoPE of one lane's EPL columns: the partner half of the row is LPR / 2 lanes away
template <typename T, int D, int EPL, int LPR>
__device__ __forceinline__ void rope_one(Vec16<T> &x, int col, const float *cs_t, const float *sn_t) {
    Vec16<T> xp;
    {
        uint4 mine = *reinterpret_cast<const uint4 *>(x.v), other;
        other.x = __shfl_xor_sync(0xffffffffu, mine.x, LPR / 2);
        other.y = __shfl_xor_sync(0xffffffffu, mine.y, LPR / 2);
        other.z = __shfl_xor_sync(0xffffffffu, mine.z, LPR / 2);
        other.w = __shfl_xor_sync(0xffffffffu, mine.w, LPR / 2);
        *reinterpret_cast<uint4 *>(xp.v) = other;
    }
    const bool lo = col < D / 2;
#pragma unroll
    for (int j = 0; j < EPL; ++j) {
        const int c = (col + j) & (D / 2 - 1);
        // each product rounded on its own (__fmul_rn: never fused into the sum), as the RoPE kernel does
        const float a = round_t<T>(__fmul_rn(to_f(x.v[j]), cs_t[c])), b = round_t<T>(__fmul_rn(to_f(xp.v[j]), sn_t[c]));
        x.v[j] = from_f<T>(lo ? a - b : a + b);
    }
}

// RoPE folded into the decode attention: none, the base-10000 rule, or the angle p x inv_freq[c] from a table of the model's
// frequencies (RoPE's optional inv_freq input, f32 [D / 2])
enum RopeMode : int { ROPE_NONE = 0, ROPE_BASE = 1, ROPE_TABLE = 2 };

// the cache holds FP8 E4M3 codes.  A namespace-scope constant: a constexpr local in the attention bodies would change how
// their unquantised instantiations compile
template <typename KT> constexpr bool KV8 = std::is_same_v<KT, uint8_t>;

// FP8 E4M3 KV cache (cache element type uint8_t; an element's value is e4m3(code) * scale[KV head]).  Every E4M3 value is exact
// in f16, so codes widen through cvt.rn.f16x2.e4m3x2 with no loss, for bf16 activations too; scales enter only in fp32.
// 16 codes (one 16-byte load) -> 16 fp32 values
__device__ __forceinline__ void e4m3x16_to_f(const uint4 raw, float (&f)[16]) {
    const uint32_t w[4] = {raw.x, raw.y, raw.z, raw.w};
#pragma unroll
    for (int i = 0; i < 4; ++i)
#pragma unroll
        for (int h = 0; h < 2; ++h) {
            const uint32_t h2 = e4m3x2_to<__half>(w[i] >> (16 * h));
            const float2 x = __half22float2(*reinterpret_cast<const __half2 *>(&h2));
            f[4 * i + 2 * h] = x.x;
            f[4 * i + 2 * h + 1] = x.y;
        }
}
// the append's quantiser: code = cvt.rn.satfinite.e4m3(fp32(x) / scale), the division correctly rounded (not a multiply by a
// reciprocal), so that a host restatement matches it bit for bit
template <typename T> __device__ __forceinline__ uint2 quantise_e4m3x8(const Vec16<T> &x, float scale) {
    uint32_t c[4];
#pragma unroll
    for (int i = 0; i < 4; ++i)
        c[i] = f32x2_to_e4m3x2(__fdiv_rn(to_f(x.v[2 * i]), scale), __fdiv_rn(to_f(x.v[2 * i + 1]), scale));
    return make_uint2(c[0] | (c[1] << 16), c[2] | (c[3] << 16));
}
template <typename T> __device__ __forceinline__ uint4 quantise_e4m3x16(const Vec16<T> (&x)[2], float scale) {
    const uint2 lo = quantise_e4m3x8(x[0], scale), hi = quantise_e4m3x8(x[1], scale);
    return make_uint4(lo.x, lo.y, hi.x, hi.y);
}
// a lane's 16 bytes of a cache row as elements v[j] that to_f reads: f16 / bf16 / fp32 as stored (widened where they are
// used), FP8 codes decoded to fp32 here
template <typename KT> __device__ __forceinline__ auto ld_cache_row(const KT *p) {
    if constexpr (KV8<KT>) {
        struct { float v[16]; } r;
        e4m3x16_to_f(*reinterpret_cast<const uint4 *>(p), r.v);
        return r;
    } else {
        return ld16(p);
    }
}

constexpr int AS_MAX_B = 1024;  // batch rows whose (position, chunk count) the CTA keeps in shared memory

template <typename T, typename KT, int D, int WARPS, int U, int ROPE, bool WIN = false>
__device__ __forceinline__ void
    attn_stream_body(KT *__restrict__ kcache, KT *__restrict__ vcache, const T *__restrict__ q,
                       const T *__restrict__ kin, const T *__restrict__ vin, const void *__restrict__ position_id,
                       int pos_flags, T *__restrict__ out, int Smax, int BH, float *__restrict__ partial,
                       int slots_per_head, int *__restrict__ tickets, const void *__restrict__ rope_pos,
                       int rope_pos_dtype, int H, const float *__restrict__ k_scale, const float *__restrict__ v_scale,
                       const float *__restrict__ inv_freq, int window = 0) {
    using C = RowCfg<KT, D>;
    constexpr int EPL = C::EPL, LPR = C::LPR, RPW = C::RPW;
    constexpr int VE = Vec16<T>::N, NV = EPL / VE;            // a lane's EPL activations: NV 16-byte vectors (FP8: 2)
    constexpr int CH = WARPS * RPW * U;                       // cache rows per chunk
    constexpr int CHUNK_BYTES = CH * D * (int)sizeof(KT);     // 16 KiB for every dtype and width
    constexpr int CONSUMERS = WARPS * 32;
    extern __shared__ __align__(128) unsigned char ring[];    // stages x { K chunk | V chunk }
    __shared__ __align__(8) uint64_t full[AS_STAGES], empty[AS_STAGES];
    __shared__ float s_m[WARPS], s_l[WARPS];
    __shared__ float s_acc[WARPS][D];
    __shared__ float s_cs[D / 2], s_sn[D / 2];
    __shared__ int s_last;
    __shared__ int s_pos[AS_MAX_B];       // clamped position of batch row b
    __shared__ int s_pre[AS_MAX_B + 1];   // (head, chunk) units before batch row b; s_pre[B] = total

    pdl_trigger();
    const int pos_dtype = pos_flags & 0xff;
    const bool per_row = (pos_flags & ITB_POS_PER_ROW) != 0;
    // ITB_POS_IN_STEP: the position tensor / RoPE positions / cache rows below the position may have been written by a
    // kernel of THIS step (an ONNX graph that computes position_ids or concatenates the past in-graph): nothing is read
    // ahead of griddepcontrol.wait.  Otherwise they are a whole step old (graph inputs, the previous step's appends) and
    // the producer starts streaming while the previous kernel of the chain drains.
    if (pos_flags & ITB_POS_IN_STEP) pdl_wait();
    const int Bn = BH / H;
    // span(p): the cache rows read below position p -- all p of them, or (WIN) the last window - 1, from lo = p - span(p).
    // Units, offsets and the dealing count from lo, so a windowed head at p runs exactly as an unwindowed one at span(p)
    // over the cache rows from lo up
    auto span = [&](int p) { return WIN ? min(p, window - 1) : p; };
    // (WIN) ITB_POS_RING: the caches are a ring, position p in row cache_row(p, Smax, rolling) = p mod Smax
    const bool rolling = WIN && (pos_flags & ITB_POS_RING) != 0;
    if (threadIdx.x == 0) {
        for (int s = 0; s < AS_STAGES; ++s) {
            mbar_init(&full[s], 1);
            mbar_init(&empty[s], WARPS);
        }
        fence_mbar_init();
    }
    for (int b = threadIdx.x; b < Bn; b += blockDim.x) {
        if constexpr (WIN) {
            s_pos[b] = win_pos(position_id, pos_dtype, per_row ? b : 0, Smax, rolling);
        } else {
            int p = pos_dtype == ITB_I64 ? read_pos<int64_t>(position_id, per_row ? b : 0)
                                         : read_pos<int32_t>(position_id, per_row ? b : 0);
            s_pos[b] = min(max(p, 0), Smax - 1);
        }
    }
    __syncthreads();
    if (threadIdx.x == 0) {
        int acc = 0;
        for (int b = 0; b < Bn; ++b) {
            s_pre[b] = acc;
            acc += H * (span(s_pos[b]) / CH + 1);  // chunks per head of row b; the last one holds rows [.., pos) + the appended row
        }
        s_pre[Bn] = acc;
    }
    __syncthreads();
    // Everything this step produced (q, k, v) is read by the consumers, after their wait; this kernel's own append
    // touches row `pos` only, which the bulk loads never include.  Over a ring that row, pos mod Smax, holds position
    // pos - Smax or older, and Smax >= window (check_ring) puts that below the window, so no chunk includes it either.

    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    const int64_t total = s_pre[Bn], G = min((int64_t)gridDim.x, total);
    // this CTA's contiguous range of (head, chunk) units: [u0, u0 + nunits), starting at (bh, c) inside batch row b.
    // G = CTAs that take part: never more than there are units, so every one owns >= 1 unit and the CTAs sharing a head
    // are consecutive
    if (blockIdx.x >= G) return;
    int nunits, bh, c, brow, pos, nch;
    {
        const int64_t u0 = blockIdx.x * total / G, u1 = (blockIdx.x + 1) * total / G;
        nunits = (int)(u1 - u0);
        brow = 0;
        while (brow + 1 < Bn && s_pre[brow + 1] <= u0) ++brow;
        pos = s_pos[brow];
        nch = span(pos) / CH + 1;
        const int r = (int)(u0 - s_pre[brow]);
        bh = brow * H + r / nch;
        c = r % nch;
    }
    auto next_unit = [&]() {  // (bh, c) -> the next unit; entering a new batch row refreshes its position
        if (++c == nch) {
            c = 0;
            ++bh;
            if (bh % H == 0 && bh < BH) {
                brow = bh / H;
                pos = s_pos[brow];
                nch = span(pos) / CH + 1;
            }
        }
    };

    if (warp == WARPS) {
        // ---------------- producer: one elected lane streams chunks into the ring ----------------
        if (lane == 0) {
            const uint64_t policy = l2_policy_evict_first();
            int st = 0, ph = 0;
            for (int it = 0; it < nunits; ++it) {
                mbar_wait(&empty[st], ph ^ 1);
                const int rows = min(CH, span(pos) - c * CH);
                if constexpr (WIN) {
                    if (rows > 0)
                        win_chunk_load<KT, D>(ring + (size_t)st * 2 * CHUNK_BYTES, CHUNK_BYTES, kcache, vcache, bh, Smax,
                                              pos - span(pos) + c * CH, rows, rolling, &full[st], policy);
                    else
                        mbar_arrive(&full[st]);
                } else if (rows > 0) {
                    const uint32_t bytes = (uint32_t)rows * D * (uint32_t)sizeof(KT);
                    const int64_t off = ((int64_t)bh * Smax + (pos - span(pos)) + (int64_t)c * CH) * D;
                    mbar_expect_tx(&full[st], 2 * bytes);
                    bulk_load_1d(ring + (size_t)st * 2 * CHUNK_BYTES, kcache + off, bytes, &full[st], policy);
                    bulk_load_1d(ring + (size_t)st * 2 * CHUNK_BYTES + CHUNK_BYTES, vcache + off, bytes, &full[st], policy);
                } else {
                    mbar_arrive(&full[st]);
                }
                next_unit();
                if (++st == AS_STAGES) { st = 0; ph ^= 1; }
            }
        }
        return;
    }

    // ---------------- consumers ----------------
    // RoPE cos / sin table of the CTA's first batch row: the RoPE positions (and an inv_freq table, a graph weight) are
    // step-old like the cache position, so the powf / sincosf chain runs ahead of the wait; recomputed only when a later
    // segment changes batch row
    int table_b = -1;
    auto rope_table = [&](int b) {
        if (threadIdx.x < D / 2) {
            const float p = rope_pos_dtype == ITB_I64 ? (float)(int)((const int64_t *)rope_pos)[b]
                                                      : (float)((const int32_t *)rope_pos)[b];
            const float freq = ROPE == ROPE_TABLE ? __fmul_rn(p, inv_freq[threadIdx.x])
                                                  : p * powf(10000.f, -(float)(threadIdx.x * 2) / (float)D);
            s_cs[threadIdx.x] = round_t<T>(cosf(freq));
            s_sn[threadIdx.x] = round_t<T>(sinf(freq));
        }
        named_bar_sync(1, CONSUMERS);
        table_b = b;
    };
    if (ROPE) rope_table(bh / H);
    pdl_wait();  // (a no-op the second time under ITB_POS_IN_STEP)
    const int sub = lane / LPR;
    const int col = (lane % LPR) * EPL;
    float qf[EPL], m = -INFINITY, l = 0.f, acc[EPL];
    bool seg_from_start = false;
    int st = 0, ph = 0;
    for (int it = 0; it < nunits; ++it) {
        if (it == 0 || c == 0) {
            // new head segment: reset the running softmax, fetch (and rotate) q
            seg_from_start = c == 0;
            m = -INFINITY;
            l = 0.f;
#pragma unroll
            for (int j = 0; j < EPL; ++j) acc[j] = 0.f;
            Vec16<T> qv[NV];
#pragma unroll
            for (int h = 0; h < NV; ++h) qv[h] = ld16(q + (int64_t)bh * D + col + VE * h);
            if (ROPE) {
                if (bh / H != table_b) rope_table(bh / H);  // (every earlier reader is behind the previous segment's barriers)
#pragma unroll
                for (int h = 0; h < NV; ++h) rope_one<T, D, VE, LPR>(qv[h], col + VE * h, s_cs, s_sn);
            }
            float qs = attn_scale<D>();
            if constexpr (KV8<KT>) qs = k_scale[bh % H] * attn_scale<D>();
#pragma unroll
            for (int j = 0; j < VE; ++j)
#pragma unroll
                for (int h = 0; h < NV; ++h) qf[VE * h + j] = to_f(qv[h].v[j]) * qs;
        }
        const int nvalid = span(pos) - c * CH;  // cache rows of this chunk that exist (<= 0: only the appended row)
        const unsigned char *kb = ring + (size_t)st * 2 * CHUNK_BYTES, *vb = kb + CHUNK_BYTES;
        mbar_wait(&full[st], ph);
#ifndef ATTN_DBG_NOCOMPUTE  // (debug builds only: measures the bare HBM -> smem ring)
        const KT *ks = reinterpret_cast<const KT *>(kb) + (warp * U * RPW + sub) * D + col;
        const KT *vs = reinterpret_cast<const KT *>(vb) + (warp * U * RPW + sub) * D + col;
        if (nvalid >= CH) {
            // full chunk (every chunk but a head's last): branch-free, so the U rows' load / dot / shuffle chains interleave
            float sc[U];
#pragma unroll
            for (int uu = 0; uu < U; ++uu) {
                const auto kv = ld_cache_row(ks + uu * RPW * D);
                float d = 0.f;
#pragma unroll
                for (int j = 0; j < EPL; ++j) d += qf[j] * to_f(kv.v[j]);
                sc[uu] = d;
            }
#pragma unroll
            for (int o = LPR / 2; o > 0; o >>= 1) {
#pragma unroll
                for (int uu = 0; uu < U; ++uu) sc[uu] += __shfl_xor_sync(0xffffffffu, sc[uu], o);
            }
            float mx = m;
#pragma unroll
            for (int uu = 0; uu < U; ++uu) mx = fmaxf(mx, sc[uu]);
            const float corr = expf(m - mx);  // m = -inf -> 0
            l *= corr;
#pragma unroll
            for (int j = 0; j < EPL; ++j) acc[j] *= corr;
#pragma unroll
            for (int uu = 0; uu < U; ++uu) {
                const auto vv = ld_cache_row(vs + uu * RPW * D);
                const float p = expf(sc[uu] - mx);
                l += p;
#pragma unroll
                for (int j = 0; j < EPL; ++j) acc[j] = fmaf(p, to_f(vv.v[j]), acc[j]);
            }
            m = mx;
        } else {
            float sc[U];
            bool ok[U];
#pragma unroll
            for (int uu = 0; uu < U; ++uu) {
                ok[uu] = (warp * U + uu) * RPW + sub < nvalid;
                float d = 0.f;
                if (ok[uu]) {
                    const auto kv = ld_cache_row(ks + uu * RPW * D);
#pragma unroll
                    for (int j = 0; j < EPL; ++j) d += qf[j] * to_f(kv.v[j]);
                }
#pragma unroll
                for (int o = LPR / 2; o > 0; o >>= 1) d += __shfl_xor_sync(0xffffffffu, d, o);
                sc[uu] = ok[uu] ? d : -INFINITY;
            }
            float mx = m;
#pragma unroll
            for (int uu = 0; uu < U; ++uu) mx = fmaxf(mx, sc[uu]);
            if (mx > -INFINITY) {
                const float corr = expf(m - mx);  // m = -inf -> 0
                l *= corr;
#pragma unroll
                for (int j = 0; j < EPL; ++j) acc[j] *= corr;
#pragma unroll
                for (int uu = 0; uu < U; ++uu) {
                    if (ok[uu]) {
                        const auto vv = ld_cache_row(vs + uu * RPW * D);
                        const float p = expf(sc[uu] - mx);
                        l += p;
#pragma unroll
                        for (int j = 0; j < EPL; ++j) acc[j] = fmaf(p, to_f(vv.v[j]), acc[j]);
                    }
                }
                m = mx;
            }
        }
#endif
        __syncwarp();
        if (lane == 0) mbar_arrive(&empty[st]);  // this warp is done with the stage
        if (++st == AS_STAGES) { st = 0; ph ^= 1; }

        const bool last_chunk = c == nch - 1;
        if (last_chunk && warp == 0) {
            // the row appended this step: rotate k if asked, store k / v in place, add its contribution from registers.  FP8
            // quantises k / v in registers, and the row contributes through its codes, decoded (kdec / vdec)
            const int64_t src = (int64_t)bh * D + col;
            Vec16<T> kx[NV];
#pragma unroll
            for (int h = 0; h < NV; ++h) kx[h] = ld16(kin + src + VE * h);
            if (ROPE) {
#pragma unroll
                for (int h = 0; h < NV; ++h) rope_one<T, D, VE, LPR>(kx[h], col + VE * h, s_cs, s_sn);
            }
            float kdec[EPL];
            uint4 kcodes;
            if constexpr (KV8<KT>) {
                kcodes = quantise_e4m3x16(kx, k_scale[bh % H]);
                e4m3x16_to_f(kcodes, kdec);
            }
            float d = 0.f;
#pragma unroll
            for (int j = 0; j < EPL; ++j) d += qf[j] * (KV8<KT> ? kdec[j] : to_f(kx[0].v[j]));
#pragma unroll
            for (int o = LPR / 2; o > 0; o >>= 1) d += __shfl_xor_sync(0xffffffffu, d, o);
            if (sub == 0) {
                Vec16<T> vx;
                float vdec[EPL];
                if constexpr (KV8<KT>) {
                    const uint4 vcodes = quantise_e4m3x16({ld16(vin + src), ld16(vin + src + VE)}, v_scale[bh % H]);
                    *reinterpret_cast<uint4 *>(kcache + ((int64_t)bh * Smax + (WIN ? cache_row(pos, Smax, rolling) : pos)) * D + col) = kcodes;
                    *reinterpret_cast<uint4 *>(vcache + ((int64_t)bh * Smax + (WIN ? cache_row(pos, Smax, rolling) : pos)) * D + col) = vcodes;
                    e4m3x16_to_f(vcodes, vdec);
                } else {
                    vx = ld16(vin + src);
                    st16(kcache + ((int64_t)bh * Smax + (WIN ? cache_row(pos, Smax, rolling) : pos)) * D + col, kx[0]);
                    st16(vcache + ((int64_t)bh * Smax + (WIN ? cache_row(pos, Smax, rolling) : pos)) * D + col, vx);
                }
                const float mx2 = fmaxf(m, d);
                const float corr = expf(m - mx2), pnew = expf(d - mx2);
                l = l * corr + pnew;
#pragma unroll
                for (int j = 0; j < EPL; ++j) acc[j] = fmaf(pnew, KV8<KT> ? vdec[j] : to_f(vx.v[j]), acc[j] * corr);
                m = mx2;
            }
        }

        if (last_chunk || it == nunits - 1) {
            // ---- segment end: fold sub-rows, warps, and (when the head is shared between CTAs) the other CTAs' partials
#pragma unroll
            for (int o = LPR; o < 32; o <<= 1) {
                const float m2 = __shfl_xor_sync(0xffffffffu, m, o);
                const float l2 = __shfl_xor_sync(0xffffffffu, l, o);
                const float mm = fmaxf(m, m2);
                const float c1 = mm > -INFINITY ? expf(m - mm) : 0.f, c2 = mm > -INFINITY ? expf(m2 - mm) : 0.f;
                l = l * c1 + l2 * c2;
#pragma unroll
                for (int j = 0; j < EPL; ++j) {
                    const float a2 = __shfl_xor_sync(0xffffffffu, acc[j], o);
                    acc[j] = acc[j] * c1 + a2 * c2;
                }
                m = mm;
            }
            if (sub == 0) {
#pragma unroll
                for (int j = 0; j < EPL; ++j) s_acc[warp][col + j] = acc[j];
                if (lane == 0) {
                    s_m[warp] = m;
                    s_l[warp] = l;
                }
            }
            named_bar_sync(1, CONSUMERS);
            const bool whole = seg_from_start && last_chunk;
            // which CTAs share this head:  cta(u) = floor(((u + 1) G - 1) / total)
            const int64_t hu0 = (int64_t)s_pre[brow] + (int64_t)(bh - brow * H) * nch;  // first unit of this head
            const int first_cta = (int)(((hu0 + 1) * G - 1) / total);
            const int last_cta = (int)(((hu0 + nch) * G - 1) / total);
            const int nseg = last_cta - first_cta + 1;
            float *slots = partial + (int64_t)bh * slots_per_head * (D + 2);
            auto out_val = [&](float A, float L) {  // FP8: V's scale, once
                if constexpr (KV8<KT>) return from_f<T>(A / L * v_scale[bh % H]);
                else return from_f<T>(A / L);
            };
            if (threadIdx.x < D) {
                const int d = threadIdx.x;
                float mw = -INFINITY;
#pragma unroll
                for (int w = 0; w < WARPS; ++w) mw = fmaxf(mw, s_m[w]);
                float L = 0.f, A = 0.f;
#pragma unroll
                for (int w = 0; w < WARPS; ++w) {
                    const float cw = s_m[w] > -INFINITY ? expf(s_m[w] - mw) : 0.f;
                    L += s_l[w] * cw;
                    A += s_acc[w][d] * cw;
                }
                if (whole) {
                    out[(int64_t)bh * D + d] = out_val(A, L);
                } else {
                    float *pp = slots + (int64_t)((int)blockIdx.x - first_cta) * (D + 2);
                    __stcg(pp + 2 + d, A);
                    if (d == 0) {
                        __stcg(pp, mw);
                        __stcg(pp + 1, L);
                    }
                    __threadfence();
                }
            }
            if (!whole) {
                named_bar_sync(1, CONSUMERS);
                if (threadIdx.x == 0) {
                    const int old = atomicAdd(tickets + bh, 1);
                    s_last = old == nseg - 1;
                    if (s_last) tickets[bh] = 0;  // self-cleaning: every other sharer has already arrived
                    __threadfence();
                }
                named_bar_sync(1, CONSUMERS);
                if (s_last && threadIdx.x < D) {
                    const int d = threadIdx.x;
                    float mw = -INFINITY;
                    for (int s = 0; s < nseg; ++s) mw = fmaxf(mw, __ldcg(slots + (int64_t)s * (D + 2)));
                    float L = 0.f, A = 0.f;
                    for (int s = 0; s < nseg; ++s) {
                        const float *pp = slots + (int64_t)s * (D + 2);
                        const float ms = __ldcg(pp);
                        const float cw = ms > -INFINITY ? expf(ms - mw) : 0.f;
                        L += __ldcg(pp + 1) * cw;
                        A += __ldcg(pp + 2 + d) * cw;
                    }
                    out[(int64_t)bh * D + d] = out_val(A, L);
                }
            }
            named_bar_sync(1, CONSUMERS);  // s_acc / s_m / s_last are reused by the next segment
        }
        next_unit();
    }
}

// ------------------------------------------------------------------------------------------------------------------
// attn_gqa_kernel: grouped-query decode, Hq = G x Hkv query heads with G > 1; query head i reads KV head i / G (HF
// repeat_kv order).  The pipeline of attn_stream_kernel (flattened units in equal contiguous ranges over 2 x 132 CTAs,
// cp.async.bulk producer, full/empty mbarrier ring, last-arriving CTA merges in CTA order) with the unit
// (batch row, KV head, query group, 16 KiB chunk).  A query group is up to QT tiles of 16 query rows (rows past the
// group's heads are zero padding): G <= 16 runs one tile, G > 16 groups of two, NQG = ceil(G / 32) groups per KV head.
// For G <= 32 there is one group, so every K and V row is read from HBM once per step and used by all G query heads;
// larger G (multi-query attention with 33+ heads) reads the KV head once per group.  Per chunk:
//   S = Q K^T   warp w takes chunk rows [w CH/8, (w + 1) CH/8) of every query row -- mma.sync m16n8k16 with fp32
//               accumulators for f16 / bf16 (D/16 k16 steps over NT = CH/64 n8 tiles), FFMA for fp32 -- and scales them
//               by 1/sqrt(D) in fp32;
//   softmax     the warps' row maxima and row sums meet in shared memory, every consumer derives the same running (m, l);
//   O += P V    f16 / bf16: P enters the tensor core as two T operands, hi = P rounded to T and lo = P - hi rounded to T
//               (two MMAs), so each weight keeps 16 (bf16) / 22 (f16) significant bits instead of T's 8 / 11 -- rounding P
//               once, as FlashAttention does, was measured at up to 2 ulp of bf16 off the oracle on short contexts.
//               Warp w owns output columns [D/8 w, D/8 (w + 1)) of every query row (NJ = D/64 n8 tiles), so O is never
//               merged across warps.  At D = 64 that is one n8 tile per warp over a 128-row chunk: every warp still issues
//               the same MMAs per chunk row as at D = 128, and the warps stay independent.
// The row appended this step is stored into the ring slot after the last chunk's cache rows and takes part in that
// chunk's products like any other row; group 0 also stores it in place.
// ------------------------------------------------------------------------------------------------------------------
constexpr int GQ_WARPS = 8;

template <typename T, int D, typename KT = T> struct GqaCfg {  // KT: the cache element type
    static constexpr int CH = 16384 / (D * (int)sizeof(KT));  // cache rows per 16 KiB chunk: 64 / 128 (f16 / bf16), 32 / 64 (fp32),
                                                              // 128 / 256 (FP8)
    static constexpr int NC = CH / (GQ_WARPS * 4);           // S columns per thread: 2 / 4, 1 / 2
    static constexpr int NT = NC / 2;                        // f16 / bf16: n8 tiles of S per warp
    static constexpr int NJ = D / (8 * GQ_WARPS);            // n8 tiles of O per warp
    static constexpr int QLD = D + 16 / (int)sizeof(T);      // +16 B per row: ldmatrix rows fall in distinct banks
    static constexpr int PLD = CH + 16 / (int)sizeof(T);
};

template <typename T, typename KT, int D, int QT, int ROPE, bool WIN = false, typename... Scale>
__device__ __forceinline__ void
    attn_gqa_body(KT *__restrict__ kcache, KT *__restrict__ vcache, const T *__restrict__ q,
                    const T *__restrict__ kin, const T *__restrict__ vin, const void *__restrict__ position_id,
                    int pos_flags, T *__restrict__ out, int Smax, int Bn, int Hkv, int G, int NQG,
                    float *__restrict__ partial, int slots_per_head, int *__restrict__ tickets, const void *__restrict__ rope_pos, int rope_pos_dtype,
                    const float *__restrict__ inv_freq, int window, const Scale *__restrict__... kv_scale) {
    // kv_scale: k_scale, v_scale for an FP8 cache, nothing for the others (unused scale parameters alone change how the
    // unquantised kernels compile)
    using C = RowCfg<T, D>;  // row-load layout of q and the appended k / v
    using Q = GqaCfg<T, D, KT>;
    constexpr int EPL = C::EPL, LPR = C::LPR, RPW = C::RPW;
    constexpr int CH = Q::CH, NC = Q::NC, NT = Q::NT, NJ = Q::NJ, QLD = Q::QLD, PLD = Q::PLD;
    constexpr int GP = 16 * QT;  // padded query rows
    constexpr int CHUNK_BYTES = CH * D * (int)sizeof(KT);
    constexpr int CONSUMERS = GQ_WARPS * 32;
    constexpr bool MMA = sizeof(T) == 2;
    constexpr float kScale = attn_scale<D>();
    extern __shared__ __align__(128) unsigned char ring[];  // stages x { K chunk | V chunk }
    __shared__ __align__(8) uint64_t full[AS_STAGES], empty[AS_STAGES];
    __shared__ __align__(16) T s_q[GP * QLD];   // (rotated) query rows of the current query group
    __shared__ __align__(16) T s_p[GP * PLD];   // P of the current chunk, rounded to T
    __shared__ __align__(16) T s_plo[MMA ? GP * PLD : 1];  // f16 / bf16: P - s_p, rounded to T
    __shared__ float s_red[2][GQ_WARPS][GP];    // per-warp row maxima / row sums of the current chunk
    __shared__ float s_cs[D / 2], s_sn[D / 2];
    __shared__ int s_last;
    __shared__ int s_pre[AS_MAX_B + 1];  // (KV head, query group, chunk) units before batch row b; s_pre[B] = total

    pdl_trigger();
    const int pos_dtype = pos_flags & 0xff;
    const bool per_row = (pos_flags & ITB_POS_PER_ROW) != 0;
    if (pos_flags & ITB_POS_IN_STEP) pdl_wait();  // (see attn_stream_kernel)
    // (WIN) ITB_POS_RING as in attn_stream_body, the flag read where it is used: a named local for it changes how the
    // unwindowed fp32 instantiations compile
    auto pos_of = [&](int b) {
        if constexpr (WIN) {
            return win_pos(position_id, pos_dtype, per_row ? b : 0, Smax, (pos_flags & ITB_POS_RING) != 0);
        } else {
            const int p = pos_dtype == ITB_I64 ? read_pos<int64_t>(position_id, per_row ? b : 0)
                                               : read_pos<int32_t>(position_id, per_row ? b : 0);
            return min(max(p, 0), Smax - 1);
        }
    };
    auto span = [&](int p) { return WIN ? min(p, window - 1) : p; };  // (see attn_stream_body)
    if (threadIdx.x == 0) {
        for (int s = 0; s < AS_STAGES; ++s) {
            mbar_init(&full[s], 1);
            mbar_init(&empty[s], GQ_WARPS);
        }
        fence_mbar_init();
    }
    // V rows past a chunk's valid rows enter the P.V product with P = 0: they must hold finite values, so the ring starts
    // zeroed (later it only ever holds cache rows)
    for (int i = threadIdx.x; i < AS_STAGES * 2 * CHUNK_BYTES / 16; i += blockDim.x)
        reinterpret_cast<uint4 *>(ring)[i] = make_uint4(0, 0, 0, 0);
    fence_proxy_async();
    const int HV = Hkv * NQG;  // (KV head, query group) segments per batch row
    for (int b = threadIdx.x; b < Bn; b += blockDim.x) s_pre[b] = HV * (span(pos_of(b)) / CH + 1);
    __syncthreads();
    if (threadIdx.x == 0) {
        int acc = 0;
        for (int b = 0; b < Bn; ++b) {
            const int n = s_pre[b];
            s_pre[b] = acc;
            acc += n;
        }
        s_pre[Bn] = acc;
    }
    __syncthreads();

    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    const int BH = Bn * HV;
    const int64_t total = s_pre[Bn], ncta = min((int64_t)gridDim.x, total);
    if (blockIdx.x >= ncta) return;
    int nunits, bh, c, brow, pos, nch;  // bh = (b * Hkv + KV head) * NQG + query group
    {
        const int64_t u0 = blockIdx.x * total / ncta, u1 = (blockIdx.x + 1) * total / ncta;
        nunits = (int)(u1 - u0);
        brow = 0;
        while (brow + 1 < Bn && s_pre[brow + 1] <= u0) ++brow;
        pos = pos_of(brow);
        nch = span(pos) / CH + 1;
        const int r = (int)(u0 - s_pre[brow]);
        bh = brow * HV + r / nch;
        c = r % nch;
    }
    auto next_unit = [&]() {
        if (++c == nch) {
            c = 0;
            ++bh;
            if (bh % HV == 0 && bh < BH) {
                brow = bh / HV;
                pos = pos_of(brow);
                nch = span(pos) / CH + 1;
            }
        }
    };

    if (warp == GQ_WARPS) {
        // ---------------- producer (as attn_stream_kernel) ----------------
        if (lane == 0) {
            const uint64_t policy = l2_policy_evict_first();
            int st = 0, ph = 0;
            for (int it = 0; it < nunits; ++it) {
                mbar_wait(&empty[st], ph ^ 1);
                const int rows = min(CH, span(pos) - c * CH);
                if (rows > 0) {
                    if constexpr (WIN) {
                        win_chunk_load<KT, D>(ring + (size_t)st * 2 * CHUNK_BYTES, CHUNK_BYTES, kcache, vcache, bh / NQG, Smax,
                                              pos - span(pos) + c * CH, rows, (pos_flags & ITB_POS_RING) != 0, &full[st], policy);
                    } else {
                        const uint32_t bytes = (uint32_t)rows * D * (uint32_t)sizeof(KT);
                        const int64_t off = ((int64_t)(bh / NQG) * Smax + (pos - span(pos)) + (int64_t)c * CH) * D;
                        mbar_expect_tx(&full[st], 2 * bytes);
                        bulk_load_1d(ring + (size_t)st * 2 * CHUNK_BYTES, kcache + off, bytes, &full[st], policy);
                        bulk_load_1d(ring + (size_t)st * 2 * CHUNK_BYTES + CHUNK_BYTES, vcache + off, bytes, &full[st], policy);
                    }
                } else {
                    mbar_arrive(&full[st]);
                }
                next_unit();
                if (++st == AS_STAGES) { st = 0; ph ^= 1; }
            }
        }
        return;
    }

    // ---------------- consumers ----------------
    int table_b = -1;
    auto rope_table = [&](int b) {
        if (threadIdx.x < D / 2) {
            const float p = rope_pos_dtype == ITB_I64 ? (float)(int)((const int64_t *)rope_pos)[b]
                                                      : (float)((const int32_t *)rope_pos)[b];
            const float freq = ROPE == ROPE_TABLE ? __fmul_rn(p, inv_freq[threadIdx.x])
                                                  : p * powf(10000.f, -(float)(threadIdx.x * 2) / (float)D);
            s_cs[threadIdx.x] = round_t<T>(cosf(freq));
            s_sn[threadIdx.x] = round_t<T>(sinf(freq));
        }
        named_bar_sync(1, CONSUMERS);
        table_b = b;
    };
    if (ROPE) rope_table(bh / HV);
    pdl_wait();
    const int sub = lane / LPR, col = (lane % LPR) * EPL;  // row-load layout (q, appended k / v)
    const int qr = lane >> 2, qc = lane & 3;               // fragment layout: rows qr, qr + 8 of each 16-row tile
    const int cw = warp * (CH / GQ_WARPS);                 // first chunk row of this warp's S columns
    // o[t][j][2h + e]: row 16t + qr + 8h, column 8 NJ w + 8j + 2qc + e
    float m_run[QT][2], l_run[QT][2], o[QT][NJ][4];
    bool seg_from_start = false;
    int st = 0, ph = 0;
    int64_t q0 = 0;  // first query head of the segment's group
    int gq = 0;      // query heads in the segment's group (<= GP)
    for (int it = 0; it < nunits; ++it) {
        if (it == 0 || c == 0) {
            // new segment: reset the running softmax, stage the group's query rows (rotated if asked)
            seg_from_start = c == 0;
#pragma unroll
            for (int t = 0; t < QT; ++t)
#pragma unroll
                for (int h = 0; h < 2; ++h) {
                    m_run[t][h] = -INFINITY;
                    l_run[t][h] = 0.f;
#pragma unroll
                    for (int j = 0; j < NJ; ++j) o[t][j][2 * h] = o[t][j][2 * h + 1] = 0.f;
                }
            if (ROPE && bh / HV != table_b) rope_table(bh / HV);
            // query heads [kvh G + qg GP, + gq) of batch row b
            q0 = (int64_t)(bh / NQG) * G + (int64_t)(bh % NQG) * GP;
            gq = min(GP, G - (bh % NQG) * GP);
            const T *qh = q + q0 * D;
            for (int r0 = warp * RPW; r0 < GP; r0 += GQ_WARPS * RPW) {
                const int r = r0 + sub;
                Vec16<T> x;
                *reinterpret_cast<uint4 *>(x.v) = make_uint4(0, 0, 0, 0);
                if (r < gq) x = ld16(qh + (int64_t)r * D + col);
                if (ROPE) rope_one<T, D, EPL, LPR>(x, col, s_cs, s_sn);
                st16(s_q + r * QLD + col, x);
            }
            named_bar_sync(1, CONSUMERS);
        }
        const int nvalid = span(pos) - c * CH;  // cache rows of this chunk below the position (last chunk: < CH)
        const bool last_chunk = c == nch - 1;
        KT *ks = reinterpret_cast<KT *>(ring + (size_t)st * 2 * CHUNK_BYTES), *vs = ks + CH * D;
        mbar_wait(&full[st], ph);
        int nrows = min(nvalid, CH);
        if (last_chunk) {
            // the row appended this step: rotate k if asked, store k / v into ring row nvalid, and (group 0) in place
            if (warp == 0) {
                const int64_t kv = bh / NQG;
#pragma unroll
                for (int r0 = 0; r0 < 2; r0 += RPW) {
                    const int which = r0 + sub;  // 0: k, 1: v
                    Vec16<T> x = ld16((which == 0 ? kin : vin) + kv * D + col);
                    if (ROPE) {
                        Vec16<T> xr = x;
                        rope_one<T, D, EPL, LPR>(xr, col, s_cs, s_sn);
                        if (which == 0) x = xr;
                    }
                    if (RPW <= 2 || which < 2) {  // (D = 64, 2-byte types: sub-rows 2, 3 only took part in the shuffles)
                        if constexpr (KV8<KT>) {
                            // quantised in registers; the ring row holds the codes, so the row contributes through them
                            const float *const scales[2] = {kv_scale...};
                            const uint2 codes = quantise_e4m3x8(x, scales[which][kv % Hkv]);
                            if (bh % NQG == 0)
                                *reinterpret_cast<uint2 *>((which == 0 ? kcache : vcache) + (kv * Smax + (WIN ? cache_row(pos, Smax, (pos_flags & ITB_POS_RING) != 0) : pos)) * D + col) = codes;
                            *reinterpret_cast<uint2 *>((which == 0 ? ks : vs) + nvalid * D + col) = codes;
                        } else {
                            if (bh % NQG == 0) st16((which == 0 ? kcache : vcache) + (kv * Smax + (WIN ? cache_row(pos, Smax, (pos_flags & ITB_POS_RING) != 0) : pos)) * D + col, x);
                            st16((which == 0 ? ks : vs) + nvalid * D + col, x);
                        }
                    }
                }
                fence_proxy_async();  // the producer's next bulk copy into this stage must land after these stores
            }
            named_bar_sync(1, CONSUMERS);
            nrows = nvalid + 1;
        }

        // ---- S = Q K^T for this warp's chunk rows, scaled, masked past nrows: s[t][h][e] = S[16t + qr + 8h][cw + NC qc + e]
        float s[QT][2][NC];
        if constexpr (KV8<KT>) {
            // The k (head-dim) order inside each 64-column block is permuted, alike for Q and K, so that a thread's B
            // fragments come from one 16-byte load of codes: k16 step 4jj + st, fragment column pair 2qc + {0,1} (+8) <->
            // columns 64jj + 16qc + 4st + {0,1} ({2,3}).  n8 tile j, B column n = chunk row cw + NC (n >> 1) + 2j + (n & 1):
            // the thread's accumulator columns 2qc, 2qc + 1 of every tile land on its NC consecutive chunk rows.
            constexpr int KS = D / 16;
            const float *const scales[2] = {kv_scale...};
            const float ksc = scales[0][(bh / NQG) % Hkv] * kScale;  // the KV head's K scale with 1/sqrt(D)
            uint32_t kf[NT][KS][2];
            const int krow = cw + NC * (qr >> 1) + (qr & 1);
#pragma unroll
            for (int j = 0; j < NT; ++j)
#pragma unroll
                for (int jj = 0; jj < D / 64; ++jj) {
                    const uint4 raw = *reinterpret_cast<const uint4 *>(ks + (krow + 2 * j) * D + 64 * jj + 16 * qc);
                    const uint32_t w[4] = {raw.x, raw.y, raw.z, raw.w};
#pragma unroll
                    for (int st4 = 0; st4 < 4; ++st4) {
                        kf[j][4 * jj + st4][0] = e4m3x2_to<T>(w[st4]);
                        kf[j][4 * jj + st4][1] = e4m3x2_to<T>(w[st4] >> 16);
                    }
                }
#pragma unroll
            for (int t = 0; t < QT; ++t) {
                float acc[NT][4];
#pragma unroll
                for (int j = 0; j < NT; ++j) acc[j][0] = acc[j][1] = acc[j][2] = acc[j][3] = 0.f;
#pragma unroll
                for (int jj = 0; jj < D / 64; ++jj) {
                    const T *qa = s_q + (16 * t + qr) * QLD + 64 * jj + 16 * qc;
                    const uint4 x0 = *reinterpret_cast<const uint4 *>(qa), x1 = *reinterpret_cast<const uint4 *>(qa + 8);
                    const uint4 y0 = *reinterpret_cast<const uint4 *>(qa + 8 * QLD), y1 = *reinterpret_cast<const uint4 *>(qa + 8 * QLD + 8);
                    const uint32_t wa[8] = {x0.x, x0.y, x0.z, x0.w, x1.x, x1.y, x1.z, x1.w};
                    const uint32_t wb[8] = {y0.x, y0.y, y0.z, y0.w, y1.x, y1.y, y1.z, y1.w};
#pragma unroll
                    for (int st4 = 0; st4 < 4; ++st4) {
                        uint32_t a[4] = {wa[2 * st4], wb[2 * st4], wa[2 * st4 + 1], wb[2 * st4 + 1]};
#pragma unroll
                        for (int j = 0; j < NT; ++j) mma_m16n8k16<T>(acc[j], a, kf[j][4 * jj + st4][0], kf[j][4 * jj + st4][1]);
                    }
                }
#pragma unroll
                for (int j = 0; j < NT; ++j)
#pragma unroll
                    for (int h = 0; h < 2; ++h)
#pragma unroll
                        for (int e = 0; e < 2; ++e) s[t][h][2 * j + e] = acc[j][2 * h + e] * ksc;
            }
        } else if constexpr (MMA) {
            // n8 tile j, B row n = chunk row cw + NC (n >> 1) + 2j + (n & 1): the thread's accumulator columns 2qc, 2qc + 1 of
            // every tile land on its NC consecutive chunk rows (NT = 1: row cw + n)
            constexpr int KS = D / 16;  // k16 steps
            uint32_t kf[NT][KS][2];
            const int krow = NT == 1 ? (lane & 7) : NC * ((lane & 7) >> 1) + (lane & 1);
#pragma unroll
            for (int j = 0; j < NT; ++j)
#pragma unroll
                for (int jj = 0; jj < KS / 2; ++jj)
                    ldmatrix_x4(kf[j][2 * jj][0], kf[j][2 * jj][1], kf[j][2 * jj + 1][0], kf[j][2 * jj + 1][1],
                                smem_u32(ks + (cw + krow + 2 * j) * D + 32 * jj + 8 * (lane >> 3)));
#pragma unroll
            for (int t = 0; t < QT; ++t) {
                float acc[NT][4];
#pragma unroll
                for (int j = 0; j < NT; ++j) acc[j][0] = acc[j][1] = acc[j][2] = acc[j][3] = 0.f;
#pragma unroll
                for (int kk = 0; kk < KS; ++kk) {
                    uint32_t a[4];
                    ldmatrix_x4(a[0], a[1], a[2], a[3], smem_u32(s_q + (16 * t + (lane & 15)) * QLD + 16 * kk + 8 * (lane >> 4)));
#pragma unroll
                    for (int j = 0; j < NT; ++j) mma_m16n8k16<T>(acc[j], a, kf[j][kk][0], kf[j][kk][1]);
                }
#pragma unroll
                for (int j = 0; j < NT; ++j)
#pragma unroll
                    for (int h = 0; h < 2; ++h)
#pragma unroll
                        for (int e = 0; e < 2; ++e) s[t][h][2 * j + e] = acc[j][2 * h + e] * kScale;
            }
        } else {
            const float *kr0 = reinterpret_cast<const float *>(ks) + (cw + NC * qc) * D;
#pragma unroll
            for (int e = 0; e < NC; ++e) {
                const float *kr = kr0 + e * D;
#pragma unroll
                for (int t = 0; t < QT; ++t)
#pragma unroll
                    for (int h = 0; h < 2; ++h) {
                        const float *qrow = reinterpret_cast<const float *>(s_q) + (16 * t + qr + 8 * h) * QLD;
                        float d = 0.f;
#pragma unroll 8
                        for (int dd = 0; dd < D; dd += 4) {
                            const float4 a = *reinterpret_cast<const float4 *>(qrow + dd);
                            const float4 b = *reinterpret_cast<const float4 *>(kr + dd);
                            d = fmaf(a.x, b.x, d);
                            d = fmaf(a.y, b.y, d);
                            d = fmaf(a.z, b.z, d);
                            d = fmaf(a.w, b.w, d);
                        }
                        s[t][h][e] = d * kScale;
                    }
            }
        }
        // ---- softmax: chunk row maxima across the warps, then P and its row sums
#pragma unroll
        for (int t = 0; t < QT; ++t)
#pragma unroll
            for (int h = 0; h < 2; ++h) {
                float mx = -INFINITY;
#pragma unroll
                for (int e = 0; e < NC; ++e) {
                    if (cw + NC * qc + e >= nrows) s[t][h][e] = -INFINITY;
                    mx = fmaxf(mx, s[t][h][e]);
                }
                mx = fmaxf(mx, __shfl_xor_sync(0xffffffffu, mx, 1));
                mx = fmaxf(mx, __shfl_xor_sync(0xffffffffu, mx, 2));
                if (qc == 0) s_red[0][warp][16 * t + qr + 8 * h] = mx;
            }
        named_bar_sync(1, CONSUMERS);
        float corr[QT][2];
#pragma unroll
        for (int t = 0; t < QT; ++t)
#pragma unroll
            for (int h = 0; h < 2; ++h) {
                const int r = 16 * t + qr + 8 * h;
                float cm = -INFINITY;
#pragma unroll
                for (int w = 0; w < GQ_WARPS; ++w) cm = fmaxf(cm, s_red[0][w][r]);
                const float mnew = fmaxf(m_run[t][h], cm);  // finite: every chunk has >= 1 row
                float sum = 0.f;
                __align__(NC * sizeof(T)) T hi[NC], lo[NC];
#pragma unroll
                for (int e = 0; e < NC; ++e) {
                    const float p = expf(s[t][h][e] - mnew);  // masked: exp(-inf) = 0
                    hi[e] = from_f<T>(p);
                    lo[e] = from_f<T>(p - to_f(hi[e]));
                    sum += p;
                }
                if constexpr (MMA) {
                    using PW = std::conditional_t<NC == 2, uint32_t, std::conditional_t<NC == 4, uint2, uint4>>;  // the thread's NC weights in one store
                    *reinterpret_cast<PW *>(s_p + r * PLD + cw + NC * qc) = *reinterpret_cast<const PW *>(hi);
                    *reinterpret_cast<PW *>(s_plo + r * PLD + cw + NC * qc) = *reinterpret_cast<const PW *>(lo);
                } else {
#pragma unroll
                    for (int e = 0; e < NC; ++e) s_p[r * PLD + cw + NC * qc + e] = hi[e];
                }
                sum += __shfl_xor_sync(0xffffffffu, sum, 1);
                sum += __shfl_xor_sync(0xffffffffu, sum, 2);
                if (qc == 0) s_red[1][warp][r] = sum;
                corr[t][h] = expf(m_run[t][h] - mnew);  // m_run = -inf -> 0
                m_run[t][h] = mnew;
            }
        named_bar_sync(1, CONSUMERS);
#pragma unroll
        for (int t = 0; t < QT; ++t)
#pragma unroll
            for (int h = 0; h < 2; ++h) {
                float ls = 0.f;
#pragma unroll
                for (int w = 0; w < GQ_WARPS; ++w) ls += s_red[1][w][16 * t + qr + 8 * h];
                l_run[t][h] = l_run[t][h] * corr[t][h] + ls;
#pragma unroll
                for (int j = 0; j < NJ; ++j) {
                    o[t][j][2 * h] *= corr[t][h];
                    o[t][j][2 * h + 1] *= corr[t][h];
                }
            }
        // ---- O += P V over output columns [8 NJ w, 8 NJ (w + 1))
        if constexpr (KV8<KT>) {
            // B fragment of k16 step kk, tile j: V codes of chunk rows 16kk + 2qc + {0, 1} (b0) and + {8, 9} (b1) in column
            // 8 NJ w + NJ qr + j: one NJ-byte load per row serves every tile, so the tiles' columns interleave
            const KT *vcol = vs + 8 * NJ * warp + NJ * qr;
#pragma unroll 4
            for (int kk = 0; kk < CH / 16; ++kk) {
                const KT *r0 = vcol + (16 * kk + 2 * qc) * D;
                uint32_t x[4];
#pragma unroll
                for (int i = 0; i < 4; ++i) {
                    const KT *ri = r0 + ((i & 1) + 8 * (i >> 1)) * D;  // rows +0, +1, +8, +9
                    if constexpr (NJ == 2) x[i] = *reinterpret_cast<const uint16_t *>(ri);
                    else x[i] = *ri;
                }
#pragma unroll
                for (int j = 0; j < NJ; ++j) {
                    const uint32_t sel = j == 0 ? 0x0040u : 0x0051u;  // byte j of the two rows -> a code pair
                    const uint32_t b0 = e4m3x2_to<T>(__byte_perm(x[0], x[1], sel));
                    const uint32_t b1 = e4m3x2_to<T>(__byte_perm(x[2], x[3], sel));
#pragma unroll
                    for (int t = 0; t < QT; ++t) {
                        const int off = (16 * t + (lane & 15)) * PLD + 16 * kk + 8 * (lane >> 4);
                        uint32_t a[4];
                        ldmatrix_x4(a[0], a[1], a[2], a[3], smem_u32(s_plo + off));
                        mma_m16n8k16<T>(o[t][j], a, b0, b1);
                        ldmatrix_x4(a[0], a[1], a[2], a[3], smem_u32(s_p + off));
                        mma_m16n8k16<T>(o[t][j], a, b0, b1);
                    }
                }
            }
        } else if constexpr (MMA && NJ == 2) {
#pragma unroll
            for (int kk = 0; kk < CH / 16; ++kk) {
                uint32_t b0, b1, b2, b3;
                ldmatrix_x4_trans(b0, b1, b2, b3,
                                  smem_u32(vs + (16 * kk + (lane & 7) + 8 * ((lane >> 3) & 1)) * D + 16 * warp + 8 * (lane >> 4)));
#pragma unroll
                for (int t = 0; t < QT; ++t) {
                    const int off = (16 * t + (lane & 15)) * PLD + 16 * kk + 8 * (lane >> 4);
                    uint32_t a[4];
                    ldmatrix_x4(a[0], a[1], a[2], a[3], smem_u32(s_plo + off));
                    mma_m16n8k16<T>(o[t][0], a, b0, b1);
                    mma_m16n8k16<T>(o[t][1], a, b2, b3);
                    ldmatrix_x4(a[0], a[1], a[2], a[3], smem_u32(s_p + off));
                    mma_m16n8k16<T>(o[t][0], a, b0, b1);
                    mma_m16n8k16<T>(o[t][1], a, b2, b3);
                }
            }
        } else if constexpr (MMA) {
            // one n8 tile per warp: a single transposed x4 load holds the V fragments of two k16 steps (rows 32 kk2 + lane)
#pragma unroll
            for (int kk2 = 0; kk2 < CH / 32; ++kk2) {
                uint32_t b[4];
                ldmatrix_x4_trans(b[0], b[1], b[2], b[3], smem_u32(vs + (32 * kk2 + lane) * D + 8 * warp));
#pragma unroll
                for (int half = 0; half < 2; ++half)
#pragma unroll
                    for (int t = 0; t < QT; ++t) {
                        const int off = (16 * t + (lane & 15)) * PLD + 32 * kk2 + 16 * half + 8 * (lane >> 4);
                        uint32_t a[4];
                        ldmatrix_x4(a[0], a[1], a[2], a[3], smem_u32(s_plo + off));
                        mma_m16n8k16<T>(o[t][0], a, b[2 * half], b[2 * half + 1]);
                        ldmatrix_x4(a[0], a[1], a[2], a[3], smem_u32(s_p + off));
                        mma_m16n8k16<T>(o[t][0], a, b[2 * half], b[2 * half + 1]);
                    }
            }
        } else {
            const float *vcol = reinterpret_cast<const float *>(vs) + 8 * NJ * warp + 2 * qc;
            const float *pf = reinterpret_cast<const float *>(s_p);
            for (int k = 0; k < nrows; ++k) {
                const float2 v0 = *reinterpret_cast<const float2 *>(vcol + k * D);
                const float2 v1 = *reinterpret_cast<const float2 *>(vcol + k * D + 8 * (NJ - 1));  // (NJ = 1: v0 again, unused)
#pragma unroll
                for (int t = 0; t < QT; ++t)
#pragma unroll
                    for (int h = 0; h < 2; ++h) {
                        const float p = pf[(16 * t + qr + 8 * h) * PLD + k];
                        o[t][0][2 * h] = fmaf(p, v0.x, o[t][0][2 * h]);
                        o[t][0][2 * h + 1] = fmaf(p, v0.y, o[t][0][2 * h + 1]);
                        if constexpr (NJ == 2) {
                            o[t][NJ - 1][2 * h] = fmaf(p, v1.x, o[t][NJ - 1][2 * h]);
                            o[t][NJ - 1][2 * h + 1] = fmaf(p, v1.y, o[t][NJ - 1][2 * h + 1]);
                        }
                    }
            }
        }
        __syncwarp();
        if (lane == 0) mbar_arrive(&empty[st]);
        if (++st == AS_STAGES) { st = 0; ph ^= 1; }

        if (last_chunk || it == nunits - 1) {
            // ---- segment end: write O / l, or this CTA's partial; the last CTA of a shared segment merges its gq rows
            const bool whole = seg_from_start && last_chunk;
            const int64_t hu0 = (int64_t)s_pre[brow] + (int64_t)(bh - brow * HV) * nch;  // first unit of this segment
            const int first_cta = (int)(((hu0 + 1) * ncta - 1) / total);
            const int last_cta = (int)(((hu0 + nch) * ncta - 1) / total);
            const int nseg = last_cta - first_cta + 1;
            // o[t][j][2h + e] is column 8 NJ w + 2 CE qc + CJ j + CE e: FP8 interleaves the n8 tiles' columns (see O += P V)
            constexpr int CJ = KV8<KT> ? 1 : 8, CE = KV8<KT> ? NJ : 1;
            auto out_val = [&](float A, float L) {  // FP8: the KV head's V scale, once
                if constexpr (KV8<KT>) {
                    const float *const scales[2] = {kv_scale...};
                    return from_f<T>(A / L * scales[1][(bh / NQG) % Hkv]);
                }
                else return from_f<T>(A / L);
            };
#pragma unroll
            for (int t = 0; t < QT; ++t)
#pragma unroll
                for (int h = 0; h < 2; ++h) {
                    const int r = 16 * t + qr + 8 * h;
                    if (r >= gq) continue;
                    if (whole) {
                        T *orow = out + (q0 + r) * D + 8 * NJ * warp + 2 * CE * qc;
#pragma unroll
                        for (int j = 0; j < NJ; ++j) {
                            orow[CJ * j] = out_val(o[t][j][2 * h], l_run[t][h]);
                            orow[CJ * j + CE] = out_val(o[t][j][2 * h + 1], l_run[t][h]);
                        }
                    } else {
                        float *pp = partial + ((q0 + r) * slots_per_head + ((int)blockIdx.x - first_cta)) * (D + 2);
#pragma unroll
                        for (int j = 0; j < NJ; ++j) {
                            __stcg(pp + 2 + 8 * NJ * warp + CJ * j + 2 * CE * qc, o[t][j][2 * h]);
                            __stcg(pp + 2 + 8 * NJ * warp + CJ * j + 2 * CE * qc + CE, o[t][j][2 * h + 1]);
                        }
                        if (warp == 0 && qc == 0) {
                            __stcg(pp, m_run[t][h]);
                            __stcg(pp + 1, l_run[t][h]);
                        }
                    }
                }
            if (!whole) {
                __threadfence();
                named_bar_sync(1, CONSUMERS);
                if (threadIdx.x == 0) {
                    const int old = atomicAdd(tickets + bh, 1);
                    s_last = old == nseg - 1;
                    if (s_last) tickets[bh] = 0;  // self-cleaning: every other sharer has already arrived
                    __threadfence();
                }
                named_bar_sync(1, CONSUMERS);
                if (s_last) {
                    for (int i = threadIdx.x; i < gq * D; i += CONSUMERS) {
                        const int r = i / D, d = i % D;
                        const float *slots = partial + (q0 + r) * slots_per_head * (D + 2);
                        float mw = -INFINITY;
                        for (int s2 = 0; s2 < nseg; ++s2) mw = fmaxf(mw, __ldcg(slots + (int64_t)s2 * (D + 2)));
                        float L = 0.f, A = 0.f;
                        for (int s2 = 0; s2 < nseg; ++s2) {
                            const float *pp = slots + (int64_t)s2 * (D + 2);
                            const float cw2 = expf(__ldcg(pp) - mw);  // every partial holds >= 1 row: finite m
                            L += __ldcg(pp + 1) * cw2;
                            A += __ldcg(pp + 2 + d) * cw2;
                        }
                        out[(q0 + r) * D + d] = out_val(A, L);
                    }
                }
            }
            named_bar_sync(1, CONSUMERS);  // s_q / s_last are reused by the next segment
        }
        next_unit();
    }
}

// The kernels: one name per head width, so that the 128-wide kernels keep the names profiles and tests know them by.
// KT: the cache element type
#define ITB_ATTN_STREAM_ARGS(KT)                                                                                        \
    KT *__restrict__ kcache, KT *__restrict__ vcache, const T *__restrict__ q, const T *__restrict__ kin,            \
        const T *__restrict__ vin, const void *__restrict__ position_id, int pos_flags, T *__restrict__ out, int Smax, \
        int BH, float *__restrict__ partial, int slots_per_head, int *__restrict__ tickets,                           \
        const void *__restrict__ rope_pos, int rope_pos_dtype, int H
#define ITB_ATTN_STREAM_PASS                                                                                            \
    kcache, vcache, q, kin, vin, position_id, pos_flags, out, Smax, BH, partial, slots_per_head, tickets, rope_pos,   \
        rope_pos_dtype, H
#define ITB_ATTN_GQA_ARGS(KT)                                                                                           \
    KT *__restrict__ kcache, KT *__restrict__ vcache, const T *__restrict__ q, const T *__restrict__ kin,            \
        const T *__restrict__ vin, const void *__restrict__ position_id, int pos_flags, T *__restrict__ out, int Smax, \
        int Bn, int Hkv, int G, int NQG, float *__restrict__ partial, int slots_per_head, int *__restrict__ tickets,   \
        const void *__restrict__ rope_pos, int rope_pos_dtype
#define ITB_ATTN_GQA_PASS                                                                                               \
    kcache, vcache, q, kin, vin, position_id, pos_flags, out, Smax, Bn, Hkv, G, NQG, partial, slots_per_head,         \
        tickets, rope_pos, rope_pos_dtype

template <typename T, int WARPS, int U, bool ROPE>
__global__ void __launch_bounds__((WARPS + 1) * 32, AS_CTAS_PER_SM) attn_stream_kernel(ITB_ATTN_STREAM_ARGS(T)) {
    attn_stream_body<T, T, 128, WARPS, U, ROPE ? ROPE_BASE : ROPE_NONE>(ITB_ATTN_STREAM_PASS, nullptr, nullptr, nullptr);  // (pdl_trigger / pdl_wait inside)
}
template <typename T, int WARPS, int U, bool ROPE>
__global__ void __launch_bounds__((WARPS + 1) * 32, AS_CTAS_PER_SM) attn_stream64_kernel(ITB_ATTN_STREAM_ARGS(T)) {
    attn_stream_body<T, T, 64, WARPS, U, ROPE ? ROPE_BASE : ROPE_NONE>(ITB_ATTN_STREAM_PASS, nullptr, nullptr, nullptr);  // (pdl_trigger / pdl_wait inside)
}
template <typename T, int QT, bool ROPE>
__global__ void __launch_bounds__((GQ_WARPS + 1) * 32, AS_CTAS_PER_SM) attn_gqa_kernel(ITB_ATTN_GQA_ARGS(T)) {
    attn_gqa_body<T, T, 128, QT, ROPE ? ROPE_BASE : ROPE_NONE>(ITB_ATTN_GQA_PASS, nullptr, 0);  // (pdl_trigger / pdl_wait inside)
}
template <typename T, int QT, bool ROPE>
__global__ void __launch_bounds__((GQ_WARPS + 1) * 32, AS_CTAS_PER_SM) attn_gqa64_kernel(ITB_ATTN_GQA_ARGS(T)) {
    attn_gqa_body<T, T, 64, QT, ROPE ? ROPE_BASE : ROPE_NONE>(ITB_ATTN_GQA_PASS, nullptr, 0);  // (pdl_trigger / pdl_wait inside)
}

// FP8 E4M3 caches: uint8_t codes + one fp32 scale per KV head, f16 / bf16 activations, both widths in one name each
template <typename T, int D, int WARPS, int U, bool ROPE>
__global__ void __launch_bounds__((WARPS + 1) * 32, AS_CTAS_PER_SM)
    attn_stream_kv8_kernel(ITB_ATTN_STREAM_ARGS(uint8_t), const float *__restrict__ k_scale, const float *__restrict__ v_scale) {
    attn_stream_body<T, uint8_t, D, WARPS, U, ROPE ? ROPE_BASE : ROPE_NONE>(ITB_ATTN_STREAM_PASS, k_scale, v_scale, nullptr);  // (pdl_trigger / pdl_wait inside)
}
template <typename T, int D, int QT, bool ROPE>
__global__ void __launch_bounds__((GQ_WARPS + 1) * 32, AS_CTAS_PER_SM)
    attn_gqa_kv8_kernel(ITB_ATTN_GQA_ARGS(uint8_t), const float *__restrict__ k_scale, const float *__restrict__ v_scale) {
    attn_gqa_body<T, uint8_t, D, QT, ROPE ? ROPE_BASE : ROPE_NONE>(ITB_ATTN_GQA_PASS, nullptr, 0, k_scale, v_scale);  // (pdl_trigger / pdl_wait inside)
}

// RoPE from an inv_freq table: one name per body for every cache type and width (k_scale / v_scale: FP8 caches only)
template <typename T, typename KT, int D, int WARPS, int U>
__global__ void __launch_bounds__((WARPS + 1) * 32, AS_CTAS_PER_SM)
    attn_stream_freq_kernel(ITB_ATTN_STREAM_ARGS(KT), const float *__restrict__ inv_freq, const float *__restrict__ k_scale,
                            const float *__restrict__ v_scale) {
    attn_stream_body<T, KT, D, WARPS, U, ROPE_TABLE>(ITB_ATTN_STREAM_PASS, k_scale, v_scale, inv_freq);  // (pdl_trigger / pdl_wait inside)
}
template <typename T, typename KT, int D, int QT>
__global__ void __launch_bounds__((GQ_WARPS + 1) * 32, AS_CTAS_PER_SM)
    attn_gqa_freq_kernel(ITB_ATTN_GQA_ARGS(KT), const float *__restrict__ inv_freq, const float *__restrict__ k_scale,
                         const float *__restrict__ v_scale) {
    if constexpr (KV8<KT>) attn_gqa_body<T, KT, D, QT, ROPE_TABLE>(ITB_ATTN_GQA_PASS, inv_freq, 0, k_scale, v_scale);
    else attn_gqa_body<T, KT, D, QT, ROPE_TABLE>(ITB_ATTN_GQA_PASS, inv_freq, 0);  // (pdl_trigger / pdl_wait inside)
}

// Sliding window (window >= 1): a query at position p reads cache rows (p - window, p], its own row included.  One name per
// body for every cache type, width and RoPE mode (inv_freq: ROPE_TABLE only; k_scale / v_scale: FP8 caches only)
template <typename T, typename KT, int D, int WARPS, int U, int ROPE>
__global__ void __launch_bounds__((WARPS + 1) * 32, AS_CTAS_PER_SM)
    attn_stream_win_kernel(ITB_ATTN_STREAM_ARGS(KT), const float *__restrict__ inv_freq, const float *__restrict__ k_scale,
                           const float *__restrict__ v_scale, int window) {
    attn_stream_body<T, KT, D, WARPS, U, ROPE, true>(ITB_ATTN_STREAM_PASS, k_scale, v_scale, inv_freq, window);  // (pdl_trigger / pdl_wait inside)
}
template <typename T, typename KT, int D, int QT, int ROPE>
__global__ void __launch_bounds__((GQ_WARPS + 1) * 32, AS_CTAS_PER_SM)
    attn_gqa_win_kernel(ITB_ATTN_GQA_ARGS(KT), const float *__restrict__ inv_freq, const float *__restrict__ k_scale,
                        const float *__restrict__ v_scale, int window) {
    if constexpr (KV8<KT>) attn_gqa_body<T, KT, D, QT, ROPE, true>(ITB_ATTN_GQA_PASS, inv_freq, window, k_scale, v_scale);
    else attn_gqa_body<T, KT, D, QT, ROPE, true>(ITB_ATTN_GQA_PASS, inv_freq, window);  // (pdl_trigger / pdl_wait inside)
}

}  // namespace itb

using namespace itb;

static int stream_slots_per_head(int S_max) { return S_max / 32 + 1; }  // >= chunks per head for every dtype and width

extern "C" int64_t it_b200_attention_kvcache_workspace(int B, int H, int S_max, int D) {
    return (int64_t)B * H * stream_slots_per_head(S_max) * (D + 2) * sizeof(float);
}

template <typename T, typename KT, int D, int ROPE>
static int launch_attn_stream(KT *kc, KT *vc, const T *q, const T *k, const T *v, const void *position_id, int pos_flags,
                              const void *rope_pos, int rope_pos_dtype, const float *inv_freq, T *out, int BH, int H, int S_max,
                              float *workspace, const float *k_scale, const float *v_scale, int window, cudaStream_t st) {
    constexpr int WARPS = 8, U = 4;  // consumer warps x rows per lane and chunk
    constexpr int CH = WARPS * RowCfg<KT, D>::RPW * U;
    constexpr int smem = AS_STAGES * 2 * CH * D * (int)sizeof(KT);
    constexpr const char *what = KV8<KT> ? "AttentionKVCache(FP8 cache): streaming kernel" : "AttentionKVCache: streaming kernel";
    int *tickets = stream_tickets(st, BH);
    if (!tickets) ITB_FAIL("%s: no ticket pool", what);
    const int64_t max_units = (int64_t)BH * (S_max / CH + 1);
    const int grid = (int)std::min<int64_t>(max_units, (int64_t)AS_CTAS_PER_SM * kNumSMs);
    auto go = [&](auto kern, auto... extra) {  // extra: the inv_freq table, FP8 scales
        return launch(what, kern, {dim3(grid), dim3((WARPS + 1) * 32), smem, st}, kc, vc, q, k, v, position_id, pos_flags, out,
                      S_max, BH, workspace, stream_slots_per_head(S_max), tickets, rope_pos, rope_pos_dtype, H, extra...);
    };
    if (window > 0) return go(attn_stream_win_kernel<T, KT, D, WARPS, U, ROPE>, inv_freq, k_scale, v_scale, window);
    constexpr bool R = ROPE == ROPE_BASE;
    if constexpr (ROPE == ROPE_TABLE) return go(attn_stream_freq_kernel<T, KT, D, WARPS, U>, inv_freq, k_scale, v_scale);
    else if constexpr (std::is_same_v<KT, uint8_t>) return go(attn_stream_kv8_kernel<T, D, WARPS, U, R>, k_scale, v_scale);
    else return go(D == 128 ? attn_stream_kernel<T, WARPS, U, R> : attn_stream64_kernel<T, WARPS, U, R>);
}

template <typename T, typename KT, int D, int QT, int ROPE>
static int launch_attn_gqa(KT *kc, KT *vc, const T *q, const T *k, const T *v, const void *position_id, int pos_flags,
                           const void *rope_pos, int rope_pos_dtype, const float *inv_freq, T *out, int B, int Hkv, int G, int S_max,
                           float *workspace, const float *k_scale, const float *v_scale, int window, cudaStream_t st) {
    constexpr int CH = GqaCfg<T, D, KT>::CH;
    constexpr int smem = AS_STAGES * 2 * CH * D * (int)sizeof(KT);
    constexpr const char *what = KV8<KT> ? "AttentionKVCache(FP8 cache): grouped-query kernel" : "AttentionKVCache: grouped-query kernel";
    const int nqg = (G + 16 * QT - 1) / (16 * QT);  // query groups per KV head
    int *tickets = stream_tickets(st, B * Hkv * nqg);
    if (!tickets) ITB_FAIL("%s: no ticket pool", what);
    const int64_t max_units = (int64_t)B * Hkv * nqg * (S_max / CH + 1);
    const int grid = (int)std::min<int64_t>(max_units, (int64_t)AS_CTAS_PER_SM * kNumSMs);
    auto go = [&](auto kern, auto... extra) {  // extra: the inv_freq table, FP8 scales
        return launch(what, kern, {dim3(grid), dim3((GQ_WARPS + 1) * 32), smem, st}, kc, vc, q, k, v, position_id, pos_flags,
                      out, S_max, B, Hkv, G, nqg, workspace, stream_slots_per_head(S_max), tickets, rope_pos, rope_pos_dtype,
                      extra...);
    };
    if (window > 0) return go(attn_gqa_win_kernel<T, KT, D, QT, ROPE>, inv_freq, k_scale, v_scale, window);
    constexpr bool R = ROPE == ROPE_BASE;
    if constexpr (ROPE == ROPE_TABLE) return go(attn_gqa_freq_kernel<T, KT, D, QT>, inv_freq, k_scale, v_scale);
    else if constexpr (std::is_same_v<KT, uint8_t>) return go(attn_gqa_kv8_kernel<T, D, QT, R>, k_scale, v_scale);
    else return go(D == 128 ? attn_gqa_kernel<T, QT, R> : attn_gqa64_kernel<T, QT, R>);
}

// the kernel for head width D and G = Hq / Hkv, with RoPE folded in when rope_pos is given (angles from inv_freq when that
// is given too).  G > 1 takes one query tile of 16 rows for G <= 16, else groups of two tiles (four tiles spill registers
// and, for fp32, exceed the static shared memory)
template <typename T, typename KT, int D>
static int launch_attn_width(KT *kc, KT *vc, const T *q, const T *k, const T *v, const void *position_id, int pos_flags,
                             const void *rope_pos, int rope_pos_dtype, const float *inv_freq, T *out, int B, int Hq, int Hkv,
                             int S_max, float *workspace, const float *k_scale, const float *v_scale, int window,
                             cudaStream_t st) {
    const int G = Hq / Hkv;
    auto go = [&](auto rope) {
        constexpr int R = decltype(rope)::value;
        const void *rp = R ? rope_pos : nullptr;
        const int rpd = R ? rope_pos_dtype : 0;
        if (G == 1)
            return launch_attn_stream<T, KT, D, R>(kc, vc, q, k, v, position_id, pos_flags, rp, rpd, inv_freq, out, B * Hq, Hq,
                                                   S_max, workspace, k_scale, v_scale, window, st);
        if (G <= 16)
            return launch_attn_gqa<T, KT, D, 1, R>(kc, vc, q, k, v, position_id, pos_flags, rp, rpd, inv_freq, out, B, Hkv, G,
                                                   S_max, workspace, k_scale, v_scale, window, st);
        return launch_attn_gqa<T, KT, D, 2, R>(kc, vc, q, k, v, position_id, pos_flags, rp, rpd, inv_freq, out, B, Hkv, G, S_max,
                                               workspace, k_scale, v_scale, window, st);
    };
    if (!rope_pos) return go(std::integral_constant<int, ROPE_NONE>{});
    return inv_freq ? go(std::integral_constant<int, ROPE_TABLE>{}) : go(std::integral_constant<int, ROPE_BASE>{});
}

// Hq query heads over Hkv cache heads.  Hq == Hkv runs attn_stream_kernel; Hq = G Hkv, G > 1, runs attn_gqa_kernel.
// k_scale non-null: the caches hold FP8 E4M3 codes (attn_*_kv8_kernel).
// inv_freq non-null: the folded RoPE's angles are p x inv_freq[c] (f32 [D / 2], checked by the caller).
static int attention_impl(int dtype, void *k_cache, void *v_cache, const void *q, const void *k, const void *v,
                          const void *position_id, int pos_flags, const void *rope_pos, int rope_pos_dtype, void *out,
                          int B, int Hq, int Hkv, int S_max, int D, void *workspace, int64_t workspace_bytes,
                          void *stream, const float *k_scale = nullptr, const float *v_scale = nullptr,
                          const float *inv_freq = nullptr, int window = 0) {
    const int H = Hq;
    const int pos_dtype = pos_flags & 0xff;
    // 128: the reference's only width (attention_kvcache.cu:154); 64: GPT-2 / TinyLlama heads (extension)
    ITB_CHECK(D == 64 || D == 128, "AttentionKVCache: head dim %d is not supported (64 or 128)", D);
    ITB_CHECK(pos_dtype == ITB_I32 || pos_dtype == ITB_U32 || pos_dtype == ITB_I64,
              "AttentionKVCache: position dtype %d must be int32/uint32/int64", pos_dtype);
    ITB_CHECK(window > 0 || !(pos_flags & ITB_POS_RING),
              "AttentionKVCache: a rolling cache (ITB_POS_RING) needs a window: it_b200_attention_kvcache_window");
    ITB_CHECK(!rope_pos || rope_pos_dtype == ITB_I32 || rope_pos_dtype == ITB_U32 || rope_pos_dtype == ITB_I64,
              "AttentionKVCache: rope position dtype %d must be int32/uint32/int64", rope_pos_dtype);
    ITB_CHECK(aligned16(k_cache) && aligned16(v_cache) && aligned16(q) && aligned16(k) && aligned16(v),
              "AttentionKVCache: tensors must be 16-byte aligned");
    const int BH = B * H;
    if (BH == 0) return 0;
    ITB_CHECK(Hkv > 0 && Hq % Hkv == 0, "AttentionKVCache: %d query heads are not a multiple of %d KV heads", Hq, Hkv);
    ITB_CHECK(B <= AS_MAX_B && BH <= 65536, "AttentionKVCache: batch %d x heads %d beyond the kernel's limits (%d rows, 65536 heads)",
              B, H, AS_MAX_B);
    const int64_t need = it_b200_attention_kvcache_workspace(B, H, S_max, D);
    ITB_CHECK(workspace && workspace_bytes >= need, "AttentionKVCache: workspace %lld < %lld bytes",
              (long long)workspace_bytes, (long long)need);
    auto st = (cudaStream_t)stream;
    if (k_scale) {
        ITB_CHECK(dtype == ITB_F16 || dtype == ITB_BF16, "AttentionKVCache(FP8 cache): q / k / v must be f16 or bf16 (dtype %d)", dtype);
        ITB_CHECK(v_scale, "AttentionKVCache(FP8 cache): the V scale is missing");
        ITB_CHECK(((reinterpret_cast<uintptr_t>(k_scale) | reinterpret_cast<uintptr_t>(v_scale)) & 3) == 0,
                  "AttentionKVCache(FP8 cache): scales must be 4-byte aligned");
        auto fp8 = [&](auto tag) {
            using T = decltype(tag);
            auto go = D == 64 ? launch_attn_width<T, uint8_t, 64> : launch_attn_width<T, uint8_t, 128>;
            return go((uint8_t *)k_cache, (uint8_t *)v_cache, (const T *)q, (const T *)k, (const T *)v, position_id, pos_flags,
                      rope_pos, rope_pos_dtype, inv_freq, (T *)out, B, Hq, Hkv, S_max, (float *)workspace, k_scale, v_scale, window, st);
        };
        return dtype == ITB_F16 ? fp8(__half{}) : fp8(__nv_bfloat16{});
    }
    ITB_DISPATCH_FLOAT(dtype, "AttentionKVCache", {
        auto go = D == 64 ? launch_attn_width<T, T, 64> : launch_attn_width<T, T, 128>;
        return go((T *)k_cache, (T *)v_cache, (const T *)q, (const T *)k, (const T *)v, position_id, pos_flags, rope_pos,
                  rope_pos_dtype, inv_freq, (T *)out, B, Hq, Hkv, S_max, (float *)workspace, nullptr, nullptr, window, st);
    });
    return 0;
}

extern "C" int it_b200_attention_kvcache(int dtype, void *k_cache, void *v_cache, const void *q, const void *k,
                                         const void *v, const void *position_id, int pos_dtype, void *out, int B,
                                         int H, int S_max, int D, void *workspace, int64_t workspace_bytes,
                                         void *stream) {
    return attention_impl(dtype, k_cache, v_cache, q, k, v, position_id, pos_dtype, nullptr, 0, out, B, H, H, S_max, D,
                          workspace, workspace_bytes, stream);
}

extern "C" int it_b200_attention_kvcache_gqa(int dtype, void *k_cache, void *v_cache, const void *q, const void *k,
                                             const void *v, const void *position_id, int pos_flags, const void *rope_pos,
                                             int rope_pos_dtype, void *out, int B, int Hq, int Hkv, int S_max, int D,
                                             void *workspace, int64_t workspace_bytes, void *stream) {
    return attention_impl(dtype, k_cache, v_cache, q, k, v, position_id, pos_flags, rope_pos, rope_pos_dtype, out, B, Hq,
                          Hkv, S_max, D, workspace, workspace_bytes, stream);
}

extern "C" int it_b200_attention_kvcache_rope(int dtype, void *k_cache, void *v_cache, const void *q_pre,
                                              const void *k_pre, const void *v, const void *position_id, int pos_dtype,
                                              const void *rope_pos, int rope_pos_dtype, void *out, int B, int H,
                                              int S_max, int D, void *workspace, int64_t workspace_bytes, void *stream) {
    ITB_CHECK(rope_pos != nullptr, "AttentionKVCache+RoPE: rope positions missing");
    return attention_impl(dtype, k_cache, v_cache, q_pre, k_pre, v, position_id, pos_dtype, rope_pos, rope_pos_dtype, out,
                          B, H, H, S_max, D, workspace, workspace_bytes, stream);
}

extern "C" int it_b200_attention_kvcache_fp8(int dtype, void *k_cache, void *v_cache, const void *k_scale, const void *v_scale,
                                             const void *q, const void *k, const void *v, const void *position_id, int pos_flags,
                                             const void *rope_pos, int rope_pos_dtype, void *out, int B, int Hq, int Hkv,
                                             int S_max, int D, void *workspace, int64_t workspace_bytes, void *stream) {
    ITB_CHECK(k_scale && v_scale, "AttentionKVCache(FP8 cache): k_scale and v_scale are required");
    return attention_impl(dtype, k_cache, v_cache, q, k, v, position_id, pos_flags, rope_pos, rope_pos_dtype, out, B, Hq, Hkv,
                          S_max, D, workspace, workspace_bytes, stream, (const float *)k_scale, (const float *)v_scale);
}

// a RoPE inv_freq table: f32, at least D / 2 entries, 4-byte aligned, and only with RoPE positions
static int check_inv_freq(const char *what, const void *rope_pos, const void *inv_freq, int freq_dtype, int64_t freq_len, int D) {
    ITB_CHECK(inv_freq, "%s: inv_freq table missing", what);
    ITB_CHECK(rope_pos, "%s: an inv_freq table needs RoPE positions", what);
    ITB_CHECK(freq_dtype == ITB_F32, "%s: inv_freq must be f32 (dtype %d)", what, freq_dtype);
    ITB_CHECK(freq_len >= D / 2, "%s: inv_freq has %lld entries, dim_head %d needs %d", what, (long long)freq_len, D, D / 2);
    ITB_CHECK((reinterpret_cast<uintptr_t>(inv_freq) & 3) == 0, "%s: inv_freq must be 4-byte aligned", what);
    return 0;
}

extern "C" int it_b200_attention_kvcache_gqa_freq(int dtype, void *k_cache, void *v_cache, const void *q, const void *k,
                                                  const void *v, const void *position_id, int pos_flags, const void *rope_pos,
                                                  int rope_pos_dtype, const void *inv_freq, int freq_dtype, int64_t freq_len,
                                                  void *out, int B, int Hq, int Hkv, int S_max, int D, void *workspace,
                                                  int64_t workspace_bytes, void *stream) {
    if (check_inv_freq("AttentionKVCache+RoPE", rope_pos, inv_freq, freq_dtype, freq_len, D)) return 1;
    return attention_impl(dtype, k_cache, v_cache, q, k, v, position_id, pos_flags, rope_pos, rope_pos_dtype, out, B, Hq,
                          Hkv, S_max, D, workspace, workspace_bytes, stream, nullptr, nullptr, (const float *)inv_freq);
}

extern "C" int it_b200_attention_kvcache_fp8_freq(int dtype, void *k_cache, void *v_cache, const void *k_scale,
                                                  const void *v_scale, const void *q, const void *k, const void *v,
                                                  const void *position_id, int pos_flags, const void *rope_pos,
                                                  int rope_pos_dtype, const void *inv_freq, int freq_dtype, int64_t freq_len,
                                                  void *out, int B, int Hq, int Hkv, int S_max, int D, void *workspace,
                                                  int64_t workspace_bytes, void *stream) {
    ITB_CHECK(k_scale && v_scale, "AttentionKVCache(FP8 cache): k_scale and v_scale are required");
    if (check_inv_freq("AttentionKVCache(FP8 cache)+RoPE", rope_pos, inv_freq, freq_dtype, freq_len, D)) return 1;
    return attention_impl(dtype, k_cache, v_cache, q, k, v, position_id, pos_flags, rope_pos, rope_pos_dtype, out, B, Hq, Hkv,
                          S_max, D, workspace, workspace_bytes, stream, (const float *)k_scale, (const float *)v_scale,
                          (const float *)inv_freq);
}

// Sliding-window decode over every cache type: k_scale / v_scale non-null, FP8 E4M3 codes; rope_pos non-null, RoPE folded in
// (inv_freq non-null: the table's angles, else base 10000).  window >= 1: the query at position p reads rows (p - window, p];
// window 0 runs the unwindowed kernels, as it_b200_attention_kvcache_gqa / _fp8 / _gqa_freq / _fp8_freq do.  ITB_POS_RING:
// the caches are a ring of S_max rows (check_ring)
extern "C" int it_b200_attention_kvcache_window(int dtype, void *k_cache, void *v_cache, const void *k_scale, const void *v_scale,
                                                const void *q, const void *k, const void *v, const void *rope_pos, int rope_pos_dtype,
                                                const void *inv_freq, int freq_dtype, int64_t freq_len, int window,
                                                const void *position_id, int pos_flags, void *out, int B, int Hq, int Hkv, int S_max,
                                                int D, void *workspace, int64_t workspace_bytes, void *stream) {
    ITB_CHECK(window >= 0, "AttentionKVCache: window %d is negative", window);
    if ((pos_flags & ITB_POS_RING) && check_ring("AttentionKVCache", window, S_max, 1)) return 1;
    ITB_CHECK(!k_scale == !v_scale, "AttentionKVCache(FP8 cache): k_scale and v_scale go together");
    if (inv_freq && check_inv_freq(k_scale ? "AttentionKVCache(FP8 cache)+RoPE" : "AttentionKVCache+RoPE", rope_pos, inv_freq,
                                   freq_dtype, freq_len, D))
        return 1;
    return attention_impl(dtype, k_cache, v_cache, q, k, v, position_id, pos_flags, rope_pos, rope_pos_dtype, out, B, Hq, Hkv,
                          S_max, D, workspace, workspace_bytes, stream, (const float *)k_scale, (const float *)v_scale,
                          (const float *)inv_freq, window);
}
