// attention.cu -- AttentionKVCache decode kernel (q-len 1) for sm_90a.
//
// Replaces reference _attention_kvcache_kernel_128_1/_2 (src/kernels/cuda/attention_kvcache.cu:8-169,
// wrapper attention_kvcache.cc:8-56).  Contract kept from the reference:
//   * seq_length = position_id[0] + 1 for every batch row (.cu:17) -- unless the caller asks for PER-ROW positions
//     (ITB_POS_PER_ROW: row b attends to position_id[b] + 1 rows and appends at position_id[b]; SURVEY 8(f-3): ragged
//     batches cannot be served with the reference's element-0 rule)
//   * k, v are appended IN PLACE into the cache INPUT tensors at position_id[0] (.cu:49-53, 89-93)
//   * cache layout [B, H, S_max, 128] contiguous; q/k/v/out [B, H, 1, 128]; scale 1/sqrt(128) (.cu:72)
// Differences by design (DESIGN.md): numerically stable online softmax instead of the reference's
// exp without max-subtraction (same mathematics; quirk q1), f16/bf16 caches in addition to fp32,
// no 2 GiB scratch round trip -- a single kernel when B*H alone fills the 132 SMs.
//
// HBM-bound: every K and V row up to position p is read exactly once with 128-bit loads; a warp
// holds RPW = 32/LPR rows per load instruction (LPR = lanes per 128-wide row: 16 for 2-byte types,
// 32 for fp32), U independent K and V loads are issued before any arithmetic so each lane keeps
// 2*U 16-byte requests in flight.
#include <algorithm>
#include <string>

#include "common.cuh"
#include "gemm.cuh"  // mbarrier / bulk-copy PTX helpers

namespace itb {

constexpr int kD = 128;

template <typename T> struct RowCfg {
    static constexpr int EPL = 16 / sizeof(T);  // elements per lane per row
    static constexpr int LPR = kD / EPL;        // lanes per row
    static constexpr int RPW = 32 / LPR;        // rows per warp-load
};

template <typename P> __device__ __forceinline__ int read_pos(const void *p, int i) { return (int)((const P *)p)[i]; }

// ------------------------------------------------------------------------------------------------------------------
// attn_stream_kernel: the production decode kernel.  Same arithmetic per cache row as attn_decode_kernel, but
//   * the (head, 64-row chunk) work units of the whole batch are FLATTENED and dealt out in equal contiguous ranges to
//     a persistent grid of 2 x 132 CTAs -- a head count that is not a multiple of the CTA slots no longer costs a
//     partly filled last wave, as a split-per-head grid does;
//   * every chunk of K rows and of V rows is ONE contiguous 16 KiB range of the cache ([B,H,S,128] layout), so a
//     producer warp streams it HBM -> shared memory with cp.async.bulk (TMA 1-D) through a full/empty mbarrier ring;
//     bytes in flight are set by the ring depth (2 x 32 KiB per CTA), not by registers per thread;
//   * a head whose units straddle two or three CTAs is finished by the LAST of them to arrive (self-cleaning ticket per
//     head), which merges the (m, l, acc) partials in CTA order -- deterministic, no second kernel.
// The in-place append and the appended row's contribution are done by the CTA that owns the head's last chunk, from
// registers; chunk loads stop at row pos-1, so the append never races the bulk reads.
// ------------------------------------------------------------------------------------------------------------------
constexpr int AS_STAGES = 2;  // ring depth
constexpr int AS_CTAS_PER_SM = 2;

template <typename T, int EPL, int LPR>
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
    const bool lo = col < kD / 2;
#pragma unroll
    for (int j = 0; j < EPL; ++j) {
        const int c = (col + j) & (kD / 2 - 1);
        // each product rounded on its own (__fmul_rn: never fused into the sum), as the RoPE kernel does
        const float a = round_t<T>(__fmul_rn(to_f(x.v[j]), cs_t[c])), b = round_t<T>(__fmul_rn(to_f(xp.v[j]), sn_t[c]));
        x.v[j] = from_f<T>(lo ? a - b : a + b);
    }
}

constexpr int AS_MAX_B = 1024;  // batch rows whose (position, chunk count) the CTA keeps in shared memory

template <typename T, int WARPS, int U, bool ROPE>
__global__ void __launch_bounds__((WARPS + 1) * 32, AS_CTAS_PER_SM)
    attn_stream_kernel(T *__restrict__ kcache, T *__restrict__ vcache, const T *__restrict__ q,
                       const T *__restrict__ kin, const T *__restrict__ vin, const void *__restrict__ position_id,
                       int pos_flags, T *__restrict__ out, int Smax, int BH, float *__restrict__ partial,
                       int slots_per_head, int *__restrict__ tickets, const void *__restrict__ rope_pos,
                       int rope_pos_dtype, int H) {
    using C = RowCfg<T>;
    constexpr int EPL = C::EPL, LPR = C::LPR, RPW = C::RPW;
    constexpr int CH = WARPS * RPW * U;                       // cache rows per chunk
    constexpr int CHUNK_BYTES = CH * kD * (int)sizeof(T);     // 16 KiB for every dtype
    constexpr int CONSUMERS = WARPS * 32;
    extern __shared__ __align__(128) unsigned char ring[];    // stages x { K chunk | V chunk }
    __shared__ __align__(8) uint64_t full[AS_STAGES], empty[AS_STAGES];
    __shared__ float s_m[WARPS], s_l[WARPS];
    __shared__ float s_acc[WARPS][kD];
    __shared__ float s_cs[kD / 2], s_sn[kD / 2];
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
    if (threadIdx.x == 0) {
        for (int s = 0; s < AS_STAGES; ++s) {
            mbar_init(&full[s], 1);
            mbar_init(&empty[s], WARPS);
        }
        fence_mbar_init();
    }
    for (int b = threadIdx.x; b < Bn; b += blockDim.x) {
        int p = pos_dtype == ITB_I64 ? read_pos<int64_t>(position_id, per_row ? b : 0)
                                     : read_pos<int32_t>(position_id, per_row ? b : 0);
        s_pos[b] = min(max(p, 0), Smax - 1);
    }
    __syncthreads();
    if (threadIdx.x == 0) {
        int acc = 0;
        for (int b = 0; b < Bn; ++b) {
            s_pre[b] = acc;
            acc += H * (s_pos[b] / CH + 1);  // chunks per head of row b; the last one holds rows [.., pos) + the appended row
        }
        s_pre[Bn] = acc;
    }
    __syncthreads();
    // Everything this step produced (q, k, v) is read by the consumers, after their wait; this kernel's own append
    // touches row `pos` only, which the bulk loads never include.

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
        nch = pos / CH + 1;
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
                nch = pos / CH + 1;
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
                const int rows = min(CH, pos - c * CH);
                if (rows > 0) {
                    const uint32_t bytes = (uint32_t)rows * kD * (uint32_t)sizeof(T);
                    const int64_t off = ((int64_t)bh * Smax + (int64_t)c * CH) * kD;
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
    // RoPE cos / sin table of the CTA's first batch row: the RoPE positions are a step-old graph input like the cache
    // position, so the powf / sincosf chain runs ahead of the wait; recomputed only when a later segment changes batch row
    int table_b = -1;
    auto rope_table = [&](int b) {
        if (threadIdx.x < kD / 2) {
            const float p = rope_pos_dtype == ITB_I64 ? (float)(int)((const int64_t *)rope_pos)[b]
                                                      : (float)((const int32_t *)rope_pos)[b];
            const float freq = p * powf(10000.f, -(float)(threadIdx.x * 2) / (float)kD);
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
            Vec16<T> qv = ld16(q + (int64_t)bh * kD + col);
            if (ROPE) {
                if (bh / H != table_b) rope_table(bh / H);  // (every earlier reader is behind the previous segment's barriers)
                rope_one<T, EPL, LPR>(qv, col, s_cs, s_sn);
            }
#pragma unroll
            for (int j = 0; j < EPL; ++j) qf[j] = to_f(qv.v[j]) * 0.08838834764831845f;  // 1/sqrt(128)
        }
        const int nvalid = pos - c * CH;  // cache rows of this chunk that exist (<= 0: only the appended row)
        const unsigned char *kb = ring + (size_t)st * 2 * CHUNK_BYTES, *vb = kb + CHUNK_BYTES;
        mbar_wait(&full[st], ph);
#ifndef ATTN_DBG_NOCOMPUTE  // (debug builds only: measures the bare HBM -> smem ring)
        const T *ks = reinterpret_cast<const T *>(kb) + (warp * U * RPW + sub) * kD + col;
        const T *vs = reinterpret_cast<const T *>(vb) + (warp * U * RPW + sub) * kD + col;
        if (nvalid >= CH) {
            // full chunk (every chunk but a head's last): branch-free, so the U rows' load / dot / shuffle chains interleave
            float sc[U];
#pragma unroll
            for (int uu = 0; uu < U; ++uu) {
                const Vec16<T> kv = ld16(ks + uu * RPW * kD);
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
                const Vec16<T> vv = ld16(vs + uu * RPW * kD);
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
                    const Vec16<T> kv = ld16(ks + uu * RPW * kD);
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
                        const Vec16<T> vv = ld16(vs + uu * RPW * kD);
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
            // the row appended this step: rotate k if asked, store k / v in place, add its contribution from registers
            Vec16<T> knew = ld16(kin + (int64_t)bh * kD + col);
            if (ROPE) rope_one<T, EPL, LPR>(knew, col, s_cs, s_sn);
            float d = 0.f;
#pragma unroll
            for (int j = 0; j < EPL; ++j) d += qf[j] * to_f(knew.v[j]);
#pragma unroll
            for (int o = LPR / 2; o > 0; o >>= 1) d += __shfl_xor_sync(0xffffffffu, d, o);
            if (sub == 0) {
                const Vec16<T> vnew = ld16(vin + (int64_t)bh * kD + col);
                st16(kcache + ((int64_t)bh * Smax + pos) * kD + col, knew);
                st16(vcache + ((int64_t)bh * Smax + pos) * kD + col, vnew);
                const float mx2 = fmaxf(m, d);
                const float corr = expf(m - mx2), pnew = expf(d - mx2);
                l = l * corr + pnew;
#pragma unroll
                for (int j = 0; j < EPL; ++j) acc[j] = fmaf(pnew, to_f(vnew.v[j]), acc[j] * corr);
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
            float *slots = partial + (int64_t)bh * slots_per_head * (kD + 2);
            if (threadIdx.x < kD) {
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
                    out[(int64_t)bh * kD + d] = from_f<T>(A / L);
                } else {
                    float *pp = slots + (int64_t)((int)blockIdx.x - first_cta) * (kD + 2);
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
                if (s_last && threadIdx.x < kD) {
                    const int d = threadIdx.x;
                    float mw = -INFINITY;
                    for (int s = 0; s < nseg; ++s) mw = fmaxf(mw, __ldcg(slots + (int64_t)s * (kD + 2)));
                    float L = 0.f, A = 0.f;
                    for (int s = 0; s < nseg; ++s) {
                        const float *pp = slots + (int64_t)s * (kD + 2);
                        const float ms = __ldcg(pp);
                        const float cw = ms > -INFINITY ? expf(ms - mw) : 0.f;
                        L += __ldcg(pp + 1) * cw;
                        A += __ldcg(pp + 2 + d) * cw;
                    }
                    out[(int64_t)bh * kD + d] = from_f<T>(A / L);
                }
            }
            named_bar_sync(1, CONSUMERS);  // s_acc / s_m / s_last are reused by the next segment
        }
        next_unit();
    }
}

}  // namespace itb

using namespace itb;

static int stream_slots_per_head(int S_max) { return S_max / 32 + 1; }  // >= chunks per head for every dtype

extern "C" int64_t it_b200_attention_kvcache_workspace(int B, int H, int S_max, int D) {
    (void)D;
    return (int64_t)B * H * stream_slots_per_head(S_max) * (kD + 2) * sizeof(float);
}

template <typename T, bool ROPE>
static int launch_attn_stream(T *kc, T *vc, const T *q, const T *k, const T *v, const void *position_id, int pos_flags,
                              const void *rope_pos, int rope_pos_dtype, T *out, int BH, int H, int S_max,
                              float *workspace, cudaStream_t st) {
    constexpr int WARPS = 8, U = 4;  // consumer warps x rows per lane and chunk
    constexpr int CH = WARPS * RowCfg<T>::RPW * U;
    const size_t smem = (size_t)AS_STAGES * 2 * CH * kD * sizeof(T);
    auto kern = attn_stream_kernel<T, WARPS, U, ROPE>;
    // the attribute is per DEVICE: a process may own runtimes on several GPUs
    if (cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem) != cudaSuccess) return 1;
    int *tickets = stream_tickets(st, BH);
    if (!tickets) return 1;
    const int64_t max_units = (int64_t)BH * (S_max / CH + 1);
    const int grid = (int)std::min<int64_t>(max_units, (int64_t)AS_CTAS_PER_SM * kNumSMs);
    cudaError_t e = launch_k(kern, dim3(grid), dim3((WARPS + 1) * 32), smem, st, kc, vc, q, k, v, position_id, pos_flags,
                             out, S_max, BH, workspace, stream_slots_per_head(S_max), tickets, rope_pos, rope_pos_dtype, H);
    return e == cudaSuccess ? 0 : 1;
}

static int attention_impl(int dtype, void *k_cache, void *v_cache, const void *q, const void *k, const void *v,
                          const void *position_id, int pos_flags, const void *rope_pos, int rope_pos_dtype, void *out,
                          int B, int H, int S_max, int D, void *workspace, int64_t workspace_bytes, void *stream) {
    const int pos_dtype = pos_flags & 0xff;
    ITB_CHECK(D == kD, "AttentionKVCache: head dim %d != 128 (reference attention_kvcache.cu:154)", D);
    ITB_CHECK(pos_dtype == ITB_I32 || pos_dtype == ITB_U32 || pos_dtype == ITB_I64,
              "AttentionKVCache: position dtype %d must be int32/uint32/int64", pos_dtype);
    ITB_CHECK(!rope_pos || rope_pos_dtype == ITB_I32 || rope_pos_dtype == ITB_U32 || rope_pos_dtype == ITB_I64,
              "AttentionKVCache: rope position dtype %d must be int32/uint32/int64", rope_pos_dtype);
    ITB_CHECK(aligned16(k_cache) && aligned16(v_cache) && aligned16(q) && aligned16(k) && aligned16(v),
              "AttentionKVCache: tensors must be 16-byte aligned");
    const int BH = B * H;
    if (BH == 0) return 0;
    ITB_CHECK(B <= AS_MAX_B && BH <= 65536, "AttentionKVCache: batch %d x heads %d beyond the kernel's limits (%d rows, 65536 heads)",
              B, H, AS_MAX_B);
    const int64_t need = it_b200_attention_kvcache_workspace(B, H, S_max, D);
    ITB_CHECK(workspace && workspace_bytes >= need, "AttentionKVCache: workspace %lld < %lld bytes",
              (long long)workspace_bytes, (long long)need);
    auto st = (cudaStream_t)stream;
    ITB_DISPATCH_FLOAT(dtype, "AttentionKVCache", {
        int rc = rope_pos ? launch_attn_stream<T, true>((T *)k_cache, (T *)v_cache, (const T *)q, (const T *)k,
                                                        (const T *)v, position_id, pos_flags, rope_pos,
                                                        rope_pos_dtype, (T *)out, BH, H, S_max, (float *)workspace, st)
                          : launch_attn_stream<T, false>((T *)k_cache, (T *)v_cache, (const T *)q, (const T *)k,
                                                         (const T *)v, position_id, pos_flags, nullptr, 0, (T *)out,
                                                         BH, H, S_max, (float *)workspace, st);
        ITB_CHECK(rc == 0, "AttentionKVCache: streaming kernel launch failed: %s",
                  cudaGetErrorString(cudaGetLastError()));
        ITB_LAUNCH_CHECK("AttentionKVCache");
    });
    return 0;
}

extern "C" int it_b200_attention_kvcache(int dtype, void *k_cache, void *v_cache, const void *q, const void *k,
                                         const void *v, const void *position_id, int pos_dtype, void *out, int B,
                                         int H, int S_max, int D, void *workspace, int64_t workspace_bytes,
                                         void *stream) {
    return attention_impl(dtype, k_cache, v_cache, q, k, v, position_id, pos_dtype, nullptr, 0, out, B, H, S_max, D,
                          workspace, workspace_bytes, stream);
}

extern "C" int it_b200_attention_kvcache_rope(int dtype, void *k_cache, void *v_cache, const void *q_pre,
                                              const void *k_pre, const void *v, const void *position_id, int pos_dtype,
                                              const void *rope_pos, int rope_pos_dtype, void *out, int B, int H,
                                              int S_max, int D, void *workspace, int64_t workspace_bytes, void *stream) {
    ITB_CHECK(rope_pos != nullptr, "AttentionKVCache+RoPE: rope positions missing");
    return attention_impl(dtype, k_cache, v_cache, q_pre, k_pre, v, position_id, pos_dtype, rope_pos, rope_pos_dtype, out,
                          B, H, S_max, D, workspace, workspace_bytes, stream);
}
