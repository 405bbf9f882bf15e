// decode_stack.cu -- the persistent decode kernel: a whole stack of Llama decoder layers (and, phase by phase, any
// chain of skinny GEMMs + AttentionKVCache) in ONE launch on sm_90a.
//
// Replaces, per decoder layer, the eight launches the fused schedule still issued in round 1 (RMSNorm, grouped q/k/v GEMM,
// RoPE+AttentionKVCache, o-proj GEMM+Add, RMSNorm, grouped gate/up GEMM, Silu*Mul, down GEMM+Add; reference run loop
// src/cuda/cuda_runtime.cc:180-200 dispatching matmul.cc / rms_norm.cu / rope.cu / attention_kvcache.cu / unary.cu /
// element_wise.cu) with five PHASES of one persistent grid, separated by a grid-wide barrier in L2:
//     [RMSNorm ->] q/k/v GEMM | RoPE + attention | o-proj GEMM + residual | [RMSNorm ->] gate/up GEMM | [Silu*Mul ->] down GEMM + residual
// Design (one CTA per SM, 14 warps, ~210 KB of shared memory):
//   * ONE byte stream through ONE shared-memory ring for the whole launch: a producer lane streams every weight tile
//     (TMA 2-D, 128B swizzle, two [64k x 64n] boxes = 16 KiB per stage) and every K / V cache chunk (cp.async.bulk, 16 KiB)
//     of ALL phases in program order.  Weights and cache rows below the position are a step old, so the producer never
//     waits for a phase barrier: the ring keeps filling while the consumers finish a phase, run the barrier and start the
//     next one -- HBM does not idle at phase boundaries the way it does at kernel boundaries.
//   * GEMM phases run on the tensor core through wgmma, swap-AB: the 128 weight columns of a stage are the A operand
//     (MN-major, two m64 halves), the 16 activation rows the K-major B operand (N = 16); one warpgroup issues the MMAs, holds
//     the fp32 accumulator [128 x 16] in registers, releases ring stages through mbarriers and parks each finished tile in
//     one of 4 shared-memory buffers (the epilogue of one tile overlaps the MMAs of the next).
//   * the flattened (tile, k-chunk) units of a phase are dealt to the CTAs in equal contiguous ranges (stream-K): every CTA
//     streams the same number of bytes (+-1 stage).  A tile shared by several CTAs is finished by the LAST of them to
//     arrive (self-cleaning ticket), which sums the fp32 partial tiles in CTA order -- deterministic -- and applies the
//     epilogue (store / + residual, each stage rounded to the storage type exactly like the separate kernels).
//   * the activation operand rides the same ring (2 KiB per stage, TMA from L2, issued after the phase barrier) and is
//     TRANSFORMED in shared memory on its way to the tensor core: RMSNorm (per-row 1/rms from per-tile partial sums of squares
//     written by the producing phase's epilogue, summed in tile order) or Silu(gate) * up -- so the norm / activation
//     kernels and their round trips disappear while every intermediate keeps the rounding of the operator graph.
//   * attention phases: the same ring carries K and V chunks; eight warps do the online softmax from shared memory exactly
//     like attn_stream_kernel (attention.cu), RoPE of q / k folded in, in-place append, per-head partial merge by ticket.
#include <algorithm>
#include <cstdlib>
#include <cstring>
#include <map>
#include <mutex>
#include <vector>

#include "decode_stack.cuh"
#include "gemm.cuh"

namespace itb {

constexpr int DS_STAGES = 8;
constexpr int DS_W_BYTES = 16384;                       // [64 k x 128 n] weights, or one 64-row K / V chunk
constexpr int DS_X_BYTES = 2048;                        // [16 rows x 64 k] activations
constexpr int DS_STAGE_BYTES = DS_W_BYTES + 2 * DS_X_BYTES;  // + second activation box (Silu*Mul: gate | up)
constexpr int DS_EPI_WARPS = 4, DS_XF_WARPS = 4;
constexpr int DS_WARP_MMA = 8, DS_WARP_W = 12, DS_WARP_X = 13;  // MMA warpgroup = warps 8..11
constexpr int DS_THREADS = 14 * 32;
constexpr int DS_ACC_BUFS = 4;
constexpr int DS_ACC_BYTES = DS_ROWS * ACC_LD * 4;     // one parked accumulator [16 columns][ACC_LD]
constexpr int DS_KD = 128;                              // head dim (reference attention_kvcache.cu:154)
constexpr int DS_CH = 64;                               // cache rows per chunk
constexpr int DS_MAX_B = 64;                            // batch rows the attention bookkeeping holds
constexpr int DS_CONS_WARPS = 8;
constexpr int DS_NORMW_MAX = 4096;

__device__ __forceinline__ unsigned ld_acquire_u32(const unsigned *p) {
    unsigned v;
    asm volatile("ld.acquire.gpu.global.u32 %0, [%1];" : "=r"(v) : "l"(p) : "memory");
    return v;
}
__device__ __forceinline__ unsigned ld_relaxed_u32(const unsigned *p) {
    unsigned v;
    asm volatile("ld.relaxed.gpu.global.u32 %0, [%1];" : "=r"(v) : "l"(p) : "memory");
    return v;
}
__device__ __forceinline__ unsigned long long ds_now() {
    unsigned long long t;
    asm volatile("mov.u64 %0, %%globaltimer;" : "=l"(t));
    return t;
}
__device__ __forceinline__ void fence_proxy_async_all() { asm volatile("fence.proxy.async;" ::: "memory"); }
// 16-byte load that bypasses L1: everything an earlier PHASE of the same launch wrote (other SMs, same addresses re-used
// across layers by the planner) must come from L2
template <typename T> __device__ __forceinline__ Vec16<T> ld16_cg(const T *p) {
    Vec16<T> r;
    uint4 u;
    asm volatile("ld.global.cg.v4.u32 {%0,%1,%2,%3}, [%4];" : "=r"(u.x), "=r"(u.y), "=r"(u.z), "=r"(u.w) : "l"(p) : "memory");
    *reinterpret_cast<uint4 *>(r.v) = u;
    return r;
}
template <typename T> __device__ __forceinline__ float ld_cg_f(const T *p) {
    unsigned short u;
    asm volatile("ld.global.cg.u16 %0, [%1];" : "=h"(u) : "l"(p) : "memory");
    T t;
    *reinterpret_cast<unsigned short *>(&t) = u;
    return to_f(t);
}

// generation barrier over the whole grid: {count, gen}.  The last arriver resets the count and bumps the generation; a CTA
// arrives at barrier p only after it has OBSERVED barrier p-1 complete (phase_done), so neither the reset nor an early
// arrival can race with the previous barrier.
__device__ __forceinline__ void grid_arrive(unsigned *bar, unsigned nctas) {
    __threadfence();
    fence_proxy_async_all();  // our generic-proxy stores are read by other CTAs' TMA (async proxy) after the barrier
    const unsigned old = atomicAdd(bar, 1u);
    if (old == nctas - 1) {
        bar[0] = 0u;
        __threadfence();
        atomicAdd(bar + 1, 1u);
    }
}
__device__ __forceinline__ void ds_report(int site, int phase, unsigned gc, unsigned extra);
__device__ __forceinline__ void grid_wait(const unsigned *bar, unsigned gen0, unsigned target, int phase) {
    // polled with RELAXED loads (an acquire load drags a whole-L1 invalidation, CCTL.IVALL, through the SM on every probe);
    // one acquire fence once the generation has been seen
    unsigned spins = 0;
    while ((unsigned)(ld_relaxed_u32(bar + 1) - gen0) < target) {
        ++spins;
        if (spins == (1u << 18)) ds_report(3 /*DSW_X_GRID*/, phase, ld_acquire_u32(bar), ld_acquire_u32(bar + 1) - gen0);
        if (spins > (1u << 24)) __trap();  // a protocol bug must trap, not hang the box
    }
    __threadfence();
    fence_proxy_async_all();
}

template <typename T, int EPL, int LPR>
__device__ __forceinline__ void ds_rope_one(Vec16<T> &x, int col, const float *cs_t, const float *sn_t) {
    Vec16<T> xp;
    {
        uint4 mine = *reinterpret_cast<const uint4 *>(x.v), other;
        other.x = __shfl_xor_sync(0xffffffffu, mine.x, LPR / 2);
        other.y = __shfl_xor_sync(0xffffffffu, mine.y, LPR / 2);
        other.z = __shfl_xor_sync(0xffffffffu, mine.z, LPR / 2);
        other.w = __shfl_xor_sync(0xffffffffu, mine.w, LPR / 2);
        *reinterpret_cast<uint4 *>(xp.v) = other;
    }
    const bool lo = col < DS_KD / 2;
#pragma unroll
    for (int j = 0; j < EPL; ++j) {
        const int c = (col + j) & (DS_KD / 2 - 1);
        // each product rounded on its own (__fmul_rn: never fused into the sum), as the RoPE kernel does
        const float a = round_t<T>(__fmul_rn(to_f(x.v[j]), cs_t[c])), b = round_t<T>(__fmul_rn(to_f(xp.v[j]), sn_t[c]));
        x.v[j] = from_f<T>(lo ? a - b : a + b);
    }
}

// ---- stall diagnostics: a wait that exceeds its budget records {site, phase, stage counter, parity} in host-mapped memory
// (it_b200_decode_stack_debug) and keeps waiting for a second budget -- so every stuck role gets to report -- before it traps
__device__ unsigned *g_ds_dbg = nullptr;
enum { DSW_W_EMPTY = 1, DSW_X_WISSUED, DSW_X_GRID, DSW_MMA_ACC, DSW_MMA_READY, DSW_XF_PHASE, DSW_XF_FULL, DSW_EPI_ACC, DSW_ATT_PHASE,
       DSW_ATT_FULLK, DSW_ATT_FULLV };
__device__ __forceinline__ void ds_report(int site, int phase, unsigned gc, unsigned extra) {
    unsigned *d = g_ds_dbg;
    if (d) {
        unsigned *r = d + ((size_t)blockIdx.x * 16 + (site & 15)) * 4;
        r[0] = 0xD5000000u | (unsigned)site;
        r[1] = (unsigned)phase;
        r[2] = gc;
        r[3] = extra;
        __threadfence_system();
    }
}
// role progress marks: slot 11 + role -> {0xD6.., phase entered}
__device__ __forceinline__ void ds_mark(int role, int phase) {
    unsigned *d = g_ds_dbg;
    if (d) {
        unsigned *r = d + ((size_t)blockIdx.x * 16 + 11 + role) * 4;
        r[0] = 0xD6000000u | (unsigned)role;
        r[1] = (unsigned)phase;
    }
}
__device__ __forceinline__ void ds_mbar_wait(uint64_t *bar, uint32_t parity, int site, int phase, unsigned gc, long long &waited) {
    if (mbar_try_wait(bar, parity)) return;
    const long long t0 = clock64();
    uint32_t spins = 0;
    while (!mbar_try_wait(bar, parity)) {
        ++spins;
        if (spins == (1u << 20)) ds_report(site, phase, gc, parity);
        if (spins > (1u << 25)) __trap();
    }
    waited += clock64() - t0;
}
// chunk probe (tools/ds_trace.py): CTA 0, phase 5 (= second layer's q/k/v GEMM), first 64 chunks: globaltimer at
//   0 W producer starts waiting for the stage   1 weight TMA issued   2 stage full (transform warp)   3 transform done
//   4 MMA thread saw `ready`   5 MMAs + commit issued   6 activation TMA issued
__device__ __forceinline__ void ds_probe(unsigned long long *trace, int nph, int p, int64_t i, int k) {
    if (trace && blockIdx.x == 0 && p == 5 && i < 64)
        trace[(size_t)gridDim.x * nph * 2 + (size_t)gridDim.x * 16 + (size_t)i * 8 + k] = ds_now();
}
// per-role accounting (tools/ds_trace.py): cycles spent blocked on an mbarrier vs. the role's whole life
__device__ __forceinline__ void ds_role_stats(unsigned long long *trace, int nph, int role, long long waited, long long t_begin) {
    if (trace) {
        unsigned long long *r = trace + (size_t)gridDim.x * nph * 2 + ((size_t)blockIdx.x * 8 + role) * 2;
        r[0] = (unsigned long long)waited;
        r[1] = (unsigned long long)(clock64() - t_begin);
    }
}

struct DsShared {
    alignas(8) uint64_t full[DS_STAGES], ready[DS_STAGES], empty[DS_STAGES];
    alignas(8) uint64_t acc_full[DS_ACC_BUFS], acc_empty[DS_ACC_BUFS];
    volatile int phase_done;       // grid barriers known to be complete (published by the X producer)
    volatile unsigned w_issued;    // ring stages the weight producer has claimed so far (global stage counter)
    unsigned gen0;                 // grid-barrier generation when this launch began
    float rinv[DS_ROWS];
    alignas(16) unsigned short normw[DS_NORMW_MAX];  // the RMSNorm weight of the running phase (K <= DS_NORMW_MAX)
    float ss[DS_EPI_WARPS][DS_ROWS];
    int last_flag;
    // attention
    float a_m[DS_CONS_WARPS], a_l[DS_CONS_WARPS];
    float a_acc[DS_CONS_WARPS][DS_KD];
    float cs[DS_KD / 2], sn[DS_KD / 2];
    int a_last;
    int pos[DS_MAX_B];
    int pre[DS_MAX_B + 1];
};

// this CTA's contiguous range [u0, u1) of `total` units
__device__ __forceinline__ void ds_range(int64_t total, int cta, int nctas, int64_t &u0, int64_t &u1, int64_t &geff) {
    geff = total < (int64_t)nctas ? total : (int64_t)nctas;
    if (geff <= 0 || cta >= geff) {
        u0 = u1 = 0;
        return;
    }
    u0 = cta * total / geff;
    u1 = (cta + 1) * total / geff;
}

template <typename T>
__global__ void __launch_bounds__(DS_THREADS, 1) decode_stack_kernel(const DsProgram prog) {
    extern __shared__ uint8_t ds_smem_raw[];
    uint8_t *ring = ds_smem_raw + ((1024u - (smem_u32(ds_smem_raw) & 1023u)) & 1023u);
    __shared__ DsShared sh;

    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    const int cta = blockIdx.x, nctas = gridDim.x;
    const DsPhase *__restrict__ phases = prog.phases;
    const int nph = prog.nphases;

    pdl_trigger();
    const bool in_step = (prog.pos_flags & ITB_POS_IN_STEP) != 0;
    if (in_step) pdl_wait();
    if (threadIdx.x == 0) {
        for (int s = 0; s < DS_STAGES; ++s) {
            mbar_init(&sh.full[s], 1);
            mbar_init(&sh.ready[s], DS_XF_WARPS);
            mbar_init(&sh.empty[s], DS_CONS_WARPS);
        }
        for (int b = 0; b < DS_ACC_BUFS; ++b) {
            mbar_init(&sh.acc_full[b], 128);  // every MMA thread after parking its fragment
            mbar_init(&sh.acc_empty[b], DS_EPI_WARPS);
        }
        fence_mbar_init();
        sh.phase_done = 0;
        sh.w_issued = 0;
    }
    // attention bookkeeping (positions are a step old unless ITB_POS_IN_STEP): clamped position per batch row and the
    // (head, chunk) units before each row -- shared by every attention phase of the program (same H, S_max)
    int attH = 0, attS = 0;
    for (int p = 0; p < nph; ++p)
        if (phases[p].kind == DS_ATTN) {
            attH = phases[p].H;
            attS = phases[p].S_max;
            break;
        }
    const int Bn = prog.rows;
    if (attH) {
        const int pos_dtype = prog.pos_flags & 0xff;
        const bool per_row = (prog.pos_flags & ITB_POS_PER_ROW) != 0;
        for (int b = threadIdx.x; b < Bn; b += blockDim.x) {
            const int i = per_row ? b : 0;
            int pv = pos_dtype == ITB_I64 ? (int)((const int64_t *)prog.position_id)[i] : (int)((const int32_t *)prog.position_id)[i];
            sh.pos[b] = min(max(pv, 0), attS - 1);
        }
    }
    __syncthreads();
    if (attH && threadIdx.x == 0) {
        int acc = 0;
        for (int b = 0; b < Bn; ++b) {
            sh.pre[b] = acc;
            acc += attH * (sh.pos[b] / DS_CH + 1);
        }
        sh.pre[Bn] = acc;
    }
    __syncthreads();
    float *acc_sm = reinterpret_cast<float *>(ring + DS_STAGES * DS_STAGE_BYTES);  // [DS_ACC_BUFS] parked accumulators
    const int64_t att_total = attH ? sh.pre[Bn] : 0;

    // walk of this CTA's attention units
    struct AttWalk {
        int nunits, bh, c, brow, pos, nch;
    };
    auto att_start = [&](AttWalk &w) {
        int64_t u0, u1, geff;
        ds_range(att_total, cta, nctas, u0, u1, geff);
        w.nunits = (int)(u1 - u0);
        w.brow = 0;
        while (w.brow + 1 < Bn && sh.pre[w.brow + 1] <= u0) ++w.brow;
        w.pos = sh.pos[w.brow];
        w.nch = w.pos / DS_CH + 1;
        const int r = (int)(u0 - sh.pre[w.brow]);
        w.bh = w.brow * attH + r / w.nch;
        w.c = r % w.nch;
    };
    auto att_next = [&](AttWalk &w) {
        if (++w.c == w.nch) {
            w.c = 0;
            ++w.bh;
            if (w.bh % attH == 0 && w.bh < Bn * attH) {
                w.brow = w.bh / attH;
                w.pos = sh.pos[w.brow];
                w.nch = w.pos / DS_CH + 1;
            }
        }
    };
    int att_units_mine = 0;
    if (attH) {
        int64_t u0, u1, geff;
        ds_range(att_total, cta, nctas, u0, u1, geff);
        att_units_mine = (int)(u1 - u0);
    }

    if (warp == DS_WARP_W) {
        // =========================== weight / cache producer: the whole program's byte stream ===========================
        if (lane == 0) {
            const uint64_t pol = l2_policy_evict_first();
            unsigned gc = 0;
            long long waited = 0;
            const long long t_begin = clock64();
            for (int p = 0; p < nph; ++p) {
                const DsPhase &ph = phases[p];
                ds_mark(0, p);
                if (ph.kind == DS_GEMM) {
                    const int ntiles = ph.ntiles, kchunks = ph.kchunks, S = ph.nsplit, tpg = ph.tiles_per_group;
                    const int nunits = ntiles * S;
                    const uint32_t tx = DS_W_BYTES + (ph.xform == DS_XF_SILU_MUL ? 2 : 1) * DS_X_BYTES;
                    int s = gc % DS_STAGES;
                    uint32_t par = ((gc / DS_STAGES) & 1) ^ 1;
                    int probe_i = 0;
                    for (int unit = cta; unit < nunits; unit += nctas) {
                        const int tile = unit % ntiles, sp = unit / ntiles;
                        const int kb = sp * kchunks / S, ke = (sp + 1) * kchunks / S;
                        const int n0 = (tile % tpg) * 128;
                        const CUtensorMap *map = &ph.mapW[tile / tpg];
                        for (int kc = kb; kc < ke; ++kc, ++gc, ++probe_i) {
                            ds_probe(prog.trace, nph, p, probe_i, 0);
                            ds_mbar_wait(&sh.empty[s], par, DSW_W_EMPTY, p, gc, waited);
                            mbar_expect_tx(&sh.full[s], tx);
                            uint8_t *dst = ring + (size_t)s * DS_STAGE_BYTES;
                            tma_load_2d(dst, map, &sh.full[s], n0, kc * 64, pol);
                            tma_load_2d(dst + DS_W_BYTES / 2, map, &sh.full[s], n0 + 64, kc * 64, pol);
                            sh.w_issued = gc + 1;
                            ds_probe(prog.trace, nph, p, probe_i, 1);
                            if (++s == DS_STAGES) {
                                s = 0;
                                par ^= 1;
                            }
                        }
                    }
                } else {
                    AttWalk w;
                    att_start(w);
                    const T *kcache = (const T *)ph.kcache, *vcache = (const T *)ph.vcache;
                    for (int it = 0; it < w.nunits; ++it, gc += 2) {
                        const int sk = gc % DS_STAGES, sv = (gc + 1) % DS_STAGES;
                        const int rows = min(DS_CH, w.pos - w.c * DS_CH);
                        const uint32_t bytes = rows > 0 ? (uint32_t)rows * DS_KD * (uint32_t)sizeof(T) : 0;
                        const int64_t off = ((int64_t)w.bh * attS + (int64_t)w.c * DS_CH) * DS_KD;
                        ds_mbar_wait(&sh.empty[sk], ((gc / DS_STAGES) & 1) ^ 1, DSW_W_EMPTY, p, gc, waited);
                        if (bytes) {
                            mbar_expect_tx(&sh.full[sk], bytes);
                            bulk_load_1d(ring + (size_t)sk * DS_STAGE_BYTES, kcache + off, bytes, &sh.full[sk], pol);
                        } else {
                            mbar_arrive(&sh.full[sk]);
                        }
                        ds_mbar_wait(&sh.empty[sv], (((gc + 1) / DS_STAGES) & 1) ^ 1, DSW_W_EMPTY, p, gc + 1, waited);
                        if (bytes) {
                            mbar_expect_tx(&sh.full[sv], bytes);
                            bulk_load_1d(ring + (size_t)sv * DS_STAGE_BYTES, vcache + off, bytes, &sh.full[sv], pol);
                        } else {
                            mbar_arrive(&sh.full[sv]);
                        }
                        sh.w_issued = gc + 2;
                        att_next(w);
                    }
                }
            }
            ds_role_stats(prog.trace, nph, 0, waited, t_begin);
            pdl_wait();
        }
    } else if (warp == DS_WARP_X) {
        // ============ activation producer + this CTA's grid-barrier waiter (publishes phase_done to the other warps) ============
        // the generation is sampled after griddepcontrol.wait (the previous kernel may be another decode_stack launch still
        // using the barrier) and BEFORE this CTA's arriver thread can reach barrier 0 (named barrier 4 with warps 0..7): no
        // barrier of this launch can complete until every CTA has sampled
        if (lane == 0) {
            pdl_wait();
            sh.gen0 = ld_acquire_u32(prog.grid_bar + 1);
        }
        __syncwarp();
        named_bar_sync(4, (DS_EPI_WARPS + DS_XF_WARPS + 1) * 32);
        if (lane == 0) {
            const uint64_t pol = l2_policy_evict_last();
            const unsigned gen0 = sh.gen0;
            unsigned gc = 0;
            for (int p = 0; p < nph; ++p) {
                const DsPhase &ph = phases[p];
                ds_mark(1, p);
                if (p > 0) grid_wait(prog.grid_bar, gen0, (unsigned)p, p);
                sh.phase_done = p;
                if (prog.trace) prog.trace[((size_t)cta * nph + p) * 2] = ds_now();
                if (ph.kind == DS_GEMM) {
                    const int ntiles = ph.ntiles, kchunks = ph.kchunks, S = ph.nsplit;
                    const int nunits = ntiles * S;
                    const bool two = ph.xform == DS_XF_SILU_MUL;
                    const CUtensorMap *mx = &ph.mapX, *mx2 = &ph.mapX2;
                    int s = gc % DS_STAGES, probe_i = 0;
                    for (int unit = cta; unit < nunits; unit += nctas) {
                        const int sp = unit / ntiles;
                        const int kb = sp * kchunks / S, ke = (sp + 1) * kchunks / S;
                        for (int kc = kb; kc < ke; ++kc, ++gc, ++probe_i) {
                            unsigned spins = 0;
                            while (sh.w_issued <= gc) {
                                ++spins;
                                if (spins == (1u << 21)) ds_report(DSW_X_WISSUED, p, gc, sh.w_issued);
                                if (spins > (1u << 27)) __trap();
                            }
                            uint8_t *dst = ring + (size_t)s * DS_STAGE_BYTES + DS_W_BYTES;
                            tma_load_2d(dst, mx, &sh.full[s], kc * 64, 0, pol);
                            if (two) tma_load_2d(dst + DS_X_BYTES, mx2, &sh.full[s], kc * 64, 0, pol);
                            ds_probe(prog.trace, nph, p, probe_i, 6);
                            if (++s == DS_STAGES) s = 0;
                        }
                    }
                } else {
                    gc += 2u * (unsigned)att_units_mine;
                }
            }
            // the last phase's barrier is not waited for by anybody: the kernel boundary orders its outputs
        }
    } else if (warp >= DS_WARP_MMA && warp < DS_WARP_MMA + 4) {
        // =========================== MMA warpgroup: drives the tensor core ===========================
        const bool leader = (threadIdx.x & 127) == 0;
        const uint32_t ring_u32 = smem_u32(ring);
        unsigned gc = 0, seg = 0;
        long long waited = 0;
        const long long t_begin = clock64();
        for (int p = 0; p < nph; ++p) {
            const DsPhase &ph = phases[p];
            if (leader) ds_mark(2, p);
            if (ph.kind != DS_GEMM) {
                gc += 2u * (unsigned)att_units_mine;
                continue;
            }
            // never run ahead of the previous phase: the `ready` barriers are also advanced by the attention consumers, and one
            // parity bit cannot tell their completion of an EARLIER use of a stage from the one this warpgroup waits for
            {
                unsigned spins = 0;
                while (sh.phase_done < p) {
                    ++spins;
                    if (spins == (1u << 21) && leader) ds_report(DSW_MMA_ACC, p, gc, 0xFFFFu);
                    if (spins > (1u << 27)) __trap();
                }
            }
            const int ntiles = ph.ntiles, kchunks = ph.kchunks, S = ph.nsplit;
            const int nunits = ntiles * S;
            int s = gc % DS_STAGES, probe_i = 0;
            uint32_t par = (gc / DS_STAGES) & 1;
            for (int unit = cta; unit < nunits; unit += nctas) {
                const int sp = unit / ntiles;
                const int kb = sp * kchunks / S, ke = (sp + 1) * kchunks / S;
                const unsigned buf = seg % DS_ACC_BUFS;
                float d0[DS_ROWS / 2], d1[DS_ROWS / 2];  // weight columns 0..63 / 64..127 of the tile
#pragma unroll
                for (int j = 0; j < DS_ROWS / 2; ++j) d0[j] = d1[j] = 0.f;
                for (int kc = kb; kc < ke; ++kc, ++gc, ++probe_i) {
                    ds_mbar_wait(&sh.ready[s], par, DSW_MMA_READY, p, gc, waited);
                    if (leader) ds_probe(prog.trace, nph, p, probe_i, 4);
                    const uint32_t wb = ring_u32 + s * DS_STAGE_BYTES, xb = wb + DS_W_BYTES;
                    wg_fence();
#pragma unroll
                    for (int kk = 0; kk < 4; ++kk) {
                        // A: the [64k x 64n] box of each half (8 KB apart), 8-row k groups 1 KB apart (SBO), one k16 step = 2 KB
                        const uint64_t a_desc = gmma_desc_sw128(wb + kk * 2048, DS_W_BYTES / 2, 1024);
                        // B: [16 rows x 128 B], 8-row groups 1 KB apart, one k16 step = 32 B inside the row
                        const uint64_t b_desc = gmma_desc_sw128(xb + kk * 32, 0, 1024);
                        Wgmma<T, DS_ROWS>::template mma<1, 0>(d0, a_desc, b_desc, 1u);
                        Wgmma<T, DS_ROWS>::template mma<1, 0>(d1, a_desc + ((DS_W_BYTES / 2) >> 4), b_desc, 1u);
                    }
                    wg_commit();
                    wg_wait<0>();
                    if (leader) {
                        mbar_arrive_n(&sh.empty[s], DS_CONS_WARPS);
                        ds_probe(prog.trace, nph, p, probe_i, 5);
                    }
                    if (++s == DS_STAGES) {
                        s = 0;
                        par ^= 1;
                    }
                }
                ds_mbar_wait(&sh.acc_empty[buf], ((seg / DS_ACC_BUFS) & 1) ^ 1, DSW_MMA_ACC, p, seg, waited);
                acc_park<DS_ROWS>(d0, acc_sm + buf * (DS_ACC_BYTES / 4), 0);
                acc_park<DS_ROWS>(d1, acc_sm + buf * (DS_ACC_BYTES / 4), 64);
                mbar_arrive(&sh.acc_full[buf]);
                ++seg;
            }
        }
        if (leader) ds_role_stats(prog.trace, nph, 2, waited, t_begin);
    }

    // ------------------------------------------------------------------------------------------------------------------
    // warps 0..7: epilogue (0-3) / transform (4-7) in GEMM phases, attention consumers in attention phases
    // ------------------------------------------------------------------------------------------------------------------
    if (warp < DS_EPI_WARPS + DS_XF_WARPS) {
        pdl_wait();
        named_bar_sync(4, (DS_EPI_WARPS + DS_XF_WARPS + 1) * 32);
        const bool is_epi = warp < DS_EPI_WARPS;
        const int xt = threadIdx.x - DS_EPI_WARPS * 32;  // transform thread index 0..127
        unsigned gc = 0, seg = 0;
        long long waited = 0;
        const long long t_begin = clock64();
        const int rows = prog.rows;
        for (int p = 0; p < nph; ++p) {
            const DsPhase &ph = phases[p];
            if (threadIdx.x == 0) ds_mark(3, p);
            if (xt == 0) ds_mark(4, p);
            if (ph.kind == DS_GEMM) {
                const int ntiles = ph.ntiles, kchunks = ph.kchunks, S = ph.nsplit, K = ph.K;
                const int nunits = ntiles * S;
                if (!is_epi) {
                    // ---------------- transform warps ----------------
                    const int xform = ph.xform;
                    const T *norm_w = (const T *)ph.norm_w;
                    const bool w_in_smem = xform == DS_XF_RMSNORM && K <= DS_NORMW_MAX && K % 8 == 0;
                    if (xform == DS_XF_RMSNORM) {
                        named_bar_sync(3, DS_XF_WARPS * 32);  // the previous norm phase's readers of rinv / normw are done
                        // the RMSNorm weight (a constant) goes to shared memory ahead of the phase barrier
                        if (w_in_smem)
                            for (int i = xt; i < K / 8; i += DS_XF_WARPS * 32)
                                *reinterpret_cast<uint4 *>(&sh.normw[i * 8]) = *reinterpret_cast<const uint4 *>(norm_w + i * 8);
                        unsigned spins = 0;
                        while (sh.phase_done < p) {
                            ++spins;
                            if (spins == (1u << 21) && xt == 0) ds_report(DSW_XF_PHASE, p, gc, sh.phase_done);
                            if (spins > (1u << 27)) __trap();
                        }
                        if (ph.ss_in) {
                            // 8 threads per row, each sums every 8th tile's partial (independent loads in flight), then a
                            // fixed xor tree over the 8 lanes: deterministic, ~1 L2 round trip instead of one per tile
                            const int r = xt >> 3, c8 = xt & 7;
                            const float *sp_ = ph.ss_in + r;
                            const int nt = ph.ss_in_tiles;
                            float part = 0.f;
#pragma unroll 4
                            for (int tt = c8; tt < nt; tt += 8) part += __ldcg(sp_ + tt * DS_ROWS);
                            part += __shfl_xor_sync(0xffffffffu, part, 4);
                            part += __shfl_xor_sync(0xffffffffu, part, 2);
                            part += __shfl_xor_sync(0xffffffffu, part, 1);
                            if (c8 == 0) sh.rinv[r] = rsqrtf(part / (float)K + 0.00001f);
                        } else {
                            // no producer phase (first layer: the rows come from the embedding gather): reduce them here
                            const T *xr = (const T *)ph.x_raw;
                            const int xw = warp - DS_EPI_WARPS;
                            for (int r = xw; r < DS_ROWS; r += DS_XF_WARPS) {
                                float ssum = 0.f;
                                if (r < rows)
                                    for (int i = lane; i < K / 8; i += 32) {
                                        const Vec16<T> a = ld16_cg(xr + (int64_t)r * K + i * 8);
#pragma unroll
                                        for (int j = 0; j < Vec16<T>::N; ++j) {
                                            const float f = to_f(a.v[j]);
                                            ssum += f * f;
                                        }
                                    }
                                ssum = warp_sum(ssum);
                                if (lane == 0) sh.rinv[r] = rsqrtf(ssum / (float)K + 0.00001f);
                            }
                        }
                        named_bar_sync(3, DS_XF_WARPS * 32);
                    }
                    const int t = xt >> 3, c = xt & 7;                       // row, 16-byte chunk of this thread
                    const int sw_off = t * 128 + ((c ^ (t & 7)) << 4);        // 128B-swizzled position inside the X box
                    const float rinv = xform == DS_XF_RMSNORM ? sh.rinv[t] : 0.f;
                    int s = gc % DS_STAGES, probe_i = 0;
                    uint32_t par = (gc / DS_STAGES) & 1;
                    for (int unit = cta; unit < nunits; unit += nctas) {
                        const int sp = unit / ntiles;
                        const int kb = sp * kchunks / S, ke = (sp + 1) * kchunks / S;
                        for (int kc = kb; kc < ke; ++kc, ++gc, ++probe_i) {
                            ds_mbar_wait(&sh.full[s], par, DSW_XF_FULL, p, gc, waited);
                            if (xt == 0) ds_probe(prog.trace, nph, p, probe_i, 2);
                            if (xform != DS_XF_NONE) {
                                uint8_t *xs = ring + (size_t)s * DS_STAGE_BYTES + DS_W_BYTES;
                                Vec16<T> a = *reinterpret_cast<const Vec16<T> *>(xs + sw_off), o;
                                if (xform == DS_XF_RMSNORM) {
                                    const int k0 = kc * 64 + c * 8;
                                    Vec16<T> w;
                                    if (w_in_smem) {
                                        if (k0 < K) w = *reinterpret_cast<const Vec16<T> *>(&sh.normw[k0]);
                                        else
#pragma unroll
                                            for (int j = 0; j < 8; ++j) w.v[j] = from_f<T>(0.f);
                                    } else {
#pragma unroll
                                        for (int j = 0; j < 8; ++j) w.v[j] = k0 + j < K ? norm_w[k0 + j] : from_f<T>(0.f);
                                    }
#pragma unroll
                                    for (int j = 0; j < 8; ++j) o.v[j] = from_f<T>(round_t<T>(to_f(a.v[j]) * rinv) * to_f(w.v[j]));
                                } else {
                                    const Vec16<T> b = *reinterpret_cast<const Vec16<T> *>(xs + DS_X_BYTES + sw_off);
#pragma unroll
                                    for (int j = 0; j < 8; ++j) {
                                        const float g = to_f(a.v[j]);
                                        o.v[j] = from_f<T>(round_t<T>(g / (1.f + expf(-g))) * to_f(b.v[j]));
                                    }
                                }
                                *reinterpret_cast<Vec16<T> *>(xs + sw_off) = o;
                                fence_proxy_async();  // generic-proxy smem writes -> visible to the tensor core (async proxy)
                            }
                            __syncwarp();
                            if (lane == 0) mbar_arrive(&sh.ready[s]);
                            if (xt == 0) ds_probe(prog.trace, nph, p, probe_i, 3);
                            if (++s == DS_STAGES) {
                                s = 0;
                                par ^= 1;
                            }
                        }
                    }
                } else {
                    // ---------------- epilogue warps: accumulator -> (partial tile, ticket, fix-up) -> output ----------------
                    const int quad = warp & 3;
                    const int col = quad * 32 + lane;  // column inside the tile == row of the parked accumulator
                    const int tpg = ph.tiles_per_group, npg = ph.n_per_group, epi = ph.epi;
                    float *partial = ph.partial;
                    int *tickets = ph.tickets;
                    for (int unit = cta; unit < nunits; unit += nctas) {
                        const int tile = unit % ntiles, sp = unit / ntiles;
                        const int kb = sp * kchunks / S, ke = (sp + 1) * kchunks / S;
                        const unsigned buf = seg % DS_ACC_BUFS;
                        ds_mbar_wait(&sh.acc_full[buf], (seg / DS_ACC_BUFS) & 1, DSW_EPI_ACC, p, seg, waited);
                        uint32_t v[16];
                        acc_row<16>(acc_sm + buf * (DS_ACC_BYTES / 4), col, 0, v);
                        __syncwarp();
                        if (lane == 0) mbar_arrive(&sh.acc_empty[buf]);
                        ++seg;
                        gc += (unsigned)(ke - kb);
                        bool do_epi = true;
                        if (S > 1) {
                            // split-K: every split parks its fp32 partial tile; the LAST to arrive (ticket) sums them in split order
                            float *slot = partial + ((int64_t)tile * S + sp) * (DS_ROWS * 128);
#pragma unroll
                            for (int j = 0; j < DS_ROWS; ++j) __stcg(slot + j * 128 + col, __uint_as_float(v[j]));
                            __threadfence();
                            named_bar_sync(1, DS_EPI_WARPS * 32);
                            if (threadIdx.x == 0) {
                                const int old = atomicAdd(tickets + tile, 1);
                                sh.last_flag = old == S - 1;
                                if (sh.last_flag) tickets[tile] = 0;  // self-cleaning: every other split has arrived
                                __threadfence();
                            }
                            named_bar_sync(1, DS_EPI_WARPS * 32);
                            do_epi = sh.last_flag != 0;
                            if (do_epi) {
                                const float *base = partial + (int64_t)tile * S * (DS_ROWS * 128);
                                float f[DS_ROWS];
#pragma unroll
                                for (int j = 0; j < DS_ROWS; ++j) f[j] = 0.f;
                                for (int sidx = 0; sidx < S; ++sidx)
#pragma unroll
                                    for (int j = 0; j < DS_ROWS; ++j) f[j] += __ldcg(base + sidx * (DS_ROWS * 128) + j * 128 + col);
#pragma unroll
                                for (int j = 0; j < DS_ROWS; ++j) v[j] = __float_as_uint(f[j]);
                            }
                        }
                        if (do_epi) {
                            const int g = tile / tpg, n = (tile % tpg) * 128 + col;
                            const bool nok = n < npg;
                            T *out = (T *)ph.out[g];
                            if (epi == DS_EPI_STORE) {
                                if (nok)
#pragma unroll
                                    for (int j = 0; j < DS_ROWS; ++j)
                                        if (j < rows) out[(int64_t)j * npg + n] = from_f<T>(__uint_as_float(v[j]));
                            } else {
                                const T *res = (const T *)ph.residual;
                                float resv[DS_ROWS];
#pragma unroll
                                for (int j = 0; j < DS_ROWS; ++j) resv[j] = (nok && j < rows) ? ld_cg_f(res + (int64_t)j * npg + n) : 0.f;
                                float sq[DS_ROWS];
#pragma unroll
                                for (int j = 0; j < DS_ROWS; ++j) {
                                    // MatMul output rounded as the separate kernel stores it, then Add(residual, .) rounded
                                    const float f = round_t<T>(resv[j] + round_t<T>(__uint_as_float(v[j])));
                                    if (nok && j < rows) out[(int64_t)j * npg + n] = from_f<T>(f);
                                    sq[j] = (nok && j < rows) ? f * f : 0.f;
                                }
                                if (ph.ss_out) {
#pragma unroll
                                    for (int j = 0; j < DS_ROWS; ++j) {
                                        const float w = warp_sum(sq[j]);
                                        if (lane == 0) sh.ss[quad][j] = w;
                                    }
                                    named_bar_sync(1, DS_EPI_WARPS * 32);
                                    if (threadIdx.x < DS_ROWS)
                                        __stcg(ph.ss_out + tile * DS_ROWS + threadIdx.x,
                                               ((sh.ss[0][threadIdx.x] + sh.ss[1][threadIdx.x]) + sh.ss[2][threadIdx.x]) + sh.ss[3][threadIdx.x]);
                                    named_bar_sync(1, DS_EPI_WARPS * 32);
                                }
                            }
                        }
                    }
                    // phase done for this CTA: publish and arrive at the grid barrier
                    named_bar_sync(1, DS_EPI_WARPS * 32);
                    if (threadIdx.x == 0 && p + 1 < nph) {
                        // never arrive at barrier p before barrier p-1 has completed (a CTA without work in this phase would
                        // otherwise mix its arrival into the previous barrier's count)
                        unsigned spins = 0;
                        while (sh.phase_done < p) {
                            ++spins;
                            if (spins == (1u << 21)) ds_report(DSW_EPI_ACC, p, gc, 0xFFFFu);
                            if (spins > (1u << 27)) __trap();
                        }
                        if (prog.trace) prog.trace[((size_t)cta * nph + p) * 2 + 1] = ds_now();
                        grid_arrive(prog.grid_bar, (unsigned)nctas);
                    }
                }
                continue;
            }

            // ======================= attention phase: warps 0..7 are the consumers =======================
            {
                unsigned spins = 0;
                while (sh.phase_done < p) {
                    ++spins;
                    if (spins == (1u << 21) && threadIdx.x == 0) ds_report(DSW_ATT_PHASE, p, gc, sh.phase_done);
                    if (spins > (1u << 27)) __trap();
                }
            }
            constexpr int EPL = 16 / sizeof(T), LPR = DS_KD / EPL, RPW = 32 / LPR;
            constexpr int U = DS_CH / (DS_CONS_WARPS * RPW);
            constexpr int CONSUMERS = DS_CONS_WARPS * 32;
            const int H = ph.H, Smax = ph.S_max;
            T *kcache = (T *)ph.kcache, *vcache = (T *)ph.vcache;
            const T *q = (const T *)ph.q, *kin = (const T *)ph.k, *vin = (const T *)ph.v;
            T *outp = (T *)ph.attn_out;
            AttWalk w;
            att_start(w);
            int table_b = -1;
            auto rope_table = [&](int b) {
                if (threadIdx.x < DS_KD / 2) {
                    const float pp = prog.rope_pos_dtype == ITB_I64 ? (float)(int)((const int64_t *)prog.rope_pos)[b]
                                                                   : (float)((const int32_t *)prog.rope_pos)[b];
                    const float freq = pp * powf(10000.f, -(float)(threadIdx.x * 2) / (float)DS_KD);
                    sh.cs[threadIdx.x] = round_t<T>(cosf(freq));
                    sh.sn[threadIdx.x] = round_t<T>(sinf(freq));
                }
                named_bar_sync(2, CONSUMERS);
                table_b = b;
            };
            const bool rope = prog.rope_pos != nullptr;
            if (rope && w.nunits > 0) rope_table(w.bh / H);
            const int sub = lane / LPR;
            const int colq = (lane % LPR) * EPL;
            float qf[EPL], m = -INFINITY, l = 0.f, acc[EPL];
            bool seg_from_start = false;
            const int64_t geff = att_total < (int64_t)nctas ? att_total : (int64_t)nctas;
            for (int it = 0; it < w.nunits; ++it, gc += 2) {
                const int bh = w.bh, c = w.c, pos = w.pos, nch = w.nch;
                if (it == 0 || c == 0) {
                    seg_from_start = c == 0;
                    m = -INFINITY;
                    l = 0.f;
#pragma unroll
                    for (int j = 0; j < EPL; ++j) acc[j] = 0.f;
                    Vec16<T> qv = ld16_cg(q + (int64_t)bh * DS_KD + colq);
                    if (rope) {
                        if (bh / H != table_b) rope_table(bh / H);
                        ds_rope_one<T, EPL, LPR>(qv, colq, sh.cs, sh.sn);
                    }
#pragma unroll
                    for (int j = 0; j < EPL; ++j) qf[j] = to_f(qv.v[j]) * 0.08838834764831845f;  // 1/sqrt(128)
                }
                const int nvalid = pos - c * DS_CH;
                const int sk = gc % DS_STAGES, sv = (gc + 1) % DS_STAGES;
                const unsigned char *kb = ring + (size_t)sk * DS_STAGE_BYTES, *vb = ring + (size_t)sv * DS_STAGE_BYTES;
                ds_mbar_wait(&sh.full[sk], (gc / DS_STAGES) & 1, DSW_ATT_FULLK, p, gc, waited);
                ds_mbar_wait(&sh.full[sv], ((gc + 1) / DS_STAGES) & 1, DSW_ATT_FULLV, p, gc + 1, waited);
                const T *ks = reinterpret_cast<const T *>(kb) + (warp * U * RPW + sub) * DS_KD + colq;
                const T *vs = reinterpret_cast<const T *>(vb) + (warp * U * RPW + sub) * DS_KD + colq;
                if (nvalid >= DS_CH) {
                    // full chunk (every chunk but a head's last): branch-free, so the U rows' load / dot / shuffle chains interleave
                    float sc[U];
#pragma unroll
                    for (int uu = 0; uu < U; ++uu) {
                        const Vec16<T> kv = ld16(ks + uu * RPW * DS_KD);
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
                        const Vec16<T> vv = ld16(vs + uu * RPW * DS_KD);
                        const float pe = expf(sc[uu] - mx);
                        l += pe;
#pragma unroll
                        for (int j = 0; j < EPL; ++j) acc[j] = fmaf(pe, to_f(vv.v[j]), acc[j]);
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
                            const Vec16<T> kv = ld16(ks + uu * RPW * DS_KD);
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
                                const Vec16<T> vv = ld16(vs + uu * RPW * DS_KD);
                                const float pe = expf(sc[uu] - mx);
                                l += pe;
#pragma unroll
                                for (int j = 0; j < EPL; ++j) acc[j] = fmaf(pe, to_f(vv.v[j]), acc[j]);
                            }
                        }
                        m = mx;
                    }
                }
                __syncwarp();
                if (lane == 0) {
                    mbar_arrive(&sh.empty[sk]);
                    mbar_arrive(&sh.empty[sv]);
                    if (warp >= DS_EPI_WARPS) {  // keeps the `ready` barriers' parity in step with the stage counter
                        mbar_arrive(&sh.ready[sk]);
                        mbar_arrive(&sh.ready[sv]);
                    }
                }

                const bool last_chunk = c == nch - 1;
                if (last_chunk && warp == 0) {
                    // the row appended this step: rotate k, store k / v in place, add its contribution from registers
                    Vec16<T> knew = ld16_cg(kin + (int64_t)bh * DS_KD + colq);
                    if (rope) ds_rope_one<T, EPL, LPR>(knew, colq, sh.cs, sh.sn);
                    float d = 0.f;
#pragma unroll
                    for (int j = 0; j < EPL; ++j) d += qf[j] * to_f(knew.v[j]);
#pragma unroll
                    for (int o = LPR / 2; o > 0; o >>= 1) d += __shfl_xor_sync(0xffffffffu, d, o);
                    if (sub == 0) {
                        const Vec16<T> vnew = ld16_cg(vin + (int64_t)bh * DS_KD + colq);
                        st16(kcache + ((int64_t)bh * Smax + pos) * DS_KD + colq, knew);
                        st16(vcache + ((int64_t)bh * Smax + pos) * DS_KD + colq, vnew);
                        const float mx2 = fmaxf(m, d);
                        const float corr = expf(m - mx2), pnew = expf(d - mx2);
                        l = l * corr + pnew;
#pragma unroll
                        for (int j = 0; j < EPL; ++j) acc[j] = fmaf(pnew, to_f(vnew.v[j]), acc[j] * corr);
                        m = mx2;
                    }
                }

                if (last_chunk || it == w.nunits - 1) {
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
                        for (int j = 0; j < EPL; ++j) sh.a_acc[warp][colq + j] = acc[j];
                        if (lane == 0) {
                            sh.a_m[warp] = m;
                            sh.a_l[warp] = l;
                        }
                    }
                    named_bar_sync(2, CONSUMERS);
                    const bool whole = seg_from_start && last_chunk;
                    const int64_t hu0 = (int64_t)sh.pre[w.brow] + (int64_t)(bh - w.brow * H) * nch;  // first unit of this head
                    const int first_cta = (int)(((hu0 + 1) * geff - 1) / att_total);
                    const int last_cta = (int)(((hu0 + nch) * geff - 1) / att_total);
                    const int nsg = last_cta - first_cta + 1;
                    float *slots = ph.attn_partial + (int64_t)bh * ph.slots_per_head * (DS_KD + 2);
                    if (threadIdx.x < DS_KD) {
                        const int d = threadIdx.x;
                        float mw = -INFINITY;
#pragma unroll
                        for (int ww = 0; ww < DS_CONS_WARPS; ++ww) mw = fmaxf(mw, sh.a_m[ww]);
                        float L = 0.f, A = 0.f;
#pragma unroll
                        for (int ww = 0; ww < DS_CONS_WARPS; ++ww) {
                            const float cw = sh.a_m[ww] > -INFINITY ? expf(sh.a_m[ww] - mw) : 0.f;
                            L += sh.a_l[ww] * cw;
                            A += sh.a_acc[ww][d] * cw;
                        }
                        if (whole) {
                            outp[(int64_t)bh * DS_KD + d] = from_f<T>(A / L);
                        } else {
                            float *pp = slots + (int64_t)(cta - first_cta) * (DS_KD + 2);
                            __stcg(pp + 2 + d, A);
                            if (d == 0) {
                                __stcg(pp, mw);
                                __stcg(pp + 1, L);
                            }
                            __threadfence();
                        }
                    }
                    if (!whole) {
                        named_bar_sync(2, CONSUMERS);
                        if (threadIdx.x == 0) {
                            const int old = atomicAdd(ph.attn_tickets + bh, 1);
                            sh.a_last = old == nsg - 1;
                            if (sh.a_last) ph.attn_tickets[bh] = 0;
                            __threadfence();
                        }
                        named_bar_sync(2, CONSUMERS);
                        if (sh.a_last && threadIdx.x < DS_KD) {
                            const int d = threadIdx.x;
                            float mw = -INFINITY;
                            for (int sidx = 0; sidx < nsg; ++sidx) mw = fmaxf(mw, __ldcg(slots + (int64_t)sidx * (DS_KD + 2)));
                            float L = 0.f, A = 0.f;
                            for (int sidx = 0; sidx < nsg; ++sidx) {
                                const float *pp = slots + (int64_t)sidx * (DS_KD + 2);
                                const float ms = __ldcg(pp);
                                const float cw = ms > -INFINITY ? expf(ms - mw) : 0.f;
                                L += __ldcg(pp + 1) * cw;
                                A += __ldcg(pp + 2 + d) * cw;
                            }
                            outp[(int64_t)bh * DS_KD + d] = from_f<T>(A / L);
                        }
                    }
                    named_bar_sync(2, CONSUMERS);  // a_acc / a_m / a_last are reused by the next segment
                }
                att_next(w);
            }
            named_bar_sync(2, CONSUMERS);
            if (threadIdx.x == 0 && p + 1 < nph) {
                if (prog.trace) prog.trace[((size_t)cta * nph + p) * 2 + 1] = ds_now();
                grid_arrive(prog.grid_bar, (unsigned)nctas);  // (phase_done >= p: waited above)
            }
        }
        if (threadIdx.x == 0) ds_role_stats(prog.trace, nph, 3, waited, t_begin);
        if (xt == 0) ds_role_stats(prog.trace, nph, 4, waited, t_begin);
    }

}

// ======================================================================================================================
// host side: program construction (cached per argument set) + launch
// ======================================================================================================================
struct DsDeviceState {
    unsigned int *grid_bar = nullptr;
    int sms = 0;
};
static DsDeviceState &ds_device_state() {
    static DsDeviceState st[64];
    int dev = 0;
    cudaGetDevice(&dev);
    dev &= 63;
    if (!st[dev].grid_bar) {
        cudaMalloc(&st[dev].grid_bar, 256);
        cudaMemset(st[dev].grid_bar, 0, 256);
        cudaDeviceGetAttribute(&st[dev].sms, cudaDevAttrMultiProcessorCount, dev);
        cudaDeviceSynchronize();
    }
    return st[dev];
}

// split-K factor of a GEMM phase: units = ntiles x S are dealt to the persistent CTAs in WAVES (unit = cta + wave * nctas,
// unit -> (split = unit / ntiles, tile = unit % ntiles)), so the CTAs of a wave stream ADJACENT column tiles over the SAME k
// rows in lock-step -- the DRAM-page locality a row-major [K, N] weight needs (contiguous
// per-CTA k ranges scatter the concurrent reads over many DRAM pages).  S = the smallest factor whose wave fill is within 2 % of the best.
int ds_pick_split(int ntiles, int kchunks, int nctas) {
    const int smax = std::max(1, std::min(16, kchunks / 2));
    double eff[17] = {0};
    double best_eff = 0.0;
    for (int S = 1; S <= smax; ++S) {
        const int64_t units = (int64_t)ntiles * S;
        const int64_t waves = (units + nctas - 1) / nctas;
        const int per = (kchunks + S - 1) / S;  // time ~ waves x (longest unit); work ~ ntiles x kchunks
        eff[S] = (double)ntiles * kchunks / ((double)waves * per * nctas);
        best_eff = std::max(best_eff, eff[S]);
    }
    for (int S = 1; S <= smax; ++S)
        if (eff[S] >= best_eff - 0.02) return S;  // the smallest split within 2 % of the best: fewer partial tiles to park and sum
    return 1;
}
int ds_max_slots(int ntiles, int kchunks, int nctas) { return ds_pick_split(ntiles, kchunks, nctas); }

}  // namespace itb

using namespace itb;

static unsigned long long *g_ds_trace = nullptr;
// phase timeline (tools/ds_trace.py): device buffer of >= 132 * nphases * 2 u64, or NULL to switch it off
extern "C" void it_b200_decode_stack_trace(void *dev_buf) { g_ds_trace = (unsigned long long *)dev_buf; }

// A cached program: phases in device memory + the tickets it owns (self-cleaning, so zeroed once)
struct DsCacheEntry {
    std::vector<uint8_t> key;
    DsPhase *dev_phases = nullptr;
    int *tickets = nullptr;
    int nphases = 0;
};
static std::mutex g_ds_mu;
static std::vector<DsCacheEntry> g_ds_cache;

static int ds_launch(int dtype, const DsPhase *dev_phases, int nph, int rows, const void *position_id, int pos_flags,
                     const void *rope_pos, int rope_pos_dtype, cudaStream_t st) {
    DsDeviceState &ds = ds_device_state();
    ITB_CHECK(ds.grid_bar != nullptr && ds.sms > 0, "decode_stack: device state allocation failed");
    DsProgram prog{};
    prog.phases = dev_phases;
    prog.nphases = nph;
    prog.rows = rows;
    prog.position_id = position_id;
    prog.pos_flags = pos_flags;
    prog.rope_pos = rope_pos;
    prog.rope_pos_dtype = rope_pos_dtype;
    prog.grid_bar = ds.grid_bar;
    prog.trace = g_ds_trace;
    const int smem = DS_STAGES * DS_STAGE_BYTES + DS_ACC_BUFS * DS_ACC_BYTES + 1024;
    cudaError_t e;
    if (dtype == ITB_BF16) {
        e = cudaFuncSetAttribute(decode_stack_kernel<__nv_bfloat16>, cudaFuncAttributeMaxDynamicSharedMemorySize, smem);
        ITB_CHECK(e == cudaSuccess, "decode_stack: smem attribute: %s", cudaGetErrorString(e));
        e = launch_k(decode_stack_kernel<__nv_bfloat16>, dim3(ds.sms), dim3(DS_THREADS), smem, st, prog);
    } else {
        e = cudaFuncSetAttribute(decode_stack_kernel<__half>, cudaFuncAttributeMaxDynamicSharedMemorySize, smem);
        ITB_CHECK(e == cudaSuccess, "decode_stack: smem attribute: %s", cudaGetErrorString(e));
        e = launch_k(decode_stack_kernel<__half>, dim3(ds.sms), dim3(DS_THREADS), smem, st, prog);
    }
    ITB_CHECK(e == cudaSuccess, "decode_stack: launch failed: %s", cudaGetErrorString(e));
    ITB_LAUNCH_CHECK("decode_stack");
    return 0;
}

struct DsScratch {
    char *base;
    int64_t off = 0;
    void *take(int64_t bytes) {
        off = (off + 255) & ~255ll;
        void *p = base + off;
        off += bytes;
        return p;
    }
};

static bool ds_fill_gemm(DsPhase &ph, int rows, const DsGemmDesc &d, int nctas) {
    memset(&ph, 0, sizeof(ph));
    ph.kind = DS_GEMM;
    ph.ngroups = d.ngroups;
    ph.n_per_group = d.n_per_group;
    ph.K = d.K;
    ph.tiles_per_group = (d.n_per_group + 127) / 128;
    ph.ntiles = ph.tiles_per_group * d.ngroups;
    ph.kchunks = (d.K + 63) / 64;
    ph.xform = d.xform;
    ph.epi = d.epi;
    for (int g = 0; g < d.ngroups; ++g) {
        if (!make_tma_2d_b16(&ph.mapW[g], d.W[g], (uint64_t)d.K, (uint64_t)d.n_per_group, (uint64_t)d.n_per_group, 64, 64, 128)) return false;
        ph.out[g] = d.out[g];
    }
    if (!make_tma_2d_b16(&ph.mapX, d.X, (uint64_t)rows, (uint64_t)d.K, (uint64_t)d.K, DS_ROWS, 64, 128)) return false;
    if (d.xform == DS_XF_SILU_MUL && !make_tma_2d_b16(&ph.mapX2, d.X2, (uint64_t)rows, (uint64_t)d.K, (uint64_t)d.K, DS_ROWS, 64, 128))
        return false;
    ph.residual = d.residual;
    ph.norm_w = d.norm_w;
    ph.x_raw = d.X;
    ph.nsplit = ds_pick_split(ph.ntiles, ph.kchunks, nctas);
    ph.slots_per_tile = ph.nsplit;
    return true;
}

static int64_t ds_scratch_bytes(int max_tiles, int max_slots, int BH, int S_max) {
    const int64_t part = (int64_t)max_tiles * max_slots * DS_ROWS * 128 * 4;
    const int64_t attn = BH ? (int64_t)BH * (S_max / DS_CH + 2) * (DS_KD + 2) * 4 : 0;
    return 2 * (part + 256) + 2 * ((int64_t)max_tiles * DS_ROWS * 4 + 256) + attn + 1024;
}

extern "C" int64_t it_b200_decode_stack_workspace(int n_layers, int B, int d_model, int H, int S_max, int ffn) {
    (void)n_layers;
    // the split factors, hence the partial slots, depend on the grid: size for the one the launch uses (one CTA per SM of the
    // current device); kNumSMs only when no device answers
    const int sms = ds_device_state().sms;
    const int nctas = sms > 0 ? sms : kNumSMs;
    int max_tiles = 0, max_slots = 0;
    const int dl = H * DS_KD;
    const int shapes[4][3] = {{3, dl, d_model}, {1, d_model, dl}, {2, ffn, d_model}, {1, d_model, ffn}};  // groups, N, K
    for (auto &sh : shapes) {
        const int tiles = sh[0] * ((sh[1] + 127) / 128), kch = (sh[2] + 63) / 64;
        max_tiles = std::max(max_tiles, tiles);
        max_slots = std::max(max_slots, ds_max_slots(tiles, kch, nctas));
    }
    return ds_scratch_bytes(max_tiles, max_slots + 1, B * H, S_max);
}

// scratch: fp32 partial tiles (two regions, alternating by phase), per-tile sums of squares (two regions), attention partial
// slots -- all from the caller's workspace (no persistence needed); tickets from the cache entry (must stay zero between uses)
static int ds_assign_scratch(std::vector<DsPhase> &phs, void *workspace, int64_t workspace_bytes, int BH, int S_max, int **tickets_out) {
    int max_tiles = 1, max_slots = 1;
    for (auto &ph : phs)
        if (ph.kind == DS_GEMM) {
            max_tiles = std::max(max_tiles, ph.ntiles);
            max_slots = std::max(max_slots, ph.slots_per_tile);
        }
    ITB_CHECK(ds_scratch_bytes(max_tiles, max_slots, BH, S_max) <= workspace_bytes, "decode_stack: workspace %lld < %lld bytes",
              (long long)workspace_bytes, (long long)ds_scratch_bytes(max_tiles, max_slots, BH, S_max));
    DsScratch sc{(char *)workspace};
    const int64_t part_bytes = (int64_t)max_tiles * max_slots * DS_ROWS * 128 * 4;
    float *part[2] = {(float *)sc.take(part_bytes), (float *)sc.take(part_bytes)};
    float *ss[2] = {(float *)sc.take((int64_t)max_tiles * DS_ROWS * 4), (float *)sc.take((int64_t)max_tiles * DS_ROWS * 4)};
    const int slots_per_head = S_max / DS_CH + 2;
    float *attn_part = BH ? (float *)sc.take((int64_t)BH * slots_per_head * (DS_KD + 2) * 4) : nullptr;
    int *tickets = nullptr;
    const size_t nt = (size_t)max_tiles * 2 + (size_t)BH;
    cudaError_t ce = cudaMalloc(&tickets, nt * sizeof(int));
    ITB_CHECK(ce == cudaSuccess, "decode_stack: cudaMalloc(tickets): %s", cudaGetErrorString(ce));
    cudaMemset(tickets, 0, nt * sizeof(int));
    *tickets_out = tickets;
    int gi = 0, ssi = 0;
    const float *prev_ss = nullptr;
    int prev_ss_tiles = 0;
    const void *prev_res_out = nullptr;
    for (auto &ph : phs) {
        if (ph.kind == DS_GEMM) {
            ph.partial = part[gi & 1];
            ph.tickets = tickets + (gi & 1) * max_tiles;
            ++gi;
            if (ph.xform == DS_XF_RMSNORM && prev_ss && prev_res_out == ph.x_raw) {
                ph.ss_in = prev_ss;  // (otherwise nullptr: the kernel reduces x_raw itself)
                ph.ss_in_tiles = prev_ss_tiles;
            }
            if (ph.epi == DS_EPI_RESIDUAL) {
                ph.ss_out = ss[ssi & 1];
                prev_ss = ph.ss_out;
                prev_ss_tiles = ph.ntiles;
                prev_res_out = ph.out[0];
                ++ssi;
            }
        } else {
            ph.attn_partial = attn_part;
            ph.attn_tickets = tickets + 2 * max_tiles;
            ph.slots_per_head = slots_per_head;
        }
    }
    return 0;
}

// look the program up by the raw argument bytes; build (tensor maps, scratch, upload) only on a miss
template <typename Build>
static int ds_run_cached(int dtype, int rows, const std::vector<uint8_t> &key_in, Build build, void *workspace,
                         int64_t workspace_bytes, int BH, int S_max, const void *position_id, int pos_flags,
                         const void *rope_pos, int rope_pos_dtype, cudaStream_t st) {
    std::lock_guard<std::mutex> lock(g_ds_mu);
    std::vector<uint8_t> k = key_in;
    int dev = 0;
    cudaGetDevice(&dev);
    k.push_back((uint8_t)dev);
    DsCacheEntry *hit = nullptr;
    for (auto &e : g_ds_cache)
        if (e.key == k) hit = &e;
    if (!hit) {
        // first use (never during a CUDA-graph capture: the runtime runs every graph once eagerly before capturing)
        cudaStreamCaptureStatus cs = cudaStreamCaptureStatusNone;
        cudaStreamIsCapturing(st, &cs);
        ITB_CHECK(cs == cudaStreamCaptureStatusNone, "decode_stack: program not built before capture (run the graph once eagerly)");
        std::vector<DsPhase> phs;
        if (int rc = build(phs)) return rc;
        DsCacheEntry e;
        e.key = k;
        e.nphases = (int)phs.size();
        if (int rc = ds_assign_scratch(phs, workspace, workspace_bytes, BH, S_max, &e.tickets)) return rc;
        cudaError_t ce = cudaMalloc(&e.dev_phases, sizeof(DsPhase) * phs.size());
        ITB_CHECK(ce == cudaSuccess, "decode_stack: cudaMalloc(program): %s", cudaGetErrorString(ce));
        ce = cudaMemcpy(e.dev_phases, phs.data(), sizeof(DsPhase) * phs.size(), cudaMemcpyHostToDevice);
        ITB_CHECK(ce == cudaSuccess, "decode_stack: upload(program): %s", cudaGetErrorString(ce));
        // An evicted entry's device program may still be baked into a CUDA graph captured earlier (graph replay launches the kernel
        // with the pointer it was captured with), so old programs are DROPPED from the lookup table but never freed: a few KB per
        // (shape, pointer set) ever seen, bounded by what the process builds.
        if (g_ds_cache.size() > 256) g_ds_cache.erase(g_ds_cache.begin());
        g_ds_cache.push_back(e);
        hit = &g_ds_cache.back();
    }
    return ds_launch(dtype, hit->dev_phases, hit->nphases, rows, position_id, pos_flags, rope_pos, rope_pos_dtype, st);
}

static int ds_sms() { return ds_device_state().sms; }

// stall diagnostics (tools/ds_debug.py): allocates host-mapped memory the kernel's wait sites report into; returns the HOST
// pointer (132 CTAs x 16 sites x 4 words), which stays readable after a trap killed the context
extern "C" void *it_b200_decode_stack_debug(void) {
    static unsigned *host = nullptr;
    if (!host) {
        unsigned *dev = nullptr;
        if (cudaHostAlloc((void **)&host, 256 * 16 * 4 * sizeof(unsigned), cudaHostAllocMapped) != cudaSuccess) return nullptr;
        memset(host, 0, 256 * 16 * 4 * sizeof(unsigned));
        cudaHostGetDevicePointer((void **)&dev, host, 0);
        cudaMemcpyToSymbol(g_ds_dbg, &dev, sizeof(dev));
    }
    return host;
}

// ---- test / head entry point: a chain of GEMM phases over <= 16 rows ------------------------------------------------------
extern "C" int it_b200_decode_gemm_chain(int dtype, int rows, int n_phases, const int *ngroups, const void *const *W,
                                         void *const *out, const int *n_per_group, const int *K, const int *xform,
                                         const int *epi, const void *const *X, const void *const *X2,
                                         const void *const *residual, const void *const *norm_w, void *workspace,
                                         int64_t workspace_bytes, void *stream) {
    ITB_CHECK(dtype == ITB_BF16 || dtype == ITB_F16, "decode_gemm_chain: dtype %d must be f16 / bf16", dtype);
    ITB_CHECK(rows >= 1 && rows <= DS_ROWS, "decode_gemm_chain: %d rows > %d", rows, DS_ROWS);
    ITB_CHECK(n_phases >= 1 && n_phases <= 8, "decode_gemm_chain: bad phase count %d", n_phases);
    auto st = (cudaStream_t)stream;
    std::vector<DsGemmDesc> descs(n_phases);
    std::vector<uint8_t> key;
    auto push = [&](const void *p, size_t n) { key.insert(key.end(), (const uint8_t *)p, (const uint8_t *)p + n); };
    int wi = 0;
    for (int p = 0; p < n_phases; ++p) {
        DsGemmDesc &d = descs[p];
        memset(&d, 0, sizeof(d));
        d.ngroups = ngroups[p];
        ITB_CHECK(d.ngroups >= 1 && d.ngroups <= DS_MAX_GROUPS, "decode_gemm_chain: bad group count");
        for (int g = 0; g < d.ngroups; ++g, ++wi) {
            d.W[g] = W[wi];
            d.out[g] = out[wi];
        }
        d.n_per_group = n_per_group[p];
        d.K = K[p];
        d.xform = xform[p];
        d.epi = epi[p];
        d.X = X[p];
        d.X2 = X2 ? X2[p] : nullptr;
        d.residual = residual ? residual[p] : nullptr;
        d.norm_w = norm_w ? norm_w[p] : nullptr;
        ITB_CHECK(d.n_per_group % 8 == 0 && d.K % 8 == 0 && d.n_per_group >= 8 && d.K >= 8, "decode_gemm_chain: N and K must be multiples of 8");
        ITB_CHECK(d.epi != DS_EPI_RESIDUAL || (d.residual && d.ngroups == 1), "decode_gemm_chain: residual epilogue needs one group + a residual");
        ITB_CHECK(d.xform != DS_XF_RMSNORM || d.norm_w, "decode_gemm_chain: RMSNorm transform needs the weight");
        ITB_CHECK(d.xform != DS_XF_SILU_MUL || d.X2, "decode_gemm_chain: Silu*Mul transform needs both operands");
        ITB_CHECK(aligned16(d.X) && (!d.X2 || aligned16(d.X2)), "decode_gemm_chain: operands must be 16-byte aligned");
        push(&d, sizeof(d));
    }
    push(&workspace, sizeof(workspace));
    int misc[2] = {rows, dtype};
    push(misc, sizeof(misc));
    auto build = [&](std::vector<DsPhase> &phs) -> int {
        const int nctas = ds_sms();
        phs.resize(n_phases);
        for (int p = 0; p < n_phases; ++p)
            ITB_CHECK(ds_fill_gemm(phs[p], rows, descs[p], nctas), "decode_gemm_chain: cuTensorMapEncodeTiled failed");
        return 0;
    };
    return ds_run_cached(dtype, rows, key, build, workspace, workspace_bytes, 0, 0, nullptr, ITB_I64, nullptr, 0, st);
}

// ---- the decoder stack ----------------------------------------------------------------------------------------------------
extern "C" int it_b200_llama_decode_stack(int dtype, int n_layers, const itb_llama_layer *layers, const void *x_in,
                                          const void *position_id, int pos_flags, const void *rope_pos, int rope_pos_dtype,
                                          int B, int d_model, int H, int S_max, int ffn, void *workspace,
                                          int64_t workspace_bytes, void *stream) {
    ITB_CHECK(dtype == ITB_BF16 || dtype == ITB_F16, "llama_decode_stack: dtype %d must be f16 / bf16", dtype);
    ITB_CHECK(B >= 1 && B <= DS_ROWS && B <= DS_MAX_B, "llama_decode_stack: batch %d > %d rows", B, DS_ROWS);
    ITB_CHECK(n_layers >= 1 && n_layers <= 128, "llama_decode_stack: bad layer count %d", n_layers);
    ITB_CHECK(d_model % 8 == 0 && ffn % 8 == 0 && H >= 1, "llama_decode_stack: d_model / ffn must be multiples of 8");
    const int pos_dtype = pos_flags & 0xff;
    ITB_CHECK(pos_dtype == ITB_I32 || pos_dtype == ITB_U32 || pos_dtype == ITB_I64, "llama_decode_stack: position dtype %d", pos_dtype);
    ITB_CHECK(!rope_pos || rope_pos_dtype == ITB_I32 || rope_pos_dtype == ITB_U32 || rope_pos_dtype == ITB_I64,
              "llama_decode_stack: rope position dtype %d", rope_pos_dtype);
    const int dl = H * DS_KD;  // local attention width (tensor parallel: H = local heads)
    auto st = (cudaStream_t)stream;
    std::vector<uint8_t> key;
    auto push = [&](const void *p, size_t n) { key.insert(key.end(), (const uint8_t *)p, (const uint8_t *)p + n); };
    push(layers, sizeof(itb_llama_layer) * (size_t)n_layers);
    push(&x_in, sizeof(x_in));
    push(&workspace, sizeof(workspace));
    int misc[8] = {dtype, B, d_model, H, S_max, ffn, pos_flags, rope_pos_dtype};
    push(misc, sizeof(misc));
    push(&position_id, sizeof(position_id));
    push(&rope_pos, sizeof(rope_pos));
    auto build = [&](std::vector<DsPhase> &phs) -> int {
        const int nctas = ds_sms();
        phs.reserve((size_t)n_layers * 5);
        const void *x = x_in;
        DsPhase ph;
        for (int li = 0; li < n_layers; ++li) {
            const itb_llama_layer &L = layers[li];
            DsGemmDesc d;
            // (1) RMSNorm -> q / k / v
            memset(&d, 0, sizeof(d));
            d.ngroups = 3;
            d.W[0] = L.wq; d.W[1] = L.wk; d.W[2] = L.wv;
            d.out[0] = L.q; d.out[1] = L.k; d.out[2] = L.v;
            d.n_per_group = dl; d.K = d_model; d.xform = DS_XF_RMSNORM; d.epi = DS_EPI_STORE;
            d.X = x; d.norm_w = L.ln1_w;
            ITB_CHECK(ds_fill_gemm(ph, B, d, nctas), "llama_decode_stack: tensor map (qkv) failed");
            phs.push_back(ph);
            // (2) RoPE + attention
            memset(&ph, 0, sizeof(ph));
            ph.kind = DS_ATTN;
            ph.kcache = L.k_cache; ph.vcache = L.v_cache;
            ph.q = L.q; ph.k = L.k; ph.v = L.v;
            ph.attn_out = L.attn_out;
            ph.H = H; ph.S_max = S_max;
            phs.push_back(ph);
            // (3) o-proj + residual
            memset(&d, 0, sizeof(d));
            d.ngroups = 1;
            d.W[0] = L.wo; d.out[0] = L.x_mid;
            d.n_per_group = d_model; d.K = dl; d.xform = DS_XF_NONE; d.epi = DS_EPI_RESIDUAL;
            d.X = L.attn_out; d.residual = x;
            ITB_CHECK(ds_fill_gemm(ph, B, d, nctas), "llama_decode_stack: tensor map (o) failed");
            phs.push_back(ph);
            // (4) RMSNorm -> gate / up
            memset(&d, 0, sizeof(d));
            d.ngroups = 2;
            d.W[0] = L.wg; d.W[1] = L.wu;
            d.out[0] = L.gate; d.out[1] = L.up;
            d.n_per_group = ffn; d.K = d_model; d.xform = DS_XF_RMSNORM; d.epi = DS_EPI_STORE;
            d.X = L.x_mid; d.norm_w = L.ln2_w;
            ITB_CHECK(ds_fill_gemm(ph, B, d, nctas), "llama_decode_stack: tensor map (gate/up) failed");
            phs.push_back(ph);
            // (5) Silu(gate) * up -> down + residual
            memset(&d, 0, sizeof(d));
            d.ngroups = 1;
            d.W[0] = L.wd; d.out[0] = L.x_out;
            d.n_per_group = d_model; d.K = ffn; d.xform = DS_XF_SILU_MUL; d.epi = DS_EPI_RESIDUAL;
            d.X = L.gate; d.X2 = L.up; d.residual = L.x_mid;
            ITB_CHECK(ds_fill_gemm(ph, B, d, nctas), "llama_decode_stack: tensor map (down) failed");
            phs.push_back(ph);
            x = L.x_out;
        }
        return 0;
    };
    return ds_run_cached(dtype, B, key, build, workspace, workspace_bytes, B * H, S_max, position_id, pos_flags, rope_pos,
                         rope_pos_dtype, st);
}
