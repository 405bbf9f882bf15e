// allreduce.cu -- one-shot all-reduce over NVLink peer memory, fused with the residual Add and the RMSNorm that
// follow it in a tensor-parallel decoder layer (examples/distributed/parallel_opt.py inserts AllReduceSum after
// every row-split MatMul; the graph then does Add(residual) and RMSNorm).
//
// Replaces, for the decode message size (tokens x d_model, 128 KiB at B = 16): ncclAllReduce on the runtime stream
// (reference src/kernels/cuda/all_reduce.cc:8-63) + the Add kernel + the RMSNorm kernel = 3 launches and a
// latency-bound collective, with ONE kernel:
//   every rank owns a symmetric comm workspace (cudaMalloc'ed, exported with cudaIpc, opened by all peers):
//       epoch[row] | (flags, unused by the LL protocol) | data[2][rank][row][2 * row_bytes]
//   CTA `row` of rank r:  (1) PUSHES its partial row into data[e&1][r][row] of every peer as "LL" packets: every 8 bytes
//   on the wire are {4 bytes of payload, 4-byte tag = e+1}, so the DATA IS ITS OWN FLAG -- no fence.sys, no separate
//   flag store, no second NVLink round trip (the 8-byte store atomicity NCCL's LL protocol relies on);  (2) polls the
//   world's packets in its LOCAL buffer with volatile 16-byte loads until every tag reads e+1;  (3) sums the world
//   partials in rank order in fp32 (identical on every rank), rounds to the storage dtype, adds the residual, stores;
//   optionally RMS-normalises the new residual row in the same pass and stores that too;  (4) bumps epoch[row].
// Double buffering by epoch parity makes a trailing barrier unnecessary (a rank can only start epoch e+2 after every
// peer finished reading epoch e's buffer).  No host involvement: CUDA-graph-capturable, PDL-chained.
// A peer that never shows up (crashed rank, start-up skew beyond the poll budget) does NOT trap the context: the poll
// gives up after ~2^26 probes, raises *timeout_flag (host-mapped memory the runtime checks after every synchronise) and
// lets the step finish with garbage, so every rank gets a recoverable infini::Exception instead of a sticky fatal error.
// Ordering contract: epoch[row] is handed from one all-reduce launch to the next through TRANSITIVE completion -- every
// kernel of this library executes griddepcontrol.wait on every path before it exits (tests/test_host_cpu.py checks the
// sources), so "my predecessor finished" implies "everything before it finished".
#include <algorithm>
#include <cstdlib>
#include <string>

#include "common.cuh"

namespace itb {

constexpr int AR_MAX_WORLD = 8;
constexpr int AR_MAX_ROWS = 64;
constexpr int AR_MAX_ROW_BYTES = 16384;

struct ArPeers {
    void *ws[AR_MAX_WORLD];  // comm workspace of every rank as mapped in THIS process (ws[rank] = local)
};

__host__ __device__ inline size_t ar_epoch_off() { return 0; }
__host__ __device__ inline size_t ar_flags_off() { return 1024; }
__host__ __device__ inline size_t ar_data_off() { return 1024 + (size_t)2 * AR_MAX_ROWS * AR_MAX_WORLD * sizeof(int); }
constexpr int AR_SLOT_BYTES = 2 * AR_MAX_ROW_BYTES;  // LL packets double the row
__host__ __device__ inline size_t ar_workspace_bytes() {
    return ar_data_off() + (size_t)2 * AR_MAX_WORLD * AR_MAX_ROWS * AR_SLOT_BYTES;
}

__device__ __forceinline__ void st_release_sys(int *p, int v) {
    asm volatile("st.release.sys.global.s32 [%0], %1;" ::"l"(p), "r"(v) : "memory");
}
__device__ __forceinline__ int ld_acquire_sys(const int *p) {
    int v;
    asm volatile("ld.acquire.sys.global.s32 %0, [%1];" : "=r"(v) : "l"(p) : "memory");
    return v;
}

__device__ __forceinline__ uint4 ld_volatile_v4(const void *p) {
    uint4 v;
    asm volatile("ld.volatile.global.v4.u32 {%0,%1,%2,%3}, [%4];" : "=r"(v.x), "=r"(v.y), "=r"(v.z), "=r"(v.w) : "l"(p) : "memory");
    return v;
}
__device__ __forceinline__ void st_volatile_v4(void *p, uint4 v) {
    asm volatile("st.volatile.global.v4.u32 [%0], {%1,%2,%3,%4};" ::"l"(p), "r"(v.x), "r"(v.y), "r"(v.z), "r"(v.w) : "memory");
}

// LL protocol: the row travels as {payload word, tag} pairs; a reader that sees both tags of a 16-byte packet has the data
template <typename T>
__global__ void __launch_bounds__(512) allreduce_ll_kernel(ArPeers peers, int world, int rank, const T *__restrict__ in,
                                                           const T *__restrict__ residual, const T *__restrict__ norm_w,
                                                           T *__restrict__ out, T *__restrict__ out_norm, int hidden,
                                                           int *timeout_flag) {
    constexpr int V = Vec16<T>::N;
    __shared__ float red[32];
    pdl_trigger();
    const int row = blockIdx.x;
    char *local = (char *)peers.ws[rank];
    int *epoch_p = (int *)(local + ar_epoch_off()) + row;
    const int nv = hidden / V;
    pdl_wait();  // `in` comes from the preceding row-split MatMul; epoch[row] from the previous all-reduce kernel
    // only CTA `row` of this stream's kernels ever writes epoch[row]; unsigned, so that the count wraps past INT_MAX (2^31
    // all-reduces of one row) without signed overflow: tag and parity follow the bits through the wrap
    const uint32_t e = (uint32_t)*epoch_p;
    const int b = e & 1;
    const uint32_t tag = e + 1u;
    bool gave_up = false;
    const size_t slot = (((size_t)b * AR_MAX_WORLD + rank) * AR_MAX_ROWS + row) * AR_SLOT_BYTES;

    // (1) push: vector i of my partial row -> packets 2i, 2i+1 of my slot on every rank (own copy included)
    for (int i = threadIdx.x; i < nv; i += blockDim.x) {
        const uint4 w = *reinterpret_cast<const uint4 *>(in + (size_t)row * hidden + i * V);
        const uint4 p0 = make_uint4(w.x, tag, w.y, tag), p1 = make_uint4(w.z, tag, w.w, tag);
        for (int p = 0; p < world; ++p) {
            char *dst = (char *)peers.ws[p] + ar_data_off() + slot + (size_t)i * 32;
            st_volatile_v4(dst, p0);
            st_volatile_v4(dst + 16, p1);
        }
    }
    // (2)+(3) poll the world's packets in local memory, reduce in rank order, residual add, optional RMSNorm
    float ss = 0.f;
    for (int i = threadIdx.x; i < nv; i += blockDim.x) {
        float acc[V];
#pragma unroll
        for (int j = 0; j < V; ++j) acc[j] = 0.f;
        const char *src0 = local + ar_data_off() + (((size_t)b * AR_MAX_WORLD) * AR_MAX_ROWS + row) * AR_SLOT_BYTES + (size_t)i * 32;
        constexpr size_t kRankStride = (size_t)AR_MAX_ROWS * AR_SLOT_BYTES;
        uint4 pa[AR_MAX_WORLD], pc[AR_MAX_WORLD];
#pragma unroll
        for (int p = 0; p < AR_MAX_WORLD; ++p)  // every rank's packets requested before the first tag is examined
            if (p < world) {
                pa[p] = ld_volatile_v4(src0 + p * kRankStride);
                pc[p] = ld_volatile_v4(src0 + p * kRankStride + 16);
            }
#pragma unroll
        for (int p = 0; p < AR_MAX_WORLD; ++p)
            if (p < world) {
                unsigned spins = 0;
                while (!gave_up && (pa[p].y != tag || pa[p].w != tag || pc[p].y != tag || pc[p].w != tag)) {
                    if (++spins > (1u << 26)) {  // a dead peer must neither hang the box nor kill the context
                        gave_up = true;
                        if (timeout_flag) *(volatile int *)timeout_flag = 1 + rank * 16 + p;
                        else __trap();
                        break;
                    }
                    pa[p] = ld_volatile_v4(src0 + p * kRankStride);
                    pc[p] = ld_volatile_v4(src0 + p * kRankStride + 16);
                }
                Vec16<T> v;
                *reinterpret_cast<uint4 *>(v.v) = make_uint4(pa[p].x, pa[p].z, pc[p].x, pc[p].z);
#pragma unroll
                for (int j = 0; j < V; ++j) acc[j] += to_f(v.v[j]);
            }
        Vec16<T> r, o;
        if (residual) r = ld16(residual + (size_t)row * hidden + i * V);
#pragma unroll
        for (int j = 0; j < V; ++j) {
            float x = round_t<T>(acc[j]);                          // the AllReduce output, as stored by the separate op
            if (residual) x = round_t<T>(to_f(r.v[j]) + x);        // Add(residual, allreduce)
            o.v[j] = from_f<T>(x);
            ss += x * x;
        }
        st16(out + (size_t)row * hidden + i * V, o);
    }
    if (norm_w) {
        const float rinv = rsqrtf(block_sum(ss, red) / (float)hidden + 0.00001f);
        for (int i = threadIdx.x; i < nv; i += blockDim.x) {
            const Vec16<T> x = ld16(out + (size_t)row * hidden + i * V), w = ld16(norm_w + i * V);
            Vec16<T> o;
#pragma unroll
            for (int j = 0; j < V; ++j) o.v[j] = from_f<T>(round_t<T>(to_f(x.v[j]) * rinv) * to_f(w.v[j]));
            st16(out_norm + (size_t)row * hidden + i * V, o);
        }
    }
    __syncthreads();
    if (threadIdx.x == 0) *epoch_p = (int)(e + 1u);
}

}  // namespace itb

using namespace itb;

extern "C" int64_t it_b200_allreduce_workspace_bytes(void) { return (int64_t)ar_workspace_bytes(); }

extern "C" int it_b200_allreduce_fused(int dtype, const void *in, const void *residual, const void *norm_w, void *out,
                                       void *out_norm, int tokens, int hidden, void *const *peer_ws, int world,
                                       int rank, int *timeout_flag, void *stream) {
    ITB_CHECK(world >= 1 && world <= AR_MAX_WORLD && rank >= 0 && rank < world, "allreduce_fused: bad world/rank %d/%d",
              world, rank);
    ITB_CHECK(tokens >= 0 && tokens <= AR_MAX_ROWS, "allreduce_fused: %d rows > %d", tokens, AR_MAX_ROWS);
    ITB_CHECK(hidden * dtype_size(dtype) <= AR_MAX_ROW_BYTES && (hidden * dtype_size(dtype)) % 16 == 0,
              "allreduce_fused: row of %d elements unsupported", hidden);
    ITB_CHECK(aligned16(in) && aligned16(out) && (!residual || aligned16(residual)) && (!norm_w || aligned16(norm_w)) &&
                  (!out_norm || aligned16(out_norm)),
              "allreduce_fused: tensors must be 16-byte aligned");
    ITB_CHECK((norm_w == nullptr) == (out_norm == nullptr), "allreduce_fused: norm weight and norm output go together");
    if (tokens == 0) return 0;
    ArPeers peers{};
    for (int p = 0; p < world; ++p) {
        ITB_CHECK(peer_ws[p] != nullptr, "allreduce_fused: peer workspace %d not mapped", p);
        peers.ws[p] = peer_ws[p];
    }
    ITB_DISPATCH_FLOAT(dtype, "allreduce_fused", {
        int threads = std::min(512, std::max(32, ((hidden / Vec16<T>::N + 31) / 32) * 32));
        return launch("allreduce_fused", allreduce_ll_kernel<T>, {dim3(tokens), dim3(threads), 0, (cudaStream_t)stream}, peers,
                      world, rank, (const T *)in, (const T *)residual, (const T *)norm_w, (T *)out, (T *)out_norm, hidden,
                      timeout_flag);
    });
    return 0;
}
