// gemm_simt.cu -- shape-generic batched GEMM on the CUDA cores (fp32 FFMA, fp32 accumulate).
//
// This is the exact-fp32 path of MatMul (the reference runs fp32 GEMMs with TF32 disabled,
// examples/distributed/cuda/cuda_launch.py:123-124, so tensor-core TF32 is not a legal substitute)
// and the catch-all for shapes / alignments the tensor-core kernels (gemm_skinny.cu,
// gemm_tc.cu) do not take.  64x64x16 tiles, 256 threads, 4x4 register micro-tile, any
// transA/transB, stride-0 batch broadcast, fused bias (+ activation) epilogue.
#include "common.cuh"
#include "gemm.cuh"

namespace itb {

template <typename T>
__global__ void __launch_bounds__(256) gemm_simt_kernel(GemmArgs g) {
    pdl_trigger();
    pdl_wait();
    constexpr int BM = 64, BN = 64, BK = 16;
    __shared__ float As[BK][BM + 4];
    __shared__ float Bs[BK][BN + 4];
    const int64_t batch = blockIdx.z;
    const T *A = (const T *)g.A + batch * g.stride_a;
    const T *B = (const T *)g.B + batch * g.stride_b;
    T *C = (T *)g.C + batch * (int64_t)g.m * g.n;
    const int m0 = blockIdx.y * BM, n0 = blockIdx.x * BN;
    const int tx = threadIdx.x & 15, ty = threadIdx.x >> 4;
    float acc[4][4] = {};
    for (int k0 = 0; k0 < g.k; k0 += BK) {
        // A tile -> As[k][m]
        for (int i = threadIdx.x; i < BM * BK; i += 256) {
            int mm, kk;
            if (g.trans_a) { mm = i % BM; kk = i / BM; } else { kk = i % BK; mm = i / BK; }
            int gm = m0 + mm, gk = k0 + kk;
            float v = 0.f;
            if (gm < g.m && gk < g.k)
                v = to_f(g.trans_a ? A[(int64_t)gk * g.m + gm] : A[(int64_t)gm * g.k + gk]);
            As[kk][mm] = v;
        }
        for (int i = threadIdx.x; i < BN * BK; i += 256) {
            int nn, kk;
            if (g.trans_b) { kk = i % BK; nn = i / BK; } else { nn = i % BN; kk = i / BN; }
            int gn = n0 + nn, gk = k0 + kk;
            float v = 0.f;
            if (gn < g.n && gk < g.k)
                v = to_f(g.trans_b ? B[(int64_t)gn * g.k + gk] : B[(int64_t)gk * g.n + gn]);
            Bs[kk][nn] = v;
        }
        __syncthreads();
#pragma unroll
        for (int kk = 0; kk < BK; ++kk) {
            float a[4], b[4];
#pragma unroll
            for (int i = 0; i < 4; ++i) a[i] = As[kk][ty * 4 + i];
#pragma unroll
            for (int j = 0; j < 4; ++j) b[j] = Bs[kk][tx * 4 + j];
#pragma unroll
            for (int i = 0; i < 4; ++i)
#pragma unroll
                for (int j = 0; j < 4; ++j) acc[i][j] = fmaf(a[i], b[j], acc[i][j]);
        }
        __syncthreads();
    }
#pragma unroll
    for (int i = 0; i < 4; ++i) {
        int gm = m0 + ty * 4 + i;
        if (gm >= g.m) continue;
#pragma unroll
        for (int j = 0; j < 4; ++j) {
            int gn = n0 + tx * 4 + j;
            if (gn >= g.n) continue;
            float v = acc[i][j];
            if (g.bias) {
                if (g.act & ITB_ACT_ROUND_BEFORE_BIAS) v = round_t<T>(v);
                v += to_f(((const T *)g.bias)[batch * g.bias_sb + gm * g.bias_sm + gn * g.bias_sn]);
            }
            C[(int64_t)gm * g.n + gn] = from_f<T>(gemm_act(g.act, v));
        }
    }
}

int launch_gemm_simt(int dtype, const GemmArgs &g, cudaStream_t st) {
    dim3 grid((g.n + 63) / 64, (g.m + 63) / 64, (unsigned)g.batch);
    ITB_CHECK(grid.y < 65536 && grid.z < 65536, "matmul(simt): grid too large (m=%d, batch=%lld)", g.m,
              (long long)g.batch);
    ITB_DISPATCH_FLOAT(dtype, "matmul(simt)", { return launch("matmul(simt)", gemm_simt_kernel<T>, {grid, dim3(256), 0, st}, g); });
    return 0;
}

}  // namespace itb
