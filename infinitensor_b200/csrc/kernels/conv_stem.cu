// conv_stem.cu -- the first convolution of an image network: few input channels (C <= 4, e.g. RGB), NCHW input, NHWC output.
//
// C = 3 is no shape for the TMA im2col path (a pixel's channel vector is 6 bytes), and the im2col + GEMM path writes and re-reads
// a 187 MB im2col matrix for it (ResNet-50, batch 64).  Here each CTA stages the input patch of a
// 16 x 16 block of output pixels in shared memory -- channel-interleaved and padded to 4 channels, 8 bytes per pixel -- and the
// warps build their mma.sync A fragments straight from that patch: with k = (r, s padded to a multiple of 4, c padded to 4), one
// k16 step is four consecutive filter taps of one filter row, a fragment register is one 32-bit shared-memory load, and the 32
// lanes of a load read 128 contiguous bytes (8 output columns x 4 taps... stride 2: 16 B apart, see a_off below).
//   grid: persistent, a few CTAs per SM, each walking (image, block row, block column) tiles; filters [F <= 64][k] stay in smem
//   warp w of 8: output rows 2w, 2w+1 of the block = two m16 tiles x 8 n8 tiles, fp32 accumulators in registers
//   epilogue: BatchNorm (folded to one FMA) + ReLU, fp16/bf16 through a per-warp padded staging tile, 16-byte NHWC stores
// Replaces cudnnConvolutionForward (+ BatchNorm + Relu kernels) for the stem (reference src/kernels/cuda/conv.cc:143-168).
#include <algorithm>

#include "conv_shapes.h"
#include "gemm.cuh"

namespace itb {

constexpr int ST_TH = 16, ST_TW = 16;          // output block
constexpr int ST_WARPS = 8, ST_THREADS = 256;
constexpr int ST_FMAX = 64;
constexpr int ST_STG_PITCH = 144;              // staging row: 64 filters x 2 B + 16 B pad (conflict-free 4-byte writes)

struct StemParams {
    const void *x, *w;
    void *y;
    const float *bn_mean, *bn_var, *bn_scale, *bn_bias;
    float bn_eps;
    int relu;
    int N, C, H, W, F, R, S, OH, OW, ph, pw, sh, sw;
    int tiles_h, tiles_w, tiles;
    int PH, PW;        // patch rows / columns (pixels)
    int S4;            // taps per filter row padded to a multiple of 4
    int ksteps;        // R * S4 / 4
    int wpitch;        // halves per filter row in smem (K + 8: conflict-free B fragment loads)
};

template <typename T>
__global__ void __launch_bounds__(ST_THREADS, 2) conv_stem_kernel(StemParams p) {
    extern __shared__ __align__(16) uint8_t smem[];
    const int K = p.ksteps * 16;
    T *w_sm = reinterpret_cast<T *>(smem);                                       // [64][wpitch]
    float2 *bn_sm = reinterpret_cast<float2 *>(w_sm + ST_FMAX * p.wpitch);     // [64] {a, b}
    uint8_t *stg_sm = reinterpret_cast<uint8_t *>(bn_sm + ST_FMAX);            // [8 warps][32 pixels][144 B]
    uint2 *patch = reinterpret_cast<uint2 *>(stg_sm + ST_WARPS * 32 * ST_STG_PITCH);  // [PH][PW] x 4 channels

    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31, g = lane >> 2, t = lane & 3;
    pdl_trigger();
    // ---- filters -> smem [f][k], k = (r * S4 + s) * 4 + c, zero where s >= S, c >= C, f >= F (constants: read before the wait)
    {
        const T *W = (const T *)p.w;
        const int RS = p.R * p.S;
        for (int i = threadIdx.x; i < ST_FMAX * (K / 4); i += ST_THREADS) {
            const int f = i / (K / 4), tap = i - f * (K / 4);
            const int r = tap / p.S4, s = tap - r * p.S4;
            T v[4];
#pragma unroll
            for (int c = 0; c < 4; ++c)
                v[c] = (f < p.F && s < p.S && c < p.C) ? W[(f * p.C + c) * RS + r * p.S + s] : from_f<T>(0.f);
            *reinterpret_cast<uint2 *>(w_sm + f * p.wpitch + tap * 4) = *reinterpret_cast<const uint2 *>(v);
        }
        for (int f = threadIdx.x; f < ST_FMAX; f += ST_THREADS) {
            float2 ab = make_float2(f < p.F ? 1.f : 0.f, 0.f);
            if (f < p.F && p.bn_scale) {
                ab.x = p.bn_scale[f] * bn_rs(p.bn_var[f], p.bn_eps);
                ab.y = __fmaf_rn(-p.bn_mean[f], ab.x, p.bn_bias[f]);
            }
            bn_sm[f] = ab;
        }
    }
    pdl_wait();
    const T *X = (const T *)p.x;
    T *Y = (T *)p.y;
    uint8_t *my_stg = stg_sm + warp * 32 * ST_STG_PITCH;
    const int patch_px = p.PH * p.PW;

    for (int tile = blockIdx.x; tile < p.tiles; tile += gridDim.x) {
        const int tw = tile % p.tiles_w;
        const int th = (tile / p.tiles_w) % p.tiles_h;
        const int n = tile / (p.tiles_w * p.tiles_h);
        const int oh0 = th * ST_TH, ow0 = tw * ST_TW;
        const int ih0 = oh0 * p.sh - p.ph, iw0 = ow0 * p.sw - p.pw;
        __syncthreads();  // the previous tile's fragments have been read (and, first time, the filters are in place)
        // ---- input patch: [PH][PW] pixels x {c0, c1, c2, c3} (zero outside the image / beyond C); reads run along w per channel
        for (int i = threadIdx.x; i < patch_px; i += ST_THREADS) {
            const int py = i / p.PW, px = i - py * p.PW;
            const int ih = ih0 + py, iw = iw0 + px;
            T v[4];
            const bool in = ih >= 0 && ih < p.H && iw >= 0 && iw < p.W;
#pragma unroll
            for (int c = 0; c < 4; ++c)
                v[c] = (in && c < p.C) ? X[(((int64_t)n * p.C + c) * p.H + ih) * p.W + iw] : from_f<T>(0.f);
            patch[i] = *reinterpret_cast<const uint2 *>(v);
        }
        __syncthreads();

        // ---- main loop: warp = output rows 2w, 2w+1 of the block; m16 tile rows g / g+8 = output columns g / g+8
        float acc[2][8][4];
#pragma unroll
        for (int mt = 0; mt < 2; ++mt)
#pragma unroll
            for (int nt = 0; nt < 8; ++nt)
#pragma unroll
                for (int e = 0; e < 4; ++e) acc[mt][nt][e] = 0.f;
        // word (4-byte) offsets into the patch: pixel (py, px) channel pair cp -> (py * PW + px) * 2 + cp
        const int a_lane = (g * p.sw + (t >> 1)) * 2 + (t & 1);  // + 8 columns: + 8 * sw * 2; upper k half: + 2 taps = + 4
        const uint32_t *patch_w = reinterpret_cast<const uint32_t *>(patch);
        const uint32_t *wsm_w = reinterpret_cast<const uint32_t *>(w_sm);
        const int b_lane = g * (p.wpitch / 2) + t;  // word offset of B[k = 2t, 2t+1][n = g] in [f][k]; n8 tile nt: + 8 nt rows
        int ks = 0;
        for (int r = 0; r < p.R; ++r) {
            for (int s0 = 0; s0 < p.S4; s0 += 4, ++ks) {
                uint32_t a[2][4];
#pragma unroll
                for (int mt = 0; mt < 2; ++mt) {
                    const int py = (2 * warp + mt) * p.sh + r;
                    const uint32_t *row = patch_w + (py * p.PW + s0) * 2 + a_lane;
                    a[mt][0] = row[0];                  // (row g,     k 2t..2t+1)
                    a[mt][1] = row[8 * p.sw * 2];       // (row g + 8, k 2t..2t+1)
                    a[mt][2] = row[4];                  // (row g,     k 2t+8..)
                    a[mt][3] = row[8 * p.sw * 2 + 4];   // (row g + 8, k 2t+8..)
                }
                const uint32_t *bk = wsm_w + b_lane + ks * 8;
#pragma unroll
                for (int nt = 0; nt < 8; ++nt) {
                    const uint32_t b0 = bk[nt * 8 * (p.wpitch / 2)], b1 = bk[nt * 8 * (p.wpitch / 2) + 4];
                    mma_m16n8k16<T>(acc[0][nt], a[0], b0, b1);
                    mma_m16n8k16<T>(acc[1][nt], a[1], b0, b1);
                }
            }
        }

        // ---- epilogue: BN + ReLU, through the warp's staging tile ([32 pixels][64 f], padded rows), 16-byte NHWC stores
#pragma unroll
        for (int mt = 0; mt < 2; ++mt)
#pragma unroll
            for (int nt = 0; nt < 8; ++nt) {
                const float2 ab0 = bn_sm[nt * 8 + 2 * t], ab1 = bn_sm[nt * 8 + 2 * t + 1];
#pragma unroll
                for (int h = 0; h < 2; ++h) {  // rows g / g + 8
                    float x0 = __fmaf_rn(acc[mt][nt][2 * h], ab0.x, ab0.y), x1 = __fmaf_rn(acc[mt][nt][2 * h + 1], ab1.x, ab1.y);
                    if (p.relu) {
                        x0 = fmaxf(x0, 0.f);
                        x1 = fmaxf(x1, 0.f);
                    }
                    T pr[2] = {from_f<T>(x0), from_f<T>(x1)};
                    *reinterpret_cast<uint32_t *>(my_stg + (mt * 16 + g + 8 * h) * ST_STG_PITCH + (nt * 8 + 2 * t) * 2) =
                        *reinterpret_cast<const uint32_t *>(pr);
                }
            }
        __syncwarp();
        const int f8 = p.F / 8;
#pragma unroll
        for (int i = 0; i < 8; ++i) {
            const int px = i * 4 + (lane >> 3), ch = lane & 7;  // staging pixel (mt * 16 + column), 16-byte chunk
            const int oh = oh0 + 2 * warp + (px >> 4), ow = ow0 + (px & 15);
            if (oh < p.OH && ow < p.OW && ch < f8) {
                const uint4 v = *reinterpret_cast<const uint4 *>(my_stg + px * ST_STG_PITCH + ch * 16);
                *reinterpret_cast<uint4 *>(Y + (((int64_t)n * p.OH + oh) * p.OW + ow) * p.F + ch * 8) = v;
            }
        }
        __syncwarp();
    }
}

static int stem_smem(const StemParams &p) {
    return ST_FMAX * p.wpitch * 2 + ST_FMAX * 8 + ST_WARPS * 32 * ST_STG_PITCH + p.PH * p.PW * 8;
}

template <typename T>
static int launch_stem_t(const StemParams &p, int smem, int64_t tiles, cudaStream_t st) {
    const int ctas_per_sm = std::max(1, std::min(2, (220 * 1024) / (smem + 1024)));
    return launch("conv(stem)", conv_stem_kernel<T>,
                  {dim3((unsigned)std::min<int64_t>(tiles, (int64_t)kNumSMs * ctas_per_sm)), dim3(ST_THREADS), smem, st}, p);
}

}  // namespace itb

using namespace itb;

extern "C" int it_b200_conv2d_stem_supported(int dtype, int C, int F, int R, int S, int ph, int pw, int sh, int sw, int dh, int dw,
                                             int groups) {
    return conv_stem_ok(dtype, C, F, R, S, ph, pw, sh, sw, dh, dw, groups) ? 1 : 0;
}

extern "C" int it_b200_conv2d_stem(int dtype, const void *x, const void *w, void *y, int N, int C, int H, int W, int F, int R, int S,
                                   int ph, int pw, int sh, int sw, const float *bn_mean, const float *bn_var, const float *bn_scale,
                                   const float *bn_bias, float bn_eps, int relu, void *stream) {
    ITB_CHECK(conv_stem_ok(dtype, C, F, R, S, ph, pw, sh, sw, 1, 1, 1),
              "conv(stem): f16 / bf16, C <= 4, F <= 64 (F %% 8 == 0), filters up to 7 x 8, strides <= 2: C=%d F=%d %dx%d", C, F, R, S);
    ITB_CHECK((bn_scale == nullptr) == (bn_mean == nullptr) && (bn_scale == nullptr) == (bn_var == nullptr) &&
                  (bn_scale == nullptr) == (bn_bias == nullptr),
              "conv(stem): the four BatchNorm parameter vectors go together");
    ITB_CHECK(aligned16(y), "conv(stem): y must be 16-byte aligned");
    StemParams p{};
    p.x = x;
    p.w = w;
    p.y = y;
    p.bn_mean = bn_mean;
    p.bn_var = bn_var;
    p.bn_scale = bn_scale;
    p.bn_bias = bn_bias;
    p.bn_eps = bn_eps;
    p.relu = relu;
    p.N = N;
    p.C = C;
    p.H = H;
    p.W = W;
    p.F = F;
    p.R = R;
    p.S = S;
    conv_out_hw(H, W, R, S, ph, pw, sh, sw, 1, 1, p.OH, p.OW);
    if ((int64_t)N * p.OH * p.OW <= 0) return 0;
    p.ph = ph;
    p.pw = pw;
    p.sh = sh;
    p.sw = sw;
    p.tiles_h = (p.OH + ST_TH - 1) / ST_TH;
    p.tiles_w = (p.OW + ST_TW - 1) / ST_TW;
    const int64_t tiles = (int64_t)N * p.tiles_h * p.tiles_w;
    ITB_CHECK(tiles < (1ll << 31), "conv(stem): too many output blocks");
    p.tiles = (int)tiles;
    p.S4 = ((S + 3) / 4) * 4;
    p.ksteps = R * p.S4 / 4;
    p.PH = (ST_TH - 1) * sh + R;
    p.PW = (ST_TW - 1) * sw + p.S4;
    p.wpitch = p.ksteps * 16 + 8;
    const int smem = stem_smem(p);
    auto st = (cudaStream_t)stream;
    if (dtype == ITB_F16) return launch_stem_t<__half>(p, smem, tiles, st);
    return launch_stem_t<__nv_bfloat16>(p, smem, tiles, st);
}
