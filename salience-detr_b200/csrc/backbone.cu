// ResNet backbone in token layout (ResNetBackbone.forward_tokens): the two kernels before the first Bottleneck.  Every
// convolution of the blocks is sdetr_conv2d_f16x3 (neck.cu).
//
//   sdetr_resnet_stem            conv 7x7, stride 2, padding 3, 3 -> 64 channels, folded FrozenBatchNorm bias and ReLU, from
//                                the NCHW fp32 image batch to (b, Ho*Wo, 64) token rows.  Plain fp32 FMAs on the CUDA cores, taps
//                                summed in (channel, ky, kx) order: the stem is under 3 % of the backbone's operations.
//   sdetr_maxpool3x3s2_tokens    3x3 / stride 2 / padding 1 max-pool on token rows, 16-byte channel vectors.
//   sdetr_frozen_bn_fold         a convolution weight with its FrozenBatchNorm folded in, on the device (the training path
//                                re-folds every call): float64 arithmetic, each operation rounded alone.
#include <math.h>

#include "common.cuh"

namespace sdetr {

// Stem tile: 16 x 16 output pixels x 64 channels per CTA of 256 threads.  Thread t owns channels 8 (t & 7) .. + 7 of the 8
// consecutive output pixels (row (t >> 3) >> 1, columns 8 ((t >> 3) & 1) .. + 7).  Shared memory: the CTA's weights as
// [147 taps][64 channels], then the input tile with its halo, [3][37][37] (zero where it falls outside the image).
constexpr int kStemTile = 16, kStemThreads = 256, kStemTaps = 147, kStemC = 64;
constexpr int kStemIn = (kStemTile - 1) * 2 + 7;  // 37 input rows / columns per tile
constexpr int kStemSmem = (kStemTaps * kStemC + 3 * kStemIn * kStemIn) * 4;

__global__ void __launch_bounds__(kStemThreads) resnet_stem_kernel(const float *__restrict__ x, int H, int W, int Ho, int Wo,
                                                                   const float *__restrict__ w /* (147, 64) */,
                                                                   const float *__restrict__ bias, float *__restrict__ y) {
    extern __shared__ float sm[];
    float *sw = sm, *sx = sm + kStemTaps * kStemC;
    const int tid = threadIdx.x, n = blockIdx.z, oy0 = blockIdx.y * kStemTile, ox0 = blockIdx.x * kStemTile;
    const int iy0 = oy0 * 2 - 3, ix0 = ox0 * 2 - 3;
    for (int i = tid; i < kStemTaps * kStemC / 4; i += kStemThreads)
        reinterpret_cast<float4 *>(sw)[i] = __ldg(reinterpret_cast<const float4 *>(w) + i);
    const float *xn = x + (int64_t)n * 3 * H * W;
    for (int i = tid; i < 3 * kStemIn * kStemIn; i += kStemThreads) {
        const int c = i / (kStemIn * kStemIn), r = (i / kStemIn) % kStemIn, col = i % kStemIn;
        const int iy = iy0 + r, ix = ix0 + col;
        sx[i] = (unsigned)iy < (unsigned)H && (unsigned)ix < (unsigned)W ? __ldg(xn + ((int64_t)c * H + iy) * W + ix) : 0.f;
    }
    __syncthreads();

    const int cg = (tid & 7) * 8, pg = tid >> 3, row = pg >> 1, col0 = (pg & 1) * 8;
    float acc[8][8];
#pragma unroll
    for (int j = 0; j < 8; ++j)
#pragma unroll
        for (int k = 0; k < 8; ++k) acc[j][k] = 0.f;
    for (int c = 0; c < 3; ++c) {
        for (int ky = 0; ky < 7; ++ky) {
            const float *xr = sx + (c * kStemIn + row * 2 + ky) * kStemIn + col0 * 2;
            const float *wr = sw + ((c * 7 + ky) * 7) * kStemC + cg;
#pragma unroll
            for (int kx = 0; kx < 7; ++kx) {
                const float4 wa = *reinterpret_cast<const float4 *>(wr + kx * kStemC);
                const float4 wb = *reinterpret_cast<const float4 *>(wr + kx * kStemC + 4);
                const float wv[8] = {wa.x, wa.y, wa.z, wa.w, wb.x, wb.y, wb.z, wb.w};
#pragma unroll
                for (int j = 0; j < 8; ++j) {
                    const float v = xr[2 * j + kx];
#pragma unroll
                    for (int k = 0; k < 8; ++k) acc[j][k] = fmaf(v, wv[k], acc[j][k]);
                }
            }
        }
    }
    const float4 ba = __ldg(reinterpret_cast<const float4 *>(bias + cg)), bb = __ldg(reinterpret_cast<const float4 *>(bias + cg + 4));
    const int oy = oy0 + row;
    if (oy >= Ho) return;
#pragma unroll
    for (int j = 0; j < 8; ++j) {
        const int ox = ox0 + col0 + j;
        if (ox >= Wo) break;
        float *dst = y + ((int64_t)n * Ho * Wo + (int64_t)oy * Wo + ox) * kStemC + cg;
        reinterpret_cast<float4 *>(dst)[0] = make_float4(relu_nan(acc[j][0] + ba.x), relu_nan(acc[j][1] + ba.y),
                                                         relu_nan(acc[j][2] + ba.z), relu_nan(acc[j][3] + ba.w));
        reinterpret_cast<float4 *>(dst)[1] = make_float4(relu_nan(acc[j][4] + bb.x), relu_nan(acc[j][5] + bb.y),
                                                         relu_nan(acc[j][6] + bb.z), relu_nan(acc[j][7] + bb.w));
    }
}

// torch's max_pool2d rule per element: a value replaces the running maximum when it is larger or NaN, so a NaN in the window
// gives NaN; padding never enters the window (the maximum starts at -inf, and every window holds at least one pixel).
__device__ __forceinline__ float pool_max(float m, float v) { return (v > m || isnan(v)) ? v : m; }

__global__ void maxpool3x3s2_tokens_kernel(const float *__restrict__ x, int64_t x_pitch, int64_t ldx, int batch, int H, int W,
                                           int C, int Ho, int Wo, float *__restrict__ y, int64_t y_pitch, int64_t ldy) {
    const int c4 = C >> 2, hwo = Ho * Wo;
    const int64_t total = (int64_t)batch * hwo * c4;
    for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (int64_t)gridDim.x * blockDim.x) {
        const int c = (int)(i % c4) * 4;
        const int64_t r = i / c4;
        const int n = (int)(r / hwo), pix = (int)(r - (int64_t)n * hwo), oy = pix / Wo, ox = pix - oy * Wo;
        float4 m = make_float4(-INFINITY, -INFINITY, -INFINITY, -INFINITY);
        const float *xn = x + (int64_t)n * x_pitch + c;
        for (int ky = 0; ky < 3; ++ky) {
            const int iy = oy * 2 - 1 + ky;
            if ((unsigned)iy >= (unsigned)H) continue;
            for (int kx = 0; kx < 3; ++kx) {
                const int ix = ox * 2 - 1 + kx;
                if ((unsigned)ix >= (unsigned)W) continue;
                const float4 v = ldg_f4(xn + ((int64_t)iy * W + ix) * ldx);
                m.x = pool_max(m.x, v.x), m.y = pool_max(m.y, v.y), m.z = pool_max(m.z, v.z), m.w = pool_max(m.w, v.w);
            }
        }
        *reinterpret_cast<float4 *>(y + (int64_t)n * y_pitch + (int64_t)pix * ldy + c) = m;
    }
}

// s = weight * rsqrt(var + eps), w_folded = w * s, bias_folded = bias - mean * s: each in float64 with its own rounding (no
// contraction), as torch computes them op by op, then rounded to fp32 once; rsqrt is the same libdevice function torch calls
__device__ __forceinline__ double frozen_bn_scale(const float *weight, const float *var, double eps, int c) {
    return __dmul_rn((double)__ldg(weight + c), rsqrt(__dadd_rn((double)__ldg(var + c), eps)));
}

__global__ void frozen_bn_fold_kernel(const float *__restrict__ w, int cout, int64_t per_co, const float *__restrict__ bn_w,
                                      const float *__restrict__ bn_b, const float *__restrict__ mean, const float *__restrict__ var,
                                      double eps, float *__restrict__ w_folded, float *__restrict__ scale, float *__restrict__ bias) {
    const int64_t n = (int64_t)cout * per_co;
    for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (int64_t)gridDim.x * blockDim.x) {
        const int c = (int)(i / per_co);
        const double s = frozen_bn_scale(bn_w, var, eps, c);
        w_folded[i] = __double2float_rn(__dmul_rn((double)w[i], s));
        if (i - (int64_t)c * per_co == 0) {
            if (scale) scale[c] = __double2float_rn(s);
            if (bias) bias[c] = __double2float_rn(__dsub_rn((double)__ldg(bn_b + c), __dmul_rn((double)__ldg(mean + c), s)));
        }
    }
}

}  // namespace sdetr

using namespace sdetr;

extern "C" int sdetr_resnet_stem(const float *x, int batch, int H, int W, const float *weight, const float *bias, float *y,
                                 sdetr_stream_t stream) {
    SDETR_REQUIRE(x && weight && bias && y, SDETR_ERR_INVALID_ARG, "resnet_stem: null pointer");
    SDETR_REQUIRE(batch >= 0 && H > 0 && W > 0, SDETR_ERR_INVALID_ARG, "resnet_stem: bad sizes");
    SDETR_REQUIRE(aligned16(weight) && aligned16(bias) && aligned16(y), SDETR_ERR_INVALID_ARG,
                  "resnet_stem: weight, bias and y must be 16-byte aligned");
    const int Ho = (H + 6 - 7) / 2 + 1, Wo = (W + 6 - 7) / 2 + 1;
    SDETR_REQUIRE((int64_t)batch * 3 * H * W < (1LL << 40) && (int64_t)Ho * Wo < (1LL << 31) && batch < 65536,
                  SDETR_ERR_INVALID_ARG, "resnet_stem: image too large");
    if (batch == 0) return SDETR_OK;
    static PerDeviceOnce once;
    SDETR_OPT_IN_SMEM(once, resnet_stem_kernel, kStemSmem, "resnet_stem");
    const dim3 grid((unsigned)((Wo + kStemTile - 1) / kStemTile), (unsigned)((Ho + kStemTile - 1) / kStemTile), (unsigned)batch);
    resnet_stem_kernel<<<grid, kStemThreads, kStemSmem, (cudaStream_t)stream>>>(x, H, W, Ho, Wo, weight, bias, y);
    return check_launch("resnet_stem");
}

extern "C" int sdetr_maxpool3x3s2_tokens(const float *x, int64_t x_pitch, int64_t ldx, int batch, int H, int W, int C, float *y,
                                         int64_t y_pitch, int64_t ldy, sdetr_stream_t stream) {
    SDETR_REQUIRE(x && y, SDETR_ERR_INVALID_ARG, "maxpool3x3s2_tokens: null pointer");
    SDETR_REQUIRE(batch >= 0 && H > 0 && W > 0 && C > 0 && C % 4 == 0, SDETR_ERR_INVALID_ARG,
                  "maxpool3x3s2_tokens: bad sizes (C a multiple of 4)");
    SDETR_REQUIRE(aligned16(x) && x_pitch % 4 == 0 && ldx % 4 == 0 && ldx >= C && aligned16(y) && y_pitch % 4 == 0 &&
                      ldy % 4 == 0 && ldy >= C,
                  SDETR_ERR_INVALID_ARG, "maxpool3x3s2_tokens: operands, pitches and row strides must be 16-byte aligned");
    const int Ho = (H + 2 - 3) / 2 + 1, Wo = (W + 2 - 3) / 2 + 1;
    const int64_t total = (int64_t)batch * Ho * Wo * (C / 4);
    if (total == 0) return SDETR_OK;
    const int64_t want = (total + 255) / 256, cap = 8LL * sm_count();
    maxpool3x3s2_tokens_kernel<<<(unsigned)(want < cap ? want : cap), 256, 0, (cudaStream_t)stream>>>(x, x_pitch, ldx, batch, H, W,
                                                                                                       C, Ho, Wo, y, y_pitch, ldy);
    return check_launch("maxpool3x3s2_tokens");
}

extern "C" int sdetr_frozen_bn_fold(const float *w, int Cout, int64_t per_cout, const float *bn_weight, const float *bn_bias,
                                    const float *running_mean, const float *running_var, double eps, float *w_folded,
                                    float *scale, float *bias, sdetr_stream_t stream) {
    SDETR_REQUIRE(w && bn_weight && bn_bias && running_mean && running_var && w_folded, SDETR_ERR_INVALID_ARG,
                  "frozen_bn_fold: null pointer");
    SDETR_REQUIRE(Cout > 0 && per_cout > 0, SDETR_ERR_INVALID_ARG, "frozen_bn_fold: bad sizes");
    const int64_t n = (int64_t)Cout * per_cout, want = (n + 255) / 256, cap = 8LL * sm_count();
    frozen_bn_fold_kernel<<<(unsigned)(want < cap ? want : cap), 256, 0, (cudaStream_t)stream>>>(
        w, Cout, per_cout, bn_weight, bn_bias, running_mean, running_var, eps, w_folded, scale, bias);
    return check_launch("frozen_bn_fold");
}
