// ConvNeXt backbone in token layout (ConvNeXtBackbone.forward_tokens): the kernels around the pointwise GEMMs.  Both
// Linears of every CNBlock and every 2x2 / stride-2 downsampling convolution run on sdetr_gemm_f16x3_ex (gemm_f16x3.cu).
//
//   sdetr_convnext_stem                conv 4x4, stride 4, 3 -> C channels with bias, then LayerNorm over C (affine), from the
//                                      NCHW fp32 image batch to (b, Ho*Wo, C) token rows.  fp32 FMAs, taps in (c, ky, kx) order
//                                      (patch_stem_kernel<4, 0> of patch_stem.cuh).
//   sdetr_dwconv7x7_layernorm_tokens   depthwise conv 7x7, padding 3, with bias, then LayerNorm over C (affine), token rows in,
//                                      token rows out (a separate buffer: the block input stays the residual).
//   sdetr_layernorm_tokens_s2d         LayerNorm over C of token rows, written space-to-depth: output row (y, x) of the
//                                      (H / 2) x (W / 2) map holds LayerNorm(x[2y + dy, 2x + dx]) at columns (2 dy + dx) C + c.
//
// One warp per token row with the two-pass LayerNorm of layernorm_rows.cuh: a NaN anywhere in the row (or in a convolution
// window feeding it) makes the whole row NaN, as in torch.
#include <math.h>

#include "common.cuh"
#include "layernorm_rows.cuh"
#include "patch_stem.cuh"

namespace sdetr {

constexpr int kCnMaxJ = kStemMaxJ;     // C <= 64 * 24 = 1536
constexpr int kCnWarps = kStemWarps;   // token rows per CTA of 256 threads

__global__ void __launch_bounds__(32 * kCnWarps) dwconv7x7_layernorm_kernel(const float *__restrict__ x, int batch, int H, int W, int C,
                                                                             const float *__restrict__ w /* (49, C) */,
                                                                             const float *__restrict__ bias,
                                                                             const float *__restrict__ g,
                                                                             const float *__restrict__ beta, float eps,
                                                                             float *__restrict__ y) {
    const int lane = threadIdx.x & 31, nj = C >> 6;
    const int64_t tok = (int64_t)blockIdx.x * kCnWarps + (threadIdx.x >> 5), hw = (int64_t)H * W;
    if (tok >= batch * hw) return;
    const int n = (int)(tok / hw), pix = (int)(tok - n * hw), oy = pix / W, ox = pix - oy * W;
    float2 v[kCnMaxJ];
#pragma unroll
    for (int j = 0; j < kCnMaxJ; ++j) v[j] = make_float2(0.f, 0.f);
    const float *xn = x + (int64_t)n * hw * C + 2 * lane;
    for (int ky = 0; ky < 7; ++ky) {
        const int iy = oy + ky - 3;
        if ((unsigned)iy >= (unsigned)H) continue;  // zero padding contributes nothing
        for (int kx = 0; kx < 7; ++kx) {
            const int ix = ox + kx - 3;
            if ((unsigned)ix >= (unsigned)W) continue;
            const float *xr = xn + ((int64_t)iy * W + ix) * C, *wr = w + (ky * 7 + kx) * C + 2 * lane;
#pragma unroll
            for (int j = 0; j < kCnMaxJ; ++j)
                if (j < nj) {
                    const float2 xv = __ldg(reinterpret_cast<const float2 *>(xr + 64 * j));
                    const float2 wv = __ldg(reinterpret_cast<const float2 *>(wr + 64 * j));
                    v[j].x = fmaf(xv.x, wv.x, v[j].x), v[j].y = fmaf(xv.y, wv.y, v[j].y);
                }
        }
    }
#pragma unroll
    for (int j = 0; j < kCnMaxJ; ++j)
        if (j < nj) {
            const float2 bv = __ldg(reinterpret_cast<const float2 *>(bias + 64 * j + 2 * lane));
            v[j].x += bv.x, v[j].y += bv.y;
        }
    cn_layernorm_store(v, nj, C, lane, g, beta, eps, y + tok * C);
}

// one warp per (output pixel, d = 2 dy + dx): the input row (2 oy + dy, 2 ox + dx) normalised into the output row's slot d
__global__ void __launch_bounds__(32 * kCnWarps) layernorm_s2d_kernel(const float *__restrict__ x, int batch, int H, int W, int C,
                                                                       int Ho, int Wo, const float *__restrict__ g,
                                                                       const float *__restrict__ beta, float eps,
                                                                       float *__restrict__ y) {
    const int lane = threadIdx.x & 31, nj = C >> 6;
    const int64_t item = (int64_t)blockIdx.x * kCnWarps + (threadIdx.x >> 5), hwo = (int64_t)Ho * Wo;
    if (item >= batch * hwo * 4) return;
    const int d = (int)(item & 3);
    const int64_t tok = item >> 2;
    const int n = (int)(tok / hwo), pix = (int)(tok - n * hwo), oy = pix / Wo, ox = pix - oy * Wo;
    const float *xr = x + ((int64_t)n * H * W + (int64_t)(2 * oy + (d >> 1)) * W + 2 * ox + (d & 1)) * C + 2 * lane;
    float2 v[kCnMaxJ];
#pragma unroll
    for (int j = 0; j < kCnMaxJ; ++j) v[j] = j < nj ? __ldg(reinterpret_cast<const float2 *>(xr + 64 * j)) : make_float2(0.f, 0.f);
    cn_layernorm_store(v, nj, C, lane, g, beta, eps, y + tok * 4 * C + d * C);
}

inline unsigned cn_blocks(int64_t warps) { return (unsigned)((warps + kCnWarps - 1) / kCnWarps); }

}  // namespace sdetr

using namespace sdetr;

#define CN_CHECK_C(what)                                                                                                       \
    SDETR_REQUIRE(C > 0 && C % 64 == 0 && C <= 64 * kCnMaxJ, SDETR_ERR_UNSUPPORTED, what ": C=%d must be a multiple of 64 up to %d", \
                  C, 64 * kCnMaxJ)

extern "C" int sdetr_convnext_stem(const float *x, int batch, int H, int W, int C, const float *weight, const float *bias,
                                   const float *ln_weight, const float *ln_bias, float eps, float *y, sdetr_stream_t stream) {
    SDETR_REQUIRE(x && weight && bias && ln_weight && ln_bias && y, SDETR_ERR_INVALID_ARG, "convnext_stem: null pointer");
    SDETR_REQUIRE(batch >= 0 && H > 0 && W > 0 && eps >= 0.f, SDETR_ERR_INVALID_ARG, "convnext_stem: bad sizes");
    CN_CHECK_C("convnext_stem");
    SDETR_REQUIRE(aligned16(weight) && aligned16(bias) && aligned16(ln_weight) && aligned16(ln_bias) && aligned16(y),
                  SDETR_ERR_INVALID_ARG, "convnext_stem: weight, biases and y must be 16-byte aligned");
    const int Ho = H / 4, Wo = W / 4;
    const int64_t toks = (int64_t)batch * Ho * Wo;
    SDETR_REQUIRE((int64_t)batch * 3 * H * W < (1LL << 40) && toks < (1LL << 31), SDETR_ERR_INVALID_ARG, "convnext_stem: image too large");
    if (toks == 0) return SDETR_OK;
    patch_stem_kernel<4, 0><<<cn_blocks(toks), 32 * kCnWarps, 0, (cudaStream_t)stream>>>(x, batch, H, W, Ho, Wo, C, weight, bias,
                                                                                           ln_weight, ln_bias, eps, y);
    return check_launch("convnext_stem");
}

extern "C" int sdetr_dwconv7x7_layernorm_tokens(const float *x, int batch, int H, int W, int C, const float *weight,
                                                const float *bias, const float *ln_weight, const float *ln_bias, float eps, float *y,
                                                sdetr_stream_t stream) {
    SDETR_REQUIRE(x && weight && bias && ln_weight && ln_bias && y, SDETR_ERR_INVALID_ARG, "dwconv7x7_layernorm_tokens: null pointer");
    SDETR_REQUIRE(batch >= 0 && H > 0 && W > 0 && eps >= 0.f, SDETR_ERR_INVALID_ARG, "dwconv7x7_layernorm_tokens: bad sizes");
    CN_CHECK_C("dwconv7x7_layernorm_tokens");
    SDETR_REQUIRE(x != y, SDETR_ERR_INVALID_ARG, "dwconv7x7_layernorm_tokens: y must not alias x");
    SDETR_REQUIRE(aligned16(x) && aligned16(weight) && aligned16(bias) && aligned16(ln_weight) && aligned16(ln_bias) && aligned16(y),
                  SDETR_ERR_INVALID_ARG, "dwconv7x7_layernorm_tokens: operands must be 16-byte aligned");
    const int64_t toks = (int64_t)batch * H * W;
    SDETR_REQUIRE(toks < (1LL << 31), SDETR_ERR_INVALID_ARG, "dwconv7x7_layernorm_tokens: map too large");
    if (toks == 0) return SDETR_OK;
    dwconv7x7_layernorm_kernel<<<cn_blocks(toks), 32 * kCnWarps, 0, (cudaStream_t)stream>>>(x, batch, H, W, C, weight, bias,
                                                                                              ln_weight, ln_bias, eps, y);
    return check_launch("dwconv7x7_layernorm_tokens");
}

extern "C" int sdetr_layernorm_tokens_s2d(const float *x, int batch, int H, int W, int C, const float *ln_weight,
                                          const float *ln_bias, float eps, float *y, sdetr_stream_t stream) {
    SDETR_REQUIRE(x && ln_weight && ln_bias && y, SDETR_ERR_INVALID_ARG, "layernorm_tokens_s2d: null pointer");
    SDETR_REQUIRE(batch >= 0 && H > 0 && W > 0 && eps >= 0.f, SDETR_ERR_INVALID_ARG, "layernorm_tokens_s2d: bad sizes");
    CN_CHECK_C("layernorm_tokens_s2d");
    SDETR_REQUIRE(x != y, SDETR_ERR_INVALID_ARG, "layernorm_tokens_s2d: y must not alias x");
    SDETR_REQUIRE(aligned16(x) && aligned16(ln_weight) && aligned16(ln_bias) && aligned16(y), SDETR_ERR_INVALID_ARG,
                  "layernorm_tokens_s2d: operands must be 16-byte aligned");
    const int Ho = H / 2, Wo = W / 2;
    const int64_t items = (int64_t)batch * Ho * Wo * 4;
    SDETR_REQUIRE(items < (1LL << 31), SDETR_ERR_INVALID_ARG, "layernorm_tokens_s2d: map too large");
    if (items == 0) return SDETR_OK;
    layernorm_s2d_kernel<<<cn_blocks(items), 32 * kCnWarps, 0, (cudaStream_t)stream>>>(x, batch, H, W, C, Ho, Wo, ln_weight, ln_bias,
                                                                                         eps, y);
    return check_launch("layernorm_tokens_s2d");
}
