// The patch-embedding stem of the token-layout backbones: conv K x K, stride 4, padding P, 3 -> C channels with bias, then
// LayerNorm over C (affine), from the NCHW fp32 image batch to (b, Ho*Wo, C) token rows.  One warp per output pixel, fp32 FMAs,
// taps in (c, ky, kx) order, then the bias; a tap outside the image reads zero.  Instances: <4, 0> the ConvNeXt / Swin stem
// (sdetr_convnext_stem, convnext.cu), <7, 2> the FocalNet stem (sdetr_focalnet_stem, focalnet.cu).
#pragma once

#include "layernorm_rows.cuh"

namespace sdetr {

constexpr int kStemMaxJ = 24;   // C <= 64 * 24 = 1536
constexpr int kStemWarps = 8;   // token rows per CTA of 256 threads

template <int K, int P>
__global__ void __launch_bounds__(32 * kStemWarps) patch_stem_kernel(const float *__restrict__ x, int batch, int H, int W, int Ho,
                                                                      int Wo, int C, const float *__restrict__ w /* (3 K K, C) */,
                                                                      const float *__restrict__ bias, const float *__restrict__ g,
                                                                      const float *__restrict__ beta, float eps,
                                                                      float *__restrict__ y) {
    const int lane = threadIdx.x & 31, nj = C >> 6;
    const int64_t tok = (int64_t)blockIdx.x * kStemWarps + (threadIdx.x >> 5), hw = (int64_t)Ho * Wo;
    if (tok >= batch * hw) return;
    const int n = (int)(tok / hw), pix = (int)(tok - n * hw), oy = pix / Wo, ox = pix - oy * Wo;
    float2 v[kStemMaxJ];
#pragma unroll
    for (int j = 0; j < kStemMaxJ; ++j) v[j] = make_float2(0.f, 0.f);
    const int y0 = 4 * oy - P, x0 = 4 * ox - P;  // P == 0: every tap is inside the image
    const float *xn = x + (int64_t)n * 3 * H * W + (int64_t)y0 * W + x0;
    for (int c = 0; c < 3; ++c)
        for (int ky = 0; ky < K; ++ky) {
            if (P > 0 && (unsigned)(y0 + ky) >= (unsigned)H) continue;  // zero rows contribute nothing
#pragma unroll(P > 0 ? 1 : K)  // unrolling the padded instance's checked taps costs registers
            for (int kx = 0; kx < K; ++kx) {
                if (P > 0 && (unsigned)(x0 + kx) >= (unsigned)W) continue;
                const float xv = __ldg(xn + ((int64_t)c * H + ky) * W + kx);  // one address per warp: a broadcast
                const float *wr = w + (int64_t)((c * K + ky) * K + kx) * C + 2 * lane;
#pragma unroll
                for (int j = 0; j < kStemMaxJ; ++j)
                    if (j < nj) {
                        const float2 wv = __ldg(reinterpret_cast<const float2 *>(wr + 64 * j));
                        v[j].x = fmaf(xv, wv.x, v[j].x), v[j].y = fmaf(xv, wv.y, v[j].y);
                    }
            }
        }
#pragma unroll
    for (int j = 0; j < kStemMaxJ; ++j)
        if (j < nj) {
            const float2 bv = __ldg(reinterpret_cast<const float2 *>(bias + 64 * j + 2 * lane));
            v[j].x += bv.x, v[j].y += bv.y;
        }
    cn_layernorm_store(v, nj, C, lane, g, beta, eps, y + tok * C);
}

}  // namespace sdetr
