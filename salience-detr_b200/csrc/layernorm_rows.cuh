// One-warp-per-row LayerNorm shared by the token-layout backbones (convnext.cu, swin.cu, focalnet.cu, patch_stem.cuh).
//
// The row lives in registers: lane l owns the channel pairs 64 j + 2 l, j < nj = C / 64 <= MaxJ.  Two passes (mean, then the
// mean of squared deviations) with butterfly warp sums, so the result is order-fixed, a NaN anywhere in the row makes the
// whole row NaN as in torch, and a constant row gives (x - mean) * rsqrt(eps) = 0 times the weight plus the bias.
#pragma once

namespace sdetr {

__device__ __forceinline__ float cn_warp_sum(float v) {
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
    return v;
}

// mean and 1 / sqrt(variance + eps) of the row held in v (lane's pairs 64 j + 2 lane, j < nj)
template <int MaxJ>
__device__ __forceinline__ void cn_layernorm_stats(const float2 (&v)[MaxJ], int nj, int C, float eps, float &mean, float &rstd) {
    float s = 0.f;
#pragma unroll
    for (int j = 0; j < MaxJ; ++j)
        if (j < nj) s += v[j].x + v[j].y;
    mean = cn_warp_sum(s) / (float)C;
    float q = 0.f;
#pragma unroll
    for (int j = 0; j < MaxJ; ++j)
        if (j < nj) {
            const float dx = v[j].x - mean, dy = v[j].y - mean;
            q = fmaf(dx, dx, q), q = fmaf(dy, dy, q);
        }
    rstd = rsqrtf(cn_warp_sum(q) / (float)C + eps);
}

// LayerNorm of the row held in v (lane's pairs 64 j + 2 lane) -> dst[c]
template <int MaxJ>
__device__ __forceinline__ void cn_layernorm_store(const float2 (&v)[MaxJ], int nj, int C, int lane, const float *__restrict__ g,
                                                   const float *__restrict__ b, float eps, float *__restrict__ dst) {
    float mean, rstd;
    cn_layernorm_stats(v, nj, C, eps, mean, rstd);
#pragma unroll
    for (int j = 0; j < MaxJ; ++j)
        if (j < nj) {
            const int c = 64 * j + 2 * lane;
            const float2 gw = __ldg(reinterpret_cast<const float2 *>(g + c)), bw = __ldg(reinterpret_cast<const float2 *>(b + c));
            *reinterpret_cast<float2 *>(dst + c) = make_float2((v[j].x - mean) * rstd * gw.x + bw.x, (v[j].y - mean) * rstd * gw.y + bw.y);
        }
}

}  // namespace sdetr
