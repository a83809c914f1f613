// Backward of the coarse-to-fine score upsample -- sdetr_upsample_bilinear_ac_backward.
//
// The salience filter's training path resizes each coarser level's score map with
// F.interpolate(mode="bilinear", align_corners=True) (salience_transformer.py:134-143).  torch's CUDA backward of that op
// scatters every fine pixel's gradient into its four coarse corners with atomics, so its result depends on the order of the
// additions, and it raises under torch.use_deterministic_algorithms(True).  This kernel is the same operator in gather
// form: one thread per coarse cell walks, in row-major order, the fine pixels whose stencil contains the cell, sums their
// weighted gradients in registers and writes the cell once.  The stencil is torch's forward one, in the same fp32 arithmetic:
//     scale = (in - 1) / (out - 1)  (0 when out == 1),  src = scale * dst,  i0 = (int)src,  i1 = i0 + (i0 < in - 1),
//     lambda = src - i0;  the cell i0 gets weight 1 - lambda, the cell i1 gets lambda (both when i0 == i1).
#include "common.cuh"

namespace sdetr {

// weight of coarse index c in the stencil of fine index d along one axis; `member` = c is one of its two corners
__device__ __forceinline__ float ac_axis_weight(float scale, int d, int in, int c, bool &member) {
    const float src = scale * (float)d;
    const int i0 = (int)src;
    const int i1 = i0 + (i0 < in - 1 ? 1 : 0);
    const float l1 = src - (float)i0, l0 = 1.f - l1;
    member = i0 == c || i1 == c;
    return (i0 == c ? l0 : 0.f) + (i1 == c ? l1 : 0.f);
}

// fine indices [lo, hi] whose stencil can contain coarse index c (a margin of one index beyond the exact bounds; every
// candidate is then tested with the forward's own arithmetic)
__device__ __forceinline__ void ac_fine_range(float scale, double inv_scale, int c, int out, int &lo, int &hi) {
    if (scale == 0.f) {  // out == 1 or in == 1: every fine index reads coarse index 0 (and 1 with weight 0)
        lo = 0, hi = out - 1;
        return;
    }
    lo = (int)floor((c - 1) * inv_scale) - 1;
    hi = (int)ceil((c + 1) * inv_scale) + 1;
    lo = lo < 0 ? 0 : lo;
    hi = hi > out - 1 ? out - 1 : hi;
}

__global__ void __launch_bounds__(256) upsample_bilinear_ac_bwd_kernel(const float *__restrict__ gf, int64_t planes, int H,
                                                                       int W, int Hc, int Wc, float sy, float sx,
                                                                       double inv_sy, double inv_sx, float *__restrict__ gc) {
    const int64_t t = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (t >= planes * Hc * Wc) return;
    const int j = (int)(t % Wc), i = (int)((t / Wc) % Hc);
    const int64_t plane = t / ((int64_t)Hc * Wc);
    const float *g = gf + plane * H * W;
    int y0, y1, x0, x1;
    ac_fine_range(sy, inv_sy, i, H, y0, y1);
    ac_fine_range(sx, inv_sx, j, W, x0, x1);
    float acc = 0.f;
    for (int y = y0; y <= y1; ++y) {
        bool my;
        const float wy = ac_axis_weight(sy, y, Hc, i, my);
        if (!my) continue;
        for (int x = x0; x <= x1; ++x) {
            bool mx;
            const float wx = ac_axis_weight(sx, x, Wc, j, mx);
            if (mx) acc += (wy * wx) * __ldg(g + (int64_t)y * W + x);
        }
    }
    gc[t] = acc;
}

}  // namespace sdetr

using namespace sdetr;

extern "C" int sdetr_upsample_bilinear_ac_backward(const float *grad_fine, int planes, int H, int W, int Hc, int Wc,
                                                   float *grad_coarse, sdetr_stream_t stream) {
    SDETR_REQUIRE(grad_fine && grad_coarse, SDETR_ERR_INVALID_ARG, "upsample_bilinear_ac_backward: null pointer");
    SDETR_REQUIRE(planes >= 0 && H > 0 && W > 0 && Hc > 0 && Wc > 0, SDETR_ERR_INVALID_ARG,
                  "upsample_bilinear_ac_backward: non-positive size");
    if (planes == 0) return SDETR_OK;
    // torch's area_pixel_compute_scale with align_corners (fp32 accumulation type of float inputs)
    const float sy = H > 1 ? (float)(Hc - 1) / (float)(H - 1) : 0.f;
    const float sx = W > 1 ? (float)(Wc - 1) / (float)(W - 1) : 0.f;
    const int64_t cells = (int64_t)planes * Hc * Wc;
    upsample_bilinear_ac_bwd_kernel<<<(unsigned)((cells + 255) / 256), 256, 0, (cudaStream_t)stream>>>(
        grad_fine, planes, H, W, Hc, Wc, sy, sx, sy > 0.f ? 1.0 / sy : 0.0, sx > 0.f ? 1.0 / sx : 0.0, grad_coarse);
    return check_launch("upsample_bilinear_ac_backward");
}
