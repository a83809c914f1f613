// FocalNet backbone in token layout (FocalNetBackbone.forward_tokens): the kernels around the Linears.  Every Linear of a block
// (f, h, proj, fc1, fc2) runs on sdetr_gemm_f16x3_ex (gemm_f16x3.cu), each downsample's 3x3 / stride-2 convolution on
// sdetr_conv2d_f16x3 (neck.cu) and its LayerNorm, like the output norms, on sdetr_layernorm_tokens (swin.cu).
//
//   sdetr_focalnet_stem               conv 7x7, stride 4, padding 2 with the map rounded up (ceil(H / 4) x ceil(W / 4)), then
//                                     LayerNorm over C: patch_stem_kernel<7, 2> of patch_stem.cuh.
//   sdetr_focal_level_tokens          one focal level: ctx_{l+1} = GELU(dwconv_k(ctx_l)) and ctx_all += ctx_{l+1} * gate_l, the
//                                     last level also per-tile channel sums of ctx_L for the global context.  k in {3, 5, 7, 9}.
//   sdetr_focal_global_context        ctx_all += GELU(mean_HW(ctx_L)) * gate_L, then / (L + 1) when normalize_modulator is set;
//                                     the partial sums reduced in a fixed order.
//   sdetr_focal_modulate              q * h, elementwise.
//   sdetr_layernorm_scale_add_tokens  t += gamma * LayerNorm(y), the post-LN residual of a block, in place.
//
// The focal kernels tile each image's rows the same way: tile p of image n holds rows [8 R p, 8 R (p + 1)), warp w the rows
// 8 R p + w + 8 i (i < R), one lane per channel pair of a 64-channel slice (grid.y).  R is the smallest count that keeps the
// tiles per image at most kFnMaxTiles, so the global-context kernel's reduction reads at most that many partial rows.
#include <math.h>

#include "common.cuh"
#include "layernorm_rows.cuh"
#include "patch_stem.cuh"

namespace sdetr {

constexpr int kFnWarps = 8;       // warps per CTA of 256 threads
constexpr int kFnMaxTiles = 128;  // row tiles per image
constexpr int kFnLnMaxJ = 24;     // sdetr_layernorm_scale_add_tokens: C <= 64 * 24 = 1536

__device__ __forceinline__ float fn_gelu(float x) { return 0.5f * x * (1.f + erff(x * 0.70710678118654752f)); }

__device__ __forceinline__ float2 fn_ldg2(const float *p) { return __ldg(reinterpret_cast<const float2 *>(p)); }

// rows per warp R and tiles per image of an hw-pixel map
inline int fn_rows_per_warp(int64_t hw) {
    const int64_t r = (hw + kFnWarps * kFnMaxTiles - 1) / (kFnWarps * kFnMaxTiles);
    return (int)(r < 1 ? 1 : r);
}
inline int fn_tiles(int64_t hw) {
    const int64_t rows = (int64_t)kFnWarps * fn_rows_per_warp(hw);
    return (int)((hw + rows - 1) / rows);
}

// Grid (tiles, C / 64, batch).  ctx / gate: image n's row r at (n H W + r) * ld.  ctx_all, out: contiguous (batch, H W, C).  The
// products and sums are rounded one by one, as torch's ctx_all = ctx_all + ctx * gates[:, l:l+1] (level 0 adds to the integer 0).
template <int K, bool Last>
__global__ void __launch_bounds__(32 * kFnWarps) focal_level_kernel(const float *__restrict__ ctx, int64_t ld_ctx,
                                                                     const float *__restrict__ gate, int64_t ld_gate,
                                                                     const float *__restrict__ w /* (K K, C) */, int H, int W, int C,
                                                                     int R, int first, float *__restrict__ out,
                                                                     float *__restrict__ ctx_all, float *__restrict__ part) {
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5, tile = blockIdx.x, n = blockIdx.z;
    const int c = blockIdx.y * 64 + 2 * lane, HW = H * W;
    const int64_t img = (int64_t)n * HW;
    const float *cn = ctx + img * ld_ctx + c;
    float2 s = make_float2(0.f, 0.f);
    for (int i = 0; i < R; ++i) {
        const int pix = (tile * R + i) * kFnWarps + warp;
        if (pix >= HW) break;
        const int oy = pix / W, ox = pix - oy * W;
        float2 a = make_float2(0.f, 0.f);
        for (int ky = 0; ky < K; ++ky) {
            const int iy = oy + ky - K / 2;
            if ((unsigned)iy >= (unsigned)H) continue;  // zero padding contributes nothing
#pragma unroll
            for (int kx = 0; kx < K; ++kx) {
                const int ix = ox + kx - K / 2;
                if ((unsigned)ix >= (unsigned)W) continue;
                const float2 xv = fn_ldg2(cn + ((int64_t)iy * W + ix) * ld_ctx), wv = fn_ldg2(w + (ky * K + kx) * C + c);
                a.x = fmaf(xv.x, wv.x, a.x), a.y = fmaf(xv.y, wv.y, a.y);
            }
        }
        const float2 p = make_float2(fn_gelu(a.x), fn_gelu(a.y));
        const float g = __ldg(gate + (img + pix) * ld_gate);
        float2 *ap = reinterpret_cast<float2 *>(ctx_all + (img + pix) * C + c);
        float2 acc = first ? make_float2(0.f, 0.f) : *ap;
        acc.x = __fadd_rn(acc.x, __fmul_rn(p.x, g)), acc.y = __fadd_rn(acc.y, __fmul_rn(p.y, g));
        *ap = acc;
        if (out) *reinterpret_cast<float2 *>(out + (img + pix) * C + c) = p;
        if (Last) s.x += p.x, s.y += p.y;
    }
    if (Last) {
        __shared__ float2 red[kFnWarps][32];
        red[warp][lane] = s;
        __syncthreads();
        if (warp == 0) {
            float2 t = red[0][lane];
#pragma unroll
            for (int u = 1; u < kFnWarps; ++u) t.x += red[u][lane].x, t.y += red[u][lane].y;
            *reinterpret_cast<float2 *>(part + ((int64_t)n * gridDim.x + tile) * C + c) = t;
        }
    }
}

// Grid (tiles, C / 64, batch), the focal level kernels' tiling.  Warp w sums the partial rows p = w, w + 8, ... in order, warp
// 0 adds the eight warp sums in order: every CTA of an image gets the same bits.  Then over the CTA's rows
// ctx_all = (ctx_all + GELU(sum / HW) * gate) [/ divisor], each operation rounded on its own.
__global__ void __launch_bounds__(32 * kFnWarps) focal_global_kernel(const float *__restrict__ part, int tiles,
                                                                      const float *__restrict__ gate, int64_t ld_gate, int H, int W,
                                                                      int C, int R, float divisor, float *__restrict__ ctx_all) {
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5, n = blockIdx.z;
    const int c = blockIdx.y * 64 + 2 * lane, HW = H * W;
    __shared__ float2 red[kFnWarps][32];
    __shared__ float2 glob[32];
    float2 s = make_float2(0.f, 0.f);
    for (int p = warp; p < tiles; p += kFnWarps) {
        const float2 v = fn_ldg2(part + ((int64_t)n * tiles + p) * C + c);
        s.x += v.x, s.y += v.y;
    }
    red[warp][lane] = s;
    __syncthreads();
    if (warp == 0) {
        float2 t = red[0][lane];
#pragma unroll
        for (int u = 1; u < kFnWarps; ++u) t.x += red[u][lane].x, t.y += red[u][lane].y;
        glob[lane] = make_float2(fn_gelu(__fdiv_rn(t.x, (float)HW)), fn_gelu(__fdiv_rn(t.y, (float)HW)));
    }
    __syncthreads();
    const float2 gl = glob[lane];
    const int64_t img = (int64_t)n * HW;
    for (int i = 0; i < R; ++i) {
        const int pix = (blockIdx.x * R + i) * kFnWarps + warp;
        if (pix >= HW) break;
        const float g = __ldg(gate + (img + pix) * ld_gate);
        float2 *ap = reinterpret_cast<float2 *>(ctx_all + (img + pix) * C + c);
        float2 a = *ap;
        a.x = __fadd_rn(a.x, __fmul_rn(gl.x, g)), a.y = __fadd_rn(a.y, __fmul_rn(gl.y, g));
        if (divisor != 0.f) a.x = __fdiv_rn(a.x, divisor), a.y = __fdiv_rn(a.y, divisor);
        *ap = a;
    }
}

// y = q * h over (rows, C), four channels per thread; q row r at r * ld_q, h and y contiguous, y may be h
__global__ void focal_modulate_kernel(const float *__restrict__ q, int64_t ld_q, const float *h, int64_t rows, int C, float *y) {
    const int c4 = C >> 2;
    const int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= rows * c4) return;
    const int64_t r = i / c4;
    const int c = (int)(i - r * c4) * 4;
    const float4 a = __ldg(reinterpret_cast<const float4 *>(q + r * ld_q + c));
    const float4 b = reinterpret_cast<const float4 *>(h)[i];
    reinterpret_cast<float4 *>(y)[i] = make_float4(__fmul_rn(a.x, b.x), __fmul_rn(a.y, b.y), __fmul_rn(a.z, b.z), __fmul_rn(a.w, b.w));
}

// one warp per row: t = t + gamma * LayerNorm(y), the LayerNorm of cn_layernorm_store, the product and the sum rounded on their own
__global__ void __launch_bounds__(32 * kFnWarps) layernorm_scale_add_kernel(const float *__restrict__ y, int64_t rows, int C,
                                                                             const float *__restrict__ g, const float *__restrict__ beta,
                                                                             float eps, const float *__restrict__ gamma,
                                                                             float *__restrict__ t) {
    const int lane = threadIdx.x & 31, nj = C >> 6;
    const int64_t tok = (int64_t)blockIdx.x * kFnWarps + (threadIdx.x >> 5);
    if (tok >= rows) return;
    const float *yr = y + tok * C + 2 * lane;
    float2 v[kFnLnMaxJ];
#pragma unroll
    for (int j = 0; j < kFnLnMaxJ; ++j) v[j] = j < nj ? fn_ldg2(yr + 64 * j) : make_float2(0.f, 0.f);
    float mean, rstd;
    cn_layernorm_stats(v, nj, C, eps, mean, rstd);
#pragma unroll
    for (int j = 0; j < kFnLnMaxJ; ++j)
        if (j < nj) {
            const int c = 64 * j + 2 * lane;
            const float2 gw = fn_ldg2(g + c), bw = fn_ldg2(beta + c), gm = fn_ldg2(gamma + c);
            float2 *tp = reinterpret_cast<float2 *>(t + tok * C + c);
            float2 tv = *tp;
            const float lx = (v[j].x - mean) * rstd * gw.x + bw.x, ly = (v[j].y - mean) * rstd * gw.y + bw.y;
            tv.x = __fadd_rn(tv.x, __fmul_rn(gm.x, lx)), tv.y = __fadd_rn(tv.y, __fmul_rn(gm.y, ly));
            *tp = tv;
        }
}

template <int K>
void fn_launch_level(bool last, dim3 grid, cudaStream_t s, const float *ctx, int64_t ld_ctx, const float *gate, int64_t ld_gate,
                     const float *w, int H, int W, int C, int R, int first, float *out, float *ctx_all, float *part) {
    if (last)
        focal_level_kernel<K, true><<<grid, 32 * kFnWarps, 0, s>>>(ctx, ld_ctx, gate, ld_gate, w, H, W, C, R, first, out, ctx_all, part);
    else
        focal_level_kernel<K, false><<<grid, 32 * kFnWarps, 0, s>>>(ctx, ld_ctx, gate, ld_gate, w, H, W, C, R, first, out, ctx_all,
                                                                    part);
}

}  // namespace sdetr

using namespace sdetr;

#define FN_CHECK_MAP(what)                                                                                                         \
    SDETR_REQUIRE(batch >= 0 && batch <= 65535 && H > 0 && W > 0 && (int64_t)H * W < (1LL << 31), SDETR_ERR_INVALID_ARG,          \
                  what ": bad sizes");                                                                                             \
    SDETR_REQUIRE(C > 0 && C % 64 == 0 && C <= 64 * kFnLnMaxJ, SDETR_ERR_UNSUPPORTED, what ": C=%d must be a multiple of 64 up to %d", \
                  C, 64 * kFnLnMaxJ)

extern "C" int sdetr_focalnet_stem(const float *x, int batch, int H, int W, int C, const float *weight, const float *bias,
                                   const float *ln_weight, const float *ln_bias, float eps, float *y, sdetr_stream_t stream) {
    SDETR_REQUIRE(x && weight && bias && ln_weight && ln_bias && y, SDETR_ERR_INVALID_ARG, "focalnet_stem: null pointer");
    SDETR_REQUIRE(batch >= 0 && H > 0 && W > 0 && eps >= 0.f, SDETR_ERR_INVALID_ARG, "focalnet_stem: bad sizes");
    SDETR_REQUIRE(C > 0 && C % 64 == 0 && C <= 64 * kStemMaxJ, SDETR_ERR_UNSUPPORTED, "focalnet_stem: C=%d must be a multiple of 64 up to %d",
                  C, 64 * kStemMaxJ);
    SDETR_REQUIRE(aligned16(weight) && aligned16(bias) && aligned16(ln_weight) && aligned16(ln_bias) && aligned16(y),
                  SDETR_ERR_INVALID_ARG, "focalnet_stem: weight, biases and y must be 16-byte aligned");
    const int Ho = (H + 3) / 4, Wo = (W + 3) / 4;
    const int64_t toks = (int64_t)batch * Ho * Wo;
    SDETR_REQUIRE((int64_t)batch * 3 * H * W < (1LL << 40) && toks < (1LL << 31), SDETR_ERR_INVALID_ARG, "focalnet_stem: image too large");
    if (toks == 0) return SDETR_OK;
    patch_stem_kernel<7, 2><<<(unsigned)((toks + kStemWarps - 1) / kStemWarps), 32 * kStemWarps, 0, (cudaStream_t)stream>>>(
        x, batch, H, W, Ho, Wo, C, weight, bias, ln_weight, ln_bias, eps, y);
    return check_launch("focalnet_stem");
}

extern "C" int64_t sdetr_focal_context_workspace_floats(int batch, int H, int W, int C) {
    if (batch < 0 || H <= 0 || W <= 0 || C <= 0) return 0;
    return (int64_t)batch * fn_tiles((int64_t)H * W) * C;
}

extern "C" int sdetr_focal_level_tokens(const float *ctx, int64_t ld_ctx, const float *gate, int64_t ld_gate, const float *weight,
                                        int ksize, int batch, int H, int W, int C, int first, float *out, float *ctx_all,
                                        float *partials, int64_t partials_floats, sdetr_stream_t stream) {
    SDETR_REQUIRE(ctx && gate && weight && ctx_all && (out || partials), SDETR_ERR_INVALID_ARG, "focal_level_tokens: null pointer");
    FN_CHECK_MAP("focal_level_tokens");
    SDETR_REQUIRE(ksize == 3 || ksize == 5 || ksize == 7 || ksize == 9, SDETR_ERR_UNSUPPORTED,
                  "focal_level_tokens: kernel size %d is not one of 3, 5, 7, 9", ksize);
    SDETR_REQUIRE(ld_ctx >= C && ld_ctx % 2 == 0 && ld_gate >= 1, SDETR_ERR_INVALID_ARG, "focal_level_tokens: bad row strides");
    SDETR_REQUIRE(((uintptr_t)ctx & 7u) == 0 && aligned16(weight) && aligned16(ctx_all) && (!out || aligned16(out)) &&
                      (!partials || aligned16(partials)),
                  SDETR_ERR_INVALID_ARG, "focal_level_tokens: operands must be aligned (ctx 8 bytes, the rest 16)");
    SDETR_REQUIRE(out != ctx && ctx_all != ctx && (!out || out != ctx_all), SDETR_ERR_INVALID_ARG,
                  "focal_level_tokens: out, ctx_all and ctx must not alias");
    SDETR_REQUIRE(!partials || partials_floats >= sdetr_focal_context_workspace_floats(batch, H, W, C), SDETR_ERR_WORKSPACE,
                  "focal_level_tokens: partials too small");
    SDETR_REQUIRE((int64_t)batch * H * W * (ld_ctx > C ? ld_ctx : C) < (1LL << 40), SDETR_ERR_INVALID_ARG, "focal_level_tokens: map too large");
    if (batch == 0) return SDETR_OK;
    const int64_t hw = (int64_t)H * W;
    const int R = fn_rows_per_warp(hw);
    const dim3 grid((unsigned)fn_tiles(hw), (unsigned)(C / 64), (unsigned)batch);
    const bool last = partials != nullptr;
    const cudaStream_t s = (cudaStream_t)stream;
    switch (ksize) {
        case 3: fn_launch_level<3>(last, grid, s, ctx, ld_ctx, gate, ld_gate, weight, H, W, C, R, first, out, ctx_all, partials); break;
        case 5: fn_launch_level<5>(last, grid, s, ctx, ld_ctx, gate, ld_gate, weight, H, W, C, R, first, out, ctx_all, partials); break;
        case 7: fn_launch_level<7>(last, grid, s, ctx, ld_ctx, gate, ld_gate, weight, H, W, C, R, first, out, ctx_all, partials); break;
        default: fn_launch_level<9>(last, grid, s, ctx, ld_ctx, gate, ld_gate, weight, H, W, C, R, first, out, ctx_all, partials); break;
    }
    return check_launch("focal_level_tokens");
}

extern "C" int sdetr_focal_global_context(const float *partials, int64_t partials_floats, const float *gate, int64_t ld_gate,
                                          int batch, int H, int W, int C, int focal_level, int normalize, float *ctx_all,
                                          sdetr_stream_t stream) {
    SDETR_REQUIRE(partials && gate && ctx_all, SDETR_ERR_INVALID_ARG, "focal_global_context: null pointer");
    FN_CHECK_MAP("focal_global_context");
    SDETR_REQUIRE(focal_level >= 1 && ld_gate >= 1, SDETR_ERR_INVALID_ARG, "focal_global_context: bad focal level or gate stride");
    SDETR_REQUIRE(aligned16(partials) && aligned16(ctx_all), SDETR_ERR_INVALID_ARG, "focal_global_context: operands must be 16-byte aligned");
    SDETR_REQUIRE(partials_floats >= sdetr_focal_context_workspace_floats(batch, H, W, C), SDETR_ERR_WORKSPACE,
                  "focal_global_context: partials too small");
    if (batch == 0) return SDETR_OK;
    const int64_t hw = (int64_t)H * W;
    const int tiles = fn_tiles(hw);
    const dim3 grid((unsigned)tiles, (unsigned)(C / 64), (unsigned)batch);
    focal_global_kernel<<<grid, 32 * kFnWarps, 0, (cudaStream_t)stream>>>(partials, tiles, gate, ld_gate, H, W, C, fn_rows_per_warp(hw),
                                                                          normalize ? (float)(focal_level + 1) : 0.f, ctx_all);
    return check_launch("focal_global_context");
}

extern "C" int sdetr_focal_modulate(const float *q, int64_t ld_q, const float *h, int64_t rows, int C, float *y, sdetr_stream_t stream) {
    SDETR_REQUIRE(q && h && y, SDETR_ERR_INVALID_ARG, "focal_modulate: null pointer");
    SDETR_REQUIRE(rows >= 0 && C > 0 && C % 4 == 0 && ld_q >= C && ld_q % 4 == 0, SDETR_ERR_INVALID_ARG, "focal_modulate: bad sizes");
    SDETR_REQUIRE(aligned16(q) && aligned16(h) && aligned16(y), SDETR_ERR_INVALID_ARG, "focal_modulate: operands must be 16-byte aligned");
    SDETR_REQUIRE(y != q, SDETR_ERR_INVALID_ARG, "focal_modulate: y must not alias q");
    const int64_t n = rows * (C / 4);
    SDETR_REQUIRE(n < (1LL << 40), SDETR_ERR_INVALID_ARG, "focal_modulate: too many rows");
    if (n == 0) return SDETR_OK;
    focal_modulate_kernel<<<(unsigned)((n + 255) / 256), 256, 0, (cudaStream_t)stream>>>(q, ld_q, h, rows, C, y);
    return check_launch("focal_modulate");
}

extern "C" int sdetr_layernorm_scale_add_tokens(const float *y, int64_t rows, int C, const float *ln_weight, const float *ln_bias,
                                                float eps, const float *gamma, float *t, sdetr_stream_t stream) {
    SDETR_REQUIRE(y && ln_weight && ln_bias && gamma && t, SDETR_ERR_INVALID_ARG, "layernorm_scale_add_tokens: null pointer");
    SDETR_REQUIRE(rows >= 0 && eps >= 0.f, SDETR_ERR_INVALID_ARG, "layernorm_scale_add_tokens: bad sizes");
    SDETR_REQUIRE(C > 0 && C % 64 == 0 && C <= 64 * kFnLnMaxJ, SDETR_ERR_UNSUPPORTED,
                  "layernorm_scale_add_tokens: C=%d must be a multiple of 64 up to %d", C, 64 * kFnLnMaxJ);
    SDETR_REQUIRE(y != t, SDETR_ERR_INVALID_ARG, "layernorm_scale_add_tokens: t must not alias y");
    SDETR_REQUIRE(aligned16(y) && aligned16(ln_weight) && aligned16(ln_bias) && aligned16(gamma) && aligned16(t), SDETR_ERR_INVALID_ARG,
                  "layernorm_scale_add_tokens: operands must be 16-byte aligned");
    SDETR_REQUIRE(rows < (1LL << 36), SDETR_ERR_INVALID_ARG, "layernorm_scale_add_tokens: too many rows");
    if (rows == 0) return SDETR_OK;
    layernorm_scale_add_kernel<<<(unsigned)((rows + kFnWarps - 1) / kFnWarps), 32 * kFnWarps, 0, (cudaStream_t)stream>>>(
        y, rows, C, ln_weight, ln_bias, eps, gamma, t);
    return check_launch("layernorm_scale_add_tokens");
}
