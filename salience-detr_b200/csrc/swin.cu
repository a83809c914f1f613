// Swin Transformer backbone in token layout (SwinTransformerBackbone.forward_tokens): the kernels around the Linears.  Every
// Linear of a block and each PatchMerging reduction runs on sdetr_gemm_f16x3_ex (gemm_f16x3.cu), the stem on
// sdetr_convnext_stem (convnext.cu).
//
//   sdetr_window_attention_tokens        shifted-window multi-head attention of V1 Swin from the QKV projection's output:
//                                        padding, cyclic shift, window partition and reverse in index arithmetic, relative
//                                        position bias and the shift mask; fp32 FMAs, one CTA per (window, head).
//   sdetr_patch_merge_layernorm_tokens   the 2x2 space-to-depth concatenation of PatchMerging with its LayerNorm over 4 C.
//   sdetr_layernorm_tokens               LayerNorm over C of contiguous token rows, C up to 1536.
//
// Both LayerNorms are the one-warp-per-row two-pass LayerNorm of layernorm_rows.cuh.
#include <math.h>

#include "common.cuh"
#include "layernorm_rows.cuh"

namespace sdetr {

constexpr int kSwWarps = 8;        // warps per CTA of 256 threads
constexpr int kSwHd = 32;          // head dim (every Swin arch): one lane per channel of a head
constexpr int kSwMaxN = 144;       // tokens per window (12 x 12)
constexpr int kSwLnMaxJ = 24;      // sdetr_layernorm_tokens: C <= 64 * 24 = 1536
constexpr int kSwMergeMaxJ = 48;   // sdetr_patch_merge_layernorm_tokens: 4 C <= 64 * 48 = 3072

// One CTA per (image, window, head).  Window token t sits at (r, c) = (wy * wh + t / ww, wx * ww + t % ww) of the rolled,
// padded frame and reads the source pixel ((r + sh) mod pad_H, (c + sw) mod pad_W); a source outside the H x W map is a pad
// token, a zero row after norm1, whose key and value are the qkv bias.  K and V of the window go to shared memory, then one
// warp per query row: lanes over keys for the logits (q * hd^-0.5) . k + bias[h, i, j] + mask, warp max and sum, p = e / sum,
// then lane = channel for p . V.  mask is -100 where the region ids of i and j differ (0 without a shift), added and kept in
// the softmax as in the reference.  Pad queries are not computed: their outputs are dropped.
__global__ void __launch_bounds__(32 * kSwWarps) window_attention_kernel(const float *__restrict__ qkv,
                                                                          const float *__restrict__ qkv_bias,
                                                                          const float *__restrict__ rel_bias, int H, int W, int C,
                                                                          int wh, int ww, int sh, int sw, int pad_H, int pad_W,
                                                                          int nwx, int nwin, float *__restrict__ y) {
    __shared__ float ks[kSwMaxN * (kSwHd + 1)];  // padded rows: lanes reading 32 different keys hit 32 banks
    __shared__ float vs[kSwMaxN * kSwHd];
    __shared__ float qs[kSwWarps][kSwHd];
    __shared__ float ps[kSwWarps][kSwMaxN];
    __shared__ int src[kSwMaxN];   // source pixel of each window token, -1 for a pad token
    __shared__ int reg[kSwMaxN];   // region id of each window token
    const int n = blockIdx.x / nwin, win = blockIdx.x - n * nwin, wy = win / nwx, wx = win - wy * nwx, h = blockIdx.y;
    const int N = wh * ww, lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    const int64_t ld = 3LL * C;
    const float *base = qkv + (int64_t)n * H * W * ld;
    for (int t = threadIdx.x; t < N; t += blockDim.x) {
        const int r = wy * wh + t / ww, c = wx * ww + t % ww;
        int sr = r + sh, sc = c + sw;
        sr -= sr >= pad_H ? pad_H : 0;
        sc -= sc >= pad_W ? pad_W : 0;
        src[t] = (sr < H && sc < W) ? sr * W + sc : -1;
        const int rh = r < pad_H - wh ? 0 : (r < pad_H - sh ? 1 : 2), rw = c < pad_W - ww ? 0 : (c < pad_W - sw ? 1 : 2);
        reg[t] = 3 * rh + rw;
    }
    __syncthreads();
    for (int e = threadIdx.x; e < N * kSwHd; e += blockDim.x) {
        const int t = e >> 5, d = e & 31, s = src[t];
        const int kc = C + h * kSwHd + d, vc = 2 * C + h * kSwHd + d;
        const float *row = s >= 0 ? base + (int64_t)s * ld : qkv_bias;
        ks[t * (kSwHd + 1) + d] = __ldg(row + kc);
        vs[t * kSwHd + d] = __ldg(row + vc);
    }
    __syncthreads();
    const float scale = 0.17677669529663687f;  // 32^-0.5
    const float *bias_h = rel_bias + (int64_t)h * N * N;
    for (int i = warp; i < N; i += kSwWarps) {
        const int si = src[i];
        if (si < 0) continue;
        qs[warp][lane] = __ldg(base + (int64_t)si * ld + h * kSwHd + lane) * scale;
        __syncwarp();
        const int ri = reg[i];
        float l[kSwMaxN / 32 + 1];
        float mx = -INFINITY;
#pragma unroll
        for (int u = 0; u < kSwMaxN / 32 + 1; ++u) {
            const int j = lane + 32 * u;
            l[u] = -INFINITY;
            if (j < N) {
                const float *kr = ks + j * (kSwHd + 1);
                float a = 0.f;
#pragma unroll
                for (int d = 0; d < kSwHd; ++d) a = fmaf(qs[warp][d], kr[d], a);
                a += __ldg(bias_h + i * N + j);
                a += reg[j] == ri ? 0.f : -100.f;
                l[u] = a;
                mx = fmaxf(mx, a);
            }
        }
#pragma unroll
        for (int o = 16; o > 0; o >>= 1) mx = fmaxf(mx, __shfl_xor_sync(0xffffffffu, mx, o));
        float sum = 0.f;
#pragma unroll
        for (int u = 0; u < kSwMaxN / 32 + 1; ++u)
            if (lane + 32 * u < N) {
                l[u] = expf(l[u] - mx);
                sum += l[u];
            }
        sum = cn_warp_sum(sum);
#pragma unroll
        for (int u = 0; u < kSwMaxN / 32 + 1; ++u)
            if (lane + 32 * u < N) ps[warp][lane + 32 * u] = l[u] / sum;
        __syncwarp();
        float o = 0.f;
        for (int j = 0; j < N; ++j) o = fmaf(ps[warp][j], vs[j * kSwHd + lane], o);
        y[((int64_t)n * H * W + si) * C + h * kSwHd + lane] = o;
        __syncwarp();  // qs and ps are rewritten by the warp's next row
    }
}

// one warp per output row (oy, ox): columns (2 dx + dy) C + c hold x(2 oy + dy, 2 ox + dx, c), zero outside the map
__global__ void __launch_bounds__(32 * kSwWarps) patch_merge_layernorm_kernel(const float *__restrict__ x, int batch, int H, int W,
                                                                               int C, int Ho, int Wo, const float *__restrict__ g,
                                                                               const float *__restrict__ beta, float eps,
                                                                               float *__restrict__ y) {
    const int lane = threadIdx.x & 31, nj = C >> 4;  // 4 C / 64
    const int64_t tok = (int64_t)blockIdx.x * kSwWarps + (threadIdx.x >> 5), hwo = (int64_t)Ho * Wo;
    if (tok >= batch * hwo) return;
    const int n = (int)(tok / hwo), pix = (int)(tok - n * hwo), oy = pix / Wo, ox = pix - oy * Wo;
    const float *xn = x + (int64_t)n * H * W * C;
    float2 v[kSwMergeMaxJ];
#pragma unroll
    for (int j = 0; j < kSwMergeMaxJ; ++j) {
        v[j] = make_float2(0.f, 0.f);
        if (j < nj) {
            const int col = 64 * j + 2 * lane, q = col / C, c = col - q * C;
            const int iy = 2 * oy + (q & 1), ix = 2 * ox + (q >> 1);
            if (iy < H && ix < W) v[j] = __ldg(reinterpret_cast<const float2 *>(xn + ((int64_t)iy * W + ix) * C + c));
        }
    }
    cn_layernorm_store(v, nj, 4 * C, lane, g, beta, eps, y + tok * 4 * C);
}

__global__ void __launch_bounds__(32 * kSwWarps) layernorm_rows_kernel(const float *__restrict__ x, int64_t rows, int C,
                                                                        const float *__restrict__ g, const float *__restrict__ beta,
                                                                        float eps, float *__restrict__ y) {
    const int lane = threadIdx.x & 31, nj = C >> 6;
    const int64_t tok = (int64_t)blockIdx.x * kSwWarps + (threadIdx.x >> 5);
    if (tok >= rows) return;
    const float *xr = x + tok * C + 2 * lane;
    float2 v[kSwLnMaxJ];
#pragma unroll
    for (int j = 0; j < kSwLnMaxJ; ++j) v[j] = j < nj ? __ldg(reinterpret_cast<const float2 *>(xr + 64 * j)) : make_float2(0.f, 0.f);
    cn_layernorm_store(v, nj, C, lane, g, beta, eps, y + tok * C);
}

inline unsigned sw_blocks(int64_t warps) { return (unsigned)((warps + kSwWarps - 1) / kSwWarps); }

}  // namespace sdetr

using namespace sdetr;

extern "C" int sdetr_window_attention_tokens(const float *qkv, const float *qkv_bias, const float *rel_bias, int batch, int H, int W,
                                             int C, int num_heads, int window_h, int window_w, int shift_h, int shift_w, float *y,
                                             sdetr_stream_t stream) {
    SDETR_REQUIRE(qkv && qkv_bias && rel_bias && y, SDETR_ERR_INVALID_ARG, "window_attention_tokens: null pointer");
    SDETR_REQUIRE(batch >= 0 && H > 0 && W > 0 && num_heads > 0 && window_h > 0 && window_w > 0, SDETR_ERR_INVALID_ARG,
                  "window_attention_tokens: bad sizes");
    SDETR_REQUIRE(C == kSwHd * num_heads, SDETR_ERR_UNSUPPORTED, "window_attention_tokens: C=%d must be %d * num_heads (%d)", C,
                  kSwHd, num_heads);
    SDETR_REQUIRE(window_h * window_w <= kSwMaxN, SDETR_ERR_UNSUPPORTED, "window_attention_tokens: window %dx%d over %d tokens",
                  window_h, window_w, kSwMaxN);
    SDETR_REQUIRE(shift_h >= 0 && shift_h < window_h && shift_w >= 0 && shift_w < window_w, SDETR_ERR_UNSUPPORTED,
                  "window_attention_tokens: shift (%d, %d) outside [0, window)", shift_h, shift_w);
    SDETR_REQUIRE(y != qkv, SDETR_ERR_INVALID_ARG, "window_attention_tokens: y must not alias qkv");
    SDETR_REQUIRE((int64_t)H * W < (1LL << 31) && (int64_t)batch * H * W * 3 * C < (1LL << 40), SDETR_ERR_INVALID_ARG,
                  "window_attention_tokens: map too large");
    // the reference's rules: pad to whole windows, no shift in a dimension the window covers
    const int pad_H = (H + window_h - 1) / window_h * window_h, pad_W = (W + window_w - 1) / window_w * window_w;
    if (window_h >= pad_H) shift_h = 0;
    if (window_w >= pad_W) shift_w = 0;
    const int nwx = pad_W / window_w, nwin = (pad_H / window_h) * nwx;
    SDETR_REQUIRE((int64_t)batch * nwin < (1LL << 31) && num_heads <= 65535, SDETR_ERR_INVALID_ARG,
                  "window_attention_tokens: too many windows");
    if (batch == 0) return SDETR_OK;
    const dim3 grid((unsigned)(batch * nwin), (unsigned)num_heads);
    window_attention_kernel<<<grid, 32 * kSwWarps, 0, (cudaStream_t)stream>>>(qkv, qkv_bias, rel_bias, H, W, C, window_h, window_w,
                                                                              shift_h, shift_w, pad_H, pad_W, nwx, nwin, y);
    return check_launch("window_attention_tokens");
}

extern "C" int sdetr_patch_merge_layernorm_tokens(const float *x, int batch, int H, int W, int C, const float *ln_weight,
                                                  const float *ln_bias, float eps, float *y, sdetr_stream_t stream) {
    SDETR_REQUIRE(x && ln_weight && ln_bias && y, SDETR_ERR_INVALID_ARG, "patch_merge_layernorm_tokens: null pointer");
    SDETR_REQUIRE(batch >= 0 && H > 0 && W > 0 && eps >= 0.f, SDETR_ERR_INVALID_ARG, "patch_merge_layernorm_tokens: bad sizes");
    SDETR_REQUIRE(C > 0 && C % 16 == 0 && 4 * C <= 64 * kSwMergeMaxJ, SDETR_ERR_UNSUPPORTED,
                  "patch_merge_layernorm_tokens: C=%d must be a multiple of 16 up to %d", C, 16 * kSwMergeMaxJ);
    SDETR_REQUIRE(x != y, SDETR_ERR_INVALID_ARG, "patch_merge_layernorm_tokens: y must not alias x");
    SDETR_REQUIRE(aligned16(x) && aligned16(ln_weight) && aligned16(ln_bias) && aligned16(y), SDETR_ERR_INVALID_ARG,
                  "patch_merge_layernorm_tokens: operands must be 16-byte aligned");
    const int Ho = (H + 1) / 2, Wo = (W + 1) / 2;
    const int64_t toks = (int64_t)batch * Ho * Wo;
    SDETR_REQUIRE(toks < (1LL << 31) && (int64_t)batch * H * W * C < (1LL << 40), SDETR_ERR_INVALID_ARG,
                  "patch_merge_layernorm_tokens: map too large");
    if (toks == 0) return SDETR_OK;
    patch_merge_layernorm_kernel<<<sw_blocks(toks), 32 * kSwWarps, 0, (cudaStream_t)stream>>>(x, batch, H, W, C, Ho, Wo, ln_weight,
                                                                                               ln_bias, eps, y);
    return check_launch("patch_merge_layernorm_tokens");
}

extern "C" int sdetr_layernorm_tokens(const float *x, int64_t rows, int C, const float *ln_weight, const float *ln_bias, float eps,
                                      float *y, sdetr_stream_t stream) {
    SDETR_REQUIRE(x && ln_weight && ln_bias && y, SDETR_ERR_INVALID_ARG, "layernorm_tokens: null pointer");
    SDETR_REQUIRE(rows >= 0 && eps >= 0.f, SDETR_ERR_INVALID_ARG, "layernorm_tokens: bad sizes");
    SDETR_REQUIRE(C > 0 && C % 64 == 0 && C <= 64 * kSwLnMaxJ, SDETR_ERR_UNSUPPORTED,
                  "layernorm_tokens: C=%d must be a multiple of 64 up to %d", C, 64 * kSwLnMaxJ);
    SDETR_REQUIRE(x != y, SDETR_ERR_INVALID_ARG, "layernorm_tokens: y must not alias x");
    SDETR_REQUIRE(aligned16(x) && aligned16(ln_weight) && aligned16(ln_bias) && aligned16(y), SDETR_ERR_INVALID_ARG,
                  "layernorm_tokens: operands must be 16-byte aligned");
    SDETR_REQUIRE(rows < (1LL << 36), SDETR_ERR_INVALID_ARG, "layernorm_tokens: too many rows");
    if (rows == 0) return SDETR_OK;
    layernorm_rows_kernel<<<sw_blocks(rows), 32 * kSwWarps, 0, (cudaStream_t)stream>>>(x, rows, C, ln_weight, ln_bias, eps, y);
    return check_launch("layernorm_tokens");
}
