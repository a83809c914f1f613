// Encoder FFN -- sdetr_ffn_fused_layernorm:   y = LayerNorm(x + linear2(ReLU(linear1(x))))
// (reference models/bricks/salience_transformer.py:347-351 `forward_ffn` + :391 `norm2`; C = 256, any hidden width % 128 == 0).
//
// Three launches on the 3xFP16 wgmma kernel of wgmma.cuh (same error-compensated products, scalings and accumulation as
// sdetr_gemm_f16x3_pre, fp32-class accuracy):
//   H = x W1^T + b1                       (M, hidden) fp32 in the workspace
//   P = ReLU(H) W2^T + b2                 the ReLU is fused into the second GEMM's operand load; P goes to the workspace, or
//                                         straight to y without LayerNorm
//   y = LayerNorm(x + P) * gamma + beta   ffn_finish_kernel, one warp per row (x may alias y).
// Deterministic: no atomics, a fixed reduction order per row.
#include "wgmma.cuh"

namespace sdetr {

constexpr int kFD = 256;  // model width: K of linear1, N of linear2

__global__ void __launch_bounds__(256) ffn_finish_kernel(const float *x /* may alias y */, int64_t ldx, const float *__restrict__ partial,
                                                         const float *__restrict__ gamma, const float *__restrict__ beta, float eps,
                                                         int64_t rows, float *y) {
    const int lane = threadIdx.x & 31;
    const int64_t row = (int64_t)blockIdx.x * 8 + (threadIdx.x >> 5);
    if (row >= rows) return;
    float4 v[2];
    float s = 0.f;
#pragma unroll
    for (int i = 0; i < 2; ++i) {
        const int c = i * 128 + lane * 4;
        const float4 a = ld_stream_f4(partial + row * kFD + c), r = *reinterpret_cast<const float4 *>(x + row * ldx + c);
        v[i] = make_float4(r.x + a.x, r.y + a.y, r.z + a.z, r.w + a.w);
        s += (v[i].x + v[i].y) + (v[i].z + v[i].w);
    }
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) s += __shfl_xor_sync(0xffffffffu, s, o);
    const float mean = s / (float)kFD;
    float ss = 0.f;
#pragma unroll
    for (int i = 0; i < 2; ++i) {
        const float dx = v[i].x - mean, dy = v[i].y - mean, dz = v[i].z - mean, dw = v[i].w - mean;
        ss += (dx * dx + dy * dy) + (dz * dz + dw * dw);
    }
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) ss += __shfl_xor_sync(0xffffffffu, ss, o);
    const float rstd = rsqrtf(ss / (float)kFD + eps);
#pragma unroll
    for (int i = 0; i < 2; ++i) {
        const int c = i * 128 + lane * 4;
        const float4 g = ldg_f4(gamma + c), bt = ldg_f4(beta + c);
        float4 o;
        o.x = (v[i].x - mean) * rstd * g.x + bt.x, o.y = (v[i].y - mean) * rstd * g.y + bt.y;
        o.z = (v[i].z - mean) * rstd * g.z + bt.z, o.w = (v[i].w - mean) * rstd * g.w + bt.w;
        *reinterpret_cast<float4 *>(y + row * kFD + c) = o;
    }
}

}  // namespace sdetr

using namespace sdetr;

extern "C" int64_t sdetr_ffn_fused_workspace_floats(int M, int hidden) {
    if (M <= 0 || hidden <= 0 || hidden % 128) return 0;
    return (int64_t)M * (hidden + kFD);  // H, then P
}

extern "C" int sdetr_ffn_fused_layernorm(const float *x, int64_t ldx, const void *w1_hi, const void *w1_lo, float w1_scale,
                                         const float *b1, const void *w2_hi, const void *w2_lo, float w2_scale, const float *b2,
                                         const float *gamma, const float *beta, float eps, int M, int hidden, float *workspace,
                                         int64_t workspace_floats, float *y, sdetr_stream_t stream) {
    SDETR_REQUIRE(x && w1_hi && w1_lo && w2_hi && w2_lo && b1 && workspace && y, SDETR_ERR_INVALID_ARG, "ffn_fused: null pointer");
    SDETR_REQUIRE((gamma == nullptr) == (beta == nullptr), SDETR_ERR_INVALID_ARG, "ffn_fused: gamma and beta go together");
    SDETR_REQUIRE(M >= 0 && hidden > 0 && hidden % 128 == 0, SDETR_ERR_UNSUPPORTED, "ffn_fused: hidden=%d must be a multiple of 128", hidden);
    SDETR_REQUIRE(w1_scale > 0.f && w2_scale > 0.f, SDETR_ERR_INVALID_ARG, "ffn_fused: weight scales must be positive");
    SDETR_REQUIRE(ldx % 4 == 0 && ldx >= kFD && aligned16(x) && aligned16(w1_hi) && aligned16(w1_lo) && aligned16(w2_hi) &&
                      aligned16(w2_lo) && aligned16(workspace) && aligned16(y),
                  SDETR_ERR_INVALID_ARG, "ffn_fused: operands must be 16-byte aligned with a 16-byte row pitch");
    if (M == 0) return SDETR_OK;
    SDETR_REQUIRE(workspace_floats >= (int64_t)M * (hidden + kFD), SDETR_ERR_INVALID_ARG,
                  "ffn_fused: workspace of %lld floats is smaller than sdetr_ffn_fused_workspace_floats", (long long)workspace_floats);
    CUtensorMap m1h, m1l, m2h, m2l;
    SDETR_REQUIRE(make_map_2d(&m1h, CU_TENSOR_MAP_DATA_TYPE_FLOAT16, 2, w1_hi, hidden, kFD, kFD, 64, kGN) &&
                      make_map_2d(&m1l, CU_TENSOR_MAP_DATA_TYPE_FLOAT16, 2, w1_lo, hidden, kFD, kFD, 64, kGN) &&
                      make_map_2d(&m2h, CU_TENSOR_MAP_DATA_TYPE_FLOAT16, 2, w2_hi, kFD, hidden, hidden, 64, kGN) &&
                      make_map_2d(&m2l, CU_TENSOR_MAP_DATA_TYPE_FLOAT16, 2, w2_lo, kFD, hidden, hidden, 64, kGN),
                  SDETR_ERR_CUDA, "ffn_fused: cuTensorMapEncodeTiled failed");
    float *h = workspace, *part = gamma ? workspace + (int64_t)M * hidden : y;
    const Gemm3xParams p1{b1, h, hidden, M, hidden, kFD, 0, kActScale, 1.f / (kActScale * w1_scale), nullptr, nullptr};
    int rc = launch_gemm3x<true, false>(x, ldx, m1h, m1l, p1, stream, "ffn_fused/linear1");
    if (rc != SDETR_OK) return rc;
    const Gemm3xParams p2{b2, part, kFD, M, kFD, hidden, 1, kActScale, 1.f / (kActScale * w2_scale), nullptr, nullptr};
    rc = launch_gemm3x<true, false>(h, hidden, m2h, m2l, p2, stream, "ffn_fused/linear2");
    if (rc != SDETR_OK || !gamma) return rc;
    ffn_finish_kernel<<<(unsigned)((M + 7) / 8), 256, 0, (cudaStream_t)stream>>>(x, ldx, part, gamma, beta, eps, M, y);
    return check_launch("ffn_fused/finish");
}
