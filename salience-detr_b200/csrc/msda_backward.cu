// MSDA core backward for sm_90a -- sdetr_msda_backward.
//
// Reference semantics: models/bricks/ops/cuda/ms_deform_im2col_cuda.cuh:76-148 (bilinear backward helper)
// and :290-392 (the kernel variant selected at head_dim 32, `case 32` :1129-1150), host wrapper
// ms_deform_attn_cuda.cu:75-145.
//
// Design: as in the forward, a group of D/4 lanes owns one (image, query, head) and keeps the 128-bit
// row layout.  Per sampling point the group
//   * re-reads the four corner rows (128-bit loads),
//   * adds  w_corner * attn * grad_out  into grad_value with ONE vector red.global.add.v4.f32 per lane and
//     corner (the reference issues four scalar atomicAdds per thread),
//   * reduces  d/d(attn)  and  d/d(loc)  over the head dimension with warp shuffles (the reference stages
//     them in shared memory and lets thread 0 add them up serially, .cuh:366-382).
#include "common.cuh"

namespace sdetr {

constexpr int kBwdThreads = 256;

struct MsdaBwdParams {
    const float *value;
    const int64_t *shapes, *lsi;
    const float *loc, *attn, *gout;
    float *gvalue, *gloc, *gattn;
    int batch, nv, heads, nq, L, P;
};

__device__ __forceinline__ float dot4(const float4 &a, const float4 &b) {
    return fmaf(a.x, b.x, fmaf(a.y, b.y, fmaf(a.z, b.z, a.w * b.w)));
}
__device__ __forceinline__ void red_add_f4(float *p, float s, const float4 &g) {
    atomicAdd(reinterpret_cast<float4 *>(p), make_float4(s * g.x, s * g.y, s * g.z, s * g.w));  // red.global.add.v4.f32
}

template <int D>
__global__ void __launch_bounds__(kBwdThreads) msda_bwd_kernel(const MsdaBwdParams p) {
    constexpr int LANES = D / 4;
    constexpr int GROUPS = kBwdThreads / LANES;
    const int lane = threadIdx.x % LANES;
    int64_t item = (int64_t)blockIdx.x * GROUPS + threadIdx.x / LANES;
    const bool active = item < (int64_t)p.batch * p.nq * p.heads;
    if (!active) item = 0;  // keep every lane in the shuffles
    const int m = (int)(item % p.heads);
    const int64_t row = item / p.heads;  // (image, query)
    const int b = (int)(row / p.nq);
    const int NP = p.L * p.P;
    const float4 go = ldg_f4(p.gout + item * D + lane * 4);
    const int64_t vimg = (int64_t)b * p.nv * p.heads * D;
    for (int l = 0; l < p.L; ++l) {
        const int H = (int)__ldg(p.shapes + 2 * l), W = (int)__ldg(p.shapes + 2 * l + 1);
        const float Hf = (float)H, Wf = (float)W;
        const int64_t lvl = vimg + __ldg(p.lsi + l) * p.heads * D + (int64_t)m * D + lane * 4;
        for (int pt = 0; pt < p.P; ++pt) {
            const int64_t k = item * NP + l * p.P + pt;
            const float x = __ldg(p.loc + 2 * k), y = __ldg(p.loc + 2 * k + 1), a = __ldg(p.attn + k);
            const float h_im = fmaf(y, Hf, -0.5f), w_im = fmaf(x, Wf, -0.5f);
            const bool in = h_im > -1.f && w_im > -1.f && h_im < Hf && w_im < Wf;
            float g_a = 0.f, g_x = 0.f, g_y = 0.f;
            if (in) {  // group-uniform branch
                const float hf = floorf(h_im), wf = floorf(w_im);
                const int y0 = (int)hf, x0 = (int)wf;
                const float ly = h_im - hf, lx = w_im - wf, hy = 1.f - ly, hx = 1.f - lx;
                const bool top = y0 >= 0, bot = y0 + 1 <= H - 1, lef = x0 >= 0, rig = x0 + 1 <= W - 1;
                const int64_t o00 = lvl + (int64_t)(y0 * W + x0) * p.heads * D;
                const int64_t o01 = o00 + (int64_t)p.heads * D, o10 = o00 + (int64_t)W * p.heads * D;
                const int64_t o11 = o10 + (int64_t)p.heads * D;
                const float4 z = make_float4(0.f, 0.f, 0.f, 0.f);
                const float4 v00 = (top && lef) ? ldg_f4(p.value + o00) : z;
                const float4 v01 = (top && rig) ? ldg_f4(p.value + o01) : z;
                const float4 v10 = (bot && lef) ? ldg_f4(p.value + o10) : z;
                const float4 v11 = (bot && rig) ? ldg_f4(p.value + o11) : z;
                const float d00 = dot4(go, v00), d01 = dot4(go, v01), d10 = dot4(go, v10), d11 = dot4(go, v11);
                g_a = hy * hx * d00 + hy * lx * d01 + ly * hx * d10 + ly * lx * d11;       // .cuh:145
                g_x = Wf * a * (-hy * d00 + hy * d01 - ly * d10 + ly * d11);               // .cuh:146 (grad_w_weight)
                g_y = Hf * a * (-hx * d00 - lx * d01 + hx * d10 + lx * d11);               // .cuh:147 (grad_h_weight)
                if (active) {
                    if (top && lef) red_add_f4(p.gvalue + o00, hy * hx * a, go);
                    if (top && rig) red_add_f4(p.gvalue + o01, hy * lx * a, go);
                    if (bot && lef) red_add_f4(p.gvalue + o10, ly * hx * a, go);
                    if (bot && rig) red_add_f4(p.gvalue + o11, ly * lx * a, go);
                }
            }
#pragma unroll
            for (int o = LANES / 2; o > 0; o >>= 1) {
                g_a += __shfl_xor_sync(0xffffffffu, g_a, o, LANES);
                g_x += __shfl_xor_sync(0xffffffffu, g_x, o, LANES);
                g_y += __shfl_xor_sync(0xffffffffu, g_y, o, LANES);
            }
            if (active && lane == 0) {
                p.gattn[k] = g_a;
                *reinterpret_cast<float2 *>(p.gloc + 2 * k) = make_float2(g_x, g_y);
            }
        }
    }
}

}  // namespace sdetr

using namespace sdetr;

extern "C" int sdetr_msda_backward(const float *value, const int64_t *spatial_shapes, const int64_t *level_start_index,
                                   const float *sampling_loc, const float *attn_weight, const float *grad_output,
                                   float *grad_value, float *grad_sampling_loc, float *grad_attn_weight, int batch,
                                   int num_value, int num_heads, int head_dim, int num_levels, int num_query,
                                   int num_points, sdetr_stream_t stream) {
    SDETR_REQUIRE(value && spatial_shapes && level_start_index && sampling_loc && attn_weight && grad_output &&
                      grad_value && grad_sampling_loc && grad_attn_weight,
                  SDETR_ERR_INVALID_ARG, "msda_backward: null pointer");
    SDETR_REQUIRE(batch > 0 && num_value > 0 && num_heads > 0 && num_levels > 0 && num_points > 0 && num_query >= 0,
                  SDETR_ERR_INVALID_ARG, "msda_backward: non-positive size");
    SDETR_REQUIRE(num_levels <= kMaxLevels, SDETR_ERR_UNSUPPORTED, "msda_backward: more than %d levels", kMaxLevels);
    SDETR_REQUIRE(aligned16(value) && aligned16(grad_output) && aligned16(grad_value) &&
                      (reinterpret_cast<uintptr_t>(grad_sampling_loc) & 7u) == 0,
                  SDETR_ERR_INVALID_ARG, "msda_backward: 16-byte alignment required");
    cudaStream_t s = (cudaStream_t)stream;
    cudaError_t e = cudaMemsetAsync(grad_value, 0, sizeof(float) * (size_t)batch * num_value * num_heads * head_dim, s);
    SDETR_REQUIRE(e == cudaSuccess, SDETR_ERR_CUDA, "msda_backward: memset: %s", cudaGetErrorString(e));
    if (num_query == 0) return SDETR_OK;
    MsdaBwdParams p{value, spatial_shapes, level_start_index, sampling_loc, attn_weight, grad_output,
                    grad_value, grad_sampling_loc, grad_attn_weight, batch, num_value, num_heads, num_query,
                    num_levels, num_points};
    const int64_t items = (int64_t)batch * num_query * num_heads;
#define SDETR_BWD(DD)                                                                                       \
    case DD: {                                                                                              \
        constexpr int G = kBwdThreads / (DD / 4);                                                           \
        msda_bwd_kernel<DD><<<(unsigned)((items + G - 1) / G), kBwdThreads, 0, s>>>(p);                      \
    } break;
    switch (head_dim) {
        SDETR_BWD(4) SDETR_BWD(8) SDETR_BWD(16) SDETR_BWD(32) SDETR_BWD(64) SDETR_BWD(128)
        default:
            SDETR_REQUIRE(false, SDETR_ERR_UNSUPPORTED, "msda_backward: head_dim %d not in {4,8,16,32,64,128}", head_dim);
    }
#undef SDETR_BWD
    return check_launch("msda_backward");
}
