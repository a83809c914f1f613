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
//
// Deterministic variant (sdetr_msda_backward_deterministic, template flag DET): the same kernel, but each corner
// contribution  (w_corner * attn) * grad_out  is multiplied by an exact power of two 2^s, rounded to int64 and added into an
// int64 accumulator with red.global.add.u64.  Integer addition is associative, so the sums do not depend on the order of the
// additions (launch order, grid, query order).  s is computed on the device (msda_det_scale_kernel) so that
//     max|grad_out| * max|attn| * num_query * num_points * 2^s <= 2^62:
// a value element belongs to one level and one image, and per query it receives at most P corner weights <= 1, so no sum
// can overflow.  A last elementwise pass (msda_det_finalize_kernel) writes grad_value = float(acc) * 2^-s, or NaN everywhere
// when grad_out or attn held a non-finite value.  grad_loc / grad_attn are computed by the same code as the atomic kernel.
#include "common.cuh"

namespace sdetr {

constexpr int kBwdThreads = 256;

// device state of the deterministic variant, at the end of its workspace (zeroed by every call)
struct MsdaDetState {
    unsigned int max_gout, max_attn;  // bit patterns of max|grad_out|, max|attn| (non-negative floats order like their bits)
    unsigned int nonfinite;           // grad_out or attn held a NaN / inf
    unsigned int blocks_done;
    int shift;                        // s of the scale 2^s
    int pad[3];
};

struct MsdaBwdParams {
    const float *value;
    const int64_t *shapes, *lsi;
    const float *loc, *attn, *gout;
    float *gvalue, *gloc, *gattn;
    int batch, nv, heads, nq, L, P;
    long long *gacc;                  // DET: int64 accumulator of grad_value * 2^s (b,Nv,M,D)
    const MsdaDetState *det;          // DET: the scale
};

__device__ __forceinline__ float dot4(const float4 &a, const float4 &b) {
    return fmaf(a.x, b.x, fmaf(a.y, b.y, fmaf(a.z, b.z, a.w * b.w)));
}
__device__ __forceinline__ void red_add_f4(float *p, float s, const float4 &g) {
    atomicAdd(reinterpret_cast<float4 *>(p), make_float4(s * g.x, s * g.y, s * g.z, s * g.w));  // red.global.add.v4.f32
}
// The same products s * g, scaled by 2^shift (exact in double), rounded to nearest and added as int64 (red.global.add.u64).
// g holds the row elements lane, lane + LANES, lane + 2 LANES, lane + 3 LANES (p points at element `lane`): each of the four
// reductions of a lane group then covers one contiguous run of LANES * 8 bytes.
template <int LANES>
__device__ __forceinline__ void red_add_i64x4(long long *p, float s, const float4 &g, double scale) {
    unsigned long long *q = reinterpret_cast<unsigned long long *>(p);
    atomicAdd(q + 0 * LANES, (unsigned long long)__double2ll_rn((double)(s * g.x) * scale));
    atomicAdd(q + 1 * LANES, (unsigned long long)__double2ll_rn((double)(s * g.y) * scale));
    atomicAdd(q + 2 * LANES, (unsigned long long)__double2ll_rn((double)(s * g.z) * scale));
    atomicAdd(q + 3 * LANES, (unsigned long long)__double2ll_rn((double)(s * g.w) * scale));
}

// max|grad_out|, max|attn| and the non-finite flag in one launch; the last block to finish derives s
__global__ void __launch_bounds__(256) msda_det_scale_kernel(const float *__restrict__ gout, int64_t n_gout,
                                                             const float *__restrict__ attn, int64_t n_attn,
                                                             int64_t contributions /* num_query * num_points */,
                                                             MsdaDetState *__restrict__ st) {
    bool bad = false;
    const float mg = block_max(thread_absmax(gout, n_gout, bad));
    const float ma = block_max(thread_absmax(attn, n_attn, bad));
    bad = __syncthreads_or(bad);
    __shared__ bool last;
    if (threadIdx.x == 0) {
        atomicMax(&st->max_gout, __float_as_uint(mg));
        atomicMax(&st->max_attn, __float_as_uint(ma));
        if (bad) atomicOr(&st->nonfinite, 1u);
        __threadfence();
        last = atomicAdd(&st->blocks_done, 1u) == gridDim.x - 1;
    }
    __syncthreads();
    if (last && threadIdx.x == 0) {
        __threadfence();
        const float amg = __uint_as_float(atomicAdd(&st->max_gout, 0u)), ama = __uint_as_float(atomicAdd(&st->max_attn, 0u));
        int shift = 0;
        if (atomicAdd(&st->nonfinite, 0u) == 0u && amg > 0.f && ama > 0.f) {
            int eg, ea, ec = 0;
            frexpf(amg, &eg);  // max|grad_out| < 2^eg: its power of two rounded up
            frexpf(ama, &ea);
            while ((1ll << ec) < contributions) ++ec;
            shift = 62 - eg - ea - ec;  // in [-257, 358]: 2^shift is a normal double
        }
        st->shift = shift;
    }
}

// grad_value = float(acc) * 2^-s, 4 elements per thread (n % 4 == 0); NaN everywhere after a non-finite input
__global__ void __launch_bounds__(256) msda_det_finalize_kernel(const long long *__restrict__ acc, int64_t n,
                                                                const MsdaDetState *__restrict__ st, float *__restrict__ gv) {
    const int64_t i = ((int64_t)blockIdx.x * blockDim.x + threadIdx.x) * 4;
    if (i >= n) return;
    const int shift = st->shift;
    const bool bad = st->nonfinite != 0u;
    const longlong2 a = *reinterpret_cast<const longlong2 *>(acc + i), c = *reinterpret_cast<const longlong2 *>(acc + i + 2);
    float4 r = make_float4(ldexpf(__ll2float_rn(a.x), -shift), ldexpf(__ll2float_rn(a.y), -shift),
                           ldexpf(__ll2float_rn(c.x), -shift), ldexpf(__ll2float_rn(c.y), -shift));
    if (bad) r = make_float4(__int_as_float(0x7fffffff), __int_as_float(0x7fffffff), __int_as_float(0x7fffffff),
                             __int_as_float(0x7fffffff));
    *reinterpret_cast<float4 *>(gv + i) = r;
}

template <int D, bool DET>
__global__ void __launch_bounds__(kBwdThreads) msda_bwd_kernel(const MsdaBwdParams p) {
    constexpr int LANES = D / 4;
    double scale = 0.0;
    if constexpr (DET) scale = ldexp(1.0, p.det->shift);
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
    float4 gt = go;  // DET: the row elements lane + k * LANES (coalesced integer reductions)
    if constexpr (DET) {
        const float *g = p.gout + item * D + lane;
        gt = make_float4(__ldg(g), __ldg(g + LANES), __ldg(g + 2 * LANES), __ldg(g + 3 * LANES));
    }
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
                    if constexpr (DET) {
                        const int64_t t = -3 * lane;  // o.. point at element 4 * lane of the row, gt wants element lane
                        if (top && lef) red_add_i64x4<LANES>(p.gacc + o00 + t, hy * hx * a, gt, scale);
                        if (top && rig) red_add_i64x4<LANES>(p.gacc + o01 + t, hy * lx * a, gt, scale);
                        if (bot && lef) red_add_i64x4<LANES>(p.gacc + o10 + t, ly * hx * a, gt, scale);
                        if (bot && rig) red_add_i64x4<LANES>(p.gacc + o11 + t, ly * lx * a, gt, scale);
                    } else {
                        if (top && lef) red_add_f4(p.gvalue + o00, hy * hx * a, go);
                        if (top && rig) red_add_f4(p.gvalue + o01, hy * lx * a, go);
                        if (bot && lef) red_add_f4(p.gvalue + o10, ly * hx * a, go);
                        if (bot && rig) red_add_f4(p.gvalue + o11, ly * lx * a, go);
                    }
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

// empty_queries_may_be_null: with num_query == 0 the five per-query arrays are empty and may be NULL
static int msda_bwd_check(const float *value, const int64_t *spatial_shapes, const int64_t *level_start_index,
                          const float *sampling_loc, const float *attn_weight, const float *grad_output, float *grad_value,
                          float *grad_sampling_loc, float *grad_attn_weight, int batch, int num_value, int num_heads,
                          int num_levels, int num_query, int num_points, bool empty_queries_may_be_null, const char *what) {
    const bool per_query = (sampling_loc && attn_weight && grad_output && grad_sampling_loc && grad_attn_weight) ||
                           (empty_queries_may_be_null && num_query == 0);
    SDETR_REQUIRE(value && spatial_shapes && level_start_index && grad_value && per_query, SDETR_ERR_INVALID_ARG,
                  "%s: null pointer", what);
    SDETR_REQUIRE(batch > 0 && num_value > 0 && num_heads > 0 && num_levels > 0 && num_points > 0 && num_query >= 0,
                  SDETR_ERR_INVALID_ARG, "%s: non-positive size", what);
    SDETR_REQUIRE(num_levels <= kMaxLevels, SDETR_ERR_UNSUPPORTED, "%s: more than %d levels", what, kMaxLevels);
    SDETR_REQUIRE(aligned16(value) && aligned16(grad_output) && aligned16(grad_value) &&
                      (reinterpret_cast<uintptr_t>(grad_sampling_loc) & 7u) == 0,
                  SDETR_ERR_INVALID_ARG, "%s: 16-byte alignment required", what);
    return SDETR_OK;
}

template <bool DET>
static int msda_bwd_launch(const MsdaBwdParams &p, int head_dim, cudaStream_t s, const char *what) {
    const int64_t items = (int64_t)p.batch * p.nq * p.heads;
#define SDETR_BWD(DD)                                                                                       \
    case DD: {                                                                                              \
        constexpr int G = kBwdThreads / (DD / 4);                                                           \
        msda_bwd_kernel<DD, DET><<<(unsigned)((items + G - 1) / G), kBwdThreads, 0, s>>>(p);                 \
    } break;
    switch (head_dim) {
        SDETR_BWD(4) SDETR_BWD(8) SDETR_BWD(16) SDETR_BWD(32) SDETR_BWD(64) SDETR_BWD(128)
        default:
            SDETR_REQUIRE(false, SDETR_ERR_UNSUPPORTED, "%s: head_dim %d not in {4,8,16,32,64,128}", what, head_dim);
    }
#undef SDETR_BWD
    return check_launch(what);
}

static bool supported_head_dim(int d) { return d == 4 || d == 8 || d == 16 || d == 32 || d == 64 || d == 128; }

extern "C" int sdetr_msda_backward(const float *value, const int64_t *spatial_shapes, const int64_t *level_start_index,
                                   const float *sampling_loc, const float *attn_weight, const float *grad_output,
                                   float *grad_value, float *grad_sampling_loc, float *grad_attn_weight, int batch,
                                   int num_value, int num_heads, int head_dim, int num_levels, int num_query,
                                   int num_points, sdetr_stream_t stream) {
    int rc = msda_bwd_check(value, spatial_shapes, level_start_index, sampling_loc, attn_weight, grad_output, grad_value,
                            grad_sampling_loc, grad_attn_weight, batch, num_value, num_heads, num_levels, num_query,
                            num_points, false, "msda_backward");
    if (rc != SDETR_OK) return rc;
    cudaStream_t s = (cudaStream_t)stream;
    cudaError_t e = cudaMemsetAsync(grad_value, 0, sizeof(float) * (size_t)batch * num_value * num_heads * head_dim, s);
    SDETR_REQUIRE(e == cudaSuccess, SDETR_ERR_CUDA, "msda_backward: memset: %s", cudaGetErrorString(e));
    if (num_query == 0) return SDETR_OK;
    MsdaBwdParams p{value, spatial_shapes, level_start_index, sampling_loc, attn_weight, grad_output,
                    grad_value, grad_sampling_loc, grad_attn_weight, batch, num_value, num_heads, num_query,
                    num_levels, num_points, nullptr, nullptr};
    return msda_bwd_launch<false>(p, head_dim, s, "msda_backward");
}

extern "C" size_t sdetr_msda_backward_deterministic_workspace(int batch, int num_value, int num_heads, int head_dim) {
    if (batch <= 0 || num_value <= 0 || num_heads <= 0 || head_dim <= 0) return 0;
    return sizeof(long long) * (size_t)batch * num_value * num_heads * head_dim + sizeof(MsdaDetState);
}

extern "C" int sdetr_msda_backward_deterministic(const float *value, const int64_t *spatial_shapes,
                                                 const int64_t *level_start_index, const float *sampling_loc,
                                                 const float *attn_weight, const float *grad_output, float *grad_value,
                                                 float *grad_sampling_loc, float *grad_attn_weight, int batch,
                                                 int num_value, int num_heads, int head_dim, int num_levels,
                                                 int num_query, int num_points, void *workspace, size_t workspace_bytes,
                                                 sdetr_stream_t stream) {
    const char *what = "msda_backward_deterministic";
    int rc = msda_bwd_check(value, spatial_shapes, level_start_index, sampling_loc, attn_weight, grad_output, grad_value,
                            grad_sampling_loc, grad_attn_weight, batch, num_value, num_heads, num_levels, num_query,
                            num_points, true, what);
    if (rc != SDETR_OK) return rc;
    SDETR_REQUIRE(supported_head_dim(head_dim), SDETR_ERR_UNSUPPORTED, "%s: head_dim %d not in {4,8,16,32,64,128}", what,
                  head_dim);
    SDETR_REQUIRE(workspace && aligned16(workspace), SDETR_ERR_INVALID_ARG, "%s: workspace must be a 16-byte aligned pointer",
                  what);
    const size_t need = sdetr_msda_backward_deterministic_workspace(batch, num_value, num_heads, head_dim);
    SDETR_REQUIRE(workspace_bytes >= need, SDETR_ERR_WORKSPACE, "%s: workspace of %zu bytes, %zu needed", what,
                  workspace_bytes, need);
    cudaStream_t s = (cudaStream_t)stream;
    const int64_t n = (int64_t)batch * num_value * num_heads * head_dim;
    if (num_query == 0) {
        cudaError_t e = cudaMemsetAsync(grad_value, 0, sizeof(float) * (size_t)n, s);
        SDETR_REQUIRE(e == cudaSuccess, SDETR_ERR_CUDA, "%s: memset: %s", what, cudaGetErrorString(e));
        return SDETR_OK;
    }
    long long *acc = static_cast<long long *>(workspace);
    MsdaDetState *st = reinterpret_cast<MsdaDetState *>(acc + n);  // n % 4 == 0: 32-byte aligned
    cudaError_t e = cudaMemsetAsync(workspace, 0, need, s);  // accumulator and state
    SDETR_REQUIRE(e == cudaSuccess, SDETR_ERR_CUDA, "%s: memset: %s", what, cudaGetErrorString(e));

    const int64_t n_gout = (int64_t)batch * num_query * num_heads * head_dim;
    const int64_t n_attn = (int64_t)batch * num_query * num_heads * num_levels * num_points;
    const int64_t want = ((n_gout > n_attn ? n_gout : n_attn) / 4 + 255) / 256;
    const int blocks = (int)(want < 1 ? 1 : (want > 4 * sm_count() ? 4 * sm_count() : want));
    msda_det_scale_kernel<<<blocks, 256, 0, s>>>(grad_output, n_gout, attn_weight, n_attn, (int64_t)num_query * num_points, st);
    if ((rc = check_launch(what)) != SDETR_OK) return rc;

    MsdaBwdParams p{value, spatial_shapes, level_start_index, sampling_loc, attn_weight, grad_output,
                    grad_value, grad_sampling_loc, grad_attn_weight, batch, num_value, num_heads, num_query,
                    num_levels, num_points, acc, st};
    if ((rc = msda_bwd_launch<true>(p, head_dim, s, what)) != SDETR_OK) return rc;

    msda_det_finalize_kernel<<<(unsigned)((n / 4 + 255) / 256), 256, 0, s>>>(acc, n, st, grad_value);
    return check_launch(what);
}
