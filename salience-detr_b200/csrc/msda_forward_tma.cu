// MSDA core forward, TMA-staged variant -- per-level value windows in shared memory (option "msda_tma").
//
// Reference semantics as msda_forward.cu (ms_deform_im2col_cuda.cuh:226-288; ms_deform_attn.py:322-349 for the fused part).
//
// Why: the L1 gather of msda_forward.cu can be bounded by the cache's tag stage rather than its data stage (multi-line
// requests are replayed line by line even when every access hits); a shared-memory row costs one 128-byte wavefront.  So this variant
// stages, per CTA, the part of every level's value map that its queries sample into shared memory with TMA and gathers
// from there:
//   * CTA = one head x `chunk` consecutive queries of the spatial tile order (as the head-major schedule of
//     msda_forward.cu), 256 threads, 8-lane groups;
//   * pass 1 (cheap): every (query, point) location is computed once to find, per level, the top-left corner of the
//     chunk's sampling footprint (warp-shuffle + shared-memory atomic minima);
//   * one elected thread issues FOUR cp.async.bulk.tensor.4d loads (one tensor map per level over (channel, x, y, image),
//     box = 32 channels x BX x BY tokens of this head) anchored at that corner, completing on one mbarrier; out-of-map
//     coordinates are zero-filled by the TMA unit, which IS the bilinear zero padding of the reference;
//   * pass 2 = the gather of msda_forward.cu (owner-computes setup, shared-memory broadcast) with each corner row read from
//     the window by one LDS.128 per lane when the 2x2 footprint lies inside the window, else by the global-memory path
//     (any offset stays correct; only speed depends on the windows fitting).
// Windows: 22x15, 15x12, 12x10, 10x9 tokens (levels 0..3) = 720 rows x 128 B = 90 KB: two CTAs per SM, so one CTA's
// TMA wait overlaps the other's gather.
#include <cuda.h>

#include "msda.cuh"

namespace sdetr {

namespace {

constexpr int kT = 256, kL = 4, kP = 4, kNP = 16, kD = 32, kLanes = 8, kGroups = kT / kLanes;
// window extents (tokens) per level; two CTAs per SM must fit (2 x ~106 KB)
__host__ __device__ constexpr int BX(int l) { return l == 0 ? 22 : l == 1 ? 15 : l == 2 ? 12 : 10; }
__host__ __device__ constexpr int BY(int l) { return l == 0 ? 15 : l == 1 ? 12 : l == 2 ? 10 : 9; }
__host__ __device__ constexpr int win_off(int l) { return l == 0 ? 0 : win_off(l - 1) + BX(l - 1) * BY(l - 1) * 128; }
constexpr int kWinBytes = win_off(kL);
constexpr int kBcW = 336, kBcPk = 80;  // per-group broadcast strides (bytes), as in msda_forward.cu
constexpr int kSmemTma = kWinBytes + kGroups * (kBcW + kBcPk) + 128;

struct Geo {
    int H, W;
    float Hf, Wf;
    int64_t start;
};

struct Setup {
    uint32_t packed;  // bits 0..11 x, 12..23 y of the clamped top-left corner, bit 30 dx, bit 31 dy; 0 weights when out of map
    float w00, w01, w10, w11;
};

__device__ __forceinline__ Setup make_setup_xy(float x, float y, float a, int H, int W, float Hf, float Wf) {
    Setup s;
    const float h_im = fmaf(y, Hf, -0.5f), w_im = fmaf(x, Wf, -0.5f);           // .cuh:274-275
    const bool in = h_im > -1.f && w_im > -1.f && h_im < Hf && w_im < Wf;        // .cuh:277
    const float hf = floorf(h_im), wf = floorf(w_im);
    const int y0 = (int)hf, x0 = (int)wf;
    const float ly = h_im - hf, lx = w_im - wf, hy = 1.f - ly, hx = 1.f - lx;
    const bool top = y0 >= 0, bot = y0 + 1 <= H - 1, lef = x0 >= 0, rig = x0 + 1 <= W - 1;
    // selected, not multiplied: a non-finite location (in == false, NaN fractions) contributes exactly 0 like the reference's
    // branch (.cuh:277) and like msda_backward.cu, instead of 0 * NaN
    s.w00 = (in && top && lef) ? a * hy * hx : 0.f;
    s.w01 = (in && top && rig) ? a * hy * lx : 0.f;
    s.w10 = (in && bot && lef) ? a * ly * hx : 0.f;
    s.w11 = (in && bot && rig) ? a * ly * lx : 0.f;
    const int rt = max(y0, 0), rb = min(y0 + 1, H - 1), cl = max(x0, 0), cr = min(x0 + 1, W - 1);
    s.packed = in ? ((uint32_t)cl | ((uint32_t)rt << 12) | ((uint32_t)(cr - cl) << 30) | ((uint32_t)(rb - rt) << 31)) : 0u;
    return s;
}

__device__ __forceinline__ uint32_t smem_u32(const void *p) { return (uint32_t)__cvta_generic_to_shared(p); }
__device__ __forceinline__ const float *row_ptr(const char *base, uint32_t index, uint32_t stride_bytes) {
    uint64_t r;
    asm("mad.wide.u32 %0, %1, %2, %3;" : "=l"(r) : "r"(index), "r"(stride_bytes), "l"(reinterpret_cast<uint64_t>(base)));
    return reinterpret_cast<const float *>(r);
}
__device__ __forceinline__ void fma4(float4 &acc, float w, const float4 &v) {
    acc.x = fmaf(w, v.x, acc.x), acc.y = fmaf(w, v.y, acc.y), acc.z = fmaf(w, v.z, acc.z), acc.w = fmaf(w, v.w, acc.w);
}

struct TmaMaps {
    CUtensorMap m[kL];
};

template <bool FUSED>
__global__ void __launch_bounds__(kT, 2) msda_fwd_tma_kernel(const MsdaFwdParams p, const __grid_constant__ TmaMaps maps) {
    extern __shared__ __align__(128) uint8_t tsm[];
    uint8_t *win = reinterpret_cast<uint8_t *>((reinterpret_cast<uintptr_t>(tsm) + 127) & ~(uintptr_t)127);
    char *bc = reinterpret_cast<char *>(win + kWinBytes);
    __shared__ int s_min[kL][2];
    __shared__ __align__(8) uint64_t s_bar;
    const int lane = threadIdx.x % kLanes, grp = threadIdx.x / kLanes;
    const int b = blockIdx.z, m = blockIdx.y;
    Geo geo[kL];
#pragma unroll
    for (int l = 0; l < kL; ++l) {
        geo[l].H = (int)__ldg(p.shapes + 2 * l);
        geo[l].W = (int)__ldg(p.shapes + 2 * l + 1);
        geo[l].Hf = (float)geo[l].H, geo[l].Wf = (float)geo[l].W;
        geo[l].start = __ldg(p.lsi + l);
    }
    if (threadIdx.x < kL * 2) s_min[threadIdx.x >> 1][threadIdx.x & 1] = 0x7fffffff;
    if (threadIdx.x == 0) {
        asm volatile("mbarrier.init.shared::cta.b64 [%0], 1;" ::"r"(smem_u32(&s_bar)));
        asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
    }
    __syncthreads();

    const int q_first = blockIdx.x * p.chunk + grp;
    const int q_last = min(p.nq, (int)(blockIdx.x + 1) * p.chunk) - 1;
    const int iters = (p.chunk + kGroups - 1) / kGroups;
    // this lane's two points: e0 = lane (levels 0..1), e1 = lane + 8 (levels 2..3)
    const int l0 = lane >> 2, l1 = 2 + (lane >> 2);

    // ---- pass 1: footprint corner per level (top-left pixel of every in-map sample) --------------------------------------
    {
        int mnx0 = 0x7fffffff, mny0 = 0x7fffffff, mnx1 = 0x7fffffff, mny1 = 0x7fffffff;
        for (int it = 0; it < iters; ++it) {
            const int qi = q_first + it * kGroups;
            if (qi > q_last) break;  // group-uniform; no shuffles in this pass
            const int q = __ldg(p.order + (int64_t)b * p.nq + qi);
            const int64_t row = (int64_t)b * p.nq + q, qm = row * p.heads + m;
            const float Wf0 = l0 ? geo[1].Wf : geo[0].Wf, Hf0 = l0 ? geo[1].Hf : geo[0].Hf;
            const float Wf1 = l1 == 3 ? geo[3].Wf : geo[2].Wf, Hf1 = l1 == 3 ? geo[3].Hf : geo[2].Hf;
            float x0, y0, x1, y1;
            if constexpr (FUSED) {
                const float *offs = p.proj + row * p.proj_stride + (int64_t)m * 2 * kNP;
                const float2 o0 = __ldg(reinterpret_cast<const float2 *>(offs) + lane);
                const float2 o1 = __ldg(reinterpret_cast<const float2 *>(offs) + lane + 8);
                const float *rrow = p.ref + row * (p.ref_dim * kL);
                fused_location<kP>(rrow, l0, p.ref_dim, o0.x, o0.y, Wf0, Hf0, x0, y0);
                fused_location<kP>(rrow, l1, p.ref_dim, o1.x, o1.y, Wf1, Hf1, x1, y1);
            } else {
                const float2 a0 = __ldg(reinterpret_cast<const float2 *>(p.loc + qm * (2 * kNP)) + lane);
                const float2 a1 = __ldg(reinterpret_cast<const float2 *>(p.loc + qm * (2 * kNP)) + lane + 8);
                x0 = a0.x, y0 = a0.y, x1 = a1.x, y1 = a1.y;
            }
            const float hx0 = fmaf(x0, Wf0, -0.5f), hy0 = fmaf(y0, Hf0, -0.5f), hx1 = fmaf(x1, Wf1, -0.5f), hy1 = fmaf(y1, Hf1, -0.5f);
            if (hx0 > -1.f && hy0 > -1.f && hx0 < Wf0 && hy0 < Hf0) mnx0 = min(mnx0, max((int)floorf(hx0), 0)), mny0 = min(mny0, max((int)floorf(hy0), 0));
            if (hx1 > -1.f && hy1 > -1.f && hx1 < Wf1 && hy1 < Hf1) mnx1 = min(mnx1, max((int)floorf(hx1), 0)), mny1 = min(mny1, max((int)floorf(hy1), 0));
        }
        // lanes with the same (lane >> 2) hold the same level: reduce over lane bits 0,1 and over the 4 groups of the warp
#pragma unroll
        for (int o = 1; o <= 2; o <<= 1) {
            mnx0 = min(mnx0, __shfl_xor_sync(0xffffffffu, mnx0, o)), mny0 = min(mny0, __shfl_xor_sync(0xffffffffu, mny0, o));
            mnx1 = min(mnx1, __shfl_xor_sync(0xffffffffu, mnx1, o)), mny1 = min(mny1, __shfl_xor_sync(0xffffffffu, mny1, o));
        }
#pragma unroll
        for (int o = 8; o <= 16; o <<= 1) {
            mnx0 = min(mnx0, __shfl_xor_sync(0xffffffffu, mnx0, o)), mny0 = min(mny0, __shfl_xor_sync(0xffffffffu, mny0, o));
            mnx1 = min(mnx1, __shfl_xor_sync(0xffffffffu, mnx1, o)), mny1 = min(mny1, __shfl_xor_sync(0xffffffffu, mny1, o));
        }
        if ((threadIdx.x & 31) == 0 || (threadIdx.x & 31) == 4) {  // lane 0 of the warp: levels 0 / 2; lane 4: levels 1 / 3
            atomicMin(&s_min[l0][0], mnx0), atomicMin(&s_min[l0][1], mny0);
            atomicMin(&s_min[l1][0], mnx1), atomicMin(&s_min[l1][1], mny1);
        }
    }
    __syncthreads();
    int wx0[kL], wy0[kL];
#pragma unroll
    for (int l = 0; l < kL; ++l) {
        wx0[l] = s_min[l][0] == 0x7fffffff ? 0 : s_min[l][0];
        wy0[l] = s_min[l][1] == 0x7fffffff ? 0 : s_min[l][1];
    }
    if (threadIdx.x == 0) {
        asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(smem_u32(&s_bar)), "r"(kWinBytes) : "memory");
#pragma unroll
        for (int l = 0; l < kL; ++l)
            asm volatile(
                "cp.async.bulk.tensor.4d.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1, {%3, %4, %5, %6}], [%2];" ::"r"(
                    smem_u32(win + win_off(l))),
                "l"(reinterpret_cast<uint64_t>(&maps.m[l])), "r"(smem_u32(&s_bar)), "r"(m * kD), "r"(wx0[l]), "r"(wy0[l]), "r"(b)
                : "memory");
    }
    // wait for the windows (phase 0)
    asm volatile(
        "{\n\t"
        ".reg .pred p;\n\t"
        "WAIT_%=:\n\t"
        "mbarrier.try_wait.parity.shared::cta.b64 p, [%0], 0;\n\t"
        "@p bra DONE_%=;\n\t"
        "bra WAIT_%=;\n\t"
        "DONE_%=:\n\t"
        "}\n" ::"r"(smem_u32(&s_bar))
        : "memory");

    // ---- pass 2: setup (owner computes, shared-memory broadcast) + gather from the windows --------------------------------
    char *wsm = bc + grp * kBcW;
    char *pksm = bc + kGroups * kBcW + grp * kBcPk;
    const uint32_t tsb = (uint32_t)p.v_tstride * 4u;
    const char *vhead = reinterpret_cast<const char *>(p.value + (int64_t)b * p.v_bstride + (int64_t)m * kD + lane * 4);
    for (int it = 0; it < iters; ++it) {
        int qi = q_first + it * kGroups;
        const bool active = qi <= q_last;
        qi = min(qi, q_last);
        const int q = __ldg(p.order + (int64_t)b * p.nq + qi);
        const int64_t row = (int64_t)b * p.nq + q, qm = row * p.heads + m;
        float lx[2], ly[2], la[2];
        if constexpr (FUSED) {
            const float *prow = p.proj + row * p.proj_stride;
            const float *offs = prow + (int64_t)m * 2 * kNP;
            const float *logit = prow + (int64_t)p.heads * 2 * kNP + (int64_t)m * kNP;
            const float2 o0 = __ldg(reinterpret_cast<const float2 *>(offs) + lane), o1 = __ldg(reinterpret_cast<const float2 *>(offs) + lane + 8);
            la[0] = __ldg(logit + lane), la[1] = __ldg(logit + lane + 8);
            const float mx = group_max<kLanes>(fmaxf(la[0], la[1]));
            la[0] = __expf(la[0] - mx), la[1] = __expf(la[1] - mx);
            const float inv = __frcp_rn(group_sum<kLanes>(la[0] + la[1]));
            la[0] *= inv, la[1] *= inv;
            const float *rrow = p.ref + row * (p.ref_dim * kL);
            fused_location<kP>(rrow, l0, p.ref_dim, o0.x, o0.y, l0 ? geo[1].Wf : geo[0].Wf, l0 ? geo[1].Hf : geo[0].Hf, lx[0], ly[0]);
            fused_location<kP>(rrow, l1, p.ref_dim, o1.x, o1.y, l1 == 3 ? geo[3].Wf : geo[2].Wf, l1 == 3 ? geo[3].Hf : geo[2].Hf, lx[1], ly[1]);
            if (active) {
                if (p.loc_out) {
                    reinterpret_cast<float2 *>(p.loc_out + qm * (2 * kNP))[lane] = make_float2(lx[0], ly[0]);
                    reinterpret_cast<float2 *>(p.loc_out + qm * (2 * kNP))[lane + 8] = make_float2(lx[1], ly[1]);
                }
                if (p.attn_out) p.attn_out[qm * kNP + lane] = la[0], p.attn_out[qm * kNP + lane + 8] = la[1];
            }
        } else {
            const float2 a0 = __ldg(reinterpret_cast<const float2 *>(p.loc + qm * (2 * kNP)) + lane);
            const float2 a1 = __ldg(reinterpret_cast<const float2 *>(p.loc + qm * (2 * kNP)) + lane + 8);
            lx[0] = a0.x, ly[0] = a0.y, lx[1] = a1.x, ly[1] = a1.y;
            la[0] = __ldg(p.attn + qm * kNP + lane), la[1] = __ldg(p.attn + qm * kNP + lane + 8);
        }
        const Setup s0 = make_setup_xy(lx[0], ly[0], la[0], l0 ? geo[1].H : geo[0].H, l0 ? geo[1].W : geo[0].W,
                                       l0 ? geo[1].Hf : geo[0].Hf, l0 ? geo[1].Wf : geo[0].Wf);
        const Setup s1 = make_setup_xy(lx[1], ly[1], la[1], l1 == 3 ? geo[3].H : geo[2].H, l1 == 3 ? geo[3].W : geo[2].W,
                                       l1 == 3 ? geo[3].Hf : geo[2].Hf, l1 == 3 ? geo[3].Wf : geo[2].Wf);
        *reinterpret_cast<float4 *>(wsm + lane * 16) = make_float4(s0.w00, s0.w01, s0.w10, s0.w11);
        *reinterpret_cast<float4 *>(wsm + (lane + 8) * 16) = make_float4(s1.w00, s1.w01, s1.w10, s1.w11);
        *reinterpret_cast<uint32_t *>(pksm + lane * 4) = s0.packed;
        *reinterpret_cast<uint32_t *>(pksm + (lane + 8) * 4) = s1.packed;
        __syncwarp();
        float4 acc = make_float4(0.f, 0.f, 0.f, 0.f);
#pragma unroll
        for (int l = 0; l < kL; ++l) {
            const uint4 pk4 = *reinterpret_cast<const uint4 *>(pksm + l * 16);
            const uint32_t pks[4] = {pk4.x, pk4.y, pk4.z, pk4.w};
            const char *lvl_base = vhead + geo[l].start * (int64_t)tsb;
            const uint8_t *wl = win + win_off(l) + lane * 16;
            const uint32_t W = (uint32_t)geo[l].W;
            float4 v[kP][4], w[kP];
#pragma unroll
            for (int pt = 0; pt < kP; ++pt) {
                w[pt] = *reinterpret_cast<const float4 *>(wsm + (l * kP + pt) * 16);
                const uint32_t pk = pks[pt];
                const uint32_t x = pk & 0xfffu, y = (pk >> 12) & 0xfffu, dx = (pk >> 30) & 1u, dy = pk >> 31;
                const uint32_t rx = x - (uint32_t)wx0[l], ry = y - (uint32_t)wy0[l];
                if (rx < (uint32_t)(BX(l) - 1) && ry < (uint32_t)(BY(l) - 1)) {  // the 2x2 footprint lies inside the window
                    const uint8_t *r00 = wl + (ry * BX(l) + rx) * 128;
                    v[pt][0] = *reinterpret_cast<const float4 *>(r00);
                    v[pt][1] = *reinterpret_cast<const float4 *>(r00 + dx * 128);
                    v[pt][2] = *reinterpret_cast<const float4 *>(r00 + dy * (BX(l) * 128));
                    v[pt][3] = *reinterpret_cast<const float4 *>(r00 + dy * (BX(l) * 128) + dx * 128);
                } else {  // outside the staged window: global-memory path (clamped addresses, zero weights when out of map)
                    const uint32_t i00 = y * W + x, i01 = i00 + dx, i10 = i00 + dy * W, i11 = i10 + dx;
                    v[pt][0] = ldg_f4(row_ptr(lvl_base, i00, tsb));
                    v[pt][1] = ldg_f4(row_ptr(lvl_base, i01, tsb));
                    v[pt][2] = ldg_f4(row_ptr(lvl_base, i10, tsb));
                    v[pt][3] = ldg_f4(row_ptr(lvl_base, i11, tsb));
                }
            }
#pragma unroll
            for (int pt = 0; pt < kP; ++pt) {
                fma4(acc, w[pt].x, v[pt][0]);
                fma4(acc, w[pt].y, v[pt][1]);
                fma4(acc, w[pt].z, v[pt][2]);
                fma4(acc, w[pt].w, v[pt][3]);
            }
        }
        __syncwarp();
        if (active) st_stream_f4(p.out + qm * kD + lane * 4, acc);
    }
}

typedef CUresult (*EncodeTiledFn)(CUtensorMap *, CUtensorMapDataType, cuuint32_t, void *, const cuuint64_t *, const cuuint64_t *,
                                  const cuuint32_t *, const cuuint32_t *, CUtensorMapInterleave, CUtensorMapSwizzle,
                                  CUtensorMapL2promotion, CUtensorMapFloatOOBfill);
EncodeTiledFn encode_fn() {
    static EncodeTiledFn fn = nullptr;
    if (!fn) {
        void *p = nullptr;
        cudaDriverEntryPointQueryResult q;
        if (cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &p, cudaEnableDefault, &q) == cudaSuccess && q == cudaDriverEntryPointSuccess)
            fn = reinterpret_cast<EncodeTiledFn>(p);
    }
    return fn;
}

}  // namespace

extern int g_msda_host_shapes[2 * kMaxLevels + 1];  // msda_forward.cu (sdetr_msda_set_host_shapes)

int launch_msda_tma(const MsdaFwdParams &p, bool fused, cudaStream_t stream) {
    // level shapes are needed on the host for the tensor maps: ONE small device->host copy per call would break the
    // "no synchronisation" contract, so the caller-visible entry point only routes here when the shapes were given as
    // host integers (sdetr_msda_set_host_shapes) -- benchmarking variant, see include/sdetr_b200.h
    SDETR_REQUIRE(g_msda_host_shapes[0] == kL, SDETR_ERR_UNSUPPORTED, "msda_tma: host level shapes not set (sdetr_msda_set_host_shapes)");
    EncodeTiledFn enc = encode_fn();
    SDETR_REQUIRE(enc, SDETR_ERR_CUDA, "msda_tma: cuTensorMapEncodeTiled unavailable");
    TmaMaps maps;
    int64_t start = 0;
    for (int l = 0; l < kL; ++l) {
        const int H = g_msda_host_shapes[1 + 2 * l], W = g_msda_host_shapes[2 + 2 * l];
        const cuuint64_t dims[4] = {(cuuint64_t)p.heads * kD, (cuuint64_t)W, (cuuint64_t)H, (cuuint64_t)p.batch};
        const cuuint64_t strides[3] = {(cuuint64_t)p.v_tstride * 4, (cuuint64_t)W * p.v_tstride * 4, (cuuint64_t)p.v_bstride * 4};
        const cuuint32_t box[4] = {(cuuint32_t)kD, (cuuint32_t)BX(l), (cuuint32_t)BY(l), 1};
        const cuuint32_t estr[4] = {1, 1, 1, 1};
        const CUresult r = enc(&maps.m[l], CU_TENSOR_MAP_DATA_TYPE_FLOAT32, 4, const_cast<float *>(p.value + start * p.v_tstride), dims,
                               strides, box, estr, CU_TENSOR_MAP_INTERLEAVE_NONE, CU_TENSOR_MAP_SWIZZLE_NONE,
                               CU_TENSOR_MAP_L2_PROMOTION_L2_128B, CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
        SDETR_REQUIRE(r == CUDA_SUCCESS, SDETR_ERR_CUDA, "msda_tma: cuTensorMapEncodeTiled failed for level %d (%d)", l, (int)r);
        start += (int64_t)H * W;
    }
    SDETR_REQUIRE(start == p.nv, SDETR_ERR_INVALID_ARG, "msda_tma: host level shapes hold %lld tokens, num_value %d", (long long)start, p.nv);
    static PerDeviceOnce o1, o2;
    SDETR_OPT_IN_SMEM(o1, msda_fwd_tma_kernel<true>, kSmemTma, "msda_tma");
    SDETR_OPT_IN_SMEM(o2, msda_fwd_tma_kernel<false>, kSmemTma, "msda_tma");
    dim3 grid((p.nq + p.chunk - 1) / p.chunk, p.heads, p.batch);
    if (fused) msda_fwd_tma_kernel<true><<<grid, kT, kSmemTma, stream>>>(p, maps);
    else msda_fwd_tma_kernel<false><<<grid, kT, kSmemTma, stream>>>(p, maps);
    return check_launch("msda_forward/tma");
}

}  // namespace sdetr
