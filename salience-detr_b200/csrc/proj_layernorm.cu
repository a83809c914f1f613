// Encoder output projection with its residual and norm1 -- sdetr_gemm_f16x3_add_layernorm:
//   q = LayerNorm(q + (A . W^T * 2^-(4+s) + bias)) * gamma + beta        A, q (M,256) fp32; W (256,256) as a 3xFP16 pair
//
// Bit for bit what sdetr_gemm_f16x3_pre (C = A . W^T + bias) followed by sdetr_add_layernorm(q, C, ..., y = q) computes, in
// one launch and without the M x 256 round trip of C:
//   * the product is gemm3x_kernel<true, false>'s: per 64-wide k-block the same 12 m64n128k16 wgmma (lo.hi first, from 0),
//     added into an fp32 sum that starts at 0.f in k-block order; then fma(acc, 2^-(4+s), bias);
//   * the LayerNorm is add_layernorm_kernel's at C = 256 (tokens.cu): "lane" L of a row owns columns 4L..4L+3 and
//     128+4L..131+4L, its partial is (0 + ((v0 + v1) + (v2 + v3))) + (the same over the second four), the 32 partials are
//     combined in the xor-16/8/4/2/1 butterfly order, mean = s / 256, the squares as fma(dx, dx, dy * dy) + fma(dz, dz, dw * dw),
//     rstd = rsqrtf(ss / 256 + eps) and y = fma((v - mean) * rstd, gamma, beta).  Every step is written with the _rn
//     intrinsics, so no contraction can differ from that kernel's.
//
// CTA: persistent over 128-row panels, one TMA producer thread (warpgroup 0) and two consumer warpgroups of 64 rows each
// that own all 256 columns of their rows.  A stage holds a k-block of A (two 128 x 32 fp32 boxes) and of W_hi / W_lo for
// output columns 0-127 and 128-255 (96 KB; two stages).  Per k-block a warpgroup splits its A fragments once and runs
// the 12-wgmma chain for each 128-column half into d, adding d into acc[0, 64) and acc[64, 128).
// In the wgmma layout a thread holds column pairs 8j + 2q + {0,1} of rows r0 and r0 + 8; one exchange with the
// neighbouring lane of its quad turns them into the 4-column groups of add_layernorm_kernel's lanes: thread q keeps the
// groups of lanes L = 2j + (q >> 1) with j = q & 1 (mod 2), so the butterfly steps 16, 8, 4 are in registers and 2, 1 are
// quad shuffles (xor 1, xor 2).
#include "wgmma.cuh"

namespace sdetr {

constexpr int kPD = 256;                     // model width: K and N
constexpr int kPStageBytes = 6 * kGBox;      // A (2 boxes), W_hi / W_lo of columns 0-127, W_hi / W_lo of 128-255
constexpr int kPStages = 2;
constexpr int kPSmem = kPStages * kPStageBytes + 1024 /* alignment */ + 256 /* barriers */;

struct ProjLnParams {
    const float *bias, *gamma, *beta;  // bias may be NULL
    float eps, out_scale;              // out_scale: 1 / (kActScale * w_scale)
    float *q;                          // (M, 256) residual in, LayerNorm out
    int M;
};

// Sum of a row's 32 lane partials in add_layernorm_kernel's butterfly order.  part[i] is lane 4i + 2 odd + (q >> 1)'s
// partial: lane xor 16 / 8 / 4 is i xor 4 / 2 / 1 (this thread), xor 2 is the quad neighbour q ^ 1, xor 1 is q ^ 2.
// Each step adds two values, the same sum in both lanes of a pair.
__device__ __forceinline__ float butterfly_sum(const float (&part)[8]) {
    float a[4], b[2];
#pragma unroll
    for (int i = 0; i < 4; ++i) a[i] = __fadd_rn(part[i], part[i + 4]);
#pragma unroll
    for (int i = 0; i < 2; ++i) b[i] = __fadd_rn(a[i], a[i + 2]);
    float t = __fadd_rn(b[0], b[1]);
    t = __fadd_rn(t, __shfl_xor_sync(0xffffffffu, t, 1));
    return __fadd_rn(t, __shfl_xor_sync(0xffffffffu, t, 2));
}

__global__ void __launch_bounds__(kGThreads, 1)
    proj_layernorm_kernel(const __grid_constant__ CUtensorMap ma, const __grid_constant__ CUtensorMap mh,
                          const __grid_constant__ CUtensorMap ml, const ProjLnParams p) {
    extern __shared__ uint8_t smem_raw[];
    uint8_t *smem = reinterpret_cast<uint8_t *>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~uintptr_t(1023));
    uint64_t *full = reinterpret_cast<uint64_t *>(smem + kPStages * kPStageBytes);
    uint64_t *empty = full + kPStages;
    if (threadIdx.x == 0) {
        for (int s = 0; s < kPStages; ++s) mbar_init(full + s, 1), mbar_init(empty + s, 8);  // 8 consumer warps release
        asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
    }
    __syncthreads();
    const int panels = (p.M + kGM - 1) / kGM, kblocks = kPD / 64;
    const int wg = threadIdx.x >> 7, tid = threadIdx.x & 127;

    if (wg == 0) {  // ---- producer
        asm volatile("setmaxnreg.dec.sync.aligned.u32 24;");
        if (tid == 0) {
            int s = 0;
            uint32_t ph = 0;
            for (int pnl = blockIdx.x; pnl < panels; pnl += gridDim.x) {
                for (int kb = 0; kb < kblocks; ++kb) {
                    mbar_wait(empty + s, ph ^ 1);
                    uint8_t *st = smem + s * kPStageBytes;
                    mbar_expect_tx(full + s, 6 * kGBox);
                    tma_load_2d(&ma, full + s, st, kb * 64, pnl * kGM);
                    tma_load_2d(&ma, full + s, st + kGBox, kb * 64 + 32, pnl * kGM);
#pragma unroll
                    for (int half = 0; half < 2; ++half) {
                        tma_load_2d(&mh, full + s, st + (2 + 2 * half) * kGBox, kb * 64, half * kGN);
                        tma_load_2d(&ml, full + s, st + (3 + 2 * half) * kGBox, kb * 64, half * kGN);
                    }
                    if (++s == kPStages) s = 0, ph ^= 1;
                }
            }
        }
        return;
    }

    // ---- consumers: warpgroup wg owns panel rows [64 (wg - 1), 64 wg), all 256 columns
    asm volatile("setmaxnreg.inc.sync.aligned.u32 240;");
    const int warp = tid >> 5, lane = tid & 31, g = lane >> 2, q = lane & 3;
    const int r0 = (wg - 1) * 64 + warp * 16 + g;  // this thread's fragment rows: r0, r0 + 8
    const int odd = q & 1;
    int s = 0;
    uint32_t ph = 0;
    float acc[128], d[64];  // acc[64 half + 4j + 2h + e] = (row r0 + 8h, column 128 half + 8j + 2q + e)
    uint32_t ahi[4][4], alo[4][4];
    for (int pnl = blockIdx.x; pnl < panels; pnl += gridDim.x) {
#pragma unroll
        for (int i = 0; i < 128; ++i) acc[i] = 0.f;
        for (int kb = 0; kb < kblocks; ++kb) {
            uint8_t *st = smem + s * kPStageBytes;
            gemm3x_stage_in<true, false>(st, full + s, ph, r0, q, 0, kActScale, ahi, alo);
#pragma unroll
            for (int half = 0; half < 2; ++half) {
                gemm3x_issue<true>(d, ahi, alo, st + 2 * half * kGBox);  // W_hi / W_lo of this half follow the A boxes
                wgmma_wait_all();
#pragma unroll
                for (int i = 0; i < 64; ++i) acc[64 * half + i] = __fadd_rn(acc[64 * half + i], d[i]);
            }
            if (lane == 0) mbar_arrive(empty + s);
            if (++s == kPStages) s = 0, ph ^= 1;
        }

        // Row by row (r0, then r0 + 8), so that the first row's values are dead before the second's are rewritten.
        // Exchange within lane pairs (q, q ^ 1): afterwards group (half, i) = columns cb + 128 half + 16 i .. + 3 of the row
        // in acc[64 half + 8i + 2h + {0, 1}] (first two) and acc[64 half + 8i + 4 + 2h + {0, 1}] (last two), cb = 8 odd +
        // 4 (q >> 1): add_layernorm_kernel's lane 2 (2i + odd) + (q >> 1) of that half.
        const int cb = 8 * odd + 4 * (q >> 1);
#pragma unroll
        for (int h = 0; h < 2; ++h) {
#pragma unroll
            for (int half = 0; half < 2; ++half)
#pragma unroll
                for (int i = 0; i < 8; ++i) {
                    float &e0 = acc[64 * half + 8 * i + 2 * h], &e1 = acc[64 * half + 8 * i + 2 * h + 1];          // j = 2i
                    float &o0 = acc[64 * half + 8 * i + 4 + 2 * h], &o1 = acc[64 * half + 8 * i + 4 + 2 * h + 1];  // j = 2i + 1
                    const float r0v = __shfl_xor_sync(0xffffffffu, odd ? e0 : o0, 1);
                    const float r1v = __shfl_xor_sync(0xffffffffu, odd ? e1 : o1, 1);
                    // even q: (own j = 2i pair, partner's j = 2i pair); odd q: (partner's j = 2i + 1 pair, own j = 2i + 1 pair)
                    if (odd) e0 = r0v, e1 = r1v;
                    else o0 = r0v, o1 = r1v;
                }
            const int64_t row = (int64_t)pnl * kGM + r0 + 8 * h;
            float *qrow = p.q + (row < p.M ? row : 0) * kPD + cb;
            float part[8];
#pragma unroll
            for (int i = 0; i < 8; ++i) {
                float sum = 0.f;
#pragma unroll
                for (int half = 0; half < 2; ++half) {
                    const int c = half * 128 + 16 * i;
                    const float4 b = p.bias ? ldg_f4(p.bias + cb + c) : make_float4(0.f, 0.f, 0.f, 0.f);
                    const float4 x = *reinterpret_cast<const float4 *>(qrow + c);
                    float &v0 = acc[64 * half + 8 * i + 2 * h], &v1 = acc[64 * half + 8 * i + 2 * h + 1];
                    float &v2 = acc[64 * half + 8 * i + 4 + 2 * h], &v3 = acc[64 * half + 8 * i + 4 + 2 * h + 1];
                    v0 = __fadd_rn(x.x, __fmaf_rn(v0, p.out_scale, b.x));
                    v1 = __fadd_rn(x.y, __fmaf_rn(v1, p.out_scale, b.y));
                    v2 = __fadd_rn(x.z, __fmaf_rn(v2, p.out_scale, b.z));
                    v3 = __fadd_rn(x.w, __fmaf_rn(v3, p.out_scale, b.w));
                    sum = __fadd_rn(sum, __fadd_rn(__fadd_rn(v0, v1), __fadd_rn(v2, v3)));
                }
                part[i] = sum;
            }
            const float mean = __fdiv_rn(butterfly_sum(part), (float)kPD);
#pragma unroll
            for (int i = 0; i < 8; ++i) {
                float sq = 0.f;
#pragma unroll
                for (int half = 0; half < 2; ++half) {
                    const float dx = __fsub_rn(acc[64 * half + 8 * i + 2 * h], mean);
                    const float dy = __fsub_rn(acc[64 * half + 8 * i + 2 * h + 1], mean);
                    const float dz = __fsub_rn(acc[64 * half + 8 * i + 4 + 2 * h], mean);
                    const float dw = __fsub_rn(acc[64 * half + 8 * i + 4 + 2 * h + 1], mean);
                    sq = __fadd_rn(sq, __fadd_rn(__fmaf_rn(dx, dx, __fmul_rn(dy, dy)), __fmaf_rn(dz, dz, __fmul_rn(dw, dw))));
                }
                part[i] = sq;
            }
            const float rstd = rsqrtf(__fadd_rn(__fdiv_rn(butterfly_sum(part), (float)kPD), p.eps));
            if (row >= p.M) continue;  // (rows past M computed from row 0's residual; nothing of them is written)
#pragma unroll
            for (int half = 0; half < 2; ++half)
#pragma unroll
                for (int i = 0; i < 8; ++i) {
                    const int c = half * 128 + 16 * i;
                    const float4 gm = ldg_f4(p.gamma + cb + c), bt = ldg_f4(p.beta + cb + c);
                    float4 o;
                    o.x = __fmaf_rn(__fmul_rn(__fsub_rn(acc[64 * half + 8 * i + 2 * h], mean), rstd), gm.x, bt.x);
                    o.y = __fmaf_rn(__fmul_rn(__fsub_rn(acc[64 * half + 8 * i + 2 * h + 1], mean), rstd), gm.y, bt.y);
                    o.z = __fmaf_rn(__fmul_rn(__fsub_rn(acc[64 * half + 8 * i + 4 + 2 * h], mean), rstd), gm.z, bt.z);
                    o.w = __fmaf_rn(__fmul_rn(__fsub_rn(acc[64 * half + 8 * i + 4 + 2 * h + 1], mean), rstd), gm.w, bt.w);
                    *reinterpret_cast<float4 *>(qrow + c) = o;
                }
        }
    }
}

}  // namespace sdetr

using namespace sdetr;

extern "C" int sdetr_gemm_f16x3_add_layernorm(const float *A, int64_t lda, const void *W_hi, const void *W_lo, float w_scale,
                                              const float *bias, const float *gamma, const float *beta, float eps, float *q, int M,
                                              sdetr_stream_t stream) {
    SDETR_REQUIRE(A && W_hi && W_lo && gamma && beta && q, SDETR_ERR_INVALID_ARG, "gemm_f16x3_add_layernorm: null pointer");
    SDETR_REQUIRE(M >= 0, SDETR_ERR_INVALID_ARG, "gemm_f16x3_add_layernorm: bad sizes");
    SDETR_REQUIRE(w_scale > 0.f, SDETR_ERR_INVALID_ARG, "gemm_f16x3_add_layernorm: weight scale must be positive");
    SDETR_REQUIRE(lda % 4 == 0 && lda >= kPD && aligned16(A) && aligned16(W_hi) && aligned16(W_lo) && aligned16(q) &&
                      (!bias || aligned16(bias)) && aligned16(gamma) && aligned16(beta),
                  SDETR_ERR_INVALID_ARG, "gemm_f16x3_add_layernorm: operands must be 16-byte aligned with 16-byte row pitch");
    if (M == 0) return SDETR_OK;
    CUtensorMap ma, mh, ml;
    SDETR_REQUIRE(make_map_2d(&ma, CU_TENSOR_MAP_DATA_TYPE_FLOAT32, 4, A, M, kPD, lda, 32, kGM) &&
                      make_map_2d(&mh, CU_TENSOR_MAP_DATA_TYPE_FLOAT16, 2, W_hi, kPD, kPD, kPD, 64, kGN) &&
                      make_map_2d(&ml, CU_TENSOR_MAP_DATA_TYPE_FLOAT16, 2, W_lo, kPD, kPD, kPD, 64, kGN),
                  SDETR_ERR_CUDA, "gemm_f16x3_add_layernorm: cuTensorMapEncodeTiled failed");
    const ProjLnParams p{bias, gamma, beta, eps, 1.f / (kActScale * w_scale), q, M};
    static PerDeviceOnce once;
    SDETR_OPT_IN_SMEM(once, proj_layernorm_kernel, kPSmem, "gemm_f16x3_add_layernorm");
    const int panels = (M + kGM - 1) / kGM, ctas = persistent_ctas();
    proj_layernorm_kernel<<<panels < ctas ? panels : ctas, kGThreads, kPSmem, (cudaStream_t)stream>>>(ma, mh, ml, p);
    return check_launch("gemm_f16x3_add_layernorm");
}
