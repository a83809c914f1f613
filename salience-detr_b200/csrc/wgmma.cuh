// Hopper (sm_90a) tensor-core GEMM with fp32-class accuracy, shared by gemm_f16x3.cu, gemm_tf32x3.cu and ffn_fused.cu:
//   C[M,N] = act(A)[M,K] . W[N,K]^T * out_scale + bias,   A fp32, W given as a (hi, lo) pair (or raw fp32 for 3xTF32).
// The product is error-compensated: A_lo.W_hi + A_hi.W_lo + A_hi.W_hi with hi = round(x), lo = round(x - hi) in the MMA
// input type, which keeps ~22 significand bits per operand (fp16 or TF32 pieces; see include/sdetr_b200.h).
//
// Structure (one CTA per SM, persistent over 128 x 128 output tiles, row-panel-major so neighbouring CTAs share A):
//   warpgroup 0, one thread:  TMA producer -- per k-block the fp32 A box(es) and the W_hi / W_lo boxes (128-byte swizzle)
//                             into a ring of stages, completion on the stage's `full` mbarrier;
//   warpgroups 1 and 2:       64 rows each.  Per k-block every thread reads its register fragment of A from the swizzled
//                             stage, applies the input activation (and the fp16 range scaling), splits it into hi / lo
//                             registers, and issues wgmma.mma_async with A from registers and W from shared memory
//                             (m64n128k16 .f16 or m64n128k8 .tf32, fp32 accumulators in registers); after the k-block's
//                             wgmma group completes each warp releases the stage on its `empty` mbarrier and adds the
//                             k-block's product to a second set of fp32 registers with ordinary round-to-nearest adds
//                             (the tensor core's own accumulation truncates: over K = 2048 that alone costs ~3 bits).
//                             The epilogue scales, adds the bias and stores straight from those registers.  The loop
//                             runs one k-block ahead, across tiles: the next k-block's fragments are split, and the
//                             previous tile's epilogue runs, while the current k-block's wgmma group is in flight.
//                             The fragments are read with shared-window loads, and the loop is compiled once per
//                             input activation, so the split has no per-element activation test.
// Registers: setmaxnreg moves them from the producer warpgroup (40) to the two consumer warpgroups (232 each).
#pragma once
#include <cuda.h>
#include <cuda_fp16.h>

#include "common.cuh"

namespace sdetr {

// ---- PTX wrappers --------------------------------------------------------------------------------------------------
__device__ __forceinline__ uint32_t smem_u32(const void *p) { return (uint32_t)__cvta_generic_to_shared(p); }

__device__ __forceinline__ void mbar_init(uint64_t *bar, uint32_t count) {
    asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(smem_u32(bar)), "r"(count));
}
__device__ __forceinline__ void mbar_arrive(uint64_t *bar) {
    asm volatile("mbarrier.arrive.shared::cta.b64 _, [%0];" ::"r"(smem_u32(bar)) : "memory");
}
__device__ __forceinline__ void mbar_expect_tx(uint64_t *bar, uint32_t bytes) {
    asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(smem_u32(bar)), "r"(bytes) : "memory");
}
__device__ __forceinline__ void mbar_wait(uint64_t *bar, uint32_t parity) {
    asm volatile(
        "{\n\t"
        ".reg .pred p;\n\t"
        "WAIT_%=:\n\t"
        "mbarrier.try_wait.parity.shared::cta.b64 p, [%0], %1;\n\t"
        "@p bra DONE_%=;\n\t"
        "bra WAIT_%=;\n\t"
        "DONE_%=:\n\t"
        "}\n" ::"r"(smem_u32(bar)),
        "r"(parity)
        : "memory");
}
__device__ __forceinline__ void tma_load_2d(const CUtensorMap *map, uint64_t *bar, void *dst, int c0, int c1) {
    asm volatile(
        "cp.async.bulk.tensor.2d.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1, {%3, %4}], [%2];" ::"r"(
            smem_u32(dst)),
        "l"(reinterpret_cast<uint64_t>(map)), "r"(smem_u32(bar)), "r"(c0), "r"(c1)
        : "memory");
}
__device__ __forceinline__ void named_bar_sync(int id, int threads) {
    asm volatile("bar.sync %0, %1;" ::"r"(id), "r"(threads) : "memory");
}

// shared-memory matrix descriptor of a K-major operand tile: rows of 128 bytes, SWIZZLE_128B, 8-row groups 1024 bytes
// apart (start >> 4 in [0,14), leading offset 1 (unused with this swizzle), stride offset 1024 >> 4 in [32,46),
// layout type 1 = 128-byte swizzle in [62,64))
__device__ __forceinline__ uint64_t wgmma_desc(uint32_t smem_addr) {
    return (uint64_t)((smem_addr & 0x3ffffu) >> 4) | (1ull << 16) | (64ull << 32) | (1ull << 62);
}
__device__ __forceinline__ void wgmma_fence() { asm volatile("wgmma.fence.sync.aligned;" ::: "memory"); }
__device__ __forceinline__ void wgmma_commit() { asm volatile("wgmma.commit_group.sync.aligned;" ::: "memory"); }
__device__ __forceinline__ void wgmma_wait_all() { asm volatile("wgmma.wait_group.sync.aligned 0;" ::: "memory"); }

#define SDETR_WGMMA_D64                                                                                                           \
    "{%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, %16, %17, %18, %19, %20, %21, %22, %23, %24, %25, %26, " \
    "%27, %28, %29, %30, %31, %32, %33, %34, %35, %36, %37, %38, %39, %40, %41, %42, %43, %44, %45, %46, %47, %48, %49, %50, %51, "  \
    "%52, %53, %54, %55, %56, %57, %58, %59, %60, %61, %62, %63}, "
#define SDETR_WGMMA_D64_OPS(d)                                                                                                    \
    "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]), "+f"(d[8]), "+f"(d[9]),       \
        "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]), "+f"(d[16]), "+f"(d[17]), "+f"(d[18]),      \
        "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23]), "+f"(d[24]), "+f"(d[25]), "+f"(d[26]), "+f"(d[27]),      \
        "+f"(d[28]), "+f"(d[29]), "+f"(d[30]), "+f"(d[31]), "+f"(d[32]), "+f"(d[33]), "+f"(d[34]), "+f"(d[35]), "+f"(d[36]),      \
        "+f"(d[37]), "+f"(d[38]), "+f"(d[39]), "+f"(d[40]), "+f"(d[41]), "+f"(d[42]), "+f"(d[43]), "+f"(d[44]), "+f"(d[45]),      \
        "+f"(d[46]), "+f"(d[47]), "+f"(d[48]), "+f"(d[49]), "+f"(d[50]), "+f"(d[51]), "+f"(d[52]), "+f"(d[53]), "+f"(d[54]),      \
        "+f"(d[55]), "+f"(d[56]), "+f"(d[57]), "+f"(d[58]), "+f"(d[59]), "+f"(d[60]), "+f"(d[61]), "+f"(d[62]), "+f"(d[63])

// d (64 x 128 fp32 per warpgroup) = (accumulate ? d : 0) + a (64 x 16 fp16, registers) . b (16 x 128 fp16, K-major in shared
// memory)
__device__ __forceinline__ void wgmma_f16_rs(float (&d)[64], const uint32_t (&a)[4], uint64_t desc_b, int accumulate) {
    asm volatile("{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %69, 0;\n\t"
                 "wgmma.mma_async.sync.aligned.m64n128k16.f32.f16.f16 " SDETR_WGMMA_D64
                 "{%64, %65, %66, %67}, %68, p, 1, 1, 0;\n\t}"
                 : SDETR_WGMMA_D64_OPS(d)
                 : "r"(a[0]), "r"(a[1]), "r"(a[2]), "r"(a[3]), "l"(desc_b), "r"(accumulate));
}
// d (64 x 128 fp32 per warpgroup) = (accumulate ? d : 0) + a (64 x 8 tf32, registers) . b (8 x 128 tf32, K-major in shared
// memory)
__device__ __forceinline__ void wgmma_tf32_rs(float (&d)[64], const uint32_t (&a)[4], uint64_t desc_b, int accumulate) {
    asm volatile("{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %69, 0;\n\t"
                 "wgmma.mma_async.sync.aligned.m64n128k8.f32.tf32.tf32 " SDETR_WGMMA_D64
                 "{%64, %65, %66, %67}, %68, p, 1, 1;\n\t}"
                 : SDETR_WGMMA_D64_OPS(d)
                 : "r"(a[0]), "r"(a[1]), "r"(a[2]), "r"(a[3]), "l"(desc_b), "r"(accumulate));
}

#define SDETR_WGMMA_D32                                                                                                           \
    "{%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, %16, %17, %18, %19, %20, %21, %22, %23, %24, %25, %26, " \
    "%27, %28, %29, %30, %31}, "
#define SDETR_WGMMA_D32_OPS(d)                                                                                                    \
    "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]), "+f"(d[8]), "+f"(d[9]),       \
        "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]), "+f"(d[16]), "+f"(d[17]), "+f"(d[18]),      \
        "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23]), "+f"(d[24]), "+f"(d[25]), "+f"(d[26]), "+f"(d[27]),      \
        "+f"(d[28]), "+f"(d[29]), "+f"(d[30]), "+f"(d[31])

// d (64 x 128 fp32 per warpgroup) = (accumulate ? d : 0) + a (64 x 16 fp16) . b (16 x 128 fp16), both K-major in shared memory
__device__ __forceinline__ void wgmma_f16_ss(float (&d)[64], uint64_t desc_a, uint64_t desc_b, int accumulate) {
    asm volatile("{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %66, 0;\n\t"
                 "wgmma.mma_async.sync.aligned.m64n128k16.f32.f16.f16 " SDETR_WGMMA_D64
                 "%64, %65, p, 1, 1, 0, 0;\n\t}"
                 : SDETR_WGMMA_D64_OPS(d)
                 : "l"(desc_a), "l"(desc_b), "r"(accumulate));
}
// d (64 x 64 fp32 per warpgroup) = (accumulate ? d : 0) + a (64 x 16 fp16) . b (16 x 64 fp16), both K-major in shared memory
__device__ __forceinline__ void wgmma_f16_ss_n64(float (&d)[32], uint64_t desc_a, uint64_t desc_b, int accumulate) {
    asm volatile("{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %34, 0;\n\t"
                 "wgmma.mma_async.sync.aligned.m64n64k16.f32.f16.f16 " SDETR_WGMMA_D32
                 "%32, %33, p, 1, 1, 0, 0;\n\t}"
                 : SDETR_WGMMA_D32_OPS(d)
                 : "l"(desc_a), "l"(desc_b), "r"(accumulate));
}

// d (64 x 64 fp32 per warpgroup) = (accumulate ? d : 0) + a (64 x 16 fp16, registers) . b (16 x 64 fp16, K-major in shared
// memory)
__device__ __forceinline__ void wgmma_f16_rs_n64(float (&d)[32], const uint32_t (&a)[4], uint64_t desc_b, int accumulate) {
    asm volatile("{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %37, 0;\n\t"
                 "wgmma.mma_async.sync.aligned.m64n64k16.f32.f16.f16 " SDETR_WGMMA_D32
                 "{%32, %33, %34, %35}, %36, p, 1, 1, 0;\n\t}"
                 : SDETR_WGMMA_D32_OPS(d)
                 : "r"(a[0]), "r"(a[1]), "r"(a[2]), "r"(a[3]), "l"(desc_b), "r"(accumulate));
}

// (x0, x1) -> packed hi (f16x2: x0 in the low half = the lower k index) and packed lo of the residuals
__device__ __forceinline__ void split2(float x0, float x1, uint32_t &hi, uint32_t &lo) {
    const __half2 h = __floats2half2_rn(x0, x1);
    const float2 hf = __half22float2(h);
    const __half2 l = __floats2half2_rn(x0 - hf.x, x1 - hf.y);
    hi = *reinterpret_cast<const uint32_t *>(&h);
    lo = *reinterpret_cast<const uint32_t *>(&l);
}
// round to the nearest TF32 value, ties away from zero; NaN and inf pass unchanged (the carry of the rounding add would
// run a NaN's high mantissa bits through the exponent into the sign: 0x7fffffff would become -0)
__device__ __forceinline__ float tf32_rn(float x) {
    const uint32_t u = __float_as_uint(x);
    return (u & 0x7f800000u) == 0x7f800000u ? x : __uint_as_float((u + 0x1000u) & 0xffffe000u);
}
__device__ __forceinline__ float gelu_erf(float x) { return 0.5f * x * (1.f + erff(x * 0.70710678118654752f)); }
__device__ __forceinline__ float apply_act(float x, int act) { return act == 1 ? relu_nan(x) : act == 2 ? gelu_erf(x) : x; }

// element (r, c) of a 128-row x 32-fp32 box written by TMA with SWIZZLE_128B (16-byte chunk index XOR row % 8)
__device__ __forceinline__ const float *swz_f32(const uint8_t *box, int r, int c) {
    return reinterpret_cast<const float *>(box + r * 128 + ((((c >> 2) ^ (r & 7)) << 4) | ((c & 3) << 2)));
}

// shared-memory loads through the shared window (a generic load of the same address takes the longer generic path)
__device__ __forceinline__ float2 lds_f32x2(const float *p) {
    float2 v;
    asm volatile("ld.shared.v2.f32 {%0, %1}, [%2];" : "=f"(v.x), "=f"(v.y) : "r"(smem_u32(p)));
    return v;
}
__device__ __forceinline__ float lds_f32(const float *p) {
    float v;
    asm volatile("ld.shared.f32 %0, [%1];" : "=f"(v) : "r"(smem_u32(p)));
    return v;
}

// ---- the kernel ------------------------------------------------------------------------------------------------------
constexpr int kGM = 128, kGN = 128;   // CTA tile
constexpr int kGThreads = 384;        // warpgroup 0: TMA producer; warpgroups 1, 2: MMA + epilogue
constexpr int kGBox = 128 * 128;      // 16 KB: 128 rows x 128 bytes, one SWIZZLE_128B TMA box
constexpr float kActScale = 16.f;     // fp16 form: exact activation pre-scale (range argument in include/sdetr_b200.h)

template <bool F16>
struct Gemm3xShape {
    static constexpr int kK = F16 ? 64 : 32;                        // k-block: one 128-byte row of W
    static constexpr int kABoxes = F16 ? 2 : 1;                     // fp32 A boxes of 32 columns per k-block
    static constexpr int kStageBytes = (kABoxes + 2) * kGBox;       // A box(es), W_hi, W_lo
    static constexpr int kStages = F16 ? 3 : 4;                     // 192 KB of ring either way
    static constexpr int kSmem = kStages * kStageBytes + 1024 /* alignment */ + 256 /* barriers */;
};

struct Gemm3xParams {
    const float *bias;         // (N) or NULL
    float *C;
    int64_t ldc;
    int M, N, K, act;          // act: 0 none, 1 ReLU, 2 exact GELU on A
    float a_scale, out_scale;  // A multiplier before the split and accumulator multiplier (fp16 form; 1 for TF32)
    const float *a_scale_dev;  // fp16 form with device scales: a_scale = *a_scale_dev, out_scale = 1 / (a_scale * *w_scale_dev)
    const float *w_scale_dev;
    const float *col_scale;    // EX only: per-column scale s (N) or NULL
    const float *Z;            // EX only: residual z (M rows, pitch ldz) or NULL; may alias C
    int64_t ldz;
    const float *row_scale;    // ROWMAX only: s (M); C[row] = max over the N columns of (acc * out_scale + bias), times s[row]
};

// Consumer side of one k-block, first half: wait until stage `st` has landed (SPLIT_W: split its raw W in place, both
// consumer warpgroups, before any wgmma reads it), then read this thread's A fragments and split them into hi / lo.
template <bool F16, bool SPLIT_W>
__device__ __forceinline__ void gemm3x_stage_in(uint8_t *st, uint64_t *full, uint32_t ph, int r0, int q, int act,
                                                float a_scale, uint32_t (&ahi)[4][4], uint32_t (&alo)[4][4]) {
    using S = Gemm3xShape<F16>;
    mbar_wait(full, ph);
    if (SPLIT_W) {
        uint8_t *w_hi = st + S::kABoxes * kGBox, *w_lo = w_hi + kGBox;
        for (int i = threadIdx.x - 128; i < kGBox / 16; i += 256) {
            const float4 w = reinterpret_cast<const float4 *>(w_hi)[i];
            float4 h, l;
            h.x = tf32_rn(w.x), h.y = tf32_rn(w.y), h.z = tf32_rn(w.z), h.w = tf32_rn(w.w);
            l.x = tf32_rn(w.x - h.x), l.y = tf32_rn(w.y - h.y), l.z = tf32_rn(w.z - h.z), l.w = tf32_rn(w.w - h.w);
            reinterpret_cast<float4 *>(w_hi)[i] = h;
            reinterpret_cast<float4 *>(w_lo)[i] = l;
        }
        asm volatile("fence.proxy.async.shared::cta;" ::: "memory");  // generic-proxy writes -> wgmma operand reads
        named_bar_sync(1, 256);
    }
#pragma unroll
    for (int kk = 0; kk < 4; ++kk) {
        if (F16) {  // m64k16: (r0, c..c+1), (r0+8, c..c+1), (r0, c+8..c+9), (r0+8, c+8..c+9)
            const uint8_t *box = st + (kk >> 1) * kGBox;
            const int c = (kk & 1) * 16 + 2 * q;
#pragma unroll
            for (int j = 0; j < 4; ++j) {
                const float2 x = lds_f32x2(swz_f32(box, r0 + (j & 1) * 8, c + (j >> 1) * 8));
                split2(apply_act(x.x, act) * a_scale, apply_act(x.y, act) * a_scale, ahi[kk][j], alo[kk][j]);
            }
        } else {  // m64k8: (r0, c), (r0+8, c), (r0, c+4), (r0+8, c+4)
            const int c = kk * 8 + q;
#pragma unroll
            for (int j = 0; j < 4; ++j) {
                const float x = apply_act(lds_f32(swz_f32(st, r0 + (j & 1) * 8, c + (j >> 1) * 4)), act), h = tf32_rn(x);
                ahi[kk][j] = __float_as_uint(h), alo[kk][j] = __float_as_uint(tf32_rn(x - h));
            }
        }
    }
}

// Second half: the k-block's 12 wgmma into d (d = alo.W_hi first, then += ahi.W_lo, += ahi.W_hi per 32 bytes of K), one
// commit group.  The caller waits for it before it touches d or rewrites ahi / alo.
template <bool F16>
__device__ __forceinline__ void gemm3x_issue(float (&d)[64], const uint32_t (&ahi)[4][4], const uint32_t (&alo)[4][4],
                                             const uint8_t *st) {
    using S = Gemm3xShape<F16>;
    wgmma_fence();
    const uint32_t bh = smem_u32(st + S::kABoxes * kGBox), bl = bh + kGBox;
#pragma unroll
    for (int kk = 0; kk < 4; ++kk) {  // 32 bytes of K per step in either type
        if (F16) {
            wgmma_f16_rs(d, alo[kk], wgmma_desc(bh + kk * 32), kk);
            wgmma_f16_rs(d, ahi[kk], wgmma_desc(bl + kk * 32), 1);
            wgmma_f16_rs(d, ahi[kk], wgmma_desc(bh + kk * 32), 1);
        } else {
            wgmma_tf32_rs(d, alo[kk], wgmma_desc(bh + kk * 32), kk);
            wgmma_tf32_rs(d, ahi[kk], wgmma_desc(bl + kk * 32), 1);
            wgmma_tf32_rs(d, ahi[kk], wgmma_desc(bh + kk * 32), 1);
        }
    }
    wgmma_commit();
}

// ROWMAX epilogue of a tile that holds all N <= 128 columns: C[row] = max_c (acc * out_scale + bias[c]) * row_scale[row], the
// column values computed as the plain epilogue computes them and their max taken in class_max_kernel's order (tokens.cu):
// lane l of a row's warp there folds columns l, l + 32, l + 64, l + 96 from -inf, then the xor-16/8/4/2/1 butterfly, each
// step fmax_nan(own, partner) and lane 0's result kept.  Column l = 8a + 2q + e (a < 4, e < 2) sits in this thread's
// acc[4 (a + 4k) + 2h + e], so the lane partials of a = 0..3 are this thread's; the steps 16 and 8 combine them in registers,
// 4 and 2 are quad shuffles and 1 is the last register step.
__device__ __forceinline__ void gemm3x_rowmax_epilogue(const Gemm3xParams &p, const float (&acc)[64], int m0, int r0, int q,
                                                       float out_scale) {
    float b[16][2];
#pragma unroll
    for (int j = 0; j < 16; ++j)
#pragma unroll
        for (int e = 0; e < 2; ++e) {
            const int col = 8 * j + 2 * q + e;
            b[j][e] = p.bias && col < p.N ? __ldg(p.bias + col) : 0.f;
        }
#pragma unroll
    for (int h = 0; h < 2; ++h) {
        float v[4][2];  // lane partials of lanes 8a + 2q + e
#pragma unroll
        for (int a = 0; a < 4; ++a)
#pragma unroll
            for (int e = 0; e < 2; ++e) {
                float m = -INFINITY;
#pragma unroll
                for (int k = 0; k < 4; ++k)
                    if (8 * (a + 4 * k) + 2 * q + e < p.N)
                        m = fmax_nan(m, __fmaf_rn(acc[4 * (a + 4 * k) + 2 * h + e], out_scale, b[a + 4 * k][e]));
                v[a][e] = m;
            }
        float w[4][2];
#pragma unroll
        for (int a = 0; a < 4; ++a)
#pragma unroll
            for (int e = 0; e < 2; ++e) w[a][e] = fmax_nan(v[a][e], v[a ^ 2][e]);  // xor 16
        float x[2];
#pragma unroll
        for (int e = 0; e < 2; ++e) {
            x[e] = fmax_nan(w[0][e], w[1][e]);                                        // xor 8 (lanes 2q + e remain)
            x[e] = fmax_nan(x[e], __shfl_xor_sync(0xffffffffu, x[e], 2));            // xor 4
            x[e] = fmax_nan(x[e], __shfl_xor_sync(0xffffffffu, x[e], 1));            // xor 2
        }
        const int row = m0 + r0 + 8 * h;
        if (q == 0 && row < p.M) p.C[row] = fmax_nan(x[0], x[1]) * __ldg(p.row_scale + row);  // xor 1, lane 0
    }
}

// Epilogue of tile t: C = acc * out_scale + bias (EX: C = z + s * (acc * out_scale + bias), s and z optional; each thread
// reads its z elements before it writes the same C elements, so z may alias C; ROWMAX: gemm3x_rowmax_epilogue).
// acc[4j + {0,1}] = (row r0, cols 8j + 2q + {0,1}), acc[4j + {2,3}] = (row r0 + 8, same cols).
template <bool EX, bool ROWMAX>
__device__ __forceinline__ void gemm3x_epilogue(const Gemm3xParams &p, const float (&acc)[64], int t, int n_tiles, int r0, int q,
                                                float out_scale) {
    const int m0 = (t / n_tiles) * kGM, n0 = (t % n_tiles) * kGN;
    if (ROWMAX) {
        gemm3x_rowmax_epilogue(p, acc, m0, r0, q, out_scale);
        return;
    }
    const bool pair = (p.ldc & 1) == 0 && (reinterpret_cast<uintptr_t>(p.C) & 7) == 0;
#pragma unroll
    for (int j = 0; j < 16; ++j) {
        const int col = n0 + 8 * j + 2 * q;
        if (col >= p.N) continue;
        const bool two = col + 1 < p.N;
        const float b0 = p.bias ? __ldg(p.bias + col) : 0.f, b1 = (p.bias && two) ? __ldg(p.bias + col + 1) : 0.f;
#pragma unroll
        for (int h = 0; h < 2; ++h) {
            const int row = m0 + r0 + 8 * h;
            if (row >= p.M) continue;
            float *dst = p.C + (int64_t)row * p.ldc + col;
            float v0 = acc[4 * j + 2 * h] * out_scale + b0, v1 = acc[4 * j + 2 * h + 1] * out_scale + b1;
            if (EX) {
                if (p.col_scale) v0 = __ldg(p.col_scale + col) * v0, v1 = two ? __ldg(p.col_scale + col + 1) * v1 : v1;
                if (p.Z) {
                    const float *z = p.Z + (int64_t)row * p.ldz + col;
                    v0 = z[0] + v0, v1 = two ? z[1] + v1 : v1;
                }
            }
            if (two && pair) {
                *reinterpret_cast<float2 *>(dst) = make_float2(v0, v1);
            } else {
                dst[0] = v0;
                if (two) dst[1] = v1;
            }
        }
    }
}

// Keeps the register A operands of a waited-for wgmma group allocated up to this point.  wgmma reads them after it
// issues, but ptxas hands their registers to values computed under the MMA (the next k-block's fragments) unless they
// are read again after the wait.  This is that read: stores under a predicate that is never true (`never`, false on every
// launch), one issue slot per four registers.
__device__ __forceinline__ void wgmma_hold(const uint32_t (&a)[4][4], bool never) {
#pragma unroll
    for (int kk = 0; kk < 4; ++kk)
        asm volatile("{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %4, 0;\n\t@p st.shared.v4.b32 [%5], {%0, %1, %2, %3};\n\t}" ::"r"(a[kk][0]),
                     "r"(a[kk][1]), "r"(a[kk][2]), "r"(a[kk][3]), "r"((int)never), "r"(0u)
                     : "memory");
}

// The consumer loop of gemm3x_kernel, with the input activation fixed at compile time.
template <bool F16, bool SPLIT_W, bool EX, bool ROWMAX, int ACT>
__device__ __forceinline__ void gemm3x_consume(const Gemm3xParams &p, uint8_t *smem, uint64_t *full, uint64_t *empty, int tiles,
                                               int n_tiles, int kblocks, int r0, int q, int lane, float a_scale, float out_scale) {
    using S = Gemm3xShape<F16>;
    // One k-block ahead, across tile boundaries: after issuing k-block j's wgmma group, wait for k-block j + 1's stage
    // (k-block 0 of the CTA's next tile after a tile's last one) and split its fragments into the other register set;
    // when j is a tile's k-block 0, the previous tile's epilogue runs there too.  Only then wait for the group, release
    // its stage and add d to acc.  The group's fragments are held to that wait (wgmma_hold), so the next k-block's split
    // never lands in a register that an in-flight wgmma still reads.
    float d[64], acc[64];  // d: the k-block's product (tensor-core accumulation), acc: the tile's sum
    uint32_t ahi[4][4], alo[4][4], nhi[4][4], nlo[4][4];
#pragma unroll
    for (int i = 0; i < 64; ++i) acc[i] = 0.f;
    int t = blockIdx.x, kb = 0, s = 0;
    uint32_t ph = 0;
    if (t >= tiles) return;
    gemm3x_stage_in<F16, SPLIT_W>(smem, full, 0, r0, q, ACT, a_scale, ahi, alo);
    for (;;) {  // k-block kb of tile t, from stage s, fragments in ahi / alo
        gemm3x_issue<F16>(d, ahi, alo, smem + s * S::kStageBytes);
        const int ns = s + 1 == S::kStages ? 0 : s + 1;
        const uint32_t nph = ns == 0 ? ph ^ 1 : ph;
        const bool last = kb + 1 == kblocks;
        const int nt = last ? t + (int)gridDim.x : t;
        const bool more = nt < tiles;
        if (kb == 0 && t != (int)blockIdx.x) {
            gemm3x_epilogue<EX, ROWMAX>(p, acc, t - (int)gridDim.x, n_tiles, r0, q, out_scale);
#pragma unroll
            for (int i = 0; i < 64; ++i) acc[i] = 0.f;  // not acc = d below: 0.f + d turns a -0 product into +0
        }
        if (more) gemm3x_stage_in<F16, SPLIT_W>(smem + ns * S::kStageBytes, full + ns, nph, r0, q, ACT, a_scale, nhi, nlo);
        wgmma_wait_all();
        wgmma_hold(ahi, p.ldc < 0), wgmma_hold(alo, p.ldc < 0);
        if (lane == 0) mbar_arrive(empty + s);
#pragma unroll
        for (int i = 0; i < 64; ++i) acc[i] += d[i];
        if (!more) break;
        s = ns, ph = nph;
        t = nt, kb = last ? 0 : kb + 1;
#pragma unroll
        for (int kk = 0; kk < 4; ++kk)
#pragma unroll
            for (int j = 0; j < 4; ++j) ahi[kk][j] = nhi[kk][j], alo[kk][j] = nlo[kk][j];
    }
    gemm3x_epilogue<EX, ROWMAX>(p, acc, t, n_tiles, r0, q, out_scale);
}

// F16: fp16 pieces (W given as a pre-scaled fp16 pair).  !F16: TF32 pieces; SPLIT_W: W arrives raw (fp32) in the W_hi slot
// and the consumer warpgroups split it in place into W_hi / W_lo with the arithmetic of sdetr_split_tf32_pair.  EX: the
// epilogue also applies the per-column scale and the residual of Gemm3xParams (instances without it compile as before).
// ROWMAX: one n-tile (N <= 128), and the epilogue writes one value per row (gemm3x_rowmax_epilogue) instead of the tile.
template <bool F16, bool SPLIT_W, bool EX = false, bool ROWMAX = false>
__global__ void __launch_bounds__(kGThreads, 1)
    gemm3x_kernel(const __grid_constant__ CUtensorMap ma, const __grid_constant__ CUtensorMap mh,
                  const __grid_constant__ CUtensorMap ml, const Gemm3xParams p) {
    using S = Gemm3xShape<F16>;
    extern __shared__ uint8_t smem_raw[];
    uint8_t *smem = reinterpret_cast<uint8_t *>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~uintptr_t(1023));
    uint64_t *full = reinterpret_cast<uint64_t *>(smem + S::kStages * S::kStageBytes);
    uint64_t *empty = full + S::kStages;
    if (threadIdx.x == 0) {
        for (int s = 0; s < S::kStages; ++s) mbar_init(full + s, 1), mbar_init(empty + s, 8);  // 8 consumer warps release
        asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
    }
    __syncthreads();
    const int n_tiles = (p.N + kGN - 1) / kGN, tiles = n_tiles * ((p.M + kGM - 1) / kGM), kblocks = p.K / S::kK;
    const int wg = threadIdx.x >> 7, tid = threadIdx.x & 127;

    if (wg == 0) {  // ---- producer
        asm volatile("setmaxnreg.dec.sync.aligned.u32 40;");
        if (tid == 0) {
            int s = 0;
            uint32_t ph = 0;
            for (int t = blockIdx.x; t < tiles; t += gridDim.x) {
                const int m0 = (t / n_tiles) * kGM, n0 = (t % n_tiles) * kGN;
                for (int kb = 0; kb < kblocks; ++kb) {
                    mbar_wait(empty + s, ph ^ 1);
                    uint8_t *st = smem + s * S::kStageBytes;
                    mbar_expect_tx(full + s, (S::kABoxes + (SPLIT_W ? 1 : 2)) * kGBox);
#pragma unroll
                    for (int b = 0; b < S::kABoxes; ++b) tma_load_2d(&ma, full + s, st + b * kGBox, kb * S::kK + b * 32, m0);
                    tma_load_2d(&mh, full + s, st + S::kABoxes * kGBox, kb * S::kK, n0);
                    if (!SPLIT_W) tma_load_2d(&ml, full + s, st + (S::kABoxes + 1) * kGBox, kb * S::kK, n0);
                    if (++s == S::kStages) s = 0, ph ^= 1;
                }
            }
        }
        return;
    }

    // ---- consumers: warpgroup wg owns tile rows [64 (wg - 1), 64 wg)
    asm volatile("setmaxnreg.inc.sync.aligned.u32 232;");
    const int warp = tid >> 5, lane = tid & 31, g = lane >> 2, q = lane & 3;
    const int r0 = (wg - 1) * 64 + warp * 16 + g;  // this thread's fragment rows: r0, r0 + 8
    float a_scale = 1.f, out_scale = 1.f;
    if (F16) {
        a_scale = p.a_scale_dev ? __ldg(p.a_scale_dev) : p.a_scale;
        out_scale = p.a_scale_dev ? 1.f / (a_scale * __ldg(p.w_scale_dev)) : p.out_scale;
    }
    switch (p.act) {  // one copy of the loop per activation keeps its test out of the per-element split
        case 1: gemm3x_consume<F16, SPLIT_W, EX, ROWMAX, 1>(p, smem, full, empty, tiles, n_tiles, kblocks, r0, q, lane, a_scale, out_scale); break;
        case 2: gemm3x_consume<F16, SPLIT_W, EX, ROWMAX, 2>(p, smem, full, empty, tiles, n_tiles, kblocks, r0, q, lane, a_scale, out_scale); break;
        default: gemm3x_consume<F16, SPLIT_W, EX, ROWMAX, 0>(p, smem, full, empty, tiles, n_tiles, kblocks, r0, q, lane, a_scale, out_scale);
    }
}

// ---- host side: tensor-map encoder through the runtime's driver entry point (no -lcuda) ------------------------------
typedef CUresult (*EncodeTiledFn)(CUtensorMap *, CUtensorMapDataType, cuuint32_t, void *, const cuuint64_t *, const cuuint64_t *,
                                  const cuuint32_t *, const cuuint32_t *, CUtensorMapInterleave, CUtensorMapSwizzle,
                                  CUtensorMapL2promotion, CUtensorMapFloatOOBfill);

inline EncodeTiledFn get_encode() {
    static EncodeTiledFn fn = nullptr;
    if (!fn) {
        void *p = nullptr;
        cudaDriverEntryPointQueryResult q;
        if (cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &p, cudaEnableDefault, &q) == cudaSuccess &&
            q == cudaDriverEntryPointSuccess)
            fn = reinterpret_cast<EncodeTiledFn>(p);
    }
    return fn;
}

// 2-D tensor (rows, cols) of `elem_bytes`-wide elements with row stride ld (elements); box = (box_cols, box_rows);
// box_cols * elem_bytes must be 128 (one SWIZZLE_128B row).  Out-of-range rows / columns of a box read as zero.
inline bool make_map_2d(CUtensorMap *m, CUtensorMapDataType dt, int elem_bytes, const void *base, int64_t rows, int64_t cols,
                        int64_t ld, int box_cols, int box_rows) {
    EncodeTiledFn enc = get_encode();
    if (!enc) return false;
    const cuuint64_t dims[2] = {(cuuint64_t)cols, (cuuint64_t)rows};
    const cuuint64_t strides[1] = {(cuuint64_t)ld * (cuuint64_t)elem_bytes};
    const cuuint32_t box[2] = {(cuuint32_t)box_cols, (cuuint32_t)box_rows};
    const cuuint32_t estr[2] = {1, 1};
    return enc(m, dt, 2, const_cast<void *>(base), dims, strides, box, estr, CU_TENSOR_MAP_INTERLEAVE_NONE,
               CU_TENSOR_MAP_SWIZZLE_128B, CU_TENSOR_MAP_L2_PROMOTION_L2_256B, CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE) == CUDA_SUCCESS;
}

// A (M,K) fp32 with row pitch lda; W maps made by the caller (F16: fp16 boxes of 64 x 128, else fp32 boxes of 32 x 128)
template <bool F16, bool SPLIT_W, bool EX = false, bool ROWMAX = false>
inline int launch_gemm3x(const float *A, int64_t lda, const CUtensorMap &mh, const CUtensorMap &ml, const Gemm3xParams &p,
                         sdetr_stream_t stream, const char *what) {
    using S = Gemm3xShape<F16>;
    CUtensorMap ma;
    SDETR_REQUIRE(make_map_2d(&ma, CU_TENSOR_MAP_DATA_TYPE_FLOAT32, 4, A, p.M, p.K, lda, 32, kGM), SDETR_ERR_CUDA,
                  "%s: cuTensorMapEncodeTiled failed", what);
    static PerDeviceOnce once;
    SDETR_OPT_IN_SMEM(once, (gemm3x_kernel<F16, SPLIT_W, EX, ROWMAX>), S::kSmem, what);
    const int tiles = ((p.N + kGN - 1) / kGN) * ((p.M + kGM - 1) / kGM), ctas = persistent_ctas();
    gemm3x_kernel<F16, SPLIT_W, EX, ROWMAX><<<tiles < ctas ? tiles : ctas, kGThreads, S::kSmem, (cudaStream_t)stream>>>(ma, mh, ml, p);
    return check_launch(what);
}

}  // namespace sdetr
