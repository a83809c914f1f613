// Encoder FFN -- sdetr_ffn_fused_layernorm:   y = LayerNorm(x + linear2(ReLU(linear1(x))))
// (reference models/bricks/salience_transformer.py:347-351 `forward_ffn` + :391 `norm2`; C = 256, any hidden width % 128 == 0).
//
// One persistent sm_90a kernel keeps the hidden activations on chip: only the weights stream from L2.  The arithmetic is
// that of sdetr_gemm_f16x3_pre applied twice (3xFP16 error-compensated products, exact power-of-two scalings, every
// 64-wide k-block's tensor-core product added into the fp32 sum with a round-to-nearest add):
//   H = acc1 * 2^-(4+s1) + b1  ->  ReLU  ->  x16  ->  fp16 hi / lo        per 64-wide hidden chunk, in shared memory
//   OUT += H . W2[:, chunk]^T                                             fp32 registers, 64 rows x 256 per warpgroup
//   y = LayerNorm(x + OUT * 2^-(4+s2) + b2) * gamma + beta                (or y = OUT * 2^-(4+s2) + b2 without gamma / beta)
//
// Work: a unit is one (128-row panel, hidden chunk); CTA i of G takes units [U i / G, U (i+1) / G) of U = panels * chunks,
// so small layers still fill the GPU.  A panel whose chunks all fall to one CTA is finished in that CTA's epilogue (x may
// alias y: only that CTA reads those rows).  A panel shared by several CTAs gets per-CTA raw sums in the workspace; a
// second launch (ffn_finish_kernel) adds them in CTA order and applies bias, residual and LayerNorm.  No atomics: the
// result is bit-reproducible at a given grid.
//
// CTA: warpgroup 0, one thread, is the TMA producer of a ring of 16 KB weight stages: per chunk 4 stages of W1 (hi + lo
// of 64 hidden rows x 64 k, k-blocks 0-3), then W2 hi and W2 lo of output columns 0-127, then of 128-255 (128 x 64 k each).
// Warpgroups 1 and 2 split the panel by rows (64 each) and both consume every stage, so each weight byte read from L2
// feeds 128 rows.  Per chunk a warpgroup computes linear1 for its rows (m64n64, x hi / lo read from shared memory, where
// it was split once per panel), writes H as hi / lo fp16 into its own H tile, and runs linear2 into all 256 output columns
// (two m64n128 groups, H from shared memory).  No warpgroup reads the other's x rows or H, so the two synchronise only
// through the weight ring and drift apart freely: one's H epilogue overlaps the other's tensor work.  Each output row sits
// in one quad of lanes, so LayerNorm reduces with quad shuffles.  Registers: setmaxnreg moves them from the producer
// warpgroup (24) to the consumers (240 each); 192 accumulators are live at most.
#include "wgmma.cuh"

namespace sdetr {

constexpr int kFD = 256;                           // model width: K of linear1, N of linear2
constexpr int kFM = 128;                           // rows of a panel: 64 per consumer warpgroup
constexpr int kFC = 64;                            // hidden columns of a chunk
constexpr int kFXTile = kFM * 128;                 // 16 KB: 128 rows x 64 fp16, SWIZZLE_128B
constexpr int kFXBytes = 2 * (kFD / 64) * kFXTile; // x hi, x lo: 4 k-block tiles each
constexpr int kFHTile = 64 * 128;                  // 8 KB: 64 rows x 64 fp16
constexpr int kFHBytes = 2 * kFHTile;              // one warpgroup's H chunk: hi tile, lo tile
constexpr int kFStages = 4;                        // of kGBox = 16 KB
constexpr int kFSlot = kFM * kFD;                  // floats of one partial panel in the workspace
constexpr int kFSmem = kFXBytes + 2 * kFHBytes + kFStages * kGBox + 1024 /* alignment */ + 128 /* barriers */;

struct FfnParams {
    const float *x;  // may alias y
    int64_t ldx;
    const float *b1, *b2, *gamma, *beta;
    float eps, out1, out2;  // out1, out2: 1 / (kActScale * w_scale) of linear1, linear2
    int M, chunks, units;
    float *part;  // CTA i's partial panels: slot 2i (its first panel) and 2i + 1 (its last)
    float *y;
};

__host__ __device__ inline int ffn_range_lo(int i, int units, int ctas) { return (int)((int64_t)units * i / ctas); }

__device__ __forceinline__ void proxy_fence_and_sync(int bar) {
    asm volatile("fence.proxy.async.shared::cta;" ::: "memory");  // generic-proxy writes -> wgmma operand reads
    named_bar_sync(bar, 128);
}
__device__ __forceinline__ void st_shared_u32(uint32_t addr, uint32_t v) {
    asm volatile("st.shared.u32 [%0], %1;" ::"r"(addr), "r"(v) : "memory");
}
__device__ __forceinline__ void st_shared_v2(uint32_t addr, uint2 v) {
    asm volatile("st.shared.v2.u32 [%0], {%1, %2};" ::"r"(addr), "r"(v.x), "r"(v.y) : "memory");
}

__global__ void __launch_bounds__(kGThreads, 1)
    ffn_fused_kernel(const __grid_constant__ CUtensorMap m1h, const __grid_constant__ CUtensorMap m1l,
                     const __grid_constant__ CUtensorMap m2h, const __grid_constant__ CUtensorMap m2l, const FfnParams p) {
    extern __shared__ uint8_t smem_raw[];
    uint8_t *smem = reinterpret_cast<uint8_t *>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~uintptr_t(1023));
    uint8_t *xs = smem, *hs = smem + kFXBytes, *ring = hs + 2 * kFHBytes;
    uint64_t *full = reinterpret_cast<uint64_t *>(ring + kFStages * kGBox), *empty = full + kFStages;
    if (threadIdx.x == 0) {
        for (int s = 0; s < kFStages; ++s) mbar_init(full + s, 1), mbar_init(empty + s, 8);  // 8 consumer warps release
        asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
    }
    __syncthreads();
    const int lo = ffn_range_lo(blockIdx.x, p.units, gridDim.x), hi = ffn_range_lo(blockIdx.x + 1, p.units, gridDim.x);
    const int wg = threadIdx.x >> 7, tid = threadIdx.x & 127;

    if (wg == 0) {  // ---- producer: 8 stages per chunk, so a W2 hi / lo pair always lands in stages (0, 1) or (2, 3)
        asm volatile("setmaxnreg.dec.sync.aligned.u32 24;");
        if (tid == 0) {
            int s = 0;
            uint32_t ph = 0;
            for (int u = lo; u < hi; ++u) {
                const int h0 = (u % p.chunks) * kFC;
                for (int t = 0; t < 8; ++t) {
                    mbar_wait(empty + s, ph ^ 1);
                    uint8_t *st = ring + s * kGBox;
                    mbar_expect_tx(full + s, kGBox);
                    if (t < 4) {  // W1 rows [h0, h0 + 64), k-block t: hi, lo
                        tma_load_2d(&m1h, full + s, st, t * 64, h0);
                        tma_load_2d(&m1l, full + s, st + kFHTile, t * 64, h0);
                    } else {      // W2 rows (output columns) [128 half, +128), k-block h0 of the hidden width: hi, then lo
                        tma_load_2d((t & 1) ? &m2l : &m2h, full + s, st, h0, ((t - 4) >> 1) * 128);
                    }
                    if (++s == kFStages) s = 0, ph ^= 1;
                }
            }
        }
        return;
    }

    // ---- consumers: warpgroup cw = wg - 1 owns rows [64 cw, 64 cw + 64) of every panel, all 256 output columns
    asm volatile("setmaxnreg.inc.sync.aligned.u32 240;");
    const int cw = wg - 1, bar = 1 + cw;
    const int warp = tid >> 5, lane = tid & 31, g = lane >> 2, q = lane & 3;
    const int r0 = warp * 16 + g;  // this thread's fragment rows within the warpgroup's 64: r0, r0 + 8
    const uint32_t ah = smem_u32(hs + cw * kFHBytes), al = ah + kFHTile;  // this warpgroup's H tile: hi, lo
    const uint32_t xsa = smem_u32(xs), xh0 = xsa + cw * kFHTile, xl0 = xh0 + kFXBytes / 2;  // rows 64 cw.. of the x tiles
    int s = 0;
    uint32_t ph = 0;
    float acc[128], d[64], acc1[32], d1[32];
    for (int u = lo; u < hi;) {
        const int pnl = u / p.chunks, c_begin = u % p.chunks, c_end = min(p.chunks, c_begin + (hi - u));
        const int64_t m0 = (int64_t)pnl * kFM + 64 * cw;  // the warpgroup's first row
        // its x rows -> x16, hi / lo fp16, swizzled k-block tiles (its readers of the previous panel passed the last
        // chunk's barrier)
        for (int i = tid; i < 64 * kFD / 4; i += 128) {
            const int r = i >> 6, c4 = i & 63, rt = 64 * cw + r;
            float4 v = make_float4(0.f, 0.f, 0.f, 0.f);
            if (m0 + r < p.M) v = *reinterpret_cast<const float4 *>(p.x + (m0 + r) * p.ldx + 4 * c4);
            uint2 h, l;
            split2(v.x * kActScale, v.y * kActScale, h.x, l.x);
            split2(v.z * kActScale, v.w * kActScale, h.y, l.y);
            const int off = (c4 >> 4) * kFXTile + rt * 128 + ((((c4 & 15) >> 1) ^ (rt & 7)) << 4) + (c4 & 1) * 8;
            st_shared_v2(xsa + off, h);
            st_shared_v2(xsa + kFXBytes / 2 + off, l);
        }
        proxy_fence_and_sync(bar);
#pragma unroll
        for (int i = 0; i < 128; ++i) acc[i] = 0.f;
        for (int c = c_begin; c < c_end; ++c) {
            // linear1: H[:, 64 c .. +64), K = 256 in 4 k-blocks
#pragma unroll
            for (int i = 0; i < 32; ++i) acc1[i] = 0.f;
            for (int kb = 0; kb < 4; ++kb) {
                mbar_wait(full + s, ph);
                const uint32_t bh = smem_u32(ring + s * kGBox), bl = bh + kFHTile;
                const uint32_t xh = xh0 + kb * kFXTile, xl = xl0 + kb * kFXTile;
                wgmma_fence();
#pragma unroll
                for (int kk = 0; kk < 4; ++kk) {
                    wgmma_f16_ss_n64(d1, wgmma_desc(xl + kk * 32), wgmma_desc(bh + kk * 32), kk);
                    wgmma_f16_ss_n64(d1, wgmma_desc(xh + kk * 32), wgmma_desc(bl + kk * 32), 1);
                    wgmma_f16_ss_n64(d1, wgmma_desc(xh + kk * 32), wgmma_desc(bh + kk * 32), 1);
                }
                wgmma_commit();
                wgmma_wait_all();
                if (lane == 0) mbar_arrive(empty + s);
                if (++s == kFStages) s = 0, ph ^= 1;
#pragma unroll
                for (int i = 0; i < 32; ++i) acc1[i] += d1[i];
            }
            // every warp of the warpgroup has finished its linear2 of the previous chunk: the H tile may be rewritten
            named_bar_sync(bar, 128);
            // H = acc1 * out1 + b1 -> ReLU -> x16 -> hi / lo
#pragma unroll
            for (int j = 0; j < 8; ++j) {
                const int col = c * kFC + 8 * j + 2 * q;
                const float bb0 = __ldg(p.b1 + col), bb1 = __ldg(p.b1 + col + 1);
#pragma unroll
                for (int h = 0; h < 2; ++h) {
                    const int r = r0 + 8 * h;
                    const float v0 = relu_nan(acc1[4 * j + 2 * h] * p.out1 + bb0) * kActScale;
                    const float v1 = relu_nan(acc1[4 * j + 2 * h + 1] * p.out1 + bb1) * kActScale;
                    uint32_t vh, vl;
                    split2(v0, v1, vh, vl);
                    const int off = r * 128 + ((j ^ (r & 7)) << 4) + 4 * q;
                    st_shared_u32(ah + off, vh);
                    st_shared_u32(al + off, vl);
                }
            }
            proxy_fence_and_sync(bar);
            // linear2: OUT[:, 128 half .. +128) += H(chunk c) . W2^T, one k-block; W2 hi in stage s, lo in stage s + 1
#pragma unroll
            for (int half = 0; half < 2; ++half) {
                mbar_wait(full + s, ph);
                mbar_wait(full + s + 1, ph);
                const uint32_t bh = smem_u32(ring + s * kGBox), bl = bh + kGBox;
                wgmma_fence();
#pragma unroll
                for (int kk = 0; kk < 4; ++kk) {
                    wgmma_f16_ss(d, wgmma_desc(al + kk * 32), wgmma_desc(bh + kk * 32), kk);
                    wgmma_f16_ss(d, wgmma_desc(ah + kk * 32), wgmma_desc(bl + kk * 32), 1);
                    wgmma_f16_ss(d, wgmma_desc(ah + kk * 32), wgmma_desc(bh + kk * 32), 1);
                }
                wgmma_commit();
                wgmma_wait_all();
                if (lane == 0) mbar_arrive(empty + s), mbar_arrive(empty + s + 1);
                if ((s += 2) == kFStages) s = 0, ph ^= 1;
#pragma unroll
                for (int i = 0; i < 64; ++i) acc[64 * half + i] += d[i];
            }
        }
        // epilogue: acc[64 half + 4j + {0,1}] = (row r0, cols 128 half + 8j + 2q + {0,1}), acc[64 half + 4j + {2,3}] =
        // (row r0 + 8, same cols)
        if (c_begin == 0 && c_end == p.chunks) {
            if (p.gamma) {
                // row sums and squares per 128-column half, quad-reduced, then the halves added: the order of the
                // kernel's earlier column split across the warpgroups, so its LayerNorm is unchanged to the bit
                float sum[2][2] = {{0.f, 0.f}, {0.f, 0.f}};
#pragma unroll
                for (int half = 0; half < 2; ++half)
#pragma unroll
                    for (int h = 0; h < 2; ++h) {
                        const int64_t row = m0 + r0 + 8 * h;
#pragma unroll
                        for (int j = 0; j < 16; ++j) {
                            const int col = half * 128 + 8 * j + 2 * q;
                            const float bb0 = p.b2 ? __ldg(p.b2 + col) : 0.f, bb1 = p.b2 ? __ldg(p.b2 + col + 1) : 0.f;
                            float2 xv = make_float2(0.f, 0.f);
                            if (row < p.M) xv = *reinterpret_cast<const float2 *>(p.x + row * p.ldx + col);
                            float &a0 = acc[64 * half + 4 * j + 2 * h], &a1 = acc[64 * half + 4 * j + 2 * h + 1];
                            a0 = xv.x + (a0 * p.out2 + bb0);
                            a1 = xv.y + (a1 * p.out2 + bb1);
                            sum[half][h] += a0 + a1;
                        }
                    }
                float mean[2], rstd[2], ss[2][2] = {{0.f, 0.f}, {0.f, 0.f}};
#pragma unroll
                for (int h = 0; h < 2; ++h) {
#pragma unroll
                    for (int half = 0; half < 2; ++half) {
                        sum[half][h] += __shfl_xor_sync(0xffffffffu, sum[half][h], 1);
                        sum[half][h] += __shfl_xor_sync(0xffffffffu, sum[half][h], 2);
                    }
                    mean[h] = (sum[0][h] + sum[1][h]) / (float)kFD;
                }
#pragma unroll
                for (int half = 0; half < 2; ++half)
#pragma unroll
                    for (int j = 0; j < 16; ++j)
#pragma unroll
                        for (int h = 0; h < 2; ++h) {
                            const float e0 = acc[64 * half + 4 * j + 2 * h] - mean[h], e1 = acc[64 * half + 4 * j + 2 * h + 1] - mean[h];
                            ss[half][h] += e0 * e0 + e1 * e1;
                        }
#pragma unroll
                for (int h = 0; h < 2; ++h) {
#pragma unroll
                    for (int half = 0; half < 2; ++half) {
                        ss[half][h] += __shfl_xor_sync(0xffffffffu, ss[half][h], 1);
                        ss[half][h] += __shfl_xor_sync(0xffffffffu, ss[half][h], 2);
                    }
                    rstd[h] = rsqrtf((ss[0][h] + ss[1][h]) / (float)kFD + p.eps);
                }
#pragma unroll
                for (int h = 0; h < 2; ++h) {
                    const int64_t row = m0 + r0 + 8 * h;
                    if (row >= p.M) continue;
#pragma unroll
                    for (int half = 0; half < 2; ++half)
#pragma unroll
                        for (int j = 0; j < 16; ++j) {
                            const int col = half * 128 + 8 * j + 2 * q;
                            const float2 gm = *reinterpret_cast<const float2 *>(p.gamma + col);
                            const float2 bt = *reinterpret_cast<const float2 *>(p.beta + col);
                            *reinterpret_cast<float2 *>(p.y + row * kFD + col) =
                                make_float2((acc[64 * half + 4 * j + 2 * h] - mean[h]) * rstd[h] * gm.x + bt.x,
                                            (acc[64 * half + 4 * j + 2 * h + 1] - mean[h]) * rstd[h] * gm.y + bt.y);
                        }
                }
            } else {
#pragma unroll
                for (int h = 0; h < 2; ++h) {
                    const int64_t row = m0 + r0 + 8 * h;
                    if (row >= p.M) continue;
#pragma unroll
                    for (int half = 0; half < 2; ++half)
#pragma unroll
                        for (int j = 0; j < 16; ++j) {
                            const int col = half * 128 + 8 * j + 2 * q;
                            const float bb0 = p.b2 ? __ldg(p.b2 + col) : 0.f, bb1 = p.b2 ? __ldg(p.b2 + col + 1) : 0.f;
                            *reinterpret_cast<float2 *>(p.y + row * kFD + col) =
                                make_float2(acc[64 * half + 4 * j + 2 * h] * p.out2 + bb0, acc[64 * half + 4 * j + 2 * h + 1] * p.out2 + bb1);
                        }
                }
            }
        } else {  // raw partial sums of a shared panel
            float *dst = p.part + (int64_t)(2 * blockIdx.x + (u == lo ? 0 : 1)) * kFSlot + 64 * cw * kFD;
#pragma unroll
            for (int h = 0; h < 2; ++h)
#pragma unroll
                for (int half = 0; half < 2; ++half)
#pragma unroll
                    for (int j = 0; j < 16; ++j)
                        *reinterpret_cast<float2 *>(dst + (r0 + 8 * h) * kFD + half * 128 + 8 * j + 2 * q) =
                            make_float2(acc[64 * half + 4 * j + 2 * h], acc[64 * half + 4 * j + 2 * h + 1]);
        }
        u += c_end - c_begin;
    }
}

// Rows of panels shared by several CTAs: OUT = the CTAs' partial sums in CTA order, y = LayerNorm(x + OUT * out2 + b2) (or
// OUT * out2 + b2 without gamma / beta).  One warp per row; rows of panels finished in the fused kernel return at once.
__global__ void __launch_bounds__(256) ffn_finish_kernel(const FfnParams p, int ctas) {
    const int lane = threadIdx.x & 31;
    const int64_t row = (int64_t)blockIdx.x * 8 + (threadIdx.x >> 5);
    if (row >= p.M) return;
    const int pnl = (int)(row / kFM), u0 = pnl * p.chunks, u1 = u0 + p.chunks - 1;
    int i0 = (int)((int64_t)u0 * ctas / p.units);
    while (ffn_range_lo(i0 + 1, p.units, ctas) <= u0) ++i0;
    int i1 = i0;
    while (ffn_range_lo(i1 + 1, p.units, ctas) <= u1) ++i1;
    if (i0 == i1) return;
    float4 v[2] = {make_float4(0.f, 0.f, 0.f, 0.f), make_float4(0.f, 0.f, 0.f, 0.f)};
    for (int i = i0; i <= i1; ++i) {
        const int first = ffn_range_lo(i, p.units, ctas) / p.chunks;
        const float *src = p.part + (int64_t)(2 * i + (pnl == first ? 0 : 1)) * kFSlot + (row % kFM) * kFD;
#pragma unroll
        for (int k = 0; k < 2; ++k) {
            const float4 a = *reinterpret_cast<const float4 *>(src + k * 128 + lane * 4);
            v[k].x += a.x, v[k].y += a.y, v[k].z += a.z, v[k].w += a.w;
        }
    }
    float s = 0.f;
#pragma unroll
    for (int k = 0; k < 2; ++k) {
        const int c = k * 128 + lane * 4;
        const float4 b = p.b2 ? ldg_f4(p.b2 + c) : make_float4(0.f, 0.f, 0.f, 0.f);
        v[k].x = v[k].x * p.out2 + b.x, v[k].y = v[k].y * p.out2 + b.y, v[k].z = v[k].z * p.out2 + b.z, v[k].w = v[k].w * p.out2 + b.w;
        if (p.gamma) {
            const float4 r = *reinterpret_cast<const float4 *>(p.x + row * p.ldx + c);
            v[k].x += r.x, v[k].y += r.y, v[k].z += r.z, v[k].w += r.w;
        }
        s += (v[k].x + v[k].y) + (v[k].z + v[k].w);
    }
    if (!p.gamma) {
#pragma unroll
        for (int k = 0; k < 2; ++k) *reinterpret_cast<float4 *>(p.y + row * kFD + k * 128 + lane * 4) = v[k];
        return;
    }
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) s += __shfl_xor_sync(0xffffffffu, s, o);
    const float mean = s / (float)kFD;
    float ss = 0.f;
#pragma unroll
    for (int k = 0; k < 2; ++k) {
        const float dx = v[k].x - mean, dy = v[k].y - mean, dz = v[k].z - mean, dw = v[k].w - mean;
        ss += (dx * dx + dy * dy) + (dz * dz + dw * dw);
    }
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) ss += __shfl_xor_sync(0xffffffffu, ss, o);
    const float rstd = rsqrtf(ss / (float)kFD + p.eps);
#pragma unroll
    for (int k = 0; k < 2; ++k) {
        const int c = k * 128 + lane * 4;
        const float4 gm = ldg_f4(p.gamma + c), bt = ldg_f4(p.beta + c);
        float4 o;
        o.x = (v[k].x - mean) * rstd * gm.x + bt.x, o.y = (v[k].y - mean) * rstd * gm.y + bt.y;
        o.z = (v[k].z - mean) * rstd * gm.z + bt.z, o.w = (v[k].w - mean) * rstd * gm.w + bt.w;
        *reinterpret_cast<float4 *>(p.y + row * kFD + c) = o;
    }
}

}  // namespace sdetr

using namespace sdetr;

extern "C" int64_t sdetr_ffn_fused_workspace_floats(int M, int hidden) {
    if (M <= 0 || hidden <= 0 || hidden % 128) return 0;
    return (int64_t)M * (hidden + kFD);  // an upper bound: the kernel uses at most two 128 x 256 slots per CTA
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
    SDETR_REQUIRE(make_map_2d(&m1h, CU_TENSOR_MAP_DATA_TYPE_FLOAT16, 2, w1_hi, hidden, kFD, kFD, 64, kFC) &&
                      make_map_2d(&m1l, CU_TENSOR_MAP_DATA_TYPE_FLOAT16, 2, w1_lo, hidden, kFD, kFD, 64, kFC) &&
                      make_map_2d(&m2h, CU_TENSOR_MAP_DATA_TYPE_FLOAT16, 2, w2_hi, kFD, hidden, hidden, 64, kGN) &&
                      make_map_2d(&m2l, CU_TENSOR_MAP_DATA_TYPE_FLOAT16, 2, w2_lo, kFD, hidden, hidden, 64, kGN),
                  SDETR_ERR_CUDA, "ffn_fused: cuTensorMapEncodeTiled failed");
    const int chunks = hidden / kFC, units = ((M + kFM - 1) / kFM) * chunks;
    int ctas = persistent_ctas();
    if (ctas > units) ctas = units;
    // The grid is narrowed to the CTAs whose two 128 x 256 partial panels fit in the workspace of M * (hidden + 256) floats.
    // That only binds for small M: at hidden 2048 it allows about M / 28 CTAs (M = 128: 4), which passes an H100's SM count
    // from about 3800 rows on.
    const int64_t slot_ctas = workspace_floats / (2 * kFSlot);
    if (ctas > slot_ctas) ctas = slot_ctas > 1 ? (int)slot_ctas : 1;
    const FfnParams p{x, ldx, b1, b2, gamma, beta, eps, 1.f / (kActScale * w1_scale), 1.f / (kActScale * w2_scale),
                      M, chunks, units, workspace, y};
    static PerDeviceOnce once;
    SDETR_OPT_IN_SMEM(once, ffn_fused_kernel, kFSmem, "ffn_fused");
    ffn_fused_kernel<<<ctas, kGThreads, kFSmem, (cudaStream_t)stream>>>(m1h, m1l, m2h, m2l, p);
    int rc = check_launch("ffn_fused");
    bool shared_panel = false;  // some CTA's range starts inside a panel
    for (int i = 1; i < ctas && !shared_panel; ++i) shared_panel = ffn_range_lo(i, units, ctas) % chunks != 0;
    if (rc != SDETR_OK || !shared_panel) return rc;
    ffn_finish_kernel<<<(unsigned)((M + 7) / 8), 256, 0, (cudaStream_t)stream>>>(p, ctas);
    return check_launch("ffn_fused/finish");
}
