// Token-layout convolutions (the RepVGG-PluX neck, the ChannelMapper and the ResNet backbone) and the neck's other kernels
// (models/necks/repnet.py:125-245).
//
//   sdetr_conv2d_f16x3            implicit-GEMM convolution (k = 1 or 3, stride 1 or 2, padding k / 2, groups), bias, optional
//                                 residual operand and none / ReLU / SiLU epilogue.  Same 3xFP16 arithmetic as sdetr_gemm_f16x3_scaled: the activation is
//                                 multiplied by a power-of-two device scalar, split into fp16 hi / lo in registers and used as
//                                 the wgmma A operand; the weight arrives as a pre-split pair (scale 2^s, also a device scalar);
//                                 lo.hi + hi.lo + hi.hi per 16-wide k step, and every 64-wide k-block's tensor-core sum is added
//                                 into fp32 registers with round-to-nearest adds.
//   sdetr_conv2d_f16x3_dgrad      its input gradient (stride 1: the same kernel on dY with flipped weights; stride 2: the
//                                 kernel's transposed mode), residual gradient and ReLU mask in the epilogue.
//   sdetr_conv2d_f16x3_wgrad      its weight gradient (split over the pixel range, splits summed in order), with an optional
//                                 per-output-channel scale.
//   sdetr_conv2d_f16x3_split_weight  the fp16 weight pairs of the forward and the input gradient, in one pass.
//   sdetr_context_gate            SqueezeAndExcitation (models/bricks/basic.py:29-54, a GCNet attention pool) + the block's
//                                 residual: out = sigmoid(W2 ReLU(W1 ctx)) * y + x (+ z), ctx = softmax(y . w_mask + b_mask) . y.
//   sdetr_upsample_nearest_concat [nearest(hi) | lo] into one 2C-wide operand (torch's nearest index rule), and its backward.
//
// Operands are token rows: pixel (py, px) of image n, channel c at base + n * pitch + (py * W + px) * ld + c (floats), so a
// level slice of a (b, Nv, C) tensor is a valid operand without a copy.
//
// Convolution tile: 64 output pixels (consecutive in (n, py, px) order) x 64 output channels per CTA of one warpgroup.  The
// k loop runs over taps x 64-channel blocks of the group's input channels; per k-block the CTA copies the 64 x 64 fp32
// activation rows (cp.async, zero-filled where the tap falls outside the map: that is the padding) and the 64 x 64 W_hi /
// W_lo tiles (128-byte swizzle, the layout wgmma reads) into a 3-stage ring.
#include <cuda_fp16.h>
#include <math.h>

#include "wgmma.cuh"

namespace sdetr {

constexpr int kCvM = 64, kCvN = 64, kCvK = 64, kCvStages = 3, kCvThreads = 128;
constexpr int kCvABytes = kCvM * kCvK * 4;  // 16 KB: fp32 activation rows of 256 bytes
constexpr int kCvBBytes = kCvN * kCvK * 2;  // 8 KB: one of W_hi / W_lo, rows of 128 bytes
constexpr int kCvStageBytes = kCvABytes + 2 * kCvBBytes;
constexpr int kCvSmem = kCvStages * kCvStageBytes + 1024 /* alignment */;
constexpr int kActReLU = 1, kActSiLU = 3;  // act codes of the convolution's epilogue (0 none)

struct ConvParams {
    const float *x;
    int64_t x_pitch, ldx;
    const __half *w_hi, *w_lo;  // (Cout, k, k, Cin / groups) row-major
    const float *a_scale, *w_scale, *bias;
    const float *z;  // residual added before the activation (NULL: none); may alias y
    int64_t z_pitch, ldz;
    const float *m;  // ReLU mask source (NULL: none): the output is 0 where m <= 0 (torch's threshold_backward); not y
    int64_t m_pitch, ldm;
    float *y;
    int64_t y_pitch, ldy;
    int H, W, Ho, Wo, M, cin_g, cout_g, ksize, stride, act;
};

__device__ __forceinline__ void cp_async16(void *dst, const void *src, bool ok) {
    asm volatile("cp.async.cg.shared.global [%0], [%1], 16, %2;" ::"r"(smem_u32(dst)), "l"(src), "r"(ok ? 16 : 0) : "memory");
}
__device__ __forceinline__ void cp_async_commit() { asm volatile("cp.async.commit_group;" ::: "memory"); }
__device__ __forceinline__ void cp_async_wait_1() { asm volatile("cp.async.wait_group 1;" ::: "memory"); }
__device__ __forceinline__ float silu(float x) { return x / (1.f + expf(-x)); }

// TRANSPOSED: the input gradient of a stride-2 convolution.  x is dY (H x W), y is dX (Ho x Wo), W the flipped, per-group
// transposed weights (see sdetr_conv2d_f16x3_dgrad); output pixel (oy, ox) with tap (ky, kx) reads x[(oy - pad + ky) / 2,
// (ox - pad + kx) / 2] when both are even and in range, and zero otherwise.
template <bool TRANSPOSED>
__global__ void __launch_bounds__(kCvThreads) conv_f16x3_kernel(const ConvParams p) {
    extern __shared__ uint8_t smem_raw[];
    uint8_t *smem = reinterpret_cast<uint8_t *>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~uintptr_t(1023));
    const int tid = threadIdx.x, m0 = blockIdx.x * kCvM, n0 = blockIdx.y * kCvN;
    const int cin0 = (n0 / p.cout_g) * p.cin_g;
    const int cblocks = p.cin_g / kCvK, kblocks = p.ksize * p.ksize * cblocks, pad = p.ksize >> 1, hwo = p.Ho * p.Wo;
    const int64_t kw = (int64_t)p.ksize * p.ksize * p.cin_g;

    // activation rows this thread copies: tile rows (tid >> 4) + 8 j, 16-byte chunk tid & 15 of each 256-byte row
    const int ac = tid & 15;
    const float *arow[8];
    int iy0[8], ix0[8];
#pragma unroll
    for (int j = 0; j < 8; ++j) {
        const int m = m0 + (tid >> 4) + 8 * j;
        arow[j] = p.x, iy0[j] = -(1 << 28), ix0[j] = 0;  // a row past M: every tap out of bounds -> zeros
        if (m < p.M) {
            const int n = m / hwo, pix = m - n * hwo, oy = pix / p.Wo, ox = pix - oy * p.Wo;
            arow[j] = p.x + (int64_t)n * p.x_pitch + cin0 + ac * 4;
            iy0[j] = oy * (TRANSPOSED ? 1 : p.stride) - pad, ix0[j] = ox * (TRANSPOSED ? 1 : p.stride) - pad;
        }
    }
    auto load_stage = [&](int s, int kb) {
        uint8_t *st = smem + s * kCvStageBytes;
        const int t = kb / cblocks, cb = kb - t * cblocks, ky = t / p.ksize, kx = t - ky * p.ksize;
#pragma unroll
        for (int j = 0; j < 8; ++j) {
            const int r = (tid >> 4) + 8 * j;
            int iy = iy0[j] + ky, ix = ix0[j] + kx;
            bool ok;
            if (TRANSPOSED) {
                ok = ((iy | ix) & 1) == 0 && (unsigned)iy < 2u * p.H && (unsigned)ix < 2u * p.W;
                iy >>= 1, ix >>= 1;
            } else {
                ok = (unsigned)iy < (unsigned)p.H && (unsigned)ix < (unsigned)p.W;
            }
            const float *src = ok ? arow[j] + ((int64_t)iy * p.W + ix) * p.ldx + cb * kCvK : p.x;
            cp_async16(st + r * 256 + ((ac ^ (r & 7)) << 4), src, ok);
        }
#pragma unroll
        for (int j = 0; j < 8; ++j) {  // W_hi rows (j < 4), W_lo rows (j >= 4): 8 16-byte chunks per 128-byte row
            const int i = (tid + 128 * j) & 511, r = i >> 3, c = i & 7;
            const __half *src = (j < 4 ? p.w_hi : p.w_lo) + (int64_t)(n0 + r) * kw + (int64_t)kb * kCvK + c * 8;
            cp_async16(st + kCvABytes + (j >> 2) * kCvBBytes + r * 128 + ((c ^ (r & 7)) << 4), src, true);
        }
    };

    const float a_scale = __ldg(p.a_scale), out_scale = 1.f / (a_scale * __ldg(p.w_scale));
    const int warp = tid >> 5, lane = tid & 31, g = lane >> 2, q = lane & 3, r0 = warp * 16 + g;
    float d[32], acc[32];
#pragma unroll
    for (int i = 0; i < 32; ++i) acc[i] = 0.f;
#pragma unroll
    for (int s = 0; s < kCvStages - 1; ++s) {
        if (s < kblocks) load_stage(s, s);
        cp_async_commit();
    }
    for (int kb = 0; kb < kblocks; ++kb) {
        cp_async_wait_1();
        asm volatile("fence.proxy.async.shared::cta;" ::: "memory");  // cp.async (generic proxy) writes -> wgmma operand reads
        __syncthreads();  // also: every warp is done with the stage the next copy overwrites
        if (kb + kCvStages - 1 < kblocks) load_stage((kb + kCvStages - 1) % kCvStages, kb + kCvStages - 1);
        cp_async_commit();
        const uint8_t *st = smem + (kb % kCvStages) * kCvStageBytes;
        uint32_t ahi[4][4], alo[4][4];
#pragma unroll
        for (int kk = 0; kk < 4; ++kk) {  // m64k16 fragment: (r0, c..c+1), (r0+8, c..c+1), (r0, c+8..c+9), (r0+8, c+8..c+9)
#pragma unroll
            for (int j = 0; j < 4; ++j) {
                const int row = r0 + (j & 1) * 8, col = kk * 16 + 2 * q + (j >> 1) * 8;
                const float2 x =
                    *reinterpret_cast<const float2 *>(st + row * 256 + ((((col >> 2) ^ (row & 7)) << 4) | ((col & 3) << 2)));
                split2(x.x * a_scale, x.y * a_scale, ahi[kk][j], alo[kk][j]);
            }
        }
        wgmma_fence();
        const uint32_t bh = smem_u32(st + kCvABytes), bl = bh + kCvBBytes;
#pragma unroll
        for (int kk = 0; kk < 4; ++kk) {
            wgmma_f16_rs_n64(d, alo[kk], wgmma_desc(bh + kk * 32), kk);
            wgmma_f16_rs_n64(d, ahi[kk], wgmma_desc(bl + kk * 32), 1);
            wgmma_f16_rs_n64(d, ahi[kk], wgmma_desc(bh + kk * 32), 1);
        }
        wgmma_commit();
        wgmma_wait_all();
#pragma unroll
        for (int i = 0; i < 32; ++i) acc[i] += d[i];
    }
    // epilogue: acc[4j + 2h + e] = (tile row r0 + 8h, column 8j + 2q + e)
#pragma unroll
    for (int h = 0; h < 2; ++h) {
        const int m = m0 + r0 + 8 * h;
        if (m >= p.M) continue;
        const int n = m / hwo, pix = m - n * hwo;
        float *dst = p.y + (int64_t)n * p.y_pitch + (int64_t)pix * p.ldy + n0;
        // z is read by the thread that then writes the same two floats of y, so z may alias y
        const float *zr = p.z ? p.z + (int64_t)n * p.z_pitch + (int64_t)pix * p.ldz + n0 : nullptr;
        const float *mr = p.m ? p.m + (int64_t)n * p.m_pitch + (int64_t)pix * p.ldm + n0 : nullptr;
#pragma unroll
        for (int j = 0; j < 8; ++j) {
            const int col = 8 * j + 2 * q;
            float v0 = acc[4 * j + 2 * h] * out_scale + (p.bias ? __ldg(p.bias + n0 + col) : 0.f);
            float v1 = acc[4 * j + 2 * h + 1] * out_scale + (p.bias ? __ldg(p.bias + n0 + col + 1) : 0.f);
            if (zr) {
                const float2 r = *reinterpret_cast<const float2 *>(zr + col);
                v0 += r.x, v1 += r.y;
            }
            if (p.act == kActSiLU) v0 = silu(v0), v1 = silu(v1);
            else if (p.act == kActReLU) v0 = relu_nan(v0), v1 = relu_nan(v1);
            if (mr) {  // a NaN in m lets the value through, a NaN value stays NaN
                const float2 r = *reinterpret_cast<const float2 *>(mr + col);
                if (r.x <= 0.f) v0 = 0.f;
                if (r.y <= 0.f) v1 = 0.f;
            }
            *reinterpret_cast<float2 *>(dst + col) = make_float2(v0, v1);
        }
    }
}

// ---- context gate ---------------------------------------------------------------------------------------------------------
// Three launches, every sum in a fixed order (no atomics): per chunk of kGateChunk pixels the chunk's logit maximum m_c,
// s_c = sum exp(l - m_c) and ctx_c = sum exp(l - m_c) y; per image the chunks combined in chunk order and the gate; then the
// elementwise gate * y + x (+ z).
constexpr int kGateChunk = 128, kGateThreads = 256;

__global__ void __launch_bounds__(kGateThreads) gate_partial_kernel(const float *__restrict__ y, int64_t y_pitch, int64_t ldy,
                                                                    int HW, int C, const float *__restrict__ w_mask,
                                                                    const float *__restrict__ b_mask, int nchunk,
                                                                    float *__restrict__ part /* (b, nchunk, C + 2) */) {
    __shared__ float e[kGateChunk];
    __shared__ float stat[2];
    const int n = blockIdx.y, p0 = blockIdx.x * kGateChunk, np = min(kGateChunk, HW - p0);
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    const float *yb = y + (int64_t)n * y_pitch + (int64_t)p0 * ldy;
    for (int i = warp; i < np; i += kGateThreads / 32) {  // logits: one warp per pixel, lanes over channels
        const float *row = yb + (int64_t)i * ldy;
        float s = 0.f;
        for (int c = lane; c < C; c += 32) s = fmaf(row[c], __ldg(w_mask + c), s);
#pragma unroll
        for (int o = 16; o > 0; o >>= 1) s += __shfl_xor_sync(0xffffffffu, s, o);
        if (lane == 0) e[i] = s + __ldg(b_mask);
    }
    __syncthreads();
    if (threadIdx.x == 0) {
        float m = e[0];
        for (int i = 1; i < np; ++i) m = fmaxf(m, e[i]);
        stat[0] = m;
    }
    __syncthreads();
    const float m = stat[0];
    if (threadIdx.x < np) e[threadIdx.x] = expf(e[threadIdx.x] - m);
    __syncthreads();
    float *out = part + ((int64_t)n * nchunk + blockIdx.x) * (C + 2);
    if (threadIdx.x == 0) {
        float s = 0.f;
        for (int i = 0; i < np; ++i) s += e[i];
        out[C] = m, out[C + 1] = s;
    }
    for (int c = threadIdx.x; c < C; c += kGateThreads) {
        float s = 0.f;
        for (int i = 0; i < np; ++i) s = fmaf(e[i], yb[(int64_t)i * ldy + c], s);
        out[c] = s;
    }
}

// per image: ctx = sum_c ctx_c exp(m_c - M) / sum_c s_c exp(m_c - M); gate = sigmoid(W2 ReLU(W1 ctx))
__global__ void __launch_bounds__(kGateThreads) gate_combine_kernel(const float *__restrict__ part, int nchunk, int C, int R,
                                                                    const float *__restrict__ w1 /* (R, C) */,
                                                                    const float *__restrict__ w2 /* (C, R) */,
                                                                    float *__restrict__ gate /* (b, C) */) {
    extern __shared__ float sh[];  // ctx[C], hidden[R]
    float *ctx = sh, *hid = sh + C;
    const int n = blockIdx.x;
    const float *pb = part + (int64_t)n * nchunk * (C + 2);
    float M = -INFINITY;
    for (int k = 0; k < nchunk; ++k) M = fmaxf(M, pb[(int64_t)k * (C + 2) + C]);
    float S = 0.f;
    for (int k = 0; k < nchunk; ++k) S += pb[(int64_t)k * (C + 2) + C + 1] * expf(pb[(int64_t)k * (C + 2) + C] - M);
    for (int c = threadIdx.x; c < C; c += kGateThreads) {
        float s = 0.f;
        for (int k = 0; k < nchunk; ++k) s = fmaf(pb[(int64_t)k * (C + 2) + c], expf(pb[(int64_t)k * (C + 2) + C] - M), s);
        ctx[c] = s / S;
    }
    __syncthreads();
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    for (int j = warp; j < R; j += kGateThreads / 32) {
        float s = 0.f;
        for (int c = lane; c < C; c += 32) s = fmaf(__ldg(w1 + (int64_t)j * C + c), ctx[c], s);
#pragma unroll
        for (int o = 16; o > 0; o >>= 1) s += __shfl_xor_sync(0xffffffffu, s, o);
        if (lane == 0) hid[j] = relu_nan(s);  // torch's ReLU: a NaN context (a NaN anywhere in the image) stays NaN
    }
    __syncthreads();
    for (int c = threadIdx.x; c < C; c += kGateThreads) {
        float s = 0.f;
        for (int j = 0; j < R; ++j) s = fmaf(__ldg(w2 + (int64_t)c * R + j), hid[j], s);
        gate[(int64_t)n * C + c] = 1.f / (1.f + expf(-s));
    }
}

struct Rows {  // a token-row operand: base + n * pitch + pixel * ld
    const float *p;
    int64_t pitch, ld;
    __device__ __forceinline__ float4 at(int n, int pix, int c) const {
        return *reinterpret_cast<const float4 *>(p + (int64_t)n * pitch + (int64_t)pix * ld + c);
    }
};

__global__ void gate_apply_kernel(Rows y, Rows x, Rows z, const float *__restrict__ gate, int batch, int HW, int C, float *out,
                                  int64_t o_pitch, int64_t ldo) {
    const int c4 = C >> 2;
    const int64_t total = (int64_t)batch * HW * c4;
    for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (int64_t)gridDim.x * blockDim.x) {
        const int c = (int)(i % c4) * 4;
        const int64_t r = i / c4;
        const int n = (int)(r / HW), pix = (int)(r - (int64_t)n * HW);
        const float4 gv = *reinterpret_cast<const float4 *>(gate + (int64_t)n * C + c), yv = y.at(n, pix, c), xv = x.at(n, pix, c);
        float4 o = make_float4(fmaf(gv.x, yv.x, xv.x), fmaf(gv.y, yv.y, xv.y), fmaf(gv.z, yv.z, xv.z), fmaf(gv.w, yv.w, xv.w));
        if (z.p) {
            const float4 zv = z.at(n, pix, c);
            o.x += zv.x, o.y += zv.y, o.z += zv.z, o.w += zv.w;
        }
        *reinterpret_cast<float4 *>(out + (int64_t)n * o_pitch + (int64_t)pix * ldo + c) = o;
    }
}

// ---- nearest upsample + concat ------------------------------------------------------------------------------------------
// torch's nearest rule (UpSampleNearest: nearest_neighbor_compute_source_index): src = min(floor(dst * (float)in / out), in - 1)
__device__ __forceinline__ int nearest_src(int dst, int in, int out) {
    const float scale = (float)in / (float)out;
    return min((int)floorf((float)dst * scale), in - 1);
}

__global__ void upsample_concat_kernel(Rows hi, int Hi, int Wi, Rows lo, int Ho, int Wo, int batch, int C, float *dst,
                                       int64_t d_pitch, int64_t ldd) {
    const int c4 = (2 * C) >> 2, hwo = Ho * Wo;
    const int64_t total = (int64_t)batch * hwo * c4;
    for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (int64_t)gridDim.x * blockDim.x) {
        const int c = (int)(i % c4) * 4;
        const int64_t r = i / c4;
        const int n = (int)(r / hwo), pix = (int)(r - (int64_t)n * hwo);
        float4 v;
        if (c < C) {
            const int oy = pix / Wo, ox = pix - oy * Wo;
            v = hi.at(n, nearest_src(oy, Hi, Ho) * Wi + nearest_src(ox, Wi, Wo), c);
        } else {
            v = lo.at(n, pix, c - C);
        }
        *reinterpret_cast<float4 *>(dst + (int64_t)n * d_pitch + (int64_t)pix * ldd + c) = v;
    }
}

// gradient of the hi half: each source pixel sums its destination range [first_dst(s), first_dst(s + 1)) per axis, rows then
// columns in order (no atomics).  first_dst(s): the first destination whose nearest_src is >= s (nearest_src is monotonic).
__device__ __forceinline__ int first_dst(int s, int in, int out) {
    int lo = 0, hi = out;
    while (lo < hi) {
        const int mid = (lo + hi) >> 1;
        if (nearest_src(mid, in, out) >= s) hi = mid; else lo = mid + 1;
    }
    return lo;
}

__global__ void upsample_concat_backward_kernel(Rows g, int Ho, int Wo, int Hi, int Wi, int batch, int C, float *dst,
                                                int64_t d_pitch, int64_t ldd) {
    const int c4 = C >> 2, hwi = Hi * Wi;
    const int64_t total = (int64_t)batch * hwi * c4;
    for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (int64_t)gridDim.x * blockDim.x) {
        const int c = (int)(i % c4) * 4;
        const int64_t r = i / c4;
        const int n = (int)(r / hwi), pix = (int)(r - (int64_t)n * hwi), sy = pix / Wi, sx = pix - sy * Wi;
        const int y0 = first_dst(sy, Hi, Ho), y1 = first_dst(sy + 1, Hi, Ho);
        const int x0 = first_dst(sx, Wi, Wo), x1 = first_dst(sx + 1, Wi, Wo);
        float4 s = make_float4(0.f, 0.f, 0.f, 0.f);
        for (int oy = y0; oy < y1; ++oy)
            for (int ox = x0; ox < x1; ++ox) {
                const float4 v = g.at(n, oy * Wo + ox, c);
                s.x += v.x, s.y += v.y, s.z += v.z, s.w += v.w;
            }
        *reinterpret_cast<float4 *>(dst + (int64_t)n * d_pitch + (int64_t)pix * ldd + c) = s;
    }
}

// ---- convolution weight gradient ---------------------------------------------------------------------------------------
// dW[co, ci, ky, kx] = sum over output pixels m of dY[m, co] . X[shift(m, ky, kx), ci], per group.  One CTA (one warpgroup) per
// 64 (co) x 64 (ci) tile of one tap and one split of the pixel range: a GEMM with M = co, N = ci, K = pixels.  Per 64-pixel
// k-block the CTA copies the dY and X rows (fp32, cp.async, X zero-filled outside the map) into a 3-stage ring; dY^T is the
// register A operand (split in registers, like the forward's activation); X is split into fp16 hi / lo and written TRANSPOSED
// (pixel-contiguous, 128-byte swizzle) into one shared W_hi / W_lo-shaped pair, so wgmma reads it K-major.  Each split writes
// its partial tile to the workspace; a second launch sums the splits in split order (bit-reproducible, no atomics) into the
// (Cout, Cin / groups, k, k) layout.
constexpr int kWgStageBytes = 2 * kCvABytes;
constexpr int kWgSmem = kCvStages * kWgStageBytes + 2 * kCvBBytes + 1024 /* alignment */;
constexpr int kWgTargetCtas = 512;  // splits = ceil(512 / tiles) at most: a function of the shape alone, so the bits are too

struct WgradParams {
    const float *dy;
    int64_t dy_pitch, lddy;
    const float *x;
    int64_t x_pitch, ldx;
    const float *dy_scale, *x_scale;
    float *part;  // (splits, Cout, cin_g, k, k)
    int H, W, Ho, Wo, M, Cout, cin_g, cout_g, ksize, stride, kb_per_split;
};

__global__ void __launch_bounds__(kCvThreads) conv_wgrad_f16x3_kernel(const WgradParams p) {
    extern __shared__ uint8_t smem_raw[];
    uint8_t *smem = reinterpret_cast<uint8_t *>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~uintptr_t(1023));
    uint8_t *bhi = smem + kCvStages * kWgStageBytes, *blo = bhi + kCvBBytes;
    const int tid = threadIdx.x, taps = p.ksize * p.ksize, ci_tiles = p.cin_g / kCvN;
    const int tap = blockIdx.x % taps, cit = (blockIdx.x / taps) % ci_tiles, cot = blockIdx.x / (taps * ci_tiles);
    const int co0 = cot * kCvM, ci0 = cit * kCvN, xc0 = (co0 / p.cout_g) * p.cin_g + ci0;
    const int ky = tap / p.ksize, kx = tap - ky * p.ksize, pad = p.ksize >> 1, hwo = p.Ho * p.Wo;
    const int kb0 = blockIdx.y * p.kb_per_split, kb1 = min(kb0 + p.kb_per_split, (p.M + kCvK - 1) / kCvK), kblocks = kb1 - kb0;
    const int ac = tid & 15;

    auto load_stage = [&](int s, int kb) {
        uint8_t *st = smem + s * kWgStageBytes;
#pragma unroll
        for (int j = 0; j < 8; ++j) {
            const int r = (tid >> 4) + 8 * j, m = kb * kCvK + r;
            bool okd = false, okx = false;
            const float *sd = p.dy, *sx = p.x;
            if (m < p.M) {
                const int n = m / hwo, pix = m - n * hwo, oy = pix / p.Wo, ox = pix - oy * p.Wo;
                const int iy = oy * p.stride - pad + ky, ix = ox * p.stride - pad + kx;
                okd = true, sd = p.dy + (int64_t)n * p.dy_pitch + (int64_t)pix * p.lddy + co0 + ac * 4;
                okx = (unsigned)iy < (unsigned)p.H && (unsigned)ix < (unsigned)p.W;
                if (okx) sx = p.x + (int64_t)n * p.x_pitch + ((int64_t)iy * p.W + ix) * p.ldx + xc0 + ac * 4;
            }
            const int off = r * 256 + ((ac ^ (r & 7)) << 4);
            cp_async16(st + off, sd, okd);
            cp_async16(st + kCvABytes + off, sx, okx);
        }
    };

    const float ds = __ldg(p.dy_scale), xs = __ldg(p.x_scale), out_scale = 1.f / (ds * xs);
    const int warp = tid >> 5, lane = tid & 31, g = lane >> 2, q = lane & 3, r0 = warp * 16 + g;
    float d[32], acc[32];
#pragma unroll
    for (int i = 0; i < 32; ++i) acc[i] = 0.f;
#pragma unroll
    for (int s = 0; s < kCvStages - 1; ++s) {
        if (s < kblocks) load_stage(s, kb0 + s);
        cp_async_commit();
    }
    for (int kb = 0; kb < kblocks; ++kb) {
        cp_async_wait_1();
        __syncthreads();  // the stage has landed; every warp is done with W_hi / W_lo and the stage the next copy overwrites
        if (kb + kCvStages - 1 < kblocks) load_stage((kb + kCvStages - 1) % kCvStages, kb0 + kb + kCvStages - 1);
        cp_async_commit();
        const uint8_t *st = smem + (kb % kCvStages) * kWgStageBytes, *sx = st + kCvABytes;
        // X (pixel, ci) -> hi / lo (ci, pixel): thread = channel tid & 63, 8-pixel chunks (tid >> 6) + 2 jj
#pragma unroll
        for (int jj = 0; jj < 4; ++jj) {
            const int ci = tid & 63, ch = (tid >> 6) + 2 * jj;
            uint32_t h[4], l[4];
#pragma unroll
            for (int e = 0; e < 4; ++e) {
                const int p0 = ch * 8 + 2 * e, p1 = p0 + 1;
                const float v0 = *reinterpret_cast<const float *>(sx + p0 * 256 + ((((ci >> 2) ^ (p0 & 7)) << 4) | ((ci & 3) << 2)));
                const float v1 = *reinterpret_cast<const float *>(sx + p1 * 256 + ((((ci >> 2) ^ (p1 & 7)) << 4) | ((ci & 3) << 2)));
                split2(v0 * xs, v1 * xs, h[e], l[e]);
            }
            const int off = ci * 128 + ((ch ^ (ci & 7)) << 4);
            *reinterpret_cast<uint4 *>(bhi + off) = make_uint4(h[0], h[1], h[2], h[3]);
            *reinterpret_cast<uint4 *>(blo + off) = make_uint4(l[0], l[1], l[2], l[3]);
        }
        asm volatile("fence.proxy.async.shared::cta;" ::: "memory");  // generic-proxy writes -> wgmma operand reads
        __syncthreads();
        uint32_t ahi[4][4], alo[4][4];
#pragma unroll
        for (int kk = 0; kk < 4; ++kk) {  // A = dY^T: row = output channel, column = pixel
#pragma unroll
            for (int j = 0; j < 4; ++j) {
                const int co = r0 + (j & 1) * 8, px = kk * 16 + 2 * q + (j >> 1) * 8;
                const float v0 = *reinterpret_cast<const float *>(st + px * 256 + ((((co >> 2) ^ (px & 7)) << 4) | ((co & 3) << 2)));
                const float v1 =
                    *reinterpret_cast<const float *>(st + (px + 1) * 256 + ((((co >> 2) ^ ((px + 1) & 7)) << 4) | ((co & 3) << 2)));
                split2(v0 * ds, v1 * ds, ahi[kk][j], alo[kk][j]);
            }
        }
        wgmma_fence();
        const uint32_t bh = smem_u32(bhi), bl = smem_u32(blo);
#pragma unroll
        for (int kk = 0; kk < 4; ++kk) {
            wgmma_f16_rs_n64(d, alo[kk], wgmma_desc(bh + kk * 32), kk);
            wgmma_f16_rs_n64(d, ahi[kk], wgmma_desc(bl + kk * 32), 1);
            wgmma_f16_rs_n64(d, ahi[kk], wgmma_desc(bh + kk * 32), 1);
        }
        wgmma_commit();
        wgmma_wait_all();
#pragma unroll
        for (int i = 0; i < 32; ++i) acc[i] += d[i];
    }
    // acc[4j + 2h + e] = (output channel co0 + r0 + 8h, input channel ci0 + 8j + 2q + e)
    float *part = p.part + (int64_t)blockIdx.y * p.Cout * p.cin_g * taps;
#pragma unroll
    for (int h = 0; h < 2; ++h) {
        const int64_t row = (int64_t)(co0 + r0 + 8 * h) * p.cin_g;
#pragma unroll
        for (int j = 0; j < 8; ++j)
#pragma unroll
            for (int e = 0; e < 2; ++e) part[(row + ci0 + 8 * j + 2 * q + e) * taps + tap] = acc[4 * j + 2 * h + e] * out_scale;
    }
}

// dw = the splits summed in split order, times cout_scale[co] when it is not NULL (one rounded product after the sum)
__global__ void wgrad_reduce_kernel(const float *__restrict__ part, int splits, int64_t n, const float *__restrict__ cout_scale,
                                    int64_t per_co, float *__restrict__ dw) {
    for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (int64_t)gridDim.x * blockDim.x) {
        float s = 0.f;
        for (int k = 0; k < splits; ++k) s += part[(int64_t)k * n + i];
        dw[i] = cout_scale ? s * __ldg(cout_scale + i / per_co) : s;
    }
}

// split of the pixel range: (splits, k-blocks per split), from the shape alone
inline void wgrad_splits(int64_t M, int tiles, int &splits, int &per) {
    const int kblocks = (int)((M + kCvK - 1) / kCvK);
    if (kblocks == 0) {
        splits = 0, per = 1;
        return;
    }
    int want = (kWgTargetCtas + tiles - 1) / tiles;
    want = want < 1 ? 1 : (want > kblocks ? kblocks : want);
    per = (kblocks + want - 1) / want;
    splits = (kblocks + per - 1) / per;
}

// the channel / kernel shapes sdetr_conv2d_f16x3_wgrad takes (its workspace size function answers 0 for the others)
inline bool wgrad_shape_ok(int Cin, int Cout, int groups, int ksize) {
    return Cin > 0 && Cout > 0 && groups > 0 && Cin % groups == 0 && Cout % groups == 0 && (Cin / groups) % kCvK == 0 &&
           (Cout / groups) % kCvN == 0 && (ksize == 1 || ksize == 3);
}

// one pass over a (Cout, Cin / groups, k, k) weight: the fp16 pair of the forward layout (Cout, k, k, Cin / groups) and, when
// asked, of the input-gradient layout (Cin, k, k, Cout / groups) flipped in both spatial axes -- the arithmetic of
// sdetr_split_f16_pair_dev with one device scale for both
__global__ void split_conv_weight_kernel(const float *__restrict__ w, int cout, int cin_g, int groups, int ksize,
                                         const float *__restrict__ scale_dev, __half *__restrict__ f_hi, __half *__restrict__ f_lo,
                                         __half *__restrict__ d_hi, __half *__restrict__ d_lo) {
    const int taps = ksize * ksize, cout_g = cout / groups;
    const int64_t n = (int64_t)cout * cin_g * taps;
    const float scale = __ldg(scale_dev);
    for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (int64_t)gridDim.x * blockDim.x) {
        const int tap = (int)(i % taps), ci = (int)((i / taps) % cin_g), co = (int)(i / ((int64_t)taps * cin_g));
        const float x = w[i] * scale;
        const __half h = __float2half_rn(x), l = __float2half_rn(x - __half2float(h));
        const int64_t fi = ((int64_t)co * taps + tap) * cin_g + ci;
        f_hi[fi] = h, f_lo[fi] = l;
        if (d_hi) {
            const int g = co / cout_g;
            const int64_t di = ((int64_t)(g * cin_g + ci) * taps + (taps - 1 - tap)) * cout_g + (co - g * cout_g);
            d_hi[di] = h, d_lo[di] = l;
        }
    }
}

inline bool rows_ok(const float *p, int64_t pitch, int64_t ld) { return aligned16(p) && pitch % 4 == 0 && ld % 4 == 0; }
inline int elementwise_blocks(int64_t total) {
    const int64_t want = (total + 255) / 256, cap = 8LL * sm_count();
    return (int)(want < 1 ? 1 : (want > cap ? cap : want));
}

}  // namespace sdetr

using namespace sdetr;

extern "C" int sdetr_conv2d_f16x3(const float *x, int64_t x_pitch, int64_t ldx, int batch, int H, int W, int Cin,
                                  const float *a_scale_dev, const void *W_hi, const void *W_lo, const float *w_scale_dev,
                                  const float *bias, const float *z, int64_t z_pitch, int64_t ldz, int Cout, int groups, int ksize,
                                  int stride, int act, float *y, int64_t y_pitch, int64_t ldy, sdetr_stream_t stream) {
    SDETR_REQUIRE(x && a_scale_dev && W_hi && W_lo && w_scale_dev && y, SDETR_ERR_INVALID_ARG, "conv2d_f16x3: null pointer");
    SDETR_REQUIRE(batch >= 0 && H >= 0 && W >= 0 && Cin > 0 && Cout > 0 && groups > 0, SDETR_ERR_INVALID_ARG,
                  "conv2d_f16x3: bad sizes");
    SDETR_REQUIRE((ksize == 1 || ksize == 3) && (stride == 1 || stride == 2) && (act == 0 || act == kActReLU || act == kActSiLU),
                  SDETR_ERR_UNSUPPORTED, "conv2d_f16x3: takes kernel 1 or 3, stride 1 or 2, act 0 (none), 1 (ReLU) or 3 (SiLU)");
    SDETR_REQUIRE(Cin % groups == 0 && Cout % groups == 0 && (Cin / groups) % kCvK == 0 && (Cout / groups) % kCvN == 0,
                  SDETR_ERR_UNSUPPORTED, "conv2d_f16x3: Cin/groups=%d and Cout/groups=%d must be multiples of 64",
                  Cin / groups, Cout / groups);
    SDETR_REQUIRE(rows_ok(x, x_pitch, ldx) && ldx >= Cin && aligned16(W_hi) && aligned16(W_lo), SDETR_ERR_INVALID_ARG,
                  "conv2d_f16x3: x, its pitch and row stride and the weights must be 16-byte aligned");
    SDETR_REQUIRE((reinterpret_cast<uintptr_t>(y) & 7) == 0 && y_pitch % 2 == 0 && ldy % 2 == 0 && ldy >= Cout,
                  SDETR_ERR_INVALID_ARG, "conv2d_f16x3: y, its pitch and row stride must be 8-byte aligned");
    SDETR_REQUIRE(!z || ((reinterpret_cast<uintptr_t>(z) & 7) == 0 && z_pitch % 2 == 0 && ldz % 2 == 0 && ldz >= Cout),
                  SDETR_ERR_INVALID_ARG, "conv2d_f16x3: z, its pitch and row stride must be 8-byte aligned");
    const int pad = ksize / 2, Ho = H > 0 ? (H + 2 * pad - ksize) / stride + 1 : 0, Wo = W > 0 ? (W + 2 * pad - ksize) / stride + 1 : 0;
    const int64_t M = (int64_t)batch * Ho * Wo;
    SDETR_REQUIRE(M < (1LL << 31) - kCvM, SDETR_ERR_INVALID_ARG, "conv2d_f16x3: too many output pixels");
    if (M == 0) return SDETR_OK;
    static PerDeviceOnce once;
    SDETR_OPT_IN_SMEM(once, conv_f16x3_kernel<false>, kCvSmem, "conv2d_f16x3");
    const ConvParams p{x, x_pitch, ldx, reinterpret_cast<const __half *>(W_hi), reinterpret_cast<const __half *>(W_lo), a_scale_dev,
                       w_scale_dev, bias, z, z_pitch, ldz, nullptr, 0, 0, y, y_pitch, ldy, H, W, Ho, Wo, (int)M, Cin / groups,
                       Cout / groups, ksize, stride, act};
    const dim3 grid((unsigned)((M + kCvM - 1) / kCvM), (unsigned)(Cout / kCvN));
    conv_f16x3_kernel<false><<<grid, kCvThreads, kCvSmem, (cudaStream_t)stream>>>(p);
    return check_launch("conv2d_f16x3");
}

extern "C" int64_t sdetr_conv2d_f16x3_wgrad_workspace_floats(int batch, int Ho, int Wo, int Cin, int Cout, int groups, int ksize) {
    if (batch <= 0 || Ho <= 0 || Wo <= 0 || !wgrad_shape_ok(Cin, Cout, groups, ksize)) return 0;
    const int tiles = (Cout / kCvM) * ((Cin / groups) / kCvN) * ksize * ksize;
    int splits, per;
    wgrad_splits((int64_t)batch * Ho * Wo, tiles, splits, per);
    return (int64_t)splits * Cout * (Cin / groups) * ksize * ksize;
}

extern "C" int sdetr_conv2d_f16x3_wgrad(const float *dy, int64_t dy_pitch, int64_t lddy, const float *dy_scale_dev,
                                        const float *x, int64_t x_pitch, int64_t ldx, const float *x_scale_dev, int batch, int H,
                                        int W, int Cin, int Cout, int groups, int ksize, int stride, const float *cout_scale,
                                        float *workspace, int64_t workspace_floats, float *dw, sdetr_stream_t stream) {
    SDETR_REQUIRE(dy && dy_scale_dev && x && x_scale_dev && dw && workspace, SDETR_ERR_INVALID_ARG, "conv2d_f16x3_wgrad: null pointer");
    SDETR_REQUIRE(batch >= 0 && H >= 0 && W >= 0 && Cin > 0 && Cout > 0 && groups > 0, SDETR_ERR_INVALID_ARG,
                  "conv2d_f16x3_wgrad: bad sizes");
    SDETR_REQUIRE((ksize == 1 || ksize == 3) && (stride == 1 || stride == 2), SDETR_ERR_UNSUPPORTED,
                  "conv2d_f16x3_wgrad: takes kernel 1 or 3, stride 1 or 2");
    SDETR_REQUIRE(wgrad_shape_ok(Cin, Cout, groups, 1), SDETR_ERR_UNSUPPORTED,
                  "conv2d_f16x3_wgrad: Cin/groups=%d and Cout/groups=%d must be multiples of 64", Cin / groups, Cout / groups);
    SDETR_REQUIRE(rows_ok(dy, dy_pitch, lddy) && lddy >= Cout && rows_ok(x, x_pitch, ldx) && ldx >= Cin, SDETR_ERR_INVALID_ARG,
                  "conv2d_f16x3_wgrad: dy, x, their pitches and row strides must be 16-byte aligned");
    const int pad = ksize / 2, Ho = H > 0 ? (H + 2 * pad - ksize) / stride + 1 : 0, Wo = W > 0 ? (W + 2 * pad - ksize) / stride + 1 : 0;
    const int64_t M = (int64_t)batch * Ho * Wo, n = (int64_t)Cout * (Cin / groups) * ksize * ksize;
    SDETR_REQUIRE(M < (1LL << 31) - kCvM, SDETR_ERR_INVALID_ARG, "conv2d_f16x3_wgrad: too many output pixels");
    const int tiles = (Cout / kCvM) * ((Cin / groups) / kCvN) * ksize * ksize;
    int splits, per;
    wgrad_splits(M, tiles, splits, per);
    SDETR_REQUIRE(aligned16(workspace) && workspace_floats >= (int64_t)splits * n, SDETR_ERR_INVALID_ARG,
                  "conv2d_f16x3_wgrad: workspace too small or not 16-byte aligned");
    if (splits > 0) {
        static PerDeviceOnce once;
        SDETR_OPT_IN_SMEM(once, conv_wgrad_f16x3_kernel, kWgSmem, "conv2d_f16x3_wgrad");
        const WgradParams p{dy, dy_pitch, lddy, x, x_pitch, ldx, dy_scale_dev, x_scale_dev, workspace, H, W, Ho, Wo, (int)M, Cout,
                            Cin / groups, Cout / groups, ksize, stride, per};
        conv_wgrad_f16x3_kernel<<<dim3((unsigned)tiles, (unsigned)splits), kCvThreads, kWgSmem, (cudaStream_t)stream>>>(p);
        const int rc = check_launch("conv2d_f16x3_wgrad");
        if (rc) return rc;
    }
    wgrad_reduce_kernel<<<elementwise_blocks(n), 256, 0, (cudaStream_t)stream>>>(workspace, splits, n, cout_scale,
                                                                                  n / Cout, dw);
    return check_launch("conv2d_f16x3_wgrad (split sum)");
}

extern "C" int sdetr_conv2d_f16x3_dgrad(const float *dy, int64_t dy_pitch, int64_t lddy, int batch, int Hy, int Wy, int Cin,
                                        const float *a_scale_dev, const void *W_hi, const void *W_lo, const float *w_scale_dev,
                                        const float *z, int64_t z_pitch, int64_t ldz, const float *m, int64_t m_pitch, int64_t ldm,
                                        int Cout, int groups, int ksize, int stride, int H, int W, float *dx, int64_t dx_pitch,
                                        int64_t lddx, sdetr_stream_t stream) {
    SDETR_REQUIRE(dy && a_scale_dev && W_hi && W_lo && w_scale_dev && dx, SDETR_ERR_INVALID_ARG, "conv2d_f16x3_dgrad: null pointer");
    SDETR_REQUIRE(batch >= 0 && H >= 0 && W >= 0 && Cin > 0 && Cout > 0 && groups > 0, SDETR_ERR_INVALID_ARG,
                  "conv2d_f16x3_dgrad: bad sizes");
    SDETR_REQUIRE((ksize == 1 || ksize == 3) && (stride == 1 || stride == 2), SDETR_ERR_UNSUPPORTED,
                  "conv2d_f16x3_dgrad: takes kernel 1 or 3, stride 1 or 2");
    SDETR_REQUIRE(Cin % groups == 0 && Cout % groups == 0 && (Cin / groups) % kCvK == 0 && (Cout / groups) % kCvN == 0,
                  SDETR_ERR_UNSUPPORTED, "conv2d_f16x3_dgrad: Cin/groups=%d and Cout/groups=%d must be multiples of 64",
                  Cin / groups, Cout / groups);
    const int pad = ksize / 2, hy = H > 0 ? (H + 2 * pad - ksize) / stride + 1 : 0, wy = W > 0 ? (W + 2 * pad - ksize) / stride + 1 : 0;
    SDETR_REQUIRE(Hy == hy && Wy == wy, SDETR_ERR_INVALID_ARG,
                  "conv2d_f16x3_dgrad: dY is %dx%d, a stride-%d convolution of %dx%d gives %dx%d", Hy, Wy, stride, H, W, hy, wy);
    SDETR_REQUIRE(rows_ok(dy, dy_pitch, lddy) && lddy >= Cin && aligned16(W_hi) && aligned16(W_lo), SDETR_ERR_INVALID_ARG,
                  "conv2d_f16x3_dgrad: dy, its pitch and row stride and the weights must be 16-byte aligned");
    SDETR_REQUIRE((reinterpret_cast<uintptr_t>(dx) & 7) == 0 && dx_pitch % 2 == 0 && lddx % 2 == 0 && lddx >= Cout,
                  SDETR_ERR_INVALID_ARG, "conv2d_f16x3_dgrad: dx, its pitch and row stride must be 8-byte aligned");
    SDETR_REQUIRE(!z || ((reinterpret_cast<uintptr_t>(z) & 7) == 0 && z_pitch % 2 == 0 && ldz % 2 == 0 && ldz >= Cout),
                  SDETR_ERR_INVALID_ARG, "conv2d_f16x3_dgrad: z, its pitch and row stride must be 8-byte aligned");
    SDETR_REQUIRE(!m || ((reinterpret_cast<uintptr_t>(m) & 7) == 0 && m_pitch % 2 == 0 && ldm % 2 == 0 && ldm >= Cout),
                  SDETR_ERR_INVALID_ARG, "conv2d_f16x3_dgrad: m, its pitch and row stride must be 8-byte aligned");
    SDETR_REQUIRE(m != dx, SDETR_ERR_INVALID_ARG, "conv2d_f16x3_dgrad: m must not alias dx");
    const int64_t M = (int64_t)batch * H * W;
    SDETR_REQUIRE(M < (1LL << 31) - kCvM, SDETR_ERR_INVALID_ARG, "conv2d_f16x3_dgrad: too many output pixels");
    if (M == 0) return SDETR_OK;
    // stride 1: the forward kernel on dY with the flipped weights (dY and dX share the map size); stride 2: its transposed mode
    const ConvParams p{dy, dy_pitch, lddy, reinterpret_cast<const __half *>(W_hi), reinterpret_cast<const __half *>(W_lo), a_scale_dev,
                       w_scale_dev, nullptr, z, z_pitch, ldz, m, m_pitch, ldm, dx, dx_pitch, lddx, Hy, Wy, H, W, (int)M,
                       Cin / groups, Cout / groups, ksize, stride == 1 ? 1 : 2, 0};
    const dim3 grid((unsigned)((M + kCvM - 1) / kCvM), (unsigned)(Cout / kCvN));
    if (stride == 1) {
        static PerDeviceOnce once;
        SDETR_OPT_IN_SMEM(once, conv_f16x3_kernel<false>, kCvSmem, "conv2d_f16x3_dgrad");
        conv_f16x3_kernel<false><<<grid, kCvThreads, kCvSmem, (cudaStream_t)stream>>>(p);
    } else {
        static PerDeviceOnce once;
        SDETR_OPT_IN_SMEM(once, conv_f16x3_kernel<true>, kCvSmem, "conv2d_f16x3_dgrad");
        conv_f16x3_kernel<true><<<grid, kCvThreads, kCvSmem, (cudaStream_t)stream>>>(p);
    }
    return check_launch("conv2d_f16x3_dgrad");
}

extern "C" int64_t sdetr_context_gate_workspace_floats(int batch, int HW, int C) {
    if (batch <= 0 || HW <= 0 || C <= 0) return 0;
    return (int64_t)batch * ((HW + kGateChunk - 1) / kGateChunk) * (C + 2) + (int64_t)batch * C;
}

extern "C" int sdetr_context_gate(const float *y, int64_t y_pitch, int64_t ldy, const float *x, int64_t x_pitch, int64_t ldx,
                                  const float *z, int64_t z_pitch, int64_t ldz, int batch, int HW, int C, const float *w_mask,
                                  const float *b_mask, const float *w1, const float *w2, int R, float *workspace,
                                  int64_t workspace_floats, float *out, int64_t out_pitch, int64_t ldo, sdetr_stream_t stream) {
    SDETR_REQUIRE(y && x && w_mask && b_mask && w1 && w2 && out && workspace, SDETR_ERR_INVALID_ARG, "context_gate: null pointer");
    SDETR_REQUIRE(batch >= 0 && HW > 0 && C > 0 && R > 0, SDETR_ERR_INVALID_ARG, "context_gate: bad sizes");
    SDETR_REQUIRE(C % 4 == 0 && C + R <= 12 * 1024, SDETR_ERR_UNSUPPORTED, "context_gate: C=%d must be a multiple of 4 and C + R at most 12288", C);
    SDETR_REQUIRE(rows_ok(y, y_pitch, ldy) && rows_ok(x, x_pitch, ldx) && (!z || rows_ok(z, z_pitch, ldz)) &&
                      rows_ok(out, out_pitch, ldo) && aligned16(workspace),
                  SDETR_ERR_INVALID_ARG, "context_gate: operands, pitches and row strides must be 16-byte aligned");
    if (batch == 0) return SDETR_OK;
    SDETR_REQUIRE(workspace_floats >= sdetr_context_gate_workspace_floats(batch, HW, C), SDETR_ERR_INVALID_ARG,
                  "context_gate: workspace too small");
    const int nchunk = (HW + kGateChunk - 1) / kGateChunk;
    float *gate = workspace, *part = workspace + (int64_t)batch * C;  // gate first: 16-byte aligned for the float4 reads
    gate_partial_kernel<<<dim3(nchunk, batch), kGateThreads, 0, (cudaStream_t)stream>>>(y, y_pitch, ldy, HW, C, w_mask, b_mask,
                                                                                         nchunk, part);
    int rc = check_launch("context_gate (partial sums)");
    if (rc) return rc;
    gate_combine_kernel<<<batch, kGateThreads, (C + R) * sizeof(float), (cudaStream_t)stream>>>(part, nchunk, C, R, w1, w2, gate);
    rc = check_launch("context_gate (combine)");
    if (rc) return rc;
    gate_apply_kernel<<<elementwise_blocks((int64_t)batch * HW * (C / 4)), 256, 0, (cudaStream_t)stream>>>(
        Rows{y, y_pitch, ldy}, Rows{x, x_pitch, ldx}, Rows{z, z_pitch, ldz}, gate, batch, HW, C, out, out_pitch, ldo);
    return check_launch("context_gate (apply)");
}

extern "C" int sdetr_upsample_nearest_concat(const float *hi, int64_t hi_pitch, int64_t ldh, int Hi, int Wi, const float *lo,
                                             int64_t lo_pitch, int64_t ldl, int Ho, int Wo, int batch, int C, float *dst,
                                             int64_t dst_pitch, int64_t ldd, sdetr_stream_t stream) {
    SDETR_REQUIRE(hi && lo && dst, SDETR_ERR_INVALID_ARG, "upsample_nearest_concat: null pointer");
    SDETR_REQUIRE(batch >= 0 && Hi > 0 && Wi > 0 && Ho >= 0 && Wo >= 0 && C > 0 && C % 4 == 0, SDETR_ERR_INVALID_ARG,
                  "upsample_nearest_concat: bad sizes (C a multiple of 4)");
    SDETR_REQUIRE(rows_ok(hi, hi_pitch, ldh) && rows_ok(lo, lo_pitch, ldl) && rows_ok(dst, dst_pitch, ldd), SDETR_ERR_INVALID_ARG,
                  "upsample_nearest_concat: operands, pitches and row strides must be 16-byte aligned");
    const int64_t total = (int64_t)batch * Ho * Wo * (C / 2);
    if (total == 0) return SDETR_OK;
    upsample_concat_kernel<<<elementwise_blocks(total), 256, 0, (cudaStream_t)stream>>>(Rows{hi, hi_pitch, ldh}, Hi, Wi,
                                                                                         Rows{lo, lo_pitch, ldl}, Ho, Wo, batch, C,
                                                                                         dst, dst_pitch, ldd);
    return check_launch("upsample_nearest_concat");
}

extern "C" int sdetr_upsample_nearest_concat_backward(const float *g, int64_t g_pitch, int64_t ldg, int Ho, int Wo, int Hi, int Wi,
                                                      int batch, int C, float *d_hi, int64_t d_pitch, int64_t ldd,
                                                      sdetr_stream_t stream) {
    SDETR_REQUIRE(g && d_hi, SDETR_ERR_INVALID_ARG, "upsample_nearest_concat_backward: null pointer");
    SDETR_REQUIRE(batch >= 0 && Hi > 0 && Wi > 0 && Ho > 0 && Wo > 0 && C > 0 && C % 4 == 0, SDETR_ERR_INVALID_ARG,
                  "upsample_nearest_concat_backward: bad sizes (C a multiple of 4)");
    SDETR_REQUIRE(rows_ok(g, g_pitch, ldg) && ldg >= C && rows_ok(d_hi, d_pitch, ldd) && ldd >= C, SDETR_ERR_INVALID_ARG,
                  "upsample_nearest_concat_backward: operands, pitches and row strides must be 16-byte aligned");
    const int64_t total = (int64_t)batch * Hi * Wi * (C / 4);
    if (total == 0) return SDETR_OK;
    upsample_concat_backward_kernel<<<elementwise_blocks(total), 256, 0, (cudaStream_t)stream>>>(Rows{g, g_pitch, ldg}, Ho, Wo, Hi,
                                                                                                  Wi, batch, C, d_hi, d_pitch, ldd);
    return check_launch("upsample_nearest_concat_backward");
}

extern "C" int sdetr_conv2d_f16x3_split_weight(const float *w, int Cout, int Cin, int groups, int ksize, const float *scale_dev,
                                               void *fwd_hi, void *fwd_lo, void *dgrad_hi, void *dgrad_lo, sdetr_stream_t stream) {
    SDETR_REQUIRE(w && scale_dev && fwd_hi && fwd_lo && (dgrad_hi == nullptr) == (dgrad_lo == nullptr), SDETR_ERR_INVALID_ARG,
                  "conv2d_f16x3_split_weight: null pointer (dgrad_hi and dgrad_lo go together)");
    SDETR_REQUIRE(Cout > 0 && Cin > 0 && groups > 0 && Cin % groups == 0 && Cout % groups == 0 && (ksize == 1 || ksize == 3),
                  SDETR_ERR_INVALID_ARG, "conv2d_f16x3_split_weight: bad sizes");
    const int64_t n = (int64_t)Cout * (Cin / groups) * ksize * ksize;
    split_conv_weight_kernel<<<elementwise_blocks(n), 256, 0, (cudaStream_t)stream>>>(
        w, Cout, Cin / groups, groups, ksize, scale_dev, reinterpret_cast<__half *>(fwd_hi), reinterpret_cast<__half *>(fwd_lo),
        reinterpret_cast<__half *>(dgrad_hi), reinterpret_cast<__half *>(dgrad_lo));
    return check_launch("conv2d_f16x3_split_weight");
}
