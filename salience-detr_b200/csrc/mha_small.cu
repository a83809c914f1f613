// The 300-token pre-attention of an encoder layer (reference salience_transformer.py:366-379): top-k tokens -> gather
// -> nn.MultiheadAttention(256, 8) self-attention (q = k = tok + pos, v = tok) -> residual -> LayerNorm -> scatter.
//
// The block is tiny (600 rows at bs=2) and latency-bound: as library calls it was 3 SGEMMs + an SDPA kernel + gather /
// LayerNorm / scatter kernels, ~95 us per layer.  Here it is three fp32 SIMT kernels:
//   mha_in_proj_kernel        gather + (tok + pos) + the packed in-projection (q | k | v), one launch
//   attn_rows_kernel          softmax(q k^T / sqrt(d)) v per (image, head, query tile): K^T / V / scores live in shared
//                             memory, the two products are register-tiled so they are FMA-bound, not LDS-bound
//   mha_out_proj_ln_scatter   out-projection + residual + LayerNorm + scatter back into the layer's query buffer
// Weights arrive TRANSPOSED ((in, out) row-major; the host caches the transposes per parameter version) so weight tiles
// stream into shared memory with coalesced rows and conflict-free stores.  All arithmetic is fp32 FMA (no tensor cores:
// the block is ~0.5 GFLOP and the strict-fp32 parity mode must stay bit-stable).
#include "common.cuh"

namespace sdetr {

// ---- gather + in-projection -----------------------------------------------------------------------------------------
// rows = batch * k selected tokens; out columns [0, 2C) use A = tok + pos (q and k), [2C, 3C) use A = tok (v).
// CTA tile: 32 rows x 128 columns, full K = C resident in shared memory (activation TRANSPOSED, [kk][row]); thread tile
// 4 rows x 4 columns, a warp = one row group x 32 column groups: per kk one broadcast 128-bit load of 4 activations and
// one 128-bit load of 4 weights feed 16 FMAs (the first version, 2 x 4 tiles, was shared-memory-bandwidth bound).
constexpr int kInRows = 32, kInCols = 128, kInThreads = 256, kInPitch = kInRows + 4;

__device__ __forceinline__ void cp_async16(float *smem_dst, const float *gmem_src) {
    const uint32_t d = (uint32_t)__cvta_generic_to_shared(smem_dst);
    asm volatile("cp.async.cg.shared.global [%0], [%1], 16;" ::"r"(d), "l"(gmem_src) : "memory");
}

template <int C>
__global__ void __launch_bounds__(kInThreads) mha_in_proj_kernel(const float *__restrict__ tokens, const float *__restrict__ pos,
                                                                 const int64_t *__restrict__ index, int nq, int k, int rows,
                                                                 const float *__restrict__ w_t /* (C, 3C) */,
                                                                 const float *__restrict__ bias /* 3C */,
                                                                 float *__restrict__ t_out /* (rows, C) */,
                                                                 float *__restrict__ qkv /* (rows, 3C) */) {
    extern __shared__ __align__(16) float sm_in[];
    float *At = sm_in;                        // [C][36]: At[kk][row]
    float *Ws = sm_in + C * kInPitch;         // [C][128]
    const int row0 = blockIdx.x * kInRows, n0 = blockIdx.y * kInCols;
    const bool add_pos = n0 < 2 * C, write_t = n0 == 2 * C;
    const int tid = threadIdx.x;
    // weight tile: rows kk of W^T, columns [n0, n0 + 128): asynchronous copies, all in flight at once
    for (int item = tid; item < C * (kInCols / 4); item += kInThreads) {
        const int kk = item / (kInCols / 4), c = (item % (kInCols / 4)) * 4;
        cp_async16(Ws + kk * kInCols + c, w_t + (int64_t)kk * (3 * C) + n0 + c);
    }
    asm volatile("cp.async.commit_group;" ::: "memory");
    // activation tile: gathered rows (+ pos), lane <-> row so the transposed stores are conflict-free; loads batched
    constexpr int kPer = kInRows * (C / 4) / kInThreads;
    float4 tv[kPer], pv[kPer];
#pragma unroll
    for (int u = 0; u < kPer; ++u) {
        const int item = tid + u * kInThreads;
        const int i = item % kInRows, c = (item / kInRows) * 4;
        const int r = row0 + i;
        tv[u] = make_float4(0.f, 0.f, 0.f, 0.f), pv[u] = tv[u];
        if (r < rows) {
            const int b = r / k;
            const int64_t src = ((int64_t)b * nq + __ldg(index + r)) * C + c;
            tv[u] = ldg_f4(tokens + src);
            if (add_pos) pv[u] = ldg_f4(pos + src);
        }
    }
#pragma unroll
    for (int u = 0; u < kPer; ++u) {
        const int item = tid + u * kInThreads;
        const int i = item % kInRows, c = (item / kInRows) * 4;
        const int r = row0 + i;
        if (write_t && r < rows) *reinterpret_cast<float4 *>(t_out + (int64_t)r * C + c) = tv[u];
        At[(c + 0) * kInPitch + i] = tv[u].x + pv[u].x, At[(c + 1) * kInPitch + i] = tv[u].y + pv[u].y;
        At[(c + 2) * kInPitch + i] = tv[u].z + pv[u].z, At[(c + 3) * kInPitch + i] = tv[u].w + pv[u].w;
    }
    asm volatile("cp.async.wait_group 0;" ::: "memory");
    __syncthreads();
    const int tx = tid & 31, ty = tid >> 5;
    const float *ap = At + ty * 4, *wp = Ws + tx * 4;
    float4 acc[4];
#pragma unroll
    for (int i = 0; i < 4; ++i) acc[i] = make_float4(0.f, 0.f, 0.f, 0.f);
#pragma unroll 8
    for (int kk = 0; kk < C; ++kk) {
        const float4 a = *reinterpret_cast<const float4 *>(ap + kk * kInPitch);
        const float4 w = *reinterpret_cast<const float4 *>(wp + kk * kInCols);
        acc[0].x = fmaf(a.x, w.x, acc[0].x), acc[0].y = fmaf(a.x, w.y, acc[0].y), acc[0].z = fmaf(a.x, w.z, acc[0].z), acc[0].w = fmaf(a.x, w.w, acc[0].w);
        acc[1].x = fmaf(a.y, w.x, acc[1].x), acc[1].y = fmaf(a.y, w.y, acc[1].y), acc[1].z = fmaf(a.y, w.z, acc[1].z), acc[1].w = fmaf(a.y, w.w, acc[1].w);
        acc[2].x = fmaf(a.z, w.x, acc[2].x), acc[2].y = fmaf(a.z, w.y, acc[2].y), acc[2].z = fmaf(a.z, w.z, acc[2].z), acc[2].w = fmaf(a.z, w.w, acc[2].w);
        acc[3].x = fmaf(a.w, w.x, acc[3].x), acc[3].y = fmaf(a.w, w.y, acc[3].y), acc[3].z = fmaf(a.w, w.z, acc[3].z), acc[3].w = fmaf(a.w, w.w, acc[3].w);
    }
    const float4 bv = ldg_f4(bias + n0 + tx * 4);
#pragma unroll
    for (int i = 0; i < 4; ++i) {
        const int r = row0 + ty * 4 + i;
        if (r < rows)
            *reinterpret_cast<float4 *>(qkv + (int64_t)r * (3 * C) + n0 + tx * 4) =
                make_float4(acc[i].x + bv.x, acc[i].y + bv.y, acc[i].z + bv.z, acc[i].w + bv.w);
    }
}

// ---- attention over a few hundred tokens, head_dim 32 --------------------------------------------------------------
// grid (heads, batch, query tiles); 512 threads.  Shared memory: K^T [32][n_pad], V [n][32], Q^T tile [32][q_pad]
// (pre-scaled), scores / probabilities TRANSPOSED Pt [n_pad][q_pad], 1/row-sum.  Both products use 4x4 register
// tiles fed by two 128-bit shared-memory loads per 16 FMAs (shared-memory bandwidth was the limit of the first version).
constexpr int kAttThreads = 512;

__global__ void __launch_bounds__(kAttThreads) attn_rows_kernel(const float *__restrict__ q, const float *__restrict__ kmat,
                                                                const float *__restrict__ v, int64_t stride_qk,
                                                                int64_t stride_v, float *__restrict__ out, int n, int heads,
                                                                float scale, int q_tile, int n_pad) {
    extern __shared__ __align__(16) float sm_att[];
    const int q_pad = q_tile <= 36 ? 36 : 68;     // >= q_tile (a multiple of 4, <= 64) and == 4 (mod 32)
    float *Kt = sm_att;                           // [32][n_pad]
    float *Vs = Kt + 32 * n_pad;                  // [n][32]
    float *Qt = Vs + (size_t)n * 32;              // [32][q_pad]
    float *Pt = Qt + 32 * q_pad;                  // [n_pad][q_pad]
    float *inv = Pt + (size_t)n_pad * q_pad;      // [q_tile]
    float *red = inv + q_tile;                    // [splits][q_tile][32] partial outputs
    const int h = blockIdx.x, b = blockIdx.y, tid = threadIdx.x;
    const int q_base = blockIdx.z * q_tile;
    const int q_cnt = min(q_tile, n - q_base);
    if (q_cnt <= 0) return;
    const float *qb = q + (int64_t)b * n * stride_qk + h * 32;
    const float *kb = kmat + (int64_t)b * n * stride_qk + h * 32;
    const float *vb = v + (int64_t)b * n * stride_v + h * 32;
    // K transposed (thread <-> key: conflict-free stores), V row-major, Q transposed and pre-scaled
    for (int item = tid; item < 8 * n; item += kAttThreads) {
        const int c4 = item / n, j = item - c4 * n;
        const float4 kv = ldg_f4(kb + (int64_t)j * stride_qk + c4 * 4);
        Kt[(c4 * 4) * n_pad + j] = kv.x, Kt[(c4 * 4 + 1) * n_pad + j] = kv.y;
        Kt[(c4 * 4 + 2) * n_pad + j] = kv.z, Kt[(c4 * 4 + 3) * n_pad + j] = kv.w;
    }
    for (int item = tid; item < 32 * (n_pad - n); item += kAttThreads) {  // zero the key padding (read by the 4-key tiles)
        const int c = item / (n_pad - n), j = n + item % (n_pad - n);
        Kt[c * n_pad + j] = 0.f;
    }
    for (int item = tid; item < 8 * n; item += kAttThreads) {
        const int j = item >> 3, c = (item & 7) * 4;
        *reinterpret_cast<float4 *>(Vs + j * 32 + c) = ldg_f4(vb + (int64_t)j * stride_v + c);
    }
    for (int item = tid; item < 8 * q_tile; item += kAttThreads) {
        const int c4 = item / q_tile, i = item - c4 * q_tile;
        float4 qv = make_float4(0.f, 0.f, 0.f, 0.f);
        if (i < q_cnt) qv = ldg_f4(qb + (int64_t)(q_base + i) * stride_qk + c4 * 4);
        Qt[(c4 * 4) * q_pad + i] = qv.x * scale, Qt[(c4 * 4 + 1) * q_pad + i] = qv.y * scale;
        Qt[(c4 * 4 + 2) * q_pad + i] = qv.z * scale, Qt[(c4 * 4 + 3) * q_pad + i] = qv.w * scale;
    }
    __syncthreads();
    // S^T = K (Q * scale)^T: thread tile 4 keys x 4 queries
    {
        const int tiles_k = (n + 3) >> 2, groups = q_tile >> 2;
        for (int id = tid; id < groups * tiles_k; id += kAttThreads) {
            const int qg = id / tiles_k, j4 = (id - qg * tiles_k) * 4;
            const float *kp = Kt + j4, *qp = Qt + qg * 4;
            float4 s0 = make_float4(0.f, 0.f, 0.f, 0.f), s1 = s0, s2 = s0, s3 = s0;  // s_i: key j4 + i, 4 queries
#pragma unroll 8
            for (int c = 0; c < 32; ++c) {
                const float4 kv = *reinterpret_cast<const float4 *>(kp + c * n_pad);
                const float4 qv = *reinterpret_cast<const float4 *>(qp + c * q_pad);
                s0.x = fmaf(kv.x, qv.x, s0.x), s0.y = fmaf(kv.x, qv.y, s0.y), s0.z = fmaf(kv.x, qv.z, s0.z), s0.w = fmaf(kv.x, qv.w, s0.w);
                s1.x = fmaf(kv.y, qv.x, s1.x), s1.y = fmaf(kv.y, qv.y, s1.y), s1.z = fmaf(kv.y, qv.z, s1.z), s1.w = fmaf(kv.y, qv.w, s1.w);
                s2.x = fmaf(kv.z, qv.x, s2.x), s2.y = fmaf(kv.z, qv.y, s2.y), s2.z = fmaf(kv.z, qv.z, s2.z), s2.w = fmaf(kv.z, qv.w, s2.w);
                s3.x = fmaf(kv.w, qv.x, s3.x), s3.y = fmaf(kv.w, qv.y, s3.y), s3.z = fmaf(kv.w, qv.z, s3.z), s3.w = fmaf(kv.w, qv.w, s3.w);
            }
            float *pp = Pt + j4 * q_pad + qg * 4;
            *reinterpret_cast<float4 *>(pp) = s0;
            *reinterpret_cast<float4 *>(pp + q_pad) = s1;
            *reinterpret_cast<float4 *>(pp + 2 * q_pad) = s2;
            *reinterpret_cast<float4 *>(pp + 3 * q_pad) = s3;
        }
    }
    __syncthreads();
    // softmax over the keys of each query (a column of Pt); warp <-> group of 4 queries, lane <-> key, 128-bit accesses
    // (q_pad % 32 == 4 keeps them bank-conflict free); unnormalised probabilities stay in Pt
    {
        const int warp = tid >> 5, lane = tid & 31;
        for (int qg = warp; qg * 4 < q_cnt; qg += kAttThreads / 32) {
            float *p = Pt + qg * 4;
            float4 mx = make_float4(-INFINITY, -INFINITY, -INFINITY, -INFINITY);
            for (int j = lane; j < n; j += 32) {
                const float4 x = *reinterpret_cast<const float4 *>(p + j * q_pad);
                mx.x = fmaxf(mx.x, x.x), mx.y = fmaxf(mx.y, x.y), mx.z = fmaxf(mx.z, x.z), mx.w = fmaxf(mx.w, x.w);
            }
#pragma unroll
            for (int o = 16; o > 0; o >>= 1) {
                mx.x = fmaxf(mx.x, __shfl_xor_sync(0xffffffffu, mx.x, o)), mx.y = fmaxf(mx.y, __shfl_xor_sync(0xffffffffu, mx.y, o));
                mx.z = fmaxf(mx.z, __shfl_xor_sync(0xffffffffu, mx.z, o)), mx.w = fmaxf(mx.w, __shfl_xor_sync(0xffffffffu, mx.w, o));
            }
            float4 sum = make_float4(0.f, 0.f, 0.f, 0.f);
            for (int j = lane; j < n; j += 32) {
                float4 x = *reinterpret_cast<const float4 *>(p + j * q_pad);
                x.x = expf(x.x - mx.x), x.y = expf(x.y - mx.y), x.z = expf(x.z - mx.z), x.w = expf(x.w - mx.w);
                *reinterpret_cast<float4 *>(p + j * q_pad) = x;
                sum.x += x.x, sum.y += x.y, sum.z += x.z, sum.w += x.w;
            }
#pragma unroll
            for (int o = 16; o > 0; o >>= 1) {
                sum.x += __shfl_xor_sync(0xffffffffu, sum.x, o), sum.y += __shfl_xor_sync(0xffffffffu, sum.y, o);
                sum.z += __shfl_xor_sync(0xffffffffu, sum.z, o), sum.w += __shfl_xor_sync(0xffffffffu, sum.w, o);
            }
            if (lane == 0) *reinterpret_cast<float4 *>(inv + qg * 4) = make_float4(1.f / sum.x, 1.f / sum.y, 1.f / sum.z, 1.f / sum.w);
        }
    }
    __syncthreads();
    // O = P V: thread = (key split, 4 queries, 4 channels); partial sums reduced through shared memory in split order
    {
        const int groups = q_tile >> 2, per_split = groups * 8;
        const int splits = kAttThreads / per_split;  // >= 1 (q_tile <= 64)
        const int s = tid / per_split, rem = tid - s * per_split;
        const int qg = rem >> 3, d4 = (rem & 7) * 4;
        if (s < splits) {
            const int chunk = (n + splits - 1) / splits, j0 = s * chunk, j1 = min(n, j0 + chunk);
            float4 a0 = make_float4(0.f, 0.f, 0.f, 0.f), a1 = a0, a2 = a0, a3 = a0;  // a_i: query qg*4 + i, 4 channels
            const float *pp = Pt + qg * 4, *vp = Vs + d4;
#pragma unroll 4
            for (int j = j0; j < j1; ++j) {
                const float4 pv = *reinterpret_cast<const float4 *>(pp + j * q_pad);
                const float4 vv = *reinterpret_cast<const float4 *>(vp + j * 32);
                a0.x = fmaf(pv.x, vv.x, a0.x), a0.y = fmaf(pv.x, vv.y, a0.y), a0.z = fmaf(pv.x, vv.z, a0.z), a0.w = fmaf(pv.x, vv.w, a0.w);
                a1.x = fmaf(pv.y, vv.x, a1.x), a1.y = fmaf(pv.y, vv.y, a1.y), a1.z = fmaf(pv.y, vv.z, a1.z), a1.w = fmaf(pv.y, vv.w, a1.w);
                a2.x = fmaf(pv.z, vv.x, a2.x), a2.y = fmaf(pv.z, vv.y, a2.y), a2.z = fmaf(pv.z, vv.z, a2.z), a2.w = fmaf(pv.z, vv.w, a2.w);
                a3.x = fmaf(pv.w, vv.x, a3.x), a3.y = fmaf(pv.w, vv.y, a3.y), a3.z = fmaf(pv.w, vv.z, a3.z), a3.w = fmaf(pv.w, vv.w, a3.w);
            }
            float *rp = red + ((size_t)s * q_tile + qg * 4) * 32 + d4;
            *reinterpret_cast<float4 *>(rp) = a0;
            *reinterpret_cast<float4 *>(rp + 32) = a1;
            *reinterpret_cast<float4 *>(rp + 64) = a2;
            *reinterpret_cast<float4 *>(rp + 96) = a3;
        }
        __syncthreads();
        for (int id = tid; id < q_cnt * 8; id += kAttThreads) {
            const int i = id >> 3, c = (id & 7) * 4;
            float4 acc = *reinterpret_cast<const float4 *>(red + (size_t)i * 32 + c);
            for (int t = 1; t < splits; ++t) {
                const float4 x = *reinterpret_cast<const float4 *>(red + ((size_t)t * q_tile + i) * 32 + c);
                acc.x += x.x, acc.y += x.y, acc.z += x.z, acc.w += x.w;
            }
            const float sc = inv[i];
            *reinterpret_cast<float4 *>(out + ((int64_t)b * n + q_base + i) * (heads * 32) + h * 32 + c) =
                make_float4(acc.x * sc, acc.y * sc, acc.z * sc, acc.w * sc);
        }
    }
}

// ---- out-projection + residual + LayerNorm + scatter ---------------------------------------------------------------
// 8 rows per CTA, all C output columns (so the LayerNorm row statistics stay inside the CTA); 128 threads, thread tile
// 4 rows x 4 columns on a transposed activation tile; W^T streams through shared memory in 64-row chunks,
// double-buffered with cp.async.
constexpr int kOutRows = 8, kOutThreads = 128, kOutChunk = 64;

template <int C>
__global__ void __launch_bounds__(kOutThreads) mha_out_proj_ln_scatter_kernel(
    const float *__restrict__ attn /* (rows, C) */, const float *__restrict__ t /* (rows, C) */,
    const float *__restrict__ w_t /* (C, C) */, const float *__restrict__ bias, const float *__restrict__ gamma,
    const float *__restrict__ beta, float eps, const int64_t *__restrict__ index, float *__restrict__ dst /* (b, nq, C) */,
    const float *__restrict__ pos /* (b, nq, C) or null */, float *__restrict__ dst_sum /* (b, nq, C) or null */, int nq,
    int k, int rows) {
    static_assert(C == 256, "thread mapping assumes 64 column groups of 4");
    extern __shared__ __align__(16) float sm_out[];
    float *At = sm_out;                          // [C][8]: At[kk][row]
    float *Ws = At + C * kOutRows;               // 2 x [64][C]
    float *Ys = Ws + 2 * kOutChunk * C;          // [8][C]
    const int tid = threadIdx.x, row0 = blockIdx.x * kOutRows;
    auto load_chunk = [&](int chunk, int buf) {
        const float *src = w_t + (int64_t)chunk * kOutChunk * C;
        float *d = Ws + buf * kOutChunk * C;
        for (int item = tid; item < kOutChunk * C / 4; item += kOutThreads) cp_async16(d + item * 4, src + item * 4);
        asm volatile("cp.async.commit_group;" ::: "memory");
    };
    load_chunk(0, 0);
    {
        constexpr int kPer = kOutRows * (C / 4) / kOutThreads;
        float4 av[kPer];
#pragma unroll
        for (int u = 0; u < kPer; ++u) {
            const int item = tid + u * kOutThreads;
            const int i = item % kOutRows, c = (item / kOutRows) * 4;
            const int r = row0 + i;
            av[u] = r < rows ? ldg_f4(attn + (int64_t)r * C + c) : make_float4(0.f, 0.f, 0.f, 0.f);
        }
#pragma unroll
        for (int u = 0; u < kPer; ++u) {
            const int item = tid + u * kOutThreads;
            const int i = item % kOutRows, c = (item / kOutRows) * 4;
            At[(c + 0) * kOutRows + i] = av[u].x, At[(c + 1) * kOutRows + i] = av[u].y;
            At[(c + 2) * kOutRows + i] = av[u].z, At[(c + 3) * kOutRows + i] = av[u].w;
        }
    }
    const int tx = tid & 63, ty = tid >> 6;
    const float *ap = At + ty * 4;
    float4 acc[4];
#pragma unroll
    for (int i = 0; i < 4; ++i) acc[i] = make_float4(0.f, 0.f, 0.f, 0.f);
    constexpr int kChunks = C / kOutChunk;
    for (int chunk = 0; chunk < kChunks; ++chunk) {
        if (chunk + 1 < kChunks) {
            load_chunk(chunk + 1, (chunk + 1) & 1);
            asm volatile("cp.async.wait_group 1;" ::: "memory");
        } else {
            asm volatile("cp.async.wait_group 0;" ::: "memory");
        }
        __syncthreads();
        const float *wp = Ws + (chunk & 1) * kOutChunk * C + tx * 4;
        const int kbase = chunk * kOutChunk;
#pragma unroll 8
        for (int kk = 0; kk < kOutChunk; ++kk) {
            const float4 a = *reinterpret_cast<const float4 *>(ap + (kbase + kk) * kOutRows);
            const float4 w = *reinterpret_cast<const float4 *>(wp + kk * C);
            acc[0].x = fmaf(a.x, w.x, acc[0].x), acc[0].y = fmaf(a.x, w.y, acc[0].y), acc[0].z = fmaf(a.x, w.z, acc[0].z), acc[0].w = fmaf(a.x, w.w, acc[0].w);
            acc[1].x = fmaf(a.y, w.x, acc[1].x), acc[1].y = fmaf(a.y, w.y, acc[1].y), acc[1].z = fmaf(a.y, w.z, acc[1].z), acc[1].w = fmaf(a.y, w.w, acc[1].w);
            acc[2].x = fmaf(a.z, w.x, acc[2].x), acc[2].y = fmaf(a.z, w.y, acc[2].y), acc[2].z = fmaf(a.z, w.z, acc[2].z), acc[2].w = fmaf(a.z, w.w, acc[2].w);
            acc[3].x = fmaf(a.w, w.x, acc[3].x), acc[3].y = fmaf(a.w, w.y, acc[3].y), acc[3].z = fmaf(a.w, w.z, acc[3].z), acc[3].w = fmaf(a.w, w.w, acc[3].w);
        }
        __syncthreads();  // everyone is done with this buffer before the chunk after next overwrites it
    }
    // + bias + residual -> Ys
    {
        const float4 bv = ldg_f4(bias + tx * 4);
#pragma unroll
        for (int i = 0; i < 4; ++i) {
            const int r = row0 + ty * 4 + i;
            float4 tr = make_float4(0.f, 0.f, 0.f, 0.f);
            if (r < rows) tr = ldg_f4(t + (int64_t)r * C + tx * 4);
            *reinterpret_cast<float4 *>(Ys + (ty * 4 + i) * C + tx * 4) =
                make_float4(tr.x + (acc[i].x + bv.x), tr.y + (acc[i].y + bv.y), tr.z + (acc[i].z + bv.z), tr.w + (acc[i].w + bv.w));
        }
    }
    __syncthreads();
    // LayerNorm (same arithmetic as add_layernorm_kernel) + scatter: each warp takes rows warp, warp + 4
    const int warp = tid >> 5, lane = tid & 31;
    for (int rr = warp; rr < kOutRows; rr += kOutThreads / 32) {
        const int r = row0 + rr;
        if (r >= rows) break;
        float4 vv[C / 128];
        float s = 0.f;
#pragma unroll
        for (int i = 0; i < C / 128; ++i) {
            vv[i] = *reinterpret_cast<const float4 *>(Ys + rr * C + i * 128 + lane * 4);
            s += (vv[i].x + vv[i].y) + (vv[i].z + vv[i].w);
        }
#pragma unroll
        for (int o = 16; o > 0; o >>= 1) s += __shfl_xor_sync(0xffffffffu, s, o);
        const float mean = s / (float)C;
        float ss = 0.f;
#pragma unroll
        for (int i = 0; i < C / 128; ++i) {
            const float dx = vv[i].x - mean, dy = vv[i].y - mean, dz = vv[i].z - mean, dw = vv[i].w - mean;
            ss += (dx * dx + dy * dy) + (dz * dz + dw * dw);
        }
#pragma unroll
        for (int o = 16; o > 0; o >>= 1) ss += __shfl_xor_sync(0xffffffffu, ss, o);
        const float rstd = rsqrtf(ss / (float)C + eps);
        const int b = r / k;
        const int64_t drow_off = ((int64_t)b * nq + __ldg(index + r)) * C;
        float *drow = dst + drow_off;
#pragma unroll
        for (int i = 0; i < C / 128; ++i) {
            const int c = i * 128 + lane * 4;
            const float4 g = ldg_f4(gamma + c), bt = ldg_f4(beta + c);
            float4 o;
            o.x = (vv[i].x - mean) * rstd * g.x + bt.x, o.y = (vv[i].y - mean) * rstd * g.y + bt.y;
            o.z = (vv[i].z - mean) * rstd * g.z + bt.z, o.w = (vv[i].w - mean) * rstd * g.w + bt.w;
            *reinterpret_cast<float4 *>(drow + c) = o;
            if (dst_sum) {  // keep the layer's `query + query_pos` buffer current for the rewritten rows
                const float4 pp = ldg_f4(pos + drow_off + c);
                *reinterpret_cast<float4 *>(dst_sum + drow_off + c) = make_float4(o.x + pp.x, o.y + pp.y, o.z + pp.z, o.w + pp.w);
            }
        }
    }
}

}  // namespace sdetr

using namespace sdetr;

extern "C" int sdetr_mha_in_proj(const float *tokens, const float *pos, const int64_t *index, int batch, int num_rows, int k,
                                 int channels, const float *w_in_t, const float *b_in, float *t_out, float *qkv,
                                 sdetr_stream_t stream) {
    SDETR_REQUIRE(batch > 0 && num_rows > 0 && k >= 0 && k <= num_rows, SDETR_ERR_INVALID_ARG, "mha_in_proj: bad sizes");
    SDETR_REQUIRE(channels == 256, SDETR_ERR_UNSUPPORTED, "mha_in_proj: channels %d (only 256)", channels);
    if (k == 0) return SDETR_OK;  // no rows: the empty index and outputs may be null
    SDETR_REQUIRE(tokens && pos && index && w_in_t && b_in && t_out && qkv, SDETR_ERR_INVALID_ARG, "mha_in_proj: null pointer");
    SDETR_REQUIRE(aligned16(tokens) && aligned16(pos) && aligned16(w_in_t) && aligned16(b_in) && aligned16(t_out) && aligned16(qkv),
                  SDETR_ERR_INVALID_ARG, "mha_in_proj: 16-byte alignment required");
    constexpr int C = 256;
    const int rows = batch * k;
    const size_t smem = (size_t)(C * kInPitch + C * kInCols) * sizeof(float);
    static PerDeviceOnce once;
    SDETR_OPT_IN_SMEM(once, mha_in_proj_kernel<C>, smem, "mha_in_proj");
    dim3 grid((rows + kInRows - 1) / kInRows, 3 * C / kInCols);
    mha_in_proj_kernel<C><<<grid, kInThreads, smem, (cudaStream_t)stream>>>(tokens, pos, index, num_rows, k, rows, w_in_t, b_in,
                                                                            t_out, qkv);
    return check_launch("mha_in_proj");
}

static int launch_attention(const float *q, const float *kmat, const float *v, int64_t stride_qk, int64_t stride_v, float *out,
                            int batch, int n, int heads, int head_dim, cudaStream_t stream, const char *what) {
    SDETR_REQUIRE(q && kmat && v && out, SDETR_ERR_INVALID_ARG, "%s: null pointer", what);
    SDETR_REQUIRE(batch > 0 && n > 0 && heads > 0, SDETR_ERR_INVALID_ARG, "%s: bad sizes", what);
    SDETR_REQUIRE(head_dim == 32, SDETR_ERR_UNSUPPORTED, "%s: head_dim %d (only 32)", what, head_dim);
    SDETR_REQUIRE(aligned16(q) && aligned16(kmat) && aligned16(v) && aligned16(out) && stride_qk % 4 == 0 && stride_v % 4 == 0,
                  SDETR_ERR_INVALID_ARG, "%s: 16-byte alignment required", what);
    const int sms = sm_count();
    // one CTA per SM: as many query tiles as fit in one wave
    const int slots = sms / (batch * heads) > 0 ? sms / (batch * heads) : 1;
    int q_tile = (n + slots - 1) / slots;
    q_tile = (q_tile + 3) & ~3;
    if (q_tile < 8) q_tile = 8;
    if (q_tile > 64) q_tile = 64;
    const int n_pad = ((n + 3) & ~3) + 4;
    const size_t limit = 220 * 1024;
    auto smem_for = [&](int qt) {  // K^T, V, Q^T, P^T, 1/sum, split partials (kAttThreads / (2 qt) splits of qt x 32)
        const int splits = kAttThreads / ((qt >> 2) * 8);
        const int q_pad = qt <= 36 ? 36 : 68;
        return ((size_t)32 * n_pad + (size_t)n * 32 + (size_t)32 * q_pad + (size_t)n_pad * q_pad + qt +
                (size_t)splits * qt * 32) * sizeof(float);
    };
    while (q_tile > 8 && smem_for(q_tile) > limit) q_tile -= 4;  // long sequences: smaller query tiles
    SDETR_REQUIRE(smem_for(q_tile) <= limit, SDETR_ERR_UNSUPPORTED, "%s: %d tokens do not fit in shared memory", what, n);
    const size_t smem = smem_for(q_tile);
    static PerDeviceOnce once;
    SDETR_OPT_IN_SMEM(once, attn_rows_kernel, 220 * 1024, what);
    dim3 grid(heads, batch, (n + q_tile - 1) / q_tile);
    attn_rows_kernel<<<grid, kAttThreads, smem, stream>>>(q, kmat, v, stride_qk, stride_v, out, n, heads,
                                                          1.f / sqrtf((float)head_dim), q_tile, n_pad);
    return check_launch(what);
}

extern "C" int sdetr_attention_qkv(const float *qkv, float *out, int batch, int n, int heads, int head_dim,
                                   sdetr_stream_t stream) {
    const int64_t c = (int64_t)heads * head_dim;
    return launch_attention(qkv, qkv ? qkv + c : nullptr, qkv ? qkv + 2 * c : nullptr, 3 * c, 3 * c, out, batch, n, heads,
                            head_dim, (cudaStream_t)stream, "attention_qkv");
}

extern "C" int sdetr_mha_out_proj_ln_scatter(const float *attn, const float *t, const float *w_out_t, const float *b_out,
                                             const float *gamma, const float *beta, float eps, const int64_t *index,
                                             float *dst, const float *pos, float *dst_sum, int batch, int num_rows, int k,
                                             int channels, sdetr_stream_t stream) {
    SDETR_REQUIRE(batch > 0 && num_rows > 0 && k >= 0 && k <= num_rows, SDETR_ERR_INVALID_ARG, "mha_out_proj_ln_scatter: bad sizes");
    SDETR_REQUIRE(channels == 256, SDETR_ERR_UNSUPPORTED, "mha_out_proj_ln_scatter: channels %d (only 256)", channels);
    if (k == 0) return SDETR_OK;  // no rows: the empty index and inputs may be null
    SDETR_REQUIRE(attn && t && w_out_t && b_out && gamma && beta && index && dst, SDETR_ERR_INVALID_ARG,
                  "mha_out_proj_ln_scatter: null pointer");
    SDETR_REQUIRE((pos == nullptr) == (dst_sum == nullptr) && aligned16(pos) && aligned16(dst_sum), SDETR_ERR_INVALID_ARG,
                  "mha_out_proj_ln_scatter: pos and dst_sum go together (16-byte aligned)");
    SDETR_REQUIRE(aligned16(attn) && aligned16(t) && aligned16(w_out_t) && aligned16(b_out) && aligned16(gamma) && aligned16(beta) &&
                      aligned16(dst),
                  SDETR_ERR_INVALID_ARG, "mha_out_proj_ln_scatter: 16-byte alignment required");
    constexpr int C = 256;
    const int rows = batch * k;
    const size_t smem = (size_t)(C * kOutRows + 2 * kOutChunk * C + kOutRows * C) * sizeof(float);
    static PerDeviceOnce once;
    SDETR_OPT_IN_SMEM(once, mha_out_proj_ln_scatter_kernel<C>, smem, "mha_out_proj_ln_scatter");
    mha_out_proj_ln_scatter_kernel<C><<<(rows + kOutRows - 1) / kOutRows, kOutThreads, smem, (cudaStream_t)stream>>>(
        attn, t, w_out_t, b_out, gamma, beta, eps, index, dst, pos, dst_sum, num_rows, k, rows);
    return check_launch("mha_out_proj_ln_scatter");
}
