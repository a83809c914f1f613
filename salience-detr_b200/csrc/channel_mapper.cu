// ChannelMapper in token layout (models/necks/channel_mapper.py:8-80): the kernels behind ChannelMapper.forward_tokens and the
// transformer's front end for features that are already tokens.
//
//   sdetr_group_norm_tokens  nn.GroupNorm of every level of a (b, Nv, C) token buffer, three launches for all levels:
//                            (1) one CTA per (image, 64-token tile of a level) computes, per channel, the Welford (mean, M2)
//                                of its rows (in the frame shifted by the tile's first row); (2) one CTA per (group, level, image) merges the tiles' and channels' partials
//                                with Chan's formula in a fixed order and writes (mean, rstd); (3) the affine apply, same tiles
//                                as (1).  No atomics: the result depends only on the data, never on the grid or launch order.
//   sdetr_group_norm_tokens_backward  its gradient: the forward's (1) and (2) recompute the statistics, then (1') per-tile sums
//                            of dy and dy * xhat, (2') one CTA per (group, level, image) forms the two group means, (3') per
//                            (level, channel) dgamma / dbeta, (4') the element-wise dx.  Equally free of atomics.
//   sdetr_token_lpos_keep    lpos = pos + level_embeds[l], x = (feat + lpos) * keep, on token rows: the same fp32 operations in
//                            the same order as sdetr_flatten_tokens[_pos], so both outputs are bit-identical to theirs.
#include <math.h>

#include "common.cuh"

namespace sdetr {

constexpr int kGnTile = 64;           // tokens per partial-statistics tile
constexpr int kGnCombineThreads = 128;

struct GnLevels {
    int size[kMaxLevels], start[kMaxLevels], tile0[kMaxLevels + 1];
    int L;
};

__device__ __forceinline__ int gn_level_of_tile(const GnLevels &lv, int tile) {
    int l = 0;
#pragma unroll
    for (int u = 1; u < kMaxLevels; ++u)
        if (u < lv.L && tile >= lv.tile0[u]) l = u;
    return l;
}

// Chan et al.: (na, ma, M2a) <- (na, ma, M2a) + (nb, mb, M2b)
__device__ __forceinline__ void chan_merge(float &na, float &ma, float &qa, float nb, float mb, float qb) {
    if (nb == 0.f) return;
    if (na == 0.f) {
        na = nb, ma = mb, qa = qb;
        return;
    }
    const float n = na + nb, d = mb - ma, f = nb / n;
    ma = ma + d * f;
    qa = qa + qb + d * d * na * f;
    na = n;
}

// threads = C4 * R: thread (r, j) owns channels 4j .. 4j+3 and the tile's rows r, r + R, ...
__global__ void gn_partial_kernel(const float *__restrict__ x, int64_t pitch, int C, GnLevels lv, int total_tiles,
                                  float *__restrict__ pmean, float *__restrict__ pm2) {
    extern __shared__ float gn_smem[];
    const int C4 = C / 4, R = blockDim.x / C4;
    const int j = threadIdx.x % C4, r = threadIdx.x / C4;
    const int tile = blockIdx.x, b = blockIdx.y;
    const int l = gn_level_of_tile(lv, tile);
    const int t0 = (tile - lv.tile0[l]) * kGnTile;
    const int rows = min(kGnTile, lv.size[l] - t0);
    const float *src = x + (int64_t)b * pitch + (int64_t)(lv.start[l] + t0) * C + 4 * j;
    // every lane works in the frame shifted by the tile's first row: the running means stay O(std) even when |mean| >> std
    const float4 k = ldg_f4(src);
    float4 mean = make_float4(0.f, 0.f, 0.f, 0.f), m2 = mean;
    int n = 0;
    for (int t = r; t < rows; t += R) {
        float4 v = ld_stream_f4(src + (int64_t)t * C);
        v.x -= k.x, v.y -= k.y, v.z -= k.z, v.w -= k.w;
        ++n;
        const float inv = 1.f / (float)n;
        float d;
        d = v.x - mean.x, mean.x += d * inv, m2.x += d * (v.x - mean.x);
        d = v.y - mean.y, mean.y += d * inv, m2.y += d * (v.y - mean.y);
        d = v.z - mean.z, mean.z += d * inv, m2.z += d * (v.z - mean.z);
        d = v.w - mean.w, mean.w += d * inv, m2.w += d * (v.w - mean.w);
    }
    float *sm = gn_smem, *sq = gn_smem + R * C;  // [R][C] each
    *reinterpret_cast<float4 *>(sm + r * C + 4 * j) = mean;
    *reinterpret_cast<float4 *>(sq + r * C + 4 * j) = m2;
    __syncthreads();
    if (r != 0) return;
    // lanes r = 0 .. R-1 merged in order; lane r holds ceil((rows - r) / R) rows
    const int64_t o = ((int64_t)b * total_tiles + tile) * C + 4 * j;
#pragma unroll
    for (int e = 0; e < 4; ++e) {
        float na = 0.f, ma = 0.f, qa = 0.f;
        for (int u = 0; u < R; ++u) {
            const float nb = (float)(u < rows ? (rows - u + R - 1) / R : 0);
            chan_merge(na, ma, qa, nb, sm[u * C + 4 * j + e], sq[u * C + 4 * j + e]);
        }
        pmean[o + e] = ma + (e == 0 ? k.x : e == 1 ? k.y : e == 2 ? k.z : k.w);
        pm2[o + e] = qa;
    }
}

// one CTA per (group, level, image): the level's tiles x the group's channels, each thread a strided share in order, then a
// fixed tree.  stats[(b * L + l) * G + g] = (mean, rstd)
__global__ void __launch_bounds__(kGnCombineThreads) gn_combine_kernel(const float *__restrict__ pmean, const float *__restrict__ pm2,
                                                                       int C, int G, GnLevels lv, int total_tiles, float eps,
                                                                       float2 *__restrict__ stats) {
    __shared__ float sn[kGnCombineThreads], sm[kGnCombineThreads], sq[kGnCombineThreads];
    const int g = blockIdx.x, l = blockIdx.y, b = blockIdx.z, cg = C / G;
    int size = 0, tile0 = 0, ntiles = 0;  // lv.*[l] by selection: a dynamic index into the parameter struct would go to local memory
#pragma unroll
    for (int u = 0; u < kMaxLevels; ++u)
        if (u == l) size = lv.size[u], tile0 = lv.tile0[u], ntiles = lv.tile0[u + 1] - lv.tile0[u];
    const int64_t items = (int64_t)ntiles * cg;
    const float *pm = pmean + ((int64_t)b * total_tiles + tile0) * C, *pq = pm2 + ((int64_t)b * total_tiles + tile0) * C;
    const float shift = __ldg(pm + g * cg);  // merged in the frame of the first partial mean: the merge sums stay O(std)
    float na = 0.f, ma = 0.f, qa = 0.f;
    for (int64_t k = threadIdx.x; k < items; k += kGnCombineThreads) {
        const int tl = (int)(k / cg), c = g * cg + (int)(k % cg);
        const float nb = (float)min(kGnTile, size - tl * kGnTile);
        chan_merge(na, ma, qa, nb, __ldg(pm + (int64_t)tl * C + c) - shift, __ldg(pq + (int64_t)tl * C + c));
    }
    sn[threadIdx.x] = na, sm[threadIdx.x] = ma, sq[threadIdx.x] = qa;
    __syncthreads();
    for (int s = kGnCombineThreads / 2; s > 0; s >>= 1) {
        if ((int)threadIdx.x < s) {
            float n0 = sn[threadIdx.x], m0 = sm[threadIdx.x], q0 = sq[threadIdx.x];
            chan_merge(n0, m0, q0, sn[threadIdx.x + s], sm[threadIdx.x + s], sq[threadIdx.x + s]);
            sn[threadIdx.x] = n0, sm[threadIdx.x] = m0, sq[threadIdx.x] = q0;
        }
        __syncthreads();
    }
    if (threadIdx.x == 0) {
        const float var = fmaxf(sq[0] / sn[0], 0.f);  // biased, as nn.GroupNorm
        stats[((int64_t)b * lv.L + l) * G + g] = make_float2(shift + sm[0], rsqrtf(var + eps));
    }
}

// y = (x - mean) * (rstd * gamma) + beta; y may alias x (each element is read, then written, by the same thread)
__global__ void gn_apply_kernel(const float *x, float *y, int64_t pitch, int C, int G, GnLevels lv,
                                const float *__restrict__ gamma, const float *__restrict__ beta,
                                const float2 *__restrict__ stats) {
    const int C4 = C / 4, R = blockDim.x / C4;
    const int j = threadIdx.x % C4, r = threadIdx.x / C4, c = 4 * j, cg = C / G;
    const int tile = blockIdx.x, b = blockIdx.y;
    const int l = gn_level_of_tile(lv, tile);
    const int t0 = (tile - lv.tile0[l]) * kGnTile;
    const int rows = min(kGnTile, lv.size[l] - t0);
    const float4 ga = ldg_f4(gamma + (int64_t)l * C + c), be = ldg_f4(beta + (int64_t)l * C + c);
    const float2 *st = stats + ((int64_t)b * lv.L + l) * G;
    const float2 s0 = st[(c + 0) / cg], s1 = st[(c + 1) / cg], s2 = st[(c + 2) / cg], s3 = st[(c + 3) / cg];
    const float a0 = s0.y * ga.x, a1 = s1.y * ga.y, a2 = s2.y * ga.z, a3 = s3.y * ga.w;
    const int64_t base = (int64_t)b * pitch + (int64_t)(lv.start[l] + t0) * C + c;
    for (int t = r; t < rows; t += R) {
        const int64_t o = base + (int64_t)t * C;
        const float4 v = *reinterpret_cast<const float4 *>(x + o);
        *reinterpret_cast<float4 *>(y + o) = make_float4(fmaf(v.x - s0.x, a0, be.x), fmaf(v.y - s1.x, a1, be.y),
                                                         fmaf(v.z - s2.x, a2, be.z), fmaf(v.w - s3.x, a3, be.w));
    }
}

// ---- backward: (dy, x) -> dx = rstd * (gamma dy - mean_grp(gamma dy) - xhat mean_grp(gamma dy xhat)), dgamma, dbeta ------------
__device__ __forceinline__ float4 sm4(const float *p, int c) { return *reinterpret_cast<const float4 *>(p + c); }

// (1) same tiles and threads as gn_partial_kernel: per channel, sum of dy and of dy * xhat over the tile's rows, each lane in row
// order, the lanes in order.  pdy / pdyx: [b][tile][C]
__global__ void gnb_partial_kernel(const float *__restrict__ dy, const float *__restrict__ x, int64_t pitch, int C, int G,
                                   GnLevels lv, int total_tiles, const float2 *__restrict__ stats, float *__restrict__ pdy,
                                   float *__restrict__ pdyx) {
    extern __shared__ float gn_smem[];
    const int C4 = C / 4, R = blockDim.x / C4;
    const int j = threadIdx.x % C4, r = threadIdx.x / C4, c = 4 * j, cg = C / G;
    const int tile = blockIdx.x, b = blockIdx.y;
    const int l = gn_level_of_tile(lv, tile);
    const int t0 = (tile - lv.tile0[l]) * kGnTile;
    const int rows = min(kGnTile, lv.size[l] - t0);
    const float2 *st = stats + ((int64_t)b * lv.L + l) * G;
    const float2 s0 = st[(c + 0) / cg], s1 = st[(c + 1) / cg], s2 = st[(c + 2) / cg], s3 = st[(c + 3) / cg];
    const int64_t base = (int64_t)b * pitch + (int64_t)(lv.start[l] + t0) * C + c;
    float4 sd = make_float4(0.f, 0.f, 0.f, 0.f), sx = sd;
    for (int t = r; t < rows; t += R) {
        const int64_t o = base + (int64_t)t * C;
        const float4 g = ld_stream_f4(dy + o), v = ld_stream_f4(x + o);
        sd.x += g.x, sx.x = fmaf(g.x, (v.x - s0.x) * s0.y, sx.x);
        sd.y += g.y, sx.y = fmaf(g.y, (v.y - s1.x) * s1.y, sx.y);
        sd.z += g.z, sx.z = fmaf(g.z, (v.z - s2.x) * s2.y, sx.z);
        sd.w += g.w, sx.w = fmaf(g.w, (v.w - s3.x) * s3.y, sx.w);
    }
    float *sm = gn_smem, *sq = gn_smem + R * C;  // [R][C] each
    *reinterpret_cast<float4 *>(sm + r * C + c) = sd;
    *reinterpret_cast<float4 *>(sq + r * C + c) = sx;
    __syncthreads();
    if (r != 0) return;
    float4 a = sm4(sm, c), q = sm4(sq, c);
    for (int u = 1; u < R; ++u) {
        const float4 p = sm4(sm + u * C, c), w = sm4(sq + u * C, c);
        a.x += p.x, a.y += p.y, a.z += p.z, a.w += p.w;
        q.x += w.x, q.y += w.y, q.z += w.z, q.w += w.w;
    }
    const int64_t o = ((int64_t)b * total_tiles + tile) * C + c;
    *reinterpret_cast<float4 *>(pdy + o) = a;
    *reinterpret_cast<float4 *>(pdyx + o) = q;
}

// (2) one CTA per (group, level, image): the level's tiles x the group's channels, gamma applied per channel, each thread a
// strided share in order, then a fixed tree.  coef[(b * L + l) * G + g] = (mean_grp(gamma dy), mean_grp(gamma dy xhat))
__global__ void __launch_bounds__(kGnCombineThreads) gnb_combine_kernel(const float *__restrict__ pdy, const float *__restrict__ pdyx,
                                                                        const float *__restrict__ gamma, int C, int G, GnLevels lv,
                                                                        int total_tiles, float2 *__restrict__ coef) {
    __shared__ float s1[kGnCombineThreads], s2[kGnCombineThreads];
    const int g = blockIdx.x, l = blockIdx.y, b = blockIdx.z, cg = C / G;
    int size = 0, tile0 = 0, ntiles = 0;  // lv.*[l] by selection, as in gn_combine_kernel
#pragma unroll
    for (int u = 0; u < kMaxLevels; ++u)
        if (u == l) size = lv.size[u], tile0 = lv.tile0[u], ntiles = lv.tile0[u + 1] - lv.tile0[u];
    const int64_t items = (int64_t)ntiles * cg;
    const float *pd = pdy + ((int64_t)b * total_tiles + tile0) * C, *px = pdyx + ((int64_t)b * total_tiles + tile0) * C;
    const float *ga = gamma + (int64_t)l * C;
    float a1 = 0.f, a2 = 0.f;
    for (int64_t k = threadIdx.x; k < items; k += kGnCombineThreads) {
        const int tl = (int)(k / cg), c = g * cg + (int)(k % cg);
        const float gc = __ldg(ga + c);
        a1 = fmaf(gc, __ldg(pd + (int64_t)tl * C + c), a1);
        a2 = fmaf(gc, __ldg(px + (int64_t)tl * C + c), a2);
    }
    s1[threadIdx.x] = a1, s2[threadIdx.x] = a2;
    __syncthreads();
    for (int s = kGnCombineThreads / 2; s > 0; s >>= 1) {
        if ((int)threadIdx.x < s) s1[threadIdx.x] += s1[threadIdx.x + s], s2[threadIdx.x] += s2[threadIdx.x + s];
        __syncthreads();
    }
    if (threadIdx.x == 0) {
        const float inv_n = 1.f / ((float)size * (float)cg);
        coef[((int64_t)b * lv.L + l) * G + g] = make_float2(s1[0] * inv_n, s2[0] * inv_n);
    }
}

constexpr int kGnParamLanes = 8;  // gnb_param_kernel: CTA (32 channels, kGnParamLanes lanes)

// (3) one CTA per (32 channels, level): dgamma[l, c] = sum of pdyx, dbeta[l, c] = sum of pdy over the level's (image, tile)
// partials; lane u of a channel sums the partials u, u + kGnParamLanes, ... in (image, tile) order, the lanes in order.  Either
// output may be NULL.
__global__ void __launch_bounds__(32 * kGnParamLanes) gnb_param_kernel(const float *__restrict__ pdy, const float *__restrict__ pdyx,
                                                                       int batch, int C, GnLevels lv, int total_tiles,
                                                                       float *__restrict__ dgamma, float *__restrict__ dbeta) {
    __shared__ float sg[kGnParamLanes][32], sb[kGnParamLanes][32];
    const int l = blockIdx.y, c = blockIdx.x * 32 + threadIdx.x, u = threadIdx.y;
    int tile0 = 0, ntiles = 0;
#pragma unroll
    for (int v = 0; v < kMaxLevels; ++v)
        if (v == l) tile0 = lv.tile0[v], ntiles = lv.tile0[v + 1] - lv.tile0[v];
    float ag = 0.f, ab = 0.f;
    if (c < C) {
        const int items = batch * ntiles;
        for (int k = u; k < items; k += kGnParamLanes) {
            const int64_t o = ((int64_t)(k / ntiles) * total_tiles + tile0 + k % ntiles) * C + c;
            ag += __ldg(pdyx + o), ab += __ldg(pdy + o);
        }
    }
    sg[u][threadIdx.x] = ag, sb[u][threadIdx.x] = ab;
    __syncthreads();
    if (u != 0 || c >= C) return;
    for (int v = 1; v < kGnParamLanes; ++v) ag += sg[v][threadIdx.x], ab += sb[v][threadIdx.x];
    if (dgamma) dgamma[(int64_t)l * C + c] = ag;
    if (dbeta) dbeta[(int64_t)l * C + c] = ab;
}

// (4) dx = rstd * (gamma dy - m1 - xhat m2), same tiles and threads as gn_apply_kernel; dx may alias x or dy (each element is
// read, then written, by the same thread)
__global__ void gnb_apply_kernel(const float *dy, const float *x, float *dx, int64_t pitch, int C, int G, GnLevels lv,
                                 const float *__restrict__ gamma, const float2 *__restrict__ stats, const float2 *__restrict__ coef) {
    const int C4 = C / 4, R = blockDim.x / C4;
    const int j = threadIdx.x % C4, r = threadIdx.x / C4, c = 4 * j, cg = C / G;
    const int tile = blockIdx.x, b = blockIdx.y;
    const int l = gn_level_of_tile(lv, tile);
    const int t0 = (tile - lv.tile0[l]) * kGnTile;
    const int rows = min(kGnTile, lv.size[l] - t0);
    const float4 ga = ldg_f4(gamma + (int64_t)l * C + c);
    const int64_t sidx = ((int64_t)b * lv.L + l) * G;
    const float2 s0 = stats[sidx + (c + 0) / cg], s1 = stats[sidx + (c + 1) / cg], s2 = stats[sidx + (c + 2) / cg],
                 s3 = stats[sidx + (c + 3) / cg];
    const float2 k0 = coef[sidx + (c + 0) / cg], k1 = coef[sidx + (c + 1) / cg], k2 = coef[sidx + (c + 2) / cg],
                 k3 = coef[sidx + (c + 3) / cg];
    const int64_t base = (int64_t)b * pitch + (int64_t)(lv.start[l] + t0) * C + c;
    for (int t = r; t < rows; t += R) {
        const int64_t o = base + (int64_t)t * C;
        const float4 g = *reinterpret_cast<const float4 *>(dy + o), v = *reinterpret_cast<const float4 *>(x + o);
        float4 d;
        d.x = s0.y * (fmaf(ga.x, g.x, -k0.x) - (v.x - s0.x) * s0.y * k0.y);
        d.y = s1.y * (fmaf(ga.y, g.y, -k1.x) - (v.y - s1.x) * s1.y * k1.y);
        d.z = s2.y * (fmaf(ga.z, g.z, -k2.x) - (v.z - s2.x) * s2.y * k2.y);
        d.w = s3.y * (fmaf(ga.w, g.w, -k3.x) - (v.w - s3.x) * s3.y * k3.y);
        *reinterpret_cast<float4 *>(dx + o) = d;
    }
}

struct LevelStarts {
    int start[kMaxLevels];
    int L;
};

// same operations as flatten_tokens(_vec)_kernel: pv = pos + level_embed; x = (feat + pv) * keep
__global__ void __launch_bounds__(256) token_lpos_keep_kernel(const float *__restrict__ feat, const float *pos,
                                                              const float *__restrict__ level_embeds, const float *__restrict__ keep,
                                                              LevelStarts ls, int nv, int C, int64_t total4, float *lpos,
                                                              float *__restrict__ x) {
    const int C4 = C / 4;
    for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < total4; i += (int64_t)gridDim.x * blockDim.x) {
        const int64_t row = i / C4;
        const int c = (int)(i - row * C4) * 4, t = (int)(row % nv);
        int l = 0;
#pragma unroll
        for (int u = 1; u < kMaxLevels; ++u)
            if (u < ls.L && t >= ls.start[u]) l = u;
        const float4 le = ldg_f4(level_embeds + (int64_t)l * C + c);
        const float4 p = *reinterpret_cast<const float4 *>(pos + row * C + c);
        const float4 f = ldg_f4(feat + row * C + c);
        const float k = __ldg(keep + row);
        const float4 pv = make_float4(p.x + le.x, p.y + le.y, p.z + le.z, p.w + le.w);
        *reinterpret_cast<float4 *>(lpos + row * C + c) = pv;
        *reinterpret_cast<float4 *>(x + row * C + c) =
            make_float4((f.x + pv.x) * k, (f.y + pv.y) * k, (f.z + pv.z) * k, (f.w + pv.w) * k);
    }
}

// levels of the host size array -> token starts and tile table; false when a size is not positive
static bool gn_levels(const int32_t *level_size_host, int num_levels, GnLevels &lv, int &nv) {
    lv = GnLevels{};
    lv.L = num_levels;
    int tiles = 0;
    nv = 0;
    for (int l = 0; l < num_levels; ++l) {
        if (level_size_host[l] <= 0) return false;
        lv.size[l] = level_size_host[l], lv.start[l] = nv, lv.tile0[l] = tiles;
        nv += level_size_host[l];
        tiles += (level_size_host[l] + kGnTile - 1) / kGnTile;
    }
    lv.tile0[num_levels] = tiles;
    return true;
}

static int gn_threads(int C) {
    const int C4 = C / 4;
    return C4 >= 256 ? C4 : C4 * (256 / C4);
}

}  // namespace sdetr

using namespace sdetr;

extern "C" int64_t sdetr_group_norm_tokens_workspace_floats(int batch, int channels, int num_groups, int num_levels,
                                                            const int32_t *level_size_host) {
    if (batch <= 0 || channels <= 0 || num_groups <= 0 || num_levels <= 0 || num_levels > kMaxLevels || !level_size_host) return 0;
    GnLevels lv;
    int nv;
    if (!gn_levels(level_size_host, num_levels, lv, nv)) return 0;
    return 2LL * batch * lv.tile0[num_levels] * channels + 2LL * batch * num_levels * num_groups;
}

extern "C" int sdetr_group_norm_tokens(const float *x, float *y, int64_t pitch, int batch, int channels, int num_levels,
                                       const int32_t *level_size_host, const float *gamma, const float *beta, int num_groups,
                                       float eps, float *workspace, int64_t workspace_floats, sdetr_stream_t stream) {
    SDETR_REQUIRE(x && y && level_size_host && gamma && beta && workspace, SDETR_ERR_INVALID_ARG, "group_norm_tokens: null pointer");
    SDETR_REQUIRE(batch >= 0 && batch <= 65535 && channels > 0 && num_groups > 0 && num_levels > 0, SDETR_ERR_INVALID_ARG,
                  "group_norm_tokens: bad sizes");
    SDETR_REQUIRE(num_levels <= kMaxLevels, SDETR_ERR_UNSUPPORTED, "group_norm_tokens: at most %d levels", kMaxLevels);
    SDETR_REQUIRE(channels % 4 == 0 && channels <= 4096 && channels % num_groups == 0, SDETR_ERR_UNSUPPORTED,
                  "group_norm_tokens: channels=%d must be a multiple of 4, at most 4096, and divisible by num_groups=%d", channels,
                  num_groups);
    SDETR_REQUIRE(eps >= 0.f, SDETR_ERR_INVALID_ARG, "group_norm_tokens: eps must not be negative");
    SDETR_REQUIRE(aligned16(x) && aligned16(y) && aligned16(gamma) && aligned16(beta) && pitch % 4 == 0, SDETR_ERR_INVALID_ARG,
                  "group_norm_tokens: x, y, gamma, beta and the image pitch must be 16-byte aligned");
    GnLevels lv;
    int nv;
    SDETR_REQUIRE(gn_levels(level_size_host, num_levels, lv, nv), SDETR_ERR_INVALID_ARG, "group_norm_tokens: empty level");
    SDETR_REQUIRE(pitch >= (int64_t)nv * channels, SDETR_ERR_INVALID_ARG, "group_norm_tokens: image pitch below Nv * C");
    if (batch == 0) return SDETR_OK;
    SDETR_REQUIRE(workspace_floats >= sdetr_group_norm_tokens_workspace_floats(batch, channels, num_groups, num_levels, level_size_host),
                  SDETR_ERR_WORKSPACE, "group_norm_tokens: workspace too small");
    const int tiles = lv.tile0[num_levels], threads = gn_threads(channels);
    float *pmean = workspace, *pm2 = workspace + (int64_t)batch * tiles * channels;
    float2 *stats = reinterpret_cast<float2 *>(pm2 + (int64_t)batch * tiles * channels);
    SDETR_REQUIRE((reinterpret_cast<uintptr_t>(stats) & 7) == 0, SDETR_ERR_INVALID_ARG, "group_norm_tokens: workspace misaligned");
    const size_t smem = 2 * sizeof(float) * (size_t)threads * 4;  // [R][C] mean and M2
    gn_partial_kernel<<<dim3(tiles, batch), threads, smem, (cudaStream_t)stream>>>(x, pitch, channels, lv, tiles, pmean, pm2);
    int rc = check_launch("group_norm_tokens (partials)");
    if (rc) return rc;
    gn_combine_kernel<<<dim3(num_groups, num_levels, batch), kGnCombineThreads, 0, (cudaStream_t)stream>>>(
        pmean, pm2, channels, num_groups, lv, tiles, eps, stats);
    rc = check_launch("group_norm_tokens (combine)");
    if (rc) return rc;
    gn_apply_kernel<<<dim3(tiles, batch), threads, 0, (cudaStream_t)stream>>>(x, y, pitch, channels, num_groups, lv, gamma, beta,
                                                                             stats);
    return check_launch("group_norm_tokens (apply)");
}

extern "C" int64_t sdetr_group_norm_tokens_backward_workspace_floats(int batch, int channels, int num_groups, int num_levels,
                                                                     const int32_t *level_size_host) {
    const int64_t fwd = sdetr_group_norm_tokens_workspace_floats(batch, channels, num_groups, num_levels, level_size_host);
    return fwd ? fwd + 2LL * batch * num_levels * num_groups : 0;  // + the (m1, m2) table
}

extern "C" int sdetr_group_norm_tokens_backward(const float *dy, const float *x, float *dx, int64_t pitch, int batch, int channels,
                                                int num_levels, const int32_t *level_size_host, const float *gamma, int num_groups,
                                                float eps, float *dgamma, float *dbeta, float *workspace, int64_t workspace_floats,
                                                sdetr_stream_t stream) {
    SDETR_REQUIRE(dy && x && dx && level_size_host && gamma && workspace, SDETR_ERR_INVALID_ARG,
                  "group_norm_tokens_backward: null pointer");
    SDETR_REQUIRE(batch >= 0 && batch <= 65535 && channels > 0 && num_groups > 0 && num_levels > 0, SDETR_ERR_INVALID_ARG,
                  "group_norm_tokens_backward: bad sizes");
    SDETR_REQUIRE(num_levels <= kMaxLevels, SDETR_ERR_UNSUPPORTED, "group_norm_tokens_backward: at most %d levels", kMaxLevels);
    SDETR_REQUIRE(channels % 4 == 0 && channels <= 4096 && channels % num_groups == 0, SDETR_ERR_UNSUPPORTED,
                  "group_norm_tokens_backward: channels=%d must be a multiple of 4, at most 4096, and divisible by num_groups=%d",
                  channels, num_groups);
    SDETR_REQUIRE(eps >= 0.f, SDETR_ERR_INVALID_ARG, "group_norm_tokens_backward: eps must not be negative");
    SDETR_REQUIRE(aligned16(dy) && aligned16(x) && aligned16(dx) && aligned16(gamma) && pitch % 4 == 0, SDETR_ERR_INVALID_ARG,
                  "group_norm_tokens_backward: dy, x, dx, gamma and the image pitch must be 16-byte aligned");
    GnLevels lv;
    int nv;
    SDETR_REQUIRE(gn_levels(level_size_host, num_levels, lv, nv), SDETR_ERR_INVALID_ARG, "group_norm_tokens_backward: empty level");
    SDETR_REQUIRE(pitch >= (int64_t)nv * channels, SDETR_ERR_INVALID_ARG, "group_norm_tokens_backward: image pitch below Nv * C");
    if (batch == 0) return SDETR_OK;
    SDETR_REQUIRE(workspace_floats >=
                      sdetr_group_norm_tokens_backward_workspace_floats(batch, channels, num_groups, num_levels, level_size_host),
                  SDETR_ERR_WORKSPACE, "group_norm_tokens_backward: workspace too small");
    const int tiles = lv.tile0[num_levels], threads = gn_threads(channels);
    // the forward's statistics, recomputed by its own kernels (the same bits); then the partials' space holds the backward's
    float *p0 = workspace, *p1 = workspace + (int64_t)batch * tiles * channels;
    float2 *stats = reinterpret_cast<float2 *>(p1 + (int64_t)batch * tiles * channels);
    float2 *coef = stats + (int64_t)batch * num_levels * num_groups;
    SDETR_REQUIRE((reinterpret_cast<uintptr_t>(stats) & 7) == 0, SDETR_ERR_INVALID_ARG,
                  "group_norm_tokens_backward: workspace misaligned");
    const size_t smem = 2 * sizeof(float) * (size_t)threads * 4;
    cudaStream_t s = (cudaStream_t)stream;
    gn_partial_kernel<<<dim3(tiles, batch), threads, smem, s>>>(x, pitch, channels, lv, tiles, p0, p1);
    int rc = check_launch("group_norm_tokens_backward (statistics partials)");
    if (rc) return rc;
    gn_combine_kernel<<<dim3(num_groups, num_levels, batch), kGnCombineThreads, 0, s>>>(p0, p1, channels, num_groups, lv, tiles, eps,
                                                                                       stats);
    if ((rc = check_launch("group_norm_tokens_backward (statistics combine)"))) return rc;
    gnb_partial_kernel<<<dim3(tiles, batch), threads, smem, s>>>(dy, x, pitch, channels, num_groups, lv, tiles, stats, p0, p1);
    if ((rc = check_launch("group_norm_tokens_backward (partials)"))) return rc;
    gnb_combine_kernel<<<dim3(num_groups, num_levels, batch), kGnCombineThreads, 0, s>>>(p0, p1, gamma, channels, num_groups, lv,
                                                                                        tiles, coef);
    if ((rc = check_launch("group_norm_tokens_backward (combine)"))) return rc;
    if (dgamma || dbeta) {
        gnb_param_kernel<<<dim3((channels + 31) / 32, num_levels), dim3(32, kGnParamLanes), 0, s>>>(p0, p1, batch, channels, lv, tiles,
                                                                                                   dgamma, dbeta);
        if ((rc = check_launch("group_norm_tokens_backward (dgamma, dbeta)"))) return rc;
    }
    gnb_apply_kernel<<<dim3(tiles, batch), threads, 0, s>>>(dy, x, dx, pitch, channels, num_groups, lv, gamma, stats, coef);
    return check_launch("group_norm_tokens_backward (dx)");
}

extern "C" int sdetr_token_lpos_keep(const float *feat, const float *pos, const float *level_embeds, const float *keep,
                                     const int32_t *level_size_host, int batch, int channels, int num_levels, float *lpos,
                                     float *x, sdetr_stream_t stream) {
    SDETR_REQUIRE(feat && pos && level_embeds && keep && level_size_host && lpos && x, SDETR_ERR_INVALID_ARG,
                  "token_lpos_keep: null pointer");
    SDETR_REQUIRE(batch >= 0 && channels > 0 && num_levels > 0, SDETR_ERR_INVALID_ARG, "token_lpos_keep: bad sizes");
    SDETR_REQUIRE(num_levels <= kMaxLevels && channels % 4 == 0, SDETR_ERR_UNSUPPORTED,
                  "token_lpos_keep: at most %d levels and channels a multiple of 4 (got %d)", kMaxLevels, channels);
    SDETR_REQUIRE(aligned16(feat) && aligned16(pos) && aligned16(level_embeds) && aligned16(lpos) && aligned16(x),
                  SDETR_ERR_INVALID_ARG, "token_lpos_keep: feat, pos, level_embeds, lpos and x must be 16-byte aligned");
    LevelStarts ls{};
    ls.L = num_levels;
    int nv = 0;
    for (int l = 0; l < num_levels; ++l) {
        SDETR_REQUIRE(level_size_host[l] > 0, SDETR_ERR_INVALID_ARG, "token_lpos_keep: level %d is empty", l);
        ls.start[l] = nv;
        nv += level_size_host[l];
    }
    const int64_t total4 = (int64_t)batch * nv * (channels / 4);
    if (total4 == 0) return SDETR_OK;
    const int64_t want = (total4 + 255) / 256, cap = 16LL * sm_count();
    token_lpos_keep_kernel<<<(unsigned)(want < cap ? want : cap), 256, 0, (cudaStream_t)stream>>>(
        feat, pos, level_embeds, keep, ls, nv, channels, total4, lpos, x);
    return check_launch("token_lpos_keep");
}
