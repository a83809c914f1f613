// Token movement and small fused elementwise kernels around the encoder layers (sm_90a).
//
// Reference semantics: models/bricks/salience_transformer.py:134-143 (score modulation), :366 (mc score),
// :390-391/:349-350 (residual + LayerNorm), :417-432 + :454-461 (reference points + four gathers),
// :474-485 (scatter back), :488-495 + position_encoding.py:81-95 (background embedding),
// models/bricks/ms_deform_attn.py:318-319 (zero the value rows of padded tokens).
//
// All kernels are HBM-streaming: one warp owns one token row and moves it with 128-bit loads/stores,
// several independent loads in flight per lane; index/mask lookups are warp-uniform.
#include "common.cuh"

namespace sdetr {

constexpr int kRowThreads = 256;  // 8 warps = 8 rows per CTA

struct LevelsDev {
    int L;
    int H[kMaxLevels], W[kMaxLevels];
    int64_t start[kMaxLevels];
};

__device__ __forceinline__ void load_levels(LevelsDev &lv, const int64_t *shapes, const int64_t *lsi, int L) {
    lv.L = L;
#pragma unroll
    for (int l = 0; l < kMaxLevels; ++l)
        if (l < L) {
            lv.H[l] = (int)__ldg(shapes + 2 * l), lv.W[l] = (int)__ldg(shapes + 2 * l + 1);
            lv.start[l] = __ldg(lsi + l);
        }
}
__device__ __forceinline__ void token_to_lyx(const LevelsDev &lv, int64_t t, int &l, int &y, int &x) {
    l = 0;
#pragma unroll
    for (int u = 1; u < kMaxLevels; ++u)
        if (u < lv.L && t >= lv.start[u]) l = u;
    int Wl = lv.W[0];
    int64_t st = lv.start[0];
#pragma unroll
    for (int u = 1; u < kMaxLevels; ++u)
        if (u == l) Wl = lv.W[u], st = lv.start[u];
    const int r = (int)(t - st);
    y = r / Wl, x = r - y * Wl;
}

// ---- gather (:454-461) ---------------------------------------------------------------------------------
__global__ void __launch_bounds__(kRowThreads) token_gather_kernel(
    const float *__restrict__ tokens, const float *__restrict__ pos, const float *__restrict__ fg,
    const float *__restrict__ vr, const int64_t *__restrict__ inds, int64_t inds_stride,
    const int64_t *__restrict__ shapes, const int64_t *__restrict__ lsi, int batch, int nv, int C, int L, int nq,
    float *__restrict__ query, float *__restrict__ query_pos, float *__restrict__ fg_q, float *__restrict__ ref_q,
    float *__restrict__ query_sum /* may be null */) {
    const int lane = threadIdx.x & 31;
    const int64_t row = (int64_t)blockIdx.x * (kRowThreads / 32) + (threadIdx.x >> 5);
    if (row >= (int64_t)batch * nq) return;
    const int b = (int)(row / nq), q = (int)(row - (int64_t)b * nq);
    const int64_t t = __ldg(inds + (int64_t)b * inds_stride + q);
    const float *src_t = tokens + ((int64_t)b * nv + t) * C;
    const float *src_p = pos + ((int64_t)b * nv + t) * C;
    float *dst_t = query + row * C, *dst_p = query_pos + row * C;
    for (int c = lane * 4; c < C; c += 256) {  // two rows x two 128-bit loads in flight per lane
        const bool two = c + 128 < C;
        const float4 a0 = ld_stream_f4(src_t + c), p0 = ld_stream_f4(src_p + c);
        float4 a1, p1;
        if (two) a1 = ld_stream_f4(src_t + c + 128), p1 = ld_stream_f4(src_p + c + 128);
        st_stream_f4(dst_t + c, a0), st_stream_f4(dst_p + c, p0);
        if (two) st_stream_f4(dst_t + c + 128, a1), st_stream_f4(dst_p + c + 128, p1);
        if (query_sum) {
            st_stream_f4(query_sum + row * C + c, make_float4(a0.x + p0.x, a0.y + p0.y, a0.z + p0.z, a0.w + p0.w));
            if (two) st_stream_f4(query_sum + row * C + c + 128, make_float4(a1.x + p1.x, a1.y + p1.y, a1.z + p1.z, a1.w + p1.w));
        }
    }
    if (lane == 0) fg_q[row] = __ldg(fg + (int64_t)b * nv + t);
    // reference points (:417-432): ((x+.5)/(vr_x*W), (y+.5)/(vr_y*H)) of the token's own level, times every
    // level's valid ratio -- same fp32 operations in the same order as the reference
    LevelsDev lv;
    load_levels(lv, shapes, lsi, L);
    int l, y, x;
    token_to_lyx(lv, t, l, y, x);
    int Hl = lv.H[0], Wl = lv.W[0];
#pragma unroll
    for (int u = 1; u < kMaxLevels; ++u)
        if (u == l) Hl = lv.H[u], Wl = lv.W[u];
    const float *v = vr + (int64_t)b * L * 2;
    const float rx = ((float)x + 0.5f) / (__ldg(v + 2 * l) * (float)Wl);
    const float ry = ((float)y + 0.5f) / (__ldg(v + 2 * l + 1) * (float)Hl);
    if (lane < L)
        *reinterpret_cast<float2 *>(ref_q + (row * L + lane) * 2) =
            make_float2(rx * __ldg(v + 2 * lane), ry * __ldg(v + 2 * lane + 1));
}

// ---- scatter back (:474-485) ----------------------------------------------------------------------------
__global__ void __launch_bounds__(kRowThreads) token_scatter_kernel(float *__restrict__ tokens,
                                                                    const float *__restrict__ query,
                                                                    const int64_t *__restrict__ inds,
                                                                    int64_t inds_stride,
                                                                    const int32_t *__restrict__ focus, int batch,
                                                                    int nv, int C, int nq) {
    const int lane = threadIdx.x & 31;
    const int64_t row = (int64_t)blockIdx.x * (kRowThreads / 32) + (threadIdx.x >> 5);
    if (row >= (int64_t)batch * nq) return;
    const int b = (int)(row / nq), q = (int)(row - (int64_t)b * nq);
    if (q >= __ldg(focus + b)) return;  // only the first focus_token_nums[b] rows are written back
    const int64_t t = __ldg(inds + (int64_t)b * inds_stride + q);
    const float *src = query + row * C;
    float *dst = tokens + ((int64_t)b * nv + t) * C;
    for (int c = lane * 4; c < C; c += 256) {
        const bool two = c + 128 < C;
        const float4 a0 = ld_stream_f4(src + c);
        float4 a1;
        if (two) a1 = ld_stream_f4(src + c + 128);
        st_stream_f4(dst + c, a0);
        if (two) st_stream_f4(dst + c + 128, a1);
    }
}

// ---- background embedding (:488-495) --------------------------------------------------------------------
__global__ void mark_flags_kernel(const int64_t *__restrict__ inds, int64_t inds_stride, int num, int batch, int nv,
                                  uint8_t *__restrict__ flags) {
    const int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= (int64_t)batch * num) return;
    const int b = (int)(i / num), q = (int)(i - (int64_t)b * num);
    flags[(int64_t)b * nv + __ldg(inds + (int64_t)b * inds_stride + q)] = 1;
}

__global__ void __launch_bounds__(kRowThreads) background_embed_kernel(
    float *__restrict__ tokens, const uint8_t *__restrict__ mask, const uint8_t *__restrict__ flags,
    const float *__restrict__ row_embed, const float *__restrict__ col_embed, const int64_t *__restrict__ shapes,
    const int64_t *__restrict__ lsi, int batch, int nv, int C, int L, int num_embeddings) {
    const int lane = threadIdx.x & 31;
    const int64_t row = (int64_t)blockIdx.x * (kRowThreads / 32) + (threadIdx.x >> 5);
    if (row >= (int64_t)batch * nv) return;
    if (__ldg(mask + row) || flags[row]) return;
    const int t = (int)(row % nv);
    LevelsDev lv;
    load_levels(lv, shapes, lsi, L);
    int l, y, x;
    token_to_lyx(lv, t, l, y, x);
    y = min(y, num_embeddings - 1), x = min(x, num_embeddings - 1);  // never read outside the tables (host validates)
    const int half = C / 2;
    float *dst = tokens + row * C;
    for (int c = lane * 4; c < C; c += 128) {
        const float *e = c < half ? col_embed + (int64_t)x * half + c : row_embed + (int64_t)y * half + (c - half);
        const float4 ev = ldg_f4(e);
        float4 v = *reinterpret_cast<float4 *>(dst + c);
        v.x += ev.x, v.y += ev.y, v.z += ev.z, v.w += ev.w;
        *reinterpret_cast<float4 *>(dst + c) = v;
    }
}

// ---- coarse-to-fine score modulation (:134-143) -----------------------------------------------------------
__global__ void __launch_bounds__(kRowThreads) score_modulate_kernel(const float *__restrict__ mem, int64_t mem_bs,
                                                                     const float *__restrict__ coarse, int64_t coarse_bs,
                                                                     const float *__restrict__ alpha, int alpha_index,
                                                                     int batch, int H, int W, int Hc, int Wc, int C,
                                                                     float *__restrict__ out) {
    const int lane = threadIdx.x & 31;
    const int64_t row = (int64_t)blockIdx.x * (kRowThreads / 32) + (threadIdx.x >> 5);
    const int HW = H * W;
    if (row >= (int64_t)batch * HW) return;
    const int b = (int)(row / HW), r = (int)(row - (int64_t)b * HW);
    const int y = r / W, x = r - y * W;
    // ATen upsample_bilinear2d, align_corners=True: src = dst * (in-1)/(out-1)
    const float sy = H > 1 ? (float)(Hc - 1) / (float)(H - 1) : 0.f;
    const float sx = W > 1 ? (float)(Wc - 1) / (float)(W - 1) : 0.f;
    const float fy = sy * (float)y, fx = sx * (float)x;
    const int y0 = (int)fy, x0 = (int)fx;
    const int y1 = y0 + (y0 < Hc - 1 ? 1 : 0), x1 = x0 + (x0 < Wc - 1 ? 1 : 0);
    const float ly = fy - (float)y0, lx = fx - (float)x0, hy = 1.f - ly, hx = 1.f - lx;
    const float *cs = coarse + (int64_t)b * coarse_bs;
    const float up = hy * (hx * __ldg(cs + y0 * Wc + x0) + lx * __ldg(cs + y0 * Wc + x1)) +
                     ly * (hx * __ldg(cs + y1 * Wc + x0) + lx * __ldg(cs + y1 * Wc + x1));
    const float a = __ldg(alpha + alpha_index);
    const float *src = mem + (int64_t)b * mem_bs + (int64_t)r * C;
    float *dst = out + row * C;
    for (int c = lane * 4; c < C; c += 128) {
        const float4 m = ld_stream_f4(src + c);
        float4 o;
        o.x = m.x + m.x * up * a, o.y = m.y + m.y * up * a, o.z = m.z + m.z * up * a, o.w = m.w + m.w * up * a;
        *reinterpret_cast<float4 *>(dst + c) = o;
    }
}

// ---- zero the value rows of padded tokens (ms_deform_attn.py:318-319) ------------------------------------
__global__ void __launch_bounds__(kRowThreads) zero_masked_rows_kernel(float *__restrict__ rows, int64_t row_stride,
                                                                       int row_floats,
                                                                       const uint8_t *__restrict__ mask,
                                                                       int64_t num_rows) {
    const int lane = threadIdx.x & 31;
    const int64_t row = (int64_t)blockIdx.x * (kRowThreads / 32) + (threadIdx.x >> 5);
    if (row >= num_rows || !__ldg(mask + row)) return;
    float *dst = rows + row * row_stride;
    for (int c = lane * 4; c < row_floats; c += 128) *reinterpret_cast<float4 *>(dst + c) = make_float4(0.f, 0.f, 0.f, 0.f);
}

// ---- mc_score = max_c(logits) * fg (:366) ---------------------------------------------------------------
__global__ void __launch_bounds__(kRowThreads) class_max_kernel(const float *__restrict__ logits, int64_t pitch,
                                                                const float *__restrict__ fg, int64_t rows, int nc,
                                                                float *__restrict__ out) {
    const int lane = threadIdx.x & 31;
    const int64_t row = (int64_t)blockIdx.x * (kRowThreads / 32) + (threadIdx.x >> 5);
    if (row >= rows) return;
    float m = -INFINITY;
    for (int c = lane; c < nc; c += 32) m = fmaxf(m, __ldg(logits + row * pitch + c));
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) m = fmaxf(m, __shfl_xor_sync(0xffffffffu, m, o));
    if (lane == 0) out[row] = m * __ldg(fg + row);
}

// ---- y = LayerNorm(x + r) (:390-391, :349-350) ------------------------------------------------------------
__global__ void __launch_bounds__(kRowThreads) add_layernorm_kernel(const float *x /* may alias y */,
                                                                    const float *r,
                                                                    const float *__restrict__ gamma,
                                                                    const float *__restrict__ beta, float eps,
                                                                    int64_t rows, int C, float *y) {
    const int lane = threadIdx.x & 31;
    const int64_t row = (int64_t)blockIdx.x * (kRowThreads / 32) + (threadIdx.x >> 5);
    if (row >= rows) return;
    float4 v[8];
    float s = 0.f;
#pragma unroll
    for (int i = 0; i < 8; ++i) {
        const int c = i * 128 + lane * 4;
        if (c < C) {
            const float4 a = *reinterpret_cast<const float4 *>(x + row * C + c);
            const float4 bb = r ? *reinterpret_cast<const float4 *>(r + row * C + c) : make_float4(0.f, 0.f, 0.f, 0.f);
            v[i] = make_float4(a.x + bb.x, a.y + bb.y, a.z + bb.z, a.w + bb.w);
            s += (v[i].x + v[i].y) + (v[i].z + v[i].w);
        }
    }
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) s += __shfl_xor_sync(0xffffffffu, s, o);
    const float mean = s / (float)C;
    float ss = 0.f;
#pragma unroll
    for (int i = 0; i < 8; ++i) {
        const int c = i * 128 + lane * 4;
        if (c < C) {
            const float dx = v[i].x - mean, dy = v[i].y - mean, dz = v[i].z - mean, dw = v[i].w - mean;
            ss += (dx * dx + dy * dy) + (dz * dz + dw * dw);
        }
    }
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) ss += __shfl_xor_sync(0xffffffffu, ss, o);
    const float rstd = rsqrtf(ss / (float)C + eps);
#pragma unroll
    for (int i = 0; i < 8; ++i) {
        const int c = i * 128 + lane * 4;
        if (c < C) {
            const float4 g = ldg_f4(gamma + c), bt = ldg_f4(beta + c);
            float4 o;
            o.x = (v[i].x - mean) * rstd * g.x + bt.x, o.y = (v[i].y - mean) * rstd * g.y + bt.y;
            o.z = (v[i].z - mean) * rstd * g.z + bt.z, o.w = (v[i].w - mean) * rstd * g.w + bt.w;
            *reinterpret_cast<float4 *>(y + row * C + c) = o;
        }
    }
}

static inline unsigned row_blocks(int64_t rows) { return (unsigned)((rows + (kRowThreads / 32) - 1) / (kRowThreads / 32)); }

}  // namespace sdetr

using namespace sdetr;

extern "C" int sdetr_token_gather(const float *tokens, const float *pos, const float *fg, const float *valid_ratios,
                                  const int64_t *inds, int64_t inds_stride, const int64_t *spatial_shapes,
                                  const int64_t *level_start_index, int batch, int num_value, int channels,
                                  int num_levels, int num_query, float *query, float *query_pos, float *fg_q,
                                  float *ref_q, float *query_sum, sdetr_stream_t stream) {
    SDETR_REQUIRE(tokens && pos && fg && valid_ratios && inds && spatial_shapes && level_start_index && query &&
                      query_pos && fg_q && ref_q,
                  SDETR_ERR_INVALID_ARG, "token_gather: null pointer");
    SDETR_REQUIRE(batch > 0 && num_value > 0 && num_query >= 0 && num_levels > 0 && num_levels <= kMaxLevels,
                  SDETR_ERR_INVALID_ARG, "token_gather: bad sizes");
    SDETR_REQUIRE(channels % 4 == 0 && aligned16(tokens) && aligned16(pos) && aligned16(query) && aligned16(query_pos),
                  SDETR_ERR_INVALID_ARG, "token_gather: rows must be 16-byte aligned, channels %% 4 == 0");
    if (num_query == 0) return SDETR_OK;
    token_gather_kernel<<<row_blocks((int64_t)batch * num_query), kRowThreads, 0, (cudaStream_t)stream>>>(
        tokens, pos, fg, valid_ratios, inds, inds_stride, spatial_shapes, level_start_index, batch, num_value, channels,
        num_levels, num_query, query, query_pos, fg_q, ref_q, query_sum);
    return check_launch("token_gather");
}

extern "C" int sdetr_token_scatter(float *tokens, const float *query, const int64_t *inds, int64_t inds_stride,
                                   const int32_t *focus_token_nums, int batch, int num_value, int channels,
                                   int num_query, sdetr_stream_t stream) {
    SDETR_REQUIRE(tokens && query && inds && focus_token_nums, SDETR_ERR_INVALID_ARG, "token_scatter: null pointer");
    SDETR_REQUIRE(batch > 0 && num_value > 0 && num_query >= 0, SDETR_ERR_INVALID_ARG, "token_scatter: bad sizes");
    SDETR_REQUIRE(channels % 4 == 0 && aligned16(tokens) && aligned16(query), SDETR_ERR_INVALID_ARG,
                  "token_scatter: rows must be 16-byte aligned, channels %% 4 == 0");
    if (num_query == 0) return SDETR_OK;
    token_scatter_kernel<<<row_blocks((int64_t)batch * num_query), kRowThreads, 0, (cudaStream_t)stream>>>(
        tokens, query, inds, inds_stride, focus_token_nums, batch, num_value, channels, num_query);
    return check_launch("token_scatter");
}

extern "C" int sdetr_background_embed(float *tokens, const uint8_t *mask, const int64_t *last_inds,
                                      int64_t inds_stride, int num_last, const float *row_embed,
                                      const float *col_embed, int num_embeddings, const int64_t *spatial_shapes,
                                      const int64_t *spatial_shapes_host, const int64_t *level_start_index, int batch,
                                      int num_value, int channels, int num_levels, uint8_t *flags,
                                      sdetr_stream_t stream) {
    SDETR_REQUIRE(tokens && mask && last_inds && row_embed && col_embed && spatial_shapes && level_start_index && flags,
                  SDETR_ERR_INVALID_ARG, "background_embed: null pointer");
    SDETR_REQUIRE(batch > 0 && num_value > 0 && num_last >= 0 && num_levels > 0 && num_levels <= kMaxLevels &&
                      num_embeddings > 0,
                  SDETR_ERR_INVALID_ARG, "background_embed: bad sizes");
    if (spatial_shapes_host) {  // the reference's nn.Embedding lookup fails for an index >= num_embeddings
        for (int l = 0; l < num_levels; ++l)
            SDETR_REQUIRE(spatial_shapes_host[2 * l] <= num_embeddings && spatial_shapes_host[2 * l + 1] <= num_embeddings,
                          SDETR_ERR_INVALID_ARG,
                          "background_embed: level %d is %lld x %lld but the embedding tables hold %d rows/columns "
                          "(max_num_embedding)",
                          l, (long long)spatial_shapes_host[2 * l], (long long)spatial_shapes_host[2 * l + 1], num_embeddings);
    }
    SDETR_REQUIRE(channels % 8 == 0 && aligned16(tokens) && aligned16(row_embed) && aligned16(col_embed),
                  SDETR_ERR_INVALID_ARG, "background_embed: channels %% 8 == 0 and 16-byte alignment required");
    cudaStream_t s = (cudaStream_t)stream;
    cudaError_t e = cudaMemsetAsync(flags, 0, (size_t)batch * num_value, s);
    SDETR_REQUIRE(e == cudaSuccess, SDETR_ERR_CUDA, "background_embed: memset: %s", cudaGetErrorString(e));
    if (num_last > 0) {
        const int64_t n = (int64_t)batch * num_last;
        mark_flags_kernel<<<(unsigned)((n + 255) / 256), 256, 0, s>>>(last_inds, inds_stride, num_last, batch, num_value,
                                                                      flags);
        int rc = check_launch("background_embed/mark");
        if (rc) return rc;
    }
    background_embed_kernel<<<row_blocks((int64_t)batch * num_value), kRowThreads, 0, s>>>(
        tokens, mask, flags, row_embed, col_embed, spatial_shapes, level_start_index, batch, num_value, channels,
        num_levels, num_embeddings);
    return check_launch("background_embed");
}

extern "C" int sdetr_score_modulate(const float *mem, int64_t mem_batch_stride, const float *coarse_score,
                                    int64_t coarse_batch_stride, const float *alpha, int alpha_index, int batch,
                                    int H, int W, int Hc, int Wc, int channels, float *out, sdetr_stream_t stream) {
    SDETR_REQUIRE(mem && coarse_score && alpha && out, SDETR_ERR_INVALID_ARG, "score_modulate: null pointer");
    SDETR_REQUIRE(batch > 0 && H > 0 && W > 0 && Hc > 0 && Wc > 0 && alpha_index >= 0, SDETR_ERR_INVALID_ARG,
                  "score_modulate: bad sizes");
    SDETR_REQUIRE(channels % 4 == 0 && aligned16(mem) && aligned16(out) && mem_batch_stride % 4 == 0,
                  SDETR_ERR_INVALID_ARG, "score_modulate: 16-byte alignment required");
    score_modulate_kernel<<<row_blocks((int64_t)batch * H * W), kRowThreads, 0, (cudaStream_t)stream>>>(
        mem, mem_batch_stride, coarse_score, coarse_batch_stride, alpha, alpha_index, batch, H, W, Hc, Wc, channels, out);
    return check_launch("score_modulate");
}

extern "C" int sdetr_zero_masked_rows(float *rows, int64_t row_stride, int row_floats, const uint8_t *mask,
                                      int64_t num_rows, sdetr_stream_t stream) {
    SDETR_REQUIRE(rows && mask, SDETR_ERR_INVALID_ARG, "zero_masked_rows: null pointer");
    SDETR_REQUIRE(num_rows >= 0 && row_floats > 0 && row_floats % 4 == 0 && row_stride % 4 == 0 && aligned16(rows),
                  SDETR_ERR_INVALID_ARG, "zero_masked_rows: bad sizes / alignment");
    if (num_rows == 0) return SDETR_OK;
    zero_masked_rows_kernel<<<row_blocks(num_rows), kRowThreads, 0, (cudaStream_t)stream>>>(rows, row_stride, row_floats,
                                                                                           mask, num_rows);
    return check_launch("zero_masked_rows");
}

extern "C" int sdetr_class_max_times_fg(const float *logits, int64_t row_pitch, const float *fg, int64_t rows,
                                        int num_classes, float *out, sdetr_stream_t stream) {
    SDETR_REQUIRE(logits && fg && out, SDETR_ERR_INVALID_ARG, "class_max_times_fg: null pointer");
    SDETR_REQUIRE(rows >= 0 && num_classes > 0 && row_pitch >= num_classes, SDETR_ERR_INVALID_ARG,
                  "class_max_times_fg: bad sizes");
    if (rows == 0) return SDETR_OK;
    class_max_kernel<<<row_blocks(rows), kRowThreads, 0, (cudaStream_t)stream>>>(logits, row_pitch, fg, rows, num_classes, out);
    return check_launch("class_max_times_fg");
}

extern "C" int sdetr_add_layernorm(const float *x, const float *r, const float *gamma, const float *beta, float eps,
                                   int64_t rows, int channels, float *y, sdetr_stream_t stream) {
    SDETR_REQUIRE(x && gamma && beta && y, SDETR_ERR_INVALID_ARG, "add_layernorm: null pointer");
    SDETR_REQUIRE(rows >= 0 && channels > 0 && channels <= 1024 && channels % 4 == 0, SDETR_ERR_UNSUPPORTED,
                  "add_layernorm: channels %d must be a multiple of 4 and <= 1024", channels);
    SDETR_REQUIRE(aligned16(x) && aligned16(y) && (!r || aligned16(r)) && aligned16(gamma) && aligned16(beta),
                  SDETR_ERR_INVALID_ARG, "add_layernorm: 16-byte alignment required");
    if (rows == 0) return SDETR_OK;
    add_layernorm_kernel<<<row_blocks(rows), kRowThreads, 0, (cudaStream_t)stream>>>(x, r, gamma, beta, eps, rows,
                                                                                     channels, y);
    return check_launch("add_layernorm");
}

// ---- 3xTF32 operand split --------------------------------------------------------------------------------
// The dense projections run on the tensor cores with fp32-class accuracy: x = hi + lo with hi = tf32(x),
// lo = tf32(x - hi); A' = [A_hi | A_hi | A_lo], B' = [B_hi | B_lo | B_hi] so that one TF32 GEMM over K' = 3K
// computes A_hi.B_hi + A_hi.B_lo + A_lo.B_hi with fp32 accumulation (dropped terms are O(2^-22)).  Every
// operand value is exactly representable in TF32, so the tensor-core products are exact.
namespace sdetr {
__device__ __forceinline__ float tf32_round(float x) {
    uint32_t u;
    asm("cvt.rna.tf32.f32 %0, %1;" : "=r"(u) : "f"(x));
    return __uint_as_float(u);
}
// out layout: (rows, K/chunk, 3, chunk): every K-chunk carries its own [hi|hi|lo] (or [hi|lo|hi]) triple, so a
// long reduction can be issued as several GEMMs accumulated in fp32 by the GEMM epilogue (beta = 1) -- the tensor
// core's own accumulator truncates, and its error grows linearly with the reduction length.
__global__ void __launch_bounds__(256) split_tf32_kernel(const float *__restrict__ x, int64_t x_stride, int64_t rows, int K,
                                                        int chunk, int layout_b, int relu, float *__restrict__ out) {
    const int64_t vec = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;  // one float4 of one row
    const int kv = K / 4;
    if (vec >= rows * kv) return;
    const int64_t r = vec / kv;
    const int c = (int)(vec - r * kv) * 4;
    float4 v = ld_stream_f4(x + r * x_stride + c);
    if (relu == 1) {
        v.x = fmaxf(v.x, 0.f), v.y = fmaxf(v.y, 0.f), v.z = fmaxf(v.z, 0.f), v.w = fmaxf(v.w, 0.f);
    } else if (relu == 2) {  // exact (erf) GELU
        v.x = 0.5f * v.x * (1.f + erff(v.x * 0.70710678118654752f)), v.y = 0.5f * v.y * (1.f + erff(v.y * 0.70710678118654752f));
        v.z = 0.5f * v.z * (1.f + erff(v.z * 0.70710678118654752f)), v.w = 0.5f * v.w * (1.f + erff(v.w * 0.70710678118654752f));
    }
    float4 hi, lo;
    hi.x = tf32_round(v.x), hi.y = tf32_round(v.y), hi.z = tf32_round(v.z), hi.w = tf32_round(v.w);
    lo.x = tf32_round(v.x - hi.x), lo.y = tf32_round(v.y - hi.y), lo.z = tf32_round(v.z - hi.z), lo.w = tf32_round(v.w - hi.w);
    const int ck = c / chunk, cc = c - ck * chunk;
    float *o = out + r * 3 * (int64_t)K + (int64_t)ck * 3 * chunk + cc;
    *reinterpret_cast<float4 *>(o) = hi;
    *reinterpret_cast<float4 *>(o + chunk) = layout_b ? lo : hi;
    *reinterpret_cast<float4 *>(o + 2 * chunk) = layout_b ? hi : lo;
}
}  // namespace sdetr

extern "C" int sdetr_split_tf32(const float *x, int64_t x_row_stride, int64_t rows, int K, int chunk, int layout_b,
                                int relu, float *out, sdetr_stream_t stream) {
    SDETR_REQUIRE(x && out, SDETR_ERR_INVALID_ARG, "split_tf32: null pointer");
    SDETR_REQUIRE(chunk > 0 && chunk % 4 == 0 && K % chunk == 0, SDETR_ERR_INVALID_ARG,
                  "split_tf32: chunk %d must divide K %d and be a multiple of 4", chunk, K);
    SDETR_REQUIRE(rows >= 0 && K > 0 && K % 4 == 0 && x_row_stride % 4 == 0 && aligned16(x) && aligned16(out),
                  SDETR_ERR_INVALID_ARG, "split_tf32: K %% 4 == 0 and 16-byte alignment required");
    if (rows == 0) return SDETR_OK;
    const int64_t vecs = rows * (K / 4);
    split_tf32_kernel<<<(unsigned)((vecs + 255) / 256), 256, 0, (cudaStream_t)stream>>>(x, x_row_stride, rows, K, chunk,
                                                                                       layout_b, relu, out);
    return check_launch("split_tf32");
}

// ---- MaskPredictor middle (salience_transformer.py:40-45): z = GELU(z); z[:, :, half:] = mean over the image's tokens ----
// Two launches: (1) GELU in place on the local half + per-CTA partial column sums of GELU(global half), (2) every CTA
// adds the partials in a fixed order (bit-reproducible, no atomics) and writes the mean over its rows' global half.
namespace sdetr {
constexpr int kMeanThreads = 256;
__device__ __forceinline__ float gelu_exact(float x) { return 0.5f * x * (1.f + erff(x * 0.70710678118654752f)); }

__global__ void __launch_bounds__(kMeanThreads) gelu_colsum_kernel(float *__restrict__ z, int n, int C, int half, int chunks,
                                                                   float *__restrict__ partial /* (b, chunks, C - half) */) {
    __shared__ float4 red[kMeanThreads];
    const int b = blockIdx.y, chunk = blockIdx.x;
    const int vec = C / 4, lanes = kMeanThreads / vec;          // threads per row, rows in flight
    const int cv = threadIdx.x % vec, rl = threadIdx.x / vec;
    const int rows_per = (n + chunks - 1) / chunks, r0 = chunk * rows_per, r1 = min(n, r0 + rows_per);
    const bool global_half = cv * 4 >= half;
    float4 acc = make_float4(0.f, 0.f, 0.f, 0.f);
    if (rl < lanes) {
        float *base = z + (int64_t)b * n * C + cv * 4;
        int r = r0 + rl;
        for (; r + 3 * lanes < r1; r += 4 * lanes) {  // four independent rows per iteration: loads in flight together
            float4 x[4];
#pragma unroll
            for (int u = 0; u < 4; ++u) x[u] = *reinterpret_cast<const float4 *>(base + (int64_t)(r + u * lanes) * C);
#pragma unroll
            for (int u = 0; u < 4; ++u) {
                x[u].x = gelu_exact(x[u].x), x[u].y = gelu_exact(x[u].y), x[u].z = gelu_exact(x[u].z), x[u].w = gelu_exact(x[u].w);
                if (global_half) acc.x += x[u].x, acc.y += x[u].y, acc.z += x[u].z, acc.w += x[u].w;
                else *reinterpret_cast<float4 *>(base + (int64_t)(r + u * lanes) * C) = x[u];
            }
        }
        for (; r < r1; r += lanes) {
            float4 x = *reinterpret_cast<const float4 *>(base + (int64_t)r * C);
            x.x = gelu_exact(x.x), x.y = gelu_exact(x.y), x.z = gelu_exact(x.z), x.w = gelu_exact(x.w);
            if (global_half) acc.x += x.x, acc.y += x.y, acc.z += x.z, acc.w += x.w;
            else *reinterpret_cast<float4 *>(base + (int64_t)r * C) = x;
        }
    }
    red[threadIdx.x] = acc;
    __syncthreads();
    if (rl == 0 && global_half) {
        float4 t = red[cv];
        for (int l = 1; l < lanes; ++l) {
            const float4 y = red[l * vec + cv];
            t.x += y.x, t.y += y.y, t.z += y.z, t.w += y.w;
        }
        *reinterpret_cast<float4 *>(partial + ((int64_t)b * chunks + chunk) * (C - half) + (cv * 4 - half)) = t;
    }
}

// chunks_in partial sums per image (fixed order) -> mean -> broadcast over this CTA's rows
__global__ void __launch_bounds__(kMeanThreads) colmean_broadcast_kernel(float *__restrict__ z, int n, int C, int half,
                                                                         int chunks_in, int chunks,
                                                                         const float *__restrict__ partial) {
    __shared__ __align__(16) float mean[1024];
    __shared__ __align__(16) float part[kMeanThreads / 32][1024];
    const int b = blockIdx.y, chunk = blockIdx.x, g = C - half;
    // every warp adds a contiguous slice of the partial rows (128-bit loads, lane <-> 4 columns), then the warps' sums
    // are added in warp order: a fixed order, so the mean is bit-reproducible
    {
        const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31, warps = kMeanThreads / 32;
        const int per = (chunks_in + warps - 1) / warps, k0 = warp * per, k1 = min(chunks_in, k0 + per);
        for (int c = lane * 4; c < g; c += 128) {
            const float *p = partial + (int64_t)b * chunks_in * g + c;
            float4 t0 = make_float4(0.f, 0.f, 0.f, 0.f), t1 = t0;
            int k = k0;
            for (; k + 1 < k1; k += 2) {
                const float4 x = ldg_f4(p + (int64_t)k * g), y = ldg_f4(p + (int64_t)(k + 1) * g);
                t0.x += x.x, t0.y += x.y, t0.z += x.z, t0.w += x.w;
                t1.x += y.x, t1.y += y.y, t1.z += y.z, t1.w += y.w;
            }
            if (k < k1) {
                const float4 x = ldg_f4(p + (int64_t)k * g);
                t0.x += x.x, t0.y += x.y, t0.z += x.z, t0.w += x.w;
            }
            *reinterpret_cast<float4 *>(&part[warp][c]) = make_float4(t0.x + t1.x, t0.y + t1.y, t0.z + t1.z, t0.w + t1.w);
        }
        __syncthreads();
        for (int c = threadIdx.x; c < g; c += kMeanThreads) {
            float t = part[0][c];
            for (int w = 1; w < warps; ++w) t += part[w][c];
            mean[c] = t / (float)n;
        }
    }
    __syncthreads();
    const int gv = g / 4, lanes = kMeanThreads / gv;
    const int cv = threadIdx.x % gv, rl = threadIdx.x / gv;
    const int rows_per = (n + chunks - 1) / chunks, r0 = chunk * rows_per, r1 = min(n, r0 + rows_per);
    if (rl >= lanes) return;
    const float4 m = *reinterpret_cast<const float4 *>(mean + cv * 4);
    for (int r = r0 + rl; r < r1; r += lanes)
        *reinterpret_cast<float4 *>(z + ((int64_t)b * n + r) * C + half + cv * 4) = m;
}
}  // namespace sdetr

extern "C" size_t sdetr_gelu_colmean_workspace(int batch, int num_rows, int channels, int half) {
    (void)num_rows;
    return (size_t)(batch + 1184) * (size_t)(channels - half) * sizeof(float);  // <= 1184 / batch (+1) partial rows per image
}

extern "C" int sdetr_gelu_colmean(float *z, int batch, int num_rows, int channels, int half, void *workspace,
                                  size_t workspace_bytes, sdetr_stream_t stream) {
    SDETR_REQUIRE(z && workspace, SDETR_ERR_INVALID_ARG, "gelu_colmean: null pointer");
    SDETR_REQUIRE(batch > 0 && num_rows > 0 && channels > 0 && channels % 4 == 0 && channels <= 1024 && half >= 0 &&
                      half < channels && half % 4 == 0 && (channels - half) % 4 == 0 && aligned16(z) && aligned16(workspace),
                  SDETR_ERR_INVALID_ARG, "gelu_colmean: bad sizes / alignment");
    SDETR_REQUIRE(channels / 4 <= kMeanThreads, SDETR_ERR_UNSUPPORTED, "gelu_colmean: channels %d > %d", channels, 4 * kMeanThreads);
    SDETR_REQUIRE(workspace_bytes >= sdetr_gelu_colmean_workspace(batch, num_rows, channels, half), SDETR_ERR_WORKSPACE,
                  "gelu_colmean: workspace too small");
    // pass 1 is a read-modify-write stream: up to 8 resident CTAs per SM so enough loads are in flight;
    // pass 2 only stores (and every CTA re-adds the partials), one wave is enough
    int chunks1 = (num_rows + 31) / 32, chunks2 = (num_rows + 63) / 64;
    const int sms = sm_count(), cap1 = 4 * sms / batch > 0 ? 4 * sms / batch : 1, cap2 = sms / batch > 0 ? sms / batch : 1;
    if (chunks1 > cap1) chunks1 = cap1;
    if (chunks2 > cap2) chunks2 = cap2;
    cudaStream_t s = (cudaStream_t)stream;
    gelu_colsum_kernel<<<dim3(chunks1, batch), kMeanThreads, 0, s>>>(z, num_rows, channels, half, chunks1, (float *)workspace);
    int rc = check_launch("gelu_colmean/colsum");
    if (rc) return rc;
    colmean_broadcast_kernel<<<dim3(chunks2, batch), kMeanThreads, 0, s>>>(z, num_rows, channels, half, chunks1, chunks2,
                                                                           (const float *)workspace);
    return check_launch("gelu_colmean/broadcast");
}

// ---- generic row gather / scatter by index (the 300-token pre-attention, salience_transformer.py:368-379) ----
namespace sdetr {
__global__ void __launch_bounds__(kRowThreads) rows_gather_kernel(const float *__restrict__ src, const int64_t *__restrict__ idx,
                                                                  int batch, int n, int k, int C, float *__restrict__ out) {
    const int lane = threadIdx.x & 31;
    const int64_t row = (int64_t)blockIdx.x * (kRowThreads / 32) + (threadIdx.x >> 5);
    if (row >= (int64_t)batch * k) return;
    const int b = (int)(row / k);
    const float *s = src + ((int64_t)b * n + __ldg(idx + row)) * C;
    for (int c = lane * 4; c < C; c += 128) st_stream_f4(out + row * C + c, ld_stream_f4(s + c));
}
__global__ void __launch_bounds__(kRowThreads) rows_scatter_kernel(float *__restrict__ dst, const int64_t *__restrict__ idx,
                                                                   int batch, int n, int k, int C, const float *__restrict__ src) {
    const int lane = threadIdx.x & 31;
    const int64_t row = (int64_t)blockIdx.x * (kRowThreads / 32) + (threadIdx.x >> 5);
    if (row >= (int64_t)batch * k) return;
    const int b = (int)(row / k);
    float *d = dst + ((int64_t)b * n + __ldg(idx + row)) * C;
    for (int c = lane * 4; c < C; c += 128) st_stream_f4(d + c, ld_stream_f4(src + row * C + c));
}
}  // namespace sdetr

extern "C" int sdetr_rows_gather(const float *src, const int64_t *index, int batch, int num_rows, int k, int channels,
                                 float *out, sdetr_stream_t stream) {
    SDETR_REQUIRE(src && index && out, SDETR_ERR_INVALID_ARG, "rows_gather: null pointer");
    SDETR_REQUIRE(batch > 0 && num_rows > 0 && k >= 0 && channels % 4 == 0 && aligned16(src) && aligned16(out),
                  SDETR_ERR_INVALID_ARG, "rows_gather: bad sizes / alignment");
    if (k == 0) return SDETR_OK;
    rows_gather_kernel<<<row_blocks((int64_t)batch * k), kRowThreads, 0, (cudaStream_t)stream>>>(src, index, batch, num_rows, k,
                                                                                                channels, out);
    return check_launch("rows_gather");
}

extern "C" int sdetr_rows_scatter(float *dst, const int64_t *index, int batch, int num_rows, int k, int channels,
                                  const float *src, sdetr_stream_t stream) {
    SDETR_REQUIRE(dst && index && src, SDETR_ERR_INVALID_ARG, "rows_scatter: null pointer");
    SDETR_REQUIRE(batch > 0 && num_rows > 0 && k >= 0 && channels % 4 == 0 && aligned16(src) && aligned16(dst),
                  SDETR_ERR_INVALID_ARG, "rows_scatter: bad sizes / alignment");
    if (k == 0) return SDETR_OK;
    rows_scatter_kernel<<<row_blocks((int64_t)batch * k), kRowThreads, 0, (cudaStream_t)stream>>>(dst, index, batch, num_rows, k,
                                                                                                 channels, src);
    return check_launch("rows_scatter");
}

// ---- front end: (b,C,H_l,W_l) feature / position maps -> token layout (SURVEY.md 8(f)-2) ------------------------
// One pass replaces flatten_multi_level x2, `pos + level_embed`, `feat + lpos` and the keep-mask multiply
// (models/bricks/base_transformer.py:21-32,104; salience_transformer.py:107-113): 32x32 (channel x token) tiles are
// transposed through shared memory so both the NCHW reads and the token-major writes are coalesced.
namespace sdetr {
struct FlattenArgs {
    const float *feat[kMaxLevels], *pos[kMaxLevels];
    int size[kMaxLevels], start[kMaxLevels], tile0[kMaxLevels + 1];  // tokens per level, token offset, first tile
    int level[kMaxLevels];  // the entry's level index in the caller's numbering (row of level_embeds)
    int L;
};
static std::atomic<int> g_flatten_vec{1};
__global__ void __launch_bounds__(256) flatten_tokens_kernel(FlattenArgs a, const float *__restrict__ level_embeds,
                                                             const float *__restrict__ keep, int nv, int C,
                                                             float *__restrict__ feat_tok, float *__restrict__ lpos_tok,
                                                             float *__restrict__ x_tok, const float *__restrict__ pos_tok) {
    // pos_tok != nullptr: the position embedding is already in token layout (b,Nv,C) (sdetr_sine_pos_tokens) -- only the
    // feature maps are transposed here
    __shared__ float sf[32][33], sp[32][33];
    int l = 0;
#pragma unroll
    for (int u = 1; u < kMaxLevels; ++u)
        if (u < a.L && (int)blockIdx.x >= a.tile0[u]) l = u;
    const int t0 = ((int)blockIdx.x - a.tile0[l]) * 32, c0 = blockIdx.y * 32, b = blockIdx.z;
    const int hw = a.size[l];
    const int tx = threadIdx.x & 31, ty = threadIdx.x >> 5;  // 32 x 8
    const float *f = a.feat[l] + ((int64_t)b * C + c0) * hw, *p = pos_tok ? nullptr : a.pos[l] + ((int64_t)b * C + c0) * hw;
#pragma unroll
    for (int i = 0; i < 4; ++i) {
        const int c = ty + 8 * i, t = t0 + tx;
        const bool ok = t < hw && c0 + c < C;
        sf[c][tx] = ok ? __ldg(f + (int64_t)c * hw + t) : 0.f;
        if (!pos_tok) sp[c][tx] = ok ? __ldg(p + (int64_t)c * hw + t) + __ldg(level_embeds + a.level[l] * C + c0 + c) : 0.f;
    }
    __syncthreads();
#pragma unroll
    for (int i = 0; i < 4; ++i) {
        const int t = t0 + ty + 8 * i, c = c0 + tx;
        if (t < hw && c < C) {
            const int64_t row = (int64_t)b * nv + a.start[l] + t;
            const float fv = sf[tx][ty + 8 * i];
            const float pv = pos_tok ? __ldg(pos_tok + row * C + c) + __ldg(level_embeds + a.level[l] * C + c) : sp[tx][ty + 8 * i];
            feat_tok[row * C + c] = fv;
            lpos_tok[row * C + c] = pv;
            x_tok[row * C + c] = (fv + pv) * __ldg(keep + row);
        }
    }
}

// Vectorised variant for levels whose token count is a multiple of 4 (16-byte aligned channel rows): each thread loads a
// 4 channel x 4 token block as four float4 (tokens contiguous in NCHW), transposes it in registers and stores, per token, a float4
// of 4 channels.  A warp = 4 token groups x 8 channel groups: reads are 64-byte runs of a channel row, writes full 128-byte lines
// of a token row; no shared memory, 1/4 of the memory instructions of the tile kernel above (3.2 -> ~5 TB/s on 228 MB at config 2).
// Block = 8 warps = the same 16 tokens x 256 channels (grid.y covers C in steps of 256).
__global__ void __launch_bounds__(256) flatten_tokens_vec_kernel(FlattenArgs a, const float *__restrict__ level_embeds,
                                                                 const float *__restrict__ keep, int nv, int C,
                                                                 float *__restrict__ feat_tok, float *__restrict__ lpos_tok,
                                                                 float *__restrict__ x_tok, const float *__restrict__ pos_tok) {
    int l = 0;
#pragma unroll
    for (int u = 1; u < kMaxLevels; ++u)
        if (u < a.L && (int)blockIdx.x >= a.tile0[u]) l = u;
    const int hw = a.size[l], b = blockIdx.z;
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    const int t = ((int)blockIdx.x - a.tile0[l]) * 16 + (lane >> 3) * 4;          // first of this thread's 4 tokens
    const int c = blockIdx.y * 256 + warp * 32 + (lane & 7) * 4;                 // first of its 4 channels
    if (t >= hw || c >= C) return;                                               // hw % 4 == 0: a token group is all-in or all-out
    const float *f = a.feat[l] + ((int64_t)b * C + c) * hw + t;
    float4 fr[4], pr[4];
#pragma unroll
    for (int i = 0; i < 4; ++i) fr[i] = ld_stream_f4(f + (int64_t)i * hw);      // channel c + i, tokens t .. t + 3
    const float4 le = ldg_f4(level_embeds + a.level[l] * C + c);
    const int64_t row0 = (int64_t)b * nv + a.start[l] + t;
    if (pos_tok) {
#pragma unroll
        for (int j = 0; j < 4; ++j) pr[j] = ld_stream_f4(pos_tok + (row0 + j) * C + c);  // token t + j, channels c .. c + 3
    } else {
        const float *p = a.pos[l] + ((int64_t)b * C + c) * hw + t;
        float4 q[4];
#pragma unroll
        for (int i = 0; i < 4; ++i) q[i] = ld_stream_f4(p + (int64_t)i * hw);
        pr[0] = make_float4(q[0].x, q[1].x, q[2].x, q[3].x), pr[1] = make_float4(q[0].y, q[1].y, q[2].y, q[3].y);
        pr[2] = make_float4(q[0].z, q[1].z, q[2].z, q[3].z), pr[3] = make_float4(q[0].w, q[1].w, q[2].w, q[3].w);
    }
    const float4 ft[4] = {make_float4(fr[0].x, fr[1].x, fr[2].x, fr[3].x), make_float4(fr[0].y, fr[1].y, fr[2].y, fr[3].y),
                          make_float4(fr[0].z, fr[1].z, fr[2].z, fr[3].z), make_float4(fr[0].w, fr[1].w, fr[2].w, fr[3].w)};
#pragma unroll
    for (int j = 0; j < 4; ++j) {
        const float4 pv = make_float4(pr[j].x + le.x, pr[j].y + le.y, pr[j].z + le.z, pr[j].w + le.w);
        const float k = __ldg(keep + row0 + j);
        const int64_t o = (row0 + j) * C + c;
        *reinterpret_cast<float4 *>(feat_tok + o) = ft[j];
        *reinterpret_cast<float4 *>(lpos_tok + o) = pv;
        *reinterpret_cast<float4 *>(x_tok + o) = make_float4((ft[j].x + pv.x) * k, (ft[j].y + pv.y) * k, (ft[j].z + pv.z) * k, (ft[j].w + pv.w) * k);
    }
}
}  // namespace sdetr

static int flatten_tokens_impl(const float *const *feats_host, const float *const *pos_host, const float *pos_tokens,
                               const float *level_embeds, const float *keep, const int32_t *level_size_host, int batch,
                               int channels, int num_levels, float *feat_tok, float *lpos_tok, float *x_tok,
                               sdetr_stream_t stream) {
    SDETR_REQUIRE(feats_host && (pos_host || pos_tokens) && level_embeds && keep && level_size_host && feat_tok && lpos_tok && x_tok,
                  SDETR_ERR_INVALID_ARG, "flatten_tokens: null pointer");
    SDETR_REQUIRE(batch > 0 && channels > 0 && num_levels > 0 && num_levels <= kMaxLevels, SDETR_ERR_INVALID_ARG,
                  "flatten_tokens: bad sizes");
    FlattenArgs a{};
    a.L = num_levels;
    int nv = 0, tiles = 0;
    for (int l = 0; l < num_levels; ++l) {
        SDETR_REQUIRE(feats_host[l] && (pos_tokens || pos_host[l]) && level_size_host[l] > 0, SDETR_ERR_INVALID_ARG,
                      "flatten_tokens: level %d", l);
        a.feat[l] = feats_host[l], a.pos[l] = pos_tokens ? nullptr : pos_host[l], a.size[l] = level_size_host[l], a.start[l] = nv, a.tile0[l] = tiles;
        nv += level_size_host[l];
        tiles += (level_size_host[l] + 31) / 32;
    }
    a.tile0[num_levels] = tiles;
    // levels with hw % 4 == 0 (16-byte aligned channel rows) go to the vectorised kernel, the others to the tile kernel
    bool vec_ok = channels % 4 == 0 && aligned16(feat_tok) && aligned16(lpos_tok) && aligned16(x_tok) && aligned16(level_embeds) &&
                  (!pos_tokens || aligned16(pos_tokens)) && g_flatten_vec.load();
    FlattenArgs v{}, r{};
    int vt = 0, rt = 0;
    for (int l = 0; l < num_levels; ++l) {
        const bool lv = vec_ok && level_size_host[l] % 4 == 0 && aligned16(feats_host[l]) && (pos_tokens || aligned16(pos_host[l]));
        FlattenArgs &d = lv ? v : r;
        int &dt = lv ? vt : rt;
        d.feat[d.L] = a.feat[l], d.pos[d.L] = a.pos[l], d.size[d.L] = a.size[l], d.start[d.L] = a.start[l], d.tile0[d.L] = dt;
        dt += lv ? (level_size_host[l] + 15) / 16 : (level_size_host[l] + 31) / 32;
        // level_embeds is indexed by the ORIGINAL level: the kernels add level_embeds + l * C, so pass a per-entry offset
        d.level[d.L] = l;
        ++d.L;
    }
    v.tile0[v.L] = vt, r.tile0[r.L] = rt;
    if (v.L) {
        dim3 grid(vt, (channels + 255) / 256, batch);
        flatten_tokens_vec_kernel<<<grid, 256, 0, (cudaStream_t)stream>>>(v, level_embeds, keep, nv, channels, feat_tok, lpos_tok, x_tok,
                                                                          pos_tokens);
        const int rc = check_launch("flatten_tokens/vec");
        if (rc != SDETR_OK) return rc;
    }
    if (r.L) {
        dim3 grid(rt, (channels + 31) / 32, batch);
        flatten_tokens_kernel<<<grid, 256, 0, (cudaStream_t)stream>>>(r, level_embeds, keep, nv, channels, feat_tok, lpos_tok, x_tok,
                                                                      pos_tokens);
        return check_launch("flatten_tokens");
    }
    return SDETR_OK;
}

extern "C" int sdetr_flatten_set_vectorized(int enable) {  // testing knob: 0 = every level through the shared-memory tile kernel
    g_flatten_vec = enable ? 1 : 0;
    return SDETR_OK;
}

extern "C" int sdetr_flatten_tokens(const float *const *feats_host, const float *const *pos_host, const float *level_embeds,
                                    const float *keep, const int32_t *level_size_host, int batch, int channels,
                                    int num_levels, float *feat_tok, float *lpos_tok, float *x_tok, sdetr_stream_t stream) {
    return flatten_tokens_impl(feats_host, pos_host, nullptr, level_embeds, keep, level_size_host, batch, channels, num_levels,
                               feat_tok, lpos_tok, x_tok, stream);
}

extern "C" int sdetr_flatten_tokens_pos(const float *const *feats_host, const float *pos_tokens, const float *level_embeds,
                                        const float *keep, const int32_t *level_size_host, int batch, int channels,
                                        int num_levels, float *feat_tok, float *lpos_tok, float *x_tok, sdetr_stream_t stream) {
    SDETR_REQUIRE(pos_tokens, SDETR_ERR_INVALID_ARG, "flatten_tokens_pos: null position tokens");
    return flatten_tokens_impl(feats_host, nullptr, pos_tokens, level_embeds, keep, level_size_host, batch, channels, num_levels,
                               feat_tok, lpos_tok, x_tok, stream);
}

// ---- layout hand-off to / from a convolutional neck (salience_transformer.py:185-192) -----------------------------------------
// tokens (b,Nv,C) <-> per-level NCHW maps (b,C,H_l*W_l): 32x32 tiles transposed through shared memory, both directions
// coalesced.  to_maps != 0: tokens -> maps (the reference's split + transpose + contiguous + reshape); else maps -> tokens
// (its flatten(2).transpose(1,2) + cat).
namespace sdetr {
__global__ void __launch_bounds__(256) token_map_transpose_kernel(FlattenArgs a, int nv, int C, float *__restrict__ tokens,
                                                                  int to_maps) {
    __shared__ float tile[32][33];
    int l = 0;
#pragma unroll
    for (int u = 1; u < kMaxLevels; ++u)
        if (u < a.L && (int)blockIdx.x >= a.tile0[u]) l = u;
    const int t0 = ((int)blockIdx.x - a.tile0[l]) * 32, c0 = blockIdx.y * 32, b = blockIdx.z;
    const int hw = a.size[l];
    const int tx = threadIdx.x & 31, ty = threadIdx.x >> 5;  // 32 x 8
    float *map = const_cast<float *>(a.feat[l]) + ((int64_t)b * C + c0) * hw;
    float *tok = tokens + ((int64_t)b * nv + a.start[l]) * C;
    if (to_maps) {
#pragma unroll
        for (int i = 0; i < 4; ++i) {  // read tokens: consecutive channels of one token are contiguous
            const int t = t0 + ty + 8 * i, c = c0 + tx;
            tile[ty + 8 * i][tx] = (t < hw && c < C) ? tok[(int64_t)t * C + c] : 0.f;
        }
        __syncthreads();
#pragma unroll
        for (int i = 0; i < 4; ++i) {  // write maps: consecutive tokens of one channel are contiguous
            const int c = ty + 8 * i, t = t0 + tx;
            if (t < hw && c0 + c < C) map[(int64_t)c * hw + t] = tile[tx][c];
        }
    } else {
#pragma unroll
        for (int i = 0; i < 4; ++i) {
            const int c = ty + 8 * i, t = t0 + tx;
            tile[c][tx] = (t < hw && c0 + c < C) ? map[(int64_t)c * hw + t] : 0.f;
        }
        __syncthreads();
#pragma unroll
        for (int i = 0; i < 4; ++i) {
            const int t = t0 + ty + 8 * i, c = c0 + tx;
            if (t < hw && c < C) tok[(int64_t)t * C + c] = tile[tx][ty + 8 * i];
        }
    }
}
}  // namespace sdetr

extern "C" int sdetr_token_map_transpose(float *tokens, float *const *maps_host, const int32_t *level_size_host, int batch,
                                         int channels, int num_levels, int to_maps, sdetr_stream_t stream) {
    SDETR_REQUIRE(tokens && maps_host && level_size_host, SDETR_ERR_INVALID_ARG, "token_map_transpose: null pointer");
    SDETR_REQUIRE(batch > 0 && batch <= 65535 && channels > 0 && num_levels > 0 && num_levels <= kMaxLevels, SDETR_ERR_INVALID_ARG,
                  "token_map_transpose: bad sizes");
    FlattenArgs a{};
    a.L = num_levels;
    int nv = 0, tiles = 0;
    for (int l = 0; l < num_levels; ++l) {
        SDETR_REQUIRE(maps_host[l] && level_size_host[l] > 0, SDETR_ERR_INVALID_ARG, "token_map_transpose: level %d", l);
        a.feat[l] = maps_host[l], a.size[l] = level_size_host[l], a.start[l] = nv, a.tile0[l] = tiles;
        nv += level_size_host[l];
        tiles += (level_size_host[l] + 31) / 32;
    }
    a.tile0[num_levels] = tiles;
    dim3 grid(tiles, (channels + 31) / 32, batch);
    token_map_transpose_kernel<<<grid, 256, 0, (cudaStream_t)stream>>>(a, nv, channels, tokens, to_maps);
    return check_launch("token_map_transpose");
}

// ---- pre-attention gather: t = q[top], x = t + pos[top] (salience_transformer.py:368-371) -----------------------------
namespace sdetr {
__global__ void __launch_bounds__(kRowThreads) rows_gather_add_kernel(const float *__restrict__ src, const float *__restrict__ pos,
                                                                      const int64_t *__restrict__ idx, int batch, int n, int k,
                                                                      int C, float *__restrict__ t, float *__restrict__ x) {
    const int lane = threadIdx.x & 31;
    const int64_t row = (int64_t)blockIdx.x * (kRowThreads / 32) + (threadIdx.x >> 5);
    if (row >= (int64_t)batch * k) return;
    const int b = (int)(row / k);
    const int64_t srow = ((int64_t)b * n + __ldg(idx + row)) * C;
    for (int c = lane * 4; c < C; c += 128) {
        const float4 a = ld_stream_f4(src + srow + c), p = ld_stream_f4(pos + srow + c);
        st_stream_f4(t + row * C + c, a);
        st_stream_f4(x + row * C + c, make_float4(a.x + p.x, a.y + p.y, a.z + p.z, a.w + p.w));
    }
}
}  // namespace sdetr

extern "C" int sdetr_rows_gather_add(const float *src, const float *pos, const int64_t *index, int batch, int num_rows, int k,
                                     int channels, float *t, float *x, sdetr_stream_t stream) {
    SDETR_REQUIRE(src && pos && index && t && x, SDETR_ERR_INVALID_ARG, "rows_gather_add: null pointer");
    SDETR_REQUIRE(batch > 0 && num_rows > 0 && k >= 0 && channels % 4 == 0 && aligned16(src) && aligned16(pos) && aligned16(t) &&
                      aligned16(x),
                  SDETR_ERR_INVALID_ARG, "rows_gather_add: bad sizes / alignment");
    if (k == 0) return SDETR_OK;
    rows_gather_add_kernel<<<row_blocks((int64_t)batch * k), kRowThreads, 0, (cudaStream_t)stream>>>(src, pos, index, batch,
                                                                                                    num_rows, k, channels, t, x);
    return check_launch("rows_gather_add");
}

