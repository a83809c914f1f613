/*
 * TEST INFRASTRUCTURE ONLY -- CPU oracle for the Salience-DETR encoder hot path.
 *
 * A plain-C restatement of the reference algorithm (xiuqhou/Salience-DETR) used as the parity
 * checker for the sm_90a kernels.  Nothing on the product path may link or call this file; only
 * tests/, __graft_entry__.smoke() and bench.py's cpu_baseline / --impl reference legs do.
 *
 * Pinning: the reference ships no tests or golden vectors (SURVEY.md section 4), so this oracle is
 * pinned against OUTPUTS OF THE REFERENCE ITSELF, produced by importing the unmodified reference
 * Python modules in the build container (oracle/make_golden.py -> tests/golden/ *.npz) and checked
 * by tests/test_oracle_golden.py.
 *
 * Reference lines restated here (paths relative to the reference root):
 *   MSDA core forward   models/bricks/ops/cuda/ms_deform_im2col_cuda.cuh:22-73, 226-288
 *                       (numerically equivalent to models/bricks/ms_deform_attn.py:159-212)
 *   MSDA core backward  models/bricks/ops/cuda/ms_deform_im2col_cuda.cuh:76-148, 290-392
 *   salience selection  models/bricks/salience_transformer.py:146-168
 *   token gather        models/bricks/salience_transformer.py:454-461
 *   reference points    models/bricks/salience_transformer.py:417-432
 *   scatter back        models/bricks/salience_transformer.py:474-485
 *   background embed    models/bricks/salience_transformer.py:488-495,
 *                       models/bricks/position_encoding.py:68-95
 *
 * Tie order: torch.topk / torch.sort leave the order of equal keys unspecified.  This oracle (and
 * the CUDA kernels) use the canonical total order "larger score first, then smaller token index";
 * tests compare against the reference on tie-free inputs, or tie groups as sets.
 */
#include <math.h>
#include <stdint.h>
#include <stdlib.h>
#include <string.h>

typedef struct {
    int batch, num_value, heads, head_dim, levels, num_query, points;
} msda_dims;

/* value token (y, x) of one level for head m; NULL when the corner lies outside the map */
static inline const float *corner_ptr(const float *level_base, int H, int W, int heads, int head_dim,
                                      int m, int y, int x) {
    if (y < 0 || x < 0 || y > H - 1 || x > W - 1) return NULL;
    return level_base + ((size_t)(y * W + x) * heads + m) * head_dim;
}

/* ---- MSDA core forward: .cuh:226-288 (+ bilinear helper :22-73) --------------------------- */
void oracle_msda_forward(const float *value, const int64_t *shapes, const int64_t *lsi,
                         const float *loc, const float *attn, float *out, int batch, int num_value,
                         int heads, int head_dim, int levels, int num_query, int points) {
    const int D = head_dim;
#pragma omp parallel for collapse(2) schedule(static)
    for (int b = 0; b < batch; ++b) {
        for (int q = 0; q < num_query; ++q) {
            for (int m = 0; m < heads; ++m) {
                float *o = out + (((size_t)b * num_query + q) * heads + m) * D;
                for (int c = 0; c < D; ++c) o[c] = 0.f;
                const size_t lw = (((size_t)b * num_query + q) * heads + m) * levels * points;
                for (int l = 0; l < levels; ++l) {
                    const int H = (int)shapes[2 * l], W = (int)shapes[2 * l + 1];
                    const float *base = value + ((size_t)b * num_value + lsi[l]) * heads * D;
                    for (int p = 0; p < points; ++p) {
                        const float lx = loc[(lw + l * points + p) * 2 + 0];
                        const float ly = loc[(lw + l * points + p) * 2 + 1];
                        const float a = attn[lw + l * points + p];
                        const float h_im = ly * H - 0.5f, w_im = lx * W - 0.5f; /* :274-275 */
                        if (!(h_im > -1 && w_im > -1 && h_im < H && w_im < W)) continue; /* :277 */
                        const int y0 = (int)floorf(h_im), x0 = (int)floorf(w_im);
                        const float fy = h_im - y0, fx = w_im - x0;
                        const float gy = 1 - fy, gx = 1 - fx;
                        const float *v1 = corner_ptr(base, H, W, heads, D, m, y0, x0);
                        const float *v2 = corner_ptr(base, H, W, heads, D, m, y0, x0 + 1);
                        const float *v3 = corner_ptr(base, H, W, heads, D, m, y0 + 1, x0);
                        const float *v4 = corner_ptr(base, H, W, heads, D, m, y0 + 1, x0 + 1);
                        const float w1 = gy * gx, w2 = gy * fx, w3 = fy * gx, w4 = fy * fx;
                        for (int c = 0; c < D; ++c) {
                            const float s = w1 * (v1 ? v1[c] : 0.f) + w2 * (v2 ? v2[c] : 0.f) +
                                            w3 * (v3 ? v3[c] : 0.f) + w4 * (v4 ? v4[c] : 0.f);
                            o[c] += a * s;
                        }
                    }
                }
            }
        }
    }
}

/* ---- MSDA core backward: .cuh:290-392 (+ helper :76-148) ---------------------------------
 * grad_value must be zero-initialised by the caller (reference: at::zeros_like, .cu:113).
 * Serial over queries inside one image so the += on grad_value needs no atomics; images run in
 * parallel. */
void oracle_msda_backward(const float *value, const int64_t *shapes, const int64_t *lsi,
                          const float *loc, const float *attn, const float *grad_out,
                          float *grad_value, float *grad_loc, float *grad_attn, int batch,
                          int num_value, int heads, int head_dim, int levels, int num_query,
                          int points) {
    const int D = head_dim;
#pragma omp parallel for schedule(static)
    for (int b = 0; b < batch; ++b) {
        for (int q = 0; q < num_query; ++q) {
            for (int m = 0; m < heads; ++m) {
                const float *go = grad_out + (((size_t)b * num_query + q) * heads + m) * D;
                const size_t lw = (((size_t)b * num_query + q) * heads + m) * levels * points;
                for (int l = 0; l < levels; ++l) {
                    const int H = (int)shapes[2 * l], W = (int)shapes[2 * l + 1];
                    const size_t lvl_off = ((size_t)b * num_value + lsi[l]) * heads * D;
                    const float *base = value + lvl_off;
                    float *gbase = grad_value + lvl_off;
                    for (int p = 0; p < points; ++p) {
                        const size_t k = lw + l * points + p;
                        grad_loc[2 * k] = grad_loc[2 * k + 1] = 0.f;
                        grad_attn[k] = 0.f;
                        const float lx = loc[2 * k], ly = loc[2 * k + 1], a = attn[k];
                        const float h_im = ly * H - 0.5f, w_im = lx * W - 0.5f;
                        if (!(h_im > -1 && w_im > -1 && h_im < H && w_im < W)) continue;
                        const int y0 = (int)floorf(h_im), x0 = (int)floorf(w_im);
                        const float fy = h_im - y0, fx = w_im - x0, gy = 1 - fy, gx = 1 - fx;
                        const int ys[4] = {y0, y0, y0 + 1, y0 + 1};
                        const int xs[4] = {x0, x0 + 1, x0, x0 + 1};
                        const float cw[4] = {gy * gx, gy * fx, fy * gx, fy * fx};
                        /* d(sample)/dy and d(sample)/dx coefficients per corner (:108-141) */
                        const float dy[4] = {-gx, -fx, gx, fx};
                        const float dx[4] = {-gy, gy, -fy, fy};
                        float acc_a = 0.f, acc_x = 0.f, acc_y = 0.f;
                        for (int c = 0; c < D; ++c) {
                            const float g = go[c], ga = g * a;
                            float s = 0.f, sy = 0.f, sx = 0.f;
                            for (int j = 0; j < 4; ++j) {
                                const float *v = corner_ptr(base, H, W, heads, D, m, ys[j], xs[j]);
                                if (!v) continue;
                                s += cw[j] * v[c];
                                sy += dy[j] * v[c];
                                sx += dx[j] * v[c];
                                gbase[(v - base) + c] += cw[j] * ga;
                            }
                            acc_a += g * s;
                            acc_x += (float)W * sx * ga;
                            acc_y += (float)H * sy * ga;
                        }
                        grad_attn[k] = acc_a;
                        grad_loc[2 * k] = acc_x;
                        grad_loc[2 * k + 1] = acc_y;
                    }
                }
            }
        }
    }
}

/* ---- salience selection: salience_transformer.py:146-168 ---------------------------------- */
typedef struct {
    float score;
    int64_t index;
} cand_t;

/* canonical total order: larger score first, then smaller token index */
static int cand_before(const void *pa, const void *pb) {
    const cand_t *a = (const cand_t *)pa, *b = (const cand_t *)pb;
    if (a->score > b->score) return -1;
    if (a->score < b->score) return 1;
    return (a->index > b->index) - (a->index < b->index);
}

/*
 * raw_score (b, Nv): MaskPredictor output per token, levels concatenated (finest first)
 * mask      (b, Nv): 1 = padding
 * hw[l], lsi[l]    : level sizes / start offsets;  k[l] = level_token_nums[l]  (py:120)
 * -> selected_inds (b, K) int64, selected_score (b, K), K = sum k[l]   (py:150-158)
 * -> foreground_score (b, Nv)                                          (py:166-168)
 */
void oracle_salience_select(const float *raw_score, const uint8_t *mask, const int64_t *lsi,
                            const int64_t *hw, const int32_t *k, int batch, int num_value,
                            int levels, int64_t *selected_inds, float *selected_score,
                            float *foreground_score) {
    int K = 0;
    for (int l = 0; l < levels; ++l) K += k[l];
    /* batch-global minima: per level (py:146 `score.min()`) and over everything (py:168) */
    float gmin = INFINITY;
    float *lmin = (float *)malloc(sizeof(float) * levels);
    for (int l = 0; l < levels; ++l) {
        lmin[l] = INFINITY;
        for (int b = 0; b < batch; ++b)
            for (int64_t t = 0; t < hw[l]; ++t) {
                const float s = raw_score[(size_t)b * num_value + lsi[l] + t];
                if (s < lmin[l]) lmin[l] = s;
            }
        if (lmin[l] < gmin) gmin = lmin[l];
    }
    int64_t maxhw = 0;
    for (int l = 0; l < levels; ++l)
        if (hw[l] > maxhw) maxhw = hw[l];
    cand_t *lvl = (cand_t *)malloc(sizeof(cand_t) * (size_t)maxhw);
    cand_t *all = (cand_t *)malloc(sizeof(cand_t) * (size_t)(K > 0 ? K : 1));
    for (int b = 0; b < batch; ++b) {
        int n = 0;
        for (int l = 0; l < levels; ++l) {
            for (int64_t t = 0; t < hw[l]; ++t) {
                const size_t g = (size_t)b * num_value + lsi[l] + t;
                lvl[t].score = mask[g] ? lmin[l] : raw_score[g]; /* masked_fill(mask, min) py:146 */
                lvl[t].index = lsi[l] + t;                       /* + level_start_index  py:151 */
            }
            qsort(lvl, (size_t)hw[l], sizeof(cand_t), cand_before); /* topk(k_l)  py:150 */
            for (int j = 0; j < k[l]; ++j) all[n++] = lvl[j];
        }
        qsort(all, (size_t)K, sizeof(cand_t), cand_before); /* cat + sort(desc) + gather py:156-158 */
        for (int j = 0; j < K; ++j) {
            selected_inds[(size_t)b * K + j] = all[j].index;
            selected_score[(size_t)b * K + j] = all[j].score;
        }
        for (int t = 0; t < num_value; ++t) {
            const size_t g = (size_t)b * num_value + t;
            foreground_score[g] = mask[g] ? gmin : raw_score[g]; /* py:167-168 */
        }
    }
    free(lvl);
    free(all);
    free(lmin);
}

/* ---- token budgets: salience_transformer.py:117-121,161-165 -------------------------------
 * fp32 multiply then truncation, exactly as `(int64 * float32_buffer).int()` does. */
void oracle_token_budgets(const uint8_t *mask, const int64_t *lsi, const int64_t *hw, int batch,
                          int num_value, int levels, const float *level_ratio, int num_layers,
                          const float *layer_ratio, int32_t *level_token_nums /* (L) */,
                          int32_t *focus_token_nums /* (b) */, int64_t *layer_num_query /* (layers) */) {
    for (int l = 0; l < levels; ++l) level_token_nums[l] = 0;
    for (int b = 0; b < batch; ++b) {
        int32_t total = 0;
        for (int l = 0; l < levels; ++l) {
            int64_t valid = 0;
            for (int64_t t = 0; t < hw[l]; ++t) valid += !mask[(size_t)b * num_value + lsi[l] + t];
            const int32_t f = (int32_t)((float)valid * level_ratio[l]);
            if (f > level_token_nums[l]) level_token_nums[l] = f;
            total += f;
        }
        focus_token_nums[b] = total;
    }
    int64_t K = 0;
    for (int l = 0; l < levels; ++l) K += level_token_nums[l];
    for (int j = 0; j < num_layers; ++j) layer_num_query[j] = (int64_t)((float)K * layer_ratio[j]);
}

/* ---- reference points of the selected tokens: py:417-432 gathered by py:458-461 ----------- */
static void token_to_lyx(int64_t t, const int64_t *lsi, const int64_t *shapes, int levels, int *l,
                         int *y, int *x) {
    int lv = levels - 1;
    while (lv > 0 && t < lsi[lv]) --lv;
    const int64_t r = t - lsi[lv];
    *l = lv;
    *y = (int)(r / shapes[2 * lv + 1]);
    *x = (int)(r % shapes[2 * lv + 1]);
}

/*
 * Fused restatement of the four gathers py:454-461.  inds has row stride inds_stride (a prefix
 * view of selected_inds).  ref_q[b,q,l',:] = ((x+.5)/(vr[b,lv,0]*W), (y+.5)/(vr[b,lv,1]*H)) * vr[b,l',:]
 */
void oracle_token_gather(const float *tokens, const float *pos, const float *fg,
                         const float *valid_ratios /* (b,L,2) */, const int64_t *inds,
                         int64_t inds_stride, const int64_t *shapes, const int64_t *lsi, int batch,
                         int num_value, int channels, int levels, int num_query, float *query,
                         float *query_pos, float *fg_q, float *ref_q) {
#pragma omp parallel for collapse(2) schedule(static)
    for (int b = 0; b < batch; ++b)
        for (int q = 0; q < num_query; ++q) {
            const int64_t t = inds[(size_t)b * inds_stride + q];
            const size_t src = ((size_t)b * num_value + t) * channels;
            const size_t dst = ((size_t)b * num_query + q) * channels;
            memcpy(query + dst, tokens + src, sizeof(float) * channels);
            memcpy(query_pos + dst, pos + src, sizeof(float) * channels);
            fg_q[(size_t)b * num_query + q] = fg[(size_t)b * num_value + t];
            int lv, y, x;
            token_to_lyx(t, lsi, shapes, levels, &lv, &y, &x);
            const float *vr = valid_ratios + (size_t)b * levels * 2;
            const float rx = ((float)x + 0.5f) / (vr[2 * lv] * (float)shapes[2 * lv + 1]);
            const float ry = ((float)y + 0.5f) / (vr[2 * lv + 1] * (float)shapes[2 * lv]);
            float *r = ref_q + ((size_t)b * num_query + q) * levels * 2;
            for (int l2 = 0; l2 < levels; ++l2) {
                r[2 * l2] = rx * vr[2 * l2];
                r[2 * l2 + 1] = ry * vr[2 * l2 + 1];
            }
        }
}

/* ---- scatter back: py:474-485 (in place on `tokens`; first min(focus[b], Nq) rows only) ---- */
void oracle_token_scatter(float *tokens, const float *query, const int64_t *inds, int64_t inds_stride,
                          const int32_t *focus_token_nums, int batch, int num_value, int channels,
                          int num_query) {
    for (int b = 0; b < batch; ++b) {
        int n = focus_token_nums[b] < num_query ? focus_token_nums[b] : num_query;
        for (int q = 0; q < n; ++q) {
            const int64_t t = inds[(size_t)b * inds_stride + q];
            memcpy(tokens + ((size_t)b * num_value + t) * channels,
                   query + ((size_t)b * num_query + q) * channels, sizeof(float) * channels);
        }
    }
}

/* ---- background embedding: py:488-495, position_encoding.py:81-95 --------------------------
 * tokens[b,t,:] += [col_embed[x] | row_embed[y]] unless t is padding or among the last layer's
 * query indices. */
void oracle_background_embed(float *tokens, const uint8_t *mask, const int64_t *last_inds,
                             int64_t inds_stride, int num_last, const float *row_embed,
                             const float *col_embed, const int64_t *shapes, const int64_t *lsi,
                             int batch, int num_value, int channels, int levels) {
    const int half = channels / 2;
    uint8_t *skip = (uint8_t *)malloc((size_t)num_value);
    for (int b = 0; b < batch; ++b) {
        memcpy(skip, mask + (size_t)b * num_value, (size_t)num_value);
        for (int q = 0; q < num_last; ++q) skip[last_inds[(size_t)b * inds_stride + q]] = 1;
        for (int t = 0; t < num_value; ++t) {
            if (skip[t]) continue;
            int lv, y, x;
            token_to_lyx(t, lsi, shapes, levels, &lv, &y, &x);
            float *o = tokens + ((size_t)b * num_value + t) * channels;
            for (int c = 0; c < half; ++c) {
                o[c] += col_embed[(size_t)x * half + c];
                o[half + c] += row_embed[(size_t)y * half + c];
            }
        }
    }
    free(skip);
}

/* ---- coarse-to-fine modulation: salience_transformer.py:134-143 ----------------------------
 * up = bilinear resize (align_corners=True) of the coarser level's score map to (H,W);
 * out = mem + mem * up * alpha.  Follows ATen's upsample_bilinear2d index arithmetic:
 * src = dst * (in-1)/(out-1) (scale computed in fp32), lambda from the fp32 source coordinate. */
void oracle_score_modulate(const float *mem /* (b,H*W,C) */, const float *coarse /* (b,Hc*Wc) */,
                           float alpha, int batch, int H, int W, int Hc, int Wc, int channels,
                           float *out) {
    const float sy = H > 1 ? (float)(Hc - 1) / (float)(H - 1) : 0.f;
    const float sx = W > 1 ? (float)(Wc - 1) / (float)(W - 1) : 0.f;
#pragma omp parallel for collapse(2) schedule(static)
    for (int b = 0; b < batch; ++b)
        for (int y = 0; y < H; ++y) {
            const float fy = sy * (float)y;
            const int y0 = (int)fy, y1 = y0 + (y0 < Hc - 1 ? 1 : 0);
            const float ly = fy - (float)y0, hy = 1.f - ly;
            for (int x = 0; x < W; ++x) {
                const float fx = sx * (float)x;
                const int x0 = (int)fx, x1 = x0 + (x0 < Wc - 1 ? 1 : 0);
                const float lx = fx - (float)x0, hx = 1.f - lx;
                const float *c = coarse + (size_t)b * Hc * Wc;
                const float up = hy * (hx * c[y0 * Wc + x0] + lx * c[y0 * Wc + x1]) +
                                 ly * (hx * c[y1 * Wc + x0] + lx * c[y1 * Wc + x1]);
                const size_t o = ((size_t)b * H * W + (size_t)y * W + x) * channels;
                for (int ch = 0; ch < channels; ++ch) out[o + ch] = mem[o + ch] + mem[o + ch] * up * alpha;
            }
        }
}
