/*
 * sdetr_b200.h -- C-ABI of the H100-native (sm_90a) Salience-DETR encoder hot path.
 *
 * This is the drop-in boundary: plain pointers and sizes, no torch types.  All pointers are DEVICE
 * pointers unless the parameter name ends in `_host`.  Every call is asynchronous on `stream`
 * (a cudaStream_t passed as void*) of the CURRENT device, allocates nothing, never synchronises, and is
 * re-entrant across streams, threads and devices (per-device kernel attributes are set on first use per device).
 * The only process-global state are the knobs sdetr_set_option / sdetr_set_persistent_ctas (atomics: a call reads them once
 * at launch).  Return value: 0 on success, negative sdetr_status on error (message: sdetr_last_error(),
 * thread-local).  Launch errors are RETURNED (the reference only printf's them:
 * models/bricks/ops/cuda/ms_deform_im2col_cuda.cuh:937-941, 1310-1314).
 *
 * Citations below are relative to the reference root (xiuqhou/Salience-DETR @ 6262e05).
 * "(b,Nq,M,L,P,2)" etc. are row-major contiguous shapes; fp32 unless stated.
 */
#ifndef SDETR_B200_H
#define SDETR_B200_H

#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

typedef void *sdetr_stream_t; /* cudaStream_t */

enum sdetr_status {
    SDETR_OK = 0,
    SDETR_ERR_INVALID_ARG = -1, /* null pointer, non-positive size, misaligned pointer */
    SDETR_ERR_UNSUPPORTED = -2, /* shape outside the compiled kernel family */
    SDETR_ERR_CUDA = -3,        /* cudaGetLastError() after a launch */
    SDETR_ERR_WORKSPACE = -4    /* workspace too small */
};

/* library version (major*10000 + minor*100 + patch) and last error string of the calling thread */
int sdetr_version(void);
const char *sdetr_last_error(void);
/* number of kernels this library has launched in the calling process (bench.py "gpu_launches") */
unsigned long long sdetr_launch_count(void);
/* The persistent tensor-core kernels (the sdetr_gemm_* entry points, sdetr_ffn_fused_layernorm) launch one CTA per SM and leave no room
 * for anything else on it; n > 0 caps them at n CTAs so that concurrently running streams (other lanes of a pipeline) find free
 * SMs for their small kernels.  0 (default) = every SM.  Process-wide. */
int sdetr_set_persistent_ctas(int n);

/* process-wide tuning knobs (benchmark sweeps): "msda_min_blocks" (2..4 resident CTAs/SM the specialised
 * MSDA kernel is compiled for), "msda_chunk" (queries per CTA in the head-major schedule). */
int sdetr_set_option(const char *name, int value);

/* ------------------------------------------------------------------------------------------------
 * MSDA core forward.  Replaces `_C.ms_deform_attn_forward`
 *   (models/bricks/ops/cuda/ms_deform_attn_cuda.cu:12-72, kernel ms_deform_im2col_cuda.cuh:226-288;
 *    numerically the same op as multi_scale_deformable_attn_pytorch, models/bricks/ms_deform_attn.py:159-212)
 *   out[b,q,m,:] = sum_{l,p} attn[b,q,m,l,p] * bilinear_zero_pad(value_l[b,:,m,:], loc[b,q,m,l,p])
 *   pixel coords  x = loc_x*W_l - 0.5, y = loc_y*H_l - 0.5 (align_corners=False).
 * value (b,Nv,M,D); spatial_shapes (L,2) int64 (H,W); level_start_index (L) int64 -- both on the device,
 * exactly the tensors the reference op receives; sampling_loc (b,Nq,M,L,P,2); attn_weight (b,Nq,M,L,P);
 * output (b,Nq,M*D), fully overwritten.  The reference's im2col_step batching (.cu:42-66) has no
 * numerical effect and is not needed (one launch covers the whole batch).
 */
int sdetr_msda_forward(const float *value, const int64_t *spatial_shapes, const int64_t *level_start_index,
                       const float *sampling_loc, const float *attn_weight, float *output, int batch,
                       int num_value, int num_heads, int head_dim, int num_levels, int num_query,
                       int num_points, sdetr_stream_t stream);

/* Extended form used by the encoder mirror:
 *  - value_batch_stride / value_token_stride (in floats) let `value` be a column slice of a wider
 *    projection buffer (the six layers' value_proj outputs share one GEMM; salience_transformer.py:452
 *    feeds the SAME value tokens to every layer);
 *  - query_order (b,Nq) int32, nullable: permutation giving the PROCESSING order of the queries
 *    (spatially tiled for L1 locality; results are written to their original rows);
 *  - schedule: 0 = query-major (4 queries x all heads per CTA), 1 = head-major chunks
 *    (one head of `chunk` consecutive queries of the processing order per CTA). */
int sdetr_msda_forward_ex(const float *value, int64_t value_batch_stride, int64_t value_token_stride,
                          const int64_t *spatial_shapes, const int64_t *level_start_index,
                          const float *sampling_loc, const float *attn_weight, float *output, int batch,
                          int num_value, int num_heads, int head_dim, int num_levels, int num_query,
                          int num_points, const int32_t *query_order, int schedule, sdetr_stream_t stream);

/* Fused attention-weight softmax + sampling-location arithmetic + MSDA core
 *   (models/bricks/ms_deform_attn.py:322-344 fused into the core, 2-d reference points):
 *   proj (b,Nq,proj_stride): per query, M*L*P*2 raw sampling offsets followed by M*L*P raw attention
 *   logits (the concatenated sampling_offsets | attention_weights Linear output);
 *   ref_points (b,Nq,L,2);  loc = ref + off / (W_l,H_l);  attn = softmax over the L*P logits of a head.
 *   loc_out / attn_out: nullable; when given they receive sampling_locations / attention_weights in the
 *   reference layouts (needed by the backward).  Other arguments as sdetr_msda_forward_ex. */
int sdetr_msda_fused_forward(const float *value, int64_t value_batch_stride, int64_t value_token_stride,
                             const int64_t *spatial_shapes, const int64_t *level_start_index,
                             const float *ref_points, const float *proj, int64_t proj_stride, float *output,
                             float *loc_out, float *attn_out, int batch, int num_value, int num_heads,
                             int head_dim, int num_levels, int num_query, int num_points,
                             const int32_t *query_order, int schedule, sdetr_stream_t stream);

/* Same with 4-d reference BOXES (cx, cy, w, h), the decoder's cross-attention (ms_deform_attn.py:345-349):
 * ref_boxes (b,Nq,L,4), 16-byte aligned;  loc = ref_xy + off / P * ref_wh * 0.5  (the reference's operation order). */
int sdetr_msda_fused_forward_boxes(const float *value, int64_t value_batch_stride, int64_t value_token_stride,
                                   const int64_t *spatial_shapes, const int64_t *level_start_index,
                                   const float *ref_boxes, const float *proj, int64_t proj_stride, float *output,
                                   float *loc_out, float *attn_out, int batch, int num_value, int num_heads, int head_dim,
                                   int num_levels, int num_query, int num_points, const int32_t *query_order, int schedule,
                                   sdetr_stream_t stream);

/* Benchmarking variant "msda_tma" (sdetr_set_option("msda_tma", 1); D = 32, L = 4, P = 4, head-major schedule with a query
 * order): the fused / plain forward stages per-level value windows in shared memory with TMA (csrc/msda_forward_tma.cu).
 * TMA tensor maps are encoded on the host, which needs the level shapes as HOST integers: give them here once per
 * geometry (process-global; the default path reads the shapes from the device tensors and needs none of this). */
int sdetr_msda_set_host_shapes(int num_levels, const int32_t *level_h_host, const int32_t *level_w_host);

/* Two-stage proposal selection, NMS on token indices (SalienceTransformer.nms_on_topk_index, salience_transformer.py:
 * 249-295 = torchvision.ops.batched_nms over boxes (x-1,y-1,x+1,y+1) on each (image, level) grid).  topk_index (b,k) int64:
 * candidate tokens in descending score order (the rank decides who suppresses whom).  kept_index (b,k) int64 receives the
 * surviving tokens in the same order (first kept_count[b] entries valid), keep_flag (b,k) uint8 (nullable) the per-
 * candidate verdict.  k < 65535; the rank table (2 bytes per token) lives in shared memory: num_value up to ~98 000.
 * A box is suppressed when its float32 IoU > iou_threshold; torchvision compares with a double threshold, so a caller
 * holding a double passes the largest float not above it (cabi.nms_iou_threshold_f32), not the nearest one. */
int sdetr_nms_topk_index(const int64_t *topk_index, int batch, int k, int num_value, int num_levels,
                         const int32_t *level_h_host, const int32_t *level_w_host, float iou_threshold, int64_t *kept_index,
                         int32_t *kept_count, uint8_t *keep_flag, sdetr_stream_t stream);


/* MSDA core backward.  Replaces `_C.ms_deform_attn_backward`
 *   (ms_deform_attn_cuda.cu:75-145; kernels ms_deform_im2col_cuda.cuh:76-148, 290-392).
 * grad_output (b,Nq,M*D) -> grad_value (b,Nv,M,D), grad_sampling_loc, grad_attn_weight (shapes of the
 * inputs).  All three outputs are fully written (grad_value is zeroed on `stream` first; the reference
 * allocates zeros, .cu:113-115).  grad_value accumulates with fp32 red.global adds like the reference's
 * atomicAdd (run-to-run order of additions is not deterministic). */
int sdetr_msda_backward(const float *value, const int64_t *spatial_shapes, const int64_t *level_start_index,
                        const float *sampling_loc, const float *attn_weight, const float *grad_output,
                        float *grad_value, float *grad_sampling_loc, float *grad_attn_weight, int batch,
                        int num_value, int num_heads, int head_dim, int num_levels, int num_query,
                        int num_points, sdetr_stream_t stream);

/* Deterministic MSDA core backward: the contract of sdetr_msda_backward (same arguments, checks and head dims
 * {4,8,16,32,64,128}), and grad_value is BIT-IDENTICAL for identical inputs whatever the launch order, the grid or the order
 * of the queries.  grad_sampling_loc and grad_attn_weight are computed by the same code as sdetr_msda_backward's and are
 * bit-identical to its results.
 * grad_value accumulates in fixed point: each corner contribution (w_corner * attn) * grad_out is multiplied by one exact
 * power of two 2^s, rounded to int64 and added with integer atomics (associative: the order of additions cannot matter).
 * s is computed on the device (no host read; the call can be captured in a CUDA graph) so that
 * max|grad_out| * max|attn| * num_query * num_points * 2^s <= 2^62 with both maxima rounded up to powers of two; no sum can
 * overflow.  The absolute error of a grad_value entry is at most (its number of contributions / 2 + 1) * 2^-s.
 * Non-finite values: a non-finite sampling location contributes exactly 0 (as in sdetr_msda_backward); a NaN or infinity
 * anywhere in grad_output or attn_weight makes EVERY grad_value entry NaN.
 * workspace: sdetr_msda_backward_deterministic_workspace() bytes, 16-byte aligned = the int64 accumulator
 * (8 * b*Nv*M*D bytes) and 32 bytes of scale / flag / reduction state; zeroed on `stream` by the call.  Too small:
 * SDETR_ERR_WORKSPACE.  Cost: four 8-byte integer reductions per lane and corner where the fp32 path issues one 16-byte one. */
size_t sdetr_msda_backward_deterministic_workspace(int batch, int num_value, int num_heads, int head_dim);
int sdetr_msda_backward_deterministic(const float *value, const int64_t *spatial_shapes, const int64_t *level_start_index,
                                      const float *sampling_loc, const float *attn_weight, const float *grad_output,
                                      float *grad_value, float *grad_sampling_loc, float *grad_attn_weight, int batch,
                                      int num_value, int num_heads, int head_dim, int num_levels, int num_query,
                                      int num_points, void *workspace, size_t workspace_bytes, sdetr_stream_t stream);

/* Backward of the coarse-to-fine score upsample F.interpolate(mode="bilinear", align_corners=True) from (planes, Hc, Wc) to
 * (planes, H, W) (salience_transformer.py:134-143), deterministic: in gather form, each coarse cell sums the weighted
 * gradients of the fine pixels whose stencil contains it, in row-major order, and is written once (no atomics; torch's
 * CUDA backward of the op scatters with atomics).  The stencil uses the fp32 quantities of torch's forward:
 * scale = (in-1)/(out-1), src = scale*dst, i0 = (int)src, i1 = i0 + (i0 < in-1), lambda = src - i0.
 * grad_fine (planes,H,W) -> grad_coarse (planes,Hc,Wc), fully written. */
int sdetr_upsample_bilinear_ac_backward(const float *grad_fine, int planes, int H, int W, int Hc, int Wc, float *grad_coarse,
                                        sdetr_stream_t stream);

/* ------------------------------------------------------------------------------------------------
 * Hierarchical salience token filter (models/bricks/salience_transformer.py:146-168), one call:
 *   per level l: v = where(mask, min over the whole (b,HW_l) score tensor, score)       (:146)
 *                top-k_l of v per image, indices offset by level_start                  (:150-151)
 *   concatenate levels, sort by score descending, reorder indices                       (:156-158)
 *   foreground_score = where(mask, min over the whole (b,Nv) tensor, score)             (:166-168)
 * Order of equal scores (unspecified in torch.topk/sort): larger score first, then smaller token index.
 * As in torch.sort, -0 == +0 and every NaN (either sign) ranks above +inf.  A minimum over scores that hold a
 * NaN is the NaN 0x7fffffff; of +0 and -0 it is -0.  selected_score keeps the bits of the score ranked.
 * raw_score (b,Nv); mask (b,Nv) uint8, 1 = padding; level_start_host / level_size_host / level_k_host:
 * HOST int32 arrays of length num_levels (k_l = level_token_nums, :120; k_l <= size_l).
 * -> selected_inds (b,K) int64, selected_score (b,K) (both may be NULL when K = 0), foreground_score (b,Nv),
 * K = sum k_l.
 * tile_order (b,K) int32, nullable: positions 0..K-1 of each image's selected list ordered by the
 * spatial cell of their token (cell_px x cell_px image pixels; level-l token = level_stride_host[l] px):
 * the processing order handed to sdetr_msda_forward_ex after sdetr_order_prefixes().
 * workspace: sdetr_salience_select_workspace() bytes, 256-byte aligned.
 */
size_t sdetr_salience_select_workspace(int batch, int num_value, int num_levels);
int sdetr_salience_select(const float *raw_score, const uint8_t *mask, const int32_t *level_start_host,
                          const int32_t *level_size_host, const int32_t *level_k_host,
                          const int32_t *level_width_host, const int32_t *level_stride_host, int cell_px,
                          int batch, int num_value, int num_levels, int64_t *selected_inds,
                          float *selected_score, float *foreground_score, int32_t *tile_order,
                          void *workspace, size_t workspace_bytes, sdetr_stream_t stream);

/* Per-layer prefixes of the processing order: for each layer j (prefix length nq_host[j] of the selected
 * list, salience_transformer.py:161-165) emit the positions < nq_j in tile order:
 * out_orders + order_offset_host[j] : (b, nq_j) int32. */
int sdetr_order_prefixes(const int32_t *tile_order, int batch, int K, int num_layers,
                         const int32_t *nq_host, const int64_t *order_offset_host, int32_t *out_orders,
                         sdetr_stream_t stream);

/* Generic segmented top-k by score (descending, NaNs first; ties: smaller position first).  Used for the
 * "top-300 most salient tokens" pre-attention selection (salience_transformer.py:366-367).
 * score (segments, n) -> topk_index (segments, k) int64 positions within the segment.
 * workspace: sdetr_topk_workspace() bytes. */
size_t sdetr_topk_workspace(int segments, int n);
int sdetr_topk_desc(const float *score, int segments, int n, int k, int64_t *topk_index, void *workspace,
                    size_t workspace_bytes, sdetr_stream_t stream);

/* ------------------------------------------------------------------------------------------------
 * Token movement around the encoder layers (models/bricks/salience_transformer.py:454-495).
 */

/* Fused four-way gather (:454-461).  inds: int64, row stride inds_stride (a prefix view of selected_inds).
 * tokens/pos (b,Nv,C), fg (b,Nv), valid_ratios (b,L,2) ->
 * query (b,Nq,C), query_pos (b,Nq,C), fg_q (b,Nq), ref_q (b,Nq,L,2) where ref_q is the gathered row of
 * get_reference_points (:417-432), recomputed from the token's (level,y,x) with identical fp32 arithmetic.
 * query_sum (b,Nq,C), may be NULL: query + query_pos, the `with_pos_embed` input of the layer's attention (:381). */
int sdetr_token_gather(const float *tokens, const float *pos, const float *fg, const float *valid_ratios,
                       const int64_t *inds, int64_t inds_stride, const int64_t *spatial_shapes,
                       const int64_t *level_start_index, int batch, int num_value, int channels,
                       int num_levels, int num_query, float *query, float *query_pos, float *fg_q,
                       float *ref_q, float *query_sum, sdetr_stream_t stream);

/* In-place scatter-back (:474-485): tokens[b, inds[b,q], :] = query[b,q,:] for q < min(focus[b], Nq).
 * focus_token_nums (b) int32 on the device (no host sync, unlike the reference's per-image slicing). */
int sdetr_token_scatter(float *tokens, const float *query, const int64_t *inds, int64_t inds_stride,
                        const int32_t *focus_token_nums, int batch, int num_value, int channels,
                        int num_query, sdetr_stream_t stream);

/* Background embedding (:488-495, position_encoding.py:81-95), in place:
 * tokens[b,t,:] += [col_embed[x] | row_embed[y]] unless mask[b,t] or t in last_inds[b,:num_last].
 * row_embed / col_embed: (num_embeddings, channels/2) tables (max_num_embedding, :400-407).  A feature map taller or
 * wider than the table is an index error in the reference (nn.Embedding): pass the HOST copy of the level shapes in
 * spatial_shapes_host ((L,2) int64 [H,W], may be NULL) to get SDETR_ERR_INVALID_ARG for it; the kernel itself never
 * reads outside the tables (indices are clamped).  flags: (b,Nv) uint8 scratch. */
int sdetr_background_embed(float *tokens, const uint8_t *mask, const int64_t *last_inds, int64_t inds_stride,
                           int num_last, const float *row_embed, const float *col_embed, int num_embeddings,
                           const int64_t *spatial_shapes, const int64_t *spatial_shapes_host,
                           const int64_t *level_start_index, int batch, int num_value, int channels,
                           int num_levels, uint8_t *flags, sdetr_stream_t stream);

/* Coarse-to-fine score modulation (:134-143): out = mem + mem * up * alpha[alpha_index], up = bilinear resize
 * (align_corners=True) of the coarser level's score map (b,Hc*Wc) to (H,W).  mem/out (b,H*W,C) with row
 * strides; alpha is read on the device. */
int sdetr_score_modulate(const float *mem, int64_t mem_batch_stride, const float *coarse_score,
                         int64_t coarse_batch_stride, const float *alpha, int alpha_index, int batch, int H,
                         int W, int Hc, int Wc, int channels, float *out, sdetr_stream_t stream);

/* value rows of padded tokens -> 0 (ms_deform_attn.py:318-319), only masked rows are touched.
 * rows: (b*Nv) rows of `row_floats` contiguous floats at stride row_stride. */
int sdetr_zero_masked_rows(float *rows, int64_t row_stride, int row_floats, const uint8_t *mask,
                           int64_t num_rows, sdetr_stream_t stream);

/* MaskPredictor middle (salience_transformer.py:40-45), in place on z (b,num_rows,channels):
 * z = GELU(z) (exact erf form); then z[b,:,half:] = mean over the num_rows tokens of image b (padded tokens included,
 * like the reference).  Deterministic two-pass reduction; workspace from sdetr_gelu_colmean_workspace. */
size_t sdetr_gelu_colmean_workspace(int batch, int num_rows, int channels, int half);
int sdetr_gelu_colmean(float *z, int batch, int num_rows, int channels, int half, void *workspace,
                       size_t workspace_bytes, sdetr_stream_t stream);

/* mc_score = max_c(class_logits) * fg (:366).  logits (rows, num_classes) with row pitch row_pitch -> out (rows). */
int sdetr_class_max_times_fg(const float *logits, int64_t row_pitch, const float *fg, int64_t rows, int num_classes,
                             float *out, sdetr_stream_t stream);

/* y = LayerNorm(x + r) * gamma + beta (:390-391, :349-350); rows of `channels` (<= 1024, multiple of 4).
 * May run in place (y == x). */
int sdetr_add_layernorm(const float *x, const float *r, const float *gamma, const float *beta, float eps,
                        int64_t rows, int channels, float *y, sdetr_stream_t stream);

/* Front end (SURVEY.md 8(f)-2): per-level NCHW maps -> token layout in one pass (base_transformer.py:21-32,
 * salience_transformer.py:107-113):  feat_tok[b,t,:] = feat_l[b,:,y,x];  lpos_tok = pos_l + level_embeds[l];
 * x_tok = (feat_tok + lpos_tok) * keep[b,t]  (keep = ~padding & proposal-valid, base_transformer.py:100-108).
 * feats_host / pos_host: HOST arrays of num_levels device pointers to (b,C,H_l*W_l) fp32; level_size_host = H_l*W_l. */
int sdetr_flatten_tokens(const float *const *feats_host, const float *const *pos_host, const float *level_embeds,
                         const float *keep, const int32_t *level_size_host, int batch, int channels, int num_levels,
                         float *feat_tok, float *lpos_tok, float *x_tok, sdetr_stream_t stream);

/* Same, with the position embedding already in token layout (b,Nv,C) (sdetr_sine_pos_tokens): only the feature maps are
 * transposed; lpos_tok = pos_tokens + level_embeds[l]. */
int sdetr_flatten_tokens_pos(const float *const *feats_host, const float *pos_tokens, const float *level_embeds,
                             const float *keep, const int32_t *level_size_host, int batch, int channels, int num_levels,
                             float *feat_tok, float *lpos_tok, float *x_tok, sdetr_stream_t stream);
/* testing knob: 1 (default) = levels with a token count % 4 == 0 use the vectorised register-transpose kernel; 0 = all levels
 * through the 32x32 shared-memory tile kernel.  Results are bit-identical. */
int sdetr_flatten_set_vectorized(int enable);

/* Salience supervision targets (training side of the filter; SalienceCriterion.get_mask_single_level with noise_scale 0,
 * models/detectors/salience_detr.py:64-114): target[b,t] = max over the boxes that contain the token's pixel centre
 * ((x+.5) stride_x, (y+.5) stride_y) of 1 - sqrt(dx^2 + dy^2) / 2, and 0 unless one containing box has its largest border
 * distance in (limit_lo[l], limit_hi[l]].  boxes (b,max_boxes,4) xyxy in pixels, 16-byte aligned; num_boxes (b,) int32. */
int sdetr_salience_targets(const float *boxes_xyxy, const int32_t *num_boxes, int max_boxes, int batch, int num_value,
                           int num_levels, const int32_t *level_h_host, const int32_t *level_w_host, const float *stride_y_host,
                           const float *stride_x_host, const float *limit_lo_host, const float *limit_hi_host, float *target,
                           sdetr_stream_t stream);

/* Layout hand-off to / from a convolutional neck (salience_transformer.py:185-192): tokens (b,Nv,C) <-> per-level NCHW
 * maps; maps_host = HOST array of num_levels device pointers to (b,C,H_l*W_l) fp32.  to_maps != 0: tokens -> maps (the
 * reference's split + transpose + contiguous + reshape); to_maps == 0: maps -> tokens (flatten(2).transpose(1,2) + cat). */
int sdetr_token_map_transpose(float *tokens, float *const *maps_host, const int32_t *level_size_host, int batch, int channels,
                              int num_levels, int to_maps, sdetr_stream_t stream);

/* Everything the path derives from the padding masks, in two launches (replaces ~60 ATen launches and makes a fresh-mask
 * batch cheap).  mask (b,Nv) uint8 (1 = padding), levels given by host (H_l, W_l).
 *   valid_token_nums[b,l] = #valid tokens;  focus_token_nums[b,l] = int(float(valid) * level_filter_ratio[l])
 *     (salience_transformer.py:116-119: fp32 multiply, truncation);
 *   valid_ratios[b,l] = (valid W of the first row / W_l, valid H of the first column / H_l)   (base_transformer.py:48-56);
 *   keep[b,t] = 1.0 iff the token is not padded and its proposal centre ((x+.5)/valid_W, (y+.5)/valid_H) and size
 *     0.05 * 2^l lie in (0.01, 0.99)   (base_transformer.py:84-108);
 *   ynorm / xnorm[b,t] = (cumsum of the valid mask along y / x + pos_offset) / (last + pos_eps) * pos_scale, the
 *     normalised coordinates of PositionEmbeddingSine (models/bricks/position_encoding.py:48-56), fp32, same op order. */
int sdetr_mask_plan(const uint8_t *mask, int batch, int num_value, int num_levels, const int32_t *level_h_host,
                    const int32_t *level_w_host, const float *level_filter_ratio_host, float pos_offset, float pos_eps,
                    float pos_scale, float *ynorm, float *xnorm, int32_t *valid_token_nums, int32_t *focus_token_nums,
                    float *valid_ratios, float *keep, sdetr_stream_t stream);
/* pos_tokens[r, :] = [sin/cos(ynorm[r] / dim_ty[j]) (j < F) | sin/cos(xnorm[r] / dim_tx[j])], sin on even j, cos on odd j
 * (position_encoding.py:58-64); rows = b*Nv, F = num_pos_feats (multiple of 4), dim_t* = temperature^(2 (j//2) / F). */
int sdetr_sine_pos_tokens(const float *ynorm, const float *xnorm, const float *dim_ty, const float *dim_tx, int64_t rows,
                          int num_pos_feats, float *pos_tokens, sdetr_stream_t stream);

/* Dense self-attention core of the 300-token pre-attention (salience_transformer.py:372-376; the attention inside
 * nn.MultiheadAttention): out = softmax(Q K^T / sqrt(d)) V per (image, head).  qkv (b,n,3,heads,d): the packed
 * projected queries, keys and values (what sdetr_mha_in_proj writes); out (b,n,heads*d).  head_dim must be 32; K^T, V
 * and the score tile live in shared memory: n up to ~460, larger n returns SDETR_ERR_UNSUPPORTED. */
int sdetr_attention_qkv(const float *qkv, float *out, int batch, int n, int heads, int head_dim, sdetr_stream_t stream);

/* Pre-attention front (salience_transformer.py:368-372 + the packed in-projection of nn.MultiheadAttention):
 * t_out[b,j,:] = tokens[b,index[b,j],:];  x = t + pos[b,index[b,j],:];
 * qkv[b,j,:] = [x Wq^T + bq | x Wk^T + bk | t Wv^T + bv].
 * tokens/pos (b,num_rows,C); index (b,k) int64; w_in_t = in_proj_weight TRANSPOSED, (C,3C) row-major; b_in (3C);
 * t_out (b,k,C); qkv (b,k,3C).  channels must be 256.  fp32 FMA arithmetic. */
int sdetr_mha_in_proj(const float *tokens, const float *pos, const int64_t *index, int batch, int num_rows, int k,
                      int channels, const float *w_in_t, const float *b_in, float *t_out, float *qkv,
                      sdetr_stream_t stream);

/* Pre-attention back (salience_transformer.py:373-379): y = LayerNorm(t + attn Wo^T + bo) with (gamma, beta, eps);
 * dst[b,index[b,j],:] = y[b,j,:] (indices unique per image).  attn, t (b,k,C); w_out_t = out_proj.weight TRANSPOSED
 * (C,C); dst (b,num_rows,C), updated in place.  channels must be 256.
 * Optional (both or neither): pos (b,num_rows,C) and dst_sum (b,num_rows,C) -- the same rows of dst_sum receive
 * y + pos[b,index[b,j],:], keeping a `query + query_pos` buffer (sdetr_token_gather's query_sum) current. */
int sdetr_mha_out_proj_ln_scatter(const float *attn, const float *t, const float *w_out_t, const float *b_out,
                                  const float *gamma, const float *beta, float eps, const int64_t *index, float *dst,
                                  const float *pos, float *dst_sum, int batch, int num_rows, int k, int channels,
                                  sdetr_stream_t stream);

/* Row gather / scatter by per-image index (the top-k tokens of the pre-attention, salience_transformer.py:368-379),
 * indices unique per image; src/dst (b,num_rows,C), index (b,k) int64.
 * t[b,j,:] = src[b,index[b,j],:],  x[b,j,:] = t[b,j,:] + pos[b,index[b,j],:]  (:368-371 in one pass) */
int sdetr_rows_gather_add(const float *src, const float *pos, const int64_t *index, int batch, int num_rows, int k,
                          int channels, float *t, float *x, sdetr_stream_t stream);
/* dst[b,index[b,j],:] = src[b,j,:] */
int sdetr_rows_scatter(float *dst, const int64_t *index, int batch, int num_rows, int k, int channels, const float *src,
                       sdetr_stream_t stream);

/* 3xTF32 operand split for the dense projections (tensor cores with fp32-class accuracy):
 * x (rows, K) with row stride x_row_stride -> out (rows, K/chunk, 3, chunk): per K-chunk [hi | hi | lo]
 * (layout_b = 0, activations) or [hi | lo | hi] (layout_b = 1, weights), hi = tf32(x), lo = tf32(x - hi);
 * relu != 0 applies max(x, 0) first (fuses the FFN activation, salience_transformer.py:348).  A TF32 GEMM over
 * a chunk's 3*chunk columns of both operands yields A_hi.B_hi + A_hi.B_lo + A_lo.B_hi for that chunk; chunks are
 * accumulated by the GEMM epilogue in fp32 (chunk == K: a single GEMM). */
int sdetr_split_tf32(const float *x, int64_t x_row_stride, int64_t rows, int K, int chunk, int layout_b, int relu,
                     float *out, sdetr_stream_t stream);

/* Dense projection on the tensor cores with fp32-class accuracy (hand-written sm_90a wgmma GEMM):
 *   C[M,N] = act(A)[M,K] . W[N,K]^T + bias,  act = ReLU (relu_a = 1, salience_transformer.py:348), exact GELU (relu_a = 2, :23-29) or identity (0).
 * A (M,K) row pitch lda floats; W_hi/W_lo (N,K) contiguous = sdetr_split_tf32_pair(W); bias (N) nullable;
 * C (M,N) row pitch ldc.  K % 32 == 0; A/W 16-byte aligned, lda % 4 == 0.  The activation is split into TF32 pieces
 * inside the kernel (no extra HBM pass); products A_hi.W_hi + A_hi.W_lo + A_lo.W_hi accumulate in fp32 registers.
 * Replaces the cuBLAS path for: value_proj / sampling_offsets|attention_weights / output_proj
 * (models/bricks/ms_deform_attn.py:316,322-328,375), FFN (salience_transformer.py:347-351), class head (:462),
 * MaskPredictor (:16-47), enc_output (base_transformer.py:111). */
/* Same contract with the RAW weight W (N,K): the kernel splits both operands itself (32 KB instead of 48 KB of TMA
 * traffic per k-block), with the arithmetic of sdetr_split_tf32_pair: results are bit-identical to the pre-split form. */
int sdetr_gemm_3xtf32_raw(const float *A, int64_t lda, const float *W, const float *bias, float *C, int64_t ldc, int M,
                          int N, int K, int act, sdetr_stream_t stream);
int sdetr_split_tf32_pair(const float *w, int64_t count, float *w_hi, float *w_lo, sdetr_stream_t stream);
int sdetr_gemm_3xtf32(const float *A, int64_t lda, const float *W_hi, const float *W_lo, const float *bias, float *C,
                      int64_t ldc, int M, int N, int K, int relu_a, sdetr_stream_t stream);
/* Same contract and kernel as sdetr_gemm_3xtf32 (pre-split weight): one CTA per SM walks the output tiles, the weight
 * halves arrive as two TMA tiles per stage and only the activation is converted in the kernel. */
int sdetr_gemm_3xtf32_pre(const float *A, int64_t lda, const float *W_hi, const float *W_lo, const float *bias, float *C,
                          int64_t ldc, int M, int N, int K, int act, sdetr_stream_t stream);

/* ---- "3xFP16": the same error-compensated product on wgmma .f16 ---------------------------------------------------------
 * An fp16 significand is as wide as a TF32 one (11 bits), so  A_hi.W_hi + A_hi.W_lo + A_lo.W_hi  with
 * hi = fp16(x), lo = fp16(x - hi) keeps the 22 significand bits per operand of 3xTF32 at twice the MMA rate and half the
 * weight bytes.  Exponent range is restored by exact power-of-two scalings: the kernel multiplies the activation by 16
 * before the split (full accuracy for 2^-7 <= |x| < 4094, absolute error floor 2^-29 below, inf/NaN above), the caller
 * scales the weight by `scale` = 2^s with max|scale * W| in [2^13, 2^14) when splitting, and the epilogue multiplies the
 * fp32 accumulator by 2^-(4+s) before the bias.  Replaces the same reference projections as sdetr_gemm_3xtf32
 * (models/bricks/ms_deform_attn.py:316,322-328,375; salience_transformer.py:347-351,462,16-47; base_transformer.py:111).
 * W (N,K) fp32 contiguous -> W_hi, W_lo (N,K) fp16 (2-byte elements, 16-byte aligned). */
int sdetr_split_f16_pair(const float *W, int64_t count, float scale, void *W_hi, void *W_lo, sdetr_stream_t stream);
/* C[M,N] = act(A)[M,K] . W^T + bias, W given as the pair above and the `w_scale` it was split with; K % 64 == 0;
 * A (M,K) fp32 with row pitch lda (floats, multiple of 4); act: 0 none, 1 ReLU, 2 exact GELU applied to A on load;
 * C row pitch ldc (TMA stores when ldc % 4 == 0). */
int sdetr_gemm_f16x3_pre(const float *A, int64_t lda, const void *W_hi, const void *W_lo, float w_scale, const float *bias,
                         float *C, int64_t ldc, int M, int N, int K, int act, sdetr_stream_t stream);
/* The encoder's class-score head and its per-row max in one launch: out[row] = max_c (A . W^T + bias)[row, c] * row_scale[row],
 * with the product of sdetr_gemm_f16x3_pre (W split by sdetr_split_f16_pair with scale w_scale; N <= 128; K % 64 == 0) and
 * the max of sdetr_class_max_times_fg (a NaN value propagates): bit for bit that pair, without the M x N logits. */
int sdetr_gemm_f16x3_rowmax(const float *A, int64_t lda, const void *W_hi, const void *W_lo, float w_scale, const float *bias,
                            const float *row_scale, float *out, int M, int N, int K, sdetr_stream_t stream);
/* An encoder layer's output projection, residual and norm1 in one launch: q = LayerNorm(q + A . W^T + bias) * gamma + beta,
 * A (M,256) with row pitch lda, W (256,256) split by sdetr_split_f16_pair with scale w_scale, q (M,256) contiguous and
 * rewritten in place; bias may be NULL.  Bit for bit sdetr_gemm_f16x3_pre followed by sdetr_add_layernorm(q, C, ..., q). */
int sdetr_gemm_f16x3_add_layernorm(const float *A, int64_t lda, const void *W_hi, const void *W_lo, float w_scale,
                                   const float *bias, const float *gamma, const float *beta, float eps, float *q, int M,
                                   sdetr_stream_t stream);
/* The same product with BOTH scales as device scalars (powers of two; sdetr_pow2_scale): the kernel multiplies A by *a_scale_dev
 * instead of the fixed 16 (activations of unknown magnitude: gradients), the weight pair was split with *w_scale_dev
 * (sdetr_split_f16_pair_dev: weights that change every training step, no host read of max|W|), and the epilogue divides both out.
 * No host synchronisation anywhere.  No fused input activation. */
int sdetr_gemm_f16x3_scaled(const float *A, int64_t lda, const float *a_scale_dev, const void *W_hi, const void *W_lo,
                            const float *w_scale_dev, const float *bias, float *C, int64_t ldc, int M, int N, int K,
                            sdetr_stream_t stream);
int sdetr_split_f16_pair_dev(const float *W, int64_t count, const float *scale_dev, void *W_hi, void *W_lo, sdetr_stream_t stream);
/* *scale = 2^s with max|x| * 2^s in [2^(target_log2 - 1), 2^target_log2) (1 for an all-zero x); one launch, deterministic.
 * state: 8 bytes of device memory, zero before the first call (the kernel leaves them zero). */
int sdetr_pow2_scale(const float *x, int64_t count, int target_log2, void *state, float *scale, sdetr_stream_t stream);

/* ---- MaskPredictor of one small feature level in two launches ---------------------------------------------------------------
 * Replaces, for a level of few token rows, score modulation + MaskPredictor (models/bricks/salience_transformer.py:16-47, :134-143):
 * x = m + m * bilinear(coarse_score, align_corners=True) * alpha[alpha_index] (coarse_score NULL: x = m), LayerNorm, Linear(C,C),
 * GELU, token mean of the upper half of the channels (over the H*W tokens of each image), Linear(C,C/2), GELU, Linear(C/2,C/4),
 * GELU, Linear(C/4,1).  channels must be 256.  fp32 FMA arithmetic.
 * mem: first token row of the level in image 0, rows of `channels` floats, images mem_batch_stride floats apart;
 * weights TRANSPOSED to (in, out) row-major: w1_t (C,C), w2a_t (C,C/2), w2b_t (C/2,C/4); w2c (C/4);
 * out: the level's raw scores, H*W per image, images out_batch_stride floats apart;
 * workspace: sdetr_mask_predictor_level_workspace_floats(batch, H, W) floats. */
int64_t sdetr_mask_predictor_level_workspace_floats(int batch, int H, int W);
int sdetr_mask_predictor_level(const float *mem, int64_t mem_batch_stride, int batch, int H, int W, int channels,
                               const float *coarse_score, int64_t coarse_batch_stride, int Hc, int Wc, const float *alpha,
                               int alpha_index, const float *ln_gamma, const float *ln_beta, float eps, const float *w1_t,
                               const float *b1, const float *w2a_t, const float *b2a, const float *w2b_t, const float *b2b,
                               const float *w2c, const float *b2c, float *workspace, int64_t workspace_floats, float *out,
                               int64_t out_batch_stride, sdetr_stream_t stream);

/* ---- encoder FFN: y = LayerNorm(x + linear2(ReLU(linear1(x)))) ------------------------------------------------------------
 * Replaces `forward_ffn` + `norm2` of the encoder layer (models/bricks/salience_transformer.py:347-351, :391) for embed_dim 256:
 * one persistent kernel computes linear1, ReLU and linear2 per 64-row panel with the hidden activations kept in shared memory,
 * and adds the residual and normalises in its epilogue; panels whose hidden chunks are spread over several CTAs are summed
 * (in a fixed order: bit-reproducible) and normalised by a second, row-wise launch.
 * Same 3xFP16 arithmetic and value domain as sdetr_gemm_f16x3_pre (both weights given as sdetr_split_f16_pair pairs with
 * their scales; W1 (hidden,256), W2 (256,hidden); hidden % 128 == 0).
 * x (M,256) fp32 with row pitch ldx (floats); y (M,256) contiguous, may alias x when ldx == 256;
 * gamma == beta == NULL: y = linear2(ReLU(linear1(x))) without residual / LayerNorm.  b2 == NULL: linear2 without bias.
 * workspace: sdetr_ffn_fused_workspace_floats(M, hidden) = M * (hidden + 256) floats, an upper bound (per-CTA partial sums of
 * shared panels; the grid is narrowed to what it holds). */
int64_t sdetr_ffn_fused_workspace_floats(int M, int hidden);
int sdetr_ffn_fused_layernorm(const float *x, int64_t ldx, const void *W1_hi, const void *W1_lo, float w1_scale, const float *b1,
                              const void *W2_hi, const void *W2_lo, float w2_scale, const float *b2, const float *gamma,
                              const float *beta, float eps, int M, int hidden, float *workspace, int64_t workspace_floats, float *y,
                              sdetr_stream_t stream);

/* ---- RepVGG-PluX neck in token layout (models/necks/repnet.py:125-245; RepVGGPluXNetwork.forward_tokens) ------------------
 * Operands are token rows: pixel (py, px) of image n, channel c at base + n * pitch + (py * W + px) * ld + c (floats), so a
 * level slice of a (b, Nv, C) tensor is an operand as it is.
 *
 * Convolution y = act(conv(x, W) + bias + z), kernel ksize x ksize (1 or 3), padding ksize / 2, stride 1 or 2, `groups` groups;
 * act 0 none, 1 ReLU (NaN propagates, as torch.relu), 3 SiLU.  Implicit GEMM on wgmma with the 3xFP16 arithmetic of
 * sdetr_gemm_f16x3_scaled: x is multiplied by the power-of-two device scalar *a_scale_dev (sdetr_pow2_scale with target 12)
 * before its hi / lo split, W (Cout, ksize, ksize, Cin / groups) row-major was split with *w_scale_dev
 * (sdetr_conv2d_f16x3_split_weight or sdetr_split_f16_pair_dev), the epilogue divides both out.  Cin / groups and Cout / groups
 * multiples of 64 (else SDETR_ERR_UNSUPPORTED); x, x_pitch, ldx 16-byte aligned; y, y_pitch, ldy 8-byte aligned;
 * Ho = (H + 2 (ksize / 2) - ksize) / stride + 1, likewise Wo.  bias may be NULL.  The residual operand z (token rows, Cout
 * wide; NULL: none) is added before the activation; z, z_pitch, ldz 8-byte aligned; z may alias y (each element is read before
 * it is written, by the same thread).  A Bottleneck's conv3 -> bn3 -> += identity -> ReLU is one call. */
int sdetr_conv2d_f16x3(const float *x, int64_t x_pitch, int64_t ldx, int batch, int H, int W, int Cin, const float *a_scale_dev,
                       const void *W_hi, const void *W_lo, const float *w_scale_dev, const float *bias, const float *z,
                       int64_t z_pitch, int64_t ldz, int Cout, int groups, int ksize, int stride, int act, float *y,
                       int64_t y_pitch, int64_t ldy, sdetr_stream_t stream);
/* Context gate of a RepVggPluXBlock (SqueezeAndExcitation, models/bricks/basic.py:29-54, plus the block's residual), per image
 * of HW pixels: p = softmax over the pixels of (y . w_mask + *b_mask); ctx = sum p y; gate = sigmoid(W2 ReLU(W1 ctx)) with
 * w1 (R, C), w2 (C, R) row-major; out = gate * y + x (+ z when z is not NULL).  Three launches; every reduction is summed in a
 * fixed order (bit-reproducible).  C % 4 == 0; all row operands 16-byte aligned; out may alias x or z.
 * workspace: sdetr_context_gate_workspace_floats(batch, HW, C) floats, 16-byte aligned. */
int64_t sdetr_context_gate_workspace_floats(int batch, int HW, int C);
int sdetr_context_gate(const float *y, int64_t y_pitch, int64_t ldy, const float *x, int64_t x_pitch, int64_t ldx, const float *z,
                       int64_t z_pitch, int64_t ldz, int batch, int HW, int C, const float *w_mask, const float *b_mask,
                       const float *w1, const float *w2, int R, float *workspace, int64_t workspace_floats, float *out,
                       int64_t out_pitch, int64_t ldo, sdetr_stream_t stream);
/* dst[:, :, 0:C] = nearest-upsampled hi (Hi, Wi) -> (Ho, Wo) with torch's index rule src = min(floor(dst * (float)in / out),
 * in - 1); dst[:, :, C:2C] = lo (Ho, Wo).  C % 4 == 0; all row operands 16-byte aligned. */
int sdetr_upsample_nearest_concat(const float *hi, int64_t hi_pitch, int64_t ldh, int Hi, int Wi, const float *lo, int64_t lo_pitch,
                                  int64_t ldl, int Ho, int Wo, int batch, int C, float *dst, int64_t dst_pitch, int64_t ldd,
                                  sdetr_stream_t stream);
/* Training.  One pass over a convolution weight w (Cout, Cin / groups, k, k) in PyTorch's layout with the device scale
 * *scale_dev (sdetr_pow2_scale, target 14): the fp16 pair (fwd_hi, fwd_lo) in sdetr_conv2d_f16x3's (Cout, k, k, Cin / groups)
 * layout and, unless dgrad_hi == dgrad_lo == NULL, the pair of the input-gradient weights W' (Cin, k, k, Cout / groups),
 * flipped in both spatial axes and transposed per group: W'[g Cin_g + ci, ky, kx, co] = W[g Cout_g + co, ci, k - 1 - ky,
 * k - 1 - kx].  The arithmetic of sdetr_split_f16_pair_dev. */
int sdetr_conv2d_f16x3_split_weight(const float *w, int Cout, int Cin, int groups, int ksize, const float *scale_dev, void *fwd_hi,
                                    void *fwd_lo, void *dgrad_hi, void *dgrad_lo, sdetr_stream_t stream);
/* Weight gradient of y = conv(x, W) (the family of sdetr_conv2d_f16x3; x: H x W, Cin channels; dy: Ho x Wo, Cout channels):
 * dw[co, ci, ky, kx] = sum over output pixels of dy[pixel, co] x[shifted pixel, g Cin_g + ci], written fp32 in PyTorch's
 * (Cout, Cin / groups, k, k) layout.  3xFP16 on wgmma: dy and x are multiplied by their power-of-two device scalars
 * (sdetr_pow2_scale, target 12) before the hi / lo split.  The pixel range is split over CTAs by a rule of the shape alone and
 * the partial sums are added in split order: bit-reproducible.  Each output row co is multiplied by cout_scale[co] (Cout
 * floats; NULL: none) in the split sum's write, one fp32 product of the same sum: the gradient of a weight W whose forward
 * ran W * s (a folded FrozenBatchNorm scale s) is this call with s.  Two launches.  dy, x, their pitches and row strides
 * 16-byte aligned; workspace: sdetr_conv2d_f16x3_wgrad_workspace_floats(batch, Ho, Wo, Cin, Cout, groups, ksize) floats,
 * 16-byte aligned (0 for an unsupported shape). */
int64_t sdetr_conv2d_f16x3_wgrad_workspace_floats(int batch, int Ho, int Wo, int Cin, int Cout, int groups, int ksize);
int sdetr_conv2d_f16x3_wgrad(const float *dy, int64_t dy_pitch, int64_t lddy, const float *dy_scale_dev, const float *x,
                             int64_t x_pitch, int64_t ldx, const float *x_scale_dev, int batch, int H, int W, int Cin, int Cout,
                             int groups, int ksize, int stride, const float *cout_scale, float *workspace, int64_t workspace_floats,
                             float *dw, sdetr_stream_t stream);
/* Input gradient of y = conv(x, W) with a fused epilogue: dx = (conv^T(dy, W) + z), then 0 where m <= 0.  dy: Hy x Wy with Cin
 * channels (the forward's Cout); dx: H x W with Cout channels (the forward's Cin); Hy, Wy must be the forward's output size of
 * H, W; W_hi / W_lo: the input-gradient pair W' of sdetr_conv2d_f16x3_split_weight.  Stride 1 is sdetr_conv2d_f16x3 on dy with
 * W'.  Stride 2 is the transposed convolution with W': output pixel (iy, ix) with tap (ky, kx) reads dY[(iy - pad + ky) / 2,
 * (ix - pad + kx) / 2] when both are even and in range, zero otherwise.  z (token rows, Cout wide; NULL: none) may alias dx
 * (read before written, by the same thread); m (NULL: none) is the ReLU mask source of torch's threshold_backward(grad, m, 0):
 * a NaN in m lets the value through, a NaN value stays NaN; m must not alias dx.  No bias, no activation.  Operand rules of
 * sdetr_conv2d_f16x3; z, m, their pitches and row strides 8-byte aligned. */
int sdetr_conv2d_f16x3_dgrad(const float *dy, int64_t dy_pitch, int64_t lddy, int batch, int Hy, int Wy, int Cin,
                             const float *a_scale_dev, const void *W_hi, const void *W_lo, const float *w_scale_dev, const float *z,
                             int64_t z_pitch, int64_t ldz, const float *m, int64_t m_pitch, int64_t ldm, int Cout, int groups,
                             int ksize, int stride, int H, int W, float *dx, int64_t dx_pitch, int64_t lddx, sdetr_stream_t stream);
/* Gradient of the hi half of sdetr_upsample_nearest_concat: d_hi (Hi x Wi) = for each source pixel, the sum of g[:, :, 0:C] over
 * the destination pixels (Ho x Wo) that read it, rows then columns in order (no atomics: deterministic).  The lo half's gradient
 * is g[:, :, C:2C] itself.  C % 4 == 0; all row operands 16-byte aligned. */
int sdetr_upsample_nearest_concat_backward(const float *g, int64_t g_pitch, int64_t ldg, int Ho, int Wo, int Hi, int Wi, int batch,
                                           int C, float *d_hi, int64_t d_pitch, int64_t ldd, sdetr_stream_t stream);

/* ---- ChannelMapper in token layout (models/necks/channel_mapper.py:8-80; ChannelMapper.forward_tokens) ----------------------
 * GroupNorm of every level of a token buffer (nn.GroupNorm per level, models/bricks/misc.py:97-98): image n, token t, channel c
 * at x + n * pitch + t * C + c (floats); level l = the level_size_host[l] tokens after the previous levels'.  Statistics per
 * (image, level, group of C / num_groups consecutive channels) over all H*W*C/G elements of the level (padding pixels included,
 * as nn.GroupNorm): per-tile Welford (count, mean, M2) partials merged with Chan's formula in a fixed order (no atomics; the
 * result is bit-identical from run to run and does not depend on the grid); biased variance, rstd = rsqrt(var + eps);
 * y = (x - mean) * rstd * gamma[l] + beta[l].  gamma / beta: (num_levels, C) row-major.  y may alias x (same pitch and rows).
 * C % 4 == 0, C <= 4096, C % num_groups == 0 (else SDETR_ERR_UNSUPPORTED); x, y, gamma, beta, pitch 16-byte aligned.
 * Three launches for all levels.  workspace: sdetr_group_norm_tokens_workspace_floats(...) floats, 8-byte aligned. */
int64_t sdetr_group_norm_tokens_workspace_floats(int batch, int channels, int num_groups, int num_levels, const int32_t *level_size_host);
int sdetr_group_norm_tokens(const float *x, float *y, int64_t pitch, int batch, int channels, int num_levels,
                            const int32_t *level_size_host, const float *gamma, const float *beta, int num_groups, float eps,
                            float *workspace, int64_t workspace_floats, sdetr_stream_t stream);
/* The transformer's front end for features that are already tokens (salience_transformer.py:107-113 without the flatten):
 * lpos = pos + level_embeds[l];  x = (feat + lpos) * keep[b,t]  -- the operations of sdetr_flatten_tokens[_pos] in the same
 * order, so lpos and x are bit-identical to theirs for the same values.  feat, pos, lpos, x (b,Nv,C) contiguous, 16-byte
 * aligned; keep (b,Nv); level_embeds (L,C); lpos may alias pos.  C % 4 == 0.  One launch. */
int sdetr_token_lpos_keep(const float *feat, const float *pos, const float *level_embeds, const float *keep,
                          const int32_t *level_size_host, int batch, int channels, int num_levels, float *lpos, float *x,
                          sdetr_stream_t stream);

/* ---- Detection loss: HungarianMatcher + HybridSetCriterion.calculate_loss (models/matcher/hungarian_matcher.py:7-91,
 * models/bricks/set_criterion.py:14-212, models/bricks/losses.py:15-21) ---------------------------------------------------
 * One problem is one (output, image) pair.  Its descriptor names the output's rows in place: query q's K class logits at
 * logits + q * logit_stride (classes contiguous) and its cxcywh box at boxes + q * box_stride (4 contiguous floats), so slices
 * of a stacked (layers, b, Q, K) tensor need no copy.  gt_boxes (num_gt, 4) cxcywh and gt_labels (num_gt) int64 are
 * contiguous; gt_labels NULL means every label is 0 (two_stage_binary_cls).  src / tgt (query, gt) index pairs are int64.
 * The table (at most SDETR_SET_MAX_PROBLEMS problems) travels to the device as a kernel parameter: no copy, no sync. */
#define SDETR_SET_MAX_PROBLEMS 128
#define SDETR_SET_MAX_QUERIES 4096
typedef struct sdetr_set_problem {
    const float *logits;
    const float *boxes;
    const float *gt_boxes;
    const int64_t *gt_labels;
    int64_t *src;       /* sdetr_set_match: written, num_gt entries, ascending queries; loss: read, num_pairs entries */
    int64_t *tgt;
    float *grad_logits; /* sdetr_set_loss_backward: (Q, K) contiguous, fully written */
    float *grad_boxes;  /* sdetr_set_loss_backward: (Q, 4) contiguous, fully written (0 on unmatched rows) */
    int64_t logit_stride;
    int64_t box_stride;
    int32_t num_queries; /* Q >= 1 */
    int32_t num_gt;
    int32_t num_pairs;   /* loss only */
    int32_t output;      /* loss only: row of the (num_outputs, 3) loss tensor this problem adds to */
} sdetr_set_problem;
/* Exact minimum-cost assignment of every problem's gts (rows) to its queries (columns), one CTA per problem, one launch:
 * cost = cost_bbox * L1(pred, gt) + cost_class * focal(pos - neg at the gt label, +1e-6 inside the logs) - cost_giou * GIoU in
 * fp32; shortest augmenting path with fp64 duals, ties to the lowest column.  Writes src (ascending query indices) / tgt of each
 * problem (num_gt pairs; nothing when num_gt == 0) and status[i] = 0.  A non-finite cost, or a gt label outside
 * [0, num_classes), sets status[i] = 1 and writes the pairs (k, k) instead (scipy / the reference's indexing raise there).  Q <= SDETR_SET_MAX_QUERIES and num_gt <= Q (else
 * SDETR_ERR_UNSUPPORTED).  workspace: sdetr_set_match_workspace_floats(...) floats (the cost matrices). */
int64_t sdetr_set_match_workspace_floats(const sdetr_set_problem *problems_host, int num_problems);
int sdetr_set_match(const sdetr_set_problem *problems_host, int num_problems, int num_classes, float cost_class, float cost_bbox,
                    float cost_giou, float alpha, float gamma, int32_t *status, float *workspace, int64_t workspace_floats,
                    sdetr_stream_t stream);
/* The solver of sdetr_set_match on given costs: problem i's (num_gt, num_queries) row-major fp32 matrix (rows gts, columns
 * queries) starts at cost + sum over the earlier problems of num_gt * num_queries.  Only num_queries, num_gt, src and tgt of
 * the descriptors are read.  Same outputs, status and limits as sdetr_set_match.  One launch. */
int sdetr_set_assign(const sdetr_set_problem *problems_host, int num_problems, const float *cost, int64_t cost_floats,
                     int32_t *status, sdetr_stream_t stream);
/* loss[o] = (varifocal class loss, L1, sum of 1 - GIoU) of the matched pairs of every problem with output == o, divided by
 * num_boxes (*num_boxes_dev when not NULL, else num_boxes_host).  Class target t = onehot * IoU(pair) and weight
 * w = (1 - alpha) sigmoid(x)^gamma (1 - onehot) + t, both detached; the loss sums w * BCEwithlogits(x, t) over all Q x K logits.
 * Sums run in a fixed order without float atomics (bit-reproducible).  A problem with status[i] != 0 (status may be NULL), a
 * pair index out of range or a gt label outside [0, num_classes) makes its output's losses NaN.  Two launches; workspace: sdetr_set_loss_workspace_floats(...). */
int64_t sdetr_set_loss_workspace_floats(const sdetr_set_problem *problems_host, int num_problems);
int sdetr_set_loss_forward(const sdetr_set_problem *problems_host, int num_problems, int num_outputs, int num_classes, float alpha,
                           float gamma, const int32_t *status, float num_boxes_host, const float *num_boxes_dev, float *workspace,
                           int64_t workspace_floats, float *loss, sdetr_stream_t stream);
/* Gradients of sum(grad_loss * loss) w.r.t. every problem's logits and boxes, into grad_logits / grad_boxes: w (sigmoid(x) - t)
 * per logit; sign(pred - gt) (0 at 0) and the GIoU gradient with torch autograd's conventions (max / min ties split half and
 * half, clamp(min=0) passes where its input is >= 0) per matched box.  grad_loss (num_outputs, 3) contiguous.  One launch. */
int sdetr_set_loss_backward(const sdetr_set_problem *problems_host, int num_problems, int num_outputs, int num_classes, float alpha,
                            float gamma, const int32_t *status, float num_boxes_host, const float *num_boxes_dev,
                            const float *grad_loss, sdetr_stream_t stream);

/* ---- Contrastive denoising queries: GenerateCDNQueries.forward after its random draws (models/bricks/denoising.py:178-329,
 * generate_query_masks :64-76) and the denoising-loss indices of DNDETRDetector.compute_dn_loss
 * (models/detectors/base_detector.py:205-218) ---------------------------------------------------------------------------------
 * Image i has num_gt gts: gt_labels (num_gt) int64 and gt_boxes (num_gt, 4) cxcywh fp32, both contiguous.  The table (at most
 * SDETR_CDN_MAX_IMAGES images) travels to the device as a kernel parameter: no copy, no sync. */
#define SDETR_CDN_MAX_IMAGES 128
typedef struct sdetr_cdn_image {
    const int64_t *gt_labels;
    const float *gt_boxes;
    int32_t num_gt;
    int32_t reserved;
} sdetr_cdn_image;
/* With m = max_gt (the largest num_gt), G = groups, S = the sum of the num_gt and D = 2 G m, the reference's draws over its
 * repeated gt list of n = 2 G S entries (entry r S + (gts of the images before i) + t is copy r < 2G of image i's gt t):
 *   label_rand (n) fp32 and label_randint (n) int64: the label draws, both NULL when label_noise_prob * 0.5 == 0;
 *   box_randint (n, 4) fp32 in {0, 1} and box_rand (n, 4) fp32: the box draws, both NULL when box_noise_scale == 0.
 * Copy r of gt t lands in slot r m + t of its image; copy 2g is the positive and 2g + 1 the negative of group g.  Writes
 *   label_queries (b, D, C) = label_encoder.weight row of the noised label where(label_rand < label_threshold, label_randint,
 *     label), NaN where that label is outside [0, num_classes) (an IndexError in the reference), zeros in padding slots;
 *   box_queries (b, D, 4) = inverse_sigmoid of the noised box (diff = wh / 2 for both corners, sign = randint * 2 - 1, +1 on
 *     the negative copies, xyxy + (part * diff) * box_noise_scale, clamp(0, 1), back to cxcywh), zeros in padding slots;
 *     every operation rounded separately, as the reference's chain of torch kernels;
 *   noised_labels (b, D) int32: the label of each slot, -1 in padding slots and where the label is out of range;
 *   attn_mask (T, T) bytes (torch.bool), T = D + num_queries: generate_query_masks(2m);
 *   status (b) int32: 1 where one of the image's noised labels is outside [0, num_classes), else 0.
 * weight_rows / weight_cols: the shape of `weight` (label_encoder.weight), must be (num_classes, embed_dim).  One launch. */
int sdetr_cdn_queries(const sdetr_cdn_image *images_host, int num_images, const float *label_rand, const int64_t *label_randint,
                      const float *box_randint, const float *box_rand, float label_threshold, float box_noise_scale,
                      const float *weight, int num_classes, int embed_dim, int weight_rows, int weight_cols, int num_queries,
                      int groups, int max_gt, float *label_queries, float *box_queries, int32_t *noised_labels, uint8_t *attn_mask,
                      int32_t *status, sdetr_stream_t stream);
/* grad_weight (num_classes, embed_dim), fully written: row k = the sum over the slots s < num_slots with noised_labels[s] == k,
 * in ascending s, of grad_label_queries[s, :] ((num_slots, embed_dim) contiguous).  No atomics: bit-reproducible.  One launch. */
int sdetr_cdn_queries_backward(const float *grad_label_queries, const int32_t *noised_labels, int64_t num_slots, int num_classes,
                               int embed_dim, float *grad_weight, sdetr_stream_t stream);
/* indices (2, P) int64, P = groups * sum of num_gt_host: image after image, the pairs (g * max_gt + t, t) for g < groups,
 * t < num_gt_host[i] (g outer): row 0 the query, row 1 the gt.  max_gt: the reference's max_gt_num_per_image (2 m for CDN).
 * One launch (none when P == 0). */
int sdetr_cdn_loss_indices(const int32_t *num_gt_host, int num_images, int groups, int max_gt, int64_t *indices,
                           sdetr_stream_t stream);

/* ---- Detection post-processing: PostProcess.forward (models/bricks/post_process.py:21-74) ------------------------------------
 * pred_logits (b, Q, K) fp32: element (i, q, c) at i * logits_batch_stride + q * logits_query_stride + c (a query slice such as
 * dn_post_process's outputs_class[:, :, pad:, :] needs no copy); pred_boxes (b, Q, 4) cxcywh fp32 likewise with unit coordinate
 * stride; target_sizes (b, 2) contiguous (h, w) of dtype sizes_dtype (SDETR_SIZES_*).  Per image, in one CTA:
 *   scores (b, k) fp32: the k largest p = sigmoid(logit) (bit-identical to torch.sigmoid on CUDA) over the Q * K flat indices,
 *     ordered by p descending, ties by smaller flat index, NaN first (= torch.sort(p, descending=True, stable=True)[:k]);
 *   labels (b, k) int64: flat index % K;  boxes (b, k, 4) fp32: the box of query flat index / K as
 *     (cx - 0.5 w, cy - 0.5 h, cx + 0.5 w, cy + 0.5 h) * (img_w, img_h, img_w, img_h), every operation rounded separately.
 * A filter is on when its threshold is > 0.  Then entry j is kept iff (confidence off or score > confidence_score) and (NMS off
 * or no kept entry ranked before j has IoU > iou_threshold with it: greedy NMS over all k boxes in this order, torchvision's
 * IoU); the kept entries are compacted to the front of each image's row in order and count (b) int32 holds how many.  Rows
 * past count are left unwritten.  With both filters off count may be NULL (else it receives k).
 * 1 <= k <= min(Q * K, SDETR_POSTPROCESS_MAX_K) (a larger k: SDETR_ERR_UNSUPPORTED), Q * K < 2^31.  workspace:
 * sdetr_postprocess_workspace(b, Q, K) bytes.  One launch, no synchronisation. */
#define SDETR_POSTPROCESS_MAX_K 4096
enum { SDETR_SIZES_INT64 = 0, SDETR_SIZES_INT32 = 1, SDETR_SIZES_FLOAT32 = 2 };
size_t sdetr_postprocess_workspace(int batch, int num_queries, int num_classes);
int sdetr_postprocess(const float *pred_logits, int64_t logits_batch_stride, int64_t logits_query_stride, const float *pred_boxes,
                      int64_t boxes_batch_stride, int64_t boxes_query_stride, const void *target_sizes, int sizes_dtype, int batch,
                      int num_queries, int num_classes, int k, float confidence_score, float iou_threshold, float *scores,
                      int64_t *labels, float *boxes, int32_t *count, void *workspace, size_t workspace_bytes,
                      sdetr_stream_t stream);
/* ---- ResNet backbone in token layout (models/backbones/resnet.py; ResNetBackbone.forward_tokens) ---------------------------
 * The stem: y = ReLU(conv(x, W) + bias), conv 7x7, stride 2, padding 3, 3 -> 64 channels.  x: the (batch, 3, H, W) NCHW
 * contiguous fp32 image batch; weight (147, 64) = W[co, c, ky, kx] at row (c * 7 + ky) * 7 + kx, column co (the folded
 * FrozenBatchNorm scale already in it); bias (64); y: (batch, Ho * Wo, 64) contiguous token rows, Ho = (H + 6 - 7) / 2 + 1,
 * likewise Wo.  fp32 FMAs, taps summed in (c, ky, kx) order; NaN propagates through the ReLU.  weight, bias, y 16-byte
 * aligned.  One launch. */
int sdetr_resnet_stem(const float *x, int batch, int H, int W, const float *weight, const float *bias, float *y,
                      sdetr_stream_t stream);
/* 3x3, stride 2, padding 1 max-pool on token rows (H x W, C channels) -> (Ho x Wo) with Ho = (H + 2 - 3) / 2 + 1, likewise Wo
 * (torch's max_pool2d, ceil_mode off).  Padding acts as -inf; a NaN in a window gives NaN.  C % 4 == 0; operands, pitches and
 * row strides 16-byte aligned.  One launch. */
/* w (Cout, per_cout) fp32 with a FrozenBatchNorm folded in: s = weight * rsqrt(running_var + eps), w_folded = w * s, and (each
 * optional) scale = s, bias = bias - running_mean * s, per output channel.  Computed in float64 with every operation rounded on
 * its own, then rounded to fp32: the values of the same fold in float64 torch, with no host read.  One launch. */
int sdetr_frozen_bn_fold(const float *w, int Cout, int64_t per_cout, const float *bn_weight, const float *bn_bias,
                         const float *running_mean, const float *running_var, double eps, float *w_folded, float *scale,
                         float *bias, sdetr_stream_t stream);
int sdetr_maxpool3x3s2_tokens(const float *x, int64_t x_pitch, int64_t ldx, int batch, int H, int W, int C, float *y,
                              int64_t y_pitch, int64_t ldy, sdetr_stream_t stream);
/* The projection GEMM of sdetr_gemm_f16x3_scaled (both scales device scalars, no host synchronisation) with the CNBlock
 * additions: C = z + s * (act(A) . W^T + bias), act applied to A as it loads (0 none, 1 ReLU, 2 exact GELU), s = col_scale (N)
 * per output column or NULL (none), z = Z (M rows, pitch ldz) or NULL (none).  Z may alias C: every element of z is read by
 * the thread that writes the same element of C, before it writes it.  |GELU(x)| <= |x|, so a_scale_dev taken over A
 * (sdetr_pow2_scale, target 12) also bounds the activated values.  K % 64 == 0; A, W_hi, W_lo 16-byte aligned, lda % 4 == 0.
 * With act 0, col_scale and Z NULL it writes the bits of sdetr_gemm_f16x3_scaled.  One launch. */
int sdetr_gemm_f16x3_ex(const float *A, int64_t lda, const float *a_scale_dev, const void *W_hi, const void *W_lo,
                        const float *w_scale_dev, const float *bias, const float *col_scale, const float *Z, int64_t ldz, float *C,
                        int64_t ldc, int M, int N, int K, int act, sdetr_stream_t stream);
/* ---- ConvNeXt backbone in token layout (models/backbones/convnext.py; ConvNeXtBackbone.forward_tokens) ----------------------
 * C % 64 == 0 and C <= 1536 for all three; token rows (batch, H * W, C) contiguous; LayerNorms over C with eps, weight and
 * bias (C); two-pass mean / variance per row in fp32, a NaN in a row's inputs gives a NaN row.  Operands 16-byte aligned.
 * The stem: y = LayerNorm(conv(x, W) + bias), conv 4x4, stride 4, no padding, 3 -> C.  x: (batch, 3, H, W) NCHW contiguous
 * fp32; weight (48, C) = W[co, c, ky, kx] at row (c * 4 + ky) * 4 + kx, column co; y: (batch, (H / 4) * (W / 4), C) (torch's
 * floor: trailing rows / columns are dropped).  fp32 FMAs, taps in (c, ky, kx) order, then the bias.  One launch. */
int sdetr_convnext_stem(const float *x, int batch, int H, int W, int C, const float *weight, const float *bias,
                        const float *ln_weight, const float *ln_bias, float eps, float *y, sdetr_stream_t stream);
/* y = LayerNorm(dwconv(x) + bias): depthwise 7x7, padding 3 (zeros), weight (49, C) = W[c, 0, ky, kx] at row ky * 7 + kx.  y is
 * (batch, H * W, C) and must not alias x.  One launch. */
int sdetr_dwconv7x7_layernorm_tokens(const float *x, int batch, int H, int W, int C, const float *weight, const float *bias,
                                     const float *ln_weight, const float *ln_bias, float eps, float *y, sdetr_stream_t stream);
/* LayerNorm of token rows written space-to-depth: y (batch, (H / 2) * (W / 2), 4 C), row (oy, ox) holding LayerNorm(x[2 oy + dy,
 * 2 ox + dx]) at columns (2 dy + dx) * C + c; an odd last row / column is dropped.  A 2x2 / stride-2 convolution is then one
 * GEMM with K = 4 C against its weight permuted to (Cout, 2, 2, Cin).  y must not alias x.  One launch. */
int sdetr_layernorm_tokens_s2d(const float *x, int batch, int H, int W, int C, const float *ln_weight, const float *ln_bias,
                               float eps, float *y, sdetr_stream_t stream);
/* ---- Swin Transformer backbone in token layout (models/backbones/swin.py; SwinTransformerBackbone.forward_tokens) -----------
 * Token rows (batch, H * W, C) contiguous in raster order.  The Linears run on sdetr_gemm_f16x3_ex, the stem on
 * sdetr_convnext_stem.
 * Shifted-window multi-head attention of V1 Swin (shifted_window_attention without its projections): qkv (batch, H * W, 3 C) is
 * the QKV Linear's output with q, k, v of head h at columns s * C + 32 h + d; qkv_bias (3 C); rel_bias (num_heads, N, N), N =
 * window_h * window_w <= 144, the expanded relative position bias; C = 32 num_heads; 0 <= shift < window per dimension, the
 * block's nominal shift.  The map is padded to pad_H = ceil(H / window_h) window_h (pad_W likewise); the shift is zeroed in a
 * dimension where the window is at least the padded size; window coordinate r of the rolled frame reads source row
 * (r + shift_h) mod pad_H (columns likewise).  A pad position is a zero row before the QKV Linear, so its key and value are the
 * qkv bias; it is not masked, and its query output is dropped.  Logits (q * 32^-0.5) . k + rel_bias[h, i, j], plus -100 where the
 * region ids 3 id_h + id_w of i and j differ (id_h: 0 on [0, pad_H - window_h), 1 on [pad_H - window_h, pad_H - shift_h), 2 on
 * the rest, of the rolled row; id_w likewise).  Softmax with expf, fp32 FMAs.  y (batch, H * W, C), every row written; y must
 * not alias qkv.  One launch. */
int sdetr_window_attention_tokens(const float *qkv, const float *qkv_bias, const float *rel_bias, int batch, int H, int W, int C,
                                  int num_heads, int window_h, int window_w, int shift_h, int shift_w, float *y,
                                  sdetr_stream_t stream);
/* PatchMerging's LayerNorm: y (batch, ceil(H / 2) * ceil(W / 2), 4 C), row (oy, ox) the LayerNorm over 4 C (weight and bias
 * (4 C)) of the concatenation [x(2 oy, 2 ox), x(2 oy + 1, 2 ox), x(2 oy, 2 ox + 1), x(2 oy + 1, 2 ox + 1)], i.e. column
 * (2 dx + dy) C + c; pixels outside the map are zeros that take part in the statistics.  C % 16 == 0, 4 C <= 3072.  Two-pass
 * mean / variance in fp32; a NaN input pixel gives a NaN row.  Operands 16-byte aligned, y must not alias x.  One launch. */
int sdetr_patch_merge_layernorm_tokens(const float *x, int batch, int H, int W, int C, const float *ln_weight,
                                       const float *ln_bias, float eps, float *y, sdetr_stream_t stream);
/* y = LayerNorm(x) over C of rows contiguous token rows (weight and bias (C)), C % 64 == 0, C <= 1536.  Two-pass mean / variance
 * in fp32; a NaN in a row gives a NaN row.  Operands 16-byte aligned, y must not alias x.  One launch. */
int sdetr_layernorm_tokens(const float *x, int64_t rows, int C, const float *ln_weight, const float *ln_bias, float eps, float *y,
                           sdetr_stream_t stream);
/* ---- FocalNet backbone in token layout (models/backbones/focalnet.py; FocalNetBackbone.forward_tokens) ---------------------
 * Token rows (batch, H * W, C) in raster order, C % 64 == 0 and C <= 1536.  The Linears of a block (f, h, proj, fc1, fc2) run on
 * sdetr_gemm_f16x3_ex, a downsample's 3x3 / stride-2 convolution on sdetr_conv2d_f16x3, its LayerNorm and the output norms on
 * sdetr_layernorm_tokens.  GELU is the exact one.
 * The stem: y = LayerNorm(conv(x, W) + bias), conv 7x7, stride 4, padding 2, 3 -> C, on the image zero-padded on the right and
 * bottom to a multiple of 4 (PatchEmbed): y (batch, ceil(H / 4) * ceil(W / 4), C), every tap outside the image a zero.  x: (batch,
 * 3, H, W) NCHW contiguous fp32; weight (147, C) = W[co, c, ky, kx] at row (c * 7 + ky) * 7 + kx, column co.  fp32 FMAs, taps in
 * (c, ky, kx) order, then the bias (sdetr_convnext_stem's body).  Two-pass LayerNorm per row.  One launch. */
int sdetr_focalnet_stem(const float *x, int batch, int H, int W, int C, const float *weight, const float *bias,
                        const float *ln_weight, const float *ln_bias, float eps, float *y, sdetr_stream_t stream);
/* The floats of the partial channel sums that the last focal level writes and sdetr_focal_global_context reads: batch times
 * the row tiles of an H x W map (at most 128) times C. */
int64_t sdetr_focal_context_workspace_floats(int batch, int H, int W, int C);
/* One focal level of FocalModulation: p = GELU(dwconv_k(ctx)), depthwise k x k, padding k / 2 (zeros), no bias, weight (k * k, C)
 * = W[c, 0, ky, kx] at row ky * k + kx, k in {3, 5, 7, 9}; then ctx_all = ctx_all + p * gate per pixel (first: 0 + p * gate),
 * the product and the sum rounded on their own, as the reference's chain.  ctx and gate: pixel r of image n at (n H W + r) *
 * ld_ctx (ld_gate), e.g. column slices of f's output; ctx 8-byte aligned, ld_ctx even.  out (batch, H * W, C) receives p, or NULL;
 * ctx_all (batch, H * W, C) is read (unless first) and written.  partials (sdetr_focal_context_workspace_floats) or NULL: on the
 * last level the per-tile channel sums of p for sdetr_focal_global_context, each in a fixed order.  out, ctx_all and ctx must not
 * alias.  fp32 FMAs.  One launch. */
int sdetr_focal_level_tokens(const float *ctx, int64_t ld_ctx, const float *gate, int64_t ld_gate, const float *weight, int ksize,
                             int batch, int H, int W, int C, int first, float *out, float *ctx_all, float *partials,
                             int64_t partials_floats, sdetr_stream_t stream);
/* The global context of FocalModulation: m = GELU(mean over the image's H * W pixels of ctx_L), the partial sums of the last
 * focal level reduced in a fixed order (repeated calls give the same bits; a NaN pixel poisons its image), then in place
 * ctx_all = ctx_all + m * gate, divided by (focal_level + 1) when normalize is set, each operation rounded on its own.  gate:
 * pixel r of image n at (n H W + r) * ld_gate.  One launch. */
int sdetr_focal_global_context(const float *partials, int64_t partials_floats, const float *gate, int64_t ld_gate, int batch, int H,
                               int W, int C, int focal_level, int normalize, float *ctx_all, sdetr_stream_t stream);
/* y = q * h over rows x C (C % 4 == 0): q row r at r * ld_q (ld_q % 4 == 0), h and y contiguous; y may be h, not q.  Operands
 * 16-byte aligned.  One launch. */
int sdetr_focal_modulate(const float *q, int64_t ld_q, const float *h, int64_t rows, int C, float *y, sdetr_stream_t stream);
/* The post-LN residual of a FocalModulationBlock: t = t + gamma * LayerNorm(y) in place, y and t contiguous rows of C, gamma (C),
 * the LayerNorm of sdetr_layernorm_tokens, the product and the sum rounded on their own.  t must not alias y; operands 16-byte
 * aligned.  One launch. */
int sdetr_layernorm_scale_add_tokens(const float *y, int64_t rows, int C, const float *ln_weight, const float *ln_bias, float eps,
                                     const float *gamma, float *t, sdetr_stream_t stream);
#ifdef __cplusplus
}
#endif
#endif /* SDETR_B200_H */
