// Contrastive denoising queries of a Salience-DETR training step: GenerateCDNQueries.forward after its random draws
// (models/bricks/denoising.py:178-329, generate_query_masks :64-76), the embedding backward of its label queries, and the
// denoising-loss indices of DNDETRDetector.compute_dn_loss (models/detectors/base_detector.py:205-218).
//
// The per-image gt table travels by value as a __grid_constant__ kernel parameter: no torch.cat, no host-to-device copy, so
// a step that calls these entry points never synchronises and can be captured in a CUDA graph.
//
// Bit parity with the reference's chain of separate torch kernels: every multiply and add below is an explicit
// __fmul_rn / __fadd_rn / __fsub_rn (nvcc would otherwise contract a*b+c into an FMA), and logf is the full-precision
// CUDA math library function torch's log kernel calls.
#include <math.h>
#include <string.h>

#include "common.cuh"

namespace sdetr {
namespace {

constexpr int kRowWarps = 8;  // slots per CTA of the query job (one warp per slot)
constexpr int kThreads = 32 * kRowWarps;
constexpr int kMaskBytesPerThread = 4;
constexpr int kGradThreads = 128;

struct ImageTable {
    sdetr_cdn_image im[SDETR_CDN_MAX_IMAGES];
};

struct CountTable {
    int32_t n[SDETR_CDN_MAX_IMAGES];
};

__device__ __forceinline__ float clamp01(float x) { return isnan(x) ? x : fminf(fmaxf(x, 0.f), 1.f); }  // torch clamp(0, 1)
__device__ __forceinline__ float clamp_min(float x, float lo) { return isnan(x) ? x : fmaxf(x, lo); }    // torch clamp(min=)

// util/misc.py:31-35: x = clamp(x, 0, 1); log(clamp(x, min=eps) / clamp(1 - x, min=eps)), eps = 1e-3 as float32
__device__ __forceinline__ float inverse_sigmoid(float x) {
    const float eps = 1e-3f;
    x = clamp01(x);
    return logf(__fdiv_rn(clamp_min(x, eps), clamp_min(__fsub_rn(1.f, x), eps)));
}

// The query job: one warp per (image i, slot j) of the (b, 2*G*m) denoising queries.  Slot j = r*m + t holds copy r of gt t;
// its flat index in the reference's repeated, concatenated gt list is r*S + off_i + t (S = sum of the gt counts).
__device__ void query_slot(const ImageTable &tab, int slot, int D, int m, int64_t S,
                           const float *__restrict__ label_rand, const int64_t *__restrict__ label_randint,
                           const float *__restrict__ box_randint, const float *__restrict__ box_rand, float label_threshold,
                           float box_noise_scale, const float *__restrict__ weight, int K, int C, float *__restrict__ label_q,
                           float *__restrict__ box_q, int32_t *__restrict__ noised_labels) {
    const int lane = threadIdx.x & 31;
    const int i = slot / D, j = slot - i * D;
    const int r = j / m, t = j - r * m;
    float *qrow = label_q + (int64_t)slot * C;
    float *brow = box_q + (int64_t)slot * 4;
    if (t >= tab.im[i].num_gt) {  // padding: zeros, no label
        for (int c = lane; c < C; c += 32) qrow[c] = 0.f;
        if (lane < 4) brow[lane] = 0.f;
        if (lane == 0) noised_labels[slot] = -1;
        return;
    }
    int64_t off = 0;
    for (int k = 0; k < i; ++k) off += tab.im[k].num_gt;
    const int64_t f = (int64_t)r * S + off + t;

    // label noise: where(rand < label_noise_prob * 0.5, randint(0, K), label)
    int64_t lab = tab.im[i].gt_labels[t];
    if (label_rand && label_rand[f] < label_threshold) lab = label_randint[f];
    const bool ok = lab >= 0 && lab < K;
    const float *wrow = weight + (ok ? lab : 0) * (int64_t)C;
    for (int c = lane; c < C; c += 32) qrow[c] = ok ? wrow[c] : NAN;  // an nn.Embedding lookup; NaN where it would raise
    if (lane == 0) noised_labels[slot] = ok ? (int32_t)lab : -1;

    if (lane == 0) {
        const float *gb = tab.im[i].gt_boxes + 4 * (int64_t)t;
        const float cx = gb[0], cy = gb[1], w = gb[2], h = gb[3];
        float o[4] = {cx, cy, w, h};
        if (box_rand) {  // GenerateCDNQueries.apply_box_noise
            const float diff[4] = {__fdiv_rn(w, 2.f), __fdiv_rn(h, 2.f), __fdiv_rn(w, 2.f), __fdiv_rn(h, 2.f)};
            float xy[4] = {__fsub_rn(cx, __fmul_rn(0.5f, w)), __fsub_rn(cy, __fmul_rn(0.5f, h)),
                           __fadd_rn(cx, __fmul_rn(0.5f, w)), __fadd_rn(cy, __fmul_rn(0.5f, h))};
            const bool negative = r & 1;
#pragma unroll
            for (int k = 0; k < 4; ++k) {
                const float sign = __fsub_rn(__fmul_rn(box_randint[4 * f + k], 2.f), 1.f);
                float part = box_rand[4 * f + k];
                if (negative) part = __fadd_rn(part, 1.f);
                part = __fmul_rn(part, sign);
                xy[k] = clamp01(__fadd_rn(xy[k], __fmul_rn(__fmul_rn(part, diff[k]), box_noise_scale)));
            }
            o[0] = __fdiv_rn(__fadd_rn(xy[0], xy[2]), 2.f);
            o[1] = __fdiv_rn(__fadd_rn(xy[1], xy[3]), 2.f);
            o[2] = __fsub_rn(xy[2], xy[0]);
            o[3] = __fsub_rn(xy[3], xy[1]);
        }
#pragma unroll
        for (int k = 0; k < 4; ++k) brow[k] = inverse_sigmoid(o[k]);
    }
}

// Grid: [query blocks | status blocks | mask blocks].
__global__ void __launch_bounds__(kThreads) cdn_queries_kernel(
    const __grid_constant__ ImageTable tab, int b, int m, int G, int num_queries, int64_t S, int query_blocks,
    int status_blocks, const float *__restrict__ label_rand, const int64_t *__restrict__ label_randint,
    const float *__restrict__ box_randint, const float *__restrict__ box_rand, float label_threshold, float box_noise_scale,
    const float *__restrict__ weight, int K, int C, float *__restrict__ label_q, float *__restrict__ box_q,
    int32_t *__restrict__ noised_labels, uint8_t *__restrict__ attn_mask, int32_t *__restrict__ status) {
    // sizes fit in int32 (checked on the host): 64-bit divisions would be calls
    const int D = 2 * G * m;  // denoising queries per image
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    int blk = blockIdx.x;
    if (blk < query_blocks) {
        const int slot = blk * kRowWarps + warp;
        if (slot < b * D)
            query_slot(tab, slot, D, m, S, label_rand, label_randint, box_randint, box_rand, label_threshold,
                       box_noise_scale, weight, K, C, label_q, box_q, noised_labels);
        return;
    }
    blk -= query_blocks;
    if (blk < status_blocks) {  // status[i] = 1 when one of image i's noised labels lies outside [0, K)
        const int i = blk * kRowWarps + warp;
        if (i >= b) return;
        const int n = tab.im[i].num_gt;
        int64_t off = 0;
        for (int k = 0; k < i; ++k) off += tab.im[k].num_gt;
        bool bad = false;
        for (int e = lane; e < 2 * G * n; e += 32) {
            const int r = e / n, t = e - r * n;
            const int64_t f = (int64_t)r * S + off + t;
            int64_t lab = tab.im[i].gt_labels[t];
            if (label_rand && label_rand[f] < label_threshold) lab = label_randint[f];
            bad |= lab < 0 || lab >= K;
        }
        bad = __any_sync(0xffffffffu, bad);
        if (lane == 0) status[i] = bad ? 1 : 0;
        return;
    }
    blk -= status_blocks;
    // generate_query_masks(2m): a matching query sees no denoising query; a denoising query sees only its own group of 2m
    const int T = D + num_queries, gs = 2 * m;
    const int e0 = (blk * kThreads + threadIdx.x) * kMaskBytesPerThread;
#pragma unroll
    for (int k = 0; k < kMaskBytesPerThread; ++k) {
        const int e = e0 + k;
        if (e >= T * T) break;
        const int row = e / T, col = e - row * T;
        bool hide;
        if (row >= D) hide = col < D;
        else hide = col < D && col / gs != row / gs;
        attn_mask[e] = hide;
    }
}

// grad_weight[k, c] = sum over the slots s with noised_labels[s] == k, in ascending s, of grad[s, c]: one thread per
// (class, column), fixed order, no atomics -- bit-reproducible.
__global__ void __launch_bounds__(kGradThreads) cdn_queries_backward_kernel(const float *__restrict__ grad,
                                                                             const int32_t *__restrict__ noised_labels,
                                                                             int64_t num_slots, int C,
                                                                             float *__restrict__ grad_weight) {
    const int k = blockIdx.y;
    const int c = blockIdx.x * kGradThreads + threadIdx.x;
    if (c >= C) return;
    float acc = 0.f;
    for (int64_t s = 0; s < num_slots; ++s)
        if (noised_labels[s] == k) acc = __fadd_rn(acc, grad[s * C + c]);
    grad_weight[(int64_t)k * C + c] = acc;
}

// (g * 2m + t, t) for g < G, t < n_i, image after image; src in indices[0, P), tgt in indices[P, 2P), P = G * sum n_i
__global__ void cdn_loss_indices_kernel(const __grid_constant__ CountTable tab, int b, int G, int max_gt, int64_t P,
                                        int64_t *__restrict__ indices) {
    const int64_t e = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (e >= P) return;
    int64_t base = 0;
    int i = 0;
    for (; i < b; ++i) {
        const int64_t cnt = (int64_t)G * tab.n[i];
        if (e < base + cnt) break;
        base += cnt;
    }
    const int n = tab.n[i];
    const int64_t k = e - base;
    const int64_t g = k / n, t = k - g * n;
    indices[e] = g * max_gt + t;
    indices[P + e] = t;
}

int check_images(const sdetr_cdn_image *ims, int num_images, const char *what) {
    SDETR_REQUIRE(ims || num_images == 0, SDETR_ERR_INVALID_ARG, "%s: null pointer (images_host)", what);
    SDETR_REQUIRE(num_images >= 0 && num_images <= SDETR_CDN_MAX_IMAGES, SDETR_ERR_INVALID_ARG, "%s: %d images (0..%d per call)",
                  what, num_images, SDETR_CDN_MAX_IMAGES);
    for (int i = 0; i < num_images; ++i) {
        SDETR_REQUIRE(ims[i].num_gt >= 0, SDETR_ERR_INVALID_ARG, "%s: image %d has %d gts", what, i, ims[i].num_gt);
        SDETR_REQUIRE(ims[i].num_gt == 0 || (ims[i].gt_labels && ims[i].gt_boxes), SDETR_ERR_INVALID_ARG,
                      "%s: null pointer (image %d gt_labels / gt_boxes)", what, i);
    }
    return SDETR_OK;
}

}  // namespace
}  // namespace sdetr

using namespace sdetr;

extern "C" int sdetr_cdn_queries(const sdetr_cdn_image *images_host, int num_images, const float *label_rand,
                                 const int64_t *label_randint, const float *box_randint, const float *box_rand,
                                 float label_threshold, float box_noise_scale, const float *weight, int num_classes,
                                 int embed_dim, int weight_rows, int weight_cols, int num_queries, int groups, int max_gt,
                                 float *label_queries, float *box_queries, int32_t *noised_labels, uint8_t *attn_mask,
                                 int32_t *status, sdetr_stream_t stream) {
    int rc = check_images(images_host, num_images, "sdetr_cdn_queries");
    if (rc) return rc;
    SDETR_REQUIRE(num_images >= 1, SDETR_ERR_INVALID_ARG, "sdetr_cdn_queries: no images");
    SDETR_REQUIRE(num_classes >= 1 && embed_dim >= 1 && num_queries >= 0 && groups >= 1 && max_gt >= 0, SDETR_ERR_INVALID_ARG,
                  "sdetr_cdn_queries: bad sizes (K %d, C %d, queries %d, groups %d, max_gt %d)", num_classes, embed_dim,
                  num_queries, groups, max_gt);
    SDETR_REQUIRE(weight_rows == num_classes && weight_cols == embed_dim, SDETR_ERR_INVALID_ARG,
                  "sdetr_cdn_queries: label_encoder.weight is (%d, %d), expected (num_classes %d, embed_dim %d)", weight_rows,
                  weight_cols, num_classes, embed_dim);
    int64_t S = 0;
    int mx = 0;
    for (int i = 0; i < num_images; ++i) S += images_host[i].num_gt, mx = images_host[i].num_gt > mx ? images_host[i].num_gt : mx;
    SDETR_REQUIRE(mx == max_gt, SDETR_ERR_INVALID_ARG, "sdetr_cdn_queries: max_gt %d, the largest gt count is %d", max_gt, mx);
    SDETR_REQUIRE(!label_rand == !label_randint && !box_rand == !box_randint, SDETR_ERR_INVALID_ARG,
                  "sdetr_cdn_queries: give both label draws and both box draws, or neither");
    const int64_t D = 2 * (int64_t)groups * max_gt, T = D + num_queries;
    SDETR_REQUIRE(weight && attn_mask && status, SDETR_ERR_INVALID_ARG, "sdetr_cdn_queries: null pointer (weight / attn_mask / status)");
    SDETR_REQUIRE(D == 0 || (label_queries && box_queries && noised_labels), SDETR_ERR_INVALID_ARG,
                  "sdetr_cdn_queries: null pointer (label_queries / box_queries / noised_labels)");
    SDETR_REQUIRE(S == 0 || ((label_rand || label_threshold <= 0.f) && (box_rand || box_noise_scale <= 0.f)), SDETR_ERR_INVALID_ARG,
                  "sdetr_cdn_queries: a noise parameter is positive but its draws are missing");
    const int64_t query_blocks = ((int64_t)num_images * D + kRowWarps - 1) / kRowWarps;
    const int64_t status_blocks = (num_images + kRowWarps - 1) / kRowWarps;
    const int64_t per_block = (int64_t)kThreads * kMaskBytesPerThread;
    const int64_t mask_blocks = (T * T + per_block - 1) / per_block;
    const int64_t blocks = query_blocks + status_blocks + mask_blocks;
    SDETR_REQUIRE(T * T + per_block < INT32_MAX && num_images * D < INT32_MAX,
                  SDETR_ERR_UNSUPPORTED, "sdetr_cdn_queries: %lld denoising + %d matching queries is too many", (long long)D,
                  num_queries);
    ImageTable tab;
    memset(&tab, 0, sizeof(tab));
    for (int i = 0; i < num_images; ++i) tab.im[i] = images_host[i];
    cdn_queries_kernel<<<(unsigned)blocks, kThreads, 0, (cudaStream_t)stream>>>(
        tab, num_images, max_gt, groups, num_queries, S, (int)query_blocks, (int)status_blocks, label_rand, label_randint, box_randint,
        box_rand, label_threshold, box_noise_scale, weight, num_classes, embed_dim, label_queries, box_queries, noised_labels,
        attn_mask, status);
    return check_launch("sdetr_cdn_queries");
}

extern "C" int sdetr_cdn_queries_backward(const float *grad_label_queries, const int32_t *noised_labels, int64_t num_slots,
                                          int num_classes, int embed_dim, float *grad_weight, sdetr_stream_t stream) {
    SDETR_REQUIRE(num_classes >= 1 && embed_dim >= 1 && num_slots >= 0, SDETR_ERR_INVALID_ARG,
                  "sdetr_cdn_queries_backward: bad sizes (K %d, C %d, slots %lld)", num_classes, embed_dim, (long long)num_slots);
    SDETR_REQUIRE(num_classes <= 65535, SDETR_ERR_UNSUPPORTED, "sdetr_cdn_queries_backward: %d classes (at most 65535)", num_classes);
    SDETR_REQUIRE(grad_weight && (num_slots == 0 || (grad_label_queries && noised_labels)), SDETR_ERR_INVALID_ARG,
                  "sdetr_cdn_queries_backward: null pointer");
    const dim3 grid((embed_dim + kGradThreads - 1) / kGradThreads, num_classes);
    cdn_queries_backward_kernel<<<grid, kGradThreads, 0, (cudaStream_t)stream>>>(grad_label_queries, noised_labels, num_slots,
                                                                                 embed_dim, grad_weight);
    return check_launch("sdetr_cdn_queries_backward");
}

extern "C" int sdetr_cdn_loss_indices(const int32_t *num_gt_host, int num_images, int groups, int max_gt, int64_t *indices,
                                      sdetr_stream_t stream) {
    SDETR_REQUIRE(num_gt_host || num_images == 0, SDETR_ERR_INVALID_ARG, "sdetr_cdn_loss_indices: null pointer (num_gt_host)");
    SDETR_REQUIRE(num_images >= 0 && num_images <= SDETR_CDN_MAX_IMAGES, SDETR_ERR_INVALID_ARG,
                  "sdetr_cdn_loss_indices: %d images (0..%d per call)", num_images, SDETR_CDN_MAX_IMAGES);
    SDETR_REQUIRE(groups >= 1 && max_gt >= 0, SDETR_ERR_INVALID_ARG, "sdetr_cdn_loss_indices: groups %d, max_gt %d", groups, max_gt);
    CountTable tab;
    memset(&tab, 0, sizeof(tab));
    int64_t P = 0;
    for (int i = 0; i < num_images; ++i) {
        SDETR_REQUIRE(num_gt_host[i] >= 0 && num_gt_host[i] <= max_gt, SDETR_ERR_INVALID_ARG,
                      "sdetr_cdn_loss_indices: image %d has %d gts (0..max_gt %d)", i, num_gt_host[i], max_gt);
        tab.n[i] = num_gt_host[i];
        P += (int64_t)groups * num_gt_host[i];
    }
    SDETR_REQUIRE(P == 0 || indices, SDETR_ERR_INVALID_ARG, "sdetr_cdn_loss_indices: null pointer (indices)");
    if (P == 0) return SDETR_OK;
    cdn_loss_indices_kernel<<<(unsigned)((P + 255) / 256), 256, 0, (cudaStream_t)stream>>>(tab, num_images, groups, max_gt, P,
                                                                                          indices);
    return check_launch("sdetr_cdn_loss_indices");
}
