// Detection post-processing for sm_90a -- sdetr_postprocess.
//
// Reference semantics: PostProcess.forward (models/bricks/post_process.py:21-74): sigmoid of the class logits, top-k over the
// flattened (query, class) scores of each image, label = index % K, query = index / K, the query's cxcywh box converted to
// xyxy and scaled by (w, h, w, h) of the image; optionally a confidence filter (score > confidence) AND greedy NMS
// (torchvision.ops.nms) over all k boxes, then the kept entries in order.  The reference runs ~a dozen torch launches, plus
// per-image host round trips and NMS calls when a filter is on; here each image is one 1024-thread CTA of ONE launch:
//   1. the sigmoid of every logit, as a descending-order key (desc_key) in the workspace -- bit-identical to torch.sigmoid
//      on CUDA (1 / (1 + expf(-x)), each operation rounded on its own);
//   2. top-k with the machinery of sdetr_topk_desc (select.cuh): radix select of the k-th key, stable compaction of the
//      winners in index order, bitonic sort of the (key, index) composites in shared memory.  Order: probability
//      descending, ties by smaller flat index, NaN first == torch.sort(p, descending=True, stable=True)[:k];
//   3. decode of the winners with every torch operation rounded separately (no contraction into FMAs);
//   4. with a filter on: the keep flag, greedy NMS in top-k order in chunks of 32 (the CTA tests the chunk's pairs, one
//      warp resolves the chunk in rank order with bit operations, then the CTA suppresses the later boxes that overlap the
//      chunk's kept ones -- exactly the sequential greedy result), and an ordered block scan that compacts the kept entries
//      and writes the count.
#include "select.cuh"

namespace sdetr {

static_assert(kTopkFast == SDETR_POSTPROCESS_MAX_K, "the C-ABI limit is the winner buffer of the single-CTA top-k");

// torch.sigmoid on CUDA: one / (one + std::exp(-a)) in fp32, full-precision expf, IEEE division
__device__ __forceinline__ float sigmoid_rn(float x) { return __fdiv_rn(1.f, __fadd_rn(1.f, expf(-x))); }

// torchvision's IoU test (nms_kernel.cu devIoU): widths clamped at 0, inter / (area_a + area_b - inter) > threshold.  A
// zero-area pair gives 0 / 0 = NaN, which never suppresses.
__device__ __forceinline__ bool iou_above(float4 a, float4 b, float threshold) {
    const float w = fmaxf(__fsub_rn(fminf(a.z, b.z), fmaxf(a.x, b.x)), 0.f);
    const float h = fmaxf(__fsub_rn(fminf(a.w, b.w), fmaxf(a.y, b.y)), 0.f);
    const float inter = __fmul_rn(w, h);
    const float sa = __fmul_rn(__fsub_rn(a.z, a.x), __fsub_rn(a.w, a.y));
    const float sb = __fmul_rn(__fsub_rn(b.z, b.x), __fsub_rn(b.w, b.y));
    return __fdiv_rn(inter, __fsub_rn(__fadd_rn(sa, sb), inter)) > threshold;
}

// bytes of dynamic shared memory per candidate when a filter is on: its box, its score and its suppression flag
constexpr int kPostFilterBytes = 16 + 4 + 1;

__global__ void __launch_bounds__(kSortThreads) postprocess_kernel(
    const float *__restrict__ logits, int64_t logits_bs, int64_t logits_qs, const float *__restrict__ pred_boxes,
    int64_t boxes_bs, int64_t boxes_qs, const void *__restrict__ target_sizes, int sizes_dtype, int Q, int K, int k, int N,
    float confidence, float iou_threshold, uint32_t *keys, float *__restrict__ out_scores, int64_t *__restrict__ out_labels,
    float *__restrict__ out_boxes, int32_t *__restrict__ count) {
    __shared__ SelectSmem sm;
    extern __shared__ float4 filt[];  // filters on: k boxes, k scores, k suppression flags
    unsigned long long *win = reinterpret_cast<unsigned long long *>(sm.hist);  // free once radix_select returned
    const int b = blockIdx.x, tid = threadIdx.x, n = Q * K;
    const float *lg = logits + (int64_t)b * logits_bs;
    const float *pb = pred_boxes + (int64_t)b * boxes_bs;
    auto logit = [=](int i) {
        const int q = i / K;
        return __ldg(lg + (int64_t)q * logits_qs + (i - q * K));
    };
    // 1. keys of the probabilities; plain loads below (not __ldg): this CTA wrote them.  kBatch logits are loaded before any
    //    is used, so that each thread has that many HBM reads in flight; (query, class) of index i steps along with i instead
    //    of being divided out for every element.
    constexpr int kBatch = 8;
    uint32_t *kw = keys + (int64_t)b * n;
    const int step_q = kSortThreads / K, step_c = kSortThreads % K;
    int q = tid / K, c = tid % K;
    for (int i0 = tid; i0 < n; i0 += kBatch * kSortThreads) {
        float x[kBatch];
#pragma unroll
        for (int u = 0; u < kBatch; ++u) {
            x[u] = i0 + u * kSortThreads < n ? __ldg(lg + (int64_t)q * logits_qs + c) : 0.f;
            q += step_q, c += step_c;
            if (c >= K) c -= K, ++q;
        }
#pragma unroll
        for (int u = 0; u < kBatch; ++u)
            if (i0 + u * kSortThreads < n) kw[i0 + u * kSortThreads] = desc_key(sigmoid_rn(x[u]));
    }
    __syncthreads();
    auto key = [=](int i) { return kw[i]; };
    // 2. top-k in canonical order
    uint32_t T, need;
    radix_select(key, n, k, T, need, sm);
    for (int j = tid; j < N; j += kSortThreads) win[j] = ~0ull;
    __syncthreads();
    stable_compact(key, n, T, need,
                   [&](uint32_t pos, int i, uint32_t kv) { win[pos] = ((unsigned long long)kv << 32) | (uint32_t)i; }, sm);
    __syncthreads();
    bitonic_sort_smem(win, N);
    // 3. decode: torch's _box_cxcywh_to_xyxy, then * (img_w, img_h, img_w, img_h) converted to fp32
    float img_h, img_w;
    if (sizes_dtype == SDETR_SIZES_INT64) {
        img_h = (float)((const int64_t *)target_sizes)[2 * b], img_w = (float)((const int64_t *)target_sizes)[2 * b + 1];
    } else if (sizes_dtype == SDETR_SIZES_INT32) {
        img_h = (float)((const int32_t *)target_sizes)[2 * b], img_w = (float)((const int32_t *)target_sizes)[2 * b + 1];
    } else {
        img_h = ((const float *)target_sizes)[2 * b], img_w = ((const float *)target_sizes)[2 * b + 1];
    }
    auto flat = [&](int j) { return (int)(win[j] & 0xffffffffull); };
    auto box_of = [&](int i) {
        const float *p = pb + (int64_t)(i / K) * boxes_qs;
        const float cx = __ldg(p), cy = __ldg(p + 1), hw = __fmul_rn(0.5f, __ldg(p + 2)), hh = __fmul_rn(0.5f, __ldg(p + 3));
        return make_float4(__fmul_rn(__fsub_rn(cx, hw), img_w), __fmul_rn(__fsub_rn(cy, hh), img_h),
                           __fmul_rn(__fadd_rn(cx, hw), img_w), __fmul_rn(__fadd_rn(cy, hh), img_h));
    };
    auto store = [&](int pos, float s, int i, float4 bx) {
        const int64_t o = (int64_t)b * k + pos;
        out_scores[o] = s;
        out_labels[o] = i % K;
        float *ob = out_boxes + o * 4;
        ob[0] = bx.x, ob[1] = bx.y, ob[2] = bx.z, ob[3] = bx.w;
    };
    const bool conf_on = confidence > 0.f, nms_on = iou_threshold > 0.f;
    if (!conf_on && !nms_on) {
        for (int j = tid; j < k; j += kSortThreads) {
            const int i = flat(j);
            store(j, sigmoid_rn(logit(i)), i, box_of(i));
        }
        if (count && tid == 0) count[b] = k;
        return;
    }
    // 4. filters
    float4 *sbox = filt;
    float *sscore = reinterpret_cast<float *>(filt + k);
    uint8_t *supp = reinterpret_cast<uint8_t *>(sscore + k);
    for (int j = tid; j < k; j += kSortThreads) {
        const int i = flat(j);
        sbox[j] = box_of(i), sscore[j] = sigmoid_rn(logit(i)), supp[j] = 0;
    }
    __syncthreads();
    if (nms_on) {
        __shared__ unsigned rows[kSortWarps], chunk_kept;
        const int lane = tid & 31, warp = tid >> 5;
        static_assert(kSortWarps == 32, "one warp per box of a 32-box chunk");
        for (int c0 = 0; c0 < k; c0 += 32) {
            // rows[w]: the later boxes of the chunk that its box w overlaps, one pair per thread
            const int j = c0 + lane;
            const bool over = lane > warp && j < k && iou_above(sbox[c0 + warp], sbox[j], iou_threshold);
            const unsigned row = __ballot_sync(0xffffffffu, over);
            if (lane == 0) rows[warp] = row;
            __syncthreads();
            if (warp == 0) {  // greedy inside the chunk, in rank order
                unsigned alive = __ballot_sync(0xffffffffu, j < k && !supp[j]);
                for (int t = 0; t < 32; ++t)
                    if ((alive >> t) & 1u) alive &= ~rows[t];
                if (j < k && !((alive >> lane) & 1u)) supp[j] = 1;
                if (lane == 0) chunk_kept = alive;
            }
            __syncthreads();
            // the chunk's kept boxes suppress later ones: a warp per later box, lane t tests the chunk's box t
            const unsigned kept = chunk_kept;
            for (int l = c0 + 32 + warp; kept && l < k; l += kSortWarps) {
                if (supp[l]) continue;  // warp-uniform
                const bool hit = ((kept >> lane) & 1u) && iou_above(sbox[c0 + lane], sbox[l], iou_threshold);
                if (__any_sync(0xffffffffu, hit) && lane == 0) supp[l] = 1;
            }
            __syncthreads();
        }
    }
    // ordered compaction: each thread owns a contiguous run of ranks
    const int per = (k + kSortThreads - 1) / kSortThreads;
    const int begin = min(k, tid * per), end = min(k, begin + per);
    auto keep = [&](int j) { return !supp[j] && (!conf_on || sscore[j] > confidence); };
    uint32_t mine = 0, pos, unused;
    for (int j = begin; j < end; ++j) mine += keep(j);
    block_scan_pair(mine, 0u, pos, unused, sm);
    for (int j = begin; j < end; ++j)
        if (keep(j)) store(pos++, sscore[j], flat(j), sbox[j]);
    if (tid == kSortThreads - 1) count[b] = (int32_t)pos;
}

static int next_pow2(int x) {
    int p = 1;
    while (p < x) p <<= 1;
    return p;
}

}  // namespace sdetr

using namespace sdetr;

extern "C" size_t sdetr_postprocess_workspace(int batch, int num_queries, int num_classes) {
    if (batch <= 0 || num_queries <= 0 || num_classes <= 0) return 0;
    return (size_t)batch * num_queries * num_classes * sizeof(uint32_t);
}

extern "C" int sdetr_postprocess(const float *pred_logits, int64_t logits_batch_stride, int64_t logits_query_stride,
                                 const float *pred_boxes, int64_t boxes_batch_stride, int64_t boxes_query_stride,
                                 const void *target_sizes, int sizes_dtype, int batch, int num_queries, int num_classes, int k,
                                 float confidence_score, float iou_threshold, float *scores, int64_t *labels, float *boxes,
                                 int32_t *count, void *workspace, size_t workspace_bytes, sdetr_stream_t stream) {
    SDETR_REQUIRE(pred_logits && pred_boxes && target_sizes && scores && labels && boxes && workspace, SDETR_ERR_INVALID_ARG,
                  "postprocess: null pointer");
    const bool filters = confidence_score > 0.f || iou_threshold > 0.f;
    SDETR_REQUIRE(count || !filters, SDETR_ERR_INVALID_ARG, "postprocess: null pointer (count is needed with a filter on)");
    SDETR_REQUIRE(batch > 0 && num_queries > 0 && num_classes > 0, SDETR_ERR_INVALID_ARG,
                  "postprocess: bad sizes (batch %d, queries %d, classes %d)", batch, num_queries, num_classes);
    const int64_t n = (int64_t)num_queries * num_classes;
    SDETR_REQUIRE(n < ((int64_t)1 << 31), SDETR_ERR_UNSUPPORTED, "postprocess: %lld scores per image, at most 2^31 - 1",
                  (long long)n);
    SDETR_REQUIRE(k >= 1 && k <= n, SDETR_ERR_INVALID_ARG, "postprocess: k=%d outside [1, %lld]", k, (long long)n);
    SDETR_REQUIRE(k <= kTopkFast, SDETR_ERR_UNSUPPORTED, "postprocess: k=%d, at most %d (the single-CTA top-k limit)", k,
                  kTopkFast);
    SDETR_REQUIRE(sizes_dtype == SDETR_SIZES_INT64 || sizes_dtype == SDETR_SIZES_INT32 || sizes_dtype == SDETR_SIZES_FLOAT32,
                  SDETR_ERR_INVALID_ARG, "postprocess: bad target_sizes dtype code %d", sizes_dtype);
    SDETR_REQUIRE(workspace_bytes >= sdetr_postprocess_workspace(batch, num_queries, num_classes), SDETR_ERR_WORKSPACE,
                  "postprocess: workspace too small");
    const size_t smem = filters ? (size_t)k * kPostFilterBytes : 0;
    static PerDeviceOnce once;
    SDETR_OPT_IN_SMEM(once, postprocess_kernel, kTopkFast * kPostFilterBytes, "postprocess");
    postprocess_kernel<<<batch, kSortThreads, smem, (cudaStream_t)stream>>>(
        pred_logits, logits_batch_stride, logits_query_stride, pred_boxes, boxes_batch_stride, boxes_query_stride, target_sizes,
        sizes_dtype, num_queries, num_classes, k, next_pow2(k), confidence_score, iou_threshold, (uint32_t *)workspace, scores,
        labels, boxes, count);
    return check_launch("postprocess");
}
