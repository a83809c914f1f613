// Detection loss of a Salience-DETR training step: the HungarianMatcher's cost matrix and exact assignment
// (models/matcher/hungarian_matcher.py:41-91) and HybridSetCriterion.calculate_loss (models/bricks/set_criterion.py:84-131,
// 174-212), forward and backward, for every (output, image) problem of a step in O(1) launches.
//
// The problem table travels by value as a __grid_constant__ kernel parameter: no host-to-device copy, so a step that calls
// these entry points stays capturable in a CUDA graph and never synchronises.
#include <math.h>
#include <string.h>

#include "common.cuh"

namespace sdetr {
namespace {

constexpr int kSolverThreads = 256;
constexpr int kLossThreads = 256;
constexpr int kRowsPerBlock = 32;  // queries per CTA of the loss kernels

struct ProblemTable {
    sdetr_set_problem p[SDETR_SET_MAX_PROBLEMS];
};

struct Box {
    float x0, y0, x1, y1;
};

__device__ __forceinline__ Box cxcywh_to_xyxy(const float *b) {  // torchvision _box_cxcywh_to_xyxy
    const float cx = b[0], cy = b[1], w = b[2], h = b[3];
    return {cx - 0.5f * w, cy - 0.5f * h, cx + 0.5f * w, cy + 0.5f * h};
}

__device__ __forceinline__ float clamp0(float x) { return x < 0.f ? 0.f : x; }  // clamp(min=0); NaN passes through

// torchvision box_iou / generalized_box_iou for one pair
__device__ __forceinline__ void pair_iou(const Box &a, const Box &b, float &iou, float &giou) {
    const float area1 = (a.x1 - a.x0) * (a.y1 - a.y0), area2 = (b.x1 - b.x0) * (b.y1 - b.y0);
    const float w = clamp0(fminf(a.x1, b.x1) - fmaxf(a.x0, b.x0)), h = clamp0(fminf(a.y1, b.y1) - fmaxf(a.y0, b.y0));
    const float inter = w * h, uni = area1 + area2 - inter;
    iou = inter / uni;
    const float wi = clamp0(fmaxf(a.x1, b.x1) - fminf(a.x0, b.x0)), hi = clamp0(fmaxf(a.y1, b.y1) - fminf(a.y0, b.y0));
    const float areai = wi * hi;
    giou = iou - (areai - uni) / areai;
}

__device__ __forceinline__ float pow_gamma(float x, float gamma) { return gamma == 2.f ? x * x : powf(x, gamma); }

__device__ __forceinline__ float sigmoidf(float x) { return 1.f / (1.f + expf(-x)); }

// binary_cross_entropy_with_logits(x, t) without weight
__device__ __forceinline__ float bce_logits(float x, float t) { return fmaxf(x, 0.f) - x * t + log1pf(expf(-fabsf(x))); }

__device__ __forceinline__ int64_t label_of(const sdetr_set_problem &p, int64_t g) { return p.gt_labels ? p.gt_labels[g] : 0; }

__device__ __forceinline__ float block_sum(float v, float *red) {  // fixed-order sum over the block, result in every thread
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
    __syncthreads();
    if ((threadIdx.x & 31) == 0) red[threadIdx.x >> 5] = v;
    __syncthreads();
    float s = 0.f;
    for (int w = 0; w < (int)(blockDim.x >> 5); ++w) s += red[w];
    return s;
}

// ---- matching: cost matrix + shortest augmenting path, one CTA per problem -----------------------------------------------
// Rows are gts (n), columns queries (Q), n <= Q.  Shortest augmenting path with dual potentials (Jonker & Volgenant 1987;
// the rectangular form of Crouse, "On implementing 2D rectangular assignment algorithms", IEEE TAES 2016): one Dijkstra
// search per row over the reduced costs c[i][j] - u[i] - v[j] >= 0, then a dual update that keeps them non-negative and
// an augmentation along the path.  Duals and path lengths are fp64; each Dijkstra step is a block-wide arg-min over the
// columns not yet reached (ties to the lowest column index), so the result is bit-reproducible.
struct ArgMin {
    double v;
    int j;
};
__device__ __forceinline__ bool better(double a, int ja, double b, int jb) { return a < b || (a == b && ja < jb); }

__device__ __forceinline__ ArgMin block_argmin(double v, int j, ArgMin *red) {
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) {
        const double ov = __shfl_xor_sync(0xffffffffu, v, o);
        const int oj = __shfl_xor_sync(0xffffffffu, j, o);
        if (better(ov, oj, v, j)) v = ov, j = oj;
    }
    if ((threadIdx.x & 31) == 0) red[threadIdx.x >> 5] = {v, j};
    __syncthreads();
    ArgMin r = red[0];
    for (int w = 1; w < kSolverThreads / 32; ++w)
        if (better(red[w].v, red[w].j, r.v, r.j)) r = red[w];
    return r;
}

// kCost: compute the cost matrices into cost_ws; else cost_ws holds them (sdetr_set_assign).
template <bool kCost>
__global__ void __launch_bounds__(kSolverThreads) set_match_kernel(const __grid_constant__ ProblemTable tab, float w_class,
                                                                   float w_bbox, float w_giou, float alpha, float gamma, int K,
                                                                   int32_t *__restrict__ status, float *__restrict__ cost_ws) {
    const int pi = blockIdx.x, tid = threadIdx.x;
    const sdetr_set_problem &p = tab.p[pi];
    const int n = p.num_gt, Q = p.num_queries;
    int64_t ws_off = 0;
    for (int k = 0; k < pi; ++k) ws_off += (int64_t)tab.p[k].num_gt * tab.p[k].num_queries;
    float *cost = cost_ws + ws_off;

    __shared__ int s_bad;
    __shared__ ArgMin s_red[kSolverThreads / 32];
    __shared__ int s_row, s_sink;
    __shared__ double s_minval;
    if (tid == 0) s_bad = 0;
    __syncthreads();
    if (n == 0) {
        if (tid == 0) status[pi] = 0;
        return;
    }

    // cost[i][j] = w_bbox * |pred_j - gt_i|_1 + w_class * (pos - neg)(x[j, label_i]) + w_giou * -GIoU(pred_j, gt_i)
    // a gt label outside [0, K) is an IndexError in the reference: the problem is invalid, its logits are not read
    if (kCost)
        for (int i = tid; i < n; i += kSolverThreads) {
            const int64_t lab = label_of(p, i);
            if (lab < 0 || lab >= K) s_bad = 1;
        }
    __syncthreads();
    bool bad = false;
    if (!kCost)
        for (int64_t e = tid; e < (int64_t)n * Q; e += kSolverThreads) bad |= !(fabsf(cost[e]) <= FLT_MAX);
    for (int i = 0; kCost && !s_bad && i < n; ++i) {
        const float *gb = p.gt_boxes + 4 * i;
        const Box g = cxcywh_to_xyxy(gb);
        const int64_t lab = label_of(p, i);
        for (int j = tid; j < Q; j += kSolverThreads) {
            const float *pb = p.boxes + j * p.box_stride;
            const float x = p.logits[j * p.logit_stride + lab];
            const float pr = sigmoidf(x);
            const float neg = -(1.f - alpha) * pow_gamma(pr, gamma) * logf(1.f - pr + 1e-6f);
            const float pos = -alpha * pow_gamma(1.f - pr, gamma) * logf(pr + 1e-6f);
            const float l1 = fabsf(pb[0] - gb[0]) + fabsf(pb[1] - gb[1]) + fabsf(pb[2] - gb[2]) + fabsf(pb[3] - gb[3]);
            float iou, giou;
            pair_iou(cxcywh_to_xyxy(pb), g, iou, giou);
            const float c = w_bbox * l1 + w_class * (pos - neg) + w_giou * -giou;
            bad |= !(fabsf(c) <= FLT_MAX);
            cost[(int64_t)i * Q + j] = c;
        }
    }
    if (bad) s_bad = 1;  // benign race: every writer stores 1
    __syncthreads();
    if (s_bad) {  // scipy raises ValueError here; a sync-free caller gets a status word and a defined assignment instead
        for (int i = tid; i < n; i += kSolverThreads) p.src[i] = i, p.tgt[i] = i;
        if (tid == 0) status[pi] = 1;
        return;
    }

    extern __shared__ __align__(16) unsigned char smem[];
    double *v = reinterpret_cast<double *>(smem);  // column duals
    double *spc = v + Q;                           // shortest path lengths to the columns
    double *u = spc + Q;                           // row duals
    int *path = reinterpret_cast<int *>(u + n);    // row preceding column j on the shortest path
    int *row4col = path + Q;
    int *col4row = row4col + Q;
    unsigned char *col_done = reinterpret_cast<unsigned char *>(col4row + n);
    unsigned char *row_seen = col_done + Q;
    for (int j = tid; j < Q; j += kSolverThreads) v[j] = 0.0, spc[j] = INFINITY, row4col[j] = -1, col_done[j] = 0;
    for (int i = tid; i < n; i += kSolverThreads) u[i] = 0.0, col4row[i] = -1, row_seen[i] = 0;
    __syncthreads();

    for (int cur = 0; cur < n; ++cur) {
        if (tid == 0) s_row = cur, s_minval = 0.0, s_sink = -1;
        __syncthreads();
        while (true) {
            const int i = s_row;
            const double minval = s_minval, ui = u[i];
            if (tid == 0) row_seen[i] = 1;
            const float *crow = cost + (int64_t)i * Q;
            double best = INFINITY;
            int bj = 0x7fffffff;
            for (int j = tid; j < Q; j += kSolverThreads) {
                if (col_done[j]) continue;
                const double r = minval + (double)crow[j] - ui - v[j];
                double s = spc[j];
                if (r < s) path[j] = i, spc[j] = s = r;
                if (s < best) best = s, bj = j;
            }
            const ArgMin m = block_argmin(best, bj, s_red);
            if (tid == 0) {
                s_minval = m.v;
                col_done[m.j] = 1;
                if (row4col[m.j] < 0) s_sink = m.j;
                else s_row = row4col[m.j];
            }
            __syncthreads();
            if (s_sink >= 0) break;
        }
        const double minval = s_minval;
        for (int i = tid; i < n; i += kSolverThreads) {
            if (!row_seen[i]) continue;
            u[i] += i == cur ? minval : minval - spc[col4row[i]];
            row_seen[i] = 0;
        }
        __syncthreads();
        for (int j = tid; j < Q; j += kSolverThreads) {
            if (col_done[j]) v[j] -= minval - spc[j];
            spc[j] = INFINITY, col_done[j] = 0;
        }
        if (tid == 0) {  // augment along the path back to `cur`
            int j = s_sink;
            while (true) {
                const int i = path[j];
                row4col[j] = i;
                const int prev = col4row[i];
                col4row[i] = j;
                if (i == cur) break;
                j = prev;
            }
        }
        __syncthreads();
    }

    // pairs in ascending query order (scipy's row_ind order for the (Q, n) matrix)
    for (int i = tid; i < n; i += kSolverThreads) {
        const int c = col4row[i];
        int rank = 0;
        for (int k = 0; k < n; ++k) rank += col4row[k] < c;
        p.src[rank] = c;
        p.tgt[rank] = i;
    }
    if (tid == 0) status[pi] = 0;
}

// ---- loss: per CTA kRowsPerBlock queries of one problem ----------------------------------------------------------------
__device__ __forceinline__ int locate_block(const ProblemTable &tab, int count, int b, int &r0) {
    int pi = 0;
    for (; pi < count; ++pi) {
        const int nb = (tab.p[pi].num_queries + kRowsPerBlock - 1) / kRowsPerBlock;
        if (b < nb) break;
        b -= nb;
    }
    r0 = b * kRowsPerBlock;
    return pi;
}

// The matched pairs whose query falls in [r0, r0 + rows): gt index per row (-1: unmatched), the detached IoU of the pair.
// Returns false when a pair's indices or its gt label (>= K) are out of range (the reference raises IndexError there).
__device__ __forceinline__ bool rows_of_block(const sdetr_set_problem &p, int K, int r0, int rows, int *gt_of, float *iou_of) {
    __shared__ int s_bad;
    if (threadIdx.x == 0) s_bad = 0;
    for (int q = threadIdx.x; q < rows; q += blockDim.x) gt_of[q] = -1;
    __syncthreads();
    for (int k = threadIdx.x; k < p.num_pairs; k += blockDim.x) {
        const int64_t q = p.src[k], g = p.tgt[k];
        if (q < 0 || q >= p.num_queries || g < 0 || g >= p.num_gt || label_of(p, g) < 0 || label_of(p, g) >= K) {
            s_bad = 1;
            continue;
        }
        if (q < r0 || q >= r0 + rows) continue;
        float iou, giou;
        pair_iou(cxcywh_to_xyxy(p.boxes + q * p.box_stride), cxcywh_to_xyxy(p.gt_boxes + 4 * g), iou, giou);
        gt_of[q - r0] = (int)g;
        iou_of[q - r0] = iou;
    }
    __syncthreads();
    return !s_bad;
}

__global__ void __launch_bounds__(kLossThreads) set_loss_partials_kernel(const __grid_constant__ ProblemTable tab, int count,
                                                                         int K, float alpha, float gamma,
                                                                         const int32_t *__restrict__ status,
                                                                         float *__restrict__ partials) {
    int r0;
    const int pi = locate_block(tab, count, blockIdx.x, r0);
    const sdetr_set_problem &p = tab.p[pi];
    const int rows = min(kRowsPerBlock, p.num_queries - r0);
    __shared__ int gt_of[kRowsPerBlock];
    __shared__ float iou_of[kRowsPerBlock];
    __shared__ float red[kLossThreads / 32];
    const bool ok = rows_of_block(p, K, r0, rows, gt_of, iou_of) && !(status && status[pi]);

    // varifocal loss: t = onehot * IoU, w = (1 - alpha) sigma^gamma (1 - onehot) + t, sum of w * BCE(x, t)
    float acc = 0.f;
    for (int e = threadIdx.x; e < rows * K; e += kLossThreads) {
        const int q = e / K, c = e - q * K;
        const float x = p.logits[(int64_t)(r0 + q) * p.logit_stride + c];
        const int g = gt_of[q];
        if (g >= 0 && label_of(p, g) == c) {
            const float t = iou_of[q];
            acc += t * bce_logits(x, t);
        } else {
            acc += (1.f - alpha) * pow_gamma(sigmoidf(x), gamma) * bce_logits(x, 0.f);
        }
    }
    // L1 and 1 - GIoU of the matched rows
    float l1 = 0.f, lg = 0.f;
    if (threadIdx.x < rows && gt_of[threadIdx.x] >= 0) {
        const float *pb = p.boxes + (int64_t)(r0 + threadIdx.x) * p.box_stride;
        const float *gb = p.gt_boxes + 4 * gt_of[threadIdx.x];
        l1 = fabsf(pb[0] - gb[0]) + fabsf(pb[1] - gb[1]) + fabsf(pb[2] - gb[2]) + fabsf(pb[3] - gb[3]);
        float iou, giou;
        pair_iou(cxcywh_to_xyxy(pb), cxcywh_to_xyxy(gb), iou, giou);
        lg = 1.f - giou;
    }
    acc = block_sum(acc, red);
    l1 = block_sum(l1, red);
    lg = block_sum(lg, red);
    if (threadIdx.x == 0) {
        float *o = partials + 3 * (int64_t)blockIdx.x;
        o[0] = ok ? acc : NAN;
        o[1] = ok ? l1 : NAN;
        o[2] = ok ? lg : NAN;
    }
}

// loss[o] = (sum of the partials of output o's CTAs, in CTA order) / num_boxes
__global__ void set_loss_finalize_kernel(const __grid_constant__ ProblemTable tab, int count, int num_outputs,
                                         const float *__restrict__ partials, float num_boxes_host,
                                         const float *__restrict__ num_boxes_dev, float *__restrict__ loss) {
    const int o = blockIdx.x * blockDim.x + threadIdx.x;
    if (o >= num_outputs) return;
    double s[3] = {0.0, 0.0, 0.0};
    int64_t b = 0;
    for (int pi = 0; pi < count; ++pi) {
        const int nb = (tab.p[pi].num_queries + kRowsPerBlock - 1) / kRowsPerBlock;
        if (tab.p[pi].output == o)
            for (int k = 0; k < nb; ++k)
                for (int c = 0; c < 3; ++c) s[c] += (double)partials[3 * (b + k) + c];
        b += nb;
    }
    const float nbx = num_boxes_dev ? *num_boxes_dev : num_boxes_host;
    for (int c = 0; c < 3; ++c) loss[3 * o + c] = (float)s[c] / nbx;
}

// d(1 - GIoU)/d(pred cxcywh) with torch autograd's conventions: max / min ties split the gradient half and half,
// clamp(min=0) passes it where the input is >= 0.
__device__ __forceinline__ float dmax_a(float a, float b) { return a > b ? 1.f : (a == b ? 0.5f : 0.f); }  // d max(a,b)/da
__device__ __forceinline__ float dmin_a(float a, float b) { return a < b ? 1.f : (a == b ? 0.5f : 0.f); }

__device__ void giou_loss_grad(const float *pb, const float *gb, float scale, float *d) {
    const Box a = cxcywh_to_xyxy(pb), b = cxcywh_to_xyxy(gb);
    const float aw = a.x1 - a.x0, ah = a.y1 - a.y0;
    const float area1 = aw * ah, area2 = (b.x1 - b.x0) * (b.y1 - b.y0);
    const float iw_raw = fminf(a.x1, b.x1) - fmaxf(a.x0, b.x0), ih_raw = fminf(a.y1, b.y1) - fmaxf(a.y0, b.y0);
    const float iw = clamp0(iw_raw), ih = clamp0(ih_raw);
    const float inter = iw * ih, uni = area1 + area2 - inter;
    const float ew_raw = fmaxf(a.x1, b.x1) - fminf(a.x0, b.x0), eh_raw = fmaxf(a.y1, b.y1) - fminf(a.y0, b.y0);
    const float ew = clamp0(ew_raw), eh = clamp0(eh_raw);
    const float areai = ew * eh;
    // giou = inter / uni - (areai - uni) / areai; the loss is 1 - giou, so every partial below carries -scale
    const float g_giou = -scale;
    const float g_inter_direct = g_giou / uni;
    const float g_uni = g_giou * (-inter / (uni * uni) + 1.f / areai);
    const float g_areai = g_giou * (-uni / (areai * areai));
    const float g_inter = g_inter_direct - g_uni;
    const float g_area1 = g_uni;
    float dx0 = 0.f, dy0 = 0.f, dx1 = 0.f, dy1 = 0.f;
    // area1 = (x1 - x0) (y1 - y0)
    dx1 += g_area1 * ah, dx0 -= g_area1 * ah, dy1 += g_area1 * aw, dy0 -= g_area1 * aw;
    // inter = clamp(min(x1) - max(x0)) * clamp(min(y1) - max(y0))
    const float giw = iw_raw >= 0.f ? g_inter * ih : 0.f, gih = ih_raw >= 0.f ? g_inter * iw : 0.f;
    dx1 += giw * dmin_a(a.x1, b.x1), dx0 -= giw * dmax_a(a.x0, b.x0);
    dy1 += gih * dmin_a(a.y1, b.y1), dy0 -= gih * dmax_a(a.y0, b.y0);
    // areai = clamp(max(x1) - min(x0)) * clamp(max(y1) - min(y0))
    const float gew = ew_raw >= 0.f ? g_areai * eh : 0.f, geh = eh_raw >= 0.f ? g_areai * ew : 0.f;
    dx1 += gew * dmax_a(a.x1, b.x1), dx0 -= gew * dmin_a(a.x0, b.x0);
    dy1 += geh * dmax_a(a.y1, b.y1), dy0 -= geh * dmin_a(a.y0, b.y0);
    // x0 = cx - w/2, x1 = cx + w/2
    d[0] = dx0 + dx1, d[1] = dy0 + dy1, d[2] = 0.5f * (dx1 - dx0), d[3] = 0.5f * (dy1 - dy0);
}

__global__ void __launch_bounds__(kLossThreads) set_loss_backward_kernel(const __grid_constant__ ProblemTable tab, int count,
                                                                         int K, float alpha, float gamma,
                                                                         const int32_t *__restrict__ status,
                                                                         float num_boxes_host,
                                                                         const float *__restrict__ num_boxes_dev,
                                                                         const float *__restrict__ grad_loss) {
    int r0;
    const int pi = locate_block(tab, count, blockIdx.x, r0);
    const sdetr_set_problem &p = tab.p[pi];
    const int rows = min(kRowsPerBlock, p.num_queries - r0);
    __shared__ int gt_of[kRowsPerBlock];
    __shared__ float iou_of[kRowsPerBlock];
    const bool ok = rows_of_block(p, K, r0, rows, gt_of, iou_of) && !(status && status[pi]);
    const float nbx = num_boxes_dev ? *num_boxes_dev : num_boxes_host;
    const float g_cls = grad_loss[3 * p.output] / nbx, g_l1 = grad_loss[3 * p.output + 1] / nbx,
                g_giou = grad_loss[3 * p.output + 2] / nbx;

    // d/dx of w * BCE(x, t) with w and t detached: w (sigma(x) - t)
    for (int e = threadIdx.x; e < rows * K; e += kLossThreads) {
        const int q = e / K, c = e - q * K;
        const float x = p.logits[(int64_t)(r0 + q) * p.logit_stride + c];
        const int g = gt_of[q];
        const float s = sigmoidf(x);
        float d;
        if (g >= 0 && label_of(p, g) == c) {
            const float t = iou_of[q];
            d = t * (s - t);
        } else {
            d = (1.f - alpha) * pow_gamma(s, gamma) * s;
        }
        p.grad_logits[(int64_t)(r0 + q) * K + c] = ok ? g_cls * d : NAN;
    }
    for (int e = threadIdx.x; e < rows * 4; e += kLossThreads) {
        const int q = e >> 2, k = e & 3;
        const int g = gt_of[q];
        float d = 0.f;
        if (g >= 0) {
            const float *pb = p.boxes + (int64_t)(r0 + q) * p.box_stride, *gb = p.gt_boxes + 4 * g;
            const float diff = pb[k] - gb[k];
            float dg[4];
            giou_loss_grad(pb, gb, g_giou, dg);
            d = g_l1 * (diff > 0.f ? 1.f : (diff < 0.f ? -1.f : 0.f)) + dg[k];
        }
        p.grad_boxes[(int64_t)(r0 + q) * 4 + k] = ok ? d : NAN;
    }
}

// ---- host-side checks ----------------------------------------------------------------------------------------------------
int check_problems(const sdetr_set_problem *ps, int count, int num_outputs, int num_classes, bool for_match, bool for_grad,
                   bool costs_given = false) {
    SDETR_REQUIRE(ps || count == 0, SDETR_ERR_INVALID_ARG, "set criterion: null pointer (problems_host)");
    SDETR_REQUIRE(count >= 0 && count <= SDETR_SET_MAX_PROBLEMS, SDETR_ERR_INVALID_ARG,
                  "set criterion: %d problems (0..%d per call)", count, SDETR_SET_MAX_PROBLEMS);
    SDETR_REQUIRE(num_classes >= 1, SDETR_ERR_INVALID_ARG, "set criterion: num_classes %d", num_classes);
    for (int i = 0; i < count; ++i) {
        const sdetr_set_problem &p = ps[i];
        SDETR_REQUIRE(costs_given || (p.logits && p.boxes), SDETR_ERR_INVALID_ARG, "set criterion: null pointer (problem %d logits / boxes)", i);
        SDETR_REQUIRE(p.num_queries >= 1 && p.num_gt >= 0 && p.num_pairs >= 0, SDETR_ERR_INVALID_ARG,
                      "set criterion: problem %d has bad sizes (Q %d, gt %d, pairs %d)", i, p.num_queries, p.num_gt, p.num_pairs);
        SDETR_REQUIRE(costs_given || (p.logit_stride >= num_classes && p.box_stride >= 4), SDETR_ERR_INVALID_ARG,
                      "set criterion: problem %d row strides (%lld, %lld) below (num_classes, 4)", i, (long long)p.logit_stride,
                      (long long)p.box_stride);
        SDETR_REQUIRE(costs_given || p.num_gt == 0 || p.gt_boxes, SDETR_ERR_INVALID_ARG, "set criterion: null pointer (problem %d gt_boxes)", i);
        if (for_match) {
            SDETR_REQUIRE(p.num_queries <= SDETR_SET_MAX_QUERIES, SDETR_ERR_UNSUPPORTED,
                          "set criterion: problem %d has %d queries, the solver holds at most %d", i, p.num_queries,
                          SDETR_SET_MAX_QUERIES);
            SDETR_REQUIRE(p.num_gt <= p.num_queries, SDETR_ERR_UNSUPPORTED,
                          "set criterion: problem %d has %d gts for %d queries (n > Q)", i, p.num_gt, p.num_queries);
            SDETR_REQUIRE(p.num_gt == 0 || (p.src && p.tgt), SDETR_ERR_INVALID_ARG, "set criterion: null pointer (problem %d src / tgt)", i);
        } else {
            SDETR_REQUIRE(p.output >= 0 && p.output < num_outputs, SDETR_ERR_INVALID_ARG,
                          "set criterion: problem %d names output %d of %d", i, p.output, num_outputs);
            SDETR_REQUIRE(p.num_pairs == 0 || (p.src && p.tgt), SDETR_ERR_INVALID_ARG,
                          "set criterion: null pointer (problem %d src / tgt)", i);
            SDETR_REQUIRE(!for_grad || (p.grad_logits && p.grad_boxes), SDETR_ERR_INVALID_ARG,
                          "set criterion: null pointer (problem %d grad_logits / grad_boxes)", i);
        }
    }
    return SDETR_OK;
}

int64_t loss_blocks(const sdetr_set_problem *ps, int count) {
    int64_t b = 0;
    for (int i = 0; i < count; ++i) b += (ps[i].num_queries + kRowsPerBlock - 1) / kRowsPerBlock;
    return b;
}

ProblemTable table_of(const sdetr_set_problem *ps, int count) {
    ProblemTable t;
    memset(&t, 0, sizeof(t));
    for (int i = 0; i < count; ++i) t.p[i] = ps[i];
    return t;
}

PerDeviceOnce g_match_once, g_assign_once;
constexpr int kMatchSmemMax = 38 * SDETR_SET_MAX_QUERIES + 16;

}  // namespace
}  // namespace sdetr

using namespace sdetr;

extern "C" int64_t sdetr_set_match_workspace_floats(const sdetr_set_problem *problems_host, int num_problems) {
    if (!problems_host || num_problems < 0 || num_problems > SDETR_SET_MAX_PROBLEMS) return -1;
    int64_t f = 0;
    for (int i = 0; i < num_problems; ++i) f += (int64_t)problems_host[i].num_gt * problems_host[i].num_queries;
    return f;
}

extern "C" int sdetr_set_match(const sdetr_set_problem *problems_host, int num_problems, int num_classes, float cost_class,
                               float cost_bbox, float cost_giou, float alpha, float gamma, int32_t *status, float *workspace,
                               int64_t workspace_floats, sdetr_stream_t stream) {
    int rc = check_problems(problems_host, num_problems, 0, num_classes, true, false);
    if (rc) return rc;
    SDETR_REQUIRE(status || num_problems == 0, SDETR_ERR_INVALID_ARG, "sdetr_set_match: null pointer (status)");
    const int64_t need = sdetr_set_match_workspace_floats(problems_host, num_problems);
    SDETR_REQUIRE(need == 0 || workspace, SDETR_ERR_INVALID_ARG, "sdetr_set_match: null pointer (workspace)");
    SDETR_REQUIRE(workspace_floats >= need, SDETR_ERR_WORKSPACE, "sdetr_set_match: workspace %lld floats < %lld",
                  (long long)workspace_floats, (long long)need);
    if (num_problems == 0) return SDETR_OK;
    int qmax = 1;
    for (int i = 0; i < num_problems; ++i) qmax = problems_host[i].num_queries > qmax ? problems_host[i].num_queries : qmax;
    const size_t smem = 38 * (size_t)qmax + 16;  // v, spc, u (fp64); path, row4col, col4row (int); two flag bytes; n <= Q
    SDETR_OPT_IN_SMEM(g_match_once, set_match_kernel<true>, kMatchSmemMax, "sdetr_set_match");
    const ProblemTable tab = table_of(problems_host, num_problems);
    set_match_kernel<true><<<num_problems, kSolverThreads, smem, (cudaStream_t)stream>>>(tab, cost_class, cost_bbox, cost_giou,
                                                                                         alpha, gamma, num_classes, status,
                                                                                         workspace);
    return check_launch("sdetr_set_match");
}

extern "C" int sdetr_set_assign(const sdetr_set_problem *problems_host, int num_problems, const float *cost, int64_t cost_floats,
                                int32_t *status, sdetr_stream_t stream) {
    int rc = check_problems(problems_host, num_problems, 0, 1, true, false, true);
    if (rc) return rc;
    SDETR_REQUIRE(status || num_problems == 0, SDETR_ERR_INVALID_ARG, "sdetr_set_assign: null pointer (status)");
    const int64_t need = sdetr_set_match_workspace_floats(problems_host, num_problems);
    SDETR_REQUIRE(need == 0 || cost, SDETR_ERR_INVALID_ARG, "sdetr_set_assign: null pointer (cost)");
    SDETR_REQUIRE(cost_floats >= need, SDETR_ERR_INVALID_ARG, "sdetr_set_assign: cost holds %lld floats, the problems need %lld",
                  (long long)cost_floats, (long long)need);
    if (num_problems == 0) return SDETR_OK;
    int qmax = 1;
    for (int i = 0; i < num_problems; ++i) qmax = problems_host[i].num_queries > qmax ? problems_host[i].num_queries : qmax;
    SDETR_OPT_IN_SMEM(g_assign_once, set_match_kernel<false>, kMatchSmemMax, "sdetr_set_assign");
    const ProblemTable tab = table_of(problems_host, num_problems);
    set_match_kernel<false><<<num_problems, kSolverThreads, 38 * (size_t)qmax + 16, (cudaStream_t)stream>>>(
        tab, 0.f, 0.f, 0.f, 0.f, 0.f, 1, status, const_cast<float *>(cost));
    return check_launch("sdetr_set_assign");
}

extern "C" int64_t sdetr_set_loss_workspace_floats(const sdetr_set_problem *problems_host, int num_problems) {
    if (!problems_host || num_problems < 0 || num_problems > SDETR_SET_MAX_PROBLEMS) return -1;
    return 3 * loss_blocks(problems_host, num_problems);
}

extern "C" int sdetr_set_loss_forward(const sdetr_set_problem *problems_host, int num_problems, int num_outputs,
                                      int num_classes, float alpha, float gamma, const int32_t *status, float num_boxes_host,
                                      const float *num_boxes_dev, float *workspace, int64_t workspace_floats, float *loss,
                                      sdetr_stream_t stream) {
    int rc = check_problems(problems_host, num_problems, num_outputs, num_classes, false, false);
    if (rc) return rc;
    SDETR_REQUIRE(num_outputs >= 1 && num_outputs <= SDETR_SET_MAX_PROBLEMS, SDETR_ERR_INVALID_ARG,
                  "sdetr_set_loss_forward: %d outputs", num_outputs);
    SDETR_REQUIRE(loss, SDETR_ERR_INVALID_ARG, "sdetr_set_loss_forward: null pointer (loss)");
    const int64_t need = 3 * loss_blocks(problems_host, num_problems);
    SDETR_REQUIRE(need == 0 || workspace, SDETR_ERR_INVALID_ARG, "sdetr_set_loss_forward: null pointer (workspace)");
    SDETR_REQUIRE(workspace_floats >= need, SDETR_ERR_WORKSPACE, "sdetr_set_loss_forward: workspace %lld floats < %lld",
                  (long long)workspace_floats, (long long)need);
    const ProblemTable tab = table_of(problems_host, num_problems);
    if (need) {
        set_loss_partials_kernel<<<(unsigned)(need / 3), kLossThreads, 0, (cudaStream_t)stream>>>(tab, num_problems, num_classes,
                                                                                                   alpha, gamma, status, workspace);
        if ((rc = check_launch("sdetr_set_loss_forward (partials)"))) return rc;
    }
    set_loss_finalize_kernel<<<1, 128, 0, (cudaStream_t)stream>>>(tab, num_problems, num_outputs, workspace, num_boxes_host,
                                                                  num_boxes_dev, loss);
    return check_launch("sdetr_set_loss_forward (finalize)");
}

extern "C" int sdetr_set_loss_backward(const sdetr_set_problem *problems_host, int num_problems, int num_outputs,
                                       int num_classes, float alpha, float gamma, const int32_t *status, float num_boxes_host,
                                       const float *num_boxes_dev, const float *grad_loss, sdetr_stream_t stream) {
    int rc = check_problems(problems_host, num_problems, num_outputs, num_classes, false, true);
    if (rc) return rc;
    SDETR_REQUIRE(grad_loss, SDETR_ERR_INVALID_ARG, "sdetr_set_loss_backward: null pointer (grad_loss)");
    const int64_t blocks = loss_blocks(problems_host, num_problems);
    if (!blocks) return SDETR_OK;
    const ProblemTable tab = table_of(problems_host, num_problems);
    set_loss_backward_kernel<<<(unsigned)blocks, kLossThreads, 0, (cudaStream_t)stream>>>(
        tab, num_problems, num_classes, alpha, gamma, status, num_boxes_host, num_boxes_dev, grad_loss);
    return check_launch("sdetr_set_loss_backward");
}
