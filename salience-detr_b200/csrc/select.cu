// Hierarchical salience token filter for sm_90a -- sdetr_salience_select, sdetr_order_prefixes,
// sdetr_topk_desc.
//
// Reference semantics: models/bricks/salience_transformer.py:146-168 (masked_fill with the batch-global
// minimum, per-level topk, concatenate + descending sort + gather, foreground score) and :366-367
// (top-k of the pre-attention).  The reference expands this into ~25 ATen launches per level plus
// host synchronisations (`topk(k=tensor)`); here the whole filter is five small kernels with no host
// round trip.
//
// Core primitive: a segmented LSD radix sort, one 1024-thread CTA per segment, 8-bit digits, keys are
// fp32 scores mapped to uint32 so that ascending key order == descending score order.  The sort is
// STABLE and the initial order is the token index, so equal scores come out by ascending index -- the
// canonical tie order shared with the oracle (torch leaves it unspecified).  Ranking inside a warp
// uses __match_any_sync; per-warp digit histograms live in shared memory; data ping-pongs through
// global (L2-resident) buffers, so any segment length works (level 0 of the 5-scale config: 67 200).
#include "common.cuh"

namespace sdetr {

constexpr int kSortThreads = 1024;
constexpr int kSortWarps = kSortThreads / 32;

struct LevelTable {
    int L;
    int start[kMaxLevels], size[kMaxLevels], k[kMaxLevels], koff[kMaxLevels + 1];
    int width[kMaxLevels], stride[kMaxLevels];
};

struct SortSmem {
    uint32_t hist[256 * kSortWarps];  // [digit][warp]
    uint32_t warp_tot[kSortWarps];
};

// One radix pass over `n` elements.  load(i) -> (key, val);  results to (dk, dv).
template <class Load>
__device__ __forceinline__ void radix_pass(Load load, int n, int shift, uint32_t *dk, uint32_t *dv, SortSmem &sm) {
    const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
    const int chunk = (((n + kSortWarps - 1) / kSortWarps) + 31) & ~31;
    const int begin = warp * chunk, end = min(n, begin + chunk);
    for (int i = tid; i < 256 * kSortWarps; i += kSortThreads) sm.hist[i] = 0;
    __syncthreads();
    // A: per-warp digit histogram
    for (int base = begin; base < end; base += 32) {
        const int i = base + lane;
        const bool valid = i < end;
        const unsigned act = __ballot_sync(0xffffffffu, valid);
        if (valid) {
            uint32_t key, val;
            load(i, key, val);
            const uint32_t d = (key >> shift) & 255u;
            const unsigned peers = __match_any_sync(act, d);
            if (lane == __ffs(peers) - 1) sm.hist[d * kSortWarps + warp] += __popc(peers);
        }
        __syncwarp();
    }
    __syncthreads();
    // B: exclusive scan over hist in (digit, warp) order; thread t owns entries [8t, 8t+8)
    {
        uint32_t v[8], s = 0;
#pragma unroll
        for (int j = 0; j < 8; ++j) v[j] = sm.hist[tid * 8 + j], s += v[j];
        uint32_t inc = s;
#pragma unroll
        for (int o = 1; o < 32; o <<= 1) {
            const uint32_t t = __shfl_up_sync(0xffffffffu, inc, o);
            if (lane >= o) inc += t;
        }
        if (lane == 31) sm.warp_tot[warp] = inc;
        __syncthreads();
        if (warp == 0) {
            uint32_t w = sm.warp_tot[lane], winc = w;
#pragma unroll
            for (int o = 1; o < 32; o <<= 1) {
                const uint32_t t = __shfl_up_sync(0xffffffffu, winc, o);
                if (lane >= o) winc += t;
            }
            sm.warp_tot[lane] = winc - w;
        }
        __syncthreads();
        uint32_t run = sm.warp_tot[warp] + inc - s;
#pragma unroll
        for (int j = 0; j < 8; ++j) sm.hist[tid * 8 + j] = run, run += v[j];
    }
    __syncthreads();
    // C: stable scatter
    for (int base = begin; base < end; base += 32) {
        const int i = base + lane;
        const bool valid = i < end;
        const unsigned act = __ballot_sync(0xffffffffu, valid);
        if (valid) {
            uint32_t key, val;
            load(i, key, val);
            const uint32_t d = (key >> shift) & 255u;
            const unsigned peers = __match_any_sync(act, d);
            const uint32_t pos = sm.hist[d * kSortWarps + warp] + __popc(peers & ((1u << lane) - 1u));
            dk[pos] = key, dv[pos] = val;
            __syncwarp(peers);
            if (lane == __ffs(peers) - 1) sm.hist[d * kSortWarps + warp] += __popc(peers);
        }
        __syncwarp();
    }
    __syncthreads();  // also makes the global writes of this pass visible to the whole CTA
}

// Full 32-bit sort: load0 -> a -> b -> a -> b.  Result in (kb, vb).
template <class Load0>
__device__ __forceinline__ void block_radix_sort(Load0 load0, int n, uint32_t *ka, uint32_t *va, uint32_t *kb,
                                                 uint32_t *vb, SortSmem &sm) {
    radix_pass(load0, n, 0, ka, va, sm);
    // plain (coherent) loads: these buffers are written by this same kernel
    auto from_a = [=](int i, uint32_t &k, uint32_t &v) { k = ((volatile uint32_t *)ka)[i], v = ((volatile uint32_t *)va)[i]; };
    auto from_b = [=](int i, uint32_t &k, uint32_t &v) { k = ((volatile uint32_t *)kb)[i], v = ((volatile uint32_t *)vb)[i]; };
    radix_pass(from_a, n, 8, kb, vb, sm);
    radix_pass(from_b, n, 16, ka, va, sm);
    radix_pass(from_a, n, 24, kb, vb, sm);
}


// ---- radix select + stable compaction + bitonic sort (the fast path) ------------------------------------------
// A full LSD sort of a 16 800-token level costs ~200 us in one CTA (latency-bound passes).  Selection does
// not need it: (1) find the k-th best key with four 8-bit histogram passes (all 1024 threads, per-warp private
// histograms), (2) emit the winners in index order with one block-wide scan (ties at the threshold: lowest
// indices first), (3) order the <= 16 384 survivors of an image with a shared-memory bitonic sort on unique
// 64-bit (key, index) composites.  Same canonical order as the LSD path, ~10x less time.
struct SelectSmem {
    alignas(8) uint32_t hist[kSortWarps * 256];  // [warp][digit]
    uint32_t total[256];
    uint32_t scan[kSortWarps * 2];
    uint32_t prefix, kth, need;
};

// k-th smallest key (1-based k, 1 <= k <= n) over key(i), i < n.  Returns T and how many keys == T belong
// to the k smallest (the rest of them are cut).  All threads of the CTA must call it.
template <class KeyFn>
__device__ __forceinline__ void radix_select(KeyFn key, int n, int k, uint32_t &T, uint32_t &need_eq, SelectSmem &sm) {
    const int tid = threadIdx.x, warp = tid >> 5;
    uint32_t prefix = 0, mask = 0, remaining = (uint32_t)k;
    for (int shift = 24; shift >= 0; shift -= 8) {
        for (int i = tid; i < kSortWarps * 256; i += kSortThreads) sm.hist[i] = 0;
        __syncthreads();
        for (int i = tid; i < n; i += kSortThreads) {
            const uint32_t kv = key(i);
            if ((kv & mask) == prefix) atomicAdd(&sm.hist[warp * 256 + ((kv >> shift) & 255u)], 1u);
        }
        __syncthreads();
        if (tid < 256) {
            uint32_t t = 0;
#pragma unroll 8
            for (int w = 0; w < kSortWarps; ++w) t += sm.hist[w * 256 + tid];
            sm.total[tid] = t;
        }
        __syncthreads();
        if (warp == 0) {  // 256 bins: each lane scans 8 consecutive bins
            const int lane = tid;
            uint32_t v[8], s = 0;
#pragma unroll
            for (int j = 0; j < 8; ++j) v[j] = sm.total[lane * 8 + j], s += v[j];
            uint32_t inc = s;
#pragma unroll
            for (int o = 1; o < 32; o <<= 1) {
                const uint32_t t = __shfl_up_sync(0xffffffffu, inc, o);
                if (lane >= o) inc += t;
            }
            uint32_t before = inc - s;  // keys in bins below lane*8
            if (remaining > before && remaining <= inc) {  // the k-th key falls into this lane's bins
#pragma unroll
                for (int j = 0; j < 8; ++j) {
                    if (remaining > before && remaining <= before + v[j]) {
                        sm.prefix = prefix | ((uint32_t)(lane * 8 + j) << shift);
                        sm.need = remaining - before;
                    }
                    before += v[j];
                }
            }
        }
        __syncthreads();
        prefix = sm.prefix, remaining = sm.need;
        mask |= 255u << shift;
        __syncthreads();
    }
    T = prefix, need_eq = remaining;
}

// block-wide exclusive scan of a pair of counters (one value pair per thread)
__device__ __forceinline__ void block_scan_pair(uint32_t a, uint32_t b, uint32_t &ea, uint32_t &eb, SelectSmem &sm) {
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    uint32_t ia = a, ib = b;
#pragma unroll
    for (int o = 1; o < 32; o <<= 1) {
        const uint32_t ta = __shfl_up_sync(0xffffffffu, ia, o), tb = __shfl_up_sync(0xffffffffu, ib, o);
        if (lane >= o) ia += ta, ib += tb;
    }
    if (lane == 31) sm.scan[warp * 2] = ia, sm.scan[warp * 2 + 1] = ib;
    __syncthreads();
    if (warp == 0) {
        const uint32_t wa = sm.scan[lane * 2], wb = sm.scan[lane * 2 + 1];
        uint32_t xa = wa, xb = wb;
#pragma unroll
        for (int o = 1; o < 32; o <<= 1) {
            const uint32_t ta = __shfl_up_sync(0xffffffffu, xa, o), tb = __shfl_up_sync(0xffffffffu, xb, o);
            if (lane >= o) xa += ta, xb += tb;
        }
        sm.scan[lane * 2] = xa - wa, sm.scan[lane * 2 + 1] = xb - wb;
    }
    __syncthreads();
    ea = sm.scan[warp * 2] + ia - a, eb = sm.scan[warp * 2 + 1] + ib - b;
    __syncthreads();
}

// Emit, in index order, the k best of key(i): all keys < T plus the first need_eq keys == T.
// emit(position, i, key).  Each thread owns a contiguous run of indices.
template <class KeyFn, class Emit>
__device__ __forceinline__ void stable_compact(KeyFn key, int n, uint32_t T, uint32_t need_eq, Emit emit, SelectSmem &sm) {
    const int ipt = (n + kSortThreads - 1) / kSortThreads;
    const int begin = min(n, (int)threadIdx.x * ipt), end = min(n, begin + ipt);
    uint32_t better = 0, equal = 0;
    for (int i = begin; i < end; ++i) {
        const uint32_t kv = key(i);
        better += kv < T, equal += kv == T;
    }
    uint32_t eb, ee;
    block_scan_pair(better, equal, eb, ee, sm);
    for (int i = begin; i < end; ++i) {
        const uint32_t kv = key(i);
        if (kv < T) {
            emit(eb + min(ee, need_eq), i, kv);
            ++eb;
        } else if (kv == T) {
            if (ee < need_eq) emit(eb + ee, i, kv);
            ++ee;
        }
    }
}

// in-place ascending bitonic sort of N (power of two) 64-bit keys in shared memory, 1024 threads
__device__ __forceinline__ void bitonic_sort_smem(unsigned long long *a, int N) {
    // Compare-exchange distance j <= 32: the 32 pairs a warp owns (pair indices 32B .. 32B+31, for every B it visits) stay
    // inside elements [64B, 64B+64) for this and all following smaller distances, so those stages only need __syncwarp;
    // block-wide barriers remain for j >= 64 and at the hand-over between the two regimes (9 instead of 45 for N = 512).
    auto stage = [&](int k, int j) {
        for (int i = threadIdx.x; i < (N >> 1); i += kSortThreads) {
            const int lo = ((i & ~(j - 1)) << 1) | (i & (j - 1));
            const int hi = lo | j;
            const unsigned long long x = a[lo], y = a[hi];
            const bool up = (lo & k) == 0;
            if ((x > y) == up) a[lo] = y, a[hi] = x;
        }
    };
    for (int k = 2; k <= N; k <<= 1) {
        int j = k >> 1;
        for (; j >= 64; j >>= 1) {
            stage(k, j);
            __syncthreads();
        }
        for (; j > 0; j >>= 1) {
            stage(k, j);
            __syncwarp();
        }
        if (k >= 64) __syncthreads();  // the next k starts with a cross-warp distance (or the caller reads the result)
    }
    __syncthreads();
}

constexpr int kBitonicMax = 16384;  // 128 KB of shared memory

// ---- kernels ---------------------------------------------------------------------------------------------

// per-level minimum over the whole (batch, HW_l) score tensor (salience_transformer.py:146 `score.min()`)
__global__ void __launch_bounds__(1024) level_min_kernel(const float *__restrict__ raw, LevelTable tb, int batch,
                                                         int nv, float *__restrict__ lmin) {
    __shared__ float red[32];
    const int l = blockIdx.x;
    float m = INFINITY;
    const int total = batch * tb.size[l];
    for (int i = threadIdx.x; i < total; i += blockDim.x) {
        const int b = i / tb.size[l], t = i - b * tb.size[l];
        m = fminf(m, __ldg(raw + (int64_t)b * nv + tb.start[l] + t));
    }
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) m = fminf(m, __shfl_xor_sync(0xffffffffu, m, o));
    if ((threadIdx.x & 31) == 0) red[threadIdx.x >> 5] = m;
    __syncthreads();
    if (threadIdx.x < 32) {
        m = red[threadIdx.x];
#pragma unroll
        for (int o = 16; o > 0; o >>= 1) m = fminf(m, __shfl_xor_sync(0xffffffffu, m, o));
        if (threadIdx.x == 0) lmin[l] = m;
    }
}

// foreground_score = where(mask, global min, raw)  (salience_transformer.py:166-168)
__global__ void foreground_kernel(const float *__restrict__ raw, const uint8_t *__restrict__ mask,
                                  const float *__restrict__ lmin, int L, int64_t total, float *__restrict__ fg) {
    float g = INFINITY;
    for (int l = 0; l < L; ++l) g = fminf(g, __ldg(lmin + l));
    for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (int64_t)gridDim.x * blockDim.x)
        fg[i] = mask[i] ? g : raw[i];
}

// segment = (image, level): sort every token of the level by (filled score desc, index asc)
__global__ void __launch_bounds__(kSortThreads) level_sort_kernel(const float *__restrict__ raw,
                                                                  const uint8_t *__restrict__ mask,
                                                                  const float *__restrict__ lmin, LevelTable tb, int nv,
                                                                  uint32_t *ka, uint32_t *va, uint32_t *kb,
                                                                  uint32_t *vb) {
    __shared__ SortSmem sm;
    const int b = blockIdx.x / tb.L, l = blockIdx.x % tb.L;
    const int64_t off = (int64_t)b * nv + tb.start[l];
    const float fill = __ldg(lmin + l);
    const int start = tb.start[l];
    auto load0 = [=](int i, uint32_t &k, uint32_t &v) {
        const float s = __ldg(mask + off + i) ? fill : __ldg(raw + off + i);
        k = desc_key(s), v = (uint32_t)(start + i);
    };
    block_radix_sort(load0, tb.size[l], ka + off, va + off, kb + off, vb + off, sm);
}

// segment = image: merge the per-level top-k_l prefixes by one more sort (cat + sort + gather, :156-158),
// then emit selected_inds / selected_score.
__global__ void __launch_bounds__(kSortThreads) merge_sort_kernel(const uint32_t *lk, const uint32_t *lv, LevelTable tb,
                                                                  int nv, int K, uint32_t *ka, uint32_t *va,
                                                                  uint32_t *kb, uint32_t *vb,
                                                                  int64_t *__restrict__ sel_inds,
                                                                  float *__restrict__ sel_score) {
    __shared__ SortSmem sm;
    const int b = blockIdx.x;
    const int64_t src = (int64_t)b * nv, dst = (int64_t)b * K;
    auto load0 = [=](int j, uint32_t &k, uint32_t &v) {
        int l = 0;
#pragma unroll
        for (int t = 1; t < kMaxLevels; ++t)
            if (t < tb.L && j >= tb.koff[t]) l = t;
        const int64_t s = src + tb.start[l] + (j - tb.koff[l]);
        k = lk[s], v = lv[s];
    };
    block_radix_sort(load0, K, ka + dst, va + dst, kb + dst, vb + dst, sm);
    for (int j = threadIdx.x; j < K; j += blockDim.x) {
        sel_inds[dst + j] = (int64_t)((volatile uint32_t *)vb)[dst + j];
        sel_score[dst + j] = desc_key_inv(((volatile uint32_t *)kb)[dst + j]);
    }
}

// segment = image: order the K selected positions by the spatial cell of their token
__global__ void __launch_bounds__(kSortThreads) tile_order_kernel(const uint32_t *sel_tok /* (b,K) token index */,
                                                                  LevelTable tb, int K, int cell_px, int cells_x,
                                                                  uint32_t *ka, uint32_t *va, uint32_t *kb,
                                                                  uint32_t *vb, int32_t *__restrict__ tile_order) {
    __shared__ SortSmem sm;
    const int b = blockIdx.x;
    const int64_t dst = (int64_t)b * K;
    auto load0 = [=](int j, uint32_t &k, uint32_t &v) {
        const int t = (int)sel_tok[dst + j];
        int l = 0;
#pragma unroll
        for (int u = 1; u < kMaxLevels; ++u)
            if (u < tb.L && t >= tb.start[u]) l = u;
        const int r = t - tb.start[l];
        const int y = r / tb.width[l], x = r - y * tb.width[l];
        const int cy = (y * tb.stride[l] + tb.stride[l] / 2) / cell_px;
        const int cx = (x * tb.stride[l] + tb.stride[l] / 2) / cell_px;
        k = ((uint32_t)(cy * cells_x + cx) << 3) | (uint32_t)l;
        v = (uint32_t)j;
    };
    block_radix_sort(load0, K, ka + dst, va + dst, kb + dst, vb + dst, sm);
    for (int j = threadIdx.x; j < K; j += blockDim.x) tile_order[dst + j] = (int32_t)((volatile uint32_t *)vb)[dst + j];
}

// (image, layer): positions < nq_j of tile_order, order preserved (stream compaction)
struct PrefixTable {
    int layers;
    int nq[16];
    int64_t off[16];
};
__global__ void __launch_bounds__(1024) order_prefix_kernel(const int32_t *__restrict__ tile_order, int K,
                                                            PrefixTable pt, int32_t *__restrict__ out) {
    __shared__ int warp_cnt[32];
    __shared__ int base_s;
    const int b = blockIdx.x, j = blockIdx.y;
    const int nq = pt.nq[j];
    int32_t *dst = out + pt.off[j] + (int64_t)b * nq;
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    if (threadIdx.x == 0) base_s = 0;
    __syncthreads();
    for (int s = 0; s < K; s += blockDim.x) {
        const int i = s + threadIdx.x;
        const int pos = i < K ? __ldg(tile_order + (int64_t)b * K + i) : K;
        const bool keep = pos < nq;
        const unsigned bal = __ballot_sync(0xffffffffu, keep);
        if (lane == 0) warp_cnt[warp] = __popc(bal);
        __syncthreads();
        int before = 0, tot = 0;
        for (int w = 0; w < 32; ++w) {
            const int c = warp_cnt[w];
            before += (w < warp) ? c : 0;
            tot += c;
        }
        const int base = base_s;
        if (keep) dst[base + before + __popc(bal & ((1u << lane) - 1u))] = pos;
        __syncthreads();
        if (threadIdx.x == 0) base_s = base + tot;
        __syncthreads();
    }
}

// generic segmented top-k (descending, ties by position): salience_transformer.py:366-367
__global__ void __launch_bounds__(kSortThreads) topk_kernel(const float *__restrict__ score, int n, int k, uint32_t *ka,
                                                            uint32_t *va, uint32_t *kb, uint32_t *vb,
                                                            int64_t *__restrict__ out) {
    __shared__ SortSmem sm;
    const int64_t off = (int64_t)blockIdx.x * n;
    auto load0 = [=](int i, uint32_t &key, uint32_t &v) { key = desc_key(__ldg(score + off + i)), v = (uint32_t)i; };
    block_radix_sort(load0, n, ka + off, va + off, kb + off, vb + off, sm);
    for (int j = threadIdx.x; j < k; j += blockDim.x)
        out[(int64_t)blockIdx.x * k + j] = (int64_t)((volatile uint32_t *)vb)[off + j];
}


// ---- fast-path kernels ---------------------------------------------------------------------------------------
// (image, level): top-k_l selection -> candidates (key, token) in index order at [b*K + koff[l] ...)
__global__ void __launch_bounds__(kSortThreads) level_select_kernel(const float *__restrict__ raw,
                                                                    const uint8_t *__restrict__ mask,
                                                                    const float *__restrict__ lmin, LevelTable tb, int nv,
                                                                    int K, uint32_t *__restrict__ ck,
                                                                    uint32_t *__restrict__ cv) {
    __shared__ SelectSmem sm;
    const int b = blockIdx.x / tb.L, l = blockIdx.x % tb.L;
    const int k = tb.k[l];
    if (k == 0) return;
    const int64_t off = (int64_t)b * nv + tb.start[l];
    const float fill = __ldg(lmin + l);
    auto key = [=](int i) { return desc_key(__ldg(mask + off + i) ? fill : __ldg(raw + off + i)); };
    uint32_t T, need;
    radix_select(key, tb.size[l], k, T, need, sm);
    const int64_t dst = (int64_t)b * K + tb.koff[l];
    const uint32_t start = (uint32_t)tb.start[l];
    stable_compact(key, tb.size[l], T, need,
                   [=](uint32_t pos, int i, uint32_t kv) { ck[dst + pos] = kv, cv[dst + pos] = start + (uint32_t)i; }, sm);
}

// image: order the K candidates by (score desc, token asc) and emit selected_inds / selected_score; then, if
// requested, the spatial-cell processing order of the sorted list.  K <= kBitonicMax.
__global__ void __launch_bounds__(kSortThreads) merge_bitonic_kernel(const uint32_t *__restrict__ ck,
                                                                     const uint32_t *__restrict__ cv, LevelTable tb,
                                                                     int K, int N, int cell_px, int cells_x,
                                                                     int64_t *__restrict__ sel_inds,
                                                                     float *__restrict__ sel_score,
                                                                     int32_t *__restrict__ tile_order) {
    extern __shared__ unsigned long long keys[];
    const int b = blockIdx.x;
    const int64_t base = (int64_t)b * K;
    for (int j = threadIdx.x; j < N; j += kSortThreads)
        keys[j] = j < K ? ((unsigned long long)ck[base + j] << 32) | cv[base + j] : ~0ull;
    __syncthreads();
    bitonic_sort_smem(keys, N);
    for (int j = threadIdx.x; j < K; j += kSortThreads) {
        const unsigned long long e = keys[j];
        sel_inds[base + j] = (int64_t)(e & 0xffffffffull);
        sel_score[base + j] = desc_key_inv((uint32_t)(e >> 32));
    }
    if (!tile_order) return;
    __syncthreads();
    for (int j = threadIdx.x; j < N; j += kSortThreads) {
        unsigned long long e = ~0ull;
        if (j < K) {
            const int t = (int)(keys[j] & 0xffffffffull);
            int l = 0;
#pragma unroll
            for (int u = 1; u < kMaxLevels; ++u)
                if (u < tb.L && t >= tb.start[u]) l = u;
            const int r = t - tb.start[l];
            const int y = r / tb.width[l], x = r - y * tb.width[l];
            const int cy = (y * tb.stride[l] + tb.stride[l] / 2) / cell_px;
            const int cx = (x * tb.stride[l] + tb.stride[l] / 2) / cell_px;
            e = ((unsigned long long)(((uint32_t)(cy * cells_x + cx) << 3) | (uint32_t)l) << 32) | (uint32_t)j;
        }
        __syncthreads();  // every thread has read keys[j] of this round before anyone overwrites it
        keys[j] = e;
    }
    __syncthreads();
    bitonic_sort_smem(keys, N);
    for (int j = threadIdx.x; j < K; j += kSortThreads) tile_order[base + j] = (int32_t)(keys[j] & 0xffffffffull);
}

// segment: top-k (k <= 2048) by radix select + compaction + bitonic sort of the winners
constexpr int kTopkFast = 4096;  // winners alias the 32 KB histogram buffer (the decoder's two-stage top-3600 takes this path)
__global__ void __launch_bounds__(kSortThreads) topk_select_kernel(const float *__restrict__ score, int n, int k, int N,
                                                                   int64_t *__restrict__ out) {
    __shared__ SelectSmem sm;
    static_assert(sizeof(sm.hist) >= kTopkFast * sizeof(unsigned long long), "winner buffer aliases the histograms");
    unsigned long long *win = reinterpret_cast<unsigned long long *>(sm.hist);  // free once radix_select returned
    const int64_t off = (int64_t)blockIdx.x * n;
    auto key = [=](int i) { return desc_key(__ldg(score + off + i)); };
    uint32_t T, need;
    radix_select(key, n, k, T, need, sm);
    for (int j = threadIdx.x; j < N; j += kSortThreads) win[j] = ~0ull;
    __syncthreads();
    stable_compact(key, n, T, need,
                   [&](uint32_t pos, int i, uint32_t kv) { win[pos] = ((unsigned long long)kv << 32) | (uint32_t)i; }, sm);
    __syncthreads();
    bitonic_sort_smem(win, N);
    for (int j = threadIdx.x; j < k; j += kSortThreads) out[(int64_t)blockIdx.x * k + j] = (int64_t)(win[j] & 0xffffffffull);
}


// ---- fastest path: per-(image, level) select + sort, rank merge across levels, counting tile order ------------
// The single-CTA bitonic sort of all K candidates is bound by ONE SM's shared-memory bandwidth (K*8 B read +
// written per stage, 105 stages at K = 11 363 -> ~170 us).  Sorting each level's winners inside the CTA that
// selected them (b*L CTAs in parallel, <= 8192 elements each) and merging by rank -- every candidate's final
// position is its rank in its own list plus binary-search ranks in the other lists, one thread per candidate,
// all SMs -- gives the same order ~5x faster.
// A level's winners are further cut into SLICES of at most kSlice candidates (by position in index order), one CTA per
// (image, slice): every CTA of a level redoes the (cheap, L2-resident) threshold search and prefix scan over the whole
// level but compacts and sorts only its own slice -- a 2048-element bitonic sort (66 stages) instead of an 8192-element
// one (91 stages on 4x the data) on the critical path, and 16 CTAs instead of 8 at config 2.  The rank merge below does
// not care how the candidates were partitioned into sorted lists.
constexpr int kSlice = 2048;
constexpr int kMaxLists = 32;

struct ListTable {
    int n;
    int level[kMaxLists], lo[kMaxLists], cnt[kMaxLists], off[kMaxLists + 1];  // winners [lo, lo+cnt) of `level` -> sorted[off ..]
};

__global__ void __launch_bounds__(kSortThreads) level_select_sort_kernel(const float *__restrict__ raw,
                                                                         const uint8_t *__restrict__ mask,
                                                                         const float *__restrict__ lmin, LevelTable tb,
                                                                         ListTable lt, int nv, int K,
                                                                         unsigned long long *__restrict__ sorted) {
    __shared__ SelectSmem sm;
    static_assert(sizeof(sm.hist) >= kSlice * sizeof(unsigned long long), "slice buffer aliases the histograms");
    unsigned long long *comp = reinterpret_cast<unsigned long long *>(sm.hist);  // free once radix_select returned
    const int b = blockIdx.x / lt.n, li = blockIdx.x % lt.n;
    const int l = lt.level[li], k = tb.k[l];
    const uint32_t lo = (uint32_t)lt.lo[li], cnt = (uint32_t)lt.cnt[li];
    int N = 1;
    while (N < (int)cnt) N <<= 1;
    const int64_t off = (int64_t)b * nv + tb.start[l];
    const float fill = __ldg(lmin + l);
    auto key = [=](int i) { return desc_key(__ldg(mask + off + i) ? fill : __ldg(raw + off + i)); };
    uint32_t T, need;
    radix_select(key, tb.size[l], k, T, need, sm);
    __syncthreads();
    for (int j = cnt + threadIdx.x; j < N; j += kSortThreads) comp[j] = ~0ull;
    const uint32_t start = (uint32_t)tb.start[l];
    stable_compact(key, tb.size[l], T, need,
                   [&](uint32_t pos, int i, uint32_t kv) {
                       if (pos - lo < cnt) comp[pos - lo] = ((unsigned long long)kv << 32) | (start + (uint32_t)i);
                   },
                   sm);
    __syncthreads();
    bitonic_sort_smem(comp, N);
    const int64_t dst = (int64_t)b * K + lt.off[li];
    for (int j = threadIdx.x; j < (int)cnt; j += kSortThreads) sorted[dst + j] = comp[j];
}

__device__ __forceinline__ int lower_bound_u64(const unsigned long long *a, int n, unsigned long long key) {
    int lo = 0, hi = n;
    while (lo < hi) {
        const int mid = (lo + hi) >> 1;
        if (a[mid] < key) lo = mid + 1;
        else hi = mid;
    }
    return lo;
}

__global__ void __launch_bounds__(256) merge_rank_kernel(const unsigned long long *__restrict__ sorted, ListTable lt, int K,
                                                         int batch, int64_t *__restrict__ sel_inds,
                                                         float *__restrict__ sel_score) {
    const int64_t g = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (g >= (int64_t)batch * K) return;
    const int b = (int)(g / K), j = (int)(g - (int64_t)b * K);
    int li = 0;
    for (int t = 1; t < lt.n; ++t)
        if (j >= lt.off[t]) li = t;
    const unsigned long long *base = sorted + (int64_t)b * K;
    const unsigned long long key = base[j];
    int pos = j - lt.off[li];
    for (int t = 0; t < lt.n; ++t)
        if (t != li) pos += lower_bound_u64(base + lt.off[t], lt.cnt[t], key);
    sel_inds[(int64_t)b * K + pos] = (int64_t)(key & 0xffffffffull);
    sel_score[(int64_t)b * K + pos] = desc_key_inv((uint32_t)(key >> 32));
}

// image: processing order = counting sort of the selected positions by (spatial cell, level).  The order inside
// a bin is whatever the atomics produce; MSDA results do not depend on the processing order.
__global__ void __launch_bounds__(kSortThreads) tile_count_kernel(const int64_t *__restrict__ sel_inds, LevelTable tb, int K,
                                                                  int cell_px, int cells_x, int bins,
                                                                  int32_t *__restrict__ tile_order) {
    extern __shared__ uint32_t hist[];  // bins + 1
    __shared__ uint32_t wsum[kSortWarps];
    const int b = blockIdx.x;
    const int64_t base = (int64_t)b * K;
    auto bin_of = [&](int j) {
        const int t = (int)sel_inds[base + j];
        int l = 0;
#pragma unroll
        for (int u = 1; u < kMaxLevels; ++u)
            if (u < tb.L && t >= tb.start[u]) l = u;
        const int r = t - tb.start[l];
        const int y = r / tb.width[l], x = r - y * tb.width[l];
        const int cy = (y * tb.stride[l] + tb.stride[l] / 2) / cell_px;
        const int cx = (x * tb.stride[l] + tb.stride[l] / 2) / cell_px;
        return min(bins - 1, ((cy * cells_x + cx) << 3) | l);
    };
    for (int i = threadIdx.x; i < bins; i += kSortThreads) hist[i] = 0;
    __syncthreads();
    for (int j = threadIdx.x; j < K; j += kSortThreads) atomicAdd(&hist[bin_of(j)], 1u);
    __syncthreads();
    // exclusive scan of `bins` counters: each thread owns a contiguous run
    const int per = (bins + kSortThreads - 1) / kSortThreads;
    const int lo = min(bins, (int)threadIdx.x * per), hi = min(bins, lo + per);
    uint32_t s = 0;
    for (int i = lo; i < hi; ++i) s += hist[i];
    uint32_t inc = s;
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
#pragma unroll
    for (int o = 1; o < 32; o <<= 1) {
        const uint32_t t = __shfl_up_sync(0xffffffffu, inc, o);
        if (lane >= o) inc += t;
    }
    if (lane == 31) wsum[warp] = inc;
    __syncthreads();
    if (warp == 0) {
        const uint32_t w = wsum[lane];
        uint32_t x = w;
#pragma unroll
        for (int o = 1; o < 32; o <<= 1) {
            const uint32_t t = __shfl_up_sync(0xffffffffu, x, o);
            if (lane >= o) x += t;
        }
        wsum[lane] = x - w;
    }
    __syncthreads();
    uint32_t run = wsum[warp] + inc - s;
    for (int i = lo; i < hi; ++i) {
        const uint32_t c = hist[i];
        hist[i] = run;
        run += c;
    }
    __syncthreads();
    for (int j = threadIdx.x; j < K; j += kSortThreads) tile_order[base + atomicAdd(&hist[bin_of(j)], 1u)] = j;
}

static int next_pow2(int x) {
    int p = 1;
    while (p < x) p <<= 1;
    return p;
}

static inline size_t align256(size_t x) { return (x + 255) & ~(size_t)255; }

}  // namespace sdetr

using namespace sdetr;

extern "C" size_t sdetr_salience_select_workspace(int batch, int num_value, int num_levels) {
    (void)num_levels;
    // level minima + 4 level-sort buffers (b*Nv u32) + 4 merge/tile-sort buffers (b*K <= b*Nv u32)
    return 256 + 8 * align256((size_t)batch * num_value * sizeof(uint32_t));
}

extern "C" int sdetr_salience_select(const float *raw_score, const uint8_t *mask, const int32_t *level_start_host,
                                     const int32_t *level_size_host, const int32_t *level_k_host,
                                     const int32_t *level_width_host, const int32_t *level_stride_host, int cell_px,
                                     int batch, int num_value, int num_levels, int64_t *selected_inds,
                                     float *selected_score, float *foreground_score, int32_t *tile_order,
                                     void *workspace, size_t workspace_bytes, sdetr_stream_t stream) {
    SDETR_REQUIRE(raw_score && mask && level_start_host && level_size_host && level_k_host && selected_inds &&
                      selected_score && foreground_score && workspace,
                  SDETR_ERR_INVALID_ARG, "salience_select: null pointer");
    SDETR_REQUIRE(batch > 0 && num_value > 0 && num_levels > 0 && num_levels <= kMaxLevels, SDETR_ERR_INVALID_ARG,
                  "salience_select: bad sizes (batch %d, num_value %d, levels %d)", batch, num_value, num_levels);
    SDETR_REQUIRE(workspace_bytes >= sdetr_salience_select_workspace(batch, num_value, num_levels),
                  SDETR_ERR_WORKSPACE, "salience_select: workspace too small");
    SDETR_REQUIRE(!tile_order || (level_width_host && level_stride_host && cell_px > 0), SDETR_ERR_INVALID_ARG,
                  "salience_select: tile_order needs level widths/strides and cell_px");
    LevelTable tb{};
    tb.L = num_levels;
    int K = 0, cover = 0, max_w_px = 0;
    for (int l = 0; l < num_levels; ++l) {
        tb.start[l] = level_start_host[l], tb.size[l] = level_size_host[l], tb.k[l] = level_k_host[l];
        tb.koff[l] = K;
        SDETR_REQUIRE(tb.k[l] >= 0 && tb.k[l] <= tb.size[l] && tb.start[l] == cover, SDETR_ERR_INVALID_ARG,
                      "salience_select: level %d: k=%d size=%d start=%d", l, tb.k[l], tb.size[l], tb.start[l]);
        K += tb.k[l];
        cover += tb.size[l];
        if (tile_order) {
            tb.width[l] = level_width_host[l], tb.stride[l] = level_stride_host[l];
            SDETR_REQUIRE(tb.width[l] > 0 && tb.stride[l] > 0, SDETR_ERR_INVALID_ARG, "salience_select: bad width/stride");
            if (tb.width[l] * tb.stride[l] > max_w_px) max_w_px = tb.width[l] * tb.stride[l];
        }
    }
    tb.koff[num_levels] = K;
    SDETR_REQUIRE(cover == num_value, SDETR_ERR_INVALID_ARG, "salience_select: levels cover %d of %d tokens", cover,
                  num_value);
    cudaStream_t s = (cudaStream_t)stream;
    char *ws = (char *)workspace;
    float *lmin = (float *)ws;
    const size_t bufsz = align256((size_t)batch * num_value * sizeof(uint32_t));
    uint32_t *buf[8];
    for (int i = 0; i < 8; ++i) buf[i] = (uint32_t *)(ws + 256 + i * bufsz);

    level_min_kernel<<<num_levels, 1024, 0, s>>>(raw_score, tb, batch, num_value, lmin);
    int rc = check_launch("salience_select/level_min");
    if (rc) return rc;
    const int64_t total = (int64_t)batch * num_value;
    const int64_t fg_cap = 8 * (int64_t)sm_count(), fg_blocks = (total + 255) / 256 < fg_cap ? (total + 255) / 256 : fg_cap;
    foreground_kernel<<<(unsigned)fg_blocks, 256, 0, s>>>(raw_score, mask, lmin, num_levels, total, foreground_score);
    if ((rc = check_launch("salience_select/foreground"))) return rc;
    if (K == 0) return SDETR_OK;
    int kmax = 0;
    for (int l = 0; l < num_levels; ++l) kmax = tb.k[l] > kmax ? tb.k[l] : kmax;
    const int cells_x = tile_order ? (max_w_px + cell_px - 1) / cell_px + 1 : 1;
    int bins = 0;
    if (tile_order) {
        int max_h_px = 0;
        for (int l = 0; l < num_levels; ++l) {
            const int hpx = (tb.size[l] / tb.width[l]) * tb.stride[l];
            max_h_px = hpx > max_h_px ? hpx : max_h_px;
        }
        bins = (((max_h_px + cell_px - 1) / cell_px + 1) * cells_x) << 3;
    }
    ListTable lt{};
    for (int l = 0; l < num_levels; ++l)
        for (int lo = 0; lo < tb.k[l]; lo += kSlice) {
            if (lt.n < kMaxLists) {
                lt.level[lt.n] = l, lt.lo[lt.n] = lo, lt.cnt[lt.n] = tb.k[l] - lo < kSlice ? tb.k[l] - lo : kSlice;
                lt.off[lt.n] = tb.koff[l] + lo;
            }
            ++lt.n;
        }
    if (lt.n <= kMaxLists && bins <= 12000) {
        // fastest path: select + sort per (image, slice of a level), rank merge, counting-sort processing order
        lt.off[lt.n] = K;
        unsigned long long *sorted = reinterpret_cast<unsigned long long *>(buf[0]);  // b*K u64 <= two u32 buffers
        level_select_sort_kernel<<<batch * lt.n, kSortThreads, 0, s>>>(raw_score, mask, lmin, tb, lt, num_value, K, sorted);
        if ((rc = check_launch("salience_select/level_select_sort"))) return rc;
        const int64_t cand = (int64_t)batch * K;
        merge_rank_kernel<<<(unsigned)((cand + 255) / 256), 256, 0, s>>>(sorted, lt, K, batch, selected_inds, selected_score);
        if ((rc = check_launch("salience_select/merge_rank"))) return rc;
        if (tile_order) {
            tile_count_kernel<<<batch, kSortThreads, (size_t)(bins + 1) * sizeof(uint32_t), s>>>(selected_inds, tb, K, cell_px,
                                                                                                cells_x, bins, tile_order);
            if ((rc = check_launch("salience_select/tile_count"))) return rc;
        }
        return SDETR_OK;
    }
    if (K <= kBitonicMax) {
        // radix select per (image, level) -> one bitonic merge per image (+ processing order)
        level_select_kernel<<<batch * num_levels, kSortThreads, 0, s>>>(raw_score, mask, lmin, tb, num_value, K, buf[0],
                                                                        buf[1]);
        if ((rc = check_launch("salience_select/level_select"))) return rc;
        const int N = next_pow2(K);
        const size_t smem = (size_t)N * sizeof(unsigned long long);
        static PerDeviceOnce once_b;
        SDETR_OPT_IN_SMEM(once_b, merge_bitonic_kernel, kBitonicMax * (int)sizeof(unsigned long long), "salience_select");
        merge_bitonic_kernel<<<batch, kSortThreads, smem, s>>>(buf[0], buf[1], tb, K, N, tile_order ? cell_px : 1,
                                                               cells_x, selected_inds, selected_score, tile_order);
        return check_launch("salience_select/merge_bitonic");
    }
    // large-K fallback (e.g. the 5-scale geometry, K = 45 570): segmented LSD radix sorts through global memory
    level_sort_kernel<<<batch * num_levels, kSortThreads, 0, s>>>(raw_score, mask, lmin, tb, num_value, buf[0], buf[1],
                                                                  buf[2], buf[3]);
    if ((rc = check_launch("salience_select/level_sort"))) return rc;
    merge_sort_kernel<<<batch, kSortThreads, 0, s>>>(buf[2], buf[3], tb, num_value, K, buf[4], buf[5], buf[6], buf[7],
                                                     selected_inds, selected_score);
    if ((rc = check_launch("salience_select/merge_sort"))) return rc;
    if (tile_order) {
        const int cells_x = (max_w_px + cell_px - 1) / cell_px + 1;
        // sorted token indices are in buf[7]; reuse the level-sort buffers as ping-pong space
        tile_order_kernel<<<batch, kSortThreads, 0, s>>>(buf[7], tb, K, cell_px, cells_x, buf[0], buf[1], buf[2], buf[3],
                                                         tile_order);
        if ((rc = check_launch("salience_select/tile_order"))) return rc;
    }
    return SDETR_OK;
}

extern "C" int sdetr_order_prefixes(const int32_t *tile_order, int batch, int K, int num_layers,
                                    const int32_t *nq_host, const int64_t *order_offset_host, int32_t *out_orders,
                                    sdetr_stream_t stream) {
    SDETR_REQUIRE(tile_order && nq_host && order_offset_host && out_orders, SDETR_ERR_INVALID_ARG,
                  "order_prefixes: null pointer");
    SDETR_REQUIRE(batch > 0 && K > 0 && num_layers > 0 && num_layers <= 16, SDETR_ERR_INVALID_ARG,
                  "order_prefixes: bad sizes");
    PrefixTable pt{};
    pt.layers = num_layers;
    for (int j = 0; j < num_layers; ++j) {
        SDETR_REQUIRE(nq_host[j] >= 0 && nq_host[j] <= K, SDETR_ERR_INVALID_ARG, "order_prefixes: nq[%d]=%d > K=%d", j,
                      nq_host[j], K);
        pt.nq[j] = nq_host[j], pt.off[j] = order_offset_host[j];
    }
    order_prefix_kernel<<<dim3(batch, num_layers), 1024, 0, (cudaStream_t)stream>>>(tile_order, K, pt, out_orders);
    return check_launch("order_prefixes");
}

extern "C" size_t sdetr_topk_workspace(int segments, int n) {
    return 4 * align256((size_t)segments * n * sizeof(uint32_t));
}

extern "C" int sdetr_topk_desc(const float *score, int segments, int n, int k, int64_t *topk_index, void *workspace,
                               size_t workspace_bytes, sdetr_stream_t stream) {
    SDETR_REQUIRE(score && topk_index && workspace, SDETR_ERR_INVALID_ARG, "topk_desc: null pointer");
    SDETR_REQUIRE(segments > 0 && n > 0 && k >= 0 && k <= n, SDETR_ERR_INVALID_ARG, "topk_desc: k=%d n=%d", k, n);
    SDETR_REQUIRE(workspace_bytes >= sdetr_topk_workspace(segments, n), SDETR_ERR_WORKSPACE,
                  "topk_desc: workspace too small");
    if (k == 0) return SDETR_OK;
    if (k <= kTopkFast) {
        topk_select_kernel<<<segments, kSortThreads, 0, (cudaStream_t)stream>>>(score, n, k, next_pow2(k), topk_index);
        return check_launch("topk_desc/select");
    }
    const size_t bufsz = align256((size_t)segments * n * sizeof(uint32_t));
    char *ws = (char *)workspace;
    topk_kernel<<<segments, kSortThreads, 0, (cudaStream_t)stream>>>(score, n, k, (uint32_t *)ws,
                                                                     (uint32_t *)(ws + bufsz),
                                                                     (uint32_t *)(ws + 2 * bufsz),
                                                                     (uint32_t *)(ws + 3 * bufsz), topk_index);
    return check_launch("topk_desc");
}
