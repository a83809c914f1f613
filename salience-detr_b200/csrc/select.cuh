// Single-CTA top-k machinery shared by select.cu (sdetr_salience_select, sdetr_topk_desc) and postprocess.cu
// (sdetr_postprocess): radix select of the k-th key, stable compaction of the winners in index order, and a
// shared-memory bitonic sort.  Keys are uint32 whose ascending order is the wanted order (desc_key in common.cuh).
#pragma once
#include "common.cuh"

namespace sdetr {

constexpr int kSortThreads = 1024;
constexpr int kSortWarps = kSortThreads / 32;

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

// Largest k of a single-CTA top-k: its winners (64-bit composites) alias the 32 KB SelectSmem histograms.
constexpr int kTopkFast = 4096;  // (the decoder's two-stage top-3600 takes this path)

}  // namespace sdetr
