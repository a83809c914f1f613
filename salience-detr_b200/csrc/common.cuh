// Shared helpers of the sm_90a kernels behind include/sdetr_b200.h.
#pragma once
#include <cuda_runtime.h>
#include <float.h>
#include <stdint.h>
#include <stdio.h>

#include <atomic>

#include "../../include/sdetr_b200.h"

namespace sdetr {

constexpr int kMaxLevels = 8;

// thread-local error string + process-wide launch counter (defined in api.cu)
void set_error(const char *fmt, ...);
void count_launch(int n = 1);

inline int check_launch(const char *what) {
    cudaError_t e = cudaGetLastError();
    if (e != cudaSuccess) {
        set_error("%s: %s", what, cudaGetErrorString(e));
        return SDETR_ERR_CUDA;
    }
    count_launch();
    return SDETR_OK;
}

#define SDETR_REQUIRE(cond, code, ...)  \
    do {                                \
        if (!(cond)) {                  \
            sdetr::set_error(__VA_ARGS__); \
            return (code);              \
        }                               \
    } while (0)

// Per-DEVICE one-time setup (cudaFuncSetAttribute opt-ins are per device): a bit per device ordinal, set after the
// attribute call succeeded.  Two threads racing on the first use both set the (idempotent) attribute.
struct PerDeviceOnce {
    std::atomic<uint64_t> done[4];
    bool need(int &dev) {
        if (cudaGetDevice(&dev) != cudaSuccess) dev = 0;
        return !((done[(dev >> 6) & 3].load(std::memory_order_acquire) >> (dev & 63)) & 1ull);
    }
    void mark(int dev) { done[(dev >> 6) & 3].fetch_or(1ull << (dev & 63), std::memory_order_release); }
};
#define SDETR_OPT_IN_SMEM(once, kernel, bytes, what)                                                                  \
    do {                                                                                                              \
        int dev_;                                                                                                     \
        if ((once).need(dev_)) {                                                                                      \
            cudaError_t e_ = cudaFuncSetAttribute(kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)(bytes)); \
            SDETR_REQUIRE(e_ == cudaSuccess, SDETR_ERR_CUDA, "%s: smem attribute: %s", what, cudaGetErrorString(e_)); \
            (once).mark(dev_);                                                                                        \
        }                                                                                                             \
    } while (0)

int sm_count();  // SMs of the CURRENT device (cached per device ordinal; api.cu)
int persistent_ctas();  // CTAs of a persistent one-per-SM kernel: sm_count(), or the cap of sdetr_set_persistent_ctas

inline bool aligned16(const void *p) { return (reinterpret_cast<uintptr_t>(p) & 15u) == 0; }

// ---- device helpers -------------------------------------------------------------------------------
// torch.relu: a NaN propagates (as the canonical NaN; fmaxf would return the 0).  One max.NaN instruction, the cost of fmaxf.
__device__ __forceinline__ float relu_nan(float x) {
    float r;
    asm("max.NaN.f32 %0, %1, 0f00000000;" : "=f"(r) : "f"(x));
    return r;
}
// torch.max: a NaN operand propagates (as the canonical NaN; fmaxf would return the other operand).  One max.NaN instruction.
__device__ __forceinline__ float fmax_nan(float a, float b) {
    float r;
    asm("max.NaN.f32 %0, %1, %2;" : "=f"(r) : "f"(a), "f"(b));
    return r;
}

__device__ __forceinline__ float4 ldg_f4(const float *p) { return __ldg(reinterpret_cast<const float4 *>(p)); }

// streaming (read-once) 128-bit load / store: keep L1 for the gathered value tiles
__device__ __forceinline__ float4 ld_stream_f4(const float *p) {
    float4 r;
    asm volatile("ld.global.nc.L1::no_allocate.v4.f32 {%0,%1,%2,%3}, [%4];"
                 : "=f"(r.x), "=f"(r.y), "=f"(r.z), "=f"(r.w)
                 : "l"(p));
    return r;
}
__device__ __forceinline__ void st_stream_f4(float *p, const float4 &v) {
    asm volatile("st.global.L1::no_allocate.v4.f32 [%0], {%1,%2,%3,%4};" ::"l"(p), "f"(v.x), "f"(v.y), "f"(v.z),
                 "f"(v.w)
                 : "memory");
}

// ---- max|x| in one launch (sdetr_pow2_scale, the deterministic MSDA backward's scale) ----------------------------------
// This thread's grid-stride share of max|x[0, n)|.  fmaxf skips NaN: `nonfinite` is set when a NaN or an infinity is seen.
// 16-byte aligned x is read with 128-bit streaming loads, any other x element by element.  FINITE_ONLY: infinities count
// as 0 too (the maximum of the finite entries).
template <bool FINITE_ONLY>
__device__ __forceinline__ float abs_for_max(float v) {
    const float a = fabsf(v);
    return FINITE_ONLY && !(a <= FLT_MAX) ? 0.f : a;
}
template <bool FINITE_ONLY = false>
__device__ __forceinline__ float thread_absmax(const float *__restrict__ x, int64_t n, bool &nonfinite) {
    float m = 0.f;
    bool bad = false;
    const int64_t t = (int64_t)blockIdx.x * blockDim.x + threadIdx.x, nt = (int64_t)gridDim.x * blockDim.x;
    if ((reinterpret_cast<uintptr_t>(x) & 15u) == 0) {
        for (int64_t i = t * 4; i < n; i += nt * 4) {
            if (i + 3 < n) {
                const float4 v = ld_stream_f4(x + i);
                m = fmaxf(m, fmaxf(fmaxf(abs_for_max<FINITE_ONLY>(v.x), abs_for_max<FINITE_ONLY>(v.y)),
                                   fmaxf(abs_for_max<FINITE_ONLY>(v.z), abs_for_max<FINITE_ONLY>(v.w))));
                bad |= !(fabsf(v.x) <= FLT_MAX) | !(fabsf(v.y) <= FLT_MAX) | !(fabsf(v.z) <= FLT_MAX) | !(fabsf(v.w) <= FLT_MAX);
            } else {
                for (int64_t j = i; j < n; ++j) m = fmaxf(m, abs_for_max<FINITE_ONLY>(x[j])), bad |= !(fabsf(x[j]) <= FLT_MAX);
            }
        }
    } else {
        for (int64_t i = t; i < n; i += nt) m = fmaxf(m, abs_for_max<FINITE_ONLY>(x[i])), bad |= !(fabsf(x[i]) <= FLT_MAX);
    }
    nonfinite |= bad;
    return m;
}
// Maximum of m over the block, in thread 0 (blockDim.x a multiple of 32).  Safe to call repeatedly in one kernel.
__device__ __forceinline__ float block_max(float m) {
    __shared__ float wm[32];
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) m = fmaxf(m, __shfl_xor_sync(0xffffffffu, m, o));
    __syncthreads();  // wm may still be read by an earlier call
    if ((threadIdx.x & 31) == 0) wm[threadIdx.x >> 5] = m;
    __syncthreads();
    if (threadIdx.x == 0)
        for (int w = 1; w < (int)(blockDim.x >> 5); ++w) m = fmaxf(m, wm[w]);
    return m;
}

// fp32 -> uint32 whose ascending order is the DESCENDING order of the floats, as torch.sort(descending=True) orders
// them: -0 == +0, and every NaN (either sign, any payload) is one key that comes first.
__device__ __forceinline__ uint32_t desc_key(float f) {
    if (f != f) return 0u;
    if (f == 0.f) f = 0.f;  // canonicalise -0
    uint32_t u = __float_as_uint(f);
    u = (u & 0x80000000u) ? ~u : (u | 0x80000000u);  // ascending-orderable
    return ~u;  // +inf -> 0x007fffff; no number maps to 0, the key of the NaNs
}
// the inverse for every key but those of a zero (gives +0) and of the NaNs (gives the NaN 0x7fffffff)
__device__ __forceinline__ float desc_key_inv(uint32_t k) {
    uint32_t u = ~k;
    u = (u & 0x80000000u) ? (u & 0x7fffffffu) : ~u;
    return __uint_as_float(u);
}

}  // namespace sdetr
