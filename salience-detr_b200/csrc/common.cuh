// Shared helpers of the sm_90a kernels behind include/sdetr_b200.h.
#pragma once
#include <cuda_runtime.h>
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

// fp32 -> uint32 whose ascending order is the DESCENDING order of the floats (-0 == +0, NaN first).
__device__ __forceinline__ uint32_t desc_key(float f) {
    if (f == 0.f) f = 0.f;  // canonicalise -0
    uint32_t u = __float_as_uint(f);
    u = (u & 0x80000000u) ? ~u : (u | 0x80000000u);  // ascending-orderable
    return ~u;
}
__device__ __forceinline__ float desc_key_inv(uint32_t k) {
    uint32_t u = ~k;
    u = (u & 0x80000000u) ? (u & 0x7fffffffu) : ~u;
    return __uint_as_float(u);
}

}  // namespace sdetr
