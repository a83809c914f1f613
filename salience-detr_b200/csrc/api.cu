// Library-level entry points: version, thread-local error string, launch counter.
#include <stdarg.h>

#include <atomic>

#include "common.cuh"

namespace sdetr {
static thread_local char g_error[512] = "";
static std::atomic<unsigned long long> g_launches{0};

void set_error(const char *fmt, ...) {
    va_list ap;
    va_start(ap, fmt);
    vsnprintf(g_error, sizeof(g_error), fmt, ap);
    va_end(ap);
}
int sm_count() {
    static std::atomic<int> cache[256];
    int dev = 0;
    if (cudaGetDevice(&dev) != cudaSuccess) return 132;
    int v = cache[dev & 255].load(std::memory_order_relaxed);
    if (!v) {
        if (cudaDeviceGetAttribute(&v, cudaDevAttrMultiProcessorCount, dev) != cudaSuccess || v <= 0) v = 132;
        cache[dev & 255].store(v, std::memory_order_relaxed);
    }
    return v;
}
static std::atomic<int> g_persistent_cap{0};
int persistent_ctas() {
    const int cap = g_persistent_cap.load(std::memory_order_relaxed), sms = sm_count();
    return cap > 0 && cap < sms ? cap : sms;
}
void count_launch(int n) { g_launches.fetch_add((unsigned long long)n, std::memory_order_relaxed); }
}  // namespace sdetr

extern "C" int sdetr_set_persistent_ctas(int n) {
    sdetr::g_persistent_cap.store(n > 0 ? n : 0, std::memory_order_relaxed);
    return SDETR_OK;
}
extern "C" int sdetr_version(void) { return 100; }  // 0.1.0
extern "C" const char *sdetr_last_error(void) { return sdetr::g_error; }
extern "C" unsigned long long sdetr_launch_count(void) { return sdetr::g_launches.load(std::memory_order_relaxed); }
