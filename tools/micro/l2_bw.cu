// L2 -> SM read bandwidth: one CTA per SM streams the same 4 MB buffer (the fp16 hi / lo weights of the fused encoder FFN at
// hidden 2048) over and over, (a) with 128-bit loads that bypass L1, (b) with bulk async copies (the TMA engine, as the FFN
// kernel reads its weights) into a shared-memory ring of 3 or 6 copies of 32 KB in flight per SM (3: the FFN's ring).  Timed
// with CUDA events; prints the card name and power limit, which belong beside the numbers.  This is the ceiling to set the
// FFN's weight traffic (tools/bench_ffn.py) against.
//   nvcc -gencode arch=compute_90a,code=sm_90a -o l2_bw l2_bw.cu && ./l2_bw
#include <cstdint>
#include <cstdio>
#include <cuda_runtime.h>

constexpr int kBytes = 4 << 20;
constexpr int kChunk = 32 << 10;  // one bulk copy
constexpr int kMaxStages = 6;     // bulk copies in flight per SM

__global__ void __launch_bounds__(1024, 1) ldg_kernel(const int4 *buf, int reps, int *sink) {
    const int n = kBytes / 16, start = (int)((int64_t)blockIdx.x * n / gridDim.x);
    int acc = 0;
    for (int r = 0; r < reps; ++r)
        for (int i = threadIdx.x; i < n; i += 8 * blockDim.x) {
            int4 v[8];
#pragma unroll
            for (int k = 0; k < 8; ++k) {
                const int j = i + k * blockDim.x;
                v[k] = j < n ? __ldcg(buf + (j + start) % n) : make_int4(0, 0, 0, 0);
            }
#pragma unroll
            for (int k = 0; k < 8; ++k) acc ^= v[k].x ^ v[k].y ^ v[k].z ^ v[k].w;
        }
    if (acc == 0x7fffffff) sink[0] = acc;  // keeps the loads
}

__global__ void __launch_bounds__(32, 1) bulk_kernel(const uint8_t *buf, int reps, int stages) {
    extern __shared__ __align__(128) uint8_t ring[];
    __shared__ __align__(8) uint64_t full[kMaxStages];
    if (threadIdx.x != 0) return;
    const uint32_t bar0 = (uint32_t)__cvta_generic_to_shared(full);
    for (int s = 0; s < stages; ++s) asm volatile("mbarrier.init.shared::cta.b64 [%0], 1;" ::"r"(bar0 + 8 * s));
    asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
    const int chunks = kBytes / kChunk, start = (int)((int64_t)blockIdx.x * chunks / gridDim.x);
    uint32_t phase = 0;
    for (int t = 0; t < reps * chunks; ++t) {
        const int s = t % stages;
        const uint32_t bar = bar0 + 8 * s;
        if (t >= stages) {  // the copy that last used this stage has landed
            asm volatile(
                "{\n\t.reg .pred p;\n\tW_%=:\n\tmbarrier.try_wait.parity.shared::cta.b64 p, [%0], %1;\n\t@!p bra W_%=;\n\t}" ::"r"(bar),
                "r"((phase >> s) & 1u)
                : "memory");
            phase ^= 1u << s;
        }
        asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(bar), "r"(kChunk) : "memory");
        asm volatile("cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];" ::"r"(
                         (uint32_t)__cvta_generic_to_shared(ring + s * kChunk)),
                     "l"(buf + (int64_t)((t + start) % chunks) * kChunk), "r"(kChunk), "r"(bar)
                     : "memory");
    }
    for (int t = reps * chunks; t < reps * chunks + stages; ++t) {  // drain
        const int s = t % stages;
        asm volatile(
            "{\n\t.reg .pred p;\n\tW_%=:\n\tmbarrier.try_wait.parity.shared::cta.b64 p, [%0], %1;\n\t@!p bra W_%=;\n\t}" ::"r"(bar0 + 8 * s),
            "r"((phase >> s) & 1u)
            : "memory");
        phase ^= 1u << s;
    }
}

template <typename F>
double gbps(int ctas, int reps, F launch) {
    cudaEvent_t a, b;
    cudaEventCreate(&a), cudaEventCreate(&b);
    for (int w = 0; w < 3; ++w) launch();
    cudaEventRecord(a);
    const int n = 20;
    for (int i = 0; i < n; ++i) launch();
    cudaEventRecord(b);
    cudaEventSynchronize(b);
    float ms = 0.f;
    cudaEventElapsedTime(&ms, a, b);
    return (double)n * ctas * reps * kBytes / (ms * 1e-3) / 1e9;
}

int main() {
    cudaDeviceProp prop;
    cudaGetDeviceProperties(&prop, 0);
    char power[64] = "unknown";
    if (FILE *f = popen("nvidia-smi --query-gpu=power.limit --format=csv,noheader -i 0", "r")) {
        if (!fgets(power, sizeof power, f)) snprintf(power, sizeof power, "unknown\n");
        pclose(f);
    }
    printf("card: %s, power limit %s", prop.name, power);
    uint8_t *buf;
    int *sink;
    cudaMalloc(&buf, kBytes), cudaMalloc(&sink, 4);
    cudaMemset(buf, 1, kBytes);
    const int sms = prop.multiProcessorCount, reps = 16;
    cudaFuncSetAttribute(bulk_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, kMaxStages * kChunk);
    const double ldg = gbps(sms, reps, [&] { ldg_kernel<<<sms, 1024>>>(reinterpret_cast<const int4 *>(buf), reps, sink); });
    const double bulk3 = gbps(sms, reps, [&] { bulk_kernel<<<sms, 32, 3 * kChunk>>>(buf, reps, 3); });
    const double bulk6 = gbps(sms, reps, [&] { bulk_kernel<<<sms, 32, kMaxStages * kChunk>>>(buf, reps, kMaxStages); });
    const cudaError_t e = cudaDeviceSynchronize();
    if (e != cudaSuccess) {
        printf("error: %s\n", cudaGetErrorString(e));
        return 1;
    }
    printf("{\"sms\": %d, \"buffer_mb\": 4, \"ldg128_gbps\": %.0f, \"bulk_copy_96kb_in_flight_gbps\": %.0f, "
           "\"bulk_copy_192kb_in_flight_gbps\": %.0f}\n", sms, ldg, bulk3, bulk6);
    return 0;
}
