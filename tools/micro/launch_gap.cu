// Kernel-to-kernel gap inside a CUDA graph on this GPU, with and without programmatic dependent launch, for small kernels and
// for kernels that opt into the maximum dynamic shared memory (carve-out switches).  nvcc -arch=sm_90a -o launch_gap launch_gap.cu
#include <cstdio>
#include <cuda_runtime.h>
#include <vector>

__global__ void small_kernel(float *p, int pdl) {
    if (pdl) asm volatile("griddepcontrol.wait;" ::: "memory");
    if (threadIdx.x == 0 && blockIdx.x == 0) p[0] += 1.f;
    if (pdl) asm volatile("griddepcontrol.launch_dependents;" ::: "memory");
}
__global__ void __launch_bounds__(512, 1) big_kernel(float *p, int pdl) {
    extern __shared__ float sm[];
    if (pdl) asm volatile("griddepcontrol.wait;" ::: "memory");
    sm[threadIdx.x] = p[0];
    __syncthreads();
    if (threadIdx.x == 0 && blockIdx.x == 0) p[0] = sm[1] + 1.f;
    if (pdl) asm volatile("griddepcontrol.launch_dependents;" ::: "memory");
}
// ~10 us of work on every SM, so that the gap is measured between kernels that really occupy the machine
__global__ void __launch_bounds__(512, 1) busy_kernel(float *p, int pdl, int iters) {
    extern __shared__ float sm[];
    sm[threadIdx.x] = 0.f;  // prologue independent of the predecessor
    __syncthreads();
    if (pdl) asm volatile("griddepcontrol.wait;" ::: "memory");
    float a = p[0];
    for (int i = 0; i < iters; ++i) a = a * 1.0000001f + 1e-9f;
    if (pdl) asm volatile("griddepcontrol.launch_dependents;" ::: "memory");
    if (a == 123.456f) p[1] = a;
    if (threadIdx.x == 0 && blockIdx.x == 0) p[0] = a * 0.f + 1.f;
}

template <typename F>
float time_graph(int n, F launch) {
    cudaStream_t s;
    cudaStreamCreate(&s);
    cudaGraph_t g;
    cudaGraphExec_t ge;
    cudaStreamBeginCapture(s, cudaStreamCaptureModeGlobal);
    for (int i = 0; i < n; ++i) launch(s, i);
    if (cudaStreamEndCapture(s, &g) != cudaSuccess) { printf("capture failed: %s\n", cudaGetErrorString(cudaGetLastError())); return -1; }
    if (cudaGraphInstantiate(&ge, g, 0) != cudaSuccess) { printf("instantiate failed: %s\n", cudaGetErrorString(cudaGetLastError())); return -1; }
    cudaEvent_t a, b;
    cudaEventCreate(&a), cudaEventCreate(&b);
    for (int w = 0; w < 3; ++w) cudaGraphLaunch(ge, s);
    cudaStreamSynchronize(s);
    cudaEventRecord(a, s);
    for (int r = 0; r < 10; ++r) cudaGraphLaunch(ge, s);
    cudaEventRecord(b, s);
    cudaStreamSynchronize(s);
    float ms;
    cudaEventElapsedTime(&ms, a, b);
    if (cudaGetLastError() != cudaSuccess) printf("error\n");
    return ms * 1000.f / (10.f * n);
}

template <typename K, typename... Args>
void launch_attr(K kernel, dim3 grid, dim3 block, size_t smem, cudaStream_t s, bool pdl, Args... args) {
    cudaLaunchConfig_t cfg{};
    cfg.gridDim = grid, cfg.blockDim = block, cfg.dynamicSmemBytes = smem, cfg.stream = s;
    cudaLaunchAttribute at[1];
    at[0].id = cudaLaunchAttributeProgrammaticStreamSerialization;
    at[0].val.programmaticStreamSerializationAllowed = 1;
    cfg.attrs = at, cfg.numAttrs = pdl ? 1 : 0;
    cudaLaunchKernelEx(&cfg, kernel, args...);
}

int main() {
    float *p;
    cudaMalloc(&p, 1024);
    cudaMemset(p, 0, 1024);
    const int big = 227 * 1024;
    cudaFuncSetAttribute(big_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, big);
    cudaFuncSetAttribute(busy_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, big);
    const int n = 200;
    for (int pdl = 0; pdl < 2; ++pdl) {
        printf("pdl=%d  small 1 CTA:            %.2f us per node\n", pdl, time_graph(n, [&](cudaStream_t s, int) { launch_attr(small_kernel, 1, 32, 0, s, pdl, p, pdl); }));
        printf("pdl=%d  small 132 CTAs x 256:   %.2f us per node\n", pdl, time_graph(n, [&](cudaStream_t s, int) { launch_attr(small_kernel, 132, 256, 0, s, pdl, p, pdl); }));
        printf("pdl=%d  227 KB smem 132 x 512:  %.2f us per node\n", pdl, time_graph(n, [&](cudaStream_t s, int) { launch_attr(big_kernel, 132, 512, big, s, pdl, p, pdl); }));
        printf("pdl=%d  alternating small/227KB: %.2f us per node\n", pdl, time_graph(n, [&](cudaStream_t s, int i) {
            if (i & 1) launch_attr(big_kernel, 132, 512, big, s, pdl, p, pdl); else launch_attr(small_kernel, 132, 256, 0, s, pdl, p, pdl); }));
        for (int iters : {2000, 20000}) {
            printf("pdl=%d  busy(%d iters) 227 KB 132 x 512: %.2f us per node\n", pdl, iters, time_graph(n, [&](cudaStream_t s, int) { launch_attr(busy_kernel, 132, 512, big, s, pdl, p, pdl, iters); }));
            printf("pdl=%d  busy(%d iters) alternating with small: %.2f us per PAIR\n", pdl, iters, 2 * time_graph(n, [&](cudaStream_t s, int i) {
                if (i & 1) launch_attr(busy_kernel, 132, 512, big, s, pdl, p, pdl, iters); else launch_attr(small_kernel, 132, 256, 0, s, pdl, p, pdl); }));
        }
    }
    return 0;
}
