// Dense projection GEMM of the path -- sdetr_gemm_f16x3_pre / _scaled ("3xFP16", fp32-class accuracy).
//
//   C[M,N] = act(A)[M,K] . W[N,K]^T + bias        fp32 in / fp32 out
//
// Same projections as gemm_tf32x3.cu (models/bricks/ms_deform_attn.py:316,322-328,375; salience_transformer.py:347-351,
// :462, :16-47; base_transformer.py:111).  An fp16 significand is as wide as a TF32 one (11 bits), so the same
// error-compensated product
//
//       x = hi + lo,  hi = fp16(x),  lo = fp16(x - hi)          C ~= A_hi.W_hi + A_hi.W_lo + A_lo.W_hi  (fp32 accumulate)
//
// keeps 22 significand bits per operand exactly like 3xTF32 (Ootomo & Yokota, "Recovering single precision accuracy from
// Tensor Cores ...", 2022), but runs on wgmma .f16: twice the K per instruction and twice the dense rate of TF32, and half
// the weight bytes through shared memory.  What fp16 lacks is exponent range; it is restored with exact power-of-two
// scalings: the activation is multiplied by 16 before the split (full accuracy for 2^-7 <= |x| < 4094, an ABSOLUTE error
// floor of 2^-29 below that, inf -> NaN above: documented domain of this entry point), the weight by a per-tensor 2^s that
// puts max|W| in [2^13, 2^14) when it is pre-split (cached per parameter), and the epilogue multiplies the accumulator by
// the exact inverse 2^-(4+s) before adding the bias.
//
// The kernel is gemm3x_kernel<true, false> of wgmma.cuh: k-blocks of 64, stage = A as two 128x32 fp32 boxes + W_hi + W_lo
// as 128x64 fp16 tiles (64 KB, three stages); per k-block and warpgroup 4 k-steps x {lo.hi, hi.lo, hi.hi} = 12 wgmma
// m64n128k16 with the split activation in registers.
#include <cuda_fp16.h>

#include "wgmma.cuh"

namespace sdetr {

// weight split: (N,K) fp32 -> W_hi = fp16(scale * W), W_lo = fp16(scale * W - W_hi)   (scale: a power of two)
__global__ void split_f16_pair_kernel(const float *__restrict__ w, int64_t n, float scale, __half *__restrict__ hi,
                                      __half *__restrict__ lo) {
    const int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    const float x = w[i] * scale;
    const __half h = __float2half_rn(x);
    hi[i] = h, lo[i] = __float2half_rn(x - __half2float(h));
}

}  // namespace sdetr

using namespace sdetr;

extern "C" int sdetr_split_f16_pair(const float *w, int64_t count, float scale, void *w_hi, void *w_lo, sdetr_stream_t stream) {
    SDETR_REQUIRE(w && w_hi && w_lo, SDETR_ERR_INVALID_ARG, "split_f16_pair: null pointer");
    SDETR_REQUIRE(scale > 0.f, SDETR_ERR_INVALID_ARG, "split_f16_pair: scale must be positive (a power of two)");
    if (count <= 0) return SDETR_OK;
    split_f16_pair_kernel<<<(unsigned)((count + 255) / 256), 256, 0, (cudaStream_t)stream>>>(
        w, count, scale, reinterpret_cast<__half *>(w_hi), reinterpret_cast<__half *>(w_lo));
    return check_launch("split_f16_pair");
}

static int gemm_f16x3_impl(const float *A, int64_t lda, const void *W_hi, const void *W_lo, float w_scale, const float *a_scale_dev,
                           const float *w_scale_dev,
                           const float *bias, float *C, int64_t ldc, int M, int N, int K, int act, sdetr_stream_t stream) {
    SDETR_REQUIRE(A && W_hi && W_lo && C, SDETR_ERR_INVALID_ARG, "gemm_f16x3_pre: null pointer");
    SDETR_REQUIRE(M >= 0 && N > 0 && K > 0 && act >= 0 && act <= 2, SDETR_ERR_INVALID_ARG, "gemm_f16x3_pre: bad sizes / activation");
    SDETR_REQUIRE(K % Gemm3xShape<true>::kK == 0, SDETR_ERR_UNSUPPORTED, "gemm_f16x3_pre: K=%d must be a multiple of %d", K,
                  Gemm3xShape<true>::kK);
    SDETR_REQUIRE(w_scale > 0.f, SDETR_ERR_INVALID_ARG, "gemm_f16x3_pre: weight scale must be positive");
    SDETR_REQUIRE(lda % 4 == 0 && aligned16(A) && aligned16(W_hi) && aligned16(W_lo) && lda >= K && ldc >= N,
                  SDETR_ERR_INVALID_ARG, "gemm_f16x3_pre: operands must be 16-byte aligned with 16-byte row pitch");
    if (M == 0) return SDETR_OK;
    CUtensorMap mh, ml;
    SDETR_REQUIRE(make_map_2d(&mh, CU_TENSOR_MAP_DATA_TYPE_FLOAT16, 2, W_hi, N, K, K, 64, kGN) &&
                      make_map_2d(&ml, CU_TENSOR_MAP_DATA_TYPE_FLOAT16, 2, W_lo, N, K, K, 64, kGN),
                  SDETR_ERR_CUDA, "gemm_f16x3_pre: cuTensorMapEncodeTiled failed");
    const Gemm3xParams p{bias, C, ldc, M, N, K, act, kActScale, 1.f / (kActScale * w_scale), a_scale_dev, w_scale_dev};
    return launch_gemm3x<true, false>(A, lda, mh, ml, p, stream, "gemm_f16x3_pre");
}


extern "C" int sdetr_gemm_f16x3_pre(const float *A, int64_t lda, const void *W_hi, const void *W_lo, float w_scale,
                                    const float *bias, float *C, int64_t ldc, int M, int N, int K, int act,
                                    sdetr_stream_t stream) {
    return gemm_f16x3_impl(A, lda, W_hi, W_lo, w_scale, nullptr, nullptr, bias, C, ldc, M, N, K, act, stream);
}

extern "C" int sdetr_gemm_f16x3_scaled(const float *A, int64_t lda, const float *a_scale_dev, const void *W_hi, const void *W_lo,
                                       const float *w_scale_dev, const float *bias, float *C, int64_t ldc, int M, int N, int K,
                                       sdetr_stream_t stream) {
    SDETR_REQUIRE(a_scale_dev && w_scale_dev, SDETR_ERR_INVALID_ARG, "gemm_f16x3_scaled: null scale pointer");
    return gemm_f16x3_impl(A, lda, W_hi, W_lo, 1.f, a_scale_dev, w_scale_dev, bias, C, ldc, M, N, K, 0, stream);
}

// The CNBlock form: C = z + s * (act(A) . W^T * out_scale + bias) with device scales (sdetr_gemm_f16x3_ex in the header).
// |GELU(x)| = |x| Phi(x) <= |x|, so the activation scale taken over A (pow2_scale, target 12) also bounds GELU(A) * a_scale
// below 2^12: the fp16 split cannot overflow whichever activation is applied on load.
extern "C" int sdetr_gemm_f16x3_ex(const float *A, int64_t lda, const float *a_scale_dev, const void *W_hi, const void *W_lo,
                                   const float *w_scale_dev, const float *bias, const float *col_scale, const float *Z, int64_t ldz,
                                   float *C, int64_t ldc, int M, int N, int K, int act, sdetr_stream_t stream) {
    SDETR_REQUIRE(A && a_scale_dev && W_hi && W_lo && w_scale_dev && C, SDETR_ERR_INVALID_ARG, "gemm_f16x3_ex: null pointer");
    SDETR_REQUIRE(M >= 0 && N > 0 && K > 0 && act >= 0 && act <= 2, SDETR_ERR_INVALID_ARG, "gemm_f16x3_ex: bad sizes / activation");
    SDETR_REQUIRE(K % Gemm3xShape<true>::kK == 0, SDETR_ERR_UNSUPPORTED, "gemm_f16x3_ex: K=%d must be a multiple of %d", K,
                  Gemm3xShape<true>::kK);
    SDETR_REQUIRE(lda % 4 == 0 && aligned16(A) && aligned16(W_hi) && aligned16(W_lo) && lda >= K && ldc >= N &&
                      (Z == nullptr || ldz >= N),
                  SDETR_ERR_INVALID_ARG, "gemm_f16x3_ex: operands must be 16-byte aligned with 16-byte row pitch");
    if (M == 0) return SDETR_OK;
    CUtensorMap mh, ml;
    SDETR_REQUIRE(make_map_2d(&mh, CU_TENSOR_MAP_DATA_TYPE_FLOAT16, 2, W_hi, N, K, K, 64, kGN) &&
                      make_map_2d(&ml, CU_TENSOR_MAP_DATA_TYPE_FLOAT16, 2, W_lo, N, K, K, 64, kGN),
                  SDETR_ERR_CUDA, "gemm_f16x3_ex: cuTensorMapEncodeTiled failed");
    const Gemm3xParams p{bias, C, ldc, M, N, K, act, 1.f, 1.f, a_scale_dev, w_scale_dev, col_scale, Z, ldz};
    return launch_gemm3x<true, false, true>(A, lda, mh, ml, p, stream, "gemm_f16x3_ex");
}

namespace sdetr {
__global__ void split_f16_pair_dev_kernel(const float *__restrict__ w, int64_t n, const float *__restrict__ scale_dev,
                                          __half *__restrict__ hi, __half *__restrict__ lo) {
    const int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    const float x = w[i] * __ldg(scale_dev);
    const __half h = __float2half_rn(x);
    hi[i] = h, lo[i] = __float2half_rn(x - __half2float(h));
}
}  // namespace sdetr

extern "C" int sdetr_split_f16_pair_dev(const float *w, int64_t count, const float *scale_dev, void *w_hi, void *w_lo,
                                        sdetr_stream_t stream) {
    SDETR_REQUIRE(w && scale_dev && w_hi && w_lo, SDETR_ERR_INVALID_ARG, "split_f16_pair_dev: null pointer");
    if (count <= 0) return SDETR_OK;
    split_f16_pair_dev_kernel<<<(unsigned)((count + 255) / 256), 256, 0, (cudaStream_t)stream>>>(
        w, count, scale_dev, reinterpret_cast<__half *>(w_hi), reinterpret_cast<__half *>(w_lo));
    return check_launch("split_f16_pair_dev");
}

// ---- power-of-two scale that brings max|x| to [2^(t-1), 2^t): one launch (the last block to finish publishes the result) ----
namespace sdetr {
__global__ void __launch_bounds__(256) pow2_scale_kernel(const float *__restrict__ x, int64_t n, int target_log2,
                                                         unsigned int *__restrict__ state /* [0] max bits, [1] blocks done */,
                                                         float *__restrict__ scale) {
    // the scale comes from the finite entries: a NaN or inf propagates through the GEMM whatever the scale, and an inf
    // counted here would give a scale that flushes every finite entry to zero in fp16
    bool nonfinite = false;
    const float m = block_max(thread_absmax<true>(x, n, nonfinite));
    __shared__ bool last;
    if (threadIdx.x == 0) {
        atomicMax(state, __float_as_uint(m));             // non-negative floats order like their bit patterns
        __threadfence();
        last = atomicAdd(state + 1, 1u) == gridDim.x - 1;
    }
    __syncthreads();
    if (last && threadIdx.x == 0) {
        __threadfence();
        const float amax = __uint_as_float(atomicAdd(state, 0u));
        int e = 0;
        float s = 1.f;
        if (amax > 0.f) {
            frexpf(amax, &e);                              // amax = f * 2^e, f in [0.5, 1)
            int sh = target_log2 - e;                      // amax * 2^sh in [2^(t-1), 2^t)
            sh = sh > 60 ? 60 : (sh < -60 ? -60 : sh);         // the product of two such scales stays finite
            s = ldexpf(1.f, sh);
        }
        *scale = s;
        state[0] = 0u, state[1] = 0u;                      // ready for the next call on this stream
    }
}
}  // namespace sdetr

extern "C" int sdetr_pow2_scale(const float *x, int64_t count, int target_log2, void *state /* 8 zeroed bytes */, float *scale,
                                sdetr_stream_t stream) {
    SDETR_REQUIRE(x && state && scale, SDETR_ERR_INVALID_ARG, "pow2_scale: null pointer");
    SDETR_REQUIRE(count > 0 && target_log2 >= -100 && target_log2 <= 100 && aligned16(x), SDETR_ERR_INVALID_ARG, "pow2_scale: bad arguments");
    const int64_t want = (count / 4 + 255) / 256;
    const int blocks = (int)(want < 1 ? 1 : (want > 4 * sm_count() ? 4 * sm_count() : want));
    pow2_scale_kernel<<<blocks, 256, 0, (cudaStream_t)stream>>>(x, count, target_log2, reinterpret_cast<unsigned int *>(state), scale);
    return check_launch("pow2_scale");
}
