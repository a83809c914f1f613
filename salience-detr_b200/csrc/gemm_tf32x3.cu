// Dense projection GEMM of the path, TF32 form -- sdetr_gemm_3xtf32 / _pre / _raw.
//
//   C[M,N] = act(A)[M,K] . W[N,K]^T + bias        fp32 in / fp32 out, fp32-class accuracy ("3xTF32")
//
// These are the only true dense GEMMs of the path (models/bricks/ms_deform_attn.py:316,322-328,375 value / offset /
// weight / output projections; salience_transformer.py:347-351 FFN; :462 class head; :16-47 MaskPredictor;
// base_transformer.py:111 enc_output).  The kernel is gemm3x_kernel<false, *> of wgmma.cuh: k-blocks of 32 fp32 (one
// 128-byte swizzled row), stage = A box + W_hi + W_lo (48 KB, four stages); the activation is split into TF32 pieces in
// registers (x = hi + lo, hi = tf32(x), lo = tf32(x - hi), optional ReLU / GELU fused in) and each warpgroup issues
// 4 k-steps x {lo.hi, hi.lo, hi.hi} = 12 wgmma m64n128k8 .tf32 per k-block.  The weight arrives pre-split
// (sdetr_split_tf32_pair, cached by the caller per parameter) or raw (sdetr_gemm_3xtf32_raw: the consumer warpgroups split
// the landed W tile in place with the same arithmetic, so both forms give bit-identical results).
#include "wgmma.cuh"

namespace sdetr {

// weight split: (N,K) -> W_hi, W_lo (both (N,K), TF32-representable)
__global__ void split_pair_kernel(const float *__restrict__ w, int64_t n, float *__restrict__ hi, float *__restrict__ lo) {
    const int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    const float x = w[i], h = tf32_rn(x);
    hi[i] = h, lo[i] = tf32_rn(x - h);
}

// 2-D fp32 tensor (rows, cols) with row stride ld (floats); box = 32 cols x 128 rows, 128-byte swizzle
static bool make_map(CUtensorMap *m, const float *base, int64_t rows, int64_t cols, int64_t ld) {
    return make_map_2d(m, CU_TENSOR_MAP_DATA_TYPE_FLOAT32, 4, base, rows, cols, ld, 32, kGN);
}

static int gemm_3xtf32_impl(const float *A, int64_t lda, const float *W_hi, const float *W_lo, const float *bias, float *C,
                            int64_t ldc, int M, int N, int K, int act, sdetr_stream_t stream, const char *what) {
    const bool raw = W_lo == nullptr;  // sdetr_gemm_3xtf32_raw: W_hi is the raw weight
    SDETR_REQUIRE(A && W_hi && C, SDETR_ERR_INVALID_ARG, "%s: null pointer", what);
    SDETR_REQUIRE(M >= 0 && N > 0 && K > 0 && act >= 0 && act <= 2, SDETR_ERR_INVALID_ARG, "%s: bad sizes / activation", what);
    SDETR_REQUIRE(K % Gemm3xShape<false>::kK == 0, SDETR_ERR_UNSUPPORTED, "%s: K=%d must be a multiple of %d", what, K,
                  Gemm3xShape<false>::kK);
    SDETR_REQUIRE(lda % 4 == 0 && aligned16(A) && aligned16(W_hi) && (raw || aligned16(W_lo)) && lda >= K && ldc >= N,
                  SDETR_ERR_INVALID_ARG, "%s: operands must be 16-byte aligned with 16-byte row pitch", what);
    if (M == 0) return SDETR_OK;
    CUtensorMap mh, ml;
    SDETR_REQUIRE(make_map(&mh, W_hi, N, K, K) && (raw || make_map(&ml, W_lo, N, K, K)), SDETR_ERR_CUDA,
                  "%s: cuTensorMapEncodeTiled failed", what);
    if (raw) ml = mh;
    const Gemm3xParams p{bias, C, ldc, M, N, K, act, 1.f, 1.f, nullptr, nullptr};
    return raw ? launch_gemm3x<false, true>(A, lda, mh, ml, p, stream, what)
               : launch_gemm3x<false, false>(A, lda, mh, ml, p, stream, what);
}

}  // namespace sdetr

using namespace sdetr;

extern "C" int sdetr_gemm_3xtf32_raw(const float *A, int64_t lda, const float *W, const float *bias, float *C, int64_t ldc,
                                     int M, int N, int K, int act, sdetr_stream_t stream) {
    SDETR_REQUIRE(W, SDETR_ERR_INVALID_ARG, "gemm_3xtf32_raw: null pointer");
    return gemm_3xtf32_impl(A, lda, W, nullptr, bias, C, ldc, M, N, K, act, stream, "gemm_3xtf32_raw");
}

extern "C" int sdetr_split_tf32_pair(const float *w, int64_t count, float *w_hi, float *w_lo, sdetr_stream_t stream) {
    SDETR_REQUIRE(w && w_hi && w_lo, SDETR_ERR_INVALID_ARG, "split_tf32_pair: null pointer");
    if (count <= 0) return SDETR_OK;
    split_pair_kernel<<<(unsigned)((count + 255) / 256), 256, 0, (cudaStream_t)stream>>>(w, count, w_hi, w_lo);
    return check_launch("split_tf32_pair");
}

extern "C" int sdetr_gemm_3xtf32(const float *A, int64_t lda, const float *W_hi, const float *W_lo, const float *bias,
                                 float *C, int64_t ldc, int M, int N, int K, int relu_a, sdetr_stream_t stream) {
    SDETR_REQUIRE(W_lo, SDETR_ERR_INVALID_ARG, "gemm_3xtf32: null pointer");
    return gemm_3xtf32_impl(A, lda, W_hi, W_lo, bias, C, ldc, M, N, K, relu_a, stream, "gemm_3xtf32");
}

extern "C" int sdetr_gemm_3xtf32_pre(const float *A, int64_t lda, const float *W_hi, const float *W_lo, const float *bias,
                                     float *C, int64_t ldc, int M, int N, int K, int act, sdetr_stream_t stream) {
    SDETR_REQUIRE(W_lo, SDETR_ERR_INVALID_ARG, "gemm_3xtf32_pre: null pointer");
    return gemm_3xtf32_impl(A, lda, W_hi, W_lo, bias, C, ldc, M, N, K, act, stream, "gemm_3xtf32_pre");
}
