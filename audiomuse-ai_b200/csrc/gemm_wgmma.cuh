// bf16 x bf16 -> fp32 GEMM on the Hopper tensor cores (wgmma + TMA), sm_90a.
//
//   D[m, n] = epi( alpha * sum_k A[m, k] * B[n, k] )        A: [M, K] row-major (K-major)
//                                                            B: [N, K] row-major (K-major)
//   epi(v)  = act(v + bias[n] - col_sub[n]) + residual[m, n] ; D is bf16 or fp32.
//
// Users: the encoder's 1x1 convolutions / linear layers (encoder.cu; A = NHWC activations,
// B = folded conv weights) and the k-NN bf16 filter pass (knn.cu; A = queries, B = library).
#pragma once

#include "common.cuh"

namespace am {
namespace gemm {

struct Epilogue {
  float alpha = 1.0f;
  const float* bias = nullptr;              // [N] added
  const float* col_sub = nullptr;           // [N] subtracted (k-NN euclidean: ||x||^2)
  int act = 0;                              // 0 none, 1 relu6, 2 relu, 3 hardswish (model_spec.cuh ActKind)
  const __nv_bfloat16* residual = nullptr;  // [M, ld_res] added after act
  int64_t ld_res = 0;
  // k-NN: besides D, write the maximum of every 32-column chunk of epi(...) (columns >= N count as -inf):
  // chunk_max[m * ld_cm + n / 32].  The selection kernel finds its threshold and the few chunks that can hold answers
  // from these (1/32 of the score matrix) and then touches only those chunks of D.
  float* chunk_max = nullptr;
  int64_t ld_cm = 0;
};

// true when the device can run the wgmma path (sm_90) and the driver exports
// cuTensorMapEncodeTiled
bool available();

// lda/ldb in elements, multiples of 8 (16-byte TMA row pitch).  ldd in elements of D; a bf16 D leaves through TMA
// stores, so its ldd is a multiple of 8 and its base 16-byte aligned.  A residual needs an even ld_res and a 4-byte
// aligned base; chunk maxima need an fp32 D.
// m_fastest: enumerate tiles with the M index fastest (B tile shared by consecutive CTAs;
// right when A is small, e.g. k-NN queries); otherwise N fastest (A tile shared).
int gemm_bf16(const __nv_bfloat16* A, int64_t M, int64_t lda, const __nv_bfloat16* B, int64_t N,
              int64_t ldb, int K, void* D, int64_t ldd, bool d_is_f32, const Epilogue& ep,
              bool m_fastest, cudaStream_t st);

// The TMA map of the wgmma kernels' K-major operands: a 2-D bf16 matrix of `rows` rows of `inner` elements,
// `pitch_elems` apart (a multiple of 8), loaded in 64 x box_rows boxes with SWIZZLE_128B, zero fill outside.
// map_out: 128-byte CUtensorMap.
int encode_map_bf16(void* map_out, const void* base, int64_t inner, int64_t rows, int64_t pitch_elems, int box_rows);

// The TMA map of a dense NHWC bf16 activation [n, h, w, c] (c a multiple of 8), loaded in boxes of 64 channels x
// box_w x box_h pixels of one image, zero fill outside (negative coordinates included): with `swizzle` as K-major
// SWIZZLE_128B rows (one row per pixel, x fastest), without as plain 128-byte rows.
int encode_map_nhwc_bf16(void* map_out, const void* base, int64_t n, int64_t h, int64_t w, int64_t c, int box_w,
                         int box_h, bool swizzle);

// reference implementation on CUDA cores (slow; used only by the on-device self test)
int gemm_bf16_simt(const __nv_bfloat16* A, int64_t M, int64_t lda, const __nv_bfloat16* B, int64_t N,
                   int64_t ldb, int K, void* D, int64_t ldd, bool d_is_f32, const Epilogue& ep,
                   cudaStream_t st);

// S[q, j] = Qb[q, :] . Xb[j, :]  (2*dot - xnorm2[j] when xnorm2 != NULL), fp32 out; CM != NULL: also the maximum of
// every 32 consecutive scores, CM[q, j / 32].  Qb has `qrows` rows (multiple of 128, zero padded).
inline int scores_bf16(const __nv_bfloat16* Qb, int qrows, const __nv_bfloat16* Xb, int64_t N, int dpad, float* S,
                       int64_t ldS, float* CM, int64_t ldCM, const float* xnorm2, cudaStream_t st) {
  Epilogue ep;
  ep.alpha = xnorm2 ? 2.0f : 1.0f;
  ep.col_sub = xnorm2;
  ep.chunk_max = CM;
  ep.ld_cm = CM ? ldCM : 0;
  return gemm_bf16(Qb, qrows, dpad, Xb, N, dpad, dpad, S, ldS, true, ep, /*m_fastest=*/true, st);
}

}  // namespace gemm
}  // namespace am
