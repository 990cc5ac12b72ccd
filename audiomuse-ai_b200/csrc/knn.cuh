// What the k-NN index (knn.cu) and the candidate post-processing on top of it (knn_walks.cu) share: the index and the
// metric constants.
#pragma once

#include "common.cuh"

namespace am {
constexpr int kMetricCos = 0, kMetricL2 = 1, kMetricIp = 2;
}  // namespace am

struct am_index {
  int64_t N = 0;
  int d = 0;
  int metric = 0;
  am::DevBuf<float> X;        // [N, d] stored rows (unit-normalised for cosine)
  am::DevBuf<float> xnorm2;   // [N] squared norms (euclidean)
  am::DevBuf<__nv_bfloat16> Xb;  // [N, dpad] bf16 copy for the tensor-core filter
  am::DevBuf<float> xres;     // [N] ||x - bf16(x)||_2 (bf16 filter bound)
  int dpad = 0;
  float max_norm = 1.0f;      // max ||x|| over stored rows
  float xres_max = 0.0f;      // max ||x - bf16(x)|| over stored rows
};
