// k-means Lloyd step: the path choice and the step object (kmeans.cu), the tensor-core plan (kmeans_tc.cu: split-bf16
// copy of the data set + scratch, reused across iterations) and the exact fp32 argmin both paths share.
#pragma once

#include "common.cuh"

#include <memory>

namespace am {

// How many Lloyd steps the split-bf16 copy of the rows is paid back over (kmeans_use_tensor_cores)
enum class KMeansUse { kPlan, kFit, kAssign };
bool kmeans_use_tensor_cores(int64_t N, int d, int k, KMeansUse use);

// The exact fp32 argmin of row x over centres j0 + kStep u, u < NC (those >= k skipped), by a whole warp: each lane
// takes features lane, lane + 32, ... with fmaf, one warp_sum tree per centre, v_j = cn_j - 2 x.c_j, and a strict "<"
// in increasing j (the lowest index wins ties).  assign_kernel and recheck_kernel both decide with it, which is why a
// row the tensor-core step rechecks gets the CUDA-core label.  kLdg = false reads C with plain loads, for
// centres in shared memory or written by the same kernel (kmeans_batch.cu); the arithmetic is the same.
template <bool kLdg>
__device__ __forceinline__ float ld_centre(const float* p) {
  if constexpr (kLdg) return __ldg(p);
  else return *p;
}

template <int NC, int kStep, bool kLdg = true>
__device__ __forceinline__ void exact_argmin(const float* x, int d, const float* C, const float* cn, int k, int lane,
                                             int j0, float& best, int& best_j) {
  float acc[NC] = {};
  // one centre reads through a row pointer, several by index: the faster code for each, with the same arithmetic
  const float* c0 = C + (int64_t)j0 * d;
  for (int i = lane; i < d; i += 32) {
    const float xv = __ldg(&x[i]);
#pragma unroll
    for (int u = 0; u < NC; ++u) {
      const int j = j0 + kStep * u;
      if (j < k) acc[u] = fmaf(xv, ld_centre<kLdg>(NC == 1 ? &c0[i] : &C[(int64_t)j * d + i]), acc[u]);
    }
  }
  float b = best;
  int bj = best_j;  // the running minimum in locals: its update compiles to selects
#pragma unroll
  for (int u = 0; u < NC; ++u) {
    const int j = j0 + kStep * u;
    const float a = warp_sum(acc[u]);
    if (j < k) {
      const float v = cn[j] - 2.0f * a;
      if (v < b) {
        b = v;
        bj = j;
      }
    }
  }
  best = b;
  best_j = bj;
}

namespace kmtc {

struct Plan {
  const float* X = nullptr;  // caller's rows (device), must outlive the plan
  int64_t N = 0;
  int d = 0, k = 0, dp = 0, kp = 0;
  DevBuf<__nv_bfloat16> Xs, Cs;  // [N, 2*dp] hi | lo ; [2*kp, dp] hi rows, lo rows
  DevBuf<float> xn, cn, scratch_sums;
  DevBuf<int> scal;  // [0] max ||c||^2 bits, [1] rows in the last step's recheck list
  DevBuf<int32_t> recheck;
  alignas(64) unsigned char map_x[128];
  alignas(64) unsigned char map_c[128];

  int create(cudaStream_t st);  // on a Plan{X, N, d, k}
  int step(const float* C_dev, int32_t* labels, float* sums, float* counts, double* inertia_dev, float* dist,
           cudaStream_t st);  // am_kmeans_plan::step on the tensor cores
  int launch_accumulate(float* sums, float* counts, double* inertia_dev, const float* C_dev, const int32_t* labels,
                        cudaStream_t st);
};

}  // namespace kmtc
}  // namespace am

// One Lloyd step over the device rows X [N, d] (they must outlive it), built as am_kmeans_plan{X, N, d, k} and then
// create(): the tensor-core plan, or assign_kernel + accumulate_kernel on CUDA cores with the centre norms in `cn`.
struct am_kmeans_plan {
  const float* X = nullptr;
  int64_t N = 0;
  int d = 0, k = 0;
  std::unique_ptr<am::kmtc::Plan> tc;  // the tensor-core path, or
  am::DevBuf<float> cn;                // the CUDA-core path's centre norms
  am::DevBuf<double> inert;            // float64 inertia behind am_kmeans_plan_step's f32 output

  int create(bool tensor_cores, cudaStream_t st);
  // labels i32[N]; sums f32[k, d], counts f32[k] (the tensor-core path fills them only with sums) and inertia f64[1]
  // (each optional) are OVERWRITTEN; dist f32[N] (optional) = squared distance of each row to its centre
  int step(const float* C, int32_t* labels, float* sums, float* counts, double* inertia, float* dist, cudaStream_t st);
};
