// Tensor-core Lloyd step (kmeans_tc.cu): plan = split-bf16 copy of the data set + scratch, reused across iterations.
#pragma once

#include "common.cuh"

namespace am {
namespace kmtc {

// true when the wgmma path can serve this problem (k <= 128; sm_90; AM_KMEANS_SIMT unset)
bool usable(int64_t N, int d, int k);

struct Plan {
  int64_t N = 0;
  int d = 0, k = 0, dp = 0, kp = 0;
  const float* X = nullptr;      // caller's rows (device), must outlive the plan
  DevBuf<__nv_bfloat16> Xs, Cs;  // [N, 2*dp] hi | lo ; [2*kp, dp] hi rows, lo rows
  DevBuf<float> xn, cn, scratch_sums;
  DevBuf<int> scal;
  DevBuf<int32_t> recheck;
  DevBuf<double> inertia64;
  alignas(64) unsigned char map_x[128];
  alignas(64) unsigned char map_c[128];

  int create(const float* X_dev, int64_t N, int d, int k, cudaStream_t st);
  // one E-step (+ M-step partial sums when `sums` is given): labels i32[N]; sums f32[k, d], counts f32[k] and
  // inertia f64[1] are OVERWRITTEN; dist f32[N] (optional) = squared distance to the assigned centre
  int step(const float* C_dev, int32_t* labels, float* sums, float* counts, double* inertia_dev, float* dist,
           cudaStream_t st);
  int last_recheck_count(cudaStream_t st, int* out);
  int launch_accumulate(float* sums, float* counts, double* inertia_dev, const float* C_dev, const int32_t* labels,
                        cudaStream_t st);
};

}  // namespace kmtc
}  // namespace am
