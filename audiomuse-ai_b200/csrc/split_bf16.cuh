// Split-bf16 row copy shared by the tensor-core k-means (kmeans_tc.cu) and the silhouette kernel (cluster_metrics.cu):
//   X f32 [N, d] -> Xs bf16 [N, 2*dp] = [hi | lo]  (x = hi + lo + O(2^-18 x)),  xn[N] = ||x||^2 (fp32);
//   dp = d rounded up to 64 (zero padded) so that a row is a whole number of 64-wide TMA K chunks.
#pragma once

#include "common.cuh"

namespace am {

// one warp per row
static __global__ void __launch_bounds__(256)
split_rows_kernel(const float* __restrict__ X, int64_t N, int d, int dp, __nv_bfloat16* __restrict__ Xs,
                  float* __restrict__ xn) {
  const int lane = threadIdx.x & 31;
  const int64_t warps = (int64_t)gridDim.x * (blockDim.x >> 5);
  for (int64_t row = (int64_t)blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5); row < N; row += warps) {
    const float* x = X + row * d;
    __nv_bfloat16* o = Xs + row * 2 * dp;
    float acc = 0.f;
    for (int i = lane; i < dp; i += 32) {
      const float v = i < d ? x[i] : 0.f;
      acc = fmaf(v, v, acc);
      const __nv_bfloat16 hi = __float2bfloat16_rn(v);
      o[i] = hi;
      o[dp + i] = __float2bfloat16_rn(v - __bfloat162float(hi));
    }
    acc = warp_sum(acc);
    if (lane == 0 && xn) xn[row] = acc;
  }
}

}  // namespace am
