// Debug entry point of the k-means Lloyd step (NOT part of libaudiomuse_b200.so: built into
// libaudiomuse_b200_debug.so, declared in include/audiomuse_b200_debug.h; used by tests/test_gpu_kmeans.py and
// tools/kmeans_bench.py).  Runs one step on the path the caller names instead of the one kmeans_use_tensor_cores
// picks, so the tensor-core step can be compared with the exact CUDA-core step on the same shape.
#include "../common.cuh"
#include "../kmeans_tc.cuh"
#include "../../../include/audiomuse_b200_debug.h"

extern "C" AM_API int am_debug_kmeans_step(int path, const float* X_dev, int64_t N, int d, int k,
                                           const float* centers_dev, int32_t* labels_dev, float* sums_dev,
                                           float* counts_dev, float* inertia_dev, float* dist_dev, void* stream) {
  using namespace am;
  AM_CHECK(path == 0 || path == 1, "am_debug_kmeans_step: path %d", path);
  AM_CHECK(X_dev && centers_dev && labels_dev, "am_debug_kmeans_step: NULL argument");
  AM_CHECK(N > 0 && d > 0 && k > 0, "am_debug_kmeans_step: bad shape");
  AM_TRY(ensure_init());
  AM_CHECK(path == 1 || kmeans_use_tensor_cores(N, d, k, KMeansUse::kPlan),
           "am_debug_kmeans_step: the tensor-core step does not take N=%lld d=%d k=%d", (long long)N, d, k);
  am_kmeans_plan p{X_dev, N, d, k};
  AM_TRY(p.create(path == 0, (cudaStream_t)stream));
  AM_TRY(am_kmeans_plan_step(&p, centers_dev, labels_dev, sums_dev, counts_dev, inertia_dev, dist_dev, stream));
  AM_CUDA(cudaStreamSynchronize((cudaStream_t)stream));
  return AM_OK;
}
