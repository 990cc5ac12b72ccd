// The k-means definitions both drivers follow, kept in one place so that am_kmeans_fit (kmeans.cu, host-driven, one
// problem on the whole GPU) and am_kmeans_fit_batch (kmeans_batch.cu, one CTA per (problem, init)) pick the same
// k-means++ rows and stop at the same step by construction: the seeding generator and its draw count, the per-row
// D^2 chains, the two-level D^2 sampling scan over 1024-row blocks, sklearn's scaled tolerance and the order in which
// empty clusters take rows.
#pragma once

#include "common.cuh"

#include <algorithm>
#include <cmath>

namespace am {

// the seeding generator: init r of a fit consumes kpp_draws_per_init(k) uniforms after those of inits 0 .. r-1
struct SplitMix {
  uint64_t s;
  __host__ __device__ uint64_t next() {
    uint64_t z = (s += 0x9e3779b97f4a7c15ull);
    z = (z ^ (z >> 30)) * 0xbf58476d1ce4e5b9ull;
    z = (z ^ (z >> 27)) * 0x94d049bb133111ebull;
    return z ^ (z >> 31);
  }
  __host__ __device__ double uniform() { return (double)(next() >> 11) * (1.0 / 9007199254740992.0); }
};
constexpr uint64_t kKmeansSeedMix = 0x5851f42d4c957f2dull;  // SplitMix{seed ^ kKmeansSeedMix}

// greedy k-means++ (sklearn's _kmeans_plusplus): L = 2 + floor(ln k) local trials per centre, at most kMaxTrials
constexpr int kMaxTrials = 8;
inline int kpp_trials(int k) { return std::min(kMaxTrials, 2 + (int)std::log((double)k)); }
// the first row, then L candidates for each further centre
inline int kpp_draws_per_init(int k) { return 1 + (k - 1) * kpp_trials(k); }
constexpr int kKppBlock = 1024;  // rows per D^2 block: the sampling scan walks block sums, then one block's rows

// acc[l] = ||x - c_l||^2 for the nl (<= L) centres c_l = cand + l * stride, by a whole warp: lane-strided fmaf of the
// differences and one warp_sum tree per centre.  Every lane gets the same values.
template <int L>
__device__ __forceinline__ void d2_chains(const float* x, const float* cand, int64_t stride, int nl, int d, int lane,
                                          float (&acc)[L]) {
#pragma unroll
  for (int l = 0; l < L; ++l) acc[l] = 0.f;
  for (int i = lane; i < d; i += 32) {
    const float xv = x[i];
#pragma unroll
    for (int l = 0; l < L; ++l) {
      if (l < nl) {
        const float df = xv - cand[(int64_t)l * stride + i];
        acc[l] = fmaf(df, df, acc[l]);
      }
    }
  }
#pragma unroll
  for (int l = 0; l < L; ++l)
    if (l < nl) acc[l] = warp_sum(acc[l]);
}

// ||v||^2 of one row by a whole warp (lane-strided fmaf, one warp_sum tree): the centre and row norms of exact_argmin
__device__ __forceinline__ float warp_sq_norm(const float* v, int d, int lane) {
  float acc = 0.f;
  for (int i = lane; i < d; i += 32) acc = fmaf(v[i], v[i], acc);
  return warp_sum(acc);
}

// D^2 sampling, with r = u * (sum of the block sums in block order): the block whose running sum passes r, then the
// row inside it; r is reduced in place as the scan goes
template <class T>
__host__ __device__ inline int64_t kpp_scan(const T* w, int64_t n, double& r) {
  int64_t b = 0;
  for (; b < n - 1; ++b) {
    if (r < w[b]) break;
    r -= w[b];
  }
  return b;
}

// sklearn: tol_ = mean(var(X, axis=0)) * tol, from float64 column sums s1 and sums of squares s2 of N rows; mean[c]
// receives the column means rounded to float32 (the shift Lloyd runs under)
__host__ __device__ inline double kmeans_tol_abs(const double* s1, const double* s2, int64_t N, int d, float tol,
                                                 float* mean) {
  double var_mean = 0.0;
  for (int c = 0; c < d; ++c) {
    const double mu = s1[c] / N;
    var_mean += s2[c] / N - mu * mu;
    mean[c] = (float)mu;
  }
  return var_mean / d * tol;
}

// sklearn's _relocate_empty_clusters_dense hands the empty clusters, in index order, the rows farthest from their
// centres: row a goes before row b when it is farther, ties to the lower index
__host__ __device__ inline bool relocate_before(float da, int64_t a, float db, int64_t b) {
  return da > db || (da == db && a < b);
}

}  // namespace am
