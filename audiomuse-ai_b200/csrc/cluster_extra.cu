// PCA and DBSCAN for the clustering task (SURVEY 8(f4); tasks/clustering_gpu.py:151-278: cuml.decomposition.PCA and
// cuml.cluster.DBSCAN with scikit-learn as the fallback -- scikit-learn's results are the bar).
//
// PCA   am_pca_moments: column means + covariance (n - 1 normalisation), accumulated in float64 on the device -- H100 has
//       FP64 to spare (N d^2 DFMA: 2.6e10 for 100 k x 512) and the eigenvectors of a float32 covariance would not match
//       LAPACK's to better than 1e-4.  The d x d eigenproblem stays on the host (numpy / LAPACK, like the reference's
//       Python); am_pca_project applies (X - mean) W^T on the device, centring against the float64 mean in float64 (a
//       float32 mean would cost |mean| * 2^-24 per coordinate, which is large next to a small spread).
// DBSCAN brute force, exact: one pass of tiled squared distances (fp32 differences, float64 re-check inside a relative
//       1e-5 band around eps^2, against eps^2 formed in float64 from the caller's double eps) writes the eps-neighbourhood
//       relation as an N x N bit matrix (1.25 GB at 100 k rows) and the neighbour counts; core points = count >=
//       min_samples (the point itself included, as scikit-learn); clusters = connected components of the core-core
//       relation, found in one pass by lock-free union-find (each edge hooks the larger root under the smaller with
//       atomicCAS, then a compress pass), so the work does not depend on the index order of the points and no iteration
//       cap can cut a component short; every root is the lowest core index of its component; a border point takes the
//       SMALLEST root among its core neighbours -- which is what scikit-learn's index-ordered depth-first expansion
//       produces, clusters being numbered by their lowest core index.
#include "common.cuh"
#include "host_call.cuh"

#include <algorithm>
#include <vector>

namespace am {

// ---------------------------------------------------------------- PCA
// column sums in float64: grid.y row slabs, one thread per column
__global__ void col_sum_kernel(const float* __restrict__ X, int64_t N, int d, double* __restrict__ sum) {
  const int c = blockIdx.x * blockDim.x + threadIdx.x;
  if (c >= d) return;
  const int64_t rows = (N + gridDim.y - 1) / gridDim.y, r0 = (int64_t)blockIdx.y * rows, r1 = min(N, r0 + rows);
  double acc = 0.0;
  for (int64_t r = r0; r < r1; ++r) acc += (double)X[r * d + c];
  atomicAdd(&sum[c], acc);
}

// C[i, j] += sum_r (X[r, i] - mu_i)(X[r, j] - mu_j) over this CTA's row slab; 64 x 64 tile per CTA, 4 x 4 per thread
constexpr int kCovTile = 64, kCovRows = 16;
__global__ void __launch_bounds__(256)
cov_kernel(const float* __restrict__ X, int64_t N, int d, const double* __restrict__ mean, double* __restrict__ Cov) {
  __shared__ double sa[kCovRows][kCovTile + 1], sb[kCovRows][kCovTile + 1];
  const int ti = blockIdx.x, tj = blockIdx.y;
  if (tj < ti) return;   // symmetric: upper tiles only, mirrored by the caller's finish kernel
  const int tx = threadIdx.x & 15, ty = threadIdx.x >> 4;
  const int64_t rows = (N + gridDim.z - 1) / gridDim.z, r0 = (int64_t)blockIdx.z * rows, r1 = min(N, r0 + rows);
  double acc[4][4] = {};
  for (int64_t rb = r0; rb < r1; rb += kCovRows) {
    for (int e = threadIdx.x; e < kCovRows * kCovTile; e += 256) {
      const int rr = e / kCovTile, cc = e - rr * kCovTile;
      const int64_t r = rb + rr;
      const int ci = ti * kCovTile + cc, cj = tj * kCovTile + cc;
      sa[rr][cc] = (r < r1 && ci < d) ? (double)X[r * d + ci] - mean[ci] : 0.0;
      sb[rr][cc] = (r < r1 && cj < d) ? (double)X[r * d + cj] - mean[cj] : 0.0;
    }
    __syncthreads();
#pragma unroll
    for (int rr = 0; rr < kCovRows; ++rr) {
      double a[4], b[4];
#pragma unroll
      for (int u = 0; u < 4; ++u) {
        a[u] = sa[rr][ty * 4 + u];
        b[u] = sb[rr][tx * 4 + u];
      }
#pragma unroll
      for (int u = 0; u < 4; ++u)
#pragma unroll
        for (int v = 0; v < 4; ++v) acc[u][v] = fma(a[u], b[v], acc[u][v]);
    }
    __syncthreads();
  }
#pragma unroll
  for (int u = 0; u < 4; ++u)
#pragma unroll
    for (int v = 0; v < 4; ++v) {
      const int i = ti * kCovTile + ty * 4 + u, j = tj * kCovTile + tx * 4 + v;
      if (i < d && j < d) atomicAdd(&Cov[(int64_t)i * d + j], acc[u][v]);
    }
}

__global__ void cov_finish_kernel(double* __restrict__ Cov, int d, double inv) {
  const int64_t e = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (e >= (int64_t)d * d) return;
  const int i = (int)(e / d), j = (int)(e - (int64_t)i * d);
  if ((j / kCovTile) < (i / kCovTile)) return;   // lower tiles are written from their mirror
  const double v = Cov[e] * inv;
  Cov[e] = v;
  if ((j / kCovTile) > (i / kCovTile)) Cov[(int64_t)j * d + i] = v;
}

// Y[r, c] = sum_i (X[r, i] - mu_i) W[c, i]  (centring and accumulation in float64); one warp per row, the centred row in
// shared memory (rounded to float once, after the float64 subtraction)
__global__ void __launch_bounds__(256)
pca_project_kernel(const float* __restrict__ X, int64_t N, int d, const double* __restrict__ mean, const float* __restrict__ W,
                   int k, float* __restrict__ Y) {
  extern __shared__ float s_row[];   // [8 warps][d]
  const int lane = threadIdx.x & 31, wib = threadIdx.x >> 5;
  float* xr = s_row + (size_t)wib * d;
  for (int64_t r = (int64_t)blockIdx.x * 8 + wib; r < N; r += (int64_t)gridDim.x * 8) {
    for (int i = lane; i < d; i += 32) xr[i] = (float)((double)X[r * d + i] - mean[i]);
    __syncwarp();
    for (int c = 0; c < k; ++c) {
      double acc = 0.0;
      const float* w = W + (int64_t)c * d;
      for (int i = lane; i < d; i += 32) acc = fma((double)xr[i], (double)__ldg(w + i), acc);
#pragma unroll
      for (int o = 16; o > 0; o >>= 1) acc += __shfl_xor_sync(0xffffffffu, acc, o);
      if (lane == 0) Y[r * k + c] = (float)acc;
    }
    __syncwarp();
  }
}

// ---------------------------------------------------------------- DBSCAN
// adjacency bits + neighbour counts.  Tile: 64 rows (i) x 64 rows (j); thread (ty, tx) owns a 4 x 4 block of pairs.
constexpr int kDbTile = 64, kDbK = 32;
__global__ void __launch_bounds__(256)
dbscan_adj_kernel(const float* __restrict__ X, int N, int d, float eps2, double eps2_exact, uint32_t* __restrict__ adj,
                  int words, int* __restrict__ count) {
  __shared__ float sa[kDbK][kDbTile + 1], sb[kDbK][kDbTile + 1];
  __shared__ uint32_t sbits[kDbTile][2];
  const int i0 = blockIdx.y * kDbTile, j0 = blockIdx.x * kDbTile;
  const int tx = threadIdx.x & 15, ty = threadIdx.x >> 4;
  float acc[4][4] = {};
  for (int k0 = 0; k0 < d; k0 += kDbK) {
    for (int e = threadIdx.x; e < kDbK * kDbTile; e += 256) {
      const int rr = e / kDbK, kk = e - rr * kDbK;   // consecutive threads walk a row: coalesced
      const int k = k0 + kk;
      sa[kk][rr] = (i0 + rr < N && k < d) ? X[(int64_t)(i0 + rr) * d + k] : 0.f;
      sb[kk][rr] = (j0 + rr < N && k < d) ? X[(int64_t)(j0 + rr) * d + k] : 0.f;
    }
    __syncthreads();
#pragma unroll 8
    for (int kk = 0; kk < kDbK; ++kk) {
      float a[4], b[4];
#pragma unroll
      for (int u = 0; u < 4; ++u) {
        a[u] = sa[kk][ty * 4 + u];
        b[u] = sb[kk][tx * 4 + u];
      }
#pragma unroll
      for (int u = 0; u < 4; ++u)
#pragma unroll
        for (int v = 0; v < 4; ++v) {
          const float t = a[u] - b[v];
          acc[u][v] = fmaf(t, t, acc[u][v]);
        }
    }
    __syncthreads();
  }
  if (threadIdx.x < kDbTile * 2) sbits[threadIdx.x >> 1][threadIdx.x & 1] = 0u;
  __syncthreads();
#pragma unroll
  for (int u = 0; u < 4; ++u) {
    const int i = i0 + ty * 4 + u;
    uint32_t bits = 0u;
#pragma unroll
    for (int v = 0; v < 4; ++v) {
      const int j = j0 + tx * 4 + v;
      if (i >= N || j >= N) continue;
      bool in = acc[u][v] <= eps2;
      if (fabsf(acc[u][v] - eps2) <= 1e-5f * eps2 + 1e-12f) {   // too close to call in fp32: decide in float64
        double s = 0.0;
        for (int k = 0; k < d; ++k) {
          const double t = (double)X[(int64_t)i * d + k] - (double)X[(int64_t)j * d + k];
          s = fma(t, t, s);
        }
        in = s <= eps2_exact;
      }
      if (in) bits |= 1u << (tx * 4 + v & 31);
    }
    if (bits) atomicOr(&sbits[ty * 4 + u][(tx * 4) >> 5], bits);
  }
  __syncthreads();
  if (threadIdx.x < kDbTile * 2) {
    const int r = threadIdx.x >> 1, h = threadIdx.x & 1, i = i0 + r;
    const uint32_t b = sbits[r][h];
    if (i < N && (j0 >> 5) + h < words) {
      adj[(int64_t)i * words + (j0 >> 5) + h] = b;
      if (b) atomicAdd(&count[i], __popc(b));
    }
  }
}

// label[i] = i for core points (a forest of singletons), INT_MAX otherwise
__global__ void dbscan_init_kernel(const int* __restrict__ count, int N, int min_samples, int* __restrict__ label,
                                   unsigned char* __restrict__ core) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= N) return;
  const bool c = count[i] >= min_samples;
  core[i] = c ? 1 : 0;
  label[i] = c ? i : 0x7fffffff;
}

// Union-find forest over the core points, stored in label[]: label[x] == x for a root, label[x] < x otherwise.  A root
// only stops being one by a successful atomicCAS that hangs it under a smaller index, and every other write stores an
// ancestor, so a parent read at any time is an ancestor, and the root of a tree is its smallest index.
__device__ __forceinline__ int uf_find(int* parent, int x) {
  for (;;) {   // path halving; terminates because a parent is always smaller than its child
    const int p = __ldcg(parent + x);
    if (p == x) return x;
    const int gp = __ldcg(parent + p);
    if (gp == p) return p;
    // x is not a root, so no atomicCAS targets it.  The store may overwrite a nearer ancestor written meanwhile by
    // another thread; any ancestor is a valid parent while hooking, but not as a final label (see the compress kernel).
    parent[x] = gp;
    x = gp;
  }
}

// hooking: the larger root goes under the smaller; a failed atomicCAS means that root was just hooked elsewhere, so
// continue from its new root.  Each failure moves one of the two to a smaller index, so the loop ends.
__device__ __forceinline__ void uf_union(int* parent, int a, int b) {
  a = uf_find(parent, a);
  b = uf_find(parent, b);
  while (a != b) {
    if (a > b) {
      const int t = a;
      a = b;
      b = t;
    }
    const int old = atomicCAS(parent + b, b, a);
    if (old == b) return;
    b = uf_find(parent, old);
  }
}

// every core-core edge of row i is hooked once from each end; one warp per row, one pass over the bit matrix
__global__ void __launch_bounds__(256)
dbscan_hook_kernel(const uint32_t* __restrict__ adj, int words, int N, const unsigned char* __restrict__ core,
                   int* __restrict__ label) {
  const int lane = threadIdx.x & 31;
  const int i = blockIdx.x * 8 + (threadIdx.x >> 5);
  if (i >= N || !core[i]) return;
  const uint32_t* row = adj + (int64_t)i * words;
  for (int w = lane; w < words; w += 32) {
    uint32_t b = row[w];
    while (b) {
      const int j = w * 32 + __ffs(b) - 1;
      b &= b - 1;
      if (j != i && core[j]) uf_union(label, i, j);
    }
  }
}

// after every hook: each core point takes its root, the lowest core index of its component.  The walk writes nothing
// but label[i] itself: a path-halving store from another thread could land after label[i] = root and put a
// non-root ancestor back.
__global__ void dbscan_compress_kernel(int N, const unsigned char* __restrict__ core, int* __restrict__ label) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= N || !core[i]) return;
  int r = i;
  for (int p = __ldcg(label + r); p != r; p = __ldcg(label + r)) r = p;
  label[i] = r;
}

// border points: the smallest component label among core neighbours (noise: none)
__global__ void __launch_bounds__(256)
dbscan_border_kernel(const uint32_t* __restrict__ adj, int words, int N, const unsigned char* __restrict__ core,
                     const int* __restrict__ label, int* __restrict__ out) {
  const int lane = threadIdx.x & 31;
  const int i = blockIdx.x * 8 + (threadIdx.x >> 5);
  if (i >= N) return;
  int best = core[i] ? label[i] : 0x7fffffff;
  if (!core[i]) {
    const uint32_t* row = adj + (int64_t)i * words;
    for (int w = lane; w < words; w += 32) {
      uint32_t b = row[w];
      while (b) {
        const int j = w * 32 + __ffs(b) - 1;
        b &= b - 1;
        if (core[j]) best = min(best, label[j]);
      }
    }
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) best = min(best, __shfl_xor_sync(0xffffffffu, best, o));
  }
  if (lane == 0) out[i] = best == 0x7fffffff ? -1 : best;
}

}  // namespace am

using namespace am;

extern "C" int am_pca_moments(const float* X, int64_t N, int d, double* mean, double* cov) {
  AM_CHECK(X && mean && cov && N >= 2 && d >= 1 && d <= 8192, "am_pca_moments: bad argument (need N >= 2, 1 <= d <= 8192)");
  cudaStream_t st;
  AM_TRY(HostCall::thread_stream(&st));
  HostCall call(st, 0, HostCall::Memory::Owned);
  float* dX;
  double *dM, *dC;
  call.up(&dX, X, (size_t)N * d);
  call.device(&dM, (size_t)d, 0);
  call.down(&dC, (size_t)d * d, cov, 0);
  AM_TRY(call.start());
  const int slabs = (int)std::max<int64_t>(1, std::min<int64_t>(64, N / 256));
  AM_LAUNCH(col_sum_kernel, dim3((unsigned)ceil_div(d, 128), (unsigned)slabs), 128, 0, st, dX, N, d, dM);
  std::vector<double> hm((size_t)d);
  AM_CUDA(cudaMemcpyAsync(hm.data(), dM, (size_t)d * 8, cudaMemcpyDeviceToHost, st));
  AM_CUDA(cudaStreamSynchronize(st));
  for (int c = 0; c < d; ++c) hm[(size_t)c] /= (double)N;
  AM_CUDA(cudaMemcpyAsync(dM, hm.data(), (size_t)d * 8, cudaMemcpyHostToDevice, st));
  const int tiles = ceil_div(d, kCovTile);
  const int zs = (int)std::max<int64_t>(1, std::min<int64_t>(N / 512, (int64_t)4 * sm_count() / std::max(1, tiles * (tiles + 1) / 2)));
  AM_LAUNCH(cov_kernel, dim3((unsigned)tiles, (unsigned)tiles, (unsigned)std::max(1, zs)), 256, 0, st, dX, N, d, dM, dC);
  AM_LAUNCH(cov_finish_kernel, (unsigned)(((int64_t)d * d + 255) / 256), 256, 0, st, dC, d, 1.0 / (double)(N - 1));
  AM_TRY(call.finish());
  std::copy(hm.begin(), hm.end(), mean);
  return AM_OK;
}

extern "C" int am_pca_project(const float* X, int64_t N, int d, const double* mean, const float* components, int k,
                              float* Y) {
  AM_CHECK(X && mean && components && Y && N >= 1 && d >= 1 && k >= 1 && d <= 8192, "am_pca_project: bad argument");
  cudaStream_t st;
  AM_TRY(HostCall::thread_stream(&st));
  HostCall call(st, 0, HostCall::Memory::Owned);
  float *dX, *dW, *dY;
  double* dM;
  call.up(&dX, X, (size_t)N * d);
  call.up(&dM, mean, (size_t)d);
  call.up(&dW, components, (size_t)k * d);
  call.down(&dY, (size_t)N * k, Y);
  AM_TRY(call.start());
  const size_t smem = (size_t)8 * d * 4;
  AM_CHECK(smem <= 200 * 1024, "am_pca_project: %d features do not fit the row buffer", d);
  AM_TRY(allow_dynamic_smem<pca_project_kernel>(200 * 1024));
  const int grid = (int)std::max<int64_t>(1, std::min<int64_t>((N + 7) / 8, (int64_t)sm_count() * 8));
  AM_LAUNCH(pca_project_kernel, grid, 256, smem, st, dX, N, d, dM, dW, k, dY);
  return call.finish();
}

extern "C" int am_dbscan(const float* X, int64_t N64, int d, double eps, int min_samples, int32_t* labels, int* n_clusters) {
  AM_CHECK(X && labels && N64 >= 1 && N64 <= (1 << 20) && d >= 1 && eps > 0.0 && eps * eps <= 3.0e38 && min_samples >= 1,
           "am_dbscan: bad argument (1 <= N <= 2^20, 0 < eps, eps^2 finite in float, min_samples >= 1)");
  const int N = (int)N64, words = (N + 31) / 32;
  cudaStream_t st;
  AM_TRY(HostCall::thread_stream(&st));
  HostCall call(st, 0, HostCall::Memory::Owned);
  std::vector<int> h((size_t)N);
  float* dX;
  uint32_t* adj;
  int *count, *label, *out;
  unsigned char* core;
  call.up(&dX, X, (size_t)N * d);
  call.down(&out, (size_t)N, h.data());
  call.device(&adj, (size_t)N * words, 0);
  call.device(&count, (size_t)N, 0);
  call.device(&label, (size_t)N);
  call.device(&core, (size_t)N);
  AM_TRY(call.start());
  const unsigned tiles = (unsigned)ceil_div(N, kDbTile);
  const double eps2 = eps * eps;
  AM_LAUNCH(dbscan_adj_kernel, dim3(tiles, tiles), 256, 0, st, dX, N, d, (float)eps2, eps2, adj, words, count);
  AM_LAUNCH(dbscan_init_kernel, (unsigned)ceil_div(N, 256), 256, 0, st, count, N, min_samples, label, core);
  AM_LAUNCH(dbscan_hook_kernel, (unsigned)ceil_div(N, 8), 256, 0, st, adj, words, N, core, label);
  AM_LAUNCH(dbscan_compress_kernel, (unsigned)ceil_div(N, 256), 256, 0, st, N, core, label);
  AM_LAUNCH(dbscan_border_kernel, (unsigned)ceil_div(N, 8), 256, 0, st, adj, words, N, core, label, out);
  AM_TRY(call.finish());
  // component labels are the lowest core index of each component: number them in that order (scikit-learn's numbering)
  std::vector<int> roots;
  for (int i = 0; i < N; ++i)
    if (h[(size_t)i] == i) roots.push_back(i);   // a root is a core point labelled with itself; ascending already
  std::vector<int> rank((size_t)N, -1);
  for (size_t r = 0; r < roots.size(); ++r) rank[(size_t)roots[r]] = (int)r;
  for (int i = 0; i < N; ++i) labels[i] = h[(size_t)i] < 0 ? -1 : rank[(size_t)h[(size_t)i]];
  if (n_clusters) *n_clusters = (int)roots.size();
  return AM_OK;
}
