// UMAP's fuzzy k-NN graph and SGD layout (tasks/song_alchemy.py:272-287 runs umap.UMAP(n_components=2) on the host).
// The host (projection.umap_fit_transform) fits a, b, runs the spectral initialisation through the spectral.cu
// eigensolver and calls the layout; everything O(N) lives here.
//
// Graph (am_umap_plan_create), umap-learn 0.5's fuzzy_simplicial_set with local_connectivity = 1, float64 throughout:
//   k-NN lists               the exact euclidean index of knn.cu (ids ascending distance, ties to the lower id)
//   self_first_kernel        per row: the row itself first, then its k - 1 nearest other rows; true euclidean distances
//                            recomputed in float64 from the ids, and the row sums of those distances
//   sum_kernel               the mean of all N k distances (one CTA, fixed order)
//   smooth_knn_kernel        per row (one thread): rho = the smallest non-zero distance, sigma by the 64-step bisection
//                            to sum_{j >= 1} exp(-(d_j - rho) / sigma) = log2 k, the 1e-3 mean floor; memberships
//   knn_csr_build            (spectral.cu) the fuzzy union W = A + A^T - A o A^T as a CSR, columns ascending
//   max_kernel + prune       entries with w < max(w) / n_epochs dropped; epochs_per_sample = n_epochs / (n_epochs w / max)
//
// Layout (am_umap_plan_layout), one launch per epoch, Jacobi: every vertex reads the previous epoch's embedding and
// writes its own row of the next one, so the result does not depend on scheduling and no atomics are needed.  Both
// directions of an edge carry the same schedule (W is symmetric), and umap moves both endpoints of a sampled edge, so
// a vertex's attraction is twice its sampled row entries' terms; its repulsion comes from the negative samples of its
// own row entries.  Negative samples are drawn from a counter-based hash of (seed, epoch, entry, sample).
#include "common.cuh"

#include <algorithm>
#include <cmath>
#include <memory>

struct am_umap_plan {
  int64_t N = 0;
  int k = 0;
  int n_epochs = 0;
  int64_t nnz = 0;
  float knn_ms = 0.f, graph_ms = 0.f, layout_ms = 0.f;
  am::Stream st;
  am::DevBuf<int64_t> indptr;           // the pruned graph
  am::DevBuf<int32_t> indices;
  am::DevBuf<double> w, eps;            // its weights and epochs_per_sample
  am::DevBuf<double> rho, sigma;
  am::DevBuf<double> next_s, next_n;    // epoch_of_next_sample, epoch_of_next_negative_sample
  am::DevBuf<float> Y0, Y1;             // the embedding, double-buffered
};

namespace am {
namespace um {

constexpr int kSmoothIters = 64;
constexpr double kSmoothTol = 1e-5;
constexpr double kMinKDistScale = 1e-3;

__device__ __forceinline__ uint64_t splitmix64(uint64_t x) {
  x += 0x9E3779B97F4A7C15ull;
  x = (x ^ (x >> 30)) * 0xBF58476D1CE4E5B9ull;
  x = (x ^ (x >> 27)) * 0x94D049BB133111EBull;
  return x ^ (x >> 31);
}

// one warp per row: ids_out[i] = [i, the first k - 1 ids of ids_in[i] other than i], dist = ||x_i - x_j|| in float64
__global__ void __launch_bounds__(256)
self_first_kernel(const float* __restrict__ X, int64_t N, int d, const int64_t* __restrict__ ids_in, int k,
                  int64_t* __restrict__ ids_out, double* __restrict__ dist, double* __restrict__ row_sum) {
  const int lane = threadIdx.x & 31;
  const int64_t row = (int64_t)blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5);
  if (row >= N) return;
  const int64_t* in = ids_in + row * k;
  int64_t* out = ids_out + row * k;
  if (lane == 0) {
    out[0] = row;
    int n = 1;
    for (int p = 0; p < k && n < k; ++p)
      if (in[p] != row) out[n++] = in[p];
  }
  __syncwarp();
  const float* xi = X + row * d;
  double rs = 0.0;
  for (int p = 0; p < k; ++p) {
    const float* xj = X + out[p] * d;
    double s = 0.0;
    for (int c = lane; c < d; c += 32) {
      const double t = (double)xi[c] - (double)xj[c];
      s = fma(t, t, s);
    }
    const double dv = sqrt(warp_sum(s));
    rs += dv;
    if (lane == 0) dist[row * k + p] = dv;
  }
  if (lane == 0) row_sum[row] = rs;
}

// out[0] = sum of v[0, n), one CTA of 1024 threads: strided partial sums, then a fixed tree
__global__ void __launch_bounds__(1024) sum_kernel(const double* __restrict__ v, int64_t n, double* __restrict__ out) {
  __shared__ double part[1024];
  double s = 0.0;
  for (int64_t i = threadIdx.x; i < n; i += 1024) s += v[i];
  part[threadIdx.x] = s;
  __syncthreads();
  for (int h = 512; h > 0; h >>= 1) {
    if ((int)threadIdx.x < h) part[threadIdx.x] += part[threadIdx.x + h];
    __syncthreads();
  }
  if (threadIdx.x == 0) out[0] = part[0];
}

// out[0] = max of v[0, n) (0 when n == 0), one CTA of 1024 threads
__global__ void __launch_bounds__(1024) max_kernel(const double* __restrict__ v, int64_t n, double* __restrict__ out) {
  __shared__ double part[1024];
  double m = 0.0;
  for (int64_t i = threadIdx.x; i < n; i += 1024) m = fmax(m, v[i]);
  part[threadIdx.x] = m;
  __syncthreads();
  for (int h = 512; h > 0; h >>= 1) {
    if ((int)threadIdx.x < h) part[threadIdx.x] = fmax(part[threadIdx.x], part[threadIdx.x + h]);
    __syncthreads();
  }
  if (threadIdx.x == 0) out[0] = part[0];
}

// one thread per row: umap-learn's smooth_knn_dist (local_connectivity 1, bandwidth 1) and the membership strengths
__global__ void smooth_knn_kernel(const int64_t* __restrict__ ids, const double* __restrict__ dist,
                                  const double* __restrict__ row_sum, const double* __restrict__ total, int64_t N, int k,
                                  double* __restrict__ rho_out, double* __restrict__ sigma_out, double* __restrict__ memb) {
  const int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= N) return;
  const double* di = dist + i * k;
  const double target = log2((double)k);
  double rho = 0.0;
  bool has = false;
  for (int j = 0; j < k; ++j)
    if (di[j] > 0.0 && (!has || di[j] < rho)) {
      rho = di[j];
      has = true;
    }
  double lo = 0.0, hi = INFINITY, mid = 1.0;
  for (int it = 0; it < kSmoothIters; ++it) {
    double psum = 0.0;
    for (int j = 1; j < k; ++j) {
      const double t = di[j] - rho;
      psum += t > 0.0 ? exp(-(t / mid)) : 1.0;
    }
    if (fabs(psum - target) < kSmoothTol) break;
    if (psum > target) {
      hi = mid;
      mid = (lo + hi) / 2.0;
    } else {
      lo = mid;
      mid = isinf(hi) ? mid * 2.0 : (lo + hi) / 2.0;
    }
  }
  double sigma = mid;
  const double floor_d = kMinKDistScale * (rho > 0.0 ? row_sum[i] / k : total[0] / ((double)N * k));
  if (sigma < floor_d) sigma = floor_d;
  rho_out[i] = rho;
  sigma_out[i] = sigma;
  for (int j = 0; j < k; ++j) {
    double m;
    if (ids[i * k + j] == i) m = 0.0;
    else if (di[j] - rho <= 0.0 || sigma == 0.0) m = 1.0;
    else m = exp(-((di[j] - rho) / sigma));
    memb[i * k + j] = m;
  }
}

// one warp per row: the number of entries with w >= thr[0] / n_epochs
__global__ void __launch_bounds__(256)
prune_count_kernel(const int64_t* __restrict__ indptr, int64_t N, const double* __restrict__ w,
                   const double* __restrict__ wmax, int n_epochs, int* __restrict__ cnt) {
  const int lane = threadIdx.x & 31;
  const int64_t row = (int64_t)blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5);
  if (row >= N) return;
  const double thr = wmax[0] / (double)n_epochs;
  int c = 0;
  for (int64_t p = indptr[row] + lane; p < indptr[row + 1]; p += 32) c += w[p] >= thr;
#pragma unroll
  for (int s = 16; s > 0; s >>= 1) c += __shfl_xor_sync(0xffffffffu, c, s);
  if (lane == 0) cnt[row] = c;
}

// one warp per row: the kept entries in order, and epochs_per_sample = n_epochs / (n_epochs * (w / max))
__global__ void __launch_bounds__(256)
prune_copy_kernel(const int64_t* __restrict__ indptr, const int32_t* __restrict__ indices, const double* __restrict__ w,
                  int64_t N, const double* __restrict__ wmax, int n_epochs, const int64_t* __restrict__ out_ptr,
                  int32_t* __restrict__ out_idx, double* __restrict__ out_w, double* __restrict__ out_eps) {
  const int lane = threadIdx.x & 31;
  const int64_t row = (int64_t)blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5);
  if (row >= N) return;
  const double mx = wmax[0], thr = mx / (double)n_epochs, ne = (double)n_epochs;
  int64_t out = out_ptr[row];
  for (int64_t p0 = indptr[row]; p0 < indptr[row + 1]; p0 += 32) {
    const int64_t p = p0 + lane;
    const bool keep = p < indptr[row + 1] && w[p] >= thr;
    const unsigned m = __ballot_sync(0xffffffffu, keep);
    if (keep) {
      const int64_t pos = out + __popc(m & ((1u << lane) - 1u));
      out_idx[pos] = indices[p];
      out_w[pos] = w[p];
      out_eps[pos] = ne / (ne * (w[p] / mx));
    }
    out += __popc(m);
  }
}

__global__ void schedule_init_kernel(const double* __restrict__ eps, int64_t nnz, double neg_rate,
                                     double* __restrict__ next_s, double* __restrict__ next_n) {
  for (int64_t e = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; e < nnz; e += (int64_t)gridDim.x * blockDim.x) {
    next_s[e] = eps[e];
    next_n[e] = eps[e] / neg_rate;
  }
}

__device__ __forceinline__ double clip4(double v) { return fmin(fmax(v, -4.0), 4.0); }

// One epoch n, one warp per vertex i; lanes stride over i's row entries and accumulate in float64, the lanes' sums are
// combined by a fixed shuffle tree.  Y_out[i] = Y_in[i] + alpha (2 sum_attr + sum_rep).
__global__ void __launch_bounds__(256)
layout_epoch_kernel(const int64_t* __restrict__ indptr, const int32_t* __restrict__ indices,
                    const double* __restrict__ eps, double* __restrict__ next_s, double* __restrict__ next_n, int64_t N,
                    const float2* __restrict__ Y_in, float2* __restrict__ Y_out, double a, double b, double gamma,
                    double alpha, double neg_rate, int n, uint64_t seed) {
  const int lane = threadIdx.x & 31;
  const int64_t i = (int64_t)blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5);
  if (i >= N) return;
  const float2 yi = Y_in[i];
  const double xi = yi.x, zi = yi.y;
  const double fn = (double)n;
  const uint64_t epoch_key = splitmix64(seed ^ ((uint64_t)n * 0xD1B54A32D192ED03ull));
  double ax = 0.0, az = 0.0, rx = 0.0, rz = 0.0;
  for (int64_t e = indptr[i] + lane; e < indptr[i + 1]; e += 32) {
    const double ns = next_s[e];
    if (ns > fn) continue;
    const double ep = eps[e];
    const float2 yj = Y_in[indices[e]];
    const double dx = xi - yj.x, dz = zi - yj.y;
    const double d2 = dx * dx + dz * dz;
    if (d2 > 0.0) {
      const double c = -2.0 * a * b * pow(d2, b - 1.0) / (a * pow(d2, b) + 1.0);
      ax += clip4(c * dx);
      az += clip4(c * dz);
    }
    next_s[e] = ns + ep;
    const double epn = ep / neg_rate;
    const double nn0 = next_n[e];
    const int n_neg = (int)((fn - nn0) / epn);
    const uint64_t entry_key = splitmix64(epoch_key ^ (uint64_t)e);
    for (int p = 0; p < n_neg; ++p) {
      const int64_t kk = (int64_t)(splitmix64(entry_key ^ (uint64_t)p) % (uint64_t)N);
      if (kk == i) continue;
      const float2 yk = Y_in[kk];
      const double ux = xi - yk.x, uz = zi - yk.y;
      const double q2 = ux * ux + uz * uz;
      if (q2 <= 0.0) continue;  // coincident points push each other nowhere
      const double c = 2.0 * gamma * b / ((0.001 + q2) * (a * pow(q2, b) + 1.0));
      if (c > 0.0) {
        rx += clip4(c * ux);
        rz += clip4(c * uz);
      }
    }
    next_n[e] = nn0 + (double)n_neg * epn;
  }
  const double gx = warp_sum(2.0 * ax + rx), gz = warp_sum(2.0 * az + rz);
  if (lane == 0) Y_out[i] = make_float2((float)(xi + alpha * gx), (float)(zi + alpha * gz));
}

int warp_rows_grid(int64_t rows) { return (int)std::max<int64_t>(1, (rows + 7) / 8); }

}  // namespace um
}  // namespace am

using namespace am;

extern "C" int am_umap_plan_create(const float* X, int64_t N, int d, int n_neighbors, int n_epochs,
                                   am_umap_plan** out) {
  AM_CHECK(X && out && N >= 2 && d >= 1, "am_umap_plan_create: bad argument (need X, out, N >= 2, d >= 1)");
  AM_CHECK(N <= (int64_t)INT32_MAX, "am_umap_plan_create: N = %lld exceeds 2^31 - 1 (int32 column indices)",
           (long long)N);
  AM_CHECK(n_neighbors >= 1 && n_neighbors <= N, "am_umap_plan_create: n_neighbors = %d outside [1, N = %lld]",
           n_neighbors, (long long)N);
  AM_CHECK(n_epochs >= 1, "am_umap_plan_create: n_epochs = %d must be positive", n_epochs);
  *out = nullptr;
  AM_TRY(ensure_init());
  std::unique_ptr<am_umap_plan> p(new am_umap_plan());
  p->N = N;
  p->k = n_neighbors;
  p->n_epochs = n_epochs;
  AM_TRY(p->st.create());
  Event ev[3];
  for (auto& e : ev) AM_TRY(e.create());
  cudaStream_t st = p->st.s;
  const int k = n_neighbors;
  DevBuf<float> dX, kdist;
  DevBuf<int64_t> kids, ids, u_ptr;
  DevBuf<double> dist, row_sum, total, memb, u_w, wmax;
  DevBuf<int32_t> u_idx;
  DevBuf<int> cnt;
  AM_TRY(knn_self_query(X, N, d, k, st, ev[0], ev[1], dX, kids, kdist));
  AM_TRY(ids.alloc((size_t)N * k));
  AM_TRY(dist.alloc((size_t)N * k));
  AM_TRY(row_sum.alloc((size_t)N));
  AM_TRY(total.alloc(1));
  AM_TRY(memb.alloc((size_t)N * k));
  AM_TRY(p->rho.alloc((size_t)N));
  AM_TRY(p->sigma.alloc((size_t)N));
  AM_LAUNCH(um::self_first_kernel, um::warp_rows_grid(N), 256, 0, st, dX.p, N, d, kids.p, k, ids.p, dist.p,
            row_sum.p);
  AM_LAUNCH(um::sum_kernel, 1, 1024, 0, st, row_sum.p, N, total.p);
  AM_LAUNCH(um::smooth_knn_kernel, (unsigned)((N + 127) / 128), 128, 0, st, ids.p, dist.p, row_sum.p, total.p, N, k,
            p->rho.p, p->sigma.p, memb.p);
  int64_t u_nnz = 0;
  AM_TRY(knn_csr_build(ids.p, memb.p, N, k, st, u_ptr, u_idx, nullptr, nullptr, &u_w, &u_nnz));
  AM_TRY(wmax.alloc(1));
  AM_TRY(cnt.alloc((size_t)N));
  AM_TRY(p->indptr.alloc((size_t)N + 1));
  AM_LAUNCH(um::max_kernel, 1, 1024, 0, st, u_w.p, u_nnz, wmax.p);
  AM_LAUNCH(um::prune_count_kernel, um::warp_rows_grid(N), 256, 0, st, u_ptr.p, N, u_w.p, wmax.p, n_epochs, cnt.p);
  AM_TRY(csr_scan(cnt.p, N, p->indptr.p, st));
  AM_CUDA(cudaMemcpyAsync(&p->nnz, p->indptr.p + N, 8, cudaMemcpyDeviceToHost, st));
  AM_CUDA(cudaStreamSynchronize(st));
  const size_t m = (size_t)std::max<int64_t>(1, p->nnz);
  AM_TRY(p->indices.alloc(m));
  AM_TRY(p->w.alloc(m));
  AM_TRY(p->eps.alloc(m));
  AM_TRY(p->next_s.alloc(m));
  AM_TRY(p->next_n.alloc(m));
  AM_TRY(p->Y0.alloc((size_t)N * 2));
  AM_TRY(p->Y1.alloc((size_t)N * 2));
  AM_LAUNCH(um::prune_copy_kernel, um::warp_rows_grid(N), 256, 0, st, u_ptr.p, u_idx.p, u_w.p, N, wmax.p, n_epochs,
            p->indptr.p, p->indices.p, p->w.p, p->eps.p);
  AM_CUDA(cudaEventRecord(ev[2].e, st));
  AM_CUDA(cudaStreamSynchronize(st));
  AM_TRY(add_elapsed_ms(p->knn_ms, ev[0], ev[1]));
  AM_TRY(add_elapsed_ms(p->graph_ms, ev[1], ev[2]));
  *out = p.release();
  return AM_OK;
}

extern "C" int am_umap_plan_info(const am_umap_plan* p, int64_t* nnz, int* n_neighbors, int* n_epochs, float* knn_ms,
                                 float* graph_ms, float* layout_ms) {
  AM_CHECK(p, "am_umap_plan_info: NULL plan");
  if (nnz) *nnz = p->nnz;
  if (n_neighbors) *n_neighbors = p->k;
  if (n_epochs) *n_epochs = p->n_epochs;
  if (knn_ms) *knn_ms = p->knn_ms;
  if (graph_ms) *graph_ms = p->graph_ms;
  if (layout_ms) *layout_ms = p->layout_ms;
  return AM_OK;
}

extern "C" int am_umap_plan_graph(am_umap_plan* p, int64_t* indptr, int32_t* indices, double* weights, double* rho,
                                  double* sigma, double* epochs_per_sample) {
  AM_CHECK(p, "am_umap_plan_graph: NULL plan");
  cudaStream_t st = p->st.s;
  const size_t nnz = (size_t)p->nnz, N = (size_t)p->N;
  if (indptr) AM_CUDA(cudaMemcpyAsync(indptr, p->indptr.p, (N + 1) * 8, cudaMemcpyDeviceToHost, st));
  if (indices && nnz) AM_CUDA(cudaMemcpyAsync(indices, p->indices.p, nnz * 4, cudaMemcpyDeviceToHost, st));
  if (weights && nnz) AM_CUDA(cudaMemcpyAsync(weights, p->w.p, nnz * 8, cudaMemcpyDeviceToHost, st));
  if (epochs_per_sample && nnz) AM_CUDA(cudaMemcpyAsync(epochs_per_sample, p->eps.p, nnz * 8, cudaMemcpyDeviceToHost, st));
  if (rho) AM_CUDA(cudaMemcpyAsync(rho, p->rho.p, N * 8, cudaMemcpyDeviceToHost, st));
  if (sigma) AM_CUDA(cudaMemcpyAsync(sigma, p->sigma.p, N * 8, cudaMemcpyDeviceToHost, st));
  AM_CUDA(cudaStreamSynchronize(st));
  return AM_OK;
}

extern "C" int am_umap_plan_layout(am_umap_plan* p, float* emb, int epochs, double a, double b, double gamma,
                                   double alpha0, double neg_rate, uint64_t seed) {
  AM_CHECK(p && emb, "am_umap_plan_layout: NULL argument");
  AM_CHECK(epochs >= 0 && epochs <= p->n_epochs, "am_umap_plan_layout: epochs = %d outside [0, n_epochs = %d]", epochs,
           p->n_epochs);
  AM_CHECK(a > 0.0 && b > 0.0 && gamma >= 0.0 && neg_rate > 0.0 && std::isfinite(a) && std::isfinite(b) &&
               std::isfinite(gamma) && std::isfinite(alpha0) && std::isfinite(neg_rate),
           "am_umap_plan_layout: need finite a > 0, b > 0, gamma >= 0, neg_rate > 0 and alpha0");
  cudaStream_t st = p->st.s;
  const int64_t N = p->N;
  Event ev[2];
  for (auto& e : ev) AM_TRY(e.create());
  AM_CUDA(cudaMemcpyAsync(p->Y0.p, emb, (size_t)N * 8, cudaMemcpyHostToDevice, st));
  if (p->nnz > 0)
    AM_LAUNCH(um::schedule_init_kernel, (unsigned)std::min<int64_t>((p->nnz + 255) / 256, (int64_t)sm_count() * 8),
              256, 0, st, p->eps.p, p->nnz, neg_rate, p->next_s.p, p->next_n.p);
  AM_CUDA(cudaEventRecord(ev[0].e, st));
  float* cur = p->Y0.p;
  float* nxt = p->Y1.p;
  for (int n = 0; n < epochs; ++n) {
    const double alpha = alpha0 * (1.0 - (double)n / (double)p->n_epochs);
    AM_LAUNCH(um::layout_epoch_kernel, um::warp_rows_grid(N), 256, 0, st, p->indptr.p, p->indices.p, p->eps.p,
              p->next_s.p, p->next_n.p, N, reinterpret_cast<const float2*>(cur), reinterpret_cast<float2*>(nxt), a, b,
              gamma, alpha, neg_rate, n, seed);
    std::swap(cur, nxt);
  }
  AM_CUDA(cudaEventRecord(ev[1].e, st));
  AM_CUDA(cudaMemcpyAsync(emb, cur, (size_t)N * 8, cudaMemcpyDeviceToHost, st));
  AM_CUDA(cudaStreamSynchronize(st));
  p->layout_ms = 0.f;  // the latest layout's time, not a sum over calls
  return add_elapsed_ms(p->layout_ms, ev[0], ev[1]);
}

extern "C" void am_umap_plan_free(am_umap_plan* p) {
  if (p && p->st.s) cudaStreamSynchronize(p->st.s);
  delete p;
}
