// K5: Lloyd k-means (sm_90a).  Replaces cuml.cluster.KMeans(...).fit_predict as called by
// tasks/clustering_gpu.py:100-123 (k-means++ init, n_init restarts, labels + cluster_centers_).
//
// Per Lloyd iteration, k <= 128 (kmeans_tc.cu): the assignment is a split-bf16 wgmma GEMM with a fused argmin
// epilogue (+ an exact fp32 recheck of near-ties), the partial sums a sort-by-label pass that reads every row
// once -- two passes over the data per iteration, HBM-bound.  This file keeps the driver (k-means++ seeding,
// sklearn's tolerance / empty-cluster rules, restarts) and the CUDA-core kernels that serve k > 128 and small
// problems:
//   assign   one warp per point; centres streamed through L1/L2; argmin_c (||c||^2 - 2 x.c) by exact_argmin
//            (kmeans_tc.cuh), lowest index wins ties; inertia accumulated in float64  (compute-bound on CUDA cores);
//   update   label-segmented column sums in shared memory ([k, W] slab per CTA, W columns),
//            flushed with one global atomicAdd per (centre, column) per CTA.
// Multi-GPU (dist.py): rows stay sharded; am_kmeans_plan_step / am_kmeans_assign_dev produce per-rank partial
// sums / counts which the host all-reduces (NCCL) before dividing.
#include "common.cuh"
#include "gemm_wgmma.cuh"
#include "host_call.cuh"
#include "kmeans_common.cuh"
#include "kmeans_tc.cuh"

#include <algorithm>
#include <cmath>

namespace am {

__global__ void center_norms_kernel(const float* __restrict__ C, int k, int d, float* __restrict__ cn) {
  const int j = blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5);
  const int lane = threadIdx.x & 31;
  if (j >= k) return;
  const float acc = warp_sq_norm(C + (int64_t)j * d, d, lane);
  if (lane == 0) cn[j] = acc;
}

// one warp per point; each lane keeps up to 16 features of x in registers per 512-chunk
__global__ void __launch_bounds__(256)
assign_kernel(const float* __restrict__ X, int64_t N, int d, const float* __restrict__ C,
              const float* __restrict__ cn, int k, int32_t* __restrict__ labels,
              float* __restrict__ counts, double* __restrict__ inertia, float* __restrict__ dist) {
  __shared__ double s_inertia[8];
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  const int warps = blockDim.x >> 5;
  double local = 0.0;
  for (int64_t row = (int64_t)blockIdx.x * warps + warp; row < N; row += (int64_t)gridDim.x * warps) {
    const float* x = X + row * d;
    float best = INFINITY;
    int best_j = 0;
    const float xn = warp_sq_norm(x, d, lane);
    for (int j = 0; j < k; ++j) exact_argmin<1, 1>(x, d, C, cn, k, lane, j, best, best_j);
    if (lane == 0) {
      labels[row] = best_j;
      if (counts) atomicAdd(&counts[best_j], 1.0f);
      if (dist) dist[row] = fmaxf(best + xn, 0.0f);
      local += (double)fmaxf(best + xn, 0.0f);
    }
  }
  if (lane == 0) s_inertia[warp] = local;
  __syncthreads();
  if (threadIdx.x == 0 && inertia) {
    double t = 0.0;
    for (int w = 0; w < warps; ++w) t += s_inertia[w];
    atomicAdd(inertia, t);
  }
}

// sums[label[i], c0:c0+W] += X[i, c0:c0+W] for a chunk of points, via a smem slab [k, W]
__global__ void __launch_bounds__(256)
accumulate_kernel(const float* __restrict__ X, int64_t N, int d, const int32_t* __restrict__ labels, int k,
                  int W, int points_per_cta, float* __restrict__ sums) {
  extern __shared__ float s_acc[];  // [k * W]
  const int c0 = blockIdx.y * W;
  const int wcols = min(W, d - c0);
  for (int i = threadIdx.x; i < k * W; i += blockDim.x) s_acc[i] = 0.f;
  __syncthreads();
  const int64_t p0 = (int64_t)blockIdx.x * points_per_cta;
  const int64_t p1 = min(N, p0 + points_per_cta);
  const int rows_per_iter = blockDim.x / W;  // W divides blockDim.x
  const int col = threadIdx.x % W, r = threadIdx.x / W;
  for (int64_t p = p0 + r; p < p1; p += rows_per_iter) {
    if (col < wcols) atomicAdd(&s_acc[labels[p] * W + col], X[p * d + c0 + col]);
  }
  __syncthreads();
  for (int i = threadIdx.x; i < k * W; i += blockDim.x) {
    const int j = i / W, c = i % W;
    const float v = s_acc[i];
    if (c < wcols && v != 0.f) atomicAdd(&sums[(int64_t)j * d + c0 + c], v);
  }
}

// C_new = sums / counts; shift2 += ||C_new - C||^2.  A cluster that is still empty takes the new centre of cluster
// `big` (sklearn's _average_centers: the first largest cluster), or keeps its centre when big < 0.
__global__ void update_centers_kernel(const float* __restrict__ sums, const float* __restrict__ counts, int k,
                                      int d, int big, float* __restrict__ C, double* __restrict__ shift2) {
  const int j = blockIdx.x;
  const int src = counts[j] > 0.f || big < 0 ? j : big;
  const float cnt = counts[src];
  double local = 0.0;
  for (int i = threadIdx.x; i < d; i += blockDim.x) {
    const float old = C[(int64_t)j * d + i];
    const float nw = cnt > 0.f ? sums[(int64_t)src * d + i] / cnt : old;
    C[(int64_t)j * d + i] = nw;
    const double df = (double)nw - (double)old;
    local += df * df;
  }
  local = warp_sum(local);
  if ((threadIdx.x & 31) == 0) atomicAdd(shift2, local);
}

// sklearn's _relocate_empty_clusters_dense (sklearn/cluster/_k_means_common.pyx): each empty cluster takes the
// point that is farthest from its own centre (next farthest for the next empty cluster, ...); that point's row
// leaves the sums / counts of the cluster it was assigned to.  One CTA, the reassignments are sequential because
// two of them may hit the same donor cluster.  Labels are NOT changed here (as in sklearn: the next E-step does).
__global__ void relocate_empty_kernel(const float* __restrict__ X, int d, const int32_t* __restrict__ labels,
                                      const int64_t* __restrict__ far_rows, const int32_t* __restrict__ empty_ids,
                                      int n_empty, float* __restrict__ sums, float* __restrict__ counts) {
  for (int e = 0; e < n_empty; ++e) {
    const int64_t row = far_rows[e];
    const int donor = labels[row], target = empty_ids[e];
    for (int i = threadIdx.x; i < d; i += blockDim.x) {
      const float v = X[row * d + i];
      sums[(int64_t)donor * d + i] -= v;
      sums[(int64_t)target * d + i] = v;
    }
    __syncthreads();
    if (threadIdx.x == 0) {
      counts[target] = 1.0f;
      counts[donor] -= 1.0f;
    }
    __syncthreads();
  }
}

// X[i, :] -= mu (sign < 0) or += mu (sign > 0) for the N rows of X [N, d]
__global__ void shift_rows_kernel(float* __restrict__ X, int64_t N, int d, const float* __restrict__ mu, int sign) {
  const int64_t n = N * d;
  for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (int64_t)gridDim.x * blockDim.x)
    X[i] = sign < 0 ? X[i] - mu[i % d] : X[i] + mu[i % d];
}

// per-feature sums of X and X^2 in float64 (column means and sklearn's tol scaling)
__global__ void column_moments_kernel(const float* __restrict__ X, int64_t N, int d, double* __restrict__ s1,
                                      double* __restrict__ s2) {
  const int c = blockIdx.x * blockDim.x + threadIdx.x;
  if (c >= d) return;
  const int64_t chunk = (N + gridDim.y - 1) / gridDim.y;
  const int64_t p0 = (int64_t)blockIdx.y * chunk, p1 = min(N, p0 + chunk);
  double a = 0.0, b = 0.0;
  for (int64_t p = p0; p < p1; ++p) {
    const double v = (double)X[p * d + c];
    a += v;
    b += v * v;
  }
  atomicAdd(&s1[c], a);
  atomicAdd(&s2[c], b);
}

// k-means++: mind2[i] = min(mind2[i], ||x_i - c||^2); per-block partial sums of mind2
__global__ void __launch_bounds__(256)
pp_update_kernel(const float* __restrict__ X, int64_t N, int d, const float* __restrict__ c, int first,
                 float* __restrict__ mind2, double* __restrict__ block_sums) {
  __shared__ double s_part[8];
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  const int64_t base = (int64_t)blockIdx.x * kKppBlock;
  double part = 0.0;
  for (int r = warp; r < kKppBlock; r += 8) {
    const int64_t row = base + r;
    if (row >= N) break;
    float acc[1];
    d2_chains<1>(X + row * d, c, 0, 1, d, lane, acc);
    if (lane == 0) {
      const float m = first ? acc[0] : fminf(mind2[row], acc[0]);
      mind2[row] = m;
      part += (double)m;
    }
  }
  if (lane == 0) s_part[warp] = part;
  __syncthreads();
  if (threadIdx.x == 0) {
    double t = 0.0;
    for (int w = 0; w < 8; ++w) t += s_part[w];
    block_sums[blockIdx.x] = t;
  }
}

// greedy k-means++ (sklearn's _kmeans_plusplus): for each of L candidate rows, the potential
// sum_i min(mind2[i], ||x_i - c_l||^2); per-block partial sums -> block_pot[block][L]
__global__ void __launch_bounds__(256)
pp_trial_kernel(const float* __restrict__ X, int64_t N, int d, const float* __restrict__ cand, int L,
                const float* __restrict__ mind2, double* __restrict__ block_pot) {
  __shared__ double s_part[8][kMaxTrials];
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  const int64_t base = (int64_t)blockIdx.x * kKppBlock;
  double part[kMaxTrials];
#pragma unroll
  for (int l = 0; l < kMaxTrials; ++l) part[l] = 0.0;
  for (int r = warp; r < kKppBlock; r += 8) {
    const int64_t row = base + r;
    if (row >= N) break;
    float acc[kMaxTrials];
    d2_chains<kMaxTrials>(X + row * d, cand, d, L, d, lane, acc);
    const float m = mind2[row];
#pragma unroll
    for (int l = 0; l < kMaxTrials; ++l)
      if (l < L) part[l] += (double)fminf(m, acc[l]);
  }
  if (lane == 0) {
#pragma unroll
    for (int l = 0; l < kMaxTrials; ++l) s_part[warp][l] = part[l];
  }
  __syncthreads();
  if (threadIdx.x < kMaxTrials) {
    double t = 0.0;
    for (int w = 0; w < 8; ++w) t += s_part[w][threadIdx.x];
    block_pot[(int64_t)blockIdx.x * kMaxTrials + threadIdx.x] = t;
  }
}

static int launch_accumulate(const float* X, int64_t N, int d, const int32_t* labels, int k, float* sums,
                             cudaStream_t st) {
  const int W = k <= 128 ? 128 : (k <= 256 ? 64 : 32);
  const size_t smem = (size_t)k * W * 4;
  AM_CHECK(smem <= 200 * 1024, "kmeans: k=%d too large for the shared-memory accumulation slab", k);
  AM_TRY(allow_dynamic_smem<accumulate_kernel>(200 * 1024));
  const int ppc = 4096;
  dim3 grid((unsigned)((N + ppc - 1) / ppc), (unsigned)ceil_div(d, W));
  AM_LAUNCH(accumulate_kernel, grid, 256, smem, st, X, N, d, labels, k, W, ppc, sums);
  return AM_OK;
}

__global__ void f64_to_f32_kernel(const double* in, float* out) { out[0] = (float)in[0]; }

// The one choice between the two Lloyd steps.  The tensor-core step (kmeans_tc.cu) is eligible when
// gemm::available(), 1 <= k <= 128 (the widest assign_tc_kernel), 1 <= d <= 4096 (the recheck band assumes fp32
// accumulation over at most 4096 terms) and 1 <= N < 2^31 (int32 row lists).  It first builds a split-bf16 copy of
// the rows, so it serves
//   KMeansUse::kPlan     every eligible shape: a plan is made to be stepped many times;
//   KMeansUse::kFit      an eligible shape with N k d >= 5e7 (a whole am_kmeans_fit);
//   KMeansUse::kAssign   an eligible shape with N k d >= 2e9 (one am_kmeans_assign_dev step pays for the copy alone).
// Everything else runs on CUDA cores, the only path for k > 128 or d > 4096.
bool kmeans_use_tensor_cores(int64_t N, int d, int k, KMeansUse use) {
  if (!gemm::available() || k < 1 || k > 128 || d < 1 || d > 4096 || N < 1 || N >= ((int64_t)1 << 31)) return false;
  const double work = (double)N * k * d;
  return use == KMeansUse::kPlan || (use == KMeansUse::kFit && work >= 5e7) ||
         (use == KMeansUse::kAssign && work >= 2e9);
}

}  // namespace am

using namespace am;

int am_kmeans_plan::create(bool tensor_cores, cudaStream_t st) {
  AM_TRY(inert.alloc(1));
  if (!tensor_cores) return cn.alloc(k);
  tc.reset(new kmtc::Plan{X, N, d, k});
  return tc->create(st);
}

int am_kmeans_plan::step(const float* C, int32_t* labels, float* sums, float* counts, double* inertia, float* dist,
                         cudaStream_t st) {
  if (tc) return tc->step(C, labels, sums, counts, inertia, dist, st);
  AM_LAUNCH(center_norms_kernel, ceil_div(k, 8), 256, 0, st, C, k, d, cn.p);
  if (counts) AM_CUDA(cudaMemsetAsync(counts, 0, (size_t)k * 4, st));
  if (inertia) AM_CUDA(cudaMemsetAsync(inertia, 0, 8, st));
  const int grid = (int)std::max<int64_t>(1, std::min<int64_t>((N + 7) / 8, (int64_t)sm_count() * 8));
  AM_LAUNCH(assign_kernel, grid, 256, 0, st, X, N, d, C, cn.p, k, labels, counts, inertia, dist);
  if (sums) {
    AM_CUDA(cudaMemsetAsync(sums, 0, (size_t)k * d * 4, st));
    AM_TRY(launch_accumulate(X, N, d, labels, k, sums, st));
  }
  return AM_OK;
}

extern "C" int am_kmeans_assign_dev(const float* X_dev, int64_t N, int d, const float* centers_dev, int k,
                                    int32_t* labels_dev, float* sums_dev, float* counts_dev, float* inertia_dev,
                                    void* stream) {
  AM_CHECK(X_dev && centers_dev && labels_dev, "am_kmeans_assign_dev: NULL argument");
  AM_CHECK(N > 0 && d > 0 && k > 0, "am_kmeans_assign_dev: bad shape");
  AM_TRY(ensure_init());
  am_kmeans_plan p{X_dev, N, d, k};
  AM_TRY(p.create(kmeans_use_tensor_cores(N, d, k, KMeansUse::kAssign), (cudaStream_t)stream));
  AM_TRY(am_kmeans_plan_step(&p, centers_dev, labels_dev, sums_dev, counts_dev, inertia_dev, nullptr, stream));
  AM_CUDA(cudaStreamSynchronize((cudaStream_t)stream));  // the step's scratch is freed on return
  return AM_OK;
}

// ---- iterative device API: the split-bf16 copy of the rows is built once and reused by every Lloyd step
extern "C" int am_kmeans_plan_create(const float* X_dev, int64_t N, int d, int k, void* stream, am_kmeans_plan** out) {
  AM_CHECK(out != nullptr, "am_kmeans_plan_create: out is NULL");
  *out = nullptr;
  AM_CHECK(X_dev && N > 0 && d > 0 && k > 0, "am_kmeans_plan_create: bad argument");
  AM_TRY(ensure_init());
  std::unique_ptr<am_kmeans_plan> p(new am_kmeans_plan{X_dev, N, d, k});
  AM_TRY(p->create(kmeans_use_tensor_cores(N, d, k, KMeansUse::kPlan), (cudaStream_t)stream));
  *out = p.release();
  return AM_OK;
}

extern "C" void am_kmeans_plan_free(am_kmeans_plan* p) {
  if (p) cudaDeviceSynchronize();
  delete p;
}

// rows the last step handed to the exact recheck kernel (near-ties inside the tensor-core error band); synchronises
extern "C" int am_kmeans_plan_last_recheck(am_kmeans_plan* p, void* stream, int* n_rows) {
  AM_CHECK(p && n_rows, "am_kmeans_plan_last_recheck: NULL argument");
  *n_rows = 0;
  if (!p->tc) return AM_OK;
  AM_CUDA(cudaMemcpyAsync(n_rows, p->tc->scal.p + 1, sizeof(int), cudaMemcpyDeviceToHost, (cudaStream_t)stream));
  AM_CUDA(cudaStreamSynchronize((cudaStream_t)stream));
  return AM_OK;
}

extern "C" int am_kmeans_plan_uses_tensor_cores(const am_kmeans_plan* p) { return p && p->tc ? 1 : 0; }

extern "C" int am_kmeans_plan_step(am_kmeans_plan* p, const float* centers_dev, int32_t* labels_dev, float* sums_dev,
                                   float* counts_dev, float* inertia_dev, float* dist_dev, void* stream) {
  AM_CHECK(p && centers_dev && labels_dev, "am_kmeans_plan_step: NULL argument");
  cudaStream_t st = (cudaStream_t)stream;
  AM_TRY(p->step(centers_dev, labels_dev, sums_dev, counts_dev, inertia_dev ? p->inert.p : nullptr, dist_dev, st));
  if (inertia_dev) AM_LAUNCH(f64_to_f32_kernel, 1, 1, 0, st, p->inert.p, inertia_dev);
  return AM_OK;  // stream-ordered: no synchronisation
}

// sklearn: tol_ = mean(var(X, axis=0)) * tol; mean[d] = the column means of X (rounded to float32)
static int scaled_tolerance(const float* X, int64_t N, int d, float tol, cudaStream_t st, double* tol_abs,
                            std::vector<float>& mean) {
  DevBuf<double> mom;
  AM_TRY(mom.alloc((size_t)2 * d));
  AM_CUDA(cudaMemsetAsync(mom.p, 0, (size_t)2 * d * 8, st));
  dim3 grid(ceil_div(d, 128), (unsigned)std::max<int64_t>(1, std::min<int64_t>(256, N / 1024)));
  AM_LAUNCH(column_moments_kernel, grid, 128, 0, st, X, N, d, mom.p, mom.p + d);
  std::vector<double> hm((size_t)2 * d);
  AM_CUDA(cudaMemcpyAsync(hm.data(), mom.p, hm.size() * 8, cudaMemcpyDeviceToHost, st));
  AM_CUDA(cudaStreamSynchronize(st));
  mean.resize((size_t)d);
  *tol_abs = kmeans_tol_abs(hm.data(), hm.data() + d, N, d, tol, mean.data());
  return AM_OK;
}

// greedy k-means++ into C [k, d] (D^2 sampling with 2 + ln k local trials, as sklearn / cuML do), on the device scratch
// mind2 f32[N], bsum f64[nblk], cand f32[kMaxTrials, d], bpot f64[nblk, kMaxTrials] (nblk 1024-row blocks)
static int kmeanspp_seed(const float* X, int64_t N, int d, int k, SplitMix& rng, float* C, float* mind2,
                         double* bsum, float* cand, double* bpot, cudaStream_t st) {
  const int64_t nblk = (N + kKppBlock - 1) / kKppBlock;
  std::vector<double> hbs(nblk), hpot((size_t)nblk * kMaxTrials);
  std::vector<float> hblock(kKppBlock);
  const int L = kpp_trials(k);
  int64_t pick = std::min<int64_t>((int64_t)(rng.uniform() * N), N - 1);
  AM_CUDA(cudaMemcpyAsync(C, X + (size_t)pick * d, (size_t)d * 4, cudaMemcpyDeviceToDevice, st));
  AM_LAUNCH(pp_update_kernel, (unsigned)nblk, 256, 0, st, X, N, d, C, 1, mind2, bsum);
  for (int j = 1; j < k; ++j) {
    AM_CUDA(cudaMemcpyAsync(hbs.data(), bsum, nblk * 8, cudaMemcpyDeviceToHost, st));
    AM_CUDA(cudaStreamSynchronize(st));
    double total = 0.0;
    for (double v : hbs) total += v;
    int64_t cand_row[kMaxTrials];
    for (int l = 0; l < L; ++l) {
      double r = rng.uniform() * total;
      const int64_t b0 = kpp_scan(hbs.data(), nblk, r) * kKppBlock, cnt = std::min<int64_t>(kKppBlock, N - b0);
      AM_CUDA(cudaMemcpyAsync(hblock.data(), mind2 + b0, cnt * 4, cudaMemcpyDeviceToHost, st));
      AM_CUDA(cudaStreamSynchronize(st));
      cand_row[l] = b0 + kpp_scan(hblock.data(), cnt, r);
      AM_CUDA(cudaMemcpyAsync(cand + (size_t)l * d, X + (size_t)cand_row[l] * d, (size_t)d * 4,
                              cudaMemcpyDeviceToDevice, st));
    }
    AM_LAUNCH(pp_trial_kernel, (unsigned)nblk, 256, 0, st, X, N, d, cand, L, mind2, bpot);
    AM_CUDA(cudaMemcpyAsync(hpot.data(), bpot, (size_t)nblk * kMaxTrials * 8, cudaMemcpyDeviceToHost, st));
    AM_CUDA(cudaStreamSynchronize(st));
    int best = 0;
    double best_pot = INFINITY;
    for (int l = 0; l < L; ++l) {
      double pot = 0.0;
      for (int64_t b = 0; b < nblk; ++b) pot += hpot[(size_t)b * kMaxTrials + l];
      if (pot < best_pot) {
        best_pot = pot;
        best = l;
      }
    }
    AM_CUDA(cudaMemcpyAsync(C + (size_t)j * d, cand + (size_t)best * d, (size_t)d * 4, cudaMemcpyDeviceToDevice,
                            st));
    if (j < k - 1)
      AM_LAUNCH(pp_update_kernel, (unsigned)nblk, 256, 0, st, X, N, d, C + (size_t)j * d, 0, mind2, bsum);
  }
  return AM_OK;
}

// sklearn's Lloyd from the centres in C, at most max_iter steps: after each E-step, empty clusters are relocated as
// sklearn does it, then the centres move; stops once the squared shift is <= tol_abs.  *n_iter = the steps run.
static int lloyd(am_kmeans_plan& step, int max_iter, double tol_abs, float* C, int32_t* labels, float* sums,
                 float* counts, float* dist, double* shift2_dev, cudaStream_t st, int* n_iter) {
  const int64_t N = step.N;
  const int d = step.d, k = step.k;
  std::vector<float> hcounts((size_t)k), hdist;
  DevBuf<int64_t> far_dev;
  DevBuf<int32_t> empty_dev;
  int it = 0;
  for (it = 1; it <= max_iter; ++it) {
    AM_TRY(step.step(C, labels, sums, counts, nullptr, dist, st));
    // empty clusters are relocated the way sklearn's Lloyd does it (rare: costs one [k] read-back per
    // iteration, and the [N] distances only when a cluster actually emptied)
    AM_CUDA(cudaMemcpyAsync(hcounts.data(), counts, (size_t)k * 4, cudaMemcpyDeviceToHost, st));
    AM_CUDA(cudaStreamSynchronize(st));
    std::vector<int32_t> empty;
    for (int j = 0; j < k; ++j)
      if (hcounts[j] == 0.f) empty.push_back(j);
    int big = -1;
    if (!empty.empty()) {
      hdist.resize((size_t)N);
      AM_CUDA(cudaMemcpyAsync(hdist.data(), dist, (size_t)N * 4, cudaMemcpyDeviceToHost, st));
      AM_CUDA(cudaStreamSynchronize(st));
    }
    // as sklearn: with every row on its centre (more clusters than distinct rows) relocation is pointless, and the
    // empty clusters move to the first largest cluster's centre instead
    if (!empty.empty() && *std::max_element(hdist.begin(), hdist.end()) == 0.f)
      big = (int)(std::max_element(hcounts.begin(), hcounts.end()) - hcounts.begin());
    else if (!empty.empty()) {
      std::vector<int64_t> order((size_t)N);
      for (int64_t i = 0; i < N; ++i) order[(size_t)i] = i;
      std::partial_sort(order.begin(), order.begin() + (int64_t)empty.size(), order.end(), [&](int64_t a, int64_t b) {
        return relocate_before(hdist[(size_t)a], a, hdist[(size_t)b], b);
      });
      AM_TRY(far_dev.alloc(empty.size()));
      AM_TRY(empty_dev.alloc(empty.size()));
      AM_CUDA(cudaMemcpyAsync(far_dev.p, order.data(), empty.size() * 8, cudaMemcpyHostToDevice, st));
      AM_CUDA(cudaMemcpyAsync(empty_dev.p, empty.data(), empty.size() * 4, cudaMemcpyHostToDevice, st));
      AM_LAUNCH(relocate_empty_kernel, 1, 256, 0, st, step.X, d, labels, far_dev.p, empty_dev.p, (int)empty.size(), sums,
                counts);
      AM_CUDA(cudaStreamSynchronize(st));  // far_dev / empty_dev are reused next time
    }
    AM_CUDA(cudaMemsetAsync(shift2_dev, 0, 8, st));
    AM_LAUNCH(update_centers_kernel, k, 128, 0, st, sums, counts, k, d, big, C, shift2_dev);
    double shift2 = 0.0;
    AM_CUDA(cudaMemcpyAsync(&shift2, shift2_dev, 8, cudaMemcpyDeviceToHost, st));
    AM_CUDA(cudaStreamSynchronize(st));
    if (shift2 <= tol_abs) break;
  }
  *n_iter = std::min(it, max_iter);
  return AM_OK;
}

extern "C" int am_kmeans_fit(const float* X, int64_t N, int d, int k, int n_init, int max_iter, float tol,
                             uint64_t seed, const float* init_centers, float* centers, int32_t* labels,
                             float* inertia, int* n_iter) {
  AM_CHECK(X && centers && labels, "am_kmeans_fit: NULL buffer");
  AM_CHECK(N > 0 && d > 0 && k > 0 && k <= N, "am_kmeans_fit: need 0 < k <= N (N=%lld k=%d)", (long long)N, k);
  AM_CHECK(max_iter > 0 && n_init > 0, "am_kmeans_fit: max_iter and n_init must be positive");
  cudaStream_t st;
  AM_TRY(HostCall::thread_stream(&st));
  const int64_t nblk = (N + kKppBlock - 1) / kKppBlock;
  HostCall call(st, 0, HostCall::Memory::Owned);
  float *dX, *dC, *dBestC, *sums, *counts, *dist, *mind2, *cand, *dmean;
  int32_t *dL, *dBestL;
  double *scal, *bsum, *bpot;
  call.up(&dX, X, (size_t)N * d);
  call.down(&dBestC, (size_t)k * d, centers);
  call.down(&dBestL, (size_t)N, labels);
  call.device(&dC, (size_t)k * d);
  call.device(&sums, (size_t)k * d);
  call.device(&counts, (size_t)k);
  call.device(&dist, (size_t)N);
  call.device(&dL, (size_t)N);
  call.device(&scal, 2);  // [0] inertia, [1] shift2
  call.device(&dmean, (size_t)d);
  call.device(&mind2, init_centers ? 0 : (size_t)N);  // k-means++ scratch
  call.device(&bsum, init_centers ? 0 : (size_t)nblk);
  call.device(&cand, init_centers ? 0 : (size_t)kMaxTrials * d);
  call.device(&bpot, init_centers ? 0 : (size_t)nblk * kMaxTrials);
  AM_TRY(call.start());
  double tol_abs = 0.0;
  std::vector<float> hmean;
  AM_TRY(scaled_tolerance(dX, N, d, tol, st, &tol_abs, hmean));
  // as sklearn's KMeans.fit: Lloyd runs on the rows minus their column means, whose fp32 distances then do not lose
  // ||mean||^2 to cancellation (seeding, tolerance and inertia do not change under the shift)
  AM_CUDA(cudaMemcpyAsync(dmean, hmean.data(), (size_t)d * 4, cudaMemcpyHostToDevice, st));
  const auto shift_grid = [](int64_t n) { return (int)std::max<int64_t>(1, std::min<int64_t>((n + 255) / 256, (int64_t)sm_count() * 8)); };
  AM_LAUNCH(shift_rows_kernel, shift_grid((int64_t)N * d), 256, 0, st, dX, N, d, dmean, -1);
  am_kmeans_plan step{dX, N, d, k};
  AM_TRY(step.create(kmeans_use_tensor_cores(N, d, k, KMeansUse::kFit), st));

  SplitMix rng{seed ^ kKmeansSeedMix};
  double best_inertia = INFINITY;
  int best_iters = 0;
  for (int run = 0; run < (init_centers ? 1 : n_init); ++run) {
    if (init_centers) {
      AM_CUDA(cudaMemcpyAsync(dC, init_centers, (size_t)k * d * 4, cudaMemcpyHostToDevice, st));
      AM_LAUNCH(shift_rows_kernel, shift_grid((int64_t)k * d), 256, 0, st, dC, (int64_t)k, d, dmean, -1);
    } else AM_TRY(kmeanspp_seed(dX, N, d, k, rng, dC, mind2, bsum, cand, bpot, st));
    int it = 0;
    AM_TRY(lloyd(step, max_iter, tol_abs, dC, dL, sums, counts, dist, scal + 1, st, &it));
    // final E-step: labels and inertia consistent with the returned centres
    AM_TRY(step.step(dC, dL, nullptr, nullptr, scal, nullptr, st));
    double inert = 0.0;
    AM_CUDA(cudaMemcpyAsync(&inert, scal, 8, cudaMemcpyDeviceToHost, st));
    AM_CUDA(cudaStreamSynchronize(st));
    if (inert < best_inertia) {  // keep the best restart
      best_inertia = inert;
      best_iters = it;
      AM_CUDA(cudaMemcpyAsync(dBestC, dC, (size_t)k * d * 4, cudaMemcpyDeviceToDevice, st));
      AM_CUDA(cudaMemcpyAsync(dBestL, dL, (size_t)N * 4, cudaMemcpyDeviceToDevice, st));
    }
  }
  AM_LAUNCH(shift_rows_kernel, shift_grid((int64_t)k * d), 256, 0, st, dBestC, (int64_t)k, d, dmean, 1);
  AM_TRY(call.finish());
  if (inertia) *inertia = (float)best_inertia;
  if (n_iter) *n_iter = best_iters;
  return AM_OK;
}
