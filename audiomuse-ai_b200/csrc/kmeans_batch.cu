// Batched k-means (sm_90a): many small, ragged problems fitted at once, for the clustering task's RQ batches
// (tasks/clustering.py:175-227, one KMeans(k, init='k-means++', n_init=10) per iteration).  Each (problem, init) runs
// whole on one CTA of a persistent grid, largest problems first: k-means++ seeding, Lloyd with sklearn's empty-cluster
// rule and tolerance, and the final E-step, with no host round trip in between.  Every decision follows the
// definitions of kmeans_common.cuh and exact_argmin (kmeans_tc.cuh), which am_kmeans_fit follows too.
//
//   prep_kernel    one CTA per problem: float64 column moments (one thread per column, rows in order), the scaled
//                  tolerance and column means, then the rows shifted by the means in place;
//   fit_kernel     one CTA per (problem, init), 8 warps: centres, column sums and counts in shared memory; D^2 and
//                  E-step one warp per row; column sums one thread per column over the rows in order; every
//                  float64 reduction in a fixed order.  So a result depends on nothing but its own problem and init;
//   select_kernel  one CTA per problem: the first init with the strictly lowest inertia, centres shifted back.
#include "common.cuh"
#include "host_call.cuh"
#include "kmeans_common.cuh"
#include "kmeans_tc.cuh"

#include <algorithm>
#include <cmath>
#include <vector>

namespace am {
namespace kb {

constexpr int kThreads = 256, kWarps = kThreads / 32;
constexpr int64_t kMaxRows = AM_KMEANS_BATCH_MAX_ROWS;  // the block sums live in shared memory
// shared memory: centres [k, d], sums [max(k, 8), d] (the k-means++ candidates during seeding), norms [k], counts [k]
// and the block sums f64[ceil(N / 1024)]
constexpr size_t kSmemLimit = (size_t)2 * AM_KMEANS_BATCH_MAX_KD * 4 + 8 + (size_t)(kMaxRows / kKppBlock) * 8;

struct Task {
  int64_t x0;    // first element of the problem's rows
  int64_t scr;   // first row of this (problem, init)'s labels / D^2 scratch
  int64_t cen;   // first element of its centres
  int64_t draw;  // its first k-means++ draw
  int n, d, k, trials;  // trials: kpp_trials(k)
  int problem, init, id;  // id: its place in problem order, where the results go
};

__host__ __device__ inline int cand_rows(int k) { return k > kMaxTrials ? k : kMaxTrials; }
// the floats, then the block sums at the next 8-byte boundary
__host__ __device__ inline size_t bsum_offset(int d, int k) {
  return (((size_t)(k + cand_rows(k)) * d + 2 * (size_t)k) * 4 + 7) / 8 * 8;
}
inline size_t smem_bytes(int n, int d, int k) {
  return bsum_offset(d, k) + (size_t)((n + kKppBlock - 1) / kKppBlock) * 8;
}

__global__ void __launch_bounds__(kThreads)
prep_kernel(float* __restrict__ X, const int64_t* __restrict__ x0, const int64_t* __restrict__ rows0,
            const int32_t* __restrict__ dims, const int64_t* __restrict__ mean0, float tol, float* __restrict__ mean,
            double* __restrict__ tol_abs) {
  extern __shared__ double s_mom[];  // [2, d]
  const int p = blockIdx.x, d = dims[p];
  const int64_t n = rows0[p + 1] - rows0[p];
  float* x = X + x0[p];
  for (int c = threadIdx.x; c < d; c += kThreads) {
    double a = 0.0, b = 0.0;
    for (int64_t r = 0; r < n; ++r) {
      const double v = (double)x[r * d + c];
      a += v;
      b += v * v;
    }
    s_mom[c] = a;
    s_mom[d + c] = b;
  }
  __syncthreads();
  float* mu = mean + mean0[p];
  if (threadIdx.x == 0) tol_abs[p] = kmeans_tol_abs(s_mom, s_mom + d, n, d, tol, mu);
  __syncthreads();
  for (int64_t e = threadIdx.x; e < n * d; e += kThreads) x[e] -= mu[e % d];
}

// one 1024-row block of D^2 work: warp w takes rows w, w + 8, ... (as pp_update_kernel / pp_trial_kernel do), each
// warp's float64 partials go to s_part[w][l], and thread l < nl adds sum_w s_part[w][l] to its `acc`
template <class RowFn>
__device__ __forceinline__ void kpp_block(int64_t b, int64_t n, int nl, double (*s_part)[kMaxTrials], RowFn row_fn,
                                          double& acc) {
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  double part[kMaxTrials];
#pragma unroll
  for (int l = 0; l < kMaxTrials; ++l) part[l] = 0.0;
  for (int r = warp; r < kKppBlock; r += kWarps) {
    const int64_t row = b * kKppBlock + r;
    if (row >= n) break;
    row_fn(row, lane, part);
  }
  if (lane == 0)
    for (int l = 0; l < kMaxTrials; ++l) s_part[warp][l] = part[l];
  __syncthreads();
  if ((int)threadIdx.x < nl) {
    double t = 0.0;
    for (int w = 0; w < kWarps; ++w) t += s_part[w][threadIdx.x];
    acc += t;
  }
  __syncthreads();
}

// float64 sum of one value per thread, in thread order by warp trees then warps in order; every thread gets it
__device__ __forceinline__ double block_sum(double v, double* s_red) {
  v = warp_sum(v);
  if ((threadIdx.x & 31) == 0) s_red[threadIdx.x >> 5] = v;
  __syncthreads();
  double t = 0.0;
  for (int w = 0; w < kWarps; ++w) t += s_red[w];
  __syncthreads();
  return t;
}

__global__ void __launch_bounds__(kThreads)
fit_kernel(const float* __restrict__ X, const Task* __restrict__ tasks, int n_tasks, int* __restrict__ counter,
           const double* __restrict__ draws, const double* __restrict__ tol_abs, int max_iter,
           int32_t* __restrict__ labels, float* __restrict__ dist, float* __restrict__ centres,
           double* __restrict__ inertia, int32_t* __restrict__ n_iter, int32_t* __restrict__ kpp,
           const int64_t* __restrict__ kpp0) {
  extern __shared__ __align__(16) unsigned char smem[];
  __shared__ double s_part[kWarps][kMaxTrials];
  __shared__ double s_red[kWarps], s_pot[kMaxTrials];
  __shared__ int64_t s_cand[kMaxTrials];
  __shared__ int64_t s_far;
  __shared__ float s_fard[kWarps];
  __shared__ int64_t s_farr[kWarps];
  __shared__ int s_task, s_big, s_nempty;
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;

  for (;;) {
    if (threadIdx.x == 0) s_task = atomicAdd(counter, 1);
    __syncthreads();
    const int t = s_task;
    __syncthreads();
    if (t >= n_tasks) return;
    const Task T = tasks[t];
    const int n = T.n, d = T.d, k = T.k;
    const float* x = X + T.x0;
    const int64_t nblk = (n + kKppBlock - 1) / kKppBlock;
    float* C = reinterpret_cast<float*>(smem);
    float* S = C + (size_t)k * d;
    float* cn = S + (size_t)cand_rows(k) * d;
    float* cnt = cn + k;
    double* bsum = reinterpret_cast<double*>(smem + bsum_offset(d, k));
    int32_t* lab = labels + T.scr;
    float* m2 = dist + T.scr;  // D^2 to the nearest chosen centre while seeding, the E-step's distances after
    int32_t* kp = kpp ? kpp + kpp0[T.problem] + (int64_t)T.init * k : nullptr;
    const double* u = draws + T.draw;

    // ---- greedy k-means++ (kmeanspp_seed in kmeans.cu, its host scans run here by thread l for trial l)
    const int L = T.trials;
    {
      const int64_t pick = min((int64_t)(u[0] * n), (int64_t)n - 1);
      for (int i = threadIdx.x; i < d; i += kThreads) C[i] = x[pick * d + i];
      if (kp && threadIdx.x == 0) kp[0] = (int32_t)pick;
      __syncthreads();
    }
    // m2 = min(m2, D^2 to centre c), and the block sums of m2
    auto update = [&](const float* c, bool first) {
      for (int64_t b = 0; b < nblk; ++b) {
        double s = 0.0;
        kpp_block(b, n, 1, s_part,
                  [&](int64_t row, int ln, double* part) {
                    float acc[1];
                    d2_chains<1>(x + row * d, c, 0, 1, d, ln, acc);
                    if (ln == 0) {
                      const float m = first ? acc[0] : fminf(m2[row], acc[0]);
                      m2[row] = m;
                      part[0] += (double)m;
                    }
                  },
                  s);
        if (threadIdx.x == 0) bsum[b] = s;
      }
      __syncthreads();
    };
    update(C, true);
    for (int j = 1; j < k; ++j) {
      if ((int)threadIdx.x < L) {
        double total = 0.0;
        for (int64_t b = 0; b < nblk; ++b) total += bsum[b];
        double r = u[1 + (int64_t)(j - 1) * L + threadIdx.x] * total;
        const int64_t b0 = kpp_scan(bsum, nblk, r) * kKppBlock;
        const int64_t cnt_b = min((int64_t)kKppBlock, (int64_t)n - b0);
        s_cand[threadIdx.x] = b0 + kpp_scan(m2 + b0, cnt_b, r);
      }
      __syncthreads();
      for (int e = threadIdx.x; e < L * d; e += kThreads) S[e] = x[s_cand[e / d] * d + e % d];
      __syncthreads();
      double pot = 0.0;
      for (int64_t b = 0; b < nblk; ++b)
        kpp_block(b, n, L, s_part,
                  [&](int64_t row, int ln, double* part) {
                    float acc[kMaxTrials];
                    d2_chains<kMaxTrials>(x + row * d, S, d, L, d, ln, acc);
                    const float m = m2[row];
#pragma unroll
                    for (int l = 0; l < kMaxTrials; ++l)
                      if (l < L) part[l] += (double)fminf(m, acc[l]);
                  },
                  pot);
      if ((int)threadIdx.x < L) s_pot[threadIdx.x] = pot;
      __syncthreads();
      int best = 0;
      double best_pot = INFINITY;
      for (int l = 0; l < L; ++l)
        if (s_pot[l] < best_pot) {
          best_pot = s_pot[l];
          best = l;
        }
      for (int i = threadIdx.x; i < d; i += kThreads) C[(size_t)j * d + i] = S[(size_t)best * d + i];
      if (kp && threadIdx.x == 0) kp[j] = (int32_t)s_cand[best];
      __syncthreads();
      if (j < k - 1) update(C + (size_t)j * d, false);
    }

    // ---- Lloyd (lloyd in kmeans.cu): E-step, column sums, sklearn's empty-cluster relocation, centre update; once the
    // squared shift is <= tol_abs or after max_iter steps, one more E-step gives the returned labels and inertia
    const double tol = tol_abs[T.problem];
    int it = 0;
    bool stop = false;
    for (;;) {
      for (int j = warp; j < k; j += kWarps) {
        const float v = warp_sq_norm(C + (size_t)j * d, d, lane);
        if (lane == 0) cn[j] = v;
      }
      for (int j = threadIdx.x; j < k; j += kThreads) cnt[j] = 0.f;
      __syncthreads();
      double local = 0.0;
      for (int64_t row = warp; row < n; row += kWarps) {
        const float* xr = x + row * d;
        const float xn = warp_sq_norm(xr, d, lane);
        float best = INFINITY;
        int best_j = 0;
        for (int j = 0; j < k; j += 4) exact_argmin<4, 1, false>(xr, d, C, cn, k, lane, j, best, best_j);
        if (lane == 0) {
          const float dd = fmaxf(best + xn, 0.0f);
          lab[row] = best_j;
          m2[row] = dd;
          atomicAdd(&cnt[best_j], 1.0f);  // integer counts: exact in any order
          local += (double)dd;
        }
      }
      if (stop) {
        const double tot = block_sum(local, s_red);
        if (threadIdx.x == 0) {
          inertia[T.id] = tot;
          n_iter[T.id] = it;
        }
        break;
      }
      ++it;
      for (int e = threadIdx.x; e < k * d; e += kThreads) S[e] = 0.f;
      __syncthreads();
      for (int c = threadIdx.x; c < d; c += kThreads)
        for (int64_t row = 0; row < n; ++row) S[(size_t)lab[row] * d + c] += x[row * d + c];
      // the clusters empty after the E-step, in index order (over the norms, which the next pass recomputes)
      int* empty = reinterpret_cast<int*>(cn);
      if (threadIdx.x == 0) {
        int ne = 0, big = 0;
        for (int j = 0; j < k; ++j) {
          if (cnt[j] == 0.f) empty[ne++] = j;
          if (cnt[j] > cnt[big]) big = j;
        }
        s_nempty = ne;
        s_big = big;
      }
      __syncthreads();
      int big = -1;
      const int n_empty = s_nempty;
      if (n_empty > 0) {
        float mx = 0.f;
        for (int64_t row = threadIdx.x; row < n; row += kThreads) mx = fmaxf(mx, m2[row]);
        for (int o = 16; o; o >>= 1) mx = fmaxf(mx, __shfl_xor_sync(0xffffffffu, mx, o));
        if (lane == 0) s_fard[warp] = mx;
        __syncthreads();
        float all_max = 0.f;
        for (int w = 0; w < kWarps; ++w) all_max = fmaxf(all_max, s_fard[w]);
        __syncthreads();
        if (all_max == 0.f) big = s_big;  // every row on its centre: the empty clusters take the first largest one's
        else
          for (int e = 0; e < n_empty; ++e) {  // the e-th empty cluster takes the e-th farthest row
            float bd = -1.f;
            long long br = -1;
            for (int64_t row = threadIdx.x; row < n; row += kThreads)
              if (m2[row] >= 0.f && (br < 0 || relocate_before(m2[row], row, bd, br))) {
                bd = m2[row];
                br = row;
              }
            for (int o = 16; o; o >>= 1) {
              const float od = __shfl_xor_sync(0xffffffffu, bd, o);
              const long long orow = __shfl_xor_sync(0xffffffffu, br, o);
              if (orow >= 0 && (br < 0 || relocate_before(od, orow, bd, br))) {
                bd = od;
                br = orow;
              }
            }
            if (lane == 0) {
              s_fard[warp] = bd;
              s_farr[warp] = br;
            }
            __syncthreads();
            if (threadIdx.x == 0) {
              float fd = -1.f;
              int64_t fr = -1;
              for (int w = 0; w < kWarps; ++w)
                if (s_farr[w] >= 0 && (fr < 0 || relocate_before(s_fard[w], s_farr[w], fd, fr))) {
                  fd = s_fard[w];
                  fr = s_farr[w];
                }
              s_far = fr;
            }
            __syncthreads();
            // relocate_empty_kernel: the row leaves its cluster's sums and count
            const int64_t row = s_far;
            const int donor = lab[row], target = empty[e];
            for (int i = threadIdx.x; i < d; i += kThreads) {
              const float v = x[row * d + i];
              S[(size_t)donor * d + i] -= v;
              S[(size_t)target * d + i] = v;
            }
            __syncthreads();
            if (threadIdx.x == 0) {
              cnt[target] = 1.0f;
              cnt[donor] -= 1.0f;
              m2[row] = -1.f;  // taken
            }
            __syncthreads();
          }
      }
      // update_centers_kernel: a cluster still empty takes cluster big's new centre
      double sh = 0.0;
      for (int e = threadIdx.x; e < k * d; e += kThreads) {
        const int j = e / d, i = e - j * d;
        const int src = cnt[j] > 0.f || big < 0 ? j : big;
        const float cv = cnt[src];
        const float old = C[e];
        const float nw = cv > 0.f ? S[(size_t)src * d + i] / cv : old;
        C[e] = nw;
        const double df = (double)nw - (double)old;
        sh += df * df;
      }
      stop = block_sum(sh, s_red) <= tol || it == max_iter;
    }
    for (int e = threadIdx.x; e < k * d; e += kThreads) centres[T.cen + e] = C[e];
    __syncthreads();
  }
}

// per problem: the first init with the strictly lowest inertia; its centres shifted back by the column means
__global__ void __launch_bounds__(kThreads)
select_kernel(const Task* __restrict__ tasks, const int32_t* __restrict__ first_task, int n_init,
              const int64_t* __restrict__ rows0, const int64_t* __restrict__ cen0, const int64_t* __restrict__ mean0,
              const float* __restrict__ mean, const int32_t* __restrict__ lab_scr, const float* __restrict__ cen_scr,
              const double* __restrict__ inertia_scr, const int32_t* __restrict__ it_scr, float* __restrict__ centres,
              int32_t* __restrict__ labels, float* __restrict__ inertia, int32_t* __restrict__ n_iter) {
  const int p = blockIdx.x;
  const int t0 = first_task[p];
  int best = t0;
  double best_inertia = INFINITY;
  for (int r = 0; r < n_init; ++r)
    if (inertia_scr[t0 + r] < best_inertia) {
      best_inertia = inertia_scr[t0 + r];
      best = t0 + r;
    }
  const Task& T = tasks[best];
  const float* mu = mean + mean0[p];
  for (int e = threadIdx.x; e < T.k * T.d; e += kThreads) centres[cen0[p] + e] = cen_scr[T.cen + e] + mu[e % T.d];
  for (int r = threadIdx.x; r < T.n; r += kThreads) labels[rows0[p] + r] = lab_scr[T.scr + r];
  if (threadIdx.x == 0) {
    inertia[p] = (float)best_inertia;
    n_iter[p] = it_scr[best];
  }
}

}  // namespace kb
}  // namespace am

using namespace am;

extern "C" int am_kmeans_fit_batch(const float* rows, const int64_t* row_offsets, int64_t n_rows, const int32_t* dims,
                                   const int32_t* ks, int n_problems, int n_init, int max_iter, float tol,
                                   const uint64_t* seeds, float* centers, const int64_t* center_offsets,
                                   int32_t* labels, float* inertia, int32_t* n_iter, int32_t* kpp_rows) {
  using namespace kb;
  AM_CHECK(rows && row_offsets && dims && ks && seeds && centers && center_offsets && labels && inertia && n_iter,
           "am_kmeans_fit_batch: a required pointer is NULL");
  AM_CHECK(n_problems >= 1 && n_init >= 1 && max_iter >= 1 && tol >= 0.f,
           "am_kmeans_fit_batch: need n_problems >= 1, n_init >= 1, max_iter >= 1, tol >= 0");
  AM_CHECK(row_offsets[0] == 0 && row_offsets[n_problems] == n_rows && center_offsets[0] == 0,
           "am_kmeans_fit_batch: row_offsets must run from 0 to n_rows and center_offsets start at 0");
  const int P = n_problems;
  std::vector<int64_t> x0(P + 1, 0), mean0(P + 1, 0), kpp0(P + 1, 0), draw0(P + 1, 0);
  for (int p = 0; p < P; ++p) {
    const int64_t n = row_offsets[p + 1] - row_offsets[p];
    const int d = dims[p], k = ks[p];
    AM_CHECK(d >= 1 && k >= 1 && n >= k, "am_kmeans_fit_batch: problem %d needs d >= 1 and 1 <= k <= N (N=%lld d=%d k=%d)",
             p, (long long)n, d, k);
    AM_CHECK(n <= kMaxRows, "am_kmeans_fit_batch: problem %d has %lld rows, more than AM_KMEANS_BATCH_MAX_ROWS = %lld",
             p, (long long)n, (long long)kMaxRows);
    AM_CHECK((int64_t)cand_rows(k) * (d + 1) <= AM_KMEANS_BATCH_MAX_KD,
             "am_kmeans_fit_batch: problem %d: max(k, 8) * (d + 1) = %lld exceeds AM_KMEANS_BATCH_MAX_KD = %d", p,
             (long long)cand_rows(k) * (d + 1), AM_KMEANS_BATCH_MAX_KD);
    AM_CHECK(center_offsets[p + 1] - center_offsets[p] == (int64_t)k * d,
             "am_kmeans_fit_batch: problem %d: center_offsets must step by k * d", p);
    x0[p + 1] = x0[p] + n * d;
    mean0[p + 1] = mean0[p] + d;
    kpp0[p + 1] = kpp0[p] + (int64_t)n_init * k;
    draw0[p + 1] = draw0[p] + (int64_t)n_init * kpp_draws_per_init(k);
  }
  for (int64_t e = 0; e < x0[P]; ++e)
    AM_CHECK(std::isfinite(rows[e]), "am_kmeans_fit_batch: a row holds NaN or infinity (element %lld)", (long long)e);

  // every (problem, init), its scratch, and the k-means++ draws of each problem's SplitMix stream
  std::vector<Task> tasks;
  std::vector<int32_t> first_task(P);
  std::vector<double> draws((size_t)std::max<int64_t>(1, draw0[P]));
  int64_t scr = 0, cen = 0;
  int dmax = 1;
  size_t smem = 0;
  for (int p = 0; p < P; ++p) {
    const int n = (int)(row_offsets[p + 1] - row_offsets[p]), d = dims[p], k = ks[p];
    SplitMix rng{seeds[p] ^ kKmeansSeedMix};
    for (int64_t i = draw0[p]; i < draw0[p + 1]; ++i) draws[(size_t)i] = rng.uniform();
    first_task[p] = (int)tasks.size();
    for (int r = 0; r < n_init; ++r) {
      tasks.push_back(Task{x0[p], scr, cen, draw0[p] + (int64_t)r * kpp_draws_per_init(k), n, d, k, kpp_trials(k), p, r,
                           (int)tasks.size()});
      scr += n;
      cen += (int64_t)k * d;
    }
    dmax = std::max(dmax, d);
    smem = std::max(smem, smem_bytes(n, d, k));
  }
  const int n_tasks = (int)tasks.size();
  // the largest problems first, so that the persistent grid does not end on one long fit
  std::vector<Task> order(tasks);
  std::stable_sort(order.begin(), order.end(), [](const Task& a, const Task& b) {
    return (double)a.n * a.k * a.d > (double)b.n * b.k * b.d;
  });

  cudaStream_t st;
  AM_TRY(HostCall::thread_stream(&st));
  HostCall call(st, 0, HostCall::Memory::Owned);
  float *dX, *dC, *dI, *dMean, *dDist, *dCen;
  int64_t *dRow0, *dX0, *dMean0, *dCen0, *dKpp0;
  int32_t *dDims, *dFirst, *dL, *dIt, *dKpp, *dLab, *dItS;
  double *dDraws, *dTol, *dInert;
  Task *dTasks, *dOrder;
  int* dCounter;
  call.up(&dX, rows, (size_t)x0[P]);
  call.up(&dRow0, row_offsets, (size_t)P + 1);
  call.up(&dX0, x0.data(), (size_t)P + 1);
  call.up(&dMean0, mean0.data(), (size_t)P + 1);
  call.up(&dCen0, center_offsets, (size_t)P + 1);
  call.up(&dKpp0, kpp0.data(), (size_t)P + 1);
  call.up(&dDims, dims, (size_t)P);
  call.up(&dFirst, first_task.data(), (size_t)P);
  call.up(&dDraws, draws.data(), draws.size());
  call.up(&dTasks, tasks.data(), (size_t)n_tasks);
  call.up(&dOrder, order.data(), (size_t)n_tasks);
  call.down(&dC, (size_t)center_offsets[P], centers);
  call.down(&dL, (size_t)n_rows, labels);
  call.down(&dI, (size_t)P, inertia);
  call.down(&dIt, (size_t)P, n_iter);
  call.down(&dKpp, kpp_rows ? (size_t)kpp0[P] : 0, kpp_rows);
  call.device(&dMean, (size_t)mean0[P]);
  call.device(&dTol, (size_t)P);
  call.device(&dLab, (size_t)scr);
  call.device(&dDist, (size_t)scr);
  call.device(&dCen, (size_t)cen);
  call.device(&dInert, (size_t)n_tasks);
  call.device(&dItS, (size_t)n_tasks);
  call.device(&dCounter, 1, 0);
  AM_TRY(call.start());

  AM_LAUNCH(prep_kernel, P, kThreads, (size_t)16 * dmax, st, dX, dX0, dRow0, dDims, dMean0, tol, dMean, dTol);
  AM_TRY(allow_dynamic_smem<fit_kernel>(kSmemLimit));
  int per_sm = 0;
  AM_CUDA(cudaOccupancyMaxActiveBlocksPerMultiprocessor(&per_sm, fit_kernel, kThreads, smem));
  const int grid = std::max(1, std::min(n_tasks, std::max(1, per_sm) * sm_count()));
  AM_LAUNCH(fit_kernel, grid, kThreads, smem, st, dX, dOrder, n_tasks, dCounter, dDraws, dTol, max_iter, dLab, dDist,
            dCen, dInert, dItS, kpp_rows ? dKpp : nullptr, dKpp0);
  AM_LAUNCH(select_kernel, P, kThreads, 0, st, dTasks, dFirst, n_init, dRow0, dCen0, dMean0, dMean, dLab, dCen, dInert,
            dItS, dC, dL, dI, dIt);
  return call.finish();
}
