// The artist-similarity GMM sweep (tasks/artist_gmm_manager.select_optimal_gmm_components :63-126 and fit_artist_gmm
// :129-216): for every artist and every K of its range, scikit-learn's GaussianMixture(K, covariance_type='diag',
// max_iter, n_init, random_state=42).fit and bic, then the first K with the strictly lowest BIC.  oracle/artist_gmm.py
// states the arithmetic; this file follows it step for step in float64 on float32 rows.
//
// Phase 1 (fit_kernel), one problem (artist, K, init) per CTA from start to finish, on a persistent grid that takes
// problems in decreasing order of cost (n K d) from an atomic counter; the counter only schedules, so a problem's result
// does not depend on which CTA ran it or on what else is in the batch:
//   column means and the k-means tolerance 1e-4 mean(var(X)); |x - mean|^2 per row
//   k-means++ on the centred rows: the first centre comes from the host (choice(n, p=uniform) is a function of n and
//            the draw only); each further centre: a fixed-order scan of closest_dist_sq, searchsorted of the draws,
//            the candidates' potentials, the first lowest
//   Lloyd    argmin |c|^2 - 2 x.c (ties: lowest), centre sums per column in row order, empty clusters reseeded with
//            the farthest point, strict or tolerance convergence, one more assignment when not strict
//   EM       the first M-step from the one-hot labels, then E-step / M-step until |change| < tol or max_iter; a
//            covariance <= 0 marks the problem failed; at the end score(X) of the final parameters (one more E pass),
//            so phase 2 needs no pass over the rows
// Phase 2 (select_kernel), one CTA per artist: per K the first init with the strictly greater bound, its BIC, the
// first K with the strictly lowest BIC, and the float32 gather of that fit's parameters.
//
// Every reduction has a fixed order: a warp reduces a row with the xor butterfly, per-row results are summed warp by
// warp in row order and the 8 warp partials in warp order, and column sums run over the rows in order.  No atomics
// touch the arithmetic.  The per-problem products are [n x d] x [d x K <= 16]: too narrow for wgmma, and float64 is
// what keeps the decisions equal to scikit-learn's, so this is CUDA-core code by design.
#include "common.cuh"

#include <algorithm>
#include <cmath>
#include <numeric>

namespace am {
namespace ag {

constexpr int kThreads = 256;
constexpr int kWarps = kThreads / 32;
constexpr int kMaxK = AM_ARTIST_GMM_MAX_K;
constexpr int kMaxTrials = 4;                 // 2 + floor(ln K) for K <= 16
constexpr int kSmemBytes = AM_ARTIST_GMM_SMEM_BYTES;
constexpr int kKMeansMaxIter = 300;
constexpr double kKMeansTol = 1e-4;
constexpr double kEps = 2.220446049250313e-16;
constexpr double kLog2Pi = 1.8378770664093453;
constexpr size_t kScratchBudget = size_t(1) << 30;   // device scratch per chunk of artists

__host__ __device__ inline int n_local_trials(int K) { return 2 + (K >= 3) + (K >= 8); }   // 2 + int(log(K))
__host__ __device__ inline int draws_per_init(int K) { return 1 + (K - 1) * n_local_trials(K); }

struct Problem {
  int artist;       // index within the chunk
  int K;
  int init;
  int first;        // the first k-means++ centre (row within the artist)
  int64_t row0;     // first row in the batch
  int n;
  int out;          // (artist_global * kMaxK + K - 1) * n_init + init
  int64_t dscr;     // offset of its double scratch
  int64_t iscr;     // offset of its int scratch
};

struct Result {
  double lower_bound, score;
  int n_iter, converged, failed, pad;
};

__host__ __device__ inline int64_t scratch_doubles(int n, int d, int K) {
  const int rb = std::max(K, n_local_trials(K) + 2);
  return (int64_t)d + n + (int64_t)n * rb + 4LL * K * d + 8 * kMaxK;
}

// ---------------------------------------------------------------- block reductions (fixed order)
__device__ __forceinline__ double block_sum(double v, double* red) {
  v = warp_sum(v);
  const int w = threadIdx.x >> 5;
  __syncthreads();
  if ((threadIdx.x & 31) == 0) red[w] = v;
  __syncthreads();
  double s = 0.0;
#pragma unroll
  for (int i = 0; i < kWarps; ++i) s += red[i];
  __syncthreads();
  return s;
}

struct Ctx {
  const float* X;   // the artist's rows (shared memory when staged, else global)
  int n, d, K;
  const double* mean;
};

__device__ __forceinline__ double xc(const Ctx& c, int i, int col) {
  return (double)c.X[(int64_t)i * c.d + col] - c.mean[col];
}

// one warp per row; v[j] = sum_col xc(i, col) * Y_j[col] for the rows of the nc centred data rows ids[] (k-means++)
// or for K double vectors (Lloyd)
template <int M>
__device__ __forceinline__ void row_dots_rows(const Ctx& c, int i, const int* ids, int m, double* v) {
  const int lane = threadIdx.x & 31;
  double acc[M];
#pragma unroll
  for (int j = 0; j < M; ++j) acc[j] = 0.0;
  for (int col = lane; col < c.d; col += 32) {
    const double x = xc(c, i, col);
#pragma unroll
    for (int j = 0; j < M; ++j)
      if (j < m) acc[j] = fma(x, xc(c, ids[j], col), acc[j]);
  }
#pragma unroll
  for (int j = 0; j < M; ++j) v[j] = warp_sum(acc[j]);
}

// ---------------------------------------------------------------- phase 1
struct Shared {
  double red[kWarps];
  double pot[kMaxTrials];
  double kv[kMaxK];
  double scan[kThreads];
  int cand[kMaxTrials];
  int idx[kMaxK];
  int cnt[kMaxK];
  int flag;
  int prob;
  double tol;
};

__global__ void __launch_bounds__(kThreads, 2)
fit_kernel(const float* __restrict__ Xall, int d, const Problem* __restrict__ probs, int n_probs, int* __restrict__ counter,
           const double* __restrict__ draws, int n_init, int max_iter, double em_tol, double reg_covar,
           double* __restrict__ dscr, int* __restrict__ iscr, Result* __restrict__ res, int32_t* __restrict__ kpp_out,
           int32_t* __restrict__ labels_out, int64_t labels_stride) {
  extern __shared__ __align__(16) unsigned char smem[];
  __shared__ Shared sh;
  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  for (;;) {
    if (tid == 0) sh.prob = atomicAdd(counter, 1);
    __syncthreads();
    const int pi = sh.prob;
    __syncthreads();
    if (pi >= n_probs) return;
    const Problem P = probs[pi];
    const int n = P.n, K = P.K, L = n_local_trials(K);
    const int rb = max(K, L + 2);
    double* mean = dscr + P.dscr;
    double* xsq = mean + d;
    double* rowbuf = xsq + n;
    double* kd = rowbuf + (int64_t)n * rb;
    double* Ca = kd;                          // Lloyd: centres; EM: means
    double* Cb = kd + (int64_t)K * d;         // Lloyd: new centres; EM: covariances
    double* mp = kd + 2LL * K * d;            // EM: means * precisions
    double* pr = kd + 3LL * K * d;            // EM: precisions
    double* kvec = kd + 4LL * K * d;          // 8 x kMaxK: nk, A, logdet, logw, weights
    double* nk = kvec;
    double* Ak = kvec + kMaxK;
    double* ldet = kvec + 2 * kMaxK;
    double* logw = kvec + 3 * kMaxK;
    double* wts = kvec + 4 * kMaxK;
    int* labels = iscr + P.iscr;
    int* labels_old = labels + n;

    // rows: staged in shared memory when they fit, else read through L2; responsibilities likewise
    const float* Xg = Xall + P.row0 * d;
    const size_t row_bytes = (size_t)n * d * sizeof(float);
    const float* X = Xg;
    size_t used = 0;
    if (row_bytes <= (size_t)kSmemBytes) {
      float* xs = reinterpret_cast<float*>(smem);
      for (int64_t e = tid; e < (int64_t)n * d; e += kThreads) xs[e] = Xg[e];
      X = xs;
      used = (row_bytes + 15) / 16 * 16;
    }
    double* resp = rowbuf;
    if (used + (size_t)n * K * sizeof(double) <= (size_t)kSmemBytes) resp = reinterpret_cast<double*>(smem + used);
    __syncthreads();
    Ctx c{X, n, d, K, mean};

    // ---- column means, tolerance, squared norms of the centred rows
    double vpart = 0.0;
    for (int col = tid; col < d; col += kThreads) {
      double s = 0.0;
      for (int i = 0; i < n; ++i) s += (double)X[(int64_t)i * d + col];
      const double m = s / n;
      double v = 0.0;
      for (int i = 0; i < n; ++i) {
        const double t = (double)X[(int64_t)i * d + col] - m;
        v = fma(t, t, v);
      }
      mean[col] = m;
      vpart += v / n;
    }
    const double km_tol = block_sum(vpart, sh.red) / d * kKMeansTol;
    for (int i = warp; i < n; i += kWarps) {
      double s = 0.0;
      for (int col = lane; col < d; col += 32) {
        const double t = xc(c, i, col);
        s = fma(t, t, s);
      }
      s = warp_sum(s);
      if (lane == 0) xsq[i] = s;
    }
    __syncthreads();

    // ---- k-means++
    const double* u = draws + (int64_t)P.init * draws_per_init(K);
    double* closest = rowbuf;
    double* cs = rowbuf + n;
    double* cd = rowbuf + 2LL * n;            // L candidate distance rows
    if (tid == 0) sh.idx[0] = P.first;
    __syncthreads();
    {
      double part = 0.0;
      const int c0 = sh.idx[0];
      for (int i = warp; i < n; i += kWarps) {
        double v;
        row_dots_rows<1>(c, i, &c0, 1, &v);
        const double dist = fmax((-2.0 * v + xsq[c0]) + xsq[i], 0.0);
        if (lane == 0) closest[i] = dist;
        part += dist;
      }
      if (lane != 0) part = 0.0;
      double pot = block_sum(part, sh.red);
      int pos = 1;
      for (int cc = 1; cc < K; ++cc) {
        // cumsum of closest in row order: contiguous chunks per thread, the chunk totals scanned by one thread
        const int chunk = (n + kThreads - 1) / kThreads;
        const int b0 = min(n, tid * chunk), b1 = min(n, b0 + chunk);
        double s = 0.0;
        for (int i = b0; i < b1; ++i) s += closest[i];
        double* tot = sh.scan;
        __syncthreads();
        tot[tid] = s;
        __syncthreads();
        if (tid == 0) {
          double run = 0.0;
          for (int t = 0; t < kThreads; ++t) {
            const double v = tot[t];
            tot[t] = run;
            run += v;
          }
        }
        __syncthreads();
        s = tot[tid];
        for (int i = b0; i < b1; ++i) {
          s += closest[i];
          cs[i] = s;
        }
        __syncthreads();
        if (tid < L) {
          const double rv = u[pos + tid] * pot;
          int lo = 0, hi = n;                      // first i with cs[i] >= rv (searchsorted, side='left')
          while (lo < hi) {
            const int mid = (lo + hi) >> 1;
            if (cs[mid] < rv) lo = mid + 1; else hi = mid;
          }
          sh.cand[tid] = min(lo, n - 1);
        }
        __syncthreads();
        pos += L;
        double pp[kMaxTrials] = {0.0, 0.0, 0.0, 0.0};
        for (int i = warp; i < n; i += kWarps) {
          double v[kMaxTrials];
          row_dots_rows<kMaxTrials>(c, i, sh.cand, L, v);
#pragma unroll
          for (int j = 0; j < kMaxTrials; ++j) {
            if (j < L) {
              const double dist = fmin(closest[i], fmax((-2.0 * v[j] + xsq[sh.cand[j]]) + xsq[i], 0.0));
              if (lane == 0) cd[(int64_t)j * n + i] = dist;
              pp[j] += dist;
            }
          }
        }
        for (int j = 0; j < L; ++j) {
          const double t = block_sum(lane == 0 ? pp[j] : 0.0, sh.red);
          if (tid == 0) sh.pot[j] = t;
        }
        __syncthreads();
        int best = 0;
        for (int j = 1; j < L; ++j)
          if (sh.pot[j] < sh.pot[best]) best = j;
        pot = sh.pot[best];
        for (int i = tid; i < n; i += kThreads) closest[i] = cd[(int64_t)best * n + i];
        if (tid == 0) sh.idx[cc] = sh.cand[best];
        __syncthreads();
      }
    }
    if (kpp_out && tid < K) kpp_out[(int64_t)P.out * kMaxK + tid] = sh.idx[tid];

    // ---- Lloyd
    for (int e = tid; e < K * d; e += kThreads) Ca[e] = xc(c, sh.idx[e / d], e % d);
    for (int i = tid; i < n; i += kThreads) labels_old[i] = -1;
    __syncthreads();
    double* C = Ca;
    double* Cn = Cb;
    bool strict = false;
    auto assign = [&](const double* Cc) {
      for (int k = warp; k < K; k += kWarps) {
        double s = 0.0;
        for (int col = lane; col < d; col += 32) s = fma(Cc[(int64_t)k * d + col], Cc[(int64_t)k * d + col], s);
        s = warp_sum(s);
        if (lane == 0) sh.kv[k] = s;
      }
      __syncthreads();
      for (int i = warp; i < n; i += kWarps) {
        double acc[kMaxK];
#pragma unroll
        for (int k = 0; k < kMaxK; ++k) acc[k] = 0.0;
        for (int col = lane; col < d; col += 32) {
          const double x = xc(c, i, col);
#pragma unroll
          for (int k = 0; k < kMaxK; ++k)
            if (k < K) acc[k] = fma(x, Cc[(int64_t)k * d + col], acc[k]);
        }
        int lab = 0;
        double best = 0.0;
#pragma unroll
        for (int k = 0; k < kMaxK; ++k) {
          if (k < K) {
            const double v = sh.kv[k] - 2.0 * warp_sum(acc[k]);
            if (k == 0 || v < best) {
              best = v;
              lab = k;
            }
          }
        }
        if (lane == 0) labels[i] = lab;
      }
      __syncthreads();
    };
    for (int it = 0; it < kKMeansMaxIter; ++it) {
      assign(C);
      // centre sums, one thread per column over the rows in order
      for (int col = tid; col < d; col += kThreads) {
        double acc[kMaxK];
#pragma unroll
        for (int k = 0; k < kMaxK; ++k) acc[k] = 0.0;
        for (int i = 0; i < n; ++i) {
          const int lab = labels[i];
          const double x = xc(c, i, col);
#pragma unroll
          for (int k = 0; k < kMaxK; ++k)
            if (k == lab) acc[k] += x;
        }
        for (int k = 0; k < K; ++k) Cn[(int64_t)k * d + col] = acc[k];
      }
      if (tid < K) {
        int m = 0;
        for (int i = 0; i < n; ++i) m += labels[i] == tid;
        sh.cnt[tid] = m;
      }
      int changed = 0;
      for (int i = tid; i < n; i += kThreads) changed |= labels[i] != labels_old[i];
      changed = __syncthreads_or(changed);
      unsigned empty = 0;         // the clusters empty after this assignment; a reseed may empty another, which stays
      for (int k = 0; k < K; ++k) empty |= (sh.cnt[k] == 0 ? 1u : 0u) << k;
      if (empty) {
        // reseed each empty cluster with the farthest remaining point from its centre (ties: the lowest row)
        double* far = rowbuf;
        for (int i = warp; i < n; i += kWarps) {
          double s = 0.0;
          const int lab = labels[i];
          for (int col = lane; col < d; col += 32) {
            const double t = xc(c, i, col) - C[(int64_t)lab * d + col];
            s = fma(t, t, s);
          }
          s = warp_sum(s);
          if (lane == 0) far[i] = s;
        }
        __syncthreads();
        for (int k = 0; k < K; ++k) {
          if (!(empty >> k & 1u)) continue;
          if (tid == 0) {
            int f = 0;
            for (int i = 1; i < n; ++i)
              if (far[i] > far[f]) f = i;
            sh.flag = f;
          }
          __syncthreads();
          const int f = sh.flag;
          const int old = labels[f];
          for (int col = tid; col < d; col += kThreads) {
            const double x = xc(c, f, col);
            Cn[(int64_t)old * d + col] -= x;
            Cn[(int64_t)k * d + col] = x;
          }
          __syncthreads();
          if (tid == 0) {
            sh.cnt[k] = 1;
            sh.cnt[old] -= 1;
            far[f] = -1.0;
          }
          __syncthreads();
        }
      }
      for (int e = tid; e < K * d; e += kThreads) {
        const int w = sh.cnt[e / d];
        if (w > 0) Cn[e] *= 1.0 / (double)w;
      }
      __syncthreads();
      for (int k = warp; k < K; k += kWarps) {
        double s = 0.0;
        for (int col = lane; col < d; col += 32) {
          const double t = Cn[(int64_t)k * d + col] - C[(int64_t)k * d + col];
          s = fma(t, t, s);
        }
        s = warp_sum(s);
        if (lane == 0) sh.kv[k] = sqrt(s);
      }
      __syncthreads();
      double* t = C;
      C = Cn;
      Cn = t;
      if (!changed) {
        strict = true;
        break;
      }
      double shift = 0.0;
      for (int k = 0; k < K; ++k) shift += sh.kv[k] * sh.kv[k];
      __syncthreads();
      if (shift <= km_tol) break;
      for (int i = tid; i < n; i += kThreads) labels_old[i] = labels[i];
      __syncthreads();
    }
    if (!strict) assign(C);
    if (labels_out)
      for (int i = tid; i < n; i += kThreads)
        labels_out[(int64_t)((K - 1) * n_init + P.init) * labels_stride + P.row0 + i] = labels[i];

    // ---- EM: the first M-step from the one-hot labels
    double* means = Ca;
    double* cov = Cb;
    int failed = 0;
    if (tid < K) {
      int m = 0;
      for (int i = 0; i < n; ++i) m += labels[i] == tid;
      nk[tid] = (double)m + 10.0 * kEps;
    }
    __syncthreads();
    for (int col = tid; col < d; col += kThreads) {
      double a1[kMaxK], a2[kMaxK];
#pragma unroll
      for (int k = 0; k < kMaxK; ++k) a1[k] = a2[k] = 0.0;
      for (int i = 0; i < n; ++i) {
        const int lab = labels[i];
        const double x = (double)X[(int64_t)i * d + col];
        const double x2 = x * x;
#pragma unroll
        for (int k = 0; k < kMaxK; ++k)
          if (k == lab) {
            a1[k] += x;
            a2[k] += x2;
          }
      }
      for (int k = 0; k < K; ++k) {
        const double m = a1[k] / nk[k];
        const double v = a2[k] / nk[k] - m * m + reg_covar;
        means[(int64_t)k * d + col] = m;
        cov[(int64_t)k * d + col] = v;
        failed |= !(v > 0.0) && !(v != v);
      }
    }
    if (tid < K) wts[tid] = nk[tid] / n;
    failed = __syncthreads_or(failed);

    // precisions, their log-determinants and the per-component constants of the E-step
    auto prepare = [&]() {
      for (int e = tid; e < K * d; e += kThreads) {
        const double pc = 1.0 / sqrt(cov[e]);
        const double p = pc * pc;
        pr[e] = p;
        mp[e] = means[e] * p;
      }
      __syncthreads();
      for (int k = warp; k < K; k += kWarps) {
        double a = 0.0, l = 0.0;
        for (int col = lane; col < d; col += 32) {
          const int64_t e = (int64_t)k * d + col;
          a += means[e] * means[e] * pr[e];
          l += log(1.0 / sqrt(cov[e]));
        }
        a = warp_sum(a);
        l = warp_sum(l);
        if (lane == 0) {
          Ak[k] = a;
          ldet[k] = l;
          logw[k] = log(wts[k]);
        }
      }
      __syncthreads();
    };
    // E pass: mean log-normaliser; writes the responsibilities when w_resp
    auto estep = [&](bool w_resp) -> double {
      double part = 0.0;
      for (int i = warp; i < n; i += kWarps) {
        double a1[kMaxK], a2[kMaxK];
#pragma unroll
        for (int k = 0; k < kMaxK; ++k) a1[k] = a2[k] = 0.0;
        for (int col = lane; col < d; col += 32) {
          const double x = (double)X[(int64_t)i * d + col];
          const double x2 = x * x;
#pragma unroll
          for (int k = 0; k < kMaxK; ++k)
            if (k < K) {
              a1[k] = fma(x, mp[(int64_t)k * d + col], a1[k]);
              a2[k] = fma(x2, pr[(int64_t)k * d + col], a2[k]);
            }
        }
        double wl[kMaxK];
        double mx = -INFINITY;
#pragma unroll
        for (int k = 0; k < kMaxK; ++k)
          if (k < K) {
            const double lp = (Ak[k] - 2.0 * warp_sum(a1[k])) + warp_sum(a2[k]);
            wl[k] = (-0.5 * (d * kLog2Pi + lp) + ldet[k]) + logw[k];
            mx = fmax(mx, wl[k]);
          }
        // scikit-learn's logsumexp: the maxima split off, the rest through log1p
        double m = 0.0, s = 0.0;
        const double shift = isfinite(mx) ? mx : 0.0;
#pragma unroll
        for (int k = 0; k < kMaxK; ++k)
          if (k < K) {
            if (wl[k] == mx) m += 1.0;
            else s += exp(wl[k] - shift);
          }
        if (s != 0.0) s = s / m;
        const double norm = (log1p(s) + log(m)) + mx;
        if (w_resp && lane < K) {
#pragma unroll
          for (int k = 0; k < kMaxK; ++k)
            if (k == lane) resp[(int64_t)i * K + k] = exp(wl[k] - norm);
        }
        part += norm;
      }
      if (lane != 0) part = 0.0;
      return block_sum(part, sh.red) / n;
    };
    auto mstep = [&]() -> int {
      if (tid < K) {
        double s = 0.0;
        for (int i = 0; i < n; ++i) s += resp[(int64_t)i * K + tid];
        nk[tid] = s + 10.0 * kEps;
      }
      __syncthreads();
      int bad = 0;
      for (int col = tid; col < d; col += kThreads) {
        double a1[kMaxK], a2[kMaxK];
#pragma unroll
        for (int k = 0; k < kMaxK; ++k) a1[k] = a2[k] = 0.0;
        for (int i = 0; i < n; ++i) {
          const double x = (double)X[(int64_t)i * d + col];
          const double x2 = x * x;
          const double* r = resp + (int64_t)i * K;
#pragma unroll
          for (int k = 0; k < kMaxK; ++k)
            if (k < K) {
              a1[k] = fma(r[k], x, a1[k]);
              a2[k] = fma(r[k], x2, a2[k]);
            }
        }
        for (int k = 0; k < K; ++k) {
          const double m = a1[k] / nk[k];
          const double v = a2[k] / nk[k] - m * m + reg_covar;
          means[(int64_t)k * d + col] = m;
          cov[(int64_t)k * d + col] = v;
          bad |= !(v > 0.0) && !(v != v);
        }
      }
      if (tid == 0) {
        double s = 0.0;
        for (int k = 0; k < K; ++k) s += nk[k];
        for (int k = 0; k < K; ++k) wts[k] = nk[k] / s;
      }
      return __syncthreads_or(bad);
    };

    double lb = -INFINITY;
    int n_iter = 0, converged = 0;
    if (!failed) {
      prepare();
      for (n_iter = 1; n_iter <= max_iter; ++n_iter) {
        const double prev = lb;
        lb = estep(true);
        __syncthreads();
        if (mstep()) {
          failed = 1;
          break;
        }
        prepare();
        if (fabs(lb - prev) < em_tol) {
          converged = 1;
          break;
        }
      }
      if (n_iter > max_iter) n_iter = max_iter;
    }
    double score = NAN;
    if (!failed) score = estep(false);
    if (tid == 0) res[P.out] = Result{lb, score, n_iter, converged, failed, 0};
    __syncthreads();
  }
}

// ---------------------------------------------------------------- phase 2
__global__ void __launch_bounds__(kThreads)
select_kernel(const Problem* __restrict__ first_prob, const int* __restrict__ art_first, int a0, const int64_t* offsets,
              const int* __restrict__ k_lo, const int* __restrict__ k_hi, int d, int n_init, const Result* __restrict__ res,
              const double* __restrict__ dscr, int32_t* __restrict__ chosen, double* __restrict__ bic,
              uint8_t* __restrict__ failed, double* __restrict__ lb_out, int32_t* __restrict__ it_out,
              uint8_t* __restrict__ conv_out, float* __restrict__ w_out, float* __restrict__ m_out,
              float* __restrict__ c_out) {
  __shared__ int s_best_k, s_best_prob;
  const int a = a0 + blockIdx.x;
  const int n = (int)(offsets[a + 1] - offsets[a]);
  if (threadIdx.x == 0) {
    double best_bic = INFINITY;
    int best_k = 0, best_p = -1;
    for (int K = 1; K <= kMaxK; ++K) {
      const int o = (a * kMaxK + K - 1);
      if (K < k_lo[a] || K > k_hi[a]) {
        bic[o] = NAN;
        failed[o] = 0;
        continue;
      }
      bool f = K > n;
      int bi = 0;
      double bl = -INFINITY;
      for (int i = 0; i < n_init && !f; ++i) {
        const Result r = res[o * n_init + i];
        f = r.failed != 0;
        lb_out[o * n_init + i] = r.lower_bound;
        it_out[o * n_init + i] = r.n_iter;
        conv_out[o * n_init + i] = (uint8_t)r.converged;
        if (r.lower_bound > bl || bl == -INFINITY) {
          bl = r.lower_bound;
          bi = i;
        }
      }
      failed[o] = f;
      if (f) {
        bic[o] = NAN;
        continue;
      }
      const double sc = res[o * n_init + bi].score;
      const double b = -2.0 * sc * n + (double)(2 * K * d + K - 1) * log((double)n);
      bic[o] = b;
      if (b < best_bic) {
        best_bic = b;
        best_k = K;
        best_p = art_first[a] + (K - k_lo[a]) * n_init + bi;
      }
    }
    chosen[a] = best_k;
    s_best_k = best_k;
    s_best_prob = best_p;
  }
  __syncthreads();
  if (s_best_prob < 0) return;
  const int K = s_best_k;
  const Problem& P = first_prob[s_best_prob];
  const double* kd = dscr + P.dscr + d + P.n + (int64_t)P.n * max(K, n_local_trials(K) + 2);
  for (int e = threadIdx.x; e < K * d; e += kThreads) {
    m_out[(int64_t)a * kMaxK * d + e] = (float)kd[e];
    c_out[(int64_t)a * kMaxK * d + e] = (float)kd[(int64_t)K * d + e];
  }
  if ((int)threadIdx.x < K) w_out[a * kMaxK + threadIdx.x] = (float)kd[4LL * K * d + 4 * kMaxK + threadIdx.x];
}

}  // namespace ag
}  // namespace am

using namespace am;

extern "C" int am_artist_gmm_fit(const float* rows, int64_t n_rows, int d, const int64_t* offsets, int n_artists,
                                 const int32_t* k_lo, const int32_t* k_hi, int n_init, int max_iter, double tol,
                                 double reg_covar, const double* draws, int64_t n_draws, int32_t* chosen_k,
                                 double* bic, uint8_t* failed, double* lower_bound, int32_t* n_iter,
                                 uint8_t* converged, float* weights, float* means, float* covariances, int32_t* kpp,
                                 int32_t* labels, float* phase_ms) {
  using namespace ag;
  AM_CHECK(rows && offsets && k_lo && k_hi && draws && chosen_k && bic && failed && lower_bound && n_iter &&
               converged && weights && means && covariances,
           "am_artist_gmm_fit: a required pointer is null");
  AM_CHECK(n_artists >= 1 && n_rows >= 1 && d >= 1 && d <= AM_ARTIST_GMM_MAX_D,
           "am_artist_gmm_fit: need n_artists >= 1, n_rows >= 1, 1 <= d <= %d (got %d, %lld, %d)",
           AM_ARTIST_GMM_MAX_D, n_artists, (long long)n_rows, d);
  AM_CHECK(n_init >= 1 && n_init <= 8 && max_iter >= 1 && tol >= 0.0 && reg_covar >= 0.0,
           "am_artist_gmm_fit: need 1 <= n_init <= 8, max_iter >= 1, tol >= 0, reg_covar >= 0");
  AM_CHECK(offsets[0] == 0 && offsets[n_artists] == n_rows, "am_artist_gmm_fit: offsets must run from 0 to n_rows");
  int kmax = 0;
  for (int a = 0; a < n_artists; ++a) {
    const int64_t n = offsets[a + 1] - offsets[a];
    AM_CHECK(n >= 1 && n <= INT32_MAX, "am_artist_gmm_fit: artist %d has %lld rows", a, (long long)n);
    AM_CHECK(k_lo[a] >= 1 && k_hi[a] <= kMaxK, "am_artist_gmm_fit: artist %d: K range [%d, %d] outside [1, %d]", a,
             k_lo[a], k_hi[a], kMaxK);
    kmax = std::max(kmax, (int)k_hi[a]);
  }
  AM_CHECK(kmax == 0 || n_draws >= (int64_t)n_init * draws_per_init(kmax),
           "am_artist_gmm_fit: %lld draws, K = %d with n_init = %d needs %d", (long long)n_draws, kmax, n_init,
           n_init * draws_per_init(kmax));
  for (int64_t e = 0; e < n_rows * d; ++e)
    AM_CHECK(std::isfinite(rows[e]), "am_artist_gmm_fit: row %lld has a NaN or infinity", (long long)(e / d));
  AM_TRY(ensure_init());

  // every problem (artist, K, init) with K <= n; the first k-means++ centre is choice(n, p=uniform) on the host
  const int A = n_artists;
  std::vector<Problem> all;
  std::vector<int> art_first(A, 0);
  for (int a = 0; a < A; ++a) {
    const int n = (int)(offsets[a + 1] - offsets[a]);
    art_first[a] = (int)all.size();
    std::vector<double> cdf;
    for (int K = k_lo[a]; K <= k_hi[a]; ++K)
      for (int i = 0; i < n_init; ++i) {
        Problem p{};
        p.K = K;
        p.init = i;
        p.n = n;
        p.row0 = offsets[a];
        p.out = (a * kMaxK + K - 1) * n_init + i;
        p.artist = a;
        p.first = -1;
        if (K <= n) {
          if (cdf.empty()) {
            cdf.resize(n);
            double s = 0.0;
            const double pw = 1.0 / n;
            for (int r = 0; r < n; ++r) cdf[r] = (s += pw);
            const double last = cdf[n - 1];
            for (int r = 0; r < n; ++r) cdf[r] /= last;
          }
          const double u = draws[(int64_t)i * draws_per_init(K)];
          p.first = (int)(std::upper_bound(cdf.begin(), cdf.end(), u) - cdf.begin());
        }
        all.push_back(p);
      }
  }

  Stream st;
  AM_TRY(st.create());
  cudaStream_t s = st.s;
  cudaEvent_t ev[4] = {};
  for (auto& e : ev) AM_CUDA(cudaEventCreate(&e));
  struct EvGuard {
    cudaEvent_t* e;
    ~EvGuard() {
      for (int i = 0; i < 4; ++i)
        if (e[i]) cudaEventDestroy(e[i]);
    }
  } evg{ev};
  const int P_all = (int)all.size();
  DevBuf<float> dX, dW, dM, dC;
  DevBuf<int64_t> dOff;
  DevBuf<int> dLo, dHi, dFirst, dCounter;
  DevBuf<double> dDraws, dBic, dLb;
  DevBuf<int32_t> dChosen, dIt, dKpp, dLab;
  DevBuf<uint8_t> dFailed, dConv;
  DevBuf<Result> dRes;
  DevBuf<Problem> dProbs;
  AM_TRY(dX.alloc((size_t)n_rows * d));
  AM_TRY(dOff.alloc(A + 1));
  AM_TRY(dLo.alloc(A));
  AM_TRY(dHi.alloc(A));
  AM_TRY(dFirst.alloc(A));
  AM_TRY(dCounter.alloc(1));
  AM_TRY(dDraws.alloc(std::max<int64_t>(1, n_draws)));
  AM_TRY(dBic.alloc((size_t)A * kMaxK));
  AM_TRY(dFailed.alloc((size_t)A * kMaxK));
  AM_TRY(dLb.alloc((size_t)A * kMaxK * n_init));
  AM_TRY(dIt.alloc((size_t)A * kMaxK * n_init));
  AM_TRY(dConv.alloc((size_t)A * kMaxK * n_init));
  AM_TRY(dRes.alloc((size_t)A * kMaxK * n_init));
  AM_TRY(dChosen.alloc(A));
  AM_TRY(dW.alloc((size_t)A * kMaxK));
  AM_TRY(dM.alloc((size_t)A * kMaxK * d));
  AM_TRY(dC.alloc((size_t)A * kMaxK * d));
  AM_TRY(dProbs.alloc(std::max(1, P_all)));
  if (kpp) AM_TRY(dKpp.alloc((size_t)A * kMaxK * n_init * kMaxK));
  if (labels) AM_TRY(dLab.alloc((size_t)kMaxK * n_init * n_rows));
  AM_CUDA(cudaMemcpyAsync(dX.p, rows, (size_t)n_rows * d * 4, cudaMemcpyHostToDevice, s));
  AM_CUDA(cudaMemcpyAsync(dOff.p, offsets, (A + 1) * 8, cudaMemcpyHostToDevice, s));
  AM_CUDA(cudaMemcpyAsync(dLo.p, k_lo, A * 4, cudaMemcpyHostToDevice, s));
  AM_CUDA(cudaMemcpyAsync(dHi.p, k_hi, A * 4, cudaMemcpyHostToDevice, s));
  AM_CUDA(cudaMemcpyAsync(dFirst.p, art_first.data(), A * 4, cudaMemcpyHostToDevice, s));
  AM_CUDA(cudaMemcpyAsync(dDraws.p, draws, n_draws * 8, cudaMemcpyHostToDevice, s));
  AM_CUDA(cudaMemsetAsync(dW.p, 0, dW.n * 4, s));
  AM_CUDA(cudaMemsetAsync(dM.p, 0, dM.n * 4, s));
  AM_CUDA(cudaMemsetAsync(dC.p, 0, dC.n * 4, s));
  AM_CUDA(cudaMemsetAsync(dLb.p, 0xff, dLb.n * 8, s));       // NaN: an init that never ran
  AM_CUDA(cudaMemsetAsync(dIt.p, 0, dIt.n * 4, s));
  AM_CUDA(cudaMemsetAsync(dConv.p, 0, dConv.n, s));
  if (kpp) AM_CUDA(cudaMemsetAsync(dKpp.p, 0xff, dKpp.n * 4, s));
  if (labels) AM_CUDA(cudaMemsetAsync(dLab.p, 0xff, dLab.n * 4, s));
  {
    // problems with K > n never run: they report failed
    std::vector<Result> init_res((size_t)A * kMaxK * n_init, Result{NAN, NAN, 0, 0, 1, 0});
    AM_CUDA(cudaMemcpyAsync(dRes.p, init_res.data(), init_res.size() * sizeof(Result), cudaMemcpyHostToDevice, s));
    AM_CUDA(cudaStreamSynchronize(s));
  }
  AM_CUDA(cudaMemcpyAsync(dProbs.p, all.data(), P_all * sizeof(Problem), cudaMemcpyHostToDevice, s));
  AM_TRY(allow_dynamic_smem<fit_kernel>(kSmemBytes));

  // chunks of whole artists whose scratch fits the budget
  float fit_ms = 0.f, sel_ms = 0.f;
  DevBuf<double> dscr;
  DevBuf<int> iscr;
  int a0 = 0;
  while (a0 < A) {
    int a1 = a0;
    int64_t dsz = 0, isz = 0;
    std::vector<Problem> runs;
    while (a1 < A) {
      int64_t add_d = 0, add_i = 0;
      for (int p = art_first[a1]; p < (a1 + 1 < A ? art_first[a1 + 1] : P_all); ++p)
        if (all[p].K <= all[p].n) {
          add_d += scratch_doubles(all[p].n, d, all[p].K);
          add_i += 2LL * all[p].n;
        }
      if (a1 > a0 && (size_t)(dsz + add_d) * 8 + (size_t)(isz + add_i) * 4 > kScratchBudget) break;
      for (int p = art_first[a1]; p < (a1 + 1 < A ? art_first[a1 + 1] : P_all); ++p)
        if (all[p].K <= all[p].n) {
          all[p].dscr = dsz;
          all[p].iscr = isz;
          dsz += scratch_doubles(all[p].n, d, all[p].K);
          isz += 2LL * all[p].n;
          runs.push_back(all[p]);
        }
      ++a1;
    }
    // the gather in phase 2 reads each problem's scratch offsets
    const int pb = art_first[a0], pe = a1 < A ? art_first[a1] : P_all;
    if (pe > pb)
      AM_CUDA(cudaMemcpyAsync(dProbs.p + pb, all.data() + pb, (pe - pb) * sizeof(Problem), cudaMemcpyHostToDevice, s));
    std::stable_sort(runs.begin(), runs.end(), [](const Problem& x, const Problem& y) {
      return (int64_t)x.n * x.K > (int64_t)y.n * y.K;
    });
    DevBuf<Problem> dRuns;
    AM_TRY(dRuns.alloc(std::max<size_t>(1, runs.size())));
    if (!runs.empty())
      AM_CUDA(cudaMemcpyAsync(dRuns.p, runs.data(), runs.size() * sizeof(Problem), cudaMemcpyHostToDevice, s));
    AM_TRY(dscr.ensure((size_t)std::max<int64_t>(1, dsz)));
    AM_TRY(iscr.ensure((size_t)std::max<int64_t>(1, isz)));
    AM_CUDA(cudaMemsetAsync(dCounter.p, 0, 4, s));
    AM_CUDA(cudaEventRecord(ev[0], s));
    if (!runs.empty()) {
      const int grid = std::min<int>((int)runs.size(), 2 * sm_count());
      AM_LAUNCH(fit_kernel, grid, kThreads, kSmemBytes, s, dX.p, d, dRuns.p, (int)runs.size(), dCounter.p, dDraws.p,
                n_init, max_iter, tol, reg_covar, dscr.p, iscr.p, dRes.p, kpp ? dKpp.p : nullptr,
                labels ? dLab.p : nullptr, n_rows);
    }
    AM_CUDA(cudaEventRecord(ev[1], s));
    AM_LAUNCH(select_kernel, a1 - a0, kThreads, 0, s, dProbs.p, dFirst.p, a0, dOff.p, dLo.p, dHi.p, d, n_init, dRes.p,
              dscr.p, dChosen.p, dBic.p, dFailed.p, dLb.p, dIt.p, dConv.p, dW.p, dM.p, dC.p);
    AM_CUDA(cudaEventRecord(ev[2], s));
    AM_CUDA(cudaStreamSynchronize(s));
    float ms = 0.f;
    AM_CUDA(cudaEventElapsedTime(&ms, ev[0], ev[1]));
    fit_ms += ms;
    AM_CUDA(cudaEventElapsedTime(&ms, ev[1], ev[2]));
    sel_ms += ms;
    a0 = a1;
  }
  AM_CUDA(cudaMemcpyAsync(chosen_k, dChosen.p, A * 4, cudaMemcpyDeviceToHost, s));
  AM_CUDA(cudaMemcpyAsync(bic, dBic.p, dBic.n * 8, cudaMemcpyDeviceToHost, s));
  AM_CUDA(cudaMemcpyAsync(failed, dFailed.p, dFailed.n, cudaMemcpyDeviceToHost, s));
  AM_CUDA(cudaMemcpyAsync(lower_bound, dLb.p, dLb.n * 8, cudaMemcpyDeviceToHost, s));
  AM_CUDA(cudaMemcpyAsync(n_iter, dIt.p, dIt.n * 4, cudaMemcpyDeviceToHost, s));
  AM_CUDA(cudaMemcpyAsync(converged, dConv.p, dConv.n, cudaMemcpyDeviceToHost, s));
  AM_CUDA(cudaMemcpyAsync(weights, dW.p, dW.n * 4, cudaMemcpyDeviceToHost, s));
  AM_CUDA(cudaMemcpyAsync(means, dM.p, dM.n * 4, cudaMemcpyDeviceToHost, s));
  AM_CUDA(cudaMemcpyAsync(covariances, dC.p, dC.n * 4, cudaMemcpyDeviceToHost, s));
  if (kpp) AM_CUDA(cudaMemcpyAsync(kpp, dKpp.p, dKpp.n * 4, cudaMemcpyDeviceToHost, s));
  if (labels) AM_CUDA(cudaMemcpyAsync(labels, dLab.p, dLab.n * 4, cudaMemcpyDeviceToHost, s));
  AM_CUDA(cudaStreamSynchronize(s));
  if (phase_ms) {
    phase_ms[0] = fit_ms;
    phase_ms[1] = sel_ms;
  }
  return AM_OK;
}
