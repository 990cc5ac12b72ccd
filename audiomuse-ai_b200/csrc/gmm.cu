// The clustering task's Gaussian mixture (tasks/clustering_helper._apply_clustering_model, method 'gmm'):
// scikit-learn's GaussianMixture(K, covariance_type='full', init_params='k-means++', n_init, tol, reg_covar).fit_predict
// in float64.  All n_init inits advance together as one batch of C = n_init K components; an init that has converged
// is masked out of every later launch, so its parameters stay those after its last M-step.
//
//   seeding   sklearn.cluster.kmeans_plusplus on the rows, all inits at once: per step the float64 distances from every
//             init's candidate rows to every row (kpp_dist_kernel), then per init the candidate with the lowest
//             potential, the scan of closest_dist_sq and the searchsorted of the host's draws (kpp_pick_kernel)
//   init      the M-step below on the one-hot responsibilities of the seed rows, weights nk / N
//   E-step    X P_c on the float64 tensor cores (mma.sync m16n8k16 f64, DMMA), only the k-slabs on or above the
//             diagonal of the upper-triangular P_c; the epilogue subtracts mu_c P_c, sums the squares and adds
//             log det and log w; only log_prob[c, n] is written (estep_kernel)
//   normalise logsumexp over an init's K components per row, the responsibilities in place, the lower bound
//   M-step    nk; resp^T X on DMMA; per component the upper-triangle 64 x 64 tiles of (resp (X - mu))^T (X - mu) on
//             DMMA, the long row axis split into chunks whose partial sums are added in chunk order (gram_kernel)
//   Cholesky  one CTA per component, 32-column panels staged in shared memory (chol_kernel); the triangular inverse
//             one CTA per (component, 32-column panel) by forward substitution (trinv_kernel); a pivot <= 0 or not
//             finite sets the ill-defined flag instead of failing the launch
//
// am_gmm_fit runs the same seeding, initialisation, normaliser, convergence loop, best-init choice and labelling for
// every covariance_type.  For 'diag', 'tied' and 'spherical' only the covariance M-step, the precision factor and the
// E-step differ from 'full', each in scikit-learn 1.9's operation order:
//
//   diag      resp^T (X o X) on DMMA (gram_kernel<false> on a device copy of X o X), cov = (that / nk - mu^2) + reg,
//             prec_chol = 1 / sqrt(cov) (diag_cov_kernel); the E-step runs the DMMA products X (mu o prec)^T and
//             (X o X) prec^T in one kernel and adds them as (sum mu^2 prec - 2 X (mu o prec)^T) + (X o X) prec^T
//             (lin_estep_kernel)
//   spherical the diag covariance averaged over the features; the E-step product is X mu^T, scaled by the precision
//             after the dot product, plus |x|^2 prec
//   tied      X^T X once per fit (gram_kernel<true> with unit weights and zero means), then per init
//             cov = (X^T X - sum_k nk mu mu^T) / sum nk + reg (tied_cov_kernel), the same Cholesky and inverse as 'full'
//             over n_init matrices, and an E-step that forms X P once per (row tile, init) and loops over the init's K
//             components in the epilogue (estep_kernel<true>)
//
// Every reduction runs in a fixed order and no floating-point atomics are used, so two calls give bit-identical
// results.
#include "common.cuh"
#include "host_call.cuh"

#include <algorithm>
#include <cmath>
#include <vector>

namespace am {
namespace gm {

constexpr int kThreads = 256;
constexpr int kWarps = kThreads / 32;
constexpr int kMaxTrials = 8;                 // 2 + floor(ln K) for K <= 512
constexpr int kPanel = 32;
constexpr double kEps = 2.220446049250313e-16;
constexpr double kLog2Pi = 1.8378770664093453;

int n_local_trials(int K) { return 2 + (int)std::log((double)K); }

// D += A B, m16n8k16, float64 operands and accumulators (DMMA.16x8x16 on sm_90).  Fragments (g = lane / 4,
// t = lane % 4): a[i] = A[g + 8 (i & 1)][t + 4 (i >> 1)], b[i] = B[t + 4 i][g], c = D[g][2t, 2t + 1], D[g + 8][2t, 2t + 1]
__device__ __forceinline__ void dmma(double (&c)[4], const double (&a)[8], const double (&b)[4]) {
  asm volatile(
      "mma.sync.aligned.m16n8k16.row.col.f64.f64.f64.f64 {%0,%1,%2,%3}, {%4,%5,%6,%7,%8,%9,%10,%11}, "
      "{%12,%13,%14,%15}, {%0,%1,%2,%3};"
      : "+d"(c[0]), "+d"(c[1]), "+d"(c[2]), "+d"(c[3])
      : "d"(a[0]), "d"(a[1]), "d"(a[2]), "d"(a[3]), "d"(a[4]), "d"(a[5]), "d"(a[6]), "d"(a[7]), "d"(b[0]), "d"(b[1]),
        "d"(b[2]), "d"(b[3]));
}

__device__ __forceinline__ double block_sum(double v, double* red) {
  v = warp_sum(v);
  const int w = threadIdx.x >> 5;
  __syncthreads();
  if ((threadIdx.x & 31) == 0) red[w] = v;
  __syncthreads();
  double s = 0.0;
  for (int i = 0; i < (int)(blockDim.x >> 5); ++i) s += red[i];
  __syncthreads();
  return s;
}

// ---------------------------------------------------------------- k-means++
__global__ void rownorm_kernel(const double* __restrict__ X, int64_t N, int dp, double* __restrict__ xsq) {
  const int lane = threadIdx.x & 31;
  for (int64_t i = (int64_t)blockIdx.x * kWarps + (threadIdx.x >> 5); i < N; i += (int64_t)gridDim.x * kWarps) {
    double s = 0.0;
    for (int c = lane; c < dp; c += 32) s = fma(X[i * dp + c], X[i * dp + c], s);
    s = warp_sum(s);
    if (lane == 0) xsq[i] = s;
  }
}

constexpr int kKppRows = 64;    // rows per kpp_dist CTA

// blockIdx.y = init: dist[init][j][i] = min(closest[init][i], max((-2 x_i.x_cj + |x_cj|^2) + |x_i|^2, 0)) for the L
// candidates cj, and the CTA's partial potentials part[init][j][blockIdx.x] (rows in order, warps in order)
__global__ void __launch_bounds__(kThreads)
kpp_dist_kernel(const double* __restrict__ X, int64_t N, int64_t Np, int dp, const double* __restrict__ xsq,
                const int* __restrict__ cand, int L, const double* __restrict__ closest, double* __restrict__ dist,
                double* __restrict__ part) {
  extern __shared__ __align__(16) double cs[];   // [L][dp]
  __shared__ double red[kWarps][kMaxTrials];
  const int init = blockIdx.y, lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  const int* cd = cand + init * kMaxTrials;
  for (int e = threadIdx.x; e < L * dp; e += kThreads) cs[e] = X[(int64_t)cd[e / dp] * dp + e % dp];
  __syncthreads();
  double pp[kMaxTrials];
#pragma unroll
  for (int j = 0; j < kMaxTrials; ++j) pp[j] = 0.0;
  const int64_t r0 = (int64_t)blockIdx.x * kKppRows;
  for (int64_t i = r0 + warp; i < std::min(N, r0 + kKppRows); i += kWarps) {
    double v[kMaxTrials];
#pragma unroll
    for (int j = 0; j < kMaxTrials; ++j) v[j] = 0.0;
    for (int c = lane; c < dp; c += 32) {
      const double x = X[i * dp + c];
#pragma unroll
      for (int j = 0; j < kMaxTrials; ++j)
        if (j < L) v[j] = fma(x, cs[j * dp + c], v[j]);
    }
    const double cl = closest[init * Np + i];
#pragma unroll
    for (int j = 0; j < kMaxTrials; ++j)
      if (j < L) {
        const double dd = fmin(cl, fmax((-2.0 * warp_sum(v[j]) + xsq[cd[j]]) + xsq[i], 0.0));
        if (lane == 0) dist[((int64_t)init * kMaxTrials + j) * Np + i] = dd;
        pp[j] += dd;
      }
  }
  if (lane == 0)
#pragma unroll
    for (int j = 0; j < kMaxTrials; ++j) red[warp][j] = pp[j];
  __syncthreads();
  if ((int)threadIdx.x < L) {
    double s = 0.0;
    for (int w = 0; w < kWarps; ++w) s += red[w][threadIdx.x];
    part[((int64_t)init * kMaxTrials + threadIdx.x) * gridDim.x + blockIdx.x] = s;
  }
}

constexpr int kPickThreads = 1024;

// one CTA per init: centre cc is the candidate with the lowest potential (first on a tie); then, when another centre
// follows, the scan of the new closest_dist_sq and the searchsorted of its L draws
__global__ void __launch_bounds__(kPickThreads)
kpp_pick_kernel(int64_t N, int64_t Np, int K, int cc, int L, int nb, const double* __restrict__ part,
                const double* __restrict__ dist, double* __restrict__ closest, double* __restrict__ cums,
                int* __restrict__ cand, int* __restrict__ idx, const double* __restrict__ draws, int64_t per_init,
                int L_next) {
  __shared__ double tot[kPickThreads];
  __shared__ int s_best;
  __shared__ double s_pot;
  const int init = blockIdx.x, tid = threadIdx.x;
  if (tid == 0) {
    int best = 0;
    double bp = 0.0;
    for (int j = 0; j < L; ++j) {
      double s = 0.0;
      for (int b = 0; b < nb; ++b) s += part[((int64_t)init * kMaxTrials + j) * nb + b];
      if (j == 0 || s < bp) {
        bp = s;
        best = j;
      }
    }
    s_best = best;
    s_pot = bp;
    idx[init * K + cc] = cand[init * kMaxTrials + best];
  }
  __syncthreads();
  const double* src = dist + ((int64_t)init * kMaxTrials + s_best) * Np;
  double* cl = closest + init * Np;
  for (int64_t i = tid; i < N; i += kPickThreads) cl[i] = src[i];
  if (cc + 1 >= K) return;
  // cumsum in row order: a contiguous chunk per thread, the chunk totals scanned by one thread
  const int64_t chunk = (N + kPickThreads - 1) / kPickThreads;
  const int64_t b0 = std::min(N, tid * chunk), b1 = std::min(N, b0 + chunk);
  double s = 0.0;
  for (int64_t i = b0; i < b1; ++i) s += src[i];
  tot[tid] = s;
  __syncthreads();
  if (tid == 0) {
    double run = 0.0;
    for (int t = 0; t < kPickThreads; ++t) {
      const double v = tot[t];
      tot[t] = run;
      run += v;
    }
  }
  __syncthreads();
  double* cs = cums + init * Np;
  s = tot[tid];
  for (int64_t i = b0; i < b1; ++i) {
    s += src[i];
    cs[i] = s;
  }
  __syncthreads();
  if (tid < L_next) {
    const double rv = draws[init * per_init + 1 + (int64_t)cc * L_next + tid] * s_pot;
    int64_t lo = 0, hi = N;                      // first i with cs[i] >= rv (searchsorted, side='left')
    while (lo < hi) {
      const int64_t mid = (lo + hi) >> 1;
      if (cs[mid] < rv) lo = mid + 1; else hi = mid;
    }
    cand[init * kMaxTrials + tid] = (int)std::min(lo, N - 1);
  }
}

__global__ void fill_kernel(double* __restrict__ p, int64_t n, double v) {
  for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (int64_t)gridDim.x * blockDim.x) p[i] = v;
}

// xx = x o x elementwise
__global__ void square_kernel(const double* __restrict__ x, int64_t n, double* __restrict__ xx) {
  for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (int64_t)gridDim.x * blockDim.x)
    xx[i] = x[i] * x[i];
}

__global__ void onehot_kernel(const int* __restrict__ idx, int C, int64_t Np, double* __restrict__ resp) {
  const int c = blockIdx.x * blockDim.x + threadIdx.x;
  if (c < C) resp[c * Np + idx[c]] = 1.0;
}

// ---------------------------------------------------------------- M-step
// nk[c] = sum_n resp[c, n] + 10 eps
__global__ void __launch_bounds__(kThreads)
nk_kernel(const double* __restrict__ resp, int64_t Np, int K, const int* __restrict__ active, double* __restrict__ nk) {
  __shared__ double red[kWarps];
  const int c = blockIdx.x;
  if (!active[c / K]) return;
  double s = 0.0;
  for (int64_t i = threadIdx.x; i < Np; i += kThreads) s += resp[c * Np + i];
  s = block_sum(s, red);
  if (threadIdx.x == 0) nk[c] = s + 10.0 * kEps;
}

constexpr int kTile = 64;       // gram output tile
constexpr int kBK = 32;         // rows per shared-memory stage
constexpr int kLd = kTile + 4;  // padded stride: the fragment loads of a half-warp hit 16 distinct bank pairs

// kCov = false: out[s][c][j] partial of sum_n resp[c, n] X[n, j], a 64 x 64 tile per (component tile, column tile).
// kCov = true: per component c and upper tile (ti <= tj), partial of sum_n resp[c, n] (X - mu_c)[n, i] (X - mu_c)[n, j].
// blockIdx.z: the row chunk s.
template <bool kCov>
__global__ void __launch_bounds__(kThreads)
gram_kernel(const double* __restrict__ X, const double* __restrict__ resp, const double* __restrict__ means,
            int64_t Np, int dp, int C, int K, const int* __restrict__ active, int64_t chunk_rows,
            double* __restrict__ out) {
  __shared__ __align__(16) double Us[kBK][kLd];
  __shared__ __align__(16) double Vs[kBK][kLd];
  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5, g = lane >> 2, t = lane & 3;
  const int d64 = (dp + kTile - 1) / kTile * kTile;
  int c = 0, i0 = 0, j0 = 0;
  if (kCov) {
    c = blockIdx.x;
    if (!active[c / K]) return;
    const int nt = d64 / kTile;
    int p = blockIdx.y, ti = 0;
    while (p >= nt - ti) {
      p -= nt - ti;
      ++ti;
    }
    i0 = ti * kTile;
    j0 = (ti + p) * kTile;
  } else {
    i0 = blockIdx.x * kTile;   // components
    j0 = blockIdx.y * kTile;   // columns
    bool any = false;          // a tile of converged inits only keeps its means
    for (int q = i0; q < min(C, i0 + kTile); q += K) any |= active[q / K] != 0;
    if (!any && (min(C, i0 + kTile) - 1) / K != i0 / K) any = active[(min(C, i0 + kTile) - 1) / K] != 0;
    if (!any) return;
  }
  const int64_t n_beg = blockIdx.z * chunk_rows, n_end = std::min(Np, n_beg + chunk_rows);
  const double* mu = kCov ? means + (int64_t)c * dp : nullptr;
  const int mt = warp & 3, nh = warp >> 2;
  double acc[4][4];
#pragma unroll
  for (int a = 0; a < 4; ++a)
#pragma unroll
    for (int b = 0; b < 4; ++b) acc[a][b] = 0.0;
  for (int64_t n0 = n_beg; n0 < n_end; n0 += kBK) {
#pragma unroll
    for (int q = 0; q < kBK * kTile / kThreads; ++q) {
      const int e = tid + q * kThreads;
      if (kCov) {
        const int r = e >> 6, m = e & 63;
        const int64_t n = n0 + r;
        const double rs = resp[(int64_t)c * Np + n];
        const int ci = i0 + m, cj = j0 + m;
        const double xi = ci < dp ? X[n * dp + ci] - mu[ci] : 0.0;
        const double xj = cj < dp ? X[n * dp + cj] - mu[cj] : 0.0;
        Us[r][m] = rs * xi;
        Vs[r][m] = xj;
      } else {
        const int r = e & 31, m = e >> 5;    // U: consecutive threads walk one component's row range
        const int cc = i0 + m;
        Us[r][m] = cc < C ? resp[(int64_t)cc * Np + n0 + r] : 0.0;
        const int r2 = e >> 6, m2 = e & 63;
        const int cj = j0 + m2;
        Vs[r2][m2] = cj < dp ? X[(n0 + r2) * dp + cj] : 0.0;
      }
    }
    __syncthreads();
#pragma unroll
    for (int kk = 0; kk < kBK; kk += 16) {
      double a[8];
#pragma unroll
      for (int i = 0; i < 8; ++i) a[i] = Us[kk + t + 4 * (i >> 1)][mt * 16 + g + 8 * (i & 1)];
#pragma unroll
      for (int nt = 0; nt < 4; ++nt) {
        double b[4];
#pragma unroll
        for (int i = 0; i < 4; ++i) b[i] = Vs[kk + t + 4 * i][nh * 32 + nt * 8 + g];
        dmma(acc[nt], a, b);
      }
    }
    __syncthreads();
  }
  const int row = mt * 16 + g;
#pragma unroll
  for (int nt = 0; nt < 4; ++nt) {
    const int col = nh * 32 + nt * 8 + 2 * t;
    if (kCov) {
      double* o = out + ((int64_t)blockIdx.z * C + c) * d64 * d64;
      o[(int64_t)(i0 + row) * d64 + j0 + col] = acc[nt][0];
      o[(int64_t)(i0 + row) * d64 + j0 + col + 1] = acc[nt][1];
      o[(int64_t)(i0 + row + 8) * d64 + j0 + col] = acc[nt][2];
      o[(int64_t)(i0 + row + 8) * d64 + j0 + col + 1] = acc[nt][3];
    } else {
      const int Cp = gridDim.x * kTile;
      double* o = out + (int64_t)blockIdx.z * Cp * d64;
      o[(int64_t)(i0 + row) * d64 + j0 + col] = acc[nt][0];
      o[(int64_t)(i0 + row) * d64 + j0 + col + 1] = acc[nt][1];
      o[(int64_t)(i0 + row + 8) * d64 + j0 + col] = acc[nt][2];
      o[(int64_t)(i0 + row + 8) * d64 + j0 + col + 1] = acc[nt][3];
    }
  }
}

// means[c][j] = (sum over chunks in order) / nk[c]
__global__ void means_reduce_kernel(const double* __restrict__ part, int S, int Cp, int d64, int dp, int K,
                                    const int* __restrict__ active, const double* __restrict__ nk,
                                    double* __restrict__ means) {
  const int c = blockIdx.x, j = threadIdx.x;
  if (!active[c / K] || j >= dp) return;
  double s = 0.0;
  for (int q = 0; q < S; ++q) s += part[((int64_t)q * Cp + c) * d64 + j];
  means[(int64_t)c * dp + j] = s / nk[c];
}

// cov[c][i][j] = (sum over chunks in order of the upper entry) / nk[c] + reg_covar on the diagonal, mirrored
__global__ void cov_reduce_kernel(const double* __restrict__ part, int S, int C, int d64, int d, int dp, int K,
                                  const int* __restrict__ active, const double* __restrict__ nk, double reg_covar,
                                  double* __restrict__ cov) {
  const int c = blockIdx.x, i = blockIdx.y;
  if (!active[c / K]) return;
  for (int j = threadIdx.x; j < d; j += blockDim.x) {
    const int a = std::min(i, j), b = std::max(i, j);
    double s = 0.0;
    for (int q = 0; q < S; ++q) s += part[((int64_t)q * C + c) * d64 * d64 + (int64_t)a * d64 + b];
    s = s / nk[c];
    if (i == j) s += reg_covar;
    cov[((int64_t)c * dp + i) * dp + j] = s;
  }
}

// weights: nk / sum of the init's nk (M-step) or nk / N (initialisation)
__global__ void weights_kernel(const double* __restrict__ nk, int n_init, int K, const int* __restrict__ active,
                               double n_rows, double* __restrict__ w) {
  const int init = blockIdx.x * blockDim.x + threadIdx.x;
  if (init >= n_init || !active[init]) return;
  double s = 0.0;
  if (n_rows > 0.0) {
    s = n_rows;
  } else {
    for (int k = 0; k < K; ++k) s += nk[init * K + k];
  }
  for (int k = 0; k < K; ++k) w[init * K + k] = nk[init * K + k] / s;
}

// diag / spherical (sph), one CTA per component, thread j = feature (d <= kThreads): the diag covariance
// cov_j = ((sum over chunks in order of resp^T (X o X)) / nk - mu_j^2) + reg_covar.
// diag: cov[c][j], prec[c][j] = 1 / sqrt(cov_j) (any cov_j <= 0 sets *fail), logdet = sum_j log prec_j, and the E-step
// columns W[c] = [mu o prec_chol^2 | prec_chol^2] (stride 2 dp), cst[c] = sum_j mu_j^2 prec_chol_j^2.
// spherical: cov[c] = mean_j cov_j, prec[c] = 1 / sqrt(cov[c]) (cov[c] <= 0 sets *fail), logdet = d log prec,
// scale[c] = prec^2 and cst[c] = sum_j mu_j^2 (the E-step columns are the means themselves).
__global__ void __launch_bounds__(kThreads)
diag_cov_kernel(bool sph, const double* __restrict__ part, int S, int Cp, int d64, int d, int dp, int K,
                const int* __restrict__ active, const double* __restrict__ nk, const double* __restrict__ means,
                const double* __restrict__ w, double reg_covar, double* __restrict__ cov, double* __restrict__ prec,
                double* __restrict__ W, double* __restrict__ cst, double* __restrict__ scale,
                double* __restrict__ logdet, double* __restrict__ logw, int* __restrict__ fail) {
  __shared__ double red[kWarps];
  const int c = blockIdx.x, j = threadIdx.x;
  if (!active[c / K]) return;
  double v = 0.0, mu = 0.0;
  if (j < d) {
    double s = 0.0;
    for (int q = 0; q < S; ++q) s += part[((int64_t)q * Cp + c) * d64 + j];
    mu = means[(int64_t)c * dp + j];
    v = (s / nk[c] - __dmul_rn(mu, mu)) + reg_covar;   // mu^2 rounded before the subtraction, as scikit-learn
  }
  if (!sph) {
    double ld = 0.0, m2 = 0.0;
    if (j < d) {
      if (v <= 0.0) *fail = 1;
      const double pc = 1.0 / sqrt(v), p = pc * pc;
      cov[(int64_t)c * dp + j] = v;
      prec[(int64_t)c * dp + j] = pc;
      W[(int64_t)c * 2 * dp + j] = mu * p;
      W[(int64_t)c * 2 * dp + dp + j] = p;
      ld = log(pc);
      m2 = mu * mu * p;
    }
    const double tl = block_sum(ld, red);
    const double tm = block_sum(m2, red);
    if (j == 0) {
      logdet[c] = tl;
      cst[c] = tm;
      logw[c] = log(w[c]);
    }
  } else {
    const double tv = block_sum(v, red);
    const double tm = block_sum(mu * mu, red);
    if (j == 0) {
      const double cv = tv / d;
      if (cv <= 0.0) *fail = 1;
      const double pc = 1.0 / sqrt(cv);
      cov[c] = cv;
      prec[c] = pc;
      scale[c] = pc * pc;
      cst[c] = tm;
      logdet[c] = d * log(pc);
      logw[c] = log(w[c]);
    }
  }
}

// tied, blockIdx.x = init, blockIdx.y = row i: cov[init][i][j] = (XtX[i][j] - sum_k (nk_k mu_ki) mu_kj) / sum_k nk_k,
// + reg_covar on the diagonal
__global__ void __launch_bounds__(kThreads)
tied_cov_kernel(const double* __restrict__ xtx, int d, int dp, int K, const int* __restrict__ active,
                const double* __restrict__ nk, const double* __restrict__ means, double reg_covar,
                double* __restrict__ cov) {
  const int init = blockIdx.x, i = blockIdx.y;
  if (!active[init]) return;
  const double* n = nk + (int64_t)init * K;
  const double* mu = means + (int64_t)init * K * dp;
  double tot = 0.0;
  for (int k = 0; k < K; ++k) tot += n[k];
  for (int j = threadIdx.x; j < d; j += kThreads) {
    double m2 = 0.0;
    for (int k = 0; k < K; ++k) m2 = fma(mu[(int64_t)k * dp + i] * n[k], mu[(int64_t)k * dp + j], m2);
    double s = (xtx[(int64_t)i * dp + j] - m2) / tot;
    if (i == j) s += reg_covar;
    cov[((int64_t)init * dp + i) * dp + j] = s;
  }
}

// ---------------------------------------------------------------- Cholesky, inverse, E-step constants
// One CTA per component: cov = L L^T into Lw (lower, row-major, stride dp), 32-column panels left to right.  A panel's
// rows are updated with the finished columns (the panel's own rows of L staged in shared memory), then factored in
// shared memory.  A pivot that is <= 0 or not finite sets *fail.
__global__ void __launch_bounds__(kThreads)
chol_kernel(const double* __restrict__ cov, int d, int dp, int K, const int* __restrict__ active,
            double* __restrict__ Lw, int* __restrict__ fail) {
  extern __shared__ __align__(16) double sm[];
  double* Lq = sm;                       // [kPanel][dp]
  double* Pn = sm + kPanel * dp;         // [dp][kPanel + 1]
  constexpr int ld = kPanel + 1;
  const int c = blockIdx.x, tid = threadIdx.x;
  if (!active[c / K]) return;
  const double* A = cov + (int64_t)c * dp * dp;
  double* L = Lw + (int64_t)c * dp * dp;
  for (int c0 = 0; c0 < d; c0 += kPanel) {
    const int w = min(kPanel, d - c0), rows = d - c0;
    for (int e = tid; e < w * c0; e += kThreads) Lq[(e / c0) * dp + e % c0] = L[(int64_t)(c0 + e / c0) * dp + e % c0];
    __syncthreads();
    for (int task = tid; task < rows * 4; task += kThreads) {
      const int r = task >> 2, jg = (task & 3) * 8;
      const double* Lr = L + (int64_t)(c0 + r) * dp;
      double acc[8];
#pragma unroll
      for (int u = 0; u < 8; ++u) acc[u] = 0.0;
      for (int k = 0; k < c0; ++k) {
        const double l = Lr[k];
#pragma unroll
        for (int u = 0; u < 8; ++u) acc[u] = fma(l, Lq[(jg + u) * dp + k], acc[u]);
      }
#pragma unroll
      for (int u = 0; u < 8; ++u)
        if (jg + u < w) Pn[r * ld + jg + u] = A[(int64_t)(c0 + r) * dp + c0 + jg + u] - acc[u];
    }
    __syncthreads();
    for (int jj = 0; jj < w; ++jj) {
      const double p = Pn[jj * ld + jj];
      if (!(p > 0.0) || !isfinite(p)) {
        if (tid == 0) *fail = 1;
        return;
      }
      const double s = sqrt(p);
      for (int r = jj + 1 + tid; r < rows; r += kThreads) Pn[r * ld + jj] /= s;
      __syncthreads();
      if (tid == 0) Pn[jj * ld + jj] = s;
      const int nc = w - jj - 1;
      for (int e = tid; e < (rows - jj - 1) * nc; e += kThreads) {
        const int r = jj + 1 + e / nc, q = jj + 1 + e % nc;
        Pn[r * ld + q] -= Pn[r * ld + jj] * Pn[q * ld + jj];
      }
      __syncthreads();
    }
    for (int e = tid; e < rows * w; e += kThreads) {
      const int r = e / w, q = e % w;
      L[(int64_t)(c0 + r) * dp + c0 + q] = r >= q ? Pn[r * ld + q] : 0.0;
    }
    __syncthreads();
  }
}

// blockIdx.x = component, blockIdx.y = 32-column panel of Z = L^-1: forward substitution down the rows,
// Z[i][j] = (delta_ij - sum_{k < i} L[i][k] Z[k][j]) / L[i][i]; 8 threads per column split k and add their partial
// sums with a fixed butterfly.  The precision Cholesky is P = Z^T (upper).
__global__ void __launch_bounds__(kThreads)
trinv_kernel(const double* __restrict__ Lw, int d, int dp, int K, const int* __restrict__ active,
             const int* __restrict__ fail, double* __restrict__ prec) {
  extern __shared__ __align__(16) double Zp[];   // [d - c0][kPanel]
  const int c = blockIdx.x, c0 = blockIdx.y * kPanel, tid = threadIdx.x;
  if (!active[c / K] || *fail || c0 >= d) return;
  const int jj = tid >> 3, kg = tid & 7, w = min(kPanel, d - c0);
  const double* L = Lw + (int64_t)c * dp * dp;
  for (int i = c0; i < d; ++i) {
    const double* Li = L + (int64_t)i * dp;
    double s = 0.0;
    for (int k = c0 + kg; k < i; k += 8) s = fma(Li[k], Zp[(k - c0) * kPanel + jj], s);
    s += __shfl_xor_sync(0xffffffffu, s, 1);
    s += __shfl_xor_sync(0xffffffffu, s, 2);
    s += __shfl_xor_sync(0xffffffffu, s, 4);
    if (kg == 0) Zp[(i - c0) * kPanel + jj] = ((i == c0 + jj ? 1.0 : 0.0) - s) / Li[i];
    __syncthreads();
  }
  double* P = prec + (int64_t)c * dp * dp;
  for (int e = tid; e < w * d; e += kThreads) {
    const int q = e / d, i = e % d;
    P[(int64_t)(c0 + q) * dp + i] = i >= c0 + q ? Zp[(i - c0) * kPanel + q] : 0.0;
  }
}

// mP[c] = mu_c P_c, logdet[c] = sum log diag P_c, logw[c] = log w_c; kTied: P_c is the init's one matrix
template <bool kTied>
__global__ void __launch_bounds__(kThreads)
prep_kernel(const double* __restrict__ means, const double* __restrict__ prec, const double* __restrict__ w, int d,
            int dp, int K, const int* __restrict__ active, double* __restrict__ mP, double* __restrict__ logdet,
            double* __restrict__ logw) {
  __shared__ double red[kWarps];
  const int c = blockIdx.x;
  if (!active[c / K]) return;
  const double* P = prec + (int64_t)(kTied ? c / K : c) * dp * dp;
  const double* mu = means + (int64_t)c * dp;
  double ld = 0.0;
  for (int j = threadIdx.x; j < d; j += kThreads) {
    double s = 0.0;
    for (int k = 0; k <= j; ++k) s = fma(mu[k], P[(int64_t)k * dp + j], s);
    mP[(int64_t)c * dp + j] = s;
    ld = log(P[(int64_t)j * dp + j]);
  }
  // fixed order: thread j's term, j < 256 = kThreads >= d
  const double t = block_sum(ld, red);
  if (threadIdx.x == 0) {
    logdet[c] = t;
    logw[c] = log(w[c]);
  }
}

// ---------------------------------------------------------------- E-step
constexpr int kEM = 64;          // rows per E-step CTA
constexpr int kXLd = 16 + 4;

// blockIdx.x = 64-row tile, blockIdx.y = component: lp[c][n] = -0.5 (d log 2 pi + |x_n P_c - mu_c P_c|^2) + log det
// P_c + log w_c.  Warp w owns rows 16 (w & 3) .. + 16 and the n-tiles 2 j + (w >> 2), j < 16, so the skipped
// below-diagonal slabs cost both column halves alike.
// kTied: blockIdx.y = init, P is the init's one matrix; X P is formed once and the epilogue runs for each of the
// init's K components in turn.
template <bool kTied>
__global__ void __launch_bounds__(kThreads)
estep_kernel(const double* __restrict__ X, int64_t Np, int d, int dp, int K, const int* __restrict__ active,
             const double* __restrict__ prec, const double* __restrict__ mP, const double* __restrict__ logdet,
             const double* __restrict__ logw, double* __restrict__ lp) {
  extern __shared__ __align__(16) double sm[];
  double* Xs = sm;                       // [kEM][kXLd]
  double* Ps = sm + kEM * kXLd;          // [16][dp + 4]
  __shared__ double red[2][kEM];
  const int c = blockIdx.y;
  if (!active[kTied ? c : c / K]) return;
  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5, g = lane >> 2, t = lane & 3;
  const int mt = warp & 3, h = warp >> 2, pld = dp + 4;
  const int64_t r0 = (int64_t)blockIdx.x * kEM;
  const double* P = prec + (int64_t)c * dp * dp;
  double acc[16][4];
#pragma unroll
  for (int j = 0; j < 16; ++j)
#pragma unroll
    for (int q = 0; q < 4; ++q) acc[j][q] = 0.0;
  for (int s0 = 0; s0 < dp; s0 += 16) {
    for (int e = tid; e < kEM * 16; e += kThreads) Xs[(e >> 4) * kXLd + (e & 15)] = X[(r0 + (e >> 4)) * dp + s0 + (e & 15)];
    const int wc = dp - s0;              // P[k][j] = 0 for j < k: only the columns from s0 on
    for (int e = tid; e < 16 * wc; e += kThreads) {
      const int k = e / wc, j = s0 + e % wc;
      Ps[k * pld + j] = P[(int64_t)(s0 + k) * dp + j];
    }
    __syncthreads();
    double a[8];
#pragma unroll
    for (int i = 0; i < 8; ++i) a[i] = Xs[(mt * 16 + g + 8 * (i & 1)) * kXLd + t + 4 * (i >> 1)];
#pragma unroll
    for (int j = 0; j < 16; ++j) {
      const int n0 = (2 * j + h) * 8;
      if (n0 >= s0 && n0 < dp) {
        double b[4];
#pragma unroll
        for (int i = 0; i < 4; ++i) b[i] = Ps[(t + 4 * i) * pld + n0 + g];
        dmma(acc[j], a, b);
      }
    }
    __syncthreads();
  }
  // full: one pass for component c; tied: one pass per component of init c, on the same X P
  for (int k = 0; k < (kTied ? K : 1); ++k) {
    const int ck = kTied ? c * K + k : c;
    const double* m = mP + (int64_t)ck * dp;
    double sa = 0.0, sb = 0.0;
#pragma unroll
    for (int j = 0; j < 16; ++j) {
      const int n0 = (2 * j + h) * 8;
      if (n0 < dp) {
        const double m0 = m[n0 + 2 * t], m1 = m[n0 + 2 * t + 1];
        const double y0 = acc[j][0] - m0, y1 = acc[j][1] - m1, y2 = acc[j][2] - m0, y3 = acc[j][3] - m1;
        sa = fma(y0, y0, sa);
        sa = fma(y1, y1, sa);
        sb = fma(y2, y2, sb);
        sb = fma(y3, y3, sb);
      }
    }
    sa += __shfl_xor_sync(0xffffffffu, sa, 1);
    sa += __shfl_xor_sync(0xffffffffu, sa, 2);
    sb += __shfl_xor_sync(0xffffffffu, sb, 1);
    sb += __shfl_xor_sync(0xffffffffu, sb, 2);
    if (t == 0) {
      red[h][mt * 16 + g] = sa;
      red[h][mt * 16 + g + 8] = sb;
    }
    __syncthreads();
    if (tid < kEM) {
      const double sq = red[0][tid] + red[1][tid];
      lp[(int64_t)ck * Np + r0 + tid] = (-0.5 * (d * kLog2Pi + sq) + logdet[ck]) + logw[ck];
    }
    if (kTied) __syncthreads();   // red is reused by the next component
  }
}

// diag / spherical (sph) E-step: blockIdx.x = 64-row tile, blockIdx.y = 64-component tile, the products
// t2[n][c] = sum_k X[n][k] W[c][k] and (diag) t3[n][c] = sum_k X2[n][k] W[c][dp + k] on DMMA (the fragment layout of
// gram_kernel), X2 the device copy of X o X, W row-major [C][ka] (diag: [mu o prec | prec], ka = 2 dp; spherical: the
// means, ka = dp).  Then, in scikit-learn's order,
//   diag:      log_prob = (cst[c] - 2 t2) + t3                               (sum mu^2 prec - 2 X (mu prec)^T + X^2 prec^T)
//   spherical: log_prob = (cst[c] s - 2 (t2 s)) + xsq[n] s,  s = scale[c]    (sum mu^2 prec - 2 (X mu^T) prec + |x|^2 prec)
// and lp[c][n] = -0.5 (d log 2 pi + log_prob) + log det + log w, for the components of active inits only.  Every
// product is rounded before it is added (__dmul_rn keeps nvcc from fusing it into an FMA), as numpy rounds it.
__global__ void __launch_bounds__(kThreads)
lin_estep_kernel(bool sph, const double* __restrict__ X, const double* __restrict__ X2, int64_t Np, int d, int dp,
                 int C, int K, const int* __restrict__ active, const double* __restrict__ W, int ka,
                 const double* __restrict__ cst, const double* __restrict__ scale, const double* __restrict__ xsq,
                 const double* __restrict__ logdet, const double* __restrict__ logw, double* __restrict__ lp) {
  __shared__ __align__(16) double Us[kBK][kLd];
  __shared__ __align__(16) double Vs[kBK][kLd];
  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5, g = lane >> 2, t = lane & 3;
  const int64_t r0 = (int64_t)blockIdx.x * kTile;
  const int c0 = blockIdx.y * kTile;
  bool any = false;            // a tile of converged inits is left alone
  for (int q = c0; q < min(C, c0 + kTile); q += K) any |= active[q / K] != 0;
  if (!any && (min(C, c0 + kTile) - 1) / K != c0 / K) any = active[(min(C, c0 + kTile) - 1) / K] != 0;
  if (!any) return;
  const int mt = warp & 3, nh = warp >> 2;
  // acc += A[rows] W[components][woff ...]^T over the dp columns of A
  auto product = [&](const double* __restrict__ A, int woff, double (&acc)[4][4]) {
#pragma unroll
    for (int a = 0; a < 4; ++a)
#pragma unroll
      for (int b = 0; b < 4; ++b) acc[a][b] = 0.0;
    for (int k0 = 0; k0 < dp; k0 += kBK) {
#pragma unroll
      for (int q = 0; q < kBK * kTile / kThreads; ++q) {
        const int e = tid + q * kThreads;
        const int r = e & 31, m = e >> 5;    // consecutive threads walk one row's (one component's) k range
        const int k = k0 + r;
        Us[r][m] = k < dp ? A[(r0 + m) * dp + k] : 0.0;
        Vs[r][m] = (c0 + m < C && k < dp) ? W[(int64_t)(c0 + m) * ka + woff + k] : 0.0;
      }
      __syncthreads();
#pragma unroll
      for (int kk = 0; kk < kBK; kk += 16) {
        double a[8];
#pragma unroll
        for (int i = 0; i < 8; ++i) a[i] = Us[kk + t + 4 * (i >> 1)][mt * 16 + g + 8 * (i & 1)];
#pragma unroll
        for (int nt = 0; nt < 4; ++nt) {
          double b[4];
#pragma unroll
          for (int i = 0; i < 4; ++i) b[i] = Vs[kk + t + 4 * i][nh * 32 + nt * 8 + g];
          dmma(acc[nt], a, b);
        }
      }
      __syncthreads();
    }
  };
  double t2[4][4], t3[4][4];
  product(X, 0, t2);
  if (!sph) product(X2, dp, t3);
#pragma unroll
  for (int nt = 0; nt < 4; ++nt)
#pragma unroll
    for (int q = 0; q < 4; ++q) {
      const int64_t n = r0 + mt * 16 + g + 8 * (q >> 1);
      const int c = c0 + nh * 32 + nt * 8 + 2 * t + (q & 1);
      if (c >= C || !active[c / K]) continue;
      double lpv;
      if (sph) {
        const double s = scale[c];
        lpv = (__dmul_rn(cst[c], s) - 2.0 * __dmul_rn(t2[nt][q], s)) + __dmul_rn(xsq[n], s);
      } else {
        lpv = (cst[c] - 2.0 * t2[nt][q]) + t3[nt][q];
      }
      lp[(int64_t)c * Np + n] = (-0.5 * (__dmul_rn(d, kLog2Pi) + lpv) + logdet[c]) + logw[c];
    }
}

// thread per (row, init): scipy's logsumexp over the init's K log-probabilities (the maxima split off, the rest
// through log1p), then log_resp = lp - norm.  labels == nullptr: resp = exp(log_resp) in place of lp and
// lpn[init][n] = norm (padded rows get resp 0).  labels != nullptr: labels[n] = argmax log_resp (first maximum).
__global__ void norm_kernel(double* __restrict__ lp, int64_t N, int64_t Np, int K, const int* __restrict__ active,
                            double* __restrict__ lpn, int64_t* __restrict__ labels) {
  const int init = blockIdx.y;
  if (!active[init]) return;
  const int64_t n = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (n >= Np) return;
  double* col = lp + (int64_t)init * K * Np + n;
  if (n >= N) {
    if (!labels)
      for (int k = 0; k < K; ++k) col[k * Np] = 0.0;
    return;
  }
  double mx = -INFINITY;
  for (int k = 0; k < K; ++k) mx = fmax(mx, col[k * Np]);
  const double shift = isfinite(mx) ? mx : 0.0;
  double cnt = 0.0, s = 0.0;
  for (int k = 0; k < K; ++k) {
    const double v = col[k * Np];
    if (v == mx) cnt += 1.0;
    else s += exp(v - shift);
  }
  if (s != 0.0) s = s / cnt;
  const double norm = (log1p(s) + log(cnt)) + mx;
  if (labels) {
    int best = 0;
    double bv = -INFINITY;
    for (int k = 0; k < K; ++k) {
      const double v = col[k * Np] - norm;
      if (k == 0 || v > bv) {
        bv = v;
        best = k;
      }
    }
    labels[n] = best;
    return;
  }
  for (int k = 0; k < K; ++k) col[k * Np] = exp(col[k * Np] - norm);
  lpn[init * Np + n] = norm;
}

__global__ void __launch_bounds__(kThreads)
lb_kernel(const double* __restrict__ lpn, int64_t N, int64_t Np, const int* __restrict__ active, double* __restrict__ lb) {
  __shared__ double red[kWarps];
  const int init = blockIdx.x;
  if (!active[init]) return;
  double s = 0.0;
  for (int64_t i = threadIdx.x; i < N; i += kThreads) s += lpn[init * Np + i];
  s = block_sum(s, red);
  if (threadIdx.x == 0) lb[init] = s / (double)N;
}

// out[k][i][j] = src[(c0 + k)][i][j] for i < rows, j < cols (strides sp between rows, sc between components)
__global__ void pack_kernel(const double* __restrict__ src, int c0, int K, int rows, int cols, int sp, int64_t sc,
                            double* __restrict__ out) {
  const int64_t total = (int64_t)K * rows * cols;
  for (int64_t e = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; e < total; e += (int64_t)gridDim.x * blockDim.x) {
    const int64_t k = e / ((int64_t)rows * cols);
    const int r = (int)(e / cols % rows), q = (int)(e % cols);
    out[e] = src[(c0 + k) * sc + (int64_t)r * sp + q];
  }
}

}  // namespace gm
}  // namespace am

using namespace am;

extern "C" int am_gmm_fit(const double* X, int64_t N, int d, int K, int type, int n_init, int max_iter, double tol,
                          double reg_covar, const double* draws, int64_t n_draws, double* weights, double* means,
                          double* covariances, double* precisions_cholesky, double* lower_bounds, int32_t* n_iter,
                          int32_t* converged, int32_t* best_init, int64_t* labels, int32_t* ill_defined, int32_t* kpp,
                          double* init_lower_bounds, int32_t* init_n_iter, int32_t* init_converged, float* phase_ms) {
  using namespace gm;
  AM_CHECK(type == AM_GMM_FULL || type == AM_GMM_DIAG || type == AM_GMM_TIED || type == AM_GMM_SPHERICAL,
           "am_gmm_fit: covariance_type %d is not AM_GMM_FULL, AM_GMM_DIAG, AM_GMM_TIED or AM_GMM_SPHERICAL", type);
  AM_CHECK(X && draws && weights && means && covariances && precisions_cholesky && lower_bounds && n_iter &&
               converged && best_init && labels && ill_defined,
           "am_gmm_fit: a required pointer is null");
  AM_CHECK(d >= 1 && d <= AM_GMM_MAX_D && K >= 1 && K <= AM_GMM_MAX_K,
           "am_gmm_fit: need 1 <= d <= %d and 1 <= K <= %d (got d = %d, K = %d)", AM_GMM_MAX_D, AM_GMM_MAX_K, d, K);
  AM_CHECK(N >= K && N <= ((int64_t)1 << 31) - 64, "am_gmm_fit: need K <= N < 2^31 - 64 (got N = %lld, K = %d)",
           (long long)N, K);
  AM_CHECK(n_init >= 1 && max_iter >= 1 && tol >= 0.0 && reg_covar >= 0.0,
           "am_gmm_fit: need n_init >= 1, max_iter >= 1, tol >= 0, reg_covar >= 0");
  AM_CHECK((int64_t)n_init * K <= AM_GMM_MAX_COMPONENTS, "am_gmm_fit: n_init K = %lld components exceeds %d",
           (long long)n_init * K, AM_GMM_MAX_COMPONENTS);
  const int L = n_local_trials(K);
  const int64_t per_init = 1 + (int64_t)(K - 1) * L;
  AM_CHECK(n_draws >= n_init * per_init, "am_gmm_fit: %lld draws, K = %d with n_init = %d needs %lld",
           (long long)n_draws, K, n_init, (long long)(n_init * per_init));
  const bool full = type == AM_GMM_FULL, tied = type == AM_GMM_TIED, sph = type == AM_GMM_SPHERICAL;
  const bool lin = type == AM_GMM_DIAG || sph;       // the E-step is one product of the rows with per-component columns

  const int dp = (d + 15) / 16 * 16, d64 = (dp + kTile - 1) / kTile * kTile;
  const int64_t Np = (N + kEM - 1) / kEM * kEM;
  const int C = n_init * K;
  const int Cp = (C + kTile - 1) / kTile * kTile;
  const int ka = sph ? dp : 2 * dp;                 // diag / spherical: row stride of the E-step columns W
  const int Cm = tied ? n_init : C;                 // covariance and precision matrices (tied: one per init)

  // the first centre of each init: choice(N, p=uniform) = searchsorted(cumsum(1/N) / last, u, 'right')
  std::vector<int> cand0((size_t)n_init * kMaxTrials, 0);
  {
    std::vector<double> cdf(N);
    double s = 0.0;
    const double pw = 1.0 / (double)N;
    for (int64_t r = 0; r < N; ++r) cdf[r] = (s += pw);
    const double last = cdf[N - 1];
    for (int64_t r = 0; r < N; ++r) cdf[r] /= last;
    for (int i = 0; i < n_init; ++i)
      cand0[(size_t)i * kMaxTrials] =
          (int)(std::upper_bound(cdf.begin(), cdf.end(), draws[i * per_init]) - cdf.begin());
  }

  // split the long row axis so that each M-step product has a few waves of CTAs
  const int sms = sm_count();
  const int64_t row_blocks = Np / kBK;
  auto split = [&](int64_t tiles, int64_t& chunk) {
    int64_t S = std::max<int64_t>(1, (4LL * sms + tiles - 1) / tiles);
    S = std::min(S, row_blocks);
    chunk = (row_blocks + S - 1) / S * kBK;
    return (int)((Np + chunk - 1) / chunk);
  };
  const int cov_tiles = (d64 / kTile) * (d64 / kTile + 1) / 2;
  int64_t mchunk = 0, cchunk = 0;
  const int Sm = split((int64_t)(Cp / kTile) * (d64 / kTile), mchunk);
  const int Sc = split((int64_t)(tied ? 1 : C) * cov_tiles, cchunk);   // tied: the one X^T X

  cudaStream_t s;
  AM_TRY(HostCall::thread_stream(&s));
  Event ev[9];
  for (auto& e : ev) AM_TRY(e.create());

  const int nb_kpp = (int)((N + kKppRows - 1) / kKppRows);
  const size_t cov_n = full ? (size_t)C * dp * dp : tied ? (size_t)n_init * dp * dp : sph ? (size_t)C : (size_t)C * dp;
  const size_t out_n = full ? (size_t)K * d * d : tied ? (size_t)d * d : sph ? (size_t)K : (size_t)K * d;
  const size_t pack_n = std::max(out_n, (size_t)K * d);   // dOut also stages the means
  const size_t x_n = (size_t)Np * dp, close_n = (size_t)n_init * Np;
  std::vector<int> act(n_init, 1);
  const int one = 1;
  HostCall call(s, 0, HostCall::Memory::Owned);
  double *dX, *dXsq, *dResp, *dClose, *dCums, *dDist, *dPart, *dNk, *dW, *dLogw, *dLogdet, *dMeans, *dMP, *dCov, *dLw,
      *dPrec, *dLpn, *dLb, *dPm, *dPc, *dOut, *dDraws;
  double *dX2, *dPm2, *dWcol, *dCst, *dScale, *dXtX, *dUnit, *dZero;   // diag / spherical / tied only
  int *dCand, *dIdx, *dActive, *dFail, *dOn;
  int64_t* dLab;
  call.up(&dCand, cand0.data(), cand0.size());
  call.up(&dDraws, draws, (size_t)n_init * per_init);
  call.up(&dActive, act.data(), (size_t)n_init);
  call.up(&dOn, &one, tied ? 1 : 0);
  call.down(&dLab, (size_t)N, labels);
  call.device(&dX, x_n, 0);   // the rows are copied in after start(), pitched
  call.device(&dXsq, (size_t)Np, 0);
  call.device(&dMeans, (size_t)C * dp, 0);
  call.device(&dMP, full || tied ? (size_t)C * dp : 0, 0);
  call.device(&dPrec, cov_n, 0);
  call.device(&dPc, full || tied ? (size_t)Sc * (tied ? 1 : C) * d64 * d64 : 0, 0);
  call.device(&dWcol, lin && !sph ? (size_t)C * ka : 0, 0);
  call.device(&dFail, 1, 0);
  call.device(&dResp, (size_t)C * Np, 0);
  call.device(&dZero, tied ? (size_t)dp : 0, 0);
  call.device(&dClose, close_n);
  call.device(&dCums, (size_t)n_init * Np);
  call.device(&dDist, (size_t)n_init * kMaxTrials * Np);
  call.device(&dPart, (size_t)n_init * kMaxTrials * nb_kpp);
  call.device(&dNk, (size_t)C);
  call.device(&dW, (size_t)C);
  call.device(&dLogw, (size_t)C);
  call.device(&dLogdet, (size_t)C);
  call.device(&dCov, cov_n);
  call.device(&dLpn, (size_t)n_init * Np);
  call.device(&dLb, (size_t)n_init);
  call.device(&dPm, (size_t)Sm * Cp * d64);
  call.device(&dOut, pack_n);
  call.device(&dIdx, (size_t)C);
  call.device(&dLw, full || tied ? cov_n : 0);
  call.device(&dX2, lin ? x_n : 0);
  call.device(&dPm2, lin ? (size_t)Sm * Cp * d64 : 0);
  call.device(&dCst, lin ? (size_t)C : 0);
  call.device(&dScale, sph ? (size_t)C : 0);
  call.device(&dXtX, tied ? (size_t)dp * dp : 0);
  call.device(&dUnit, tied ? (size_t)Np : 0);
  AM_TRY(call.start());
  AM_CUDA(cudaMemcpy2DAsync(dX, (size_t)dp * 8, X, (size_t)d * 8, (size_t)d * 8, (size_t)N, cudaMemcpyHostToDevice, s));

  const size_t chol_smem = ((size_t)kPanel * dp + (size_t)dp * (kPanel + 1)) * 8;
  const size_t trinv_smem = (size_t)dp * kPanel * 8;
  const size_t estep_smem = ((size_t)kEM * kXLd + 16 * (size_t)(dp + 4)) * 8;
  AM_TRY(allow_dynamic_smem<kpp_dist_kernel>((size_t)kMaxTrials * AM_GMM_MAX_D * 8));
  AM_TRY(allow_dynamic_smem<chol_kernel>(((size_t)kPanel * AM_GMM_MAX_D + (size_t)AM_GMM_MAX_D * (kPanel + 1)) * 8));
  AM_TRY(allow_dynamic_smem<trinv_kernel>((size_t)AM_GMM_MAX_D * kPanel * 8));
  AM_TRY(allow_dynamic_smem<estep_kernel<false>>(((size_t)kEM * kXLd + 16 * (size_t)(AM_GMM_MAX_D + 4)) * 8));
  AM_TRY(allow_dynamic_smem<estep_kernel<true>>(((size_t)kEM * kXLd + 16 * (size_t)(AM_GMM_MAX_D + 4)) * 8));

  // ---- k-means++
  AM_CUDA(cudaEventRecord(ev[0].e, s));
  AM_LAUNCH(rownorm_kernel, grid_for(N * 32), kThreads, 0, s, dX, N, dp, dXsq);
  AM_LAUNCH(fill_kernel, grid_for(close_n), 256, 0, s, dClose, (int64_t)close_n, (double)INFINITY);
  for (int cc = 0; cc < K; ++cc) {
    const int Lc = cc == 0 ? 1 : L;
    AM_LAUNCH(kpp_dist_kernel, dim3(nb_kpp, n_init), kThreads, (size_t)Lc * dp * 8, s, dX, N, Np, dp, dXsq,
              dCand, Lc, dClose, dDist, dPart);
    AM_LAUNCH(kpp_pick_kernel, n_init, kPickThreads, 0, s, N, Np, K, cc, Lc, nb_kpp, dPart, dDist, dClose,
              dCums, dCand, dIdx, dDraws, per_init, L);
  }
  AM_LAUNCH(onehot_kernel, ceil_div(C, 256), 256, 0, s, dIdx, C, Np, dResp);
  if (lin) AM_LAUNCH(square_kernel, grid_for(x_n), 256, 0, s, dX, (int64_t)x_n, dX2);
  if (tied) {   // X^T X over all rows, unweighted: gram_kernel<true> with one component, unit weights, zero mean
    AM_LAUNCH(fill_kernel, grid_for(Np), 256, 0, s, dUnit, Np, 1.0);
    AM_LAUNCH(gram_kernel<true>, dim3(1, cov_tiles, Sc), kThreads, 0, s, dX, dUnit, dZero, Np, dp, 1, 1, dOn,
              cchunk, dPc);
    AM_LAUNCH(cov_reduce_kernel, dim3(1, d), 256, 0, s, dPc, Sc, 1, d64, d, dp, 1, dOn, dUnit, 0.0, dXtX);
  }
  AM_CUDA(cudaEventRecord(ev[1].e, s));

  // ---- M-step (init = true: the initialisation's weights nk / N) and the precision factors
  auto mstep = [&](bool init, const Event& e_mid) -> int {
    AM_LAUNCH(nk_kernel, C, kThreads, 0, s, dResp, Np, K, dActive, dNk);
    AM_LAUNCH(gram_kernel<false>, dim3(Cp / kTile, d64 / kTile, Sm), kThreads, 0, s, dX, dResp, dMeans, Np, dp,
              C, K, dActive, mchunk, dPm);
    AM_LAUNCH(means_reduce_kernel, C, d64, 0, s, dPm, Sm, Cp, d64, dp, K, dActive, dNk, dMeans);
    if (full) {
      AM_LAUNCH(gram_kernel<true>, dim3(C, cov_tiles, Sc), kThreads, 0, s, dX, dResp, dMeans, Np, dp, C, K,
                dActive, cchunk, dPc);
      AM_LAUNCH(cov_reduce_kernel, dim3(C, d), 256, 0, s, dPc, Sc, C, d64, d, dp, K, dActive, dNk, reg_covar,
                dCov);
    } else if (tied) {
      AM_LAUNCH(tied_cov_kernel, dim3(n_init, d), kThreads, 0, s, dXtX, d, dp, K, dActive, dNk, dMeans,
                reg_covar, dCov);
    } else {
      AM_LAUNCH(gram_kernel<false>, dim3(Cp / kTile, d64 / kTile, Sm), kThreads, 0, s, dX2, dResp, dMeans, Np,
                dp, C, K, dActive, mchunk, dPm2);
    }
    AM_LAUNCH(weights_kernel, ceil_div(n_init, 64), 64, 0, s, dNk, n_init, K, dActive, init ? (double)N : 0.0,
              dW);
    AM_CUDA(cudaEventRecord(e_mid.e, s));
    if (lin) {
      AM_LAUNCH(diag_cov_kernel, C, kThreads, 0, s, sph, dPm2, Sm, Cp, d64, d, dp, K, dActive, dNk, dMeans, dW, reg_covar,
                dCov, dPrec, dWcol, dCst, dScale, dLogdet, dLogw, dFail);
      return AM_OK;
    }
    const int kc = full ? K : 1;                     // components per covariance matrix's active flag
    AM_LAUNCH(chol_kernel, Cm, kThreads, chol_smem, s, dCov, d, dp, kc, dActive, dLw, dFail);
    AM_LAUNCH(trinv_kernel, dim3(Cm, ceil_div(d, kPanel)), kThreads, trinv_smem, s, dLw, d, dp, kc, dActive,
              dFail, dPrec);
    if (tied)
      AM_LAUNCH(prep_kernel<true>, C, kThreads, 0, s, dMeans, dPrec, dW, d, dp, K, dActive, dMP, dLogdet,
                dLogw);
    else
      AM_LAUNCH(prep_kernel<false>, C, kThreads, 0, s, dMeans, dPrec, dW, d, dp, K, dActive, dMP, dLogdet,
                dLogw);
    return AM_OK;
  };
  auto estep = [&]() -> int {
    if (lin) {
      AM_LAUNCH(lin_estep_kernel, dim3((unsigned)(Np / kTile), Cp / kTile), kThreads, 0, s, sph, dX, sph ? nullptr : dX2, Np, d, dp,
                C, K, dActive, sph ? dMeans : dWcol, ka, dCst, dScale, dXsq, dLogdet, dLogw, dResp);
    } else if (tied) {
      AM_LAUNCH(estep_kernel<true>, dim3((unsigned)(Np / kEM), n_init), kThreads, estep_smem, s, dX, Np, d, dp, K,
                dActive, dPrec, dMP, dLogdet, dLogw, dResp);
    } else {
      AM_LAUNCH(estep_kernel<false>, dim3((unsigned)(Np / kEM), C), kThreads, estep_smem, s, dX, Np, d, dp, K,
                dActive, dPrec, dMP, dLogdet, dLogw, dResp);
    }
    return AM_OK;
  };
  auto normalise = [&](int64_t* lab) -> int {
    AM_LAUNCH(norm_kernel, dim3((unsigned)ceil_div((int)Np, 256), n_init), 256, 0, s, dResp, N, Np, K, dActive,
              dLpn, lab);
    if (!lab) AM_LAUNCH(lb_kernel, n_init, kThreads, 0, s, dLpn, N, Np, dActive, dLb);
    return AM_OK;
  };

  float ms[5] = {0.f, 0.f, 0.f, 0.f, 0.f};   // seeding, E-step, normaliser, M-step, precision factors
  AM_TRY(mstep(true, ev[2]));
  AM_CUDA(cudaEventRecord(ev[3].e, s));
  int fail = 0;
  AM_CUDA(cudaMemcpyAsync(&fail, dFail, 4, cudaMemcpyDeviceToHost, s));
  AM_CUDA(cudaStreamSynchronize(s));
  AM_TRY(add_elapsed_ms(ms[0], ev[0], ev[1]));
  AM_TRY(add_elapsed_ms(ms[3], ev[1], ev[2]));
  AM_TRY(add_elapsed_ms(ms[4], ev[2], ev[3]));
  if (kpp) AM_CUDA(cudaMemcpy(kpp, dIdx, (size_t)C * 4, cudaMemcpyDeviceToHost));

  std::vector<double> lb(n_init, -INFINITY), traj((size_t)n_init * max_iter, NAN);
  std::vector<int> it_of(n_init, 0), conv_of(n_init, 0);
  int running = n_init;
  for (int it = 1; it <= max_iter && running > 0 && !fail; ++it) {
    AM_CUDA(cudaEventRecord(ev[4].e, s));
    AM_TRY(estep());
    AM_CUDA(cudaEventRecord(ev[5].e, s));
    AM_TRY(normalise(nullptr));
    AM_CUDA(cudaEventRecord(ev[6].e, s));
    AM_TRY(mstep(false, ev[7]));
    AM_CUDA(cudaEventRecord(ev[8].e, s));
    std::vector<double> got(n_init);
    AM_CUDA(cudaMemcpyAsync(got.data(), dLb, n_init * 8, cudaMemcpyDeviceToHost, s));
    AM_CUDA(cudaMemcpyAsync(&fail, dFail, 4, cudaMemcpyDeviceToHost, s));
    AM_CUDA(cudaStreamSynchronize(s));
    AM_TRY(add_elapsed_ms(ms[1], ev[4], ev[5]));
    AM_TRY(add_elapsed_ms(ms[2], ev[5], ev[6]));
    AM_TRY(add_elapsed_ms(ms[3], ev[6], ev[7]));
    AM_TRY(add_elapsed_ms(ms[4], ev[7], ev[8]));
    for (int i = 0; i < n_init; ++i) {
      if (!act[i]) continue;
      const double prev = lb[i];
      lb[i] = got[i];
      traj[(size_t)i * max_iter + it - 1] = got[i];
      it_of[i] = it;
      if (std::fabs(got[i] - prev) < tol) {
        conv_of[i] = 1;
        act[i] = 0;
        --running;
      }
    }
    if (running > 0) AM_CUDA(cudaMemcpyAsync(dActive, act.data(), n_init * 4, cudaMemcpyHostToDevice, s));
  }
  *ill_defined = fail ? 1 : 0;
  if (fail) return AM_OK;

  // the first init with the strictly greatest final bound
  int best = 0;
  double bmax = -INFINITY;
  for (int i = 0; i < n_init; ++i)
    if (lb[i] > bmax || bmax == -INFINITY) {
      bmax = lb[i];
      best = i;
    }
  *best_init = best;
  *n_iter = it_of[best];
  *converged = conv_of[best];
  for (int q = 0; q < max_iter; ++q) lower_bounds[q] = traj[(size_t)best * max_iter + q];
  if (init_lower_bounds) std::copy(traj.begin(), traj.end(), init_lower_bounds);
  if (init_n_iter) std::copy(it_of.begin(), it_of.end(), init_n_iter);
  if (init_converged) std::copy(conv_of.begin(), conv_of.end(), init_converged);

  // labels: one more E-step on the best init's parameters
  std::fill(act.begin(), act.end(), 0);
  act[best] = 1;
  AM_CUDA(cudaMemcpyAsync(dActive, act.data(), n_init * 4, cudaMemcpyHostToDevice, s));
  AM_TRY(estep());
  AM_TRY(normalise(dLab));
  const int c0 = best * K;
  AM_CUDA(cudaMemcpyAsync(weights, dW + c0, (size_t)K * 8, cudaMemcpyDeviceToHost, s));
  AM_LAUNCH(pack_kernel, grid_for((int64_t)K * d), 256, 0, s, dMeans, c0, K, 1, d, dp, (int64_t)dp, dOut);
  AM_CUDA(cudaMemcpyAsync(means, dOut, (size_t)K * d * 8, cudaMemcpyDeviceToHost, s));
  AM_TRY(call.finish());  // the labels
  // covariances and precisions_cholesky in scikit-learn's shapes: full [K, d, d], tied [d, d], diag [K, d],
  // spherical [K]
  const int pc0 = tied ? best : c0, pK = tied ? 1 : K, rows = full || tied ? d : 1, cols = sph ? 1 : d;
  const int64_t sc = full || tied ? (int64_t)dp * dp : sph ? 1 : dp;
  for (int q = 0; q < 2; ++q) {
    AM_LAUNCH(pack_kernel, grid_for((int64_t)out_n), 256, 0, s, q ? dPrec : dCov, pc0, pK, rows, cols, dp, sc,
              dOut);
    AM_CUDA(cudaMemcpyAsync(q ? precisions_cholesky : covariances, dOut, out_n * 8, cudaMemcpyDeviceToHost, s));
    AM_CUDA(cudaStreamSynchronize(s));
  }
  if (phase_ms)
    for (int q = 0; q < 5; ++q) phase_ms[q] = ms[q];
  return AM_OK;
}
