// Spectral clustering's graph and eigensolver (tasks/clustering_gpu.py:312-335 wraps sklearn.cluster.SpectralClustering
// with affinity='nearest_neighbors', assign_labels='kmeans').  The host (clustering_gpu.spectral_embedding) runs
// Chebyshev-filtered subspace iteration; everything O(N) lives here, the host only sees b x b matrices.
//
// Graph (am_spectral_plan_create), scikit-learn's kneighbors_graph(include_self=True) -> A = 0.5 (C + C^T) -> W = A
// without its diagonal (scipy's normed laplacian ignores it), deg = row sums of W, dd = sqrt(deg):
//   k-NN lists               the exact euclidean index of knn.cu, every row a query (ids ascending distance, ties to
//                            the lower id: the same lists as a float64 ranking)
//   count_edges_kernel       per row: its own list entries + the entries that name it (the transpose), self dropped
//   scan_kernel              exclusive scan -> raw row offsets
//   scatter_edges_kernel     both directions of every edge (atomic cursors: the order inside a row is arbitrary ...)
//   sort_rows_kernel         ... so each row is rank-sorted (one warp per row, O(len^2 / 32)); a column present twice
//                            is an edge in both lists (weight 1), once an edge in one list (weight 0.5)
//   compact_rows_kernel      merge -> CSR indices i32 / weights f32, deg and dd in float64
//   normalise_kernel         s_ij = w_ij / dd_j / dd_i (scipy's order), float64: the values of S = D^-1/2 W D^-1/2
// The same count / scan / scatter / sort / compact steps build UMAP's fuzzy union (knn_csr_build with memberships,
// called from umap.cu); am_spectral_plan_create_csr starts from a given float64 graph (degree_kernel for dd).
//
// Eigensolver steps, float64 throughout (the wanted eigenvalues can be packed 1e-3 apart, so the block is never
// rounded to fp32):
//   cheb_spmm_kernel         Y_out = alpha (S Y - c Y) - beta Y_prev: one warp per row, lanes across 128 columns of
//                            the gathered neighbour rows; the three-term recurrence is fused into the SpMM epilogue
//   gram_kernel + reduce     G = V^T V, H = V^T (S V): 32 x 32 output tiles per row chunk, partials summed in a
//                            fixed order (deterministic)
//   rowmul_kernel            V Q (rotation), the Ritz residuals ||S V q - theta V q|| and the embedding V Q / dd
#include "common.cuh"

#include <algorithm>
#include <cmath>
#include <memory>

struct am_spectral_plan {
  int64_t N = 0;
  int k_nn = 0;
  int b = 0, ld = 0;  // block width, row stride (b rounded up to 32; padding columns stay 0)
  int64_t nnz = 0;
  int64_t n_spmm = 0;
  float knn_ms = 0.f, graph_ms = 0.f;
  am::Stream st;
  am::DevBuf<int64_t> indptr;
  am::DevBuf<int32_t> indices;
  am::DevBuf<float> w;    // W's values (0.5 or 1)
  am::DevBuf<double> s;   // S's values
  am::DevBuf<double> dd;  // sqrt(deg)
  am::DevBuf<double> V, Y, SV;  // the block, the recurrence's second buffer, S V
  am::DevBuf<double> part, red, Qd, theta;
};

namespace am {
namespace sp {

constexpr int kCols = 128;   // columns per SpMM warp: 4 per lane
constexpr int kRotRows = 64; // rows per rowmul CTA (8 per warp)
constexpr int kQChunk = 128; // rows of Q staged in shared memory per step

__global__ void count_edges_kernel(const int64_t* __restrict__ ids, int64_t N, int k, int* __restrict__ cnt) {
  const int64_t total = N * k;
  for (int64_t e = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; e < total; e += (int64_t)gridDim.x * blockDim.x) {
    const int64_t i = e / k, j = ids[e];
    if (j == i || j < 0 || j >= N) continue;
    atomicAdd(&cnt[i], 1);
    atomicAdd(&cnt[j], 1);
  }
}

// exclusive scan of cnt[N] -> off[N + 1]; one CTA of 1024 threads, each summing a contiguous chunk
__global__ void __launch_bounds__(1024) scan_kernel(const int* __restrict__ cnt, int64_t N, int64_t* __restrict__ off) {
  __shared__ int64_t part[1024];
  const int t = threadIdx.x;
  const int64_t chunk = (N + 1023) / 1024;
  const int64_t lo = std::min<int64_t>(N, t * chunk), hi = std::min<int64_t>(N, lo + chunk);
  int64_t s = 0;
  for (int64_t i = lo; i < hi; ++i) s += cnt[i];
  part[t] = s;
  __syncthreads();
  if (t == 0) {
    int64_t run = 0;
    for (int u = 0; u < 1024; ++u) {
      const int64_t v = part[u];
      part[u] = run;
      run += v;
    }
    off[N] = run;
  }
  __syncthreads();
  int64_t run = part[t];
  for (int64_t i = lo; i < hi; ++i) {
    off[i] = run;
    run += cnt[i];
  }
}

// memb (optional): a value per list entry, carried with both directions into raw_v
__global__ void scatter_edges_kernel(const int64_t* __restrict__ ids, int64_t N, int k, const int64_t* __restrict__ off,
                                     int* __restrict__ cursor, int32_t* __restrict__ raw, const double* __restrict__ memb,
                                     double* __restrict__ raw_v) {
  const int64_t total = N * k;
  for (int64_t e = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; e < total; e += (int64_t)gridDim.x * blockDim.x) {
    const int64_t i = e / k, j = ids[e];
    if (j == i || j < 0 || j >= N) continue;
    const int64_t pi = off[i] + atomicAdd(&cursor[i], 1), pj = off[j] + atomicAdd(&cursor[j], 1);
    raw[pi] = (int32_t)j;
    raw[pj] = (int32_t)i;
    if (memb) raw_v[pi] = raw_v[pj] = memb[e];
  }
}

// one warp per row: rank sort of the row's columns (ties by position) into `sorted` (and raw_v's values, when given,
// into sorted_v), and the number of distinct columns
__global__ void __launch_bounds__(256)
sort_rows_kernel(const int64_t* __restrict__ off, int64_t N, const int32_t* __restrict__ raw, int32_t* __restrict__ sorted,
                 int* __restrict__ ucnt, const double* __restrict__ raw_v, double* __restrict__ sorted_v) {
  const int lane = threadIdx.x & 31;
  const int64_t warps = (int64_t)gridDim.x * (blockDim.x >> 5);
  for (int64_t row = (int64_t)blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5); row < N; row += warps) {
    const int64_t base = off[row];
    const int L = (int)(off[row + 1] - base);
    const int32_t* r = raw + base;
    int32_t* o = sorted + base;
    for (int p = lane; p < L; p += 32) {
      const int32_t x = r[p];
      int rank = 0;
      for (int q = 0; q < L; ++q) {
        const int32_t y = r[q];
        rank += (y < x) || (y == x && q < p);
      }
      o[rank] = x;
      if (raw_v) sorted_v[base + rank] = raw_v[base + p];
    }
    __syncwarp();
    int u = 0;
    for (int p = lane; p < L; p += 32) u += (p == 0 || o[p] != o[p - 1]);
#pragma unroll
    for (int s = 16; s > 0; s >>= 1) u += __shfl_xor_sync(0xffffffffu, u, s);
    if (lane == 0) ucnt[row] = u;
  }
}

// one warp per row: distinct columns -> CSR.  Affinity (kFuzzy false): weight 1 for a column present twice (i in j's
// list and j in i's), 0.5 otherwise; deg = the row sum (exact: multiples of 0.5), dd = sqrt(deg).  Fuzzy union (kFuzzy
// true, UMAP's W = A + A^T - A o A^T): from the carried memberships, a + b - a b for a column present twice (the same
// value in either order), a for one present once, into w64; w and dd are not written.
template <bool kFuzzy>
__global__ void __launch_bounds__(256)
compact_rows_kernel(const int64_t* __restrict__ off, int64_t N, const int32_t* __restrict__ sorted,
                    const int64_t* __restrict__ indptr, int32_t* __restrict__ indices, float* __restrict__ w,
                    double* __restrict__ dd, const double* __restrict__ sorted_v, double* __restrict__ w64) {
  const int lane = threadIdx.x & 31;
  const int64_t warps = (int64_t)gridDim.x * (blockDim.x >> 5);
  for (int64_t row = (int64_t)blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5); row < N; row += warps) {
    const int64_t base = off[row];
    const int L = (int)(off[row + 1] - base);
    const int32_t* s = sorted + base;
    int64_t out = indptr[row];
    double deg = 0.0;
    for (int p0 = 0; p0 < L; p0 += 32) {
      const int p = p0 + lane;
      const bool valid = p < L;
      const int32_t x = valid ? s[p] : 0;
      const bool first = valid && (p == 0 || s[p - 1] != x);
      const unsigned m = __ballot_sync(0xffffffffu, first);
      if (first) {
        const bool twice = p + 1 < L && s[p + 1] == x;
        const int64_t pos = out + __popc(m & ((1u << lane) - 1u));
        indices[pos] = x;
        if (kFuzzy) {
          const double a = sorted_v[base + p], b = twice ? sorted_v[base + p + 1] : 0.0;
          w64[pos] = twice ? a + b - a * b : a;
        } else {
          const float wt = twice ? 1.0f : 0.5f;
          w[pos] = wt;
          deg += wt;
        }
      }
      out += __popc(m);
    }
    if (kFuzzy) continue;
    deg = warp_sum(deg);
    if (lane == 0) dd[row] = sqrt(deg);
  }
}

// one warp per row: deg = the row sum of a float64 W (lanes strided over the row, then a fixed shuffle tree), dd = sqrt
__global__ void __launch_bounds__(256)
degree_kernel(const int64_t* __restrict__ indptr, int64_t N, const double* __restrict__ w, double* __restrict__ dd) {
  const int lane = threadIdx.x & 31;
  const int64_t warps = (int64_t)gridDim.x * (blockDim.x >> 5);
  for (int64_t row = (int64_t)blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5); row < N; row += warps) {
    double deg = 0.0;
    for (int64_t p = indptr[row] + lane; p < indptr[row + 1]; p += 32) deg += w[p];
    deg = warp_sum(deg);
    if (lane == 0) dd[row] = sqrt(deg);
  }
}

template <typename T>
__global__ void __launch_bounds__(256)
normalise_kernel(const int64_t* __restrict__ indptr, int64_t N, const int32_t* __restrict__ indices,
                 const T* __restrict__ w, const double* __restrict__ dd, double* __restrict__ s) {
  const int lane = threadIdx.x & 31;
  const int64_t warps = (int64_t)gridDim.x * (blockDim.x >> 5);
  for (int64_t row = (int64_t)blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5); row < N; row += warps) {
    const double di = dd[row];
    for (int64_t p = indptr[row] + lane; p < indptr[row + 1]; p += 32) s[p] = (double)w[p] / dd[indices[p]] / di;
  }
}

__device__ __forceinline__ uint64_t splitmix64(uint64_t x) {
  x += 0x9E3779B97F4A7C15ull;
  x = (x ^ (x >> 30)) * 0xBF58476D1CE4E5B9ull;
  x = (x ^ (x >> 27)) * 0x94D049BB133111EBull;
  return x ^ (x >> 31);
}

// seeded start block: uniform in [-1, 1) for the b columns, 0 in the padding
__global__ void init_block_kernel(double* __restrict__ V, int64_t N, int b, int ld, uint64_t seed) {
  const int64_t total = N * ld;
  for (int64_t e = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; e < total; e += (int64_t)gridDim.x * blockDim.x) {
    const int c = (int)(e % ld);
    const uint64_t h = splitmix64(seed ^ splitmix64((uint64_t)e));
    V[e] = c < b ? (double)(h >> 11) * 0x1.0p-52 - 1.0 : 0.0;
  }
}

// out[i, :] = alpha (sum_j s_ij Y[j, :] - c Y[i, :]) - beta P[i, :]; out may alias P (each row reads its own P row
// before the same lanes write it), never Y.  One warp per row; blockIdx.y picks 128 columns, 4 per lane.
__global__ void __launch_bounds__(256)
cheb_spmm_kernel(const int64_t* __restrict__ indptr, const int32_t* __restrict__ indices, const double* __restrict__ s,
                 int64_t N, int ld, const double* __restrict__ Y, const double* P, double* out, double alpha,
                 double c, double beta) {
  const int lane = threadIdx.x & 31;
  const int64_t row = (int64_t)blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5);
  if (row >= N) return;
  const int col0 = blockIdx.y * kCols + lane;
  double acc[4] = {0.0, 0.0, 0.0, 0.0};
  const int64_t p0 = indptr[row], p1 = indptr[row + 1];
  for (int64_t pb = p0; pb < p1; pb += 32) {
    const int n = (int)std::min<int64_t>(32, p1 - pb);
    int32_t jl = 0;
    double sl = 0.0;
    if (lane < n) {
      jl = indices[pb + lane];
      sl = s[pb + lane];
    }
    for (int t = 0; t < n; ++t) {
      const int32_t j = __shfl_sync(0xffffffffu, jl, t);
      const double sv = __shfl_sync(0xffffffffu, sl, t);
      const double* y = Y + (int64_t)j * ld + col0;
#pragma unroll
      for (int q = 0; q < 4; ++q)
        if (col0 + 32 * q < ld) acc[q] = fma(sv, __ldg(y + 32 * q), acc[q]);  // uniform: ld is a multiple of 32
    }
  }
  const double* yi = Y + row * ld + col0;
  const double* pi = P ? P + row * ld + col0 : nullptr;
  double* o = out + row * ld + col0;
#pragma unroll
  for (int q = 0; q < 4; ++q) {
    if (col0 + 32 * q >= ld) continue;
    double v = alpha * (acc[q] - c * yi[32 * q]);
    if (pi) v -= beta * pi[32 * q];
    o[32 * q] = v;
  }
}

// part[p][r, c] = sum over rows of chunk p of A[:, r] B[:, c] for one 32 x 32 output tile (blockIdx.x, blockIdx.y)
__global__ void __launch_bounds__(256)
gram_kernel(const double* __restrict__ A, const double* __restrict__ B, int64_t N, int b, int ld, int64_t rows_per_chunk,
            double* __restrict__ part) {
  __shared__ double As[32][33], Bs[32][33];
  const int tx = threadIdx.x & 31, ty = threadIdx.x >> 5;
  const int r0 = blockIdx.x * 32, c0 = blockIdx.y * 32;
  const int64_t lo = (int64_t)blockIdx.z * rows_per_chunk, hi = std::min<int64_t>(N, lo + rows_per_chunk);
  double acc[4] = {0.0, 0.0, 0.0, 0.0};
  for (int64_t base = lo; base < hi; base += 32) {
    for (int rr = ty; rr < 32; rr += 8) {
      const int64_t row = base + rr;
      const bool ok = row < hi;
      As[rr][tx] = ok && r0 + tx < ld ? A[row * ld + r0 + tx] : 0.0;
      Bs[rr][tx] = ok && c0 + tx < ld ? B[row * ld + c0 + tx] : 0.0;
    }
    __syncthreads();
#pragma unroll 8
    for (int rr = 0; rr < 32; ++rr) {
      const double bv = Bs[rr][tx];
#pragma unroll
      for (int q = 0; q < 4; ++q) acc[q] = fma(As[rr][ty * 4 + q], bv, acc[q]);
    }
    __syncthreads();
  }
  double* out = part + (int64_t)blockIdx.z * b * b;
#pragma unroll
  for (int q = 0; q < 4; ++q) {
    const int r = r0 + ty * 4 + q, c = c0 + tx;
    if (r < b && c < b) out[(int64_t)r * b + c] = acc[q];
  }
}

// out[e] = sum_{p < P} part[p * E + e], in p order
__global__ void reduce_parts_kernel(const double* __restrict__ part, int P, int64_t E, double* __restrict__ out) {
  for (int64_t e = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; e < E; e += (int64_t)gridDim.x * blockDim.x) {
    double s = 0.0;
    for (int p = 0; p < P; ++p) s += part[(int64_t)p * E + e];
    out[e] = s;
  }
}

enum RowMul { kRotate = 0, kResidual = 1, kEmbed = 2 };

// Products of the block with a b x ncols matrix Q (row-major, Q[l * ncols + c]); CTA = 64 rows x 32 columns, 8 rows per
// warp, lane = column.  Q is staged 128 rows at a time in shared memory; the block's row values reach the lanes by
// shuffles.
//   kRotate    out[i, c] = (V Q)[i, c] for c < ncols, 0 for ncols <= c < ld
//   kResidual  per CTA and column: sum_i ((W Q)[i, c] - theta_c (V Q)[i, c])^2 and sum_i (V Q)[i, c]^2 -> part
//              [gridDim.x][2][ncols], W = S V
//   kEmbed     emb[i, c] = (V Q)[i, c] / dd[i], [N, ncols]
template <int kMode>
__global__ void __launch_bounds__(256)
rowmul_kernel(const double* __restrict__ V, const double* __restrict__ W, int64_t N, int b, int ld,
              const double* __restrict__ Q, int ncols, const double* __restrict__ theta, const double* __restrict__ dd,
              double* __restrict__ out, double* __restrict__ emb, double* __restrict__ part) {
  __shared__ double Qs[kQChunk][32];
  __shared__ double red[2][8][32];
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  const int c = blockIdx.y * 32 + lane;
  const int64_t row0 = (int64_t)blockIdx.x * kRotRows + warp * 8;
  const int nr = (int)max((int64_t)0, min((int64_t)8, N - row0));  // rows of this warp, uniform
  double av[8], aw[8];
#pragma unroll
  for (int r = 0; r < 8; ++r) av[r] = aw[r] = 0.0;
  for (int l0 = 0; l0 < b; l0 += kQChunk) {
    const int nl = min(kQChunk, b - l0);
    __syncthreads();
    for (int e = threadIdx.x; e < kQChunk * 32; e += 256) {
      const int l = e >> 5, cc = blockIdx.y * 32 + (e & 31);
      Qs[l][e & 31] = (l < nl && cc < ncols) ? Q[(int64_t)(l0 + l) * ncols + cc] : 0.0;
    }
    __syncthreads();
    for (int t = 0; t < nl; t += 32) {
      const bool lv = t + lane < nl;
      double vl[8], wl[8];
#pragma unroll
      for (int r = 0; r < 8; ++r) {
        const int64_t at = (row0 + r) * ld + l0 + t + lane;
        vl[r] = (r < nr && lv) ? V[at] : 0.0;
        wl[r] = (kMode == kResidual && r < nr && lv) ? W[at] : 0.0;
      }
#pragma unroll 4
      for (int u = 0; u < 32; ++u) {  // rows of Qs past nl are 0
        const double q = Qs[t + u][lane];
#pragma unroll
        for (int r = 0; r < 8; ++r) {
          av[r] = fma(__shfl_sync(0xffffffffu, vl[r], u), q, av[r]);
          if (kMode == kResidual) aw[r] = fma(__shfl_sync(0xffffffffu, wl[r], u), q, aw[r]);
        }
      }
    }
  }
  if (kMode == kRotate) {
    if (c >= ld) return;
#pragma unroll
    for (int r = 0; r < 8; ++r) {
      const int64_t row = row0 + r;
      if (row < N) out[row * ld + c] = c < ncols ? av[r] : 0.0;
    }
  } else if (kMode == kEmbed) {
    if (c >= ncols) return;
#pragma unroll
    for (int r = 0; r < 8; ++r) {
      const int64_t row = row0 + r;
      if (row < N) emb[row * ncols + c] = av[r] / dd[row];
    }
  } else {
    const double th = c < ncols ? theta[c] : 0.0;
    double rs = 0.0, us = 0.0;
#pragma unroll
    for (int r = 0; r < 8; ++r) {
      if (r >= nr) continue;
      const double d = aw[r] - th * av[r];
      rs = fma(d, d, rs);
      us = fma(av[r], av[r], us);
    }
    red[0][warp][lane] = rs;
    red[1][warp][lane] = us;
    __syncthreads();
    if (warp == 0 && c < ncols) {
      double a = 0.0, u = 0.0;
      for (int w8 = 0; w8 < 8; ++w8) {
        a += red[0][w8][lane];
        u += red[1][w8][lane];
      }
      part[(int64_t)blockIdx.x * 2 * ncols + c] = a;
      part[(int64_t)blockIdx.x * 2 * ncols + ncols + c] = u;
    }
  }
}

int row_grid(int64_t rows) {
  return (int)std::max<int64_t>(1, std::min<int64_t>((rows + 7) / 8, (int64_t)sm_count() * 16));
}
int flat_grid(int64_t n) { return (int)std::max<int64_t>(1, std::min<int64_t>((n + 255) / 256, (int64_t)sm_count() * 8)); }

int spmm(am_spectral_plan* p, const double* Y, const double* P, double* out, double alpha, double c, double beta) {
  const dim3 grid((unsigned)((p->N + 7) / 8), (unsigned)ceil_div(p->ld, kCols));
  AM_LAUNCH(cheb_spmm_kernel, grid, 256, 0, p->st.s, p->indptr.p, p->indices.p, p->s.p, p->N, p->ld, Y, P, out, alpha,
            c, beta);
  ++p->n_spmm;
  return AM_OK;
}

// G = A^T B into `dst` (b x b, device)
int gram(am_spectral_plan* p, const double* A, const double* B, double* dst) {
  const int tiles = ceil_div(p->b, 32);
  const int64_t max_chunks = std::max<int64_t>(1, (p->N + 31) / 32);
  const int chunks = (int)std::min<int64_t>(max_chunks, std::max<int64_t>(1, (4LL * sm_count() + tiles * tiles - 1) /
                                                                                  ((int64_t)tiles * tiles)));
  const int64_t rows_per_chunk = round_up((size_t)((p->N + chunks - 1) / chunks), 32);
  const int used = (int)((p->N + rows_per_chunk - 1) / rows_per_chunk);
  const int64_t E = (int64_t)p->b * p->b;
  AM_TRY(p->part.ensure((size_t)used * E));
  AM_LAUNCH(gram_kernel, dim3((unsigned)tiles, (unsigned)tiles, (unsigned)used), 256, 0, p->st.s, A, B, p->N, p->b, p->ld,
            rows_per_chunk, p->part.p);
  AM_LAUNCH(reduce_parts_kernel, flat_grid(E), 256, 0, p->st.s, p->part.p, used, E, dst);
  return AM_OK;
}

int upload_q(am_spectral_plan* p, const double* Q, int ncols) {
  AM_TRY(p->Qd.ensure((size_t)p->b * ncols));
  AM_CUDA(cudaMemcpyAsync(p->Qd.p, Q, (size_t)p->b * ncols * 8, cudaMemcpyHostToDevice, p->st.s));
  return AM_OK;
}

// the block buffers and the seeded start block V (synchronises)
int init_block(am_spectral_plan* p, uint64_t seed) {
  const size_t blk = (size_t)p->N * p->ld;
  AM_TRY(p->V.alloc(blk));
  AM_TRY(p->Y.alloc(blk));
  AM_TRY(p->SV.alloc(blk));
  AM_TRY(p->red.alloc((size_t)2 * p->b * p->b));
  AM_LAUNCH(init_block_kernel, flat_grid((int64_t)blk), 256, 0, p->st.s, p->V.p, p->N, p->b, p->ld, seed);
  AM_CUDA(cudaStreamSynchronize(p->st.s));
  return AM_OK;
}

dim3 rowmul_grid(const am_spectral_plan* p, int ncols) {
  return dim3((unsigned)((p->N + kRotRows - 1) / kRotRows), (unsigned)ceil_div(ncols, 32));
}

}  // namespace sp

int csr_scan(const int* cnt, int64_t N, int64_t* off, cudaStream_t st) {
  AM_LAUNCH(sp::scan_kernel, 1, 1024, 0, st, cnt, N, off);
  return AM_OK;
}

int knn_csr_build(const int64_t* ids, const double* memb, int64_t N, int k, cudaStream_t st, DevBuf<int64_t>& indptr,
                  DevBuf<int32_t>& indices, DevBuf<float>* w32, DevBuf<double>* dd, DevBuf<double>* w64, int64_t* nnz) {
  const bool fuzzy = memb != nullptr;
  DevBuf<int64_t> off;
  DevBuf<int> cnt, cursor;
  DevBuf<int32_t> raw, sorted;
  DevBuf<double> raw_v, sorted_v;
  AM_TRY(cnt.alloc((size_t)N));
  AM_TRY(cursor.alloc((size_t)N));
  AM_TRY(off.alloc((size_t)N + 1));
  AM_TRY(indptr.alloc((size_t)N + 1));
  if (!fuzzy) AM_TRY(dd->alloc((size_t)N));
  AM_CUDA(cudaMemsetAsync(cnt.p, 0, (size_t)N * 4, st));
  AM_CUDA(cudaMemsetAsync(cursor.p, 0, (size_t)N * 4, st));
  const int eg = sp::flat_grid(N * k), rg = sp::row_grid(N);
  AM_LAUNCH(sp::count_edges_kernel, eg, 256, 0, st, ids, N, k, cnt.p);
  AM_LAUNCH(sp::scan_kernel, 1, 1024, 0, st, cnt.p, N, off.p);
  int64_t raw_nnz = 0;
  AM_CUDA(cudaMemcpyAsync(&raw_nnz, off.p + N, 8, cudaMemcpyDeviceToHost, st));
  AM_CUDA(cudaStreamSynchronize(st));
  AM_TRY(raw.alloc((size_t)std::max<int64_t>(1, raw_nnz)));
  AM_TRY(sorted.alloc((size_t)std::max<int64_t>(1, raw_nnz)));
  if (fuzzy) {
    AM_TRY(raw_v.alloc((size_t)std::max<int64_t>(1, raw_nnz)));
    AM_TRY(sorted_v.alloc((size_t)std::max<int64_t>(1, raw_nnz)));
  }
  AM_LAUNCH(sp::scatter_edges_kernel, eg, 256, 0, st, ids, N, k, off.p, cursor.p, raw.p, memb, raw_v.p);
  AM_LAUNCH(sp::sort_rows_kernel, rg, 256, 0, st, off.p, N, raw.p, sorted.p, cnt.p, raw_v.p, sorted_v.p);
  AM_LAUNCH(sp::scan_kernel, 1, 1024, 0, st, cnt.p, N, indptr.p);
  AM_CUDA(cudaMemcpyAsync(nnz, indptr.p + N, 8, cudaMemcpyDeviceToHost, st));
  AM_CUDA(cudaStreamSynchronize(st));
  AM_TRY(indices.alloc((size_t)std::max<int64_t>(1, *nnz)));
  if (fuzzy) {
    AM_TRY(w64->alloc((size_t)std::max<int64_t>(1, *nnz)));
    AM_LAUNCH(sp::compact_rows_kernel<true>, rg, 256, 0, st, off.p, N, sorted.p, indptr.p, indices.p, nullptr, nullptr,
              sorted_v.p, w64->p);
  } else {
    AM_TRY(w32->alloc((size_t)std::max<int64_t>(1, *nnz)));
    AM_LAUNCH(sp::compact_rows_kernel<false>, rg, 256, 0, st, off.p, N, sorted.p, indptr.p, indices.p, w32->p, dd->p,
              nullptr, nullptr);
  }
  // the scratch buffers are freed on return: finish with them first
  AM_CUDA(cudaStreamSynchronize(st));
  return AM_OK;
}

int knn_self_query(const float* X, int64_t N, int d, int k, cudaStream_t st, const Event& t0, const Event& t1,
                   DevBuf<float>& dX, DevBuf<int64_t>& ids, DevBuf<float>& dist) {
  AM_TRY(dX.alloc((size_t)N * d));
  AM_CUDA(cudaMemcpyAsync(dX.p, X, (size_t)N * d * 4, cudaMemcpyHostToDevice, st));
  AM_TRY(ids.alloc((size_t)N * k));
  AM_TRY(dist.alloc((size_t)N * k));
  AM_CUDA(cudaEventRecord(t0.e, st));
  am_index* idx = nullptr;
  AM_TRY(am_knn_build_dev(dX.p, N, d, 1, st, &idx));
  const int qs = am_knn_query_dev(idx, dX.p, (int)N, k, 0, ids.p, dist.p, st);
  am_knn_free(idx);
  AM_TRY(qs);
  AM_CUDA(cudaEventRecord(t1.e, st));
  return AM_OK;
}

}  // namespace am

using namespace am;

extern "C" int am_spectral_plan_create(const float* X, int64_t N, int d, int n_neighbors, int block, uint64_t seed,
                                       am_spectral_plan** out) {
  AM_CHECK(X && out && N >= 2 && d >= 1, "am_spectral_plan_create: bad argument (need X, out, N >= 2, d >= 1)");
  AM_CHECK(N <= (int64_t)INT32_MAX, "am_spectral_plan_create: N = %lld exceeds 2^31 - 1 (int32 column indices)",
           (long long)N);
  AM_CHECK(n_neighbors >= 2 && n_neighbors <= N, "am_spectral_plan_create: n_neighbors = %d outside [2, N = %lld]",
           n_neighbors, (long long)N);
  AM_CHECK(block >= 1 && block <= N, "am_spectral_plan_create: block = %d outside [1, N = %lld]", block, (long long)N);
  *out = nullptr;
  AM_TRY(ensure_init());
  std::unique_ptr<am_spectral_plan> p(new am_spectral_plan());
  p->N = N;
  p->k_nn = n_neighbors;
  p->b = block;
  p->ld = (int)round_up((size_t)block, 32);
  AM_TRY(p->st.create());
  cudaStream_t st = p->st.s;
  Event ev[3];
  for (auto& e : ev) AM_TRY(e.create());
  DevBuf<float> dX, dist;
  DevBuf<int64_t> ids;
  AM_TRY(knn_self_query(X, N, d, n_neighbors, st, ev[0], ev[1], dX, ids, dist));
  AM_TRY(knn_csr_build(ids.p, nullptr, N, n_neighbors, st, p->indptr, p->indices, &p->w, &p->dd, nullptr, &p->nnz));
  AM_TRY(p->s.alloc((size_t)std::max<int64_t>(1, p->nnz)));
  AM_LAUNCH(sp::normalise_kernel<float>, sp::row_grid(N), 256, 0, st, p->indptr.p, N, p->indices.p, p->w.p, p->dd.p,
            p->s.p);
  AM_CUDA(cudaEventRecord(ev[2].e, st));
  AM_TRY(sp::init_block(p.get(), seed));
  AM_TRY(add_elapsed_ms(p->knn_ms, ev[0], ev[1]));
  AM_TRY(add_elapsed_ms(p->graph_ms, ev[1], ev[2]));
  *out = p.release();
  return AM_OK;
}

extern "C" int am_spectral_plan_create_csr(const int64_t* indptr, const int32_t* indices, const double* weights,
                                           int64_t N, int block, uint64_t seed, am_spectral_plan** out) {
  AM_CHECK(indptr && out && N >= 1, "am_spectral_plan_create_csr: bad argument (need indptr, out, N >= 1)");
  AM_CHECK(N <= (int64_t)INT32_MAX, "am_spectral_plan_create_csr: N = %lld exceeds 2^31 - 1", (long long)N);
  AM_CHECK(block >= 1 && block <= N, "am_spectral_plan_create_csr: block = %d outside [1, N = %lld]", block,
           (long long)N);
  const int64_t nnz = indptr[N];
  AM_CHECK(indptr[0] == 0 && nnz >= 0 && (nnz == 0 || (indices && weights)),
           "am_spectral_plan_create_csr: bad CSR (indptr[0] must be 0; indices and weights needed when nnz > 0)");
  for (int64_t i = 0; i < N; ++i)
    AM_CHECK(indptr[i + 1] > indptr[i], "am_spectral_plan_create_csr: row %lld is empty (zero degree)", (long long)i);
  for (int64_t e = 0; e < nnz; ++e)
    AM_CHECK(indices[e] >= 0 && indices[e] < N && weights[e] > 0.0 && std::isfinite(weights[e]),
             "am_spectral_plan_create_csr: entry %lld has a column outside [0, N) or a weight that is not finite and "
             "positive", (long long)e);
  *out = nullptr;
  AM_TRY(ensure_init());
  std::unique_ptr<am_spectral_plan> p(new am_spectral_plan());
  p->N = N;
  p->b = block;
  p->ld = (int)round_up((size_t)block, 32);
  p->nnz = nnz;
  AM_TRY(p->st.create());
  cudaStream_t st = p->st.s;
  DevBuf<double> w;
  AM_TRY(p->indptr.alloc((size_t)N + 1));
  AM_TRY(p->indices.alloc((size_t)nnz));
  AM_TRY(w.alloc((size_t)nnz));
  AM_TRY(p->s.alloc((size_t)nnz));
  AM_TRY(p->dd.alloc((size_t)N));
  AM_CUDA(cudaMemcpyAsync(p->indptr.p, indptr, ((size_t)N + 1) * 8, cudaMemcpyHostToDevice, st));
  AM_CUDA(cudaMemcpyAsync(p->indices.p, indices, (size_t)nnz * 4, cudaMemcpyHostToDevice, st));
  AM_CUDA(cudaMemcpyAsync(w.p, weights, (size_t)nnz * 8, cudaMemcpyHostToDevice, st));
  AM_LAUNCH(sp::degree_kernel, sp::row_grid(N), 256, 0, st, p->indptr.p, N, w.p, p->dd.p);
  AM_LAUNCH(sp::normalise_kernel<double>, sp::row_grid(N), 256, 0, st, p->indptr.p, N, p->indices.p, w.p, p->dd.p,
            p->s.p);
  AM_TRY(sp::init_block(p.get(), seed));  // synchronises before w is freed
  *out = p.release();
  return AM_OK;
}

extern "C" int am_spectral_plan_info(const am_spectral_plan* p, int64_t* nnz, int* block, int64_t* n_spmm,
                                     float* knn_ms, float* graph_ms) {
  AM_CHECK(p, "am_spectral_plan_info: NULL plan");
  if (nnz) *nnz = p->nnz;
  if (block) *block = p->b;
  if (n_spmm) *n_spmm = p->n_spmm;
  if (knn_ms) *knn_ms = p->knn_ms;
  if (graph_ms) *graph_ms = p->graph_ms;
  return AM_OK;
}

extern "C" int am_spectral_plan_graph(am_spectral_plan* p, int64_t* indptr, int32_t* indices, float* data, double* dd) {
  AM_CHECK(p, "am_spectral_plan_graph: NULL plan");
  AM_CHECK(!data || !p->nnz || p->w.p, "am_spectral_plan_graph: a plan made from a CSR keeps no float32 W");
  cudaStream_t st = p->st.s;
  if (indptr) AM_CUDA(cudaMemcpyAsync(indptr, p->indptr.p, ((size_t)p->N + 1) * 8, cudaMemcpyDeviceToHost, st));
  if (indices && p->nnz) AM_CUDA(cudaMemcpyAsync(indices, p->indices.p, (size_t)p->nnz * 4, cudaMemcpyDeviceToHost, st));
  if (data && p->nnz) AM_CUDA(cudaMemcpyAsync(data, p->w.p, (size_t)p->nnz * 4, cudaMemcpyDeviceToHost, st));
  if (dd) AM_CUDA(cudaMemcpyAsync(dd, p->dd.p, (size_t)p->N * 8, cudaMemcpyDeviceToHost, st));
  AM_CUDA(cudaStreamSynchronize(st));
  return AM_OK;
}

extern "C" int am_spectral_plan_iterate(am_spectral_plan* p, const double* Q, int degree, double cut, double* G,
                                        double* H) {
  AM_CHECK(p && G && H, "am_spectral_plan_iterate: NULL argument");
  AM_CHECK(degree >= 0 && (degree == 0 || (cut > -1.0 && cut < 1.0)),
           "am_spectral_plan_iterate: need degree >= 0 and, with a filter, -1 < cut < 1 (got %d, %g)", degree, cut);
  cudaStream_t st = p->st.s;
  if (Q) {
    AM_TRY(sp::upload_q(p, Q, p->b));
    AM_LAUNCH(sp::rowmul_kernel<sp::kRotate>, sp::rowmul_grid(p, p->ld), 256, 0, st, p->V.p, nullptr, p->N, p->b, p->ld,
              p->Qd.p, p->b, nullptr, nullptr, p->Y.p, nullptr, nullptr);
    std::swap(p->V.p, p->Y.p);
  }
  if (degree > 0) {
    // scaled Chebyshev filter: p_m(x) = T_m((x - c) / e) / T_m(t0), damping [-1, cut] and equal to 1 at x = 1;
    // sigma_k = T_{k-1}(t0) / T_k(t0) keeps every coefficient finite
    const double e = (cut + 1.0) / 2.0, c = (cut - 1.0) / 2.0, t0 = (1.0 - c) / e;
    double sigma = 1.0 / t0;
    AM_TRY(sp::spmm(p, p->V.p, nullptr, p->Y.p, sigma / e, c, 0.0));  // Y = p_1(S) V
    double* cur = p->Y.p;   // p_k(S) V
    double* prev = p->V.p;  // p_{k-1}(S) V
    for (int k = 1; k < degree; ++k) {
      const double sn = 1.0 / (2.0 * t0 - sigma);
      AM_TRY(sp::spmm(p, cur, prev, prev, 2.0 * sn / e, c, sigma * sn));
      std::swap(cur, prev);
      sigma = sn;
    }
    p->V.p = cur;
    p->Y.p = prev;
  }
  AM_TRY(sp::spmm(p, p->V.p, nullptr, p->SV.p, 1.0, 0.0, 0.0));
  AM_TRY(sp::gram(p, p->V.p, p->V.p, p->red.p));
  AM_TRY(sp::gram(p, p->V.p, p->SV.p, p->red.p + (size_t)p->b * p->b));
  const size_t bb = (size_t)p->b * p->b * 8;
  AM_CUDA(cudaMemcpyAsync(G, p->red.p, bb, cudaMemcpyDeviceToHost, st));
  AM_CUDA(cudaMemcpyAsync(H, p->red.p + (size_t)p->b * p->b, bb, cudaMemcpyDeviceToHost, st));
  AM_CUDA(cudaStreamSynchronize(st));
  return AM_OK;
}

extern "C" int am_spectral_plan_residuals(am_spectral_plan* p, const double* Q, const double* theta, int ncols,
                                          double* res, double* norms) {
  AM_CHECK(p && Q && theta && res && ncols >= 1 && ncols <= p->b,
           "am_spectral_plan_residuals: bad argument (need Q, theta, res and 1 <= ncols <= block)");
  cudaStream_t st = p->st.s;
  AM_TRY(sp::upload_q(p, Q, ncols));
  AM_TRY(p->theta.ensure((size_t)ncols));
  AM_CUDA(cudaMemcpyAsync(p->theta.p, theta, (size_t)ncols * 8, cudaMemcpyHostToDevice, st));
  const dim3 grid = sp::rowmul_grid(p, ncols);
  AM_TRY(p->part.ensure((size_t)grid.x * 2 * ncols));
  AM_LAUNCH(sp::rowmul_kernel<sp::kResidual>, grid, 256, 0, st, p->V.p, p->SV.p, p->N, p->b, p->ld, p->Qd.p, ncols,
            p->theta.p, nullptr, nullptr, nullptr, p->part.p);
  AM_LAUNCH(sp::reduce_parts_kernel, sp::flat_grid(2 * ncols), 256, 0, st, p->part.p, (int)grid.x, (int64_t)2 * ncols,
            p->red.p);
  std::vector<double> h((size_t)2 * ncols);
  AM_CUDA(cudaMemcpyAsync(h.data(), p->red.p, h.size() * 8, cudaMemcpyDeviceToHost, st));
  AM_CUDA(cudaStreamSynchronize(st));
  for (int c = 0; c < ncols; ++c) {
    const double u = std::sqrt(h[(size_t)ncols + c]);
    res[c] = u > 0.0 ? std::sqrt(h[(size_t)c]) / u : INFINITY;
    if (norms) norms[c] = u;
  }
  return AM_OK;
}

extern "C" int am_spectral_plan_embed(am_spectral_plan* p, const double* Q, int ncols, double* out) {
  AM_CHECK(p && Q && out && ncols >= 1 && ncols <= p->b,
           "am_spectral_plan_embed: bad argument (need Q, out and 1 <= ncols <= block)");
  cudaStream_t st = p->st.s;
  AM_TRY(sp::upload_q(p, Q, ncols));
  DevBuf<double> emb;
  AM_TRY(emb.alloc((size_t)p->N * ncols));
  AM_LAUNCH(sp::rowmul_kernel<sp::kEmbed>, sp::rowmul_grid(p, ncols), 256, 0, st, p->V.p, nullptr, p->N, p->b, p->ld,
            p->Qd.p, ncols, nullptr, p->dd.p, nullptr, emb.p, nullptr);
  AM_CUDA(cudaMemcpyAsync(out, emb.p, (size_t)p->N * ncols * 8, cudaMemcpyDeviceToHost, st));
  AM_CUDA(cudaStreamSynchronize(st));
  return AM_OK;
}

extern "C" void am_spectral_plan_free(am_spectral_plan* p) {
  if (p && p->st.s) cudaStreamSynchronize(p->st.s);
  delete p;
}
