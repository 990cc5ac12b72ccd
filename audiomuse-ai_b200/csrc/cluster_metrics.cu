// Clustering scores for the clustering task's fitness (tasks/clustering_helper.py:462-470: scikit-learn's
// silhouette_score, davies_bouldin_score and calinski_harabasz_score on the [N, d] matrix that was just clustered).
//
// The rows are first put in label order on the device (host counting sort -> permutation + per-label segment offsets,
// then a gather), so every cluster is one contiguous segment of rows.
//
// Silhouette (O(N^2 d), the hot path)
//   split_rows_kernel         sorted rows -> Xs bf16 [N, 2*dp] = [hi | lo] (split_bf16.cuh)
//   silhouette_tc_kernel      CTA (row tile of 128, column range): warpgroup 0 TMA-streams A_hi, A_lo [128 x 64] of the
//                             row tile and B_hi, B_lo [128 x 64] of one column block per 64-wide K chunk into a 3-stage
//                             mbarrier ring; warpgroups 1-2 (64 rows each) run
//                               D += A_hi.B_hi + A_lo.B_hi + A_hi.B_lo + A_lo.B_lo (wgmma m64n128k16, fp32 registers)
//                             A first launch over the diagonal blocks only stores xn_i = D_ii: the squared norms in
//                             the same arithmetic as every D_ij, so identical rows cancel exactly.  (k-means drops
//                             the lo.lo product; here it would leave d~^2 short by sum (lo_i - lo_j)^2 for EVERY pair,
//                             a bias that does not average out of the mean silhouette.)  The full launch
//                             then takes, from the registers, d_ij = sqrt(max(xn_i + xn_j - 2 D_ij, 0)) (0 on the diagonal)
//                             summed over each label segment the block spans (fp32 inside a block, <= 32 terms per
//                             thread and row), carried in float64 across blocks, merged over the 4 threads of a row
//                             and added to S[i, label] when the segment ends.  Only S f64[N, L] is written: the N x N
//                             distance matrix never exists in memory.
//   silhouette_finish_kernel  a = S[i, own] / (n_own - 1), b = min_{c != own} S[i, c] / n_c, s = (b - a) / max(a, b);
//                             0 for singleton clusters and for 0 / 0 (scikit-learn's nan_to_num); per-sample values
//                             go out in the caller's row order, their float64 sum to one accumulator.
//
// Davies-Bouldin and Calinski-Harabasz (O(N d), HBM bound), float64 accumulation:
//   seg_col_sum_kernel        per-label column sums -> centroids (centroid_kernel)
//   seg_dist_kernel           per-label sums of ||x - c|| and ||x - c||^2
//   host                      the L x L centroid step and scikit-learn's special cases.
#include "gemm_wgmma.cuh"
#include "host_call.cuh"
#include "split_bf16.cuh"
#include "tma_pipeline.cuh"

#include <algorithm>
#include <cmath>
#include <vector>

namespace am {
namespace cm {

using namespace ptx;
using pipe::kChunkK;
using pipe::kThreads;

constexpr int kTile = 128;   // rows of a CTA tile = columns of a column block
constexpr int kStages = 3;
constexpr int kOpTile = kTile * kChunkK * 2;  // one bf16 128 x 64 operand tile: 16 KiB
constexpr int kStageBytes = 4 * kOpTile;      // A_hi, A_lo, B_hi, B_lo
using Ring = pipe::Ring<kStages>;
constexpr size_t kSmem = Ring::smem_bytes(kStageBytes, kStages, 0);

// one warp per row: Xp[i] = X[perm[i]]
__global__ void __launch_bounds__(256)
gather_rows_kernel(const float* __restrict__ X, int64_t N, int d, const int32_t* __restrict__ perm,
                   float* __restrict__ Xp) {
  const int lane = threadIdx.x & 31;
  const int64_t warps = (int64_t)gridDim.x * (blockDim.x >> 5);
  for (int64_t row = (int64_t)blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5); row < N; row += warps) {
    const float* x = X + (int64_t)perm[row] * d;
    float* o = Xp + row * d;
    for (int i = lane; i < d; i += 32) o[i] = x[i];
  }
}

struct SilArgs {
  int64_t N;
  int dp, L;
  int col_blocks;        // ceil(N / 128)
  int blocks_per_split;  // column blocks per CTA (grid.y splits the column range)
  float* xn;             // [N] D_ii of the sorted rows: written by the diagonal pass, read by the full pass
  const int32_t* seg;    // [N] label of each sorted row
  const int32_t* off;    // [L + 1] segment offsets
  double* S;             // [N, L] sum of distances from sorted row i to the rows of label c (zeroed by the caller)
};

// kDiag: only the diagonal block of each row tile, writing xn[i] = D_ii (the squared norm in the same tensor-core
// arithmetic as every D_ij, so that d_ij is exactly 0 for identical rows); otherwise the column range of grid.y.
template <bool kDiag>
__global__ void __launch_bounds__(kThreads, 1)
silhouette_tc_kernel(const __grid_constant__ CUtensorMap map_x, const SilArgs a) {
  extern __shared__ __align__(1024) uint8_t smem_raw[];
  Ring ring(smem_raw, kStageBytes, kStages, 0);

  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int num_kb = a.dp / kChunkK;
  const int tile = blockIdx.x;
  const int b_begin = kDiag ? tile : blockIdx.y * a.blocks_per_split;
  const int b_end = kDiag ? tile + 1 : min(a.col_blocks, b_begin + a.blocks_per_split);  // never empty

  if (threadIdx.x == 0) {
    prefetch_tensormap(&map_x);
    ring.init();
  }
  __syncthreads();

  if (warp < 4) {
    regs_producer();
    if (warp == 0 && elect_one_sync()) {
      for (int b = b_begin; b < b_end; ++b) {
        for (int kb = 0; kb < num_kb; ++kb) {
          const Ring::Slot s = ring.acquire();
          tma_load_2d(s.smem, &map_x, s.bar, kb * kChunkK, tile * kTile);                    // A hi
          tma_load_2d(s.smem + kOpTile, &map_x, s.bar, a.dp + kb * kChunkK, tile * kTile);   // A lo
          tma_load_2d(s.smem + 2 * kOpTile, &map_x, s.bar, kb * kChunkK, b * kTile);         // B hi
          tma_load_2d(s.smem + 3 * kOpTile, &map_x, s.bar, a.dp + kb * kChunkK, b * kTile);  // B lo
        }
      }
    }
    return;
  }
  regs_consumer();
  // ===================== consumers: warpgroup g owns tile rows [64 g, 64 g + 64) =====================
  const int wg = (threadIdx.x >> 7) - 1;
  const int quad = lane & 3;
  const int64_t N = a.N;
  const int64_t row0 = (int64_t)tile * kTile + wg * 64 + ((threadIdx.x & 127) >> 5) * 16 + (lane >> 2);
  float xr[2] = {0.f, 0.f};
  if (!kDiag) {
#pragma unroll
    for (int h = 0; h < 2; ++h) xr[h] = row0 + 8 * h < N ? a.xn[row0 + 8 * h] : 0.f;
  }
  double run[2] = {0.0, 0.0};  // this thread's share of the current segment's sum, per row
  float acc[64];
#pragma unroll
  for (int i = 0; i < 64; ++i) acc[i] = 0.f;
  for (int b = b_begin; b < b_end; ++b) {
    for (int kb = 0; kb < num_kb; ++kb) {
      const uint32_t s = ring.wait();
      const uint32_t rows = (uint32_t)(wg * 64 * 128);
      pipe::mma_chunk_split<128, true>(acc, s + rows, s + kOpTile + rows, s + 2 * kOpTile, s + 3 * kOpTile, kb);
      ring.release();
    }
    const int64_t c0 = (int64_t)b * kTile;
    if constexpr (kDiag) {
#pragma unroll
      for (int j = 0; j < 16; ++j)
#pragma unroll
        for (int e = 0; e < 2; ++e)
#pragma unroll
          for (int h = 0; h < 2; ++h) {
            const int64_t col = c0 + 8 * j + 2 * quad + e;
            if (col == row0 + 8 * h && col < N) a.xn[col] = acc[4 * j + 2 * h + e];
          }
    } else {
      // ===================== fused epilogue: distances in place, then per-segment sums =====================
#pragma unroll
      for (int j = 0; j < 16; ++j)
#pragma unroll
        for (int e = 0; e < 2; ++e) {
          const int64_t col = c0 + 8 * j + 2 * quad + e;
          const float xc = col < N ? a.xn[col] : 0.f;
#pragma unroll
          for (int h = 0; h < 2; ++h) {
            const float v = sqrtf(fmaxf(fmaf(-2.0f, acc[4 * j + 2 * h + e], xr[h] + xc), 0.f));
            acc[4 * j + 2 * h + e] = col == row0 + 8 * h ? 0.f : v;
          }
        }
      // the block's columns are sorted by label: it spans the segments seg[c0] .. seg[cend - 1]
      const int64_t cend = min(c0 + kTile, N);
      const int s_last = __ldg(&a.seg[cend - 1]);
      for (int s = __ldg(&a.seg[c0]); s <= s_last; ++s) {
        const int64_t s_hi = __ldg(&a.off[s + 1]);
        const int lo = (int)(max((int64_t)__ldg(&a.off[s]), c0) - c0), hi = (int)(min(s_hi, cend) - c0);
        float part[2] = {0.f, 0.f};
#pragma unroll
        for (int j = 0; j < 16; ++j)
#pragma unroll
          for (int e = 0; e < 2; ++e) {
            const int c = 8 * j + 2 * quad + e;
            if (c >= lo && c < hi) {
              part[0] += acc[4 * j + e];
              part[1] += acc[4 * j + 2 + e];
            }
          }
        run[0] += (double)part[0];
        run[1] += (double)part[1];
        // flush when the segment ends in this block, or this CTA's column range ends inside it (another CTA adds the rest)
        if (s_hi <= cend || b == b_end - 1) {
#pragma unroll
          for (int h = 0; h < 2; ++h) {
            double t = run[h];
            t += __shfl_xor_sync(0xffffffffu, t, 1);
            t += __shfl_xor_sync(0xffffffffu, t, 2);
            const int64_t row = row0 + 8 * h;
            if (quad == 0 && row < N) atomicAdd(&a.S[row * a.L + s], t);
            run[h] = 0.0;
          }
        }
      }
    }
  }
}

// one warp per sorted row i: the silhouette of i from S; samples in the caller's order (perm), sum of s in *total
__global__ void __launch_bounds__(256)
silhouette_finish_kernel(const double* __restrict__ S, int64_t N, int L, const int32_t* __restrict__ seg,
                         const int32_t* __restrict__ off, const int32_t* __restrict__ perm, float* __restrict__ samples,
                         double* __restrict__ total) {
  __shared__ double s_part[8];
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  const int64_t warps = (int64_t)gridDim.x * 8;
  double local = 0.0;
  for (int64_t i = (int64_t)blockIdx.x * 8 + warp; i < N; i += warps) {
    const int own = seg[i];
    const double* row = S + i * L;
    double b = INFINITY;
    for (int c = lane; c < L; c += 32)
      if (c != own) b = fmin(b, row[c] / (double)(off[c + 1] - off[c]));
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) b = fmin(b, __shfl_xor_sync(0xffffffffu, b, o));
    if (lane == 0) {
      const int n_own = off[own + 1] - off[own];
      double s = 0.0;  // singleton cluster (0 / 0 in scikit-learn) -> 0
      if (n_own > 1) {
        const double a = row[own] / (double)(n_own - 1), m = fmax(a, b);
        s = m > 0.0 ? (b - a) / m : 0.0;  // a = b = 0 (duplicates across clusters): 0 / 0 -> 0
      }
      samples[perm[i]] = (float)s;
      local += s;
    }
  }
  if (lane == 0) s_part[warp] = local;
  __syncthreads();
  if (threadIdx.x == 0) {
    double t = 0.0;
    for (int w = 0; w < 8; ++w) t += s_part[w];
    atomicAdd(total, t);
  }
}

// per-label column sums of the sorted rows (float64): one thread per column walks a slab of rows (grid.y slabs) and
// flushes at every segment boundary
__global__ void seg_col_sum_kernel(const float* __restrict__ Xp, int64_t N, int d, const int32_t* __restrict__ seg,
                                   double* __restrict__ sums) {
  const int c = blockIdx.x * blockDim.x + threadIdx.x;
  if (c >= d) return;
  const int64_t rows = (N + gridDim.y - 1) / gridDim.y, r0 = (int64_t)blockIdx.y * rows, r1 = min(N, r0 + rows);
  if (r0 >= r1) return;
  int cur = seg[r0];
  double acc = 0.0;
  for (int64_t r = r0; r < r1; ++r) {
    const int s = seg[r];
    if (s != cur) {
      atomicAdd(&sums[(int64_t)cur * d + c], acc);
      acc = 0.0;
      cur = s;
    }
    acc += (double)Xp[r * d + c];
  }
  atomicAdd(&sums[(int64_t)cur * d + c], acc);
}

// sums -> centroids in place
__global__ void centroid_kernel(double* __restrict__ cent, int L, int d, const int32_t* __restrict__ off) {
  const int64_t e = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (e >= (int64_t)L * d) return;
  const int k = (int)(e / d);
  cent[e] /= (double)(off[k + 1] - off[k]);
}

// per-label sums of ||x - c|| and ||x - c||^2 (float64): a warp walks `chunk` consecutive sorted rows
__global__ void __launch_bounds__(256)
seg_dist_kernel(const float* __restrict__ Xp, int64_t N, int d, const int32_t* __restrict__ seg,
                const double* __restrict__ cent, int64_t chunk, double* __restrict__ dsum, double* __restrict__ dsq) {
  const int lane = threadIdx.x & 31;
  const int64_t w = (int64_t)blockIdx.x * 8 + (threadIdx.x >> 5);
  const int64_t r0 = w * chunk, r1 = min(N, r0 + chunk);
  if (r0 >= r1) return;
  int cur = seg[r0];
  double a1 = 0.0, a2 = 0.0;
  for (int64_t r = r0; r < r1; ++r) {
    const int s = seg[r];
    if (s != cur) {
      if (lane == 0) {
        atomicAdd(&dsum[cur], a1);
        atomicAdd(&dsq[cur], a2);
      }
      a1 = a2 = 0.0;
      cur = s;
    }
    const float* x = Xp + r * d;
    const double* c = cent + (int64_t)s * d;
    double q = 0.0;
    for (int i = lane; i < d; i += 32) {
      const double t = (double)x[i] - c[i];
      q = fma(t, t, q);
    }
    q = warp_sum(q);
    a1 += sqrt(q);
    a2 += q;
  }
  if (lane == 0) {
    atomicAdd(&dsum[cur], a1);
    atomicAdd(&dsq[cur], a2);
  }
}

}  // namespace cm
}  // namespace am

using namespace am;
using namespace am::cm;

extern "C" int am_cluster_scores(const float* X, int64_t N, int d, const int32_t* labels, int n_labels, int which,
                                 double* scores, float* samples) {
  AM_CHECK(X && labels && scores && N >= 2 && d >= 1 && d <= 8192 && which >= 1 && which <= 7,
           "am_cluster_scores: bad argument (need N >= 2, 1 <= d <= 8192, which in 1..7)");
  AM_CHECK(n_labels >= 2 && n_labels < N,
           "am_cluster_scores: Number of labels is %d. Valid values are 2 to n_samples - 1 (inclusive)", n_labels);
  // the permutation and the TMA row coordinates are int32; S = f64[N, L] is capped at 16 GiB
  AM_CHECK(N <= (int64_t)INT32_MAX - kTile, "am_cluster_scores: N = %lld rows exceeds the limit of 2^31 - 129",
           (long long)N);
  const bool sil = which & 1, dbch = (which & 6) != 0;
  AM_CHECK(!sil || N * (int64_t)n_labels <= ((int64_t)1 << 31),
           "am_cluster_scores: silhouette needs N * n_labels <= 2^31 (S is f64[N, n_labels]); got %lld x %d",
           (long long)N, n_labels);
  const int L = n_labels;
  // counting sort of the labels: perm lists the rows label by label, off[c] .. off[c + 1] is label c's segment
  std::vector<int32_t> off((size_t)L + 1, 0), perm((size_t)N), seg((size_t)N);
  for (int64_t i = 0; i < N; ++i) {
    const int32_t c = labels[i];
    AM_CHECK(c >= 0 && c < L, "am_cluster_scores: label %d of row %lld is outside [0, %d)", c, (long long)i, L);
    ++off[(size_t)c + 1];
  }
  for (int c = 0; c < L; ++c) {
    AM_CHECK(off[(size_t)c + 1] > 0, "am_cluster_scores: label %d has no rows (labels must be 0 .. n_labels - 1)", c);
    off[(size_t)c + 1] += off[(size_t)c];
  }
  {
    std::vector<int32_t> cursor(off.begin(), off.end() - 1);
    for (int64_t i = 0; i < N; ++i) perm[(size_t)cursor[(size_t)labels[i]]++] = (int32_t)i;
    for (int c = 0; c < L; ++c)
      std::fill(seg.begin() + off[(size_t)c], seg.begin() + off[(size_t)c + 1], c);
  }
  cudaStream_t st;
  AM_TRY(HostCall::thread_stream(&st));
  AM_CHECK(!sil || gemm::available(), "am_cluster_scores: the silhouette kernel needs an sm_90 device with TMA");
  HostCall call(st, 0, HostCall::Memory::Owned);
  float *dX, *dXp;
  int32_t *dPerm, *dSeg, *dOff;
  call.up(&dX, X, (size_t)N * d);
  call.up(&dPerm, perm.data(), (size_t)N);
  call.up(&dSeg, seg.data(), (size_t)N);
  call.up(&dOff, off.data(), (size_t)L + 1);
  call.device(&dXp, (size_t)N * d);
  AM_TRY(call.start());
  const int row_grid = (int)std::max<int64_t>(1, std::min<int64_t>((N + 7) / 8, (int64_t)sm_count() * 16));
  AM_LAUNCH(gather_rows_kernel, row_grid, 256, 0, st, dX, N, d, dPerm, dXp);

  if (sil) {
    const int dp = (int)round_up((size_t)d, 64);
    DevBuf<__nv_bfloat16> Xs;
    DevBuf<float> xn, dSamples;
    DevBuf<double> S, total;
    AM_TRY(Xs.alloc((size_t)N * 2 * dp));
    AM_TRY(xn.alloc((size_t)N));
    AM_TRY(dSamples.alloc((size_t)N));
    AM_TRY(S.alloc((size_t)N * L));
    AM_TRY(total.alloc(1));
    AM_CUDA(cudaMemsetAsync(S.p, 0, (size_t)N * L * 8, st));
    AM_CUDA(cudaMemsetAsync(total.p, 0, 8, st));
    AM_LAUNCH(split_rows_kernel, row_grid, 256, 0, st, dXp, N, d, dp, Xs.p, nullptr);
    CUtensorMap map;
    AM_TRY(gemm::encode_map_bf16(&map, Xs.p, 2 * dp, N, 2 * dp, kTile));
    SilArgs a{};
    a.N = N;
    a.dp = dp;
    a.L = L;
    a.col_blocks = (int)((N + kTile - 1) / kTile);
    const int tiles = a.col_blocks;
    // about four CTAs per SM in all, so that the last wave is a small share of the work
    int splits = (int)std::min<int64_t>(a.col_blocks, std::max<int64_t>(1, (4LL * sm_count() + tiles - 1) / tiles));
    a.blocks_per_split = (a.col_blocks + splits - 1) / splits;
    splits = (a.col_blocks + a.blocks_per_split - 1) / a.blocks_per_split;  // every split non-empty
    a.xn = xn.p;
    a.seg = dSeg;
    a.off = dOff;
    a.S = S.p;
    AM_TRY(allow_dynamic_smem<silhouette_tc_kernel<true>>(kSmem));
    AM_TRY(allow_dynamic_smem<silhouette_tc_kernel<false>>(kSmem));
    AM_LAUNCH(silhouette_tc_kernel<true>, dim3((unsigned)tiles, 1u), kThreads, kSmem, st, map, a);
    AM_LAUNCH(silhouette_tc_kernel<false>, dim3((unsigned)tiles, (unsigned)splits), kThreads, kSmem, st, map, a);
    AM_LAUNCH(silhouette_finish_kernel, row_grid, 256, 0, st, S.p, N, L, dSeg, dOff, dPerm, dSamples.p,
              total.p);
    double t = 0.0;
    AM_CUDA(cudaMemcpyAsync(&t, total.p, 8, cudaMemcpyDeviceToHost, st));
    if (samples) AM_CUDA(cudaMemcpyAsync(samples, dSamples.p, (size_t)N * 4, cudaMemcpyDeviceToHost, st));
    AM_CUDA(cudaStreamSynchronize(st));
    scores[0] = t / (double)N;
  }

  if (dbch) {
    DevBuf<double> cent, dsum, dsq;
    AM_TRY(cent.alloc((size_t)L * d));
    AM_TRY(dsum.alloc((size_t)L));
    AM_TRY(dsq.alloc((size_t)L));
    AM_CUDA(cudaMemsetAsync(cent.p, 0, (size_t)L * d * 8, st));
    AM_CUDA(cudaMemsetAsync(dsum.p, 0, (size_t)L * 8, st));
    AM_CUDA(cudaMemsetAsync(dsq.p, 0, (size_t)L * 8, st));
    const int slabs = (int)std::max<int64_t>(1, std::min<int64_t>(1024, N / 64));
    AM_LAUNCH(seg_col_sum_kernel, dim3((unsigned)ceil_div(d, 128), (unsigned)slabs), 128, 0, st, dXp, N, d,
              dSeg, cent.p);
    AM_LAUNCH(centroid_kernel, (unsigned)(((int64_t)L * d + 255) / 256), 256, 0, st, cent.p, L, d, dOff);
    const int64_t warps = (int64_t)sm_count() * 64;
    const int64_t chunk = std::max<int64_t>(1, (N + warps - 1) / warps);
    const int64_t used = (N + chunk - 1) / chunk;
    AM_LAUNCH(seg_dist_kernel, (unsigned)((used + 7) / 8), 256, 0, st, dXp, N, d, dSeg, cent.p, chunk, dsum.p,
              dsq.p);
    std::vector<double> hc((size_t)L * d), hs((size_t)L), hq((size_t)L);
    AM_CUDA(cudaMemcpyAsync(hc.data(), cent.p, (size_t)L * d * 8, cudaMemcpyDeviceToHost, st));
    AM_CUDA(cudaMemcpyAsync(hs.data(), dsum.p, (size_t)L * 8, cudaMemcpyDeviceToHost, st));
    AM_CUDA(cudaMemcpyAsync(hq.data(), dsq.p, (size_t)L * 8, cudaMemcpyDeviceToHost, st));
    AM_CUDA(cudaStreamSynchronize(st));
    if (which & 4) {  // sklearn.metrics.calinski_harabasz_score
      std::vector<double> mean((size_t)d, 0.0);
      for (int k = 0; k < L; ++k) {
        const double n = (double)(off[(size_t)k + 1] - off[(size_t)k]);
        for (int c = 0; c < d; ++c) mean[(size_t)c] += n * hc[(size_t)k * d + c];
      }
      for (int c = 0; c < d; ++c) mean[(size_t)c] /= (double)N;
      double extra = 0.0, intra = 0.0;
      for (int k = 0; k < L; ++k) {
        double e = 0.0;
        for (int c = 0; c < d; ++c) {
          const double t = hc[(size_t)k * d + c] - mean[(size_t)c];
          e += t * t;
        }
        extra += (double)(off[(size_t)k + 1] - off[(size_t)k]) * e;
        intra += hq[(size_t)k];
      }
      scores[2] = intra == 0.0 ? 1.0 : extra * (double)(N - L) / (intra * (double)(L - 1));
    }
    if (which & 2) {  // sklearn.metrics.davies_bouldin_score
      std::vector<double> s((size_t)L), cd((size_t)L * L);
      bool intra_zero = true, cent_zero = true;  // np.allclose(..., 0): every |value| <= 1e-8
      for (int k = 0; k < L; ++k) {
        s[(size_t)k] = hs[(size_t)k] / (double)(off[(size_t)k + 1] - off[(size_t)k]);
        intra_zero = intra_zero && std::fabs(s[(size_t)k]) <= 1e-8;
      }
      for (int k = 0; k < L; ++k)
        for (int m = 0; m < L; ++m) {
          double q = 0.0;
          for (int c = 0; c < d; ++c) {
            const double t = hc[(size_t)k * d + c] - hc[(size_t)m * d + c];
            q += t * t;
          }
          cd[(size_t)k * L + m] = std::sqrt(q);
          cent_zero = cent_zero && cd[(size_t)k * L + m] <= 1e-8;
        }
      if (intra_zero || cent_zero) {
        scores[1] = 0.0;
      } else {
        double acc = 0.0;
        for (int k = 0; k < L; ++k) {
          double best = -INFINITY;
          for (int m = 0; m < L; ++m) {
            const double dist = cd[(size_t)k * L + m];  // a distance of exactly 0 counts as infinite
            best = std::max(best, dist == 0.0 ? 0.0 : (s[(size_t)k] + s[(size_t)m]) / dist);
          }
          acc += best;
        }
        scores[1] = acc / (double)L;
      }
    }
  }
  return AM_OK;
}
