// K5 on the tensor cores: one Lloyd E-step + M-step partial sums for k <= 128 clusters (sm_90a).
//
// Replaces cuml.cluster.KMeans's assignment GEMM (tasks/clustering_gpu.py:100-123; SURVEY 2.4 K5).
//
//   split (once per data set)   X f32 [N, d] -> Xs bf16 [N, 2*dp] = [hi | lo]  (x = hi + lo + O(2^-18 x)),
//                               xn[N] = ||x||^2;  dp = d rounded up to 64 (zero padded).
//   per iteration
//     centre prep               C f32 [k, d] -> Cs bf16 [2*kp, dp] = rows [0, kp): hi, [kp, 2kp): lo;  cn[j] = ||c_j||^2
//                               (+inf for the padded rows j >= k), cmax = max ||c_j||.
//     assign_tc_kernel          persistent warp-specialised CTAs of three warpgroups, a tile = 128 points:
//                                 warpgroup 0     TMA: per 64-wide K chunk the A_hi, A_lo [128 x 64] and B [2kp x 64]
//                                                 tiles (SWIZZLE_128B) into a 3-stage mbarrier ring;
//                                 warpgroups 1-2  64 points each: wgmma.mma_async m64n{kp}k16 into fp32 registers,
//                                                 D += A_hi.B_hi + A_lo.B_hi + A_hi.B_lo   -- an fp32-class dot product
//                                                 (dropped term lo.lo <= 2^-18 |x||c|); then the FUSED ARGMIN
//                                                 EPILOGUE from the registers: v_j = cn_j - 2 D_j, running best /
//                                                 second best per thread, merged over the 4 threads of a row; writes
//                                                 label and distance, nothing else -- the [N, k] score matrix never
//                                                 exists in memory.
//                               A point whose runner-up is within the proven error band of the best
//                               (2^-11 ||x|| max||c||) is appended to a recheck list.
//     recheck_kernel            exact fp32 argmin (exact_argmin, shared with kmeans.cu's assign_kernel) for the
//                               listed points only: labels equal the exact-arithmetic labels for EVERY point.
//     accumulate_sorted_kernel  M-step partial sums: a CTA counting-sorts the labels of its 2048-point slab in
//                               shared memory, then each warp walks one label segment: rows are read once, as whole
//                               coalesced rows, summed in registers, the exact ||x - c||^2 taken on the way (inertia),
//                               and flushed with one red.global.add per (cluster, column) per slab -- no
//                               shared-memory atomics on the data path.
//
// HBM traffic per iteration: Xs once (assign) + X once (accumulate) = 2 * N * d * 4 bytes.
#include "kmeans_tc.cuh"

#include "gemm_wgmma.cuh"
#include "split_bf16.cuh"
#include "tma_pipeline.cuh"

#include <algorithm>
#include <cmath>

namespace am {
namespace kmtc {

using namespace ptx;
using pipe::kChunkK;
using pipe::kThreads;

constexpr int kTileM = 128;
constexpr int kATile = kTileM * kChunkK * 2;  // 16 KiB
constexpr int kSlabMax = 4096;                // most points one accumulate CTA sorts at a time

// ---------------------------------------------------------------- split passes
// the rows: split_rows_kernel (split_bf16.cuh, shared with the silhouette kernel)
// one warp per centre row (incl. the padded rows): Cs, cn, and the max norm (as int bits of a non-negative float)
__global__ void __launch_bounds__(256)
split_centers_kernel(const float* __restrict__ C, int k, int d, int kp, int dp, __nv_bfloat16* __restrict__ Cs,
                     float* __restrict__ cn, int* __restrict__ cmax2_bits) {
  const int lane = threadIdx.x & 31;
  const int j = blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5);
  if (j >= kp) return;
  float acc = 0.f;
  for (int i = lane; i < dp; i += 32) {
    const float v = (j < k && i < d) ? C[(int64_t)j * d + i] : 0.f;
    acc = fmaf(v, v, acc);
    const __nv_bfloat16 hi = __float2bfloat16_rn(v);
    Cs[(int64_t)j * dp + i] = hi;
    Cs[(int64_t)(kp + j) * dp + i] = __float2bfloat16_rn(v - __bfloat162float(hi));
  }
  acc = warp_sum(acc);
  if (lane == 0) {
    cn[j] = j < k ? acc : INFINITY;
    if (j < k) atomicMax(cmax2_bits, __float_as_int(acc));
  }
}

// ---------------------------------------------------------------- assignment GEMM with the fused argmin epilogue
struct AssignArgs {
  int64_t N;
  int kp, dp, k;
  int tiles;
  const float* cn;        // [kp]
  const float* xn;        // [N]
  const int* cmax2_bits;  // max ||c||^2
  int32_t* labels;        // [N]
  float* dist;            // [N] or NULL: max(best + xn, 0)
  int* n_recheck;         // counter
  int32_t* recheck;       // [N] row list
  float band_scale;       // 2^-11
};

constexpr int kStages = 3;
using Ring = pipe::Ring<kStages>;

// per stage: A_hi, A_lo [128 x 64], then B [2 KP x 64] = centres hi rows, lo rows
template <int KP>
constexpr int stage_bytes() { return 2 * kATile + 2 * KP * kChunkK * 2; }

// (best, index, runner-up) of two disjoint candidate sets; equal scores keep the lower centre index
__device__ __forceinline__ void merge_best(float& best, int& best_j, float& second, float b2, int j2, float s2) {
  if (b2 < best || (b2 == best && j2 < best_j)) {
    second = fminf(s2, best);
    best = b2;
    best_j = j2;
  } else {
    second = fminf(second, b2);
  }
}

template <int KP>
__global__ void __launch_bounds__(kThreads, 1)
assign_tc_kernel(const __grid_constant__ CUtensorMap map_x, const __grid_constant__ CUtensorMap map_c, const AssignArgs args) {
  extern __shared__ __align__(1024) uint8_t smem_raw[];
  Ring ring(smem_raw, stage_bytes<KP>(), kStages, KP * sizeof(float));
  float* s_cn = reinterpret_cast<float*>(ring.extra());  // [KP]

  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int num_kb = args.dp / kChunkK;

  if (threadIdx.x == 0) {
    prefetch_tensormap(&map_x);
    prefetch_tensormap(&map_c);
    ring.init();
  }
  for (int i = threadIdx.x; i < KP; i += kThreads) s_cn[i] = args.cn[i];
  __syncthreads();

  if (warp < 4) {
    regs_producer();
    if (warp == 0 && elect_one_sync()) {
      for (int tile = blockIdx.x; tile < args.tiles; tile += gridDim.x) {
        for (int kb = 0; kb < num_kb; ++kb) {
          const Ring::Slot s = ring.acquire();
          tma_load_2d(s.smem, &map_x, s.bar, kb * kChunkK, tile * kTileM);                    // hi
          tma_load_2d(s.smem + kATile, &map_x, s.bar, args.dp + kb * kChunkK, tile * kTileM);  // lo
          tma_load_2d(s.smem + 2 * kATile, &map_c, s.bar, kb * kChunkK, 0);                    // centres hi | lo
        }
      }
    }
    return;
  }
  regs_consumer();
  // ===================== consumers: warpgroup g owns tile rows [64 g, 64 g + 64) =====================
  const int wg = (threadIdx.x >> 7) - 1;
  const int quad = lane & 3;
  const float cmax = sqrtf(__int_as_float(*args.cmax2_bits));
  float acc[KP / 2];
#pragma unroll
  for (int i = 0; i < KP / 2; ++i) acc[i] = 0.f;
  for (int tile = blockIdx.x; tile < args.tiles; tile += gridDim.x) {
    for (int kb = 0; kb < num_kb; ++kb) {
      const uint32_t s = ring.wait();
      const uint32_t rows = (uint32_t)(wg * 64 * 128);
      pipe::mma_chunk_split<KP, false>(acc, s + rows, s + kATile + rows, s + 2 * kATile,
                                       s + 2 * kATile + (uint32_t)KP * 128u, kb);
      ring.release();
    }
    // ===================== fused argmin epilogue: a quad of threads = two points =====================
    const int64_t row0 = (int64_t)tile * kTileM + wg * 64 + ((threadIdx.x & 127) >> 5) * 16 + (lane >> 2);
#pragma unroll
    for (int h = 0; h < 2; ++h) {
      const int64_t row = row0 + 8 * h;
      float best = INFINITY, second = INFINITY;
      int best_j = 0;  // a label in range even for a row whose scores are all NaN / +inf
#pragma unroll
      for (int j = 0; j < KP / 8; ++j) {  // this thread's columns in increasing order
#pragma unroll
        for (int e = 0; e < 2; ++e) {
          const int c = 8 * j + 2 * quad + e;
          const float s = fmaf(-2.0f, acc[4 * j + 2 * h + e], s_cn[c]);  // +inf for padded centres
          if (s < best) {
            second = best;
            best = s;
            best_j = c;
          } else if (s < second) {
            second = s;
          }
        }
      }
#pragma unroll
      for (int o = 1; o <= 2; o <<= 1) {
        const float b2 = __shfl_xor_sync(0xffffffffu, best, o);
        const int j2 = __shfl_xor_sync(0xffffffffu, best_j, o);
        const float s2 = __shfl_xor_sync(0xffffffffu, second, o);
        merge_best(best, best_j, second, b2, j2, s2);
      }
      if (quad == 0 && row < args.N) {
        const float xn = __ldg(&args.xn[row]);
        args.labels[row] = best_j;
        if (args.dist) args.dist[row] = fmaxf(best + xn, 0.f);
        // |x.c~ - x.c| <= 2^-13 ||x|| max||c||, so |v~ - v| <= 2^-12 ||x|| max||c|| per centre (split-bf16 residuals +
        // fp32 accumulation over dp terms; measured on H100 up to 0.21 x 2^-12 at d = 4096 on non-negative data).
        // A runner-up within twice that of the winner (the band, 2^-11) may be the exact winner: the exact kernel
        // decides.  cn's own rounding is not in the band: it is the same fp32 value the CUDA-core step uses.
        const float band = args.band_scale * sqrtf(xn) * cmax;
        if (second - best <= band) {
          const int slot = atomicAdd(args.n_recheck, 1);
          args.recheck[slot] = (int32_t)row;
        }
      }
    }
  }
}

// exact fp32 argmin for the listed rows (exact_argmin, kmeans_tc.cuh, as assign_kernel decides).  One CTA per row,
// the centres dealt round-robin to its 8 warps (a single warp walking all k centres took ~0.3 ms per row, and a
// kernel is as slow as its slowest row); each warp keeps four dot products in flight, centres j0 + 8 u (u < 4).
__global__ void __launch_bounds__(256)
recheck_kernel(const float* __restrict__ X, int d, const float* __restrict__ C, const float* __restrict__ cn, int k,
               const int* __restrict__ n_recheck, const int32_t* __restrict__ recheck, int32_t* __restrict__ labels,
               float* __restrict__ dist) {
  __shared__ float s_best[8];
  __shared__ int s_idx[8];
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  const int n = *n_recheck;
  for (int q = blockIdx.x; q < n; q += gridDim.x) {
    const int64_t row = recheck[q];
    const float* x = X + row * d;
    float xn = 0.f;
    for (int i = lane; i < d; i += 32) xn = fmaf(x[i], x[i], xn);
    xn = warp_sum(xn);
    float best = INFINITY;
    int best_j = 0x7fffffff;
    for (int j0 = warp; j0 < k; j0 += 32) exact_argmin<4, 8>(x, d, C, cn, k, lane, j0, best, best_j);
    if (lane == 0) {
      s_best[warp] = best;
      s_idx[warp] = best_j;
    }
    __syncthreads();
    if (threadIdx.x == 0) {
      float b = s_best[0];
      int bj = s_idx[0];
      for (int w = 1; w < 8; ++w)
        if (s_best[w] < b || (s_best[w] == b && s_idx[w] < bj)) {
          b = s_best[w];
          bj = s_idx[w];
        }
      labels[row] = bj;
      if (dist) dist[row] = fmaxf(b + xn, 0.0f);
    }
    __syncthreads();
  }
}

// ---------------------------------------------------------------- M-step partial sums
// sums[j, :] += sum of the rows labelled j; counts[j] += their number; inertia += sum ||x - c_label||^2 (exact, fp32
// per row, float64 across rows).  kMaxChunks 128-column float4 chunks per lane cover d <= 512 in registers.
template <int kVec>
__global__ void __launch_bounds__(256)
accumulate_sorted_kernel(const float* __restrict__ X, int64_t N, int d, const int32_t* __restrict__ labels, int k,
                         const float* __restrict__ C, int slab, float* __restrict__ sums, float* __restrict__ counts,
                         double* __restrict__ inertia) {
  extern __shared__ int s_mem[];
  int* s_hist = s_mem;            // [k + 1] start offsets after the scan
  int* s_cursor = s_hist + k + 1;  // [k]
  int* s_order = s_cursor + k;    // [slab] rows of the slab grouped by label
  __shared__ double s_inertia[8];
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  double local = 0.0;
  // the grid is sized to ONE resident wave (a second, partial wave doubled the kernel's time): every CTA takes the same
  // number of slabs
  for (int64_t p0 = (int64_t)blockIdx.x * slab; p0 < N; p0 += (int64_t)gridDim.x * slab) {
    const int np = (int)min((int64_t)slab, N - p0);
    __syncthreads();
    for (int i = threadIdx.x; i <= k; i += blockDim.x) s_hist[i] = 0;
    __syncthreads();
    for (int i = threadIdx.x; i < np; i += blockDim.x) atomicAdd(&s_hist[labels[p0 + i] + 1], 1);
    __syncthreads();
    if (warp == 0) {  // inclusive scan of the k + 1 bins
      int carry = 0;
      for (int base = 0; base <= k; base += 32) {
        const int idx = base + lane;
        int v = idx <= k ? s_hist[idx] : 0;
#pragma unroll
        for (int o = 1; o < 32; o <<= 1) {
          const int t = __shfl_up_sync(0xffffffffu, v, o);
          if (lane >= o) v += t;
        }
        v += carry;
        if (idx <= k) s_hist[idx] = v;
        carry = __shfl_sync(0xffffffffu, v, 31);
      }
    }
    __syncthreads();
    for (int i = threadIdx.x; i < k; i += blockDim.x) s_cursor[i] = s_hist[i];
    __syncthreads();
    for (int i = threadIdx.x; i < np; i += blockDim.x) {
      const int slot = atomicAdd(&s_cursor[labels[p0 + i]], 1);
      s_order[slot] = i;
    }
    __syncthreads();
    constexpr int kMaxChunks = 4;  // 4 x 32 lanes x kVec columns per pass (512 columns with float4 loads)
    for (int col0 = 0; col0 < d; col0 += kMaxChunks * 32 * kVec) {
      for (int j = warp; j < k; j += 8) {
        const int s0 = s_hist[j], s1 = s_hist[j + 1];
        if (s0 == s1) continue;
        float acc[kMaxChunks][kVec], cj[kMaxChunks][kVec];
#pragma unroll
        for (int q = 0; q < kMaxChunks; ++q)
#pragma unroll
          for (int e = 0; e < kVec; ++e) {
            const int col = col0 + (q * 32 + lane) * kVec + e;
            acc[q][e] = 0.f;
            cj[q][e] = col < d ? __ldg(&C[(int64_t)j * d + col]) : 0.f;
          }
        float dsum = 0.f;
        auto consume = [&](const float (&v)[kMaxChunks][kVec]) {
          float dloc = 0.f;
#pragma unroll
          for (int q = 0; q < kMaxChunks; ++q)
#pragma unroll
            for (int e = 0; e < kVec; ++e) {
              acc[q][e] += v[q][e];
              const float a = v[q][e] - cj[q][e];
              dloc = fmaf(a, a, dloc);
            }
          dsum += dloc;
        };
        auto load = [&](int s, float (&v)[kMaxChunks][kVec]) {
          const float* x = X + (p0 + s_order[s]) * d;
#pragma unroll
          for (int q = 0; q < kMaxChunks; ++q) {
            const int col = col0 + (q * 32 + lane) * kVec;
            if constexpr (kVec == 4) {
              float4 t = make_float4(0.f, 0.f, 0.f, 0.f);
              if (col < d) t = __ldg(reinterpret_cast<const float4*>(x + col));
              v[q][0] = t.x; v[q][1] = t.y; v[q][2] = t.z; v[q][3] = t.w;
            } else {
              v[q][0] = col < d ? __ldg(x + col) : 0.f;
            }
          }
        };
        // padded columns load 0 and their centre entry is 0: they add nothing to sums or distances
        int s = s0;
        for (; s + 1 < s1; s += 2) {  // two rows in flight per warp
          float va[kMaxChunks][kVec], vb[kMaxChunks][kVec];
          load(s, va);
          load(s + 1, vb);
          consume(va);
          consume(vb);
        }
        if (s < s1) {
          float va[kMaxChunks][kVec];
          load(s, va);
          consume(va);
        }
#pragma unroll
        for (int q = 0; q < kMaxChunks; ++q)
#pragma unroll
          for (int e = 0; e < kVec; ++e) {
            const int col = col0 + (q * 32 + lane) * kVec + e;
            if (col < d) atomicAdd(&sums[(int64_t)j * d + col], acc[q][e]);
          }
        dsum = warp_sum(dsum);
        if (lane == 0) {
          local += (double)dsum;
          if (col0 == 0 && counts) atomicAdd(&counts[j], (float)(s1 - s0));
        }
      }
    }
  }
  if (lane == 0) s_inertia[warp] = local;
  __syncthreads();
  if (threadIdx.x == 0 && inertia) {
    double t = 0.0;
    for (int w = 0; w < 8; ++w) t += s_inertia[w];
    atomicAdd(inertia, t);
  }
}

// ---------------------------------------------------------------- host
int Plan::create(cudaStream_t st) {
  dp = (int)round_up((size_t)d, 64);
  kp = (int)round_up((size_t)k, 16);
  AM_TRY(Xs.alloc((size_t)N * 2 * dp));
  AM_TRY(xn.alloc((size_t)N));
  AM_TRY(Cs.alloc((size_t)2 * kp * dp));
  AM_TRY(cn.alloc((size_t)kp));
  AM_TRY(scal.alloc(2));  // [0] max ||c||^2 bits, [1] recheck counter
  AM_TRY(recheck.alloc((size_t)N));
  const int grid = (int)std::max<int64_t>(1, std::min<int64_t>((N + 7) / 8, (int64_t)sm_count() * 16));
  AM_LAUNCH(split_rows_kernel, grid, 256, 0, st, X, N, d, dp, Xs.p, xn.p);
  AM_TRY(gemm::encode_map_bf16(map_x, Xs.p, 2 * dp, N, 2 * dp, kTileM));
  AM_TRY(gemm::encode_map_bf16(map_c, Cs.p, dp, 2 * kp, dp, 2 * kp));
  return AM_OK;
}

int Plan::launch_accumulate(float* sums, float* counts, double* inertia_dev, const float* C_dev, const int32_t* labels,
                            cudaStream_t st) {
  // one resident wave: 3 CTAs per SM (register limited), each takes ceil(N / grid) points in slabs of <= kSlabMax
  const int64_t ctas = (int64_t)sm_count() * 3;
  int slab = (int)std::min<int64_t>(kSlabMax, std::max<int64_t>(256, (N + ctas - 1) / ctas));
  const int64_t n_slabs = (N + slab - 1) / slab;
  const unsigned grid = (unsigned)std::min<int64_t>(n_slabs, ctas);
  const size_t smem = (size_t)(2 * k + 1 + slab) * sizeof(int);
  if (d % 4 == 0) {
    AM_LAUNCH(accumulate_sorted_kernel<4>, grid, 256, smem, st, X, N, d, labels, k, C_dev, slab, sums, counts, inertia_dev);
  } else {
    AM_LAUNCH(accumulate_sorted_kernel<1>, grid, 256, smem, st, X, N, d, labels, k, C_dev, slab, sums, counts, inertia_dev);
  }
  return AM_OK;
}

template <int KP>
static int launch_assign(const Plan& p, const AssignArgs& a, cudaStream_t st) {
  const size_t smem = Ring::smem_bytes(stage_bytes<KP>(), kStages, KP * sizeof(float));
  AM_TRY(allow_dynamic_smem<assign_tc_kernel<KP>>(smem));
  const int grid = std::min(a.tiles, sm_count());
  AM_LAUNCH(assign_tc_kernel<KP>, grid, kThreads, smem, st, *reinterpret_cast<const CUtensorMap*>(p.map_x),
            *reinterpret_cast<const CUtensorMap*>(p.map_c), a);
  return AM_OK;
}

int Plan::step(const float* C_dev, int32_t* labels, float* sums, float* counts, double* inertia_dev, float* dist,
               cudaStream_t st) {
  AM_CUDA(cudaMemsetAsync(scal.p, 0, 2 * sizeof(int), st));
  AM_LAUNCH(split_centers_kernel, ceil_div(kp, 8), 256, 0, st, C_dev, k, d, kp, dp, Cs.p, cn.p, scal.p);
  AssignArgs a{};
  a.N = N;
  a.kp = kp;
  a.dp = dp;
  a.k = k;
  a.tiles = (int)((N + kTileM - 1) / kTileM);
  a.cn = cn.p;
  a.xn = xn.p;
  a.cmax2_bits = scal.p;
  a.labels = labels;
  a.dist = dist;
  a.n_recheck = scal.p + 1;
  a.recheck = recheck.p;
  a.band_scale = 1.0f / 2048.0f;
  switch (kp) {
    case 16: AM_TRY(launch_assign<16>(*this, a, st)); break;
    case 32: AM_TRY(launch_assign<32>(*this, a, st)); break;
    case 48: AM_TRY(launch_assign<48>(*this, a, st)); break;
    case 64: AM_TRY(launch_assign<64>(*this, a, st)); break;
    case 80: AM_TRY(launch_assign<80>(*this, a, st)); break;
    case 96: AM_TRY(launch_assign<96>(*this, a, st)); break;
    case 112: AM_TRY(launch_assign<112>(*this, a, st)); break;
    case 128: AM_TRY(launch_assign<128>(*this, a, st)); break;
    default:
      set_error("kmeans: no assignment kernel for %d centres", kp);
      return AM_ERR_INVALID;
  }
  AM_LAUNCH(recheck_kernel, sm_count() * 8, 256, 0, st, X, d, C_dev, cn.p, k, scal.p + 1, recheck.p, labels, dist);
  if (sums) {
    AM_CUDA(cudaMemsetAsync(sums, 0, (size_t)k * d * 4, st));
    if (counts) AM_CUDA(cudaMemsetAsync(counts, 0, (size_t)k * 4, st));
    if (inertia_dev) AM_CUDA(cudaMemsetAsync(inertia_dev, 0, 8, st));
    AM_TRY(launch_accumulate(sums, counts, inertia_dev, C_dev, labels, st));
  } else if (inertia_dev) {  // final E-step: inertia only (sums go to scratch-free path: counts ignored)
    AM_CUDA(cudaMemsetAsync(inertia_dev, 0, 8, st));
    AM_TRY(scratch_sums.ensure((size_t)k * d));
    AM_CUDA(cudaMemsetAsync(scratch_sums.p, 0, (size_t)k * d * 4, st));
    AM_TRY(launch_accumulate(scratch_sums.p, nullptr, inertia_dev, C_dev, labels, st));
  }
  return AM_OK;
}

}  // namespace kmtc
}  // namespace am
