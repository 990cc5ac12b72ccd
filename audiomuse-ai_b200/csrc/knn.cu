// K4: exact brute-force k-NN index (sm_90a).  Replaces the voyager.Index object
// (tasks/voyager_manager.py:183,1397,1447,1580,1681; tasks/clap_text_search.py:173,263,493).
//
// Exactness by construction ("filter with a proven bound, then re-rank in float64"):
//   1. approximate scores s~[q, j] for every stored row, with |s~ - s| <= eps
//      (fp32 SIMT pass: eps from the fp32 dot-product error bound;
//       bf16 tensor-core pass (gemm_wgmma.cuh): eps from the bf16 rounding residual norms);
//   2. per query: T = k-th largest s~ (radix select).  Every exact top-k row satisfies
//      s~ >= T - 2*eps, so {j : s~_j >= T - 2 eps} is a superset of the answer;
//   3. the superset (k + a handful) is re-scored with float64 accumulation from the stored
//      float32 rows and sorted by (distance asc, id asc); the first k are returned.
//   If the superset overflows the on-chip candidate buffer (k > ~4000, e.g. the reference's
//   k = len(index) max-distance scan, voyager_manager.py:1681) a full float64 pass + global
//   bitonic sort answers instead.
#include "host_call.cuh"
#include "knn.cuh"

#include <algorithm>
#include <cmath>
#include <functional>
#include <memory>

#include "gemm_wgmma.cuh"

namespace am {

constexpr int kCandCap = 4096;       // on-chip candidate capacity per query
constexpr int kCmChunk = 32;         // the GEMM epilogue also writes the maximum of every 32 consecutive scores
constexpr int kCmMaxK = 512;         // chunk-max selection: k-th largest chunk maximum as the threshold
constexpr int kCmChunkCap = 2048;    // flagged chunks a query may have on chip
constexpr int kSelThreads = 1024;

// ---------------------------------------------------------------- build kernels
// one warp per row: squared norm in float64; optional in-place unit normalisation
__global__ void row_prepare_kernel(float* __restrict__ X, int64_t N, int d, int normalize,
                                   float* __restrict__ norm2_out) {
  const int64_t row = (int64_t)blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5);
  const int lane = threadIdx.x & 31;
  if (row >= N) return;
  float* x = X + row * d;
  double acc = 0.0;
  for (int i = lane; i < d; i += 32) {
    const double v = (double)x[i];
    acc += v * v;
  }
  acc = warp_sum(acc);
  double nrm = sqrt(acc);
  if (normalize) {
    if (nrm == 0.0) nrm = 1.0;
    for (int i = lane; i < d; i += 32) x[i] = (float)((double)x[i] / nrm);
    __syncwarp();
    double a2 = 0.0;
    for (int i = lane; i < d; i += 32) {
      const double v = (double)x[i];
      a2 += v * v;
    }
    acc = warp_sum(a2);
  }
  if (lane == 0 && norm2_out) norm2_out[row] = (float)acc;
}

// bf16 copy (zero-padded to dpad) + residual norm ||x - bf16(x)||
__global__ void row_to_bf16_kernel(const float* __restrict__ X, int64_t N, int d, int dpad,
                                   __nv_bfloat16* __restrict__ Xb, float* __restrict__ res) {
  const int64_t row = (int64_t)blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5);
  const int lane = threadIdx.x & 31;
  if (row >= N) return;
  const float* x = X + row * d;
  __nv_bfloat16* y = Xb + row * dpad;
  float acc = 0.0f;
  for (int i = lane; i < dpad; i += 32) {
    const float v = i < d ? x[i] : 0.0f;
    const __nv_bfloat16 h = __float2bfloat16_rn(v);
    y[i] = h;
    const float r = v - __bfloat162float(h);
    acc = fmaf(r, r, acc);
  }
  acc = warp_sum(acc);
  if (lane == 0) res[row] = sqrtf(acc) * 1.0001f;
}

// ---------------------------------------------------------------- fp32 scoring pass
// score = q.x (cosine / ip) or 2 q.x - ||x||^2 (euclidean; larger = closer).
// One warp per stored row, kQT queries per pass kept in shared memory.
constexpr int kQT = 8;
__global__ void __launch_bounds__(256)
score_f32_kernel(const float* __restrict__ X, const float* __restrict__ xnorm2, int64_t N, int d,
                 const float* __restrict__ Q, int nq, int q0, int metric, float* __restrict__ S, int64_t ldS) {
  extern __shared__ __align__(16) float s_q[];  // [kQT][d]
  const int nqt = min(kQT, nq - q0);
  for (int i = threadIdx.x; i < nqt * d; i += blockDim.x) s_q[i] = Q[(int64_t)q0 * d + i];
  __syncthreads();
  const int lane = threadIdx.x & 31;
  const int warps = blockDim.x >> 5;
  const int64_t stride = (int64_t)gridDim.x * warps;
  if ((d & 3) == 0) {
    // 16-byte loads, two rows in flight per warp: the single-query pass is a pure HBM stream (N d 4 bytes) and
    // scalar loads of one row at a time left it at 2.5 TB/s
    const int d4 = d >> 2;
    const float4* s_q4 = reinterpret_cast<const float4*>(s_q);
    for (int64_t row = (int64_t)blockIdx.x * warps + (threadIdx.x >> 5); row < N; row += 2 * stride) {
      const int64_t row_b = row + stride;
      const bool has_b = row_b < N;
      const float4* xa = reinterpret_cast<const float4*>(X + row * d);
      const float4* xb = reinterpret_cast<const float4*>(X + (has_b ? row_b : row) * d);
      float acc_a[kQT], acc_b[kQT];
#pragma unroll
      for (int t = 0; t < kQT; ++t) acc_a[t] = acc_b[t] = 0.0f;
      for (int i = lane; i < d4; i += 32) {
        const float4 va = __ldg(&xa[i]), vb = __ldg(&xb[i]);
#pragma unroll
        for (int t = 0; t < kQT; ++t) {
          if (t < nqt) {
            const float4 qv = s_q4[t * d4 + i];
            acc_a[t] = fmaf(va.w, qv.w, fmaf(va.z, qv.z, fmaf(va.y, qv.y, fmaf(va.x, qv.x, acc_a[t]))));
            acc_b[t] = fmaf(vb.w, qv.w, fmaf(vb.z, qv.z, fmaf(vb.y, qv.y, fmaf(vb.x, qv.x, acc_b[t]))));
          }
        }
      }
#pragma unroll
      for (int t = 0; t < kQT; ++t) {
        acc_a[t] = warp_sum(acc_a[t]);
        acc_b[t] = warp_sum(acc_b[t]);
      }
      if (lane == 0) {
        const float xna = metric == kMetricL2 ? xnorm2[row] : 0.0f;
        const float xnb = (metric == kMetricL2 && has_b) ? xnorm2[row_b] : 0.0f;
        for (int t = 0; t < nqt; ++t) {
          S[(int64_t)(q0 + t) * ldS + row] = metric == kMetricL2 ? 2.0f * acc_a[t] - xna : acc_a[t];
          if (has_b) S[(int64_t)(q0 + t) * ldS + row_b] = metric == kMetricL2 ? 2.0f * acc_b[t] - xnb : acc_b[t];
        }
      }
    }
    return;
  }
  for (int64_t row = (int64_t)blockIdx.x * warps + (threadIdx.x >> 5); row < N; row += stride) {
    const float* x = X + row * d;
    float acc[kQT];
#pragma unroll
    for (int t = 0; t < kQT; ++t) acc[t] = 0.0f;
    for (int i = lane; i < d; i += 32) {
      const float v = __ldg(&x[i]);
#pragma unroll
      for (int t = 0; t < kQT; ++t)
        if (t < nqt) acc[t] = fmaf(v, s_q[t * d + i], acc[t]);
    }
#pragma unroll
    for (int t = 0; t < kQT; ++t) acc[t] = warp_sum(acc[t]);
    if (lane == 0) {
      const float xn = metric == kMetricL2 ? xnorm2[row] : 0.0f;
      for (int t = 0; t < nqt; ++t)
        S[(int64_t)(q0 + t) * ldS + row] = metric == kMetricL2 ? 2.0f * acc[t] - xn : acc[t];
    }
  }
}

// ---------------------------------------------------------------- bf16 scoring pass for a handful of queries
// The single-query (radius walk, "similar to this track") case is one pass over the library and nothing else, so it
// should read the 2-byte copy, not the 4-byte one: same approximate scores as the tensor-core filter (bf16 x bf16 products
// are exact in fp32, fp32 accumulation), same proven bound, half the HBM bytes -- and the per-32 maxima the selection
// kernel steers by come out of the same pass instead of a second kernel.  One warp per chunk of 32 rows; a lane holds
// 8 kSegs elements of every query in registers; the row sums are reduced with butterflies and lane r keeps row r.
template <int kQ, int kSegs>
__global__ void __launch_bounds__(256)
score_bf16_small_kernel(const __nv_bfloat16* __restrict__ Xb, const float* __restrict__ xnorm2, int64_t N, int d, int dpad,
                        const float* __restrict__ Q, int nq, int q0, int metric, float* __restrict__ S, int64_t ldS,
                        float* __restrict__ CM, int64_t ldCM, int64_t n_chunks, double* __restrict__ qnorm,
                        float* __restrict__ qres) {
  const int lane = threadIdx.x & 31;
  const int64_t gw = (int64_t)blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5);
  const int64_t total = (int64_t)gridDim.x * (blockDim.x >> 5);
  // query preparation (what query_prepare_kernel does, redone by every warp -- d is a few hundred -- so that the single
  // query costs one launch less): float64 norm, cosine: normalise, round to bf16, norm of the rounding residual
  float qv[kQ][kSegs][8];
#pragma unroll
  for (int t = 0; t < kQ; ++t) {
    const bool have = q0 + t < nq;
    const float* x = Q + (int64_t)(have ? q0 + t : q0) * d;
    float raw[kSegs][8];
    double acc = 0.0;
#pragma unroll
    for (int sg = 0; sg < kSegs; ++sg)
#pragma unroll
      for (int e = 0; e < 8; ++e) {
        const int i = sg * 256 + lane * 8 + e;
        raw[sg][e] = (have && i < d) ? __ldg(x + i) : 0.f;
        acc += (double)raw[sg][e] * (double)raw[sg][e];
      }
    acc = warp_sum(acc);
    const double nrm = sqrt(acc);
    const double scale = (metric == kMetricCos) ? (nrm == 0.0 ? 1.0 : 1.0 / nrm) : 1.0;
    float racc = 0.f;
#pragma unroll
    for (int sg = 0; sg < kSegs; ++sg)
#pragma unroll
      for (int e = 0; e < 8; ++e) {
        const float v = (float)((double)raw[sg][e] * scale);
        const __nv_bfloat16 h = __float2bfloat16_rn(v);
        qv[t][sg][e] = __bfloat162float(h);
        const float r = v - qv[t][sg][e];
        racc = fmaf(r, r, racc);
      }
    racc = warp_sum(racc);
    if (gw == 0 && lane == 0 && have) {
      qnorm[q0 + t] = (metric == kMetricCos) ? (nrm == 0.0 ? 1.0 : nrm) : nrm;
      qres[q0 + t] = sqrtf(racc) * 1.0001f;
    }
  }
  for (int64_t chunk = gw; chunk < n_chunks; chunk += total) {
    const int64_t j0 = chunk * 32;
    float mine[kQ];
#pragma unroll
    for (int t = 0; t < kQ; ++t) mine[t] = 0.f;
#pragma unroll 4
    for (int r = 0; r < 32; ++r) {
      const int64_t row = j0 + r < N ? j0 + r : N - 1;   // rows beyond N: any valid row, masked below
      float acc[kQ];
#pragma unroll
      for (int t = 0; t < kQ; ++t) acc[t] = 0.f;
#pragma unroll
      for (int sg = 0; sg < kSegs; ++sg) {
        const uint4 raw = __ldg(reinterpret_cast<const uint4*>(Xb + row * dpad + sg * 256 + lane * 8));
        const __nv_bfloat162* h = reinterpret_cast<const __nv_bfloat162*>(&raw);
#pragma unroll
        for (int e = 0; e < 4; ++e) {
          const float2 f = __bfloat1622float2(h[e]);
#pragma unroll
          for (int t = 0; t < kQ; ++t) acc[t] = fmaf(f.y, qv[t][sg][2 * e + 1], fmaf(f.x, qv[t][sg][2 * e], acc[t]));
        }
      }
#pragma unroll
      for (int t = 0; t < kQ; ++t) {
        const float sum = warp_sum(acc[t]);
        if (lane == r) mine[t] = sum;
      }
    }
    const int64_t row = j0 + lane;
    const bool ok = row < N;
    const float xn = (metric == kMetricL2 && ok) ? xnorm2[row] : 0.f;
#pragma unroll
    for (int t = 0; t < kQ; ++t) {
      if (q0 + t < nq) {   // warp-uniform
        const float sc = metric == kMetricL2 ? 2.0f * mine[t] - xn : mine[t];
        if (ok) S[(int64_t)(q0 + t) * ldS + row] = sc;
        float m = ok ? sc : -INFINITY;
#pragma unroll
        for (int o = 16; o > 0; o >>= 1) m = fmaxf(m, __shfl_xor_sync(0xffffffffu, m, o));
        if (lane == 0) CM[(int64_t)(q0 + t) * ldCM + chunk] = m;
      }
    }
  }
}

// ---------------------------------------------------------------- query preparation
// per query: float64 norm; normalised fp32 copy (cosine) for the scoring pass; bf16 copy +
// residual norm for the tensor-core filter.
__global__ void query_prepare_kernel(const float* __restrict__ Q, int nq, int d, int dpad, int metric,
                                     float* __restrict__ Qs, double* __restrict__ qnorm,
                                     __nv_bfloat16* __restrict__ Qb, float* __restrict__ qres) {
  const int q = blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5);
  const int lane = threadIdx.x & 31;
  if (q >= nq) return;
  const float* x = Q + (int64_t)q * d;
  double acc = 0.0;
  for (int i = lane; i < d; i += 32) acc += (double)x[i] * (double)x[i];
  acc = warp_sum(acc);
  double nrm = sqrt(acc);
  const double scale = (metric == kMetricCos) ? (nrm == 0.0 ? 1.0 : 1.0 / nrm) : 1.0;
  if (lane == 0) qnorm[q] = (metric == kMetricCos) ? (nrm == 0.0 ? 1.0 : nrm) : nrm;
  float racc = 0.0f;
  for (int i = lane; i < dpad; i += 32) {
    const float v = i < d ? (float)((double)x[i] * scale) : 0.0f;
    if (i < d) Qs[(int64_t)q * d + i] = v;
    if (Qb) {
      const __nv_bfloat16 h = __float2bfloat16_rn(v);
      Qb[(int64_t)q * dpad + i] = h;
      const float r = v - __bfloat162float(h);
      racc = fmaf(r, r, racc);
    }
  }
  if (Qb) {
    racc = warp_sum(racc);
    if (lane == 0) qres[q] = sqrtf(racc) * 1.0001f;
  }
}

// ---------------------------------------------------------------- select + exact re-rank
__device__ __forceinline__ unsigned f2key(float f) {  // monotone: larger float -> larger key
  const unsigned u = __float_as_uint(f);
  return (u & 0x80000000u) ? ~u : (u | 0x80000000u);
}
__device__ __forceinline__ float key2f(unsigned k) {
  const unsigned u = (k & 0x80000000u) ? (k & 0x7fffffffu) : ~k;
  return __uint_as_float(u);
}

// count `bin` (when `valid`) into this warp's private histogram.  Two leader-election rounds fold the
// lanes that share the most common bins into one atomic each; what is left goes in individually.
__device__ __forceinline__ void hist_add(unsigned* hist, unsigned bin, bool valid, int lane) {
  unsigned active = __ballot_sync(0xffffffffu, valid);
#pragma unroll
  for (int round = 0; round < 2; ++round) {
    if (active == 0u) return;  // warp-uniform
    const int leader = __ffs(active) - 1;
    const unsigned lb = __shfl_sync(0xffffffffu, bin, leader);
    const unsigned same = __ballot_sync(0xffffffffu, valid && bin == lb) & active;
    if (lane == leader) atomicAdd(&hist[lb], (unsigned)__popc(same));
    active &= ~same;
  }
  if ((active >> lane) & 1u) atomicAdd(&hist[bin], 1u);
}

struct SelectParams {
  const float* S;        // [nq, ldS] approximate scores (larger = closer)
  int64_t ldS;
  int64_t N;
  int d;
  int metric;
  int k;
  const float* X;        // [N, d]
  const float* xnorm2;   // [N] (euclidean)
  const float* Q;        // [nq, d] raw queries
  const double* qnorm;   // [nq]
  float eps_abs;         // fp32-accumulation part of the score error bound (per unit of ||q|| when eps_scales_with_q)
  int eps_scales_with_q; // inner product / euclidean: multiply eps_abs by this query's norm
  const float* qres;     // per-query bf16 residual norm (NULL on the fp32 pass)
  const float* xres;     // per-row bf16 residual norm (NULL on the fp32 pass)
  float xres_max;
  float xnorm_max;
  int64_t* ids;          // [nq, k]
  float* dist;           // [nq, k]
  int* overflow;         // [nq] set to 1 if the candidate superset did not fit
  // chunk-max selection (select_cm_kernel): the GEMM epilogue also wrote the maximum of every 32 scores
  const float* CM;       // [nq, ldCM]
  int64_t ldCM;
  int64_t n_chunks;      // ceil(N / 32)
};

// float64 distance of query q to stored row `row`, one warp.  d % 4 == 0: 16-byte loads, all of a lane's loads issued
// before the first FMA (the re-rank of ~k candidates is latency bound: a query's survivors are read exactly once)
__device__ __forceinline__ double exact_distance(const SelectParams& p, int q, int64_t row, int lane) {
  const float* x = p.X + row * p.d;
  const float* qv = p.Q + (int64_t)q * p.d;
  double acc = 0.0, xn = 0.0;
  const bool need_xn = p.metric == kMetricL2;
  if ((p.d & 3) == 0 && ((reinterpret_cast<uintptr_t>(qv) | reinterpret_cast<uintptr_t>(x)) & 15) == 0) {
    const float4* x4 = reinterpret_cast<const float4*>(x);
    const float4* q4 = reinterpret_cast<const float4*>(qv);
    const int n4 = p.d >> 2;
    for (int i0 = lane; i0 < n4; i0 += 128) {  // up to 4 vector pairs in flight per lane
      float4 a[4], b[4];
#pragma unroll
      for (int u = 0; u < 4; ++u) {
        const int i = i0 + 32 * u;
        a[u] = i < n4 ? __ldg(&x4[i]) : make_float4(0.f, 0.f, 0.f, 0.f);
        b[u] = i < n4 ? __ldg(&q4[i]) : make_float4(0.f, 0.f, 0.f, 0.f);
      }
#pragma unroll
      for (int u = 0; u < 4; ++u) {
        acc = fma((double)a[u].x, (double)b[u].x, acc);
        acc = fma((double)a[u].y, (double)b[u].y, acc);
        acc = fma((double)a[u].z, (double)b[u].z, acc);
        acc = fma((double)a[u].w, (double)b[u].w, acc);
        if (need_xn) {
          xn = fma((double)a[u].x, (double)a[u].x, xn);
          xn = fma((double)a[u].y, (double)a[u].y, xn);
          xn = fma((double)a[u].z, (double)a[u].z, xn);
          xn = fma((double)a[u].w, (double)a[u].w, xn);
        }
      }
    }
  } else {
    for (int i = lane; i < p.d; i += 32) {
      const double v = (double)__ldg(&x[i]);
      acc = fma(v, (double)__ldg(&qv[i]), acc);
      if (need_xn) xn = fma(v, v, xn);
    }
  }
  acc = warp_sum(acc);
  if (p.metric == kMetricCos) return 1.0 - acc / p.qnorm[q];
  if (p.metric == kMetricIp) return 1.0 - acc;
  // squared L2 = ||q||^2 - 2 q.x + ||x||^2, all in float64
  xn = warp_sum(xn);
  const double qn = p.qnorm[q];
  return fmax(qn * qn - 2.0 * acc + xn, 0.0);
}

struct SelShared {
  unsigned (*hist)[256];  // [kSelThreads / 32][256] per-warp private histograms
  unsigned* tot;          // [256]
  unsigned* prefix;
  unsigned* remaining;
};

// radix select of the kk-th largest of `cnt` floats at `src` (a global row read through __ldg, or shared memory).
// Per-warp private histograms: scores of one query cluster in a handful of exponent bins, so a single shared
// histogram serialises on a few addresses; privatised, a bin is only contended by the 32 lanes of one warp and
// the 32 partial histograms are summed once per pass.  All kSelThreads threads of the CTA must call it.
__device__ float radix_kth(const SelShared& sh, const float* src, int64_t cnt, unsigned kk, bool global_src) {
  const int tid = threadIdx.x;
  unsigned* my_hist = sh.hist[tid >> 5];
  if (tid == 0) {
    *sh.prefix = 0;
    *sh.remaining = kk;
  }
  unsigned mask = 0;
  for (int shift = 24; shift >= 0; shift -= 8) {
    for (int i = tid; i < (kSelThreads / 32) * 256; i += kSelThreads) (&sh.hist[0][0])[i] = 0;
    __syncthreads();
    const unsigned prefix = *sh.prefix;
    // 8 scores per thread per iteration (two 16-byte loads in flight): the row is latency bound otherwise
    const int lane = tid & 31;
    const int64_t n8 = (cnt + 7) >> 3;  // rows are padded to a multiple of 4 floats and 16-byte aligned
    for (int64_t base = 0; base < n8; base += kSelThreads) {
      const int64_t v = base + tid;
      float4 f0 = make_float4(0.f, 0.f, 0.f, 0.f), f1 = f0;
      const bool in0 = v < n8 && (v * 8) < cnt, in1 = v < n8 && (v * 8 + 4) < cnt;
      if (global_src) {
        if (in0) f0 = __ldg(reinterpret_cast<const float4*>(src) + 2 * v);
        if (in1) f1 = __ldg(reinterpret_cast<const float4*>(src) + 2 * v + 1);
      } else {
        if (in0) f0 = reinterpret_cast<const float4*>(src)[2 * v];
        if (in1) f1 = reinterpret_cast<const float4*>(src)[2 * v + 1];
      }
      const float fv[8] = {f0.x, f0.y, f0.z, f0.w, f1.x, f1.y, f1.z, f1.w};
#pragma unroll
      for (int e = 0; e < 8; ++e) {
        const unsigned key = f2key(fv[e]);
        const bool ok = (v < n8) && (v * 8 + e < cnt) && ((key & mask) == prefix);
        hist_add(my_hist, (key >> shift) & 255u, ok, lane);
      }
    }
    __syncthreads();
    if (tid < 256) {
      unsigned t = 0;
#pragma unroll 8
      for (int w = 0; w < kSelThreads / 32; ++w) t += sh.hist[w][tid];
      sh.tot[tid] = t;
    }
    __syncthreads();
    if (tid == 0) {
      unsigned rem = *sh.remaining;
      int b = 255;
      for (; b > 0; --b) {
        if (sh.tot[b] >= rem) break;
        rem -= sh.tot[b];
      }
      *sh.prefix = prefix | ((unsigned)b << shift);
      *sh.remaining = rem;
    }
    mask |= 255u << shift;
    __syncthreads();
  }
  return key2f(*sh.prefix);
}

// bound on |s~ - s| for query q (see the header of this file)
__device__ __forceinline__ float score_eps(const SelectParams& p, int q) {
  // the dot-product rounding error is proportional to ||q|| ||x||: using the query's OWN norm keeps T - 2 eps a proven
  // bound when a query is far larger than the stored rows (ADVICE r1: the bound used to assume ||q|| <= 2 max||x||)
  float eps = p.eps_abs * (p.eps_scales_with_q ? fmaxf((float)p.qnorm[q], 1e-30f) : 1.0f);
  if (p.qres) {
    // |q.x - qb.xb| <= ||q-qb|| ||x|| + ||qb|| ||x-xb||  (Cauchy-Schwarz), plus fp32 accumulation
    const float qr = p.qres[q];
    const float qn = (p.metric == kMetricCos) ? 1.0f : (float)p.qnorm[q];
    eps += qr * p.xnorm_max + (qn + qr) * p.xres_max;
    if (p.metric == kMetricL2) eps *= 2.0f;
  }
  return eps;
}

// one compare-exchange of a bitonic network sorting by (distance asc, id asc): the pair (lo, hi) is put in ascending
// order when `up`, in descending order otherwise
template <class I>
__device__ __forceinline__ void bitonic_exchange(double* dist, int* ids, I lo, I hi, bool up) {
  const double dl = dist[lo], dh = dist[hi];
  const int il = ids[lo], ih = ids[hi];
  const bool gt = (dl > dh) || (dl == dh && il > ih);
  if (gt == up) {
    dist[lo] = dh;
    dist[hi] = dl;
    ids[lo] = ih;
    ids[hi] = il;
  }
}

// exact float64 distances of the `count` candidate rows in c_id (one warp per candidate), bitonic sort by
// (distance asc, id asc), first k written out.  All threads of the CTA; c_id / c_dist hold kCandCap entries.
__device__ void rerank_sort_emit(const SelectParams& p, int q, unsigned count, double* c_dist, int* c_id) {
  const int tid = threadIdx.x;
  const int lane = tid & 31, warp = tid >> 5;
  for (unsigned c = warp; c < count; c += kSelThreads / 32) {
    const double dd = exact_distance(p, q, c_id[c], lane);
    if (lane == 0) c_dist[c] = dd;
  }
  unsigned n2 = 1;
  while (n2 < count) n2 <<= 1;
  for (unsigned c = count + tid; c < n2; c += kSelThreads) {
    c_dist[c] = INFINITY;
    c_id[c] = 0x7fffffff;
  }
  __syncthreads();
  for (unsigned size = 2; size <= n2; size <<= 1) {
    for (unsigned stride = size >> 1; stride > 0; stride >>= 1) {
      for (unsigned t = tid; t < n2 / 2; t += kSelThreads) {
        const unsigned lo = 2 * t - (t & (stride - 1));
        bitonic_exchange(c_dist, c_id, lo, lo + stride, (lo & size) == 0);
      }
      __syncthreads();
    }
  }
  for (int i = tid; i < p.k; i += kSelThreads) {
    p.ids[(int64_t)q * p.k + i] = (int64_t)c_id[i];
    p.dist[(int64_t)q * p.k + i] = (float)c_dist[i];
  }
  if (tid == 0) p.overflow[q] = 0;
}

__global__ void __launch_bounds__(kSelThreads, 2) select_rerank_kernel(SelectParams p) {
  __shared__ unsigned s_hist[kSelThreads / 32][256];
  __shared__ unsigned s_tot[256];
  __shared__ unsigned s_prefix, s_remaining, s_count;
  extern __shared__ __align__(16) unsigned char s_dyn[];
  double* c_dist = reinterpret_cast<double*>(s_dyn);                  // [kCandCap]
  int* c_id = reinterpret_cast<int*>(c_dist + kCandCap);              // [kCandCap]
  const SelShared sh{s_hist, s_tot, &s_prefix, &s_remaining};

  const int q = blockIdx.x;
  const int tid = threadIdx.x;
  const float* S = p.S + (int64_t)q * p.ldS;
  const int64_t N = p.N;

  // ---- a lower bound T of the k-th largest score.  k <= kSelThreads / 2: every thread takes the maximum of its
  // (interleaved) share of the row in ONE light pass; the k-th largest of those kSelThreads maxima is the k-th
  // largest of a subset of the row, hence <= the row's k-th largest -- and in practice within a few ranks of
  // it, so the candidate superset below stays ~k + tens.  (Exactness only needs T <= true k-th: the superset
  // {s~ >= T - 2 eps} then contains every exact top-k row.)  Larger k: exact radix select over the whole row
  // (four histogram passes -- what every query paid before; 2.2 ms per 4096 queries of a 100 k library).
  float kth;
  if (p.k <= kSelThreads / 2) {  // beyond that the bound loosens: k = 1000 of 1024 maxima admits ~4 k candidates
    float m = -INFINITY;
    const int64_t n8 = (N + 7) >> 3;
    for (int64_t v = tid; v < n8; v += kSelThreads) {
      float4 f0 = make_float4(-INFINITY, -INFINITY, -INFINITY, -INFINITY), f1 = f0;
      if (v * 8 < N) f0 = __ldg(reinterpret_cast<const float4*>(S) + 2 * v);
      if (v * 8 + 4 < N) f1 = __ldg(reinterpret_cast<const float4*>(S) + 2 * v + 1);
      const float fv[8] = {f0.x, f0.y, f0.z, f0.w, f1.x, f1.y, f1.z, f1.w};
#pragma unroll
      for (int e = 0; e < 8; ++e)
        if (v * 8 + e < N) m = fmaxf(m, fv[e]);
    }
    float* s_max = reinterpret_cast<float*>(s_dyn);  // [kSelThreads]; the candidate buffers are not live yet
    s_max[tid] = m;
    __syncthreads();
    kth = radix_kth(sh, s_max, kSelThreads, (unsigned)p.k, false);
  } else {
    kth = radix_kth(sh, S, N, (unsigned)p.k, true);
  }

  // ---- candidate superset: s~ >= kth - 2*eps   (eps: bound on |s~ - s|)
  const float thr = kth - 2.0f * score_eps(p, q) - 1e-30f;
  if (tid == 0) s_count = 0;
  __syncthreads();
  {
    const int64_t n4 = (N + 3) >> 2;
    for (int64_t v = tid; v < n4; v += kSelThreads) {
      const float4 f = __ldg(reinterpret_cast<const float4*>(S) + v);
      const float fv[4] = {f.x, f.y, f.z, f.w};
#pragma unroll
      for (int e = 0; e < 4; ++e) {
        const int64_t i = v * 4 + e;
        if (i < N && fv[e] >= thr) {
          const unsigned slot = atomicAdd(&s_count, 1u);
          if (slot < (unsigned)kCandCap) c_id[slot] = (int)i;
        }
      }
    }
  }
  __syncthreads();
  const unsigned count = s_count;
  if (count > (unsigned)kCandCap) {
    if (tid == 0) p.overflow[q] = 1;
    return;
  }
  rerank_sort_emit(p, q, count, c_dist, c_id);
}

// per-32 maxima of score rows written by the fp32 scoring pass (the tensor-core GEMM writes them in its epilogue):
// one warp per (query, chunk), a coalesced 128-byte read
__global__ void __launch_bounds__(256)
chunk_max_rows_kernel(const float* __restrict__ S, int64_t ldS, int64_t N, int nq, int64_t n_chunks, float* __restrict__ CM,
                      int64_t ldCM) {
  const int lane = threadIdx.x & 31;
  const int64_t total = (int64_t)nq * n_chunks;
  for (int64_t w = (int64_t)blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5); w < total; w += (int64_t)gridDim.x * (blockDim.x >> 5)) {
    const int64_t q = w / n_chunks, c = w - q * n_chunks;
    const int64_t col = c * 32 + lane;
    float v = col < N ? __ldg(&S[q * ldS + col]) : -INFINITY;
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) v = fmaxf(v, __shfl_xor_sync(0xffffffffu, v, o));
    if (lane == 0) CM[q * ldCM + c] = v;
  }
}

// ---- chunk-max selection (k <= kCmMaxK).  The GEMM epilogue wrote, beside the
// scores, the maximum of every 32 consecutive ones (CM: 1/32 of the bytes).  Per query:
//   T   = k-th largest chunk maximum -- the k-th largest of a SUBSET of the scores, hence a lower bound of the true
//         k-th largest, and tight (the top k scores sit in ~k different chunks);
//   only chunks whose maximum >= T - 2 eps can hold answers (k + a few): their 32 scores are read back from S and
//   filtered with the same proven bound; the survivors go through the float64 re-rank + sort.
// Each query thus reads N / 32 maxima + ~k x 128 bytes of scores instead of streaming its 4 N-byte row twice
// (select_rerank_kernel): the row of scores is written by the GEMM but almost never read.
// The kernel is written for latency (a query's work is tiny): six block-wide phases, no histogram passes --
//   thread maxima of the chunk maxima -> k-th largest of those 1024 values by rank counting (still the k-th largest of
//   a subset of the scores: a valid lower bound) -> flagged chunks (re-read by the few threads that own one) -> one warp
//   per flagged chunk reads its 32 scores -> one warp per survivor computes the float64 distance -> rank-counting sort.
__global__ void __launch_bounds__(kSelThreads, 2) select_cm_kernel(SelectParams p) {
  __shared__ float s_max[kSelThreads];
  __shared__ float s_thr;
  __shared__ unsigned s_count, s_chunks;
  extern __shared__ __align__(16) unsigned char s_dyn[];
  double* c_dist = reinterpret_cast<double*>(s_dyn);      // [kCandCap]
  int* c_id = reinterpret_cast<int*>(c_dist + kCandCap);  // [kCandCap]
  int* c_chunk = reinterpret_cast<int*>(c_dist);          // [kCmChunkCap] flagged chunks (dead before c_dist is written)
  const int q = blockIdx.x;
  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  const float* CM = p.CM + (int64_t)q * p.ldCM;
  const float* S = p.S + (int64_t)q * p.ldS;
  float m = -INFINITY;
  for (int64_t i = tid; i < p.n_chunks; i += kSelThreads) m = fmaxf(m, __ldg(&CM[i]));
  s_max[tid] = m;
  if (tid == 0) {
    s_count = 0;
    s_chunks = 0;
  }
  __syncthreads();
  // k-th largest of G group maxima by rank counting (G^2 comparisons: G = 256 when that leaves enough groups beside
  // the k winners, else all 1024 thread maxima); ties by index, rank k - 1 <=> k-th largest
  const int G = p.k <= 128 ? 256 : kSelThreads;
  if (G == 256) {
    float g4 = -INFINITY;
    if (tid < 256) {
      const float4 o = reinterpret_cast<const float4*>(s_max)[tid];
      g4 = fmaxf(fmaxf(o.x, o.y), fmaxf(o.z, o.w));
    }
    __syncthreads();
    if (tid < 256) s_max[tid] = g4;
    __syncthreads();
  }
  if (tid < G) {
    const float mm = s_max[tid];
    int rank = 0;
    const float4* s4 = reinterpret_cast<const float4*>(s_max);
    for (int j = 0; j < G / 4; ++j) {
      const float4 o = s4[j];
      rank += (o.x > mm || (o.x == mm && 4 * j < tid)) + (o.y > mm || (o.y == mm && 4 * j + 1 < tid)) +
              (o.z > mm || (o.z == mm && 4 * j + 2 < tid)) + (o.w > mm || (o.w == mm && 4 * j + 3 < tid));
    }
    if (rank == p.k - 1) s_thr = mm - 2.0f * score_eps(p, q) - 1e-30f;
  }
  __syncthreads();
  const float thr = s_thr;
  if (m >= thr) {  // only threads whose own maximum reaches the threshold re-read their share (L1 / L2 hits)
    for (int64_t i = tid; i < p.n_chunks; i += kSelThreads) {
      if (__ldg(&CM[i]) >= thr) {
        const unsigned slot = atomicAdd(&s_chunks, 1u);
        if (slot < (unsigned)kCmChunkCap) c_chunk[slot] = (int)i;
      }
    }
  }
  __syncthreads();
  const unsigned n_flag = s_chunks;
  if (n_flag > (unsigned)kCmChunkCap) {
    if (tid == 0) p.overflow[q] = 1;
    return;
  }
  // one warp per flagged chunk: lane = column inside the chunk (one coalesced 128-byte read of S)
  for (unsigned w = warp; w < n_flag; w += kSelThreads / 32) {
    const int64_t col = (int64_t)c_chunk[w] * kCmChunk + lane;
    if (col < p.N && __ldg(&S[col]) >= thr) {
      const unsigned slot = atomicAdd(&s_count, 1u);
      if (slot < (unsigned)kCandCap) c_id[slot] = (int)col;
    }
  }
  __syncthreads();
  const unsigned count = s_count;
  if (count > (unsigned)kCandCap || count < (unsigned)p.k) {  // (count < k cannot happen; guarded)
    if (tid == 0) p.overflow[q] = 1;
    return;
  }
  __syncthreads();  // c_chunk (aliasing c_dist) is dead from here
  if (count > (unsigned)kSelThreads) {
    rerank_sort_emit(p, q, count, c_dist, c_id);  // many survivors (duplicates, huge k): bitonic sort
    return;
  }
  for (unsigned c = warp; c < count; c += kSelThreads / 32) {
    const double dd = exact_distance(p, q, c_id[c], lane);
    if (lane == 0) c_dist[c] = dd;
  }
  __syncthreads();
  if (tid < (int)count) {  // rank-counting sort by (distance asc, id asc): one pass, no further barriers
    const double dm = c_dist[tid];
    const int im = c_id[tid];
    int rank = 0;
    for (unsigned j = 0; j < count; ++j) {
      const double dj = c_dist[j];
      rank += (dj < dm || (dj == dm && c_id[j] < im)) ? 1 : 0;
    }
    if (rank < p.k) {
      p.ids[(int64_t)q * p.k + rank] = (int64_t)im;
      p.dist[(int64_t)q * p.k + rank] = (float)dm;
    }
  }
  if (tid == 0) p.overflow[q] = 0;
}

// ---------------------------------------------------------------- full-sort fallback (large k)
__global__ void exact_all_kernel(SelectParams p, int q, int64_t npad, double* __restrict__ dist,
                                 int* __restrict__ ids) {
  const int64_t row = (int64_t)blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5);
  const int lane = threadIdx.x & 31;
  if (row >= npad) return;
  double dd = INFINITY;
  if (row < p.N) dd = exact_distance(p, q, row, lane);
  if (lane == 0) {
    dist[row] = dd;
    ids[row] = row < p.N ? (int)row : 0x7fffffff;
  }
}

__global__ void bitonic_step_kernel(double* __restrict__ dist, int* __restrict__ ids, int64_t npad,
                                    unsigned size, unsigned stride) {
  const int64_t t = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (t >= npad / 2) return;
  const int64_t lo = 2 * t - (t & (int64_t)(stride - 1));
  bitonic_exchange(dist, ids, lo, lo + (int64_t)stride, (lo & size) == 0);
}

__global__ void emit_topk_kernel(const double* __restrict__ dist, const int* __restrict__ ids, int k,
                                 int64_t* __restrict__ out_ids, float* __restrict__ out_dist) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i < k) {
    out_ids[i] = ids[i];
    out_dist[i] = (float)dist[i];
  }
}

static int full_sort_query(const SelectParams& p, int q, cudaStream_t st) {
  int64_t npad = 1;
  while (npad < p.N) npad <<= 1;
  DevBuf<double> dist;
  DevBuf<int> ids;
  AM_TRY(dist.alloc(npad));
  AM_TRY(ids.alloc(npad));
  AM_LAUNCH(exact_all_kernel, (unsigned)((npad + 7) / 8), 256, 0, st, p, q, npad, dist.p, ids.p);
  const unsigned blocks = (unsigned)((npad / 2 + 255) / 256);
  for (unsigned size = 2; size <= npad; size <<= 1)
    for (unsigned stride = size >> 1; stride > 0; stride >>= 1)
      AM_LAUNCH(bitonic_step_kernel, std::max(1u, blocks), 256, 0, st, dist.p, ids.p, npad, size, stride);
  AM_LAUNCH(emit_topk_kernel, ceil_div(p.k, 256), 256, 0, st, dist.p, ids.p, p.k,
            p.ids + (int64_t)q * p.k, p.dist + (int64_t)q * p.k);
  AM_CUDA(cudaStreamSynchronize(st));
  return AM_OK;
}

// ---------------------------------------------------------------- farthest stored row
// get_max_distance_for_id (voyager_manager.py:1660-1702) walks query(k = N) -- (float64 distance asc, row asc), each
// distance returned as float32 -- and keeps the first strict maximum of the float32 distances, skipping the target.
// Among the rows at the float32 maximum that is the smallest float64 distance, then the smallest row.  One pass computes
// every distance with exact_distance on the query the query path prepares, so each is the value query() returns; each
// warp keeps its best row, each block reduces its warps', and one block reduces the blocks'.  A NaN distance never wins
// (dist > max is false), as in the reference's loop.
constexpr int kFarThreads = 256;

struct FarBest {
  float f;    // the float32 distance query() returns
  double dd;  // the float64 distance it orders by
  int64_t row;  // -1: none
};

__device__ __forceinline__ bool far_better(const FarBest& a, const FarBest& b) {
  if (a.row < 0) return false;
  if (b.row < 0) return true;
  return a.f > b.f || (a.f == b.f && (a.dd < b.dd || (a.dd == b.dd && a.row < b.row)));
}

// the block's best of `cand` (one per thread), written by thread 0 to *out
__device__ __forceinline__ void far_block_reduce(FarBest cand, FarBest* out) {
  __shared__ FarBest s_best[kFarThreads / 32];
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  for (int o = 16; o > 0; o >>= 1) {
    FarBest other;
    other.f = __shfl_down_sync(0xffffffffu, cand.f, o);
    other.dd = __shfl_down_sync(0xffffffffu, cand.dd, o);
    other.row = __shfl_down_sync(0xffffffffu, cand.row, o);
    if (lane + o < 32 && far_better(other, cand)) cand = other;
  }
  if (lane == 0) s_best[warp] = cand;
  __syncthreads();
  if (threadIdx.x == 0) {
    FarBest best = s_best[0];
    for (int w = 1; w < kFarThreads / 32; ++w)
      if (far_better(s_best[w], best)) best = s_best[w];
    *out = best;
  }
}

// pass 1: one warp per row, grid-stride; block b's best to part[b]
__global__ void __launch_bounds__(kFarThreads) farthest_kernel(SelectParams p, int64_t exclude_row,
                                                               FarBest* __restrict__ part) {
  const int lane = threadIdx.x & 31;
  const int64_t warps = (int64_t)gridDim.x * (kFarThreads / 32);
  FarBest best{0.f, 0.0, -1};
  for (int64_t row = (int64_t)blockIdx.x * (kFarThreads / 32) + (threadIdx.x >> 5); row < p.N; row += warps) {
    const double dd = exact_distance(p, 0, row, lane);
    const FarBest c{(float)dd, dd, row};
    if (row != exclude_row && !isnan(c.f) && far_better(c, best)) best = c;
  }
  if (lane != 0) best.row = -1;  // every lane holds the warp's best; lane 0 speaks for it
  far_block_reduce(best, &part[blockIdx.x]);
}

// pass 2: one block over the blocks' bests
__global__ void __launch_bounds__(kFarThreads) farthest_reduce_kernel(const FarBest* __restrict__ part, int n_part,
                                                                      int64_t* __restrict__ out_row,
                                                                      float* __restrict__ out_dist) {
  __shared__ FarBest s_out;
  FarBest best{0.f, 0.0, -1};
  for (int b = threadIdx.x; b < n_part; b += kFarThreads)
    if (far_better(part[b], best)) best = part[b];
  far_block_reduce(best, &s_out);
  if (threadIdx.x == 0) {
    *out_row = s_out.row;
    *out_dist = s_out.row >= 0 ? s_out.f : 0.0f;
  }
}

static float reduce_max_host(const float* dev, int64_t n, cudaStream_t st, int* status) {
  std::vector<float> h(n);
  cudaError_t e = cudaMemcpyAsync(h.data(), dev, n * 4, cudaMemcpyDeviceToHost, st);
  if (e == cudaSuccess) e = cudaStreamSynchronize(st);
  if (e != cudaSuccess) {
    *status = cuda_fail(e, "D2H norms", __FILE__, __LINE__);
    return 0.f;
  }
  float m = 0.f;
  for (float v : h) m = std::max(m, v);
  *status = AM_OK;
  return m;
}

// ---------------------------------------------------------------- stored rows by id
__global__ void gather_rows_kernel(const float* __restrict__ X, int64_t N, int d, const int64_t* __restrict__ ids, int n,
                                   float* __restrict__ out) {
  const int64_t total = (int64_t)n * d;
  for (int64_t t = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; t < total; t += (int64_t)gridDim.x * blockDim.x) {
    const int64_t r = t / d;
    const int c = (int)(t - r * d);
    const int64_t row = ids[r];
    out[t] = (row >= 0 && row < N) ? X[row * d + c] : nanf("");
  }
}

}  // namespace am

using namespace am;

// the body of am_knn_build (X in host memory, kind = cudaMemcpyHostToDevice, on a stream of its own) and
// am_knn_build_dev (X in device memory, kind = cudaMemcpyDeviceToDevice, on the caller's stream `st`)
static int build_index(const char* fn, const float* X, int64_t N, int d, int metric, cudaMemcpyKind kind, cudaStream_t st,
                       am_index** out) {
  AM_CHECK(out != nullptr, "%s: out is NULL", fn);
  *out = nullptr;
  AM_CHECK(N >= 0 && d > 0 && (X != nullptr || N == 0), "%s: bad shape N=%lld d=%d", fn, (long long)N, d);
  AM_CHECK(metric >= 0 && metric <= 2, "%s: metric must be 0 (cosine), 1 (euclidean) or 2 (ip)", fn);
  AM_CHECK(N < (int64_t)0x7fffffff, "%s: at most 2^31-2 rows", fn);  // row ids are int, 0x7fffffff marks padding
  AM_TRY(ensure_init());
  Stream own;
  if (kind == cudaMemcpyHostToDevice) {
    AM_TRY(own.create());
    st = own.s;
  }
  std::unique_ptr<am_index> idx(new am_index());
  idx->N = N;
  idx->d = d;
  idx->metric = metric;
  AM_TRY(idx->X.alloc(std::max<size_t>((size_t)N * d, 1)));
  AM_TRY(idx->xnorm2.alloc(std::max<int64_t>(N, 1)));
  if (N > 0) {
    AM_CUDA(cudaMemcpyAsync(idx->X.p, X, (size_t)N * d * 4, kind, st));
    AM_LAUNCH(row_prepare_kernel, (unsigned)((N + 7) / 8), 256, 0, st, idx->X.p, N, d, metric == kMetricCos ? 1 : 0,
              idx->xnorm2.p);
    int s;
    const float m2 = reduce_max_host(idx->xnorm2.p, N, st, &s);
    AM_TRY(s);
    idx->max_norm = std::sqrt(m2) * 1.0001f;
    // bf16 copy for the tensor-core filter
    idx->dpad = (int)round_up(d, 64);
    AM_TRY(idx->Xb.alloc((size_t)N * idx->dpad));
    AM_TRY(idx->xres.alloc(N));
    AM_LAUNCH(row_to_bf16_kernel, (unsigned)((N + 7) / 8), 256, 0, st, idx->X.p, N, d, idx->dpad, idx->Xb.p, idx->xres.p);
    idx->xres_max = reduce_max_host(idx->xres.p, N, st, &s);
    AM_TRY(s);
  }
  *out = idx.release();
  return AM_OK;
}

extern "C" int am_knn_build(const float* X, int64_t N, int d, int metric, am_index** out) {
  return build_index("am_knn_build", X, N, d, metric, cudaMemcpyHostToDevice, nullptr, out);
}

extern "C" int am_knn_build_dev(const float* X_dev, int64_t N, int d, int metric, void* stream, am_index** out) {
  return build_index("am_knn_build_dev", X_dev, N, d, metric, cudaMemcpyDeviceToDevice, (cudaStream_t)stream, out);
}

extern "C" void am_knn_free(am_index* idx) { delete idx; }

// ---------------------------------------------------------------- query plan
// Everything about a query call that follows from (index, nq, k, mode), decided before anything is launched.
enum class Scorer {
  None,       // the full sort computes every distance itself
  F32,        // score_f32_kernel over the fp32 rows (+ chunk_max_rows_kernel for the chunk-max selection)
  Bf16Small,  // score_bf16_small_kernel: one pass over the bf16 rows per 1-4 queries, which also prepares the queries
              // and writes the chunk maxima
  Bf16Gemm,   // the wgmma GEMM over the bf16 rows, chunk maxima from its epilogue for the chunk-max selection
};
enum class Selection { ChunkMax, Rows, FullSort };  // select_cm_kernel, select_rerank_kernel, full_sort_query

struct QueryPlan {
  Scorer scorer;
  Selection select;
  int per_pass;      // queries per pass
  int qrows;         // rows of the per-pass query buffers (the GEMM's A operand: a multiple of 128, zero padded)
  SelectParams sel;  // shapes, error bound and index rows of the selection; the run adds the per-pass pointers
  size_t n_cm, n_s, n_qs, n_qb, n_qres;  // elements of the scratch buffers (qnorm and the overflow flags: qrows each)
};

static int plan_query(const am_index* idx, int nq, int k, int mode, QueryPlan* pl) {
  const int64_t N = idx->N;
  const int d = idx->d;
  const bool want_tensor = (mode == 2) || (mode == 0 && nq >= 16 && N >= 4096);
  const bool use_tensor = want_tensor && gemm::available();
  AM_CHECK(!(mode == 2 && !use_tensor), "am_knn_query: tensor-core filter unavailable on this device");
  SelectParams& p = pl->sel;
  p = SelectParams{};
  p.N = N;
  p.d = d;
  p.metric = idx->metric;
  p.k = k;
  p.X = idx->X.p;
  p.xnorm2 = idx->xnorm2.p;
  p.xnorm_max = idx->max_norm;
  p.ldS = round_up(N, 4);
  p.n_chunks = (N + kCmChunk - 1) / kCmChunk;
  p.ldCM = round_up(p.n_chunks, 8);
  // chunk-max selection when the k-th largest chunk maximum leaves enough chunks beside the k winners
  const bool chunk_max = k <= kCmMaxK && p.n_chunks >= 4 * (int64_t)k;
  if (k > kCandCap - 64) {
    pl->select = Selection::FullSort;
    pl->scorer = Scorer::None;
  } else {
    pl->select = chunk_max ? Selection::ChunkMax : Selection::Rows;
    if (use_tensor)
      pl->scorer = Scorer::Bf16Gemm;
    else if (mode == 0 && chunk_max && (idx->dpad == 256 || idx->dpad == 512 || idx->dpad == 1024))
      pl->scorer = Scorer::Bf16Small;
    else
      pl->scorer = Scorer::F32;
  }
  const bool gemm = pl->scorer == Scorer::Bf16Gemm, small = pl->scorer == Scorer::Bf16Small;
  // passes of at most 3 << 28 scores (3 GiB)
  pl->per_pass = (int)std::max<int64_t>(1, std::min<int64_t>(nq, (int64_t)(3ll << 28) / p.ldS));
  if (gemm) pl->per_pass = std::max(128, pl->per_pass / 128 * 128);
  pl->qrows = gemm ? (int)round_up(std::min(nq, pl->per_pass), 128) : std::min(nq, pl->per_pass);
  const size_t qrows = (size_t)pl->qrows;
  pl->n_cm = pl->select == Selection::ChunkMax ? qrows * p.ldCM : 0;
  pl->n_s = pl->scorer == Scorer::None ? 0 : qrows * p.ldS;
  pl->n_qs = small ? 0 : qrows * d;
  pl->n_qb = gemm ? qrows * idx->dpad : 0;
  pl->n_qres = (gemm || small) ? qrows : 0;
  // fp32 accumulation error: <= (d * 2^-24 * 1.01) * ||q|| ||x||  (any summation order).  It scales with ||q|| ||x||:
  // cosine queries are unit vectors; for inner product / euclidean the kernel multiplies by the query's own norm
  // (score_eps), so a query far larger than the stored rows is covered
  const float fp32_rel = (float)d * 6.1e-8f;
  p.eps_scales_with_q = idx->metric == kMetricCos ? 0 : 1;
  if (gemm || small) {  // bf16 products: the rounding residuals of both sides enter the bound (score_eps)
    p.xres = idx->xres.p;
    p.xres_max = idx->xres_max;
    p.eps_abs = fp32_rel * idx->max_norm;
  } else {  // fp32 pass: |s~ - s| <= d 2^-24 ||q|| ||x|| per dot product (x2 for the euclidean score 2 q.x - ||x||^2,
            // plus the rounding of the stored fp32 ||x||^2)
    p.eps_abs = fp32_rel * idx->max_norm * (idx->metric == kMetricL2 ? 2.0f : 1.0f) +
                (idx->metric == kMetricL2 ? 1.2e-7f * idx->max_norm * idx->max_norm : 0.0f);
  }
  return AM_OK;
}

struct QueryBufs {
  float *CM, *S, *Qs;
  double* qnorm;
  int* overflow;
  __nv_bfloat16* Qb;
  float* qres;
  std::vector<int> flags;  // host: the overflow flags of the last pass
};

template <int kQ, int kSegs>
static int score_small_launch(const am_index* idx, const QueryPlan& pl, const QueryBufs& b, const float* Qc, int nc, int t0,
                              int grid, cudaStream_t st) {
  AM_LAUNCH((score_bf16_small_kernel<kQ, kSegs>), grid, 256, 0, st, idx->Xb.p, idx->xnorm2.p, idx->N, idx->d, idx->dpad, Qc,
            nc, t0, idx->metric, b.S, pl.sel.ldS, b.CM, pl.sel.ldCM, pl.sel.n_chunks, b.qnorm, b.qres);
  return AM_OK;
}

// the pass's queries four, two or one per launch
template <int kSegs>
static int score_small(const am_index* idx, const QueryPlan& pl, const QueryBufs& b, const float* Qc, int nc,
                       cudaStream_t st) {
  const int grid = (int)std::max<int64_t>(1, std::min<int64_t>((pl.sel.n_chunks + 7) / 8, (int64_t)sm_count() * 8));
  for (int t0 = 0; t0 < nc;) {
    const int kq = nc - t0 >= 4 ? 4 : (nc - t0 >= 2 ? 2 : 1);
    if (kq == 4) AM_TRY((score_small_launch<4, kSegs>(idx, pl, b, Qc, nc, t0, grid, st)));
    else if (kq == 2) AM_TRY((score_small_launch<2, kSegs>(idx, pl, b, Qc, nc, t0, grid, st)));
    else AM_TRY((score_small_launch<1, kSegs>(idx, pl, b, Qc, nc, t0, grid, st)));
    t0 += kq;
  }
  return AM_OK;
}

// The scratch of a query plan, as parts of `call`.  The overflow flags of a pass come back into b->flags.
static void query_parts(HostCall& call, const QueryPlan& pl, int nq, QueryBufs* b) {
  b->flags.resize(std::min(nq, pl.per_pass));
  call.device(&b->CM, pl.n_cm);
  call.device(&b->S, pl.n_s);
  call.device(&b->Qs, pl.n_qs);
  call.device(&b->qnorm, (size_t)pl.qrows);
  call.down(&b->overflow, b->flags.size(), b->flags.data());
  call.device(&b->Qb, pl.n_qb);
  call.device(&b->qres, pl.n_qres);
}

// The host side of a query's passes.  fetch(q0, nc, false) brings the overflow flags of the pass's nc queries into
// b.flags and synchronises; fetch(q0, nc, true) runs after flagged queries were answered by the full sort and brings
// the pass's results to wherever the caller wants them.
using FetchPass = std::function<int(int q0, int nc, bool results_only)>;

// Runs a checked query (1 <= k <= N, nq >= 1) on device pointers, in the scratch query_parts declared.
static int knn_query_impl(const am_index* idx, const QueryPlan& pl, const QueryBufs& b, const float* Q_dev, int nq, int k,
                          int64_t* ids_dev, float* dist_dev, cudaStream_t st, const FetchPass& fetch) {
  const int64_t N = idx->N;
  const int d = idx->d;
  const bool gemm = pl.scorer == Scorer::Bf16Gemm, small = pl.scorer == Scorer::Bf16Small;
  SelectParams p = pl.sel;
  p.S = b.S;
  p.CM = b.CM;
  p.qnorm = b.qnorm;
  p.qres = (gemm || small) ? b.qres : nullptr;
  p.overflow = b.overflow;
  const size_t sel_smem = (size_t)kCandCap * (sizeof(double) + sizeof(int));
  for (int q0 = 0; q0 < nq; q0 += pl.per_pass) {
    const int nc = std::min(pl.per_pass, nq - q0);
    p.Q = Q_dev + (int64_t)q0 * d;
    p.ids = ids_dev + (int64_t)q0 * k;
    p.dist = dist_dev + (int64_t)q0 * k;
    // 1. queries: norms, normalised fp32 copy, bf16 copy + residual norm
    if (gemm) AM_CUDA(cudaMemsetAsync(b.Qb, 0, (size_t)pl.qrows * idx->dpad * sizeof(__nv_bfloat16), st));
    if (!small)
      AM_LAUNCH(query_prepare_kernel, ceil_div(nc, 8), 256, 0, st, p.Q, nc, d, idx->dpad, idx->metric, b.Qs, b.qnorm,
                gemm ? b.Qb : nullptr, gemm ? b.qres : nullptr);
    // 2. approximate scores, and their per-32 maxima for the chunk-max selection
    switch (pl.scorer) {
      case Scorer::None:
        break;
      case Scorer::F32: {
        const int grid = std::max(1, std::min<int>((int)((N + 7) / 8), sm_count() * 8));
        for (int t0 = 0; t0 < nc; t0 += kQT)
          AM_LAUNCH(score_f32_kernel, grid, 256, (size_t)kQT * d * 4, st, idx->X.p, idx->xnorm2.p, N, d, b.Qs, nc, t0,
                    idx->metric, b.S, p.ldS);
        if (pl.select == Selection::ChunkMax) {
          const int64_t warps = (int64_t)nc * p.n_chunks;
          AM_LAUNCH(chunk_max_rows_kernel, (unsigned)std::min<int64_t>((warps + 7) / 8, (int64_t)sm_count() * 16), 256, 0,
                    st, b.S, p.ldS, N, nc, p.n_chunks, b.CM, p.ldCM);
        }
        break;
      }
      case Scorer::Bf16Small:
        if (idx->dpad == 256) AM_TRY(score_small<1>(idx, pl, b, p.Q, nc, st));
        else if (idx->dpad == 512) AM_TRY(score_small<2>(idx, pl, b, p.Q, nc, st));
        else AM_TRY(score_small<4>(idx, pl, b, p.Q, nc, st));
        break;
      case Scorer::Bf16Gemm:  // bf16 x bf16 -> fp32 in registers, euclidean fix-up in the epilogue
        AM_TRY(gemm::scores_bf16(b.Qb, pl.qrows, idx->Xb.p, N, idx->dpad, b.S, p.ldS,
                                 pl.select == Selection::ChunkMax ? b.CM : nullptr, p.ldCM,
                                 idx->metric == kMetricL2 ? idx->xnorm2.p : nullptr, st));
        break;
    }
    // 3. selection + exact re-rank; a query whose candidates do not fit on chip raises its overflow flag
    switch (pl.select) {
      case Selection::ChunkMax:
        AM_TRY(allow_dynamic_smem<select_cm_kernel>(sel_smem));
        AM_LAUNCH(select_cm_kernel, nc, kSelThreads, sel_smem, st, p);
        break;
      case Selection::Rows:
        AM_TRY(allow_dynamic_smem<select_rerank_kernel>(sel_smem));
        AM_LAUNCH(select_rerank_kernel, nc, kSelThreads, sel_smem, st, p);
        break;
      case Selection::FullSort:
        break;
    }
    // 4. overflow flags to the host; flagged queries (all of them for the full sort) answered by the full sort
    const bool all = pl.select == Selection::FullSort;
    if (!all) AM_TRY(fetch(q0, nc, false));
    bool any = false;
    for (int q = 0; q < nc; ++q)
      if (all || b.flags[q]) {
        AM_TRY(full_sort_query(p, q, st));
        any = true;
      }
    if (any) AM_TRY(fetch(q0, nc, true));
  }
  return AM_OK;
}

// the size checks of both query entry points
static int check_query(const am_index* idx, int nq, int k) {
  AM_CHECK(nq >= 0 && k >= 0, "am_knn_query: negative size");
  if (k > idx->N) {
    set_error("am_knn_query: k=%d exceeds the %lld stored vectors (voyager.RecallError)", k, (long long)idx->N);
    return AM_ERR_RECALL;
  }
  return AM_OK;
}

extern "C" int am_knn_query_dev(const am_index* idx, const float* Q_dev, int nq, int k, int mode, int64_t* ids_dev,
                                float* dist_dev, void* stream) {
  AM_CHECK(idx && Q_dev && ids_dev && dist_dev, "am_knn_query_dev: NULL argument");
  AM_TRY(check_query(idx, nq, k));
  if (nq == 0 || k == 0) return AM_OK;
  QueryPlan pl;
  AM_TRY(plan_query(idx, nq, k, mode, &pl));
  const cudaStream_t st = (cudaStream_t)stream;
  // the caller's stream, nothing pinned: only the overflow flags come back
  HostCall call(st, 0, HostCall::Memory::Pool);
  QueryBufs b;
  query_parts(call, pl, nq, &b);
  AM_TRY(call.start());
  return knn_query_impl(idx, pl, b, Q_dev, nq, k, ids_dev, dist_dev, st,
                        [&](int, int, bool results_only) { return results_only ? AM_OK : call.finish(); });
}

extern "C" int am_knn_query(const am_index* idx, const float* Q, int nq, int k, int mode, int64_t* ids, float* dist) {
  AM_CHECK(idx && (Q || nq == 0) && (ids || nq * (int64_t)k == 0) && (dist || nq * (int64_t)k == 0),
           "am_knn_query: NULL argument");
  AM_TRY(check_query(idx, nq, k));
  if (nq == 0 || k == 0) return AM_OK;
  cudaStream_t st;
  AM_TRY(HostCall::thread_stream(&st));
  QueryPlan pl;
  AM_TRY(plan_query(idx, nq, k, mode, &pl));
  HostCall call(st, kStageLimit, HostCall::Memory::Pool);
  float *dQ, *dD;
  int64_t* dI;
  call.up(&dQ, Q, (size_t)nq * idx->d);
  call.down(&dI, (size_t)nq * k, ids);
  call.down(&dD, (size_t)nq * k, dist);
  QueryBufs b;
  query_parts(call, pl, nq, &b);
  AM_TRY(call.start());
  // a call of one pass brings its results back with the flags (a single query: 3 host-side CUDA calls besides the
  // launches); otherwise, and after full sorts, the pass's rows are copied straight to the caller's arrays
  return knn_query_impl(idx, pl, b, dQ, nq, k, dI, dD, st, [&](int q0, int nc, bool results_only) -> int {
    if (!results_only && nc == nq) return call.finish();
    if (!results_only) AM_CUDA(cudaMemcpyAsync(b.flags.data(), b.overflow, nc * sizeof(int), cudaMemcpyDeviceToHost, st));
    const int64_t r0 = (int64_t)q0 * k;
    AM_CUDA(cudaMemcpyAsync(ids + r0, dI + r0, (size_t)nc * k * 8, cudaMemcpyDeviceToHost, st));
    AM_CUDA(cudaMemcpyAsync(dist + r0, dD + r0, (size_t)nc * k * 4, cudaMemcpyDeviceToHost, st));
    AM_CUDA(cudaStreamSynchronize(st));
    return AM_OK;
  });
}

extern "C" int am_knn_get_vectors(const am_index* idx, const int64_t* ids, int n, float* out) {
  AM_CHECK(idx && (n == 0 || (ids && out)), "am_knn_get_vectors: NULL argument");
  AM_CHECK(n >= 0, "am_knn_get_vectors: negative count");
  if (n == 0) return AM_OK;
  for (int i = 0; i < n; ++i)
    AM_CHECK(ids[i] >= 0 && ids[i] < idx->N, "am_knn_get_vectors: id %lld out of range [0, %lld)", (long long)ids[i],
             (long long)idx->N);
  cudaStream_t st;
  AM_TRY(HostCall::thread_stream(&st));
  // a whole library (Index._materialise_rows) goes straight to the caller's array instead of pinning its size for good
  HostCall call(st, kStageLimit, HostCall::Memory::Pool);
  int64_t* d_ids;
  float* d_out;
  call.up(&d_ids, ids, (size_t)n);
  call.down(&d_out, (size_t)n * idx->d, out);
  AM_TRY(call.start());
  const int grid = (int)std::max<int64_t>(1, std::min<int64_t>(((int64_t)n * idx->d + 255) / 256, (int64_t)sm_count() * 8));
  AM_LAUNCH(gather_rows_kernel, grid, 256, 0, st, idx->X.p, idx->N, idx->d, d_ids, n, d_out);
  return call.finish();
}

extern "C" int am_knn_farthest(const am_index* idx, const float* query, int64_t exclude_row, int64_t* out_row,
                               float* out_dist) {
  AM_CHECK(idx && query && out_row && out_dist, "am_knn_farthest: NULL argument");
  AM_CHECK(exclude_row >= -1 && exclude_row < idx->N, "am_knn_farthest: excluded row %lld out of range",
           (long long)exclude_row);
  *out_row = -1;
  *out_dist = 0.0f;
  if (idx->N == 0) return AM_OK;
  cudaStream_t st;
  AM_TRY(HostCall::thread_stream(&st));
  const int d = idx->d;
  const int n_part = (int)std::max<int64_t>(1, std::min<int64_t>((idx->N + 7) / 8, (int64_t)sm_count() * 8));
  HostCall call(st, HostCall::kAlways, HostCall::Memory::Pool);
  float *dQ, *dQs, *dD;
  double* qnorm;
  int64_t* dR;
  FarBest* part;
  call.up(&dQ, query, (size_t)d);
  call.down(&dR, 1, out_row);
  call.down(&dD, 1, out_dist);
  call.device(&dQs, (size_t)d);
  call.device(&qnorm, 1);
  call.device(&part, (size_t)n_part);
  AM_TRY(call.start());
  // the query as knn_query_impl prepares it for a single query of k = N (query_prepare_kernel, then exact_distance)
  AM_LAUNCH(query_prepare_kernel, 1, 256, 0, st, dQ, 1, d, idx->dpad, idx->metric, dQs, qnorm, nullptr, nullptr);
  SelectParams p{};
  p.N = idx->N;
  p.d = d;
  p.metric = idx->metric;
  p.X = idx->X.p;
  p.xnorm2 = idx->xnorm2.p;
  p.Q = dQ;
  p.qnorm = qnorm;
  AM_LAUNCH(farthest_kernel, n_part, kFarThreads, 0, st, p, exclude_row, part);
  AM_LAUNCH(farthest_reduce_kernel, 1, kFarThreads, 0, st, part, n_part, dR, dD);
  return call.finish();
}
