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
#include "common.cuh"

#include <math_constants.h>

#include <algorithm>
#include <cmath>
#include <memory>

#include "gemm_wgmma.cuh"

namespace am {

constexpr int kMetricCos = 0, kMetricL2 = 1, kMetricIp = 2;
constexpr int kCandCap = 4096;       // on-chip candidate capacity per query
constexpr int kCmChunk = 32;         // the GEMM epilogue also writes the maximum of every 32 consecutive scores
constexpr int kCmMaxK = 512;         // chunk-max selection: k-th largest chunk maximum as the threshold
constexpr int kCmChunkCap = 2048;    // flagged chunks a query may have on chip
constexpr int kSelThreads = 1024;

}  // namespace am

struct am_index {
  int64_t N = 0;
  int d = 0;
  int metric = 0;
  am::DevBuf<float> X;        // [N, d] stored rows (unit-normalised for cosine)
  am::DevBuf<float> xnorm2;   // [N] squared norms (euclidean)
  am::DevBuf<__nv_bfloat16> Xb;  // [N, dpad] bf16 copy for the tensor-core filter
  am::DevBuf<float> xres;     // [N] ||x - bf16(x)||_2 (bf16 filter bound)
  int dpad = 0;
  float max_norm = 1.0f;      // max ||x|| over stored rows
  float xres_max = 0.0f;      // max ||x - bf16(x)|| over stored rows
};

namespace am {

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


// ---------------------------------------------------------------- duplicate filter on device
// voyager_manager.py:526-617 (_filter_by_distance) + :487-524 (_compute_distance_batch): walk a result list in
// order and drop an item whose DIRECT distance (get_direct_distance, :99-140: cosine = 1 - cos with both norms
// recomputed, euclidean = ||a - b||, not squared) to a recently kept item is below the threshold.  "Recently
// kept": lists of <= `batch` items compare with the last `lookback` kept items; longer lists are cut into
// batches of `batch`, and an item is compared with the last `lookback` items kept BEFORE its batch plus
// everything kept so far inside the batch.  One CTA per list; the walk is sequential, the comparisons of one
// item are spread over the warps; float64 accumulation.
constexpr int kFilterThreads = 256;
constexpr int kFilterCap = 4096;  // items per list

// get_direct_distance (voyager_manager.py:99-140) between stored rows a and b, one warp, float64 accumulation:
// euclidean ||a - b||, otherwise 1 - cos (+inf when either row is zero)
__device__ __forceinline__ double direct_distance(const float* a, const float* b, int d, int metric, int lane) {
  double dot = 0.0, na = 0.0, nb = 0.0, d2 = 0.0;
  for (int t = lane; t < d; t += 32) {
    const double av = (double)__ldg(&a[t]), bv = (double)__ldg(&b[t]);
    dot = fma(av, bv, dot);
    na = fma(av, av, na);
    nb = fma(bv, bv, nb);
    const double df = av - bv;
    d2 = fma(df, df, d2);
  }
  dot = warp_sum(dot);
  na = warp_sum(na);
  nb = warp_sum(nb);
  d2 = warp_sum(d2);
  if (metric == kMetricL2) return sqrt(d2);
  const double den = sqrt(na) * sqrt(nb);
  return den == 0.0 ? INFINITY : 1.0 - fmin(1.0, fmax(-1.0, dot / den));
}

// The first kept item that item i of a list is compared with: the last `lookback` kept ones, or in a list longer
// than the batch, the last `lookback` kept before i's batch (kept_at_batch) and every one kept since.
__device__ __forceinline__ int filter_window_start(int kept, int kept_at_batch, bool batched, int lookback) {
  return max(0, (batched ? kept_at_batch : kept) - lookback);
}

__global__ void __launch_bounds__(kFilterThreads)
filter_by_distance_kernel(const float* __restrict__ X, int64_t N, int d, int metric, const int64_t* __restrict__ ids,
                          int n, double threshold, int lookback, int batch, unsigned char* __restrict__ keep) {
  __shared__ int s_kept[kFilterCap];
  __shared__ int s_close;
  const int64_t* my_ids = ids + (int64_t)blockIdx.x * n;
  unsigned char* my_keep = keep + (int64_t)blockIdx.x * n;
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31, warps = kFilterThreads / 32;
  int kept = 0, base = 0;  // base: number kept when the current batch started
  const bool batched = n > batch;
  for (int i = 0; i < n; ++i) {
    if (batched && i % batch == 0) base = kept;
    const int64_t row = my_ids[i];
    if (threadIdx.x == 0) s_close = 0;
    __syncthreads();
    bool valid = row >= 0 && row < N;  // the reference skips items whose vector is missing
    if (valid) {
      const int start = filter_window_start(kept, base, batched, lookback);
      const float* a = X + row * d;
      for (int j = start + warp; j < kept; j += warps) {
        const double dist = direct_distance(a, X + (int64_t)s_kept[j] * d, d, metric, lane);
        if (lane == 0 && dist < threshold) s_close = 1;
      }
    }
    __syncthreads();
    const bool keep_it = valid && !s_close;
    if (threadIdx.x == 0) {
      my_keep[i] = keep_it ? 1 : 0;
      if (keep_it) s_kept[kept] = (int)row;
    }
    if (keep_it) ++kept;
    __syncthreads();
  }
}


// ---------------------------------------------------------------- radius walk on device
// voyager_manager.py:941-1367 (_execute_radius_walk) over the candidates _radius_walk_get_candidates (:842-938) leaves,
// in one CTA.  The reference's steps and the state that restates each:
//   * anchor distances (:927, get_direct_distance) in float64, one warp per candidate; the stable sort by that distance
//     (:968) is a bitonic sort of (distance bits, input position) keys -- distances are >= 0 or +inf, so their bit
//     patterns order like the values, and the position breaks ties the way a stable sort keeps them;
//   * buckets of 50 in that order (:956, :970-974), walked one after the other until the playlist holds n songs (what
//     the window-doubling loop at :1261-1281 amounts to);
//   * the first song is sorted[0] (:1008-1013); its artist counts (:1041-1047) but not per bucket;
//   * each bucket starts at its first unused candidate (:1091-1103; in bucket 0 that skips sorted[0]), accepted if it
//     passes the artist rules and otherwise only dropped from the bucket (:1140-1163);
//   * then greedily: score = 0.7 d(prev, cand) + 0.3 float32(d(anchor, cand)) (:1222), the first strict minimum in
//     bucket order wins (:1223), prev is the last song APPENDED (:1174), and the bucket ends when no candidate passes;
//   * the artist rules (:1120-1136, :1188-1211) apply when eliminate_duplicates and the cap is > 0: one song per artist
//     per bucket, and an artist already in 2 buckets or at the cap is refused;
//   * once the playlist holds n songs nothing later changes it (:1146, :1237, :1262), so the walk stops there;
//   * _avoid_triple_adjacent (:1287-1318) on the final order.
// Per-candidate state lives in global scratch (sort keys, per-artist counters, the playlist); only the distances from
// the current song to the <= 50 candidates of the bucket are in shared memory.  Warp 0 keeps the books, every warp
// computes distances.
constexpr int kWalkThreads = 1024;
constexpr int kWalkBucket = 50;    // BUCKET_SIZE, voyager_manager.py:956
constexpr unsigned long long kWalkMissing = ~0ull;  // sort key of a candidate that is not in the index: after +inf

__device__ __forceinline__ double walk_key_dist(unsigned long long k) { return __longlong_as_double((long long)k); }

// artists[c] of input position c (-1: no artist); count / buckets / mark: per artist, the songs taken, the buckets it
// has a song in, and the last bucket it took a song in
__device__ __forceinline__ bool walk_artist_ok(int a, int bucket, int cap, const int* count, const int* buckets,
                                               const int* mark) {
  return a < 0 || !(mark[a] == bucket || buckets[a] >= 2 || count[a] >= cap);
}

__global__ void __launch_bounds__(kWalkThreads)
radius_walk_kernel(const float* __restrict__ X, int64_t N, int d, int metric, const float* __restrict__ anchor,
                   const int64_t* __restrict__ rows, const int32_t* __restrict__ artists, int n_cand, int n,
                   int artist_rules, int cap, int64_t npad, unsigned long long* key, int* ord, int* count,
                   int* buckets, int* mark, int* playlist, int32_t* __restrict__ out_pos,
                   double* __restrict__ out_dist, int32_t* __restrict__ out_count) {
  __shared__ double s_dprev[kWalkBucket];
  __shared__ unsigned long long s_elig;  // candidates of the bucket that may be taken next
  __shared__ int s_valid, s_len, s_prev_pos;  // valid candidates, playlist length, input position of the last song
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31, warps = kWalkThreads / 32;
  if (threadIdx.x == 0) s_valid = 0;
  __syncthreads();

  // ---- anchor distances and sort keys (padding sorts after every candidate)
  for (int64_t i = warp; i < npad; i += warps) {
    unsigned long long k = kWalkMissing;
    const int64_t row = i < n_cand ? rows[i] : -1;
    if (row >= 0 && row < N) {
      k = (unsigned long long)__double_as_longlong(direct_distance(X + row * d, anchor, d, metric, lane));
      if (lane == 0) atomicAdd(&s_valid, 1);
    }
    if (lane == 0) {
      key[i] = k;
      ord[i] = (int)i;
    }
  }
  __syncthreads();
  // ---- bitonic sort of (key, position) ascending
  for (int64_t kk = 2; kk <= npad; kk <<= 1) {
    for (int64_t j = kk >> 1; j > 0; j >>= 1) {
      for (int64_t i = threadIdx.x; i < npad; i += kWalkThreads) {
        const int64_t l = i ^ j;
        if (l > i) {
          const unsigned long long ki = key[i], kl = key[l];
          const int oi = ord[i], ol = ord[l];
          const bool i_after = ki > kl || (ki == kl && oi > ol);
          if (i_after == ((i & kk) == 0)) {
            key[i] = kl;
            key[l] = ki;
            ord[i] = ol;
            ord[l] = oi;
          }
        }
      }
      __syncthreads();
    }
  }

  // ---- the walk; sorted index s -> input position ord[s], anchor distance key[s]
  const int m = s_valid;
  if (threadIdx.x == 0) {
    s_len = 0;
    if (m > 0 && n > 0) {  // the first song (:1008-1013, :1041-1047)
      playlist[0] = 0;
      s_len = 1;
      s_prev_pos = ord[0];
      const int a = artists[ord[0]];
      if (a >= 0) count[a] += 1;
    }
  }
  __syncthreads();
  for (int b = 0;; ++b) {
    const bool go = (int64_t)b * kWalkBucket < m && s_len < n;  // read by every thread before warp 0 writes again
    __syncthreads();
    if (!go) break;
    const int base = b * kWalkBucket, nb = min(kWalkBucket, m - base);
    // warp 0's books for this bucket: candidates still available, playlist length, the artist of each lane's two
    // candidates (j = lane, lane + 32)
    unsigned long long avail = ((1ull << nb) - 1) & ~(b == 0 ? 1ull : 0ull);  // bucket 0 holds the first song
    int len = 0, art[2] = {-1, -1};
    // the candidates that may be taken next (a warp-wide ballot)
    auto eligible = [&]() {
      unsigned long long e = 0;
      for (int h = 0; h < 2; ++h) {
        const int j = lane + 32 * h;
        const bool ok = j < nb && ((avail >> j) & 1) &&
                        (!artist_rules || walk_artist_ok(art[h], b, cap, count, buckets, mark));
        e |= (unsigned long long)__ballot_sync(0xffffffffu, ok) << (32 * h);
      }
      return e;
    };
    // take sorted index base + j (the bookkeeping of :1141-1161 / :1232-1253); lane 0 writes, the warp reads back
    auto accept = [&](int j) {
      avail &= ~(1ull << j);
      if (lane == 0) {
        if (len < n) {
          playlist[len] = base + j;
          s_prev_pos = ord[base + j];
        }
        const int a = artists[ord[base + j]];
        if (a >= 0) {
          count[a] += 1;
          if (mark[a] != b) {
            mark[a] = b;
            buckets[a] += 1;
          }
        }
      }
      if (len < n) ++len;
      __syncwarp();
    };
    if (warp == 0) {
      len = s_len;
      for (int h = 0; h < 2; ++h) {
        const int j = lane + 32 * h;
        if (j < nb) art[h] = artists[ord[base + j]];
      }
      if (avail) {  // the start (:1105-1163): the first available candidate, taken if the artist rules allow it
        const int start = __ffsll((long long)avail) - 1;
        if ((eligible() >> start) & 1) accept(start);
        else avail &= ~(1ull << start);
      }
      const unsigned long long e = len < n ? eligible() : 0ull;
      if (lane == 0) {
        s_len = len;
        s_elig = e;
      }
    }
    // greedy steps (:1166-1253): every warp computes d(prev, cand) for the eligible candidates, warp 0 picks
    for (;;) {
      __syncthreads();  // s_elig / s_prev_pos published
      const unsigned long long e = s_elig;
      if (e == 0) break;
      const float* prev = X + rows[s_prev_pos] * d;
      for (int j = warp; j < nb; j += warps)
        if ((e >> j) & 1) {
          const double dist = direct_distance(X + rows[ord[base + j]] * d, prev, d, metric, lane);
          if (lane == 0) s_dprev[j] = dist;
        }
      __syncthreads();  // distances ready
      if (warp == 0) {
        double best = INFINITY;  // a score must be strictly below +inf and below every earlier one (:1179, :1223)
        int best_j = INT_MAX;
        for (int h = 0; h < 2; ++h) {
          const int j = lane + 32 * h;
          if (j < nb && ((e >> j) & 1)) {
            const double a32 = (double)(float)walk_key_dist(key[base + j]);  // the bucket's float32 array (:983)
            const double score = __dadd_rn(__dmul_rn(0.7, s_dprev[j]), __dmul_rn(0.3, a32));
            if (score < best) {
              best = score;
              best_j = j;
            }
          }
        }
        for (int o = 16; o > 0; o >>= 1) {  // the first minimum in bucket order
          const double ob = __shfl_xor_sync(0xffffffffu, best, o);
          const int oj = __shfl_xor_sync(0xffffffffu, best_j, o);
          if (ob < best || (ob == best && oj < best_j)) {
            best = ob;
            best_j = oj;
          }
        }
        unsigned long long next = 0;
        if (best_j != INT_MAX) {
          accept(best_j);
          if (len < n) next = eligible();
        }
        if (lane == 0) {
          s_len = len;
          s_elig = next;
        }
      }
    }
  }

  // ---- _avoid_triple_adjacent (:1287-1318) on the playlist, then the outputs
  const int L = s_len;
  if (threadIdx.x == 0) {
    auto author = [&](int t) { return artists[ord[playlist[t]]]; };
    int i = 0;
    while (i <= L - 3) {
      const int a1 = author(i);
      if (a1 >= 0 && a1 == author(i + 1) && a1 == author(i + 2)) {
        int j = i + 3;
        while (j < L && author(j) == a1) ++j;
        if (j < L) {  // swap the third with the first later song by another artist, then look at i again
          const int t = playlist[i + 2];
          playlist[i + 2] = playlist[j];
          playlist[j] = t;
          continue;
        }
      }
      ++i;
    }
    *out_count = L;
  }
  __syncthreads();
  for (int t = threadIdx.x; t < L; t += kWalkThreads) {
    out_pos[t] = ord[playlist[t]];
    out_dist[t] = walk_key_dist(key[playlist[t]]);
  }
}


// ---------------------------------------------------------------- song path walk on device
// path_manager.py:180-317 (_find_best_songs_for_job) over the chain find_nearest_neighbors_by_vector
// (voyager_manager.py:1547-1657) runs on each job's k-NN prefix, for a sequence of jobs, in one CTA.  One pass over a
// job's candidates in k-NN order does every stage, because each stage only looks at what came before it:
//   * _filter_by_distance (:526-617): the item is compared with the kept window (filter_window_start) in the
//     VOYAGER_METRIC distance; with no lookback the list is unchanged;
//   * same-song dedupe (:1625-1636): an item without details, or whose signature this job already let through, is out;
//   * the raw-author cap (:1638-1653, only when eliminate_duplicates and the cap is > 0; falsy authors are out);
//   * [:n]: the pass ends after the n-th item that got this far;
//   * acceptance (path_manager.py:211-291): used rows and signatures, the normalised-author cap, then the lookbacks
//     against the path's last songs and this job's found songs, in PATH_DISTANCE_METRIC; the job ends once it has
//     its songs.  A job that falls short gives back what it took (:294-312).
// Per candidate, every warp computes the distances the decision may need (filter window, path window, found window)
// and the threads look for the row among the used rows; then thread 0 decides and keeps the books.
constexpr int kPathThreads = 512;

// get_distance (path_manager.py:27-52): euclidean ||a - b||, angular arccos(clip(cos)) / pi (+inf when either row is
// zero).  cos = 1 - (1 - cos) is exact for cos >= 0.5, which covers every distance below the thresholds.
__device__ __forceinline__ double path_distance(const float* a, const float* b, int d, int metric, int lane) {
  const double dd = direct_distance(a, b, d, metric, lane);
  if (metric == kMetricL2 || dd == INFINITY) return dd;
  return acos(1.0 - dd) / CUDART_PI;
}

struct SongPathArgs {
  const float* X;
  int64_t N;
  int d;
  int n_jobs;
  const int32_t* job_off;     // [n_jobs + 1] candidate ranges
  const int32_t* job_n;       // [n_jobs] the by-vector n (k_search)
  const int32_t* job_need;    // [n_jobs] num_to_find
  const int64_t* cand_row;    // [n_cand] stored row, -1: no vector
  const int32_t* cand_sig;    // (title, author) signature key, -1: no details
  const int32_t* cand_author; // normalised author key
  const int32_t* cand_raw;    // raw author key, -1: falsy author
  int64_t* used_row;          // [n_used + sum(need)] in / out
  int32_t* n_used;
  unsigned char* used_sig;    // [n_sig] in / out
  int32_t* author_count;      // [n_author] in / out
  int64_t* path_row;          // [n_path + sum(need)] in / out: the start song first
  int32_t* n_path;
  int64_t end_row;
  am_song_path_cfg cfg;
  int32_t* seen;              // [n_sig] scratch: the job that last let the signature through, -1 initially
  int32_t* raw_mark;          // [n_raw] scratch: the job that last counted the raw author, -1 initially
  int32_t* raw_count;         // [n_raw] scratch
  int32_t* kept;              // [2 x max candidates per job] scratch: the filter's kept positions, then the job's found
  int32_t* out_found;         // [n_jobs]
  int32_t* out_pos;           // [sum(need)] accepted candidates, in path order
  int32_t* out_failed;        // first failed job when stopping on failure, else -1
  double* out_dist;           // [n_path + sum(need)] distances between consecutive songs of the path and the end song
};

__global__ void __launch_bounds__(kPathThreads) song_path_kernel(const SongPathArgs a) {
  __shared__ int s_close;      // bit 0: filter window, bit 1: path window, bit 2: found window
  __shared__ int s_used, s_stop;
  __shared__ int s_kept, s_batch_kept, s_found, s_prod, s_n_used, s_n_path, s_n_out;
  const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31, warps = kPathThreads / 32;
  const am_song_path_cfg& c = a.cfg;
  const int lb_f = c.filter_lookback, lb_p = c.path_lookback;
  for (int j = tid; j < a.n_jobs; j += kPathThreads) a.out_found[j] = 0;  // jobs after a stop are not run
  if (tid == 0) {
    s_n_used = *a.n_used;
    s_n_path = *a.n_path;
    s_n_out = 0;
    *a.out_failed = -1;
  }
  __syncthreads();
  for (int j = 0; j < a.n_jobs; ++j) {
    const int base = a.job_off[j], m = a.job_off[j + 1] - base, n = a.job_n[j], need = a.job_need[j];
    const bool batched = m > c.filter_batch;
    if (tid == 0) {
      s_kept = s_batch_kept = s_found = s_prod = s_stop = 0;
    }
    const int used0 = s_n_used;  // the rows this job adds are given back by truncation
    __syncthreads();
    int found_all = 0;  // thread 0: songs found so far
    for (int i = 0; i < m; ++i) {
      const int64_t row = a.cand_row[base + i];
      const bool valid = row >= 0 && row < a.N;
      if (tid == 0) {
        s_close = 0;
        s_used = 0;
        if (batched && i % c.filter_batch == 0) s_batch_kept = s_kept;
      }
      __syncthreads();
      if (valid) {
        const int kept = s_kept, found = s_found, np = s_n_path;
        const int f0 = lb_f > 0 ? filter_window_start(kept, s_batch_kept, batched, lb_f) : kept;
        const int nf = kept - f0, npw = min(lb_p, np), nq = min(lb_p, found);
        const float* x = a.X + row * a.d;
        for (int t = warp; t < nf + npw + nq; t += warps) {
          int64_t other;
          int metric, bit;
          double thr;
          if (t < nf) {
            other = a.cand_row[base + a.kept[f0 + t]];
            metric = c.voyager_metric;
            thr = c.filter_threshold;
            bit = 1;
          } else if (t < nf + npw) {
            other = a.path_row[np - npw + (t - nf)];
            metric = c.path_metric;
            thr = c.path_threshold;
            bit = 2;
          } else {
            other = a.cand_row[base + a.kept[m + found - nq + (t - nf - npw)]];
            metric = c.path_metric;
            thr = c.path_threshold;
            bit = 4;
          }
          const float* y = a.X + other * a.d;
          const double dist = bit == 1 ? direct_distance(x, y, a.d, metric, lane) : path_distance(x, y, a.d, metric, lane);
          if (lane == 0 && dist < thr) atomicOr(&s_close, bit);
        }
      }
      for (int t = tid; t < s_n_used; t += kPathThreads)
        if (a.used_row[t] == row) s_used = 1;
      __syncthreads();
      if (tid == 0) {
        const int close = s_close;
        bool pass = true;
        if (lb_f > 0) {  // _filter_by_distance: items without a vector are dropped, the kept ones form the window
          pass = valid && !(close & 1);
          if (pass) a.kept[s_kept++] = i;
        }
        const int sig = a.cand_sig[base + i];
        if (pass && sig < 0) pass = false;
        if (pass) {
          if (a.seen[sig] == j) pass = false;
          else a.seen[sig] = j;
        }
        if (pass && c.voyager_cap > 0) {
          const int r = a.cand_raw[base + i];
          if (r < 0) {
            pass = false;
          } else {
            if (a.raw_mark[r] != j) {
              a.raw_mark[r] = j;
              a.raw_count[r] = 0;
            }
            if (a.raw_count[r] >= c.voyager_cap) pass = false;
            else a.raw_count[r] += 1;
          }
        }
        if (pass) {
          s_prod += 1;
          const int au = a.cand_author[base + i];
          const bool ok = !s_used && !a.used_sig[sig] && !(c.path_cap > 0 && a.author_count[au] >= c.path_cap) && valid &&
                          !(close & 2) && !(close & 4);
          if (ok) {
            ++found_all;
            s_found = found_all;
            a.used_row[s_n_used++] = row;
            a.used_sig[sig] = 1;
            a.author_count[au] += 1;
            a.out_pos[s_n_out + found_all - 1] = base + i;
            a.kept[m + found_all - 1] = i;  // the job's found list, behind the filter's (<= m entries each)
          }
          if (found_all >= need || s_prod >= n) s_stop = 1;
        }
      }
      __syncthreads();
      if (s_stop) break;
    }
    if (tid == 0) {
      const int found = s_found;
      if (found < need) {  // roll back (:294-312)
        for (int t = 0; t < found; ++t) {
          const int p = base + a.kept[m + t];
          a.used_sig[a.cand_sig[p]] = 0;
          int& cnt = a.author_count[a.cand_author[p]];
          cnt = max(0, cnt - 1);
        }
        s_n_used = used0;
        a.out_found[j] = 0;
        if (c.stop_on_failure) {
          *a.out_failed = j;
          s_stop = 2;
        }
      } else {
        for (int t = 0; t < found; ++t) a.path_row[s_n_path++] = a.cand_row[base + a.kept[m + t]];
        s_n_out += found;
        a.out_found[j] = found;
      }
    }
    __syncthreads();
    if (s_stop == 2) break;
  }
  // distances between consecutive songs of the path, the end song last
  const int np = s_n_path;
  for (int t = warp; t < np; t += warps) {
    const int64_t r0 = a.path_row[t], r1 = t + 1 < np ? a.path_row[t + 1] : a.end_row;
    const double dist = path_distance(a.X + r0 * a.d, a.X + r1 * a.d, a.d, c.path_metric, lane);
    if (lane == 0) a.out_dist[t] = dist;
  }
  if (tid == 0) {
    *a.n_used = s_n_used;
    *a.n_path = np;
  }
}


// ---------------------------------------------------------------- candidate post-processing helpers
// Direct distances (get_direct_distance, voyager_manager.py:99-140) between all pairs of `n` stored rows: what the
// radius walk (voyager_manager.py:1166-1258: score = 0.7 d(prev, cand) + 0.3 d(anchor, cand)) and the path logic
// recompute pair by pair with get_vector round trips.  One warp per pair (upper triangle), float64 accumulation.
__global__ void __launch_bounds__(256)
pairwise_direct_kernel(const float* __restrict__ X, int64_t N, int d, int metric, const int64_t* __restrict__ ids, int n,
                       float* __restrict__ out) {
  const int lane = threadIdx.x & 31;
  const int64_t pairs = (int64_t)n * (n + 1) / 2;
  for (int64_t pidx = (int64_t)blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5); pidx < pairs;
       pidx += (int64_t)gridDim.x * (blockDim.x >> 5)) {
    // pidx -> (i <= j) in the row-major upper triangle
    int i = (int)((2.0 * n + 1.0 - sqrt((2.0 * n + 1.0) * (2.0 * n + 1.0) - 8.0 * (double)pidx)) * 0.5);
    while ((int64_t)i * n - (int64_t)i * (i - 1) / 2 > pidx) --i;
    while ((int64_t)(i + 1) * n - (int64_t)(i + 1) * i / 2 <= pidx) ++i;
    const int j = i + (int)(pidx - ((int64_t)i * n - (int64_t)i * (i - 1) / 2));
    const int64_t ra = ids[i], rb = ids[j];
    float res = INFINITY;  // a missing vector: the reference returns +inf
    if (ra >= 0 && ra < N && rb >= 0 && rb < N) res = (float)direct_distance(X + ra * d, X + rb * d, d, metric, lane);
    if (lane == 0) {
      out[(int64_t)i * n + j] = res;
      out[(int64_t)j * n + i] = res;
    }
  }
}

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
extern "C" int64_t am_knn_size(const am_index* idx) { return idx ? idx->N : 0; }
extern "C" int am_knn_dim(const am_index* idx) { return idx ? idx->d : 0; }

extern "C" int am_knn_get_vector(const am_index* idx, int64_t id, float* out) {
  return am_knn_get_vectors(idx, &id, 1, out);
}

// one stream-ordered allocation carved into the temporaries of a query call (a call used to make nine cudaMallocAsync /
// cudaFreeAsync pairs: ~20 us of the ~110 us a single query took through the host API)
struct Arena {
  AsyncBuf<char> buf;
  size_t off = 0;
  static size_t pad(size_t bytes) { return round_up(bytes, 256); }
  int reserve(size_t bytes, cudaStream_t st) {
    off = 0;
    return buf.alloc(bytes, st);
  }
  template <class T>
  T* take(size_t count) {
    T* r = reinterpret_cast<T*>(buf.p + off);
    off += pad(count * sizeof(T));
    return r;
  }
};
// pinned host staging of the calling thread (query in, [ids | dist | overflow] out in ONE copy each way)
struct HostStage {
  void* p = nullptr;
  size_t cap = 0;
  ~HostStage() {
    if (p) cudaFreeHost(p);
  }
  int ensure(size_t bytes) {
    if (bytes <= cap) return AM_OK;
    if (p) cudaFreeHost(p);
    p = nullptr;
    cap = 0;
    cudaError_t e = cudaHostAlloc(&p, bytes, cudaHostAllocDefault);
    if (e != cudaSuccess) return cuda_fail(e, "cudaHostAlloc", __FILE__, __LINE__);
    cap = bytes;
    return AM_OK;
  }
};

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

// Runs a checked query (1 <= k <= N, nq >= 1) on device pointers.  host_ids / host_dist (optional): the host entry point's
// destinations -- results are copied there in the same stream round trip as the overflow flags (one synchronisation per
// pass instead of two; a single query is latency bound on exactly these).  merged != NULL: the caller laid out
// [ids | dist | overflow] contiguously from ids_dev (256-byte padded parts) and owns a pinned staging buffer of that size:
// results and flags travel in one device-to-host copy.  Scratch is allocated per call so the entry points are re-entrant.
static int knn_query_impl(const am_index* idx, const float* Q_dev, int nq, int k, int mode, int64_t* ids_dev, float* dist_dev,
                          cudaStream_t st, int64_t* host_ids, float* host_dist, int* overflow_dev = nullptr,
                          HostStage* merged = nullptr) {
  QueryPlan pl;
  AM_TRY(plan_query(idx, nq, k, mode, &pl));
  const int64_t N = idx->N;
  const int d = idx->d;
  const bool gemm = pl.scorer == Scorer::Bf16Gemm, small = pl.scorer == Scorer::Bf16Small;
  Arena arena;
  AM_TRY(arena.reserve(Arena::pad(pl.n_cm * 4) + Arena::pad(pl.n_s * 4) + Arena::pad(pl.n_qs * 4) +
                           Arena::pad((size_t)pl.qrows * 8) + Arena::pad((size_t)pl.qrows * 4) + Arena::pad(pl.n_qb * 2) +
                           Arena::pad(pl.n_qres * 4),
                       st));
  QueryBufs b;
  b.CM = arena.take<float>(pl.n_cm);
  b.S = arena.take<float>(pl.n_s);
  b.Qs = arena.take<float>(pl.n_qs);
  b.qnorm = arena.take<double>((size_t)pl.qrows);
  b.overflow = overflow_dev ? overflow_dev : arena.take<int>((size_t)pl.qrows);
  b.Qb = arena.take<__nv_bfloat16>(pl.n_qb);
  b.qres = arena.take<float>(pl.n_qres);
  SelectParams p = pl.sel;
  p.S = b.S;
  p.CM = b.CM;
  p.qnorm = b.qnorm;
  p.qres = (gemm || small) ? b.qres : nullptr;
  p.overflow = b.overflow;
  const size_t sel_smem = (size_t)kCandCap * (sizeof(double) + sizeof(int));
  std::vector<int> h_overflow;
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
    // 4. results and overflow flags to the host; flagged queries (all of them for the full sort) answered by the full sort
    h_overflow.assign(nc, 1);
    if (pl.select != Selection::FullSort) {
      if (merged && host_ids && nc == nq) {
        const size_t o_dist = Arena::pad((size_t)nq * k * 8), o_ovf = o_dist + Arena::pad((size_t)nq * k * 4);
        const size_t bytes = o_ovf + (size_t)nq * sizeof(int);
        AM_CUDA(cudaMemcpyAsync(merged->p, ids_dev, bytes, cudaMemcpyDeviceToHost, st));
        AM_CUDA(cudaStreamSynchronize(st));
        const char* h = static_cast<const char*>(merged->p);
        std::memcpy(host_ids, h, (size_t)nq * k * 8);
        std::memcpy(host_dist, h + o_dist, (size_t)nq * k * 4);
        std::memcpy(h_overflow.data(), h + o_ovf, (size_t)nq * sizeof(int));
      } else {
        AM_CUDA(cudaMemcpyAsync(h_overflow.data(), b.overflow, nc * sizeof(int), cudaMemcpyDeviceToHost, st));
        if (host_ids) {
          AM_CUDA(cudaMemcpyAsync(host_ids + (int64_t)q0 * k, p.ids, (size_t)nc * k * 8, cudaMemcpyDeviceToHost, st));
          AM_CUDA(cudaMemcpyAsync(host_dist + (int64_t)q0 * k, p.dist, (size_t)nc * k * 4, cudaMemcpyDeviceToHost, st));
        }
        AM_CUDA(cudaStreamSynchronize(st));
      }
    }
    bool any = false;
    for (int q = 0; q < nc; ++q)
      if (h_overflow[q]) {
        AM_TRY(full_sort_query(p, q, st));
        any = true;
      }
    if (any && host_ids) {  // rows answered by the exact full sort are copied again
      AM_CUDA(cudaMemcpyAsync(host_ids + (int64_t)q0 * k, p.ids, (size_t)nc * k * 8, cudaMemcpyDeviceToHost, st));
      AM_CUDA(cudaMemcpyAsync(host_dist + (int64_t)q0 * k, p.dist, (size_t)nc * k * 4, cudaMemcpyDeviceToHost, st));
      AM_CUDA(cudaStreamSynchronize(st));
    }
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
  return knn_query_impl(idx, Q_dev, nq, k, mode, ids_dev, dist_dev, (cudaStream_t)stream, nullptr, nullptr);
}

extern "C" int am_knn_query_ex(const am_index* idx, const float* Q, int nq, int k, int mode, int64_t* ids,
                               float* dist) {
  AM_CHECK(idx && (Q || nq == 0) && (ids || nq * (int64_t)k == 0) && (dist || nq * (int64_t)k == 0),
           "am_knn_query: NULL argument");
  AM_TRY(check_query(idx, nq, k));
  if (nq == 0 || k == 0) return AM_OK;
  AM_TRY(ensure_init());
  static thread_local Stream st;  // one stream per calling thread (Flask gthread x4): re-entrant
  AM_TRY(st.create());
  // device: [Q | ids | dist | overflow] in one allocation; host: one pinned staging buffer per thread -- the query goes up
  // and [ids | dist | overflow] comes back in one copy each (a single query: 3 host-side CUDA calls besides the launches)
  static thread_local HostStage pin;
  const size_t b_q = Arena::pad((size_t)nq * idx->d * 4), b_ids = Arena::pad((size_t)nq * k * 8), b_dist = Arena::pad((size_t)nq * k * 4);
  const size_t b_ovf = Arena::pad((size_t)nq * sizeof(int));
  const bool small = b_q + b_ids + b_dist + b_ovf <= ((size_t)2 << 20);   // (1.37 M vs 1.15 M QPS at 256 queries) beyond that the two extra host copies cost more than they save
  Arena blk;
  AM_TRY(blk.reserve(b_q + b_ids + b_dist + b_ovf, st.s));
  float* dQ = blk.take<float>((size_t)nq * idx->d);
  int64_t* dI = blk.take<int64_t>((size_t)nq * k);
  float* dD = blk.take<float>((size_t)nq * k);
  int* dO = blk.take<int>((size_t)nq);
  if (small) {
    AM_TRY(pin.ensure(std::max(b_q, b_ids + b_dist + b_ovf)));
    std::memcpy(pin.p, Q, (size_t)nq * idx->d * 4);
    AM_CUDA(cudaMemcpyAsync(dQ, pin.p, (size_t)nq * idx->d * 4, cudaMemcpyHostToDevice, st.s));
    return knn_query_impl(idx, dQ, nq, k, mode, dI, dD, st.s, ids, dist, dO, &pin);
  }
  AM_CUDA(cudaMemcpyAsync(dQ, Q, (size_t)nq * idx->d * 4, cudaMemcpyHostToDevice, st.s));
  return knn_query_impl(idx, dQ, nq, k, mode, dI, dD, st.s, ids, dist);
}

extern "C" int am_knn_query(const am_index* idx, const float* Q, int nq, int k, int64_t* ids, float* dist) {
  return am_knn_query_ex(idx, Q, nq, k, 0, ids, dist);
}

extern "C" int am_knn_filter_by_distance(const am_index* idx, const int64_t* ids, int n_lists, int n, float threshold,
                                         int lookback, int batch, unsigned char* keep) {
  AM_CHECK(idx && (ids || n_lists * n == 0) && (keep || n_lists * n == 0), "am_knn_filter_by_distance: NULL argument");
  AM_CHECK(n_lists >= 0 && n >= 0 && n <= kFilterCap, "am_knn_filter_by_distance: list length %d exceeds %d", n, kFilterCap);
  AM_CHECK(batch > 0, "am_knn_filter_by_distance: batch must be positive");
  if (n_lists == 0 || n == 0) return AM_OK;
  if (lookback <= 0) {  // the reference returns the list unchanged
    std::memset(keep, 1, (size_t)n_lists * n);
    return AM_OK;
  }
  AM_TRY(ensure_init());
  static thread_local Stream tst;  // re-entrant like am_knn_query
  AM_TRY(tst.create());
  cudaStream_t st = tst.s;
  AsyncBuf<int64_t> d_ids;
  AsyncBuf<unsigned char> d_keep;
  AM_TRY(d_ids.alloc((size_t)n_lists * n, st));
  AM_TRY(d_keep.alloc((size_t)n_lists * n, st));
  AM_CUDA(cudaMemcpyAsync(d_ids.p, ids, (size_t)n_lists * n * 8, cudaMemcpyHostToDevice, st));
  AM_LAUNCH(filter_by_distance_kernel, n_lists, kFilterThreads, 0, st, idx->X.p, idx->N, idx->d, idx->metric, d_ids.p, n,
            (double)threshold, lookback, batch, d_keep.p);
  AM_CUDA(cudaMemcpyAsync(keep, d_keep.p, (size_t)n_lists * n, cudaMemcpyDeviceToHost, st));
  AM_CUDA(cudaStreamSynchronize(st));
  return AM_OK;
}

extern "C" int am_knn_pairwise(const am_index* idx, const int64_t* ids, int n, float* out) {
  AM_CHECK(idx && (n == 0 || (ids && out)), "am_knn_pairwise: NULL argument");
  AM_CHECK(n >= 0 && n <= 8192, "am_knn_pairwise: n = %d out of range [0, 8192]", n);
  if (n == 0) return AM_OK;
  AM_TRY(ensure_init());
  static thread_local Stream tst;
  AM_TRY(tst.create());
  cudaStream_t st = tst.s;
  AsyncBuf<int64_t> d_ids;
  AsyncBuf<float> d_out;
  AM_TRY(d_ids.alloc((size_t)n, st));
  AM_TRY(d_out.alloc((size_t)n * n, st));
  AM_CUDA(cudaMemcpyAsync(d_ids.p, ids, (size_t)n * 8, cudaMemcpyHostToDevice, st));
  const int64_t pairs = (int64_t)n * (n + 1) / 2;
  const int grid = (int)std::max<int64_t>(1, std::min<int64_t>((pairs + 7) / 8, (int64_t)sm_count() * 8));
  AM_LAUNCH(pairwise_direct_kernel, grid, 256, 0, st, idx->X.p, idx->N, idx->d, idx->metric, d_ids.p, n, d_out.p);
  AM_CUDA(cudaMemcpyAsync(out, d_out.p, (size_t)n * n * 4, cudaMemcpyDeviceToHost, st));
  AM_CUDA(cudaStreamSynchronize(st));
  return AM_OK;
}

extern "C" int am_knn_get_vectors(const am_index* idx, const int64_t* ids, int n, float* out) {
  AM_CHECK(idx && (n == 0 || (ids && out)), "am_knn_get_vectors: NULL argument");
  AM_CHECK(n >= 0, "am_knn_get_vectors: negative count");
  if (n == 0) return AM_OK;
  for (int i = 0; i < n; ++i)
    AM_CHECK(ids[i] >= 0 && ids[i] < idx->N, "am_knn_get_vectors: id %lld out of range [0, %lld)", (long long)ids[i],
             (long long)idx->N);
  AM_TRY(ensure_init());
  static thread_local Stream tst;
  AM_TRY(tst.create());
  cudaStream_t st = tst.s;
  AsyncBuf<int64_t> d_ids;
  AsyncBuf<float> d_out;
  AM_TRY(d_ids.alloc((size_t)n, st));
  AM_TRY(d_out.alloc((size_t)n * idx->d, st));
  AM_CUDA(cudaMemcpyAsync(d_ids.p, ids, (size_t)n * 8, cudaMemcpyHostToDevice, st));
  const int grid = (int)std::max<int64_t>(1, std::min<int64_t>(((int64_t)n * idx->d + 255) / 256, (int64_t)sm_count() * 8));
  AM_LAUNCH(gather_rows_kernel, grid, 256, 0, st, idx->X.p, idx->N, idx->d, d_ids.p, n, d_out.p);
  AM_CUDA(cudaMemcpyAsync(out, d_out.p, (size_t)n * idx->d * 4, cudaMemcpyDeviceToHost, st));
  AM_CUDA(cudaStreamSynchronize(st));
  return AM_OK;
}

extern "C" int am_knn_radius_walk(const am_index* idx, const float* anchor, const int64_t* rows, const int32_t* artists,
                                  int n_cand, int n, int eliminate_duplicates, int max_songs_per_artist, int metric,
                                  int32_t* out_pos, double* out_dist, int32_t* out_count) {
  AM_CHECK(idx && anchor && out_count && (n_cand == 0 || (rows && artists)) && (n == 0 || (out_pos && out_dist)),
           "am_knn_radius_walk: NULL argument");
  AM_CHECK(n_cand >= 0 && n >= 0, "am_knn_radius_walk: negative size (n_cand = %d, n = %d)", n_cand, n);
  AM_CHECK(metric == kMetricCos || metric == kMetricL2, "am_knn_radius_walk: metric %d is not 0 (angular) or 1 (euclidean)",
           metric);
  *out_count = 0;
  if (n_cand == 0 || n == 0) return AM_OK;
  int n_art = 0;
  for (int i = 0; i < n_cand; ++i) {
    AM_CHECK(artists[i] >= -1, "am_knn_radius_walk: artist id %d at %d is below -1", artists[i], i);
    n_art = std::max(n_art, artists[i] + 1);
  }
  int64_t npad = 1;
  while (npad < n_cand) npad <<= 1;
  const int n_out = std::min(n, n_cand);
  AM_TRY(ensure_init());
  static thread_local Stream tst;  // re-entrant like am_knn_query
  AM_TRY(tst.create());
  cudaStream_t st = tst.s;
  // inputs [anchor | rows | artists] go up in one copy, outputs [count | pos | dist] come back in one
  const size_t b_anchor = Arena::pad((size_t)idx->d * 4), b_rows = Arena::pad((size_t)n_cand * 8),
               b_art = Arena::pad((size_t)n_cand * 4);
  const size_t b_cnt = Arena::pad(4), b_pos = Arena::pad((size_t)n_out * 4), b_dist = Arena::pad((size_t)n_out * 8);
  const size_t b_in = b_anchor + b_rows + b_art, b_out = b_cnt + b_pos + b_dist;
  const size_t b_scratch = Arena::pad((size_t)npad * 8) + Arena::pad((size_t)npad * 4) + 3 * Arena::pad((size_t)n_art * 4) +
                           Arena::pad((size_t)n_out * 4);
  static thread_local HostStage pin;
  AM_TRY(pin.ensure(std::max(b_in, b_out)));
  char* h = static_cast<char*>(pin.p);
  std::memcpy(h, anchor, (size_t)idx->d * 4);
  std::memcpy(h + b_anchor, rows, (size_t)n_cand * 8);
  std::memcpy(h + b_anchor + b_rows, artists, (size_t)n_cand * 4);
  Arena blk;
  AM_TRY(blk.reserve(b_in + b_out + b_scratch, st));
  float* d_anchor = blk.take<float>(idx->d);
  int64_t* d_rows = blk.take<int64_t>(n_cand);
  int32_t* d_art = blk.take<int32_t>(n_cand);
  int32_t* d_cnt = blk.take<int32_t>(1);
  int32_t* d_pos = blk.take<int32_t>(n_out);
  double* d_dist = blk.take<double>(n_out);
  unsigned long long* d_key = blk.take<unsigned long long>(npad);
  int* d_ord = blk.take<int>(npad);
  int* d_count = blk.take<int>(n_art);
  int* d_buckets = blk.take<int>(n_art);
  int* d_mark = blk.take<int>(n_art);
  int* d_playlist = blk.take<int>(n_out);
  AM_CUDA(cudaMemcpyAsync(d_anchor, h, b_in, cudaMemcpyHostToDevice, st));
  if (n_art > 0) {
    AM_CUDA(cudaMemsetAsync(d_count, 0, 2 * Arena::pad((size_t)n_art * 4), st));    // count, buckets
    AM_CUDA(cudaMemsetAsync(d_mark, 0xff, (size_t)n_art * 4, st));                  // mark = -1: no bucket yet
  }
  const int rules = eliminate_duplicates && max_songs_per_artist > 0;
  AM_LAUNCH(radius_walk_kernel, 1, kWalkThreads, 0, st, idx->X.p, idx->N, idx->d, metric, d_anchor, d_rows, d_art,
            n_cand, n_out, rules, max_songs_per_artist, npad, d_key, d_ord, d_count, d_buckets, d_mark, d_playlist, d_pos,
            d_dist, d_cnt);
  AM_CUDA(cudaMemcpyAsync(h, d_cnt, b_out, cudaMemcpyDeviceToHost, st));
  AM_CUDA(cudaStreamSynchronize(st));
  int32_t cnt = 0;
  std::memcpy(&cnt, h, 4);
  std::memcpy(out_pos, h + b_cnt, (size_t)cnt * 4);
  std::memcpy(out_dist, h + b_cnt + b_pos, (size_t)cnt * 8);
  *out_count = cnt;
  return AM_OK;
}

extern "C" int am_knn_song_path(const am_index* idx, const am_song_path_cfg* cfg, int n_jobs, const int32_t* job_off,
                                const int32_t* job_n, const int32_t* job_need, const int64_t* cand_rows,
                                const int32_t* cand_sig, const int32_t* cand_author, const int32_t* cand_author_raw,
                                int n_sig, int n_author, int64_t* used_rows, int32_t* n_used, unsigned char* used_sig,
                                int32_t* author_count, int64_t* path_rows, int32_t* n_path, int64_t end_row,
                                int32_t* out_found, int32_t* out_pos, int32_t* out_failed, double* out_dist) {
  AM_CHECK(idx && cfg && n_used && n_path && out_failed && (n_jobs == 0 || (job_off && job_n && job_need && out_found)),
           "am_knn_song_path: NULL argument");
  AM_CHECK(n_jobs >= 0 && n_sig >= 0 && n_author >= 0 && *n_used >= 0 && *n_path >= 1,
           "am_knn_song_path: negative size, or no start song in the path");
  AM_CHECK(cfg->voyager_metric == kMetricCos || cfg->voyager_metric == kMetricL2, "am_knn_song_path: voyager_metric %d",
           cfg->voyager_metric);
  AM_CHECK(cfg->path_metric == kMetricCos || cfg->path_metric == kMetricL2, "am_knn_song_path: path_metric %d",
           cfg->path_metric);
  AM_CHECK(cfg->filter_batch > 0, "am_knn_song_path: filter_batch must be positive");
  AM_CHECK(end_row >= 0 && end_row < idx->N, "am_knn_song_path: end row %lld out of range", (long long)end_row);
  AM_CHECK(n_jobs == 0 || job_off[0] == 0, "am_knn_song_path: job_off[0] must be 0");
  int64_t total_need = 0;
  int max_m = 0;
  for (int j = 0; j < n_jobs; ++j) {
    AM_CHECK(job_off[j + 1] >= job_off[j] && job_n[j] >= 1 && job_need[j] >= 1,
             "am_knn_song_path: job %d: bad range, n or num_to_find", j);
    total_need += job_need[j];
    max_m = std::max(max_m, job_off[j + 1] - job_off[j]);
  }
  const int n_cand = n_jobs ? job_off[n_jobs] : 0;
  AM_CHECK(n_cand == 0 || (cand_rows && cand_sig && cand_author && cand_author_raw), "am_knn_song_path: NULL candidates");
  AM_CHECK(total_need == 0 || out_pos, "am_knn_song_path: NULL out_pos");
  int n_raw = 0;
  for (int i = 0; i < n_cand; ++i) {
    AM_CHECK(cand_sig[i] >= -1 && cand_sig[i] < n_sig && cand_author[i] >= 0 && cand_author[i] < n_author &&
                 cand_author_raw[i] >= -1,
             "am_knn_song_path: candidate %d has a key out of range", i);
    n_raw = std::max(n_raw, cand_author_raw[i] + 1);
  }
  const int nu = *n_used, np = *n_path;
  for (int t = 0; t < np; ++t)
    AM_CHECK(path_rows[t] >= 0 && path_rows[t] < idx->N, "am_knn_song_path: path row %d out of range", t);
  const int64_t cap_used = nu + total_need, cap_path = np + total_need;
  AM_TRY(ensure_init());
  static thread_local Stream tst;  // re-entrant like am_knn_query
  AM_TRY(tst.create());
  cudaStream_t st = tst.s;
  using A = Arena;
  // [inputs | state | outputs | scratch]: inputs and state go up in one copy, state and outputs come back in one
  const size_t b_in = A::pad((n_jobs + 1) * 4) + 2 * A::pad(n_jobs * 4) + A::pad((size_t)n_cand * 8) + 3 * A::pad((size_t)n_cand * 4);
  const size_t b_state = A::pad(16) + A::pad(cap_used * 8) + A::pad(cap_path * 8) + A::pad((size_t)n_author * 4) + A::pad(n_sig);
  const size_t b_out = A::pad(n_jobs * 4) + A::pad(total_need * 4) + A::pad(cap_path * 8);
  const size_t b_scratch = A::pad((size_t)n_sig * 4) + 2 * A::pad((size_t)n_raw * 4) + A::pad((size_t)2 * max_m * 4);
  static thread_local HostStage pin;
  AM_TRY(pin.ensure(b_in + b_state + b_out));
  Arena blk;
  AM_TRY(blk.reserve(b_in + b_state + b_out + b_scratch, st));
  char* const d0 = blk.buf.p;
  int32_t* d_off = blk.take<int32_t>(n_jobs + 1);
  int32_t* d_n = blk.take<int32_t>(n_jobs);
  int32_t* d_need = blk.take<int32_t>(n_jobs);
  int64_t* d_row = blk.take<int64_t>(n_cand);
  int32_t* d_sig = blk.take<int32_t>(n_cand);
  int32_t* d_au = blk.take<int32_t>(n_cand);
  int32_t* d_raw = blk.take<int32_t>(n_cand);
  int32_t* d_hdr = blk.take<int32_t>(4);  // n_used, n_path, failed
  int64_t* d_used = blk.take<int64_t>(cap_used);
  int64_t* d_path = blk.take<int64_t>(cap_path);
  int32_t* d_count = blk.take<int32_t>(n_author);
  unsigned char* d_usig = blk.take<unsigned char>(n_sig);
  int32_t* d_found = blk.take<int32_t>(n_jobs);
  int32_t* d_pos = blk.take<int32_t>(total_need);
  double* d_dist = blk.take<double>(cap_path);
  int32_t* d_seen = blk.take<int32_t>(n_sig);
  int32_t* d_mark = blk.take<int32_t>(n_raw);
  int32_t* d_rcount = blk.take<int32_t>(n_raw);
  int32_t* d_kept = blk.take<int32_t>((size_t)2 * max_m);
  char* h = static_cast<char*>(pin.p);
  auto put = [&](const void* src, const void* dev, size_t bytes) {
    if (bytes) std::memcpy(h + (static_cast<const char*>(dev) - d0), src, bytes);
  };
  put(job_off, d_off, (n_jobs ? n_jobs + 1 : 0) * 4);
  put(job_n, d_n, n_jobs * 4);
  put(job_need, d_need, n_jobs * 4);
  put(cand_rows, d_row, (size_t)n_cand * 8);
  put(cand_sig, d_sig, (size_t)n_cand * 4);
  put(cand_author, d_au, (size_t)n_cand * 4);
  put(cand_author_raw, d_raw, (size_t)n_cand * 4);
  const int32_t hdr[4] = {nu, np, -1, 0};
  put(hdr, d_hdr, 16);
  put(used_rows, d_used, (size_t)nu * 8);
  put(path_rows, d_path, (size_t)np * 8);
  put(author_count, d_count, (size_t)n_author * 4);
  put(used_sig, d_usig, (size_t)n_sig);
  AM_CUDA(cudaMemcpyAsync(d0, h, b_in + b_state, cudaMemcpyHostToDevice, st));
  AM_CUDA(cudaMemsetAsync(d_seen, 0xff, A::pad((size_t)n_sig * 4) + A::pad((size_t)n_raw * 4), st));  // seen, raw_mark: -1
  SongPathArgs a{idx->X.p, idx->N, idx->d, n_jobs, d_off, d_n, d_need, d_row, d_sig, d_au, d_raw, d_used, d_hdr, d_usig,
                 d_count, d_path, d_hdr + 1, end_row, *cfg, d_seen, d_mark, d_rcount, d_kept, d_found, d_pos, d_hdr + 2,
                 d_dist};
  AM_LAUNCH(song_path_kernel, 1, kPathThreads, 0, st, a);
  char* const s0 = reinterpret_cast<char*>(d_hdr);
  AM_CUDA(cudaMemcpyAsync(h + (s0 - d0), s0, b_state + b_out, cudaMemcpyDeviceToHost, st));
  AM_CUDA(cudaStreamSynchronize(st));
  auto get = [&](void* dst, const void* dev, size_t bytes) {
    if (bytes) std::memcpy(dst, h + (static_cast<const char*>(dev) - d0), bytes);
  };
  int32_t out_hdr[4];
  get(out_hdr, d_hdr, 16);
  int64_t taken = 0;
  get(out_found, d_found, n_jobs * 4);
  for (int j = 0; j < n_jobs; ++j) taken += out_found[j];
  AM_CHECK(out_hdr[0] >= nu && out_hdr[0] <= cap_used && out_hdr[1] >= np && out_hdr[1] <= cap_path && taken <= total_need,
           "am_knn_song_path: inconsistent result (used %d of %lld, path %d of %lld, taken %lld of %lld)", out_hdr[0],
           (long long)cap_used, out_hdr[1], (long long)cap_path, (long long)taken, (long long)total_need);
  *n_used = out_hdr[0];
  *n_path = out_hdr[1];
  *out_failed = out_hdr[2];
  get(out_pos, d_pos, taken * 4);
  get(used_rows, d_used, (size_t)out_hdr[0] * 8);
  get(path_rows, d_path, (size_t)out_hdr[1] * 8);
  get(author_count, d_count, (size_t)n_author * 4);
  get(used_sig, d_usig, (size_t)n_sig);
  get(out_dist, d_dist, (size_t)out_hdr[1] * 8);
  return AM_OK;
}
