// Kernels of the graph-driven encoder path that are NOT part of the PhiNet fast path: first convolution with
// an arbitrary small kernel, depthwise K x K with any activation, squeeze-excite, and the head's row program.
// Included by encoder.cu and depthwise.cu (hence static kernels).  Layout conventions as in encoder.cu (NHWC bf16, channels padded to 16).
#pragma once

#include "common.cuh"
#include "model_spec.cuh"

namespace am {

__device__ __forceinline__ float apply_act(int kind, float v) {
  switch (kind) {
    case kActRelu6: return fminf(fmaxf(v, 0.f), 6.f);
    case kActRelu: return fmaxf(v, 0.f);
    case kActHardSwish: return v * fminf(fmaxf(v * (1.0f / 6.0f) + 0.5f, 0.f), 1.f);
    case kActGelu: return 0.5f * v * (1.0f + erff(v * 0.70710678118654752440f));
    case kActSigmoid: return 1.0f / (1.0f + expf(-v));
    case kActHardSigmoid: return fminf(fmaxf(v * (1.0f / 6.0f) + 0.5f, 0.f), 1.f);
    case kActTanh: return tanhf(v);
    default: return v;
  }
}

__device__ __forceinline__ uint4 pack8_bf16(const float (&o)[8]) {
  uint4 pk;
  __nv_bfloat162 t;
  t = __floats2bfloat162_rn(o[0], o[1]); pk.x = *reinterpret_cast<uint32_t*>(&t);
  t = __floats2bfloat162_rn(o[2], o[3]); pk.y = *reinterpret_cast<uint32_t*>(&t);
  t = __floats2bfloat162_rn(o[4], o[5]); pk.z = *reinterpret_cast<uint32_t*>(&t);
  t = __floats2bfloat162_rn(o[6], o[7]); pk.w = *reinterpret_cast<uint32_t*>(&t);
  return pk;
}

// First convolution, Cin = 1: mel f32 [B, n_mels, T] -> NHWC bf16 [B, Ho, Wo, Cp].
// h_is_time: image (H, W) = (time, mel) (PhiNet view) else (mel, time) (plain NCHW view of the input).
// Per-mel affine (bn0) applied to in-range samples; padding contributes exact zeros.
// One thread = one output pixel x one 8-channel group; weights [kh*kw, Cp] + bias staged in shared memory.
static __global__ void __launch_bounds__(256)
conv_first_kernel(const float* __restrict__ mel, int B, int n_mels, int T, int Ho, int Wo, int kh, int kw, int stride,
                  int pad_t, int pad_l, int h_is_time, const float* __restrict__ sc, const float* __restrict__ sh,
                  const float* __restrict__ w /* [kh*kw, cp] */, const float* __restrict__ bias, int cp, int act,
                  __nv_bfloat16* __restrict__ out) {
  extern __shared__ float s_w[];  // [(kh*kw + 1) * cp]
  const int taps = kh * kw;
  for (int i = threadIdx.x; i < (taps + 1) * cp; i += blockDim.x) s_w[i] = i < taps * cp ? w[i] : bias[i - taps * cp];
  __syncthreads();
  const int groups = cp >> 3;
  const int64_t total = (int64_t)B * Ho * Wo * groups;
  const int H = h_is_time ? T : n_mels, W = h_is_time ? n_mels : T;
  for (int64_t idx = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; idx < total; idx += (int64_t)gridDim.x * blockDim.x) {
    const int g = (int)(idx % groups);
    int64_t r = idx / groups;
    const int wo = (int)(r % Wo);
    r /= Wo;
    const int ho = (int)(r % Ho);
    const int b = (int)(r / Ho);
    const float* m = mel + (int64_t)b * n_mels * T;
    float o[8];
#pragma unroll
    for (int e = 0; e < 8; ++e) o[e] = s_w[taps * cp + g * 8 + e];
    for (int dy = 0; dy < kh; ++dy) {
      const int h = ho * stride + dy - pad_t;
      if (h < 0 || h >= H) continue;
      for (int dx = 0; dx < kw; ++dx) {
        const int x = wo * stride + dx - pad_l;
        if (x < 0 || x >= W) continue;
        const int mi = h_is_time ? x : h, ti = h_is_time ? h : x;
        float v = __ldg(&m[(int64_t)mi * T + ti]);
        if (sc) v = fmaf(v, __ldg(&sc[mi]), __ldg(&sh[mi]));
        const float* wt = s_w + (dy * kw + dx) * cp + g * 8;
#pragma unroll
        for (int e = 0; e < 8; ++e) o[e] = fmaf(v, wt[e], o[e]);
      }
    }
#pragma unroll
    for (int e = 0; e < 8; ++e) o[e] = apply_act(act, o[e]);
    *reinterpret_cast<uint4*>(out + (((int64_t)b * Ho + ho) * Wo + wo) * cp + g * 8) = pack8_bf16(o);
  }
}

// Depthwise K x K (K odd, <= 7), stride 1 / 2, arbitrary zero padding, folded BN bias, any trunk activation.
// fp32 accumulation.  One thread = one output pixel x one 8-channel group (coalesced 16-byte accesses).
static __global__ void __launch_bounds__(256)
depthwise_generic_kernel(const __nv_bfloat16* __restrict__ in, int B, int H, int W, int cp, int Ho, int Wo, int k,
                         int stride, int pad_t, int pad_l, const float* __restrict__ w /* [k*k, cp] */,
                         const float* __restrict__ bias, int act, __nv_bfloat16* __restrict__ out) {
  const int groups = cp >> 3;
  const int64_t total = (int64_t)B * Ho * Wo * groups;
  for (int64_t idx = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; idx < total; idx += (int64_t)gridDim.x * blockDim.x) {
    const int g = (int)(idx % groups);
    int64_t r = idx / groups;
    const int wo = (int)(r % Wo);
    r /= Wo;
    const int ho = (int)(r % Ho);
    const int b = (int)(r / Ho);
    const int c0 = g * 8;
    float o[8];
    {
      const float4 b0 = __ldg(reinterpret_cast<const float4*>(bias + c0));
      const float4 b1 = __ldg(reinterpret_cast<const float4*>(bias + c0 + 4));
      o[0] = b0.x; o[1] = b0.y; o[2] = b0.z; o[3] = b0.w; o[4] = b1.x; o[5] = b1.y; o[6] = b1.z; o[7] = b1.w;
    }
    for (int dy = 0; dy < k; ++dy) {
      const int h = ho * stride + dy - pad_t;
      if (h < 0 || h >= H) continue;
      for (int dx = 0; dx < k; ++dx) {
        const int x = wo * stride + dx - pad_l;
        if (x < 0 || x >= W) continue;
        const uint4 raw = __ldg(reinterpret_cast<const uint4*>(in + (((int64_t)b * H + h) * W + x) * cp + c0));
        const __nv_bfloat162* h2 = reinterpret_cast<const __nv_bfloat162*>(&raw);
        const float* wt = w + (dy * k + dx) * cp + c0;
        const float4 w0 = __ldg(reinterpret_cast<const float4*>(wt)), w1 = __ldg(reinterpret_cast<const float4*>(wt + 4));
        const float2 p0 = __bfloat1622float2(h2[0]), p1 = __bfloat1622float2(h2[1]), p2 = __bfloat1622float2(h2[2]),
                     p3 = __bfloat1622float2(h2[3]);
        o[0] = fmaf(p0.x, w0.x, o[0]); o[1] = fmaf(p0.y, w0.y, o[1]); o[2] = fmaf(p1.x, w0.z, o[2]); o[3] = fmaf(p1.y, w0.w, o[3]);
        o[4] = fmaf(p2.x, w1.x, o[4]); o[5] = fmaf(p2.y, w1.y, o[5]); o[6] = fmaf(p3.x, w1.z, o[6]); o[7] = fmaf(p3.y, w1.w, o[7]);
      }
    }
#pragma unroll
    for (int e = 0; e < 8; ++e) o[e] = apply_act(act, o[e]);
    *reinterpret_cast<uint4*>(out + (((int64_t)b * Ho + ho) * Wo + wo) * cp + c0) = pack8_bf16(o);
  }
}

// squeeze: mean over (H, W) of NHWC bf16 -> f32 [B, C].  grid (ceil(C / 64), B), 256 threads: 64 channels x 4 pixel lanes.
static __global__ void __launch_bounds__(256)
channel_mean_kernel(const __nv_bfloat16* __restrict__ in, int HW, int cp, int C, float* __restrict__ out) {
  __shared__ float s_part[4][64];
  const int c = blockIdx.x * 64 + (threadIdx.x & 63), lane = threadIdx.x >> 6, b = blockIdx.y;
  float acc = 0.f;
  if (c < C)
    for (int p = lane; p < HW; p += 4) acc += __bfloat162float(in[((int64_t)b * HW + p) * cp + c]);
  s_part[lane][threadIdx.x & 63] = acc;
  __syncthreads();
  if (lane == 0 && c < C)
    out[(int64_t)b * C + c] = (s_part[0][threadIdx.x] + s_part[1][threadIdx.x] + s_part[2][threadIdx.x] + s_part[3][threadIdx.x]) / (float)HW;
}

// the two tiny fully connected layers of a squeeze-excite gate, one CTA per window:
// gate[b, c] = gate_act( W2 . inner_act( W1 . mean[b] + b1 ) + b2 )
static __global__ void __launch_bounds__(256)
se_gate_kernel(const float* __restrict__ mean, int C, int Cm, const float* __restrict__ w1, const float* __restrict__ b1,
               const float* __restrict__ w2, const float* __restrict__ b2, int inner_act, int gate_act,
               float* __restrict__ gate) {
  extern __shared__ float s_se[];  // [C] mean, [Cm] hidden
  float* s_m = s_se;
  float* s_h = s_se + C;
  const int b = blockIdx.x, warp = threadIdx.x >> 5, lane = threadIdx.x & 31, nw = blockDim.x >> 5;
  for (int i = threadIdx.x; i < C; i += blockDim.x) s_m[i] = mean[(int64_t)b * C + i];
  __syncthreads();
  for (int j = warp; j < Cm; j += nw) {
    float acc = 0.f;
    for (int i = lane; i < C; i += 32) acc = fmaf(w1[(int64_t)j * C + i], s_m[i], acc);
    acc = warp_sum(acc);
    if (lane == 0) s_h[j] = apply_act(inner_act, acc + b1[j]);
  }
  __syncthreads();
  for (int c = warp; c < C; c += nw) {
    float acc = 0.f;
    for (int j = lane; j < Cm; j += 32) acc = fmaf(w2[(int64_t)c * Cm + j], s_h[j], acc);
    acc = warp_sum(acc);
    if (lane == 0) gate[(int64_t)b * C + c] = apply_act(gate_act, acc + b2[c]);
  }
}

// excite: y[b, p, c] = x[b, p, c] * gate[b, c]   (8 channels per thread)
static __global__ void __launch_bounds__(256)
se_scale_kernel(const __nv_bfloat16* __restrict__ in, int64_t HW, int cp, int C, const float* __restrict__ gate, int B,
                __nv_bfloat16* __restrict__ out) {
  const int groups = cp >> 3;
  const int64_t total = (int64_t)B * HW * groups;
  for (int64_t idx = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; idx < total; idx += (int64_t)gridDim.x * blockDim.x) {
    const int g = (int)(idx % groups);
    const int64_t pix = idx / groups;
    const int b = (int)(pix / HW);
    const uint4 raw = *reinterpret_cast<const uint4*>(in + pix * cp + g * 8);
    const __nv_bfloat162* h2 = reinterpret_cast<const __nv_bfloat162*>(&raw);
    float o[8];
#pragma unroll
    for (int q = 0; q < 4; ++q) {
      const float2 f = __bfloat1622float2(h2[q]);
      const int c = g * 8 + 2 * q;
      o[2 * q] = c < C ? f.x * gate[(int64_t)b * C + c] : 0.f;
      o[2 * q + 1] = c + 1 < C ? f.y * gate[(int64_t)b * C + c + 1] : 0.f;
    }
    *reinterpret_cast<uint4*>(out + pix * cp + g * 8) = pack8_bf16(o);
  }
}

// ---------------------------------------------------------------- head row program (f32 [n, dim])
static __global__ void vec_unary_kernel(const float* __restrict__ x, int64_t n, int act, float* __restrict__ y) {
  for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (int64_t)gridDim.x * blockDim.x)
    y[i] = apply_act(act, x[i]);
}
static __global__ void vec_add_kernel(const float* __restrict__ a, const float* __restrict__ b, int64_t n, float* __restrict__ y) {
  for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (int64_t)gridDim.x * blockDim.x) y[i] = a[i] + b[i];
}
static __global__ void vec_affine_kernel(const float* __restrict__ x, int64_t n, int dim, const float* __restrict__ scale,
                                  const float* __restrict__ shift, float* __restrict__ y) {
  for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (int64_t)gridDim.x * blockDim.x) {
    const int c = (int)(i % dim);
    float v = x[i];
    if (scale) v *= scale[c];
    if (shift) v += shift[c];
    y[i] = v;
  }
}

__device__ __forceinline__ float block_sum_256(float v, float* s_red, float* s_out) {
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  v = warp_sum(v);
  if (lane == 0) s_red[warp] = v;
  __syncthreads();
  if (warp == 0) {
    float t = lane < (int)(blockDim.x >> 5) ? s_red[lane] : 0.f;
    t = warp_sum(t);
    if (lane == 0) *s_out = t;
  }
  __syncthreads();
  const float r = *s_out;
  __syncthreads();
  return r;
}

// one CTA per row: y = (x - mean) * rsqrt(var + eps) * g + b
static __global__ void __launch_bounds__(256)
vec_layernorm_kernel(const float* __restrict__ x, int E, const float* __restrict__ g, const float* __restrict__ bt, float eps,
                     float* __restrict__ y) {
  __shared__ float s_red[32];
  __shared__ float s_out;
  const float* a = x + (int64_t)blockIdx.x * E;
  float loc = 0.f;
  for (int i = threadIdx.x; i < E; i += blockDim.x) loc += a[i];
  const float mean = block_sum_256(loc, s_red, &s_out) / (float)E;
  loc = 0.f;
  for (int i = threadIdx.x; i < E; i += blockDim.x) {
    const float d = a[i] - mean;
    loc = fmaf(d, d, loc);
  }
  const float rstd = rsqrtf(block_sum_256(loc, s_red, &s_out) / (float)E + eps);
  for (int i = threadIdx.x; i < E; i += blockDim.x) y[(int64_t)blockIdx.x * E + i] = (a[i] - mean) * rstd * g[i] + bt[i];
}

// one CTA per row: y = x / max(||x||, eps)
static __global__ void __launch_bounds__(256)
vec_l2norm_kernel(const float* __restrict__ x, int E, float eps, float* __restrict__ y) {
  __shared__ float s_red[32];
  __shared__ float s_out;
  const float* a = x + (int64_t)blockIdx.x * E;
  float loc = 0.f;
  for (int i = threadIdx.x; i < E; i += blockDim.x) loc = fmaf(a[i], a[i], loc);
  const float nrm = fmaxf(sqrtf(block_sum_256(loc, s_red, &s_out)), eps);
  for (int i = threadIdx.x; i < E; i += blockDim.x) y[(int64_t)blockIdx.x * E + i] = a[i] / nrm;
}

}  // namespace am
