// The 3x3 / pad 1 / ReLU6 depthwise of the layer-by-layer path (depthwise.cuh): the two packed-fp16 kernels, the
// overflow test that admits a layer to them, and the launch that picks a kernel from the shape.
#include "depthwise.cuh"

#include <cuda_fp16.h>

#include <cmath>

#include "encoder_generic.cuh"

namespace am {

// depthwise 3x3, pad 1, stride s, folded BN, ReLU6.  NHWC bf16.
// A thread owns 8 channels (one 16-byte vector) of a vertical strip of kDwRows output rows at one
// output column: the 9 x 8 folded weights live in registers, each input row (3 taps) is loaded once
// and scattered into the (up to three) output rows it feeds, so the input is read ~(s*R+2)/R times
// from L1/L2 instead of 9.  Consecutive threads = consecutive channel groups (coalesced 16 B).
constexpr int kDwRows = 4;
constexpr int kDwThreads = 128;

__device__ __forceinline__ void dw_load_row(const __nv_bfloat16* base, int h, int H, int W, int cp, int x0,
                                            uint4 (&raw)[3]) {
#pragma unroll
  for (int dx = 0; dx < 3; ++dx) {
    const int x = x0 + dx;
    raw[dx] = make_uint4(0u, 0u, 0u, 0u);
    if (h >= 0 && h < H && x >= 0 && x < W)
      raw[dx] = __ldg(reinterpret_cast<const uint4*>(base + ((int64_t)h * W + x) * cp));
  }
}

template <int kStride>
__global__ void __launch_bounds__(kDwThreads, 3)
depthwise_kernel(const __nv_bfloat16* __restrict__ in, int B, int H, int W, int cp, int Ho, int Wo,
                 const float* __restrict__ w /* [9, cp] */, const float* __restrict__ bias,
                 __nv_bfloat16* __restrict__ out) {
  const int groups = cp >> 3;
  const int strips = (Ho + kDwRows - 1) / kDwRows;
  const int64_t total = (int64_t)B * strips * Wo * groups;
  const int64_t idx = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (idx >= total) return;
  const int g = (int)(idx % groups);
  int64_t r = idx / groups;
  const int wo = (int)(r % Wo);
  r /= Wo;
  const int strip = (int)(r % strips);
  const int b = (int)(r / strips);
  const int c0 = g * 8;
  const int ho0 = strip * kDwRows;
  const int nrows = min(kDwRows, Ho - ho0);

  // packed fp16 arithmetic (HFMA2): inputs are post-ReLU6
  // (|x| <= 6, bf16 -> fp16 is exact there), 9 taps; half the FMAs and half the weight registers of fp32
  __half2 wt[9][4];
#pragma unroll
  for (int t = 0; t < 9; ++t) {
    const float4 w0 = __ldg(reinterpret_cast<const float4*>(w + t * cp + c0));
    const float4 w1 = __ldg(reinterpret_cast<const float4*>(w + t * cp + c0 + 4));
    wt[t][0] = __floats2half2_rn(w0.x, w0.y);
    wt[t][1] = __floats2half2_rn(w0.z, w0.w);
    wt[t][2] = __floats2half2_rn(w1.x, w1.y);
    wt[t][3] = __floats2half2_rn(w1.z, w1.w);
  }
  __half2 acc[kDwRows][4];
  {
    const float4 b0 = __ldg(reinterpret_cast<const float4*>(bias + c0));
    const float4 b1 = __ldg(reinterpret_cast<const float4*>(bias + c0 + 4));
#pragma unroll
    for (int i = 0; i < kDwRows; ++i) {
      acc[i][0] = __floats2half2_rn(b0.x, b0.y);
      acc[i][1] = __floats2half2_rn(b0.z, b0.w);
      acc[i][2] = __floats2half2_rn(b1.x, b1.y);
      acc[i][3] = __floats2half2_rn(b1.z, b1.w);
    }
  }
  const int x0 = wo * kStride - 1;
  const int h_first = ho0 * kStride - 1;
  constexpr int kInRows = (kDwRows - 1) * kStride + 3;
  const __nv_bfloat16* base = in + ((int64_t)b * H) * W * cp + c0;
  // software pipeline: the loads of input row ir+1 are in flight while row ir is consumed
  uint4 cur[3], nxt[3];
  dw_load_row(base, h_first, H, W, cp, x0, cur);
#pragma unroll
  for (int ir = 0; ir < kInRows; ++ir) {
    if (ir + 1 < kInRows) dw_load_row(base, h_first + ir + 1, H, W, cp, x0, nxt);
    __half2 px[3][4];
#pragma unroll
    for (int dx = 0; dx < 3; ++dx) {
      const __nv_bfloat162* h2 = reinterpret_cast<const __nv_bfloat162*>(&cur[dx]);
#pragma unroll
      for (int q = 0; q < 4; ++q) px[dx][q] = __float22half2_rn(__bfloat1622float2(h2[q]));
    }
    // input row ir feeds output row o with kernel row dy = ir - o*stride, 0 <= dy < 3
#pragma unroll
    for (int dy = 0; dy < 3; ++dy) {
      const int num = ir - dy;
      if (num < 0 || (num % kStride) != 0) continue;
      const int o = num / kStride;
      if (o >= kDwRows) continue;
#pragma unroll
      for (int dx = 0; dx < 3; ++dx)
#pragma unroll
        for (int j = 0; j < 4; ++j) acc[o][j] = __hfma2(px[dx][j], wt[dy * 3 + dx][j], acc[o][j]);
    }
#pragma unroll
    for (int dx = 0; dx < 3; ++dx) cur[dx] = nxt[dx];
  }
  const __half2 h_zero = __floats2half2_rn(0.f, 0.f), h_six = __floats2half2_rn(6.f, 6.f);
#pragma unroll
  for (int o = 0; o < kDwRows; ++o) {
    if (o < nrows) {
      uint4 pk;
      uint32_t* pw = reinterpret_cast<uint32_t*>(&pk);
#pragma unroll
      for (int j = 0; j < 4; ++j) {
        const float2 f = __half22float2(__hmin2(__hmax2(acc[o][j], h_zero), h_six));
        const __nv_bfloat162 t = __floats2bfloat162_rn(f.x, f.y);
        pw[j] = *reinterpret_cast<const uint32_t*>(&t);
      }
      *reinterpret_cast<uint4*>(out + ((((int64_t)b * Ho + ho0 + o) * Wo + wo) * cp) + c0) = pk;
    }
  }
}

// Row-sliding depthwise 3x3 for the NARROW late maps (W <= 16: blocks 6-9).  A thread owns 8 channels of a strip
// of 2 output rows and walks the output columns, keeping a 3-column window of the input rows in registers: every
// input pixel is loaded ONCE (the strip kernel above loads it from three threads -- in three different CTAs once
// the channel count exceeds the CTA size -- and those re-reads went to L2).  Packed fp16 arithmetic as above.
constexpr int kDwRowR = 2;

template <int kStride>
__global__ void __launch_bounds__(kDwThreads, 3)
depthwise_row_kernel(const __nv_bfloat16* __restrict__ in, int B, int H, int W, int cp, int Ho, int Wo,
                     const float* __restrict__ w /* [9, cp] */, const float* __restrict__ bias,
                     __nv_bfloat16* __restrict__ out) {
  constexpr int IR = (kDwRowR - 1) * kStride + 3;  // input rows feeding the strip
  const int groups = cp >> 3;
  const int strips = (Ho + kDwRowR - 1) / kDwRowR;
  const int64_t total = (int64_t)B * strips * groups;
  const int64_t idx = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (idx >= total) return;
  const int g = (int)(idx % groups);
  const int64_t r = idx / groups;
  const int strip = (int)(r % strips);
  const int b = (int)(r / strips);
  const int c0 = g * 8;
  const int ho0 = strip * kDwRowR;
  __half2 wt[9][4], bv[4];
#pragma unroll
  for (int t = 0; t < 9; ++t) {
    const float4 w0 = __ldg(reinterpret_cast<const float4*>(w + t * cp + c0));
    const float4 w1 = __ldg(reinterpret_cast<const float4*>(w + t * cp + c0 + 4));
    wt[t][0] = __floats2half2_rn(w0.x, w0.y);
    wt[t][1] = __floats2half2_rn(w0.z, w0.w);
    wt[t][2] = __floats2half2_rn(w1.x, w1.y);
    wt[t][3] = __floats2half2_rn(w1.z, w1.w);
  }
  {
    const float4 b0 = __ldg(reinterpret_cast<const float4*>(bias + c0));
    const float4 b1 = __ldg(reinterpret_cast<const float4*>(bias + c0 + 4));
    bv[0] = __floats2half2_rn(b0.x, b0.y);
    bv[1] = __floats2half2_rn(b0.z, b0.w);
    bv[2] = __floats2half2_rn(b1.x, b1.y);
    bv[3] = __floats2half2_rn(b1.z, b1.w);
  }
  const int h_first = ho0 * kStride - 1;
  const __nv_bfloat16* base = in + ((int64_t)b * H) * W * cp + c0;
  auto load_raw = [&](int x, uint4 (&raw)[IR]) {
#pragma unroll
    for (int ir = 0; ir < IR; ++ir) {
      const int h = h_first + ir;
      raw[ir] = make_uint4(0u, 0u, 0u, 0u);
      if (h >= 0 && h < H && x >= 0 && x < W) raw[ir] = __ldg(reinterpret_cast<const uint4*>(base + ((int64_t)h * W + x) * cp));
    }
  };
  auto unpack = [&](const uint4 (&raw)[IR], __half2 (&col)[IR][4]) {
#pragma unroll
    for (int ir = 0; ir < IR; ++ir) {
      const __nv_bfloat162* h2 = reinterpret_cast<const __nv_bfloat162*>(&raw[ir]);
#pragma unroll
      for (int q = 0; q < 4; ++q) col[ir][q] = __float22half2_rn(__bfloat1622float2(h2[q]));
    }
  };
  const __half2 h_zero = __floats2half2_rn(0.f, 0.f), h_six = __floats2half2_rn(6.f, 6.f);
  __half2 ca[IR][4], cb[IR][4], cc[IR][4];  // input columns x-1, x, x+1 of the current output column
  uint4 raw[IR], raw2[IR];
  load_raw(-1, raw);
  unpack(raw, ca);
  if (kStride == 1) {
    load_raw(0, raw);
    unpack(raw, cb);
  }
  load_raw(kStride == 1 ? 1 : 0, raw);  // prefetch for the first column
  if (kStride == 2) load_raw(1, raw2);
  for (int wo = 0; wo < Wo; ++wo) {
    if (kStride == 1) {
      unpack(raw, cc);
      if (wo + 1 < Wo) load_raw(wo + 2, raw);  // next column's loads fly under this column's arithmetic
    } else {
      unpack(raw, cb);
      unpack(raw2, cc);
      if (wo + 1 < Wo) {
        load_raw(2 * wo + 2, raw);
        load_raw(2 * wo + 3, raw2);
      }
    }
#pragma unroll
    for (int o = 0; o < kDwRowR; ++o) {
      if (ho0 + o < Ho) {
        __half2 acc[4];
#pragma unroll
        for (int j = 0; j < 4; ++j) acc[j] = bv[j];
#pragma unroll
        for (int dy = 0; dy < 3; ++dy) {
          const int ir = o * kStride + dy;
#pragma unroll
          for (int j = 0; j < 4; ++j) {
            acc[j] = __hfma2(ca[ir][j], wt[dy * 3 + 0][j], acc[j]);
            acc[j] = __hfma2(cb[ir][j], wt[dy * 3 + 1][j], acc[j]);
            acc[j] = __hfma2(cc[ir][j], wt[dy * 3 + 2][j], acc[j]);
          }
        }
        uint4 pk;
        uint32_t* pw = reinterpret_cast<uint32_t*>(&pk);
#pragma unroll
        for (int j = 0; j < 4; ++j) {
          const float2 f = __half22float2(__hmin2(__hmax2(acc[j], h_zero), h_six));
          const __nv_bfloat162 t = __floats2bfloat162_rn(f.x, f.y);
          pw[j] = *reinterpret_cast<const uint32_t*>(&t);
        }
        *reinterpret_cast<uint4*>(out + ((((int64_t)b * Ho + ho0 + o) * Wo + wo) * cp) + c0) = pk;
      }
    }
    // slide the window
#pragma unroll
    for (int ir = 0; ir < IR; ++ir)
#pragma unroll
      for (int j = 0; j < 4; ++j) {
        if (kStride == 1) {
          ca[ir][j] = cb[ir][j];
          cb[ir][j] = cc[ir][j];
        } else {
          ca[ir][j] = cc[ir][j];
        }
      }
  }
}

bool dw3x3_fp16_safe(const std::vector<float>& w, const std::vector<float>& bias, int cp, bool relu6_input) {
  if (!relu6_input) return false;
  for (int c = 0; c < cp; ++c) {
    double m = std::fabs((double)bias[(size_t)c]);
    for (int t = 0; t < 9; ++t) m += 6.0 * std::fabs((double)w[(size_t)t * cp + c]);
    if (!(m < 32768.0)) return false;  // NaN weights are not safe either
  }
  return true;
}

int dw3x3(const __nv_bfloat16* in, int B, int H, int W, int cp, int stride, const float* w, const float* bias, bool fp16,
          __nv_bfloat16* out, cudaStream_t st, int* kernel) {
  AM_CHECK(stride == 1 || stride == 2, "depthwise: stride %d", stride);
  const int Ho = (H - 1) / stride + 1, Wo = (W - 1) / stride + 1;
  AM_CHECK(B > 0 && H > 0 && W > 0 && cp % 8 == 0, "depthwise: empty input or channels not a multiple of 8");
  if (!fp16) {
    if (kernel) *kernel = kDwGeneric;
    AM_LAUNCH(depthwise_generic_kernel, grid_for((int64_t)B * Ho * Wo * (cp / 8)), 256, 0, st, in, B, H, W, cp, Ho, Wo,
              3, stride, 1, 1, w, bias, (int)kActRelu6, out);
    return AM_OK;
  }
  const int strips = (Ho + kDwRows - 1) / kDwRows;
  const int64_t total = (int64_t)B * strips * Wo * (cp / 8);
  const unsigned grid = (unsigned)((total + kDwThreads - 1) / kDwThreads);
  const int rstrips = (Ho + kDwRowR - 1) / kDwRowR;
  const int64_t rtotal = (int64_t)B * rstrips * (cp / 8);
  if (W <= 16 && rtotal >= (int64_t)sm_count() * 8 * kDwThreads) {
    // narrow late maps with enough (window, strip, channel group) work items to fill the GPU
    if (kernel) *kernel = kDwRow;
    const unsigned rgrid = (unsigned)((rtotal + kDwThreads - 1) / kDwThreads);
    if (stride == 1) {
      AM_LAUNCH(depthwise_row_kernel<1>, rgrid, kDwThreads, 0, st, in, B, H, W, cp, Ho, Wo, w, bias, out);
    } else {
      AM_LAUNCH(depthwise_row_kernel<2>, rgrid, kDwThreads, 0, st, in, B, H, W, cp, Ho, Wo, w, bias, out);
    }
  } else {
    if (kernel) *kernel = kDwStrip;
    if (stride == 1) {
      AM_LAUNCH(depthwise_kernel<1>, grid, kDwThreads, 0, st, in, B, H, W, cp, Ho, Wo, w, bias, out);
    } else {
      AM_LAUNCH(depthwise_kernel<2>, grid, kDwThreads, 0, st, in, B, H, W, cp, Ho, Wo, w, bias, out);
    }
  }
  return AM_OK;
}

}  // namespace am
