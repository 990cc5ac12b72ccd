// The log-mel plan and the register FFT-2048, shared by the log-mel kernel (mel.cu) and the track-feature spectrum pass
// (track_features.cu), which also reads the plan's window and twiddle tables.
#pragma once

#include "common.cuh"

namespace am {

constexpr int kNfft = 2048;
constexpr int kNc = 1024;       // complex FFT length
constexpr int kFramesPerCta = 16;
constexpr int kWarps = 8;
constexpr int kThreads = kWarps * 32;
constexpr int kTrStride = 33;   // padded row stride of the per-warp transpose buffer

struct MelTables {
  float* window;      // [2048]
  float2* fft_tw;     // [32*32]  fft_tw[k1*32 + n2] = W_1024^(n2*k1)
  float2* post_tw;    // [1024]   W_2048^k
  int* band_start;    // [n_mels] first FFT bin with non-zero weight
  int* band_len;      // [n_mels]
  int* band_off;      // [n_mels] offset into weights
  float* weights;     // [nnz]
};

}  // namespace am

struct am_mel_plan {
  am_mel_cfg cfg;
  int center;    // cfg.framing as mel_kernel takes it: 1 reflect pad n_fft/2, 0 no padding, 2 zero pad n_fft/2
  am::MelTables t;
  int max_bin;   // highest FFT bin with non-zero mel weight
  int nnz;
  am::DevBuf<char> storage;
};

namespace am {

// ---------------------------------------------------------------- device: 32-point FFT
// Only ever called with compile-time indices (fft32_stage's template arguments and unrolled loop counters), so every
// call folds to a constant.
__host__ __device__ constexpr float cos32(int i) {  // cos(2*pi*i/32), i in [0,16)
  switch (i) {
    case 0: return 1.0f;
    case 1: return 0.98078528040323044913f;
    case 2: return 0.92387953251128675613f;
    case 3: return 0.83146961230254523708f;
    case 4: return 0.70710678118654752440f;
    case 5: return 0.55557023301960222474f;
    case 6: return 0.38268343236508977173f;
    case 7: return 0.19509032201612826785f;
    case 8: return 0.0f;
    case 9: return -0.19509032201612826785f;
    case 10: return -0.38268343236508977173f;
    case 11: return -0.55557023301960222474f;
    case 12: return -0.70710678118654752440f;
    case 13: return -0.83146961230254523708f;
    case 14: return -0.92387953251128675613f;
    default: return -0.98078528040323044913f;
  }
}
// sin(2*pi*i/32) for i in [0,16): sin(x) = cos(x - pi/2) -> index i-8; cos is even.
__host__ __device__ constexpr float sin32i(int i) { return cos32(i >= 8 ? i - 8 : 8 - i); }

__host__ __device__ constexpr int rev5(int i) {
  return ((i & 1) << 4) | ((i & 2) << 2) | (i & 4) | ((i & 8) >> 2) | ((i & 16) >> 4);
}

// One radix-2 decimation-in-frequency stage of butterfly span kHalf.  The stage is a template argument so that
// every index and twiddle is a compile-time constant: with a runtime `half` loop nvcc kept the stage loop rolled,
// put re/im in local memory and looked the twiddles up through an indirect branch.  Products that feed a later
// addition are rounded on their own (__fmul_rn): straight-line code would otherwise let nvcc contract them into
// FMAs and change the result in the last bits.
template <int kHalf>
__device__ __forceinline__ void fft32_stage(float (&re)[32], float (&im)[32]) {
#pragma unroll
  for (int base = 0; base < 32; base += 2 * kHalf) {
#pragma unroll
    for (int j = 0; j < kHalf; ++j) {
      const int a = base + j, b = a + kHalf;
      const float ar = re[a], ai = im[a], br = re[b], bi = im[b];
      re[a] = ar + br;
      im[a] = ai + bi;
      const float dr = ar - br, di = ai - bi;
      const int idx = j * (16 / kHalf);  // twiddle W_32^idx = cos - i sin
      if (idx == 0) {
        re[b] = dr;
        im[b] = di;
      } else if (idx == 8) {  // * (-i)
        re[b] = di;
        im[b] = -dr;
      } else if (idx == 4) {  // * (1 - i)/sqrt2
        re[b] = __fmul_rn(dr + di, 0.70710678118654752440f);
        im[b] = __fmul_rn(di - dr, 0.70710678118654752440f);
      } else if (idx == 12) {  // * (-1 - i)/sqrt2
        re[b] = __fmul_rn(di - dr, 0.70710678118654752440f);
        im[b] = __fmul_rn(-(dr + di), 0.70710678118654752440f);
      } else {
        const float c = cos32(idx), s = sin32i(idx);
        re[b] = fmaf(dr, c, di * s);
        im[b] = fmaf(di, c, -dr * s);
      }
    }
  }
}

// In-place radix-2 decimation-in-frequency, forward (e^{-i...}).  Input natural order,
// output bit-reversed: X[k] is left in element rev5(k).  Straight-line code; trivial
// twiddles cost no multiplies.
__device__ __forceinline__ void fft32(float (&re)[32], float (&im)[32]) {
  fft32_stage<16>(re, im);
  fft32_stage<8>(re, im);
  fft32_stage<4>(re, im);
  fft32_stage<2>(re, im);
  fft32_stage<1>(re, im);
}

// ---------------------------------------------------------------- device: one frame's power spectrum
// One warp: x[0..2048) (staged samples of the frame) times win -> rFFT-2048 -> |X[k]|^2 into tr[k] for the bins of the
// first kK2 32-bin groups, and tr[1024] when nyquist.  2048 real samples -> 1024-point complex FFT as 32 x 32 (each lane
// does two radix-2 32-point FFTs in registers, twiddles from s_tw) -> real-FFT split (partner bins via warp shuffle).
// tr is the warp's 32 x kTrStride transpose buffer; the caller __syncwarp()s before reading it.
template <int kK2>
__device__ __forceinline__ void warp_power_spectrum(const float* __restrict__ x, const float* __restrict__ win,
                                                    const float2* __restrict__ s_tw, const float2* __restrict__ post_tw,
                                                    float* __restrict__ tr, int lane, bool nyquist) {
  float re[32], im[32];
  // ---- z[n] = x[2n]w[2n] + i x[2n+1]w[2n+1];  lane = n2, element n1 holds z[32*n1 + n2]
  const float2* xf = reinterpret_cast<const float2*>(x);
  const float2* wf = reinterpret_cast<const float2*>(win);
#pragma unroll
  for (int n1 = 0; n1 < 32; ++n1) {
    const float2 x = xf[32 * n1 + lane];
    const float2 w = wf[32 * n1 + lane];
    re[n1] = __fmul_rn(x.x, w.x);  // not contracted into the first butterflies
    im[n1] = __fmul_rn(x.y, w.y);
  }
  fft32(re, im);  // element i = Y[k1 = rev5(i)] for this n2
  // ---- twiddle W_1024^(n2*k1) and transpose to lane = k1, element = n2
#pragma unroll
  for (int i = 0; i < 32; ++i) {
    const int k1 = rev5(i);
    const float2 w = s_tw[k1 * 32 + lane];
    const float r = re[i], q = im[i];
    re[i] = fmaf(r, w.x, -q * w.y);
    im[i] = fmaf(r, w.y, q * w.x);
  }
#pragma unroll
  for (int i = 0; i < 32; ++i) tr[rev5(i) * kTrStride + lane] = re[i];
  __syncwarp();
#pragma unroll
  for (int n2 = 0; n2 < 32; ++n2) re[n2] = tr[lane * kTrStride + n2];
  __syncwarp();
#pragma unroll
  for (int i = 0; i < 32; ++i) tr[rev5(i) * kTrStride + lane] = im[i];
  __syncwarp();
#pragma unroll
  for (int n2 = 0; n2 < 32; ++n2) im[n2] = tr[lane * kTrStride + n2];
  __syncwarp();
  fft32(re, im);  // element i = Z[k1 + 32*k2], k1 = lane, k2 = rev5(i)

  // ---- real-FFT split + power:  X[k] = (Z[k]+Z*[N-k])/2 - (i/2) W_2048^k (Z[k]-Z*[N-k])
  const int partner = (32 - lane) & 31;
#pragma unroll
  for (int i = 0; i < 32; ++i) {
    const int k2 = rev5(i);
    if (k2 < kK2) {  // compile time
      float pr = __shfl_sync(0xffffffffu, re[31 - i], partner);
      float pi = __shfl_sync(0xffffffffu, im[31 - i], partner);
      if (lane == 0) {  // N-k = 32*(32-k2): same lane, element rev5((32-k2)&31)
        pr = re[rev5((32 - k2) & 31)];
        pi = im[rev5((32 - k2) & 31)];
      }
      const int k = lane + 32 * k2;
      const float2 w = __ldg(&post_tw[k]);  // (cos, -sin)
      const float er = re[i] + pr, ei = im[i] - pi;
      const float orr = re[i] - pr, oi = im[i] + pi;
      const float xr = 0.5f * (er + fmaf(w.x, oi, w.y * orr));
      const float xi = 0.5f * (ei - fmaf(w.x, orr, -w.y * oi));
      tr[k] = fmaf(xr, xr, xi * xi);
    }
  }
  if (nyquist && lane == 0) {  // Nyquist bin: X[1024] = Re Z[0] - Im Z[0]
    const float ny = re[0] - im[0];
    tr[kNc] = ny * ny;
  }
}

}  // namespace am
