// analyze_track's tempo, energy and key inputs (tasks/analysis.py:344-348) for a batch of ragged tracks  (sm_90a)
//
// Restates librosa 0.11.0's beat.beat_track (tempo only), feature.rms and feature.chroma_stft as analyze_track calls
// them: n_fft 2048, hop 512, periodic Hann, center=True with zero padding, so a track of n samples has T = 1 + n / 512
// frames.  oracle/track_features.py is the float64 statement of every step below.
//
//   tempo   am_mel_batch_dev on a center = 2 (zero pad) plan: 128 slaney mels up to sr/2 in dB      (mel_kernel)
//           per-track maximum of the dB spectrogram (the top_db = 80 clip is against it)           tf_db_max_kernel
//           clip, first difference, clamp at 0, median over the mels, 3 frames of left pad           tf_onset_kernel
//           tempogram: linear-ramp pad, Hann window, autocorrelation, inf-normalisation, summed
//           over frames per block (float64)                                                         tf_tempogram_kernel
//           mean over frames, blocks summed in order                                                 tf_tempogram_reduce
//           argmax(log1p(1e6 tg) + log-normal prior) over 8 s of lags: on the host (win doubles per track)
//   rms     frame -> sum of squares of the unwindowed samples                                        tf_spectrum_kernel
//   chroma  frame -> Hann -> rFFT-2048 (mel.cuh's register FFT) -> |.|^2 -> piptrack peaks, compacted
//           per frame (mag and residual histogram bin)                                               tf_spectrum_kernel
//           exact median of the track's peak mags (radix select on the float bits), the 100-bin
//           residual histogram of the peaks at or above it, its first fullest bin                    tf_tuning_kernel
//           filters.chroma(sr, 2048, tuning) per track (float64 -> float32)                          tf_chroma_fb_kernel
//           the spectrum again (recomputed, not stored), chromafb @ S, per-frame max normalisation   tf_spectrum_kernel
//
// Tracks are zero-padded to the longest track of their group, which is exact: librosa pads with zeros too, and only
// each track's own T frames are kept.  Every reduction has a fixed order and no floating-point atomics are used, so
// two calls give identical bits and a track gives the same result alone as in any batch.
#include "host_call.cuh"
#include "mel.cuh"

#include <algorithm>
#include <cmath>
#include <type_traits>

namespace am {

constexpr int kTfMels = 128;
constexpr int kTfHop = 512;
constexpr int kHistBins = 100;
constexpr int kTgFrames = 64;      // frames of one tempogram block
constexpr int kTgThreads = 256;
constexpr int kTgMaxWin = 1024;    // lags: floor(8 sr / 512) <= 750 for sr <= 48 kHz
constexpr int kTuneThreads = 1024;
constexpr size_t kWorkspaceBytes = size_t(2) << 30;   // per group of tracks

// np.linspace(-0.5, 0.5, 101)[i] for i < 100: i * 0.01 + (-0.5), each step rounded
__host__ __device__ inline double hist_edge(int i) {
#ifdef __CUDA_ARCH__
  return __dadd_rn(__dmul_rn((double)i, 0.01), -0.5);
#else
  return (double)i * 0.01 + -0.5;
#endif
}

// ------------------------------------------------------------------------------------------------ padding
__global__ void tf_pad_kernel(const float* __restrict__ x, const long long* __restrict__ off, int L,
                              float* __restrict__ out) {
  const int b = blockIdx.y;
  const long long o = off[b], n = off[b + 1] - o;
  for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < L; i += (long long)gridDim.x * blockDim.x)
    out[(long long)b * L + i] = i < n ? x[o + i] : 0.f;
}

// ------------------------------------------------------------------------------------------------ onset envelope
// max over the track's own frames of the dB mel spectrogram [B, 128, Tmax]
__global__ void tf_db_max_kernel(const float* __restrict__ db, const int* __restrict__ T_of, int Tmax,
                                 float* __restrict__ out) {
  __shared__ float red[32];
  const int b = blockIdx.x, T = T_of[b];
  const float* d = db + (long long)b * kTfMels * Tmax;
  float m = -INFINITY;
  for (long long i = threadIdx.x; i < (long long)kTfMels * T; i += blockDim.x) {
    const int mel = (int)(i / T), t = (int)(i % T);
    m = fmaxf(m, d[(long long)mel * Tmax + t]);
  }
  for (int o = 16; o; o >>= 1) m = fmaxf(m, __shfl_xor_sync(0xffffffffu, m, o));
  if ((threadIdx.x & 31) == 0) red[threadIdx.x >> 5] = m;
  __syncthreads();
  if (threadIdx.x < 32) {
    m = threadIdx.x < (blockDim.x >> 5) ? red[threadIdx.x] : -INFINITY;
    for (int o = 16; o; o >>= 1) m = fmaxf(m, __shfl_xor_sync(0xffffffffu, m, o));
    if (threadIdx.x == 0) out[b] = m;
  }
}

// env[t] = median over the mels of max(0, c[t-2] - c[t-3]), c = max(dB, max - 80) (float32, as librosa's), 0 for
// t < 3.  One warp per frame; the 128 values are sorted by a bitonic network in the warp's shared slice.
__global__ void __launch_bounds__(256) tf_onset_kernel(const float* __restrict__ db, const float* __restrict__ db_max,
                                                       const int* __restrict__ T_of,
                                                       const long long* __restrict__ foff, int Tmax,
                                                       float* __restrict__ env) {
  __shared__ float s[8][kTfMels];
  const int b = blockIdx.y, lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  const int t = blockIdx.x * 8 + warp, T = T_of[b];
  if (t >= T) return;
  float* e = env + foff[b];
  if (t < 3) {
    if (lane == 0) e[t] = 0.f;
    return;
  }
  const float floor_db = db_max[b] - 80.0f;
  const float* d = db + (long long)b * kTfMels * Tmax;
  float* v = s[warp];
#pragma unroll
  for (int q = 0; q < 4; ++q) {
    const int m = lane + 32 * q;
    const float cur = fmaxf(d[(long long)m * Tmax + t - 2], floor_db);
    const float prev = fmaxf(d[(long long)m * Tmax + t - 3], floor_db);
    v[m] = fmaxf(0.f, cur - prev);
  }
  __syncwarp();
  for (int k = 2; k <= kTfMels; k <<= 1) {
    for (int j = k >> 1; j > 0; j >>= 1) {
#pragma unroll
      for (int q = 0; q < 4; ++q) {
        const int i = lane + 32 * q, l = i ^ j;
        if (l > i) {
          const float a = v[i], c = v[l];
          const bool up = (i & k) == 0;
          if (up ? a > c : a < c) {
            v[i] = c;
            v[l] = a;
          }
        }
      }
      __syncwarp();
    }
  }
  if (lane == 0) e[t] = __fmul_rn(__fadd_rn(v[kTfMels / 2 - 1], v[kTfMels / 2]), 0.5f);
}

// ------------------------------------------------------------------------------------------------ tempogram
// Block (blk, b) sums, over frames t in [blk * 64, +64) of track b, the inf-normalised autocorrelation of
// env_pad[t .. t + win) * hann_win (float64), env_pad the envelope padded by win/2 on both sides with a linear ramp to
// 0 (np.pad mode='linear_ramp').  part[b, blk, k] = that sum; any[b, blk] = 1 when an envelope value is non-zero.
__global__ void __launch_bounds__(kTgThreads) tf_tempogram_kernel(const float* __restrict__ env,
                                                                  const int* __restrict__ T_of,
                                                                  const long long* __restrict__ foff, int win,
                                                                  int n_blk, double* __restrict__ part,
                                                                  int* __restrict__ any) {
  __shared__ double s_hann[kTgMaxWin];
  __shared__ double s_w[kTgMaxWin];
  __shared__ double s_red[kTgThreads / 32];
  constexpr int kLags = kTgMaxWin / kTgThreads;
  const int b = blockIdx.y, blk = blockIdx.x, tid = threadIdx.x;
  const int T = T_of[b], h = win / 2;
  const float* e = env + foff[b];
  double acc[kLags];
#pragma unroll
  for (int q = 0; q < kLags; ++q) acc[q] = 0.0;
  for (int j = tid; j < win; j += kTgThreads) s_hann[j] = 0.5 - 0.5 * cos(2.0 * M_PI * j / win);
  const int t_lo = blk * kTgFrames, t_hi = min(T, t_lo + kTgFrames);
  const float edge = e[T - 1];
  int nz = 0;
  for (int t = t_lo; t < t_hi; ++t) {
    __syncthreads();
    for (int j = tid; j < win; j += kTgThreads) {
      const int p = t + j - h;   // index into the unpadded envelope
      float x;
      if (p < 0) {
        x = (float)((double)(p + h) * ((double)e[0] / h));
      } else if (p >= T) {
        x = (float)((double)(h - 1 - (p - T)) * ((double)edge / h));
      } else {
        x = e[p];
      }
      s_w[j] = (double)x * s_hann[j];
    }
    if (tid == 0) nz |= e[t] != 0.f;
    __syncthreads();
    double r[kLags];
    double m = 0.0;
#pragma unroll
    for (int q = 0; q < kLags; ++q) {
      const int k = tid + q * kTgThreads;
      double s = 0.0;
      if (k < win)
        for (int j = 0; j + k < win; ++j) s = fma(s_w[j], s_w[j + k], s);
      r[q] = s;
      m = fmax(m, fabs(s));
    }
    for (int o = 16; o; o >>= 1) m = fmax(m, __shfl_xor_sync(0xffffffffu, m, o));
    if ((tid & 31) == 0) s_red[tid >> 5] = m;
    __syncthreads();
    m = s_red[0];
#pragma unroll
    for (int w = 1; w < kTgThreads / 32; ++w) m = fmax(m, s_red[w]);
    if (m < 2.2250738585072014e-308) m = 1.0;   // np.finfo(float64).tiny: all-zero frames stay 0
#pragma unroll
    for (int q = 0; q < kLags; ++q) acc[q] += r[q] / m;
  }
  double* o = part + ((long long)b * n_blk + blk) * win;
#pragma unroll
  for (int q = 0; q < kLags; ++q) {
    const int k = tid + q * kTgThreads;
    if (k < win) o[k] = acc[q];
  }
  if (tid == 0) any[b * n_blk + blk] = nz;
}

// tg[b, k] = sum over blocks (in order) / T; any_b = OR of the blocks' flags
__global__ void tf_tempogram_reduce(const double* __restrict__ part, const int* __restrict__ any_part,
                                    const int* __restrict__ T_of, int win, int n_blk, double* __restrict__ tg,
                                    int* __restrict__ any) {
  const int b = blockIdx.x, T = T_of[b], nb = (T + kTgFrames - 1) / kTgFrames;
  for (int k = threadIdx.x; k < win; k += blockDim.x) {
    double s = 0.0;
    for (int i = 0; i < nb; ++i) s += part[((long long)b * n_blk + i) * win + k];
    tg[(long long)b * win + k] = s / T;
  }
  if (threadIdx.x == 0) {
    int a = 0;
    for (int i = 0; i < nb; ++i) a |= any_part[b * n_blk + i];
    any[b] = a;
  }
}

// ------------------------------------------------------------------------------------------------ spectrum pass
struct TfSpecArgs {
  const float* pad;            // [B, L] zero-padded samples
  const int* T_of;             // [B]
  const long long* n_of;       // [B] samples per track
  const long long* foff;       // [B + 1] frame offsets
  int L;
  int sr;
  int kmin, kmax;              // piptrack's bins: fmin <= rfftfreq < fmax
  int cap;                     // peak slots per frame
  float* rms;                  // [sum T]            (pass 1, optional)
  float* pk_mag;               // [sum T, cap]       (pass 1, optional)
  unsigned char* pk_bin;       // [sum T, cap]
  int* pk_count;               // [sum T]
  const float* chroma_fb;      // [B, 12, 1025]     (pass 2)
  float* chroma;               // [12 * sum T]: track b at 12 foff[b], row-major (12, T_b)
};

// residual of a peak's pitch in semitones, (12 log2(f / 27.5)) mod 1 shifted into [-0.5, 0.5), and its histogram bin
// against np.linspace(-0.5, 0.5, 101) (left-closed bins, the last closed on the right)
__device__ __forceinline__ int residual_bin(float pitch) {
  const double x = 12.0 * log2((double)pitch / 27.5);
  double r = fmod(x, 1.0);
  if (r < 0.0) r += 1.0;
  if (r >= 0.5) r -= 1.0;
  int i = (int)floor((r + 0.5) * kHistBins);
  i = min(max(i, 0), kHistBins - 1);
  while (i > 0 && r < hist_edge(i)) --i;
  while (i < kHistBins - 1 && r >= hist_edge(i + 1)) ++i;
  return i;
}

template <bool kChroma>
__global__ void __launch_bounds__(kThreads, 2) tf_spectrum_kernel(TfSpecArgs a, MelTables tb) {
  extern __shared__ __align__(16) unsigned char smem_raw[];
  constexpr int n_stage = (kFramesPerCta - 1) * kTfHop + kNfft;
  float* s_x = reinterpret_cast<float*>(smem_raw);                        // [n_stage]
  float* s_win = s_x + n_stage;                                           // [2048]
  float2* s_tw = reinterpret_cast<float2*>(s_win + kNfft);                // [1024]
  float* s_tr = reinterpret_cast<float*>(s_tw + 32 * 32);                 // [8][32*33]

  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  const int b = blockIdx.y, T = a.T_of[b];
  const int t0 = blockIdx.x * kFramesPerCta;
  if (t0 >= T) return;
  const int nf = min(kFramesPerCta, T - t0);
  const long long n = a.n_of[b];
  const float* x = a.pad + (long long)b * a.L;
  const int count = (nf - 1) * kTfHop + kNfft;
  const long long p0 = (long long)t0 * kTfHop - kNfft / 2;
  for (int i = tid; i < n_stage; i += kThreads) {
    const long long src = p0 + i;
    s_x[i] = (i < count && src >= 0 && src < n) ? x[src] : 0.f;
  }
  for (int i = tid; i < kNfft; i += kThreads) s_win[i] = tb.window[i];
  for (int i = tid; i < 32 * 32; i += kThreads) s_tw[i] = tb.fft_tw[i];
  __syncthreads();

  float* tr = s_tr + warp * 32 * kTrStride;
  const long long fo = a.foff[b];
  for (int f = warp; f < nf; f += kWarps) {
    const int t = t0 + f;
    const float* xf = s_x + f * kTfHop;
    if (!kChroma && a.rms) {
      double ss = 0.0;
      for (int i = lane; i < kNfft; i += 32) ss = fma((double)xf[i], (double)xf[i], ss);
      for (int o = 16; o; o >>= 1) ss += __shfl_xor_sync(0xffffffffu, ss, o);
      if (lane == 0) a.rms[fo + t] = (float)sqrt(ss / kNfft);
    }
    warp_power_spectrum<32>(xf, s_win, s_tw, tb.post_tw, tr, lane, true);
    __syncwarp();
    if constexpr (!kChroma) {
      if (a.pk_mag) {
        // piptrack: threshold 0.1 x the frame's maximum over all bins; a peak is a localmax of S * (S > ref)
        float m = 0.f;
        for (int k = lane; k <= kNc; k += 32) m = fmaxf(m, tr[k]);
        for (int o = 16; o; o >>= 1) m = fmaxf(m, __shfl_xor_sync(0xffffffffu, m, o));
        const float ref = __fmul_rn(0.1f, m);
        float* pm = a.pk_mag + (fo + t) * a.cap;
        unsigned char* pb = a.pk_bin + (fo + t) * a.cap;
        int cnt = 0;
        for (int k0 = a.kmin; k0 < a.kmax; k0 += 32) {
          const int k = k0 + lane;
          bool peak = false;
          float mag = 0.f;
          int bin = 0;
          if (k < a.kmax) {
            const float sm = tr[k - 1], s0 = tr[k], sp = tr[k + 1];
            const float ym = sm > ref ? sm : 0.f, y0 = s0 > ref ? s0 : 0.f, yp = sp > ref ? sp : 0.f;
            peak = y0 > ym && y0 >= yp;
            if (peak) {
              // librosa 0.11 _parabolic_interpolation and np.gradient, float32 without contraction
              const float pa = __fsub_rn(__fadd_rn(sp, sm), __fmul_rn(2.f, s0));
              const float pbv = __fdiv_rn(__fsub_rn(sp, sm), 2.f);
              const float shift = fabsf(pbv) >= fabsf(pa) ? 0.f : __fdiv_rn(-pbv, pa);
              mag = __fadd_rn(s0, __fmul_rn(__fmul_rn(0.5f, pbv), shift));
              const float pitch = (float)(((double)k + (double)shift) * (double)a.sr / (double)kNfft);
              bin = residual_bin(pitch);
            }
          }
          const unsigned bal = __ballot_sync(0xffffffffu, peak);
          if (peak) {
            const int slot = cnt + __popc(bal & ((1u << lane) - 1));
            pm[slot] = mag;
            pb[slot] = (unsigned char)bin;
          }
          cnt += __popc(bal);
        }
        if (lane == 0) a.pk_count[fo + t] = cnt;
      }
    } else {
      const float* fb = a.chroma_fb + (long long)b * 12 * (kNc + 1);
      float c[12];
#pragma unroll
      for (int q = 0; q < 12; ++q) c[q] = 0.f;
      for (int k = lane; k <= kNc; k += 32) {
        const float s = tr[k];
#pragma unroll
        for (int q = 0; q < 12; ++q) c[q] = fmaf(__ldg(fb + q * (kNc + 1) + k), s, c[q]);
      }
      float m = 0.f;
#pragma unroll
      for (int q = 0; q < 12; ++q) {
        for (int o = 16; o; o >>= 1) c[q] += __shfl_xor_sync(0xffffffffu, c[q], o);
        m = fmaxf(m, fabsf(c[q]));
      }
      if (m < 1.17549435e-38f) m = 1.f;   // np.finfo(float32).tiny: all-zero frames stay 0
      if (lane < 12) {
        float v = c[0];
#pragma unroll
        for (int q = 1; q < 12; ++q)
          if (lane == q) v = c[q];
        a.chroma[12 * fo + (long long)lane * T + t] = __fdiv_rn(v, m);
      }
    }
    __syncwarp();
  }
}

static size_t tf_spectrum_smem() {
  return ((kFramesPerCta - 1) * kTfHop + kNfft + kNfft + 2 * 32 * 32 + (size_t)kWarps * 32 * kTrStride) * sizeof(float);
}

// ------------------------------------------------------------------------------------------------ tuning
// One block per track.  The median of all peak mags (np.median: the middle value, or the float32 mean of the two
// middle values) by an exact radix select on the float bits (mags are >= 0, so their bits order like their values),
// then the histogram of the bins of the peaks with mag >= median, and tuning = the left edge of its first fullest bin.
__device__ unsigned tf_select(const float* __restrict__ pm, const int* __restrict__ cnt, int T, int cap,
                              unsigned rank, int* hist /* [256] */, unsigned* s_state /* [2] */) {
  unsigned prefix = 0, mask = 0;
  for (int shift = 24; shift >= 0; shift -= 8) {
    for (int i = threadIdx.x; i < 256; i += blockDim.x) hist[i] = 0;
    __syncthreads();
    for (int t = threadIdx.x; t < T; t += blockDim.x) {
      const int c = cnt[t];
      for (int j = 0; j < c; ++j) {
        const unsigned u = __float_as_uint(pm[(long long)t * cap + j]);
        if ((u & mask) == prefix) atomicAdd(&hist[(u >> shift) & 255], 1);
      }
    }
    __syncthreads();
    if (threadIdx.x == 0) {
      unsigned r = rank, d = 0;
      while (r >= (unsigned)hist[d]) r -= hist[d++];
      s_state[0] = prefix | (d << shift);
      s_state[1] = r;
    }
    __syncthreads();
    prefix = s_state[0];
    rank = s_state[1];
    mask |= 255u << shift;
    __syncthreads();
  }
  return prefix;
}

__global__ void __launch_bounds__(kTuneThreads) tf_tuning_kernel(const float* __restrict__ pk_mag,
                                                                 const unsigned char* __restrict__ pk_bin,
                                                                 const int* __restrict__ pk_count,
                                                                 const int* __restrict__ T_of,
                                                                 const long long* __restrict__ foff, int cap,
                                                                 float* __restrict__ thr_out,
                                                                 int* __restrict__ hist_out,
                                                                 double* __restrict__ tuning) {
  __shared__ int hist[256];
  __shared__ unsigned s_state[2];
  __shared__ unsigned long long s_n;
  const int b = blockIdx.x, T = T_of[b];
  const long long fo = foff[b];
  const float* pm = pk_mag + fo * cap;
  const unsigned char* pb = pk_bin + fo * cap;
  const int* cnt = pk_count + fo;
  if (threadIdx.x == 0) s_n = 0;
  __syncthreads();
  unsigned long long n_loc = 0;
  for (int t = threadIdx.x; t < T; t += blockDim.x) n_loc += cnt[t];
  atomicAdd(&s_n, n_loc);
  __syncthreads();
  const unsigned long long N = s_n;
  if (N == 0) {   // pitch_tuning of an empty set: 0.0
    if (threadIdx.x < kHistBins) hist_out[b * kHistBins + threadIdx.x] = 0;
    if (threadIdx.x == 0) {
      thr_out[b] = 0.f;
      tuning[b] = 0.0;
    }
    return;
  }
  const float v1 = __uint_as_float(tf_select(pm, cnt, T, cap, (unsigned)((N - 1) / 2), hist, s_state));
  float thr = v1;
  if (N % 2 == 0) {
    const float v2 = __uint_as_float(tf_select(pm, cnt, T, cap, (unsigned)(N / 2), hist, s_state));
    thr = __fdiv_rn(__fadd_rn(v1, v2), 2.f);
  }
  for (int i = threadIdx.x; i < 256; i += blockDim.x) hist[i] = 0;
  __syncthreads();
  for (int t = threadIdx.x; t < T; t += blockDim.x) {
    const int c = cnt[t];
    for (int j = 0; j < c; ++j)
      if (pm[(long long)t * cap + j] >= thr) atomicAdd(&hist[pb[(long long)t * cap + j]], 1);
  }
  __syncthreads();
  if (threadIdx.x < kHistBins) hist_out[b * kHistBins + threadIdx.x] = hist[threadIdx.x];
  if (threadIdx.x == 0) {
    int best = 0;
    for (int i = 1; i < kHistBins; ++i)
      if (hist[i] > hist[best]) best = i;
    thr_out[b] = thr;
    tuning[b] = hist_edge(best);
  }
}

// ------------------------------------------------------------------------------------------------ chroma filterbank
// filters.chroma(sr, 2048, n_chroma=12, tuning, ctroct=5, octwidth=2, norm=2, base_c=True) in float64, stored float32:
// fb[b, c, k] for k <= 1024.  One block per track, one thread per FFT bin.
__device__ __forceinline__ double tf_frqbin(int k, double step, double a16) {
  // 12 * hz_to_octs(k * sr / 2048); the DC bin is 1.5 octaves below bin 1
  if (k == 0) return 12.0 * log2(step / a16) - 18.0;
  return 12.0 * log2(((double)k * step) / a16);
}

__global__ void tf_chroma_fb_kernel(const double* __restrict__ tuning, int sr, float* __restrict__ fb) {
  const int b = blockIdx.x;
  const double a440 = 440.0 * pow(2.0, tuning[b] / 12.0);
  const double a16 = a440 / 16.0;
  const double step = (double)sr / (double)kNfft;   // np.linspace(0, sr, 2048, endpoint=False)
  for (int k = threadIdx.x; k <= kNc; k += blockDim.x) {
    const double f0 = tf_frqbin(k, step, a16), f1 = tf_frqbin(k + 1, step, a16);
    const double bw = fmax(f1 - f0, 1.0);
    double w[12];
    double len = 0.0;
#pragma unroll
    for (int c = 0; c < 12; ++c) {
      double d = f0 - (double)c;
      d = fmod(d + 6.0 + 120.0, 12.0);
      if (d < 0.0) d += 12.0;
      d -= 6.0;
      const double q = 2.0 * d / bw;
      w[c] = exp(-0.5 * (q * q));
      len += w[c] * w[c];
    }
    len = sqrt(len);
    if (len < 2.2250738585072014e-308) len = 1.0;
    const double o = (f0 / 12.0 - 5.0) / 2.0;
    const double oct = exp(-0.5 * (o * o));
#pragma unroll
    for (int c = 0; c < 12; ++c) fb[((long long)b * 12 + c) * (kNc + 1) + k] = (float)(w[(c + 3) % 12] / len * oct);
  }
}

}  // namespace am

// ================================================================================================ host API
using namespace am;

struct am_track_features_plan {
  int sr;
  int win;           // tempogram lags
  int kmin, kmax;    // piptrack bins
  int cap;           // peak slots per frame
  am_mel_plan* mel = nullptr;
  ~am_track_features_plan() { am_mel_plan_free(mel); }
};

extern "C" int am_track_features_plan_create(int sr, am_track_features_plan** out) {
  AM_CHECK(out != nullptr, "am_track_features_plan_create: out is NULL");
  *out = nullptr;
  AM_CHECK(sr >= AM_TRACK_FEATURES_MIN_SR && sr <= AM_TRACK_FEATURES_MAX_SR,
           "track features: sample rate %d outside [%d, %d]", sr, AM_TRACK_FEATURES_MIN_SR, AM_TRACK_FEATURES_MAX_SR);
  AM_TRY(ensure_init());
  auto* p = new am_track_features_plan();
  p->sr = sr;
  p->win = (int)((long long)(8.0 * sr) / kTfHop);
  // np.fft.rfftfreq(2048, 1/sr): k * (1 / (2048 * (1 / sr))); fmin 150 <= f < min(4000, sr / 2)
  const double val = 1.0 / (kNfft * (1.0 / sr));
  const double fmax = std::min(4000.0, (double)sr / 2);
  int lo = -1, hi = -1;
  for (int k = 0; k <= kNc; ++k) {
    const double f = k * val;
    if (150.0 <= f && f < fmax) {
      if (lo < 0) lo = k;
      hi = k;
    }
  }
  p->kmin = lo;
  p->kmax = hi + 1;
  p->cap = (int)round_up((size_t)((p->kmax - p->kmin + 2) / 2), 32);
  am_mel_cfg cfg{sr, kNfft, kTfHop, kTfMels, 0.0f, (float)sr / 2.0f, 0, /* framing: zero pad */ 2, 0};
  int s = am_mel_plan_create(&cfg, &p->mel);
  if (s == AM_OK) s = allow_dynamic_smem<tf_spectrum_kernel<false>>(tf_spectrum_smem());
  if (s == AM_OK) s = allow_dynamic_smem<tf_spectrum_kernel<true>>(tf_spectrum_smem());
  if (s != AM_OK) {
    delete p;
    return s;
  }
  *out = p;
  return AM_OK;
}

extern "C" void am_track_features_plan_free(am_track_features_plan* plan) { delete plan; }

extern "C" int am_track_features_plan_info(const am_track_features_plan* plan, int* win, int* kmin, int* kmax) {
  AM_CHECK(plan != nullptr, "am_track_features_plan_info: plan is NULL");
  if (win) *win = plan->win;
  if (kmin) *kmin = plan->kmin;
  if (kmax) *kmax = plan->kmax;
  return AM_OK;
}

namespace {

// bpm[k] = 60 sr / (512 k), bpm[0] = inf; argmax(log1p(1e6 tg) + logprior), logprior = -0.5 (log2 bpm - log2 120)^2
// and -inf below the first lag whose bpm is under 320 (feature/rhythm.py tempo)
double tempo_from_tg(const double* tg, int win, int sr) {
  std::vector<double> bpm(win);
  bpm[0] = INFINITY;
  for (int k = 1; k < win; ++k) bpm[k] = 60.0 * sr / (kTfHop * (double)k);
  int max_idx = 0;
  while (max_idx < win && !(bpm[max_idx] < 320.0)) ++max_idx;
  if (max_idx == win) max_idx = 0;   // np.argmax of an all-False mask
  int best = -1;
  double best_v = 0.0;
  for (int k = 0; k < win; ++k) {
    const double d = (std::log2(bpm[k]) - std::log2(120.0)) / 1.0;
    const double lp = k < max_idx ? -INFINITY : -0.5 * (d * d);
    const double v = std::log1p(1e6 * tg[k]) + lp;
    if (best < 0 || v > best_v) {
      best = k;
      best_v = v;
    }
  }
  return bpm[best];
}

struct Group {
  int b0, nb;
  long long L;
  int Tmax;
};

// Device buffers of one group of tracks, carved from one allocation: carve(nullptr, ...) returns the bytes needed.
struct Workspace {
  float* x;  float* pad;  long long* off;  long long* n;  long long* foff;  int* T;
  float* db;  float* db_max;  float* env;  double* part;  int* any_part;  double* tg;  int* any;   // tempo
  float* rms;                                                                                     // rms
  float* pk_mag;  unsigned char* pk_bin;  int* pk_count;  float* thr;  int* hist;  double* tuning;
  float* fb;  float* chroma;                                                                      // chroma
};

size_t carve(char* base, Workspace& w, int nb, long long L, int Tmax, long long n_in, long long nT, int win, int cap,
             bool tempo, bool rms, bool chroma) {
  size_t o = 0;
  auto take = [&](auto*& p, size_t count, bool on = true) {
    using T = std::remove_reference_t<decltype(*p)>;
    p = nullptr;
    if (!on) return;
    if (base) p = reinterpret_cast<T*>(base + o);
    o = round_up(o + count * sizeof(T), 256);
  };
  const int n_blk = (Tmax + kTgFrames - 1) / kTgFrames;
  take(w.x, n_in);
  take(w.pad, (size_t)nb * L);
  take(w.off, nb + 1);
  take(w.n, nb);
  take(w.foff, nb + 1);
  take(w.T, nb);
  take(w.db, (size_t)nb * kTfMels * Tmax, tempo);
  take(w.db_max, nb, tempo);
  take(w.env, nT, tempo);
  take(w.part, (size_t)nb * n_blk * win, tempo);
  take(w.any_part, (size_t)nb * n_blk, tempo);
  take(w.tg, (size_t)nb * win, tempo);
  take(w.any, nb, tempo);
  take(w.rms, nT, rms);
  take(w.pk_mag, (size_t)nT * cap, chroma);
  take(w.pk_bin, (size_t)nT * cap, chroma);
  take(w.pk_count, nT, chroma);
  take(w.thr, nb, chroma);
  take(w.hist, (size_t)nb * kHistBins, chroma);
  take(w.tuning, nb, chroma);
  take(w.fb, (size_t)nb * 12 * (kNc + 1), chroma);
  take(w.chroma, (size_t)nT * 12, chroma);
  return o;
}

}  // namespace

extern "C" int am_track_features(const am_track_features_plan* plan, const float* samples, const int64_t* offsets,
                                 int n_tracks, int what, double* tempo, float* rms, float* chroma, double* tuning,
                                 float* onset_env, double* tempogram, int32_t* histogram, float* threshold) {
  AM_CHECK(plan != nullptr, "am_track_features: plan is NULL");
  AM_CHECK(n_tracks >= 1 && samples && offsets, "am_track_features: need n_tracks >= 1, samples and offsets");
  AM_CHECK(what >= 1 && what <= (AM_TF_TEMPO | AM_TF_RMS | AM_TF_CHROMA), "am_track_features: bad what flags %d",
           what);
  const bool want_tempo = what & AM_TF_TEMPO, want_rms = what & AM_TF_RMS, want_chroma = what & AM_TF_CHROMA;
  AM_CHECK(!want_tempo || tempo, "am_track_features: tempo output is NULL");
  AM_CHECK(!want_rms || rms, "am_track_features: rms output is NULL");
  AM_CHECK(!want_chroma || chroma, "am_track_features: chroma output is NULL");
  AM_CHECK(offsets[0] == 0, "am_track_features: offsets[0] must be 0");
  for (int i = 0; i < n_tracks; ++i) {
    const long long n = offsets[i + 1] - offsets[i];
    AM_CHECK(n >= 1, "am_track_features: track %d is empty", i);
    AM_CHECK(n <= (long long)INT32_MAX - kNfft, "am_track_features: track %d is too long", i);
  }
  for (long long i = 0; i < offsets[n_tracks]; ++i)
    AM_CHECK(std::isfinite(samples[i]), "am_track_features: sample %lld is not finite", i);

  const int win = plan->win, cap = plan->cap;
  std::vector<int> T(n_tracks);
  std::vector<long long> foff(n_tracks + 1, 0);
  for (int i = 0; i < n_tracks; ++i) {
    T[i] = 1 + (int)((offsets[i + 1] - offsets[i]) / kTfHop);
    foff[i + 1] = foff[i] + T[i];
  }
  // groups of consecutive tracks whose workspace (padded to the group's longest track) fits kWorkspaceBytes
  auto need = [&](int b0, int nb, long long L, int Tm) {
    Workspace w;
    return carve(nullptr, w, nb, L, Tm, offsets[b0 + nb] - offsets[b0], foff[b0 + nb] - foff[b0], win, cap,
                 want_tempo, want_rms, want_chroma);
  };
  std::vector<Group> groups;
  size_t ws_max = 0;
  for (int i = 0; i < n_tracks;) {
    Group g{i, 0, 0, 0};
    while (i < n_tracks) {
      const long long L = std::max<long long>(g.L, offsets[i + 1] - offsets[i]);
      const int Tm = std::max(g.Tmax, T[i]);
      if (g.nb > 0 && need(g.b0, g.nb + 1, L, Tm) > kWorkspaceBytes) break;
      g.L = L;
      g.Tmax = Tm;
      ++g.nb;
      ++i;
    }
    ws_max = std::max(ws_max, need(g.b0, g.nb, g.L, g.Tmax));
    groups.push_back(g);
  }

  cudaStream_t st;
  AM_TRY(HostCall::thread_stream(&st));
  HostCall call(st, 0, HostCall::Memory::Owned);
  char* ws;
  call.device(&ws, ws_max);
  AM_TRY(call.start());
  for (const Group& g : groups) {
    const int nb = g.nb;
    const long long L = g.L;
    const int Tmax = g.Tmax;
    const long long n_in = offsets[g.b0 + nb] - offsets[g.b0];
    const long long nT = foff[g.b0 + nb] - foff[g.b0];
    const int n_blk = (Tmax + kTgFrames - 1) / kTgFrames;
    Workspace w;
    carve(ws, w, nb, L, Tmax, n_in, nT, win, cap, want_tempo, want_rms, want_chroma);
    float* d_x = w.x;
    float* d_pad = w.pad;
    long long* d_off = w.off;
    long long* d_n = w.n;
    long long* d_foff = w.foff;
    int* d_T = w.T;
    std::vector<long long> h_off(nb + 1), h_n(nb), h_foff(nb + 1);
    for (int i = 0; i <= nb; ++i) {
      h_off[i] = offsets[g.b0 + i] - offsets[g.b0];
      h_foff[i] = foff[g.b0 + i] - foff[g.b0];
    }
    for (int i = 0; i < nb; ++i) h_n[i] = h_off[i + 1] - h_off[i];
    AM_CUDA(cudaMemcpyAsync(d_x, samples + offsets[g.b0], n_in * 4, cudaMemcpyHostToDevice, st));
    AM_CUDA(cudaMemcpyAsync(d_off, h_off.data(), (nb + 1) * 8, cudaMemcpyHostToDevice, st));
    AM_CUDA(cudaMemcpyAsync(d_n, h_n.data(), nb * 8, cudaMemcpyHostToDevice, st));
    AM_CUDA(cudaMemcpyAsync(d_foff, h_foff.data(), (nb + 1) * 8, cudaMemcpyHostToDevice, st));
    AM_CUDA(cudaMemcpyAsync(d_T, T.data() + g.b0, nb * 4, cudaMemcpyHostToDevice, st));
    AM_LAUNCH(tf_pad_kernel, dim3((unsigned)std::min<long long>(ceil_div((int)std::min<long long>(L, INT32_MAX), 256), 4096), nb), 256, 0, st,
              d_x, d_off, (int)L, d_pad);

    if (want_tempo) {
      float *d_db = w.db, *d_dbmax = w.db_max, *d_env = w.env;
      double *d_part = w.part, *d_tg = w.tg;
      int *d_anyp = w.any_part, *d_any = w.any;
      AM_TRY(am_mel_batch_dev(plan->mel, d_pad, 0, nb, (int)L, d_db, st));
      AM_LAUNCH(tf_db_max_kernel, nb, 1024, 0, st, d_db, d_T, Tmax, d_dbmax);
      AM_LAUNCH(tf_onset_kernel, dim3(ceil_div(Tmax, 8), nb), 256, 0, st, d_db, d_dbmax, d_T, d_foff, Tmax, d_env);
      AM_LAUNCH(tf_tempogram_kernel, dim3(n_blk, nb), kTgThreads, 0, st, d_env, d_T, d_foff, win, n_blk, d_part,
                d_anyp);
      AM_LAUNCH(tf_tempogram_reduce, nb, 256, 0, st, d_part, d_anyp, d_T, win, n_blk, d_tg, d_any);
      std::vector<double> h_tg((size_t)nb * win);
      std::vector<int> h_any(nb);
      AM_CUDA(cudaMemcpyAsync(h_tg.data(), d_tg, h_tg.size() * 8, cudaMemcpyDeviceToHost, st));
      AM_CUDA(cudaMemcpyAsync(h_any.data(), d_any, nb * 4, cudaMemcpyDeviceToHost, st));
      if (onset_env)
        AM_CUDA(cudaMemcpyAsync(onset_env + foff[g.b0], d_env, nT * 4, cudaMemcpyDeviceToHost, st));
      AM_CUDA(cudaStreamSynchronize(st));
      for (int i = 0; i < nb; ++i)
        tempo[g.b0 + i] = h_any[i] ? tempo_from_tg(h_tg.data() + (size_t)i * win, win, plan->sr) : 0.0;
      if (tempogram) std::memcpy(tempogram + (size_t)g.b0 * win, h_tg.data(), h_tg.size() * 8);
    }
    if (want_rms || want_chroma) {
      TfSpecArgs a{};
      a.pad = d_pad;
      a.T_of = d_T;
      a.n_of = d_n;
      a.foff = d_foff;
      a.L = (int)L;
      a.sr = plan->sr;
      a.kmin = plan->kmin;
      a.kmax = plan->kmax;
      a.cap = cap;
      float* d_rms = w.rms;
      float* d_thr = w.thr;
      int* d_hist = w.hist;
      double* d_tun = w.tuning;
      float* d_chroma = w.chroma;
      a.rms = d_rms;
      a.pk_mag = w.pk_mag;
      a.pk_bin = w.pk_bin;
      a.pk_count = w.pk_count;
      a.chroma_fb = w.fb;
      a.chroma = d_chroma;
      const dim3 grid(ceil_div(Tmax, kFramesPerCta), nb);
      AM_LAUNCH(tf_spectrum_kernel<false>, grid, kThreads, tf_spectrum_smem(), st, a, plan->mel->t);
      if (want_chroma) {
        AM_LAUNCH(tf_tuning_kernel, nb, kTuneThreads, 0, st, a.pk_mag, a.pk_bin, a.pk_count, d_T, d_foff, cap,
                  d_thr, d_hist, d_tun);
        AM_LAUNCH(tf_chroma_fb_kernel, nb, 256, 0, st, d_tun, plan->sr, w.fb);
        AM_LAUNCH(tf_spectrum_kernel<true>, grid, kThreads, tf_spectrum_smem(), st, a, plan->mel->t);
        AM_CUDA(cudaMemcpyAsync(chroma + 12 * foff[g.b0], d_chroma, nT * 12 * 4, cudaMemcpyDeviceToHost, st));
        if (tuning) AM_CUDA(cudaMemcpyAsync(tuning + g.b0, d_tun, nb * 8, cudaMemcpyDeviceToHost, st));
        if (threshold) AM_CUDA(cudaMemcpyAsync(threshold + g.b0, d_thr, nb * 4, cudaMemcpyDeviceToHost, st));
        if (histogram)
          AM_CUDA(cudaMemcpyAsync(histogram + (size_t)g.b0 * kHistBins, d_hist, (size_t)nb * kHistBins * 4,
                                  cudaMemcpyDeviceToHost, st));
      }
      if (want_rms) AM_CUDA(cudaMemcpyAsync(rms + foff[g.b0], d_rms, nT * 4, cudaMemcpyDeviceToHost, st));
      AM_CUDA(cudaStreamSynchronize(st));
    }
  }
  return AM_OK;
}
