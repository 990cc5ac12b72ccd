// Decode + resample front end (SURVEY 8(f) row 1): what tasks/analysis.py:170-250 (robust_load_audio_with_fallback ->
// librosa.load(path, sr=48000, mono=True, duration=AUDIO_LOAD_TIMEOUT)) does before the CLAP path sees a waveform.
//
//   am_wav_info / am_wav_decode_mono   host: RIFF/WAVE reader (PCM 8 / 16 / 24 / 32 bit, IEEE float 32 / 64, also
//                                      behind WAVE_FORMAT_EXTENSIBLE), any channel count, down-mixed to mono float32
//                                      by the channel mean (librosa.to_mono).  Integer scaling follows libsndfile's
//                                      float read (x / 2^(bits-1)), which is what librosa.load returns.
//   am_resample                        device: rational polyphase resampler, the algorithm of
//                                      scipy.signal.resample_poly (zero-phase Kaiser(5.0)-windowed sinc of half length
//                                      10 max(up, down), gain up, cut-off 1 / max(up, down)); the common real-library
//                                      case 44.1 kHz -> 48 kHz is up / down = 160 / 147, 21 taps per output sample.
//                                      librosa itself resamples with soxr_hq (not installable here): PARITY UNPINNED
//                                      against librosa for non-48 kHz files; pinned against scipy's resample_poly.
//   am_audio_to_segments_dev           device form of am_pcm_to_segments (clip, * 32767 -> int16 by truncation, the
//                                      10 s / 5 s-hop windows incl. the right-aligned tail; clap_analyzer.py:502-523)
//                                      so a resampled waveform never returns to the host.
// Other containers (mp3 / flac / ogg ...) stay with the reference's own loader (pydub / ffmpeg): decode stays on host.
#include "common.cuh"
#include "host_call.cuh"

#include <algorithm>
#include <cmath>
#include <cstdio>
#include <cstdlib>
#include <map>
#include <memory>
#include <mutex>
#include <numeric>

namespace am {

// ---------------------------------------------------------------- RIFF / WAVE
struct WavFmt {
  int format = 0;        // 1 = PCM, 3 = IEEE float
  int channels = 0;
  int sample_rate = 0;
  int bits = 0;
  int block_align = 0;
  int64_t data_offset = 0, data_bytes = 0;
};

static uint32_t rd32(const uint8_t* p) { return (uint32_t)p[0] | ((uint32_t)p[1] << 8) | ((uint32_t)p[2] << 16) | ((uint32_t)p[3] << 24); }
static uint16_t rd16(const uint8_t* p) { return (uint16_t)(p[0] | (p[1] << 8)); }

static int parse_wav_header(FILE* f, const char* path, WavFmt* w) {
  uint8_t hdr[12];
  if (std::fread(hdr, 1, 12, f) != 12 || std::memcmp(hdr, "RIFF", 4) != 0 || std::memcmp(hdr + 8, "WAVE", 4) != 0) {
    set_error("am_wav: %s is not a RIFF/WAVE file", path);
    return AM_ERR_IO;
  }
  bool have_fmt = false;
  for (;;) {
    uint8_t ck[8];
    if (std::fread(ck, 1, 8, f) != 8) break;
    const uint32_t size = rd32(ck + 4);
    if (std::memcmp(ck, "fmt ", 4) == 0) {
      uint8_t b[40] = {0};
      const size_t n = std::min<size_t>(size, sizeof b);
      if (std::fread(b, 1, n, f) != n || n < 16) break;
      w->format = rd16(b);
      w->channels = rd16(b + 2);
      w->sample_rate = (int)rd32(b + 4);
      w->block_align = rd16(b + 12);
      w->bits = rd16(b + 14);
      if (w->format == 0xFFFE && n >= 26) w->format = rd16(b + 24);  // WAVE_FORMAT_EXTENSIBLE: sub-format GUID's first word
      if (size > n) std::fseek(f, (long)(size - n), SEEK_CUR);
      if (size & 1) std::fseek(f, 1, SEEK_CUR);
      have_fmt = true;
    } else if (std::memcmp(ck, "data", 4) == 0) {
      if (!have_fmt) break;
      w->data_offset = std::ftell(f);
      std::fseek(f, 0, SEEK_END);
      const int64_t remain = (int64_t)std::ftell(f) - w->data_offset;
      w->data_bytes = std::min<int64_t>((int64_t)size, remain);  // streamed files write 0xFFFFFFFF / a short count
      if (size == 0xFFFFFFFFu || size == 0) w->data_bytes = remain;
      const bool ok_fmt = (w->format == 1 && (w->bits == 8 || w->bits == 16 || w->bits == 24 || w->bits == 32)) ||
                          (w->format == 3 && (w->bits == 32 || w->bits == 64));
      if (!ok_fmt || w->channels <= 0 || w->sample_rate <= 0) {
        set_error("am_wav: %s: unsupported encoding (format tag %d, %d bits, %d channels)", path, w->format, w->bits, w->channels);
        return AM_ERR_INVALID;
      }
      if (w->block_align <= 0) w->block_align = w->channels * w->bits / 8;
      return AM_OK;
    } else {
      std::fseek(f, (long)(size + (size & 1)), SEEK_CUR);
    }
  }
  set_error("am_wav: %s has no usable fmt / data chunks", path);
  return AM_ERR_IO;
}

// ---------------------------------------------------------------- resampler
// h = up * firwin(2 * half + 1, 1 / max(up, down), window = kaiser(5.0)), as scipy.signal.resample_poly builds it
static double bessel_i0(double x) {
  double sum = 1.0, term = 1.0;
  const double q = x * x / 4.0;
  for (int k = 1; k < 200; ++k) {
    term *= q / ((double)k * k);
    sum += term;
    if (term < 1e-18 * sum) break;
  }
  return sum;
}

struct ResamplePlanHost {
  int up = 1, down = 1, half = 0, taps = 0;   // taps per phase
  int64_t n_pre_pad = 0, n_pre_remove = 0;
  std::vector<float> poly;                    // [up][taps]: poly[p][i] = h_padded[p + i * up]
};

static void build_filter(int up, int down, ResamplePlanHost* rp) {
  rp->up = up;
  rp->down = down;
  const int maxr = std::max(up, down);
  const int half = 10 * maxr;
  rp->half = half;
  const int n = 2 * half + 1;
  const double fc = 1.0 / maxr, beta = 5.0;
  std::vector<double> h((size_t)n);
  double sum = 0.0;
  const double i0b = bessel_i0(beta);
  for (int i = 0; i < n; ++i) {
    const double m = (double)i - half;
    const double x = fc * m;
    const double sinc = x == 0.0 ? 1.0 : std::sin(M_PI * x) / (M_PI * x);
    const double r = 2.0 * i / (n - 1) - 1.0;
    const double win = bessel_i0(beta * std::sqrt(std::max(0.0, 1.0 - r * r))) / i0b;
    h[(size_t)i] = fc * sinc * win;
    sum += h[(size_t)i];
  }
  for (double& v : h) v = v / sum * up;  // firwin scales to unit DC gain; resample_poly multiplies by up
  // scipy pads the filter in front so that the output is phase aligned: n_pre_pad = down - half % down
  int64_t pre_pad = down - half % down, pre_remove = (half + pre_pad) / down;
  rp->n_pre_pad = pre_pad;
  rp->n_pre_remove = pre_remove;
  const int64_t hp_len = pre_pad + n;
  rp->taps = (int)((hp_len + up - 1) / up);
  rp->poly.assign((size_t)up * rp->taps, 0.f);
  for (int64_t j = 0; j < n; ++j) {
    const int64_t q = j + pre_pad;
    rp->poly[(size_t)(q % up) * rp->taps + (size_t)(q / up)] = (float)h[(size_t)j];
  }
}

// y[k] = sum_i poly[phase][i] * x[base - i],  t = (k + n_pre_remove) * down, phase = t % up, base = t / up
// (the upfirdn identity: output sample t of the zero-stuffed, filtered signal; float64 accumulation)
__global__ void __launch_bounds__(256)
resample_kernel(const float* __restrict__ x, int64_t n_in, const float* __restrict__ poly, int up, int down, int taps,
                int64_t pre_remove, float* __restrict__ y, int64_t n_out) {
  extern __shared__ float s_poly[];
  for (int i = threadIdx.x; i < up * taps; i += blockDim.x) s_poly[i] = poly[i];
  __syncthreads();
  for (int64_t k = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; k < n_out; k += (int64_t)gridDim.x * blockDim.x) {
    const int64_t t = (k + pre_remove) * down;
    const int phase = (int)(t % up);
    const int64_t base = t / up;
    const float* p = s_poly + phase * taps;
    double acc = 0.0;
    for (int i = 0; i < taps; ++i) {
      const int64_t j = base - i;
      if (j >= 0 && j < n_in) acc = fma((double)p[i], (double)__ldg(&x[j]), acc);
    }
    y[k] = (float)acc;
  }
}

// clip, * 32767 -> int16 (truncation), windows of `seg` samples every `hop`, right-aligned tail window when
// n_seg * hop < L (clap_analyzer.py:502-523); window s starts at start[s]; samples beyond L are zero (short tracks)
__global__ void __launch_bounds__(256)
audio_to_segments_kernel(const float* __restrict__ audio, int64_t L, int seg, int hop, int n_regular, int n_seg,
                         int16_t* __restrict__ out) {
  const int64_t total = (int64_t)n_seg * seg;
  for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (int64_t)gridDim.x * blockDim.x) {
    const int s = (int)(i / seg);
    const int64_t o = i - (int64_t)s * seg;
    const int64_t start = s < n_regular ? (int64_t)s * hop : L - seg;
    const int64_t j = start + o;
    float v = (j >= 0 && j < L) ? audio[j] : 0.f;
    v = fminf(fmaxf(v, -1.0f), 1.0f) * 32767.0f;
    out[i] = (int16_t)v;  // float -> int conversion truncates toward zero, like numpy's astype(int16)
  }
}

}  // namespace am

using namespace am;

struct ResamplePlan {
  ResamplePlanHost host;
  DevBuf<float> poly_dev;
};

extern "C" int am_wav_info(const char* path, int* sample_rate, int* channels, int64_t* frames, int* bits) {
  AM_CHECK(path != nullptr, "am_wav_info: NULL path");
  FILE* f = std::fopen(path, "rb");
  if (!f) {
    set_error("am_wav: cannot open %s", path);
    return AM_ERR_IO;
  }
  WavFmt w;
  const int s = parse_wav_header(f, path, &w);
  std::fclose(f);
  AM_TRY(s);
  if (sample_rate) *sample_rate = w.sample_rate;
  if (channels) *channels = w.channels;
  if (frames) *frames = w.data_bytes / w.block_align;
  if (bits) *bits = w.format == 3 ? -w.bits : w.bits;
  return AM_OK;
}

extern "C" int am_wav_decode_mono(const char* path, int64_t max_frames, float* out, int64_t cap, int64_t* n_frames,
                                  int* sample_rate) {
  AM_CHECK(path && n_frames, "am_wav_decode_mono: NULL argument");
  FILE* f = std::fopen(path, "rb");
  if (!f) {
    set_error("am_wav: cannot open %s", path);
    return AM_ERR_IO;
  }
  WavFmt w;
  int s = parse_wav_header(f, path, &w);
  if (s != AM_OK) {
    std::fclose(f);
    return s;
  }
  int64_t frames = w.data_bytes / w.block_align;
  if (max_frames >= 0) frames = std::min(frames, max_frames);
  *n_frames = frames;
  if (sample_rate) *sample_rate = w.sample_rate;
  if (!out) {  // size query
    std::fclose(f);
    return AM_OK;
  }
  if (cap < frames) {
    std::fclose(f);
    set_error("am_wav_decode_mono: buffer of %lld frames, file has %lld", (long long)cap, (long long)frames);
    return AM_ERR_INVALID;
  }
  std::fseek(f, (long)w.data_offset, SEEK_SET);
  const int ch = w.channels, bps = w.bits / 8;
  const int64_t chunk = 1 << 16;
  std::vector<uint8_t> buf((size_t)chunk * w.block_align);
  for (int64_t f0 = 0; f0 < frames; f0 += chunk) {
    const int64_t nf = std::min(chunk, frames - f0);
    const size_t got = std::fread(buf.data(), (size_t)w.block_align, (size_t)nf, f);
    if ((int64_t)got != nf) {
      std::fclose(f);
      set_error("am_wav: short read on %s", path);
      return AM_ERR_IO;
    }
    if (w.format == 1 && w.bits == 16 && ch <= 2 && w.block_align == 2 * ch) {
      // PCM16 mono / stereo: the common library file; branch-free loops the compiler vectorises
      const int16_t* q = reinterpret_cast<const int16_t*>(buf.data());
      float* o = out + f0;
      if (ch == 1) {
        for (int64_t i = 0; i < nf; ++i) o[i] = (float)q[i] / 32768.0f;
      } else {
        for (int64_t i = 0; i < nf; ++i) o[i] = ((float)q[2 * i] / 32768.0f + (float)q[2 * i + 1] / 32768.0f) / 2.0f;
      }
      continue;
    }
    for (int64_t i = 0; i < nf; ++i) {
      const uint8_t* p = buf.data() + (size_t)i * w.block_align;
      float acc = 0.f;
      for (int c = 0; c < ch; ++c, p += bps) {
        float v;
        if (w.format == 3) {
          if (w.bits == 32) std::memcpy(&v, p, 4);
          else {
            double dv;
            std::memcpy(&dv, p, 8);
            v = (float)dv;
          }
        } else if (w.bits == 16) {
          v = (float)(int16_t)rd16(p) / 32768.0f;
        } else if (w.bits == 8) {
          v = ((float)p[0] - 128.0f) / 128.0f;
        } else if (w.bits == 24) {
          const int32_t q = (int32_t)((uint32_t)p[0] << 8 | (uint32_t)p[1] << 16 | (uint32_t)p[2] << 24) >> 8;
          v = (float)q / 8388608.0f;
        } else {
          v = (float)((double)(int32_t)rd32(p) / 2147483648.0);
        }
        acc += v;  // float32 channel sum in channel order, then / channels: numpy's mean over the channel axis
      }
      out[f0 + i] = ch == 1 ? acc : acc / (float)ch;
    }
  }
  std::fclose(f);
  return AM_OK;
}

// One call per file for the common case (a 48 kHz WAV): decode -> mono float32 -> the reference's clip / * 32767 / int16
// truncation / 10 s windows (am_pcm_to_segments), no Python-side temporaries; the GIL is released for the whole call,
// so a thread pool scales with the cores.  seg == NULL reports *n_seg and *duration_sec only.  A file at another rate
// returns AM_ERR_INVALID ("needs resampling"): the caller goes through am_wav_decode_mono + am_resample.
extern "C" int am_wav_to_segments(const char* path, double max_seconds, int16_t* seg, int max_seg, int* n_seg,
                                  double* duration_sec) {
  AM_CHECK(path && n_seg, "am_wav_to_segments: NULL argument");
  int sr = 0, ch = 0, bits = 0;
  int64_t frames = 0;
  AM_TRY(am_wav_info(path, &sr, &ch, &frames, &bits));
  if (sr != 48000) {
    set_error("am_wav_to_segments: %s is at %d Hz: needs resampling", path, sr);
    return AM_ERR_INVALID;
  }
  const int64_t limit = max_seconds >= 0 ? (int64_t)(max_seconds * sr) : -1;
  const int64_t L = limit >= 0 ? std::min(frames, limit) : frames;
  AM_CHECK(L > 0, "am_wav_to_segments: %s holds no audio", path);
  *n_seg = am_num_segments(L);
  if (duration_sec) *duration_sec = (double)L / sr;
  if (!seg) return AM_OK;
  AM_CHECK(max_seg >= *n_seg, "am_wav_to_segments: room for %d windows, need %d", max_seg, *n_seg);
  std::vector<float> audio((size_t)L);
  int64_t got = 0;
  AM_TRY(am_wav_decode_mono(path, L, audio.data(), L, &got, &sr));
  return am_pcm_to_segments(audio.data(), got, seg, max_seg, n_seg);
}

static int resample_plan_create(int sr_in, int sr_out, ResamplePlan** out) {
  AM_CHECK(sr_in > 0 && sr_out > 0, "am_resample: bad rates %d -> %d", sr_in, sr_out);
  const int g = std::gcd(sr_in, sr_out);
  const int up = sr_out / g, down = sr_in / g;
  AM_CHECK(up <= 1024 && down <= 4096, "am_resample: %d -> %d needs up / down = %d / %d (unsupported ratio)", sr_in,
           sr_out, up, down);
  AM_TRY(ensure_init());
  auto p = std::make_unique<ResamplePlan>();
  build_filter(up, down, &p->host);
  AM_CHECK((size_t)up * p->host.taps * 4 <= 200 * 1024, "am_resample: polyphase table too large");
  AM_TRY(p->poly_dev.alloc(p->host.poly.size()));
  AM_CUDA(cudaMemcpy(p->poly_dev.p, p->host.poly.data(), p->host.poly.size() * 4, cudaMemcpyHostToDevice));
  *out = p.release();
  return AM_OK;
}

static int64_t resample_out_len(const ResamplePlan* p, int64_t n_in) {
  return (n_in * p->host.up + p->host.down - 1) / p->host.down;  // ceil(n * up / down), as resample_poly
}

static int resample_dev(const ResamplePlan* p, const float* x_dev, int64_t n_in, float* y_dev, cudaStream_t stream) {
  const int64_t n_out = resample_out_len(p, n_in);
  const size_t smem = p->host.poly.size() * 4;  // <= 200 KiB (resample_plan_create)
  AM_TRY(allow_dynamic_smem<resample_kernel>(200 * 1024));
  const int grid = (int)std::max<int64_t>(1, std::min<int64_t>((n_out + 255) / 256, (int64_t)sm_count() * 8));
  AM_LAUNCH(resample_kernel, grid, 256, smem, stream, x_dev, n_in, p->poly_dev.p, p->host.up, p->host.down,
            p->host.taps, p->host.n_pre_remove, y_dev, n_out);
  return AM_OK;
}

// x f32[n_in] at sr_in -> y f32[ceil(n_in * up / down)] at sr_out.  Re-entrant and stream-ordered (called
// from decoder threads while the encoder runs): the plan of a rate pair is built once and cached, scratch comes from
// the stream-ordered pool of the calling thread's own stream -- no cudaMalloc / cudaFree, which would wait for every
// kernel in flight on the device.
extern "C" int am_resample(const float* x, int64_t n_in, int sr_in, int sr_out, float* y, int64_t cap, int64_t* n_out) {
  AM_CHECK(x && y && n_out && n_in > 0, "am_resample: bad argument");
  static std::mutex mu;
  static std::map<std::pair<int, int>, ResamplePlan*> plans;  // process lifetime
  ResamplePlan* p = nullptr;
  {
    std::lock_guard<std::mutex> lk(mu);
    auto it = plans.find({sr_in, sr_out});
    if (it == plans.end()) {
      AM_TRY(resample_plan_create(sr_in, sr_out, &p));
      plans[{sr_in, sr_out}] = p;
    } else {
      p = it->second;
    }
  }
  *n_out = resample_out_len(p, n_in);
  AM_CHECK(cap >= *n_out, "am_resample: output buffer of %lld samples, need %lld", (long long)cap, (long long)*n_out);
  cudaStream_t st;
  AM_TRY(HostCall::thread_stream(&st));
  HostCall call(st, 0, HostCall::Memory::Pool);
  float *dx, *dy;
  call.up(&dx, x, (size_t)n_in);
  call.down(&dy, (size_t)*n_out, y);
  AM_TRY(call.start());
  AM_TRY(resample_dev(p, dx, n_in, dy, st));
  return call.finish();
}

// windows a waveform of L samples produces (clap_analyzer.py:510-521): 1 when L <= 480000, else the regular windows
// plus the tail window when n_regular * hop < L
extern "C" int am_num_segments(int64_t L) {
  const int64_t seg = 480000, hop = 240000;
  if (L <= seg) return 1;
  int n = 0;
  for (int64_t start = 0; start + seg <= L; start += hop) ++n;
  if ((int64_t)n * hop < L) ++n;
  return n;
}

extern "C" int am_audio_to_segments_dev(const float* audio_dev, int64_t L, int16_t* seg_dev, int max_seg, int* n_seg,
                                        void* stream) {
  AM_CHECK(audio_dev && n_seg && L > 0, "am_audio_to_segments_dev: bad argument");
  const int seg = 480000, hop = 240000;
  const int total = am_num_segments(L);
  *n_seg = total;
  if (!seg_dev) return AM_OK;
  AM_CHECK(max_seg >= total, "am_audio_to_segments_dev: room for %d windows, need %d", max_seg, total);
  int n_regular = 0;
  if (L <= seg) n_regular = 1;  // single zero-padded window starting at 0
  else
    for (int64_t start = 0; start + seg <= L; start += hop) ++n_regular;
  AM_TRY(ensure_init());
  const int grid = (int)std::min<int64_t>(((int64_t)total * seg + 255) / 256, (int64_t)sm_count() * 8);
  AM_LAUNCH(audio_to_segments_kernel, grid, 256, 0, (cudaStream_t)stream, audio_dev, L, seg, hop, n_regular, total, seg_dev);
  return AM_OK;
}
