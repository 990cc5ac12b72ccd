// K2 + K3: student CLAP audio encoder, batched (sm_90a).
//
// Replaces the per-segment onnxruntime call of tasks/clap_analyzer.py:534 and the numpy pooling
// at :552-562.  Architecture: student_clap/models/student_onnx_model.py (bn0 over mel bins ->
// PhiNet inverted-residual trunk (ReLU6, no SE: compatibility=True) -> 1x1 stride-2 conv to 2048
// -> spatial mean -> Projection (linear1, GELU, linear2, residual, LayerNorm) -> L2).
//
// Data layout in HBM: activations are NHWC bf16 [B, H, W, Cp] with Cp = channels rounded up to 16
// (padded channels are exact zeros: zero weight rows + zero bias), so every 1x1 convolution is
// one K-major GEMM  D[B*H*W, Cout] = A[B*H*W, Cin] x W[Cout, Cin]^T  on the wgmma path
// (gemm.cu) with the folded-BatchNorm bias, ReLU6 and the residual add fused in its epilogue.
// Depthwise 3x3 (+BN+ReLU6) is a bandwidth kernel over 8-channel (16-byte) vectors (depthwise.cu).  The stem
// (bn0 + pad + 3x3 stride-2 on the single input channel + 1x1 + BN + ReLU6) reads the fp32
// log-mel directly and is computed in fp32.  The head (<= 2.5 MMAC per window) runs in fp32.
#include "common.cuh"
#include "host_call.cuh"

#include <algorithm>
#include <cmath>
#include <cstdio>
#include <functional>
#include <memory>

#include "depthwise.cuh"
#include "encoder_generic.cuh"
#include "fused_block.cuh"
#include "gemm_wgmma.cuh"
#include "model_spec.cuh"

namespace am {

struct Layer {
  int type = 0;
  int cin = 0, cout = 0, cin_p = 0, cout_p = 0;
  int kh = 1, kw = 1;
  int stride = 1, act = 0, block_start = 0, residual = 0;
  int pad_t = 0, pad_b = 0, pad_l = 0, pad_r = 0;
  int h_is_time = 1, gate_act = 0, cmid = 0;
  DevBuf<__nv_bfloat16> w_bf16;  // pointwise: [cout_p, cin_p]
  DevBuf<float> w_f32;           // depthwise: [k*k, c_p]; stem: dw[9]; first conv: [kh*kw, c_p]; squeeze-excite: fc1 [cmid, c]
  DevBuf<float> bias;            // [cout_p]  (squeeze-excite: fc1 bias [cmid])
  DevBuf<float> aux0, aux1, aux2;  // stem / first conv: per-mel scale / shift (+ stem pw scale); squeeze-excite: fc2 [c, cmid], fc2 bias
  DevBuf<float> fused_params;    // 3x3 depthwise: its weights, bias and the preceding pointwise layer's bias per 64-channel chunk (fused::pack_params)
  bool dw_fp16 = false;          // 3x3 depthwise: layer by layer, the packed-fp16 kernels cannot overflow on it (dw3x3_fp16_safe)
  // true for the 3x3 / pad 1 / ReLU6 depthwise the packed-fp16 kernels and the fused block kernel implement
  bool dw_fast() const {
    return type == kDepthwise && kh == 3 && kw == 3 && pad_t == 1 && pad_b == 1 && pad_l == 1 && pad_r == 1 && act == kActRelu6;
  }
};

// one operation of the head's row program (model_spec.cuh: VecOp) with its weights on the device
struct HeadOp {
  int kind = 0, a = -1, b = -1, dst = -1, K = 0, N = 0, act = 0, stride = 1;
  float eps = 0.f, eps2 = 0.f;
  DevBuf<float> w, bias;          // LayerNorm gain / shift, affine scale / shift; kVecLinear: bias
  DevBuf<__nv_bfloat16> w3;       // kVecLinear: bf16 [N, 3*Kp] = [hi | lo | hi] (see split3_kernel)
  bool has_w = false, has_bias = false;
};

static inline int pad16(int c) { return (int)round_up((size_t)c, 16); }

// ---------------------------------------------------------------- kernels
// stem: mel f32 [B, n_mels, T] -> NHWC bf16 [B, Ho, Wo, Cp];  image H = time, W = mel bin.
// A CTA owns a tile of 32 output rows (time) x 8 output columns (mel) of one window.
//   phase 1: one thread per pixel computes the single-channel 3x3 stride-2 response; lanes of a warp
//            walk the TIME axis (contiguous in the mel layout), so each tap is a 256-byte strided read
//            instead of 32 scattered sectors;
//   phase 2: the 256 responses are expanded to Cp channels, consecutive threads writing consecutive
//            16-byte groups (8 pixels x Cp x 2 B contiguous runs per output row).
constexpr int kStemTH = 32, kStemTW = 8;

__global__ void __launch_bounds__(256)
stem_kernel(const float* __restrict__ mel, int B, int n_mels, int T, int Ho, int Wo, int pad_t, int pad_l,
            const float* __restrict__ bn_scale, const float* __restrict__ bn_shift,
            const float* __restrict__ dw, const float* __restrict__ pw_scale,
            const float* __restrict__ pw_shift, int cp, __nv_bfloat16* __restrict__ out) {
  __shared__ float s_v[kStemTH * kStemTW];
  extern __shared__ float s_pw[];  // [2 * cp]: scale, shift
  const int groups = cp >> 3;
  const int tiles_h = (Ho + kStemTH - 1) / kStemTH, tiles_w = (Wo + kStemTW - 1) / kStemTW;
  const int64_t n_tiles = (int64_t)B * tiles_h * tiles_w;
  for (int i = threadIdx.x; i < cp; i += 256) {
    s_pw[i] = pw_scale[i];
    s_pw[cp + i] = pw_shift[i];
  }
  float wdw[9];
#pragma unroll
  for (int i = 0; i < 9; ++i) wdw[i] = __ldg(&dw[i]);
  // phase-2 mapping: a thread keeps ONE channel group (its 8 scales + 8 shifts live in registers) and
  // walks the tile's pixels; consecutive threads = consecutive groups of one pixel, then the next pixel,
  // so a warp still writes contiguous 16-byte runs.  (Reading the 16 constants from shared memory per
  // item made the kernel LSU-bound at 3x its write roofline.)
  const int g_step = groups < 256 ? groups : 256;
  const int pix_lanes = 256 / g_step;
  const int g0 = (int)threadIdx.x % g_step, pl = (int)threadIdx.x / g_step;
  float sc[8], sh[8];
  int g_regs = -1;
  __syncthreads();
  if (pl < pix_lanes) {
#pragma unroll
    for (int e = 0; e < 8; ++e) {
      sc[e] = s_pw[g0 * 8 + e];
      sh[e] = s_pw[cp + g0 * 8 + e];
    }
    g_regs = g0;
  }
  for (int64_t tile = blockIdx.x; tile < n_tiles; tile += gridDim.x) {
    const int tw = (int)(tile % tiles_w);
    const int64_t t1 = tile / tiles_w;
    const int th = (int)(t1 % tiles_h);
    const int b = (int)(t1 / tiles_h);
    const int ho0 = th * kStemTH, wo0 = tw * kStemTW;
    __syncthreads();
    {
      const int hl = threadIdx.x & (kStemTH - 1), wl = threadIdx.x / kStemTH;  // lanes walk the time axis
      const int ho = ho0 + hl, wo = wo0 + wl;
      float v = 0.f;
      if (ho < Ho && wo < Wo) {
        const float* m = mel + (int64_t)b * n_mels * T;
#pragma unroll
        for (int dx = 0; dx < 3; ++dx) {
          const int w = 2 * wo + dx - pad_l;
          if (w < 0 || w >= n_mels) continue;
          const float bsc = __ldg(&bn_scale[w]), bsh = __ldg(&bn_shift[w]);
#pragma unroll
          for (int dy = 0; dy < 3; ++dy) {
            const int h = 2 * ho + dy - pad_t;
            if (h < 0 || h >= T) continue;
            v = fmaf(wdw[dy * 3 + dx], fmaf(__ldg(&m[(int64_t)w * T + h]), bsc, bsh), v);
          }
        }
      }
      s_v[hl * kStemTW + wl] = v;
    }
    __syncthreads();
    const int nw = min(kStemTW, Wo - wo0), nh = min(kStemTH, Ho - ho0);
    for (int g = g0; g < groups && pl < pix_lanes; g += g_step) {
      if (g != g_regs) {  // only when groups > 256 (never for the shipped students)
#pragma unroll
        for (int e = 0; e < 8; ++e) {
          sc[e] = s_pw[g * 8 + e];
          sh[e] = s_pw[cp + g * 8 + e];
        }
        g_regs = g;
      }
      for (int p = pl; p < nh * nw; p += pix_lanes) {
        const int hl = (nw == kStemTW) ? (p >> 3) : p / nw;  // ragged right-edge tiles only
        const int wl = p - hl * nw;
        const float v = s_v[hl * kStemTW + wl];
      float o8[8];
#pragma unroll
      for (int e = 0; e < 8; ++e) o8[e] = relu6f(fmaf(v, sc[e], sh[e]));
      uint4 pk;
      __nv_bfloat162 t;
      t = __floats2bfloat162_rn(o8[0], o8[1]); pk.x = *reinterpret_cast<uint32_t*>(&t);
      t = __floats2bfloat162_rn(o8[2], o8[3]); pk.y = *reinterpret_cast<uint32_t*>(&t);
      t = __floats2bfloat162_rn(o8[4], o8[5]); pk.z = *reinterpret_cast<uint32_t*>(&t);
      t = __floats2bfloat162_rn(o8[6], o8[7]); pk.w = *reinterpret_cast<uint32_t*>(&t);
      const int64_t pix = ((int64_t)b * Ho + ho0 + hl) * Wo + wo0 + wl;
      *reinterpret_cast<uint4*>(out + (pix * groups + g) * 8) = pk;
      }
    }
  }
}

// head step 1: mean over the positions a 1x1 stride-s conv visits -> f32 [B, C]
__global__ void strided_mean_kernel(const __nv_bfloat16* __restrict__ in, int H, int W, int cp, int C, int stride,
                                    float* __restrict__ out) {
  const int b = blockIdx.x;
  const int hs = (H + stride - 1) / stride, ws = (W + stride - 1) / stride;
  const float inv = 1.0f / (float)(hs * ws);
  for (int c = threadIdx.x; c < C; c += blockDim.x) {
    float acc = 0.f;
    for (int h = 0; h < H; h += stride)
      for (int w = 0; w < W; w += stride) acc += __bfloat162float(in[(((int64_t)b * H + h) * W + w) * cp + c]);
    out[(int64_t)b * C + c] = acc * inv;
  }
}

// fp32 -> three bf16 terms so that ONE bf16 tensor-core GEMM over K' = 3*Kp reproduces the fp32 product to ~2^-16:
//   x = hi + lo (+ 2^-17 x),  A' = [hi | hi | lo],  W' = [hi | lo | hi]  =>  A'.W'^T = hi.hi + hi.lo + lo.hi
// (the dropped lo.lo term is 2^-18).  The head's three linears are 0.7 GFLOP in total: on CUDA cores they were
// latency bound at 0.45 ms, as split-bf16 GEMMs on the wgmma kernel they are a few microseconds each.
__global__ void __launch_bounds__(256)
split3_kernel(const float* __restrict__ x, int B, int K, int Kp, int in_act, __nv_bfloat16* __restrict__ out) {
  const int64_t n = (int64_t)B * Kp;
  for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (int64_t)gridDim.x * blockDim.x) {
    const int64_t b = i / Kp;
    const int k = (int)(i - b * Kp);
    float v = 0.f;
    if (k < K) {
      v = apply_act(in_act, x[b * K + k]);
    }
    const __nv_bfloat16 hi = __float2bfloat16_rn(v);
    const __nv_bfloat16 lo = __float2bfloat16_rn(v - __bfloat162float(hi));
    __nv_bfloat16* o = out + b * 3 * Kp + k;
    o[0] = hi;
    o[Kp] = hi;
    o[2 * Kp] = lo;
  }
}

// W fp32 [N, K] -> bf16 [N, 3*Kp] = [hi | lo | hi]
static int upload_split3(DevBuf<__nv_bfloat16>& dst, const std::vector<float>& w, int N, int K) {
  const int Kp = (int)round_up((size_t)K, 8);
  std::vector<__nv_bfloat16> h((size_t)N * 3 * Kp, __float2bfloat16_rn(0.f));
  for (int n = 0; n < N; ++n)
    for (int k = 0; k < K; ++k) {
      const float v = w[(size_t)n * K + k];
      const __nv_bfloat16 hi = __float2bfloat16_rn(v);
      const __nv_bfloat16 lo = __float2bfloat16_rn(v - __bfloat162float(hi));
      __nv_bfloat16* o = h.data() + (size_t)n * 3 * Kp + k;
      o[0] = hi;
      o[Kp] = lo;
      o[2 * Kp] = hi;
    }
  AM_TRY(dst.alloc(h.size()));
  AM_CUDA(cudaMemcpy(dst.p, h.data(), h.size() * sizeof(__nv_bfloat16), cudaMemcpyHostToDevice));
  return AM_OK;
}

// head final: z = LayerNorm(e1 + e2) * g + b ; out = z / max(||z||, eps2)   (one CTA per row)
__global__ void __launch_bounds__(256)
head_finalize_kernel(const float* __restrict__ e1, const float* __restrict__ e2, int E, const float* __restrict__ g,
                     const float* __restrict__ bt, float eps, float eps2, float* __restrict__ out) {
  __shared__ float s_red[32];
  __shared__ float s_stat[2];
  const int b = blockIdx.x, tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  const float* a = e1 + (int64_t)b * E;
  const float* c = e2 + (int64_t)b * E;
  auto block_sum = [&](float v) {
    v = warp_sum(v);
    if (lane == 0) s_red[warp] = v;
    __syncthreads();
    float t = 0.f;
    if (warp == 0) {
      t = lane < (blockDim.x >> 5) ? s_red[lane] : 0.f;
      t = warp_sum(t);
      if (lane == 0) s_stat[0] = t;
    }
    __syncthreads();
    const float r = s_stat[0];
    __syncthreads();
    return r;
  };
  float loc = 0.f;
  for (int i = tid; i < E; i += blockDim.x) loc += a[i] + c[i];
  const float mean = block_sum(loc) / (float)E;
  loc = 0.f;
  for (int i = tid; i < E; i += blockDim.x) {
    const float d = a[i] + c[i] - mean;
    loc = fmaf(d, d, loc);
  }
  const float var = block_sum(loc) / (float)E;
  const float rstd = rsqrtf(var + eps);
  loc = 0.f;
  for (int i = tid; i < E; i += blockDim.x) {
    const float z = (a[i] + c[i] - mean) * rstd * g[i] + bt[i];
    loc = fmaf(z, z, loc);
  }
  const float nrm = fmaxf(sqrtf(block_sum(loc)), eps2);
  for (int i = tid; i < E; i += blockDim.x) {
    const float z = (a[i] + c[i] - mean) * rstd * g[i] + bt[i];
    out[(int64_t)b * E + i] = z / nrm;
  }
}

// K3: per-track mean of window embeddings, then / (||.|| + 1e-9)   (clap_analyzer.py:552-562)
__global__ void __launch_bounds__(256)
track_pool_kernel(const float* __restrict__ seg_emb, const int32_t* __restrict__ seg_off, int E,
                  float* __restrict__ out) {
  __shared__ float s_red[8];
  __shared__ float s_norm;
  const int t = blockIdx.x, tid = threadIdx.x;
  const int s0 = seg_off[t], s1 = seg_off[t + 1];
  const int n = s1 - s0;
  float loc = 0.f;
  for (int i = tid; i < E; i += blockDim.x) {
    float acc = 0.f;
    for (int s = s0; s < s1; ++s) acc += seg_emb[(int64_t)s * E + i];
    const float m = n > 0 ? acc / (float)n : 0.f;
    out[(int64_t)t * E + i] = m;
    loc = fmaf(m, m, loc);
  }
  loc = warp_sum(loc);
  if ((tid & 31) == 0) s_red[tid >> 5] = loc;
  __syncthreads();
  if (tid == 0) {
    float tot = 0.f;
    for (int w = 0; w < (int)(blockDim.x >> 5); ++w) tot += s_red[w];
    s_norm = sqrtf(tot) + 1e-9f;
  }
  __syncthreads();
  if (n > 0)
    for (int i = tid; i < E; i += blockDim.x) out[(int64_t)t * E + i] /= s_norm;
}

template <typename T>
static int upload(DevBuf<T>& dst, const std::vector<T>& src) {
  AM_TRY(dst.alloc(std::max<size_t>(src.size(), 1)));
  if (!src.empty()) AM_CUDA(cudaMemcpy(dst.p, src.data(), src.size() * sizeof(T), cudaMemcpyHostToDevice));
  return AM_OK;
}

static std::vector<float> padded(const std::vector<float>& v, size_t n) {
  std::vector<float> o(n, 0.f);
  std::copy(v.begin(), v.begin() + std::min(n, v.size()), o.begin());
  return o;
}

struct Shape {
  int H, W;
};

// One launch group of the trunk.
enum StepKind { kStepStem, kStepConvFirst, kStepFused, kStepPointwise, kStepDw3x3, kStepDwGeneric, kStepSqueezeExcite };

struct Step {
  int kind = 0;
  size_t first = 0, last = 0;  // layers [first, last] it runs; kStepFused: [expansion,] depthwise, projection
  Shape in{0, 0}, out{0, 0};
  int cout_p = 0;              // padded channels of its output
  bool starts_block = false;   // its input is the residual source until the next such step
  fused::BlockDesc desc{};     // kStepFused
  fused::Plan plan;
};

// What runs for windows of T frames: every decision that depends on the shapes is taken here, once.  run_steps, the
// workspace sizes and the flop counts of am_clap_flops_* all read it.
struct ForwardPlan {
  int T = 0;  // 0: not built
  std::vector<Step> steps;
  size_t late_step = 0;  // steps [0, late_step) are the early phase
  Shape split{0, 0};     // input of the late phase: shape and padded channels
  int split_c = 0;
  // per-window elements of the largest layer output of each phase, the expanded tensors included (blocks run layer by
  // layer with AM_FUSED_BLOCKS=0 or when a block does not fit the fused kernel)
  size_t early_act = 0, late_act = 0;
};

}  // namespace am

struct am_model {
  int n_mels = 0, emb = 0;
  std::string source;
  std::vector<std::unique_ptr<am::Layer>> layers;
  std::vector<std::unique_ptr<am::HeadOp>> head;  // row program: pool, linears, ..., the last op writes the embedding
  std::vector<int> reg_dim;
  std::vector<std::unique_ptr<am::DevBuf<float>>> regs;  // head registers f32 [n, reg_dim]
  int head_cin = 0, head_cin_p = 0;                      // channels the trunk hands to the head's pooling
  // workspace (grown on demand, reused across calls; one user thread per model)
  am::DevBuf<__nv_bfloat16> act[3];
  am::DevBuf<float> mel_ws, seg_emb, se_mean, se_gate;
  am::DevBuf<__nv_bfloat16> a3;       // head GEMM operand [n, 3 * Kp] (split3_kernel)
  am::DevBuf<__nv_bfloat16> late_in;  // [n, H, W, C] output of the early layers for all windows of a call
  int late_sub = 256;                 // windows per pass of the late phase
  size_t act_elems = 0;
  am::ForwardPlan plan;               // of the window length of the latest call (plan_for)
  am::Stream stream;         // compute stream of the host-pointer entry points
  am::Stream copy_stream;    // H2D staging stream (host API): copies of chunk i+1 overlap compute of chunk i
  am::DevBuf<int16_t> pcm_stage[2];
  am::DevBuf<int32_t> off_stage;
  am::DevBuf<float> out_stage;
  am::Event ev_copied[2], ev_done[2];
  // submitted-but-not-collected host calls (am_clap_embed_tracks_submit / _collect): results land in pinned
  // staging first, so the D2H is truly asynchronous and the NEXT call's H2D + early blocks overlap this call's tail
  struct Ticket {
    am::PinnedBuf<float> stage;
    float* user_out = nullptr;
    size_t count = 0;
    am::Event ready;
    bool open = false;
  } tickets[2];
  unsigned n_submitted = 0, n_collected = 0;
  bool slot_used[2] = {false, false};
  am_mel_plan* host_plan = nullptr;  // mel plan of the host entry point, cached per cfg (building one = host trig
  am_mel_cfg host_plan_cfg{};        // tables + cudaMalloc + upload: ~1 ms, was paid on every call)
  int fused_blocks = 1;      // AM_FUSED_BLOCKS=0: every block layer by layer (fused_block.cu otherwise)
  ~am_model() {
    if (host_plan) am_mel_plan_free(host_plan);
  }
};

namespace am {

// output extent of a spatial layer (first conv / stem / depthwise); 1x1 layers keep the shape
static Shape layer_out(const Layer& l, Shape s) {
  if (l.type == kDepthwise || l.type == kConvFirst || l.type == kStem)
    return {(s.H + l.pad_t + l.pad_b - l.kh) / l.stride + 1, (s.W + l.pad_l + l.pad_r - l.kw) / l.stride + 1};
  return s;
}

// ModelSpec -> device model: pads channels to 16, converts weights to the kernels' layouts, validates the chain
static int build_model(am_model* m, const ModelSpec& spec) {
  m->n_mels = spec.n_mels;
  m->emb = spec.emb;
  m->source = spec.source;
  if (spec.layers.empty() || (spec.layers[0].type != kStem && spec.layers[0].type != kConvFirst) || spec.head.empty() ||
      spec.emb <= 0 || spec.n_mels <= 0) {
    set_error("weights: model must start with a convolution on the mel spectrogram and end with a head");
    return AM_ERR_IO;
  }
  int c = 0;
  for (size_t li = 0; li < spec.layers.size(); ++li) {
    const LayerSpec& S = spec.layers[li];
    auto L = std::make_unique<Layer>();
    L->type = S.type;
    L->cin = S.cin;
    L->cout = S.cout;
    L->cin_p = pad16(S.cin);
    L->cout_p = pad16(S.cout);
    L->kh = S.kh;
    L->kw = S.kw;
    L->stride = S.stride;
    L->act = S.act;
    L->block_start = S.block_start;
    L->residual = S.residual;
    L->pad_t = S.pad_t;
    L->pad_b = S.pad_b;
    L->pad_l = S.pad_l;
    L->pad_r = S.pad_r;
    L->h_is_time = S.h_is_time;
    L->gate_act = S.gate_act;
    L->cmid = S.cmid;
    if (li > 0 && S.cin != c) {
      set_error("weights: layer %zu expects %d input channels, previous layer produces %d", li, S.cin, c);
      return AM_ERR_IO;
    }
    if (li > 0 && (S.type == kStem || S.type == kConvFirst)) {
      set_error("weights: layer %zu: a first convolution in the middle of the trunk", li);
      return AM_ERR_IO;
    }
    if (S.type == kStem) {
      AM_TRY(upload(L->aux0, S.aux0));
      AM_TRY(upload(L->aux1, S.aux1));
      AM_TRY(upload(L->w_f32, S.w));
      AM_TRY(upload(L->aux2, padded(S.aux2, L->cout_p)));
      AM_TRY(upload(L->bias, padded(S.bias, L->cout_p)));
    } else if (S.type == kConvFirst) {
      const int taps = S.kh * S.kw;
      if (S.w.size() != (size_t)S.cout * taps || S.bias.size() != (size_t)S.cout ||
          (!S.aux0.empty() && (S.aux0.size() != (size_t)spec.n_mels || S.aux1.size() != (size_t)spec.n_mels))) {
        set_error("weights: malformed first convolution");
        return AM_ERR_IO;
      }
      std::vector<float> wt((size_t)taps * L->cout_p, 0.f);
      for (int o = 0; o < S.cout; ++o)
        for (int t = 0; t < taps; ++t) wt[(size_t)t * L->cout_p + o] = S.w[(size_t)o * taps + t];
      AM_TRY(upload(L->w_f32, wt));
      AM_TRY(upload(L->bias, padded(S.bias, L->cout_p)));
      if (!S.aux0.empty()) {
        AM_TRY(upload(L->aux0, S.aux0));
        AM_TRY(upload(L->aux1, S.aux1));
      }
    } else if (S.type == kPointwise) {
      if (S.w.size() != (size_t)S.cin * S.cout || S.bias.size() != (size_t)S.cout) {
        set_error("weights: malformed pointwise layer %zu", li);
        return AM_ERR_IO;
      }
      std::vector<__nv_bfloat16> wb((size_t)L->cout_p * L->cin_p, __float2bfloat16_rn(0.f));
      for (int o = 0; o < S.cout; ++o)
        for (int i = 0; i < S.cin; ++i) wb[(size_t)o * L->cin_p + i] = __float2bfloat16_rn(S.w[(size_t)o * S.cin + i]);
      AM_TRY(upload(L->w_bf16, wb));
      AM_TRY(upload(L->bias, padded(S.bias, L->cout_p)));
    } else if (S.type == kDepthwise) {
      const int taps = S.kh * S.kw;
      if (S.w.size() != (size_t)S.cin * taps || S.bias.size() != (size_t)S.cin) {
        set_error("weights: malformed depthwise layer %zu", li);
        return AM_ERR_IO;
      }
      std::vector<float> wt((size_t)taps * L->cin_p, 0.f);
      for (int ch = 0; ch < S.cin; ++ch)
        for (int t = 0; t < taps; ++t) wt[(size_t)t * L->cin_p + ch] = S.w[(size_t)ch * taps + t];
      AM_TRY(upload(L->w_f32, wt));
      AM_TRY(upload(L->bias, padded(S.bias, L->cin_p)));
      if (L->dw_fast()) {  // the fused kernel's parameters; the expansion bias matters only when fused_block_at fuses it
        const LayerSpec& prev = spec.layers[li - 1];  // li > 0: the first layer is a stem or first convolution
        const bool relu6_in = prev.act == kActRelu6 && (prev.type == kStem || prev.type == kConvFirst || prev.type == kPointwise);
        L->dw_fp16 = dw3x3_fp16_safe(wt, padded(S.bias, L->cin_p), L->cin_p, relu6_in);
        const LayerSpec* E = prev.type == kPointwise ? &prev : nullptr;
        const std::vector<float> b1 = E ? padded(E->bias, L->cin_p) : std::vector<float>();
        AM_TRY(upload(L->fused_params, fused::pack_params(wt, padded(S.bias, L->cin_p), E ? &b1 : nullptr, L->cin_p)));
      }
    } else if (S.type == kSqueezeExcite) {
      if (S.w.size() != (size_t)S.cmid * S.cin || S.bias.size() != (size_t)S.cmid || S.aux0.size() != (size_t)S.cin * S.cmid ||
          S.aux1.size() != (size_t)S.cin) {
        set_error("weights: malformed squeeze-excite layer %zu", li);
        return AM_ERR_IO;
      }
      AM_TRY(upload(L->w_f32, S.w));
      AM_TRY(upload(L->bias, S.bias));
      AM_TRY(upload(L->aux0, S.aux0));
      AM_TRY(upload(L->aux1, S.aux1));
    } else {
      set_error("weights: unknown layer type %d", S.type);
      return AM_ERR_IO;
    }
    c = S.cout;
    m->layers.push_back(std::move(L));
  }
  // ---- head program
  m->reg_dim = spec.reg_dim;
  for (int rdim : spec.reg_dim) {
    (void)rdim;
    m->regs.push_back(std::make_unique<DevBuf<float>>());
  }
  for (size_t q = 0; q < spec.head.size(); ++q) {
    const VecOp& S = spec.head[q];
    auto H = std::make_unique<HeadOp>();
    H->kind = S.kind;
    H->a = S.a;
    H->b = S.b;
    H->dst = S.dst;
    H->K = S.K;
    H->N = S.N;
    H->act = S.act;
    H->stride = S.stride;
    H->eps = S.eps;
    H->eps2 = S.eps2;
    auto reg_ok = [&](int r) { return r >= 0 && r < spec.n_regs; };
    if (!reg_ok(S.dst) || (S.kind != kVecPool && !reg_ok(S.a)) || ((S.kind == kVecAdd || S.kind == kVecAddLnL2) && !reg_ok(S.b))) {
      set_error("weights: head op %zu references an unknown register", q);
      return AM_ERR_IO;
    }
    if (S.kind == kVecPool) {
      if (q != 0 || S.N != c) {
        set_error("weights: the head must start by pooling the trunk's %d channels", c);
        return AM_ERR_IO;
      }
      m->head_cin = c;
      m->head_cin_p = pad16(c);
    } else if (S.kind == kVecLinear) {
      if (S.w.size() != (size_t)S.N * S.K || (!S.bias.empty() && S.bias.size() != (size_t)S.N) || spec.reg_dim[(size_t)S.a] != S.K ||
          spec.reg_dim[(size_t)S.dst] != S.N) {
        set_error("weights: malformed linear in the head (op %zu)", q);
        return AM_ERR_IO;
      }
      AM_TRY(upload_split3(H->w3, S.w, S.N, S.K));
      H->has_w = true;
      if (!S.bias.empty()) {
        AM_TRY(upload(H->bias, S.bias));
        H->has_bias = true;
      }
    } else if (S.kind == kVecAffine || S.kind == kVecLayerNorm || S.kind == kVecAddLnL2) {
      const size_t dim = (size_t)spec.reg_dim[(size_t)S.dst];
      if ((!S.w.empty() && S.w.size() != dim) || (!S.bias.empty() && S.bias.size() != dim) ||
          (S.kind != kVecAffine && (S.w.empty() || S.bias.empty()))) {
        set_error("weights: malformed row op %zu in the head", q);
        return AM_ERR_IO;
      }
      if (!S.w.empty()) {
        AM_TRY(upload(H->w, S.w));
        H->has_w = true;
      }
      if (!S.bias.empty()) {
        AM_TRY(upload(H->bias, S.bias));
        H->has_bias = true;
      }
    }
    m->head.push_back(std::move(H));
  }
  if (m->head.empty() || m->head[0]->kind != kVecPool || spec.reg_dim[(size_t)m->head.back()->dst] != m->emb) {
    set_error("weights: the head must start with the spatial pooling and end with the %d-d embedding", m->emb);
    return AM_ERR_IO;
  }
  return AM_OK;
}

// The trunk runs in two phases.  EARLY = stem + the leading layers whose input maps are large (at least
// kEarlyMinPositions positions per window): processed chunk by chunk, so host->device copies of the next chunk hide
// under it and one chunk already fills the GPU.  LATE = everything after (small tensors): processed ONCE for all
// windows of the call, so the deep, narrow layers get full-size grids.  The split falls on a block boundary (a
// residual add reads its block's input).
constexpr int64_t kEarlyMinPositions = 4096;

// Layers from `i` (a block start) form an inverted-residual block the fused kernel runs: [1x1 expand + ReLU6] ->
// 3x3 depthwise + ReLU6 -> linear 1x1, all inside [i, hi) and fitting fused::plan at input shape `s`.
static bool fused_block_at(const am_model* m, size_t i, size_t hi, Shape s, Step* st) {
  const auto& L = m->layers;
  if (!m->fused_blocks || !L[i]->block_start) return false;
  int e = -1;
  size_t k = i;
  if (L[k]->type == kPointwise && L[k]->act == kActRelu6 && L[k]->stride == 1) e = (int)k++;
  if (k + 1 >= hi || k + 1 >= L.size()) return false;
  const Layer& D = *L[k];
  const Layer& P = *L[k + 1];
  if (!D.dw_fast() || P.type != kPointwise || P.act != kActNone || P.stride != 1 || P.cin_p != D.cin_p) return false;
  if (e >= 0 && L[(size_t)e]->cout_p != D.cin_p) return false;
  fused::BlockDesc& d = st->desc;
  d = fused::BlockDesc{};
  d.H = s.H;
  d.W = s.W;
  d.cin_p = e >= 0 ? L[(size_t)e]->cin_p : D.cin_p;
  d.cmid_p = D.cin_p;
  d.cout_p = P.cout_p;
  d.stride = D.stride;
  d.has_expand = e >= 0 ? 1 : 0;
  d.residual = P.residual;
  st->first = i;
  st->last = k + 1;
  return fused::plan(d, &st->plan);
}

static int build_plan(const am_model* m, int T, ForwardPlan* p) {
  const auto& L = m->layers;
  *p = ForwardPlan{};
  const Layer& stem = *L[0];
  Shape s = layer_out(stem, stem.h_is_time ? Shape{T, m->n_mels} : Shape{m->n_mels, T});
  AM_CHECK(s.H > 0 && s.W > 0, "encoder: input of %d frames x %d mels is too small", T, m->n_mels);
  AM_CHECK(stem.type == kStem || (size_t)(stem.kh * stem.kw + 1) * stem.cout_p * sizeof(float) <= 48 * 1024,
           "encoder: first convolution with %d x %d taps x %d channels does not fit in shared memory", stem.kh, stem.kw,
           stem.cout_p);
  // first layer of the late phase
  size_t split = 1;
  for (Shape w = s; split < L.size(); ++split) {
    if (L[split]->block_start && (int64_t)w.H * w.W < kEarlyMinPositions) break;
    w = layer_out(*L[split], w);
  }
  Step st;
  st.kind = stem.type == kStem ? kStepStem : kStepConvFirst;
  st.in = st.out = s;
  st.cout_p = stem.cout_p;
  p->steps.push_back(st);
  p->late_step = 1;
  p->early_act = (size_t)s.H * s.W * stem.cout_p;
  for (size_t i = 1; i < L.size();) {
    const bool late = i >= split;
    const int prev = p->steps.back().kind;
    st = Step{};
    st.in = s;
    st.starts_block = L[i]->block_start || i == split || prev == kStepStem || prev == kStepConvFirst || prev == kStepFused;
    if (fused_block_at(m, i, late ? L.size() : split, s, &st)) {
      st.kind = kStepFused;
    } else {
      const Layer& l = *L[i];
      st.first = st.last = i;
      switch (l.type) {
        case kPointwise: st.kind = kStepPointwise; break;
        case kDepthwise: st.kind = l.dw_fast() ? kStepDw3x3 : kStepDwGeneric; break;
        case kSqueezeExcite: st.kind = kStepSqueezeExcite; break;
        default: set_error("encoder: layer %zu of type %d cannot run here", i, l.type); return AM_ERR_INVALID;
      }
      AM_CHECK(l.type != kSqueezeExcite || (size_t)(l.cin + l.cmid) * sizeof(float) <= 48 * 1024,
               "encoder: squeeze-excite over %d channels does not fit in shared memory", l.cin);
    }
    size_t& act = late ? p->late_act : p->early_act;
    for (i = st.first; i <= st.last; ++i) {
      s = layer_out(*L[i], s);
      AM_CHECK(s.H > 0 && s.W > 0, "encoder: depthwise layer %zu has an empty output", i);
      act = std::max(act, (size_t)s.H * s.W * L[i]->cout_p);
    }
    st.out = s;
    st.cout_p = L[st.last]->cout_p;
    p->steps.push_back(st);
    if (!late) p->late_step = p->steps.size();
  }
  p->split = p->steps[p->late_step - 1].out;
  p->split_c = p->steps[p->late_step - 1].cout_p;
  p->T = T;
  return AM_OK;
}

// the model's plan for windows of T frames: rebuilt when T changes (a session runs one window length)
static int plan_for(am_model* m, int T, const ForwardPlan** out) {
  if (m->plan.T != T) AM_TRY(build_plan(m, T, &m->plan));
  *out = &m->plan;
  return AM_OK;
}

// Launches steps [lo, hi) of the plan on `nb` windows.  lo == 0: starts from the log-mel (stem); else from `in`.
// The last step writes to `final_out` when given, else to a workspace buffer; *out is what it wrote.
static int run_steps(am_model* m, const ForwardPlan& p, const float* mel_dev, const __nv_bfloat16* in, size_t lo, size_t hi,
                     int nb, __nv_bfloat16* final_out, const __nv_bfloat16** out, cudaStream_t st) {
  const __nv_bfloat16* cur = in;
  const __nv_bfloat16* block_in = in;
  for (size_t q = lo; q < hi; ++q) {
    const Step& t = p.steps[q];
    const Layer& l = *m->layers[t.last];
    if (t.starts_block) block_in = cur;
    __nv_bfloat16* dst = q + 1 == hi ? final_out : nullptr;
    for (auto& b : m->act)
      if (!dst && b.p != cur && b.p != block_in) dst = b.p;
    const Shape s = t.in, o = t.out;
    switch (t.kind) {
      case kStepStem: {
        const int64_t n_tiles = (int64_t)nb * ((o.H + kStemTH - 1) / kStemTH) * ((o.W + kStemTW - 1) / kStemTW);
        const int grid = (int)std::max<int64_t>(1, std::min<int64_t>(n_tiles, (int64_t)sm_count() * 8));
        AM_LAUNCH(stem_kernel, grid, 256, (size_t)l.cout_p * 8, st, mel_dev, nb, m->n_mels, p.T, o.H, o.W, l.pad_t, l.pad_l,
                  l.aux0.p, l.aux1.p, l.w_f32.p, l.aux2.p, l.bias.p, l.cout_p, dst);
        break;
      }
      case kStepConvFirst: {
        const size_t smem = (size_t)(l.kh * l.kw + 1) * l.cout_p * sizeof(float);
        const int grid = grid_for((int64_t)nb * o.H * o.W * (l.cout_p / 8));
        AM_LAUNCH(conv_first_kernel, grid, 256, smem, st, mel_dev, nb, m->n_mels, p.T, o.H, o.W, l.kh, l.kw, l.stride, l.pad_t,
                  l.pad_l, l.h_is_time, l.aux0.p, l.aux1.p, l.w_f32.p, l.bias.p, l.cout_p, l.act, dst);
        break;
      }
      case kStepFused: {  // the whole block in one kernel (fused_block.cu)
        const Layer& D = *m->layers[t.last - 1];
        AM_TRY(fused::run(t.desc, t.plan, cur, t.desc.has_expand ? m->layers[t.first]->w_bf16.p : nullptr, D.fused_params.p,
                          l.w_bf16.p, l.bias.p, dst, nb, st));
        break;
      }
      case kStepDwGeneric:
        AM_LAUNCH(depthwise_generic_kernel, grid_for((int64_t)nb * o.H * o.W * (l.cout_p / 8)), 256, 0, st, cur, nb, s.H, s.W,
                  l.cin_p, o.H, o.W, l.kh, l.stride, l.pad_t, l.pad_l, l.w_f32.p, l.bias.p, l.act, dst);
        break;
      case kStepDw3x3:
        AM_TRY(dw3x3(cur, nb, s.H, s.W, l.cin_p, l.stride, l.w_f32.p, l.bias.p, l.dw_fp16, dst, st, nullptr));
        break;
      case kStepSqueezeExcite: {
        const int HW = s.H * s.W;
        AM_TRY(m->se_mean.ensure((size_t)nb * l.cin));
        AM_TRY(m->se_gate.ensure((size_t)nb * l.cin));
        AM_LAUNCH(channel_mean_kernel, dim3((unsigned)ceil_div(l.cin, 64), (unsigned)nb), 256, 0, st, cur, HW, l.cin_p, l.cin,
                  m->se_mean.p);
        const size_t smem = (size_t)(l.cin + l.cmid) * sizeof(float);
        AM_LAUNCH(se_gate_kernel, nb, 256, smem, st, m->se_mean.p, l.cin, l.cmid, l.w_f32.p, l.bias.p, l.aux0.p, l.aux1.p, l.act,
                  l.gate_act, m->se_gate.p);
        AM_LAUNCH(se_scale_kernel, grid_for((int64_t)nb * HW * (l.cin_p / 8)), 256, 0, st, cur, (int64_t)HW, l.cin_p, l.cin,
                  m->se_gate.p, nb, dst);
        break;
      }
      case kStepPointwise: {
        gemm::Epilogue ep;
        ep.bias = l.bias.p;
        ep.act = l.act;
        if (l.residual) {
          ep.residual = block_in;
          ep.ld_res = l.cout_p;
        }
        AM_TRY(gemm::gemm_bf16(cur, (int64_t)nb * s.H * s.W, l.cin_p, l.w_bf16.p, l.cout_p, l.cin_p, l.cin_p, dst, l.cout_p, false,
                               ep, /*m_fastest=*/false, st));
        break;
      }
    }
    cur = dst;
  }
  *out = cur;
  return AM_OK;
}

// EARLY phase of `nb` windows (log-mel at mel_dev): result appended to m->late_in at window offset b0
static int forward_early(am_model* m, const ForwardPlan& p, const float* mel_dev, int nb, int b0, cudaStream_t st) {
  const size_t per_win = (size_t)p.split.H * p.split.W * p.split_c;
  const __nv_bfloat16* o;
  return run_steps(m, p, mel_dev, nullptr, 0, p.late_step, nb, m->late_in.p + (size_t)b0 * per_win, &o, st);
}

// LATE phase for all `n` windows + the head program's pooling (for a 1x1 stride-s conv in front of the mean, the
// mean over the positions the conv visits commutes with it: the conv runs on the pooled rows)
static int forward_late(am_model* m, const ForwardPlan& p, int n, cudaStream_t st) {
  const size_t per_win = (size_t)p.split.H * p.split.W * p.split_c;
  const Shape so = p.steps.back().out;
  const HeadOp& pool = *m->head[0];
  for (int b0 = 0; b0 < n; b0 += m->late_sub) {
    const int nb = std::min(m->late_sub, n - b0);
    const __nv_bfloat16* o = m->late_in.p + (size_t)b0 * per_win;
    AM_TRY(run_steps(m, p, nullptr, o, p.late_step, p.steps.size(), nb, nullptr, &o, st));
    AM_LAUNCH(strided_mean_kernel, nb, 256, 0, st, o, so.H, so.W, m->head_cin_p, m->head_cin, pool.stride,
              m->regs[(size_t)pool.dst]->p + (size_t)b0 * m->head_cin);
  }
  return AM_OK;
}

// head row program for `n` windows at once, ops [lo, hi) (default: all after the pooling); the last op writes out_dev
static int head_forward(am_model* m, int n, float* out_dev, cudaStream_t st, size_t lo = 1, size_t hi = SIZE_MAX) {
  if (n <= 0) return AM_OK;
  const int64_t rows = n;
  for (size_t q = lo; q < std::min(hi, m->head.size()); ++q) {
    const HeadOp& h = *m->head[q];
    const bool last = q + 1 == m->head.size();
    float* dst = last ? out_dev : m->regs[(size_t)h.dst]->p;
    const float* a = h.a >= 0 ? m->regs[(size_t)h.a]->p : nullptr;
    const float* b = h.b >= 0 ? m->regs[(size_t)h.b]->p : nullptr;
    const int dim = m->reg_dim[(size_t)h.dst];
    const int egrid = grid_for(rows * dim);
    switch (h.kind) {
      case kVecLinear: {
        const int Kp = (int)round_up((size_t)h.K, 8);
        const int grid = (int)std::min<int64_t>(((int64_t)n * Kp + 255) / 256, (int64_t)sm_count() * 8);
        AM_LAUNCH(split3_kernel, grid, 256, 0, st, a, n, h.K, Kp, h.act, m->a3.p);
        gemm::Epilogue ep;
        ep.bias = h.has_bias ? h.bias.p : nullptr;
        AM_TRY(gemm::gemm_bf16(m->a3.p, n, 3 * Kp, h.w3.p, h.N, 3 * Kp, 3 * Kp, dst, h.N, /*d_is_f32=*/true, ep, false, st));
        break;
      }
      case kVecUnary:
        AM_LAUNCH(vec_unary_kernel, egrid, 256, 0, st, a, rows * dim, h.act, dst);
        break;
      case kVecAdd:
        AM_LAUNCH(vec_add_kernel, egrid, 256, 0, st, a, b, rows * dim, dst);
        break;
      case kVecAffine:
        AM_LAUNCH(vec_affine_kernel, egrid, 256, 0, st, a, rows * dim, dim, h.has_w ? h.w.p : nullptr,
                  h.has_bias ? h.bias.p : nullptr, dst);
        break;
      case kVecLayerNorm:
        AM_LAUNCH(vec_layernorm_kernel, n, 256, 0, st, a, dim, h.w.p, h.bias.p, h.eps, dst);
        break;
      case kVecL2Norm:
        AM_LAUNCH(vec_l2norm_kernel, n, 256, 0, st, a, dim, h.eps2, dst);
        break;
      case kVecAddLnL2:
        AM_LAUNCH(head_finalize_kernel, n, 256, 0, st, a, b, dim, h.w.p, h.bias.p, h.eps, h.eps2, dst);
        break;
      default:
        set_error("encoder: head op %zu of kind %d cannot run here", q, h.kind);
        return AM_ERR_INVALID;
    }
  }
  return AM_OK;
}

// Windows per pass: the early phase takes at most kMaxSub (256 measured 1 % faster than 128), and few enough that one
// activation buffer stays within kEarlyActBudget elements (the buffers hold every layer output, ~50 MB per 10 s window
// for the shipped student, so 256 windows would need three 14 GB buffers); the late phase takes at most kLateSub.
constexpr int kMaxSub = 256, kLateSub = 256;
constexpr size_t kEarlyActBudget = (size_t)1 << 30;  // bf16 elements = 2 GiB per buffer

static int early_sub(const ForwardPlan& p, int n) {
  const int cap = (int)std::max<size_t>(1, kEarlyActBudget / std::max<size_t>(1, p.early_act));
  return std::min({std::max(n, 1), kMaxSub, cap});
}

static int ensure_workspace(am_model* m, const ForwardPlan& p, int nb, int n_total) {
  const size_t nt = (size_t)std::max(n_total, 1);
  m->late_sub = (int)std::min<size_t>(nt, (size_t)kLateSub);
  const size_t need = std::max(p.early_act * (size_t)nb, p.late_act * (size_t)m->late_sub);
  if (need > m->act_elems) {
    for (auto& b : m->act) b.release();
    for (auto& b : m->act) AM_TRY(b.alloc(std::max<size_t>(need, 16)));
    m->act_elems = need;
  }
  AM_TRY(m->late_in.ensure(nt * (size_t)p.split.H * p.split.W * p.split_c));
  size_t kmax = 8;
  for (size_t r = 0; r < m->regs.size(); ++r) {
    AM_TRY(m->regs[r]->ensure(nt * (size_t)m->reg_dim[r]));
    kmax = std::max(kmax, round_up((size_t)m->reg_dim[r], 8));
  }
  AM_TRY(m->a3.ensure(nt * 3 * kmax));
  return AM_OK;
}

// ---------------------------------------------------------------- debug trace (csrc/debug/encoder_debug.cu)
// Hidden like every symbol without AM_API: libaudiomuse_b200.so does not export these, the debug library calls them.

// the plan for windows of T frames as flat records (include/audiomuse_b200_debug.h, am_debug_encoder_plan)
int debug_encoder_plan(am_model* m, int T, std::vector<int>* steps, std::vector<int>* layers, std::vector<int>* head,
                       std::vector<float>* head_eps, int* late_step) {
  const ForwardPlan* p;
  AM_TRY(plan_for(m, T, &p));
  for (const Step& t : p->steps)
    steps->insert(steps->end(), {t.kind, (int)t.first, (int)t.last, t.in.H, t.in.W, t.out.H, t.out.W, t.cout_p,
                                 t.starts_block ? 1 : 0});
  for (const auto& l : m->layers)
    layers->insert(layers->end(), {l->type, l->cin, l->cout, l->kh, l->kw, l->stride, l->pad_t, l->pad_b, l->pad_l,
                                   l->pad_r, l->act, l->gate_act, l->cmid, l->h_is_time, l->residual, l->block_start,
                                   l->cin_p, l->cout_p});
  for (const auto& h : m->head) {
    head->insert(head->end(), {h->kind, h->a, h->b, h->dst, h->K, h->N, h->act, h->stride});
    head_eps->insert(head_eps->end(), {h->eps, h->eps2});
  }
  *late_step = (int)p->late_step;
  return AM_OK;
}

// One forward pass of B windows (mel_dev) through run_steps / forward_late / head_forward, as am_clap_embed_dev runs
// it, with every intermediate handed to the callbacks (after a stream synchronise):
//   on_step(q, out, elems): step q's output for all B windows, bf16 NHWC.  The steps run unchanged: each one is
//     observed by re-running the prefix of its phase ([0, q], or [late_step, q] on the early phase's late_in) with
//     step q writing to a separate buffer, in the phase's own window chunks.
//   on_head(q, out, elems): head op q's result f32 [B, dim] (op 0: the pooling); the ops run one head_forward each.
// The last op writes the embedding to out_dev.
int debug_encoder_trace(am_model* m, const float* mel_dev, int B, int T, float* out_dev,
                        const std::function<int(size_t, const __nv_bfloat16*, size_t)>& on_step,
                        const std::function<int(size_t, const float*, size_t)>& on_head) {
  cudaStream_t st = m->stream.s;
  const ForwardPlan* p;
  AM_TRY(plan_for(m, T, &p));
  const int sub = early_sub(*p, B);
  AM_TRY(ensure_workspace(m, *p, sub, B));
  size_t most = 0;
  for (const Step& t : p->steps) most = std::max(most, (size_t)t.out.H * t.out.W * t.cout_p);
  DevBuf<__nv_bfloat16> obs;
  AM_TRY(obs.alloc(most * B));
  const __nv_bfloat16* o;
  auto observe = [&](size_t q) -> int {
    AM_CUDA(cudaStreamSynchronize(st));
    const Step& t = p->steps[q];
    return on_step(q, obs.p, (size_t)B * t.out.H * t.out.W * t.cout_p);
  };
  for (size_t q = 0; q < p->late_step; ++q) {
    const size_t per = (size_t)p->steps[q].out.H * p->steps[q].out.W * p->steps[q].cout_p;
    for (int b0 = 0; b0 < B; b0 += sub)
      AM_TRY(run_steps(m, *p, mel_dev + (size_t)b0 * m->n_mels * T, nullptr, 0, q + 1, std::min(sub, B - b0),
                       obs.p + (size_t)b0 * per, &o, st));
    AM_TRY(observe(q));
  }
  for (int b0 = 0; b0 < B; b0 += sub)
    AM_TRY(forward_early(m, *p, mel_dev + (size_t)b0 * m->n_mels * T, std::min(sub, B - b0), b0, st));
  const size_t per_win = (size_t)p->split.H * p->split.W * p->split_c;
  for (size_t q = p->late_step; q < p->steps.size(); ++q) {
    const size_t per = (size_t)p->steps[q].out.H * p->steps[q].out.W * p->steps[q].cout_p;
    for (int b0 = 0; b0 < B; b0 += m->late_sub)
      AM_TRY(run_steps(m, *p, nullptr, m->late_in.p + (size_t)b0 * per_win, p->late_step, q + 1,
                       std::min(m->late_sub, B - b0), obs.p + (size_t)b0 * per, &o, st));
    AM_TRY(observe(q));
  }
  AM_TRY(forward_late(m, *p, B, st));
  AM_CUDA(cudaStreamSynchronize(st));
  AM_TRY(on_head(0, m->regs[(size_t)m->head[0]->dst]->p, (size_t)B * m->head_cin));
  for (size_t q = 1; q < m->head.size(); ++q) {
    AM_TRY(head_forward(m, B, out_dev, st, q, q + 1));
    AM_CUDA(cudaStreamSynchronize(st));
    const HeadOp& h = *m->head[q];
    const float* r = q + 1 == m->head.size() ? out_dev : m->regs[(size_t)h.dst]->p;
    AM_TRY(on_head(q, r, (size_t)B * m->reg_dim[(size_t)h.dst]));
  }
  return AM_OK;
}

}  // namespace am

using namespace am;

static int finish_load(am_model* m, const am::ModelSpec& spec, am_model** out) {
  int s = build_model(m, spec);
  if (s == AM_OK) s = m->stream.create();
  if (s != AM_OK) {
    delete m;
    return s;
  }
  if (const char* fb = std::getenv("AM_FUSED_BLOCKS")) m->fused_blocks = std::atoi(fb) != 0;
  if (!gemm::available()) {
    set_error("am_clap_load: the wgmma GEMM path is unavailable on this device; no fallback is shipped");
    delete m;
    return AM_ERR_NO_DEVICE;
  }
  *out = m;
  return AM_OK;
}

// `path` (may be NULL) locates external tensor data of an ONNX model (model.onnx.data next to the model file)
static int load_any(const void* blob, size_t nbytes, const char* path, am::ModelSpec* spec) {
  if (looks_like_onnx(blob, nbytes)) return load_onnx_spec(blob, nbytes, path, spec);
  return load_amw1_spec(blob, nbytes, spec);
}

extern "C" int am_clap_load_mem(const void* blob, size_t nbytes, am_model** out) {
  AM_CHECK(out != nullptr, "am_clap_load_mem: out is NULL");
  *out = nullptr;
  AM_CHECK(blob != nullptr && nbytes >= 20, "am_clap_load_mem: empty blob");
  ModelSpec spec;
  AM_TRY(load_any(blob, nbytes, nullptr, &spec));
  AM_TRY(ensure_init());
  return finish_load(new am_model(), spec, out);
}

static int read_file(const char* path, std::vector<uint8_t>* buf) {
  FILE* f = std::fopen(path, "rb");
  if (!f) {
    set_error("am_clap_load: cannot open %s", path);
    return AM_ERR_IO;
  }
  std::fseek(f, 0, SEEK_END);
  const long n = std::ftell(f);
  std::fseek(f, 0, SEEK_SET);
  buf->resize((size_t)std::max<long>(n, 0));
  const size_t got = n > 0 ? std::fread(buf->data(), 1, (size_t)n, f) : 0;
  std::fclose(f);
  if (n <= 0 || got != (size_t)n) {
    set_error("am_clap_load: short read on %s", path);
    return AM_ERR_IO;
  }
  return AM_OK;
}

extern "C" int am_clap_load(const char* path, am_model** out) {
  AM_CHECK(out != nullptr && path != nullptr, "am_clap_load: NULL argument");
  *out = nullptr;
  std::vector<uint8_t> buf;
  AM_TRY(read_file(path, &buf));
  ModelSpec spec;
  AM_TRY(load_any(buf.data(), buf.size(), path, &spec));
  AM_TRY(ensure_init());
  return finish_load(new am_model(), spec, out);
}

static const char* act_name(int a) {
  static const char* names[] = {"none", "relu6", "relu", "hardswish", "gelu", "sigmoid", "hardsigmoid", "tanh"};
  return a >= 0 && a < 8 ? names[a] : "?";
}

// one line per layer / head op of the lowered program
static std::string describe_spec(const ModelSpec& sp) {
  char line[256];
  std::string o;
  std::snprintf(line, sizeof line, "source %s; n_mels %d; embedding %d; %zu layers; %zu head ops\n", sp.source.c_str(), sp.n_mels,
                sp.emb, sp.layers.size(), sp.head.size());
  o += line;
  for (size_t i = 0; i < sp.layers.size(); ++i) {
    const LayerSpec& l = sp.layers[i];
    static const char* tn[] = {"stem", "pointwise", "depthwise", "head", "conv_first", "squeeze_excite"};
    std::snprintf(line, sizeof line, "L%-3zu %-14s %4d -> %4d  k %dx%d s %d pad %d,%d,%d,%d act %s%s%s%s", i,
                  l.type >= 0 && l.type < 6 ? tn[l.type] : "?", l.cin, l.cout, l.kh, l.kw, l.stride, l.pad_t, l.pad_b, l.pad_l,
                  l.pad_r, act_name(l.act), l.residual ? " +residual" : "", l.block_start ? " [block]" : "",
                  (l.type == kStem || l.type == kConvFirst) ? (l.h_is_time ? " H=time" : " H=mel") : "");
    o += line;
    if (l.type == kSqueezeExcite) {
      std::snprintf(line, sizeof line, " mid %d gate %s", l.cmid, act_name(l.gate_act));
      o += line;
    }
    o += "\n";
  }
  static const char* hn[] = {"pool", "linear", "unary", "add", "affine", "layernorm", "l2norm", "add_layernorm_l2"};
  for (size_t i = 0; i < sp.head.size(); ++i) {
    const VecOp& h = sp.head[i];
    std::snprintf(line, sizeof line, "H%-3zu %-16s r%d%s -> r%d  K %d N %d act %s stride %d bias %d\n", i,
                  h.kind >= 0 && h.kind < 8 ? hn[h.kind] : "?", h.a, h.b >= 0 ? (std::string(",r") + std::to_string(h.b)).c_str() : "",
                  h.dst, h.K, h.N, act_name(h.act), h.stride, h.bias.empty() ? 0 : 1);
    o += line;
  }
  return o;
}

// host-only (no GPU): parse + lower a model file and describe the resulting program
extern "C" int am_clap_describe_file(const char* path, char* buf, int cap) {
  AM_CHECK(path != nullptr, "am_clap_describe_file: NULL path");
  std::vector<uint8_t> data;
  AM_TRY(read_file(path, &data));
  ModelSpec spec;
  AM_TRY(load_any(data.data(), data.size(), path, &spec));
  const std::string d = describe_spec(spec);
  if (buf && cap > 0) {
    const size_t n = std::min((size_t)cap - 1, d.size());
    std::memcpy(buf, d.data(), n);
    buf[n] = 0;
  }
  return (int)d.size() + 1;
}

// frees every workspace buffer (activations, staging, head registers); the next call re-allocates what it needs.
// The cleanup step of the reference's OOM retry (tasks/clap_analyzer.py:536-549 -> cleanup_cuda_memory).
extern "C" int am_clap_release_workspace(am_model* m) {
  AM_CHECK(m != nullptr, "am_clap_release_workspace: NULL model");
  AM_CHECK(m->n_submitted == m->n_collected, "am_clap_release_workspace: submitted calls are still in flight");
  AM_CUDA(cudaDeviceSynchronize());
  for (auto& b : m->act) b.release();
  m->act_elems = 0;
  m->late_in.release();
  m->a3.release();
  m->mel_ws.release();
  m->seg_emb.release();
  m->se_mean.release();
  m->se_gate.release();
  for (auto& r : m->regs) r->release();
  for (auto& b : m->pcm_stage) b.release();
  m->off_stage.release();
  m->out_stage.release();
  m->slot_used[0] = m->slot_used[1] = false;
  return AM_OK;
}

extern "C" void am_clap_free(am_model* m) {
  if (m) cudaDeviceSynchronize();
  delete m;
}
extern "C" int am_clap_embedding_dim(const am_model* m) { return m ? m->emb : 0; }
extern "C" int am_clap_n_mels(const am_model* m) { return m ? m->n_mels : 0; }

static double head_macs(const am_model* m) {
  double macs = 0.0;
  for (const auto& h : m->head)
    if (h->kind == kVecLinear) macs += (double)h->K * h->N;
  return macs;
}

// MACs of one window in the step's 1x1 convolutions and in its other layers
static void step_macs(const am_model* m, const Step& t, double* pointwise, double* other) {
  *pointwise = *other = 0.0;
  Shape s = t.in;
  for (size_t i = t.first; i <= t.last; ++i) {
    const Layer& l = *m->layers[i];
    if (l.type == kPointwise) {
      *pointwise += (double)s.H * s.W * l.cin * (double)l.cout;
      continue;
    }
    s = t.out;
    if (l.type == kStem) *other += (double)s.H * s.W * (9.0 + l.cout);
    if (l.type == kConvFirst) *other += (double)s.H * s.W * l.kh * l.kw * l.cout;
    if (l.type == kDepthwise) *other += (double)s.H * s.W * l.cin * l.kh * l.kw;
    if (l.type == kSqueezeExcite) *other += 2.0 * l.cin * l.cmid;
  }
}

extern "C" double am_clap_flops_per_segment(const am_model* m, int T) {
  ForwardPlan p;
  if (!m || m->layers.empty() || build_plan(m, T, &p) != AM_OK) return 0.0;
  double macs = head_macs(m);
  for (const Step& t : p.steps) {
    double pw, other;
    step_macs(m, t, &pw, &other);
    macs += pw + other;
  }
  return 2.0 * macs;
}

// flops (2 x MAC) of one window of T frames executed by the GEMM kernel and by the fused block kernel (pointwise +
// depthwise inside fused blocks), and the fused blocks' algorithmic HBM bytes (block input + output, bf16): sums over
// the steps run_steps launches
extern "C" int am_clap_flops_split(const am_model* m, int T, double* gemm_flops, double* fused_flops,
                                   double* fused_bytes) {
  AM_CHECK(m && gemm_flops && fused_flops && fused_bytes && !m->layers.empty(), "am_clap_flops_split: bad argument");
  ForwardPlan p;
  AM_TRY(build_plan(m, T, &p));
  double g = 0.0, f = 0.0, fb = 0.0;
  for (const Step& t : p.steps) {
    double pw, other;
    step_macs(m, t, &pw, &other);
    if (t.kind == kStepFused) {
      f += 2.0 * (pw + other);
      fb += 2.0 * ((double)t.in.H * t.in.W * t.desc.cin_p + (double)t.out.H * t.out.W * t.desc.cout_p);
    } else if (t.kind == kStepPointwise) {
      g += 2.0 * pw;
    }
  }
  *gemm_flops = g;
  *fused_flops = f;
  *fused_bytes = fb;
  return AM_OK;
}

extern "C" int am_clap_embed_dev(am_model* m, const float* mel_dev, int B, int T, float* out_dev, void* stream) {
  AM_CHECK(m && mel_dev && out_dev, "am_clap_embed_dev: NULL argument");
  AM_CHECK(B >= 0 && T > 0, "am_clap_embed_dev: bad shape B=%d T=%d", B, T);
  cudaStream_t st = (cudaStream_t)stream;
  const ForwardPlan* p;
  AM_TRY(plan_for(m, T, &p));
  const int sub = early_sub(*p, B);
  AM_TRY(ensure_workspace(m, *p, sub, B));
  for (int b0 = 0; b0 < B; b0 += sub) {
    const int nb = std::min(sub, B - b0);
    AM_TRY(forward_early(m, *p, mel_dev + (size_t)b0 * m->n_mels * T, nb, b0, st));
  }
  AM_TRY(forward_late(m, *p, B, st));
  return head_forward(m, B, out_dev, st);
}

extern "C" int am_clap_embed(am_model* m, const float* mel, int B, int T, float* out) {
  AM_CHECK(m && mel && out, "am_clap_embed: NULL argument");
  AM_CHECK(B >= 0 && T > 0, "am_clap_embed: bad shape B=%d T=%d", B, T);
  if (B == 0) return AM_OK;
  HostCall call(m->stream.s, 0, HostCall::Memory::Owned);
  float *d_mel, *d_out;
  call.up(&d_mel, mel, (size_t)B * m->n_mels * T);
  call.down(&d_out, (size_t)B * m->emb, out);
  AM_TRY(call.start());
  AM_TRY(am_clap_embed_dev(m, d_mel, B, T, d_out, m->stream.s));
  return call.finish();
}

extern "C" int am_clap_embed_tracks_dev(am_model* m, const am_mel_plan* plan, const int16_t* pcm_dev, int n_samples,
                                        const int32_t* seg_offsets_dev, int n_tracks, int n_segments, float* out_dev,
                                        void* stream) {
  AM_CHECK(m && plan && out_dev && seg_offsets_dev, "am_clap_embed_tracks_dev: NULL argument");
  AM_CHECK(n_tracks >= 0 && n_segments >= 0 && (pcm_dev || n_segments == 0), "am_clap_embed_tracks_dev: bad sizes");
  if (n_tracks == 0) return AM_OK;
  cudaStream_t st = (cudaStream_t)stream;
  const int T = mel_plan_frames(plan, n_samples);
  if (T < 0) return T;
  const ForwardPlan* p;
  AM_TRY(plan_for(m, T, &p));
  const int sub = early_sub(*p, n_segments);
  AM_TRY(ensure_workspace(m, *p, sub, n_segments));
  AM_TRY(m->mel_ws.ensure((size_t)sub * m->n_mels * T));
  AM_TRY(m->seg_emb.ensure((size_t)std::max(n_segments, 1) * m->emb));
  for (int b0 = 0; b0 < n_segments; b0 += sub) {
    const int nb = std::min(sub, n_segments - b0);
    AM_TRY(am_mel_batch_dev(plan, pcm_dev + (size_t)b0 * n_samples, 1, nb, n_samples, m->mel_ws.p, st));
    AM_TRY(forward_early(m, *p, m->mel_ws.p, nb, b0, st));
  }
  AM_TRY(forward_late(m, *p, n_segments, st));
  AM_TRY(head_forward(m, n_segments, m->seg_emb.p, st));
  AM_LAUNCH(track_pool_kernel, n_tracks, 256, 0, st, m->seg_emb.p, seg_offsets_dev, m->emb, out_dev);
  return AM_OK;
}

extern "C" int am_clap_embed_tracks_collect(am_model* m) {
  AM_CHECK(m != nullptr, "am_clap_embed_tracks_collect: NULL model");
  AM_CHECK(m->n_collected < m->n_submitted, "am_clap_embed_tracks_collect: nothing was submitted");
  am_model::Ticket& t = m->tickets[m->n_collected & 1];
  ++m->n_collected;
  t.open = false;
  if (t.count == 0) return AM_OK;
  AM_CUDA(cudaEventSynchronize(t.ready.e));
  std::memcpy(t.user_out, t.stage.p, t.count * sizeof(float));
  return AM_OK;
}

extern "C" int am_clap_embed_tracks_submit(am_model* m, const am_mel_cfg* cfg, const int16_t* pcm, int n_samples,
                                           const int32_t* seg_offsets, int n_tracks, float* out) {
  AM_CHECK(m && cfg && seg_offsets && out, "am_clap_embed_tracks: NULL argument");
  AM_CHECK(n_tracks >= 0, "am_clap_embed_tracks: negative track count");
  // the encoder is defined on CLAP's mel only: reflect padding and power_to_db
  AM_CHECK(cfg->n_mels == m->n_mels && cfg->transpose == 0 && cfg->framing == 0 && cfg->log_mode == 0,
           "am_clap_embed_tracks: mel cfg does not match the model");
  AM_CHECK(m->n_submitted - m->n_collected < 2, "am_clap_embed_tracks_submit: two calls are already in flight; collect one");
  const bool warm = m->n_submitted > m->n_collected;  // an earlier batch is still running
  am_model::Ticket& tk = m->tickets[m->n_submitted & 1];
  if (n_tracks == 0) {
    tk.user_out = out;
    tk.count = 0;
    tk.open = true;
    ++m->n_submitted;
    return AM_OK;
  }
  // Everything that can fail without touching the stream (argument checks, allocations) happens BEFORE the ticket
  // is opened: a failed submit leaves n_submitted == what it was, so the session stays usable (a single OOM in a
  // bulk scan used to leave an uncollectable ticket behind).
  const int n_segments = seg_offsets[n_tracks];
  AM_CHECK(seg_offsets[0] == 0 && n_segments >= 0 && (pcm || n_segments == 0), "am_clap_embed_tracks: bad seg_offsets");
  if (!m->host_plan || std::memcmp(&m->host_plan_cfg, cfg, sizeof(am_mel_cfg)) != 0) {
    if (m->host_plan) am_mel_plan_free(m->host_plan);
    m->host_plan = nullptr;
    AM_TRY(am_mel_plan_create(cfg, &m->host_plan));
    m->host_plan_cfg = *cfg;
  }
  am_mel_plan* plan = m->host_plan;
  cudaStream_t st = m->stream.s;
  AM_TRY(m->copy_stream.create());
  cudaStream_t cs = m->copy_stream.s;
  for (int i = 0; i < 2; ++i) {
    AM_TRY(m->ev_copied[i].create(cudaEventDisableTiming));
    AM_TRY(m->ev_done[i].create(cudaEventDisableTiming));
  }
  const int T = mel_plan_frames(plan, n_samples);
  if (T < 0) return T;
  const ForwardPlan* p;
  AM_TRY(plan_for(m, T, &p));
  const int sub = early_sub(*p, n_segments);
  // (growing a workspace buffer while a batch is in flight is safe: cudaFree waits for the device)
  AM_TRY(ensure_workspace(m, *p, sub, n_segments));
  AM_TRY(m->mel_ws.ensure((size_t)sub * m->n_mels * T));
  AM_TRY(m->seg_emb.ensure((size_t)std::max(n_segments, 1) * m->emb));
  for (auto& b : m->pcm_stage) AM_TRY(b.ensure((size_t)sub * n_samples));
  AM_TRY(m->off_stage.ensure((size_t)n_tracks + 1));
  AM_TRY(m->out_stage.ensure((size_t)n_tracks * m->emb));
  const size_t out_count = (size_t)n_tracks * m->emb;
  AM_TRY(tk.stage.ensure(out_count));
  AM_TRY(tk.ready.create(cudaEventDisableTiming));
  if (std::getenv("AM_TEST_FAIL_SUBMIT")) {  // test hook: a submit that fails after its allocations (tests/test_gpu_encoder.py)
    set_error("am_clap_embed_tracks_submit: out of memory (injected by AM_TEST_FAIL_SUBMIT)");
    return AM_ERR_OOM;
  }
  auto enqueue = [&]() -> int {
    AM_CUDA(cudaMemcpyAsync(m->off_stage.p, seg_offsets, (size_t)(n_tracks + 1) * 4, cudaMemcpyHostToDevice, st));
    // double-buffered pipeline: H2D of chunk c+1 (copy stream) overlaps mel + early trunk of chunk c.  The
    // copy runs ~3x faster than the compute it hides under, so only the FIRST chunk's copy is exposed:
    // chunks grow 16, 32, 64, then `sub`: a copy is ~2.2x faster than the compute it hides under, so each chunk may
    // be at most ~2.2x the previous one (8 / 24 / 96 measured slower: the small chunks under-fill the GPU).
    int c = 0;
    for (int b0 = 0; b0 < n_segments; ++c) {
      // a batch submitted while another is still in flight has its copies hidden under that one: two big chunks
      const int want = warm ? (sub + 1) / 2 : (c == 0 ? 16 : (c == 1 ? 32 : (c == 2 ? 64 : sub)));
      const int nb = std::min(std::min(want, sub), n_segments - b0);
      const int slot = c & 1;
      // slot free again (its last reader may belong to the previous, still running, submitted call)
      if (m->slot_used[slot]) AM_CUDA(cudaStreamWaitEvent(cs, m->ev_done[slot].e, 0));
      m->slot_used[slot] = true;
      AM_CUDA(cudaMemcpyAsync(m->pcm_stage[slot].p, pcm + (size_t)b0 * n_samples, (size_t)nb * n_samples * 2,
                              cudaMemcpyHostToDevice, cs));
      AM_CUDA(cudaEventRecord(m->ev_copied[slot].e, cs));
      AM_CUDA(cudaStreamWaitEvent(st, m->ev_copied[slot].e, 0));
      AM_TRY(am_mel_batch_dev(plan, m->pcm_stage[slot].p, 1, nb, n_samples, m->mel_ws.p, st));
      AM_CUDA(cudaEventRecord(m->ev_done[slot].e, st));  // the mel kernel was the staging slot's only reader
      AM_TRY(forward_early(m, *p, m->mel_ws.p, nb, b0, st));
      b0 += nb;
    }
    AM_TRY(forward_late(m, *p, n_segments, st));
    AM_TRY(head_forward(m, n_segments, m->seg_emb.p, st));
    AM_LAUNCH(track_pool_kernel, n_tracks, 256, 0, st, m->seg_emb.p, m->off_stage.p, m->emb, m->out_stage.p);
    AM_CUDA(cudaMemcpyAsync(tk.stage.p, m->out_stage.p, out_count * 4, cudaMemcpyDeviceToHost, st));
    AM_CUDA(cudaEventRecord(tk.ready.e, st));
    return AM_OK;
  };
  const int s = enqueue();
  if (s != AM_OK) {  // a launch / copy failed half way: let the stream drain, keep the ticket closed
    cudaStreamSynchronize(st);
    cudaStreamSynchronize(cs);
    return s;
  }
  tk.user_out = out;
  tk.count = out_count;
  tk.open = true;
  ++m->n_submitted;
  return AM_OK;
}

extern "C" int am_clap_embed_tracks(am_model* m, const am_mel_cfg* cfg, const int16_t* pcm, int n_samples,
                                    const int32_t* seg_offsets, int n_tracks, float* out) {
  AM_CHECK(m != nullptr, "am_clap_embed_tracks: NULL argument");
  AM_CHECK(m->n_submitted == m->n_collected, "am_clap_embed_tracks: submitted calls are still in flight; collect them first");
  AM_TRY(am_clap_embed_tracks_submit(m, cfg, pcm, n_samples, seg_offsets, n_tracks, out));  // transactional: no ticket on failure
  return am_clap_embed_tracks_collect(m);
}
