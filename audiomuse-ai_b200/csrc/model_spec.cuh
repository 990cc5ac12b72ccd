// Host-side description of an audio encoder, produced by a loader (AMW1 blob reader in amw1_model.cu, ONNX graph
// lowering in onnx_model.cu) and consumed by encoder.cu's build_model(): folded fp32 weights + the layer program.
//
// The trunk is a chain of NHWC layers (one live residual source at a time: the input of the latest
// `block_start` layer); the head is a small register program on f32 [n, dim] rows.
#pragma once

#include <cstdint>
#include <string>
#include <vector>

namespace am {

enum LayerType { kStem = 0, kPointwise = 1, kDepthwise = 2, kHead = 3, kConvFirst = 4, kSqueezeExcite = 5 };
enum ActKind { kActNone = 0, kActRelu6 = 1, kActRelu = 2, kActHardSwish = 3, kActGelu = 4, kActSigmoid = 5,
               kActHardSigmoid = 6, kActTanh = 7 };

struct LayerSpec {
  int type = 0;
  int cin = 0, cout = 0;
  int kh = 1, kw = 1, stride = 1;
  int pad_t = 0, pad_b = 0, pad_l = 0, pad_r = 0;
  int act = 0, residual = 0, block_start = 0;
  int h_is_time = 1;  // kStem / kConvFirst: image H axis is the mel spectrogram's time axis (else: the mel axis)
  int gate_act = kActHardSigmoid;  // kSqueezeExcite: gate non-linearity; `act` is the inner one
  int cmid = 0;                    // kSqueezeExcite: reduced width
  // kStem:        aux0 / aux1 = per-mel scale / shift, w = dw[9], aux2 = pw scale[cout], bias = pw shift[cout]
  // kConvFirst:   aux0 / aux1 = per-mel scale / shift (may be empty), w = [cout, kh*kw], bias[cout]
  // kPointwise:   w = [cout, cin], bias[cout]
  // kDepthwise:   w = [c, kh*kw], bias[c]
  // kSqueezeExcite: w = fc1 [cmid, c], bias = fc1 bias [cmid], aux0 = fc2 [c, cmid], aux1 = fc2 bias [c]
  std::vector<float> w, bias, aux0, aux1, aux2;
};

enum VecOpKind {
  kVecPool = 0,       // dst[n, C] = mean over the (h % s == 0, w % s == 0) positions of the trunk output
  kVecLinear = 1,     // dst = in_act(src) . W[N, K]^T + bias
  kVecUnary = 2,      // dst = act(src)
  kVecAdd = 3,        // dst = a + b
  kVecAffine = 4,     // dst = src * scale[dim] + shift[dim]   (either may be empty)
  kVecLayerNorm = 5,  // dst = (src - mean) / sqrt(var + eps) * g + b
  kVecL2Norm = 6,     // dst = src / max(||src||, eps)
  kVecAddLnL2 = 7     // dst = L2(LayerNorm(a + b))   (peephole fusion of the three above)
};

struct VecOp {
  int kind = 0;
  int a = -1, b = -1, dst = -1;  // register ids
  int K = 0, N = 0;              // kVecLinear: in / out width; others: N = row width
  int act = 0;                   // kVecLinear: activation applied to the INPUT; kVecUnary: the activation
  int stride = 1;                // kVecPool
  float eps = 0.f, eps2 = 0.f;   // LayerNorm eps / L2 clamp
  std::vector<float> w, bias;    // kVecLinear: W[N, K], bias[N]; kVecAffine: scale / shift; LayerNorm: g / b
};

struct ModelSpec {
  int n_mels = 0, emb = 0;
  std::vector<LayerSpec> layers;
  std::vector<VecOp> head;
  int n_regs = 0;
  std::vector<int> reg_dim;
  std::string source;  // "AMW1" or "ONNX (ir N, opset M, K nodes)"
};

// onnx_model.cu: reads a ModelProto (+ external data next to `path` when given) and lowers it.
// Returns AM_OK or an am_status with am_last_error() naming the unsupported node / pattern.
int load_onnx_spec(const void* data, size_t nbytes, const char* path, ModelSpec* out);
bool looks_like_onnx(const void* data, size_t nbytes);
// amw1_model.cu: reads an AMW1 blob (audiomuse-ai_b200/weights.py).  AM_OK, or AM_ERR_IO with am_last_error() set.
int load_amw1_spec(const void* blob, size_t nbytes, ModelSpec* spec);

}  // namespace am
