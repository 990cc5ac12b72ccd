// Debug trace of the encoder (NOT part of libaudiomuse_b200.so: built into libaudiomuse_b200_debug.so, declared in
// include/audiomuse_b200_debug.h; used by tests/test_gpu_encoder_steps_exact.py).  The plan and the forward pass come
// from encoder.cu's debug_encoder_plan / debug_encoder_trace, which run the encoder's own dispatch.
#include "../common.cuh"
#include "../../../include/audiomuse_b200_debug.h"

#include <functional>
#include <vector>

namespace am {
// encoder.cu
int debug_encoder_plan(am_model* m, int T, std::vector<int>* steps, std::vector<int>* layers, std::vector<int>* head,
                       std::vector<float>* head_eps, int* late_step);
int debug_encoder_trace(am_model* m, const float* mel_dev, int B, int T, float* out_dev,
                        const std::function<int(size_t, const __nv_bfloat16*, size_t)>& on_step,
                        const std::function<int(size_t, const float*, size_t)>& on_head);
}  // namespace am

extern "C" AM_API int am_debug_encoder_plan(am_model* m, int T, int* counts, int* steps, int* layers, int* head,
                                            float* head_eps) {
  using namespace am;
  AM_CHECK(m && counts && T > 0, "am_debug_encoder_plan: bad argument");
  std::vector<int> s, l, h;
  std::vector<float> e;
  int late = 0;
  AM_TRY(debug_encoder_plan(m, T, &s, &l, &h, &e, &late));
  counts[0] = (int)(s.size() / AM_TRACE_STEP_INTS);
  counts[1] = late;
  counts[2] = (int)(l.size() / AM_TRACE_LAYER_INTS);
  counts[3] = (int)(h.size() / AM_TRACE_HEAD_INTS);
  if (steps) std::copy(s.begin(), s.end(), steps);
  if (layers) std::copy(l.begin(), l.end(), layers);
  if (head) std::copy(h.begin(), h.end(), head);
  if (head_eps) std::copy(e.begin(), e.end(), head_eps);
  return AM_OK;
}

extern "C" AM_API int am_debug_encoder_trace(am_model* m, const float* mel, int B, int T, uint16_t* steps_out,
                                             float* head_out, float* emb) {
  using namespace am;
  AM_CHECK(m && mel && steps_out && head_out && emb && B > 0 && T > 0, "am_debug_encoder_trace: bad argument");
  const int n_mels = am_clap_n_mels(m), E = am_clap_embedding_dim(m);
  DevBuf<float> d_mel, d_emb;
  AM_TRY(d_mel.alloc((size_t)B * n_mels * T));
  AM_TRY(d_emb.alloc((size_t)B * E));
  AM_CUDA(cudaMemcpy(d_mel.p, mel, (size_t)B * n_mels * T * sizeof(float), cudaMemcpyHostToDevice));
  size_t step_off = 0, head_off = 0;
  auto on_step = [&](size_t, const __nv_bfloat16* out, size_t n) -> int {
    AM_CUDA(cudaMemcpy(steps_out + step_off, out, n * sizeof(uint16_t), cudaMemcpyDeviceToHost));
    step_off += n;
    return AM_OK;
  };
  auto on_head = [&](size_t, const float* out, size_t n) -> int {
    AM_CUDA(cudaMemcpy(head_out + head_off, out, n * sizeof(float), cudaMemcpyDeviceToHost));
    head_off += n;
    return AM_OK;
  };
  AM_TRY(debug_encoder_trace(m, d_mel.p, B, T, d_emb.p, on_step, on_head));
  AM_CUDA(cudaMemcpy(emb, d_emb.p, (size_t)B * E * sizeof(float), cudaMemcpyDeviceToHost));
  return AM_OK;
}
