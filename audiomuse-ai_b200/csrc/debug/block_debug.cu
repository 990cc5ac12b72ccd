// Debug entry point of the inverted-residual block (NOT part of libaudiomuse_b200.so: built into
// libaudiomuse_b200_debug.so, declared in include/audiomuse_b200_debug.h; used by tests/test_gpu_block_exact.py).
// Runs one block on host operands either fused (fused_block.cu) or layer by layer, through the same calls the
// encoder's run_steps makes for it.
#include "../common.cuh"
#include "../depthwise.cuh"
#include "../fused_block.cuh"
#include "../gemm_wgmma.cuh"
#include "../model_spec.cuh"
#include "../../../include/audiomuse_b200_debug.h"

#include <vector>

namespace {

template <typename T>
int upload(am::DevBuf<T>& d, const void* h, size_t n) {
  AM_TRY(d.alloc(n));
  AM_CUDA(cudaMemcpy(d.p, h, n * sizeof(T), cudaMemcpyHostToDevice));
  return AM_OK;
}

template <typename T>
int download(void* h, const am::DevBuf<T>& d, size_t n) {
  AM_CUDA(cudaMemcpy(h, d.p, n * sizeof(T), cudaMemcpyDeviceToHost));
  return AM_OK;
}

}  // namespace

extern "C" AM_API int am_debug_block(int path, int B, int H, int W, int cin_p, int cmid_p, int cout_p, int stride,
                                     int has_expand, int residual, const uint16_t* X, const uint16_t* W1,
                                     const float* b1, const float* wd, const float* bd, const uint16_t* W2,
                                     const float* b2, uint16_t* Y, uint16_t* E_out, uint16_t* D_out, int* info) {
  using namespace am;
  AM_CHECK(path >= 0 && path <= 2, "am_debug_block: path %d", path);
  AM_CHECK(B > 0 && H > 0 && W > 0 && (stride == 1 || stride == 2), "am_debug_block: bad shape");
  AM_CHECK(cin_p > 0 && cmid_p > 0 && cout_p > 0 && cin_p % 16 == 0 && cmid_p % 16 == 0 && cout_p % 16 == 0,
           "am_debug_block: channel counts must be positive multiples of 16");
  AM_CHECK(has_expand || cin_p == cmid_p, "am_debug_block: a block without expansion has cin_p == cmid_p");
  AM_CHECK(!residual || (stride == 1 && cin_p == cout_p), "am_debug_block: a residual needs stride 1, cin_p == cout_p");
  AM_CHECK(info, "am_debug_block: NULL info");

  fused::Plan pl;
  fused::BlockDesc d{};
  if (path != 1) {  // the plan first: a rejected shape launches nothing
    d.H = H;
    d.W = W;
    d.cin_p = cin_p;
    d.cmid_p = cmid_p;
    d.cout_p = cout_p;
    d.stride = stride;
    d.has_expand = has_expand ? 1 : 0;
    d.residual = residual ? 1 : 0;
    AM_CHECK(fused::plan(d, &pl), "am_debug_block: the fused kernel does not take this block");
    if (path == 2) {
      *info = pl.tile_h;
      return AM_OK;
    }
  }

  AM_CHECK(X && wd && bd && W2 && b2 && Y && (!has_expand || (W1 && b1)), "am_debug_block: NULL operand");
  AM_TRY(ensure_init());
  const int Ho = (H - 1) / stride + 1, Wo = (W - 1) / stride + 1;
  const size_t n_x = (size_t)B * H * W * cin_p, n_e = (size_t)B * H * W * cmid_p;
  const size_t n_d = (size_t)B * Ho * Wo * cmid_p, n_y = (size_t)B * Ho * Wo * cout_p;
  const std::vector<float> h_wd(wd, wd + (size_t)9 * cmid_p), h_bd(bd, bd + cmid_p);

  DevBuf<__nv_bfloat16> dX, dW1, dW2, dE, dD, dY;
  DevBuf<float> db1, dwd, dbd, db2, dparams;
  AM_TRY(upload(dX, X, n_x));
  AM_TRY(upload(dW2, W2, (size_t)cout_p * cmid_p));
  AM_TRY(upload(db2, b2, cout_p));
  if (has_expand) {
    AM_TRY(upload(dW1, W1, (size_t)cmid_p * cin_p));
    AM_TRY(upload(db1, b1, cmid_p));
  }
  AM_TRY(dY.alloc(n_y));
  AM_CUDA(cudaMemset(dY.p, 0xff, n_y * 2));  // NaN: an output the kernel leaves unwritten cannot pass as a value

  if (path == 0) {
    const std::vector<float> h_b1 = has_expand ? std::vector<float>(b1, b1 + cmid_p) : std::vector<float>();
    const std::vector<float> packed = fused::pack_params(h_wd, h_bd, has_expand ? &h_b1 : nullptr, cmid_p);
    AM_TRY(upload(dparams, packed.data(), packed.size()));
    AM_TRY(fused::run(d, pl, dX.p, has_expand ? dW1.p : nullptr, dparams.p, dW2.p, db2.p, dY.p, B, nullptr));
    *info = pl.stages;
  } else {
    AM_TRY(upload(dwd, wd, (size_t)9 * cmid_p));
    AM_TRY(upload(dbd, bd, cmid_p));
    AM_TRY(dD.alloc(n_d));
    AM_CUDA(cudaMemset(dD.p, 0xff, n_d * 2));
    const __nv_bfloat16* dw_in = dX.p;
    if (has_expand) {  // 1x1 expansion + bias + ReLU6
      AM_TRY(dE.alloc(n_e));
      AM_CUDA(cudaMemset(dE.p, 0xff, n_e * 2));
      gemm::Epilogue ep;
      ep.bias = db1.p;
      ep.act = kActRelu6;
      AM_TRY(gemm::gemm_bf16(dX.p, (int64_t)B * H * W, cin_p, dW1.p, cmid_p, cin_p, cin_p, dE.p, cmid_p, false, ep,
                             /*m_fastest=*/false, nullptr));
      dw_in = dE.p;
    }
    // the encoder's input bound: after a ReLU6 expansion, else none
    const bool fp16 = dw3x3_fp16_safe(h_wd, h_bd, cmid_p, has_expand != 0);
    AM_TRY(dw3x3(dw_in, B, H, W, cmid_p, stride, dwd.p, dbd.p, fp16, dD.p, nullptr, info));
    gemm::Epilogue ep;
    ep.bias = db2.p;
    if (residual) {
      ep.residual = dX.p;
      ep.ld_res = cout_p;
    }
    AM_TRY(gemm::gemm_bf16(dD.p, (int64_t)B * Ho * Wo, cmid_p, dW2.p, cout_p, cmid_p, cmid_p, dY.p, cout_p, false, ep,
                           /*m_fastest=*/false, nullptr));
  }
  AM_CUDA(cudaDeviceSynchronize());
  AM_TRY(download(Y, dY, n_y));
  if (path == 1 && E_out && has_expand) AM_TRY(download(E_out, dE, n_e));
  if (path == 1 && D_out) AM_TRY(download(D_out, dD, n_d));
  return AM_OK;
}
