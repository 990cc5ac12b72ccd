// Debug entry points of the wgmma GEMM (NOT part of libaudiomuse_b200.so: built into libaudiomuse_b200_debug.so,
// declared in include/audiomuse_b200_debug.h; used by tests/test_gpu_gemm.py and tools/gemm_bench.py).
#include "../common.cuh"
#include "../gemm_wgmma.cuh"
#include "../../../include/audiomuse_b200_debug.h"

#include <cmath>
#include <vector>

// ---------------------------------------------------------------- on-device self test (debug C ABI)
// Runs the wgmma kernel and the SIMT reference on seeded bf16 operands and returns the
// largest |difference| through *max_abs_diff.  flags: bit0 bias, bit1 relu6, bit2 residual,
// bit3 fp32 output, bit4 m_fastest, bit5 col_sub with alpha = 2.
extern "C" AM_API int am_selftest_gemm(int M, int N, int K, int flags, double* max_abs_diff) {
  using namespace am;
  AM_CHECK(max_abs_diff != nullptr && M > 0 && N > 0 && K > 0, "am_selftest_gemm: bad argument");
  AM_TRY(ensure_init());
  const int lda = (int)round_up(K, 8), ldd = (int)round_up(N, 8);
  std::vector<__nv_bfloat16> hA((size_t)M * lda), hB((size_t)N * lda), hR((size_t)M * ldd);
  std::vector<float> hbias(N), hsub(N);
  uint32_t s = 12345u + (uint32_t)(M * 31 + N * 17 + K);
  auto rnd = [&]() {
    s = s * 1664525u + 1013904223u;
    return ((s >> 8) & 0xffff) / 65536.0f - 0.5f;
  };
  for (auto& v : hA) v = __float2bfloat16_rn(rnd());
  for (auto& v : hB) v = __float2bfloat16_rn(rnd());
  for (auto& v : hR) v = __float2bfloat16_rn(rnd());
  for (auto& v : hbias) v = rnd();
  for (auto& v : hsub) v = rnd();
  const bool f32 = flags & 8;
  DevBuf<__nv_bfloat16> dA, dB, dR;
  DevBuf<float> dbias, dsub;
  DevBuf<char> d1, d2;
  AM_TRY(dA.alloc(hA.size()));
  AM_TRY(dB.alloc(hB.size()));
  AM_TRY(dR.alloc(hR.size()));
  AM_TRY(dbias.alloc(N));
  AM_TRY(dsub.alloc(N));
  const size_t out_bytes = (size_t)M * ldd * (f32 ? 4 : 2);
  AM_TRY(d1.alloc(out_bytes));
  AM_TRY(d2.alloc(out_bytes));
  AM_CUDA(cudaMemcpy(dA.p, hA.data(), hA.size() * 2, cudaMemcpyHostToDevice));
  AM_CUDA(cudaMemcpy(dB.p, hB.data(), hB.size() * 2, cudaMemcpyHostToDevice));
  AM_CUDA(cudaMemcpy(dR.p, hR.data(), hR.size() * 2, cudaMemcpyHostToDevice));
  AM_CUDA(cudaMemcpy(dbias.p, hbias.data(), N * 4, cudaMemcpyHostToDevice));
  AM_CUDA(cudaMemcpy(dsub.p, hsub.data(), N * 4, cudaMemcpyHostToDevice));
  AM_CUDA(cudaMemset(d1.p, 0, out_bytes));
  AM_CUDA(cudaMemset(d2.p, 0, out_bytes));
  gemm::Epilogue ep;
  if (flags & 1) ep.bias = dbias.p;
  if (flags & 2) ep.act = 1;
  if ((flags & 4) && !f32) {
    ep.residual = dR.p;
    ep.ld_res = ldd;
  }
  if (flags & 32) {
    ep.col_sub = dsub.p;
    ep.alpha = 2.0f;
  }
  AM_TRY(gemm::gemm_bf16(dA.p, M, lda, dB.p, N, lda, K, d1.p, ldd, f32, ep, (flags & 16) != 0, nullptr));
  AM_TRY(gemm::gemm_bf16_simt(dA.p, M, lda, dB.p, N, lda, K, d2.p, ldd, f32, ep, nullptr));
  AM_CUDA(cudaDeviceSynchronize());
  std::vector<char> h1(out_bytes), h2(out_bytes);
  AM_CUDA(cudaMemcpy(h1.data(), d1.p, out_bytes, cudaMemcpyDeviceToHost));
  AM_CUDA(cudaMemcpy(h2.data(), d2.p, out_bytes, cudaMemcpyDeviceToHost));
  double worst = 0.0;
  for (int m = 0; m < M; ++m)
    for (int n = 0; n < N; ++n) {
      double a, b;
      if (f32) {
        a = reinterpret_cast<float*>(h1.data())[(size_t)m * ldd + n];
        b = reinterpret_cast<float*>(h2.data())[(size_t)m * ldd + n];
      } else {
        a = __bfloat162float(reinterpret_cast<__nv_bfloat16*>(h1.data())[(size_t)m * ldd + n]);
        b = __bfloat162float(reinterpret_cast<__nv_bfloat16*>(h2.data())[(size_t)m * ldd + n]);
      }
      const double df = std::fabs(a - b);
      if (!(df <= worst)) worst = df;  // NaN propagates
    }
  *max_abs_diff = worst;
  return AM_OK;
}

extern "C" AM_API int am_bench_gemm(int M, int N, int K, int iters, double* ms_per_launch) {
  using namespace am;
  AM_CHECK(ms_per_launch != nullptr && M > 0 && N > 0 && K > 0 && iters > 0, "am_bench_gemm: bad argument");
  AM_TRY(ensure_init());
  const int lda = (int)round_up(K, 8), ldd = (int)round_up(N, 8);
  DevBuf<__nv_bfloat16> dA, dB, dD;
  AM_TRY(dA.alloc((size_t)M * lda));
  AM_TRY(dB.alloc((size_t)N * lda));
  AM_TRY(dD.alloc((size_t)M * ldd));
  AM_CUDA(cudaMemset(dA.p, 0x3c, (size_t)M * lda * 2));  // bf16 0x3c3c = 0.0115: finite, non-trivial
  AM_CUDA(cudaMemset(dB.p, 0x3c, (size_t)N * lda * 2));
  gemm::Epilogue ep;
  cudaEvent_t e0, e1;
  AM_CUDA(cudaEventCreate(&e0));
  AM_CUDA(cudaEventCreate(&e1));
  int rc = gemm::gemm_bf16(dA.p, M, lda, dB.p, N, lda, K, dD.p, ldd, false, ep, false, nullptr);
  if (rc == AM_OK) {
    cudaEventRecord(e0, nullptr);
    for (int i = 0; i < iters && rc == AM_OK; ++i)
      rc = gemm::gemm_bf16(dA.p, M, lda, dB.p, N, lda, K, dD.p, ldd, false, ep, false, nullptr);
    cudaEventRecord(e1, nullptr);
    cudaError_t ce = cudaEventSynchronize(e1);
    float ms = 0.f;
    if (ce == cudaSuccess) ce = cudaEventElapsedTime(&ms, e0, e1);
    if (ce != cudaSuccess && rc == AM_OK) {
      set_error("am_bench_gemm: %s", cudaGetErrorString(ce));
      rc = AM_ERR_CUDA;
    }
    *ms_per_launch = (double)ms / iters;
  }
  cudaEventDestroy(e0);
  cudaEventDestroy(e1);
  return rc;
}
