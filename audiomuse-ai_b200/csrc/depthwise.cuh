// The 3x3 / pad 1 / ReLU6 depthwise of the layer-by-layer path (depthwise.cu), shared by the encoder and the
// block debug entry (debug/block_debug.cu) so that both pick the same kernel for the same shape.
#pragma once

#include "common.cuh"

#include <vector>

namespace am {

// the kernel dw3x3 launched
enum DwKernel { kDwStrip = 0, kDwRow = 1, kDwGeneric = 2 };

// True when the packed-fp16 kernels (depthwise_kernel, depthwise_row_kernel) cannot overflow on this layer: its input
// follows a ReLU6 (0 <= x <= 6), and for every channel |bias| + 6 * sum |w|, a bound on every partial sum, stays below
// 2^15, half the fp16 range (65504), so no converted weight or bias and no partial sum reaches inf.  Otherwise the
// layer runs in fp32 (depthwise_generic_kernel).  w [9, cp], bias [cp], fp32 as uploaded.
bool dw3x3_fp16_safe(const std::vector<float>& w, const std::vector<float>& bias, int cp, bool relu6_input);

// out = bf16(relu6(dw3x3(in, pad 1, stride) + bias)): in [B, H, W, cp] -> out [B, Ho, Wo, cp] NHWC bf16, w [9, cp] and
// bias [cp] fp32 on the device.  fp16: the layer passed dw3x3_fp16_safe.  *kernel (may be NULL) = the DwKernel run.
int dw3x3(const __nv_bfloat16* in, int B, int H, int W, int cp, int stride, const float* w, const float* bias, bool fp16,
          __nv_bfloat16* out, cudaStream_t st, int* kernel);

}  // namespace am
