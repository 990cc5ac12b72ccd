// Fused inverted-residual block (expand 1x1 -> depthwise 3x3 -> project 1x1 [+ residual]) on wgmma: see
// fused_block.cu.
#pragma once

#include "common.cuh"

namespace am {
namespace fused {

struct BlockDesc {
  int H, W;                       // input spatial size (per window)
  int cin_p, cmid_p, cout_p;      // channel counts, padded to 16
  int stride;                     // depthwise stride (1 or 2), pad 1
  int has_expand;                 // 0: block without expansion conv (cmid == cin)
  int residual;                   // add the block input (stride 1, cin == cout)
};

struct Plan {
  size_t smem_bytes = 0;
  int stages = 1;  // depth of the per-chunk weight ring: as many stages as fit, up to 4
  int tile_h = 8;  // output rows (time) of a tile, 8 columns wide: 8, or 16 at stride 1 where the ring stays as deep
};

// false when the block does not fit the kernel (Cout > 256, shared memory)
bool plan(const BlockDesc& d, Plan* out);

// The kernel's per-chunk parameters of a 3x3 depthwise layer of c_p channels: for every 64 channels, one contiguous
// [11][64] fp32 block of the 9 tap weights (wd [9, c_p]), the bias (bd [c_p]) and the preceding expansion's bias (b1
// [c_p]; zeros when NULL), zero past c_p, so that one bulk copy loads a chunk's parameters.
std::vector<float> pack_params(const std::vector<float>& wd, const std::vector<float>& bd, const std::vector<float>* b1,
                               int c_p);

// W1 [cmid_p, cin_p] bf16 (NULL without an expansion conv); params = pack_params(depthwise, expansion bias);
// W2 [cout_p, cmid_p] bf16, b2 [cout_p]; X [B, H, W, cin_p] -> Y [B, Ho, Wo, cout_p], NHWC bf16
int run(const BlockDesc& d, const Plan& p, const __nv_bfloat16* X, const __nv_bfloat16* W1, const float* params,
        const __nv_bfloat16* W2, const float* b2, __nv_bfloat16* Y, int B, cudaStream_t st);

}  // namespace fused
}  // namespace am
