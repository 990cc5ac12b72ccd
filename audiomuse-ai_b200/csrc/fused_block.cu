// Fused inverted-residual block on sm_90a: [1x1 expand + ReLU6] -> 3x3 depthwise + ReLU6 -> 1x1 project [+ residual]
// in one kernel, so the expanded tensor (6x the block width) never goes to HBM.
//
// One warpgroup per 8 x 8 output tile of one window.  The input halo tile (10 x 10 pixels at stride 1, 17 x 17 at
// stride 2) is loaded once into shared memory as K-major 128-byte-swizzled bf16 tiles.  The expansion channels are
// then walked in chunks of 64:
//   expansion   wgmma m64n64k16 over the halo rows, fp32 accumulators in registers -> + bias, ReLU6 -> bf16 halo tile
//               E [halo pixels x 64] in shared memory (pixels outside the image are zero: the depthwise pads with 0);
//   depthwise   3 x 3 taps from E in fp32 (a thread = 8 channels of one output pixel) + bias, ReLU6 -> bf16, written
//               as the K-major swizzled A operand [64 pixels x 64 channels] of
//   projection  wgmma m64n64k16 into up to four 64-column register accumulator blocks (Cout <= 256), accumulated
//               over the chunks.
// Epilogue: + bias (+ the block input for a residual block) -> bf16, straight from the registers.
// Blocks without an expansion conv read E from the input directly.  Rounding follows the layer-by-layer path: the
// expansion and the depthwise output are rounded to bf16, every sum is fp32.
#include "fused_block.cuh"

#include "ptx_sm90.cuh"

namespace am {
namespace fused {

using namespace ptx;

constexpr int kTile = 8;        // output tile edge: 64 pixels = one m64 projection
constexpr int kChunk = 64;      // expansion channels per pass = one 128-byte swizzle row of projection K
constexpr int kThreads = 128;   // one warpgroup
constexpr int kMaxCout = 256;
constexpr size_t kSmemMax = 232448;

template <int S>
constexpr int halo() { return (kTile - 1) * S + 3; }
template <int S>
constexpr int halo_rows() { return (halo<S>() * halo<S>() + 63) / 64 * 64; }

// byte offset of (row, 16-byte chunk) in a K-major SWIZZLE_128B tile (rows of 64 bf16, 8-row atoms of 1024 bytes)
__device__ __forceinline__ uint32_t sw128(uint32_t row, uint32_t chunk) {
  return (row << 7) + (((chunk ^ row) & 7u) << 4);
}

struct Args {
  const __nv_bfloat16* X;   // [B, H, W, cin_p]
  const __nv_bfloat16* W1;  // [cmid_p, cin_p] (has_expand)
  const float* b1;          // [cmid_p]
  const float* wd;          // [9, cmid_p]
  const float* bd;          // [cmid_p]
  const __nv_bfloat16* W2;  // [cout_p, cmid_p]
  const float* b2;          // [cout_p]
  __nv_bfloat16* Y;         // [B, Ho, Wo, cout_p]
  int H, W, Ho, Wo, tiles_y, tiles_x;
  int cin_p, cmid_p, cout_p, residual;
};

struct Layout {  // shared-memory carve-up (byte offsets from the 1024-aligned base)
  uint32_t xs, w1s, w2s, a2, e, total;
};

__host__ __device__ inline Layout layout(int S, bool has_expand, int cin_p, int cout_p) {
  const uint32_t hr = (uint32_t)(((S == 1 ? 10 * 10 : 17 * 17) + 63) / 64 * 64);
  const uint32_t kbx = has_expand ? (uint32_t)((cin_p + 63) / 64) : 0u;
  const uint32_t n2 = (uint32_t)((cout_p + 63) / 64 * 64);
  Layout l;
  l.xs = 0;
  l.w1s = l.xs + kbx * hr * 128;
  l.w2s = l.w1s + kbx * kChunk * 128;
  l.a2 = l.w2s + n2 * 128;
  l.e = l.a2 + 64 * 128;
  l.total = l.e + hr * 128;
  return l;
}

template <int S, bool kExpand>
__global__ void __launch_bounds__(kThreads)
fused_block_kernel(const Args a) {
  extern __shared__ __align__(1024) uint8_t smem_raw[];
  uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~(uintptr_t)1023);
  constexpr int HALO = halo<S>(), HPX = HALO * HALO, HR = halo_rows<S>();
  const Layout L = layout(S, kExpand, a.cin_p, a.cout_p);
  uint8_t* xs = smem + L.xs;
  uint8_t* w1s = smem + L.w1s;
  uint8_t* w2s = smem + L.w2s;
  uint8_t* a2 = smem + L.a2;
  __nv_bfloat16* e = reinterpret_cast<__nv_bfloat16*>(smem + L.e);  // [HR][64], plain rows of 128 bytes

  const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31, quad = lane & 3;
  const int per_img = a.tiles_y * a.tiles_x;
  const int b = blockIdx.x / per_img;
  const int ty = (blockIdx.x % per_img) / a.tiles_x, tx = blockIdx.x % a.tiles_x;
  const int oy0 = ty * kTile, ox0 = tx * kTile;
  const int gy0 = oy0 * S - 1, gx0 = ox0 * S - 1;  // image position of halo pixel (0, 0)
  const __nv_bfloat16* Xb = a.X + (int64_t)b * a.H * a.W * a.cin_p;
  auto in_image = [&](int hp, int& gy, int& gx) {
    gy = gy0 + hp / HALO;
    gx = gx0 + hp % HALO;
    return hp < HPX && gy >= 0 && gy < a.H && gx >= 0 && gx < a.W;
  };
  const uint4 zero4 = make_uint4(0u, 0u, 0u, 0u);

  const int kbx = (a.cin_p + 63) / 64;
  if (kExpand) {  // input halo tile, once: [kbx][HR rows][64 channels]
    for (int it = tid; it < kbx * HR * 8; it += kThreads) {
      const int c = it & 7, p = (it >> 3) % HR, kb = (it >> 3) / HR;
      const int ch = kb * 64 + c * 8;
      int gy, gx;
      uint4 v = zero4;
      if (ch < a.cin_p && in_image(p, gy, gx)) v = *reinterpret_cast<const uint4*>(Xb + ((int64_t)gy * a.W + gx) * a.cin_p + ch);
      *reinterpret_cast<uint4*>(xs + kb * HR * 128 + sw128(p, c)) = v;
    }
  }

  const int n2_blocks = (a.cout_p + 63) / 64;
  float acc2[4][32];
#pragma unroll
  for (int nb = 0; nb < 4; ++nb)
#pragma unroll
    for (int i = 0; i < 32; ++i) acc2[nb][i] = 0.f;

  for (int c0 = 0; c0 < a.cmid_p; c0 += kChunk) {
    const int nch = min(kChunk, a.cmid_p - c0);
    __syncthreads();  // the previous chunk's readers of w1s / w2s / E / A2 are done
    if (kExpand) {
      for (int it = tid; it < kbx * kChunk * 8; it += kThreads) {
        const int c = it & 7, r = (it >> 3) % kChunk, kb = (it >> 3) / kChunk;
        const int ch = kb * 64 + c * 8;
        uint4 v = zero4;
        if (r < nch && ch < a.cin_p) v = *reinterpret_cast<const uint4*>(a.W1 + (int64_t)(c0 + r) * a.cin_p + ch);
        *reinterpret_cast<uint4*>(w1s + kb * kChunk * 128 + sw128(r, c)) = v;
      }
    } else {  // no expansion: E is the input's channel chunk
      for (int it = tid; it < HR * 8; it += kThreads) {
        const int c = it & 7, p = it >> 3;
        int gy, gx;
        uint4 v = zero4;
        if (c * 8 < nch && in_image(p, gy, gx))
          v = *reinterpret_cast<const uint4*>(Xb + ((int64_t)gy * a.W + gx) * a.cin_p + c0 + c * 8);
        *reinterpret_cast<uint4*>(e + p * 64 + c * 8) = v;
      }
    }
    for (int it = tid; it < n2_blocks * 64 * 8; it += kThreads) {
      const int c = it & 7, r = it >> 3;
      uint4 v = zero4;
      if (r < a.cout_p && c * 8 < nch) v = *reinterpret_cast<const uint4*>(a.W2 + (int64_t)r * a.cmid_p + c0 + c * 8);
      *reinterpret_cast<uint4*>(w2s + sw128(r, c)) = v;
    }
    fence_proxy_async();  // generic-proxy writes -> visible to the wgmma (async proxy) reads
    __syncthreads();

    if (kExpand) {
      for (int m = 0; m < HR / 64; ++m) {
        float acc1[32];
#pragma unroll
        for (int i = 0; i < 32; ++i) acc1[i] = 0.f;
        wgmma_fence();
        for (int kb = 0; kb < kbx; ++kb) {
          const uint64_t da = make_smem_desc(smem_u32(xs + kb * HR * 128 + m * 64 * 128));
          const uint64_t db = make_smem_desc(smem_u32(w1s + kb * kChunk * 128));
          const int ksteps = min(4, (a.cin_p - kb * 64) / 16);
          for (int ks = 0; ks < ksteps; ++ks)
            Wgmma<64>::mma(acc1, da + (uint64_t)(ks * 2), db + (uint64_t)(ks * 2), (kb | ks) ? 1u : 0u);
        }
        wgmma_commit();
        wgmma_wait_all();
        reg_fence(acc1);
#pragma unroll
        for (int h = 0; h < 2; ++h) {
          const int p = m * 64 + warp * 16 + (lane >> 2) + 8 * h;
          int gy, gx;
          const bool inside = in_image(p, gy, gx);
#pragma unroll
          for (int j = 0; j < 8; ++j) {
            const int col = 8 * j + 2 * quad;
            float f0 = 0.f, f1 = 0.f;
            if (inside && col < nch) {
              f0 = relu6f(acc1[4 * j + 2 * h] + __ldg(&a.b1[c0 + col]));
              f1 = relu6f(acc1[4 * j + 2 * h + 1] + __ldg(&a.b1[c0 + col + 1]));
            }
            *reinterpret_cast<__nv_bfloat162*>(e + p * 64 + col) = __floats2bfloat162_rn(f0, f1);
          }
        }
      }
      __syncthreads();
    } else {
      __syncthreads();
    }

    // depthwise: item = 8 channels of one output pixel
    for (int it = tid; it < 64 * 8; it += kThreads) {
      const int g = it & 7, px = it >> 3;
      const int oy = px >> 3, ox = px & 7;
      uint4 out = zero4;
      if (g * 8 < nch) {
        const int cg = c0 + g * 8;
        float acc[8];
#pragma unroll
        for (int q = 0; q < 8; ++q) acc[q] = __ldg(&a.bd[cg + q]);
#pragma unroll
        for (int dy = 0; dy < 3; ++dy)
#pragma unroll
          for (int dx = 0; dx < 3; ++dx) {
            const int hp = (oy * S + dy) * HALO + ox * S + dx;
            const uint4 v = *reinterpret_cast<const uint4*>(e + hp * 64 + g * 8);
            const __nv_bfloat162* v2 = reinterpret_cast<const __nv_bfloat162*>(&v);
            const float* w = a.wd + (dy * 3 + dx) * a.cmid_p + cg;
#pragma unroll
            for (int q = 0; q < 4; ++q) {
              const float2 f = __bfloat1622float2(v2[q]);
              acc[2 * q] = fmaf(f.x, __ldg(&w[2 * q]), acc[2 * q]);
              acc[2 * q + 1] = fmaf(f.y, __ldg(&w[2 * q + 1]), acc[2 * q + 1]);
            }
          }
        __nv_bfloat162 o2[4];
#pragma unroll
        for (int q = 0; q < 4; ++q) o2[q] = __floats2bfloat162_rn(relu6f(acc[2 * q]), relu6f(acc[2 * q + 1]));
        out = *reinterpret_cast<const uint4*>(o2);
      }
      *reinterpret_cast<uint4*>(a2 + sw128(px, g)) = out;
    }
    fence_proxy_async();
    __syncthreads();

    // projection: acc2 += A2 [64 x nch] . W2_chunk [Cout x nch]^T
    wgmma_fence();
    const uint64_t da = make_smem_desc(smem_u32(a2));
#pragma unroll
    for (int nb = 0; nb < 4; ++nb) {
      if (nb < n2_blocks) {
        const uint64_t db = make_smem_desc(smem_u32(w2s + nb * 64 * 128));
        for (int ks = 0; ks < nch / 16; ++ks)
          Wgmma<64>::mma(acc2[nb], da + (uint64_t)(ks * 2), db + (uint64_t)(ks * 2), (c0 | ks) ? 1u : 0u);
      }
    }
    wgmma_commit();
    wgmma_wait_all();
#pragma unroll
    for (int nb = 0; nb < 4; ++nb) reg_fence(acc2[nb]);
  }

  // epilogue: + bias (+ block input) -> bf16
#pragma unroll
  for (int h = 0; h < 2; ++h) {
    const int px = warp * 16 + (lane >> 2) + 8 * h;
    const int oy = oy0 + (px >> 3), ox = ox0 + (px & 7);
    if (oy >= a.Ho || ox >= a.Wo) continue;
    const int64_t pix = ((int64_t)b * a.Ho + oy) * a.Wo + ox;
#pragma unroll
    for (int nb = 0; nb < 4; ++nb) {
      if (nb >= n2_blocks) continue;
#pragma unroll
      for (int j = 0; j < 8; ++j) {
        const int n = nb * 64 + 8 * j + 2 * quad;
        if (n >= a.cout_p) continue;
        float f0 = acc2[nb][4 * j + 2 * h] + __ldg(&a.b2[n]);
        float f1 = acc2[nb][4 * j + 2 * h + 1] + __ldg(&a.b2[n + 1]);
        if (a.residual) {  // stride 1, cin_p == cout_p: the block input at the same pixel
          const float2 r = __bfloat1622float2(*reinterpret_cast<const __nv_bfloat162*>(a.X + pix * a.cin_p + n));
          f0 += r.x;
          f1 += r.y;
        }
        *reinterpret_cast<__nv_bfloat162*>(a.Y + pix * a.cout_p + n) = __floats2bfloat162_rn(f0, f1);
      }
    }
  }
}

bool plan(const BlockDesc& d, Plan* out) {
  if (d.stride != 1 && d.stride != 2) return false;
  if (d.cout_p > kMaxCout || d.cout_p % 16 || d.cmid_p % 16 || d.cin_p % 16) return false;
  if (!d.has_expand && d.cin_p != d.cmid_p) return false;
  if (d.residual && (d.stride != 1 || d.cin_p != d.cout_p)) return false;
  const Layout l = layout(d.stride, d.has_expand != 0, d.cin_p, d.cout_p);
  out->smem_bytes = (size_t)l.total + 1024;
  return out->smem_bytes <= kSmemMax;
}

template <int S, bool kExpand>
static int launch(const Args& a, int B, size_t smem, cudaStream_t st) {
  AM_TRY((allow_dynamic_smem<fused_block_kernel<S, kExpand>>(kSmemMax)));
  const int64_t grid = (int64_t)B * a.tiles_y * a.tiles_x;
  AM_CHECK(grid < ((int64_t)1 << 31), "fused block: %lld tiles is too many for one launch", (long long)grid);
  AM_LAUNCH((fused_block_kernel<S, kExpand>), (unsigned)grid, kThreads, smem, st, a);
  return AM_OK;
}

int run(const BlockDesc& d, const Plan& p, const __nv_bfloat16* X, const __nv_bfloat16* W1, const float* b1,
        const float* wd, const float* bd, const __nv_bfloat16* W2, const float* b2, __nv_bfloat16* Y, int B,
        cudaStream_t st) {
  AM_CHECK(X && wd && bd && W2 && b2 && Y && (!d.has_expand || (W1 && b1)), "fused block: NULL operand");
  Args a{};
  a.X = X;
  a.W1 = W1;
  a.b1 = b1;
  a.wd = wd;
  a.bd = bd;
  a.W2 = W2;
  a.b2 = b2;
  a.Y = Y;
  a.H = d.H;
  a.W = d.W;
  a.Ho = (d.H - 1) / d.stride + 1;  // 3 x 3, pad 1
  a.Wo = (d.W - 1) / d.stride + 1;
  a.tiles_y = (a.Ho + kTile - 1) / kTile;
  a.tiles_x = (a.Wo + kTile - 1) / kTile;
  a.cin_p = d.cin_p;
  a.cmid_p = d.cmid_p;
  a.cout_p = d.cout_p;
  a.residual = d.residual;
  if (d.stride == 1) return d.has_expand ? launch<1, true>(a, B, p.smem_bytes, st) : launch<1, false>(a, B, p.smem_bytes, st);
  return d.has_expand ? launch<2, true>(a, B, p.smem_bytes, st) : launch<2, false>(a, B, p.smem_bytes, st);
}

}  // namespace fused
}  // namespace am
