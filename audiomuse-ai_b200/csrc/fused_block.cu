// Fused inverted-residual block on sm_90a: [1x1 expand + ReLU6] -> 3x3 depthwise + ReLU6 -> 1x1 project [+ residual]
// in one kernel, so the expanded tensor (6x the block width) never goes to HBM.
//
// Persistent, warp-specialised CTA of three warpgroups (tma_pipeline.cuh), each CTA looping over output tiles 8 mel
// columns wide and 8 time rows high, or 16 (the tall tile) for a stride-1 block with cout_p <= 128 whose ring stays
// as deep (plan()); the height is a kernel parameter, chosen outside every K loop:
//   warpgroup 0   TMA producer (one elected lane): per tile the input halo (10 x 10 pixels at stride 1, 18 x 10 for
//                 the tall tile, 17 x 17 at stride 2) through a 4-D NHWC tensor map as K-major 128-byte-swizzled
//                 bf16 rows, zero filled outside the image and past cin_p; per 64-channel chunk of the expansion, into
//                 a ring of as many stages as fit (up to 4): the W1 and W2 chunks (2-D maps, zero filled past cmid_p /
//                 cout_p) or, without an expansion conv, the input's channel chunk itself, and the chunk's depthwise
//                 weights and biases and expansion bias in one bulk copy (packed per chunk at model load,
//                 pack_params).  The next tile's halo and first chunks load while the consumers finish the current
//                 tile.
//   warpgroups 1, 2   consumers, sharing one tile; per chunk:
//     expansion   transposed, E^T = W1 chunk . halo^T, so the halo pixels are the MMA's N: each warpgroup one
//                 contiguous run of 8-pixel atoms (wgmma m64n152k16 / m64n144k16 at stride 2, m64n56k16 / m64n48k16
//                 at stride 1, m64n96k16 / m64n88k16 for the tall tile's 184 halo rows); fp32 accumulators -> + bias,
//                 ReLU6 -> bf16, stored back pixel-major by stmatrix
//                 .trans into the halo tile E [halo pixels x 64, 16-byte groups XOR-swizzled by pixel] (pixels
//                 outside the image are zero: the depthwise pads with 0, and relu6(bias) need not be);
//     depthwise   3 x 3 taps from E in fp32 (a thread = 2 channels of one output column, walking its input rows) +
//                 bias, ReLU6 -> bf16, written as the K-major swizzled A operand [tile pixels x 64 channels] of
//     projection  wgmma into register accumulators, accumulated over the chunks in ascending order: for an 8 x 8
//                 tile m64n(Cout / 2)k16, one half of the output columns per warpgroup (Cout <= 256); for a tall
//                 tile m64n(Cout)k16, 64 of A's 128 rows per warpgroup (Cout <= 128).
//   With two or more stages the chunks overlap: chunk c + 1's expansion MMAs are issued before chunk c's depthwise and
//   run under it (they write only registers), and its epilogue refills E after chunk c's projection.  Two named
//   barriers per chunk order E and the A operand between the consumer warpgroups; both retire their projection before
//   the first, so one A buffer serves.
// Epilogue: + bias (+ the block input for a residual block) -> bf16, straight from the registers; every bias and
// residual value is loaded before the first store.
// Rounding follows the layer-by-layer path: the expansion and the depthwise output are rounded to bf16, every sum is
// fp32, in the same order for every element.
#include "fused_block.cuh"

#include <type_traits>

#include "gemm_wgmma.cuh"
#include "tma_pipeline.cuh"

namespace am {
namespace fused {

using namespace ptx;

constexpr int kTile = 8;        // output tile width (mel columns), and the height of the square tile: 64 pixels
constexpr int kTallTile = 16;   // height (time rows) of the tall tile at stride 1: 128 pixels
constexpr int kChunk = 64;      // expansion channels per pass = one 128-byte swizzle row of projection K
constexpr int kMaxCout = 256;
constexpr int kMaxStages = 4;
constexpr size_t kSmemMax = 232448;
constexpr uint32_t kConsumerBar = 1;  // named barrier of the two consumer warpgroups
// per stage after W1 / W2, and per chunk in pack_params: depthwise weights [9][64], depthwise bias [64], expansion
// bias [64], fp32
constexpr int kParamRows = 9 + 1 + 1;
constexpr uint32_t kDwBytes = kParamRows * kChunk * 4;
using Ring = pipe::Ring<kMaxStages>;

// the input halo of a tile th output rows high: halo(S) pixels wide, halo_h high, halo_px pixels
__host__ __device__ constexpr int halo(int S) { return (kTile - 1) * S + 3; }
__host__ __device__ constexpr int halo_h(int S, int th) { return (th - 1) * S + 3; }
__host__ __device__ constexpr int halo_px(int S, int th) { return halo_h(S, th) * halo(S); }
// shared-memory rows of one 64-channel block of the halo: the 8 x 8 tile's rounded to 64, the tall tile's to whole
// 8-pixel atoms (184 for 180 pixels: at 192 block 2 of the shipped student would lose a ring stage)
__host__ __device__ constexpr int halo_rows(int S, int th) {
  return th == kTile ? (halo_px(S, th) + 63) / 64 * 64 : (halo_px(S, th) + 7) / 8 * 8;
}
// the expansion's split of the halo pixels, rounded up to whole 8-pixel atoms, between the two consumer warpgroups
__host__ __device__ constexpr int en0(int px) { return ((px + 7) / 8 + 1) / 2 * 8; }
__host__ __device__ constexpr int en1(int px) { return (px + 7) / 8 * 8 - en0(px); }

constexpr uint32_t round1k(uint32_t v) { return (v + 1023u) & ~1023u; }

// element offset of channel group g (8 channels) of pixel p in E: rows of 64 bf16, the 16-byte groups XOR-swizzled
// by the pixel so that the expansion epilogue's stores (8 pixels of one group per warp) hit distinct banks
__device__ __forceinline__ int e_off(int p, int g) { return p * 64 + ((g ^ (p & 7)) << 3); }

// byte offset of (row, 16-byte chunk) in a K-major SWIZZLE_128B tile (rows of 64 bf16, 8-row atoms of 1024 bytes)
__device__ __forceinline__ uint32_t sw128(uint32_t row, uint32_t chunk) {
  return (row << 7) + (((chunk ^ row) & 7u) << 4);
}

// Shared memory: the ring of per-chunk stages, then the kernel's own region (offsets from its start).
//   stage (expand):     [W1 chunk: kbx x 64 rows x 128 B][W2 chunk: n2 rows x 128 B][depthwise params]
//   stage (no expand):  [input chunk: halo pixels x 128 B][W2 chunk][depthwise params]
//   own region:         [input halo: kbx x hr rows x 128 B][projection A: tile pixels x 128 B][E: halo pixels x 128 B]
//                       [2 barriers]
struct Layout {
  uint32_t stage, w2, dw;     // stage bytes, offsets of W2 and the depthwise params inside a stage
  uint32_t xs, a2, e, bars, extra;
  int hr;                     // halo_rows of the tile
  int th;                     // output rows of a tile: kTile, or kTallTile at stride 1
  int stages;
  size_t smem;
};

static Layout layout(int S, int th, bool has_expand, int cin_p, int cout_p, int stages) {
  const uint32_t hr = (uint32_t)halo_rows(S, th), hpx = (uint32_t)halo_px(S, th);
  const uint32_t kbx = has_expand ? (uint32_t)((cin_p + 63) / 64) : 0u;
  const uint32_t n2 = (uint32_t)((cout_p + 63) / 64 * 64);
  Layout l;
  l.w2 = has_expand ? kbx * kChunk * 128 : round1k(hpx * 128);
  l.dw = l.w2 + n2 * 128;
  l.stage = round1k(l.dw + kDwBytes);
  l.xs = 0;
  l.a2 = l.xs + kbx * hr * 128;
  l.e = l.a2 + (uint32_t)(th * kTile * 128);
  l.bars = l.e + (has_expand ? hpx * 128 : 0u);
  l.extra = l.bars + 2 * sizeof(uint64_t);
  l.hr = (int)hr;
  l.th = th;
  l.stages = stages;
  l.smem = Ring::smem_bytes(l.stage, stages, l.extra);
  return l;
}

struct Args {
  const __nv_bfloat16* X;   // [B, H, W, cin_p] (the residual)
  const float* params;      // [cmid_p / 64 rounded up][kParamRows][64] (pack_params)
  const float* b2;          // [cout_p]
  __nv_bfloat16* Y;         // [B, Ho, Wo, cout_p]
  int H, W, Ho, Wo, tiles_y, tiles_x, num_tiles;
  int cin_p, cmid_p, cout_p, residual;
  Layout l;
};

// Per-phase cycle counters of a measurement build (-DAM_FUSED_PHASES, tools/fused_block_phases.py): one thread of each
// warpgroup sums clock64 deltas per phase and adds them, per CTA, to g_phase_cycles[warpgroup]; run() prints the sums
// of every launch to stderr.  A default build compiles PhaseClock to nothing.
enum Phase { kRingWait, kHaloWait, kExpandMma, kExpandEpi, kDepthwise, kProjectMma, kBarrier, kEpilogue, kIssue, kNumPhases };
#ifdef AM_FUSED_PHASES
static const char* const kPhaseNames[kNumPhases] = {"ring_wait", "halo_wait", "expand_mma", "expand_epi", "depthwise",
                                                     "project_mma", "barrier", "epilogue", "issue"};
__device__ unsigned long long g_phase_cycles[3][kNumPhases];
__device__ __forceinline__ long long clock_now() {
  long long v;
  asm volatile("mov.u64 %0, %%clock64;" : "=l"(v));
  return v;
}
struct PhaseClock {
  uint32_t acc[kNumPhases];  // 32 bits: a CTA's cycles in one phase of one launch stay far below 2^32
  long long t;
  __device__ __forceinline__ PhaseClock() : acc{}, t(clock_now()) {}
  __device__ __forceinline__ void lap(Phase p) {
    const long long n = clock_now();
    acc[p] += (uint32_t)(n - t);
    t = n;
  }
  __device__ __forceinline__ void flush(int wg) {
    for (int p = 0; p < kNumPhases; ++p) atomicAdd(&g_phase_cycles[wg][p], (unsigned long long)acc[p]);
  }
};
#else
struct PhaseClock {
  __device__ __forceinline__ void lap(Phase) {}
  __device__ __forceinline__ void flush(int) {}
};
#endif

template <int S, bool kExpand>
__global__ void __launch_bounds__(pipe::kThreads, 1)
fused_block_kernel(const __grid_constant__ CUtensorMap map_x, const __grid_constant__ CUtensorMap map_w1,
                   const __grid_constant__ CUtensorMap map_w2, const Args a) {
  extern __shared__ __align__(1024) uint8_t smem_raw[];
  constexpr int HALO = halo(S);  // halo pixels per row, for both tile heights
  constexpr int PX8 = halo_px(S, kTile), PXT = halo_px(S, kTallTile);
  // The tile height is a kernel parameter, so the choice is uniform across the CTA; stride 2 takes 8 x 8 tiles only.
  const bool tall = S == 1 && a.l.th == kTallTile;
  const int hpx = tall ? PXT : PX8, hr = a.l.hr;
  Ring ring(smem_raw, a.l.stage, a.l.stages, a.l.extra);
  uint8_t* own = ring.extra();
  uint8_t* xs = own + a.l.xs;
  uint8_t* a2 = own + a.l.a2;
  uint64_t* xs_full = reinterpret_cast<uint64_t*>(own + a.l.bars);  // halo landed (TMA -> consumers)
  uint64_t* xs_empty = xs_full + 1;                                 // last expansion of the tile done (consumers -> TMA)

  const int per_img = a.tiles_y * a.tiles_x;
  const int kbx = (a.cin_p + 63) / 64;
  const int n2_blocks = (a.cout_p + 63) / 64;

  if (threadIdx.x == 0) {
    prefetch_tensormap(&map_x);
    if (kExpand) prefetch_tensormap(&map_w1);
    prefetch_tensormap(&map_w2);
    mbar_init(xs_full, 1);
    mbar_init(xs_empty, pipe::kConsumerThreads);
    ring.init();  // fences the barrier initialisations above too
  }
  __syncthreads();

  if (threadIdx.x < 128) {
    regs_producer();
    // ===================== TMA producer =====================
    if (threadIdx.x < 32 && elect_one_sync()) {
      PhaseClock clk;
      uint32_t xs_phase = 0;
      for (int tile = blockIdx.x; tile < a.num_tiles; tile += gridDim.x) {
        const int b = tile / per_img, ty = (tile % per_img) / a.tiles_x, tx = tile % a.tiles_x;
        const int gy0 = ty * a.l.th * S - 1, gx0 = tx * kTile * S - 1;  // image position of halo pixel (0, 0)
        if (kExpand) {
          clk.lap(kIssue);
          mbar_wait(xs_empty, xs_phase ^ 1);
          clk.lap(kHaloWait);
          mbar_expect_tx(xs_full, (uint32_t)(kbx * hpx * 128));
          for (int kb = 0; kb < kbx; ++kb) tma_load_4d(xs + kb * hr * 128, &map_x, xs_full, kb * 64, gx0, gy0, b);
          xs_phase ^= 1;
        }
        for (int c0 = 0; c0 < a.cmid_p; c0 += kChunk) {
          const uint32_t tx_bytes = (kExpand ? (uint32_t)kbx * kChunk * 128 : (uint32_t)hpx * 128) +
                                    (uint32_t)n2_blocks * 64 * 128 + kDwBytes;
          clk.lap(kIssue);
          const Ring::Slot s = ring.acquire(tx_bytes);
          clk.lap(kRingWait);
          if (kExpand) {
            for (int kb = 0; kb < kbx; ++kb) tma_load_2d(s.smem + kb * kChunk * 128, &map_w1, s.bar, kb * 64, c0);
          } else {
            tma_load_4d(s.smem, &map_x, s.bar, c0, gx0, gy0, b);
          }
          tma_load_2d(s.smem + a.l.w2, &map_w2, s.bar, c0, 0);
          bulk_load(s.smem + a.l.dw, a.params + (int64_t)c0 * kParamRows, kDwBytes, s.bar);
        }
      }
      clk.lap(kIssue);
      clk.flush(0);
    }
    return;
  }
  regs_consumer();
  // ===================== consumers: warpgroups 1 and 2 =====================
  const int ct = threadIdx.x - 128;          // 0 .. 255
  // warp-uniform by construction (a shuffle result), so branches on it keep the wgmmas on a converged path
  const int wg = __shfl_sync(0xffffffffu, ct >> 7, 0), wt = ct & 127;
  const int warp = wt >> 5, lane = wt & 31, quad = lane & 3;
  __nv_bfloat16* e_own = reinterpret_cast<__nv_bfloat16*>(own + a.l.e);  // [HPX][64], plain rows of 128 bytes
  const int nchunks = (a.cmid_p + kChunk - 1) / kChunk;
  // With two or more stages chunk c + 1's expansion reads its stage while chunk c's is still held; a one-stage ring
  // cannot hold both, so there the expansion waits for chunk c's projection and the stage it frees.
  const bool ahead = a.l.stages > 1;

  // Calls f(std::integral_constant<int, tile height>), so that the code for each tile height has its sizes as
  // compile-time constants; the choice is made once, outside every K loop.
  auto with_tile = [&](auto f) {
    if constexpr (S == 1) {
      if (tall) return f(std::integral_constant<int, kTallTile>{});
    }
    return f(std::integral_constant<int, kTile>{});
  };

  // The expansion runs transposed, E^T [64 channels x halo pixels] = W1 chunk . halo^T: the stage's W1 chunk (64
  // K-major rows) is the A operand and the halo rows are B, so the halo pixels are the MMA's wide dimension.  The
  // pixels, rounded up to whole 8-row atoms, split between the warpgroups as evenly as whole atoms allow (en0 / en1):
  // 152 + 144 at stride 2, 56 + 48 at stride 1, 96 + 88 for the tall tile.  Halo rows past the halo's pixels are stale
  // and give accumulator columns that are never stored.
  // The projection: an 8 x 8 tile gives each warpgroup all 64 rows of A and one half of the output columns,
  // [wg half, (wg + 1) half); a tall tile gives each warpgroup 64 of A's 128 rows and all cout_p (<= 128) columns.
  const int half = a.cout_p / 2;
  const int proj_n = tall ? a.cout_p : half;       // columns of this warpgroup's projection MMA
  const int proj_col = tall ? 0 : wg * half;       // its first output column
  const int proj_row = tall ? 64 * wg : 0;         // its first row of A (output pixel of the tile)

  // the first MMA of every expansion and of every tile's projection overwrites (scale_d = 0)
  constexpr int kAcc1 = en0(S == 1 ? PXT : PX8) / 2;  // the widest expansion of the kernel's tile heights
  float acc1[kAcc1];  // expansion: channels 16 warp + lane / 4 (+ 8) of pixels p0 + 8 j + 2 quad (+ 1)
  float acc2[kMaxCout / 4];  // projection: output columns proj_col + 8 j + 2 quad (+ 1), j < proj_n / 8
#pragma unroll
  for (int i = 0; i < kAcc1; ++i) acc1[i] = 0.f;
#pragma unroll
  for (int i = 0; i < kMaxCout / 4; ++i) acc2[i] = 0.f;

  // acc1 = W1 chunk . this warpgroup's halo rows^T, issued and committed, not waited for
  // (the width is chosen outside the K loop, so that each warpgroup's MMAs form one straight run ptxas can batch)
  auto expand_issue = [&](const uint8_t* stage) {
    const uint32_t w1 = smem_u32(stage);
    auto issue = [&](auto width, int p0) {
      const uint32_t px = smem_u32(xs) + (uint32_t)(p0 * 128);
      for (int kb = 0; kb < kbx; ++kb) {
        const uint64_t da = make_smem_desc(w1 + (uint32_t)(kb * kChunk * 128));
        const uint64_t db = make_smem_desc(px + (uint32_t)(kb * hr * 128));
        const int ksteps = min(4, (a.cin_p - kb * 64) / 16);
        for (int ks = 0; ks < ksteps; ++ks)
          wgmma_into<decltype(width)::value>(acc1, da + (uint64_t)(ks * 2), db + (uint64_t)(ks * 2),
                                             (kb | ks) ? 1u : 0u);
      }
    };
    wgmma_fence();
    with_tile([&](auto th) {
      constexpr int PX = halo_px(S, decltype(th)::value);
      if (wg == 0) issue(std::integral_constant<int, en0(PX)>{}, 0);
      else issue(std::integral_constant<int, en1(PX)>{}, en0(PX));
    });
    wgmma_commit();
  };
  // Bit 2 j + k of this thread's mask: halo pixel p0 + 8 j + 2 quad + k of its warpgroup lies inside the image.  It
  // depends on the tile only, so it is computed once per tile rather than in every chunk's epilogue.  The pixels'
  // halo coordinates do not depend on the tile; the empty asm keeps the compiler from hoisting all 2 x en0 / 4 of
  // them out of the tile loop, where they would not fit in the registers the chunk loop leaves.
  auto inside_mask = [&](int gy0, int gx0) {
    return with_tile([&](auto th) {
      constexpr int EN0 = en0(halo_px(S, decltype(th)::value));
      int p0 = wg * EN0 + 2 * quad;
      asm volatile("" : "+r"(p0));
      uint64_t m = 0;
#pragma unroll
      for (int j = 0; j < EN0 / 8; ++j)
#pragma unroll
        for (int k = 0; k < 2; ++k) {
          const int p = p0 + 8 * j + k;
          const int gy = gy0 + p / HALO, gx = gx0 + p % HALO;
          if (gy >= 0 && gy < a.H && gx >= 0 && gx < a.W) m |= 1ull << (2 * j + k);
        }
      return m;
    });
  };
  // E pixels of this warpgroup = relu6(acc1 + b1), zero outside the image and past the chunk's channels.  A thread's
  // bf16 pair (channel r + 8 h, pixels 8 j + 2 quad, + 1) is one register of the 8 x 8 fragment (pixel group j,
  // channel group 2 warp + h); stmatrix .trans writes the fragments back pixel-major, each pixel's 8 channels one
  // 16-byte group at e_off, so E keeps the layout the depthwise reads.  The pixel groups past the halo's last whole
  // atom (warpgroup 1's last one) store element by element, stopping at the halo's last pixel.
  auto expand_epilogue = [&](const uint8_t* stage, int nch, uint64_t inside) {
    reg_fence(acc1);
    const float* b1 = reinterpret_cast<const float*>(stage + a.l.dw) + 10 * kChunk;
    const int r = 16 * warp + (lane >> 2);
    const float bias[2] = {b1[r], b1[r + 8]};
    // a channel past the chunk's stores zeros: its bits of the mask below are cleared
    const uint32_t keep[2] = {r < nch ? ~0u : 0u, r + 8 < nch ? ~0u : 0u};
    // The zero cases clear the bf16 halves of the packed pair (pixel 2 quad in the low half, the next in the high
    // one): relu6f maps every input, NaN included, to a finite value, so masking after the conversion gives the same
    // bits as selecting 0 before it.
    auto pack = [&](int j, int h) {  // the fragment register of pixel group j, channel group 2 warp + h
      const uint32_t bits = (uint32_t)(inside >> (2 * j));
      const uint32_t mask = ((bits & 1u) * 0xffffu | (bits & 2u) * 0x7fff8000u) & keep[h];
      const __nv_bfloat162 v = __floats2bfloat162_rn(relu6f(acc1[4 * j + 2 * h] + bias[h]),
                                                     relu6f(acc1[4 * j + 2 * h + 1] + bias[h]));
      return *reinterpret_cast<const uint32_t*>(&v) & mask;
    };
    auto store = [&](auto wgc, auto th) {
      constexpr int HPX = halo_px(S, decltype(th)::value);
      constexpr int P0 = decltype(wgc)::value * en0(HPX);
      constexpr int NG = (decltype(wgc)::value ? en1(HPX) : en0(HPX)) / 8;  // pixel groups of this warpgroup
      constexpr int NFULL = (HPX - P0) / 8 < NG ? (HPX - P0) / 8 : NG;     // those entirely below HPX
      // lane 8 i + k addresses row k of matrix i: pixel group j + i / 2, channel group 2 warp + i % 2
      const int mi = lane >> 3;
      const uint32_t e_base = smem_u32(e_own);
#pragma unroll
      for (int j = 0; j + 1 < NFULL; j += 2) {
        const int p = P0 + 8 * (j + (mi >> 1)) + (lane & 7);
        stmatrix_x4_trans(e_base + 2 * e_off(p, 2 * warp + (mi & 1)), pack(j, 0), pack(j, 1), pack(j + 1, 0),
                          pack(j + 1, 1));
      }
      if (NFULL % 2) {
        const int p = P0 + 8 * (NFULL - 1) + (lane & 7);
        stmatrix_x2_trans(e_base + 2 * e_off(p, 2 * warp + (mi & 1)), pack(NFULL - 1, 0), pack(NFULL - 1, 1));
      }
#pragma unroll
      for (int j = NFULL; j < NG; ++j)
#pragma unroll
        for (int h = 0; h < 2; ++h) {
          const uint32_t v = pack(j, h);
#pragma unroll
          for (int k = 0; k < 2; ++k) {
            const int p = P0 + 8 * j + 2 * quad + k;
            if (p < HPX)
              reinterpret_cast<uint16_t*>(e_own)[e_off(p, 2 * warp + h) + (lane >> 2)] = (uint16_t)(v >> (16 * k));
          }
        }
    };
    with_tile([&](auto th) {
      if (wg == 0) store(std::integral_constant<int, 0>{}, th);
      else store(std::integral_constant<int, 1>{}, th);
    });
  };

  PhaseClock clk;
  uint32_t xs_phase = 0;
  for (int tile = blockIdx.x; tile < a.num_tiles; tile += gridDim.x) {
    const int b = tile / per_img, ty = (tile % per_img) / a.tiles_x, tx = tile % a.tiles_x;
    const int oy0 = ty * a.l.th, ox0 = tx * kTile;
    const int gy0 = oy0 * S - 1, gx0 = ox0 * S - 1;
    const uint64_t inside = kExpand ? inside_mask(gy0, gx0) : 0;
    if (kExpand) {
      mbar_wait(xs_full, xs_phase);
      xs_phase ^= 1;
      clk.lap(kHaloWait);
      const uint8_t* s0 = ring.wait_ptr();
      clk.lap(kRingWait);
      expand_issue(s0);
      wgmma_wait<0>();
      clk.lap(kExpandMma);
      expand_epilogue(s0, min(kChunk, a.cmid_p), inside);
      if (nchunks == 1) mbar_arrive(xs_empty);  // this thread's reads of the halo are complete
      clk.lap(kExpandEpi);
    }

    for (int c = 0; c < nchunks; ++c) {
      const int c0 = c * kChunk, nch = min(kChunk, a.cmid_p - c0);
      const bool next = kExpand && c + 1 < nchunks;  // chunk c + 1's expansion runs in this iteration
      uint8_t* sp = ring.wait_ptr();  // returns at once when the expansion already waited for it
      clk.lap(kRingWait);
      const float* dwp = reinterpret_cast<const float*>(sp + a.l.dw);
      const __nv_bfloat16* e = kExpand ? e_own : reinterpret_cast<const __nv_bfloat16*>(sp);
      // E is complete, and both warpgroups' previous projection has finished reading A
      named_bar_sync(kConsumerBar, pipe::kConsumerThreads);
      clk.lap(kBarrier);
      const uint8_t* sn = nullptr;  // chunk c + 1's stage
      if (next && ahead) {
        sn = ring.wait_ahead_ptr();
        clk.lap(kRingWait);
        expand_issue(sn);
        clk.lap(kExpandMma);
      }

      // depthwise: a thread = one channel pair (2 cp, 2 cp + 1) of one output column ox, a warp = all 64 channels of
      // that column, so every E load and A store of a warp is one 128-byte pixel row (conflict-free under the XOR
      // swizzles).  The thread walks the column's input rows top to bottom, converts each of the row's 3 taps once and
      // adds it into every output row that uses it; per output the order stays bias, then dy and dx ascending.  The
      // 8 x 8 tile keeps its 8 output rows and stores them at the end; the tall tile stores each of its 16 rows as
      // soon as its last tap is in, so only about 3 rows of accumulators are live.
      with_tile([&](auto th) {
        constexpr int TH = decltype(th)::value, HH = halo_h(S, TH);
        const int ox = ct >> 5, cp = lane, g = cp >> 2;
        // A row 8 oy + ox: its swizzle depends on ox only (sw128 takes the row mod 8)
        uint8_t* arow = a2 + sw128(ox, g) + 4 * (cp & 3);
        auto put = [&](int oy, uint32_t v) { *reinterpret_cast<uint32_t*>(arow + oy * kTile * 128) = v; };
        if (2 * cp < nch) {
          float2 w[9];
#pragma unroll
          for (int t = 0; t < 9; ++t) w[t] = *reinterpret_cast<const float2*>(dwp + t * kChunk + 2 * cp);
          const float2 bias = *reinterpret_cast<const float2*>(dwp + 9 * kChunk + 2 * cp);
          float2 acc[TH];
#pragma unroll
          for (int oy = 0; oy < TH; ++oy) acc[oy] = bias;
          auto out = [&](int oy) {  // bf16 pair of output row oy
            const __nv_bfloat162 o = __floats2bfloat162_rn(relu6f(acc[oy].x), relu6f(acc[oy].y));
            return *reinterpret_cast<const uint32_t*>(&o);
          };
          // halo pixel ox * S + d (d = iy * HALO + dx) is at col[d & 7] + 64 d: its swizzle depends on d only mod 8
          const __nv_bfloat16* col[8];
#pragma unroll
          for (int k = 0; k < 8; ++k) col[k] = e + ox * S * 64 + ((g ^ ((ox * S + k) & 7)) << 3) + 2 * (cp & 3);
#pragma unroll
          for (int iy = 0; iy < HH; ++iy) {
            float2 v[3];
#pragma unroll
            for (int dx = 0; dx < 3; ++dx) {
              const int d = iy * HALO + dx;
              v[dx] = __bfloat1622float2(*reinterpret_cast<const __nv_bfloat162*>(col[d & 7] + d * 64));
            }
#pragma unroll
            for (int dy = 0; dy < 3; ++dy) {  // output row oy takes input row iy as its tap row dy
              if (iy < dy || (iy - dy) % S != 0 || (iy - dy) / S >= TH) continue;
              const int oy = (iy - dy) / S;
#pragma unroll
              for (int dx = 0; dx < 3; ++dx) {
                acc[oy].x = fmaf(v[dx].x, w[dy * 3 + dx].x, acc[oy].x);
                acc[oy].y = fmaf(v[dx].y, w[dy * 3 + dx].y, acc[oy].y);
              }
            }
            if constexpr (TH != kTile) {  // stride 1: input row iy is output row iy - 2's last tap row
              if (iy >= 2) put(iy - 2, out(iy - 2));
            }
          }
          if constexpr (TH == kTile) {
#pragma unroll
            for (int oy = 0; oy < TH; ++oy) put(oy, out(oy));
          }
        } else {  // a lane past the chunk's channels writes zeros
#pragma unroll
          for (int oy = 0; oy < TH; ++oy) put(oy, 0u);
        }
      });
      fence_proxy_async();  // generic-proxy writes of A -> visible to the wgmma (async proxy) reads
      clk.lap(kDepthwise);
      // A is complete, and both warpgroups are done reading E
      named_bar_sync(kConsumerBar, pipe::kConsumerThreads);
      clk.lap(kBarrier);

      // projection: acc2 += A2 rows [proj_row, + 64) . W2_chunk rows [proj_col, + proj_n)^T, one MMA of width proj_n
      // per k step
      wgmma_fence();
      {
        const uint64_t da = make_smem_desc(smem_u32(a2) + (uint32_t)(proj_row * 128));
        const uint64_t db = make_smem_desc(smem_u32(sp) + a.l.w2 + (uint32_t)(proj_col * 128));
        auto project = [&](auto width) {
          for (int ks = 0; ks < nch / 16; ++ks)
            wgmma_into<decltype(width)::value>(acc2, da + (uint64_t)(ks * 2), db + (uint64_t)(ks * 2),
                                               (c0 | ks) ? 1u : 0u);
        };
        // cout_p is a multiple of 16 and at most kMaxCout, and at most 128 for a tall tile (plan())
        switch (proj_n) {
          case 8: project(std::integral_constant<int, 8>{}); break;
          case 16: project(std::integral_constant<int, 16>{}); break;
          case 24: project(std::integral_constant<int, 24>{}); break;
          case 32: project(std::integral_constant<int, 32>{}); break;
          case 40: project(std::integral_constant<int, 40>{}); break;
          case 48: project(std::integral_constant<int, 48>{}); break;
          case 56: project(std::integral_constant<int, 56>{}); break;
          case 64: project(std::integral_constant<int, 64>{}); break;
          case 72: project(std::integral_constant<int, 72>{}); break;
          case 80: project(std::integral_constant<int, 80>{}); break;
          case 88: project(std::integral_constant<int, 88>{}); break;
          case 96: project(std::integral_constant<int, 96>{}); break;
          case 104: project(std::integral_constant<int, 104>{}); break;
          case 112: project(std::integral_constant<int, 112>{}); break;
          case 120: project(std::integral_constant<int, 120>{}); break;
          case 128: project(std::integral_constant<int, 128>{}); break;
        }
      }
      wgmma_commit();
      clk.lap(kProjectMma);

      if (next && !ahead) {  // one stage: chunk c + 1 lands only once chunk c's stage is free
        wgmma_wait<0>();
        ring.release();
        sn = ring.wait_ptr();
        clk.lap(kRingWait);
        expand_issue(sn);
      }
      // Retires chunk c + 1's expansion too.  Waiting for it alone (wait_group 1) and running its epilogue under the
      // projection makes ptxas serialise the wgmmas (C7514), so the two retire together.
      wgmma_wait<0>();
      reg_fence(acc2);
      if (!next || ahead) ring.release();
      clk.lap(kProjectMma);
      if (next) {
        expand_epilogue(sn, min(kChunk, a.cmid_p - c0 - kChunk), inside);
        if (c + 2 == nchunks) mbar_arrive(xs_empty);  // this thread's reads of the halo are complete
        clk.lap(kExpandEpi);
      }
    }

    // epilogue: + bias (+ block input) -> bf16.  A thread holds pixels proj_row + 16 warp + lane / 4 (+ 8) of the tile,
    // columns proj_col + 8 j + 2 quad (+ 1).  Every bias and residual value is loaded before the first store: as far as
    // the compiler knows Y may alias b2 and X, so a load placed after a store would wait for it, one global-load
    // latency per column pair.
    {
      constexpr int J = kMaxCout / 16;  // column groups of 8 a warpgroup holds at most
      bool in[2];
      int64_t pix[2];
#pragma unroll
      for (int h = 0; h < 2; ++h) {
        const int px = proj_row + warp * 16 + (lane >> 2) + 8 * h;
        const int oy = oy0 + (px >> 3), ox = ox0 + (px & 7);
        in[h] = oy < a.Ho && ox < a.Wo;
        pix[h] = ((int64_t)b * a.Ho + oy) * a.Wo + ox;
      }
      float2 bias[J];
      uint32_t res[2][J];  // bf16 pairs of the block input (stride 1, cin_p == cout_p) at the same pixel
#pragma unroll
      for (int j = 0; j < J; ++j) {
        bias[j] = make_float2(0.f, 0.f);
        res[0][j] = res[1][j] = 0u;
        if (8 * j >= proj_n) continue;
        const int n = proj_col + 8 * j + 2 * quad;
        bias[j] = make_float2(__ldg(&a.b2[n]), __ldg(&a.b2[n + 1]));
#pragma unroll
        for (int h = 0; h < 2; ++h)
          if (a.residual && in[h]) res[h][j] = *reinterpret_cast<const uint32_t*>(a.X + pix[h] * a.cin_p + n);
      }
#pragma unroll
      for (int h = 0; h < 2; ++h) {
        if (!in[h]) continue;
#pragma unroll
        for (int j = 0; j < J; ++j) {
          if (8 * j >= proj_n) break;
          const int n = proj_col + 8 * j + 2 * quad;
          float f0 = acc2[4 * j + 2 * h] + bias[j].x;
          float f1 = acc2[4 * j + 2 * h + 1] + bias[j].y;
          if (a.residual) {
            f0 += __uint_as_float(res[h][j] << 16);
            f1 += __uint_as_float(res[h][j] & 0xffff0000u);
          }
          *reinterpret_cast<__nv_bfloat162*>(a.Y + pix[h] * a.cout_p + n) = __floats2bfloat162_rn(f0, f1);
        }
      }
    }
    clk.lap(kEpilogue);
  }
  if (wt == 0) clk.flush(1 + wg);
}

// The shapes the fused path takes: those whose single-buffered tile working set (input halo, one W1 and W2 chunk,
// the projection A operand and E, all at whole 64-row granularity) fits in shared memory.  This is the rule of the
// earlier single-warpgroup kernel, kept so that exactly the same blocks fuse (the rest run layer by layer) rather
// than the set drifting with this kernel's layout.  Every such shape fits that layout with at least one stage: a
// one-stage layout is never larger for blocks with an expansion (E holds only the halo pixels, not 64-row blocks), and
// at most 48 bytes larger for the no-expansion blocks, whose working set is far below the limit.
static bool fits(const BlockDesc& d) {
  const size_t hr = (size_t)halo_rows(d.stride, kTile);
  const size_t kbx = d.has_expand ? (size_t)((d.cin_p + 63) / 64) : 0;
  const size_t n2 = (size_t)((d.cout_p + 63) / 64 * 64);
  const size_t set = kbx * hr * 128 + kbx * kChunk * 128 + n2 * 128 + 64 * 128 + hr * 128;
  return set + 1024 <= kSmemMax;
}

bool plan(const BlockDesc& d, Plan* out) {
  if (d.stride != 1 && d.stride != 2) return false;
  if (d.cout_p > kMaxCout || d.cout_p % 16 || d.cmid_p % 16 || d.cin_p % 16) return false;
  if (!d.has_expand && d.cin_p != d.cmid_p) return false;
  if (d.residual && (d.stride != 1 || d.cin_p != d.cout_p)) return false;
  if (!fits(d)) return false;
  auto deepest = [&](int th) {  // the layout with as many ring stages as fit
    Layout l = layout(d.stride, th, d.has_expand != 0, d.cin_p, d.cout_p, kMaxStages);
    for (int s = kMaxStages - 1; s >= 1 && l.smem > kSmemMax; --s)
      l = layout(d.stride, th, d.has_expand != 0, d.cin_p, d.cout_p, s);
    return l;
  };
  Layout l = deepest(kTile);
  // The tall tile halves the per-pixel share of each chunk's fixed costs (barriers, ring and halo waits, MMA issue)
  // and runs the expansion over 184 halo pixels per 128 outputs instead of 104 per 64.  It needs stride 1, cout_p <=
  // 128 so that one warpgroup's projection over all the columns keeps 64 accumulator registers, and as deep a ring as
  // the 8 x 8 tile: a shallower ring would stall the pipeline more than the tile saves.
  if (d.stride == 1 && d.cout_p <= 128) {
    const Layout t = deepest(kTallTile);
    if (t.smem <= kSmemMax && t.stages == l.stages) l = t;
  }
  out->stages = l.stages;
  out->tile_h = l.th;
  out->smem_bytes = l.smem;
  return out->smem_bytes <= kSmemMax;
}

template <int S, bool kExpand>
static int launch(const CUtensorMap& mx, const CUtensorMap& m1, const CUtensorMap& m2, const Args& a, size_t smem,
                  cudaStream_t st) {
  AM_TRY((allow_dynamic_smem<fused_block_kernel<S, kExpand>>(kSmemMax)));
  const int grid = std::max(1, std::min(a.num_tiles, sm_count()));
#ifdef AM_FUSED_PHASES
  void* counters = nullptr;
  AM_CUDA(cudaGetSymbolAddress(&counters, g_phase_cycles));
  AM_CUDA(cudaMemsetAsync(counters, 0, sizeof(g_phase_cycles), st));
#endif
  AM_LAUNCH((fused_block_kernel<S, kExpand>), grid, pipe::kThreads, smem, st, mx, m1, m2, a);
#ifdef AM_FUSED_PHASES
  unsigned long long c[3][kNumPhases];
  AM_CUDA(cudaStreamSynchronize(st));
  AM_CUDA(cudaMemcpyFromSymbol(c, g_phase_cycles, sizeof(c)));
  std::fprintf(stderr, "fused_phases H=%d W=%d cin=%d cmid=%d cout=%d S=%d stages=%d grid=%d tiles=%d", a.H, a.W,
               a.cin_p, a.cmid_p, a.cout_p, S, a.l.stages, grid, a.num_tiles);
  for (int w = 0; w < 3; ++w)
    for (int p = 0; p < kNumPhases; ++p) std::fprintf(stderr, " wg%d.%s=%llu", w, kPhaseNames[p], c[w][p]);
  std::fprintf(stderr, "\n");
#endif
  return AM_OK;
}

std::vector<float> pack_params(const std::vector<float>& wd, const std::vector<float>& bd, const std::vector<float>* b1,
                               int c_p) {
  const int chunks = (c_p + kChunk - 1) / kChunk;
  std::vector<float> out((size_t)chunks * kParamRows * kChunk, 0.f);
  for (int c = 0; c < c_p; ++c) {
    float* q = &out[((size_t)(c / kChunk) * kParamRows) * kChunk + c % kChunk];
    for (int t = 0; t < 9; ++t) q[t * kChunk] = wd[(size_t)t * c_p + c];
    q[9 * kChunk] = bd[c];
    if (b1) q[10 * kChunk] = (*b1)[c];
  }
  return out;
}

int run(const BlockDesc& d, const Plan& p, const __nv_bfloat16* X, const __nv_bfloat16* W1, const float* params,
        const __nv_bfloat16* W2, const float* b2, __nv_bfloat16* Y, int B, cudaStream_t st) {
  AM_CHECK(X && params && W2 && b2 && Y && (!d.has_expand || W1), "fused block: NULL operand");
  auto aligned16 = [](const void* q) { return (reinterpret_cast<uintptr_t>(q) & 15) == 0; };
  AM_CHECK(aligned16(X) && aligned16(W2) && aligned16(params) && (!d.has_expand || aligned16(W1)),
           "fused block: operands must be 16-byte aligned (TMA)");
  Args a{};
  a.X = X;
  a.params = params;
  a.b2 = b2;
  a.Y = Y;
  a.H = d.H;
  a.W = d.W;
  a.Ho = (d.H - 1) / d.stride + 1;  // 3 x 3, pad 1
  a.Wo = (d.W - 1) / d.stride + 1;
  AM_CHECK(p.tile_h == kTile || (p.tile_h == kTallTile && d.stride == 1 && d.cout_p <= 128),
           "fused block: plan does not match the block");
  a.tiles_y = (a.Ho + p.tile_h - 1) / p.tile_h;
  a.tiles_x = (a.Wo + kTile - 1) / kTile;
  const int64_t tiles = (int64_t)B * a.tiles_y * a.tiles_x;
  AM_CHECK(tiles < ((int64_t)1 << 31), "fused block: %lld tiles is too many for one launch", (long long)tiles);
  a.num_tiles = (int)tiles;
  a.cin_p = d.cin_p;
  a.cmid_p = d.cmid_p;
  a.cout_p = d.cout_p;
  a.residual = d.residual;
  const Layout l = layout(d.stride, p.tile_h, d.has_expand != 0, d.cin_p, d.cout_p, p.stages);
  AM_CHECK(l.smem == p.smem_bytes, "fused block: plan does not match the block");
  a.l = l;

  CUtensorMap mx, m1, m2;
  AM_TRY(gemm::encode_map_nhwc_bf16(&mx, X, B, d.H, d.W, d.cin_p, halo(d.stride), halo_h(d.stride, p.tile_h), true));
  AM_TRY(gemm::encode_map_bf16(&m2, W2, d.cmid_p, d.cout_p, d.cmid_p, (d.cout_p + 63) / 64 * 64));
  if (d.has_expand) AM_TRY(gemm::encode_map_bf16(&m1, W1, d.cin_p, d.cmid_p, d.cin_p, kChunk));
  else m1 = m2;  // unused
  if (d.stride == 1) return d.has_expand ? launch<1, true>(mx, m1, m2, a, l.smem, st) : launch<1, false>(mx, m1, m2, a, l.smem, st);
  return d.has_expand ? launch<2, true>(mx, m1, m2, a, l.smem, st) : launch<2, false>(mx, m1, m2, a, l.smem, st);
}

}  // namespace fused
}  // namespace am
