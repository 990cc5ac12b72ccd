// Warpgroup-MMA / TMA GEMM for sm_90a (see gemm_wgmma.cuh for the contract).
//
// Persistent CTA of 384 threads (three warpgroups), one CTA per SM, tile = 128 rows x BN columns:
//   warpgroup 0   TMA producer (one elected lane of warp 0): cp.async.bulk.tensor loads of the A tile [128 x 64]
//                 and the B tile [BN x 64] (bf16, 128-byte swizzle) into a shared-memory ring of up to 4 stages;
//   warpgroups 1, 2   consumers, rows [0, 64) and [64, 128) of the tile: wgmma.mma_async m64nBNk16 straight from
//                 the swizzled tiles into fp32 register accumulators, then the epilogue from registers:
//                 alpha / bias / ReLU6 / residual -> bf16 or fp32 (+ the k-NN chunk maxima).  A bf16 tile is staged
//                 in shared memory and leaves through TMA stores (cp.async.bulk.tensor ... bulk_group) that one
//                 thread of the warpgroup issues; the warpgroup goes straight on to the next tile's MMAs and waits
//                 for the stores to have read the staging tile only before it writes that tile again.
// The ring and its barriers are tma_pipeline.cuh's.  While the consumers run an epilogue the producer is already
// filling the ring with the next tile's first K blocks.
#include "gemm_wgmma.cuh"
#include "tma_pipeline.cuh"

#include <mutex>

namespace am {
namespace gemm {

using pipe::kChunkK;
using pipe::kThreads;

constexpr int kBlockM = 128;
constexpr int kStages = 4;             // at most; fewer when a wide B tile would not fit
constexpr int kATileBytes = kBlockM * kChunkK * 2;  // 16 KiB
constexpr int kMaxBlockN = 256;
constexpr size_t kSmemMax = 232448;    // 227 KiB: the opt-in limit of one block on sm_90
using Ring = pipe::Ring<kStages>;

using namespace ptx;

struct KernelArgs {
  int64_t M, N;
  int K;
  int block_n;
  int tiles_m, tiles_n;
  int m_fastest;
  void* D;
  int64_t ldd;
  int d_is_f32;
  int d_vec;      // fp32 D rows allow 2-element vector stores (even ldd, aligned base)
  float alpha;
  const float* bias;
  const float* col_sub;
  int act;
  const __nv_bfloat16* residual;  // bf16 D only; ld_res even and a 4-byte aligned base (2-element loads)
  int64_t ld_res;
  float* chunk_max;  // k-NN: per-32-column maxima beside D (see Epilogue::chunk_max)
  int64_t ld_cm;
  int stages;     // smem ring depth
};

// The bf16 staging tile of one consumer warpgroup: its 64 rows x BN columns as the boxes of the TMA stores, BN / 64
// boxes of 64 columns (128-byte rows, SWIZZLE_128B), then, when BN % 64 != 0, one narrower box of the last BN % 64
// columns through a second tensor map: 32- and 64-byte rows with the matching SWIZZLE_32B / _64B, 96-byte rows
// unswizzled.  Every box starts 1024-byte aligned.  The swizzles spread a warp's fragment stores (8 rows x 4 column
// pairs) over all 32 banks; only the 96-byte box has two-way conflicts.
template <int BN>
constexpr int stage_bytes() { return 64 * BN * 2; }
constexpr int tail_swizzle_bytes(int tail_cols) { return tail_cols == 16 ? 32 : tail_cols == 32 ? 64 : 0; }

// byte offset in the staging tile of the bf16 pair at (row r, even column c)
template <int BN>
__device__ __forceinline__ uint32_t stage_offset(int r, int c) {
  constexpr int kTail = BN % 64;
  if (c < BN - kTail) {  // a 64-column box: 16-byte chunk index ^= row % 8
    const uint32_t o = (uint32_t)(r * 128 + (c % 64) * 2);
    return (uint32_t)(c / 64) * 8192u + (o ^ (((o >> 7) & 7u) << 4));
  }
  const uint32_t o = (uint32_t)(r * kTail * 2 + (c - (BN - kTail)) * 2);
  constexpr int kSw = tail_swizzle_bytes(kTail);
  const uint32_t sw = kSw == 32 ? ((o >> 7) & 1u) << 4 : kSw == 64 ? ((o >> 7) & 3u) << 4 : 0u;
  return (uint32_t)(BN / 64) * 8192u + (o ^ sw);
}

__device__ __forceinline__ void tile_coords(const KernelArgs& a, int tile, int& m_blk, int& n_blk) {
  if (a.m_fastest) {
    m_blk = tile % a.tiles_m;
    n_blk = tile / a.tiles_m;
  } else {
    n_blk = tile % a.tiles_n;
    m_blk = tile / a.tiles_n;
  }
}

__device__ __forceinline__ float epi_act(float v, int act) {
  if (act == 1) return relu6f(v);
  if (act == 2) return fmaxf(v, 0.f);                                         // ReLU
  if (act == 3) return v * fminf(fmaxf(fmaf(v, 1.0f / 6.0f, 0.5f), 0.f), 1.f);  // HardSwish
  return v;
}

// bias[n] - col_sub[n] of this thread's column pair n, n + 1 (0 outside the matrix), loaded once per tile
__device__ __forceinline__ void epi_cols(const KernelArgs& a, bool has_cols, int64_t n, float& cb0, float& cb1) {
  cb0 = 0.f;
  cb1 = 0.f;
  if (!has_cols) return;
  if (n < a.N) {
    if (a.bias) cb0 += __ldg(&a.bias[n]);
    if (a.col_sub) cb0 -= __ldg(&a.col_sub[n]);
  }
  if (n + 1 < a.N) {
    if (a.bias) cb1 += __ldg(&a.bias[n + 1]);
    if (a.col_sub) cb1 -= __ldg(&a.col_sub[n + 1]);
  }
}

// act(alpha * v + cb): the epilogue before the residual
__device__ __forceinline__ float epi_value(const KernelArgs& a, float v, float cb) {
  if (a.alpha != 1.0f) v *= a.alpha;
  return epi_act(v + cb, a.act);
}

template <int BN>
__global__ void __launch_bounds__(kThreads, 1)
gemm_wgmma_kernel(const __grid_constant__ CUtensorMap map_a, const __grid_constant__ CUtensorMap map_b,
                  const __grid_constant__ CUtensorMap map_d, const __grid_constant__ CUtensorMap map_d_tail,
                  const KernelArgs args) {
  extern __shared__ __align__(1024) uint8_t smem_raw[];
  // after the ring, for a bf16 D: the two consumer warpgroups' staging tiles
  Ring ring(smem_raw, kATileBytes + BN * kChunkK * 2, args.stages, args.d_is_f32 ? 0 : 2 * stage_bytes<BN>());

  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int num_tiles = args.tiles_m * args.tiles_n;

  if (threadIdx.x == 0) {
    prefetch_tensormap(&map_a);
    prefetch_tensormap(&map_b);
    if (!args.d_is_f32) {
      if (BN >= 64) prefetch_tensormap(&map_d);
      if (BN % 64 != 0) prefetch_tensormap(&map_d_tail);
    }
    ring.init();
  }
  __syncthreads();

  if (warp < 4) {
    regs_producer();
    // ===================== TMA producer =====================
    if (warp == 0 && elect_one_sync()) {
      const int num_kb = (args.K + kChunkK - 1) / kChunkK;
      for (int tile = blockIdx.x; tile < num_tiles; tile += gridDim.x) {
        int m_blk, n_blk;
        tile_coords(args, tile, m_blk, n_blk);
        for (int kb = 0; kb < num_kb; ++kb) {
          const Ring::Slot s = ring.acquire();
          tma_load_2d(s.smem, &map_a, s.bar, kb * kChunkK, m_blk * kBlockM);
          tma_load_2d(s.smem + kATileBytes, &map_b, s.bar, kb * kChunkK, n_blk * BN);
        }
      }
    }
    return;
  }
  regs_consumer();
  // ===================== consumers: warpgroups 1 and 2 =====================
  const int wg = (threadIdx.x >> 7) - 1;      // 0: tile rows [0, 64), 1: [64, 128)
  const int wt = threadIdx.x & 127;
  const int quad = lane & 3;
  const bool has_cols = (args.bias != nullptr) || (args.col_sub != nullptr);
  float acc[BN / 2];
#pragma unroll
  for (int i = 0; i < BN / 2; ++i) acc[i] = 0.f;
  for (int tile = blockIdx.x; tile < num_tiles; tile += gridDim.x) {
    int m_blk, n_blk;
    tile_coords(args, tile, m_blk, n_blk);
    pipe::mma_k_loop<BN>(ring, acc, (uint32_t)(wg * 64 * 128), (uint32_t)kATileBytes, args.K);
    // ---- epilogue straight from the accumulator registers, each read once (an accumulator written by any other
    //      instruction would make ptxas serialise every wgmma of the kernel)
    const int64_t n_base = (int64_t)n_blk * BN;
    const int64_t row0 = (int64_t)m_blk * kBlockM + wg * 64 + (wt >> 5) * 16 + (lane >> 2);
    if (!args.d_is_f32) {  // bf16: fragment -> swizzled staging tile -> TMA stores (rows >= M, columns >= N clipped)
      uint8_t* stg = ring.extra() + wg * stage_bytes<BN>();
      const int r_lo = (wt >> 5) * 16 + (lane >> 2);
      if (wt == 0) bulk_wait_group_read<0>();  // the previous tile's stores have read the staging tile ...
      named_bar_sync(1 + wg, 128);             // ... before any thread of the warpgroup writes it again
#pragma unroll
      for (int j = 0; j < BN / 8; ++j) {
        const int64_t n = n_base + 8 * j + 2 * quad;  // this thread's two columns: n, n + 1
        float cb0, cb1;
        epi_cols(args, has_cols, n, cb0, cb1);
#pragma unroll
        for (int h = 0; h < 2; ++h) {
          const int64_t row = row0 + 8 * h;
          float f0 = epi_value(args, acc[4 * j + 2 * h], cb0), f1 = epi_value(args, acc[4 * j + 2 * h + 1], cb1);
          if (args.residual && row < args.M && n < args.N) {
            const __nv_bfloat16* r = args.residual + row * args.ld_res + n;
            if (n + 1 < args.N) {
              const float2 rv = __bfloat1622float2(*reinterpret_cast<const __nv_bfloat162*>(r));
              f0 += rv.x;
              f1 += rv.y;
            } else {
              f0 += __bfloat162float(r[0]);
            }
          }
          *reinterpret_cast<__nv_bfloat162*>(stg + stage_offset<BN>(r_lo + 8 * h, 8 * j + 2 * quad)) =
              __floats2bfloat162_rn(f0, f1);
        }
      }
      fence_proxy_async();  // the staging writes are visible to the TMA unit's reads
      named_bar_sync(1 + wg, 128);
      if (wt == 0) {
        const int row_tile = m_blk * kBlockM + wg * 64;
#pragma unroll
        for (int b = 0; b < BN / 64; ++b) tma_store_2d(&map_d, stg + b * 8192, (int)n_base + 64 * b, row_tile);
        if (BN % 64 != 0) tma_store_2d(&map_d_tail, stg + (BN / 64) * 8192, (int)n_base + BN - BN % 64, row_tile);
        bulk_commit_group();
      }
      continue;
    }
    // fp32 D, stored from registers; k-NN: the maximum of every 32-column chunk (columns >= N excluded); BN % 32 == 0 when chunk_max is set
    float mx[2] = {-INFINITY, -INFINITY};
#pragma unroll
    for (int j = 0; j < BN / 8; ++j) {
      const int64_t n = n_base + 8 * j + 2 * quad;
      const bool pair = n + 1 < args.N;
      float cb0, cb1;
      epi_cols(args, has_cols, n, cb0, cb1);
#pragma unroll
      for (int h = 0; h < 2; ++h) {
        const int64_t row = row0 + 8 * h;
        float f0 = epi_value(args, acc[4 * j + 2 * h], cb0), f1 = epi_value(args, acc[4 * j + 2 * h + 1], cb1);
        if (args.chunk_max) {
          if (n < args.N) mx[h] = fmaxf(mx[h], f0);
          if (pair) mx[h] = fmaxf(mx[h], f1);
        }
        if (row >= args.M || n >= args.N) continue;
        float* d = reinterpret_cast<float*>(args.D) + row * args.ldd + n;
        if (pair && args.d_vec) {
          *reinterpret_cast<float2*>(d) = make_float2(f0, f1);
        } else {
          d[0] = f0;
          if (pair) d[1] = f1;
        }
      }
      if (args.chunk_max && j % 4 == 3) {
#pragma unroll
        for (int h = 0; h < 2; ++h) {
          mx[h] = fmaxf(mx[h], __shfl_xor_sync(0xffffffffu, mx[h], 1));
          mx[h] = fmaxf(mx[h], __shfl_xor_sync(0xffffffffu, mx[h], 2));
          const int64_t row = row0 + 8 * h;
          const int64_t n0 = n_base + 8 * (j - 3);
          if (quad == 0 && row < args.M && n0 < args.N) args.chunk_max[row * args.ld_cm + (n0 >> 5)] = mx[h];
          mx[h] = -INFINITY;
        }
      }
    }
  }
  if (!args.d_is_f32 && wt == 0) bulk_wait_group<0>();  // the last tile's stores are done before the CTA exits
}

// ---------------------------------------------------------------- SIMT reference (self test only)
__global__ void gemm_simt_kernel(const __nv_bfloat16* __restrict__ A, int64_t M, int64_t lda,
                                 const __nv_bfloat16* __restrict__ B, int64_t N, int64_t ldb, int K,
                                 KernelArgs args) {
  const int64_t n = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  const int64_t m = blockIdx.y;
  if (n >= N || m >= M) return;
  float acc = 0.f;
  for (int k = 0; k < K; ++k) acc = fmaf(__bfloat162float(A[m * lda + k]), __bfloat162float(B[n * ldb + k]), acc);
  float v = acc * args.alpha;
  if (args.bias) v += args.bias[n];
  if (args.col_sub) v -= args.col_sub[n];
  if (args.act == 1) v = relu6f(v);
  else if (args.act == 2) v = fmaxf(v, 0.f);
  else if (args.act == 3) v *= fminf(fmaxf(fmaf(v, 1.0f / 6.0f, 0.5f), 0.f), 1.f);
  if (args.d_is_f32) {
    reinterpret_cast<float*>(args.D)[m * args.ldd + n] = v;
  } else {
    if (args.residual) v += __bfloat162float(args.residual[m * args.ld_res + n]);
    reinterpret_cast<__nv_bfloat16*>(args.D)[m * args.ldd + n] = __float2bfloat16_rn(v);
  }
}

// ---------------------------------------------------------------- host
typedef CUresult (*EncodeTiledFn)(CUtensorMap*, CUtensorMapDataType, cuuint32_t, void*, const cuuint64_t*,
                                  const cuuint64_t*, const cuuint32_t*, const cuuint32_t*, CUtensorMapInterleave,
                                  CUtensorMapSwizzle, CUtensorMapL2promotion, CUtensorMapFloatOOBfill);

static EncodeTiledFn g_encode = nullptr;
static std::once_flag g_encode_once;

static EncodeTiledFn get_encode() {
  std::call_once(g_encode_once, [] {
    void* fn = nullptr;
    cudaDriverEntryPointQueryResult qres;
    cudaError_t e = cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &fn, cudaEnableDefault, &qres);
    if (e == cudaSuccess && qres == cudaDriverEntryPointSuccess) g_encode = reinterpret_cast<EncodeTiledFn>(fn);
    cudaGetLastError();
  });
  return g_encode;
}

bool available() { return ensure_init() == AM_OK && device_cc() == 90 && get_encode() != nullptr; }

int encode_map_bf16(void* map_out, const void* base, int64_t inner, int64_t rows, int64_t pitch_elems, int box_rows) {
  AM_CHECK(get_encode() != nullptr, "cuTensorMapEncodeTiled unavailable");
  const cuuint64_t dims[2] = {(cuuint64_t)inner, (cuuint64_t)rows};
  const cuuint64_t strides[1] = {(cuuint64_t)pitch_elems * 2};
  const cuuint32_t box[2] = {(cuuint32_t)kChunkK, (cuuint32_t)box_rows};
  const cuuint32_t estr[2] = {1, 1};
  CUresult r = get_encode()(reinterpret_cast<CUtensorMap*>(map_out), CU_TENSOR_MAP_DATA_TYPE_BFLOAT16, 2,
                            const_cast<void*>(base), dims, strides, box, estr, CU_TENSOR_MAP_INTERLEAVE_NONE,
                            CU_TENSOR_MAP_SWIZZLE_128B, CU_TENSOR_MAP_L2_PROMOTION_L2_256B,
                            CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
  if (r != CUDA_SUCCESS) {
    set_error("cuTensorMapEncodeTiled failed (%d) inner=%lld rows=%lld pitch=%lld box_rows=%d", (int)r,
              (long long)inner, (long long)rows, (long long)pitch_elems, box_rows);
    return AM_ERR_CUDA;
  }
  return AM_OK;
}

int encode_map_nhwc_bf16(void* map_out, const void* base, int64_t n, int64_t h, int64_t w, int64_t c, int box_w,
                         int box_h, bool swizzle) {
  AM_CHECK(get_encode() != nullptr, "cuTensorMapEncodeTiled unavailable");
  const cuuint64_t dims[4] = {(cuuint64_t)c, (cuuint64_t)w, (cuuint64_t)h, (cuuint64_t)n};
  const cuuint64_t strides[3] = {(cuuint64_t)(c * 2), (cuuint64_t)(w * c * 2), (cuuint64_t)(h * w * c * 2)};
  const cuuint32_t box[4] = {(cuuint32_t)kChunkK, (cuuint32_t)box_w, (cuuint32_t)box_h, 1};
  const cuuint32_t estr[4] = {1, 1, 1, 1};
  CUresult r = get_encode()(reinterpret_cast<CUtensorMap*>(map_out), CU_TENSOR_MAP_DATA_TYPE_BFLOAT16, 4,
                            const_cast<void*>(base), dims, strides, box, estr, CU_TENSOR_MAP_INTERLEAVE_NONE,
                            swizzle ? CU_TENSOR_MAP_SWIZZLE_128B : CU_TENSOR_MAP_SWIZZLE_NONE,
                            CU_TENSOR_MAP_L2_PROMOTION_L2_256B, CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
  if (r != CUDA_SUCCESS) {
    set_error("cuTensorMapEncodeTiled failed (%d) nhwc=[%lld, %lld, %lld, %lld] box=%dx%d", (int)r, (long long)n,
              (long long)h, (long long)w, (long long)c, box_w, box_h);
    return AM_ERR_CUDA;
  }
  return AM_OK;
}

// The TMA map a bf16 D leaves through: [rows, cols] with rows `pitch_elems` apart (a multiple of 8), stored in boxes
// of box_cols x 64 rows swizzled as stage_offset lays them out.
static int encode_map_d(CUtensorMap* map_out, void* D, int64_t cols, int64_t rows, int64_t pitch_elems, int box_cols) {
  const cuuint64_t dims[2] = {(cuuint64_t)cols, (cuuint64_t)rows};
  const cuuint64_t strides[1] = {(cuuint64_t)pitch_elems * 2};
  const cuuint32_t box[2] = {(cuuint32_t)box_cols, 64};
  const cuuint32_t estr[2] = {1, 1};
  const int sw = box_cols == 64 ? 128 : tail_swizzle_bytes(box_cols);
  const CUtensorMapSwizzle swizzle = sw == 128  ? CU_TENSOR_MAP_SWIZZLE_128B
                                     : sw == 64 ? CU_TENSOR_MAP_SWIZZLE_64B
                                     : sw == 32 ? CU_TENSOR_MAP_SWIZZLE_32B
                                                : CU_TENSOR_MAP_SWIZZLE_NONE;
  CUresult r = get_encode()(map_out, CU_TENSOR_MAP_DATA_TYPE_BFLOAT16, 2, D, dims, strides, box, estr,
                            CU_TENSOR_MAP_INTERLEAVE_NONE, swizzle, CU_TENSOR_MAP_L2_PROMOTION_NONE,
                            CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
  if (r != CUDA_SUCCESS) {
    set_error("cuTensorMapEncodeTiled failed (%d) for D: cols=%lld rows=%lld pitch=%lld box_cols=%d", (int)r,
              (long long)cols, (long long)rows, (long long)pitch_elems, box_cols);
    return AM_ERR_CUDA;
  }
  return AM_OK;
}

// tile widths gemm_wgmma_kernel is instantiated for (the switch in gemm_bf16)
static bool gemm_has_n(int n) {
  return n == 16 || n == 32 || n == 48 || n == 64 || n == 80 || n == 96 || n == 112 || n == 128 || n == 144 ||
         n == 160 || n == 192 || n == 224 || n == 256;
}

// the smallest instantiated tile width >= n (n <= kMaxBlockN)
static int tile_n_for(int n) {
  for (int c = 16; c <= kMaxBlockN; c += 16)
    if (c >= n && gemm_has_n(c)) return c;
  return kMaxBlockN;
}

// N <= 256: one tile of the smallest width that holds N.  Wider: the width of at least 128 that pads N the least
// (ties to the wider tile, fewer re-reads of A), e.g. 288 = 2 x 144, 1360 -> 11 x 128, 2592 = 18 x 144.  The k-NN
// scores (chunk maxima) keep near-equal tiles of at most 256 columns, rounded to the 32-column chunks.
static int pick_block_n(int64_t N, bool chunk_max) {
  const int64_t n16 = (int64_t)round_up((size_t)N, 16);
  int bn;
  if (n16 <= kMaxBlockN) {
    bn = (int)n16;
  } else if (!chunk_max) {
    int best = kMaxBlockN;
    for (int c = kMaxBlockN; c >= 128; c -= 16) {
      if (!gemm_has_n(c)) continue;
      if ((N + c - 1) / c * c < (N + best - 1) / best * best) best = c;
    }
    return best;
  } else {
    const int64_t tiles = (n16 + kMaxBlockN - 1) / kMaxBlockN;
    bn = (int)round_up((size_t)((n16 + tiles - 1) / tiles), 16);
  }
  if (chunk_max) bn = std::min(kMaxBlockN, (int)round_up((size_t)bn, 32));  // chunk c <-> columns [32c, 32c + 32)
  return tile_n_for(bn);
}

static KernelArgs make_args(int64_t M, int64_t N, int K, void* D, int64_t ldd, bool d_is_f32, const Epilogue& ep,
                            bool m_fastest) {
  KernelArgs a{};
  a.M = M;
  a.N = N;
  a.K = K;
  a.block_n = pick_block_n(N, ep.chunk_max != nullptr);
  a.tiles_m = (int)((M + kBlockM - 1) / kBlockM);
  a.tiles_n = (int)((N + a.block_n - 1) / a.block_n);
  a.m_fastest = m_fastest ? 1 : 0;
  a.D = D;
  a.ldd = ldd;
  a.d_is_f32 = d_is_f32 ? 1 : 0;
  a.d_vec = (ldd % 2 == 0 && (reinterpret_cast<uintptr_t>(D) & (d_is_f32 ? 7 : 3)) == 0) ? 1 : 0;
  a.alpha = ep.alpha;
  a.bias = ep.bias;
  a.col_sub = ep.col_sub;
  a.act = ep.act;
  a.chunk_max = ep.chunk_max;
  a.ld_cm = ep.ld_cm;
  a.residual = ep.residual;
  a.ld_res = ep.ld_res;
  return a;
}

template <int BN>
static int launch_bn(const CUtensorMap& map_a, const CUtensorMap& map_b, KernelArgs& args, cudaStream_t st) {
  AM_TRY(allow_dynamic_smem<gemm_wgmma_kernel<BN>>(kSmemMax));
  CUtensorMap map_d = map_a, map_d_tail = map_a;  // unused for an fp32 D, and for the box kind BN lacks
  if (!args.d_is_f32) {
    if (BN >= 64) AM_TRY(encode_map_d(&map_d, args.D, args.N, args.M, args.ldd, 64));
    if (BN % 64 != 0) AM_TRY(encode_map_d(&map_d_tail, args.D, args.N, args.M, args.ldd, BN % 64));
  }
  const size_t stage_bytes = (size_t)kATileBytes + (size_t)BN * kChunkK * 2;
  const size_t extra = args.d_is_f32 ? 0 : 2 * (size_t)gemm::stage_bytes<BN>();
  args.stages = (int)std::min<size_t>(kStages, (kSmemMax - Ring::smem_bytes(0, 0, extra)) / stage_bytes);
  const size_t smem = Ring::smem_bytes(stage_bytes, args.stages, extra);
  const int tiles = args.tiles_m * args.tiles_n;
  const int grid = std::max(1, std::min(tiles, sm_count()));
  AM_LAUNCH(gemm_wgmma_kernel<BN>, grid, kThreads, smem, st, map_a, map_b, map_d, map_d_tail, args);
  return AM_OK;
}

int gemm_bf16(const __nv_bfloat16* A, int64_t M, int64_t lda, const __nv_bfloat16* B, int64_t N, int64_t ldb, int K,
              void* D, int64_t ldd, bool d_is_f32, const Epilogue& ep, bool m_fastest, cudaStream_t st) {
  AM_CHECK(A && B && D, "gemm: NULL operand");
  AM_CHECK(M > 0 && N > 0 && K > 0, "gemm: empty problem M=%lld N=%lld K=%d", (long long)M, (long long)N, K);
  AM_CHECK(lda % 8 == 0 && ldb % 8 == 0, "gemm: lda/ldb must be multiples of 8 elements (TMA 16-byte pitch)");
  AM_CHECK((reinterpret_cast<uintptr_t>(A) & 15) == 0 && (reinterpret_cast<uintptr_t>(B) & 15) == 0,
           "gemm: operands must be 16-byte aligned");
  AM_CHECK(d_is_f32 || (ldd % 8 == 0 && (reinterpret_cast<uintptr_t>(D) & 15) == 0),
           "gemm: a bf16 D needs ldd a multiple of 8 elements and a 16-byte aligned base (TMA stores)");
  AM_CHECK(d_is_f32 || !ep.chunk_max, "gemm: chunk maxima need an fp32 D");
  AM_CHECK(!ep.residual || (ep.ld_res % 2 == 0 && (reinterpret_cast<uintptr_t>(ep.residual) & 3) == 0),
           "gemm: the residual needs an even ld_res and a 4-byte aligned base");
  AM_CHECK(available(), "gemm: wgmma path unavailable (needs sm_90 and cuTensorMapEncodeTiled)");
  KernelArgs args = make_args(M, N, K, D, ldd, d_is_f32, ep, m_fastest);
  CUtensorMap map_a, map_b;
  AM_TRY(encode_map_bf16(&map_a, A, K, M, lda, kBlockM));
  AM_TRY(encode_map_bf16(&map_b, B, K, N, ldb, args.block_n));
  switch (args.block_n) {
    case 16: return launch_bn<16>(map_a, map_b, args, st);
    case 32: return launch_bn<32>(map_a, map_b, args, st);
    case 48: return launch_bn<48>(map_a, map_b, args, st);
    case 64: return launch_bn<64>(map_a, map_b, args, st);
    case 80: return launch_bn<80>(map_a, map_b, args, st);
    case 96: return launch_bn<96>(map_a, map_b, args, st);
    case 112: return launch_bn<112>(map_a, map_b, args, st);
    case 128: return launch_bn<128>(map_a, map_b, args, st);
    case 144: return launch_bn<144>(map_a, map_b, args, st);
    case 160: return launch_bn<160>(map_a, map_b, args, st);
    case 192: return launch_bn<192>(map_a, map_b, args, st);
    case 224: return launch_bn<224>(map_a, map_b, args, st);
    case 256: return launch_bn<256>(map_a, map_b, args, st);
  }
  set_error("gemm: no kernel for a %d-column tile", args.block_n);
  return AM_ERR_INVALID;
}

int gemm_bf16_simt(const __nv_bfloat16* A, int64_t M, int64_t lda, const __nv_bfloat16* B, int64_t N, int64_t ldb,
                   int K, void* D, int64_t ldd, bool d_is_f32, const Epilogue& ep, cudaStream_t st) {
  AM_CHECK(A && B && D && M > 0 && N > 0 && K > 0, "gemm_simt: bad problem");
  AM_CHECK(M <= 65535, "gemm_simt: M too large for the self-test kernel");
  KernelArgs args = make_args(M, N, K, D, ldd, d_is_f32, ep, false);
  dim3 grid((unsigned)((N + 127) / 128), (unsigned)M);
  AM_LAUNCH(gemm_simt_kernel, grid, 128, 0, st, A, M, lda, B, N, ldb, K, args);
  return AM_OK;
}

}  // namespace gemm
}  // namespace am
