// Warpgroup-MMA / TMA GEMM for sm_90a (see gemm_wgmma.cuh for the contract).
//
// Persistent CTA of 384 threads (three warpgroups), one CTA per SM, tile = 128 rows x BN columns:
//   warpgroup 0   TMA producer (one elected lane of warp 0): cp.async.bulk.tensor loads of the A tile [128 x 64]
//                 and the B tile [BN x 64] (bf16, 128-byte swizzle) into a shared-memory ring of up to 4 stages;
//   warpgroups 1, 2   consumers, rows [0, 64) and [64, 128) of the tile: wgmma.mma_async m64nBNk16 straight from
//                 the swizzled tiles into fp32 register accumulators, then the epilogue from registers:
//                 alpha / bias / ReLU6 / residual -> bf16 or fp32 (+ the k-NN chunk maxima); a bf16 tile goes through
//                 shared memory so that global stores are whole 16-byte chunks of consecutive columns.
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
  int d_vec;      // D rows allow 2-element vector stores (even ldd, aligned base)
  float alpha;
  const float* bias;
  const float* col_sub;
  int act;
  const __nv_bfloat16* residual;
  int64_t ld_res;
  int res_vec;    // residual rows allow 2-element vector loads
  float* chunk_max;  // k-NN: per-32-column maxima beside D (see Epilogue::chunk_max)
  int64_t ld_cm;
  int stages;     // smem ring depth
  int staged;     // bf16 D leaves through a shared-memory tile as whole 16-byte row chunks (coalesced)
};

// per consumer warpgroup: 64 rows of the tile, rows padded by 16 bytes so the fragment writes spread over the banks
template <int BN>
constexpr int stage_pitch() { return BN * 2 + 16; }

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

template <int BN>
__global__ void __launch_bounds__(kThreads, 1)
gemm_wgmma_kernel(const __grid_constant__ CUtensorMap map_a, const __grid_constant__ CUtensorMap map_b,
                  const KernelArgs args) {
  extern __shared__ __align__(1024) uint8_t smem_raw[];
  // after the ring: [2][64][stage_pitch] bf16 output tiles when args.staged
  Ring ring(smem_raw, kATileBytes + BN * kChunkK * 2, args.stages, args.staged ? 2 * 64 * stage_pitch<BN>() : 0);

  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int num_tiles = args.tiles_m * args.tiles_n;
  const int num_kb = (args.K + kChunkK - 1) / kChunkK;

  if (threadIdx.x == 0) {
    prefetch_tensormap(&map_a);
    prefetch_tensormap(&map_b);
    ring.init();
  }
  __syncthreads();

  if (warp < 4) {
    regs_producer();
    // ===================== TMA producer =====================
    if (warp == 0 && elect_one_sync()) {
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
    for (int kb = 0; kb < num_kb; ++kb) {
      const uint32_t s = ring.wait();
      const int ksteps = min(kChunkK, args.K - kb * kChunkK + 15) / 16;  // skip all-zero K tails
      pipe::mma_chunk<BN>(acc, s + (uint32_t)(wg * 64 * 128), s + kATileBytes, ksteps, kb);
      ring.release();
    }
    // ---- epilogue straight from the accumulator registers
    const int64_t n_base = (int64_t)n_blk * BN;
    const int64_t row0 = (int64_t)m_blk * kBlockM + wg * 64 + (wt >> 5) * 16 + (lane >> 2);
#pragma unroll
    for (int j = 0; j < BN / 8; ++j) {
      const int64_t n = n_base + 8 * j + 2 * quad;  // this thread's two columns: n, n + 1
      float cb0 = 0.f, cb1 = 0.f;
      if (has_cols) {
        if (n < args.N) {
          if (args.bias) cb0 += __ldg(&args.bias[n]);
          if (args.col_sub) cb0 -= __ldg(&args.col_sub[n]);
        }
        if (n + 1 < args.N) {
          if (args.bias) cb1 += __ldg(&args.bias[n + 1]);
          if (args.col_sub) cb1 -= __ldg(&args.col_sub[n + 1]);
        }
      }
#pragma unroll
      for (int h = 0; h < 2; ++h) {
        float& f0 = acc[4 * j + 2 * h];
        float& f1 = acc[4 * j + 2 * h + 1];
        if (args.alpha != 1.0f) {
          f0 *= args.alpha;
          f1 *= args.alpha;
        }
        f0 = epi_act(f0 + cb0, args.act);
        f1 = epi_act(f1 + cb1, args.act);
      }
    }
    if (args.staged) {  // bf16: fragment -> shared tile -> 16-byte row chunks
      uint8_t* stg = ring.extra() + wg * 64 * stage_pitch<BN>();
      const int r_lo = (wt >> 5) * 16 + (lane >> 2);
#pragma unroll
      for (int h = 0; h < 2; ++h) {
        const int64_t row = row0 + 8 * h;
#pragma unroll
        for (int j = 0; j < BN / 8; ++j) {
          const int64_t n = n_base + 8 * j + 2 * quad;
          float f0 = acc[4 * j + 2 * h], f1 = acc[4 * j + 2 * h + 1];
          if (args.residual && row < args.M && n < args.N) {  // N % 8 == 0 here: both columns exist
            const float2 rv = __bfloat1622float2(
                *reinterpret_cast<const __nv_bfloat162*>(args.residual + row * args.ld_res + n));
            f0 += rv.x;
            f1 += rv.y;
          }
          *reinterpret_cast<__nv_bfloat162*>(stg + (r_lo + 8 * h) * stage_pitch<BN>() + (8 * j + 2 * quad) * 2) =
              __floats2bfloat162_rn(f0, f1);
        }
      }
      asm volatile("bar.sync %0, 128;" ::"r"(1 + wg) : "memory");
      const int64_t tile_row0 = (int64_t)m_blk * kBlockM + wg * 64;
      for (int idx = wt; idx < 64 * (BN / 8); idx += 128) {
        const int r = idx / (BN / 8), c8 = idx - r * (BN / 8);
        const int64_t row = tile_row0 + r, n = n_base + 8 * c8;
        if (row < args.M && n < args.N)
          *reinterpret_cast<uint4*>(reinterpret_cast<__nv_bfloat16*>(args.D) + row * args.ldd + n) =
              *reinterpret_cast<const uint4*>(stg + r * stage_pitch<BN>() + c8 * 16);
      }
      asm volatile("bar.sync %0, 128;" ::"r"(1 + wg) : "memory");  // the tile is read before the next one is staged
      continue;
    }
    if (args.chunk_max) {  // k-NN: the maximum of every 32-column chunk (columns >= N excluded); BN % 32 == 0 here
#pragma unroll
      for (int c = 0; c < BN / 32; ++c) {
        float mx[2] = {-INFINITY, -INFINITY};
#pragma unroll
        for (int j = 4 * c; j < 4 * c + 4; ++j) {
          const int64_t n = n_base + 8 * j + 2 * quad;
#pragma unroll
          for (int h = 0; h < 2; ++h) {
            if (n < args.N) mx[h] = fmaxf(mx[h], acc[4 * j + 2 * h]);
            if (n + 1 < args.N) mx[h] = fmaxf(mx[h], acc[4 * j + 2 * h + 1]);
          }
        }
#pragma unroll
        for (int h = 0; h < 2; ++h) {
          mx[h] = fmaxf(mx[h], __shfl_xor_sync(0xffffffffu, mx[h], 1));
          mx[h] = fmaxf(mx[h], __shfl_xor_sync(0xffffffffu, mx[h], 2));
          const int64_t row = row0 + 8 * h;
          const int64_t n0 = n_base + 32 * c;
          if (quad == 0 && row < args.M && n0 < args.N) args.chunk_max[row * args.ld_cm + (n0 >> 5)] = mx[h];
        }
      }
    }
#pragma unroll
    for (int h = 0; h < 2; ++h) {
      const int64_t row = row0 + 8 * h;
      if (row >= args.M) continue;
#pragma unroll
      for (int j = 0; j < BN / 8; ++j) {
        const int64_t n = n_base + 8 * j + 2 * quad;
        if (n >= args.N) continue;
        const bool pair = n + 1 < args.N;
        float f0 = acc[4 * j + 2 * h], f1 = acc[4 * j + 2 * h + 1];
        if (args.d_is_f32) {
          float* d = reinterpret_cast<float*>(args.D) + row * args.ldd + n;
          if (pair && args.d_vec) {
            *reinterpret_cast<float2*>(d) = make_float2(f0, f1);
          } else {
            d[0] = f0;
            if (pair) d[1] = f1;
          }
        } else {
          if (args.residual) {
            const __nv_bfloat16* r = args.residual + row * args.ld_res + n;
            if (pair && args.res_vec) {
              const float2 rv = __bfloat1622float2(*reinterpret_cast<const __nv_bfloat162*>(r));
              f0 += rv.x;
              f1 += rv.y;
            } else {
              f0 += __bfloat162float(r[0]);
              if (pair) f1 += __bfloat162float(r[1]);
            }
          }
          __nv_bfloat16* d = reinterpret_cast<__nv_bfloat16*>(args.D) + row * args.ldd + n;
          if (pair && args.d_vec) {
            *reinterpret_cast<__nv_bfloat162*>(d) = __floats2bfloat162_rn(f0, f1);
          } else {
            d[0] = __float2bfloat16_rn(f0);
            if (pair) d[1] = __float2bfloat16_rn(f1);
          }
        }
      }
    }
  }
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

// tile widths gemm_wgmma_kernel is instantiated for (the switch in gemm_bf16)
static bool gemm_has_n(int n) {
  return n == 16 || n == 32 || n == 48 || n == 64 || n == 80 || n == 96 || n == 112 || n == 128 || n == 160 ||
         n == 192 || n == 224 || n == 256;
}

// the smallest instantiated tile width >= n (n <= kMaxBlockN)
static int tile_n_for(int n) {
  for (int c = 16; c <= kMaxBlockN; c += 16)
    if (c >= n && gemm_has_n(c)) return c;
  return kMaxBlockN;
}

static int pick_block_n(int64_t N, bool chunk_max) {
  const int64_t n16 = (int64_t)round_up((size_t)N, 16);
  int bn;
  if (n16 <= kMaxBlockN) {
    bn = (int)n16;
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
  a.res_vec = (ep.ld_res % 2 == 0 && (reinterpret_cast<uintptr_t>(ep.residual) & 3) == 0) ? 1 : 0;
  a.staged = (!d_is_f32 && !ep.chunk_max && N % 8 == 0 && ldd % 8 == 0 && (reinterpret_cast<uintptr_t>(D) & 15) == 0 &&
              (!ep.residual || (ep.ld_res % 2 == 0 && (reinterpret_cast<uintptr_t>(ep.residual) & 3) == 0))) ? 1 : 0;
  return a;
}

template <int BN>
static int launch_bn(const CUtensorMap& map_a, const CUtensorMap& map_b, KernelArgs& args, cudaStream_t st) {
  AM_TRY(allow_dynamic_smem<gemm_wgmma_kernel<BN>>(kSmemMax));
  const size_t stage_bytes = (size_t)kATileBytes + (size_t)BN * kChunkK * 2;
  const size_t extra = args.staged ? 2 * 64 * stage_pitch<BN>() : 0;
  args.stages = (int)std::min<size_t>(kStages, (kSmemMax - Ring::smem_bytes(0, 0, extra)) / stage_bytes);
  const size_t smem = Ring::smem_bytes(stage_bytes, args.stages, extra);
  const int tiles = args.tiles_m * args.tiles_n;
  const int grid = std::max(1, std::min(tiles, sm_count()));
  AM_LAUNCH(gemm_wgmma_kernel<BN>, grid, kThreads, smem, st, map_a, map_b, args);
  return AM_OK;
}

int gemm_bf16(const __nv_bfloat16* A, int64_t M, int64_t lda, const __nv_bfloat16* B, int64_t N, int64_t ldb, int K,
              void* D, int64_t ldd, bool d_is_f32, const Epilogue& ep, bool m_fastest, cudaStream_t st) {
  AM_CHECK(A && B && D, "gemm: NULL operand");
  AM_CHECK(M > 0 && N > 0 && K > 0, "gemm: empty problem M=%lld N=%lld K=%d", (long long)M, (long long)N, K);
  AM_CHECK(lda % 8 == 0 && ldb % 8 == 0, "gemm: lda/ldb must be multiples of 8 elements (TMA 16-byte pitch)");
  AM_CHECK((reinterpret_cast<uintptr_t>(A) & 15) == 0 && (reinterpret_cast<uintptr_t>(B) & 15) == 0,
           "gemm: operands must be 16-byte aligned");
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
