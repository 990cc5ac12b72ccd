// The warp-specialised TMA -> wgmma main loop shared by gemm_wgmma_kernel (gemm.cu), assign_tc_kernel (kmeans_tc.cu),
// silhouette_tc_kernel (cluster_metrics.cu) and fused_block_kernel (fused_block.cu).
//
// A CTA of three warpgroups: warpgroup 0 is the producer (one elected lane of warp 0 issues the TMA loads), warpgroups
// 1 and 2 are consumers (64 rows of the 128-row tile each).  Operand tiles travel through a ring of shared-memory
// stages guarded by two mbarrier arrays: `full` (TMA -> consumers, transaction counted) and `empty` (consumers ->
// TMA, one arrival per consumer thread).  Every thread that takes part keeps its own stage / phase position.
//
// Dynamic shared memory: [alignment slack][stages x stage_bytes][extra_bytes of the kernel's own][full][empty].
#pragma once

#include "ptx_sm90.cuh"

namespace am {
namespace pipe {

constexpr int kThreads = 384;          // producer warpgroup + two consumer warpgroups
constexpr int kConsumerThreads = 256;
constexpr int kChunkK = 64;            // K per stage: 64 bf16 = one 128-byte swizzle row

// kMaxStages barrier pairs are reserved whatever the run-time stage count (the GEMM picks it per tile width).
template <int kMaxStages>
struct Ring {
  // the dynamic shared memory a launch requests for this layout; 1024 bytes of slack for the SWIZZLE_128B alignment
  __host__ __device__ static constexpr size_t smem_bytes(size_t stage_bytes, int stages, size_t extra_bytes) {
    return 1024 + (size_t)stages * stage_bytes + extra_bytes + 2 * kMaxStages * sizeof(uint64_t);
  }

  uint8_t* base;  // stage i at base + i * stage_bytes, 1024-byte aligned
  uint64_t* full;
  uint64_t* empty;
  uint32_t stage_bytes;
  int stages;
  int stage = 0;
  uint32_t phase = 0;

  __device__ __forceinline__ Ring(uint8_t* smem_raw, uint32_t stage_bytes_, int stages_, uint32_t extra_bytes)
      // an offset from smem_raw rather than an integer round trip, so that the compiler still knows every pointer
      // into the ring is shared memory and emits LDS / STS for the kernels' own accesses instead of generic LD / ST
      : base(smem_raw + ((1024u - (ptx::smem_u32(smem_raw) & 1023u)) & 1023u)),
        full(reinterpret_cast<uint64_t*>(base + stages_ * stage_bytes_ + extra_bytes)),
        empty(full + kMaxStages),
        stage_bytes(stage_bytes_),
        stages(stages_) {}

  // the kernel's own region after the ring
  __device__ __forceinline__ uint8_t* extra() const { return base + stages * stage_bytes; }

  // thread 0, before the CTA's first __syncthreads
  __device__ __forceinline__ void init() const {
    for (int i = 0; i < stages; ++i) {
      ptx::mbar_init(&full[i], 1);
      ptx::mbar_init(&empty[i], kConsumerThreads);
    }
    ptx::fence_barrier_init();
    ptx::fence_proxy_async();
  }

  // producer: waits until the consumers have freed the next stage and arms its `full` barrier for a whole stage of
  // TMA bytes; the caller issues the loads of the stage into `smem`, completing on `bar`
  struct Slot {
    uint8_t* smem;
    uint64_t* bar;
  };
  __device__ __forceinline__ Slot acquire() { return acquire(stage_bytes); }
  // ... or for `tx_bytes`, when the loads of a stage do not fill it
  __device__ __forceinline__ Slot acquire(uint32_t tx_bytes) {
    ptx::mbar_wait(&empty[stage], phase ^ 1);
    ptx::mbar_expect_tx(&full[stage], tx_bytes);
    const Slot s{base + stage * stage_bytes, &full[stage]};
    advance();
    return s;
  }

  // consumer: waits until the next stage has landed and returns its shared-memory address ...
  __device__ __forceinline__ uint32_t wait() const { return ptx::smem_u32(wait_ptr()); }
  // ... or its generic address, for ordinary loads from the stage
  __device__ __forceinline__ uint8_t* wait_ptr() const {
    ptx::mbar_wait(&full[stage], phase);
    return base + stage * stage_bytes;
  }
  // ... or, still holding that stage, waits for the one after it without advancing (needs stages > 1)
  __device__ __forceinline__ uint8_t* wait_ahead_ptr() const {
    const int next = stage + 1 == stages ? 0 : stage + 1;
    ptx::mbar_wait(&full[next], next == 0 ? phase ^ 1 : phase);
    return base + next * stage_bytes;
  }
  // ... and hands it back to the producer once this thread's MMAs have read it
  __device__ __forceinline__ void release() {
    ptx::mbar_arrive(&empty[stage]);
    advance();
  }

 private:
  __device__ __forceinline__ void advance() {
    if (++stage == stages) {
      stage = 0;
      phase ^= 1;
    }
  }
};

// The GEMM's whole K loop with one wgmma group in flight: the MMAs of chunk kb are issued and committed, then the
// group of chunk kb - 1 is retired (wgmma.wait_group 1) and its stage released, so the tensor pipe never drains between
// K chunks.  D[64 x N] = sum over the ceil(K / 64) chunks of A[64 x 64] . B[N x 64]^T (K-major SWIZZLE_128B tiles, the
// A tile at byte offset a_off and the B tile at b_off of each stage), 16-wide K steps in order, all-zero K tails
// skipped.  Returns with every MMA complete and every stage released; the accumulators are touched by no other
// instruction until then.
template <int N, int kMaxStages>
__device__ __forceinline__ void mma_k_loop(Ring<kMaxStages>& ring, float (&acc)[N / 2], uint32_t a_off, uint32_t b_off,
                                           int K) {
  const int num_kb = (K + kChunkK - 1) / kChunkK;
  int rd = ring.stage;  // the stage read next: one ahead of ring.stage (the one released next) inside the loop
  uint32_t rd_phase = ring.phase;
  ptx::wgmma_fence();
#pragma unroll 1
  for (int kb = 0; kb < num_kb; ++kb) {
    ptx::mbar_wait(&ring.full[rd], rd_phase);
    const uint32_t s = ptx::smem_u32(ring.base + rd * ring.stage_bytes);
    if (++rd == ring.stages) {
      rd = 0;
      rd_phase ^= 1;
    }
    const uint64_t da = ptx::make_smem_desc(s + a_off), db = ptx::make_smem_desc(s + b_off);
    const int ksteps = min(kChunkK, K - kb * kChunkK + 15) / 16;  // skip all-zero K tails
#pragma unroll 1
    for (int ks = 0; ks < ksteps; ++ks)
      ptx::Wgmma<N>::mma(acc, da + (uint64_t)(ks * 2), db + (uint64_t)(ks * 2), (kb | ks) ? 1u : 0u);
    ptx::wgmma_commit();
    if (kb > 0) {
      ptx::wgmma_wait<1>();
      ring.release();
    }
  }
  ptx::wgmma_wait<0>();
  ring.release();
  ptx::reg_fence(acc);
}

// The split-bf16 form, x = hi + lo: D (+)= A_hi.B_hi + A_lo.B_hi + A_hi.B_lo (+ A_lo.B_lo when kLoLo), in that order
// per 16-wide K step, over a whole 64-wide chunk.
template <int N, bool kLoLo>
__device__ __forceinline__ void mma_chunk_split(float (&acc)[N / 2], uint32_t a_hi, uint32_t a_lo, uint32_t b_hi,
                                                uint32_t b_lo, int kb) {
  const uint64_t d_ahi = ptx::make_smem_desc(a_hi), d_alo = ptx::make_smem_desc(a_lo);
  const uint64_t d_bhi = ptx::make_smem_desc(b_hi), d_blo = ptx::make_smem_desc(b_lo);
  ptx::wgmma_fence();
#pragma unroll
  for (int ks = 0; ks < kChunkK / 16; ++ks) {
    const uint64_t o = (uint64_t)(ks * 2);  // 16 bf16 = 32 bytes along K inside the swizzle atom
    ptx::Wgmma<N>::mma(acc, d_ahi + o, d_bhi + o, (kb | ks) ? 1u : 0u);
    ptx::Wgmma<N>::mma(acc, d_alo + o, d_bhi + o, 1u);
    ptx::Wgmma<N>::mma(acc, d_ahi + o, d_blo + o, 1u);
    if constexpr (kLoLo) ptx::Wgmma<N>::mma(acc, d_alo + o, d_blo + o, 1u);
  }
  ptx::wgmma_commit();
  ptx::wgmma_wait_all();
  ptx::reg_fence(acc);
}

}  // namespace pipe
}  // namespace am
