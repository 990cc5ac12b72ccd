// Shared host/device helpers for libaudiomuse_b200.so (sm_90a only).
#pragma once

#include <cuda_runtime.h>
#include <cuda_bf16.h>

#include <atomic>
#include <cstdarg>
#include <cstdint>
#include <cstdio>
#include <cstring>
#include <string>
#include <vector>

#include "../../include/audiomuse_b200.h"

namespace am {

// ---------------------------------------------------------------- error plumbing
void set_error(const char* fmt, ...);
int cuda_fail(cudaError_t e, const char* what, const char* file, int line);
extern std::atomic<uint64_t> g_launches;

#define AM_CUDA(expr)                                                   \
  do {                                                                  \
    cudaError_t _e = (expr);                                            \
    if (_e != cudaSuccess) return ::am::cuda_fail(_e, #expr, __FILE__, __LINE__); \
  } while (0)

#define AM_CHECK(cond, ...)              \
  do {                                   \
    if (!(cond)) {                       \
      ::am::set_error(__VA_ARGS__);      \
      return AM_ERR_INVALID;             \
    }                                    \
  } while (0)

#define AM_TRY(expr)            \
  do {                          \
    int _s = (expr);            \
    if (_s != AM_OK) return _s; \
  } while (0)

// Optional per-launch CUDA-event timing (am_profile_enable): bench.py reads the per-kernel
// device time of the timed region from it.  Disabled: one relaxed atomic load per launch.
extern std::atomic<int> g_prof_on;
void prof_mark(const char* name, cudaStream_t st, int end);

// every kernel launch goes through this so bench.py can report gpu_launches
#define AM_LAUNCH(kernel, grid, block, smem, stream, ...)                 \
  do {                                                                    \
    const bool _prof = ::am::g_prof_on.load(std::memory_order_relaxed) != 0; \
    if (_prof) ::am::prof_mark(#kernel, (stream), 0);                     \
    kernel<<<(grid), (block), (smem), (stream)>>>(__VA_ARGS__);           \
    if (_prof) ::am::prof_mark(#kernel, (stream), 1);                     \
    ::am::g_launches.fetch_add(1, std::memory_order_relaxed);             \
    cudaError_t _le = cudaGetLastError();                                 \
    if (_le != cudaSuccess) return ::am::cuda_fail(_le, #kernel, __FILE__, __LINE__); \
  } while (0)

int ensure_init();          // lazy context creation; AM_OK or error
int mel_plan_frames(const am_mel_plan* plan, int n_samples);  // mel.cu: frames T, or AM_ERR_INVALID (too short)
int sm_count();             // SMs of the active device
int device_cc();            // major*10+minor

// Lets kKernel launch with up to `bytes` of dynamic shared memory.  The attribute is set by the first call for each
// kernel (the static's initialisation is thread safe, so concurrent first launches set it once and all wait for it);
// every call passes that kernel's same constant limit.
template <auto kKernel>
int allow_dynamic_smem(size_t bytes) {
  static const cudaError_t e = cudaFuncSetAttribute(kKernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)bytes);
  return e == cudaSuccess ? AM_OK : cuda_fail(e, "cudaFuncSetAttribute(MaxDynamicSharedMemorySize)", __FILE__, __LINE__);
}

// ---------------------------------------------------------------- RAII device / pinned buffers
template <typename T>
struct DevBuf {
  T* p = nullptr;
  size_t n = 0;
  DevBuf() = default;
  DevBuf(const DevBuf&) = delete;
  DevBuf& operator=(const DevBuf&) = delete;
  ~DevBuf() { release(); }
  void release() {
    if (p) cudaFree(p);
    p = nullptr;
    n = 0;
  }
  int alloc(size_t count) {
    release();
    if (count == 0) return AM_OK;
    cudaError_t e = cudaMalloc(&p, count * sizeof(T));
    if (e != cudaSuccess) {
      p = nullptr;
      return cuda_fail(e, "cudaMalloc", __FILE__, __LINE__);
    }
    n = count;
    return AM_OK;
  }
  int ensure(size_t count) { return count <= n ? AM_OK : alloc(count); }
};

template <typename T>
struct PinnedBuf {
  T* p = nullptr;
  size_t n = 0;
  PinnedBuf() = default;
  PinnedBuf(const PinnedBuf&) = delete;
  PinnedBuf& operator=(const PinnedBuf&) = delete;
  ~PinnedBuf() {
    if (p) cudaFreeHost(p);
  }
  int ensure(size_t count) {
    if (count <= n) return AM_OK;
    if (p) cudaFreeHost(p);
    p = nullptr;
    n = 0;
    cudaError_t e = cudaMallocHost(&p, count * sizeof(T));
    if (e != cudaSuccess) {
      p = nullptr;
      return cuda_fail(e, "cudaMallocHost", __FILE__, __LINE__);
    }
    n = count;
    return AM_OK;
  }
};

struct Stream {
  cudaStream_t s = nullptr;
  ~Stream() {
    if (s) cudaStreamDestroy(s);
  }
  int create() {
    if (s) return AM_OK;
    cudaError_t e = cudaStreamCreateWithFlags(&s, cudaStreamNonBlocking);
    return e == cudaSuccess ? AM_OK : cuda_fail(e, "cudaStreamCreate", __FILE__, __LINE__);
  }
};

struct Event {
  cudaEvent_t e = nullptr;
  Event() = default;
  Event(const Event&) = delete;
  Event& operator=(const Event&) = delete;
  ~Event() {
    if (e) cudaEventDestroy(e);
  }
  int create(unsigned flags = cudaEventDefault) {
    if (e) return AM_OK;
    cudaError_t r = cudaEventCreateWithFlags(&e, flags);
    if (r == cudaSuccess) return AM_OK;
    e = nullptr;
    return cuda_fail(r, "cudaEventCreate", __FILE__, __LINE__);
  }
};

// ms += the time between two completed events recorded with timing
inline int add_elapsed_ms(float& ms, const Event& from, const Event& to) {
  float t = 0.f;
  cudaError_t r = cudaEventElapsedTime(&t, from.e, to.e);
  if (r != cudaSuccess) return cuda_fail(r, "cudaEventElapsedTime", __FILE__, __LINE__);
  ms += t;
  return AM_OK;
}

inline size_t round_up(size_t x, size_t m) { return (x + m - 1) / m * m; }
inline int ceil_div(int a, int b) { return (a + b - 1) / b; }
// blocks of 256 threads for a grid-stride kernel over `total_threads` items: at most 16 per SM
inline int grid_for(int64_t total_threads) {
  const int64_t blocks = (total_threads + 255) / 256;
  return (int)(blocks < 1 ? 1 : (blocks < (int64_t)sm_count() * 16 ? blocks : (int64_t)sm_count() * 16));
}

// ---------------------------------------------------------------- symmetrised k-NN graphs (spectral.cu)
// The k exact euclidean nearest rows of every row of host X f32[N, d] (knn.cu's index, ids ascending distance): X is
// uploaded into dX, which stays with the caller, and ids i64[N, k] and dist f32[N, k] are filled; all three are
// allocated here.  t0 and t1 are recorded on `st` around the index build and query.  Stream-ordered.
int knn_self_query(const float* X, int64_t N, int d, int k, cudaStream_t st, const Event& t0, const Event& t1,
                   DevBuf<float>& dX, DevBuf<int64_t>& ids, DevBuf<float>& dist);
// CSR of k-NN lists ids i64[N, k] (device; a row's own id and ids outside [0, N) are skipped), columns ascending per
// row.  memb == nullptr: the affinity 0.5 (C + C^T) into w32 (0.5 or 1) and dd = sqrt(row sums).  memb f64[N, k] (a
// value per list entry): the fuzzy union A + A^T - A o A^T into w64.  Allocates the outputs; synchronises.
int knn_csr_build(const int64_t* ids, const double* memb, int64_t N, int k, cudaStream_t st, DevBuf<int64_t>& indptr,
                  DevBuf<int32_t>& indices, DevBuf<float>* w32, DevBuf<double>* dd, DevBuf<double>* w64,
                  int64_t* nnz);
// exclusive scan of cnt i32[N] into off i64[N + 1] (off[N] = the total), stream-ordered
int csr_scan(const int* cnt, int64_t N, int64_t* off, cudaStream_t st);

// ---------------------------------------------------------------- device helpers
#ifdef __CUDACC__
__device__ __forceinline__ float warp_sum(float v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
  return v;
}
__device__ __forceinline__ double warp_sum(double v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
  return v;
}
__device__ __forceinline__ float relu6f(float v) { return fminf(fmaxf(v, 0.0f), 6.0f); }
#endif

}  // namespace am
