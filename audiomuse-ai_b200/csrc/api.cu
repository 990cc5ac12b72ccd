// Library lifecycle, error reporting, launch accounting (C ABI: include/audiomuse_b200.h).
#include "common.cuh"

#include <map>
#include <mutex>

namespace am {

static thread_local std::string t_error;
std::atomic<uint64_t> g_launches{0};
static std::mutex g_init_mu;
static std::atomic<int> g_inited{0};
static int g_sms = 0, g_cc = 0;

void set_error(const char* fmt, ...) {
  char buf[1024];
  va_list ap;
  va_start(ap, fmt);
  vsnprintf(buf, sizeof buf, fmt, ap);
  va_end(ap);
  t_error = buf;
}

int cuda_fail(cudaError_t e, const char* what, const char* file, int line) {
  const bool oom = (e == cudaErrorMemoryAllocation);
  // "out of memory" keeps tasks/memory_utils.py's OOM detection (string match) working
  set_error("%s%s failed: %s (%s:%d)", oom ? "out of memory: " : "", what, cudaGetErrorString(e), file,
            line);
  cudaGetLastError();  // clear the sticky-free error state
  return oom ? AM_ERR_OOM : AM_ERR_CUDA;
}

// ---------------------------------------------------------------- launch profiler
std::atomic<int> g_prof_on{0};
struct ProfRec {
  const char* name;
  cudaEvent_t e0, e1;
};
static std::mutex g_prof_mu;
static std::vector<ProfRec> g_prof;

void prof_mark(const char* name, cudaStream_t st, int end) {
  std::lock_guard<std::mutex> lk(g_prof_mu);
  if (!end) {
    ProfRec r{name, nullptr, nullptr};
    if (cudaEventCreate(&r.e0) != cudaSuccess || cudaEventCreate(&r.e1) != cudaSuccess) return;
    cudaEventRecord(r.e0, st);
    g_prof.push_back(r);
  } else if (!g_prof.empty() && g_prof.back().name == name) {
    cudaEventRecord(g_prof.back().e1, st);
  }
}

int ensure_init() {
  if (g_inited.load(std::memory_order_acquire)) return AM_OK;
  return am_init(-1);
}
int sm_count() { return g_sms; }
int device_cc() { return g_cc; }

}  // namespace am

using namespace am;

extern "C" int am_init(int device_ordinal) {
  std::lock_guard<std::mutex> lk(g_init_mu);
  int n = 0;
  cudaError_t e = cudaGetDeviceCount(&n);
  if (e != cudaSuccess || n == 0) {
    set_error("no CUDA device visible (%s); libaudiomuse_b200 has no CPU fallback",
              e == cudaSuccess ? "device count 0" : cudaGetErrorString(e));
    cudaGetLastError();
    return AM_ERR_NO_DEVICE;
  }
  if (device_ordinal >= 0) {
    AM_CHECK(device_ordinal < n, "am_init: device %d out of range (%d visible)", device_ordinal, n);
    AM_CUDA(cudaSetDevice(device_ordinal));
  }
  int dev = 0;
  AM_CUDA(cudaGetDevice(&dev));
  cudaDeviceProp p;
  AM_CUDA(cudaGetDeviceProperties(&p, dev));
  if (p.major != 9 || p.minor != 0) {
    set_error("device %d is sm_%d%d; this library is built for sm_90a (H100) only", dev, p.major, p.minor);
    return AM_ERR_NO_DEVICE;
  }
  g_sms = p.multiProcessorCount;
  g_cc = p.major * 10 + p.minor;
  AM_CUDA(cudaFree(0));
  {  // keep stream-ordered scratch cached in the default pool instead of returning it at every sync
    cudaMemPool_t pool;
    if (cudaDeviceGetDefaultMemPool(&pool, dev) == cudaSuccess) {
      uint64_t thr = UINT64_MAX;
      cudaMemPoolSetAttribute(pool, cudaMemPoolAttrReleaseThreshold, &thr);
    }
    cudaGetLastError();
  }
  g_inited.store(1, std::memory_order_release);
  return AM_OK;
}

extern "C" void am_shutdown(void) {
  std::lock_guard<std::mutex> lk(g_init_mu);
  if (g_inited.load()) cudaDeviceSynchronize();
  g_inited.store(0);
}

extern "C" const char* am_last_error(void) { return t_error.c_str(); }
extern "C" int am_version(void) { return 100; }
extern "C" uint64_t am_launch_count(void) { return g_launches.load(std::memory_order_relaxed); }

// ---------------------------------------------------------------- profiler C ABI
extern "C" void am_profile_enable(int on) {
  g_prof_on.store(on ? 1 : 0, std::memory_order_relaxed);
}

// Writes a JSON object {"kernel name": {"ms": total_device_ms, "count": launches}, ...} for every
// launch recorded since the last report, then clears the records.  Returns the number of bytes
// needed (excluding the NUL); call with cap = 0 to size the buffer.  Synchronises the device.
extern "C" int am_profile_report(char* buf, int cap) {
  static thread_local std::string cached;
  if (buf == nullptr || cap <= 0 || cached.empty()) {
    cudaDeviceSynchronize();
    std::lock_guard<std::mutex> lk(g_prof_mu);
    std::map<std::string, std::pair<double, long>> agg;
    for (auto& r : g_prof) {
      float ms = 0.f;
      if (cudaEventElapsedTime(&ms, r.e0, r.e1) == cudaSuccess) {
        auto& a = agg[r.name];
        a.first += ms;
        a.second += 1;
      }
      cudaEventDestroy(r.e0);
      cudaEventDestroy(r.e1);
    }
    cudaGetLastError();
    g_prof.clear();
    cached = "{";
    bool first = true;
    for (auto& kv : agg) {
      char tmp[512];
      snprintf(tmp, sizeof tmp, "%s\"%s\": {\"ms\": %.6f, \"count\": %ld}", first ? "" : ", ", kv.first.c_str(),
               kv.second.first, kv.second.second);
      cached += tmp;
      first = false;
    }
    cached += "}";
  }
  const int need = (int)cached.size();
  if (buf != nullptr && cap > need) {
    std::memcpy(buf, cached.c_str(), need + 1);
    cached.clear();
  }
  return need;
}
