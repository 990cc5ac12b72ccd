// The memory and stream of a host-pointer entry point call (host_call.cuh).
#include "host_call.cuh"

#include <algorithm>

namespace am {

int HostCall::thread_stream(cudaStream_t* st) {
  AM_TRY(ensure_init());
  static thread_local Stream s;  // one per calling thread (Flask gthread x4), so the entry points are re-entrant
  AM_TRY(s.create());
  *st = s.s;
  return AM_OK;
}

HostCall::~HostCall() {
  if (!dev_) return;
  if (mem_ == Memory::Pool) cudaFreeAsync(dev_, st_);
  else cudaFree(dev_);
}

int HostCall::start() {
  auto rank = [](const Part& p) { return p.dir != Device ? (int)p.dir : Device + (p.fill < 0 ? 256 : p.fill); };
  std::stable_sort(parts_.begin(), parts_.end(), [&](const Part& a, const Part& b) { return rank(a) < rank(b); });
  size_t off = 0;
  for (Part& p : parts_) {
    p.off = off;
    off += round_up(p.bytes, 256);
    if (p.dir == Up) back_begin_ = off;
    if (p.dir <= Both) up_end_ = off;
    if (p.dir <= Down) back_end_ = off;
  }
  if (off) {
    const bool pool = mem_ == Memory::Pool;
    const cudaError_t e = pool ? cudaMallocAsync((void**)&dev_, off, st_) : cudaMalloc((void**)&dev_, off);
    if (e != cudaSuccess) {
      dev_ = nullptr;
      return cuda_fail(e, pool ? "cudaMallocAsync" : "cudaMalloc", __FILE__, __LINE__);
    }
  }
  for (const Part& p : parts_) {
    char* ptr = dev_ + p.off;
    std::memcpy(p.slot, &ptr, sizeof ptr);
  }
  staged_ = back_end_ <= limit_;  // [up | both | down] starts at 0
  if (staged_) {
    static thread_local PinnedBuf<char> mirror;  // grows to the largest staged call of the thread
    AM_TRY(mirror.ensure(back_end_));
    host_ = mirror.p;
    for (const Part& p : parts_)
      if (p.up_bytes) std::memcpy(host_ + p.off, p.src, p.up_bytes);
    if (up_end_) AM_CUDA(cudaMemcpyAsync(dev_, host_, up_end_, cudaMemcpyHostToDevice, st_));
  } else {
    for (const Part& p : parts_)
      if (p.up_bytes) AM_CUDA(cudaMemcpyAsync(dev_ + p.off, p.src, p.up_bytes, cudaMemcpyHostToDevice, st_));
  }
  for (size_t i = 0, j; i < parts_.size(); i = j) {  // one memset per run of adjacent parts with the same fill byte
    const Part& p = parts_[i];
    for (j = i + 1; j < parts_.size() && p.fill >= 0 && parts_[j].fill == p.fill;) ++j;
    const size_t end = parts_[j - 1].off + round_up(parts_[j - 1].bytes, 256);
    if (p.fill >= 0 && end > p.off) AM_CUDA(cudaMemsetAsync(dev_ + p.off, p.fill, end - p.off, st_));
  }
  return AM_OK;
}

int HostCall::finish() {
  if (staged_ && back_end_ > back_begin_)
    AM_CUDA(cudaMemcpyAsync(host_ + back_begin_, dev_ + back_begin_, back_end_ - back_begin_, cudaMemcpyDeviceToHost,
                            st_));
  for (const Part& p : parts_)
    if (!staged_ && p.dst && p.bytes) AM_CUDA(cudaMemcpyAsync(p.dst, dev_ + p.off, p.bytes, cudaMemcpyDeviceToHost, st_));
  AM_CUDA(cudaStreamSynchronize(st_));
  for (const Part& p : parts_)
    if (staged_ && p.dst && p.bytes) std::memcpy(p.dst, host_ + p.off, p.bytes);
  return AM_OK;
}

}  // namespace am
