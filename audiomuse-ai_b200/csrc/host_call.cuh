// The device memory of one host-pointer entry point call (host_call.cu).
#pragma once

#include <cstring>
#include <type_traits>
#include <vector>

#include "common.cuh"

namespace am {

// A host call whose transfers fit in 2 MiB stages them through pinned memory: one query of 256 runs at 1.37 M instead of
// 1.15 M queries/s.  Beyond that the copies into and out of the pinned mirror cost more than they save.
constexpr size_t kStageLimit = (size_t)2 << 20;

// The device memory of one host call, declared part by part, in one allocation laid out
// [up | both ways | down | device-only, same fill bytes together]: start() copies everything that goes up in one range
// and fills each run of same-byte parts with one memset, finish() copies everything that comes back in one range.
// Staged (what crosses the bus fits in stage_limit), both ranges travel through the calling thread's pinned mirror;
// otherwise each part is copied straight from or to the caller's arrays, so a large call pins nothing.  finish() copies
// a part with a host array there in full; a part whose returned length depends on the result has none and is read
// through mirror() / get() (staged calls only).  Device pointers are set by start() and live as long as the call.
//
// Pool: the block comes from the stream-ordered pool, with no device-wide synchronisation on allocation or free, for
// calls that run often on small inputs.  Owned: a plain cudaMalloc freed with the call, for calls whose scratch is too
// large to leave reserved in the pool (am_init keeps what the pool has reserved).
class HostCall {
 public:
  enum class Memory { Pool, Owned };
  static constexpr size_t kAlways = ~size_t(0);
  HostCall(cudaStream_t st, size_t stage_limit, Memory mem) : st_(st), limit_(stage_limit), mem_(mem) {}
  HostCall(const HostCall&) = delete;
  HostCall& operator=(const HostCall&) = delete;
  ~HostCall();

  template <class T>
  void up(T** dev, const std::remove_const_t<T>* src, size_t count) {
    parts_.push_back(Part{dev, Up, count * sizeof(T), count * sizeof(T), src, nullptr, -1});
  }
  // `count` elements on the device, the first n_up from src; all of them come back to dst unless it is null
  template <class T>
  void both(T** dev, const std::remove_const_t<T>* src, size_t n_up, size_t count, T* dst = nullptr) {
    parts_.push_back(Part{dev, Both, count * sizeof(T), n_up * sizeof(T), src, dst, -1});
  }
  // fill >= 0: start() sets every byte to it first, for elements the launches may leave unwritten
  template <class T>
  void down(T** dev, size_t count, T* dst = nullptr, int fill = -1) {
    parts_.push_back(Part{dev, Down, count * sizeof(T), 0, nullptr, dst, fill});
  }
  template <class T>
  void device(T** dev, size_t count, int fill = -1) {
    parts_.push_back(Part{dev, Device, count * sizeof(T), 0, nullptr, nullptr, fill});
  }

  int start();   // allocate, copy up, fill
  int finish();  // copy back, synchronise, copy the parts with a host array there
  template <class T>
  const T* mirror(const T* dev) const {
    return reinterpret_cast<const T*>(host_ + (reinterpret_cast<const char*>(dev) - dev_));
  }
  template <class T>
  void get(T* dst, const T* dev, size_t count) const {  // the first `count` elements of a part, from the mirror
    if (count) std::memcpy(dst, mirror(dev), count * sizeof(T));
  }

  // the calling thread's stream, shared by its host calls (each synchronises before it returns); initialises the
  // library on first use
  static int thread_stream(cudaStream_t* st);

 private:
  enum Dir { Up, Both, Down, Device };
  struct Part {
    void* slot;  // the caller's device pointer variable
    Dir dir;
    size_t bytes, up_bytes;
    const void* src;
    void* dst;
    int fill;
    size_t off = 0;
  };
  cudaStream_t st_;
  size_t limit_;
  Memory mem_;
  std::vector<Part> parts_;
  char* dev_ = nullptr;
  char* host_ = nullptr;
  size_t up_end_ = 0, back_begin_ = 0, back_end_ = 0;
  bool staged_ = false;
};

}  // namespace am
