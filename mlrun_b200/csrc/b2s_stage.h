// b2s_stage.h -- host-side staging that the serving runtime (b2s_runtime.cu), the point-in-time join (b2s_pit.cu) and the
// windowed aggregations (b2s_agg.cu) share: one device block per call for its inputs, outputs and scratch, device and
// pinned arrays and CUDA events that free themselves, and the call's launch count.  Host code only.  Its names live in the
// including unit's anonymous namespace, so none is exported.
#pragma once
#include <cuda_runtime.h>

#include <cstddef>
#include <cstdint>
#include <memory>
#include <vector>

#include "../../include/b200serve.h"
#include "b2s_internal.h"

namespace {

// The kernel launches of one call: what it reports in b2s_stats::kernels, added to the library's count as they are made.
struct Launches {
  int n = 0;
  void add(int k) {
    n += k;
    b2s_int_count_launches(k);
  }
};

// Synchronises a stream when it leaves scope.  Destructors run in reverse order of declaration: declared before a
// DeviceBlock it waits for the block's free, declared after it it waits before the free.
struct SyncOnExit {
  cudaStream_t st;
  ~SyncOnExit() { cudaStreamSynchronize(st); }
};

// B2S_ERR_INVALID unless p is device memory of the library's device, aligned to `align` bytes
inline int check_on_device(const void* p, int align, const char* what, int i) {
  if (misaligned(p, align)) return b2s_int_fail(B2S_ERR_INVALID, "%s %d: not %d-byte aligned", what, i, align);
  int32_t dev = -1;
  if (int rc = b2s_pointer_device(p, &dev)) return rc;
  if (dev != b2s_int_device())
    return b2s_int_fail(B2S_ERR_INVALID, "%s %d: %s, not memory of the library's device %d", what, i, dev < 0 ? "host memory" : "another device's memory",
                        b2s_int_device());
  return B2S_OK;
}

// CUDA events, destroyed when the array leaves scope.
class Events {
 public:
  Events() = default;
  Events(const Events&) = delete;
  Events& operator=(const Events&) = delete;
  ~Events() {
    for (cudaEvent_t e : ev_) cudaEventDestroy(e);
  }
  int create(int n, unsigned flags = cudaEventDefault) {
    for (int i = 0; i < n; ++i) {
      cudaEvent_t e = nullptr;
      B2S_CUDA_TRY(cudaEventCreateWithFlags(&e, flags));
      ev_.push_back(e);
    }
    return B2S_OK;
  }
  cudaEvent_t operator[](size_t i) const { return ev_[i]; }
  const cudaEvent_t* data() const { return ev_.data(); }
  size_t size() const { return ev_.size(); }

 private:
  std::vector<cudaEvent_t> ev_;
};

// Device and pinned host arrays, freed when their owner goes.  allocate() frees the old array before it makes the new one:
// a failed allocation leaves the owner empty, never dangling.
struct CudaFree {
  void operator()(void* p) const { cudaFree(p); }
};
struct CudaFreeHost {
  void operator()(void* p) const { cudaFreeHost(p); }
};
template <class T>
using DeviceArray = std::unique_ptr<T[], CudaFree>;
template <class T>
using PinnedArray = std::unique_ptr<T[], CudaFreeHost>;

template <class T>
int allocate(DeviceArray<T>& a, size_t bytes) {
  a.reset();
  void* p = nullptr;
  B2S_CUDA_TRY(cudaMalloc(&p, bytes));
  a.reset(static_cast<T*>(p));
  return B2S_OK;
}
template <class T>
int allocate(PinnedArray<T>& a, size_t bytes) {
  a.reset();
  void* p = nullptr;
  B2S_CUDA_TRY(cudaMallocHost(&p, bytes));
  a.reset(static_cast<T*>(p));
  return B2S_OK;
}

// Every device array of one call in a single cudaMallocAsync, each region 256-byte aligned.  Regions are laid out first,
// each with the pointer that is to address it; alloc() makes the block and sets those pointers.  An input is uploaded by
// upload(); an output of n elements is copied back to its destination by download() for a range of rows.  The block is
// freed on its stream when it leaves scope: a caller that copies back on another stream synchronises that one first.
class DeviceBlock {
 public:
  struct Out {
    void* dst;    // where the rows go (host memory for download(); any memory for a caller that moves them itself)
    size_t off;   // the region's offset in the block
    size_t elem;  // bytes per row
  };

  explicit DeviceBlock(cudaStream_t st) : st_(st) {}
  DeviceBlock(const DeviceBlock&) = delete;
  DeviceBlock& operator=(const DeviceBlock&) = delete;
  ~DeviceBlock() {
    if (base_) cudaFreeAsync(base_, st_);
  }

  template <class T>
  size_t scratch(T*& dev, size_t bytes) {
    const size_t off = total_;
    total_ += (bytes + 255) / 256 * 256;
    binds_.push_back({&dev, off, [](void* p, char* at) { *static_cast<T**>(p) = static_cast<T*>(static_cast<void*>(at)); }});
    return off;
  }
  template <class T>
  void input(T*& dev, const void* src, size_t bytes) {
    ins_.push_back({src, scratch(dev, bytes), bytes});
  }
  template <class T>
  void output(T*& dev, void* dst, size_t elem, int64_t n) {
    outs_.push_back({dst, scratch(dev, (size_t)n * elem), elem});
  }

  int alloc() {
    B2S_CUDA_TRY(cudaMallocAsync(&base_, total_, st_));
    for (const Bind& b : binds_) b.set(b.ptr, base_ + b.off);
    return B2S_OK;
  }
  int upload() const {
    for (const In& i : ins_) B2S_CUDA_TRY(cudaMemcpyAsync(base_ + i.off, i.src, i.bytes, cudaMemcpyHostToDevice, st_));
    return B2S_OK;
  }
  // rows [q0, q1) of every output, on stream st
  int download(int64_t q0, int64_t q1, cudaStream_t st) const {
    for (const Out& o : outs_)
      B2S_CUDA_TRY(cudaMemcpyAsync(static_cast<char*>(o.dst) + q0 * o.elem, base_ + o.off + q0 * o.elem, (size_t)(q1 - q0) * o.elem,
                                   cudaMemcpyDeviceToHost, st));
    return B2S_OK;
  }
  const std::vector<Out>& outputs() const { return outs_; }
  void* at(size_t off) const { return base_ + off; }

 private:
  struct In {
    const void* src;
    size_t off, bytes;
  };
  struct Bind {  // *ptr (a T*) = the region at off
    void* ptr;
    size_t off;
    void (*set)(void* ptr, char* at);
  };
  cudaStream_t st_;
  char* base_ = nullptr;
  size_t total_ = 0;
  std::vector<In> ins_;
  std::vector<Out> outs_;
  std::vector<Bind> binds_;
};

}  // namespace
