// lm_buffer.h -- owners of the library's device memory, pinned host memory, streams and events.
//
// An owner that holds nothing makes no CUDA call, so host-only handles and machines without a device never touch the
// runtime.  The owners never zero, copy or synchronise: growth policy, memsets and copies stay with the caller, and so
// does the choice of where a free may happen (a cudaFree waits for the whole device).
#pragma once
#include <cuda_runtime.h>
#include <stddef.h>

#include <algorithm>
#include <type_traits>
#include <utility>
#include <vector>

struct DeviceAlloc {
  static cudaError_t alloc(void** p, size_t bytes) { return cudaMalloc(p, bytes); }
  static void release(void* p) { cudaFree(p); }
};
struct PinnedAlloc {
  static cudaError_t alloc(void** p, size_t bytes) { return cudaMallocHost(p, bytes); }
  static void release(void* p) { cudaFreeHost(p); }
};

// Owning, move-only array of size() elements of T.  Its size changes only once an allocation has succeeded: after a
// failed one it holds nothing and its size is 0.
template <typename T, typename A>
class CudaArray {
 public:
  CudaArray() = default;
  CudaArray(const CudaArray&) = delete;
  CudaArray& operator=(const CudaArray&) = delete;
  CudaArray(CudaArray&& o) noexcept : p_(o.p_), n_(o.n_) { o.p_ = nullptr; o.n_ = 0; }
  CudaArray& operator=(CudaArray&& o) noexcept {
    if (this != &o) {
      reset();
      std::swap(p_, o.p_);
      std::swap(n_, o.n_);
    }
    return *this;
  }
  ~CudaArray() { reset(); }

  T* get() const { return p_; }
  // host access: pinned memory only (a device pointer must not be dereferenced on the host)
  T& operator[](size_t i) const {
    static_assert(std::is_same<A, PinnedAlloc>::value, "operator[] reads on the host: PinnedArray only");
    return p_[i];
  }
  size_t size() const { return n_; }
  bool empty() const { return n_ == 0; }

  // Exactly n elements: the old memory is freed first, then n elements are allocated (none for n = 0).
  cudaError_t assign(size_t n) {
    reset();
    if (n == 0) return cudaSuccess;
    void* p = nullptr;
    const cudaError_t e = A::alloc(&p, n * sizeof(T));
    if (e != cudaSuccess) return e;
    p_ = static_cast<T*>(p);
    n_ = n;
    return cudaSuccess;
  }
  // Grow only: n <= size() keeps the memory, a larger n is assign(n).
  cudaError_t reserve(size_t n) { return n <= n_ ? cudaSuccess : assign(n); }
  void reset() {
    if (p_) A::release(p_);
    p_ = nullptr;
    n_ = 0;
  }

 private:
  T* p_ = nullptr;
  size_t n_ = 0;
};

template <typename T>
using DeviceArray = CudaArray<T, DeviceAlloc>;
template <typename T>
using PinnedArray = CudaArray<T, PinnedAlloc>;

// a = exactly max(v.size(), min_n) elements, then v copied to its front on stream st (not waited for).
template <typename T>
cudaError_t upload(DeviceArray<T>& a, const std::vector<T>& v, cudaStream_t st, size_t min_n = 0) {
  cudaError_t e = a.assign(std::max(v.size(), min_n));
  if (e == cudaSuccess && !v.empty()) e = cudaMemcpyAsync(a.get(), v.data(), v.size() * sizeof(T), cudaMemcpyHostToDevice, st);
  return e;
}

struct StreamKind {
  using handle = cudaStream_t;
  static cudaError_t create(cudaStream_t* h, unsigned flags) { return cudaStreamCreateWithFlags(h, flags); }
  static void destroy(cudaStream_t h) { cudaStreamDestroy(h); }
};
struct EventKind {
  using handle = cudaEvent_t;
  static cudaError_t create(cudaEvent_t* h, unsigned flags) { return cudaEventCreateWithFlags(h, flags); }
  static void destroy(cudaEvent_t h) { cudaEventDestroy(h); }
};

// Owning, move-only stream or event: created with its flags by create(), destroyed with its owner.  A failed create
// leaves it empty.
template <typename K>
class CudaHandle {
 public:
  using handle = typename K::handle;
  CudaHandle() = default;
  CudaHandle(const CudaHandle&) = delete;
  CudaHandle& operator=(const CudaHandle&) = delete;
  CudaHandle(CudaHandle&& o) noexcept : h_(o.h_) { o.h_ = nullptr; }
  CudaHandle& operator=(CudaHandle&& o) noexcept {
    if (this != &o) {
      reset();
      std::swap(h_, o.h_);
    }
    return *this;
  }
  ~CudaHandle() { reset(); }

  handle get() const { return h_; }
  cudaError_t create(unsigned flags) {
    reset();
    handle h = nullptr;
    const cudaError_t e = K::create(&h, flags);
    if (e == cudaSuccess) h_ = h;
    return e;
  }
  void reset() {
    if (h_) K::destroy(h_);
    h_ = nullptr;
  }

 private:
  handle h_ = nullptr;
};

using Stream = CudaHandle<StreamKind>;
using Event = CudaHandle<EventKind>;
