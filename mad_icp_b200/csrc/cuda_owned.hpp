// cuda_owned.hpp -- move-only owners of the CUDA resources the library holds: device and pinned buffers, events, streams
// and executable graphs.  An owner releases its handle when it is destroyed or given another one.  Allocation stays the
// plain CUDA call, which returns a cudaError_t (CK) and writes the new handle through put().
#pragma once
#include <cuda_runtime.h>

#include <utility>

namespace madicp {

template <class H, auto Release>
class Owned {
 public:
  Owned() = default;
  Owned(Owned&& o) noexcept : h_(std::exchange(o.h_, H{})) {}
  Owned& operator=(Owned&& o) noexcept {
    if (this != &o) {
      reset();
      h_ = std::exchange(o.h_, H{});
    }
    return *this;
  }
  ~Owned() { reset(); }

  void reset() {
    if (h_) Release(h_);
    h_ = H{};
  }
  // releases the handle held, if any, and returns where an allocation or creation call writes the new one
  H* put() {
    reset();
    return &h_;
  }
  H get() const { return h_; }
  operator H() const { return h_; }
  H operator->() const { return h_; }

 private:
  H h_{};
};

template <class T>
using DevPtr = Owned<T*, cudaFree>;  // cudaMalloc
template <class T>
using HostPtr = Owned<T*, cudaFreeHost>;  // cudaMallocHost / cudaHostAlloc
using Event = Owned<cudaEvent_t, cudaEventDestroy>;
using Stream = Owned<cudaStream_t, cudaStreamDestroy>;
using GraphExec = Owned<cudaGraphExec_t, cudaGraphExecDestroy>;

}  // namespace madicp
