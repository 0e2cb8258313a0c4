// The few THC (pre-ATen CUDA runtime) names the reference's NMS extension (mmdet/ops/nms/src/nms_kernel.cu) uses,
// restated on the CUDA runtime so that its unmodified source compiles against a current torch.  Test
// infrastructure only: see oracle/ref_build.py.
#pragma once
#include <cuda_runtime.h>
#include <ATen/Context.h>
#include <c10/util/Exception.h>
#include <cstddef>

struct THCState {};

inline void* THCudaMalloc(THCState*, size_t size) {
  void* p = nullptr;
  const cudaError_t err = cudaMalloc(&p, size);
  TORCH_CHECK(err == cudaSuccess, "THCudaMalloc: ", cudaGetErrorString(err));
  return p;
}

inline void THCudaFree(THCState*, void* p) {
  const cudaError_t err = cudaFree(p);
  TORCH_CHECK(err == cudaSuccess, "THCudaFree: ", cudaGetErrorString(err));
}

#define THCudaCheck(expr)                                                           \
  do {                                                                              \
    const cudaError_t thc_err_ = (expr);                                            \
    TORCH_CHECK(thc_err_ == cudaSuccess, "CUDA error: ", cudaGetErrorString(thc_err_)); \
  } while (0)

// The extension asks `at::globalContext().lazyInitCUDA()` for its THCState; current torch has no such member.
// Everything that includes this header after ATen sees `at::globalContext()` resolve to a context whose
// lazyInitCUDA() returns the (stateless) THCState above.
namespace at {
struct RefThcContext {
  THCState* lazyInitCUDA() {
    static THCState state;
    return &state;
  }
};
inline RefThcContext& ref_thc_context() {
  static RefThcContext ctx;
  return ctx;
}
}  // namespace at
#define globalContext ref_thc_context
