// KCCA: the pairwise kernel matrices of sklearn's PAIRWISE_KERNEL_FUNCTIONS (see ccab_pairwise_kernel in
// include/ccab200.h).
#pragma once

#include <cuda_runtime.h>
#include <stddef.h>
#include <stdint.h>

namespace ccab {

// metric ids: the CCAB_KERNEL_* constants of include/ccab200.h
enum KernelMetric : int {
  kKernelLinear = 0,
  kKernelPoly = 1,
  kKernelRbf = 2,
  kKernelSigmoid = 3,
  kKernelCosine = 4,
  kKernelLaplacian = 5,
  kKernelChi2 = 6,
  kKernelAdditiveChi2 = 7,
};

size_t pairwise_kernel_workspace_bytes(int metric, int64_t nx, int64_t ny);
template <typename T>
int pairwise_kernel(int metric, const T* X, int64_t nx, int64_t ldx, const T* Y, int64_t ny, int64_t ldy, int d,
                    double gamma, double degree, double coef0, double* K, int64_t ldk, void* ws, size_t ws_bytes,
                    cudaStream_t stream);

}  // namespace ccab
