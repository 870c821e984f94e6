// Rectangular fp32 GEMM on the Hopper tensor cores (wgmma TF32, 3xTF32 split formed while staging into
// shared memory) -- the solver-stage companion of the moment kernel K1.  See tgemm.cu.
#pragma once
#include "common.cuh"

namespace ccab {

struct TgemmArgs {
  int transa = 0, transb = 0;  // op(X) = X^T when set (row-major storage, like ccab_gemm)
  int m = 0, n = 0, k = 0;     // C (m x n) = alpha * op(A) (m x k) * op(B) (k x n) + beta * C
  float alpha = 1.f, beta = 0.f;
  const float* A = nullptr;
  int64_t lda = 0, strideA = 0;   // stride*: elements between consecutive matrices of the batch
  const float* B = nullptr;
  int64_t ldb = 0, strideB = 0;
  float* C = nullptr;             // may be NULL when only the transposed copy is wanted (beta must be 0)
  int64_t ldc = 0, strideC = 0;
  float* Ct = nullptr;            // optional: C^T (n x m, row-major, ldct) written as well
  int64_t ldct = 0, strideCt = 0;
  int batch = 1;
  int batch2 = 1;                 // optional second batch dimension (strides *2): matrix (b, b2) at X + b*stride + b2*stride2
  int64_t strideA2 = 0, strideB2 = 0, strideC2 = 0, strideCt2 = 0;
  int force_bn = 0;               // 0: heuristic; 64 / 128: column-tile width (128 makes an n <= 128 product safe in place)
  int lower_only = 0;             // skip 128 x BN tiles that lie strictly above the diagonal (SYRK-type updates)
};

// The staging loads need 16-byte aligned base pointers / leading dimensions / batch strides.  False -> use the FMA kernel.
bool tgemm_supported(const TgemmArgs& a);

// Asynchronous on `stream`.  Returns 0, <0 bad argument, >0 cudaError_t.
int tgemm(const TgemmArgs& a, cudaStream_t stream);

}  // namespace ccab
