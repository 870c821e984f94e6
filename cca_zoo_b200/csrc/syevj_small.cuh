// Single-CTA two-sided Jacobi eigensolver for small symmetric matrices (see syevj_small.cu).
#pragma once
#include "common.cuh"

namespace ccab {

template <typename T>
bool syevj_small_supported(int n);   // n <= 128 (float) / 104 (double): two copies of H and of a column slice of V must fit one CTA's shared memory

// For each of `batch` symmetric matrices A_b = A + b * strideA (n x n, lda): eigenvalues descending into
// evals + b * strideE, eigenvectors as ROWS of evt + b * strideV (n x n, ldv).  info_dev[b] (device, may be NULL) =
// sweeps used, negated when the off-diagonal mass did not reach the tolerance.  One launch, no host sync.
template <typename T>
int syevj_small(int n, int batch, const T* A, int64_t lda, int64_t strideA, T* evals, int64_t strideE, T* evt,
                int64_t ldv, int64_t strideV, int* info_dev, cudaStream_t stream);

}  // namespace ccab
