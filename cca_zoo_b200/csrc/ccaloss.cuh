// Fused small-matrix stage of the deep-CCA objective (see ccaloss.cu).
#pragma once
#include "common.cuh"

namespace ccab {

// C: (d1+d2) x (d1+d2) block covariance of [z1 z2] (row-major).  Outputs (device): loss[1], G11 (d1 x d1),
// P (d1 x d2), G22 (d2 x d2), min_pivot[1] (smallest elimination pivot of S11 / S22 = squared Cholesky pivot).
template <typename T>
int ccaloss_small(const T* C, int64_t ldc, int d1, int d2, double eps, T* loss, T* G11, T* P, T* G22, T* min_pivot,
                  cudaStream_t stream);

// Widths <= 64, everything after the moment pass in ONE single-CTA launch: reads the moment buffer of ccab_moments
// (two views, each padded to one 128-column block) directly, forms S = cov + eps I, inverts S11 and S22 side by side
// (Gauss-Jordan in shared memory), P, loss, G11, G22.  saved = G11 | P | G22 | mean1 | mean2 (T), flags[0..1] = 1 when
// the smallest pivot of S11 / S22 is <= eps / 4, flags[2] = 1 when a moment is not finite.  n_dev (device, may be
// NULL): the sample count is read there instead of `n` (an all-reduced global batch), and saved gains N behind the means.
template <typename T>
int ccaloss_small_forward(const double* moments, int Dp, double n, int d1, int d2, double eps, T* loss, T* saved,
                          int* flags, cudaStream_t stream, const double* n_dev = nullptr);

// g1 = 2/(n-1) center(z1 G11 - z2 P^T) go, g2 = 2/(n-1) center(z2 G22 - z1 P) go in ONE launch (64 rows per CTA); the
// centring is algebraic: the column means of the products follow from the saved means of z1 / z2.  global: the n rows
// are one shard of a global batch whose means and count N (saved[.. + d1 + d2]) the forward saved; 2/(N-1) scales.
template <typename T>
int ccaloss_small_backward(int d1, int d2, const T* z1, int64_t ld1, const T* z2, int64_t ld2, int64_t n,
                           const T* saved, const T* grad_out, T* g1, int64_t ldg1, T* g2, int64_t ldg2,
                           cudaStream_t stream, bool global = false);

}  // namespace ccab
