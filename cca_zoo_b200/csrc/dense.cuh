// Small dense glue on CUDA cores (exact fp32 / fp64 FMA): GEMM with optional transposes, whitening
// scale of eigenvector rows, Frobenius norm.  None of these is on the roofline-critical path; they
// connect K1 (moments) to K3/K4 (Jacobi) at sizes D <= a few thousand.
#pragma once
#include "common.cuh"

namespace ccab {

// Batched GEMM descriptor shared by the FMA kernel (any T) and the tcgen05 kernel (float, see tgemm.cuh):
// matrix (b, b2) of the batch lives at X + b * strideX + b2 * strideX2.
template <typename T>
struct GemmArgs {
  int transa = 0, transb = 0;
  int m = 0, n = 0, k = 0;
  T alpha = T(1), beta = T(0);
  const T* A = nullptr;
  int64_t lda = 0, strideA = 0, strideA2 = 0;
  const T* B = nullptr;
  int64_t ldb = 0, strideB = 0, strideB2 = 0;
  T* C = nullptr;                 // may be NULL when only Ct is wanted
  int64_t ldc = 0, strideC = 0, strideC2 = 0;
  T* Ct = nullptr;                // optional transposed copy (n x m, row-major)
  int64_t ldct = 0, strideCt = 0, strideCt2 = 0;
  int batch = 1, batch2 = 1;
  int lower_only = 0;             // skip output tiles strictly above the diagonal
  void* splitk_ws = nullptr;      // optional scratch: thin products split their reduction over CTAs / a batch and
  size_t splitk_ws_bytes = 0;     // add the partial tiles in a fixed order (deterministic); unused when too small
};
template <typename T>
int gemm_fma(const GemmArgs<T>& g, cudaStream_t stream);   // exact FMA tiles on the CUDA cores
template <typename T>
int xgemm(const GemmArgs<T>& g, cudaStream_t stream);      // float: tcgen05 when TMA-addressable, else gemm_fma

// Whitening factors from an eigendecomposition (covariance form of svd_whiten,
// cca_zoo/_utils/_linalg.py:30-38):  for eigenpair j (descending, rows of Vt)
//   keep_j = lam_j > rank_tol * lam_0  and  j < max_rank
//   g_j    = keep_j ? 1 / sqrt(((1 - c) * max(lam_j, lam_floor) + c + floor_add) * scale) : 0
//   Wt[j,:] = g_j * Vt[j,:]
// and *rank_out = #kept.  `floor_dev` (may be null) points at a device scalar added to floor_add.
template <typename T>
int whiten_rows(int d, const T* lam, const T* Vt, int64_t ldv, double c, double floor_add, const T* floor_dev,
                double scale, double rank_tol, int max_rank, double lam_floor, T* Wt, int64_t ldw, T* g_out,
                int* rank_out, cudaStream_t stream);

// B[i,j] = A[i,j] * (r ? r[i] : 1) * (c ? c[j] : 1), optionally c_pow/r_pow applied first:
// factor = pow(value, pow) with pow in {1, -1, -0.5} encoded as 0, 1, 2.   (m x n row-major, in place ok)
template <typename T>
int scale_rows_cols(int m, int n, const T* A, int64_t lda, const T* r, int r_pow, const T* c, int c_pow, T* B,
                    int64_t ldb, cudaStream_t stream);

// A[:, j] -= mean_i A[i, j]   (m x n row-major, in place)
template <typename T>
int center_columns(int m, int n, T* A, int64_t lda, cudaStream_t stream);

// A[i, :] = (A[i, :] - r) * s[0]   (m x n row-major, in place; r: device T[n], s: device T[1])
template <typename T>
int row_sub_scale(int64_t m, int n, T* A, int64_t lda, const T* r, const T* s, cudaStream_t stream);

// out[0] = ||A||_F (m x n, row-major)
template <typename T>
int frobenius_norm(int m, int n, const T* A, int64_t lda, T* out, cudaStream_t stream);

}  // namespace ccab
