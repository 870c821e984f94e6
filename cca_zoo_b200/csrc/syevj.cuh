// One-sided block Jacobi eigensolver / SVD (kernels K3/K4 of DESIGN.md).
#pragma once
#include "common.cuh"

namespace ccab {

template <typename T>
struct JacobiArgs {
  const T* in;              // input matrix (batched)
  int64_t ld_in;            // leading dimension of the input
  int64_t batch_stride_in;  // elements between consecutive matrices
  int colmajor_in;          // 1: in[j*ld + i] is element (i,j); 0: in[i*ld + j]
  int m, n, batch;          // rows, columns (vectors rotated), number of matrices
  int svd_mode;             // 0: symmetric eigenproblem (m == n), 1: singular value decomposition
  double shift;             // symmetric mode: solve A + shift*I (make it PSD), values are un-shifted
  double tol;               // <=0: 4*eps*sqrt(m)
  int max_sweeps;           // <=0: default
  T* out_vals;              // [batch][n] descending (eigenvalues / singular values), may be null
  int64_t vals_stride;
  T* out_right;             // [batch][n][ld_right]: row j = j-th right vector (eigenvector), may be null
  int64_t ld_right, right_stride;
  T* out_left;              // SVD mode: [batch][n][ld_left]: row j = j-th left vector (length m), may be null
  int64_t ld_left, left_stride;
  int* info;                // host: info[0] = sweeps used
  float* final_offdiag;     // host: largest normalised off-diagonal Gram entry of the last sweep
};

template <typename T>
size_t jacobi_workspace_bytes(int m, int n, int batch);

// NOTE: synchronises `stream` once per sweep (the convergence flag is read on the host).
template <typename T>
int jacobi_solve(const JacobiArgs<T>& a, void* ws, size_t ws_bytes, cudaStream_t stream);

}  // namespace ccab
