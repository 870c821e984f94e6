// CCAR3 (CCA by reduced-rank regression): the row-sparse ADMM on the block moments and the fourth-power row sum of
// the Ledoit-Wolf shrinkage (see ccab_ccar3_admm / ccab_row_norm4_sum in include/ccab200.h).
#pragma once

#include <cuda_runtime.h>
#include <stddef.h>
#include <stdint.h>

namespace ccab {

constexpr int kCcar3MaxQ = 512;        // widest Y: a CTA keeps 8 x 8 fragments of every output row in registers
constexpr int kCcar3MaxP = 16384;      // widest X: M = (Sx + (rho + eps) I)^-1 is p x p float64 (2 GB)
constexpr int kCcar3MaxGrid = 1024;    // partial-sum slots of the residual reduction
constexpr int kCcar3InfoDoubles = 4;   // iterations, primal, dual, stop flag

size_t ccar3_admm_workspace_bytes(int p, int q);
int ccar3_admm(int p, int q, const double* M, int64_t ldm, const double* B0, int64_t ldb, double kappa, double rho,
               double tol, int max_iter, double* Z, int64_t ldz, double* U, int64_t ldu, double* info, void* ws,
               size_t ws_bytes, cudaStream_t stream);

size_t row_norm4_sum_workspace_bytes(int64_t n);
template <typename T>
int row_norm4_sum(int64_t n, int d, const T* Y, int64_t ldy, const double* mean, double* out, void* ws,
                  size_t ws_bytes, cudaStream_t stream);

}  // namespace ccab
