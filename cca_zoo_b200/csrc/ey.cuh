// Eckart-Young gradient estimators (CCA_EY, PLS_EY, MCCA_EY): momentum steps on the EY loss (see ccab_ey_fit in
// include/ccab200.h).
#pragma once

#include <cuda_runtime.h>
#include <stddef.h>
#include <stdint.h>

#include "moments.cuh"

namespace ccab {

constexpr int kEyMaxK = 32;          // latent dimensions one fit may carry (register-resident rows of W)
constexpr int kEyStateHeader = 8;    // doubles in front of W and the velocity in the state block

struct EyParams {
  int k, n_steps, batch;  // batch = 0: covariance route
  double c, lr, momentum, tol;
};

size_t ey_fit_workspace_bytes(const ColumnLayout& L, int k, int batch);
int ey_fit(const ColumnLayout& L, const EyParams& p, const double* cov, int dtype, const void* const* views,
           const int64_t* ld, const int32_t* idx, double* state, void* ws, size_t ws_bytes, cudaStream_t stream);

}  // namespace ccab
