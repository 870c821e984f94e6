// Sparse / ALS estimators on the block Gram matrix (see ccab_als_fit in include/ccab200.h).
#pragma once

#include <cuda_runtime.h>
#include <stddef.h>
#include <stdint.h>

#include "moments.cuh"

namespace ccab {

// estimator kinds of ccab_als_fit (CCAB_ALS_* in include/ccab200.h)
enum AlsKind { kAlsPls = 0, kAlsPmd = 1, kAlsParkhomenko = 2, kAlsSpan = 3, kAlsAdmm = 4, kAlsElastic = 5, kAlsIpls = 6 };

// regression: ElasticCCA / SCCA_IPLS (kinds 5, 6) need more (the eigendecompositions of the diagonal blocks)
size_t als_fit_workspace_bytes(const ColumnLayout& L, bool regression);
int als_fit(int kind, const ColumnLayout& L, const double* G, double g_scale, double n_samples, const double* params,
            double mu, const double* init, int k, int max_iter, double tol, double* W_out, int* iters_out, void* ws,
            size_t ws_bytes, cudaStream_t stream);

}  // namespace ccab
