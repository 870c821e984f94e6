// Held-out scores of a batch of fitted candidates from the block covariance of the test rows (see ccab_cv_scores in
// include/ccab200.h).
#pragma once

#include <cuda_runtime.h>
#include <stddef.h>
#include <stdint.h>

#include "moments.cuh"   // kMaxViews

namespace ccab {

size_t cv_scores_workspace_bytes(int n_views, const int64_t* dims, int64_t n_cols);
int cv_scores(int n_views, const int64_t* dims, const double* C, int64_t ldc, double n, const double* W, int64_t ldw,
              int G, int k_max, const int* k_of, double* corr, double* score, void* ws,
              cudaStream_t stream);

}  // namespace ccab
