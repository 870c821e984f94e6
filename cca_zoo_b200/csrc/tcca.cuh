// TCCA (tensor CCA): the Khatri-Rao contraction that builds the whitened cross-moment tensor, and CP-ALS on that
// tensor (see ccab_tcca_moment / ccab_tcca_fit in include/ccab200.h).
#pragma once

#include <cuda_runtime.h>
#include <stddef.h>
#include <stdint.h>

namespace ccab {

constexpr int kTccaMaxViews = 8;
constexpr int kTccaMaxK = 64;
constexpr int64_t kTccaMaxEntries = (int64_t)1 << 25;   // prod p_i: M in float64 is 256 MB
constexpr int kTccaMaxIter = 100;                       // tensorly's n_iter_max: length of the rec history
constexpr int kTccaHeader = 8;                          // doubles in front of the rec history in the state block

// Problem sizes shared by the entry points; returns non-zero (with the error set) when they are out of range.
int tcca_check_dims(int n_views, const int64_t* dims);

int tcca_moment_plan(int n_views, const int64_t* dims, int64_t n, int nsplit);   // splits of n the contraction uses
size_t tcca_moment_workspace_bytes(int n_views, const int64_t* dims, int64_t n, int nsplit);
int tcca_moment(int n_views, const int64_t* dims, int64_t n, const double* const* Z, const int64_t* ldz, double scale,
                int nsplit, double* M, void* ws, size_t ws_bytes, cudaStream_t stream);

int tcca_moment_adjoint(int n_views, const int64_t* dims, int64_t n, const double* M, const double* const* H,
                        const int64_t* ldh, double scale, const double* dscale, double* const* Y, const int64_t* ldy,
                        cudaStream_t stream);

size_t tcca_state_doubles(int n_views, const int64_t* dims, int k);
size_t tcca_fit_workspace_bytes(int n_views, const int64_t* dims, int k);
int tcca_fit(int n_views, const int64_t* dims, int k, const double* M, const double* const* evecs, const double* lam0,
             const double* rand, int start, int n_iter, double* state, void* ws, size_t ws_bytes, cudaStream_t stream);

}  // namespace ccab
