// Device-side fit assembly (see fit.cu): moments -> weights without a host round trip.
#pragma once
#include "common.cuh"
#include "moments.cuh"

namespace ccab {

// Result block = [ header: double[kFitHeaderDoubles] | mean: double[D] | sigma: T[k] | W_1: T[d_1 x k] | W_2 ... ],
// every section 256-byte aligned (offsets from *_result_layout).  Header:
//   [0] status bit mask (0 = the weights are valid)   [1] n_total   [2] residual ||T^T U - V diag(sigma)||_F
//   [3] sigma_1   [4] 1-based index of the first failed Cholesky (0 = none)   [5] sweeps of the Ritz eigensolve
constexpr int kFitHeaderDoubles = 32;
constexpr int kFitNotPositiveDefinite = 1;  // a ridge block (or a CholQR Gram matrix) failed the pivot test
constexpr int kFitNotConverged = 2;         // the subspace iteration / Ritz solve missed the tolerance
constexpr int kFitNonFinite = 4;            // NaN / inf in the moments (i.e. in the input)
constexpr int kFitTooFewSamples = 8;        // n <= max(d_i): the covariance blocks are rank deficient by construction

template <typename T>
size_t rcca_fit_workspace_bytes(int d1, int d2, int k, int p);
template <typename T>
void rcca_fit_result_layout(int d1, int d2, int k, int p, int64_t* offsets /* mean, sigma, W1, W2, total */);
// c: host double[2].  n_dev (device, may be NULL) overrides n_host.  p = width of the iterated block (k + oversampling).
template <typename T>
int rcca_fit(const ColumnLayout& L, const double* moments, const double* n_dev, double n_host, int center,
             const double* c, int k, int p, int iters, void* result, size_t result_bytes, void* ws, size_t ws_bytes,
             cudaStream_t stream);

// MCCA (cca_zoo/linear/_mcca.py:113-173, pca=False form): result block = header | mean | eigenvalues T[k] | W_1 .. W_m
// (offsets: mean, values, W_1 .. W_m, total = m + 3 entries).  c: host double[m], eps_floor: the reference's eps.
template <typename T>
size_t mcca_fit_workspace_bytes(const ColumnLayout& L, int k, int p);
template <typename T>
void mcca_fit_result_layout(const ColumnLayout& L, int k, int p, int64_t* offsets);
template <typename T>
int mcca_fit(const ColumnLayout& L, const double* moments, const double* n_dev, double n_host, int center,
             const double* c, double eps_floor, int k, int p, int iters, void* result, size_t result_bytes, void* ws,
             size_t ws_bytes, cudaStream_t stream);

// ---- deep-CCA objective on the device (cca_zoo/deep/objectives.py:61-102), any widths, nothing read back ----
// saved (T[d1*d1 + d1*d2 + d2*d2 + d1 + d2]) = G11 | P | G22 | means for the analytic backward; flags_out (device int[3]) = Cholesky
// status of S11, S22 (pivot^2 <= eps / 4 counts as failure) and a non-finite-input flag, to be checked lazily.
template <typename T>
size_t ccaloss_workspace_bytes(const ColumnLayout& L, int64_t n, int precision);
template <typename T>
int ccaloss_forward(const ColumnLayout& L, int precision, const void* z1, int64_t ld1, const void* z2, int64_t ld2,
                    int64_t n, double eps, T* loss, T* saved, int* flags_out, void* ws, size_t ws_bytes,
                    cudaStream_t stream);
// g1 / g2 (n x d1 / n x d2) <- 2/(n-1) center(z1 G11 - z2 P^T) * grad_out[0] and the symmetric expression
template <typename T>
int ccaloss_backward(int d1, int d2, const T* z1, int64_t ld1, const T* z2, int64_t ld2, int64_t n, const T* saved,
                     const T* grad_out, T* g1, int64_t ldg1, T* g2, int64_t ldg2, cudaStream_t stream);

// ---- global batch (moments all-reduced over data-parallel ranks) ----
// The stage of ccaloss_forward after the moment pass, from a given buffer whose sample count N is read at n_dev[0]
// (device).  saved (T[d1*d1 + d1*d2 + d2*d2 + d1 + d2 + 1]) = G11 | P | G22 | global means | N; flags as above.
template <typename T>
size_t ccaloss_fwd_moments_workspace_bytes(const ColumnLayout& L);
template <typename T>
int ccaloss_forward_moments(const ColumnLayout& L, const double* moments, const double* n_dev, double eps, T* loss,
                            T* saved, int* flags_out, void* ws, size_t ws_bytes, cudaStream_t stream);
// This shard's rows (n >= 0) of dL/dz of the global loss: g1 <- 2/(N-1) (z1 G11 - z2 P^T - 1 r_1^T) grad_out[0] with
// r_1 = mu_1^T G11 - mu_2^T P^T from the saved global means, g2 symmetric.  No collective.
template <typename T>
int ccaloss_backward_global(int d1, int d2, const T* z1, int64_t ld1, const T* z2, int64_t ld2, int64_t n,
                            const T* saved, const T* grad_out, T* g1, int64_t ldg1, T* g2, int64_t ldg2,
                            cudaStream_t stream);

}  // namespace ccab
