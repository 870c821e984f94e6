// GFA (Group Factor Analysis): the mean-field variational loop iterated on the Gram matrix (see ccab_gfa_fit in
// include/ccab200.h).
#pragma once

#include <cuda_runtime.h>
#include <stddef.h>
#include <stdint.h>

#include "moments.cuh"

namespace ccab {

constexpr int kGfaMaxK = 64;        // latent dimensions one fit may carry
constexpr int kGfaHeader = 16;      // doubles of counters in front of the state block

// Offsets (in doubles) of the state block of a fit with capacity K over D features; every per-view array has
// kMaxViews slots and every k x k matrix leading dimension K, so the layout depends on (K, D) only.
struct GfaLayout {
  size_t y_const, a_ard, a_tau, tau, b_tau, alpha, b_ard, cov_w, ww, cov_z, zz, index, W, B0, B1, GB0, GB1, total;
};
GfaLayout gfa_layout(int K, int D);

size_t gfa_fit_workspace_bytes(const ColumnLayout& L, int k);
int gfa_fit(const ColumnLayout& L, int k, const double* G, double n_samples, const double* XtZ0, double tol,
            int drop_k, int n_steps, double* state, void* ws, size_t ws_bytes, cudaStream_t stream);

}  // namespace ccab
