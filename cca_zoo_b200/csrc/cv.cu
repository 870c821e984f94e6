// Held-out scores of G fitted candidates from the block covariance C of the test rows (ccab_cv_scores).
//
// For candidate b, latent dimension j (column c = b * k_max + j of W) and views i, l:
//   S_il = w_i^T C_il w_l,   den_i = max'(sqrt(S_ii (n - 1))) / sqrt(n - 1)   (max'(x) = x > 1e-12 ? x : 1)
//   corr[b, j] = sum_{i != l} S_il / (den_i den_l) / (m (m - 1)),   score[b] = mean_{j < k_of[b]} corr[b, j]
// which is average_pairwise_correlations of the projected test rows, written in the covariance (as
// BaseModel._pairwise_correlations_device does for one model).
//
// Two stages:
//   1. Y_l = C[:, block l] W[block l, :] for every view l: m GEMMs on the fp64 tensor pipe (xgemm<double>), D x G k_max
//      each, into the workspace;
//   2. cv_scores_kernel, one CTA per candidate: for each of its dimensions the diagonal S_ii, then the normalised
//      off-diagonal sum sum_{r in block i} W[r, c] sum_{l != i} Y_l[r, c] / den_l.  Every reduction runs in a fixed
//      order (strided per-thread sums, a shuffle butterfly, warps in index order), so repeated calls are bit-identical.
#include "cv.cuh"

#include <cmath>

#include "common.cuh"
#include "dense.cuh"

namespace ccab {
namespace {

constexpr int kThreads = 256;
constexpr int kWarps = kThreads / 32;

struct CvLayout {
  int m;
  int off[kMaxViews + 1];   // row offset of each view's block in C and W
};

__device__ __forceinline__ double warp_sum(double v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
  return v;
}

// tot[i] = sum over the CTA of s[i], i < m (warps added in index order)
__device__ __forceinline__ void block_sums(const double (&s)[kMaxViews], int m, double (*red)[kWarps], double* tot) {
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
#pragma unroll
  for (int i = 0; i < kMaxViews; ++i) {
    if (i < m) {
      const double v = warp_sum(s[i]);
      if (lane == 0) red[i][warp] = v;
    }
  }
  __syncthreads();
  if (threadIdx.x < m) {
    double t = 0.0;
#pragma unroll
    for (int w = 0; w < kWarps; ++w) t += red[threadIdx.x][w];
    tot[threadIdx.x] = t;
  }
  __syncthreads();
}

__global__ void __launch_bounds__(kThreads) cv_scores_kernel(const CvLayout L, double nm1,
                                                             const double* __restrict__ W, int64_t ldw,
                                                             const double* __restrict__ Y, int64_t ldy,
                                                             int64_t ystride, int k_max,
                                                             const int* __restrict__ k_of,
                                                             double* __restrict__ corr, double* __restrict__ score) {
  __shared__ double red[kMaxViews][kWarps];
  __shared__ double tot[kMaxViews];
  __shared__ double den[kMaxViews];
  const int b = blockIdx.x, m = L.m;
  const int kb = min(max(k_of[b], 0), k_max);
  const double sq = sqrt(nm1);
  double total = 0.0;
  for (int j = 0; j < k_max; ++j) {
    const int64_t c = (int64_t)b * k_max + j;
    if (j >= kb) {
      if (threadIdx.x == 0) corr[c] = 0.0;
      continue;
    }
    double s[kMaxViews];
#pragma unroll
    for (int i = 0; i < kMaxViews; ++i) {
      s[i] = 0.0;
      if (i < m) {
        const double* Yi = Y + i * ystride;
        for (int r = L.off[i] + threadIdx.x; r < L.off[i + 1]; r += kThreads)
          s[i] = fma(W[(int64_t)r * ldw + c], Yi[(int64_t)r * ldy + c], s[i]);
      }
    }
    block_sums(s, m, red, tot);
    if (threadIdx.x < m) {
      const double nrm = sqrt(tot[threadIdx.x] * nm1);
      den[threadIdx.x] = (nrm > 1e-12 ? nrm : 1.0) / sq;
    }
    __syncthreads();
#pragma unroll
    for (int i = 0; i < kMaxViews; ++i) {
      s[i] = 0.0;
      if (i < m) {
        for (int r = L.off[i] + threadIdx.x; r < L.off[i + 1]; r += kThreads) {
          double y = 0.0;
#pragma unroll
          for (int l = 0; l < kMaxViews; ++l)
            if (l < m && l != i) y += Y[l * ystride + (int64_t)r * ldy + c] / den[l];
          s[i] = fma(W[(int64_t)r * ldw + c], y, s[i]);
        }
      }
    }
    block_sums(s, m, red, tot);
    if (threadIdx.x == 0) {
      double off = 0.0;
      for (int i = 0; i < m; ++i) off += tot[i] / den[i];
      const double v = off / (double)(m * (m - 1));
      corr[c] = v;
      total += v;
    }
    __syncthreads();   // tot / den are rewritten for the next dimension
  }
  if (threadIdx.x == 0) score[b] = kb > 0 ? total / kb : 0.0;
}

}  // namespace

size_t cv_scores_workspace_bytes(int n_views, const int64_t* dims, int64_t n_cols) {
  int64_t D = 0;
  for (int v = 0; v < n_views; ++v) D += dims[v];
  return (size_t)n_views * (size_t)D * (size_t)n_cols * sizeof(double) + 256;
}

int cv_scores(int n_views, const int64_t* dims, const double* C, int64_t ldc, double n, const double* W, int64_t ldw,
              int G, int k_max, const int* k_of, double* corr, double* score, void* ws,
              cudaStream_t stream) {
  CvLayout L;
  L.m = n_views;
  L.off[0] = 0;
  for (int v = 0; v < n_views; ++v) L.off[v + 1] = L.off[v] + (int)dims[v];
  const int D = L.off[n_views];
  const int64_t ncol = (int64_t)G * k_max;
  double* Y = reinterpret_cast<double*>((reinterpret_cast<uintptr_t>(ws) + 255) & ~(uintptr_t)255);
  const int64_t ystride = (int64_t)D * ncol;
  for (int l = 0; l < n_views; ++l) {
    GemmArgs<double> g;
    g.m = D; g.n = (int)ncol; g.k = (int)dims[l];
    g.A = C + L.off[l]; g.lda = ldc;
    g.B = W + (int64_t)L.off[l] * ldw; g.ldb = ldw;
    g.C = Y + l * ystride; g.ldc = ncol;
    const int rc = xgemm<double>(g, stream);
    if (rc) return rc;
  }
  cv_scores_kernel<<<G, kThreads, 0, stream>>>(L, n - 1.0, W, ldw, Y, ncol, ystride, k_max, k_of, corr, score);
  count_launches(1);
  CCAB_CUDA(cudaGetLastError());
  return 0;
}

}  // namespace ccab
