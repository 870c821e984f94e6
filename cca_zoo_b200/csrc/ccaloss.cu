// K6: fused small-matrix stage of the deep-CCA objective (cca_zoo/deep/objectives.py:86-102) for encoder
// widths d1, d2 <= 64: ONE single-CTA launch turns the block covariance of [z1 z2] into the loss and the
// three small matrices its analytic gradient needs.
//
//   S11 = C11 + eps I, S22 = C22 + eps I, S12 = C12
//   I1 = S11^-1, I2 = S22^-1      in-place Gauss-Jordan without pivoting (safe for SPD); its pivots are the
//                                 squared Cholesky pivots, whose minimum is returned so the caller can certify
//                                 that the reference's clamp(min=eps) of the eigenvalues is inactive
//   P  = I1 S12 I2                loss = -<P, S12> = -|| S11^-1/2 S12 S22^-1/2 ||_F^2
//   G11 = P S21 I1, G22 = I2 S21 P                      (dL/dS11, dL/dS22; dL/dS12 = -2 P; SURVEY.md §3.4)
//
// Everything lives in shared memory (6 matrices of 64 x 65), 1024 threads, two block barriers per
// elimination step.
#include "ccaloss.cuh"

#include "chol_device.cuh"

namespace ccab {

constexpr int kLD = 64;
constexpr int kLP = kLD + 1;

template <typename T>
__device__ void spd_inverse_inplace(T* A, int d, T* rowk, T* colk, T* minpiv_s) {
  for (int k = 0; k < d; ++k) {
    for (int i = threadIdx.x; i < d; i += blockDim.x) {
      rowk[i] = A[k * kLP + i];
      colk[i] = A[i * kLP + k];
    }
    __syncthreads();
    const T p = rowk[k];
    if (threadIdx.x == 0) *minpiv_s = fmin(*minpiv_s, p);
    const T ip = T(1) / p;
    for (int e = threadIdx.x; e < d * d; e += blockDim.x) {
      const int i = e / d, j = e % d;
      const T rkj = (j == k ? T(1) : rowk[j]) * ip;
      T v;
      if (i == k) v = rkj;
      else v = (j == k ? T(0) : A[i * kLP + j]) - colk[i] * rkj;
      A[i * kLP + j] = v;
    }
    __syncthreads();
  }
}

// Cm (m x n) = op(A) op(B) with k the contraction length; all operands in shared memory (stride kLP)
template <typename T, int TA, int TB>
__device__ void smem_matmul(const T* A, const T* B, T* Cm, int m, int n, int k) {
  for (int e = threadIdx.x; e < m * n; e += blockDim.x) {
    const int i = e / n, j = e % n;
    T acc = 0;
    for (int t = 0; t < k; ++t) {
      const T a = TA ? A[t * kLP + i] : A[i * kLP + t];
      const T b = TB ? B[j * kLP + t] : B[t * kLP + j];
      acc = fma(a, b, acc);
    }
    Cm[i * kLP + j] = acc;
  }
  __syncthreads();
}

template <typename T>
__global__ void __launch_bounds__(1024) ccaloss_small_kernel(const T* __restrict__ C, int64_t ldc, int d1, int d2,
                                                             T eps, T* __restrict__ loss, T* __restrict__ G11,
                                                             T* __restrict__ Pout, T* __restrict__ G22,
                                                             T* __restrict__ min_pivot) {
  extern __shared__ __align__(16) unsigned char ccl_smem[];
  T* I1 = reinterpret_cast<T*>(ccl_smem);   // S11 -> S11^-1
  T* I2 = I1 + kLD * kLP;                    // S22 -> S22^-1
  T* S12 = I2 + kLD * kLP;
  T* Tm = S12 + kLD * kLP;
  T* Pm = Tm + kLD * kLP;
  T* Gm = Pm + kLD * kLP;
  T* rowk = Gm + kLD * kLP;                  // [64]
  T* colk = rowk + kLD;                      // [64]
  T* red = colk + kLD;                       // [32]
  T* minpiv = red + 32;                      // [1]
  for (int e = threadIdx.x; e < d1 * d1; e += blockDim.x) {
    const int i = e / d1, j = e % d1;
    I1[i * kLP + j] = C[(size_t)i * ldc + j] + (i == j ? eps : T(0));
  }
  for (int e = threadIdx.x; e < d2 * d2; e += blockDim.x) {
    const int i = e / d2, j = e % d2;
    I2[i * kLP + j] = C[(size_t)(d1 + i) * ldc + d1 + j] + (i == j ? eps : T(0));
  }
  for (int e = threadIdx.x; e < d1 * d2; e += blockDim.x) {
    const int i = e / d2, j = e % d2;
    S12[i * kLP + j] = C[(size_t)i * ldc + d1 + j];
  }
  if (threadIdx.x == 0) *minpiv = T(3.0e38);
  __syncthreads();
  spd_inverse_inplace(I1, d1, rowk, colk, minpiv);
  spd_inverse_inplace(I2, d2, rowk, colk, minpiv);
  smem_matmul<T, 0, 0>(I1, S12, Tm, d1, d2, d1);      // Tm = I1 S12
  smem_matmul<T, 0, 0>(Tm, I2, Pm, d1, d2, d2);       // P  = I1 S12 I2
  T acc = 0;
  for (int e = threadIdx.x; e < d1 * d2; e += blockDim.x) {
    const int i = e / d2, j = e % d2;
    acc = fma(Pm[i * kLP + j], S12[i * kLP + j], acc);
    Pout[(size_t)i * d2 + j] = Pm[i * kLP + j];
  }
  for (int o = 16; o > 0; o >>= 1) acc += __shfl_xor_sync(0xffffffffu, acc, o);
  if ((threadIdx.x & 31) == 0) red[threadIdx.x >> 5] = acc;
  __syncthreads();
  if (threadIdx.x < 32) {
    acc = threadIdx.x < (blockDim.x >> 5) ? red[threadIdx.x] : T(0);
    for (int o = 16; o > 0; o >>= 1) acc += __shfl_xor_sync(0xffffffffu, acc, o);
    if (threadIdx.x == 0) {
      loss[0] = -acc;
      min_pivot[0] = *minpiv;
    }
  }
  __syncthreads();
  smem_matmul<T, 0, 1>(Pm, S12, Tm, d1, d1, d2);      // Tm = P S12^T            (d1 x d1)
  smem_matmul<T, 0, 0>(Tm, I1, Gm, d1, d1, d1);       // G11 = P S21 I1
  for (int e = threadIdx.x; e < d1 * d1; e += blockDim.x) G11[e] = Gm[(e / d1) * kLP + e % d1];
  __syncthreads();
  smem_matmul<T, 1, 0>(S12, Pm, Tm, d2, d2, d1);      // Tm = S12^T P            (d2 x d2)
  smem_matmul<T, 0, 0>(I2, Tm, Gm, d2, d2, d2);       // G22 = I2 S21 P
  for (int e = threadIdx.x; e < d2 * d2; e += blockDim.x) G22[e] = Gm[(e / d2) * kLP + e % d2];
}

template <typename T>
int ccaloss_small(const T* C, int64_t ldc, int d1, int d2, double eps, T* loss, T* G11, T* P, T* G22, T* min_pivot,
                  cudaStream_t stream) {
  CCAB_CHECK_ARG(d1 >= 1 && d2 >= 1 && d1 <= kLD && d2 <= kLD, "ccaloss_small supports widths 1..64, got %d, %d", d1,
                 d2);
  CCAB_CHECK_ARG(ldc >= d1 + d2, "ldc too small");
  const size_t smem = sizeof(T) * (6 * kLD * kLP + 2 * kLD + 33);
  CCAB_CUDA(cudaFuncSetAttribute(ccaloss_small_kernel<T>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
  ccaloss_small_kernel<T><<<1, 1024, smem, stream>>>(C, ldc, d1, d2, (T)eps, loss, G11, P, G22, min_pivot);
  count_launches(1);
  CCAB_CUDA(cudaGetLastError());
  return 0;
}


// =============================================================================================================
// widths <= 64: the whole objective after the moment pass in one launch, the whole backward in one launch
// =============================================================================================================
namespace {

// Gauss-Jordan inversion of TWO SPD matrices side by side (threads [0, 512) work on A1, [512, 1024) on A2; the step
// loop runs max(d1, d2) times with two block barriers per step for both).  minpiv_s[0..1] <- smallest pivots.
template <typename T>
__device__ void spd_inverse_pair(T* A1, int d1, T* A2, int d2, T* rowk, T* colk, T* minpiv_s) {
  const int half = threadIdx.x >> 9;                 // 0 / 1
  const int t = threadIdx.x & 511;
  T* A = half ? A2 : A1;
  const int d = half ? d2 : d1;
  T* rk = rowk + half * kLD;
  T* ck = colk + half * kLD;
  const int steps = d1 > d2 ? d1 : d2;
  for (int k = 0; k < steps; ++k) {
    const bool on = k < d;
    if (on)
      for (int i = t; i < d; i += 512) {
        rk[i] = A[k * kLP + i];
        ck[i] = A[i * kLP + k];
      }
    __syncthreads();
    if (on) {
      const T p = rk[k];
      if (t == 0) minpiv_s[half] = fmin(minpiv_s[half], p);
      const T ip = T(1) / p;
      for (int e = t; e < d * d; e += 512) {
        const int i = e / d, j = e % d;
        const T rkj = (j == k ? T(1) : rk[j]) * ip;
        T v;
        if (i == k) v = rkj;
        else v = (j == k ? T(0) : A[i * kLP + j]) - ck[i] * rkj;
        A[i * kLP + j] = v;
      }
    }
    __syncthreads();
  }
}

// Cm (m x n) = op(A) op(B), operands in shared memory (stride kLP); 4 x 2 register tiles: a warp owns 4 rows, a lane
// the columns lane, lane + 32 -- A values are warp broadcasts, B values conflict-free
template <typename T, int TA, int TB>
__device__ void smem_matmul4(const T* A, const T* B, T* Cm, int m, int n, int k) {
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31, nwarps = blockDim.x >> 5;
  for (int r0 = warp * 4; r0 < m; r0 += nwarps * 4) {
    T acc[4][2];
#pragma unroll
    for (int i = 0; i < 4; ++i) acc[i][0] = acc[i][1] = T(0);
    for (int t = 0; t < k; ++t) {
      T a[4], b[2];
#pragma unroll
      for (int i = 0; i < 4; ++i) a[i] = (r0 + i < m) ? (TA ? A[t * kLP + r0 + i] : A[(r0 + i) * kLP + t]) : T(0);
#pragma unroll
      for (int j = 0; j < 2; ++j) {
        const int c = lane + 32 * j;
        b[j] = (c < n) ? (TB ? B[c * kLP + t] : B[t * kLP + c]) : T(0);
      }
#pragma unroll
      for (int i = 0; i < 4; ++i) {
        acc[i][0] = fma(a[i], b[0], acc[i][0]);
        acc[i][1] = fma(a[i], b[1], acc[i][1]);
      }
    }
#pragma unroll
    for (int i = 0; i < 4; ++i)
#pragma unroll
      for (int j = 0; j < 2; ++j) {
        const int c = lane + 32 * j;
        if (r0 + i < m && c < n) Cm[(r0 + i) * kLP + c] = acc[i][j];
      }
  }
  __syncthreads();
}

// S_h^-1 for the two (<= 64 x 64, identity-padded) SPD matrices side by side: threads [0, 512) work on A1, the rest on
// A2, both halves in lockstep (the barriers are common).  Cholesky by one warp per 32 x 32 block (chol_device.cuh),
// panel by row-wise forward substitution, inverse of the factor by one warp per diagonal block plus one
// recursive-doubling step, then A <- X^T X with X = L^-1.  X1 / X2 / tmp are scratch (64 x 65, 64 x 65, 64 x 65).
// notpd[h] != 0 when a pivot of matrix h is <= piv_tol.
template <typename T>
__device__ void chol_inverse_pair(T* A1, int d1, T* A2, int d2, T* X1, T* X2, T* tmp, T* dinv, T piv_tol, int* notpd) {
  const int half = threadIdx.x >> 9, t = threadIdx.x & 511, hw = t >> 5, lane = t & 31;
  T* A = half ? A2 : A1;
  T* X = half ? X2 : X1;
  T* tm = tmp + half * 32 * kLP;
  T* dv = dinv + half * kLD;
  const int d = half ? d2 : d1;
  const bool two = d > 32;                         // this half has a second 32-block with data
  const bool any_two = d1 > 32 || d2 > 32;         // uniform over the CTA
  for (int e = t; e < kLD * kLD; e += 512) X[(e / kLD) * kLP + e % kLD] = T(0);
  if (t < kLD) dv[t] = T(1);
  __syncthreads();
  if (hw == 0) warp_chol_32<T, kLP>(A, dv, 0, d, 0, piv_tol, notpd + half);
  __syncthreads();
  if (any_two) {
    if (two && t < 32) {                           // panel row 32 + t <- a L_00^-T
      T* row = A + (32 + t) * kLP;
      T a[32];
#pragma unroll
      for (int c = 0; c < 32; ++c) a[c] = row[c];
#pragma unroll
      for (int c = 0; c < 32; ++c) {
        T v = a[c];
#pragma unroll
        for (int k = 0; k < c; ++k) v = fma(-a[k], A[c * kLP + k], v);
        a[c] = v * dv[c];
      }
#pragma unroll
      for (int c = 0; c < 32; ++c) row[c] = a[c];
    }
    __syncthreads();
    if (two)
      for (int e = t; e < 32 * 32; e += 512) {     // trailing update, lower part
        const int r = 32 + e / 32, c = 32 + e % 32;
        if (c > r) continue;
        T acc = T(0);
#pragma unroll 8
        for (int k = 0; k < 32; ++k) acc = fma(A[r * kLP + k], A[c * kLP + k], acc);
        A[r * kLP + c] -= acc;
      }
    __syncthreads();
    if (two && hw == 0) warp_chol_32<T, kLP>(A, dv, 32, d, 0, piv_tol, notpd + half);
    __syncthreads();
  }
  if (hw == 0) warp_trinv_32<T, kLP>(A, dv, X, 0);
  if (hw == 1) {
    if (two) warp_trinv_32<T, kLP>(A, dv, X, 32);
    else X[(32 + lane) * kLP + 32 + lane] = T(1);   // padding block: identity
  }
  __syncthreads();
  if (any_two) {                                   // X_10 = -X_11 (L_10 X_00)
    if (two)
      for (int e = t; e < 32 * 32; e += 512) {
        const int rr = e / 32, cc = e % 32;
        T acc = T(0);
        for (int k = cc; k < 32; ++k) acc = fma(A[(32 + rr) * kLP + k], X[k * kLP + cc], acc);
        tm[rr * kLP + cc] = acc;
      }
    __syncthreads();
    if (two)
      for (int e = t; e < 32 * 32; e += 512) {
        const int rr = e / 32, cc = e % 32;
        T acc = T(0);
        for (int k = 0; k <= rr; ++k) acc = fma(X[(32 + rr) * kLP + 32 + k], tm[k * kLP + cc], acc);
        X[(32 + rr) * kLP + cc] = -acc;
      }
    __syncthreads();
  }
  smem_matmul4<T, 1, 0>(X1, X1, A1, kLD, kLD, kLD);   // S^-1 = X^T X (all threads, one matrix after the other)
  smem_matmul4<T, 1, 0>(X2, X2, A2, kLD, kLD, kLD);
}

template <typename T>
__global__ void __launch_bounds__(1024) ccaloss_small_fwd_kernel(const double* __restrict__ mom, int Dp, double n_host,
                                                                 const double* __restrict__ n_dev, int d1, int d2,
                                                                 T eps, T* __restrict__ loss, T* __restrict__ saved,
                                                                 int* __restrict__ flags) {
  extern __shared__ __align__(16) unsigned char ccl_smem[];
  T* I1 = reinterpret_cast<T*>(ccl_smem);   // S11 -> S11^-1
  T* I2 = I1 + kLD * kLP;                    // S22 -> S22^-1
  T* S12 = I2 + kLD * kLP;
  T* Tm = S12 + kLD * kLP;
  T* Pm = Tm + kLD * kLP;
  T* Tm2 = Pm + kLD * kLP;
  T* rowk = Tm2 + kLD * kLP;                 // [2][64]
  T* colk = rowk + 2 * kLD;                  // [2][64]
  T* red = colk + 2 * kLD;                   // [32]
  T* minpiv = red + 32;                      // [2]
  __shared__ int bad;
  __shared__ int notpd[2];
  const double* M = mom;
  const double* s = mom + (size_t)Dp * Dp;
  const int o2 = 128;                        // padded offset of view 2 (each view occupies one 128-column block)
  if (threadIdx.x == 0) { minpiv[0] = T(3.0e38); minpiv[1] = T(3.0e38); bad = 0; notpd[0] = notpd[1] = 0; }
  for (int e = threadIdx.x; e < kLD * kLD; e += blockDim.x) {   // identity padding up to 64 x 64
    const int i = e / kLD, j = e % kLD;
    I1[i * kLP + j] = I2[i * kLP + j] = (i == j) ? T(1) : T(0);
  }
  __syncthreads();
  const double n = n_dev ? n_dev[0] : n_host;    // global batch: the all-reduced count, read on the device
  const double inv = 1.0 / (n - 1.0), inv_n = 1.0 / n;
  int notfinite = 0;
  for (int e = threadIdx.x; e < d1 * d1; e += blockDim.x) {
    const int i = e / d1, j = e % d1;
    const double m = M[(size_t)min(i, j) * Dp + max(i, j)];
    notfinite |= !isfinite(m);
    I1[i * kLP + j] = (T)((m - s[i] * s[j] * inv_n) * inv) + (i == j ? eps : T(0));
  }
  for (int e = threadIdx.x; e < d2 * d2; e += blockDim.x) {
    const int i = e / d2, j = e % d2;
    const double m = M[(size_t)(o2 + min(i, j)) * Dp + o2 + max(i, j)];
    notfinite |= !isfinite(m);
    I2[i * kLP + j] = (T)((m - s[o2 + i] * s[o2 + j] * inv_n) * inv) + (i == j ? eps : T(0));
  }
  for (int e = threadIdx.x; e < d1 * d2; e += blockDim.x) {
    const int i = e / d2, j = e % d2;
    const double m = M[(size_t)i * Dp + o2 + j];
    notfinite |= !isfinite(m);
    S12[i * kLP + j] = (T)((m - s[i] * s[o2 + j] * inv_n) * inv);
  }
  if (notfinite) bad = 1;
  T* G11 = saved;
  T* Pout = saved + (size_t)d1 * d1;
  T* G22 = Pout + (size_t)d1 * d2;
  T* mean = G22 + (size_t)d2 * d2;
  for (int i = threadIdx.x; i < d1 + d2; i += blockDim.x) mean[i] = (T)(s[i < d1 ? i : o2 + i - d1] * inv_n);
  if (n_dev && threadIdx.x == 0) mean[d1 + d2] = (T)n;   // global batch: N rides behind the means for the backward
  __syncthreads();
  chol_inverse_pair(I1, d1, I2, d2, Tm, Tm2, Pm, rowk, T(0.25) * eps, notpd);
  smem_matmul4<T, 0, 0>(I1, S12, Tm, d1, d2, d1);      // Tm  = A1 S12          (Q)
  smem_matmul4<T, 0, 0>(S12, I2, Tm2, d1, d2, d2);     // Tm2 = S12 A2          (Q2)
  smem_matmul4<T, 0, 0>(Tm, I2, Pm, d1, d2, d2);       // P   = A1 S12 A2
  T acc = 0;
  for (int e = threadIdx.x; e < d1 * d2; e += blockDim.x) {
    const int i = e / d2, j = e % d2;
    acc = fma(Pm[i * kLP + j], S12[i * kLP + j], acc);
    Pout[(size_t)i * d2 + j] = Pm[i * kLP + j];
  }
  for (int o = 16; o > 0; o >>= 1) acc += __shfl_xor_sync(0xffffffffu, acc, o);
  if ((threadIdx.x & 31) == 0) red[threadIdx.x >> 5] = acc;
  __syncthreads();
  if (threadIdx.x < 32) {
    acc = threadIdx.x < (blockDim.x >> 5) ? red[threadIdx.x] : T(0);
    for (int o = 16; o > 0; o >>= 1) acc += __shfl_xor_sync(0xffffffffu, acc, o);
    if (threadIdx.x == 0) {
      loss[0] = -acc;
      flags[0] = notpd[0] != 0;
      flags[1] = notpd[1] != 0;
      flags[2] = bad;
    }
  }
  __syncthreads();
  smem_matmul4<T, 0, 1>(Pm, Tm, I1, d1, d1, d2);       // G11 = P Q^T   (I1 is free now)
  for (int e = threadIdx.x; e < d1 * d1; e += blockDim.x) G11[e] = I1[(e / d1) * kLP + e % d1];
  smem_matmul4<T, 1, 0>(Tm2, Pm, I2, d2, d2, d1);      // G22 = Q2^T P
  for (int e = threadIdx.x; e < d2 * d2; e += blockDim.x) G22[e] = I2[(e / d2) * kLP + e % d2];
}

// 64 rows per CTA, 256 threads: thread (row r = tid / 4, column phase q = tid % 4) owns the columns q, q + 4, ..
template <typename T>
__global__ void __launch_bounds__(256) ccaloss_small_bwd_kernel(int d1, int d2, const T* __restrict__ z1, int64_t ld1,
                                                                const T* __restrict__ z2, int64_t ld2, int64_t n,
                                                                const T* __restrict__ saved,
                                                                const T* __restrict__ grad_out, T* __restrict__ g1,
                                                                int64_t ldg1, T* __restrict__ g2, int64_t ldg2,
                                                                bool global) {
  extern __shared__ __align__(16) unsigned char ccb_smem[];
  T* G11 = reinterpret_cast<T*>(ccb_smem);   // [64][65] each
  T* Ps = G11 + kLD * kLP;
  T* G22 = Ps + kLD * kLP;
  T* Z1 = G22 + kLD * kLP;                    // [64 rows][65]
  T* Z2 = Z1 + kLD * kLP;
  T* r1 = Z2 + kLD * kLP;                     // [64]
  T* r2 = r1 + kLD;
  T* m1 = r2 + kLD;
  T* m2 = m1 + kLD;
  const int tid = threadIdx.x;
  const T* sG11 = saved;
  const T* sP = saved + (size_t)d1 * d1;
  const T* sG22 = sP + (size_t)d1 * d2;
  const T* smean = sG22 + (size_t)d2 * d2;
  for (int e = tid; e < d1 * d1; e += 256) G11[(e / d1) * kLP + e % d1] = sG11[e];
  for (int e = tid; e < d1 * d2; e += 256) Ps[(e / d2) * kLP + e % d2] = sP[e];
  for (int e = tid; e < d2 * d2; e += 256) G22[(e / d2) * kLP + e % d2] = sG22[e];
  if (tid < d1) m1[tid] = smean[tid];
  if (tid < d2) m2[tid] = smean[d1 + tid];
  const int64_t row0 = (int64_t)blockIdx.x * 64;
  for (int e = tid; e < 64 * d1; e += 256) {
    const int r = e / d1, c = e % d1;
    Z1[r * kLP + c] = row0 + r < n ? z1[(row0 + r) * ld1 + c] : T(0);
  }
  for (int e = tid; e < 64 * d2; e += 256) {
    const int r = e / d2, c = e % d2;
    Z2[r * kLP + c] = row0 + r < n ? z2[(row0 + r) * ld2 + c] : T(0);
  }
  __syncthreads();
  // column means of the un-centred products: r1 = m1^T G11 - m2^T P^T, r2 = m2^T G22 - m1^T P
  if (tid < d1) {
    T a = 0;
    for (int k = 0; k < d1; ++k) a = fma(m1[k], G11[k * kLP + tid], a);
    for (int k = 0; k < d2; ++k) a = fma(-m2[k], Ps[tid * kLP + k], a);
    r1[tid] = a;
  } else if (tid >= 64 && tid < 64 + d2) {
    const int c = tid - 64;
    T a = 0;
    for (int k = 0; k < d2; ++k) a = fma(m2[k], G22[k * kLP + c], a);
    for (int k = 0; k < d1; ++k) a = fma(-m1[k], Ps[k * kLP + c], a);
    r2[c] = a;
  }
  __syncthreads();
  const int r = tid >> 2, q = tid & 3;
  // global batch: n counts this shard's rows only; the scale takes the all-reduced N saved behind the means
  const double nm1 = global ? (double)smean[d1 + d2] - 1.0 : (double)(n - 1);
  const T scale = (T)(2.0 / nm1) * (grad_out ? grad_out[0] : T(1));
  T a1[16], a2[16];
#pragma unroll
  for (int j = 0; j < 16; ++j) a1[j] = a2[j] = T(0);
  for (int k = 0; k < d1; ++k) {
    const T x = Z1[r * kLP + k];
#pragma unroll
    for (int j = 0; j < 16; ++j) {
      a1[j] = fma(x, G11[k * kLP + q + 4 * j], a1[j]);       // z1 G11
      a2[j] = fma(-x, Ps[k * kLP + q + 4 * j], a2[j]);       // - z1 P
    }
  }
  for (int k = 0; k < d2; ++k) {
    const T y = Z2[r * kLP + k];
#pragma unroll
    for (int j = 0; j < 16; ++j) {
      a1[j] = fma(-y, Ps[(q + 4 * j) * kLP + k], a1[j]);     // - z2 P^T
      a2[j] = fma(y, G22[k * kLP + q + 4 * j], a2[j]);       // z2 G22
    }
  }
  if (row0 + r < n) {
#pragma unroll
    for (int j = 0; j < 16; ++j) {
      const int c = q + 4 * j;
      if (c < d1) g1[(row0 + r) * ldg1 + c] = (a1[j] - r1[c]) * scale;
      if (c < d2) g2[(row0 + r) * ldg2 + c] = (a2[j] - r2[c]) * scale;
    }
  }
}

}  // namespace

template <typename T>
int ccaloss_small_forward(const double* moments, int Dp, double n, int d1, int d2, double eps, T* loss, T* saved,
                          int* flags, cudaStream_t stream, const double* n_dev) {
  CCAB_CHECK_ARG(d1 >= 1 && d2 >= 1 && d1 <= kLD && d2 <= kLD && Dp == 256, "ccaloss_small_forward: widths 1..64");
  const size_t smem = sizeof(T) * (6 * kLD * kLP + 4 * kLD + 40);
  static bool attr_done[64] = {};
  int dev = 0;
  CCAB_CUDA(cudaGetDevice(&dev));
  if (dev < 0 || dev >= 64 || !attr_done[dev]) {
    CCAB_CUDA(cudaFuncSetAttribute(ccaloss_small_fwd_kernel<T>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
    if (dev >= 0 && dev < 64) attr_done[dev] = true;
  }
  ccaloss_small_fwd_kernel<T><<<1, 1024, smem, stream>>>(moments, Dp, n, n_dev, d1, d2, (T)eps, loss, saved, flags);
  count_launches(1);
  CCAB_CUDA(cudaGetLastError());
  return 0;
}

template <typename T>
int ccaloss_small_backward(int d1, int d2, const T* z1, int64_t ld1, const T* z2, int64_t ld2, int64_t n,
                           const T* saved, const T* grad_out, T* g1, int64_t ldg1, T* g2, int64_t ldg2,
                           cudaStream_t stream, bool global) {
  CCAB_CHECK_ARG(d1 >= 1 && d2 >= 1 && d1 <= kLD && d2 <= kLD && n >= (global ? 0 : 2),
                 "ccaloss_small_backward: widths 1..64");
  if (n == 0) return 0;                            // a rank without rows in a global batch
  const size_t smem = sizeof(T) * (5 * kLD * kLP + 4 * kLD);
  static bool attr_done[64] = {};
  int dev = 0;
  CCAB_CUDA(cudaGetDevice(&dev));
  if (dev < 0 || dev >= 64 || !attr_done[dev]) {
    CCAB_CUDA(cudaFuncSetAttribute(ccaloss_small_bwd_kernel<T>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
    if (dev >= 0 && dev < 64) attr_done[dev] = true;
  }
  ccaloss_small_bwd_kernel<T><<<(unsigned)ceil_div(n, 64), 256, smem, stream>>>(d1, d2, z1, ld1, z2, ld2, n, saved,
                                                                                grad_out, g1, ldg1, g2, ldg2, global);
  count_launches(1);
  CCAB_CUDA(cudaGetLastError());
  return 0;
}

template int ccaloss_small_forward<float>(const double*, int, double, int, int, double, float*, float*, int*,
                                          cudaStream_t, const double*);
template int ccaloss_small_forward<double>(const double*, int, double, int, int, double, double*, double*, int*,
                                           cudaStream_t, const double*);
template int ccaloss_small_backward<float>(int, int, const float*, int64_t, const float*, int64_t, int64_t, const float*,
                                           const float*, float*, int64_t, float*, int64_t, cudaStream_t, bool);
template int ccaloss_small_backward<double>(int, int, const double*, int64_t, const double*, int64_t, int64_t,
                                            const double*, const double*, double*, int64_t, double*, int64_t,
                                            cudaStream_t, bool);

template int ccaloss_small<float>(const float*, int64_t, int, int, double, float*, float*, float*, float*, float*,
                                  cudaStream_t);
template int ccaloss_small<double>(const double*, int64_t, int, int, double, double*, double*, double*, double*,
                                   double*, cudaStream_t);

}  // namespace ccab
