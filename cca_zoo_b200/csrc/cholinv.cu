// Blocked Cholesky factorisation WITH the explicit inverse of the factor, batched:
//     R = L L^T,   Linv = L^-1      (R symmetric positive definite, n x n, lower triangle referenced)
//
// This is the whitening step of the solver stage in its GEMM-friendly form: with Linv in hand,
// T = L1^-1 C12 L2^-T, K_ij = L_i^-1 C_ij L_j^-T, the weights L_i^-T U_k and S_ii^-1 = Linv^T Linv of the deep-CCA
// objective are all plain products for the tensor-core GEMM (tgemm.cu) -- no triangular solves remain.
// It replaces LAPACK's potrf/trsm inside scipy.linalg.eigh(A, B) (cca_zoo/_utils/_linalg.py:67-71), the
// ridge whitening of cca_zoo/_utils/_linalg.py:30-38 in Cholesky form, and _inv_sqrtm's role in
// cca_zoo/deep/objectives.py:94-97 (round 1 did this with 64-wide kernels: 124 dependent launches for n = 1024).
//
//   chol_diag_inv_kernel : one CTA per matrix factors a diagonal block (<= NB x NB, NB = 128 for float, 64 for
//       double) in shared memory AND inverts the factor.  32 x 32 sub-blocks: warp 0 factors / inverts a sub-block
//       warp-synchronously in registers (row per lane, shuffles, no block barrier), all warps apply the panel
//       and trailing updates; the inverse's off-diagonal sub-blocks follow by recursive doubling
//       (X_BA = -X_BB L_BA X_AA).  ~10 block barriers per 32 columns instead of 64.
//   potrf_inv (host) : right-looking over NB-wide block columns -- diagonal kernel, panel  P = A_panel Dinv^T  and
//       trailing update  A22 -= P P^T  as two GEMMs (lower tiles only) -- then Linv assembled from the diagonal
//       inverses by recursive doubling over block pairs (2 batched GEMMs per level, log2(n / NB) levels).
//       n = 1024: 24 + 6 launches, batched over the views.
#include "cholinv.cuh"

#include <type_traits>

#include "chol_device.cuh"
#include "dense.cuh"
#include "tgemm.cuh"

namespace ccab {

template <typename T>
int potrf_panel_gemm(const GemmArgs<T>& g, T* scratch, int64_t strideScratch, cudaStream_t stream);

namespace {

template <typename T>
struct DiagCfg;
template <>
struct DiagCfg<float> {
  static constexpr int NB = 128;
  static constexpr int kThreads = 512;
};
template <>
struct DiagCfg<double> {
  static constexpr int NB = 64;
  static constexpr int kThreads = 256;   // warp 0 holds a 32 x 32 row and column in registers: 128+ per thread
};

// C[r][c] (+)= sign * sum_{k in [k0, k1)} A(r, k) * B(k, c) for r in [0, M), c in [0, Nc), all in shared memory.
// Warp-centric register tiling: a warp takes 4 rows at a time, lane l the columns l, l + 32, ... -- the A values are
// warp broadcasts, the B values conflict-free; 4 + NT loads per 4 * NT FMAs.  BT: B(k, c) = Bm[c * ldb + k] (the
// A A^T form of the trailing update) else Bm[k * ldb + c].  tri: 0 none, 1 = only c <= r is needed (lower part),
// klo / khi: per-tile reduction bounds for triangular operands (see the callers).
template <typename T, int NT, bool BT, typename KLo, typename KHi>
__device__ __forceinline__ void smem_mm(T* Cm, int ldc, const T* Am, int lda, const T* Bm, int ldb, int M, int Nc,
                                        T sign, bool accumulate, bool lower_only, KLo klo, KHi khi, int nthreads) {
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31, nwarps = nthreads >> 5;
  for (int r0 = warp * 4; r0 < M; r0 += nwarps * 4) {
    T acc[4][NT];
#pragma unroll
    for (int i = 0; i < 4; ++i)
#pragma unroll
      for (int j = 0; j < NT; ++j) acc[i][j] = T(0);
    const int kb = klo(r0), ke = khi(r0);
#pragma unroll 4
    for (int k = kb; k < ke; ++k) {
      T a[4], b[NT];
#pragma unroll
      for (int i = 0; i < 4; ++i) a[i] = (r0 + i < M) ? Am[(r0 + i) * lda + k] : T(0);
#pragma unroll
      for (int j = 0; j < NT; ++j) {
        const int c = lane + 32 * j;
        b[j] = (c < Nc) ? (BT ? Bm[c * ldb + k] : Bm[k * ldb + c]) : T(0);
      }
#pragma unroll
      for (int i = 0; i < 4; ++i)
#pragma unroll
        for (int j = 0; j < NT; ++j) acc[i][j] = fma(a[i], b[j], acc[i][j]);
    }
#pragma unroll
    for (int i = 0; i < 4; ++i)
#pragma unroll
      for (int j = 0; j < NT; ++j) {
        const int r = r0 + i, c = lane + 32 * j;
        if (r < M && c < Nc && (!lower_only || c <= r)) {
          const T v = sign * acc[i][j];
          Cm[r * ldc + c] = accumulate ? Cm[r * ldc + c] + v : v;
        }
      }
  }
}

template <typename T, int NB, int kDiagThreads>
__global__ void __launch_bounds__(kDiagThreads, 1)
chol_diag_inv_kernel(T* __restrict__ A, int64_t lda, int64_t strideA, int nb, int j0, T* __restrict__ Dinv,
                     int64_t strideDinv, double piv_tol, const double* __restrict__ piv_tol_dev,
                     int* __restrict__ info) {
  constexpr int LD = NB + 1;
  constexpr int HB = NB / 2;
  constexpr int NSUB = NB / 32;
  extern __shared__ __align__(16) unsigned char cdi_smem[];
  T* S = reinterpret_cast<T*>(cdi_smem);
  T* X = S + NB * LD;
  T* Tm = X + NB * LD;            // [HB][HB + 1]
  T* dinv_s = Tm + HB * (HB + 1); // [NB]
  __shared__ int bad;
  T* Ab = A + (size_t)blockIdx.x * strideA;
  T* Db = Dinv + (size_t)blockIdx.x * strideDinv;
  const int tid = threadIdx.x;
  const T tol = (T)(piv_tol_dev ? piv_tol_dev[blockIdx.x] : piv_tol);
  if (tid == 0) bad = 0;
  {
    // 8 independent global loads in flight per thread (a load-then-store loop serialises on the memory latency);
    // the strict upper triangle is loaded too (it lies inside the matrix) but never used
    constexpr int kPer = NB * NB / kDiagThreads;
    static_assert(kPer % 8 == 0 && NB * NB % kDiagThreads == 0, "load tiling");
    for (int base = 0; base < kPer; base += 8) {
      T v[8];
#pragma unroll
      for (int u = 0; u < 8; ++u) {
        const int e = tid + (base + u) * kDiagThreads;
        const int r = e / NB, c = e % NB;
        v[u] = (r < nb && c < nb) ? Ab[(size_t)r * lda + c] : T(0);
      }
#pragma unroll
      for (int u = 0; u < 8; ++u) {
        const int e = tid + (base + u) * kDiagThreads;
        const int r = e / NB, c = e % NB;
        T w = (r == c) ? T(1) : T(0);            // padding: identity
        if (r < nb && c < nb) w = c <= r ? v[u] : T(0);
        S[r * LD + c] = w;
        X[r * LD + c] = T(0);
      }
    }
  }
  if (tid < NB) dinv_s[tid] = T(1);
  __syncthreads();

  const int nsub = (nb + 31) / 32;
  for (int jb = 0; jb < nsub; ++jb) {
    const int rb = jb * 32;
    if (tid < 32) warp_chol_32<T, LD>(S, dinv_s, rb, nb, j0, tol, &bad);
    __syncthreads();
    if (jb + 1 >= nsub) break;                  // nothing below / to the right
    const int r0 = rb + 32;
    const int R = nsub * 32 - r0;               // rows that hold data
    // ---- panel: row r of the block column <- a_r L_jj^-T by forward substitution, one thread per row ----
    if (tid < R) {
      T* row = S + (r0 + tid) * LD + rb;
      T a[32];
#pragma unroll
      for (int c = 0; c < 32; ++c) a[c] = row[c];
      // column-oriented: once a[c] is final, the 31 - c later entries take their update independently (a short
      // dependent chain of 32 scale + update steps instead of 496 chained FMAs)
#pragma unroll
      for (int c = 0; c < 32; ++c) {
        a[c] *= dinv_s[rb + c];
#pragma unroll
        for (int j = c + 1; j < 32; ++j) a[j] = fma(-a[c], S[(rb + j) * LD + rb + c], a[j]);   // warp broadcast
      }
#pragma unroll
      for (int c = 0; c < 32; ++c) row[c] = a[c];
    }
    __syncthreads();
    // ---- trailing update (lower part): S[r][c] -= sum_k P[r][k] P[c][k] ----
    smem_mm<T, NSUB - 1, true>(S + r0 * LD + r0, LD, S + r0 * LD + rb, LD, S + r0 * LD + rb, LD, R, R, T(-1), true,
                               true, [](int) { return 0; }, [](int) { return 32; }, kDiagThreads);
    __syncthreads();
  }

  // ---- inverse: the diagonal sub-blocks by one warp each ... ----
  if (tid < 32 * NSUB) {
    const int w = tid >> 5;
    if (w < nsub) warp_trinv_32<T, LD>(S, dinv_s, X, w * 32);
    else if ((tid & 31) == 0)
      for (int i = 0; i < 32; ++i) X[(w * 32 + i) * LD + w * 32 + i] = T(1);    // padding block: identity
  }
  __syncthreads();
  // ---- ... the off-diagonal sub-blocks by recursive doubling: X_BA = -X_BB (L_BA X_AA) ----
  for (int s = 32; s < NB; s *= 2) {
    const int npairs = NB / (2 * s);
    for (int pi = 0; pi < npairs; ++pi) {
      const int a0 = 2 * pi * s, b0 = a0 + s;
      // Tm = L_BA X_AA: X_AA is lower triangular, column c needs k >= c only -- a 4-row tile shares the bound 0
      if (s == 32)
        smem_mm<T, 1, false>(Tm + pi * s * (HB + 1), HB + 1, S + b0 * LD + a0, LD, X + a0 * LD + a0, LD, s, s, T(1),
                             false, false, [](int) { return 0; }, [s](int) { return s; }, kDiagThreads);
      else
        smem_mm<T, 2, false>(Tm + pi * s * (HB + 1), HB + 1, S + b0 * LD + a0, LD, X + a0 * LD + a0, LD, s, s, T(1),
                             false, false, [](int) { return 0; }, [s](int) { return s; }, kDiagThreads);
    }
    __syncthreads();
    for (int pi = 0; pi < npairs; ++pi) {
      const int a0 = 2 * pi * s, b0 = a0 + s;
      // X_BA = -X_BB Tm: X_BB lower triangular, row r needs k <= r only
      if (s == 32)
        smem_mm<T, 1, false>(X + b0 * LD + a0, LD, X + b0 * LD + b0, LD, Tm + pi * s * (HB + 1), HB + 1, s, s, T(-1),
                             false, false, [](int) { return 0; }, [s](int r0) { return min(s, r0 + 4); }, kDiagThreads);
      else
        smem_mm<T, 2, false>(X + b0 * LD + a0, LD, X + b0 * LD + b0, LD, Tm + pi * s * (HB + 1), HB + 1, s, s, T(-1),
                             false, false, [](int) { return 0; }, [s](int r0) { return min(s, r0 + 4); }, kDiagThreads);
    }
    __syncthreads();
  }

  for (int e = tid; e < NB * NB; e += kDiagThreads) {
    const int r = e / NB, c = e % NB;
    if (r < nb && c < nb) Ab[(size_t)r * lda + c] = S[r * LD + c];       // L (strict upper of the block zeroed)
    Db[(size_t)r * NB + c] = (r < nb && c < nb) ? X[r * LD + c] : T(0);
  }
  if (tid == 0 && bad) atomicCAS(info + blockIdx.x, 0, bad);
}

// Linv <- 0 everywhere, then the inverted diagonal blocks on the block diagonal
template <typename T>
__global__ void linv_init_kernel(T* __restrict__ Linv, int64_t ldi, int64_t strideL, int n, int NB,
                                 const T* __restrict__ Dinv, int64_t strideD) {
  T* Lb = Linv + (size_t)blockIdx.y * strideL;
  const T* Db = Dinv + (size_t)blockIdx.y * strideD;
  const size_t total = (size_t)n * n;
  for (size_t e = blockIdx.x * (size_t)blockDim.x + threadIdx.x; e < total; e += (size_t)gridDim.x * blockDim.x) {
    const int r = (int)(e / n), c = (int)(e % n);
    T v = T(0);
    if (r / NB == c / NB) v = Db[(size_t)(r / NB) * NB * NB + (size_t)(r % NB) * NB + (c % NB)];
    Lb[(size_t)r * ldi + c] = v;
  }
}

}  // namespace

template <typename T>
int potrf_inv_block(T* A, int64_t lda, int64_t strideA, int nb, int j0, T* Dinv, int64_t strideDinv, double piv_tol,
                    const double* piv_tol_dev, int* info, int batch, cudaStream_t stream) {
  constexpr int NB = DiagCfg<T>::NB;
  constexpr int kDiagThreads = DiagCfg<T>::kThreads;
  CCAB_CHECK_ARG(nb >= 1 && nb <= NB, "diagonal block of %d exceeds %d", nb, NB);
  const size_t smem = sizeof(T) * (2 * NB * (NB + 1) + (NB / 2) * (NB / 2 + 1) + NB);
  static bool attr_done[64] = {};
  int dev = 0;
  CCAB_CUDA(cudaGetDevice(&dev));
  if (dev < 0 || dev >= 64 || !attr_done[dev]) {
    CCAB_CUDA(cudaFuncSetAttribute(chol_diag_inv_kernel<T, NB, kDiagThreads>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
    if (dev >= 0 && dev < 64) attr_done[dev] = true;
  }
  chol_diag_inv_kernel<T, NB, kDiagThreads><<<batch, kDiagThreads, smem, stream>>>(A, lda, strideA, nb, j0, Dinv, strideDinv, piv_tol,
                                                                                  piv_tol_dev, info);
  count_launches(1);
  CCAB_CUDA(cudaGetLastError());
  return 0;
}

template <typename T>
int potrf_inv_block_size() {
  return DiagCfg<T>::NB;
}

template <typename T>
size_t potrf_inv_workspace_bytes(int n, int batch) {
  constexpr int NB = DiagCfg<T>::NB;
  const size_t nblk = (size_t)ceil_div(n, NB);
  const size_t dinv = nblk * NB * NB;            // inverted diagonal blocks
  const size_t tmp = (size_t)n * ((size_t)n / 2 + NB);  // L_BA X_AA of every pair of one doubling level
  return sizeof(T) * (dinv + tmp) * (size_t)batch + 256;
}

template <typename T>
int potrf_inv(int n, int batch, T* A, int64_t lda, int64_t strideA, T* Linv, int64_t ldi, int64_t strideLinv,
              double piv_tol, const double* piv_tol_dev, int* info, void* ws, size_t ws_bytes, cudaStream_t stream) {
  constexpr int NB = DiagCfg<T>::NB;
  CCAB_CHECK_ARG(n >= 1 && batch >= 1 && lda >= n && ldi >= n, "bad potrf_inv shape");
  CCAB_CHECK_ARG(ws_bytes >= potrf_inv_workspace_bytes<T>(n, batch), "potrf_inv workspace too small");
  CCAB_CHECK_ARG(batch == 1 || (strideA > 0 && strideLinv > 0), "potrf_inv: batch strides missing");
  const int nblk = (int)ceil_div(n, NB);
  T* w = reinterpret_cast<T*>((reinterpret_cast<uintptr_t>(ws) + 255) & ~uintptr_t(255));
  const int64_t strideD = (int64_t)nblk * NB * NB;
  T* Dinv = w;
  const int64_t strideT = (int64_t)n * (n / 2 + NB);
  T* Tmp = w + strideD * batch;
  CCAB_CUDA(cudaMemsetAsync(info, 0, sizeof(int) * batch, stream));

  for (int jb = 0; jb < nblk; ++jb) {
    const int j0 = jb * NB, nb = std::min(NB, n - j0);
    int rc = potrf_inv_block<T>(A + (size_t)j0 * lda + j0, lda, strideA, nb, j0, Dinv + (size_t)jb * NB * NB, strideD,
                                piv_tol, piv_tol_dev, info, batch, stream);
    if (rc) return rc;
    const int rows = n - j0 - nb;
    if (rows <= 0) continue;
    GemmArgs<T> g;   // panel: P = A_panel * Dinv_jj^T   (in place: a tile reads its rows completely before writing)
    g.transa = 0; g.transb = 1; g.m = rows; g.n = nb; g.k = nb;
    g.A = A + (size_t)(j0 + nb) * lda + j0; g.lda = lda; g.strideA = strideA;
    g.B = Dinv + (size_t)jb * NB * NB; g.ldb = NB; g.strideB = strideD;
    g.C = A + (size_t)(j0 + nb) * lda + j0; g.ldc = lda; g.strideC = strideA;
    g.batch = batch;
    rc = potrf_panel_gemm<T>(g, Tmp, strideT, stream);
    if (rc) return rc;
    GemmArgs<T> u;   // trailing: A22 -= P P^T, lower tiles
    u.transa = 0; u.transb = 1; u.m = rows; u.n = rows; u.k = nb; u.alpha = T(-1); u.beta = T(1);
    u.A = g.C; u.lda = lda; u.strideA = strideA;
    u.B = g.C; u.ldb = lda; u.strideB = strideA;
    u.C = A + (size_t)(j0 + nb) * lda + (j0 + nb); u.ldc = lda; u.strideC = strideA;
    u.batch = batch; u.lower_only = 1;
    rc = xgemm<T>(u, stream);
    if (rc) return rc;
  }

  // ---- Linv: diagonal blocks, then off-diagonal blocks level by level ----
  {
    const size_t total = (size_t)n * n;
    dim3 grid((unsigned)std::min<size_t>((total + 255) / 256, 1184), (unsigned)batch);
    linv_init_kernel<T><<<grid, 256, 0, stream>>>(Linv, ldi, strideLinv, n, NB, Dinv, strideD);
    count_launches(1);
    CCAB_CUDA(cudaGetLastError());
  }
  for (int64_t s = NB; s < n; s *= 2) {
    const int npairs_all = (int)ceil_div(n, 2 * s);
    // pairs whose B block is a full s x s block can share one batched launch; a ragged last pair goes alone
    int nfull = 0;
    for (int i = 0; i < npairs_all; ++i)
      if ((2 * i + 2) * s <= n) nfull = i + 1;
    for (int pass = 0; pass < 2; ++pass) {
      int i0, np;
      int64_t bs;
      if (pass == 0) {
        if (nfull == 0) continue;
        i0 = 0; np = nfull; bs = s;
      } else {
        if (nfull == npairs_all) continue;
        i0 = nfull; np = 1;
        bs = n - (2 * (int64_t)i0 + 1) * s;
        if (bs <= 0) continue;
      }
      const int64_t a0 = 2 * (int64_t)i0 * s, b0 = a0 + s;
      const int64_t pair_stride_a = 2 * s * (lda + 1), pair_stride_i = 2 * s * (ldi + 1);
      GemmArgs<T> g1;   // Tmp = L[B, A] * Linv[A, A]
      g1.m = (int)bs; g1.n = (int)s; g1.k = (int)s;
      g1.A = A + (size_t)b0 * lda + a0; g1.lda = lda; g1.strideA = pair_stride_a; g1.strideA2 = strideA;
      g1.B = Linv + (size_t)a0 * ldi + a0; g1.ldb = ldi; g1.strideB = pair_stride_i; g1.strideB2 = strideLinv;
      g1.C = Tmp + (size_t)i0 * s * s; g1.ldc = s; g1.strideC = s * s; g1.strideC2 = strideT;
      g1.batch = np; g1.batch2 = batch;
      int rc = xgemm<T>(g1, stream);
      if (rc) return rc;
      GemmArgs<T> g2;   // Linv[B, A] = -Linv[B, B] * Tmp
      g2.m = (int)bs; g2.n = (int)s; g2.k = (int)bs; g2.alpha = T(-1);
      g2.A = Linv + (size_t)b0 * ldi + b0; g2.lda = ldi; g2.strideA = pair_stride_i; g2.strideA2 = strideLinv;
      g2.B = g1.C; g2.ldb = s; g2.strideB = s * s; g2.strideB2 = strideT;
      g2.C = Linv + (size_t)b0 * ldi + a0; g2.ldc = ldi; g2.strideC = pair_stride_i; g2.strideC2 = strideLinv;
      g2.batch = np; g2.batch2 = batch;
      rc = xgemm<T>(g2, stream);
      if (rc) return rc;
    }
  }
  return 0;
}

// The panel product overwrites its own A operand.  The tensor-core kernel reads a tile's whole A rows (all of K)
// before its epilogue writes them and no other tile reads those rows, so in place is safe there; the FMA kernel
// tiles N in 64-column blocks whose CTAs would read columns another CTA has already overwritten, so it goes through
// a scratch copy.
template <typename T>
int potrf_panel_gemm(const GemmArgs<T>& g, T* scratch, int64_t strideScratch, cudaStream_t stream) {
  if (std::is_same<T, float>::value && g.n <= 128) {
    TgemmArgs a;
    a.transa = g.transa; a.transb = g.transb; a.m = g.m; a.n = g.n; a.k = g.k;
    a.A = reinterpret_cast<const float*>(g.A); a.lda = g.lda; a.strideA = g.strideA;
    a.B = reinterpret_cast<const float*>(g.B); a.ldb = g.ldb; a.strideB = g.strideB;
    a.C = reinterpret_cast<float*>(g.C); a.ldc = g.ldc; a.strideC = g.strideC;
    a.batch = g.batch;
    a.force_bn = 128;   // ONE column tile per row block: the in-place condition
    if (tgemm_supported(a)) return tgemm(a, stream);
  }
  if (g.n <= 64) return xgemm<T>(g, stream);      // one 64-column tile covers the panel in every kernel: same argument
  GemmArgs<T> t = g;
  t.C = scratch; t.ldc = g.n; t.strideC = strideScratch;
  int rc = gemm_fma<T>(t, stream);
  if (rc) return rc;
  for (int b = 0; b < g.batch; ++b) {
    CCAB_CUDA(cudaMemcpy2DAsync(g.C + (size_t)b * g.strideC, (size_t)g.ldc * sizeof(T), scratch + (size_t)b * strideScratch,
                                (size_t)g.n * sizeof(T), (size_t)g.n * sizeof(T), (size_t)g.m, cudaMemcpyDeviceToDevice,
                                stream));
  }
  return 0;
}

template int potrf_inv<float>(int, int, float*, int64_t, int64_t, float*, int64_t, int64_t, double, const double*, int*,
                              void*, size_t, cudaStream_t);
template int potrf_inv<double>(int, int, double*, int64_t, int64_t, double*, int64_t, int64_t, double, const double*,
                               int*, void*, size_t, cudaStream_t);
template size_t potrf_inv_workspace_bytes<float>(int, int);
template size_t potrf_inv_workspace_bytes<double>(int, int);
template int potrf_inv_block_size<float>();
template int potrf_inv_block_size<double>();
template int potrf_inv_block<float>(float*, int64_t, int64_t, int, int, float*, int64_t, double, const double*, int*,
                                    int, cudaStream_t);
template int potrf_inv_block<double>(double*, int64_t, int64_t, int, int, double*, int64_t, double, const double*, int*,
                                     int, cudaStream_t);

}  // namespace ccab
