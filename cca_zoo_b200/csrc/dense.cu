#include "dense.cuh"

#include <algorithm>

#include "tgemm.cuh"

namespace ccab {

// 64x64 output tile, 16-deep k chunks, 256 threads, 4x4 register tile per thread.  blockIdx.z walks the batch
// (b2 * batch1 + b1).  Exact FMA in T: the path for float64, for shapes TMA cannot address and for tiny products.
template <typename T, int TA, int TB>
__global__ void __launch_bounds__(256) gemm_kernel(const GemmArgs<T> g) {
  constexpr int KC = 16;
  __shared__ T As[KC][64 + 4];
  __shared__ T Bs[KC][64 + 4];
  const int m = g.m, n = g.n, k = g.k;
  const int m0 = blockIdx.y * 64, n0 = blockIdx.x * 64;
  if (g.lower_only && n0 >= m0 + 64) return;
  const int b1 = (int)blockIdx.z % g.batch, b2 = (int)blockIdx.z / g.batch;
  const T* __restrict__ A = g.A + (size_t)b1 * g.strideA + (size_t)b2 * g.strideA2;
  const T* __restrict__ B = g.B + (size_t)b1 * g.strideB + (size_t)b2 * g.strideB2;
  const int64_t lda = g.lda, ldb = g.ldb;
  const int tx = threadIdx.x & 15, ty = threadIdx.x >> 4;
  T acc[4][4];
#pragma unroll
  for (int i = 0; i < 4; ++i)
#pragma unroll
    for (int j = 0; j < 4; ++j) acc[i][j] = T(0);

  for (int k0 = 0; k0 < k; k0 += KC) {
    // A tile -> As[kk][mm]
    if (TA) {  // op(A) = A^T : stored k x m, contiguous along m
      const int mm = threadIdx.x & 63, kk0 = threadIdx.x >> 6;
#pragma unroll
      for (int i = 0; i < KC / 4; ++i) {
        const int kk = kk0 + 4 * i;
        As[kk][mm] = (k0 + kk < k && m0 + mm < m) ? A[(size_t)(k0 + kk) * lda + m0 + mm] : T(0);
      }
    } else {  // stored m x k, contiguous along k
      const int kk = threadIdx.x & 15, mm0 = threadIdx.x >> 4;
#pragma unroll
      for (int i = 0; i < 4; ++i) {
        const int mm = mm0 + 16 * i;
        As[kk][mm] = (k0 + kk < k && m0 + mm < m) ? A[(size_t)(m0 + mm) * lda + k0 + kk] : T(0);
      }
    }
    // B tile -> Bs[kk][nn]
    if (TB) {  // op(B) = B^T : stored n x k, contiguous along k
      const int kk = threadIdx.x & 15, nn0 = threadIdx.x >> 4;
#pragma unroll
      for (int i = 0; i < 4; ++i) {
        const int nn = nn0 + 16 * i;
        Bs[kk][nn] = (k0 + kk < k && n0 + nn < n) ? B[(size_t)(n0 + nn) * ldb + k0 + kk] : T(0);
      }
    } else {  // stored k x n, contiguous along n
      const int nn = threadIdx.x & 63, kk0 = threadIdx.x >> 6;
#pragma unroll
      for (int i = 0; i < KC / 4; ++i) {
        const int kk = kk0 + 4 * i;
        Bs[kk][nn] = (k0 + kk < k && n0 + nn < n) ? B[(size_t)(k0 + kk) * ldb + n0 + nn] : T(0);
      }
    }
    __syncthreads();
#pragma unroll
    for (int kk = 0; kk < KC; ++kk) {
      T a[4], b[4];
#pragma unroll
      for (int i = 0; i < 4; ++i) { a[i] = As[kk][ty * 4 + i]; b[i] = Bs[kk][tx * 4 + i]; }
#pragma unroll
      for (int i = 0; i < 4; ++i)
#pragma unroll
        for (int j = 0; j < 4; ++j) acc[i][j] = fma(a[i], b[j], acc[i][j]);
    }
    __syncthreads();
  }
  T* C = g.C ? g.C + (size_t)b1 * g.strideC + (size_t)b2 * g.strideC2 : nullptr;
  T* Ct = g.Ct ? g.Ct + (size_t)b1 * g.strideCt + (size_t)b2 * g.strideCt2 : nullptr;
#pragma unroll
  for (int i = 0; i < 4; ++i) {
    const int r = m0 + ty * 4 + i;
    if (r >= m) continue;
#pragma unroll
    for (int j = 0; j < 4; ++j) {
      const int cidx = n0 + tx * 4 + j;
      if (cidx >= n) continue;
      T v = g.alpha * acc[i][j];
      if (C) {
        if (g.beta != T(0)) v += g.beta * C[(size_t)r * g.ldc + cidx];
        C[(size_t)r * g.ldc + cidx] = v;
      }
      if (Ct) Ct[(size_t)cidx * g.ldct + r] = v;
    }
  }
}

template <typename T>
int gemm_fma(const GemmArgs<T>& g, cudaStream_t stream) {
  CCAB_CHECK_ARG(g.m >= 0 && g.n >= 0 && g.k >= 0 && g.batch >= 1 && g.batch2 >= 1, "bad gemm shape");
  CCAB_CHECK_ARG(g.C || g.Ct, "gemm: no output");
  CCAB_CHECK_ARG(g.C || g.beta == T(0), "gemm: beta != 0 needs C");
  if (g.m == 0 || g.n == 0) return 0;
  dim3 grid((unsigned)ceil_div(g.n, 64), (unsigned)ceil_div(g.m, 64), (unsigned)(g.batch * g.batch2));
  if (!g.transa && !g.transb) gemm_kernel<T, 0, 0><<<grid, 256, 0, stream>>>(g);
  else if (g.transa && !g.transb) gemm_kernel<T, 1, 0><<<grid, 256, 0, stream>>>(g);
  else if (!g.transa && g.transb) gemm_kernel<T, 0, 1><<<grid, 256, 0, stream>>>(g);
  else gemm_kernel<T, 1, 1><<<grid, 256, 0, stream>>>(g);
  count_launches(1);
  CCAB_CUDA(cudaGetLastError());
  return 0;
}
template int gemm_fma<float>(const GemmArgs<float>&, cudaStream_t);
template int gemm_fma<double>(const GemmArgs<double>&, cudaStream_t);

// ---------------------------------------------------------------------------------------------------------------
// float64 GEMM on the fp64 tensor pipe: mma.sync.aligned.m8n8k4.f64 (DMMA; tcgen05 has no f64 kind).  64 x 64 output
// tile, 8 warps x (4 x 2) m8n8 fragments, 16-deep k chunks staged through skewed shared tiles ([k][64 + 8] doubles:
// conflict-free 64-bit fragment loads) and double-buffered through registers (the global loads of chunk c + 1 are in
// flight while chunk c is multiplied).  Same GemmArgs contract as the FMA kernel; it carries the float64 solver stage
// (MCCA / GCCA whitening, K assembly, subspace iteration) that np.cov's upcast imposes
// (cca_zoo/linear/_mcca.py:150-152).
// ---------------------------------------------------------------------------------------------------------------
__device__ __forceinline__ void dmma_884(double& c0, double& c1, double a, double b) {
  asm volatile("mma.sync.aligned.m8n8k4.row.col.f64.f64.f64.f64 {%0, %1}, {%2}, {%3}, {%0, %1};"
               : "+d"(c0), "+d"(c1)
               : "d"(a), "d"(b));
}

template <int TA, int TB>
__global__ void __launch_bounds__(256) dgemm_mma_kernel(const GemmArgs<double> g, int nsplit, int kchunk,
                                                        double* __restrict__ partial) {
  constexpr int KC = 16, LDS = 64 + 4;   // row stride = 8 banks (mod 32): the 4 k-rows x 8 columns of a fragment load hit 32 distinct banks
  __shared__ double As[2][KC][LDS];
  __shared__ double Bs[2][KC][LDS];
  const int m = g.m, n = g.n;
  const int m0 = blockIdx.y * 64, n0 = blockIdx.x * 64;
  if (g.lower_only && n0 >= m0 + 64) return;
  const int split = (int)blockIdx.z % nsplit, bz = (int)blockIdx.z / nsplit;
  const int kbeg = split * kchunk;
  const int k = min(g.k, kbeg + kchunk);        // this CTA reduces over [kbeg, k)
  const int b1 = bz % g.batch, b2 = bz / g.batch;
  const double* __restrict__ A = g.A + (size_t)b1 * g.strideA + (size_t)b2 * g.strideA2;
  const double* __restrict__ B = g.B + (size_t)b1 * g.strideB + (size_t)b2 * g.strideB2;
  const int64_t lda = g.lda, ldb = g.ldb;
  const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
  const int wm = (warp & 1) * 32, wn = (warp >> 1) * 16;
  const int gq = lane >> 2, tq = lane & 3;

  double ra[4], rb[4];
  auto load_regs = [&](int k0) {
    if (TA) {  // stored k x m
      const int mm = tid & 63, kk0 = tid >> 6;
#pragma unroll
      for (int i = 0; i < 4; ++i) {
        const int kk = kk0 + 4 * i;
        ra[i] = (k0 + kk < k && m0 + mm < m) ? A[(size_t)(k0 + kk) * lda + m0 + mm] : 0.0;
      }
    } else {   // stored m x k
      const int kk = tid & 15, mm0 = tid >> 4;
#pragma unroll
      for (int i = 0; i < 4; ++i) {
        const int mm = mm0 + 16 * i;
        ra[i] = (k0 + kk < k && m0 + mm < m) ? A[(size_t)(m0 + mm) * lda + k0 + kk] : 0.0;
      }
    }
    if (TB) {  // stored n x k
      const int kk = tid & 15, nn0 = tid >> 4;
#pragma unroll
      for (int i = 0; i < 4; ++i) {
        const int nn = nn0 + 16 * i;
        rb[i] = (k0 + kk < k && n0 + nn < n) ? B[(size_t)(n0 + nn) * ldb + k0 + kk] : 0.0;
      }
    } else {   // stored k x n
      const int nn = tid & 63, kk0 = tid >> 6;
#pragma unroll
      for (int i = 0; i < 4; ++i) {
        const int kk = kk0 + 4 * i;
        rb[i] = (k0 + kk < k && n0 + nn < n) ? B[(size_t)(k0 + kk) * ldb + n0 + nn] : 0.0;
      }
    }
  };
  auto store_regs = [&](int buf) {
    if (TA) {
      const int mm = tid & 63, kk0 = tid >> 6;
#pragma unroll
      for (int i = 0; i < 4; ++i) As[buf][kk0 + 4 * i][mm] = ra[i];
    } else {
      const int kk = tid & 15, mm0 = tid >> 4;
#pragma unroll
      for (int i = 0; i < 4; ++i) As[buf][kk][mm0 + 16 * i] = ra[i];
    }
    if (TB) {
      const int kk = tid & 15, nn0 = tid >> 4;
#pragma unroll
      for (int i = 0; i < 4; ++i) Bs[buf][kk][nn0 + 16 * i] = rb[i];
    } else {
      const int nn = tid & 63, kk0 = tid >> 6;
#pragma unroll
      for (int i = 0; i < 4; ++i) Bs[buf][kk0 + 4 * i][nn] = rb[i];
    }
  };

  double acc[4][2][2];
#pragma unroll
  for (int i = 0; i < 4; ++i)
#pragma unroll
    for (int j = 0; j < 2; ++j) acc[i][j][0] = acc[i][j][1] = 0.0;

  load_regs(kbeg);
  store_regs(0);
  __syncthreads();
  int buf = 0;
  for (int k0 = kbeg; k0 < k; k0 += KC) {
    const bool more = k0 + KC < k;
    if (more) load_regs(k0 + KC);
#pragma unroll
    for (int kk = 0; kk < KC; kk += 4) {
      double a[4], b[2];
#pragma unroll
      for (int i = 0; i < 4; ++i) a[i] = As[buf][kk + tq][wm + 8 * i + gq];
#pragma unroll
      for (int j = 0; j < 2; ++j) b[j] = Bs[buf][kk + tq][wn + 8 * j + gq];
#pragma unroll
      for (int i = 0; i < 4; ++i)
#pragma unroll
        for (int j = 0; j < 2; ++j) dmma_884(acc[i][j][0], acc[i][j][1], a[i], b[j]);
    }
    if (more) {
      store_regs(buf ^ 1);   // the other buffer was last read one iteration ago (barrier below separates them)
      __syncthreads();
      buf ^= 1;
    }
  }
  if (nsplit > 1) {   // partial tile of this split: [bz][split][m][n], summed in fixed order by the reduce kernel
    double* Pp = partial + ((size_t)bz * nsplit + split) * (size_t)m * n;
#pragma unroll
    for (int i = 0; i < 4; ++i)
#pragma unroll
      for (int j = 0; j < 2; ++j)
#pragma unroll
        for (int e = 0; e < 2; ++e) {
          const int r = m0 + wm + 8 * i + gq, c = n0 + wn + 8 * j + 2 * tq + e;
          if (r < m && c < n) Pp[(size_t)r * n + c] = acc[i][j][e];
        }
    return;
  }
  double* C = g.C ? g.C + (size_t)b1 * g.strideC + (size_t)b2 * g.strideC2 : nullptr;
  double* Ct = g.Ct ? g.Ct + (size_t)b1 * g.strideCt + (size_t)b2 * g.strideCt2 : nullptr;
#pragma unroll
  for (int i = 0; i < 4; ++i)
#pragma unroll
    for (int j = 0; j < 2; ++j)
#pragma unroll
      for (int e = 0; e < 2; ++e) {
        const int r = m0 + wm + 8 * i + gq, c = n0 + wn + 8 * j + 2 * tq + e;
        if (r >= m || c >= n) continue;
        double v = g.alpha * acc[i][j][e];
        if (C) {
          if (g.beta != 0.0) v += g.beta * C[(size_t)r * g.ldc + c];
          C[(size_t)r * g.ldc + c] = v;
        }
        if (Ct) Ct[(size_t)c * g.ldct + r] = v;
      }
}

// C (+ Ct) = alpha * sum_s partial[s] + beta * C, splits added in index order; partial[bz][s] is m x ldp
template <typename T>
__global__ void splitk_reduce_kernel(const GemmArgs<T> g, int nsplit, const T* __restrict__ partial, int64_t ldp) {
  const size_t mn = (size_t)g.m * g.n;
  const size_t slab = (size_t)g.m * ldp;
  const int bz = blockIdx.y, b1 = bz % g.batch, b2 = bz / g.batch;
  T* C = g.C ? g.C + (size_t)b1 * g.strideC + (size_t)b2 * g.strideC2 : nullptr;
  T* Ct = g.Ct ? g.Ct + (size_t)b1 * g.strideCt + (size_t)b2 * g.strideCt2 : nullptr;
  const T* Pp = partial + (size_t)bz * nsplit * slab;
  for (size_t e = blockIdx.x * (size_t)blockDim.x + threadIdx.x; e < mn; e += (size_t)gridDim.x * blockDim.x) {
    const int r = (int)(e / g.n), c = (int)(e % g.n);
    if (g.lower_only && (c / 64) > (r / 64)) continue;
    T acc = T(0);
    for (int s = 0; s < nsplit; ++s) acc += Pp[(size_t)s * slab + (size_t)r * ldp + c];
    T v = (T)g.alpha * acc;
    if (C) {
      if (g.beta != 0.0) v += (T)g.beta * C[(size_t)r * g.ldc + c];
      C[(size_t)r * g.ldc + c] = v;
    }
    if (Ct) Ct[(size_t)c * g.ldct + r] = v;
  }
}

int gemm_dmma(const GemmArgs<double>& g, cudaStream_t stream) {
  CCAB_CHECK_ARG(g.m >= 0 && g.n >= 0 && g.k >= 0 && g.batch >= 1 && g.batch2 >= 1, "bad gemm shape");
  CCAB_CHECK_ARG(g.C || g.Ct, "gemm: no output");
  CCAB_CHECK_ARG(g.C || g.beta == 0.0, "gemm: beta != 0 needs C");
  if (g.m == 0 || g.n == 0) return 0;
  const int64_t tiles = ceil_div(g.n, 64) * ceil_div(g.m, 64) * g.batch * g.batch2;
  // thin products (few output tiles, long reduction) leave most SMs idle: split the reduction when scratch is given
  int nsplit = 1;
  if (g.splitk_ws && tiles < 74 && g.k >= 512) {
    nsplit = (int)std::min<int64_t>(std::min<int64_t>(8, 148 / tiles), g.k / 256);
    const size_t need = (size_t)g.batch * g.batch2 * nsplit * (size_t)g.m * g.n * sizeof(double);
    if (nsplit < 2 || need > g.splitk_ws_bytes) nsplit = 1;
  }
  int kchunk = g.k;
  if (nsplit > 1) {
    kchunk = (int)(ceil_div(ceil_div(g.k, nsplit), 16) * 16);
    nsplit = (int)ceil_div(g.k, kchunk);
  }
  double* partial = static_cast<double*>(g.splitk_ws);
  dim3 grid((unsigned)ceil_div(g.n, 64), (unsigned)ceil_div(g.m, 64), (unsigned)(g.batch * g.batch2 * nsplit));
  if (!g.transa && !g.transb) dgemm_mma_kernel<0, 0><<<grid, 256, 0, stream>>>(g, nsplit, kchunk, partial);
  else if (g.transa && !g.transb) dgemm_mma_kernel<1, 0><<<grid, 256, 0, stream>>>(g, nsplit, kchunk, partial);
  else if (!g.transa && g.transb) dgemm_mma_kernel<0, 1><<<grid, 256, 0, stream>>>(g, nsplit, kchunk, partial);
  else dgemm_mma_kernel<1, 1><<<grid, 256, 0, stream>>>(g, nsplit, kchunk, partial);
  count_launches(1);
  if (nsplit > 1) {
    const size_t mn = (size_t)g.m * g.n;
    dim3 rgrid((unsigned)std::min<size_t>((mn + 255) / 256, 592), (unsigned)(g.batch * g.batch2));
    splitk_reduce_kernel<double><<<rgrid, 256, 0, stream>>>(g, nsplit, partial, g.n);
    count_launches(1);
  }
  CCAB_CUDA(cudaGetLastError());
  return 0;
}

// tensor pipe when the operands are float32 and TMA-addressable and the product is big enough to amortise the
// pipeline fill; exact FMA tiles otherwise
template <>
int xgemm<float>(const GemmArgs<float>& g, cudaStream_t stream) {
  TgemmArgs a;
  a.transa = g.transa; a.transb = g.transb; a.m = g.m; a.n = g.n; a.k = g.k; a.alpha = g.alpha; a.beta = g.beta;
  a.A = g.A; a.lda = g.lda; a.strideA = g.strideA; a.strideA2 = g.strideA2;
  a.B = g.B; a.ldb = g.ldb; a.strideB = g.strideB; a.strideB2 = g.strideB2;
  a.C = g.C; a.ldc = g.ldc; a.strideC = g.strideC; a.strideC2 = g.strideC2;
  a.Ct = g.Ct; a.ldct = g.ldct; a.strideCt = g.strideCt; a.strideCt2 = g.strideCt2;
  a.batch = g.batch; a.batch2 = g.batch2; a.lower_only = g.lower_only;
  const bool big = (int64_t)g.m * g.n * g.k >= ((int64_t)1 << 21) && g.k >= 16;   // >= 128^3: the pipeline fill (~9 us) pays off
  if (big && tgemm_supported(a)) {
    // thin products (few 128 x 64 output tiles, long reduction) occupy a handful of SMs for k / 32 pipeline steps:
    // when the caller lends scratch, run equal k-slices as a batch and add the partial tiles in slice order
    // (deterministic).  Slices along a K-major operand overlap in memory (batch stride < row stride), which TMA
    // tensor maps allow; should the encoder refuse, the unsplit product below still runs.
    const int64_t tiles = ceil_div(g.m, 128) * ceil_div(g.n, 64);
    if (g.splitk_ws && g.batch == 1 && g.batch2 == 1 && !g.lower_only && tiles <= 24 && g.k >= 512) {
      int ns = (int)std::min<int64_t>(std::min<int64_t>(8, 148 / tiles), g.k / 128);
      while (ns >= 2 && (g.k % ns != 0 || (g.k / ns) % 32 != 0)) --ns;
      const int64_t ldp = ceil_div(g.n, 4) * 4;
      const size_t need = (size_t)ns * g.m * ldp * sizeof(float);
      if (ns >= 2 && need <= g.splitk_ws_bytes && (reinterpret_cast<uintptr_t>(g.splitk_ws) & 15) == 0) {
        const int kc = g.k / ns;
        TgemmArgs b = a;
        b.k = kc; b.alpha = 1.0; b.beta = 0.0;
        b.C = static_cast<float*>(g.splitk_ws); b.ldc = ldp; b.strideC = (int64_t)g.m * ldp;
        b.Ct = nullptr;
        b.batch = ns;
        b.strideA = g.transa ? (int64_t)kc * g.lda : kc;
        b.strideB = g.transb ? kc : (int64_t)kc * g.ldb;
        if (tgemm_supported(b) && tgemm(b, stream) == 0) {
          const size_t mn = (size_t)g.m * g.n;
          splitk_reduce_kernel<float><<<(unsigned)std::min<size_t>((mn + 255) / 256, 592), 256, 0, stream>>>(
              g, ns, static_cast<const float*>(g.splitk_ws), ldp);
          count_launches(1);
          CCAB_CUDA(cudaGetLastError());
          return 0;
        }
      }
    }
    return tgemm(a, stream);
  }
  return gemm_fma<float>(g, stream);
}
template <>
int xgemm<double>(const GemmArgs<double>& g, cudaStream_t stream) {
  if (g.k >= 8) return gemm_dmma(g, stream);   // fp64 tensor pipe (DMMA)
  return gemm_fma<double>(g, stream);
}

template <typename T>
__global__ void whiten_rows_kernel(int d, const T* __restrict__ lam, const T* __restrict__ Vt, int64_t ldv, double c,
                                   double floor_add, const T* __restrict__ floor_dev, double scale, double rank_tol,
                                   int max_rank, double lam_floor, T* __restrict__ Wt, int64_t ldw, T* __restrict__ g_out,
                                   int* __restrict__ rank_out) {
  const int j = blockIdx.x;
  const double l0 = fmax((double)lam[0], 0.0);
  const double lj = (double)lam[j];
  const bool keep = (lj > rank_tol * l0) && (j < max_rank);
  const double fl = floor_add + (floor_dev ? (double)floor_dev[0] : 0.0);
  const double g = keep ? 1.0 / sqrt(((1.0 - c) * fmax(lj, lam_floor) + c + fl) * scale) : 0.0;
  for (int i = threadIdx.x; i < d; i += blockDim.x) Wt[(size_t)j * ldw + i] = (T)(g * (double)Vt[(size_t)j * ldv + i]);
  if (threadIdx.x == 0) {
    if (g_out) g_out[j] = (T)g;
    if (rank_out && keep) atomicAdd(rank_out, 1);
  }
}

template <typename T>
int whiten_rows(int d, const T* lam, const T* Vt, int64_t ldv, double c, double floor_add, const T* floor_dev,
                double scale, double rank_tol, int max_rank, double lam_floor, T* Wt, int64_t ldw, T* g_out,
                int* rank_out, cudaStream_t stream) {
  CCAB_CHECK_ARG(d >= 1, "bad dimension");
  if (rank_out) CCAB_CUDA(cudaMemsetAsync(rank_out, 0, sizeof(int), stream));
  whiten_rows_kernel<T><<<d, 128, 0, stream>>>(d, lam, Vt, ldv, c, floor_add, floor_dev, scale, rank_tol, max_rank,
                                               lam_floor, Wt, ldw, g_out, rank_out); count_launches(1);
  CCAB_CUDA(cudaGetLastError());
  return 0;
}
template int whiten_rows<float>(int, const float*, const float*, int64_t, double, double, const float*, double, double,
                                int, double, float*, int64_t, float*, int*, cudaStream_t);
template int whiten_rows<double>(int, const double*, const double*, int64_t, double, double, const double*, double,
                                 double, int, double, double*, int64_t, double*, int*, cudaStream_t);

template <typename T>
__device__ __forceinline__ T pow_code(T v, int code) {
  if (code == 1) return T(1) / v;
  if (code == 2) return T(1) / sqrt(v);
  return v;
}

// columns on grid.x, rows on grid.y with a grid-stride loop: gridDim.y stops at 65535, the row count does not
template <typename T>
__global__ void scale_kernel(int m, int n, const T* __restrict__ A, int64_t lda, const T* __restrict__ r, int r_pow,
                             const T* __restrict__ c, int c_pow, T* __restrict__ B, int64_t ldb) {
  const int j = blockIdx.x * blockDim.x + threadIdx.x;
  if (j >= n) return;
  const T fc = c ? pow_code(c[j], c_pow) : T(1);
  for (int i = blockIdx.y; i < m; i += gridDim.y) {
    T f = T(1);
    if (r) f *= pow_code(r[i], r_pow);
    if (c) f *= fc;
    B[(size_t)i * ldb + j] = A[(size_t)i * lda + j] * f;
  }
}

template <typename T>
int scale_rows_cols(int m, int n, const T* A, int64_t lda, const T* r, int r_pow, const T* c, int c_pow, T* B,
                    int64_t ldb, cudaStream_t stream) {
  CCAB_CHECK_ARG(m >= 0 && n >= 0, "bad shape");
  if (m == 0 || n == 0) return 0;
  const unsigned rows = (unsigned)std::min(m, 65535);
  scale_kernel<T><<<dim3((unsigned)ceil_div(n, 128), rows), 128, 0, stream>>>(m, n, A, lda, r, r_pow, c, c_pow, B,
                                                                              ldb); count_launches(1);
  CCAB_CUDA(cudaGetLastError());
  return 0;
}
template int scale_rows_cols<float>(int, int, const float*, int64_t, const float*, int, const float*, int, float*,
                                    int64_t, cudaStream_t);
template int scale_rows_cols<double>(int, int, const double*, int64_t, const double*, int, const double*, int, double*,
                                     int64_t, cudaStream_t);

// one block per 32 columns; fixed-order reduction over rows (deterministic)
template <typename T>
__global__ void center_columns_kernel(int m, int n, T* __restrict__ A, int64_t lda) {
  __shared__ double part[32][33];
  const int j = blockIdx.x * 32 + (threadIdx.x & 31);
  const int rg = threadIdx.x >> 5;  // 32 row groups
  double acc = 0.0;
  if (j < n)
    for (int i = rg; i < m; i += 32) acc += (double)A[(size_t)i * lda + j];
  part[rg][threadIdx.x & 31] = acc;
  __syncthreads();
  if (rg == 0) {
    double s = 0.0;
    for (int k = 0; k < 32; ++k) s += part[k][threadIdx.x & 31];
    part[0][threadIdx.x & 31] = s / (double)m;
  }
  __syncthreads();
  const T mu = (T)part[0][threadIdx.x & 31];
  if (j < n)
    for (int i = rg; i < m; i += 32) A[(size_t)i * lda + j] -= mu;
}

template <typename T>
int center_columns(int m, int n, T* A, int64_t lda, cudaStream_t stream) {
  if (m == 0 || n == 0) return 0;
  center_columns_kernel<T><<<(unsigned)ceil_div(n, 32), 1024, 0, stream>>>(m, n, A, lda); count_launches(1);
  CCAB_CUDA(cudaGetLastError());
  return 0;
}
template int center_columns<float>(int, int, float*, int64_t, cudaStream_t);
template int center_columns<double>(int, int, double*, int64_t, cudaStream_t);

// one thread per element of a 32-column strip, grid-stride over the rows
template <typename T>
__global__ void row_sub_scale_kernel(int64_t m, int n, T* __restrict__ A, int64_t lda, const T* __restrict__ r,
                                     const T* __restrict__ s) {
  const int j = blockIdx.x * 32 + (threadIdx.x & 31);
  if (j >= n) return;
  const T rj = r[j], sc = s[0];
  for (int64_t i = (int64_t)blockIdx.y * (blockDim.x >> 5) + (threadIdx.x >> 5); i < m;
       i += (int64_t)gridDim.y * (blockDim.x >> 5))
    A[i * lda + j] = (A[i * lda + j] - rj) * sc;
}

template <typename T>
int row_sub_scale(int64_t m, int n, T* A, int64_t lda, const T* r, const T* s, cudaStream_t stream) {
  CCAB_CHECK_ARG(m >= 0 && n >= 0 && lda >= n, "row_sub_scale: bad shape");
  CCAB_CHECK_ARG(r && s, "row_sub_scale: r and s are required");
  if (m == 0 || n == 0) return 0;
  const unsigned gy = (unsigned)std::min<int64_t>(ceil_div(m, 8), 1024);
  row_sub_scale_kernel<T><<<dim3((unsigned)ceil_div(n, 32), gy), 256, 0, stream>>>(m, n, A, lda, r, s);
  count_launches(1);
  CCAB_CUDA(cudaGetLastError());
  return 0;
}
template int row_sub_scale<float>(int64_t, int, float*, int64_t, const float*, const float*, cudaStream_t);
template int row_sub_scale<double>(int64_t, int, double*, int64_t, const double*, const double*, cudaStream_t);

// Two passes in one CTA.  Pass 1 finds max |a| and the exponent e that puts max |a| 2^-e in [0.5, 1); pass 2 sums
// (a 2^-e)^2 in a fixed order and the norm is 2^e sqrt(sum).  The scaling is exact and moves every square by the even
// power 2^-2e, so at ordinary scales the result is sqrt(sum a^2) bit for bit, while the squares can neither overflow
// (entries past 2^511) nor vanish (entries below 2^-537): frob(2^k A) = 2^k frob(A) exactly over the whole range.
template <typename T>
__global__ void frobenius_kernel(int m, int n, const T* __restrict__ A, int64_t lda, T* __restrict__ out) {
  __shared__ double red[32];
  __shared__ int e_s;
  const size_t total = (size_t)m * n;
  double mx = 0.0;
  for (size_t i = threadIdx.x; i < total; i += blockDim.x) mx = fmax(mx, fabs((double)A[(i / n) * lda + (i % n)]));
  for (int o = 16; o > 0; o >>= 1) mx = fmax(mx, __shfl_xor_sync(0xffffffffu, mx, o));
  if ((threadIdx.x & 31) == 0) red[threadIdx.x >> 5] = mx;
  __syncthreads();
  if (threadIdx.x < 32) {
    mx = threadIdx.x < (blockDim.x >> 5) ? red[threadIdx.x] : 0.0;
    for (int o = 16; o > 0; o >>= 1) mx = fmax(mx, __shfl_xor_sync(0xffffffffu, mx, o));
    if (threadIdx.x == 0) {
      int e = 0;                                // zero matrix: sum 0; inf: e = 0 keeps the inf
      if (isfinite(mx) && mx > 0.0) frexp(mx, &e);
      e_s = e;
    }
  }
  __syncthreads();
  const int e = e_s;
  double acc = 0.0;
  for (size_t i = threadIdx.x; i < total; i += blockDim.x) {
    const double v = ldexp((double)A[(i / n) * lda + (i % n)], -e);
    acc += v * v;
  }
  for (int o = 16; o > 0; o >>= 1) acc += __shfl_xor_sync(0xffffffffu, acc, o);
  if ((threadIdx.x & 31) == 0) red[threadIdx.x >> 5] = acc;
  __syncthreads();
  if (threadIdx.x < 32) {
    acc = threadIdx.x < (blockDim.x >> 5) ? red[threadIdx.x] : 0.0;
    for (int o = 16; o > 0; o >>= 1) acc += __shfl_xor_sync(0xffffffffu, acc, o);
    if (threadIdx.x == 0) out[0] = (T)ldexp(sqrt(acc), e);
  }
}

template <typename T>
int frobenius_norm(int m, int n, const T* A, int64_t lda, T* out, cudaStream_t stream) {
  frobenius_kernel<T><<<1, 1024, 0, stream>>>(m, n, A, lda, out); count_launches(1);  // deterministic single-block reduction
  CCAB_CUDA(cudaGetLastError());
  return 0;
}
template int frobenius_norm<float>(int, int, const float*, int64_t, float*, cudaStream_t);
template int frobenius_norm<double>(int, int, const double*, int64_t, double*, cudaStream_t);

}  // namespace ccab
