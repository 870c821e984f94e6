// TCCA on the device (see ccab_tcca_moment / ccab_tcca_fit in include/ccab200.h).
//
// krprod_moment: M_(0) = Z_1^T KR(Z_2, ..., Z_m) / n, the mode-0 unfolding of the whitened cross-moment tensor, as
// one GEMM-shaped contraction over the samples on the fp64 tensor pipe.  The B operand (n x prod_{i>1} p_i) is never
// stored: each 16 x 64 slice of it is generated in shared memory as the elementwise product of the Z_2 .. Z_m entries
// of the slice's samples at every column's multi-index.
//
// CP-ALS: tensorly's unnormalised ALS on M as a fixed launch sequence, 3 m + 1 kernels per iteration (MTTKRP, solve
// and Gram per mode, then the reconstruction error).  Every kernel returns at once when the stop flag of the state
// block is set, so the host enqueues all iterations without reading anything back.
#include "tcca.cuh"

#include <algorithm>

#include "common.cuh"
#include "dense.cuh"

namespace ccab {

int tcca_check_dims(int n_views, const int64_t* dims) {
  CCAB_CHECK_ARG(dims && n_views >= 2 && n_views <= kTccaMaxViews, "TCCA needs 2 to %d views, got n_views = %d",
                 kTccaMaxViews, n_views);
  int64_t prod = 1;
  for (int i = 0; i < n_views; ++i) {
    CCAB_CHECK_ARG(dims[i] >= 1, "view %d has width %lld", i, (long long)dims[i]);
    prod *= dims[i];
    CCAB_CHECK_ARG(prod <= kTccaMaxEntries, "the tensor has more than 2^25 entries (prod of the view widths)");
  }
  return 0;
}

// ---------------------------------------------------------------------------------------------------------------
// Khatri-Rao contraction
// ---------------------------------------------------------------------------------------------------------------
struct KrArgs {
  const double* Z[kTccaMaxViews];
  int64_t ld[kTccaMaxViews];
  int p[kTccaMaxViews];
  int nv;
  int64_t n, kchunk;
  int p1, P;          // M is p1 x P (P = prod_{i>1} p_i)
  double scale;
  double* M;
  double* partial;    // nsplit > 1: [split][p1][P] slabs
};

__device__ __forceinline__ void tcca_dmma_884(double& c0, double& c1, double a, double b) {
  asm volatile("mma.sync.aligned.m8n8k4.row.col.f64.f64.f64.f64 {%0, %1}, {%2}, {%3}, {%0, %1};"
               : "+d"(c0), "+d"(c1)
               : "d"(a), "d"(b));
}

// 64 x 64 output tile, 8 warps x (4 x 2) m8n8 fragments, 16 samples per k step, register double buffering (the
// tiling of dgemm_mma_kernel).  blockIdx.z is the split of the samples.
__global__ void __launch_bounds__(256) krprod_moment_kernel(const KrArgs a) {
  constexpr int KC = 16, LDS = 64 + 4;
  __shared__ double As[2][KC][LDS];
  __shared__ double Bs[2][KC][LDS];
  const int m0 = blockIdx.y * 64, n0 = blockIdx.x * 64;
  const int64_t kbeg = (int64_t)blockIdx.z * a.kchunk;
  const int64_t kend = min(a.n, kbeg + a.kchunk);
  const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
  const int wm = (warp & 1) * 32, wn = (warp >> 1) * 16;
  const int gq = lane >> 2, tq = lane & 3;
  const int mm = tid & 63, kk0 = tid >> 6;       // row mm of the A slice, column mm of the B slice
  const bool row_ok = m0 + mm < a.p1;
  const bool col_ok = n0 + mm < a.P;
  // the multi-index of this thread's B column, once: C-order flattening of (i_2, ..., i_m), the last view fastest
  int idx[kTccaMaxViews];
  {
    int rest = col_ok ? n0 + mm : 0;
#pragma unroll
    for (int v = kTccaMaxViews - 1; v >= 1; --v) {
      idx[v] = 0;
      if (v < a.nv) {
        idx[v] = rest % a.p[v];
        rest /= a.p[v];
      }
    }
  }

  double ra[4], rb[4];
  auto load_regs = [&](int64_t k0) {
#pragma unroll
    for (int i = 0; i < 4; ++i) {
      const int64_t s = k0 + kk0 + 4 * i;
      const bool in = s < kend;
      ra[i] = (in && row_ok) ? a.Z[0][s * a.ld[0] + m0 + mm] : 0.0;
      double b = 0.0;
      if (in && col_ok) {
        b = a.Z[1][s * a.ld[1] + idx[1]];
#pragma unroll
        for (int v = 2; v < kTccaMaxViews; ++v)
          if (v < a.nv) b *= a.Z[v][s * a.ld[v] + idx[v]];
      }
      rb[i] = b;
    }
  };
  auto store_regs = [&](int buf) {
#pragma unroll
    for (int i = 0; i < 4; ++i) {
      As[buf][kk0 + 4 * i][mm] = ra[i];
      Bs[buf][kk0 + 4 * i][mm] = rb[i];
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
  for (int64_t k0 = kbeg; k0 < kend; k0 += KC) {
    const bool more = k0 + KC < kend;
    if (more) load_regs(k0 + KC);
#pragma unroll
    for (int kk = 0; kk < KC; kk += 4) {
      double fa[4], fb[2];
#pragma unroll
      for (int i = 0; i < 4; ++i) fa[i] = As[buf][kk + tq][wm + 8 * i + gq];
#pragma unroll
      for (int j = 0; j < 2; ++j) fb[j] = Bs[buf][kk + tq][wn + 8 * j + gq];
#pragma unroll
      for (int i = 0; i < 4; ++i)
#pragma unroll
        for (int j = 0; j < 2; ++j) tcca_dmma_884(acc[i][j][0], acc[i][j][1], fa[i], fb[j]);
    }
    if (more) {
      store_regs(buf ^ 1);
      __syncthreads();
      buf ^= 1;
    }
  }
  double* out = a.partial ? a.partial + (size_t)blockIdx.z * a.p1 * a.P : a.M;
  const double f = a.partial ? 1.0 : a.scale;
#pragma unroll
  for (int i = 0; i < 4; ++i)
#pragma unroll
    for (int j = 0; j < 2; ++j)
#pragma unroll
      for (int e = 0; e < 2; ++e) {
        const int r = m0 + wm + 8 * i + gq, c = n0 + wn + 8 * j + 2 * tq + e;
        if (r < a.p1 && c < a.P) out[(size_t)r * a.P + c] = f * acc[i][j][e];
      }
}

// M = scale * sum_s partial[s], the splits added in index order
__global__ void krprod_reduce_kernel(const double* __restrict__ partial, int nsplit, size_t count, double scale,
                                     double* __restrict__ M) {
  for (size_t e = blockIdx.x * (size_t)blockDim.x + threadIdx.x; e < count; e += (size_t)gridDim.x * blockDim.x) {
    double s = 0.0;
    for (int q = 0; q < nsplit; ++q) s += partial[(size_t)q * count + e];
    M[e] = scale * s;
  }
}

static int64_t tcca_columns(int n_views, const int64_t* dims) {
  int64_t P = 1;
  for (int i = 1; i < n_views; ++i) P *= dims[i];
  return P;
}

// Sample chunk of each split: a multiple of the 16-sample k step.  Automatic plans split only when the output tiles
// cannot fill the GPU (about two CTAs per SM), keeping at least 1024 samples per split.
static int64_t tcca_kchunk(int n_views, const int64_t* dims, int64_t n, int nsplit) {
  const int64_t tiles = ceil_div(tcca_columns(n_views, dims), 64) * ceil_div(dims[0], 64);
  int64_t ns = nsplit;
  if (ns <= 0) ns = tiles >= 264 ? 1 : std::min<int64_t>(ceil_div(264, tiles), ceil_div(n, 1024));
  ns = std::max<int64_t>(1, std::min<int64_t>(ns, ceil_div(n, 16)));
  return ceil_div(ceil_div(n, ns), 16) * 16;
}

int tcca_moment_plan(int n_views, const int64_t* dims, int64_t n, int nsplit) {
  return (int)ceil_div(n, tcca_kchunk(n_views, dims, n, nsplit));
}

size_t tcca_moment_workspace_bytes(int n_views, const int64_t* dims, int64_t n, int nsplit) {
  const int ns = tcca_moment_plan(n_views, dims, n, nsplit);
  if (ns <= 1) return 0;
  return (size_t)ns * dims[0] * tcca_columns(n_views, dims) * sizeof(double);
}

int tcca_moment(int n_views, const int64_t* dims, int64_t n, const double* const* Z, const int64_t* ldz, double scale,
                int nsplit, double* M, void* ws, size_t ws_bytes, cudaStream_t stream) {
  KrArgs a = {};
  a.nv = n_views;
  for (int i = 0; i < n_views; ++i) {
    a.Z[i] = Z[i];
    a.ld[i] = ldz[i];
    a.p[i] = (int)dims[i];
  }
  a.n = n;
  a.p1 = (int)dims[0];
  a.P = (int)tcca_columns(n_views, dims);
  a.scale = scale;
  a.M = M;
  a.kchunk = tcca_kchunk(n_views, dims, n, nsplit);
  const int ns = (int)ceil_div(n, a.kchunk);
  if (ns > 1) {
    CCAB_CHECK_ARG(ws && ws_bytes >= tcca_moment_workspace_bytes(n_views, dims, n, nsplit),
                   "krprod_moment: workspace too small for %d splits", ns);
    a.partial = static_cast<double*>(ws);
  }
  dim3 grid((unsigned)ceil_div(a.P, 64), (unsigned)ceil_div(a.p1, 64), (unsigned)ns);
  krprod_moment_kernel<<<grid, 256, 0, stream>>>(a);
  count_launches(1);
  if (ns > 1) {
    const size_t count = (size_t)a.p1 * a.P;
    krprod_reduce_kernel<<<(unsigned)std::min<size_t>((count + 255) / 256, 1184), 256, 0, stream>>>(a.partial, ns,
                                                                                                    count, scale, M);
    count_launches(1);
  }
  CCAB_CUDA(cudaGetLastError());
  return 0;
}

// ---------------------------------------------------------------------------------------------------------------
// Khatri-Rao adjoint
// ---------------------------------------------------------------------------------------------------------------
struct KrAdjArgs {
  const double* H[kTccaMaxViews];
  int64_t ldh[kTccaMaxViews];
  double* Y[kTccaMaxViews];
  int64_t ldy[kTccaMaxViews];
  int p[kTccaMaxViews];
  int stride[kTccaMaxViews];    // C-order strides of M
  int nv;
  int64_t n;
  double scale;
  const double* dscale;         // optional device factor
  const double* M;
};

// Y_i = f * KR_{j != i}(H_j) M_(i)^T for the mode i = blockIdx.z: a 64 x 64 tile (samples x mode-i index) of an
// (n x P_i) x (P_i x k_i) product, with the tiling of krprod_moment_kernel.  The reduction runs over the positions
// of the other modes (C order, the last of them fastest) in steps of 16; each thread owns one position q of the step
// and tracks its multi-index as mixed-radix digits, advanced by the digits of 16 with one conditional subtraction per
// digit.  From it the thread generates the KR entries of 4 samples (the A slice) and reads M at 4 mode-i indices
// through the mode-i stride (the B slice): no permuted copy of M.  One CTA owns the whole reduction of its tile, so
// the summation order is fixed.
__global__ void __launch_bounds__(256) krprod_adjoint_kernel(const KrAdjArgs a) {
  constexpr int KC = 16, LDS = 64 + 4;
  __shared__ double As[2][KC][LDS];   // [position][sample]
  __shared__ double Bs[2][KC][LDS];   // [position][mode-i index]
  const int mode = blockIdx.z, ki = a.p[mode];
  const int64_t m0 = (int64_t)blockIdx.x * 64;
  const int n0 = blockIdx.y * 64;
  if (n0 >= ki) return;
  const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
  const int wm = (warp & 1) * 32, wn = (warp >> 1) * 16;
  const int gq = lane >> 2, tq = lane & 3;
  const int q = tid & 15, g = tid >> 4;
  const int64_t si = a.stride[mode];
  int P = 1;
#pragma unroll
  for (int v = 0; v < kTccaMaxViews; ++v)
    if (v < a.nv && v != mode) P *= a.p[v];
  // digits of q and of the step 16 (both mod P) over the other modes
  int dig[kTccaMaxViews], inc[kTccaMaxViews];
  {
    int r0 = q % P, r1 = KC % P;
#pragma unroll
    for (int v = kTccaMaxViews - 1; v >= 0; --v) {
      dig[v] = inc[v] = 0;
      if (v < a.nv && v != mode) {
        dig[v] = r0 % a.p[v];
        r0 /= a.p[v];
        inc[v] = r1 % a.p[v];
        r1 /= a.p[v];
      }
    }
  }

  double ra[4], rb[4];
  auto load_regs = [&](int k0) {
    const bool in = k0 + q < P;
    int64_t off = 0;
#pragma unroll
    for (int v = 0; v < kTccaMaxViews; ++v)
      if (v < a.nv && v != mode) off += (int64_t)dig[v] * a.stride[v];
#pragma unroll
    for (int r = 0; r < 4; ++r) {
      const int64_t s = m0 + g + 16 * r;
      double x = 0.0;
      if (in && s < a.n) {
        x = 1.0;
#pragma unroll
        for (int v = 0; v < kTccaMaxViews; ++v)
          if (v < a.nv && v != mode) x *= a.H[v][s * a.ldh[v] + dig[v]];
      }
      ra[r] = x;
      const int c = n0 + 4 * g + r;
      rb[r] = (in && c < ki) ? a.M[off + c * si] : 0.0;
    }
    int carry = 0;
#pragma unroll
    for (int v = kTccaMaxViews - 1; v >= 0; --v) {
      if (v < a.nv && v != mode) {
        const int d = dig[v] + inc[v] + carry;
        carry = d >= a.p[v];
        dig[v] = carry ? d - a.p[v] : d;
      }
    }
  };
  auto store_regs = [&](int buf) {
#pragma unroll
    for (int r = 0; r < 4; ++r) {
      As[buf][q][g + 16 * r] = ra[r];
      Bs[buf][q][4 * g + r] = rb[r];
    }
  };

  double acc[4][2][2];
#pragma unroll
  for (int i = 0; i < 4; ++i)
#pragma unroll
    for (int j = 0; j < 2; ++j) acc[i][j][0] = acc[i][j][1] = 0.0;

  load_regs(0);
  store_regs(0);
  __syncthreads();
  int buf = 0;
  for (int k0 = 0; k0 < P; k0 += KC) {
    const bool more = k0 + KC < P;
    if (more) load_regs(k0 + KC);
#pragma unroll
    for (int kk = 0; kk < KC; kk += 4) {
      double fa[4], fb[2];
#pragma unroll
      for (int i = 0; i < 4; ++i) fa[i] = As[buf][kk + tq][wm + 8 * i + gq];
#pragma unroll
      for (int j = 0; j < 2; ++j) fb[j] = Bs[buf][kk + tq][wn + 8 * j + gq];
#pragma unroll
      for (int i = 0; i < 4; ++i)
#pragma unroll
        for (int j = 0; j < 2; ++j) tcca_dmma_884(acc[i][j][0], acc[i][j][1], fa[i], fb[j]);
    }
    if (more) {
      store_regs(buf ^ 1);
      __syncthreads();
      buf ^= 1;
    }
  }
  const double f = a.dscale ? a.scale * *a.dscale : a.scale;
  double* Y = a.Y[mode];
  const int64_t ldy = a.ldy[mode];
#pragma unroll
  for (int i = 0; i < 4; ++i)
#pragma unroll
    for (int j = 0; j < 2; ++j)
#pragma unroll
      for (int e = 0; e < 2; ++e) {
        const int64_t r = m0 + wm + 8 * i + gq;
        const int c = n0 + wn + 8 * j + 2 * tq + e;
        if (r < a.n && c < ki) Y[r * ldy + c] = f * acc[i][j][e];
      }
}

int tcca_moment_adjoint(int n_views, const int64_t* dims, int64_t n, const double* M, const double* const* H,
                        const int64_t* ldh, double scale, const double* dscale, double* const* Y, const int64_t* ldy,
                        cudaStream_t stream) {
  KrAdjArgs a = {};
  a.nv = n_views;
  int64_t P = 1, kmax = 1;
  for (int i = n_views - 1; i >= 0; --i) {
    a.H[i] = H[i];
    a.ldh[i] = ldh[i];
    a.Y[i] = Y[i];
    a.ldy[i] = ldy[i];
    a.p[i] = (int)dims[i];
    a.stride[i] = (int)P;
    P *= dims[i];
    kmax = std::max<int64_t>(kmax, dims[i]);
  }
  a.n = n;
  a.scale = scale;
  a.dscale = dscale;
  a.M = M;
  dim3 grid((unsigned)ceil_div(n, 64), (unsigned)ceil_div(kmax, 64), (unsigned)n_views);
  krprod_adjoint_kernel<<<grid, 256, 0, stream>>>(a);
  count_launches(1);
  CCAB_CUDA(cudaGetLastError());
  return 0;
}

// ---------------------------------------------------------------------------------------------------------------
// CP-ALS
// ---------------------------------------------------------------------------------------------------------------
struct AlsArgs {
  int nv, k, P;
  int p[kTccaMaxViews];
  int stride[kTccaMaxViews];     // C-order strides of M
  int64_t foff[kTccaMaxViews];   // offset (doubles) of factor j (p_j x k row-major) in the state block
  int64_t goff;                  // offset of the factor Grams (m x k x k)
  const double* M;
  double* st;
  double* mt;                    // MTTKRP of the current mode, p_j x k
};

__device__ __forceinline__ bool tcca_stopped(const double* st) {
  return st[1] != 0.0 || st[0] >= (double)kTccaMaxIter;
}

// sum over the block of NT threads in a fixed order; every thread gets the result
template <int NT>
__device__ __forceinline__ double tcca_block_sum(double v, double* sh) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
  if ((threadIdx.x & 31) == 0) sh[threadIdx.x >> 5] = v;
  __syncthreads();
  double s = 0.0;
#pragma unroll
  for (int w = 0; w < NT / 32; ++w) s += sh[w];
  __syncthreads();
  return s;
}

// Start factors (blockIdx.y = mode j, blockIdx.x = column r): eigenvector r of M_(j) M_(j)^T with its entry of
// largest |value| (the first on ties) made positive, mode 0 scaled by sigma_r = sqrt(lambda_r); columns r >= p_j
// from the caller's random block.
struct StartArgs {
  const double* E[kTccaMaxViews];   // eigenvectors as rows (p_j x p_j, descending)
  const double* lam0;               // eigenvalues of mode 0
  const double* rand;               // random columns of the modes with p_j < k, p_j x (k - p_j) each, in mode order
  int64_t roff[kTccaMaxViews];
};

__global__ void __launch_bounds__(256) tcca_start_kernel(const AlsArgs a, const StartArgs s) {
  __shared__ double bv[256];
  __shared__ int bi[256];
  const int j = blockIdx.y, r = blockIdx.x, k = a.k, p = a.p[j];
  double* F = a.st + a.foff[j];
  if (r >= p) {
    const double* R = s.rand + s.roff[j];
    for (int i = threadIdx.x; i < p; i += 256) F[(size_t)i * k + r] = R[(size_t)i * (k - p) + (r - p)];
    return;
  }
  const double* u = s.E[j] + (size_t)r * p;
  double best = -1.0;
  int at = p;
  for (int i = threadIdx.x; i < p; i += 256) {
    const double v = fabs(u[i]);
    if (v > best) { best = v; at = i; }
  }
  bv[threadIdx.x] = best;
  bi[threadIdx.x] = at;
  __syncthreads();
  for (int h = 128; h > 0; h >>= 1) {
    if (threadIdx.x < h) {
      const double v2 = bv[threadIdx.x + h];
      const int i2 = bi[threadIdx.x + h];
      if (v2 > bv[threadIdx.x] || (v2 == bv[threadIdx.x] && i2 < bi[threadIdx.x])) {
        bv[threadIdx.x] = v2;
        bi[threadIdx.x] = i2;
      }
    }
    __syncthreads();
  }
  const double lead = u[bi[0]];
  const double sign = lead > 0.0 ? 1.0 : (lead < 0.0 ? -1.0 : 0.0);
  const double sigma = j == 0 ? sqrt(fmax(s.lam0[r], 0.0)) : 1.0;
  for (int i = threadIdx.x; i < p; i += 256) F[(size_t)i * k + r] = u[i] * sign * sigma;
}

// Gram F_j^T F_j of modes j0 + blockIdx.y, entry blockIdx.x (row-major k x k)
__global__ void __launch_bounds__(128) tcca_gram_kernel(const AlsArgs a, int j0) {
  __shared__ double sh[4];
  if (tcca_stopped(a.st)) return;
  const int j = j0 + blockIdx.y, k = a.k, r = blockIdx.x / k, c = blockIdx.x % k;
  const double* F = a.st + a.foff[j];
  double acc = 0.0;
  for (int i = threadIdx.x; i < a.p[j]; i += 128) acc += F[(size_t)i * k + r] * F[(size_t)i * k + c];
  acc = tcca_block_sum<128>(acc, sh);
  if (threadIdx.x == 0) a.st[a.goff + (size_t)j * k * k + blockIdx.x] = acc;
}

// MTTKRP of mode j: mt[i, r] = sum over the slice M[.., i, ..] of M * prod_{l != j} F_l[i_l, r].  Block (i, 16-column
// chunk of r); each thread walks the slice with stride 256, then one fixed-order block reduction per column.
__global__ void __launch_bounds__(256) tcca_mttkrp_kernel(const AlsArgs a, int j) {
  constexpr int RC = 16;
  __shared__ double sh[8];
  if (tcca_stopped(a.st)) return;
  const int i = blockIdx.x, r0 = blockIdx.y * RC, k = a.k;
  const int R = min(RC, k - r0);
  const int pj = a.p[j], sj = a.stride[j];
  const int T = a.P / pj;
  double acc[RC];
#pragma unroll
  for (int q = 0; q < RC; ++q) acc[q] = 0.0;
  for (int t = threadIdx.x; t < T; t += 256) {
    const int hi = t / sj;
    const int off = (hi * pj + i) * sj + (t - hi * sj);
    const double x = a.M[off];
    const double* rows[kTccaMaxViews];
#pragma unroll
    for (int l = 0; l < kTccaMaxViews; ++l)
      rows[l] = (l < a.nv && l != j) ? a.st + a.foff[l] + (size_t)((off / a.stride[l]) % a.p[l]) * k + r0 : nullptr;
#pragma unroll
    for (int q = 0; q < RC; ++q) {
      if (q < R) {
        double w = x;
#pragma unroll
        for (int l = 0; l < kTccaMaxViews; ++l)
          if (rows[l]) w *= rows[l][q];
        acc[q] += w;
      }
    }
  }
#pragma unroll
  for (int q = 0; q < RC; ++q) {
    const double s = tcca_block_sum<256>(acc[q], sh);
    if (threadIdx.x == 0 && q < R) a.mt[(size_t)i * k + r0 + q] = s;
  }
}

// F_j = solve(V^T, mt^T)^T with V the Hadamard product of the other modes' Grams: every block factorises V^T (LU with
// partial pivoting, the LAPACK getrf convention, in shared memory) and solves 64 rows.  An exactly zero pivot (where
// numpy.linalg.solve raises LinAlgError) sets the singular bit and the stop flag.
__global__ void __launch_bounds__(64) tcca_solve_kernel(const AlsArgs a, int j) {
  extern __shared__ double sm[];
  __shared__ int piv[kTccaMaxK];
  __shared__ int singular;
  if (tcca_stopped(a.st)) return;
  const int k = a.k, ld = k + 1, tid = threadIdx.x;
  double* LU = sm;
  double* X = sm + (size_t)k * ld;
  for (int e = tid; e < k * k; e += 64) {
    const int r = e / k, c = e % k;
    double v = 1.0;
    for (int l = 0; l < a.nv; ++l)
      if (l != j) v *= a.st[a.goff + (size_t)l * k * k + (size_t)c * k + r];   // V^T[r][c] = V[c][r]
    LU[r * ld + c] = v;
  }
  if (tid == 0) singular = 0;
  __syncthreads();
  for (int c = 0; c < k; ++c) {
    if (tid == 0) {
      int p = c;
      double best = fabs(LU[c * ld + c]);
      for (int r = c + 1; r < k; ++r)
        if (fabs(LU[r * ld + c]) > best) { best = fabs(LU[r * ld + c]); p = r; }
      piv[c] = p;
      if (LU[p * ld + c] == 0.0) singular = 1;
    }
    __syncthreads();
    const int p = piv[c];
    if (p != c && tid < k) {
      const double t = LU[c * ld + tid];
      LU[c * ld + tid] = LU[p * ld + tid];
      LU[p * ld + tid] = t;
    }
    __syncthreads();
    const double d = LU[c * ld + c];
    if (d != 0.0) {
      for (int r = c + 1 + tid; r < k; r += 64) {
        const double l = LU[r * ld + c] / d;
        LU[r * ld + c] = l;
        for (int cc = c + 1; cc < k; ++cc) LU[r * ld + cc] -= l * LU[c * ld + cc];
      }
    }
    __syncthreads();
  }
  if (singular) {
    if (blockIdx.x == 0 && tid == 0) {
      a.st[2] = 1.0;
      a.st[1] = 1.0;
    }
    return;
  }
  const int row = blockIdx.x * 64 + tid;
  if (row >= a.p[j]) return;
  double* x = X + (size_t)tid * ld;
  for (int c = 0; c < k; ++c) x[c] = a.mt[(size_t)row * k + c];
  for (int c = 0; c < k; ++c) {
    const int p = piv[c];
    if (p != c) {
      const double t = x[c];
      x[c] = x[p];
      x[p] = t;
    }
  }
  for (int c = 0; c < k; ++c)
    for (int r = c + 1; r < k; ++r) x[r] -= LU[r * ld + c] * x[c];
  for (int c = k - 1; c >= 0; --c) {
    double s = x[c];
    for (int cc = c + 1; cc < k; ++cc) s -= LU[c * ld + cc] * x[cc];
    x[c] = s / LU[c * ld + c];
  }
  double* F = a.st + a.foff[j] + (size_t)row * k;
  for (int c = 0; c < k; ++c) F[c] = x[c];
}

// rec = sqrt(|‖M‖² + sum(Hadamard of all Grams) - 2 <mt_{m-1}, F_{m-1}>|) / ‖M‖, the rec history, the stop test
// (|rec_prev - rec| < 1e-8 from the second iteration on) and the iteration count
__global__ void __launch_bounds__(256) tcca_rec_kernel(const AlsArgs a) {
  __shared__ double sh[8];
  if (tcca_stopped(a.st)) return;
  const int k = a.k, last = a.nv - 1;
  double cp = 0.0;
  for (int e = threadIdx.x; e < k * k; e += 256) {
    double w = 1.0;
    for (int l = 0; l < a.nv; ++l) w *= a.st[a.goff + (size_t)l * k * k + e];
    cp += w;
  }
  cp = tcca_block_sum<256>(cp, sh);
  const double* F = a.st + a.foff[last];
  double ip = 0.0;
  for (int e = threadIdx.x; e < a.p[last] * k; e += 256) ip += a.mt[e] * F[e];
  ip = tcca_block_sum<256>(ip, sh);
  if (threadIdx.x == 0) {
    const double norm = a.st[3];
    const double rec = sqrt(fabs(norm * norm + cp - 2.0 * ip)) / norm;
    const int it = (int)a.st[0];
    a.st[kTccaHeader + it] = rec;
    if (it >= 1 && fabs(a.st[kTccaHeader + it - 1] - rec) < 1e-8) a.st[1] = 1.0;
    a.st[0] = (double)(it + 1);
  }
}

static int64_t tcca_sum_dims(int n_views, const int64_t* dims) {
  int64_t s = 0;
  for (int i = 0; i < n_views; ++i) s += dims[i];
  return s;
}

size_t tcca_state_doubles(int n_views, const int64_t* dims, int k) {
  return (size_t)kTccaHeader + kTccaMaxIter + (size_t)k * tcca_sum_dims(n_views, dims) + (size_t)n_views * k * k;
}

size_t tcca_fit_workspace_bytes(int n_views, const int64_t* dims, int k) {
  int64_t pmax = 1;
  for (int i = 0; i < n_views; ++i) pmax = std::max<int64_t>(pmax, dims[i]);
  return (size_t)pmax * k * sizeof(double);
}

int tcca_fit(int n_views, const int64_t* dims, int k, const double* M, const double* const* evecs, const double* lam0,
             const double* rand, int start, int n_iter, double* state, void* ws, size_t ws_bytes, cudaStream_t stream) {
  CCAB_CHECK_ARG(ws && ws_bytes >= tcca_fit_workspace_bytes(n_views, dims, k), "tcca_fit: workspace too small");
  AlsArgs a = {};
  a.nv = n_views;
  a.k = k;
  int64_t P = 1, at = kTccaHeader + kTccaMaxIter;
  for (int i = n_views - 1; i >= 0; --i) {
    a.stride[i] = (int)P;
    P *= dims[i];
  }
  for (int i = 0; i < n_views; ++i) {
    a.p[i] = (int)dims[i];
    a.foff[i] = at;
    at += (int64_t)k * dims[i];
  }
  a.goff = at;
  a.P = (int)P;
  a.M = M;
  a.st = state;
  a.mt = static_cast<double*>(ws);
  const size_t solve_smem = (size_t)(k + 64) * (k + 1) * sizeof(double);
  CCAB_CUDA(cudaFuncSetAttribute(tcca_solve_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)solve_smem));
  if (start) {
    StartArgs s = {};
    int64_t roff = 0;
    for (int i = 0; i < n_views; ++i) {
      CCAB_CHECK_ARG(evecs[i], "tcca_fit: no eigenvectors for mode %d", i);
      s.E[i] = evecs[i];
      s.roff[i] = roff;
      if (dims[i] < k) roff += dims[i] * (k - dims[i]);
    }
    CCAB_CHECK_ARG(lam0 && (roff == 0 || rand), "tcca_fit: the start needs the mode-0 eigenvalues and %lld random "
                   "entries", (long long)roff);
    s.lam0 = lam0;
    s.rand = rand;
    CCAB_CUDA(cudaMemsetAsync(state, 0, (kTccaHeader + kTccaMaxIter) * sizeof(double), stream));
    tcca_start_kernel<<<dim3((unsigned)k, (unsigned)n_views), 256, 0, stream>>>(a, s);
    tcca_gram_kernel<<<dim3((unsigned)(k * k), (unsigned)n_views), 128, 0, stream>>>(a, 0);
    count_launches(2);
    int rc = frobenius_norm<double>(1, (int)P, M, P, state + 3, stream);
    if (rc) return rc;
  }
  for (int it = 0; it < std::min(n_iter, kTccaMaxIter); ++it) {
    for (int j = 0; j < n_views; ++j) {
      tcca_mttkrp_kernel<<<dim3((unsigned)dims[j], (unsigned)ceil_div(k, 16)), 256, 0, stream>>>(a, j);
      tcca_solve_kernel<<<(unsigned)ceil_div(dims[j], 64), 64, solve_smem, stream>>>(a, j);
      tcca_gram_kernel<<<dim3((unsigned)(k * k), 1), 128, 0, stream>>>(a, j);
    }
    tcca_rec_kernel<<<1, 256, 0, stream>>>(a);
    count_launches(3 * n_views + 1);
  }
  CCAB_CUDA(cudaGetLastError());
  return 0;
}

}  // namespace ccab
