// Pairwise kernel matrices K = k(X, Y) in float64 (see ccab_pairwise_kernel in include/ccab200.h).
//
// Inner-product metrics (linear, poly, sigmoid, rbf, cosine): X Y^T on the fp64 tensor pipe (DMMA m8n8k4) in the
// tiling of dgemm_mma_kernel, with the metric applied in the epilogue.  rbf and cosine read per-row squared norms /
// inverse norms from a pre-pass.  Distance metrics (laplacian, chi2, additive_chi2): shared-memory tiles and FMA
// sums over the features.  Each output element is summed over the features in one fixed order, so reruns are
// bit-identical.  The elementwise steps follow sklearn's order of operations (sklearn/metrics/pairwise.py).
#include "kcca.cuh"

#include "common.cuh"

namespace ccab {

template <typename T>
__device__ __forceinline__ double ld64(const T* p) { return (double)__ldg(p); }

__device__ __forceinline__ void kcca_dmma_884(double& c0, double& c1, double a, double b) {
  asm volatile("mma.sync.aligned.m8n8k4.row.col.f64.f64.f64.f64 {%0, %1}, {%2}, {%3}, {%0, %1};"
               : "+d"(c0), "+d"(c1)
               : "d"(a), "d"(b));
}

// out[r] = sum_k x[r,k]^2 (inv == 0) or its inverse square root, 0 for a zero row (inv != 0; sklearn's normalize
// leaves zero rows at zero).  One warp per row; lane-strided partial sums and a butterfly: a fixed order.
template <typename T>
__global__ void __launch_bounds__(256) row_norms_kernel(const T* __restrict__ X, int64_t n, int64_t ldx, int d,
                                                        int inv, double* __restrict__ out) {
  const int64_t r = (int64_t)blockIdx.x * 8 + (threadIdx.x >> 5);
  const int lane = threadIdx.x & 31;
  if (r >= n) return;
  double s = 0.0;
  for (int k = lane; k < d; k += 32) {
    const double v = ld64(X + r * ldx + k);
    s = fma(v, v, s);
  }
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) s += __shfl_xor_sync(0xffffffffu, s, o);
  if (lane == 0) out[r] = inv ? (s > 0.0 ? 1.0 / sqrt(s) : 0.0) : s;
}

struct KernelArgs {
  int64_t nx, ny, ldx, ldy, ldk;
  int d, metric, same;
  double gamma, degree, coef0;
  const double* xn;   // rbf: squared row norms of X; cosine: inverse row norms
  const double* yn;
  double* K;
};

// the metric applied to one inner product v = x_r . y_c (numpy's order of operations, no contraction)
__device__ __forceinline__ double inner_epilogue(const KernelArgs& a, double v, int64_t r, int64_t c) {
  switch (a.metric) {
    case kKernelPoly:
      return pow(__dadd_rn(__dmul_rn(v, a.gamma), a.coef0), a.degree);
    case kKernelSigmoid:
      return tanh(__dadd_rn(__dmul_rn(v, a.gamma), a.coef0));
    case kKernelRbf: {
      // euclidean_distances(squared=True): (-2 x.y + |x|^2) + |y|^2, clamped at 0, exact 0 on the diagonal of X vs X
      double dist = __dadd_rn(__dadd_rn(__dmul_rn(-2.0, v), a.xn[r]), a.yn[c]);
      dist = fmax(dist, 0.0);
      if (a.same && r == c) dist = 0.0;
      return exp(__dmul_rn(dist, -a.gamma));
    }
    case kKernelCosine:
      return __dmul_rn(__dmul_rn(v, a.xn[r]), a.yn[c]);
    default:
      return v;
  }
}

// 64 x 64 output tile of X Y^T, 8 warps x (4 x 2) m8n8 fragments, 16-feature chunks double-buffered through
// registers (the layout of dgemm_mma_kernel with op(A) = X, op(B) = Y^T).
template <typename T>
__global__ void __launch_bounds__(256) kernel_mma_kernel(const KernelArgs a, const T* __restrict__ X,
                                                         const T* __restrict__ Y) {
  constexpr int KC = 16, LDS = 64 + 4;
  __shared__ double As[2][KC][LDS];
  __shared__ double Bs[2][KC][LDS];
  const int64_t m0 = (int64_t)blockIdx.y * 64, n0 = (int64_t)blockIdx.x * 64;
  const int d = a.d;
  const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
  const int wm = (warp & 1) * 32, wn = (warp >> 1) * 16;
  const int gq = lane >> 2, tq = lane & 3;
  const int kk = tid & 15, rr0 = tid >> 4;

  double ra[4], rb[4];
  auto load_regs = [&](int k0) {
#pragma unroll
    for (int i = 0; i < 4; ++i) {
      const int64_t rr = rr0 + 16 * i;
      const bool kin = k0 + kk < d;
      ra[i] = (kin && m0 + rr < a.nx) ? ld64(X + (m0 + rr) * a.ldx + k0 + kk) : 0.0;
      rb[i] = (kin && n0 + rr < a.ny) ? ld64(Y + (n0 + rr) * a.ldy + k0 + kk) : 0.0;
    }
  };
  auto store_regs = [&](int buf) {
#pragma unroll
    for (int i = 0; i < 4; ++i) {
      As[buf][kk][rr0 + 16 * i] = ra[i];
      Bs[buf][kk][rr0 + 16 * i] = rb[i];
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
  for (int k0 = 0; k0 < d; k0 += KC) {
    const bool more = k0 + KC < d;
    if (more) load_regs(k0 + KC);
#pragma unroll
    for (int k4 = 0; k4 < KC; k4 += 4) {
      double fa[4], fb[2];
#pragma unroll
      for (int i = 0; i < 4; ++i) fa[i] = As[buf][k4 + tq][wm + 8 * i + gq];
#pragma unroll
      for (int j = 0; j < 2; ++j) fb[j] = Bs[buf][k4 + tq][wn + 8 * j + gq];
#pragma unroll
      for (int i = 0; i < 4; ++i)
#pragma unroll
        for (int j = 0; j < 2; ++j) kcca_dmma_884(acc[i][j][0], acc[i][j][1], fa[i], fb[j]);
    }
    if (more) {
      store_regs(buf ^ 1);   // the other buffer was last read one iteration ago (the barrier below separates them)
      __syncthreads();
      buf ^= 1;
    }
  }
#pragma unroll
  for (int i = 0; i < 4; ++i)
#pragma unroll
    for (int j = 0; j < 2; ++j)
#pragma unroll
      for (int e = 0; e < 2; ++e) {
        const int64_t r = m0 + wm + 8 * i + gq, c = n0 + wn + 8 * j + 2 * tq + e;
        if (r < a.nx && c < a.ny) a.K[r * a.ldk + c] = inner_epilogue(a, acc[i][j][e], r, c);
      }
}

// 64 x 64 output tile of a distance metric, 16-feature chunks staged in shared memory, 4 x 4 outputs per thread.
// Padding features are 0 in both operands and add exactly nothing (|0 - 0| = 0; chi2 skips a zero denominator).
template <typename T>
__global__ void __launch_bounds__(256) kernel_dist_kernel(const KernelArgs a, const T* __restrict__ X,
                                                          const T* __restrict__ Y) {
  constexpr int KC = 16, LDS = 64 + 4;
  __shared__ double Xs[KC][LDS];
  __shared__ double Ys[KC][LDS];
  const int64_t m0 = (int64_t)blockIdx.y * 64, n0 = (int64_t)blockIdx.x * 64;
  const int tid = threadIdx.x, tx = tid & 15, ty = tid >> 4;
  const int kk = tid & 15, rr0 = tid >> 4;
  const bool l1 = a.metric == kKernelLaplacian;
  double acc[4][4];
#pragma unroll
  for (int i = 0; i < 4; ++i)
#pragma unroll
    for (int j = 0; j < 4; ++j) acc[i][j] = 0.0;

  for (int k0 = 0; k0 < a.d; k0 += KC) {
#pragma unroll
    for (int i = 0; i < 4; ++i) {
      const int64_t rr = rr0 + 16 * i;
      const bool kin = k0 + kk < a.d;
      Xs[kk][rr] = (kin && m0 + rr < a.nx) ? ld64(X + (m0 + rr) * a.ldx + k0 + kk) : 0.0;
      Ys[kk][rr] = (kin && n0 + rr < a.ny) ? ld64(Y + (n0 + rr) * a.ldy + k0 + kk) : 0.0;
    }
    __syncthreads();
#pragma unroll 4
    for (int k = 0; k < KC; ++k) {
      double x[4], y[4];
#pragma unroll
      for (int i = 0; i < 4; ++i) { x[i] = Xs[k][ty * 4 + i]; y[i] = Ys[k][tx * 4 + i]; }
#pragma unroll
      for (int i = 0; i < 4; ++i)
#pragma unroll
        for (int j = 0; j < 4; ++j) {
          if (l1) {
            acc[i][j] = __dadd_rn(acc[i][j], fabs(__dsub_rn(x[i], y[j])));
          } else {   // sklearn's _chi2_kernel_fast: (x - y)^2 / (x + y) over the features with x + y != 0
            const double num = __dsub_rn(x[i], y[j]), den = __dadd_rn(x[i], y[j]);
            if (den != 0.0) acc[i][j] = __dadd_rn(acc[i][j], __ddiv_rn(__dmul_rn(num, num), den));
          }
        }
    }
    __syncthreads();
  }
#pragma unroll
  for (int i = 0; i < 4; ++i) {
    const int64_t r = m0 + ty * 4 + i;
    if (r >= a.nx) continue;
#pragma unroll
    for (int j = 0; j < 4; ++j) {
      const int64_t c = n0 + tx * 4 + j;
      if (c >= a.ny) continue;
      double v;
      if (l1) v = exp(__dmul_rn(-a.gamma, acc[i][j]));   // exp(-gamma * manhattan_distances)
      else if (a.metric == kKernelChi2) v = exp(__dmul_rn(-acc[i][j], a.gamma));
      else v = -acc[i][j];
      a.K[r * a.ldk + c] = v;
    }
  }
}

static bool needs_norms(int metric) { return metric == kKernelRbf || metric == kKernelCosine; }

size_t pairwise_kernel_workspace_bytes(int metric, int64_t nx, int64_t ny) {
  return needs_norms(metric) ? (size_t)(nx + ny) * sizeof(double) : 0;
}

template <typename T>
int pairwise_kernel(int metric, const T* X, int64_t nx, int64_t ldx, const T* Y, int64_t ny, int64_t ldy, int d,
                    double gamma, double degree, double coef0, double* K, int64_t ldk, void* ws, size_t ws_bytes,
                    cudaStream_t stream) {
  KernelArgs a;
  a.nx = nx; a.ny = ny; a.ldx = ldx; a.ldy = ldy; a.ldk = ldk;
  a.d = d; a.metric = metric;
  a.same = (const void*)X == (const void*)Y && nx == ny && ldx == ldy;   // sklearn's `X is Y` (Y=None)
  a.gamma = gamma; a.degree = degree; a.coef0 = coef0;
  a.xn = a.yn = nullptr;
  a.K = K;
  if (nx == 0 || ny == 0) return 0;
  if (needs_norms(metric)) {
    CCAB_CHECK_ARG(ws && ws_bytes >= pairwise_kernel_workspace_bytes(metric, nx, ny),
                   "pairwise_kernel: workspace of %zu bytes < %zu", ws_bytes,
                   pairwise_kernel_workspace_bytes(metric, nx, ny));
    double* xn = static_cast<double*>(ws);
    double* yn = xn + nx;
    const int inv = metric == kKernelCosine;
    row_norms_kernel<T><<<(unsigned)ceil_div(nx, 8), 256, 0, stream>>>(X, nx, ldx, d, inv, xn);
    count_launches(1);
    if (a.same) {
      yn = xn;
    } else {
      row_norms_kernel<T><<<(unsigned)ceil_div(ny, 8), 256, 0, stream>>>(Y, ny, ldy, d, inv, yn);
      count_launches(1);
    }
    a.xn = xn;
    a.yn = yn;
  }
  dim3 grid((unsigned)ceil_div(ny, 64), (unsigned)ceil_div(nx, 64));
  if (metric <= kKernelCosine) kernel_mma_kernel<T><<<grid, 256, 0, stream>>>(a, X, Y);
  else kernel_dist_kernel<T><<<grid, 256, 0, stream>>>(a, X, Y);
  count_launches(1);
  CCAB_CUDA(cudaGetLastError());
  return 0;
}

template int pairwise_kernel<float>(int, const float*, int64_t, int64_t, const float*, int64_t, int64_t, int, double,
                                    double, double, double*, int64_t, void*, size_t, cudaStream_t);
template int pairwise_kernel<double>(int, const double*, int64_t, int64_t, const double*, int64_t, int64_t, int,
                                     double, double, double, double*, int64_t, void*, size_t, cudaStream_t);

}  // namespace ccab
