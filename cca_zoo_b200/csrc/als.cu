// Sparse / ALS estimators (PLS_ALS, SCCA_PMD, ParkhomenkoCCA, SCCA_Span, SCCA_ADMM) iterated on the block Gram
// matrix G = [X_1 .. X_m]^T [X_1 .. X_m] instead of the samples.
//
// Every quantity the reference's data-space loop forms is a function of G and the weights:
//   target of view i   t = sum_{j != i} X_j w_j,   ||t||^2 = sum_{j,l != i} P_jl,   P_jl = w_j^T G_jl w_l
//   X_i^T t            = sum_{j != i} G_ij w_j
//   deflation          X_i <- X_i Q_i,  Q_i = I - w_i a_i^T / s_i,  a_i = G_ii w_i,  s_i = P_ii
// so one latent dimension is a loop of block mat-vecs R[j][r] = G[r, block j] . w_j over rows of G, with the
// per-view thresholding in between.  One persistent cooperative kernel (als_dimension) runs the whole loop of one
// dimension: the mat-vec phases are spread over every warp of the grid (one warp per row), the per-view
// post-processing (target normalisation, soft thresholding, the PMD bisection, the Span radix select, the ADMM
// steps, the convergence test) runs on CTA 0, and grid barriers separate the phases.  Every reduction has a fixed
// order (warp butterflies, block trees, sums over rows in row order), so repeated fits are bit-identical.
//
// Traffic of one Gauss-Seidel sweep: the update of view i reads the rows of block i (p_i x D), the diagonal block
// product with the new w_i (p_i x p_i) is read in the phase of view i+1 -- G once per sweep.  An ADMM iteration
// (Jacobi order) reads G once.
#include <cooperative_groups.h>

#include <algorithm>

#include "als.cuh"
#include "common.cuh"

namespace ccab {
namespace cg = cooperative_groups;

namespace {

constexpr int kThreads = 1024;
constexpr int kWarps = kThreads / 32;
constexpr int kBisect = 50;  // halvings of the PMD threshold interval (cca_zoo/linear/_iterative.py:246)

struct AlsArgs {
  int kind, m, D, k, d, max_iter;
  int off[kMaxViews + 1];
  double param[kMaxViews];  // PMD: L1 bound tau*sqrt(p); Parkhomenko / ADMM: tau; Span: span
  double mu, tol, n;
  const double* G;     // workspace copy (deflated between dimensions)
  const double* init;  // k x D initial weights (unit per view)
  double* W_out;       // D x k
  int* iters_out;      // k
  double* R;           // m x D block mat-vec results
  double* w;           // D current weights
  double* z;           // D (ADMM)
  double* eta;         // D (ADMM)
  double* f;           // D deflation coefficients a_i / s_i
  double* rowsq;       // D sums of squares of the diagonal-block row segments (ADMM step size)
  double* P;           // m x m
  double* fro;         // m   ||G_ii||_F
  int* done;           // convergence flag of the current sweep
};

__device__ __forceinline__ double warp_sum(double v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
  return v;
}
__device__ __forceinline__ double warp_max(double v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v = fmax(v, __shfl_xor_sync(0xffffffffu, v, o));
  return v;
}

// Block-wide sum (or max), returned to every thread; fixed order: per-thread partial, warp butterfly, warp 0 tree.
template <bool MAX>
__device__ double block_reduce(double v, double* red) {
  const int lane = threadIdx.x & 31, wid = threadIdx.x >> 5;
  v = MAX ? warp_max(v) : warp_sum(v);
  __syncthreads();  // red may still be read by the previous reduction
  if (lane == 0) red[wid] = v;
  __syncthreads();
  if (wid == 0) {
    double x = red[lane];
    x = MAX ? warp_max(x) : warp_sum(x);
    if (lane == 0) red[kWarps] = x;
  }
  __syncthreads();
  return red[kWarps];
}

__device__ __forceinline__ double soft(double x, double t) { return copysign(fmax(fabs(x) - t, 0.0), x); }

// R[j][r] = G[r, block j] . w_j for the rows of up to two row ranges [r0, r0 + n0) (blocks in mask0) and
// [r1, r1 + n1) (blocks in mask1); one warp per row, four independent accumulators per lane.  With `rowsq` the warp
// also stores the sum of squares of the row's diagonal-block segment.
__device__ void matvec(const AlsArgs& a, int r0, int n0, unsigned mask0, int r1, int n1, unsigned mask1,
                       bool rowsq) {
  const int lane = threadIdx.x & 31;
  const int gwarp = (blockIdx.x * blockDim.x + threadIdx.x) >> 5;
  const int nwarps = (gridDim.x * blockDim.x) >> 5;
  for (int t = gwarp; t < n0 + n1; t += nwarps) {
    const int r = t < n0 ? r0 + t : r1 + (t - n0);
    const unsigned mask = t < n0 ? mask0 : mask1;
    const double* row = a.G + (size_t)r * a.D;
    for (int j = 0; j < a.m; ++j) {
      if (!((mask >> j) & 1u)) continue;
      const int o = a.off[j], p = a.off[j + 1] - o;
      const double* g = row + o;
      const double* w = a.w + o;
      double s0 = 0.0, s1 = 0.0, s2 = 0.0, s3 = 0.0, q = 0.0;
      int c = lane;
      for (; c + 96 < p; c += 128) {
        const double g0 = __ldg(g + c), g1 = __ldg(g + c + 32), g2 = __ldg(g + c + 64), g3 = __ldg(g + c + 96);
        s0 = fma(g0, w[c], s0);
        s1 = fma(g1, w[c + 32], s1);
        s2 = fma(g2, w[c + 64], s2);
        s3 = fma(g3, w[c + 96], s3);
        if (rowsq) q += (g0 * g0 + g1 * g1) + (g2 * g2 + g3 * g3);
      }
      for (; c < p; c += 32) {
        const double g0 = __ldg(g + c);
        s0 = fma(g0, w[c], s0);
        if (rowsq) q += g0 * g0;
      }
      const double s = warp_sum((s0 + s1) + (s2 + s3));
      if (lane == 0) a.R[(size_t)j * a.D + r] = s;
      if (rowsq && r >= o && r < o + p) {
        q = warp_sum(q);
        if (lane == 0) a.rowsq[r] = q;
      }
    }
  }
}

// CTA 0: P_jl = w_j^T R[l][rows of j] for all pairs (R from a full mat-vec pass)
__device__ void all_pairs(const AlsArgs& a, double* red) {
  for (int j = 0; j < a.m; ++j)
    for (int l = j; l < a.m; ++l) {
      double s = 0.0;
      for (int r = a.off[j] + threadIdx.x; r < a.off[j + 1]; r += blockDim.x) s = fma(a.w[r], a.R[(size_t)l * a.D + r], s);
      s = block_reduce<false>(s, red);
      if (threadIdx.x == 0) a.P[j * a.m + l] = a.P[l * a.m + j] = s;
    }
  __syncthreads();
}

// CTA 0: xs[0..p) = X_i^T t / ||t|| (unnormalised when ||t|| <= 1e-12, as the reference)
__device__ void target(const AlsArgs& a, int i, double* xs) {
  double tn2 = 0.0;
  for (int j = 0; j < a.m; ++j)
    for (int l = 0; l < a.m; ++l)
      if (j != i && l != i) tn2 += a.P[j * a.m + l];
  const double tn = sqrt(fmax(tn2, 0.0));
  const int o = a.off[i], p = a.off[i + 1] - o;
  for (int r = threadIdx.x; r < p; r += blockDim.x) {
    double x = 0.0;
    for (int j = 0; j < a.m; ++j)
      if (j != i) x += a.R[(size_t)j * a.D + o + r];
    xs[r] = tn > 1e-12 ? x / tn : x;
  }
  __syncthreads();
}

// CTA 0: xs /= ||xs|| when the norm exceeds 1e-12
__device__ void normalise(double* xs, int p, double* red) {
  double s = 0.0;
  for (int r = threadIdx.x; r < p; r += blockDim.x) s = fma(xs[r], xs[r], s);
  const double nrm = sqrt(block_reduce<false>(s, red));
  if (nrm > 1e-12)
    for (int r = threadIdx.x; r < p; r += blockDim.x) xs[r] /= nrm;
  __syncthreads();
}

// CTA 0: the s-th largest |xs| (1 <= s <= p) by an MSB-first radix select over the bit patterns of the non-negative
// doubles (their unsigned order is their numeric order); integer histogram counts, so the result is exact.
__device__ double kth_largest_abs(const double* xs, int p, int s, unsigned* hist, unsigned long long* sel) {
  unsigned long long prefix = 0ull, mask = 0ull;
  unsigned remaining = (unsigned)s;
  for (int shift = 56; shift >= 0; shift -= 8) {
    for (int b = threadIdx.x; b < 256; b += blockDim.x) hist[b] = 0u;
    __syncthreads();
    for (int r = threadIdx.x; r < p; r += blockDim.x) {
      const unsigned long long key = (unsigned long long)__double_as_longlong(fabs(xs[r]));
      if ((key & mask) == prefix) atomicAdd(&hist[(key >> shift) & 255ull], 1u);
    }
    __syncthreads();
    if (threadIdx.x == 0) {
      int b = 255;
      for (; b > 0 && hist[b] < remaining; --b) remaining -= hist[b];
      sel[0] = (unsigned long long)b;
      sel[1] = remaining;
    }
    __syncthreads();
    prefix |= sel[0] << shift;
    remaining = (unsigned)sel[1];
    mask |= 255ull << shift;
    __syncthreads();
  }
  return __longlong_as_double((long long)prefix);
}

struct Smem {
  double red[kWarps + 1];
  unsigned hist[256];
  unsigned long long sel[2];
  double dmax;
};

// CTA 0: Gauss-Seidel update of view i from R[j][rows of i] (j != i); `pend` >= 0 names the view whose diagonal
// product R[pend][rows of pend] was formed with its new weights in the phase just finished.
__device__ void gs_update(const AlsArgs& a, int i, int pend, double* xs, Smem& sm) {
  if (pend >= 0) {
    double s = 0.0;
    for (int r = a.off[pend] + threadIdx.x; r < a.off[pend + 1]; r += blockDim.x)
      s = fma(a.w[r], a.R[(size_t)pend * a.D + r], s);
    s = block_reduce<false>(s, sm.red);
    if (threadIdx.x == 0) a.P[pend * a.m + pend] = s;
    __syncthreads();
  }
  const int o = a.off[i], p = a.off[i + 1] - o;
  target(a, i, xs);
  if (a.kind == kAlsParkhomenko) {
    for (int r = threadIdx.x; r < p; r += blockDim.x) xs[r] = soft(xs[r], a.param[i]);
    __syncthreads();
  } else if (a.kind == kAlsSpan) {
    const int s = (int)a.param[i];
    if (s < p) {
      const double thr = kth_largest_abs(xs, p, s, sm.hist, sm.sel);
      for (int r = threadIdx.x; r < p; r += blockDim.x)
        if (!(fabs(xs[r]) >= thr)) xs[r] = 0.0;
      __syncthreads();
    }
  } else if (a.kind == kAlsPmd) {
    double l1 = 0.0, mx = 0.0;
    for (int r = threadIdx.x; r < p; r += blockDim.x) {
      l1 += fabs(xs[r]);
      mx = fmax(mx, fabs(xs[r]));
    }
    l1 = block_reduce<false>(l1, sm.red);
    const double bound = a.param[i];
    if (l1 > bound) {
      double lo = 0.0, hi = block_reduce<true>(mx, sm.red);
      for (int it = 0; it < kBisect; ++it) {
        const double mid = (lo + hi) / 2.0;
        double s = 0.0;
        for (int r = threadIdx.x; r < p; r += blockDim.x) s += fmax(fabs(xs[r]) - mid, 0.0);
        if (block_reduce<false>(s, sm.red) > bound) lo = mid;
        else hi = mid;
      }
      const double thr = (lo + hi) / 2.0;
      for (int r = threadIdx.x; r < p; r += blockDim.x) xs[r] = soft(xs[r], thr);
      __syncthreads();
    }
  }
  normalise(xs, p, sm.red);
  double dd = 0.0;
  for (int r = threadIdx.x; r < p; r += blockDim.x) {
    const double e = xs[r] - a.w[o + r];
    dd = fma(e, e, dd);
    a.w[o + r] = xs[r];
  }
  dd = block_reduce<false>(dd, sm.red);
  if (threadIdx.x == 0) sm.dmax = fmax(sm.dmax, sqrt(dd));
  for (int j = 0; j < a.m; ++j) {
    if (j == i) continue;
    double s = 0.0;
    for (int r = threadIdx.x; r < p; r += blockDim.x) s = fma(a.w[o + r], a.R[(size_t)j * a.D + o + r], s);
    s = block_reduce<false>(s, sm.red);
    if (threadIdx.x == 0) a.P[i * a.m + j] = a.P[j * a.m + i] = s;
  }
  __syncthreads();
}

// CTA 0: one ADMM iteration (Jacobi order: every target from the weights at the start) from a full R pass
__device__ void admm_update(const AlsArgs& a, double* xs, Smem& sm) {
  all_pairs(a, sm.red);
  for (int i = 0; i < a.m; ++i) {
    const int o = a.off[i], p = a.off[i + 1] - o;
    target(a, i, xs);
    const double step = a.fro[i] / a.n + a.mu, thr = a.param[i] / a.mu;
    double zz = 0.0;
    for (int r = threadIdx.x; r < p; r += blockDim.x) {
      const double wi = a.w[o + r], ei = a.eta[o + r];
      const double g = a.R[(size_t)i * a.D + o + r] - xs[r] + a.mu * (wi - a.z[o + r] + ei);
      const double wt = wi - g / step;
      const double zi = soft(wt + ei, thr);
      xs[r] = wt;
      a.z[o + r] = zi;
      zz = fma(zi, zi, zz);
    }
    const double zn = sqrt(block_reduce<false>(zz, sm.red));
    double dd = 0.0;
    for (int r = threadIdx.x; r < p; r += blockDim.x) {
      double zi = a.z[o + r];
      if (zn > 1.0) zi /= zn;
      a.z[o + r] = zi;
      a.eta[o + r] = a.eta[o + r] + xs[r] - zi;
      const double e = zi - a.w[o + r];
      dd = fma(e, e, dd);
    }
    dd = block_reduce<false>(dd, sm.red);
    if (threadIdx.x == 0) sm.dmax = fmax(sm.dmax, sqrt(dd));
  }
  for (int r = threadIdx.x; r < a.D; r += blockDim.x) a.w[r] = a.z[r];
  __syncthreads();
}

__global__ void __launch_bounds__(kThreads, 1) als_dimension(AlsArgs a) {
  extern __shared__ double xs[];  // CTA 0: the vector of the view being updated
  __shared__ Smem sm;
  cg::grid_group grid = cg::this_grid();
  const bool lead = blockIdx.x == 0;
  const unsigned all = (1u << a.m) - 1u;
  const bool admm = a.kind == kAlsAdmm;

  for (int r = blockIdx.x * blockDim.x + threadIdx.x; r < a.D; r += gridDim.x * blockDim.x) {
    const double v = a.init[(size_t)a.d * a.D + r];
    a.w[r] = v;
    a.z[r] = v;
    a.eta[r] = 0.0;
  }
  grid.sync();
  matvec(a, 0, a.D, all, 0, 0, 0u, admm);
  grid.sync();
  if (lead) {
    all_pairs(a, sm.red);
    if (admm)
      for (int i = 0; i < a.m; ++i) {
        double s = 0.0;
        for (int r = a.off[i] + threadIdx.x; r < a.off[i + 1]; r += blockDim.x) s += a.rowsq[r];
        s = block_reduce<false>(s, sm.red);
        if (threadIdx.x == 0) a.fro[i] = sqrt(s);
      }
  }

  int iters = 0;
  for (int it = 0; it < a.max_iter; ++it) {
    if (lead && threadIdx.x == 0) sm.dmax = 0.0;
    if (admm) {
      if (it > 0) {
        matvec(a, 0, a.D, all, 0, 0, 0u, false);
        grid.sync();
      }
      if (lead) admm_update(a, xs, sm);
    } else {
      for (int i = 0; i < a.m; ++i) {
        const int prev = i > 0 ? i - 1 : a.m - 1;
        const bool fresh = it == 0 && i == 0;  // R of view 0 comes from the full pass
        if (!fresh) {
          // rows of view i against the other blocks, and the diagonal block of the view just updated
          matvec(a, a.off[i], a.off[i + 1] - a.off[i], all & ~(1u << i), a.off[prev], a.off[prev + 1] - a.off[prev],
                 1u << prev, false);
          grid.sync();
        }
        if (lead) gs_update(a, i, fresh ? -1 : prev, xs, sm);
        if (i + 1 < a.m) grid.sync();
      }
    }
    if (lead && threadIdx.x == 0) *a.done = sm.dmax < a.tol ? 1 : 0;
    grid.sync();
    iters = it + 1;
    if (*(volatile int*)a.done) break;
  }

  // final weights: Y = G E (= R), S = E^T G E (= P) and F for the deflation of the next dimension
  matvec(a, 0, a.D, all, 0, 0, 0u, false);
  grid.sync();
  if (lead) {
    all_pairs(a, sm.red);
    for (int i = 0; i < a.m; ++i) {
      const double s = a.P[i * a.m + i];
      for (int r = a.off[i] + threadIdx.x; r < a.off[i + 1]; r += blockDim.x) {
        a.f[r] = s > 1e-12 ? a.R[(size_t)i * a.D + r] / s : 0.0;
        a.W_out[(size_t)r * a.k + a.d] = a.w[r];
      }
    }
    if (threadIdx.x == 0) a.iters_out[a.d] = iters;
  }
}

// G <- G - Y F^T - F Y^T + F S F^T with Y[r][i] = R[i][r], F[r][i] = f[r] for i = view of r (else 0), S = P.
// (a + b) and f[r] f[c] are symmetric in (r, c), so G stays exactly symmetric.
__device__ __forceinline__ int view_of(int x, const ColumnLayout& L) {
  int v = 0;
#pragma unroll
  for (int u = 1; u < kMaxViews; ++u) v += (u < L.n_views && x >= L.coff[u]) ? 1 : 0;
  return v;
}

__global__ void als_deflate(double* G, int D, int m, ColumnLayout L, const double* R, const double* f,
                            const double* P) {
  for (int r = blockIdx.x; r < D; r += gridDim.x) {
    const int vr = view_of(r, L);
    const double fr = f[r];
    double* row = G + (size_t)r * D;
    for (int c = threadIdx.x; c < D; c += blockDim.x) {
      const int vc = view_of(c, L);
      const double fc = f[c];
      const double t = R[(size_t)vc * D + r] * fc + fr * R[(size_t)vr * D + c];
      row[c] = row[c] - t + (fr * fc) * P[vr * m + vc];
    }
  }
}

__global__ void als_scale_copy(const double* __restrict__ src, double* __restrict__ dst, size_t n, double s) {
  for (size_t i = blockIdx.x * (size_t)blockDim.x + threadIdx.x; i < n; i += (size_t)gridDim.x * blockDim.x)
    dst[i] = src[i] * s;
}

struct AlsWorkspace {
  size_t g, r, w, z, eta, f, rowsq, p, fro, done, total;  // byte offsets
};

AlsWorkspace als_workspace(const ColumnLayout& L) {
  auto al = [](size_t x) { return (x + 255) / 256 * 256; };
  const size_t D = (size_t)L.D, m = (size_t)L.n_views;
  AlsWorkspace w;
  w.g = 0;
  w.r = w.g + al(8 * D * D);
  w.w = w.r + al(8 * m * D);
  w.z = w.w + al(8 * D);
  w.eta = w.z + al(8 * D);
  w.f = w.eta + al(8 * D);
  w.rowsq = w.f + al(8 * D);
  w.p = w.rowsq + al(8 * D);
  w.fro = w.p + al(8 * kMaxViews * kMaxViews);
  w.done = w.fro + al(8 * kMaxViews);
  w.total = w.done + 256;
  return w;
}

}  // namespace

size_t als_fit_workspace_bytes(const ColumnLayout& L) { return als_workspace(L).total + 256; }

int als_fit(int kind, const ColumnLayout& L, const double* G, double g_scale, double n_samples, const double* params,
            double mu, const double* init, int k, int max_iter, double tol, double* W_out, int* iters_out, void* ws,
            size_t ws_bytes, cudaStream_t stream) {
  CCAB_CHECK_ARG(ws_bytes >= als_fit_workspace_bytes(L), "workspace too small: %zu < %zu", ws_bytes,
                 als_fit_workspace_bytes(L));
  int maxp = 0;
  for (int v = 0; v < L.n_views; ++v) maxp = L.dims[v] > maxp ? L.dims[v] : maxp;
  const size_t smem = (size_t)maxp * sizeof(double);
  int dev = 0, sms = 0, optin = 0;
  CCAB_CUDA(cudaGetDevice(&dev));
  CCAB_CUDA(cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, dev));
  CCAB_CUDA(cudaDeviceGetAttribute(&optin, cudaDevAttrMaxSharedMemoryPerBlockOptin, dev));
  CCAB_CHECK_ARG(smem + sizeof(Smem) <= (size_t)optin, "a view of %d features does not fit the shared memory of the ALS kernel",
                 maxp);
  CCAB_CUDA(cudaFuncSetAttribute(als_dimension, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
  int per_sm = 0;
  CCAB_CUDA(cudaOccupancyMaxActiveBlocksPerMultiprocessor(&per_sm, als_dimension, kThreads, smem));
  CCAB_CHECK_ARG(per_sm >= 1, "the ALS kernel cannot be resident on this device");

  uintptr_t base = ((uintptr_t)ws + 255) / 256 * 256;
  const AlsWorkspace o = als_workspace(L);
  AlsArgs a;
  a.kind = kind;
  a.m = L.n_views;
  a.D = L.D;
  a.k = k;
  a.max_iter = max_iter;
  for (int v = 0; v <= L.n_views; ++v) a.off[v] = L.coff[v];
  for (int v = 0; v < kMaxViews; ++v) a.param[v] = 0.0;
  for (int v = 0; v < L.n_views; ++v)
    a.param[v] = kind == kAlsPmd ? params[v] * sqrt((double)L.dims[v]) : (kind == kAlsPls ? 0.0 : params[v]);
  a.mu = mu;
  a.tol = tol;
  a.n = n_samples;
  double* Gw = reinterpret_cast<double*>(base + o.g);
  a.G = Gw;
  a.init = init;
  a.W_out = W_out;
  a.iters_out = iters_out;
  a.R = reinterpret_cast<double*>(base + o.r);
  a.w = reinterpret_cast<double*>(base + o.w);
  a.z = reinterpret_cast<double*>(base + o.z);
  a.eta = reinterpret_cast<double*>(base + o.eta);
  a.f = reinterpret_cast<double*>(base + o.f);
  a.rowsq = reinterpret_cast<double*>(base + o.rowsq);
  a.P = reinterpret_cast<double*>(base + o.p);
  a.fro = reinterpret_cast<double*>(base + o.fro);
  a.done = reinterpret_cast<int*>(base + o.done);

  const size_t nn = (size_t)L.D * L.D;
  als_scale_copy<<<(unsigned)std::min<size_t>(ceil_div(nn, 256), 4 * (size_t)sms), 256, 0, stream>>>(G, Gw, nn,
                                                                                                   g_scale);
  CCAB_CUDA(cudaGetLastError());
  int launches = 1;
  for (int d = 0; d < k; ++d) {
    a.d = d;
    void* args[] = {&a};
    CCAB_CUDA(cudaLaunchCooperativeKernel((const void*)als_dimension, dim3(per_sm * sms), dim3(kThreads), args, smem,
                                          stream));
    ++launches;
    if (d + 1 < k) {
      als_deflate<<<(unsigned)std::min(L.D, 8 * sms), 256, 0, stream>>>(Gw, L.D, L.n_views, L, a.R, a.f, a.P);
      CCAB_CUDA(cudaGetLastError());
      ++launches;
    }
  }
  count_launches(launches);
  return 0;
}

}  // namespace ccab
