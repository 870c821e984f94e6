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
// ElasticCCA / SCCA_IPLS (kinds 5, 6) replace the thresholding by a penalised regression of view i on the target,
//   min_w  1/2 w^T Q_i w - b_i^T w + lam_i ||w||_1,   Q_i = G_ii / n + rho_i I,   b_i = X_i^T t / (||t|| n),
// lam_i = alpha_i l1_i, rho_i = alpha_i (1 - l1_i) (sklearn's Lasso / ElasticNet objectives over n) or alpha_i / n
// (Ridge, l1_i = 0: ||y - X w||^2 + alpha ||w||^2).  The target
// of ElasticCCA includes view i itself.  CTA 0 solves it:
//   lam_i == 0   w = V (Lam / n + rho)^+ V^T b with the eigendecomposition G_ii = V Lam V^T of this dimension
//                (jacobi_solve on the host side, once per dimension): the minimum-norm solution when Q_i is singular
//                (always from the second dimension on at alpha = 0: deflation maps the previous w_i to zero);
//   lam_i > 0    cyclic coordinate descent from the current w_i on the rows of G_ii, the gradient Q w - b recomputed
//                exactly after every sweep, until the KKT residual is <= kKktTol * max(1, ||b||_inf).
// SCCA_IPLS then divides by the population std of X_i w, sqrt(w^T G_ii w / n - (mu_i^T w)^2), mu_i the column means
// of the (deflated) view, deflated with the view (mu_i <- mu_i - (mu_i^T w_i) a_i / s_i).
//
// Traffic of one Gauss-Seidel sweep: the update of view i reads the rows of block i (p_i x D), the diagonal block
// product with the new w_i (p_i x p_i) is read in the phase of view i+1 -- G once per sweep.  An ADMM iteration
// (Jacobi order) reads G once.
#include <cooperative_groups.h>

#include <algorithm>
#include <cstring>

#include "als.cuh"
#include "common.cuh"
#include "syevj.cuh"

namespace ccab {
namespace cg = cooperative_groups;

namespace {

constexpr int kThreads = 1024;
constexpr int kWarps = kThreads / 32;
constexpr int kRegThreads = 512;  // CTA size of the regression kinds
constexpr int kBisect = 50;  // halvings of the PMD threshold interval (cca_zoo/linear/_iterative.py:246)
constexpr double kKktTol = 1e-12;  // regression kinds: KKT residual bound relative to max(1, ||b||_inf)
// coordinate-descent sweeps per sub-problem at most: the max_iter of the reference's sklearn Lasso / ElasticNet.  A
// sub-problem that does not reach kKktTol in them is reported (negated sweep count of its dimension).
constexpr int kCdSweeps = 1000;

struct AlsArgs {
  int kind, m, D, k, d, max_iter;
  int off[kMaxViews + 1];
  double param[kMaxViews];  // PMD: L1 bound tau*sqrt(p); Parkhomenko / ADMM: tau; Span: span
  double rho[kMaxViews], lam[kMaxViews];  // ElasticCCA / IPLS: alpha (1 - l1), alpha l1
  double mu, tol, n;  // mu: ADMM penalty; regression kinds: the relative eigenvalue cut of the lam == 0 solve
  int maxp;                                // widest view (the dynamic shared memory holds 3 vectors of it)
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
  const double* V;     // regression kinds, lam == 0: eigenvectors of G_ii as rows, p_i x p_i at V + voff[i]
  const double* ev;    // D: eigenvalues of G_ii (descending per view)
  double* colmean;     // D: IPLS column means of the deflated views
  size_t voff[kMaxViews];
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
// A CTA of fewer than kWarps warps must zero red[] once first: the slots of its missing warps then stay 0 (the regression
// kinds only take maxima of non-negative values).
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
  const bool self = a.kind == kAlsElastic;  // ElasticCCA: the sum of ALL views' scores
  double tn2 = 0.0;
  for (int j = 0; j < a.m; ++j)
    for (int l = 0; l < a.m; ++l)
      if (self || (j != i && l != i)) tn2 += a.P[j * a.m + l];
  const double tn = sqrt(fmax(tn2, 0.0));
  const int o = a.off[i], p = a.off[i + 1] - o;
  for (int r = threadIdx.x; r < p; r += blockDim.x) {
    double x = 0.0;
    for (int j = 0; j < a.m; ++j)
      if (self || j != i) x += a.R[(size_t)j * a.D + o + r];
    xs[r] = tn > 1e-12 ? x / tn : x;
  }
  __syncthreads();
}

// CTA 0: y[r] = sum_c Gd[r * ld + c] x[c] for r < p (one warp per row, lanes over columns)
__device__ void cta_matvec(const double* Gd, int ld, int p, const double* x, double* y) {
  const int lane = threadIdx.x & 31, wid = threadIdx.x >> 5;
  for (int r = wid; r < p; r += (int)(blockDim.x >> 5)) {
    const double* g = Gd + (size_t)r * ld;
    double s0 = 0.0, s1 = 0.0;
    int c = lane;
    for (; c + 32 < p; c += 64) {
      s0 = fma(__ldg(g + c), x[c], s0);
      s1 = fma(__ldg(g + c + 32), x[c + 32], s1);
    }
    if (c < p) s0 = fma(__ldg(g + c), x[c], s0);
    const double s = warp_sum(s0 + s1);
    if (lane == 0) y[r] = s;
  }
  __syncthreads();
}

// CTA 0: the largest KKT residual of min 1/2 w^T Q w - b^T w + lam ||w||_1 at w, g = Q w - b
__device__ double kkt_residual(const double* w, const double* g, int p, double lam, double* red) {
  double r = 0.0;
  for (int c = threadIdx.x; c < p; c += blockDim.x)
    r = fmax(r, w[c] != 0.0 ? fabs(g[c] + copysign(lam, w[c])) : fmax(fabs(g[c]) - lam, 0.0));
  return block_reduce<true>(r, red);
}

// CTA 0: the penalised regression of one view (see the header) on its diagonal block Gd (p x p, leading dimension ld),
// V / ev its eigenvectors (rows) / eigenvalues, w0 its current weights, cm its column means.  In: xs = X_i^T t / ||t||;
// out: xs = the new w_i.  u, g: scratch vectors of p doubles in shared memory.
__device__ void regress(int kind, const double* Gd, int ld, int p, double n, double rho, double lam, double rcond,
                        const double* V, const double* ev, const double* w0, const double* cm, double* xs,
                        double* u, double* g, double* red, double* bcast, int* fail) {
  double bmax = 0.0;
  for (int r = threadIdx.x; r < p; r += blockDim.x) {
    xs[r] /= n;  // b
    bmax = fmax(bmax, fabs(xs[r]));
  }
  bmax = block_reduce<true>(bmax, red);
  if (lam == 0.0) {
    // w = V diag(1 / mu_k) V^T b over the eigenvalues mu_k = ev_k / n + rho above rcond * mu_max
    const double cut = rcond * fmax(ev[0] / n + rho, 0.0);
    cta_matvec(V, p, p, xs, u);
    for (int k = threadIdx.x; k < p; k += blockDim.x) {
      const double mk = ev[k] / n + rho;
      u[k] = mk > cut ? u[k] / mk : 0.0;
    }
    __syncthreads();
    for (int r = threadIdx.x; r < p; r += blockDim.x) {
      double s = 0.0;
      for (int k = 0; k < p; ++k) s = fma(V[(size_t)k * p + r], u[k], s);
      g[r] = s;
    }
    __syncthreads();
    for (int r = threadIdx.x; r < p; r += blockDim.x) xs[r] = g[r];
    __syncthreads();
  } else {
    // cyclic coordinate descent on Q_i from the current w_i (u holds w, g the gradient Q w - b)
    const double tol = kKktTol * fmax(1.0, bmax);
    for (int r = threadIdx.x; r < p; r += blockDim.x) u[r] = w0[r];
    __syncthreads();
    for (int sweep = 0;; ++sweep) {
      cta_matvec(Gd, ld, p, u, g);
      for (int r = threadIdx.x; r < p; r += blockDim.x) g[r] = g[r] / n + rho * u[r] - xs[r];
      __syncthreads();
      if (kkt_residual(u, g, p, lam, red) <= tol) break;
      if (sweep == kCdSweeps) {
        if (threadIdx.x == 0) *fail = 1;
        break;
      }
      for (int j = 0; j < p; ++j) {
        if (threadIdx.x == 0) {
          const double q = Gd[(size_t)j * ld + j] / n + rho;
          const double wj = u[j];
          const double nw = q > 0.0 ? soft(wj * q - g[j], lam) / q : 0.0;
          bcast[0] = nw - wj;
          u[j] = nw;
        }
        __syncthreads();
        const double dl = bcast[0];
        if (dl != 0.0) {
          const double* row = Gd + (size_t)j * ld;
          for (int r = threadIdx.x; r < p; r += blockDim.x) g[r] = fma(dl, row[r] / n + (r == j ? rho : 0.0), g[r]);
        }
        __syncthreads();
      }
    }
    for (int r = threadIdx.x; r < p; r += blockDim.x) xs[r] = u[r];
    __syncthreads();
  }
  if (kind == kAlsIpls) {
    // divide by the population std of the score X_i w when it exceeds 1e-12
    cta_matvec(Gd, ld, p, xs, u);
    double q = 0.0, mw = 0.0;
    for (int r = threadIdx.x; r < p; r += blockDim.x) {
      q = fma(xs[r], u[r], q);
      mw = fma(cm[r], xs[r], mw);
    }
    q = block_reduce<false>(q, red);
    mw = block_reduce<false>(mw, red);
    const double sd = sqrt(fmax(q / n - mw * mw, 0.0));
    if (sd > 1e-12)
      for (int r = threadIdx.x; r < p; r += blockDim.x) xs[r] /= sd;
    __syncthreads();
  }
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
  double bcast;
  int cd_fail;  // a coordinate descent of this dimension stopped at kCdSweeps
};

// CTA 0: Gauss-Seidel update of view i from R[j][rows of i] (j != i); `pend` >= 0 names the view whose diagonal
// product R[pend][rows of pend] was formed with its new weights in the phase just finished.
template <bool REG>
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
  } else if (REG) {
    regress(a.kind, a.G + (size_t)o * a.D + o, a.D, p, a.n, a.rho[i], a.lam[i], a.mu, a.V + a.voff[i], a.ev + o,
            a.w + o, a.colmean + o, xs, xs + a.maxp, xs + 2 * a.maxp, sm.red, &sm.bcast, &sm.cd_fail);
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
  if (!REG) normalise(xs, p, sm.red);
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

// REG: the regression kinds (ElasticCCA, SCCA_IPLS); a separate instantiation keeps their solver out of the register
// allocation of the other kinds, and its 512-thread CTAs give the solver 128 registers
template <bool REG>
__global__ void __launch_bounds__(REG ? kRegThreads : kThreads, 1) als_dimension(AlsArgs a) {
  extern __shared__ double xs[];  // CTA 0: the vector of the view being updated
  __shared__ Smem sm;
  cg::grid_group grid = cg::this_grid();
  const bool lead = blockIdx.x == 0;
  const unsigned all = (1u << a.m) - 1u;
  const bool admm = a.kind == kAlsAdmm;
  if (REG)
    for (int t = threadIdx.x; t <= kWarps; t += blockDim.x) sm.red[t] = 0.0;  // see block_reduce
  if (REG && threadIdx.x == 0) sm.cd_fail = 0;

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
          // (ElasticCCA: view i's own block too, its target includes X_i w_i)
          matvec(a, a.off[i], a.off[i + 1] - a.off[i], REG && a.kind == kAlsElastic ? all : all & ~(1u << i), a.off[prev],
                 a.off[prev + 1] - a.off[prev], 1u << prev, false);
          grid.sync();
        }
        if (lead) gs_update<REG>(a, i, fresh ? -1 : prev, xs, sm);
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
    if (REG && a.kind == kAlsIpls)  // deflate the column means with the view: mu_i <- mu_i - (mu_i^T w_i) f_i
      for (int i = 0; i < a.m; ++i) {
        double s = 0.0;
        for (int r = a.off[i] + threadIdx.x; r < a.off[i + 1]; r += blockDim.x) s = fma(a.colmean[r], a.w[r], s);
        s = block_reduce<false>(s, sm.red);
        for (int r = a.off[i] + threadIdx.x; r < a.off[i + 1]; r += blockDim.x) a.colmean[r] -= s * a.f[r];
        __syncthreads();
      }
    if (threadIdx.x == 0) a.iters_out[a.d] = REG && sm.cd_fail ? -iters : iters;
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
  size_t g, r, w, z, eta, f, rowsq, p, fro, done, v, ev, colmean, jac, total;  // byte offsets
};

AlsWorkspace als_workspace(const ColumnLayout& L, bool reg) {
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
  w.v = w.ev = w.colmean = w.jac = w.total = w.done + 256;
  if (!reg) return w;
  // regression kinds only: the eigenvectors of every G_ii, the eigenvalues, the IPLS column means, the eigensolver's
  size_t vv = 0, jac = 0;
  for (int i = 0; i < L.n_views; ++i) {
    vv += (size_t)L.dims[i] * L.dims[i];
    jac = std::max(jac, jacobi_workspace_bytes<double>(L.dims[i], L.dims[i], 1));
  }
  w.ev = w.v + al(8 * vv);
  w.colmean = w.ev + al(8 * D);
  w.jac = w.colmean + al(8 * D);
  w.total = w.jac + al(jac);
  return w;
}

}  // namespace

size_t als_fit_workspace_bytes(const ColumnLayout& L, bool regression) {
  return als_workspace(L, regression).total + 256;
}

int als_fit(int kind, const ColumnLayout& L, const double* G, double g_scale, double n_samples, const double* params,
            double mu, const double* init, int k, int max_iter, double tol, double* W_out, int* iters_out, void* ws,
            size_t ws_bytes, cudaStream_t stream) {
  const bool reg = kind == kAlsElastic || kind == kAlsIpls;
  CCAB_CHECK_ARG(ws_bytes >= als_fit_workspace_bytes(L, reg), "workspace too small: %zu < %zu", ws_bytes,
                 als_fit_workspace_bytes(L, reg));
  int maxp = 0;
  for (int v = 0; v < L.n_views; ++v) maxp = L.dims[v] > maxp ? L.dims[v] : maxp;
  const size_t smem = (size_t)maxp * sizeof(double) * (reg ? 3 : 1);
  int dev = 0, sms = 0, optin = 0;
  CCAB_CUDA(cudaGetDevice(&dev));
  CCAB_CUDA(cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, dev));
  CCAB_CUDA(cudaDeviceGetAttribute(&optin, cudaDevAttrMaxSharedMemoryPerBlockOptin, dev));
  CCAB_CHECK_ARG(smem + sizeof(Smem) <= (size_t)optin, "a view of %d features does not fit the shared memory of the ALS kernel",
                 maxp);
  const void* kern = reg ? (const void*)als_dimension<true> : (const void*)als_dimension<false>;
  CCAB_CUDA(cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
  int per_sm = 0;
  const int threads = reg ? kRegThreads : kThreads;
  CCAB_CUDA(cudaOccupancyMaxActiveBlocksPerMultiprocessor(&per_sm, kern, threads, smem));
  CCAB_CHECK_ARG(per_sm >= 1, "the ALS kernel cannot be resident on this device");

  uintptr_t base = ((uintptr_t)ws + 255) / 256 * 256;
  const AlsWorkspace o = als_workspace(L, reg);
  AlsArgs a;
  a.kind = kind;
  a.m = L.n_views;
  a.D = L.D;
  a.k = k;
  a.max_iter = max_iter;
  for (int v = 0; v <= L.n_views; ++v) a.off[v] = L.coff[v];
  a.maxp = maxp;
  for (int v = 0; v < kMaxViews; ++v) a.param[v] = a.rho[v] = a.lam[v] = 0.0;
  for (int v = 0; v < L.n_views; ++v) {
    if (reg) {
      // Ridge (l1 = 0) minimises ||y - X w||^2 + alpha ||w||^2, not divided by n
      a.rho[v] = params[2 * v + 1] == 0.0 ? params[2 * v] / n_samples : params[2 * v] * (1.0 - params[2 * v + 1]);
      a.lam[v] = params[2 * v] * params[2 * v + 1];
    } else {
      a.param[v] = kind == kAlsPmd ? params[v] * sqrt((double)L.dims[v]) : (kind == kAlsPls ? 0.0 : params[v]);
    }
  }
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
  double* V = reinterpret_cast<double*>(base + o.v);
  double* ev = reinterpret_cast<double*>(base + o.ev);
  a.V = V;
  a.ev = ev;
  a.colmean = reinterpret_cast<double*>(base + o.colmean);
  bool need_eig = false;
  for (int v = 0, acc = 0; v < L.n_views; ++v) {
    a.voff[v] = (size_t)acc;
    acc += L.dims[v] * L.dims[v];
    need_eig = need_eig || (reg && a.lam[v] == 0.0);
  }
  if (kind == kAlsIpls)
    CCAB_CUDA(cudaMemcpyAsync(a.colmean, params + 2 * L.n_views, sizeof(double) * L.D, cudaMemcpyHostToDevice, stream));

  const size_t nn = (size_t)L.D * L.D;
  als_scale_copy<<<(unsigned)std::min<size_t>(ceil_div(nn, 256), 4 * (size_t)sms), 256, 0, stream>>>(G, Gw, nn,
                                                                                                   g_scale);
  CCAB_CUDA(cudaGetLastError());
  int launches = 1;
  for (int d = 0; d < k; ++d) {
    a.d = d;
    // lam == 0 views of the regression kinds: the eigendecomposition of this dimension's G_ii (synchronises the stream)
    for (int v = 0; need_eig && v < L.n_views; ++v) {
      if (a.lam[v] != 0.0) continue;
      JacobiArgs<double> ja;
      memset(&ja, 0, sizeof(ja));
      ja.in = Gw + (size_t)L.coff[v] * L.D + L.coff[v];
      ja.ld_in = L.D;
      ja.batch_stride_in = 0;
      ja.colmajor_in = 1;  // symmetric
      ja.m = ja.n = L.dims[v];
      ja.batch = 1;
      ja.out_vals = ev + L.coff[v];
      ja.vals_stride = L.dims[v];
      ja.out_right = V + a.voff[v];
      ja.ld_right = L.dims[v];
      ja.right_stride = (int64_t)L.dims[v] * L.dims[v];
      int info = 0;
      ja.info = &info;
      const int rc = jacobi_solve<double>(ja, reinterpret_cast<void*>(base + o.jac), o.total - o.jac, stream);
      if (rc) return rc;
      CCAB_CHECK_ARG(info > 0, "the eigensolver of view %d did not converge (dimension %d)", v, d);
    }
    void* args[] = {&a};
    CCAB_CUDA(cudaLaunchCooperativeKernel(kern, dim3(per_sm * sms), dim3(threads), args, smem,
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
