// GFA (Group Factor Analysis, cca_zoo/probabilistic/_gfa.py): the closed-form mean-field variational loop, every
// iteration of a chunk inside ONE persistent cooperative kernel (gfa_steps), the state carried between calls in a
// caller-owned device block (layout: gfa_layout, documented with ccab_gfa_fit in include/ccab200.h).
//
// From the first Z update on, the latent mean is z = X B with B = [tau_1 W_1; ...; tau_m W_m] cov_z (D x k), so the
// loop is a function of the Gram matrix G = X^T X (centred when the views are) and of GB = G B:
//   X_m^T z = (GB)_m,  z^T z = B^T G B,  sum z o (X_m W_m) = sum (GB)_m o W_m,  mean(z^2, 0) = diag(B^T G B) / n,
//   ||z - z'||^2 = tr((B - B')^T (GB - GB')),  ||z'||^2 = tr(B'^T GB').
// Only the first W update reads the random start z0, through X^T z0 (XtZ0).  Phases of one iteration, separated by
// grid barriers (CTA 0 does the k x k algebra while the other CTAs wait at the next barrier):
//   1. CTA 0: cov_w_m = (1/tau_m) T o inv(T o zz + I / tau_m),  T = t t^T,  t = alpha_m^-1/2      (Cholesky)
//   2. W_m = tau_m (GB)_m cov_w_m                                                      (rows of W, all CTAs)
//   3. ww_m = W_m^T W_m                                                                (one warp per entry)
//   4. CTA 0: ww_m += d_m cov_w_m, the ARD update of alpha_m, cov_z = inv(I + sum_m tau_m ww_m)
//   5. B = [tau_m W_m] cov_z                                                           (rows of B)
//   6. GB = G B in 32-row tiles, the columns split into a fixed number of slices;  7. the slices summed in order
//   8. B^T GB, the per-view cross terms sum (GB)_m o W_m and the terms of the stopping statistic (one warp each)
//   9. CTA 0: zz = B^T G B + n cov_z, the tau update, pruning (columns compacted in place, in index order), the
//      patience counter and the stop flag; then phase 1 of the next iteration.
// GB and B of the previous iteration stay in the second buffer of a pair (the header's parity picks the current
// one), so the stopping statistic needs no second pass over G.  Every reduction has a fixed order and there are no
// floating-point atomics: repeated fits are bit-identical, and so is any split of the iterations into calls.
#include <cooperative_groups.h>

#include <algorithm>
#include <cmath>

#include "common.cuh"
#include "gfa.cuh"

namespace ccab {
namespace cg = cooperative_groups;

namespace {

constexpr int kThreads = 256;
constexpr int kWarps = kThreads / 32;
constexpr int kXpt = kGfaMaxK / kWarps;  // latent columns per thread in the G B tiles
constexpr int kTile = 32;                // rows of G B per tile (one per lane)
constexpr int kCh = 32;                  // columns of G staged per round
constexpr int kItems = 128;              // target number of (tile, slice) work items of G B
constexpr size_t kCholSmem = 128 << 10;  // shared memory for the batched k x k factorisations

constexpr double kArdBeta0 = 1e-14;
constexpr double kTauBeta0 = 1e-14;
constexpr double kDropTol = 1e-7;
constexpr int kPatience = 1000;

// header slots
constexpr int hIters = 0, hK = 1, hStable = 2, hStop = 3, hParity = 4, hRel = 5, hPrunes = 6;

struct GfaArgs {
  int m, D, K, S, cps, n_steps, drop_k, nb;  // nb: matrices per batched factorisation
  int off[kMaxViews + 1];
  double n, tol;
  const double* G;
  const double* XtZ0;
  double* st;
  double* part;  // S x K x D partials of G B (S > 1)
  double* red;   // B^T GB (K x K) | cross (kMaxViews x K) | stop terms (2 x K)
  GfaLayout o;
};

__device__ __forceinline__ double warp_sum(double v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
  return v;
}

__device__ __forceinline__ int gwarp() { return (blockIdx.x * blockDim.x + threadIdx.x) >> 5; }
__device__ __forceinline__ int nwarps() { return (gridDim.x * blockDim.x) >> 5; }

__device__ __forceinline__ int view_of(const GfaArgs& a, int r) {
  int v = 0;
  for (int u = 1; u < a.m; ++u) v += r >= a.off[u] ? 1 : 0;
  return v;
}

// In place: nb symmetric positive definite k x k matrices (leading dimension k, shared memory) -> their inverses,
// via the lower Cholesky factor L and inv = L^-T L^-1.  Li: scratch of the same size.  All threads of the block.
__device__ void chol_inv(double* A, double* Li, int nb, int k) {
  const int kk = k * k;
  for (int j = 0; j < k; ++j) {
    __syncthreads();
    for (int t = threadIdx.x; t < nb * k; t += blockDim.x) {
      const int b = t / k, i = t % k;
      double* a = A + b * kk;
      if (i > j) a[i * k + j] /= sqrt(a[j * k + j]);
    }
    __syncthreads();
    const int nt = k - j - 1;
    for (int t = threadIdx.x; t < nb * nt * nt; t += blockDim.x) {
      const int b = t / (nt * nt), r = t % (nt * nt), i = j + 1 + r / nt, l = j + 1 + r % nt;
      double* a = A + b * kk;
      if (l <= i) a[i * k + l] -= a[i * k + j] * a[l * k + j];
    }
    for (int b = threadIdx.x; b < nb; b += blockDim.x) A[b * kk + j * k + j] = sqrt(A[b * kk + j * k + j]);
  }
  __syncthreads();
  for (int t = threadIdx.x; t < nb * k; t += blockDim.x) {  // columns of L^-1 by forward substitution
    const int b = t / k, c = t % k;
    const double* a = A + b * kk;
    double* li = Li + b * kk;
    for (int i = 0; i < c; ++i) li[i * k + c] = 0.0;
    for (int i = c; i < k; ++i) {
      double s = i == c ? 1.0 : 0.0;
      for (int l = c; l < i; ++l) s -= a[i * k + l] * li[l * k + c];
      li[i * k + c] = s / a[i * k + i];
    }
  }
  __syncthreads();
  for (int t = threadIdx.x; t < nb * kk; t += blockDim.x) {
    const int b = t / kk, i = (t % kk) / k, j = t % k;
    const double* li = Li + b * kk;
    double s = 0.0;
    for (int l = max(i, j); l < k; ++l) s += li[l * k + i] * li[l * k + j];
    A[t] = s;
  }
  __syncthreads();
}

struct Ptr {
  double *hdr, *y_const, *a_ard, *a_tau, *tau, *b_tau, *alpha, *b_ard, *cov_w, *ww, *cov_z, *zz, *index, *W;
  double* B[2];
  double* GB[2];
};

__device__ Ptr pointers(const GfaArgs& a) {
  Ptr p;
  double* s = a.st;
  p.hdr = s;
  p.y_const = s + a.o.y_const;
  p.a_ard = s + a.o.a_ard;
  p.a_tau = s + a.o.a_tau;
  p.tau = s + a.o.tau;
  p.b_tau = s + a.o.b_tau;
  p.alpha = s + a.o.alpha;
  p.b_ard = s + a.o.b_ard;
  p.cov_w = s + a.o.cov_w;
  p.ww = s + a.o.ww;
  p.cov_z = s + a.o.cov_z;
  p.zz = s + a.o.zz;
  p.index = s + a.o.index;
  p.W = s + a.o.W;
  p.B[0] = s + a.o.B0;
  p.B[1] = s + a.o.B1;
  p.GB[0] = s + a.o.GB0;
  p.GB[1] = s + a.o.GB1;
  return p;
}

// phase 1 (CTA 0): cov_w of every view from zz, alpha and tau
__device__ void phase_cov_w(const GfaArgs& a, const Ptr& p, int k, double* sm) {
  const int K = a.K, kk = k * k;
  double* A = sm;
  double* Li = sm + a.nb * kk;
  for (int v0 = 0; v0 < a.m; v0 += a.nb) {
    const int nb = min(a.nb, a.m - v0);
    __syncthreads();
    for (int t = threadIdx.x; t < nb * kk; t += blockDim.x) {
      const int v = v0 + t / kk, i = (t % kk) / k, j = t % k;
      const double T = (1.0 / sqrt(p.alpha[v * K + i])) * (1.0 / sqrt(p.alpha[v * K + j]));
      A[t] = T * p.zz[i * K + j] + (i == j ? 1.0 / p.tau[v] : 0.0);
    }
    chol_inv(A, Li, nb, k);
    for (int t = threadIdx.x; t < nb * kk; t += blockDim.x) {
      const int v = v0 + t / kk, i = (t % kk) / k, j = t % k;
      const double T = (1.0 / sqrt(p.alpha[v * K + i])) * (1.0 / sqrt(p.alpha[v * K + j]));
      p.cov_w[((size_t)v * K + i) * K + j] = (1.0 / p.tau[v]) * T * A[t];
    }
  }
  __syncthreads();
}

// phases 2 and 5: out[x][r] = s_r sum_y in[y][r] M_v[y][x] for the rows r of view v, M_v = mat + v * mstride,
// s_r = scale[v]; one thread per (row, group of 8 latent columns)
__device__ void rows_times(const GfaArgs& a, int k, const double* in, const double* mat, size_t mstride,
                           const double* scale, bool scale_in, double* out) {
  const int K = a.K, D = a.D, ng = (k + 7) / 8;
  for (int t = blockIdx.x * blockDim.x + threadIdx.x; t < D * ng; t += gridDim.x * blockDim.x) {
    const int r = t % D, x0 = (t / D) * 8;
    const int v = view_of(a, r);
    const double* M = mat + v * mstride;
    const double s = scale[v];
    double acc[8];
#pragma unroll
    for (int j = 0; j < 8; ++j) acc[j] = 0.0;
    for (int y = 0; y < k; ++y) {
      const double iv = scale_in ? s * in[(size_t)y * D + r] : in[(size_t)y * D + r];
#pragma unroll
      for (int j = 0; j < 8; ++j)
        if (x0 + j < k) acc[j] = fma(iv, M[y * K + x0 + j], acc[j]);
    }
#pragma unroll
    for (int j = 0; j < 8; ++j)
      if (x0 + j < k) out[(size_t)(x0 + j) * D + r] = scale_in ? acc[j] : s * acc[j];
  }
}

// phase 3: ww_m = W_m^T W_m (upper triangle computed, mirrored), one warp per entry
__device__ void phase_ww(const GfaArgs& a, const Ptr& p, int k) {
  const int lane = threadIdx.x & 31, K = a.K, D = a.D;
  for (int t = gwarp(); t < a.m * k * k; t += nwarps()) {
    const int v = t / (k * k), x = (t % (k * k)) / k, y = t % k;
    if (x > y) continue;
    const double* wx = p.W + (size_t)x * D;
    const double* wy = p.W + (size_t)y * D;
    double s = 0.0;
    for (int r = a.off[v] + lane; r < a.off[v + 1]; r += 32) s = fma(wx[r], wy[r], s);
    s = warp_sum(s);
    if (lane == 0) {
      p.ww[((size_t)v * K + x) * K + y] = s;
      p.ww[((size_t)v * K + y) * K + x] = s;
    }
  }
}

// phase 4 (CTA 0): ww_m += d_m cov_w_m, the ARD update, cov_z
__device__ void phase_cov_z(const GfaArgs& a, const Ptr& p, int k, double* sm) {
  const int K = a.K, kk = k * k;
  for (int t = threadIdx.x; t < a.m * kk; t += blockDim.x) {
    const int v = t / kk, i = (t % kk) / k, j = t % k;
    const size_t e = ((size_t)v * K + i) * K + j;
    p.ww[e] += (double)(a.off[v + 1] - a.off[v]) * p.cov_w[e];
  }
  __syncthreads();
  for (int t = threadIdx.x; t < a.m * k; t += blockDim.x) {
    const int v = t / k, x = t % k;
    const double b = kArdBeta0 + p.ww[((size_t)v * K + x) * K + x] / 2.0;
    p.b_ard[v * K + x] = b;
    p.alpha[v * K + x] = p.a_ard[v] / b;
  }
  for (int t = threadIdx.x; t < kk; t += blockDim.x) {
    const int i = t / k, j = t % k;
    double s = i == j ? 1.0 : 0.0;
    for (int v = 0; v < a.m; ++v) s = s + p.tau[v] * p.ww[((size_t)v * K + i) * K + j];
    sm[t] = s;
  }
  chol_inv(sm, sm + kk, 1, k);
  for (int t = threadIdx.x; t < kk; t += blockDim.x) p.cov_z[(t / k) * K + t % k] = sm[t];
  __syncthreads();
}

// phase 6: G B, or its column-slice partials
__device__ void phase_gb(const GfaArgs& a, int k, const double* B, double* GB, double* sm) {
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5, D = a.D;
  double* Gs = sm;               // kCh x kTile
  double* Bs = sm + kCh * kTile; // k x kCh
  const int tiles = (D + kTile - 1) / kTile;
  for (int item = blockIdx.x; item < tiles * a.S; item += gridDim.x) {
    const int tile = item % tiles, s = item / tiles;
    const int r0 = tile * kTile;
    const int c_begin = s * a.cps * kCh, c_end = min(D, (s + 1) * a.cps * kCh);
    double acc[kXpt];
#pragma unroll
    for (int j = 0; j < kXpt; ++j) acc[j] = 0.0;
    for (int c0 = c_begin; c0 < c_end; c0 += kCh) {
      const int cn = min(kCh, c_end - c0);
      __syncthreads();
      // G is symmetric: row c0 + c of G holds column c0 + c, so the tile is read along rows (coalesced)
      for (int e = threadIdx.x; e < kCh * kTile; e += blockDim.x) {
        const int c = e / kTile, r = e % kTile;
        Gs[e] = (c < cn && r0 + r < D) ? a.G[(size_t)(c0 + c) * D + r0 + r] : 0.0;
      }
      for (int e = threadIdx.x; e < k * kCh; e += blockDim.x) {
        const int x = e / kCh, c = e % kCh;
        Bs[e] = c < cn ? B[(size_t)x * D + c0 + c] : 0.0;
      }
      __syncthreads();
      for (int c = 0; c < cn; ++c) {
        const double g = Gs[c * kTile + lane];
#pragma unroll
        for (int j = 0; j < kXpt; ++j) {
          const int x = warp + kWarps * j;
          if (x < k) acc[j] = fma(g, Bs[x * kCh + c], acc[j]);
        }
      }
    }
    const int r = r0 + lane;
    if (r < D) {
      double* out = a.S > 1 ? a.part + (size_t)s * a.K * D : GB;
#pragma unroll
      for (int j = 0; j < kXpt; ++j) {
        const int x = warp + kWarps * j;
        if (x < k) out[(size_t)x * D + r] = acc[j];
      }
    }
  }
}

// phase 8: B^T GB (upper triangle), the per-view cross terms and the stopping-statistic terms; one warp per task
__device__ void phase_reduce(const GfaArgs& a, const Ptr& p, int k, const double* B, const double* GB,
                             const double* Bp, const double* GBp, bool stop_terms) {
  const int lane = threadIdx.x & 31, K = a.K, D = a.D;
  double* btgb = a.red;
  double* cross = a.red + K * K;
  double* stopt = cross + kMaxViews * K;
  const int n1 = k * k, n2 = n1 + a.m * k, n3 = n2 + (stop_terms ? 2 * k : 0);
  for (int t = gwarp(); t < n3; t += nwarps()) {
    double s = 0.0;
    if (t < n1) {
      const int x = t / k, y = t % k;
      if (x > y) continue;
      const double* bx = B + (size_t)x * D;
      const double* gy = GB + (size_t)y * D;
      for (int r = lane; r < D; r += 32) s = fma(bx[r], gy[r], s);
      s = warp_sum(s);
      if (lane == 0) btgb[x * K + y] = btgb[y * K + x] = s;
    } else if (t < n2) {
      const int v = (t - n1) / k, x = (t - n1) % k;
      const double* g = GB + (size_t)x * D;
      const double* w = p.W + (size_t)x * D;
      for (int r = a.off[v] + lane; r < a.off[v + 1]; r += 32) s = fma(g[r], w[r], s);
      s = warp_sum(s);
      if (lane == 0) cross[v * K + x] = s;
    } else {
      const int q = (t - n2) / k, x = (t - n2) % k;
      const double* b = B + (size_t)x * D;
      const double* g = GB + (size_t)x * D;
      const double* bp = Bp + (size_t)x * D;
      const double* gp = GBp + (size_t)x * D;
      if (q == 0)
        for (int r = lane; r < D; r += 32) s = fma(b[r] - bp[r], g[r] - gp[r], s);
      else
        for (int r = lane; r < D; r += 32) s = fma(bp[r], gp[r], s);
      s = warp_sum(s);
      if (lane == 0) stopt[q * K + x] = s;
    }
  }
}

// compact the rows keep[0..nk) of a k-row, ld-D array in place (keep ascending, keep[j] >= j)
__device__ void compact_rows(double* X, const int* keep, int nk, int D) {
  for (int j = 0; j < nk; ++j) {
    if (keep[j] != j)
      for (int r = threadIdx.x; r < D; r += blockDim.x) X[(size_t)j * D + r] = X[(size_t)keep[j] * D + r];
    __syncthreads();
  }
}

// compact a k x k matrix (leading dimension K) to its rows and columns keep[0..nk), through shared memory
__device__ void compact_kk(double* M, const int* keep, int nk, int K, double* sm) {
  __syncthreads();
  for (int t = threadIdx.x; t < nk * nk; t += blockDim.x) sm[t] = M[keep[t / nk] * K + keep[t % nk]];
  __syncthreads();
  for (int t = threadIdx.x; t < nk * nk; t += blockDim.x) M[(t / nk) * K + t % nk] = sm[t];
  __syncthreads();
}

struct Cta0 {
  int keep[kGfaMaxK];
  int nk, k, stop;
};

// phase 9 (CTA 0): zz, tau, pruning, the stopping rule; updates the header.  Returns the new k.
__device__ void phase_update(const GfaArgs& a, const Ptr& p, int k, int cur, int iters, double* sm, Cta0& c0) {
  const int K = a.K, lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  const double* btgb = a.red;
  const double* cross = a.red + K * K;
  const double* stopt = cross + kMaxViews * K;
  for (int t = threadIdx.x; t < k * k; t += blockDim.x) {
    const int i = t / k, j = t % k;
    p.zz[i * K + j] = btgb[i * K + j] + a.n * p.cov_z[i * K + j];
  }
  __syncthreads();
  for (int v = warp; v < a.m; v += kWarps) {  // tau: one warp per view
    double s = 0.0;
    for (int t = lane; t < k * k; t += 32) s += p.ww[((size_t)v * K + t / k) * K + t % k] * p.zz[(t / k) * K + t % k];
    s = warp_sum(s);
    if (lane == 0) {
      double cr = 0.0;
      for (int x = 0; x < k; ++x) cr += cross[v * K + x];
      const double b = kTauBeta0 + (p.y_const[v] + s - 2.0 * cr) / 2.0;
      p.b_tau[v] = b;
      p.tau[v] = p.a_tau[v] / b;
    }
  }
  if (threadIdx.x == 0) {
    int nk = 0;
    for (int x = 0; x < k; ++x)
      if (!a.drop_k || btgb[x * K + x] / a.n > kDropTol) c0.keep[nk++] = x;
    const bool pruned = a.drop_k && nk > 0 && nk != k;
    c0.nk = pruned ? nk : k;
    double* hdr = p.hdr;
    double stable = hdr[hStable];
    hdr[hRel] = NAN;
    if (pruned) {
      stable = 0.0;
      hdr[hPrunes] += 1.0;
    } else if (iters > 0) {
      double num = 0.0, den = 0.0;
      for (int x = 0; x < k; ++x) num += stopt[x];
      for (int x = 0; x < k; ++x) den += stopt[K + x];
      const double rel = sqrt(num) / fmax(sqrt(den), 1e-300);
      hdr[hRel] = rel;
      stable = rel < a.tol ? stable + 1.0 : 0.0;
    }
    hdr[hStable] = stable;
    hdr[hIters] = (double)(iters + 1);
    hdr[hK] = (double)c0.nk;
    hdr[hParity] = (double)cur;
    c0.stop = stable >= kPatience ? 1 : 0;
    hdr[hStop] = c0.stop ? 1.0 : 0.0;
  }
  __syncthreads();
  const int nk = c0.nk;
  if (nk != k) {
    compact_rows(p.B[cur], c0.keep, nk, a.D);
    compact_rows(p.GB[cur], c0.keep, nk, a.D);
    compact_rows(p.W, c0.keep, nk, a.D);
    for (int v = 0; v < a.m; ++v) {
      compact_kk(p.cov_w + (size_t)v * K * K, c0.keep, nk, K, sm);
      compact_kk(p.ww + (size_t)v * K * K, c0.keep, nk, K, sm);
    }
    compact_kk(p.cov_z, c0.keep, nk, K, sm);
    compact_kk(p.zz, c0.keep, nk, K, sm);
    if (threadIdx.x < a.m) {
      const int v = threadIdx.x;
      for (int j = 0; j < nk; ++j) {
        p.alpha[v * K + j] = p.alpha[v * K + c0.keep[j]];
        p.b_ard[v * K + j] = p.b_ard[v * K + c0.keep[j]];
      }
    }
    if (threadIdx.x == kThreads - 1)
      for (int j = 0; j < nk; ++j) p.index[j] = p.index[c0.keep[j]];
  }
  c0.k = nk;
  __syncthreads();
}

__global__ void __launch_bounds__(kThreads) gfa_steps(GfaArgs a) {
  extern __shared__ double sm[];
  __shared__ Cta0 c0;
  cg::grid_group grid = cg::this_grid();
  const Ptr p = pointers(a);
  if (__ldcg(p.hdr + hStop) != 0.0) return;  // a previous call stopped the fit: every block returns before a barrier
  int iters = (int)__ldcg(p.hdr + hIters);
  int k = (int)__ldcg(p.hdr + hK);
  int cur = (int)__ldcg(p.hdr + hParity);
  if (blockIdx.x == 0) phase_cov_w(a, p, k, sm);
  grid.sync();
  for (int t = 0; t < a.n_steps; ++t) {
    const double* XZ = iters == 0 ? a.XtZ0 : p.GB[cur];
    rows_times(a, k, XZ, p.cov_w, (size_t)a.K * a.K, p.tau, false, p.W);
    grid.sync();
    phase_ww(a, p, k);
    grid.sync();
    if (blockIdx.x == 0) phase_cov_z(a, p, k, sm);
    grid.sync();
    const int nxt = cur ^ 1;
    rows_times(a, k, p.W, p.cov_z, 0, p.tau, true, p.B[nxt]);
    grid.sync();
    phase_gb(a, k, p.B[nxt], p.GB[nxt], sm);
    grid.sync();
    if (a.S > 1) {
      const size_t kd = (size_t)k * a.D, KD = (size_t)a.K * a.D;
      for (size_t e = (size_t)blockIdx.x * blockDim.x + threadIdx.x; e < kd; e += (size_t)gridDim.x * blockDim.x) {
        double s = 0.0;
        for (int q = 0; q < a.S; ++q) s += a.part[q * KD + e];
        p.GB[nxt][e] = s;
      }
      grid.sync();
    }
    phase_reduce(a, p, k, p.B[nxt], p.GB[nxt], p.B[cur], p.GB[cur], iters > 0);
    grid.sync();
    if (blockIdx.x == 0) {
      phase_update(a, p, k, nxt, iters, sm, c0);
      if (!c0.stop && t + 1 < a.n_steps) phase_cov_w(a, p, c0.k, sm);
    }
    grid.sync();
    cur = nxt;
    ++iters;
    k = (int)__ldcg(p.hdr + hK);
    if (__ldcg(p.hdr + hStop) != 0.0) break;
  }
}

struct GfaWorkspace {
  size_t part, red, total;
  int S, cps;
};

GfaWorkspace gfa_workspace(const ColumnLayout& L, int K) {
  auto al = [](size_t x) { return (x + 255) / 256 * 256; };
  GfaWorkspace w;
  const int tiles = (L.D + kTile - 1) / kTile, chunks = (L.D + kCh - 1) / kCh;
  int S = std::max(1, std::min(chunks, kItems / tiles));
  w.cps = (chunks + S - 1) / S;
  w.S = (chunks + w.cps - 1) / w.cps;
  w.part = 0;
  w.red = w.part + (w.S > 1 ? al(8 * (size_t)w.S * K * L.D) : 0);
  w.total = w.red + al(8 * ((size_t)K * K + (size_t)(kMaxViews + 2) * K));
  return w;
}

int chol_batch(int m, int K) { return std::max(1, std::min(m, (int)(kCholSmem / (16 * (size_t)K * K)))); }

size_t smem_bytes(int m, int K) {
  const size_t gemm = 8 * (size_t)(kCh * kTile + K * kCh);
  const size_t chol = 16 * (size_t)chol_batch(m, K) * K * K;
  return std::max(gemm, chol);
}

}  // namespace

GfaLayout gfa_layout(int K, int D) {
  GfaLayout o;
  const size_t V = kMaxViews, k = (size_t)K, kk = k * k, kd = k * (size_t)D;
  o.y_const = kGfaHeader;
  o.a_ard = o.y_const + V;
  o.a_tau = o.a_ard + V;
  o.tau = o.a_tau + V;
  o.b_tau = o.tau + V;
  o.alpha = o.b_tau + V;
  o.b_ard = o.alpha + V * k;
  o.cov_w = o.b_ard + V * k;
  o.ww = o.cov_w + V * kk;
  o.cov_z = o.ww + V * kk;
  o.zz = o.cov_z + kk;
  o.index = o.zz + kk;
  o.W = o.index + k;
  o.B0 = o.W + kd;
  o.B1 = o.B0 + kd;
  o.GB0 = o.B1 + kd;
  o.GB1 = o.GB0 + kd;
  o.total = o.GB1 + kd;
  return o;
}

size_t gfa_fit_workspace_bytes(const ColumnLayout& L, int k) { return gfa_workspace(L, k).total + 256; }

int gfa_fit(const ColumnLayout& L, int k, const double* G, double n_samples, const double* XtZ0, double tol,
            int drop_k, int n_steps, double* state, void* ws, size_t ws_bytes, cudaStream_t stream) {
  CCAB_CHECK_ARG(ws_bytes >= gfa_fit_workspace_bytes(L, k), "workspace too small: %zu < %zu", ws_bytes,
                 gfa_fit_workspace_bytes(L, k));
  if (n_steps == 0) return 0;
  const GfaWorkspace o = gfa_workspace(L, k);
  uintptr_t base = ((uintptr_t)ws + 255) / 256 * 256;
  GfaArgs a;
  a.m = L.n_views;
  a.D = L.D;
  a.K = k;
  a.S = o.S;
  a.cps = o.cps;
  a.n_steps = n_steps;
  a.drop_k = drop_k ? 1 : 0;
  a.nb = chol_batch(L.n_views, k);
  for (int v = 0; v <= L.n_views; ++v) a.off[v] = L.coff[v];
  for (int v = L.n_views + 1; v <= kMaxViews; ++v) a.off[v] = L.D;
  a.n = n_samples;
  a.tol = tol;
  a.G = G;
  a.XtZ0 = XtZ0;
  a.st = state;
  a.part = reinterpret_cast<double*>(base + o.part);
  a.red = reinterpret_cast<double*>(base + o.red);
  a.o = gfa_layout(k, L.D);

  const void* fn = (const void*)gfa_steps;
  const size_t smem = smem_bytes(L.n_views, k);
  CCAB_CUDA(cudaFuncSetAttribute(fn, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
  int dev = 0, sms = 0, per_sm = 0;
  CCAB_CUDA(cudaGetDevice(&dev));
  CCAB_CUDA(cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, dev));
  CCAB_CUDA(cudaOccupancyMaxActiveBlocksPerMultiprocessor(&per_sm, fn, kThreads, smem));
  CCAB_CHECK_ARG(per_sm >= 1, "the GFA kernel cannot be resident on this device");
  void* args[] = {&a};
  CCAB_CUDA(cudaLaunchCooperativeKernel(fn, dim3(per_sm * sms), dim3(kThreads), args, smem, stream));
  count_launches(1);
  return 0;
}

}  // namespace ccab
