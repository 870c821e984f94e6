// Eckart-Young gradient estimators (CCA_EY, PLS_EY, MCCA_EY): momentum steps on the EY loss
//   L = -2 tr(C_ey - c V) + tr(Vb Vb),  Vb = (1 - c) V + c B,  B = (1/m) sum_i W_i^T W_i,
// every step of a chunk inside ONE persistent cooperative kernel (ey_steps), the state (W, velocity, previous
// objective, step count, stop flag) carried between calls in a caller-owned device block.
//
// Two routes, with m views and k latent dimensions:
//   * covariance route (full batch): everything the reference's full-batch step forms is a function of the centred
//     block covariance C.  With Y_ij = C_ij W_j, V = (1/m) sum_i W_i^T Y_ii, C_ey = (1/m) sum_ij W_i^T Y_ij and
//       g_i = (4/m) [c Y_ii + (1 - c) Y_ii Vb - sum_j Y_ij] + (4c/m) W_i Vb.
//     Phases: Y = C blockdiag(W) in row tiles (C read once), the k x k products, the row-local update, B of the
//     updated weights.  The cost does not depend on n.
//   * mini-batch route: the bs rows idx[step] are gathered straight from the views (float32 or float64, any ld).
//     Z_i = X_b,i W_i, Zc_i = Z_i - mean, S = sum_j Zc_j, V = sum_i Zc_i^T Zc_i / (m (bs - 1)),
//     C_ey = S^T S / (m (bs - 1)), T_i = 4 / (m (bs - 1)) (c Zc_i + (1 - c) Zc_i Vb - S) and
//       g_i = X_b,i^T T_i + (4c/m) W_i Vb.
//     The columns of T_i sum to zero, so the centring of X cancels from the gradient: the views are read raw.
// The objective pairs V and C_ey of the PRE-update representations with B of the POST-update weights (as the
// reference does); a step stops the fit when |prev_obj - obj| < tol, which a NaN objective never satisfies.
//
// Grid barriers separate the phases; every reduction has a fixed order (warp butterflies, sums over rows or batch
// slices in index order) and no floating-point atomics, so repeated fits are bit-identical.
#include <cooperative_groups.h>

#include <algorithm>
#include <cmath>

#include "common.cuh"
#include "ey.cuh"

namespace ccab {
namespace cg = cooperative_groups;

namespace {

constexpr int kThreads = 256;
constexpr int kWarps = kThreads / 32;
constexpr int kChunk = 128;       // columns of W staged in shared memory per round of a row tile
constexpr int kSliceRows = 128;   // batch rows per partial of X_b^T T
constexpr int kMaxSlices = 64;

struct EyArgs {
  int m, D, k, batch, n_steps, nslices, slice;
  int off[kMaxViews + 1];   // column offset of each view
  int toff[kMaxViews + 1];  // first 32-feature tile of each view
  double c, lr, mom, tol;
  const double* cov;        // covariance route: D x D
  const void* X[kMaxViews];
  int64_t ld[kMaxViews];
  const int32_t* idx;       // mini-batch route: n_steps x batch row indices
  double* state;            // header | W (k x D) | velocity (k x D)
  double* ya;               // covariance: Y_ii (k x D); mini-batch: Z (batch x m x k)
  double* yb;               // covariance: sum_j Y_ij (k x D); mini-batch: T (batch x m x k)
  double* part;             // mini-batch: nslices x k x D partials of X_b^T T
  double* kk;               // V | C_ey | B[0] | B[1] (k x k each) | batch means (m x k)
};

struct Smem {
  double w[kEyMaxK * kChunk];  // staged columns of W
  double vb[kEyMaxK * kEyMaxK];
  double obj;
  int stop;
};

__device__ __forceinline__ double warp_sum(double v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
  return v;
}

__device__ __forceinline__ int gwarp() { return (blockIdx.x * blockDim.x + threadIdx.x) >> 5; }
__device__ __forceinline__ int nwarps() { return (gridDim.x * blockDim.x) >> 5; }

__device__ __forceinline__ int view_of(const EyArgs& a, int r) {
  int v = 0;
  for (int u = 1; u < a.m; ++u) v += r >= a.off[u] ? 1 : 0;
  return v;
}

// acc[x] = sum_s row[s] W[x, off_j + s] over the p_j columns of view j for the row of this warp (row == nullptr:
// zeros), reduced over the warp (every lane holds the sums).  Called by all threads of the block: the columns of W
// are staged in shared memory kChunk at a time and shared by the block's warps.
template <typename T>
__device__ void tile_rows(const EyArgs& a, const T* row, int j, const double* W, Smem& sm, double* acc) {
  const int lane = threadIdx.x & 31;
  const int o = a.off[j], p = a.off[j + 1] - o;
#pragma unroll
  for (int x = 0; x < kEyMaxK; ++x) acc[x] = 0.0;
  for (int c0 = 0; c0 < p; c0 += kChunk) {
    const int cn = min(kChunk, p - c0);
    __syncthreads();
    for (int e = threadIdx.x; e < a.k * kChunk; e += blockDim.x) {
      const int x = e / kChunk, s = e % kChunk;
      sm.w[e] = s < cn ? W[(size_t)x * a.D + o + c0 + s] : 0.0;
    }
    __syncthreads();
    if (row)
      for (int s = lane; s < cn; s += 32) {
        const double v = (double)row[c0 + s];
#pragma unroll
        for (int x = 0; x < kEyMaxK; ++x)
          if (x < a.k) acc[x] = fma(v, sm.w[x * kChunk + s], acc[x]);
      }
  }
#pragma unroll
  for (int x = 0; x < kEyMaxK; ++x)
    if (x < a.k) acc[x] = warp_sum(acc[x]);
}

// B[x][y] = (1/m) sum_r W[x][r] W[y][r]; one warp per entry
__device__ void gram(const EyArgs& a, const double* W, double* B) {
  const int lane = threadIdx.x & 31;
  for (int t = gwarp(); t < a.k * a.k; t += nwarps()) {
    const double* wx = W + (size_t)(t / a.k) * a.D;
    const double* wy = W + (size_t)(t % a.k) * a.D;
    double s = 0.0;
    for (int r = lane; r < a.D; r += 32) s = fma(wx[r], wy[r], s);
    s = warp_sum(s);
    if (lane == 0) B[t] = s / a.m;
  }
}

// shared Vb = (1 - c) V + c B
__device__ void blend(const EyArgs& a, const double* V, const double* B, Smem& sm) {
  __syncthreads();
  for (int e = threadIdx.x; e < a.k * a.k; e += blockDim.x) sm.vb[e] = (1.0 - a.c) * V[e] + a.c * B[e];
  __syncthreads();
}

// ---- covariance route -----------------------------------------------------------------------------------------
// Y_ii (ya) and sum_j Y_ij (yb) for every row r of C, eight rows per block tile
__device__ void cov_products(const EyArgs& a, const double* W, Smem& sm) {
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  double acc[kEyMaxK];
  for (int tile = blockIdx.x; tile < (a.D + kWarps - 1) / kWarps; tile += gridDim.x) {
    const int r = tile * kWarps + warp;
    const bool live = r < a.D;
    const int vr = live ? view_of(a, r) : -1;
    for (int j = 0; j < a.m; ++j) {
      tile_rows<double>(a, live ? a.cov + (size_t)r * a.D + a.off[j] : nullptr, j, W, sm, acc);
      if (!live) continue;
#pragma unroll
      for (int x = 0; x < kEyMaxK; ++x)
        if (x < a.k && lane == x) {
          if (j == vr) a.ya[(size_t)x * a.D + r] = acc[x];
          double* ys = a.yb + (size_t)x * a.D + r;
          *ys = j == 0 ? acc[x] : *ys + acc[x];
        }
    }
  }
}

// V = (1/m) W^T Y_ii and C_ey = (1/m) W^T sum_j Y_ij over all rows; one warp per entry
__device__ void cov_kk(const EyArgs& a, const double* W) {
  const int lane = threadIdx.x & 31, kk = a.k * a.k;
  for (int t = gwarp(); t < 2 * kk; t += nwarps()) {
    const int e = t % kk;
    const double* wx = W + (size_t)(e / a.k) * a.D;
    const double* y = (t < kk ? a.ya : a.yb) + (size_t)(e % a.k) * a.D;
    double s = 0.0;
    for (int r = lane; r < a.D; r += 32) s = fma(wx[r], y[r], s);
    s = warp_sum(s);
    if (lane == 0) a.kk[t] = s / a.m;
  }
}

// ---- mini-batch route -----------------------------------------------------------------------------------------
template <typename T>
__device__ void mb_project(const EyArgs& a, const int32_t* idx, const double* W, Smem& sm) {
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  const int tv = (a.batch + kWarps - 1) / kWarps;
  double acc[kEyMaxK];
  for (int tile = blockIdx.x; tile < a.m * tv; tile += gridDim.x) {
    const int i = tile / tv, b = (tile % tv) * kWarps + warp;
    const bool live = b < a.batch;
    const T* row = live ? static_cast<const T*>(a.X[i]) + (int64_t)idx[b] * a.ld[i] : nullptr;
    tile_rows<T>(a, row, i, W, sm, acc);
    if (!live) continue;
#pragma unroll
    for (int x = 0; x < kEyMaxK; ++x)
      if (x < a.k && lane == x) a.ya[((size_t)b * a.m + i) * a.k + x] = acc[x];
  }
}

// batch means of Z (m x k); one warp per entry
__device__ void mb_means(const EyArgs& a, double* mu) {
  const int lane = threadIdx.x & 31;
  for (int t = gwarp(); t < a.m * a.k; t += nwarps()) {
    const int i = t / a.k, x = t % a.k;
    double s = 0.0;
    for (int b = lane; b < a.batch; b += 32) s += a.ya[((size_t)b * a.m + i) * a.k + x];
    s = warp_sum(s);
    if (lane == 0) mu[t] = s / a.batch;
  }
}

// V and C_ey of the centred batch representations; one warp per entry
__device__ void mb_kk(const EyArgs& a, const double* mu) {
  const int lane = threadIdx.x & 31, kk = a.k * a.k, m = a.m, k = a.k;
  for (int t = gwarp(); t < 2 * kk; t += nwarps()) {
    const int e = t % kk, x = e / k, y = e % k;
    double s = 0.0;
    for (int b = lane; b < a.batch; b += 32) {
      const double* z = a.ya + (size_t)b * m * k;
      if (t < kk) {
        for (int i = 0; i < m; ++i) s = fma(z[i * k + x] - mu[i * k + x], z[i * k + y] - mu[i * k + y], s);
      } else {
        double sx = 0.0, sy = 0.0;
        for (int i = 0; i < m; ++i) {
          sx += z[i * k + x] - mu[i * k + x];
          sy += z[i * k + y] - mu[i * k + y];
        }
        s = fma(sx, sy, s);
      }
    }
    s = warp_sum(s);
    if (lane == 0) a.kk[t] = s / ((double)m * (a.batch - 1));
  }
}

// T (batch x m x k), one thread per (batch row, view)
__device__ void mb_targets(const EyArgs& a, const double* mu, const Smem& sm) {
  const int m = a.m, k = a.k;
  const double scale = 4.0 / ((double)m * (a.batch - 1));
  for (int t = blockIdx.x * blockDim.x + threadIdx.x; t < a.batch * m; t += gridDim.x * blockDim.x) {
    const int b = t / m, i = t % m;
    const double* z = a.ya + (size_t)b * m * k;
    double zc[kEyMaxK], s[kEyMaxK];
#pragma unroll
    for (int x = 0; x < kEyMaxK; ++x)
      if (x < k) {
        zc[x] = z[i * k + x] - mu[i * k + x];
        double acc = 0.0;
        for (int j = 0; j < m; ++j) acc += z[j * k + x] - mu[j * k + x];
        s[x] = acc;
      }
    double* out = a.yb + (size_t)t * k;
#pragma unroll
    for (int y = 0; y < kEyMaxK; ++y)
      if (y < k) {
        double zv = 0.0;
#pragma unroll
        for (int x = 0; x < kEyMaxK; ++x)
          if (x < k) zv = fma(zc[x], sm.vb[x * k + y], zv);
        out[y] = scale * (a.c * zc[y] + (1.0 - a.c) * zv - s[y]);
      }
  }
}

// partials of X_b^T T: one warp per (32 features of one view, batch slice); lanes walk the features (coalesced reads
// of the gathered rows), T is read as a broadcast
template <typename T>
__device__ void mb_gradient(const EyArgs& a, const int32_t* idx) {
  const int lane = threadIdx.x & 31, k = a.k;
  const int ntiles = a.toff[a.m];
  for (int t = gwarp(); t < ntiles * a.nslices; t += nwarps()) {
    const int tile = t % ntiles, sl = t / ntiles;
    int i = 0;
    while (tile >= a.toff[i + 1]) ++i;
    const int p = a.off[i + 1] - a.off[i];
    const int f = (tile - a.toff[i]) * 32 + lane;
    const bool live = f < p;
    const T* X = static_cast<const T*>(a.X[i]);
    double acc[kEyMaxK];
#pragma unroll
    for (int x = 0; x < kEyMaxK; ++x) acc[x] = 0.0;
    const int b1 = min(a.batch, (sl + 1) * a.slice);
    for (int b = sl * a.slice; b < b1; ++b) {
      const double xv = live ? (double)X[(int64_t)idx[b] * a.ld[i] + f] : 0.0;
      const double* tb = a.yb + ((size_t)b * a.m + i) * k;
#pragma unroll
      for (int x = 0; x < kEyMaxK; ++x)
        if (x < k) acc[x] = fma(xv, tb[x], acc[x]);
    }
    if (live) {
#pragma unroll
      for (int x = 0; x < kEyMaxK; ++x)
        if (x < k) a.part[((size_t)sl * k + x) * a.D + a.off[i] + f] = acc[x];
    }
  }
}

// ---- shared: row-local gradient, momentum and weight update ------------------------------------------------------
template <bool COV>
__device__ void update(const EyArgs& a, double* W, double* vel, const Smem& sm) {
  const int k = a.k, D = a.D;
  const double cm = 4.0 * a.c / a.m;
  for (int r = blockIdx.x * blockDim.x + threadIdx.x; r < D; r += gridDim.x * blockDim.x) {
    double w[kEyMaxK], g[kEyMaxK];
#pragma unroll
    for (int x = 0; x < kEyMaxK; ++x)
      if (x < k) w[x] = W[(size_t)x * D + r];
    if (COV) {
      double yd[kEyMaxK];
#pragma unroll
      for (int x = 0; x < kEyMaxK; ++x)
        if (x < k) yd[x] = a.ya[(size_t)x * D + r];
#pragma unroll
      for (int y = 0; y < kEyMaxK; ++y)
        if (y < k) {
          double yv = 0.0;
#pragma unroll
          for (int x = 0; x < kEyMaxK; ++x)
            if (x < k) yv = fma(yd[x], sm.vb[x * k + y], yv);
          g[y] = (4.0 / a.m) * (a.c * yd[y] + (1.0 - a.c) * yv - a.yb[(size_t)y * D + r]);
        }
    } else {
#pragma unroll
      for (int y = 0; y < kEyMaxK; ++y)
        if (y < k) {
          double s = 0.0;
          for (int sl = 0; sl < a.nslices; ++sl) s += a.part[((size_t)sl * k + y) * D + r];
          g[y] = s;
        }
    }
#pragma unroll
    for (int y = 0; y < kEyMaxK; ++y)
      if (y < k) {
        double wv = 0.0;
#pragma unroll
        for (int x = 0; x < kEyMaxK; ++x)
          if (x < k) wv = fma(w[x], sm.vb[x * k + y], wv);
        const double gy = g[y] + cm * wv;
        double* v = vel + (size_t)y * D + r;
        const double nv = a.mom * *v - a.lr * gy;
        *v = nv;
        W[(size_t)y * D + r] = w[y] + nv;
      }
  }
}

// objective from V, C_ey (pre-update representations) and B of the updated weights; every block computes the same
// value in the same order, so all agree on the stop decision without another barrier
__device__ double objective(const EyArgs& a, const double* Bn) {
  const int k = a.k;
  const double* V = a.kk;
  const double* Ce = a.kk + k * k;
  double tr = 0.0, q = 0.0;
  for (int x = 0; x < k; ++x) tr += Ce[x * k + x] - a.c * V[x * k + x];
  for (int x = 0; x < k; ++x)
    for (int y = 0; y < k; ++y)
      q += ((1.0 - a.c) * V[x * k + y] + a.c * Bn[x * k + y]) * ((1.0 - a.c) * V[y * k + x] + a.c * Bn[y * k + x]);
  return -2.0 * tr + q;
}

template <typename T, bool COV>
__global__ void __launch_bounds__(kThreads) ey_steps(EyArgs a) {
  __shared__ Smem sm;
  cg::grid_group grid = cg::this_grid();
  double* hdr = a.state;  // prev_obj, steps, stop, last obj
  double* W = a.state + kEyStateHeader;
  double* vel = W + (size_t)a.k * a.D;
  const int kk = a.k * a.k;
  double* B[2] = {a.kk + 2 * kk, a.kk + 3 * kk};
  double* mu = a.kk + 4 * kk;

  if (hdr[2] != 0.0) return;  // a previous call stopped the fit: every block returns before any barrier
  double prev = hdr[0];
  const double steps0 = hdr[1];
  gram(a, W, B[0]);
  grid.sync();
  for (int t = 0; t < a.n_steps; ++t) {
    const double* Bc = B[t & 1];
    double* Bn = B[(t + 1) & 1];
    if (COV) {
      cov_products(a, W, sm);
      grid.sync();
      cov_kk(a, W);
      grid.sync();
      blend(a, a.kk, Bc, sm);
      update<true>(a, W, vel, sm);
    } else {
      const int32_t* idx = a.idx + (size_t)t * a.batch;
      mb_project<T>(a, idx, W, sm);
      grid.sync();
      mb_means(a, mu);
      grid.sync();
      mb_kk(a, mu);
      grid.sync();
      blend(a, a.kk, Bc, sm);
      mb_targets(a, mu, sm);
      grid.sync();
      mb_gradient<T>(a, idx);
      grid.sync();
      update<false>(a, W, vel, sm);
    }
    grid.sync();
    gram(a, W, Bn);
    grid.sync();
    if (threadIdx.x == 0) {
      const double obj = objective(a, Bn);
      sm.obj = obj;
      sm.stop = fabs(prev - obj) < a.tol ? 1 : 0;
      if (blockIdx.x == 0) {
        hdr[0] = obj;
        hdr[1] = steps0 + t + 1;
        hdr[2] = sm.stop ? 1.0 : 0.0;
        hdr[3] = fabs(prev - obj);
      }
    }
    __syncthreads();
    prev = sm.obj;
    const bool stop = sm.stop != 0;
    if (stop) break;
  }
}

struct EyWorkspace {
  size_t ya, yb, part, kk, total;  // byte offsets
  int nslices, slice;
};

EyWorkspace ey_workspace(const ColumnLayout& L, int k, int batch) {
  auto al = [](size_t x) { return (x + 255) / 256 * 256; };
  const size_t D = (size_t)L.D, m = (size_t)L.n_views, K = (size_t)k;
  EyWorkspace w;
  w.nslices = batch > 0 ? (int)std::min<int64_t>(kMaxSlices, ceil_div(batch, kSliceRows)) : 0;
  w.slice = batch > 0 ? (int)ceil_div(batch, w.nslices) : 0;
  const size_t rows = batch > 0 ? 8 * (size_t)batch * m * K : 8 * K * D;
  w.ya = 0;
  w.yb = w.ya + al(rows);
  w.part = w.yb + al(rows);
  w.kk = w.part + al(8 * (size_t)w.nslices * K * D);
  w.total = w.kk + al(8 * (4 * K * K + m * K));
  return w;
}

template <typename T, bool COV>
int launch(EyArgs& a, cudaStream_t stream) {
  const void* fn = (const void*)ey_steps<T, COV>;
  int dev = 0, sms = 0, per_sm = 0;
  CCAB_CUDA(cudaGetDevice(&dev));
  CCAB_CUDA(cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, dev));
  CCAB_CUDA(cudaOccupancyMaxActiveBlocksPerMultiprocessor(&per_sm, fn, kThreads, 0));
  CCAB_CHECK_ARG(per_sm >= 1, "the EY kernel cannot be resident on this device");
  void* args[] = {&a};
  CCAB_CUDA(cudaLaunchCooperativeKernel(fn, dim3(per_sm * sms), dim3(kThreads), args, 0, stream));
  count_launches(1);
  return 0;
}

}  // namespace

size_t ey_fit_workspace_bytes(const ColumnLayout& L, int k, int batch) { return ey_workspace(L, k, batch).total + 256; }

int ey_fit(const ColumnLayout& L, const EyParams& p, const double* cov, int dtype, const void* const* views,
           const int64_t* ld, const int32_t* idx, double* state, void* ws, size_t ws_bytes, cudaStream_t stream) {
  CCAB_CHECK_ARG(ws_bytes >= ey_fit_workspace_bytes(L, p.k, p.batch), "workspace too small: %zu < %zu", ws_bytes,
                 ey_fit_workspace_bytes(L, p.k, p.batch));
  if (p.n_steps == 0) return 0;
  const EyWorkspace o = ey_workspace(L, p.k, p.batch);
  uintptr_t base = ((uintptr_t)ws + 255) / 256 * 256;
  EyArgs a;
  a.m = L.n_views;
  a.D = L.D;
  a.k = p.k;
  a.batch = p.batch;
  a.n_steps = p.n_steps;
  a.nslices = o.nslices;
  a.slice = o.slice;
  a.toff[0] = 0;
  for (int v = 0; v <= L.n_views; ++v) a.off[v] = L.coff[v];
  for (int v = 0; v < L.n_views; ++v) a.toff[v + 1] = a.toff[v] + (int)ceil_div(L.dims[v], 32);
  a.c = p.c;
  a.lr = p.lr;
  a.mom = p.momentum;
  a.tol = p.tol;
  a.cov = cov;
  for (int v = 0; v < kMaxViews; ++v) {
    a.X[v] = v < L.n_views && views ? views[v] : nullptr;
    a.ld[v] = v < L.n_views && ld ? ld[v] : 0;
  }
  a.idx = idx;
  a.state = state;
  a.ya = reinterpret_cast<double*>(base + o.ya);
  a.yb = reinterpret_cast<double*>(base + o.yb);
  a.part = reinterpret_cast<double*>(base + o.part);
  a.kk = reinterpret_cast<double*>(base + o.kk);
  if (p.batch == 0) return launch<double, true>(a, stream);
  if (dtype == 0) return launch<float, false>(a, stream);
  return launch<double, false>(a, stream);
}

}  // namespace ccab
