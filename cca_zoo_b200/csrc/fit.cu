// Fit assembly on the device: from the (all-reduced) moment buffer to the weights, as ONE asynchronous call per
// estimator -- no host read-back between the moment pass and the result (SURVEY.md §8b: the fit behind the C ABI).
//
//   rcca_fit : cca_zoo/linear/_rcca.py:83-101 in covariance / Cholesky form
//       C = (M - s s^T / n) / (n - 1)                      cov_ridge_kernel (also R_i = (1-c_i) C_ii + c_i I, max diag,
//                                                           finiteness flag; n is read from device memory)
//       R_i = L_i L_i^T, Linv_i = L_i^-1                    potrf_inv (cholinv.cu), both views batched when d1 == d2
//       T = Linv_1 C_12 Linv_2^T                            2 GEMMs (tgemm.cu for float)
//       leading k singular triplets of T                    blocked subspace iteration: Z <- orth(T^T T Z) with CholQR
//                                                           (Gram GEMM + single-launch Cholesky/inverse + GEMM), then
//                                                           Rayleigh-Ritz through the single-CTA Jacobi eigensolver
//       weights_i = Linv_i^T U_k / V_k                      2 GEMMs, written into the result block
//   Every decision the host used to take from a read-back (pivot failures, CholQR rank loss, convergence of the
//   iteration, finiteness of the input, n > d) is written into the header of the result block instead; the host copies
//   the block once, checks the status word and re-runs through the eigen route when it is non-zero.
#include "fit.cuh"

#include <cmath>
#include <type_traits>

#include "ccaloss.cuh"
#include "cholinv.cuh"
#include "dense.cuh"
#include "moments.cuh"
#include "syevj_small.cuh"

namespace ccab {

namespace {

inline size_t al256(size_t x) { return (x + 255) & ~size_t(255); }
inline int64_t r4(int64_t x) { return (x + 3) & ~int64_t(3); }

struct CovRidgeParams {
  int n_views, D, Dp;
  int dims[kMaxViews];
  int coff[kMaxViews + 1];
  int poff[kMaxViews + 1];
  double c[kMaxViews];
  double ridge_add[kMaxViews]; // R_v = (1 - c_v) C_vv + (c_v + ridge_add_v) I
  void* R[kMaxViews];          // ridge block of view v (may be NULL)
  long long ldr[kMaxViews];
};
struct PivotTolParams {
  int n_views;
  double c[kMaxViews], rank_tol[kMaxViews];
  double floor;   // lower bound of the tolerance (MCCA's eps floor: lambda_min(B) < eps must not pass)
};

__device__ __forceinline__ int view_of(const CovRidgeParams& p, int g) {
  int v = 0;
  while (v + 1 < p.n_views && p.coff[v + 1] <= g) ++v;
  return v;
}

// C (D x D, ldc) = covariance from the moments; R_v (dims[v] x dims[v], ldr[v]) = (1 - c_v) C_vv + c_v I;
// dmax[v] = max diag(C_vv) (float bits, atomicMax: non-negative values order like integers); flags[0] |= 1 when a
// moment is not finite; mean (double[D]).
template <typename T>
__global__ void cov_ridge_kernel(const CovRidgeParams p, const double* __restrict__ mom, const double* __restrict__ n_dev,
                                 double n_host, int center, T* __restrict__ C, int64_t ldc, double* __restrict__ mean,
                                 unsigned* __restrict__ dmax, int* __restrict__ flags) {
  const double n_total = n_dev ? n_dev[0] : n_host;
  const double* M = mom;
  const double* s = mom + (size_t)p.Dp * p.Dp;
  const int gi = blockIdx.y * blockDim.y + threadIdx.y;
  const int gj = blockIdx.x * blockDim.x + threadIdx.x;
  if (gi >= p.D || gj >= p.D) return;
  const int vi = view_of(p, gi), vj = view_of(p, gj);
  const int pi = p.poff[vi] + gi - p.coff[vi], pj = p.poff[vj] + gj - p.coff[vj];
  const int r = min(pi, pj), c = max(pi, pj);
  double v = M[(size_t)r * p.Dp + c];
  if (!isfinite(v)) atomicOr(flags, 1);
  if (center) v -= s[pi] * s[pj] / n_total;
  v /= (n_total - 1.0);
  C[(size_t)gi * ldc + gj] = (T)v;
  if (vi == vj && p.R[vi]) {
    const double cv = p.c[vi];
    const double rv = (1.0 - cv) * v + (gi == gj ? cv + p.ridge_add[vi] : 0.0);
    static_cast<T*>(p.R[vi])[(size_t)(gi - p.coff[vi]) * p.ldr[vi] + (gj - p.coff[vj])] = (T)rv;
    if (gi == gj && dmax) atomicMax(dmax + vi, __float_as_uint(fmaxf((float)v, 0.f)));
  }
  if (gi == 0 && mean) mean[gj] = center ? s[pj] / n_total : 0.0;
  if (gi == 0 && gj == 0 && !(n_total >= 2.0)) atomicOr(flags, 2);
}

// pivot tolerance of view v: rank_tol_v * ((1 - c_v) dmax_v + c_v)   (the covariance-space image of the reference's
// s > 0 filter on the regularised spectrum, _solvers._rank_tol)
__global__ void pivot_tol_kernel(const PivotTolParams q, const unsigned* __restrict__ dmax, double* __restrict__ tol) {
  const int v = threadIdx.x;
  if (v < q.n_views) tol[v] = fmax(q.floor, q.rank_tol[v] * ((1.0 - q.c[v]) * (double)__uint_as_float(dmax[v]) + q.c[v]));
}

// counter-based standard normal start block (splitmix64 hash + Box-Muller): reproducible, no generator state
template <typename T>
__global__ void randn_kernel(T* __restrict__ Z, int64_t ld, int rows, int cols, unsigned long long seed) {
  const size_t total = (size_t)rows * cols;
  for (size_t e = blockIdx.x * (size_t)blockDim.x + threadIdx.x; e < total; e += (size_t)gridDim.x * blockDim.x) {
    unsigned long long x = seed + 0x9E3779B97F4A7C15ull * (e + 1);
    x = (x ^ (x >> 30)) * 0xBF58476D1CE4E5B9ull;
    x = (x ^ (x >> 27)) * 0x94D049BB133111EBull;
    x ^= x >> 31;
    const double u1 = ((double)(unsigned)(x >> 32) + 1.0) * (1.0 / 4294967297.0);
    const double u2 = (double)(unsigned)(x & 0xffffffffu) * (1.0 / 4294967296.0);
    const double g = sqrt(-2.0 * log(u1)) * cospi(2.0 * u2);
    Z[(e / cols) * ld + (e % cols)] = (T)g;
  }
}

// sig_j = sqrt(max(lam_j, 0)) for j < k; U[:, j] *= 1 / sig_j (0 when sig_j == 0)
template <typename T>
__global__ void ritz_scale_kernel(T* __restrict__ U, int64_t ldu, int rows, int k, const T* __restrict__ lam,
                                  T* __restrict__ sig) {
  const int j = blockIdx.x * blockDim.x + threadIdx.x;
  const int i = blockIdx.y;
  if (j >= k) return;
  const T s = sqrt(fmax(lam[j], T(0)));
  if (i == 0 && sig) sig[j] = s;
  U[(size_t)i * ldu + j] *= s > T(0) ? T(1) / s : T(0);
}

// stats[0] = || E - V diag(sig) ||_F^2, stats[1] = sig_0 (sym: |sig_0| + shift).  Row slabs over the blocks, partial
// sums added in block order by the last block to finish (counter zeroed by the caller): deterministic, one launch.
constexpr int kResidBlocks = 64;
template <typename T>
__global__ void __launch_bounds__(256)
residual_kernel(const T* __restrict__ E, int64_t lde, const T* __restrict__ V, int64_t ldv, int rows, int k,
                const T* __restrict__ sig, double shift, int sym, double* __restrict__ stats,
                double* __restrict__ partial, unsigned* __restrict__ counter) {
  __shared__ double red[8];
  __shared__ bool last;
  const int per = (rows + gridDim.x - 1) / gridDim.x;
  const int r0 = blockIdx.x * per;
  const int nr = max(0, min(rows, r0 + per) - r0);
  double acc = 0.0;
  for (int e = threadIdx.x; e < nr * k; e += blockDim.x) {
    const int i = r0 + e / k, j = e % k;
    const double d = (double)E[(size_t)i * lde + j] - (double)V[(size_t)i * ldv + j] * (double)sig[j];
    acc += d * d;
  }
  for (int o = 16; o > 0; o >>= 1) acc += __shfl_xor_sync(0xffffffffu, acc, o);
  if ((threadIdx.x & 31) == 0) red[threadIdx.x >> 5] = acc;
  __syncthreads();
  if (threadIdx.x == 0) {
    double t = 0.0;
    for (int w = 0; w < (int)(blockDim.x >> 5); ++w) t += red[w];
    partial[blockIdx.x] = t;
    __threadfence();
    last = atomicAdd(counter, 1u) == gridDim.x - 1;
    if (last) {
      __threadfence();
      double tot = 0.0;
      for (unsigned b = 0; b < gridDim.x; ++b) tot += *reinterpret_cast<volatile double*>(partial + b);
      stats[0] = tot;
      stats[1] = sym ? fabs((double)sig[0]) + shift : (double)sig[0];
      *counter = 0u;
    }
  }
}

// header of the result block: see FitHeader in fit.cuh
__global__ void fit_status_kernel(double* __restrict__ hdr, const int* __restrict__ flags, const int* __restrict__ infos,
                                  int n_infos, const int* __restrict__ rr_info, const double* __restrict__ stats,
                                  const double* __restrict__ n_dev, double n_host, double resid_tol, int k, int max_d) {
  if (threadIdx.x != 0) return;
  const double n_total = n_dev ? n_dev[0] : n_host;
  int status = 0;
  if (flags[0] & 1) status |= kFitNonFinite;
  if (flags[0] & 2) status |= kFitTooFewSamples;
  int first_bad = 0;
  for (int i = 0; i < n_infos; ++i)
    if (infos[i] != 0 && !first_bad) first_bad = i + 1;
  if (first_bad) status |= kFitNotPositiveDefinite;
  const double resid = sqrt(fmax(stats[0], 0.0)), s1 = stats[1];
  if (!(s1 > 0.0) || !(resid <= resid_tol * s1 * sqrt((double)k))) status |= kFitNotConverged;
  if (rr_info && rr_info[0] <= 0) status |= kFitNotConverged;
  if (!(n_total > (double)max_d)) status |= kFitTooFewSamples;
  hdr[0] = (double)status;
  hdr[1] = n_total;
  hdr[2] = resid;
  hdr[3] = s1;
  hdr[4] = (double)first_bad;
  hdr[5] = rr_info ? (double)rr_info[0] : 0.0;
}

template <typename T>
double eps_of() {
  return std::is_same<T, float>::value ? 1.1920928955078125e-7 : 2.220446049250313e-16;
}
// residual tolerance of the subspace iteration relative to sigma_1 sqrt(k): 200 eps in float, and no tighter than 1e-10
// in double -- the vectors are then accurate to 1e-10 / gap, far inside the 1e-5 parity bar, while 200 eps (4e-14) would
// cost twice the iterations for nothing
template <typename T>
double resid_tol_of() {
  return std::max(200.0 * eps_of<T>(), 1e-10);
}

// ---------------------------------------------------------------------------------------------
// CholQR: Zout (rows x p) = Zin * chol(Zin^T Zin)^-T ; info slot must be zero on entry
// ---------------------------------------------------------------------------------------------
template <typename T>
struct CholQrWs {
  T* G;      // p x ldg
  T* Ginv;   // max(p, NB) square
  void* pws;
  size_t pws_bytes;
  int64_t ldg;
  void* splitk_ws = nullptr;   // scratch for the split reduction of the (single-tile, long-k) Gram product in float64
  size_t splitk_ws_bytes = 0;
};

template <typename T>
int cholqr(const T* Zin, int64_t ldz, T* Zout, int64_t ldo, int rows, int p, const CholQrWs<T>& w, int* info,
           cudaStream_t s) {
  GemmArgs<T> g;
  g.transa = 1; g.m = p; g.n = p; g.k = rows;
  g.A = Zin; g.lda = ldz; g.B = Zin; g.ldb = ldz; g.C = w.G; g.ldc = w.ldg;
  g.splitk_ws = w.splitk_ws; g.splitk_ws_bytes = w.splitk_ws_bytes;
  int rc = xgemm<T>(g, s);
  if (rc) return rc;
  const int NB = potrf_inv_block_size<T>();
  int64_t ldi;
  if (p <= NB) {
    rc = potrf_inv_block<T>(w.G, w.ldg, 0, p, 0, w.Ginv, 0, 0.0, nullptr, info, 1, s);
    ldi = NB;
  } else {
    int* tmp_info = info;   // potrf_inv clears its info slot itself: accumulate through a scratch int
    rc = potrf_inv<T>(p, 1, w.G, w.ldg, 0, w.Ginv, w.ldg, 0, 0.0, nullptr, tmp_info, w.pws, w.pws_bytes, s);
    ldi = w.ldg;
  }
  if (rc) return rc;
  GemmArgs<T> q;   // Zout = Zin * Ginv^T
  q.transb = 1; q.m = rows; q.n = p; q.k = p;
  q.A = Zin; q.lda = ldz; q.B = w.Ginv; q.ldb = ldi; q.C = Zout; q.ldc = ldo;
  return xgemm<T>(q, s);
}

struct RccaPlan {
  int d1, d2, D, k, p;
  int64_t ldC, ld1, ld2, ldT, ldp, ldk;
  size_t oC, oR, oLinv, oT1, oT, oZ, oZ2, oY, oG, oGinv, oH, oLam, oVy, oU, oV, oE, oPws, oSplit, oSmall, total;
  size_t pws_bytes, split_bytes;
  size_t r_mean, r_sig, r_w1, r_w2, r_total;
};

template <typename T>
RccaPlan make_rcca_plan(int d1, int d2, int k, int p) {
  RccaPlan P;
  P.d1 = d1; P.d2 = d2; P.D = d1 + d2; P.k = k; P.p = p;
  P.ldC = r4(P.D); P.ld1 = r4(d1); P.ld2 = r4(d2); P.ldT = r4(d2); P.ldp = r4(p); P.ldk = r4(k);
  const int NB = potrf_inv_block_size<T>();
  const int dm = std::max(d1, d2);
  size_t o = 0;
  auto take = [&](size_t elems) { size_t at = o; o += al256(elems * sizeof(T)); return at; };
  P.oC = take((size_t)P.D * P.ldC);
  // the two ridge blocks / inverses as ONE strided batch when the views have the same width
  P.oR = take(2 * (size_t)dm * r4(dm));
  P.oLinv = take(2 * (size_t)dm * r4(dm));
  P.oT1 = take((size_t)d1 * P.ldT);
  P.oT = take((size_t)d1 * P.ldT);
  P.oZ = take((size_t)d2 * P.ldp);
  P.oZ2 = take((size_t)d2 * P.ldp);
  P.oY = take((size_t)d1 * P.ldp);
  P.oG = take((size_t)p * P.ldp);
  P.oGinv = take((size_t)std::max(p, NB) * std::max<int64_t>(P.ldp, NB));
  P.oH = take((size_t)p * P.ldp);
  P.oLam = take((size_t)p);
  P.oVy = take((size_t)p * P.ldp);
  P.oU = take((size_t)d1 * P.ldk);
  P.oV = take((size_t)d2 * P.ldk);
  P.oE = take((size_t)d2 * P.ldk);
  P.pws_bytes = std::max(potrf_inv_workspace_bytes<T>(dm, 2), potrf_inv_workspace_bytes<T>(p, 1));
  P.oPws = o; o += al256(P.pws_bytes);
  P.split_bytes = 8 * (size_t)dm * r4(std::max(p, k)) * sizeof(T);   // k-slices of the thin products (xgemm)
  P.oSplit = o; o += al256(P.split_bytes);
  P.oSmall = o; o += 4096;   // flags, infos, dmax, tolerances, stats, device pointer tables
  P.total = o + 256;
  size_t r = sizeof(double) * kFitHeaderDoubles;
  P.r_mean = r; r += al256(sizeof(double) * P.D);
  P.r_sig = r; r += al256(sizeof(T) * k);
  P.r_w1 = r; r += al256(sizeof(T) * (size_t)d1 * k);
  P.r_w2 = r; r += al256(sizeof(T) * (size_t)d2 * k);
  P.r_total = r;
  return P;
}

}  // namespace

// 0 for every shape rcca_fit refuses: the workspace query is also the question "does the one-call fit take this?"
template <typename T>
size_t rcca_fit_workspace_bytes(int d1, int d2, int k, int p) {
  if (!(k >= 1 && p >= k && p <= std::min(d1, d2) && syevj_small_supported<T>(p))) return 0;
  return make_rcca_plan<T>(d1, d2, k, p).total;
}

template <typename T>
void rcca_fit_result_layout(int d1, int d2, int k, int p, int64_t* offsets) {
  RccaPlan P = make_rcca_plan<T>(d1, d2, k, p);
  offsets[0] = (int64_t)P.r_mean;
  offsets[1] = (int64_t)P.r_sig;
  offsets[2] = (int64_t)P.r_w1;
  offsets[3] = (int64_t)P.r_w2;
  offsets[4] = (int64_t)P.r_total;
}

template <typename T>
int rcca_fit(const ColumnLayout& L, const double* moments, const double* n_dev, double n_host, int center,
             const double* c, int k, int p, int iters, void* result, size_t result_bytes, void* ws, size_t ws_bytes,
             cudaStream_t s) {
  CCAB_CHECK_ARG(L.n_views == 2, "rcca_fit needs exactly 2 views");
  const int d1 = L.dims[0], d2 = L.dims[1], D = L.D;
  CCAB_CHECK_ARG(k >= 1 && p >= k && p <= std::min(d1, d2), "rcca_fit: need 1 <= k <= p <= min(d1, d2), got k=%d p=%d", k,
                 p);
  CCAB_CHECK_ARG(syevj_small_supported<T>(p), "rcca_fit: subspace width %d exceeds the single-CTA eigensolver", p);
  CCAB_CHECK_ARG(iters >= 1 && iters <= 64, "rcca_fit: bad iteration count %d", iters);
  RccaPlan P = make_rcca_plan<T>(d1, d2, k, p);
  CCAB_CHECK_ARG(ws_bytes >= P.total, "rcca_fit workspace too small: %zu < %zu", ws_bytes, P.total);
  CCAB_CHECK_ARG(result_bytes >= P.r_total, "rcca_fit result block too small: %zu < %zu", result_bytes, P.r_total);
  uint8_t* w = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(ws) + 255) & ~uintptr_t(255));
  uint8_t* res = static_cast<uint8_t*>(result);
  CCAB_CHECK_ARG((reinterpret_cast<uintptr_t>(res) & 255) == 0, "rcca_fit: result block must be 256-byte aligned");
  auto at = [&](size_t off) { return reinterpret_cast<T*>(w + off); };
  T* C = at(P.oC);
  const bool batched = d1 == d2;
  const int64_t ldR = r4(std::max(d1, d2));
  const int64_t strideR = (int64_t)std::max(d1, d2) * ldR;
  T* R1 = at(P.oR);
  T* R2 = R1 + strideR;
  T* Li1 = at(P.oLinv);
  T* Li2 = Li1 + strideR;
  const int64_t ldr1 = batched ? ldR : P.ld1, ldr2 = batched ? ldR : P.ld2;
  T *T1 = at(P.oT1), *Tm = at(P.oT), *Z = at(P.oZ), *Z2 = at(P.oZ2), *Y = at(P.oY), *H = at(P.oH), *lam = at(P.oLam),
    *Vy = at(P.oVy), *U = at(P.oU), *V = at(P.oV), *E = at(P.oE);
  CholQrWs<T> cq;
  cq.G = at(P.oG);
  cq.Ginv = at(P.oGinv);
  cq.pws = w + P.oPws;
  cq.pws_bytes = P.pws_bytes;
  cq.ldg = P.ldp;
  cq.splitk_ws = w + P.oSplit;
  cq.splitk_ws_bytes = P.split_bytes;
  auto thin = [&](GemmArgs<T>& g) { g.splitk_ws = cq.splitk_ws; g.splitk_ws_bytes = cq.splitk_ws_bytes; };
  // small device scratch
  uint8_t* sm = w + P.oSmall;
  int* flags = reinterpret_cast<int*>(sm);                     // [1]
  int* infos = flags + 4;                                      // [2 + iters + 2] potrf, CholQR passes
  const int n_infos = 2 + iters + 2;
  int* rr_info = infos + 80;                                   // [1]
  unsigned* dmax = reinterpret_cast<unsigned*>(sm + 512);      // [2]
  double* tol = reinterpret_cast<double*>(sm + 1024);          // [2]
  double* stats = tol + 8;                                     // [2]
  double* resid_part = reinterpret_cast<double*>(sm + 1280);   // [kResidBlocks]
  unsigned* resid_cnt = reinterpret_cast<unsigned*>(sm + 1280 + 8 * kResidBlocks);

  CCAB_CUDA(cudaMemsetAsync(sm, 0, 2048, s));
  double* hdr = reinterpret_cast<double*>(res);
  double* mean = reinterpret_cast<double*>(res + P.r_mean);
  T* sig = reinterpret_cast<T*>(res + P.r_sig);
  T* W1 = reinterpret_cast<T*>(res + P.r_w1);
  T* W2 = reinterpret_cast<T*>(res + P.r_w2);

  // ---- covariance + ridge blocks ----
  {
    CovRidgeParams cp;
    memset(&cp, 0, sizeof(cp));
    cp.n_views = 2; cp.D = D; cp.Dp = L.Dp;
    for (int v = 0; v < 2; ++v) { cp.dims[v] = L.dims[v]; cp.c[v] = c[v]; }
    for (int v = 0; v <= 2; ++v) { cp.coff[v] = L.coff[v]; cp.poff[v] = L.poff[v]; }
    cp.R[0] = R1; cp.R[1] = R2; cp.ldr[0] = ldr1; cp.ldr[1] = ldr2;
    dim3 block(32, 8), grid((unsigned)ceil_div(D, 32), (unsigned)ceil_div(D, 8));
    cov_ridge_kernel<T><<<grid, block, 0, s>>>(cp, moments, n_dev, n_host, center, C, P.ldC, mean, dmax, flags);
    count_launches(1);
    PivotTolParams q;
    memset(&q, 0, sizeof(q));
    q.n_views = 2;
    q.c[0] = c[0]; q.c[1] = c[1];
    q.rank_tol[0] = d1 * eps_of<T>(); q.rank_tol[1] = d2 * eps_of<T>();
    pivot_tol_kernel<<<1, 32, 0, s>>>(q, dmax, tol);
    count_launches(1);
    CCAB_CUDA(cudaGetLastError());
  }
  // ---- Cholesky + inverse of both ridge blocks ----
  int rc;
  if (batched) {
    rc = potrf_inv<T>(d1, 2, R1, ldR, strideR, Li1, ldR, strideR, 0.0, tol, infos, cq.pws, cq.pws_bytes, s);
    if (rc) return rc;
  } else {
    rc = potrf_inv<T>(d1, 1, R1, ldr1, 0, Li1, ldr1, 0, 0.0, tol, infos, cq.pws, cq.pws_bytes, s);
    if (rc) return rc;
    rc = potrf_inv<T>(d2, 1, R2, ldr2, 0, Li2, ldr2, 0, 0.0, tol + 1, infos + 1, cq.pws, cq.pws_bytes, s);
    if (rc) return rc;
  }
  // ---- T = Linv1 C12 Linv2^T ----
  {
    GemmArgs<T> g;
    g.m = d1; g.n = d2; g.k = d1;
    g.A = Li1; g.lda = ldr1; g.B = C + d1; g.ldb = P.ldC; g.C = T1; g.ldc = P.ldT;
    rc = xgemm<T>(g, s);
    if (rc) return rc;
    GemmArgs<T> h;
    h.transb = 1; h.m = d1; h.n = d2; h.k = d2;
    h.A = T1; h.lda = P.ldT; h.B = Li2; h.ldb = ldr2; h.C = Tm; h.ldc = P.ldT;
    rc = xgemm<T>(h, s);
    if (rc) return rc;
  }
  // ---- subspace iteration: Z <- orth(T^T (T Z)) ----
  {
    const size_t total = (size_t)d2 * p;
    randn_kernel<T><<<(unsigned)std::min<size_t>((total + 255) / 256, 592), 256, 0, s>>>(Z, P.ldp, d2, p, 0x1234ull);
    count_launches(1);
    CCAB_CUDA(cudaGetLastError());
  }
  int info_slot = 2;
  // With d2 <= d1 the Gram matrix A = T^T T fits the (now free) T1 buffer: one product per iteration instead of two.
  // Only the SUBSPACE is iterated with A (its rounding moves the dominant subspace by ~eps); the Rayleigh-Ritz step
  // and the residual below use T itself.
  const bool gram = d2 <= d1 && iters >= 2;
  if (gram) {
    GemmArgs<T> g;
    g.transa = 1; g.m = d2; g.n = d2; g.k = d1; g.A = Tm; g.lda = P.ldT; g.B = Tm; g.ldb = P.ldT; g.C = T1; g.ldc = P.ldT;
    rc = xgemm<T>(g, s);
    if (rc) return rc;
  }
  for (int it = 0; it < iters; ++it) {
    if (gram) {
      GemmArgs<T> a;   // Z2 = (T^T T) Z, as A^T Z: the k-slices of both operands are then whole row blocks
      a.transa = 1; a.m = d2; a.n = p; a.k = d2; a.A = T1; a.lda = P.ldT; a.B = Z; a.ldb = P.ldp; a.C = Z2; a.ldc = P.ldp;
      thin(a);
      rc = xgemm<T>(a, s);
      if (rc) return rc;
    } else {
      GemmArgs<T> a;   // Y = T Z
      a.m = d1; a.n = p; a.k = d2; a.A = Tm; a.lda = P.ldT; a.B = Z; a.ldb = P.ldp; a.C = Y; a.ldc = P.ldp;
      rc = xgemm<T>(a, s);
      if (rc) return rc;
      GemmArgs<T> b;   // Z2 = T^T Y
      b.transa = 1; b.m = d2; b.n = p; b.k = d1; b.A = Tm; b.lda = P.ldT; b.B = Y; b.ldb = P.ldp; b.C = Z2; b.ldc = P.ldp;
      rc = xgemm<T>(b, s);
      if (rc) return rc;
    }
    rc = cholqr<T>(Z2, P.ldp, Z, P.ldp, d2, p, cq, infos + info_slot++, s);
    if (rc) return rc;
    if (it == iters - 1) {   // second pass on the last iterate: orthonormal to working precision
      rc = cholqr<T>(Z, P.ldp, Z2, P.ldp, d2, p, cq, infos + info_slot++, s);
      if (rc) return rc;
      std::swap(Z, Z2);
    }
  }
  // ---- Rayleigh-Ritz on Y = T Z: Y^T Y = Vy diag(sig^2) Vy^T ; U = Y Vy diag(1/sig), V = Z Vy ----
  {
    GemmArgs<T> a;
    a.m = d1; a.n = p; a.k = d2; a.A = Tm; a.lda = P.ldT; a.B = Z; a.ldb = P.ldp; a.C = Y; a.ldc = P.ldp;
    thin(a);
    rc = xgemm<T>(a, s);
    if (rc) return rc;
    GemmArgs<T> h;
    h.transa = 1; h.m = p; h.n = p; h.k = d1; h.A = Y; h.lda = P.ldp; h.B = Y; h.ldb = P.ldp; h.C = H; h.ldc = P.ldp;
    thin(h);
    rc = xgemm<T>(h, s);
    if (rc) return rc;
    rc = syevj_small<T>(p, 1, H, P.ldp, 0, lam, p, Vy, P.ldp, 0, rr_info, s);
    if (rc) return rc;
    GemmArgs<T> u;   // U = Y Vy_k   (rows of Vy are the eigenvectors: op(B) = Vy[:k]^T)
    u.transb = 1; u.m = d1; u.n = k; u.k = p; u.A = Y; u.lda = P.ldp; u.B = Vy; u.ldb = P.ldp; u.C = U; u.ldc = P.ldk;
    rc = xgemm<T>(u, s);
    if (rc) return rc;
    ritz_scale_kernel<T><<<dim3((unsigned)ceil_div(k, 128), (unsigned)d1), 128, 0, s>>>(U, P.ldk, d1, k, lam, sig);
    count_launches(1);
    GemmArgs<T> v;   // V = Z Vy_k
    v.transb = 1; v.m = d2; v.n = k; v.k = p; v.A = Z; v.lda = P.ldp; v.B = Vy; v.ldb = P.ldp; v.C = V; v.ldc = P.ldk;
    rc = xgemm<T>(v, s);
    if (rc) return rc;
    GemmArgs<T> e;   // E = T^T U  (compare with V diag(sig))
    e.transa = 1; e.m = d2; e.n = k; e.k = d1; e.A = Tm; e.lda = P.ldT; e.B = U; e.ldb = P.ldk; e.C = E; e.ldc = P.ldk;
    thin(e);
    rc = xgemm<T>(e, s);
    if (rc) return rc;
    residual_kernel<T><<<kResidBlocks, 256, 0, s>>>(E, P.ldk, V, P.ldk, d2, k, sig, 0.0, 0, stats, resid_part, resid_cnt);
    count_launches(1);
    CCAB_CUDA(cudaGetLastError());
  }
  // ---- weights = Linv^T U / V ----
  {
    GemmArgs<T> a;
    a.transa = 1; a.m = d1; a.n = k; a.k = d1; a.A = Li1; a.lda = ldr1; a.B = U; a.ldb = P.ldk; a.C = W1; a.ldc = k;
    thin(a);
    rc = xgemm<T>(a, s);
    if (rc) return rc;
    GemmArgs<T> b;
    b.transa = 1; b.m = d2; b.n = k; b.k = d2; b.A = Li2; b.lda = ldr2; b.B = V; b.ldb = P.ldk; b.C = W2; b.ldc = k;
    thin(b);
    rc = xgemm<T>(b, s);
    if (rc) return rc;
  }
  fit_status_kernel<<<1, 32, 0, s>>>(hdr, flags, infos, n_infos, rr_info, stats, n_dev, n_host, resid_tol_of<T>(), k,
                                    std::max(d1, d2));
  count_launches(1);
  CCAB_CUDA(cudaGetLastError());
  return 0;
}


// =============================================================================================================
// mcca_fit : cca_zoo/linear/_mcca.py:113-173 (pca=False form) through the Cholesky reduction of A v = lam B v
//   B_i = (1-c_i) C_ii + c_i I = L_i L_i^T (batched when the views have one width), K_ij = L_i^-1 C_ij L_j^-T (i != j,
//   zero diagonal blocks), largest k eigenpairs of K by blocked subspace iteration on K + shift I
//   (shift = 1 / (1 - max c) >= -lambda_min(K): the whitened cross blocks have ||K|| <= (m-1) / (1 - max c) ... the
//   shift only has to make the iterated matrix positive on the wanted end), Rayleigh-Ritz through the two-sided
//   single-CTA Jacobi (which needs no shift), v_i = sqrt(m) L_i^-T y_i  (v^T B v = 1 with B / m, scipy's normalisation).
//   The eps floor of _build_B (:170-172) is only active when lambda_min(B) < eps: the pivot tolerance of the Cholesky
//   is raised to eps so that such problems fail the factorisation and are declined to the host-assembled eigen route.
// =============================================================================================================
namespace {

struct MccaPlan {
  int m, D, k, p, dmax;
  bool equal;
  int64_t ldC, ldR, strideR, ldp, ldk;
  int off[kMaxViews + 1];
  size_t oC, oR, oLinv, oTmp, oK, oZ, oZ2, oY, oG, oGinv, oH, oLam, oVy, oZr, oE, oPws, oSplit, oSmall, total;
  size_t pws_bytes, split_bytes;
  size_t r_mean, r_val, r_w[kMaxViews], r_total;
};

template <typename T>
MccaPlan make_mcca_plan(const ColumnLayout& L, int k, int p) {
  MccaPlan P;
  P.m = L.n_views; P.D = L.D; P.k = k; P.p = p;
  P.dmax = 0;
  P.equal = true;
  for (int v = 0; v < P.m; ++v) {
    P.dmax = std::max(P.dmax, L.dims[v]);
    if (L.dims[v] != L.dims[0]) P.equal = false;
    P.off[v] = L.coff[v];
  }
  P.off[P.m] = L.D;
  P.ldC = r4(P.D); P.ldR = r4(P.dmax); P.strideR = (int64_t)P.dmax * P.ldR; P.ldp = r4(p); P.ldk = r4(k);
  const int NB = potrf_inv_block_size<T>();
  size_t o = 0;
  auto take = [&](size_t elems) { size_t at = o; o += al256(elems * sizeof(T)); return at; };
  P.oC = take((size_t)P.D * P.ldC);
  P.oR = take((size_t)P.m * P.strideR);
  P.oLinv = take((size_t)P.m * P.strideR);
  P.oTmp = take((size_t)P.dmax * P.ldR);
  P.oK = take((size_t)P.D * P.ldC);
  P.oZ = take((size_t)P.D * P.ldp);
  P.oZ2 = take((size_t)P.D * P.ldp);
  P.oY = take((size_t)P.D * P.ldp);
  P.oG = take((size_t)p * P.ldp);
  P.oGinv = take((size_t)std::max(p, NB) * std::max<int64_t>(P.ldp, NB));
  P.oH = take((size_t)p * P.ldp);
  P.oLam = take((size_t)p);
  P.oVy = take((size_t)p * P.ldp);
  P.oZr = take((size_t)P.D * P.ldk);
  P.oE = take((size_t)P.D * P.ldk);
  P.pws_bytes = std::max(potrf_inv_workspace_bytes<T>(P.dmax, P.m), potrf_inv_workspace_bytes<T>(p, 1));
  P.oPws = o; o += al256(P.pws_bytes);
  P.split_bytes = 8 * (size_t)P.D * p * sizeof(T);
  P.oSplit = o; o += al256(P.split_bytes);
  P.oSmall = o; o += 4096;
  P.total = o + 256;
  size_t r = sizeof(double) * kFitHeaderDoubles;
  P.r_mean = r; r += al256(sizeof(double) * P.D);
  P.r_val = r; r += al256(sizeof(T) * k);
  for (int v = 0; v < P.m; ++v) { P.r_w[v] = r; r += al256(sizeof(T) * (size_t)L.dims[v] * k); }
  P.r_total = r;
  return P;
}

template <typename T>
__global__ void copy_vals_kernel(const T* __restrict__ src, T* __restrict__ dst, int k) {
  const int j = blockIdx.x * blockDim.x + threadIdx.x;
  if (j < k) dst[j] = src[j];
}

}  // namespace

// 0 for every shape mcca_fit refuses (as rcca_fit_workspace_bytes)
template <typename T>
size_t mcca_fit_workspace_bytes(const ColumnLayout& L, int k, int p) {
  if (!(L.n_views >= 2 && k >= 1 && p >= k && p <= L.D && syevj_small_supported<T>(p))) return 0;
  return make_mcca_plan<T>(L, k, p).total;
}

template <typename T>
void mcca_fit_result_layout(const ColumnLayout& L, int k, int p, int64_t* offsets) {
  MccaPlan P = make_mcca_plan<T>(L, k, p);
  offsets[0] = (int64_t)P.r_mean;
  offsets[1] = (int64_t)P.r_val;
  for (int v = 0; v < P.m; ++v) offsets[2 + v] = (int64_t)P.r_w[v];
  offsets[2 + P.m] = (int64_t)P.r_total;
}

template <typename T>
int mcca_fit(const ColumnLayout& L, const double* moments, const double* n_dev, double n_host, int center,
             const double* c, double eps_floor, int k, int p, int iters, void* result, size_t result_bytes, void* ws,
             size_t ws_bytes, cudaStream_t s) {
  const int m = L.n_views, D = L.D;
  CCAB_CHECK_ARG(m >= 2, "mcca_fit needs at least 2 views");
  CCAB_CHECK_ARG(k >= 1 && p >= k && p <= D, "mcca_fit: need 1 <= k <= p <= D, got k=%d p=%d", k, p);
  CCAB_CHECK_ARG(syevj_small_supported<T>(p), "mcca_fit: subspace width %d exceeds the single-CTA eigensolver", p);
  CCAB_CHECK_ARG(iters >= 1 && iters <= 60, "mcca_fit: bad iteration count %d", iters);
  double cmax = 0.0;
  for (int v = 0; v < m; ++v) cmax = std::max(cmax, c[v]);
  CCAB_CHECK_ARG(cmax <= 0.9, "mcca_fit: max c = %g > 0.9 (no a-priori shift); use the host-assembled route", cmax);
  MccaPlan P = make_mcca_plan<T>(L, k, p);
  CCAB_CHECK_ARG(ws_bytes >= P.total, "mcca_fit workspace too small: %zu < %zu", ws_bytes, P.total);
  CCAB_CHECK_ARG(result_bytes >= P.r_total, "mcca_fit result block too small: %zu < %zu", result_bytes, P.r_total);
  uint8_t* w = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(ws) + 255) & ~uintptr_t(255));
  uint8_t* res = static_cast<uint8_t*>(result);
  CCAB_CHECK_ARG((reinterpret_cast<uintptr_t>(res) & 255) == 0, "mcca_fit: result block must be 256-byte aligned");
  auto at = [&](size_t off) { return reinterpret_cast<T*>(w + off); };
  T *C = at(P.oC), *R = at(P.oR), *Linv = at(P.oLinv), *Tmp = at(P.oTmp), *K = at(P.oK), *Z = at(P.oZ), *Z2 = at(P.oZ2),
    *Y = at(P.oY), *H = at(P.oH), *lam = at(P.oLam), *Vy = at(P.oVy), *Zr = at(P.oZr), *E = at(P.oE);
  CholQrWs<T> cq;
  cq.G = at(P.oG);
  cq.Ginv = at(P.oGinv);
  cq.pws = w + P.oPws;
  cq.pws_bytes = P.pws_bytes;
  cq.ldg = P.ldp;
  cq.splitk_ws = w + P.oSplit;
  cq.splitk_ws_bytes = P.split_bytes;
  uint8_t* sm = w + P.oSmall;
  int* flags = reinterpret_cast<int*>(sm);
  int* infos = flags + 4;                                      // [m + iters + 4]
  const int n_infos = m + iters + 4;
  int* rr_info = infos + 100;
  unsigned* dmax = reinterpret_cast<unsigned*>(sm + 512);
  double* tol = reinterpret_cast<double*>(sm + 1024);          // [m]
  double* stats = tol + kMaxViews;                             // [2]
  double* resid_part = reinterpret_cast<double*>(sm + 1280);   // [kResidBlocks]
  unsigned* resid_cnt = reinterpret_cast<unsigned*>(sm + 1280 + 8 * kResidBlocks);
  CCAB_CUDA(cudaMemsetAsync(sm, 0, 2048, s));
  CCAB_CUDA(cudaMemsetAsync(K, 0, sizeof(T) * (size_t)D * P.ldC, s));
  double* hdr = reinterpret_cast<double*>(res);
  double* mean = reinterpret_cast<double*>(res + P.r_mean);
  T* vals = reinterpret_cast<T*>(res + P.r_val);

  // ---- covariance + ridge blocks (np.cov always centres: the caller passes center accordingly) ----
  {
    CovRidgeParams cp;
    memset(&cp, 0, sizeof(cp));
    cp.n_views = m; cp.D = D; cp.Dp = L.Dp;
    PivotTolParams q;
    memset(&q, 0, sizeof(q));
    q.n_views = m;
    for (int v = 0; v < m; ++v) {
      cp.dims[v] = L.dims[v]; cp.c[v] = c[v];
      cp.R[v] = R + (size_t)v * P.strideR; cp.ldr[v] = P.ldR;
      q.c[v] = c[v]; q.rank_tol[v] = L.dims[v] * eps_of<T>();
    }
    for (int v = 0; v <= m; ++v) { cp.coff[v] = L.coff[v]; cp.poff[v] = L.poff[v]; }
    q.floor = eps_floor;
    dim3 block(32, 8), grid((unsigned)ceil_div(D, 32), (unsigned)ceil_div(D, 8));
    cov_ridge_kernel<T><<<grid, block, 0, s>>>(cp, moments, n_dev, n_host, center, C, P.ldC, mean, dmax, flags);
    count_launches(1);
    pivot_tol_kernel<<<1, 32, 0, s>>>(q, dmax, tol);
    count_launches(1);
    CCAB_CUDA(cudaGetLastError());
  }
  int rc;
  if (P.equal) {
    rc = potrf_inv<T>(L.dims[0], m, R, P.ldR, P.strideR, Linv, P.ldR, P.strideR, 0.0, tol, infos, cq.pws, cq.pws_bytes, s);
    if (rc) return rc;
  } else {
    for (int v = 0; v < m; ++v) {
      rc = potrf_inv<T>(L.dims[v], 1, R + (size_t)v * P.strideR, P.ldR, 0, Linv + (size_t)v * P.strideR, P.ldR, 0, 0.0,
                        tol + v, infos + v, cq.pws, cq.pws_bytes, s);
      if (rc) return rc;
    }
  }
  // ---- K_ij = Linv_i C_ij Linv_j^T (and its mirror) ----
  for (int i = 0; i < m; ++i)
    for (int j = i + 1; j < m; ++j) {
      const int di = L.dims[i], dj = L.dims[j];
      GemmArgs<T> g;
      g.m = di; g.n = dj; g.k = di;
      g.A = Linv + (size_t)i * P.strideR; g.lda = P.ldR;
      g.B = C + (size_t)P.off[i] * P.ldC + P.off[j]; g.ldb = P.ldC; g.C = Tmp; g.ldc = P.ldR;
      rc = xgemm<T>(g, s);
      if (rc) return rc;
      GemmArgs<T> h;
      h.transb = 1; h.m = di; h.n = dj; h.k = dj;
      h.A = Tmp; h.lda = P.ldR; h.B = Linv + (size_t)j * P.strideR; h.ldb = P.ldR;
      h.C = K + (size_t)P.off[i] * P.ldC + P.off[j]; h.ldc = P.ldC;
      h.Ct = K + (size_t)P.off[j] * P.ldC + P.off[i]; h.ldct = P.ldC;
      rc = xgemm<T>(h, s);
      if (rc) return rc;
    }
  // ---- subspace iteration on K + shift I ----
  // K + I / (1 - max c) is positive semi-definite, so lambda_min(K) >= -1 / (1 - max c): half of that bound as the shift
  // keeps every wanted (positive) eigenvalue ahead of the negative end in magnitude and damps the unwanted middle of
  // the spectrum twice as fast as the full bound would
  const double shift = 0.5 / (1.0 - cmax);
  {
    const size_t total = (size_t)D * p;
    randn_kernel<T><<<(unsigned)std::min<size_t>((total + 255) / 256, 592), 256, 0, s>>>(Z2, P.ldp, D, p, 0x4321ull);
    count_launches(1);
    CCAB_CUDA(cudaGetLastError());
  }
  int slot = m;
  rc = cholqr<T>(Z2, P.ldp, Z, P.ldp, D, p, cq, infos + slot++, s);
  if (rc) return rc;
  for (int it = 0; it < iters; ++it) {
    CCAB_CUDA(cudaMemcpy2DAsync(Y, P.ldp * sizeof(T), Z, P.ldp * sizeof(T), (size_t)p * sizeof(T), (size_t)D,
                                cudaMemcpyDeviceToDevice, s));
    GemmArgs<T> a;   // Y = K Z + shift Z
    a.m = D; a.n = p; a.k = D; a.beta = (T)shift; a.A = K; a.lda = P.ldC; a.B = Z; a.ldb = P.ldp; a.C = Y; a.ldc = P.ldp;
    a.splitk_ws = cq.splitk_ws; a.splitk_ws_bytes = cq.splitk_ws_bytes;
    rc = xgemm<T>(a, s);
    if (rc) return rc;
    if (it % 2 == 0 && it != iters - 1) {   // orthonormalise every second product: cond grows by (|lam_1|+s)/(lam_p+s)
      std::swap(Y, Z);                      // per step, far inside what one CholQR pass absorbs
      continue;
    }
    rc = cholqr<T>(Y, P.ldp, Z, P.ldp, D, p, cq, infos + slot++, s);
    if (rc) return rc;
    if (it == iters - 1) {
      rc = cholqr<T>(Z, P.ldp, Z2, P.ldp, D, p, cq, infos + slot++, s);
      if (rc) return rc;
      std::swap(Z, Z2);
    }
  }
  // ---- Rayleigh-Ritz: H = Z^T K Z ----
  {
    GemmArgs<T> a;
    a.m = D; a.n = p; a.k = D; a.A = K; a.lda = P.ldC; a.B = Z; a.ldb = P.ldp; a.C = Y; a.ldc = P.ldp;   // Y = K Z
    a.splitk_ws = cq.splitk_ws; a.splitk_ws_bytes = cq.splitk_ws_bytes;
    rc = xgemm<T>(a, s);
    if (rc) return rc;
    GemmArgs<T> h;
    h.transa = 1; h.m = p; h.n = p; h.k = D; h.A = Z; h.lda = P.ldp; h.B = Y; h.ldb = P.ldp; h.C = H; h.ldc = P.ldp;
    h.splitk_ws = cq.splitk_ws; h.splitk_ws_bytes = cq.splitk_ws_bytes;
    rc = xgemm<T>(h, s);
    if (rc) return rc;
    rc = syevj_small<T>(p, 1, H, P.ldp, 0, lam, p, Vy, P.ldp, 0, rr_info, s);
    if (rc) return rc;
    GemmArgs<T> u;   // Ritz vectors Zr = Z Q_k
    u.transb = 1; u.m = D; u.n = k; u.k = p; u.A = Z; u.lda = P.ldp; u.B = Vy; u.ldb = P.ldp; u.C = Zr; u.ldc = P.ldk;
    rc = xgemm<T>(u, s);
    if (rc) return rc;
    GemmArgs<T> e;   // E = (K Z) Q_k
    e.transb = 1; e.m = D; e.n = k; e.k = p; e.A = Y; e.lda = P.ldp; e.B = Vy; e.ldb = P.ldp; e.C = E; e.ldc = P.ldk;
    rc = xgemm<T>(e, s);
    if (rc) return rc;
    residual_kernel<T><<<kResidBlocks, 256, 0, s>>>(E, P.ldk, Zr, P.ldk, D, k, lam, shift, 1, stats, resid_part, resid_cnt);
    copy_vals_kernel<T><<<(unsigned)ceil_div(k, 128), 128, 0, s>>>(lam, vals, k);
    count_launches(2);
    CCAB_CUDA(cudaGetLastError());
  }
  // ---- v_i = sqrt(m) Linv_i^T y_i ----
  for (int v = 0; v < m; ++v) {
    GemmArgs<T> a;
    a.transa = 1; a.m = L.dims[v]; a.n = k; a.k = L.dims[v]; a.alpha = (T)std::sqrt((double)m);
    a.A = Linv + (size_t)v * P.strideR; a.lda = P.ldR; a.B = Zr + (size_t)P.off[v] * P.ldk; a.ldb = P.ldk;
    a.C = reinterpret_cast<T*>(res + P.r_w[v]); a.ldc = k;
    rc = xgemm<T>(a, s);
    if (rc) return rc;
  }
  fit_status_kernel<<<1, 32, 0, s>>>(hdr, flags, infos, n_infos, rr_info, stats, n_dev, n_host, resid_tol_of<T>(), k,
                                    P.dmax);
  count_launches(1);
  CCAB_CUDA(cudaGetLastError());
  return 0;
}

template size_t mcca_fit_workspace_bytes<float>(const ColumnLayout&, int, int);
template size_t mcca_fit_workspace_bytes<double>(const ColumnLayout&, int, int);
template void mcca_fit_result_layout<float>(const ColumnLayout&, int, int, int64_t*);
template void mcca_fit_result_layout<double>(const ColumnLayout&, int, int, int64_t*);
template int mcca_fit<float>(const ColumnLayout&, const double*, const double*, double, int, const double*, double, int,
                             int, int, void*, size_t, void*, size_t, cudaStream_t);
template int mcca_fit<double>(const ColumnLayout&, const double*, const double*, double, int, const double*, double, int,
                              int, int, void*, size_t, void*, size_t, cudaStream_t);

// =============================================================================================================
// Deep-CCA objective (cca_zoo/deep/objectives.py:61-102) on the device, any widths, no host read-back.
//   forward : moments of [z1 z2] -> S_ii = C_ii + eps I, S_12 -> batched Cholesky + inverse ->
//             A_i = S_ii^-1 = Linv_i^T Linv_i, Q = A_1 S_12, Q2 = S_12 A_2, P = Q A_2 = S_11^-1 S_12 S_22^-1,
//             loss = -<P, S_12> (= -||S_11^-1/2 S_12 S_22^-1/2||_F^2: the reference's eigvalsh(T^T T).sum() is a trace),
//             G_11 = P Q^T = P S_21 S_11^-1, G_22 = Q2^T P = S_22^-1 S_21 P        (7 GEMMs, tcgen05 for float)
//   backward: dL/dz_1 = 2/(n-1) center(z_1 G_11 - z_2 P^T) go, dL/dz_2 = 2/(n-1) center(z_2 G_22 - z_1 P) go
//             (SURVEY.md §3.4; 4 tall GEMMs + 2 centring passes; `go` is the upstream gradient, read on the device)
//   flags[0..1] = Cholesky status of S_11 / S_22 with pivot^2 <= eps / 4 counted as failure (S_ii = C_ii + eps I has
//   lambda_min >= eps in exact arithmetic: a smaller pivot means rounding destroyed the ridge; the caller re-runs through
//   the eigen route, which clamps like the reference); checked lazily by the host.
// =============================================================================================================
namespace {

// loss[0] = -sum_ij P[i][j] * S12[i][j]: per-block partial sums (fixed assignment of elements to blocks), then one
// warp adds the partials in index order -- deterministic
template <typename T>
__global__ void loss_dot_partial_kernel(const T* __restrict__ P, int64_t ldp, const T* __restrict__ S, int64_t lds, int d1,
                                        int d2, double* __restrict__ partial) {
  __shared__ double red[32];
  double acc = 0.0;
  const int total = d1 * d2;
  for (int e = blockIdx.x * blockDim.x + threadIdx.x; e < total; e += gridDim.x * blockDim.x) {
    const int i = e / d2, j = e - i * d2;
    acc += (double)P[(size_t)i * ldp + j] * (double)S[(size_t)i * lds + j];
  }
  for (int o = 16; o > 0; o >>= 1) acc += __shfl_xor_sync(0xffffffffu, acc, o);
  if ((threadIdx.x & 31) == 0) red[threadIdx.x >> 5] = acc;
  __syncthreads();
  if (threadIdx.x == 0) {
    double t = 0.0;
    for (int w = 0; w < (int)(blockDim.x >> 5); ++w) t += red[w];
    partial[blockIdx.x] = t;
  }
}
template <typename T>
__global__ void loss_dot_final_kernel(const double* __restrict__ partial, int nparts, T* __restrict__ loss) {
  if (threadIdx.x == 0) {
    double t = 0.0;
    for (int i = 0; i < nparts; ++i) t += partial[i];
    loss[0] = (T)(-t);
  }
}

// column sums of A (m x n) over row slabs: part[slab][j] (fixed order inside a slab)
template <typename T>
__global__ void colsum_partial_kernel(int m, int n, const T* __restrict__ A, int64_t lda, int rows_per_slab,
                                      double* __restrict__ part) {
  __shared__ double sh[8][33];
  const int j = blockIdx.x * 32 + (threadIdx.x & 31);
  const int rg = threadIdx.x >> 5;   // 8 row groups
  const int r0 = blockIdx.y * rows_per_slab, r1 = min(m, r0 + rows_per_slab);
  double acc = 0.0;
  if (j < n)
    for (int i = r0 + rg; i < r1; i += 8) acc += (double)A[(size_t)i * lda + j];
  sh[rg][threadIdx.x & 31] = acc;
  __syncthreads();
  if (rg == 0 && j < n) {
    double t = 0.0;
    for (int k = 0; k < 8; ++k) t += sh[k][threadIdx.x & 31];
    part[(size_t)blockIdx.y * n + j] = t;
  }
}
// A[i][j] = (A[i][j] - mean_j) * scale[0], mean_j from the slab partials (added in slab order)
template <typename T>
__global__ void center_apply_kernel(int m, int n, T* __restrict__ A, int64_t lda, const double* __restrict__ part,
                                    int nslabs, const T* __restrict__ scale) {
  const int j = blockIdx.x * 32 + (threadIdx.x & 31);
  if (j >= n) return;
  double t = 0.0;
  for (int k = 0; k < nslabs; ++k) t += part[(size_t)k * n + j];
  const T mu = (T)(t / (double)m);
  const T sc = scale ? scale[0] : T(1);
  const int rows_per_block = (m + gridDim.y - 1) / gridDim.y;
  const int r0 = blockIdx.y * rows_per_block, r1 = min(m, r0 + rows_per_block);
  for (int i = r0 + (threadIdx.x >> 5); i < r1; i += blockDim.x >> 5) A[(size_t)i * lda + j] = (A[(size_t)i * lda + j] - mu) * sc;
}

// A[:, j] = (A[:, j] - mean_i A[i, j]) * scale[0]   (one block per 32 columns; fixed-order reduction)
template <typename T>
__global__ void center_scale_kernel(int m, int n, T* __restrict__ A, int64_t lda, const T* __restrict__ scale) {
  __shared__ double part[32][33];
  const int j = blockIdx.x * 32 + (threadIdx.x & 31);
  const int rg = threadIdx.x >> 5;
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
  const T sc = scale ? scale[0] : T(1);
  if (j < n)
    for (int i = rg; i < m; i += 32) A[(size_t)i * lda + j] = (A[(size_t)i * lda + j] - mu) * sc;
}

// Per-device scratch of the backward's centring (2 x 32 slabs x up to 4096 columns of partial sums, 2 MB), allocated
// once with the stream-ordered allocator: the backward entry point takes no workspace argument.
double* center_scratch(cudaStream_t) {
  static double* buf[64] = {};
  int dev = 0;
  if (cudaGetDevice(&dev) != cudaSuccess || dev < 0 || dev >= 64) return nullptr;
  if (!buf[dev]) {
    if (cudaMalloc(reinterpret_cast<void**>(&buf[dev]), sizeof(double) * 2 * 32 * 4096) != cudaSuccess) {
      set_error("could not allocate the 2 MB centring scratch");
      return nullptr;
    }
  }
  return buf[dev];
}

struct LossPlan {
  int d1, d2, D, Dp;
  int64_t ldC, ldR, strideR;
  bool batched;
  size_t oMom, oMomWs, oC, oR, oLinv, oA, oQ, oQ2, oPws, oSmall, oMean, total;
  size_t mom_ws_bytes, pws_bytes;
  size_t sG11, sP, sG22, s_total;   // element offsets inside `saved`
};

// from_moments: the stage after a given (all-reduced) moment buffer -- no moment sections, a double[D] for the means
template <typename T>
LossPlan make_loss_plan(const ColumnLayout& L, int64_t n, int precision, bool from_moments = false) {
  LossPlan P;
  P.d1 = L.dims[0]; P.d2 = L.dims[1]; P.D = L.D; P.Dp = L.Dp;
  P.ldC = r4(P.D);
  const int dm = std::max(P.d1, P.d2);
  P.ldR = r4(dm);
  P.strideR = (int64_t)dm * P.ldR;
  P.batched = P.d1 == P.d2;
  size_t o = 0;
  auto take = [&](size_t bytes) { size_t at = o; o += al256(bytes); return at; };
  if (from_moments) {
    P.oMom = P.oMomWs = 0;
    P.mom_ws_bytes = 0;
    P.oMean = take(sizeof(double) * (size_t)P.D);
  } else {
    P.oMom = take(sizeof(double) * ((size_t)P.Dp * P.Dp + P.Dp));
    P.mom_ws_bytes = std::max(moments_workspace_bytes(std::is_same<T, float>::value ? 0 : 1, precision, L, n),
                              moments_workspace_bytes(std::is_same<T, float>::value ? 0 : 1, 2, L, n)) + 512;
    P.oMomWs = take(P.mom_ws_bytes);
    P.oMean = 0;
  }
  P.oC = take(sizeof(T) * (size_t)P.D * P.ldC);
  P.oR = take(sizeof(T) * 2 * (size_t)P.strideR);
  P.oLinv = take(sizeof(T) * 2 * (size_t)P.strideR);
  P.oA = take(sizeof(T) * 2 * (size_t)P.strideR);
  P.oQ = take(sizeof(T) * (size_t)P.d1 * r4(P.d2));
  P.oQ2 = take(sizeof(T) * (size_t)P.d1 * r4(P.d2));
  P.pws_bytes = potrf_inv_workspace_bytes<T>(dm, 2);
  P.oPws = take(P.pws_bytes);
  P.oSmall = take(4096);
  P.total = o + 256;
  P.sG11 = 0;
  P.sP = (size_t)P.d1 * P.d1;
  P.sG22 = P.sP + (size_t)P.d1 * P.d2;
  P.s_total = P.sG22 + (size_t)P.d2 * P.d2;
  return P;
}

}  // namespace

template <typename T>
size_t ccaloss_workspace_bytes(const ColumnLayout& L, int64_t n, int precision) {
  return make_loss_plan<T>(L, n, precision).total;
}

namespace {

// saved[0 .. D) = (T) mean, saved[D] = (T) N: the global means and count behind G11 | P | G22 (wide global forward)
template <typename T>
__global__ void saved_tail_kernel(const double* __restrict__ mean, int D, const double* __restrict__ n_dev,
                                  T* __restrict__ tail) {
  for (int i = blockIdx.x * blockDim.x + threadIdx.x; i <= D; i += gridDim.x * blockDim.x)
    tail[i] = (T)(i < D ? mean[i] : n_dev[0]);
}

// Wide widths, everything after the moment pass: covariance + ridge blocks, batched Cholesky + inverse, 7 GEMMs, loss.
// n_dev == NULL: n_host rows (the fused local forward).  n_dev != NULL: an all-reduced buffer whose count is read on the
// device; the global means and N are appended to `saved` for ccaloss_backward_global.
template <typename T>
int loss_stage(const LossPlan& P, const ColumnLayout& L, uint8_t* w, const double* mom, const double* n_dev, double n_host,
               double eps, T* loss, T* saved, int* flags_out, cudaStream_t s) {
  const int d1 = P.d1, d2 = P.d2, D = P.D;
  T* C = reinterpret_cast<T*>(w + P.oC);
  T* R1 = reinterpret_cast<T*>(w + P.oR);
  T* R2 = R1 + P.strideR;
  T* Li1 = reinterpret_cast<T*>(w + P.oLinv);
  T* Li2 = Li1 + P.strideR;
  T* A1 = reinterpret_cast<T*>(w + P.oA);
  T* A2 = A1 + P.strideR;
  T* Q = reinterpret_cast<T*>(w + P.oQ);
  T* Q2 = reinterpret_cast<T*>(w + P.oQ2);
  const int64_t ldq = r4(d2);
  uint8_t* sm = w + P.oSmall;
  int* flags = reinterpret_cast<int*>(sm);
  unsigned* dmax = reinterpret_cast<unsigned*>(sm + 512);
  const int64_t ldr1 = P.batched ? P.ldR : r4(d1), ldr2 = P.batched ? P.ldR : r4(d2);
  T* G11 = saved + P.sG11;
  T* Pm = saved + P.sP;
  T* G22 = saved + P.sG22;

  double* mean = n_dev ? reinterpret_cast<double*>(w + P.oMean) : nullptr;
  int rc;
  CCAB_CUDA(cudaMemsetAsync(sm, 0, 1024, s));
  {
    CovRidgeParams cp;
    memset(&cp, 0, sizeof(cp));
    cp.n_views = 2; cp.D = D; cp.Dp = L.Dp;
    for (int v = 0; v < 2; ++v) { cp.dims[v] = L.dims[v]; cp.c[v] = 0.0; cp.ridge_add[v] = eps; }
    for (int v = 0; v <= 2; ++v) { cp.coff[v] = L.coff[v]; cp.poff[v] = L.poff[v]; }
    cp.R[0] = R1; cp.R[1] = R2; cp.ldr[0] = ldr1; cp.ldr[1] = ldr2;
    dim3 block(32, 8), grid((unsigned)ceil_div(D, 32), (unsigned)ceil_div(D, 8));
    cov_ridge_kernel<T><<<grid, block, 0, s>>>(cp, mom, n_dev, n_host, 1, C, P.ldC, mean, dmax, flags + 4);
    count_launches(1);
    CCAB_CUDA(cudaGetLastError());
  }
  const double piv_tol = 0.25 * eps;   // a pivot^2 below the ridge itself: S_ii lost its definiteness to rounding
  if (P.batched) {
    rc = potrf_inv<T>(d1, 2, R1, P.ldR, P.strideR, Li1, P.ldR, P.strideR, piv_tol, nullptr, flags, w + P.oPws, P.pws_bytes, s);
    if (rc) return rc;
  } else {
    rc = potrf_inv<T>(d1, 1, R1, ldr1, 0, Li1, ldr1, 0, piv_tol, nullptr, flags, w + P.oPws, P.pws_bytes, s);
    if (rc) return rc;
    rc = potrf_inv<T>(d2, 1, R2, ldr2, 0, Li2, ldr2, 0, piv_tol, nullptr, flags + 1, w + P.oPws, P.pws_bytes, s);
    if (rc) return rc;
  }
  // A_i = Linv_i^T Linv_i
  if (P.batched) {
    GemmArgs<T> g;
    g.transa = 1; g.m = d1; g.n = d1; g.k = d1;
    g.A = Li1; g.lda = P.ldR; g.strideA = P.strideR; g.B = Li1; g.ldb = P.ldR; g.strideB = P.strideR;
    g.C = A1; g.ldc = P.ldR; g.strideC = P.strideR; g.batch = 2;
    rc = xgemm<T>(g, s);
    if (rc) return rc;
  } else {
    for (int v = 0; v < 2; ++v) {
      GemmArgs<T> g;
      const int d = v ? d2 : d1;
      const int64_t ld = v ? ldr2 : ldr1;
      g.transa = 1; g.m = d; g.n = d; g.k = d;
      g.A = v ? Li2 : Li1; g.lda = ld; g.B = g.A; g.ldb = ld; g.C = v ? A2 : A1; g.ldc = ld;
      rc = xgemm<T>(g, s);
      if (rc) return rc;
    }
  }
  const T* S12 = C + d1;
  {
    GemmArgs<T> g;   // Q = A1 S12
    g.m = d1; g.n = d2; g.k = d1; g.A = A1; g.lda = ldr1; g.B = S12; g.ldb = P.ldC; g.C = Q; g.ldc = ldq;
    rc = xgemm<T>(g, s);
    if (rc) return rc;
    GemmArgs<T> h;   // Q2 = S12 A2
    h.m = d1; h.n = d2; h.k = d2; h.A = S12; h.lda = P.ldC; h.B = A2; h.ldb = ldr2; h.C = Q2; h.ldc = ldq;
    rc = xgemm<T>(h, s);
    if (rc) return rc;
    GemmArgs<T> p;   // P = Q A2
    p.m = d1; p.n = d2; p.k = d2; p.A = Q; p.lda = ldq; p.B = A2; p.ldb = ldr2; p.C = Pm; p.ldc = d2;
    rc = xgemm<T>(p, s);
    if (rc) return rc;
    GemmArgs<T> a;   // G11 = P Q^T
    a.transb = 1; a.m = d1; a.n = d1; a.k = d2; a.A = Pm; a.lda = d2; a.B = Q; a.ldb = ldq; a.C = G11; a.ldc = d1;
    rc = xgemm<T>(a, s);
    if (rc) return rc;
    GemmArgs<T> b;   // G22 = Q2^T P
    b.transa = 1; b.m = d2; b.n = d2; b.k = d1; b.A = Q2; b.lda = ldq; b.B = Pm; b.ldb = d2; b.C = G22; b.ldc = d2;
    rc = xgemm<T>(b, s);
    if (rc) return rc;
  }
  {
    double* partial = reinterpret_cast<double*>(sm + 2048);   // [64]
    loss_dot_partial_kernel<T><<<64, 256, 0, s>>>(Pm, d2, S12, P.ldC, d1, d2, partial);
    loss_dot_final_kernel<T><<<1, 32, 0, s>>>(partial, 64, loss);
    count_launches(2);
  }
  CCAB_CUDA(cudaGetLastError());
  if (n_dev) {
    saved_tail_kernel<T><<<1, 256, 0, s>>>(mean, D, n_dev, saved + P.s_total);
    count_launches(1);
    CCAB_CUDA(cudaGetLastError());
  }
  // flags_out[0..1] = Cholesky status, [2] = non-finite moments
  CCAB_CUDA(cudaMemcpyAsync(flags_out, flags, 2 * sizeof(int), cudaMemcpyDeviceToDevice, s));
  CCAB_CUDA(cudaMemcpyAsync(flags_out + 2, flags + 4, sizeof(int), cudaMemcpyDeviceToDevice, s));
  return 0;
}

}  // namespace

template <typename T>
int ccaloss_forward(const ColumnLayout& L, int precision, const void* z1, int64_t ld1, const void* z2, int64_t ld2,
                    int64_t n, double eps, T* loss, T* saved, int* flags_out, void* ws, size_t ws_bytes, cudaStream_t s) {
  CCAB_CHECK_ARG(L.n_views == 2 && n >= 2, "ccaloss_forward: two views and at least 2 samples");
  LossPlan P = make_loss_plan<T>(L, n, precision);
  CCAB_CHECK_ARG(ws_bytes >= P.total, "ccaloss workspace too small: %zu < %zu", ws_bytes, P.total);
  uint8_t* w = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(ws) + 255) & ~uintptr_t(255));
  const int d1 = P.d1, d2 = P.d2;
  double* mom = reinterpret_cast<double*>(w + P.oMom);

  // ---- moments of [z1 z2] ----
  const void* views[2] = {z1, z2};
  const int64_t lds[2] = {ld1, ld2};
  int rc;
  if (std::max(d1, d2) <= 64) {
    // narrow representations (config 3's k = 64): the moment pass (exact FMA, HBM / latency bound) and ONE single-CTA
    // launch for everything else
    rc = moments_simt<T>(L, views, lds, n, mom, w + P.oMomWs, P.mom_ws_bytes, s);
    if (rc) return rc;
    return ccaloss_small_forward<T>(mom, L.Dp, (double)n, d1, d2, eps, loss, saved, flags_out, s);
  }
  if (std::is_same<T, float>::value && precision != 2)
    rc = moments_tf32(L, views, lds, n, precision, mom, w + P.oMomWs, P.mom_ws_bytes, s);
  else
    rc = moments_simt<T>(L, views, lds, n, mom, w + P.oMomWs, P.mom_ws_bytes, s);
  if (rc) return rc;
  return loss_stage<T>(P, L, w, mom, nullptr, (double)n, eps, loss, saved, flags_out, s);
}

template <typename T>
size_t ccaloss_fwd_moments_workspace_bytes(const ColumnLayout& L) {
  return make_loss_plan<T>(L, 0, 2, true).total;
}

template <typename T>
int ccaloss_forward_moments(const ColumnLayout& L, const double* mom, const double* n_dev, double eps, T* loss,
                            T* saved, int* flags_out, void* ws, size_t ws_bytes, cudaStream_t s) {
  CCAB_CHECK_ARG(L.n_views == 2 && mom && n_dev, "ccaloss_forward_moments: two views, a moment buffer and n_dev");
  LossPlan P = make_loss_plan<T>(L, 0, 2, true);
  CCAB_CHECK_ARG(ws_bytes >= P.total, "ccaloss workspace too small: %zu < %zu", ws_bytes, P.total);
  uint8_t* w = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(ws) + 255) & ~uintptr_t(255));
  if (std::max(P.d1, P.d2) <= 64)
    return ccaloss_small_forward<T>(mom, L.Dp, 0.0, P.d1, P.d2, eps, loss, saved, flags_out, s, n_dev);
  return loss_stage<T>(P, L, w, mom, n_dev, 0.0, eps, loss, saved, flags_out, s);
}

template <typename T>
int ccaloss_backward(int d1, int d2, const T* z1, int64_t ld1, const T* z2, int64_t ld2, int64_t n, const T* saved,
                     const T* grad_out, T* g1, int64_t ldg1, T* g2, int64_t ldg2, cudaStream_t s) {
  CCAB_CHECK_ARG(n >= 2 && d1 >= 1 && d2 >= 1, "ccaloss_backward: bad shape");
  if (std::max(d1, d2) <= 64)
    return ccaloss_small_backward<T>(d1, d2, z1, ld1, z2, ld2, n, saved, grad_out, g1, ldg1, g2, ldg2, s);
  const T* G11 = saved;
  const T* Pm = saved + (size_t)d1 * d1;
  const T* G22 = Pm + (size_t)d1 * d2;
  const T a = (T)(2.0 / (double)(n - 1));
  GemmArgs<T> g;
  g.m = (int)n; g.n = d1; g.k = d1; g.alpha = a; g.A = z1; g.lda = ld1; g.B = G11; g.ldb = d1; g.C = g1; g.ldc = ldg1;
  int rc = xgemm<T>(g, s);
  if (rc) return rc;
  GemmArgs<T> h;   // g1 -= a z2 P^T
  h.transb = 1; h.m = (int)n; h.n = d1; h.k = d2; h.alpha = -a; h.beta = T(1);
  h.A = z2; h.lda = ld2; h.B = Pm; h.ldb = d2; h.C = g1; h.ldc = ldg1;
  rc = xgemm<T>(h, s);
  if (rc) return rc;
  GemmArgs<T> u;
  u.m = (int)n; u.n = d2; u.k = d2; u.alpha = a; u.A = z2; u.lda = ld2; u.B = G22; u.ldb = d2; u.C = g2; u.ldc = ldg2;
  rc = xgemm<T>(u, s);
  if (rc) return rc;
  GemmArgs<T> v;   // g2 -= a z1 P
  v.m = (int)n; v.n = d2; v.k = d1; v.alpha = -a; v.beta = T(1);
  v.A = z1; v.lda = ld1; v.B = Pm; v.ldb = d2; v.C = g2; v.ldc = ldg2;
  rc = xgemm<T>(v, s);
  if (rc) return rc;
  // centring: slab partial sums, then subtract and scale (the scratch lives behind the gradients' own columns: none is
  // available here, so the caller-provided `part` buffer is carved from g-independent static device scratch)
  {
    const int nslabs = (int)std::min<int64_t>(32, ceil_div(n, 128));
    const int rows_per_slab = (int)ceil_div(n, nslabs);
    double* part = std::max(d1, d2) <= 4096 ? center_scratch(s) : nullptr;
    if (!part) {   // wider than the scratch (or no scratch): the single-pass kernel
      center_scale_kernel<T><<<(unsigned)ceil_div(d1, 32), 1024, 0, s>>>((int)n, d1, g1, ldg1, grad_out);
      center_scale_kernel<T><<<(unsigned)ceil_div(d2, 32), 1024, 0, s>>>((int)n, d2, g2, ldg2, grad_out);
      count_launches(2);
      CCAB_CUDA(cudaGetLastError());
      return 0;
    }
    for (int v = 0; v < 2; ++v) {
      T* g = v ? g2 : g1;
      const int d = v ? d2 : d1;
      const int64_t ldg = v ? ldg2 : ldg1;
      double* pv = part + (size_t)v * 32 * 4096;
      colsum_partial_kernel<T><<<dim3((unsigned)ceil_div(d, 32), (unsigned)nslabs), 256, 0, s>>>((int)n, d, g, ldg,
                                                                                                 rows_per_slab, pv);
      center_apply_kernel<T><<<dim3((unsigned)ceil_div(d, 32), 32), 256, 0, s>>>((int)n, d, g, ldg, pv, nslabs, grad_out);
    }
    count_launches(4);
  }
  CCAB_CUDA(cudaGetLastError());
  return 0;
}

namespace {

// Epilogue of the global backward, for g_v = z_v G_vv - z_w P^(T) over this shard's rows (blockIdx.z = v): subtract the
// column means of the whole batch's products, r_1 = mu_1^T G11 - mu_2^T P^T, r_2 = mu_2^T G22 - mu_1^T P (a small product
// of the saved global means), and scale by 2/(N-1) grad_out with N saved behind the means.  Each block recomputes r for
// its 32 columns (8 row groups over the contraction, added in group order: every block gets the same bits), then
// rewrites its slab of rows.
template <typename T>
__global__ void __launch_bounds__(256) ccaloss_global_center_kernel(int64_t m, int d1, int d2, T* __restrict__ g1,
                                                                    int64_t ldg1, T* __restrict__ g2, int64_t ldg2,
                                                                    const T* __restrict__ saved,
                                                                    const T* __restrict__ grad_out, int rows_per_block) {
  __shared__ double part[8][33];
  const int v = blockIdx.z;
  const int d = v ? d2 : d1, dw = v ? d1 : d2;
  const int lane = threadIdx.x & 31, rg = threadIdx.x >> 5;
  const int j = blockIdx.x * 32 + lane;
  if (blockIdx.x * 32 >= d) return;                  // uniform over the block
  const T* G11 = saved;
  const T* Pm = G11 + (size_t)d1 * d1;
  const T* G22 = Pm + (size_t)d1 * d2;
  const T* mu = G22 + (size_t)d2 * d2;               // mu_1 | mu_2 | N
  const T* Gv = v ? G22 : G11;
  const T* mv = v ? mu + d1 : mu;
  const T* mw = v ? mu : mu + d1;
  double acc = 0.0;
  if (j < d) {
    for (int k = rg; k < d; k += 8) acc += (double)mv[k] * (double)Gv[(size_t)k * d + j];
    // v = 0: (mu_2^T P^T)_j = sum_k mu_2[k] P[j][k];  v = 1: (mu_1^T P)_j = sum_k mu_1[k] P[k][j]
    for (int k = rg; k < dw; k += 8)
      acc -= (double)mw[k] * (double)(v ? Pm[(size_t)k * d2 + j] : Pm[(size_t)j * d2 + k]);
  }
  part[rg][lane] = acc;
  __syncthreads();
  if (rg == 0) {
    double t = 0.0;
    for (int k = 0; k < 8; ++k) t += part[k][lane];
    part[0][lane] = t;
  }
  __syncthreads();
  if (j >= d) return;
  const T r = (T)part[0][lane];
  const T sc = (T)(2.0 / ((double)mu[d1 + d2] - 1.0)) * (grad_out ? grad_out[0] : T(1));
  T* g = v ? g2 : g1;
  const int64_t ldg = v ? ldg2 : ldg1;
  const int64_t r0 = (int64_t)blockIdx.y * rows_per_block, r1 = min(m, r0 + (int64_t)rows_per_block);
  for (int64_t i = r0 + rg; i < r1; i += 8) g[i * ldg + j] = (g[i * ldg + j] - r) * sc;
}

}  // namespace

template <typename T>
int ccaloss_backward_global(int d1, int d2, const T* z1, int64_t ld1, const T* z2, int64_t ld2, int64_t n,
                            const T* saved, const T* grad_out, T* g1, int64_t ldg1, T* g2, int64_t ldg2,
                            cudaStream_t s) {
  CCAB_CHECK_ARG(n >= 0 && d1 >= 1 && d2 >= 1, "ccaloss_backward_global: bad shape");
  if (n == 0) return 0;                              // a rank without rows: nothing to write
  if (std::max(d1, d2) <= 64)
    return ccaloss_small_backward<T>(d1, d2, z1, ld1, z2, ld2, n, saved, grad_out, g1, ldg1, g2, ldg2, s, true);
  const T* G11 = saved;
  const T* Pm = saved + (size_t)d1 * d1;
  const T* G22 = Pm + (size_t)d1 * d2;
  GemmArgs<T> g;   // g1 = z1 G11
  g.m = (int)n; g.n = d1; g.k = d1; g.A = z1; g.lda = ld1; g.B = G11; g.ldb = d1; g.C = g1; g.ldc = ldg1;
  int rc = xgemm<T>(g, s);
  if (rc) return rc;
  GemmArgs<T> h;   // g1 -= z2 P^T
  h.transb = 1; h.m = (int)n; h.n = d1; h.k = d2; h.alpha = T(-1); h.beta = T(1);
  h.A = z2; h.lda = ld2; h.B = Pm; h.ldb = d2; h.C = g1; h.ldc = ldg1;
  rc = xgemm<T>(h, s);
  if (rc) return rc;
  GemmArgs<T> u;   // g2 = z2 G22
  u.m = (int)n; u.n = d2; u.k = d2; u.A = z2; u.lda = ld2; u.B = G22; u.ldb = d2; u.C = g2; u.ldc = ldg2;
  rc = xgemm<T>(u, s);
  if (rc) return rc;
  GemmArgs<T> v;   // g2 -= z1 P
  v.m = (int)n; v.n = d2; v.k = d1; v.alpha = T(-1); v.beta = T(1);
  v.A = z1; v.lda = ld1; v.B = Pm; v.ldb = d2; v.C = g2; v.ldc = ldg2;
  rc = xgemm<T>(v, s);
  if (rc) return rc;
  const int row_blocks = (int)std::min<int64_t>(64, ceil_div(n, 64));
  const int rows_per_block = (int)ceil_div(n, row_blocks);
  dim3 grid((unsigned)ceil_div(std::max(d1, d2), 32), (unsigned)row_blocks, 2);
  ccaloss_global_center_kernel<T><<<grid, 256, 0, s>>>(n, d1, d2, g1, ldg1, g2, ldg2, saved, grad_out, rows_per_block);
  count_launches(1);
  CCAB_CUDA(cudaGetLastError());
  return 0;
}

template size_t ccaloss_fwd_moments_workspace_bytes<float>(const ColumnLayout&);
template size_t ccaloss_fwd_moments_workspace_bytes<double>(const ColumnLayout&);
template int ccaloss_forward_moments<float>(const ColumnLayout&, const double*, const double*, double, float*, float*,
                                            int*, void*, size_t, cudaStream_t);
template int ccaloss_forward_moments<double>(const ColumnLayout&, const double*, const double*, double, double*,
                                             double*, int*, void*, size_t, cudaStream_t);
template int ccaloss_backward_global<float>(int, int, const float*, int64_t, const float*, int64_t, int64_t,
                                            const float*, const float*, float*, int64_t, float*, int64_t, cudaStream_t);
template int ccaloss_backward_global<double>(int, int, const double*, int64_t, const double*, int64_t, int64_t,
                                             const double*, const double*, double*, int64_t, double*, int64_t,
                                             cudaStream_t);
template size_t ccaloss_workspace_bytes<float>(const ColumnLayout&, int64_t, int);
template size_t ccaloss_workspace_bytes<double>(const ColumnLayout&, int64_t, int);
template int ccaloss_forward<float>(const ColumnLayout&, int, const void*, int64_t, const void*, int64_t, int64_t, double,
                                    float*, float*, int*, void*, size_t, cudaStream_t);
template int ccaloss_forward<double>(const ColumnLayout&, int, const void*, int64_t, const void*, int64_t, int64_t, double,
                                     double*, double*, int*, void*, size_t, cudaStream_t);
template int ccaloss_backward<float>(int, int, const float*, int64_t, const float*, int64_t, int64_t, const float*,
                                     const float*, float*, int64_t, float*, int64_t, cudaStream_t);
template int ccaloss_backward<double>(int, int, const double*, int64_t, const double*, int64_t, int64_t, const double*,
                                      const double*, double*, int64_t, double*, int64_t, cudaStream_t);

template size_t rcca_fit_workspace_bytes<float>(int, int, int, int);
template size_t rcca_fit_workspace_bytes<double>(int, int, int, int);
template void rcca_fit_result_layout<float>(int, int, int, int, int64_t*);
template void rcca_fit_result_layout<double>(int, int, int, int, int64_t*);
template int rcca_fit<float>(const ColumnLayout&, const double*, const double*, double, int, const double*, int, int, int,
                             void*, size_t, void*, size_t, cudaStream_t);
template int rcca_fit<double>(const ColumnLayout&, const double*, const double*, double, int, const double*, int, int,
                              int, void*, size_t, void*, size_t, cudaStream_t);

}  // namespace ccab
