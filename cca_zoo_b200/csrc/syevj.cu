// K3/K4: symmetric eigensolver and SVD by one-sided block Jacobi (Hestenes), batched.
//
// The working matrix G (m x n, column-major: each column contiguous) starts as A (symmetric mode) or
// as the matrix to factor (SVD mode), multiplied by the power of two that brings max |G| into [0.5, 1) (exact; the
// values are scaled back at the end); V (n x n) starts as I.  Columns are grouped in blocks of
// kB = 16.  One round of the round-robin tournament handles nb/2 disjoint block pairs; for a pair
// the 32-column panel P = [G_p G_q] gets
//     (a) its Gram matrix  W = P^T P                      (jacobi_gram_kernel, row-split partials)
//     (b) the small symmetric eigenproblem W = Q L Q^T    (jacobi_solve_kernel: parallel two-sided
//         Jacobi in shared memory, 256 pair-blocks per step, ping-pong buffers, one barrier/step)
//     (c) the update  [G;V]_panel <- [G;V]_panel Q        (jacobi_apply_kernel)
// nb-1 rounds make a sweep; sweeps repeat until the largest normalised off-diagonal Gram entry seen
// in a sweep drops below tol.  At convergence G = A V has orthogonal columns:
//     symmetric mode : lambda_j = v_j . g_j  (Rayleigh quotient, sign included)
//     SVD mode       : sigma_j = |g_j|, u_j = g_j / sigma_j.
// Results are sorted descending and written as ROWS (row j = j-th vector).
//
// Replaces the LAPACK calls behind np.linalg.svd / scipy.linalg.eigh / np.linalg.eigvalsh /
// torch.linalg.eigh at cca_zoo/_utils/_linalg.py:28,67-71, cca_zoo/linear/_rcca.py:97,
// cca_zoo/linear/_mcca.py:117,170, cca_zoo/linear/_gcca.py:102, cca_zoo/deep/objectives.py:19.
#include "syevj.cuh"

#include <cooperative_groups.h>

#include <algorithm>
#include <cmath>
#include <cstring>
#include <cstdlib>
#include <type_traits>

namespace ccab {

constexpr int kB = 16;        // column block width
constexpr int kS = 2 * kB;    // panel width
constexpr int kSP = kS + 1;   // padded smem stride

template <typename T>
__device__ __forceinline__ T neg_inf();
template <>
__device__ __forceinline__ float neg_inf<float>() { return __int_as_float(0xff800000); }
template <>
__device__ __forceinline__ double neg_inf<double>() { return __longlong_as_double(0xfff0000000000000ULL); }

template <typename T>
struct Eps;
template <>
struct Eps<float> { static constexpr float v = 5.9604645e-8f; };
template <>
struct Eps<double> { static constexpr double v = 1.1102230246251565e-16; };

// round-robin tournament on `np` players (np even): pair i of round r
__host__ __device__ __forceinline__ void rr_pair(int np, int r, int i, int& p, int& q) {
  const int m1 = np - 1;
  int a, b;
  if (i == 0) {
    a = m1;
    b = r % m1;
  } else {
    a = (r + i) % m1;
    b = (r - i + m1) % m1;
  }
  p = a < b ? a : b;
  q = a < b ? b : a;
}

// Rotation (c, s) that annihilates a_pq of [[app, apq], [apq, aqq]]:  t = h / (d + sgn(d) sqrt(d^2 + h^2))
// with d = aqq - app, h = 2 apq; c = 1/sqrt(1 + t^2), s = t c.  Fast reciprocal / rsqrt are enough: the
// accumulated Q is re-orthonormalised before it is applied (reorthonormalise below).
__device__ __forceinline__ void jacobi_cs(float app, float aqq, float apq, float& c, float& s, bool& rotated) {
  const float e = Eps<float>::v;
  if (apq * apq <= e * e * fabsf(app * aqq) || apq == 0.f) {
    c = 1.f;
    s = 0.f;
    return;
  }
  const float d = aqq - app, h = 2.f * apq;
  const float r = sqrtf(fmaf(d, d, h * h));
  const float t = __fdividef(h, d + copysignf(r, d));
  c = rsqrtf(fmaf(t, t, 1.f));
  s = t * c;
  rotated = true;
}
__device__ __forceinline__ void jacobi_cs(double app, double aqq, double apq, double& c, double& s, bool& rotated) {
  const double e = Eps<double>::v;
  if (apq * apq <= e * e * fabs(app * aqq) || apq == 0.0) {
    c = 1.0;
    s = 0.0;
    return;
  }
  const double d = aqq - app, h = 2.0 * apq;
  const double r = sqrt(fma(d, d, h * h));
  const double t = h / (d + copysign(r, d));
  c = rsqrt(fma(t, t, 1.0));
  s = t * c;
  rotated = true;
}

// One sweep of parallel cyclic two-sided Jacobi on a 32 x 32 symmetric matrix in shared memory, 256 threads.
// Thread (i, j) owns the 2x2 block of rotation pairs (i, j) in each of the 31 tournament steps; lanes
// 0..15 of every warp each compute the rotation of pair `lane` once and the warp shares them by shuffle.
// Wa/Wb: ping-pong copies (stride 33), Q: accumulated rotations (stride 33, starts as I), pairs: the
// (S-1) x 16 tournament table.  Returns the buffer holding the rotated matrix.
template <typename T, int S>
__device__ T* small_syevj(T* Wa, T* Wb, T* Q, const uchar2* pairs) {
  static_assert(S == 32, "the thread mapping below is written for 32 x 32 panels and 256 threads");
  constexpr int H = S / 2;
  constexpr int SP = S + 1;
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  const int j = lane & 15;
  const int i = 2 * warp + (lane >> 4);
  T* cur = Wa;
  T* nxt = Wb;
  for (int step = 0; step < S - 1; ++step) {
    const uchar2 pq = pairs[step * H + j];
    const int pj = pq.x, qj = pq.y;
    T cj, sj;
    bool rj = false;
    jacobi_cs(cur[pj * SP + pj], cur[qj * SP + qj], cur[pj * SP + qj], cj, sj, rj);
    const T ci = __shfl_sync(0xffffffffu, cj, i);
    const T si = __shfl_sync(0xffffffffu, sj, i);
    const int pi = __shfl_sync(0xffffffffu, pj, i);
    const int qi = __shfl_sync(0xffffffffu, qj, i);
    const bool ri = __shfl_sync(0xffffffffu, (int)rj, i) != 0;
    const T x00 = cur[pi * SP + pj], x01 = cur[pi * SP + qj];
    const T x10 = cur[qi * SP + pj], x11 = cur[qi * SP + qj];
    const T y00 = cj * x00 - sj * x01, y01 = sj * x00 + cj * x01;
    const T y10 = cj * x10 - sj * x11, y11 = sj * x10 + cj * x11;
    T z00 = ci * y00 - si * y10, z10 = si * y00 + ci * y10;
    T z01 = ci * y01 - si * y11, z11 = si * y01 + ci * y11;
    if (i == j && ri) { z01 = T(0); z10 = T(0); }
    nxt[pi * SP + pj] = z00;
    nxt[pi * SP + qj] = z01;
    nxt[qi * SP + pj] = z10;
    nxt[qi * SP + qj] = z11;
    if (ri) {  // Q <- Q J_i for rows j and j+H (each (row, pair) owned by exactly one thread)
#pragma unroll
      for (int hh = 0; hh < 2; ++hh) {
        const int r = j + hh * H;
        const T a = Q[r * SP + pi], b = Q[r * SP + qi];
        Q[r * SP + pi] = ci * a - si * b;
        Q[r * SP + qi] = si * a + ci * b;
      }
    }
    __syncthreads();
    T* tmp = cur; cur = nxt; nxt = tmp;
  }
  return cur;
}

// tournament table in shared memory: pairs[step * 16 + i] = (p, q), p < q
template <int S>
__device__ void fill_pair_table(uchar2* pairs) {
  for (int e = threadIdx.x; e < (S - 1) * (S / 2); e += blockDim.x) {
    int p, q;
    rr_pair(S, e / (S / 2), e % (S / 2), p, q);
    pairs[e] = make_uchar2((unsigned char)p, (unsigned char)q);
  }
}

// ---------------------------------------------------------------------------------------------
// (a) partial Gram of a panel over a row range
// ---------------------------------------------------------------------------------------------
template <typename T>
struct JacobiCtx {
  T* G;          // [batch][n_pad cols][ldg]      column-major
  T* V;          // [batch][n_pad cols][n_pad]    column-major
  T* Wpart;      // [batch][npairs][R][kS*kS]
  T* Qm;         // [batch][npairs][kS*kS]        row-major Q
  int* skip;     // [batch][npairs]
  unsigned* stat;  // [batch] max off-diagonal ratio of the sweep (float bits)
  float* null2;    // [batch] squared column norm below which a column is numerical noise: (n eps)^2 ||G||_F^2
  int* expo;       // [batch] G was multiplied by 2^-expo before the sweeps (max |G| in [0.5, 1))
  int m, n_pad, nb, npairs, R;
  int64_t ldg;
  int rows_per_part;
};

template <typename T>
__global__ void __launch_bounds__(256) jacobi_gram_kernel(const JacobiCtx<T> c, int round) {
  constexpr int KR = 64;
  __shared__ T Ps[KR][kSP];
  const int pair = blockIdx.x, part = blockIdx.y, b = blockIdx.z;
  int p, q;
  rr_pair(c.nb, round, pair, p, q);
  const T* G = c.G + (size_t)b * c.n_pad * c.ldg;
  const int r0 = part * c.rows_per_part;
  const int r1 = min(r0 + c.rows_per_part, c.m);
  const int tx = threadIdx.x & 15, ty = threadIdx.x >> 4;
  T acc00 = 0, acc01 = 0, acc10 = 0, acc11 = 0;
  const int lr = threadIdx.x & 63, lc0 = threadIdx.x >> 6;
  for (int r = r0; r < r1; r += KR) {
#pragma unroll
    for (int i = 0; i < kS / 4; ++i) {
      const int col = lc0 + 4 * i;
      const int gcol = (col < kB ? p * kB + col : q * kB + col - kB);
      const int row = r + lr;
      Ps[lr][col] = row < r1 ? G[(size_t)gcol * c.ldg + row] : T(0);
    }
    __syncthreads();
#pragma unroll 8
    for (int k = 0; k < KR; ++k) {
      const T a0 = Ps[k][2 * ty], a1 = Ps[k][2 * ty + 1];
      const T b0 = Ps[k][2 * tx], b1 = Ps[k][2 * tx + 1];
      acc00 = fma(a0, b0, acc00);
      acc01 = fma(a0, b1, acc01);
      acc10 = fma(a1, b0, acc10);
      acc11 = fma(a1, b1, acc11);
    }
    __syncthreads();
  }
  T* W = c.Wpart + (((size_t)b * c.npairs + pair) * c.R + part) * (kS * kS);
  W[(2 * ty) * kS + 2 * tx] = acc00;
  W[(2 * ty) * kS + 2 * tx + 1] = acc01;
  W[(2 * ty + 1) * kS + 2 * tx] = acc10;
  W[(2 * ty + 1) * kS + 2 * tx + 1] = acc11;
}

// ---------------------------------------------------------------------------------------------
// (b) small eigenproblem of the panel Gram matrix -> Q (columns sorted by descending eigenvalue)
// ---------------------------------------------------------------------------------------------
// One Newton-Schulz step Q <- Q + Q (I - Q^T Q) / 2: the product of hundreds of rotations drifts from
// orthogonality by O(#rotations * eps) (tiny rotations round c to 1 and inflate norms systematically);
// this pulls Q back to eps-level so that V and G = A V stay consistent over thousands of panel updates.
// E: scratch S x S (stride SP).  All threads of the block call this.
template <typename T, int S>
__device__ void reorthonormalise(T* Q, T* E, T* Qn) {
  constexpr int SP = S + 1;
  for (int e = threadIdx.x; e < S * S; e += blockDim.x) {
    const int i = e / S, j = e % S;
    T acc = (i == j) ? T(1) : T(0);
#pragma unroll 8
    for (int k = 0; k < S; ++k) acc = fma(-Q[k * SP + i], Q[k * SP + j], acc);
    E[i * SP + j] = acc;
  }
  __syncthreads();
  for (int e = threadIdx.x; e < S * S; e += blockDim.x) {
    const int i = e / S, j = e % S;
    T acc = T(0);
#pragma unroll 8
    for (int k = 0; k < S; ++k) acc = fma(Q[i * SP + k], E[k * SP + j], acc);
    Qn[i * SP + j] = Q[i * SP + j] + T(0.5) * acc;
  }
  __syncthreads();
}

template <typename T>
__global__ void __launch_bounds__(256) jacobi_solve_kernel(const JacobiCtx<T> c, T tol) {
  __shared__ T Wa[kS * kSP];
  __shared__ T Wb[kS * kSP];
  __shared__ T Q[kS * kSP];
  __shared__ int rank_of[kS];
  __shared__ float ratio_s;
  __shared__ uchar2 pairs[(kS - 1) * (kS / 2)];
  fill_pair_table<kS>(pairs);
  const int pair = blockIdx.x, b = blockIdx.y;
  const T* Wp = c.Wpart + ((size_t)b * c.npairs + pair) * c.R * (kS * kS);
  if (threadIdx.x == 0) ratio_s = 0.f;
  for (int e = threadIdx.x; e < kS * kS; e += blockDim.x) {
    T acc = 0;
    for (int r = 0; r < c.R; ++r) acc += Wp[(size_t)r * kS * kS + e];  // fixed order: deterministic
    const int i = e / kS, j = e % kS;
    Wa[i * kSP + j] = acc;
    Q[i * kSP + j] = (i == j) ? T(1) : T(0);
  }
  __syncthreads();
  // convergence statistic: max_{i<j} |w_ij| / sqrt(w_ii w_jj)
  const float null2_b = c.null2[b];
  float myr = 0.f;
  for (int e = threadIdx.x; e < kS * kS; e += blockDim.x) {
    const int i = e / kS, j = e % kS;
    if (i < j) {
      // columns at the rounding-noise level of the matrix (rank-deficient input) have no direction: the cosine
      // between them and anything else is noise and must not keep the iteration "unconverged" forever
      const T wi = Wa[i * kSP + i], wj = Wa[j * kSP + j];
      const T d = wi * wj;
      const T w = fabs(Wa[i * kSP + j]);
      if (d > T(0) && w > T(0) && (float)wi > null2_b && (float)wj > null2_b) myr = fmaxf(myr, (float)(w / sqrt(d)));
    }
  }
  for (int o = 16; o > 0; o >>= 1) myr = fmaxf(myr, __shfl_xor_sync(0xffffffffu, myr, o));
  if ((threadIdx.x & 31) == 0 && myr > 0.f) atomicMax(reinterpret_cast<int*>(&ratio_s), __float_as_int(myr));
  __syncthreads();
  const float ratio = ratio_s;
  if (threadIdx.x == 0) {
    atomicMax(c.stat + b, __float_as_uint(ratio));
    c.skip[(size_t)b * c.npairs + pair] = (ratio <= (float)tol) ? 1 : 0;
  }
  if (ratio <= (float)tol) return;  // panel already orthogonal: Q = I, apply kernel skips it

  T* fin = small_syevj<T, kS>(Wa, Wb, Q, pairs);
  __syncthreads();
  if (threadIdx.x < kS) {
    const int i = threadIdx.x;
    const T li = fin[i * kSP + i];
    int rk = 0;
    for (int j = 0; j < kS; ++j) {
      const T lj = fin[j * kSP + j];
      rk += (lj > li || (lj == li && j < i)) ? 1 : 0;
    }
    rank_of[i] = rk;
  }
  __syncthreads();
  T* other = (fin == Wa) ? Wb : Wa;   // free ping-pong buffer: scratch for I - Q^T Q
  T* Qn = fin;                         // the diagonalised matrix is no longer needed after ranking
  reorthonormalise<T, kS>(Q, other, Qn);
  T* Qo = c.Qm + ((size_t)b * c.npairs + pair) * (kS * kS);
  for (int e = threadIdx.x; e < kS * kS; e += blockDim.x) {
    const int r = e / kS, i = e % kS;
    Qo[r * kS + rank_of[i]] = Qn[r * kSP + i];
  }
}

// ---------------------------------------------------------------------------------------------
// (c) panel update: rows of [G;V] times Q
// ---------------------------------------------------------------------------------------------
template <typename T>
__global__ void __launch_bounds__(128) jacobi_apply_kernel(const JacobiCtx<T> c, int round) {
  __shared__ T Qs[kS * kS];
  const int pair = blockIdx.x, b = blockIdx.z;
  if (c.skip[(size_t)b * c.npairs + pair]) return;
  int p, q;
  rr_pair(c.nb, round, pair, p, q);
  const T* Qg = c.Qm + ((size_t)b * c.npairs + pair) * (kS * kS);
  for (int e = threadIdx.x; e < kS * kS; e += blockDim.x) Qs[e] = Qg[e];
  __syncthreads();
  // row chunks: first ceil(m/128) chunks cover G, the rest cover V
  const int gchunks = (c.m + 127) / 128;
  int chunk = blockIdx.y;
  T* base;
  int64_t ld;
  int rows;
  if (chunk < gchunks) {
    base = c.G + (size_t)b * c.n_pad * c.ldg;
    ld = c.ldg;
    rows = c.m;
  } else {
    chunk -= gchunks;
    base = c.V + (size_t)b * c.n_pad * c.n_pad;
    ld = c.n_pad;
    rows = c.n_pad;
  }
  const int row = chunk * 128 + threadIdx.x;
  if (row >= rows) return;
  T x[kS], y[kS];
#pragma unroll
  for (int k = 0; k < kS; ++k) {
    const int gcol = (k < kB ? p * kB + k : q * kB + k - kB);
    x[k] = base[(size_t)gcol * ld + row];
    y[k] = T(0);
  }
#pragma unroll
  for (int k = 0; k < kS; ++k) {
#pragma unroll
    for (int j = 0; j < kS; ++j) y[j] = fma(x[k], Qs[k * kS + j], y[j]);
  }
#pragma unroll
  for (int k = 0; k < kS; ++k) {
    const int gcol = (k < kB ? p * kB + k : q * kB + k - kB);
    base[(size_t)gcol * ld + row] = y[k];
  }
}

// ---------------------------------------------------------------------------------------------
// fused round: one thread-block CLUSTER per block pair.  Each CTA of the cluster keeps its row slice of
// the [G;V] panel in shared memory, the partial Gram matrices are summed over the cluster through
// distributed shared memory (fixed order => every CTA holds the identical W and derives the identical Q),
// the small eigenproblem is solved redundantly per CTA and applied to the resident slice.  One launch per
// round, the panel is read once and written once.
// ---------------------------------------------------------------------------------------------
namespace cg = cooperative_groups;

template <typename T>
__global__ void __launch_bounds__(256) jacobi_round_fused_kernel(const JacobiCtx<T> c, int round, T tol, int cs,
                                                                 int rows_g, int rows_v) {
  extern __shared__ __align__(16) unsigned char fused_smem[];
  cg::cluster_group cluster = cg::this_cluster();
  const int rank = (int)cluster.block_rank();
  const int pair = blockIdx.x / cs, b = blockIdx.y;
  const int rows = rows_g + rows_v;
  const int LS = rows | 1;  // odd leading dimension: conflict-free column access
  T* Ps = reinterpret_cast<T*>(fused_smem);                 // [kS][LS]
  T* Wpart = Ps + (size_t)kS * LS;                          // [kS*kS] dense partial Gram
  T* Wa = Wpart + kS * kS;                                  // [kS*kSP]
  T* Wb = Wa + kS * kSP;
  T* Q = Wb + kS * kSP;
  uchar2* pairs = reinterpret_cast<uchar2*>(Q + kS * kSP);  // [(kS-1)*16]
  int* rank_of = reinterpret_cast<int*>(pairs + (kS - 1) * (kS / 2));
  float* ratio_s = reinterpret_cast<float*>(rank_of + kS);

  int p, q;
  rr_pair(c.nb, round, pair, p, q);
  T* Gb = c.G + (size_t)b * c.n_pad * c.ldg;
  T* Vb = c.V + (size_t)b * c.n_pad * c.n_pad;
  const int g0 = rank * rows_g, v0 = rank * rows_v;
  const int gn = max(0, min(rows_g, c.m - g0)), vn = max(0, min(rows_v, c.n_pad - v0));

  fill_pair_table<kS>(pairs);
  if (threadIdx.x == 0) *ratio_s = 0.f;
  // ---- load the slice (coalesced along rows) ----
  for (int k = 0; k < kS; ++k) {
    const int gcol = (k < kB ? p * kB + k : q * kB + k - kB);
    const T* gsrc = Gb + (size_t)gcol * c.ldg + g0;
    const T* vsrc = Vb + (size_t)gcol * c.n_pad + v0;
    T* dst = Ps + (size_t)k * LS;
    for (int r = threadIdx.x; r < rows; r += blockDim.x) {
      T v = T(0);
      if (r < rows_g) { if (r < gn) v = gsrc[r]; }
      else if (r - rows_g < vn) v = vsrc[r - rows_g];
      dst[r] = v;
    }
  }
  __syncthreads();
  // ---- partial Gram over the G rows of this CTA ----
  {
    const int tx = threadIdx.x & 15, ty = threadIdx.x >> 4;
    const T* a0p = Ps + (size_t)(2 * ty) * LS;
    const T* a1p = a0p + LS;
    const T* b0p = Ps + (size_t)(2 * tx) * LS;
    const T* b1p = b0p + LS;
    T acc00 = 0, acc01 = 0, acc10 = 0, acc11 = 0;
#pragma unroll 4
    for (int r = 0; r < gn; ++r) {
      const T a0 = a0p[r], a1 = a1p[r], b0 = b0p[r], b1 = b1p[r];
      acc00 = fma(a0, b0, acc00);
      acc01 = fma(a0, b1, acc01);
      acc10 = fma(a1, b0, acc10);
      acc11 = fma(a1, b1, acc11);
    }
    Wpart[(2 * ty) * kS + 2 * tx] = acc00;
    Wpart[(2 * ty) * kS + 2 * tx + 1] = acc01;
    Wpart[(2 * ty + 1) * kS + 2 * tx] = acc10;
    Wpart[(2 * ty + 1) * kS + 2 * tx + 1] = acc11;
  }
  cluster.sync();
  // ---- cluster-wide sum through distributed shared memory, same order in every CTA ----
  for (int e = threadIdx.x; e < kS * kS; e += blockDim.x) {
    T acc = 0;
    for (int r = 0; r < cs; ++r) acc += cluster.map_shared_rank(Wpart, r)[e];
    const int i = e / kS, j = e % kS;
    Wa[i * kSP + j] = acc;
    Q[i * kSP + j] = (i == j) ? T(1) : T(0);
  }
  cluster.sync();  // all remote reads done: CTAs are independent from here on
  // ---- convergence statistic of this panel ----
  const float null2_b = c.null2[b];
  float myr = 0.f;
  for (int e = threadIdx.x; e < kS * kS; e += blockDim.x) {
    const int i = e / kS, j = e % kS;
    if (i < j) {
      // columns at the rounding-noise level of the matrix (rank-deficient input) have no direction: the cosine
      // between them and anything else is noise and must not keep the iteration "unconverged" forever
      const T wi = Wa[i * kSP + i], wj = Wa[j * kSP + j];
      const T d = wi * wj;
      const T w = fabs(Wa[i * kSP + j]);
      if (d > T(0) && w > T(0) && (float)wi > null2_b && (float)wj > null2_b) myr = fmaxf(myr, (float)(w / sqrt(d)));
    }
  }
  for (int o = 16; o > 0; o >>= 1) myr = fmaxf(myr, __shfl_xor_sync(0xffffffffu, myr, o));
  if ((threadIdx.x & 31) == 0 && myr > 0.f) atomicMax(reinterpret_cast<int*>(ratio_s), __float_as_int(myr));
  __syncthreads();
  const float ratio = *ratio_s;
  if (rank == 0 && threadIdx.x == 0) atomicMax(c.stat + b, __float_as_uint(ratio));
  if (ratio <= (float)tol) return;  // uniform over the cluster (identical W everywhere)

  T* fin = small_syevj<T, kS>(Wa, Wb, Q, pairs);
  __syncthreads();
  if (threadIdx.x < kS) {
    const int i = threadIdx.x;
    const T li = fin[i * kSP + i];
    int rk = 0;
    for (int j = 0; j < kS; ++j) {
      const T lj = fin[j * kSP + j];
      rk += (lj > li || (lj == li && j < i)) ? 1 : 0;
    }
    rank_of[i] = rk;
  }
  __syncthreads();
  T* other = (fin == Wa) ? Wb : Wa;
  reorthonormalise<T, kS>(Q, other, fin);  // fin <- orthonormalised Q (stride kSP)
  // Qs: dense, column-permuted (sorted) copy for the apply loop, reuse Wpart
  for (int e = threadIdx.x; e < kS * kS; e += blockDim.x) {
    const int r = e / kS, i = e % kS;
    Wpart[r * kS + rank_of[i]] = fin[r * kSP + i];
  }
  __syncthreads();
  // ---- apply to the resident slice, write back (coalesced along rows) ----
  for (int r = threadIdx.x; r < rows; r += blockDim.x) {
    const bool isg = r < rows_g;
    const int lr = isg ? r : r - rows_g;
    if (lr >= (isg ? gn : vn)) continue;
    T x[kS], y[kS];
#pragma unroll
    for (int k = 0; k < kS; ++k) {
      x[k] = Ps[(size_t)k * LS + r];
      y[k] = T(0);
    }
#pragma unroll
    for (int k = 0; k < kS; ++k) {
#pragma unroll
      for (int j = 0; j < kS; ++j) y[j] = fma(x[k], Wpart[k * kS + j], y[j]);
    }
    T* dstbase = isg ? (Gb + g0 + lr) : (Vb + v0 + lr);
    const int64_t ld = isg ? c.ldg : (int64_t)c.n_pad;
#pragma unroll
    for (int k = 0; k < kS; ++k) {
      const int gcol = (k < kB ? p * kB + k : q * kB + k - kB);
      dstbase[(size_t)gcol * ld] = y[k];
    }
  }
}

template <typename T>
static size_t fused_smem_bytes(int rows) {
  const int LS = rows | 1;
  return ((size_t)kS * LS + kS * kS + 3 * kS * kSP) * sizeof(T) + (kS - 1) * (kS / 2) * sizeof(uchar2) +
         kS * sizeof(int) + 64;
}

// ---------------------------------------------------------------------------------------------
// setup / teardown kernels
// ---------------------------------------------------------------------------------------------
// G[col j][row i] = in[j*ld_in + i] (colmajor_in) or in[i*ld_in + j]; padded columns zero; V = I.
template <typename T>
__global__ void jacobi_init_kernel(const T* __restrict__ in, int64_t ld_in, int64_t batch_stride_in,
                                   int colmajor_in, int m, int n, JacobiCtx<T> c, T shift) {
  const int b = blockIdx.z;
  const T* A = in + (size_t)b * batch_stride_in;
  T* G = c.G + (size_t)b * c.n_pad * c.ldg;
  T* V = c.V + (size_t)b * c.n_pad * c.n_pad;
  const int col = blockIdx.y;
  for (int row = blockIdx.x * blockDim.x + threadIdx.x; row < max(c.m, c.n_pad);
       row += gridDim.x * blockDim.x) {
    if (row < c.m) {
      T v = T(0);
      if (col < n) {
        v = colmajor_in ? A[(size_t)col * ld_in + row] : A[(size_t)row * ld_in + col];
        if (row == col) v += shift;
      }
      G[(size_t)col * c.ldg + row] = v;
    }
    if (row < c.n_pad) V[(size_t)col * c.n_pad + row] = (row == col) ? T(1) : T(0);
  }
  if (blockIdx.x == 0 && blockIdx.y == 0 && threadIdx.x == 0) c.stat[b] = 0u;
}

// One block per matrix, fixed-order reductions (deterministic):
//  * expo[b] = the exponent of max |G_b| (frexp), and G_b <- 2^-expo G_b, so that max |G_b| lies in [0.5, 1).  The
//    sweeps form products of four entries (w_ii w_jj in the convergence test, a_pp a_qq and a_pq^2 in the rotation
//    test), and the noise floor below is kept in float: away from unit scale these under- or overflow (a float64
//    covariance of data at 1e-12, a float32 matrix with entries near 1e9), no pair gets a ratio, and the sweep
//    reports convergence with V still the identity.  A power of two is exact, so the solve of 2^k A is the solve of A
//    bit for bit and jacobi_values_kernel multiplies the values back by 2^expo.  A zero matrix keeps expo = 0.
//  * null2[b] = (n eps)^2 ||G_b||_F^2 of the normalised G_b.  n eps ||A||_F bounds the rounding error of a column of
//    A V (|fl(A v) - A v| <= n eps |A| |v|), so a column below it carries no direction.  A larger floor stops refining
//    genuine columns: at 10 n eps ||A||_F, a float32 n = 2700 SPD matrix with eigenvalues in [0.01, 1] had every
//    eigenvalue below 0.048 left unrefined (eigenvalue errors of 7.6e-3).
template <typename T>
__global__ void jacobi_scale_kernel(const JacobiCtx<T> c, int n) {
  __shared__ double red[32];
  __shared__ int expo_s;
  const int b = blockIdx.x;
  T* G = c.G + (size_t)b * c.n_pad * c.ldg;
  // ldg == m (make_plan): the n columns of G_b are one run of n m elements, walked without a division per element
  const size_t total = (size_t)n * c.m;
  T amax = T(0);
#pragma unroll 4
  for (size_t e = threadIdx.x; e < total; e += blockDim.x) amax = fmax(amax, fabs(G[e]));
  for (int o = 16; o > 0; o >>= 1) amax = fmax(amax, __shfl_xor_sync(0xffffffffu, amax, o));
  if ((threadIdx.x & 31) == 0) red[threadIdx.x >> 5] = (double)amax;
  __syncthreads();
  if (threadIdx.x == 0) {
    double t = 0.0;
    for (int w = 0; w < (int)(blockDim.x >> 5); ++w) t = fmax(t, red[w]);
    int ex = 0;
    if (t > 0.0) frexp(t, &ex);
    expo_s = ex;
    c.expo[b] = ex;
  }
  __syncthreads();
  const int ex = expo_s;
  double acc = 0.0;
#pragma unroll 4
  for (size_t e = threadIdx.x; e < total; e += blockDim.x) {
    const T v = ldexp(G[e], -ex);
    G[e] = v;
    acc += (double)v * (double)v;
  }
  for (int o = 16; o > 0; o >>= 1) acc += __shfl_xor_sync(0xffffffffu, acc, o);
  if ((threadIdx.x & 31) == 0) red[threadIdx.x >> 5] = acc;
  __syncthreads();
  if (threadIdx.x == 0) {
    double t = 0.0;
    for (int w = 0; w < (int)(blockDim.x >> 5); ++w) t += red[w];
    const double ne = (double)n * (double)Eps<T>::v;
    c.null2[b] = (float)fmin(ne * ne * t, 3.0e38);   // norm threshold n eps ||G||_F
  }
}

__global__ void jacobi_reset_stat_kernel(unsigned* stat, int batch) {
  if (threadIdx.x < batch) stat[threadIdx.x] = 0u;
}

// one warp per column: value (Rayleigh quotient or norm), pad detection, optional normalisation of G.  The value is
// formed in the scale of the normalised G and multiplied back by 2^expo (exact).
template <typename T>
__global__ void jacobi_values_kernel(JacobiCtx<T> c, int n, int svd_mode, T shift, T* __restrict__ vals,
                                     T* __restrict__ vnorm) {
  const int b = blockIdx.y;
  const int col = blockIdx.x * (blockDim.x / 32) + (threadIdx.x >> 5);
  const int lane = threadIdx.x & 31;
  if (col >= c.n_pad) return;
  T* g = c.G + (size_t)b * c.n_pad * c.ldg + (size_t)col * c.ldg;
  const T* v = c.V + (size_t)b * c.n_pad * c.n_pad + (size_t)col * c.n_pad;
  T acc = 0, padw = 0, vv = 0;
  if (svd_mode) {
    for (int i = lane; i < c.m; i += 32) acc = fma(g[i], g[i], acc);
  } else {
    for (int i = lane; i < n; i += 32) acc = fma(v[i], g[i], acc);
  }
  for (int i = lane; i < n; i += 32) vv = fma(v[i], v[i], vv);
  for (int i = n + lane; i < c.n_pad; i += 32) padw = fma(v[i], v[i], padw);
  for (int o = 16; o > 0; o >>= 1) {
    acc += __shfl_xor_sync(0xffffffffu, acc, o);
    padw += __shfl_xor_sync(0xffffffffu, padw, o);
    vv += __shfl_xor_sync(0xffffffffu, vv, o);
  }
  const int ex = c.expo[b];
  T val;
  if (padw > T(0.5)) {
    val = neg_inf<T>();  // padding direction: sorts last, never output
  } else if (svd_mode) {
    const T nrm = sqrt(acc);
    const T inv = nrm > T(0) ? T(1) / nrm : T(0);
    for (int i = lane; i < c.m; i += 32) g[i] *= inv;
    val = ldexp(nrm, ex);
  } else {
    // Rayleigh quotient of the (re-normalised) vector, un-shifted by the shift in the same scale
    val = ldexp((vv > T(0) ? acc / vv : acc) - ldexp(shift, -ex), ex);
  }
  if (lane == 0) {
    vals[(size_t)b * c.n_pad + col] = val;
    vnorm[(size_t)b * c.n_pad + col] = vv > T(0) ? T(1) / sqrt(vv) : T(1);
  }
}

// rank-by-counting sort (descending) + gather of the vectors as rows
template <typename T>
__global__ void jacobi_rank_kernel(const T* __restrict__ vals, int n_pad, int* __restrict__ rank) {
  const int b = blockIdx.y;
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n_pad) return;
  const T* v = vals + (size_t)b * n_pad;
  const T vi = v[i];
  int rk = 0;
  for (int j = 0; j < n_pad; ++j) {
    const T vj = v[j];
    rk += (vj > vi || (vj == vi && j < i)) ? 1 : 0;
  }
  rank[(size_t)b * n_pad + i] = rk;
}

template <typename T>
__global__ void jacobi_gather_kernel(JacobiCtx<T> c, int n, const T* __restrict__ vals,
                                     const T* __restrict__ vnorm, const int* __restrict__ rank, T* __restrict__ out_vals,
                                     int64_t vals_stride, T* __restrict__ out_right, int64_t ld_right,
                                     int64_t right_stride, T* __restrict__ out_left, int64_t ld_left,
                                     int64_t left_stride) {
  const int b = blockIdx.y, col = blockIdx.x;
  const int rk = rank[(size_t)b * c.n_pad + col];
  if (rk >= n) return;  // padding directions
  if (threadIdx.x == 0 && out_vals) out_vals[(size_t)b * vals_stride + rk] = vals[(size_t)b * c.n_pad + col];
  if (out_right) {
    const T* v = c.V + (size_t)b * c.n_pad * c.n_pad + (size_t)col * c.n_pad;
    T* o = out_right + (size_t)b * right_stride + (size_t)rk * ld_right;
    const T sc = vnorm[(size_t)b * c.n_pad + col];
    for (int i = threadIdx.x; i < n; i += blockDim.x) o[i] = v[i] * sc;
  }
  if (out_left) {
    const T* g = c.G + (size_t)b * c.n_pad * c.ldg + (size_t)col * c.ldg;
    T* o = out_left + (size_t)b * left_stride + (size_t)rk * ld_left;
    for (int i = threadIdx.x; i < c.m; i += blockDim.x) o[i] = g[i];
  }
}

// ---------------------------------------------------------------------------------------------
// host driver
// ---------------------------------------------------------------------------------------------
// Pinned landing buffer of the per-sweep convergence flags.  Grow-only and kept for the life of the calling
// thread: cudaMallocHost / cudaFreeHost cost 0.5-10 ms per call (the free synchronises the device), which used to
// dominate every small eigensolve.  Portable so that one process driving several devices can share it.
static unsigned* pinned_stat_buffer(size_t count) {
  static thread_local unsigned* buf = nullptr;
  static thread_local size_t cap = 0;
  if (count > cap) {
    if (buf) cudaFreeHost(buf);
    buf = nullptr;
    cap = 0;
    const size_t want = std::max<size_t>(count, 1024);
    if (cudaHostAlloc(reinterpret_cast<void**>(&buf), want * sizeof(unsigned), cudaHostAllocPortable) != cudaSuccess) {
      buf = nullptr;
      return nullptr;
    }
    cap = want;
  }
  return buf;
}

namespace {
inline size_t al(size_t x) { return (x + 255) & ~size_t(255); }

template <typename T>
struct Plan {
  int n_pad, nb, npairs, R, rows_per_part;
  int64_t ldg;
  size_t oG, oV, oW, oQ, oSkip, oStat, oNull, oExpo, oVals, oNorm, oRank, total;
};

template <typename T>
Plan<T> make_plan(int m, int n, int batch) {
  Plan<T> P;
  P.n_pad = (int)ceil_div(n, kS) * kS;
  P.nb = P.n_pad / kB;
  P.npairs = P.nb / 2;
  P.ldg = m;
  // enough Gram partials to fill the machine, at least 128 rows each
  int R = (int)std::max<int64_t>(1, std::min<int64_t>(ceil_div(m, 128), ceil_div(4 * 148, (int64_t)P.npairs * batch)));
  R = std::min(R, 16);
  P.rows_per_part = (int)ceil_div(ceil_div(m, R), 64) * 64;
  P.R = (int)ceil_div(m, P.rows_per_part);
  size_t o = 0;
  P.oG = o; o += al((size_t)batch * P.n_pad * P.ldg * sizeof(T));
  P.oV = o; o += al((size_t)batch * P.n_pad * P.n_pad * sizeof(T));
  P.oW = o; o += al((size_t)batch * P.npairs * P.R * kS * kS * sizeof(T));
  P.oQ = o; o += al((size_t)batch * P.npairs * kS * kS * sizeof(T));
  P.oSkip = o; o += al((size_t)batch * P.npairs * sizeof(int));
  P.oStat = o; o += al((size_t)batch * sizeof(unsigned));
  P.oNull = o; o += al((size_t)batch * sizeof(float));
  P.oExpo = o; o += al((size_t)batch * sizeof(int));
  P.oVals = o; o += al((size_t)batch * P.n_pad * sizeof(T));
  P.oNorm = o; o += al((size_t)batch * P.n_pad * sizeof(T));
  P.oRank = o; o += al((size_t)batch * P.n_pad * sizeof(int));
  P.total = o + 256;
  return P;
}
}  // namespace

template <typename T>
size_t jacobi_workspace_bytes(int m, int n, int batch) {
  return make_plan<T>(m, n, batch).total;
}

template <typename T>
int jacobi_solve(const JacobiArgs<T>& a, void* ws, size_t ws_bytes, cudaStream_t stream) {
  const int m = a.m, n = a.n, batch = a.batch;
  CCAB_CHECK_ARG(m >= 1 && n >= 1 && batch >= 1 && batch <= 1024, "bad jacobi shape m=%d n=%d batch=%d", m, n,
                 batch);
  CCAB_CHECK_ARG(a.svd_mode || m == n, "symmetric mode needs a square matrix");
  Plan<T> P = make_plan<T>(m, n, batch);
  CCAB_CHECK_ARG(ws_bytes >= P.total, "workspace too small: %zu < %zu", ws_bytes, P.total);
  uint8_t* w = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(ws) + 255) & ~uintptr_t(255));
  JacobiCtx<T> c;
  c.G = reinterpret_cast<T*>(w + P.oG);
  c.V = reinterpret_cast<T*>(w + P.oV);
  c.Wpart = reinterpret_cast<T*>(w + P.oW);
  c.Qm = reinterpret_cast<T*>(w + P.oQ);
  c.skip = reinterpret_cast<int*>(w + P.oSkip);
  c.stat = reinterpret_cast<unsigned*>(w + P.oStat);
  c.null2 = reinterpret_cast<float*>(w + P.oNull);
  c.expo = reinterpret_cast<int*>(w + P.oExpo);
  T* vals = reinterpret_cast<T*>(w + P.oVals);
  T* vnorm = reinterpret_cast<T*>(w + P.oNorm);
  int* rank = reinterpret_cast<int*>(w + P.oRank);
  c.m = m;
  c.n_pad = P.n_pad;
  c.nb = P.nb;
  c.npairs = P.npairs;
  c.R = P.R;
  c.ldg = P.ldg;
  c.rows_per_part = P.rows_per_part;

  const T shift = a.svd_mode ? T(0) : (T)a.shift;
  {
    const int rows = std::max(m, P.n_pad);
    dim3 grid((unsigned)std::min<int64_t>(ceil_div(rows, 256), 64), P.n_pad, batch);
    jacobi_init_kernel<T><<<grid, 256, 0, stream>>>(a.in, a.ld_in, a.batch_stride_in, a.colmajor_in, m, n, c, shift); count_launches(1);
    jacobi_scale_kernel<T><<<batch, 1024, 0, stream>>>(c, n); count_launches(1);
    CCAB_CUDA(cudaGetLastError());
  }
  const T tol = a.tol > 0 ? (T)a.tol : (T)(4.0 * (double)Eps<T>::v * std::sqrt((double)m));
  // the same cap for both precisions: the block sweeps spend a phase that grows with n before the quadratic one sets in
  // (a float32 n = 2700 SPD matrix with eigenvalues spread over [0.01, 1] converges in its 17th sweep, to eigenvalue
  // errors of 0.005 n eps ||A||), and the cap only costs time on a solve that would otherwise be reported unconverged.
  // Rank-deficient blocks have a long phase of their own: the columns of the null cluster keep normalised
  // off-diagonals near 1 until their norms fall below the noise floor, then the sweep converges at once (a 300 x 300
  // float64 covariance of rank 150, 900 samples: 25 sweeps), so the cap leaves room well beyond that
  const int max_sweeps = a.max_sweeps > 0 ? a.max_sweeps : 64;
  // fused cluster path: smallest cluster (<= 8 CTAs) whose row slice fits comfortably in shared memory; when none
  // fits (large m), each round runs as three kernels (gram / solve / apply)
  int cs = 0, rows_g = 0, rows_v = 0;
  size_t fused_bytes = 0;
  for (int cand = 1; cand <= 8; cand *= 2) {
    const int rg = (int)ceil_div(m, cand), rv = (int)ceil_div(P.n_pad, cand);
    const size_t bytes = fused_smem_bytes<T>(rg + rv);
    const size_t limit = (size_t)P.npairs * batch * cand >= 296 ? 100 * 1024 : 200 * 1024;
    if (bytes <= limit) {
      cs = cand; rows_g = rg; rows_v = rv; fused_bytes = bytes;
      // prefer more CTAs per pair while the machine is not full
      if ((size_t)P.npairs * batch * cand >= 148 || cand == 8) break;
    }
  }
  if (cs) {
    cudaError_t e = cudaFuncSetAttribute(jacobi_round_fused_kernel<T>, cudaFuncAttributeMaxDynamicSharedMemorySize,
                                         (int)fused_bytes);
    if (e != cudaSuccess) return cuda_fail(e, "cudaFuncSetAttribute(jacobi_round_fused_kernel)");
  }
  const int rounds = P.nb - 1;
  const int apply_chunks = (int)(ceil_div(m, 128) + ceil_div(P.n_pad, 128));
  int sweeps_done = 0;
  float last_ratio = -1.f;
  unsigned* h_stat = pinned_stat_buffer((size_t)batch);
  CCAB_CHECK_ARG(h_stat != nullptr, "could not allocate the pinned convergence-flag buffer");
  int rc = 0;
  for (int sweep = 0; sweep < max_sweeps; ++sweep) {
    for (int r = 0; r < rounds; ++r) {
      if (cs) {
        cudaLaunchConfig_t cfg;
        memset(&cfg, 0, sizeof(cfg));
        cfg.gridDim = dim3(P.npairs * cs, batch, 1);
        cfg.blockDim = dim3(256, 1, 1);
        cfg.dynamicSmemBytes = fused_bytes;
        cfg.stream = stream;
        cudaLaunchAttribute attr[1];
        attr[0].id = cudaLaunchAttributeClusterDimension;
        attr[0].val.clusterDim.x = cs;
        attr[0].val.clusterDim.y = 1;
        attr[0].val.clusterDim.z = 1;
        cfg.attrs = attr;
        cfg.numAttrs = 1;
        cudaError_t le = cudaLaunchKernelEx(&cfg, jacobi_round_fused_kernel<T>, c, r, tol, cs, rows_g, rows_v);
        if (le != cudaSuccess) { rc = cuda_fail(le, "jacobi_round_fused_kernel launch"); break; }
        count_launches(1);
      } else {
        jacobi_gram_kernel<T><<<dim3(P.npairs, P.R, batch), 256, 0, stream>>>(c, r); count_launches(1);
        jacobi_solve_kernel<T><<<dim3(P.npairs, batch), 256, 0, stream>>>(c, tol); count_launches(1);
        jacobi_apply_kernel<T><<<dim3(P.npairs, apply_chunks, batch), 128, 0, stream>>>(c, r); count_launches(1);
      }
    }
    if (rc) break;
    cudaError_t e = cudaGetLastError();
    if (e != cudaSuccess) { rc = cuda_fail(e, "jacobi sweep launch"); break; }
    e = cudaMemcpyAsync(h_stat, c.stat, sizeof(unsigned) * batch, cudaMemcpyDeviceToHost, stream);
    if (e == cudaSuccess) e = cudaStreamSynchronize(stream);
    if (e != cudaSuccess) { rc = cuda_fail(e, "jacobi sweep sync"); break; }
    ++sweeps_done;
    float worst = 0.f;
    for (int b = 0; b < batch; ++b) {
      float f;
      memcpy(&f, &h_stat[b], 4);
      worst = std::max(worst, f);
    }
    last_ratio = worst;
    if (getenv("CCAB_JACOBI_VERBOSE")) fprintf(stderr, "[syevj] sweep %d worst offdiag %.3e (tol %.3e)\n", sweep, worst, (double)tol);
    if (worst <= (float)tol) break;
    jacobi_reset_stat_kernel<<<1, 1024, 0, stream>>>(c.stat, batch); count_launches(1);
  }
  if (rc) return rc;
  // "no silent fallback": a solve that ran out of sweeps reports it -- info[0] = -sweeps, and the call fails unless the
  // caller asked for the diagnostics (info != NULL) and therefore handles the sign itself
  const bool converged = last_ratio >= 0.f && last_ratio <= (float)tol;
  if (a.info) { a.info[0] = converged ? sweeps_done : -sweeps_done; }
  if (a.final_offdiag) *a.final_offdiag = last_ratio;
  if (!converged && !a.info) {
    set_error("Jacobi iteration did not converge in %d sweeps (normalised off-diagonal %.3e > tolerance %.3e)",
              sweeps_done, (double)last_ratio, (double)tol);
    return -20;
  }

  jacobi_values_kernel<T><<<dim3((unsigned)ceil_div(P.n_pad, 8), batch), 256, 0, stream>>>(c, n, a.svd_mode, shift, vals, vnorm); count_launches(1);
  jacobi_rank_kernel<T><<<dim3((unsigned)ceil_div(P.n_pad, 256), batch), 256, 0, stream>>>(vals, P.n_pad, rank); count_launches(1);
  jacobi_gather_kernel<T><<<dim3(P.n_pad, batch), 128, 0, stream>>>(
      c, n, vals, vnorm, rank, a.out_vals, a.vals_stride, a.out_right, a.ld_right, a.right_stride, a.out_left, a.ld_left,
      a.left_stride); count_launches(1);
  CCAB_CUDA(cudaGetLastError());
  return 0;
}

template size_t jacobi_workspace_bytes<float>(int, int, int);
template size_t jacobi_workspace_bytes<double>(int, int, int);
template int jacobi_solve<float>(const JacobiArgs<float>&, void*, size_t, cudaStream_t);
template int jacobi_solve<double>(const JacobiArgs<double>&, void*, size_t, cudaStream_t);

}  // namespace ccab
