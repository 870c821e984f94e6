// Small symmetric eigensolver: ONE single-CTA launch per matrix (n <= 128 float / 96 double), everything in shared
// memory, no host involvement -- the Rayleigh-Ritz step of the subspace iteration (p x p, p = k + oversampling)
// and any other small, well-conditioned symmetric problem of the solver stage.
//
// Classical two-sided Jacobi with the round-robin (tournament) parallel ordering: per step n/2 disjoint index pairs
// are rotated at once.  Thread i < n/2 computes the rotation of pair i from the current 2 x 2 pivot block; then the
// (n/2)^2 2 x 2 blocks  H[{p_i,q_i}, {p_j,q_j}]  are each updated by ONE thread (row rotation of pair i, column
// rotation of pair j -- the blocks partition H, so there is no hazard) and the eigenvector rows are rotated
// alongside.  Two block barriers per step, n - 1 steps per sweep, software-pipelined: the rotations of step t + 1 are
// computed (by n/2 threads) while the other threads rotate the eigenvectors of step t; only the upper triangle of H
// is kept.  The off-diagonal mass seen during a sweep decides convergence on the device.  Eigenvalues are returned in descending order with the eigenvectors as rows.
// H is solved multiplied by the power of two that brings max |H| into [0.5, 1), and the eigenvalues are scaled back.
//
// Two-sided Jacobi resolves eigenvalues to eps * ||H|| (absolute): right for the Ritz problem, whose block is well
// conditioned; the whitening eigenproblems (tiny eigenvalues matter relatively) stay on the one-sided solver of
// syevj.cu.  Replaces, with the subspace iteration around it, scipy.linalg.eigh / np.linalg.svd of
// cca_zoo/_utils/_linalg.py:64-73 and cca_zoo/linear/_rcca.py:97 when only the leading k pairs are wanted.
#include "syevj_small.cuh"

#include <cmath>

namespace ccab {

namespace {

constexpr int kSmallThreads = 512;
constexpr int kSmallMaxN = 128;                      // (n/2)^2 2 x 2 blocks over 1024 threads: 4 per thread
constexpr int kHB = ((kSmallMaxN / 2) * (kSmallMaxN / 2 + 1) / 2 + kSmallThreads - 1) / kSmallThreads;   // upper-triangle pair blocks per thread
constexpr int kVB = ((kSmallMaxN / 2) * (kSmallMaxN / 4) + kSmallThreads - 64 - 1) / (kSmallThreads - 64);   // V items per non-rotation thread: (n/2) * ceil(n/4) <= 2048

template <typename T>
struct SmallEps;
template <>
struct SmallEps<float> {
  static constexpr float v = 1.1920929e-7f;
};
template <>
struct SmallEps<double> {
  static constexpr double v = 2.220446049250313e-16;
};

// Position bookkeeping of the tournament: the matrix is PHYSICALLY permuted after every step so that the rotation
// pairs are always the adjacent positions (2i, 2i+1) -- all addresses are affine in the block indices, no index
// tables.  Brent-Luk movement on the 2 x (N/2) array top[i] = position 2i, bot[i] = position 2i+1: top[0] stays,
// bot[0] -> top[1], top[i] -> top[i+1], top[last] -> bot[last], bot[i] -> bot[i-1].
__device__ __forceinline__ int rr_dest(int r, int N) {
  if (r == 0 || N == 2) return r;
  if (r == 1) return 2;
  if (r & 1) return r - 2;                 // bot[i] -> bot[i-1]
  return r + 2 < N ? r + 2 : N - 1;        // top[i] -> top[i+1], the last one drops to the bottom row
}

__device__ __forceinline__ float fast_sqrt(float x) { return __fsqrt_rn(x); }
__device__ __forceinline__ double fast_sqrt(double x) { return sqrt(x); }
__device__ __forceinline__ float fast_rsqrt(float x) {
  const float r = rsqrtf(x);
  return r * fmaf(-0.5f * x * r, r, 1.5f);
}
__device__ __forceinline__ double fast_rsqrt(double x) { return 1.0 / sqrt(x); }
__device__ __forceinline__ float fast_div(float a, float b) { return __fdividef(a, b); }
__device__ __forceinline__ double fast_div(double a, double b) { return a / b; }

template <typename T>
struct alignas(2 * sizeof(T)) Rot2 {
  T s, tau;   // Rutishauser: x' = x - s (y + tau x), y' = y + s (x - tau y)
};

template <typename T>
__global__ void __launch_bounds__(kSmallThreads, 1)
syevj_small_kernel(const T* __restrict__ A, int64_t lda, int64_t strideA, int n, T* __restrict__ evals,
                   int64_t strideE, T* __restrict__ evt, int64_t ldv, int64_t strideV, int max_sweeps, T tol,
                   int* __restrict__ info) {
  // grid = (nsplit, batch): every CTA of a matrix runs the SAME rotations on its own copy of H (identical
  // arithmetic, hence identical bits) and accumulates the eigenvector columns [c0, c1) only -- the V update is
  // as large as the H update and splits without any communication.
  extern __shared__ __align__(16) unsigned char sv_smem[];
  const int N = (n + 1) & ~1;      // even number of positions; for odd n one of them is a bye (zero row / column)
  const int LD = N + 2;            // even: the two columns of a pair sit in one aligned 2-vector
  const int m2 = N / 2;
  const int nsplit = gridDim.x;
  const int cw = (n + nsplit - 1) / nsplit;              // eigenvector columns of this CTA
  const int c0 = blockIdx.x * cw;
  const int c1 = min(n, c0 + cw);
  const int ncol = max(0, c1 - c0);
  const int LDV = cw + 1;
  T* const H0 = reinterpret_cast<T*>(sv_smem);
  T* const H1 = H0 + (size_t)N * LD;
  T* const V0 = H1 + (size_t)N * LD;
  T* const V1 = V0 + (size_t)N * LDV;
  T* red = V1 + (size_t)N * LDV;                         // [32]
  Rot2<T>* rot = reinterpret_cast<Rot2<T>*>((reinterpret_cast<uintptr_t>(red + 32) + 15) & ~uintptr_t(15));   // [2][m2]
  int* label = reinterpret_cast<int*>(rot + 2 * m2);     // [2][N] original index held by a position (-1: the bye)
  int* rank = label + 2 * N;                             // [N]
  __shared__ int done;
  __shared__ int expo;
  const int tid = threadIdx.x;
  const int warp = tid >> 5, lane = tid & 31;
  const T* Ab = A + (size_t)blockIdx.y * strideA;

  // ---- load (symmetrised), V = I (own columns), max |H| ----
  T amax = T(0);
#pragma unroll 4
  for (int e = tid; e < N * N; e += kSmallThreads) {
    const int r = e / N, c = e % N;
    T v = T(0);
    if (r < n && c < n) v = T(0.5) * (Ab[(size_t)r * lda + c] + Ab[(size_t)c * lda + r]);
    H0[r * LD + c] = v;
    amax = fmax(amax, fabs(v));
  }
  for (int e = tid; e < N * cw; e += kSmallThreads) {
    const int r = e / cw, c = e % cw;
    V0[r * LDV + c] = (r == c0 + c && r < n) ? T(1) : T(0);
  }
  if (tid < N) label[tid] = tid < n ? tid : -1;
  for (int o = 16; o > 0; o >>= 1) amax = fmax(amax, __shfl_xor_sync(0xffffffffu, amax, o));
  if (lane == 0) red[warp] = amax;
  if (tid == 0) done = 0;
  __syncthreads();
  // ---- H <- 2^-expo H with max |H| in [0.5, 1), ||H||_F^2 ----
  // The rotation and convergence tests below compare sums of squares: away from unit scale they under- or overflow
  // (a float32 matrix with entries near 1e20 makes ||H||_F^2 infinite and the first sweep "converged").  A power of
  // two is exact, so the solve of 2^k A is the solve of A bit for bit; the eigenvalues are scaled back when written.
  // A zero matrix keeps expo = 0.
  {
    for (int w = 0; w < kSmallThreads / 32; ++w) amax = fmax(amax, red[w]);
    int ex = 0;
    if (amax > T(0)) frexp(amax, &ex);
    if (tid == 0) expo = ex;
    __syncthreads();
    T fro_local = T(0);
#pragma unroll 4
    for (int e = tid; e < N * N; e += kSmallThreads) {
      const int r = e / N, c = e % N;
      const T v = ldexp(H0[r * LD + c], -ex);
      H0[r * LD + c] = v;
      fro_local = fma(v, v, fro_local);
    }
    for (int o = 16; o > 0; o >>= 1) fro_local += __shfl_xor_sync(0xffffffffu, fro_local, o);
    if (lane == 0) red[warp] = fro_local;
  }
  __syncthreads();
  T fro2 = T(0);
  for (int w = 0; w < kSmallThreads / 32; ++w) fro2 += red[w];
  __syncthreads();

  // static work assignment: upper-triangle pair blocks (i <= j), V items (pair, column)
  const int nt = m2 * (m2 + 1) / 2;
  int bi[kHB], bj[kHB];
#pragma unroll
  for (int u = 0; u < kHB; ++u) {
    int t = tid + u * kSmallThreads;
    bi[u] = -1; bj[u] = 0;
    if (t < nt) {
      int i = 0, rowlen = m2;
      while (t >= rowlen) { t -= rowlen; ++i; --rowlen; }
      bi[u] = i; bj[u] = i + t;
    }
  }
  // V items go to the threads that do not compute rotations (tid >= 64): the two run side by side in phase B
  constexpr int kVThreads = kSmallThreads - 64;
  int vi[kVB], vc[kVB];
#pragma unroll
  for (int u = 0; u < kVB; ++u) {
    const int e = (tid - 64) + u * kVThreads;
    const bool ok = tid >= 64 && ncol > 0 && e < m2 * ncol;
    vi[u] = ok ? e / ncol : -1;
    vc[u] = ok ? e % ncol : 0;
  }

  // rotation of the adjacent pair (2 tid, 2 tid + 1) of Hs into rbuf[tid]; returns the off-diagonal mass it removes.
  // Only the UPPER triangle of H is maintained (element (r, c) lives at [min][max]): half the scattered stores.
  auto make_rotation = [&](const T* Hs, Rot2<T>* rbuf) -> T {
    const int p = 2 * tid, q = p + 1;
    const T hpp = Hs[p * LD + p], hqq = Hs[q * LD + q], hpq = Hs[p * LD + q];
    T sn = T(0), tau = T(0);
    // the whole CTA waits for these few threads: keep the dependent chain short (4 special-function ops).
    // With z = (hqq - hpp) / 2 and r = hypot(z, hpq):  tan = hpq / (z + sign(z) r)  (the smaller root),
    // c = 1 / sqrt(1 + tan^2), s = tan c, tau = s / (1 + c).  The rotation only has to be orthogonal to
    // rounding (it is, by construction of the update from s and tau) and ANNIHILATE approximately: a pivot left
    // at 1e-7 of its size is finished off by the next sweep, so fast reciprocals are good enough in float.
    if (hpq * hpq > SmallEps<T>::v * SmallEps<T>::v * T(1e-4) * fabs(hpp * hqq) && hpq != T(0)) {
      const T z = T(0.5) * (hqq - hpp);
      const T r = fast_sqrt(fma(z, z, hpq * hpq));
      const T tt = fast_div(hpq, z + (z >= T(0) ? r : -r));
      const T c = fast_rsqrt(fma(tt, tt, T(1)));
      sn = tt * c;
      tau = fast_div(sn, T(1) + c);
    }
    Rot2<T> r;
    r.s = sn; r.tau = tau;
    rbuf[tid] = r;
    return T(2) * hpq * hpq;
  };

  // Software pipeline: per step  A: H update with rot[rc] (all threads)  | barrier |
  //                              B: rotations of the NEXT step from the new H (tid < m2) alongside the eigenvector
  //                                 update of THIS step with rot[rc] (tid >= 64)                      | barrier |
  // so the few threads of the rotation chain no longer stall the whole CTA.
  int cur = 0, rc = 0, sweeps = 0;
  T off_local = T(0), off_next = T(0);
  if (tid < m2) off_local = make_rotation(H0, rot);
  __syncthreads();
  for (int sweep = 0; sweep < max_sweeps; ++sweep) {
    for (int t = 0; t < N - 1; ++t) {
      const T* H = cur ? H1 : H0;
      T* Hn = cur ? H0 : H1;
      const T* V = cur ? V1 : V0;
      T* Vn = cur ? V0 : V1;
      const Rot2<T>* rcur = rot + rc * m2;
      Rot2<T>* rnext = rot + (rc ^ 1) * m2;
      // ---- phase A: H <- J^T H J on the upper-triangle pair blocks, written to the NEXT buffer at the positions the
      // tournament moves them to (reads and writes never touch the same buffer) ----
      if (tid < N) label[(cur ^ 1) * N + rr_dest(tid, N)] = label[cur * N + tid];
#pragma unroll
      for (int u = 0; u < kHB; ++u) {
        if (bi[u] < 0) continue;
        const int i = bi[u], j = bj[u];
        const Rot2<T> ri = rcur[i], rj = rcur[j];
        const T* h0 = H + (2 * i) * LD + 2 * j;
        const T a = h0[0], b = h0[1], d = h0[LD + 1];
        const T c_ = i == j ? b : h0[LD];             // the pivot block's lower element is its upper one
        const T a1 = a - ri.s * (c_ + ri.tau * a), c1 = c_ + ri.s * (a - ri.tau * c_);
        const T b1 = b - ri.s * (d + ri.tau * b), d1 = d + ri.s * (b - ri.tau * d);
        T a2 = a1 - rj.s * (b1 + rj.tau * a1), b2 = b1 + rj.s * (a1 - rj.tau * b1);
        T c2 = c1 - rj.s * (d1 + rj.tau * c1), d2 = d1 + rj.s * (c1 - rj.tau * d1);
        const int rp = rr_dest(2 * i, N), rq = rr_dest(2 * i + 1, N), cp = rr_dest(2 * j, N), cq = rr_dest(2 * j + 1, N);
        if (i == j) {                               // pivot block: annihilated exactly (kept when not rotated)
          if (ri.s != T(0)) b2 = T(0);
          Hn[rp * LD + rp] = a2;
          Hn[rq * LD + rq] = d2;
          Hn[min(rp, rq) * LD + max(rp, rq)] = b2;
        } else {
          Hn[min(rp, cp) * LD + max(rp, cp)] = a2;
          Hn[min(rp, cq) * LD + max(rp, cq)] = b2;
          Hn[min(rq, cp) * LD + max(rq, cp)] = c2;
          Hn[min(rq, cq) * LD + max(rq, cq)] = d2;
        }
      }
      __syncthreads();
      // ---- phase B ----
      if (tid < m2) {
        const T o = make_rotation(Hn, rnext);
        if (t == N - 2) off_next = o; else off_local += o;   // the last one already belongs to the next sweep
      }
#pragma unroll
      for (int u = 0; u < kVB; ++u) {
        if (vi[u] < 0) continue;
        const Rot2<T> r = rcur[vi[u]];
        const int p = 2 * vi[u];
        const T vp = V[p * LDV + vc[u]], vq = V[(p + 1) * LDV + vc[u]];
        Vn[rr_dest(p, N) * LDV + vc[u]] = vp - r.s * (vq + r.tau * vp);
        Vn[rr_dest(p + 1, N) * LDV + vc[u]] = vq + r.s * (vp - r.tau * vq);
      }
      __syncthreads();
      cur ^= 1;
      rc ^= 1;
    }
    ++sweeps;
    for (int o = 16; o > 0; o >>= 1) off_local += __shfl_xor_sync(0xffffffffu, off_local, o);
    if (lane == 0) red[warp] = off_local;
    __syncthreads();
    if (tid == 0) {
      T off2 = T(0);
      for (int w = 0; w < kSmallThreads / 32; ++w) off2 += red[w];
      done = !(off2 > tol * tol * fro2);
    }
    __syncthreads();
    if (done) break;
    off_local = off_next;
    off_next = T(0);
  }

  // ---- sort (rank by counting, descending; ties by position) and write ----
  const T* H = cur ? H1 : H0;
  const T* V = cur ? V1 : V0;
  const int* lab = label + cur * N;
  if (tid < N) {
    int rk = -1;
    if (lab[tid] >= 0) {
      const T li = H[tid * LD + tid];
      rk = 0;
      for (int j = 0; j < N; ++j) {
        if (lab[j] < 0) continue;
        const T lj = H[j * LD + j];
        rk += (lj > li || (lj == li && j < tid)) ? 1 : 0;
      }
      if (evals && blockIdx.x == 0) evals[(size_t)blockIdx.y * strideE + rk] = ldexp(li, expo);
    }
    rank[tid] = rk;
  }
  __syncthreads();
  if (evt) {
    T* Eb = evt + (size_t)blockIdx.y * strideV;
    for (int e = tid; e < N * ncol; e += kSmallThreads) {
      const int r = e / ncol, c = e - r * ncol;
      if (rank[r] >= 0) Eb[(size_t)rank[r] * ldv + c0 + c] = V[r * LDV + c];
    }
  }
  if (tid == 0 && info && blockIdx.x == 0) info[blockIdx.y] = done ? sweeps : -sweeps;
}

inline int small_nsplit(int n) { return n >= 64 ? 4 : (n >= 24 ? 2 : 1); }

template <typename T>
size_t small_smem_bytes(int n) {
  const int N = (n + 1) & ~1;
  const int cw = (n + small_nsplit(n) - 1) / small_nsplit(n);
  return sizeof(T) * (2 * (size_t)N * (N + 2) + 2 * (size_t)N * (cw + 1) + 32) + sizeof(Rot2<T>) * (size_t)N +
         sizeof(int) * 3 * (size_t)N + 128;
}

}  // namespace

template <typename T>
bool syevj_small_supported(int n) {
  return n >= 1 && n <= kSmallMaxN && small_smem_bytes<T>(n) <= 220 * 1024;
}

template <typename T>
int syevj_small(int n, int batch, const T* A, int64_t lda, int64_t strideA, T* evals, int64_t strideE, T* evt,
                int64_t ldv, int64_t strideV, int* info_dev, cudaStream_t stream) {
  CCAB_CHECK_ARG(syevj_small_supported<T>(n), "syevj_small: n = %d does not fit one CTA's shared memory", n);
  CCAB_CHECK_ARG(batch >= 1 && lda >= n && (!evt || ldv >= n), "bad syevj_small shape");
  const size_t smem = small_smem_bytes<T>(n);
  CCAB_CUDA(cudaFuncSetAttribute(syevj_small_kernel<T>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
  const int max_sweeps = sizeof(T) == 4 ? 14 : 18;
  const T tol = T(4) * SmallEps<T>::v * (T)std::sqrt((double)n);
  syevj_small_kernel<T><<<dim3(small_nsplit(n), batch), kSmallThreads, smem, stream>>>(A, lda, strideA, n, evals, strideE, evt, ldv, strideV,
                                                               max_sweeps, tol, info_dev);
  count_launches(1);
  CCAB_CUDA(cudaGetLastError());
  return 0;
}

template bool syevj_small_supported<float>(int);
template bool syevj_small_supported<double>(int);
template int syevj_small<float>(int, int, const float*, int64_t, int64_t, float*, int64_t, float*, int64_t, int64_t,
                                int*, cudaStream_t);
template int syevj_small<double>(int, int, const double*, int64_t, int64_t, double*, int64_t, double*, int64_t, int64_t,
                                 int*, cudaStream_t);

}  // namespace ccab
