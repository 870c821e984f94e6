// CCAR3 on the device (see ccab_ccar3_admm / ccab_row_norm4_sum in include/ccab200.h).
//
// ccar3_admm_kernel: the reference's row-sparse ADMM (cca_zoo/linear/_ccar3.py:_admm_row_sparse_rrr) in inverse form,
//   B = B0 + rho M (Z - U),   Z_old = Z,   Z = shrink_rows(B + U),   U = U + B - Z,
// with M = (Sx + (rho + eps) I)^-1 and B0 = M Sxy Sy^-1/2 formed once by the caller.  ONE persistent cooperative
// kernel runs every iteration.  Each CTA owns whole rows of B, Z and U (row blocks of 8 nr rows, strided over the
// grid), so the row norms of the group shrink are CTA-local:
//   1. the CTA's rows of M W (W = Z - U of the previous iteration, p x q) on the fp64 tensor pipe (mma.sync m8n8k4
//      f64), 16-wide k slices of M and W double-buffered through shared memory by cp.async;
//   2. the epilogue B = B0 + rho (M W) into a shared tile, then one warp per row: the row norm of B + U, the shrink,
//      the new Z, U and W = Z - U, and the squared residuals ||Z - B||^2, ||Z_old - Z||^2 of the row;
//   3. each CTA writes its two residual sums to its slot; ONE grid barrier; every CTA adds the slots in slot order
//      (so every CTA takes the same stop decision) and leaves the loop when max(primal, dual) < tol.
// W is double-buffered across iterations (read W[it & 1], write W[(it + 1) & 1]), as are the residual slots, so the
// single barrier per iteration is the only synchronisation.  Every sum has a fixed order: reruns are bit-identical.
//
// Traffic per iteration: every active CTA reads all of W (p x q_pad doubles) and its rows of M from L2, i.e.
// G * 8 p q_pad + 8 p^2 bytes for G active CTAs, and writes its rows of Z, U and W.  The fragment registers limit a
// CTA to 8 x 8 fragments per warp of one row block: q <= 512 (kCcar3MaxQ).
//
// row_norm4_kernel: sum_s ||y_s - mean||^4 in float64 over a float32 / float64 view with any row stride, one warp per
// row, a grid fixed by n alone, and the per-block sums added in block order by a second single-block launch.
#include "ccar3.cuh"

#include <cooperative_groups.h>

#include <algorithm>

#include "common.cuh"

namespace ccab {
namespace cg = cooperative_groups;

namespace {

constexpr int kThreads = 256;
constexpr int kWarps = kThreads / 32;
constexpr int KC = 16;  // k slice of the product

struct AdmmArgs {
  int p, q, qp, nr, nblk, max_iter;
  const double* M;
  int64_t ldm;
  const double* B0;
  int64_t ldb;
  double kappa, rho, tol;
  double* Z;
  int64_t ldz;
  double* U;
  int64_t ldu;
  double* W;     // two p x qp buffers (columns q .. qp zero)
  double* part;  // two buffers of kCcar3MaxGrid (primal^2, dual^2) slots
  double* info;
};

__device__ __forceinline__ void ccar3_dmma_884(double& c0, double& c1, double a, double b) {
  asm volatile("mma.sync.aligned.m8n8k4.row.col.f64.f64.f64.f64 {%0, %1}, {%2}, {%3}, {%0, %1};"
               : "+d"(c0), "+d"(c1)
               : "d"(a), "d"(b));
}

// 8-byte copy global -> shared through L1 (M never changes); src_bytes = 0 writes a zero
__device__ __forceinline__ void cp_async8(void* dst, const void* src, int src_bytes) {
  asm volatile("cp.async.ca.shared.global [%0], [%1], 8, %2;" ::"r"(smem_u32(dst)), "l"(src), "r"(src_bytes)
               : "memory");
}
// 16-byte copy global -> shared bypassing L1 (W is rewritten by other CTAs every iteration)
__device__ __forceinline__ void cp_async16_cg(void* dst, const void* src, int src_bytes) {
  asm volatile("cp.async.cg.shared.global [%0], [%1], 16, %2;" ::"r"(smem_u32(dst)), "l"(src), "r"(src_bytes)
               : "memory");
}
__device__ __forceinline__ void cp_async_commit() { asm volatile("cp.async.commit_group;" ::: "memory"); }
template <int N>
__device__ __forceinline__ void cp_async_wait() { asm volatile("cp.async.wait_group %0;" ::"n"(N) : "memory"); }

__device__ __forceinline__ double warp_sum(double v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
  return v;
}

// shared memory: the two k-slice stages (M slice as [k][row], W slice as [k][col]), aliased by the epilogue tile
__host__ __device__ inline size_t stage_doubles(int NR, int qp) { return (size_t)2 * KC * ((8 * NR + 4) + (qp + 4)); }
__host__ __device__ inline size_t tile_doubles(int NR, int qp) { return (size_t)8 * NR * (qp + 2); }

template <int NR, int NJ>
__global__ void __launch_bounds__(kThreads, 1) ccar3_admm_kernel(const AdmmArgs a) {
  extern __shared__ __align__(16) double smem[];
  __shared__ double red[kWarps][2];
  __shared__ double res[2];
  cg::grid_group grid = cg::this_grid();
  const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
  const int gq = lane >> 2, tq = lane & 3;
  const int qp = a.qp, ldw = qp + 4, ldt = qp + 2, ncb = qp / 8;
  const int rows = 8 * a.nr;
  constexpr int LDM = 8 * NR + 4;
  double* Ms = smem;                          // [2][KC][LDM]
  double* Ws = smem + 2 * KC * LDM;           // [2][KC][ldw]
  double* T = smem;                           // [rows][ldt] (after the product)
  const size_t wsz = (size_t)a.p * qp;

  // Z = U = 0 on the rows this CTA owns (nobody else touches them)
  for (int blk = blockIdx.x; blk < a.nblk; blk += gridDim.x)
    for (int r = warp; r < rows; r += kWarps) {
      const int gr = blk * rows + r;
      if (gr >= a.p) break;
      for (int c = lane; c < a.q; c += 32) {
        a.Z[(int64_t)gr * a.ldz + c] = 0.0;
        a.U[(int64_t)gr * a.ldu + c] = 0.0;
      }
    }

  const int nk = (a.p + KC - 1) / KC;
  double primal = 0.0, dual = 0.0;
  int it = 0;
  bool stop = false;
  while (it < a.max_iter) {
    const double* Wc = a.W + (size_t)(it & 1) * wsz;
    double* Wn = a.W + (size_t)((it + 1) & 1) * wsz;
    double pr_cta = 0.0, du_cta = 0.0;
    for (int blk = blockIdx.x; blk < a.nblk; blk += gridDim.x) {
      const int r0 = blk * rows;
      auto stage = [&](int buf, int k0) {
        double* ms = Ms + buf * KC * LDM;
        for (int idx = tid; idx < rows * KC; idx += kThreads) {
          const int r = idx / KC, k = idx % KC, gr = r0 + r, gk = k0 + k;
          const bool ok = gr < a.p && gk < a.p;
          cp_async8(ms + k * LDM + r, ok ? a.M + (int64_t)gr * a.ldm + gk : a.M, ok ? 8 : 0);
        }
        double* ws = Ws + buf * KC * ldw;
        const int half = qp / 2;
        for (int idx = tid; idx < KC * half; idx += kThreads) {
          const int k = idx / half, c = 2 * (idx % half), gk = k0 + k;
          const bool ok = gk < a.p;
          cp_async16_cg(ws + k * ldw + c, ok ? Wc + (size_t)gk * qp + c : Wc, ok ? 16 : 0);
        }
        cp_async_commit();
      };

      double acc[NR][NJ][2];
#pragma unroll
      for (int i = 0; i < NR; ++i)
#pragma unroll
        for (int j = 0; j < NJ; ++j) acc[i][j][0] = acc[i][j][1] = 0.0;

      stage(0, 0);
      for (int kc = 0; kc < nk; ++kc) {
        if (kc + 1 < nk) {
          stage((kc + 1) & 1, (kc + 1) * KC);
          cp_async_wait<1>();
        } else {
          cp_async_wait<0>();
        }
        __syncthreads();
        const double* ms = Ms + (kc & 1) * KC * LDM;
        const double* ws = Ws + (kc & 1) * KC * ldw;
#pragma unroll
        for (int kk = 0; kk < KC; kk += 4) {
          double fa[NR], fb[NJ];
#pragma unroll
          for (int i = 0; i < NR; ++i) fa[i] = ms[(kk + tq) * LDM + 8 * i + gq];
#pragma unroll
          for (int j = 0; j < NJ; ++j) {
            const int cb = warp + kWarps * j;
            fb[j] = cb < ncb ? ws[(kk + tq) * ldw + 8 * cb + gq] : 0.0;
          }
#pragma unroll
          for (int i = 0; i < NR; ++i)
#pragma unroll
            for (int j = 0; j < NJ; ++j)
              if (i < a.nr && warp + kWarps * j < ncb) ccar3_dmma_884(acc[i][j][0], acc[i][j][1], fa[i], fb[j]);
        }
        __syncthreads();
      }

      // B = B0 + rho (M W) into the tile (the stages are free: the last __syncthreads above)
#pragma unroll
      for (int i = 0; i < NR; ++i)
#pragma unroll
        for (int j = 0; j < NJ; ++j) {
          const int cb = warp + kWarps * j;
          if (i < a.nr && cb < ncb) {
#pragma unroll
            for (int e = 0; e < 2; ++e) {
              const int r = 8 * i + gq, c = 8 * cb + 2 * tq + e, gr = r0 + r;
              if (gr < a.p && c < a.q) T[r * ldt + c] = fma(a.rho, acc[i][j][e], a.B0[(int64_t)gr * a.ldb + c]);
            }
          }
        }
      __syncthreads();

      // one warp per row: the group shrink and the updates of Z, U and W
      double pr = 0.0, du = 0.0;
      for (int r = warp; r < rows; r += kWarps) {
        const int gr = r0 + r;
        if (gr >= a.p) break;
        double* z = a.Z + (int64_t)gr * a.ldz;
        double* u = a.U + (int64_t)gr * a.ldu;
        double* w = Wn + (size_t)gr * qp;
        const double* t = T + r * ldt;
        double ss = 0.0;
        for (int c = lane; c < a.q; c += 32) {
          const double zn = t[c] + u[c];
          ss = fma(zn, zn, ss);
        }
        const double nrm = sqrt(warp_sum(ss));
        const double s = nrm > 0.0 ? fmax(0.0, 1.0 - a.kappa / nrm) : 0.0;
        for (int c = lane; c < a.q; c += 32) {
          const double b = t[c], uo = u[c], zo = z[c];
          const double zn = (b + uo) * s;
          const double un = (uo + b) - zn;
          const double d1 = zn - b, d2 = zo - zn;
          pr = fma(d1, d1, pr);
          du = fma(d2, d2, du);
          z[c] = zn;
          u[c] = un;
          w[c] = zn - un;
        }
      }
      pr = warp_sum(pr);
      du = warp_sum(du);
      if (lane == 0) {
        red[warp][0] = pr;
        red[warp][1] = du;
      }
      __syncthreads();
      if (tid == 0)
        for (int v = 0; v < kWarps; ++v) {
          pr_cta += red[v][0];
          du_cta += red[v][1];
        }
      __syncthreads();
    }
    double* slot = a.part + (size_t)(it & 1) * 2 * kCcar3MaxGrid;
    if (tid == 0) {
      slot[2 * blockIdx.x] = pr_cta;
      slot[2 * blockIdx.x + 1] = du_cta;
    }
    grid.sync();
    if (warp == 0) {
      double s0 = 0.0, s1 = 0.0;
      for (int c = lane; c < (int)gridDim.x; c += 32) {
        s0 += __ldcg(slot + 2 * c);
        s1 += __ldcg(slot + 2 * c + 1);
      }
      s0 = warp_sum(s0);
      s1 = warp_sum(s1);
      if (lane == 0) {
        const double sp = sqrt((double)a.p);
        res[0] = sqrt(s0) / sp;
        res[1] = sqrt(s1) / sp;
      }
    }
    __syncthreads();
    primal = res[0];
    dual = res[1];
    ++it;
    stop = fmax(primal, dual) < a.tol;
    if (stop) break;
  }
  if (blockIdx.x == 0 && tid == 0) {
    a.info[0] = (double)it;
    a.info[1] = primal;
    a.info[2] = dual;
    a.info[3] = stop ? 1.0 : 0.0;
  }
}

template <int NR, int NJ>
int launch_admm(AdmmArgs a, cudaStream_t stream) {
  const void* fn = (const void*)ccar3_admm_kernel<NR, NJ>;
  const size_t smem = sizeof(double) * std::max(stage_doubles(NR, a.qp), tile_doubles(NR, a.qp));
  CCAB_CUDA(cudaFuncSetAttribute(fn, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
  int dev = 0, sms = 0, per_sm = 0;
  CCAB_CUDA(cudaGetDevice(&dev));
  CCAB_CUDA(cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, dev));
  CCAB_CUDA(cudaOccupancyMaxActiveBlocksPerMultiprocessor(&per_sm, fn, kThreads, smem));
  CCAB_CHECK_ARG(per_sm >= 1, "the CCAR3 ADMM kernel cannot be resident on this device");
  const int resident = std::min(per_sm * sms, kCcar3MaxGrid);
  // row blocks of 8 nr rows: at least 32 rows per block (fewer CTAs re-reading W from L2) unless the grid would
  // otherwise need more than one pass over its row blocks
  const int want = (int)ceil_div(a.p, 8 * (int64_t)resident);
  a.nr = std::min(NR, std::max(want, 4));
  a.nblk = (int)ceil_div(a.p, 8 * (int64_t)a.nr);
  const int grid = std::min(a.nblk, resident);
  void* args[] = {&a};
  CCAB_CUDA(cudaLaunchCooperativeKernel(fn, dim3(grid), dim3(kThreads), args, smem, stream));
  count_launches(1);
  return 0;
}

template <typename T>
__global__ void __launch_bounds__(kThreads) row_norm4_kernel(int64_t n, int d, const T* __restrict__ Y, int64_t ldy,
                                                             const double* __restrict__ mean, double* part) {
  __shared__ double red[kWarps];
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  double acc = 0.0;
  for (int64_t r = (int64_t)blockIdx.x * kWarps + warp; r < n; r += (int64_t)gridDim.x * kWarps) {
    const T* y = Y + r * ldy;
    double s = 0.0;
    for (int c = lane; c < d; c += 32) {
      const double v = (double)y[c] - mean[c];
      s = fma(v, v, s);
    }
    s = warp_sum(s);
    acc = fma(s, s, acc);
  }
  if (lane == 0) red[warp] = acc;
  __syncthreads();
  if (threadIdx.x == 0) {
    double t = 0.0;
    for (int v = 0; v < kWarps; ++v) t += red[v];
    part[blockIdx.x] = t;
  }
}

__global__ void __launch_bounds__(32) sum_partials_kernel(const double* __restrict__ part, int nb, double* out) {
  double s = 0.0;
  for (int b = threadIdx.x; b < nb; b += 32) s += part[b];
  s = warp_sum(s);
  if (threadIdx.x == 0) out[0] = s;
}

constexpr int kNorm4MaxBlocks = 1024;

int norm4_blocks(int64_t n) { return (int)std::max<int64_t>(1, std::min<int64_t>(ceil_div(n, kWarps), kNorm4MaxBlocks)); }

}  // namespace

size_t ccar3_admm_workspace_bytes(int p, int q) {
  const int qp = (int)ceil_div(q, 8) * 8;
  return sizeof(double) * ((size_t)2 * p * qp + (size_t)2 * 2 * kCcar3MaxGrid);
}

int ccar3_admm(int p, int q, const double* M, int64_t ldm, const double* B0, int64_t ldb, double kappa, double rho,
               double tol, int max_iter, double* Z, int64_t ldz, double* U, int64_t ldu, double* info, void* ws,
               size_t ws_bytes, cudaStream_t stream) {
  CCAB_CHECK_ARG(ws && ws_bytes >= ccar3_admm_workspace_bytes(p, q), "ccar3_admm: workspace too small");
  CCAB_CHECK_ARG(reinterpret_cast<uintptr_t>(ws) % 16 == 0, "ccar3_admm: workspace not 16-byte aligned");
  AdmmArgs a = {};
  a.p = p;
  a.q = q;
  a.qp = (int)ceil_div(q, 8) * 8;
  a.max_iter = max_iter;
  a.M = M;
  a.ldm = ldm;
  a.B0 = B0;
  a.ldb = ldb;
  a.kappa = kappa;
  a.rho = rho;
  a.tol = tol;
  a.Z = Z;
  a.ldz = ldz;
  a.U = U;
  a.ldu = ldu;
  a.W = static_cast<double*>(ws);
  a.part = a.W + (size_t)2 * p * a.qp;
  a.info = info;
  // W of the first iteration is Z - U = 0; the padding columns stay 0 in both buffers
  CCAB_CUDA(cudaMemsetAsync(a.W, 0, sizeof(double) * (size_t)2 * p * a.qp, stream));
  int rc;
  if (a.qp <= 64)
    rc = launch_admm<8, 1>(a, stream);
  else if (a.qp <= 128)
    rc = launch_admm<8, 2>(a, stream);
  else if (a.qp <= 256)
    rc = launch_admm<8, 4>(a, stream);
  else
    rc = launch_admm<4, 8>(a, stream);
  if (rc) return rc;
  CCAB_CUDA(cudaGetLastError());
  return 0;
}

size_t row_norm4_sum_workspace_bytes(int64_t n) { return sizeof(double) * (size_t)norm4_blocks(n); }

template <typename T>
int row_norm4_sum(int64_t n, int d, const T* Y, int64_t ldy, const double* mean, double* out, void* ws,
                  size_t ws_bytes, cudaStream_t stream) {
  CCAB_CHECK_ARG(ws && ws_bytes >= row_norm4_sum_workspace_bytes(n), "row_norm4_sum: workspace too small");
  const int nb = norm4_blocks(n);
  double* part = static_cast<double*>(ws);
  row_norm4_kernel<T><<<nb, kThreads, 0, stream>>>(n, d, Y, ldy, mean, part);
  sum_partials_kernel<<<1, 32, 0, stream>>>(part, nb, out);
  count_launches(2);
  CCAB_CUDA(cudaGetLastError());
  return 0;
}
template int row_norm4_sum<float>(int64_t, int, const float*, int64_t, const double*, double*, void*, size_t,
                                  cudaStream_t);
template int row_norm4_sum<double>(int64_t, int, const double*, int64_t, const double*, double*, void*, size_t,
                                   cudaStream_t);

}  // namespace ccab
