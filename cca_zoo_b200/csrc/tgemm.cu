// tgemm: C = alpha * op(A) * op(B) + beta * C in fp32-grade arithmetic on the Hopper tensor cores (wgmma, 3xTF32).
//
// The solver stage after K1 (Cholesky panels and trailing updates, L^-1 assembly, T = L1^-1 C12 L2^-T, the
// subspace iteration, the back-substitution of the weights, the tall products of the deep-CCA backward) is a
// chain of small and medium GEMMs.  This kernel puts them on the tensor pipe with the machinery of K1:
//
//   * operands straight from row-major storage, both majors: wgmma reads TF32 operands only K-major, so the
//     256 threads of the CTA stage each 32-index slice of op(A) and op(B) into K-major 128-byte swizzled shared
//     tiles (TileStager: float4 loads along a contiguous reduction index, a transposing store otherwise), and all
//     four op() combinations of ccab_gemm share one mainloop without any transposed copy in global memory;
//   * 3xTF32 with the split formed while staging: hi = truncated fp32, lo = rna_tf32(x - hi), three wgmmas per
//     k-step (lo*hi, hi*lo, hi*hi); double-buffered, the global loads of the next slice in flight during the MMAs;
//   * 128 x BN output tiles, two warpgroups of 64 rows each; the fp32 register accumulator of the tensor cores is
//     added into a second register set after every slice (round-to-nearest adds), which keeps a K = 512 product at
//     fp32 grade;
//   * batched through blockIdx.z.
//
// Out-of-range rows / columns / reduction indices are staged as zeros, so no shape needs padding.
// Replaces the FMA products behind cca_zoo/linear/_rcca.py:96,100, cca_zoo/linear/_mcca.py:131 and
// cca_zoo/deep/objectives.py:97 (and the LAPACK level-3 calls inside scipy.linalg.eigh / numpy.linalg.svd).
#include "tgemm.cuh"

namespace ccab {
namespace {

constexpr int kTgThreads = 256;
constexpr int kBM = 128;
constexpr int kKC = 32;       // reduction indices per slice = one 128-byte K-major row
constexpr int kRun = 1;       // slices per accumulator run (32 reduction indices)

struct TgParams {
  const float* A;
  const float* B;
  long long lda, strideA, strideA2, ldb, strideB, strideB2;
  float* C;
  long long ldc, strideC, strideC2;
  float* Ct;
  long long ldct, strideCt, strideCt2;
  int batch1;  // blockIdx.z = b2 * batch1 + b1
  int M, N, K;
  float alpha, beta;
  int lower_only;
  int vec_c;  // rows of C can be read / written as float4
};

template <int BN>
struct TgCfg {
  static constexpr int kATile = kBM * kKC * 4;
  static constexpr int kBTile = BN * kKC * 4;
  static constexpr int kStage = 2 * (kATile + kBTile);  // A hi, A lo, B hi, B lo
  static constexpr int kSmem = 2 * kStage + 1024;
};

template <bool AK, bool BK, int BN>
__global__ void __launch_bounds__(kTgThreads, 1) tgemm_kernel(const __grid_constant__ TgParams p) {
  using Cfg = TgCfg<BN>;
  constexpr int R = BN / 2;   // accumulator registers per thread
  const int m0 = blockIdx.y * kBM, n0 = blockIdx.x * BN;
  const int bz = (int)blockIdx.z % p.batch1, bz2 = (int)blockIdx.z / p.batch1;
  if (p.lower_only && n0 >= m0 + kBM) return;

  extern __shared__ uint8_t smem_raw[];
  uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~uintptr_t(1023));

  // op(A) row m, reduction index k: A[m * lda + k] (AK) or A[k * lda + m]; op(B)^T row n likewise with BK
  const float* Ab = p.A + (size_t)bz * p.strideA + (size_t)bz2 * p.strideA2 + (AK ? (size_t)m0 * p.lda : (size_t)m0);
  const float* Bb = p.B + (size_t)bz * p.strideB + (size_t)bz2 * p.strideB2 + (BK ? (size_t)n0 * p.ldb : (size_t)n0);
  const int nch = (p.K + kKC - 1) / kKC;
  TileStager<AK, kBM> sa;
  TileStager<BK, BN> sb;
  auto load = [&](int c) {
    const int k0 = c * kKC, ks = min(kKC, p.K - k0);
    sa.load(Ab + (AK ? (size_t)k0 : (size_t)k0 * p.lda), p.lda, p.M - m0, ks, true);
    sb.load(Bb + (BK ? (size_t)k0 : (size_t)k0 * p.ldb), p.ldb, p.N - n0, ks, true);
  };
  auto store = [&](int buf) {
    uint8_t* st = smem + buf * Cfg::kStage;
    sa.template store<true>(st, st + Cfg::kATile);
    sb.template store<true>(st + 2 * Cfg::kATile, st + 2 * Cfg::kATile + Cfg::kBTile);
  };

  float acc[R], tot[R];
#pragma unroll
  for (int i = 0; i < R; ++i) acc[i] = tot[i] = 0.f;
  const int wg = threadIdx.x >> 7;
  load(0);
  store(0);
  fence_proxy_async_smem();
  __syncthreads();
  for (int c = 0; c < nch; ++c) {
    const uint32_t st = smem_u32(smem + (c & 1) * Cfg::kStage);
    const uint32_t a0 = st + wg * 64 * 128, b0 = st + 2 * Cfg::kATile;
    wgmma_fence();
#pragma unroll
    for (int kk = 0; kk < kKC / 8; ++kk) {
      const uint64_t a_hi = wgmma_desc_k128(a0 + 32 * kk), a_lo = wgmma_desc_k128(a0 + Cfg::kATile + 32 * kk);
      const uint64_t b_hi = wgmma_desc_k128(b0 + 32 * kk), b_lo = wgmma_desc_k128(b0 + Cfg::kBTile + 32 * kk);
      wgmma_tf32<BN>(acc, a_lo, b_hi);   // small cross terms first
      wgmma_tf32<BN>(acc, a_hi, b_lo);
      wgmma_tf32<BN>(acc, a_hi, b_hi);
    }
    wgmma_commit();
    const bool more = c + 1 < nch;
    if (more) load(c + 1);
    wgmma_wait_all();
    wgmma_fence_regs<R>(acc);
    if (!more || (c + 1) % kRun == 0) {
#pragma unroll
      for (int i = 0; i < R; ++i) {
        tot[i] += acc[i];
        acc[i] = 0.f;
      }
    }
    if (more) store((c + 1) & 1);   // that stage was last read by the wgmmas of slice c - 1, retired before the barrier
    fence_proxy_async_smem();
    __syncthreads();
  }

  // ---- epilogue: fragment element r of a thread is (row lane/4 + 8*((r/2)%2), column 8*(r/4) + 2*(lane%4) + r%2)
  const int warp = (threadIdx.x >> 5) & 3, lane = threadIdx.x & 31;
  float* Cb = p.C ? p.C + (size_t)bz * p.strideC + (size_t)bz2 * p.strideC2 : nullptr;
  float* Ctb = p.Ct ? p.Ct + (size_t)bz * p.strideCt + (size_t)bz2 * p.strideCt2 : nullptr;
#pragma unroll
  for (int r = 0; r < R; r += 2) {
    const int row = m0 + wg * 64 + warp * 16 + (lane >> 2) + 8 * ((r >> 1) & 1);
    const int col = n0 + 8 * (r >> 2) + 2 * (lane & 3);
    if (row >= p.M) continue;
    float v0 = p.alpha * tot[r], v1 = p.alpha * tot[r + 1];
    if (Cb) {
      float* crow = Cb + (size_t)row * p.ldc + col;
      if (p.vec_c && col + 2 <= p.N) {   // col is even and ldc % 4 == 0: an aligned float2
        float2* c2 = reinterpret_cast<float2*>(crow);
        if (p.beta != 0.f) {
          const float2 o = *c2;
          v0 += p.beta * o.x;
          v1 += p.beta * o.y;
        }
        *c2 = make_float2(v0, v1);
      } else {
        if (col < p.N) {
          if (p.beta != 0.f) v0 += p.beta * crow[0];
          crow[0] = v0;
        }
        if (col + 1 < p.N) {
          if (p.beta != 0.f) v1 += p.beta * crow[1];
          crow[1] = v1;
        }
      }
    }
    if (Ctb) {
      if (col < p.N) Ctb[(size_t)col * p.ldct + row] = v0;
      if (col + 1 < p.N) Ctb[(size_t)(col + 1) * p.ldct + row] = v1;
    }
  }
}

template <bool AK, bool BK, int BN>
int launch(const TgParams& prm, dim3 grid, cudaStream_t stream) {
  using Cfg = TgCfg<BN>;
  static bool attr_done[64] = {};   // cudaFuncSetAttribute is per device
  int dev = 0;
  CCAB_CUDA(cudaGetDevice(&dev));
  if (dev < 0 || dev >= 64 || !attr_done[dev]) {
    CCAB_CUDA(cudaFuncSetAttribute(tgemm_kernel<AK, BK, BN>, cudaFuncAttributeMaxDynamicSharedMemorySize, Cfg::kSmem));
    if (dev >= 0 && dev < 64) attr_done[dev] = true;
  }
  tgemm_kernel<AK, BK, BN><<<grid, kTgThreads, Cfg::kSmem, stream>>>(prm);
  count_launches(1);
  CCAB_CUDA(cudaGetLastError());
  return 0;
}

inline bool aligned16(const void* p) { return (reinterpret_cast<uintptr_t>(p) & 15) == 0; }

}  // namespace

bool tgemm_supported(const TgemmArgs& a) {
  if (a.m < 1 || a.n < 1 || a.k < 1 || a.batch < 1) return false;
  if (!a.A || !a.B || !aligned16(a.A) || !aligned16(a.B)) return false;
  if (a.lda % 4 || a.ldb % 4) return false;
  if (a.batch > 1 && (a.strideA % 4 || a.strideB % 4 || a.strideA <= 0 || a.strideB <= 0)) return false;
  if (a.batch2 < 1 || (a.batch2 > 1 && (a.strideA2 % 4 || a.strideB2 % 4 || a.strideA2 <= 0 || a.strideB2 <= 0))) return false;
  return true;
}

int tgemm(const TgemmArgs& a, cudaStream_t stream) {
  CCAB_CHECK_ARG(tgemm_supported(a), "tgemm: operands must be 16-byte aligned with leading dimensions % 4 == 0");
  CCAB_CHECK_ARG(a.C || a.Ct, "tgemm: no output");
  CCAB_CHECK_ARG(a.C || a.beta == 0.f, "tgemm: beta != 0 needs C");
  const bool AK = !a.transa;  // op(A) = A (m x k row-major): reduction index contiguous
  const bool BK = a.transb != 0;  // op(B) = B^T with B stored n x k: reduction index contiguous
  CCAB_CHECK_ARG(a.lda >= (AK ? a.k : a.m) && a.ldb >= (BK ? a.k : a.n), "tgemm: leading dimension too small");
  const int64_t tiles128 = ceil_div(a.m, kBM) * ceil_div(a.n, 128) * a.batch * a.batch2;
  int BN = (a.n > 64 && tiles128 >= 96) ? 128 : 64;
  if (a.force_bn == 64 || a.force_bn == 128) BN = a.force_bn;
  TgParams prm;
  memset(&prm, 0, sizeof(prm));
  prm.A = a.A;
  prm.lda = a.lda;
  prm.strideA = a.strideA;
  prm.strideA2 = a.strideA2;
  prm.B = a.B;
  prm.ldb = a.ldb;
  prm.strideB = a.strideB;
  prm.strideB2 = a.strideB2;
  prm.C = a.C;
  prm.ldc = a.ldc;
  prm.strideC = a.strideC;
  prm.strideC2 = a.strideC2;
  prm.Ct = a.Ct;
  prm.ldct = a.ldct;
  prm.strideCt = a.strideCt;
  prm.strideCt2 = a.strideCt2;
  prm.batch1 = a.batch;
  prm.M = a.m;
  prm.N = a.n;
  prm.K = a.k;
  prm.alpha = a.alpha;
  prm.beta = a.beta;
  prm.lower_only = a.lower_only;
  prm.vec_c = a.C && aligned16(a.C) && a.ldc % 4 == 0 && a.strideC % 4 == 0 && a.strideC2 % 4 == 0;
  dim3 grid((unsigned)ceil_div(a.n, BN), (unsigned)ceil_div(a.m, kBM), (unsigned)(a.batch * a.batch2));
#define CCAB_TG(AK_, BK_)                                                       \
  (BN == 128 ? launch<AK_, BK_, 128>(prm, grid, stream) : launch<AK_, BK_, 64>(prm, grid, stream))
  if (AK && BK) return CCAB_TG(true, true);
  if (AK && !BK) return CCAB_TG(true, false);
  if (!AK && BK) return CCAB_TG(false, true);
  return CCAB_TG(false, false);
#undef CCAB_TG
}

}  // namespace ccab
