// K1: block moments M = X^T X (+ column sums) of the hstacked views, upper block triangle only.
//
//   * moments_wgmma_kernel : Hopper wgmma (TF32, fp32 accumulators in registers), 128 x 128 tiles of the upper
//     block triangle, split over the sample axis.  A producer / consumer pipeline on mbarriers: TMA loads of the raw
//     sample slices, two transpose warpgroups that write them as K-major swizzled shared tiles, two wgmma
//     warpgroups.  Optional 3xTF32 (hi / lo copies in shared memory, 3 MMAs per k-step) for fp32-grade accuracy.
//   * moments_x3b_pair_kernel : the same pipeline for 3xTF32 with the two cross terms as bf16 MMAs (2 instead of 3
//     units of tensor work), on 256 x 128 pair tiles: one transposed B block feeds two A blocks.
//     Column sums are exact fp32 sums of the loaded values.
//   * moments_simt_kernel : exact FMA (fp32) tile kernel, the non-tensor reference path;
//     moments_dmma_kernel : float64 inputs on the fp64 tensor pipe (mma.sync m8n8k4.f64).
//   * reduce / covariance kernels (K2): fixed-order sum of the split partials into a double
//     moment buffer (the all-reduce payload), then C = (M - s s^T / n) / (n - 1).
//
// Replaces, in covariance form, the tall SVDs / np.cov calls of the reference:
//   cca_zoo/_utils/_linalg.py:28, cca_zoo/linear/_rcca.py:96, cca_zoo/linear/_mcca.py:150-152,166,
//   cca_zoo/linear/_gcca.py:101, cca_zoo/deep/objectives.py:83-92.
#include "moments.cuh"

#include <mutex>
#include <type_traits>

namespace ccab {

// =============================================================================================
// layout
// =============================================================================================
int make_layout(int n_views, const int64_t* dims, ColumnLayout* L) {
  CCAB_CHECK_ARG(n_views >= 1 && n_views <= kMaxViews, "n_views must be in [1,%d], got %d", kMaxViews,
                 n_views);
  L->n_views = n_views;
  L->coff[0] = 0;
  L->poff[0] = 0;
  int nb = 0;
  for (int v = 0; v < n_views; ++v) {
    CCAB_CHECK_ARG(dims[v] >= 1 && dims[v] <= kMaxBlocks * kBlk, "bad view width %lld", (long long)dims[v]);
    L->dims[v] = (int)dims[v];
    int b = (int)ceil_div(dims[v], kBlk);
    nb += b;
    L->coff[v + 1] = L->coff[v] + (int)dims[v];
    L->poff[v + 1] = L->poff[v] + b * kBlk;
  }
  CCAB_CHECK_ARG(nb <= kMaxBlocks, "total padded width %d exceeds %d", nb * kBlk, kMaxBlocks * kBlk);
  L->nblocks = nb;
  L->D = L->coff[n_views];
  L->Dp = nb * kBlk;
  return 0;
}

// optional timing of the tensor-core moment kernel alone (bench.py roofline): events on the launching stream
static bool g_prof_on = false;
static cudaEvent_t g_prof_e0 = nullptr, g_prof_e1 = nullptr;
static bool g_prof_valid = false;
void moments_profile_enable(int on) {
  g_prof_on = on != 0;
  g_prof_valid = false;
  if (g_prof_on && !g_prof_e0) {
    cudaEventCreate(&g_prof_e0);
    cudaEventCreate(&g_prof_e1);
  }
}
float moments_profile_last_ms() {
  if (!g_prof_valid) return -1.f;
  float ms = -1.f;
  if (cudaEventSynchronize(g_prof_e1) != cudaSuccess) return -1.f;
  if (cudaEventElapsedTime(&ms, g_prof_e0, g_prof_e1) != cudaSuccess) return -1.f;
  return ms;
}

// =============================================================================================
// wgmma kernel
// =============================================================================================
// One CTA = one 128 x 128 tile (A block bi, B block bj >= bi) of M over one split of the sample axis, taken in 32-sample
// slices by four warpgroups that meet only on mbarriers:
//   * thread 0 issues the TMA loads of the raw row-major [32 samples x 128 columns] slice of each column block, as
//     four [32 x 32] boxes with 128-byte swizzle, into a ring of raw stages (a diagonal tile loads only A).  Rows past
//     n_rows and columns past the view's width arrive as zeros;
//   * warpgroups 0 and 1 transpose the B block of each raw stage into the K-major, 128-byte-swizzled operand tiles
//     wgmma reads from shared memory (the sample index is the strided one of row-major X, and wgmma reads TF32 only
//     K-major): hi, and in 3xTF32 mode lo, in a ring of operand stages.  Thread (h, m) owns column m and the 4-sample
//     groups of parity h.  A diagonal tile transposes its one block, which serves as B, and takes the exact fp32
//     column sums here;
//   * warpgroups 2 and 3 each run the wgmmas of 64 rows of the tile, three k-steps of MMAs in flight while the
//     fragments of the next are loaded.  They load their A fragments straight from the raw stage into registers
//     (registers have no major-ness requirement) and split hi / lo there; the 3xTF32 mode issues lo*hi + hi*lo + hi*hi
//     per k-step.
// Per 3xTF32 slice of an off-diagonal tile the mainloop moves about 192 KB through shared memory: 32 KB of TMA writes,
// 16 KB of transpose reads, 32 KB of hi / lo stores of B, 16 KB of A fragment loads and 96 KB of wgmma B reads.
// The swizzle makes the raw reads conflict-free for both readers: a transpose warp reads one 128-byte box row, and a
// fragment load takes samples {0,5,2,7} (then {4,1,6,3}) of a k-step on lanes t = lane % 4 = 0..3, so the 32 lanes
// hit 32 distinct banks.
struct WgParams {
  CUtensorMap map[kMaxViews];   // view v: {width, rows} fp32, row pitch lds[v], box 32 columns x 32 rows, 128B swizzle
  uint8_t blk_view[kMaxBlocks];
  int blk_col0[kMaxBlocks];
  float* partial;      // [S][Dp][Dp]
  float* partial_sum;  // [S][Dp]
  int64_t n_rows, rows_per_split;
  int64_t row_base;    // first row of this pass in the tensor maps
  int nblocks, Dp;
};
static_assert(sizeof(WgParams) <= 4096, "kernel parameter space");

constexpr int kWgXpose = 256;              // two transpose warpgroups
constexpr int kWgThreads = kWgXpose + 256;  // + two MMA warpgroups
constexpr int kWgKC = 32;                  // samples per slice = one 128-byte K-major row
constexpr int kWgTile = kBlk * kWgKC * 4;  // bytes of one 128 x 32 fp32 tile (raw column block or operand copy)
constexpr int kWgBox = 32 * kWgKC * 4;     // bytes of one [32 samples x 32 columns] TMA box

// Byte offset of element (sample k, column m) in the raw slice of a column block: box m / 32, swizzled as TMA stores it
__device__ __forceinline__ uint32_t raw_offset(int k, int m) {
  return (uint32_t)(m >> 5) * kWgBox + k128_offset(k, (m & 31) >> 2) + (uint32_t)(m & 3) * 4;
}

// Operand arithmetic of moments_wgmma_kernel: one TF32 pass, 3xTF32
enum class K1Mode { TF32, X3 };

template <K1Mode M>
struct WgCfg {
  static constexpr int kOps = M == K1Mode::TF32 ? 1 : 2;   // B operand tiles: hi (+ lo)
  static constexpr int kOpStage = kOps * kWgTile;
  static constexpr int kRawStage = 2 * kWgTile;    // raw A block, raw B block
  static constexpr int kOpStages = M == K1Mode::TF32 ? 3 : 2;
  // a raw stage is held until the MMA warps have loaded its A fragments, up to kOpStages slices after its transpose
  static constexpr int kRawStages = 5;
  static constexpr int kBarOff = kOpStages * kOpStage + kRawStages * kRawStage;
  static constexpr int kSumOff = kBarOff + 2 * (kOpStages + kRawStages) * 8;       // odd column sums
  static constexpr int kSmem = kSumOff + kBlk * 4 + 1024;   // + alignment slack
};
static_assert(WgCfg<K1Mode::X3>::kSmem <= 227 * 1024 && WgCfg<K1Mode::TF32>::kSmem <= 227 * 1024,
              "shared memory per block");
static_assert(WgCfg<K1Mode::X3>::kRawStages > WgCfg<K1Mode::X3>::kOpStages &&
              WgCfg<K1Mode::TF32>::kRawStages > WgCfg<K1Mode::TF32>::kOpStages,
              "the refill of a raw stage must not wait on the MMA warps' current slice");

template <K1Mode M>
__global__ void __launch_bounds__(kWgThreads, 1) moments_wgmma_kernel(const __grid_constant__ WgParams p) {
  using Cfg = WgCfg<M>;
  constexpr bool X3 = M == K1Mode::X3;
  constexpr int NO = Cfg::kOpStages, NR = Cfg::kRawStages;
  extern __shared__ uint8_t smem_raw[];
  // offset (not an integer round trip) so that the compiler still sees shared-memory pointers: LDS / STS, not LD / ST
  uint8_t* smem = smem_raw + ((1024u - (smem_u32(smem_raw) & 1023u)) & 1023u);
  uint8_t* ops = smem;                          // operand stages (1024-byte aligned: swizzle atoms)
  uint8_t* raw = smem + NO * Cfg::kOpStage;     // raw stages
  uint64_t* raw_full = reinterpret_cast<uint64_t*>(smem + Cfg::kBarOff);
  uint64_t* raw_empty = raw_full + NR;
  uint64_t* op_full = raw_empty + NR;
  uint64_t* op_empty = op_full + NO;

  int t = blockIdx.x, bi = 0, rowlen = p.nblocks;   // tile decode over the upper block triangle
  while (t >= rowlen) { t -= rowlen; ++bi; --rowlen; }
  const int bj = bi + t;
  const bool diag = bi == bj;
  const int split = blockIdx.y;
  const int64_t r0 = (int64_t)split * p.rows_per_split;
  const int64_t r1 = min(r0 + p.rows_per_split, p.n_rows);
  const int nch = r1 > r0 ? (int)((r1 - r0 + kWgKC - 1) / kWgKC) : 0;

  if (threadIdx.x == 0) {
    for (int s = 0; s < NR; ++s) {
      mbar_init(&raw_full[s], 1);
      mbar_init(&raw_empty[s], kWgXpose + 8);   // every transpose thread and one lane of each MMA warp
    }
    for (int s = 0; s < NO; ++s) {
      mbar_init(&op_full[s], kWgXpose);
      mbar_init(&op_empty[s], 8);       // one lane of each MMA warp
    }
    fence_mbar_init();
  }
  __syncthreads();

  if (threadIdx.x < kWgXpose) {
    // ---- TMA issue (thread 0) and transpose warpgroups ----
    setmaxnreg_dec<80>();
    const int m = threadIdx.x % kBlk, h = threadIdx.x / kBlk;   // column, parity of its 4-sample groups
    const CUtensorMap* mapA = &p.map[p.blk_view[bi]];
    const CUtensorMap* mapB = &p.map[p.blk_view[bj]];
    const int colA = p.blk_col0[bi], colB = p.blk_col0[bj];
    auto issue = [&](int c) {
      const int s = c % NR;
      const int row = (int)(p.row_base + r0 + (int64_t)c * kWgKC);
      uint8_t* dst = raw + s * Cfg::kRawStage;
      mbar_arrive_expect_tx(&raw_full[s], diag ? kWgTile : 2 * kWgTile);
#pragma unroll
      for (int q = 0; q < kBlk / 32; ++q) {
        tma_load_2d(dst + q * kWgBox, mapA, &raw_full[s], colA + 32 * q, row);
        if (!diag) tma_load_2d(dst + kWgTile + q * kWgBox, mapB, &raw_full[s], colB + 32 * q, row);
      }
    };
    if (threadIdx.x == 0)
      for (int c = 0; c < min(NR, nch); ++c) issue(c);

    float csum = 0.f;   // column m of a diagonal tile over the 4-sample groups of parity h
    auto transpose = [&](const uint8_t* src, uint8_t* hi, uint8_t* lo, bool sums) {
#pragma unroll
      for (int j = 0; j < kWgKC / 8; ++j) {
        const int kg = 2 * j + h;
        float v[4];
#pragma unroll
        for (int e = 0; e < 4; ++e)   // a warp reads one 128-byte box row: conflict-free
          v[e] = *reinterpret_cast<const float*>(src + raw_offset(4 * kg + e, m));
        const uint32_t off = k128_offset(m, kg);
        *reinterpret_cast<float4*>(hi + off) = make_float4(tf32_hi(v[0]), tf32_hi(v[1]), tf32_hi(v[2]), tf32_hi(v[3]));
        if (X3)
          *reinterpret_cast<float4*>(lo + off) = make_float4(tf32_residual(v[0]), tf32_residual(v[1]),
                                                             tf32_residual(v[2]), tf32_residual(v[3]));
        if (sums) csum += (v[0] + v[1]) + (v[2] + v[3]);
      }
    };
    for (int c = 0; c < nch; ++c) {
      const int sr = c % NR, so = c % NO;
      mbar_wait(&raw_full[sr], (c / NR) & 1);
      mbar_wait(&op_empty[so], ((c / NO) & 1) ^ 1);   // the MMAs of slice c - NO have retired
      uint8_t* dst = ops + so * Cfg::kOpStage;
      transpose(raw + sr * Cfg::kRawStage + (diag ? 0 : kWgTile), dst, dst + kWgTile, diag);
      fence_proxy_async_smem();   // the generic-proxy stores become visible to wgmma (async proxy)
      mbar_arrive(&raw_empty[sr]);
      mbar_arrive(&op_full[so]);
      // Refill the raw stage of slice c - NO + 1: the MMA warps hand back slice c - NO (seen above) as they load the
      // last A fragments of slice c - NO + 1, so this wait is short and does not hold the transpose back behind them.
      const int rf = c + NR - NO + 1;
      if (threadIdx.x == 0 && rf >= NR && rf < nch) {
        mbar_wait(&raw_empty[rf % NR], (rf / NR - 1) & 1);
        issue(rf);
      }
    }
    if (diag) {   // even + odd groups
      float* odd = reinterpret_cast<float*>(smem + Cfg::kSumOff);
      if (h) odd[m] = csum;
      asm volatile("bar.sync 1, %0;" ::"n"(kWgXpose) : "memory");
      if (!h) p.partial_sum[(size_t)split * p.Dp + bi * kBlk + m] = csum + odd[m];
    }
  } else {
    // ---- MMA warpgroups ----
    setmaxnreg_inc<168>();
    const int wg = (threadIdx.x - kWgXpose) >> 7, lane = threadIdx.x & 31, t = lane & 3;
    // Raw-stage offsets of this thread's A fragment elements in k-step 0 (k-step kk adds kk * 1024): rows m and m + 8
    // of the tile, and the two samples of lane t, t and t + 4.  The first load takes sample kx, the second kx ^ 4, so
    // that the lanes of one load hit distinct swizzle chunks; odd t gets its samples in the swapped order.
    const int m = wg * 64 + ((threadIdx.x >> 5) & 3) * 16 + (lane >> 2);
    const int kx = t ^ ((t & 1) << 2);
    const bool swap = t & 1;
    const uint32_t o00 = raw_offset(kx, m), o01 = raw_offset(kx ^ 4, m);
    const uint32_t o10 = raw_offset(kx, m + 8), o11 = raw_offset(kx ^ 4, m + 8);
    float acc[64];
#pragma unroll
    for (int i = 0; i < 64; ++i) acc[i] = 0.f;
    wgmma_fence_regs<64>(acc);   // keeps the zeroing out of the wgmma pipeline (else ptxas serialises the wgmmas)
    // One wgmma group per step, so that the fragment registers of a step are free once its group of the previous
    // slice has retired.  A step is one k-step of 8 samples: a ring of four k-step fragments, 32 registers in 3xTF32
    // mode, with three groups in flight while the next fragments are loaded.  (Two whole-slice fragment sets do not fit
    // next to the accumulators in the 128 registers a 512-thread CTA compiles to.)
    constexpr int KS = kWgKC / 8;          // steps per slice
    constexpr int KR = Cfg::kOps * 4;      // fragment registers per step: 0..3 TF32 hi, 4..7 TF32 lo
    uint32_t fa[KS][KR] = {};
    for (int c = 0; c < nch; ++c) {
      const int sr = c % NR, so = c % NO;
      mbar_wait(&raw_full[sr], (c / NR) & 1);
      const uint8_t* a_src = raw + sr * Cfg::kRawStage;   // the A block (a diagonal tile's only block)
      const uint32_t b0 = smem_u32(ops + so * Cfg::kOpStage);
#pragma unroll
      for (int kk = 0; kk < KS; ++kk) {
        wgmma_wait<KS - 1>();   // step kk of slice c - 1 has retired: its fragment registers may be rewritten
        // ... and not before: keeping them live up to here makes ptxas give each step registers of its own (else it
        // may reuse one set and serialise the wgmmas)
        wgmma_fence_regs<KR>(fa[kk]);
        // the last step of slice c - 1 has retired with it: hand that slice's operand stage back
        if (kk == KS - 1 && c > 0 && lane == 0) mbar_arrive(&op_empty[(c - 1) % NO]);
        {
          const uint8_t* s = a_src + kk * 1024;
          const float v00 = *reinterpret_cast<const float*>(s + o00), v01 = *reinterpret_cast<const float*>(s + o01);
          const float v10 = *reinterpret_cast<const float*>(s + o10), v11 = *reinterpret_cast<const float*>(s + o11);
          const float a[4] = {swap ? v01 : v00, swap ? v11 : v10, swap ? v00 : v01, swap ? v10 : v11};
#pragma unroll
          for (int i = 0; i < 4; ++i) {
            fa[kk][i] = __float_as_uint(tf32_hi(a[i]));
            if constexpr (X3) fa[kk][4 + i] = __float_as_uint(tf32_residual(a[i]));
          }
        }
        wgmma_fence_regs<KR>(fa[kk]);
        if (kk == KS - 1) {
          __syncwarp();
          if (lane == 0) mbar_arrive(&raw_empty[sr]);   // every lane of the warp has read the slice's A fragments
        }
        if (kk == 0) mbar_wait(&op_full[so], (c / NO) & 1);
        wgmma_fence();
        const uint64_t b_hi = wgmma_desc_k128(b0 + 32 * kk);
        if constexpr (X3) {
          const uint64_t b_lo = wgmma_desc_k128(b0 + kWgTile + 32 * kk);
          wgmma_tf32_ra<128>(acc, &fa[kk][4], b_hi);   // small cross terms first
          wgmma_tf32_ra<128>(acc, &fa[kk][0], b_lo);
        }
        wgmma_tf32_ra<128>(acc, &fa[kk][0], b_hi);
        wgmma_commit();
      }
    }
    wgmma_wait_all();
    wgmma_fence_regs<64>(acc);

    // ---- epilogue: fragments -> partial slab of this split ----
    const int warp = (threadIdx.x >> 5) & 3;
    float* P = p.partial + (size_t)split * p.Dp * p.Dp;
    const int row0 = bi * kBlk + wg * 64 + warp * 16 + (lane >> 2);
    const int col0 = bj * kBlk + 2 * (lane & 3);
#pragma unroll
    for (int r = 0; r < 64; r += 2) {
      const int row = row0 + 8 * ((r >> 1) & 1), col = col0 + 8 * (r >> 2);
      *reinterpret_cast<float2*>(P + (size_t)row * p.Dp + col) = make_float2(acc[r], acc[r + 1]);
    }
  }
}

// =============================================================================================
// tf32x3b pair-tile kernel
// =============================================================================================
// 3xTF32 with the cross terms as bf16 MMAs: hi*hi stays a TF32 MMA per k-step of 8 samples, and lo*hi + hi*lo run as
// bf16 m64n128k16 MMAs per k16 step of 16 samples, at twice the TF32 rate.  hi = trunc_tf32(x); the bf16 copies are
// rne_bf16(hi) and rne_bf16(x - hi).  A bf16 k16 step takes its k index in the order of the registers an MMA thread
// already holds for two TF32 k-steps: logical k 2t, 2t+1, 2t+8, 2t+9 of the step are samples t, t+4, 8+t, 12+t.  (Any
// sample permutation leaves X^T X unchanged as long as A and B share it.)  So the bf16 A fragment is packed from the
// TF32 fragment's registers, and chunk e (16 bytes) of a row of the bf16 B tile holds the pairs (8e+t, 8e+t+4),
// t = 0..3.  The bf16 tile is one 128 x 128-byte K-major tile with 128-byte swizzle: hi in bytes 0..63 of a row (k16
// steps 0, 1), lo in bytes 64..127.  An operand stage is the TF32 hi tile and this tile, 32 KB.
//
// One CTA = one pair tile over one split of the sample axis: A blocks 2i and 2i + 1 against a B block j >= 2i, i.e.
// 256 x 128 of M, so that each transposed B slice feeds two A blocks.  Pair i has the tiles j = 2i .. nblocks - 1:
//   * j > 2i + 1 loads A0 | A1 | B (48 KB per raw stage);
//   * j = 2i + 1: B is A1; both A blocks are loaded, the tile holds sub-tiles (2i, 2i+1) and the diagonal (2i+1, 2i+1);
//   * j = 2i: B is A0; only A0 is loaded and only the diagonal (2i, 2i) is computed: sub-tile (2i+1, 2i) lies below
//     the block diagonal, and the second MMA warpgroup idles.  A lone last block (odd nblocks) is this case.
// The tiles with j in {2i, 2i+1} take the exact fp32 column sums of block j, so each block's sums are written once.
// For nblocks = 16 that is 72 pair tiles instead of 136 unit tiles.  Three roles meet only on mbarriers:
//   * thread 0 issues the TMA loads of each slice (as moments_wgmma_kernel) into a ring of raw stages;
//   * one transpose warpgroup, thread m owning column m of B: the K-major TF32 hi tile and the bf16 hi | lo tile;
//   * two MMA warpgroups, warpgroup g owning the 128 rows of A block 2i + g as two m64n128 accumulators (128
//     registers).  A fragments come straight from the raw stage as in moments_wgmma_kernel.  A step is one k16 step
//     of one 64-row group: 2 TF32 + 2 bf16 MMAs in one wgmma group, four steps per slice, a ring of four steps of
//     fragment registers (64) with three groups in flight.  Every output element sees the MMAs of the unit-tile
//     kernel in the same order (per k16 step: lo*hi, hi*lo, hi*hi of its two k-steps), over the same 2048-sample
//     accumulator runs, so the partials are bit for bit those of 128 x 128 tiles.
// Per slice of a j > 2i + 1 tile (two unit tiles of MMA work, 2048 tensor clocks) the shared-memory traffic is about
// 48 KB TMA, 16 KB transpose reads, 32 KB stores, 32 KB A fragments and 128 KB B reads: 128 KB per unit tile instead
// of 160 KB.
// At config 2 on an H100 the loads bind it, not shared memory: alone they take 80 % of the MMA time (9.8 GB from L2),
// and they overlap with the MMAs only in part (DESIGN.md §4).
constexpr int kPrXpose = 128;                  // one transpose warpgroup (its thread 0 issues the TMA loads)
constexpr int kPrThreads = kPrXpose + 256;     // + two MMA warpgroups
struct PairCfg {
  static constexpr int kOpStage = 2 * kWgTile;    // TF32 hi tile | bf16 hi | lo tile
  static constexpr int kRawStage = 3 * kWgTile;   // raw A0 | A1 | B
  static constexpr int kOpStages = 2;
  static constexpr int kRawStages = 3;
  static constexpr int kFrag = 4;                 // steps of A fragment registers
  static constexpr int kBarOff = kOpStages * kOpStage + kRawStages * kRawStage;
  static constexpr int kSmem = kBarOff + 2 * (kOpStages + kRawStages) * 8 + 1024;   // + alignment slack
  // registers: 128 x 56 + 256 x 224 = 384 x 168, what the CTA is allocated at launch
  static constexpr int kXposeRegs = 56, kMmaRegs = 224;
};
static_assert(PairCfg::kSmem <= 227 * 1024, "shared memory per block");
static_assert(PairCfg::kRawStages > PairCfg::kOpStages,
              "the refill of a raw stage must not wait on the MMA warps' current slice");
static_assert(kPrXpose * PairCfg::kXposeRegs + 256 * PairCfg::kMmaRegs <= kPrThreads * (65536 / kPrThreads / 8 * 8),
              "the register budgets must fit in what the CTA is allocated at launch");
static_assert(4 % PairCfg::kFrag == 0, "a slice is four steps");

// pair tiles of the upper block triangle of nblocks blocks: sum over i of nblocks - 2i
inline int pair_tiles(int nblocks) {
  int n = 0;
  for (int i = 0; 2 * i < nblocks; ++i) n += nblocks - 2 * i;
  return n;
}

__global__ void __launch_bounds__(kPrThreads, 1) moments_x3b_pair_kernel(const __grid_constant__ WgParams p) {
  constexpr int NO = PairCfg::kOpStages, NR = PairCfg::kRawStages, NF = PairCfg::kFrag;
  extern __shared__ uint8_t smem_raw[];
  uint8_t* smem = smem_raw + ((1024u - (smem_u32(smem_raw) & 1023u)) & 1023u);
  uint8_t* ops = smem;                              // operand stages (1024-byte aligned: swizzle atoms)
  uint8_t* raw = smem + NO * PairCfg::kOpStage;     // raw stages
  uint64_t* raw_full = reinterpret_cast<uint64_t*>(smem + PairCfg::kBarOff);
  uint64_t* raw_empty = raw_full + NR;
  uint64_t* op_full = raw_empty + NR;
  uint64_t* op_empty = op_full + NO;

  int t = blockIdx.x, i = 0, rowlen = p.nblocks;   // pair tile decode
  while (t >= rowlen) { t -= rowlen; ++i; rowlen -= 2; }
  const int a0 = 2 * i, bj = a0 + t;
  const int nload = min(t, 2) + 1;   // raw blocks per slice: A0 (j = 2i); A0, A1 (j = 2i + 1); A0, A1, B
  const int na = min(nload, 2);      // A blocks with work, one MMA warpgroup each
  const int bslot = nload - 1;       // where B sits in the raw stage
  const bool diag = t < 2;           // B is an A block: its column sums
  const int split = blockIdx.y;
  const int64_t r0 = (int64_t)split * p.rows_per_split;
  const int64_t r1 = min(r0 + p.rows_per_split, p.n_rows);
  const int nch = r1 > r0 ? (int)((r1 - r0 + kWgKC - 1) / kWgKC) : 0;

  if (threadIdx.x == 0) {
    for (int s = 0; s < NR; ++s) {
      mbar_init(&raw_full[s], 1);
      mbar_init(&raw_empty[s], kPrXpose + 4 * na);   // every transpose thread and one lane of each working MMA warp
    }
    for (int s = 0; s < NO; ++s) {
      mbar_init(&op_full[s], kPrXpose);
      mbar_init(&op_empty[s], 4 * na);
    }
    fence_mbar_init();
  }
  __syncthreads();

  if (threadIdx.x < kPrXpose) {
    // ---- TMA issue (thread 0) and the transpose warpgroup ----
    setmaxnreg_dec<PairCfg::kXposeRegs>();
    const int m = threadIdx.x;   // column of B
    auto issue = [&](int c) {
      const int s = c % NR;
      const int row = (int)(p.row_base + r0 + (int64_t)c * kWgKC);
      uint8_t* dst = raw + s * PairCfg::kRawStage;
      mbar_arrive_expect_tx(&raw_full[s], nload * kWgTile);
      for (int b = 0; b < nload; ++b) {
        const int blk = b < 2 ? a0 + b : bj;
        const CUtensorMap* map = &p.map[p.blk_view[blk]];
#pragma unroll
        for (int q = 0; q < kBlk / 32; ++q)
          tma_load_2d(dst + b * kWgTile + q * kWgBox, map, &raw_full[s], p.blk_col0[blk] + 32 * q, row);
      }
    };
    if (threadIdx.x == 0)
      for (int c = 0; c < min(NR, nch); ++c) issue(c);

    // column m of a diagonal tile over k16 steps 0 and 1 of each slice, added at the end (as two transpose threads
    // of a unit tile sum them)
    float csum[2] = {0.f, 0.f};
    for (int c = 0; c < nch; ++c) {
      const int sr = c % NR, so = c % NO;
      mbar_wait(&raw_full[sr], (c / NR) & 1);
      mbar_wait(&op_empty[so], ((c / NO) & 1) ^ 1);   // the MMAs of slice c - NO have retired
      const uint8_t* src = raw + sr * PairCfg::kRawStage + bslot * kWgTile;
      uint8_t* hi = ops + so * PairCfg::kOpStage;
      uint8_t* lo = hi + kWgTile;   // the bf16 tile: hi | lo pairs of k-step e in chunks e | 4 + e
#pragma unroll
      for (int e = 0; e < 4; ++e) {   // k-step of 8 samples
        float v[8], x[8];
#pragma unroll
        for (int k = 0; k < 8; ++k) {   // a warp reads one 128-byte box row: conflict-free
          v[k] = *reinterpret_cast<const float*>(src + raw_offset(8 * e + k, m));
          x[k] = tf32_hi(v[k]);
        }
        *reinterpret_cast<float4*>(hi + k128_offset(m, 2 * e)) = make_float4(x[0], x[1], x[2], x[3]);
        *reinterpret_cast<float4*>(hi + k128_offset(m, 2 * e + 1)) = make_float4(x[4], x[5], x[6], x[7]);
        *reinterpret_cast<uint4*>(lo + k128_offset(m, e)) =
            make_uint4(pack_bf16x2(x[0], x[4]), pack_bf16x2(x[1], x[5]), pack_bf16x2(x[2], x[6]),
                       pack_bf16x2(x[3], x[7]));
        *reinterpret_cast<uint4*>(lo + k128_offset(m, 4 + e)) =
            make_uint4(pack_bf16x2(v[0] - x[0], v[4] - x[4]), pack_bf16x2(v[1] - x[1], v[5] - x[5]),
                       pack_bf16x2(v[2] - x[2], v[6] - x[6]), pack_bf16x2(v[3] - x[3], v[7] - x[7]));
        if (diag) csum[e >> 1] += ((v[0] + v[1]) + (v[2] + v[3])) + ((v[4] + v[5]) + (v[6] + v[7]));
      }
      fence_proxy_async_smem();   // the generic-proxy stores become visible to wgmma (async proxy)
      mbar_arrive(&raw_empty[sr]);
      mbar_arrive(&op_full[so]);
      // Refill the raw stage of slice c - NO + 1: the MMA warps hand it back as they load its last A fragments, about
      // when they hand back the operand stage of slice c - NO (seen above), so this wait is short.
      const int rf = c + NR - NO + 1;
      if (threadIdx.x == 0 && rf >= NR && rf < nch) {
        mbar_wait(&raw_empty[rf % NR], (rf / NR - 1) & 1);
        issue(rf);
      }
    }
    if (diag) p.partial_sum[(size_t)split * p.Dp + bj * kBlk + m] = csum[0] + csum[1];
  } else {
    // ---- MMA warpgroups ----
    setmaxnreg_inc<PairCfg::kMmaRegs>();
    const int g = (threadIdx.x - kPrXpose) >> 7;   // A block a0 + g
    if (g >= na) return;                          // sub-tile below the block diagonal
    const int lane = threadIdx.x & 31, t4 = lane & 3, warp = (threadIdx.x >> 5) & 3;
    // Raw-stage offsets of this thread's A fragment elements in k-step 0 of row group 0, as in moments_wgmma_kernel
    // (k-step kk adds kk * 1024, row group 1 (rows + 64) two boxes)
    const int m = warp * 16 + (lane >> 2);
    const int kx = t4 ^ ((t4 & 1) << 2);
    const bool swap = t4 & 1;
    const uint32_t o00 = raw_offset(kx, m), o01 = raw_offset(kx ^ 4, m);
    const uint32_t o10 = raw_offset(kx, m + 8), o11 = raw_offset(kx ^ 4, m + 8);
    float acc[2][64];
#pragma unroll
    for (int r = 0; r < 2; ++r) {
#pragma unroll
      for (int k = 0; k < 64; ++k) acc[r][k] = 0.f;
      wgmma_fence_regs<64>(acc[r]);   // keeps the zeroing out of the wgmma pipeline
    }
    // fragment registers of a step: 0..3 and 4..7 TF32 hi of its two k-steps, 8..11 bf16 hi, 12..15 bf16 lo
    uint32_t fa[NF][16] = {};
    for (int c = 0; c < nch; ++c) {
      const int sr = c % NR, so = c % NO;
      mbar_wait(&raw_full[sr], (c / NR) & 1);
      const uint8_t* a_src = raw + sr * PairCfg::kRawStage + g * kWgTile;
      const uint32_t b0 = smem_u32(ops + so * PairCfg::kOpStage);
#pragma unroll
      for (int s = 0; s < 4; ++s) {   // step s: k16 step kk of row group r
        const int kk = s >> 1, r = s & 1, f = s % NF;
        wgmma_wait<NF - 1>();   // the group that last read fa[f] has retired
        wgmma_fence_regs<16>(fa[f]);
        // ... and with it the last step of slice c - 1: hand that slice's operand stage back
        if (s == NF - 1 && c > 0 && lane == 0) mbar_arrive(&op_empty[(c - 1) % NO]);
#pragma unroll
        for (int q = 0; q < 2; ++q) {
          const uint8_t* src = a_src + (2 * kk + q) * 1024 + r * 2 * kWgBox;
          const float v00 = *reinterpret_cast<const float*>(src + o00), v01 = *reinterpret_cast<const float*>(src + o01);
          const float v10 = *reinterpret_cast<const float*>(src + o10), v11 = *reinterpret_cast<const float*>(src + o11);
          const float a[4] = {swap ? v01 : v00, swap ? v11 : v10, swap ? v00 : v01, swap ? v10 : v11};
          float x[4];
#pragma unroll
          for (int k = 0; k < 4; ++k) {
            x[k] = tf32_hi(a[k]);
            fa[f][4 * q + k] = __float_as_uint(x[k]);
          }
          // bf16 register 2q + h: row + 8h, samples t (low half) and t + 4 of k-step q of the step
#pragma unroll
          for (int h = 0; h < 2; ++h) {
            fa[f][8 + 2 * q + h] = pack_bf16x2(x[h], x[h + 2]);
            fa[f][12 + 2 * q + h] = pack_bf16x2(a[h] - x[h], a[h + 2] - x[h + 2]);
          }
        }
        wgmma_fence_regs<16>(fa[f]);
        if (s == 3) {
          __syncwarp();
          if (lane == 0) mbar_arrive(&raw_empty[sr]);   // every lane of the warp has read the slice's A fragments
        }
        if (s == 0) mbar_wait(&op_full[so], (c / NO) & 1);
        wgmma_fence();
        // bf16 tile: hi of k16 step kk at 32 kk, lo at 64 + 32 kk
        wgmma_bf16_ra<128>(acc[r], &fa[f][12], wgmma_desc_k128(b0 + kWgTile + 32 * kk));        // lo * hi
        wgmma_bf16_ra<128>(acc[r], &fa[f][8], wgmma_desc_k128(b0 + kWgTile + 64 + 32 * kk));    // hi * lo
        wgmma_tf32_ra<128>(acc[r], &fa[f][0], wgmma_desc_k128(b0 + 64 * kk));
        wgmma_tf32_ra<128>(acc[r], &fa[f][4], wgmma_desc_k128(b0 + 64 * kk + 32));
        wgmma_commit();
      }
    }
    wgmma_wait_all();
    wgmma_fence_regs<64>(acc[0]);
    wgmma_fence_regs<64>(acc[1]);

    // ---- epilogue: fragments -> partial slab of this split ----
    float* P = p.partial + (size_t)split * p.Dp * p.Dp;
    const int col0 = bj * kBlk + 2 * t4;
#pragma unroll
    for (int r = 0; r < 2; ++r) {
      const int row0 = (a0 + g) * kBlk + r * 64 + m;
#pragma unroll
      for (int k = 0; k < 64; k += 2) {
        const int row = row0 + 8 * ((k >> 1) & 1), col = col0 + 8 * (k >> 2);
        *reinterpret_cast<float2*>(P + (size_t)row * p.Dp + col) = make_float2(acc[r][k], acc[r][k + 1]);
      }
    }
  }
}

// =============================================================================================
// exact SIMT kernel (fp32 / fp64), 64x64 tiles inside the same padded tile space
// =============================================================================================
struct SimtParams {
  const void* view_ptr[kMaxViews];
  int64_t view_ld[kMaxViews];
  int view_dim[kMaxViews];
  int view_poff[kMaxViews + 1];
  int n_views;
  int64_t n_rows;
  int64_t rows_per_split;
  int nb64, Dp;
  void* partial;      // T [S][Dp][Dp]
  void* partial_sum;  // T [S][Dp]
};

template <typename T>
__global__ void __launch_bounds__(256) moments_simt_kernel(const SimtParams p) {
  constexpr int KC = 16;
  __shared__ T As[KC][64];
  __shared__ T Bs[KC][64];
  // tile decode over the upper triangle of nb64 x nb64
  int t = blockIdx.x, bi = 0, rowlen = p.nb64;
  while (t >= rowlen) { t -= rowlen; ++bi; --rowlen; }
  const int bj = bi + t;
  const int split = blockIdx.y;
  const int64_t r0 = split * p.rows_per_split;
  const int64_t r1 = min(r0 + p.rows_per_split, p.n_rows);

  auto locate = [&](int pcol0, int& v, int& c0) {
    v = 0;
    while (v + 1 < p.n_views && p.view_poff[v + 1] <= pcol0) ++v;
    c0 = pcol0 - p.view_poff[v];
  };
  int vA, cA, vB, cB;
  locate(bi * 64, vA, cA);
  locate(bj * 64, vB, cB);
  const T* XA = static_cast<const T*>(p.view_ptr[vA]);
  const T* XB = static_cast<const T*>(p.view_ptr[vB]);
  const int64_t ldA = p.view_ld[vA], ldB = p.view_ld[vB];
  const int dA = p.view_dim[vA], dB = p.view_dim[vB];

  const int tx = threadIdx.x & 15, ty = threadIdx.x >> 4;
  T acc[4][4];
#pragma unroll
  for (int i = 0; i < 4; ++i)
#pragma unroll
    for (int j = 0; j < 4; ++j) acc[i][j] = T(0);
  T csum[4] = {T(0), T(0), T(0), T(0)};
  // One accumulator run covers at most kRun rows (as plan_tc bounds the 3xTF32 runs): a fp32 sum over all n rows of a
  // split would drift by eps * sqrt(n).  Every kRun rows the run is folded into float64 registers and restarts.
  constexpr int kRun = 2048;
  double fold[4][4], fold_sum[4];
#pragma unroll
  for (int i = 0; i < 4; ++i) {
    fold_sum[i] = 0.0;
#pragma unroll
    for (int j = 0; j < 4; ++j) fold[i][j] = 0.0;
  }
  auto fold_run = [&]() {
#pragma unroll
    for (int i = 0; i < 4; ++i) {
      fold_sum[i] += (double)csum[i];
      csum[i] = T(0);
#pragma unroll
      for (int j = 0; j < 4; ++j) {
        fold[i][j] += (double)acc[i][j];
        acc[i][j] = T(0);
      }
    }
  };

  const int lc = threadIdx.x & 63, lr = threadIdx.x >> 6;  // loader: 4 rows x 64 cols per pass
  for (int64_t r = r0; r < r1; r += KC) {
    if (r > r0 && (r - r0) % kRun == 0) fold_run();
#pragma unroll
    for (int i = 0; i < KC / 4; ++i) {
      const int kr = lr + 4 * i;
      const int64_t row = r + kr;
      const bool rv = row < r1;
      As[kr][lc] = (rv && cA + lc < dA) ? XA[row * ldA + cA + lc] : T(0);
      Bs[kr][lc] = (rv && cB + lc < dB) ? XB[row * ldB + cB + lc] : T(0);
    }
    __syncthreads();
#pragma unroll
    for (int k = 0; k < KC; ++k) {
      T a[4], b[4];
#pragma unroll
      for (int i = 0; i < 4; ++i) { a[i] = As[k][ty * 4 + i]; b[i] = Bs[k][tx * 4 + i]; }
#pragma unroll
      for (int i = 0; i < 4; ++i)
#pragma unroll
        for (int j = 0; j < 4; ++j) acc[i][j] = fma(a[i], b[j], acc[i][j]);
      if (ty == 0) {
#pragma unroll
        for (int j = 0; j < 4; ++j) csum[j] += b[j];
      }
    }
    __syncthreads();
  }
  fold_run();   // a split of at most kRun rows writes its fp32 sums unchanged
  T* P = static_cast<T*>(p.partial) + (size_t)split * p.Dp * p.Dp;
#pragma unroll
  for (int i = 0; i < 4; ++i)
#pragma unroll
    for (int j = 0; j < 4; ++j)
      P[(size_t)(bi * 64 + ty * 4 + i) * p.Dp + bj * 64 + tx * 4 + j] = (T)fold[i][j];
  if (bi == bj && ty == 0) {
    T* S = static_cast<T*>(p.partial_sum) + (size_t)split * p.Dp;
#pragma unroll
    for (int j = 0; j < 4; ++j) S[bi * 64 + tx * 4 + j] = (T)fold_sum[j];
  }
}

// =============================================================================================
// fp64 tensor-core variant of the exact kernel: mma.sync.aligned.m8n8k4.row.col.f64 (DMMA; wgmma has no
// f64 kind).  Same 64x64 tiles, same partial layout and split planning as moments_simt_kernel.
// 8 warps; warp w owns the 32 x 16 sub-tile (rows 32*(w&1), cols 16*(w>>1)) = 4 x 2 m8n8 fragments.
// Shared tiles are [k][64 + 8] doubles: the 16-bank skew between consecutive k rows makes the 64-bit
// fragment loads conflict-free (two wavefronts, the minimum for 32 lanes x 8 bytes).
// =============================================================================================
__device__ __forceinline__ void dmma_m8n8k4(double& c0, double& c1, double a, double b) {
  asm volatile("mma.sync.aligned.m8n8k4.row.col.f64.f64.f64.f64 {%0, %1}, {%2}, {%3}, {%0, %1};"
               : "+d"(c0), "+d"(c1)
               : "d"(a), "d"(b));
}

__global__ void __launch_bounds__(256) moments_dmma_kernel(const SimtParams p) {
  constexpr int KC = 16;
  constexpr int LDS = 64 + 4;   // row stride = 8 banks (mod 32): fragment loads (4 k-rows x 8 columns) are conflict-free
  __shared__ double As[2][KC][LDS];   // double buffered: one block barrier per 16-row chunk
  __shared__ double Bs[2][KC][LDS];
  int t = blockIdx.x, bi = 0, rowlen = p.nb64;
  while (t >= rowlen) { t -= rowlen; ++bi; --rowlen; }
  const int bj = bi + t;
  const int split = blockIdx.y;
  const int64_t r0 = split * p.rows_per_split;
  const int64_t r1 = min(r0 + p.rows_per_split, p.n_rows);

  auto locate = [&](int pcol0, int& v, int& c0) {
    v = 0;
    while (v + 1 < p.n_views && p.view_poff[v + 1] <= pcol0) ++v;
    c0 = pcol0 - p.view_poff[v];
  };
  int vA, cA, vB, cB;
  locate(bi * 64, vA, cA);
  locate(bj * 64, vB, cB);
  const double* XA = static_cast<const double*>(p.view_ptr[vA]);
  const double* XB = static_cast<const double*>(p.view_ptr[vB]);
  const int64_t ldA = p.view_ld[vA], ldB = p.view_ld[vB];
  const int dA = p.view_dim[vA], dB = p.view_dim[vB];

  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int wm = (warp & 1) * 32, wn = (warp >> 1) * 16;
  const int gq = lane >> 2, tq = lane & 3;     // fragment coordinates: row/col group and k index
  double acc[4][2][2];
#pragma unroll
  for (int i = 0; i < 4; ++i)
#pragma unroll
    for (int j = 0; j < 2; ++j) acc[i][j][0] = acc[i][j][1] = 0.0;
  double csum = 0.0;                            // column sums: thread c < 64 of a diagonal tile sums column c

  const int lc = threadIdx.x & 63, lr = threadIdx.x >> 6;
  // register prefetch: the global loads of chunk c + 1 are in flight while the tensor pipe works on chunk c
  double ra[KC / 4], rb[KC / 4];
  auto gload = [&](int64_t r) {
#pragma unroll
    for (int i = 0; i < KC / 4; ++i) {
      const int64_t row = r + lr + 4 * i;
      const bool rv = row < r1;
      ra[i] = (rv && cA + lc < dA) ? XA[row * ldA + cA + lc] : 0.0;
      rb[i] = (rv && cB + lc < dB) ? XB[row * ldB + cB + lc] : 0.0;
    }
  };
  auto sstore = [&](int buf) {
#pragma unroll
    for (int i = 0; i < KC / 4; ++i) {
      As[buf][lr + 4 * i][lc] = ra[i];
      Bs[buf][lr + 4 * i][lc] = rb[i];
    }
  };
  gload(r0);
  sstore(0);
  __syncthreads();
  int buf = 0;
  for (int64_t r = r0; r < r1; r += KC, buf ^= 1) {
    const bool more = r + KC < r1;
    if (more) gload(r + KC);
#pragma unroll
    for (int k0 = 0; k0 < KC; k0 += 4) {
      double a[4], b[2];
#pragma unroll
      for (int i = 0; i < 4; ++i) a[i] = As[buf][k0 + tq][wm + 8 * i + gq];   // A[m][k] = X[k][m]
#pragma unroll
      for (int j = 0; j < 2; ++j) b[j] = Bs[buf][k0 + tq][wn + 8 * j + gq];   // B[k][n] = X[k][n]
#pragma unroll
      for (int i = 0; i < 4; ++i)
#pragma unroll
        for (int j = 0; j < 2; ++j) dmma_m8n8k4(acc[i][j][0], acc[i][j][1], a[i], b[j]);
    }
    if (bi == bj && threadIdx.x < 64) {
#pragma unroll
      for (int k = 0; k < KC; ++k) csum += Bs[buf][k][threadIdx.x];
    }
    if (more) sstore(buf ^ 1);   // the other buffer was last read before the previous barrier
    __syncthreads();
  }
  double* P = static_cast<double*>(p.partial) + (size_t)split * p.Dp * p.Dp;
#pragma unroll
  for (int i = 0; i < 4; ++i)
#pragma unroll
    for (int j = 0; j < 2; ++j) {
      const int row = bi * 64 + wm + 8 * i + gq;       // C fragment: row = lane/4, cols = (lane%4)*2 + {0,1}
      const int col = bj * 64 + wn + 8 * j + 2 * tq;
      *reinterpret_cast<double2*>(P + (size_t)row * p.Dp + col) = make_double2(acc[i][j][0], acc[i][j][1]);
    }
  if (bi == bj && threadIdx.x < 64)
    static_cast<double*>(p.partial_sum)[(size_t)split * p.Dp + bi * 64 + threadIdx.x] = csum;
}

// =============================================================================================
// K2: reduce split partials (fixed order => deterministic) and finalise the covariance
// =============================================================================================
// valid_blk: partial tiles exist for block-row <= block-col where blocks are `blk` wide.
// ldp: leading dimension (and row count) of each partial slab, >= Dp
template <typename T>
__global__ void reduce_partials_kernel(const T* __restrict__ partial, const T* __restrict__ partial_sum,
                                       int S, int Dp, int ldp, int blk, double* __restrict__ out,
                                       int accumulate = 0) {
  const size_t total = (size_t)Dp * Dp + (partial_sum ? Dp : 0);   // partial_sum == NULL: the sums come from elsewhere
  const size_t slab = (size_t)ldp * ldp;
  for (size_t i = blockIdx.x * (size_t)blockDim.x + threadIdx.x; i < total;
       i += (size_t)gridDim.x * blockDim.x) {
    double acc = 0.0;
    if (i < (size_t)Dp * Dp) {
      const int r = (int)(i / Dp), c = (int)(i % Dp);
      if (r / blk <= c / blk) {
        // 8 independent loads in flight, added in split order (the sum is the same as the plain loop's)
        const T* src = partial + (size_t)r * ldp + c;
        int s = 0;
        for (; s + 8 <= S; s += 8) {
          T v[8];
#pragma unroll
          for (int u = 0; u < 8; ++u) v[u] = src[(size_t)(s + u) * slab];
#pragma unroll
          for (int u = 0; u < 8; ++u) acc += (double)v[u];
        }
        for (; s < S; ++s) acc += (double)src[(size_t)s * slab];
      }
    } else {
      const size_t j = i - (size_t)Dp * Dp;
      for (int s = 0; s < S; ++s) acc += (double)partial_sum[(size_t)s * ldp + j];
    }
    out[i] = accumulate ? out[i] + acc : acc;
  }
}

struct CovParams {
  int n_views, D, Dp;
  int dims[kMaxViews];
  int coff[kMaxViews + 1];
  int poff[kMaxViews + 1];
};

__device__ __forceinline__ int compact_to_padded(const CovParams& p, int g) {
  int v = 0;
  while (v + 1 < p.n_views && p.coff[v + 1] <= g) ++v;
  return p.poff[v] + (g - p.coff[v]);
}

template <typename Tout>
__global__ void covariance_kernel(const CovParams p, const double* __restrict__ mom, double n_total,
                                  int center, Tout* __restrict__ C, int64_t ldc, Tout* __restrict__ mean) {
  const double* M = mom;
  const double* s = mom + (size_t)p.Dp * p.Dp;
  const int gi = blockIdx.y * blockDim.y + threadIdx.y;
  const int gj = blockIdx.x * blockDim.x + threadIdx.x;
  if (gi >= p.D || gj >= p.D) return;
  const int pi = compact_to_padded(p, gi), pj = compact_to_padded(p, gj);
  const int r = min(pi, pj), c = max(pi, pj);  // upper block triangle (and exact symmetry)
  double v = M[(size_t)r * p.Dp + c];
  if (center) v -= s[pi] * s[pj] / n_total;
  C[(size_t)gi * ldc + gj] = (Tout)(v / (n_total - 1.0));
  if (gi == 0 && mean) mean[gj] = (Tout)(center ? s[pj] / n_total : 0.0);
}

// =============================================================================================
// host side
// =============================================================================================
namespace {

int sm_count() {
  static int n[64] = {};   // per device ordinal (a process may drive several GPUs)
  int dev = 0;
  cudaGetDevice(&dev);
  if (dev < 0 || dev >= 64) return 132;
  if (!n[dev]) {
    cudaDeviceGetAttribute(&n[dev], cudaDevAttrMultiProcessorCount, dev);
    if (n[dev] <= 0) n[dev] = 132;
  }
  return n[dev];
}

struct TcPlan {
  int total_chunks, num_splits, chunks_per_split, ntiles;
  size_t partial_bytes, sum_bytes;
};

TcPlan plan_tc(const ColumnLayout& L, int64_t n_rows, int mode) {
  const bool x3 = mode != 0;   // 0: one TF32 pass, 1: 3xTF32, 3: 3xTF32 with bf16 cross terms
  TcPlan P;
  P.total_chunks = (int)ceil_div(n_rows, kWgKC);
  P.ntiles = L.nblocks * (L.nblocks + 1) / 2;
  // about four waves of CTAs, so that the tile count does not leave a mostly idle last wave.  Counted in 128 x 128
  // unit tiles also for the pair-tile kernel of mode 3, so that every mode splits the sample axis alike.
  int S = (int)ceil_div(4 * sm_count(), P.ntiles);
  int max_splits = 64;
  if (x3) {
    // The 3xTF32 mode exists for fp32-grade results: one fp32 accumulator run is bounded to 2048 samples and the
    // fixed-order float64 reduction of the split partials does the long sum.
    S = std::max<int64_t>(S, ceil_div(n_rows, 2048));
    max_splits = 256;
  }
  const int min_chunks = 8;  // keep the per-CTA prologue / epilogue amortised
  S = (int)std::min<int64_t>(S, std::max<int64_t>(1, P.total_chunks / min_chunks));
  // keep the split partials below 2 GiB
  const int64_t slab = (int64_t)L.Dp * L.Dp * (int64_t)sizeof(float);
  max_splits = (int)std::max<int64_t>(1, std::min<int64_t>(max_splits, ((int64_t)2 << 30) / slab));
  S = std::min(S, max_splits);
  S = std::max(1, std::min(S, P.total_chunks));
  P.chunks_per_split = (int)ceil_div(P.total_chunks, S);
  P.num_splits = (int)ceil_div(P.total_chunks, P.chunks_per_split);
  P.partial_bytes = (size_t)P.num_splits * L.Dp * L.Dp * sizeof(float);
  P.sum_bytes = (size_t)P.num_splits * L.Dp * sizeof(float);
  return P;
}

// rows one pass of the 3xTF32 modes may take: the split count that keeps the partials below 2 GiB (<= 256) times the
// 2048-sample accumulator run
int64_t tc_rows_cap(const ColumnLayout& L, int mode) {
  if (mode == 0) return (int64_t)1 << 31;
  const int64_t slab = (int64_t)L.Dp * L.Dp * (int64_t)sizeof(float);
  const int64_t max_splits = std::max<int64_t>(1, std::min<int64_t>(256, ((int64_t)2 << 30) / slab));
  return max_splits * 2048;
}

inline size_t align256(size_t x) { return (x + 255) & ~size_t(255); }

struct SimtPlan {
  int nb64, ntiles, num_splits;
  int64_t rows_per_split;
};

SimtPlan plan_simt(const ColumnLayout& L, int64_t n_rows) {
  SimtPlan P;
  P.nb64 = L.Dp / 64;
  P.ntiles = P.nb64 * (P.nb64 + 1) / 2;
  int S = 1;
  if (P.ntiles < 2 * sm_count()) S = (2 * sm_count()) / P.ntiles;
  S = (int)std::min<int64_t>(S, std::max<int64_t>(1, n_rows / 64));   // mini-batches: fill the machine with short slabs
  S = std::max(1, std::min(S, 64));
  P.rows_per_split = ceil_div(ceil_div(n_rows, S), 16) * 16;
  P.num_splits = (int)ceil_div(n_rows, P.rows_per_split);
  return P;
}

}  // namespace

size_t moments_workspace_bytes(int dtype, int precision, const ColumnLayout& L, int64_t n_rows) {
  if (precision == 2 || dtype == 1) {
    SimtPlan P = plan_simt(L, n_rows);
    size_t el = dtype == 1 ? 8 : 4;
    return align256((size_t)P.num_splits * L.Dp * L.Dp * el) + align256((size_t)P.num_splits * L.Dp * el);
  }
  TcPlan P = plan_tc(L, std::min(n_rows, tc_rows_cap(L, precision)), precision);   // sized for one pass
  return align256(P.partial_bytes) + align256(P.sum_bytes) + 256;
}

namespace {

typedef CUresult (*EncodeTiledFn)(CUtensorMap*, CUtensorMapDataType, cuuint32_t, void*, const cuuint64_t*,
                                  const cuuint64_t*, const cuuint32_t*, const cuuint32_t*, CUtensorMapInterleave,
                                  CUtensorMapSwizzle, CUtensorMapL2promotion, CUtensorMapFloatOOBfill);

// cuTensorMapEncodeTiled through the runtime's driver entry point (no link against libcuda)
EncodeTiledFn encode_fn() {
  static EncodeTiledFn fn = nullptr;
  static std::once_flag once;
  std::call_once(once, [] {
    void* f = nullptr;
    cudaDriverEntryPointQueryResult q;
    if (cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &f, cudaEnableDefault, &q) == cudaSuccess &&
        q == cudaDriverEntryPointSuccess)
      fn = reinterpret_cast<EncodeTiledFn>(f);
  });
  return fn;
}

// Row-major fp32 view (n_rows x d, row pitch ld floats) read in [32 rows x 32 columns] boxes with 128-byte swizzle
// (see raw_offset); elements past column d or row n_rows read as zero, also in boxes that lie wholly past column d.
int encode_view_map(CUtensorMap* map, const void* ptr, int64_t n_rows, int64_t d, int64_t ld) {
  EncodeTiledFn enc = encode_fn();
  if (!enc) {
    set_error("cuTensorMapEncodeTiled entry point not available (driver too old?)");
    return -2;
  }
  cuuint64_t gdim[2] = {(cuuint64_t)d, (cuuint64_t)n_rows};
  cuuint64_t gstride[1] = {(cuuint64_t)ld * 4};
  cuuint32_t box[2] = {32, (cuuint32_t)kWgKC};
  cuuint32_t estr[2] = {1, 1};
  CUresult r = enc(map, CU_TENSOR_MAP_DATA_TYPE_FLOAT32, 2, const_cast<void*>(ptr), gdim, gstride, box, estr,
                   CU_TENSOR_MAP_INTERLEAVE_NONE, CU_TENSOR_MAP_SWIZZLE_128B, CU_TENSOR_MAP_L2_PROMOTION_L2_256B,
                   CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
  if (r != CUDA_SUCCESS) {
    set_error("cuTensorMapEncodeTiled failed with CUresult %d (d=%lld n=%lld ld=%lld)", (int)r, (long long)d,
              (long long)n_rows, (long long)ld);
    return -3;
  }
  return 0;
}

int moments_tf32_pass(const ColumnLayout& L, WgParams& prm, int64_t row_base, int64_t n_rows, int mode,
                      double* moments_out, void* ws, size_t ws_bytes, cudaStream_t stream, int accumulate);

}  // namespace

// The 3xTF32 modes bound one accumulator run to 2048 samples (plan_tc) and the split partials to 2 GiB: inputs longer
// than tc_rows_cap() rows are processed in equal passes whose float64 moments add up in moments_out (the moments are
// additive over rows; partials are sized for one pass).  The tensor maps span all rows; a pass offsets the row
// coordinate.
int moments_tf32(const ColumnLayout& L, const void* const* views, const int64_t* lds, int64_t n_rows, int mode,
                 double* moments_out, void* ws, size_t ws_bytes, cudaStream_t stream) {
  CCAB_CHECK_ARG(n_rows >= 1 && n_rows < (int64_t)1 << 31, "n_rows out of range");
  for (int v = 0; v < L.n_views; ++v)
    CCAB_CHECK_ARG((reinterpret_cast<uintptr_t>(views[v]) & 15) == 0 && lds[v] % 4 == 0,
                   "TF32 moments need 16-byte aligned views and lds %% 4 == 0 (view %d: ld %lld)", v,
                   (long long)lds[v]);
  {
    int dev = 0;   // bind the primary context to this thread before the driver-API tensor-map encoder
    CCAB_CUDA(cudaGetDevice(&dev));
    CCAB_CUDA(cudaSetDevice(dev));
  }
  WgParams prm;
  memset(&prm, 0, sizeof(prm));
  for (int v = 0; v < L.n_views; ++v) {
    int rc = encode_view_map(&prm.map[v], views[v], n_rows, L.dims[v], lds[v]);
    if (rc) return rc;
  }
  int b = 0;
  for (int v = 0; v < L.n_views; ++v)
    for (int c = 0; c < L.dims[v]; c += kBlk, ++b) {
      prm.blk_view[b] = (uint8_t)v;
      prm.blk_col0[b] = c;
    }
  const int64_t cap = tc_rows_cap(L, mode);
  if (n_rows <= cap) return moments_tf32_pass(L, prm, 0, n_rows, mode, moments_out, ws, ws_bytes, stream, 0);
  const int64_t npass = ceil_div(n_rows, cap);
  const int64_t per = std::min(cap, ceil_div(ceil_div(n_rows, npass), 2048) * 2048);
  int pass = 0;
  for (int64_t r0 = 0; r0 < n_rows; r0 += per, ++pass) {
    int rc = moments_tf32_pass(L, prm, r0, std::min(per, n_rows - r0), mode, moments_out, ws, ws_bytes, stream,
                               pass > 0);
    if (rc) return rc;
  }
  return 0;
}

namespace {
template <K1Mode M>
int launch_wgmma(dim3 grid, const WgParams& prm, cudaStream_t stream) {
  // function attributes are per device / context: set on every call
  CCAB_CUDA(cudaFuncSetAttribute(moments_wgmma_kernel<M>, cudaFuncAttributeMaxDynamicSharedMemorySize,
                                 WgCfg<M>::kSmem));
  moments_wgmma_kernel<M><<<grid, kWgThreads, WgCfg<M>::kSmem, stream>>>(prm);
  return 0;
}

int launch_x3b_pair(int num_splits, const WgParams& prm, cudaStream_t stream) {
  CCAB_CUDA(cudaFuncSetAttribute(moments_x3b_pair_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize,
                                 PairCfg::kSmem));
  moments_x3b_pair_kernel<<<dim3(pair_tiles(prm.nblocks), num_splits), kPrThreads, PairCfg::kSmem, stream>>>(prm);
  return 0;
}

// One pass over rows [row_base, row_base + n_rows).  Its splits end on multiples of 32 rows from row_base, and a pass
// that is not the last ends on a multiple of 2048, so no slice reads rows of the next pass.
int moments_tf32_pass(const ColumnLayout& L, WgParams& prm, int64_t row_base, int64_t n_rows, int mode,
                      double* moments_out, void* ws, size_t ws_bytes, cudaStream_t stream, int accumulate) {
  TcPlan P = plan_tc(L, n_rows, mode);
  const size_t need = align256(P.partial_bytes) + align256(P.sum_bytes) + 256;
  CCAB_CHECK_ARG(ws_bytes >= need, "workspace too small: %zu < %zu", ws_bytes, need);
  uint8_t* w = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(ws) + 255) & ~uintptr_t(255));
  float* d_partial = reinterpret_cast<float*>(w);
  float* d_partial_sum = reinterpret_cast<float*>(w + align256(P.partial_bytes));

  prm.partial = d_partial;
  prm.partial_sum = d_partial_sum;
  prm.n_rows = n_rows;
  prm.rows_per_split = (int64_t)P.chunks_per_split * kWgKC;
  prm.row_base = row_base;
  prm.nblocks = L.nblocks;
  prm.Dp = L.Dp;
  dim3 grid(P.ntiles, P.num_splits);
  if (g_prof_on) cudaEventRecord(g_prof_e0, stream);
  int rc = mode == 3   ? launch_x3b_pair(P.num_splits, prm, stream)
           : mode != 0 ? launch_wgmma<K1Mode::X3>(grid, prm, stream)
                       : launch_wgmma<K1Mode::TF32>(grid, prm, stream);
  if (rc) return rc;
  count_launches(1);
  CCAB_CUDA(cudaGetLastError());
  if (g_prof_on) {
    cudaEventRecord(g_prof_e1, stream);
    g_prof_valid = true;
  }

  const size_t total = (size_t)L.Dp * L.Dp + L.Dp;
  int rblocks = (int)std::min<size_t>((total + 255) / 256, (size_t)sm_count() * 8);
  reduce_partials_kernel<float><<<rblocks, 256, 0, stream>>>(d_partial, d_partial_sum, P.num_splits, L.Dp, L.Dp,
                                                            kBlk, moments_out, accumulate); count_launches(1);
  CCAB_CUDA(cudaGetLastError());
  return 0;
}
}  // namespace

template <typename T>
int moments_simt(const ColumnLayout& L, const void* const* views, const int64_t* lds, int64_t n_rows,
                 double* moments_out, void* ws, size_t ws_bytes, cudaStream_t stream) {
  CCAB_CHECK_ARG(n_rows >= 1, "n_rows must be positive");
  SimtPlan P = plan_simt(L, n_rows);
  const size_t pb = align256((size_t)P.num_splits * L.Dp * L.Dp * sizeof(T));
  const size_t sb = align256((size_t)P.num_splits * L.Dp * sizeof(T));
  CCAB_CHECK_ARG(ws_bytes >= pb + sb, "workspace too small: %zu < %zu", ws_bytes, pb + sb);
  uint8_t* w = static_cast<uint8_t*>(ws);
  SimtParams prm;
  memset(&prm, 0, sizeof(prm));
  for (int v = 0; v < L.n_views; ++v) {
    prm.view_ptr[v] = views[v];
    prm.view_ld[v] = lds[v];
    prm.view_dim[v] = L.dims[v];
  }
  for (int v = 0; v <= L.n_views; ++v) prm.view_poff[v] = L.poff[v];
  prm.n_views = L.n_views;
  prm.n_rows = n_rows;
  prm.rows_per_split = P.rows_per_split;
  prm.nb64 = P.nb64;
  prm.Dp = L.Dp;
  prm.partial = w;
  prm.partial_sum = w + pb;
  // partial sums of non-diagonal 64-blocks inside a 128-block are never written by the kernel: the
  // reducer only reads what a tile wrote (block-triangle test at 64 granularity).
  dim3 grid(P.ntiles, P.num_splits);
  if constexpr (std::is_same<T, double>::value)
    moments_dmma_kernel<<<grid, 256, 0, stream>>>(prm);
  else
    moments_simt_kernel<T><<<grid, 256, 0, stream>>>(prm);
  count_launches(1);
  CCAB_CUDA(cudaGetLastError());
  const size_t total = (size_t)L.Dp * L.Dp + L.Dp;
  int rblocks = (int)std::min<size_t>((total + 255) / 256, (size_t)sm_count() * 8);
  reduce_partials_kernel<T><<<rblocks, 256, 0, stream>>>(static_cast<const T*>(prm.partial),
                                                        static_cast<const T*>(prm.partial_sum), P.num_splits,
                                                        L.Dp, L.Dp, 64, moments_out); count_launches(1);
  CCAB_CUDA(cudaGetLastError());
  return 0;
}

template int moments_simt<float>(const ColumnLayout&, const void* const*, const int64_t*, int64_t, double*, void*,
                                 size_t, cudaStream_t);
template int moments_simt<double>(const ColumnLayout&, const void* const*, const int64_t*, int64_t, double*, void*,
                                  size_t, cudaStream_t);

// =============================================================================================
// exchange-step packing (SURVEY.md §8e): only the upper triangle of 128 x 128 blocks of the moment matrix carries
// information; the all-reduced message is  [ upper blocks (row-major over bi <= bj) | column sums | n | reserved ].
// For D = 2048 that is 17.9 MB of float64 instead of 33.6 MB.
// =============================================================================================
__global__ void pack_moments_kernel(const double* __restrict__ mom, int nblocks, int Dp, double n_local,
                                    double* __restrict__ packed) {
  // blockIdx.x walks the upper-triangle blocks, then one extra "block" for the column sums and the tail
  const int nt = nblocks * (nblocks + 1) / 2;
  const int t = blockIdx.x;
  if (t < nt) {
    int bi = 0, rem = t, rowlen = nblocks;
    while (rem >= rowlen) { rem -= rowlen; ++bi; --rowlen; }
    const int bj = bi + rem;
    const double* src = mom + (size_t)bi * kBlk * Dp + (size_t)bj * kBlk;
    double* dst = packed + (size_t)t * kBlk * kBlk;
    for (int e = threadIdx.x; e < kBlk * kBlk; e += blockDim.x) dst[e] = src[(size_t)(e / kBlk) * Dp + (e % kBlk)];
  } else {
    double* dst = packed + (size_t)nt * kBlk * kBlk;
    const double* s = mom + (size_t)Dp * Dp;
    for (int e = threadIdx.x; e < Dp; e += blockDim.x) dst[e] = s[e];
    if (threadIdx.x == 0) { dst[Dp] = n_local; dst[Dp + 1] = 0.0; }
  }
}

__global__ void unpack_moments_kernel(const double* __restrict__ packed, int nblocks, int Dp, double* __restrict__ mom) {
  const int nt = nblocks * (nblocks + 1) / 2;
  const int bi = blockIdx.y, bj = blockIdx.x;
  if (bi < nblocks) {
    double* dst = mom + (size_t)bi * kBlk * Dp + (size_t)bj * kBlk;
    if (bj >= bi) {
      const int t = bi * nblocks - bi * (bi - 1) / 2 + (bj - bi);
      const double* src = packed + (size_t)t * kBlk * kBlk;
      for (int e = threadIdx.x; e < kBlk * kBlk; e += blockDim.x) dst[(size_t)(e / kBlk) * Dp + (e % kBlk)] = src[e];
    } else {
      for (int e = threadIdx.x; e < kBlk * kBlk; e += blockDim.x) dst[(size_t)(e / kBlk) * Dp + (e % kBlk)] = 0.0;
    }
  } else if (bj == 0) {
    const double* src = packed + (size_t)nt * kBlk * kBlk;
    double* s = mom + (size_t)Dp * Dp;
    for (int e = threadIdx.x; e < Dp; e += blockDim.x) s[e] = src[e];
  }
}

// =============================================================================================
// Fused exchange step over NVLink / NVSwitch (SURVEY.md §8e "v2"): ONE kernel packs the upper block triangle of the
// local moments into a symmetric-memory buffer, meets the other ranks on per-CTA flags in their signal pads, reduces
// its slice of the message INSIDE THE SWITCH (multimem.ld_reduce on the multicast address: one load returns the sum
// over all ranks), broadcasts the sums with multimem.st, meets the ranks again and scatters the totals back into the
// moment buffer.  No NCCL call, no intermediate launch; every element is reduced exactly once, so all ranks receive
// bit-identical totals.  CTA c of every rank owns the same column of regions {(owner rho, c)}: it needs no grid-wide
// synchronisation, only its own flag row.  The buffers / flags come from torch's symmetric memory (parallel.py).
// =============================================================================================
__device__ __forceinline__ double multimem_ld_reduce_add_f64(const double* mc_addr) {
  double v;
  asm volatile("multimem.ld_reduce.relaxed.sys.global.add.f64 %0, [%1];" : "=d"(v) : "l"(mc_addr) : "memory");
  return v;
}
__device__ __forceinline__ void multimem_st_f64(double* mc_addr, double v) {
  asm volatile("multimem.st.relaxed.sys.global.f64 [%0], %1;" ::"l"(mc_addr), "d"(v) : "memory");
}
__device__ __forceinline__ void st_release_sys_u32(uint32_t* p, uint32_t v) {
  asm volatile("st.release.sys.global.u32 [%0], %1;" ::"l"(p), "r"(v) : "memory");
}
__device__ __forceinline__ uint32_t ld_acquire_sys_u32(const uint32_t* p) {
  uint32_t v;
  asm volatile("ld.acquire.sys.global.u32 %0, [%1];" : "=r"(v) : "l"(p) : "memory");
  return v;
}

struct ExchangeParams {
  double* mom;            // local moment buffer [Dp*Dp + Dp]
  double* sym;            // this rank's symmetric buffer (local address), >= world * chunk doubles
  double* mc;             // multicast address of the same buffer
  uint32_t* const* pads;  // device array [world]: signal pad of every rank (peer-mapped)
  double* n_total_out;    // device scalar (may be NULL)
  double n_local;
  long long packed;       // doubles in the message (upper blocks | column sums | n | reserved)
  long long chunk;        // doubles per owner rank (world * chunk >= packed)
  int rank, world, nblocks, Dp;
  unsigned epoch;         // 2 flag values per call: epoch, epoch + 1 (monotonic; compared with >=)
};

__device__ __forceinline__ const double* packed_src(const ExchangeParams& p, long long e, int nt) {
  // element e of the message -> its home in the moment buffer
  const long long blk = e / (kBlk * kBlk);
  if (blk < nt) {
    int bi = 0, rem = (int)blk, rowlen = p.nblocks;
    while (rem >= rowlen) { rem -= rowlen; ++bi; --rowlen; }
    const int bj = bi + rem;
    const int off = (int)(e - blk * (kBlk * kBlk));
    return p.mom + ((size_t)bi * kBlk + off / kBlk) * p.Dp + (size_t)bj * kBlk + (off % kBlk);
  }
  const long long t = e - (long long)nt * kBlk * kBlk;
  return t < p.Dp ? p.mom + (size_t)p.Dp * p.Dp + t : nullptr;   // tail: n, reserved
}

__device__ __forceinline__ void exchange_barrier(const ExchangeParams& p, unsigned value) {
  // all threads of the CTA have finished their writes to symmetric / peer memory
  __threadfence_system();
  __syncthreads();
  if ((int)threadIdx.x < p.world)
    st_release_sys_u32(p.pads[threadIdx.x] + (size_t)blockIdx.x * p.world + p.rank, value);
  if ((int)threadIdx.x < p.world) {
    const uint32_t* slot = p.pads[p.rank] + (size_t)blockIdx.x * p.world + threadIdx.x;
    unsigned spins = 0;
    while ((int)(ld_acquire_sys_u32(slot) - value) < 0) {
      if (++spins > (1u << 26)) {   // ~ seconds: a lost peer must not hang the box
        printf("ccab: exchange barrier timed out (rank %d cta %d peer %d)\n", p.rank, blockIdx.x, threadIdx.x);
        __trap();
      }
    }
  }
  __syncthreads();
}

__global__ void __launch_bounds__(512) exchange_nvls_kernel(const ExchangeParams p) {
  const int nt = p.nblocks * (p.nblocks + 1) / 2;
  const long long sub = (p.chunk + gridDim.x - 1) / gridDim.x;   // doubles per (owner, CTA) region
  const long long r0 = (long long)blockIdx.x * sub;
  const long long r1 = r0 + sub < p.chunk ? r0 + sub : p.chunk;
  // ---- pack this CTA's column of regions ----
  for (int rho = 0; rho < p.world; ++rho) {
    const long long base = (long long)rho * p.chunk;
    for (long long i = r0 + threadIdx.x; i < r1; i += blockDim.x) {
      const long long e = base + i;
      double v = 0.0;
      if (e < p.packed) {
        const double* src = packed_src(p, e, nt);
        v = src ? *src : (e == (long long)nt * kBlk * kBlk + p.Dp ? p.n_local : 0.0);
      }
      p.sym[e] = v;
    }
  }
  exchange_barrier(p, p.epoch);
  // ---- reduce the own region in the switch and broadcast it ----
  {
    const long long base = (long long)p.rank * p.chunk;
    for (long long i = r0 + threadIdx.x; i < r1; i += blockDim.x) {
      const double v = multimem_ld_reduce_add_f64(p.mc + base + i);
      multimem_st_f64(p.mc + base + i, v);
    }
  }
  exchange_barrier(p, p.epoch + 1);
  // ---- scatter the totals back ----
  for (int rho = 0; rho < p.world; ++rho) {
    const long long base = (long long)rho * p.chunk;
    for (long long i = r0 + threadIdx.x; i < r1; i += blockDim.x) {
      const long long e = base + i;
      if (e >= p.packed) continue;
      const double v = p.sym[e];
      const double* dst = packed_src(p, e, nt);
      if (dst) *const_cast<double*>(dst) = v;
      else if (e == (long long)nt * kBlk * kBlk + p.Dp && p.n_total_out) *p.n_total_out = v;
    }
  }
}

int moments_exchange_nvls(const ColumnLayout& L, double* mom, double n_local, double* sym_local, double* sym_multicast,
                          void* const* pads_dev, int rank, int world, int pad_slots, int64_t sym_doubles,
                          unsigned epoch, double* n_total_out, cudaStream_t stream) {
  CCAB_CHECK_ARG(world >= 2 && world <= 64 && rank >= 0 && rank < world, "bad rank / world %d / %d", rank, world);
  CCAB_CHECK_ARG(mom && sym_local && sym_multicast && pads_dev, "null pointer argument");
  ExchangeParams p;
  memset(&p, 0, sizeof(p));
  p.mom = mom; p.sym = sym_local; p.mc = sym_multicast;
  p.pads = reinterpret_cast<uint32_t* const*>(pads_dev);
  p.n_total_out = n_total_out; p.n_local = n_local;
  p.packed = moments_packed_size(L);
  p.chunk = ceil_div(ceil_div(p.packed, world), 2) * 2;
  CCAB_CHECK_ARG(sym_doubles >= p.chunk * world, "symmetric buffer too small: %lld < %lld doubles", (long long)sym_doubles,
                 (long long)(p.chunk * world));
  p.rank = rank; p.world = world; p.nblocks = L.nblocks; p.Dp = L.Dp; p.epoch = epoch;
  int grid = std::min(64, pad_slots / world);
  CCAB_CHECK_ARG(grid >= 1, "signal pad too small for %d ranks", world);
  grid = (int)std::min<int64_t>(grid, std::max<int64_t>(1, p.chunk / 512));
  exchange_nvls_kernel<<<grid, 512, 0, stream>>>(p);
  count_launches(1);
  CCAB_CUDA(cudaGetLastError());
  return 0;
}

// =============================================================================================
// Shifted accumulation (numerical safety of the one-pass covariance): C = (M - s s^T / n) / (n - 1) cancels
// catastrophically when a column's mean dominates its spread -- the relative error of C is eps_prod * (mean / std)^2
// with eps_prod the product / accumulation error of the moment kernel (1e-7 .. 1e-6 for the 3xTF32 modes).  Covariance
// is shift invariant, so the moments of X - x0 (x0 = pilot mean of the leading rows) are accumulated instead and the
// raw moments are rebuilt in float64 afterwards, where 53 bits absorb the cancellation:
//     M = M' + x0 s'^T + s' x0^T + n x0 x0^T,   s = s' + n x0.
// pilot_kernel : x0 and the ratio mean^2 / var per column from <= 4096 leading rows (one block per 32 columns)
// shift_kernel : Xs = X - x0
// unshift_kernel: the float64 correction above on the padded moment buffer (upper block triangle)
// =============================================================================================
template <typename T>
__global__ void pilot_kernel(const T* __restrict__ X, int64_t rows, int d, int64_t ld, T* __restrict__ x0,
                             float* __restrict__ ratio_max) {
  __shared__ double s1[32][33], s2[32][33];
  const int j = blockIdx.x * 32 + (threadIdx.x & 31);
  const int rg = threadIdx.x >> 5;
  double a = 0.0, b = 0.0;
  const double ref = j < d ? (double)X[j] : 0.0;     // first row as a provisional origin: the pilot itself must not cancel
  if (j < d)
    for (int64_t i = rg; i < rows; i += 32) {
      const double v = (double)X[i * ld + j] - ref;
      a += v;
      b += v * v;
    }
  s1[rg][threadIdx.x & 31] = a;
  s2[rg][threadIdx.x & 31] = b;
  __syncthreads();
  if (rg == 0 && j < d) {
    double sa = 0.0, sb = 0.0;
    for (int k = 0; k < 32; ++k) { sa += s1[k][threadIdx.x & 31]; sb += s2[k][threadIdx.x & 31]; }
    const double mean = sa / (double)rows;
    const double var = fmax(sb / (double)rows - mean * mean, 0.0);
    const double m0 = ref + mean;
    x0[j] = (T)m0;
    const double r = var > 0.0 ? m0 * m0 / var : (m0 != 0.0 ? 1e30 : 0.0);
    atomicMax(reinterpret_cast<unsigned*>(ratio_max), __float_as_uint((float)fmin(r, 1e30)));
  }
}

template <typename T>
__global__ void shift_kernel(const T* __restrict__ X, int64_t n, int d, int64_t ldx, const T* __restrict__ x0,
                             T* __restrict__ Xs, int64_t lds) {
  const int64_t total = n * (int64_t)d;
  for (int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; i < total; i += (int64_t)gridDim.x * blockDim.x) {
    const int64_t r = i / d;
    const int c = (int)(i - r * d);
    Xs[r * lds + c] = X[r * ldx + c] - x0[c];
  }
}

struct UnshiftParams {
  int n_views, Dp;
  int dims[kMaxViews];
  int poff[kMaxViews + 1];
  const void* x0[kMaxViews];   // per view, in the views' dtype
  int is_f64;
};
__device__ __forceinline__ double unshift_x0(const UnshiftParams& p, int pc) {
  int v = 0;
  while (v + 1 < p.n_views && p.poff[v + 1] <= pc) ++v;
  const int c = pc - p.poff[v];
  if (c >= p.dims[v] || !p.x0[v]) return 0.0;
  return p.is_f64 ? static_cast<const double*>(p.x0[v])[c] : (double)static_cast<const float*>(p.x0[v])[c];
}
__global__ void unshift_kernel(const UnshiftParams p, double* __restrict__ mom, double n) {
  double* M = mom;
  double* s = mom + (size_t)p.Dp * p.Dp;
  const size_t total = (size_t)p.Dp * p.Dp;
  for (size_t e = blockIdx.x * (size_t)blockDim.x + threadIdx.x; e < total; e += (size_t)gridDim.x * blockDim.x) {
    const int r = (int)(e / p.Dp), c = (int)(e % p.Dp);
    if (r / kBlk > c / kBlk) continue;
    const double ar = unshift_x0(p, r), ac = unshift_x0(p, c);
    if (ar == 0.0 && ac == 0.0) continue;
    M[e] += ar * s[c] + s[r] * ac + n * ar * ac;      // s still holds the shifted sums here
  }
}
__global__ void unshift_sums_kernel(const UnshiftParams p, double* __restrict__ mom, double n) {
  double* s = mom + (size_t)p.Dp * p.Dp;
  const int c = blockIdx.x * blockDim.x + threadIdx.x;
  if (c < p.Dp) s[c] += n * unshift_x0(p, c);
}

template <typename T>
int column_pilot(const T* X, int64_t rows, int d, int64_t ld, T* x0, float* ratio_max, cudaStream_t stream) {
  CCAB_CHECK_ARG(rows >= 1 && d >= 1 && ld >= d, "bad pilot shape");
  pilot_kernel<T><<<(unsigned)ceil_div(d, 32), 1024, 0, stream>>>(X, rows, d, ld, x0, ratio_max);
  count_launches(1);
  CCAB_CUDA(cudaGetLastError());
  return 0;
}
template <typename T>
int shift_rows(const T* X, int64_t n, int d, int64_t ldx, const T* x0, T* Xs, int64_t lds, cudaStream_t stream) {
  const int64_t total = n * (int64_t)d;
  if (total == 0) return 0;
  shift_kernel<T><<<(unsigned)std::min<int64_t>(ceil_div(total, 256), (int64_t)sm_count() * 16), 256, 0, stream>>>(
      X, n, d, ldx, x0, Xs, lds);
  count_launches(1);
  CCAB_CUDA(cudaGetLastError());
  return 0;
}
template int column_pilot<float>(const float*, int64_t, int, int64_t, float*, float*, cudaStream_t);
template int column_pilot<double>(const double*, int64_t, int, int64_t, double*, float*, cudaStream_t);
template int shift_rows<float>(const float*, int64_t, int, int64_t, const float*, float*, int64_t, cudaStream_t);
template int shift_rows<double>(const double*, int64_t, int, int64_t, const double*, double*, int64_t, cudaStream_t);

int moments_unshift(const ColumnLayout& L, double* mom, const void* const* x0, int is_f64, double n,
                    cudaStream_t stream) {
  UnshiftParams p;
  memset(&p, 0, sizeof(p));
  p.n_views = L.n_views; p.Dp = L.Dp; p.is_f64 = is_f64;
  for (int v = 0; v < L.n_views; ++v) { p.dims[v] = L.dims[v]; p.x0[v] = x0[v]; }
  for (int v = 0; v <= L.n_views; ++v) p.poff[v] = L.poff[v];
  const size_t total = (size_t)L.Dp * L.Dp;
  unshift_kernel<<<(unsigned)std::min<size_t>((total + 255) / 256, (size_t)sm_count() * 8), 256, 0, stream>>>(p, mom, n);
  unshift_sums_kernel<<<(unsigned)ceil_div(L.Dp, 256), 256, 0, stream>>>(p, mom, n);   // after M: M used the shifted s
  count_launches(2);
  CCAB_CUDA(cudaGetLastError());
  return 0;
}

int64_t moments_packed_size(const ColumnLayout& L) {
  const int64_t nt = (int64_t)L.nblocks * (L.nblocks + 1) / 2;
  return nt * kBlk * kBlk + L.Dp + 2;
}

int moments_pack(const ColumnLayout& L, const double* mom, double n_local, double* packed, cudaStream_t stream) {
  const int nt = L.nblocks * (L.nblocks + 1) / 2;
  pack_moments_kernel<<<nt + 1, 256, 0, stream>>>(mom, L.nblocks, L.Dp, n_local, packed);
  count_launches(1);
  CCAB_CUDA(cudaGetLastError());
  return 0;
}

int moments_unpack(const ColumnLayout& L, const double* packed, double* mom, cudaStream_t stream) {
  unpack_moments_kernel<<<dim3(L.nblocks, L.nblocks + 1), 256, 0, stream>>>(packed, L.nblocks, L.Dp, mom);
  count_launches(1);
  CCAB_CUDA(cudaGetLastError());
  return 0;
}

template <typename Tout>
int covariance_from_moments(const ColumnLayout& L, const double* moments, double n_total, int center, Tout* C,
                            int64_t ldc, Tout* mean, cudaStream_t stream) {
  CCAB_CHECK_ARG(n_total >= 2.0, "need at least 2 samples for a covariance, got %g", n_total);
  CCAB_CHECK_ARG(ldc >= L.D, "ldc too small");
  CovParams p;
  p.n_views = L.n_views;
  p.D = L.D;
  p.Dp = L.Dp;
  for (int v = 0; v < kMaxViews; ++v) p.dims[v] = v < L.n_views ? L.dims[v] : 0;
  for (int v = 0; v <= kMaxViews; ++v) {
    p.coff[v] = v <= L.n_views ? L.coff[v] : L.D;
    p.poff[v] = v <= L.n_views ? L.poff[v] : L.Dp;
  }
  dim3 block(32, 8);
  dim3 grid((unsigned)ceil_div(L.D, 32), (unsigned)ceil_div(L.D, 8));
  covariance_kernel<Tout><<<grid, block, 0, stream>>>(p, moments, n_total, center, C, ldc, mean); count_launches(1);
  CCAB_CUDA(cudaGetLastError());
  return 0;
}

template int covariance_from_moments<float>(const ColumnLayout&, const double*, double, int, float*, int64_t, float*,
                                            cudaStream_t);
template int covariance_from_moments<double>(const ColumnLayout&, const double*, double, int, double*, int64_t,
                                             double*, cudaStream_t);

}  // namespace ccab
