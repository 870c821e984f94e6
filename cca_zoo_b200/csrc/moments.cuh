// Block-moment stage (kernels K1/K2 of DESIGN.md): M = [X1..Xm]^T [X1..Xm], s = 1^T X.
#pragma once
#include <cuda_bf16.h>
#include <cuda_fp16.h>

#include "common.cuh"

namespace ccab {

constexpr int kMaxViews = 8;
constexpr int kBlk = 128;        // column-block width of the padded tile space
constexpr int kMaxBlocks = 128;  // D_padded <= 16384

// Column layout shared by every kernel of the moment stage.  Each view's columns are padded to a
// multiple of 128 in *tile space*; "compact" is the hstacked view order the reference uses
// (cca_zoo/linear/_mcca.py:150: np.hstack(views)).
struct ColumnLayout {
  int n_views;
  int nblocks;               // total 128-column blocks
  int D;                     // compact width  = sum(dims)
  int Dp;                    // padded width   = nblocks * 128
  int dims[kMaxViews];       // view widths
  int coff[kMaxViews + 1];   // compact offset of each view
  int poff[kMaxViews + 1];   // padded  offset of each view
};

int make_layout(int n_views, const int64_t* dims, ColumnLayout* out);

// Arithmetic type of a view element: 16-bit views are converted on load and accumulated in fp32, and their pilot
// origin and shifted copy are fp32.
template <typename T>
struct Wide { using type = T; };
template <>
struct Wide<__nv_bfloat16> { using type = float; };
template <>
struct Wide<__half> { using type = float; };
template <typename T>
using wide_t = typename Wide<T>::type;

// --- launchers (all asynchronous on `stream`) -------------------------------------------------
// precision: 0 = TF32 single pass (wgmma), 1 = 3xTF32 split (wgmma), 2 = exact SIMT FMA,
//            3 = 3xTF32 with the two cross terms as bf16 MMAs (hi*hi in TF32): 2 instead of 3 units of tensor work,
//            the same split plan and passes as 1.
// dtype: CCAB_F32, CCAB_F64, CCAB_BF16 or CCAB_F16; every tensor precision of a 16-bit dtype is the 16-bit wgmma
// kernel (mode kModeBf16 / kModeF16 of moments_tf32).
size_t moments_workspace_bytes(int dtype, int precision, const ColumnLayout& L, int64_t n_rows);

// modes of moments_tf32 beyond the float32 precisions 0, 1 and 3: bf16 / fp16 views, one wgmma per k16 step (the
// products are exact in fp32), with the split plan and passes of the 3xTF32 modes
constexpr int kModeBf16 = 4, kModeF16 = 5;

int moments_tf32(const ColumnLayout& L, const void* const* views, const int64_t* lds, int64_t n_rows,
                 int mode /* 0, 1, 3, kModeBf16 or kModeF16 */, double* moments_out, void* ws, size_t ws_bytes,
                 cudaStream_t stream);

template <typename T>
int moments_simt(const ColumnLayout& L, const void* const* views, const int64_t* lds, int64_t n_rows,
                 double* moments_out, void* ws, size_t ws_bytes, cudaStream_t stream);

// moments (double[Dp*Dp + Dp], padded, upper block triangle) -> compact covariance + means
template <typename Tout>
int covariance_from_moments(const ColumnLayout& L, const double* moments, double n_total, int center,
                            Tout* C, int64_t ldc, Tout* mean, cudaStream_t stream);
// the same with the sample count read at n_dev[0] on the device (an all-reduced count; N < 2 gives inf / NaN entries)
template <typename Tout>
int covariance_from_moments_ndev(const ColumnLayout& L, const double* moments, const double* n_dev, int center,
                                 Tout* C, int64_t ldc, Tout* mean, cudaStream_t stream);

// exchange-step message: upper triangle of 128 x 128 blocks | column sums | n | reserved (all float64)
int64_t moments_packed_size(const ColumnLayout& L);
int moments_pack(const ColumnLayout& L, const double* moments, double n_local, double* packed, cudaStream_t stream);
int moments_unpack(const ColumnLayout& L, const double* packed, double* moments, cudaStream_t stream);

// Shifted accumulation: pilot statistics of the leading rows, Xs = X - x0, and the float64 correction that turns the
// moments of the shifted data back into raw moments (see moments.cu).
// x0 and Xs are wide_t<T>: float32 for 16-bit views.
template <typename T>
int column_pilot(const T* X, int64_t rows, int d, int64_t ld, wide_t<T>* x0, float* ratio_max, cudaStream_t stream);
template <typename T>
int shift_rows(const T* X, int64_t n, int d, int64_t ldx, const wide_t<T>* x0, wide_t<T>* Xs, int64_t lds,
               cudaStream_t stream);
int moments_unshift(const ColumnLayout& L, double* moments, const void* const* x0, int is_f64, double n,
                    cudaStream_t stream);

// Fused exchange step on symmetric memory (pack + in-switch reduction with multimem + unpack in ONE kernel).
// sym_local / sym_multicast: local and multicast address of a symmetric buffer of sym_doubles doubles
// (>= world * ceil(packed / world)); pads_dev: device array of the world signal-pad pointers (uint32, pad_slots
// entries each, zero-initialised once); epoch: 2 x the call counter, identical on all ranks, strictly increasing.
int moments_exchange_nvls(const ColumnLayout& L, double* moments, double n_local, double* sym_local,
                          double* sym_multicast, void* const* pads_dev, int rank, int world, int pad_slots,
                          int64_t sym_doubles, unsigned epoch, double* n_total_out, cudaStream_t stream);

// CUDA-event timing of the tensor-core moment kernel launch alone (for bench.py's roofline line)
void moments_profile_enable(int on);
float moments_profile_last_ms();

}  // namespace ccab
