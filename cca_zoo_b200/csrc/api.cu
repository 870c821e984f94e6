// C ABI of libccab200 (see include/ccab200.h).  Thin argument checking + dispatch; no exceptions
// leave this file.
#include "../../include/ccab200.h"

#include <cstdarg>
#include <cmath>
#include <cstring>
#include <atomic>
#include <exception>

#include "als.cuh"
#include "ccaloss.cuh"
#include "ccar3.cuh"
#include "cv.cuh"
#include "cholinv.cuh"
#include "common.cuh"
#include "gfa.cuh"
#include "kcca.cuh"
#include "dense.cuh"
#include "ey.cuh"
#include "fit.cuh"
#include "moments.cuh"
#include "syevj.cuh"
#include "syevj_small.cuh"
#include "tcca.cuh"
#include "tgemm.cuh"

namespace ccab {
static thread_local char g_err[512] = "";
void set_error(const char* fmt, ...) {
  va_list ap;
  va_start(ap, fmt);
  vsnprintf(g_err, sizeof(g_err), fmt, ap);
  va_end(ap);
}
static std::atomic<long> g_launches{0};
void count_launches(int n) { g_launches.fetch_add(n, std::memory_order_relaxed); }
long launch_count() { return g_launches.load(std::memory_order_relaxed); }
int cuda_fail(cudaError_t e, const char* what) {
  set_error("CUDA error %d (%s) at %s", (int)e, cudaGetErrorString(e), what);
  return (int)e;
}
}  // namespace ccab

using namespace ccab;

#define CCAB_TRY try {
#define CCAB_CATCH                                 \
  }                                                \
  catch (const std::exception& e) {                \
    set_error("internal exception: %s", e.what()); \
    return -100;                                   \
  }                                                \
  catch (...) {                                    \
    set_error("internal exception");               \
    return -100;                                   \
  }

static int require_device() {
  int dev = 0;
  cudaError_t e = cudaGetDevice(&dev);
  if (e != cudaSuccess) return cuda_fail(e, "cudaGetDevice (no CUDA device: libccab200 has no CPU fallback)");
  int major = 0;
  cudaDeviceGetAttribute(&major, cudaDevAttrComputeCapabilityMajor, dev);
  if (major != 9) {
    set_error("libccab200 is built for sm_90a (Hopper) only; device %d has compute capability major %d", dev, major);
    return -10;
  }
  return 0;
}

extern "C" {

int ccab_version(void) { return 100; }
int64_t ccab_launch_count(void) { return (int64_t)launch_count(); }
const char* ccab_last_error(void) { return g_err; }

int64_t ccab_moments_size(int n_views, const int64_t* dims) {
  ColumnLayout L;
  if (make_layout(n_views, dims, &L)) return -1;
  return (int64_t)L.Dp * L.Dp + L.Dp;
}
int64_t ccab_moments_padded_dim(int n_views, const int64_t* dims) {
  ColumnLayout L;
  if (make_layout(n_views, dims, &L)) return -1;
  return L.Dp;
}

size_t ccab_moments_workspace_bytes(int dtype, int precision, int n_views, const int64_t* dims, int64_t n_rows) {
  ColumnLayout L;
  if (make_layout(n_views, dims, &L)) return 0;
  return moments_workspace_bytes(dtype, precision, L, n_rows) + 512;
}

int ccab_moments(int dtype, int precision, int n_views, const void* const* views, const int64_t* dims,
                 const int64_t* lds, int64_t n_rows, double* moments, void* workspace, size_t workspace_bytes,
                 void* stream) {
  CCAB_TRY
  CCAB_CHECK_ARG(dtype == CCAB_F32 || dtype == CCAB_F64 || dtype == CCAB_BF16 || dtype == CCAB_F16, "bad dtype %d",
                 dtype);
  CCAB_CHECK_ARG(precision >= 0 && precision <= 3, "bad precision %d", precision);
  CCAB_CHECK_ARG(!(dtype == CCAB_F64 && precision != CCAB_PREC_EXACT),
                 "float64 inputs support CCAB_PREC_EXACT only (the TF32 tensor-core path has no f64 kind)");
  CCAB_CHECK_ARG(views && dims && lds && moments && workspace, "null pointer argument");
  ColumnLayout L;
  int rc = make_layout(n_views, dims, &L);
  if (rc) return rc;
  for (int v = 0; v < n_views; ++v) {
    CCAB_CHECK_ARG(views[v] != nullptr, "view %d is NULL", v);
    CCAB_CHECK_ARG(lds[v] >= dims[v], "lds[%d] < dims[%d]", v, v);
  }
  rc = require_device();
  if (rc) return rc;
  cudaStream_t s = static_cast<cudaStream_t>(stream);
  if (precision == CCAB_PREC_EXACT) {
    if (dtype == CCAB_F32) return moments_simt<float>(L, views, lds, n_rows, moments, workspace, workspace_bytes, s);
    if (dtype == CCAB_BF16)
      return moments_simt<__nv_bfloat16>(L, views, lds, n_rows, moments, workspace, workspace_bytes, s);
    if (dtype == CCAB_F16) return moments_simt<__half>(L, views, lds, n_rows, moments, workspace, workspace_bytes, s);
    return moments_simt<double>(L, views, lds, n_rows, moments, workspace, workspace_bytes, s);
  }
  // every tensor precision of a 16-bit dtype is the 16-bit wgmma kernel: its products are exact, nothing to split
  const int mode = dtype == CCAB_BF16 ? kModeBf16 : dtype == CCAB_F16 ? kModeF16 : precision;
  return moments_tf32(L, views, lds, n_rows, mode, moments, workspace, workspace_bytes, s);
  CCAB_CATCH
}

int64_t ccab_moments_packed_size(int n_views, const int64_t* dims) {
  ColumnLayout L;
  if (make_layout(n_views, dims, &L)) return -1;
  return moments_packed_size(L);
}

int ccab_moments_pack(int n_views, const int64_t* dims, const double* moments, double n_local, double* packed,
                      void* stream) {
  CCAB_TRY
  CCAB_CHECK_ARG(dims && moments && packed, "null pointer argument");
  ColumnLayout L;
  int rc = make_layout(n_views, dims, &L);
  if (rc) return rc;
  rc = require_device();
  if (rc) return rc;
  return moments_pack(L, moments, n_local, packed, static_cast<cudaStream_t>(stream));
  CCAB_CATCH
}

int ccab_moments_unpack(int n_views, const int64_t* dims, const double* packed, double* moments, void* stream) {
  CCAB_TRY
  CCAB_CHECK_ARG(dims && moments && packed, "null pointer argument");
  ColumnLayout L;
  int rc = make_layout(n_views, dims, &L);
  if (rc) return rc;
  rc = require_device();
  if (rc) return rc;
  return moments_unpack(L, packed, moments, static_cast<cudaStream_t>(stream));
  CCAB_CATCH
}

int ccab_moments_exchange_nvls(int n_views, const int64_t* dims, double* moments, double n_local, double* sym_local,
                               double* sym_multicast, void* const* signal_pads_dev, int rank, int world,
                               int pad_slots, int64_t sym_doubles, unsigned epoch, double* n_total_out, void* stream) {
  CCAB_TRY
  CCAB_CHECK_ARG(dims && moments, "null pointer argument");
  ColumnLayout L;
  int rc = make_layout(n_views, dims, &L);
  if (rc) return rc;
  rc = require_device();
  if (rc) return rc;
  return moments_exchange_nvls(L, moments, n_local, sym_local, sym_multicast, signal_pads_dev, rank, world, pad_slots,
                               sym_doubles, epoch, n_total_out, static_cast<cudaStream_t>(stream));
  CCAB_CATCH
}

int ccab_column_pilot(int dtype, const void* X, int64_t rows, int d, int64_t ld, void* x0, float* ratio_max_dev,
                      void* stream) {
  CCAB_TRY
  CCAB_CHECK_ARG(dtype == CCAB_F32 || dtype == CCAB_F64 || dtype == CCAB_BF16 || dtype == CCAB_F16, "bad dtype %d",
                 dtype);
  CCAB_CHECK_ARG(X && x0 && ratio_max_dev, "null pointer argument");
  int rc = require_device();
  if (rc) return rc;
  cudaStream_t s = static_cast<cudaStream_t>(stream);
  if (dtype == CCAB_F32)
    return column_pilot<float>(static_cast<const float*>(X), rows, d, ld, static_cast<float*>(x0), ratio_max_dev, s);
  if (dtype == CCAB_BF16)
    return column_pilot<__nv_bfloat16>(static_cast<const __nv_bfloat16*>(X), rows, d, ld, static_cast<float*>(x0),
                                       ratio_max_dev, s);
  if (dtype == CCAB_F16)
    return column_pilot<__half>(static_cast<const __half*>(X), rows, d, ld, static_cast<float*>(x0), ratio_max_dev, s);
  return column_pilot<double>(static_cast<const double*>(X), rows, d, ld, static_cast<double*>(x0), ratio_max_dev, s);
  CCAB_CATCH
}

int ccab_shift_rows(int dtype, const void* X, int64_t n, int d, int64_t ldx, const void* x0, void* Xs, int64_t lds,
                    void* stream) {
  CCAB_TRY
  CCAB_CHECK_ARG(dtype == CCAB_F32 || dtype == CCAB_F64 || dtype == CCAB_BF16 || dtype == CCAB_F16, "bad dtype %d",
                 dtype);
  CCAB_CHECK_ARG(X && x0 && Xs && ldx >= d && lds >= d, "bad argument");
  int rc = require_device();
  if (rc) return rc;
  cudaStream_t s = static_cast<cudaStream_t>(stream);
  if (dtype == CCAB_F32)
    return shift_rows<float>(static_cast<const float*>(X), n, d, ldx, static_cast<const float*>(x0),
                             static_cast<float*>(Xs), lds, s);
  if (dtype == CCAB_BF16)
    return shift_rows<__nv_bfloat16>(static_cast<const __nv_bfloat16*>(X), n, d, ldx, static_cast<const float*>(x0),
                                     static_cast<float*>(Xs), lds, s);
  if (dtype == CCAB_F16)
    return shift_rows<__half>(static_cast<const __half*>(X), n, d, ldx, static_cast<const float*>(x0),
                              static_cast<float*>(Xs), lds, s);
  return shift_rows<double>(static_cast<const double*>(X), n, d, ldx, static_cast<const double*>(x0),
                            static_cast<double*>(Xs), lds, s);
  CCAB_CATCH
}

int ccab_moments_unshift(int dtype, int n_views, const int64_t* dims, double* moments, const void* const* x0,
                         double n_rows, void* stream) {
  CCAB_TRY
  CCAB_CHECK_ARG(dtype == CCAB_F32 || dtype == CCAB_F64, "bad dtype %d", dtype);
  CCAB_CHECK_ARG(dims && moments && x0, "null pointer argument");
  ColumnLayout L;
  int rc = make_layout(n_views, dims, &L);
  if (rc) return rc;
  rc = require_device();
  if (rc) return rc;
  return moments_unshift(L, moments, x0, dtype == CCAB_F64, n_rows, static_cast<cudaStream_t>(stream));
  CCAB_CATCH
}

int ccab_covariance(int out_dtype, int n_views, const int64_t* dims, const double* moments, double n_total,
                    int center, void* C, int64_t ldc, void* mean, void* stream) {
  CCAB_TRY
  CCAB_CHECK_ARG(out_dtype == CCAB_F32 || out_dtype == CCAB_F64, "bad dtype %d", out_dtype);
  CCAB_CHECK_ARG(dims && moments && C, "null pointer argument");
  ColumnLayout L;
  int rc = make_layout(n_views, dims, &L);
  if (rc) return rc;
  rc = require_device();
  if (rc) return rc;
  cudaStream_t s = static_cast<cudaStream_t>(stream);
  if (out_dtype == CCAB_F32)
    return covariance_from_moments<float>(L, moments, n_total, center, static_cast<float*>(C), ldc,
                                          static_cast<float*>(mean), s);
  return covariance_from_moments<double>(L, moments, n_total, center, static_cast<double*>(C), ldc,
                                         static_cast<double*>(mean), s);
  CCAB_CATCH
}

int ccab_covariance_ndev(int out_dtype, int n_views, const int64_t* dims, const double* moments, const double* n_dev,
                         int center, void* C, int64_t ldc, void* mean, void* stream) {
  CCAB_TRY
  CCAB_CHECK_ARG(out_dtype == CCAB_F32 || out_dtype == CCAB_F64, "bad dtype %d", out_dtype);
  CCAB_CHECK_ARG(dims && moments && n_dev && C, "null pointer argument");
  ColumnLayout L;
  int rc = make_layout(n_views, dims, &L);
  if (rc) return rc;
  rc = require_device();
  if (rc) return rc;
  cudaStream_t s = static_cast<cudaStream_t>(stream);
  if (out_dtype == CCAB_F32)
    return covariance_from_moments_ndev<float>(L, moments, n_dev, center, static_cast<float*>(C), ldc,
                                               static_cast<float*>(mean), s);
  return covariance_from_moments_ndev<double>(L, moments, n_dev, center, static_cast<double*>(C), ldc,
                                              static_cast<double*>(mean), s);
  CCAB_CATCH
}

size_t ccab_syevj_workspace_bytes(int dtype, int n, int batch) {
  if (n < 1 || batch < 1) return 0;
  return dtype == CCAB_F32 ? jacobi_workspace_bytes<float>(n, n, batch) : jacobi_workspace_bytes<double>(n, n, batch);
}

}  // extern "C"

template <typename T>
static int syevj_t(int n, int batch, const void* A, int64_t lda, int64_t batch_stride, double shift, void* evals,
                   void* evecs_t, int64_t ldv, int* info, float* info_offdiag, void* ws, size_t wsb, cudaStream_t s) {
  JacobiArgs<T> a;
  memset(&a, 0, sizeof(a));
  a.in = static_cast<const T*>(A);
  a.ld_in = lda;
  a.batch_stride_in = batch_stride;
  a.colmajor_in = 1;  // symmetric: either reading order is the same matrix, this one is coalesced
  a.m = n;
  a.n = n;
  a.batch = batch;
  a.svd_mode = 0;
  a.shift = shift;
  a.out_vals = static_cast<T*>(evals);
  a.vals_stride = n;
  a.out_right = static_cast<T*>(evecs_t);
  a.ld_right = ldv;
  a.right_stride = (int64_t)n * ldv;
  a.info = info;
  a.final_offdiag = info_offdiag;
  return jacobi_solve<T>(a, ws, wsb, s);
}

extern "C" {

int ccab_syevj(int dtype, int n, int batch, const void* A, int64_t lda, int64_t batch_stride, double shift,
               void* evals, void* evecs_t, int64_t ldv, int* info, float* info_offdiag, void* workspace,
               size_t workspace_bytes, void* stream) {
  CCAB_TRY
  CCAB_CHECK_ARG(dtype == CCAB_F32 || dtype == CCAB_F64, "bad dtype %d", dtype);
  CCAB_CHECK_ARG(n >= 1 && batch >= 1, "bad shape n=%d batch=%d", n, batch);
  CCAB_CHECK_ARG(A && workspace, "null pointer argument");
  CCAB_CHECK_ARG(lda >= n && (evecs_t == nullptr || ldv >= n), "leading dimension too small");
  int rc = require_device();
  if (rc) return rc;
  cudaStream_t s = static_cast<cudaStream_t>(stream);
  if (dtype == CCAB_F32)
    return syevj_t<float>(n, batch, A, lda, batch_stride, shift, evals, evecs_t, ldv, info, info_offdiag, workspace,
                          workspace_bytes, s);
  return syevj_t<double>(n, batch, A, lda, batch_stride, shift, evals, evecs_t, ldv, info, info_offdiag, workspace,
                         workspace_bytes, s);
  CCAB_CATCH
}

int ccab_syevj_small(int dtype, int n, int batch, const void* A, int64_t lda, int64_t stride_a, void* evals,
                     void* evecs_t, int64_t ldv, int* info_dev, void* stream) {
  CCAB_TRY
  CCAB_CHECK_ARG(dtype == CCAB_F32 || dtype == CCAB_F64, "bad dtype %d", dtype);
  CCAB_CHECK_ARG(A != nullptr, "null pointer argument");
  int rc = require_device();
  if (rc) return rc;
  cudaStream_t s = static_cast<cudaStream_t>(stream);
  if (dtype == CCAB_F32)
    return syevj_small<float>(n, batch, static_cast<const float*>(A), lda, stride_a, static_cast<float*>(evals), n,
                              static_cast<float*>(evecs_t), ldv, (int64_t)n * ldv, info_dev, s);
  return syevj_small<double>(n, batch, static_cast<const double*>(A), lda, stride_a, static_cast<double*>(evals), n,
                             static_cast<double*>(evecs_t), ldv, (int64_t)n * ldv, info_dev, s);
  CCAB_CATCH
}

size_t ccab_gesvj_workspace_bytes(int dtype, int m, int n) {
  if (n < 1 || m < 1) return 0;
  return dtype == CCAB_F32 ? jacobi_workspace_bytes<float>(m, n, 1) : jacobi_workspace_bytes<double>(m, n, 1);
}

}  // extern "C"

template <typename T>
static int gesvj_t(int m, int n, const void* A, int64_t lda, void* sigma, void* right_t, int64_t ldr, void* left_t,
                   int64_t ldl, int* info, float* info_offdiag, void* ws, size_t wsb, cudaStream_t s) {
  JacobiArgs<T> a;
  memset(&a, 0, sizeof(a));
  a.in = static_cast<const T*>(A);
  a.ld_in = lda;
  a.batch_stride_in = 0;
  a.colmajor_in = 1;
  a.m = m;
  a.n = n;
  a.batch = 1;
  a.svd_mode = 1;
  a.out_vals = static_cast<T*>(sigma);
  a.vals_stride = n;
  a.out_right = static_cast<T*>(right_t);
  a.ld_right = ldr;
  a.out_left = static_cast<T*>(left_t);
  a.ld_left = ldl;
  a.info = info;
  a.final_offdiag = info_offdiag;
  return jacobi_solve<T>(a, ws, wsb, s);
}

extern "C" {

int ccab_gesvj(int dtype, int m, int n, const void* A, int64_t lda, void* sigma, void* right_t, int64_t ldr,
               void* left_t, int64_t ldl, int* info, float* info_offdiag, void* workspace, size_t workspace_bytes,
               void* stream) {
  CCAB_TRY
  CCAB_CHECK_ARG(dtype == CCAB_F32 || dtype == CCAB_F64, "bad dtype %d", dtype);
  CCAB_CHECK_ARG(m >= 1 && n >= 1, "bad shape m=%d n=%d", m, n);
  CCAB_CHECK_ARG(A && workspace, "null pointer argument");
  CCAB_CHECK_ARG(lda >= m, "lda < m");
  CCAB_CHECK_ARG((right_t == nullptr || ldr >= n) && (left_t == nullptr || ldl >= m), "leading dimension too small");
  int rc = require_device();
  if (rc) return rc;
  cudaStream_t s = static_cast<cudaStream_t>(stream);
  if (dtype == CCAB_F32)
    return gesvj_t<float>(m, n, A, lda, sigma, right_t, ldr, left_t, ldl, info, info_offdiag, workspace,
                          workspace_bytes, s);
  return gesvj_t<double>(m, n, A, lda, sigma, right_t, ldr, left_t, ldl, info, info_offdiag, workspace,
                         workspace_bytes, s);
  CCAB_CATCH
}

int ccab_gemm(int dtype, int transa, int transb, int m, int n, int k, double alpha, const void* A, int64_t lda,
              const void* B, int64_t ldb, double beta, void* C, int64_t ldc, void* stream) {
  CCAB_TRY
  CCAB_CHECK_ARG(dtype == CCAB_F32 || dtype == CCAB_F64, "bad dtype %d", dtype);
  CCAB_CHECK_ARG(A && B && C, "null pointer argument");
  int rc = require_device();
  if (rc) return rc;
  cudaStream_t s = static_cast<cudaStream_t>(stream);
  if (dtype == CCAB_F32) {   // tensor pipe (wgmma, 3xTF32) when TMA can address the operands, FMA tiles otherwise
    GemmArgs<float> g;
    g.transa = transa; g.transb = transb; g.m = m; g.n = n; g.k = k; g.alpha = (float)alpha; g.beta = (float)beta;
    g.A = static_cast<const float*>(A); g.lda = lda; g.B = static_cast<const float*>(B); g.ldb = ldb;
    g.C = static_cast<float*>(C); g.ldc = ldc;
    return xgemm<float>(g, s);
  }
  GemmArgs<double> g;   // fp64 tensor pipe (mma.sync m8n8k4.f64)
  g.transa = transa; g.transb = transb; g.m = m; g.n = n; g.k = k; g.alpha = alpha; g.beta = beta;
  g.A = static_cast<const double*>(A); g.lda = lda; g.B = static_cast<const double*>(B); g.ldb = ldb;
  g.C = static_cast<double*>(C); g.ldc = ldc;
  return xgemm<double>(g, s);
  CCAB_CATCH
}

int ccab_gemm_tc(int transa, int transb, int m, int n, int k, double alpha, const void* A, int64_t lda,
                 int64_t stride_a, const void* B, int64_t ldb, int64_t stride_b, double beta, void* C, int64_t ldc,
                 int64_t stride_c, void* Ct, int64_t ldct, int64_t stride_ct, int batch, int lower_only,
                 void* stream) {
  CCAB_TRY
  CCAB_CHECK_ARG(A && B && (C || Ct), "null pointer argument");
  CCAB_CHECK_ARG(m >= 1 && n >= 1 && k >= 1 && batch >= 1, "bad shape m=%d n=%d k=%d batch=%d", m, n, k, batch);
  CCAB_CHECK_ARG((!C || ldc >= n) && (!Ct || ldct >= m), "output leading dimension too small");
  int rc = require_device();
  if (rc) return rc;
  TgemmArgs a;
  a.transa = transa;
  a.transb = transb;
  a.m = m;
  a.n = n;
  a.k = k;
  a.alpha = (float)alpha;
  a.beta = (float)beta;
  a.A = static_cast<const float*>(A);
  a.lda = lda;
  a.strideA = stride_a;
  a.B = static_cast<const float*>(B);
  a.ldb = ldb;
  a.strideB = stride_b;
  a.C = static_cast<float*>(C);
  a.ldc = ldc;
  a.strideC = stride_c;
  a.Ct = static_cast<float*>(Ct);
  a.ldct = ldct;
  a.strideCt = stride_ct;
  a.batch = batch;
  a.lower_only = lower_only;
  return tgemm(a, static_cast<cudaStream_t>(stream));
  CCAB_CATCH
}

int ccab_whiten_rows(int dtype, int d, const void* lam, const void* Vt, int64_t ldv, double c, double floor_add,
                     const void* floor_dev, double scale, double rank_tol, int max_rank, double lam_floor, void* Wt,
                     int64_t ldw, void* g_out, int* rank_out, void* stream) {
  CCAB_TRY
  CCAB_CHECK_ARG(dtype == CCAB_F32 || dtype == CCAB_F64, "bad dtype %d", dtype);
  CCAB_CHECK_ARG(lam && Vt && Wt, "null pointer argument");
  CCAB_CHECK_ARG(scale > 0.0, "scale must be positive");
  int rc = require_device();
  if (rc) return rc;
  cudaStream_t s = static_cast<cudaStream_t>(stream);
  if (dtype == CCAB_F32)
    return whiten_rows<float>(d, static_cast<const float*>(lam), static_cast<const float*>(Vt), ldv, c, floor_add,
                              static_cast<const float*>(floor_dev), scale, rank_tol, max_rank, lam_floor,
                              static_cast<float*>(Wt), ldw, static_cast<float*>(g_out), rank_out, s);
  return whiten_rows<double>(d, static_cast<const double*>(lam), static_cast<const double*>(Vt), ldv, c, floor_add,
                             static_cast<const double*>(floor_dev), scale, rank_tol, max_rank, lam_floor,
                             static_cast<double*>(Wt), ldw, static_cast<double*>(g_out), rank_out, s);
  CCAB_CATCH
}

int ccab_ccaloss_small(int dtype, int d1, int d2, const void* C, int64_t ldc, double eps, void* loss, void* G11,
                       void* P, void* G22, void* min_pivot, void* stream) {
  CCAB_TRY
  CCAB_CHECK_ARG(dtype == CCAB_F32 || dtype == CCAB_F64, "bad dtype %d", dtype);
  CCAB_CHECK_ARG(C && loss && G11 && P && G22 && min_pivot, "null pointer argument");
  int rc = require_device();
  if (rc) return rc;
  cudaStream_t s = static_cast<cudaStream_t>(stream);
  if (dtype == CCAB_F32)
    return ccaloss_small<float>(static_cast<const float*>(C), ldc, d1, d2, eps, static_cast<float*>(loss),
                                static_cast<float*>(G11), static_cast<float*>(P), static_cast<float*>(G22),
                                static_cast<float*>(min_pivot), s);
  return ccaloss_small<double>(static_cast<const double*>(C), ldc, d1, d2, eps, static_cast<double*>(loss),
                               static_cast<double*>(G11), static_cast<double*>(P), static_cast<double*>(G22),
                               static_cast<double*>(min_pivot), s);
  CCAB_CATCH
}

size_t ccab_potrf_inv_workspace_bytes(int dtype, int n, int batch) {
  if (n < 1 || batch < 1) return 0;
  return dtype == CCAB_F32 ? potrf_inv_workspace_bytes<float>(n, batch) : potrf_inv_workspace_bytes<double>(n, batch);
}

int ccab_potrf_inv(int dtype, int n, int batch, void* A, int64_t lda, int64_t stride_a, void* Linv, int64_t ldi,
                   int64_t stride_i, double pivot_tol, int* info_dev, void* workspace, size_t workspace_bytes,
                   void* stream) {
  CCAB_TRY
  CCAB_CHECK_ARG(dtype == CCAB_F32 || dtype == CCAB_F64, "bad dtype %d", dtype);
  CCAB_CHECK_ARG(A && Linv && info_dev && workspace, "null pointer argument");
  int rc = require_device();
  if (rc) return rc;
  cudaStream_t s = static_cast<cudaStream_t>(stream);
  if (dtype == CCAB_F32)
    return potrf_inv<float>(n, batch, static_cast<float*>(A), lda, stride_a, static_cast<float*>(Linv), ldi, stride_i,
                            pivot_tol, nullptr, info_dev, workspace, workspace_bytes, s);
  return potrf_inv<double>(n, batch, static_cast<double*>(A), lda, stride_a, static_cast<double*>(Linv), ldi, stride_i,
                           pivot_tol, nullptr, info_dev, workspace, workspace_bytes, s);
  CCAB_CATCH
}

size_t ccab_rcca_fit_workspace_bytes(int dtype, const int64_t* dims, int k, int p) {
  if (!dims || dims[0] < 1 || dims[1] < 1 || (dtype != CCAB_F32 && dtype != CCAB_F64)) return 0;
  return dtype == CCAB_F32 ? rcca_fit_workspace_bytes<float>((int)dims[0], (int)dims[1], k, p)
                           : rcca_fit_workspace_bytes<double>((int)dims[0], (int)dims[1], k, p);
}

int ccab_rcca_fit_result_layout(int dtype, const int64_t* dims, int k, int p, int64_t* offsets) {
  CCAB_TRY
  CCAB_CHECK_ARG(dims && offsets && dims[0] >= 1 && dims[1] >= 1 && k >= 1 && p >= k, "bad argument");
  if (dtype == CCAB_F32) rcca_fit_result_layout<float>((int)dims[0], (int)dims[1], k, p, offsets);
  else rcca_fit_result_layout<double>((int)dims[0], (int)dims[1], k, p, offsets);
  return 0;
  CCAB_CATCH
}

int ccab_rcca_fit(int dtype, const int64_t* dims, const double* moments, const double* n_total_dev, double n_total,
                  int center, const double* c, int k, int p, int iters, void* result, size_t result_bytes,
                  void* workspace, size_t workspace_bytes, void* stream) {
  CCAB_TRY
  CCAB_CHECK_ARG(dtype == CCAB_F32 || dtype == CCAB_F64, "bad dtype %d", dtype);
  CCAB_CHECK_ARG(dims && moments && c && result && workspace, "null pointer argument");
  ColumnLayout L;
  int rc = make_layout(2, dims, &L);
  if (rc) return rc;
  rc = require_device();
  if (rc) return rc;
  cudaStream_t s = static_cast<cudaStream_t>(stream);
  if (dtype == CCAB_F32)
    return rcca_fit<float>(L, moments, n_total_dev, n_total, center, c, k, p, iters, result, result_bytes, workspace,
                           workspace_bytes, s);
  return rcca_fit<double>(L, moments, n_total_dev, n_total, center, c, k, p, iters, result, result_bytes, workspace,
                          workspace_bytes, s);
  CCAB_CATCH
}

size_t ccab_ccaloss_workspace_bytes(int dtype, int precision, int d1, int d2, int64_t n) {
  int64_t dims[2] = {d1, d2};
  ColumnLayout L;
  if (make_layout(2, dims, &L)) return 0;
  if (dtype == CCAB_F64) precision = CCAB_PREC_EXACT;
  return dtype == CCAB_F32 ? ccaloss_workspace_bytes<float>(L, n, precision)
                           : ccaloss_workspace_bytes<double>(L, n, precision);
}

int ccab_ccaloss_fwd(int dtype, int precision, const void* z1, int64_t ld1, const void* z2, int64_t ld2, int64_t n,
                     int d1, int d2, double eps, void* loss, void* saved, int* flags_dev, void* workspace,
                     size_t workspace_bytes, void* stream) {
  CCAB_TRY
  CCAB_CHECK_ARG(dtype == CCAB_F32 || dtype == CCAB_F64, "bad dtype %d", dtype);
  CCAB_CHECK_ARG(precision >= 0 && precision <= 3, "bad precision %d", precision);
  CCAB_CHECK_ARG(z1 && z2 && loss && saved && flags_dev && workspace, "null pointer argument");
  CCAB_CHECK_ARG(ld1 >= d1 && ld2 >= d2, "leading dimension too small");
  int64_t dims[2] = {d1, d2};
  ColumnLayout L;
  int rc = make_layout(2, dims, &L);
  if (rc) return rc;
  rc = require_device();
  if (rc) return rc;
  cudaStream_t s = static_cast<cudaStream_t>(stream);
  if (dtype == CCAB_F32)
    return ccaloss_forward<float>(L, precision, z1, ld1, z2, ld2, n, eps, static_cast<float*>(loss),
                                  static_cast<float*>(saved), flags_dev, workspace, workspace_bytes, s);
  return ccaloss_forward<double>(L, CCAB_PREC_EXACT, z1, ld1, z2, ld2, n, eps, static_cast<double*>(loss),
                                 static_cast<double*>(saved), flags_dev, workspace, workspace_bytes, s);
  CCAB_CATCH
}

int ccab_ccaloss_bwd(int dtype, const void* z1, int64_t ld1, const void* z2, int64_t ld2, int64_t n, int d1, int d2,
                     const void* saved, const void* grad_out, void* g1, int64_t ldg1, void* g2, int64_t ldg2,
                     void* stream) {
  CCAB_TRY
  CCAB_CHECK_ARG(dtype == CCAB_F32 || dtype == CCAB_F64, "bad dtype %d", dtype);
  CCAB_CHECK_ARG(z1 && z2 && saved && g1 && g2, "null pointer argument");
  CCAB_CHECK_ARG(ld1 >= d1 && ld2 >= d2 && ldg1 >= d1 && ldg2 >= d2, "leading dimension too small");
  int rc = require_device();
  if (rc) return rc;
  cudaStream_t s = static_cast<cudaStream_t>(stream);
  if (dtype == CCAB_F32)
    return ccaloss_backward<float>(d1, d2, static_cast<const float*>(z1), ld1, static_cast<const float*>(z2), ld2, n,
                                   static_cast<const float*>(saved), static_cast<const float*>(grad_out),
                                   static_cast<float*>(g1), ldg1, static_cast<float*>(g2), ldg2, s);
  return ccaloss_backward<double>(d1, d2, static_cast<const double*>(z1), ld1, static_cast<const double*>(z2), ld2, n,
                                  static_cast<const double*>(saved), static_cast<const double*>(grad_out),
                                  static_cast<double*>(g1), ldg1, static_cast<double*>(g2), ldg2, s);
  CCAB_CATCH
}

size_t ccab_ccaloss_fwd_moments_workspace_bytes(int dtype, int d1, int d2) {
  int64_t dims[2] = {d1, d2};
  ColumnLayout L;
  if (make_layout(2, dims, &L)) return 0;
  return dtype == CCAB_F32 ? ccaloss_fwd_moments_workspace_bytes<float>(L) : ccaloss_fwd_moments_workspace_bytes<double>(L);
}

int ccab_ccaloss_fwd_moments(int dtype, int d1, int d2, const double* moments, const double* n_dev, double eps,
                             void* loss, void* saved, int* flags_dev, void* workspace, size_t workspace_bytes,
                             void* stream) {
  CCAB_TRY
  CCAB_CHECK_ARG(dtype == CCAB_F32 || dtype == CCAB_F64, "bad dtype %d", dtype);
  CCAB_CHECK_ARG(moments && n_dev && loss && saved && flags_dev && workspace, "null pointer argument");
  int64_t dims[2] = {d1, d2};
  ColumnLayout L;
  int rc = make_layout(2, dims, &L);
  if (rc) return rc;
  rc = require_device();
  if (rc) return rc;
  cudaStream_t s = static_cast<cudaStream_t>(stream);
  if (dtype == CCAB_F32)
    return ccaloss_forward_moments<float>(L, moments, n_dev, eps, static_cast<float*>(loss), static_cast<float*>(saved),
                                          flags_dev, workspace, workspace_bytes, s);
  return ccaloss_forward_moments<double>(L, moments, n_dev, eps, static_cast<double*>(loss),
                                         static_cast<double*>(saved), flags_dev, workspace, workspace_bytes, s);
  CCAB_CATCH
}

int ccab_ccaloss_bwd_global(int dtype, const void* z1, int64_t ld1, const void* z2, int64_t ld2, int64_t n_local, int d1,
                            int d2, const void* saved, const void* grad_out, void* g1, int64_t ldg1, void* g2,
                            int64_t ldg2, void* stream) {
  CCAB_TRY
  CCAB_CHECK_ARG(dtype == CCAB_F32 || dtype == CCAB_F64, "bad dtype %d", dtype);
  CCAB_CHECK_ARG(saved && (n_local == 0 || (z1 && z2 && g1 && g2)), "null pointer argument");
  CCAB_CHECK_ARG(ld1 >= d1 && ld2 >= d2 && ldg1 >= d1 && ldg2 >= d2, "leading dimension too small");
  int rc = require_device();
  if (rc) return rc;
  cudaStream_t s = static_cast<cudaStream_t>(stream);
  if (dtype == CCAB_F32)
    return ccaloss_backward_global<float>(d1, d2, static_cast<const float*>(z1), ld1, static_cast<const float*>(z2),
                                          ld2, n_local, static_cast<const float*>(saved),
                                          static_cast<const float*>(grad_out), static_cast<float*>(g1), ldg1,
                                          static_cast<float*>(g2), ldg2, s);
  return ccaloss_backward_global<double>(d1, d2, static_cast<const double*>(z1), ld1, static_cast<const double*>(z2),
                                         ld2, n_local, static_cast<const double*>(saved),
                                         static_cast<const double*>(grad_out), static_cast<double*>(g1), ldg1,
                                         static_cast<double*>(g2), ldg2, s);
  CCAB_CATCH
}

size_t ccab_mcca_fit_workspace_bytes(int dtype, int n_views, const int64_t* dims, int k, int p) {
  ColumnLayout L;
  if (!dims || make_layout(n_views, dims, &L) || (dtype != CCAB_F32 && dtype != CCAB_F64)) return 0;
  return dtype == CCAB_F32 ? mcca_fit_workspace_bytes<float>(L, k, p) : mcca_fit_workspace_bytes<double>(L, k, p);
}

int ccab_mcca_fit_result_layout(int dtype, int n_views, const int64_t* dims, int k, int p, int64_t* offsets) {
  CCAB_TRY
  CCAB_CHECK_ARG(dims && offsets && k >= 1 && p >= k, "bad argument");
  ColumnLayout L;
  int rc = make_layout(n_views, dims, &L);
  if (rc) return rc;
  if (dtype == CCAB_F32) mcca_fit_result_layout<float>(L, k, p, offsets);
  else mcca_fit_result_layout<double>(L, k, p, offsets);
  return 0;
  CCAB_CATCH
}

int ccab_mcca_fit(int dtype, int n_views, const int64_t* dims, const double* moments, const double* n_total_dev,
                  double n_total, int center, const double* c, double eps, int k, int p, int iters, void* result,
                  size_t result_bytes, void* workspace, size_t workspace_bytes, void* stream) {
  CCAB_TRY
  CCAB_CHECK_ARG(dtype == CCAB_F32 || dtype == CCAB_F64, "bad dtype %d", dtype);
  CCAB_CHECK_ARG(dims && moments && c && result && workspace, "null pointer argument");
  ColumnLayout L;
  int rc = make_layout(n_views, dims, &L);
  if (rc) return rc;
  rc = require_device();
  if (rc) return rc;
  cudaStream_t s = static_cast<cudaStream_t>(stream);
  if (dtype == CCAB_F32)
    return mcca_fit<float>(L, moments, n_total_dev, n_total, center, c, eps, k, p, iters, result, result_bytes,
                           workspace, workspace_bytes, s);
  return mcca_fit<double>(L, moments, n_total_dev, n_total, center, c, eps, k, p, iters, result, result_bytes, workspace,
                          workspace_bytes, s);
  CCAB_CATCH
}

size_t ccab_als_fit_workspace_bytes(int n_views, const int64_t* dims) {
  ColumnLayout L;
  if (!dims || n_views < 2 || make_layout(n_views, dims, &L)) return 0;
  return als_fit_workspace_bytes(L, false);
}

size_t ccab_als_regression_workspace_bytes(int n_views, const int64_t* dims) {
  ColumnLayout L;
  if (!dims || n_views < 2 || make_layout(n_views, dims, &L)) return 0;
  return als_fit_workspace_bytes(L, true);
}

int ccab_als_fit(int kind, int n_views, const int64_t* dims, const double* G, double g_scale, double n_samples,
                 const double* params, double mu, const double* init, int k, int max_iter, double tol, double* W_out,
                 int* iters_out, void* workspace, size_t workspace_bytes, void* stream) {
  CCAB_TRY
  CCAB_CHECK_ARG(kind >= CCAB_ALS_PLS && kind <= CCAB_ALS_IPLS, "bad ALS kind %d", kind);
  CCAB_CHECK_ARG(n_views >= 2, "the ALS estimators need at least 2 views, got %d", n_views);
  CCAB_CHECK_ARG(dims && G && init && W_out && iters_out && workspace, "null pointer argument");
  CCAB_CHECK_ARG(kind == CCAB_ALS_PLS || params, "params is NULL");
  CCAB_CHECK_ARG(k >= 1 && max_iter >= 0, "bad k %d / max_iter %d", k, max_iter);
  CCAB_CHECK_ARG(kind != CCAB_ALS_ADMM || (mu > 0.0 && n_samples > 0.0), "ADMM needs mu > 0 and n_samples > 0");
  ColumnLayout L;
  int rc = make_layout(n_views, dims, &L);
  if (rc) return rc;
  const bool reg = kind == CCAB_ALS_ELASTIC || kind == CCAB_ALS_IPLS;
  for (int v = 0; reg && v < n_views; ++v) {
    const double alpha = params[2 * v], l1 = params[2 * v + 1];
    CCAB_CHECK_ARG(alpha >= 0.0 && alpha < INFINITY, "alpha[%d] = %g is not a finite non-negative number", v, alpha);
    CCAB_CHECK_ARG(l1 >= 0.0 && l1 <= 1.0, "l1_ratio[%d] = %g is not in [0, 1]", v, l1);
    CCAB_CHECK_ARG(dims[v] <= 2048, "view %d has %lld features; ElasticCCA / SCCA_IPLS take at most 2048 per view", v,
                   (long long)dims[v]);
  }
  CCAB_CHECK_ARG(!reg || n_samples > 0.0, "ElasticCCA / SCCA_IPLS need n_samples > 0");
  CCAB_CHECK_ARG(!reg || (mu >= 0.0 && mu < 1.0), "the eigenvalue cut mu = %g of ElasticCCA / SCCA_IPLS is not in [0, 1)",
                 mu);
  for (int v = 0; kind != CCAB_ALS_PLS && !reg && v < n_views; ++v) {
    CCAB_CHECK_ARG(params[v] >= 0.0, "params[%d] = %g is negative", v, params[v]);
    CCAB_CHECK_ARG(kind != CCAB_ALS_SPAN || (params[v] >= 1.0 && params[v] == (double)(int64_t)params[v]),
                   "span[%d] = %g is not a positive integer", v, params[v]);
  }
  rc = require_device();
  if (rc) return rc;
  return als_fit(kind, L, G, g_scale, n_samples, params, mu, init, k, max_iter, tol, W_out, iters_out, workspace,
                 workspace_bytes, static_cast<cudaStream_t>(stream));
  CCAB_CATCH
}

size_t ccab_ey_fit_workspace_bytes(int n_views, const int64_t* dims, int k, int batch) {
  ColumnLayout L;
  if (!dims || n_views < 2 || k < 1 || k > kEyMaxK || batch < 0 || batch == 1 || make_layout(n_views, dims, &L))
    return 0;
  return ey_fit_workspace_bytes(L, k, batch);
}

int ccab_ey_fit(int n_views, const int64_t* dims, int k, double c, double learning_rate, double momentum, double tol,
                int n_steps, const double* cov, int dtype, const void* const* views, const int64_t* ld, int batch,
                const int32_t* idx, double* state, void* workspace, size_t workspace_bytes, void* stream) {
  CCAB_TRY
  CCAB_CHECK_ARG(n_views >= 2, "the EY estimators need at least 2 views, got %d", n_views);
  CCAB_CHECK_ARG(dims && state && workspace, "null pointer argument");
  CCAB_CHECK_ARG(k >= 1 && k <= kEyMaxK, "k = %d: the EY fit supports 1 <= k <= %d", k, kEyMaxK);
  CCAB_CHECK_ARG(n_steps >= 0, "bad n_steps %d", n_steps);
  CCAB_CHECK_ARG(c >= 0.0 && c <= 1.0, "c = %g is outside [0, 1]", c);
  if (cov) {
    CCAB_CHECK_ARG(batch == 0, "the covariance route takes batch = 0, got %d", batch);
  } else {
    CCAB_CHECK_ARG(batch >= 2, "the mini-batch route needs batch >= 2, got %d", batch);
    CCAB_CHECK_ARG(views && ld && idx, "null pointer argument");
    CCAB_CHECK_ARG(dtype == CCAB_F32 || dtype == CCAB_F64, "bad dtype %d", dtype);
  }
  ColumnLayout L;
  int rc = make_layout(n_views, dims, &L);
  if (rc) return rc;
  for (int v = 0; !cov && v < n_views; ++v) {
    CCAB_CHECK_ARG(views[v], "views[%d] is NULL", v);
    CCAB_CHECK_ARG(ld[v] >= dims[v], "ld[%d] = %lld < dims[%d] = %lld", v, (long long)ld[v], v, (long long)dims[v]);
  }
  rc = require_device();
  if (rc) return rc;
  EyParams p;
  p.k = k;
  p.n_steps = n_steps;
  p.batch = cov ? 0 : batch;
  p.c = c;
  p.lr = learning_rate;
  p.momentum = momentum;
  p.tol = tol;
  return ey_fit(L, p, cov, dtype, views, ld, idx, state, workspace, workspace_bytes, static_cast<cudaStream_t>(stream));
  CCAB_CATCH
}

size_t ccab_tcca_moment_workspace_bytes(int n_views, const int64_t* dims, int64_t n, int nsplit) {
  if (tcca_check_dims(n_views, dims) || n < 1) return 0;
  return tcca_moment_workspace_bytes(n_views, dims, n, nsplit);
}

int ccab_tcca_moment(int n_views, const int64_t* dims, int64_t n, const double* const* Z, const int64_t* ldz,
                     double scale, int nsplit, double* M, void* workspace, size_t workspace_bytes, void* stream) {
  CCAB_TRY
  int rc = tcca_check_dims(n_views, dims);
  if (rc) return rc;
  CCAB_CHECK_ARG(n >= 1, "krprod_moment needs at least one sample, got n = %lld", (long long)n);
  CCAB_CHECK_ARG(Z && ldz && M, "null pointer argument");
  for (int i = 0; i < n_views; ++i)
    CCAB_CHECK_ARG(Z[i] && ldz[i] >= dims[i], "view %d: null pointer or leading dimension %lld < width %lld", i,
                   (long long)ldz[i], (long long)dims[i]);
  rc = require_device();
  if (rc) return rc;
  return tcca_moment(n_views, dims, n, Z, ldz, scale, nsplit, M, workspace, workspace_bytes,
                     static_cast<cudaStream_t>(stream));
  CCAB_CATCH
}

int ccab_tcca_moment_adjoint(int n_views, const int64_t* dims, int64_t n, const double* M, const double* const* H,
                             const int64_t* ldh, double scale, const double* scale_dev, double* const* Y,
                             const int64_t* ldy, void* stream) {
  CCAB_TRY
  int rc = tcca_check_dims(n_views, dims);
  if (rc) return rc;
  CCAB_CHECK_ARG(n >= 1, "krprod_adjoint needs at least one sample, got n = %lld", (long long)n);
  CCAB_CHECK_ARG(H && ldh && Y && ldy && M, "null pointer argument");
  for (int i = 0; i < n_views; ++i) {
    CCAB_CHECK_ARG(dims[i] <= (int64_t)65535 * 64, "view %d has width %lld; the adjoint supports at most %d", i,
                   (long long)dims[i], 65535 * 64);
    CCAB_CHECK_ARG(H[i] && ldh[i] >= dims[i], "H[%d]: null pointer or leading dimension %lld < width %lld", i,
                   (long long)ldh[i], (long long)dims[i]);
    CCAB_CHECK_ARG(Y[i] && ldy[i] >= dims[i], "Y[%d]: null pointer or leading dimension %lld < width %lld", i,
                   (long long)ldy[i], (long long)dims[i]);
  }
  rc = require_device();
  if (rc) return rc;
  return tcca_moment_adjoint(n_views, dims, n, M, H, ldh, scale, scale_dev, Y, ldy, static_cast<cudaStream_t>(stream));
  CCAB_CATCH
}

int64_t ccab_tcca_state_size(int n_views, const int64_t* dims, int k) {
  if (tcca_check_dims(n_views, dims)) return -1;
  if (k < 1 || k > kTccaMaxK) {
    set_error("k = %d: the TCCA fit supports 1 <= k <= %d", k, kTccaMaxK);
    return -1;
  }
  return (int64_t)tcca_state_doubles(n_views, dims, k);
}

size_t ccab_tcca_fit_workspace_bytes(int n_views, const int64_t* dims, int k) {
  if (tcca_check_dims(n_views, dims) || k < 1 || k > kTccaMaxK) return 0;
  return tcca_fit_workspace_bytes(n_views, dims, k);
}

int ccab_tcca_fit(int n_views, const int64_t* dims, int k, const double* M, const double* const* evecs,
                  const double* lam0, const double* rand, int start, int n_iter, double* state, void* workspace,
                  size_t workspace_bytes, void* stream) {
  CCAB_TRY
  int rc = tcca_check_dims(n_views, dims);
  if (rc) return rc;
  CCAB_CHECK_ARG(k >= 1 && k <= kTccaMaxK, "k = %d: the TCCA fit supports 1 <= k <= %d", k, kTccaMaxK);
  CCAB_CHECK_ARG(n_iter >= 0, "bad n_iter %d", n_iter);
  CCAB_CHECK_ARG(M && state && (!start || evecs), "null pointer argument");
  rc = require_device();
  if (rc) return rc;
  return tcca_fit(n_views, dims, k, M, evecs, lam0, rand, start, n_iter, state, workspace, workspace_bytes,
                  static_cast<cudaStream_t>(stream));
  CCAB_CATCH
}

size_t ccab_row_norm4_sum_workspace_bytes(int64_t n) {
  if (n < 1) return 0;
  return row_norm4_sum_workspace_bytes(n);
}

int ccab_row_norm4_sum(int dtype, int64_t n, int d, const void* Y, int64_t ldy, const double* mean, double* out,
                       void* workspace, size_t workspace_bytes, void* stream) {
  CCAB_TRY
  CCAB_CHECK_ARG(dtype == CCAB_F32 || dtype == CCAB_F64, "bad dtype %d", dtype);
  CCAB_CHECK_ARG(n >= 1 && d >= 1, "bad shape n=%lld d=%d", (long long)n, d);
  CCAB_CHECK_ARG(ldy >= d, "leading dimension %lld < width %d", (long long)ldy, d);
  CCAB_CHECK_ARG(Y && mean && out, "null pointer argument");
  int rc = require_device();
  if (rc) return rc;
  cudaStream_t s = static_cast<cudaStream_t>(stream);
  if (dtype == CCAB_F32)
    return row_norm4_sum<float>(n, d, static_cast<const float*>(Y), ldy, mean, out, workspace, workspace_bytes, s);
  return row_norm4_sum<double>(n, d, static_cast<const double*>(Y), ldy, mean, out, workspace, workspace_bytes, s);
  CCAB_CATCH
}

size_t ccab_ccar3_admm_workspace_bytes(int p, int q) {
  if (p < 1 || p > kCcar3MaxP || q < 1 || q > kCcar3MaxQ) return 0;
  return ccar3_admm_workspace_bytes(p, q);
}

int ccab_ccar3_admm(int p, int q, const double* M, int64_t ldm, const double* B0, int64_t ldb, double kappa,
                    double rho, double tol, int max_iter, double* Z, int64_t ldz, double* U, int64_t ldu,
                    double* info, void* workspace, size_t workspace_bytes, void* stream) {
  CCAB_TRY
  CCAB_CHECK_ARG(p >= 1 && p <= kCcar3MaxP && q >= 1 && q <= kCcar3MaxQ,
                 "ccar3_admm supports 1 <= p <= %d and 1 <= q <= %d, got p = %d, q = %d", kCcar3MaxP, kCcar3MaxQ, p, q);
  CCAB_CHECK_ARG(max_iter >= 1, "bad max_iter %d", max_iter);
  CCAB_CHECK_ARG(rho > 0.0 && tol > 0.0 && kappa >= 0.0, "ccar3_admm needs rho > 0, tol > 0 and kappa >= 0");
  CCAB_CHECK_ARG(ldm >= p && ldb >= q && ldz >= q && ldu >= q, "leading dimension too small");
  CCAB_CHECK_ARG(M && B0 && Z && U && info, "null pointer argument");
  int rc = require_device();
  if (rc) return rc;
  return ccar3_admm(p, q, M, ldm, B0, ldb, kappa, rho, tol, max_iter, Z, ldz, U, ldu, info, workspace,
                    workspace_bytes, static_cast<cudaStream_t>(stream));
  CCAB_CATCH
}

size_t ccab_cv_scores_workspace_bytes(int n_views, const int64_t* dims, int G, int k_max) {
  if (n_views < 2 || n_views > kMaxViews || !dims || G < 1 || k_max < 1) return 0;
  for (int v = 0; v < n_views; ++v)
    if (dims[v] < 1) return 0;
  return cv_scores_workspace_bytes(n_views, dims, (int64_t)G * k_max);
}

int ccab_cv_scores(int n_views, const int64_t* dims, const double* C, int64_t ldc, double n, const double* W,
                   int64_t ldw, int G, int k_max, const int* k_of, double* corr, double* score, void* workspace,
                   size_t workspace_bytes, void* stream) {
  CCAB_TRY
  CCAB_CHECK_ARG(n_views >= 2 && n_views <= kMaxViews, "cv_scores needs 2 to %d views, got %d", kMaxViews,
                 n_views);
  CCAB_CHECK_ARG(dims && C && W && k_of && corr && score && workspace, "null pointer argument");
  int64_t D = 0;
  for (int v = 0; v < n_views; ++v) {
    CCAB_CHECK_ARG(dims[v] >= 1, "bad view width %lld", (long long)dims[v]);
    D += dims[v];
  }
  CCAB_CHECK_ARG(D <= (1 << 20), "total width %lld is too large", (long long)D);
  CCAB_CHECK_ARG(G >= 1 && k_max >= 1 && (int64_t)G * k_max <= (1 << 24), "bad candidate shape G = %d, k_max = %d", G,
                 k_max);
  CCAB_CHECK_ARG(ldc >= D && ldw >= (int64_t)G * k_max, "leading dimension too small");
  CCAB_CHECK_ARG(n >= 2.0, "at least 2 held-out samples are needed, got n = %g", n);
  CCAB_CHECK_ARG(workspace_bytes >= cv_scores_workspace_bytes(n_views, dims, (int64_t)G * k_max),
                 "workspace too small: %zu bytes", workspace_bytes);
  int rc = require_device();
  if (rc) return rc;
  return cv_scores(n_views, dims, C, ldc, n, W, ldw, G, k_max, k_of, corr, score, workspace,
                   static_cast<cudaStream_t>(stream));
  CCAB_CATCH
}

size_t ccab_pairwise_kernel_workspace_bytes(int metric, int64_t nx, int64_t ny) {
  if (metric < CCAB_KERNEL_LINEAR || metric > CCAB_KERNEL_ADDITIVE_CHI2 || nx < 0 || ny < 0) return 0;
  return pairwise_kernel_workspace_bytes(metric, nx, ny);
}

int ccab_pairwise_kernel(int metric, int dtype, const void* X, int64_t nx, int64_t ldx, const void* Y, int64_t ny,
                         int64_t ldy, int d, double gamma, double degree, double coef0, double* K, int64_t ldk,
                         void* workspace, size_t workspace_bytes, void* stream) {
  CCAB_TRY
  CCAB_CHECK_ARG(metric >= CCAB_KERNEL_LINEAR && metric <= CCAB_KERNEL_ADDITIVE_CHI2, "bad kernel metric %d", metric);
  CCAB_CHECK_ARG(dtype == CCAB_F32 || dtype == CCAB_F64, "bad dtype %d", dtype);
  CCAB_CHECK_ARG(nx >= 0 && ny >= 0 && d >= 1, "bad shape nx=%lld ny=%lld d=%d", (long long)nx, (long long)ny, d);
  CCAB_CHECK_ARG(ldx >= d && ldy >= d && ldk >= ny, "leading dimension too small");
  CCAB_CHECK_ARG(nx <= ((int64_t)1 << 31) && ny <= ((int64_t)1 << 31), "pairwise_kernel: more than 2^31 rows");
  CCAB_CHECK_ARG((X && Y && K) || nx == 0 || ny == 0, "null pointer argument");
  int rc = require_device();
  if (rc) return rc;
  cudaStream_t s = static_cast<cudaStream_t>(stream);
  if (dtype == CCAB_F32)
    return pairwise_kernel<float>(metric, static_cast<const float*>(X), nx, ldx, static_cast<const float*>(Y), ny,
                                  ldy, d, gamma, degree, coef0, K, ldk, workspace, workspace_bytes, s);
  return pairwise_kernel<double>(metric, static_cast<const double*>(X), nx, ldx, static_cast<const double*>(Y), ny,
                                 ldy, d, gamma, degree, coef0, K, ldk, workspace, workspace_bytes, s);
  CCAB_CATCH
}

size_t ccab_gfa_fit_workspace_bytes(int n_views, const int64_t* dims, int k) {
  ColumnLayout L;
  if (!dims || n_views < 1 || k < 1 || k > kGfaMaxK || make_layout(n_views, dims, &L)) return 0;
  return gfa_fit_workspace_bytes(L, k);
}

int ccab_gfa_fit(int n_views, const int64_t* dims, int k, const double* G, double n_samples, const double* XtZ0,
                 double tol, int drop_k, int n_steps, double* state, void* workspace, size_t workspace_bytes,
                 void* stream) {
  CCAB_TRY
  CCAB_CHECK_ARG(n_views >= 1, "GFA needs at least 1 view, got %d", n_views);
  CCAB_CHECK_ARG(dims && G && XtZ0 && state && workspace, "null pointer argument");
  CCAB_CHECK_ARG(k >= 1 && k <= kGfaMaxK, "k = %d: the GFA fit supports 1 <= k <= %d", k, kGfaMaxK);
  CCAB_CHECK_ARG(n_steps >= 0, "bad n_steps %d", n_steps);
  CCAB_CHECK_ARG(n_samples > 0.0, "n_samples = %g is not positive", n_samples);
  ColumnLayout L;
  int rc = make_layout(n_views, dims, &L);
  if (rc) return rc;
  rc = require_device();
  if (rc) return rc;
  return gfa_fit(L, k, G, n_samples, XtZ0, tol, drop_k, n_steps, state, workspace, workspace_bytes,
                 static_cast<cudaStream_t>(stream));
  CCAB_CATCH
}

int ccab_scale(int dtype, int m, int n, const void* A, int64_t lda, const void* r, int r_pow, const void* c,
               int c_pow, void* B, int64_t ldb, void* stream) {
  CCAB_TRY
  CCAB_CHECK_ARG(dtype == CCAB_F32 || dtype == CCAB_F64, "bad dtype %d", dtype);
  CCAB_CHECK_ARG((A && B) || m == 0 || n == 0, "null pointer argument");   // an empty tensor may have no storage
  CCAB_CHECK_ARG(r_pow >= 0 && r_pow <= 2 && c_pow >= 0 && c_pow <= 2, "bad power code");
  int rc = require_device();
  if (rc) return rc;
  cudaStream_t s = static_cast<cudaStream_t>(stream);
  if (dtype == CCAB_F32)
    return scale_rows_cols<float>(m, n, static_cast<const float*>(A), lda, static_cast<const float*>(r), r_pow,
                                  static_cast<const float*>(c), c_pow, static_cast<float*>(B), ldb, s);
  return scale_rows_cols<double>(m, n, static_cast<const double*>(A), lda, static_cast<const double*>(r), r_pow,
                                 static_cast<const double*>(c), c_pow, static_cast<double*>(B), ldb, s);
  CCAB_CATCH
}

int ccab_center_columns(int dtype, int m, int n, void* A, int64_t lda, void* stream) {
  CCAB_TRY
  CCAB_CHECK_ARG(dtype == CCAB_F32 || dtype == CCAB_F64, "bad dtype %d", dtype);
  CCAB_CHECK_ARG(A != nullptr || m == 0 || n == 0, "null pointer argument");
  int rc = require_device();
  if (rc) return rc;
  cudaStream_t s = static_cast<cudaStream_t>(stream);
  if (dtype == CCAB_F32) return center_columns<float>(m, n, static_cast<float*>(A), lda, s);
  return center_columns<double>(m, n, static_cast<double*>(A), lda, s);
  CCAB_CATCH
}

int ccab_row_sub_scale(int dtype, int64_t m, int n, void* A, int64_t lda, const void* r, const void* s_dev,
                       void* stream) {
  CCAB_TRY
  CCAB_CHECK_ARG(dtype == CCAB_F32 || dtype == CCAB_F64, "bad dtype %d", dtype);
  CCAB_CHECK_ARG(A != nullptr || m == 0 || n == 0, "null pointer argument");
  int rc = require_device();
  if (rc) return rc;
  cudaStream_t s = static_cast<cudaStream_t>(stream);
  if (dtype == CCAB_F32)
    return row_sub_scale<float>(m, n, static_cast<float*>(A), lda, static_cast<const float*>(r),
                                static_cast<const float*>(s_dev), s);
  return row_sub_scale<double>(m, n, static_cast<double*>(A), lda, static_cast<const double*>(r),
                               static_cast<const double*>(s_dev), s);
  CCAB_CATCH
}

int ccab_frobenius_norm(int dtype, int m, int n, const void* A, int64_t lda, void* out, void* stream) {
  CCAB_TRY
  CCAB_CHECK_ARG(dtype == CCAB_F32 || dtype == CCAB_F64, "bad dtype %d", dtype);
  CCAB_CHECK_ARG(out && (A || m == 0 || n == 0), "null pointer argument");
  CCAB_CHECK_ARG(m >= 0 && n >= 0, "bad shape");
  int rc = require_device();
  if (rc) return rc;
  cudaStream_t s = static_cast<cudaStream_t>(stream);
  if (dtype == CCAB_F32)
    return frobenius_norm<float>(m, n, static_cast<const float*>(A), lda, static_cast<float*>(out), s);
  return frobenius_norm<double>(m, n, static_cast<const double*>(A), lda, static_cast<double*>(out), s);
  CCAB_CATCH
}

int ccab_profile_moments(int enable) {
  moments_profile_enable(enable);
  return 0;
}
double ccab_profile_moments_last_ms(void) { return (double)moments_profile_last_ms(); }

}  // extern "C"
