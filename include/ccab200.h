/* libccab200 -- C ABI of the H100-native CCA hot path.
 *
 * The reference (jameschapman19/cca_zoo) is pure Python and has NO FFI boundary for this path
 * (SURVEY.md §8b); this header is the boundary a maintainer would bind with ctypes (see
 * INTEGRATION.md).  Each entry point names the reference code it replaces.
 *
 * Conventions
 *   - every pointer marked "device" is a CUDA device pointer owned by the caller (PyTorch's caching
 *     allocator in the Python binding); the library never allocates device memory, the caller passes
 *     a workspace sized by the matching *_workspace_bytes call;
 *   - matrices are row-major with an explicit leading dimension unless stated otherwise;
 *   - `stream` is a cudaStream_t passed as void*; calls are asynchronous on it, except ccab_syevj /
 *     ccab_gesvj which synchronise it once per Jacobi sweep to read the convergence flag;
 *   - return 0 = OK, <0 = bad argument / unsupported, >0 = cudaError_t.  ccab_last_error() gives the
 *     message of the last failure on the calling thread.  No C++ exception crosses the ABI.
 *   - dtype: CCAB_F32 / CCAB_F64.  The 16-bit codes CCAB_BF16 / CCAB_F16 are accepted by ccab_moments,
 *     ccab_moments_workspace_bytes, ccab_column_pilot and ccab_shift_rows only; every other entry point rejects them
 *     as a bad dtype.  There is no CPU fallback: without a sm_90a device every compute entry point fails.
 */
#ifndef CCAB200_H
#define CCAB200_H

#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#define CCAB_F32 0
#define CCAB_F64 1
#define CCAB_BF16 2 /* bfloat16 views: the moments and the pilot / shift of the shifted accumulation only */
#define CCAB_F16 3  /* float16 views: likewise */

/* arithmetic of the moment kernel (ccab_moments `precision`) */
#define CCAB_PREC_TF32 0   /* fp32 in, one wgmma TF32 pass, fp32 accumulate               */
#define CCAB_PREC_TF32X3 1 /* fp32 in, hi/lo split + 3 wgmma passes: fp32-grade accuracy          */
#define CCAB_PREC_EXACT 2  /* FMA in the input dtype on CUDA cores (the only choice for CCAB_F64)  */
#define CCAB_PREC_TF32X3B 3 /* 3xTF32 with the two cross terms as bf16 MMAs: fp32-grade, 2/3 the tensor work */
/* For CCAB_BF16 / CCAB_F16 views, CCAB_PREC_TF32, _TF32X3 and _TF32X3B all select the one 16-bit wgmma kernel: the
 * product of two bf16 or two fp16 values is exact in fp32, so there is nothing to split.  Its fp32 accumulator runs
 * span at most 2048 samples and are summed in float64, as in the 3xTF32 modes.  CCAB_PREC_EXACT converts on load and
 * runs FMA in fp32 on CUDA cores, with the same 2048-sample runs folded into float64. */

#define CCAB_MAX_VIEWS 8

int ccab_version(void);
const char* ccab_last_error(void);
/* kernels launched by this library since it was loaded (bench.py's gpu_launches) */
int64_t ccab_launch_count(void);

/* ---- K1: block moments --------------------------------------------------------------------------
 * M = [X_1 .. X_m]^T [X_1 .. X_m] and s = 1^T [X_1 .. X_m] over the n_rows samples this process
 * holds.  Output `moments` (device, double) has ccab_moments_size() entries: a Dp x Dp padded matrix
 * (each view padded to a multiple of 128 columns) followed by the Dp column sums.  Entries M[r][c] with r <= c are
 * the moments; entries below the 128-block diagonal are zero; the strictly lower part (r > c) of a diagonal
 * 128 x 128 block is unspecified and no consumer reads it.  The buffer is additive over row shards: all-reduce(sum) it
 * across ranks before ccab_covariance.
 * Replaces: np.linalg.svd(X) cca_zoo/_utils/_linalg.py:28, X1_w.T @ X2_w cca_zoo/linear/_rcca.py:96,
 * np.cov(...) cca_zoo/linear/_mcca.py:150-152,166 and cca_zoo/linear/_gcca.py:101,
 * z.T @ z cca_zoo/deep/objectives.py:86-92; the column sums replace v.mean(axis=0) cca_zoo/_base.py:97.
 * views[v]: device pointer to an n_rows x dims[v] row-major array with leading dimension lds[v]
 * (tensor-core paths read the views with TMA: they need 16-byte aligned pointers and a row pitch that is a multiple of
 * 16 bytes -- lds[v] % 4 == 0 for float32, lds[v] % 8 == 0 for bf16 / fp16 -- and return -1 otherwise). */
int64_t ccab_moments_size(int n_views, const int64_t* dims);
int64_t ccab_moments_padded_dim(int n_views, const int64_t* dims);
size_t ccab_moments_workspace_bytes(int dtype, int precision, int n_views, const int64_t* dims, int64_t n_rows);
int ccab_moments(int dtype, int precision, int n_views, const void* const* views, const int64_t* dims,
                 const int64_t* lds, int64_t n_rows, double* moments, void* workspace, size_t workspace_bytes,
                 void* stream);

/* ---- shifted accumulation (numerical safety of the one-pass covariance) -----------------------------------------------
 * (M - s s^T / n) cancels catastrophically when a column's mean dominates its spread: the relative error of the
 * covariance is eps_prod * (mean / std)^2, eps_prod ~ 1e-7 .. 1e-6 for float32 inputs.  The reference centres the data
 * first (cca_zoo/_base.py:96-99); covariance being shift invariant, the same is had in one pass by accumulating the
 * moments of X - x0 and rebuilding the raw moments in float64:
 *   ccab_column_pilot   x0[j] = mean of column j over the first `rows` rows (device, in the view's dtype; float32
 *                       for 16-bit views);
 *                       ratio_max_dev[0] = max(ratio_max_dev[0], max_j mean_j^2 / var_j)   (zero it first)
 *   ccab_shift_rows     Xs = X - x0   (one extra pass, only taken when the pilot says it matters; Xs is float32 for
 *                       16-bit views, whose shifted copy then takes the float32 moment route and whose
 *                       ccab_moments_unshift runs with dtype CCAB_F32)
 *   ccab_moments        ... on Xs ...
 *   ccab_moments_unshift  M += x0 s^T + s x0^T + n x0 x0^T, s += n x0 in float64 (x0: per view device pointers or NULL)
 * after which the buffer holds the raw moments again: additive over row shards, all-reducible, whatever x0 each rank
 * chose. */
int ccab_column_pilot(int dtype, const void* X, int64_t rows, int d, int64_t ld, void* x0, float* ratio_max_dev,
                      void* stream);
int ccab_shift_rows(int dtype, const void* X, int64_t n, int d, int64_t ldx, const void* x0, void* Xs, int64_t lds,
                    void* stream);
int ccab_moments_unshift(int dtype, int n_views, const int64_t* dims, double* moments, const void* const* x0,
                         double n_rows, void* stream);

/* ---- exchange step of a sample-sharded fit (SURVEY.md §8e) ---------------------------------------------------------
 * ccab_moments_pack gathers what the all-reduce has to carry into ONE contiguous float64 message of
 * ccab_moments_packed_size() entries: the upper triangle of 128 x 128 blocks of M (row-major over block pairs),
 * the column sums, the local sample count n and one reserved slot.  Sum it over the ranks (NCCL all-reduce over
 * NVLink), then ccab_moments_unpack restores the moment buffer of ccab_moments (zero below the block diagonal, the
 * diagonal blocks copied whole, so their strictly lower parts stay as unspecified as in ccab_moments);
 * packed[size - 2] is the total sample count, which ccab_rcca_fit / ccab_mcca_fit read on the device (n_total_dev). */
int64_t ccab_moments_packed_size(int n_views, const int64_t* dims);
int ccab_moments_pack(int n_views, const int64_t* dims, const double* moments, double n_local, double* packed,
                      void* stream);
int ccab_moments_unpack(int n_views, const int64_t* dims, const double* packed, double* moments, void* stream);

/* Fused exchange step over NVLink / NVSwitch: pack -> in-switch all-reduce -> unpack in ONE kernel, no NCCL call.
 * Needs a symmetric-memory buffer of `sym_doubles` float64 (>= world * ceil(ccab_moments_packed_size / world),
 * rounded up to even) mapped on every rank with a multicast (NVLS) address, and the ranks' signal pads (uint32 flags,
 * `pad_slots` entries each, zeroed once) -- torch.distributed._symmetric_memory provides both (cca_zoo_b200/parallel.py).
 * Each CTA packs its column of the message, meets the peers on its own flag row (st.release.sys / ld.acquire.sys),
 * reduces this rank's slice with multimem.ld_reduce.add.f64 (the switch adds the ranks' copies), broadcasts it with
 * multimem.st, meets the peers again and scatters the totals into `moments`; n_total_out (device, may be NULL)
 * receives the summed sample count.  `epoch` must be the same on every rank and grow by 2 per call.
 * The result is bit-identical on all ranks (every element is reduced once, in the switch). */
int ccab_moments_exchange_nvls(int n_views, const int64_t* dims, double* moments, double n_local, double* sym_local,
                               double* sym_multicast, void* const* signal_pads_dev, int rank, int world,
                               int pad_slots, int64_t sym_doubles, unsigned epoch, double* n_total_out, void* stream);

/* ---- K2: covariance from (all-reduced) moments ---------------------------------------------------
 * C = (M - s s^T / n_total) / (n_total - 1) (center != 0) or M / (n_total - 1), compact D x D
 * (D = sum dims, hstack order), full symmetric, in out_dtype; mean = s / n_total (or 0).
 * Replaces: the centring of cca_zoo/_base.py:96-99 plus the 1/(n-1) scalings listed above. */
int ccab_covariance(int out_dtype, int n_views, const int64_t* dims, const double* moments, double n_total,
                    int center, void* C, int64_t ldc, void* mean, void* stream);
/* The same with n_total read at n_dev[0] (device): the count of an all-reduced buffer needs no host read-back.
 * N < 2 is not refused here (nothing is read back): C then holds inf / NaN. */
int ccab_covariance_ndev(int out_dtype, int n_views, const int64_t* dims, const double* moments, const double* n_dev,
                         int center, void* C, int64_t ldc, void* mean, void* stream);

/* ---- K3: batched symmetric eigensolver (one-sided block Jacobi) ----------------------------------
 * For each of `batch` symmetric n x n matrices A_b (device, row-major == column-major, lda, stride
 * batch_stride elements): eigenvalues descending into evals[b*n ..], eigenvectors as ROWS of
 * evecs_t[b] (n x n, ldv): evecs_t[b][j,:] is the unit eigenvector of the j-th largest eigenvalue.
 * `shift` is added to the diagonal before solving and removed from the eigenvalues afterwards; pass a
 * value >= -lambda_min for indefinite matrices (the one-sided method needs A + shift*I to be PSD to
 * separate +/- pairs).  info[0] (host, may be NULL) = sweeps used, NEGATED when the iteration ran out of sweeps before
 * reaching the tolerance (with info == NULL such a call fails instead), info_offdiag (host, may be NULL) =
 * last normalised off-diagonal.
 * Replaces: scipy.linalg.eigh cca_zoo/_utils/_linalg.py:64-71, np.linalg.eigvalsh
 * cca_zoo/linear/_mcca.py:170,194 cca_zoo/linear/_gcca.py:102, sklearn PCA cca_zoo/linear/_mcca.py:117,
 * torch.linalg.eigh cca_zoo/deep/objectives.py:19, and (via covariance form) the tall SVD of
 * cca_zoo/_utils/_linalg.py:28. */
size_t ccab_syevj_workspace_bytes(int dtype, int n, int batch);
int ccab_syevj(int dtype, int n, int batch, const void* A, int64_t lda, int64_t batch_stride, double shift,
               void* evals, void* evecs_t, int64_t ldv, int* info, float* info_offdiag, void* workspace,
               size_t workspace_bytes, void* stream);

/* Small symmetric eigenproblems (n <= 128 float / 104 double), batched, ONE single-CTA launch per matrix, no host
 * synchronisation: two-sided Jacobi with tournament ordering in shared memory.  Same outputs as ccab_syevj
 * (descending eigenvalues, eigenvectors as rows; evals / evecs_t contiguous per matrix: n and n x ldv); absolute
 * accuracy eps * ||A|| (use ccab_syevj when tiny eigenvalues matter relatively).  info_dev[b] (device int[batch],
 * may be NULL) = sweeps used, negated if the tolerance was not reached.
 * Replaces the Rayleigh-Ritz eigensolve of the top-k route (scipy.linalg.eigh subset_by_index,
 * cca_zoo/_utils/_linalg.py:64-73). */
int ccab_syevj_small(int dtype, int n, int batch, const void* A, int64_t lda, int64_t stride_a, void* evals,
                     void* evecs_t, int64_t ldv, int* info_dev, void* stream);

/* ---- K4: singular value decomposition (one-sided Jacobi) -----------------------------------------
 * G is m x n given by COLUMNS: column j is the contiguous array A + j*lda (length m) -- i.e. a
 * row-major n x m buffer holds G^T.  Outputs (descending): sigma[n]; right_t (n x n, ldr): row j =
 * j-th right singular vector; left_t (n x m, ldl): row j = j-th left singular vector (unit, length m;
 * zero for sigma_j = 0).  Any output may be NULL.
 * Replaces: np.linalg.svd(cross_cov) cca_zoo/linear/_rcca.py:97. */
size_t ccab_gesvj_workspace_bytes(int dtype, int m, int n);
int ccab_gesvj(int dtype, int m, int n, const void* A, int64_t lda, void* sigma, void* right_t, int64_t ldr,
               void* left_t, int64_t ldl, int* info, float* info_offdiag, void* workspace, size_t workspace_bytes,
               void* stream);

/* ---- dense glue ----------------------------------------------------------------------------------
 * C (m x n) = alpha * op(A) * op(B) + beta * C, row-major; transX != 0 means op(X) = X^T.
 * float32 operands that TMA can address (16-byte aligned, leading dimensions % 4 == 0) run on the tensor pipe
 * (ccab_gemm_tc: 3xTF32, fp32-grade); everything else as exact FMA tiles.
 * Replaces the small products W1^T C12 W2, W @ U (cca_zoo/linear/_rcca.py:96,100), components_.T @ w
 * (cca_zoo/linear/_mcca.py:131) and the S11^-1/2 S12 S22^-1/2 chain (cca_zoo/deep/objectives.py:97). */
int ccab_gemm(int dtype, int transa, int transb, int m, int n, int k, double alpha, const void* A, int64_t lda,
              const void* B, int64_t ldb, double beta, void* C, int64_t ldc, void* stream);

/* Tensor-core variant of ccab_gemm for float32 (wgmma TF32, 3xTF32 split formed in shared memory:
 * fp32-grade products, fp32 accumulation in TMEM), batched: matrix b of the batch lives at X + b * stride_x.
 * Optionally also (or only: C may be NULL when beta == 0) writes the transpose Ct (n x m, row-major, ldct).
 * lower_only != 0 skips the 128-row output tiles that lie strictly above the diagonal (SYRK-type updates).
 * Needs 16-byte aligned A / B with lda, ldb (and the batch strides) multiples of 4; otherwise returns < 0 and the
 * caller uses ccab_gemm.  Replaces the same reference products as ccab_gemm, on the tensor pipe. */
int ccab_gemm_tc(int transa, int transb, int m, int n, int k, double alpha, const void* A, int64_t lda,
                 int64_t stride_a, const void* B, int64_t ldb, int64_t stride_b, double beta, void* C, int64_t ldc,
                 int64_t stride_c, void* Ct, int64_t ldct, int64_t stride_ct, int batch, int lower_only,
                 void* stream);

/* Whitening rows from an eigendecomposition (covariance form of svd_whiten,
 * cca_zoo/_utils/_linalg.py:30-38; also B^-1/2 of cca_zoo/linear/_mcca.py:163-173 and R_i of
 * cca_zoo/linear/_gcca.py:101-105):
 *   keep_j  = lam[j] > rank_tol * max(lam[0],0)  &&  j < max_rank
 *   g_j     = keep_j ? ((1-c)*max(lam[j],lam_floor) + c + floor_add + (floor_dev ? *floor_dev : 0))^-1/2
 *                      * scale^-1/2 : 0
 *   Wt[j,:] = g_j * Vt[j,:]            g_out[j] = g_j (may be NULL)      *rank_out = #kept (device int)
 * lam_floor = 0 with c = 0, floor_add = eps reproduces clamp(eigh(S + eps I), min=eps)
 * (cca_zoo/deep/objectives.py:19-21); pass -inf-like (e.g. -1e300) to disable the clamp. */
int ccab_whiten_rows(int dtype, int d, const void* lam, const void* Vt, int64_t ldv, double c, double floor_add,
                     const void* floor_dev, double scale, double rank_tol, int max_rank, double lam_floor, void* Wt,
                     int64_t ldw, void* g_out, int* rank_out, void* stream);

/* ---- K6: fused small-matrix stage of the deep-CCA objective (widths d1, d2 <= 64) -------------------
 * From the (d1+d2)^2 block covariance C of [z1 z2] (device, row-major): S_ii = C_ii + eps I,
 * P = S11^-1 S12 S22^-1, loss[0] = -<P, S12> = -||S11^-1/2 S12 S22^-1/2||_F^2, G11 = P S21 S11^-1 (d1 x d1),
 * G22 = S22^-1 S21 P (d2 x d2), P (d1 x d2), and min_pivot[0] = the smallest elimination pivot of S11/S22:
 * min_pivot > 4 eps certifies that the eigenvalue clamp of the reference is inactive (otherwise callers take
 * the eigen route).  One single-CTA launch.
 * Replaces: _inv_sqrtm x2, the T / T^T T products and eigvalsh of cca_zoo/deep/objectives.py:94-102 (forward)
 * and supplies the matrices of the analytic backward (SURVEY.md §3.4). */
int ccab_ccaloss_small(int dtype, int d1, int d2, const void* C, int64_t ldc, double eps, void* loss, void* G11,
                       void* P, void* G22, void* min_pivot, void* stream);

/* ---- Cholesky route of the generalised problem ----------------------------------------------------
 * Batched blocked Cholesky WITH the explicit inverse of the factor (the GEMM-friendly form of the whitening):
 * for each of `batch` SPD matrices A_b = A + b * stride_a (n x n row-major, lower triangle referenced)
 *   lower triangle of A_b <- L_b,   Linv_b = Linv + b * stride_i (n x n, ldi) <- L_b^-1 (zeros above the diagonal).
 * info_dev[b] (device int[batch]) = 0 or the 1-based index of the first pivot <= pivot_tol (matrix not numerically
 * positive definite: callers fall back to the eigen route).
 * Diagonal blocks (128 wide for float, 64 for double) are factored AND inverted by one single-CTA launch each
 * (warp-synchronous 32 x 32 sub-blocks); panels, trailing updates and the assembly of L^-1 by recursive doubling are
 * GEMMs (wgmma for float).  With Linv,  T = L1^-1 C12 L2^-T  and the weights  L_i^-T U_k  are plain products.
 * Replaces LAPACK potrf / trsm inside scipy.linalg.eigh(A, B) (cca_zoo/_utils/_linalg.py:67-71) and, in Cholesky
 * form, the whitening of cca_zoo/_utils/_linalg.py:30-38 and _inv_sqrtm of cca_zoo/deep/objectives.py:9-21. */
size_t ccab_potrf_inv_workspace_bytes(int dtype, int n, int batch);
int ccab_potrf_inv(int dtype, int n, int batch, void* A, int64_t lda, int64_t stride_a, void* Linv, int64_t ldi,
                   int64_t stride_i, double pivot_tol, int* info_dev, void* workspace, size_t workspace_bytes,
                   void* stream);

/* ---- the fit behind the ABI: rCCA / CCA / PLS ----------------------------------------------------------------------
 * From the (all-reduced) moment buffer of ccab_moments to the weights in ONE asynchronous call: covariance, ridge
 * blocks R_i = (1-c_i) C_ii + c_i I, batched Cholesky + inverse, T = L1^-1 C12 L2^-T, the leading k singular triplets
 * of T by blocked subspace iteration (block width p >= k, `iters` products with T^T T, CholQR, Rayleigh-Ritz) and
 * weights_i = L_i^-T U_k / V_k.  Nothing is read back by the library: every decision that needs a host (pivot
 * failures, rank loss, convergence, NaN / inf in the input, n <= d) is reported in the header of the result block.
 *   result (device, 256-byte aligned, ccab_rcca_fit_result_layout offsets[4] bytes):
 *     double header[32] | double mean[D] | T sigma[k] | T W1[d1 x k] | T W2[d2 x k]      (offsets[0..3] = byte offsets)
 *     header[0] = status bits (0 = valid): 1 a block is not positive definite, 2 not converged, 4 non-finite input,
 *                 8 too few samples (n <= max d_i);  header[1] = n_total;  [2] residual;  [3] sigma_1;
 *                 [4] index of the first failed factorisation;  [5] sweeps of the Ritz eigensolve
 *   n_total_dev (device double, may be NULL) overrides n_total: the sample count can ride in the all-reduced message.
 *   p must satisfy k <= p <= min(d1, d2) and p <= 128 (float) / 104 (double), the sizes ccab_syevj_small takes.
 *   ccab_rcca_fit_workspace_bytes returns 0 for every (dtype, dims, k, p) the fit refuses, so callers ask it first.
 *   dtype = arithmetic of the whole solve (CCAB_F32 uses wgmma GEMMs).
 * Replaces cca_zoo/linear/_rcca.py:83-101 (via cca_zoo/_utils/_linalg.py:9-41) after the moment pass. */
size_t ccab_rcca_fit_workspace_bytes(int dtype, const int64_t* dims, int k, int p);
int ccab_rcca_fit_result_layout(int dtype, const int64_t* dims, int k, int p, int64_t* offsets /* [5] */);
int ccab_rcca_fit(int dtype, const int64_t* dims, const double* moments, const double* n_total_dev, double n_total,
                  int center, const double* c, int k, int p, int iters, void* result, size_t result_bytes,
                  void* workspace, size_t workspace_bytes, void* stream);

/* ---- the fit behind the ABI: MCCA -------------------------------------------------------------------------------------
 * Same contract as ccab_rcca_fit for m >= 2 views: B_i = (1-c_i) C_ii + c_i I = L_i L_i^T (batched Cholesky + inverse
 * when the views share one width), K_ij = L_i^-1 C_ij L_j^-T, the k largest eigenpairs of K by blocked subspace
 * iteration on K + I / (1 - max c) with a Rayleigh-Ritz step, v_i = sqrt(m) L_i^-T y_i (v^T (B/m) v = 1 as scipy).
 * Result block: double header[32] | double mean[D] | T eigenvalues[k] | T W_1[d_1 x k] | .. | T W_m; offsets has m + 3
 * entries (mean, eigenvalues, W_1 .. W_m, total).  `eps` is the reference's floor on lambda_min(B): a block whose pivots
 * fall below it fails the factorisation (status bit 1) and the caller takes the eigen route, which applies the floor.
 * Needs max c <= 0.9 and k <= p <= D with p <= 128 (float) / 104 (double); ccab_mcca_fit_workspace_bytes returns 0
 * for every (dtype, dims, k, p) the fit refuses (also for fewer than 2 views).
 * Replaces cca_zoo/linear/_mcca.py:113-173 (_build_A, _build_B, gevp of cca_zoo/_utils/_linalg.py:44-73). */
size_t ccab_mcca_fit_workspace_bytes(int dtype, int n_views, const int64_t* dims, int k, int p);
int ccab_mcca_fit_result_layout(int dtype, int n_views, const int64_t* dims, int k, int p, int64_t* offsets);
int ccab_mcca_fit(int dtype, int n_views, const int64_t* dims, const double* moments, const double* n_total_dev,
                  double n_total, int center, const double* c, double eps, int k, int p, int iters, void* result,
                  size_t result_bytes, void* workspace, size_t workspace_bytes, void* stream);

/* ---- the sparse / ALS estimators behind the ABI ----------------------------------------------------------------------
 * PLS_ALS, SCCA_PMD, ParkhomenkoCCA, SCCA_Span and SCCA_ADMM iterated on the block Gram matrix g_scale * G (D x D,
 * device, row-major, symmetric; pass the covariance with g_scale = n - 1) instead of the samples, all k latent
 * dimensions in ONE asynchronous call: per dimension one persistent cooperative kernel (every sweep, every view update,
 * the thresholding and the convergence test: max_i ||w_i - w_i_prev|| < tol, at most max_iter sweeps), then the
 * deflation X_i <- X_i (I - w_i a_i^T / s_i) as a rank-2m update of a workspace copy of G.  Fixed-order reductions
 * only: repeated calls give bit-identical results.
 *   kind       CCAB_ALS_*
 *   params     per-view (host, n_views doubles): PMD tau (L1 bound tau * sqrt(d_i)), Parkhomenko / ADMM tau, Span span
 *              (1 <= span); ignored (may be NULL) for PLS_ALS
 *              ElasticCCA / SCCA_IPLS: 2 * n_views doubles (alpha_i >= 0, l1_ratio_i in [0, 1]) per view; SCCA_IPLS
 *              then D more: the column means of the views (zeros when they are centred)
 *   mu         ADMM penalty; n_samples: the ADMM step 1 / (||G_ii||_F / n_samples + mu), the n of the regressions.
 *              ElasticCCA / SCCA_IPLS: mu in [0, 1) is the relative eigenvalue cut of the alpha l1 = 0 solve
 *              (eigenvalues of G_ii / n + rho at or below mu times the largest count as zero)
 *   init       device, k x D: the initial weights of each dimension (unit norm per view)
 *   W_out      device, D x k row-major (hstack of the views' weights);  iters_out: device int[k], sweeps per dimension
 *              (ElasticCCA / SCCA_IPLS: negated when a coordinate descent of that dimension stopped at its 1000 sweeps
 *              above the KKT bound)
 * Needs 2 <= n_views <= 8; the widest view must fit the shared memory of one CTA (up to ~28000 features).
 * ElasticCCA and SCCA_IPLS solve each view update as the penalised regression of sklearn's Ridge / Lasso / ElasticNet
 * on the Gram matrix, min 1/2 w^T (G_ii / n + rho I) w - b^T w + alpha l1 ||w||_1 (rho = alpha (1 - l1), Ridge:
 * alpha / n_samples), to a KKT residual of 1e-12 max(1, ||b||_inf): the minimum-norm solution through an
 * eigendecomposition of G_ii per dimension when alpha l1 = 0 (this synchronises the stream once per eigensolver
 * sweep, so those calls are not asynchronous), cyclic coordinate descent otherwise (at most 1000 sweeps, the max_iter
 * of sklearn's solvers).  Views of at most 2048 features; their workspace is ccab_als_regression_workspace_bytes
 * (ccab_als_fit_workspace_bytes is that of kinds 0-4).
 * Replaces cca_zoo/linear/_iterative.py:65-117 (fit / _fit_single with the _update_weight of each model) and
 * deflate (cca_zoo/_utils/_linalg.py:91-116). */
#define CCAB_ALS_PLS 0
#define CCAB_ALS_PMD 1
#define CCAB_ALS_PARKHOMENKO 2
#define CCAB_ALS_SPAN 3
#define CCAB_ALS_ADMM 4
#define CCAB_ALS_ELASTIC 5
#define CCAB_ALS_IPLS 6
size_t ccab_als_fit_workspace_bytes(int n_views, const int64_t* dims);
size_t ccab_als_regression_workspace_bytes(int n_views, const int64_t* dims);
int ccab_als_fit(int kind, int n_views, const int64_t* dims, const double* G, double g_scale, double n_samples,
                 const double* params, double mu, const double* init, int k, int max_iter, double tol, double* W_out,
                 int* iters_out, void* workspace, size_t workspace_bytes, void* stream);

/* ---- the Eckart-Young gradient estimators behind the ABI -------------------------------------------------------------
 * CCA_EY, PLS_EY (c = 1) and MCCA_EY: up to n_steps momentum steps on the EY loss
 *   L = -2 tr(C_ey - c V) + tr(Vb Vb),  Vb = (1 - c) V + c B,  B = (1/m) sum_i W_i^T W_i
 * (vel = momentum * vel - learning_rate * g;  W += vel), ALL in one persistent cooperative launch, asynchronous, no
 * host synchronisation.  The fit state lives in a caller-owned device block of 8 + 2 * k * D doubles:
 *   state[0] previous objective (+inf before the first step), state[1] steps taken, state[2] stop flag,
 *   state[3] |change of the objective| of the last step, state[4..7] reserved (zero),
 *   then W (k x D: W[x * D + r] is row r of the hstacked weights, column x) and the velocity (same layout).
 * A step whose |prev_obj - obj| < tol sets the stop flag; once it is set, later steps and later calls do nothing (a
 * NaN objective never sets it).  Call repeatedly to run a fit in chunks.
 *   cov        covariance route (full batch): the centred D x D block covariance (device, row-major, float64);
 *              views / ld / idx are ignored and batch must be 0.
 *   batch > 1  mini-batch route (cov NULL): step s of this call uses rows idx[s * batch .. (s + 1) * batch) (device
 *              int32) gathered straight from the raw views (device pointers, all `dtype`, row-major with leading
 *              dimension ld[i] >= dims[i]); the batch is centred inside the step.
 * Needs 2 <= n_views <= 8 and 1 <= k <= 32.  Fixed-order reductions only: repeated calls give bit-identical results.
 * Replaces cca_zoo/linear/gradient/_base.py:113-130 with _derivative / _objective of
 * cca_zoo/linear/gradient/_cca_ey.py:195-225. */
size_t ccab_ey_fit_workspace_bytes(int n_views, const int64_t* dims, int k, int batch);
int ccab_ey_fit(int n_views, const int64_t* dims, int k, double c, double learning_rate, double momentum, double tol,
                int n_steps, const double* cov, int dtype, const void* const* views, const int64_t* ld, int batch,
                const int32_t* idx, double* state, void* workspace, size_t workspace_bytes, void* stream);

/* ---- GFA (Group Factor Analysis) behind the ABI ----------------------------------------------------------------------
 * Up to n_steps iterations of the closed-form mean-field variational loop, iterated on the Gram matrix: from the first
 * Z update on the latent mean is z = X B, B = [tau_1 W_1; ...; tau_m W_m] cov_z, so each iteration costs one D x D x k
 * product G B whatever n is.  ALL iterations run in one persistent cooperative launch, asynchronous, no host
 * synchronisation; float64 throughout, fixed-order reductions only (repeated calls give bit-identical results, and any
 * split of the iterations into calls gives the same state bit for bit).
 *   G          the float64 Gram matrix X^T X of the hstacked views (centred when the fit centres), D x D, row-major,
 *              symmetric (the kernel reads its rows as columns)
 *   n_samples  n (the zz = z^T z + n cov_z term and the pruning statistic mean(z^2, 0) = diag(B^T G B) / n)
 *   XtZ0       X^T z0 stored transposed (k x D row-major: XtZ0[x * D + r]), z0 the random start; read by the first
 *              iteration only
 *   tol        relative change of z below which an iteration counts as quiet; 1000 quiet iterations in a row, with no
 *              pruning, set the stop flag, after which later iterations and later calls do nothing
 *   drop_k     non-zero: columns whose mean(z^2) is not above 1e-7 are pruned (unless all are), compacting every
 *              array of the state in place in index order
 * The caller-owned state block (doubles; K = k the capacity, D = sum(dims), 8 slots per per-view array):
 *   [0] iterations done  [1] active columns k'  [2] quiet iterations in a row  [3] stop flag  [4] parity (which of
 *   the B / GB pairs is current)  [5] relative change of the last iteration (NaN when not compared)  [6] prunes
 *   [7..15] reserved; then y_const[8] (tr G_mm), a_ard[8], a_tau[8], tau[8], b_tau[8], alpha[8][K], b_ard[8][K],
 *   cov_w[8][K][K], ww[8][K][K], cov_z[K][K], zz[K][K], index[K] (original column of each active one), W[K][D],
 *   B[2][K][D], GB[2][K][D].  Matrices keep leading dimension K; column x of W, B, GB is the row x * D .. x * D + D.
 *   The caller initialises it (header zero, k' = K; the constants; tau = 1e3; b_tau, b_ard = 1e-14; alpha from the
 *   data variance; zz = z0^T z0 + n I; index = 0..K-1).
 * Needs 1 <= n_views <= 8 and 1 <= k <= 64 (workspace_bytes returns 0 otherwise).
 * Replaces the loop of GFA.fit, cca_zoo/probabilistic/_gfa.py:217-286. */
size_t ccab_gfa_fit_workspace_bytes(int n_views, const int64_t* dims, int k);
int ccab_gfa_fit(int n_views, const int64_t* dims, int k, const double* G, double n_samples, const double* XtZ0,
                 double tol, int drop_k, int n_steps, double* state, void* workspace, size_t workspace_bytes,
                 void* stream);

/* ---- TCCA (tensor CCA) behind the ABI ---------------------------------------------------------------------------------
 * ccab_tcca_moment: M = scale * Z_1^T KR(Z_2, ..., Z_m), the mode-0 unfolding (p_1 x prod_{i>1} p_i, row-major) of
 * the cross-moment tensor of the whitened views.  KR is the row-wise Khatri-Rao product flattened in C order (the
 * last view's index fastest), so M reshaped to p_1 x ... x p_m is the tensor itself.  Z[i] are float64 n x p_i
 * row-major device matrices with leading dimension ldz[i] >= p_i.  One contraction over the samples on the fp64 tensor
 * pipe (DMMA); the Khatri-Rao operand is generated in shared memory and never stored.  nsplit <= 0 picks the number of
 * sample splits from the shape (splits when the output tiles cannot fill the GPU); the partial slabs are added in a
 * fixed order, no atomics, so repeated calls are bit-identical.  workspace_bytes (0 when unsplit) sizes the slabs.
 * Needs 2 <= n_views <= 8, every p_i >= 1, prod p_i <= 2^25, n >= 1.
 * Replaces the n x p_1 x ... x p_m outer-product array of TCCA.fit, cca_zoo/linear/_tcca.py:99-109. */
size_t ccab_tcca_moment_workspace_bytes(int n_views, const int64_t* dims, int64_t n, int nsplit);
int ccab_tcca_moment(int n_views, const int64_t* dims, int64_t n, const double* const* Z, const int64_t* ldz,
                     double scale, int nsplit, double* M, void* workspace, size_t workspace_bytes, void* stream);

/* ccab_tcca_moment_adjoint: the adjoint of the contraction of ccab_tcca_moment in every mode, in one launch:
 *   Y[i] = f * KR_{j != i}(H_j) M_(i)^T,   Y[i][s, a] = f * sum_{idx: idx_i = a} M[idx] prod_{j != i} H_j[s, idx_j],
 * f = scale * (*scale_dev) (scale alone when scale_dev is NULL; scale_dev is a device double, never read back).
 * M is the tensor in C order (prod p_i float64 entries, as ccab_tcca_moment writes it), read through the mode-i
 * strides: no permuted copy.  H[i] are float64 n x p_i row-major device matrices (leading dimension ldh[i] >= p_i),
 * Y[i] float64 n x p_i row-major outputs (ldy[i] >= p_i).  Each (n x P_i) x (P_i x p_i) product, P_i = prod_{j != i}
 * p_j, runs on the fp64 tensor pipe (DMMA) with the Khatri-Rao operand generated in shared memory from the H_j rows,
 * never stored.  Every output tile sums its whole reduction in one fixed order, with no splits and no atomics:
 * repeated calls are bit-identical, and no workspace is needed.
 * Needs 2 <= n_views <= 8, 1 <= p_i <= 65535 * 64, prod p_i <= 2^25, n >= 1.
 * With M = ccab_tcca_moment(H) at scale 1/n and f = 1/n, Y[i] is the gradient of ||M||_F^2 / 2 with respect to
 * H_i: the backward of the deep tensor-CCA objective (TCCALoss). */
int ccab_tcca_moment_adjoint(int n_views, const int64_t* dims, int64_t n, const double* M, const double* const* H,
                             const int64_t* ldh, double scale, const double* scale_dev, double* const* Y,
                             const int64_t* ldy, void* stream);

/* ccab_tcca_fit: up to n_iter iterations of tensorly's parafac ALS (unnormalised, exact solve per mode, stop when
 * |rec_prev - rec| < 1e-8 from the second iteration on, at most 100 iterations in all) on the tensor M (float64,
 * prod p_i entries in C order), asynchronous: a fixed launch sequence in which every kernel returns at once once the
 * stop flag is set, fixed-order reductions only (repeated calls are bit-identical).
 * start != 0 first writes the start state from the leading eigenvectors of the unfolding Grams M_(j) M_(j)^T:
 *   evecs[j]   p_j x p_j row-major device matrix whose row r is the eigenvector of the r-th largest eigenvalue
 *   lam0       the eigenvalues of mode 0 (descending, device): column r of mode 0 is scaled by sqrt(max(lam0[r], 0))
 *   rand       (device) the random start columns of every mode with p_j < k, p_j x (k - p_j) row-major each, in mode
 *              order (tensorly draws them with one RandomState in that order); may be NULL when there are none
 *   Column r < min(k, p_j) is eigenvector r with its entry of largest |value| (the first on ties) made positive.
 * State block (doubles, size ccab_tcca_state_size): [0] iterations done [1] stop flag [2] singular (an exactly zero
 * pivot in the solve of some mode, where numpy.linalg.solve raises; it also sets the stop flag) [3] ||M||_F
 * [4..7] zero; rec[100] (the reconstruction error of every iteration); the factors F_j (p_j x k row-major) in mode
 * order; their Grams F_j^T F_j (k x k each).
 * Needs 2 <= n_views <= 8, 1 <= k <= 64, prod p_i <= 2^25 (state_size returns -1, workspace_bytes 0 otherwise).
 * Replaces tensorly.decomposition.parafac(M, k, random_state=...) of TCCA.fit, cca_zoo/linear/_tcca.py:111-117. */
int64_t ccab_tcca_state_size(int n_views, const int64_t* dims, int k);
size_t ccab_tcca_fit_workspace_bytes(int n_views, const int64_t* dims, int k);
int ccab_tcca_fit(int n_views, const int64_t* dims, int k, const double* M, const double* const* evecs,
                  const double* lam0, const double* rand, int start, int n_iter, double* state, void* workspace,
                  size_t workspace_bytes, void* stream);

/* ---- KCCA: pairwise kernel matrices ------------------------------------------------------------------------------
 * ccab_pairwise_kernel: K = k(X, Y) (nx x ny float64, row-major, ldk) for the metric names of sklearn's
 * PAIRWISE_KERNEL_FUNCTIONS, computed as sklearn.metrics.pairwise_kernels does:
 *   LINEAR         x.y
 *   POLY           (gamma x.y + coef0)^degree                     (pow with a float degree)
 *   RBF            exp(-gamma max(|x|^2 + |y|^2 - 2 x.y, 0))      (0 distance on the diagonal when X is Y)
 *   SIGMOID        tanh(gamma x.y + coef0)
 *   COSINE         x.y / (|x| |y|)                                (0 for a zero row)
 *   LAPLACIAN      exp(-gamma sum_k |x_k - y_k|)
 *   CHI2           exp(-gamma sum_k (x_k - y_k)^2 / (x_k + y_k))  (terms with x_k + y_k = 0 skipped)
 *   ADDITIVE_CHI2  -sum_k (x_k - y_k)^2 / (x_k + y_k)
 * X (nx x d, ldx) and Y (ny x d, ldy) are row-major device matrices in `dtype` (float32 is widened to float64 on
 * load); "X is Y" means the same pointer, row count and leading dimension.  The inner-product metrics run on the fp64
 * tensor pipe (DMMA) with the metric fused into the epilogue, after a row-norm pre-pass for RBF / COSINE; the
 * distance metrics run as FMA tiles.  Every element is summed over the features in one fixed order: repeated calls
 * are bit-identical.  CHI2 / ADDITIVE_CHI2 need non-negative input, which the caller checks (sklearn raises).
 * workspace_bytes: (nx + ny) doubles for RBF / COSINE, 0 otherwise.
 * Replaces sklearn.metrics.pairwise_kernels of KCCA.fit / KCCA.transform, cca_zoo/nonparametric/_kcca.py:137-183. */
#define CCAB_KERNEL_LINEAR 0
#define CCAB_KERNEL_POLY 1
#define CCAB_KERNEL_RBF 2
#define CCAB_KERNEL_SIGMOID 3
#define CCAB_KERNEL_COSINE 4
#define CCAB_KERNEL_LAPLACIAN 5
#define CCAB_KERNEL_CHI2 6
#define CCAB_KERNEL_ADDITIVE_CHI2 7
size_t ccab_pairwise_kernel_workspace_bytes(int metric, int64_t nx, int64_t ny);
int ccab_pairwise_kernel(int metric, int dtype, const void* X, int64_t nx, int64_t ldx, const void* Y, int64_t ny,
                         int64_t ldy, int d, double gamma, double degree, double coef0, double* K, int64_t ldk,
                         void* workspace, size_t workspace_bytes, void* stream);

/* ---- CCAR3: reduced-rank-regression CCA -------------------------------------------------------------------------
 * ccab_row_norm4_sum: out[0] (device double) = sum_s ||y_s - mean||^4 over the n rows of Y (n x d row-major, ldy,
 * float32 or float64 in `dtype`), centred on the fly with mean (device double[d]); accumulated in float64 in a fixed
 * order (one warp per row, a grid chosen from n alone, block sums added in block order): repeated calls are
 * bit-identical.  It is the one data-dependent term of the Ledoit-Wolf shrinkage that the block moments lack.
 * Replaces the sum of (X^2)^T X^2 inside sklearn.covariance.ledoit_wolf_shrinkage, behind
 * LedoitWolf().fit(Y) in CCAR3.fit, cca_zoo/linear/_ccar3.py:221. */
size_t ccab_row_norm4_sum_workspace_bytes(int64_t n);
int ccab_row_norm4_sum(int dtype, int64_t n, int d, const void* Y, int64_t ldy, const double* mean, double* out,
                       void* workspace, size_t workspace_bytes, void* stream);

/* ccab_ccar3_admm: the row-sparse group-lasso ADMM of CCAR3 in inverse form on float64 device matrices,
 *   B = B0 + rho M (Z - U);   Z_old = Z;   Z = row_shrink(B + U);   U = U + B - Z,
 *   row_shrink scales each row r by max(0, 1 - kappa / ||r||) (rows of norm 0 stay 0),
 * from Z = U = 0 (both are overwritten, p x q row-major, ldz / ldu), for up to max_iter iterations, stopping after
 * the first iteration with max(||Z - B||_F, ||Z_old - Z||_F) / sqrt(p) < tol.  M = (Sx + (rho + eps) I)^-1 is p x p
 * (ldm), B0 = M Sxy Sy^-1/2 is p x q (ldb), kappa = lambda / rho.  Z holds the result (exact zero rows).
 * info (device double[4]) = iterations done, the last primal and dual residuals, and 1 if the tolerance stopped the
 * loop (0 when max_iter did).  One persistent cooperative launch, one grid barrier per iteration, no host
 * synchronisation; the products run on the fp64 tensor pipe (DMMA) and every sum has a fixed order, so repeated calls
 * are bit-identical.  1 <= p <= 16384, 1 <= q <= 512; workspace_bytes is 0 outside them.
 * Replaces _admm_row_sparse_rrr, cca_zoo/linear/_ccar3.py:37-80 (two LU solves of order p per iteration). */
size_t ccab_ccar3_admm_workspace_bytes(int p, int q);
int ccab_ccar3_admm(int p, int q, const double* M, int64_t ldm, const double* B0, int64_t ldb, double kappa,
                    double rho, double tol, int max_iter, double* Z, int64_t ldz, double* U, int64_t ldu,
                    double* info, void* workspace, size_t workspace_bytes, void* stream);

/* ---- held-out scores of a batch of fitted candidates (the cross-validation scoring of GridSearchCV) --------------
 * C (device, D x D float64, ldc) is the covariance of n held-out rows, D = sum(dims), 2 <= n_views <= CCAB_MAX_VIEWS.
 * W (device, D x G k_max float64, row-major, ldw) packs G candidates: column b k_max + j holds dimension j of candidate
 * b (the views' weight blocks stacked by rows), zero past k_of[b] (device int32[G], 1 <= k_of[b] <= k_max).
 * corr (device, G x k_max) receives the average off-diagonal pairwise correlation of the projected rows per dimension
 * (zero past k_of[b]), score (device, G) its mean over the first k_of[b] dimensions: per pair
 * S_il = w_i^T C_il w_l / (den_i den_l) with den_i = sqrt(S_ii (n - 1)), or 1 when that is <= 1e-12, over sqrt(n - 1).
 * The products C[:, block l] W[block l, :] run on the fp64 tensor pipe; every sum has a fixed order, so repeated calls
 * are bit-identical.  workspace_bytes is 0 for arguments the entry point refuses.
 * Replaces one clone / fit / score cycle's score(), cca_zoo/_base.py:153-194, per candidate and split. */
size_t ccab_cv_scores_workspace_bytes(int n_views, const int64_t* dims, int G, int k_max);
int ccab_cv_scores(int n_views, const int64_t* dims, const double* C, int64_t ldc, double n, const double* W,
                   int64_t ldw, int G, int k_max, const int* k_of, double* corr, double* score, void* workspace,
                   size_t workspace_bytes, void* stream);

/* ---- the deep-CCA objective behind the ABI (any widths) ---------------------------------------------------------
 * ccab_ccaloss_fwd: loss[0] = -|| S11^-1/2 S12 S22^-1/2 ||_F^2 with S_ii = cov(z_i) + eps I, from the moment pass over
 * [z1 z2] (precision as in ccab_moments), a batched Cholesky + inverse and 7 GEMMs; `saved`
 * (T[d1*d1 + d1*d2 + d2*d2 + d1 + d2]) receives G11 = P S21 S11^-1 | P = S11^-1 S12 S22^-1 | G22 = S22^-1 S21 P | the
 * column means of z1, z2 (written by the fused path for widths <= 64) for the backward.
 * Nothing is read back: flags_dev (device int[3]) = Cholesky status of S11, S22 (a pivot^2 <= eps / 4 counts as a failure:
 * rounding destroyed the ridge; the caller re-runs through the eigen route, which clamps like the reference) and a
 * non-finite-input flag -- check lazily.
 * ccab_ccaloss_bwd: g1 = 2/(n-1) center(z1 G11 - z2 P^T) * grad_out[0], g2 = 2/(n-1) center(z2 G22 - z1 P) * grad_out[0]
 * (grad_out: device scalar, may be NULL = 1).  4 tall GEMMs (wgmma for float) + the centring (slab partial sums in a
 * 2 MB per-device scratch that this entry point allocates on first use -- the one exception to "the library never
 * allocates": it takes no workspace argument); widths <= 64 run as ONE fused launch instead.
 * Replaces cca_zoo/deep/objectives.py:9-21,79-102 and torch autograd through two eigh + eigvalsh. */
size_t ccab_ccaloss_workspace_bytes(int dtype, int precision, int d1, int d2, int64_t n);
int ccab_ccaloss_fwd(int dtype, int precision, const void* z1, int64_t ld1, const void* z2, int64_t ld2, int64_t n,
                     int d1, int d2, double eps, void* loss, void* saved, int* flags_dev, void* workspace,
                     size_t workspace_bytes, void* stream);
int ccab_ccaloss_bwd(int dtype, const void* z1, int64_t ld1, const void* z2, int64_t ld2, int64_t n, int d1, int d2,
                     const void* saved, const void* grad_out, void* g1, int64_t ldg1, void* g2, int64_t ldg2,
                     void* stream);

/* ---- the deep-CCA objective of a global batch (data-parallel ranks, moments all-reduced before the loss) ----------
 * ccab_ccaloss_fwd_moments: the stage of ccab_ccaloss_fwd after its moment pass, from `moments` (the ccab_moments
 * buffer of [z1 z2], summed over the ranks) with the sample count N read at n_dev[0] on the device.  Same loss and
 * flags; `saved` (T[d1*d1 + d1*d2 + d2*d2 + d1 + d2 + 1]) = G11 | P | G22 | global column means of z1, z2 | N.
 * ccab_ccaloss_bwd_global: this rank's n_local rows (0 allowed) of the gradient of the global loss,
 *   g1 = 2/(N-1) (z1 G11 - z2 P^T - 1 (mu1^T G11 - mu2^T P^T)) * grad_out[0],  g2 symmetric,
 * with mu and N from `saved`: 4 GEMMs over the local rows and one epilogue launch (widths <= 64: one fused launch).
 * Neither reads anything back, and the backward needs nothing from the other ranks. */
size_t ccab_ccaloss_fwd_moments_workspace_bytes(int dtype, int d1, int d2);
int ccab_ccaloss_fwd_moments(int dtype, int d1, int d2, const double* moments, const double* n_dev, double eps,
                             void* loss, void* saved, int* flags_dev, void* workspace, size_t workspace_bytes,
                             void* stream);
int ccab_ccaloss_bwd_global(int dtype, const void* z1, int64_t ld1, const void* z2, int64_t ld2, int64_t n_local, int d1,
                            int d2, const void* saved, const void* grad_out, void* g1, int64_t ldg1, void* g2,
                            int64_t ldg2, void* stream);

/* B[i,j] = A[i,j] * f(r[i]) * f(c[j]); r / c may be NULL; *_pow: 0 -> x, 1 -> 1/x, 2 -> 1/sqrt(x).
 * (column scalings such as diag(sigma)^-1/2 in the GCCA back-substitution, cca_zoo/linear/_gcca.py:109) */
int ccab_scale(int dtype, int m, int n, const void* A, int64_t lda, const void* r, int r_pow, const void* c,
               int c_pow, void* B, int64_t ldb, void* stream);

/* A[:, j] -= mean_i A[i, j] in place (the centring Jacobian of cca_zoo/deep/objectives.py:83-84) */
int ccab_center_columns(int dtype, int m, int n, void* A, int64_t lda, void* stream);

/* A[i, :] = (A[i, :] - r) * s[0] in place (m x n row-major; r: device T[n], s: device T[1]): the centring of a
 * global-batch gradient by the all-reduced column means, with a scale that may depend on the device-side count */
int ccab_row_sub_scale(int dtype, int64_t m, int n, void* A, int64_t lda, const void* r, const void* s, void* stream);

/* out[0] (device) = ||A||_F of an m x n row-major matrix */
int ccab_frobenius_norm(int dtype, int m, int n, const void* A, int64_t lda, void* out, void* stream);

/* Measurement hook: when enabled, CUDA events are recorded on the caller's stream immediately around the
 * tensor-core moment-kernel launch of ccab_moments (TF32 paths); ccab_profile_moments_last_ms() waits for the
 * last pair and returns the kernel's duration in ms (-1 if none). */
int ccab_profile_moments(int enable);
double ccab_profile_moments_last_ms(void);

#ifdef __cplusplus
}
#endif
#endif /* CCAB200_H */
