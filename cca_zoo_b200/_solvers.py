"""Covariance-space solvers on the device (everything after the all-reduce; replicated per rank).

Input: the compact block covariance ``C`` (D x D CUDA tensor) of the hstacked views.  All arithmetic
runs in libccab200 kernels (Jacobi eigensolver / SVD, GEMM, scalings); torch supplies buffers, views
and the handful of scalar read-backs (ranks, floors) that decide shapes on the host.
Algebra: SURVEY.md §3.1-3.3, checked against the reference by oracle/restatement.py (cov_* forms).
"""
from __future__ import annotations

import os

import numpy as np
import torch

from . import ops


def _slices(dims):
    off = np.concatenate([[0], np.cumsum(dims)]).astype(int)
    return [slice(int(off[i]), int(off[i + 1])) for i in range(len(dims))]


def _eps(dtype):
    return float(torch.finfo(dtype).eps)


class _two_streams:
    """Fork the current stream into two side streams and join them back on exit: independent per-view
    chains of small latency-bound kernels (Cholesky factorisations and inverses) overlap."""

    _pool = {}

    def __init__(self, device):
        self.device = device

    def __enter__(self):
        key = (self.device.index, torch.cuda.current_stream(self.device).cuda_stream)
        if key not in self._pool:
            self._pool[key] = [torch.cuda.Stream(self.device), torch.cuda.Stream(self.device)]
        self.streams = self._pool[key]
        self.main = torch.cuda.current_stream(self.device)
        ev = torch.cuda.Event()
        ev.record(self.main)
        for st in self.streams:
            st.wait_event(ev)
        return self.streams

    def __exit__(self, *exc):
        for st in self.streams:
            ev = torch.cuda.Event()
            ev.record(st)
            self.main.wait_event(ev)
        return False


def _rank_tol(d, dtype):
    """Relative eigenvalue threshold below which a direction of a d x d covariance block is treated as
    numerically null: the covariance-space image of the reference's ``s > 0`` filter
    (cca_zoo/_utils/_linalg.py:30).  d * eps is the noise level of the computed spectrum (entries carry
    O(eps) relative error, the spectral norm of that perturbation grows like d); it does NOT grow with the
    number of samples."""
    return d * _eps(dtype)


def _regularised_rank_tol(lam, c, d):
    """Threshold (relative to lambda_max) below which a direction of C_ii is dropped by the eigen route.

    The reference filters on ``s > 0`` (cca_zoo/_utils/_linalg.py:30), which in floating point only removes exact
    zeros; what makes a direction unusable is a numerically null REGULARISED eigenvalue (1-c) lam + c.  So the test
    is (1-c) lam + c > tol ((1-c) lam_max + c): for c = 0 the plain relative filter lam > tol lam_max (there the
    reference itself returns 1e13-sized weights for the null directions), for any practical ridge c > tol lam_max
    nothing is dropped -- exactly what the reference and the Cholesky route (pivot test on the regularised block) do.
    Returned in the form the kernel wants: keep iff lam > value * lam_max (-1 keeps everything)."""
    tol = _rank_tol(d, lam.dtype)
    if c == 0.0:
        return tol
    if c >= 1.0:
        return -1.0
    lam_max = max(float(lam[0].item()), 0.0)            # one host read-back; the eigen route is the slow path anyway
    thr = (tol * ((1.0 - c) * lam_max + c) - c) / (1.0 - c)
    if thr < 0.0 or lam_max == 0.0:
        return -1.0
    return thr / lam_max


def _block_eigh(C, dims):
    """Eigendecomposition of every diagonal block C_ii; equal-sized blocks go in one batched call."""
    sl = _slices(dims)
    lams, vts = [None] * len(dims), [None] * len(dims)
    by_size = {}
    for i, d in enumerate(dims):
        by_size.setdefault(d, []).append(i)
    for d, idx in by_size.items():
        A = torch.stack([C[sl[i], sl[i]] for i in idx]).contiguous()
        ev, evt = ops.syevj(A)
        for b, i in enumerate(idx):
            lams[i], vts[i] = ev[b], evt[b]
    return lams, vts


def _cholqr(Y, flags, passes=1):
    """Orthonormalise the columns of Y (n x p) by CholQR: G = Y^T Y = L L^T, returns Y L^-T.
    The device-side Cholesky status flags are appended to ``flags`` (checked once, later, by the caller):
    a non-zero flag means the block lost rank."""
    for _ in range(passes):
        Ginv, info = ops.potrf_inv_(ops.gemm(Y, Y, transa=True))
        flags.append(info)
        Y = ops.gemm(Y, Ginv, transb=True)
    return Y


def topk_svd(T, k, max_rounds=4, iters_per_round=5, oversample=None, seed=1234):
    """Leading k singular triplets of T (d1 x d2) by blocked subspace iteration + Rayleigh-Ritz.

    Z <- orth(T^T T Z) repeated (one CholQR pass per iteration: enough to keep the block
    well-conditioned; the last one is done twice); then the Jacobi SVD of the thin block Y = T Z (d1 x p)
    gives U, sigma and V = Z V_y.  Converged when ||T^T U_k - V_k diag(sigma)||_F <= tol sigma_1 sqrt(k) (the
    other residual T v_j - sigma_j u_j vanishes by construction).  Returns (sigma[k], Ut[k,d1], Vt[k,d2]) or
    None if it does not converge (no spectral gap after the block) or a block loses rank: the caller then
    runs the full Jacobi SVD.  One host read-back per round.
    """
    d1, d2 = T.shape
    if oversample is None:
        oversample = int(os.environ.get("CCAB_TOPK_OVERSAMPLE", "0")) or max(32, k // 2)
    p = min(min(d1, d2), k + oversample)
    gen = torch.Generator(device=T.device).manual_seed(seed)
    # a Gaussian start block is well conditioned by itself (cond ~ (sqrt(d)+sqrt(p))/(sqrt(d)-sqrt(p))):
    # no orthonormalisation needed before the first product
    Z = torch.randn((d2, p), generator=gen, device=T.device, dtype=T.dtype)
    flags = []
    tol = 200.0 * _eps(T.dtype)
    iters_per_round = int(os.environ.get("CCAB_TOPK_ITERS", "0")) or iters_per_round
    for _ in range(max_rounds):
        for it in range(iters_per_round):
            # one application of T^T T between orthonormalisations: the block's condition number grows by
            # (sigma_1/sigma_p)^2 per step, far below what a single CholQR pass tolerates
            Y = ops.gemm(T, Z)                                    # d1 x p
            Z = _cholqr(ops.gemm(T, Y, transa=True), flags,       # d2 x p
                         passes=2 if it == iters_per_round - 1 else 1)
        # Rayleigh-Ritz on Y = T Z (d1 x p): Y^T Y = Vy diag(sig^2) Vy^T (p x p Jacobi eigensolve; the block is
        # well conditioned -- sigma_1/sigma_p is a few units -- so squaring costs nothing at the top), then
        # U = Y Vy diag(1/sig), V = Z Vy
        Y = ops.gemm(T, Z)                                  # d1 x p
        sig2, Vy_t = ops.syevj(ops.gemm(Y, Y, transa=True))
        sig = sig2.clamp_min(0).sqrt()
        Ut = ops.scale(ops.gemm(Vy_t[:k], Y, transb=True), rows=sig[:k], rows_pow=-1)   # k x d1
        Vt = ops.gemm(Vy_t[:k], Z, transb=True)             # k x d2 : rows of (Z Vy)^T
        E = ops.gemm(Ut, T)                                 # rows: u_j^T T
        E -= ops.scale(Vt, rows=sig[:k])
        stats = torch.stack([ops.frobenius_norm(E)[0], sig[0], torch.stack(flags).max().to(T.dtype).reshape(())])
        resid, s1, bad = (float(x) for x in stats.cpu())    # the round's single host read-back
        if os.environ.get("CCAB_DEBUG_TOPK"):
            print(f"[topk_svd] p={p} iters={iters_per_round} resid={resid:.3e} limit={tol * s1 * (k ** 0.5):.3e}")
        if bad != 0.0 or not (s1 > 0.0):
            return None
        if resid <= tol * s1 * (k ** 0.5):
            return sig[:k], Ut, Vt
        flags = []
        Z = ops.gemm(Z, Vy_t, transb=True)                  # continue from the Ritz basis (all p vectors)
    return None


def topk_eigsh(K, k, shift, max_rounds=6, iters_per_round=8, seed=4321):
    """Largest-k (algebraic) eigenpairs of the symmetric matrix K by blocked subspace iteration on
    K + shift*I (shift >= -lambda_min(K) so that the shifted matrix is PSD) with Rayleigh-Ritz through the
    Jacobi eigensolver.  Returns (evals[k] descending, evecs_t[k, D]) or None when the residual
    ||K Z_k - Z_k diag(theta)||_F does not reach tol (no gap after the block): callers then run the full
    Jacobi solve.  One host read-back per round."""
    D = K.shape[0]
    p = min(D, max(2 * k, k + 32))
    gen = torch.Generator(device=K.device).manual_seed(seed)
    Z = torch.randn((D, p), generator=gen, device=K.device, dtype=K.dtype)
    flags = []
    Z = _cholqr(Z, flags, passes=2)
    tol = 200.0 * _eps(K.dtype)
    for _ in range(max_rounds):
        for it in range(iters_per_round):
            Y = ops.gemm(K, Z)
            if shift != 0.0:
                Y.add_(Z, alpha=shift)
            Z = _cholqr(Y, flags, passes=2 if it == iters_per_round - 1 else 1)
        KZ = ops.gemm(K, Z)                                   # D x p
        H = ops.gemm(Z, KZ, transa=True)                      # p x p Rayleigh quotient matrix
        H = 0.5 * (H + H.T)
        nrm = ops.frobenius_norm(H)
        theta, Qt = ops.syevj(H, shift=float(nrm.item()))     # descending
        Zr_t = ops.gemm(Qt[:k], Z, transb=True)               # k x D : Ritz vectors as rows
        E = ops.gemm(Qt[:k], KZ, transb=True)                 # rows: (K z_j)^T
        E -= ops.scale(Zr_t, rows=theta[:k])
        stats = torch.stack([ops.frobenius_norm(E)[0], theta[0].abs() + abs(shift),
                             torch.stack(flags).max().to(K.dtype).reshape(())])
        resid, scale, bad = (float(x) for x in stats.cpu())
        if bad != 0.0 or not (scale > 0.0):
            return None
        if resid <= tol * scale * (k ** 0.5):
            return theta[:k], Zr_t
        flags = []
        Z = ops.gemm(Z, Qt, transb=True)
    return None


def _cholesky_whiteners(C, dims, c, scales, eps_floor):
    """Per view: R_i = (1-c_i) C_ii + c_i I = L_i L_i^T and Linv_i = sqrt(scale_i) L_i^-1.
    Returns the list of Linv_i, or None when a block is not numerically positive definite or when
    lambda_min(R_i) cannot be certified >= eps_floor (then the reference's eps floor, _mcca.py:170-172 /
    _gcca.py:102-104, might be active and the eigen route must decide).  The certificate is
    lambda_min(R) = 1 / ||R^-1||_2 >= 1 / ||L^-1||_F^2."""
    sl = _slices(dims)
    out, flags, norms = [], [], []
    for i, s in enumerate(sl):
        R = (1.0 - c[i]) * C[s, s]
        R.diagonal().add_(c[i])
        dmax = R.diagonal().max()
        Linv, info = ops.potrf_inv_(R, pivot_tol=0.0)
        flags.append(info)
        norms.append(torch.stack([ops.frobenius_norm(Linv)[0], dmax]))
        out.append(Linv)
    stats = torch.cat([torch.stack(flags).max().to(C.dtype).reshape(1), torch.stack(norms).reshape(-1)]).cpu()
    if float(stats[0]) != 0.0:
        return None
    for i in range(len(dims)):
        fro, dmax = float(stats[1 + 2 * i]), float(stats[2 + 2 * i])
        if not (fro > 0.0) or not np.isfinite(fro):
            return None
        lam_min_lb = 1.0 / (fro * fro)
        if lam_min_lb < eps_floor or lam_min_lb < _rank_tol(dims[i], C.dtype) * dmax:
            return None
    return [Linv if scales[i] == 1.0 else Linv.mul_(scales[i] ** 0.5) for i, Linv in enumerate(out)]


def mcca_weights_cholesky(C, dims, latent_dimensions, c, eps):
    """MCCA through the Cholesky reduction of the generalised problem (what scipy.linalg.eigh(A, B) does,
    cca_zoo/_utils/_linalg.py:67-71): B_i = R_i/m = L_B L_B^T, K_ij = Linv_i C_ij Linv_j^T (i != j, zero
    diagonal blocks), largest eigenpairs of K by subspace iteration, v_i = sqrt(m) Linv_i^T y_i (v^T B v = 1)."""
    m = len(dims)
    sl = _slices(dims)
    D = C.shape[0]
    k = min(latent_dimensions, D)
    if 4 * k > D:
        return None
    Linv = _cholesky_whiteners(C, dims, c, [1.0] * m, eps)
    if Linv is None:
        return None
    K = torch.zeros((D, D), dtype=C.dtype, device=C.device)
    for i in range(m):
        for j in range(i + 1, m):
            tmp = ops.gemm(Linv[i], C[sl[i], sl[j]])
            ops.gemm(tmp, Linv[j], transb=True, out=K[sl[i], sl[j]])
            K[sl[j], sl[i]] = K[sl[i], sl[j]].T
    cmax = max(c)
    shift = 1.0 / (1.0 - cmax) if cmax <= 0.9 else float(ops.frobenius_norm(K).item())
    res = topk_eigsh(K, k, shift)
    if res is None:
        return None
    _, Yt = res
    return [ops.gemm(Linv[i], Yt[:, sl[i]], transa=True, transb=True, alpha=m ** 0.5) for i in range(m)]


def _pad_null_components(weights, k_out):
    """The reference takes eigenvectors of the n x n matrix, so it returns min(k, n) components even when that
    exceeds the total width D (cca_zoo/_utils/_linalg.py:65); the extra eigenvectors belong to the zero eigenvalue,
    are orthogonal to every view's column space, and pinv(X_i) maps them to zero weights.  Same shape, exact zeros."""
    k = weights[0].shape[1]
    if k_out <= k:
        return weights
    return [torch.cat([w, torch.zeros((w.shape[0], k_out - k), dtype=w.dtype, device=w.device)], dim=1)
            for w in weights]


def gcca_weights_cholesky(C, dims, n_samples, latent_dimensions, c, mu, eps, second_moment=None):
    """GCCA primal form with Cholesky whiteners: Wt_i = sqrt(mu_i) L_i^-1, G = (n-1) Wt C Wt^T (PSD), top-k of
    G by subspace iteration, W_i = C_ii^-1 [C Wt^T U]_i sig^-1/2 (C_ii^-1 from its own Cholesky factor).
    ``second_moment`` (center=False): see ``gcca_weights``."""
    Cd = C if second_moment is None else second_moment
    m = len(dims)
    sl = _slices(dims)
    D = C.shape[0]
    k = min(latent_dimensions, D, n_samples)
    if 4 * k > D:
        return None
    Wt = _cholesky_whiteners(C, dims, c, mu, eps)       # Wt_i = sqrt(mu_i) L_i^-1: a zero view weight zeroes the whitener
    if Wt is None:
        return None
    # factors of the UNregularised blocks for pinv(X_i) = C_ii^-1 X_i^T/(n-1) (full column rank certified); a view with
    # mu_i = 0 is ignored by the eigenproblem but still gets weights (the reference: cca_zoo/linear/_gcca.py:105,109)
    Lc = _cholesky_whiteners(Cd, dims, [0.0] * m, [1.0] * m, 0.0) \
        if (Cd is not C or any(ci != 0.0 for ci in c) or any(x == 0.0 for x in mu)) \
        else [w / (mu[i] ** 0.5) for i, w in enumerate(Wt)]
    if Lc is None:
        return None
    G = torch.empty((D, D), dtype=C.dtype, device=C.device)
    for i in range(m):
        for j in range(i, m):
            tmp = ops.gemm(Wt[i], Cd[sl[i], sl[j]])
            ops.gemm(tmp, Wt[j], transb=True, alpha=float(n_samples - 1), out=G[sl[i], sl[j]])
            if j > i:
                G[sl[j], sl[i]] = G[sl[i], sl[j]].T
    res = topk_eigsh(G, k, 0.0)
    if res is None:
        return None
    sig, Ut = res
    P = torch.empty((D, k), dtype=C.dtype, device=C.device)
    for i in range(m):
        ops.gemm(Wt[i], Ut[:, sl[i]], transa=True, transb=True, out=P[sl[i]])
    CP = ops.gemm(Cd, P)
    out = []
    for i in range(m):
        t1 = ops.gemm(Lc[i], CP[sl[i]])                 # Linv CP_i
        wi = ops.gemm(Lc[i], t1, transa=True)           # Linv^T Linv CP_i = C_ii^-1 CP_i
        out.append(ops.scale(wi, cols=sig, cols_pow=-0.5))
    return _pad_null_components(out, min(latent_dimensions, n_samples))


def rcca_weights_cholesky(C, dims, n_samples, latent_dimensions, c):
    """rCCA through the Cholesky form of the whitening (same weights as ``rcca_weights`` up to sign):
    R_i = (1-c_i) C_ii + c_i I = L_i L_i^T ; T = L_1^-1 C_12 L_2^-T ; weights = L_i^-T U_k / V_k.
    Returns None when a regularised block is not numerically positive definite (the eigen route, which
    reproduces the reference's rank handling, is used instead)."""
    s1, s2 = _slices(dims)
    Linv, infos = [], []
    dmax = torch.stack([C[s, s].diagonal().max() for s in (s1, s2)]).cpu()      # one read-back for both views
    with _two_streams(C.device) as streams:
        for i, s in enumerate((s1, s2)):
            with torch.cuda.stream(streams[i]):       # the two factorisations are independent: run them abreast
                R = (1.0 - c[i]) * C[s, s]
                R.diagonal().add_(c[i])
                tol = _rank_tol(dims[i], C.dtype) * ((1.0 - c[i]) * float(dmax[i]) + c[i])
                # explicit L^-1: everything downstream -- T and the back-substitution of the k weight vectors --
                # becomes plain GEMMs.  R is ridge-regularised and certified positive definite, so
                # cond(L) = sqrt(cond(R)) is benign.
                Li, info = ops.potrf_inv_(R, pivot_tol=tol)
                Linv.append(Li)
                infos.append(info)
    if int(torch.stack(infos).max().item()) != 0:
        return None
    T = ops.gemm(ops.gemm(Linv[0], C[s1, s2]), Linv[1], transb=True)      # L1^-1 C12 L2^-T
    k = min(latent_dimensions, dims[0], dims[1])
    res = topk_svd(T, k) if 4 * k <= min(dims) else None
    if res is None:
        _, Ut, Vt = ops.gesvj(T)
        Ut, Vt = Ut[:k], Vt[:k]
    else:
        _, Ut, Vt = res
    w1 = ops.gemm(Linv[0], Ut, transa=True, transb=True)                   # L1^-T U_k   (d1 x k)
    w2 = ops.gemm(Linv[1], Vt, transa=True, transb=True)
    return [w1, w2]


def rcca_weights(C, dims, n_samples, latent_dimensions, c, solver="auto"):
    """rCCA / CCA / PLS (cca_zoo/linear/_rcca.py:83-101 in covariance form).

    C_ii = V_i L_i V_i^T ; Wt_i = diag(((1-c_i) L_i + c_i)^-1/2) V_i^T (directions with
    lam <= tol*lam_max dropped = the reference's ``s > 0`` filter, _linalg.py:30) ;
    T = Wt_1 C_12 Wt_2^T = U S V^T (one-sided Jacobi) ; weights = Wt_1^T U_k, Wt_2^T V_k.
    """
    if solver == "cholesky" or (solver == "auto" and min(dims) >= 256 and n_samples > max(dims)):
        w = rcca_weights_cholesky(C, dims, n_samples, latent_dimensions, c)
        if w is not None:
            return w
    s1, s2 = _slices(dims)
    lams, vts = _block_eigh(C, dims)
    wts, ranks = [], []
    for i in range(2):
        Wt, _, rank = ops.whiten_rows(lams[i], vts[i], c[i], rank_tol=_regularised_rank_tol(lams[i], c[i], dims[i]),
                                      max_rank=min(n_samples, dims[i]))
        wts.append(Wt)
        ranks.append(rank)
    r1, r2 = (int(r.item()) for r in ranks)  # host read-back: decides k (_rcca.py:95)
    k = min(latent_dimensions, r1, r2)
    tmp = ops.gemm(wts[0], C[s1, s2])                 # (d1 x d2)
    T = ops.gemm(tmp, wts[1], transb=True)            # (d1 x d2) in whitened coordinates
    # gesvj factors G = T^T given by columns, i.e. the row-major buffer of T itself:
    #   right vectors of G = left singular vectors U of T, left vectors of G = right singular vectors V of T
    _, Ut, Vt = ops.gesvj(T)
    w1 = ops.gemm(wts[0], Ut[:k], transa=True, transb=True)   # (d1 x k)
    w2 = ops.gemm(wts[1], Vt[:k], transa=True, transb=True)   # (d2 x k)
    return [w1, w2]


#: above this total width the dense Jacobi route (O(D^3) per sweep on a D x D matrix) is refused instead of being
#: entered silently when the top-k route declines: at D = 16384 it would run for hours
_MAX_DENSE_JACOBI = 8192


def _refuse_dense(D, what):
    if D > _MAX_DENSE_JACOBI:
        raise RuntimeError(
            f"{what}: the top-k (Cholesky + subspace iteration) route declined on a {D} x {D} problem (a block is "
            f"not positive definite, an eps floor may be active, 4k > D, or no spectral gap after the block) and "
            f"the dense Jacobi route is limited to D <= {_MAX_DENSE_JACOBI}.  Regularise (c > 0) or reduce "
            f"latent_dimensions.")


def mcca_weights(C, dims, latent_dimensions, c, eps, solver="auto"):
    """MCCA (cca_zoo/linear/_mcca.py:113-135,141-173): top-k of A v = lam B v, v^T B v = 1 with
    A = (C - blkdiag C_ii)/m, B = blkdiag((1-c_i) C_ii + c_i I)/m (+ eps floor).

    With B_i = V_i diag(b_i) V_i^T and Wt_i = diag(b_i^-1/2) V_i^T the problem becomes the standard
    symmetric one K y = lam y, K_ij = Wt_i A_ij Wt_j^T, v_i = Wt_i^T y_i.  K is indefinite (for two
    views its spectrum is +-sigma), so it is solved shifted by ||K||_F to keep +-pairs apart.
    """
    if solver == "cholesky" or (solver == "auto" and C.shape[0] >= 512):
        w = mcca_weights_cholesky(C, dims, latent_dimensions, c, eps)
        if w is not None:
            return w
    _refuse_dense(C.shape[0], "MCCA")
    m = len(dims)
    sl = _slices(dims)
    D = C.shape[0]
    lams, vts = _block_eigh(C, dims)
    # eps floor of _build_B (:170-172): lambda_min of the block-diagonal B is the min over blocks
    min_eig = min(float(((1.0 - c[i]) * lams[i][-1] + c[i]).item()) for i in range(m))
    floor = (eps - min_eig) if min_eig < eps else 0.0
    wts = []
    for i in range(m):
        Wt, _, _ = ops.whiten_rows(lams[i], vts[i], c[i], floor_add=floor, scale=1.0 / m, rank_tol=-1.0)
        wts.append(Wt)
    K = torch.zeros((D, D), dtype=C.dtype, device=C.device)
    for i in range(m):
        for j in range(i + 1, m):
            tmp = ops.gemm(wts[i], C[sl[i], sl[j]])
            ops.gemm(tmp, wts[j], transb=True, alpha=1.0 / m, out=K[sl[i], sl[j]])
            K[sl[j], sl[i]] = K[sl[i], sl[j]].T
    shift = float(ops.frobenius_norm(K).item())
    evals, evt = ops.syevj(K, shift=shift)
    k = min(latent_dimensions, D)
    return [ops.gemm(wts[i], evt[:k, sl[i]], transa=True, transb=True) for i in range(m)]


def gcca_weights(C, dims, n_samples, latent_dimensions, c, mu, eps, solver="auto", second_moment=None):
    """GCCA in primal (D x D) form (cca_zoo/linear/_gcca.py:94-109; SURVEY.md §3.3).

    reg_i = (1-c_i) L_i + c_i (+ per-view eps floor, :102-104) ; Wt_i = diag(sqrt(mu_i) reg_i^-1/2) V_i^T ;
    G = (n-1) Wt C Wt^T (block-wise) ; top-k G u = sig u ;
    W_i = pinv(C_ii) [C Wt^T u]_i sig^-1/2   (pinv from the same eigendecomposition).

    ``second_moment`` = X^T X / (n-1) WITHOUT mean subtraction, given when the estimator was built with
    ``center=False``: the reference then still regularises with ``np.cov`` (centred, :98-100) but forms
    ``v R^-1 v^T`` and ``pinv(v)`` from the raw views (:105,109), so G, the projection and the pseudo-inverse use
    the second moment while the whiteners use the covariance.
    """
    if solver == "cholesky" or (solver == "auto" and C.shape[0] >= 512):
        w = gcca_weights_cholesky(C, dims, n_samples, latent_dimensions, c, mu, eps, second_moment)
        if w is not None:
            return w
    _refuse_dense(C.shape[0], "GCCA")
    Cd = C if second_moment is None else second_moment
    m = len(dims)
    sl = _slices(dims)
    D = C.shape[0]
    lams, vts = _block_eigh(C, dims)
    lams_d, vts_d = (lams, vts) if Cd is C else _block_eigh(Cd, dims)
    wts = []
    for i in range(m):
        reg_min = float(((1.0 - c[i]) * lams[i][-1] + c[i]).item())
        floor = (eps - reg_min) if reg_min < eps else 0.0
        if mu[i] == 0.0:                                   # ignored view: zero whitener (no division by mu)
            wts.append(torch.zeros((dims[i], dims[i]), dtype=C.dtype, device=C.device))
            continue
        Wt, _, _ = ops.whiten_rows(lams[i], vts[i], c[i], floor_add=floor, scale=1.0 / mu[i], rank_tol=-1.0)
        wts.append(Wt)
    G = torch.empty((D, D), dtype=C.dtype, device=C.device)
    for i in range(m):
        for j in range(i, m):
            tmp = ops.gemm(wts[i], Cd[sl[i], sl[j]])
            ops.gemm(tmp, wts[j], transb=True, alpha=float(n_samples - 1), out=G[sl[i], sl[j]])
            if j > i:
                G[sl[j], sl[i]] = G[sl[i], sl[j]].T
    sig, evt = ops.syevj(G)
    k = min(latent_dimensions, D, n_samples)
    # P = blkdiag(Wt_i^T) U_k   (D x k)
    P = torch.empty((D, k), dtype=C.dtype, device=C.device)
    for i in range(m):
        ops.gemm(wts[i], evt[:k, sl[i]], transa=True, transb=True, out=P[sl[i]])
    CP = ops.gemm(Cd, P)                                                  # (D x k)
    out = []
    for i in range(m):
        tol = _rank_tol(dims[i], C.dtype)
        # pinv(C_ii) = V diag(1/lam | lam > tol lam_max) V^T  via whiten_rows with c=0 (g = lam^-1/2) twice
        Pinv_half, _, _ = ops.whiten_rows(lams_d[i], vts_d[i], 0.0, rank_tol=tol)   # diag(lam^-1/2) V^T
        t1 = ops.gemm(Pinv_half, CP[sl[i]])                                      # (d x k)
        wi = ops.gemm(Pinv_half, t1, transa=True)                                # V lam^-1 V^T CP_i
        out.append(ops.scale(wi, cols=sig[:k], cols_pow=-0.5))
    return _pad_null_components(out, min(latent_dimensions, n_samples))
