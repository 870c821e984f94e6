"""KTCCA restated in numpy (cca_zoo/nonparametric/_ktcca.py).  TEST INFRASTRUCTURE ONLY.

``ref_ktcca_fit``  the reference's data-space fit: invsqrt_i = inv(sqrtm((1 - c_i) K_i^2 + c_i K_i)) floored at eps per
                   view, the n x n x ... x n array of per-sample outer products of the rows of K_i invsqrt_i averaged
                   over the samples, then tensorly's ``parafac`` (oracle/tcca.py:parafac); weights_i = invsqrt_i F_i.
``eig_ktcca_fit``  the route cca_zoo_b200.nonparametric.KTCCA takes on the device: one eigendecomposition per kernel
                   matrix, the per-view floor from the eigenvalues, Z_i = V_i diag(lambda_i h_i) V_i^T, the Khatri-Rao
                   contraction M = Z_1^T KR(Z_2, ..., Z_m) / n, the Gram start and ``als_step`` of oracle/tcca.py, and
                   weights_i = V_i diag(h_i) V_i^T F_i.
"""
from __future__ import annotations

import numpy as np
from scipy.linalg import sqrtm

from oracle import tcca as TC
from oracle.kcca import _perview, kernel_settings, kernels, setup


def ref_ktcca_fit(views, k, c=0.1, eps=1e-3, center=True, random_state=None, info=None, **kernel_kw):
    """The reference's fit: (weights per view, centred training views, kernel settings).  ``info`` goes to
    ``parafac``."""
    X, _ = setup(views, center)
    m = len(X)
    st = kernel_settings(m, **kernel_kw)
    whitened, invs = [], []
    for K, ci in zip(kernels(X, st), _perview(c, 0.1, m)):
        cov = (1.0 - ci) * K @ K + ci * K
        lmin = np.linalg.eigvalsh(cov).min()
        if lmin < eps:
            cov += (eps - lmin) * np.eye(cov.shape[0])
        inv = np.linalg.inv(sqrtm(cov).real)
        whitened.append(K @ inv)
        invs.append(inv)
    M = whitened[0]
    for wk in whitened[1:]:
        for _ in range(M.ndim - 1):
            wk = np.expand_dims(wk, 1)
        M = np.expand_dims(M, -1) @ wk
    M = M.mean(axis=0)
    cp = TC.parafac(M, k, random_state=random_state, info=info)
    return [inv @ f for inv, f in zip(invs, cp.factors)], X, st


def eig_ktcca_fit(views, k, c=0.1, eps=1e-3, center=True, random_state=None, info=None, **kernel_kw):
    """The eigenbasis route: (weights per view, centred training views, kernel settings).  ``info`` (a dict) receives
    the final ALS state and min f_i per view."""
    X, _ = setup(views, center)
    m, n = len(X), X[0].shape[0]
    st = kernel_settings(m, **kernel_kw)
    Z, H, fmin = [], [], []
    for K, ci in zip(kernels(X, st), _perview(c, 0.1, m)):
        lam, U = np.linalg.eigh(K)
        f = ci * lam + (1.0 - ci) * lam * lam
        h = 1.0 / np.sqrt(f + (eps - f.min() if f.min() < eps else 0.0))
        Z.append((U * (lam * h)) @ U.T)
        H.append((U, h))
        fmin.append(float(f.min()))
    M = TC.krprod_moment(Z).reshape([n] * m)
    state = TC.gram_start(M, k, TC.random_columns(M.shape, k, TC.rng_of(random_state)))
    for _ in range(TC.N_ITER_MAX):
        TC.als_step(state, M)
        if state["stop"]:
            break
    if state["singular"]:
        raise np.linalg.LinAlgError("Singular matrix")
    if info is not None:
        info.update(state=state, fmin=fmin)
    return [U @ (h[:, None] * (U.T @ F)) for (U, h), F in zip(H, state["F"])], X, st
