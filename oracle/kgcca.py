"""KGCCA restated in numpy (cca_zoo/nonparametric/_kgcca.py).  TEST INFRASTRUCTURE ONLY.

``ref_kgcca_fit``  the reference's data-space fit: Q = sum_i mu_i K_i B_i^-1 K_i with B_i = c_i K_i + (1 - c_i) K_i^2
                   floored at eps per view, the top-k eigenvectors T of Q from scipy's eigh, weights_i = pinv(K_i) T.
``eig_kgcca_fit``  the route cca_zoo_b200.nonparametric.KGCCA takes on the device: one eigendecomposition per kernel
                   matrix, the per-view floor from the eigenvalues, Q summed in the eigenbases, the top-k eigenvectors
                   of Q and the clean pseudo-inverse (|lambda| <= n eps_mach max|lambda| zeroed).
"""
from __future__ import annotations

import numpy as np
import scipy.linalg

from oracle.kcca import _perview, kernel_settings, kernels, setup


def ref_kgcca_fit(views, k, c=0.1, eps=1e-6, center=True, view_weights=None, **kernel_kw):
    """The reference's fit: (weights per view, centred training views, kernel settings)."""
    X, _ = setup(views, center)
    m, n = len(X), X[0].shape[0]
    st = kernel_settings(m, **kernel_kw)
    Ks = kernels(X, st)
    Q = np.zeros((n, n))
    for K, ci, mi in zip(Ks, _perview(c, 0.1, m), _perview(view_weights, 1.0, m)):
        B = ci * K + (1.0 - ci) * K @ K
        lmin = np.linalg.eigvalsh(B).min()
        if lmin < eps:
            B += (eps - lmin) * np.eye(n)
        Q += mi * K @ np.linalg.inv(B) @ K
    kk = min(k, n)
    w, V = scipy.linalg.eigh(Q, subset_by_index=[n - kk, n - 1])
    T = V[:, np.argsort(w)[::-1]]
    return [np.linalg.pinv(K) @ T for K in Ks], X, st


def eig_kgcca_fit(views, k, c=0.1, eps=1e-6, center=True, view_weights=None, info=None, **kernel_kw):
    """The eigenbasis route: (weights per view, centred training views, kernel settings).  ``info`` (a dict) receives
    Q, its eigenvalues (descending) and min f_i per view."""
    X, _ = setup(views, center)
    m, n = len(X), X[0].shape[0]
    st = kernel_settings(m, **kernel_kw)
    eig = [np.linalg.eigh(K) for K in kernels(X, st)]
    Q, plus, fmin = np.zeros((n, n)), [], []
    for (lam, U), ci, mi in zip(eig, _perview(c, 0.1, m), _perview(view_weights, 1.0, m)):
        f = ci * lam + (1.0 - ci) * lam * lam
        s = eps - f.min() if f.min() < eps else 0.0
        Q += (U * (mi * lam * lam / (f + s))) @ U.T
        keep = np.abs(lam) > n * np.finfo(np.float64).eps * np.abs(lam).max()
        plus.append(np.where(keep, 1.0 / np.where(keep, lam, 1.0), 0.0))
        fmin.append(float(f.min()))
    w, Y = np.linalg.eigh(Q)
    w, Y = w[::-1], Y[:, ::-1]
    T = Y[:, :min(k, n)]
    if info is not None:
        info.update(Q=Q, evals=w, fmin=fmin)
    return [U @ (p[:, None] * (U.T @ T)) for (_, U), p in zip(eig, plus)], X, st
