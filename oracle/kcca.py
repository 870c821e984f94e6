"""KCCA restated in numpy (cca_zoo/nonparametric/_kcca.py).  TEST INFRASTRUCTURE ONLY.

``ref_kcca_fit``   the reference's data-space fit: A from np.cov of the hstacked kernel matrices, B = blockdiag(c K +
                   (1 - c) K^2) with its eps floor, the top-k generalised eigenvectors of (A, B) from scipy's eigh.
``eig_kcca_fit``   the route cca_zoo_b200.nonparametric.KCCA takes on the device: one eigendecomposition per kernel
                   matrix, the floor from the eigenvalues, the same keep rule, the whitened matrix T and its top-k
                   eigenvectors.
``kernels``        the kernel matrices as the reference builds them (sklearn's pairwise_kernels, filter_params=True).
"""
from __future__ import annotations

import numpy as np
import scipy.linalg
from scipy.linalg import block_diag
from sklearn.metrics import pairwise_kernels


def _perview(value, default, m):
    if value is None:
        return [default] * m
    return list(value) if isinstance(value, list) else [value] * m


def setup(views, center=True):
    """(views as float64, centred when ``center``; their means)."""
    views = [np.asarray(v, dtype=np.float64) for v in views]
    means = [v.mean(axis=0) if center else np.zeros(v.shape[1]) for v in views]
    return [v - mu for v, mu in zip(views, means)], means


def kernel_settings(m, kernel="linear", gamma=None, degree=1.0, coef0=1.0, kernel_params=None):
    """Per view keyword arguments of the reference's pairwise_kernels calls."""
    ker, gam = _perview(kernel, "linear", m), _perview(gamma, None, m)
    deg, co, kp = _perview(degree, 1.0, m), _perview(coef0, 1.0, m), _perview(kernel_params, {}, m)
    return [dict(metric=ker[i], gamma=gam[i], degree=deg[i], coef0=co[i], filter_params=True, **(kp[i] or {}))
            for i in range(m)]


def kernels(views, settings, test=None):
    """K_i = k_i(views_i) (or k_i(views_i, test_i) when ``test`` is given)."""
    if test is None:
        return [pairwise_kernels(v, **s) for v, s in zip(views, settings)]
    return [pairwise_kernels(v, Y=t, **s) for v, t, s in zip(views, test, settings)]


def ref_kcca_fit(views, k, c=0.1, eps=1e-3, center=True, **kernel_kw):
    """The reference's fit: (weights per view, centred training views, kernel settings)."""
    X, _ = setup(views, center)
    m = len(X)
    st = kernel_settings(m, **kernel_kw)
    Ks = kernels(X, st)
    cs = _perview(c, 0.1, m)
    A = np.cov(np.hstack(Ks), rowvar=False)
    A -= block_diag(*[np.cov(K, rowvar=False) for K in Ks])
    A /= m
    B = np.asarray(block_diag(*[ci * K + (1.0 - ci) * K @ K for ci, K in zip(cs, Ks)]))
    lmin = np.linalg.eigvalsh(B).min()
    if lmin < eps:
        B += (eps - lmin) * np.eye(B.shape[0])
    B /= m
    p = A.shape[0]
    kk = min(k, p)
    w, V = scipy.linalg.eigh(A, B, subset_by_index=[p - kk, p - 1])
    V = V[:, np.argsort(w)[::-1]]
    n = X[0].shape[0]
    return [V[i * n:(i + 1) * n] for i in range(m)], X, st


def eig_kcca_fit(views, k, c=0.1, eps=1e-3, center=True, info=None, **kernel_kw):
    """The eigenbasis route: (weights per view, centred training views, kernel settings).  ``info`` (a dict) receives
    the eigenvalues of T (descending), lambda_min(B) and the kept ranks."""
    X, _ = setup(views, center)
    m, n = len(X), X[0].shape[0]
    st = kernel_settings(m, **kernel_kw)
    Ks = kernels(X, st)
    cs = _perview(c, 0.1, m)
    eig = [np.linalg.eigh(K) for K in Ks]
    f = [ci * lam + (1.0 - ci) * lam * lam for ci, (lam, _) in zip(cs, eig)]
    fmin = min(x.min() for x in f)
    s = eps - fmin if fmin < eps else 0.0
    beta = [(x + s) / m for x in f]
    D = [lam / np.sqrt(b) / np.sqrt(m * (n - 1.0)) for (lam, _), b in zip(eig, beta)]
    cut = n * np.finfo(np.float64).eps * max(np.abs(x).max() for x in D)
    keep = [np.abs(x) > cut for x in D]
    U = [u[:, kp] for (_, u), kp in zip(eig, keep)]
    Dk = [x[kp] for x, kp in zip(D, keep)]
    r = [u.shape[1] for u in U]
    off = np.concatenate([[0], np.cumsum(r)]).astype(int)
    T = np.zeros((off[-1], off[-1]))
    for i in range(m):
        for j in range(m):
            if i != j:
                P = U[i].T @ U[j] - np.outer(U[i].sum(axis=0), U[j].sum(axis=0)) / n
                T[off[i]:off[i + 1], off[j]:off[j + 1]] = Dk[i][:, None] * P * Dk[j][None, :]
    w, Y = np.linalg.eigh(T)
    w, Y = w[::-1], Y[:, ::-1]
    kk = min(k, m * n)
    if info is not None:
        info.update(evals=w, lmin_B=fmin, ranks=r)
    Wt = [U[i] @ (Y[off[i]:off[i + 1], :kk] / np.sqrt(beta[i][keep[i]])[:, None]) for i in range(m)]
    return Wt, X, st


def transform(train_views, settings, weights, test):
    """The reference's transform: k_i(train_views_i, test_i)^T weights_i, the test views not centred."""
    return [K.T @ w for K, w in zip(kernels(train_views, settings, test), weights)]


def score(train_views, settings, weights, test):
    """The reference's score: the mean off-diagonal correlation of the transformed test views per dimension."""
    T = np.stack(transform(train_views, settings, weights, test))
    T = T - T.mean(axis=1, keepdims=True)
    nrm = np.sqrt((T ** 2).sum(axis=1, keepdims=True))
    T = T / np.where(nrm > 1e-12, nrm, 1.0)
    C = np.einsum("isd,jsd->ijd", T, T)
    m = C.shape[0]
    return (C.sum(axis=(0, 1)) - sum(C[i, i] for i in range(m))) / (m * (m - 1))


def align(w, ref):
    """``w`` with each column's sign flipped to agree with ``ref`` (the same column of all views together)."""
    s = np.sign(sum(np.sum(a * b, axis=0) for a, b in zip(w, ref)))
    s[s == 0] = 1.0
    return [a * s for a in w]


def rel_err(w, ref):
    """max over views of max|w - ref| / max|ref| after sign alignment."""
    w = align(w, ref)
    return max(float(np.abs(a - b).max()) / max(float(np.abs(b).max()), 1e-300) for a, b in zip(w, ref))
