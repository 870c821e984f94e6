"""CPU restatement (numpy, float64) of the Eckart-Young gradient estimators of the reference
(cca_zoo/linear/gradient/: CCA_EY, PLS_EY, MCCA_EY).

TEST INFRASTRUCTURE ONLY -- the checker of csrc/ey.cu, in three forms:

* ``ref_ey_fit`` -- the reference's data-space loop (cca_zoo/linear/gradient/_base.py:113-130), restated;
* ``cov_step`` -- the covariance-route step the CUDA kernel implements for full batches;
* ``mb_step`` -- the mini-batch step on the raw (uncentred) views, as the kernel gathers them.

All three return / carry the per-step ``|prev_obj - obj|`` so that callers can tell how far a ``tol`` test is from
flipping.
"""
from __future__ import annotations

import numpy as np

from .restatement import block_slices, setup_fit

EY_KINDS = ("cca", "pls", "mcca")


# ---------------------------------------------------------------------------------------------------- initialisation
def ey_init(views_, kind, k, bs, rng):
    """Initial weights (cca_zoo/_utils/_ey.py:120-126 for PLS_EY, :173-184 for CCA_EY / MCCA_EY) drawn from ``rng`` in
    the reference's order; ``views_`` are the views after _setup_fit (centred when ``center``)."""
    n = views_[0].shape[0]
    idx = rng.choice(n, bs, replace=False) if kind != "pls" else None
    out = []
    for v in views_:
        w0, _ = np.linalg.qr(rng.standard_normal((v.shape[1], k)))
        if kind != "pls":
            _, r = np.linalg.qr(v[idx] @ w0)
            w0 = w0 @ np.linalg.solve(r, np.eye(k))
        out.append(w0)
    return out


def stacked_r(z0):
    """R of the Householder QR of z0 (n x k, n >= 2k) from k of its rows and its Gram matrix only: the QR of the
    2k x k stack [z0[:k]; chol(z0^T z0 - z0[:k]^T z0[:k])^T]."""
    k = z0.shape[1]
    head = z0[:k]
    L = np.linalg.cholesky(z0.T @ z0 - head.T @ head)
    return np.linalg.qr(np.vstack([head, L.T]), mode="r")


# ---------------------------------------------------------------------------------------------------- the reference
def _cov_pair(reps):
    n, m = reps[0].shape[0], len(reps)
    cen = [z - z.mean(axis=0) for z in reps]
    k = cen[0].shape[1]
    C, V = np.zeros((k, k)), np.zeros((k, k))
    for zi in cen:
        V += zi.T @ zi / (n - 1)
        for zj in cen:
            C += zi.T @ zj / (n - 1)
    return C / m, V / m


def _objective(reps, W, c):
    C, V = _cov_pair(reps)
    B = sum(w.T @ w for w in W) / len(W)
    Vb = (1 - c) * V + c * B
    return float(-2.0 * np.trace(C - c * V) + np.trace(Vb @ Vb))


def ref_ey_fit(views, kind, k, c=0.0, learning_rate=1e-2, max_iter=1000, batch_size=None, tol=1e-6, momentum=0.9,
               random_state=None, center=True):
    """The reference's fit, restated: (weights, steps taken, per-step |prev_obj - obj|)."""
    views_, _ = setup_fit(views, center)
    c = 1.0 if kind == "pls" else c
    n, m = views_[0].shape[0], len(views_)
    bs = n if batch_size is None else min(batch_size, n)
    rng = np.random.default_rng(random_state)
    W = ey_init(views_, kind, k, bs, rng)
    vel = [np.zeros_like(w) for w in W]
    prev, deltas = np.inf, []
    for _ in range(max_iter):
        idx = rng.choice(n, bs, replace=False)
        batch = [v[idx] for v in views_]
        reps = [b @ w for b, w in zip(batch, W)]
        cen = [z - z.mean(axis=0) for z in reps]
        total = sum(cen)
        _, V = _cov_pair(reps)
        Vb = (1 - c) * V + c * sum(w.T @ w for w in W) / m
        scale = 4.0 / (m * (bs - 1))
        g = [(b - b.mean(axis=0)).T @ (scale * (c * z + (1 - c) * (z @ Vb) - total)) + (4.0 * c / m) * (w @ Vb)
             for b, z, w in zip(batch, cen, W)]
        for i, gi in enumerate(g):
            vel[i] = momentum * vel[i] - learning_rate * gi
            W[i] = W[i] + vel[i]
        obj = _objective(reps, W, c)
        deltas.append(abs(prev - obj))
        if abs(prev - obj) < tol:
            break
        prev = obj
    return W, len(deltas), deltas


# ---------------------------------------------------------------------------------------------------- kernel forms
def new_state(W):
    return {"W": [np.array(w, dtype=np.float64) for w in W], "vel": [np.zeros_like(w, dtype=np.float64) for w in W],
            "prev": np.inf, "steps": 0, "stop": False, "deltas": []}


def _finish_step(st, V, Ce, g, c, lr, momentum, tol):
    m = len(st["W"])
    for i, gi in enumerate(g):
        st["vel"][i] = momentum * st["vel"][i] - lr * gi
        st["W"][i] = st["W"][i] + st["vel"][i]
    Bn = sum(w.T @ w for w in st["W"]) / m
    Vb = (1 - c) * V + c * Bn
    obj = float(-2.0 * np.trace(Ce - c * V) + np.trace(Vb @ Vb))
    d = abs(st["prev"] - obj)
    st["deltas"].append(d)
    st["steps"] += 1
    st["stop"] = bool(d < tol)
    st["prev"] = obj


def cov_step(st, C, dims, c, lr, momentum, tol):
    """One full-batch step on the centred block covariance C (D x D)."""
    if st["stop"]:
        return
    sl = block_slices(dims)
    W, m = st["W"], len(dims)
    Y = [[C[sl[i], sl[j]] @ W[j] for j in range(m)] for i in range(m)]
    V = sum(W[i].T @ Y[i][i] for i in range(m)) / m
    Ce = sum(W[i].T @ Y[i][j] for i in range(m) for j in range(m)) / m
    Vb = (1 - c) * V + c * sum(w.T @ w for w in W) / m
    g = [4 / m * (c * Y[i][i] + (1 - c) * Y[i][i] @ Vb - sum(Y[i])) + 4 * c / m * W[i] @ Vb for i in range(m)]
    _finish_step(st, V, Ce, g, c, lr, momentum, tol)


def mb_step(st, views, idx, c, lr, momentum, tol):
    """One mini-batch step on the rows ``idx`` of the RAW views (no global centring)."""
    if st["stop"]:
        return
    W, m, bs = st["W"], len(views), len(idx)
    Xb = [np.asarray(v[idx], dtype=np.float64) for v in views]
    Z = [x @ w for x, w in zip(Xb, W)]
    Zc = [z - z.mean(axis=0) for z in Z]
    S = sum(Zc)
    V = sum(z.T @ z for z in Zc) / (m * (bs - 1))
    Ce = S.T @ S / (m * (bs - 1))
    Vb = (1 - c) * V + c * sum(w.T @ w for w in W) / m
    scale = 4.0 / (m * (bs - 1))
    g = [x.T @ (scale * (c * z + (1 - c) * z @ Vb - S)) + 4 * c / m * w @ Vb for x, z, w in zip(Xb, Zc, W)]
    _finish_step(st, V, Ce, g, c, lr, momentum, tol)


def cov_ey_fit(views, kind, k, c=0.0, learning_rate=1e-2, max_iter=1000, tol=1e-6, momentum=0.9, random_state=None,
               center=True, C=None):
    """Full-batch fit by the covariance route: (weights, steps, deltas).  ``C`` defaults to the centred covariance of
    the views in float64."""
    views_, _ = setup_fit([np.asarray(v, dtype=np.float64) for v in views], center)
    c = 1.0 if kind == "pls" else c
    n = views_[0].shape[0]
    rng = np.random.default_rng(random_state)
    st = new_state(ey_init(views_, kind, k, n, rng))
    if C is None:
        X = np.hstack(views_)
        X = X - X.mean(axis=0)
        C = X.T @ X / (n - 1)
    dims = [v.shape[1] for v in views_]
    for _ in range(max_iter):
        cov_step(st, C, dims, c, learning_rate, momentum, tol)
        if st["stop"]:
            break
    return st["W"], st["steps"], st["deltas"]


def mb_ey_fit(views, kind, k, batch_size, c=0.0, learning_rate=1e-2, max_iter=1000, tol=1e-6, momentum=0.9,
              random_state=None, center=True):
    """Mini-batch fit in the kernel's form (raw views, batch-local centring): (weights, steps, deltas)."""
    raw = [np.asarray(v, dtype=np.float64) for v in views]
    views_, _ = setup_fit(raw, center)
    c = 1.0 if kind == "pls" else c
    n = raw[0].shape[0]
    bs = min(batch_size, n)
    rng = np.random.default_rng(random_state)
    st = new_state(ey_init(views_, kind, k, bs, rng))
    for _ in range(max_iter):
        mb_step(st, raw, rng.choice(n, bs, replace=False), c, learning_rate, momentum, tol)
        if st["stop"]:
            break
    return st["W"], st["steps"], st["deltas"]
