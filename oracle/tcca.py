"""Float64 restatements of TCCA (cca_zoo/linear/_tcca.py).

TEST INFRASTRUCTURE ONLY.

  * ``parafac`` restates tensorly 0.8's default ``parafac(tensor, rank, random_state=...)`` path, the one the reference
    calls: ``init='svd'`` with sign-flipped truncated SVD starts, unnormalised ALS with an exact solve per mode, and the
    absolute reconstruction-error stop rule (tol 1e-8, at most 100 iterations).
  * ``ref_tcca_fit`` is the reference's data-space path: centred views, ``inv(sqrtm(cov))`` whiteners, the n x p_1 x
    ... x p_m outer-product array averaged over samples, then ``parafac``.
  * ``cov_tcca_fit`` is the device algorithm: moments, eigen whiteners, the Khatri-Rao contraction
    M_(0) = Z_1^T KR(Z_2, ..., Z_m) / n, the start from the eigenvectors of the unfolding Grams M_(j) M_(j)^T, then
    ``als_step`` on the state ``start_state`` returns -- the layout ``ccab_tcca_fit`` keeps on the device.
"""
from __future__ import annotations

import numpy as np
from scipy.linalg import sqrtm

N_ITER_MAX = 100
TOL = 1e-8


def unfold(M, j):
    """tensorly's unfolding: mode j first, the remaining modes in C order."""
    return np.moveaxis(M, j, 0).reshape(M.shape[j], -1)


def khatri_rao(factors):
    """Row-wise Khatri-Rao product, the first factor's row index varying slowest."""
    out = factors[0]
    for f in factors[1:]:
        out = (out[:, None, :] * f[None, :, :]).reshape(-1, out.shape[1])
    return out


def mttkrp(M, factors, j):
    return unfold(M, j) @ khatri_rao([f for i, f in enumerate(factors) if i != j])


def svd_flip(U):
    """tensorly's U-based ``svd_flip``: the entry of largest |value| of each column (the first on ties) positive."""
    rows = np.argmax(np.abs(U), axis=0)
    signs = np.sign(U[rows, np.arange(U.shape[1])])
    return U * signs


def rng_of(random_state):
    """tensorly's ``check_random_state``: the global numpy RandomState for None."""
    if random_state is None:
        return np.random.mtrand._rand
    return np.random.RandomState(random_state)


def random_columns(shape, k, rng):
    """The random start columns of every mode with p_j < k, drawn in mode order (a list with None elsewhere)."""
    return [rng.random_sample((p, k - p)) if p < k else None for p in shape]


def assemble_start(shape, k, vecs, sigma0, rand):
    """Start factors from the leading left singular vectors ``vecs[j]`` (p_j x min(k, p_j)) of every unfolding:
    the sign rule, mode 0 scaled by its singular values, then the random columns."""
    factors = []
    for j, p in enumerate(shape):
        U = svd_flip(vecs[j])
        if j == 0:
            U = U * sigma0[:U.shape[1]]
        if p < k:
            U = np.concatenate([U, rand[j]], axis=1)
        factors.append(U[:, :k])
    return factors


def new_state(M, factors):
    return {"F": [np.array(f, dtype=np.float64) for f in factors], "iters": 0, "stop": False, "singular": False,
            "rec": [], "norm": float(np.linalg.norm(M.reshape(-1)))}


def als_step(state, M):
    """One tensorly ALS iteration on ``state`` (in place): for each mode in order, V = Hadamard product of the other
    factors' Grams, F_j = solve(V^T, MTTKRP_j^T)^T; then the reconstruction error and the stop test."""
    if state["stop"]:
        return state
    F = state["F"]
    k = F[0].shape[1]
    m = len(F)
    for j in range(m):
        V = np.ones((k, k))
        for i, f in enumerate(F):
            if i != j:
                V = V * (f.T @ f)
        mt = mttkrp(M, F, j)
        try:
            F[j] = np.linalg.solve(V.T, mt.T).T
        except np.linalg.LinAlgError:
            state["singular"] = state["stop"] = True
            return state
    V = np.ones((k, k))
    for f in F:
        V = V * (f.T @ f)
    norm = state["norm"]
    rec = np.sqrt(abs(norm ** 2 + V.sum() - 2.0 * np.sum(mt * F[m - 1]))) / norm
    state["rec"].append(float(rec))
    if state["iters"] >= 1 and abs(state["rec"][-2] - rec) < TOL:
        state["stop"] = True
    state["iters"] += 1
    return state


class CPTensor:
    def __init__(self, factors):
        self.weights = np.ones(factors[0].shape[1])
        self.factors = factors


def parafac(tensor, rank, random_state=None, n_iter_max=N_ITER_MAX, info=None, **_):
    """tensorly 0.8 ``parafac`` at its defaults (float64).  ``info`` (a dict, optional) receives the iteration count,
    the reconstruction errors and the start's relative singular-value gaps."""
    M = np.asarray(tensor, dtype=np.float64)
    k = int(rank)
    rng = rng_of(random_state)
    vecs, gaps, sigma0 = [], [], None
    rand = []
    for j, p in enumerate(M.shape):
        U, S, _ = np.linalg.svd(unfold(M, j), full_matrices=False)
        kk = min(k, p)
        vecs.append(U[:, :kk])
        if j == 0:
            sigma0 = S
        if kk < len(S):
            gaps.append((S[kk - 1] - S[kk]) / S[0])
        rand.append(rng.random_sample((p, k - p)) if p < k else None)
    state = new_state(M, assemble_start(M.shape, k, vecs, sigma0, rand))
    for _ in range(n_iter_max):
        als_step(state, M)
        if state["stop"]:
            break
    if state["singular"]:
        raise np.linalg.LinAlgError("Singular matrix")
    if info is not None:
        info.update(iters=state["iters"], rec=list(state["rec"]), gaps=gaps, stop=state["stop"])
    return CPTensor(state["F"])


# --------------------------------------------------------------------------------------------------------------------
def _per_view(c, m):
    return [float(x) for x in c] if isinstance(c, (list, tuple, np.ndarray)) else [float(c)] * m


def ref_tcca_fit(views, k, center=True, c=0.0, eps=1e-6, random_state=None, info=None):
    """The reference's TCCA.fit in numpy: (weights, means)."""
    views = [np.asarray(v, dtype=np.float64) for v in views]
    means = [v.mean(axis=0) for v in views]
    if center:
        views = [v - mu for v, mu in zip(views, means)]
    cs = _per_view(c, len(views))
    whitened, invs = [], []
    for v, ci in zip(views, cs):
        cov = (1.0 - ci) * np.cov(v, rowvar=False) + ci * np.eye(v.shape[1])
        lmin = np.linalg.eigvalsh(cov).min()
        if lmin < eps:
            cov += (eps - lmin) * np.eye(cov.shape[0])
        inv = np.linalg.inv(sqrtm(cov).real)
        whitened.append(v @ inv)
        invs.append(inv)
    M = whitened[0]
    for wv in whitened[1:]:
        for _ in range(M.ndim - 1):
            wv = np.expand_dims(wv, 1)
        M = np.expand_dims(M, -1) @ wv
    M = M.mean(axis=0)
    cp = parafac(M, k, random_state=random_state, info=info)
    return [inv @ f for inv, f in zip(invs, cp.factors)], means


def whiteners(views, c=0.0, eps=1e-6):
    """Eigen whiteners S_i = V (lam + floor)^-1/2 V^T of (1 - c_i) cov_i + c_i I (cov always centred, ddof = 1)."""
    out = []
    for v, ci in zip(views, _per_view(c, len(views))):
        lam, V = np.linalg.eigh(np.cov(np.asarray(v, dtype=np.float64), rowvar=False).reshape(v.shape[1], v.shape[1]))
        lam = (1.0 - ci) * lam + ci
        if lam.min() < eps:
            lam = lam + (eps - lam.min())
        out.append((V / np.sqrt(lam)) @ V.T)
    return out


def krprod_moment(Z):
    """M_(0) = Z_1^T KR(Z_2, ..., Z_m) / n (p_1 x prod_{i>1} p_i)."""
    n = Z[0].shape[0]
    kr = Z[1]
    for z in Z[2:]:
        kr = (kr[:, :, None] * z[:, None, :]).reshape(n, -1)
    return Z[0].T @ kr / n


def gram_start(M, k, rand):
    """The device start: eigenvectors of the unfolding Grams M_(j) M_(j)^T, descending, and sigma = sqrt(lambda)."""
    vecs, sigma0 = [], None
    for j, p in enumerate(M.shape):
        A = unfold(M, j)
        lam, U = np.linalg.eigh(A @ A.T)
        lam, U = lam[::-1], U[:, ::-1]
        vecs.append(U[:, :min(k, p)])
        if j == 0:
            sigma0 = np.sqrt(np.maximum(lam, 0.0))
    return new_state(M, assemble_start(M.shape, k, vecs, sigma0, rand))


def tensor_of(views, center=True, c=0.0, eps=1e-6):
    """(M as a p_1 x ... x p_m array, whiteners, means) by the device algorithm."""
    views = [np.asarray(v, dtype=np.float64) for v in views]
    means = [v.mean(axis=0) for v in views]
    S = whiteners(views, c, eps)
    Z = [(v - mu if center else v) @ s for v, mu, s in zip(views, means, S)]
    M = krprod_moment(Z).reshape([v.shape[1] for v in views])
    return M, S, means


def cov_tcca_fit(views, k, center=True, c=0.0, eps=1e-6, random_state=None):
    """The device algorithm in float64: (weights, means, final ALS state)."""
    M, S, means = tensor_of(views, center, c, eps)
    state = gram_start(M, k, random_columns(M.shape, k, rng_of(random_state)))
    for _ in range(N_ITER_MAX):
        als_step(state, M)
        if state["stop"]:
            break
    if state["singular"]:
        raise np.linalg.LinAlgError("Singular matrix")
    return [s @ f for s, f in zip(S, state["F"])], means, state
