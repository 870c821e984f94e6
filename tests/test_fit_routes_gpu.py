"""The one-call device fits (``ops.rcca_fit`` / ``ops.mcca_fit``, csrc/fit.cu) route by route, each compared with a
float64 CPU reference that solves the identical covariance matrix.

Inputs are built so that their sample covariance is a chosen C (``_samples``); the moment buffer comes from
``ops.moments(views, "exact")`` and the reference from ``ops.covariance`` of that same buffer, so the error measured
belongs to the fit alone.  For rCCA with c = 0 the exact answer is known as well: C12 = C11^1/2 U diag(rho) V^T C22^1/2
has canonical correlations rho and weights C11^-1/2 U, C22^-1/2 V.

Routes (each selected only by shape, dtype or argument) and how a test pins which one ran -- the library's launch
counter, as the per-iteration launch delta ``launches(iters + 1) - launches(iters)`` (``PINS``):
  * Gram iteration (T^T T formed once, d2 <= d1 and iters >= 2) vs two products per iteration (d2 > d1 or iters = 1);
  * CholQR through the single diagonal-block kernel (p <= NB: 64 in float64, 128 in float32) vs blocked potrf_inv;
  * ridge blocks as one batched Cholesky (equal widths) vs one per view (total launch count of the fit);
  * MCCA: CholQR after every second product, and always after the last one.

Error bounds.  The fit reports status 0 only when its residual r = ||T^T U - V diag(sigma)||_F (header word 2) is at
most resid_tol * sigma_1 * sqrt(k), resid_tol = max(200 eps, 1e-10) (``resid_tol_of`` in fit.cu); that is asserted.
The computed T (or whitened K) differs from the exact one by the rounding of the Cholesky factor, its inverse and two
products: about sqrt(d) u sqrt(kappa) ||T|| with u the unit roundoff of the solve dtype and kappa = max cond(R_i) (the
inverse factor carries sqrt(kappa); sums of d rounded terms grow like sqrt(d) u).  With
    e = r / sigma_1 + sqrt(d) u sqrt(kappa)                    (relative backward error of the singular triplets)
  * sigma_j (eigenvalue_j):        |sigma_j - sigma_j,ref| <= e sigma_1                         (Weyl)
  * each weight vector:            ||w - w_ref|| / ||w_ref|| <= sqrt(kappa) e sigma_1 / gap     (Davis-Kahan: angle
    e sigma_1 / gap in the whitened space; mapping back through L^-T multiplies a relative error by at most
    cond(L) = sqrt(kappa)); gap = the smallest distance between consecutive sigma_1 .. sigma_k+1 of the reference
  * W_i^T R_i W_i - I, W_1^T C12 W_2 - diag(sigma):  2 e  (a rotation of the singular vectors among themselves leaves
    both identities, so the angle above does not enter; each of the two factors carries e)
MCCA reads the same with K + shift I for T: sigma_1 becomes |lambda_1| + shift and the identity is V^T (B/m) V = I.
Each bound is multiplied by a constant ``K`` fitted once to the measured values, so that the largest measured value of
every bound lies between 0.1 and 1 of it (every case prints its fractions with ``-s``).  On an H100 the largest
fractions were, rCCA: sigma 0.23, weights 0.15, identities 0.13; MCCA: eigenvalues 0.21, weights 0.13, identity
0.14.
"""
import ctypes as C

import numpy as np
import pytest
import torch

from oracle import restatement as R

pytestmark = pytest.mark.gpu

f32, f64 = torch.float32, torch.float64
UNIT = {f32: 2.0 ** -24, f64: 2.0 ** -53}
PMAX = {f32: 128, f64: 104}                    # largest block width of the single-CTA Ritz solve (syevj_small.cu)
#: constants of the bounds below (module docstring), per fit: sigma / eigenvalues, weights, identities
K = {"rcca": {"sig": 1.0, "w": 0.5, "id": 1.0}, "mcca": {"sig": 1.0, "w": 0.25, "id": 0.5}}


def resid_tol(dtype):
    return max(200 * 2 * UNIT[dtype], 1e-10)


def _launches():
    from cca_zoo_b200 import _lib

    torch.cuda.synchronize()
    return int(_lib.load().ccab_launch_count())


# --------------------------------------------------------------------------------------------------
# inputs with a chosen sample covariance
# --------------------------------------------------------------------------------------------------
def _orth(n, m, rng):
    Q, Rr = np.linalg.qr(rng.standard_normal((n, m)))
    return Q * np.sign(np.diag(Rr))


def _spd(d, kappa, rng):
    """SPD matrix with eigenvalues geomspace(1, 1/kappa): (C, Q, lam)."""
    Q = _orth(d, d, rng)
    lam = np.geomspace(1.0, 1.0 / kappa, d) if d > 1 else np.ones(1)
    return (Q * lam) @ Q.T, Q, lam


def _samples(Cm, n, mu, rng):
    """n x D data whose sample covariance (ddof 1) is Cm and whose column means are mu:
    X = sqrt(n-1) Q Cm^1/2 + 1 mu^T with Q the column-orthonormal basis of a centred random matrix."""
    G = rng.standard_normal((n, Cm.shape[0]))
    G -= G.mean(axis=0)
    Q, _ = np.linalg.qr(G)
    lam, V = np.linalg.eigh((Cm + Cm.T) / 2)
    half = (V * np.sqrt(np.clip(lam, 0.0, None))) @ V.T
    return np.sqrt(n - 1.0) * Q @ half + mu


def _split(X, dims):
    off = np.concatenate([[0], np.cumsum(dims)]).astype(int)
    return [np.ascontiguousarray(X[:, off[i]:off[i + 1]]) for i in range(len(dims))]


def _rho(r, k, p):
    """Canonical correlations: k wanted ones down to 0.55, a gap of 0.05, the rest of the block down to 0.3 (CholQR
    stays well conditioned), and a tail beyond p three orders below (one product already converges)."""
    top = np.linspace(0.9, 0.55, k) if k > 1 else np.array([0.9])
    mid = np.linspace(0.5, 0.3, p - k) if p > k else np.zeros(0)
    tail = 3e-5 * np.linspace(1.0, 0.1, r - p) if r > p else np.zeros(0)
    return np.concatenate([top, mid, tail])


def rcca_problem(d1, d2, k, p, kappa=30.0, seed=0, rho=None, mu_scale=0.5):
    """(views, exact weights, rho) for c = 0 with condition number kappa in both views."""
    rng = np.random.default_rng(seed)
    rho = _rho(min(d1, d2), k, p) if rho is None else np.asarray(rho, dtype=np.float64)
    C11, Q1, l1 = _spd(d1, kappa, rng)
    C22, Q2, l2 = _spd(d2, kappa, rng)
    r = len(rho)
    U, V = (_orth(d1, r, rng), _orth(d2, r, rng)) if r else (np.zeros((d1, 0)), np.zeros((d2, 0)))
    h1, h2 = (Q1 * np.sqrt(l1)) @ Q1.T, (Q2 * np.sqrt(l2)) @ Q2.T
    C12 = h1 @ (U * rho) @ V.T @ h2
    Cm = np.block([[C11, C12], [C12.T, C22]])
    n = d1 + d2 + 300
    X = _samples(Cm, n, mu_scale * rng.standard_normal(d1 + d2), rng)
    W1 = (Q1 / np.sqrt(l1)) @ Q1.T @ U
    W2 = (Q2 / np.sqrt(l2)) @ Q2.T @ V
    return _split(X, [d1, d2]), [W1, W2], rho


def mcca_problem(dims, k, seed=0, extra=6):
    """Views from k + extra shared latent factors plus noise: the k wanted ones strong (between-view correlations
    about 0.95 .. 0.8, so the subspace iteration on K + shift I converges in 32 products), the extra ones weaker."""
    rng = np.random.default_rng(seed)
    s2 = np.concatenate([np.geomspace(20.0, 4.0, k), np.geomspace(2.0, 0.5, extra)])
    D = int(sum(dims))
    off = np.concatenate([[0], np.cumsum(dims)]).astype(int)
    A = np.zeros((k + extra, D))
    for i, d in enumerate(dims):
        a = rng.standard_normal((k + extra, d))
        A[:, off[i]:off[i + 1]] = a / np.linalg.norm(a, axis=1, keepdims=True) * np.sqrt(s2)[:, None]
    Cm = A.T @ A + np.diag(rng.uniform(0.5, 1.5, D))
    X = _samples(Cm, D + 300, 0.3 * rng.standard_normal(D), rng)
    return _split(X, dims)


# --------------------------------------------------------------------------------------------------
# running the fits
# --------------------------------------------------------------------------------------------------
def _moments(views):
    from cca_zoo_b200 import ops

    return ops.moments([torch.from_numpy(v).cuda() for v in views], "exact")


def _reference_cov(mom, dims, n, center):
    from cca_zoo_b200 import ops

    Cd, mean = ops.covariance(mom, dims, n, center=center, dtype=f64)
    return Cd.cpu().numpy(), mean.cpu().numpy()


def fit_rcca(mom, dims, n, c, k, p, iters, dtype, center=True, n_dev=None):
    """(header, mean, sigma, [W1, W2], launches of the call) as host copies."""
    from cca_zoo_b200 import ops

    l0 = _launches()
    block, offs = ops.rcca_fit(mom, dims, None if n_dev is not None else n, n_dev, center, c, k, p, iters, dtype)
    l1 = _launches()
    hdr, mean, sig, ws = ops.decode_fit_block(block.cpu(), offs, dims, k, dtype)
    return hdr.copy(), mean.copy(), sig.astype(np.float64), [w.astype(np.float64) for w in ws], l1 - l0


def fit_mcca(mom, dims, n, c, k, p, iters, dtype=f64, center=True, eps=1e-6):
    from cca_zoo_b200 import ops

    l0 = _launches()
    block, offs = ops.mcca_fit(mom, dims, n, None, center, c, eps, k, p, iters, dtype)
    l1 = _launches()
    hdr, mean, val, ws = ops.decode_fit_block(block.cpu(), offs, dims, k, dtype)
    return hdr.copy(), mean.copy(), val.astype(np.float64), [w.astype(np.float64) for w in ws], l1 - l0


def _ridge(Cm, dims, c):
    return [(1.0 - ci) * Cm[s, s] + ci * np.eye(d) for s, d, ci in zip(R.block_slices(dims), dims, c)]


def _report(what, **ratios):
    print(f"{what}: " + "  ".join(f"{k} {v:.3f}" for k, v in ratios.items()))
    for k, v in ratios.items():
        assert v <= 1.0, f"{what}: {k} = {v:.3f} of its bound"


def check_rcca(what, out, Cm, mean_ref, dims, c, k, dtype, n, center=True):
    """Every check that needs no route knowledge: status, header, mean, sigma and weights against the reference,
    and the identities of the solution."""
    hdr, mean, sig, ws, _ = out
    assert int(hdr[0]) == 0, f"{what}: status {int(hdr[0])}"
    assert hdr[1] == n and hdr[4] == 0 and hdr[5] > 0 and hdr[3] == sig[0], (what, hdr[:6])
    assert hdr[2] <= resid_tol(dtype) * sig[0] * np.sqrt(k), (what, hdr[2])
    if center:
        assert np.array_equal(mean, mean_ref), what
    else:
        assert not mean.any(), what
    cmax = max(c)
    assert np.all(np.diff(sig) <= 0) and sig[-1] >= 0 and sig[0] <= 1.0 / (1.0 - cmax), (what, sig)
    Rs = _ridge(Cm, dims, c)
    kappa = max(np.linalg.cond(Ri) for Ri in Rs)
    ref_w_all, ref_sv_all = R.cov_rcca_fit(Cm, dims, min(dims), c, n_samples=n)
    ref_w = [w[:, :k] for w in ref_w_all]
    ref_sv = ref_sv_all[:k]
    gap = float(np.min(-np.diff(np.append(ref_sv_all, 0.0)[:k + 1])))      # nearest neighbour of any of the k
    s1 = ref_sv[0]
    e = hdr[2] / s1 + np.sqrt(max(dims)) * UNIT[dtype] * np.sqrt(kappa)
    e_sig = float(np.abs(sig - ref_sv).max())
    e_w = R.max_rel_err_per_vector(ws, ref_w)
    s1_, s2_ = R.block_slices(dims)
    e_id = max(float(np.abs(w.T @ Ri @ w - np.eye(k)).max()) for w, Ri in zip(ws, Rs))
    e_x = float(np.abs(ws[0].T @ Cm[s1_, s2_] @ ws[1] - np.diag(sig)).max())
    Kr = K["rcca"]
    _report(what, sigma=e_sig / (Kr["sig"] * e * s1), weights=e_w / (Kr["w"] * np.sqrt(kappa) * e * s1 / gap),
            ident=max(e_id, e_x) / (Kr["id"] * 2 * e))
    return ref_w, ref_sv


def check_mcca(what, out, Cm, mean_ref, dims, c, k, n, center=True, converged=True):
    """As check_rcca.  ``converged=False`` (too few products for the tolerance): the status must be exactly 2 and the
    checks that hold for any orthonormal block stay -- the Ritz values lie below the eigenvalues (interlacing) and
    V^T (B/m) V = I."""
    hdr, mean, val, ws, _ = out
    m = len(dims)
    shift = 0.5 / (1.0 - max(c))
    assert int(hdr[0]) == (0 if converged else 2), f"{what}: status {int(hdr[0])}"
    assert hdr[1] == n and hdr[4] == 0 and hdr[5] > 0 and hdr[3] == abs(val[0]) + shift, (what, hdr[:6])
    assert (hdr[2] <= resid_tol(f64) * hdr[3] * np.sqrt(k)) == converged, (what, hdr[2])
    if center:
        assert np.array_equal(mean, mean_ref), what
    else:
        assert not mean.any(), what
    assert np.all(np.diff(val) <= 0), (what, val)
    Bs = _ridge(Cm, dims, c)
    kappa = max(np.linalg.cond(Bi) if Bi.shape[0] > 1 else 1.0 for Bi in Bs)
    D = int(sum(dims))
    ref_w_all, lam_all = R.cov_mcca_fit(Cm, dims, D, c)
    ref_w = [w[:, :k] for w in ref_w_all]
    lam = lam_all[:k]
    gap = float(np.min(-np.diff(lam_all[:k + 1])))
    l1 = abs(lam[0]) + shift                   # the iterated matrix is K + shift I
    e = hdr[2] / l1 + np.sqrt(D) * UNIT[f64] * np.sqrt(kappa)
    V = np.vstack(ws)
    Bm = np.zeros((D, D))
    for s, Bi in zip(R.block_slices(dims), Bs):
        Bm[s, s] = Bi
    e_id = float(np.abs(V.T @ (Bm / m) @ V - np.eye(k)).max())
    if not converged:
        e = np.sqrt(D) * UNIT[f64] * np.sqrt(kappa)
        assert np.all(val <= lam + e * l1), (what, val, lam)
        _report(what, ident=e_id / (K["mcca"]["id"] * 2 * e))
        return ref_w, lam
    e_val = float(np.abs(val - lam).max())
    e_w = R.max_rel_err_per_vector([V], [np.vstack(ref_w)])     # one generalised eigenvector across all views
    Km = K["mcca"]
    _report(what, eigval=e_val / (Km["sig"] * e * l1), weights=e_w / (Km["w"] * np.sqrt(kappa) * e * l1 / gap),
            ident=e_id / (Km["id"] * 2 * e))
    return ref_w, lam


# --------------------------------------------------------------------------------------------------
# route pins: per-iteration launch deltas and whole-call launch counts measured on an H100
# --------------------------------------------------------------------------------------------------
PINS = {
    "rcca-256x256-p24-float64-total-it6": 59,
    "rcca-256x256-p24-float64-gram-per-iter": 4,
    "rcca-256x256-p24-float32-total-it6": 51,
    "rcca-256x256-p24-float32-gram-per-iter": 4,
    "rcca-300x260-p24-float64-total-it6": 84,
    "rcca-300x260-p24-float64-gram-per-iter": 4,
    "rcca-300x260-p24-float32-total-it6": 68,
    "rcca-300x260-p24-float32-gram-per-iter": 4,
    "rcca-64x64-p20-float64-total-it6": 46,
    "rcca-64x64-p20-float64-gram-per-iter": 4,
    "rcca-65x65-p20-float64-total-it6": 51,
    "rcca-65x65-p20-float64-gram-per-iter": 4,
    "rcca-128x128-p20-float32-total-it6": 46,
    "rcca-128x128-p20-float32-gram-per-iter": 4,
    "rcca-129x129-p20-float32-total-it6": 51,
    "rcca-129x129-p20-float32-gram-per-iter": 4,
    "rcca-300x260-p24-float64-total-it2": 68,
    "rcca-260x300-p24-float64-total-it2": 69,
    "rcca-260x300-p24-float64-two-per-iter": 5,
    "rcca-260x300-p24-float64-total-it6": 89,
    "rcca-400x360-p64-float64-total-it6": 97,
    "rcca-400x360-p64-float64-gram-per-iter": 4,
    "rcca-400x360-p65-float64-total-it6": 139,
    "rcca-400x360-p65-float64-gram-per-iter": 10,
    "rcca-400x360-p80-float64-total-it6": 139,
    "rcca-400x360-p80-float64-gram-per-iter": 10,
    "rcca-400x360-p104-float64-total-it6": 139,
    "rcca-400x360-p104-float64-gram-per-iter": 10,
    "rcca-400x360-p128-float32-total-it6": 73,
    "rcca-400x360-p128-float32-gram-per-iter": 4,
    "rcca-300x260-p17-float64-total-it6": 84,
    "rcca-300x260-p17-float64-gram-per-iter": 4,
    "rcca-300x260-p17-float32-total-it6": 68,
    "rcca-300x260-p17-float32-gram-per-iter": 4,
    "rcca-40x33-p33-float32-total-it6": 48,
    "rcca-40x33-p33-float32-gram-per-iter": 4,
    "rcca-1024x1024-p80-float64-total-it6": 159,
    "rcca-1024x1024-p80-float64-gram-per-iter": 12,
    "rcca-1024x1024-p80-float32-total-it6": 91,
    "rcca-1024x1024-p80-float32-gram-per-iter": 6,
    "mcca-2views-equal-total": 113,
    "mcca-2views-unequal-total": 120,
    "mcca-3views-equal-total": 113,
    "mcca-3views-w1-w65-total": 122,
    "mcca-8views-equal-total": 163,
    "mcca-iters1-total": 56,
    "mcca-iters2-total": 57,
    "mcca-iters3-total": 61,
    "mcca-c0.9-total": 202,
    "mcca-p80-blocked-total": 283,
    "mcca-pmax-total": 283,
    "rcca-300x260-p24-float64-total-it1": 64,
    "rcca-40x33-p33-float64-total-it6": 48,
    "rcca-40x33-p33-float64-gram-per-iter": 4,
    "mcca-2views-equal-per-iter": 1,
    "mcca-2views-unequal-per-iter": 1,
    "mcca-3views-equal-per-iter": 1,
    "mcca-3views-w1-w65-per-iter": 1,
    "mcca-8views-equal-per-iter": 1,
    "mcca-8views-unequal-total": 182,
    "mcca-8views-unequal-per-iter": 1,
    "mcca-iters2-per-iter": 1,
    "mcca-iters3-per-iter": 4,
    "mcca-c0.9-per-iter": 1,
    "mcca-p80-blocked-per-iter": 2,
    "mcca-pmax-per-iter": 2,
    "mcca-steps-4-7": (4, 1, 4),
}


def _pin(key, got):
    print(f"pin {key}: {got}")
    if key in PINS:
        assert got == PINS[key], (key, got, PINS[key])


def _iter_delta(mom, dims, n, c, k, p, iters, dtype):
    a = fit_rcca(mom, dims, n, c, k, p, iters, dtype)[4]
    b = fit_rcca(mom, dims, n, c, k, p, iters + 1, dtype)[4]
    return b - a


# --------------------------------------------------------------------------------------------------
# rCCA routes
# --------------------------------------------------------------------------------------------------
RCCA_CASES = [
    # id, d1, d2, k, p, iters, dtype
    ("ridge-batched", 256, 256, 8, 24, 6, f64),
    ("ridge-batched", 256, 256, 8, 24, 6, f32),
    ("ridge-perview", 300, 260, 8, 24, 6, f64),
    ("ridge-perview", 300, 260, 8, 24, 6, f32),
    ("potrf-1block", 64, 64, 4, 20, 6, f64),
    ("potrf-2blocks", 65, 65, 4, 20, 6, f64),
    ("potrf-1block", 128, 128, 4, 20, 6, f32),
    ("potrf-2blocks", 129, 129, 4, 20, 6, f32),
    ("gram", 300, 260, 8, 24, 2, f64),
    ("gram", 300, 260, 8, 24, 6, f64),
    ("two-product", 260, 300, 8, 24, 2, f64),
    ("two-product", 260, 300, 8, 24, 6, f64),
    ("two-product-iters1", 300, 260, 8, 24, 1, f64),
    ("cholqr-p64", 400, 360, 48, 64, 6, f64),
    ("cholqr-p65", 400, 360, 49, 65, 6, f64),
    ("cholqr-p80", 400, 360, 64, 80, 6, f64),
    ("cholqr-pmax", 400, 360, 88, 104, 6, f64),
    ("cholqr-pmax", 400, 360, 112, 128, 6, f32),
    ("k1", 300, 260, 1, 17, 6, f64),
    ("k1", 300, 260, 1, 17, 6, f32),
    ("k=p=min", 40, 33, 33, 33, 6, f64),
    ("k=p=min", 40, 33, 33, 33, 6, f32),
    ("bench", 1024, 1024, 64, 80, 6, f64),
    ("bench", 1024, 1024, 64, 80, 6, f32),
]


@pytest.mark.parametrize("name,d1,d2,k,p,iters,dtype", RCCA_CASES,
                         ids=[f"{c[0]}-{c[1]}x{c[2]}-k{c[3]}-p{c[4]}-it{c[5]}-{str(c[6])[6:]}" for c in RCCA_CASES])
def test_rcca_fit_route_matches_reference(name, d1, d2, k, p, iters, dtype):
    dims, c = [d1, d2], [0.0, 0.0]
    # one product (iters = 1) converges exactly when the cross-covariance has rank p
    views, w_exact, rho = rcca_problem(d1, d2, k, p, seed=d1 + 7 * d2 + k, rho=_rho(p, k, p) if iters == 1 else None)
    n = views[0].shape[0]
    mom = _moments(views)
    Cm, mean_ref = _reference_cov(mom, dims, n, True)
    out = fit_rcca(mom, dims, n, c, k, p, iters, dtype)
    what = f"rcca {name} {d1}x{d2} k={k} p={p} iters={iters} {dtype}"
    ref_w, ref_sv = check_rcca(what, out, Cm, mean_ref, dims, c, k, dtype, n)
    # the construction: the reference solves the chosen problem (rounding of the float64 samples only)
    assert np.abs(ref_sv - rho[:k]).max() < 1e-9 and R.max_rel_err_per_vector(ref_w, [w[:, :k] for w in w_exact]) < 1e-7
    gram = d2 <= d1 and iters >= 2
    _pin(f"rcca-{d1}x{d2}-p{p}-{str(dtype)[6:]}-total-it{iters}", out[4])
    if iters >= 2:
        _pin(f"rcca-{d1}x{d2}-p{p}-{str(dtype)[6:]}-{'gram' if gram else 'two'}-per-iter",
             _iter_delta(mom, dims, n, c, k, p, iters, dtype))


@pytest.mark.parametrize("dtype", [f64, f32])
def test_rcca_fit_ridge_and_uncentred(dtype):
    """c != 0 against the reference, and center = False: the column sums in the buffer are not used (the reference
    solves the uncentred second moments) and the mean block is zero."""
    dims, k = [300, 260], 6
    views, _, _ = rcca_problem(*dims, k, 22, seed=5, mu_scale=2.0)
    n = views[0].shape[0]
    mom = _moments(views)
    for c, center, p in (([0.3, 0.05], True, 22), ([0.0, 0.0], False, 23), ([0.2, 0.2], False, 23)):   # the means
        # add one direction to the uncentred spectrum: p = 23 keeps the block clear of the 3e-5 tail
        Cm, mean_ref = _reference_cov(mom, dims, n, center)
        out = fit_rcca(mom, dims, n, c, k, p, 12, dtype, center=center)
        check_rcca(f"rcca c={c} center={center} {dtype}", out, Cm, mean_ref, dims, c, k, dtype, n, center=center)


def test_rcca_fit_reads_the_sample_count_from_the_device():
    """n_host = 0 with n on the device (the sharded fit's all-reduced count) computes the same bits as n_host."""
    dims, k, p = [300, 260], 8, 24
    views, _, _ = rcca_problem(*dims, k, p, seed=9)
    n = views[0].shape[0]
    mom = _moments(views)
    for dtype in (f64, f32):
        a = fit_rcca(mom, dims, n, [0.1, 0.0], k, p, 6, dtype)
        b = fit_rcca(mom, dims, n, [0.1, 0.0], k, p, 6, dtype, n_dev=torch.tensor([float(n)], dtype=f64, device="cuda"))
        assert np.array_equal(a[0][:6], b[0][:6]) and np.array_equal(a[1], b[1]) and np.array_equal(a[2], b[2])
        assert all(np.array_equal(x, y) for x, y in zip(a[3], b[3])) and int(a[0][0]) == 0


# --------------------------------------------------------------------------------------------------
# MCCA routes
# --------------------------------------------------------------------------------------------------
MCCA_CASES = [
    # id, dims, k, p, iters, c
    ("2views-equal", [160, 160], 4, 36, 32, [0.0, 0.0]),
    ("2views-unequal", [160, 120], 4, 36, 32, [0.1, 0.0]),
    ("3views-equal", [100, 100, 100], 5, 37, 32, [0.0, 0.0, 0.0]),
    ("3views-w1-w65", [65, 1, 100], 4, 36, 32, [0.0, 0.0, 0.1]),
    ("8views-equal", [40] * 8, 6, 38, 32, [0.05] * 8),
    ("8views-unequal", [65, 1, 30, 50, 20, 10, 40, 64], 6, 38, 32, [0.0] * 8),
    ("iters1", [150, 120, 100], 5, 37, 1, [0.0] * 3),
    ("iters2", [150, 120, 100], 5, 37, 2, [0.0] * 3),
    ("iters3", [150, 120, 100], 5, 37, 3, [0.0] * 3),
    ("c0.9", [150, 120, 100], 5, 37, 60, [0.9, 0.5, 0.0]),
    ("p80-blocked", [200, 200, 200], 40, 80, 32, [0.0] * 3),
    ("pmax", [200, 200, 200], 52, 104, 32, [0.0] * 3),
]


@pytest.mark.parametrize("name,dims,k,p,iters,c", MCCA_CASES, ids=[c[0] for c in MCCA_CASES])
def test_mcca_fit_route_matches_reference(name, dims, k, p, iters, c):
    views = mcca_problem(dims, k, seed=len(dims) * 13 + k)
    n = views[0].shape[0]
    mom = _moments(views)
    Cm, mean_ref = _reference_cov(mom, dims, n, True)
    out = fit_mcca(mom, dims, n, c, k, p, iters)
    check_mcca(f"mcca {name} dims={dims} k={k} p={p} iters={iters} c={c}", out, Cm, mean_ref, dims, c, k, n,
               converged=iters >= 32)
    _pin(f"mcca-{name}-total", out[4])
    if iters >= 2:
        _pin(f"mcca-{name}-per-iter", out[4] - fit_mcca(mom, dims, n, c, k, p, iters - 1)[4])


def test_mcca_fit_uncentred_and_cholqr_schedule():
    """center = 0: the mean block is zero and the buffer's column sums are not used.  The CholQR schedule (after
    every second product and after the last one) shows as launches per iteration alternating with the parity."""
    dims, k, p = [150, 120, 100], 5, 37
    views = mcca_problem(dims, k, seed=3)
    n = views[0].shape[0]
    mom = _moments(views)
    Cm, _ = _reference_cov(mom, dims, n, False)
    check_mcca("mcca center=False", fit_mcca(mom, dims, n, [0.0] * 3, k, p, 32, center=False), Cm, None, dims,
               [0.0] * 3, k, n, center=False)
    counts = [fit_mcca(mom, dims, n, [0.0] * 3, k, p, it)[4] for it in (4, 5, 6, 7)]
    steps = np.diff(counts)
    print(f"mcca launches at iters 4..7: {counts}, steps {list(steps)}")
    _pin("mcca-steps-4-7", tuple(int(s) for s in steps))


# --------------------------------------------------------------------------------------------------
# status word from real inputs
# --------------------------------------------------------------------------------------------------
def _status(out):
    return int(out[0][0])


@pytest.mark.parametrize("dims", [[256, 256], [300, 260]], ids=["batched", "per-view"])
@pytest.mark.parametrize("bad", [0, 1])
def test_rcca_fit_singular_view_sets_bit_1_and_names_the_view(dims, bad):
    views, _, _ = rcca_problem(*dims, 6, 22, seed=1)
    views[bad][:, 7] = views[bad][:, 3]           # exactly singular covariance block, c = 0
    n = views[0].shape[0]
    out = fit_rcca(_moments(views), dims, n, [0.0, 0.0], 6, 22, 6, f64)
    assert _status(out) & 1 and out[0][4] == bad + 1, out[0][:6]


@pytest.mark.parametrize("dims", [[80, 80, 80], [80, 60, 70]], ids=["batched", "per-view"])
@pytest.mark.parametrize("bad", [0, 1, 2])
def test_mcca_fit_singular_view_sets_bit_1_and_names_the_view(dims, bad):
    views = mcca_problem(dims, 4, seed=2)
    views[bad][:, 5] = views[bad][:, 2]
    n = views[0].shape[0]
    out = fit_mcca(_moments(views), dims, n, [0.0] * 3, 4, 36, 32)
    assert _status(out) & 1 and out[0][4] == bad + 1, out[0][:6]


def test_mcca_fit_eps_floor_decides_at_lambda_min():
    """lambda_min(B_1) just below the reference's eps: the fit declines (bit 1, the host route applies the floor);
    just above: status 0 and the reference's answer (its floor is inactive)."""
    dims, k, p, eps = [80, 60, 70], 4, 36, 1e-6
    views = mcca_problem(dims, k, seed=4)
    Cm = np.cov(np.hstack(views), rowvar=False)
    for lam_min, want in ((0.9 * eps, 1), (1.2 * eps, 0)):
        C2 = Cm.copy()
        C2[79, :] = 0.0
        C2[:, 79] = 0.0
        C2[79, 79] = lam_min                       # its own eigenvalue and the last pivot of B_1
        rng = np.random.default_rng(8)
        X = _samples(C2, views[0].shape[0], np.zeros(sum(dims)), rng)
        vs = _split(X, dims)
        n = vs[0].shape[0]
        mom = _moments(vs)
        Cd, mean_ref = _reference_cov(mom, dims, n, True)
        assert abs(np.linalg.eigvalsh(Cd[:80, :80]).min() - lam_min) < 1e-3 * eps
        out = fit_mcca(mom, dims, n, [0.0] * 3, k, p, 32, eps=eps)
        if want:
            assert _status(out) & 1 and out[0][4] == 1, out[0][:6]
        else:
            check_mcca("mcca lambda_min just above eps", out, Cd, mean_ref, dims, [0.0] * 3, k, n)


def test_rcca_fit_not_converged_bit_2():
    dims = [300, 260]
    views, _, _ = rcca_problem(*dims, 8, 24, seed=6, rho=np.linspace(0.6, 0.59, 260))     # no gap anywhere
    n = views[0].shape[0]
    out = fit_rcca(_moments(views), dims, n, [0.0, 0.0], 8, 24, 1, f64)
    assert _status(out) == 2, out[0][:6]
    views, _, _ = rcca_problem(*dims, 8, 24, seed=6, rho=np.zeros(0))                      # C12 = 0
    out = fit_rcca(_moments(views), dims, n, [0.0, 0.0], 8, 24, 6, f64)
    assert _status(out) & 2 and np.isfinite(out[0][:6]).all(), out[0][:6]


def test_fit_non_finite_input_bit_4():
    views, _, _ = rcca_problem(300, 260, 6, 22, seed=7)
    views[1][11, 4] = np.nan
    n = views[0].shape[0]
    mom = _moments(views)
    assert _status(fit_rcca(mom, [300, 260], n, [0.1, 0.1], 6, 22, 6, f64)) & 4
    assert _status(fit_rcca(mom, [300, 260], n, [0.1, 0.1], 6, 22, 6, f32)) & 4


def test_fit_too_few_samples_bit_8():
    """n_total <= max d_i sets bit 8 (the blocks are rank deficient by construction); max d_i + 1 does not."""
    dims = [120, 90]
    rng = np.random.default_rng(12)
    for n, want in ((120, 8), (121, 0)):
        vs = [rng.standard_normal((n, d)) for d in dims]
        out = fit_rcca(_moments(vs), dims, n, [0.1, 0.1], 4, 20, 6, f64)
        assert (_status(out) & 8) == want, (n, out[0][:6])
        mout = fit_mcca(_moments(vs), dims, n, [0.1, 0.1], 4, 36, 32)
        assert (_status(mout) & 8) == want, (n, mout[0][:6])
    mom = _moments([rng.standard_normal((500, d)) for d in dims])
    assert _status(fit_rcca(mom, dims, 1, [0.1, 0.1], 4, 20, 6, f64)) & 8
    assert _status(fit_mcca(mom, dims, 1, [0.1, 0.1], 4, 36, 32)) & 8


@pytest.mark.parametrize("dtype", [f64, f32])
def test_rcca_fit_low_rank_cross_covariance_never_returns_wrong_weights(dtype):
    """C12 of exact rank r = 12 < p = 24 with k = 8 <= r: the block iterate loses rank.  Either the status word says
    so or the weights are right -- never status 0 with wrong weights."""
    dims, k, p = [300, 260], 8, 24
    rho = np.linspace(0.9, 0.4, 12)
    views, _, _ = rcca_problem(*dims, k, p, seed=10, rho=rho)
    n = views[0].shape[0]
    mom = _moments(views)
    Cm, mean_ref = _reference_cov(mom, dims, n, True)
    out = fit_rcca(mom, dims, n, [0.0, 0.0], k, p, 6, dtype)
    if _status(out):
        print(f"rank-12 cross covariance, {dtype}: status {_status(out)}")
    else:
        print(f"rank-12 cross covariance, {dtype}: status 0, weights checked")
        check_rcca(f"rcca rank 12 {dtype}", out, Cm, mean_ref, dims, [0.0, 0.0], k, dtype, n)


# --------------------------------------------------------------------------------------------------
# determinism and reads of uninitialised memory, through the C ABI
# --------------------------------------------------------------------------------------------------
def _abi_fit(kind, dims, mom, n, c, k, p, iters, dtype, fill, ws_extra=0, misalign=0):
    """The fit through ctypes with the workspace and result block pre-filled with ``fill``; returns
    (rc, block bytes, offsets)."""
    from cca_zoo_b200 import _lib

    lib = _lib.load()
    dt = _lib.F32 if dtype == f32 else _lib.F64
    d = _lib.i64_array(dims)
    m = len(dims)
    if kind == "rcca":
        offs = (C.c_int64 * 5)()
        assert lib.ccab_rcca_fit_result_layout(dt, d, k, p, offs) == 0
        wsb = lib.ccab_rcca_fit_workspace_bytes(dt, d, k, p)
    else:
        offs = (C.c_int64 * (m + 3))()
        assert lib.ccab_mcca_fit_result_layout(dt, m, d, k, p, offs) == 0
        wsb = lib.ccab_mcca_fit_workspace_bytes(dt, m, d, k, p)
    assert wsb > 0
    total = offs[len(offs) - 1]
    raw = torch.full((total + 512,), fill, dtype=torch.uint8, device="cuda")
    start = (-raw.data_ptr()) % 256 + misalign
    block = raw[start:start + total]
    ws = torch.full((wsb + ws_extra,), fill, dtype=torch.uint8, device="cuda")    # the fit aligns inside it itself
    cc = (C.c_double * m)(*c)
    stream = C.c_void_p(torch.cuda.current_stream().cuda_stream)
    if kind == "rcca":
        rc = lib.ccab_rcca_fit(dt, d, mom.data_ptr(), None, float(n), 1, cc, k, p, iters, block.data_ptr(), total,
                               ws.data_ptr(), ws.numel(), stream)
    else:
        rc = lib.ccab_mcca_fit(dt, m, d, mom.data_ptr(), None, float(n), 1, cc, 1e-6, k, p, iters, block.data_ptr(),
                               total, ws.data_ptr(), ws.numel(), stream)
    torch.cuda.synchronize()
    return rc, block.cpu().numpy(), [int(x) for x in offs]


def _written(buf, offs, dims, k, dtype):
    """The bytes the fit writes: header words 0-5, the mean, sigma / eigenvalues, the weights (not the gaps)."""
    item = 4 if dtype == f32 else 8
    parts = [buf[:48], buf[offs[0]:offs[0] + 8 * sum(dims)], buf[offs[1]:offs[1] + item * k]]
    parts += [buf[offs[2 + i]:offs[2 + i] + item * d * k] for i, d in enumerate(dims)]
    return np.concatenate(parts)


@pytest.mark.parametrize("kind,dims,k,p,dtype", [
    ("rcca", [300, 260], 8, 24, f32), ("rcca", [300, 260], 8, 24, f64), ("rcca", [400, 360], 64, 80, f64),
    ("rcca", [256, 256], 8, 24, f32), ("mcca", [65, 1, 100], 4, 36, f64), ("mcca", [200, 200, 200], 40, 80, f64)])
def test_fit_is_bitwise_independent_of_buffer_contents(kind, dims, k, p, dtype):
    if kind == "rcca":
        views, _, _ = rcca_problem(*dims, k, p, seed=21)
        c, iters = [0.1, 0.0], 6
    else:
        views = mcca_problem(dims, k, seed=21)
        c, iters = [0.0] * len(dims), 32
    n = views[0].shape[0]
    mom = _moments(views)
    got = []
    for fill in (0xFF, 0x00, 0xFF):
        rc, buf, offs = _abi_fit(kind, dims, mom, n, c, k, p, iters, dtype, fill)
        assert rc == 0
        got.append(_written(buf, offs, dims, k, dtype))
    assert int(got[0][:8].view(np.float64)[0]) == 0
    assert np.array_equal(got[0], got[1]) and np.array_equal(got[0], got[2])


# --------------------------------------------------------------------------------------------------
# refusals
# --------------------------------------------------------------------------------------------------
def test_fits_refuse_bad_arguments_with_a_message():
    from cca_zoo_b200 import _lib, ops

    rng = np.random.default_rng(0)
    dims = [300, 300]
    vs = [rng.standard_normal((700, d)) for d in dims]
    mom, n = _moments(vs), 700
    bad_r = [(9, 8, 6, f64), (4, 301, 6, f64), (4, PMAX[f64] + 1, 6, f64), (4, PMAX[f32] + 1, 6, f32),
             (4, 20, 0, f64), (4, 20, 65, f64)]
    for k, p, iters, dt in bad_r:
        with pytest.raises(ValueError, match=r"ccab_rcca_fit(_result_layout)? failed \(code -\d+\): .+"):
            ops.rcca_fit(mom, dims, n, None, True, [0.1, 0.1], k, p, iters, dt)
    for k, p, iters, dt in [(4, PMAX[f64], 6, f64), (4, PMAX[f32], 6, f32)]:       # the limits themselves are taken
        ops.rcca_fit(mom, dims, n, None, True, [0.1, 0.1], k, p, iters, dt)
    mdims = [40, 30, 50]
    mmom = _moments([rng.standard_normal((700, d)) for d in mdims])
    bad_m = [(9, 8, 6, [0.0] * 3), (4, 121, 6, [0.0] * 3), (4, PMAX[f64] + 1, 6, [0.0] * 3), (4, 36, 0, [0.0] * 3),
             (4, 36, 61, [0.0] * 3), (4, 36, 32, [0.0, 0.91, 0.0])]
    for k, p, iters, c in bad_m:
        with pytest.raises(ValueError, match=r"ccab_mcca_fit(_result_layout)? failed \(code -\d+\): .+"):
            ops.mcca_fit(mmom, mdims, n, None, True, c, 1e-6, k, p, iters, f64)
    ops.mcca_fit(mmom, mdims, n, None, True, [0.9, 0.0, 0.0], 1e-6, 4, PMAX[f64], 60, f64)
    with pytest.raises(ValueError, match=r"ccab_mcca_fit failed \(code -\d+\): .+"):
        ops.mcca_fit(_moments([vs[0]]), [300], n, None, True, [0.0], 1e-6, 4, 36, 32, f64)
    # a workspace one byte short, a result block off the 256-byte grid
    for kind, dd, mm, c, k, p, iters in (("rcca", dims, mom, [0.1, 0.1], 4, 20, 6),
                                         ("mcca", mdims, mmom, [0.0] * 3, 4, 36, 32)):
        for dt in (f32, f64):
            rc, _, _ = _abi_fit(kind, dd, mm, n, c, k, p, iters, dt, 0, ws_extra=-1)
            assert rc < 0 and "workspace too small" in _lib.last_error()
            rc, _, _ = _abi_fit(kind, dd, mm, n, c, k, p, iters, dt, 0, misalign=8)
            assert rc < 0 and "256-byte aligned" in _lib.last_error()


# --------------------------------------------------------------------------------------------------
# estimators at the float64 Ritz limit: the plans decline what the library refuses
# --------------------------------------------------------------------------------------------------
def _latent_views(n, dims, r, seed):
    rng = np.random.default_rng(seed)
    z = rng.standard_normal((n, r)) * np.geomspace(3.0, 0.3, r)
    return [z @ rng.standard_normal((r, d)) / np.sqrt(d) + rng.standard_normal((n, d)) for d in dims]


def test_mcca_k60_and_float64_rcca_k90_fit_and_match_the_oracle():
    from cca_zoo_b200.linear import MCCA, rCCA

    views = _latent_views(6000, [512] * 4, 64, seed=1)
    est = MCCA(latent_dimensions=60).fit(views)
    print(f"MCCA k=60 on 4 x 512: route {getattr(est, '_fit_info', 'host (declined by the plan)')}")
    w_ref, mu_ref = R.ref_mcca_fit(views, 60)
    assert R.max_rel_err_per_vector(est.weights_, w_ref) < 1e-6
    np.testing.assert_allclose(np.concatenate(est.means_), np.concatenate(mu_ref), rtol=1e-12, atol=1e-12)
    views = _latent_views(5000, [400, 400], 96, seed=2)
    est = rCCA(latent_dimensions=90, c=0.1).fit(views)
    print(f"float64 rCCA k=90 on 400 + 400: route {getattr(est, '_fit_info', 'host (declined by the plan)')}")
    w_ref, mu_ref = R.ref_rcca_fit(views, 90, 0.1)
    assert R.max_rel_err_per_vector(est.weights_, w_ref) < 1e-6
