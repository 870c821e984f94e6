"""The batched Cholesky-inverse ``potrf_inv`` (csrc/cholinv.cu, through ``ops.potrf_inv_``) at every size, pivot
position, stride and scale where its route changes, against CPU references (float64 for the float32 kernel, long
double for the float64 kernel).

Routes, with NB the diagonal block width (128 for float32, 64 for float64):

* ``chol_diag_inv_kernel`` factors and inverts each NB-wide diagonal block in 32-wide sub-blocks; the last block is
  padded with the identity;
* the panel ``P = A_panel Dinv^T`` runs on 3xTF32 tensor cores (float32, lda % 4 == 0), on FMA tiles through scratch
  (float32 otherwise) or on DMMA (float64); the trailing update ``A22 -= P P^T`` writes whole lower tiles, so the strict
  upper triangle of A is not preserved and only ``tril(A)`` is checked;
* Linv is assembled by recursive doubling over block pairs; a ragged last pair whose B block is narrower than 8
  columns runs its second product on the FMA kernel in float64 (n = NB + 3 and 2 NB + 5).

Accuracy is checked against bounds that hold whatever the conditioning (see ``_check_factor``), failures through
``info``, and bitwise only what the arithmetic makes exact: separate matrices of a batch, equal routes over different
strides, and powers-of-four scaling (float64 by IEEE homogeneity; float32 as the H100's reciprocal square root
behaves).
"""
import numpy as np
import pytest
import scipy.linalg.lapack as lapack
import torch

gpu = pytest.mark.gpu

NB = {torch.float32: 128, torch.float64: 64}
NP = {torch.float32: np.float32, torch.float64: np.float64}
COND = {torch.float32: 1e3, torch.float64: 1e8}
# unit of the error model: 2^-53 for float64; 2^-21 for float32, where the 3xTF32 split operands lose about 2^-21
# per product (the FMA route and the Newton-refined reciprocal square root are within it)
U = {torch.float32: 2.0 ** -21, torch.float64: 2.0 ** -53}
DTYPES = [torch.float32, torch.float64]


def _sizes(nb):
    return [1, 2, 31, 32, 33, nb - 1, nb, nb + 1, nb + 3, 2 * nb - 1, 2 * nb, 2 * nb + 1, 2 * nb + 5, 3 * nb,
            4 * nb - 1, 4 * nb + 1, 8 * nb + 3]


# --------------------------------------------------------------------------------------------------
# fixtures (checked on the CPU by test_fixtures_cpu)
# --------------------------------------------------------------------------------------------------
def graded(n, cond, seed):
    """Q diag(lam) Q^T with lam geometric from 1 down to 1 / cond, Q Haar-random; float64."""
    g = np.random.default_rng(seed)
    Q, R = np.linalg.qr(g.standard_normal((n, n)))
    Q = Q * np.sign(np.diag(R))
    lam = cond ** (-np.arange(n) / max(n - 1, 1))
    A = (Q * lam) @ Q.T
    return (A + A.T) / 2


def planted(n, j, seed):
    """A = L0 L0^T with A[j, j] lowered by L0[j, j]^2 + 1: every pivot before j is L0[k, k]^2 = 4 and the pivot at j
    is exactly -1 in exact arithmetic, far from zero in any rounding; float64."""
    g = np.random.default_rng(seed)
    L0 = np.tril(g.standard_normal((n, n)) * 0.5 / np.sqrt(n), -1) + 2.0 * np.eye(n)
    A = L0 @ L0.T
    A[j, j] -= L0[j, j] ** 2 + 1.0
    return A


def decoupled(n, j, p, seed):
    """A well-conditioned SPD matrix whose row and column j are zero but for A[j, j] = p: every L[j, k] is an exact
    zero, so the pivot at j is exactly p in any arithmetic."""
    A = graded(n, 10.0, seed)
    A[j, :] = 0.0
    A[:, j] = 0.0
    A[j, j] = p
    return A


def _potrf_info(A):
    f = lapack.spotrf if A.dtype == np.float32 else lapack.dpotrf
    return f(A, lower=1)[1]


def test_fixtures_cpu():
    """No GPU: the planted matrices make LAPACK's Cholesky fail at exactly column j, in float32 and float64, and the
    graded matrices have the intended condition numbers."""
    for dt in DTYPES:
        nb = NB[dt]
        n = 2 * nb + 1
        for j in (0, 31, 32, nb - 1, nb, nb + 31, n - 1):
            A = planted(n, j, j).astype(NP[dt])
            assert _potrf_info(A) == j + 1, (dt, j)
        assert _potrf_info(planted(n, 5, 0).astype(NP[dt])[:5, :5]) == 0
        for n in (2, 33, nb + 3, 2 * nb + 5):
            A = graded(n, COND[dt], n)
            lam = np.linalg.eigvalsh(A)
            assert abs(lam.max() / lam.min() / COND[dt] - 1) < 1e-3, (dt, n)
            assert _potrf_info(A.astype(NP[dt])) == 0
    tol = 2.0 ** -10
    A = decoupled(80, 40, tol * (1 + 2.0 ** -20), 0)
    assert np.all(A[40, :40] == 0) and np.all(A[41:, 40] == 0) and A[40, 40] > tol


# --------------------------------------------------------------------------------------------------
# bounds
# --------------------------------------------------------------------------------------------------
def _blocks(n, nb):
    return [(j0, min(j0 + nb, n)) for j0 in range(0, n, nb)]


def _check_factor(A, L, Linv, dtype, what):
    """The two bounds, with M_1 = |L| |L^T|, K = |Linv| |L| and u the unit above:

    backward error   |A - L L^T|   <= (4n + 8) u (M_1 + |L| G^T),   G = blockdiag_j(|L_jj| |X_jj| |L_jj|)
    inverse residual |Linv L - I|  <= (4n + 8) u (K + K K)

    Derivation (first order in u).  A right-looking Cholesky whose block columns are formed by substitution meets
    Higham's componentwise bound gamma_{n+1} M_1 (Accuracy and Stability of Numerical Algorithms, Thm 10.3).  Here the
    panel is instead the product P = A_p X_jj^T with the explicit inverse X_jj of the diagonal block, and
    A_p - P L_jj^T = -A_p (L_jj X_jj - I)^T - E L_jj^T with |E| <= gamma_nb |A_p| |X_jj^T|: since |A_p| <= |P| |L_jj^T|,
    both terms are bounded by gamma |P| (|L_jj| |X_jj| |L_jj|)^T, which is the |L| G^T term.  Linv's off-diagonal
    blocks come from X_BA = -X_BB (L_BA X_AA), whose residual X_BB L_BA (X_AA L_AA - I) + X_BB E_1 L_AA + E_2 L_AA
    carries the product |X_BB| |L_BA| |X_AA| |L_AA|: the extra |Linv| |L| factor of K K.  (n + 1) roundings per
    entry, doubled for the two sources in each bound, give 4n; 8u covers the diagonal L_kk = piv * rsqrt(piv)
    (reciprocal square root, product, square).  Only tril(A) is compared: the trailing update rewrites the strict
    upper triangle of the diagonal tiles."""
    n = A.shape[0]
    nb = NB[dtype]
    hp = np.longdouble if dtype == torch.float64 else np.float64
    u = U[dtype]
    gam = (4 * n + 8) * u
    Lh, Xh = L.astype(hp), Linv.astype(hp)
    aL, aX = np.abs(L).astype(np.float64), np.abs(Linv).astype(np.float64)
    R = np.abs(A.astype(hp) - Lh @ Lh.T).astype(np.float64)
    M1 = aL @ aL.T
    LG = np.zeros_like(M1)
    for j0, j1 in _blocks(n, nb):
        Gj = aL[j0:j1, j0:j1] @ aX[j0:j1, j0:j1] @ aL[j0:j1, j0:j1]
        LG[:, j0:j1] = aL[:, j0:j1] @ Gj.T
    bound = gam * (M1 + LG)
    low = np.tril(np.ones((n, n), dtype=bool))
    E = np.abs(Xh @ Lh - np.eye(n, dtype=hp)).astype(np.float64)
    K = aX @ aL
    with np.errstate(invalid="ignore"):      # 0 / 0 above the diagonal of the (lower triangular) residual
        r_bw = float((R / bound)[low].max())
        r_inv = float((E / (gam * (K + K @ K)))[low].max())
        plain_bw = float((R / (n * u * M1))[low].max())
        plain_inv = float((E / (n * u * K))[low].max())
    print(f"{what}: |A - LL^T| / bound = {r_bw:.2e} (/ n u |L||L^T| = {plain_bw:.2e}), "
          f"|Linv L - I| / bound = {r_inv:.2e} (/ n u |Linv||L| = {plain_inv:.2e})")
    assert r_bw <= 1.0, f"{what}: backward error {r_bw:.3f} of its bound"
    assert r_inv <= 1.0, f"{what}: inverse residual {r_inv:.3f} of its bound"
    assert np.all(np.triu(Linv, 1) == 0), f"{what}: Linv is not exactly zero above its diagonal"


# --------------------------------------------------------------------------------------------------
# accuracy at every route-changing size
# --------------------------------------------------------------------------------------------------
@gpu
@pytest.mark.parametrize("dtype,n", [(dt, n) for dt in DTYPES for n in _sizes(NB[dt])])
def test_potrf_inv_accuracy_at_every_block_edge(dtype, n):
    """Graded spectra at condition 1e8 (float64) / 1e3 (float32), batch 1 and batch 3 (the first matrix of the batch
    is the batch-1 matrix)."""
    from cca_zoo_b200 import ops

    mats = [graded(n, COND[dtype], 1000 * n + s).astype(NP[dtype]) for s in range(3)]
    one = torch.from_numpy(mats[0]).cuda()
    Linv1, info1 = ops.potrf_inv_(one)
    three = torch.from_numpy(np.stack(mats)).cuda()
    Linv3, info3 = ops.potrf_inv_(three)
    assert int(info1.item()) == 0 and info3.cpu().tolist() == [0, 0, 0]
    _check_factor(mats[0], np.tril(one.cpu().numpy()), Linv1.cpu().numpy(), dtype, f"{dtype} n={n} batch 1")
    for b in range(3):
        _check_factor(mats[b], np.tril(three[b].cpu().numpy()), Linv3[b].cpu().numpy(), dtype,
                      f"{dtype} n={n} batch 3 [{b}]")


# --------------------------------------------------------------------------------------------------
# info: failing pivots at every block edge, a NaN, and pivot_tol
# --------------------------------------------------------------------------------------------------
@gpu
@pytest.mark.parametrize("dtype", DTYPES)
@pytest.mark.parametrize("where", ["first", "sub-block end", "sub-block start", "block end", "block start",
                                   "inside block 2", "padded last block"])
def test_potrf_inv_info_in_the_middle_of_a_batch(dtype, where):
    """n = 2 NB + 1, so column n - 1 is alone in the padded last block.  The failing matrix sits between two good
    ones: info is [0, j + 1, 0], and the good factors and inverses are bit-identical to batch-of-one calls (each
    kernel treats the matrices of a batch separately with the same arithmetic)."""
    from cca_zoo_b200 import ops

    nb = NB[dtype]
    n = 2 * nb + 1
    j = {"first": 0, "sub-block end": 31, "sub-block start": 32, "block end": nb - 1, "block start": nb,
         "inside block 2": nb + 31, "padded last block": n - 1}[where]
    mats = [graded(n, 100.0, 7).astype(NP[dtype]), planted(n, j, j).astype(NP[dtype]),
            graded(n, 100.0, 8).astype(NP[dtype])]
    Ab = torch.from_numpy(np.stack(mats)).cuda()
    Linv, info = ops.potrf_inv_(Ab)
    assert info.cpu().tolist() == [0, j + 1, 0]
    for b in (0, 2):
        A1 = torch.from_numpy(mats[b]).cuda()
        Linv1, info1 = ops.potrf_inv_(A1)
        assert int(info1.item()) == 0
        assert torch.equal(Ab[b], A1) and torch.equal(Linv[b], Linv1), f"matrix {b} changed by its neighbour"


@gpu
@pytest.mark.parametrize("dtype", DTYPES)
def test_potrf_inv_nan_entry(dtype):
    """A NaN at A[j, i], i < j (lower triangle), reaches the pivot at j first: info = j + 1."""
    from cca_zoo_b200 import ops

    nb = NB[dtype]
    n = 2 * nb + 5
    for j, i in ((1, 0), (33, 2), (nb, nb - 1), (nb + 40, 3), (n - 1, nb + 1), (2 * nb + 2, 2 * nb)):
        A = graded(n, 100.0, j).astype(NP[dtype])
        A[j, i] = np.nan
        _, info = ops.potrf_inv_(torch.from_numpy(A).cuda())
        assert int(info.item()) == j + 1, (j, i)


@gpu
@pytest.mark.parametrize("dtype", DTYPES)
@pytest.mark.parametrize("j", [0, 45, "block 2"])
def test_potrf_inv_pivot_tol_is_strict(dtype, j):
    """The pivot at j is exactly p (``decoupled``).  With pivot_tol = 2^-10: p = tol (1 + 2^-20) passes, p = tol and
    p = tol (1 - 2^-20) fail (the test is pivot > tol)."""
    from cca_zoo_b200 import ops

    nb = NB[dtype]
    n = 2 * nb + 3
    j = nb + 17 if j == "block 2" else j
    tol = 2.0 ** -10
    for p, want in ((tol * (1 + 2.0 ** -20), 0), (tol, j + 1), (tol * (1 - 2.0 ** -20), j + 1)):
        A = decoupled(n, j, p, j).astype(NP[dtype])
        assert float(A[j, j]) == p
        _, info = ops.potrf_inv_(torch.from_numpy(A).cuda(), pivot_tol=tol)
        assert int(info.item()) == want, (p / tol - 1, int(info.item()))


# --------------------------------------------------------------------------------------------------
# strides
# --------------------------------------------------------------------------------------------------
@gpu
@pytest.mark.parametrize("dtype", DTYPES)
@pytest.mark.parametrize("pad", [12, 13])
def test_potrf_inv_2d_view(dtype, pad):
    """A view at (3, 4) of an (n + 8) x (n + pad) matrix.  pad = 12: lda % 4 == 0, the float32 panel runs on the
    tensor cores, as for a contiguous matrix, and the result equals the contiguous call bit for bit.  pad = 13: the
    float32 panel and trailing update run on FMA tiles (the panel through scratch), so the bits differ from the
    contiguous call's.  float64 takes DMMA either way and matches bit for bit.  Nothing outside the view may
    change."""
    from cca_zoo_b200 import ops

    nb = NB[dtype]
    n = 2 * nb + 44                 # a multiple of 4, so the contiguous call is TMA-addressable too
    A = graded(n, COND[dtype], 12).astype(NP[dtype])
    parent = torch.from_numpy(np.random.default_rng(1).standard_normal((n + 8, n + pad)).astype(NP[dtype])).cuda()
    parent[3:3 + n, 4:4 + n] = torch.from_numpy(A).cuda()
    before = parent.clone()
    view = parent[3:3 + n, 4:4 + n]
    assert (view.stride(0) % 4 == 0) == (pad == 12)
    Linv, info = ops.potrf_inv_(view)
    assert int(info.item()) == 0
    mask = torch.ones_like(parent, dtype=torch.bool)
    mask[3:3 + n, 4:4 + n] = False
    assert torch.equal(parent[mask], before[mask]), "potrf_inv wrote outside its view"
    _check_factor(A, np.tril(view.cpu().numpy()), Linv.cpu().numpy(), dtype, f"{dtype} view pad={pad}")
    ref = torch.from_numpy(A).cuda()
    Linv_ref, _ = ops.potrf_inv_(ref)
    same = torch.equal(torch.tril(view), torch.tril(ref)) and torch.equal(Linv, Linv_ref)
    assert same == (pad == 12 or dtype == torch.float64), "the view did not take the expected panel route"


@gpu
@pytest.mark.parametrize("dtype", DTYPES)
def test_potrf_inv_batch_stride_not_n_lda(dtype):
    """Three matrices with row stride lda = n + 4 and batch stride n * lda + 36 (a multiple of 4, so the float32 panel
    keeps the tensor cores), in a buffer filled with sentinels: bit-identical to a contiguous batch of the same
    three, and the gaps between the matrices untouched."""
    from cca_zoo_b200 import ops

    nb = NB[dtype]
    n = 2 * nb + 8
    lda, bstride = n + 4, n * (n + 4) + 36
    mats = np.stack([graded(n, COND[dtype], 30 + b) for b in range(3)]).astype(NP[dtype])
    buf = torch.full((3 * bstride + 40,), 7.25, dtype=dtype, device="cuda")
    view = torch.as_strided(buf, (3, n, n), (bstride, lda, 1), 20)
    view.copy_(torch.from_numpy(mats).cuda())
    mask = torch.ones_like(buf, dtype=torch.bool)
    torch.as_strided(mask, (3, n, n), (bstride, lda, 1), 20).fill_(False)
    Linv, info = ops.potrf_inv_(view)
    assert info.cpu().tolist() == [0, 0, 0]
    assert bool((buf[mask] == 7.25).all()), "potrf_inv wrote outside its matrices"
    ref = torch.from_numpy(mats).cuda()
    Linv_ref, _ = ops.potrf_inv_(ref)
    assert torch.equal(torch.tril(view), torch.tril(ref)) and torch.equal(Linv, Linv_ref)
    _check_factor(mats[1], np.tril(view[1].cpu().numpy()), Linv[1].cpu().numpy(), dtype, f"{dtype} batch stride")


# --------------------------------------------------------------------------------------------------
# scale
# --------------------------------------------------------------------------------------------------
@gpu
def test_potrf_inv_float64_is_exactly_homogeneous():
    """L(4^k A) = 2^k L(A) and Linv(4^k A) = 2^-k Linv(A) bit for bit, k = -240 ... 240: every step is homogeneous
    under powers of four (IEEE sqrt and division, FMA chains, DMMA) while nothing leaves the normal range.
    n = 2 NB + 5 includes the FMA product of the ragged doubling pair."""
    from cca_zoo_b200 import ops

    n = 2 * NB[torch.float64] + 5
    A = graded(n, 1e6, 240)
    A0 = torch.from_numpy(A).cuda()
    Linv0, _ = ops.potrf_inv_(A0)
    L0 = torch.tril(A0)
    _check_factor(A, L0.cpu().numpy(), Linv0.cpu().numpy(), torch.float64, "float64 n=133 k=0")
    for k in range(-240, 241, 40):
        Ak = torch.from_numpy(np.ldexp(A, 2 * k)).cuda()
        Linv, info = ops.potrf_inv_(Ak)
        assert int(info.item()) == 0
        assert torch.equal(torch.tril(Ak), L0 * 2.0 ** k), f"L at k={k}"
        assert torch.equal(Linv, Linv0 * 2.0 ** -k), f"Linv at k={k}"


@gpu
def test_potrf_inv_float32_over_scales():
    """float32, k = -30 ... 30: both bounds at every scale of 4^k A, and L(4^k A) = 2^k L(A), Linv(4^k A) =
    2^-k Linv(A) bit for bit.  The reciprocal square root goes through the hardware approximation (MUFU.RSQ) plus one
    Newton step, which no standard makes homogeneous; on an H100 it is exactly homogeneous under powers of four, and
    this test pins that."""
    from cca_zoo_b200 import ops

    n = 2 * NB[torch.float32] + 44
    A = graded(n, COND[torch.float32], 30)
    for k in range(-30, 31, 10):
        Ak = np.ldexp(A, 2 * k).astype(np.float32)
        Ad = torch.from_numpy(Ak).cuda()
        Linv, info = ops.potrf_inv_(Ad)
        assert int(info.item()) == 0
        _check_factor(Ak, np.tril(Ad.cpu().numpy()), Linv.cpu().numpy(), torch.float32, f"float32 k={k}")
        if k == -30:
            L0, X0 = torch.tril(Ad), Linv
        else:
            s = 2.0 ** (k + 30)
            assert torch.equal(torch.tril(Ad), L0 * s) and torch.equal(Linv, X0 / s), f"k={k}: not 2^k L(A) exactly"
