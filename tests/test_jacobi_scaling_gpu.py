"""Scale equivariance of the Jacobi eigensolvers and SVD (``ops.syevj``, ``ops.gesvj``, ``ops.syevj_small``).

Multiplying a matrix by 2^k is exact, and so is a solver that normalises its input by a power of two: the solve of
2^k A must be the solve of A bit for bit -- eigenvalues / singular values times 2^k, the same vectors, the same sweep
count.  Every case below checks

  (a) at k = 0, the result against float64 LAPACK on the host (the tolerances of test_kernels_gpu.py, and of
      test_shape_routes_gpu.py at the sizes of the unfused round and test_syevj_small_gpu.py for ``syevj_small``);
  (b) at every k of ``KS``, exact equivariance against the k = 0 solve;
  (c) where the solver takes a batch, that each member is scaled on its own: one call on 2^a A, A, 2^b A gives three
      results that agree bit for bit once unscaled.  (A batched call is never compared with a single call: the Gram
      partition and the cluster size of the Jacobi round depend on the batch, so those differ in rounding by design.)

The scales keep every input and every expected output in the normal range, null eigenvalues included, and reach
where the products of the convergence and rotation tests (degree 4 in the entries) under- or overflow without the
normalisation: float64 data at 1e-12 (MEG magnetometers in tesla) has a covariance near 1e-24, and a float32 matrix
with entries near 1e9 already overflows w_ii w_jj.  A solver that stops there reports convergence with V = I.
"""
import numpy as np
import pytest
import torch

from tests.test_shape_routes_gpu import _check_eigh, jacobi_cluster_size

pytestmark = pytest.mark.gpu

KS = {torch.float64: (-600, -160, -80, 0, 80, 600), torch.float32: (-70, -30, 0, 30, 70)}
TOL = {torch.float64: 1e-12, torch.float32: 5e-6}      # test_kernels_gpu.py: test_syevj_psd / test_gesvj
SMALL_TOL = {torch.float64: 1e-13, torch.float32: 3e-6}   # test_syevj_small_gpu.py
SMALL_MAX_N = {torch.float64: 104, torch.float32: 128}


def _pow2(x, k):
    """2^k x by ``torch.ldexp``, checked exact: every entry keeps its mantissa and moves its exponent by k."""
    y = torch.ldexp(x, torch.tensor(float(k), dtype=x.dtype, device=x.device))
    mx, ex = torch.frexp(x)
    my, ey = torch.frexp(y)
    nz = x != 0
    assert torch.equal(mx, my) and bool(((ey - ex)[nz] == k).all()), f"2^{k} x is not exact in {x.dtype}"
    return y


def _orth(n, g):
    Q, R = torch.linalg.qr(torch.randn(n, n, generator=g, dtype=torch.float64))
    return Q * torch.sign(torch.diagonal(R))


def _sym(lam, g):
    Q = _orth(lam.numel(), g)
    A = (Q * lam) @ Q.T
    return (A + A.T) / 2


def _assert_scaled(got, ref, k, what):
    """got == 2^k ref bit for bit (CPU tensors)."""
    assert bool(torch.isfinite(got).all()), f"{what}: non-finite output at 2^{k}"
    exp = _pow2(ref, k)
    if not torch.equal(got, exp):
        bad = (got != exp).nonzero()[0].tolist()
        raise AssertionError(f"{what}: not equivariant at 2^{k}: {int((got != exp).sum())} entries differ, first at "
                             f"{bad}: {got[tuple(bad)].item()!r} vs 2^{k} x {ref[tuple(bad)].item()!r}")


def _assert_same(got, ref, k, what):
    assert bool(torch.isfinite(got).all()), f"{what}: non-finite output at 2^{k}"
    assert torch.equal(got, ref), (f"{what}: differs at 2^{k} from the unscaled solve "
                                   f"(max |diff| {float((got.double() - ref.double()).abs().max()):.3e})")


def _anchor_eigh(A64, ev, Vt, dtype):
    """test_kernels_gpu.py::test_syevj_psd: eigenvalues, orthonormal rows, residual, descending order."""
    tol = TOL[dtype]
    n = A64.shape[-1]
    ev, Vt = ev.double(), Vt.double()
    ref = torch.linalg.eigvalsh(A64).flip(0)
    nrm = float(ref.abs().max())
    assert torch.all(ev[:-1] >= ev[1:])
    assert float((ev - ref).abs().max()) <= tol * nrm * 20
    assert float((Vt @ Vt.T - torch.eye(n, dtype=torch.float64)).abs().max()) <= tol * 50
    assert float((A64 @ Vt.T - Vt.T * ev).abs().max()) <= tol * nrm * 50


def _syevj_at(A, k, shift=0.0):
    """ops.syevj of 2^k A (shift scaled alike) -> (ev, Vt, sweeps) on the host; A on the host."""
    from cca_zoo_b200 import ops

    ev, Vt, info = ops.syevj(_pow2(A, k).cuda(), shift=shift * 2.0 ** k, return_info=True)
    assert info["converged"], f"syevj at 2^{k}: {info}"
    return ev.cpu(), Vt.cpu(), info["sweeps"]


def _syevj_equivariant(A, dtype, shift=0.0, what="syevj"):
    """(b) over KS[dtype]; returns the k = 0 solve."""
    ev0, Vt0, sw0 = _syevj_at(A, 0, shift)
    for k in KS[dtype]:
        if k == 0:
            continue
        ev, Vt, sw = _syevj_at(A, k, shift)
        _assert_scaled(ev, ev0, k, f"{what} eigenvalues")
        _assert_same(Vt, Vt0, k, f"{what} eigenvectors")
        assert sw == sw0, f"{what}: {sw} sweeps at 2^{k}, {sw0} unscaled"
    return ev0, Vt0


# --------------------------------------------------------------------------------------------------
# ops.syevj, symmetric mode
# --------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("dtype", [torch.float64, torch.float32])
@pytest.mark.parametrize("n", [50, 100])
def test_syevj_spd_is_scale_equivariant(dtype, n):
    g = torch.Generator().manual_seed(n)
    lo = -6 if dtype == torch.float64 else -3
    A = _sym(torch.logspace(0, lo, n, dtype=torch.float64), g).to(dtype)
    ev, Vt = _syevj_equivariant(A, dtype, what=f"{dtype} SPD n={n}")
    _anchor_eigh(A.double(), ev, Vt, dtype)


def test_syevj_rank_deficient_covariance_is_scale_equivariant():
    """300 x 300 float64 covariance of rank 150 from 900 samples: the columns of the null cluster only stop the sweep
    once their norms fall below the noise floor (n eps)^2 ||A||_F^2, which must follow the scale of A."""
    g = torch.Generator().manual_seed(300)
    X = torch.randn(900, 150, generator=g, dtype=torch.float64) @ torch.randn(150, 300, generator=g, dtype=torch.float64)
    X = X - X.mean(0)
    A = X.T @ X / 899
    A = (A + A.T) / 2
    ev, Vt = _syevj_equivariant(A, torch.float64, what="rank-150 covariance")
    _anchor_eigh(A, ev, Vt, torch.float64)


@pytest.mark.parametrize("dtype", [torch.float64, torch.float32])
def test_syevj_equal_eigenvalue_cluster_is_scale_equivariant(dtype):
    """An eigenvalue of multiplicity 8 in the middle of the spectrum: its vectors are any basis of the eigenspace, so
    the k = 0 solve is checked by its projector, the scaled solves by their bits."""
    g = torch.Generator().manual_seed(64)
    lam = torch.cat([torch.linspace(1.3, 1.0, 28, dtype=torch.float64), torch.full((8,), 0.7, dtype=torch.float64),
                     torch.linspace(0.4, 0.1, 28, dtype=torch.float64)])
    Q = _orth(64, g)
    A = (Q * lam) @ Q.T
    A = ((A + A.T) / 2).to(dtype)
    ev, Vt = _syevj_equivariant(A, dtype, what=f"{dtype} cluster")
    _anchor_eigh(A.double(), ev, Vt, dtype)
    tol = TOL[dtype]
    assert float((ev[28:36].double() - 0.7).abs().max()) <= tol * 1.3 * 20
    Vc = Vt[28:36].double()
    P, Pref = Vc.T @ Vc, Q[:, 28:36] @ Q[:, 28:36].T
    assert float((P - Pref).abs().max()) <= tol * 50, "eigenspace of the repeated eigenvalue"


def test_syevj_indefinite_with_shift_is_scale_equivariant():
    """The batch of test_kernels_gpu.py::test_syevj_batched_and_indefinite_with_shift (a Jordan-Wielandt matrix and a
    symmetric indefinite one), solved shifted to PSD with the shift scaled by 2^k as well."""
    g = torch.Generator().manual_seed(7)
    T = torch.randn(20, 12, generator=g, dtype=torch.float64) * 0.3
    K = torch.zeros(32, 32, dtype=torch.float64)
    K[:20, 20:] = T
    K[20:, :20] = T.T
    S = torch.randn(32, 32, generator=g, dtype=torch.float64)
    S = (S + S.T) / 2
    A = torch.stack([K, S])
    shift = float(max(torch.linalg.matrix_norm(K), torch.linalg.matrix_norm(S)))
    ev, Vt = _syevj_equivariant(A, torch.float64, shift=shift, what="shifted indefinite")
    for b, M in enumerate([K, S]):
        ref = torch.linalg.eigvalsh(M).flip(0)
        np.testing.assert_allclose(ev[b].numpy(), ref.numpy(), atol=1e-11)
        assert (M @ Vt[b].T - Vt[b].T * ev[b]).abs().max() < 1e-10
    np.testing.assert_allclose(ev[0, :12].numpy(), torch.linalg.svdvals(T).numpy(), atol=1e-11)


@pytest.mark.parametrize("dtype", [torch.float64, torch.float32])
def test_syevj_batch_members_are_scaled_each_on_its_own(dtype):
    """(c): one call on [2^lo A, A, 2^hi A, 0].  The zero member keeps the factor 1: eigenvalues 0, the identity."""
    from cca_zoo_b200 import ops

    n = 50
    g = torch.Generator().manual_seed(51)
    A = _sym(torch.logspace(0, -3, n, dtype=torch.float64), g).to(dtype)
    lo, hi = KS[dtype][0], KS[dtype][-1]
    batch = torch.stack([_pow2(A, lo), A, _pow2(A, hi), torch.zeros_like(A)])
    ev, Vt, info = ops.syevj(batch.cuda(), return_info=True)
    assert info["converged"], info
    ev, Vt = ev.cpu(), Vt.cpu()
    _anchor_eigh(A.double(), ev[1], Vt[1], dtype)
    _assert_scaled(ev[0], ev[1], lo, "member 2^lo A")
    _assert_scaled(ev[2], ev[1], hi, "member 2^hi A")
    _assert_same(Vt[0], Vt[1], lo, "member 2^lo A vectors")
    _assert_same(Vt[2], Vt[1], hi, "member 2^hi A vectors")
    assert bool((ev[3] == 0).all()), "zero member: eigenvalues"
    assert torch.equal(Vt[3], torch.eye(n, dtype=dtype)), "zero member: vectors"


@pytest.mark.parametrize("dtype,n", [(torch.float64, 1200), (torch.float32, 2700)])
def test_syevj_unfused_round_is_scale_equivariant(dtype, n):
    """The three-kernel round (gram / solve / apply) at the sizes test_shape_routes_gpu.py runs it: [A, A] and
    [2^lo A, 2^hi A] in one call each (same batch, same Gram partition, same route)."""
    from cca_zoo_b200 import ops

    assert jacobi_cluster_size(n, n, 2, dtype) == 0
    g = torch.Generator().manual_seed(n)
    A = _sym(0.01 + 0.99 * torch.rand(n, generator=g, dtype=torch.float64), g).to(dtype)
    lo, hi = KS[dtype][0], KS[dtype][-1]
    ev0, Vt0, info0 = ops.syevj(torch.stack([A, A]).cuda(), return_info=True)
    ev1, Vt1, info1 = ops.syevj(torch.stack([_pow2(A, lo), _pow2(A, hi)]).cuda(), return_info=True)
    assert info0["converged"] and info1["converged"], (info0, info1)
    assert info1["sweeps"] == info0["sweeps"], (info0, info1)
    ev0, Vt0, ev1, Vt1 = ev0.cpu(), Vt0.cpu(), ev1.cpu(), Vt1.cpu()
    _check_eigh(A.double(), ev0[0], Vt0[0], dtype, f"{dtype} n={n} unfused")
    for b, k in enumerate((lo, hi)):
        _assert_scaled(ev1[b], ev0[b], k, f"{dtype} n={n} unfused eigenvalues")
        _assert_same(Vt1[b], Vt0[b], k, f"{dtype} n={n} unfused eigenvectors")


# --------------------------------------------------------------------------------------------------
# ops.gesvj
# --------------------------------------------------------------------------------------------------
def _gesvj_at(G, k):
    from cca_zoo_b200 import ops

    sig, Rt, Lt, info = ops.gesvj(_pow2(G, k).T.contiguous().cuda(), return_info=True)
    assert info["converged"], f"gesvj at 2^{k}: {info}"
    return sig.cpu(), Rt.cpu(), Lt.cpu(), info["sweeps"]


def _gesvj_equivariant(G, dtype, ks, what):
    sig0, Rt0, Lt0, sw0 = _gesvj_at(G, 0)
    for k in ks:
        if k == 0:
            continue
        sig, Rt, Lt, sw = _gesvj_at(G, k)
        _assert_scaled(sig, sig0, k, f"{what} singular values")
        _assert_same(Rt, Rt0, k, f"{what} right vectors")
        _assert_same(Lt, Lt0, k, f"{what} left vectors")
        assert sw == sw0, f"{what}: {sw} sweeps at 2^{k}, {sw0} unscaled"
    return sig0.double(), Rt0.double(), Lt0.double()


def _anchor_svd(G64, sig, Rt, Lt, dtype, rank):
    """test_kernels_gpu.py::test_gesvj: singular values, the null ones, reconstruction, orthonormal right vectors."""
    tol = TOL[dtype]
    n = G64.shape[1]
    ref = torch.linalg.svdvals(G64)[:rank]
    assert torch.all(sig[:-1] >= sig[1:])
    assert float((sig[:rank] - ref).abs().max()) <= tol * float(ref.max()) * 20
    if rank < n:
        assert float(sig[rank:].abs().max()) <= tol * float(ref.max()) * 50
    recon = (Lt[:rank].T * sig[:rank]) @ Rt[:rank]
    assert float((recon - G64).abs().max()) <= tol * float(ref.max()) * 50
    assert float((Rt @ Rt.T - torch.eye(n, dtype=torch.float64)).abs().max()) <= tol * 50


@pytest.mark.parametrize("dtype", [torch.float64, torch.float32])
@pytest.mark.parametrize("m,n", [(40, 24), (24, 40), (96, 96), (130, 70)])
def test_gesvj_is_scale_equivariant(dtype, m, n):
    g = torch.Generator().manual_seed(m * n)
    G = torch.randn(m, n, generator=g, dtype=torch.float64).to(dtype)
    sig, Rt, Lt = _gesvj_equivariant(G, dtype, KS[dtype], f"{dtype} {m}x{n}")
    _anchor_svd(G.double(), sig, Rt, Lt, dtype, min(m, n))


@pytest.mark.parametrize("m,n,dtype", [(6000, 64, torch.float64), (12000, 64, torch.float32)])
def test_gesvj_tall_unfused_is_scale_equivariant(m, n, dtype):
    """The tall shapes of test_shape_routes_gpu.py (unfused round, ragged Gram partials) at the two extreme scales."""
    assert jacobi_cluster_size(m, n, 1, dtype) == 0
    g = torch.Generator().manual_seed(m)
    Q, _ = torch.linalg.qr(torch.randn(m, n, generator=g, dtype=torch.float64))
    G = ((Q * torch.linspace(1.0, 0.5, n, dtype=torch.float64)) @ _orth(n, g).T).to(dtype)
    ks = (KS[dtype][0], KS[dtype][-1])
    sig, Rt, Lt = _gesvj_equivariant(G, dtype, ks, f"{dtype} {m}x{n} unfused")
    _anchor_svd(G.double(), sig, Rt, Lt, dtype, n)


@pytest.mark.parametrize("dtype", [torch.float64, torch.float32])
def test_gesvj_rank_deficient_is_scale_equivariant(dtype):
    """200 x 60 of rank 30: half the columns of G V end at the noise floor, which must follow the scale of G."""
    g = torch.Generator().manual_seed(30)
    G = (torch.randn(200, 30, generator=g, dtype=torch.float64) @ torch.randn(30, 60, generator=g, dtype=torch.float64)
         / 30).to(dtype)
    sig, Rt, Lt = _gesvj_equivariant(G, dtype, KS[dtype], f"{dtype} rank 30")
    _anchor_svd(G.double(), sig, Rt, Lt, dtype, 30)


# --------------------------------------------------------------------------------------------------
# ops.syevj_small
# --------------------------------------------------------------------------------------------------
def _small_matrix(n, dtype, seed):
    g = torch.Generator().manual_seed(seed)
    X = torch.randn(n, n, generator=g, dtype=torch.float64)
    return ((X + X.T) / 2).to(dtype)


def _anchor_small(A64, lam, Vt, dtype):
    """test_syevj_small_gpu.py::test_syevj_small_matches_lapack."""
    tol = SMALL_TOL[dtype]
    n = A64.shape[-1]
    ref = torch.linalg.eigvalsh(A64).flip(-1)
    scale = float(ref.abs().max())
    lam, V = lam.double(), Vt.double()
    assert float((lam - ref).abs().max()) < tol * scale * max(1, n) ** 0.5
    assert float((V @ V.T - torch.eye(n, dtype=torch.float64)).abs().max()) < 20 * tol
    assert float((V @ A64 - lam.unsqueeze(-1) * V).abs().max()) < 30 * tol * scale


@pytest.mark.parametrize("dtype", [torch.float64, torch.float32])
@pytest.mark.parametrize("n", [7, 33, 96, "max"])
def test_syevj_small_is_scale_equivariant(dtype, n):
    from cca_zoo_b200 import ops

    n = SMALL_MAX_N[dtype] if n == "max" else n
    A = _small_matrix(n, dtype, 17 * n)
    lam0, Vt0, info0 = (t.cpu() for t in ops.syevj_small(A.cuda()))
    assert int(info0.min()) > 0, info0
    _anchor_small(A.double(), lam0, Vt0, dtype)
    for k in KS[dtype]:
        if k == 0:
            continue
        lam, Vt, info = (t.cpu() for t in ops.syevj_small(_pow2(A, k).cuda()))
        _assert_scaled(lam, lam0, k, f"syevj_small {dtype} n={n} eigenvalues")
        _assert_same(Vt, Vt0, k, f"syevj_small {dtype} n={n} eigenvectors")
        assert torch.equal(info, info0), f"syevj_small {dtype} n={n}: info {info.tolist()} at 2^{k}, {info0.tolist()}"


@pytest.mark.parametrize("dtype", [torch.float64, torch.float32])
def test_syevj_small_batch_members_are_scaled_each_on_its_own(dtype):
    """(c): one call on [2^lo A, 2^hi A]."""
    from cca_zoo_b200 import ops

    A = _small_matrix(33, dtype, 2)
    lo, hi = KS[dtype][0], KS[dtype][-1]
    lam, Vt, info = (t.cpu() for t in ops.syevj_small(torch.stack([_pow2(A, lo), _pow2(A, hi)]).cuda()))
    assert int(info.min()) > 0 and int(info[0]) == int(info[1]), info
    _anchor_small(A.double(), _pow2(lam[0], -lo), Vt[0], dtype)
    _assert_scaled(lam[1], _pow2(lam[0], -lo), hi, "syevj_small member 2^hi A")
    _assert_same(Vt[1], Vt[0], hi - lo, "syevj_small member 2^hi A vectors")


# --------------------------------------------------------------------------------------------------
# an estimator on data far from unit scale
# --------------------------------------------------------------------------------------------------
def test_rcca_eigen_route_follows_scaled_views():
    """rCCA(c=0) weights scale by exactly 1/s when the views are multiplied by s.  At s = 2^-40 (float64 data of
    standard deviation 1e-12, the size of MEG magnetometer data in tesla) the covariance blocks are near 1e-24."""
    from oracle import restatement as R

    from cca_zoo_b200.linear import rCCA

    rng = np.random.default_rng(40)
    z = rng.standard_normal((500, 3))
    views = [z @ rng.standard_normal((3, 20)) + rng.standard_normal((500, 20)),
             z @ rng.standard_normal((3, 30)) + rng.standard_normal((500, 30))]
    w0 = rCCA(latent_dimensions=3, c=0.0, solver="eigen").fit(views).weights_
    for k in (-40, 40):
        s = 2.0 ** k
        scaled = [v * s for v in views]
        ws = rCCA(latent_dimensions=3, c=0.0, solver="eigen").fit(scaled).weights_
        err = R.max_rel_err_per_vector([w * s for w in ws], w0)
        assert err < 1e-12, f"2^{k}: s w(s X) differs from w(X) by {err:.2e}"
        w_ref, _ = R.ref_rcca_fit(scaled, 3, 0.0)
        err = R.max_rel_err_per_vector(ws, w_ref)
        assert err < 1e-5, f"2^{k}: weights differ from the reference by {err:.2e}"
