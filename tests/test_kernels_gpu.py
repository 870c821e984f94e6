"""GPU parity tests of the individual kernels (through the C ABI) against float64 numpy/torch.

Tolerances are stated per test: exact / fp64 paths at round-off, TF32 at its 2^-11 input rounding,
3xTF32 at fp32 grade.
"""
import numpy as np
import pytest
import torch

pytestmark = pytest.mark.gpu


def _views(n, dims, dtype, seed=0, mean=0.0):
    g = torch.Generator().manual_seed(seed)
    z = torch.randn(n, 4, generator=g, dtype=torch.float64)
    out = []
    for d in dims:
        a = torch.randn(4, d, generator=g, dtype=torch.float64)
        out.append((z @ a + torch.randn(n, d, generator=g, dtype=torch.float64) + mean).to(dtype))
    return out


def _ref_cov(views, center=True):
    X = torch.cat([v.double() for v in views], dim=1).cpu().numpy()
    n = X.shape[0]
    if center:
        X = X - X.mean(axis=0)
    return X.T @ X / (n - 1)


@pytest.mark.parametrize("precision,dtype,rtol", [
    ("exact", torch.float64, 1e-12),
    ("exact", torch.float32, 2e-5),
    ("tf32x3", torch.float32, 2e-5),
    ("tf32x3b", torch.float32, 2e-5),     # 3xTF32 with the two cross terms as bf16 MMAs
    ("tf32", torch.float32, 3e-3),
])
@pytest.mark.parametrize("n,dims", [
    (200, [50, 50]),          # BASELINE config 1 shape
    (1000, [128, 128]),
    (777, [10, 8, 6]),        # ragged views, n not a multiple of the chunk
    (4096, [300, 130]),       # views straddling 128-blocks
    (33, [5, 7]),             # tiny
])
def test_moments_and_covariance(precision, dtype, rtol, n, dims):
    from cca_zoo_b200 import ops

    views = [v.cuda() for v in _views(n, dims, dtype, seed=n)]
    mom = ops.moments(views, precision=precision)
    Cm, mean = ops.covariance(mom, dims, n, center=True, dtype=torch.float64)
    ref = _ref_cov(views)
    scale = np.sqrt(np.outer(np.diag(ref), np.diag(ref)))
    err = np.abs(Cm.cpu().numpy() - ref) / scale
    assert err.max() < rtol, f"max normalised covariance error {err.max():.3e}"
    assert torch.equal(Cm, Cm.T), "covariance must be exactly symmetric"
    ref_mean = torch.cat([v.double() for v in views], dim=1).mean(dim=0)
    mtol = 1e-12 if dtype == torch.float64 else (3e-3 if precision == "tf32" else 1e-5)
    assert (mean.cpu() - ref_mean.cpu()).abs().max() < mtol * (1 + ref_mean.abs().max())


@pytest.mark.parametrize("precision", ["tf32x3b", "tf32x3"])
def test_inputs_longer_than_one_pass_keep_the_accumulator_run_bound(precision):
    """ADVICE r1 (low): the 2048-sample accumulator run of the 3xTF32 modes used to stretch once the split count hit its
    cap (n > 256 * 2048 rows), letting the round-toward-zero drift of TMEM back in.  Long inputs are now processed in
    equal passes whose float64 moments add up: the result IS the sum of the passes' moments (bitwise), and as accurate
    as a short input's."""
    from cca_zoo_b200 import ops

    n, dims = 1_200_000, [64, 64]          # cap = 256 splits x 2048 rows = 524288 rows per pass -> 3 passes
    cap = 256 * 2048
    npass = -(-n // cap)
    per = min(cap, -(-(-(-n // npass)) // 2048) * 2048)
    g = torch.Generator(device="cuda").manual_seed(5)
    views = [torch.randn(n, d, generator=g, device="cuda") + 0.25 for d in dims]
    mom = ops.moments(views, precision=precision)
    parts = None
    for r0 in range(0, n, per):
        m = ops.moments([v[r0:r0 + per] for v in views], precision=precision)
        parts = m if parts is None else parts + m
    assert torch.equal(mom, parts), "the passes must add up to the one-call result exactly"
    Dp = 256
    M = mom[:Dp * Dp].view(Dp, Dp)
    X = torch.cat(views, dim=1).double()
    ref_diag = (X * X).sum(dim=0)
    got = torch.cat([torch.diagonal(M)[:64], torch.diagonal(M)[128:192]])
    rel = ((got - ref_diag) / ref_diag).cpu().numpy()
    assert np.abs(rel).max() < 5e-5, f"diagonal of the raw moments off by {np.abs(rel).max():.2e}"
    s = mom[Dp * Dp:Dp * Dp + Dp]
    ref_s = X.sum(dim=0)
    got_s = torch.cat([s[:64], s[128:192]])
    assert ((got_s - ref_s).abs() / ref_s.abs()).max() < 1e-5
    Cm, _ = ops.covariance(mom, dims, n, center=True, dtype=torch.float64)
    Xc = X - X.mean(dim=0)
    ref = (Xc.T @ Xc / (n - 1)).cpu().numpy()
    scale = np.sqrt(np.outer(np.diag(ref), np.diag(ref)))
    assert (np.abs(Cm.cpu().numpy() - ref) / scale).max() < 5e-5


def test_moments_uncentred_and_nonzero_mean():
    from cca_zoo_b200 import ops

    views = [v.cuda() for v in _views(2000, [40, 24], torch.float64, seed=3, mean=5.0)]
    mom = ops.moments(views, precision="exact")
    C0, mean0 = ops.covariance(mom, [40, 24], 2000, center=False)
    X = torch.cat(views, dim=1).cpu().numpy()
    np.testing.assert_allclose(C0.cpu().numpy(), X.T @ X / 1999, rtol=1e-12)
    assert float(mean0.abs().max()) == 0.0
    C1, _ = ops.covariance(mom, [40, 24], 2000, center=True)
    np.testing.assert_allclose(C1.cpu().numpy(), _ref_cov(views), rtol=1e-9, atol=1e-9)


@pytest.mark.parametrize("precision", ["tf32x3b", "tf32x3", "exact"])
def test_badly_centred_columns_take_the_shifted_accumulation(precision):
    """Columns with |mean| = 1000 std: raw float32 moments would lose all digits of the covariance
    (eps * (mean / std)^2 ~ 1e-7 * 1e6); the pilot detects it and the shifted pass keeps float32-grade accuracy."""
    from cca_zoo_b200 import ops

    g = torch.Generator().manual_seed(3)
    n, dims = 6000, [96, 130]
    base = [torch.randn(n, d, generator=g, dtype=torch.float64) for d in dims]
    off = [torch.linspace(-1000.0, 1000.0, d, dtype=torch.float64) for d in dims]
    views64 = [b + o for b, o in zip(base, off)]
    views = [v.float().cuda() for v in views64]
    mom, x0 = ops.moments_safe(views, precision=precision)
    assert x0 is not None, "the pilot must ask for the shifted pass here"
    Cm, mean = ops.covariance(mom, dims, n, center=True, dtype=torch.float64)
    X = torch.cat([v.double().cpu() for v in views], dim=1)          # the float32 inputs, exactly
    ref = torch.cov(X.T)
    scale = torch.sqrt(torch.outer(ref.diagonal(), ref.diagonal()))
    assert float(((Cm.cpu() - ref).abs() / scale).max()) < 5e-5
    assert float((mean.cpu() - X.mean(dim=0)).abs().max()) < 1e-3
    raw = ops.moments(views, precision=precision)                     # for contrast: the unguarded one-pass form
    Cr, _ = ops.covariance(raw, dims, n, center=True, dtype=torch.float64)
    assert float(((Cr.cpu() - ref).abs() / scale).max()) > 1e-3
    centred = [v.float().cuda() for v in base]                        # well centred data: no extra pass
    _, x0c = ops.moments_safe(centred, precision=precision)
    assert x0c is None


def test_moments_are_additive_over_row_shards():
    """The multi-GPU contract: moments of row shards sum to the moments of the whole."""
    from cca_zoo_b200 import ops

    views = [v.cuda() for v in _views(3000, [96, 80], torch.float32, seed=5)]
    whole = ops.moments(views, precision="tf32x3")
    parts = ops.moments([v[:1700] for v in views], precision="tf32x3") + ops.moments(
        [v[1700:] for v in views], precision="tf32x3")
    Cw, _ = ops.covariance(whole, [96, 80], 3000)
    Cp, _ = ops.covariance(parts, [96, 80], 3000)
    assert (Cw - Cp).abs().max() < 1e-5 * Cw.abs().max()


@pytest.mark.parametrize("dtype,tol", [(torch.float64, 1e-11), (torch.float32, 2e-4)])
@pytest.mark.parametrize("ta,tb", [(False, False), (True, False), (False, True), (True, True)])
def test_gemm(dtype, tol, ta, tb):
    from cca_zoo_b200 import ops

    g = torch.Generator().manual_seed(1)
    m, n, k = 70, 130, 45
    A = torch.randn((k, m) if ta else (m, k), generator=g, dtype=torch.float64)
    B = torch.randn((n, k) if tb else (k, n), generator=g, dtype=torch.float64)
    ref = (A.T if ta else A) @ (B.T if tb else B)
    out = ops.gemm(A.to(dtype).cuda(), B.to(dtype).cuda(), transa=ta, transb=tb)
    assert (out.double().cpu() - ref).abs().max() < tol * ref.abs().max() * 10


@pytest.mark.parametrize("dtype,tol", [(torch.float64, 1e-12), (torch.float32, 5e-6)])
@pytest.mark.parametrize("n", [8, 32, 50, 64, 100, 256])
def test_syevj_psd(dtype, tol, n):
    """A v = lambda v, orthonormal rows, descending order (tests/test_linalg.py:122-141 of the reference)."""
    from cca_zoo_b200 import ops

    g = torch.Generator().manual_seed(n)
    X = torch.randn(3 * n, n, generator=g, dtype=torch.float64)
    A = (X.T @ X / (3 * n)).to(dtype)
    ev, Vt = ops.syevj(A.cuda())
    ev, Vt = ev.double().cpu(), Vt.double().cpu()
    A64 = A.double()
    ref = torch.linalg.eigvalsh(A64).flip(0)
    assert torch.all(ev[:-1] >= ev[1:])
    assert (ev - ref).abs().max() < tol * ref.abs().max() * 20
    assert (Vt @ Vt.T - torch.eye(n, dtype=torch.float64)).abs().max() < tol * 50
    resid = A64 @ Vt.T - Vt.T * ev
    assert resid.abs().max() < tol * ref.abs().max() * 50


def test_syevj_batched_and_indefinite_with_shift():
    from cca_zoo_b200 import ops

    g = torch.Generator().manual_seed(7)
    T = torch.randn(20, 12, generator=g, dtype=torch.float64) * 0.3
    K = torch.zeros(32, 32, dtype=torch.float64)          # Jordan-Wielandt: eigenvalues +-sigma
    K[:20, 20:] = T
    K[20:, :20] = T.T
    S = torch.randn(32, 32, generator=g, dtype=torch.float64)
    S = (S + S.T) / 2
    A = torch.stack([K, S]).cuda()
    shift = float(max(torch.linalg.matrix_norm(K), torch.linalg.matrix_norm(S)))
    ev, Vt = ops.syevj(A, shift=shift)
    for b, M in enumerate([K, S]):
        ref = torch.linalg.eigvalsh(M).flip(0)
        np.testing.assert_allclose(ev[b].cpu().numpy(), ref.numpy(), atol=1e-11)
        V = Vt[b].cpu()
        assert (M @ V.T - V.T * ev[b].cpu()).abs().max() < 1e-10
    sv = torch.linalg.svdvals(T)
    np.testing.assert_allclose(ev[0, :12].cpu().numpy(), sv.numpy(), atol=1e-11)


@pytest.mark.parametrize("dtype,tol", [(torch.float64, 1e-12), (torch.float32, 5e-6)])
@pytest.mark.parametrize("m,n", [(40, 24), (24, 40), (96, 96), (130, 70)])
def test_gesvj(dtype, tol, m, n):
    from cca_zoo_b200 import ops

    g = torch.Generator().manual_seed(m * n)
    G = torch.randn(m, n, generator=g, dtype=torch.float64)
    sig, Rt, Lt = ops.gesvj(G.T.contiguous().to(dtype).cuda())
    sig, Rt, Lt = sig.double().cpu(), Rt.double().cpu(), Lt.double().cpu()
    G = G.to(dtype).double()
    ref = torch.linalg.svdvals(G)
    r = min(m, n)
    assert (sig[:r] - ref).abs().max() < tol * ref.max() * 20
    if n > m:
        assert sig[m:].abs().max() < tol * ref.max() * 50
    recon = (Lt[:r].T * sig[:r]) @ Rt[:r]
    assert (recon - G).abs().max() < tol * ref.max() * 50
    assert (Rt @ Rt.T - torch.eye(n, dtype=torch.float64)).abs().max() < tol * 50


def test_whiten_rows_matches_definition():
    from cca_zoo_b200 import ops

    g = torch.Generator().manual_seed(2)
    X = torch.randn(200, 16, generator=g, dtype=torch.float64)
    Cm = (X.T @ X / 199).cuda()
    lam, Vt = ops.syevj(Cm)
    Wt, gv, rank = ops.whiten_rows(lam, Vt, c=0.2)
    W = Wt.T.cpu()
    reg = 0.8 * Cm.cpu() + 0.2 * torch.eye(16, dtype=torch.float64)
    assert (W.T @ reg @ W - torch.eye(16, dtype=torch.float64)).abs().max() < 1e-10
    assert int(rank.item()) == 16


def test_argument_errors_are_loud():
    from cca_zoo_b200 import ops

    with pytest.raises(RuntimeError, match="CUDA tensor"):
        ops.moments([torch.zeros(4, 4), torch.zeros(4, 4)])
    with pytest.raises(ValueError):
        ops.moments([torch.zeros(4, 4, device="cuda"), torch.zeros(5, 4, device="cuda")])
    with pytest.raises(ValueError):
        ops.gemm(torch.zeros(4, 5, device="cuda"), torch.zeros(4, 5, device="cuda"))


def test_topk_svd_matches_full_svd():
    from cca_zoo_b200 import _solvers

    g = torch.Generator().manual_seed(3)
    U, _ = torch.linalg.qr(torch.randn(300, 300, generator=g, dtype=torch.float64))
    V, _ = torch.linalg.qr(torch.randn(260, 260, generator=g, dtype=torch.float64))
    s = torch.cat([torch.linspace(0.9, 0.5, 20, dtype=torch.float64), 0.1 * torch.rand(240, generator=g, dtype=torch.float64)])
    T = (U[:, :260] * s) @ V.T
    sig, Ut, Vt = _solvers.topk_svd(T.cuda(), 20)
    np.testing.assert_allclose(sig.cpu().numpy(), s[:20].numpy(), rtol=1e-10)
    assert ((Ut.cpu() @ U[:, :20]).abs() - torch.eye(20, dtype=torch.float64)).abs().max() < 1e-8
    assert ((Vt.cpu() @ V[:, :20]).abs() - torch.eye(20, dtype=torch.float64)).abs().max() < 1e-8
    # slowly decaying spectrum: no gap to exploit -> reports failure, callers fall back to the full Jacobi SVD
    slow = (U[:, :260] * (1.0 - 1e-4 * torch.arange(260, dtype=torch.float64))) @ V.T
    assert _solvers.topk_svd(slow.cuda(), 20, max_rounds=1, iters_per_round=2) is None
