"""Kernel routes that only the shape, dtype and batch of the input select, each checked against a float64 CPU
reference at the shapes that select it.

* Jacobi (``ops.syevj`` / ``ops.gesvj``): the fused round at cluster sizes 1, 2, 4 and 8 and the unfused
  three-kernel round (gram / solve / apply), float32 and float64.
* ``CCALoss`` on the fused small-width kernels (widths <= 64) and the first widths past them.
* ``ops.gemm`` dispatch: float32 3xTF32 tensor cores vs FMA tiles, float64 DMMA vs FMA tiles.

Every test also pins the route it was written for, so that a planner change cannot move it elsewhere unnoticed:
Jacobi and ``CCALoss`` by the library's launch counter, the Jacobi cluster size by a copy of the host planner (checked
on the CPU), the float32 GEMM routes bitwise (the tensor route against ``gemm_tc``, the FMA route against an exact
emulation of its fma chain).
"""
import numpy as np
import pytest
import torch

U = {torch.float32: 2.0 ** -24, torch.float64: 2.0 ** -53}     # unit roundoff


def _launches():
    from cca_zoo_b200 import _lib

    torch.cuda.synchronize()
    return int(_lib.load().ccab_launch_count())


# --------------------------------------------------------------------------------------------------
# Jacobi planner: a copy of the cluster-size loop of jacobi_solve (cca_zoo_b200/csrc/syevj.cu, "fused cluster path")
# and of fused_smem_bytes.  Keep the two in step.
# --------------------------------------------------------------------------------------------------
_KS, _KSP = 32, 33


def _cdiv(a, b):
    return -(-a // b)


def jacobi_cluster_size(m, n, batch, dtype):
    """Cluster size of the fused Jacobi round for an m x n problem (m == n for syevj), 0 = unfused round."""
    es = 4 if dtype == torch.float32 else 8
    n_pad = _cdiv(n, _KS) * _KS
    npairs = n_pad // _KS
    cs = 0
    for cand in (1, 2, 4, 8):
        rows = _cdiv(m, cand) + _cdiv(n_pad, cand)
        nbytes = (_KS * (rows | 1) + _KS * _KS + 3 * _KS * _KSP) * es + (_KS - 1) * (_KS // 2) * 2 + _KS * 4 + 64
        limit = 100 * 1024 if npairs * batch * cand >= 296 else 200 * 1024
        if nbytes <= limit:
            cs = cand
            if npairs * batch * cand >= 148 or cand == 8:
                break
    return cs


def jacobi_gram_partials(m, n, batch):
    """Row partials of the unfused round's Gram kernel (make_plan in syevj.cu): (count, rows per partial)."""
    npairs = _cdiv(n, _KS)
    R = min(16, max(1, min(_cdiv(m, 128), _cdiv(4 * 148, npairs * batch))))
    rows = _cdiv(_cdiv(m, R), 64) * 64
    return _cdiv(m, rows), rows


def jacobi_launches(n, sweeps, converged, cs):
    """Launches of one syevj / gesvj call: init + scale, the rounds of every sweep, a flag reset after every sweep but
    a converged last one, then values + rank + gather."""
    n_pad = _cdiv(n, _KS) * _KS
    rounds = n_pad // 16 - 1
    f = 1 if cs else 3
    return 5 + sweeps * rounds * f + (sweeps - 1 if converged else sweeps)


# (m, n, batch) -> cluster size for both dtypes; the GPU tests below use these shapes
SYEVJ_ROUTES = [
    # (m, n, batch, dtype, cluster size)
    (64, 64, 1, torch.float32, 8),
    (64, 64, 1, torch.float64, 8),
    (64, 64, 64, torch.float32, 2),
    (64, 64, 64, torch.float64, 2),
    (128, 128, 40, torch.float32, 1),
    (128, 128, 40, torch.float64, 1),
    (32, 32, 64, torch.float32, 4),
    (32, 32, 64, torch.float64, 4),
    (1200, 1200, 1, torch.float64, 4),
    (1200, 1200, 2, torch.float64, 0),
    (1184, 1184, 2, torch.float64, 0),
    (2700, 2700, 1, torch.float32, 0),
]
GESVJ_ROUTES = [
    (6000, 64, 1, torch.float64, 0),
    (12000, 64, 1, torch.float32, 0),
]


def test_jacobi_planner_copy_reaches_every_route():
    """The shapes of this file reach cluster sizes 1, 2, 4, 8 and the unfused round in both dtypes (no GPU needed)."""
    reached = {torch.float32: set(), torch.float64: set()}
    for m, n, batch, dtype, cs in SYEVJ_ROUTES + GESVJ_ROUTES:
        assert jacobi_cluster_size(m, n, batch, dtype) == cs, (m, n, batch, dtype)
        reached[dtype].add(cs)
    for dtype, got in reached.items():
        assert got == {0, 1, 2, 4, 8}, (dtype, sorted(got))
    # the float64 6000 x 64 SVD runs 16 Gram partials and the last one is ragged; so does the float32 12000 x 64 one
    assert jacobi_gram_partials(6000, 64, 1) == (16, 384) and 6000 % 384 != 0
    assert jacobi_gram_partials(12000, 64, 1) == (16, 768) and 12000 % 768 != 0
    # the documented borders of the unfused round
    assert jacobi_cluster_size(1152, 1152, 2, torch.float64) == 4 and jacobi_cluster_size(1153, 1153, 2, torch.float64) == 0
    assert jacobi_cluster_size(1312, 1312, 1, torch.float64) == 4 and jacobi_cluster_size(1313, 1313, 1, torch.float64) == 0
    assert jacobi_cluster_size(2624, 2624, 1, torch.float32) == 8 and jacobi_cluster_size(2625, 2625, 1, torch.float32) == 0
    assert jacobi_launches(64, 3, True, 8) == 5 + 3 * 3 + 2
    assert jacobi_launches(64, 3, False, 0) == 5 + 3 * 3 * 3 + 3


# --------------------------------------------------------------------------------------------------
# Jacobi on the GPU
# --------------------------------------------------------------------------------------------------
def _orth(n, g):
    Q, R = torch.linalg.qr(torch.randn(n, n, generator=g, dtype=torch.float64))
    return Q * torch.sign(torch.diagonal(R))


def _sym(lam, g):
    Q = _orth(lam.numel(), g)
    A = (Q * lam) @ Q.T
    return (A + A.T) / 2


def _mixed_batch(n, batch, g):
    """Members that converge at different speeds: SPD, diagonal with distinct entries (every panel skipped), zero,
    rank n/2 PSD, a triply repeated eigenvalue, then SPD matrices with condition numbers from 10 to 1e6."""
    mats = [_sym(torch.logspace(0, -3, n, dtype=torch.float64), g)]
    d = torch.linspace(-1.0, 2.0, n, dtype=torch.float64)
    mats.append(torch.diag(d[torch.randperm(n, generator=g)]))
    mats.append(torch.zeros(n, n, dtype=torch.float64))
    half = torch.cat([0.5 + torch.rand(n // 2, generator=g, dtype=torch.float64),
                      torch.zeros(n - n // 2, dtype=torch.float64)])
    mats.append(_sym(half, g))
    rep = 0.2 + torch.rand(n, generator=g, dtype=torch.float64)
    rep[n // 3:n // 3 + 3] = 0.7
    mats.append(_sym(rep, g))
    for i in range(batch - len(mats)):
        mats.append(_sym(torch.logspace(0, -1 - 5 * i / max(1, batch - 6), n, dtype=torch.float64), g))
    return torch.stack(mats[:batch])


# Bounds in units of n u ||A||_2 (orthogonality: n u), rank-deficient and zero members included.  The largest errors
# seen on an H100 were 0.38 (eigenvalues), 0.21 (orthogonality) and 1.4 (residual, a rank n/2 member).
C_VAL, C_ORTH, C_RES = 2, 1, 4


def _check_eigh(A, ev, Vt, dtype, what):
    """A (float64 CPU, the dtype-rounded input), ev / Vt from syevj."""
    n = A.shape[-1]
    u = U[dtype]
    ev, Vt = ev.double().cpu(), Vt.double().cpu()
    ref = torch.linalg.eigvalsh(A).flip(0)
    nrm = float(ref.abs().max())
    e_val = float((ev - ref).abs().max())
    e_orth = float((Vt @ Vt.T - torch.eye(n, dtype=torch.float64)).abs().max())
    e_res = float((A @ Vt.T - Vt.T * ev).abs().max())
    print(f"{what}: eig {e_val / (n * u * max(nrm, 1e-300)):.3f}  orth {e_orth / (n * u):.3f}  "
          f"resid {e_res / (n * u * max(nrm, 1e-300)):.3f}  (in units of n u ||A||)")
    assert torch.all(ev[:-1] >= ev[1:]), f"{what}: eigenvalues not in descending order"
    assert e_val <= C_VAL * n * u * nrm, f"{what}: eigenvalue error {e_val:.3e}"
    assert e_orth <= C_ORTH * n * u, f"{what}: ||V V^T - I|| = {e_orth:.3e}"
    assert e_res <= C_RES * n * u * nrm, f"{what}: residual {e_res:.3e}"
    return ref


def _syevj_counted(A, cs, **kw):
    from cca_zoo_b200 import ops

    l0 = _launches()
    ev, Vt, info = ops.syevj(A, return_info=True, **kw)
    got = _launches() - l0
    assert info["converged"], f"syevj did not converge: {info}"
    n = A.shape[-1]
    assert got == jacobi_launches(n, info["sweeps"], True, cs), (
        f"launch count {got} does not match the {'fused (cluster ' + str(cs) + ')' if cs else 'unfused'} round "
        f"with {info['sweeps']} sweeps")
    print(f"syevj n={n} batch={A.shape[0] if A.dim() == 3 else 1} route cs={cs}: {info['sweeps']} sweeps, {got} launches")
    return ev, Vt, info


@pytest.mark.gpu
@pytest.mark.parametrize("dtype", [torch.float32, torch.float64])
@pytest.mark.parametrize("n,batch,cs", [(128, 40, 1), (64, 64, 2), (32, 64, 4)])
def test_syevj_mixed_batch_on_each_cluster_size(dtype, n, batch, cs):
    assert jacobi_cluster_size(n, n, batch, dtype) == cs
    g = torch.Generator().manual_seed(1000 * n + batch)
    A = _mixed_batch(n, batch, g).to(dtype)
    ev, Vt, _ = _syevj_counted(A.cuda(), cs)
    failures = []
    for b in range(batch):
        try:
            _check_eigh(A[b].double(), ev[b], Vt[b], dtype, f"{dtype} n={n} member {b}")
        except AssertionError as e:
            failures.append(str(e).splitlines()[0])
    assert not failures, failures
    # the diagonal member: every panel is skipped, the values are the sorted diagonal, the vectors a permutation
    diag = torch.diagonal(A[1])
    assert torch.equal(ev[1].cpu(), torch.sort(diag, descending=True).values)
    P = Vt[1].cpu()
    assert torch.all((P == 0) | (P == 1)) and torch.all(P.sum(0) == 1) and torch.all(P.sum(1) == 1)
    assert torch.equal(P @ diag, ev[1].cpu())
    # the zero member: exact zeros, identity vectors
    assert torch.all(ev[2] == 0) and torch.equal(Vt[2].cpu(), torch.eye(n, dtype=dtype))


@pytest.mark.gpu
def test_syevj_float64_n1200_alone_and_in_a_pair_take_cluster_4_and_the_unfused_round():
    g = torch.Generator().manual_seed(1200)
    A = _sym(0.01 + 0.99 * torch.rand(1200, generator=g, dtype=torch.float64), g)
    ev1, Vt1, _ = _syevj_counted(A.cuda(), 4)
    ev2, Vt2, _ = _syevj_counted(torch.stack([A, A]).cuda(), 0)
    _check_eigh(A, ev1, Vt1, torch.float64, "f64 n=1200 cluster 4")
    _check_eigh(A, ev2[0], Vt2[0], torch.float64, "f64 n=1200 unfused")
    assert torch.equal(ev2[0], ev2[1]) and torch.equal(Vt2[0], Vt2[1]), "identical batch members must agree bitwise"
    assert float((ev1 - ev2[0]).abs().max()) <= C_VAL * 1200 * U[torch.float64] * float(ev1.abs().max())


@pytest.mark.gpu
def test_syevj_float32_n64_alone_and_repeated_take_cluster_8_and_cluster_2():
    g = torch.Generator().manual_seed(64)
    A = _sym(torch.logspace(0, -2, 64, dtype=torch.float64), g).float()
    ev1, Vt1, _ = _syevj_counted(A.cuda(), 8)
    ev2, Vt2, _ = _syevj_counted(A.expand(64, 64, 64).contiguous().cuda(), 2)
    _check_eigh(A.double(), ev1, Vt1, torch.float32, "f32 n=64 cluster 8")
    _check_eigh(A.double(), ev2[0], Vt2[0], torch.float32, "f32 n=64 cluster 2")
    assert all(torch.equal(ev2[0], ev2[b]) and torch.equal(Vt2[0], Vt2[b]) for b in range(64))
    assert float((ev1 - ev2[0]).abs().max()) <= C_VAL * 64 * U[torch.float32] * float(ev1.abs().max())


@pytest.mark.gpu
def test_syevj_float32_n2700_unfused():
    """Eigenvalues in [0.01, 1].  The smallest lie below 10 n u ||A||_F = 0.048: a noise floor that large left their
    directions unrefined (eigenvalue errors of 7.6e-3) while the solve still reported convergence."""
    g = torch.Generator().manual_seed(2700)
    A = _sym(0.01 + 0.99 * torch.rand(2700, generator=g, dtype=torch.float64), g).float()
    ev, Vt, _ = _syevj_counted(A.cuda(), 0)
    _check_eigh(A.double(), ev, Vt, torch.float32, "f32 n=2700 unfused")


@pytest.mark.gpu
def test_syevj_indefinite_with_shift_unfused():
    """Jordan-Wielandt matrix (eigenvalues +-sigma of its block) and a symmetric indefinite matrix, shifted to PSD."""
    g = torch.Generator().manual_seed(1184)
    T = torch.randn(600, 584, generator=g, dtype=torch.float64) / 50
    K = torch.zeros(1184, 1184, dtype=torch.float64)
    K[:600, 600:] = T
    K[600:, :600] = T.T
    S = _sym(torch.linspace(-1.0, 2.0, 1184, dtype=torch.float64), g)
    A = torch.stack([K, S])
    shift = float(max(torch.linalg.matrix_norm(K), torch.linalg.matrix_norm(S)))
    ev, Vt, _ = _syevj_counted(A.cuda(), 0, shift=shift)
    for b in range(2):
        _check_eigh(A[b], ev[b], Vt[b], torch.float64, f"f64 n=1184 shifted member {b}")
    sv = torch.linalg.svdvals(T)
    assert float((ev[0, :584].cpu() - sv).abs().max()) <= C_VAL * 1184 * U[torch.float64] * float(sv[0])


@pytest.mark.gpu
@pytest.mark.parametrize("m,n,dtype", [(6000, 64, torch.float64), (12000, 64, torch.float32)])
def test_gesvj_tall_unfused_with_ragged_gram_partials(m, n, dtype):
    from cca_zoo_b200 import ops

    assert jacobi_cluster_size(m, n, 1, dtype) == 0
    g = torch.Generator().manual_seed(m)
    Q, _ = torch.linalg.qr(torch.randn(m, n, generator=g, dtype=torch.float64))
    sig_in = torch.linspace(1.0, 0.5, n, dtype=torch.float64)
    G = ((Q * sig_in) @ _orth(n, g).T).to(dtype)
    l0 = _launches()
    sig, Rt, Lt, info = ops.gesvj(G.T.contiguous().cuda(), return_info=True)
    got = _launches() - l0
    assert info["converged"], info
    assert got == jacobi_launches(n, info["sweeps"], True, 0), (got, info)
    print(f"gesvj {m}x{n} {dtype} unfused: {info['sweeps']} sweeps, {got} launches")
    G = G.double()
    sig, Rt, Lt = sig.double().cpu(), Rt.double().cpu(), Lt.double().cpu()
    ref = torch.linalg.svdvals(G)
    u, nrm, kappa = U[dtype], float(ref[0]), float(ref[0] / ref[-1])
    e_sig = float((sig - ref).abs().max())
    e_rec = float(((Lt.T * sig) @ Rt - G).abs().max())
    e_right = float((Rt @ Rt.T - torch.eye(n, dtype=torch.float64)).abs().max())
    e_left = float((Lt @ Lt.T - torch.eye(n, dtype=torch.float64)).abs().max())
    print(f"gesvj {m}x{n}: sigma {e_sig / (n * u * nrm):.3f}  recon {e_rec / (n * u * nrm):.3f}  "
          f"right {e_right / (n * u):.3f}  left {e_left / (n * u * kappa):.3f}  (units of n u [||G||, kappa])")
    assert torch.all(sig[:-1] >= sig[1:])
    # largest seen on an H100: 0.094, 0.011, 0.094 and 0.26 of these units
    assert e_sig <= n * u * nrm
    assert e_rec <= n * u * nrm
    assert e_right <= n * u
    assert e_left <= n * u * kappa


# --------------------------------------------------------------------------------------------------
# CCALoss on the fused small-width kernels
# --------------------------------------------------------------------------------------------------
def _loss_views(n, d1, d2, dtype, seed):
    """Two views sharing a 3-dimensional latent signal; cond(S_ii) stays below about 1e3."""
    g = torch.Generator().manual_seed(seed)
    t = torch.randn(n, 3, generator=g, dtype=torch.float64)
    zs = [0.5 * t @ torch.randn(3, d, generator=g, dtype=torch.float64) + torch.randn(n, d, generator=g,
                                                                                     dtype=torch.float64) + 0.3
          for d in (d1, d2)]
    return [z.to(dtype) for z in zs]


def _check_ccaloss(n, d1, d2, dtype, fwd_launches, bwd_launches):
    from cca_zoo_b200.deep import CCALoss
    from oracle.restatement import cov_ccaloss

    tol = 1e-9 if dtype == torch.float64 else 2e-4
    z1, z2 = _loss_views(n, d1, d2, dtype, seed=100 * d1 + d2 + n)
    L, ga, gb = cov_ccaloss(z1.double().numpy(), z2.double().numpy(), 1e-5)
    for layout in ("contiguous", "slices"):
        fn = CCALoss(eps=1e-5)
        if layout == "contiguous":
            a = z1.cuda().requires_grad_()
            b = z2.cuda().requires_grad_()
            za, zb, scale = a, b, 1.0
        else:                         # column slices of wider tensors (ld > d), upstream gradient 3
            a = torch.zeros(n, d1 + 7, dtype=dtype, device="cuda")
            a[:, 2:2 + d1] = z1.cuda()
            b = torch.zeros(n, d2 + 5, dtype=dtype, device="cuda")
            b[:, 3:3 + d2] = z2.cuda()
            a.requires_grad_()
            b.requires_grad_()
            za, zb, scale = a[:, 2:2 + d1], b[:, 3:3 + d2], 3.0
        l0 = _launches()
        loss = fn([za, zb])
        l1 = _launches()
        (loss * scale if scale != 1.0 else loss).backward()
        l2 = _launches()
        fn.check()
        fwd_launches(l1 - l0)
        bwd_launches(l2 - l1)
        what = f"CCALoss {dtype} n={n} ({d1},{d2}) {layout}"
        print(f"{what}: {l1 - l0} forward / {l2 - l1} backward launches")
        assert abs(loss.item() - L) <= tol * abs(L), f"{what}: loss {loss.item()!r} vs {L!r}"
        g1 = a.grad[:, 2:2 + d1] if layout == "slices" else a.grad
        g2 = b.grad[:, 3:3 + d2] if layout == "slices" else b.grad
        for got, ref in ((g1, ga), (g2, gb)):
            err = np.abs(got.double().cpu().numpy() - scale * ref).max()
            assert err <= tol * scale * np.abs(ref).max(), f"{what}: gradient error {err:.3e}"
        if layout == "slices":        # columns outside the slices receive exactly zero
            assert float(a.grad[:, :2].abs().max()) == 0 and float(a.grad[:, 2 + d1:].abs().max()) == 0
            assert float(b.grad[:, :3].abs().max()) == 0 and float(b.grad[:, 3 + d2:].abs().max()) == 0


def _eq(k):
    def check(got):
        assert got == k, f"expected {k} launches, got {got}"
    return check


def _potrf_inv_launches(n, dtype):
    from cca_zoo_b200 import ops

    A = torch.eye(n, dtype=dtype, device="cuda")
    l0 = _launches()
    ops.potrf_inv_(A)
    return _launches() - l0


@pytest.mark.gpu
@pytest.mark.parametrize("dtype", [torch.float32, torch.float64])
@pytest.mark.parametrize("n,d1,d2", [(1000, 1, 1), (1000, 1, 64), (1000, 20, 50), (1000, 50, 20), (1000, 32, 33),
                                     (1000, 33, 33), (1000, 63, 40), (1000, 64, 64), (48, 20, 33)])
def test_ccaloss_small_width_kernels(dtype, n, d1, d2):
    """Moment pass + reduction + ccaloss_small_fwd_kernel forward, ccaloss_small_bwd_kernel backward."""
    _check_ccaloss(n, d1, d2, dtype, _eq(3), _eq(1))


@pytest.mark.gpu
@pytest.mark.parametrize("dtype", [torch.float32, torch.float64])
@pytest.mark.parametrize("d1,d2", [(64, 65), (65, 65)])
def test_ccaloss_first_widths_past_the_small_kernels(dtype, d1, d2):
    """Unbatched (64, 65) and batched (65, 65) potrf_inv route.  Forward: moment pass + reduction, covariance + ridge,
    potrf_inv of S_11 and S_22 (one batched call when the widths agree, else one call each), A_i = Linv_i^T Linv_i (one
    batched product, else two), five products for Q, Q2, P, G11, G22, and the two-stage loss reduction.  Backward: four
    products and the column-sum / centring pair of each gradient."""
    p1, p2 = _potrf_inv_launches(d1, dtype), _potrf_inv_launches(d2, dtype)
    fwd = 2 + 1 + (p1 + 1 if d1 == d2 else p1 + p2 + 2) + 5 + 2
    _check_ccaloss(1000, d1, d2, dtype, _eq(fwd), _eq(8))


# --------------------------------------------------------------------------------------------------
# ops.gemm dispatch
# --------------------------------------------------------------------------------------------------
def _fma32(a, b, c):
    """Correctly rounded float32 fma(a, b, c), elementwise on float32 numpy arrays: a*b is exact in float64, the sum's
    rounding error is recovered exactly (TwoSum) and decides the float32 midpoints that a plain cast would round to
    even."""
    p = a.astype(np.float64) * b.astype(np.float64)
    c64 = c.astype(np.float64)
    s = p + c64
    bb = s - p
    e = (p - (s - bb)) + (c64 - bb)
    r = s.astype(np.float32)
    rd = r.astype(np.float64)
    other = 2.0 * s - rd
    mid = (rd != s) & (other.astype(np.float32).astype(np.float64) == other) & (e != 0)
    fixed = np.where(e > 0, np.maximum(rd, other), np.minimum(rd, other)).astype(np.float32)
    return np.where(mid, fixed, r)


def _fma_gemm32(opA, opB, alpha, beta, C):
    """What the FMA kernel computes: acc = fma(a_ik, b_kj, acc) for k in order, then alpha * acc + beta * C (alpha and
    beta powers of two, so the epilogue rounds once however it is contracted)."""
    acc = np.zeros((opA.shape[0], opB.shape[1]), dtype=np.float32)
    for t in range(opA.shape[1]):
        acc = _fma32(np.broadcast_to(opA[:, t:t + 1], acc.shape), np.broadcast_to(opB[t:t + 1, :], acc.shape), acc)
    return (np.float64(alpha) * acc.astype(np.float64) + np.float64(beta) * C.astype(np.float64)).astype(np.float32)


def _out_views(m, n, dtype, g):
    """Two parents holding identical C values: one view 16-byte aligned with ld % 4 == 0, one offset by an element."""
    C = torch.randn(m, n, generator=g, dtype=torch.float64).to(dtype)
    pa = torch.randn(m, n + 8, generator=g, dtype=torch.float64).to(dtype).cuda()
    pb = pa.clone()
    pa[:, 4:4 + n] = C.cuda()
    pb[:, 5:5 + n] = C.cuda()
    return C, (pa, pa[:, 4:4 + n]), (pb, pb[:, 5:5 + n])


def _untouched(parent, before, lo, hi):
    return torch.equal(parent[:, :lo], before[:, :lo]) and torch.equal(parent[:, hi:], before[:, hi:])


@pytest.mark.gpu
@pytest.mark.parametrize("ta,tb", [(False, False), (True, False), (False, True), (True, True)])
@pytest.mark.parametrize("m,n,k,route", [(128, 128, 128, "tensor"), (127, 128, 128, "fma"),
                                         (256, 256, 256, "fma-unaligned-A")])
def test_gemm_float32_dispatch(ta, tb, m, n, k, route):
    from cca_zoo_b200 import ops

    g = torch.Generator().manual_seed(m + n + k + 2 * ta + tb)
    ashape = (k, m) if ta else (m, k)
    A64 = torch.randn(ashape, generator=g, dtype=torch.float64)
    B64 = torch.randn((n, k) if tb else (k, n), generator=g, dtype=torch.float64)
    A, B = A64.float(), B64.float()
    Ad = A.cuda()
    if route == "fma-unaligned-A":    # a view with ld % 4 != 0: TMA cannot address it
        wide = torch.zeros(ashape[0], ashape[1] + 1, dtype=torch.float32, device="cuda")
        wide[:, :ashape[1]] = Ad
        Ad = wide[:, :ashape[1]]
        assert Ad.stride(0) % 4 != 0
    Bd = B.cuda()
    alpha, beta = -0.5, 2.0
    C, (pa, va), (pb, vb) = _out_views(m, n, torch.float32, g)
    pa0, pb0 = pa.clone(), pb.clone()
    ops.gemm(Ad, Bd, transa=ta, transb=tb, alpha=alpha, beta=beta, out=va)     # vec_c = 1 on the tensor route
    ops.gemm(Ad, Bd, transa=ta, transb=tb, alpha=alpha, beta=beta, out=vb)     # vec_c = 0 (misaligned out)
    torch.cuda.synchronize()
    assert torch.equal(va, vb), "aligned and misaligned outputs must agree bitwise"
    assert _untouched(pa, pa0, 4, 4 + n) and _untouched(pb, pb0, 5, 5 + n), "gemm wrote outside its output view"
    opA = (A.T if ta else A).double()
    opB = (B.T if tb else B).double()
    absAB = (opA.abs() @ opB.abs()).numpy()
    ref = (alpha * (opA @ opB) + beta * C.double()).numpy()
    err = np.abs(va.double().cpu().numpy() - ref)
    bound = k * U[torch.float32] * (abs(alpha) * absAB + abs(beta) * np.abs(C.double().numpy()))
    if route == "tensor":
        # the same kernel as gemm_tc with the same arguments
        tc_a = pa0[:, 4:4 + n].clone()
        tc_b = pb0.clone()[:, 5:5 + n]
        ops.gemm_tc(Ad, Bd, transa=ta, transb=tb, alpha=alpha, beta=beta, out=tc_a)
        ops.gemm_tc(Ad, Bd, transa=ta, transb=tb, alpha=alpha, beta=beta, out=tc_b)
        assert torch.equal(va, tc_a) and torch.equal(va, tc_b), "ops.gemm did not take the tensor-core route"
        ratio = float((err / bound).max())
        print(f"gemm f32 {m}x{n}x{k} ta={ta} tb={tb} 3xTF32: max error / (k u |A||B|) = {ratio:.3f}")
        assert ratio <= 0.25              # 0.032 seen on an H100: the split operands lose about 2^-21 per product
    else:
        emu = _fma_gemm32(opA.float().numpy(), opB.float().numpy(), alpha, beta, C.numpy())
        assert np.array_equal(va.cpu().numpy(), emu), "ops.gemm did not take the FMA route (or its fma chain changed)"
        ratio = float((err / bound).max())
        print(f"gemm f32 {m}x{n}x{k} ta={ta} tb={tb} FMA: max error / (k u |A||B|) = {ratio:.3f}")
        assert ratio <= (k + 1) / k       # gamma_k for the chain, one more rounding in the epilogue


def _kernel_names(fn):
    """Names of the CUDA kernels that ``fn`` launches, from the profiler's device activity."""
    from torch.profiler import ProfilerActivity, profile

    torch.cuda.synchronize()
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        fn()
        torch.cuda.synchronize()
    return [e.name for e in prof.events() if e.device_type == torch.autograd.DeviceType.CUDA]


@pytest.mark.gpu
@pytest.mark.parametrize("ta,tb", [(False, False), (True, False), (False, True), (True, True)])
@pytest.mark.parametrize("k", [1, 7, 8, 17, 1000])
def test_gemm_float64_fma_and_dmma(ta, tb, k):
    """k < 8 takes the FMA tiles, k >= 8 the DMMA kernel (pinned by the kernel names the profiler records).  Reference
    in long double (64-bit significand)."""
    from cca_zoo_b200 import ops

    g = torch.Generator().manual_seed(7 * k + 2 * ta + tb)
    alpha, beta = -0.75, 1.5
    A = torch.randn((k, 65) if ta else (65, k), dtype=torch.float64, device="cuda")
    B = torch.randn((65, k) if tb else (k, 65), dtype=torch.float64, device="cuda")
    names = _kernel_names(lambda: ops.gemm(A, B, transa=ta, transb=tb))
    want, other = ("dgemm_mma_kernel", "gemm_kernel<double") if k >= 8 else ("gemm_kernel<double", "dgemm_mma_kernel")
    assert sum(want in s for s in names) == 1 and not any(other in s for s in names), names
    for m in (1, 65, 130):
        for n in (1, 65, 130):
            A = torch.randn((k, m) if ta else (m, k), generator=g, dtype=torch.float64)
            B = torch.randn((n, k) if tb else (k, n), generator=g, dtype=torch.float64)
            C, (pa, va), _ = _out_views(m, n, torch.float64, g)
            pa0 = pa.clone()
            ops.gemm(A.cuda(), B.cuda(), transa=ta, transb=tb, alpha=alpha, beta=beta, out=va)
            opA = (A.T if ta else A).numpy().astype(np.longdouble)
            opB = (B.T if tb else B).numpy().astype(np.longdouble)
            Cl = C.numpy().astype(np.longdouble)
            ref = np.longdouble(alpha) * (opA @ opB) + np.longdouble(beta) * Cl
            bound = (k + 2) * U[torch.float64] * (abs(alpha) * (np.abs(opA) @ np.abs(opB)) + abs(beta) * np.abs(Cl))
            err = np.abs(va.cpu().numpy().astype(np.longdouble) - ref)
            assert np.all(err <= bound), f"m={m} n={n} k={k}: error / bound = {float((err / bound).max()):.3f}"
            assert _untouched(pa, pa0, 4, 4 + n), "gemm wrote outside its output view"
