"""Batched blocked Cholesky + explicit inverse (ccab_potrf_inv) against float64 torch on the host."""
import pytest
import torch

pytestmark = pytest.mark.gpu


def _spd(n, batch, dtype, seed, cond=50.0):
    g = torch.Generator().manual_seed(seed)
    X = torch.randn(batch, 3 * n, n, generator=g, dtype=torch.float64)
    A = X.transpose(1, 2) @ X / (3 * n)
    A = A + torch.eye(n, dtype=torch.float64) / cond
    return A.to(dtype)


@pytest.mark.parametrize("dtype,tol", [(torch.float32, 2e-4), (torch.float64, 1e-11)])
@pytest.mark.parametrize("n,batch", [(5, 1), (17, 1), (64, 2), (100, 1), (128, 3), (200, 2), (256, 1), (300, 1),
                                     (512, 2), (640, 1), (1000, 1), (1024, 2)])
def test_potrf_inv_matches_float64(dtype, tol, n, batch):
    from cca_zoo_b200 import ops

    A = _spd(n, batch, dtype, n + batch)
    Ad = A.cuda().clone()
    Linv, info = ops.potrf_inv_(Ad)
    assert int(info.max().item()) == 0
    L = torch.tril(Ad).double().cpu()
    A64 = A.double()
    ref = torch.linalg.cholesky(A64)
    assert float((L - ref).abs().max() / ref.abs().max()) < tol
    Li = Linv.double().cpu()
    assert float(torch.triu(Li, 1).abs().max()) == 0.0          # exact zeros above the diagonal
    eye = torch.eye(n, dtype=torch.float64)
    assert float((Li @ ref - eye).abs().max()) < 20 * tol       # L^-1 against the float64 factor
    assert float((Li.transpose(1, 2) @ Li @ A64 - eye).abs().max()) < 50 * tol


def test_potrf_inv_2d_view_inside_a_larger_matrix_and_fma_route_for_an_unaligned_row_stride():
    """Diagonal blocks of one covariance matrix as a strided batch (the rCCA use, tensor-core panels), and the FMA
    fallback for matrices whose row stride TMA cannot address."""
    from cca_zoo_b200 import ops

    C = torch.zeros(512, 512, dtype=torch.float32)
    A = _spd(256, 2, torch.float32, 3)
    C[:256, :256], C[256:, 256:] = A[0], A[1]
    Cd = C.cuda()
    blocks = torch.as_strided(Cd, (2, 256, 256), (256 * 513, 512, 1))
    Linv, info = ops.potrf_inv_(blocks)
    assert int(info.max().item()) == 0
    ref = torch.linalg.cholesky(A.double())
    assert float((Linv.double().cpu() @ ref - torch.eye(256, dtype=torch.float64)).abs().max()) < 2e-3
    # row stride 257 (not a multiple of 4): the panel and trailing-update GEMMs take the FMA kernel
    buf = torch.zeros(2 * 256 * 257, dtype=torch.float32, device="cuda")
    Ad = torch.as_strided(buf, (2, 256, 256), (256 * 257, 257, 1))
    Ad.copy_(A)
    Linv2, info2 = ops.potrf_inv_(Ad)
    assert int(info2.max().item()) == 0
    assert float((Linv2 - Linv).abs().max() / Linv.abs().max()) < 1e-4


def test_potrf_inv_flags_a_non_positive_definite_matrix():
    from cca_zoo_b200 import ops

    A = _spd(300, 2, torch.float64, 9)
    A[1, 150, 150] = -1.0
    _, info = ops.potrf_inv_(A.cuda())
    info = info.cpu()
    assert int(info[0]) == 0 and int(info[1]) == 151
