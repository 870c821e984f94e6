"""Single-CTA two-sided Jacobi eigensolver (ccab_syevj_small) against float64 LAPACK on the host."""
import pytest
import torch

pytestmark = pytest.mark.gpu


@pytest.mark.parametrize("dtype,tol", [(torch.float32, 3e-6), (torch.float64, 1e-13)])
@pytest.mark.parametrize("n,batch", [(1, 1), (2, 3), (7, 2), (32, 1), (33, 2), (64, 4), (95, 1), (96, 2), (97, 1),
                                     (104, 2), (128, 2)])
def test_syevj_small_matches_lapack(dtype, tol, n, batch):
    from cca_zoo_b200 import ops

    if dtype == torch.float64 and n > 104:
        pytest.skip("float64: two copies of H and a slice of V fit one CTA's shared memory up to n = 104")
    g = torch.Generator().manual_seed(n * 31 + batch)
    X = torch.randn(batch, n, n, generator=g, dtype=torch.float64)
    A = (X + X.transpose(1, 2)) / 2                       # indefinite: two-sided Jacobi needs no shift
    lam, Vt, info = ops.syevj_small(A.to(dtype).cuda())
    assert int(info.min().item()) > 0
    ref = torch.linalg.eigvalsh(A).flip(-1)
    scale = float(ref.abs().max())
    assert float((lam.double().cpu() - ref).abs().max()) < tol * scale * max(1, n) ** 0.5
    V = Vt.double().cpu()
    eye = torch.eye(n, dtype=torch.float64)
    assert float((V @ V.transpose(1, 2) - eye).abs().max()) < 20 * tol
    resid = V @ A - lam.double().cpu().unsqueeze(-1) * V   # rows: v^T A - lam v^T
    assert float(resid.abs().max()) < 30 * tol * scale


def test_syevj_small_gram_matrix_descending_and_repeatable():
    from cca_zoo_b200 import ops

    g = torch.Generator().manual_seed(3)
    Y = torch.randn(1024, 96, generator=g)
    H = (Y.T @ Y).cuda()
    lam1, V1, _ = ops.syevj_small(H)
    lam2, V2, _ = ops.syevj_small(H)
    assert torch.equal(lam1, lam2) and torch.equal(V1, V2)
    assert bool((lam1[:-1] >= lam1[1:]).all())
    ref = torch.linalg.eigvalsh(H.double().cpu()).flip(-1)
    assert float((lam1.double().cpu() - ref).abs().max() / ref.max()) < 3e-6
