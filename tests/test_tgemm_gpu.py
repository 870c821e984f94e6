"""wgmma GEMM (ccab_gemm_tc) against a float64 torch product: every op() combination (= every pairing of
K-major / MN-major shared-memory operands), ragged sizes (TMA zero fill), batches, alpha / beta, the transposed
copy and the lower-triangle-only mode.  Tolerance: fp32-grade (3xTF32 products, fp32 accumulation)."""
import pytest
import torch

pytestmark = pytest.mark.gpu


def _ref(A, B, ta, tb):
    a = A.double().transpose(-1, -2) if ta else A.double()
    b = B.double().transpose(-1, -2) if tb else B.double()
    return a @ b


def _rel(x, ref):
    return float((x.double() - ref).abs().max() / ref.abs().max())


@pytest.mark.parametrize("ta", [False, True])
@pytest.mark.parametrize("tb", [False, True])
@pytest.mark.parametrize("m,n,k", [(128, 128, 32), (128, 64, 256), (256, 384, 128), (1024, 1024, 1024),
                                   (200, 136, 72), (96, 96, 1000), (1000, 96, 1024), (4096, 512, 512), (36, 20, 8)])
def test_gemm_tc_matches_float64(ta, tb, m, n, k):
    from cca_zoo_b200 import ops

    g = torch.Generator(device="cuda").manual_seed(m * 7 + n * 3 + k)
    A = torch.randn((k, m) if ta else (m, k), generator=g, device="cuda")
    B = torch.randn((n, k) if tb else (k, n), generator=g, device="cuda")
    ref = _ref(A, B, ta, tb)
    out_t = torch.empty((n, m), device="cuda")
    out = ops.gemm_tc(A, B, transa=ta, transb=tb, out_t=out_t)
    assert _rel(out, ref) < 4e-6 * max(1.0, (k / 256) ** 0.5), _rel(out, ref)
    assert torch.equal(out_t, out.T.contiguous())


def test_gemm_tc_alpha_beta_views_and_batches():
    from cca_zoo_b200 import ops

    g = torch.Generator(device="cuda").manual_seed(5)
    big = torch.randn(2048, 2048, generator=g, device="cuda")
    A = big[:1024, 1024:]                      # a sub-matrix view: ld = 2048, pointer offset 4096 bytes
    B = big[1024:, :1024]
    C0 = torch.randn(1024, 1024, generator=g, device="cuda")
    C = C0.clone()
    ops.gemm_tc(A, B, transb=True, alpha=-0.5, beta=2.0, out=C)
    ref = -0.5 * (A.double() @ B.double().T) + 2.0 * C0.double()
    assert _rel(C, ref) < 6e-6
    # batched, strided like the diagonal blocks of one matrix
    X = torch.randn(3, 256, 192, generator=g, device="cuda")
    Y = torch.randn(3, 192, 320, generator=g, device="cuda")
    out = ops.gemm_tc(X, Y)
    assert _rel(out, X.double() @ Y.double()) < 5e-6
    out = ops.gemm_tc(X, X, transa=True)       # the K1 pairing (both MN-major)
    assert _rel(out, X.double().transpose(1, 2) @ X.double()) < 5e-6


def test_gemm_tc_lower_only_leaves_upper_tiles_untouched():
    from cca_zoo_b200 import ops

    g = torch.Generator(device="cuda").manual_seed(6)
    P = torch.randn(512, 128, generator=g, device="cuda")
    C0 = torch.randn(512, 512, generator=g, device="cuda")
    C = C0.clone()
    ops.gemm_tc(P, P, transb=True, alpha=-1.0, beta=1.0, out=C, lower_only=True)
    ref = C0.double() - P.double() @ P.double().T
    low = torch.tril(torch.ones(512, 512, device="cuda")).bool()
    assert _rel(torch.where(low, C.double(), torch.zeros_like(ref)), torch.where(low, ref, torch.zeros_like(ref))) < 6e-6
    blk = torch.arange(512, device="cuda") // 128
    above = blk[None, :] > blk[:, None]        # whole 128 x 128 tiles strictly above the diagonal
    assert torch.equal(C[above], C0[above])


def test_gemm_tc_is_more_accurate_than_one_tf32_pass():
    """3xTF32 must deliver fp32-grade products: error well below the 2^-11 of a single TF32 pass."""
    from cca_zoo_b200 import ops

    g = torch.Generator(device="cuda").manual_seed(8)
    A = torch.randn(512, 512, generator=g, device="cuda") + 3.0
    B = torch.randn(512, 512, generator=g, device="cuda") - 2.0
    err = _rel(ops.gemm_tc(A, B), A.double() @ B.double())
    assert err < 5e-6, err


def test_gemm_tc_rejects_misaligned_operands():
    from cca_zoo_b200 import ops

    A = torch.randn(64, 50, device="cuda")     # ld = 50: not a multiple of 4
    with pytest.raises(ValueError):
        ops.gemm_tc(A, A, transb=True)
