"""TCCALoss on bfloat16 / float16 representations: the moment pass reads them as they are, everything after it runs
in float64, the loss is float32 and the gradients come back in the representations' dtype.  Compared with TCCALoss on
float64 copies of the same values."""
import pytest
import torch

from cca_zoo_b200.deep import TCCALoss

pytestmark = pytest.mark.gpu

HALF = [torch.bfloat16, torch.float16]


def _reps(n, widths, dtype, seed):
    g = torch.Generator(device="cuda").manual_seed(seed)
    latent = torch.randn(n, 4, generator=g, device="cuda")
    return [(latent @ torch.randn(4, w, generator=g, device="cuda")
             + torch.randn(n, w, generator=g, device="cuda")).to(dtype).requires_grad_() for w in widths]


def _ulp(x, dtype):
    """One ulp of the 16-bit dtype at |x| (float64), with the smallest normal exponent as the floor."""
    mant, emin = (7, -126) if dtype == torch.bfloat16 else (10, -14)
    e = torch.floor(torch.log2(x.abs().clamp_min(2.0 ** emin)))
    return torch.pow(2.0, e - mant)


def _loss_and_grads(loss_fn, zs):
    loss = loss_fn(zs)
    grads = torch.autograd.grad(loss, zs)
    return loss.detach(), grads


# (batch, widths): the Cholesky route for three and four views, and a batch narrower than the width (eigen route)
SHAPES = [(4096, [64, 64, 64]), (4096, [32, 32, 32, 32]), (48, [64, 64])]


@pytest.mark.parametrize("dtype", HALF)
@pytest.mark.parametrize("shape", SHAPES, ids=["4096x64x3", "4096x32x4", "48x64x2_eigen"])
@pytest.mark.parametrize("verify", ["lazy", "sync"])
def test_16_bit_matches_the_float64_copy(shape, dtype, verify):
    n, widths = shape
    zs = _reps(n, widths, dtype, n + sum(widths))
    fn = TCCALoss(eps=1e-3, verify=verify)
    loss, grads = _loss_and_grads(fn, zs)
    fn.check()
    z64 = [z.detach().double().requires_grad_() for z in zs]
    loss64, grads64 = _loss_and_grads(TCCALoss(eps=1e-3, verify=verify), z64)
    assert loss.dtype == torch.float32
    assert abs(loss.item() - loss64.item()) <= 1e-5 * abs(loss64.item())
    for g, g64 in zip(grads, grads64):
        assert g.dtype == dtype
        # on the host, where pow(2, e) is exact: the tolerance is one ulp, not a rounding below it
        g, ref = g.double().cpu(), g64.to(dtype).double().cpu()
        # one ulp of the rounded float64 gradient, entries below 1 % of the largest measured in the ulp at that level
        floor = 1e-2 * ref.abs().max()
        tol = _ulp(torch.maximum(ref.abs(), floor), dtype)
        assert ((g - ref).abs() <= tol).all(), ((g - ref).abs() / tol).max().item()


@pytest.mark.parametrize("dtype", HALF)
def test_mixed_16_and_32_bit_raise(dtype):
    zs = _reps(256, [8, 8, 4], torch.float32, 0)
    mixed = [zs[0].detach().to(dtype), zs[1].detach(), zs[2].detach()]
    with pytest.raises(ValueError):
        TCCALoss()(mixed)
    with pytest.raises(ValueError):
        TCCALoss()(mixed[::-1])


def test_autocast_encoder_trains_one_step():
    torch.manual_seed(0)
    enc = [torch.nn.Sequential(torch.nn.Linear(100, 128), torch.nn.ReLU(), torch.nn.Linear(128, 16)).cuda()
           for _ in range(3)]
    opt = torch.optim.SGD([p for e in enc for p in e.parameters()], lr=1e-3)
    x = [torch.randn(1024, 100, device="cuda") for _ in range(3)]
    loss_fn = TCCALoss()
    with torch.autocast("cuda", dtype=torch.bfloat16):
        z = [e(xi) for e, xi in zip(enc, x)]
        assert z[0].dtype == torch.bfloat16
        loss = loss_fn(z)
    assert loss.dtype == torch.float32 and torch.isfinite(loss)
    loss.backward()
    loss_fn.check()
    for e in enc:
        for p in e.parameters():
            assert p.grad is not None and torch.isfinite(p.grad).all()
    opt.step()
