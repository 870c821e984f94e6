"""bfloat16 / float16 views end to end: the estimators that hand their views to ``_local_moments`` read them with the
16-bit moment kernels (no float64 copy) and solve exactly as for a float64 copy; the deep objectives take 16-bit
representations through the moment pass and run their loss stage and backward in float32."""
import numpy as np
import pytest
import torch

from cca_zoo_b200 import _lib, ops
from cca_zoo_b200.deep import CCALoss, GCCALoss, MCCALoss
from cca_zoo_b200.linear import GCCA, MCCA, PLS_ALS, rCCA
from cca_zoo_b200.model_selection import GridSearchCV

pytestmark = pytest.mark.gpu

HALF = [torch.bfloat16, torch.float16]


def _views(n, dims, dtype, integer, seed, device="cuda"):
    g = torch.Generator(device="cpu").manual_seed(seed)
    latent = torch.randn(n, 2, generator=g)
    out = []
    for d in dims:
        v = latent @ torch.randn(2, d, generator=g) + 0.5 * torch.randn(n, d, generator=g)
        if integer:
            v = (4 * v).round().clamp(-15, 15)
        out.append(v.to(dtype).to(device))
    return out


ESTIMATORS = {
    "rcca": (lambda: rCCA(latent_dimensions=2, c=0.1), [40, 30]),
    "mcca": (lambda: MCCA(latent_dimensions=2, c=0.1), [40, 30, 20]),
    "gcca": (lambda: GCCA(latent_dimensions=2, c=0.1), [40, 30, 20]),
    "pls_als": (lambda: PLS_ALS(latent_dimensions=2, random_state=0), [40, 30]),
}


def _rel(w, w_ref):
    """Largest relative difference per weight vector, up to sign."""
    worst = 0.0
    for a, b in zip(w, w_ref):
        for k in range(b.shape[1]):
            s = np.sign(a[:, k] @ b[:, k]) or 1.0
            worst = max(worst, np.abs(s * a[:, k] - b[:, k]).max() / np.abs(b[:, k]).max())
    return worst


@pytest.mark.parametrize("dtype", HALF)
@pytest.mark.parametrize("name", list(ESTIMATORS))
def test_estimators_integer_views_bit_identical_to_float64_copy(name, dtype):
    make, dims = ESTIMATORS[name]
    v = _views(3000, dims, dtype, True, 1)
    est = make().fit(v)
    ref = make().fit([x.double() for x in v])
    assert all(w.dtype == np.float64 for w in est.weights_)
    for a, b in zip(est.weights_, ref.weights_):
        np.testing.assert_array_equal(a, b)


@pytest.mark.parametrize("dtype", HALF)
@pytest.mark.parametrize("name", list(ESTIMATORS))
def test_estimators_random_views_match_float64_copy(name, dtype):
    """Tolerance 1e-3 per weight vector, the smoke check of the float32 route: the 16-bit moments carry the error of
    fp32 runs (see test_moments_half_gpu.py), the solve is the float64 one."""
    make, dims = ESTIMATORS[name]
    v = _views(5000, dims, dtype, False, 2)
    est = make().fit(v)
    ref = make().fit([x.double() for x in v])
    assert all(w.dtype == np.float64 for w in est.weights_)
    assert _rel(est.weights_, ref.weights_) < 1e-3


@pytest.mark.parametrize("dtype", HALF)
def test_partial_fit_in_two_halves(dtype):
    v = _views(4000, [40, 30], dtype, True, 3)
    est = rCCA(latent_dimensions=2, c=0.1)
    est.partial_fit([x[:2000] for x in v], solve=False)
    est.partial_fit([x[2000:] for x in v])
    ref = rCCA(latent_dimensions=2, c=0.1).fit([x.double() for x in v])
    for a, b in zip(est.weights_, ref.weights_):
        np.testing.assert_array_equal(a, b)


@pytest.mark.parametrize("dtype", HALF)
def test_gridsearch_moment_route(dtype):
    v = _views(600, [20, 15], dtype, True, 4)
    grid = {"c": [0.0, 0.3, 0.8]}
    a = GridSearchCV(rCCA(latent_dimensions=2), grid, cv=3).fit(v)
    b = GridSearchCV(rCCA(latent_dimensions=2), grid, cv=3).fit([x.double() for x in v])
    np.testing.assert_array_equal(a.cv_results_["mean_test_score"], b.cv_results_["mean_test_score"])
    assert a.best_params_ == b.best_params_


@pytest.mark.parametrize("kind", ["numpy_float16", "cpu_bfloat16"])
def test_streamed_host_views(kind):
    dtype = torch.float16 if kind == "numpy_float16" else torch.bfloat16
    v = _views(8192, [40, 30], dtype, True, 5, device="cpu")
    host = [x.numpy() for x in v] if kind == "numpy_float16" else v
    est = rCCA(latent_dimensions=2, c=0.1)
    est._stream_threshold_bytes = 0
    est._stream_chunk_rows = 1000
    calls = []
    real = ops.moments

    def spy(views, precision="tf32x3b"):
        calls.append(views[0].dtype)
        return real(views, precision=precision)

    ops.moments = spy
    try:
        est.fit(host)
    finally:
        ops.moments = real
    assert calls and set(calls) == {dtype}, calls          # every chunk reached the kernel in its own dtype
    ref = rCCA(latent_dimensions=2, c=0.1).fit([x.double().numpy() for x in v])
    for a, b in zip(est.weights_, ref.weights_):
        np.testing.assert_array_equal(a, b)


def test_badly_centred_float16_view_takes_the_shift():
    g = torch.Generator(device="cuda").manual_seed(6)
    v = [(100.0 + torch.randn(20000, 24, generator=g, device="cuda")).half(),
         torch.randn(20000, 16, generator=g, device="cuda").half()]
    _, ratio = ops.column_pilot(v)
    assert ratio > ops.SHIFT_RATIO[torch.float16]
    mom, x0 = ops.moments_safe(v)
    assert x0 is not None and all(o.dtype == torch.float32 for o in x0)
    dims = [24, 16]
    C, _ = ops.covariance(mom, dims, 20000)
    X = torch.cat([x.double() for x in v], dim=1)
    ref = torch.cov(X.T)
    d = torch.diagonal(ref)
    # the float32 route's bound (tf32x3b, 5e-5 of sqrt(C_ii C_jj)) on the shifted float32 copy
    assert ((C - ref).abs() / torch.sqrt(d[:, None] * d[None, :])).max().item() < 5e-5


def test_fit_allocates_no_float64_copy():
    n, dims = 200000, [512, 512]
    v = _views(n, dims, torch.bfloat16, False, 7)
    est = rCCA(latent_dimensions=64, c=0.1)
    est.fit([x[:4096] for x in v])                           # warm-up: library load, caches
    torch.cuda.synchronize()
    torch.cuda.reset_peak_memory_stats()
    base = torch.cuda.memory_allocated()
    est.fit(v)
    torch.cuda.synchronize()
    extra = torch.cuda.max_memory_allocated() - base
    lib = _lib.load()
    ws = lib.ccab_moments_workspace_bytes(_lib.BF16, _lib.PREC_TF32X3B, 2, _lib.i64_array(dims), n) + 512
    D = sum(dims)
    inputs = sum(x.numel() * x.element_size() for x in v)
    assert extra <= ws + 32 * D * D * 8, (extra, ws)
    assert extra < 4 * inputs                               # a float64 copy of the views alone would be 4x


# --------------------------------------------------------------------------------------------- objectives
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


LOSSES = {
    "cca": lambda **k: CCALoss(**k),
    "cca_sync": lambda **k: CCALoss(verify="sync", **k),
    "mcca": lambda **k: MCCALoss(**k),
    "mcca_sync": lambda **k: MCCALoss(verify="sync", **k),
    "gcca": lambda **k: GCCALoss(**k),
}
# (batch, width of each view): tall batches on both sides of the exact / wgmma moment choice (total width 256), and a
# batch narrower than the width (eigen route)
OBJ_SHAPES = [(4096, 64), (4096, 512), (48, 64)]


@pytest.mark.parametrize("dtype", HALF)
@pytest.mark.parametrize("shape", OBJ_SHAPES)
@pytest.mark.parametrize("name", list(LOSSES))
def test_objectives_match_the_float32_route(name, shape, dtype):
    n, w = shape
    m = 3 if name.startswith("mcca") or name == "gcca" else 2
    zs = _reps(n, [w] * m, dtype, n + w)
    make = LOSSES[name]
    loss, grads = _loss_and_grads(make(eps=1e-3), zs)
    # MCCALoss(verify="sync") on float32 input is the per-pair CCALoss loop; 16-bit input runs the moment form (the
    # global-batch body), whose float32 route is the lazy MCCALoss: compare with that (the two float32 evaluations of
    # the same loss differ by ~4e-5 relative at these shapes)
    ref_make = LOSSES["mcca"] if name == "mcca_sync" else make
    z32 = [z.detach().float().requires_grad_() for z in zs]
    loss32, grads32 = _loss_and_grads(ref_make(eps=1e-3), z32)
    z64 = [z.detach().double().requires_grad_() for z in zs]
    _, grads64 = _loss_and_grads(ref_make(eps=1e-3), z64)
    assert loss.dtype == torch.float32
    assert abs(loss.item() - loss32.item()) <= 1e-5 * abs(loss32.item())
    for g, g32, g64 in zip(grads, grads32, grads64):
        assert g.dtype == dtype
        ref = g32.to(dtype).double()
        # one ulp of the rounded float32 gradient (entries below 1 % of the largest measured in the ulp at that level),
        # plus twice the float32 route's own error against float64: the gradient is a difference of terms that cancel,
        # so two float32 evaluations of it differ by about that much whatever the order of their sums
        floor = 1e-2 * ref.abs().max()
        tol = _ulp(torch.maximum(ref.abs(), floor), dtype) + 2 * (g32.double() - g64).abs().max()
        assert ((g.double() - ref).abs() <= tol).all(), (g.double() - ref).abs().max().item()


@pytest.mark.parametrize("dtype", HALF)
@pytest.mark.parametrize("name", ["cca", "mcca", "gcca"])
def test_mixed_16_and_32_bit_raise(name, dtype):
    zs = _reps(256, [8, 8], torch.float32, 0)
    mixed = [zs[0].detach().to(dtype), zs[1].detach()]
    with pytest.raises(ValueError):
        LOSSES[name]()(mixed)
    with pytest.raises(ValueError):
        LOSSES[name]()(mixed[::-1])


def test_autocast_encoder_trains_one_step():
    torch.manual_seed(0)
    enc = [torch.nn.Sequential(torch.nn.Linear(100, 128), torch.nn.ReLU(), torch.nn.Linear(128, 32)).cuda()
           for _ in range(2)]
    opt = torch.optim.SGD([p for e in enc for p in e.parameters()], lr=1e-3)
    x = [torch.randn(1024, 100, device="cuda") for _ in range(2)]
    loss_fn = CCALoss()
    with torch.autocast("cuda", dtype=torch.bfloat16):
        z = [e(xi) for e, xi in zip(enc, x)]
        assert z[0].dtype == torch.bfloat16
        loss = loss_fn(z)
    loss.backward()
    for e in enc:
        for p in e.parameters():
            assert p.grad is not None and torch.isfinite(p.grad).all()
    opt.step()
    loss_fn.check()
