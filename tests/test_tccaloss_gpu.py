"""TCCALoss on the GPU: loss and analytic gradients against the reference's float64 autograd (the goldens of
oracle/make_golden_tccaloss.py), the eigen route for rank-deficient batches and for verify='sync' failures, the lazy
status, NaN input, no host synchronisation in the lazy path, a training loop against a torch-eager restatement, and a
shape whose outer-product array the reference cannot hold, checked against the Gram form of oracle/tccaloss.py."""
import os

import numpy as np
import pytest
import torch

from oracle import tccaloss as O
from tests import tccaloss_golden as G

pytestmark = pytest.mark.gpu
DEV = "cpu" if os.environ.get("CCAB_TESTS_ON_STANDIN") else "cuda"


@pytest.mark.parametrize("name", sorted(G.CASES))
@pytest.mark.parametrize("dtype", [torch.float64, torch.float32])
def test_loss_and_gradients_match_reference(name, dtype):
    from cca_zoo_b200.deep import TCCALoss

    c = G.CASES[name]
    tol = G.tol64(name) if dtype == torch.float64 else 1e-3
    loss_ref, grads_ref = G.outputs(name)
    zs = [torch.from_numpy(z).to(dtype).to(DEV).requires_grad_(True) for z in G.inputs(name)]
    fn = TCCALoss(eps=c["eps"])
    loss = fn(zs)
    assert loss.dim() == 0 and loss.dtype == dtype
    loss.backward()
    fn.check()
    lerr = abs(loss.item() - loss_ref) / abs(loss_ref)
    gerr = G.rel_err([z.grad.double().cpu().numpy() for z in zs], grads_ref)
    print(f"{name} {dtype}: loss {lerr:.2e} grad {gerr:.2e} (tol {tol:.1e})")
    assert lerr <= (1e-12 if dtype == torch.float64 else tol) and gerr <= tol


def _duplicate_column_views():
    """S_1 = [[4, 4], [4, 4]] exactly (integer data, n - 1 = 16): at eps = 1e-17 its Cholesky pivot is exactly 0."""
    x = np.array([2.0] * 8 + [-2.0] * 8 + [0.0])
    rng = np.random.default_rng(3)
    return [torch.from_numpy(v).cuda() for v in (np.stack([x, x], 1), rng.standard_normal((17, 3)),
                                                  rng.standard_normal((17, 2)))]


def test_sync_takes_the_eigen_route_and_lazy_reports_at_the_next_call():
    from cca_zoo_b200.deep import TCCALoss

    zs = _duplicate_column_views()
    zs = [z.requires_grad_(True) for z in zs]
    loss = TCCALoss(eps=1e-17, verify="sync")(zs)
    loss.backward()
    want, gw, _ = O.eigen_form([z.detach().cpu().numpy() for z in zs], 1e-17)
    assert abs(loss.item() - want) <= 1e-6 * abs(want)
    assert all(torch.isfinite(z.grad).all() for z in zs)
    assert G.rel_err([z.grad.cpu().numpy() for z in zs[1:]], gw[1:]) <= 1e-6
    lazy = TCCALoss(eps=1e-17)
    lazy([z.detach() for z in zs])                      # returns: nothing is read back
    good = [torch.randn(40, 3, dtype=torch.float64, device="cuda") for _ in range(3)]
    torch.cuda.synchronize()
    with pytest.raises(RuntimeError, match="not numerically positive"):
        lazy(good)
    lazy(good)
    lazy.check()


def test_nan_input_raises_value_error():
    from cca_zoo_b200.deep import TCCALoss

    zs = [torch.randn(30, 3, dtype=torch.float64, device="cuda") for _ in range(3)]
    zs[1][1, 2] = float("nan")
    with pytest.raises(ValueError, match="NaN"):
        TCCALoss(verify="sync")(zs)
    fn = TCCALoss()
    fn(zs)
    with pytest.raises(ValueError, match="NaN"):
        fn.check()
    with pytest.raises(ValueError, match="NaN"):          # rank deficient by shape: the eigen route checks at once
        TCCALoss()([z[:3] for z in zs])


def test_no_host_sync_in_the_lazy_path():
    from cca_zoo_b200.deep import TCCALoss

    zs = [torch.randn(256, w, device="cuda", requires_grad=True) for w in (8, 5, 6)]
    fn = TCCALoss()
    fn(zs).backward()                                     # warm-up: pinned status buffers, library load
    fn.check()
    torch.cuda.set_sync_debug_mode("error")
    try:
        for _ in range(2):
            fn(zs).backward()
    finally:
        torch.cuda.set_sync_debug_mode("default")
    fn.check()


def _eager_loss(zs, eps):
    """The reference's formula in torch (eigh, clamp, outer products, norm) on the device, for autograd."""
    n = zs[0].shape[0]
    H = []
    for z in zs:
        zc = z - z.mean(0)
        S = zc.T @ zc / (n - 1) + eps * torch.eye(z.shape[1], dtype=z.dtype, device=z.device)
        lam, V = torch.linalg.eigh(S)
        H.append(zc @ (V @ torch.diag(lam.clamp(min=eps).rsqrt()) @ V.T))
    letters = "abcdefgh"[:len(H)]
    M = torch.einsum(",".join("z" + c for c in letters) + "->" + letters, *H) / n
    return -torch.linalg.norm(M.reshape(-1))


def test_training_loop_matches_eager_restatement():
    from cca_zoo_b200.deep import TCCALoss

    torch.manual_seed(0)
    zl = torch.randn(300, 2, dtype=torch.float64, device="cuda")
    xs = [zl @ torch.randn(2, d, dtype=torch.float64, device="cuda")
          + 0.3 * torch.randn(300, d, dtype=torch.float64, device="cuda") for d in (10, 12, 8)]
    init = [torch.nn.Linear(d, 4).double().cuda() for d in (10, 12, 8)]
    traj = {}
    for kind in ("device", "eager"):
        encs = [torch.nn.Linear(d, 4).double().cuda() for d in (10, 12, 8)]
        for e, e0 in zip(encs, init):
            e.load_state_dict(e0.state_dict())
        opt = torch.optim.Adam([p for e in encs for p in e.parameters()], lr=1e-2)
        fn = TCCALoss(eps=1e-6)
        out = []
        for _ in range(5):
            opt.zero_grad()
            zs = [e(x) for e, x in zip(encs, xs)]
            loss = fn(zs) if kind == "device" else _eager_loss(zs, 1e-6)
            loss.backward()
            opt.step()
            out.append(loss.item())
        traj[kind] = np.array(out)
    assert traj["device"][-1] < traj["device"][0]
    assert np.abs(traj["device"] - traj["eager"]).max() <= 1e-9 * np.abs(traj["eager"]).max()


def test_shape_the_reference_cannot_hold():
    """n = 4096 and four views of width 32: the reference's outer-product array would be 4096 x 32^4 doubles
    (34 GB).  The loss is checked against ||M|| from the sample Grams, and the gradient along a random direction
    against a central difference of the device loss."""
    from cca_zoo_b200.deep import TCCALoss

    rng = np.random.default_rng(11)
    n = 4096
    zl = rng.standard_normal((n, 2))
    zs = [zl @ rng.standard_normal((2, 32)) + rng.standard_normal((n, 32)) for _ in range(4)]
    eps = 1e-5
    H = []
    for z in zs:
        zc = z - z.mean(0)
        lam, V = np.linalg.eigh(zc.T @ zc / (n - 1) + eps * np.eye(32))
        H.append(zc @ (V / np.sqrt(np.maximum(lam, eps))) @ V.T)
    want = -O.gram_norm(H)
    zd = [torch.from_numpy(z).cuda().requires_grad_(True) for z in zs]
    fn = TCCALoss(eps=eps)
    loss = fn(zd)
    loss.backward()
    fn.check()
    assert abs(loss.item() - want) <= 1e-11 * abs(want)
    d = [torch.from_numpy(rng.standard_normal((n, 32))).cuda() for _ in range(4)]
    h = 1e-4
    with torch.no_grad():
        lp = fn([z + h * e for z, e in zip(zd, d)]).item()
        lm = fn([z - h * e for z, e in zip(zd, d)]).item()
    dd = sum(float((z.grad * e).sum()) for z, e in zip(zd, d))
    assert abs((lp - lm) / (2 * h) - dd) <= 1e-6 * abs(dd)
