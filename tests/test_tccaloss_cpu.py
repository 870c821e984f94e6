"""TCCALoss without a GPU: the float64 restatement (oracle/tccaloss.py) against the reference's goldens in both
whitenings, the two gradient forms against each other, the invariance of the loss under the choice of whitener, the
Gram form of ||M||, and the host logic of ``cca_zoo_b200.deep.TCCALoss`` on the torch stand-in
(tests/fake_ops_tccaloss.py): route choice, argument errors and the status flags."""
import numpy as np
import pytest
import torch

from oracle import tccaloss as O
from tests import tccaloss_golden as G

FULL_RANK = sorted(n for n, c in G.CASES.items() if c["n"] - 1 >= max(c["widths"]))


@pytest.mark.parametrize("name", sorted(G.CASES))
def test_oracle_matches_reference(name):
    zs, eps = G.inputs(name), G.CASES[name]["eps"]
    loss_ref, grads_ref = G.outputs(name)
    forms = [O.eigen_form] + ([O.chol_form] if name in FULL_RANK else [])
    for form in forms:
        loss, grads, _ = form(zs, eps)
        assert abs(loss - loss_ref) <= 1e-12 * abs(loss_ref)
        assert G.rel_err(grads, grads_ref) <= G.tol64(name), form.__name__


def test_golden_covers_the_issue_cases():
    ms = {len(c["widths"]) for c in G.CASES.values()}
    assert {2, 3, 4, 5, 8} <= ms
    assert any(1 in c["widths"] for c in G.CASES.values())
    assert {c["eps"] for c in G.CASES.values()} == {1e-5, 1e-6}
    assert any(c["n"] - 1 < max(c["widths"]) for c in G.CASES.values())
    assert any(max(c["widths"]) > 64 for c in G.CASES.values())


@pytest.mark.parametrize("name", FULL_RANK)
def test_gradient_forms_agree(name):
    zs, eps = G.inputs(name), G.CASES[name]["eps"]
    lc, gc, ic = O.chol_form(zs, eps)
    le, ge, ie = O.eigen_form(zs, eps)
    assert abs(lc - le) <= 1e-13 * abs(le)
    assert G.rel_err(gc, ge) <= 1e-12
    assert abs(O.gram_norm(ic["H"]) + lc) <= 1e-13 * abs(lc)


def test_loss_is_invariant_under_the_whitener():
    """Swapping R_i = L_i^-T for S_i^-1/2 (or any R_i Q_i, Q_i orthogonal) leaves ||M|| unchanged."""
    zs, eps = G.inputs("m3"), G.CASES["m3"]["eps"]
    _, _, ic = O.chol_form(zs, eps)
    _, _, ie = O.eigen_form(zs, eps)
    rng = np.random.default_rng(0)
    Q = [np.linalg.qr(rng.standard_normal((h.shape[1],) * 2))[0] for h in ic["H"]]
    norms = [np.linalg.norm(O.moment(H)) for H in (ic["H"], ie["H"], [h @ q for h, q in zip(ic["H"], Q)])]
    assert max(norms) - min(norms) <= 1e-13 * norms[0]


def test_adjoint_is_the_gradient_of_the_squared_norm():
    """<Y_i, dH_i> / n = d(||M||^2 / 2) along dH_i: the contract of ccab_tcca_moment_adjoint at f = 1/n."""
    rng = np.random.default_rng(1)
    H = [rng.standard_normal((9, p)) for p in (3, 1, 4)]
    M = O.moment(H)
    Y = O.adjoint(M, H)
    for i in range(3):
        d = rng.standard_normal(H[i].shape)
        h = 1e-6
        Hp = [x + h * d if j == i else x for j, x in enumerate(H)]
        Hm = [x - h * d if j == i else x for j, x in enumerate(H)]
        fd = (np.sum(O.moment(Hp) ** 2) - np.sum(O.moment(Hm) ** 2)) / (4 * h)
        assert abs(fd - np.sum(Y[i] * d) / 9) <= 1e-7 * abs(fd)


# ------------------------------------------------------------------ host logic on the stand-in
@pytest.fixture
def standin(monkeypatch):
    from tests import fake_ops, fake_ops_tccaloss

    fake_ops_tccaloss.install(monkeypatch)
    calls = {"syevj": 0, "potrf_inv_": 0}
    for name in calls:
        real = getattr(fake_ops, name)

        def wrap(*a, _real=real, _name=name, **k):
            calls[_name] += 1
            return _real(*a, **k)

        monkeypatch.setattr(fake_ops, name, wrap)
    return calls, fake_ops_tccaloss.CALLS


@pytest.mark.parametrize("name", sorted(G.CASES))
def test_standin_matches_reference(standin, name):
    from cca_zoo_b200.deep import TCCALoss

    calls, kcalls = standin
    c = G.CASES[name]
    loss_ref, grads_ref = G.outputs(name)
    zs = [torch.from_numpy(z).requires_grad_(True) for z in G.inputs(name)]
    loss = TCCALoss(eps=c["eps"])(zs)
    loss.backward()
    assert loss.dim() == 0 and loss.dtype == torch.float64
    assert abs(loss.item() - loss_ref) <= 1e-12 * abs(loss_ref)
    assert G.rel_err([z.grad.numpy() for z in zs], grads_ref) <= G.tol64(name)
    eigen = c["n"] - 1 < max(c["widths"])
    assert (calls["syevj"] > 0) == eigen and (calls["potrf_inv_"] > 0) != eigen
    assert kcalls == {"moment": 1, "adjoint": 1}


def _duplicate_column_views():
    """A view whose two columns are equal, with integer data and n - 1 = 16: S = [[4, 4], [4, 4]] exactly, so at
    eps = 1e-17 (below the rounding of 4) its Cholesky factorisation meets an exactly zero pivot."""
    x = np.array([2.0] * 8 + [-2.0] * 8 + [0.0])
    rng = np.random.default_rng(3)
    return [np.stack([x, x], 1), rng.standard_normal((17, 3)), rng.standard_normal((17, 2))]


def test_standin_status_and_sync_route(standin):
    from cca_zoo_b200.deep import TCCALoss

    calls, _ = standin
    zs = [torch.from_numpy(z) for z in _duplicate_column_views()]
    with pytest.raises(RuntimeError, match="not numerically positive"):
        TCCALoss(eps=1e-17)(zs)              # on the stand-in the status is inspected at once
    loss = TCCALoss(eps=1e-17, verify="sync")(zs)
    assert calls["syevj"] == 3 and np.isfinite(loss.item())
    bad = [z.clone() for z in zs]
    bad[1][0, 0] = float("nan")
    for verify in ("lazy", "sync"):
        with pytest.raises(ValueError, match="NaN"):
            TCCALoss(verify=verify)(bad)


@pytest.mark.parametrize("widths,n,match", [
    ([3], 10, "2 to 8"), ([2] * 9, 10, "2 to 8"), ([3, 4], 1, "at least 2 samples"),
    ([32] * 5 + [2], 4, "2\\^25"), ([8193, 4096], 2, "2\\^25"),
])
def test_argument_errors_before_any_call(standin, widths, n, match):
    from cca_zoo_b200.deep import TCCALoss

    calls, kcalls = standin
    zs = [torch.zeros(n, w, dtype=torch.float64) for w in widths]
    with pytest.raises(ValueError, match=match):
        TCCALoss()(zs)
    assert calls == {"syevj": 0, "potrf_inv_": 0} and kcalls == {"moment": 0, "adjoint": 0}


def test_verify_argument():
    from cca_zoo_b200.deep import TCCALoss

    with pytest.raises(ValueError, match="verify"):
        TCCALoss(verify="never")
