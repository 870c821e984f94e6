"""The GFA kernel (ccab_gfa_fit through ``ops.gfa_fit``) against its float64 step restatement
(oracle/gfa.py:gram_step), state by state: after 1, 2 and 40 iterations, at k = 1 and k = 64, on 8 ragged views, at
a width where the grid-stride loops wrap, across prunes, with the stop flag set; plus chunk invariance and reruns bit
for bit."""
import numpy as np
import pytest
import torch

from cca_zoo_b200 import ops
from cca_zoo_b200.datasets import joint_data
from oracle import gfa as O

pytestmark = pytest.mark.gpu

FIELDS = ("W", "B", "GB", "cov_z", "zz", "alpha", "b_ard", "cov_w", "ww", "tau", "b_tau")


def _problem(dims, k, seed, latent=2, n=400):
    views = joint_data(n_views=len(dims), n_samples=n, n_features=list(dims), latent_dimensions=latent,
                       signal_to_noise=2.0, random_state=seed)
    G, n, dims, Xz0, zz0, dv = O.gram_inputs(views, k)
    return G, n, dims, Xz0, zz0, dv, O.y_constants(G, dims)


def _device_fit(p, tol, drop_k=True):
    G, n, dims, Xz0, zz0, dv, yc = p
    dev = torch.device("cuda")
    return ops.gfa_fit(dims, torch.from_numpy(G).to(dev), n, torch.from_numpy(Xz0).to(dev), zz0, dv, yc, tol,
                       drop_k=drop_k)


def _oracle(p, steps, tol, drop_k=True):
    G, n, dims, Xz0, zz0, dv, yc = p
    st = O.gram_state(n, dims, Xz0.shape[1], zz0, dv, yc)
    for _ in range(steps):
        O.gram_step(st, G, Xz0, tol, drop_k)
    return st


def _compare(dev, ref, tol=1e-12):
    assert dev["iters"] == ref["iters"] and dev["k"] == ref["k"] and dev["stable"] == ref["stable"]
    assert dev["stop"] == ref["stop"]
    assert np.array_equal(dev["index"], ref["index"])
    for f in FIELDS:
        a, b = np.asarray(dev[f]), np.asarray(ref[f])
        assert a.shape == b.shape, f
        err = float(np.abs(a - b).max()) / max(float(np.abs(b).max()), 1e-300)
        assert err < tol, f"{f}: {err:.2e}"


@pytest.mark.parametrize("dims,k,seed", [((10, 8), 1, 0), ((10, 8), 4, 3), ((30, 40), 64, 1),
                                         ((5, 9, 3, 7, 11, 4, 6, 8), 3, 2), ((1500, 1800, 1200), 5, 4)])
@pytest.mark.parametrize("steps", [1, 2, 40])
def test_gfa_kernel_matches_the_step_restatement(dims, k, seed, steps):
    p = _problem(dims, k, seed)
    fit = _device_fit(p, 1e-4)
    fit.run(steps)
    _compare(fit.result(), _oracle(p, steps, 1e-4))


def test_gfa_kernel_prunes_inside_a_chunk_several_times():
    p = _problem((10, 8), 8, 3)
    ref = _oracle(p, 40, 1e-4)
    assert ref["k"] == 4                      # prunes 8 -> 7 -> 6 -> 4 in iterations 7, 11, 15
    fit = _device_fit(p, 1e-4)
    fit.run(40)
    res = fit.result()
    assert res["prunes"] == 3
    _compare(res, ref)


def test_gfa_kernel_without_drop_k_keeps_every_column():
    p = _problem((10, 8), 8, 3)
    fit = _device_fit(p, 1e-4, drop_k=False)
    fit.run(40)
    res = fit.result()
    assert res["k"] == 8
    _compare(res, _oracle(p, 40, 1e-4, drop_k=False))


def test_gfa_kernel_stop_flag_freezes_the_state():
    p = _problem((10, 8), 2, 5)
    ref = _oracle(p, 3000, 1e-2)
    assert ref["stop"] and ref["iters"] < 3000
    fit = _device_fit(p, 1e-2)
    fit.run(3000)
    res = fit.result()
    _compare(res, ref, tol=1e-10)
    frozen = fit.state.clone()
    fit.run(50)
    assert fit.stopped()
    assert torch.equal(fit.state, frozen)


def test_gfa_kernel_chunks_and_reruns_are_bit_identical():
    p = _problem((10, 8), 8, 3)
    a, b, c = _device_fit(p, 1e-4), _device_fit(p, 1e-4), _device_fit(p, 1e-4)
    a.run(12)
    b.run(5)
    b.run(7)
    c.run(12)
    assert torch.equal(a.state, b.state)
    assert torch.equal(a.state, c.state)
    for split in ((1, 1, 1, 37), (20, 20)):
        d = _device_fit(p, 1e-4)
        for s in split:
            d.run(s)
        e = _device_fit(p, 1e-4)
        e.run(40)
        assert torch.equal(d.state, e.state)


def test_gfa_kernel_rejects_k_above_64():
    p = _problem((30, 40), 65, 0)
    with pytest.raises(ValueError, match="1 <= k <= 64"):
        _device_fit(p, 1e-4)
