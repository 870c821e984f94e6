"""Host-side logic of the estimators on CPU: the whole ``fit`` -- validation, moment pass, all-reduce, covariance
stage, solver routes and their fall-backs, PartialCCA / GRCCA algebra -- with tests/fake_ops.py (torch CPU, LAPACK)
standing in for the CUDA kernels.  What this checks is the PYTHON between the kernels, against the same reference
goldens the GPU tests use; the kernels themselves are checked by the ``-m gpu`` tests.
"""
import os
import socket

import numpy as np
import pytest
import torch
import torch.distributed as dist
import torch.multiprocessing as mp

from oracle import restatement as R
from tests import fake_ops
from tests import golden_io as G


@pytest.fixture
def host(monkeypatch):
    fake_ops.install(monkeypatch)


def _tol(case):
    return 2e-3 if case["dtype"] == "f32" and case["model"] in ("CCA", "rCCA", "PLS") else \
        (1e-5 if case["dtype"] == "f32" else 1e-8)


@pytest.mark.parametrize("solver", ["auto", "eigen", "cholesky"])
@pytest.mark.parametrize("name", sorted(G.CASES))
def test_estimators_through_host_logic(host, name, solver):
    from cca_zoo_b200 import linear

    case = G.CASES[name]
    views = G.case_inputs(name)
    w_ref, mu_ref, score_ref = G.case_outputs(name)
    kwargs = dict(case["kwargs"])
    if case["model"] not in ("CCA", "PLS"):
        kwargs["solver"] = solver
    elif solver != "auto":
        pytest.skip("CCA / PLS take no solver argument")
    est = getattr(linear, case["model"])(**kwargs).fit(views)
    err = R.max_rel_err_per_vector([w.astype(np.float64) for w in est.weights_], w_ref)
    assert err < _tol(case), f"{name}/{solver}: {err:.2e}"
    np.testing.assert_allclose(est.score(views), score_ref, rtol=max(_tol(case), 1e-7))
    assert est.n_samples_ == views[0].shape[0] and est.n_features_in_ == [v.shape[1] for v in views]


@pytest.mark.parametrize("name", sorted(G.PARTIAL_CASES))
def test_partialcca_through_host_logic(host, name):
    from cca_zoo_b200.linear import PartialCCA

    case = G.PARTIAL_CASES[name]
    views, Z = G.ext_inputs(name)
    ref = G.ext_outputs(name)
    est = PartialCCA(**case["kwargs"]).fit(views, partials=Z)
    tol = 1e-5 if case["dtype"] == "f32" else 1e-8
    assert R.max_rel_err_per_vector([w.astype(np.float64) for w in est.weights_], ref["w"]) < tol
    for b, br in zip(est.confound_betas_, ref["beta"]):
        np.testing.assert_allclose(b, br, rtol=1e-5, atol=1e-6 if case["dtype"] == "f32" else 1e-10)
    # row batches accumulate to the same model
    inc = PartialCCA(**case["kwargs"])
    n = views[0].shape[0]
    cut = n // 3
    inc.partial_fit([v[:cut] for v in views], partials=Z[:cut], solve=False)
    inc.partial_fit([v[cut:] for v in views], partials=Z[cut:])
    assert R.max_rel_err_per_vector(inc.weights_, est.weights_) < 1e-7


@pytest.mark.parametrize("name", sorted(G.GROUP_CASES))
def test_grcca_through_host_logic(host, name):
    from cca_zoo_b200.linear import GRCCA

    case = G.GROUP_CASES[name]
    views, groups = G.ext_inputs(name)
    ref = G.ext_outputs(name)
    est = GRCCA(**case["kwargs"]).fit(views, feature_groups=groups)
    tol = 1e-5 if case["dtype"] == "f32" else 1e-8
    assert R.max_rel_err_per_vector([w.astype(np.float64) for w in est.weights_], ref["w"]) < tol
    np.testing.assert_allclose(est.score(views), ref["score"], rtol=1e-6)


def _wide_views(n=3000, dims=(300, 280), k=6, seed=3, dtype=np.float64):
    rng = np.random.default_rng(seed)
    z = rng.standard_normal((n, k))
    return [(z @ rng.standard_normal((k, d)) * 0.4 + rng.standard_normal((n, d))).astype(dtype) for d in dims]


def test_device_fit_status_word_drives_retry_fallback_and_errors(host, monkeypatch):
    """The device-side fit reports through the header of its result block (csrc/fit.cu, include/ccab200.h): 'not
    converged' is answered by ONE more call with the larger iteration count, every other failure bit by the
    host-assembled routes, non-finite input by the reference's ValueError; ``weights_`` always match the oracle."""
    from cca_zoo_b200 import ops
    from cca_zoo_b200.linear import rCCA

    views = _wide_views()
    w_ref, _ = R.ref_rcca_fit(views, 4, 0.2)
    real = ops.rcca_fit
    seen = []

    def flaky(mom, dims, n_host, n_dev, center, c, k, p, iters, dtype):
        seen.append(iters)
        block, offsets = real(mom, dims, n_host, n_dev, center, c, k, p, iters, dtype)
        if len(seen) == 1:                                   # first attempt: pretend the tolerance was missed
            block.numpy()[:8].view(np.float64)[0] = ops.FIT_NOT_CONVERGED
        return block, offsets

    monkeypatch.setattr(ops, "rcca_fit", flaky)
    est = rCCA(latent_dimensions=4, c=0.2).fit(views)
    assert len(seen) == 2 and seen[1] > seen[0], seen
    assert est._fit_info["route"] == "device" and est._fit_info["iters"] == seen[1]
    assert R.max_rel_err_per_vector(est.weights_, w_ref) < 1e-8

    def declined(bit):
        def f(mom, dims, n_host, n_dev, center, c, k, p, iters, dtype):
            seen.append(iters)
            block, offsets = real(mom, dims, n_host, n_dev, center, c, k, p, iters, dtype)
            block.numpy()[:8].view(np.float64)[0] = bit
            return block, offsets
        return f

    for bit in (ops.FIT_NOT_POSITIVE_DEFINITE, ops.FIT_TOO_FEW_SAMPLES, ops.FIT_NOT_POSITIVE_DEFINITE | ops.FIT_NOT_CONVERGED):
        seen.clear()
        monkeypatch.setattr(ops, "rcca_fit", declined(bit))
        est = rCCA(latent_dimensions=4, c=0.2).fit(views)
        assert len(seen) == 1, "only a missed tolerance is worth a second device attempt"
        assert est._fit_info == {"route": "host", "device_status": bit}
        assert R.max_rel_err_per_vector(est.weights_, w_ref) < 1e-8
        assert est.n_samples_ == views[0].shape[0]

    monkeypatch.setattr(ops, "rcca_fit", declined(ops.FIT_NON_FINITE))
    with pytest.raises(ValueError, match="NaN or infinity"):
        rCCA(latent_dimensions=4, c=0.2).fit(views)


def test_parameter_validation_runs_once_per_parameter_set(host, monkeypatch):
    """sklearn's validation is a function of the constructor parameters alone: a re-fit with unchanged parameters skips
    it (pure host time in front of the first kernel), any change -- rebinding or in-place mutation -- repeats it, and an
    invalid value still raises at fit time as in the reference (cca_zoo/_base.py:88)."""
    from sklearn.base import BaseEstimator, clone
    from sklearn.utils._param_validation import InvalidParameterError

    from cca_zoo_b200.linear import rCCA

    calls = {"n": 0}
    real = BaseEstimator._validate_params

    def spy(self):
        calls["n"] += 1
        return real(self)

    monkeypatch.setattr(BaseEstimator, "_validate_params", spy)
    rng = np.random.default_rng(0)
    views = [rng.standard_normal((200, 10)), rng.standard_normal((200, 8))]
    est = rCCA(latent_dimensions=2, c=[0.1, 0.2])
    est.fit(views)
    est.fit(views)
    assert calls["n"] == 1
    est.c[0] = 0.3                                   # in-place mutation of a list parameter
    est.fit(views)
    assert calls["n"] == 2
    est.latent_dimensions = 0
    with pytest.raises(InvalidParameterError):
        est.fit(views)
    assert calls["n"] == 3
    est.latent_dimensions = 2                        # back to the last set that passed: nothing to re-check
    est.fit(views)
    assert calls["n"] == 3
    assert not hasattr(clone(est), "_validated_params_")      # a clone validates for itself
    clone(est).fit(views)
    assert calls["n"] == 4


def test_device_fit_plan_limits(host, monkeypatch):
    """When the one-call fit is taken (csrc/fit.cu needs p <= 128 for its single-CTA Ritz solve and 4k <= min d_i) and
    how the block width / first-try iteration count are chosen; the environment knobs are for experiments only."""
    from cca_zoo_b200.linear import MCCA, rCCA

    f32 = torch.float32
    plan = rCCA(latent_dimensions=64, c=0.1)._device_fit_plan([1024, 1024], 100000, f32)
    assert plan is not None and plan["k"] == 64 and plan["iters"] == [6, 20]
    assert rCCA(latent_dimensions=64, c=0.1, solver="eigen")._device_fit_plan([1024, 1024], 100000, f32) is None
    assert rCCA(latent_dimensions=64, c=0.1)._device_fit_plan([200, 1024], 100000, f32) is None      # narrow view
    assert rCCA(latent_dimensions=64, c=0.1)._device_fit_plan([1024, 1024], 900, f32) is None        # n <= d
    assert rCCA(latent_dimensions=120, c=0.1)._device_fit_plan([1024, 1024], 100000, f32) is None    # p would exceed 128
    assert rCCA(latent_dimensions=300, c=0.1)._device_fit_plan([1024, 1024], 100000, f32) is None    # 4k > min d
    monkeypatch.setenv("CCAB_FIT_OVERSAMPLE", "32")
    monkeypatch.setenv("CCAB_FIT_ITERS", "5")
    assert rCCA(latent_dimensions=64, c=0.1)._device_fit_plan([1024, 1024], 100000, f32)["iters"] == [5, 20]
    monkeypatch.delenv("CCAB_FIT_OVERSAMPLE")
    monkeypatch.delenv("CCAB_FIT_ITERS")
    assert MCCA(latent_dimensions=32, c=0.1)._device_fit_plan([512] * 4, 125000, f32) is not None
    assert MCCA(latent_dimensions=32, c=0.95)._device_fit_plan([512] * 4, 125000, f32) is None       # shift needs c <= 0.9
    # the float64 Ritz solve takes p <= 104: the plan asks the library with the SOLVE dtype and declines above it
    f64 = torch.float64
    assert rCCA(latent_dimensions=83, c=0.1)._device_fit_plan([400, 400], 5000, f64) is not None     # p = 103
    assert rCCA(latent_dimensions=84, c=0.1)._device_fit_plan([400, 400], 5000, f64) is None         # p = 105
    assert rCCA(latent_dimensions=84, c=0.1)._device_fit_plan([400, 400], 5000, f32) is not None     # float32: p <= 128
    assert rCCA(latent_dimensions=90, c=0.1)._device_fit_plan([400, 400], 5000, f64) is None         # p = 112
    for dt in (f32, f64):                                 # MCCA solves in float64 whatever the input dtype
        assert MCCA(latent_dimensions=52)._device_fit_plan([512] * 4, 20000, dt) is not None         # p = 104
        assert MCCA(latent_dimensions=53)._device_fit_plan([512] * 4, 20000, dt) is None             # p = 106
        assert MCCA(latent_dimensions=60)._device_fit_plan([512] * 4, 20000, dt) is None             # p = 120


def test_fit_workspace_query_answers_zero_exactly_where_the_fit_refuses():
    """ccab_rcca_fit_workspace_bytes / ccab_mcca_fit_workspace_bytes are the one owner of the fits' limits: the plans
    ask them (a pure host query, so the real library answers here too, also under the CPU stand-in)."""
    from cca_zoo_b200 import ops

    for dt, pmax in ((torch.float32, 128), (torch.float64, 104)):
        for dims, k, p in (([200, 150], 1, 1), ([200, 150], 5, 150), ([200, 150], 5, 151), ([200, 150], 6, 5),
                           ([200, 150], 0, 4), ([300, 300], 64, pmax), ([300, 300], 64, pmax + 1), ([40, 33], 33, 33)):
            want = 1 <= k <= p <= min(dims) and p <= pmax
            assert (ops.rcca_fit_workspace_bytes(dims, k, p, dt) > 0) == want, (dt, dims, k, p)
        for dims, k, p in (([64, 64], 4, 64), ([65, 1], 4, 66), ([65, 1], 4, 67), ([300] * 8, 8, pmax),
                           ([300] * 8, 8, pmax + 1), ([300], 4, 8), ([300, 300], 9, 8)):
            want = len(dims) >= 2 and 1 <= k <= p <= sum(dims) and p <= pmax
            assert (ops.mcca_fit_workspace_bytes(dims, k, p, dt) > 0) == want, (dt, dims, k, p)


def test_cholesky_and_eigen_routes_agree_on_wide_views(host):
    """min(dims) >= 256 and n > max(dims): ``auto`` takes the device-side fit (one library call); when that is not
    available the host-assembled Cholesky + subspace-iteration route; both agree with the eigen route."""
    from cca_zoo_b200 import _solvers
    from cca_zoo_b200.linear import MCCA, GCCA, rCCA

    views = _wide_views()
    w_ref, _ = R.ref_rcca_fit(views, 4, 0.2)
    auto = rCCA(latent_dimensions=4, c=0.2).fit(views)
    assert auto._fit_info["route"] == "device"
    calls = {"n": 0}
    real = _solvers.topk_svd

    def spy(*a, **kw):
        calls["n"] += 1
        return real(*a, **kw)

    _solvers.topk_svd, keep = spy, real
    plan, rCCA._device_fit_plan = rCCA._device_fit_plan, lambda self, *a: None
    try:
        hosted = rCCA(latent_dimensions=4, c=0.2).fit(views)
    finally:
        _solvers.topk_svd = keep
        rCCA._device_fit_plan = plan
    assert calls["n"] == 1, "without the device-side fit, auto must take the host-assembled top-k route here"
    assert R.max_rel_err_per_vector(hosted.weights_, w_ref) < 1e-8
    eig = rCCA(latent_dimensions=4, c=0.2, solver="eigen").fit(views)
    assert R.max_rel_err_per_vector(auto.weights_, w_ref) < 1e-8
    assert R.max_rel_err_per_vector(eig.weights_, w_ref) < 1e-8
    three = views + [_wide_views(seed=4)[0][:, :260]]
    for cls, ref in ((MCCA, R.ref_mcca_fit(three, 3, 0.1)[0]), (GCCA, None)):
        a = cls(latent_dimensions=3, c=0.1, solver="cholesky").fit(three)
        e = cls(latent_dimensions=3, c=0.1, solver="eigen").fit(three)
        assert R.max_rel_err_per_vector(a.weights_, e.weights_) < 1e-7
        if ref is not None:
            assert R.max_rel_err_per_vector(a.weights_, ref) < 1e-7


def test_cholesky_route_declines_on_a_singular_block_and_the_eigen_route_drops_the_null_directions(host):
    """Three duplicated columns make a block exactly singular: potrf reports it, the eigen route takes over and
    drops the numerically null directions (lambda <= d eps lambda_max, the covariance-space image of the
    reference's ``s > 0`` filter).  The canonical correlations then equal those of the views WITHOUT the
    duplicates (same column space).  The reference itself keeps singular values of 1e-14 in this corner
    (``s > 0`` is true for them), which yields weights of 1e13 and correlations that are off by 8e-4 -- the
    oracle's literal restatement reproduces that artefact, its covariance form does not."""
    from cca_zoo_b200.linear import rCCA

    views = _wide_views()
    w_true, mu_true = R.ref_rcca_fit(views, 3, 0.0)
    truth = R.score(views, mu_true, w_true)
    dup = [np.hstack([views[0], views[0][:, :3]]), views[1]]
    for solver in ("cholesky", "eigen"):
        est = rCCA(latent_dimensions=3, c=0.0, solver=solver).fit(dup)
        np.testing.assert_allclose(est.score(dup), truth, rtol=1e-7)
        assert np.abs(est.weights_[0]).max() < 1e3
    M, s, n = R.moments(dup)
    w_cov, _ = R.cov_rcca_fit(R.covariance_from_moments(M, s, n), [303, 280], 3, 0.0, n)
    np.testing.assert_allclose(R.score(dup, [v.mean(axis=0) for v in dup], w_cov), truth, rtol=1e-7)


def test_dense_route_is_refused_beyond_its_size_limit(host, monkeypatch):
    from cca_zoo_b200 import _solvers
    from cca_zoo_b200.linear import MCCA

    monkeypatch.setattr(_solvers, "_MAX_DENSE_JACOBI", 256)
    views = _wide_views(n=900, dims=(200, 180))
    MCCA(latent_dimensions=2, c=0.1, solver="eigen").fit([v[:, :100] for v in views])   # D = 200: allowed
    with pytest.raises(RuntimeError, match="dense Jacobi route is limited"):
        MCCA(latent_dimensions=120, c=0.1).fit(views)                                    # 4k > D: top-k declines


def test_validation_errors_match_the_reference_messages(host):
    from sklearn.exceptions import NotFittedError
    from sklearn.utils._param_validation import InvalidParameterError

    from cca_zoo_b200.linear import MCCA, rCCA

    v = _wide_views(n=50, dims=(6, 5))
    with pytest.raises(ValueError, match="exactly 2 views"):
        rCCA().fit(v + [v[0]])
    with pytest.raises(ValueError, match="same number of samples"):
        MCCA().fit([v[0], v[1][:-1]])
    with pytest.raises(ValueError, match="At least 2 views"):
        MCCA().fit(v[:1])
    with pytest.raises(InvalidParameterError):
        rCCA(c=1.5).fit(v)
    with pytest.raises(InvalidParameterError):
        MCCA(latent_dimensions=0).fit(v)
    with pytest.raises(NotFittedError):
        rCCA().transform(v)
    bad = [v[0].copy(), v[1]]
    bad[0][3, 2] = np.nan
    with pytest.raises(ValueError, match="NaN"):
        rCCA().fit(bad)


# ------------------------------------------------------------------------------------------------------------
# N > 1: the whole sharded fit (row shards -> moments -> ONE all-reduce -> replicated solve), gloo, world 2
# ------------------------------------------------------------------------------------------------------------
def _free_port():
    s = socket.socket()
    s.bind(("127.0.0.1", 0))
    port = s.getsockname()[1]
    s.close()
    return port


def _sharded_fit_worker(rank, world, port, out_dir):
    os.environ.update(MASTER_ADDR="127.0.0.1", MASTER_PORT=str(port), RANK=str(rank), WORLD_SIZE=str(world))
    dist.init_process_group("gloo", rank=rank, world_size=world)
    try:
        mpatch = pytest.MonkeyPatch()
        fake_ops.install(mpatch)
        from cca_zoo_b200 import parallel
        from cca_zoo_b200.linear import MCCA, PartialCCA, rCCA

        views = G.dataset("joint3_med")
        Z = np.random.default_rng(9).standard_normal((views[0].shape[0], 3)) + 0.4
        lo, hi = parallel.shard_rows(views[0].shape[0], rank, world)
        shard = [v[lo:hi] for v in views]
        out = {}
        out["rcca"] = rCCA(latent_dimensions=4, c=0.1).fit(shard[:2]).weights_
        m = MCCA(latent_dimensions=3, c=0.05).fit(shard)
        out["mcca"], out["mcca_n"] = m.weights_, np.array([m.n_samples_])
        p = PartialCCA(latent_dimensions=3, c=0.05).fit(shard, partials=Z[lo:hi])
        out["pcca"], out["pcca_beta"] = p.weights_, p.confound_betas_
        np.savez(os.path.join(out_dir, f"rank{rank}.npz"),
                 **{f"{k}{i}": a for k, v in out.items() for i, a in enumerate(v)})
        mpatch.undo()
    finally:
        dist.destroy_process_group()


def test_sharded_fit_world2_equals_single_process_fit(tmp_path, host):
    world = 2
    mp.spawn(_sharded_fit_worker, args=(world, _free_port(), str(tmp_path)), nprocs=world, join=True)
    r0, r1 = np.load(tmp_path / "rank0.npz"), np.load(tmp_path / "rank1.npz")
    for key in r0.files:
        assert np.array_equal(r0[key], r1[key]), f"{key}: replicated solve must be bit-identical on every rank"
    views = G.dataset("joint3_med")
    Z = np.random.default_rng(9).standard_normal((views[0].shape[0], 3)) + 0.4
    assert int(r0["mcca_n0"]) == views[0].shape[0]
    w, _ = R.ref_rcca_fit(views[:2], 4, 0.1)
    assert R.max_rel_err_per_vector([r0["rcca0"], r0["rcca1"]], w) < 1e-8
    w, _ = R.ref_mcca_fit(views, 3, 0.05)
    assert R.max_rel_err_per_vector([r0[f"mcca{i}"] for i in range(3)], w) < 1e-8
    w, _, betas = R.ref_partialcca_fit(views, Z, 3, 0.05)
    assert R.max_rel_err_per_vector([r0[f"pcca{i}"] for i in range(3)], w) < 1e-8
    for i, b in enumerate(betas):
        np.testing.assert_allclose(r0[f"pcca_beta{i}"], b, atol=1e-10)


@pytest.mark.parametrize("name", sorted(G.CENTER_CASES))
def test_center_false_semantics_through_host_logic(host, name):
    """np.cov centres inside MCCA / GCCA / GRCCA whatever ``center`` says; GCCA mixes in raw second moments; a
    ridge keeps the null directions of a rank-deficient view (goldens: oracle/make_golden_ext.py CENTER_CASES)."""
    from cca_zoo_b200 import linear

    case = G.CENTER_CASES[name]
    views, _ = G.ext_inputs(name)
    ref = G.ext_outputs(name)
    est = getattr(linear, case["model"])(**case["kwargs"]).fit(views)
    assert [w.shape for w in est.weights_] == [w.shape for w in ref["w"]]
    kk = 8 if name == "rcca_dup_ridge" else est.weights_[0].shape[1]
    tol = 1e-5 if case["dtype"] == "f32" else 1e-7
    assert R.max_rel_err_per_vector([w[:, :kk].astype(np.float64) for w in est.weights_],
                                    [w[:, :kk] for w in ref["w"]]) < tol
    np.testing.assert_allclose(est.score(views)[:kk], ref["score"][:kk], rtol=1e-5, atol=1e-8)
    if not case["kwargs"].get("center", True):
        assert all(np.all(mu == 0) for mu in est.means_)


def test_center_false_routes_agree_on_wide_views(host):
    from cca_zoo_b200.linear import GCCA, GRCCA, MCCA

    views = [v + 0.7 for v in _wide_views()] + [_wide_views(seed=4)[0][:, :260] - 0.3]
    w_m, _ = R.ref_mcca_fit(views, 3, 0.1, center=False)
    w_g, _ = R.ref_gcca_fit(views, 3, 0.1, center=False)
    groups = [np.random.default_rng(i).integers(0, 9, size=v.shape[1]) for i, v in enumerate(views)]
    w_r, _ = R.ref_grcca_fit(views, groups, 3, 0.3, 0.5, center=False)
    for solver in ("cholesky", "eigen"):
        assert R.max_rel_err_per_vector(MCCA(latent_dimensions=3, c=0.1, center=False, solver=solver)
                                        .fit(views).weights_, w_m) < 1e-7
        assert R.max_rel_err_per_vector(GCCA(latent_dimensions=3, c=0.1, center=False, solver=solver)
                                        .fit(views).weights_, w_g) < 1e-7
        assert R.max_rel_err_per_vector(GRCCA(latent_dimensions=3, c=0.3, mu=0.5, center=False, solver=solver)
                                        .fit(views, feature_groups=groups).weights_, w_r) < 1e-7


@pytest.mark.parametrize("name", sorted(G.LOSS_CASES) + sorted(G.GLOSS_CASES))
def test_objectives_through_host_logic(host, name):
    """Route selection and the analytic backward of CCALoss / MCCALoss / GCCALoss against the reference's forward
    value and autograd gradients (goldens), with the stand-in kernels."""
    from cca_zoo_b200.deep import CCALoss, GCCALoss, MCCALoss

    c = G.LOSS_CASES.get(name) or G.GLOSS_CASES[name]
    loss_ref, grads_ref = G.loss_outputs(name)
    zs = [z.clone().requires_grad_(True) for z in G.loss_inputs(name)]
    fn = {"cca": CCALoss, "mcca": MCCALoss}.get(c.get("kind"), GCCALoss)(eps=c["eps"])
    loss = fn(zs)
    assert loss.dim() == 0 and abs(loss.item() - loss_ref) < 1e-9 * abs(loss_ref)
    loss.backward()
    for z, gr in zip(zs, grads_ref):
        assert np.abs(z.grad.numpy() - gr).max() < 1e-7 * np.abs(gr).max()


def test_objectives_reject_cpu_tensors_without_the_standin():
    from cca_zoo_b200.deep import CCALoss, GCCALoss

    z = [torch.randn(8, 3), torch.randn(8, 3)]
    for fn in (CCALoss(), GCCALoss()):
        with pytest.raises(RuntimeError, match="CUDA"):
            fn(z)


def test_device_score_path_equals_the_reference_definition(host, monkeypatch):
    """pairwise correlations from ONE moment pass (W_i^T C_ij W_j normalised) == Pearson correlations of the
    transformed samples (cca_zoo/_base.py:153-174), on held-out rows, for 2 and 3 views."""
    from cca_zoo_b200._base import BaseModel
    from cca_zoo_b200.linear import MCCA, rCCA

    views = G.dataset("joint3_med")
    train = [v[:1500] for v in views]
    held = [v[1500:] for v in views]
    for est in (rCCA(latent_dimensions=4, c=0.1).fit(train[:2]), MCCA(latent_dimensions=3, c=0.05).fit(train)):
        hv = held[: est.n_views_]
        host_path = est.pairwise_correlations(hv)
        monkeypatch.setattr(BaseModel, "_device_score_threshold", 0)
        monkeypatch.setattr(torch.cuda, "is_available", lambda: True)
        dev_path = est.pairwise_correlations(hv)
        monkeypatch.undo()
        fake_ops.install(monkeypatch)
        np.testing.assert_allclose(dev_path, host_path, atol=1e-10)
        np.testing.assert_allclose(dev_path, R.pairwise_correlations(R.transform(hv, est.means_, est.weights_)),
                                   atol=1e-10)


def test_partial_fit_batches_and_torch_inputs_equal_one_fit(host):
    from cca_zoo_b200.linear import GCCA, MCCA, rCCA

    views = G.dataset("joint3_med")
    for cls, kw, nv in ((rCCA, dict(c=0.1), 2), (MCCA, dict(c=0.05), 3), (GCCA, dict(c=0.1), 3)):
        one = cls(latent_dimensions=3, **kw).fit(views[:nv])
        inc = cls(latent_dimensions=3, **kw)
        cuts = [0, 700, 1500, 2500]
        for a, b in zip(cuts[:-1], cuts[1:]):
            inc.partial_fit([v[a:b] for v in views[:nv]], solve=b == cuts[-1])
        assert R.max_rel_err_per_vector(inc.weights_, one.weights_) < 1e-9
        assert inc.n_samples_ == 2500
        tt = cls(latent_dimensions=3, **kw).fit([torch.from_numpy(v) for v in views[:nv]])
        assert R.max_rel_err_per_vector(tt.weights_, one.weights_) < 1e-12
        with pytest.raises(ValueError, match="keep the view widths"):
            inc.partial_fit([v[:10, :5] for v in views[:nv]])
