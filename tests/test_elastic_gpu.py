"""GPU tests of ElasticCCA / SCCA_IPLS (the regression kinds of ccab_als_fit): parity with the Gram-space restatement
(oracle/elastic.py:cov_elastic_fit) on the device's own covariance, with the reference's golden vectors where the
sub-problems have unique minimisers, the alpha = 0 degenerate cases, an independent KKT check, the reference's own
assertions and the invariants of the ALS family."""
import json
import os
import socket

import numpy as np
import pytest
import torch

from cca_zoo_b200.datasets import conftest_views, joint_data
from oracle import elastic as E

pytestmark = pytest.mark.gpu

_DIR = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden")
with open(os.path.join(_DIR, "reference_outputs_elastic.json")) as _f:
    META = json.load(_f)
NPZ = np.load(os.path.join(_DIR, "reference_outputs_elastic.npz"))
CASES = {c["name"]: c for c in META["cases"]}


def _cls(kind):
    from cca_zoo_b200 import linear

    return linear.ElasticCCA if kind == "elastic" else linear.SCCA_IPLS


def _views(case):
    kind, args = META["datasets"][case["dataset"]]
    if kind == "joint":
        return joint_data(**args)
    return [v[:args.get("rows")] for v in conftest_views(args["name"])]


def _golden(name):
    ws, i = [], 0
    while f"{name}/w{i}" in NPZ:
        ws.append(NPZ[f"{name}/w{i}"])
        i += 1
    return ws


def _spread_tol(case, d):
    return max(1e-6, 10.0 * max(max(s[:d + 1]) for s in case["spread"]))


def _restate(est, views, **kw):
    """cov_elastic_fit on the Gram matrix of the covariance the estimator computed on the device."""
    C, dims, n = est._fit_device(views)
    G = C.to(torch.float64).cpu().numpy() * (n - 1)
    means = est._column_means if est._kind == "ipls" and not est.center else None
    flat = est._regression_params(len(dims))
    return E.cov_elastic_fit(G, dims, n, est._kind, est.latent_dimensions, params=list(zip(flat[::2], flat[1::2])),
                             colmeans=means, max_iter=est.max_iter, tol=est.tol, random_state=est.random_state, **kw)


def _deflated(views, W, center):
    """The reference's deflated views before each dimension (cca_zoo/_utils/_linalg.py:91-116)."""
    Xs = [np.asarray(v, np.float64) - (np.asarray(v).mean(axis=0) if center else 0.0) for v in views]
    out = []
    for d in range(W[0].shape[1]):
        out.append([x.copy() for x in Xs])
        for i, x in enumerate(Xs):
            t = x @ W[i][:, d]
            s = float(t @ t)
            if s > 1e-12:
                Xs[i] = x - np.outer(t, t @ x) / s
    return out


@pytest.mark.parametrize("name", sorted(CASES))
def test_elastic_matches_restatement_and_reference(name):
    case = CASES[name]
    views = _views(case)
    est = _cls(case["model"])(**case["kwargs"])
    W_ref, iters_ref, deltas = _restate(est, views, return_info=True)
    est.fit(views)
    tol = case["kwargs"]["tol"]
    if min(abs(x - tol) for dl in deltas for x in dl) > 1e-3 * tol:
        assert est._fit_info["iters"] == iters_ref
    short = views[0].shape[0] <= max(v.shape[1] for v in views)
    for w, r in zip(est.weights_, W_ref):
        assert w.dtype == np.float64 and np.all(np.isfinite(w))
        err = float(np.abs(w - r).max())
        assert err < (1e-8 if short else 1e-9) * max(1.0, float(np.abs(r).max())), f"restatement differs by {err:.2e}"
    if case["spread"] is None:
        return
    for i, (w, g, v) in enumerate(zip(est.weights_, _golden(name), views)):
        a, l1 = case["params"][i]
        unique = a * (1.0 - l1) > 0.0
        for d in range(w.shape[1]):
            if unique or (d == 0 and v.shape[0] - 1 > v.shape[1]):
                assert float(np.abs(w[:, d] - g[:, d]).max()) <= _spread_tol(case, d), (i, d)


@pytest.mark.parametrize("name", sorted(n for n, c in CASES.items() if c["setting"] == "default"))
def test_alpha_zero_scores_and_minimum_norm(name):
    """alpha = 0: from dimension 2 on (and for n <= d_i from the first) G_ii is singular.  The weights are the
    minimum-norm ones in every dimension.  Where the reference converged (from dimension 2 on, n > d_i), the scores of
    the deflated views and the weights with the null space projected out match it.  For n <= d_i the reference's
    coordinate descent does not converge (its tight run raises ConvergenceWarning), so nothing is compared with it."""
    case = CASES[name]
    views = _views(case)
    est = _cls(case["model"])(**case["kwargs"]).fit(views)
    ref = _golden(name)
    center = case["kwargs"]["center"]
    ours, theirs = _deflated(views, est.weights_, center), _deflated(views, ref, center)
    for d in range(est.weights_[0].shape[1]):
        for i in range(len(views)):
            # minimum norm: no component in the null space of the view as deflated by this fit's own weights
            w = est.weights_[i][:, d]
            U, sv, Vt = np.linalg.svd(ours[d][i], full_matrices=False)
            R = Vt[sv > 1e-10 * sv[0]]
            assert np.linalg.norm(w - R.T @ (R @ w)) <= 1e-8 * max(1.0, np.linalg.norm(w))
    if case["spread"] is None:
        assert views[0].shape[0] <= views[0].shape[1]       # only the n <= d_i cases lack a converged reference
        return
    for d in range(1, est.weights_[0].shape[1]):
        tol = _spread_tol(case, d)
        for i in range(len(views)):
            X = theirs[d][i]
            s_ours, s_ref = X @ est.weights_[i][:, d], X @ ref[i][:, d]
            assert np.abs(s_ours - s_ref).max() <= tol * max(1.0, np.linalg.norm(X, 2))
            U, sv, Vt = np.linalg.svd(X, full_matrices=False)
            R = Vt[sv > 1e-10 * sv[0]]                   # the row space: the complement of the null space
            w = est.weights_[i][:, d]
            assert np.abs(R.T @ (R @ w) - R.T @ (R @ ref[i][:, d])).max() <= tol * max(1.0, np.abs(w).max())


def _correlated(n=400, dims=(30, 20), noise=0.03, seed=3):
    rng = np.random.default_rng(seed)
    z = rng.standard_normal((n, 2))
    return [z @ rng.standard_normal((2, p)) + noise * rng.standard_normal((n, p)) for p in dims]


def test_small_alpha_correlated_features_reports_capped_descent():
    """Lasso with a tiny alpha on nearly collinear features: cyclic coordinate descent does not reach the 1e-12 KKT
    bound in its 1000 sweeps (sklearn's max_iter).  The fit says so with a ConvergenceWarning, as the reference's
    solver does, and its weights are those of the same capped iteration restated on the host."""
    from sklearn.exceptions import ConvergenceWarning

    views = _correlated()
    est = _cls("elastic")(latent_dimensions=2, alpha=1e-4, l1_ratio=1.0, max_iter=3, tol=0.0, random_state=0)
    W_ref, iters_ref = _restate(est, views)
    assert all(it < 0 for it in iters_ref)                  # the restatement caps too
    with pytest.warns(ConvergenceWarning, match="sweep limit"):
        est.fit(views)
    assert est._fit_info["iters"] == [abs(it) for it in iters_ref]
    for w, r in zip(est.weights_, W_ref):
        assert np.all(np.isfinite(w))
        assert float(np.abs(w - r).max()) < 1e-6 * max(1.0, float(np.abs(r).max()))
    # a well-conditioned fit gives no warning
    import warnings

    with warnings.catch_warnings():
        warnings.simplefilter("error", ConvergenceWarning)
        _cls("elastic")(latent_dimensions=2, alpha=1e-2, l1_ratio=1.0, random_state=0).fit(conftest_views("two_views"))


def test_float32_inputs_n_below_d_alpha_zero():
    """n <= d_i at alpha = 0 from float32 views: the eigenvalue cut follows the accuracy of the 3xTF32 moments, so the
    null space of the float32 Gram matrix is dropped as in float64 and the weights agree with the float64 fit."""
    rng = np.random.default_rng(4)
    views = [rng.standard_normal((12, 16)), rng.standard_normal((12, 14))]
    for kind in ("elastic", "ipls"):
        kw = dict(latent_dimensions=2, tol=0.0, max_iter=4, random_state=0)
        a = _cls(kind)(**kw).fit(views)
        b = _cls(kind)(**kw).fit([v.astype(np.float32) for v in views])
        for x, y in zip(a.weights_, b.weights_):
            assert float(np.abs(x - y).max()) < 1e-3 * max(1.0, float(np.abs(x).max())), kind


def test_large_alpha_gives_zero_weights():
    views = conftest_views("three_views")
    for kind in ("elastic", "ipls"):
        est = _cls(kind)(latent_dimensions=3, alpha=50.0, l1_ratio=0.7, random_state=0).fit(views)
        for w in est.weights_:
            assert np.all(np.isfinite(w)) and np.all(w == 0.0)
        assert est._fit_info["iters"] == [2, 2, 2]


@pytest.mark.parametrize("kind", ["elastic", "ipls"])
@pytest.mark.parametrize("alpha,l1", [(0.05, 1.0), (0.05, 0.5), (0.5, 0.0), (0.0, 1.0)])
def test_last_subproblem_kkt_from_the_data(kind, alpha, l1):
    """Rebuild each view's last sub-problem of the last dimension from the data in float64 and check the fitted
    weights solve it: KKT residual <= 1e-10 (for SCCA_IPLS up to the std normalisation, undone first)."""
    views = joint_data(n_views=3, n_samples=400, n_features=[30, 20, 12], latent_dimensions=2, signal_to_noise=0.5,
                       random_state=5)
    k = 2
    est = _cls(kind)(latent_dimensions=k, alpha=alpha, l1_ratio=l1, max_iter=1, random_state=2).fit(views)
    Xs = _deflated(views, est.weights_, True)[k - 1]
    W = [w[:, k - 1] for w in est.weights_]
    n = views[0].shape[0]
    m = len(views)
    for i in range(m):            # one sweep: view i saw views < i updated, views > i at their initial weights
        init = E.als_init([v.shape[1] for v in views], k, 2)[k - 1]
        cur = [W[j] if j < i else init[j] for j in range(m)]
        t = sum(Xs[j] @ cur[j] for j in range(m) if kind == "elastic" or j != i)
        y = t / np.linalg.norm(t) if np.linalg.norm(t) > 1e-12 else t
        Q = Xs[i].T @ Xs[i] / n + (alpha / n if l1 == 0.0 else alpha * (1 - l1)) * np.eye(Xs[i].shape[1])
        b = Xs[i].T @ y / n
        w = W[i]
        if kind == "ipls":
            # undo the std normalisation: the regression solution is w * std(X w_raw) = w * c for the c >= 0 that
            # minimises the residual
            lam = alpha * l1
            c = (b @ w - lam * np.abs(w).sum()) / (w @ Q @ w) if np.any(w != 0) else 0.0
            w = c * w
        assert E.kkt_residual(Q, b, alpha * l1, w) <= 1e-10


def test_reference_assertions():
    """cca_zoo tests/linear/test_iterative.py: fit completes (two and three views), reproducibility, :222-235."""
    two, three = conftest_views("two_views"), conftest_views("three_views")
    for kind in ("elastic", "ipls"):
        cls = _cls(kind)
        assert cls(latent_dimensions=1, max_iter=50, random_state=0).fit(two).weights_[0].shape == (10, 1)
        assert len(cls(latent_dimensions=1, max_iter=50, random_state=0).fit(three).weights) == 3
        w1 = cls(latent_dimensions=1, max_iter=50, random_state=42).fit(two).weights
        w2 = cls(latent_dimensions=1, max_iter=50, random_state=42).fit(two).weights
        for a, b in zip(w1, w2):
            np.testing.assert_array_equal(a, b)
        m = cls(latent_dimensions=1, center=False, max_iter=50, random_state=0).fit(two)
        assert m.transform(two)[0].shape == (50, 1)
    m = _cls("elastic")(latent_dimensions=1, alpha=0.1, l1_ratio=1.0, max_iter=200, random_state=0).fit(two)
    assert hasattr(m, "weights_")
    m = _cls("ipls")(latent_dimensions=1, alpha=0.1, l1_ratio=1.0, max_iter=100, random_state=0).fit(two)
    assert hasattr(m, "weights_")
    # a moderate lasso penalty zeroes some weights exactly, not all
    for kind, alpha in (("elastic", 0.02), ("ipls", 0.02)):
        m = _cls(kind)(latent_dimensions=1, alpha=alpha, l1_ratio=1.0, max_iter=200, random_state=0).fit(two)
        for w in m.weights:
            assert 0 < np.sum(w == 0.0) < w.size


@pytest.mark.parametrize("kind", ["elastic", "ipls"])
def test_reruns_bit_identical_partial_fit_and_float32(kind):
    views = conftest_views("three_views")
    kw = dict(latent_dimensions=3, max_iter=300, random_state=1, alpha=0.05, l1_ratio=0.5)
    a = _cls(kind)(**kw).fit(views)
    b = _cls(kind)(**kw).fit(views)
    for x, y in zip(a.weights_, b.weights_):
        assert np.array_equal(x, y)
    p = _cls(kind)(**kw)
    for rows in (slice(0, 17), slice(17, 35), slice(35, 50)):
        p.partial_fit([v[rows] for v in views], solve=rows.stop == 50)
    for x, y in zip(a.weights_, p.weights_):
        assert float(np.abs(x - y).max()) < 1e-10
    f = _cls(kind)(**kw).fit([v.astype(np.float32) for v in views])
    for x, y in zip(f.weights_, a.weights_):
        assert x.dtype == np.float64 and float(np.abs(x - y).max()) < 1e-3


def test_one_library_call_and_one_copy(monkeypatch):
    from cca_zoo_b200 import _lib, ops

    lib = _lib.load()
    real = lib.ccab_als_fit
    calls = {"lib": 0}

    def counted(*args):
        calls["lib"] += 1
        return real(*args)

    monkeypatch.setattr(lib, "ccab_als_fit", counted)
    views = conftest_views("three_views")
    for kind in ("elastic", "ipls"):
        est = _cls(kind)(latent_dimensions=3, alpha=0.05, l1_ratio=0.5, random_state=0, center=False)
        C, dims, n = est._fit_device(views)
        params = est._view_params(dims)
        init = np.zeros((3, sum(dims)))
        init[:, 0] = init[:, 10] = init[:, 18] = 1.0
        real_cpu, copies = torch.Tensor.cpu, []

        def counted_cpu(self, *a, **k):
            copies.append(tuple(self.shape))
            return real_cpu(self, *a, **k)

        calls["lib"] = 0
        monkeypatch.setattr(torch.Tensor, "cpu", counted_cpu)
        W, iters = ops.als_fit(C, dims, n, kind, params, init, 100, 1e-6)
        monkeypatch.setattr(torch.Tensor, "cpu", real_cpu)
        assert calls["lib"] == 1 and len(copies) == 1 and W.shape == (24, 3) and np.all(np.isfinite(W))
    with pytest.raises(ValueError, match="params"):
        ops.als_fit(C, dims, n, "elastic", [0.1, 0.5], init, 10, 1e-6)


@pytest.mark.parametrize("kind,alpha,l1", [("ipls", 0.0, 1.0), ("elastic", 0.02, 0.5)])
def test_elastic_beyond_l2(kind, alpha, l1):
    """d_i = 2048 (the largest view width): G (128 MB) does not fit in L2; a few fixed sweeps."""
    views = joint_data(n_views=2, n_samples=6000, n_features=[2048, 2048], latent_dimensions=2,
                       signal_to_noise=0.2, random_state=11)
    est = _cls(kind)(latent_dimensions=2, alpha=alpha, l1_ratio=l1, tol=0.0, max_iter=3, random_state=0)
    W_ref, iters_ref = _restate(est, views)
    est.fit(views)
    assert est._fit_info["iters"] == iters_ref == [3, 3]
    for w, r in zip(est.weights_, W_ref):
        assert float(np.abs(w - r).max()) < 1e-9 * max(1.0, float(np.abs(r).max()))


def _free_port():
    s = socket.socket()
    s.bind(("127.0.0.1", 0))
    port = s.getsockname()[1]
    s.close()
    return port


def _worker(rank, world, port, out_dir):
    import torch.distributed as dist

    from cca_zoo_b200 import parallel

    os.environ.update(MASTER_ADDR="127.0.0.1", MASTER_PORT=str(port), RANK=str(rank), WORLD_SIZE=str(world))
    torch.cuda.set_device(rank)
    dist.init_process_group("nccl", rank=rank, world_size=world, device_id=torch.device("cuda", rank))
    try:
        views = joint_data(n_views=3, n_samples=3001, n_features=[40, 30, 20], latent_dimensions=3,
                           signal_to_noise=0.3, random_state=9)
        lo, hi = parallel.shard_rows(3001, rank, world)
        for kind in ("elastic", "ipls"):
            est = _cls(kind)(latent_dimensions=3, alpha=0.02, l1_ratio=0.5, random_state=0).fit([v[lo:hi] for v in views])
            np.save(os.path.join(out_dir, f"{kind}_w1_rank{rank}.npy"), est.weights_[1])
    finally:
        dist.destroy_process_group()


@pytest.mark.skipif(torch.cuda.device_count() < 2, reason="needs 2 GPUs")
def test_two_rank_fit_identical_on_both_ranks(tmp_path):
    import torch.multiprocessing as mp

    mp.spawn(_worker, args=(2, _free_port(), str(tmp_path)), nprocs=2, join=True)
    views = joint_data(n_views=3, n_samples=3001, n_features=[40, 30, 20], latent_dimensions=3, signal_to_noise=0.3,
                       random_state=9)
    for kind in ("elastic", "ipls"):
        w = [np.load(tmp_path / f"{kind}_w1_rank{r}.npy") for r in range(2)]
        assert np.array_equal(w[0], w[1])
        single = _cls(kind)(latent_dimensions=3, alpha=0.02, l1_ratio=0.5, random_state=0).fit(views)
        assert float(np.abs(w[0] - single.weights_[1]).max()) < 1e-9
