"""GridSearchCV on the device: the moment route against the generic route (sklearn's GridSearchCV through the
view-splitting wrapper, every candidate fitted and scored on its rows) for every estimator and splitter of the case
table, float32 views, badly centred views, CUDA-tensor inputs, a streamed host input, the refit, and the delegation of
``transform`` / ``score``."""
from __future__ import annotations

import numpy as np
import pytest
import torch

from cca_zoo_b200.linear import CCA, rCCA
from cca_zoo_b200.model_selection import GridSearchCV

from .gridsearch_cases import CASES, NON_PARTITION, SPLITTERS, views

pytestmark = pytest.mark.gpu


def _generic(gs):
    g = GridSearchCV(gs.estimator, gs.param_grid, cv=gs.cv, refit=gs.refit)
    g._moment_route = lambda *a: (None, False)
    return g


def _compare(moment, generic, tol):
    ra, rb = moment.cv_results_, generic.cv_results_
    assert set(ra) == set(rb)
    assert ra["params"] == rb["params"]
    split_keys = [k for k in ra if k.startswith("split")]
    a = np.array([ra[k] for k in split_keys])
    b = np.array([rb[k] for k in split_keys])
    np.testing.assert_allclose(a, b, rtol=0, atol=tol)
    np.testing.assert_array_equal(ra["rank_test_score"], rb["rank_test_score"])
    assert moment.best_params_ == generic.best_params_


@pytest.mark.parametrize("splitter", list(SPLITTERS))
@pytest.mark.parametrize("case", list(CASES))
def test_moment_route_matches_generic_float64(case, splitter):
    est, grid, m = CASES[case]
    v = views(m, n=200)
    moment = GridSearchCV(est, grid, cv=SPLITTERS[splitter]).fit(v)
    assert (moment._inner_cv is None) == (splitter not in NON_PARTITION)
    _compare(moment, _generic(moment).fit(v), 1e-10)


@pytest.mark.parametrize("case", ["rcca_c", "rcca_perview_c", "cca_k", "mcca_3", "gcca_3"])
def test_moment_route_matches_generic_float32(case):
    est, grid, m = CASES[case]
    v = views(m, n=300, dtype=np.float32)
    moment = GridSearchCV(est, grid, cv=SPLITTERS["kfold_shuffle"]).fit(v)
    _compare(moment, _generic(moment).fit(v), 1e-4)


def test_badly_centred_views():
    v = views(2, n=400, offset=1e3)
    moment = GridSearchCV(rCCA(latent_dimensions=2), {"c": [0.0, 0.3, 0.8]}, cv=4).fit(v)
    _compare(moment, _generic(moment).fit(v), 1e-8)


def test_cuda_tensor_inputs():
    v = views(2, n=300)
    tv = [torch.from_numpy(x).cuda() for x in v]
    on_dev = GridSearchCV(rCCA(), {"c": [0.1, 0.5]}, cv=SPLITTERS["kfold_shuffle"]).fit(tv)
    on_host = GridSearchCV(rCCA(), {"c": [0.1, 0.5]}, cv=SPLITTERS["kfold_shuffle"]).fit(v)
    _compare(on_dev, on_host, 1e-12)
    for w, u in zip(on_dev.best_estimator_.weights_, on_host.best_estimator_.weights_):
        np.testing.assert_array_equal(w, u)


def test_streamed_host_input():
    v = views(2, n=1 << 17, dims=(40, 40))                # 84 MB of float64: above the 64 MB streaming threshold
    assert sum(x.nbytes for x in v) >= rCCA._stream_threshold_bytes
    moment = GridSearchCV(rCCA(), {"c": [0.1, 0.6]}, cv=2).fit(v)
    _compare(moment, _generic(moment).fit(v), 1e-10)
    direct = rCCA(**moment.best_params_).fit(v)
    for w, u in zip(moment.best_estimator_.weights_, direct.weights_):
        np.testing.assert_array_equal(w, u)


@pytest.mark.parametrize("case", ["rcca_c", "mcca_3", "gcca_3", "pmd_tau", "elastic_alpha"])
def test_refit_is_bit_identical_to_fit(case):
    from sklearn.base import clone

    est, grid, m = CASES[case]
    v = views(m, n=200)
    gs = GridSearchCV(est, grid, cv=3).fit(v)
    direct = clone(est).set_params(**gs.best_params_).fit(v)
    for w, u in zip(gs.best_estimator_.weights_, direct.weights_):
        np.testing.assert_array_equal(w, u)


def test_transform_and_score_delegate():
    v = views(2, n=200)
    held = views(2, n=80, seed=3)
    gs = GridSearchCV(CCA(), {"latent_dimensions": [1, 2]}, cv=3).fit(v)
    generic = _generic(GridSearchCV(CCA(), {"latent_dimensions": [1, 2]}, cv=3)).fit(v)
    for a, b in zip(gs.transform(held), gs.best_estimator_.transform(held)):
        np.testing.assert_array_equal(a, b)
    assert gs.score(held) == pytest.approx(generic.score(held), abs=1e-12)


def test_refit_false_exceptions_match():
    v = views(2, n=200)
    errors = []
    for gs in (GridSearchCV(CCA(), {"latent_dimensions": [1, 2]}, cv=3, refit=False),
               _generic(GridSearchCV(CCA(), {"latent_dimensions": [1, 2]}, cv=3, refit=False))):
        gs.fit(v)
        row = []
        for call in (gs.transform, gs.score):
            with pytest.raises(Exception) as exc:
                call(v)
            row.append(type(exc.value))
        errors.append(row)
    assert errors[0] == errors[1] == [AttributeError, AttributeError]
