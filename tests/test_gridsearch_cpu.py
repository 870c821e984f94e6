"""GridSearchCV host logic on the torch-CPU stand-in (tests/fake_ops*.py): which route ``fit`` takes, the order of
splits and candidates, ``cv_results_`` of the moment route against the generic route (sklearn's GridSearchCV through
the view-splitting wrapper), failed fits, and the behaviours of the reference's tests/model_selection/test_search.py."""
from __future__ import annotations

import warnings

import numpy as np
import pytest
from sklearn.exceptions import FitFailedWarning
from sklearn.model_selection import KFold, ShuffleSplit, check_cv

from cca_zoo_b200 import parallel
from cca_zoo_b200.datasets import conftest_views
from cca_zoo_b200.linear import CCA, GRCCA, MCCA, PLS_EY, PartialCCA, TCCA, rCCA
from cca_zoo_b200.model_selection import GridSearchCV, _search

from . import fake_ops, fake_ops_cv, fake_ops_sparse
from .gridsearch_cases import CASES, NON_PARTITION, SPLITTERS, views


@pytest.fixture
def standin(monkeypatch):
    fake_ops.install(monkeypatch)
    fake_ops_sparse.install(monkeypatch)
    fake_ops_cv.install(monkeypatch)
    return monkeypatch


def _routes(monkeypatch):
    """Record which route each fit takes."""
    taken = []
    for name in ("_fit_generic", "_search_moments"):
        orig = getattr(GridSearchCV, name)

        def spy(self, *a, _orig=orig, _name=name, **k):
            taken.append(_name)
            return _orig(self, *a, **k)

        monkeypatch.setattr(GridSearchCV, name, spy)
    return taken


def _generic(gs):
    """The same search forced onto the generic route."""
    g = GridSearchCV(gs.estimator, gs.param_grid, cv=gs.cv, refit=gs.refit)
    g._moment_route = lambda *a: (None, False)
    return g


# ------------------------------------------------------------------------------------------------ route selection
ROUTE_TABLE = [
    # (estimator, grid, kwargs, fit_params, expected route)
    (rCCA(), {"c": [0.1, 0.2]}, {}, {}, "moment"),
    (CCA(), {"latent_dimensions": [1, 2]}, {"n_jobs": 1}, {}, "moment"),
    (MCCA(), {"c": [0.1]}, {}, {}, "moment"),
    (GRCCA(), {"c": [0.1]}, {}, {}, "generic"),                  # subclass overriding fit
    (PartialCCA(), {"c": [0.1]}, {}, {}, "generic"),
    (TCCA(), {"c": [0.1]}, {}, {}, "generic"),                   # not fitted from the block moments
    (PLS_EY(), {"c": [0.1]}, {}, {}, "generic"),
    (rCCA(), {"c": [0.1]}, {"scoring": lambda est, X, y=None: 0.0}, {}, "generic"),
    (rCCA(), {"c": [0.1], "precision": ["exact"]}, {}, {}, "generic"),
    (rCCA(), [{"c": [0.1]}, {"device": [None]}], {}, {}, "generic"),
    (rCCA(), {"c": [0.1]}, {"cv": 25}, {}, "moment"),           # 50 rows: 2 test rows per fold is the least allowed
    (rCCA(), {"c": [0.1]}, {"cv": 26}, {}, "generic"),          # ... and 26 folds leave some with 1
    (rCCA(), {"c": [0.1]}, {"cv": ShuffleSplit(2, test_size=1, random_state=0)}, {}, "generic"),
    (rCCA(), {"c": [0.1]}, {"cv": SPLITTERS["time_series"]}, {}, "generic"),     # later rows are in neither side
    (rCCA(), {"c": [0.1]}, {"cv": SPLITTERS["shuffle_split_partial"]}, {}, "generic"),
    (rCCA(), {"c": [0.1]}, {"cv": [(np.arange(2, 50), np.arange(0, 4))]}, {}, "generic"),        # overlapping sides
    (rCCA(), {"c": [0.1]}, {"cv": [(np.r_[np.arange(4, 50), 4], np.arange(0, 3))]}, {}, "generic"),  # a repeated row
    (rCCA(), {"c": [0.1]}, {"cv": [(np.arange(4, 50), np.arange(0, 4))]}, {}, "moment"),
]


@pytest.mark.parametrize("est,grid,kwargs,fit_params,expected", ROUTE_TABLE)
def test_route_selection(est, grid, kwargs, fit_params, expected):
    gs = GridSearchCV(est, grid, **{"cv": 3, **kwargs})
    _, eligible = gs._moment_route(50, None, fit_params)
    assert eligible == (expected == "moment")


def test_route_selection_fit_params_and_distributed(monkeypatch):
    gs = GridSearchCV(rCCA(), {"c": [0.1]}, cv=3)
    assert gs._moment_route(50, None, {})[1]
    assert gs._moment_route(50, None, {"groups": np.arange(50)}) == (None, False)
    monkeypatch.setattr(parallel, "is_distributed", lambda group=None: True)
    assert gs._moment_route(50, None, {}) == (None, False)


def test_fit_takes_the_selected_route(standin):
    taken = _routes(standin)
    v = conftest_views("two_views")
    GridSearchCV(rCCA(), {"c": [0.1, 0.2]}, cv=2).fit(v)
    GridSearchCV(GRCCA(), {"c": [0.1]}, cv=2).fit(v)
    assert taken == ["_search_moments", "_fit_generic"]


# ------------------------------------------------------------------------------------------------ enumeration order
@pytest.mark.parametrize("splitter", list(SPLITTERS))
def test_splits_are_sklearns(splitter):
    cv = SPLITTERS[splitter]
    gs = GridSearchCV(rCCA(), {"c": [0.1]}, cv=cv)
    got, _ = gs._moment_route(97, None, {})
    want = list(check_cv(cv, None, classifier=False).split(np.zeros((97, 18))))
    assert len(got) == len(want)
    for (a, b), (c, d) in zip(got, want):
        np.testing.assert_array_equal(a, c)
        np.testing.assert_array_equal(b, d)


def test_rows_slices_runs_and_gathers_the_rest():
    v = np.arange(40.0).reshape(20, 2)
    run = _search._rows(v, np.arange(5, 9))
    assert np.shares_memory(run, v) and np.array_equal(run, v[5:9])
    idx = np.array([1, 3, 4, 9])
    np.testing.assert_array_equal(_search._rows(v, idx), v[idx])


# ------------------------------------------------------------------------------------------------ route parity
def _assert_results_match(a, b, tol):
    ra, rb = a.cv_results_, b.cv_results_
    assert set(ra) == set(rb)
    for key in ra:
        if key.startswith("param_"):
            assert ra[key].dtype == rb[key].dtype
            np.testing.assert_array_equal(np.ma.getmaskarray(ra[key]), np.ma.getmaskarray(rb[key]))
            assert [x for x in ra[key].compressed()] == [x for x in rb[key].compressed()]
        elif key == "params":
            assert ra[key] == rb[key]
        elif key.startswith("rank_"):
            np.testing.assert_array_equal(ra[key], rb[key])
            assert ra[key].dtype == rb[key].dtype
        elif "time" not in key:
            np.testing.assert_allclose(ra[key], rb[key], rtol=0, atol=tol, equal_nan=True)
    assert a.best_params_ == b.best_params_
    assert a.best_score_ == pytest.approx(b.best_score_, abs=tol)


@pytest.mark.parametrize("splitter", ["kfold_shuffle", "shuffle_split", "time_series", "shuffle_split_partial"])
@pytest.mark.parametrize("case", list(CASES))
def test_moment_route_matches_generic_route(standin, case, splitter):
    est, grid, m = CASES[case]
    v = views(m)
    moment = GridSearchCV(est, grid, cv=SPLITTERS[splitter]).fit(v)
    assert (moment._inner_cv is None) == (splitter not in NON_PARTITION)
    generic = _generic(moment).fit(v)
    assert generic._inner_cv is not None
    _assert_results_match(moment, generic, 1e-10)
    for w, u in zip(moment.best_estimator_.weights_, generic.best_estimator_.weights_):
        np.testing.assert_array_equal(w, u)


def _fit_warnings(gs, v):
    with warnings.catch_warnings(record=True) as rec:
        warnings.simplefilter("always")
        gs.fit(v)
    return sorted({type(w.message).__name__ for w in rec if issubclass(w.category, (FitFailedWarning, UserWarning))})


def test_failed_candidate_follows_sklearns_rules(standin):
    v = views(2)
    moment = GridSearchCV(rCCA(), {"c": [0.1, 2.0, 0.5]}, cv=3)
    generic = _generic(moment)
    wm, wg = _fit_warnings(moment, v), _fit_warnings(generic, v)
    assert wm == wg == ["FitFailedWarning", "UserWarning"]
    assert np.isnan(moment.cv_results_["mean_test_score"][1])
    assert moment.cv_results_["rank_test_score"][1] == 3
    _assert_results_match(moment, generic, 1e-10)


def test_all_fits_failed_raises(standin):
    v = views(2)
    for gs in (GridSearchCV(rCCA(), {"c": [2.0, 3.0]}, cv=2), _generic(GridSearchCV(rCCA(), {"c": [2.0, 3.0]}, cv=2))):
        with pytest.raises(ValueError, match="All the 4 fits failed"):
            gs.fit(v)


def test_three_views_fail_rcca_on_both_routes(standin):
    v = views(3)
    for gs in (GridSearchCV(rCCA(), {"c": [0.1]}, cv=2), _generic(GridSearchCV(rCCA(), {"c": [0.1]}, cv=2))):
        with pytest.raises(ValueError, match="fits failed"):
            gs.fit(v)


@pytest.mark.parametrize("route", ["moment", "generic"])
def test_refit_false(standin, route):
    v = conftest_views("two_views")
    gs = GridSearchCV(CCA(), {"latent_dimensions": [1, 2]}, cv=2, refit=False)
    if route == "generic":
        gs = _generic(gs)
    gs.fit(v)
    assert not hasattr(gs, "best_estimator_")
    with pytest.raises(AttributeError, match="refit"):
        gs.transform(v)
    with pytest.raises(AttributeError, match="refit"):
        gs.score(v)


# ------------------------------------------------------------------------------------------------ the reference's tests
@pytest.fixture(params=["moment", "generic"])
def make(request, standin):
    def build(*a, **k):
        gs = GridSearchCV(*a, **k)
        return _generic(gs) if request.param == "generic" else gs
    return build


def test_fit_returns_self(make):
    gs = make(CCA(), param_grid={"latent_dimensions": [1]}, cv=2)
    assert gs.fit(conftest_views("two_views")) is gs


def test_best_params_score_and_estimator(make):
    v = conftest_views("two_views")
    gs = make(CCA(), param_grid={"latent_dimensions": [1, 2]}, cv=2).fit(v)
    assert gs.best_params_["latent_dimensions"] in [1, 2]
    assert not any(k.startswith("estimator__") for k in gs.best_params_)
    assert isinstance(gs.best_score_, float) and -1.0 <= gs.best_score_ <= 1.0
    assert len(gs.best_estimator_.transform(v)) == 2
    assert isinstance(gs.cv_results_, dict) and "mean_test_score" in gs.cv_results_


def test_multi_param_grid(make):
    gs = make(rCCA(), param_grid={"latent_dimensions": [1, 2], "c": [0.0, 0.1]}, cv=2).fit(conftest_views("two_views"))
    assert set(gs.best_params_) == {"latent_dimensions", "c"}


def test_list_of_grids(make):
    gs = make(CCA(), param_grid=[{"latent_dimensions": [1]}, {"latent_dimensions": [2]}], cv=2)
    gs.fit(conftest_views("two_views"))
    assert gs.best_params_["latent_dimensions"] in [1, 2]


def test_score_after_fit(make):
    rng = np.random.default_rng(10)
    test_views = [rng.standard_normal((20, 10)), rng.standard_normal((20, 8))]
    gs = make(CCA(), param_grid={"latent_dimensions": [1, 2]}, cv=2).fit(conftest_views("two_views"))
    s = gs.score(test_views)
    assert isinstance(s, float) and -1.0 <= s <= 1.0
    assert s == pytest.approx(float(np.mean(gs.best_estimator_.score(test_views))), abs=1e-12)


def test_n_jobs_one(make):
    gs = make(CCA(), param_grid={"latent_dimensions": [1, 2]}, cv=2, n_jobs=1).fit(conftest_views("two_views"))
    assert hasattr(gs, "best_score_")


def test_three_view_model(make):
    gs = make(MCCA(), param_grid={"latent_dimensions": [1, 2]}, cv=2).fit(conftest_views("three_views"))
    assert isinstance(gs.best_score_, float) and "latent_dimensions" in gs.best_params_


def test_transform_delegates(make):
    v = conftest_views("two_views")
    gs = make(CCA(), param_grid={"latent_dimensions": [1, 2]}, cv=2).fit(v)
    for a, b in zip(gs.transform(v), gs.best_estimator_.transform(v)):
        np.testing.assert_array_equal(a, b)


def test_kfold_without_shuffle_matches(standin):
    v = views(2, n=101)
    moment = GridSearchCV(rCCA(), {"c": [0.1, 0.4]}, cv=KFold(4)).fit(v)
    _assert_results_match(moment, _generic(moment).fit(v), 1e-10)


def test_one_shot_split_iterable_reaches_the_generic_route(standin):
    v = views(2, n=60)
    pairs = [(np.arange(1, 60), np.arange(0, 1)), (np.r_[0, np.arange(2, 60)], np.arange(1, 2))]   # 1 test row each
    gs = GridSearchCV(rCCA(), {"c": [0.1, 0.5]}, cv=(p for p in pairs)).fit(v)
    assert gs._inner_cv is not None and gs.n_splits_ == 2
    want = GridSearchCV(rCCA(), {"c": [0.1, 0.5]}, cv=pairs).fit(v)
    np.testing.assert_array_equal(gs.cv_results_["split1_test_score"], want.cv_results_["split1_test_score"])


def test_failed_scoring_gives_nan_and_sklearns_warning(standin):
    def broken(*a, **k):
        raise RuntimeError("scoring kernel failed")

    standin.setattr(_search.ops, "cv_scores", broken)
    with warnings.catch_warnings(record=True) as rec:
        warnings.simplefilter("always")
        gs = GridSearchCV(rCCA(), {"c": [0.1, 0.5]}, cv=2).fit(views(2))
    msgs = [str(w.message) for w in rec if w.category is UserWarning]
    assert sum(m.startswith("Scoring failed.") for m in msgs) == 4
    assert not any(w.category is FitFailedWarning for w in rec)
    assert np.isnan(gs.cv_results_["mean_test_score"]).all()
    np.testing.assert_array_equal(gs.cv_results_["rank_test_score"], [1, 1])
