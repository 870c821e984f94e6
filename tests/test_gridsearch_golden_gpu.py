"""GridSearchCV against the reference's GridSearchCV (tests/golden/reference_outputs_gridsearch.*, written by
oracle/make_golden_gridsearch.py on CPU): split scores, their mean, std and rank, best_params_, best_score_, the
best estimator's held-out score and the fit-failure warnings, case by case.  Every case that the moment route serves
takes it here."""
from __future__ import annotations

import json
import os
import warnings

import numpy as np
import pytest
from sklearn.model_selection import KFold, RepeatedKFold, ShuffleSplit

from cca_zoo_b200 import linear
from cca_zoo_b200.model_selection import GridSearchCV

pytestmark = pytest.mark.gpu

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "reference_outputs_gridsearch")
with open(GOLDEN + ".json") as f:
    META = json.load(f)
SPLITTERS = {
    "int4": lambda: 4,
    "kfold_shuffle": lambda: KFold(4, shuffle=True, random_state=0),
    "shuffle_split": lambda: ShuffleSplit(3, test_size=0.3, random_state=0),
    "repeated_kfold": lambda: RepeatedKFold(n_splits=3, n_repeats=2, random_state=0),
}
#: closed-form solves agree with the reference's LAPACK to rounding; the ALS solves agree to their stopping rule
TOL = {"SCCA_PMD": 1e-5, "ElasticCCA": 1e-5}
CLOSED_FORM_TOL = 1e-8


@pytest.fixture(scope="module")
def data():
    g = np.load(GOLDEN + ".npz")
    m = len(META["dims"])
    return {k: g[k] for k in g.files}, [g[f"train_{i}"] for i in range(m)], [g[f"test_{i}"] for i in range(m)]


@pytest.mark.parametrize("name", sorted(META["cases"]))
def test_matches_reference(name, data):
    g, train, test = data
    case = META["cases"][name]
    m, tol = case["n_views"], TOL.get(case["estimator"], CLOSED_FORM_TOL)
    est = getattr(linear, case["estimator"])(**case["kwargs"])
    with warnings.catch_warnings(record=True) as rec:
        warnings.simplefilter("always")
        gs = GridSearchCV(est, case["grid"], cv=SPLITTERS[case["splitter"]]()).fit(train[:m])
    assert gs._inner_cv is None                                    # the moment route
    r = gs.cv_results_
    ref = g[f"{name}__split_scores"]
    got = np.array([r[f"split{s}_test_score"] for s in range(ref.shape[1])]).T
    np.testing.assert_allclose(got, ref, rtol=0, atol=tol, equal_nan=True)
    np.testing.assert_allclose(r["mean_test_score"], g[f"{name}__mean"], rtol=0, atol=tol, equal_nan=True)
    np.testing.assert_allclose(r["std_test_score"], g[f"{name}__std"], rtol=0, atol=tol, equal_nan=True)
    np.testing.assert_array_equal(r["rank_test_score"], g[f"{name}__rank"])
    assert gs.best_params_ == case["best_params"]
    assert gs.best_score_ == pytest.approx(case["best_score"], abs=tol)
    assert gs.score(test[:m]) == pytest.approx(case["held_out_score"], abs=tol)
    got_warnings = sorted({w.category.__name__ for w in rec if w.category.__name__ in ("FitFailedWarning",
                                                                                      "UserWarning")})
    assert got_warnings == case["warnings"]
