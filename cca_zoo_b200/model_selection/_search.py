"""Grid search with cross-validation for the multiview estimators, at the reference's import path
``cca_zoo.model_selection``.

The search has the reference's interface and results (``cv_results_`` in sklearn's layout for the grid of a
view-splitting wrapper, ``estimator__<name>`` keys; ``best_params_`` without the prefix) and takes one of two routes:

* the generic route, for any estimator: the views are stacked and handed to ``sklearn.model_selection.GridSearchCV``
  through ``_MultiviewWrapper``, so every (candidate, split) is a clone / fit(train rows) / score(test rows) cycle;
* the moment route, for the estimators whose fit is a function of the block moments alone (``_MOMENT_ESTIMATORS``):
  the moments are additive over rows, so one moment pass over all rows and one over each split's test rows carry all
  the data a grid needs.  Each split's train moments are the total minus the test moments (float64), each candidate
  is fitted from them by the estimator's own solve (``BaseModel._fit_from_moments``), and all candidates of a split are
  scored against the test covariance in one device call (``ops.cv_scores``: the mean over dimensions of
  ``average_pairwise_correlations``, which is what the wrapper's ``score`` returns).  ``refit`` solves the best
  candidate from the total moments without another pass, which gives the weights ``fit(views)`` gives.

``fit`` takes the moment route when nothing it can observe rules it out (see ``_moment_route``); its ``n_jobs`` is then
unused, as nothing is spawned.
"""
from __future__ import annotations

import time
import traceback
import warnings
from typing import Any

import numpy as np
import sklearn.model_selection as skms
import torch
from scipy.stats import rankdata
from sklearn.base import BaseEstimator, clone
from sklearn.model_selection._search import _yield_masked_array_for_each_param
from sklearn.model_selection._validation import _warn_or_raise_about_fit_failures

from .. import ops, parallel
from .._validation import validate_views
from ..linear import (CCA, GCCA, MCCA, PLS, PLS_ALS, ElasticCCA, ParkhomenkoCCA, SCCA_ADMM, SCCA_IPLS, SCCA_PMD,
                      SCCA_Span, rCCA)

_PREFIX = "estimator__"

#: estimators whose ``fit`` is ``_fit_moments`` of the moment buffer of the views (exact types: subclasses that
#: override ``fit``, such as GRCCA and PartialCCA, take the generic route)
_MOMENT_ESTIMATORS = (rCCA, CCA, PLS, MCCA, GCCA, PLS_ALS, SCCA_PMD, ParkhomenkoCCA, SCCA_Span, SCCA_ADMM, ElasticCCA,
                      SCCA_IPLS)
#: parameters that change the moment pass itself rather than the solve after it
_MOMENT_PASS_PARAMS = ("precision", "device")


def _host(v):
    return v.detach().cpu().numpy() if isinstance(v, torch.Tensor) else np.asarray(v)


class _MultiviewWrapper(BaseEstimator):
    """A multiview estimator behind sklearn's single-matrix interface: ``X`` is the views stacked by columns and
    ``split_indices`` the view widths that split it again."""

    def __init__(self, estimator: BaseEstimator, split_indices: list[int]) -> None:
        self.estimator = estimator
        self.split_indices = split_indices

    def _split_views(self, X):
        edges = np.cumsum([0] + list(self.split_indices))
        return [X[:, a:b] for a, b in zip(edges[:-1], edges[1:])]

    def fit(self, X, y=None, **fit_params: Any):
        self.estimator_ = clone(self.estimator)
        self.estimator_.fit(self._split_views(X), **fit_params)
        return self

    def score(self, X, y=None) -> float:
        """Mean over the latent dimensions of the average pairwise correlations."""
        return float(np.mean(self.estimator_.score(self._split_views(X))))

    def get_params(self, deep: bool = True) -> dict[str, Any]:
        params = {"estimator": self.estimator, "split_indices": self.split_indices}
        if deep:
            params.update({_PREFIX + k: v for k, v in self.estimator.get_params(deep=True).items()})
        return params

    def set_params(self, **params: Any):
        inner = {k[len(_PREFIX):]: v for k, v in params.items() if k.startswith(_PREFIX)}
        own = {k: v for k, v in params.items() if not k.startswith(_PREFIX)}
        if own:
            super().set_params(**own)
        if inner:
            self.estimator.set_params(**inner)
        return self


def _rows(v, idx):
    """Rows ``idx`` of a view: a slice when they form one ascending run, a gather otherwise."""
    lo = int(idx[0])
    if len(idx) == int(idx[-1]) - lo + 1 and np.array_equal(idx, np.arange(lo, lo + len(idx))):
        return v[lo:lo + len(idx)]
    if isinstance(v, torch.Tensor):
        return v.index_select(0, torch.from_numpy(np.asarray(idx, dtype=np.int64)).to(v.device))
    return v[idx]


def _is_partition(train, test, n_rows: int) -> bool:
    """Whether ``train`` and ``test`` together hold every row index below ``n_rows`` exactly once."""
    if len(train) + len(test) != n_rows:
        return False
    idx = np.concatenate([train, test])
    if idx.dtype.kind not in "iu" or idx.min() < 0 or idx.max() >= n_rows:
        return False
    return bool(np.bincount(idx, minlength=n_rows).max() == 1)


class GridSearchCV:
    """Exhaustive search over a parameter grid for a multiview estimator, with cross-validated scores.

    Args:
        estimator: a multiview estimator of this package (e.g. ``cca_zoo_b200.linear.rCCA``).
        param_grid: dict, or list of dicts, of parameter names and the lists of values to try.
        cv: number of folds or a cross-validation splitter (default 5), as in sklearn.
        scoring: ``None`` scores with the estimator's ``score`` (mean over dimensions); anything else is passed to
            sklearn.
        n_jobs: jobs of the generic route (sklearn's meaning); unused on the moment route.
        refit: refit the best candidate on all rows (default True).
        verbose: sklearn's verbosity.

    After ``fit``: ``cv_results_``, ``best_score_``, ``best_params_`` and, when ``refit``, ``best_estimator_``.
    """

    def __init__(self, estimator: BaseEstimator, param_grid, cv=5, scoring=None, n_jobs=None, refit: bool = True,
                 verbose: int = 0) -> None:
        self.estimator = estimator
        self.param_grid = param_grid
        self.cv = cv
        self.scoring = scoring
        self.n_jobs = n_jobs
        self.refit = refit
        self.verbose = verbose

    def _wrapped_grid(self):
        if isinstance(self.param_grid, dict):
            return {_PREFIX + k: v for k, v in self.param_grid.items()}
        return [{_PREFIX + k: v for k, v in grid.items()} for grid in self.param_grid]

    def _moment_route(self, n_rows: int, y, fit_params):
        """(splits, eligible): the splits as a list of (train, test) index arrays, or None when the route was ruled out
        before they were enumerated, and whether the moment route applies.  It needs every split to be a partition of
        the rows (train = all rows not in test, each row once): the train moments are the total minus the test
        moments.  Splitters that leave rows out (TimeSeriesSplit, ShuffleSplit with train_size + test_size < 1) or
        index lists that repeat rows take the generic route."""
        grids = [self.param_grid] if isinstance(self.param_grid, dict) else list(self.param_grid)
        if (type(self.estimator) not in _MOMENT_ESTIMATORS or self.scoring is not None or fit_params
                or any(p in g for g in grids for p in _MOMENT_PASS_PARAMS) or parallel.is_distributed()):
            return None, False
        cv = skms.check_cv(self.cv, y, classifier=False)          # the wrapper of the generic route is no classifier
        splits = [(np.asarray(tr), np.asarray(te)) for tr, te in cv.split(np.empty((n_rows, 0)), y)]
        ok = bool(splits) and all(len(tr) >= 2 and len(te) >= 2 and _is_partition(tr, te, n_rows) for tr, te in splits)
        return splits, ok

    def fit(self, views, y=None, **fit_params: Any):
        """Search the grid on ``views`` (list of ``(n_samples, n_features_i)`` arrays or tensors); returns self."""
        splits, eligible = self._moment_route(len(views[0]), y, fit_params)
        if eligible:
            self._search_moments(views, splits)
        else:                               # splits already drawn from a one-shot iterable are handed on, not redrawn
            self._fit_generic(views, y, self.cv if splits is None else splits, **fit_params)
        return self

    # ------------------------------------------------------------------ generic route
    def _fit_generic(self, views, y, cv, **fit_params):
        arrays = [_host(v) for v in views]
        wrapper = _MultiviewWrapper(self.estimator, [a.shape[1] for a in arrays])
        self._inner_cv = skms.GridSearchCV(wrapper, self._wrapped_grid(), cv=cv, scoring=self.scoring,
                                           n_jobs=self.n_jobs, refit=self.refit, verbose=self.verbose)
        self._inner_cv.fit(np.hstack(arrays), y, **fit_params)
        self.cv_results_ = self._inner_cv.cv_results_
        self.best_index_ = self._inner_cv.best_index_
        self.best_score_ = self._inner_cv.best_score_
        self.best_params_ = {k[len(_PREFIX):]: v for k, v in self._inner_cv.best_params_.items()}
        self.n_splits_ = self._inner_cv.n_splits_
        if self.refit:
            self.best_estimator_ = self._inner_cv.best_estimator_.estimator_
            self.refit_time_ = self._inner_cv.refit_time_

    # ------------------------------------------------------------------ moment route
    def _search_moments(self, views, splits):
        self._inner_cv = None
        candidates = list(skms.ParameterGrid(self._wrapped_grid()))
        n_cand, n_splits = len(candidates), len(splits)
        if self.verbose > 0:
            print(f"Fitting {n_splits} folds for each of {n_cand} candidates, totalling {n_cand * n_splits} fits")
        validated = validate_views(views)
        base = clone(self.estimator)
        device = base._device()
        total, n_rows, dims, in_dtype = base._local_moments(validated, device)
        scores = np.full((n_cand, n_splits), np.nan)
        fit_time = np.zeros((n_cand, n_splits))
        score_time = np.zeros((n_cand, n_splits))
        errors = [[None] * n_splits for _ in range(n_cand)]
        D = int(sum(dims))
        for s, (train, test) in enumerate(splits):
            test_mom, n_test, _, _ = base._local_moments([_rows(v, test) for v in validated], device)
            train_mom = total - test_mom
            C, _ = ops.covariance(test_mom, dims, n_test, center=True, dtype=torch.float64)
            fitted = []
            for c, params in enumerate(candidates):
                est = clone(self.estimator).set_params(
                    **{k[len(_PREFIX):]: v for k, v in clone(params, safe=False).items()})
                t0 = time.perf_counter()
                try:
                    est._fit_from_moments(train_mom.clone(), len(train), dims, in_dtype)
                except Exception:
                    errors[c][s] = traceback.format_exc()
                else:
                    fitted.append((c, [np.asarray(w, dtype=np.float64) for w in est.weights_]))
                fit_time[c, s] = time.perf_counter() - t0
            if not fitted:
                continue
            t0 = time.perf_counter()
            k_of = [int(ws[0].shape[1]) for _, ws in fitted]
            k_max = max(k_of)
            W = np.zeros((D, len(fitted) * k_max))
            for b, (_, ws) in enumerate(fitted):
                W[:, b * k_max:b * k_max + k_of[b]] = np.concatenate(ws, axis=0)
            try:
                _, score = ops.cv_scores(C, dims, n_test, torch.from_numpy(W).to(device), k_of)
                score = score.cpu().numpy()                  # the one host read-back of the split
            except Exception:                                # sklearn's error_score=nan rule for a failed score
                detail = traceback.format_exc()
                score = np.full(len(fitted), np.nan)
                for _ in fitted:
                    warnings.warn("Scoring failed. The score on this train-test partition for these parameters will be "
                                  f"set to nan. Details: \n{detail}", UserWarning)
            per = (time.perf_counter() - t0) / len(fitted)
            for b, (c, _) in enumerate(fitted):
                scores[c, s] = score[b]
                score_time[c, s] = per
        _warn_or_raise_about_fit_failures([{"fit_error": e} for row in errors for e in row], np.nan)
        self.cv_results_ = self._format_results(candidates, scores, fit_time, score_time)
        self.best_index_ = int(self.cv_results_["rank_test_score"].argmin())
        self.best_score_ = self.cv_results_["mean_test_score"][self.best_index_]
        best = self.cv_results_["params"][self.best_index_]
        self.best_params_ = {k[len(_PREFIX):]: v for k, v in best.items()}
        self.n_splits_ = n_splits
        if self.refit:
            t0 = time.perf_counter()
            est = clone(self.estimator).set_params(**clone(self.best_params_, safe=False))
            self.best_estimator_ = est._fit_from_moments(total, n_rows, dims, in_dtype)
            self.refit_time_ = time.perf_counter() - t0

    @staticmethod
    def _format_results(candidates, scores, fit_time, score_time) -> dict:
        """``cv_results_`` in sklearn's layout (GridSearchCV with ``error_score=nan`` and one metric)."""
        results: dict[str, Any] = {}
        for name, arr in (("fit_time", fit_time), ("score_time", score_time)):
            results[f"mean_{name}"] = arr.mean(axis=1)
            results[f"std_{name}"] = arr.std(axis=1)
        for key, ma in _yield_masked_array_for_each_param(candidates):
            results[key] = ma
        results["params"] = candidates
        for s in range(scores.shape[1]):
            results[f"split{s}_test_score"] = scores[:, s]
        means = np.average(scores, axis=1)
        results["mean_test_score"] = means
        if np.any(~np.isfinite(means)):
            warnings.warn(f"One or more of the test scores are non-finite: {means}", category=UserWarning)
        results["std_test_score"] = np.sqrt(np.average((scores - means[:, None]) ** 2, axis=1))
        if np.isnan(means).all():
            rank = np.ones_like(means, dtype=np.int32)
        else:
            rank = rankdata(-np.nan_to_num(means, nan=np.nanmin(means) - 1), method="min").astype(np.int32)
        results["rank_test_score"] = rank
        return results

    # ------------------------------------------------------------------ delegation
    def _check_refit(self, attr: str) -> None:
        if not self.refit:
            raise AttributeError(f"This GridSearchCV instance was initialized with `refit=False`. {attr} is available "
                                 "only after refitting on the best parameters. You can refit an estimator manually "
                                 "using the `best_params_` attribute")

    def transform(self, views):
        """``best_estimator_.transform(views)``; AttributeError when ``refit=False``."""
        self._check_refit("transform")
        return self.best_estimator_.transform(views)

    def score(self, views, y=None) -> float:
        """Mean canonical correlation of ``best_estimator_`` on ``views``; AttributeError when ``refit=False``."""
        if self._inner_cv is not None:
            return float(self._inner_cv.score(np.hstack([_host(v) for v in views]), y))
        self._check_refit("score")
        return float(np.mean(self.best_estimator_.score(views)))
