"""Case table of the GridSearchCV tests: every estimator the moment route serves, with a grid of its solve parameters,
and the splitters it is run with.  Shared by the CPU tests (on the torch stand-in) and the GPU tests."""
from __future__ import annotations

import numpy as np
from sklearn.model_selection import KFold, RepeatedKFold, ShuffleSplit, TimeSeriesSplit

from cca_zoo_b200.linear import (CCA, GCCA, MCCA, PLS, PLS_ALS, ElasticCCA, ParkhomenkoCCA, SCCA_ADMM, SCCA_IPLS,
                                 SCCA_PMD, SCCA_Span, rCCA)

# name -> (estimator, param grid, number of views)
CASES = {
    "rcca_c": (rCCA(latent_dimensions=2), {"c": [0.0, 0.1, 0.5, 0.9]}, 2),
    "rcca_perview_c": (rCCA(), {"c": [[0.1, 0.5], [0.5, 0.1], 0.3]}, 2),
    "cca_k": (CCA(), {"latent_dimensions": [1, 2, 3]}, 2),
    "pls_k": (PLS(), {"latent_dimensions": [1, 2]}, 2),
    "mcca_3": (MCCA(latent_dimensions=2), {"c": [0.1, 0.5]}, 3),
    "gcca_3": (GCCA(), {"latent_dimensions": [1, 2], "c": [0.2, 0.6]}, 3),
    "pls_als": (PLS_ALS(random_state=0), {"latent_dimensions": [1, 2]}, 2),
    "pmd_tau": (SCCA_PMD(random_state=0), {"tau": [0.5, 0.9]}, 2),
    "parkhomenko": (ParkhomenkoCCA(random_state=0), {"tau": [0.01, 0.1]}, 2),
    "span": (SCCA_Span(random_state=0), {"span": [3, 6]}, 2),
    "admm": (SCCA_ADMM(random_state=0), {"tau": [0.01, 0.1]}, 2),
    "elastic_alpha": (ElasticCCA(random_state=0), {"alpha": [0.01, 0.1]}, 2),
    "ipls": (SCCA_IPLS(random_state=0), {"alpha": [0.01, 0.1]}, 2),
    "grid_list": (rCCA(), [{"c": [0.1]}, {"c": [0.5], "latent_dimensions": [2]}], 2),
}

SPLITTERS = {
    "int3": 3,
    "kfold_shuffle": KFold(4, shuffle=True, random_state=0),
    "shuffle_split": ShuffleSplit(3, test_size=0.3, random_state=0),
    "repeated_kfold": RepeatedKFold(n_splits=3, n_repeats=2, random_state=0),
    # splits that are not partitions of the rows: the search takes the generic route
    "time_series": TimeSeriesSplit(3),
    "shuffle_split_partial": ShuffleSplit(3, test_size=0.2, train_size=0.3, random_state=0),
}
NON_PARTITION = ("time_series", "shuffle_split_partial")


def views(n_views: int, n: int = 120, dims=(10, 8, 6), offset: float = 0.0, seed: int = 0, dtype=np.float64):
    """Views with two shared latent directions, so that the grid's scores differ."""
    rng = np.random.default_rng(seed)
    z = rng.standard_normal((n, 2))
    out = []
    for p in dims[:n_views]:
        out.append((z @ rng.standard_normal((2, p)) + rng.standard_normal((n, p)) + offset).astype(dtype))
    return out
