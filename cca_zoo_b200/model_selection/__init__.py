"""Model selection for the multiview estimators, at the reference's import path ``cca_zoo.model_selection``.

``GridSearchCV`` cross-validates a parameter grid.  For the estimators fitted from the block moments (rCCA, CCA, PLS,
MCCA, GCCA and the iterative estimators of ``cca_zoo_b200.linear``) it reads the data once for the moments of all rows
and once for each split's test rows, fits every candidate from the moments and scores all candidates of a split in one
device call; any other estimator is searched through ``sklearn.model_selection.GridSearchCV`` as in the reference."""
from ._search import GridSearchCV

__all__ = ["GridSearchCV"]
