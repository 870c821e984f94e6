"""cca_zoo_b200 -- H100-native drop-in for the covariance -> eigensolve hot path of cca_zoo.

``cca_zoo_b200.linear`` mirrors ``cca_zoo.linear`` (CCA, rCCA, PLS, MCCA, GCCA, PartialCCA, GRCCA, the iterative,
gradient and tensor (TCCA) estimators and CCAR3) and
``cca_zoo_b200.deep.objectives`` mirrors ``cca_zoo.deep.objectives`` (CCALoss, MCCALoss, GCCALoss) and
``cca_zoo_b200.probabilistic`` provides ``GFA`` of ``cca_zoo.probabilistic`` and
``cca_zoo_b200.nonparametric`` provides ``KCCA``, ``KGCCA`` and ``KTCCA`` of ``cca_zoo.nonparametric`` and
``cca_zoo_b200.model_selection`` provides ``GridSearchCV`` of ``cca_zoo.model_selection``.
All arithmetic runs in hand-written sm_90a kernels (libccab200.so, include/ccab200.h).
"""
__version__ = "0.1.0"
