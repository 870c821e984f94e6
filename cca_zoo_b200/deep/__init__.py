"""Deep-CCA correlation objectives on the hot path (mirrors ``cca_zoo.deep.objectives``)."""
from .objectives import CCALoss, GCCALoss, MCCALoss, TCCALoss

__all__ = ["CCALoss", "MCCALoss", "GCCALoss", "TCCALoss"]
