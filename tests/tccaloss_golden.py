"""The TCCALoss golden cases (tests/golden/reference_outputs_tccaloss.{npz,json}, oracle/make_golden_tccaloss.py):
inputs, the reference's float64 loss and gradients, and the tolerance each case's conditioning allows."""
from __future__ import annotations

import json
import os

import numpy as np

_DIR = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden")
with open(os.path.join(_DIR, "reference_outputs_tccaloss.json")) as _f:
    CASES = {c["name"]: c for c in json.load(_f)["cases"]}
_NPZ = np.load(os.path.join(_DIR, "reference_outputs_tccaloss.npz"))


def inputs(name):
    return [_NPZ[f"{name}/z{i}"] for i in range(len(CASES[name]["widths"]))]


def outputs(name):
    """(loss, [dL/dz_i]) of the reference's autograd."""
    return float(_NPZ[f"{name}/loss"][0]), [_NPZ[f"{name}/g{i}"] for i in range(len(CASES[name]["widths"]))]


def tol64(name):
    """1e-10 relative, widened to kappa * 1e-14 where S_i is ill-conditioned (the rank-deficient case)."""
    return max(1e-10, 1e-14 * CASES[name]["kappa"])


def rel_err(got, want):
    """Largest error relative to the largest entry of the reference, over all gradients."""
    return max(float(np.abs(g - w).max() / np.abs(w).max()) for g, w in zip(got, want))
