"""The CCAR3 golden cases (tests/golden/reference_outputs_ccar3.{npz,json}, oracle/make_golden_ccar3.py): their seeded
inputs, the reference's outputs and the tolerances derived from each case's spread under a 1e-15 input perturbation."""
from __future__ import annotations

import json
import os

import numpy as np

from cca_zoo_b200.datasets import conftest_views, joint_data

_DIR = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden")
with open(os.path.join(_DIR, "reference_outputs_ccar3.json")) as _f:
    META = json.load(_f)
NPZ = np.load(os.path.join(_DIR, "reference_outputs_ccar3.npz"))
CASES = {c["name"]: c for c in META["cases"]}


def inputs(name):
    """(train views, held-out views), the recipe of oracle/make_golden_ccar3.py:build_dataset."""
    kind, args = META["datasets"][CASES[name]["dataset"]]
    n_test = META["n_test"]
    if kind == "conftest":
        views = conftest_views(args["name"])
        rng = np.random.default_rng(99)
        return views, [v[:n_test] + 0.1 * rng.standard_normal(v[:n_test].shape) for v in views]
    views = joint_data(**dict(args, n_samples=args["n_samples"] + n_test))
    return [v[:-n_test] for v in views], [v[-n_test:] for v in views]


def kwargs(name):
    return dict(CASES[name]["kwargs"])


def outputs(name):
    return dict(w=[NPZ[f"{name}/w{i}"] for i in range(2)], means=[NPZ[f"{name}/mean{i}"] for i in range(2)],
                transform=[NPZ[f"{name}/transform{i}"] for i in range(2)], score=NPZ[f"{name}/score"],
                iters=CASES[name]["iters"])


def tolerance(name, key="spread_w"):
    """1000 x the case's spread, and never below 1e-10 (the float64 arithmetic of a different summation order)."""
    return max(1e3 * CASES[name][key], 1e-10)


def align(W, ref):
    """W with a joint sign per component pair (column j of both views) chosen to match ref."""
    out = [np.array(w, dtype=np.float64) for w in W]
    for j in range(ref[0].shape[1]):
        s = np.sign(sum(float(w[:, j] @ r[:, j]) for w, r in zip(out, ref)))
        for w in out:
            w[:, j] *= s if s != 0 else 1.0
    return out


def rel_err(a, b):
    num = max(float(np.abs(np.asarray(x) - np.asarray(y)).max()) for x, y in zip(a, b))
    return num / max(max(float(np.abs(np.asarray(y)).max()) for y in b), 1e-300)
