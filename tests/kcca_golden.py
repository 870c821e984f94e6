"""The KCCA golden cases (tests/golden/reference_outputs_kcca.{npz,json}, oracle/make_golden_kcca.py): their seeded
inputs, the reference's outputs and the tolerances set from each case's spread."""
from __future__ import annotations

import json
import os

import numpy as np

from cca_zoo_b200.datasets import joint_data

_DIR = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden")
with open(os.path.join(_DIR, "reference_outputs_kcca.json")) as _f:
    META = json.load(_f)
NPZ = np.load(os.path.join(_DIR, "reference_outputs_kcca.npz"))
CASES = {c["name"]: c for c in META["cases"]}


def inputs(name):
    """(train views, held-out views), the recipe of oracle/make_golden_kcca.py:build_dataset."""
    case = CASES[name]
    args = META["datasets"][case["dataset"]]
    n_test = META["n_test"]
    views = joint_data(**dict(args, n_samples=args["n_samples"] + n_test))
    if case["how"] == "abs":
        views = [np.abs(v) for v in views]
    elif case["how"] == "f32":
        views = [v.astype(np.float32).astype(np.float64) for v in views]
    return [v[:-n_test] for v in views], [v[-n_test:] for v in views]


def kwargs(name):
    return dict(CASES[name]["kwargs"])


def outputs(name):
    ws, i = [], 0
    while f"{name}/w{i}" in NPZ:
        ws.append(NPZ[f"{name}/w{i}"])
        i += 1
    return dict(w=ws, s=[NPZ[f"{name}/s{j}"] for j in range(len(ws))], transform=NPZ[f"{name}/transform"],
                score=NPZ[f"{name}/score"])


def tolerances(name):
    """(weights, scores): max(1e-9, 10 x the weight spread) and max(1e-10, 10 x the score spread)."""
    return max(1e-9, 10.0 * CASES[name]["spread_w"]), max(1e-10, 10.0 * CASES[name]["spread_s"])
