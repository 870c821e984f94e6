"""The TCCA golden cases (tests/golden/reference_outputs_tcca.{npz,json}, oracle/make_golden_tcca.py): their seeded
inputs and the reference's outputs."""
from __future__ import annotations

import json
import os

import numpy as np

from cca_zoo_b200.datasets import conftest_views, joint_data

_DIR = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden")
with open(os.path.join(_DIR, "reference_outputs_tcca.json")) as _f:
    META = json.load(_f)
NPZ = np.load(os.path.join(_DIR, "reference_outputs_tcca.npz"))
CASES = {c["name"]: c for c in META["cases"]}


def inputs(name):
    """(train views, held-out views), the recipe of oracle/make_golden_tcca.py:build_dataset."""
    kind, args = META["datasets"][CASES[name]["dataset"]]
    n_test = META["n_test"]
    if kind == "conftest":
        views = conftest_views(args["name"])
        rng = np.random.default_rng(99)
        return views, [v[:n_test] + 0.1 * rng.standard_normal(v[:n_test].shape) for v in views]
    if kind == "rankdef":
        rng = np.random.default_rng(args["seed"])
        n = args["n"] + n_test
        z = rng.standard_normal((n, 1))
        a = z @ rng.standard_normal((1, 4)) + rng.standard_normal((n, 4))
        b = z @ rng.standard_normal((1, 3)) + rng.standard_normal((n, 3))
        c = z @ rng.standard_normal((1, 2)) + rng.standard_normal((n, 2))
        views = [a, b, np.hstack([c, c[:, :1] + c[:, 1:]])]
    else:
        views = joint_data(**dict(args, n_samples=args["n_samples"] + n_test))
    return [v[:-n_test] for v in views], [v[-n_test:] for v in views]


def kwargs(name):
    return dict(CASES[name]["kwargs"])


def outputs(name):
    ws, i = [], 0
    while f"{name}/w{i}" in NPZ:
        ws.append(NPZ[f"{name}/w{i}"])
        i += 1
    return dict(w=ws, means=[NPZ[f"{name}/mean{j}"] for j in range(len(ws))], rec=NPZ[f"{name}/rec"],
                iters=CASES[name]["iters"], stop=CASES[name]["stop"], transform=NPZ[f"{name}/transform"],
                score=NPZ[f"{name}/score"])
