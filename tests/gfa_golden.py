"""The GFA golden cases (tests/golden/reference_outputs_gfa.{npz,json}, oracle/make_golden_gfa.py): their seeded
inputs and the reference's outputs."""
from __future__ import annotations

import json
import os

import numpy as np

from cca_zoo_b200.datasets import conftest_views, joint_data

_DIR = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden")
with open(os.path.join(_DIR, "reference_outputs_gfa.json")) as _f:
    META = json.load(_f)
NPZ = np.load(os.path.join(_DIR, "reference_outputs_gfa.npz"))
CASES = {c["name"]: c for c in META["cases"]}


def inputs(name):
    """(train views, held-out views), the recipe of oracle/make_golden_gfa.py:build_dataset."""
    kind, args = META["datasets"][CASES[name]["dataset"]]
    n_test = META["n_test"]
    if kind == "conftest":
        views = conftest_views(args["name"])
        rng = np.random.default_rng(99)
        return views, [v + 0.1 * rng.standard_normal(v.shape) for v in views]
    if kind == "private":
        rng = np.random.default_rng(args["seed"])
        n = args["n"] + n_test
        zs, zp = rng.standard_normal((n, 1)), rng.standard_normal((n, 1))
        y1 = zs @ rng.standard_normal((1, 5)) + zp @ rng.standard_normal((1, 5)) + 0.1 * rng.standard_normal((n, 5))
        y2 = zs @ rng.standard_normal((1, 4)) + 0.1 * rng.standard_normal((n, 4))
        views = [y1, y2]
    else:
        views = joint_data(**dict(args, n_samples=args["n_samples"] + n_test))
    return [v[:-n_test] for v in views], [v[-n_test:] for v in views]


def outputs(name):
    ws, i = [], 0
    while f"{name}/w{i}" in NPZ:
        ws.append(NPZ[f"{name}/w{i}"])
        i += 1
    post = {k.split("/post/")[1]: NPZ[k] for k in NPZ.files if k.startswith(f"{name}/post/")}
    return dict(w=ws, means=[NPZ[f"{name}/mean{j}"] for j in range(len(ws))],
                view_relevance=NPZ[f"{name}/view_relevance"], n_iter=int(NPZ[f"{name}/n_iter"][0]),
                n_components=int(NPZ[f"{name}/n_components"][0]), post=post, transform=NPZ[f"{name}/transform"],
                score=NPZ[f"{name}/score"], log_likelihood=float(NPZ[f"{name}/log_likelihood"][0]),
                loadings0=NPZ[f"{name}/loadings0"])
