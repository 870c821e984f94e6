"""The KGCCA and KTCCA golden cases (tests/golden/reference_outputs_{kgcca,ktcca}.{npz,json},
oracle/make_golden_{kgcca,ktcca}.py): their seeded inputs, the reference's outputs and the tolerances set from each
case's spread."""
from __future__ import annotations

import json
import os

import numpy as np

from cca_zoo_b200.datasets import joint_data

_DIR = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden")


class Golden:
    def __init__(self, model: str):
        with open(os.path.join(_DIR, f"reference_outputs_{model}.json")) as f:
            self.meta = json.load(f)
        self.npz = np.load(os.path.join(_DIR, f"reference_outputs_{model}.npz"))
        self.cases = {c["name"]: c for c in self.meta["cases"]}

    def inputs(self, name):
        """(train views, held-out views), the recipe of the generator's build_dataset."""
        case = self.cases[name]
        args = self.meta["datasets"][case["dataset"]]
        n_test = self.meta["n_test"]
        views = joint_data(**dict(args, n_samples=args["n_samples"] + n_test))
        if case["how"] == "abs":
            views = [np.abs(v) for v in views]
        elif case["how"] == "f32":
            views = [v.astype(np.float32).astype(np.float64) for v in views]
        return [v[:-n_test] for v in views], [v[-n_test:] for v in views]

    def kwargs(self, name):
        return dict(self.cases[name]["kwargs"])

    def outputs(self, name):
        ws, i = [], 0
        while f"{name}/w{i}" in self.npz:
            ws.append(self.npz[f"{name}/w{i}"])
            i += 1
        return dict(w=ws, s=[self.npz[f"{name}/s{j}"] for j in range(len(ws))],
                    transform=self.npz[f"{name}/transform"], score=self.npz[f"{name}/score"])

    def tolerances(self, name):
        """(weights, transform, score): max(1e-9, 10 x the weight spread) and max(1e-10, 10 x the spread) of the
        training scores and the held-out transform, or of the training scores and the held-out score."""
        c = self.cases[name]
        return (max(1e-9, 10.0 * c["spread_w"]), max(1e-10, 10.0 * max(c["spread_s"], c["spread_t"])),
                max(1e-10, 10.0 * max(c["spread_s"], c["spread_score"])))


KGCCA = Golden("kgcca")
KTCCA = Golden("ktcca")
GOLDEN = {"KGCCA": KGCCA, "KTCCA": KTCCA}
