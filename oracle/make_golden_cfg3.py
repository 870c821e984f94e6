"""Generate tests/golden/reference_outputs_cfg3.npz: the reference's CCALoss / MCCALoss value and autograd
gradients at BASELINE config 3 (batch 4096; widths 64, 512, a ragged pair, and a 3-view MCCALoss).

    python oracle/make_golden_cfg3.py          (authoring container only: needs /root/reference)

TEST INFRASTRUCTURE ONLY.  The objective is evaluated by the UNMODIFIED reference
(cca_zoo/deep/objectives.py:61-102,138-153) in float64 on seeded inputs; the fixtures travel to the GPU
box, the reference does not.  A full gradient at 4096 x 512 is 16 MB per view, so each gradient is stored as
  * every 64th row (element-wise comparison),
  * its Frobenius norm,
  * two projections  g^T r  and  g c  onto seeded probe vectors r (batch) and c (width), which see every entry.
The input recipe (SURVEY.md §8d, config 3) is rebuilt by tests/golden_io.py:cfg3_inputs.
"""
from __future__ import annotations

import json
import os
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from oracle import refshim  # noqa: E402

refshim.install()

import torch  # noqa: E402
from cca_zoo.deep.objectives import CCALoss, MCCALoss  # noqa: E402

ROW_STRIDE = 64

CASES = [
    # (name, kind, batch, widths, eps, seed)
    ("cfg3_4096x64", "cca", 4096, [64, 64], 1e-5, 0),
    ("cfg3_4096x512", "cca", 4096, [512, 512], 1e-5, 0),
    ("cfg3_4096x96x160", "cca", 4096, [96, 160], 1e-5, 1),
    ("cfg3_4096x256x200", "cca", 4096, [256, 200], 1e-5, 2),
    ("cfg3_m4096x64x3", "mcca", 4096, [64, 64, 64], 1e-5, 3),
]


def cfg3_inputs(batch, widths, seed):
    """z_i = z_l A_i + eps_i with z_l ~ N(0, I_16), A_i ~ N(0,1)^{16 x w}, eps ~ N(0, 1) (torch CPU generator)."""
    g = torch.Generator().manual_seed(seed)
    zl = torch.randn(batch, 16, generator=g, dtype=torch.float64)
    out = []
    for w in widths:
        a = torch.randn(16, w, generator=g, dtype=torch.float64)
        out.append(zl @ a + torch.randn(batch, w, generator=g, dtype=torch.float64))
    return out


def probes(batch, width, seed):
    rng = np.random.default_rng(10_000 + seed)
    return rng.standard_normal(batch), rng.standard_normal(width)


def main():
    out, meta = {}, {"row_stride": ROW_STRIDE, "cases": []}
    for name, kind, batch, widths, eps, seed in CASES:
        zs = [z.clone().requires_grad_(True) for z in cfg3_inputs(batch, widths, seed)]
        fn = CCALoss(eps=eps) if kind == "cca" else MCCALoss(eps=eps)
        loss = fn(zs)
        loss.backward()
        out[f"{name}/loss"] = np.array(loss.item())
        for i, z in enumerate(zs):
            g = z.grad.numpy()
            r, c = probes(batch, widths[i], seed + i)
            out[f"{name}/grad{i}_rows"] = g[::ROW_STRIDE].copy()
            out[f"{name}/grad{i}_fro"] = np.array(np.linalg.norm(g))
            out[f"{name}/grad{i}_tr"] = g.T @ r
            out[f"{name}/grad{i}_c"] = g @ c
        meta["cases"].append(dict(name=name, kind=kind, batch=batch, widths=widths, eps=eps, seed=seed))
        print(name, loss.item())
    gdir = os.path.join(ROOT, "tests", "golden")
    # the large float64 arrays keep 30 of their 52 mantissa bits (relative rounding <= 1e-9, far below every tolerance
    # they are checked with), which keeps the compressed file under 1 MB
    out = {k: (v.view(np.uint64) & ~np.uint64((1 << 22) - 1)).view(np.float64)
           if v.dtype == np.float64 and v.nbytes >= 16384 else v for k, v in out.items()}
    np.savez_compressed(os.path.join(gdir, "reference_outputs_cfg3.npz"), **out)
    with open(os.path.join(gdir, "reference_outputs_cfg3.json"), "w") as f:
        json.dump(meta, f, indent=1)
    print("wrote", len(out), "arrays")


if __name__ == "__main__":
    main()
