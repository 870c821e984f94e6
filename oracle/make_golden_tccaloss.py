"""Generate tests/golden/reference_outputs_tccaloss.{npz,json} from the UNMODIFIED reference: TCCALoss
(cca_zoo/deep/objectives.py:223-289), its loss and its autograd gradients in float64.

    python oracle/make_golden_tccaloss.py

TEST INFRASTRUCTURE ONLY (see make_golden.py).  The inputs are stored with the outputs.  Every case records kappa,
the largest condition number of the S_i = cov(z_i) + eps I: the gradient of a whitened objective moves by about
kappa times the rounding of its inputs, so a rank-deficient batch (kappa ~ lambda_max / eps) agrees with the
reference only to about kappa * 1e-14.  The archive is written with fixed zip timestamps: two runs give the same bytes.
"""
from __future__ import annotations

import io
import json
import os
import sys
import zipfile

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from oracle import refshim  # noqa: E402

refshim.install()

import torch  # noqa: E402
from cca_zoo.deep.objectives import TCCALoss  # noqa: E402

# name, n, widths, eps, seed
CASES = [
    ("m2", 64, [5, 4], 1e-5, 0),
    ("m3", 100, [3, 4, 5], 1e-5, 1),
    ("m3_eps6", 100, [3, 4, 5], 1e-6, 1),
    ("m4_width1", 80, [4, 1, 3, 2], 1e-5, 2),
    ("m5", 60, [3, 4, 5, 3, 4], 1e-6, 3),
    ("m8", 40, [2, 3, 2, 2, 1, 2, 3, 2], 1e-5, 4),
    ("width_crosses_64", 150, [70, 2, 3], 1e-5, 5),
    ("rank_deficient", 6, [8, 3, 4], 1e-5, 6),
]


def views(n, widths, seed):
    """Correlated representations: a shared latent plus noise (torch CPU generator, seeded)."""
    g = torch.Generator().manual_seed(seed)
    zl = torch.randn(n, 2, generator=g, dtype=torch.float64)
    return [zl @ torch.randn(2, w, generator=g, dtype=torch.float64)
            + 0.5 * torch.randn(n, w, generator=g, dtype=torch.float64) for w in widths]


def kappa(zs, eps):
    out = 1.0
    for z in zs:
        zc = z - z.mean(0)
        lam = np.linalg.eigvalsh(zc.T @ zc / (z.shape[0] - 1) + eps * np.eye(z.shape[1]))
        out = max(out, float(lam[-1] / max(lam[0], eps)))
    return out


def write_npz(path, arrays):
    with zipfile.ZipFile(path, "w", compression=zipfile.ZIP_DEFLATED) as zf:
        for name in sorted(arrays):
            buf = io.BytesIO()
            np.lib.format.write_array(buf, np.ascontiguousarray(arrays[name]), allow_pickle=False)
            info = zipfile.ZipInfo(name + ".npy", date_time=(1980, 1, 1, 0, 0, 0))
            info.compress_type = zipfile.ZIP_DEFLATED
            zf.writestr(info, buf.getvalue())


def main():
    out, meta = {}, {"cases": []}
    for name, n, widths, eps, seed in CASES:
        zs = [z.requires_grad_(True) for z in views(n, widths, seed)]
        loss = TCCALoss(eps=eps)(zs)
        loss.backward()
        for i, z in enumerate(zs):
            out[f"{name}/z{i}"] = z.detach().numpy()
            out[f"{name}/g{i}"] = z.grad.numpy()
        out[f"{name}/loss"] = np.array([loss.item()])
        meta["cases"].append(dict(name=name, n=n, widths=widths, eps=eps, seed=seed,
                                  kappa=kappa([z.detach().numpy() for z in zs], eps)))
    gdir = os.path.join(ROOT, "tests", "golden")
    write_npz(os.path.join(gdir, "reference_outputs_tccaloss.npz"), out)
    with open(os.path.join(gdir, "reference_outputs_tccaloss.json"), "w") as f:
        json.dump(meta, f, indent=1)
        f.write("\n")


if __name__ == "__main__":
    main()
