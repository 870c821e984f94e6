"""Differential fuzzing of the objectives' HOST-SIDE logic (route selection, analytic backward) against the
reference's forward + autograd.  Kernels replaced by tests/fake_ops.py.  Batches with
n - 1 <= 1.25 width (rank-deficient or barely determined batch covariance) are skipped unless --all: there the reference differentiates
through an eigendecomposition with repeated eigenvalues and its own gradient is rounding noise.
With --golden the reference's results come from tests/golden/reference_fuzz_loss.npz (recorded for seed 20240924,
200 trials by oracle/make_golden_live.py), so no reference installation is needed; that file keeps, per gradient, a
fixed sample of at most 16 rows (float32, far below the tolerances) and the Frobenius norm.

    python tools/fuzz_loss_vs_reference.py [seed] [trials] [--all] [--golden]
"""
import os
import sys
import warnings

import numpy as np
import pytest
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from tests import fake_ops  # noqa: E402
from oracle import refshim  # noqa: E402

GOLDEN = os.path.join(ROOT, "tests", "golden", "reference_fuzz_loss.npz")


def draw_trials(seed, trials, show_all=False):
    """The seeded problems, independent of any result: (kind, zs, eps, desc)."""
    g = torch.Generator().manual_seed(seed)
    rng = np.random.default_rng(seed)
    for _ in range(trials):
        kind = str(rng.choice(["CCALoss", "MCCALoss", "GCCALoss"]))
        m = 2 if kind == "CCALoss" else int(rng.integers(2, 5))
        n = int(rng.integers(4, 200))
        widths = [int(rng.integers(1, 80)) for _ in range(m)]
        if kind == "GCCALoss" or rng.random() < 0.5:
            widths = [widths[0]] * m
        eps = float(rng.choice([1e-3, 1e-4, 1e-5]))
        dt = torch.float64 if rng.random() < 0.7 else torch.float32
        lat = torch.randn(n, 3, generator=g, dtype=torch.float64)
        zs = [(lat @ torch.randn(3, w, generator=g, dtype=torch.float64) * float(rng.uniform(0, 1.5))
               + torch.randn(n, w, generator=g, dtype=torch.float64)).to(dt) for w in widths]
        # rank-deficient or barely determined batch covariance (smallest eigenvalue at the rounding level of float32)
        deficient = n - 1 <= 1.25 * (sum(widths) if kind == "GCCALoss" else max(widths))
        if deficient and not show_all:
            continue
        yield kind, zs, eps, f"{kind} n={n} widths={widths} eps={eps} {dt}"


def run(lib, kind, zs, eps):
    """(loss, gradients as float64, loss dtype name, loss dim), or the name of the exception raised."""
    zz = [z.clone().requires_grad_(True) for z in zs]
    try:
        with warnings.catch_warnings():
            warnings.simplefilter("ignore")
            loss = getattr(lib, kind)(eps=eps)(zz)
            loss.backward()
        return loss.item(), [z.grad.double().numpy() for z in zz], str(loss.dtype), loss.dim()
    except Exception as e:  # noqa: BLE001
        return type(e).__name__


def sample_rows(n):
    return np.unique(np.linspace(0, n - 1, min(n, 16)).astype(int))


def digest(grads):
    """(sampled rows, Frobenius norms) of the gradients, as stored in the golden file."""
    return [g[sample_rows(g.shape[0])] for g in grads], [float(np.linalg.norm(g)) for g in grads]


def record(seed, trials):
    refshim.install()
    from cca_zoo.deep import objectives as ref

    out = {}
    for i, (kind, zs, eps, _) in enumerate(draw_trials(seed, trials)):
        res = run(ref, kind, zs, eps)
        if isinstance(res, str):
            out[f"{i}/exception"] = np.array(res)
            continue
        out[f"{i}/loss"], out[f"{i}/dtype"], out[f"{i}/dim"] = np.array(res[0]), np.array(res[2]), np.array(res[3])
        rows, norms = digest(res[1])
        for j, (gr, nr) in enumerate(zip(rows, norms)):
            out[f"{i}/grad{j}"], out[f"{i}/gradnorm{j}"] = gr.astype(np.float32), np.array(nr)
    return out


def from_arrays(i, npz):
    if f"{i}/exception" in npz:
        return str(npz[f"{i}/exception"])
    grads, norms, j = [], [], 0
    while f"{i}/grad{j}" in npz:
        grads.append(npz[f"{i}/grad{j}"].astype(np.float64))
        norms.append(float(npz[f"{i}/gradnorm{j}"]))
        j += 1
    return float(npz[f"{i}/loss"]), (grads, norms), str(npz[f"{i}/dtype"]), int(npz[f"{i}/dim"])


def main():
    args = [a for a in sys.argv[1:] if not a.startswith("--")]
    seed = int(args[0]) if args else 0
    trials = int(args[1]) if len(args) > 1 else 200
    show_all = "--all" in sys.argv
    golden = np.load(GOLDEN) if "--golden" in sys.argv else None
    if golden is None:
        refshim.install()
        from cca_zoo.deep import objectives as ref
    fake_ops.install(pytest.MonkeyPatch())
    from cca_zoo_b200.deep import objectives as ours

    bad = 0
    for i, (kind, zs, eps, desc) in enumerate(draw_trials(seed, trials, show_all)):
        r = from_arrays(i, golden) if golden is not None else run(ref, kind, zs, eps)
        o = run(ours, kind, zs, eps)
        if isinstance(r, str) or isinstance(o, str):
            if r != o:
                bad += 1
                print("EXCEPTION", desc, "| ref", r, "| ours", o if isinstance(o, str) else "no exception")
            continue
        tol = 5e-3 if zs[0].dtype == torch.float32 else 1e-7
        dl = abs(r[0] - o[0]) / max(abs(r[0]), 1e-300)
        if golden is not None:    # the stored digest: sampled rows and norms
            (rg, rn), (og, on) = r[1], digest(o[1])
            dg = max(max(np.abs(a - b).max() / max(np.abs(a).max(), 1e-300) for a, b in zip(rg, og)),
                     max(abs(a - b) / max(a, 1e-300) for a, b in zip(rn, on)))
        else:
            dg = max(np.abs(a - b).max() / max(np.abs(a).max(), 1e-300) for a, b in zip(r[1], o[1]))
        if not (dl < tol and dg < 50 * tol) or r[2:] != o[2:]:
            bad += 1
            print(f"VALUES loss {dl:.1e} grad {dg:.1e} dtype/dim {r[2:]} {o[2:]}", desc)
    print(f"seed {seed}: {trials} trials, {bad} mismatches")
    return 1 if bad else 0


if __name__ == "__main__":
    sys.exit(main())
