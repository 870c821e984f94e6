"""Generate tests/golden/reference_outputs_ccar3.{npz,json} from the UNMODIFIED reference: CCAR3
(cca_zoo/linear/_ccar3.py).

    python oracle/make_golden_ccar3.py

TEST INFRASTRUCTURE ONLY (see make_golden.py).  Each case records the reference's weights, held-out transform and
score, the ADMM iteration count of the restatement oracle/ccar3.py:admm_ref (checked against the reference's own
weights), and the spreads: the largest change of the weights, the held-out transform and the held-out score over
three refits with the inputs perturbed by 1e-15 (relative).  A case is kept only when a last-bit difference cannot
change its result discontinuously:
  * the stopping statistic max(primal, dual) is at least 1e-3 (relative) away from tol at the last iteration and at
    the one before it;
  * every eigenvalue of Sy is at least 1e-3 (relative) away from the 1e-4 cut;
  * the final row norms of B + U are at least 1e-6 (relative) away from lambda / rho;
  * the top r_eff + 1 singular values of B are separated by at least 1e-3 (relative to the largest).
Rerunning the script reproduces the files byte for byte.
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

from cca_zoo.linear import CCAR3 as RefCCAR3  # noqa: E402

from cca_zoo_b200.datasets import conftest_views, joint_data  # noqa: E402
from oracle import ccar3 as O  # noqa: E402

N_TEST = 40
DATASETS = {
    "two_views": ("conftest", {"name": "two_views"}),
    "correlated_views": ("conftest", {"name": "correlated_views"}),
    "p_gt_n": ("joint", dict(n_views=2, n_samples=30, n_features=[60, 5], latent_dimensions=2, signal_to_noise=2.0,
                             random_state=5)),
    "ragged": ("joint", dict(n_views=2, n_samples=2000, n_features=[700, 90], latent_dimensions=3,
                             signal_to_noise=1.0, random_state=6)),
}


def _cases():
    out = []
    for ds in ("two_views", "correlated_views"):
        for lw in (True, False):
            for lam in (0.0, 0.05, 0.3):
                out.append((f"{ds}_lam{lam:g}_lw{int(lw)}", ds, dict(latent_dimensions=2, lambda_=lam,
                                                                     ledoit_wolf=lw)))
            out.append((f"{ds}_lowdim_lw{int(lw)}", ds, dict(latent_dimensions=2, highdim=False, ledoit_wolf=lw)))
    out += [
        ("uncentred", "two_views", dict(latent_dimensions=2, center=False, lambda_=0.05)),
        ("uncentred_lowdim", "correlated_views", dict(latent_dimensions=2, center=False, highdim=False)),
        ("tight_tol", "correlated_views", dict(latent_dimensions=2, lambda_=0.05, tol=1e-8, ledoit_wolf=False)),
        ("capped", "two_views", dict(latent_dimensions=2, lambda_=0.05, max_iter=5)),
        ("padded", "two_views", dict(latent_dimensions=9, lambda_=0.0)),
        ("zero_b", "two_views", dict(latent_dimensions=2, lambda_=50.0)),
        ("p_gt_n", "p_gt_n", dict(latent_dimensions=2, lambda_=0.1)),
        ("ragged", "ragged", dict(latent_dimensions=3, lambda_=0.02)),
    ]
    return out


def build_dataset(name):
    """(train views, held-out views)."""
    kind, args = DATASETS[name]
    if kind == "conftest":
        views = conftest_views(args["name"])
        rng = np.random.default_rng(99)
        return views, [v[:N_TEST] + 0.1 * rng.standard_normal(v[:N_TEST].shape) for v in views]
    views = joint_data(**dict(args, n_samples=args["n_samples"] + N_TEST))
    return [v[:-N_TEST] for v in views], [v[-N_TEST:] for v in views]


def align(W, ref):
    """W with each component pair's sign chosen to match ref (a joint sign per column of both views)."""
    out = [w.copy() for w in W]
    for j in range(ref[0].shape[1]):
        s = np.sign(sum(float(w[:, j] @ r[:, j]) for w, r in zip(W, ref)))
        for w in out:
            w[:, j] *= s if s != 0 else 1.0
    return out


def rel_err(a, b):
    num = max(float(np.abs(x - y).max()) for x, y in zip(a, b))
    den = max(max(float(np.abs(y).max()) for y in b), 1e-300)
    return num / den


def margins(views, kw):
    """The four keep conditions of the module docstring, from the restatement's instrumented ADMM."""
    kw = dict(kw)
    k = kw.pop("latent_dimensions")
    center, lam = kw.get("center", True), kw.get("lambda_", 0.0)
    rho, tol = kw.get("rho", 1.0), kw.get("tol", 1e-4)
    X, Y = [np.asarray(v, dtype=np.float64) for v in views]
    if center:
        X, Y = X - X.mean(axis=0), Y - Y.mean(axis=0)
    n, p = X.shape
    Sy = O.ledoit_wolf_data(Y)[0] if kw.get("ledoit_wolf", True) else Y.T @ Y / n
    eig = np.linalg.eigvalsh(Sy)
    cut = float(np.min(np.abs(eig - 1e-4)) / 1e-4)
    Si = O.sqrt_inv_psd(Sy)
    stop_m, row_m = np.inf, np.inf
    if kw.get("highdim", True):
        trace = []
        B, it = O.admm_ref(X, Y @ Si, lam, rho, kw.get("max_iter", 10_000), tol, kw.get("eps", 1e-8), trace)
        for t in trace[-2:]:
            stop_m = min(stop_m, abs(max(t["primal"], t["dual"]) - tol) / tol)
        if lam > 0:
            row_m = float(np.min(np.abs(trace[-1]["rownorm"] - lam / rho)) / (lam / rho))
    else:
        B, it = np.linalg.solve(X.T @ X / n + kw.get("eps", 1e-8) * np.eye(p), X.T @ (Y @ Si) / n), 0
    gap = np.inf
    if np.any(B):
        sig = np.linalg.svd(B, compute_uv=False)
        r = min(k, *B.shape)
        top = sig[:min(r + 1, sig.size)]
        if top.size > 1:
            gap = float(np.min(-np.diff(top)) / sig[0])
    return it, dict(stop=stop_m, cut=cut, row=row_m, gap=gap)


def run_case(name, ds, kw):
    views, test = build_dataset(ds)
    ref = RefCCAR3(**kw).fit(views)
    it, m = margins(views, kw)
    w_or, _ = O.ref_ccar3_fit(views, k=kw["latent_dimensions"],
                              **{a: b for a, b in kw.items() if a != "latent_dimensions"})
    err_or = rel_err(align(w_or, ref.weights_), ref.weights_) if np.any(ref.weights_[0]) else 0.0
    tr, score = ref.transform(test), ref.score(test)
    rng = np.random.default_rng(7)
    sw = st = sc = 0.0
    for _ in range(3):
        pv = [v * (1.0 + 1e-15 * rng.standard_normal(v.shape)) for v in views]
        pr = RefCCAR3(**kw).fit(pv)
        if np.any(ref.weights_[0]):
            sw = max(sw, rel_err(align(pr.weights_, ref.weights_), ref.weights_))
            st = max(st, rel_err(align(pr.transform(test), tr), tr))
        sc = max(sc, float(np.abs(np.abs(pr.score(test)) - np.abs(score)).max()))
    ok = m["stop"] >= 1e-3 and m["cut"] >= 1e-3 and m["row"] >= 1e-6 and m["gap"] >= 1e-3 and err_or < 1e-9
    print(f"{name}: iters {it} margins stop {m['stop']:.1e} cut {m['cut']:.1e} row {m['row']:.1e} gap "
          f"{m['gap']:.1e} oracle {err_or:.1e} spread w {sw:.1e} t {st:.1e} score {sc:.1e}", "" if ok else "dropped")
    return ref, tr, score, it, dict(spread_w=sw, spread_t=st, spread_score=sc), ok


def main():
    arrays, meta = {}, {"n_test": N_TEST, "datasets": DATASETS, "cases": []}
    for name, ds, kw in _cases():
        ref, tr, score, it, spread, ok = run_case(name, ds, kw)
        if not ok:
            continue
        for i, w in enumerate(ref.weights_):
            arrays[f"{name}/w{i}"] = np.asarray(w, dtype=np.float64)
            arrays[f"{name}/mean{i}"] = np.asarray(ref.means_[i], dtype=np.float64)
            arrays[f"{name}/transform{i}"] = np.asarray(tr[i], dtype=np.float64)
        arrays[f"{name}/score"] = np.asarray(score, dtype=np.float64)
        meta["cases"].append(dict(name=name, dataset=ds, kwargs=kw, iters=int(it), **spread))
    out = os.path.join(ROOT, "tests", "golden", "reference_outputs_ccar3")
    np.savez_compressed(out + ".npz", **arrays)
    with open(out + ".json", "w") as f:
        json.dump(meta, f, indent=1, sort_keys=True)
        f.write("\n")


if __name__ == "__main__":
    main()
