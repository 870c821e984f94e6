"""Differential fuzzing of the HOST-SIDE logic against the reference: random shapes, ridge values, centring flags, view weights, confounds, feature groups, dtypes.
The kernels are replaced by tests/fake_ops.py (torch CPU), so every mismatch is a divergence of the Python between
the kernels from the reference's behaviour.  Ill-posed draws (c = 0 with a rank-deficient or under-determined view,
where the reference itself returns noise-dependent output) are reported only with --all.
With --golden the reference's results come from tests/golden/reference_fuzz.npz (recorded for seed 20240924,
200 trials by oracle/make_golden_live.py), so no reference installation is needed.

    python tools/fuzz_vs_reference.py [seed] [trials] [--all] [--medium] [--golden]
"""
import os
import sys
import warnings

import numpy as np
import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from tests import fake_ops  # noqa: E402  (before refshim: the reference has its own `tests` package)
from oracle import refshim  # noqa: E402
from oracle import restatement as R  # noqa: E402

GOLDEN = os.path.join(ROOT, "tests", "golden", "reference_fuzz.npz")


def draw_trials(seed, trials, medium=False):
    """The seeded problems, independent of any result: (model, views, kw, ours_kw, extra, facts)."""
    rng = np.random.default_rng(seed)
    for _ in range(trials):
        model = str(rng.choice(["CCA", "rCCA", "PLS", "MCCA", "GCCA", "PartialCCA", "GRCCA"]))
        m = 2 if model in ("CCA", "rCCA", "PLS") else int(rng.integers(2, 5))
        n = int(rng.integers(6, 120))
        dims = [int(rng.integers(1, 30)) for _ in range(m)]
        k = int(rng.integers(1, 8))
        if medium:
            n = int(rng.integers(300, 700))
            dims = [int(rng.integers(36, 110)) for _ in range(m)]
        lat = rng.standard_normal((n, 3))
        views = [lat @ rng.standard_normal((3, d)) * rng.uniform(0, 1.5) + rng.standard_normal((n, d))
                 + rng.uniform(-1, 1) for d in dims]
        dup = rng.random() < 0.15
        if dup:
            j = int(rng.integers(0, m))
            views[j] = np.hstack([views[j], views[j][:, :1]])
            dims[j] += 1
        f32 = rng.random() < 0.25
        if f32:
            views = [v.astype(np.float32) for v in views]
        kw = dict(latent_dimensions=k, center=bool(rng.random() < 0.75))
        c = 0.0
        if model not in ("CCA", "PLS"):
            c = float(rng.choice([0.0, 0.0, 0.1, 0.5, 1.0])) if rng.random() < 0.7 else \
                [float(rng.uniform(0, 1)) for _ in range(m)]
            kw["c"] = c
        extra = {}
        ours_kw = {}
        if medium and model not in ("CCA", "PLS"):
            ours_kw["solver"] = str(rng.choice(["auto", "eigen", "cholesky"]))
        if model == "GCCA" and rng.random() < 0.5:
            kw["view_weights"] = [float(rng.uniform(0.5, 2)) for _ in range(m)]
        if model == "MCCA":
            kw["pca"] = bool(rng.random() < 0.5)
        if model == "PartialCCA":
            extra["partials"] = rng.standard_normal((n, int(rng.integers(1, 4)))) + 0.3
        if model == "GRCCA":
            kw["mu"] = float(rng.choice([0.0, 0.5, 2.0]))
            extra["feature_groups"] = [rng.integers(0, 3, size=d) for d in dims]
        cmin = 1.0 if model == "PLS" else (min(c) if isinstance(c, list) else c)
        q = extra["partials"].shape[1] if "partials" in extra else 0
        determined = (not dup) and n - 2 - q > sum(dims)     # else exact correlation-1 ties (degenerate top eigenspace)
        # c = 0 needs full-rank blocks; GCCA takes pinv(view) whatever c is; float32 inputs of an under-determined
        # problem amplify the reference's own float32 rounding (centring and pinv run in float32 there)
        well = determined or (cmin > 0 and model != "GCCA" and not f32)
        facts = dict(n=n, dims=dims, q=q, f32=f32, well=well,
                     desc=f"{'well ' if well else 'ILL  '}{model} n={n} dims={dims} f32={f32} {kw} {ours_kw}")
        yield model, views, kw, ours_kw, extra, facts


def run(lib, model, views, kw, extra):
    """What a caller sees: (weights_, means_, score, transform of the held-out half, pairwise correlations), or the
    name of the exception the fit raised."""
    try:
        with warnings.catch_warnings():
            warnings.simplefilter("ignore")
            est = getattr(lib, model)(**kw).fit(views, **extra)
            held = [v[: views[0].shape[0] // 2] for v in views]
            return dict(weights=list(est.weights_), means=[np.asarray(m) for m in est.means_],
                        score=np.asarray(est.score(views)), transform=[np.asarray(t) for t in est.transform(held)],
                        pairwise=np.asarray(est.pairwise_correlations(held)))
    except Exception as e:  # noqa: BLE001
        return type(e).__name__


def to_arrays(i, res, out):
    """Flatten one reference result into npz entries under trial index i."""
    if isinstance(res, str):
        out[f"{i}/exception"] = np.array(res)
        return
    for key in ("weights", "means", "transform"):
        for j, a in enumerate(res[key]):
            out[f"{i}/{key}{j}"] = a
    out[f"{i}/score"], out[f"{i}/pairwise"] = res["score"], res["pairwise"]


def from_arrays(i, npz):
    if f"{i}/exception" in npz:
        return str(npz[f"{i}/exception"])
    if f"{i}/score" not in npz:
        return None    # ill-posed trial that did not raise: only its exception behaviour is compared
    res = {"score": npz[f"{i}/score"], "pairwise": npz[f"{i}/pairwise"]}
    for key in ("weights", "means", "transform"):
        res[key], j = [], 0
        while f"{i}/{key}{j}" in npz:
            res[key].append(npz[f"{i}/{key}{j}"])
            j += 1
    return res


def compare(r, o, facts, show_all=False):
    """None if ours matches the reference's result r, else a description of the mismatch."""
    desc = facts["desc"]
    if isinstance(r, str) or isinstance(o, str):
        return None if r == o else f"EXCEPTION {desc} | ref: {r} | ours: {o if isinstance(o, str) else 'no exception'}"
    if r is None or (not facts["well"] and not show_all):
        return None
    if [w.shape for w in r["weights"]] != [w.shape for w in o["weights"]]:
        return f"WEIGHT SHAPES {desc} {[w.shape for w in r['weights']]} {[w.shape for w in o['weights']]}"
    dt_r = [w.dtype for w in r["weights"]] + [t.dtype for t in r["transform"]]
    dt_o = [w.dtype for w in o["weights"]] + [t.dtype for t in o["transform"]]
    if dt_r != dt_o:
        return f"DTYPES {desc} {dt_r} {dt_o}"
    tol = 2e-3 if facts["f32"] else 1e-6
    kmax = min(min(facts["dims"]), max(facts["n"] - 2 - facts["q"], 0))
    d_score = float(np.max(np.abs(r["score"] - o["score"])[np.arange(r["score"].shape[0]) < max(kmax, 1)]))
    # weights / variates only for components that are determined: inside the rank of the problem, clearly
    # correlated, and separated from both neighbours (sign-aligned per component)
    sc = r["score"]
    left = np.abs(np.diff(np.concatenate([[2.0], sc])))
    right = np.abs(np.diff(np.concatenate([sc, [-2.0]])))
    simple = (left > 1e-3) & (right > 1e-3) & (np.abs(sc) > 1e-3) & (np.arange(sc.shape[0]) < kmax)
    w_r = [np.asarray(w, dtype=np.float64) for w in r["weights"]]
    w_o = R.align_signs([np.asarray(w, dtype=np.float64) for w in o["weights"]], w_r)
    d_w = 0.0
    for a, b in zip(w_o, w_r):
        num = np.linalg.norm(a - b, axis=0)[simple]
        den = np.linalg.norm(b, axis=0)[simple]
        if num.size:
            d_w = max(d_w, float(np.max(num / np.maximum(den, 1e-300))))
    d_means = max(float(np.max(np.abs(np.asarray(a, dtype=np.float64) - np.asarray(b, dtype=np.float64))))
                  for a, b in zip(r["means"], o["means"]))
    d_pair = float(np.max(np.abs(r["pairwise"][..., simple] - o["pairwise"][..., simple]))) if simple.any() else 0.0
    if not (d_score < tol and d_w < 50 * tol and d_means < 1e-5 and d_pair < 50 * tol):
        return f"VALUES score {d_score:.1e} weights {d_w:.1e} means {d_means:.1e} pairwise {d_pair:.1e} {desc}"
    return None


def record(seed, trials):
    """The reference's results for the seeded problems (well-posed trials in full, the others by exception only)."""
    refshim.install()
    import cca_zoo.linear as ref

    out = {}
    for i, (model, views, kw, _, extra, facts) in enumerate(draw_trials(seed, trials)):
        res = run(ref, model, views, kw, extra)
        if isinstance(res, str) or facts["well"]:
            to_arrays(i, res, out)
    return out


def main():
    args = [a for a in sys.argv[1:] if not a.startswith("--")]
    seed = int(args[0]) if args else 0
    trials = int(args[1]) if len(args) > 1 else 300
    show_all = "--all" in sys.argv
    medium = "--medium" in sys.argv        # wider views, explicit solver routes (top-k route needs 4k <= width)
    golden = np.load(GOLDEN) if "--golden" in sys.argv else None
    if golden is None:
        refshim.install()
        import cca_zoo.linear as ref
    fake_ops.install(pytest.MonkeyPatch())
    from cca_zoo_b200 import linear as ours

    bad = 0
    for i, (model, views, kw, ours_kw, extra, facts) in enumerate(draw_trials(seed, trials, medium)):
        r = from_arrays(i, golden) if golden is not None else run(ref, model, views, kw, extra)
        o = run(ours, model, views, {**kw, **ours_kw}, extra)
        msg = compare(r, o, facts, show_all)
        if msg:
            bad += 1
            print(msg)
    print(f"seed {seed}: {trials} trials, {bad} mismatches")
    return 1 if bad else 0


if __name__ == "__main__":
    sys.exit(main())
