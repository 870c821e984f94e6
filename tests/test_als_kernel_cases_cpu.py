"""The reference half of tests/test_als_kernel_gpu.py on the CPU: from the trace of the float64 restatement, every
case of tests/als_kernel_cases.py must keep a margin at each discrete decision the ALS kernel takes (or sit exactly on
it by construction), its weights must move, and the table must reach every branch it is there for.  A case whose
comparison could flip between the device and numpy fails here rather than on the GPU."""
import numpy as np
import pytest

from oracle import sparse as S
from tests import als_kernel_cases as K

ALL = list(K.CASES.values())
MARGIN = 1e-8          # relative margin of every support / side decision
GUARD = 1e-6           # a 1e-12 guard value is 0 or above this fraction of its scale
EIG_GAP = 1e3          # kept and dropped eigenvalues stay this factor away from the cut


def _updates(trace):
    return [(d, u) for d, rec in enumerate(trace) for u in rec["updates"]]


def _exact_ties(case):
    return case.gen in ("span_tie", "span_zero")


def margins(case):
    """Every decision of the case's trace against its margin; returns the list of violations (empty for a good
    case)."""
    W, iters, trace = K.reference(case)
    init = K.inputs(case)[1]
    bad = []
    sl = S.block_slices(case.dims)
    for d, rec in enumerate(trace):
        sg = np.sqrt(rec["gmax"])
        for x in rec["deltas"]:
            if case.tol > 0 and abs(x - case.tol) < 1e-3 * case.tol:
                bad.append(f"dim {d}: delta {x} within 1e-3 of tol")
        for i, s in enumerate(rec["s"]):
            wn = float(W[sl[i], d] @ W[sl[i], d])
            if s != 0.0 and s <= GUARD * rec["gmax"] * wn:
                bad.append(f"dim {d} view {i}: deflation s {s}")
        for u in rec["updates"]:
            at = f"dim {d} sweep {u['sweep']} view {u['view']}"
            tau = case.params[u["view"]]
            if u["tn"] != 0.0 and u["tn"] <= GUARD * sg:
                bad.append(f"{at}: ||t|| {u['tn']}")
            if "norm" in u and u["norm"] != 0.0 and u["norm"] <= GUARD * sg:
                bad.append(f"{at}: norm {u['norm']}")
            if case.kind == "parkhomenko" and u["tau_gap"] < MARGIN * tau:
                bad.append(f"{at}: tau gap {u['tau_gap']}")
            if case.kind == "pmd":
                if abs(u["l1"] - u["bound"]) < MARGIN * u["bound"]:
                    bad.append(f"{at}: l1 {u['l1']} at the bound {u['bound']}")
                if "thr" in u and u["tau_gap"] < MARGIN * u["thr"]:
                    bad.append(f"{at}: bisection threshold gap {u['tau_gap']}")
            if case.kind == "span" and "gap" in u:
                if _exact_ties(case):
                    if not (np.array_equal(u["raw"], np.round(u["raw"])) and np.array_equal(init, np.round(init))):
                        bad.append(f"{at}: a designed tie on non-integer data")
                elif u["gap"] < MARGIN * u["thr"]:
                    bad.append(f"{at}: span gap {u['gap']}")
            if case.kind == "admm":
                if abs(u["zn"] - 1.0) < MARGIN:
                    bad.append(f"{at}: ||z|| {u['zn']} at 1")
                if u["tau_gap"] < MARGIN * tau / K.device_mu(case):
                    bad.append(f"{at}: tau gap {u['tau_gap']}")
            if "cut" in u:
                if u["kept_min"] < EIG_GAP * u["cut"] or u["dropped_max"] > u["cut"] / EIG_GAP:
                    bad.append(f"{at}: eigenvalues {u['kept_min']} / {u['dropped_max']} near the cut {u['cut']}")
            if "kkt" in u:
                sweeps = len(u["kkt"]) - 1
                if u["kkt"][-1] > u["kkt_tol"]:
                    if u["kkt"][-1] < 10 * u["kkt_tol"]:
                        bad.append(f"{at}: capped descent at KKT residual {u['kkt'][-1]}")
                else:
                    if sweeps > 500:
                        bad.append(f"{at}: descent converged in {sweeps} sweeps")
            if "sd" in u and u["sd"] != 0.0 and u["sd"] <= GUARD:
                bad.append(f"{at}: std {u['sd']}")
    return bad


@pytest.mark.parametrize("case", ALL, ids=lambda c: c.name)
def test_als_kernel_case_keeps_its_margins(case):
    W, iters, trace = K.reference(case)
    G, init, _ = K.inputs(case)
    assert G.shape == (case.D, case.D) and np.array_equal(G, G.T) and init.shape == (case.k, case.D)
    assert np.array_equal(G / (case.n - 1) * (case.n - 1), G), "G / (n - 1) does not round-trip"
    assert np.isfinite(W).all() and len(trace) == case.k
    bad = margins(case)
    assert not bad, f"{case.name}: " + "; ".join(bad[:10])
    if case.max_iter == 0:
        assert np.array_equal(W, init.T) and iters == [0] * case.k
        return
    assert np.linalg.norm(W - init.T) > 1e-3 * np.linalg.norm(init), "the weights barely move"
    if case.tol > 0:
        assert all(0 < abs(it) < case.max_iter for it in iters), f"{case.name} does not converge: {iters}"
    else:
        assert [abs(it) for it in iters] == [case.max_iter] * case.k


def _reached(case):
    """The branches the case's trace reaches."""
    _, _, trace = K.reference(case)
    ups = [u for _, u in _updates(trace)]
    out = set()
    if any(u["tn"] == 0.0 for u in ups):
        out.add("tn0")
    if any(u.get("norm") == 0.0 for u in ups):
        out.add("norm0")
    if any(s == 0.0 for rec in trace[:-1] for s in rec["s"]):
        out.add("s0")
    if case.kind == "pmd":
        if any(u["l1"] <= u["bound"] for u in ups):
            out.add("pmd_nobisect")
        if any("thr" in u for u in ups):
            out.add("pmd_bisect")
    if case.kind == "span":
        if any(u.get("gap") == 0.0 and u["thr"] > 0 for u in ups):
            out.add("span_tie")
        if any(u.get("thr") == 0.0 for u in ups):
            out.add("span_thr0")
        if any("gap" not in u for u in ups):
            out.add("span_all")
    if case.kind == "admm":
        if any(u["zn"] > 1 for u in ups):
            out.add("zn_above")
        if any(u["zn"] <= 1 for u in ups):
            out.add("zn_below")
    if any(u.get("dropped_max", -np.inf) > -np.inf for u in ups):
        out.add("eig_cut")
    if any("kkt" in u for u in ups) and any("cut" in u for u in ups):
        out.add("eig_and_cd")
    if any(u.get("sd") == 0.0 for u in ups):
        out.add("sd0")
    if case.gen == "data" and case.kind == "ipls" and case.k > 1:
        out.add("means")
    if any("kkt" in u and u["kkt"][-1] > u["kkt_tol"] for u in ups):
        out.add("capped")
    if not case.reg and case.D > K.WARPS_PER_SM[False] * K.SMS_H100:
        out.add("wrap")
    if case.reg and case.D > K.WARPS_PER_SM[True] * K.SMS_H100:
        out.add("wrap")
    return out


@pytest.mark.parametrize("case", [c for c in ALL if c.tags], ids=lambda c: c.name)
def test_als_kernel_case_reaches_its_branches(case):
    assert set(case.tags) <= _reached(case), f"{case.name}: {set(case.tags) - _reached(case)} not reached"


def test_als_kernel_cases_cover_the_table():
    cases = ALL
    for kind in K.KINDS:
        mine = [c for c in cases if c.kind == kind]
        assert {len(c.dims) for c in mine} >= {2, 3} and {c.k for c in mine} >= {1, 3}
        assert {0, 1, 2} <= {c.max_iter for c in mine if c.tol == 0} and max(c.max_iter for c in mine) >= 20
        assert any(c.tol > 0 for c in mine), kind
    widths = {p for c in cases for p in c.dims}
    assert {1, 32, 33, 64, 65, 96, 97, 127, 128, 129, 255, 257} <= widths
    m8 = [c for c in cases if len(c.dims) == 8]
    assert any(not c.reg for c in m8) and any(c.reg for c in m8)
    assert all(c.k < min(c.dims) or c.k == 1 for c in cases)
    # the wrap cases: the full pass and a Gauss-Seidel phase (rows of view i and of view i - 1) exceed the warps of an
    # H100 SXM grid; the two non-regression ones are one cheap kind and one thresholding kind
    wrap = [c for c in cases if "wrap" in c.tags]
    assert {c.kind for c in wrap} == {"pls", "span", "ipls"}
    for c in wrap:
        warps = K.WARPS_PER_SM[c.reg] * K.SMS_H100
        assert c.D > warps and max(c.dims[i] + c.dims[i - 1] for i in range(len(c.dims))) > warps
        assert not c.reg or max(c.dims) == 2048
    reached = set().union(*(_reached(c) for c in cases))
    assert {"tn0", "norm0", "s0", "pmd_nobisect", "pmd_bisect", "span_tie", "span_thr0", "span_all", "zn_above",
            "zn_below", "eig_cut", "eig_and_cd", "sd0", "means", "capped", "wrap"} <= reached
    capped = [c for c in cases if "capped" in _reached(c)]
    assert len(capped) == 1
    _, iters, _ = K.reference(capped[0])
    assert [d for d, it in enumerate(iters) if it < 0] == [1], iters
