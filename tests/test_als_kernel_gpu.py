"""The ALS kernel (``als_dimension`` and ``als_deflate`` in csrc/als.cu) driven through ``ops.als_fit`` directly, kind
by kind against the float64 Gram-space restatement (oracle/sparse.py:cov_als_fit, oracle/elastic.py:cov_elastic_fit)
at the shapes and branches where it can go wrong.  The case table and the reference half of every case live in
tests/als_kernel_cases.py; tests/test_als_kernel_cases_cpu.py certifies from the reference's trace that no discrete
decision of a case sits within rounding of its boundary, so the comparison here is tight.

Per case: W against the reference relative to its max |w| (1e-12 after at most one sweep, 1e-10 after more; for the
regression kinds at least 1e-15 times the condition number of the kept eigenvalues), equal sweep counts, equal supports for the thresholding kinds, ``max_iter = 0`` returning the initial
weights bit for bit, and a ConvergenceWarning that names exactly the dimension whose descent was capped.  Beyond the
per-case parity: the launch grid read from a profiler trace makes the wrap cases wrap, those cases rerun bit for bit,
PLS_ALS and SCCA_Span are exactly invariant under a power-of-4 scaling of G, and a regression view wider than 2048
features is refused."""
import json
import os
import subprocess
import sys
import tempfile
import warnings

import numpy as np
import pytest
import torch

from tests import als_kernel_cases as K

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
WRAP = [c for c in K.CASES.values() if "wrap" in c.tags]


def _device_fit(case, scale=1.0):
    from cca_zoo_b200 import ops

    G, init, _ = K.inputs(case)
    cov = torch.from_numpy(G * (scale / (case.n - 1))).cuda()
    return ops.als_fit(cov, case.dims, case.n, case.kind, K.device_params(case), init, case.max_iter, case.tol,
                       mu=K.device_mu(case))


def _bound(case, trace):
    """The comparison bound of a case (see the module docstring) and the condition number it came from."""
    base = K.tolerance(case)
    kappa = max([u["cut"] / (K.RCOND * u["kept_min"]) for rec in trace for u in rec["updates"] if "cut" in u],
                default=1.0)
    return max(base, 1e-15 * kappa), f"kappa {kappa:.1e}"


@pytest.mark.parametrize("case", list(K.CASES.values()), ids=lambda c: c.name)
def test_als_kernel_matches_reference(case):
    from sklearn.exceptions import ConvergenceWarning

    W_ref, iters_ref, trace = K.reference(case)
    capped = [d for d, it in enumerate(iters_ref) if it < 0]
    if capped:
        with pytest.warns(ConvergenceWarning) as rec:
            W, iters = _device_fit(case)
        msgs = [str(r.message) for r in rec if issubclass(r.category, ConvergenceWarning)]
        assert len(msgs) == 1 and f"dimension(s) {capped}" in msgs[0], msgs
    else:
        with warnings.catch_warnings():
            warnings.simplefilter("error", ConvergenceWarning)
            W, iters = _device_fit(case)
    assert iters == [abs(it) for it in iters_ref], f"sweeps {iters} != {iters_ref}"
    if case.max_iter == 0:
        assert np.array_equal(W, K.inputs(case)[1].T), "max_iter = 0 changed the initial weights"
        return
    scale = float(np.abs(W_ref).max()) or 1.0        # all weights exactly zero: compare absolutely
    err = float(np.abs(W - W_ref).max()) / scale
    bound, why = _bound(case, trace)
    print(f"{case.name}: err {err:.1e} bound {bound:.0e} ({why}) ratio {err / bound:.1e}")
    assert err <= bound, f"{case.name}: W differs by {err:.2e} (> {bound:.0e})"
    if case.kind in ("pmd", "parkhomenko", "span", "admm") or "norm0" in case.tags:
        assert np.array_equal(W == 0.0, W_ref == 0.0), "the supports differ"


def print_als_grids(trace_dir):
    """One fit of each wrap case under the profiler; prints {kernel name: [grid, block]} as JSON, read from the
    exported trace."""
    from torch.profiler import ProfilerActivity, profile

    for case in WRAP:
        K.inputs(case)
    torch.cuda.synchronize()
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        for case in WRAP:
            _device_fit(case)
        torch.cuda.synchronize()
    path = os.path.join(trace_dir, "trace.json")
    prof.export_chrome_trace(path)
    with open(path) as f:
        events = json.load(f)["traceEvents"]
    out = {}
    for e in events:
        if e.get("cat") == "kernel" and "als_dimension" in e.get("name", ""):
            assert "grid" in e.get("args", {}) and "block" in e["args"], e
            out[e["name"]] = [e["args"]["grid"], e["args"]["block"]]
    print(json.dumps(out))


def test_als_kernel_launch_grid_makes_the_loops_wrap():
    """The wrap cases have more rows than the grid has warps (one warp per row of G) in the full pass and in a
    Gauss-Seidel phase (rows of view i and of view i - 1), for both instantiations.  Read from the launch itself, so a
    change of occupancy that voided the coverage fails here.  The profiler runs in a child process, as in
    tests/test_ey_kernel_gpu.py."""
    sms = torch.cuda.get_device_properties(0).multi_processor_count
    with tempfile.TemporaryDirectory() as d:
        code = (f"import sys; sys.path.insert(0, {ROOT!r}); from tests import test_als_kernel_gpu as t; "
                f"t.print_als_grids({d!r})")
        flags = ["-s"] if sys.flags.no_user_site else []
        r = subprocess.run([sys.executable, *flags, "-c", code], capture_output=True, text=True, timeout=900)
    assert r.returncode == 0, r.stdout[-2000:] + r.stderr[-4000:]
    grids = json.loads(r.stdout.strip().splitlines()[-1])
    print(f"als_dimension grids on {sms} SMs: {grids}")
    assert len(grids) == 2, grids                    # als_dimension<false> and <true>
    for name, (grid, block) in grids.items():
        assert grid[1] == grid[2] == 1 and grid[0] % sms == 0 and block[1] == block[2] == 1, (name, grid, block)
        warps = grid[0] * block[0] // 32
        reg = "true" in name
        for case in [c for c in WRAP if c.reg == reg]:
            phase = max(case.dims[i] + case.dims[i - 1] for i in range(len(case.dims)))
            assert case.D > warps and phase > warps, (name, grid, block, case.name)


@pytest.mark.parametrize("case", WRAP, ids=lambda c: c.name)
def test_als_kernel_wrap_cases_rerun_bit_identically(case):
    W1, it1 = _device_fit(case)
    W2, it2 = _device_fit(case)
    assert it1 == it2 and np.array_equal(W1, W2)


@pytest.mark.parametrize("name", ["pls_m3_k3_it2", "span_m3_k3_it2", "span_m8_k3"])
def test_als_kernel_exact_under_power_of_4_scaling(name):
    """Every step of PLS_ALS and SCCA_Span is homogeneous in G, deflation included, and sqrt(4^e x) = 2^e sqrt(x)
    exactly: 4^8 G and 4^-8 G give the bit-identical weights and sweeps."""
    case = K.CASES[name]
    W, iters = _device_fit(case)
    for e in (8, -8):
        We, ie = _device_fit(case, scale=4.0 ** e)
        assert ie == iters and np.array_equal(We, W), e


def test_als_kernel_regression_view_past_2048_features_raises():
    from cca_zoo_b200 import ops

    dims = (2049, 3)
    D = sum(dims)
    cov = torch.eye(D, dtype=torch.float64, device="cuda")
    init = np.ones((1, D)) / 3.0
    for kind, extra in (("elastic", []), ("ipls", [0.0] * D)):
        with pytest.raises(ValueError, match="2048"):
            ops.als_fit(cov, dims, 1025, kind, [0.1, 0.5, 0.1, 0.5] + extra, init, 2, 0.0)
