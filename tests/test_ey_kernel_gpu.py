"""The EY step kernel (``ey_steps`` in csrc/ey.cu) driven through ``ops.ey_fit`` directly, step for step against the
float64 restatement of its steps (tests/fake_ops_ey.EyFit: ``oracle.ey.cov_step`` / ``mb_step``), at the shapes where
the kernel branches.  The case table and the reference half of every case live in tests/ey_kernel_cases.py.

After each compared call the whole device state block is read once and checked against the reference state: W and the
velocity relative to their max |.|, the objective, the step count, the last |prev - obj| and the stop flag.  The
tolerance is 1e-12 after the first step and 1e-10 after the rest (a few tens of steps); float32 views are held to the
same bounds, since the kernel converts each gathered element to float64 exactly.

Beyond the per-case parity: the launch grid (read from a profiler trace) is small enough that the grid-stride loops
these cases rely on do wrap; chunked calls give the bit-identical state of one call; a stop inside a call freezes the
state for every later call; a divergent fit ends in NaN weights without a stop; rows past 2^31 elements of a view are
gathered with 64-bit offsets; and, at the estimator level, chunking and column-slice views leave ``weights_`` bit for
bit unchanged."""
import json
import os
import subprocess
import sys
import tempfile

import numpy as np
import pytest
import torch

from tests import ey_kernel_cases as K
from tests import fake_ops_ey

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


# ----------------------------------------------------------------------------------------------------------- helpers
def _device_views(case, views):
    """The case's views on the device: contiguous, or columns 1 .. p of a wider NaN-filled tensor whose (odd) row
    stride is ``K.row_strides``."""
    out = []
    for v, ld in zip(views, K.row_strides(case)):
        t = torch.from_numpy(v).cuda()
        if ld != v.shape[1]:
            wide = torch.full((v.shape[0], ld), float("nan"), dtype=t.dtype, device="cuda")
            wide[:, 1:1 + v.shape[1]] = t
            t = wide[:, 1:1 + v.shape[1]]
            assert t.stride(0) == ld and not t.is_contiguous()
        out.append(t)
    return out


def _device_fit(case, tol=0.0):
    from cca_zoo_b200 import ops

    if isinstance(case, K.CovCase):
        C, init, lr = K.cov_inputs(case)
        fit = ops.ey_fit(case.dims, init, case.c, lr, K.MOMENTUM, tol, cov=torch.from_numpy(C).cuda())
        return fit, None
    views, init, lr, idx = K.mb_inputs(case)
    fit = ops.ey_fit(case.dims, init, case.c, lr, K.MOMENTUM, tol, views=_device_views(case, views), batch=case.bs)
    return fit, torch.from_numpy(idx).cuda()


def _run(fit, idx, calls):
    """Device state blocks after each call of ``calls`` (one read of the state per call)."""
    out, start = [], 0
    for n in calls:
        fit.run(n, None if idx is None else idx[start:start + n])
        out.append(fit.state.cpu().numpy().copy())
        start += n
    return out


def _check(label, k, D, dev, ref, tol):
    """Device block against reference block; returns the relative errors."""
    hd, Wd, Vd = K.split_block(dev, k, D)
    hr, Wr, Vr = K.split_block(ref, k, D)
    assert np.isfinite(Wr).all() and np.isfinite(Vr).all()
    err = {
        "W": float(np.abs(Wd - Wr).max() / np.abs(Wr).max()),
        "vel": float(np.abs(Vd - Vr).max() / np.abs(Vr).max()),
        "obj": float(abs(hd[0] - hr[0]) / abs(hr[0])),
    }
    if np.isinf(hr[3]):                              # the first step of a fit: |inf - obj|
        assert hd[3] == hr[3], f"{label}: last delta {hd[3]} != {hr[3]}"
        err["delta"] = 0.0
    else:                                            # |prev - obj|: the error of two objectives of this size
        err["delta"] = float(abs(hd[3] - hr[3]) / (abs(hr[0]) + abs(hr[3])))
    print(f"{label}: " + "  ".join(f"{n} {e:.1e}" for n, e in err.items()))
    assert hd[1] == hr[1], f"{label}: steps {hd[1]} != {hr[1]}"
    assert hd[2] == hr[2], f"{label}: stop flag {hd[2]} != {hr[2]}"
    assert not hd[4:].any(), f"{label}: the unused header words changed"
    for name, e in err.items():
        assert e <= tol, f"{label}: {name} differs by {e:.2e} (> {tol:.0e})"
    return err


def _parity(case):
    calls, ref = K.ref_schedule(case)
    fit, idx = _device_fit(case)
    dev = _run(fit, idx, calls)
    for i, tol in enumerate((K.FIRST_TOL, K.LATER_TOL)):
        _check(f"{case.name} step {sum(calls[:i + 1])}", case.k, case.D, dev[i], ref[i], tol)


# ----------------------------------------------------------------------------------------------------------- routes
@pytest.mark.parametrize("case", K.COV_CASES, ids=lambda c: c.name)
def test_ey_kernel_covariance_route_matches_reference(case):
    _parity(case)


@pytest.mark.parametrize("case", K.MB_CASES, ids=lambda c: c.name)
def test_ey_kernel_minibatch_route_matches_reference(case):
    _parity(case)


def print_ey_grids(trace_dir):
    """One step of each instantiation of ey_steps (covariance, float64 and float32 mini-batch) under the profiler;
    prints {kernel name: grid} as JSON, read from the exported trace."""
    from torch.profiler import ProfilerActivity, profile

    fits = [_device_fit(case) for case in (K.COV["k32_largeD"], K.MB["bs127_k32_m2"], K.MB["bs20000_k32_m3"])]
    torch.cuda.synchronize()
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        for fit, idx in fits:
            fit.run(1, idx)
        torch.cuda.synchronize()
    path = os.path.join(trace_dir, "trace.json")
    prof.export_chrome_trace(path)
    with open(path) as f:
        events = json.load(f)["traceEvents"]
    out = {}
    for e in events:
        if e.get("cat") == "kernel" and "ey_steps" in e.get("name", ""):
            assert "grid" in e.get("args", {}), e
            out[e["name"]] = e["args"]["grid"]
    print(json.dumps(out))


def test_ey_kernel_launch_grid_makes_the_loops_wrap():
    """The k = 32 cases wrap the one-warp-per-entry loops over the 2k^2 entries of V | C_ey (8 warps per CTA times
    the grid < 2k^2) and the large-D cases wrap the row tiles of the covariance products (8 rows per tile, D > 8 times
    the grid, with D > 16 x SMs besides).  Read from the launch itself, so a change of occupancy that voided the
    coverage fails here.  The profiler runs in a child process: a profiling session early in the pytest process left
    later sessions there (tests/test_shape_routes_gpu.py) with no kernel events."""
    sms = torch.cuda.get_device_properties(0).multi_processor_count
    with tempfile.TemporaryDirectory() as d:
        code = (f"import sys; sys.path.insert(0, {ROOT!r}); from tests import test_ey_kernel_gpu as t; "
                f"t.print_ey_grids({d!r})")
        flags = ["-s"] if sys.flags.no_user_site else []
        r = subprocess.run([sys.executable, *flags, "-c", code], capture_output=True, text=True, timeout=900)
    assert r.returncode == 0, r.stdout[-2000:] + r.stderr[-4000:]
    grids = {name: tuple(g) for name, g in json.loads(r.stdout.strip().splitlines()[-1]).items()}
    print(f"ey_steps grids on {sms} SMs: {grids}")
    assert len(grids) == 3, grids                    # the three instantiations, one launch each
    large = [c for c in K.COV_CASES if c.D > 16 * K.SMS_H100]
    assert {c.k for c in large} == {3, 17, 32}
    for name, g in grids.items():
        assert g[1] == g[2] == 1 and g[0] % sms == 0, (name, g)
        for case in [c for c in K.COV_CASES + K.MB_CASES if c.k == 32]:
            assert 8 * g[0] < 2 * case.k ** 2, (name, g, case.name)
        if "true" in name:                           # ey_steps<double, true>: the covariance route
            for case in large:
                assert case.D > 16 * sms and case.D > 8 * g[0], (g, case.name)


# ----------------------------------------------------------------------------------------------------------- state
@pytest.mark.parametrize("which", ["cov", "mb_f32", "mb_f64"])
def test_ey_kernel_chunked_calls_match_one_call(which):
    case = K.CHUNK_COV if which == "cov" else K.CHUNK_MB[which[3:]]
    blocks = []
    for calls in ((12,), (5, 7), (1,) * 12):
        fit, idx = _device_fit(case)
        _run(fit, idx, calls)
        blocks.append(fit.state.clone())
    assert torch.equal(blocks[0], blocks[1]), "run(5); run(7) differs from run(12)"
    assert torch.equal(blocks[0], blocks[2]), "12 x run(1) differs from run(12)"
    _check(f"{case.name} step 12", case.k, case.D, blocks[0].cpu().numpy(), K.ref_run(case, (12,))[0], K.LATER_TOL)


def test_ey_kernel_stop_inside_a_call_freezes_the_state():
    case = K.STOP_CASE
    tol, s, calls = K.stop_plan()
    ref = K.ref_run(case, calls, tol)
    fit, _ = _device_fit(case, tol)
    dev = _run(fit, None, calls)
    assert dev[0][1] == calls[0] and dev[0][2] == 0.0
    assert dev[1][1] == s and dev[1][2] == 1.0, f"stopped at {dev[1][1]} (flag {dev[1][2]}), expected step {s}"
    _check(f"{case.name} stop at {s}", case.k, case.D, dev[1], ref[1], K.LATER_TOL)
    assert np.array_equal(dev[2], dev[1]), "a call after the stop changed the state"
    assert fit.stopped()


def test_ey_kernel_divergence_ends_in_nan_without_stop():
    case = K.DIVERGE_CASE
    fit, _ = _device_fit(case)
    fit.run(case.steps)
    h, W, _ = K.split_block(fit.state.cpu().numpy(), case.k, case.D)
    assert np.isnan(W).all()
    assert h[1] == case.steps and h[2] == 0.0 and not fit.stopped()


def test_ey_kernel_rows_past_2_31_elements():
    """View 1 is 3 rows of a float32 storage of 2^31 + a few thousand elements, row stride 2^30 + 5: its row 2 starts
    past element 2^31, so its offset only fits in 64 bits."""
    from cca_zoo_b200 import ops

    ld, p0, p1, k, bs, steps = 2 ** 30 + 5, 7, 40, 2, 64, 6
    size = 2 * ld + p1 + 4096
    free, _ = torch.cuda.mem_get_info()
    if free < 2 * 4 * size:
        pytest.skip(f"needs {2 * 4 * size / 2**30:.1f} GiB free, {free / 2**30:.1f} GiB are")
    rng = np.random.default_rng(11)
    x = [rng.standard_normal((3, p)).astype(np.float32) + 0.5 for p in (p0, p1)]
    idx = rng.integers(0, 3, (steps, bs)).astype(np.int32)
    idx[:, 0] = 2
    init = K.orthonormal_init(rng, (p0, p1), k, 0.5)
    trace = sum(float(v.astype(np.float64).var(axis=0, ddof=1).sum()) for v in x)
    lr = 0.05 * 2 / (4 * trace)
    ref = fake_ops_ey.EyFit((p0, p1), init, 0.0, lr, K.MOMENTUM, 0.0, views=[torch.from_numpy(v) for v in x], batch=bs)
    storage = torch.empty(size, dtype=torch.float32, device="cuda")
    try:
        big = torch.as_strided(storage, (3, p1), (ld, 1))
        big.copy_(torch.from_numpy(x[1]))                # writes the 3 rows only
        fit = ops.ey_fit((p0, p1), init, 0.0, lr, K.MOMENTUM, 0.0, views=[torch.from_numpy(x[0]).cuda(), big], batch=bs)
        didx = torch.from_numpy(idx).cuda()
        start = 0
        for n, tol in ((1, K.FIRST_TOL), (steps - 1, K.LATER_TOL)):
            fit.run(n, didx[start:start + n])
            ref.run(n, torch.from_numpy(idx[start:start + n]))
            start += n
            _check(f"row offset past 2^31, step {start}", k, p0 + p1, fit.state.cpu().numpy(), K.ref_block(ref.st), tol)
        W = K.split_block(K.ref_block(ref.st), k, p0 + p1)[1]
        assert np.linalg.norm(W - init.T.reshape(-1)) > K.MOVE * np.linalg.norm(init)
    finally:
        del big, storage
        torch.cuda.empty_cache()


# ----------------------------------------------------------------------------------------------------------- estimator
def _estimator_views(dtype, rng):
    z = rng.standard_normal((600, 2))
    return [(z @ rng.standard_normal((2, p)) + rng.standard_normal((600, p)) + 1.0).astype(dtype) for p in (8, 12, 16)]


def test_ey_estimator_chunked_minibatch_fit_is_bit_identical(monkeypatch):
    from cca_zoo_b200 import linear
    from cca_zoo_b200.linear import _gradient

    views = _estimator_views(np.float64, np.random.default_rng(5))
    kw = dict(latent_dimensions=3, batch_size=50, max_iter=60, tol=0.0, learning_rate=2e-3, random_state=5)
    a = linear.MCCA_EY(**kw).fit(views)
    monkeypatch.setattr(_gradient, "_CHUNK_INDEX_BYTES", 4 * 50 * 7)    # 7 steps of 50 rows per chunk
    b = linear.MCCA_EY(**kw).fit(views)
    assert a._fit_info["calls"] == 1 and b._fit_info["calls"] == 9
    assert a._fit_info["iters"] == b._fit_info["iters"] == 60
    for x, y in zip(a.weights_, b.weights_):
        assert np.isfinite(x).all() and np.array_equal(x, y)


def test_ey_estimator_on_column_slices_matches_contiguous_views():
    """CUDA views that are column slices of wider tensors (row stride a multiple of 4 floats, so the column sums and
    the initial projection take the same GEMM route as for the contiguous copies) give bit-identical weights."""
    from cca_zoo_b200 import linear

    views = [torch.from_numpy(v).cuda() for v in _estimator_views(np.float32, np.random.default_rng(6))]
    sliced = []
    for v in views:
        wide = torch.full((v.shape[0], v.shape[1] + 8), float("nan"), dtype=v.dtype, device="cuda")
        wide[:, :v.shape[1]] = v
        sliced.append(wide[:, :v.shape[1]])
    kw = dict(latent_dimensions=3, batch_size=64, max_iter=50, tol=0.0, learning_rate=2e-3, random_state=6)
    a = linear.CCA_EY(**kw).fit(views)
    b = linear.CCA_EY(**kw).fit(sliced)
    assert a._fit_info["route"] == b._fit_info["route"] == "minibatch"
    for x, y in zip(a.weights_, b.weights_):
        assert np.isfinite(x).all() and np.array_equal(x, y)
