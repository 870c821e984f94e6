"""Differential fuzz of the host logic against the reference's recorded results (tests/golden/reference_fuzz*.npz,
made by oracle/make_golden_live.py).  A fixed seed of tools/fuzz_vs_reference.py: random shapes, ridge values,
centring flags, view weights, confounds, feature groups and dtypes must give the reference's scores, weights, means
and pairwise correlations wherever the problem is well posed and the component is determined, and raise where it
raises."""
import os
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _fuzz(tool):
    return subprocess.run([sys.executable, os.path.join(ROOT, "tools", tool), "20240924", "200", "--golden"],
                          capture_output=True, text=True, timeout=900)


def test_fixed_seed_fuzz_has_no_mismatch():
    out = _fuzz("fuzz_vs_reference.py")
    assert out.returncode == 0, out.stdout[-3000:] + out.stderr[-2000:]
    assert "0 mismatches" in out.stdout


def test_fixed_seed_loss_fuzz_has_no_mismatch():
    out = _fuzz("fuzz_loss_vs_reference.py")
    assert out.returncode == 0, out.stdout[-3000:] + out.stderr[-2000:]
    assert "0 mismatches" in out.stdout
