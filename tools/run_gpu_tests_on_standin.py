"""Pre-flight for HOST-SIDE changes when no GPU is at hand: run the estimator-level ``-m gpu`` test files with
tests/fake_ops.py (torch CPU) standing in for the kernels.  It validates the Python between the kernels against
the same goldens / oracle assertions the GPU run will make; it says nothing about the kernels themselves.

    python tools/run_gpu_tests_on_standin.py [extra pytest args]
"""
import os
import sys

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
os.chdir(ROOT)

from tests import fake_ops, fake_ops_ey, fake_ops_sparse, fake_ops_tccaloss  # noqa: E402

os.environ["CCAB_TESTS_ON_STANDIN"] = "1"
mp = pytest.MonkeyPatch()
fake_ops.install(mp)
fake_ops_sparse.install(mp)
fake_ops_ey.install(mp)
fake_ops_tccaloss.install(mp)
FILES = ["tests/test_linear_gpu.py", "tests/test_ext_gpu.py", "tests/test_zz_center_gpu.py", "tests/test_sparse_gpu.py",
         "tests/test_ey_gpu.py", "tests/test_tccaloss_gpu.py"]
# tests that move tensors to the GPU themselves or time device paths cannot run on the stand-in
SKIP = ("accepts_cuda_and_cpu_tensors or batches_tensors or device_score_path or partial_fit_and_streamed or pickle "
        "or float32_precisions or edge_shapes or transform_on_the_device or one_library_call or argument_errors "
        "or cuda_and_host_inputs or sync_takes_the_eigen_route or nan_input_raises or no_host_sync "
        "or training_loop_matches_eager or shape_the_reference_cannot_hold")
sys.exit(pytest.main([f for f in FILES if os.path.exists(f)] + ["-m", "gpu", "-q", "-k", f"not ({SKIP})", "-p",
                                                                 "no:cacheprovider"] + sys.argv[1:]))
