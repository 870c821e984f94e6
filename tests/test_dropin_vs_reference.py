"""Drop-in check of the model-selection contract: a grid search (sklearn clone / set_params / fit / score on 3-fold
splits of the samples, as the reference's GridSearchCV wrapper runs it) drives this package's estimators and must
reach the reference's cross-validated scores and best parameters (recorded by oracle/make_golden_live.py), host
logic on the torch-CPU stand-in."""
import os
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))

SCRIPT = r"""
import sys, warnings
sys.path.insert(0, %r)
from tests import fake_ops
import numpy as np, pytest
from sklearn.base import clone
from sklearn.model_selection import KFold, ParameterGrid
fake_ops.install(pytest.MonkeyPatch())
from cca_zoo_b200 import linear as ours
from oracle.make_golden_live import DROPIN_GRIDS, dropin_views
golden = np.load(%r)
views = dropin_views()
for name, (nv, grid) in DROPIN_GRIDS.items():
    v = views[:nv]
    base = getattr(ours, name)(latent_dimensions=2)
    scores = []
    for params in ParameterGrid(grid):
        fold = []
        for tr, te in KFold(3).split(v[0]):
            est = clone(base).set_params(**params)
            with warnings.catch_warnings():
                warnings.simplefilter("ignore")
                est.fit([x[tr] for x in v])
            fold.append(float(np.mean(est.score([x[te] for x in v]))))
        scores.append(np.mean(fold))
    ref = golden[f"dropin/{name}/mean_test_score"]
    assert int(np.argmax(scores)) == int(np.argmax(ref)), (name, scores, ref)
    assert np.allclose(scores, ref, atol=1e-8), (name, scores, ref)
    assert type(est).__module__.startswith("cca_zoo_b200")
print("DROPIN_OK")
"""


def test_reference_gridsearch_drives_our_estimators():
    golden = os.path.join(ROOT, "tests", "golden", "reference_live.npz")
    out = subprocess.run([sys.executable, "-c", SCRIPT % (ROOT, golden)], capture_output=True, text=True, timeout=900)
    assert "DROPIN_OK" in out.stdout, out.stdout[-2000:] + out.stderr[-3000:]
