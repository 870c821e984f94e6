"""TEST INFRASTRUCTURE ONLY: the torch-CPU stand-in for ``cca_zoo_b200.ops.tcca_moment`` / ``tcca_fit``, the
companion of tests/fake_ops.py for ``cca_zoo_b200.linear._tcca``.  It runs the float64 restatement of oracle/tcca.py
(the Khatri-Rao contraction, the Gram start and ``als_step``) with the binding's contract: the state block in the
layout of ``ops.tcca_layout``.  Nothing in the package imports this module; ``install(monkeypatch)`` swaps it in for
one test (after ``fake_ops.install``).  ``CALLS`` counts the calls and records the random start columns passed."""
from __future__ import annotations

import numpy as np
import torch

from cca_zoo_b200.ops import (TCCA_HEADER, TCCA_MAX_ENTRIES, TCCA_MAX_ITER, TCCA_MAX_K, TCCA_MAX_VIEWS,  # noqa: F401
                              decode_tcca_state, tcca_layout)
from tests import fake_ops

CALLS = {"moment": 0, "fit": 0, "rand": None}


def tcca_moment(Z, nsplit=0):
    from oracle import tcca as O

    CALLS["moment"] += 1
    return torch.from_numpy(O.krprod_moment([z.to(torch.float64).numpy() for z in Z]))


def _encode(st, dims, k):
    o = tcca_layout(dims, k)
    h = np.zeros(o["total"])
    h[0], h[1], h[2], h[3] = st["iters"], st["stop"], st["singular"], st["norm"]
    h[o["rec"]:o["rec"] + len(st["rec"])] = st["rec"]
    for f, F in zip(o["F"], st["F"]):
        h[f:f + F.size] = F.reshape(-1)
    h[o["G"]:o["total"]] = np.stack([F.T @ F for F in st["F"]]).reshape(-1)
    return torch.from_numpy(h)


def tcca_fit(M, dims, k, n_iter, rand=None, state=None):
    from oracle import tcca as O

    CALLS["fit"] += 1
    dims = [int(p) for p in dims]
    if not (1 <= k <= TCCA_MAX_K) or not (2 <= len(dims) <= TCCA_MAX_VIEWS) or np.prod(dims) > TCCA_MAX_ENTRIES:
        raise ValueError("ccab_tcca_fit: problem out of range")
    T = M.to(torch.float64).numpy().reshape(dims)
    if state is None:
        CALLS["rand"] = rand
        st = O.gram_start(T, k, rand)
    else:
        d = decode_tcca_state(state.numpy(), dims, k)
        st = {"F": d["F"], "iters": d["iters"], "stop": d["stop"], "singular": d["singular"], "rec": list(d["rec"]),
              "norm": d["norm"]}
    for _ in range(min(int(n_iter), TCCA_MAX_ITER)):
        if st["iters"] >= TCCA_MAX_ITER:
            break
        O.als_step(st, T)
    return _encode(st, dims, k)


def install(monkeypatch):
    """Route TCCA's library calls through this module (and tests/fake_ops.py) for one test."""
    import sys

    from cca_zoo_b200.linear import _tcca

    me = sys.modules[__name__]
    for name in ("tcca_moment", "tcca_fit", "tcca_layout", "decode_tcca_state", "TCCA_MAX_K", "TCCA_MAX_VIEWS",
                 "TCCA_MAX_ENTRIES", "TCCA_MAX_ITER"):
        monkeypatch.setattr(fake_ops, name, getattr(me, name), raising=False)
    monkeypatch.setattr(_tcca, "ops", fake_ops)
    CALLS.update(moment=0, fit=0, rand=None)
