"""Host logic of ``TCCALoss(global_batch=True)`` on CPU: the torch stand-in of the kernels
(tests/fake_ops_tccaloss_global.py) and two gloo processes.  Checked: two collectives per forward (the moments, then
the tensor with its marginals) and none in the backward, no read-back of N while the local shard is at least as tall
as the widths, the read-back and the eigen route on every rank when the global batch is rank deficient, a rank without
rows, NaN in one shard raising on both ranks, and that one process takes today's route call for call.  Loss and
gradient rows are compared with the float64 restatement of oracle/tccaloss.py on the concatenated batch."""
import os
import socket
import sys

import numpy as np
import pytest
import torch
import torch.distributed as dist
import torch.multiprocessing as mp

from oracle import tccaloss as O
from tests import fake_ops_tccaloss_global as FT

EPS = 1e-3


def _free_port():
    s = socket.socket()
    s.bind(("127.0.0.1", 0))
    port = s.getsockname()[1]
    s.close()
    return port


def _data(n, widths, seed):
    g = torch.Generator().manual_seed(seed)
    lat = torch.randn(n, 2, generator=g, dtype=torch.float64)
    return [lat @ torch.randn(2, w, generator=g, dtype=torch.float64) + torch.randn(n, w, generator=g, dtype=torch.float64)
            for w in widths]


# (name, widths, total rows, rows of rank 0)
CASES = [
    ("m2", [5, 4], 40, 27),
    ("m3", [6, 5, 4], 50, 31),
    ("empty_rank", [6, 5, 4], 30, 0),
    ("m4_narrow_shard", [4, 3, 3, 2], 45, 1),
    ("eigen", [8, 6, 5], 6, 2),
]


def _loss(**kw):
    from cca_zoo_b200.deep import TCCALoss

    return TCCALoss(eps=EPS, **kw)


def _worker(rank, world, port, out):
    os.environ.update(MASTER_ADDR="127.0.0.1", MASTER_PORT=str(port), RANK=str(rank), WORLD_SIZE=str(world))
    dist.init_process_group("gloo", rank=rank, world_size=world)
    monkeypatch = pytest.MonkeyPatch()
    try:
        from cca_zoo_b200 import parallel

        log = FT.install(monkeypatch)
        collectives = []
        real = parallel.dist.all_reduce
        monkeypatch.setattr(parallel.dist, "all_reduce", lambda *a, **k: (collectives.append(1), real(*a, **k))[1])
        res = {}
        for name, widths, n, n0 in CASES:
            zs = _data(n, widths, seed=len(name))
            lo, hi = (0, n0) if rank == 0 else (n0, n)
            mine = [z[lo:hi].clone().requires_grad_(True) for z in zs]
            log.clear()
            collectives.clear()
            loss = _loss(global_batch=True)(mine)
            fwd_log, fwd_coll = list(log), len(collectives)
            log.clear()
            loss.backward()
            res[name] = dict(loss=loss.detach(), grads=[z.grad for z in mine], fwd_log=fwd_log, fwd_coll=fwd_coll,
                             bwd_log=list(log), bwd_coll=len(collectives) - fwd_coll)
        zs = _data(40, [5, 4, 3], seed=7)
        zs[1][30, 2] = float("nan")                    # rank 1's shard only
        raised = []
        for verify in ("lazy", "sync"):
            mine = [z[:20] if rank == 0 else z[20:] for z in zs]
            try:
                _loss(global_batch=True, verify=verify)(mine)
                raised.append(None)
            except ValueError as err:
                raised.append(str(err))
        res["nan"] = raised
        torch.save(res, os.path.join(out, f"rank{rank}.pt"))
    finally:
        monkeypatch.undo()
        dist.destroy_process_group()


@pytest.fixture(scope="module")
def ranks(tmp_path_factory):
    out = tmp_path_factory.mktemp("tcca_global")
    # the workers import this module as ``tests.…``: the repository's own ``tests`` must come first on their path,
    # whatever other trees earlier tests of the session put in front of it
    root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    saved = list(sys.path)
    sys.path.insert(0, root)
    try:
        mp.spawn(_worker, args=(2, _free_port(), str(out)), nprocs=2, join=True)
    finally:
        sys.path[:] = saved
    return [torch.load(out / f"rank{r}.pt") for r in range(2)]


@pytest.mark.parametrize("name,widths,n,n0", CASES, ids=[c[0] for c in CASES])
def test_global_loss_and_gradients_match_the_oracle(ranks, name, widths, n, n0):
    r0, r1 = ranks[0][name], ranks[1][name]
    assert torch.equal(r0["loss"], r1["loss"]), "every rank must see the same loss"
    form = O.eigen_form if n - 1 < max(widths) else O.chol_form
    loss, grads, _ = form([z.numpy() for z in _data(n, widths, seed=len(name))], EPS)
    assert abs(float(r0["loss"]) - loss) <= 1e-10 * abs(loss)
    for i, g in enumerate(grads):
        got = torch.cat([r0["grads"][i], r1["grads"][i]]).numpy()
        assert got.shape == g.shape
        assert np.abs(got - g).max() <= 1e-10 * np.abs(g).max(), (name, i)


@pytest.mark.parametrize("name", [c[0] for c in CASES])
def test_two_collectives_per_forward_none_in_backward(ranks, name):
    for r in ranks:
        assert r[name]["fwd_coll"] == 2
        assert r[name]["bwd_coll"] == 0
        assert "moments" not in r[name]["bwd_log"]


def test_no_read_back_when_the_shard_is_tall_enough(ranks):
    for name in ("m2", "m3"):
        for r in ranks:
            assert "read_n" not in r[name]["fwd_log"], name
            assert "syevj" not in r[name]["fwd_log"]
    # rank 0 holds 1 row of width 4: it reads N once, sees N - 1 >= 4 and stays on the Cholesky route like rank 1
    narrow, tall = ranks[0]["m4_narrow_shard"]["fwd_log"], ranks[1]["m4_narrow_shard"]["fwd_log"]
    assert narrow.count("read_n") == 1 and "read_n" not in tall
    assert "potrf_inv_" in narrow and "potrf_inv_" in tall and "syevj" not in narrow + tall


def test_rank_deficient_global_batch_takes_the_eigen_route_on_every_rank(ranks):
    for r in ranks:
        log = r["eigen"]["fwd_log"]
        assert "read_n" in log and "syevj" in log
        assert "potrf_inv_" not in log
        assert log.count("moments") == 1, "no second moment pass: the eigen route works from the exchanged moments"


def test_marginals_are_contracted_for_three_views_or_more(ranks):
    assert ranks[0]["m2"]["fwd_log"].count("tcca_moment") == 1
    assert ranks[0]["m3"]["fwd_log"].count("tcca_moment") == 1 + 3
    assert ranks[0]["m4_narrow_shard"]["fwd_log"].count("tcca_moment") == 1 + 4
    for r in ranks:
        # backward: one adjoint, and per mode one two-view contraction for M_(i) M_(i)^T and M_(i) vec(Pbar_i)
        assert r["m3"]["bwd_log"].count("tcca_moment_adjoint") == 1
        assert r["m3"]["bwd_log"].count("tcca_moment") == 3


def test_a_rank_without_rows(ranks):
    r0 = ranks[0]["empty_rank"]
    assert "moments" not in r0["fwd_log"] and "tcca_moment" not in r0["fwd_log"], "no kernel on an empty batch"
    assert "tcca_moment_adjoint" not in r0["bwd_log"]
    assert [tuple(g.shape) for g in r0["grads"]] == [(0, 6), (0, 5), (0, 4)]


def test_nan_in_one_shard_raises_on_both_ranks(ranks):
    for r in ranks:
        assert len(r["nan"]) == 2
        assert all(msg is not None and "NaN" in msg for msg in r["nan"]), r["nan"]


@pytest.mark.parametrize("widths", [[5, 4], [5, 4, 3], [3, 3, 2, 2]])
def test_one_process_takes_todays_route(monkeypatch, widths):
    assert not (dist.is_available() and dist.is_initialized())
    out = []
    log = FT.install(monkeypatch)
    for glob in (False, True):
        zs = [z.clone().requires_grad_(True) for z in _data(30, widths, seed=3)]
        log.clear()
        loss = _loss(global_batch=glob)(zs)
        loss.backward()
        out.append((list(log), loss.detach(), [z.grad for z in zs]))
    assert out[0][0] == out[1][0]
    assert torch.equal(out[0][1], out[1][1])
    assert all(torch.equal(a, b) for a, b in zip(out[0][2], out[1][2]))


@pytest.mark.parametrize("dtype", [torch.bfloat16, torch.float16])
@pytest.mark.parametrize("widths,n", [([5, 4, 3], 40), ([8, 6], 6)])
def test_16_bit_takes_the_global_body_without_an_exchange(monkeypatch, dtype, widths, n):
    from tests import fake_ops as F

    log = FT.install(monkeypatch)
    seen = []
    logged = F.moments

    def moments(views, precision="tf32x3b"):
        seen.append({v.dtype for v in views})
        return logged(views, precision)

    monkeypatch.setattr(F, "moments", moments)
    zs = [z.to(dtype).requires_grad_(True) for z in _data(n, widths, seed=5)]
    loss = _loss()(zs)
    assert loss.dtype == torch.float32
    loss.backward()
    loss = loss.detach()
    assert all(z.grad.dtype == dtype for z in zs)
    eigen = n - 1 < max(widths)
    # the moment pass reads the 16-bit representations; only the eigen route adds the float64 moments of the copies
    assert seen == ([{dtype}, {torch.float64}] if eigen else [{dtype}])
    assert ("read_n" in log) == eigen
    form = O.eigen_form if eigen else O.chol_form
    ref, grads, _ = form([z.detach().double().numpy() for z in zs], EPS)
    assert abs(float(loss) - ref) <= 1e-6 * abs(ref)
    for z, g in zip(zs, grads):
        assert np.abs(z.grad.double().numpy() - g).max() <= 1e-2 * np.abs(g).max()


def test_mixed_dtypes_raise(monkeypatch):
    FT.install(monkeypatch)
    zs = _data(20, [4, 3], seed=1)
    with pytest.raises(ValueError, match="share"):
        _loss()([zs[0].to(torch.bfloat16), zs[1].to(torch.float32)])
    with pytest.raises(ValueError, match="share"):
        _loss()([zs[0].to(torch.float16), zs[1].to(torch.bfloat16)])
