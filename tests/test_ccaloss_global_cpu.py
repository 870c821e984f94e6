"""Host logic of ``global_batch=True`` (CCALoss, MCCALoss, GCCALoss) on CPU: the torch stand-in of the kernels
(tests/fake_ops_global.py) and two gloo processes.  Checked: one collective per forward and none in the backward, no
read-back of N while the local shard is at least as tall as the widths, the read-back and the eigen route when the
global batch is rank deficient, a rank without rows, and that one process takes today's route call for call."""
import os
import socket

import pytest
import torch
import torch.distributed as dist
import torch.multiprocessing as mp

from tests import fake_ops_global as FG


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


# (name, loss class, widths, total rows, rows of rank 0)
CASES = [
    ("cca_uneven", "CCALoss", [5, 4], 40, 27),
    ("cca_narrow_shard", "CCALoss", [5, 4], 40, 3),
    ("cca_eigen", "CCALoss", [8, 6], 6, 2),
    ("cca_empty_rank", "CCALoss", [5, 4], 30, 0),
    ("mcca3", "MCCALoss", [5, 4, 3], 50, 31),
    ("mcca_eigen", "MCCALoss", [6, 4, 3], 5, 2),
    ("gcca3", "GCCALoss", [4, 4, 4], 45, 20),
]


def _loss(kind, **kw):
    from cca_zoo_b200.deep import objectives

    return getattr(objectives, kind)(eps=1e-3, **kw)


def _worker(rank, world, port, out):
    os.environ.update(MASTER_ADDR="127.0.0.1", MASTER_PORT=str(port), RANK=str(rank), WORLD_SIZE=str(world))
    dist.init_process_group("gloo", rank=rank, world_size=world)
    monkeypatch = pytest.MonkeyPatch()
    try:
        from cca_zoo_b200 import parallel

        log = FG.install(monkeypatch)
        collectives = []
        real = parallel.dist.all_reduce
        monkeypatch.setattr(parallel.dist, "all_reduce", lambda *a, **k: (collectives.append(1), real(*a, **k))[1])
        res = {}
        for name, kind, widths, n, n0 in CASES:
            zs = _data(n, widths, seed=len(name))
            lo, hi = (0, n0) if rank == 0 else (n0, n)
            mine = [z[lo:hi].clone().requires_grad_(True) for z in zs]
            log.clear()
            collectives.clear()
            loss = _loss(kind, global_batch=True)(mine)
            fwd_log, fwd_coll = list(log), len(collectives)
            log.clear()
            loss.backward()
            res[name] = dict(loss=loss.detach(), grads=[z.grad for z in mine], fwd_log=fwd_log, fwd_coll=fwd_coll,
                             bwd_log=list(log), bwd_coll=len(collectives) - fwd_coll)
        torch.save(res, os.path.join(out, f"rank{rank}.pt"))
    finally:
        monkeypatch.undo()
        dist.destroy_process_group()


@pytest.fixture(scope="module")
def ranks(tmp_path_factory):
    out = tmp_path_factory.mktemp("global")
    mp.spawn(_worker, args=(2, _free_port(), str(out)), nprocs=2, join=True)
    return [torch.load(out / f"rank{r}.pt") for r in range(2)]


def _full_batch(monkeypatch, kind, widths, n, name):
    FG.install(monkeypatch)
    zs = [z.clone().requires_grad_(True) for z in _data(n, widths, seed=len(name))]
    loss = _loss(kind)(zs)
    loss.backward()
    return loss.detach(), [z.grad for z in zs]


@pytest.mark.parametrize("name,kind,widths,n,n0", CASES, ids=[c[0] for c in CASES])
def test_global_loss_and_gradients_match_the_full_batch(ranks, monkeypatch, name, kind, widths, n, n0):
    r0, r1 = ranks[0][name], ranks[1][name]
    assert torch.equal(r0["loss"], r1["loss"]), "every rank must see the same loss"
    loss, grads = _full_batch(monkeypatch, kind, widths, n, name)
    # rank-deficient batches: S_ii has eigenvalues at eps = 1e-3, so its inverse amplifies rounding ~1e3-fold
    tol = 1e-8 if "eigen" in name else 1e-10
    assert abs(float(r0["loss"]) - float(loss)) <= tol * abs(float(loss))
    for i, g in enumerate(grads):
        got = torch.cat([r0["grads"][i], r1["grads"][i]])
        assert got.shape == g.shape
        assert float((got - g).abs().max()) <= tol * float(g.abs().max()), (name, i)


@pytest.mark.parametrize("name", [c[0] for c in CASES])
def test_one_collective_per_forward_none_in_backward(ranks, name):
    for r in ranks:
        assert r[name]["fwd_coll"] == 1
        assert r[name]["bwd_coll"] == 0
        assert "moments" not in r[name]["bwd_log"]


def test_no_read_back_when_the_shard_is_tall_enough(ranks):
    for name in ("cca_uneven", "mcca3"):
        for r in ranks:
            assert "read_n" not in r[name]["fwd_log"], name
            assert "syevj" not in r[name]["fwd_log"]
    # rank 0 holds 3 rows of width 5: it reads N once, sees N - 1 >= 5 and stays on the Cholesky route like rank 1
    narrow, tall = ranks[0]["cca_narrow_shard"]["fwd_log"], ranks[1]["cca_narrow_shard"]["fwd_log"]
    assert narrow.count("read_n") == 1 and "read_n" not in tall
    assert "ccaloss_fwd_moments" in narrow and "ccaloss_fwd_moments" in tall


def test_rank_deficient_global_batch_takes_the_eigen_route_on_every_rank(ranks):
    for name in ("cca_eigen", "mcca_eigen"):
        for r in ranks:
            log = r[name]["fwd_log"]
            assert "read_n" in log and "syevj" in log, name
            assert "ccaloss_fwd_moments" not in log and "potrf_inv_" not in log


def test_a_rank_without_rows(ranks):
    r0 = ranks[0]["cca_empty_rank"]
    assert "moments" not in r0["fwd_log"], "a rank without rows launches no moment pass"
    assert [tuple(g.shape) for g in r0["grads"]] == [(0, 5), (0, 4)]


@pytest.mark.parametrize("kind,widths", [("CCALoss", [5, 4]), ("MCCALoss", [5, 4, 3]), ("GCCALoss", [4, 4, 4])])
def test_one_process_takes_todays_route(monkeypatch, kind, widths):
    assert not (dist.is_available() and dist.is_initialized())
    out = []
    log = FG.install(monkeypatch)
    for glob in (False, True):
        zs = [z.clone().requires_grad_(True) for z in _data(30, widths, seed=3)]
        log.clear()
        loss = _loss(kind, global_batch=glob)(zs)
        loss.backward()
        out.append((list(log), loss.detach(), [z.grad for z in zs]))
    assert out[0][0] == out[1][0]
    assert torch.equal(out[0][1], out[1][1])
    assert all(torch.equal(a, b) for a, b in zip(out[0][2], out[1][2]))
