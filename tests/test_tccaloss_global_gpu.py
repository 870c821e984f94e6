"""Global-batch TCCALoss on one GPU, the ranks simulated in one process.  A batch is split into shards (also into three
with one of them empty).  The shards' moment buffers and counts are summed on the device and stand in for the first
exchange; for the second, every shard's local tensor buffer (the contraction of its whitened rows and, for 3 or more
views, the marginals) is recorded in a first pass, and their sum stands in for the all-reduce in the second.  Every
shard must see the same loss bit for bit, and the concatenated gradients must match the package's own full-batch
TCCALoss in float64."""
import pytest
import torch

from cca_zoo_b200 import ops, parallel

pytestmark = pytest.mark.gpu


def _data(n, widths, seed, dtype=torch.float64):
    g = torch.Generator().manual_seed(seed)
    lat = torch.randn(n, 3, generator=g, dtype=torch.float64)
    zs = [lat @ torch.randn(3, w, generator=g, dtype=torch.float64) + torch.randn(n, w, generator=g, dtype=torch.float64)
          for w in widths]
    return [z.to(dtype).cuda() for z in zs]


def _split(zs, sizes):
    out, lo = [], 0
    for s in sizes:
        out.append([z[lo:lo + s] for z in zs])
        lo += s
    assert lo == zs[0].shape[0]
    return out


def _fake_exchange(monkeypatch, shards, tensor_total=None):
    """Sum the shards' moment buffers and counts on the device; every shard's first exchange returns that sum, and
    its second returns ``tensor_total`` (None: the local buffer as it is)."""
    dims = [int(z.shape[1]) for z in shards[0]]
    total = torch.zeros(ops.moments_size(dims), dtype=torch.float64, device="cuda")
    for sh in shards:
        if sh[0].shape[0]:
            total += ops.moments([z.contiguous() for z in sh], precision="exact")
    n_dev = torch.tensor([float(sum(sh[0].shape[0] for sh in shards))], dtype=torch.float64, device="cuda")
    monkeypatch.setattr(parallel, "is_distributed", lambda group=None: True)
    monkeypatch.setattr(parallel, "allreduce_moments_lazy",
                        lambda mom, n_local, group=None, dims=None: (total.clone(), None, n_dev.clone()))
    monkeypatch.setattr(parallel, "allreduce_sum_",
                        lambda buf, group=None: buf if tensor_total is None else buf.copy_(tensor_total))


def _tensor_total(monkeypatch, make_loss, shards):
    """First pass: every shard's local tensor buffer, summed in shard order."""
    local = []
    _fake_exchange(monkeypatch, shards)
    monkeypatch.setattr(parallel, "allreduce_sum_", lambda buf, group=None: (local.append(buf.clone()), buf)[1])
    for sh in shards:
        with torch.no_grad():
            make_loss(True)(sh)
    total = local[0].clone()
    for b in local[1:]:
        total += b
    return total


def _run_shards(monkeypatch, make_loss, zs, sizes):
    shards = _split(zs, sizes)
    total = _tensor_total(monkeypatch, make_loss, shards)
    _fake_exchange(monkeypatch, shards, total)
    losses, grads = [], []
    for sh in shards:
        mine = [z.clone().requires_grad_(True) for z in sh]
        fn = make_loss(True)
        loss = fn(mine)
        loss.backward()
        fn.check()
        losses.append(loss.detach())
        grads.append([z.grad for z in mine])
    monkeypatch.undo()
    return losses, [torch.cat([g[i] for g in grads]) for i in range(len(zs))]


def _full(make_loss, zs):
    mine = [z.clone().requires_grad_(True) for z in zs]
    loss = make_loss(False)(mine)
    loss.backward()
    return loss.detach(), [z.grad for z in mine]


def _rel(a, b):
    return float((a - b).abs().max()) / max(float(b.abs().max()), 1e-300)


def _check(losses, grads, loss_ref, grads_ref, tol):
    assert all(torch.equal(l, losses[0]) for l in losses), "every shard must see the same loss bit for bit"
    assert abs(float(losses[0]) - float(loss_ref)) <= tol * abs(float(loss_ref))
    for g, r in zip(grads, grads_ref):
        assert g.shape == r.shape
        assert _rel(g, r) <= tol, _rel(g, r)


def _tcca(eps=1e-5, verify="lazy"):
    from cca_zoo_b200.deep import TCCALoss

    return lambda glob: TCCALoss(eps=eps, precision="exact", verify=verify, global_batch=glob)


# (name, widths, N, shards): each also runs split into three with an empty middle shard
CASES = [
    ("m2", [5, 4], 40, [27, 13]),
    ("m3", [6, 5, 4], 50, [31, 19]),
    ("empty_rank", [6, 5, 4], 30, [0, 30]),
    ("m4_narrow_shard", [4, 3, 3, 2], 45, [1, 44]),
    ("eigen", [8, 6, 5], 6, [2, 4]),
    ("wide", [64, 64, 64], 4096, [2048, 1500, 548]),
    ("limit", [256, 256, 512], 1030, [515, 515]),
]


def _with_empty(sizes):
    return [sizes[0], 0, sum(sizes[1:])]


@pytest.mark.parametrize("three", [False, True], ids=["shards", "three_with_empty"])
@pytest.mark.parametrize("verify", ["lazy", "sync"])
@pytest.mark.parametrize("name,widths,n,sizes", CASES, ids=[c[0] for c in CASES])
def test_tccaloss_global_matches_full_batch(monkeypatch, name, widths, n, sizes, verify, three):
    if name == "limit" and verify == "sync":
        pytest.skip("the limit shape runs once per split, under verify='lazy'")
    zs = _data(n, widths, seed=n + sum(widths))
    eps = 1e-3 if name == "eigen" else 1e-5
    losses, grads = _run_shards(monkeypatch, _tcca(eps, verify), zs, _with_empty(sizes) if three else sizes)
    loss_ref, grads_ref = _full(_tcca(eps, verify), zs)
    _check(losses, grads, loss_ref, grads_ref, 1e-8 if name == "eigen" else 1e-10)


def _duplicate_column_views():
    x = torch.tensor([2.0] * 8 + [-2.0] * 8 + [0.0], dtype=torch.float64)
    g = torch.Generator().manual_seed(3)
    return [torch.stack([x, x], 1).cuda(), torch.randn(17, 3, generator=g, dtype=torch.float64).cuda(),
            torch.randn(17, 2, generator=g, dtype=torch.float64).cuda()]


def test_indefinite_within_view_covariance(monkeypatch):
    zs = _duplicate_column_views()                    # S_1 = C_11 + 1e-17 I is singular: the Cholesky status fails
    sizes = [1, 6, 10]
    losses, grads = _run_shards(monkeypatch, _tcca(eps=1e-17, verify="sync"), zs, sizes)
    loss_ref, _ = _full(_tcca(eps=1e-17, verify="sync"), zs)
    assert all(torch.equal(l, losses[0]) for l in losses)
    assert abs(float(losses[0]) - float(loss_ref)) <= 1e-6 * abs(float(loss_ref))
    assert all(torch.isfinite(g).all() for g in grads)
    lazy = _tcca(eps=1e-17)(True)                     # lazy: every shard reports at check()
    shards = _split(zs, sizes)
    _fake_exchange(monkeypatch, shards)
    for sh in shards:
        lazy(sh)
        with pytest.raises(RuntimeError, match="not numerically positive"):
            lazy.check()


@pytest.mark.parametrize("widths", [[5, 4, 3], [64, 64, 64]])
def test_nan_in_one_shard_raises_on_every_shard(monkeypatch, widths):
    from cca_zoo_b200.deep import TCCALoss

    zs = _data(300, widths, seed=9)
    zs[1][200, 1] = float("nan")
    shards = _split(zs, [100, 100, 100])
    _fake_exchange(monkeypatch, shards)
    for sh in shards:
        with pytest.raises(ValueError, match="NaN"):
            TCCALoss(verify="sync", global_batch=True)(sh)
        fn = TCCALoss(global_batch=True)
        fn(sh)
        with pytest.raises(ValueError, match="NaN"):
            fn.check()


@pytest.mark.parametrize("widths", [[5, 4, 3], [64, 64, 64]])
def test_tall_shards_do_not_synchronise(monkeypatch, widths):
    zs = _data(1024, widths, seed=2)
    shards = _split(zs, [400, 624])                   # both taller than the widths: nothing may be read back
    make = _tcca()
    total = _tensor_total(monkeypatch, make, shards)
    _fake_exchange(monkeypatch, shards, total)
    fns = [make(True) for _ in shards]
    mine = [[z.clone().requires_grad_(True) for z in sh] for sh in shards]

    def step():
        for fn, sh in zip(fns, mine):
            fn(sh).backward()

    step()
    torch.cuda.synchronize()
    torch.cuda.set_sync_debug_mode("error")
    try:
        step()
    finally:
        torch.cuda.set_sync_debug_mode(0)
    torch.cuda.synchronize()
    for fn in fns:
        fn.check()


def test_one_process_runs_the_per_replica_route():
    from cca_zoo_b200.deep import objectives

    zs = _data(200, [6, 5, 4], seed=1)
    out = []
    for glob in (False, True):
        mine = [z.clone().requires_grad_(True) for z in zs]
        loss = objectives.TCCALoss(global_batch=glob)(mine)
        assert loss.grad_fn.name().startswith("_TCCALossFnBackward")
        loss.backward()
        out.append((loss.detach(), [z.grad for z in mine]))
    assert torch.equal(out[0][0], out[1][0])
    assert all(torch.equal(a, b) for a, b in zip(out[0][1], out[1][1]))


def test_tcca_moment_scale_and_out():
    H = _data(300, [7, 5, 3], seed=4)
    M = ops.tcca_moment(H)
    buf = torch.full((7 * 15 + 3,), 7.0, dtype=torch.float64, device="cuda")
    S = ops.tcca_moment(H, scale=1.0, out=buf[:105])
    assert S.data_ptr() == buf.data_ptr() and torch.equal(buf[105:], torch.full((3,), 7.0, dtype=torch.float64,
                                                                                  device="cuda"))
    assert _rel(S.reshape(7, 15) / 300, M) <= 1e-14
