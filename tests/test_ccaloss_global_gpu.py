"""Global-batch CCALoss / MCCALoss / GCCALoss on one GPU, the ranks simulated in one process: a batch is split into
uneven shards (one of a single row, one shorter than the widths), the shards' moment buffers and counts are summed on
the device, and that sum stands in for the exchange while each shard runs the global forward and backward.  Every
shard must see the same loss bit for bit, and the concatenated gradients must match the package's own full-batch
evaluation."""
import numpy as np
import pytest
import torch

from cca_zoo_b200 import ops, parallel
from tests import golden_io as G

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


def _fake_exchange(monkeypatch, shards):
    """Sum the shards' moment buffers and counts on the device; every shard's exchange returns that sum."""
    dims = [int(z.shape[1]) for z in shards[0]]
    total = torch.zeros(ops.moments_size(dims), dtype=torch.float64, device="cuda")
    for sh in shards:
        if sh[0].shape[0]:
            total += ops.moments([z.contiguous() for z in sh], precision="exact")
    n_dev = torch.tensor([float(sum(sh[0].shape[0] for sh in shards))], dtype=torch.float64, device="cuda")
    monkeypatch.setattr(parallel, "is_distributed", lambda group=None: True)
    monkeypatch.setattr(parallel, "allreduce_moments_lazy",
                        lambda mom, n_local, group=None, dims=None: (total.clone(), None, n_dev.clone()))


def _run_shards(monkeypatch, make_loss, zs, sizes):
    shards = _split(zs, sizes)
    _fake_exchange(monkeypatch, shards)
    losses, grads = [], []
    for sh in shards:
        mine = [z.clone().requires_grad_(True) for z in sh]
        fn = make_loss(True)
        loss = fn(mine)
        loss.backward()
        if hasattr(fn, "check"):
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


def _cca(eps=1e-5, verify="lazy"):
    from cca_zoo_b200.deep import CCALoss

    return lambda glob: CCALoss(eps=eps, precision="exact", verify=verify, global_batch=glob)


@pytest.mark.parametrize("widths", [[5, 4], [64, 64], [65, 40], [130, 96]])
@pytest.mark.parametrize("verify", ["lazy", "sync"])
def test_ccaloss_global_matches_full_batch(monkeypatch, widths, verify):
    n = 700
    zs = _data(n, widths, seed=sum(widths))
    sizes = [1, 50, 300, n - 351]                     # one single row, one shorter than the widths
    losses, grads = _run_shards(monkeypatch, lambda g: _cca(verify=verify)(g), zs, sizes)
    loss_ref, grads_ref = _full(_cca(verify=verify), zs)
    _check(losses, grads, loss_ref, grads_ref, 1e-10)


@pytest.mark.parametrize("widths", [[5, 4, 3], [8, 8, 8], [6, 6, 6, 6], [70, 20, 33, 9]])
def test_mccaloss_global_matches_full_batch(monkeypatch, widths):
    from cca_zoo_b200.deep import MCCALoss

    n = 600
    zs = _data(n, widths, seed=len(widths) + sum(widths))
    make = lambda glob: MCCALoss(eps=1e-5, precision="exact", global_batch=glob)  # noqa: E731
    losses, grads = _run_shards(monkeypatch, make, zs, [1, 40, 259, 300])
    loss_ref, grads_ref = _full(make, zs)
    _check(losses, grads, loss_ref, grads_ref, 1e-10)


def test_gccaloss_global_matches_full_batch(monkeypatch):
    from cca_zoo_b200.deep import GCCALoss

    zs = _data(500, [6, 5, 7], seed=11)
    make = lambda glob: GCCALoss(eps=1e-5, global_batch=glob)  # noqa: E731
    losses, grads = _run_shards(monkeypatch, make, zs, [1, 4, 200, 295])
    loss_ref, grads_ref = _full(make, zs)
    _check(losses, grads, loss_ref, grads_ref, 1e-10)


@pytest.mark.parametrize("name", sorted(G.LOSS_CASES))
@pytest.mark.parametrize("dtype,tol", [(torch.float64, 1e-5), (torch.float32, 1e-3)])
def test_golden_loss_cases_split_into_shards(monkeypatch, name, dtype, tol):
    from cca_zoo_b200.deep import CCALoss, MCCALoss

    c = G.LOSS_CASES[name]
    loss_ref, grads_ref = G.loss_outputs(name)
    zs = [z.to(dtype).cuda() for z in G.loss_inputs(name)]
    n = zs[0].shape[0]
    cls = CCALoss if c["kind"] == "cca" else MCCALoss
    make = lambda glob: cls(eps=c["eps"], precision="exact", global_batch=glob)  # noqa: E731
    losses, grads = _run_shards(monkeypatch, make, zs, [1, n // 3, n - 1 - n // 3])
    assert all(torch.equal(l, losses[0]) for l in losses)
    assert abs(float(losses[0]) - loss_ref) < tol * abs(loss_ref)
    for g, gr in zip(grads, grads_ref):
        err = np.abs(g.double().cpu().numpy() - gr).max()
        assert err < tol * np.abs(gr).max()


def test_globally_rank_deficient_batch_takes_the_eigen_route(monkeypatch):
    from cca_zoo_b200.deep import MCCALoss

    zs = _data(20, [30, 24], seed=4)                 # N - 1 < width: every shard takes the eigen route
    losses, grads = _run_shards(monkeypatch, _cca(eps=1e-3), zs, [1, 7, 12])
    loss_ref, grads_ref = _full(_cca(eps=1e-3), zs)
    _check(losses, grads, loss_ref, grads_ref, 1e-8)
    zs = _data(12, [20, 14, 16], seed=6)
    make = lambda glob: MCCALoss(eps=1e-3, precision="exact", verify="sync", global_batch=glob)  # noqa: E731
    losses, grads = _run_shards(monkeypatch, make, zs, [1, 5, 6])
    loss_ref, grads_ref = _full(make, zs)
    _check(losses, grads, loss_ref, grads_ref, 1e-8)


def _duplicate_column_views():
    x = torch.tensor([2.0] * 8 + [-2.0] * 8 + [0.0], dtype=torch.float64)
    g = torch.Generator().manual_seed(3)
    return [torch.stack([x, x], 1).cuda(), torch.randn(17, 2, generator=g, dtype=torch.float64).cuda(),
            torch.randn(17, 3, generator=g, dtype=torch.float64).cuda()]


def test_indefinite_within_view_covariance_under_sync(monkeypatch):
    from cca_zoo_b200.deep import MCCALoss

    zs = _duplicate_column_views()                    # S_11 = C_11 + 1e-17 I is singular: the Cholesky status fails
    losses, grads = _run_shards(monkeypatch, _cca(eps=1e-17, verify="sync"), zs[:2], [1, 6, 10])
    loss_ref, grads_ref = _full(_cca(eps=1e-17, verify="sync"), zs[:2])
    assert all(torch.equal(l, losses[0]) for l in losses)
    assert abs(float(losses[0]) - float(loss_ref)) <= 1e-6 * abs(float(loss_ref))
    assert all(torch.isfinite(g).all() for g in grads)
    make = lambda glob: MCCALoss(eps=1e-17, precision="exact", verify="sync", global_batch=glob)  # noqa: E731
    losses, grads = _run_shards(monkeypatch, make, zs, [1, 6, 10])
    loss_ref, _ = _full(make, zs)
    assert all(torch.equal(l, losses[0]) for l in losses)
    assert abs(float(losses[0]) - float(loss_ref)) <= 1e-6 * abs(float(loss_ref))
    assert all(torch.isfinite(g).all() for g in grads)
    lazy = _cca(eps=1e-17)(True)                      # lazy: every shard reports at check()
    shards = _split(zs[:2], [1, 6, 10])
    _fake_exchange(monkeypatch, shards)
    for sh in shards:
        lazy(sh)
        with pytest.raises(RuntimeError, match="not numerically positive"):
            lazy.check()


@pytest.mark.parametrize("widths", [[5, 4], [130, 96]])
def test_nan_in_one_shard_raises_on_every_shard(monkeypatch, widths):
    from cca_zoo_b200.deep import CCALoss, MCCALoss

    zs = _data(300, widths, seed=9)
    zs[0][200, 1] = float("nan")
    shards = _split(zs, [100, 100, 100])
    _fake_exchange(monkeypatch, shards)
    for sh in shards:
        with pytest.raises(ValueError, match="NaN"):
            CCALoss(verify="sync", global_batch=True)(sh)
        fn = CCALoss(global_batch=True)
        fn(sh)
        with pytest.raises(ValueError, match="NaN"):
            fn.check()
        fn = MCCALoss(global_batch=True)
        fn(sh)
        with pytest.raises(ValueError, match="NaN"):
            fn.check()


@pytest.mark.parametrize("widths", [[5, 4], [130, 96]])
def test_ops_level_global_steps_do_not_synchronise(monkeypatch, widths):
    from cca_zoo_b200.deep import MCCALoss

    zs = _data(512, widths, seed=2)
    shards = _split(zs, [200, 312])                   # both taller than the widths: nothing may be read back
    _fake_exchange(monkeypatch, shards)
    dims = [int(w) for w in widths]
    go = torch.ones(1, dtype=torch.float64, device="cuda")
    mcca = MCCALoss(global_batch=True)

    def step():
        for sh in shards:
            mom = ops.moments(sh, precision="exact")
            total, _, n_dev = parallel.allreduce_moments_lazy(mom, sh[0].shape[0], None, dims)
            loss, saved, flags = ops.ccaloss_fwd_moments(total, n_dev, dims[0], dims[1], 1e-5, torch.float64)
            ops.ccaloss_bwd_global(sh[0], sh[1], saved, go)
            mine = [z.clone().requires_grad_(True) for z in sh]
            mcca(mine).backward()

    step()
    torch.cuda.synchronize()
    torch.cuda.set_sync_debug_mode("error")
    try:
        step()
    finally:
        torch.cuda.set_sync_debug_mode(0)
    torch.cuda.synchronize()
    mcca.check()


def test_device_count_covariance_and_row_sub_scale():
    zs = _data(300, [7, 5], seed=1)
    mom = ops.moments(zs, precision="exact")
    C, mean = ops.covariance(mom, [7, 5], 300)
    Cd, meand = ops.covariance(mom, [7, 5], torch.tensor([300.0], dtype=torch.float64, device="cuda"))
    assert torch.equal(C, Cd) and torch.equal(mean, meand)
    A = torch.randn(1000, 37, dtype=torch.float64, device="cuda")
    r = torch.randn(37, dtype=torch.float64, device="cuda")
    s = torch.tensor([0.7], dtype=torch.float64, device="cuda")
    want = (A - r) * 0.7
    assert torch.equal(ops.row_sub_scale_(A, r, s), want)
