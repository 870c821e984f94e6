"""Sample-sharded fitting: one process per GPU, each holding a row shard of every view.

The only exchange step of the path (SURVEY.md §8e): the additive moment buffer
``[M (Dp x Dp) | s (Dp) | n]`` is summed over ranks with ONE all-reduce; everything after it
(covariance finalisation, eigensolves) is replicated and bit-identical on every rank.
Backend-agnostic (NCCL on GPUs; the host logic is exercised with gloo on CPU in tests).
"""
from __future__ import annotations

import torch
import torch.distributed as dist


def is_distributed(group=None) -> bool:
    return dist.is_available() and dist.is_initialized() and dist.get_world_size(group) > 1


def pack_moments(moments: torch.Tensor, n_local: int) -> torch.Tensor:
    """Append the local row count so that it rides in the same message."""
    tail = torch.tensor([float(n_local)], dtype=moments.dtype, device=moments.device)
    return torch.cat([moments, tail])


def allreduce_moments(moments: torch.Tensor, n_local: int, group=None, dims=None):
    """Sum (moments, n) over the ranks of ``group``.  Returns (moments_total, n_total) -- one host read-back (n)."""
    if not is_distributed(group):
        return moments, int(n_local)
    mom, _, n_dev = allreduce_moments_lazy(moments, n_local, group, dims)
    return mom, int(round(float(n_dev.item())))


class _NvlsExchange:
    """Symmetric-memory state of the fused exchange kernel (csrc/moments.cu: exchange_nvls_kernel): one symmetric
    float64 buffer per message size with its multicast (NVLS) mapping and the ranks' signal pads, obtained from
    ``torch.distributed._symmetric_memory``; a call counter gives the flag epochs.  ``get`` returns None -- on every
    rank alike -- when symmetric memory or the multicast mapping is not available (then the NCCL all-reduce runs)."""

    _cache: dict = {}
    _disabled = False

    @classmethod
    def get(cls, device, n_doubles, group):
        import os

        mode = os.environ.get("CCAB_EXCHANGE", "auto")
        if cls._disabled or mode == "nccl":
            return None
        grp = group if group is not None else dist.group.WORLD
        key = (device.index, int(n_doubles), grp.group_name)
        if key in cls._cache:
            return cls._cache[key]
        world = dist.get_world_size(grp)
        ex, ok = None, 1
        try:
            import torch.distributed._symmetric_memory as symm_mem

            chunk = (-(-int(n_doubles) // world) + 1) // 2 * 2
            buf = symm_mem.empty(chunk * world, dtype=torch.float64, device=device)
            hdl = symm_mem.rendezvous(buf, grp)
            if not int(hdl.multicast_ptr):
                raise RuntimeError("no multicast (NVLS) mapping")
            pad = hdl.get_signal_pad(hdl.rank)
            pad.zero_()
            ex = cls.__new__(cls)
            ex.buf, ex.hdl, ex.calls = buf, hdl, 0
            ex.pad_slots = int(hdl.signal_pad_size) // 4
        except Exception as err:  # noqa: BLE001 -- any failure means "use NCCL", decided collectively below
            ok, ex = 0, None
            if mode == "nvls":
                raise RuntimeError(f"CCAB_EXCHANGE=nvls but symmetric memory is unavailable: {err}") from err
        flag = torch.tensor([ok], dtype=torch.int32, device=device)
        dist.all_reduce(flag, op=dist.ReduceOp.MIN, group=group)      # also orders the pad reset before the first use
        if int(flag.item()) == 0:
            cls._disabled = True
            ex = None
        cls._cache[key] = ex
        return ex

    def run(self, moments, dims, n_local):
        from . import ops

        self.calls += 1
        h = self.hdl
        return ops.moments_exchange_nvls(moments, dims, n_local, self.buf, int(h.multicast_ptr),
                                         int(h.signal_pad_ptrs_dev), int(h.rank), int(h.world_size), self.pad_slots,
                                         2 * self.calls - 1)


def allreduce_moments_lazy(moments: torch.Tensor, n_local: int, group=None, dims=None):
    """Like ``allreduce_moments`` but WITHOUT reading the sample count back: returns
    ``(moments_total, n_host, n_dev)`` where exactly one of ``n_host`` (int, single process) and ``n_dev`` (1-element
    float64 device tensor, sharded fit) is not None.  The device-side fit (``ops.rcca_fit``) takes ``n_dev`` as it is,
    so a sharded fit has no host synchronisation between the moment pass and the final copy of the weights."""
    if not is_distributed(group):
        return moments, int(n_local), None
    if moments.is_cuda and dims is not None:
        # the message carries only the upper triangle of 128 x 128 blocks, the column sums and n (half the bytes of the
        # square buffer, no torch.cat copy); packing / unpacking are two small kernels around the ONE all-reduce
        from . import _lib, ops

        size = int(_lib.load().ccab_moments_packed_size(len(dims), _lib.i64_array(dims)))
        ex = _NvlsExchange.get(moments.device, size, group)
        if ex is not None:
            # ONE kernel: pack, in-switch reduction on the NVLS multicast address, unpack (no NCCL call)
            return moments, None, ex.run(moments, dims, n_local)
        packed = ops.moments_pack(moments, dims, n_local)
        dist.all_reduce(packed, op=dist.ReduceOp.SUM, group=group)
        mom, n_dev = ops.moments_unpack(packed, dims, out=moments)
        return mom, None, n_dev
    packed = pack_moments(moments, n_local)
    dist.all_reduce(packed, op=dist.ReduceOp.SUM, group=group)
    return packed[:-1], None, packed[-1:]


def allreduce_sum_(buf: torch.Tensor, group=None) -> torch.Tensor:
    """In place: ``buf`` summed over the ranks of ``group`` with one all-reduce (the tensor exchange of the global-batch
    ``TCCALoss``); returns ``buf``."""
    dist.all_reduce(buf, op=dist.ReduceOp.SUM, group=group)
    return buf


def shard_rows(n_rows: int, rank: int, world: int):
    """Contiguous row block [lo, hi) of rank ``rank``."""
    base, rem = divmod(n_rows, world)
    lo = rank * base + min(rank, rem)
    return lo, lo + base + (1 if rank < rem else 0)
