"""Host logic of bfloat16 / float16 inputs, on the torch-CPU stand-in ops: which views reach the moment pass in their
own dtype, which routes still convert to float64, and the objectives' 16-bit route."""
import numpy as np
import pytest
import torch

from cca_zoo_b200 import _base
from cca_zoo_b200._base import BaseModel
from cca_zoo_b200.deep import CCALoss, GCCALoss, MCCALoss
from cca_zoo_b200.linear import TCCA, rCCA
from cca_zoo_b200.nonparametric import KCCA
from tests import fake_ops as F
from tests import fake_ops_global as FG


def _recording_moments_safe(monkeypatch):
    seen = []

    def moments_safe(views, precision="tf32x3b", x0=None):
        seen.append([v.dtype for v in views])
        return F.moments(views, precision), None

    monkeypatch.setattr(F, "moments_safe", moments_safe)
    return seen


def _views(dtype, n=50, dims=(6, 5)):
    g = torch.Generator().manual_seed(0)
    return [torch.randn(n, d, generator=g).to(dtype) for d in dims]


@pytest.mark.parametrize("dtype", [torch.bfloat16, torch.float16])
def test_local_moments_keeps_16_bit_tensors(monkeypatch, dtype):
    F.install(monkeypatch)
    seen = _recording_moments_safe(monkeypatch)
    mom, n, dims, in_dtype = rCCA()._local_moments(_views(dtype), torch.device("cpu"))
    assert seen == [[dtype, dtype]]
    assert in_dtype == torch.float64 and n == 50 and dims == [6, 5]


def test_local_moments_keeps_numpy_float16(monkeypatch):
    F.install(monkeypatch)
    seen = _recording_moments_safe(monkeypatch)
    views = [v.numpy() for v in _views(torch.float16)]
    _, _, _, in_dtype = rCCA()._local_moments(views, torch.device("cpu"))
    assert seen == [[torch.float16, torch.float16]] and in_dtype == torch.float64


@pytest.mark.parametrize("pair", [(torch.bfloat16, torch.float16), (torch.bfloat16, torch.float32)])
def test_local_moments_mixed_dtypes_go_to_float64(monkeypatch, pair):
    F.install(monkeypatch)
    seen = _recording_moments_safe(monkeypatch)
    views = [v.to(dt) for v, dt in zip(_views(torch.float32), pair)]
    _, _, _, in_dtype = rCCA()._local_moments(views, torch.device("cpu"))
    assert seen == [[torch.float64, torch.float64]] and in_dtype == torch.float64


def test_streamed_16_bit_chunks_stay_16_bit(monkeypatch):
    F.install(monkeypatch)
    chunks = []
    real = F.moments

    def moments(views, precision="tf32x3b"):
        chunks.append(views[0].dtype)
        return real(views, precision)

    monkeypatch.setattr(F, "moments", moments)
    est = rCCA()
    est._stream_threshold_bytes = 0
    est._stream_chunk_rows = 10
    monkeypatch.setattr(torch.cuda, "current_stream", lambda device=None: _NoStream(), raising=False)
    monkeypatch.setattr(torch.cuda, "stream", lambda s: _NullCtx(), raising=False)
    monkeypatch.setattr(torch.cuda, "Event", _NoEvent, raising=False)
    monkeypatch.setattr(_base, "_copy_stream", lambda device: _NoStream())
    monkeypatch.setattr(torch.Tensor, "record_stream", lambda self, s: None)
    monkeypatch.setattr(F, "SHIFT_RATIO", {**F.SHIFT_RATIO, torch.bfloat16: 16.0})   # the stand-in has float32/64 only
    _, n, _, in_dtype = est._local_moments(_views(torch.bfloat16, n=60), torch.device("cpu"))
    assert n == 60 and in_dtype == torch.float64
    assert chunks == [torch.bfloat16] * 6


class _NoStream:
    def wait_event(self, ev):
        pass


class _NullCtx:
    def __enter__(self):
        return self

    def __exit__(self, *a):
        return False


class _NoEvent:
    def record(self, s=None):
        pass


class _Stop(Exception):
    pass


def _record_to_device(monkeypatch):
    seen = []
    real = BaseModel._to_device

    def to_device(self, v, device):
        out = real(self, v, torch.device("cpu"))
        seen.append(out.dtype)
        raise _Stop

    monkeypatch.setattr(BaseModel, "_to_device", to_device)
    monkeypatch.setattr(BaseModel, "_device", lambda self: torch.device("cpu"))
    return seen


@pytest.mark.parametrize("make", [lambda: TCCA(latent_dimensions=1), lambda: KCCA(latent_dimensions=1)])
def test_tcca_and_kcca_still_convert_to_float64(monkeypatch, make):
    seen = _record_to_device(monkeypatch)
    with pytest.raises(_Stop):
        make().fit(_views(torch.bfloat16))
    assert seen == [torch.float64]


def test_transform_still_converts_to_float64(monkeypatch):
    seen = _record_to_device(monkeypatch)
    est = rCCA()
    est.means_ = [np.zeros(6), np.zeros(5)]
    est.weights_ = [np.ones((6, 1)), np.ones((5, 1))]
    with pytest.raises(_Stop):
        est._transform_device(_views(torch.bfloat16))
    assert seen == [torch.float64]


@pytest.mark.parametrize("dtype", [torch.bfloat16, torch.float16])
@pytest.mark.parametrize("kind,widths", [("CCALoss", [5, 4]), ("MCCALoss", [5, 4, 3]), ("GCCALoss", [4, 4, 4])])
def test_objectives_route_16_bit_to_the_moment_stage(monkeypatch, dtype, kind, widths):
    log = FG.install(monkeypatch)
    seen = []
    logged_moments = F.moments

    def moments(views, precision="tf32x3b"):
        seen.append({v.dtype for v in views})
        return logged_moments(views, precision)

    monkeypatch.setattr(F, "moments", moments)
    g = torch.Generator().manual_seed(1)
    zs = [torch.randn(40, w, generator=g).to(dtype).requires_grad_(True) for w in widths]
    loss = {"CCALoss": CCALoss, "MCCALoss": MCCALoss, "GCCALoss": GCCALoss}[kind]()(zs)
    assert loss.dtype == torch.float32
    loss.backward()
    assert seen == [{dtype}]                           # one moment pass, on the 16-bit representations as they are
    assert all(z.grad.dtype == dtype for z in zs)
    if kind != "GCCALoss":                             # GCCALoss reads N back, as its Jacobi sweeps do
        assert "read_n" not in log
