"""The TF32 moment paths read the views with TMA, which needs 16-byte aligned rows: ccab_moments rejects a view whose
pointer or leading dimension breaks that (include/ccab200.h) with an error instead of launching."""
import ctypes as C

import pytest
import torch

pytestmark = pytest.mark.gpu


def _call(views, lds, precision):
    from cca_zoo_b200 import _lib

    lib = _lib.load()
    n, dims = views[0].shape[0], _lib.i64_array([v.shape[1] for v in views])
    ptrs = (C.c_void_p * len(views))(*[v.data_ptr() for v in views])
    mom = torch.zeros(lib.ccab_moments_size(len(views), dims), dtype=torch.float64, device="cuda")
    ws = torch.empty(lib.ccab_moments_workspace_bytes(_lib.F32, precision, len(views), dims, n) + 256,
                     dtype=torch.uint8, device="cuda")
    stream = C.c_void_p(torch.cuda.current_stream().cuda_stream)
    rc = lib.ccab_moments(_lib.F32, precision, len(views), ptrs, dims, _lib.i64_array(lds), n, mom.data_ptr(),
                          ws.data_ptr(), ws.numel(), stream)
    torch.cuda.synchronize()
    return rc, _lib.last_error(), mom


@pytest.mark.parametrize("precision", [0, 1, 3])
def test_tf32_moments_reject_unaligned_views(precision):
    base = torch.randn(300, 132, device="cuda")
    ok = base[:, :130]
    rc, _, _ = _call([ok, ok], [132, 132], precision)
    assert rc == 0
    odd_ld = torch.randn(300 * 131, device="cuda").view(300, 131)
    rc, err, _ = _call([ok, odd_ld], [132, 131], precision)
    assert rc != 0 and "aligned" in err
    shifted = base.view(-1)[1:].as_strided((299, 130), (132, 1))   # 4-byte offset pointer, ld % 4 == 0
    rc, err, _ = _call([shifted, shifted], [132, 132], precision)
    assert rc != 0 and "aligned" in err
