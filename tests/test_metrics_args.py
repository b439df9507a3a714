"""CPU-only: xrb_ssim rejects bad arguments with XRB_E_BADARG before any CUDA call, and metrics.ssim rejects CPU tensors, mismatched shapes and
non-float32 images before it reaches the library."""
import ctypes as C
import math

import pytest


def _ssim(x=1, y=1, n=2, h=16, w=16, c=3, r=1.0, mf=1, mc=1, s=None, ws=1, ws_bytes=None):
    from xrnerf_b200 import _C
    lib = _C.lib
    buf = (C.c_double * 64)()
    a = C.addressof(buf)
    p = lambda v: None if not v else C.c_void_p(a)                                                    # noqa: E731
    if ws_bytes is None:
        ws_bytes = lib.xrb_ssim_workspace(n, h, w)
    return lib.xrb_ssim(p(x), p(y), n, h, w, c, r, p(mf), p(mc), p(s), p(ws), ws_bytes, None)


def test_ssim_rejects_bad_arguments_without_gpu():
    from xrnerf_b200 import _C
    lib = _C.lib
    cases = {
        'h < 7': dict(h=6), 'w < 7': dict(w=6), 'c = 0': dict(c=0), 'c = 5': dict(c=5), 'n < 0': dict(n=-1),
        'R = 0': dict(r=0.0), 'R < 0': dict(r=-1.0), 'R = inf': dict(r=math.inf), 'R = nan': dict(r=math.nan),
        'x null': dict(x=0), 'y null': dict(y=0), 'mean_full null': dict(mf=0), 'mean_crop null': dict(mc=0), 'workspace null': dict(ws=0),
        'short workspace': dict(ws_bytes=lib.xrb_ssim_workspace(2, 16, 16) - 1),
    }
    for what, kw in cases.items():
        assert _ssim(**kw) == _C.XRB_E_BADARG, what
        assert lib.xrb_last_error().startswith(b'ssim:'), what
    assert _ssim(h=6, x=0) == _C.XRB_E_BADARG and b'7x7' in lib.xrb_last_error()                      # sizes are checked first
    assert _ssim(n=0, x=0, y=0, mf=0, mc=0, ws=0, ws_bytes=0) == 0                                       # n == 0: a no-op touching no pointer
    assert _ssim(n=0, h=6) == _C.XRB_E_BADARG                                                           # ... but its sizes are still checked


def test_ssim_workspace_size_without_gpu():
    from xrnerf_b200 import _C
    lib = _C.lib
    assert lib.xrb_ssim_workspace(1, 7, 7) == 16                                                         # one 32 x 16 tile: two doubles
    assert lib.xrb_ssim_workspace(200, 800, 800) == 200 * 25 * 50 * 16
    assert lib.xrb_ssim_workspace(0, 800, 800) == 0
    assert lib.xrb_ssim_workspace(1, 6, 800) == 0 and lib.xrb_ssim_workspace(-1, 8, 8) == 0


def test_ssim_python_checks_without_gpu():
    import torch
    from xrnerf_b200 import _C, metrics
    x = torch.zeros(8, 8, 3)
    with pytest.raises(ValueError, match='same shape'):
        metrics.ssim(x, torch.zeros(8, 9, 3), 1.0)
    with pytest.raises(ValueError, match=r'\[H,W,C\]'):
        metrics.ssim(torch.zeros(8, 8), torch.zeros(8, 8), 1.0)
    with pytest.raises(_C.XrbError, match='float32'):
        metrics.ssim(x, torch.zeros(8, 8, 3, dtype=torch.float64), 1.0)
    with pytest.raises(_C.XrbError, match='float32'):
        metrics.ssim(x.half(), x.half(), 1.0)
    with pytest.raises(_C.XrbError, match='CUDA'):
        metrics.ssim(x, x, 1.0)
    m = metrics.TestMetrics(ndown=4)
    with pytest.raises(ValueError, match='no view'):
        m.summary()
