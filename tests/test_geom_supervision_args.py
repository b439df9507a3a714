"""CPU-only: the depth / opacity supervision entry points reject bad arguments before any CUDA call, and the registry builds with and without the new
cfg keys and render flag (include/xrnerf_b200.h, "Depth and opacity supervision")."""
import ctypes as C

import pytest

from cases import MIP_MODEL, NERF_MODEL, NGP_MODEL, host_buffer

BADARG = -1


def _lib():
    from xrnerf_b200 import _C
    _C.lib.xrb_last_error.restype = C.c_char_p
    return _C.lib


def test_calc_rgb_geom_argument_validation():
    lib = _lib()
    buf, a = host_buffer()
    p = C.c_void_p(a)
    ps = [p] * 7
    assert lib.xrb_rm_calc_rgb_forward_geom(*ps, -1, 0.0, 1.0, 2, 3, p, p, p, None) == BADARG
    assert lib.xrb_rm_calc_rgb_forward_geom(*ps, 0, 0.0, 1.0, 2, 3, None, None, None, None) == 0          # n == 0 touches nothing
    for k in range(10):                                                                                  # every pointer is required
        args = ps + [p, p, p]
        args[k] = None
        assert lib.xrb_rm_calc_rgb_forward_geom(*args[:7], 4, 0.0, 1.0, 2, 3, *args[7:], None) == BADARG, k
    assert lib.xrb_rm_calc_rgb_forward_geom(C.c_void_p(a + 4), *ps[1:], 4, 0.0, 1.0, 2, 3, p, p, p, None) == BADARG   # raw misaligned
    assert b'calc_rgb_forward_geom' in lib.xrb_last_error()
    bw = [p] * 8
    assert lib.xrb_rm_calc_rgb_backward_geom(*bw, 0.0, 1.0, p, p, p, p, -1, 2, 3, p, None) == BADARG
    for k in [0, 1, 2, 3, 4, 5, 6, 7]:
        args = list(bw)
        args[k] = None
        assert lib.xrb_rm_calc_rgb_backward_geom(*args, 0.0, 1.0, p, p, None, None, 4, 2, 3, p, None) == BADARG, k
    assert lib.xrb_rm_calc_rgb_backward_geom(*bw, 0.0, 1.0, None, p, p, p, 4, 2, 3, p, None) == BADARG      # forward depth missing
    assert lib.xrb_rm_calc_rgb_backward_geom(*bw, 0.0, 1.0, p, None, p, p, 4, 2, 3, p, None) == BADARG      # forward alpha missing
    assert lib.xrb_rm_calc_rgb_backward_geom(*bw, 0.0, 1.0, p, p, p, p, 4, 2, 3, None, None) == BADARG
    assert lib.xrb_rm_calc_rgb_backward_geom(*bw, 0.0, 1.0, p, p, p, p, 4, 2, 3, C.c_void_p(a + 4), None) == BADARG
    del buf


def test_nerf_composite_backward_geom_argument_validation():
    lib = _lib()
    buf, a = host_buffer()
    p = C.c_void_p(a)
    f = C.c_float
    assert lib.xrb_nerf_composite_backward_geom(p, p, p, p, p, p, -1, 8, 0, 0, f(0), f(0), 1, p, None) == BADARG
    assert lib.xrb_nerf_composite_backward_geom(p, p, p, p, p, p, 4, 0, 0, 0, f(0), f(0), 1, p, None) == BADARG
    assert lib.xrb_nerf_composite_backward_geom(p, p, p, p, p, p, 4, 8, 0, 0, f(0), f(0), 3, p, None) == -2     # density activation
    assert lib.xrb_nerf_composite_backward_geom(p, p, p, None, p, p, 4, 8, 0, 0, f(0), f(0), 1, p, None) == BADARG
    assert lib.xrb_nerf_composite_backward_geom(p, p, p, p, p, p, 4, 8, 0, 0, f(0), f(0), 1, None, None) == BADARG
    assert lib.xrb_nerf_composite_backward_geom(p, p, p, p, p, p, 4, 8, 0, 0, f(0), f(0), 1, C.c_void_p(a + 4), None) == BADARG
    assert lib.xrb_nerf_composite_backward_geom(C.c_void_p(a + 4), p, p, p, p, p, 4, 8, 0, 0, f(0), f(0), 1, p, None) == BADARG
    assert lib.xrb_nerf_composite_backward_geom(None, None, None, None, None, None, 0, 8, 0, 0, f(0), f(0), 1, None, None) == 0
    del buf


def test_geom_loss_argument_validation():
    lib = _lib()
    buf, a = host_buffer()
    p = C.c_void_p(a)
    f = C.c_float

    def call(depth=p, alpha=p, td=p, ta=p, ns=None, nsc=None, n=4, wd=1.0, wa=1.0, mean=0, gd=p, ga=p, loss=p):
        return lib.xrb_geom_loss_grad(depth, alpha, td, ta, ns, nsc, n, f(wd), f(wa), mean, gd, ga, loss, None)
    assert call(n=-1) == BADARG
    assert call(wd=-1.0) == BADARG and call(wa=float('nan')) == BADARG and call(wd=float('inf')) == BADARG
    assert call(mean=2) == BADARG
    assert call(ns=p) == BADARG and call(nsc=p) == BADARG
    assert call(loss=None) == BADARG
    for k in ('depth', 'td', 'gd'):
        assert call(**{k: None}) == BADARG, k
        assert b'depth_weight' in lib.xrb_last_error()
    for k in ('alpha', 'ta', 'ga'):
        assert call(**{k: None}) == BADARG, k
    assert call(depth=None, alpha=None, td=None, ta=None, gd=None, ga=None, loss=None, n=0) == 0
    del buf


def test_ngp_batch_depth_argument_validation():
    lib = _lib()
    buf, a = host_buffer()
    p = C.c_void_p(a)
    f = C.c_float
    k = (f(100.0), f(100.0), f(50.0), f(50.0), f(0.33))
    assert lib.xrb_ngp_batch_depth(p, 0, 8, 8, *k, p, 4, p, None) == BADARG
    assert lib.xrb_ngp_batch_depth(p, 1, 0, 8, *k, p, 4, p, None) == BADARG
    assert lib.xrb_ngp_batch_depth(p, 1, 8, 8, *k, p, -1, p, None) == BADARG
    for i in range(3):
        args = [p, p, p]
        args[i] = None
        assert lib.xrb_ngp_batch_depth(args[0], 1, 8, 8, *k, args[1], 4, args[2], None) == BADARG, i
    assert lib.xrb_ngp_batch_depth(None, 1, 8, 8, *k, None, 0, None, None) == 0
    del buf


@pytest.mark.parametrize('model', ['nerf', 'mip', 'ngp'])
def test_registry_builds_with_and_without_geometry_keys(model):
    from xrnerf_b200 import registry as R
    base = {'nerf': NERF_MODEL, 'mip': MIP_MODEL, 'ngp': NGP_MODEL}[model]
    plain = R.build_network(base)
    assert plain.depth_loss_weight == 0.0 and plain.opacity_loss_weight == 0.0 and not plain.render.geometry_grad
    cfg = dict(base['cfg'], depth_loss_weight=0.5, opacity_loss_weight=2.0)
    geo = R.build_network(dict(base, cfg=cfg, render=dict(base['render'], geometry_grad=True)))
    assert geo.depth_loss_weight == 0.5 and geo.opacity_loss_weight == 2.0 and geo.render.geometry_grad
