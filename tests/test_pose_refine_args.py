"""NGP camera pose refinement without a GPU: argument validation of the three entry points (include/xrnerf_b200.h, "NGP camera pose refinement") before
any CUDA call, the trainer's and the ray source's refusals, and the Exp map's value and Jacobian (xrnerf_b200.data) against float64 autograd."""
import ctypes as C

import pytest
import torch


def _lib():
    from xrnerf_b200 import _C
    return _C, _C.lib


def test_backward_inputs_validation():
    _C, lib = _lib()
    cfg = _C.NgpConfig(16, 2, 19, 16, 1.38191288, 64, 1, 2)
    tab = _C.NgpTable(None, None, 0)
    buf = (C.c_char * 256)()
    p = C.c_void_p((C.addressof(buf) + 15) & ~15)
    args = lambda n, d_rows, stride=3, cfg=cfg: (C.byref(cfg), C.byref(tab), p, p, stride, p, 3, p, n, None, p, p, p, d_rows, None)   # noqa: E731
    assert lib.xrb_ngp_mlp_backward_tc_inputs(*args(0, None)) == 0                                       # empty batch: no-op
    assert lib.xrb_ngp_mlp_backward_tc_inputs(*args(-1, p)) == -1 and b'bad size' in lib.xrb_last_error()
    assert lib.xrb_ngp_mlp_backward_tc_inputs(*args(4, p, stride=2)) == -1
    assert lib.xrb_ngp_mlp_backward_tc_inputs(*args(4, None)) == -1 and b'd_rows' in lib.xrb_last_error()
    odd = C.c_void_p(p.value + 4)
    a = list(args(4, p)); a[7] = odd                                                                    # dl_draw not 16-byte aligned
    assert lib.xrb_ngp_mlp_backward_tc_inputs(*a) == -1 and b'aligned' in lib.xrb_last_error()
    deep = _C.NgpConfig(16, 2, 19, 16, 1.38191288, 64, 2, 2)
    assert lib.xrb_ngp_mlp_backward_tc_inputs(*args(4, p, cfg=deep)) == -2 and b'ngp_mlp_backward_tc_inputs' in lib.xrb_last_error()
    assert lib.xrb_ngp_mlp_backward_tc(*args(4, p, cfg=deep)[:13], None) == -2                            # the parameter-only entry as before


def test_ray_grad_validation():
    _C, lib = _lib()
    buf = (C.c_char * 64)()
    p = C.c_void_p(C.addressof(buf))
    assert lib.xrb_ngp_ray_grad(None, None, None, None, None, 0, 0.0, 1.0, 1.0, None, None, None) == 0
    assert lib.xrb_ngp_ray_grad(p, p, p, p, p, -1, 0.0, 1.0, 1.0, p, p, None) == -1 and b'negative' in lib.xrb_last_error()
    assert lib.xrb_ngp_ray_grad(p, p, p, p, p, 4, 1.0, 1.0, 1.0, p, p, None) == -1 and b'aabb' in lib.xrb_last_error()
    assert lib.xrb_ngp_ray_grad(p, p, p, p, None, 4, 0.0, 1.0, 1.0, p, p, None) == -1 and b'null' in lib.xrb_last_error()


def test_pose_grad_validation():
    _C, lib = _lib()
    buf = (C.c_char * 64)()
    p = C.c_void_p(C.addressof(buf))
    assert lib.xrb_ngp_pose_grad(None, 0, None, 1, 4, 4, 1.0, 1.0, 2.0, 2.0, None, None, None, None) == 0
    assert lib.xrb_ngp_pose_grad(p, -1, p, 1, 4, 4, 1.0, 1.0, 2.0, 2.0, p, p, p, None) == -1
    assert lib.xrb_ngp_pose_grad(p, 4, p, 0, 4, 4, 1.0, 1.0, 2.0, 2.0, p, p, p, None) == -1 and b'bad arguments' in lib.xrb_last_error()
    assert lib.xrb_ngp_pose_grad(p, 4, p, 1, 4, 4, 1.0, 1.0, 2.0, 2.0, p, None, p, None) == -1 and b'null' in lib.xrb_last_error()


def test_backward_rows_d_rows_needs_tensor_cores_and_shape():
    _C, _ = _lib()
    from xrnerf_b200.ngp import NgpField
    f = NgpField()
    pts = torch.zeros(8, 3)
    out = (torch.zeros(1), torch.zeros(1), torch.zeros(1))
    with pytest.raises(_C.XrbError, match='impl 1'):
        f.backward_rows(pts, pts, torch.zeros(8, 4), out, impl=0, d_rows=torch.zeros(8, 6))
    with pytest.raises(_C.XrbError, match=r'\[>= 8, 6\]'):
        f.backward_rows(pts, pts, torch.zeros(8, 4), out, impl=1, d_rows=torch.zeros(8, 3))
    with pytest.raises(_C.XrbError, match='float32'):
        f.backward_rows(pts, pts, torch.zeros(8, 4), out, impl=1, d_rows=torch.zeros(8, 6, dtype=torch.float64))


def test_trainer_ray_grad_refuses_unsupported_field():
    from xrnerf_b200.ngp import NgpField
    from xrnerf_b200.train import NgpTrainer
    with pytest.raises(ValueError, match='tensor-core field backward'):
        NgpTrainer(NgpField(density_hidden=2, color_hidden=2), None, 128, ray_grad=True)
    with pytest.raises(ValueError, match='tensor-core field backward'):
        NgpTrainer(NgpField(), None, 128, bwd_impl=0, ray_grad=True)


def _source(**kw):
    from xrnerf_b200.data import NgpRaySource
    poses = torch.eye(4)[:, :3][None].repeat(3, 1, 1)
    return NgpRaySource(poses, torch.rand(3, 4, 5, 4), [[4.0, 0, 2.5], [0, 4.0, 2.0], [0, 0, 1]], **kw)


def test_pose_step_needs_refine_poses_and_a_refinable_batch():
    _C, _ = _lib()
    g = torch.zeros(8, 3)
    with pytest.raises(_C.XrbError, match='refine_poses=True'):
        _source().pose_step({'rays_o': g}, g, g)
    src = _source(refine_poses=True)
    with pytest.raises(_C.XrbError, match='row_idx, pose_xi'):
        src.pose_step({'rays_o': g}, g, g)
    batch = {'row_idx': torch.zeros(8, dtype=torch.int64), 'pose_xi': torch.zeros(3, 6)}
    with pytest.raises(_C.XrbError, match=r'grad_d must be float32 \[8,3\]'):
        src.pose_step(batch, g, torch.zeros(8, 2))
    with pytest.raises(_C.XrbError, match=r'grad_o must be float32 \[8,3\]'):
        src.pose_step(batch, g.double(), g)
    with pytest.raises(_C.XrbError, match='CUDA'):
        src.pose_step(batch, g, g)                       # no CPU fallback
    assert torch.equal(src.refined_poses(), src.poses) and torch.equal(_source().refined_poses(), _source().poses)


def _exp64(omega):
    x, y, z = omega.unbind(-1)
    zr = torch.zeros_like(x)
    return torch.linalg.matrix_exp(torch.stack([zr, -z, y, z, zr, -x, -y, x, zr], -1).reshape(omega.shape[:-1] + (3, 3)))


@pytest.mark.parametrize('mag', [0.0, 1e-4, 0.3])
def test_exp_jacobian_matches_f64_autograd(mag):
    """corrected_poses and pose_xi_grad (float32) against float64 autograd of torch.linalg.matrix_exp, at omega = 0, tiny and |omega| = 0.3"""
    from xrnerf_b200.data import corrected_poses, pose_xi_grad
    g = torch.Generator().manual_seed(int(mag * 1e4) + 1)
    P = torch.cat([torch.linalg.qr(torch.randn(5, 3, 3, generator=g, dtype=torch.float64))[0], torch.randn(5, 1, 3, generator=g, dtype=torch.float64)], 1)
    xi = torch.randn(5, 6, generator=g, dtype=torch.float64)
    xi[:, :3] *= mag / xi[:, :3].norm(dim=1, keepdim=True)
    xi[:, 3:] *= 0.01
    dP = torch.randn(5, 4, 3, generator=g, dtype=torch.float64)
    x = xi.clone().requires_grad_(True)
    ref_P = torch.cat([_exp64(x[:, :3]).transpose(1, 2) @ P[:, :3], (P[:, 3] + x[:, 3:])[:, None]], 1)
    (ref_g,) = torch.autograd.grad(ref_P, x, dP)
    got_P = corrected_poses(P.float(), xi.float()).double()
    got_g = pose_xi_grad(P.float(), xi.float(), dP.float()).double()
    assert float((got_P - ref_P.detach()).abs().max()) <= 1e-6
    assert float((got_g - ref_g).abs().max()) <= 1e-6 * float(dP.abs().sum(dim=(1, 2)).max())
