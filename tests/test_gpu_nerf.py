"""GPU parity of the NeRF / Mip-NeRF kernels against golden vectors produced by the reference's own PyTorch modules
(tests/golden/nerf_golden.npz) and, at larger sizes, against the numpy oracle. fp32 tolerance: 2e-5 abs/rel (scan order,
CUDA libm vs ATen CPU), gradients 1e-4 relative to the largest entry."""
import os

import numpy as np
import pytest
import torch
from cases import dev

pytestmark = pytest.mark.gpu
G = {**np.load(os.path.join(os.path.dirname(__file__), 'golden', 'nerf_golden.npz')), **np.load(os.path.join(os.path.dirname(__file__), 'golden', 'nerf_golden_embedded.npz'))}


def close(a, b, tol=2e-5):
    a = a.detach().cpu().numpy() if torch.is_tensor(a) else a
    return np.allclose(a, b, rtol=tol, atol=tol)


def test_posenc_golden():
    from xrnerf_b200.registry import BaseEmbedder
    e = BaseEmbedder(i_embed=0, multires=10, multires_dirs=4)
    d = e({'pts': dev(G['pts']), 'viewdirs': dev(G['viewdirs'])})
    assert d['embedded'].shape == (24 * 64, 90) and tuple(d['unflatten_shape']) == (24, 64)
    assert close(d['embedded'], G['embedded'], 5e-5)   # arguments up to 2^9 * 6 rad: CUDA sinf/cosf vs ATen CPU


@pytest.mark.parametrize('wb', [0, 1])
def test_nerf_render_golden_forward_backward(wb):
    from xrnerf_b200.registry import NerfRender
    t = f'render_wb{wb}.'
    r = NerfRender(white_bkgd=bool(wb), raw_noise_std=0)
    raw = dev(G[t + 'raw']).requires_grad_(True)
    data, ret = r({'raw': raw, 'z_vals': dev(G['z_vals']), 'rays_d': dev(G['rays_d'])}, is_test=True)
    for k in ('rgb', 'disp', 'acc'):
        assert close(ret[k], G[t + k]), k
    assert close(data['weights'], G[t + 'weights'])
    (ret['rgb'] * dev(G[t + 'grad_rgb'])).sum().backward()
    ref = G[t + 'd_raw']
    assert np.abs(raw.grad.cpu().numpy() - ref).max() <= 1e-4 * np.abs(ref).max()


def test_mip_render_golden_forward_backward():
    from xrnerf_b200.registry import MipNerfRender
    r = MipNerfRender(white_bkgd=True, raw_noise_std=0, rgb_padding=0.001, density_bias=-1, density_activation='softplus')
    raw = dev(G['mip.raw']).requires_grad_(True)
    data, ret = r({'raw': raw, 'z_vals': dev(G['mip.z_vals']), 'rays_d': dev(G['rays_d'])}, is_test=True)
    for k in ('rgb', 'disp', 'acc'):
        assert close(ret[k], G['mip.' + k]), k
    assert close(data['weights'], G['mip.weights'])
    (ret['rgb'] * dev(G['mip.grad_rgb'])).sum().backward()
    ref = G['mip.d_raw']
    assert np.abs(raw.grad.cpu().numpy() - ref).max() <= 1e-4 * np.abs(ref).max()


def test_sample_pdf_golden():
    from xrnerf_b200.registry.networks import sample_pdf
    from xrnerf_b200 import _C
    base = {'z_vals': dev(G['z_vals']), 'weights': dev(G['pdf.weights']), 'rays_o': dev(G['rays_o']), 'rays_d': dev(G['rays_d'])}
    d = sample_pdf(dict(base), 128, False, True)
    assert close(d['z_vals'], G['pdf.z_det']) and close(d['pts'], G['pdf.pts_det'], 5e-5)
    # caller-supplied uniforms (the reference's torch.rand path)
    z_out = torch.empty((24, 192), device='cuda')
    _C.check(_C.lib.xrb_nerf_sample_pdf(_C.ptr(base['z_vals']), _C.ptr(base['weights']), _C.ptr(base['rays_o']), _C.ptr(base['rays_d']), _C.ptr(dev(G['pdf.u'])), 24, 64, 128,
                                        _C.ptr(z_out), None, _C.stream()))
    assert close(z_out, G['pdf.z_rand'])
    assert (z_out[:, 1:] >= z_out[:, :-1]).all()


def test_mip_embed_and_resample_golden():
    from xrnerf_b200.registry import MipNerfEmbedder
    from xrnerf_b200.registry.networks import resample_along_rays
    from xrnerf_b200 import _C
    e = MipNerfEmbedder(min_deg_point=0, max_deg_point=16, min_deg_view=0, max_deg_view=4, use_viewdirs=True)
    data = {'z_vals': dev(G['mip.z_vals']), 'rays_o': dev(G['rays_o']), 'rays_d': dev(G['rays_d']), 'radii': dev(G['mip.radii']), 'viewdirs': dev(G['viewdirs'])}
    d = e(dict(data))
    assert d['embedded'].shape == G['mip.embedded'].shape
    assert close(d['embedded'], G['mip.embedded'], 1e-4)   # sin of arguments up to 2^15 * 6
    means = torch.empty((24, 32, 3), device='cuda'); covs = torch.empty((24, 32, 3), device='cuda'); emb = torch.empty_like(d['embedded'])
    _C.check(_C.lib.xrb_mip_embed(_C.ptr(data['z_vals']), _C.ptr(data['rays_o']), _C.ptr(data['rays_d']), _C.ptr(data['radii'].reshape(-1)), _C.ptr(data['viewdirs']), 24, 32, 0, 16, 0, 4,
                                  _C.ptr(emb), _C.ptr(means), _C.ptr(covs), _C.stream()))
    assert close(means, G['mip.means']) and np.allclose(covs.cpu().numpy(), G['mip.covs'], rtol=1e-4, atol=1e-9)
    d2 = resample_along_rays({'z_vals': dev(G['mip.z_vals']), 'weights': dev(G['mip.weights'])}, False, 'cone', 0.01)
    assert close(d2['z_vals'], G['mip.z_resampled'], 5e-5)


def test_composite_large_vs_numpy_oracle():
    """config-3 shape slice: 4096 rays x 192 samples"""
    from oracle import nerf_oracle as O
    from xrnerf_b200.registry import NerfRender
    rng = np.random.default_rng(0)
    n, s = 4096, 192
    raw = rng.normal(0, 1, (n, s, 4)).astype(np.float32)
    z = np.sort(rng.uniform(2, 6, (n, s)).astype(np.float32), -1)
    d = rng.normal(0, 1, (n, 3)).astype(np.float32)
    ref = O.nerf_render(raw, z, d, white_bkgd=True)
    data, ret = NerfRender(white_bkgd=True)({'raw': dev(raw), 'z_vals': dev(z), 'rays_d': dev(d)}, is_test=True)
    assert close(ret['rgb'], ref['rgb'], 5e-5) and close(ret['acc'], ref['acc'], 5e-5) and close(data['weights'], ref['weights'], 5e-5)


def test_ray_generation_golden():
    """xrb_nerf_get_rays / xrb_nerf_zvals vs the reference's GetRays(+radii)/GetViewdirs/GetZvals/PerturbZvals and get_rays_np_hash"""
    import ctypes as C
    from xrnerf_b200 import _C
    H, W, K = 12, 20, G['gen.K']
    n = H * W
    pose = np.ascontiguousarray(G['gen.pose'][:3, :4], np.float32)
    o = torch.empty((n, 3), device='cuda'); d = torch.empty((n, 3), device='cuda'); v = torch.empty((n, 3), device='cuda'); r = torch.empty((n, 1), device='cuda')
    c2w = (C.c_float * 12)(*pose.reshape(-1).tolist())
    _C.check(_C.lib.xrb_nerf_get_rays(c2w, H, W, float(K[0][0]), float(K[1][1]), float(K[0][2]), float(K[1][2]), 0, None, n, _C.ptr(o), _C.ptr(d), _C.ptr(v), _C.ptr(r), _C.stream()))
    assert close(o, G['gen.rays_o']) and close(d, G['gen.rays_d']) and close(v, G['gen.viewdirs']) and np.allclose(r.cpu().numpy(), G['gen.radii'], rtol=1e-4, atol=1e-7)
    _C.check(_C.lib.xrb_nerf_get_rays(c2w, H, W, float(K[0][0]), float(K[1][1]), float(K[0][2]), float(K[1][2]), 1, None, n, _C.ptr(o), _C.ptr(d), None, None, _C.stream()))
    assert close(o, G['gen.ngp_rays_o']) and close(d, G['gen.ngp_rays_d'])
    # a pixel subset (SelectRays) gives the same rays
    idx = torch.tensor([0, 7, 19, 20, 239, 101], dtype=torch.int32, device='cuda')
    o2 = torch.empty((6, 3), device='cuda'); d2 = torch.empty((6, 3), device='cuda')
    _C.check(_C.lib.xrb_nerf_get_rays(c2w, H, W, float(K[0][0]), float(K[1][1]), float(K[0][2]), float(K[1][2]), 1, _C.ptr(idx), 6, _C.ptr(o2), _C.ptr(d2), None, None, _C.stream()))
    assert torch.equal(d2, d[idx.long()])
    z = torch.empty((n, 64), device='cuda')
    _C.check(_C.lib.xrb_nerf_zvals(n, 64, 2.0, 6.0, 0, None, _C.ptr(z), _C.stream()))
    assert close(z, G['gen.z_lin'])
    _C.check(_C.lib.xrb_nerf_zvals(n, 64, 2.0, 6.0, 0, _C.ptr(dev(G['gen.u'])), _C.ptr(z), _C.stream()))
    assert close(z, G['gen.z_perturbed'])
    z33 = torch.empty((n, 33), device='cuda')
    _C.check(_C.lib.xrb_nerf_zvals(n, 33, 2.0, 6.0, 1, None, _C.ptr(z33), _C.stream()))
    assert close(z33, G['gen.z_lindisp'])
