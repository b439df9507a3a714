"""GPU parity of the device-side ray sources (SURVEY §8f-1) and of the randomized sampling branches against golden vectors produced by the REFERENCE's own
transforms (tests/golden/make_golden_r2.py: load_rays_hash / HashBatchSample / RandomBGColor / SelectRays / GetZvals(randomized) / resample_along_rays(randomized)
imported unmodified, their RNG draws recorded). Tolerances: rays 2e-6 abs (fp32, same expression order), blended targets 1e-6, z values 2e-5."""
import os

import numpy as np
import pytest
import torch
from cases import dev

pytestmark = pytest.mark.gpu
G = np.load(os.path.join(os.path.dirname(os.path.abspath(__file__)), 'golden', 'nerf_golden_r2.npz'))


def test_ngp_ray_source_matches_reference_table_batching_and_bg():
    from xrnerf_b200.data import NgpRaySource
    src = NgpRaySource(G['batch.poses'], G['batch.images'], G['batch.K']).cuda().shuffle(perm=G['batch.perm'])
    # the un-shuffled table itself: rows 0..23 of load_rays_hash
    head = src.rows(torch.arange(24).cuda(), u_bg=np.zeros((24, 3), np.float32))
    t = G['batch.table_head']
    assert np.abs(head['rays_o'].cpu().numpy() - t[:, :3]).max() <= 2e-6 and np.abs(head['rays_d'].cpu().numpy() - t[:, 3:6]).max() <= 2e-6
    assert np.array_equal(head['alpha'].cpu().numpy(), t[:, 9:10]) and np.array_equal(head['img_ids'].cpu().numpy(), t[:, 10:])
    for b in range(2):                                             # two consecutive HashBatchSample slices of the shuffled table, RandomBGColor on top
        out = src.next_batch(16, u_bg=G['batch.u_bg'][b])
        for k, tol in (('rays_o', 2e-6), ('rays_d', 2e-6), ('target_s', 1e-6), ('alpha', 0), ('img_ids', 0), ('bg_color', 1e-7)):
            assert np.abs(out[k].cpu().numpy() - G[f'batch.{b}.{k}']).max() <= tol, (b, k)
    # device-drawn backgrounds: uniform in [0,1), different per ray, target = rgb*alpha + bg*(1-alpha)
    out = src.next_batch(16)
    bg = out['bg_color'].cpu().numpy()
    assert (bg >= 0).all() and (bg < 1).all() and len(np.unique(bg)) > 40
    # wrap-around rule of HashBatchSample (create.py:168-171)
    src.cur_i = src.n_rows - 10
    src.next_batch(16)
    assert src.cur_i == 16


def test_select_rays_and_nerf_ray_source_match_reference():
    from xrnerf_b200.data import NerfRaySource, select_rays_indices
    H, W = G['select.image'].shape[:2]
    K, pose, img = G['select.K'], G['select.pose'], dev(G['select.image'])
    src = NerfRaySource(H, W, K, include_radius=True)
    for tag, it in (('full', 100), ('crop', 3)):
        pix = select_rays_indices(H, W, 24, iter_n=it, precrop_iters=10, precrop_frac=0.5, select_inds=G[f'select.{tag}.inds'])
        out = src.batch(pose, img, pix)
        for k, tol in (('rays_o', 1e-6), ('rays_d', 2e-6), ('target_s', 0), ('radii', 1e-7)):
            assert np.abs(out[k].cpu().numpy() - G[f'select.{tag}.{k}']).max() <= tol, (tag, k)
    pix = select_rays_indices(H, W, 50, generator=torch.Generator().manual_seed(0))
    assert len(set(pix.tolist())) == 50 and int(pix.max()) < H * W      # without replacement, inside the image


def test_randomized_zvals_and_mip_resample_match_reference():
    from xrnerf_b200 import _C
    from xrnerf_b200.registry.networks import resample_along_rays
    u = dev(G['zrand.u'])
    n, s = u.shape
    z = torch.empty((n, s), device='cuda')
    _C.check(_C.lib.xrb_nerf_zvals(n, s, 2.0, 6.0, 0, _C.ptr(u), _C.ptr(z), _C.stream()))       # GetZvals(randomized=True) == the stratified jitter of PerturbZvals on the linspace
    assert np.abs(z.cpu().numpy() - G['zrand.z']).max() <= 2e-6
    data = {'z_vals': dev(G['mipr.z_vals']), 'weights': dev(G['mipr.weights'])}
    out = resample_along_rays(data, True, 'cone', 0.01, rand=dev(G['mipr.u']))
    assert np.abs(out['z_vals'].cpu().numpy() - G['mipr.z_resampled']).max() <= 2e-5
