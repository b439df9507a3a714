"""Pins oracle/nerf_oracle.py (numpy restatement) against golden vectors produced by the reference's OWN PyTorch modules
(tests/golden/make_golden.py). CPU-only. fp32 tolerances: 1e-5 abs/rel (different summation order numpy vs ATen), bin
indices of sample_pdf exact through the sorted z_vals (1e-5)."""
import os

import numpy as np
import pytest

from oracle import nerf_oracle as O

G = {**np.load(os.path.join(os.path.dirname(__file__), 'golden', 'nerf_golden.npz')), **np.load(os.path.join(os.path.dirname(__file__), 'golden', 'nerf_golden_embedded.npz'))}


def close(a, b, tol=1e-5):
    return np.allclose(a, b, rtol=tol, atol=tol)


def test_embed_and_mlp():
    e = O.embed(G['pts'], G['viewdirs'])
    assert e.shape == G['embedded'].shape == (24 * 64, 90)
    assert close(e, G['embedded'], 2e-5)
    sd = {k[4:]: G[k] for k in G if k.startswith('mlp.')}
    raw = O.nerf_mlp(sd, G['embedded'], 63, 27).reshape(24, 64, 4)
    assert close(raw, G['raw'], 1e-4)


@pytest.mark.parametrize('wb', [0, 1])
def test_nerf_render(wb):
    t = f'render_wb{wb}.'
    r = O.nerf_render(G[t + 'raw'], G['z_vals'], G['rays_d'], white_bkgd=bool(wb))
    for k in ('rgb', 'disp', 'acc', 'weights'):
        assert close(r[k], G[t + k], 2e-5), k


def test_sample_pdf():
    z, pts, _ = O.sample_pdf(G['z_vals'], G['pdf.weights'], G['rays_o'], G['rays_d'], 128)
    assert close(z, G['pdf.z_det']) and close(pts, G['pdf.pts_det'], 2e-5)
    z, _, _ = O.sample_pdf(G['z_vals'], G['pdf.weights'], G['rays_o'], G['rays_d'], 128, u=G['pdf.u'])
    assert close(z, G['pdf.z_rand'])


def test_mip():
    means, covs = O.cast_rays(G['mip.z_vals'], G['rays_o'], G['rays_d'], G['mip.radii'])
    assert close(means, G['mip.means']) and np.allclose(covs, G['mip.covs'], rtol=1e-4, atol=1e-9)
    ipe = O.integrated_pos_enc(G['mip.means'], G['mip.covs']).reshape(-1, 96)
    pe = O.mip_pos_enc(G['viewdirs'])
    emb = np.concatenate([ipe, np.repeat(pe[:, None, :], 32, 1).reshape(-1, 27)], -1)
    assert close(emb, G['mip.embedded'], 2e-5)
    r = O.nerf_render(G['mip.raw'], G['mip.z_vals'], G['rays_d'], white_bkgd=True, rgb_padding=0.001, density_bias=-1, density_activation='softplus', mip=True)
    for k in ('rgb', 'disp', 'acc', 'weights'):
        assert close(r[k], G['mip.' + k], 2e-5), k
    z2 = O.resample_along_rays(G['mip.z_vals'], G['mip.weights'])
    assert close(z2, G['mip.z_resampled'], 2e-5)


def test_ray_generation():
    r = O.get_rays(G['gen.pose'], 12, 20, G['gen.K'])
    assert close(r['rays_o'], G['gen.rays_o']) and close(r['rays_d'], G['gen.rays_d']) and close(r['viewdirs'], G['gen.viewdirs']) and close(r['radii'], G['gen.radii'], 1e-6)
    ro, rd = O.get_rays_ngp(G['gen.pose'][:3, :4].T, 12, 20, G['gen.K'])
    assert close(ro, G['gen.ngp_rays_o']) and close(rd, G['gen.ngp_rays_d'])
    assert close(O.z_vals(240, 64, 2.0, 6.0), G['gen.z_lin']) and close(O.z_vals(240, 33, 2.0, 6.0, lindisp=True), G['gen.z_lindisp'])
    assert close(O.z_vals(240, 64, 2.0, 6.0, u=G['gen.u']), G['gen.z_perturbed'])
    assert close(G['gen.rays_o'][:, None] + G['gen.rays_d'][:, None] * G['gen.z_lin'][..., None], G['gen.pts'])
