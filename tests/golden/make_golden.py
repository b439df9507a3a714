"""Generates tests/golden/nerf_golden.npz by running the REFERENCE's own PyTorch modules (imported unmodified from
/root/reference through oracle/ref_import.py) on seeded inputs. Run in the build container only:

    python tests/golden/make_golden.py

The .npz is committed; the GPU box (no /root/reference) only reads it.
"""
import os
import sys

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, ROOT)
from oracle import ref_import as R  # noqa: E402


def main():
    torch.manual_seed(0)
    torch.set_num_threads(1)
    emb = R.load('embedders.base'); mlpm = R.load('mlps.nerf_mlp'); rnd = R.load('renders.nerf_render'); hs = R.load('networks.utils.hierarchical_sample')
    mip = R.load('networks.utils.mip'); me = R.load('embedders.mipnerf_embedder'); mr = R.load('renders.mipnerf_render')
    out = {}
    N, S = 24, 64
    rays_o = torch.rand(N, 3) * 0.2
    rays_d = torch.randn(N, 3)
    viewdirs = rays_d / rays_d.norm(dim=-1, keepdim=True)
    t = torch.linspace(0., 1., S)
    z = (2.0 * (1 - t) + 6.0 * t).expand(N, S).contiguous()
    mids = .5 * (z[..., 1:] + z[..., :-1])
    upper = torch.cat([mids, z[..., -1:]], -1); lower = torch.cat([z[..., :1], mids], -1)
    z = lower + (upper - lower) * torch.rand(z.shape)          # PerturbZvals (datasets/pipelines/augment.py:269-283)
    pts = rays_o[..., None, :] + rays_d[..., None, :] * z[..., :, None]
    # --- BaseEmbedder + NerfMLP (small width so the fixture stays small; same code path as 256)
    m = mlpm.NerfMLP(skips=[4], netdepth=8, netwidth=64, output_ch=5, use_viewdirs=True, netchunk=1024,
                     embedder=dict(type='BaseEmbedder', i_embed=0, multires=10, multires_dirs=4))
    data = {'pts': pts.clone(), 'viewdirs': viewdirs.clone()}
    e = m.embedder(dict(data))['embedded']
    data = m(data)
    raw = data['raw'].detach()
    out.update(rays_o=rays_o, rays_d=rays_d, viewdirs=viewdirs, z_vals=z, pts=pts, embedded=e.detach(), raw=raw)
    for k, v in m.state_dict().items():
        out['mlp.' + k] = v
    # --- NerfRender (white bkgd on/off), gradients wrt raw
    for wb in (False, True):
        r = rnd.NerfRender(white_bkgd=wb, raw_noise_std=0)
        raw_g = (raw * 3).clone().requires_grad_(True)
        d2, ret = r({'raw': raw_g, 'z_vals': z, 'rays_d': rays_d}, is_test=True)
        g = torch.linspace(-1, 1, N * 3).reshape(N, 3)
        (ret['rgb'] * g).sum().backward()
        tag = f'render_wb{int(wb)}.'
        out.update({tag + 'raw': raw_g.detach(), tag + 'rgb': ret['rgb'].detach(), tag + 'disp': ret['disp'].detach(), tag + 'acc': ret['acc'].detach(),
                    tag + 'weights': d2['weights'].detach(), tag + 'grad_rgb': g, tag + 'd_raw': raw_g.grad})
    # --- sample_pdf deterministic (is_test) and with a fixed u (perturb): monkeypatch torch.rand for reproducible u
    r = rnd.NerfRender(white_bkgd=False, raw_noise_std=0)
    d2, _ = r({'raw': raw * 3, 'z_vals': z, 'rays_d': rays_d}, is_test=True)
    w = d2['weights'].detach()
    dd = hs.sample_pdf({'z_vals': z, 'rays_o': rays_o, 'rays_d': rays_d, 'weights': w}, 128, False, True)
    out.update({'pdf.weights': w, 'pdf.z_det': dd['z_vals'], 'pdf.pts_det': dd['pts']})
    u = torch.rand(N, 128)
    orig = torch.rand
    torch.rand = lambda *a, **k: u
    dd = hs.sample_pdf({'z_vals': z, 'rays_o': rays_o, 'rays_d': rays_d, 'weights': w}, 128, True, False)
    torch.rand = orig
    out.update({'pdf.u': u, 'pdf.z_rand': dd['z_vals']})
    # --- Mip-NeRF: cast_rays, IPE, pos_enc, MipNerfRender, resample
    S1 = 33
    zm = torch.linspace(2., 6., S1).expand(N, S1).contiguous() + torch.rand(N, S1) * 0.05
    zm, _ = torch.sort(zm, -1)
    radii = torch.rand(N, 1) * 0.002 + 0.0005
    means, covs = mip.cast_rays(zm, rays_o, rays_d, radii, 'cone')
    embm = me.MipNerfEmbedder(min_deg_point=0, max_deg_point=16, min_deg_view=0, max_deg_view=4, use_viewdirs=True)
    ed = embm({'samples': (means, covs), 'viewdirs': viewdirs})
    out.update({'mip.z_vals': zm, 'mip.radii': radii, 'mip.means': means, 'mip.covs': covs, 'mip.embedded': ed['embedded']})
    rawm = torch.randn(N, S1 - 1, 4)
    rm_ = mr.MipNerfRender(white_bkgd=True, raw_noise_std=0, rgb_padding=0.001, density_bias=-1, density_activation='softplus')
    rawm_g = rawm.clone().requires_grad_(True)
    d3, ret = rm_({'raw': rawm_g, 'z_vals': zm, 'rays_d': rays_d}, is_test=True)
    g = torch.linspace(-1, 1, N * 3).reshape(N, 3)
    (ret['rgb'] * g).sum().backward()
    out.update({'mip.raw': rawm, 'mip.rgb': ret['rgb'].detach(), 'mip.disp': ret['disp'].detach(), 'mip.acc': ret['acc'].detach(), 'mip.weights': d3['weights'].detach(),
                'mip.grad_rgb': g, 'mip.d_raw': rawm_g.grad})
    d4 = mip.resample_along_rays({'rays_o': rays_o, 'rays_d': rays_d, 'radii': radii, 'z_vals': zm, 'weights': d3['weights'].detach().clone()}, False, 'cone', 0.01)
    out.update({'mip.z_resampled': d4['z_vals'], 'mip.means2': d4['samples'][0], 'mip.covs2': d4['samples'][1]})
    # --- ray generation (SURVEY §8 a1-a5): GetRays(+radii) / GetViewdirs / GetBounds / GetZvals / PerturbZvals / GetPts and the NGP get_rays_np_hash
    create, augment, get_rays = R.load_pipelines()
    Hh, Ww, foc = 12, 20, 27.5
    K = np.array([[foc, 0, 0.5 * Ww], [0, foc, 0.5 * Hh], [0, 0, 1]], np.float32)
    pose = torch.tensor([[0.36, -0.48, 0.8, 1.5], [0.8, 0.6, 0.0, -0.7], [-0.48, 0.64, 0.6, 2.2], [0, 0, 0, 1]], dtype=torch.float32)
    kw = dict(H=Hh, W=Ww, K=K, near=2.0, far=6.0)
    res = create.GetRays(include_radius=True, **kw)({'pose': pose})
    res = create.GetViewdirs(**kw)(res)
    res = create.GetBounds(**kw)(res)
    res['rays_o'] = res['rays_o'].reshape(-1, 3); res['rays_d_flat'] = res['rays_d'].reshape(-1, 3)
    res['near'] = res['near'].reshape(-1, 1); res['far'] = res['far'].reshape(-1, 1)
    zres = create.GetZvals(N_samples=64, lindisp=False, randomized=False, **kw)(dict(rays_o=res['rays_o'], near=res['near'], far=res['far']))
    zlin = create.GetZvals(N_samples=33, lindisp=True, randomized=False, **kw)(dict(rays_o=res['rays_o'], near=res['near'], far=res['far']))
    uz = torch.rand(Hh * Ww, 64)
    orig = torch.rand
    torch.rand = lambda *a, **k: uz
    zper = augment.PerturbZvals()({'z_vals': zres['z_vals'].clone()})
    torch.rand = orig
    ptsg = create.GetPts()({'rays_o': res['rays_o'], 'rays_d': res['rays_d_flat'], 'z_vals': zres['z_vals']})
    ro_h, rd_h = get_rays.get_rays_np_hash(Hh, Ww, K, pose[:3, :4].numpy().T.copy())
    out.update({'gen.pose': pose, 'gen.K': K, 'gen.rays_o': res['rays_o'], 'gen.rays_d': res['rays_d_flat'], 'gen.viewdirs': res['viewdirs'], 'gen.radii': res['radii'].reshape(-1, 1),
                'gen.z_lin': zres['z_vals'], 'gen.z_lindisp': zlin['z_vals'], 'gen.u': uz, 'gen.z_perturbed': zper['z_vals'], 'gen.pts': ptsg['pts'],
                'gen.ngp_rays_o': ro_h.reshape(-1, 3).astype(np.float32), 'gen.ngp_rays_d': rd_h.reshape(-1, 3).astype(np.float32)})
    # --- losses / metrics of the train steps (networks/utils/metrics.py:3-16; nerf.py:71-92, hashnerf.py:32-52, mipnerf.py:45-74)
    met = R.load('networks.utils.metrics')
    lx = torch.rand(96, 3); ly = (lx + 0.25 * torch.randn(96, 3)).clamp(0, 1)
    lxg = lx.clone().requires_grad_(True)
    h5 = met.HuberLoss(lxg, ly, 0.1, 'sum') * 5
    h5.backward()
    mse = met.img2mse(lx, ly)
    out.update({'loss.x': lx, 'loss.y': ly, 'loss.huber_sum': met.HuberLoss(lx, ly, 0.1, 'sum'), 'loss.huber_mean': met.HuberLoss(lx, ly, 0.1, 'mean'),
                'loss.huber5_grad': lxg.grad, 'loss.mse': mse, 'loss.psnr': met.mse2psnr(mse)})
    out = {k: (v.detach().numpy() if torch.is_tensor(v) else np.asarray(v)) for k, v in out.items()}
    big = ('embedded', 'mip.embedded')   # in a file of their own: every stored file stays under 1 MB
    here = os.path.dirname(os.path.abspath(__file__))
    np.savez_compressed(os.path.join(here, 'nerf_golden.npz'), **{k: v for k, v in out.items() if k not in big})
    np.savez_compressed(os.path.join(here, 'nerf_golden_embedded.npz'), **{k: out[k] for k in big})
    print('wrote nerf_golden.npz and nerf_golden_embedded.npz with', len(out), 'arrays')


if __name__ == '__main__':
    main()
