"""Fused inference path of the hierarchical NeRF (NerfNetwork.forward with N_importance > 0,
/root/reference/xrnerf/models/networks/nerf.py:39-48 + the val pipeline's GetZvals/GetPts, datasets/pipelines/create.py:486-597) for a batch of rays:

  z_vals (linspace) -> [posenc straight into fp16 tile images (wgmma operand layout), positions formed in registers] -> coarse NerfMLP (wgmma) -> composite ->
  sample_pdf (one kernel) -> posenc tiles -> fine NerfMLP (wgmma) -> composite

No [N,S,3] `pts`, no fp32 `embedded`, no per-chunk Python loop: 7 kernel launches per ray batch of any size.
"""
import torch

from . import _C
from .nerf_mlp import nerf_mlp_forward_tiles


class NerfRenderer:
    def __init__(self, network, near=2.0, far=6.0, n_samples=64):
        """network: registry NerfNetwork (mlp, mlp_fine, render); BaseEmbedder encodings."""
        self.net, self.near, self.far, self.S = network, near, far, n_samples
        e = network.mlp.embedder
        self.multires, self.multires_dirs = e.multires, e.multires_dirs

    def _mlp(self, mlp, rays_o, rays_d, viewdirs, z):
        n, s = z.shape
        rows = n * s
        enc = torch.empty(_C.lib.xrb_nerf_enc_image_bytes(rows, mlp.input_ch), dtype=torch.uint8, device=z.device)
        _C.check(_C.lib.xrb_nerf_posenc_tiles_rays(_C.ptr(rays_o), _C.ptr(rays_d), _C.ptr(z), _C.ptr(viewdirs), n, s, self.multires, self.multires_dirs, _C.ptr(enc), _C.stream()),
                 'posenc_tiles_rays')
        image, bias = mlp._packed()
        return nerf_mlp_forward_tiles(image, bias, enc, rows, mlp.input_ch, mlp.input_ch_dirs).view(n, s, 4)

    @torch.no_grad()
    def render(self, rays_o, rays_d, viewdirs):
        from .registry.networks import sample_pdf
        net = self.net
        n = rays_o.shape[0]
        rays_o, rays_d, viewdirs = (x.contiguous().float() for x in (rays_o, rays_d, viewdirs))   # the kernels read dense [n,3] rows
        t = torch.linspace(0., 1., self.S, device=rays_o.device)
        z = (self.near * (1. - t) + self.far * t).expand(n, self.S).contiguous()           # GetZvals (create.py:502-531), lindisp=False
        data = {'rays_o': rays_o, 'rays_d': rays_d, 'viewdirs': viewdirs, 'z_vals': z}
        data['raw'] = self._mlp(net.mlp, rays_o, rays_d, viewdirs, z)
        data, ret = net.render(data, is_test=True)
        if getattr(net, 'N_importance', 0) > 0:
            data['pts'] = None
            data = sample_pdf(data, net.N_importance, False, True)
            data['raw'] = self._mlp(net.mlp_fine, rays_o, rays_d, viewdirs, data['z_vals'])
            _, fine = net.render(data, is_test=True)
            ret = {'coarse_rgb': ret['rgb'], 'rgb': fine['rgb'], 'disp': fine['disp'], 'acc': fine['acc']}
        return ret


class MipNerfRenderer:
    """Fused inference path of MipNerfNetwork.forward(is_test=True) (/root/reference/xrnerf/models/networks/mipnerf.py:25-43): per level
    [cast_rays + IPE straight into fp16 tile images (wgmma operand layout)] -> the SAME NerfMLP (wgmma) -> MipNerfRender composite, with resample_along_rays
    (one kernel) between the levels: 3 launches per level + 1, no [N,S,3] means/covs, no fp32 `embedded` [N*S,123]."""

    def __init__(self, network, near=2.0, far=6.0, n_samples=128):
        self.net, self.near, self.far, self.S = network, near, far, n_samples
        e = network.mlp.embedder
        self.degs = (e.min_deg, e.max_deg, e.min_deg_view, e.max_deg_view)

    def _mlp(self, rays_o, rays_d, viewdirs, radii, z):
        mlp = self.net.mlp
        n, s = z.shape[0], z.shape[1] - 1
        rows = n * s
        enc = torch.empty(_C.lib.xrb_nerf_enc_image_bytes(rows, mlp.input_ch), dtype=torch.uint8, device=z.device)
        _C.check(_C.lib.xrb_mip_ipe_tiles_rays(_C.ptr(z), _C.ptr(rays_o), _C.ptr(rays_d), _C.ptr(radii), _C.ptr(viewdirs), n, s, *self.degs, _C.ptr(enc), _C.stream()), 'mip_ipe_tiles_rays')
        image, bias = mlp._packed()
        return nerf_mlp_forward_tiles(image, bias, enc, rows, mlp.input_ch, mlp.input_ch_dirs).view(n, s, 4)

    @torch.no_grad()
    def render(self, rays_o, rays_d, viewdirs, radii):
        from .registry.networks import resample_along_rays, merge_ret
        net = self.net
        n = rays_o.shape[0]
        rays_o, rays_d, viewdirs, radii = (x.contiguous().float() for x in (rays_o, rays_d, viewdirs, radii.reshape(-1)))
        t = torch.linspace(0., 1., self.S + 1, device=rays_o.device)
        z = (self.near * (1. - t) + self.far * t).expand(n, self.S + 1).contiguous()       # GetZvals (create.py:502-531), randomized=False
        data = {'rays_o': rays_o, 'rays_d': rays_d, 'viewdirs': viewdirs, 'radii': radii, 'z_vals': z}
        ret = {}
        for level in range(net.num_levels):
            if level > 0:
                data = resample_along_rays(data, False, net.ray_shape, net.resample_padding)
            data['raw'] = self._mlp(rays_o, rays_d, viewdirs, radii, data['z_vals'])
            data, level_ret = net.render(data, is_test=True)
            ret = level_ret if not ret else merge_ret(ret, level_ret)
        return ret
