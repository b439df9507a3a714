"""Fused inference path of the hierarchical NeRF (NerfNetwork.forward with N_importance > 0,
/root/reference/xrnerf/models/networks/nerf.py:39-48 + the val pipeline's GetZvals/GetPts, datasets/pipelines/create.py:486-597) for a set of rays:

  z_vals (given, or linspace) -> [posenc straight into fp16 tile images (wgmma operand layout), positions formed in registers] -> coarse NerfMLP (wgmma) ->
  composite -> sample_pdf (one kernel) -> posenc tiles -> fine NerfMLP (wgmma) -> composite

No [N,S,3] `pts`, no fp32 `embedded`, no per-chunk Python loop: 7 kernel launches per ray batch. Any number of rays is rendered in ray batches of
bounded size (RAY_BATCH_BYTES); every kernel on the path is ray- or row-independent, so a ray's result does not depend on the split.
"""
import torch

from . import _C
from .nerf_mlp import nerf_mlp_forward_tiles

# working-set budget of one ray batch: the encoding image of the level with the most rows, plus every level's raw, weights and z buffers
RAY_BATCH_BYTES = 2 << 30
_ACT = {'relu': 1, 'softplus': 4}


def bytes_per_ray(level_rows, input_ch, normals=False):
    """upper bound of the device bytes one ray of a batch holds at the peak: the fp16 encoding image of the largest level (xrb_nerf_enc_image_bytes per
    row: 256 B for input_ch 63, 384 B for 96) plus, per level of R rows, raw f32[R,4], weights f32[R] and z f32[R+1]. NeRF 64 + 128: 192 * 256 +
    (64 + 192) * 24 + 8 = 55 304 B; Mip-NeRF 2 x 128: 128 * 384 + 2 * 128 * 24 + 8 = 55 304 B. normals=True adds the gradient f32[R,3] of the last
    level's R rows (12 R: 57 608 B for NeRF, 56 840 B for Mip-NeRF)."""
    enc_row = _C.lib.xrb_nerf_enc_image_bytes(128, int(input_ch)) // 128
    return max(level_rows) * enc_row + sum(16 * r + 4 * r + 4 * (r + 1) for r in level_rows) + (12 * level_rows[-1] if normals else 0)


def ray_batch_size(level_rows, input_ch, budget=RAY_BATCH_BYTES, normals=False):
    """rays per batch: the largest multiple of 128 whose bytes_per_ray fit in `budget` (at least 128). At the reference shapes 38 784 rays, a peak of
    2.0 GiB plus the last encoding tile (with normals 37 248 rays for NeRF, 37 760 for Mip-NeRF)."""
    return max(128, budget // bytes_per_ray(level_rows, input_ch, normals) // 128 * 128)


def encode_rays(mlp, rays_o, rays_d, viewdirs, z, radii=None):
    """the fp16 encoding tile image of every sample of the rays, as the renderers form it: xrb_nerf_posenc_tiles_rays on z f32[n,S] (BaseEmbedder) or
    xrb_mip_ipe_tiles_rays on the interval ends z f32[n,S+1] and radii f32[n] (MipNerfEmbedder)"""
    e, mip = mlp.embedder, radii is not None
    n, s = z.shape[0], z.shape[1] - (1 if mip else 0)
    enc = torch.empty(_C.lib.xrb_nerf_enc_image_bytes(n * s, mlp.input_ch), dtype=torch.uint8, device=z.device)
    if mip:
        _C.check(_C.lib.xrb_mip_ipe_tiles_rays(_C.ptr(z), _C.ptr(rays_o), _C.ptr(rays_d), _C.ptr(radii), _C.ptr(viewdirs), n, s, e.min_deg, e.max_deg, e.min_deg_view,
                                               e.max_deg_view, _C.ptr(enc), _C.stream()), 'mip_ipe_tiles_rays')
    else:
        _C.check(_C.lib.xrb_nerf_posenc_tiles_rays(_C.ptr(rays_o), _C.ptr(rays_d), _C.ptr(z), _C.ptr(viewdirs), n, s, e.multires, e.multires_dirs, _C.ptr(enc), _C.stream()),
                 'posenc_tiles_rays')
    return enc


def density_grad_rays(mlp, enc, rays_o, rays_d, z, radii=None, density=None):
    """grad f32[n*S,3] of the raw density at every sample of the rays whose encoding image is enc (xrb_nerf_density_grad_rays, or with radii
    xrb_mip_density_grad_rays); density (f32[n*S] or None) receives the raw density"""
    mip = radii is not None
    n, s = z.shape[0], z.shape[1] - (1 if mip else 0)
    image, bias, gimage = mlp._packed(grad=True)
    grad = torch.empty((n * s, 3), dtype=torch.float32, device=z.device)
    dptr = None if density is None else _C.ptr(density)
    if mip:
        e = mlp.embedder
        _C.check(_C.lib.xrb_mip_density_grad_rays(_C.ptr(image), _C.ptr(gimage), _C.ptr(bias), _C.ptr(enc), _C.ptr(rays_o), _C.ptr(rays_d), _C.ptr(z), _C.ptr(radii), n, s,
                                                  mlp.input_ch, mlp.input_ch_dirs, e.min_deg, e.max_deg, dptr, _C.ptr(grad), _C.stream()), 'mip_density_grad_rays')
    else:
        _C.check(_C.lib.xrb_nerf_density_grad_rays(_C.ptr(image), _C.ptr(gimage), _C.ptr(bias), _C.ptr(enc), _C.ptr(rays_o), _C.ptr(rays_d), _C.ptr(z), n, s,
                                                   mlp.input_ch, mlp.input_ch_dirs, dptr, _C.ptr(grad), _C.stream()), 'nerf_density_grad_rays')
    return grad


def composite_normals(weights, grad, out):
    """out f32[n,3] <- sum_k w_k (-g_k / |g_k|) of each ray (xrb_nerf_composite_normals); weights f32[n,S], grad f32[n*S,3]"""
    n, s = weights.shape
    _C.check(_C.lib.xrb_nerf_composite_normals(_C.ptr(weights), _C.ptr(grad), n, s, _C.ptr(out), _C.stream()), 'nerf_composite_normals')


def _outputs(n, device, depth):
    out = {'rgb': torch.empty((n, 3), dtype=torch.float32, device=device), 'disp': torch.empty(n, dtype=torch.float32, device=device),
           'acc': torch.empty(n, dtype=torch.float32, device=device)}
    if depth:
        out['depth'] = torch.empty((n, 1), dtype=torch.float32, device=device)
    return out


def _composite(render, raw, z, rays_d, out, lo):
    """NerfRender / MipNerfRender forward with is_test (no raw noise) of one batch of rays, written into rows lo.. of the level's outputs; returns the
    batch's weights. With out['depth'] the kernel is xrb_nerf_composite_forward_depth, whose other outputs are bit-identical."""
    n, s = raw.shape[0], raw.shape[1]
    hi = lo + n
    weights = torch.empty((n, s), dtype=torch.float32, device=raw.device)
    args = (_C.ptr(raw), _C.ptr(z), _C.ptr(rays_d), n, s, int(render.mip), int(render.white_bkgd), float(render.rgb_padding), float(render.density_bias),
            _ACT[render.density_activation], _C.ptr(out['rgb'][lo:hi]), _C.ptr(out['disp'][lo:hi]), _C.ptr(out['acc'][lo:hi]), _C.ptr(weights))
    if 'depth' in out:
        _C.check(_C.lib.xrb_nerf_composite_forward_depth(*args, _C.ptr(out['depth'][lo:hi]), _C.stream()), 'nerf_composite_forward_depth')
    else:
        _C.check(_C.lib.xrb_nerf_composite_forward(*args, _C.stream()), 'nerf_composite_forward')
    return weights


def _merge_levels(levels):
    from .registry.networks import merge_ret
    ret = levels[0]
    for level in levels[1:]:
        ret = merge_ret(ret, level)
    return ret


def _z_rows(z_vals, n, width, near, far, device):
    """the coarse z values: z_vals checked to be [n, width], or the linspace near..far (GetZvals, create.py:502-531, lindisp=False) as one row"""
    if z_vals is None:
        t = torch.linspace(0., 1., width, device=device)
        return None, (near * (1. - t) + far * t)[None]
    if tuple(z_vals.shape) != (n, width):
        raise ValueError(f'z_vals: expected shape {(n, width)}, got {tuple(z_vals.shape)}')
    return z_vals.contiguous().float(), None


class NerfRenderer:
    def __init__(self, network, near=2.0, far=6.0, n_samples=64, ray_batch=None):
        """network: registry NerfNetwork (mlp, mlp_fine, render); BaseEmbedder encodings. near / far / n_samples make the coarse z values when render()
        is given none. ray_batch: rays per batch, None = ray_batch_size(), which keeps a batch's working set under RAY_BATCH_BYTES."""
        self.net, self.near, self.far, self.S, self.ray_batch = network, near, far, n_samples, ray_batch
        e = network.mlp.embedder
        self.multires, self.multires_dirs = e.multires, e.multires_dirs

    def _mlp(self, mlp, rays_o, rays_d, viewdirs, z):
        """the level's raw [n,S,4] and its encoding image"""
        n, s = z.shape
        enc = encode_rays(mlp, rays_o, rays_d, viewdirs, z)
        image, bias = mlp._packed()
        return nerf_mlp_forward_tiles(image, bias, enc, n * s, mlp.input_ch, mlp.input_ch_dirs).view(n, s, 4), enc

    @torch.no_grad()
    def render(self, rays_o, rays_d, viewdirs, z_vals=None, depth=False, normals=False):
        """rays_o, rays_d, viewdirs f32[n,3]; z_vals f32[n,S] the coarse z values (the val pipeline's GetZvals), None = linspace(near, far, n_samples).
        Returns NerfNetwork.forward(is_test=True)'s keys: rgb [n,3], disp [n], acc [n], and with N_importance > 0 the coarse level's as coarse_*;
        depth=True adds depth [n,1] (and coarse_depth) = sum of w * z, not divided by acc. normals=True adds normal [n,3] of the last level
        (include/xrnerf_b200.h "NeRF / Mip-NeRF normal maps"): the density gradient kernel on that level's encoding image, then the normal composite on
        its weights; every other output is unchanged.
        Peak device memory beyond the inputs and outputs: ray_batch * bytes_per_ray (about 2.0 GiB at the reference shapes) plus one 128-row
        encoding tile."""
        from .registry.networks import sample_pdf
        net = self.net
        n, dev = rays_o.shape[0], rays_o.device
        rays_o, rays_d, viewdirs = (x.contiguous().float() for x in (rays_o, rays_d, viewdirs))   # the kernels read dense [n,3] rows
        s = self.S if z_vals is None else z_vals.shape[-1]
        z_all, z_lin = _z_rows(z_vals, n, s, self.near, self.far, dev)
        n_imp = getattr(net, 'N_importance', 0)
        level_rows = [s] + ([s + n_imp] if n_imp > 0 else [])
        batch = self.ray_batch or ray_batch_size(level_rows, net.mlp.input_ch, normals=normals)
        levels = [_outputs(n, dev, depth) for _ in level_rows]
        normal = torch.empty((n, 3), dtype=torch.float32, device=dev) if normals else None
        for lo in range(0, n, batch):
            hi = min(n, lo + batch)
            o, d, vd = rays_o[lo:hi], rays_d[lo:hi], viewdirs[lo:hi]
            z = z_all[lo:hi] if z_all is not None else z_lin.expand(hi - lo, s).contiguous()
            mlp = net.mlp
            raw, enc = self._mlp(mlp, o, d, vd, z)
            weights = _composite(net.render, raw, z, d, levels[0], lo)
            if n_imp > 0:
                data = sample_pdf({'rays_o': o, 'rays_d': d, 'z_vals': z, 'weights': weights, 'pts': None}, n_imp, False, True)
                z, mlp = data['z_vals'], net.mlp_fine
                raw = enc = None                    # the coarse level's buffers are free before the fine level's are allocated
                raw, enc = self._mlp(mlp, o, d, vd, z)
                weights = _composite(net.render, raw, z, d, levels[1], lo)
            if normals:
                composite_normals(weights, density_grad_rays(mlp, enc, o, d, z), normal[lo:hi])
            raw = enc = None
        ret = _merge_levels(levels)
        if normals:
            ret['normal'] = normal
        return ret


class MipNerfRenderer:
    """Fused inference path of MipNerfNetwork.forward(is_test=True) (/root/reference/xrnerf/models/networks/mipnerf.py:25-43): per level
    [cast_rays + IPE straight into fp16 tile images (wgmma operand layout)] -> the SAME NerfMLP (wgmma) -> MipNerfRender composite, with resample_along_rays
    (one kernel) between the levels: 3 launches per level + 1 per ray batch, no [N,S,3] means/covs, no fp32 `embedded` [N*S,123]. Ray batches as NerfRenderer's."""

    def __init__(self, network, near=2.0, far=6.0, n_samples=128, ray_batch=None):
        self.net, self.near, self.far, self.S, self.ray_batch = network, near, far, n_samples, ray_batch
        e = network.mlp.embedder
        self.degs = (e.min_deg, e.max_deg, e.min_deg_view, e.max_deg_view)

    def _mlp(self, rays_o, rays_d, viewdirs, radii, z):
        """the level's raw [n,S,4] and its encoding image"""
        mlp = self.net.mlp
        n, s = z.shape[0], z.shape[1] - 1
        enc = encode_rays(mlp, rays_o, rays_d, viewdirs, z, radii)
        image, bias = mlp._packed()
        return nerf_mlp_forward_tiles(image, bias, enc, n * s, mlp.input_ch, mlp.input_ch_dirs).view(n, s, 4), enc

    @torch.no_grad()
    def render(self, rays_o, rays_d, viewdirs, radii, z_vals=None, depth=False, normals=False):
        """rays_o, rays_d, viewdirs f32[n,3], radii f32[n] or [n,1]; z_vals f32[n,S+1] the first level's interval ends (GetZvals), None =
        linspace(near, far, n_samples + 1). Returns MipNerfNetwork.forward(is_test=True)'s keys (rgb, disp, acc; earlier levels as coarse_*);
        depth=True adds depth [n,1] per level = sum of w * (z_k + z_{k+1}) / 2, not divided by acc. normals=True adds normal [n,3] of the last
        level, as NerfRenderer.render's. Peak device memory beyond the inputs and outputs as NerfRenderer.render's."""
        from .registry.networks import resample_along_rays
        net = self.net
        n, dev = rays_o.shape[0], rays_o.device
        rays_o, rays_d, viewdirs, radii = (x.contiguous().float() for x in (rays_o, rays_d, viewdirs, radii.reshape(-1)))
        s = self.S if z_vals is None else z_vals.shape[-1] - 1
        z_all, z_lin = _z_rows(z_vals, n, s + 1, self.near, self.far, dev)          # randomized=False
        level_rows = [s] * net.num_levels
        batch = self.ray_batch or ray_batch_size(level_rows, net.mlp.input_ch, normals=normals)
        levels = [_outputs(n, dev, depth) for _ in level_rows]
        normal = torch.empty((n, 3), dtype=torch.float32, device=dev) if normals else None
        for lo in range(0, n, batch):
            hi = min(n, lo + batch)
            data = {'rays_o': rays_o[lo:hi], 'rays_d': rays_d[lo:hi], 'viewdirs': viewdirs[lo:hi], 'radii': radii[lo:hi],
                    'z_vals': z_all[lo:hi] if z_all is not None else z_lin.expand(hi - lo, s + 1).contiguous()}
            for level, out in enumerate(levels):
                if level > 0:
                    data = resample_along_rays(data, False, net.ray_shape, net.resample_padding)
                raw = enc = None                    # the last level's buffers are free before this level's are allocated
                raw, enc = self._mlp(data['rays_o'], data['rays_d'], data['viewdirs'], data['radii'], data['z_vals'])
                data['weights'] = _composite(net.render, raw, data['z_vals'], data['rays_d'], out, lo)
            if normals:
                grad = density_grad_rays(net.mlp, enc, data['rays_o'], data['rays_d'], data['z_vals'], data['radii'])
                composite_normals(data['weights'], grad, normal[lo:hi])
            raw = enc = grad = None
        ret = _merge_levels(levels)
        if normals:
            ret['normal'] = normal
        return ret
