"""NerfRender / MipNerfRender / HashNerfRender with the reference's kwargs and (data, ret) protocol
(/root/reference/xrnerf/models/renders/nerf_render.py:10-98, mipnerf_render.py:11-33, hashnerf_render.py:15-177)."""
import torch
from torch import nn

from .. import _C
from .. import raymarch_cuda
from .builder import RENDERS

_ACT = {'relu': 1, 'softplus': 4}


class _CompositeFn(torch.autograd.Function):
    @staticmethod
    def forward(ctx, raw, z_vals, rays_d, mip, white_bkgd, rgb_padding, density_bias, act):
        raw = raw.contiguous().float()
        z_vals, rays_d = z_vals.contiguous().float(), rays_d.contiguous().float()
        n, s = raw.shape[0], raw.shape[1]
        rgb = torch.empty((n, 3), dtype=torch.float32, device=raw.device)
        disp = torch.empty(n, dtype=torch.float32, device=raw.device)
        acc = torch.empty(n, dtype=torch.float32, device=raw.device)
        weights = torch.empty((n, s), dtype=torch.float32, device=raw.device)
        _C.check(_C.lib.xrb_nerf_composite_forward(_C.ptr(raw), _C.ptr(z_vals), _C.ptr(rays_d), n, s, int(mip), int(white_bkgd), float(rgb_padding), float(density_bias), act,
                                                   _C.ptr(rgb), _C.ptr(disp), _C.ptr(acc), _C.ptr(weights), _C.stream()), 'nerf_composite_forward')
        ctx.save_for_backward(raw, z_vals, rays_d)
        ctx.args = (int(mip), int(white_bkgd), float(rgb_padding), float(density_bias), act)
        ctx.mark_non_differentiable(disp, acc, weights)
        return rgb, disp, acc, weights

    @staticmethod
    def backward(ctx, g_rgb, g_disp, g_acc, g_w):
        raw, z_vals, rays_d = ctx.saved_tensors
        n, s = raw.shape[0], raw.shape[1]
        d_raw = torch.empty_like(raw)
        _C.check(_C.lib.xrb_nerf_composite_backward(_C.ptr(raw), _C.ptr(z_vals), _C.ptr(rays_d), _C.ptr(g_rgb.contiguous().float()), n, s, *ctx.args, _C.ptr(d_raw), _C.stream()),
                 'nerf_composite_backward')
        return d_raw, None, None, None, None, None, None, None


class _CompositeGeomFn(torch.autograd.Function):
    """the composite with differentiable depth (sum of w * z, mid-points for Mip-NeRF; not divided by acc) and acc, for depth / opacity losses
    (xrb_nerf_composite_forward_depth, xrb_nerf_composite_backward_geom); rgb and d_raw of an rgb-only loss are bit-identical to _CompositeFn's"""

    @staticmethod
    def forward(ctx, raw, z_vals, rays_d, mip, white_bkgd, rgb_padding, density_bias, act):
        raw = raw.contiguous().float()
        z_vals, rays_d = z_vals.contiguous().float(), rays_d.contiguous().float()
        n, s = raw.shape[0], raw.shape[1]
        rgb = torch.empty((n, 3), dtype=torch.float32, device=raw.device)
        disp, acc, depth = (torch.empty(n, dtype=torch.float32, device=raw.device) for _ in range(3))
        weights = torch.empty((n, s), dtype=torch.float32, device=raw.device)
        _C.check(_C.lib.xrb_nerf_composite_forward_depth(_C.ptr(raw), _C.ptr(z_vals), _C.ptr(rays_d), n, s, int(mip), int(white_bkgd), float(rgb_padding), float(density_bias),
                                                         act, _C.ptr(rgb), _C.ptr(disp), _C.ptr(acc), _C.ptr(weights), _C.ptr(depth), _C.stream()), 'nerf_composite_forward_depth')
        ctx.save_for_backward(raw, z_vals, rays_d)
        ctx.args = (int(mip), int(white_bkgd), float(rgb_padding), float(density_bias), act)
        ctx.mark_non_differentiable(disp, weights)
        return rgb, disp, acc, weights, depth

    @staticmethod
    def backward(ctx, g_rgb, g_disp, g_acc, g_w, g_depth):
        raw, z_vals, rays_d = ctx.saved_tensors
        n, s = raw.shape[0], raw.shape[1]
        d_raw = torch.empty_like(raw)
        _C.check(_C.lib.xrb_nerf_composite_backward_geom(_C.ptr(raw), _C.ptr(z_vals), _C.ptr(rays_d), _C.ptr(g_rgb.contiguous().float()), _C.ptr(g_depth.contiguous().float()),
                                                         _C.ptr(g_acc.contiguous().float()), n, s, *ctx.args, _C.ptr(d_raw), _C.stream()), 'nerf_composite_backward_geom')
        return d_raw, None, None, None, None, None, None, None


@RENDERS.register_module()
class NerfRender(nn.Module):
    mip = False

    def __init__(self, white_bkgd=False, raw_noise_std=0, rgb_padding=0, density_bias=0, density_activation='relu', geometry_grad=False, **kwarg):
        """geometry_grad: ret also holds `depth` [n] (sum of w * z, mid-points for Mip-NeRF; not divided by acc), and `depth` and `acc` are differentiable
        (depth / opacity losses); otherwise acc is not, as in the reference"""
        super().__init__()
        if density_activation not in _ACT:
            raise NotImplementedError(density_activation)
        self.white_bkgd, self.raw_noise_std, self.rgb_padding, self.density_bias = white_bkgd, raw_noise_std, rgb_padding, density_bias
        self.density_activation = density_activation
        self.geometry_grad = bool(geometry_grad)

    def forward(self, data, is_test=False):
        raw, z_vals, rays_d = data['raw'], data['z_vals'], data['rays_d']
        _C.require_cuda(raw, z_vals, rays_d)
        noise_std = 0 if is_test else self.raw_noise_std
        if noise_std > 0.:  # nerf_render.py:68-74 draws on the CPU then moves; all BASELINE configs use 0
            raw = torch.cat([raw[..., :3], raw[..., 3:] + (torch.randn(raw[..., 3:].shape) * noise_std).to(raw.device)], -1)
        args = (raw, z_vals, rays_d, self.mip, self.white_bkgd, self.rgb_padding, self.density_bias, _ACT[self.density_activation])
        if self.geometry_grad:
            rgb, disp, acc, weights, depth = _CompositeGeomFn.apply(*args)
            data['weights'] = weights
            return data, {'rgb': rgb, 'disp': disp, 'acc': acc, 'depth': depth}
        rgb, disp, acc, weights = _CompositeFn.apply(*args)
        data['weights'] = weights
        return data, {'rgb': rgb, 'disp': disp, 'acc': acc}


@RENDERS.register_module()
class MipNerfRender(NerfRender):
    mip = True


class _CalcRgbBp(torch.autograd.Function):
    """hashnerf_render.py:60-146 (_calc_rgb_bp)"""

    @staticmethod
    def forward(ctx, raw, coords, numsteps, numsteps_c, bg, grid_mean, rgb_act, dens_act, aabb_range):
        raw = raw.contiguous()
        rgb = torch.zeros((numsteps.shape[0], 3), dtype=torch.float32, device=raw.device)
        raymarch_cuda.calc_rgb_forward_api(raw, coords, numsteps, numsteps_c, bg, int(rgb_act), int(dens_act), float(aabb_range[0]), float(aabb_range[1]), rgb)
        ctx.save_for_backward(raw, numsteps_c, coords, rgb, grid_mean)
        ctx.extro = (rgb_act, dens_act, aabb_range)
        return rgb

    @staticmethod
    def backward(ctx, grad_rgb):
        raw, numsteps_c, coords, rgb, grid_mean = ctx.saved_tensors
        rgb_act, dens_act, aabb_range = ctx.extro
        d_raw = torch.zeros_like(raw)
        raymarch_cuda.calc_rgb_backward_api(raw, numsteps_c, coords, grad_rgb.contiguous(), rgb, grid_mean, int(rgb_act), int(dens_act), float(aabb_range[0]), float(aabb_range[1]), d_raw)
        return d_raw, None, None, None, None, None, None, None, None


class _CalcRgbGeomFn(torch.autograd.Function):
    """_CalcRgbBp with differentiable alpha = 1 - T and depth = sum of w * t [n,1] (xrb_rm_calc_rgb_forward_geom / xrb_rm_calc_rgb_backward_geom); rgb and
    the colour channels of d_raw are bit-identical to _CalcRgbBp's"""

    @staticmethod
    def forward(ctx, raw, coords, numsteps, numsteps_c, bg, grid_mean, rgb_act, dens_act, aabb_range, rays_o, rays_d):
        raw = raw.contiguous()
        _C.require_cuda(raw, coords, numsteps, numsteps_c, bg, rays_o, rays_d)
        n = numsteps.shape[0]
        rgb = torch.zeros((n, 3), dtype=torch.float32, device=raw.device)
        alpha = torch.zeros((n, 1), dtype=torch.float32, device=raw.device)
        depth = torch.zeros((n, 1), dtype=torch.float32, device=raw.device)
        _C.check(_C.lib.xrb_rm_calc_rgb_forward_geom(_C.ptr(raw), _C.ptr(coords), _C.i32(numsteps), _C.i32(numsteps_c), _C.f32(bg.contiguous()), _C.f32(rays_o), _C.f32(rays_d), n,
                                                     float(aabb_range[0]), float(aabb_range[1]), int(rgb_act), int(dens_act), _C.ptr(rgb), _C.ptr(alpha), _C.ptr(depth),
                                                     _C.stream()), 'calc_rgb_forward_geom')
        ctx.save_for_backward(raw, numsteps_c, coords, rgb, grid_mean, rays_o, rays_d, alpha, depth)
        ctx.extro = (rgb_act, dens_act, aabb_range)
        return rgb, alpha, depth

    @staticmethod
    def backward(ctx, grad_rgb, grad_alpha, grad_depth):
        raw, numsteps_c, coords, rgb, grid_mean, rays_o, rays_d, alpha, depth = ctx.saved_tensors
        rgb_act, dens_act, aabb_range = ctx.extro
        d_raw = torch.zeros_like(raw)
        _C.check(_C.lib.xrb_rm_calc_rgb_backward_geom(_C.ptr(raw), _C.i32(numsteps_c), _C.ptr(coords), _C.f32(grad_rgb.contiguous()), _C.ptr(rgb), _C.f32(grid_mean), _C.ptr(rays_o),
                                                      _C.ptr(rays_d), float(aabb_range[0]), float(aabb_range[1]), _C.ptr(depth), _C.ptr(alpha), _C.f32(grad_depth.contiguous()),
                                                      _C.f32(grad_alpha.contiguous()), numsteps_c.shape[0], int(rgb_act), int(dens_act), _C.ptr(d_raw), _C.stream()),
                 'calc_rgb_backward_geom')
        return d_raw, None, None, None, None, None, None, None, None, None, None


@RENDERS.register_module()
class HashNerfRender(nn.Module):
    def __init__(self, bg_color=None, geometry_grad=False, **kwarg):
        """geometry_grad: the training path also returns differentiable `alpha` and `depth` [n,1] (sum of w * t, not divided by alpha) for depth / opacity
        losses; otherwise it returns rgb only, as in the reference"""
        super().__init__()
        self.bg_color = torch.tensor(bg_color if bg_color is not None else [0, 0, 0]).to(dtype=torch.float32)
        self.geometry_grad = bool(geometry_grad)

    def forward(self, data, sampler, is_test=False):
        raw = data['raw']
        if is_test:
            n = sampler.rays_numsteps.shape[0]
            rgb = torch.zeros((n, 3), dtype=torch.float32, device=raw.device)
            alpha = torch.zeros((n, 1), dtype=torch.float32, device=raw.device)
            raymarch_cuda.calc_rgb_influence_api(raw.contiguous(), sampler.coords, sampler.rays_numsteps, self.bg_color, int(sampler.rgb_activation), int(sampler.density_activation),
                                                 sampler.aabb_range[0], sampler.aabb_range[1], rgb, alpha)
            return data, {'rgb': rgb, 'alpha': alpha}
        if self.geometry_grad:
            rgb, alpha, depth = _CalcRgbGeomFn.apply(raw, sampler.coords, sampler.rays_numsteps, sampler.rays_numsteps_compacted, data['bg_color'].detach(),
                                                     sampler.density_grid_mean, int(sampler.rgb_activation), int(sampler.density_activation), sampler.aabb_range,
                                                     data['rays_o'].contiguous().float(), data['rays_d'].contiguous().float())
            return data, {'rgb': rgb, 'alpha': alpha, 'depth': depth}
        rgb = _CalcRgbBp.apply(raw, sampler.coords, sampler.rays_numsteps, sampler.rays_numsteps_compacted, data['bg_color'].detach(), sampler.density_grid_mean,
                               int(sampler.rgb_activation), int(sampler.density_activation), sampler.aabb_range)
        return data, {'rgb': rgb}
