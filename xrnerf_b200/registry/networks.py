"""NerfNetwork / MipNerfNetwork / HashNerfNetwork: the control flow of the reference's networks
(/root/reference/xrnerf/models/networks/nerf.py:15-180, mipnerf.py:14-74, hashnerf.py:16-52) over this package's kernels.
The mmcv-runner-facing API is kept: train_step(data, optimizer) -> {loss, log_vars, num_samples}, val_step, batchify_forward,
set_val_pipeline. Dataset/runner/hook plumbing is out of scope (SURVEY §2 rows 1-4)."""
import torch
from torch import nn

from .. import _C
from . import builder
from .builder import NETWORKS

# ---- networks/utils: metrics.py:3-16, batching.py, transforms.py (merge_ret / recover_shape)
img2mse = lambda x, y: torch.mean((x - y) ** 2)
mse2psnr = lambda x: -10. * torch.log(x) / torch.log(torch.tensor([10.], device=x.device))


def HuberLoss(x, y, delta=0.1, reduction='sum'):
    rel = (x - y).abs()
    loss = torch.where(rel > delta, rel - 0.5 * delta, 0.5 / delta * rel * rel)
    return loss.mean() if reduction == 'mean' else loss.sum()


def unfold_batching(x):
    """networks/utils/batching.py:5-12: (bs, N_per_sampler, ...) -> (bs * N_per_sampler, ...); 1-D tensors and non-tensors pass through."""
    if torch.is_tensor(x) and x.dim() > 1:
        return x.reshape((-1,) + tuple(x.shape[2:]))     # == torch.cat([x[b] for b in range(bs)], 0)
    return x


def merge_ret(ret, fine_ret):
    out = {'coarse_' + k: v for k, v in ret.items()}
    out.update(fine_ret)
    return out


class _GeomLossFn(torch.autograd.Function):
    """w_d * sum |D - D*| / c_d + w_a * sum (A - A*)^2 / c_a over the rays each term keeps (xrb_geom_loss_grad: depth only where D* is finite and > 0;
    with numsteps, only the rays the compaction kept whole), c = 1 (mean=False) or the number of rays kept"""

    @staticmethod
    def forward(ctx, depth, alpha, target_depth, target_alpha, numsteps, numsteps_c, wd, wa, mean):
        ref = depth if depth is not None else alpha
        n = ref.numel()
        vec = lambda t: None if t is None else t.detach().reshape(-1).contiguous().float()   # noqa: E731
        loss = torch.zeros(1, dtype=torch.float32, device=ref.device)
        gd = torch.zeros(n, dtype=torch.float32, device=ref.device) if depth is not None else None
        ga = torch.zeros(n, dtype=torch.float32, device=ref.device) if alpha is not None else None
        ts = [vec(t) for t in (depth, alpha, target_depth, target_alpha)]
        _C.require_cuda(*ts)
        _C.check(_C.lib.xrb_geom_loss_grad(*[_C.ptr(t) for t in ts], _C.ptr(numsteps), _C.ptr(numsteps_c), n, float(wd), float(wa), int(mean), _C.ptr(gd), _C.ptr(ga),
                                           _C.ptr(loss), _C.stream()), 'geom_loss_grad')
        ctx.save_for_backward(gd, ga)
        ctx.shapes = (None if depth is None else depth.shape, None if alpha is None else alpha.shape)
        return loss[0]

    @staticmethod
    def backward(ctx, g):
        gd, ga = ctx.saved_tensors
        sd, sa = ctx.shapes
        return (None if gd is None else (g * gd).reshape(sd), None if ga is None else (g * ga).reshape(sa), None, None, None, None, None, None, None)


def geom_loss(ret, data, depth_weight, opacity_weight, prefix='', numsteps=None, mean=True, alpha_key='acc', target_alpha_key='target_alpha'):
    """(depth term, opacity term) of one level (ret keys prefix + 'depth' / prefix + alpha_key), each None when its weight is 0 or its target is absent"""
    ns, nsc = numsteps if numsteps is not None else (None, None)
    out = []
    for w, key, tkey in ((depth_weight, 'depth', 'target_depth'), (opacity_weight, alpha_key, target_alpha_key)):
        if w > 0 and tkey in data:
            d, a = (ret[prefix + key], None) if key == 'depth' else (None, ret[prefix + key])
            out.append(_GeomLossFn.apply(d, a, data[tkey] if key == 'depth' else None, data[tkey] if key != 'depth' else None, ns, nsc,
                                         w if key == 'depth' else 0.0, w if key != 'depth' else 0.0, mean))
        else:
            out.append(None)
    return out


def recover_shape(x, src_shape):
    return x.reshape([int(v) for v in src_shape[:2]] + [-1])


def sample_pdf(data, N_samples, is_perturb=False, is_test=False):
    """hierarchical_sample.py:6-53 as one kernel (inverse CDF + merge sort + pts)."""
    z, w, o, d = (data[k].contiguous().float() for k in ('z_vals', 'weights', 'rays_o', 'rays_d'))
    _C.require_cuda(z, w, o, d)
    n, s = z.shape
    det = is_test or not is_perturb
    u = None if det else torch.rand((n, N_samples), device=z.device)
    z_out = torch.empty((n, s + N_samples), dtype=torch.float32, device=z.device)
    want_pts = not ('pts' in data and data['pts'] is None)   # the fused renderer forms positions inside the encoding kernel and asks for no pts
    pts = torch.empty((n, s + N_samples, 3), dtype=torch.float32, device=z.device) if want_pts else None
    _C.check(_C.lib.xrb_nerf_sample_pdf(_C.ptr(z), _C.ptr(w.detach()), _C.ptr(o), _C.ptr(d), _C.ptr(u), n, s, N_samples, _C.ptr(z_out), _C.ptr(pts), _C.stream()), 'sample_pdf')
    data['pts'], data['z_vals'] = pts, z_out
    return data


def resample_along_rays(data, randomized, ray_shape, resample_padding, rand=None):
    """mip.py:146-176 as one kernel (blur + piecewise-constant inverse CDF). `rand`: the [n, S+1] uniforms the reference draws with torch.rand when
    `randomized` (mip.py:31-33); default: drawn on the device."""
    if ray_shape != 'cone':
        raise NotImplementedError('ray_shape cone (the reference configs)')
    z, w = data['z_vals'].contiguous().float(), data['weights'].detach().contiguous().float()
    n, s1 = z.shape
    u = None
    if randomized:
        sdt = 1.0 / s1
        r = torch.rand((n, s1), device=z.device) if rand is None else rand.to(z.device).float()
        u = torch.arange(s1, device=z.device) * sdt + r * (sdt - torch.finfo(torch.float32).eps)
        u = torch.minimum(u, torch.tensor(1. - torch.finfo(torch.float32).eps, device=z.device)).contiguous()
    z_new = torch.empty_like(z)
    _C.check(_C.lib.xrb_mip_resample(_C.ptr(z), _C.ptr(w), _C.ptr(u), n, s1 - 1, float(resample_padding), _C.ptr(z_new), _C.stream()), 'mip_resample')
    data['z_vals'] = z_new
    return data


@NETWORKS.register_module()
class NerfNetwork(nn.Module):
    render_normals = False   # True: the fused test path also returns per-pixel normal maps of the last level (batchify_forward)

    def __init__(self, cfg, mlp=None, mlp_fine=None, render=None):
        super().__init__()
        self.phase = cfg.get('phase', 'train')
        # depth / opacity supervision (opt-in): weights of L1 depth and squared opacity terms added to the colour loss when a batch holds the targets
        self.depth_loss_weight, self.opacity_loss_weight = float(cfg.get('depth_loss_weight', 0.0)), float(cfg.get('opacity_loss_weight', 0.0))
        for k in ('chunk', 'bs_data', 'is_perturb', 'N_importance'):
            if k in cfg:
                setattr(self, k, cfg[k])
        if mlp is not None:
            self.mlp = builder.build_mlp(mlp)
        if mlp_fine is not None:
            self.mlp_fine = builder.build_mlp(mlp_fine)
        if render is not None:
            self.render = builder.build_render(render)
        self.val_pipeline = None

    def forward(self, data, is_test=False):
        data, ret = self.render(self.mlp(data), is_test)
        if self.N_importance > 0:
            data = sample_pdf(data, self.N_importance, self.is_perturb, is_test)
            _, fine_ret = self.render(self.mlp_fine(data), is_test)
            ret = merge_ret(ret, fine_ret)
        return ret

    def batchify_forward(self, data, is_test=False):
        """Inference over a whole ray set. With is_test, `fused_inference` (default True), rays on CUDA and the fused NerfMLP shape (NerfMLP._fused_ok),
        the rays go through the fused renderer (xrnerf_b200.nerf.NerfRenderer; MipNerfRenderer for Mip-NeRF) in ray batches of bounded size, on the
        pipeline's data['z_vals'] (the reference Blender configs' linspace(2, 6) when absent) and, for Mip-NeRF, data['radii']. That path also returns
        each ray's `depth` [n,1] (sum of w * z, not divided by acc; `coarse_depth` for the coarse level); `fused_ray_batch` sets its rays per batch
        (None: xrnerf_b200.nerf.ray_batch_size). Training, `fused_inference = False` and other shapes run the reference's chunk loop over forward()
        (nerf.py:50-69), which returns the reference's keys only."""
        if is_test and getattr(self, 'fused_inference', True) and self._fused_ok(data['rays_o']):
            return self._fused_forward(data)
        if is_test and self.render_normals:
            raise NotImplementedError('render_normals: normal maps come from the fused NeRF / Mip-NeRF renderer (CUDA rays, the fused NerfMLP shape); '
                                      'set fused_inference = True')
        return self._chunked_forward(data, is_test)

    def _fused_mlps(self):
        return [self.mlp] + ([self.mlp_fine] if getattr(self, 'N_importance', 0) > 0 else [])

    def _fused_ok(self, x):
        """the fused renderer serves this network: CUDA rays, NerfMLPs of the fused shape with the encoding the renderer forms (BaseEmbedder (63, 27) for
        NeRF, MipNerfEmbedder (96, 27) for Mip-NeRF), and the matching composite"""
        mip, mlps = isinstance(self, MipNerfNetwork), self._fused_mlps()
        return (x.is_cuda and bool(mlps) and getattr(self.render, 'mip', None) == mip
                and all(hasattr(m, '_fused_ok') and m._fused_ok(x) and m._is_mip() == mip for m in mlps))

    def _fused_forward(self, data):
        from ..nerf import NerfRenderer
        r = NerfRenderer(self, ray_batch=getattr(self, 'fused_ray_batch', None))
        return r.render(data['rays_o'], data['rays_d'], data['viewdirs'], z_vals=data.get('z_vals'), depth=True, normals=self.render_normals)

    def _chunked_forward(self, data, is_test):
        N = data[self.bs_data].shape[0]
        all_ret = {}
        for i in range(0, N, self.chunk):
            chunk = {k: (v[i:i + self.chunk] if torch.is_tensor(v) and v.dim() > 0 and v.shape[0] == N else v) for k, v in data.items()}
            ret = self.forward(chunk, is_test)
            for k, v in ret.items():
                all_ret.setdefault(k, []).append(v)
        return {k: torch.cat(v, 0) for k, v in all_ret.items()}

    def _geometry_wanted(self, data, alpha_key='target_alpha'):
        return (self.depth_loss_weight > 0 and 'target_depth' in data) or (self.opacity_loss_weight > 0 and alpha_key in data)

    def _forward_geometry(self, data, geometry):
        """forward() with the render's geometry_grad flag set for this call when the depth / opacity terms are wanted"""
        if not geometry:
            return self.forward(data, is_test=False)
        flag = self.render.geometry_grad
        self.render.geometry_grad = True
        try:
            return self.forward(data, is_test=False)
        finally:
            self.render.geometry_grad = flag

    def _add_geometry(self, loss, log, ret, data, levels, **kw):
        """adds the depth / opacity terms of every (prefix, multiplier) level to the loss; log_vars gain loss_depth / loss_opacity"""
        per_level = [(m, geom_loss(ret, data, self.depth_loss_weight, self.opacity_loss_weight, prefix=p, **kw)) for p, m in levels]
        for i, name in enumerate(('loss_depth', 'loss_opacity')):
            terms = [t[i] if m == 1.0 else m * t[i] for m, t in per_level if t[i] is not None]
            if terms:
                term = sum(terms[1:], terms[0])
                loss = loss + term
                log[name] = term.item()
        return loss

    def train_step(self, data, optimizer, **kwargs):
        data = {k: unfold_batching(v) for k, v in data.items()}
        geometry = self._geometry_wanted(data)
        ret = self._forward_geometry(data, geometry)
        img_loss = img2mse(ret['rgb'], data['target_s'])
        psnr = mse2psnr(img_loss)
        loss = img_loss
        if 'coarse_rgb' in ret:
            loss = loss + img2mse(ret['coarse_rgb'], data['target_s'])
        log = {}
        if geometry:   # both levels, as the colour loss
            loss = self._add_geometry(loss, log, ret, data, [('', 1.0)] + ([('coarse_', 1.0)] if 'coarse_rgb' in ret else []))
        return {'loss': loss, 'log_vars': {'loss': loss.item(), 'psnr': psnr.item(), **log}, 'num_samples': ret['rgb'].shape[0]}

    def _mark_dirty(self):
        for m in (getattr(self, 'mlp', None), getattr(self, 'mlp_fine', None)):
            if m is not None and hasattr(m, 'mark_dirty'):
                m.mark_dirty()                      # weights may have been swapped through `.data` (EMAHook) since the last pack

    def val_step(self, data, optimizer=None, **kwargs):
        """nerf.py:94-142: phase 'test' dispatches to test_step. Otherwise renders data['poses'] and, when given, data['spiral_poses'] through the
        installed val pipeline (rank 0 only in the reference; here every rank renders what it is given). Returns the reference's keys as device tensors:
        rgbs [H,W,3] and disps [H,W,1] per pose, gt_imgs (data['images'] per pose, when given), spiral_rgbs / spiral_disps, elapsed_time per pose in
        seconds (pipeline + render, CUDA events); plus psnr per pose, taken on the device against images[..., :3]. With `render_normals` also normals
        and spiral_normals: one [H,W,3] normal map per pose (batchify_forward's `normal`)."""
        if self.phase == 'test':
            return self.test_step(data, **kwargs)
        self._mark_dirty()
        data = {k: unfold_batching(v) for k, v in data.items()}
        poses, images, spiral = data['poses'], data.get('images'), data.get('spiral_poses')
        rgbs, disps, gt_imgs, psnrs, elapsed, spiral_rgbs, spiral_disps, normals, spiral_normals = [], [], [], [], [], [], [], [], []
        with torch.no_grad():
            for i in range(poses.shape[0]):
                t0, t1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                t0.record()
                d = self.val_pipeline({'pose': poses[i], 'idx': i})
                ret = self.batchify_forward(d, is_test=True)
                rgb = recover_shape(ret['rgb'], d['src_shape'])
                t1.record()
                rgbs.append(rgb); disps.append(recover_shape(ret['disp'], d['src_shape'])); elapsed.append((t0, t1))
                if 'normal' in ret:
                    normals.append(recover_shape(ret['normal'], d['src_shape']))
                if images is not None:
                    gt = images[i].to(rgb.device)
                    gt_imgs.append(gt)
                    psnrs.append(mse2psnr(img2mse(rgb, gt[..., :3])))
            for i in range(0 if spiral is None else spiral.shape[0]):
                d = self.val_pipeline({'pose': spiral[i], 'idx': i})
                ret = self.batchify_forward(d, is_test=True)
                spiral_rgbs.append(recover_shape(ret['rgb'], d['src_shape'])); spiral_disps.append(recover_shape(ret['disp'], d['src_shape']))
                if 'normal' in ret:
                    spiral_normals.append(recover_shape(ret['normal'], d['src_shape']))
        torch.cuda.synchronize()
        out = {'rgbs': rgbs, 'disps': disps, 'gt_imgs': gt_imgs, 'spiral_rgbs': spiral_rgbs, 'spiral_disps': spiral_disps,
               'elapsed_time': [a.elapsed_time(b) * 1e-3 for a, b in elapsed], 'psnr': [float(p.item()) for p in psnrs]}
        if self.render_normals:
            out['normals'], out['spiral_normals'] = normals, spiral_normals
        return out

    def test_step(self, data, **kwargs):
        """nerf.py:144-169: one test pose (data['pose'], data['image'], data['idx']) through the installed val pipeline -> rgb [H,W,3], disp [H,W,1],
        gt_img (data['image'] on the render's device) and idx (an int); with `render_normals` also normal [H,W,3]."""
        self._mark_dirty()
        data = {k: unfold_batching(v) for k, v in data.items()}
        idx = data['idx']
        idx = int(idx.item()) if torch.is_tensor(idx) else int(idx)
        with torch.no_grad():
            d = self.val_pipeline({'pose': data['pose'], 'idx': idx})
            ret = self.batchify_forward(d, is_test=True)
        rgb = recover_shape(ret['rgb'], d['src_shape'])
        out = {'rgb': rgb, 'disp': recover_shape(ret['disp'], d['src_shape']), 'gt_img': data['image'].to(rgb.device), 'idx': idx}
        if 'normal' in ret:
            out['normal'] = recover_shape(ret['normal'], d['src_shape'])
        return out

    def set_val_pipeline(self, func):
        self.val_pipeline = func

    def _mesh_mlp(self):
        """the network whose output the renderer returns"""
        return self.mlp_fine if self.N_importance > 0 else self.mlp

    def extract_mesh(self, resolution=256, threshold=50.0, box=((-1.5, -1.5, -1.5), (1.5, 1.5, 1.5))):
        """Triangle mesh of the density level set sigma = threshold -> (verts f32[V,3], faces i32[F,3]) CUDA tensors, in the world frame of the rays,
        triangles wound counter-clockwise seen from outside. The raw alpha of mlp_fine (mlp when N_importance == 0) is sampled on a resolution^3 lattice
        spanning `box` (NerfMLP.density_lattice) and meshed by xrnerf_b200.mesh.marching_cubes.

        threshold is a density sigma = act(raw + density_bias) with the renderer's activation (relu or softplus), mapped to raw alpha by
        mesh.raw_density_threshold (ValueError outside the activation's range). The default of 50 has not been checked here on a trained scene.
        The default box is the cube the Instant-NGP path's unit cube covers (synth.poses_nerf2ngp: scale 0.33, offset 0.5), so meshes of one scene
        from both networks cover the same region."""
        return self._lattice_mesh(resolution, threshold, box)

    def _lattice_mesh(self, resolution, threshold, box, sigma=None):
        """sigma: the Mip-NeRF point query's footprint (None for NeRF)"""
        from ..mesh import marching_cubes, raw_density_threshold
        r = self.render
        raw = raw_density_threshold(threshold, r.density_activation, r.density_bias)
        mlp = self._mesh_mlp()
        mlp.mark_dirty()                       # weights may have been swapped through `.data` (EMAHook) since the last pack
        with torch.no_grad():
            vol = mlp.density_lattice((resolution,) * 3, box, sigma)
            return marching_cubes(vol, raw, box)

    def extract_colored_mesh(self, resolution=256, threshold=50.0, box=((-1.5, -1.5, -1.5), (1.5, 1.5, 1.5))):
        """extract_mesh with a unit normal and a colour per vertex -> (verts f32[V,3], faces i32[F,3], normals f32[V,3], colors f32[V,3]) CUDA tensors;
        verts and faces are bit-identical to extract_mesh(resolution, threshold, box).

        normal = -g / |g| (0 where g = 0), with g the gradient of the raw alpha at the vertex (NerfMLP.density_grad). Inside is "sigma > threshold", so the
        normal points outward. The gradient comes from the training kernels' forward, the lattice from the inference kernel: the two densities agree to
        the fp16 tolerance, not bit for bit.
        color = NerfRender's rgb activation sigmoid(raw[:3]) (1 + 2 rgb_padding) - rgb_padding of the inference kernel at the vertex, with view
        direction -normal: the surface seen from outside."""
        return self._colored_lattice_mesh(resolution, threshold, box)

    def _colored_lattice_mesh(self, resolution, threshold, box, sigma=None):
        from ..mesh import outward_normals
        verts, faces = self._lattice_mesh(resolution, threshold, box, sigma)
        mlp = self._mesh_mlp()
        with torch.no_grad():
            normals = outward_normals(mlp.density_grad(verts, sigma)[1])
            colors = nerf_vertex_colors(mlp, verts, -normals, self.render.rgb_padding, sigma)
            return verts, faces, normals, colors


def nerf_vertex_colors(mlp, pts, dirs, rgb_padding, sigma=None):
    """NerfRender's rgb activation of the fused inference NerfMLP at pts f32[n,3] seen along dirs f32[n,3] (one encoding row per point,
    nerf_mlp.encode_points: BaseEmbedder, or with a MipNerfEmbedder the point query at footprint sigma)"""
    from ..nerf_mlp import encode_points, nerf_mlp_forward_tiles
    n = int(pts.shape[0])
    image, bias = mlp._packed()
    enc = torch.empty(_C.lib.xrb_nerf_enc_image_bytes(n, mlp.input_ch), dtype=torch.uint8, device=pts.device)
    encode_points(mlp, sigma, pts.contiguous().float(), dirs.contiguous().float(), 1, enc)
    raw = nerf_mlp_forward_tiles(image, bias, enc, n, mlp.input_ch, mlp.input_ch_dirs)
    return torch.sigmoid(raw[:, :3]) * (1 + 2 * rgb_padding) - rgb_padding


@NETWORKS.register_module()
class MipNerfNetwork(NerfNetwork):
    def __init__(self, cfg, mlp=None, render=None):
        super().__init__(cfg, mlp=mlp, render=render)
        self.num_levels, self.resample_padding, self.ray_shape = cfg.num_levels if hasattr(cfg, 'num_levels') else cfg['num_levels'], cfg['resample_padding'], cfg['ray_shape']
        self.use_multiscale, self.coarse_loss_mult = cfg['use_multiscale'], cfg['coarse_loss_mult']

    _NO_FOOTPRINT = "MipNerfNetwork: the field is defined on conical frusta, and a point query needs a chosen footprint: pass footprint=sigma or 'cell'"

    def _mesh_mlp(self):
        """one MLP serves every level"""
        return self.mlp

    def extract_mesh(self, resolution=256, threshold=50.0, box=((-1.5, -1.5, -1.5), (1.5, 1.5, 1.5)), footprint=None):
        """Triangle mesh of the density level set sigma_density = threshold of the point query at `footprint` -> (verts f32[V,3], faces i32[F,3]) CUDA
        tensors, in the world frame of the rays, triangles wound counter-clockwise seen from outside: NerfMLP.density_lattice (xrb_mip_density_lattice)
        on a resolution^3 lattice spanning `box`, meshed by xrnerf_b200.mesh.marching_cubes.

        Mip-NeRF's field is defined on conical frusta, so a point query needs a footprint: the isotropic Gaussian of standard deviation sigma around the
        point, encoded by the IPE (include/xrnerf_b200.h). footprint = sigma >= 0 in the rays' world frame, or 'cell': sigma = h / sqrt(12) for the
        lattice spacing h = max over axes (hi - lo) / (resolution - 1), the standard deviation of a uniform distribution over one cell, so the mesh sees
        the field filtered at its own spacing. footprint=None raises NotImplementedError; a negative or non-finite sigma or an unknown string raises
        ValueError. Neither the 'cell' default nor the threshold of 50 has been checked here on a trained scene.

        threshold is a density act(raw + density_bias) with the renderer's activation (the reference config: softplus, density_bias = -1), mapped to raw
        alpha by mesh.raw_density_threshold (ValueError outside the activation's range)."""
        if footprint is None:
            raise NotImplementedError(self._NO_FOOTPRINT)
        from ..mesh import footprint_sigma
        return self._lattice_mesh(resolution, threshold, box, footprint_sigma(footprint, (resolution,) * 3, box))

    def extract_colored_mesh(self, resolution=256, threshold=50.0, box=((-1.5, -1.5, -1.5), (1.5, 1.5, 1.5)), footprint=None):
        """extract_mesh with a unit normal and a colour per vertex -> (verts, faces, normals, colors) CUDA tensors; verts and faces are bit-identical to
        extract_mesh(resolution, threshold, box, footprint). One sigma serves the lattice, the gradient and the colours.

        normal = -g / |g| (0 where g = 0), g the gradient of the point query's raw alpha at the vertex (NerfMLP.density_grad at the same sigma); it
        points outward. color = the renderer's sigmoid(raw[:3]) (1 + 2 rgb_padding) - rgb_padding of the inference kernel on the point query at the
        vertex, with view direction -normal."""
        if footprint is None:
            raise NotImplementedError(self._NO_FOOTPRINT)
        from ..mesh import footprint_sigma
        return self._colored_lattice_mesh(resolution, threshold, box, footprint_sigma(footprint, (resolution,) * 3, box))

    def _fused_mlps(self):
        return [self.mlp] if self.ray_shape == 'cone' else []      # resample_along_rays implements the cone

    def _fused_forward(self, data):
        from ..nerf import MipNerfRenderer
        r = MipNerfRenderer(self, ray_batch=getattr(self, 'fused_ray_batch', None))
        return r.render(data['rays_o'], data['rays_d'], data['viewdirs'], data['radii'], z_vals=data.get('z_vals'), depth=True, normals=self.render_normals)

    def val_step(self, data, optimizer=None, **kwargs):
        """mipnerf.py:76-98: without use_multiscale NerfNetwork.val_step. With it, one pixel-shaped view through evaluate_once: phase 'test' returns
        rgb [H,W,3], gt_img, disp [H,W,1] and idx; validation returns rgbs, gt_imgs and disps as one-element lists. Device tensors throughout."""
        if not self.use_multiscale:
            return super().val_step(data, optimizer, **kwargs)
        rgb, image, disp, idx, *normal = self.evaluate_once(data, **kwargs)
        if self.phase == 'test':
            return dict({'rgb': rgb, 'gt_img': image, 'disp': disp, 'idx': idx}, **({'normal': normal[0]} if normal else {}))
        return dict({'rgbs': [rgb], 'gt_imgs': [image], 'disps': [disp]}, **({'normals': normal} if normal else {}))

    def evaluate_once(self, data, **kwargs):
        """mipnerf.py:100-117: data holds one view's per-pixel rays [1,H,W,...] (rays_o, rays_d, viewdirs, radii, z_vals, ..., image) and idx; every
        tensor is flattened to [H*W, -1] float32 rows and rendered by batchify_forward(is_test=True) -> (rgb [H,W,3], image [H,W,C], disp [H,W,1], idx),
        and with `render_normals` a fifth element, the normal map [H,W,3]"""
        self._mark_dirty()
        H, W = data['image'].shape[1:3]
        idx = data['idx']
        idx = int(idx.item()) if torch.is_tensor(idx) else int(idx)
        rays = {k: v.squeeze(0).reshape(H * W, -1).to(torch.float32) for k, v in data.items() if k != 'idx' and torch.is_tensor(v)}
        with torch.no_grad():
            ret = self.batchify_forward(rays, is_test=True)
        rgb = ret['rgb'].reshape((H, W, -1))
        out = (rgb, rays['image'].reshape((H, W, -1)).to(rgb.device), ret['disp'].reshape((H, W, -1)), idx)
        return out + ((ret['normal'].reshape((H, W, 3)),) if 'normal' in ret else ())

    def forward(self, data, is_test):
        randomized = not is_test
        ret = {}
        for i_level in range(self.num_levels):
            if i_level > 0:
                data = resample_along_rays(data, randomized, self.ray_shape, self.resample_padding)
            # level 0: sample_along_rays == cast_rays on the given z_vals; the Gaussians are formed inside the embedder kernel
            data, temp_ret = self.render(self.mlp(data), is_test)
            ret = temp_ret if not ret else merge_ret(ret, temp_ret)
        return ret

    def train_step(self, data, optimizer, **kwargs):
        data = {k: unfold_batching(v) for k, v in data.items()}
        geometry = self._geometry_wanted(data)
        ret = self._forward_geometry(data, geometry)
        mask = torch.broadcast_to(data['lossmult'], ret['rgb'].shape) if 'lossmult' in data else torch.ones_like(ret['rgb'])
        loss_fine = (mask * (ret['rgb'] - data['target_s']) ** 2).sum() / mask.sum()
        loss_coarse = (mask * (ret['coarse_rgb'] - data['target_s']) ** 2).sum() / mask.sum()
        loss = loss_fine + self.coarse_loss_mult * loss_coarse
        psnr = mse2psnr(loss_fine)
        log = {}
        if geometry:   # the coarse level weighted like its colour loss
            loss = self._add_geometry(loss, log, ret, data, [('', 1.0), ('coarse_', float(self.coarse_loss_mult))])
        return {'loss': loss, 'log_vars': {'loss': loss.item(), 'loss_fine': loss_fine.item(), 'loss_coarse': loss_coarse.item(), 'psnr': psnr.item(), **log},
                'num_samples': ret['rgb'].shape[0]}


@NETWORKS.register_module()
class HashNerfNetwork(NerfNetwork):
    render_normals = False   # True: the test path also returns per-pixel normal maps (batchify_forward)

    def __init__(self, cfg, sampler=None, mlp=None, render=None):
        super().__init__(cfg)
        self.sampler = builder.build_sampler(sampler)
        self.mlp = builder.build_mlp(mlp)
        self.render = builder.build_render(render)

    def forward(self, data, is_test=False):
        data = self.sampler.sample(data, self.mlp, is_test)
        data = self.mlp(data)
        data, ret = self.render(data, self.sampler, is_test)
        return ret

    def batchify_forward(self, data, is_test=False):
        """Inference over a whole ray set (hashnerf.py:69-71 via nerf.py:50-69: 4096-ray chunks, each = sample (host sync) -> 3 tcnn launches -> composite).
        Here the test path is ONE fused launch per call for any number of rays (xrb_ngp_render_fused; no chunk loop, no host sync, no [S,7]/[S,4] buffers);
        `fused_inference = False` or training falls back to the reference-shaped chunk loop over forward().
        The fused path also returns each ray's `depth` [n,1] (sum of w * t, not divided by alpha) and `disp` [n,1] (xrnerf_b200.ngp.disparity: 0 where
        alpha == 0); the reference-shaped path returns the reference's keys only.
        `render_normals` (default False) selects the normal-map output: the test path then renders through the chain (xrb_ngp_render_normals) and also
        returns each ray's `normal` [n,3] (sum of w * the samples' outward unit normals, not normalised; include/xrnerf_b200.h "Normal maps"); rgb,
        depth and disp come from the same chain render. It needs the fused path: with `fused_inference = False` it raises NotImplementedError."""
        smp = self.sampler
        normals = is_test and getattr(self, 'render_normals', False)
        if normals and not getattr(self, 'fused_inference', True):
            raise NotImplementedError('render_normals: normal maps come from the fused NGP renderer; set fused_inference = True')
        if not (is_test and getattr(self, 'fused_inference', True) and data['rays_o'].is_cuda and hasattr(smp, 'aabb_range')):
            return self._chunked_forward(data, is_test)
        from ..ngp import NgpRenderer, disparity
        smp.check_device(data)
        r = getattr(self, '_renderer', None)
        if r is None:
            r = self._renderer = NgpRenderer(self.mlp.field, aabb=tuple(float(a) for a in smp.aabb_range), near=smp.near_distance, cone=smp.cone_angle_constant,
                                             rgb_act=int(smp.rgb_activation), dens_act=int(smp.density_activation), bg=tuple(float(c) for c in self.render.bg_color))
        import xrnerf_b200.raymarch_cuda as rm
        r.calls = rm.rng_calls['ray_sampler']               # the same jitter stream the unfused path would use next (hidden static pcg32 of the reference, Q9)
        rays_o = data['rays_o'].contiguous().float()
        depth = torch.empty((rays_o.shape[0], 1), dtype=torch.float32, device=rays_o.device)
        if normals:
            return self._render_normals(r, rays_o, data['rays_d'].contiguous().float(), depth)
        rgb, alpha, _ = r.render_fused(rays_o, data['rays_d'].contiguous().float(), smp.density_grid_bitfield, depth=depth)
        rm.rng_calls['ray_sampler'] += 1
        return {'rgb': rgb.clone(), 'alpha': alpha.clone(), 'depth': depth, 'disp': disparity(depth, alpha)}

    def _render_normals(self, r, rays_o, rays_d, depth):
        """the `render_normals` view through the chain render. The sample buffer holds the renderer's budget per ray; a view that marched more rows is
        rendered again with a buffer of exactly its row count and the same call index (the same jitter), so no ray is dropped. One host read per view."""
        import xrnerf_b200.raymarch_cuda as rm
        from ..ngp import disparity
        n = rays_o.shape[0]
        normal = torch.empty((n, 3), dtype=torch.float32, device=rays_o.device)
        calls, bitfield = rm.rng_calls['ray_sampler'], self.sampler.density_grid_bitfield
        r.calls = calls
        rgb, alpha, _, counters = r.render(rays_o, rays_d, bitfield, depth=depth, normals=normal)
        marched = int(counters[1].item())
        if marched > n * r.budget:
            r.calls = calls
            rgb, alpha, _, counters = r.render(rays_o, rays_d, bitfield, depth=depth, normals=normal, max_samples=marched)
        rm.rng_calls['ray_sampler'] += 1
        return {'rgb': rgb.clone(), 'alpha': alpha.clone(), 'depth': depth, 'disp': disparity(depth, alpha), 'normal': normal}

    def val_step(self, data, optimizer=None, **kwargs):
        """hashnerf.py:54-93 (rank-0 loop over validation poses) with the image rendered by one launch and the PSNR taken on the device; every rank renders the
        poses it is given (SURVEY Q17). Returns the reference's keys plus 'psnr'; 'disps' holds one [H,W,1] disparity map per pose (the reference
        declares the list and leaves it empty, as the reference-shaped path `fused_inference = False` still does)."""
        if self.phase == 'test':
            return self.test_step(data, **kwargs)
        # validation may run right after mmcv's EMAHook swapped the parameters through `.data` (Parameter._version unchanged): rebuild the fp16 shadows, the cell
        # image and the wgmma weight image once per call instead of trusting the version key
        self.mlp.mark_dirty()
        data = {k: unfold_batching(v) for k, v in data.items()}
        poses, images = data['poses'], data.get('images')
        rgbs, disps, normals, gt_imgs, psnrs, elapsed = [], [], [], [], [], []
        with torch.no_grad():
            for i in range(poses.shape[0]):
                t0, t1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                t0.record()
                d = self.val_pipeline({'pose': poses[i], 'idx': i})
                ret = self.batchify_forward(d, is_test=True)
                rgb = recover_shape(ret['rgb'], d['src_shape'])
                if 'disp' in ret:
                    disps.append(recover_shape(ret['disp'], d['src_shape']))
                if 'normal' in ret:
                    normals.append(recover_shape(ret['normal'], d['src_shape']))
                if images is not None:
                    alpha = images[i][..., 3:].to(rgb.device)
                    gt = images[i][..., :3].to(rgb.device) * alpha
                    rgb = rgb * alpha
                    gt_imgs.append(gt)
                    psnrs.append(mse2psnr(img2mse(rgb, gt)))
                t1.record()
                rgbs.append(rgb); elapsed.append((t0, t1))
        torch.cuda.synchronize()
        out = {'rgbs': rgbs, 'disps': disps, 'gt_imgs': gt_imgs, 'elapsed_time': [a.elapsed_time(b) * 1e-3 for a, b in elapsed], 'psnr': [float(p.item()) for p in psnrs]}
        if getattr(self, 'render_normals', False):
            out['normals'] = normals      # one [H,W,3] normal map per pose (batchify_forward)
        return out

    def test_step(self, data, **kwargs):
        """hashnerf.py:95-111: one spiral pose per call; `data` already holds the pose's rays (rays_o, rays_d, src_shape, idx) from the test pipeline.
        A dict with only `poses` is run through the installed val pipeline first."""
        data = {k: unfold_batching(v) for k, v in data.items()}
        idx = data.get('idx', 0)
        idx = int(idx.item()) if torch.is_tensor(idx) else int(idx)
        if idx == 0 or not getattr(self, '_test_refreshed', False):       # first pose of a test run: the weights may have been swapped / loaded through `.data`
            self.mlp.mark_dirty()
            self._test_refreshed = True
        with torch.no_grad():
            d = data if 'rays_o' in data else self.val_pipeline({'pose': data['poses'], 'idx': idx})
            ret = self.batchify_forward(d, is_test=True)
        out = {'spiral_rgb': ret['rgb'], 'spiral_alpha': ret['alpha']}
        if 'disp' in ret:
            out['spiral_disp'] = ret['disp']
        if 'normal' in ret:
            out['spiral_normal'] = ret['normal']
        if 'src_shape' in d:
            out = {k: recover_shape(v, d['src_shape']) for k, v in out.items()}
        out['idx'] = idx
        return out

    def extract_mesh(self, resolution=256, threshold=2.5):
        """Triangle mesh of the field's density level set sigma = threshold -> (verts f32[V,3], faces i32[F,3]) CUDA tensors, vertices in the frame the
        rays are given in (the warped [0,1]^3 mapped through sampler.aabb_range; the unit cube before set_data), triangles wound counter-clockwise
        seen from outside. The density is sampled on a resolution^3 lattice over the whole warped domain (NgpField.density_lattice) and meshed by
        xrnerf_b200.mesh.marching_cubes.

        threshold is a density sigma, mapped to the network's raw output through the inverse of sampler.density_activation (ValueError outside
        its range). The default 2.5 is Instant-NGP's usual mesh threshold; it has not been checked here on a trained scene. For a Blender-frame
        mesh of a scene loaded the NGP way, pass the vertices through xrnerf_b200.mesh.ngp_to_nerf."""
        verts, faces = self._warped_mesh(resolution, threshold)
        return self._from_warped(verts), faces

    def _warped_mesh(self, resolution, threshold):
        """extract_mesh's triangles with the vertices still in the field's warped [0,1]^3 domain"""
        from ..mesh import marching_cubes, raw_density_threshold
        raw = raw_density_threshold(threshold, self.sampler.density_activation)
        self.mlp.mark_dirty()                  # weights may have been swapped through `.data` (EMAHook) since the last pack
        with torch.no_grad():
            vol = self.mlp.field.density_lattice((resolution,) * 3)
            return marching_cubes(vol, raw)

    def _from_warped(self, verts):
        lo, hi = (float(a) for a in getattr(self.sampler, 'aabb_range', (0.0, 1.0)))
        return verts * (hi - lo) + lo

    def extract_colored_mesh(self, resolution=256, threshold=2.5):
        """extract_mesh with a unit normal and a colour per vertex -> (verts f32[V,3], faces i32[F,3], normals f32[V,3], colors f32[V,3]) CUDA tensors, in
        the frame extract_mesh uses; verts and faces are bit-identical to extract_mesh(resolution, threshold).

        normal = -g / |g| (0 where g = 0), with g the gradient of the raw density at the vertex's warped position (NgpField.density_grad). Inside is
        "raw > threshold", so the normal points outward. sampler.aabb_range is a positive uniform scale, so the normals need no map. The gradient is that of
        the CUDA-core density (impl 0), while the lattice the vertices come from uses the field's impl: the two densities agree to the field's fp16
        tolerance, not bit for bit.

        color = sampler.rgb_activation(run_mlp(warped vertex, dir)[:, :3]) with dir = (1 - normal) / 2: the field seen from outside, looking along
        -normal, in the warped [0,1]^3 direction convention of the ray march (dir = (d + 1) / 2 for a unit ray direction d). A zero normal gives the
        direction (0.5, 0.5, 0.5). For the Blender frame, map verts with xrnerf_b200.mesh.ngp_to_nerf and normals with ngp_to_nerf_normals."""
        from ..mesh import activate_rgb, outward_normals
        verts_w, faces = self._warped_mesh(resolution, threshold)
        field = self.mlp.field
        with torch.no_grad():
            normals = outward_normals(field.density_grad(verts_w)[1])
            colors = activate_rgb(field.run_mlp(verts_w, (1.0 - normals) * 0.5)[:, :3], self.sampler.rgb_activation)
            return self._from_warped(verts_w), faces, normals, colors

    def train_step(self, data, optimizer, **kwargs):
        data = {k: unfold_batching(v) for k, v in data.items()}
        geometry = self._geometry_wanted(data, alpha_key='alpha')
        ret = self._forward_geometry(data, geometry)
        bs = ret['rgb'].shape[0]
        alpha = data['alpha'].detach()
        huber = HuberLoss(ret['rgb'], data['target_s'], 0.1, 'sum')
        psnr = mse2psnr(img2mse(ret['rgb'] * alpha, data['target_s'] * alpha))
        loss = huber * 5
        log = {}
        if geometry:   # reduction 'sum' like the Huber term; rays the compaction truncated drop out (their depth and alpha are partial sums)
            smp = self.sampler
            loss = self._add_geometry(loss, log, ret, data, [('', 1.0)], numsteps=(smp.rays_numsteps, smp.rays_numsteps_compacted), mean=False, alpha_key='alpha',
                                      target_alpha_key='alpha')
        return {'loss': loss, 'log_vars': {'loss': loss.item(), 'psnr': psnr.item(), **log}, 'num_samples': bs}
