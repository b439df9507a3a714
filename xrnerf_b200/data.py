"""Device-side ray sources for training (SURVEY §8f-1): the reference builds rays in DataLoader workers on the CPU
(/root/reference/xrnerf/datasets/pipelines/create.py:205-245, augment.py:12-76,:290-313; load_data/get_rays.py:72-98: a 100 x 640 000 x 11 fp32 = 2.8 GB host
table, shuffled with np.random.shuffle - "slow", hashnerf_dataset.py:44). Once the render step runs at tens of millions of rays per second that pipeline is the
bottleneck, so here a batch is generated from (pose, pixel index) on the device: no table, no H2D copy per step.

    NgpRaySource   = HashNerfDataset's ray table + HashBatchSample + RandomBGColor  (Instant-NGP training batches)
    NerfRaySource  = GetRays (+ Mip radii) + GetViewdirs + SelectRays                (one image per step, NeRF / Mip-NeRF "no_batching")
    select_rays_indices = SelectRays' coordinate construction incl. the precrop window

Randomness is explicit: the row permutation, the selection indices and the background uniforms can be passed in (parity tests against the reference's own
transforms, tests/test_gpu_data.py) or are drawn on the device.
"""
import torch

from . import _C


POSE_LR = 3e-3           # default Adam learning rate of the pose corrections (NgpRaySource.pose_step), chosen with the convergence test of tests/test_gpu_pose_refine.py (DESIGN §4.10)


def so3_exp(omega):
    """Exp of the rotation vectors omega [..., 3] -> [..., 3, 3]: I + A [w]x + B [w]x^2 with A = sin(t) / t, B = (1 - cos(t)) / t^2 = 2 sin^2(t/2) / t^2 (no
    cancellation), and their Taylor series through t^4 below t = 0.05 (truncation < 1e-11), so that the value and its autograd derivative are finite and accurate at 0"""
    t2 = (omega * omega).sum(-1, keepdim=True)[..., None]
    small = t2 < 0.0025
    t = torch.sqrt(torch.where(small, torch.ones_like(t2), t2))
    h = 0.5 * t
    a = torch.where(small, 1.0 - t2 / 6.0 + t2 * t2 / 120.0, torch.sin(t) / t)
    b = torch.where(small, 0.5 - t2 / 24.0 + t2 * t2 / 720.0, 0.5 * (torch.sin(h) / h) ** 2)
    x, y, z = omega.unbind(-1)
    zero = torch.zeros_like(x)
    K = torch.stack([zero, -z, y, z, zero, -x, -y, x, zero], -1).reshape(omega.shape[:-1] + (3, 3))
    eye = torch.eye(3, dtype=omega.dtype, device=omega.device)
    return eye + a * K + b * (K @ K)


def corrected_poses(poses43, xi):
    """NGP xforms [I,4,3] (rows 0..2: the rotation's columns, row 3: the centre) corrected by xi = (omega, rho) [I,6]: R' = R Exp(omega), o' = o + rho
    (include/xrnerf_b200.h, "NGP camera pose refinement"). Rows 0..2 of an xform are R^T, so they become Exp(omega)^T R^T."""
    rot = so3_exp(xi[:, :3]).transpose(-1, -2) @ poses43[:, :3]
    return torch.cat([rot, (poses43[:, 3] + xi[:, 3:])[:, None]], 1)


def pose_xi_grad(poses43, xi, d_poses):
    """dL/dxi [I,6] from dL/dP' [I,4,3] at the corrected poses corrected_poses(poses43, xi): autograd of the Exp map (float32)"""
    with torch.enable_grad():
        x = xi.detach().clone().requires_grad_(True)
        (g,) = torch.autograd.grad(corrected_poses(poses43, x), x, d_poses)
    return g


class NgpRaySource:
    def __init__(self, poses43, images_rgba, K, seed=0, depths=None, depth_scale=0.33, refine_poses=False):
        """poses43 [I,4,3] NGP xforms (poses_nerf2ngp, datasets/utils/hashnerf.py:4-23); images_rgba [I,H,W,4] float32; K 3x3 intrinsics.
        depths [I,H,W] (optional): z-depth images, the distance along each camera's optical axis in the dataset's units (0 or not finite: no depth); batches
        then also hold target_depth [n,1], the ray parameter of the NGP ray (xrb_ngp_batch_depth) with depth_scale the scale of poses_nerf2ngp.
        refine_poses: hold a correction xi [I,6] per image (include/xrnerf_b200.h, "NGP camera pose refinement"), initially 0, and generate every batch from
        the corrected poses; batches then also hold row_idx [n] (int64) and pose_xi [I,6], the corrections they were drawn with, and pose_step() updates xi."""
        self.poses = torch.as_tensor(poses43, dtype=torch.float32).contiguous()
        self.images = torch.as_tensor(images_rgba, dtype=torch.float32).contiguous()
        self.I, self.H, self.W = self.images.shape[:3]
        self.depths = None if depths is None else torch.as_tensor(depths, dtype=torch.float32).contiguous()
        if self.depths is not None and tuple(self.depths.shape) != (self.I, self.H, self.W):
            raise ValueError(f'depths: expected shape {(self.I, self.H, self.W)}, got {tuple(self.depths.shape)}')
        self.depth_scale = float(depth_scale)
        self.fx, self.fy, self.cx, self.cy = float(K[0][0]), float(K[1][1]), float(K[0][2]), float(K[1][2])
        self.n_rows = self.I * self.H * self.W
        self.perm = None
        self.cur_i = 0
        self.seed, self.calls = int(seed), 0
        self.refine_poses = bool(refine_poses)
        if self.refine_poses:
            self.xi, self.xi_m, self.xi_v = (torch.zeros((self.I, 6), dtype=torch.float32) for _ in range(3))
            self.pose_steps = 0

    def cuda(self, device=None):
        self.poses, self.images = self.poses.cuda(device), self.images.cuda(device)
        if self.refine_poses:
            self.xi, self.xi_m, self.xi_v = self.xi.cuda(device), self.xi_m.cuda(device), self.xi_v.cuda(device)
        if self.depths is not None:
            self.depths = self.depths.cuda(device)
        if self.perm is not None:
            self.perm = self.perm.cuda(device)
        return self

    def shuffle(self, perm=None, generator=None):
        """np.random.shuffle(rays_rgb) of the reference (hashnerf_dataset.py:41-44) as a row permutation; `perm` given for tests."""
        dev = self.images.device
        self.perm = torch.as_tensor(perm, dtype=torch.int64).to(dev).contiguous() if perm is not None else torch.randperm(self.n_rows, device=dev, generator=generator)
        self.cur_i = 0
        return self

    def next_batch(self, n_rand, u_bg=None):
        """HashBatchSample.__call__ (cur_i wraps to 0 when the next slice would reach the end, create.py:168-171) + RandomBGColor. Returns the reference's data-dict keys."""
        if self.perm is None:
            self.shuffle()
        if self.cur_i + n_rand >= self.n_rows:
            self.cur_i = 0
        rows = self.perm[self.cur_i:self.cur_i + n_rand]
        self.cur_i += n_rand
        return self.rows(rows, u_bg)

    def rows(self, row_idx, u_bg=None):
        dev = self.images.device
        _C.require_cuda(self.images, self.poses, row_idx)
        n = int(row_idx.numel())
        row_idx = row_idx.to(torch.int64).contiguous()
        f = lambda c: torch.empty((n, c), dtype=torch.float32, device=dev)
        out = dict(rays_o=f(3), rays_d=f(3), target_s=f(3), alpha=f(1), img_ids=f(1), bg_color=f(3))
        if u_bg is not None:
            u_bg = torch.as_tensor(u_bg, dtype=torch.float32).to(dev).contiguous()
        poses = self.poses
        if self.refine_poses:
            xi = self.xi.clone()
            poses = corrected_poses(self.poses, xi).contiguous()
            out.update(row_idx=row_idx, pose_xi=xi)
        _C.check(_C.lib.xrb_ngp_batch_sample(_C.f32(poses), _C.f32(self.images), self.I, self.H, self.W, self.fx, self.fy, self.cx, self.cy, _C.ptr(row_idx, torch.int64), n,
                                             _C.ptr(u_bg), self.seed, self.calls, _C.ptr(out['rays_o']), _C.ptr(out['rays_d']), _C.ptr(out['target_s']), _C.ptr(out['alpha']),
                                             _C.ptr(out['img_ids']), _C.ptr(out['bg_color']), _C.stream()), 'ngp_batch_sample')
        self.calls += 1
        if self.depths is not None:
            _C.require_cuda(self.depths)
            out['target_depth'] = f(1)
            _C.check(_C.lib.xrb_ngp_batch_depth(_C.f32(self.depths), self.I, self.H, self.W, self.fx, self.fy, self.cx, self.cy, self.depth_scale, _C.ptr(row_idx, torch.int64), n,
                                                _C.ptr(out['target_depth']), _C.stream()), 'ngp_batch_depth')
        return out

    def refined_poses(self):
        """the corrected NGP xforms [I,4,3] (the given poses without refine_poses), for rendering and export"""
        if not self.refine_poses:
            return self.poses.clone()
        return corrected_poses(self.poses, self.xi)

    def pose_step(self, batch, grad_o, grad_d, lr=POSE_LR, betas=(0.9, 0.999), eps=1e-8):
        """One Adam step on the pose corrections from the gradient of a loss with respect to the rays of `batch` (a dict this source returned): grad_o /
        grad_d [n,3], e.g. NgpTrainer(ray_grad=True)'s grad_rays_o / grad_rays_d after step(batch['rays_o'], batch['rays_d'], ...). xrb_ngp_pose_grad chains them
        to the corrected poses, autograd of the Exp map to xi, then xrb_adam_ema_step updates xi. No host synchronisation.
        The gradient is taken at the corrections the batch was drawn with (batch['pose_xi']): a batch generated before the previous pose_step (e.g. one
        prefetched for NgpTrainer.step's next_rays) yields a gradient one step stale, which Adam tolerates at these step sizes."""
        if not self.refine_poses:
            raise _C.XrbError('XRB_E_BADARG: pose_step needs NgpRaySource(..., refine_poses=True)')
        if 'pose_xi' not in batch or 'row_idx' not in batch:
            raise _C.XrbError('XRB_E_BADARG: pose_step needs a batch drawn from this source with refine_poses=True (row_idx, pose_xi)')
        row_idx, xi = batch['row_idx'], batch['pose_xi']
        n = int(row_idx.numel())
        for name, g in (('grad_o', grad_o), ('grad_d', grad_d)):
            if not torch.is_tensor(g) or g.dtype != torch.float32 or tuple(g.shape) != (n, 3):
                what = f'{g.dtype} {tuple(g.shape)}' if torch.is_tensor(g) else type(g).__name__
                raise _C.XrbError(f'XRB_E_BADARG: {name} must be float32 [{n},3], got {what}')
        _C.require_cuda(self.poses, row_idx, grad_o, grad_d)
        poses = corrected_poses(self.poses, xi).contiguous()
        grad_o, grad_d = grad_o.contiguous(), grad_d.contiguous()      # held by name until the launch: the kernel reads them
        d_poses = torch.zeros((self.I, 4, 3), dtype=torch.float32, device=self.poses.device)
        _C.check(_C.lib.xrb_ngp_pose_grad(_C.ptr(row_idx, torch.int64), n, _C.f32(poses), self.I, self.H, self.W, self.fx, self.fy, self.cx, self.cy, _C.f32(grad_o),
                                          _C.f32(grad_d), _C.f32(d_poses), _C.stream()), 'ngp_pose_grad')
        g = pose_xi_grad(self.poses, xi, d_poses).contiguous()
        self.pose_steps += 1
        _C.check(_C.lib.xrb_adam_ema_step(_C.f32(self.xi), None, _C.f32(g), _C.f32(self.xi_m), _C.f32(self.xi_v), self.xi.numel(), float(lr), float(betas[0]), float(betas[1]),
                                          float(eps), 0.0, self.pose_steps, 1.0, None, 0.0, _C.stream()), 'pose adam')
        return g


def select_rays_indices(H, W, sel_n, iter_n=0, precrop_iters=0, precrop_frac=0.5, select_inds=None, generator=None, device='cpu'):
    """SelectRays (augment.py:31-66): row-major pixel numbers of the selected rays. `select_inds` = the indices np.random.choice would return (tests); default:
    a random subset without replacement drawn with torch."""
    if precrop_iters != 0 and iter_n < precrop_iters:
        dH, dW = int(H // 2 * precrop_frac), int(W // 2 * precrop_frac)
        h0, w0, hh, ww = H // 2 - dH, W // 2 - dW, 2 * dH, 2 * dW
    else:
        h0, w0, hh, ww = 0, 0, H, W
    n_all = hh * ww
    if select_inds is None:
        select_inds = torch.randperm(n_all, generator=generator, device=device)[:sel_n]
    k = torch.as_tensor(select_inds, dtype=torch.int64)
    return ((h0 + k // ww) * W + (w0 + k % ww)).to(torch.int32)


class NerfRaySource:
    """GetRays(+radii) + GetViewdirs + SelectRays for one posed image on the device (xrb_nerf_get_rays over the selected pixels only)."""

    def __init__(self, H, W, K, include_radius=False):
        self.H, self.W = int(H), int(W)
        self.fx, self.fy, self.cx, self.cy = float(K[0][0]), float(K[1][1]), float(K[0][2]), float(K[1][2])
        self.include_radius = include_radius

    def batch(self, c2w, image_rgb, pixel_idx, depth=None, alpha=None):
        """c2w [3,4] or [4,4] camera-to-world (host or device), image_rgb [H,W,3] device tensor, pixel_idx int32[n] (select_rays_indices) ->
        rays_o, rays_d, viewdirs, target_s (+ radii). depth [H,W] (z-depth; GetRays directions have a unit camera-z component, so it is the ray's z
        already) and alpha [H,W] (optional, device) add target_depth / target_alpha [n,1] at the same pixels."""
        dev = image_rgb.device
        _C.require_cuda(image_rgb)
        pixel_idx = pixel_idx.to(device=dev, dtype=torch.int32).contiguous()
        n = int(pixel_idx.numel())
        c = torch.as_tensor(c2w, dtype=torch.float32).cpu().reshape(-1, 4)[:3].contiguous()
        c2w_host = (_C.C.c_float * 12)(*[float(v) for v in c.reshape(-1)])
        o = torch.empty((n, 3), device=dev); d = torch.empty((n, 3), device=dev); v = torch.empty((n, 3), device=dev)
        r = torch.empty((n, 1), device=dev) if self.include_radius else None
        _C.check(_C.lib.xrb_nerf_get_rays(c2w_host, self.H, self.W, self.fx, self.fy, self.cx, self.cy, 0, _C.i32(pixel_idx), n, _C.ptr(o), _C.ptr(d), _C.ptr(v), _C.ptr(r), _C.stream()),
                 'get_rays')
        out = dict(rays_o=o, rays_d=d, viewdirs=v, target_s=image_rgb.reshape(-1, image_rgb.shape[-1])[pixel_idx.long()])
        if r is not None:
            out['radii'] = r
        for key, img in (('target_depth', depth), ('target_alpha', alpha)):
            if img is not None:
                _C.require_cuda(img)
                out[key] = img.reshape(-1, 1).to(torch.float32)[pixel_idx.long()]
        return out
