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


class NgpRaySource:
    def __init__(self, poses43, images_rgba, K, seed=0, depths=None, depth_scale=0.33):
        """poses43 [I,4,3] NGP xforms (poses_nerf2ngp, datasets/utils/hashnerf.py:4-23); images_rgba [I,H,W,4] float32; K 3x3 intrinsics.
        depths [I,H,W] (optional): z-depth images, the distance along each camera's optical axis in the dataset's units (0 or not finite: no depth); batches
        then also hold target_depth [n,1], the ray parameter of the NGP ray (xrb_ngp_batch_depth) with depth_scale the scale of poses_nerf2ngp."""
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

    def cuda(self, device=None):
        self.poses, self.images = self.poses.cuda(device), self.images.cuda(device)
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
        _C.check(_C.lib.xrb_ngp_batch_sample(_C.f32(self.poses), _C.f32(self.images), self.I, self.H, self.W, self.fx, self.fy, self.cx, self.cy, _C.ptr(row_idx, torch.int64), n,
                                             _C.ptr(u_bg), self.seed, self.calls, _C.ptr(out['rays_o']), _C.ptr(out['rays_d']), _C.ptr(out['target_s']), _C.ptr(out['alpha']),
                                             _C.ptr(out['img_ids']), _C.ptr(out['bg_color']), _C.stream()), 'ngp_batch_sample')
        self.calls += 1
        if self.depths is not None:
            _C.require_cuda(self.depths)
            out['target_depth'] = f(1)
            _C.check(_C.lib.xrb_ngp_batch_depth(_C.f32(self.depths), self.I, self.H, self.W, self.fx, self.fy, self.cx, self.cy, self.depth_scale, _C.ptr(row_idx, torch.int64), n,
                                                _C.ptr(out['target_depth']), _C.stream()), 'ngp_batch_depth')
        return out


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
