"""Host-side objects of the fused Instant-NGP path: parameter storage (tcnn layouts), fp16 working copies, the packed
tensor-core weight image, and thin wrappers over the C ABI (include/xrnerf_b200.h: xrb_ngp_*).
"""
import math

import torch
from torch import nn

from . import _C

PER_LEVEL_SCALE = float(2.0 ** (math.log2(2048 * 1 / 16) / (16 - 1)))  # hashnerf_mlp.py:17-20 with bound=1 (Q6)


class NgpField(nn.Module):
    """HashNerfMLP's arithmetic (hash grid + SH + density/colour FullyFusedMLPs) as ONE kernel.

    Parameters keep tcnn's flat layouts and the reference's state_dict keys are produced by the registry class
    (xrnerf_b200.api.HashNerfMLP) that owns one of these. `impl`: 1 = wgmma tensor-core tiles, 0 = CUDA cores.
    """

    def __init__(self, n_levels=16, n_features=2, log2_hashmap_size=19, base_resolution=16, per_level_scale=PER_LEVEL_SCALE, width=64,
                 density_hidden=1, color_hidden=2, seed=1337, impl=1, n_packed_levels=None):
        super().__init__()
        # levels [0, n_packed_levels) are gathered from the cell image (xrb_ngp_table, include/xrnerf_b200.h): 7 = the five dense levels + the first two hashed
        # ones, 72.5 MB. With the 24.4 MB table that exceeds H100's 50 MB L2 (only 5 levels, 10.6 MB, or 6, 27.6 MB, fit beside it), yet on H100
        # 5, 6 and 7 levels show no measurable difference in speed (DESIGN.md §4.1). The trainer drops to 6 (the image is rebuilt after every optimiser step); 0 disables it.
        self.n_packed = 7 if n_packed_levels is None else int(n_packed_levels)
        self.cfg = _C.NgpConfig(n_levels, n_features, log2_hashmap_size, base_resolution, per_level_scale, width, density_hidden, color_hidden)
        n_hash = _C.lib.xrb_tcnn_hashgrid_num_params(self.cfg)
        if n_hash < 0:
            raise _C.XrbError(_C.lib.xrb_last_error().decode())
        g = torch.Generator().manual_seed(seed)
        self.hash_params = nn.Parameter((torch.rand(n_hash, generator=g) * 2 - 1) * 1e-4)

        def xavier(shapes):
            return torch.cat([((torch.rand(o, i, generator=g) * 2 - 1) * math.sqrt(6.0 / (i + o))).reshape(-1) for (o, i) in shapes])
        self.density_params = nn.Parameter(xavier([(width, 32)] + [(width, width)] * (density_hidden - 1) + [(16, width)]))
        self.color_params = nn.Parameter(xavier([(width, 32)] + [(width, width)] * (color_hidden - 1) + [(16, width)]))
        self.impl = impl
        self._ver = None
        self._table16 = self._dens16 = self._color16 = self._image = self._cells = self.tab = None

    # ---- fp16 working copies, cell image and packed wgmma weight image, refreshed when a master parameter changed
    def mark_dirty(self):
        """Force the next refresh(). Parameter._version does not see writes through `.data` (mmcv's EMAHook swaps parameters with
        `value.data.copy_(ema)`), so every entry point that may run after such a write calls this (val_step/test_step, load_state_dict, _apply)."""
        self._ver = None

    def _apply(self, fn, *a, **kw):
        self.mark_dirty()
        return super()._apply(fn, *a, **kw)

    def _load_from_state_dict(self, *a, **kw):
        self.mark_dirty()
        return super()._load_from_state_dict(*a, **kw)

    def _alloc(self, dev):
        self._table16 = torch.empty(self.hash_params.numel(), dtype=torch.float16, device=dev)
        self._dens16 = torch.empty(self.density_params.numel(), dtype=torch.float16, device=dev)
        self._color16 = torch.empty(self.color_params.numel(), dtype=torch.float16, device=dev)
        self._image = torch.empty(_C.lib.xrb_ngp_weight_image_bytes(self.cfg), dtype=torch.uint8, device=dev)
        nb = _C.lib.xrb_ngp_cell_image_bytes(self.cfg, self.n_packed) if self.n_packed > 0 else 0
        self._cells = torch.empty(nb, dtype=torch.uint8, device=dev) if nb else None
        self._bind_table()

    def _bind_table(self):
        """self.tab <- the xrb_ngp_table of the current fp16 table and cell image"""
        cells = self._cells is not None
        self.tab = _C.NgpTable(self._table16.data_ptr(), self._cells.data_ptr() if cells else None, self.n_packed if cells else 0)

    def use_table(self, table16=None):
        """Read the fp16 hash table from `table16`, a caller-owned fp16 tensor of hash_params.numel() elements (e.g. the working table inside a
        peer-exchange block, which other processes write), after copying the current table into it. None: from a private copy of the current table again."""
        if table16 is None:
            table16 = self._table16.clone()
        elif table16.data_ptr() == self._table16.data_ptr():
            return
        else:
            table16.copy_(self._table16)
        self._table16 = table16
        self._bind_table()

    def params_and_shadows(self):
        """(fp32 master, fp16 working copy) of the hash table, the density net and the colour net: what an optimiser updates in place before calling
        shadows_updated()"""
        return [(self.hash_params, self._table16), (self.density_params, self._dens16), (self.color_params, self._color16)]

    def set_packed_levels(self, n):
        """change how many levels the cell image holds (re-allocates and rebuilds it on the next refresh)"""
        if int(n) != self.n_packed:
            self.n_packed = int(n)
            self._table16 = None
            self.mark_dirty()

    def rebuild_cells(self):
        """cell image <- fp16 table (one kernel; called whenever the table changed)"""
        if self._cells is not None:
            _C.check(_C.lib.xrb_ngp_build_cell_image(self.cfg, _C.ptr(self._table16), self.n_packed, _C.ptr(self._cells), _C.stream()), 'build cell image')

    def _version_key(self):
        return (self.hash_params._version, self.density_params._version, self.color_params._version, self.hash_params.device)

    def refresh(self, force=False):
        if not force and self._version_key() == self._ver:
            return
        dev = self.hash_params.device
        if self._table16 is None or self._table16.device != dev:
            self._alloc(dev)
        s = _C.stream()
        _C.check(_C.lib.xrb_tcnn_cast_params(_C.ptr(self.hash_params.detach()), _C.ptr(self._table16), self.hash_params.numel(), s), 'cast hash')
        _C.check(_C.lib.xrb_tcnn_cast_params(_C.ptr(self.density_params.detach()), _C.ptr(self._dens16), self.density_params.numel(), s), 'cast density')
        _C.check(_C.lib.xrb_tcnn_cast_params(_C.ptr(self.color_params.detach()), _C.ptr(self._color16), self.color_params.numel(), s), 'cast color')
        self.shadows_updated()

    def shadows_updated(self):
        """The fp16 working copies hold the current parameters (an optimiser updated masters and copies in place, params_and_shadows()): re-pack the
        weight image, rebuild the cell image and record the parameters' versions as current, so that refresh() does not cast the masters again (a
        data-parallel trainer keeps only its own slice of the fp32 hash table up to date)."""
        _C.check(_C.lib.xrb_ngp_pack_weights(self.cfg, _C.ptr(self.density_params.detach()), _C.ptr(self.color_params.detach()), _C.ptr(self._image), _C.stream()), 'pack')
        self.rebuild_cells()
        self._ver = self._version_key()

    def run_mlp(self, pts, dirs, impl=None):
        """pts, dirs: [S,3] float32 views (row stride in floats may be > 3, e.g. coords[:, :3] / coords[:, 4:]). -> raw [S,4] f32."""
        _C.require_cuda(pts, dirs)
        self.refresh()
        return self.mlp_rows(pts, dirs, torch.empty((pts.shape[0], 4), dtype=torch.float32, device=pts.device), impl=impl)

    def mlp_rows(self, pts, dirs, out, n_rows_dev=None, impl=None):
        """run_mlp into `out` [S,4] from the working copies as they are, without refresh(): a training step between optimiser updates, where the fp32
        masters may be stale, calls this. n_rows_dev (int32 device tensor, optional): only the first min(S, n_rows_dev[0]) rows are evaluated."""
        (pp, ps), (dp, ds) = _C.rows(pts), _C.rows(dirs)
        impl = self.impl if impl is None else impl
        _C.check(_C.lib.xrb_ngp_mlp_forward(self.cfg, self.tab, _C.ptr(self._dens16), _C.ptr(self._color16), _C.ptr(self._image), pp, ps, dp, ds, pts.shape[0], _C.i32(n_rows_dev),
                                            _C.f32(out), impl, _C.stream()), 'ngp_mlp_forward')
        return out

    def forward(self, pts, dirs):
        """differentiable (w.r.t. the parameters) HashNerfMLP.run_mlp"""
        if torch.is_grad_enabled() and any(p.requires_grad for p in (self.hash_params, self.density_params, self.color_params)):
            return _FieldFn.apply(self, pts, dirs, self.hash_params, self.density_params, self.color_params)
        return self.run_mlp(pts, dirs)

    def tc_backward_ok(self):
        return (self.cfg.density_hidden, self.cfg.color_hidden) in ((1, 1), (1, 2))

    def backward_params(self, pts, dirs, grad_raw, out=None, impl=None):
        """dL/draw [S,4] -> (d_hash, d_density, d_color) fp32, accumulated into `out` if given (zero-initialised otherwise).
        impl 1 = wgmma tensor-core tiles (xrb_ngp_mlp_backward_tc), 0 = CUDA cores; default: self.impl where the tensor-core kernel is built."""
        _C.require_cuda(pts, dirs, grad_raw)
        self.refresh()
        if out is None:
            out = (torch.zeros_like(self.hash_params), torch.zeros_like(self.density_params), torch.zeros_like(self.color_params))
        return self.backward_rows(pts, dirs, grad_raw, out, impl=impl)

    def backward_rows(self, pts, dirs, grad_raw, out, n_rows_dev=None, impl=None, d_rows=None):
        """backward_params into `out` from the working copies as they are, without refresh() (see mlp_rows). n_rows_dev as in mlp_rows; the CUDA-core
        kernel (impl 0) takes its row count from the host, so with n_rows_dev it waits for the device once.
        d_rows (optional): a dense float32 [S,6] tensor that receives each effective row's (dL/dx, dL/dw), the gradient with respect to the warped
        position and direction (xrb_ngp_mlp_backward_tc_inputs, include/xrnerf_b200.h "NGP camera pose refinement"); tensor-core backward only."""
        n = pts.shape[0]
        (pp, ps), (dp, ds) = _C.rows(pts), _C.rows(dirs)
        impl = (self.impl if self.tc_backward_ok() else 0) if impl is None else impl
        if d_rows is not None:
            if impl != 1:
                raise _C.XrbError('XRB_E_BADARG: d_rows needs the tensor-core backward (impl 1)')
            if d_rows.dim() != 2 or d_rows.shape[1] != 6 or d_rows.shape[0] < n:
                raise _C.XrbError(f'XRB_E_BADARG: d_rows must be float32 [>= {n}, 6], got {tuple(d_rows.shape)}')
            _C.check(_C.lib.xrb_ngp_mlp_backward_tc_inputs(self.cfg, self.tab, _C.ptr(self._image), pp, ps, dp, ds, _C.f32(grad_raw), n, _C.i32(n_rows_dev), _C.f32(out[0]),
                                                           _C.f32(out[1]), _C.f32(out[2]), _C.f32(d_rows), _C.stream()), 'ngp_mlp_backward_tc_inputs')
            return out
        if impl == 1:
            _C.check(_C.lib.xrb_ngp_mlp_backward_tc(self.cfg, self.tab, _C.ptr(self._image), pp, ps, dp, ds, _C.f32(grad_raw), n, _C.i32(n_rows_dev), _C.f32(out[0]), _C.f32(out[1]),
                                                    _C.f32(out[2]), _C.stream()), 'ngp_mlp_backward_tc')
            return out
        if n_rows_dev is not None:
            n = min(n, int(n_rows_dev[0].item()))
        _C.check(_C.lib.xrb_ngp_mlp_backward(self.cfg, self.tab, _C.ptr(self._dens16), _C.ptr(self._color16), pp, ps, dp, ds, _C.f32(grad_raw), n, _C.f32(out[0]), _C.f32(out[1]),
                                             _C.f32(out[2]), _C.stream()), 'ngp_mlp_backward')
        return out

    def run_density(self, pts, impl=None):
        _C.require_cuda(pts)
        self.refresh()
        pp, ps = _C.rows(pts)
        n = pts.shape[0]
        out = torch.empty((n, 1), dtype=torch.float32, device=pts.device)
        impl = self.impl if impl is None else impl
        _C.check(_C.lib.xrb_ngp_density_forward(self.cfg, self.tab, _C.ptr(self._dens16), _C.ptr(self._image), pp, ps, n, _C.ptr(out), impl, _C.stream()), 'ngp_density_forward')
        return out

    def density_grad(self, pts):
        """pts: [n,3] float32 view in the warped [0,1]^3 domain (row stride may be > 3). -> (density f32[n,1], grad f32[n,3]): the raw density, bit-identical
        to run_density(pts, impl=0), and its gradient with respect to the position, on CUDA cores (xrb_ngp_density_grad, include/xrnerf_b200.h)."""
        _C.require_cuda(pts)
        self.refresh()
        pp, ps = _C.rows(pts)
        n = pts.shape[0]
        density = torch.empty((n, 1), dtype=torch.float32, device=pts.device)
        grad = torch.empty((n, 3), dtype=torch.float32, device=pts.device)
        _C.check(_C.lib.xrb_ngp_density_grad(self.cfg, self.tab, _C.ptr(self._dens16), pp, ps, n, _C.f32(density), _C.f32(grad), _C.stream()), 'ngp_density_grad')
        return density, grad

    def density_grad_tc(self, pts, density=True, order=None, n_rows_dev=None):
        """pts: [n,3] float32 view in the warped [0,1]^3 domain (row stride may be > 3, e.g. the chain's sample rows). -> (density f32[n,1] or None,
        grad f32[n,3]): the raw density, bit-identical to run_density(pts, impl=1), and its position gradient on tensor cores (xrb_ngp_density_grad_tc,
        include/xrnerf_b200.h: the gradient that the normal maps use). order (int32 device tensor, optional): slot j evaluates row order[j], a permutation
        of the effective rows; n_rows_dev (int32 device tensor, optional): only the first min(n, n_rows_dev[0]) rows are written."""
        _C.require_cuda(pts, order, n_rows_dev)
        self.refresh()
        pp, ps = _C.rows(pts)
        n = pts.shape[0]
        dens = torch.empty((n, 1), dtype=torch.float32, device=pts.device) if density else None
        grad = torch.empty((n, 3), dtype=torch.float32, device=pts.device)
        _C.check(_C.lib.xrb_ngp_density_grad_tc(self.cfg, self.tab, _C.ptr(self._image), pp, ps, n, _C.i32(n_rows_dev), _C.i32(order), _C.f32(dens), _C.f32(grad), _C.stream()),
                 'ngp_density_grad_tc')
        return dens, grad

    def density_lattice(self, shape, box=((0.0, 0.0, 0.0), (1.0, 1.0, 1.0)), impl=None):
        """Raw density on the lattice of shape (nz, ny, nx) over box = (box_min, box_max) in the warped [0,1]^3 domain -> f32[nz,ny,nx] on the field's
        device (x fastest). Lattice positions and limits: xrb_ngp_density_lattice (include/xrnerf_b200.h); each value equals run_density at that position."""
        if not self.hash_params.is_cuda:
            raise _C.XrbError('xrnerf_b200 kernels need CUDA tensors; there is no CPU fallback')
        self.refresh()
        nz, ny, nx = (int(n) for n in shape)
        dev = self.hash_params.device
        out = torch.empty((nz, ny, nx), dtype=torch.float32, device=dev)
        ws = torch.empty(_C.lib.xrb_ngp_density_lattice_workspace(), dtype=torch.uint8, device=dev)
        impl = self.impl if impl is None else impl
        _C.check(_C.lib.xrb_ngp_density_lattice(self.cfg, self.tab, _C.ptr(self._dens16), _C.ptr(self._image), nx, ny, nz, _C.float3(box[0]), _C.float3(box[1]), _C.f32(out), impl,
                                                _C.ptr(ws), _C.stream()), 'ngp_density_lattice')
        return out


class _FieldFn(torch.autograd.Function):
    """autograd bridge for NgpField.run_mlp: forward = xrb_ngp_mlp_forward, backward = xrb_ngp_mlp_backward (one kernel
    producing the gradients of all three parameter vectors). pts/dirs are not differentiated (the reference detaches them,
    hashnerf_mlp.py:58-68)."""

    @staticmethod
    def forward(ctx, field, pts, dirs, hash_params, density_params, color_params):
        ctx.field = field
        ctx.save_for_backward(pts, dirs)
        return field.run_mlp(pts, dirs)

    @staticmethod
    def backward(ctx, grad_raw):
        f = ctx.field
        pts, dirs = ctx.saved_tensors
        grad_raw = grad_raw.contiguous().to(torch.float32)
        dt, dd, dc = f.backward_params(pts, dirs, grad_raw)
        return None, None, None, dt, dd, dc


def _rays(t):
    """rays as the kernels read them: dense float32 [n,3] (a strided view - e.g. a Fortran-ordered array that came through torch.from_numpy - is
    copied, never reinterpreted)"""
    if t.dtype != torch.float32:
        raise _C.XrbError(f'XRB_E_BADARG: rays must be float32, got {t.dtype}')
    if t.dim() != 2 or t.shape[1] != 3:
        raise _C.XrbError(f'XRB_E_BADARG: rays must be [n,3], got {tuple(t.shape)}')
    return t.contiguous()


def _depth_ptr(depth, n, device, name='depth', width=1):
    """pointer of a caller-owned depth (width 1) or normal (width 3) output: a dense float32 tensor of n * width elements on the rays' device"""
    if not torch.is_tensor(depth) or depth.dtype != torch.float32 or depth.numel() != n * width or depth.device != device or (width > 1 and depth.shape[-1] != width):
        what = f'{depth.dtype} {tuple(depth.shape)} on {depth.device}' if torch.is_tensor(depth) else type(depth).__name__
        shape = f'of {n} elements' if width == 1 else f'of shape [{n},{width}]'
        raise _C.XrbError(f'XRB_E_BADARG: {name} must be a float32 tensor {shape} on {device}, got {what}')
    return _C.f32(depth)


def disparity(depth, alpha):
    """1 / max(1e-10, depth / alpha) where alpha > 0, and 0 where alpha == 0.

    NeRF's disp_map (nerf_render.py:32-36) is NaN where no weight was accumulated; an NGP image has many rays that miss the scene, and one NaN
    breaks the `x / max(x)` normalisation of a disparity video, so those rays get 0 here."""
    hit = alpha > 0
    return torch.where(hit, 1.0 / torch.clamp(depth / torch.where(hit, alpha, torch.ones_like(alpha)), min=1e-10), torch.zeros_like(alpha))


class NgpRenderer:
    """Fused inference render of a ray batch (xrb_ngp_render / xrb_ngp_render_fused): march -> field -> composite, no host sync, persistent workspace.

    samples_per_ray_budget sizes the sample buffers of the CHAIN path (n_rays * budget rows; the reference sizes them for 1024 per ray,
    ngp_grid_sampler.py:47). A ray that does not fit gets count 0 exactly like the reference (ray_sampler.cu:76-82) and renders as background:
    `overflowed(counters)` tells the caller (device-side compare, no sync), and HashNerfNetwork's validation uses the single-launch path, which
    has no sample buffer and therefore no overflow. Returned tensors are cached per batch size and OVERWRITTEN by the next call with the same
    size (pass `out=` to own them)."""

    def __init__(self, field, aabb=(0.0, 1.0), near=0.05, cone=1.0 / 256, rgb_act=2, dens_act=3, bg=(0.0, 0.0, 0.0), samples_per_ray_budget=64):
        self.field, self.aabb, self.near, self.cone = field, aabb, near, cone
        self.rgb_act, self.dens_act, self.bg = rgb_act, dens_act, tuple(bg)
        self.budget = samples_per_ray_budget
        self.calls = 0
        self._ws = None
        self._out = {}
        self._max_samples = 0

    def overflowed(self, counters):
        """0-dim bool tensor (device): did the last chain render drop rays because the batch marched more samples than the budget holds?"""
        return counters[1] > self._max_samples

    def render(self, rays_o, rays_d, bitfield, out=None, profile_events=None, depth=None, normals=None, max_samples=None):
        """profile_events: optional (torch.cuda.Event, torch.cuda.Event) recorded right before / after the field kernel (bench roofline).
        depth: optional caller-owned float32 tensor of n elements on the rays' device, filled with each ray's depth (xrb_ngp_render_depth,
        include/xrnerf_b200.h); the returned tuple is the same either way.
        normals: optional caller-owned float32 [n,3] tensor on the rays' device, filled with each ray's normal (xrb_ngp_render_normals: sum of w * the
        samples' outward unit normals, not normalised); it needs `depth` as well. max_samples: rows of the sample buffer (default n * the budget)."""
        if normals is not None and depth is None:
            raise _C.XrbError('XRB_E_BADARG: normals need a depth output as well (xrb_ngp_render_normals writes both)')
        _C.require_cuda(rays_o, rays_d, bitfield)
        rays_o, rays_d = _rays(rays_o), _rays(rays_d)
        n = rays_o.shape[0]
        depth_p = None if depth is None else _depth_ptr(depth, n, rays_o.device)
        normal_p = None if normals is None else _depth_ptr(normals, n, rays_o.device, 'normals', 3)
        f = self.field
        f.refresh()
        max_samples = n * self.budget if max_samples is None else int(max_samples)
        self._max_samples = max_samples
        ws_bytes = _C.lib.xrb_ngp_render_workspace if normal_p is None else _C.lib.xrb_ngp_render_normals_workspace
        need = ws_bytes(n, max_samples)
        if self._ws is None or self._ws.numel() < need or self._ws.device != rays_o.device:
            self._ws = torch.empty(need, dtype=torch.uint8, device=rays_o.device)
        if out is None:
            key = (n, rays_o.device)
            if key not in self._out:
                self._out[key] = (torch.empty((n, 3), dtype=torch.float32, device=rays_o.device), torch.empty((n, 1), dtype=torch.float32, device=rays_o.device),
                                  torch.empty((n, 2), dtype=torch.int32, device=rays_o.device), torch.empty(2, dtype=torch.int32, device=rays_o.device))
            out = self._out[key]
        rgb, alpha, numsteps, counters = out
        ev0 = ev1 = None
        if profile_events is not None:
            ev0, ev1 = (_C.C.c_void_p(e.cuda_event) for e in profile_events)
        head = (f.cfg, f.tab, _C.ptr(f._image), _C.u8(bitfield), _C.ptr(rays_o), _C.ptr(rays_d), n, max_samples, self.aabb[0], self.aabb[1], self.near, self.cone, 9121,
                self.calls, _C.float3(self.bg), self.rgb_act, self.dens_act, _C.f32(rgb), _C.f32(alpha))
        tail = (_C.i32(numsteps), _C.i32(counters), _C.ptr(self._ws), ev0, ev1, _C.stream())
        if depth_p is None:
            _C.check(_C.lib.xrb_ngp_render(*head, *tail), 'ngp_render')
        elif normal_p is None:
            _C.check(_C.lib.xrb_ngp_render_depth(*head, depth_p, *tail), 'ngp_render_depth')
        else:
            _C.check(_C.lib.xrb_ngp_render_normals(*head, depth_p, normal_p, *tail), 'ngp_render_normals')
        self.calls += 1
        return rgb, alpha, numsteps, counters

    def render_fused(self, rays_o, rays_d, bitfield, out=None, ws=None, depth=None):
        """Single-launch render (xrb_ngp_render_fused). Returns (rgb [n,3], alpha [n,1], n_samples i32[n]). `ws`: a zero-initialised workspace
        owned by the caller (one per stream when several batches are in flight); default: one per renderer. depth: as in render()
        (xrb_ngp_render_fused_depth)."""
        _C.require_cuda(rays_o, rays_d, bitfield)
        rays_o, rays_d = _rays(rays_o), _rays(rays_d)
        n = rays_o.shape[0]
        depth_p = None if depth is None else _depth_ptr(depth, n, rays_o.device)
        f = self.field
        f.refresh()
        if ws is None:
            if getattr(self, '_ws_fused', None) is None or self._ws_fused.device != rays_o.device:
                self._ws_fused = torch.zeros(_C.lib.xrb_ngp_render_fused_workspace(), dtype=torch.uint8, device=rays_o.device)
            ws = self._ws_fused
        if out is None:
            key = ('fused', n, rays_o.device)
            if key not in self._out:
                self._out[key] = (torch.empty((n, 3), dtype=torch.float32, device=rays_o.device), torch.empty((n, 1), dtype=torch.float32, device=rays_o.device),
                                  torch.empty(n, dtype=torch.int32, device=rays_o.device))
            out = self._out[key]
        rgb, alpha, ns = out
        head = (f.cfg, f.tab, _C.ptr(f._image), _C.u8(bitfield), _C.ptr(rays_o), _C.ptr(rays_d), n, self.aabb[0], self.aabb[1], self.near, self.cone, 9121, self.calls,
                _C.float3(self.bg), self.rgb_act, self.dens_act, _C.f32(rgb), _C.f32(alpha))
        tail = (_C.i32(ns), _C.ptr(ws), _C.stream())
        if depth_p is None:
            _C.check(_C.lib.xrb_ngp_render_fused(*head, *tail), 'ngp_render_fused')
        else:
            _C.check(_C.lib.xrb_ngp_render_fused_depth(*head, depth_p, *tail), 'ngp_render_fused_depth')
        self.calls += 1
        return rgb, alpha, ns
