"""Fused Instant-NGP training step (HashNerfNetwork.train_step, /root/reference/xrnerf/models/networks/hashnerf.py:32-52 +
ngp_grid_sampler.py:189-266 + the mmcv OptimizerHook/Adam it runs under) without host synchronisation:

  [aux stream, one step ahead]  march -> compaction            (needs only rays + occupancy bitfield, not the weights)
  [main stream]  field forward (wgmma) -> composite forward -> Huber x5 loss+grad (one kernel) -> composite backward ->
                 field backward (wgmma: dX and dW as tensor-core instructions) -> gradient exchange -> fused Adam (+ fp16 / weight-image / cell-image refresh)

Every per-sample kernel reads the compacted sample count on the device (`n_rows_dev`), so the work follows the batch actually marched.

Rays trained per step. The reference compacts a batch to `target_batch_size` = 2^18 samples by truncation in ray order (compacted_coord.cu:5-77) and keeps the
batch near that size with `update_batch_rays` (ngp_grid_sampler.py:268-281: every 16 steps n_rays <- ceil128(n_rays * 2^18 / mean compacted count)). A fixed
65 536-ray batch of the benchmark scene marches ~700 K samples, so with T = 2^18 most rays would be truncated away and never trained; `NgpTrainer` therefore
takes T as a parameter (bench: 2^20, nothing truncated), reports `trained_rays()` (rays whose every sample took part), and implements the reference's
adaptive rule for callers that size the batch like the reference does (`adaptive_n_rays`).

Data parallel (world > 1): every rank holds identical weights and takes a disjoint ray batch. The gradient exchange of the 12.2 M-entry hash table is SHARDED
(what MMDistributedDataParallel's dense fp32 all-reduce does in the reference, core/apis/train.py:28-36, at a quarter of the bytes):
  bf16 pack -> reduce-scatter (each rank receives the sum of ITS 1/world slice) -> Adam on the rank's slice of (master, exp_avg, exp_avg_sq, ema) ->
  all-gather of the refreshed fp16 working copy
so a rank moves 2 x 24.4 MB x (world-1)/world instead of 2 x 48.8 MB x (world-1)/world, and runs 1/world of the Adam pass. The fp32 master / EMA slices of
the other ranks are fetched on demand (`sync_master()`: checkpointing, validation with EMA weights). The ~10 K MLP weights use a plain fp32 all-reduce.
`grad_comm='allreduce'` keeps the dense fp32 all-reduce of round 1. The march of step k+1 runs on the aux stream while step k's exchange is in flight.
The occupancy grid is updated identically on every rank (same weights + same RNG call index => same grid, SURVEY §8e), so it needs no communication.
"""
import os

import torch

from . import _C


def shard_range(n, world, rank, align=8):
    """[begin, end) of rank's slice of an n-element vector cut into `world` equal slices of ceil(n / world) rounded up to `align` elements
    (the last slices may be short or empty); `padded` = world * slice length is the size collectives operate on."""
    per = -(-n // world)
    per = -(-per // align) * align
    b = min(rank * per, n)
    return b, min(b + per, n), per, per * world


class ShardedExchange:
    """Host logic of the sharded gradient exchange for ONE parameter vector (device-agnostic: the gloo CPU test runs it).

    reduce_scatter_sum(src)  -> this rank's slice of sum_over_ranks(src)   (src: padded wire-format vector)
    all_gather(full, mine)   -> every rank's slice written into `full` (padded)
    Backends without reduce_scatter (gloo) fall back to all_reduce + slice: same result, used only by the CPU test."""

    def __init__(self, n, group=None):
        import torch.distributed as dist
        self.dist, self.group = dist, group
        self.world = dist.get_world_size(group) if dist.is_initialized() else 1
        self.rank = dist.get_rank(group) if dist.is_initialized() else 0
        self.n = n
        self.begin, self.end, self.per, self.padded = shard_range(n, self.world, self.rank)

    def reduce_scatter_sum(self, src, out):
        assert src.numel() == self.padded and out.numel() == self.per
        if self.world == 1:
            out.copy_(src[:self.per])
            return out
        try:
            self.dist.reduce_scatter_tensor(out, src, op=self.dist.ReduceOp.SUM, group=self.group)
        except (RuntimeError, NotImplementedError):
            tmp = src.clone()
            self.dist.all_reduce(tmp, op=self.dist.ReduceOp.SUM, group=self.group)
            out.copy_(tmp[self.rank * self.per:(self.rank + 1) * self.per])
        return out

    def all_gather(self, full, mine):
        assert full.numel() == self.padded and mine.numel() == self.per
        if self.world == 1:
            full[:self.per].copy_(mine)
            return full
        try:
            self.dist.all_gather_into_tensor(full, mine, group=self.group)
        except (RuntimeError, NotImplementedError):
            parts = [torch.empty_like(mine) for _ in range(self.world)]
            self.dist.all_gather(parts, mine, group=self.group)
            full.copy_(torch.cat(parts))
        return full


class _DevView:
    """a raw device pointer as a __cuda_array_interface__ object (torch.as_tensor wraps it without copying)"""

    def __init__(self, ptr, n, typestr):
        self.__cuda_array_interface__ = {'shape': (int(n),), 'typestr': typestr, 'data': (int(ptr), False), 'version': 2}


class PeerExchange:
    """The optimiser step of the data-parallel NGP trainer as ONE exchange over NVLink peer memory (csrc/peer_adam.cu, include/xrnerf_b200.h xrb_peer_*): every rank owns an
    exchange block (flags | bf16 table gradient | fp32 MLP gradients | fp16 working table) that every other process maps through CUDA IPC. `t16` is this rank's working table INSIDE
    its block: the field reads it, the other ranks' optimiser kernels write their slices into it."""

    def __init__(self, n_table, n_mlp, group, dev):
        import torch.distributed as dist
        self.world, self.rank = dist.get_world_size(group), dist.get_rank(group)
        if self.world > 8:
            raise _C.XrbError('peer exchange: at most 8 ranks (one NVSwitch domain)')
        self.n_table, self.n_mlp = int(n_table), int(n_mlp)
        self.begin, self.end, self.per, self.padded = shard_range(n_table, self.world, self.rank)
        a16 = lambda x: (x + 15) // 16 * 16   # noqa: E731
        self.off_g16 = 128
        self.off_gmlp = a16(self.off_g16 + 2 * self.padded)
        self.off_t16 = a16(self.off_gmlp + 4 * self.n_mlp)
        self.bytes = a16(self.off_t16 + 2 * self.padded)
        # every rank must reach the same verdict (all map everything, or all fall back): failures are gathered, never raised between two collectives
        own, handle, err = _C.C.c_void_p(), (_C.C.c_char * 64)(), None
        try:
            _C.check(_C.lib.xrb_peer_alloc(self.bytes, _C.C.byref(own), handle), 'peer_alloc')
        except _C.XrbError as e:
            err = str(e)
        self.own = own.value
        handles = [None] * self.world
        dist.all_gather_object(handles, None if err else bytes(handle.raw), group=group)
        self.opened = []
        self.layout = _C.PeerLayout(self.world, self.rank, (_C.C.c_void_p * 8)(), self.off_g16, self.off_gmlp, self.off_t16, self.n_table, self.per, self.n_mlp)
        if all(h is not None for h in handles):
            for p in range(self.world):
                if p == self.rank:
                    self.layout.base[p] = self.own
                    continue
                ptr = _C.C.c_void_p()
                try:
                    _C.check(_C.lib.xrb_peer_open((_C.C.c_char * 64).from_buffer_copy(handles[p]), _C.C.byref(ptr)), f'peer_open(rank {p})')
                except _C.XrbError as e:
                    err = str(e)
                    break
                self.layout.base[p] = ptr.value
                self.opened.append(ptr.value)
        else:
            err = err or 'another rank could not allocate its exchange block'
        verdicts = [None] * self.world
        dist.all_gather_object(verdicts, err, group=group)
        if any(v is not None for v in verdicts):
            self.close()
            raise _C.XrbError('peer exchange unavailable: ' + '; '.join(f'rank {r}: {v}' for r, v in enumerate(verdicts) if v is not None))
        self.t16 = torch.as_tensor(_DevView(self.own + self.off_t16, self.padded, '<f2'), device=dev)
        self.step = 0
        dist.barrier(group=group)       # every block is mapped everywhere before anyone signals

    def check(self):
        st = _C.C.c_uint32(0)
        _C.check(_C.lib.xrb_peer_status(self.own, _C.C.byref(st), _C.stream()), 'peer_status')
        if st.value:
            raise _C.XrbError(f'peer exchange: a rank did not arrive within the kernel time-out (status {st.value}: 1 = gradients, 9 = updated slices)')

    def __del__(self):
        try:
            self.close()
        except Exception:   # noqa: BLE001  (interpreter shutdown)
            pass

    def close(self):
        """releases the mappings and this rank's block. `t16` (and anything aliasing it, e.g. a field's working table) must not be used afterwards: NgpTrainer.close() re-homes the table first."""
        if not getattr(self, 'own', None) and not getattr(self, 'opened', None):
            return
        if torch.cuda.is_available():
            torch.cuda.synchronize()
        for p in getattr(self, 'opened', []):
            _C.lib.xrb_peer_close(p)
        self.opened = []
        if getattr(self, 'own', None):
            _C.lib.xrb_peer_free(self.own)
        self.own = None


def huber5_grad(rgb, target, delta=0.1):
    """d/d rgb of 5 * HuberLoss(rgb, target, 0.1, 'sum') (networks/utils/metrics.py:8-16, hashnerf.py:39-44) and the loss value (torch restatement of
    xrb_ngp_huber5_grad, kept for the CPU tests that pin it to the reference's own metrics.py)."""
    diff = rgb - target
    rel = diff.abs()
    loss = torch.where(rel > delta, rel - 0.5 * delta, 0.5 / delta * rel * rel).sum() * 5
    grad = torch.where(rel > delta, torch.sign(diff), diff / delta) * 5
    return loss, grad


def adaptive_n_rays(n_rays, measured_total, n_steps=16, target_batch_size=1 << 18):
    """update_batch_rays (ngp_grid_sampler.py:268-281): n_rays <- min(ceil128(n_rays * T / max(measured / n_steps, 1)), 2^18)"""
    measured = max(measured_total / float(n_steps), 1.0)
    n = int(n_rays * target_batch_size / measured)
    n = (n + 127) // 128 * 128
    return min(n, 1 << 18)


class _Slot:
    """sample buffers of one in-flight batch (two slots: the march of step k+1 runs while step k trains)"""

    def __init__(self, n_rays, cap, T, dev):
        self.coords = torch.empty((cap, 7), dtype=torch.float32, device=dev)
        self.coords_c = torch.zeros((T, 7), dtype=torch.float32, device=dev)
        self.rays_index = torch.zeros((n_rays, 1), dtype=torch.int32, device=dev)
        self.numsteps = torch.zeros((n_rays, 2), dtype=torch.int32, device=dev)
        self.numsteps_c = torch.zeros((n_rays, 2), dtype=torch.int32, device=dev)
        self.counter = torch.zeros(2, dtype=torch.int32, device=dev)
        self.cnt_c = torch.zeros(2, dtype=torch.int32, device=dev)
        self.ws_march = torch.empty(_C.lib.xrb_rm_rays_sampler_workspace(n_rays), dtype=torch.uint8, device=dev)
        self.ws_compact = torch.empty(_C.lib.xrb_rm_compacted_coord_workspace(n_rays), dtype=torch.uint8, device=dev)
        self.ready = None          # event: march + compaction of the batch in this slot are done
        self.free = None           # event: the training step that used this slot has finished reading it
        self.rays = None


class NgpTrainer:
    def __init__(self, field, bitfield, n_rays, target_batch_size=1 << 18, aabb=(0.0, 1.0), near=0.05, cone=1.0 / 256, rgb_act=2, dens_act=3,
                 lr=1e-2, betas=(0.9, 0.99), eps=1e-15, weight_decay=1e-6, samples_per_ray_budget=64, group=None, ema_momentum=None, ema_warm_up=100,
                 grad_comm='auto', bwd_impl=None, depth_weight=0.0, opacity_weight=0.0, ray_grad=False):
        import torch.distributed as dist
        self.f, self.bitfield, self.n_rays, self.T = field, bitfield, n_rays, int(target_batch_size)
        self.aabb, self.near, self.cone, self.rgb_act, self.dens_act = aabb, near, cone, rgb_act, dens_act
        self.lr, self.betas, self.eps, self.wd, self.group = lr, betas, eps, weight_decay, group
        dev = field.hash_params.device
        self.dev = dev
        self.world = dist.get_world_size(group) if dist.is_available() and dist.is_initialized() else 1
        self.rank = dist.get_rank(group) if self.world > 1 else 0
        self.grad_comm = grad_comm if self.world > 1 else 'none'
        self.bwd_impl = (1 if field.tc_backward_ok() else 0) if bwd_impl is None else bwd_impl
        self.fwd_impl = 1
        self.ray_grad = bool(ray_grad)
        if self.ray_grad:
            if self.world > 1:
                raise ValueError('ray_grad: only for a single process (world size 1)')
            if self.bwd_impl != 1 or not field.tc_backward_ok():
                raise ValueError(f'ray_grad: needs the tensor-core field backward, built for (density_hidden, color_hidden) = (1,1) or (1,2); this field is '
                                 f'({field.cfg.density_hidden},{field.cfg.color_hidden}) with bwd_impl {self.bwd_impl}')
        self.params = [field.hash_params, field.density_params, field.color_params]
        if field.n_packed > 6:
            field.set_packed_levels(6)     # the cell image is rebuilt after every optimiser step: 35 us for 6 levels (27.6 MB) vs 88 us for 7
        field.refresh()
        n_hash = field.hash_params.numel()
        if self.grad_comm not in ('none', 'auto', 'sharded', 'allreduce', 'peer'):
            raise ValueError(f'grad_comm {grad_comm!r}: one of auto, peer, sharded, allreduce')
        self.px = None
        if self.grad_comm in ('auto', 'peer'):     # auto: the peer-memory exchange where CUDA IPC between the ranks works (one NVLink / NVSwitch domain), else NCCL reduce-scatter / all-gather
            try:
                self.px = PeerExchange(field.hash_params.numel(), field.density_params.numel() + field.color_params.numel(), group, dev)
                self.grad_comm = 'peer'
            except _C.XrbError:
                if self.grad_comm == 'peer':
                    raise
                self.grad_comm = 'sharded'
        self.ex = ShardedExchange(n_hash, group) if self.grad_comm in ('sharded', 'peer') else None   # peer mode: slice bounds + the rare whole-tensor gathers (state_dict, EMA)
        pad = self.ex.padded if self.ex else n_hash
        # flat fp32 gradient: [hash (padded to the collective's size) | density | colour]
        self.gflat = torch.zeros(pad + field.density_params.numel() + field.color_params.numel(), dtype=torch.float32, device=dev)
        self.g_hash = self.gflat[:n_hash]
        self.g_mlp = self.gflat[pad:]
        self.g_dens = self.g_mlp[:field.density_params.numel()]
        self.g_color = self.g_mlp[field.density_params.numel():]
        self.grads = [self.g_hash, self.g_dens, self.g_color]
        if self.px is not None:
            field.use_table(self.px.t16[:self.px.n_table])     # the field's working table lives inside this rank's exchange block (the other ranks write their slices into it)
        if self.ex:
            if self.px is None:
                self.g16 = torch.zeros(pad, dtype=torch.bfloat16, device=dev)                 # wire format of the hash gradient
                self.g16_mine = torch.zeros(self.ex.per, dtype=torch.bfloat16, device=dev)
            b, e = self.ex.begin, self.ex.end
            self.m = [torch.zeros(e - b, device=dev), torch.zeros_like(field.density_params), torch.zeros_like(field.color_params)]
            self.v = [torch.zeros(e - b, device=dev), torch.zeros_like(field.density_params), torch.zeros_like(field.color_params)]
            self.t16_pad = torch.zeros(pad, dtype=torch.float16, device=dev) if self.px is None else None   # all-gather target (padded copy of the fp16 table)
        else:
            self.m = [torch.zeros_like(p) for p in self.params]
            self.v = [torch.zeros_like(p) for p in self.params]
        self.step_n = 0
        # EMAHook(momentum=0.05) of the reference config (nerf_blender_local01.py:24), folded into the Adam pass; buffers start as copies (EMAHook.before_run)
        self.ema_momentum, self.ema_warm_up = ema_momentum, ema_warm_up
        if ema_momentum is not None:
            self.ema = [p.detach().clone() for p in self.params]
            if self.ex:
                self.ema[0] = field.hash_params.detach()[self.ex.begin:self.ex.end].clone()
        else:
            self.ema = [None] * 3
        cap = n_rays * samples_per_ray_budget
        self.slots = [_Slot(n_rays, cap, self.T, dev) for _ in range(2)]
        self.raw = torch.empty((self.T, 4), dtype=torch.float32, device=dev)
        self.draw = torch.zeros((self.T, 4), dtype=torch.float32, device=dev)
        self.rgb = torch.zeros((n_rays, 3), dtype=torch.float32, device=dev)
        self.grad_rgb = torch.zeros((n_rays, 3), dtype=torch.float32, device=dev)
        self.loss_accum = torch.zeros(1, dtype=torch.float32, device=dev)
        # depth / opacity supervision (step's target_depth / target_alpha): lambda_d sum |D - D*| + lambda_a sum (A - A*)^2 over the rays the compaction kept
        # whole, added to the 5 x Huber colour loss; the gradient reaches the field through the same loss_scale as the colour's (include/xrnerf_b200.h)
        self.depth_weight, self.opacity_weight = float(depth_weight), float(opacity_weight)
        if not (self.depth_weight >= 0.0 and self.opacity_weight >= 0.0):
            raise ValueError(f'depth_weight {depth_weight} / opacity_weight {opacity_weight}: must be >= 0')
        if self.depth_weight > 0.0 or self.opacity_weight > 0.0:
            self.alpha, self.depth, self.grad_alpha, self.grad_depth = (torch.zeros(n_rays, dtype=torch.float32, device=dev) for _ in range(4))
        # camera pose refinement (NgpRaySource.pose_step): step() also fills grad_rays_o / grad_rays_d [n_rays,3], the gradient of the loss it returns with
        # respect to the rays it was given (sample t held fixed; include/xrnerf_b200.h "NGP camera pose refinement")
        if self.ray_grad:
            self.d_rows = torch.zeros((self.T, 6), dtype=torch.float32, device=dev)
            self.grad_rays_o = torch.zeros((n_rays, 3), dtype=torch.float32, device=dev)
            self.grad_rays_d = torch.zeros((n_rays, 3), dtype=torch.float32, device=dev)
            self.inv_loss_scale = 1.0 / float(torch.tensor(128.0, dtype=torch.float32) / n_rays)   # the composite's fp32 128.f / n_rays, inverted
        self.grid_mean = torch.ones(1, dtype=torch.float32, device=dev)
        self.aux = torch.cuda.Stream(device=dev) if dev.type == 'cuda' else None
        self.trained_total = torch.zeros(1, dtype=torch.int64, device=dev)    # rays fully trained, summed over every batch prepared so far (device counter, no sync)
        self.march_calls = 0
        self.cur = 0
        self.master_stale = False

    # ------------------------------------------------------------------ march + compaction of one batch (aux stream)
    def _prepare(self, slot, rays_o, rays_d):
        from .ngp import _rays
        rays_o, rays_d = _rays(rays_o), _rays(rays_d)
        s = self.slots[slot]
        main = torch.cuda.current_stream()
        entry = torch.cuda.Event(); entry.record(main)
        with torch.cuda.stream(self.aux):
            self.aux.wait_event(entry)                 # the rays exist
            if s.free is not None:
                self.aux.wait_event(s.free)            # the step that last used this slot is done with it
            s.counter.zero_(); s.cnt_c.zero_()
            n = rays_o.shape[0]
            st = _C.stream()
            _C.check(_C.lib.xrb_rm_rays_sampler(_C.ptr(rays_o), _C.ptr(rays_d), _C.u8(self.bitfield), None, None, None, n, s.coords.shape[0], self.aabb[0], self.aabb[1], self.near,
                                                self.cone, 9121, self.march_calls, _C.ptr(s.coords), _C.ptr(s.rays_index), _C.ptr(s.numsteps), _C.ptr(s.counter), _C.ptr(s.ws_march), st),
                     'rays_sampler')
            self.march_calls += 1
            # the reference's no-grad pre-pass over ALL samples (ngp_grid_sampler.py:229-230) feeds only compacted_coord's dead transmittance loop
            # (compacted_coord.cu:41-44, SURVEY Q3): skipping it changes no result. Padding rows of coords_c are never read: every consumer takes the
            # compacted count from the device (cnt_c[1]).
            _C.check(_C.lib.xrb_rm_compacted_coord(None, _C.ptr(s.coords), _C.ptr(s.numsteps), n, self.T, _C.ptr(s.coords_c), _C.ptr(s.numsteps_c), _C.ptr(s.cnt_c[0:1]),
                                                   _C.ptr(s.cnt_c[1:2]), _C.ptr(s.ws_compact), st), 'compacted_coord')
            _C.check(_C.lib.xrb_ngp_count_trained_rays(_C.ptr(s.numsteps), _C.ptr(s.numsteps_c), n, _C.ptr(self.trained_total), st), 'count_trained_rays')
            s.ready = torch.cuda.Event(); s.ready.record(self.aux)
        s.rays = (rays_o, rays_d)                      # keep the tensors alive until the kernels ran

    # ------------------------------------------------------------------ one training step
    def step(self, rays_o, rays_d, target, bg, next_rays=None, target_depth=None, target_alpha=None):
        """Trains on (rays_o, rays_d, target, bg). next_rays = (rays_o, rays_d) of the FOLLOWING call (optional): their march starts now, on the aux
        stream, and overlaps this step's field kernels and gradient exchange. Returns the loss as a 0-dim device tensor (no sync).
        target_depth / target_alpha f32[n] or [n,1]: the depth (ray parameter t, e.g. NgpRaySource's target_depth; not finite or <= 0: no depth) and
        opacity each ray should render; used when depth_weight / opacity_weight > 0, and then the loss also holds their terms."""
        f = self.f
        s = self.slots[self.cur]
        if s.ready is None or s.rays is None or s.rays[0].data_ptr() != _ptr_of(rays_o):
            self._prepare(self.cur, rays_o, rays_d)
        if next_rays is not None:
            self._prepare(self.cur ^ 1, *next_rays)
        main = torch.cuda.current_stream()
        main.wait_event(s.ready)
        st = _C.stream()
        pts, dirs, n_rows_dev = s.coords_c[:, :3], s.coords_c[:, 4:], s.cnt_c[1:2]
        f.mlp_rows(pts, dirs, self.raw, n_rows_dev, self.fwd_impl)       # never refresh() here: the fp32 master outside this rank's slice is stale
        wd = self.depth_weight if target_depth is not None else 0.0
        wa = self.opacity_weight if target_alpha is not None else 0.0
        if wd > 0.0 or wa > 0.0:
            self._composite_geom(s, bg, target, target_depth if wd > 0.0 else None, target_alpha if wa > 0.0 else None, wd, wa, st)
        else:
            _C.check(_C.lib.xrb_rm_calc_rgb_forward(_C.ptr(self.raw), _C.ptr(s.coords_c), _C.ptr(s.numsteps), _C.ptr(s.numsteps_c), _C.f32(bg), self.n_rays, self.rgb_act,
                                                    self.dens_act, _C.ptr(self.rgb), st), 'calc_rgb_forward')
            self.loss_accum.zero_()
            _C.check(_C.lib.xrb_ngp_huber5_grad(_C.ptr(self.rgb), _C.f32(target), self.n_rays * 3, 0.1, _C.ptr(self.grad_rgb), _C.ptr(self.loss_accum), st), 'huber5')
            # rows of dL/draw beyond the compacted count are never read (n_rows_dev); rows owned by rays are all written by the kernel
            _C.check(_C.lib.xrb_rm_calc_rgb_backward(_C.ptr(self.raw), _C.ptr(s.numsteps_c), _C.ptr(s.coords_c), _C.ptr(self.grad_rgb), _C.ptr(self.rgb), _C.ptr(self.grid_mean),
                                                     self.n_rays, self.rgb_act, self.dens_act, _C.ptr(self.draw), st), 'calc_rgb_backward')
        self.gflat.zero_()
        if self.ray_grad:
            f.backward_rows(pts, dirs, self.draw, self.grads, n_rows_dev, self.bwd_impl, d_rows=self.d_rows)
            self._ray_grad(s, st)
        else:
            f.backward_rows(pts, dirs, self.draw, self.grads, n_rows_dev, self.bwd_impl)
        s.free = torch.cuda.Event(); s.free.record(main)
        self.step_n += 1
        it = self.step_n - 1                                                            # runner.iter inside after_train_iter
        mom = 0.0 if self.ema_momentum is None else min(self.ema_momentum, (1 + it) / (self.ema_warm_up + it))
        self._exchange_and_update(mom)
        f.shadows_updated()
        self.cur ^= 1
        return self.loss_accum[0]

    def _composite_geom(self, s, bg, target, target_depth, target_alpha, wd, wa, st):
        """composite forward with depth and alpha -> 5 x Huber -> depth / opacity loss (same loss_accum) -> composite backward with the geometry terms"""
        rays_o, rays_d = s.rays
        lo, hi = float(self.aabb[0]), float(self.aabb[1])
        _C.check(_C.lib.xrb_rm_calc_rgb_forward_geom(_C.ptr(self.raw), _C.ptr(s.coords_c), _C.ptr(s.numsteps), _C.ptr(s.numsteps_c), _C.f32(bg), _C.ptr(rays_o), _C.ptr(rays_d),
                                                     self.n_rays, lo, hi, self.rgb_act, self.dens_act, _C.ptr(self.rgb), _C.ptr(self.alpha), _C.ptr(self.depth), st),
                 'calc_rgb_forward_geom')
        self.loss_accum.zero_()
        _C.check(_C.lib.xrb_ngp_huber5_grad(_C.ptr(self.rgb), _C.f32(target), self.n_rays * 3, 0.1, _C.ptr(self.grad_rgb), _C.ptr(self.loss_accum), st), 'huber5')
        gd = self.grad_depth if wd > 0.0 else None
        ga = self.grad_alpha if wa > 0.0 else None
        _C.check(_C.lib.xrb_geom_loss_grad(_C.ptr(self.depth), _C.ptr(self.alpha), _ray_vec(target_depth, self.n_rays), _ray_vec(target_alpha, self.n_rays), _C.ptr(s.numsteps),
                                           _C.ptr(s.numsteps_c), self.n_rays, wd, wa, 0, _C.ptr(gd), _C.ptr(ga), _C.ptr(self.loss_accum), st), 'geom_loss_grad')
        _C.check(_C.lib.xrb_rm_calc_rgb_backward_geom(_C.ptr(self.raw), _C.ptr(s.numsteps_c), _C.ptr(s.coords_c), _C.ptr(self.grad_rgb), _C.ptr(self.rgb), _C.ptr(self.grid_mean),
                                                      _C.ptr(rays_o), _C.ptr(rays_d), lo, hi, _C.ptr(self.depth), _C.ptr(self.alpha), _C.ptr(gd), _C.ptr(ga), self.n_rays,
                                                      self.rgb_act, self.dens_act, _C.ptr(self.draw), st), 'calc_rgb_backward_geom')

    def _ray_grad(self, s, st):
        """d_rows -> grad_rays_o / grad_rays_d. dL/draw carries the composite's loss_scale = 128 / n_rays (calc_rgb.cu:92-93); its inverse restores the
        gradient of the loss step() returns (plus the composite's l1 / l2 regularisers, 0 unless rgb_act is exponential or the grid mean is below 0.01)"""
        rays_o, rays_d = s.rays
        _C.check(_C.lib.xrb_ngp_ray_grad(_C.ptr(self.d_rows), _C.ptr(s.coords_c), _C.ptr(s.numsteps_c), _C.ptr(rays_o), _C.ptr(rays_d), self.n_rays, float(self.aabb[0]),
                                         float(self.aabb[1]), self.inv_loss_scale, _C.ptr(self.grad_rays_o), _C.ptr(self.grad_rays_d), st), 'ngp_ray_grad')

    def _adam(self, p, p16, g, m, v, e, mom, div, bf16=False):
        fn = _C.lib.xrb_adam_ema_step_bf16grad if bf16 else _C.lib.xrb_adam_ema_step
        _C.check(fn(_C.ptr(p), _C.ptr(p16), _C.ptr(g), _C.ptr(m), _C.ptr(v), p.numel(), self.lr, self.betas[0], self.betas[1], self.eps, self.wd, self.step_n, div, _C.ptr(e), mom,
                    _C.stream()), 'adam')

    def close(self):
        """peer mode: give the field an ordinary fp16 table again (a copy of the working table) and release the exchange block and the mappings of the other ranks' blocks.
        Collective in effect: every rank must stop stepping before any rank closes (the others write into this block)."""
        if self.px is None:
            return
        torch.cuda.synchronize()
        if self.world > 1:
            import torch.distributed as dist
            dist.barrier(group=self.group)
        self.f.use_table(None)
        self.px.close()
        self.px = None
        self.grad_comm = 'closed'

    def _exchange_and_update(self, mom):
        import torch.distributed as dist
        f = self.f
        pairs = f.params_and_shadows()           # the MLPs' copies; the table's is the exchange block's in peer mode
        if self.grad_comm == 'peer':
            px, ex, C = self.px, self.ex, _C.C
            f.use_table(px.t16[:px.n_table])
            if px.step == 0:                 # first exchange: line the ranks up on the host once (lazy module loading / allocator warm-up differ by rank; the kernels give up after ~10 s)
                torch.cuda.synchronize()
                dist.barrier(group=self.group)
            px.step += 1
            st = _C.stream()
            _C.check(_C.lib.xrb_peer_publish_grads(C.byref(px.layout), _C.ptr(self.g_hash), _C.ptr(self.g_mlp), px.step, st), 'peer_publish_grads')
            groups = [_C.PeerMlpGroup(_C.ptr(p.data), _C.ptr(p16), _C.ptr(m), _C.ptr(v), _C.ptr(e), p.numel(), off)
                      for (p, p16), m, v, e, off in zip(pairs[1:], self.m[1:], self.v[1:], self.ema[1:], (0, f.density_params.numel()))]
            b, e_ = ex.begin, ex.end
            sl = f.hash_params.data[b:e_]
            _C.check(_C.lib.xrb_peer_adam_step(C.byref(px.layout), _C.ptr(sl) if e_ > b else None, _C.ptr(self.m[0]) if e_ > b else None, _C.ptr(self.v[0]) if e_ > b else None,
                                               _C.ptr(self.ema[0]) if (self.ema[0] is not None and e_ > b) else None, C.byref(groups[0]), C.byref(groups[1]), self.lr, self.betas[0],
                                               self.betas[1], self.eps, self.wd, self.step_n, mom if self.ema[0] is not None else 0.0, px.step, st), 'peer_adam_step')
            self.master_stale = True
            return
        if self.grad_comm == 'sharded':
            ex = self.ex
            _C.check(_C.lib.xrb_pack_bf16(_C.ptr(self.gflat[:ex.padded]), _C.ptr(self.g16), ex.padded, _C.stream()), 'pack_bf16')
            ex.reduce_scatter_sum(self.g16, self.g16_mine)
            dist.all_reduce(self.g_mlp, op=dist.ReduceOp.SUM, group=self.group)
            b, e = ex.begin, ex.end
            if e > b:
                self._adam(f.hash_params.data[b:e], self.t16_pad[b:e], self.g16_mine[:e - b], self.m[0], self.v[0], self.ema[0], mom, float(self.world), bf16=True)
            ex.all_gather(self.t16_pad, self.t16_pad[self.rank * ex.per:(self.rank + 1) * ex.per])
            pairs[0][1].copy_(self.t16_pad[:ex.n])
            self.master_stale = True
            for (p, p16), g_, m, v, e in zip(pairs[1:], self.grads[1:], self.m[1:], self.v[1:], self.ema[1:]):
                self._adam(p.data, p16, g_, m, v, e, mom, float(self.world))
            return
        div = 1.0
        if self.grad_comm == 'allreduce':
            dist.all_reduce(self.gflat, op=dist.ReduceOp.SUM, group=self.group)
            div = float(self.world)
        for (p, p16), g_, m, v, e in zip(pairs, self.grads, self.m, self.v, self.ema):
            self._adam(p.data, p16, g_, m, v, e, mom, div)

    # ------------------------------------------------------------------ bookkeeping
    def trained_rays(self, slot=None):
        """rays of the last step whose EVERY marched sample took part in the step (numsteps_c.count == numsteps.count): 0-dim device tensor. For tests and one-off queries
        (call it after a synchronize: the slot is re-marched by the aux stream two steps later); a training loop reads `trained_total`, which the aux stream keeps up to date."""
        s = self.slots[self.cur ^ 1 if slot is None else slot]
        return (s.numsteps_c[:, 0] == s.numsteps[:, 0]).sum()

    def compacted_samples(self, slot=None):
        return self.slots[self.cur ^ 1 if slot is None else slot].cnt_c[1]

    def sync_master(self):
        """sharded mode: fetch the other ranks' slices of the fp32 master table (and EMA) so that state_dict() / EMA swaps see whole tensors"""
        if self.grad_comm not in ('sharded', 'peer') or not self.master_stale:
            return
        ex, f = self.ex, self.f
        full = torch.zeros(ex.padded, dtype=torch.float32, device=self.dev)
        mine = torch.zeros(ex.per, dtype=torch.float32, device=self.dev)
        mine[:ex.end - ex.begin].copy_(f.hash_params.data[ex.begin:ex.end])
        ex.all_gather(full, mine)
        f.hash_params.data.copy_(full[:ex.n])
        self.master_stale = False

    def ema_full(self):
        """EMA of the hash table as one tensor (sharded mode gathers the slices)"""
        if self.ema[0] is None:
            return None
        if self.grad_comm not in ('sharded', 'peer'):
            return self.ema[0]
        ex = self.ex
        full = torch.zeros(ex.padded, dtype=torch.float32, device=self.dev)
        mine = torch.zeros(ex.per, dtype=torch.float32, device=self.dev)
        mine[:ex.end - ex.begin].copy_(self.ema[0])
        ex.all_gather(full, mine)
        return full[:ex.n]


def _ray_vec(t, n):
    """pointer of a per-ray f32 target ([n] or [n,1]); None -> NULL"""
    if t is None:
        return None
    if t.numel() != n:
        raise _C.XrbError(f'XRB_E_BADARG ({_C.XRB_E_BADARG}): expected {n} per-ray values, got shape {tuple(t.shape)}')
    _C.require_cuda(t)
    return _C.f32(t)


def _ptr_of(t):
    return t.data_ptr() if t.is_contiguous() else -1
