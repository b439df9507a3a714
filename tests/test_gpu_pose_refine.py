"""NGP camera pose refinement on the H100 (include/xrnerf_b200.h, "NGP camera pose refinement"): the field's input gradient, the per-ray and per-image
reductions against float64, the trainer's ray gradients and launch sequence, and that refinement recovers perturbed poses.

Rounding bounds. The field's input gradients pass through the fp16 staging of dZ at every layer: with R stagings on the way, each entry errs by at most
tau = (R + 1) 2^-11 times its absolute chain, the floor of restate64_pose.FLOOR added at every staged value (as in test_gpu_field_grad_exact; the +1 covers
fp32 accumulation). position_grad_level and sh4_grad add fp32 sums of at most 16 x 8 and 16 terms of a few products each: 64 U32 times their absolute
chain. The reductions are fp32 sums of K terms of a few products: gamma(K + 16, U32) times the sum of absolute terms.
"""
import math

import numpy as np
import pytest
import torch

from cases import dev, load_ngp_weights
from restate64 import U16, U32, Grid, gamma, hashgrid_enc16, ngp_mats, position_grad
from restate64_pose import field_masks, input_grads, ngp_rays64, ray_grad64, sh4_jacobian

pytestmark = pytest.mark.gpu


def _field(dh, ch):
    from xrnerf_b200 import synth
    from xrnerf_b200.ngp import NgpField
    f = load_ngp_weights(NgpField(density_hidden=dh, color_hidden=ch, n_packed_levels=6).cuda(),
                         synth.ngp_weights(seed=10 * dh + ch + 500, dens_hidden=dh, color_hidden=ch, hash_range=0.5))
    f.refresh()
    return f


def _sh16(dirs_d):
    from xrnerf_b200 import _C
    n = dirs_d.shape[0]
    sh = torch.empty((n, 16), dtype=torch.float16, device='cuda')
    dp, ds = _C.rows(dirs_d)
    _C.check(_C.lib.xrb_tcnn_sh4_forward(dp, ds, n, _C.ptr(sh), _C.stream()))
    return sh.cpu().numpy().astype(np.float64)


def _tau(dh, ch):
    return (dh + 1 + ch + 1 + 1) * U16


class InputCase:
    """float64 d_rows of a batch (stable rows only; unstable rows get dL/draw = 0) with its bound"""

    def __init__(self, f, pts, dirs, draw, pts_d=None, dirs_d=None):
        dh, ch = f.cfg.density_hidden, f.cfg.color_hidden
        pts_d = dev(pts) if pts_d is None else pts_d
        dirs_d = dev(dirs) if dirs_d is None else dirs_d
        dm, cm = ngp_mats(f._dens16.cpu().numpy(), dh), ngp_mats(f._color16.cpu().numpy(), ch)
        dmasks, cmasks, self.stable = field_masks(dm, cm, hashgrid_enc16(f, pts_d), _sh16(dirs_d))
        self.draw = draw.copy()
        self.draw[~self.stable] = 0.0
        genc, gcin, agenc, agcin = input_grads(dm, cm, dmasks, cmasks, self.draw.astype(np.float64), self.stable)
        gx, mx = position_grad(Grid.of(f), pts, genc, agenc)
        J = sh4_jacobian(dirs)
        gw = np.einsum('nk,nka->na', gcin[:, 15:31], J)
        mw = np.einsum('nk,nka->na', agcin[:, 15:31], np.abs(J))
        self.ref = np.concatenate([gx, gw], 1)
        self.bound = (_tau(dh, ch) + 64 * U32) * np.concatenate([mx, mw], 1)
        self.genc_mass = agenc

    def check(self, got, name):
        got = np.asarray(got, np.float64)
        err = np.abs(got - self.ref)
        assert np.isfinite(got).all(), name
        ratio = np.divide(err, self.bound, out=np.where(err > 0, np.inf, 0.0), where=self.bound > 0)
        k = np.unravel_index(int(np.argmax(ratio)), ratio.shape)
        assert ratio[k] <= 1.0, (name, k, float(ratio[k]), float(got[k]), float(self.ref[k]))
        assert self.stable.mean() >= 1 / 3, (name, float(self.stable.mean()))
        assert (np.abs(self.ref[self.stable]) > 0).mean() > 0.9, name       # not vacuous
        print(f'{name}: n={len(got)} stable={self.stable.mean():.3f} max err/bound={float(ratio[k]):.3f}')


def _batch(n, seed):
    rng = np.random.default_rng(seed)
    return rng.random((n, 3)).astype(np.float32), rng.random((n, 3)).astype(np.float32), (rng.normal(0, 1, (n, 4)) * 1e-3).astype(np.float32)


def _zeros(f):
    return torch.zeros_like(f.hash_params), torch.zeros_like(f.density_params), torch.zeros_like(f.color_params)


def _inputs(f, pts_d, dirs_d, draw_d, n_rows_dev=None, rows=None):
    rows = pts_d.shape[0] if rows is None else rows
    d_rows = torch.full((rows, 6), float('nan'), device='cuda')
    out = f.backward_rows(pts_d, dirs_d, draw_d, _zeros(f), n_rows_dev, impl=1, d_rows=d_rows)
    torch.cuda.synchronize()
    return d_rows, out


# ------------------------------------------------------------------------------------------------ field input gradient
@pytest.mark.parametrize('shape', [(1, 1), (1, 2)])
@pytest.mark.parametrize('n', [1, 129, 20001])
def test_field_input_grad_matches_f64(shape, n):
    """every entry of d_rows (dL/dx through position_grad, dL/dw through the SH derivative) within the derived bound, (1,1) and (1,2), ragged row counts"""
    f = _field(*shape)
    pts, dirs, draw = _batch(n, seed=n + 7)
    case = InputCase(f, pts, dirs, draw)
    d_rows, _ = _inputs(f, dev(pts), dev(dirs), dev(case.draw))
    if n == 1:
        got = np.asarray(d_rows.cpu().numpy(), np.float64)
        assert np.isfinite(got).all() and (case.bound.sum() == 0 or np.all(np.abs(got - case.ref) <= case.bound))
        return
    case.check(d_rows.cpu().numpy(), f'd_rows {shape} n={n}')


@pytest.mark.parametrize('count', [700, 0, 1100])
def test_field_input_grad_device_row_count_and_strided_rows(count):
    """n_rows_dev and the stride-7 coords views the trainer passes: the first min(n, count) rows are written, the others are never touched"""
    f = _field(1, 2)
    n = 1000
    n_eff = min(n, count)
    pts, dirs, draw = _batch(n, seed=31)
    coords = np.random.default_rng(32).random((n, 7)).astype(np.float32)
    coords[:, :3] = pts; coords[:, 4:] = dirs
    cd = dev(coords)
    case = InputCase(f, pts[:n_eff], dirs[:n_eff], draw[:n_eff]) if n_eff else None
    draw_k = draw.copy()
    if n_eff:
        draw_k[:n_eff] = case.draw
    d_rows, _ = _inputs(f, cd[:, :3], cd[:, 4:], dev(draw_k), torch.tensor([count], dtype=torch.int32, device='cuda'))
    got = d_rows.cpu().numpy()
    assert np.isnan(got[n_eff:]).all()
    if n_eff:
        case.check(got[:n_eff], f'd_rows n_rows_dev={count} strided')


@pytest.mark.parametrize('shape', [(1, 1), (1, 2)])
def test_field_input_grad_parameter_gradients_unchanged(shape):
    """the INPUTS kernel accumulates the parameter gradients of xrb_ngp_mlp_backward_tc: the difference is within the spread of two runs of the latter
    (both add the same per-sample terms with atomics in arrival order)"""
    f = _field(*shape)
    pts, dirs, draw = (dev(a) for a in _batch(40001, seed=3))
    a = f.backward_rows(pts, dirs, draw, _zeros(f), impl=1)
    b = f.backward_rows(pts, dirs, draw, _zeros(f), impl=1)
    _, c = _inputs(f, pts, dirs, draw)
    tiles = (40001 + 127) // 128
    for name, x, y, z in zip(('table', 'density', 'color'), a, b, c):
        spread = float((x - y).abs().max())
        scale = float(x.abs().max())
        assert scale > 0
        # a weight-gradient entry is the sum of one partial per tile, added with atomics in arrival order: reordering those additions moves it by at most
        # tiles x 2^-24 x the largest partial sum, taken here as the largest entry
        assert float((z - x).abs().max()) <= max(2 * spread, tiles * 2.0 ** -24 * scale), (name, float((z - x).abs().max()), spread, scale)


def test_field_input_grad_is_the_density_gradient():
    """at dL/draw = (0, 0, 0, 1) dL/dx is xrb_ngp_density_grad_tc's gradient (same masks; stagings at 2^12 and 2^10 differ by a power of two), and dL/dw is 0"""
    f = _field(1, 2)
    n = 20000
    pts, dirs, _ = _batch(n, seed=11)
    draw = np.zeros((n, 4), np.float32); draw[:, 3] = 1.0
    pd = dev(pts)
    d_rows, _ = _inputs(f, pd, dev(dirs), dev(draw))
    _, g = f.density_grad_tc(pd, density=False)
    case = InputCase(f, pts, dirs, draw)
    got, want = d_rows[:, :3].cpu().numpy().astype(np.float64), g.cpu().numpy().astype(np.float64)
    bound = 2 * case.bound[:, :3]
    s = case.stable
    assert np.all(np.abs(got[s] - want[s]) <= bound[s])
    assert float(d_rows[:, 3:].abs().max()) == 0.0
    print(f'density gradient: max |d_rows - density_grad_tc| = {float(np.abs(got - want).max()):.3e} (max |g| {float(np.abs(want).max()):.3e})')


# ------------------------------------------------------------------------------------------------ ray and pose reductions
def _march_rows(n_rays, seed, lo=0.0, hi=1.0):
    """rays, compacted rows (positions on the rays, count 0..40, the rows in ray order) and random d_rows"""
    rng = np.random.default_rng(seed)
    o = (rng.random((n_rays, 3)) * 2 - 0.5).astype(np.float32)
    d = rng.normal(size=(n_rays, 3)); d = (d / np.linalg.norm(d, axis=1, keepdims=True)).astype(np.float32)
    cnt = rng.integers(0, 41, n_rays); cnt[::7] = 0
    base = np.concatenate([[0], np.cumsum(cnt)[:-1]])
    rows = int(cnt.sum())
    coords = rng.random((rows, 7)).astype(np.float32)
    for r in range(n_rays):
        t = np.sort(rng.random(cnt[r])) * 1.5 + 0.05
        coords[base[r]:base[r] + cnt[r], :3] = ((o[r] + t[:, None] * d[r] - lo) / (hi - lo)).astype(np.float32)
    d_rows = rng.normal(size=(rows, 6)).astype(np.float32)
    return o, d, np.stack([cnt, base], 1).astype(np.int32), coords, d_rows


@pytest.mark.parametrize('aabb', [(0.0, 1.0), (-1.5, 2.5)])
def test_ray_grad_matches_f64(aabb):
    from xrnerf_b200 import _C
    n = 3000
    o, d, ns, coords, d_rows = _march_rows(n, seed=5, lo=aabb[0], hi=aabb[1])
    go, gd = torch.full((n, 3), float('nan'), device='cuda'), torch.full((n, 3), float('nan'), device='cuda')
    scale = 0.37
    ins = [dev(a) for a in (d_rows, coords, ns, o, d)]          # held until the kernel has run: a pointer of a freed temporary may be reused by the next
    _C.check(_C.lib.xrb_ngp_ray_grad(*(_C.ptr(a) for a in ins), n, aabb[0], aabb[1], scale, _C.ptr(go), _C.ptr(gd), _C.stream()))
    torch.cuda.synchronize()
    ro, rd, mo, md = ray_grad64(d_rows, coords, ns, o, d, aabb[0], aabb[1], scale)
    K = int(ns[:, 0].max())
    for got, ref, m in ((go, ro, mo), (gd, rd, md)):
        got = got.cpu().numpy().astype(np.float64)
        assert np.all(np.abs(got - ref) <= gamma(2 * K + 32, U32) * m + 1e-30)
    assert float(go[torch.from_numpy(ns[:, 0] == 0).cuda()].abs().max()) == 0.0


@pytest.mark.parametrize('I', [1, 3, 1100])
def test_pose_grad_matches_f64_autograd(I):
    """dL/dP' against float64 autograd of the ray generation, for I = 1, 3 and 1100 (I x 12 floats beyond 48 KB: the warp-aggregated global path)"""
    from xrnerf_b200 import _C
    H, W, fx, fy, cx, cy = 12, 10, 9.0, 8.5, 5.2, 6.1
    g = torch.Generator().manual_seed(I)
    n = 6000
    rot = torch.linalg.qr(torch.randn(I, 3, 3, generator=g, dtype=torch.float64))[0]
    poses = torch.cat([rot.transpose(1, 2), torch.randn(I, 1, 3, generator=g, dtype=torch.float64)], 1).float()
    row_idx = torch.randint(0, I * H * W, (n,), generator=g)
    go, gd = torch.randn(n, 3, generator=g), torch.randn(n, 3, generator=g)
    out = torch.zeros((I, 4, 3), device='cuda')
    ri, pc, goc, gdc = row_idx.cuda(), poses.cuda(), go.cuda(), gd.cuda()
    _C.check(_C.lib.xrb_ngp_pose_grad(_C.ptr(ri), n, _C.ptr(pc), I, H, W, fx, fy, cx, cy, _C.ptr(goc), _C.ptr(gdc), _C.ptr(out), _C.stream()))
    torch.cuda.synchronize()
    P = poses.double().requires_grad_(True)
    o, dh = ngp_rays64(P, row_idx, H, W, fx, fy, cx, cy)
    ((o * go.double()).sum() + (dh * gd.double()).sum()).backward()
    ref = P.grad.numpy()
    # mass: per ray |grad_o| on row 3, (|g| + |d^| |d^ . g|_abs) / |d~| |(x, y, 1)| on rows 0..2
    with torch.no_grad():
        img = row_idx // (H * W); pix = row_idx % (H * W)
        x = ((pix % W).double() + 0.5 - cx) / fx; y = ((pix // W).double() + 0.5 - cy) / fy
        Pd = poses.double()[img]
        dt = x[:, None] * Pd[:, 0] + y[:, None] * Pd[:, 1] + Pd[:, 2]
        nr = dt.norm(dim=1, keepdim=True); u = dt / nr
        gmag = (gd.double().abs() + u.abs() * (u.abs() * gd.double().abs()).sum(1, keepdim=True)) / nr
        inp = torch.stack([x.abs(), y.abs(), torch.ones_like(x)], 1)
        mass = torch.zeros(I, 4, 3, dtype=torch.float64)
        mass.index_add_(0, img, torch.cat([inp[:, :, None] * gmag[:, None, :], go.double().abs()[:, None, :]], 1))
        count = torch.bincount(img, minlength=I).max().item()
    got = out.cpu().numpy().astype(np.float64)
    bound = gamma(count + 32, U32) * mass.numpy()
    assert np.all(np.abs(got - ref) <= bound), float((np.abs(got - ref) / np.maximum(bound, 1e-300)).max())


# ------------------------------------------------------------------------------------------------ trainer
class _Launches:
    """the ordered device work a block of code issues, recorded where it is issued (deterministic, unlike a profiler trace, whose activity buffers can
    drop records): every entry point of the CUDA library called through xrnerf_b200._C.lib (each launches a fixed kernel sequence for its arguments),
    and every aten operator on CUDA tensors (torch's own kernels: the zero_ / copy_ of the step)"""

    def __init__(self, monkeypatch):
        from torch.utils._python_dispatch import TorchDispatchMode
        from xrnerf_b200 import _C
        self.names, self.on = [], False
        rec = self

        class Lib:
            def __getattr__(self, name):
                fn = getattr(real, name)
                if not name.startswith('xrb_') or name == 'xrb_last_error':
                    return fn

                def call(*a):
                    if rec.on:
                        rec.names.append(name)
                    return fn(*a)
                return call

        class Ops(TorchDispatchMode):
            def __torch_dispatch__(self, func, types, args=(), kwargs=None):
                out = func(*args, **(kwargs or {}))
                if rec.on and any(torch.is_tensor(t) and t.is_cuda for t in list(args) + [out] if torch.is_tensor(t)):
                    rec.names.append(str(func.overloadpacket))
                return out
        real = _C.lib
        monkeypatch.setattr(_C, 'lib', Lib())
        self.mode = Ops()

    def __enter__(self):
        self.on = True
        self.mode.__enter__()
        return self

    def __exit__(self, *exc):
        self.mode.__exit__(*exc)
        self.on = False


def _trainer_run(scene, steps=3, launches=None, **kw):
    from xrnerf_b200.ngp import NgpField
    from xrnerf_b200.train import NgpTrainer
    n = 4096
    o, d, bf = dev(scene['rays_o']), dev(scene['rays_d']), dev(scene['bitfield'])
    target = torch.full((n, 3), 0.5, device='cuda'); bg = torch.zeros((n, 3), device='cuda')
    f = NgpField(seed=5).cuda()
    tr = NgpTrainer(f, bf, n, target_batch_size=1 << 16, **kw)
    names = []
    if launches is not None:
        launches.names = names = []
        with launches:
            for _ in range(steps):
                tr.step(o, d, target, bg)
    else:
        for _ in range(steps):
            tr.step(o, d, target, bg)
    torch.cuda.synchronize()
    return tr, names


def test_trainer_flags_off_is_todays_step(scene, monkeypatch):
    """ray_grad=False issues what a trainer built without the flag issues, over 3 steps (library entry points and torch operators, in order), none of it
    the new entry points; ray_grad=True issues the same list with the field backward replaced by its input-gradient entry followed by the per-ray
    reduction"""
    rec = _Launches(monkeypatch)
    _, today = _trainer_run(scene, launches=rec)
    _, off = _trainer_run(scene, launches=rec, ray_grad=False)
    _, on = _trainer_run(scene, launches=rec, ray_grad=True)
    assert today.count('xrb_ngp_mlp_backward_tc') == 3 and today.count('xrb_ngp_mlp_forward') == 3 and len(today) > 30
    assert off == today
    assert not any(k in ('xrb_ngp_mlp_backward_tc_inputs', 'xrb_ngp_ray_grad', 'xrb_ngp_pose_grad') for k in today)
    expect = []
    for k in today:
        expect += ['xrb_ngp_mlp_backward_tc_inputs', 'xrb_ngp_ray_grad'] if k == 'xrb_ngp_mlp_backward_tc' else [k]
    assert on == expect


def test_trainer_ray_grad_is_the_chain(scene):
    """grad_rays_o / grad_rays_d equal xrb_ngp_ray_grad of the trainer's own d_rows with 1 / loss_scale, and are non-zero where rays have compacted rows"""
    from xrnerf_b200 import _C
    tr, _ = _trainer_run(scene, steps=1, ray_grad=True)
    s = tr.slots[tr.cur ^ 1]
    n_c = int(s.cnt_c[1])
    ro, rd = (t.cpu().numpy() for t in s.rays)
    go, gd, mo, md = ray_grad64(tr.d_rows[:n_c].cpu().numpy(), s.coords_c[:n_c].cpu().numpy(), s.numsteps_c.cpu().numpy(), ro, rd, 0.0, 1.0, tr.inv_loss_scale)
    K = int(s.numsteps_c[:, 0].max())
    for got, ref, m in ((tr.grad_rays_o, go, mo), (tr.grad_rays_d, gd, md)):
        got = got.cpu().numpy().astype(np.float64)
        assert np.all(np.abs(got - ref) <= gamma(2 * K + 32, U32) * m + 1e-30)
    hit = s.numsteps_c[:, 0].cpu().numpy() > 0
    assert hit.mean() > 0.3 and (np.abs(tr.grad_rays_d.cpu().numpy()[hit]).sum(1) > 0).mean() > 0.9
    assert _C.lib.xrb_abi_version() == 5


def test_ray_source_flags_off_keeps_todays_keys():
    from xrnerf_b200.data import NgpRaySource
    poses = torch.eye(4)[:, :3][None].repeat(2, 1, 1)
    src = NgpRaySource(poses, torch.rand(2, 4, 5, 4), [[4.0, 0, 2.5], [0, 4.0, 2.0], [0, 0, 1]]).cuda()
    assert set(src.next_batch(8)) == {'rays_o', 'rays_d', 'target_s', 'alpha', 'img_ids', 'bg_color'}
    ref = NgpRaySource(poses, src.images.cpu(), [[4.0, 0, 2.5], [0, 4.0, 2.0], [0, 0, 1]], refine_poses=True).cuda()
    rows = torch.arange(40, device='cuda')
    a, b = src.rows(rows, u_bg=torch.zeros(40, 3)), ref.rows(rows, u_bg=torch.zeros(40, 3))
    assert set(b) == set(a) | {'row_idx', 'pose_xi'}
    assert torch.equal(a['rays_o'], b['rays_o']) and torch.equal(a['rays_d'], b['rays_d'])     # xi = 0: Exp(0) = I exactly


# ------------------------------------------------------------------------------------------------ refinement converges
RING_RADIUS = 0.75   # camera distance from the sphere's centre: close enough that parallax tells a shift of the centre from a rotation


def _ring_poses(k, radius=1.1, height=0.35, c=0.5):
    """k NGP xforms on a ring around (c, c, c), each looking at it (camera z forward)"""
    out = []
    for i in range(k):
        a = 2 * math.pi * i / k
        o = np.array([c + radius * math.cos(a), c + radius * math.sin(a), c + height])
        z = np.array([c, c, c]) - o; z /= np.linalg.norm(z)
        x = np.cross(z, [0.0, 0.0, 1.0]); x /= np.linalg.norm(x)
        y = np.cross(z, x)
        out.append(np.stack([x, y, z, o]))
    return np.array(out, np.float32)


def _textured_sphere():
    """cases.sphere_network with a texture: level 4's feature 1 holds sin waves of the position, routed through density output 1 into the colour net
    (colour input 0 -> two hidden units +/- -> the three outputs with different gains), so colour varies over the sphere and rotation is observable"""
    from cases import sphere_network
    net, grid = sphere_network()
    f = net.mlp.field
    l, r = 4, int(grid.res[4])
    i = np.arange(r)
    z, y, x = np.meshgrid(i, i, i, indexing='ij')
    pos = (np.stack([x, y, z], -1).astype(np.float64) - 0.5) / float(grid.scale[l])
    tex = 0.5 * np.sin(2 * np.pi * 4 * pos[..., 0]) * np.cos(2 * np.pi * 3 * pos[..., 1]) + 0.5 * np.sin(2 * np.pi * 5 * pos[..., 2])
    with torch.no_grad():
        t = f.hash_params.detach().cpu().numpy().copy()
        t[2 * grid.off[l] + 1:2 * (grid.off[l] + r ** 3):2] = tex.reshape(-1).astype(np.float16).astype(np.float32)
        f.hash_params.copy_(torch.from_numpy(t))
        dp = f.density_params.detach().cpu().numpy().copy()
        dp[64 * 32 + 0] *= 100.0; dp[64 * 32 + 1] *= 100.0              # opaque sphere (as the depth-supervision test)
        dp[2 * 32 + 9], dp[3 * 32 + 9] = 1.0, -1.0                        # hidden units 2, 3 = +/- feature 1 of level 4
        dp[64 * 32 + 64 + 2], dp[64 * 32 + 64 + 3] = 1.0, -1.0            # density output 1 = the texture
        f.density_params.copy_(torch.from_numpy(dp))
        cp = np.zeros(f.color_params.numel(), np.float32)
        cp[0 * 32 + 0], cp[1 * 32 + 0] = 1.0, -1.0                        # colour input 0 = density output 1
        o = 64 * 32
        for _ in range(f.cfg.color_hidden - 1):
            cp[o + 0 * 64 + 0], cp[o + 1 * 64 + 1] = 1.0, 1.0
            o += 64 * 64
        for c, gain in enumerate((3.0, -2.0, 1.5)):
            cp[o + c * 64 + 0], cp[o + c * 64 + 1] = gain, -gain
        f.color_params.copy_(torch.from_numpy(cp))
    f.mark_dirty()
    return f


def _rot_err(Pa, Pb):
    """mean angle (degrees) between the rotations of two sets of xforms, and the mean centre distance"""
    Ra, Rb = Pa[:, :3].double(), Pb[:, :3].double()
    c = ((torch.einsum('nij,nij->n', Ra, Rb) - 1) / 2).clamp(-1, 1)
    return float(torch.rad2deg(torch.arccos(c)).mean()), float((Pa[:, 3] - Pb[:, 3]).double().norm(dim=1).mean())


def refine(radius, steps=300, lr=None, trace=()):
    """8 ring views at `radius` from the centre of a textured opaque sphere rendered from the true poses; the poses perturbed by 1-2 degrees about a random
    axis and 0.01 in the centre; `steps` steps of field lr 0 + pose_step -> (rotation error deg, centre error) before and after"""
    from xrnerf_b200.data import POSE_LR, NgpRaySource, corrected_poses
    from xrnerf_b200.ngp import NgpRenderer
    from xrnerf_b200.train import NgpTrainer
    teacher = _textured_sphere()
    true = torch.from_numpy(_ring_poses(8, radius=radius))
    Hh = Ww = 64
    K = [[70.0, 0, Ww / 2], [0, 70.0, Hh / 2], [0, 0, 1]]
    ones = torch.full((128 ** 3 * 8 // 8,), 255, dtype=torch.uint8, device='cuda')
    gt = NgpRaySource(true, torch.zeros(8, Hh, Ww, 4), K).cuda()
    b = gt.rows(torch.arange(8 * Hh * Ww, device='cuda'), u_bg=torch.zeros(8 * Hh * Ww, 3))
    rgb, alpha, _, _ = NgpRenderer(teacher, samples_per_ray_budget=1024).render(b['rays_o'], b['rays_d'], ones)
    assert 0.2 < float((alpha > 0.5).float().mean()) < 0.9
    images = torch.cat([rgb, torch.ones_like(rgb[:, :1])], 1).reshape(8, Hh, Ww, 4)
    g = torch.Generator().manual_seed(0)
    axis = torch.randn(8, 3, generator=g); axis /= axis.norm(dim=1, keepdim=True)
    ang = torch.deg2rad(1.0 + torch.rand(8, 1, generator=g))
    shift = torch.randn(8, 3, generator=g); shift *= 0.01 / shift.norm(dim=1, keepdim=True)
    noisy = corrected_poses(true, torch.cat([axis * ang, shift], 1))
    src = NgpRaySource(noisy, images.cpu(), K, refine_poses=True).cuda()
    n = 4096
    tr = NgpTrainer(teacher, ones, n, target_batch_size=1 << 22, samples_per_ray_budget=1024, lr=0.0, ray_grad=True)
    zero_bg = torch.zeros((n, 3), device='cuda')
    r0, c0 = _rot_err(src.refined_poses().cpu(), true)
    for it in range(steps):
        batch = src.next_batch(n)
        tr.step(batch['rays_o'], batch['rays_d'], batch['target_s'], zero_bg)
        src.pose_step(batch, tr.grad_rays_o, tr.grad_rays_d, lr=POSE_LR if lr is None else lr)
        if it + 1 in trace:
            print(it + 1, _rot_err(src.refined_poses().cpu(), true))
    torch.cuda.synchronize()
    r1, c1 = _rot_err(src.refined_poses().cpu(), true)
    return r0, r1, c0, c1


def test_pose_refinement_recovers_perturbed_poses():
    """refine(): at the default learning rate the mean rotation and centre errors both fall at least 5x within 300 steps"""
    r0, r1, c0, c1 = refine(RING_RADIUS)
    print(f'pose refinement: mean rotation error {r0:.3f} -> {r1:.3f} deg, mean centre error {c0:.4f} -> {c1:.4f}')
    assert r1 * 5 <= r0 and c1 * 5 <= c0
