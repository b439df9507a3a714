"""NeRF / Mip-NeRF inference through the fused renderers: NerfNetwork.batchify_forward(is_test=True) in ray batches of bounded size on the pipeline's
z values, depth from xrb_nerf_composite_forward_depth, and the networks' val_step / test_step / evaluate_once.
GPU tests compare the fused path with the reference-shaped chunk loop and with float64 restatements; the CPU tests check argument validation,
the batch-size arithmetic and the phase dispatch."""
import ctypes as C

import numpy as np
import pytest
import torch
from cases import FAR, MIP_CFG, MIP_MODEL, NEAR, NERF_MODEL, bits, nerf_net, view_rays, zvals

LEVEL_KEYS = ('rgb', 'disp', 'acc')


def _nerf_data(n, seed):
    """rays through an 800 x 800 Blender camera (the first n pixels of a view 800 wide), GetZvals(lindisp, NEAR, FAR, 64) and GetPts"""
    o, d, v, _ = view_rays(n // 800 + 1, 800, seed, radii=False)
    o, d, v = o[:n].contiguous(), d[:n].contiguous(), v[:n].contiguous()
    z = zvals(n, 64)
    return {'rays_o': o, 'rays_d': d, 'viewdirs': v, 'z_vals': z, 'pts': o[:, None] + d[:, None] * z[..., None]}


def _mip_data(n, seed):
    """as _nerf_data with GetZvals(129) and per-ray radii spread over 0.5x..2x the camera's"""
    o, d, v, r = view_rays(n // 800 + 3, 800, seed)                             # the radii take a pixel's neighbours: H >= 3
    g = torch.Generator(device='cuda').manual_seed(seed)
    r = r[:n] * (0.5 + 1.5 * torch.rand((n, 1), device='cuda', generator=g))
    return {'rays_o': o[:n].contiguous(), 'rays_d': d[:n].contiguous(), 'viewdirs': v[:n].contiguous(), 'radii': r.contiguous(), 'z_vals': zvals(n, 129)}


# ------------------------------------------------------------------------------------------------ fused == chunked

@pytest.mark.gpu
@pytest.mark.parametrize('ray_batch', [None, 384])
def test_nerf_fused_batchify_matches_chunked(ray_batch):
    """NeRF 64 + 128 on lindisp z values over [0.5, 3]: the fused path equals the reference-shaped chunk loop within the renderer tolerances
    (coarse 2e-3, fine 5e-3). 1000 rays: not a multiple of either batch size. Rendering on linspace(2, 6) instead fails the tolerance."""
    net = nerf_net(False)
    net.fused_ray_batch = ray_batch
    data = _nerf_data(1000, 1)
    with torch.no_grad():
        got = net.batchify_forward(dict(data), is_test=True)
        net.fused_inference = False
        ref = net.batchify_forward(dict(data), is_test=True)
        from xrnerf_b200.nerf import NerfRenderer
        lin = NerfRenderer(net).render(data['rays_o'], data['rays_d'], data['viewdirs'])
    assert set(ref) == {'coarse_' + k for k in LEVEL_KEYS} | set(LEVEL_KEYS)
    assert set(got) == set(ref) | {'depth', 'coarse_depth'}
    assert got['depth'].shape == (1000, 1) and got['rgb'].shape == (1000, 3) and got['disp'].shape == got['acc'].shape == (1000,)
    assert (got['coarse_rgb'] - ref['coarse_rgb']).abs().max().item() <= 2e-3
    assert (got['rgb'] - ref['rgb']).abs().max().item() <= 5e-3
    assert (got['coarse_acc'] - ref['coarse_acc']).abs().max().item() <= 2e-3
    assert (lin['coarse_rgb'] - ref['coarse_rgb']).abs().max().item() > 2e-3      # ignoring the pipeline's z values would fail the tolerance


@pytest.mark.gpu
@pytest.mark.parametrize('ray_batch', [None, 384])
def test_mip_fused_batchify_matches_chunked(ray_batch):
    """Mip-NeRF 2 x 128 with per-ray radii on lindisp z values over [0.5, 3]: fused == chunk loop within 1e-2 on rgb and acc of both levels."""
    net = nerf_net(True, seed=5)
    net.fused_ray_batch = ray_batch
    data = _mip_data(1000, 2)
    with torch.no_grad():
        got = net.batchify_forward(dict(data), is_test=True)
        net.fused_inference = False
        ref = net.batchify_forward(dict(data), is_test=True)
        from xrnerf_b200.nerf import MipNerfRenderer
        lin = MipNerfRenderer(net).render(data['rays_o'], data['rays_d'], data['viewdirs'], data['radii'])
    assert set(got) == set(ref) | {'depth', 'coarse_depth'}
    for k in ('rgb', 'coarse_rgb', 'acc', 'coarse_acc'):
        assert (got[k] - ref[k]).abs().max().item() <= 1e-2, k
    assert max((lin[k] - ref[k]).abs().max().item() for k in ('coarse_rgb', 'coarse_acc')) > 1e-2      # ignoring the pipeline's z values would fail


# ------------------------------------------------------------------------------------------------ batch split

@pytest.mark.gpu
@pytest.mark.parametrize('mip', [False, True])
def test_batch_split_is_invisible(mip):
    """one batch and batches of 200 and 333 rays (1000 rays) give bit-identical rgb, disp, acc and depth on every level"""
    from xrnerf_b200.nerf import NerfRenderer, MipNerfRenderer
    net = nerf_net(mip, seed=7)
    data = _mip_data(1000, 3) if mip else _nerf_data(1000, 3)
    outs = []
    for batch in (None, 200, 333):
        if mip:
            outs.append(MipNerfRenderer(net, ray_batch=batch).render(data['rays_o'], data['rays_d'], data['viewdirs'], data['radii'], z_vals=data['z_vals'], depth=True))
        else:
            outs.append(NerfRenderer(net, ray_batch=batch).render(data['rays_o'], data['rays_d'], data['viewdirs'], z_vals=data['z_vals'], depth=True))
    assert set(outs[0]) == {p + k for p in ('', 'coarse_') for k in LEVEL_KEYS + ('depth',)}
    for other in outs[1:]:
        for k, v in outs[0].items():
            assert torch.equal(bits(v), bits(other[k])), k


# ------------------------------------------------------------------------------------------------ depth

def _composite(raw, z, d, mip, depth, white=True, pad=0.001, bias=-1.0, act=4):
    from xrnerf_b200 import _C
    n, s = raw.shape[0], raw.shape[1]
    out = [torch.full(sh, float('nan'), device='cuda') for sh in ((n, 3), (n,), (n,), (n, s))]
    args = [_C.ptr(raw), _C.ptr(z), _C.ptr(d), n, s, int(mip), int(white), pad, bias, act] + [_C.ptr(t) for t in out]
    if depth:
        dep = torch.full((n,), float('nan'), device='cuda')
        _C.check(_C.lib.xrb_nerf_composite_forward_depth(*args, _C.ptr(dep), _C.stream()))
        return out + [dep]
    _C.check(_C.lib.xrb_nerf_composite_forward(*args, _C.stream()))
    return out


def _nerf_disp(depth, acc):
    """nerf_render.py:32-36 in fp32: 1 / max(1e-10, depth / acc), NaN propagated"""
    return 1.0 / torch.clamp(depth / acc, min=1e-10)


def _mip_disp(depth, acc, z0, zl):
    """mipnerf_render.py:18-24 in fp32: clamp(nan_to_num(depth / acc, inf), z_0, z_last)"""
    q = torch.nan_to_num(depth / acc, nan=float('inf'), posinf=float('inf'))
    return torch.maximum(torch.minimum(q, zl), z0)


def _same_bits_or_nan(a, b):
    na, nb = torch.isnan(a), torch.isnan(b)
    return torch.equal(na, nb) and torch.equal(bits(torch.where(na, 0.0, a)), bits(torch.where(nb, 0.0, b)))


@pytest.mark.gpu
@pytest.mark.parametrize('mip', [False, True])
@pytest.mark.parametrize('s', [1, 64, 129])
def test_composite_depth_entry(mip, s):
    """xrb_nerf_composite_forward_depth: rgb, disp, acc and weights bit-identical to xrb_nerf_composite_forward; depth = sum w z (mid-points when mip)
    within the fp32 summation bound gamma_(s+2) * sum |w z| of a float64 restatement on the kernel's own weights; disp = the reference formula on
    depth and acc, bit for bit, NaN where acc == 0 (rays whose densities are all zero)."""
    n = 333
    g = torch.Generator(device='cuda').manual_seed(s + 100 * mip)
    raw = torch.randn((n, s, 4), device='cuda', generator=g) * 3
    act = 4 if mip else 1
    raw[:40, :, 3] = -50.0                                                  # relu: density 0, acc 0; softplus(-51) is 7e-23
    z = (0.5 + 3 * torch.rand((n, s + int(mip)), device='cuda', generator=g)).sort(dim=-1).values.contiguous()
    d = torch.randn((n, 3), device='cuda', generator=g)
    for white in (False, True):
        base = _composite(raw, z, d, mip, False, white=white, act=act)
        rgb, disp, acc, w, depth = _composite(raw, z, d, mip, True, white=white, act=act)
        for a, b in zip(base, (rgb, disp, acc, w)):
            assert _same_bits_or_nan(a, b)
        zz = z.double()
        zm = 0.5 * (zz[:, :-1] + zz[:, 1:]) if mip else zz
        ref = (w.double() * zm).sum(1)
        gamma = (s + 2) * 2.0 ** -24 / (1 - (s + 2) * 2.0 ** -24)
        assert ((depth.double() - ref).abs() <= gamma * (w.double() * zm).abs().sum(1)).all()
        want = _mip_disp(depth, acc, z[:, 0], z[:, -1]) if mip else _nerf_disp(depth, acc)
        assert _same_bits_or_nan(disp, want)
        if not mip:
            assert torch.isnan(disp[:40]).all() and (acc[:40] == 0).all()


@pytest.mark.gpu
@pytest.mark.parametrize('mip', [False, True])
def test_renderer_disp_is_the_reference_formula_on_depth(mip):
    """the fused renderers' disp equals, bit for bit, the reference formula in fp32 on the returned depth and acc: both NeRF levels, and Mip-NeRF's first
    level (whose z_0 / z_last are the given z values); depth=False leaves the other outputs bit-identical"""
    from xrnerf_b200.nerf import NerfRenderer, MipNerfRenderer
    net = nerf_net(mip, seed=9)
    data = _mip_data(700, 4) if mip else _nerf_data(700, 4)
    if mip:
        run = lambda dep: MipNerfRenderer(net).render(data['rays_o'], data['rays_d'], data['viewdirs'], data['radii'], z_vals=data['z_vals'], depth=dep)
    else:
        run = lambda dep: NerfRenderer(net).render(data['rays_o'], data['rays_d'], data['viewdirs'], z_vals=data['z_vals'], depth=dep)
    off, on = run(False), run(True)
    assert set(on) == set(off) | {'depth', 'coarse_depth'}
    for k, v in off.items():
        assert _same_bits_or_nan(v, on[k]), k
    z = data['z_vals']
    if mip:
        assert _same_bits_or_nan(on['coarse_disp'], _mip_disp(on['coarse_depth'][:, 0], on['coarse_acc'], z[:, 0], z[:, -1]))
    else:
        for p in ('', 'coarse_'):
            assert _same_bits_or_nan(on[p + 'disp'], _nerf_disp(on[p + 'depth'][:, 0], on[p + 'acc'])), p
    lo, hi = float(z.min()), float(z.max())
    for p in ('', 'coarse_'):
        dep, acc = on[p + 'depth'][:, 0], on[p + 'acc']
        assert (dep >= 0).all() and (dep <= hi * acc * (1 + 1e-5) + 1e-6).all() and (dep >= lo * acc * (1 - 1e-5) - 1e-6).all()


# ------------------------------------------------------------------------------------------------ API

@pytest.mark.gpu
def test_nerf_val_and_test_steps():
    """val_step: the reference's keys plus psnr, [H,W,3] / [H,W,1] device tensors for the validation and spiral poses; phase 'test' -> test_step
    (rgb, gt_img, disp, idx). fused_inference = False keeps the reference's keys in batchify_forward."""
    H, W = 24, 40
    net = nerf_net(False, seed=11)
    o, d, v, _ = view_rays(H, W, 5, radii=False)
    z = zvals(H * W, 64)
    d_view = {'rays_o': o, 'rays_d': d, 'viewdirs': v, 'z_vals': z, 'pts': o[:, None] + d[:, None] * z[..., None], 'src_shape': torch.tensor([H, W, 3])}
    seen = []
    net.set_val_pipeline(lambda item: (seen.append(item['pose'].shape), dict(d_view))[1])
    images = torch.rand((1, 2, H, W, 3), device='cuda')
    out = net.val_step({'poses': torch.zeros((1, 2, 4, 4)), 'images': images, 'spiral_poses': torch.zeros((1, 3, 4, 4))})
    assert set(out) == {'rgbs', 'disps', 'gt_imgs', 'spiral_rgbs', 'spiral_disps', 'elapsed_time', 'psnr'}
    assert len(out['rgbs']) == len(out['disps']) == len(out['gt_imgs']) == len(out['elapsed_time']) == len(out['psnr']) == 2
    assert len(out['spiral_rgbs']) == len(out['spiral_disps']) == 3 and seen == [(4, 4)] * 5
    for rgb, disp in zip(out['rgbs'] + out['spiral_rgbs'], out['disps'] + out['spiral_disps']):
        assert rgb.shape == (H, W, 3) and disp.shape == (H, W, 1) and rgb.is_cuda and disp.is_cuda
    assert torch.equal(out['gt_imgs'][1], images[0, 1]) and all(t > 0 for t in out['elapsed_time'])
    with torch.no_grad():
        ret = net.batchify_forward(dict(d_view), is_test=True)
    mse = ((ret['rgb'].reshape(H, W, 3) - images[0, 0]) ** 2).mean()
    assert abs(out['psnr'][0] - float(-10 * torch.log10(mse))) <= 1e-4
    assert torch.equal(out['rgbs'][0], ret['rgb'].reshape(H, W, 3))
    net.phase = 'test'
    t = net.val_step({'pose': torch.zeros((1, 4, 4)), 'image': images[:, 0], 'idx': torch.tensor([3])})
    assert set(t) == {'rgb', 'gt_img', 'disp', 'idx'} and t['idx'] == 3
    assert t['rgb'].shape == (H, W, 3) and t['disp'].shape == (H, W, 1) and torch.equal(t['gt_img'], images[0, 0])
    net.fused_inference = False
    with torch.no_grad():
        ref = net.batchify_forward(dict(d_view), is_test=True)
    assert set(ref) == {'coarse_' + k for k in LEVEL_KEYS} | set(LEVEL_KEYS)


@pytest.mark.gpu
def test_mip_multiscale_evaluate_once():
    """use_multiscale: a pixel-shaped view (per-pixel radii) is flattened and rendered through the fused path; validation returns one-element lists,
    phase 'test' the evaluate_once keys. Without use_multiscale val_step is NerfNetwork's."""
    H, W = 20, 36
    net = nerf_net(True, seed=13, use_multiscale=True)
    o, d, v, r = view_rays(H, W, 6)
    z = zvals(H * W, 129)
    image = torch.rand((1, H, W, 3), device='cuda')
    px = lambda t: t.reshape(1, H, W, -1)
    data = {'rays_o': px(o), 'rays_d': px(d), 'viewdirs': px(v), 'radii': px(r), 'z_vals': px(z), 'lossmult': torch.ones((1, H, W, 1), device='cuda'),
            'near': torch.full((1, H, W, 1), NEAR, device='cuda'), 'far': torch.full((1, H, W, 1), FAR, device='cuda'), 'image': image, 'idx': torch.tensor([[5]])}
    with torch.no_grad():
        ref = net.batchify_forward({'rays_o': o, 'rays_d': d, 'viewdirs': v, 'radii': r, 'z_vals': z}, is_test=True)
    val = net.val_step(dict(data))
    assert set(val) == {'rgbs', 'gt_imgs', 'disps'} and all(len(x) == 1 for x in val.values())
    assert val['rgbs'][0].shape == (H, W, 3) and val['disps'][0].shape == (H, W, 1) and torch.equal(val['gt_imgs'][0], image[0])
    assert torch.equal(val['rgbs'][0], ref['rgb'].reshape(H, W, 3)) and 'depth' in ref
    net.phase = 'test'
    t = net.val_step(dict(data))
    assert set(t) == {'rgb', 'gt_img', 'disp', 'idx'} and t['idx'] == 5 and torch.equal(t['disp'], ref['disp'].reshape(H, W, 1))
    net.use_multiscale, net.phase = False, 'train'
    net.set_val_pipeline(lambda item: {'rays_o': o, 'rays_d': d, 'viewdirs': v, 'radii': r, 'z_vals': z, 'src_shape': torch.tensor([H, W, 3])})
    out = net.val_step({'poses': torch.zeros((1, 1, 4, 4)), 'images': image[None]})
    assert out['rgbs'][0].shape == (H, W, 3) and out['disps'][0].shape == (H, W, 1) and len(out['psnr']) == 1


# ------------------------------------------------------------------------------------------------ whole view

@pytest.mark.gpu
def test_whole_view_renders_in_bounded_memory():
    """a whole 800 x 800 view (640 000 rays) through NerfNetwork.val_step: the peak allocation beyond the view's inputs stays under the bound the
    renderer states (ray_batch_size * bytes_per_ray + one encoding tile), plus the two levels' outputs, the PSNR's temporaries and a repack of both MLPs"""
    from xrnerf_b200.nerf import bytes_per_ray, ray_batch_size
    H = W = 800
    n = H * W
    net = nerf_net(False, seed=17)
    o, d, v, _ = view_rays(H, W, 8, radii=False)
    view = {'rays_o': o, 'rays_d': d, 'viewdirs': v, 'z_vals': zvals(n, 64, 2.0, 6.0, False), 'src_shape': torch.tensor([H, W, 3])}
    net.set_val_pipeline(lambda item: dict(view))
    image = torch.rand((1, 1, H, W, 3), device='cuda')
    net.val_step({'poses': torch.zeros((1, 1, 4, 4)), 'images': image})        # packs the weights once
    torch.cuda.synchronize()
    base = torch.cuda.memory_allocated()
    torch.cuda.reset_peak_memory_stats()
    out = net.val_step({'poses': torch.zeros((1, 1, 4, 4)), 'images': image})
    torch.cuda.synchronize()
    peak = torch.cuda.max_memory_allocated() - base
    rows = [64, 192]
    bound = ray_batch_size(rows, 63) * bytes_per_ray(rows, 63) + 128 * 256 + n * 2 * 24 + 3 * n * 12 + (16 << 20)
    assert peak <= bound, (peak, bound)
    assert out['rgbs'][0].shape == (H, W, 3) and np.isfinite(out['psnr'][0])
    assert torch.isfinite(out['rgbs'][0]).all()


# ------------------------------------------------------------------------------------------------ CPU

def test_composite_depth_entry_validates_arguments_without_gpu():
    from xrnerf_b200 import _C
    lib = _C.lib
    buf = (C.c_char * 4096)()
    p = C.c_void_p((C.addressof(buf) + 255) & ~255)                     # 256-byte aligned host memory: never dereferenced by a rejected call
    f = C.c_float
    call = lambda n, s, act, raw, depth: lib.xrb_nerf_composite_forward_depth(raw, p, p, n, s, 0, 1, f(0), f(0), act, p, p, p, p, depth, None)
    assert call(4, 8, 1, p, None) == _C.XRB_E_BADARG and b'null' in lib.xrb_last_error()      # every other pointer is set: the missing depth is refused
    assert call(0, 8, 1, p, None) == 0                                                       # an empty batch is a no-op
    assert call(-1, 8, 1, p, p) == _C.XRB_E_BADARG and b'bad size' in lib.xrb_last_error()
    assert call(4, 0, 1, p, p) == _C.XRB_E_BADARG and b'bad size' in lib.xrb_last_error()
    assert call(4, 8, 2, p, p) == -2                                                         # XRB_E_UNSUPPORTED: relu(1) or softplus(4) only
    assert call(4, 8, 1, C.c_void_p(p.value + 4), p) == _C.XRB_E_BADARG and b'aligned' in lib.xrb_last_error()
    assert call(4, 8, 1, None, p) == _C.XRB_E_BADARG and b'null' in lib.xrb_last_error()


def test_ray_batch_size_without_gpu():
    from xrnerf_b200.nerf import RAY_BATCH_BYTES, bytes_per_ray, ray_batch_size
    assert bytes_per_ray([64, 192], 63) == 192 * 256 + (64 + 192) * 24 + 8 == 55304
    assert bytes_per_ray([128, 128], 96) == 128 * 384 + 2 * 128 * 24 + 8 == 55304
    b = ray_batch_size([64, 192], 63)
    assert b == 38784 and b % 128 == 0 and b * 55304 <= RAY_BATCH_BYTES < (b + 128) * 55304
    assert ray_batch_size([64, 192], 63, budget=1000) == 128


class _Stub:
    """stands in for batchify_forward on the CPU: records the rays it is given, returns fixed per-ray outputs"""

    def __init__(self):
        self.calls = []

    def __call__(self, data, is_test=False):
        self.calls.append((data, is_test))
        n = data['rays_o'].shape[0]
        return {'rgb': torch.full((n, 3), 0.25), 'disp': torch.full((n,), 2.0), 'acc': torch.ones(n)}


def test_test_phase_dispatch_without_gpu():
    """NerfNetwork: phase 'test' sends val_step to test_step, which renders data['pose'] through the val pipeline (this raised KeyError('poses') before);
    MipNerfNetwork with use_multiscale flattens a pixel-shaped view (per-pixel radii included) to rays in evaluate_once."""
    from xrnerf_b200 import registry as R
    H, W = 3, 5
    net = R.build_network(dict(NERF_MODEL, cfg=dict(NERF_MODEL['cfg'], phase='test')))
    net.batchify_forward = stub = _Stub()
    seen = []
    net.set_val_pipeline(lambda item: (seen.append(item), {'rays_o': torch.zeros((H * W, 3)), 'src_shape': torch.tensor([H, W, 3])})[1])
    image = torch.rand((1, H, W, 3))
    out = net.val_step({'pose': torch.eye(4)[None], 'image': image, 'idx': torch.tensor([7])})
    assert set(out) == {'rgb', 'gt_img', 'disp', 'idx'} and out['idx'] == 7 and torch.equal(out['gt_img'], image[0])
    assert out['rgb'].shape == (H, W, 3) and out['disp'].shape == (H, W, 1) and stub.calls[0][1] is True
    assert torch.equal(seen[0]['pose'], torch.eye(4)) and seen[0]['idx'] == 7
    mip = R.build_network(dict(MIP_MODEL, cfg=dict(MIP_CFG, use_multiscale=True)))
    mip.batchify_forward = stub = _Stub()
    px = lambda c: torch.rand((1, H, W, c))
    data = {'rays_o': px(3), 'rays_d': px(3), 'viewdirs': px(3), 'radii': px(1), 'z_vals': px(129), 'image': image, 'idx': torch.tensor([[2]])}
    val = mip.val_step(dict(data))
    assert set(val) == {'rgbs', 'gt_imgs', 'disps'} and val['rgbs'][0].shape == (H, W, 3) and val['disps'][0].shape == (H, W, 1)
    rays = stub.calls[0][0]
    assert rays['radii'].shape == (H * W, 1) and rays['z_vals'].shape == (H * W, 129) and torch.equal(rays['radii'][:, 0], data['radii'].reshape(-1))
    mip.phase = 'test'
    t = mip.val_step(dict(data))
    assert set(t) == {'rgb', 'gt_img', 'disp', 'idx'} and t['idx'] == 2 and torch.equal(t['gt_img'], image[0])
