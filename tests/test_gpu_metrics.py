"""Image metrics on the device (xrnerf_b200.metrics, xrb_ssim): SSIM against a float64 numpy + scipy.ndimage.uniform_filter restatement of
scikit-image's structural_similarity (the computation the reference's hooks request), its exact identities, batch and run invariance, and the
ValidateHook / TestHook summaries on real val_step outputs against the hooks' own arithmetic on host copies."""
import ctypes as C
import json
from fractions import Fraction

import numpy as np
import pytest
import torch
from cases import NERF_MODEL, NGP_MODEL, dev
from scipy.ndimage import uniform_filter


# ------------------------------------------------------------------------------------------------ oracle

def ssim_map64(x, y, R):
    """skimage.metrics.structural_similarity(x, y, multichannel=True, data_range=R, full=True)[1], restated in float64: 7x7 uniform window,
    mode 'reflect', K1 0.01, K2 0.03, sample covariance"""
    x, y = np.asarray(x, np.float64), np.asarray(y, np.float64)
    C1, C2, cn = (0.01 * R) ** 2, (0.03 * R) ** 2, 49 / 48
    S = np.empty(x.shape)
    for c in range(x.shape[-1]):
        a, b = x[..., c], y[..., c]
        f = lambda t: uniform_filter(t, size=7, mode='reflect')                                          # noqa: E731
        ux, uy, uxx, uyy, uxy = f(a), f(b), f(a * a), f(b * b), f(a * b)
        vx, vy, vxy = cn * (uxx - ux * ux), cn * (uyy - uy * uy), cn * (uxy - ux * uy)
        S[..., c] = ((2 * ux * uy + C1) * (2 * vxy + C2)) / ((ux ** 2 + uy ** 2 + C1) * (vx + vy + C2))
    return S


def ssim_entry_exact(x, y, R, h, w, c):
    """S at one entry in exact rational arithmetic from the fp32 inputs (C1, C2 as the double values (0.01 R)^2, (0.03 R)^2), rounded once to
    float64. uniform_filter's running sums drift by a few double ulps along an 800-pixel line; where 2 vxy + C2 nearly cancels, that drift moves the
    oracle's S by more than one fp32 ulp, and this settles which of the two is right."""
    H, W = x.shape[:2]
    ref = lambda i, n: -i - 1 if i < 0 else (2 * n - i - 1 if i >= n else i)                             # noqa: E731
    win = [(ref(h + i, H), ref(w + j, W)) for i in range(-3, 4) for j in range(-3, 4)]
    a = [Fraction(float(x[p + (c,)])) for p in win]
    b = [Fraction(float(y[p + (c,)])) for p in win]
    ux, uy = sum(a) / 49, sum(b) / 49
    uxx, uyy, uxy = sum(t * t for t in a) / 49, sum(t * t for t in b) / 49, sum(s * t for s, t in zip(a, b)) / 49
    C1, C2, cn = Fraction((0.01 * R) ** 2), Fraction((0.03 * R) ** 2), Fraction(49, 48)
    vx, vy, vxy = cn * (uxx - ux * ux), cn * (uyy - uy * uy), cn * (uxy - ux * uy)
    return float(((2 * ux * uy + C1) * (2 * vxy + C2)) / ((ux * ux + uy * uy + C1) * (vx + vy + C2)))


def ulps32(got, want):
    """|got - want| in units of the fp32 spacing at want, with want rounded to fp32"""
    want32 = np.asarray(want).astype(np.float32)
    return np.abs(np.asarray(got, np.float64) - want32) / np.spacing(np.abs(want32))


def hook_scores(rgb, gt, R=2.0):
    """ValidateHook / TestHook on host copies (hooks/utils.py): numpy img2mse, mse2psnr, and calculate_ssim's full-map mean at the data_range R"""
    rgb, gt = rgb.cpu().numpy(), gt.cpu().numpy()
    mse = np.mean((rgb - gt) ** 2)
    psnr = -10. * np.log(mse) / np.log(np.array([10.]))
    return float(mse), float(psnr.item()), float(ssim_map64(rgb, gt, R).mean())


def pair(shape, correlated, seed):
    g = np.random.default_rng(seed)
    x = g.random(shape, dtype=np.float32)
    y = np.clip(x + g.normal(0, 0.1, shape).astype(np.float32), 0, 1) if correlated else g.random(shape, dtype=np.float32)
    return x, y.astype(np.float32)


# ------------------------------------------------------------------------------------------------ ssim

@pytest.mark.gpu
@pytest.mark.parametrize('shape', [(7, 7, 1), (8, 13, 3), (37, 53, 3), (64, 64, 4), (800, 800, 3)])
@pytest.mark.parametrize('R', [1.0, 2.0, 0.37])
@pytest.mark.parametrize('correlated', [True, False])
def test_ssim_matches_float64_oracle(shape, R, correlated):
    """every S entry within 1 fp32 ulp of the oracle rounded to fp32 or, at the few entries where the oracle's own drift exceeds that, of the exact
    value; both means within 1e-10 (double sums in another order). At 7x7 every entry's window reads reflected borders."""
    from xrnerf_b200 import metrics
    x, y = pair(shape, correlated, seed=hash((shape, R, correlated)) % 2 ** 32)
    s, ms, smap = metrics.ssim(dev(x), dev(y), R, full=True)
    assert s.dtype == ms.dtype == torch.float64 and s.shape == ms.shape == () and smap.shape == shape and smap.dtype == torch.float32
    ref = ssim_map64(x, y, R)
    got = smap.cpu().numpy()
    off = np.argwhere(ulps32(got, ref) > 1.0)
    assert len(off) <= 16, len(off)                                                                     # the oracle's drift matters at a handful of entries
    for e in map(tuple, off):
        assert ulps32(got[e], ssim_entry_exact(x, y, R, *e)) <= 1.0, (e, float(got[e]), ref[e], ssim_entry_exact(x, y, R, *e))
    assert abs(float(s) - ref.mean()) <= 1e-10
    assert abs(float(ms) - ref[3:-3, 3:-3].mean()) <= 1e-10


@pytest.mark.gpu
@pytest.mark.parametrize('shape', [(7, 7, 1), (37, 53, 3), (64, 64, 4)])
def test_ssim_identities_are_exact(shape):
    """S(x, x) = 1 in every entry and both means; S(x, y) = S(y, x) bit for bit"""
    from xrnerf_b200 import metrics
    x, y = (dev(a) for a in pair(shape, False, seed=3))
    s, ms, smap = metrics.ssim(x, x, 0.37, full=True)
    assert float(s) == 1.0 and float(ms) == 1.0 and bool((smap == 1.0).all())
    a, b = metrics.ssim(x, y, 2.0, full=True), metrics.ssim(y, x, 2.0, full=True)
    assert all(torch.equal(u, v) for u, v in zip(a, b))


@pytest.mark.gpu
def test_ssim_of_constant_images():
    """x = a, y = b everywhere: S = (2ab + C1) / (a^2 + b^2 + C1) (the variance terms are both C2)"""
    from xrnerf_b200 import metrics
    for a, b, R in [(0.25, 0.75, 1.0), (0.1, 0.9, 2.0), (0.5, 0.5, 0.37), (0.3, 0.0, 1.0)]:
        x = torch.full((9, 12, 3), a, device='cuda')
        y = torch.full((9, 12, 3), b, device='cuda')
        a64, b64 = float(np.float32(a)), float(np.float32(b))
        C1 = (0.01 * R) ** 2
        want = (2 * a64 * b64 + C1) / (a64 ** 2 + b64 ** 2 + C1)
        s, ms, smap = metrics.ssim(x, y, R, full=True)
        assert abs(float(s) - want) <= 1e-12 and abs(float(ms) - want) <= 1e-12
        assert float((smap.double() - want).abs().max()) <= 1e-7 * max(1.0, abs(want))


@pytest.mark.gpu
def test_ssim_batch_and_run_invariance():
    """image i of a batch of 5 is bit-identical to its single call, maps included; two runs are bit-identical; a strided view is scored as its copy"""
    from xrnerf_b200 import metrics
    g = np.random.default_rng(7)
    x = dev(g.random((5, 37, 53, 3), dtype=np.float32))
    y = dev(np.clip(x.cpu().numpy() + g.normal(0, 0.2, x.shape).astype(np.float32), 0, 1))
    s, ms, smap = metrics.ssim(x, y, 1.0, full=True)
    assert s.shape == ms.shape == (5,)
    for i in range(5):
        si, msi, mapi = metrics.ssim(x[i], y[i], 1.0, full=True)
        assert torch.equal(si, s[i]) and torch.equal(msi, ms[i]) and torch.equal(mapi, smap[i])
    again = metrics.ssim(x, y, 1.0, full=True)
    assert all(torch.equal(u, v) for u, v in zip(again, (s, ms, smap)))
    xt = x[1].transpose(0, 1).contiguous().transpose(0, 1)                                               # same values, strided
    assert not xt.is_contiguous()
    st = metrics.ssim(xt, y[1], 1.0, full=True)
    assert torch.equal(st[0], s[1]) and torch.equal(st[2], smap[1])
    assert torch.equal(metrics.ssim(x, y, 1.0)[0], s)                                                    # full=False: the same means


# ------------------------------------------------------------------------------------------------ hook summaries

def _nerf_val_output(H=24, W=40):
    from xrnerf_b200 import _C, registry as R, synth
    torch.manual_seed(11)
    net = R.build_network(NERF_MODEL).cuda()
    pose = synth.pose_spherical(30.0, -30.0, 4.0)
    c2w = (C.c_float * 12)(*[float(v) for v in pose[:3, :4].reshape(-1)])
    n, f = H * W, float(synth.FOCAL) * W / 800.0
    o, d, v = (torch.empty((n, 3), device='cuda') for _ in range(3))
    _C.check(_C.lib.xrb_nerf_get_rays(c2w, H, W, f, f, W / 2.0, H / 2.0, 0, None, n, _C.ptr(o), _C.ptr(d), _C.ptr(v), None, _C.stream()), 'get_rays')
    z = torch.empty((n, 64), device='cuda')
    _C.check(_C.lib.xrb_nerf_zvals(n, 64, 2.0, 6.0, 0, None, _C.ptr(z), _C.stream()), 'zvals')
    view = {'rays_o': o, 'rays_d': d, 'viewdirs': v, 'z_vals': z, 'pts': o[:, None] + d[:, None] * z[..., None], 'src_shape': torch.tensor([H, W, 3])}
    net.set_val_pipeline(lambda item: dict(view))
    images = torch.rand((1, 3, H, W, 3), device='cuda')
    return net.val_step({'poses': torch.zeros((1, 3, 4, 4)), 'images': images})


def _ngp_val_output(scene):
    from xrnerf_b200 import registry as R, synth
    torch.manual_seed(0)
    net = R.build_network(NGP_MODEL).cuda()
    n_img = scene['poses'].shape[0]
    net.sampler.set_data(dict(poses=scene['poses'], focal=np.full((n_img, 2), synth.FOCAL), aabb_scale=1, aabb_range=(0.0, 1.0), metadata=scene['metadata']), dict(H=800, W=800))
    net.sampler.density_grid_bitfield = dev(scene['bitfield'])
    t, d, c = synth.ngp_weights(seed=3, hash_range=0.5, mlp_gain=2.0)
    with torch.no_grad():
        net.mlp.field.hash_params.copy_(dev(t)); net.mlp.field.density_params.copy_(dev(d)); net.mlp.field.color_params.copy_(dev(c))
    data = {'rays_o': dev(scene['rays_o']), 'rays_d': dev(scene['rays_d']), 'img_ids': dev(scene['img_ids'].astype(np.float32)[:, None])}
    H = W = 64                                                                                           # the scene's 4096 rays
    net.set_val_pipeline(lambda item: dict(data, src_shape=torch.tensor([H, W, 3])))
    return net.val_step({'poses': torch.zeros((1, 2, 4, 3)), 'images': torch.rand((1, 2, H, W, 4), device='cuda')})


def _check_against_hook(out, got):
    want = [hook_scores(r, g) for r, g in zip(out['rgbs'], out['gt_imgs'])]
    assert set(got) == {'mse', 'psnr', 'ssim', 'average_mse', 'average_psnr', 'average_ssim'}
    assert len(got['mse']) == len(want) >= 2
    for i, (mse, psnr, s) in enumerate(want):
        assert got['mse'][i] == pytest.approx(mse, rel=4e-6) and got['psnr'][i] == pytest.approx(psnr, abs=1e-4)
        assert abs(got['ssim'][i] - s) <= 1e-10
    for k in ('mse', 'psnr', 'ssim'):
        assert got['average_' + k] == sum(got[k]) / len(got[k])
    assert got['psnr'] == out['psnr']                                                                     # val_step's own device PSNR: 3-channel gt_imgs


@pytest.mark.gpu
def test_validate_metrics_on_nerf_val_step():
    from xrnerf_b200.metrics import validate_metrics
    out = _nerf_val_output()
    _check_against_hook(out, validate_metrics(out))


@pytest.mark.gpu
def test_validate_metrics_on_ngp_val_step(scene):
    from xrnerf_b200.metrics import validate_metrics
    out = _ngp_val_output(scene)
    assert out['gt_imgs'][0].shape == (64, 64, 3)
    _check_against_hook(out, validate_metrics(out))


@pytest.mark.gpu
def test_validate_metrics_returns_none_where_the_hook_returns():
    from xrnerf_b200.metrics import validate_metrics
    x = torch.rand((16, 16, 3), device='cuda')
    assert validate_metrics({'rgbs': [], 'gt_imgs': []}) is None
    assert validate_metrics({'rgbs': [x, x], 'gt_imgs': [torch.rand((16, 16, 4), device='cuda'), x]}) is None
    assert validate_metrics({'rgbs': [x], 'gt_imgs': [x]})['ssim'] == [1.0]


@pytest.mark.gpu
def test_test_metrics_per_scale_averages():
    """TestMetrics(ndown=4) on 8 views of 64/32/16/8 pixels a side by scale (Mip-NeRF multiscale): per-scale averages and the hook's JSON dict"""
    from xrnerf_b200.metrics import TestMetrics
    g = np.random.default_rng(5)
    m = TestMetrics(ndown=4)
    want = {s: [] for s in range(4)}
    for idx in range(8):
        side = 64 >> (idx % 4)
        x, y = pair((side, side, 3), True, seed=100 + idx)
        y = np.clip(y + g.normal(0, 0.05, y.shape).astype(np.float32), 0, 1).astype(np.float32)
        rgb, gt = dev(x), dev(y)
        m.add({'rgb': rgb, 'gt_img': gt, 'idx': idx, 'disp': None})
        want[idx % 4].append(hook_scores(rgb, gt))
    got = m.summary()
    assert set(got) == {'average_mse', 'average_psnr', 'average_ssim', 'psnrs', 'ssims'}
    for s in range(4):
        assert got['average_mse'][s] == pytest.approx(np.mean([w[0] for w in want[s]]), rel=4e-6)
        assert got['average_psnr'][s] == pytest.approx(np.mean([w[1] for w in want[s]]), abs=1e-4)
        assert abs(got['average_ssim'][s] - np.mean([w[2] for w in want[s]])) <= 1e-10
        assert got['psnrs'][s] == pytest.approx([w[1] for w in want[s]], abs=1e-4)
        assert np.allclose(got['ssims'][s], [w[2] for w in want[s]], rtol=0, atol=1e-10)
    dumped = json.loads(json.dumps({'psnrs': got['psnrs'], 'ssims': got['ssims']}))
    assert set(dumped['psnrs']) == set(dumped['ssims']) == {'0', '1', '2', '3'} and all(len(v) == 2 for v in dumped['ssims'].values())
