"""Depth from both NGP render paths (xrb_ngp_render_depth: march -> field -> composite chain; xrb_ngp_render_fused_depth: the single-launch
kernel) and the disparity maps HashNerfNetwork's validation and test steps return.

depth = sum_k T_k alpha_k t_k (not divided by alpha); disparity = 1 / max(1e-10, depth / alpha) where alpha > 0, 0 where alpha == 0.
GPU tests compare against a float64 restatement over the oracle's march and field; the CPU tests check argument validation."""
import ctypes as C

import numpy as np
import pytest
import torch
from cases import NGP_MODEL, cpu_args, dev

BG = (0.1, 0.5, 0.9)
# unwarp_dt (common.cuh): the fp32 constants of the march, evaluated in float64
MIN_DT = float(np.float32(np.float32(1.73205080757) / np.float32(1024)))
MAX_DT = MIN_DT * 128


@pytest.fixture(scope='module')
def setup():
    from xrnerf_b200 import synth
    from xrnerf_b200.ngp import NgpField
    f = NgpField().cuda()
    table, dens, color = synth.ngp_weights(seed=3, hash_range=0.5, mlp_gain=2.0)
    with torch.no_grad():
        f.hash_params.copy_(dev(table)); f.density_params.copy_(dev(dens)); f.color_params.copy_(dev(color))
    return f, table, dens, color


def sample_t(coords, ns, o, d, lo=0.0, hi=1.0):
    """float64 t of every marched row, rebuilt from its warped position: ((lo + x * (hi - lo)) - o) . d / (d . d); and each row's ray"""
    ray = np.repeat(np.arange(ns.shape[0]), ns[:, 0])
    rows = np.concatenate([np.arange(b, b + c) for c, b in ns]) if len(ray) else np.zeros(0, np.int64)
    o64, d64 = o.astype(np.float64)[ray], d.astype(np.float64)[ray]
    p = lo + coords[rows, :3].astype(np.float64) * (hi - lo)
    return ((p - o64) * d64).sum(1) / (d64 * d64).sum(1), rows, ray


def depth64(port, scene, table, dens, color, o, d, n_prior):
    """float64 depth of every ray over the oracle's march and fp32 field (exp density, as NgpRenderer's default dens_act 3); plus the largest t of
    the batch and each ray's first / last sample t"""
    c, _, ns, cnt = port.rays_sampler(o, d, scene['bitfield'], o.shape[0] * 64, n_prior_calls=n_prior)
    t, rows, ray = sample_t(c, ns, o, d)
    coords = c[rows]
    raw = port.ngp_mlp_forward(table, dens, color, np.ascontiguousarray(coords[:, :3]), np.ascontiguousarray(coords[:, 4:])).astype(np.float64)
    dt = coords[:, 3].astype(np.float64) * (MAX_DT - MIN_DT) + MIN_DT
    alpha = 1.0 - np.exp(-np.exp(raw[:, 3]) * dt)
    depth = np.zeros(o.shape[0])
    start = np.concatenate([[0], np.cumsum(ns[:, 0])])
    for i in np.nonzero(ns[:, 0])[0]:
        a = alpha[start[i]:start[i + 1]]
        T = np.concatenate([[1.0], np.cumprod(1.0 - a)[:-1]])
        depth[i] = (T * a * t[start[i]:start[i + 1]]).sum()
    return depth, ns[:, 0], t.max(), first_last_t(t, ns[:, 0])


def first_last_t(t, counts):
    start = np.concatenate([[0], np.cumsum(counts)])[:-1]
    has = counts > 0
    first, last = np.full(counts.shape, np.nan), np.full(counts.shape, np.nan)
    first[has], last[has] = t[start[has]], t[start[has] + counts[has] - 1]
    return first, last


def both(r, o, d, bf, path):
    """(rgb, alpha, counts) without depth, then (rgb, alpha, counts, depth) with depth, from the same RNG call index"""
    n = o.shape[0]
    calls = r.calls
    fn = r.render_fused if path == 'fused' else r.render
    a = [x.clone() for x in fn(o, d, bf)]
    r.calls = calls
    depth = torch.full((n, 1), -1.0, device='cuda')
    b = [x.clone() for x in fn(o, d, bf, depth=depth)]
    return a, b, depth


# ------------------------------------------------------------------------------------------------ GPU

@pytest.mark.gpu
@pytest.mark.parametrize('path', ['chain', 'fused'])
def test_depth_changes_nothing_else(scene, setup, path):
    """rgb, alpha and sample counts (chain: numsteps and counters) with depth are bit-identical to those without, on the 4096-ray batch, a whole
    800x800 view and an all-ones occupancy grid (several 64-sample march rounds per ray in the single-launch kernel)"""
    from xrnerf_b200 import synth
    from xrnerf_b200.ngp import NgpRenderer
    f = setup[0]
    bf = dev(scene['bitfield'])
    vo, vd = synth.get_rays_ngp(scene['poses'][7])
    n = 2048
    cases = [(dev(scene['rays_o']), dev(scene['rays_d']), bf, 64), (dev(vo), dev(vd), bf, 48),
             (dev(vo[:n * 300:300]), dev(vd[:n * 300:300]), torch.full_like(bf, 255), 1024)]
    for o, d, b, budget in cases:
        r = NgpRenderer(f, bg=BG, samples_per_ray_budget=budget)
        for _ in range(2):
            a, got, depth = both(r, o, d, b, path)
            assert all(torch.equal(x, y) for x, y in zip(a, got))
            assert torch.isfinite(depth).all() and (depth >= 0).all()


@pytest.mark.gpu
def test_depth_matches_float64_restatement(port, scene, setup):
    """both paths within 2e-3 x (largest t of the batch) of the float64 depth (the rgb tolerance scaled by t: the error comes from the fp16 field), and within
    5e-5 of each other; two consecutive calls, so that the advanced RNG stream is covered"""
    from xrnerf_b200.ngp import NgpRenderer
    f, table, dens, color = setup
    o, d = scene['rays_o'], scene['rays_d']
    rc, rf = NgpRenderer(f, bg=BG), NgpRenderer(f, bg=BG)
    n = o.shape[0]
    for call in range(2):
        dc, df = torch.empty(n, device='cuda'), torch.empty(n, device='cuda')
        _, _, ns_c, _ = rc.render(dev(o), dev(d), dev(scene['bitfield']), depth=dc)
        _, _, ns_f = rf.render_fused(dev(o), dev(d), dev(scene['bitfield']), depth=df)
        ref, counts, t_max, _ = depth64(port, scene, table, dens, color, o, d, call)
        assert np.array_equal(ns_c[:, 0].cpu().numpy(), counts) and np.array_equal(ns_f.cpu().numpy(), counts)
        assert ref.max() > 0.2 * t_max                                  # the scene is visible: depth is not trivially small
        assert np.abs(dc.cpu().numpy() - ref).max() <= 2e-3 * t_max
        assert np.abs(df.cpu().numpy() - ref).max() <= 2e-3 * t_max
        assert (dc - df).abs().max().item() <= 5e-5


@pytest.mark.gpu
@pytest.mark.parametrize('path', ['chain', 'fused'])
def test_depth_and_disparity_properties(port, scene, setup, path):
    """rays without samples: depth == 0 and disp == 0 exactly; where alpha > 1e-4, depth / alpha lies within [first t, last t] of the ray's samples;
    on the 4096-ray batch and on a whole 800x800 view. Slack: 1e-5, plus what fp32 allows: alpha = 1 - T and the sum of the weights in depth may
    differ by a few roundings of a value near 1 per sample (count * 2^-22 here; the scans round more often than a sequential product), which
    depth / alpha magnifies by last t / alpha."""
    from xrnerf_b200 import synth
    from xrnerf_b200.ngp import NgpRenderer, disparity
    f = setup[0]
    vo, vd = synth.get_rays_ngp(scene['poses'][21])
    for o, d, budget in ((scene['rays_o'], scene['rays_d'], 64), (vo, vd, 48)):
        r = NgpRenderer(f, bg=BG, samples_per_ray_budget=budget)
        n = o.shape[0]
        depth = torch.empty((n, 1), device='cuda')
        fn = r.render_fused if path == 'fused' else r.render
        alpha = fn(dev(o), dev(d), dev(scene['bitfield']), depth=depth)[1]
        disp = disparity(depth, alpha)
        c, _, ns, _ = port.rays_sampler(o, d, scene['bitfield'], n * budget)
        t, _, _ = sample_t(c, ns, o, d)
        first, last = first_last_t(t, ns[:, 0])
        depth, alpha, disp = depth.cpu().numpy()[:, 0], alpha.cpu().numpy()[:, 0], disp.cpu().numpy()[:, 0]
        miss = ns[:, 0] == 0
        assert miss.any() and (~miss).any()
        assert (depth[miss] == 0).all() and (disp[miss] == 0).all() and (alpha[miss] == 0).all()
        assert np.isfinite(disp).all() and (disp >= 0).all()
        hit = alpha > 1e-4
        assert hit.sum() > 100
        mean_t = depth[hit].astype(np.float64) / alpha[hit]
        slack = 1e-5 + last[hit] * ns[hit, 0] * 2.0 ** -22 / alpha[hit]
        assert (mean_t >= first[hit] - slack).all() and (mean_t <= last[hit] + slack).all()


@pytest.mark.gpu
@pytest.mark.parametrize('n', [1, 31, 33, 1000])
def test_fused_depth_ragged_sizes(scene, setup, n):
    from xrnerf_b200.ngp import NgpRenderer
    f = setup[0]
    o, d, bf = dev(scene['rays_o'][:n]), dev(scene['rays_d'][:n]), dev(scene['bitfield'])
    a, b = NgpRenderer(f, bg=(1.0, 1.0, 1.0)), NgpRenderer(f, bg=(1.0, 1.0, 1.0))
    df, dc = torch.empty(n, device='cuda'), torch.empty(n, device='cuda')
    ns = a.render_fused(o, d, bf, depth=df)[2]
    ns_u = b.render(o, d, bf, depth=dc)[2]
    assert torch.equal(ns, ns_u[:, 0]) and (df - dc).abs().max().item() <= 5e-5


@pytest.mark.gpu
def test_renderer_rejects_bad_depth_tensor(scene, setup):
    from xrnerf_b200 import _C
    from xrnerf_b200.ngp import NgpRenderer
    r = NgpRenderer(setup[0])
    o, d, bf = dev(scene['rays_o'][:64]), dev(scene['rays_d'][:64]), dev(scene['bitfield'])
    for bad in (torch.empty(64, dtype=torch.float64, device='cuda'), torch.empty(65, device='cuda'), torch.empty(64), torch.empty((64, 2), device='cuda')[:, 0]):
        for fn in (r.render, r.render_fused):
            with pytest.raises(_C.XrbError):
                fn(o, d, bf, depth=bad)
    assert r.calls == 0                                                  # refused before anything ran


@pytest.mark.gpu
def test_hashnerf_network_returns_disparity(scene):
    """batchify_forward(is_test=True) returns depth / disp [n,1]; val_step one finite [H,W,1] map per pose in `disps`; test_step `spiral_disp` [H,W,1].
    The reference-shaped path (fused_inference = False) keeps the reference's keys: `disps` stays empty."""
    from xrnerf_b200 import registry as R, synth
    from xrnerf_b200.ngp import disparity
    import xrnerf_b200.raymarch_cuda as rm
    torch.manual_seed(0)
    net = R.build_network(NGP_MODEL).cuda()
    n_img = scene['poses'].shape[0]
    net.sampler.set_data(dict(poses=scene['poses'], focal=np.full((n_img, 2), synth.FOCAL), aabb_scale=1, aabb_range=(0.0, 1.0), metadata=scene['metadata']), dict(H=800, W=800))
    net.sampler.density_grid_bitfield = dev(scene['bitfield'])
    t, d, c = synth.ngp_weights(seed=3, hash_range=0.5, mlp_gain=2.0)
    with torch.no_grad():
        net.mlp.field.hash_params.copy_(dev(t)); net.mlp.field.density_params.copy_(dev(d)); net.mlp.field.color_params.copy_(dev(c))
    data = {'rays_o': dev(scene['rays_o']), 'rays_d': dev(scene['rays_d']), 'img_ids': dev(scene['img_ids'].astype(np.float32)[:, None])}
    n = 4096
    with torch.no_grad():
        rm.reset_rng()
        got = net.batchify_forward(dict(data), is_test=True)
    assert got['depth'].shape == (n, 1) and got['disp'].shape == (n, 1) and torch.equal(got['disp'], disparity(got['depth'], got['alpha']))
    assert torch.isfinite(got['disp']).all() and (got['disp'] > 0).any()
    H = W = 64
    net.set_val_pipeline(lambda item: dict(data, src_shape=torch.tensor([H, W, 3])))
    net.phase = 'train'
    out = net.val_step({'poses': torch.zeros((1, 2, 4, 3)), 'images': torch.rand((1, 2, H, W, 4), device='cuda')})
    assert len(out['disps']) == 2 and all(x.shape == (H, W, 1) and torch.isfinite(x).all() for x in out['disps'])
    net.phase = 'test'
    sp = net.val_step({'poses': torch.zeros((1, 4, 3)), 'idx': 3})
    assert sp['spiral_disp'].shape == (H, W, 1) and sp['spiral_rgb'].shape == (H, W, 3) and sp['spiral_alpha'].shape == (H, W, 1) and sp['idx'] == 3
    net.phase = 'train'
    net.chunk, net.bs_data, net.fused_inference = 4096, 'rays_o', False
    out = net.val_step({'poses': torch.zeros((1, 1, 4, 3))})
    assert out['disps'] == [] and len(out['rgbs']) == 1


# ------------------------------------------------------------------------------------------------ CPU


def test_depth_entry_points_validate_arguments_without_gpu():
    _C, _buf, p, cfg, tab = cpu_args()
    lib = _C.lib
    bg = _C.float3(BG)
    f = C.c_float
    chain = lambda n, depth_out: lib.xrb_ngp_render_depth(cfg, tab, p, p, p, p, n, 256, f(0), f(1), f(0.05), f(1 / 256), 9121, 0, bg, 2, 3, p, p, depth_out, p, p, p,
                                                           None, None, None)
    fused = lambda n, depth_out: lib.xrb_ngp_render_fused_depth(cfg, tab, p, p, p, p, n, f(0), f(1), f(0.05), f(1 / 256), 9121, 0, bg, 2, 3, p, p, depth_out, p, p, None)
    for fn in (chain, fused):
        assert fn(4, None) == -1 and b'null' in lib.xrb_last_error()   # every other pointer is set: the missing depth output is what is refused
        assert fn(0, None) == 0                                         # an empty batch is a no-op
        assert fn(-1, p) == -1 and b'bad size' in lib.xrb_last_error()
    assert lib.xrb_ngp_render_depth(None, tab, p, p, p, p, 4, 256, f(0), f(1), f(0.05), f(1 / 256), 9121, 0, bg, 2, 3, p, p, p, p, p, p, None, None, None) == -1
    assert lib.xrb_ngp_render_depth(cfg, tab, p, p, p, p, 4, 0, f(0), f(1), f(0.05), f(1 / 256), 9121, 0, bg, 2, 3, p, p, p, p, p, p, None, None, None) == -1


def test_depth_tensor_checks_and_disparity_without_gpu():
    from xrnerf_b200 import _C
    from xrnerf_b200.ngp import _depth_ptr, disparity
    cpu = torch.device('cpu')
    ok = torch.zeros((8, 1))
    assert _depth_ptr(ok, 8, cpu).value == ok.data_ptr()
    for bad in (torch.zeros(8, dtype=torch.float64), torch.zeros(9), torch.zeros((8, 2))[:, 0], np.zeros(8, np.float32)):
        with pytest.raises(_C.XrbError):
            _depth_ptr(bad, 8, cpu)
    depth = torch.tensor([[0.0], [0.5], [0.0], [2.0]])
    alpha = torch.tensor([[0.0], [0.25], [0.5], [1.0]])
    disp = disparity(depth, alpha)[:, 0]
    assert disp[0] == 0 and disp[1] == 0.5 and disp[3] == 0.5                # no NaN where alpha == 0
    assert abs(float(disp[2]) - 1e10) <= 1e4                                 # depth / alpha clamped at 1e-10
