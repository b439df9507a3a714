"""GPU parity of the 10 raymarch_cuda replacements (xrnerf_b200.raymarch_cuda, through the C ABI) against the CPU oracle
(port, itself pinned bit-exact to the reference's own kernels in test_oracle_vs_ref.py).
Index path: bit-exact. Compositing (__expf + warp-scan association): |err| <= 2e-5 abs on colours in [0,1]."""
import numpy as np
import pytest
import torch
from cases import dev

pytestmark = pytest.mark.gpu


def _bits(a):
    return np.ascontiguousarray(a).view(np.uint32)


@pytest.fixture(scope='module')
def rm():
    import xrnerf_b200.raymarch_cuda as rm
    return rm


def gpu_march(rm, o, d, bf, cap, nprior=0, md=None, img=None, xf=None, aabb=(0.0, 1.0), near=0.05, cone=1.0 / 256):
    n = o.shape[0]
    coords = torch.zeros((cap, 7), dtype=torch.float32, device='cuda')
    ridx = torch.zeros((n, 1), dtype=torch.int32, device='cuda')
    ns = torch.zeros((n, 2), dtype=torch.int32, device='cuda')
    cnt = torch.zeros(2, dtype=torch.int32, device='cuda')
    rm.reset_rng(ray_sampler=nprior)
    rm.rays_sampler_api(dev(o), dev(d), dev(bf), None if md is None else dev(md), None if img is None else dev(img), None if xf is None else dev(xf), aabb[0], aabb[1], near, cone,
                        coords, ridx, ns, cnt)
    return coords.cpu().numpy(), ridx.cpu().numpy(), ns.cpu().numpy(), cnt.cpu().numpy()


def test_rays_sampler_bit_exact(rm, port, scene):
    s = scene
    a = port.rays_sampler(s['rays_o'], s['rays_d'], s['bitfield'], 4096 * 256)
    b = gpu_march(rm, s['rays_o'], s['rays_d'], s['bitfield'], 4096 * 256, md=s['metadata'], img=s['img_ids'], xf=s['poses'])
    assert np.array_equal(a[3], b[3]) and np.array_equal(a[2], b[2]) and np.array_equal(a[1], b[1])
    assert np.array_equal(_bits(a[0]), _bits(b[0]))


def test_rays_sampler_rng_advance_edges_overflow(rm, port, scene):
    s = scene
    o = np.array([[0.5, 0.5, -1.0], [0.5, 0.5, 0.5], [2.0, 2.0, 2.0], [0.5, -1.0, 0.5], [0.1, 0.2, -0.5]], np.float32)
    d = np.array([[0, 0, 1], [0.6, 0.0, 0.8], [1, 0, 0], [0, 1, 0], [0.3, 0.2, 0.9327379]], np.float32)
    o = np.concatenate([o, s['rays_o'][:251]]); d = np.concatenate([d, s['rays_d'][:251]])
    for cap, nprior in ((256 * 1024, 0), (700, 0), (256 * 1024, 5)):
        a = port.rays_sampler(o, d, s['bitfield'], cap, n_prior_calls=nprior)
        b = gpu_march(rm, o, d, s['bitfield'], cap, nprior=nprior)
        assert np.array_equal(a[3], b[3]) and np.array_equal(a[2], b[2]) and np.array_equal(a[1], b[1])
        assert np.array_equal(_bits(a[0]), _bits(b[0]))


def test_rays_sampler_dense_grid_1024_cap_and_empty(rm, port, scene):
    bf = np.full_like(scene['bitfield'], 255)
    o, d = scene['rays_o'][:200], scene['rays_d'][:200]
    a = port.rays_sampler(o, d, bf, 200 * 1024)
    b = gpu_march(rm, o, d, bf, 200 * 1024)
    assert np.array_equal(a[2], b[2]) and np.array_equal(_bits(a[0]), _bits(b[0]))
    z = np.zeros_like(bf)
    b = gpu_march(rm, o, d, z, 1024)
    assert b[3][1] == 0 and (b[1] == -1).all()
    # n_rays == 0 is a no-op
    gpu_march(rm, o[:0], d[:0], bf, 16)


@pytest.mark.parametrize('aabb,cone', [((0.0, 1.0), 0.0), ((0.0, 1.0), 1.0 / 64), ((-0.5, 1.5), 1.0 / 256), ((-3.5, 4.5), 1.0 / 256), ((0.1, 0.8), 0.0)])
def test_rays_sampler_any_aabb_cone(rm, port, scene, aabb, cone):
    """Which cell and cascade a tested position falls in depends on the position AND on the step at t (mip_from_dt): sparse random occupancy in EVERY cascade,
    growing steps (cone > 0), boxes that are not the unit cube and axis-parallel rays (zero direction components), bit-exact vs the oracle."""
    rng = np.random.default_rng(5)
    bf = np.zeros_like(scene['bitfield']).reshape(8, -1)
    for m in range(8):                       # a few isolated occupied cells per cascade, plus the scene's own cascade 0
        idx = rng.integers(0, bf.shape[1], 4000 if m else 400)
        bf[m, idx] |= (1 << rng.integers(0, 8, idx.size)).astype(np.uint8)
    bf[0] |= scene['bitfield'].reshape(8, -1)[0]
    bf = bf.reshape(-1)
    n = 6000
    o = (rng.uniform(-1, 2, (n, 3)) * (aabb[1] - aabb[0]) + aabb[0]).astype(np.float32)
    tgt = rng.uniform(aabb[0], aabb[1], (n, 3))
    d = tgt - o; d = (d / np.linalg.norm(d, axis=1, keepdims=True)).astype(np.float32)
    d[:50, 0] = 0; d[50:100, 1] = 0; d[100:120, :2] = 0; d[100:120, 2] = 1      # axis-parallel rays: zero components in the walk
    cap = n * 200
    a = port.rays_sampler(o, d, bf, cap, aabb=aabb, cone=cone)
    b = gpu_march(rm, o, d, bf, cap, aabb=aabb, cone=cone)
    assert int(a[3][1]) > 100                                                     # the case is not vacuous
    assert np.array_equal(a[3], b[3]) and np.array_equal(a[2], b[2]) and np.array_equal(a[1], b[1])
    assert np.array_equal(_bits(a[0]), _bits(b[0]))


def test_rays_sampler_full_image_property(rm, scene):
    """BASELINE-size property test: a whole 800x800 image; bases are the exclusive prefix sum of counts, samples sorted by ray."""
    from xrnerf_b200 import synth
    o, d = synth.get_rays_ngp(scene['poses'][3])
    c, ri, ns, cnt = gpu_march(rm, o, d, scene['bitfield'], 640000 * 48)
    counts = ns[:, 0].astype(np.int64)
    assert cnt[1] == counts.sum() and cnt[0] == 640000
    assert np.array_equal(ns[:, 1].astype(np.int64), np.concatenate([[0], np.cumsum(counts)[:-1]]))
    used = c[:cnt[1]]
    assert (used[:, :3] >= 0).all() and (used[:, :3] <= 1).all() and (used[:, 3] >= 0).all()


def test_rays_sampler_full_image_bit_exact_vs_oracle(rm, port, scene):
    """BASELINE-size parity (round-1 W1/W2): a whole 800x800 view in pixel order, marched by the CUDA path and by the oracle port: counts, bases,
    ray slots and every coords row bit for bit. The rays go through torch.from_numpy WITHOUT the test helper's ascontiguousarray, exactly as bench.py
    feeds them (a Fortran-ordered rays_o was read as different rays in round 1: the oracle gives ~10.9 samples/ray for this kind of view, that bug 23.0)."""
    from xrnerf_b200 import synth
    o, d = synth.get_rays_ngp(scene['poses'][21])
    cap = 640000 * 48
    a = port.rays_sampler(o, d, scene['bitfield'], cap)
    n = o.shape[0]
    coords = torch.zeros((cap, 7), dtype=torch.float32, device='cuda')
    ridx = torch.zeros((n, 1), dtype=torch.int32, device='cuda'); ns = torch.zeros((n, 2), dtype=torch.int32, device='cuda'); cnt = torch.zeros(2, dtype=torch.int32, device='cuda')
    rm.reset_rng(ray_sampler=0)
    rm.rays_sampler_api(torch.from_numpy(o).cuda(), torch.from_numpy(d).cuda(), dev(scene['bitfield']), None, None, None, 0.0, 1.0, 0.05, 1.0 / 256, coords, ridx, ns, cnt)
    total = int(a[3][1])
    assert 8.0 < total / n < 14.0, total / n                      # the oracle's own figure for a spiral view of this scene
    assert np.array_equal(a[3], cnt.cpu().numpy()) and np.array_equal(a[2], ns.cpu().numpy()) and np.array_equal(a[1], ridx.cpu().numpy())
    assert np.array_equal(_bits(a[0][:total]), _bits(coords[:total].cpu().numpy()))
    assert (a[2][:, 0] > 64).any()                                 # rays longer than the inline t cache exist in this view: the overflow-chunk emit path ran


def test_compacted_coord(rm, port, scene):
    s = scene
    c, _, ns, cnt = port.rays_sampler(s['rays_o'], s['rays_d'], s['bitfield'], 4096 * 256)
    coords = c[:cnt[1]]
    raw = np.zeros((cnt[1], 4), np.float32)
    for cap in (1 << 18, 20000, 1):
        a = port.compacted_coord(raw, coords, ns, cap)
        co = torch.zeros((cap, 7), dtype=torch.float32, device='cuda')
        nsc = torch.zeros((ns.shape[0], 2), dtype=torch.int32, device='cuda')
        rc = torch.zeros(1, dtype=torch.int32, device='cuda'); sc = torch.zeros(1, dtype=torch.int32, device='cuda')
        rm.compacted_coord_api(dev(raw), dev(coords), dev(ns), torch.ones(3), 2, 3, 0.0, 1.0, co, nsc, rc, sc)
        assert np.array_equal(a[1], nsc.cpu().numpy()) and a[2][0] == rc.item() and a[3][0] == sc.item()
        assert np.array_equal(_bits(a[0]), _bits(co.cpu().numpy()))


@pytest.mark.parametrize('rgb_act,dens_act', [(2, 3), (3, 1), (0, 2)])
def test_calc_rgb_forward_backward_inference(rm, port, scene, rgb_act, dens_act):
    s = scene
    c, _, ns, cnt = port.rays_sampler(s['rays_o'], s['rays_d'], s['bitfield'], 4096 * 256)
    coords = c[:cnt[1]]
    rng = np.random.default_rng(5)
    raw_all = rng.normal(0, 1.5, (cnt[1], 4)).astype(np.float32); raw_all[:, 3] += 2.0
    cc, nsc, _, _ = port.compacted_coord(raw_all, coords, ns, 30000)
    raw = raw_all[:30000].copy()
    bg = rng.random((ns.shape[0], 3)).astype(np.float32)
    f_ref = port.calc_rgb_forward(raw, cc, ns, nsc, bg, rgb_act, dens_act)
    out = torch.zeros((ns.shape[0], 3), dtype=torch.float32, device='cuda')
    rm.calc_rgb_forward_api(dev(raw), dev(cc), dev(ns), dev(nsc), dev(bg), rgb_act, dens_act, 0.0, 1.0, out)
    assert np.abs(out.cpu().numpy() - f_ref).max() <= 2e-5 * max(1.0, np.abs(f_ref).max())
    g = rng.normal(0, 1, f_ref.shape).astype(np.float32)
    for mean in (0.5, 0.001):
        b_ref = port.calc_rgb_backward(raw, nsc, cc, g, f_ref, np.array([mean], np.float32), rgb_act, dens_act)
        dl = torch.zeros((raw.shape[0], 4), dtype=torch.float32, device='cuda')
        rm.calc_rgb_backward_api(dev(raw), dev(nsc), dev(cc), dev(g), dev(f_ref), dev(np.array([mean], np.float32)), rgb_act, dens_act, 0.0, 1.0, dl)
        assert np.abs(dl.cpu().numpy() - b_ref).max() <= 5e-5 * max(1.0, np.abs(b_ref).max())
    i_ref = port.calc_rgb_inference(raw_all, coords, ns, np.array([0.2, 0.4, 0.9], np.float32), rgb_act, dens_act)
    rgb = torch.zeros((ns.shape[0], 3), dtype=torch.float32, device='cuda'); alpha = torch.zeros((ns.shape[0], 1), dtype=torch.float32, device='cuda')
    rm.calc_rgb_influence_api(dev(raw_all), dev(coords), dev(ns), torch.tensor([0.2, 0.4, 0.9]), rgb_act, dens_act, 0.0, 1.0, rgb, alpha)
    assert np.abs(rgb.cpu().numpy() - i_ref[0]).max() <= 2e-5 * max(1.0, np.abs(i_ref[0]).max())
    assert np.abs(alpha.cpu().numpy() - i_ref[1]).max() <= 2e-5


def test_long_rays_composite(rm, port, scene):
    """rays with up to 1024 samples (dense grid): product-scan error stays within tolerance"""
    bf = np.full_like(scene['bitfield'], 255)
    o, d = scene['rays_o'][:64], scene['rays_d'][:64]
    c, _, ns, cnt = port.rays_sampler(o, d, bf, 64 * 1024)
    rng = np.random.default_rng(1)
    raw = rng.normal(0, 1, (cnt[1], 4)).astype(np.float32); raw[:, 3] -= 1.0
    i_ref = port.calc_rgb_inference(raw, c[:cnt[1]], ns, np.zeros(3, np.float32))
    rgb = torch.zeros((64, 3), dtype=torch.float32, device='cuda'); alpha = torch.zeros((64, 1), dtype=torch.float32, device='cuda')
    rm.calc_rgb_influence_api(dev(raw), dev(c[:cnt[1]]), dev(ns), torch.zeros(3), 2, 3, 0.0, 1.0, rgb, alpha)
    assert np.abs(rgb.cpu().numpy() - i_ref[0]).max() <= 2e-5 and np.abs(alpha.cpu().numpy() - i_ref[1]).max() <= 2e-5


def test_grid_kernels(rm, port, scene):
    from xrnerf_b200 import synth
    n_img = 7
    focal = np.full((n_img, 2), synth.FOCAL, np.float32)
    a = port.mark_untrained(focal, scene['poses'][:n_img], n_img, (800, 800))
    g = torch.full((8 * 128 ** 3,), 7.0, dtype=torch.float32, device='cuda')  # garbage pre-fill: must be fully overwritten
    rm.mark_untrained_density_grid_api(dev(focal), dev(scene['poses'][:n_img]), g.numel(), n_img, 800, 800, g)
    assert np.array_equal(a, g.cpu().numpy())

    grid = scene['grid'].copy(); grid[128 ** 3:] = -1.0
    for step, thresh, n, nprior, mc in ((0, -0.01, 1 << 16, 0, 0), (5, 0.01, 1 << 15, 4, 0), (1, -0.01, 1 << 14, 0, 2)):
        pa, ia = port.generate_grid_samples(grid, step, n, mc, thresh, n_prior_calls=nprior)
        pos = torch.zeros((n, 3), dtype=torch.float32, device='cuda'); idx = torch.zeros(n, dtype=torch.int32, device='cuda')
        rm.reset_rng(generate_grid_samples=nprior)
        rm.generate_grid_samples_nerf_nonuniform_api(dev(grid), step, n, mc, thresh, 0.0, 1.0, pos, idx)
        assert np.array_equal(ia, idx.cpu().numpy()) and np.array_equal(_bits(pa), _bits(pos.cpu().numpy()))

    rng = np.random.default_rng(3)
    n = 1 << 16
    idx = rng.integers(0, 128 ** 3, n).astype(np.int32); idx[:100] = idx[0]
    dens = rng.normal(-3, 2, (n, 1)).astype(np.float32)
    tmp0 = np.zeros(8 * 128 ** 3, np.float32)
    a = port.splat(dens, idx, tmp0)
    t = dev(tmp0)
    rm.splat_grid_samples_nerf_max_nearest_neighbor_api(dev(dens), dev(idx), 1, n, t)
    tg = t.cpu().numpy()
    assert np.array_equal(a > 0, tg > 0) and np.abs(a - tg).max() <= 1e-5 * np.abs(a).max()  # __expf vs expf

    grid2 = scene['grid'].copy(); grid2[rng.integers(0, grid2.size, 5000)] = -1.0
    e_ref = port.ema(a, grid2)
    gg = dev(grid2)
    rm.ema_grid_samples_nerf_api(dev(a), grid2.size, 0.95, gg)
    assert np.array_equal(_bits(e_ref), _bits(gg.cpu().numpy()))

    for g_np in (e_ref, scene['grid'], np.zeros_like(grid2)):
        b_ref, m_ref = port.update_bitfield(g_np)
        mean = torch.zeros(16384, dtype=torch.float32, device='cuda'); bf = torch.zeros(8 * 128 ** 3 // 8, dtype=torch.uint8, device='cuda')
        rm.update_bitfield_api(dev(g_np), mean, bf)
        assert mean[0].item() == m_ref[0]
        assert np.array_equal(b_ref, bf.cpu().numpy())
