"""The chain render (xrb_ngp_render) evaluates the field over its samples bucketed by position: the order it uses is a permutation of the
marched rows sorted by bucket, and the rendered pixels are bit-identical to the same march evaluated in ray order."""
import numpy as np
import pytest
import torch
from cases import dev

pytestmark = pytest.mark.gpu


@pytest.fixture(scope='module')
def field():
    from xrnerf_b200 import synth
    from xrnerf_b200.ngp import NgpField
    f = NgpField().cuda()
    table, dens, color = synth.ngp_weights(seed=3, hash_range=0.5, mlp_gain=2.0)
    with torch.no_grad():
        f.hash_params.copy_(dev(table)); f.density_params.copy_(dev(dens)); f.color_params.copy_(dev(color))
    return f


def workspace_views(r, n_rays):
    """coords [max_samples,7] and the evaluation order [max_samples] inside the renderer's workspace (layout: include/xrnerf_b200.h)"""
    from xrnerf_b200 import _C
    ms = r._max_samples
    off = (_C.lib.xrb_rm_rays_sampler_workspace(n_rays) + 255) & ~255
    coords = r._ws[off:off + ms * 28].view(torch.float32).view(ms, 7)
    order = r._ws[off + ms * 44:off + ms * 48].view(torch.int32)
    return coords, order


def bucket_keys(coords):
    """the 64^3 Morton bucket of each row, as the ordering kernel computes it (NaN-safe clamp: rows past an overflowed ray hold stale memory)"""
    q = np.fmin(np.fmax(coords[:, :3] * np.float32(64), np.float32(0)), np.float32(63)).astype(np.uint32)
    key = np.zeros(len(q), np.uint32)
    for b in range(6):
        for a in range(3):
            key |= ((q[:, a] >> b) & 1) << (3 * b + a)
    return key


def render_and_check_order(f, o, d, bf, budget):
    from xrnerf_b200.ngp import NgpRenderer
    r = NgpRenderer(f, samples_per_ray_budget=budget)
    rgb, alpha, ns, cnt = r.render(o, d, bf)
    torch.cuda.synchronize()
    n = min(int(cnt[1]), r._max_samples)
    coords, order = workspace_views(r, o.shape[0])
    perm = order[:n].cpu().numpy().astype(np.int64)
    assert np.array_equal(np.sort(perm), np.arange(n))
    keys = bucket_keys(coords[:n].cpu().numpy())[perm]
    assert (np.diff(keys.astype(np.int64)) >= 0).all()           # evaluated bucket by bucket
    return r, (rgb, alpha, ns, cnt), n


def test_order_is_a_bucket_sorted_permutation_of_a_bench_batch(field):
    from xrnerf_b200 import synth
    bf, _ = synth.bitfield_from_grid_numpy(synth.lego_like_density_grid(0))
    o, d = synth.ray_batch(65536, seed=1005)[:2]
    r, out, n = render_and_check_order(field, dev(o), dev(d), dev(bf), 64)
    assert n > 65536 and not bool(r.overflowed(out[3]))


def test_order_all_ones_grid(scene, field):
    o, d = dev(scene['rays_o'][:2048]), dev(scene['rays_d'][:2048])
    ones = torch.full_like(dev(scene['bitfield']), 255)
    r, out, n = render_and_check_order(field, o, d, ones, 1024)
    assert int(out[2][:, 0].max()) > 64 and n == int(out[3][1])


def test_order_when_rays_overflow_the_sample_budget(scene, field):
    """counters[1] > max_samples: the rows past the first overflowed ray were never written by the march and still get a bucket"""
    o, d, bf = dev(scene['rays_o']), dev(scene['rays_d']), dev(scene['bitfield'])
    r, out, n = render_and_check_order(field, o, d, bf, 4)
    assert bool(r.overflowed(out[3])) and n == r._max_samples
    assert (out[2][:, 0] == 0).any()


def test_order_when_every_ray_misses(scene, field):
    o = torch.full((1000, 3), 2.0, device='cuda')                 # outside the unit box, looking away from it
    d = torch.nn.functional.normalize(torch.ones((1000, 3), device='cuda'), dim=1)
    r, out, n = render_and_check_order(field, o, d, dev(scene['bitfield']), 64)
    assert n == 0 and int(out[2][:, 0].abs().sum()) == 0 and float(out[1].abs().sum()) == 0.0


@pytest.mark.parametrize('call', [0, 3])
def test_render_is_bit_identical_to_ray_order_evaluation(scene, field, call):
    """NgpRenderer.render == rays_sampler_api -> NgpField.run_mlp (rows in ray order) -> calc_rgb_influence_api, same RNG call index"""
    import xrnerf_b200.raymarch_cuda as rm
    from xrnerf_b200.ngp import NgpRenderer
    o, d, bf = dev(scene['rays_o']), dev(scene['rays_d']), dev(scene['bitfield'])
    n_rays = o.shape[0]
    bg = (0.1, 0.5, 0.9)
    r = NgpRenderer(field, bg=bg)
    r.calls = call
    rgb, alpha, ns, cnt = (x.clone() for x in r.render(o, d, bf))
    rm.reset_rng(ray_sampler=call)
    coords = torch.zeros((n_rays * 64, 7), device='cuda'); ridx = torch.zeros((n_rays, 1), dtype=torch.int32, device='cuda')
    ns_ref = torch.zeros((n_rays, 2), dtype=torch.int32, device='cuda'); cnt_ref = torch.zeros(2, dtype=torch.int32, device='cuda')
    rm.rays_sampler_api(o, d, bf, None, None, None, r.aabb[0], r.aabb[1], r.near, r.cone, coords, ridx, ns_ref, cnt_ref)
    S = int(cnt_ref[1])
    raw = field.run_mlp(coords[:S, :3], coords[:S, 4:])
    rgb_ref = torch.empty((n_rays, 3), device='cuda'); alpha_ref = torch.empty((n_rays, 1), device='cuda')
    rm.calc_rgb_influence_api(raw, coords, ns_ref, torch.tensor(bg), r.rgb_act, r.dens_act, r.aabb[0], r.aabb[1], rgb_ref, alpha_ref)
    assert torch.equal(cnt, cnt_ref) and torch.equal(ns, ns_ref)
    assert torch.equal(rgb, rgb_ref) and torch.equal(alpha, alpha_ref)
    assert float(alpha.max()) > 0.2


def test_two_renders_are_bit_identical(field):
    """the order inside a bucket depends on atomics; the pixels do not"""
    from xrnerf_b200 import synth
    from xrnerf_b200.ngp import NgpRenderer
    bf, _ = synth.bitfield_from_grid_numpy(synth.lego_like_density_grid(0))
    o, d = (dev(x) for x in synth.ray_batch(65536, seed=7)[:2])
    r = NgpRenderer(field, bg=(0.2, 0.3, 0.4))
    a = [x.clone() for x in r.render(o, d, dev(bf))]
    r.calls = 0
    b = r.render(o, d, dev(bf))
    assert all(torch.equal(x, y) for x, y in zip(a, b))
