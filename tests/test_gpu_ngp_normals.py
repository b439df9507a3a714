"""NGP normal maps: the density gradient on tensor cores (xrb_ngp_density_grad_tc, NgpField.density_grad_tc), the chain render with normals
(xrb_ngp_render_normals, NgpRenderer.render(normals=...)) and HashNerfNetwork.render_normals. include/xrnerf_b200.h ("Normal maps") states the contract.

Gradient restatement (numpy, float64, over the kernel's fp16 weights and its fp16 encodings from xrb_tcnn_hashgrid_forward). The tensor-core forward sums in
fp32 in an order the hardware picks, so the masks are not restated exactly: a row whose hidden pre-activation lies within the forward's error bound of 0
(K 2^-22 times the sum of |w| |x| for a K-term tensor-core sum, plus the spread of the layer before's fp16 activation, which is exact unless a rounding
boundary of fp16 lies within that layer's own bound) has an ambiguous mask, and is counted and
excluded. With the masks fixed, the kernel's gradient is a sum of products: each W^T step a 64-term tensor-core sum (64 2^-22), dh - 1 fp16 stagings of d(density)/d(hidden)
(relative 2^-11, plus 2^-25 / 2^10 absolute for an entry in the fp16 subnormal range), and the 27 fp32 roundings of position_grad_level (2 + 1 + 8 + 16, as
in test_gpu_mesh_attributes). The bound is that relative factor times the same chain on absolute values, plus the subnormal terms carried down the
absolute chain, plus the float64 restatement's own gamma. Nothing in it is fitted to a run.
"""
import ctypes as C
import math

import numpy as np
import pytest
import torch

from cases import NGP_MODEL, SPHERE_C, SPHERE_R, cpu_args, dev, face_points, load_ngp_weights, ngp_density_grad, ngp_field, random_points, sphere_network
from restate64 import GAMMA_TC, U16, U32, U64, Grid, cuda_core_density_grad, field_mats, gamma, hashgrid_enc16, position_grad

f32 = np.float32
SUB = 2.0 ** -25 / 1024              # fp16 staging: half the subnormal spacing, over the 2^10 staging scale
REPORT = []


def tc_restated(field, grid, x):
    """float64 gradient, its bound and the rows whose masks are unambiguous, at x f32[n,3]"""
    mats = field_mats(field)
    a, ea = hashgrid_enc16(field, x), np.zeros((len(x), 32))           # layer input and its absolute error against the kernel's
    masks, ok = [], np.ones(len(x), bool)
    for W in mats[:-1]:
        z = a @ W.T
        ez = np.abs(W) @ ea.T
        ez = ez.T + W.shape[1] * GAMMA_TC * (np.abs(a) + ea) @ np.abs(W).T
        ok &= (np.abs(z) > ez + 2.0 ** -24).all(1)             # fp16(z) > 0 iff z > 2^-25: decided unless z is this close to 0
        m = z > 0
        masks.append(m)
        # the kernel's activation fp16(z_k) lies between the fp16 roundings of z -+ ez (rounding is monotone): exact where those agree
        lo = np.maximum(z - ez * (1 + 1e-9), 0).astype(np.float16).astype(np.float64)
        hi = np.maximum(z + ez * (1 + 1e-9), 0).astype(np.float16).astype(np.float64)
        a, ea = np.where(m, lo, 0.0), np.where(m, hi - lo, 0.0)
    dh = len(mats) - 2 + 1
    g, ga, gs = masks[-1] * mats[-1][0][None, :], masks[-1] * np.abs(mats[-1][0])[None, :], np.zeros((len(x), 64))
    for k in range(dh - 1, 0, -1):
        W = mats[k]
        g, ga = masks[k - 1] * (g @ W), masks[k - 1] * (ga @ np.abs(W))
        gs = masks[k - 1] * (gs @ np.abs(W) + SUB)
    ge, gea, ges = g @ mats[0], ga @ np.abs(mats[0]), gs @ np.abs(mats[0])
    pg, m = position_grad(grid, x, ge, gea)
    _, ms = position_grad(grid, x, ge, ges)
    rel = (1 + U16) ** (dh - 1) * (1 + 64 * dh * GAMMA_TC) * (1 + gamma(27, U32)) - 1
    return pg, (rel + gamma(64 * dh + 27, U64)) * m + (1 + rel) * ms, ok


def kernel_tc(field, pts, density=True, order=None, n_dev=None):
    d, g = field.density_grad_tc(pts, density=density, order=order, n_rows_dev=n_dev)
    return d, g


CASES = [(dh, npk) for dh in (1, 2) for npk in (0, 6, 7)]


@pytest.fixture(scope='module', params=CASES, ids=[f'dh{dh}-packed{npk}' for dh, npk in CASES])
def case(request):
    dh, npk = request.param
    f = ngp_field(dh, npk)
    return f, Grid.of(f)


# ================================================================================================================ row stage
@pytest.mark.gpu
def test_density_bit_identical_to_tensor_core_field(case):
    field, _ = case
    for n in (0, 1, 127, 129, 5000):
        x = dev(random_points(n, 30 + n)) if n else torch.empty((0, 3), device='cuda')
        rows = torch.full((n, 7), 9.0, device='cuda')
        rows[:, :3] = x
        want = field.run_density(x, impl=1) if n else torch.empty((0, 1), device='cuda')
        g_ref = None
        for pts in (x, rows[:, :3]):
            d, g = kernel_tc(field, pts)
            assert d.shape == (n, 1) and g.shape == (n, 3)
            assert torch.equal(d.view(torch.int32), want.view(torch.int32))
            assert torch.isfinite(g).all()
            g_ref = g if g_ref is None else g_ref
            assert torch.equal(g.view(torch.int32), g_ref.view(torch.int32))
        d0, g0 = kernel_tc(field, x, density=False)
        assert d0 is None and torch.equal(g0.view(torch.int32), g_ref.view(torch.int32))


@pytest.mark.gpu
def test_rows_independent_of_order_and_count(case):
    field, _ = case
    n = 3000
    x = dev(random_points(n, 41))
    _, g = kernel_tc(field, x)
    d = field.run_density(x, impl=1)
    perm = torch.randperm(n, generator=torch.Generator().manual_seed(2)).to(torch.int32).cuda()
    d1, g1 = kernel_tc(field, x, order=perm)
    assert torch.equal(d1.view(torch.int32), d.view(torch.int32)) and torch.equal(g1.view(torch.int32), g.view(torch.int32))
    m = 1234
    n_dev = torch.tensor([m], dtype=torch.int32, device='cuda')
    sub = torch.randperm(m, generator=torch.Generator().manual_seed(3)).to(torch.int32).cuda()
    order = torch.cat([sub, torch.arange(m, n, dtype=torch.int32, device='cuda')])
    d2, g2 = kernel_tc(field, x, order=order, n_dev=n_dev)
    assert torch.equal(d2[:m].view(torch.int32), d[:m].view(torch.int32)) and torch.equal(g2[:m].view(torch.int32), g[:m].view(torch.int32))


def _check(field, grid, x, what):
    _, g = kernel_tc(field, dev(x))
    g = g.cpu().numpy().astype(np.float64)
    g64, bound, ok = tc_restated(field, grid, x)
    err = np.abs(g - g64)
    bad = ~(err <= bound).all(1) & ok
    assert not bad.any(), f'{what}: {int(bad.sum())} rows beyond the bound, max err/bound {float((err / np.maximum(bound, 1e-300))[ok].max()):.3g}'
    return int((~ok).sum()), len(x), float((err / np.maximum(bound, 1e-300))[ok].max()) if ok.any() else 0.0, g, bound


@pytest.mark.gpu
def test_gradient_within_derived_bound(case):
    field, grid = case
    amb, total, worst = 0, 0, 0.0
    for x, what in ((random_points(3000, 51), 'random'), (face_points(grid, 40, 52), 'faces'), (random_points(129, 53), 'n=129')):
        a, n, w, _, _ = _check(field, grid, x, what)
        amb, total, worst = amb + a, total + n, max(worst, w)
    # one hidden layer: the masks are decided by the encodings alone. Two: a layer-1 activation whose fp16 rounding boundary lies inside the tensor-core
    # accumulation bound (K 2^-22) may be either neighbour, which widens layer 2's bound; about 1.6 % of these rows, so the limit there is 2 %
    limit = 1e-3 if field.cfg.density_hidden == 1 else 2e-2
    assert amb < limit * total, f'{amb} of {total} rows have an ambiguous mask'
    REPORT.append(f'density_grad_tc dh {field.cfg.density_hidden} / packed {field.n_packed}: max |err| / bound = {worst:.3g}, ambiguous masks {amb} of {total}')
    print(REPORT[-1])


@pytest.mark.gpu
def test_agrees_with_cuda_core_kernel(case):
    field, grid = case
    x = random_points(2000, 61)
    _, g_tc, b_tc = _check(field, grid, x, 'tc')[2:]
    _, g_cc = ngp_density_grad(field, x)
    _, _, b_cc = cuda_core_density_grad(field, grid, x)
    _, _, ok = tc_restated(field, grid, x)
    err = np.abs(g_tc - g_cc)[ok]
    assert (err <= (b_tc + b_cc)[ok]).all(), f'max err/bound {float((err / (b_tc + b_cc)[ok]).max()):.3g}'


# ================================================================================================================ render
def _ngp_field():
    from xrnerf_b200 import synth
    from xrnerf_b200.ngp import NgpField
    return load_ngp_weights(NgpField().cuda(), synth.ngp_weights(seed=3, hash_range=0.5, mlp_gain=2.0))


def _workspace_rows(r, n, max_samples):
    """(coords [max_samples,7], raw [max_samples,4], grad [max_samples,3]) of the renderer's workspace (include/xrnerf_b200.h layout)"""
    from xrnerf_b200 import _C
    a256 = lambda b: (b + 255) // 256 * 256
    ws = r._ws
    c0 = a256(_C.lib.xrb_rm_rays_sampler_workspace(n))
    fl = ws[c0:c0 + max_samples * 11 * 4].view(torch.float32)
    g0 = a256(_C.lib.xrb_ngp_render_workspace(n, max_samples) - 256)
    return fl[:max_samples * 7].view(max_samples, 7), fl[max_samples * 7:].view(max_samples, 4), ws[g0:g0 + max_samples * 12].view(torch.float32).view(max_samples, 3)


def _weights64(coords, raw, ns):
    """float64 composite weights w = T alpha of every ray's rows (dens_act 3: sigma = exp(raw)), as lists of (rows, w)"""
    min_dt = float(f32(f32(1.73205080757) / f32(1024)))
    out = []
    for c, b in ns:
        rows = np.arange(b, b + c)
        dt = coords[rows, 3].astype(np.float64) * (min_dt * 128 - min_dt) + min_dt
        a = 1.0 - np.exp(-np.exp(raw[rows, 3].astype(np.float64)) * dt)
        T = np.concatenate([[1.0], np.cumprod(1.0 - a)[:-1]])
        out.append((rows, T * a))
    return out


@pytest.mark.gpu
def test_render_normals_changes_nothing_else(scene):
    from xrnerf_b200 import synth
    from xrnerf_b200.ngp import NgpRenderer
    f = _ngp_field()
    bf = dev(scene['bitfield'])
    vo, vd = synth.get_rays_ngp(scene['poses'][7])
    for o, d, budget in ((dev(scene['rays_o']), dev(scene['rays_d']), 64), (dev(vo), dev(vd), 48)):
        n = o.shape[0]
        ra, rb = NgpRenderer(f, samples_per_ray_budget=budget), NgpRenderer(f, samples_per_ray_budget=budget)
        for call in range(2):
            da, db, nb = torch.empty(n, device='cuda'), torch.empty(n, device='cuda'), torch.empty((n, 3), device='cuda')
            a = [t.clone() for t in ra.render(o, d, bf, depth=da)]
            b = [t.clone() for t in rb.render(o, d, bf, depth=db, normals=nb)]
            for x, y in zip(a[:3] + [da], b[:3] + [db]):
                assert torch.equal(x.view(torch.int32), y.view(torch.int32))
            assert torch.isfinite(nb).all()


@pytest.mark.gpu
@pytest.mark.parametrize('n', [4096, 1, 33, 1000])
def test_render_normals_match_float64_composite(scene, n):
    """normal vs the float64 composite of the kernel's own per-row gradients with the march's weights (restated from the kernel's raw rows). Bound:
    gamma_(S+2) sum w |n| for the fp32 sums, plus 8 u per sample for the fp32 evaluation of alpha = 1 - exp(-sigma dt) and of T (absolute: the
    cancellation in 1 - exp(-x) makes it so), plus 4 u per sample for the fp32 normalisation of g."""
    from xrnerf_b200.ngp import NgpRenderer
    f = _ngp_field()
    o, d = dev(scene['rays_o'][:n]), dev(scene['rays_d'][:n])
    r = NgpRenderer(f, samples_per_ray_budget=64)
    dpt, nrm = torch.empty(n, device='cuda'), torch.empty((n, 3), device='cuda')
    _, alpha, ns, counters = r.render(o, d, dev(scene['bitfield']), depth=dpt, normals=nrm)
    assert not bool(r.overflowed(counters))
    coords, raw, grad = (t.cpu().numpy() for t in _workspace_rows(r, n, n * 64))
    ns = ns.cpu().numpy()
    g = grad.astype(np.float64)
    gl = np.linalg.norm(g, axis=1, keepdims=True)
    nhat = np.where(gl > 0, -g / np.where(gl > 0, gl, 1), 0.0)
    got = nrm.cpu().numpy().astype(np.float64)
    worst = 0.0
    for i, (rows, w) in enumerate(_weights64(coords, raw, ns)):
        S = len(rows)
        want = (w[:, None] * nhat[rows]).sum(0)
        bound = gamma(S + 2, U32) * (w[:, None] * np.abs(nhat[rows])).sum(0) + 12 * U32 * S
        err = np.abs(got[i] - want)
        assert (err <= bound).all(), (i, S, err, bound)
        worst = max(worst, float((err / bound).max()) if S else 0.0)
    assert (alpha.cpu().numpy()[ns[:, 0] > 0] > 0).any()
    assert np.all(got[ns[:, 0] == 0] == 0)
    REPORT.append(f'render normals, {n} rays: max |err| / bound = {worst:.3g}')


@pytest.mark.gpu
def test_sphere_normals_face_the_camera():
    """The sphere field of cases.sphere_network (raw = K (r - |x - c|) by trilinear interpolation of fp16 samples on level 4, K = 20 so that central
    rays become opaque). At every pixel with alpha > 0.99: N . d < 0, and the angle between the normal and the float64 composite of the analytic radial
    directions at the same samples with the same weights is within the bound derived from the trilinear error: the interpolant's gradient differs from
    the exact one by at most 3 h / (rho - sqrt(3) h) (each edge difference quotient is the derivative at a point of the edge, within sqrt(3) h of the
    sample, and |Hessian| = 1 / rho) plus 2 sqrt(3) delta / h for the fp16 samples (delta = 2^-11 (|sdf| + sqrt(3) h), the corners' largest
    magnitude), so the unit normals differ by at most twice that;
    2^-8 more covers the kernel's own arithmetic, which the row tests bound far tighter."""
    from xrnerf_b200.ngp import NgpRenderer
    net, grid = sphere_network()
    f = net.mlp.field
    K = 20.0
    with torch.no_grad():
        f.density_params[64 * 32 + 0] = K; f.density_params[64 * 32 + 1] = -K
    f.mark_dirty()
    m = 32
    u = (np.arange(m) + 0.5) / m * 0.16 - 0.08
    px, py = np.meshgrid(u, u, indexing='ij')
    o = np.stack([0.5 + px.ravel(), 0.5 + py.ravel(), np.full(m * m, -0.5)], 1).astype(f32)
    d = np.tile(np.array([[0.0, 0.0, 1.0]], f32), (m * m, 1))
    from xrnerf_b200 import synth
    bf = np.full_like(synth.bitfield_from_grid_numpy(synth.lego_like_density_grid(0))[0], 255)
    n = m * m
    r = NgpRenderer(f, samples_per_ray_budget=1024)
    dpt, nrm = torch.empty(n, device='cuda'), torch.empty((n, 3), device='cuda')
    _, alpha, ns, counters = r.render(dev(o), dev(d), dev(bf), depth=dpt, normals=nrm)
    assert not bool(r.overflowed(counters))
    coords, raw, _ = (t.cpu().numpy() for t in _workspace_rows(r, n, n * 1024))
    ns, alpha, got = ns.cpu().numpy(), alpha.cpu().numpy()[:, 0], nrm.cpu().numpy().astype(np.float64)
    h = 1.0 / float(grid.scale[4])
    opaque = alpha > 0.99
    assert opaque.sum() >= 0.9 * n
    worst, worst_bound = 0.0, 0.0
    for i, (rows, w) in enumerate(_weights64(coords, raw, ns)):
        if not opaque[i]:
            continue
        x = coords[rows, :3].astype(np.float64)
        rad = x - SPHERE_C
        rho = np.linalg.norm(rad, axis=1)
        radial = rad / rho[:, None]
        delta = U16 * (np.abs(SPHERE_R - rho) + math.sqrt(3) * h)
        E = 3 * h / np.maximum(rho - math.sqrt(3) * h, 1e-30) + 2 * math.sqrt(3) * delta / h
        e = np.where(rho > 2 * math.sqrt(3) * h, np.minimum(2.0, 2 * E + 2.0 ** -8), 2.0)
        want = (w[:, None] * radial).sum(0)
        B = np.linalg.norm(want)
        limit = math.asin(min(1.0, ((w * e).sum() + 12 * U32 * len(rows)) / B))
        assert float(got[i] @ d[i]) < 0
        ang = math.acos(max(-1.0, min(1.0, float(got[i] @ want) / (np.linalg.norm(got[i]) * B))))
        assert ang <= limit, (i, math.degrees(ang), math.degrees(limit))
        if ang > worst:
            worst, worst_bound = ang, limit
    REPORT.append(f'sphere normals: {int(opaque.sum())} opaque pixels, max angle to the radial composite {math.degrees(worst):.3f} deg (bound there {math.degrees(worst_bound):.3f} deg)')
    print(REPORT[-1])


# ================================================================================================================ network
def _net(scene):
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
    return net, data


@pytest.mark.gpu
def test_network_render_normals(scene):
    import xrnerf_b200.raymarch_cuda as rm
    from xrnerf_b200.ngp import NgpRenderer
    net, data = _net(scene)
    n, H, W = 4096, 64, 64
    net.set_val_pipeline(lambda item: dict(data, src_shape=torch.tensor([H, W, 3])))
    with torch.no_grad():
        net.phase = 'train'
        plain = net.val_step({'poses': torch.zeros((1, 1, 4, 3))})
        assert set(plain) == {'rgbs', 'disps', 'gt_imgs', 'elapsed_time', 'psnr'}
        net.phase = 'test'
        assert set(net.val_step({'poses': torch.zeros((1, 4, 3)), 'idx': 1})) == {'spiral_rgb', 'spiral_alpha', 'spiral_disp', 'idx'}
        net.render_normals = True
        rm.reset_rng(5)
        got = net.batchify_forward(dict(data), is_test=True)
        assert got['normal'].shape == (n, 3) and got['depth'].shape == (n, 1)
        r = NgpRenderer(net.mlp.field, aabb=(0.0, 1.0), near=net.sampler.near_distance, cone=net.sampler.cone_angle_constant, bg=(0.0, 0.0, 0.0))
        r.calls = 5
        dp, nm = torch.empty((n, 1), device='cuda'), torch.empty((n, 3), device='cuda')
        rgb, alpha, _, _ = r.render(data['rays_o'], data['rays_d'], net.sampler.density_grid_bitfield, depth=dp, normals=nm)
        for a, b in ((got['rgb'], rgb), (got['alpha'], alpha), (got['depth'], dp), (got['normal'], nm)):
            assert torch.equal(a.view(torch.int32), b.view(torch.int32))
        # overflow: a budget of one sample per ray re-renders the view with the marched row count and the same jitter
        budget = net._renderer.budget
        net._renderer.budget = 1
        rm.reset_rng(5)
        small = net.batchify_forward(dict(data), is_test=True)
        net._renderer.budget = budget
        for k in ('rgb', 'alpha', 'depth', 'normal'):
            assert torch.equal(small[k].view(torch.int32), got[k].view(torch.int32)), k
        net.phase = 'train'
        out = net.val_step({'poses': torch.zeros((1, 2, 4, 3))})
        assert len(out['normals']) == 2 and all(x.shape == (H, W, 3) and torch.isfinite(x).all() for x in out['normals'])
        net.phase = 'test'
        sp = net.val_step({'poses': torch.zeros((1, 4, 3)), 'idx': 2})
        assert sp['spiral_normal'].shape == (H, W, 3)
        net.fused_inference = False
        with pytest.raises(NotImplementedError):
            net.batchify_forward(dict(data), is_test=True)


@pytest.mark.gpu
def test_report():
    print('\n'.join(REPORT))


# ================================================================================================================ CPU
BAD_CFGS = lambda _C: (_C.NgpConfig(16, 2, 19, 16, 1.38191288, 64, 5, 2), _C.NgpConfig(16, 2, 19, 16, 1.38191288, 64, 0, 2),
                       _C.NgpConfig(16, 2, 19, 16, 1.38191288, 32, 1, 2), _C.NgpConfig(8, 2, 19, 16, 1.38191288, 64, 1, 2))


def test_density_grad_tc_validates_arguments_without_gpu():
    _C, _buf, p, cfg, tab = cpu_args()
    lib = _C.lib
    call = lambda cfg=cfg, tab=tab, w=p, pts=p, stride=3, n=4, nd=None, order=None, dens=p, grad=p: lib.xrb_ngp_density_grad_tc(cfg, tab, w, pts, stride, n, nd, order, dens, grad, None)
    assert call(cfg=None) == -1 and b'null' in lib.xrb_last_error()
    for bad in BAD_CFGS(_C):
        assert call(cfg=bad) == -2 and b'unsupported' in lib.xrb_last_error()
    assert call(n=-1) == -1 and b'bad size' in lib.xrb_last_error()
    assert call(stride=2) == -1 and b'bad size' in lib.xrb_last_error()
    for kw in (dict(tab=None), dict(w=None), dict(pts=None), dict(grad=None)):
        assert call(**kw) == -1 and b'null pointer' in lib.xrb_last_error(), kw
    assert call(w=C.c_void_p(p.value + 4)) == -1 and b'16-byte' in lib.xrb_last_error()
    assert call(tab=_C.NgpTable(None, None, 0)) == -1 and b'null hash table' in lib.xrb_last_error()
    assert call(tab=_C.NgpTable(p.value + 4, None, 0)) == -1 and b'aligned' in lib.xrb_last_error()
    assert call(tab=_C.NgpTable(p.value, None, 14)) == -1 and b'n_packed_levels' in lib.xrb_last_error()
    assert call(tab=_C.NgpTable(p.value, None, 6)) == -1 and b'cell image' in lib.xrb_last_error()
    assert call(n=0, tab=None, w=None, pts=None, dens=None, grad=None) == 0   # n == 0 touches no pointer


def test_render_normals_validates_arguments_without_gpu():
    _C, _buf, p, cfg, tab = cpu_args()
    lib = _C.lib
    bg = (C.c_float * 3)(0, 0, 0)

    def call(cfg=cfg, tab=tab, w=p, bf=p, o=p, d=p, n=4, ms=64, bgp=bg, rgb=p, alpha=p, depth=p, normal=p, ns=p, cnt=p, ws=p):
        return lib.xrb_ngp_render_normals(cfg, tab, w, bf, o, d, n, ms, 0.0, 1.0, 0.05, 1 / 256, 9121, 0, bgp, 2, 3, rgb, alpha, depth, normal, ns, cnt, ws, None, None, None)
    assert call(cfg=None) == -1 and b'null' in lib.xrb_last_error()
    for bad in BAD_CFGS(_C):
        assert call(cfg=bad) == -2 and b'unsupported' in lib.xrb_last_error()
    assert call(n=-1) == -1 and b'bad size' in lib.xrb_last_error()
    assert call(ms=0) == -1 and b'bad size' in lib.xrb_last_error()
    for kw in ('tab', 'w', 'bf', 'o', 'd', 'bgp', 'rgb', 'alpha', 'depth', 'normal', 'ns', 'cnt', 'ws'):
        assert call(**{kw: None}) == -1 and b'null pointer' in lib.xrb_last_error(), kw
    assert call(w=C.c_void_p(p.value + 4)) == -1 and b'16-byte' in lib.xrb_last_error()
    assert call(tab=_C.NgpTable(p.value + 4, None, 0)) == -1 and b'aligned' in lib.xrb_last_error()
    assert call(tab=_C.NgpTable(p.value, None, 6)) == -1 and b'cell image' in lib.xrb_last_error()
    assert call(n=0, tab=None, w=None, o=None, normal=None) == 0
    a256 = lambda b: (b + 255) // 256 * 256
    for n, ms in ((1, 1), (4096, 4096 * 64), (640000, 640000 * 64)):
        assert lib.xrb_ngp_render_normals_workspace(n, ms) == lib.xrb_ngp_render_workspace(n, ms) + a256(12 * ms)


def test_renderer_normals_checks_without_gpu():
    """NgpRenderer.render: normals need depth, and must be a float32 [n,3] tensor on the rays' device (checked before any launch); render_normals
    with fused_inference = False raises NotImplementedError"""
    from xrnerf_b200 import _C
    from xrnerf_b200.ngp import _depth_ptr
    n = 5
    good = torch.zeros((n, 3))
    assert _depth_ptr(good, n, good.device, 'normals', 3)
    for bad in (torch.zeros((n, 3), dtype=torch.float64), torch.zeros(n * 3), torch.zeros((n, 2)), torch.zeros((n + 1, 3)), 'x'):
        with pytest.raises(_C.XrbError, match='normals must be a float32 tensor of shape'):
            _depth_ptr(bad, n, good.device, 'normals', 3)
    with pytest.raises(_C.XrbError, match='depth must be a float32 tensor of 5 elements'):
        _depth_ptr(torch.zeros(4), n, good.device)
    from xrnerf_b200.ngp import NgpRenderer

    class _F:
        pass
    r = NgpRenderer(_F())
    with pytest.raises(_C.XrbError, match='normals need a depth output'):
        r.render(torch.zeros((n, 3)), torch.zeros((n, 3)), torch.zeros(8, dtype=torch.uint8), normals=good)
    from xrnerf_b200.registry.networks import HashNerfNetwork
    assert HashNerfNetwork.render_normals is False
    net = HashNerfNetwork.__new__(HashNerfNetwork)
    torch.nn.Module.__init__(net)
    net.sampler, net.render_normals, net.fused_inference = None, True, False
    with pytest.raises(NotImplementedError):
        net.batchify_forward({'rays_o': torch.zeros((n, 3))}, is_test=True)
