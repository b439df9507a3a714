"""NeRF / Mip-NeRF normal maps: the NerfMLP's density gradient at every sample on tensor cores (xrb_nerf_density_grad_rays,
xrb_mip_density_grad_rays, NerfMLP.density_grad_rays), the normal composite (xrb_nerf_composite_normals), the renderers' normals=True and
NerfNetwork.render_normals. include/xrnerf_b200.h ("NeRF / Mip-NeRF normal maps") states the contract.

Gradient restatement (numpy, float64) over the kernel's fp16 weights, the fp16 encodings read back from the tile image and the forward's fp16
roundings. A ReLU network's gradient depends on its inputs only through the masks, so with the masks agreed the kernel's g is a sum of products:
per W^T step a 256-term tensor-core sum (256 2^-22 per term), per staging of d(density)/d(hidden) one fp16 rounding (2^-11 relative; the per-row
power-of-two scale puts the row's largest entry in [2^14, 2^15), so an entry in fp16's subnormal range is off by at most 2^-25, 2^-39 of the row's
largest entry), two fp32 terms summed for the encoding gradient and the encoding derivative's fp32 terms (sinf / cosf / expf to a few ulp, 2^-21 each).
The bound is that relative factor times the same chain on absolute values, plus the subnormal terms carried down it, plus the float64 restatement's
own gamma. A unit whose pre-activation lies within the forward's bound of 0 (K 2^-22 sum |w| |x| plus the fp16 roundings around it) has an ambiguous
mask; with 8 x 256 units nearly every row has one, so instead of excluding rows the bound adds what each such unit can change: its |dZ| carried
down the absolute chain. Every row must lie within the bound. Nothing in it is fitted to a run.
"""
import ctypes as C

import numpy as np
import pytest
import torch

from cases import MIP_MLP, NERF_MLP, bits, nerf_net, view_rays, zvals
from restate64 import GAMMA_TC as TC, U16, columns, decode, f16, w16

REPORT = []


def _rays(mip, n, s, seed, d_zero=False):
    """n rays of an 800-wide Blender view with s samples each (z [n,s], or [n,s+1] interval ends and radii for Mip-NeRF)"""
    o, d, v, r = view_rays(n // 800 + 3, 800, seed)
    o, d, v, r = o[:n].contiguous(), d[:n].contiguous(), v[:n].contiguous(), r[:n].reshape(-1).contiguous()
    if d_zero:
        d = torch.zeros_like(d)
        r = torch.zeros_like(r)
    w = s + 1 if mip else s
    z = zvals(n, w, 2.0, 6.0, False) if w > 1 else torch.full((n, 1), 3.0, device='cuda')
    return o, d, v, z, (r if mip else None)


def _grad(mlp, o, d, v, z, r):
    from xrnerf_b200.nerf import encode_rays
    enc = encode_rays(mlp, o, d, v, z, r)
    dens, g = mlp.density_grad_rays(o, d, z, r, enc=enc)
    return enc, dens, g


def _enc_rows(enc, n_rows, ic):
    """the fp16 point-encoding columns of the tile image, float64 [n_rows, ic]"""
    return columns(enc, n_rows, (ic + 63) // 64 + 1, 0, ic).cpu().numpy()


def _positions(mip, o, d, z, r, e):
    """float64 of the fp32 positions the encoder forms, and the encoding's Jacobian J [n, ic, 3] there (float64)"""
    o, d, z = (t.cpu().numpy() for t in (o, d, z))
    if not mip:
        s = z.shape[1]
        p = (o[:, None, :] + (d[:, None, :] * z[..., None]).astype(np.float32)).astype(np.float32).reshape(-1, 3).astype(np.float64)
        n = len(p)
        J = np.zeros((n, 63, 3))
        for a in range(3):
            J[:, a, a] = 1.0
            for b in range(10):
                J[:, 3 + 6 * b + a, a] = 2.0 ** b * np.cos(2.0 ** b * p[:, a])
                J[:, 6 + 6 * b + a, a] = -2.0 ** b * np.sin(2.0 ** b * p[:, a])
        return p, J, np.zeros(n)
    r = r.cpu().numpy()
    t0, t1 = z[:, :-1].astype(np.float64), z[:, 1:].astype(np.float64)
    mu, hw = (t0 + t1) / 2, (t1 - t0) / 2
    den = 3 * mu ** 2 + hw ** 2
    t_mean = mu + 2 * mu * hw ** 2 / den
    t_var = hw ** 2 / 3 - 4 / 15 * (hw ** 4 * (12 * mu ** 2 - hw ** 2)) / den ** 2
    r_var = r[:, None].astype(np.float64) ** 2 * (mu ** 2 / 4 + 5 / 12 * hw ** 2 - 4 / 15 * hw ** 4 / den)
    dd = d.astype(np.float64)
    dm = np.maximum(1e-10, (dd ** 2).sum(1))
    mean = (dd[:, None, :] * t_mean[..., None] + o[:, None, :]).reshape(-1, 3)
    cov = (t_var[..., None] * dd[:, None, :] ** 2 + r_var[..., None] * (1 - dd[:, None, :] ** 2 / dm[:, None, None])).reshape(-1, 3)
    n = len(mean)
    J = np.zeros((n, 96, 3))
    for k in range(16):
        sc = 2.0 ** (e.min_deg + k)
        for a in range(3):
            hv = 0.5 * cov[:, a] * sc * sc
            f = np.where(hv <= 20, np.exp(-hv), 0.0) * sc
            J[:, 3 * k + a, a] = f * np.cos(mean[:, a] * sc)
            J[:, 48 + 3 * k + a, a] = -f * np.sin(mean[:, a] * sc)
    return mean, J, cov


def _restated(mlp, enc16, J):
    """float64 gradient, its bound and the rows whose masks are unambiguous"""
    W = [w16(l).cpu().numpy() for l in mlp.pts_linears]
    b = [f16(l.bias.detach().float().cpu().numpy()) for l in mlp.pts_linears]
    wa = mlp.alpha_linear.weight.detach().float().cpu().numpy()[0].astype(np.float64)
    ic = mlp.input_ch
    masks, ambs, ok = [], [], np.ones(len(enc16), bool)
    h, eh = enc16, np.zeros_like(enc16)                        # layer input and its spread against the kernel's
    for l in range(8):
        x, ex = (np.concatenate([enc16, h], 1), np.concatenate([np.zeros_like(enc16), eh], 1)) if l == 5 else (h, eh)
        z = x @ W[l].T
        ez = (np.abs(W[l]) @ ex.T).T + x.shape[1] * TC * (np.abs(x) + ex) @ np.abs(W[l]).T
        # the kernel's activation fp16(fp16(acc) + fp16(b)) lies between these two (rounding is monotone): its mask is decided where they agree
        lo = f16(f16(z - ez * (1 + 1e-9)) + b[l])
        hi = f16(f16(z + ez * (1 + 1e-9)) + b[l])
        amb = (lo > 0) != (hi > 0)
        ok &= ~amb.any(1)
        m = hi > 0                                             # an undecided unit is taken live here; amb records that the kernel may have it dead
        masks.append(m); ambs.append(amb)
        # the next layer reads the fp16 activation at the restated sum; where lo == hi (every decided unit but those with an fp16 rounding boundary
        # inside the bracket) it is the kernel's exactly, so the spread is carried only through the units where they differ
        h = np.where(m, f16(f16(z) + b[l]), 0.0)
        eh = np.where(m, hi - np.maximum(lo, 0), 0.0) * (lo != hi)
    # gu: what the undecided units can change. A unit the kernel may have dead contributes at most its own |dZ| (bounded by the absolute chain
    # before the mask), carried down the absolute chain like every other term
    g, ga = masks[7] * wa[None], masks[7] * np.abs(wa)[None]
    gs, gu = np.zeros_like(g), ambs[7] * np.abs(wa)[None]
    e5 = e5a = e5s = e5u = None
    for l in range(7, 0, -1):
        Wh = W[l][:, ic:] if l == 5 else W[l]
        if l == 5:
            Wp = W[5][:, :ic]
            e5, e5a, e5s, e5u = g @ Wp, ga @ np.abs(Wp), (gs + 2.0 ** -39 * ga.max(1, keepdims=True)) @ np.abs(Wp), gu @ np.abs(Wp)
        gs = masks[l - 1] * ((gs + 2.0 ** -39 * ga.max(1, keepdims=True)) @ np.abs(Wh))
        gu = masks[l - 1] * (gu @ np.abs(Wh)) + ambs[l - 1] * (ga @ np.abs(Wh))
        g, ga = masks[l - 1] * (g @ Wh), masks[l - 1] * (ga @ np.abs(Wh))
    e = g @ W[0] + e5
    ea = ga @ np.abs(W[0]) + e5a
    es = (gs + 2.0 ** -39 * ga.max(1, keepdims=True)) @ np.abs(W[0]) + e5s
    eu = gu @ np.abs(W[0]) + e5u
    gx = np.einsum('nc,nca->na', e, J)
    gxa = np.einsum('nc,nca->na', ea, np.abs(J))
    gxs = np.einsum('nc,nca->na', es + eu, np.abs(J))
    rel = (1 + U16) ** 8 * (1 + 256 * TC) ** 9 * (1 + 2.0 ** -23) * (1 + 2.0 ** -21) ** 2 * (1 + 100 * 2.0 ** -24) - 1
    return gx, rel * gxa + (1 + rel) * gxs + 2.0 ** -50 * gxa, ok


CASES = [(mip, sc) for mip in (False, True) for sc in (1.0, 2.0 ** -6)]
IDS = [f'{"mip" if m else "nerf"}-{"default" if s == 1 else "scaled"}' for m, s in CASES]


@pytest.mark.gpu
@pytest.mark.parametrize('mip,scale', CASES, ids=IDS)
def test_density_bit_identical_to_the_inference_kernel(mip, scale):
    """density_out == raw[:, 3] of xrb_nerf_mlp_forward on the same encoding image, for 1, 127, 129 and 5000 rows (ragged S); a row does not depend on
    the batch split (200 / 333 rays against one batch)"""
    from xrnerf_b200.nerf_mlp import nerf_mlp_forward_tiles
    net = nerf_net(mip, seed=1, scale=scale)
    mlp = net.mlp
    image, bias = mlp._packed()
    for n, s in ((1, 1), (1, 127), (3, 43), (50, 100)):
        o, d, v, z, r = _rays(mip, n, s, seed=n)
        enc, dens, g = _grad(mlp, o, d, v, z, r)
        raw = nerf_mlp_forward_tiles(image, bias, enc, n * s, mlp.input_ch, mlp.input_ch_dirs)
        assert torch.equal(bits(dens), bits(raw[:, 3].contiguous())), (n, s)
        assert torch.isfinite(g).all()
    o, d, v, z, r = _rays(mip, 533, 37, seed=9)
    _, d_all, g_all = _grad(mlp, o, d, v, z, r)
    for lo, hi in ((0, 200), (200, 533)):
        _, dp, gp = _grad(mlp, o[lo:hi], d[lo:hi], v[lo:hi], z[lo:hi], None if r is None else r[lo:hi])
        assert torch.equal(bits(dp), bits(d_all[lo * 37:hi * 37])) and torch.equal(bits(gp), bits(g_all[lo * 37:hi * 37]))


@pytest.mark.gpu
@pytest.mark.parametrize('mip,scale', CASES, ids=IDS)
def test_gradient_against_float64(mip, scale):
    net = nerf_net(mip, seed=2, scale=scale)
    mlp = net.mlp
    n, s = 40, 64
    o, d, v, z, r = _rays(mip, n, s, seed=3)
    enc, _, g = _grad(mlp, o, d, v, z, r)
    _, J, _ = _positions(mip, o, d, z, r, mlp.embedder)
    e16 = _enc_rows(enc, n * s, mlp.input_ch)
    ref, bound, ok = _restated(mlp, e16, J)
    g = g.cpu().numpy().astype(np.float64)
    excluded = int((~ok).sum())
    REPORT.append((mip, scale, excluded, n * s))
    within = (np.abs(g - ref) <= bound).all(1)
    print(f'{"mip" if mip else "nerf"} scale {scale}: {excluded} of {n * s} rows have a mask the bound cannot decide; {int(within.sum())} rows within it')
    # 8 x 256 units: nearly every row has some unit whose pre-activation lies within the forward's bound of 0, so excluding those rows would leave
    # none (DESIGN 4.8). The bound carries what each undecided unit can change instead, so every row must lie within it
    assert within.all(), float(within.mean())
    if scale != 1.0:      # d(density)/d(hidden) spans at least 2^42 from dZ_7 to dZ_0 (seven W^T steps at 2^-6 each), and g is resolved and finite
        assert np.isfinite(g).all() and (np.abs(g) > 0).all(1).mean() >= 0.9


@pytest.mark.gpu
@pytest.mark.parametrize('mip', [False, True])
def test_agrees_with_the_training_kernel_gradient(mip):
    """rays with d = 0 (and radius 0): every sample sits at o, so g must match nerf_train.density_grad at o (Mip-NeRF: sigma 0). Both paths stage
    fp16 through the same eight layers with tensor-core sums, so each is within this file's float64 bound of the restatement; they must agree within
    twice it (the training path's fixed 2^12 staging scale adds its subnormal term, negligible at these magnitudes)"""
    from xrnerf_b200 import nerf_train
    net = nerf_net(mip, seed=4)
    mlp = net.mlp
    n, s = 64, 2
    o, d, v, z, r = _rays(mip, n, s, seed=5, d_zero=True)
    o = o + torch.linspace(-0.5, 0.5, n, device='cuda')[:, None]                 # distinct points
    enc, dens, g = _grad(mlp, o, d, v, z, r)
    with torch.no_grad():
        _, gt = nerf_train.density_grad(mlp, o.repeat_interleave(s, 0).contiguous(), sigma=0.0 if mip else None)
    _, J, _ = _positions(mip, o, d, z, r, mlp.embedder)
    _, bound, ok = _restated(mlp, _enc_rows(enc, n * s, mlp.input_ch), J)
    within = ((g - gt).abs().cpu().numpy() <= 2 * bound).all(1)
    assert within.all(), float(within.mean())


@pytest.mark.gpu
@pytest.mark.parametrize('mip', [False, True])
def test_normals_change_nothing_else(mip):
    from xrnerf_b200.nerf import MipNerfRenderer, NerfRenderer
    net = nerf_net(mip, seed=6)
    o, d, v, z, r = _rays(mip, 700, 64, seed=7)
    R = MipNerfRenderer(net, ray_batch=256) if mip else NerfRenderer(net, ray_batch=256)
    args = (o, d, v, r) if mip else (o, d, v)
    a = R.render(*args, z_vals=z, depth=True)
    b = R.render(*args, z_vals=z, depth=True, normals=True)
    assert set(b) == set(a) | {'normal'} and b['normal'].shape == (700, 3)
    for k in a:
        assert torch.equal(bits(a[k]), bits(b[k])), k
    assert torch.isfinite(b['normal']).all()


@pytest.mark.gpu
@pytest.mark.parametrize('n', [1, 33, 1000])
def test_composite_against_float64(n):
    from xrnerf_b200.nerf import composite_normals
    g = torch.Generator(device='cuda').manual_seed(n)
    s = 57
    w = torch.rand((n, s), device='cuda', generator=g) * 0.05
    w[::5] = 0.0                                             # rays with all-zero weights
    gr = torch.randn((n * s, 3), device='cuda', generator=g) * 10.0 ** torch.randint(-20, 20, (n * s, 1), device='cuda', generator=g)
    gr[::7] = 0.0
    out = torch.empty((n, 3), device='cuda')
    composite_normals(w, gr, out)
    G = gr.cpu().double().numpy()
    nrm = np.linalg.norm(G, axis=1, keepdims=True)
    nk = np.where(nrm > 0, -G / np.where(nrm > 0, nrm, 1), 0.0).reshape(n, s, 3)
    W = w.cpu().double().numpy()
    ref = (W[..., None] * nk).sum(1)
    bound = ((s + 2) * 2.0 ** -24 / (1 - (s + 2) * 2.0 ** -24) + 4 * 2.0 ** -24) * (W[..., None] * np.abs(nk)).sum(1) + 1e-30
    assert (np.abs(out.cpu().double().numpy() - ref) <= bound).all()
    assert (out[::5] == 0).all()


def _octahedron(net, c):
    """density = c - (|x| + |y| + |z|) through the trunk: layer 0 forms relu(+-x_a) from encoding columns 0..2, layers 1..7 pass the 6 units through
    (skip columns zero), alpha_linear is -1 on them with bias c; every weight is 0 or +-1, exact in fp16"""
    mlp = net.mlp
    with torch.no_grad():
        for lin in mlp.pts_linears:
            lin.weight.zero_(); lin.bias.zero_()
        W0 = mlp.pts_linears[0].weight
        for a in range(3):
            W0[2 * a, a], W0[2 * a + 1, a] = 1.0, -1.0
        ic = mlp.input_ch
        for l in range(1, 8):
            off = ic if l == 5 else 0
            for u in range(6):
                mlp.pts_linears[l].weight[u, off + u] = 1.0
        mlp.alpha_linear.weight.zero_(); mlp.alpha_linear.weight[0, :6] = -1.0
        mlp.alpha_linear.bias.fill_(c)
    mlp.mark_dirty()


def _octant_rays(n, samples):
    """n rays, each from a point outside the octahedron in one of the 8 octants towards a point of that octant's face (both in the closed, convex
    octant, so every sample stays in it): (rays_o, rays_d, the octant's signs, z) with `samples` z values from 1 to 4"""
    rng = np.random.default_rng(0)
    sgn = torch.tensor(rng.choice([-1.0, 1.0], (n, 3)), device='cuda', dtype=torch.float32)
    o = sgn * torch.tensor([2.0, 1.5, 1.0], device='cuda')
    tgt = sgn * torch.tensor(rng.dirichlet([4, 4, 4], n) * 0.5, device='cuda', dtype=torch.float32)
    d = tgt - o
    d = (d / d.norm(dim=1, keepdim=True)).contiguous()
    z = torch.linspace(1.0, 4.0, samples, device='cuda')[None].repeat(n, 1).contiguous()
    return o.contiguous(), d, sgn, z


@pytest.mark.gpu
def test_octahedron_normals_nerf():
    """samples near a face of the octahedron |x| + |y| + |z| = 0.5, away from its edges, in all 8 octants (so both relu(x_a) and relu(-x_a) units are
    live somewhere): n = -g / |g| is the face's outward normal (+-1, +-1, +-1)/sqrt(3) to 1e-3 rad, and it faces the camera (n . d < 0)"""
    net = nerf_net(False, seed=8)
    _octahedron(net, 0.5)
    o, d, sgn, z = _octant_rays(512, 64)
    _, g = net.mlp.density_grad_rays(o, d, z)
    nk = -g / g.norm(dim=1, keepdim=True)
    p = (o[:, None] + d[:, None] * z[..., None]).reshape(-1, 3)
    s = sgn.repeat_interleave(64, 0)
    face = (p * s > 0.02).all(1) & ((p.abs().sum(1) - 0.5).abs() < 0.3)
    cosang = (nk[face] * s[face] * 3 ** -0.5).sum(1)
    assert face.sum() > 1000 and (cosang > np.cos(1e-3)).all()
    assert ((nk[face] * d.repeat_interleave(64, 0)[face]).sum(1) < 0).all()
    assert len(torch.unique(s[face], dim=0)) == 8


@pytest.mark.gpu
def test_octahedron_normals_mip():
    """the same weights on the Mip-NeRF IPE with min_deg 0: encoding columns 0..2 are f_a sin(mu_a), f_a = exp(-cov_a / 2), so the density is
    c - sum_a f_a |sin(mu_a)| and g_a = -sign(column a) f_a cos(mu_a) (0 where the fp16 column is 0). The expected direction is that restatement, in
    float64 at the frustum Gaussians' means and covariances and with the signs of the fp16 columns read back from the encoding image; every sample's
    normal is within 1e-3 rad of it, and where |mu_a| < 1 on all axes and the sample is near the level set it faces the camera."""
    from xrnerf_b200.nerf import encode_rays
    net = nerf_net(True, seed=9)
    _octahedron(net, 0.5)
    mlp = net.mlp
    o, d, sgn, z = _octant_rays(256, 65)
    r = torch.full((256,), 2e-3, device='cuda')
    enc = encode_rays(mlp, o, d, d, z, r)
    _, g = mlp.density_grad_rays(o, d, z, r, enc=enc)
    mean, _, cov = _positions(True, o, d, z, r, mlp.embedder)
    col = _enc_rows(enc, 256 * 64, 96)[:, :3]
    want = -np.sign(col) * np.exp(-0.5 * cov) * np.cos(mean)
    g = g.cpu().double().numpy()
    live = np.linalg.norm(want, axis=1) > 0
    assert live.mean() > 0.99
    cosang = (g[live] * want[live]).sum(1) / (np.linalg.norm(g[live], axis=1) * np.linalg.norm(want[live], axis=1))
    assert (cosang > np.cos(1e-3)).all(), float(cosang.min())
    dd = d.repeat_interleave(64, 0).cpu().double().numpy()
    near = (np.abs(mean) < 1).all(1) & (np.abs(np.abs(np.sin(mean)).sum(1) - 0.5) < 0.3) & (mean * sgn.repeat_interleave(64, 0).cpu().numpy() > 0.02).all(1)
    assert near.sum() > 500 and ((-g[near] * dd[near]).sum(1) < 0).all()


@pytest.mark.gpu
def test_network_api_and_whole_view():
    """val_step / test_step keys with render_normals on and off; a whole 800 x 800 NeRF view with normals; NotImplementedError without the fused path"""
    H, W = 24, 40
    net = nerf_net(False, seed=11)
    o, d, v, _ = view_rays(H, W, 5, radii=False)
    z = zvals(H * W, 64)
    view = {'rays_o': o, 'rays_d': d, 'viewdirs': v, 'z_vals': z, 'src_shape': torch.tensor([H, W, 3])}
    net.set_val_pipeline(lambda item: dict(view))
    images = torch.rand((1, 2, H, W, 3), device='cuda')
    out = net.val_step({'poses': torch.zeros((1, 2, 4, 4)), 'images': images, 'spiral_poses': torch.zeros((1, 1, 4, 4))})
    assert 'normals' not in out
    net.render_normals = True
    out2 = net.val_step({'poses': torch.zeros((1, 2, 4, 4)), 'images': images, 'spiral_poses': torch.zeros((1, 1, 4, 4))})
    assert len(out2['normals']) == 2 and len(out2['spiral_normals']) == 1 and out2['normals'][0].shape == (H, W, 3)
    assert torch.equal(out2['rgbs'][0], out['rgbs'][0])
    net.phase = 'test'
    t = net.val_step({'pose': torch.zeros((1, 4, 4)), 'image': images[:, 0], 'idx': torch.tensor([3])})
    assert t['normal'].shape == (H, W, 3)
    net.fused_inference = False
    with pytest.raises(NotImplementedError):
        net.batchify_forward(dict(view), is_test=True)
    mip = nerf_net(True, seed=12)
    mip.render_normals = True
    _, _, _, r = view_rays(H, W, 6)
    mview = dict(view, radii=r, z_vals=zvals(H * W, 129))
    mip.set_val_pipeline(lambda item: dict(mview))
    mo = mip.val_step({'poses': torch.zeros((1, 1, 4, 4)), 'images': images[:, :1]})
    assert mo['normals'][0].shape == (H, W, 3)
    # Mip-NeRF use_multiscale: evaluate_once returns the normal map as a fifth element, val_step as normals / normal
    ms = nerf_net(True, seed=13, use_multiscale=True)
    px = lambda t: t.reshape(1, H, W, -1)
    mdata = {'rays_o': px(o), 'rays_d': px(d), 'viewdirs': px(v), 'radii': px(r), 'z_vals': px(mview['z_vals']), 'image': images[:, 0], 'idx': torch.tensor([[4]])}
    assert len(ms.evaluate_once(dict(mdata))) == 4
    ms.render_normals = True
    rgb, _, _, idx, normal = ms.evaluate_once(dict(mdata))
    assert normal.shape == (H, W, 3) and idx == 4 and torch.isfinite(normal).all()
    val = ms.val_step(dict(mdata))
    assert set(val) == {'rgbs', 'gt_imgs', 'disps', 'normals'} and torch.equal(val['normals'][0], normal) and torch.equal(val['rgbs'][0], rgb)
    ms.phase = 'test'
    t = ms.val_step(dict(mdata))
    assert set(t) == {'rgb', 'gt_img', 'disp', 'idx', 'normal'} and torch.equal(t['normal'], normal)
    # a whole 800 x 800 view
    big = nerf_net(False, seed=17)
    big.render_normals = True
    H = W = 800
    o, d, v, _ = view_rays(H, W, 8, radii=False)
    bview = {'rays_o': o, 'rays_d': d, 'viewdirs': v, 'z_vals': zvals(H * W, 64, 2.0, 6.0, False), 'src_shape': torch.tensor([H, W, 3])}
    big.set_val_pipeline(lambda item: dict(bview))
    from xrnerf_b200.nerf import bytes_per_ray, ray_batch_size
    image = torch.rand((1, 1, H, W, 3), device='cuda')
    big.val_step({'poses': torch.zeros((1, 1, 4, 4)), 'images': image})
    torch.cuda.synchronize()
    base = torch.cuda.memory_allocated()
    torch.cuda.reset_peak_memory_stats()
    bo = big.val_step({'poses': torch.zeros((1, 1, 4, 4)), 'images': image})
    torch.cuda.synchronize()
    peak = torch.cuda.max_memory_allocated() - base
    rows = [64, 192]
    n = H * W
    bound = ray_batch_size(rows, 63, normals=True) * bytes_per_ray(rows, 63, normals=True) + 128 * 256 + n * 2 * 24 + 3 * n * 12 + n * 12 + (24 << 20)
    assert peak <= bound, (peak, bound)
    assert bo['normals'][0].shape == (H, W, 3) and torch.isfinite(bo['normals'][0]).all()


# ------------------------------------------------------------------------------------------------ CPU

def test_entry_points_validate_arguments_without_gpu():
    from xrnerf_b200 import _C
    L = _C.lib
    p = C.c_void_p(16)
    nerf = lambda n, s, ic=63, icd=27, w=p, g=p: L.xrb_nerf_density_grad_rays(w, g, p, p, p, p, p, n, s, ic, icd, None, p, None)
    mip = lambda n, s, ic=96, lo=0, hi=16, r=p: L.xrb_mip_density_grad_rays(p, p, p, p, p, p, p, r, n, s, ic, 27, lo, hi, None, p, None)
    assert nerf(-1, 4) == -1 and nerf(4, 0) == -1 and mip(-1, 4) == -1 and mip(4, 0) == -1
    assert nerf(4, 4, ic=96) == -2 and nerf(4, 4, icd=28) == -2 and mip(4, 4, ic=63) == -2 and mip(4, 4, hi=10) == -2
    assert nerf(0, 4) == 0 and mip(0, 4) == 0
    assert nerf(4, 4, w=None) == -1 and nerf(4, 4, g=None) == -1 and mip(4, 4, r=None) == -1
    assert L.xrb_nerf_density_grad_rays(C.c_void_p(17), p, p, p, p, p, p, 4, 4, 63, 27, None, p, None) == -1       # misaligned image
    assert L.xrb_nerf_composite_normals(p, p, -1, 4, p, None) == -1 and L.xrb_nerf_composite_normals(p, p, 4, 0, p, None) == -1
    assert L.xrb_nerf_composite_normals(None, None, 0, 4, None, None) == 0 and L.xrb_nerf_composite_normals(p, None, 4, 4, p, None) == -1


def test_ray_batch_size_with_normals_without_gpu():
    from xrnerf_b200.nerf import RAY_BATCH_BYTES, bytes_per_ray, ray_batch_size
    assert bytes_per_ray([64, 192], 63) == 55304 and bytes_per_ray([128, 128], 96) == 55304
    assert bytes_per_ray([64, 192], 63, normals=True) == 55304 + 12 * 192 and bytes_per_ray([128, 128], 96, normals=True) == 55304 + 12 * 128
    assert ray_batch_size([64, 192], 63) == 38784
    for rows, ic in (([64, 192], 63), ([128, 128], 96)):
        b = ray_batch_size(rows, ic, normals=True)
        assert b % 128 == 0 and b * bytes_per_ray(rows, ic, True) <= RAY_BATCH_BYTES < (b + 128) * bytes_per_ray(rows, ic, True)


def _unslab64(buf, n):
    h = np.frombuffer(buf, np.float16).reshape(n // 8, 8, 4, 8)
    rows = np.arange(n)
    out = np.zeros((n, 32), np.float16)
    for c in range(4):
        out[:, 8 * c:8 * c + 8] = h[rows >> 3, rows & 7, c ^ ((rows >> 1) & 3)]
    return out


def _unslab(buf, n):
    """an [n x 64] fp16 slab with the tile images' 128-byte swizzle"""
    from xrnerf_b200.nerf_train import Img
    return decode(Img(torch.frombuffer(bytearray(buf), dtype=torch.uint8), n * 128, 0, 1), 1, rows=n).numpy()


@pytest.mark.parametrize('mip', [False, True])
def test_grad_image_packer_without_gpu(mip):
    """pack_nerf_mlp_grad's slabs are fp16 W^T, in the stream order of the gradient kernel; pack_nerf_mlp's stream image is what it was"""
    from xrnerf_b200 import registry as R
    from xrnerf_b200.nerf_mlp import pack_nerf_mlp, pack_nerf_mlp_grad
    torch.manual_seed(3)
    mlp = R.build_mlp(MIP_MLP if mip else NERF_MLP)
    ic = mlp.input_ch
    npt = 128 if mip else 64
    img = pack_nerf_mlp_grad(mlp).numpy().tobytes()
    W = [l.weight.detach().numpy() for l in mlp.pts_linears]
    off = 0

    def wide(wt):
        nonlocal off
        for j in range(4):
            for kh in range(2):
                got = _unslab64(img[off:off + 16384], 256)
                assert np.array_equal(got, wt[:, 64 * j + 32 * kh:64 * j + 32 * kh + 32].astype(np.float16))
                off += 16384

    def points(wp):
        nonlocal off
        wt = np.zeros((npt, 256), np.float32)
        wt[:ic] = wp.T
        for j in range(4):
            got = _unslab(img[off:off + npt * 128], npt)
            assert np.array_equal(got, wt[:, 64 * j:64 * j + 64].astype(np.float16))
            off += npt * 128
    wide(W[7].T); wide(W[6].T); points(W[5][:, :ic]); wide(W[5][:, ic:].T)
    for l in (4, 3, 2, 1):
        wide(W[l].T)
    points(W[0])
    assert off == len(img)
    image, bias = pack_nerf_mlp(mlp)
    aux = 2 if mip else 1
    first = _unslab64(image.numpy().tobytes()[:16384], 256)
    assert np.array_equal(first, np.pad(W[0], ((0, 0), (0, 64 * aux - ic)))[:, :32].astype(np.float16))
    assert len(image) == 16384 * (2 * aux + 2 * 4 * 6 + 2 * (4 + aux) + 2 * 4) + 128 * 128 * (5) + 16 * 128 * 2
