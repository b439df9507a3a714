"""Depth and opacity supervision on the H100: the geometry gradients of the NGP, NeRF and Mip-NeRF composites against float64 autograd, the loss kernel, the
NGP target depth, the trainer against the registry's autograd path, and that the terms train geometry (include/xrnerf_b200.h, "Depth and opacity
supervision").

Rounding bounds. A float64 restatement differs from an fp32 kernel by rounding only. Each fp32 sum or product chain of m terms errs by at most gamma(m, U32)
times the sum of its terms' absolute values (Higham, Accuracy and Stability of Numerical Algorithms, 3.1-3.4); a gradient entry is a few such chains over at
most one ray's K samples, so each entry is bounded by gamma(4 K + 64, U32) times MAG, the sum of absolute values of the products it is made of (the
64 covers the fixed number of roundings per sample: the activations, expf / __expf within 2 ulp plus the argument's own rounding, the scans' carries).
A composite's opacity 1 - exp(-sigma delta) (expf for NeRF / Mip-NeRF, __expf for NGP) has an ABSOLUTE error of a few units of U32 rather than a
relative one (the subtraction of two numbers near 1): ALPHA_ABS = 8 U32 each, which reaches every later transmittance, so the bounds add (K + 1) ALPHA_ABS
times the transmittance-weighted absolute terms.
"""
import numpy as np
import pytest
import torch

from cases import dev, view_rays, zvals
from restate64 import U32, gamma
from restate64_geom import geom_loss64, nerf_composite64, ngp_composite64, ngp_pad

pytestmark = pytest.mark.gpu

ALPHA_ABS = 8 * U32


def _call(name, *args):
    from xrnerf_b200 import _C
    _C.check(getattr(_C.lib, name)(*args, _C.stream()), name)


# ------------------------------------------------------------------------------------------------ NeRF / Mip-NeRF composite backward
def _nerf_case(mip, white, S, n=64, seed=0):
    g = torch.Generator(device='cuda').manual_seed(seed)
    raw = torch.randn((n, S, 4), device='cuda', generator=g)
    raw[..., 3] = raw[..., 3] * 2.0 + (1.0 if mip else 0.5)          # sigma * delta <= ~0.5 per interval (see the module docstring)
    z = zvals(n, S + 1 if mip else S)
    d = torch.randn((n, 3), device='cuda', generator=g)
    d = d / d.norm(dim=-1, keepdim=True) * (1.0 + 0.5 * torch.rand((n, 1), device='cuda', generator=g))
    grads = torch.randn((n, 3), device='cuda', generator=g), torch.randn(n, device='cuda', generator=g), torch.randn(n, device='cuda', generator=g)
    args = (int(mip), int(white), 0.001 if mip else 0.0, -1.0 if mip else 0.0, 4 if mip else 1)
    return raw, z, d, grads, args


def _nerf_backward(raw, z, d, grads, args, geom=True):
    from xrnerf_b200 import _C
    n, S = raw.shape[:2]
    out = torch.empty_like(raw)
    if geom:
        g_rgb, g_d, g_a = grads
        _call('xrb_nerf_composite_backward_geom', _C.ptr(raw), _C.ptr(z), _C.ptr(d), _C.ptr(g_rgb), _C.ptr(g_d), _C.ptr(g_a), n, S, *args, _C.ptr(out))
    else:
        _call('xrb_nerf_composite_backward', _C.ptr(raw), _C.ptr(z), _C.ptr(d), _C.ptr(grads[0]), n, S, *args, _C.ptr(out))
    return out


@pytest.mark.parametrize('mip', [False, True])
@pytest.mark.parametrize('white', [False, True])
@pytest.mark.parametrize('S', [45, 64])
def test_nerf_composite_geometry_grad_matches_f64(mip, white, S):
    """d_raw of grad_rgb . rgb + grad_depth . depth + grad_acc . acc against float64 autograd of the restated composite, entry by entry within
    gamma(4 S + 64) MAG; with both geometry gradients NULL, d_raw is bit-identical to xrb_nerf_composite_backward's"""
    from xrnerf_b200 import _C
    raw, z, d, grads, args = _nerf_case(mip, white, S)
    got = _nerf_backward(raw, z, d, grads, args).double().cpu()
    r64 = raw.double().cpu().requires_grad_(True)
    g_rgb, g_d, g_a = (t.double().cpu() for t in grads)
    rgb, depth, acc, sd = nerf_composite64(r64, z.cpu(), d.cpu(), mip, white, args[2], args[3], softplus=mip)
    ((g_rgb * rgb).sum() + (g_d * depth).sum() + (g_a * acc).sum()).backward()
    want = r64.grad
    # MAG: per sample |G_k| terms and the ray's sum of w_j |G_j| (the suffix is total - prefix), times |d sigma delta / d raw|, times 1 + sum of sigma delta
    # (the relative error of a transmittance formed from that sum or product)
    with torch.no_grad():
        r = r64.detach()
        zk = 0.5 * (z[:, 1:] + z[:, :-1]).double().cpu() if mip else z.double().cpu()
        a = r[..., 3] + args[3]
        dact = torch.sigmoid(a) if mip else (a > 0).double()
        zz = z.double().cpu()
        dl = (zz[:, 1:] - zz[:, :-1]) if mip else torch.cat([zz[:, 1:] - zz[:, :-1], torch.full_like(zz[:, :1], 1e10)], 1)
        dist = dl * d.double().cpu().norm(dim=-1, keepdim=True)
        alpha = 1 - torch.exp(-sd)
        T = torch.exp(-(torch.cumsum(sd, 1) - sd)) if mip else torch.cumprod(torch.cat([torch.ones_like(alpha[:, :1]), 1 - alpha + 1e-10], 1), 1)[:, :-1]
        w = alpha * T
        s = torch.sigmoid(r[..., :3])
        c = s * (1 + 2 * args[2]) - args[2]
        G = (g_rgb.abs()[:, None, :] * (c.abs() + float(white))).sum(-1) + g_d.abs()[:, None] * zk.abs() + g_a.abs()[:, None]
        tot = (w * G).sum(1, keepdim=True)
        growth = 1 + sd.clamp_max(1e3).sum(1, keepdim=True)
        mag = torch.zeros_like(want)
        # alpha = 1 - expf(-sigma delta) carries an absolute error (ALPHA_ABS, module docstring) into w and every later transmittance
        wt = w + T * (S + 1) * ALPHA_ABS / gamma(4 * S + 64, U32)
        mag[..., :3] = g_rgb.abs()[:, None, :] * wt[..., None] * s * (1 - s) * (1 + 2 * args[2])
        mag[..., 3] = dist.clamp_max(1e10) * dact * (T * G + tot)
        mag = mag * growth[..., None]
    bound = gamma(4 * S + 64, U32) * mag
    err = (got - want).abs()
    ratio = (err / bound.clamp_min(1e-300)).reshape(-1, 4).max(0).values
    assert bool((err <= bound).all()), ('err / bound per channel', ratio.tolist(), float(err.max()), float(want.abs().max()))
    base = _nerf_backward(raw, z, d, grads, args, geom=False)
    nulls = torch.empty_like(raw)
    n = raw.shape[0]
    _call('xrb_nerf_composite_backward_geom', _C.ptr(raw), _C.ptr(z), _C.ptr(d), _C.ptr(grads[0]), None, None, n, S, *args, _C.ptr(nulls))
    assert torch.equal(base.view(torch.int32), nulls.view(torch.int32))


# ------------------------------------------------------------------------------------------------ NGP composite forward / backward
def _ngp_setup(scene, n, T):
    """the march + compaction of n scene rays (ray-order truncation at T rows) and the field's raw rows, zero padded to T"""
    import xrnerf_b200.raymarch_cuda as rm
    from xrnerf_b200.ngp import NgpField
    f = NgpField(seed=5).cuda()
    with torch.no_grad():
        f.hash_params.mul_(3000.0)
    o, d, bf = dev(scene['rays_o'][:n]), dev(scene['rays_d'][:n]), dev(scene['bitfield'])
    rm.reset_rng()
    coords = torch.zeros((n * 64, 7), device='cuda'); ridx = torch.zeros((n, 1), dtype=torch.int32, device='cuda'); ns = torch.zeros((n, 2), dtype=torch.int32, device='cuda')
    cnt = torch.zeros(2, dtype=torch.int32, device='cuda')
    rm.rays_sampler_api(o, d, bf, None, None, None, 0.0, 1.0, 0.05, 1.0 / 256, coords, ridx, ns, cnt)
    cc = torch.zeros((T, 7), device='cuda'); nsc = torch.zeros((n, 2), dtype=torch.int32, device='cuda')
    rc = torch.zeros(1, dtype=torch.int32, device='cuda'); sc = torch.zeros(1, dtype=torch.int32, device='cuda')
    rm.compacted_coord_api(None, coords, ns, None, 2, 3, 0.0, 1.0, cc, nsc, rc, sc)
    n_c = min(int(sc.item()), T)
    f.impl = 1
    raw = torch.zeros((T, 4), device='cuda')
    with torch.no_grad():
        raw[:n_c] = f(cc[:n_c, :3], cc[:n_c, 4:])
    return f, o, d, bf, cc, ns, nsc, n_c, raw


@pytest.mark.parametrize('n', [1, 33, 1000, 4096])
@pytest.mark.parametrize('T', [1 << 16, 20000])
def test_ngp_composite_geometry_matches_f64(scene, n, T):
    """MODE 4 forward: rgb bit-identical to the colour-only forward, depth and alpha bit-identical to xrb_ngp_render_depth's for the rays the compaction kept
    whole. Geometry backward: colour channels bit-identical to the colour-only backward, every channel within the module's bound of float64 autograd of the
    restated composite (loss_scale and the l1 term included)"""
    from xrnerf_b200 import _C
    from xrnerf_b200.ngp import NgpRenderer
    f, o, d, bf, cc, ns, nsc, n_c, raw = _ngp_setup(scene, n, T)
    bg = torch.rand((n, 3), device='cuda', generator=torch.Generator(device='cuda').manual_seed(1))
    rgb0, rgb4 = torch.zeros((n, 3), device='cuda'), torch.zeros((n, 3), device='cuda')
    alpha, depth = torch.zeros(n, device='cuda'), torch.zeros(n, device='cuda')
    _call('xrb_rm_calc_rgb_forward', _C.ptr(raw), _C.ptr(cc), _C.ptr(ns), _C.ptr(nsc), _C.ptr(bg), n, 2, 3, _C.ptr(rgb0))
    _call('xrb_rm_calc_rgb_forward_geom', _C.ptr(raw), _C.ptr(cc), _C.ptr(ns), _C.ptr(nsc), _C.ptr(bg), _C.ptr(o), _C.ptr(d), n, 0.0, 1.0, 2, 3, _C.ptr(rgb4), _C.ptr(alpha),
          _C.ptr(depth))
    assert torch.equal(rgb0, rgb4)
    whole = (nsc[:, 0] == ns[:, 0])
    dep_r = torch.zeros(n, device='cuda')
    _, alpha_r, ns_r, _ = NgpRenderer(f).render(o, d, bf, depth=dep_r)
    assert torch.equal(ns_r[:, 0], ns[:, 0])
    assert torch.equal(alpha[whole], alpha_r[:, 0][whole]) and torch.equal(depth[whole], dep_r[whole])
    # backward: random upstream gradients, l1 switched on (grid mean below the minimum optical thickness)
    g = torch.Generator(device='cuda').manual_seed(2)
    gr, gd, ga = torch.randn((n, 3), device='cuda', generator=g), torch.randn(n, device='cuda', generator=g), torch.randn(n, device='cuda', generator=g)
    mean = torch.zeros(1, device='cuda')
    d0, d4 = torch.zeros((T, 4), device='cuda'), torch.zeros((T, 4), device='cuda')
    _call('xrb_rm_calc_rgb_backward', _C.ptr(raw), _C.ptr(nsc), _C.ptr(cc), _C.ptr(gr), _C.ptr(rgb0), _C.ptr(mean), n, 2, 3, _C.ptr(d0))
    _call('xrb_rm_calc_rgb_backward_geom', _C.ptr(raw), _C.ptr(nsc), _C.ptr(cc), _C.ptr(gr), _C.ptr(rgb4), _C.ptr(mean), _C.ptr(o), _C.ptr(d), 0.0, 1.0, _C.ptr(depth), _C.ptr(alpha),
          _C.ptr(gd), _C.ptr(ga), n, 2, 3, _C.ptr(d4))
    assert torch.equal(d0[:n_c, :3], d4[:n_c, :3])
    dn = torch.zeros((T, 4), device='cuda')
    _call('xrb_rm_calc_rgb_backward_geom', _C.ptr(raw), _C.ptr(nsc), _C.ptr(cc), _C.ptr(gr), _C.ptr(rgb4), _C.ptr(mean), _C.ptr(o), _C.ptr(d), 0.0, 1.0, _C.ptr(depth), _C.ptr(alpha),
          None, None, n, 2, 3, _C.ptr(dn))
    assert torch.equal(d0[:n_c], dn[:n_c])
    # float64 autograd of the restatement
    r64 = raw[:n_c].double().cpu().requires_grad_(True)
    args = (cc[:n_c].cpu().numpy(), ns.cpu().numpy(), nsc.cpu().numpy(), bg.cpu().numpy(), o.cpu().numpy(), d.cpu().numpy(), 0.0, 1.0)
    rgb, A, D, (w, Ta, t, dt), m = ngp_composite64(r64, args[0], args[1], args[2], args[3], args[4], args[5], args[6], args[7])
    gr64, gd64, ga64 = gr.double().cpu(), gd.double().cpu(), ga.double().cpu()
    ((gr64 * rgb).sum() + (gd64 * D).sum() + (ga64 * A).sum()).backward()
    loss_scale = 128.0 / n
    want = loss_scale * r64.grad
    want[:, 3] -= torch.where(r64.detach()[:, 3] < 0, 1e-4, 0.0)
    got = d4[:n_c].double().cpu()
    # MAG per row, gathered from the [ray, slot] layout of the restatement
    idx, valid = ngp_pad(args[2], n_c)
    with torch.no_grad():
        rr = r64.detach()
        c = torch.sigmoid(rr[:, :3])
        K = idx.shape[1]
        rows = torch.from_numpy(idx[valid])
        c_pad = torch.zeros(w.shape + (3,), dtype=torch.float64); c_pad[m] = c[rows]
        G = (gr64.abs()[:, None, :] * c_pad).sum(-1) + gd64.abs()[:, None] * t.abs() + ga64.abs()[:, None]
        tot = (w * G).sum(1, keepdim=True) + Ta[:, -1:] * (gr64.abs() * torch.from_numpy(args[3]).abs()).sum(1, keepdim=True)
        sig = torch.zeros_like(w); sig[m] = torch.exp(rr[rows, 3])
        Tb = Ta + w
        mag_w = loss_scale * sig * dt * ((Ta * G + tot) * (1 + (K + 1) * ALPHA_ABS / gamma(4 * K + 64, U32)))
        mag_c = loss_scale * (gr64.abs()[:, None, :] * (w + Tb * (K + 1) * ALPHA_ABS / gamma(4 * K + 64, U32))[..., None] * c_pad * (1 - c_pad))
        mag = torch.zeros_like(want)
        mag[rows, 3] = mag_w[m] + 1e-4
        mag[rows, :3] = mag_c[m]
    bound = gamma(4 * K + 64, U32) * mag
    err = (got - want).abs()
    assert bool((err <= bound).all()), (float((err - bound).max()), float(err.max()), int((err > bound).sum()))


# ------------------------------------------------------------------------------------------------ loss kernel
@pytest.mark.parametrize('mean', [0, 1])
def test_geom_loss_matches_f64(mean):
    """loss and gradients against the float64 restatement, including every mask: non-finite depth, depth <= 0, truncated rays"""
    from xrnerf_b200 import _C
    n = 5000
    g = np.random.default_rng(3)
    depth, alpha = g.uniform(0.1, 2.0, n).astype(np.float32), g.uniform(0, 1, n).astype(np.float32)
    td, ta = g.uniform(0.1, 2.0, n).astype(np.float32), g.uniform(0, 1, n).astype(np.float32)
    td[::7] = np.nan; td[1::11] = np.inf; td[2::13] = 0.0; td[3::17] = -1.0
    td[4::19] = depth[4::19]                                            # |D - D*| = 0: subgradient 0
    ns = np.stack([g.integers(1, 50, n), np.zeros(n)], 1).astype(np.int32)
    nsc = ns.copy(); nsc[5::9, 0] -= 1                                  # truncated
    keep = nsc[:, 0] == ns[:, 0]
    wd, wa = 0.7, 3.0
    loss = torch.full((1,), 0.25, device='cuda')
    gd, ga = torch.full((n,), 9.0, device='cuda'), torch.full((n,), 9.0, device='cuda')
    t = [dev(v) for v in (depth, alpha, td, ta, ns, nsc)]
    _call('xrb_geom_loss_grad', *[_C.ptr(v) for v in t], n, wd, wa, mean, _C.ptr(gd), _C.ptr(ga), _C.ptr(loss))
    L, Gd, Ga = geom_loss64(depth, alpha, td, ta, keep, wd, wa, mean)
    # the loss: two fp32 sums of n terms and a scale; the gradients: one or two roundings each
    mag = wd * np.abs(np.where(keep & np.isfinite(td) & (td > 0), depth - np.nan_to_num(td), 0)).sum() + wa * (np.where(keep, alpha - ta, 0) ** 2).sum()
    mag /= (max(int(keep.sum()), 1) if mean else 1)
    assert abs(float(loss.item()) - 0.25 - L) <= gamma(n + 8, U32) * (mag + 0.25)
    assert np.all(np.abs(gd.cpu().numpy() - Gd) <= gamma(3, U32) * np.abs(Gd))
    assert np.all(np.abs(ga.cpu().numpy() - Ga) <= gamma(4, U32) * np.abs(Ga))
    dropped = ~keep
    assert (gd.cpu().numpy()[dropped] == 0).all() and (ga.cpu().numpy()[dropped] == 0).all()
    assert (gd.cpu().numpy()[~np.isfinite(td) | (td <= 0)] == 0).all()


# ------------------------------------------------------------------------------------------------ target depth
def test_ngp_batch_depth_planes():
    """xrb_ngp_batch_depth against numpy on synth poses: a plane at camera z-depth Z gives t = 0.33 Z |(x, y, 1)| within a few ulps, and o + t d lies at
    camera depth 0.33 Z"""
    from xrnerf_b200 import synth
    from xrnerf_b200.data import NgpRaySource
    I, H, W = 3, 20, 30
    poses = np.ascontiguousarray(synth.spiral_poses_ngp(I).astype(np.float32))
    Z = np.array([1.5, 2.0, 3.25], np.float32)
    depths = np.broadcast_to(Z[:, None, None], (I, H, W)).copy()
    K = [[25.0, 0, W / 2.0 - 0.3], [0, 27.0, H / 2.0 + 0.2], [0, 0, 1]]
    src = NgpRaySource(poses, np.zeros((I, H, W, 4), np.float32), K, depths=depths).cuda()
    rows = torch.arange(I * H * W, device='cuda')
    b = src.rows(rows)
    t = b['target_depth'][:, 0].double().cpu().numpy()
    r = np.arange(I * H * W); img, pix = r // (H * W), r % (H * W)
    j, i = pix // W, pix % W
    x = (i.astype(np.float32) + np.float32(0.5) - np.float32(K[0][2])) / np.float32(K[0][0])
    y = (j.astype(np.float32) + np.float32(0.5) - np.float32(K[1][2])) / np.float32(K[1][1])
    want = 0.33 * Z[img].astype(np.float64) * np.sqrt(x.astype(np.float64) ** 2 + y.astype(np.float64) ** 2 + 1.0)
    assert np.all(np.abs(t - want) <= 4 * np.spacing(want.astype(np.float32)).astype(np.float64))
    # the ray's point at t sits on the plane: its component along the camera axis (the third rotation row of the pose) is 0.33 Z
    dd = b['rays_d'].double().cpu().numpy()
    axis = poses[img, 2, :].astype(np.float64)
    axis /= np.linalg.norm(axis, axis=-1, keepdims=True)
    assert np.allclose((t[:, None] * dd * axis).sum(-1), 0.33 * Z[img], rtol=1e-5)


# ------------------------------------------------------------------------------------------------ trainer
def test_trainer_geometry_step_matches_autograd_path(scene):
    """a depth- and opacity-weighted NgpTrainer.step against the registry path (_CalcRgbGeomFn + 5 x Huber + the geometry loss through autograd), within
    the tolerances of test_trainer_step_matches_autograd_path (T = 20000: truncated rays, which the geometry terms drop)"""
    from xrnerf_b200.ngp import NgpField
    from xrnerf_b200.train import NgpTrainer, huber5_grad
    from xrnerf_b200.registry.renders import _CalcRgbGeomFn
    from xrnerf_b200.registry.networks import _GeomLossFn
    import xrnerf_b200.raymarch_cuda as rm
    T, n = 20000, 4096
    torch.manual_seed(0)
    f = NgpField(seed=5).cuda()
    with torch.no_grad():
        f.hash_params.mul_(3000.0)
    o, d, bf = dev(scene['rays_o']), dev(scene['rays_d']), dev(scene['bitfield'])
    target = torch.rand((n, 3), device='cuda'); bg = torch.rand((n, 3), device='cuda')
    td = torch.rand(n, device='cuda') + 0.3; td[::5] = float('nan'); ta = torch.rand(n, device='cuda')
    wd, wa = 2.0, 7.0
    rm.reset_rng()
    coords = torch.zeros((n * 64, 7), device='cuda'); ridx = torch.zeros((n, 1), dtype=torch.int32, device='cuda'); ns = torch.zeros((n, 2), dtype=torch.int32, device='cuda')
    cnt = torch.zeros(2, dtype=torch.int32, device='cuda')
    rm.rays_sampler_api(o, d, bf, None, None, None, 0.0, 1.0, 0.05, 1.0 / 256, coords, ridx, ns, cnt)
    cc = torch.zeros((T, 7), device='cuda'); nsc = torch.zeros((n, 2), dtype=torch.int32, device='cuda'); rc = torch.zeros(1, dtype=torch.int32, device='cuda')
    sc = torch.zeros(1, dtype=torch.int32, device='cuda')
    rm.compacted_coord_api(None, coords, ns, None, 2, 3, 0.0, 1.0, cc, nsc, rc, sc)
    n_c = min(int(sc.item()), T)
    assert int((nsc[:, 0] != ns[:, 0]).sum()) > 0
    f.impl = 1
    raw = f(cc[:n_c, :3], cc[:n_c, 4:])
    rgb, alpha, depth = _CalcRgbGeomFn.apply(raw, cc, ns, nsc, bg, torch.ones(1, device='cuda'), 2, 3, (0.0, 1.0), o, d)
    loss_ref = huber5_grad(rgb, target)[0] + _GeomLossFn.apply(depth, alpha, td, ta, ns, nsc, wd, wa, False)
    loss_ref.backward()
    g_ref = [p_.grad.clone() for p_ in (f.hash_params, f.density_params, f.color_params)]
    tr = NgpTrainer(f, bf, n, target_batch_size=T, bwd_impl=1, lr=0.0, depth_weight=wd, opacity_weight=wa)
    loss = float(tr.step(o, d, target, bg, target_depth=td, target_alpha=ta))
    torch.cuda.synchronize()
    assert abs(loss - float(loss_ref)) <= 1e-4 * abs(float(loss_ref))
    whole = nsc[:, 0] == ns[:, 0]
    assert bool((tr.grad_depth[~whole] == 0).all()) and bool((tr.grad_alpha[~whole] == 0).all())     # truncated rays: no geometry gradient
    for name, a, b in zip(('table', 'density', 'color'), tr.grads, g_ref):
        scale = float(b.abs().max())
        err = (a - b).abs()
        assert scale > 0
        assert float(err.max()) <= 1e-5 * scale, (name, float(err.max()), scale)
        assert float(torch.sqrt((err.double() ** 2).sum() / (b.double() ** 2).sum())) <= 3e-3, name


def test_trainer_zero_weights_is_todays_step(scene):
    """with both weights 0 the trainer runs today's launch sequence: over 3 steps the same kernels in the same order as a trainer built without the new
    kwargs (targets passed or not), and in the first step (same weights in both) dL/draw bit for bit, the loss and the parameter gradients within the
    spread of their atomic accumulation. The 5 x Huber sum and the field backward's gradients are accumulated with atomics in arrival order, so two runs of
    the same step differ in the last bits, and the parameters after a step (Adam divides by sqrt(v), eps = 1e-15) are not comparable bit for bit."""
    from xrnerf_b200.ngp import NgpField
    from xrnerf_b200.train import NgpTrainer
    n = 4096
    o, d, bf = dev(scene['rays_o']), dev(scene['rays_d']), dev(scene['bitfield'])
    target = torch.full((n, 3), 0.5, device='cuda'); bg = torch.zeros((n, 3), device='cuda')
    td, ta = torch.rand(n, device='cuda') + 0.3, torch.rand(n, device='cuda')
    runs = []
    for kw, step_kw in (({}, {}), (dict(depth_weight=0.0, opacity_weight=0.0), dict(target_depth=td, target_alpha=ta))):
        f = NgpField(seed=5).cuda()
        tr = NgpTrainer(f, bf, n, target_batch_size=1 << 16, **kw)
        with torch.profiler.profile(activities=[torch.profiler.ProfilerActivity.CUDA]) as prof:
            loss = tr.step(o, d, target, bg, **step_kw).clone()
            torch.cuda.synchronize()
            draw = tr.draw[:int(tr.compacted_samples())].clone()
            grads = [g.clone() for g in tr.grads]
            for _ in range(2):
                tr.step(o, d, target, bg, **step_kw)
            torch.cuda.synchronize()
        names = [e.name for e in sorted(prof.events(), key=lambda e: e.time_range.start) if e.device_type == torch.autograd.DeviceType.CUDA]
        runs.append((names, loss, draw, grads))
    (na, la, da, ga), (nb, lb, db, gb) = runs
    assert len(na) > 15 and na == nb
    assert torch.equal(da.view(torch.int32), db.view(torch.int32))
    # the 5 x Huber sum is accumulated with one atomic add per block, in arrival order: its 3 n positive terms bound the spread
    assert abs(float(la) - float(lb)) <= gamma(3 * n, U32) * float(la)
    for name, a, b in zip(('table', 'density', 'color'), ga, gb):   # the tolerances of test_trainer_step_matches_autograd_path for the wgmma backward
        scale = float(b.abs().max())
        err = (a - b).abs()
        assert scale > 0 and float(err.max()) <= 1e-5 * scale, (name, float(err.max()), scale)
        assert float(torch.sqrt((err.double() ** 2).sum() / (b.double() ** 2).sum())) <= 3e-3, name


# ------------------------------------------------------------------------------------------------ supervision trains geometry
def test_ngp_depth_and_opacity_supervision_learn_the_sphere(scene):
    """a fresh field learns a teacher's depth and silhouette from the geometry terms alone (constant colour target equal to the background): the mean depth
    error on the training rays falls at least 5x, and alpha separates the silhouette (> 0.5 inside, < 0.5 outside) on >= 95 % of the rays"""
    from cases import sphere_network
    from xrnerf_b200.ngp import NgpField, NgpRenderer
    from xrnerf_b200.train import NgpTrainer
    net, _ = sphere_network()
    teacher = net.mlp.field
    with torch.no_grad():
        teacher.density_params[64 * 32 + 0] *= 100.0                  # raw density 100 (r - |x - c|): an opaque sphere, empty space around it
        teacher.density_params[64 * 32 + 1] *= 100.0
    teacher.mark_dirty()
    n = 4096
    o, d = dev(scene['rays_o'][:n]), dev(scene['rays_d'][:n])
    ones = torch.full_like(dev(scene['bitfield']), 255)
    dstar = torch.zeros(n, device='cuda')
    _, astar, _, _ = NgpRenderer(teacher, samples_per_ray_budget=1024).render(o, d, ones, depth=dstar)
    astar = astar[:, 0].clone()
    inside = astar > 0.5
    assert 0.1 < float(inside.float().mean()) < 0.9                   # the rays see both the sphere and around it
    dstar = torch.where(inside, dstar, torch.full_like(dstar, float('nan')))   # depth where the sphere is hit, no depth elsewhere
    student = NgpField(seed=11).cuda()

    def measure():
        dep = torch.zeros(n, device='cuda')
        _, a, _, _ = NgpRenderer(student, samples_per_ray_budget=1024).render(o, d, ones, depth=dep)
        a = a[:, 0]
        return float((dep[inside] - dstar[inside]).abs().mean()), float(((a > 0.5) == inside).float().mean())
    err0, _ = measure()
    tr = NgpTrainer(student, ones, n, target_batch_size=1 << 22, samples_per_ray_budget=1024, depth_weight=1.0, opacity_weight=10.0)
    col = torch.full((n, 3), 0.5, device='cuda')
    for _ in range(300):
        tr.step(o, d, col, col, target_depth=dstar, target_alpha=astar)
    torch.cuda.synchronize()
    err1, sep = measure()
    print(f'sphere supervision: mean |D - D*| {err0:.4f} -> {err1:.4f}, silhouette separated on {100 * sep:.1f} % of rays')
    assert err1 * 5 <= err0
    assert sep >= 0.95


# ------------------------------------------------------------------------------------------------ NeRF / Mip-NeRF train_step
@pytest.mark.parametrize('mip', [False, True])
def test_nerf_train_step_geometry_terms_descend(mip):
    """one train_step with depth and opacity weights (large beside the colour term, so they dominate the gradient), then a small SGD step along -grad,
    lowers the depth and opacity terms"""
    from cases import nerf_net
    kw = dict(depth_loss_weight=5.0, opacity_loss_weight=5.0) if mip else dict(depth_loss_weight=5.0, opacity_loss_weight=5.0, N_importance=0)
    net = nerf_net(mip, seed=0, **kw)
    H = W = 32
    o, d, v, r = view_rays(H, W, seed=4)
    n = H * W
    S = 64
    t = torch.linspace(0., 1., S + 1 if mip else S, device='cuda')
    z = (2.0 * (1. - t) + 6.0 * t).expand(n, t.numel()).contiguous()
    data = {'rays_o': o[None], 'rays_d': d[None], 'viewdirs': v[None], 'z_vals': z[None], 'target_s': torch.rand((1, n, 3), device='cuda'),
            'target_depth': (3.0 + torch.rand((1, n, 1), device='cuda')), 'target_alpha': torch.ones((1, n, 1), device='cuda')}
    if mip:
        data['radii'] = r[None]
    else:
        data['pts'] = (o[:, None, :] + d[:, None, :] * z[:, :, None])[None]
    opt = torch.optim.SGD(net.parameters(), lr=1e-3)

    def terms():
        out = net.train_step(dict(data), opt)
        return out, out['log_vars']['loss_depth'], out['log_vars']['loss_opacity']
    out, ld0, lo0 = terms()
    assert not net.render.geometry_grad                                # the flag is set for the step only
    opt.zero_grad(set_to_none=True)
    out['loss'].backward()
    gsq = sum(float((p.grad.double() ** 2).sum()) for p in net.parameters() if p.grad is not None)
    assert gsq > 0
    with torch.no_grad():
        for p in net.parameters():
            if p.grad is not None:
                p.add_(p.grad, alpha=-1e-3 / max(gsq, 1.0) ** 0.5)
    net._mark_dirty()
    _, ld1, lo1 = terms()
    assert ld1 + lo1 < ld0 + lo0, (ld0, lo0, ld1, lo1)
