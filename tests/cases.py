"""The inputs the tests share: the model configs, the NGP field and NeRF network builders with their seeded weights, the NeRF views and z values,
the device copy and the host memory the CPU argument-validation tests pass. Nothing here asserts anything."""
import ctypes as C

import numpy as np
import torch

# ---------------------------------------------------------------------------------------------------------------- configs
NGP_MODEL = dict(   # configs/instant_ngp/nerf_blender_local01.py's model
    type='HashNerfNetwork', cfg=dict(phase='train', chunk=4096, bs_data='rays_o'),
    mlp=dict(type='HashNerfMLP', bound=1,
             embedder_pos=dict(n_input_dims=3, encoding_config=dict(otype='HashGrid', n_levels=16, n_features_per_level=2, log2_hashmap_size=19, base_resolution=16, interpolation='Linear')),
             embedder_dir=dict(n_input_dims=3, encoding_config=dict(otype='SphericalHarmonics', degree=4)),
             density_net=dict(n_input_dims=32, n_output_dims=16, network_config=dict(otype='FullyFusedMLP', activation='ReLU', output_activation='None', n_neurons=64, num_layers=1)),
             color_net=dict(n_output_dims=3, network_config=dict(otype='FullyFusedMLP', activation='ReLU', output_activation='None', n_neurons=64, num_layers=2))),
    sampler=dict(type='NGPGridSampler', update_grid_freq=16, update_block_size=5000000, n_rays_per_batch=4096, cone_angle_constant=0.00390625, near_distance=0.2,
                 target_batch_size=1 << 18, rgb_activation=2, density_activation=3),
    render=dict(type='HashNerfRender', bg_color=[0, 0, 0]))

# output_ch is read only without view directions (registry/mlps.py), so it changes nothing here; 5 is the reference configs' value
NERF_MLP = dict(type='NerfMLP', skips=[4], netdepth=8, netwidth=256, netchunk=1024 * 32, output_ch=5, use_viewdirs=True,
                embedder=dict(type='BaseEmbedder', i_embed=0, multires=10, multires_dirs=4))
NERF_MODEL = dict(type='NerfNetwork', cfg=dict(phase='train', N_importance=128, is_perturb=False, chunk=1024 * 32, bs_data='rays_o'), mlp=NERF_MLP, mlp_fine=NERF_MLP,
                  render=dict(type='NerfRender', white_bkgd=True, raw_noise_std=0))
MIP_MLP = dict(type='NerfMLP', skips=[4], netdepth=8, netwidth=256, netchunk=1024 * 32, use_viewdirs=True,
               embedder=dict(type='MipNerfEmbedder', min_deg_point=0, max_deg_point=16, min_deg_view=0, max_deg_view=4, use_viewdirs=True, append_identity=True))
MIP_CFG = dict(phase='train', ray_shape='cone', resample_padding=0.01, use_multiscale=False, coarse_loss_mult=0.1, num_levels=2, chunk=800, bs_data='rays_o')
MIP_RENDER = dict(type='MipNerfRender', white_bkgd=True, raw_noise_std=0, rgb_padding=0.001, density_bias=-1, density_activation='softplus')
MIP_MODEL = dict(type='MipNerfNetwork', cfg=MIP_CFG, mlp=MIP_MLP, render=MIP_RENDER)


# ---------------------------------------------------------------------------------------------------------------- memory
def dev(a, dt=None):
    """a numpy array on the GPU (converted to dt first when given)"""
    t = torch.from_numpy(np.ascontiguousarray(a))
    return (t if dt is None else t.to(dt)).cuda()


def bits(t):
    return t.contiguous().view(torch.int32)


def host_buffer(nbytes=4096):
    """(the ctypes buffer, a 256-byte aligned address of nbytes inside it): host memory a rejected call never dereferences; keep the buffer alive"""
    buf = (C.c_char * (nbytes + 256))()
    return buf, (C.addressof(buf) + 255) & ~255


def cpu_args():
    """(_C, buffer, aligned host pointer, the NGP_MODEL field's config, a table on that pointer) for the NGP entry points' argument checks"""
    from xrnerf_b200 import _C
    buf, a = host_buffer()
    p = C.c_void_p(a)
    return _C, buf, p, _C.NgpConfig(16, 2, 19, 16, 1.38191288, 64, 1, 2), _C.NgpTable(a, None, 0)


# ---------------------------------------------------------------------------------------------------------------- NGP
def load_ngp_weights(field, weights):
    """copy (table, density, colour) float32 arrays into an NgpField's parameters"""
    table, dens, color = weights
    with torch.no_grad():
        field.hash_params.copy_(torch.from_numpy(table)); field.density_params.copy_(torch.from_numpy(dens)); field.color_params.copy_(torch.from_numpy(color))
    return field


def ngp_field(dh=1, n_packed=6, seed=3):
    """an NgpField (colour net 2 hidden layers) with synth.ngp_weights(seed, hash_range 0.5, mlp_gain 2)"""
    from xrnerf_b200 import synth
    from xrnerf_b200.ngp import NgpField
    f = NgpField(density_hidden=dh, color_hidden=2, n_packed_levels=n_packed).cuda()
    return load_ngp_weights(f, synth.ngp_weights(seed=seed, dens_hidden=dh, hash_range=0.5, mlp_gain=2.0))


def ngp_network():
    """NGP_MODEL with the weights of ngp_field()"""
    from xrnerf_b200 import registry as R, synth
    net = R.build_network(NGP_MODEL).cuda()
    load_ngp_weights(net.mlp.field, synth.ngp_weights(seed=3, hash_range=0.5, mlp_gain=2.0))
    return net


def ngp_density_grad(field, x, with_density=True):
    """xrb_ngp_density_grad on x f32[n,3] through the C ABI (density=NULL when with_density is False)"""
    from xrnerf_b200 import _C
    field.refresh()
    n = len(x)
    xt = torch.from_numpy(np.ascontiguousarray(x)).cuda() if n else torch.empty((0, 3), device='cuda')
    dens = torch.full((n,), float('nan'), device='cuda')
    grad = torch.full((n, 3), float('nan'), device='cuda')
    _C.check(_C.lib.xrb_ngp_density_grad(field.cfg, field.tab, _C.ptr(field._dens16), _C.ptr(xt), 3, n, _C.f32(dens) if with_density else None, _C.f32(grad), _C.stream()),
             'density_grad')
    torch.cuda.synchronize()
    return dens.cpu().numpy().astype(np.float64), grad.cpu().numpy().astype(np.float64)


def random_points(n, seed):
    return np.random.default_rng(seed).uniform(1 / 64, 1 - 1 / 64, (n, 3)).astype(np.float32)


def face_points(grid, n_per, seed):
    """points with one coordinate exactly on a cell face of some level: fp32(scale_l * x + 0.5) is an integer"""
    rng = np.random.default_rng(seed)
    pts = []
    for l in (0, 2, 4, 5, 7, 9, 12, 15):
        for _ in range(n_per):
            k = int(rng.integers(2, int(grid.res[l]) - 1))
            x = np.float32((k - 0.5) / float(grid.scale[l]))
            for _ in range(64):
                px = grid.fma(l, np.array([x]))[0]
                if px == k:
                    break
                x = np.nextafter(x, np.float32(np.inf) if px < k else np.float32(-np.inf))
            if px != k:
                continue
            p = rng.uniform(1 / 64, 1 - 1 / 64, 3).astype(np.float32)
            p[rng.integers(0, 3)] = x
            if rng.uniform() < 0.3:                                          # on faces of two axes at once
                p[(np.argmax(p == x) + 1) % 3] = x
            pts.append(p)
    return np.stack(pts).astype(np.float32)


SPHERE_C, SPHERE_R, SPHERE_THR = 0.5, 0.3, 0.05   # raw density = fp16(r - |x - c|) at the level-4 grid points, level set raw = 0.05


def sphere_network():
    """(network, its Grid): level 4 (dense, resolution 59) holds fp16 samples of r - |x - c| in feature 0 and every other entry is 0; the density
    net has two hidden units, +enc[8] and -enc[8], and output row (+1, -1): the raw density is the trilinear interpolant of those samples"""
    from restate64 import Grid
    net = ngp_network()
    f = net.mlp.field
    grid = Grid(f.cfg)
    l, r = 4, int(grid.res[4])
    assert r == 59 and r ** 3 <= grid.off[5] - grid.off[4]
    i = np.arange(r)
    z, y, x = np.meshgrid(i, i, i, indexing='ij')                         # grid point (x, y, z) at index x + y r + z r^2
    pos = (np.stack([x, y, z], -1).astype(np.float64) - 0.5) / float(grid.scale[l])
    sdf = (SPHERE_R - np.linalg.norm(pos - SPHERE_C, axis=-1)).astype(np.float16).astype(np.float32)
    table = np.zeros(f.hash_params.numel(), np.float32)
    table[2 * grid.off[l]:2 * (grid.off[l] + r ** 3):2] = sdf.reshape(-1)
    dens = np.zeros(f.density_params.numel(), np.float32)
    dens[0 * 32 + 8], dens[1 * 32 + 8] = 1.0, -1.0                       # W_in [64][32]
    dens[64 * 32 + 0], dens[64 * 32 + 1] = 1.0, -1.0                     # W_out row 0
    with torch.no_grad():
        f.hash_params.copy_(torch.from_numpy(table)); f.density_params.copy_(torch.from_numpy(dens))
    return net, Grid.of(f)


# ---------------------------------------------------------------------------------------------------------------- NeRF / Mip-NeRF
def nerf_net(mip, seed=0, scale=1.0, **cfg):
    """NERF_MODEL or the Mip-NeRF model (cfg overrides its cfg), seeded; scale multiplies the weights of pts_linears 1..7 of every fused MLP"""
    from xrnerf_b200 import registry as R
    torch.manual_seed(seed)
    model = dict(MIP_MODEL, cfg=dict(MIP_CFG, **cfg)) if mip else dict(NERF_MODEL, cfg=dict(NERF_MODEL['cfg'], **cfg))
    net = R.build_network(model).cuda()
    if scale != 1.0:
        with torch.no_grad():
            for m in net._fused_mlps():
                for lin in m.pts_linears[1:]:
                    lin.weight.mul_(scale)
    return net


def nerf_mlp(cfg, seed, scaled=False):
    """a registry NerfMLP of cfg, seeded; scaled: weights doubled and biases uniform in [-0.5, 0.5], so units switch on and off across the box"""
    from xrnerf_b200 import registry as R
    torch.manual_seed(seed)
    mlp = R.build_mlp(cfg).cuda()
    if scaled:
        with torch.no_grad():
            for p in mlp.parameters():
                p.mul_(2.0) if p.dim() == 2 else p.uniform_(-0.5, 0.5)
    return mlp


def view_rays(H, W, seed, radii=True):
    """every pixel of an H x W view of a Blender spiral pose, Blender intrinsics scaled to the view (xrb_nerf_get_rays, GetRays + GetViewdirs)"""
    from xrnerf_b200 import _C, synth
    rng = np.random.default_rng(seed)
    pose = synth.pose_spherical(float(rng.uniform(-180, 180)), -30.0, 4.0)
    c2w = (C.c_float * 12)(*[float(v) for v in pose[:3, :4].reshape(-1)])
    n = H * W
    f = float(synth.FOCAL) * W / 800.0
    o, d, v = (torch.empty((n, 3), device='cuda') for _ in range(3))
    r = torch.empty((n, 1), device='cuda') if radii else None
    _C.check(_C.lib.xrb_nerf_get_rays(c2w, H, W, f, f, W / 2.0, H / 2.0, 0, None, n, _C.ptr(o), _C.ptr(d), _C.ptr(v), _C.ptr(r), _C.stream()), 'get_rays')
    return o, d, v, r


NEAR, FAR = 0.5, 3.0        # not the linspace(2, 6) the renderers default to


def zvals(n, s, near=NEAR, far=FAR, lindisp=True):
    from xrnerf_b200 import _C
    z = torch.empty((n, s), device='cuda')
    _C.check(_C.lib.xrb_nerf_zvals(n, s, float(near), float(far), int(lindisp), None, _C.ptr(z), _C.stream()), 'zvals')
    return z
