"""NeRF mesh export: the NerfMLP's raw alpha on a lattice (xrb_nerf_density_lattice, NerfMLP.density_lattice), its gradient with respect to the
position (NerfMLP.density_grad: the training kernels + xrb_nerf_posenc_grad), and NerfNetwork.extract_mesh / extract_colored_mesh.

The lattice is compared bit for bit with the inference kernel on the posenc_tiles encoding of the same points. The gradient is compared entry by entry
with a float64 restatement over the kernels' own fp16 weights, activations and ReLU masks. The mesh path is checked on a NerfMLP whose raw alpha is
r - (|x| + |y| + |z|): an octahedron with known volume, area and normals."""
import ctypes as C
import math

import numpy as np
import pytest
import torch
from cases import NERF_MLP, host_buffer, nerf_mlp
from restate64 import U16, U32, area, check_closed_oriented, columns, euler, lattice_coords, lattice_points, mc_oracle, trunk_grad, w16


# ---------------------------------------------------------------------------------------------------------------- CPU: argument checks
def test_density_lattice_validates_arguments_without_gpu():
    from xrnerf_b200 import _C
    lib = _C.lib
    lo, hi = _C.float3((-1.5, -1.5, -1.5)), _C.float3((1.5, 1.5, 1.5))
    buf, a = host_buffer()
    p = C.c_void_p(a)
    for n in ((1, 4, 4), (4, 1025, 4), (4, 4, -1)):
        assert lib.xrb_nerf_density_lattice(p, p, 63, 10, *n, lo, hi, p, None) == -1 and b'bad size' in lib.xrb_last_error()
    assert lib.xrb_nerf_density_lattice(p, p, 96, 10, 4, 4, 4, lo, hi, p, None) == -2 and b'input_ch 63' in lib.xrb_last_error()
    assert lib.xrb_nerf_density_lattice(p, p, 63, 8, 4, 4, 4, lo, hi, p, None) == -2
    for b0, b1 in (((0, 0, 0), (1, 0, 1)), ((0, 0, 0), (1, 1, math.inf)), ((2, 0, 0), (1, 1, 1))):
        assert lib.xrb_nerf_density_lattice(p, p, 63, 10, 4, 4, 4, _C.float3(b0), _C.float3(b1), p, None) == -1 and b'box' in lib.xrb_last_error()
    assert lib.xrb_nerf_density_lattice(p, p, 63, 10, 4, 4, 4, None, hi, p, None) == -1
    assert lib.xrb_nerf_density_lattice(None, None, 63, 10, 0, 4, 4, lo, hi, None, None) == 0            # empty lattice: a no-op
    assert lib.xrb_nerf_density_lattice(None, p, 63, 10, 4, 4, 4, lo, hi, p, None) == -1 and b'null' in lib.xrb_last_error()
    assert lib.xrb_nerf_density_lattice(p, p, 63, 10, 4, 4, 4, lo, hi, None, None) == -1
    odd = C.c_void_p(a + 4)
    assert lib.xrb_nerf_density_lattice(odd, p, 63, 10, 4, 4, 4, lo, hi, p, None) == -1 and b'aligned' in lib.xrb_last_error()


def test_posenc_grad_validates_arguments_without_gpu():
    from xrnerf_b200 import _C
    lib = _C.lib
    buf, a = host_buffer()
    p = C.c_void_p(a)
    assert lib.xrb_nerf_posenc_grad(p, -1, 10, p, 2, p, p, None) == -1 and b'bad size' in lib.xrb_last_error()
    assert lib.xrb_nerf_posenc_grad(p, 4, 11, p, 2, p, p, None) == -1
    assert lib.xrb_nerf_posenc_grad(p, 4, 10, p, 0, p, p, None) == -1 and lib.xrb_nerf_posenc_grad(p, 4, 10, p, 5, p, p, None) == -1
    assert lib.xrb_nerf_posenc_grad(None, 0, 10, None, 2, None, None, None) == 0                          # n == 0: a no-op
    for args in ((None, p, p, p), (p, None, p, p), (p, p, None, p), (p, p, p, None)):
        assert lib.xrb_nerf_posenc_grad(args[0], 4, 10, args[1], 2, args[2], args[3], None) == -1 and b'null' in lib.xrb_last_error()
    assert lib.xrb_nerf_posenc_grad(p, 4, 10, C.c_void_p(a + 4), 2, p, p, None) == -1


def test_raw_density_threshold_relu_and_softplus():
    """NerfRender's activations by name (the NGP sampler's integer codes stop at 3), with density_bias"""
    from xrnerf_b200.mesh import raw_density_threshold
    assert raw_density_threshold(50.0, 'relu') == 50.0
    assert raw_density_threshold(50.0, 'relu', density_bias=-1.0) == 51.0
    assert raw_density_threshold(0.0, 'relu', density_bias=0.5) == -0.5
    for s in (1e-3, 0.5, 3.0, 19.9):
        v = raw_density_threshold(s, 'softplus')
        assert abs(np.log1p(np.exp(v)) - s) <= 1e-12 * max(1.0, s)
        assert raw_density_threshold(s, 'softplus', density_bias=2.0) == v - 2.0
    assert raw_density_threshold(50.0, 'softplus') == 50.0                                              # softplus(v) = v above 20
    for s, act in ((-1.0, 'relu'), (0.0, 'softplus'), (-2.0, 'softplus'), (math.nan, 'softplus'), (math.inf, 'relu'), (1.0, 'tanh'), (1.0, 4)):
        with pytest.raises(ValueError):
            raw_density_threshold(s, act)


def test_mip_network_and_cpu_mlp_refuse_mesh_export():
    from xrnerf_b200 import registry as R
    from xrnerf_b200.registry.networks import MipNerfNetwork
    net = object.__new__(MipNerfNetwork)
    with pytest.raises(NotImplementedError, match='frusta'):
        net.extract_mesh(64)
    with pytest.raises(NotImplementedError, match='frusta'):
        net.extract_colored_mesh(64)
    mlp = R.build_mlp(NERF_MLP)
    with pytest.raises(NotImplementedError, match='CUDA'):
        mlp.density_lattice((4, 4, 4), ((0, 0, 0), (1, 1, 1)))
    with pytest.raises(NotImplementedError, match='CUDA'):
        mlp.density_grad(torch.zeros(4, 3))


# ---------------------------------------------------------------------------------------------------------------- GPU helpers
def _infer(mlp, pts, dirs):
    """raw f32[n,4] of the inference kernel on the posenc_tiles encoding of (pts, dirs)"""
    from xrnerf_b200 import _C
    from xrnerf_b200.nerf_mlp import nerf_mlp_forward_tiles
    n = pts.shape[0]
    enc = torch.empty(_C.lib.xrb_nerf_enc_image_bytes(n, 63), dtype=torch.uint8, device='cuda')
    _C.check(_C.lib.xrb_nerf_posenc_tiles(_C.f32(pts.contiguous()), _C.f32(dirs.contiguous()), n, 1, 10, 4, _C.ptr(enc), _C.stream()), 'posenc_tiles')
    image, bias = mlp._packed()
    return nerf_mlp_forward_tiles(image, bias, enc, n, 63, 27)


# ---------------------------------------------------------------------------------------------------------------- lattice: bit identity
@pytest.mark.gpu
@pytest.mark.parametrize('shape', [(2, 2, 2), (7, 5, 3), (9, 33, 17), (128, 128, 128)])
@pytest.mark.parametrize('scaled', [False, True])
def test_density_lattice_equals_inference_kernel_bit_for_bit(shape, scaled):
    """(nz, ny, nx); totals 8, 105, 5049 and 2^21: three are not a multiple of the 128-row tile. Boxes with negative coordinates."""
    mlp = nerf_mlp(NERF_MLP, 11, scaled)
    for box in (((-1.5, -1.5, -1.5), (1.5, 1.5, 1.5)), ((-2.0, -0.25, -3.5), (-0.5, 1.75, -1.0))):
        with torch.no_grad():
            vol = mlp.density_lattice(shape, box)
            pts = lattice_points(shape, box)
            dirs = torch.nn.functional.normalize(torch.randn_like(pts), dim=-1)
            raw = _infer(mlp, pts, dirs)
        torch.cuda.synchronize()
        assert vol.shape == shape
        assert torch.equal(vol.reshape(-1), raw[:, 3]), (shape, box, float((vol.reshape(-1) - raw[:, 3]).abs().max()))


# ---------------------------------------------------------------------------------------------------------------- gradient: float64 restatement
def _kernel_forward(mlp, pts):
    """the training kernels' forward as density_grad runs it: encoding (fp16) and the 8 hidden activations (fp16) as float64"""
    from xrnerf_b200 import _C
    from xrnerf_b200 import nerf_train as T
    n = pts.shape[0]
    nt = (n + 127) // 128
    S = mlp._tg_slabs
    enc = T.Img.new(nt, 2, 'cuda')
    vd = torch.zeros((1, 3), device='cuda')
    _C.check(_C.lib.xrb_nerf_posenc_tiles(_C.f32(pts), _C.f32(vd), n, n, 10, 4, _C.ptr(enc.buf), _C.stream()), 'posenc_tiles')
    H = [T.Img.new(nt, 4, 'cuda') for _ in range(8)]
    T._fwd(n, S, 'pts0', [enc.sub(0, 1)], H[0])
    for l in range(1, 8):
        T._fwd(n, S, f'pts{l}', ([enc.sub(0, 1), H[l - 1]] if l == 5 else [H[l - 1]]), H[l])
    return columns(enc.buf, n, 2, 0, 63), [columns(h.buf, n, 4, 0, 256) for h in H]


def _restated_grad(mlp, pts, enc, H):
    """float64 d(raw alpha)/d(position) over the fp16 weights, with the kernels' ReLU masks (fp16 activation > 0); also the same chain on absolute
    values, which bounds the rounding error"""
    e, ea = trunk_grad(mlp, H, 63)
    out, outa = e[:, :3].clone(), ea[:, :3].clone()
    for b in range(10):
        y = (pts * 2.0 ** b).double()                         # the kernel's fp32 argument, exact
        out += 2.0 ** b * (torch.cos(y) * e[:, 3 + 6 * b:6 + 6 * b] - torch.sin(y) * e[:, 6 + 6 * b:9 + 6 * b])
        outa += 2.0 ** b * (torch.cos(y).abs() * ea[:, 3 + 6 * b:6 + 6 * b] + torch.sin(y).abs() * ea[:, 6 + 6 * b:9 + 6 * b])
    return out, outa


# Rounding count of the kernel chain: the staged dZ of alpha_linear and of each of the 8 trunk layers is rounded to fp16 once (9 roundings of 2^-11),
# each fp32 contraction of <= 320 terms adds 320 * 2^-24 per layer (9 layers), the d(encoding) blocks are summed and scaled once in fp32, and the final
# contraction over 61 columns adds 64 * 2^-24 plus the sincosf error (2 ulp). |kernel - float64| <= GAMMA * (the same chain on absolute values) + ABS,
# ABS for staged values in fp16's subnormal range (2^-25 / 2^12 each).
GAMMA = 9 * U16 + 9 * 320 * U32 + 2 * U32 + 64 * U32 + 2 * 2 * U32
ABS = 1e-9


def _check_grad(mlp, pts):
    dens, grad = mlp.density_grad(pts)
    enc, H = _kernel_forward(mlp, pts)
    want, bound = _restated_grad(mlp, pts, enc, H)
    err = (grad.double() - want).abs()
    assert (err <= GAMMA * bound + ABS).all(), float((err / (GAMMA * bound + ABS)).max())
    return dens, grad, want


@pytest.mark.gpu
@pytest.mark.parametrize('n', [0, 1, 127, 129])
def test_density_grad_matches_float64_restatement(n):
    mlp = nerf_mlp(NERF_MLP, 21, scaled=True)
    torch.manual_seed(n)
    pts = (torch.rand((n, 3), device='cuda') * 3 - 1.5).contiguous()
    dens, grad = mlp.density_grad(pts)
    assert dens.shape == (n,) and grad.shape == (n, 3)
    if n == 0:
        return
    dens, grad, _ = _check_grad(mlp, pts)
    # the training forward's density agrees with the inference kernel's to the fp16 tolerance, not bit for bit
    with torch.no_grad():
        raw = _infer(mlp, pts, torch.nn.functional.normalize(torch.randn_like(pts), dim=-1))
    assert float((dens - raw[:, 3]).abs().max()) <= 2e-2 * max(1.0, float(raw[:, 3].abs().max()))


@pytest.mark.gpu
def test_density_grad_chunks_are_row_independent():
    """one chunk + 1 rows: the last rows equal the same rows run alone, bit for bit, and match the float64 restatement"""
    from xrnerf_b200 import nerf_train as T
    mlp = nerf_mlp(NERF_MLP, 22, scaled=True)
    n = T.GRAD_CHUNK + 1
    torch.manual_seed(5)
    pts = (torch.rand((n, 3), device='cuda') * 3 - 1.5).contiguous()
    dens, grad = mlp.density_grad(pts)
    tail = pts[-129:].contiguous()
    d2, g2, _ = _check_grad(mlp, tail)
    assert torch.equal(dens[-129:], d2) and torch.equal(grad[-129:], g2)


def _f64_alpha(mlp, pts):
    """the unrounded float64 raw alpha over the fp16 weights (no activation rounding) -> [n], and its pre-activations"""
    x = pts.double()
    enc = torch.cat([x] + [torch.cat([torch.sin(x * 2.0 ** b), torch.cos(x * 2.0 ** b)], -1) for b in range(10)], -1)
    h, pre = enc, []
    for l, lin in enumerate(mlp.pts_linears):
        z = h @ w16(lin).T + lin.bias.detach().double()
        pre.append(z)
        h = torch.relu(z)
        if l == 4:
            h = torch.cat([enc, h], -1)
    return (h @ w16(mlp.alpha_linear).T)[:, 0] + mlp.alpha_linear.bias.detach().double()[0], pre


@pytest.mark.gpu
def test_density_grad_matches_central_differences():
    """central differences of the unrounded float64 function, at points where its ReLU masks equal the kernels' and do not change over the stencil"""
    mlp = nerf_mlp(NERF_MLP, 23, scaled=True)
    torch.manual_seed(9)
    pts = (torch.rand((4096, 3), device='cuda') * 3 - 1.5).contiguous()
    h = 1e-6
    eye = torch.eye(3, device='cuda', dtype=torch.float64)
    mlp.density_grad(pts[:1])
    _, pre = _f64_alpha(mlp, pts)
    _, H = _kernel_forward(mlp, pts)
    keep = torch.stack([((z > 0) == (Hl > 0)).all(1) for z, Hl in zip(pre, H)], 1).all(1)
    for a in range(3):
        for sg in (-1.0, 1.0):
            _, pre_s = _f64_alpha(mlp, pts.double() + sg * h * eye[a])
            keep &= torch.stack([((z > 0) == (zs > 0)).all(1) for z, zs in zip(pre, pre_s)], 1).all(1)
    pts = pts[keep][:64].contiguous()
    assert pts.shape[0] >= 16
    _, grad = mlp.density_grad(pts)
    enc, H = _kernel_forward(mlp, pts)
    _, bound = _restated_grad(mlp, pts, enc, H)
    fd = torch.stack([(_f64_alpha(mlp, pts.double() + h * eye[a])[0] - _f64_alpha(mlp, pts.double() - h * eye[a])[0]) / (2 * h) for a in range(3)], 1)
    # a ReLU network's gradient depends on the activations only through the masks, which agree here: the kernel's GAMMA bound, twice, covers the
    # stencil's truncation (h^2 / 6 * 2^27 |e| for the 2^9-scaled sines, below 1e-7 of the bound) and its float64 roundoff (1e-16 |f| / h)
    tol = 2 * GAMMA * bound + 1e-6
    assert ((grad.double() - fd).abs() <= tol).all(), float(((grad.double() - fd).abs() / tol).max())


# ---------------------------------------------------------------------------------------------------------------- analytic field: an octahedron
R_OCT = 1.0


def _octahedron_network(rgb_padding=0.001):
    """NerfNetwork whose raw alpha is r - (|x| + |y| + |z|) and whose rgb is the view direction: pts_linears.0 takes relu(+-x_a) from the identity
    columns, layers 1-7 pass the six units through, alpha_linear sums them; views_linears.0 takes relu(+-d_a), rgb_linear forms d_a."""
    from xrnerf_b200.registry.networks import NerfNetwork
    net = NerfNetwork(dict(N_importance=0, chunk=1024, bs_data='rays_o', is_perturb=False), mlp=NERF_MLP,
                      render=dict(type='NerfRender', white_bkgd=False, raw_noise_std=0, rgb_padding=rgb_padding)).cuda()
    m = net.mlp
    with torch.no_grad():
        for p in m.parameters():
            p.zero_()
        for a in range(3):
            m.pts_linears[0].weight[2 * a, a], m.pts_linears[0].weight[2 * a + 1, a] = 1.0, -1.0
            m.views_linears[0].weight[2 * a, 256 + a], m.views_linears[0].weight[2 * a + 1, 256 + a] = 1.0, -1.0
            m.rgb_linear.weight[a, 2 * a], m.rgb_linear.weight[a, 2 * a + 1] = 1.0, -1.0
        for l in range(1, 8):
            off = 63 if l == 5 else 0
            for u in range(6):
                m.pts_linears[l].weight[u, off + u] = 1.0
        m.alpha_linear.weight[0, :6] = -1.0
        m.alpha_linear.bias[0] = R_OCT
    return net


@pytest.mark.gpu
def test_octahedron_mesh_geometry_and_normals():
    net = _octahedron_network()
    box = ((-1.5, -1.5, -1.5), (1.5, 1.5, 1.5))
    verts, faces = net.extract_mesh(resolution=128, threshold=0.0 + 1e-9, box=box)   # relu: sigma > 1e-9 <=> raw > 1e-9
    v, f = verts.cpu().numpy(), faces.cpu().numpy()
    vol = check_closed_oriented(v, f)
    assert euler(v, f) == 2
    ar = area(v, f)
    vol_exact, area_exact = 4 / 3 * R_OCT ** 3, 4 * math.sqrt(3) * R_OCT ** 2
    # the numpy oracle on the field the kernel evaluates: r - sum |fp16(x_a)| (the encoding holds the position in fp16), summed in fp32
    n = 128
    c = np.abs(lattice_coords(-1.5, 1.5, n).astype(np.float16).astype(np.float32))
    Z, Y, X = np.meshgrid(c, c, c, indexing='ij')
    ov, of = mc_oracle(np.float32(R_OCT) - ((X + Y) + Z), 1e-9, box)
    o_vol, o_area = check_closed_oriented(ov, of), area(ov, of)
    # stated bounds: within 1e-5 (relative) of the oracle's mesh (fp32 summation order of the alpha dot product), within 2 % of the analytic
    # octahedron (marching cubes cuts its edges and corners at h = 3/127)
    assert abs(vol - o_vol) <= 1e-5 * o_vol and abs(ar - o_area) <= 1e-5 * o_area, (vol, o_vol, ar, o_area)
    assert abs(vol - vol_exact) <= 2e-2 * vol_exact and abs(ar - area_exact) <= 2e-2 * area_exact, (vol, vol_exact, ar, area_exact)
    verts2, faces2, normals, colors = net.extract_colored_mesh(resolution=128, threshold=1e-9, box=box)
    assert torch.equal(verts2, verts) and torch.equal(faces2, faces)
    # every vertex off the coordinate planes: normal = sign(v) / sqrt(3), within 0.5 degrees (the gradient is exact there up to fp16 staging)
    off = (verts.abs() > 2 * 3 / 127).all(1)
    assert int(off.sum()) > 1000
    want = torch.sign(verts[off]) / math.sqrt(3)
    cosang = (normals[off] * want).sum(1).clamp(-1, 1)
    assert float(torch.rad2deg(torch.acos(cosang)).max()) <= 0.5
    # the rgb head returns the view direction, the colour is seen along -normal: sigmoid(-normal) (1 + 2p) - p, to the fp16 tolerance
    p = net.render.rgb_padding
    assert float((colors - (torch.sigmoid(-normals) * (1 + 2 * p) - p)).abs().max()) <= 2e-3


@pytest.mark.gpu
def test_colored_mesh_equals_its_parts():
    from xrnerf_b200.registry.networks import NerfNetwork
    torch.manual_seed(31)
    net = NerfNetwork(dict(N_importance=64, chunk=1024, bs_data='rays_o', is_perturb=False), mlp=NERF_MLP, mlp_fine=NERF_MLP,
                      render=dict(type='NerfRender', white_bkgd=False, raw_noise_std=0, rgb_padding=0.001)).cuda()
    with torch.no_grad():
        vol = net.mlp_fine.density_lattice((48, 48, 48), ((-1.5,) * 3, (1.5,) * 3))
    thr = float(torch.quantile(vol.reshape(-1)[::7].float(), 0.6))
    verts, faces = net.extract_mesh(resolution=48, threshold=max(thr, 1e-6))
    assert verts.shape[0] > 0
    v2, f2, normals, colors = net.extract_colored_mesh(resolution=48, threshold=max(thr, 1e-6))
    assert torch.equal(v2, verts) and torch.equal(f2, faces)
    _, g = net.mlp_fine.density_grad(verts)
    nrm = torch.linalg.vector_norm(g, dim=1, keepdim=True)
    assert torch.equal(normals, torch.where(nrm > 0, -g / nrm, torch.zeros_like(g)))
    with torch.no_grad():
        raw = _infer(net.mlp_fine, verts, -normals)
    assert torch.equal(colors, torch.sigmoid(raw[:, :3]) * (1 + 2 * 0.001) - 0.001)
