"""Mip-NeRF mesh export: the point query at footprint sigma (the IPE of the isotropic Gaussian N(p, sigma^2 I); xrb_mip_ipe_tiles_points), the
NerfMLP's raw alpha on a lattice of point queries (xrb_mip_density_lattice, NerfMLP.density_lattice(footprint=...)), its gradient with respect to the
position (NerfMLP.density_grad: the training kernels + xrb_mip_ipe_grad), and MipNerfNetwork.extract_mesh / extract_colored_mesh.

The encoder is compared with the numpy restatement of the reference's integrated_pos_enc / pos_enc (oracle.nerf_oracle). The lattice is compared bit
for bit with the encoder + the inference kernel. The gradient is compared entry by entry with a float64 restatement over the kernels' own fp16
weights, activations and ReLU masks. The mesh path is checked on a NerfMLP whose raw alpha is r - a_0 (|sin x| + |sin y| + |sin z|), built from the
band-0 sine columns, so the footprint moves the surface."""
import ctypes as C
import math

import numpy as np
import pytest
import torch
from cases import MIP_CFG, MIP_MLP, MIP_RENDER, NERF_MLP, host_buffer, nerf_mlp
from restate64 import U16, U32, area, check_closed_oriented, columns, euler, lattice_coords, lattice_points, mc_oracle, mip_bands, trunk_grad, w16

BOX = ((-1.5, -1.5, -1.5), (1.5, 1.5, 1.5))
CELL_256 = 3.0 / 255 / math.sqrt(12.0)                                  # footprint 'cell' at 256^3 over BOX: 3.4e-3
SIGMAS = [0.0, 1e-3, CELL_256, 0.05, 1.0]
HALF_PI32 = np.float32(0.5 * np.pi)


# ---------------------------------------------------------------------------------------------------------------- CPU: argument checks
def test_mip_density_lattice_validates_arguments_without_gpu():
    from xrnerf_b200 import _C
    lib = _C.lib
    lo, hi = _C.float3(BOX[0]), _C.float3(BOX[1])
    buf, a = host_buffer()
    p = C.c_void_p(a)
    for n in ((1, 4, 4), (4, 1025, 4), (4, 4, -1)):
        assert lib.xrb_mip_density_lattice(p, p, 0, 16, 0.01, *n, lo, hi, p, None) == -1 and b'bad size' in lib.xrb_last_error()
    for d0, d1 in ((0, 22), (4, 4), (5, 2), (-101, -90)):
        assert lib.xrb_mip_density_lattice(p, p, d0, d1, 0.01, 4, 4, 4, lo, hi, p, None) == -1 and b'degrees' in lib.xrb_last_error()
    for s in (-1e-6, math.nan, math.inf, -math.inf):
        assert lib.xrb_mip_density_lattice(p, p, 0, 16, s, 4, 4, 4, lo, hi, p, None) == -1 and b'sigma' in lib.xrb_last_error()
    for b0, b1 in (((0, 0, 0), (1, 0, 1)), ((0, 0, 0), (1, 1, math.inf)), ((2, 0, 0), (1, 1, 1))):
        assert lib.xrb_mip_density_lattice(p, p, 0, 16, 0.01, 4, 4, 4, _C.float3(b0), _C.float3(b1), p, None) == -1 and b'box' in lib.xrb_last_error()
    assert lib.xrb_mip_density_lattice(p, p, 0, 16, 0.01, 4, 4, 4, None, hi, p, None) == -1
    assert lib.xrb_mip_density_lattice(None, None, 0, 16, 0.01, 0, 4, 4, lo, hi, None, None) == 0            # empty lattice: a no-op
    assert lib.xrb_mip_density_lattice(None, p, 0, 16, 0.01, 4, 4, 4, lo, hi, p, None) == -1 and b'null' in lib.xrb_last_error()
    assert lib.xrb_mip_density_lattice(p, p, 0, 16, 0.01, 4, 4, 4, lo, hi, None, None) == -1
    odd = C.c_void_p(a + 4)
    assert lib.xrb_mip_density_lattice(odd, p, 0, 16, 0.01, 4, 4, 4, lo, hi, p, None) == -1 and b'aligned' in lib.xrb_last_error()
    assert lib.xrb_mip_density_lattice(p, C.c_void_p(a + 8), 0, 16, 0.01, 4, 4, 4, lo, hi, p, None) == -1 and b'aligned' in lib.xrb_last_error()
    # the NeRF lattice still refuses the Mip-NeRF layout
    assert lib.xrb_nerf_density_lattice(p, p, 96, 10, 4, 4, 4, lo, hi, p, None) == -2


def test_mip_ipe_tiles_points_validates_arguments_without_gpu():
    from xrnerf_b200 import _C
    lib = _C.lib
    buf, a = host_buffer()
    p = C.c_void_p(a)
    f = lib.xrb_mip_ipe_tiles_points
    assert f(p, p, -1, 1, 0.01, 0, 16, 0, 4, p, None) == -1 and b'bad size' in lib.xrb_last_error()
    assert f(p, p, 4, 0, 0.01, 0, 16, 0, 4, p, None) == -1
    for args in ((0, 22, 0, 4), (3, 3, 0, 4), (0, 16, 0, 11), (0, 16, 4, 3), (0, 16, -101, 4)):
        assert f(p, p, 4, 1, 0.01, *args, p, None) == -1 and b'bad size' in lib.xrb_last_error()
    for s in (-1.0, math.nan, math.inf):
        assert f(p, p, 4, 1, s, 0, 16, 0, 4, p, None) == -1 and b'sigma' in lib.xrb_last_error()
    assert f(None, None, 0, 1, 0.01, 0, 16, 0, 4, None, None) == 0                                          # n == 0: a no-op
    for args in ((None, p, p), (p, None, p), (p, p, None)):
        assert f(args[0], args[1], 4, 1, 0.01, 0, 16, 0, 4, args[2], None) == -1 and b'null' in lib.xrb_last_error()
    assert f(p, p, 4, 1, 0.01, 0, 16, 0, 4, C.c_void_p(a + 4), None) == -1 and b'misaligned' in lib.xrb_last_error()


def test_mip_ipe_grad_validates_arguments_without_gpu():
    from xrnerf_b200 import _C
    lib = _C.lib
    buf, a = host_buffer()
    p = C.c_void_p(a)
    f = lib.xrb_mip_ipe_grad
    assert f(p, -1, 0.01, 0, 16, p, 2, p, p, None) == -1 and b'bad size' in lib.xrb_last_error()
    assert f(p, 4, 0.01, 0, 22, p, 2, p, p, None) == -1 and f(p, 4, 0.01, 2, 2, p, 2, p, p, None) == -1
    assert f(p, 4, 0.01, 0, 16, p, 0, p, p, None) == -1 and f(p, 4, 0.01, 0, 16, p, 5, p, p, None) == -1
    for s in (-1.0, math.nan, -math.inf):
        assert f(p, 4, s, 0, 16, p, 2, p, p, None) == -1 and b'sigma' in lib.xrb_last_error()
    assert f(None, 0, 0.01, 0, 16, None, 2, None, None, None) == 0                                           # n == 0: a no-op
    for args in ((None, p, p, p), (p, None, p, p), (p, p, None, p), (p, p, p, None)):
        assert f(args[0], 4, 0.01, 0, 16, args[1], 2, args[2], args[3], None) == -1 and b'null' in lib.xrb_last_error()
    assert f(p, 4, 0.01, 0, 16, C.c_void_p(a + 4), 2, p, p, None) == -1


def test_footprint_sigma_values_and_validation():
    from xrnerf_b200.mesh import footprint_sigma
    assert footprint_sigma(0.0) == 0.0 and footprint_sigma(0.05) == 0.05 and footprint_sigma(1) == 1.0
    assert footprint_sigma('cell', (256, 256, 256), BOX) == pytest.approx(CELL_256, rel=1e-15)
    # (nz, ny, nx): the largest spacing of the three axes, here z: 4 / 9
    assert footprint_sigma('cell', (10, 20, 40), ((0, 0, 0), (1, 2, 4))) == pytest.approx(4 / 9 / math.sqrt(12), rel=1e-15)
    for bad in (-1e-9, -1.0, math.nan, math.inf, -math.inf, 1e39, 'edge', 'Cell'):
        with pytest.raises(ValueError):
            footprint_sigma(bad, (8, 8, 8), BOX)
    with pytest.raises(ValueError, match='lattice'):
        footprint_sigma('cell')


def test_mlp_footprint_rules_without_gpu():
    """a MipNerfEmbedder NerfMLP needs a footprint, a BaseEmbedder one takes none; the CPU refusal comes first"""
    from xrnerf_b200 import registry as R
    mip, nerf = R.build_mlp(MIP_MLP), R.build_mlp(NERF_MLP)
    assert mip._footprint(0.05) == 0.05 and mip._footprint('cell', (256,) * 3, BOX) == pytest.approx(CELL_256, rel=1e-15)
    with pytest.raises(NotImplementedError, match='footprint'):
        mip._footprint(None)
    with pytest.raises(ValueError):
        mip._footprint(-0.5)
    with pytest.raises(ValueError):
        mip._footprint('cell')                                           # density_grad has no lattice
    assert nerf._footprint(None) is None
    with pytest.raises(ValueError):
        nerf._footprint(0.01)
    for m in (mip, nerf):
        with pytest.raises(NotImplementedError, match='CUDA'):
            m.density_lattice((4, 4, 4), BOX, footprint=0.01)
        with pytest.raises(NotImplementedError, match='CUDA'):
            m.density_grad(torch.zeros(4, 3), footprint=0.01)


def test_mip_network_footprint_errors_without_gpu():
    """footprint=None raises NotImplementedError naming the frusta and how to choose a footprint; a bad footprint raises ValueError; both before any
    attribute of the network is read"""
    from xrnerf_b200.registry.networks import MipNerfNetwork
    net = object.__new__(MipNerfNetwork)
    for fn in (net.extract_mesh, net.extract_colored_mesh):
        with pytest.raises(NotImplementedError, match="frusta.*footprint=sigma or 'cell'"):
            fn(64)
        for bad in (-0.1, math.nan, math.inf, 'voxel'):
            with pytest.raises(ValueError):
                fn(64, footprint=bad)


# ---------------------------------------------------------------------------------------------------------------- GPU helpers
def _encode(pts, dirs, sigma, spr=1):
    """the point encoder's tile image (3 blocks per tile) of (pts, dirs) at footprint sigma"""
    from xrnerf_b200 import _C
    n = pts.shape[0]
    enc = torch.full((_C.lib.xrb_nerf_enc_image_bytes(n, 96),), 0xA5, dtype=torch.uint8, device='cuda')
    _C.check(_C.lib.xrb_mip_ipe_tiles_points(_C.f32(pts.contiguous()), _C.f32(dirs.contiguous()), n, spr, float(sigma), 0, 16, 0, 4, _C.ptr(enc), _C.stream()),
             'mip_ipe_tiles_points')
    return enc


def _infer(mlp, pts, dirs, sigma):
    """raw f32[n,4] of the inference kernel on the point encoder's encoding of (pts, dirs) at footprint sigma"""
    from xrnerf_b200.nerf_mlp import nerf_mlp_forward_tiles
    image, bias = mlp._packed()
    return nerf_mlp_forward_tiles(image, bias, _encode(pts, dirs, sigma), pts.shape[0], 96, 27)


def _threshold_sigma():
    """an fp32 sigma at which band 3's exponent 0.5 ((sigma^2 8) 8) is exactly 20 in fp32: the band is live, at the zeroing threshold"""
    s = np.float32(math.sqrt(40.0) / 8)
    for _ in range(2000):
        cov = s * s
        hv = np.float32(0.5) * (cov * np.float32(8) * np.float32(8))
        if hv == np.float32(20):
            return float(s)
        s = np.nextafter(s, np.float32(1) if hv < 20 else np.float32(0))
    # no fp32 sigma lands exactly: take the largest one still at or below the threshold
    while np.float32(0.5) * (s * s * np.float32(64)) > 20:
        s = np.nextafter(s, np.float32(0))
    return float(s)


# ---------------------------------------------------------------------------------------------------------------- point encoder against the reference
@pytest.mark.gpu
def test_point_encoder_matches_reference_ipe():
    """every column against integrated_pos_enc(p, sigma^2 (1,1,1)) and pos_enc(d): within the fp16 rounding of the value (2^-11 relative, 2^-25 absolute
    for subnormals) plus the two sine evaluations' error at the 2^15-scaled arguments (a few 2^-24, absolute, both sides) and one fp32 ulp of a_k.
    Dead bands (exponent above 20) are exactly zero; the direction block equals what xrb_mip_ipe_tiles_rays writes for the same direction."""
    from oracle import nerf_oracle as O
    from xrnerf_b200 import _C
    g = torch.Generator(device='cuda').manual_seed(3)
    n = 1000                                                              # 7 full tiles + a ragged one
    pts = (torch.rand((n, 3), device='cuda', generator=g) * 3 - 1.5).contiguous()
    pts[:4] = torch.tensor([[0.0, 0.0, 0.0], [1.5, -1.5, 1.5], [1e-3, -2e-7, 0.75], [-1.0, 0.5, -0.25]], device='cuda')
    dirs = torch.nn.functional.normalize(torch.randn((n, 3), device='cuda', generator=g), dim=-1).contiguous()
    p64 = pts.cpu().numpy()
    sig_thr = _threshold_sigma()
    for sigma in SIGMAS + [sig_thr]:
        enc = _encode(pts, dirs, sigma)
        got = columns(enc, n, 3, 0, 96).cpu().numpy()
        s32 = np.float32(sigma)
        want = O.integrated_pos_enc(p64, np.full_like(p64, s32 * s32), 0, 16).astype(np.float64)
        tol = (U16 + 2 * U32) * np.abs(want) + 2.0 ** -25 + 8 * U32
        assert (np.abs(got - want) <= tol).all(), (sigma, float((np.abs(got - want) / tol).max()))
        fac = mip_bands(sigma)
        dead = np.concatenate([np.repeat(fac == 0, 3)] * 2)
        assert (got[:, dead] == 0).all()
        if sigma == 1.0:
            assert dead.sum() == 6 * 13                                   # hv = 0.5, 2, 8 live; 32 and above dead
        if sigma == sig_thr:
            assert not dead[9] and dead[12] and fac[3] > 0               # band 3 exactly at the threshold: evaluated (and below fp16's range)
        d_got = columns(enc, n, 3, 2, 27).cpu().numpy()
        d_want = O.mip_pos_enc(dirs.cpu().numpy(), 0, 4).astype(np.float64)
        assert (np.abs(d_got - d_want) <= U16 * np.abs(d_want) + 8 * U32).all()
        # padding columns 96..127 and the rows past n are +0
        pad = columns(enc, (n + 127) // 128 * 128, 3, 0, 128).cpu().numpy()
        assert (pad[:, 96:] == 0).all() and (pad[n:] == 0).all()
    # the direction block, byte for byte, against the ray encoder's (one sample per ray)
    rays = _C.lib.xrb_nerf_enc_image_bytes(n, 96)
    img = torch.zeros(rays, dtype=torch.uint8, device='cuda')
    z = torch.tensor([[2.0, 2.5]], device='cuda').expand(n, 2).contiguous()
    radii = torch.full((n, 1), 1e-3, device='cuda')
    _C.check(_C.lib.xrb_mip_ipe_tiles_rays(_C.ptr(z), _C.ptr(pts), _C.ptr(dirs), _C.ptr(radii), _C.ptr(dirs), n, 1, 0, 16, 0, 4, _C.ptr(img), _C.stream()))
    mine = _encode(pts, dirs, 0.05)
    blk = lambda t: t.view(-1, 3, 16384)[:, 2]
    assert torch.equal(blk(mine), blk(img))


# ---------------------------------------------------------------------------------------------------------------- lattice: bit identity
@pytest.mark.gpu
@pytest.mark.parametrize('shape', [(2, 2, 2), (7, 5, 3), (9, 33, 17), (128, 128, 128)])
@pytest.mark.parametrize('scaled', [False, True])
def test_mip_density_lattice_equals_encoder_and_inference_kernel_bit_for_bit(shape, scaled):
    """(nz, ny, nx); totals 8, 105, 5049 and 2^21: three are not a multiple of the 128-row tile. A centred box and one with negative coordinates;
    every footprint of SIGMAS and 'cell' of the lattice itself."""
    from xrnerf_b200.mesh import footprint_sigma
    mlp = nerf_mlp(MIP_MLP, 11, scaled)
    for box in (BOX, ((-2.0, -0.25, -3.5), (-0.5, 1.75, -1.0))):
        pts = lattice_points(shape, box)
        dirs = torch.nn.functional.normalize(torch.randn_like(pts), dim=-1)
        for fp in SIGMAS + ['cell']:
            sigma = footprint_sigma(fp, shape, box)
            with torch.no_grad():
                vol = mlp.density_lattice(shape, box, footprint=fp)
                raw = _infer(mlp, pts, dirs, sigma)
            torch.cuda.synchronize()
            assert vol.shape == shape
            assert torch.equal(vol.reshape(-1), raw[:, 3]), (shape, box, fp, float((vol.reshape(-1) - raw[:, 3]).abs().max()))


# ---------------------------------------------------------------------------------------------------------------- gradient: float64 restatement
def _kernel_forward(mlp, pts, sigma):
    """the training kernels' forward as density_grad runs it: the point encoding (fp16) and the 8 hidden activations (fp16) as float64"""
    from xrnerf_b200 import nerf_train as T
    n = pts.shape[0]
    nt = (n + 127) // 128
    S = mlp._tg_slabs
    enc = _encode(pts, torch.zeros((n, 3), device='cuda'), sigma)
    img = T.Img(enc, 3 * T.BLOCK, 0, 3)
    H = [T.Img.new(nt, 4, 'cuda') for _ in range(8)]
    T._fwd(n, S, 'pts0', [img.sub(0, 2)], H[0])
    for l in range(1, 8):
        T._fwd(n, S, f'pts{l}', ([img.sub(0, 2), H[l - 1]] if l == 5 else [H[l - 1]]), H[l])
    return columns(enc, n, 3, 0, 96), [columns(h.buf, n, 4, 0, 256) for h in H]


def _restated_grad(mlp, pts, sigma, H):
    """float64 d(raw alpha)/d(position) over the fp16 weights, with the kernels' ReLU masks (fp16 activation > 0) and the library's a_k; also the same
    chain on absolute values, which bounds the rounding error, and the absolute error bound of the final contraction's cosines"""
    e, ea = trunk_grad(mlp, H, 96)
    fac = mip_bands(sigma)
    out, outa, trig = (torch.zeros_like(pts, dtype=torch.float64) for _ in range(3))
    for k in range(16):
        if fac[k] == 0:
            continue
        y32 = pts * 2.0 ** k                                  # the kernel's fp32 arguments: y exact, y + pi/2 rounded once
        y, yc = y32.double(), (y32 + float(HALF_PI32)).double()
        es, ec, eas, eac = e[:, 3 * k:3 * k + 3], e[:, 48 + 3 * k:51 + 3 * k], ea[:, 3 * k:3 * k + 3], ea[:, 48 + 3 * k:51 + 3 * k]
        out += fac[k] * 2.0 ** k * (torch.cos(y) * es + torch.cos(yc) * ec)
        outa += fac[k] * 2.0 ** k * (torch.cos(y).abs() * eas + torch.cos(yc).abs() * eac)
        trig += fac[k] * 2.0 ** k * (eas + eac)
    return out, outa, trig


# The rounding count of the kernel chain, as in tests/test_gpu_nerf_mesh.py with the Mip-NeRF widths: 9 fp16 stagings of the dZ (2^-11 each), 9 fp32
# contractions of <= 352 terms (the skip layer reads 96 + 256 columns), the two d(encoding) terms summed and scaled once in fp32, and the final
# contraction over 96 columns with three fp32 products per term. |kernel - float64| <= GAMMA * (the same chain on absolute values)
# + COS * sum_k a_k 2^deg (|e_sin| + |e_cos|) (the cosf error, 2 ulp of a value <= 1, absolute) + ABS (staged values in fp16's subnormal range).
GAMMA = 9 * U16 + 9 * 352 * U32 + 2 * U32 + 96 * U32 + 4 * U32
COS = 4 * U32
ABS = 1e-9


def _check_grad(mlp, pts, sigma):
    dens, grad = mlp.density_grad(pts, footprint=sigma)
    _, H = _kernel_forward(mlp, pts, sigma)
    want, bound, trig = _restated_grad(mlp, pts, sigma, H)
    err = (grad.double() - want).abs()
    lim = GAMMA * bound + COS * trig + ABS
    assert (err <= lim).all(), (sigma, float((err / lim).max()))
    return dens, grad, want


@pytest.mark.gpu
@pytest.mark.parametrize('n', [0, 1, 127, 129])
def test_mip_density_grad_matches_float64_restatement(n):
    mlp = nerf_mlp(MIP_MLP, 21, scaled=True)
    torch.manual_seed(n)
    pts = (torch.rand((n, 3), device='cuda') * 3 - 1.5).contiguous()
    for sigma in SIGMAS:
        dens, grad = mlp.density_grad(pts, footprint=sigma)
        assert dens.shape == (n,) and grad.shape == (n, 3)
        if n == 0:
            continue
        dens, grad, _ = _check_grad(mlp, pts, sigma)
        # the training forward's density agrees with the inference kernel's to the fp16 tolerance, not bit for bit
        with torch.no_grad():
            raw = _infer(mlp, pts, torch.nn.functional.normalize(torch.randn_like(pts), dim=-1), sigma)
        assert float((dens - raw[:, 3]).abs().max()) <= 2e-2 * max(1.0, float(raw[:, 3].abs().max()))


@pytest.mark.gpu
def test_mip_density_grad_chunks_are_row_independent():
    """one chunk + 1 rows: the last rows equal the same rows run alone, bit for bit, and match the float64 restatement"""
    from xrnerf_b200 import nerf_train as T
    mlp = nerf_mlp(MIP_MLP, 22, scaled=True)
    n = T.GRAD_CHUNK + 1
    torch.manual_seed(5)
    pts = (torch.rand((n, 3), device='cuda') * 3 - 1.5).contiguous()
    dens, grad = mlp.density_grad(pts, footprint=CELL_256)
    tail = pts[-129:].contiguous()
    d2, g2, _ = _check_grad(mlp, tail, CELL_256)
    assert torch.equal(dens[-129:], d2) and torch.equal(grad[-129:], g2)


def _f64_alpha(mlp, pts, sigma, phase):
    """the unrounded float64 raw alpha of the point query over the fp16 weights (no activation rounding) -> [n], and its pre-activations. The cos
    columns are a_k sin(y + phase), phase = the kernel's fp32 (y + pi/2) - y at the base point (the reference's expression), held over the stencil."""
    x = pts.double()
    fac = mip_bands(sigma)
    sins = [fac[k] * torch.sin(x * 2.0 ** k) for k in range(16)]
    coss = [fac[k] * torch.sin(x * 2.0 ** k + phase[k]) for k in range(16)]
    enc = torch.cat([torch.cat(sins, -1), torch.cat(coss, -1)], -1)
    h, pre = enc, []
    for l, lin in enumerate(mlp.pts_linears):
        z = h @ w16(lin).T + lin.bias.detach().double()
        pre.append(z)
        h = torch.relu(z)
        if l == 4:
            h = torch.cat([enc, h], -1)
    return (h @ w16(mlp.alpha_linear).T)[:, 0] + mlp.alpha_linear.bias.detach().double()[0], pre


@pytest.mark.gpu
@pytest.mark.parametrize('sigma', [0.0, CELL_256, 0.05])
def test_mip_density_grad_matches_central_differences(sigma):
    """central differences of the unrounded float64 function, at points where its ReLU masks equal the kernels' and do not change over the stencil.
    The step is 1e-6 scaled to the highest live band, 2^top h <= 2^9 1e-6 (NeRF's stencil at its 2^9-scaled sines), so the masks can hold over it."""
    mlp = nerf_mlp(MIP_MLP, 23, scaled=True)
    torch.manual_seed(9)
    pts = (torch.rand((4096, 3), device='cuda') * 3 - 1.5).contiguous()
    phase = lambda p: [((p * 2.0 ** k) + float(HALF_PI32)).double() - (p * 2.0 ** k).double() for k in range(16)]
    top = int(np.nonzero(mip_bands(sigma))[0].max())
    h = 1e-6 * min(1.0, 2.0 ** (9 - top))
    eye = torch.eye(3, device='cuda', dtype=torch.float64)
    mlp.density_grad(pts[:1], footprint=sigma)
    ph = phase(pts)
    _, pre = _f64_alpha(mlp, pts, sigma, ph)
    _, H = _kernel_forward(mlp, pts, sigma)
    keep = torch.stack([((z > 0) == (Hl > 0)).all(1) for z, Hl in zip(pre, H)], 1).all(1)
    for a in range(3):
        for sg in (-1.0, 1.0):
            _, pre_s = _f64_alpha(mlp, pts.double() + sg * h * eye[a], sigma, ph)
            keep &= torch.stack([((z > 0) == (zs > 0)).all(1) for z, zs in zip(pre, pre_s)], 1).all(1)
    pts = pts[keep][:64].contiguous()
    assert pts.shape[0] >= 16
    ph = phase(pts)
    _, grad = mlp.density_grad(pts, footprint=sigma)
    _, H = _kernel_forward(mlp, pts, sigma)
    _, bound, trig = _restated_grad(mlp, pts, sigma, H)
    fd = torch.stack([(_f64_alpha(mlp, pts.double() + h * eye[a], sigma, ph)[0] - _f64_alpha(mlp, pts.double() - h * eye[a], sigma, ph)[0]) / (2 * h)
                      for a in range(3)], 1)
    # the masks agree, so the kernel's bound, twice, covers the stencil's truncation (h^2 / 6 * 2^(3 top) |e| against 2^top |e|: below 5e-8 of the
    # bound) and its float64 roundoff (1e-16 |f| / h)
    tol = 2 * (GAMMA * bound + COS * trig) + 1e-6
    assert ((grad.double() - fd).abs() <= tol).all(), float(((grad.double() - fd).abs() / tol).max())


# ---------------------------------------------------------------------------------------------------------------- analytic field: sum |band-0 sine|
R_SIN = 0.7
RGB_PADDING = 0.001


def _sine_network():
    """MipNerfNetwork (softplus, density_bias -1: the reference config) whose raw alpha is r - a_0 (|sin x| + |sin y| + |sin z|) and whose rgb is the
    view direction: pts_linears.0 takes relu(+-a_0 sin x_a) from the band-0 sine columns 0..2, layers 1-7 pass the six units through, alpha_linear
    sums them; views_linears.0 takes relu(+-d_a) from the direction's identity columns, rgb_linear forms d_a."""
    from xrnerf_b200.registry.networks import MipNerfNetwork
    net = MipNerfNetwork(dict(MIP_CFG, phase='test'), mlp=MIP_MLP, render=dict(MIP_RENDER, rgb_padding=RGB_PADDING)).cuda()
    m = net.mlp
    with torch.no_grad():
        for p in m.parameters():
            p.zero_()
        for a in range(3):
            m.pts_linears[0].weight[2 * a, a], m.pts_linears[0].weight[2 * a + 1, a] = 1.0, -1.0
            m.views_linears[0].weight[2 * a, 256 + a], m.views_linears[0].weight[2 * a + 1, 256 + a] = 1.0, -1.0
            m.rgb_linear.weight[a, 2 * a], m.rgb_linear.weight[a, 2 * a + 1] = 1.0, -1.0
        for l in range(1, 8):
            off = 96 if l == 5 else 0
            for u in range(6):
                m.pts_linears[l].weight[u, off + u] = 1.0
        m.alpha_linear.weight[0, :6] = -1.0
        m.alpha_linear.bias[0] = R_SIN
    return net


@pytest.mark.gpu
@pytest.mark.parametrize('sigma', [0.0, 0.5])
def test_sine_field_mesh_geometry_normals_and_colours(sigma):
    from xrnerf_b200.mesh import raw_density_threshold
    net = _sine_network()
    a0 = mip_bands(sigma)[0]
    assert a0 == (1.0 if sigma == 0 else float(np.float32(math.exp(-0.125))))
    dens = math.log1p(math.exp(-1.0))                                    # softplus(raw - 1) at raw = 0: the level set raw = 0
    thr = raw_density_threshold(dens, 'softplus', -1.0)
    assert abs(thr) < 1e-12
    n = 128
    verts, faces = net.extract_mesh(resolution=n, threshold=dens, box=BOX, footprint=sigma)
    v, f = verts.cpu().numpy(), faces.cpu().numpy()
    vol = check_closed_oriented(v, f)
    assert euler(v, f) == 2
    ar = area(v, f)
    # the numpy oracle on the field the kernel evaluates: r - sum fp16(a_0 sin(x_a)), summed in fp32
    c = lattice_coords(-1.5, 1.5, n)
    s = np.abs((np.float32(a0) * np.sin(c)).astype(np.float16).astype(np.float32))
    Z, Y, X = np.meshgrid(s, s, s, indexing='ij')
    ov, of = mc_oracle(np.float32(R_SIN) - ((X + Y) + Z), thr, BOX)
    o_vol, o_area = check_closed_oriented(ov, of), area(ov, of)
    assert abs(vol - o_vol) <= 1e-5 * o_vol and abs(ar - o_area) <= 1e-5 * o_area, (vol, o_vol, ar, o_area)
    # vertices off the coordinate planes lie on sum |sin x_a| = r / a_0: fp16 values (3 half-ulps of 2^-11 over a_0) and linear interpolation of a
    # function with |second derivative| <= 1 over h = 3/127 (3 h^2 / 8)
    hh = 3.0 / (n - 1)
    off = (verts.abs() > 2 * hh).all(1)
    assert int(off.sum()) > 1000
    resid = torch.sin(verts[off].double()).abs().sum(1) - R_SIN / a0
    lim = 3 * 2.0 ** -12 / a0 + 3 * hh * hh / 8
    assert float(resid.abs().max()) <= lim, (float(resid.abs().max()), lim)
    if sigma > 0:   # the footprint moved the surface: far from the point field's sum |sin x_a| = r
        assert float((torch.sin(verts[off].double()).abs().sum(1) - R_SIN).abs().min()) > 20 * lim
    verts2, faces2, normals, colors = net.extract_colored_mesh(resolution=n, threshold=dens, box=BOX, footprint=sigma)
    assert torch.equal(verts2, verts) and torch.equal(faces2, faces)
    # normals off the coordinate planes: the outward direction of sign(x_a) cos(x_a), within 0.5 degrees
    vo = verts[off].double()
    want = torch.nn.functional.normalize(torch.sign(vo) * torch.cos(vo), dim=1)
    cosang = (normals[off].double() * want).sum(1).clamp(-1, 1)
    assert float(torch.rad2deg(torch.acos(cosang)).max()) <= 0.5
    # the rgb head returns the view direction, the colour is seen along -normal: sigmoid(-normal) (1 + 2p) - p, to the fp16 tolerance
    p = RGB_PADDING
    assert float((colors - (torch.sigmoid(-normals) * (1 + 2 * p) - p)).abs().max()) <= 2e-3


@pytest.mark.gpu
def test_mip_colored_mesh_equals_its_parts():
    from xrnerf_b200.mesh import footprint_sigma, marching_cubes, raw_density_threshold
    from xrnerf_b200.registry.networks import MipNerfNetwork
    torch.manual_seed(31)
    net = MipNerfNetwork(dict(MIP_CFG, phase='test'), mlp=MIP_MLP, render=dict(MIP_RENDER, rgb_padding=RGB_PADDING)).cuda()
    res = 48
    sigma = footprint_sigma('cell', (res,) * 3, BOX)
    with torch.no_grad():
        vol = net.mlp.density_lattice((res,) * 3, BOX, footprint=sigma)
    q = float(torch.quantile(vol.reshape(-1)[::7].float(), 0.6))
    dens = math.log1p(math.exp(q - 1.0))                                 # the renderer's density at raw alpha q
    verts, faces = net.extract_mesh(resolution=res, threshold=dens, footprint='cell')
    assert verts.shape[0] > 0
    v0, f0 = marching_cubes(vol, raw_density_threshold(dens, 'softplus', -1.0), BOX)
    assert torch.equal(verts, v0) and torch.equal(faces, f0)
    v2, f2, normals, colors = net.extract_colored_mesh(resolution=res, threshold=dens, footprint='cell')
    assert torch.equal(v2, verts) and torch.equal(f2, faces)
    _, g = net.mlp.density_grad(verts, footprint=sigma)
    nrm = torch.linalg.vector_norm(g, dim=1, keepdim=True)
    assert torch.equal(normals, torch.where(nrm > 0, -g / nrm, torch.zeros_like(g)))
    with torch.no_grad():
        raw = _infer(net.mlp, verts, -normals, sigma)
    assert torch.equal(colors, torch.sigmoid(raw[:, :3]) * (1 + 2 * RGB_PADDING) - RGB_PADDING)
