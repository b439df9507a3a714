"""Mesh vertex normals and colours: the field's density gradient (xrb_ngp_density_grad, NgpField.density_grad), HashNerfNetwork.extract_colored_mesh,
and the PLY attributes (xrnerf_b200.mesh.write_ply, ngp_to_nerf_normals).

Restatement (numpy; include/xrnerf_b200.h states the contract). The kernel's encodings come from xrb_tcnn_hashgrid_forward (the same hash_level and fp16
rounding as the density kernels); the density net then runs as the CUDA-core kernel does it, one sequential fp32 fma chain per unit, restated exactly
(each fp16 x fp16 product is exact, and the sum is formed in extended precision and rounded once to fp32). That gives the forward activations and masks;
the density it produces must equal the kernel's bit for bit, which is what shows the masks are the kernel's. The grid cell is restated exactly
(restate64.Grid: px = fp32(fma(scale, x, 0.5)) for every fp32 x), so the in-cell positions are the kernel's too. The restatement is
restate64.cuda_core_density_grad.

Gradient bound. With those masks and in-cell positions, the kernel's gradient is a sum of products, each of the form
    scale_l * (+-w_y w_z) * v_c * (a path of weights through the net),
computed in fp32 with at most n roundings along any product: 64 per W^T step of the net (a chain of 64 fma), then 2 for v_c . (g0, g1), 1 for the weight
product, 8 for the sum over corners and 16 for the sum over levels. So |kernel - exact| <= gamma_n * M, gamma_n = n u / (1 - n u), u = 2^-24, where M is
the same sum on absolute values; the float64 restatement adds its own gamma_n with u = 2^-53. Nothing in the bound is fitted to a run.
"""
import math

import numpy as np
import pytest
import torch
from cases import SPHERE_C, SPHERE_THR, cpu_args, face_points, ngp_density_grad, ngp_field, ngp_network, random_points, sphere_network
from restate64 import U32, U64, Grid, cuda_core_density, cuda_core_density_grad, enc_grad, field_mats, gamma, hashgrid_enc16

f32 = np.float32
REPORT = []


# ================================================================================================================ CPU-only tests
def test_density_grad_validates_arguments_without_gpu():
    _C, _buf, p, cfg, tab = cpu_args()
    lib = _C.lib
    call = lambda cfg=cfg, tab=tab, w=p, pts=p, stride=3, n=4, dens=p, grad=p: lib.xrb_ngp_density_grad(cfg, tab, w, pts, stride, n, dens, grad, None)
    assert call(cfg=None) == -1 and b'null' in lib.xrb_last_error()
    for bad in (_C.NgpConfig(16, 2, 19, 16, 1.38191288, 64, 5, 2), _C.NgpConfig(16, 2, 19, 16, 1.38191288, 64, 0, 2), _C.NgpConfig(16, 2, 19, 16, 1.38191288, 32, 1, 2),
                _C.NgpConfig(8, 2, 19, 16, 1.38191288, 64, 1, 2)):
        assert call(cfg=bad) == -2 and b'unsupported' in lib.xrb_last_error()
    assert call(n=-1) == -1 and b'bad size' in lib.xrb_last_error()
    assert call(stride=2) == -1 and b'bad size' in lib.xrb_last_error()
    for kw in (dict(tab=None), dict(w=None), dict(pts=None), dict(grad=None)):
        assert call(**kw) == -1 and b'null pointer' in lib.xrb_last_error(), kw
    assert call(tab=_C.NgpTable(None, None, 0)) == -1 and b'null hash table' in lib.xrb_last_error()
    assert call(tab=_C.NgpTable(p.value + 4, None, 0)) == -1 and b'aligned' in lib.xrb_last_error()
    assert call(tab=_C.NgpTable(p.value, None, 14)) == -1 and b'n_packed_levels' in lib.xrb_last_error()
    assert call(tab=_C.NgpTable(p.value, None, 6)) == -1 and b'cell image' in lib.xrb_last_error()
    assert call(n=0, tab=None, w=None, pts=None, dens=None, grad=None) == 0   # n == 0 touches no pointer


def _write_ply_before(path, verts, faces):
    """write_ply as it was before the vertex attributes: the byte layout a file without attributes keeps"""
    v = np.ascontiguousarray(np.asarray(verts), dtype='<f4').reshape(-1, 3)
    f = np.ascontiguousarray(np.asarray(faces), dtype='<i4').reshape(-1, 3)
    rec = np.empty(len(f), dtype=[('n', 'u1'), ('idx', '<i4', (3,))])
    rec['n'] = 3
    rec['idx'] = f
    header = ('ply\nformat binary_little_endian 1.0\n'
              f'element vertex {len(v)}\nproperty float x\nproperty float y\nproperty float z\n'
              f'element face {len(f)}\nproperty list uchar int vertex_indices\nend_header\n')
    with open(path, 'wb') as fh:
        fh.write(header.encode('ascii'))
        fh.write(v.tobytes())
        fh.write(rec.tobytes())


def test_write_ply_without_attributes_is_unchanged(tmp_path):
    from xrnerf_b200.mesh import write_ply
    rng = np.random.default_rng(1)
    for nv, nf in ((9, 11), (0, 0), (1, 0)):
        verts = rng.standard_normal((nv, 3)).astype(f32)
        faces = rng.integers(0, max(nv, 1), (nf, 3)).astype(np.int32)
        write_ply(tmp_path / 'a.ply', torch.from_numpy(verts), torch.from_numpy(faces))
        _write_ply_before(tmp_path / 'b.ply', verts, faces)
        assert (tmp_path / 'a.ply').read_bytes() == (tmp_path / 'b.ply').read_bytes()


def _parse_ply(data):
    end = data.index(b'end_header\n') + len(b'end_header\n')
    header = data[:end].decode('ascii').splitlines()
    nv = int(next(h for h in header if h.startswith('element vertex')).split()[-1])
    nf = int(next(h for h in header if h.startswith('element face')).split()[-1])
    props = [h.split()[1:] for h in header if h.startswith('property') and 'list' not in h]
    dt = np.dtype([(name, {'float': '<f4', 'uchar': 'u1'}[ty]) for ty, name in props])
    v = np.frombuffer(data[end:end + nv * dt.itemsize], dt)
    rec = np.frombuffer(data[end + nv * dt.itemsize:], dtype=[('n', 'u1'), ('idx', '<i4', (3,))])
    assert len(rec) == nf
    return header, [name for _, name in props], v, rec


def test_write_ply_with_normals_and_colors(tmp_path):
    from xrnerf_b200.mesh import write_ply
    rng = np.random.default_rng(2)
    verts = rng.standard_normal((13, 3)).astype(f32)
    faces = rng.integers(0, 13, (7, 3)).astype(np.int32)
    normals = rng.standard_normal((13, 3)).astype(f32)
    colors = rng.uniform(-0.2, 1.2, (13, 3)).astype(f32)
    colors[:2, 0] = [0.0, 1.0]                                          # the ends
    want_rgb = np.floor(np.clip(colors.astype(np.float64), 0, 1) * 255 + 0.5).astype(np.uint8)
    for kw, names in ((dict(normals=normals, colors=colors), ['x', 'y', 'z', 'nx', 'ny', 'nz', 'red', 'green', 'blue']),
                      (dict(normals=torch.from_numpy(normals)), ['x', 'y', 'z', 'nx', 'ny', 'nz']),
                      (dict(colors=torch.from_numpy(colors)), ['x', 'y', 'z', 'red', 'green', 'blue'])):
        write_ply(tmp_path / 'm.ply', torch.from_numpy(verts), torch.from_numpy(faces), **kw)
        header, props, v, rec = _parse_ply((tmp_path / 'm.ply').read_bytes())
        assert props == names
        assert header.index('element vertex 13') < header.index('property float x') < header.index('element face 7')
        assert np.array_equal(np.stack([v['x'], v['y'], v['z']], 1), verts) and np.array_equal(rec['idx'], faces) and (rec['n'] == 3).all()
        if 'normals' in kw:
            assert np.array_equal(np.stack([v['nx'], v['ny'], v['nz']], 1), normals)
        if 'colors' in kw:
            assert np.array_equal(np.stack([v['red'], v['green'], v['blue']], 1), want_rgb)


def test_ngp_to_nerf_normals_matches_the_position_map():
    from xrnerf_b200.mesh import ngp_to_nerf, ngp_to_nerf_normals
    rng = np.random.default_rng(3)
    p = torch.from_numpy(rng.uniform(0, 1, (50, 3)))
    n = torch.from_numpy(rng.standard_normal((50, 3)))
    n = n / torch.linalg.vector_norm(n, dim=1, keepdim=True)
    d = ngp_to_nerf(p + n) - ngp_to_nerf(p)
    want = d / torch.linalg.vector_norm(d, dim=1, keepdim=True)
    got = ngp_to_nerf_normals(n)
    assert torch.allclose(got, want, rtol=0, atol=1e-12)
    assert torch.equal(ngp_to_nerf_normals(torch.zeros((2, 3))), torch.zeros((2, 3))) and ngp_to_nerf_normals(torch.zeros((0, 3))).shape == (0, 3)


# ================================================================================================================ GPU tests
CASES = [(dh, npk) for dh in (1, 2) for npk in (0, 6, 7)]


@pytest.fixture(scope='module', params=CASES, ids=[f'dh{dh}-packed{npk}' for dh, npk in CASES])
def case(request):
    dh, npk = request.param
    f = ngp_field(dh, npk)
    return f, Grid.of(f)


@pytest.mark.gpu
def test_density_is_bit_identical_to_run_density(case):
    field, _ = case
    x = torch.from_numpy(random_points(5000, 10)).cuda()
    rows = torch.full((5000, 7), 9.0, device='cuda')
    rows[:, 2:5] = x
    for pts in (x, rows[:, 2:5]):
        d, g = field.density_grad(pts)
        assert d.shape == (5000, 1) and g.shape == (5000, 3) and d.dtype == torch.float32 and g.dtype == torch.float32
        want = field.run_density(pts, impl=0)
        assert torch.equal(d.view(torch.int32), want.view(torch.int32))
        assert torch.isfinite(g).all()
    assert torch.equal(field.density_grad(rows[:, 2:5])[1].view(torch.int32), field.density_grad(x)[1].view(torch.int32))


def _check_against_restatement(field, grid, x, what, with_density=True):
    dens, g = ngp_density_grad(field, x, with_density)
    if not len(x):
        return 0
    want_d, g64, bound = cuda_core_density_grad(field, grid, x)
    if with_density:
        assert np.array_equal(dens.astype(f32).view(np.uint32), want_d.astype(f32).view(np.uint32)), f'{what}: density differs from the restated CUDA-core forward'
    else:
        assert np.isnan(dens).all()
    err = np.abs(g - g64)
    assert (err <= bound).all(), f'{what}: max err/bound {float((err / np.maximum(bound, 1e-300)).max()):.3g}'
    return float((err / np.maximum(bound, 1e-300)).max())


@pytest.mark.gpu
def test_gradient_within_derived_bound(case):
    field, grid = case
    worst = _check_against_restatement(field, grid, random_points(3000, 11), 'random')
    fp = face_points(grid, 40, 12)
    assert len(fp) >= 200
    worst = max(worst, _check_against_restatement(field, grid, fp, 'faces'))
    for n in (0, 1, 127, 129):
        worst = max(worst, _check_against_restatement(field, grid, random_points(n, 13 + n), f'n={n}'))
    worst = max(worst, _check_against_restatement(field, grid, random_points(300, 14), 'density NULL', with_density=False))
    REPORT.append(f'cfg {field.cfg.density_hidden} / packed {field.n_packed}: max |err| / bound = {worst:.3g}')
    print(REPORT[-1])


def f64_density(grid, mats, x):
    """the float64 function the finite differences differentiate: exact trilinear interpolation of the fp16 table (float64 cell arithmetic), then the
    density net with fp16 weights and no activation rounding -> (density [n], hidden pre-activations list)"""
    enc = np.zeros((x.shape[0], 32))
    for l in range(16):
        px = float(grid.scale[l]) * x + 0.5
        gi = np.floor(px).astype(np.int64)
        _, w = grid.trilinear(px - gi)
        v = grid.corner_values(l, gi)
        enc[:, 2 * l:2 * l + 2] = (w[:, :, None] * v).sum(1)
    a, pre = enc, []
    for W in mats[:-1]:
        z = a @ W.T
        pre.append(z)
        a = np.maximum(z, 0)
    return a @ mats[-1][0], pre, enc


@pytest.mark.gpu
@pytest.mark.parametrize('dh', [1, 2])
def test_gradient_matches_finite_differences(dh):
    """Central differences of the float64 function (fp16 parameters, no activation rounding). Inside one cell of every level and with every ReLU
    decision fixed, that function is linear along each axis, so the difference quotient is its derivative up to float64 rounding. The kernel differs
    from it by its fp32 rounding (the restatement's bound), by its in-cell positions being fp32 (|df| <= 2^-24 (scale_l + 1) per axis, moving the
    weight products by at most the sum over the other two axes) and by the difference quotient's float64 rounding."""
    field = ngp_field(dh, 6, seed=5)
    grid = Grid.of(field)
    mats = field_mats(field)
    h = 2.0 ** -20
    x = random_points(6000, 21).astype(np.float64)
    keep = np.ones(len(x), bool)
    for l in range(16):                                                   # every level: at least 4 h scale_l from a cell face
        f = float(grid.scale[l]) * x + 0.5
        f -= np.floor(f)
        keep &= ((f > 4 * h * grid.scale[l]) & (f < 1 - 4 * h * grid.scale[l])).all(1)
    _, pre0, _ = f64_density(grid, mats, x)
    sides = []
    for a in range(3):
        for s in (-1, 1):
            xs = x.copy(); xs[:, a] += s * h
            d, pre, _ = f64_density(grid, mats, xs)
            sides.append(d)
            for z0, z in zip(pre0, pre):
                keep &= ((z0 > 0) == (z > 0)).all(1)
    xk = x.astype(f32)
    _, masks_k = cuda_core_density(mats, hashgrid_enc16(field, xk))
    for z0, mk in zip(pre0, masks_k):                                     # the kernel's masks (fp16 activation > 0) are the float64 function's
        keep &= ((z0 > 0) == mk).all(1)
    assert keep.sum() >= 1000, keep.sum()
    fd = np.stack([(sides[2 * a + 1] - sides[2 * a]) / (2 * h) for a in range(3)], 1)[keep]
    _, g = ngp_density_grad(field, xk[keep])
    _, _, bound = cuda_core_density_grad(field, grid, xk[keep])
    # the in-cell positions: the kernel's are fp32 (|df| <= 2^-24 (scale_l + 1) per axis), which moves dw_c/df_a by at most the sum of |df| over the
    # other two axes; the float64 function's are rounded too (2^-53 (scale_l + 1)), which moves each side's value by the level's |dF/df| times that
    ge, gea = enc_grad(mats, [m[keep] for m in masks_k])
    cellpos, fd_err = np.zeros((keep.sum(), 3)), np.zeros(keep.sum())
    enc_abs = np.zeros((keep.sum(), 32))
    for l in range(16):
        gi, fk = grid.cell(l, xk[keep])
        v = grid.corner_values(l, gi)
        dw, w = grid.trilinear(fk)
        sa = np.abs(v[:, :, 0]) * gea[:, None, 2 * l] + np.abs(v[:, :, 1]) * gea[:, None, 2 * l + 1]
        sc = float(grid.scale[l])
        cellpos += sc * 2 * U32 * (sc + 1) * sa.sum(1)[:, None] * 1.0001
        fd_err += 2 * U64 * (sc + 1) * (np.abs(dw).sum(2) * sa).sum(1) * 1.0001 / (2 * h)
        enc_abs[:, 2 * l:2 * l + 2] = (w[:, :, None] * np.abs(v)).sum(1)
    # and each side's float64 value is within gamma_n(u64) of its sum of absolute terms (n = 16 * 8 roundings of the encoding + the net's chains)
    mass = enc_abs @ np.abs(mats[0]).T
    for W in mats[1:-1]:
        mass = mass @ np.abs(W).T
    mass = mass @ np.abs(mats[-1][0])
    fd_err += 2 * gamma(16 * 8 + 64 * dh + 64, U64) * mass * 1.0001 / (2 * h) + U64 * np.abs(fd).max(1)
    tol = bound + cellpos + fd_err[:, None]
    err = np.abs(g - fd)
    assert (err <= tol).all(), f'max err/tol {float((err / tol).max()):.3g}'
    REPORT.append(f'finite differences, density_hidden {dh}: {int(keep.sum())} points, max |kernel - fd| / tol = {float((err / tol).max()):.3g}')
    print(REPORT[-1])


@pytest.mark.gpu
def test_sphere_normals():
    from xrnerf_b200.mesh import marching_cubes, raw_density_threshold
    net, grid = sphere_network()
    field = net.mlp.field
    sigma = math.exp(SPHERE_THR)                                         # the sampler's density activation is exponential
    verts, faces, normals, colors = net.extract_colored_mesh(resolution=128, threshold=sigma)
    assert len(faces) > 10000
    vw = marching_cubes(field.density_lattice((128,) * 3), raw_density_threshold(sigma, 3))[0]
    x = vw.cpu().numpy()
    # the kernel's gradient is the interpolant's: the restatement with d(out 0)/d(encoding) = e_8
    _, g = ngp_density_grad(field, x)
    dens, g64, bound = cuda_core_density_grad(field, grid, x)
    assert (dens > 0).all() and (np.abs(g - g64) <= bound).all()
    n = normals.cpu().numpy().astype(np.float64)
    v, fc = verts.cpu().numpy().astype(np.float64), faces.cpu().numpy()
    fn = np.cross(v[fc[:, 1]] - v[fc[:, 0]], v[fc[:, 2]] - v[fc[:, 0]])  # counter-clockwise seen from outside: outward, |.| = 2 area
    vn = np.zeros_like(v)
    for k in range(3):
        np.add.at(vn, fc[:, k], fn)
    assert ((n * vn).sum(1) > 0).all()
    radial = x.astype(np.float64) - SPHERE_C
    radial /= np.linalg.norm(radial, axis=1, keepdims=True)
    ang = lambda a, b: np.arccos(np.clip((a * b).sum(1) / np.linalg.norm(a, axis=1) / np.linalg.norm(b, axis=1), -1, 1))
    got = ang(n, radial)
    # bound: the float64 interpolant's angle, plus how far the kernel's gradient can turn from it (|err| / |g64|), plus the fp32 normalisation
    # (relative error <= 4 u per component)
    gnorm = np.linalg.norm(g64, axis=1)
    turn = np.arcsin(np.minimum(1.0, np.linalg.norm(bound, axis=1) / gnorm))
    limit = float((ang(-g64, radial) + turn).max()) + 4 * math.sqrt(3) * U32
    REPORT.append(f'sphere at 128^3: {len(x)} vertices, max angle to the radial direction {math.degrees(got.max()):.3f} deg (bound {math.degrees(limit):.3f} deg)')
    print(REPORT[-1])
    assert got.max() <= limit


@pytest.mark.gpu
def test_extract_colored_mesh_equals_its_parts():
    from xrnerf_b200.mesh import marching_cubes, activate_rgb, raw_density_threshold
    net = ngp_network()
    field = net.mlp.field
    vol = field.density_lattice((48, 48, 48))
    sigma = math.exp(float(torch.quantile(vol.reshape(-1)[::7], 0.7)))
    net.sampler.aabb_range = (-1.5, 2.5)
    verts, faces, normals, colors = net.extract_colored_mesh(resolution=48, threshold=sigma)
    v0, f0 = net.extract_mesh(resolution=48, threshold=sigma)
    assert len(f0) > 100
    assert torch.equal(verts.view(torch.int32), v0.view(torch.int32)) and torch.equal(faces, f0)
    vw = marching_cubes(field.density_lattice((48, 48, 48)), raw_density_threshold(sigma, 3))[0]
    _, g = field.density_grad(vw)
    norm = torch.linalg.vector_norm(g, dim=1, keepdim=True)
    want_n = torch.where(norm > 0, -g / norm, torch.zeros_like(g))
    assert torch.equal(normals.view(torch.int32), want_n.view(torch.int32))
    want_c = activate_rgb(field.run_mlp(vw, (-want_n + 1) / 2)[:, :3], 2)
    assert torch.equal(colors.view(torch.int32), torch.sigmoid(field.run_mlp(vw, (-want_n + 1) / 2)[:, :3]).view(torch.int32))
    assert torch.equal(colors, want_c)
    ln = torch.linalg.vector_norm(normals.double(), dim=1)
    assert ((ln == 0) | ((ln - 1).abs() <= 8 * U32)).all()
    assert (colors >= 0).all() and (colors <= 1).all()
    for t in (verts, normals, colors):
        assert t.is_cuda and t.dtype == torch.float32 and t.shape == (len(verts), 3)
    empty = net.extract_colored_mesh(resolution=32, threshold=math.exp(float(vol.max()) + 1.0))
    assert all(t.shape == (0, 3) and t.is_cuda for t in empty)


def test_report():
    for line in REPORT:
        print(line)
