"""NGP mesh export: the field's density on a lattice (xrb_ngp_density_lattice, NgpField.density_lattice), marching cubes (xrb_mc_count /
xrb_mc_emit, xrnerf_b200.mesh.marching_cubes) and HashNerfNetwork.extract_mesh.

The marching-cubes kernels are compared bit for bit, in order, with `mc_oracle`, a numpy restatement of the contract in include/xrnerf_b200.h
over the triangulation table that scripts/gen_mc_table.py generates. That the table is right is not taken from the table itself: the oracle's
meshes (CPU tests) and the kernels' meshes (GPU tests) must be closed and consistently oriented, with outward normals, the right Euler
characteristic and, at 128^3, the analytic enclosed volume and area."""
import math

import numpy as np
import pytest
import torch
from cases import NGP_MODEL, cpu_args, dev
from restate64 import GEN, area, check_closed_oriented, euler, lattice_coords, mc_oracle

f32 = np.float32


# ---------------------------------------------------------------------------------------------------------------- volumes
def grid(shape):
    nz, ny, nx = shape
    z, y, x = np.meshgrid(*(np.linspace(0, 1, n, dtype=np.float64) for n in (nz, ny, nx)), indexing='ij')
    return x, y, z


def sphere(shape, c=(0.5, 0.5, 0.5), r=0.3):
    x, y, z = grid(shape)
    return (r - np.sqrt((x - c[0]) ** 2 + (y - c[1]) ** 2 + (z - c[2]) ** 2)).astype(f32)      # > 0 inside


def torus(shape, R=0.28, r=0.1):
    x, y, z = grid(shape)
    q = np.sqrt((x - 0.5) ** 2 + (y - 0.5) ** 2) - R
    return (r - np.sqrt(q ** 2 + (z - 0.5) ** 2)).astype(f32)


def two_spheres(shape):
    return np.maximum(sphere(shape, (0.28, 0.5, 0.5), 0.18), sphere(shape, (0.72, 0.5, 0.5), 0.18))


def smooth_noise(shape, seed=0, k=6):
    """a sum of random low-frequency cosines, zero on the boundary layer's outside (multiplied by a bump) so its level sets are closed"""
    rng = np.random.default_rng(seed)
    x, y, z = grid(shape)
    v = np.zeros(x.shape)
    for _ in range(k):
        w = rng.uniform(-9, 9, 3)
        v += np.cos(w[0] * x + w[1] * y + w[2] * z + rng.uniform(0, 6.3))
    bump = (x * (1 - x) * y * (1 - y) * z * (1 - z)) * 64
    return ((v / k * 0.5 + 0.5) * bump - 0.05).astype(f32)


def single_case(case):
    """4^3 volume, outside everywhere except the corners of cell (1,1,1) that `case` sets"""
    v = np.full((4, 4, 4), -1.0, f32)
    for c in range(8):
        if (case >> c) & 1:
            v[1 + ((c >> 2) & 1), 1 + ((c >> 1) & 1), 1 + (c & 1)] = 1.0
    return v


def random_binary(shape, seed):
    rng = np.random.default_rng(seed)
    v = np.where(rng.random(shape) < 0.5, 1.0, -1.0).astype(f32) * rng.uniform(0.5, 2.0, shape).astype(f32)
    v[0], v[-1], v[:, 0], v[:, -1], v[:, :, 0], v[:, :, -1] = -1, -1, -1, -1, -1, -1
    return v


# relative error of the enclosed volume and the area at 128^3 against the analytic values. The oracle's meshes measure: sphere (r 0.3) volume
# -4.1e-4, area -2.2e-4; torus (0.28, 0.1) volume -1.29e-3, area -3.5e-4 (test_oracle_topology_and_geometry). The bounds leave 2x to 3x headroom.
VOL_RTOL, AREA_RTOL = 2.5e-3, 1e-3
SPHERE_V, SPHERE_A = 4 / 3 * math.pi * 0.3 ** 3, 4 * math.pi * 0.3 ** 2
TORUS_V, TORUS_A = 2 * math.pi ** 2 * 0.28 * 0.1 ** 2, 4 * math.pi ** 2 * 0.28 * 0.1


# ================================================================================================================ CPU tests
def test_generator_reproduces_committed_table():
    with open(GEN.HEADER) as fh:
        assert fh.read() == GEN.render_header()


def test_oracle_closed_for_every_single_cube_case():
    for case in range(1, 255):
        verts, faces = mc_oracle(single_case(case), 0.0)
        check_closed_oriented(verts, faces)
    assert mc_oracle(single_case(0), 0.0)[1].shape == (0, 3)


def test_oracle_closed_on_random_binary_volumes():
    for seed in range(20):
        verts, faces = mc_oracle(random_binary((9, 10, 11), seed), 0.0)
        check_closed_oriented(verts, faces)


def test_oracle_topology_and_geometry():
    s = mc_oracle(sphere((128, 128, 128)), 0.0)
    t = mc_oracle(torus((128, 128, 128)), 0.0)
    two = mc_oracle(two_spheres((64, 64, 64)), 0.0)
    assert euler(*s) == 2 and euler(*t) == 0 and euler(*two) == 4
    for (v, f), V, A in ((s, SPHERE_V, SPHERE_A), (t, TORUS_V, TORUS_A)):
        assert abs(check_closed_oriented(v, f) - V) <= VOL_RTOL * V
        assert abs(area(v, f) - A) <= AREA_RTOL * A
    check_closed_oriented(*mc_oracle(smooth_noise((40, 33, 47)), 0.0))


def test_mesh_entry_points_validate_arguments_without_gpu():
    _C, _buf, p, cfg, tab = cpu_args()
    lib = _C.lib
    unit = (_C.float3((0, 0, 0)), _C.float3((1, 1, 1)))
    lattice = lambda n, box=unit, out=p: lib.xrb_ngp_density_lattice(cfg, tab, p, p, n[0], n[1], n[2], box[0], box[1], out, 1, p, None)
    count = lambda n, thr=0.0, ws=p: lib.xrb_mc_count(p, n[0], n[1], n[2], thr, ws, p, None)
    emit = lambda n, thr=0.0, box=unit, verts=p: lib.xrb_mc_emit(p, n[0], n[1], n[2], thr, box[0], box[1], p, verts, p, None)
    for fn in (lattice, count, emit):
        for n in ((1, 4, 4), (4, 1025, 4), (4, 4, -2)):
            assert fn(n) == -1 and b'bad size' in lib.xrb_last_error()
        assert fn((0, 5, 5)) == 0 and fn((0, 0, 0)) == 0                   # an empty lattice is a no-op
    for box in (((0, 0, -0.01), (1, 1, 1)), ((0, 0, 0), (1, 1.5, 1)), ((0.5, 0, 0), (0.25, 1, 1)), ((0.5, 0, 0), (0.5, 1, 1)), ((float('nan'), 0, 0), (1, 1, 1))):
        assert lattice((4, 4, 4), (_C.float3(box[0]), _C.float3(box[1]))) == -1 and b'box' in lib.xrb_last_error()
    assert lattice((4, 4, 4), out=None) == -1 and b'null' in lib.xrb_last_error()
    assert lib.xrb_ngp_density_lattice(cfg, tab, p, p, 4, 4, 4, None, unit[1], p, 1, p, None) == -1
    assert lib.xrb_ngp_density_lattice(None, tab, p, p, 4, 4, 4, unit[0], unit[1], p, 1, p, None) == -1
    assert lib.xrb_ngp_density_lattice(cfg, tab, p, None, 4, 4, 4, unit[0], unit[1], p, 1, p, None) == -1 and b'weights' in lib.xrb_last_error()
    # marching cubes: any box with box_min < box_max, a threshold that is not NaN, every pointer
    assert emit((4, 4, 4), box=(_C.float3((-2, -2, -2)), _C.float3((3, 3, 3))), verts=None) == -1 and b'null' in lib.xrb_last_error()
    assert emit((4, 4, 4), box=(_C.float3((0, 0, 1)), _C.float3((1, 1, 1)))) == -1 and b'box' in lib.xrb_last_error()
    for fn in (count, emit):
        assert fn((4, 4, 4), thr=float('nan')) == -1 and b'NaN' in lib.xrb_last_error()
    assert count((4, 4, 4), ws=None) == -1 and b'null' in lib.xrb_last_error()
    assert lib.xrb_mc_count(None, 4, 4, 4, 0.0, p, p, None) == -1 and lib.xrb_mc_count(p, 4, 4, 4, 0.0, p, None, None) == -1
    assert lib.xrb_mc_workspace(1, 4, 4) == 0
    assert lib.xrb_mc_workspace(37, 64, 50) == 4 * (37 * 64 * 50 + 2 * ((37 * 64 * 50 + 255) // 256) + 4)   # 4 bytes per point + O(blocks)
    assert lib.xrb_ngp_density_lattice_workspace() == 12 * (1 << 20)


def test_write_ply_round_trip(tmp_path):
    from xrnerf_b200.mesh import write_ply
    rng = np.random.default_rng(0)
    verts = rng.standard_normal((7, 3)).astype(f32)
    faces = rng.integers(0, 7, (5, 3)).astype(np.int32)
    path = tmp_path / 'm.ply'
    write_ply(path, torch.from_numpy(verts), torch.from_numpy(faces))
    data = path.read_bytes()
    end = data.index(b'end_header\n') + len(b'end_header\n')
    header = data[:end].decode('ascii').splitlines()
    assert header[:2] == ['ply', 'format binary_little_endian 1.0']
    assert 'element vertex 7' in header and 'element face 5' in header and 'property list uchar int vertex_indices' in header
    body = data[end:]
    v = np.frombuffer(body[:7 * 12], '<f4').reshape(7, 3)
    rec = np.frombuffer(body[7 * 12:], dtype=[('n', 'u1'), ('idx', '<i4', (3,))])
    assert len(body) == 7 * 12 + 5 * 13
    assert np.array_equal(v, verts) and (rec['n'] == 3).all() and np.array_equal(rec['idx'], faces)
    write_ply(tmp_path / 'e.ply', np.zeros((0, 3), f32), np.zeros((0, 3), np.int32))
    assert (tmp_path / 'e.ply').read_bytes().endswith(b'element face 0\nproperty list uchar int vertex_indices\nend_header\n')


def test_ngp_to_nerf_recovers_camera_centres():
    from xrnerf_b200 import synth
    from xrnerf_b200.mesh import ngp_to_nerf
    poses = np.stack([synth.pose_spherical(a, -30.0, 4.0) for a in np.linspace(-180, 180, 9)[:-1]], 0)
    ngp = synth.poses_nerf2ngp(poses)                       # [I,4,3]: row 3 is the camera centre in the field's frame
    back = ngp_to_nerf(torch.from_numpy(ngp[:, 3, :]).double()).numpy()
    assert np.abs(back - poses[:, :3, 3]).max() <= 1e-6
    assert ngp_to_nerf(torch.zeros((0, 3))).shape == (0, 3)


def test_density_threshold_mapping():
    from xrnerf_b200.mesh import raw_density_threshold as raw
    assert raw(2.5, 3) == pytest.approx(math.log(2.5), abs=0) and raw(2.5, 0) == 2.5 and raw(-1.0, 0) == -1.0 and raw(2.5, 1) == 2.5 and raw(0.0, 1) == 0.0
    assert raw(0.25, 2) == pytest.approx(math.log(1 / 3), rel=1e-15)
    for act in (0, 1, 2, 3):
        for s in (0.01, 0.5, 0.99):
            r = raw(s, act)
            assert {0: r, 1: max(r, 0.0), 2: 1 / (1 + math.exp(-r)), 3: math.exp(r)}[act] == pytest.approx(s, rel=1e-12)
    for s, act in ((0.0, 3), (-1.0, 3), (-0.5, 1), (0.0, 2), (1.0, 2), (1.5, 2), (float('nan'), 0), (float('inf'), 3), (1.0, 4)):
        with pytest.raises(ValueError):
            raw(s, act)


# ================================================================================================================ GPU tests
def gpu_mc(vol, thr, box=((0, 0, 0), (1, 1, 1))):
    from xrnerf_b200.mesh import marching_cubes
    v, f = marching_cubes(dev(vol), thr, box)
    torch.cuda.synchronize()
    return v.cpu().numpy(), f.cpu().numpy()


def assert_same_mesh(got, want):
    assert got[0].dtype == np.float32 and got[1].dtype == np.int32
    assert got[0].shape == want[0].shape and got[1].shape == want[1].shape
    assert np.array_equal(got[0].view(np.uint32), want[0].view(np.uint32)), 'vertices differ from the oracle'
    assert np.array_equal(got[1], want[1]), 'triangles differ from the oracle'


def _volumes():
    rng = np.random.default_rng(5)
    plateau = np.round(sphere((30, 31, 29)) * 16).astype(f32) / 16       # many lattice values equal to the threshold 0
    return {
        'sphere': (sphere((64, 64, 64)), 0.0, ((0, 0, 0), (1, 1, 1))),
        'torus_37x64x50': (torus((50, 64, 37)), 0.0, ((-1, 0, 2), (1, 0.5, 3))),
        'two_spheres': (two_spheres((33, 47, 65)), 0.0, ((0, 0, 0), (1, 1, 1))),
        'noise': (smooth_noise((61, 40, 77), seed=2), 0.0, ((0.1, 0.2, 0.3), (0.9, 0.7, 0.8))),
        'noise_open': (rng.standard_normal((19, 23, 300)).astype(f32), 0.3, ((0, 0, 0), (1, 1, 1))),
        'plateau': (plateau, 0.0, ((0, 0, 0), (1, 1, 1))),
        'small': (sphere((2, 3, 2), r=0.8), 0.0, ((0, 0, 0), (1, 1, 1))),
    }


@pytest.mark.gpu
@pytest.mark.parametrize('name', sorted(_volumes()))
def test_marching_cubes_matches_oracle_bit_for_bit(name):
    vol, thr, box = _volumes()[name]
    want = mc_oracle(vol, thr, box)
    assert len(want[1]) > 0
    assert_same_mesh(gpu_mc(vol, thr, box), want)
    if name == 'plateau':
        assert (vol == thr).sum() > 100


@pytest.mark.gpu
def test_marching_cubes_empty_and_full_volumes():
    for vol in (np.zeros((17, 9, 33), f32), np.ones((17, 9, 33), f32)):
        v, f = gpu_mc(vol, 0.5)
        assert v.shape == (0, 3) and f.shape == (0, 3)
    v, f = gpu_mc(np.ones((17, 9, 33), f32), 0.0)                        # everything inside: the mesh is the open boundary of nothing -> empty
    assert v.shape == (0, 3) and f.shape == (0, 3)


@pytest.mark.gpu
def test_marching_cubes_closed_for_every_single_cube_case():
    for case in range(1, 255):
        got = gpu_mc(single_case(case), 0.0)
        assert_same_mesh(got, mc_oracle(single_case(case), 0.0))
        check_closed_oriented(*got)


@pytest.mark.gpu
def test_marching_cubes_closed_on_random_binary_volumes():
    for seed in range(8):
        vol = random_binary((24, 29, 31), seed)
        got = gpu_mc(vol, 0.0)
        assert_same_mesh(got, mc_oracle(vol, 0.0))
        check_closed_oriented(*got)


@pytest.mark.gpu
def test_marching_cubes_topology_and_geometry_at_128():
    s, t = gpu_mc(sphere((128, 128, 128)), 0.0), gpu_mc(torus((128, 128, 128)), 0.0)
    two = gpu_mc(two_spheres((64, 64, 64)), 0.0)
    assert euler(*s) == 2 and euler(*t) == 0 and euler(*two) == 4
    for (v, f), V, A in ((s, SPHERE_V, SPHERE_A), (t, TORUS_V, TORUS_A)):
        assert abs(check_closed_oriented(v, f) - V) <= VOL_RTOL * V
        assert abs(area(v, f) - A) <= AREA_RTOL * A
    check_closed_oriented(*two)
    check_closed_oriented(*gpu_mc(smooth_noise((70, 81, 90), seed=4), 0.0))


@pytest.fixture(scope='module')
def field():
    from xrnerf_b200 import synth
    from xrnerf_b200.ngp import NgpField
    f = NgpField().cuda()
    table, dens, color = synth.ngp_weights(seed=3, hash_range=0.5, mlp_gain=2.0)
    with torch.no_grad():
        f.hash_params.copy_(dev(table)); f.density_params.copy_(dev(dens)); f.color_params.copy_(dev(color))
    return f


def lattice_positions(shape, box):
    """[N,3] float32 positions of the lattice (x fastest), restated on the CPU with the formula of xrb_ngp_density_lattice"""
    nz, ny, nx = shape
    cx, cy, cz = (lattice_coords(box[0][a], box[1][a], n) for a, n in enumerate((nx, ny, nz)))
    z, y, x = np.meshgrid(cz, cy, cx, indexing='ij')
    return np.stack([x.reshape(-1), y.reshape(-1), z.reshape(-1)], 1)


@pytest.mark.gpu
@pytest.mark.parametrize('impl', [1, 0])
def test_density_lattice_matches_run_density(field, impl):
    for shape, box in (((64, 64, 64), ((0, 0, 0), (1, 1, 1))), ((50, 64, 37), ((0, 0, 0), (1, 1, 1))), ((33, 20, 47), ((0.1, 0.25, 0.3), (0.6, 0.9, 0.7))),
                       ((2, 3, 1024), ((0, 0.5, 0.5), (1, 0.75, 1)))):
        got = field.density_lattice(shape, box, impl=impl)
        pts = dev(lattice_positions(shape, box))
        assert float(pts.min()) >= 0 and float(pts.max()) <= 1
        want = field.run_density(pts, impl=impl).reshape(shape)
        assert got.shape == shape and torch.equal(got.view(torch.int32), want.view(torch.int32))
    big = (130, 100, 90)                                                 # more points than one staging chunk (2^20)
    got = field.density_lattice(big, impl=impl)
    assert torch.equal(got.view(torch.int32), field.run_density(dev(lattice_positions(big, ((0, 0, 0), (1, 1, 1)))), impl=impl).reshape(big).view(torch.int32))


def _network():
    from xrnerf_b200 import registry as R, synth
    net = R.build_network(NGP_MODEL).cuda()
    table, dens, color = synth.ngp_weights(seed=3, hash_range=0.5, mlp_gain=2.0)
    with torch.no_grad():
        f = net.mlp.field
        f.hash_params.copy_(dev(table)); f.density_params.copy_(dev(dens)); f.color_params.copy_(dev(color))
    return net


@pytest.mark.gpu
def test_extract_mesh_equals_its_parts():
    from xrnerf_b200.mesh import marching_cubes
    net = _network()
    field = net.mlp.field
    vol = field.density_lattice((48, 48, 48))
    thr = float(torch.quantile(vol.reshape(-1)[::7], 0.7))            # a level set that crosses this untrained field
    sigma = math.exp(thr)                                              # the sampler's density activation is exponential
    net.sampler.aabb_range = (-1.5, 2.5)
    verts, faces = net.extract_mesh(resolution=48, threshold=sigma)
    v0, f0 = marching_cubes(vol, math.log(sigma))
    assert len(f0) > 100
    assert torch.equal(faces, f0) and torch.equal(verts.view(torch.int32), (v0 * (2.5 - -1.5) + -1.5).view(torch.int32))
    v2, f2 = net.extract_mesh(resolution=48, threshold=sigma)
    assert torch.equal(v2.view(torch.int32), verts.view(torch.int32)) and torch.equal(f2, faces)
    # different weights through load_state_dict: the next mesh reflects them (the field was refreshed)
    sd = {k: v.clone() for k, v in net.state_dict().items()}
    key = next(k for k in sd if 'density_net' in k)
    sd[key] = sd[key] * 0.5
    net.load_state_dict(sd)
    v3, f3 = net.extract_mesh(resolution=48, threshold=sigma)
    assert not (v3.shape == verts.shape and torch.equal(v3, verts))
    vol3 = net.mlp.field.density_lattice((48, 48, 48))
    assert torch.equal(f3, marching_cubes(vol3, math.log(sigma))[1])
    del net.sampler.aabb_range                                           # before set_data: the unit cube
    v4, _ = net.extract_mesh(resolution=48, threshold=sigma)
    assert torch.equal(v4.view(torch.int32), (marching_cubes(vol3, math.log(sigma))[0] * (1.0 - 0.0) + 0.0).view(torch.int32))
