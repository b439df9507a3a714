"""Triangle meshes of a density volume: marching cubes on the GPU (xrb_mc_count / xrb_mc_emit, include/xrnerf_b200.h), a binary PLY writer, and
the map from the Instant-NGP field's frame back to the dataset's (Blender / NeRF) world frame.

    verts, faces = network.extract_mesh(resolution=256)          # HashNerfNetwork: vertices in the frame the rays are given in
    write_ply('mesh.ply', ngp_to_nerf(verts), faces)
    verts, faces, normals, colors = network.extract_colored_mesh(resolution=256)
    write_ply('mesh.ply', ngp_to_nerf(verts), faces, ngp_to_nerf_normals(normals), colors)

    verts, faces = nerf_network.extract_mesh(resolution=256)     # NerfNetwork: vertices and normals already in the NeRF world frame
    verts, faces, normals, colors = nerf_network.extract_colored_mesh(resolution=256)
    write_ply('mesh.ply', verts, faces, normals, colors)

    verts, faces, normals, colors = mip_network.extract_colored_mesh(resolution=256, footprint='cell')   # MipNerfNetwork: a footprint is required
"""
import numpy as np
import torch

from . import _C


def marching_cubes(volume, threshold, box=((0.0, 0.0, 0.0), (1.0, 1.0, 1.0))):
    """volume: CUDA f32[nz,ny,nx] (x fastest), each size 2..1024. -> (verts f32[V,3], faces i32[F,3]) CUDA tensors, vertices in the coordinates of
    box = (box_min, box_max), which the lattice spans. A value is inside iff it is > threshold; triangles wind counter-clockwise seen from outside.
    Order and rounding: xrb_mc_emit. Waits for the device once, to size the outputs."""
    _C.require_cuda(volume)
    if volume.dim() != 3:
        raise _C.XrbError(f'XRB_E_BADARG: volume must be [nz,ny,nx], got {tuple(volume.shape)}')
    nz, ny, nx = volume.shape
    dev = volume.device
    ws = torch.empty(_C.lib.xrb_mc_workspace(nx, ny, nz), dtype=torch.uint8, device=dev)
    counts = torch.zeros(2, dtype=torch.int32, device=dev)
    _C.check(_C.lib.xrb_mc_count(_C.f32(volume), nx, ny, nz, float(threshold), _C.ptr(ws), _C.i32(counts), _C.stream()), 'mc_count')
    n_verts, n_faces = (int(v) for v in counts.tolist())
    if n_verts < 0:
        raise _C.XrbError('marching cubes: more than 2^31 - 1 vertices or triangles')
    verts = torch.empty((n_verts, 3), dtype=torch.float32, device=dev)
    faces = torch.empty((n_faces, 3), dtype=torch.int32, device=dev)
    if n_verts:
        _C.check(_C.lib.xrb_mc_emit(_C.f32(volume), nx, ny, nz, float(threshold), _C.float3(box[0]), _C.float3(box[1]), _C.ptr(ws), _C.f32(verts), _C.i32(faces),
                                    _C.stream()), 'mc_emit')
    return verts, faces


def write_ply(path, verts, faces, normals=None, colors=None):
    """Binary little-endian PLY: `element vertex` with float x, y, z, then float nx, ny, nz when `normals` [V,3] is given, then uchar red, green, blue when
    `colors` [V,3] in [0,1] is given (each channel floor(clamp(c, 0, 1) * 255 + 0.5)), interleaved per vertex; `element face` with list uchar int
    vertex_indices."""
    v = np.ascontiguousarray(torch.as_tensor(verts).detach().cpu().numpy(), dtype='<f4').reshape(-1, 3)
    f = np.ascontiguousarray(torch.as_tensor(faces).detach().cpu().numpy(), dtype='<i4').reshape(-1, 3)
    fields, props = [('xyz', '<f4', (3,))], 'property float x\nproperty float y\nproperty float z\n'
    if normals is not None:
        fields.append(('n', '<f4', (3,)))
        props += 'property float nx\nproperty float ny\nproperty float nz\n'
    if colors is not None:
        fields.append(('rgb', 'u1', (3,)))
        props += 'property uchar red\nproperty uchar green\nproperty uchar blue\n'
    vrec = np.empty(len(v), dtype=fields)
    vrec['xyz'] = v
    if normals is not None:
        vrec['n'] = np.asarray(torch.as_tensor(normals).detach().cpu().numpy(), dtype='<f4').reshape(-1, 3)
    if colors is not None:
        c = np.asarray(torch.as_tensor(colors).detach().cpu().numpy(), dtype=np.float64).reshape(-1, 3)
        vrec['rgb'] = np.floor(np.clip(c, 0.0, 1.0) * 255.0 + 0.5).astype(np.uint8)
    rec = np.empty(len(f), dtype=[('n', 'u1'), ('idx', '<i4', (3,))])
    rec['n'] = 3
    rec['idx'] = f
    header = ('ply\nformat binary_little_endian 1.0\n'
              f'element vertex {len(v)}\n{props}'
              f'element face {len(f)}\nproperty list uchar int vertex_indices\nend_header\n')
    with open(path, 'wb') as fh:
        fh.write(header.encode('ascii'))
        fh.write(vrec.tobytes())
        fh.write(rec.tobytes())


def ngp_to_nerf(verts, scale=0.33, offset=(0.5, 0.5, 0.5)):
    """Inverse of the position map of synth.poses_nerf2ngp (and the reference's NGP loader): there a NeRF point p becomes
    (p * scale + offset)[[1, 2, 0]]; here a point q of the field's frame becomes p with p[[1, 2, 0]] = q, then (p - offset) / scale."""
    q = torch.as_tensor(verts)
    p = q[:, [2, 0, 1]]
    return (p - torch.as_tensor(offset, dtype=p.dtype, device=p.device)) / scale


def ngp_to_nerf_normals(normals):
    """Normals (directions) of the field's frame in the NeRF world frame: the axis permutation of ngp_to_nerf. Its scale is positive and uniform, so it
    drops out of a unit normal; zero normals stay zero."""
    return torch.as_tensor(normals)[:, [2, 0, 1]]


def outward_normals(g):
    """-g / |g| per row of g f32[n,3] (0 where g = 0): the outward unit normal of a level set whose inside is where the field exceeds the level"""
    norm = torch.linalg.vector_norm(g, dim=1, keepdim=True)
    return torch.where(norm > 0, -g / norm, torch.zeros_like(g))


def footprint_sigma(footprint, shape=None, box=None):
    """The standard deviation sigma of a Mip-NeRF point query (include/xrnerf_b200.h, Mip-NeRF mesh export) -> float. `footprint` is sigma itself,
    finite and >= 0, in the world frame of the rays; or 'cell': sigma = h / sqrt(12) with h = max over axes of (hi - lo) / (n - 1), the standard
    deviation of a uniform distribution over one cell of the lattice of shape (nz, ny, nx) over box = (box_min, box_max), so that a mesh sampled at
    resolution n sees the field filtered at its own spacing. ValueError for a negative or non-finite sigma or an unknown string."""
    if isinstance(footprint, str):
        if footprint != 'cell':
            raise ValueError(f"footprint must be a number sigma >= 0 or 'cell', got {footprint!r}")
        if shape is None or box is None:
            raise ValueError("footprint 'cell' needs a lattice: pass the point query's sigma")
        nz, ny, nx = (int(n) for n in shape)
        h = max([(float(box[1][a]) - float(box[0][a])) / (n - 1) for a, n in enumerate((nx, ny, nz)) if n >= 2] or [0.0])
        s = h / np.sqrt(12.0)
    else:
        s = float(footprint)
    if not (0.0 <= s <= float(np.finfo(np.float32).max)):                     # finite as the fp32 the kernels take (NaN fails too)
        raise ValueError(f'footprint sigma must be finite and >= 0, got {footprint}')
    return s


def raw_density_threshold(sigma, activation, density_bias=0.0):
    """The raw network output whose activated density is sigma (the NGP sampler's density_activation code: 0 None, 1 ReLU, 2 Logistic, 3 Exponential;
    or NerfRender's density_activation name: 'relu', or 'softplus' with threshold 20 as in the NeRF composite, the library's code 4), the activation
    applied to raw + density_bias: v > raw  <=>  act(v + density_bias) > sigma. ValueError when sigma is outside the activation's range (or the
    activation is unknown)."""
    s = float(sigma)
    act = {'relu': 1, 'softplus': 4}.get(activation, -1) if isinstance(activation, str) else int(activation)
    if act == 4 and not isinstance(activation, str):
        act = -1                                   # the sampler codes stop at 3
    if not np.isfinite(s):
        raise ValueError(f'density threshold must be finite, got {sigma}')
    return _inverse_density_act(s, act) - float(density_bias)


def _inverse_density_act(s, act):
    if act == 0:
        return s
    if act == 1:
        if s < 0:
            raise ValueError(f'a ReLU density is never negative: threshold {s}')
        return s
    if act == 4:
        if s <= 0:
            raise ValueError(f'a softplus density is positive: threshold {s}')
        return s if s > 20.0 else float(np.log(np.expm1(s)))   # softplus(v) = v above 20
    if act == 2:
        if not 0.0 < s < 1.0:
            raise ValueError(f'a logistic density lies in (0, 1): threshold {s}')
        return float(np.log(s) - np.log1p(-s))
    if act == 3:
        if s <= 0:
            raise ValueError(f'an exponential density is positive: threshold {s}')
        return float(np.log(s))
    raise ValueError('unknown density activation')


def activate_rgb(raw, activation):
    """The sampler's rgb_activation (0 None, 1 ReLU, 2 Logistic, 3 Exponential of the value clamped to [-10, 10], as the composite applies it) on a tensor"""
    act = int(activation)
    if act == 0:
        return raw
    if act == 1:
        return torch.relu(raw)
    if act == 2:
        return torch.sigmoid(raw)
    if act == 3:
        return torch.exp(torch.clamp(raw, -10.0, 10.0))
    raise ValueError(f'unknown rgb activation {activation}')
