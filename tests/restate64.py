"""float64 restatements of this project's own kernels, shared by the tests that pin them (DESIGN §2). Each function names the kernel or the layout
it restates; two kernels that compute the same thing in different arithmetic get one restatement each. Nothing here asserts a bound: a test
derives its bound from the arithmetic restated here and keeps it beside its assertion.

  * fp16 / fp32 helpers: f16, ulp16, gamma and the unit roundoffs.
  * NGP: Grid (grid_cell / grid_index / the trilinear weights / the table-gradient scatter of csrc/ngp_field.cuh), ngp_mats (the fp16 weight
    matrices of a tcnn network), hashgrid_enc16 (xrb_tcnn_hashgrid_forward, the encodings every field kernel feeds its network), and the
    CUDA-core density gradient (xrb_ngp_density_grad): cuda_core_layer, cuda_core_density, enc_grad, position_grad, cuda_core_density_grad.
  * Tile images (csrc/tc.cuh, nerf_mlp._slab): encode / decode, and columns for a block range of an image.
  * NerfMLP: w16, trunk_grad (the training kernels' d(alpha)/d(encoding) down the 8-layer trunk), emulated_fp16_forward, mip_bands.
  * Marching cubes (xrb_mc_count / xrb_mc_emit): lattice_coords, mc_oracle, and the mesh checks check_closed_oriented, area, euler.
"""
import ctypes as C
import importlib.util
import os

import numpy as np
import torch

U16 = 2.0 ** -11            # fp16 unit roundoff
U32 = 2.0 ** -24            # fp32 unit roundoff
U64 = 2.0 ** -53            # float64 unit roundoff
GAMMA_TC = 2.0 ** -22       # per-term bound of a K-term fp32 accumulation of exact products on the tensor cores (gamma = K GAMMA_TC)
f32 = np.float32


def f16(a):
    """a rounded to fp16 once and back to float64, as an array, or as a tensor on a's device when a is one (numpy's float64 -> fp16 conversion is a
    single RNE rounding)"""
    if torch.is_tensor(a):
        return torch.from_numpy(f16(a.detach().cpu().numpy())).to(a.device)
    return np.asarray(a, np.float64).astype(np.float16).astype(np.float64)


def ulp16(v):
    """fp16 spacing at |v| (the subnormal step 2^-24 below 2^-14), as an array, or a tensor when v is one"""
    if torch.is_tensor(v):
        _, e = torch.frexp(torch.clamp(v.abs(), min=2.0 ** -14))
        return torch.ldexp(torch.ones_like(v), (e - 11).to(torch.int32))
    _, e = np.frexp(np.maximum(np.abs(v), 2.0 ** -14))
    return np.ldexp(1.0, e - 11)


def gamma(n, u):
    """n u / (1 - n u): the bound on n roundings of unit roundoff u"""
    return n * u / (1 - n * u)


# ================================================================================================================ NGP
P1, P2 = 2654435761, 805459861


class Grid:
    """tcnn's multiresolution grid as csrc/ngp_field.cuh computes it, layout from xrb_tcnn_hashgrid_layout, optionally with an fp16 table.

    grid_cell forms px = fma(scale, x, 0.5) in fp32 (fma: below). grid_index is tcnn's: a hashed level (res^3 > its table size, which is then
    2^log2_hashmap_size) takes (x ^ y P1 ^ z P2) & (size - 1) over uint32, a dense one x + y res + z res^2 with one conditional subtract of the
    size (that index is below twice the size).

    The fma is exact for every fp32 input. The product of two fp32 values has at most 48 significant bits and lies inside float64's exponent
    range, so t = scale x is exact in float64; TwoSum gives hi + lo = t + 0.5 exactly. Rounding that sum to odd at float64's 53 bits (hi where
    lo = 0, else whichever of hi and its neighbour towards lo has an odd last bit) and then to nearest fp32 equals rounding the exact sum to
    nearest fp32 once, because 53 >= 24 + 2 (Boldo and Melquiond, "Emulation of FMA and correctly rounded sums: proved algorithms using
    rounding to odd", IEEE TC 2008). So no input, however small, is rounded twice."""

    def __init__(self, cfg, table16=None):
        from xrnerf_b200 import _C
        off = (C.c_uint32 * 17)(); sc = (C.c_float * 16)(); res = (C.c_uint32 * 16)()
        _C.check(_C.lib.xrb_tcnn_hashgrid_layout(cfg, off, sc, res))
        self.off = np.array(off[:], np.int64)
        self.scale = np.array(sc[:], f32)
        self.res = np.array(res[:], np.int64)
        self.hashed = self.res ** 3 > np.diff(self.off)
        self.n_entries = int(self.off[-1])
        self.table = None if table16 is None else np.asarray(table16).astype(np.float64).reshape(-1, 2)

    @classmethod
    def of(cls, field):
        """the grid of an NgpField with its current fp16 table"""
        field.refresh()
        return cls(field.cfg, field._table16.cpu().numpy())

    def fma(self, l, x):
        """fp32 fma(scale_l, x, 0.5) of fp32 x, exactly (class docstring)"""
        t = np.float64(self.scale[l]) * np.asarray(x, f32).astype(np.float64)
        hi = t + 0.5
        b = hi - t
        lo = (t - (hi - b)) + (0.5 - b)
        even = (hi.view(np.int64) & 1) == 0
        return np.where((lo != 0) & even, np.nextafter(hi, np.where(lo > 0, np.inf, -np.inf)), hi).astype(f32)

    def cell(self, l, x):
        """x f32[n,3] -> (integer cell i64[n,3], in-cell position f32 as float64 [n,3]) as grid_cell computes them"""
        px = self.fma(l, x)
        fl = np.floor(px)
        return fl.astype(np.int64), (px - fl).astype(np.float64)

    def index(self, l, gi):
        """entry index within level l [n,8] of the 8 corners of cells gi i64[n,3] (corner c = bit0 x, bit1 y, bit2 z)"""
        hs, r = int(self.off[l + 1] - self.off[l]), int(self.res[l])
        out = np.empty((gi.shape[0], 8), np.int64)
        for c in range(8):
            x, y, z = (gi[:, a] + ((c >> a) & 1) for a in range(3))
            if self.hashed[l]:
                out[:, c] = (x ^ ((y * P1) & 0xffffffff) ^ ((z * P2) & 0xffffffff)) & (hs - 1)
            else:
                idx = x + y * r + z * r * r
                out[:, c] = np.where(idx >= hs, idx - hs, idx)
        return out

    @staticmethod
    def trilinear(f):
        """(d w_c / d f [n,8,3], the weights w_c [n,8]) of in-cell positions f [n,3] (float64 of the fp32 positions)"""
        u = 1.0 - f
        dw, w = np.zeros(f.shape[:1] + (8, 3)), np.zeros(f.shape[:1] + (8,))
        for c in range(8):
            pick = [f[:, a] if (c >> a) & 1 else u[:, a] for a in range(3)]
            w[:, c] = pick[0] * pick[1] * pick[2]
            for a in range(3):
                o = [pick[b] for b in range(3) if b != a]
                dw[:, c, a] = (1.0 if (c >> a) & 1 else -1.0) * o[0] * o[1]
        return dw, w

    def corners(self, l, x):
        """(entry index [n,8] into the whole table, trilinear weight [n,8] float64) of level l at x f32[n,3]"""
        gi, f = self.cell(l, x)
        return self.off[l] + self.index(l, gi), self.trilinear(f)[1]

    def corner_values(self, l, gi):
        """fp16 feature pairs of the table at the 8 corners [n,8,2] of cells gi"""
        return self.table[self.off[l] + self.index(l, gi)]

    def scatter(self, x, genc, rows):
        """(table gradient of dL/denc [n,32], contribution count per scalar); only `rows` contribute"""
        acc = np.zeros(2 * self.n_entries); cnt = np.zeros(2 * self.n_entries)
        p, g = x[rows], genc[rows]
        for l in range(16):
            idx, w = self.corners(l, p)
            for f in range(2):
                k = (2 * idx + f).ravel()
                acc += np.bincount(k, (w * g[:, 2 * l + f:2 * l + f + 1]).ravel(), minlength=acc.size)
                cnt += np.bincount(k, minlength=acc.size)
        return acc, cnt


def ngp_mats(params, n_hidden):
    """the fp16 weight matrices W[out][in] (float64) of a tcnn network with 32 inputs, n_hidden 64-wide layers and 16 outputs from its flat
    parameters (rounded to fp16 here; already-fp16 values pass unchanged)"""
    w = f16(params)
    out, o = [], 0
    for (r, c) in [(64, 32)] + [(64, 64)] * (n_hidden - 1) + [(16, 64)]:
        out.append(w[o:o + r * c].reshape(r, c))
        o += r * c
    assert o == w.size
    return out


def hashgrid_enc16(field, pts):
    """the fp16 encodings xrb_tcnn_hashgrid_forward computes from the field's table at pts (f32 array [n,3], or rows of a CUDA tensor), as float64"""
    from xrnerf_b200 import _C
    pts = pts if torch.is_tensor(pts) else torch.from_numpy(np.ascontiguousarray(pts, f32)).cuda()
    n = pts.shape[0]
    enc = torch.empty((n, 32), dtype=torch.float16, device='cuda')
    pp, ps = _C.rows(pts)
    _C.check(_C.lib.xrb_tcnn_hashgrid_forward(field.cfg, field.tab, pp, ps, n, _C.ptr(enc), _C.stream()), 'hashgrid_forward')
    return enc.cpu().numpy().astype(np.float64)


# ---------------------------------------------------------------------------------------------------------------- CUDA-core density gradient
# The CUDA-core density runs each unit as one sequential fp32 fma chain, restated exactly here; the tensor-core kernels sum in an order the
# hardware picks, so their tests bound an interval around the float64 sum instead (test_gpu_field_grad_exact, test_gpu_ngp_normals).
def cuda_core_layer(W, x):
    """the CUDA-core layer's pre-activations: per unit a sequential fp32 fma chain over the inputs, each step rounded once (each fp16 x fp16
    product is exact, and the sum is formed in extended precision before its one rounding)"""
    s = np.zeros((x.shape[0], W.shape[0]), f32)
    for k in range(W.shape[1]):
        s = (np.longdouble(1) * W[:, k][None, :] * x[:, k][:, None] + s.astype(np.longdouble)).astype(f32)
    return s.astype(np.float64)


def cuda_core_density(mats, enc16):
    """density and hidden-layer masks as the CUDA-core density computes them (enc16: the fp16 encodings as float64)"""
    a, masks = enc16, []
    for W in mats[:-1]:
        a = f16(np.maximum(cuda_core_layer(W, a), 0))
        masks.append(a > 0)
    return f16(cuda_core_layer(mats[-1][:1], a)[:, 0]), masks


def enc_grad(mats, masks):
    """d(out 0)/d(encoding) [n,32] in float64 and the same chain on absolute values"""
    g = masks[-1] * mats[-1][0][None, :]
    ga = np.abs(g)
    for k in range(len(mats) - 2, 0, -1):
        g, ga = masks[k - 1] * (g @ mats[k]), masks[k - 1] * (ga @ np.abs(mats[k]))
    return g @ mats[0], ga @ np.abs(mats[0])


def position_grad(grid, x, ge, gea):
    """position_grad_level summed over the levels: scale_l sum_c dw_c/df (v_c . ge_l) [n,3], and the same sum on absolute values"""
    g, m = np.zeros((x.shape[0], 3)), np.zeros((x.shape[0], 3))
    for l in range(16):
        gi, f = grid.cell(l, x)
        v = grid.corner_values(l, gi)
        dw, _ = grid.trilinear(f)
        s = v[:, :, 0] * ge[:, None, 2 * l] + v[:, :, 1] * ge[:, None, 2 * l + 1]
        sa = np.abs(v[:, :, 0]) * gea[:, None, 2 * l] + np.abs(v[:, :, 1]) * gea[:, None, 2 * l + 1]
        g += float(grid.scale[l]) * (dw * s[:, :, None]).sum(1)
        m += float(grid.scale[l]) * (np.abs(dw) * sa[:, :, None]).sum(1)
    return g, m


def field_mats(field):
    """ngp_mats of the field's fp16 density weights"""
    field.refresh()
    return ngp_mats(field._dens16.cpu().numpy(), field.cfg.density_hidden)


def cuda_core_density_grad(field, grid, x):
    """xrb_ngp_density_grad at x f32[n,3]: (density as the kernel computes it, float64 gradient, its bound). The gradient is a sum of products
    with at most 64 dh + 2 + 1 + 8 + 16 fp32 roundings along any one: gamma_n(2^-24) times the absolute chain, plus the restatement's own."""
    mats = field_mats(field)
    dens, masks = cuda_core_density(mats, hashgrid_enc16(field, x))
    ge, gea = enc_grad(mats, masks)
    g, m = position_grad(grid, x, ge, gea)
    n = 64 * field.cfg.density_hidden + 2 + 1 + 8 + 16
    return dens, g, (gamma(n, U32) + gamma(n, U64)) * m


# ================================================================================================================ tile images
BLOCK = 16384               # bytes of one [128 x 64] fp16 block


def swz(rows):
    """fp16 index of element (r, k) of a [rows x 64] block or slab: byte (r >> 3) 1024 + (r & 7) 128 + (((k >> 3) ^ (r & 7)) << 4) + (k & 7) 2"""
    r, k = np.meshgrid(np.arange(rows), np.arange(64), indexing='ij')
    return (((r >> 3) * 1024 + (r & 7) * 128 + (((k >> 3) ^ (r & 7)) << 4) + (k & 7) * 2) // 2).reshape(-1)


def decode(img, n_tiles, rows=128):
    """an Img (or a raw slab arena with rows = n_pad) -> fp16 [n_tiles * rows, n_blk * 64] (torch, on the image's device)"""
    buf, stride, off, nb = img.buf, img.tile_stride // 2, img.blk_off // 2, img.n_blk
    h = buf.view(torch.float16)[:n_tiles * stride].reshape(n_tiles, stride)[:, off:off + nb * rows * 64].reshape(n_tiles, nb, rows * 64)
    idx = torch.as_tensor(swz(rows), device=buf.device)
    return h[:, :, idx].reshape(n_tiles, nb, rows, 64).permute(0, 2, 1, 3).reshape(n_tiles * rows, nb * 64)


def encode(m16):
    """fp16 [n_tiles * 128, n_blk * 64] -> tile image bytes (the inverse of decode)"""
    R, Cc = m16.shape
    nt, nb = R // 128, Cc // 64
    blocks = m16.reshape(nt, 128, nb, 64).permute(0, 2, 1, 3).reshape(nt, nb, 8192)
    out = torch.empty_like(blocks)
    out[:, :, torch.as_tensor(swz(128), device=m16.device)] = blocks
    return out.reshape(-1).view(torch.uint8)


def image(m16):
    """the Img of an fp16 matrix"""
    from xrnerf_b200.nerf_train import Img
    nb = m16.shape[1] // 64
    return Img(encode(m16), nb * BLOCK, 0, nb)


def columns(buf, n, n_blk, blk0, cols):
    """float64 [n, cols]: rows 0..n-1 of the `cols` columns starting at block blk0 of the tile image in buf (n_blk blocks per tile)"""
    from xrnerf_b200.nerf_train import Img
    return decode(Img(buf, n_blk * BLOCK, blk0 * BLOCK, (cols + 63) // 64), (n + 127) // 128)[:n, :cols].double()


# ================================================================================================================ NerfMLP
def w16(lin):
    """the fp16 weights the kernels' slabs hold, as float64 on the layer's device"""
    return f16(lin.weight)


def trunk_grad(mlp, H, input_ch):
    """d(raw alpha)/d(encoding) [n, input_ch] through the 8-layer trunk (skip at 5) over the fp16 weights, with the ReLU masks of the hidden
    activations H (fp16 activation > 0, as the training kernels stage them); also the same chain on absolute values"""
    n = H[0].shape[0]
    g, ga = w16(mlp.alpha_linear)[0].expand(n, 256), w16(mlp.alpha_linear)[0].abs().expand(n, 256)
    e = torch.zeros((n, input_ch), dtype=torch.float64, device=g.device)
    ea = torch.zeros_like(e)
    for l in range(7, -1, -1):
        m = (H[l] > 0).double()
        g, ga = g * m, ga * m                                 # dZ of layer l
        W = w16(mlp.pts_linears[l])
        if l == 0:
            e, ea = e + g @ W, ea + ga @ W.abs()
        elif l == 5:
            e, ea = e + g @ W[:, :input_ch], ea + ga @ W[:, :input_ch].abs()
            g, ga = g @ W[:, input_ch:], ga @ W[:, input_ch:].abs()
        else:
            g, ga = g @ W, ga @ W.abs()
    return e, ea


def _ste_half(t):
    """value rounded to fp16, gradient passed straight through: what storing an activation as fp16 does"""
    return t + (t.half().float() - t).detach()


def emulated_fp16_forward(mlp, x):
    """the reference's run_mlp (nerf_mlp.py:70-94) with the tensor-core path's operand precision: fp16 weights and fp16 layer inputs, fp32
    accumulation and bias, so that a comparison isolates the kernels (same ReLU pattern) from the precision choice"""
    import torch.nn.functional as F
    lin = lambda l, h: F.linear(h, _ste_half(l.weight), l.bias)
    pts, views = torch.split(_ste_half(x), [mlp.input_ch, mlp.input_ch_dirs], dim=-1)
    h = pts
    for i, l in enumerate(mlp.pts_linears):
        h = _ste_half(F.relu(lin(l, h)))
        if i in mlp.skips:
            h = torch.cat([pts, h], -1)
    alpha = lin(mlp.alpha_linear, h)
    h = torch.cat([_ste_half(lin(mlp.feature_linear, h)), views], -1)
    h = _ste_half(F.relu(lin(mlp.views_linears[0], h)))
    return torch.cat([lin(mlp.rgb_linear, h), alpha], -1)


def mip_bands(sigma, min_deg=0, max_deg=16):
    """the per-band factors a_k of a Mip-NeRF point-query launch as the library forms them: hv = 0.5 ((sigma^2 2^deg) 2^deg) in fp32,
    a_k = fp32(exp(-hv)), and the band is live iff hv <= 20 -> float64 [n_deg] (0 for a dead band)"""
    s = f32(sigma)
    cov = s * s
    out = np.zeros(max_deg - min_deg)
    for k in range(max_deg - min_deg):
        sc = f32(2.0 ** (min_deg + k))
        hv = f32(0.5) * (cov * sc * sc)
        if not hv <= 20:
            break
        out[k] = float(f32(np.exp(-np.float64(hv))))
    return out


# ================================================================================================================ marching cubes
def _gen():
    root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    spec = importlib.util.spec_from_file_location('gen_mc_table', os.path.join(root, 'scripts', 'gen_mc_table.py'))
    m = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(m)
    return m


GEN = _gen()
COUNTS, TRIS = GEN.build_table()


def lattice_coords(lo, hi, n):
    """float32 coordinates of lattice indices 0..n-1 on one axis: min(lo + i * ((hi - lo) / (n - 1)), hi), each operation rounded once"""
    lo, hi = f32(lo), f32(hi)
    step = f32(hi - lo) / f32(n - 1)
    return np.minimum(lo + np.arange(n, dtype=f32) * f32(step), hi).astype(f32)


def lattice_points(shape, box):
    """the lattice's points, x fastest, f32 [nz ny nx, 3] on the GPU"""
    nz, ny, nx = shape
    cx, cy, cz = (lattice_coords(box[0][a], box[1][a], n) for a, n in enumerate((nx, ny, nz)))
    Z, Y, X = np.meshgrid(cz, cy, cx, indexing='ij')
    return torch.from_numpy(np.stack([X, Y, Z], -1).reshape(-1, 3).copy()).cuda()


def mc_oracle(vol, threshold, box=((0, 0, 0), (1, 1, 1))):
    """(verts f32[V,3], faces i32[F,3]) of vol f32[nz,ny,nx] (x fastest), by the contract of xrb_mc_emit"""
    vol = np.ascontiguousarray(vol, f32)
    thr = f32(threshold)
    nz, ny, nx = vol.shape
    cx, cy, cz = (lattice_coords(box[0][a], box[1][a], n) for a, n in enumerate((nx, ny, nz)))
    inside = vol > thr
    cross = np.zeros((nz, ny, nx, 3), bool)                   # the edge from each point in +x, +y, +z crosses
    cross[:, :, :-1, 0] = inside[:, :, :-1] != inside[:, :, 1:]
    cross[:, :-1, :, 1] = inside[:, :-1, :] != inside[:, 1:, :]
    cross[:-1, :, :, 2] = inside[:-1, :, :] != inside[1:, :, :]
    vid = np.cumsum(cross.reshape(-1)).reshape(cross.shape).astype(np.int64) - 1
    pz, py, px, ax = np.nonzero(cross)                         # lattice-point order, then axis: the vertex order
    step = np.stack([ax == 0, ax == 1, ax == 2], 1).astype(np.int64)
    qx, qy, qz = px + step[:, 0], py + step[:, 1], pz + step[:, 2]
    vp, vq = vol[pz, py, px], vol[qz, qy, qx]
    p_in = vp > thr
    v_in, v_out = np.where(p_in, vp, vq), np.where(p_in, vq, vp)
    t = (f32(thr) - v_out).astype(f32) / (v_in - v_out).astype(f32)
    verts = np.stack([cx[px], cy[py], cz[pz]], 1).astype(f32)
    for a, (c, ip, iq) in enumerate(((cx, px, qx), (cy, py, qy), (cz, pz, qz))):
        sel = ax == a
        P, Q = c[ip[sel]], c[iq[sel]]
        pin = p_in[sel]
        Pin, Pout = np.where(pin, P, Q), np.where(pin, Q, P)
        verts[sel, a] = Pout + (t[sel] * (Pin - Pout).astype(f32)).astype(f32)
    # cells
    case = np.zeros((nz - 1, ny - 1, nx - 1), np.int64)
    for c in range(8):
        ox, oy, oz = c & 1, (c >> 1) & 1, (c >> 2) & 1
        case |= inside[oz:nz - 1 + oz, oy:ny - 1 + oy, ox:nx - 1 + ox].astype(np.int64) << c
    case = case.reshape(-1)
    n_t = COUNTS[case].astype(np.int64)
    cell = np.repeat(np.arange(case.size), n_t)
    slot = np.arange(cell.size) - np.repeat(np.cumsum(n_t) - n_t, n_t)
    edges = TRIS[case[cell], slot].astype(np.int64)                         # [F,3]
    gz, gy, gx = np.unravel_index(cell, (nz - 1, ny - 1, nx - 1))
    start = np.array([GEN.edge_corners(e)[0] for e in range(12)])
    eo = np.stack([start & 1, (start >> 1) & 1, (start >> 2) & 1], 1)    # owner offset of each edge
    ea = np.arange(12) // 4
    faces = vid[gz[:, None] + eo[edges, 2], gy[:, None] + eo[edges, 1], gx[:, None] + eo[edges, 0], ea[edges]]
    return verts, faces.astype(np.int32).reshape(-1, 3)


def check_closed_oriented(verts, faces):
    """every undirected edge in exactly two triangles, every directed edge once, every vertex used, signed volume > 0; returns the volume"""
    faces = np.asarray(faces, np.int64)
    assert faces.shape[0] > 0
    d = np.concatenate([faces[:, [0, 1]], faces[:, [1, 2]], faces[:, [2, 0]]])
    key = d[:, 0] * (1 << 32) + d[:, 1]
    assert np.unique(key).size == key.size, 'a directed edge appears twice'
    und = np.minimum(d[:, 0], d[:, 1]) * (1 << 32) + np.maximum(d[:, 0], d[:, 1])
    _, cnt = np.unique(und, return_counts=True)
    assert (cnt == 2).all(), 'an edge does not lie in exactly two triangles'
    assert np.unique(faces).size == len(verts), 'an unused vertex'
    vol = signed_volume(verts, faces)
    assert vol > 0
    return vol


def signed_volume(verts, faces):
    v = np.asarray(verts, np.float64)[np.asarray(faces, np.int64)]
    return float(np.einsum('ij,ij->i', v[:, 0], np.cross(v[:, 1], v[:, 2])).sum() / 6)


def area(verts, faces):
    v = np.asarray(verts, np.float64)[np.asarray(faces, np.int64)]
    return float(np.linalg.norm(np.cross(v[:, 1] - v[:, 0], v[:, 2] - v[:, 0]), axis=1).sum() / 2)


def euler(verts, faces):
    faces = np.asarray(faces, np.int64)
    d = np.concatenate([faces[:, [0, 1]], faces[:, [1, 2]], faces[:, [2, 0]]])
    n_edges = np.unique(np.minimum(d[:, 0], d[:, 1]) * (1 << 32) + np.maximum(d[:, 0], d[:, 1])).size
    return len(verts) - n_edges + len(faces)
