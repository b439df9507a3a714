"""Host side of the fused wgmma NerfMLP (csrc/nerf_mlp_tc.cu): packs the nn.Linear weights of the reference-shaped NerfMLP
(/root/reference/xrnerf/models/mlps/nerf_mlp.py:29-49) into the kernel's weight image — fp16 slabs, K-major, in the exact order the kernel's
TMA producer streams them — and its bias vector, and runs the kernel on the fp16 encoding tile image of the rows. Also the NerfMLP's point queries
(mesh export): the one map from its embedder, and a Mip-NeRF footprint sigma, to the point-encoder, density-lattice and encoding-gradient kernels."""
import ctypes as C

import numpy as np
import torch

from . import _C


def fused_shape(mlp):
    """the NerfMLP shape the fused kernels implement: netdepth 8, netwidth 256, skips [4], use_viewdirs, input channels (63, 27) (BaseEmbedder,
    multires 10 / 4) or (96, 27) (MipNerfEmbedder, 16 point and 4 view bands)"""
    return (mlp.use_viewdirs and len(mlp.pts_linears) == 8 and list(mlp.skips) == [4] and mlp.pts_linears[0].out_features == 256
            and (mlp.input_ch, mlp.input_ch_dirs) in ((63, 27), (96, 27)))


# ---- point queries: BaseEmbedder when sigma is None, otherwise the Mip-NeRF point query at footprint sigma (include/xrnerf_b200.h, mesh export)
def encode_points(mlp, sigma, pts, dirs, samples_per_ray, enc):
    """the encoding tile image enc (u8, xrb_nerf_enc_image_bytes) of pts f32[n,3] with view directions dirs f32[n / samples_per_ray, 3]:
    xrb_nerf_posenc_tiles or xrb_mip_ipe_tiles_points"""
    e, n = mlp.embedder, int(pts.shape[0])
    if sigma is None:
        _C.check(_C.lib.xrb_nerf_posenc_tiles(_C.f32(pts), _C.f32(dirs), n, samples_per_ray, e.multires, e.multires_dirs, _C.ptr(enc), _C.stream()), 'nerf_posenc_tiles')
    else:
        _C.check(_C.lib.xrb_mip_ipe_tiles_points(_C.f32(pts), _C.f32(dirs), n, samples_per_ray, float(sigma), e.min_deg, e.max_deg, e.min_deg_view, e.max_deg_view,
                                                 _C.ptr(enc), _C.stream()), 'mip_ipe_tiles_points')


def density_lattice(mlp, sigma, image, bias, shape, box, out):
    """out f32[nz,ny,nx] <- the raw alpha on the lattice of shape (nz, ny, nx) over box: xrb_nerf_density_lattice or xrb_mip_density_lattice"""
    e = mlp.embedder
    nz, ny, nx = shape
    lo, hi = _C.float3(box[0]), _C.float3(box[1])
    if sigma is None:
        _C.check(_C.lib.xrb_nerf_density_lattice(_C.ptr(image), _C.f32(bias), mlp.input_ch, e.multires, nx, ny, nz, lo, hi, _C.f32(out), _C.stream()),
                 'nerf_density_lattice')
    else:
        _C.check(_C.lib.xrb_mip_density_lattice(_C.ptr(image), _C.f32(bias), e.min_deg, e.max_deg, float(sigma), nx, ny, nz, lo, hi, _C.f32(out), _C.stream()),
                 'mip_density_lattice')


def encoding_grad(mlp, sigma, pts, d_enc, n_terms, scale, grad):
    """grad f32[n,3] <- the gradient with respect to pts f32[n,3] through the point encoding, from the n_terms encoding-gradient terms in the tile image
    d_enc and the staging scale at device address `scale`: xrb_nerf_posenc_grad or xrb_mip_ipe_grad"""
    e, n, scale = mlp.embedder, int(pts.shape[0]), C.c_void_p(scale)
    if sigma is None:
        _C.check(_C.lib.xrb_nerf_posenc_grad(_C.f32(pts), n, e.multires, _C.ptr(d_enc), n_terms, scale, _C.f32(grad), _C.stream()), 'nerf_posenc_grad')
    else:
        _C.check(_C.lib.xrb_mip_ipe_grad(_C.f32(pts), n, float(sigma), e.min_deg, e.max_deg, _C.ptr(d_enc), n_terms, scale, _C.f32(grad), _C.stream()), 'mip_ipe_grad')


def _slab(w_rows_by_64):
    """[N,64] float32 -> swizzled bytes (N*128). element (n,k) -> (n>>3)*1024 + (n&7)*128 + (((k>>3) ^ (n&7))<<4) + (k&7)*2"""
    n = w_rows_by_64.shape[0]
    assert w_rows_by_64.shape[1] == 64 and n % 8 == 0
    h = w_rows_by_64.astype(np.float16)
    out = np.zeros((n // 8, 8, 8, 8), np.float16)          # [row group][row in group][chunk position][elem]
    rows = np.arange(n)
    for c in range(8):
        pos = c ^ (rows & 7)
        out[rows >> 3, rows & 7, pos, :] = h[:, c * 8:(c + 1) * 8]
    return out.reshape(-1).view(np.uint8)


def _pad_cols(w, k0, k1):
    """columns [k0,k1) of w, zero-padded to 64"""
    blk = np.zeros((w.shape[0], 64), np.float32)
    k1 = min(k1, w.shape[1])
    if k1 > k0:
        blk[:, :k1 - k0] = w[:, k0:k1]
    return blk


def _slab64(w_rows_by_32):
    """[N,32] float32 -> K-major SWIZZLE_64B bytes (N*64): element (n,k) -> (n>>3)*512 + (n&7)*64 + (((k>>3) ^ ((n>>1)&3))<<4) + (k&7)*2"""
    n = w_rows_by_32.shape[0]
    assert w_rows_by_32.shape[1] == 32 and n % 8 == 0
    h = w_rows_by_32.astype(np.float16)
    out = np.zeros((n // 8, 8, 4, 8), np.float16)          # [row group][row in group][chunk position][elem]
    rows = np.arange(n)
    for c in range(4):
        pos = c ^ ((rows >> 1) & 3)
        out[rows >> 3, rows & 7, pos, :] = h[:, c * 8:(c + 1) * 8]
    return out.reshape(-1).view(np.uint8)


def pack_nerf_mlp(mlp):
    """mlp: registry NerfMLP of the fused shape (fused_shape). Returns (image u8, bias f32) on the module's device.
    Image: 16 KB slabs in the kernel's stream order — per layer, per K-block (the point / direction block first where a layer reads it):
    the 256-wide layers as two K-halves [256 x 32] (SWIZZLE_64B), views_linears.0 / rgb_linear as one [N x 64] slab (SWIZZLE_128B). Bias vector: fp32 per-layer biases, Wa[256], ba, padded to 8 floats, then an fp16 copy of the per-layer biases."""
    assert fused_shape(mlp), 'fused NerfMLP kernel: netdepth=8, netwidth=256, skips=[4], use_viewdirs=True, input channels (63, 27) or (96, 27)'
    ic, icd = mlp.input_ch, mlp.input_ch_dirs
    aux = (ic + 63) // 64
    g = lambda lin: (lin.weight.detach().float().cpu().numpy(), lin.bias.detach().float().cpu().numpy())
    H = lambda W, j, off=0: _pad_cols(W, off + 64 * j, off + 64 * (j + 1))
    layers = []   # (column blocks in K order, N, n_halves, bias)
    W, b = g(mlp.pts_linears[0])
    layers.append(([_pad_cols(W, 64 * j, 64 * (j + 1)) for j in range(aux)], 256, 2, b))          # AUX (pts block 0) [, H3 = pts block 1]
    for l in range(1, 8):
        W, b = g(mlp.pts_linears[l])
        if l == 5:   # input = cat([pts(ic), h(256)])
            Wp = W[:, :ic]
            blocks = [_pad_cols(Wp, 0, 64)] + [H(W, j, ic) for j in range(4)] + ([_pad_cols(Wp, 64, 128)] if aux == 2 else [])
        else:
            blocks = [H(W, j) for j in range(4)]
        layers.append((blocks, 256, 2, b))
    W, b = g(mlp.feature_linear)
    layers.append(([H(W, j) for j in range(4)], 256, 2, b))
    W, b = g(mlp.views_linears[0])                                                                 # [128, 256 + icd] on cat([feature, dirs]); direction block first
    layers.append(([_pad_cols(W[:, 256:], 0, 64)] + [H(W, j) for j in range(4)], 128, 1, b))
    Wr, br = g(mlp.rgb_linear)
    W16 = np.zeros((16, 128), np.float32); W16[:3] = Wr
    layers.append(([H(W16, 0), H(W16, 1)], 16, 1, np.concatenate([br, np.zeros(13, np.float32)])))
    slabs, biases = [], []
    for blocks, N, nh, b in layers:
        hw = N // nh
        for blk in blocks:
            assert blk.shape == (N, 64)
            if nh == 2:     # N=256 layers: two K-halves [256 x 32] in the 64-byte-swizzle layout (one N=256 MMA pair each: A is read once)
                for kh in range(2):
                    slabs.append(_slab64(blk[:, 32 * kh:32 * (kh + 1)]))
            else:
                slabs.append(_slab(blk))
        biases.append(b.astype(np.float32))
    layer_bias = np.concatenate(biases)
    Wa, ba = g(mlp.alpha_linear)
    f32 = np.concatenate([layer_bias, Wa[0].astype(np.float32), ba.astype(np.float32)])
    f32 = np.concatenate([f32, np.zeros((-len(f32)) % 8, np.float32)])
    h16 = layer_bias.astype(np.float16)
    h16 = np.concatenate([h16, np.zeros((-len(h16)) % 8, np.float16)])
    dev = mlp.pts_linears[0].weight.device
    return torch.from_numpy(np.concatenate(slabs)).to(dev), torch.from_numpy(np.concatenate([f32, h16.view(np.float32)])).to(dev)


def pack_nerf_mlp_grad(mlp):
    """The gradient image of the density-gradient kernel (xrb_nerf_density_grad_rays): W^T of the trunk as B operands, in the order its producer
    streams them — pts_linears.7, .6, the point columns of .5, the hidden columns of .5, then .4 .. .1, the point columns of .0. A 256-wide step is
    four K-blocks of W^T (K = the layer's outputs), each as two K-halves [256 x 32] (SWIZZLE_64B, as pack_nerf_mlp's); a point step is [NP x 64]
    slabs (SWIZZLE_128B) of W[:, :input_ch]^T zero padded to NP = 64 (NeRF) or 128 (Mip-NeRF) rows."""
    assert fused_shape(mlp), 'fused NerfMLP kernel: netdepth=8, netwidth=256, skips=[4], use_viewdirs=True, input channels (63, 27) or (96, 27)'
    ic = mlp.input_ch
    n_pts = 64 if ic <= 64 else 128
    W = [lin.weight.detach().float().cpu().numpy() for lin in mlp.pts_linears]
    slabs = []

    def wide(wt):
        for j in range(4):
            blk = wt[:, 64 * j:64 * (j + 1)]
            slabs.extend(_slab64(np.ascontiguousarray(blk[:, 32 * kh:32 * (kh + 1)])) for kh in range(2))

    def points(wp):
        wt = np.zeros((n_pts, 256), np.float32)
        wt[:ic] = wp.T
        slabs.extend(_slab(np.ascontiguousarray(wt[:, 64 * j:64 * (j + 1)])) for j in range(4))
    wide(W[7].T); wide(W[6].T); points(W[5][:, :ic]); wide(W[5][:, ic:].T)
    for l in (4, 3, 2, 1):
        wide(W[l].T)
    points(W[0])
    return torch.from_numpy(np.concatenate(slabs)).to(mlp.pts_linears[0].weight.device)


def nerf_mlp_forward(image, bias, embedded, input_ch, input_ch_dirs):
    """fp32 embedded rows [n, input_ch + input_ch_dirs] -> raw [n, 4]: packs the fp16 encoding tile image (one streaming kernel), then runs the MLP kernel,
    which TMA-loads it. image/bias come from pack_nerf_mlp."""
    _C.require_cuda(image, bias, embedded)
    embedded = embedded.contiguous().float()
    n = embedded.shape[0]
    raw = torch.empty((n, 4), dtype=torch.float32, device=embedded.device)
    enc = torch.empty(_C.lib.xrb_nerf_enc_image_bytes(n, int(input_ch)), dtype=torch.uint8, device=embedded.device)
    _C.check(_C.lib.xrb_nerf_pack_embedded(_C.ptr(embedded), n, int(input_ch), int(input_ch_dirs), _C.ptr(enc), _C.stream()), 'nerf_pack_embedded')
    return nerf_mlp_forward_tiles(image, bias, enc, n, input_ch, input_ch_dirs, raw)


def nerf_mlp_forward_tiles(image, bias, enc_image, n_rows, input_ch, input_ch_dirs, raw=None):
    """The MLP kernel on an already packed encoding tile image (xrb_nerf_pack_embedded / xrb_nerf_posenc_tiles / xrb_mip_ipe_tiles_rays);
    image/bias come from pack_nerf_mlp."""
    if raw is None:
        raw = torch.empty((n_rows, 4), dtype=torch.float32, device=enc_image.device)
    _C.check(_C.lib.xrb_nerf_mlp_forward(_C.ptr(image), _C.ptr(bias), _C.ptr(enc_image), n_rows, int(input_ch), int(input_ch_dirs), _C.ptr(raw), _C.stream()), 'nerf_mlp_forward')
    return raw
