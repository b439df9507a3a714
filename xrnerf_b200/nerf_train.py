"""NerfMLP training on tensor cores: host side of csrc/nerf_train.cu.

The reference trains NerfMLP (/root/reference/xrnerf/models/mlps/nerf_mlp.py:70-94) through torch.autograd over its nn.Linear modules (cuBLAS fp32 GEMMs, every
activation through HBM in fp32; networks/nerf.py:71-92, networks/mipnerf.py:45-74). Here `NerfMlpTrainFn` is ONE autograd node for run_mlp: its forward runs the 12 dense
layers as wgmma kernels over fp16 tile images (xrb_nerf_tg_layer) and keeps every layer input as the backward's operand; its backward runs, per layer, the input gradient
(the same weight slabs read MN-major, ReLU mask fused) and the weight / bias gradients (xrb_nerf_tg_dw: accumulators in registers across all rows). Parameters stay the
nn.Linear modules of the registry class (state_dict compatibility); their fp32 weights are re-packed into fp16 slabs at every forward (the optimiser changed them).

Numeric contract: fp16 operands, fp32 accumulation, fp16 activations and activation gradients, fp32 parameter gradients. The activation gradients are
loss-scaled by a power of two chosen on the device per backward (max |dL/draw| s in [2^12, 2^13)), so that the NeRF loss's 1e-8 .. 1e-5 gradients stay in fp16's
normal range down the trunk. tests/test_gpu_nerf_train_exact.py checks every launch and the whole chain entry by entry against float64 from the kernels' own
operands, and a Blender-sized train step to 1e-2 relative L2 per tensor; tests/test_gpu_nerf_train.py compares with the fp32 autograd path (raw 2e-2 of max,
gradients 6e-2 relative L2 per tensor).
"""
import ctypes as C

import torch

from . import _C
from . import nerf_mlp as nm

BLOCK = 16384


class TgLayer(C.Structure):
    _fields_ = [('a_base', C.c_void_p * 2), ('a_tile_stride', C.c_uint32 * 2), ('a_blk_off', C.c_uint32 * 2), ('a_n_blk', C.c_int * 2), ('n_a', C.c_int),
                ('w', C.c_void_p),
                ('slab_w_off', C.c_uint32 * 10), ('slab_bytes', C.c_uint32 * 10), ('slab_n_sub', C.c_int * 10), ('slab_a_blk0', C.c_int * 10), ('slab_d_col', C.c_int * 10),
                ('slab_first', C.c_int * 10), ('slab_n_k', C.c_int * 10), ('n_slabs', C.c_int),
                ('b_mn', C.c_int), ('mma_n', C.c_int), ('out_cols', C.c_int), ('epi', C.c_int), ('relu', C.c_int), ('bias', C.c_void_p),
                ('x_base', C.c_void_p), ('x_tile_stride', C.c_uint32), ('x_blk_off', C.c_uint32),
                ('y', C.c_void_p), ('y_tile_stride', C.c_uint32), ('y_blk_off', C.c_uint32),
                ('yf', C.c_void_p), ('yf_stride', C.c_int), ('yf_col', C.c_int), ('yf_n', C.c_int), ('yf_scale', C.c_float),
                ('n_rows', C.c_int64)]


class TgDw(C.Structure):
    _fields_ = [('z_base', C.c_void_p), ('z_tile_stride', C.c_uint32), ('z_blk_off', C.c_uint32),
                ('x_base', C.c_void_p), ('x_tile_stride', C.c_uint32), ('x_blk_off', C.c_uint32), ('x_n_blk', C.c_int),
                ('N', C.c_int), ('K', C.c_int), ('k_off', C.c_int), ('k_cols', C.c_int),
                ('dW', C.c_void_p), ('db', C.c_void_p), ('n_rows', C.c_int64), ('scale', C.c_void_p)]


_C.lib.xrb_nerf_tg_layer.restype = C.c_int
_C.lib.xrb_nerf_tg_layer.argtypes = [C.POINTER(TgLayer), C.c_void_p]
_C.lib.xrb_nerf_tg_dw.restype = C.c_int
_C.lib.xrb_nerf_tg_dw.argtypes = [C.POINTER(TgDw), C.c_void_p]


class Img:
    """a tile image (or a block range of one): device buffer + tile stride + first block + block count"""

    def __init__(self, buf, tile_stride, blk_off, n_blk):
        self.buf, self.tile_stride, self.blk_off, self.n_blk = buf, int(tile_stride), int(blk_off), int(n_blk)

    @staticmethod
    def new(n_tiles, n_blk, dev, zero=False):
        f = torch.zeros if zero else torch.empty
        return Img(f(n_tiles * n_blk * BLOCK, dtype=torch.uint8, device=dev), n_blk * BLOCK, 0, n_blk)

    def sub(self, first, n):
        return Img(self.buf, self.tile_stride, self.blk_off + first * BLOCK, n)

    @property
    def ptr(self):
        return self.buf.data_ptr()


class _Slabs:
    """fp16 weight slabs of all layers in one arena; layer -> (offset, n_pad, [ (col0, valid) per input block ])"""

    def __init__(self, mlp, P):
        self.P = P
        W = mlp.pts_linears[0].out_features
        ic, icd = mlp.input_ch, mlp.input_ch_dirs
        pts_blocks = [(64 * k, min(64, ic - 64 * k)) for k in range(P)]
        hid = lambda off: [(off + 64 * k, 64) for k in range(W // 64)]
        self.layers = {}
        specs = [('pts0', mlp.pts_linears[0], pts_blocks)]
        for l in range(1, len(mlp.pts_linears)):
            blocks = (pts_blocks + hid(ic)) if (l - 1) in mlp.skips else hid(0)
            specs.append((f'pts{l}', mlp.pts_linears[l], blocks))
        specs += [('alpha', mlp.alpha_linear, hid(0)), ('feature', mlp.feature_linear, hid(0)),
                  ('views', mlp.views_linears[0], hid(0) + [(W, icd)]), ('rgb', mlp.rgb_linear, [(0, 64), (64, 64)])]
        off = 0
        for name, lin, blocks in specs:
            n_pad = (lin.out_features + 15) // 16 * 16
            self.layers[name] = dict(lin=lin, off=off, n_pad=n_pad, blocks=blocks, slab_bytes=n_pad * 128)
            off += len(blocks) * n_pad * 128
        self.arena = torch.empty(off, dtype=torch.uint8, device=lin.weight.device)

    def pack(self):
        for L in self.layers.values():
            lin, nb = L['lin'], len(L['blocks'])
            col0 = (C.c_int * nb)(*[b[0] for b in L['blocks']]); valid = (C.c_int * nb)(*[b[1] for b in L['blocks']])
            _C.check(_C.lib.xrb_nerf_tg_pack_weights(_C.f32(lin.weight.detach()), lin.out_features, lin.in_features, L['n_pad'], nb, col0, valid,
                                                     C.c_void_p(self.arena.data_ptr() + L['off']), _C.stream()), 'tg_pack_weights')


def _layer(n_rows, a_srcs, w_arena, slabs, b_mn, mma_n, out_cols, epi, relu=0, bias=None, x=None, y=None, yf=None, yf_col=0, yf_n=0):
    L = TgLayer()
    for s, a in enumerate(a_srcs):
        L.a_base[s], L.a_tile_stride[s], L.a_blk_off[s], L.a_n_blk[s] = a.ptr, a.tile_stride, a.blk_off, a.n_blk
    L.n_a = len(a_srcs)
    L.w = w_arena.data_ptr()
    for s, (w_off, nbytes, n_sub, a_blk0, d_col, first, n_k) in enumerate(slabs):
        L.slab_w_off[s], L.slab_bytes[s], L.slab_n_sub[s], L.slab_a_blk0[s], L.slab_d_col[s], L.slab_first[s], L.slab_n_k[s] = w_off, nbytes, n_sub, a_blk0, d_col, first, n_k
    L.n_slabs = len(slabs)
    L.b_mn, L.mma_n, L.out_cols, L.epi, L.relu = b_mn, mma_n, out_cols, epi, relu
    L.bias = bias.data_ptr() if bias is not None else None
    if x is not None:
        L.x_base, L.x_tile_stride, L.x_blk_off = x.ptr, x.tile_stride, x.blk_off
    if y is not None:
        L.y, L.y_tile_stride, L.y_blk_off = y.ptr, y.tile_stride, y.blk_off
    if yf is not None:
        L.yf, L.yf_stride, L.yf_col, L.yf_n, L.yf_scale = yf.data_ptr(), yf.shape[1], yf_col, yf_n, 1.0
    L.n_rows = n_rows
    _C.check(_C.lib.xrb_nerf_tg_layer(C.byref(L), _C.stream()), 'nerf_tg_layer')


def _fwd(n_rows, S, name, a_srcs, out_img=None, relu=1, yf=None, yf_col=0, yf_n=0):
    L = S.layers[name]
    lin = L['lin']
    slabs = [(L['off'] + kb * L['slab_bytes'], L['slab_bytes'], 1, kb, 0, 1 if kb == 0 else 0, 4) for kb in range(len(L['blocks']))]
    if yf is None:
        _layer(n_rows, a_srcs, S.arena, slabs, 0, L['n_pad'], L['n_pad'], 0, relu=relu, bias=lin.bias.detach(), y=out_img)
    else:
        _layer(n_rows, a_srcs, S.arena, slabs, 0, 16, 16, 1, bias=lin.bias.detach(), yf=yf, yf_col=yf_col, yf_n=yf_n)


def _dx(n_rows, S, pairs, obs, out_img, mask=None):
    """pairs: [(layer name, dZ image)] accumulated; obs: input blocks (kb indices of the layer's slab list) whose gradient is wanted -> out_img (len(obs) blocks)"""
    a_srcs, slabs, a0 = [], [], 0
    for name, z in pairs:
        a_srcs.append(z)
    for j, ob in enumerate(obs):
        a0 = 0
        for p, (name, z) in enumerate(pairs):
            L = S.layers[name]
            n_out = L['lin'].out_features
            n_sub = max(1, n_out // 64) if n_out >= 64 else 1
            n_k = 4 if n_out >= 64 else 1
            slabs.append((L['off'] + ob * L['slab_bytes'], L['slab_bytes'], n_sub, a0, j * 64, 1 if p == 0 else 0, n_k))
            a0 += z.n_blk
    _layer(n_rows, a_srcs, S.arena, slabs, 1, 64, len(obs) * 64, 2 if mask is not None else 3, x=mask, y=out_img)


def _dw(n_rows, z, x, lin, gW, gb, k_off, k_cols, with_bias, scale=None):
    D = TgDw()
    D.z_base, D.z_tile_stride, D.z_blk_off = z.ptr, z.tile_stride, z.blk_off
    D.x_base, D.x_tile_stride, D.x_blk_off, D.x_n_blk = x.ptr, x.tile_stride, x.blk_off, x.n_blk
    D.N, D.K, D.k_off, D.k_cols = lin.out_features, lin.in_features, k_off, k_cols
    D.dW, D.db = gW.data_ptr(), (gb.data_ptr() if with_bias else None)
    D.n_rows = n_rows
    D.scale = scale.data_ptr() + 4 if scale is not None else None
    _C.check(_C.lib.xrb_nerf_tg_dw(C.byref(D), _C.stream()), 'nerf_tg_dw')


def supported(mlp):
    return nm.fused_shape(mlp)


def param_list(mlp):
    lins = list(mlp.pts_linears) + [mlp.alpha_linear, mlp.feature_linear, mlp.views_linears[0], mlp.rgb_linear]
    return lins, [t for l in lins for t in (l.weight, l.bias)]


class NerfMlpTrainFn(torch.autograd.Function):
    """run_mlp(embedded [rows, input_ch + input_ch_dirs] fp32) -> raw [rows, 4] fp32, differentiable w.r.t. every nn.Linear weight and bias of `mlp`."""

    @staticmethod
    def forward(ctx, mlp, embedded, *params):
        dev = embedded.device
        n = int(embedded.shape[0])
        nt = (n + 127) // 128
        P = (mlp.input_ch + 63) // 64
        S = getattr(mlp, '_tg_slabs', None)
        if S is None or S.arena.device != dev:
            S = mlp._tg_slabs = _Slabs(mlp, P)
        S.pack()
        enc = Img(torch.empty(_C.lib.xrb_nerf_enc_image_bytes(n, int(mlp.input_ch)), dtype=torch.uint8, device=dev), (P + 1) * BLOCK, 0, P + 1)
        emb = embedded.detach().contiguous().float()
        _C.check(_C.lib.xrb_nerf_pack_embedded(_C.ptr(emb), n, int(mlp.input_ch), int(mlp.input_ch_dirs), _C.ptr(enc.buf), _C.stream()), 'nerf_pack_embedded')
        pts, dirs = enc.sub(0, P), enc.sub(P, 1)
        H = [Img.new(nt, 4, dev) for _ in range(8)]
        F, V = Img.new(nt, 4, dev), Img.new(nt, 2, dev)
        raw = torch.empty((n, 4), dtype=torch.float32, device=dev)
        _fwd(n, S, 'pts0', [pts], H[0])
        for l in range(1, 8):
            _fwd(n, S, f'pts{l}', ([pts, H[l - 1]] if (l - 1) in mlp.skips else [H[l - 1]]), H[l])
        _fwd(n, S, 'alpha', [H[7]], yf=raw, yf_col=3, yf_n=1)
        _fwd(n, S, 'feature', [H[7]], F, relu=0)
        _fwd(n, S, 'views', [F, dirs], V)
        _fwd(n, S, 'rgb', [V], yf=raw, yf_col=0, yf_n=3)
        ctx.mlp, ctx.saved, ctx.n = mlp, (S, enc, pts, dirs, H, F, V), n
        return raw

    @staticmethod
    def backward(ctx, d_raw):
        mlp, (S, enc, pts, dirs, H, F, V), n = ctx.mlp, ctx.saved, ctx.n
        dev = d_raw.device
        nt = (n + 127) // 128
        P = S.P
        lins, params = param_list(mlp)
        g = {id(t): torch.zeros_like(t, dtype=torch.float32) for t in params}
        gw = lambda lin: (g[id(lin.weight)], g[id(lin.bias)])
        d_raw = d_raw.contiguous().float()
        z_rgb, z_alpha = Img.new(nt, 1, dev, zero=True), Img.new(nt, 1, dev, zero=True)
        sc = torch.empty(2, dtype=torch.float32, device=dev)        # [workspace, s]: the dZ staging scale, chosen on the device from max |dL/draw|
        _C.check(_C.lib.xrb_nerf_tg_pack_draw(_C.ptr(d_raw), n, _C.ptr(z_rgb.buf), _C.ptr(z_alpha.buf), _C.ptr(sc), _C.stream()), 'tg_pack_draw')
        ic, icd, W = mlp.input_ch, mlp.input_ch_dirs, 256
        # rgb_linear
        ZV = Img.new(nt, 2, dev)
        _dx(n, S, [('rgb', z_rgb)], [0, 1], ZV, mask=V)
        _dw(n, z_rgb, V, mlp.rgb_linear, *gw(mlp.rgb_linear), 0, 128, True, sc)
        # views_linears.0 on cat([feature, dirs]): only the feature part of the input gradient is needed
        ZF = Img.new(nt, 4, dev)
        _dx(n, S, [('views', ZV)], [0, 1, 2, 3], ZF, mask=None)
        _dw(n, ZV, F, mlp.views_linears[0], *gw(mlp.views_linears[0]), 0, W, True, sc)
        _dw(n, ZV, dirs, mlp.views_linears[0], *gw(mlp.views_linears[0]), W, icd, False, sc)
        # feature_linear (no activation) + alpha_linear both read h7
        Za, Zb = Img.new(nt, 4, dev), Img.new(nt, 4, dev)
        _dx(n, S, [('feature', ZF), ('alpha', z_alpha)], [0, 1, 2, 3], Za, mask=H[7])
        _dw(n, ZF, H[7], mlp.feature_linear, *gw(mlp.feature_linear), 0, W, True, sc)
        _dw(n, z_alpha, H[7], mlp.alpha_linear, *gw(mlp.alpha_linear), 0, W, True, sc)
        # trunk, top down: Za holds dZ of layer l (gradient w.r.t. its pre-activation)
        for l in range(7, 0, -1):
            lin = mlp.pts_linears[l]
            skip = (l - 1) in mlp.skips
            if skip:
                _dw(n, Za, pts, lin, *gw(lin), 0, ic, True, sc)
                _dw(n, Za, H[l - 1], lin, *gw(lin), ic, W, False, sc)
                _dx(n, S, [(f'pts{l}', Za)], [P + k for k in range(4)], Zb, mask=H[l - 1])
            else:
                _dw(n, Za, H[l - 1], lin, *gw(lin), 0, W, True, sc)
                _dx(n, S, [(f'pts{l}', Za)], [0, 1, 2, 3], Zb, mask=H[l - 1])
            Za, Zb = Zb, Za
        _dw(n, Za, pts, mlp.pts_linears[0], *gw(mlp.pts_linears[0]), 0, ic, True, sc)
        return (None, None) + tuple(g[id(t)] for t in params)


GRAD_CHUNK = 1 << 18   # rows per pass of density_grad: about 1.5 GB of tile images


def density_grad(mlp, pts, chunk=GRAD_CHUNK, sigma=None):
    """pts f32[n,3] -> (raw density f32[n], d(raw density)/d(position) f32[n,3]) of a NerfMLP, from the training kernels: the forward of
    pts_linears.0..7 and alpha_linear with saved activations, then d_raw = (0, 0, 0, 1) through alpha_linear and the trunk's input gradients down to
    the point encoding (the pts_linears.0 term and the point-block term of the skip layer pts_linears.5, ReLU masks of the forward), contracted with the
    encoding's derivative. feature_linear and the view branch are not run. In chunks of `chunk` rows.

    BaseEmbedder (input_ch 63, one point block; sigma None): the positional encoding. MipNerfEmbedder (two point blocks): the point query at
    footprint `sigma` (include/xrnerf_b200.h). The kernels are nerf_mlp.encode_points and nerf_mlp.encoding_grad.
    The staged activation gradients are fp16 at a scale of 2^12: an encoding-gradient entry above about 16 would overflow."""
    dev = pts.device
    n_all = int(pts.shape[0])
    dens = torch.empty(n_all, dtype=torch.float32, device=dev)
    grad = torch.empty((n_all, 3), dtype=torch.float32, device=dev)
    P = (mlp.input_ch + 63) // 64                                     # point blocks of the encoding
    S = getattr(mlp, '_tg_slabs', None)
    if S is None or S.arena.device != dev:
        S = mlp._tg_slabs = _Slabs(mlp, P)
    S.pack()
    vd = torch.zeros((1, 3), dtype=torch.float32, device=dev)         # any direction: the view branch is not evaluated
    for i0 in range(0, n_all, chunk):
        p = pts[i0:i0 + chunk]
        n = int(p.shape[0])
        nt = (n + 127) // 128
        enc = Img.new(nt, P + 1, dev)
        nm.encode_points(mlp, sigma, p, vd, n, enc.buf)
        pts_img = enc.sub(0, P)
        H = [Img.new(nt, 4, dev) for _ in range(8)]
        _fwd(n, S, 'pts0', [pts_img], H[0])
        for l in range(1, 8):
            _fwd(n, S, f'pts{l}', ([pts_img, H[l - 1]] if (l - 1) in mlp.skips else [H[l - 1]]), H[l])
        raw_a = dens[i0:i0 + n].view(n, 1)
        _fwd(n, S, 'alpha', [H[7]], yf=raw_a, yf_col=0, yf_n=1)
        d_raw = torch.zeros((n, 4), dtype=torch.float32, device=dev)
        d_raw[:, 3] = 1.0
        z_rgb, z_alpha = Img.new(nt, 1, dev), Img.new(nt, 1, dev)
        sc = torch.empty(2, dtype=torch.float32, device=dev)
        _C.check(_C.lib.xrb_nerf_tg_pack_draw(_C.ptr(d_raw), n, _C.ptr(z_rgb.buf), _C.ptr(z_alpha.buf), _C.ptr(sc), _C.stream()), 'tg_pack_draw')
        Za, Zb = Img.new(nt, 4, dev), Img.new(nt, 4, dev)
        d_enc = Img.new(nt, 2 * P, dev)                               # blocks 0..P-1: through pts_linears.0, P..2P-1: through the skip layer's point blocks
        _dx(n, S, [('alpha', z_alpha)], [0, 1, 2, 3], Za, mask=H[7])
        for l in range(7, 0, -1):
            if (l - 1) in mlp.skips:
                _dx(n, S, [(f'pts{l}', Za)], list(range(P)), d_enc.sub(P, P))
                _dx(n, S, [(f'pts{l}', Za)], [P + k for k in range(4)], Zb, mask=H[l - 1])
            else:
                _dx(n, S, [(f'pts{l}', Za)], [0, 1, 2, 3], Zb, mask=H[l - 1])
            Za, Zb = Zb, Za
        _dx(n, S, [('pts0', Za)], list(range(P)), d_enc.sub(0, P))
        nm.encoding_grad(mlp, sigma, p, d_enc.buf, 2, sc.data_ptr() + 4, grad[i0:i0 + n])
    return dens, grad


def run_mlp_train(mlp, embedded):
    _, params = param_list(mlp)
    return NerfMlpTrainFn.apply(mlp, embedded, *params)
