"""The NerfMLP training kernels (csrc/nerf_train.cu: xrb_nerf_tg_layer, xrb_nerf_tg_dw, xrb_nerf_tg_pack_weights, xrb_nerf_tg_pack_draw) one launch
at a time, and NerfMlpTrainFn's whole chain, against float64 restatements of the same operations, entry by entry.

Tile images are read and written by restate64's encoder / decoder, which implements the documented layout (csrc/tc.cuh, nerf_mlp._slab):
fp16 element (r, k) of a [128 x 64] block sits at byte (r >> 3) 1024 + (r & 7) 128 + (((k >> 3) ^ (r & 7)) << 4) + (k & 7) 2, and a weight slab
[n_pad x 64] uses the same formula with n_pad rows. Every reference starts from the kernel's own fp16 operands (the images handed to a launch, or
decoded from what the previous launch wrote), so its inputs are exact and no ReLU decision can differ.

Forward (tg_layer epi 0 / 1). z = sum_k a_k w_k + bias in float64 over the K = 64 x (A blocks) products the MMAs perform (padding columns
included: the slab's zero columns times the image's padding). The kernel accumulates the exact fp16 x fp16 products in fp32 on the tensor cores
(at most K 2^-22 M, M = sum_k |a_k w_k|, as in test_gpu_field_grad_exact.py) and then adds the fp32 bias once (2^-24 (|acc| + |bias|)), so its
pre-activation is within
    b = K 2^-22 M + 2^-23 (M + |bias|)
of z. Rounding to fp16 and ReLU are monotone: the fp16 output lies in [fp16(act(z - b)), fp16(act(z + b))], asserted for every entry; the fp32
head rows (epi 1) lie within b of z.
Input gradient (tg_layer b_mn = 1, epi 2 / 3). dX = dZ . W over the K dZ columns the MMAs read (16 for a 16-row head slab, the layer width
otherwise, both for the feature + alpha pair); no bias, so b = K 2^-22 M, and with epi 2 the interval is multiplied by the mask [x > 0] read from
the kernel's own x image, so the mask is exact.
Weight gradient (tg_dw). dW[o, k_off + k] += sum_r dZ[r, o] X[r, k] / s over the rows r < n, db[o] += sum_r dZ[r, o] / s (s: the staging scale,
from the device or 2^14 when none is given). A CTA keeps its
accumulators across its rows_cta = 128 ceil(tiles / CTAs per chunk) rows (tensor cores: rows_cta 2^-22 M; the bias sums are a chain of fp32 adds,
less), the flush multiplies by the exact power of two 1 / s, and the partial sums of the `per` CTAs of a chunk and the 8 bias threads of a column
meet in fp32 atomics (each 2^-24 (|pre| + M)). Hence |got - pre - ref| <= D 2^-23 (M + |pre|) with D = 2 rows_cta + 8 per, per as the launcher
computes it from the SM count. The kernel reads every row of a tile, so dZ must be zero in the padding rows (NerfMlpTrainFn keeps that: tg_pack_draw
zeroes them and every later dZ is a product of zero rows); the tests put finite garbage in X's padding rows to pin that precondition.
Chain (NerfMlpTrainFn). The forward layers are checked as above from the previous layer's decoded output. The backward is run in float64 from the
kernel's own activations and masks, and every weight and bias gradient entry must satisfy, as in test_gpu_field_grad_exact.py,
    |g - g64| <= (tau_l + D 2^-23) M'
  * tau_l = (R_l + 1) 2^-11 + Ksum_l 2^-22. R_l counts the fp16 stagings on the longest path into layer l's dZ (the head's dL/draw is one, every
    input-gradient launch above adds one: rgb 1, views 2, feature 3, alpha 1, pts7 4, ..., pts0 11); Ksum_l is the number of products of the
    dX launches on that path, whose fp32 accumulation is not covered by the 2^-11 of their rounding; the "+1" covers second-order terms.
  * A staged value v (scaled by s, the power of two tg_pack_draw chooses with max |dL/draw| s in [2^12, 2^13)) comes back as v (1 + d) + h with
    |d| <= 2^-11 and |h| <= 2^-25 (half the fp16 subnormal step): in unscaled units h <= 2^-11 FLOOR with FLOOR = 2^-25 / (s 2^-11). M' is the
    same chain on absolute values with FLOOR added to every live staged value (a row below n whose mask is on).
  * D as for tg_dw, with the larger of the two chunk counts a layer uses.
Nothing in b, tau, FLOOR or D is fitted to a run.

Sensitivity (test_altered_references_are_rejected): the same assertions reject the tg_dw reference without the last row of a ragged tile (n = 129
and 300), with the dZ scale off by a factor of 2, the Mip-NeRF / NeRF chain reference with the direction block's k_off moved by one column, and the
forward reference with one bias entry moved by one ulp of the fp16 it rounds to (seen in the rows whose input is all zero: there the
pre-activation is the bias alone and the interval is one fp16 value).

Real gradient magnitudes (test_blender_train_step_gradients): NerfNetwork.train_step and MipNerfNetwork.train_step with the Blender settings
(4096 rays, 64 + 128 samples or 2 x 128 for Mip-NeRF, white background, no perturbation) on synthetic rays, (embedded, dL/draw) captured at the
NerfMlpTrainFn boundary. The MSE over 3 x 4096 values makes dL/draw ~1e-7, where the floor term dominates M' and an entrywise bound says
little, so each tensor's relative L2 is compared with a float64 backward from the kernel's own activations. The limit is 1e-2: while every
staged value is inside fp16's normal range, each staging is a relative error of at most 2^-11 and there are at most 12 on any path, i.e.
12 2^-11 = 5.9e-3 even if every error had the same sign; a staged dZ that leaves the normal range loses relative precision without limit (0 when
it rounds to zero). The fraction of the staged dZ that is subnormal or zero in fp16 is printed per layer.
"""
import ctypes as C
import math
import time

import numpy as np
import pytest
import torch
from cases import MIP_MLP, NERF_MLP, host_buffer
from restate64 import BLOCK, GAMMA_TC, U16, decode, encode, f16, image, swz, ulp16, w16

SCALE = 16384.0             # xrb_nerf_tg_grad_scale(): the staging scale of a tg_dw launch without a device scale
REPORT = []
MODELS = {'nerf': NERF_MLP, 'mip': MIP_MLP}


def within(got, ref, bound):
    """(all |got - ref| <= bound and finite, largest err / bound, index of it)"""
    got = got.double()
    err = (got - ref).abs()
    ratio = torch.where(bound > 0, err / torch.where(bound > 0, bound, 1.0), torch.where(err > 0, math.inf, 0.0))
    k = int(torch.argmax(ratio.reshape(-1)))
    r = float(ratio.reshape(-1)[k])
    return bool(torch.isfinite(got).all()) and r <= 1.0, r, k


def interval(y16, z, b, relu, mask=None):
    """(every fp16 output inside [fp16(act(z - b)), fp16(act(z + b))] (x mask), largest |y - act(z)| / (b + half an ulp))"""
    act = (lambda v: v.clamp_min(0.0)) if relu else (lambda v: v)
    lo, hi, a = f16(act(z - b)), f16(act(z + b)), act(z)
    if mask is not None:
        lo, hi, a = (torch.where(mask, v, torch.zeros_like(v)) for v in (lo, hi, a))
    y = y16.double()
    ok = bool(torch.isfinite(y).all() and ((y >= lo) & (y <= hi)).all())
    ratio = float(((y - a).abs() / (b + 0.5 * ulp16(a.abs() + b))).max()) if y.numel() else 0.0
    return ok, ratio


def head_scale(d):
    """the staging scale tg_pack_draw chooses: the power of two s with max |dL/draw| s in [2^12, 2^13) (2^14 for an all-zero batch)"""
    m = float(d.abs().max()) if d.numel() else 0.0
    return SCALE if m == 0 else 2.0 ** (12 - math.floor(math.log2(m)))


def sm_count():
    return torch.cuda.get_device_properties(0).multi_processor_count


def dw_depth(n, n_chunks):
    """D of the tg_dw bound for one launch (the launcher's grid: per = SMs / chunks CTAs per chunk, at most one per tile)"""
    nt = (n + 127) // 128
    per = max(1, min(sm_count() // n_chunks, nt))
    return 2 * 128 * math.ceil(nt / per) + 8 * per


# ----------------------------------------------------------------------------------------------------------------------------- fixtures
@pytest.fixture(scope='module', autouse=True)
def _report():
    t0 = time.time()
    yield
    print(f'\n[nerf train exact] wall {time.time() - t0:.1f} s')
    for line in REPORT:
        print('  ' + line)
    _MLPS.clear()


_MLPS = {}


def mlp_for(kind):
    """a registry NerfMLP (default nn.Linear init, seeded) with its slab arena packed"""
    from xrnerf_b200 import nerf_train as NT
    from xrnerf_b200 import registry as R
    if kind not in _MLPS:
        torch.manual_seed(17 if kind == 'nerf' else 23)
        mlp = R.build_mlp(dict(MODELS[kind])).cuda()
        S = NT._Slabs(mlp, (mlp.input_ch + 63) // 64)
        S.pack()
        _MLPS[kind] = (mlp, S)
    return _MLPS[kind]


def b32(lin):
    return lin.bias.detach().double()


def rand16(rows, cols, seed, lo=-1.0, hi=1.0):
    g = torch.Generator(device='cuda').manual_seed(seed)
    return (torch.rand((rows, cols), device='cuda', generator=g) * (hi - lo) + lo).half()


# ----------------------------------------------------------------------------------------------------------------------------- layout
def test_tile_codec_is_the_documented_layout():
    """the test's encoder writes the bytes nerf_mlp._slab (the documented K-major 128-byte swizzle) writes, and decode inverts it"""
    from xrnerf_b200 import nerf_mlp as nm
    rng = np.random.default_rng(0)
    m = rng.normal(0, 1, (256, 128)).astype(np.float32)
    got = encode(torch.from_numpy(m).half()).numpy()
    want = np.concatenate([nm._slab(np.ascontiguousarray(m[128 * t:128 * (t + 1), 64 * b:64 * (b + 1)])) for t in range(2) for b in range(2)])
    assert np.array_equal(got, want)
    from xrnerf_b200.nerf_train import Img
    back = decode(Img(torch.from_numpy(got), 2 * BLOCK, 0, 2), 2)
    assert np.array_equal(back.numpy().view(np.uint16), m.astype(np.float16).view(np.uint16))


# ----------------------------------------------------------------------------------------------------------------------------- 1. packers
@pytest.mark.gpu
@pytest.mark.parametrize('kind', ['nerf', 'mip'])
def test_pack_weights_bit_exact(kind):
    """every slab _Slabs packs (pts0's ragged blocks, the skip layer's point blocks, the 27-column direction block at col0 = 256, the N = 1 and
    N = 3 heads padded to 16): fp16 RNE of W[row][col0 + k] for row < N and k < valid, +0 elsewhere; the arena is pre-filled with 0xA5"""
    from xrnerf_b200 import nerf_train as NT
    from xrnerf_b200 import registry as R
    torch.manual_seed(5)
    mlp = R.build_mlp(dict(MODELS[kind])).cuda()
    S = NT._Slabs(mlp, (mlp.input_ch + 63) // 64)
    S.arena.fill_(0xA5)
    S.pack()
    torch.cuda.synchronize()
    seen = set()
    for name, L in S.layers.items():
        W = L['lin'].weight.detach().cpu().numpy()
        N, n_pad = W.shape[0], L['n_pad']
        assert n_pad == (N + 15) // 16 * 16
        for kb, (col0, valid) in enumerate(L['blocks']):
            seen.add((N, W.shape[1], n_pad, col0, valid))
            off = L['off'] + kb * L['slab_bytes']
            slab = S.arena[off:off + n_pad * 128].view(torch.float16).cpu().numpy()[swz(n_pad)].reshape(n_pad, 64)
            want = np.zeros((n_pad, 64), np.float16)
            want[:N, :valid] = W[:, col0:col0 + valid].astype(np.float16)
            assert np.array_equal(slab.view(np.uint16), want.view(np.uint16)), (name, kb, col0, valid)
    ic = mlp.input_ch
    assert (128, 256 + 27, 128, 256, 27) in seen and (1, 256, 16, 192, 64) in seen and (3, 128, 16, 64, 64) in seen
    assert any(v < 64 for (_, _, _, _, v) in seen) and (256, ic, 256, 0, min(64, ic)) in seen
    REPORT.append(f'pack_weights {kind}: {len(seen)} distinct (N, K_in, n_pad, col0, valid) bit-exact')


@pytest.mark.gpu
@pytest.mark.parametrize('n', [1, 127, 128, 129, 300, 'zeros'])
def test_pack_draw_bit_exact(n):
    """fp16 RNE of dL/draw * s: rgb in columns 0..2 of one image, alpha in column 0 of the other, every other entry +0, rows >= n included
    (both images pre-filled with 0xA5). s is the power of two with max |dL/draw| s in [2^12, 2^13), written to scale[1]: the head cannot reach
    fp16's overflow. The underflow edges are pinned with max |dL/draw| = 2^-10 (s = 2^22): 2^-46 stays the smallest subnormal 2^-24, 2^-47 rounds
    to +0 (tie to even), 3 2^-48 rounds up to 2^-24, -2^-48 gives -0. An all-zero batch takes s = 2^14."""
    from xrnerf_b200 import _C
    zeros = n == 'zeros'
    n = 200 if zeros else n
    rng = np.random.default_rng(n)
    d = (rng.normal(0, 1, (n, 4)) * 1e-4).astype(np.float32)
    edges = np.array([2.0 ** -10, 2.0 ** -46, 2.0 ** -47, 3 * 2.0 ** -48, -(2.0 ** -48), -(2.0 ** -46), 1.5 * 2.0 ** -46, 0.0])
    flat = d.reshape(-1)
    flat[:min(flat.size, edges.size)] = edges[:flat.size].astype(np.float32)
    if zeros:
        d[:] = 0
    nt = (n + 127) // 128
    zr = torch.full((nt * BLOCK,), 0xA5, dtype=torch.uint8, device='cuda'); za = zr.clone()
    sc = torch.full((2,), -1.0, device='cuda')
    dd = torch.from_numpy(d).cuda()
    _C.check(_C.lib.xrb_nerf_tg_pack_draw(_C.ptr(dd), n, _C.ptr(zr), _C.ptr(za), _C.ptr(sc), _C.stream()))
    torch.cuda.synchronize()
    s_ = head_scale(torch.from_numpy(d))
    assert float(sc[1]) == s_ and (zeros or s_ == 2.0 ** 22)
    from xrnerf_b200.nerf_train import Img
    got_r = decode(Img(zr, BLOCK, 0, 1), nt).cpu().numpy().view(np.uint16)
    got_a = decode(Img(za, BLOCK, 0, 1), nt).cpu().numpy().view(np.uint16)
    s16 = (d.astype(np.float64) * s_).astype(np.float16)       # exact product, one RNE rounding
    want_r = np.zeros((nt * 128, 64), np.float16); want_r[:n, :3] = s16[:, :3]
    want_a = np.zeros((nt * 128, 64), np.float16); want_a[:n, 0] = s16[:, 3]
    assert np.array_equal(got_r, want_r.view(np.uint16)) and np.array_equal(got_a, want_a.view(np.uint16))
    if not zeros and n >= 2:
        e = s16.reshape(-1)[:8].astype(np.float64)
        assert e[0] == 4096 and e[1] == 2.0 ** -24 and e[2] == 0 and not np.signbit(s16.reshape(-1)[2]) and e[3] == 2.0 ** -24
        assert e[4] == 0 and np.signbit(s16.reshape(-1)[4]) and e[5] == -(2.0 ** -24) and e[6] == 2.0 ** -23
    assert float(np.abs(s16.astype(np.float64)).max()) < 2.0 ** 13


# ----------------------------------------------------------------------------------------------------------------------------- 2. tg_layer
class Operands:
    """random fp16 operand images for every descriptor NerfMlpTrainFn builds, at n rows, and their float64 values (rows < n)"""

    def __init__(self, kind, n, seed):
        from xrnerf_b200.nerf_train import Img
        self.mlp, self.S = mlp_for(kind)
        mlp = self.mlp
        self.n, self.nt = n, max(1, (n + 127) // 128)
        R, P = self.nt * 128, self.S.P
        self.ic, self.icd, self.P = mlp.input_ch, mlp.input_ch_dirs, P
        # encoding image: P point blocks + one direction block per tile; finite garbage in the padding columns (the slabs' zero columns cancel it)
        enc = rand16(R, (P + 1) * 64, seed)
        self.enc = Img(encode(enc), (P + 1) * BLOCK, 0, P + 1)
        self.pts, self.dirs = self.enc.sub(0, P), self.enc.sub(P, 1)
        self.pts64, self.dirs64 = enc[:n, :self.ic].double(), enc[:n, P * 64:P * 64 + self.icd].double()
        # activations: ReLU outputs (about a quarter exactly 0) for the masks; dZ images (scaled units) with garbage beyond the used columns
        act = lambda c, s: torch.clamp_min(rand16(R, c, s, -0.5, 1.5), 0).half()
        self.H_m, self.F_m, self.V_m = act(256, seed + 1), rand16(R, 256, seed + 2), act(128, seed + 3)
        self.H_m[::97] = 0                                       # dead rows: the pre-activation is the bias alone, M = 0 and the interval one fp16 value
        self.H, self.F, self.V = image(self.H_m), image(self.F_m), image(self.V_m)
        self.Z_m = {c: rand16(R, c, seed + 10 + c, -4, 4) for c in (64, 128, 256)}
        self.Z = {c: image(m) for c, m in self.Z_m.items()}

    def out(self, n_blk):
        from xrnerf_b200.nerf_train import Img
        img = Img.new(self.nt, n_blk, 'cuda')
        img.buf.fill_(0xA5)
        return img


def fwd_ref(x64, lin, K):
    W, bias = w16(lin), b32(lin)
    z = x64 @ W.T + bias
    M = x64.abs() @ W.abs().T
    return z, K * GAMMA_TC * M + 2.0 ** -23 * (M + bias.abs())


def dx_ref(pairs, mask64=None):
    """pairs [(dZ float64, W float64 restricted to the gradient's input columns, K products)] -> (z, b)"""
    z = sum(dz @ W for dz, W, _ in pairs)
    b = sum(K * GAMMA_TC * (dz.abs() @ W.abs()) for dz, W, K in pairs)
    return z, b


def run_layer_cases(kind, n, seed=1, bias_shift=None):
    """every tg_layer descriptor of NerfMlpTrainFn on random operand images; returns {case: largest err/bound}. bias_shift = (layer, column):
    the reference's bias entry moved by one fp16 ulp (sensitivity)"""
    from xrnerf_b200 import nerf_train as NT
    O = Operands(kind, n, seed)
    mlp, S, ic, icd, P = O.mlp, O.S, O.ic, O.icd, O.P
    out = {}
    H64, F64, V64 = O.H_m[:n].double(), O.F_m[:n].double(), O.V_m[:n].double()

    def fcheck(name, a_srcs, x64, relu, n_out_blk, lin):
        y = O.out(n_out_blk)
        NT._fwd(n, S, name, a_srcs, y, relu=relu)
        torch.cuda.synchronize()
        K = 64 * sum(a.n_blk for a in a_srcs)
        z, b = fwd_ref(x64, lin, K)
        if bias_shift and bias_shift[0] == name:
            c = bias_shift[1]
            z[:, c] += float(ulp16(f16(lin.bias.detach().double()[c:c + 1])))   # one ulp of the fp16 the bias rounds to
        ok, r = interval(decode(y, O.nt)[:n, :lin.out_features], z, b, relu)
        out[f'fwd {name}'] = (ok, r)

    fcheck('pts0', [O.pts], O.pts64, 1, 4, mlp.pts_linears[0])
    fcheck('pts1', [O.H], H64, 1, 4, mlp.pts_linears[1])
    fcheck('pts5', [O.pts, O.H], torch.cat([O.pts64, H64], 1), 1, 4, mlp.pts_linears[5])
    fcheck('feature', [O.H], H64, 0, 4, mlp.feature_linear)
    fcheck('views', [O.F, O.dirs], torch.cat([F64, O.dirs64], 1), 1, 2, mlp.views_linears[0])
    # the fp32 heads: alpha -> column 3, rgb -> columns 0..2 of one raw buffer; each launch leaves the other columns alone
    raw = torch.full((max(n, 1), 4), float('nan'), device='cuda')
    NT._fwd(n, S, 'alpha', [O.H], yf=raw, yf_col=3, yf_n=1)
    torch.cuda.synchronize()
    assert n == 0 or torch.isnan(raw[:, :3]).all()
    NT._fwd(n, S, 'rgb', [O.V], yf=raw, yf_col=0, yf_n=3)
    torch.cuda.synchronize()
    for name, cols, x64, lin, K in (('alpha', slice(3, 4), H64, mlp.alpha_linear, 256), ('rgb', slice(0, 3), V64, mlp.rgb_linear, 128)):
        z, b = fwd_ref(x64, lin, K)
        ok, r, _ = within(raw[:n, cols], z, b)
        out[f'fwd {name} (fp32 rows)'] = (ok, r)

    def dcheck(name, pairs_img, pairs_ref, obs, mask_img, mask64):
        y = O.out(len(obs))
        NT._dx(n, S, pairs_img, obs, y, mask=mask_img)
        torch.cuda.synchronize()
        z, b = dx_ref(pairs_ref)
        ok, r = interval(decode(y, O.nt)[:n], z, b, False, None if mask64 is None else mask64 > 0)
        out[f'dx {name}'] = (ok, r)

    Z64 = {c: m[:n].double() for c, m in O.Z_m.items()}
    W = lambda lin: w16(lin)
    z16 = O.Z[64]
    # rgb: dZ block with the 3 live columns (the rest is garbage the zero slab rows 3..15 and n_k = 1 must ignore); mask V; d_col 0, 64
    dcheck('rgb', [('rgb', z16)], [(Z64[64][:, :3], W(mlp.rgb_linear), 16)], [0, 1], O.V, V64)
    # views: the feature part only (obs 0..3: d_col 0, 64, 128, 192), no mask (epi 3)
    dcheck('views', [('views', O.Z[128])], [(Z64[128], W(mlp.views_linears[0])[:, :256], 128)], [0, 1, 2, 3], None, None)
    # feature + alpha: two A sources, 8 slabs, mask H
    dcheck('feature+alpha', [('feature', O.Z[256]), ('alpha', z16)], [(Z64[256], W(mlp.feature_linear), 256), (Z64[64][:, :1], W(mlp.alpha_linear), 16)],
           [0, 1, 2, 3], O.H, H64)
    # the skip layer: the hidden part of its input (slab blocks P..P+3)
    dcheck('pts5', [('pts5', O.Z[256])], [(Z64[256], W(mlp.pts_linears[5])[:, ic:], 256)], [P + k for k in range(4)], O.H, H64)
    dcheck('pts1', [('pts1', O.Z[256])], [(Z64[256], W(mlp.pts_linears[1]), 256)], [0, 1, 2, 3], O.H, H64)
    return out


@pytest.mark.gpu
@pytest.mark.parametrize('n', [1, 127, 128, 129, 40001])
@pytest.mark.parametrize('kind', ['nerf', 'mip'])
def test_tg_layer_every_descriptor(kind, n):
    """forward epi 0 with and without ReLU, one- and two-source A (skip, views), the fp32 heads (epi 1, yf_col / yf_n), the input gradient with
    mask (epi 2) and without (epi 3) at d_col 0 / 64 / 128 / 192, feature + alpha as one 8-slab launch; 40 001 rows = 313 tiles: every CTA takes
    several tiles and the 2-slot slab ring wraps"""
    out = run_layer_cases(kind, n)
    bad = {k: v for k, v in out.items() if not v[0]}
    REPORT.append(f'tg_layer {kind} n={n}: max err/bound ' + ' '.join(f'{k}={v[1]:.3f}' for k, v in out.items()))
    assert not bad, bad


@pytest.mark.gpu
def test_tg_layer_zero_rows_is_a_no_op():
    from xrnerf_b200 import nerf_train as NT
    O = Operands('nerf', 0, 3)
    y = O.out(4)
    before = y.buf.clone()
    raw = torch.full((1, 4), 7.0, device='cuda')
    NT._fwd(0, O.S, 'pts1', [O.H], y)
    NT._fwd(0, O.S, 'alpha', [O.H], yf=raw, yf_col=3, yf_n=1)
    NT._dx(0, O.S, [('pts1', O.Z[256])], [0, 1, 2, 3], y, mask=O.H)
    torch.cuda.synchronize()
    assert torch.equal(y.buf, before) and bool((raw == 7.0).all())


# ----------------------------------------------------------------------------------------------------------------------------- 3. tg_dw
# (name, N, K, x_n_blk, k_off, k_cols): the normal path (N = 128 / 256, 1..4 input blocks) and the transposed one (N <= 16, 2 or 4 blocks)
DW_CASES = [('pts0 nerf', 256, 63, 1, 0, 63), ('pts0 mip', 256, 96, 2, 0, 96), ('pts5 hidden', 256, 352, 4, 96, 256), ('3 blocks', 256, 200, 3, 10, 150),
            ('views dirs', 128, 283, 1, 256, 27), ('views feature', 128, 283, 4, 0, 256), ('alpha', 1, 256, 4, 0, 256), ('rgb', 3, 128, 2, 0, 128),
            ('16 ragged', 16, 110, 2, 5, 100)]


def dw_case(spec, n, with_bias, seed, drop_last=False, scale=SCALE, device_scale=None):
    """one tg_dw launch accumulating onto non-zero dW / db; returns (ok, ratio) for dW and db and the raw material for the sensitivity checks"""
    from xrnerf_b200 import nerf_train as NT
    name, N, K, xb, k_off, k_cols = spec
    nt = max(1, (n + 127) // 128)
    R = nt * 128
    zc = 64 if N <= 16 else N
    zm = rand16(R, zc, seed, -4, 4)
    zm[n:] = 0                                                   # the precondition: dZ is zero in the padding rows
    if N <= 16:
        zm[:n, N:] = 7.0                                         # columns >= N: computed by the N = 16 MMA (or not read), never flushed
    xm = rand16(R, 64 * xb, seed + 1)
    xm[n:] = 3.0                                                 # finite garbage in X's padding rows
    xm[:, k_cols:] = 5.0 if k_cols < 64 * xb else xm[:, k_cols:]   # and in the columns past k_cols
    zi, xi = image(zm), image(xm)
    g = torch.Generator(device='cuda').manual_seed(seed + 2)
    pre_w = torch.randn((N, K), device='cuda', generator=g) * 1e-3
    pre_b = torch.randn((N,), device='cuda', generator=g) * 1e-3
    dW, db = pre_w.clone(), pre_b.clone()
    lin = type('L', (), {'out_features': N, 'in_features': K})
    sc = None if device_scale is None else torch.tensor([0.0, device_scale], device='cuda')
    NT._dw(n, zi, xi, lin, dW, db, k_off, k_cols, with_bias, sc)
    torch.cuda.synchronize()
    scale = scale if device_scale is None else device_scale
    rows = n - 1 if drop_last else n
    z64, x64 = zm[:rows, :N].double(), xm[:rows, :k_cols].double()
    D = dw_depth(n, 1 if N <= 16 else N // 128) if N > 16 else dw_depth(n, xb // 2)
    refW = pre_w.double().clone(); MW = torch.zeros_like(refW)
    refW[:, k_off:k_off + k_cols] += z64.T @ x64 / scale
    MW[:, k_off:k_off + k_cols] = z64.abs().T @ x64.abs() / scale
    okW, rW, _ = within(dW, refW, D * 2.0 ** -23 * (MW + pre_w.double().abs()))
    refb = pre_b.double() + (z64.sum(0) / scale if with_bias else 0.0)
    Mb = z64.abs().sum(0) / scale if with_bias else torch.zeros(N, dtype=torch.float64, device='cuda')
    okb, rb, _ = within(db, refb, D * 2.0 ** -23 * (Mb + pre_b.double().abs()))
    return (okW, rW), (okb, rb)


def _three_tiles_per_cta():
    return 3 * sm_count() * 128 + 77


@pytest.mark.gpu
@pytest.mark.parametrize('n', [1, 127, 128, 129, 40001, 'three-tiles'])
def test_tg_dw_entrywise(n):
    """both paths, x_n_blk 1..4, ragged k_off / k_cols (63, 96, 27 at offset 256, 100 at offset 5), db NULL and non-NULL, accumulated onto
    non-zero dW and db; 'three-tiles': 3 x SMs x 128 + 77 rows, so that every CTA of every chunk takes at least 3 tiles"""
    n = _three_tiles_per_cta() if n == 'three-tiles' else n
    res = []
    for i, spec in enumerate(DW_CASES):
        for with_bias in (True, False):
            # with the bias: the staging scale from the device (2^20, as tg_pack_draw writes it); without: the fixed 2^14 (scale NULL)
            (okW, rW), (okb, rb) = dw_case(spec, n, with_bias, seed=100 + 7 * i + with_bias, device_scale=2.0 ** 20 if with_bias else None)
            assert okW and okb, (spec, n, with_bias, rW, rb)
            res.append(f'{spec[0]}{"" if with_bias else " (db NULL)"} dW={rW:.3f} db={rb:.3f}')
    REPORT.append(f'tg_dw n={n}: max err/bound ' + '; '.join(res))


@pytest.mark.gpu
def test_tg_dw_zero_rows_is_a_no_op():
    from xrnerf_b200 import nerf_train as NT
    zi, xi = image(rand16(128, 256, 1)), image(rand16(128, 256, 2))
    dW, db = torch.ones((256, 256), device='cuda'), torch.ones(256, device='cuda')
    NT._dw(0, zi, xi, type('L', (), {'out_features': 256, 'in_features': 256}), dW, db, 0, 256, True)
    torch.cuda.synchronize()
    assert bool((dW == 1).all() and (db == 1).all())


# ----------------------------------------------------------------------------------------------------------------------------- 4. the chain
def run_train_fn(kind, n, seed, d_scale=1e-3):
    """NerfMlpTrainFn forward + backward on random encodings; returns (mlp, saved images, d_raw, raw, {param: kernel gradient})"""
    from xrnerf_b200 import nerf_train as NT
    mlp, _ = mlp_for(kind)
    gen = torch.Generator().manual_seed(seed)
    x = (torch.rand((n, mlp.input_ch + mlp.input_ch_dirs), generator=gen) * 2 - 1).cuda()
    d = (torch.randn((n, 4), generator=gen) * d_scale).cuda()
    for p in mlp.parameters():
        p.grad = None
    raw = NT.run_mlp_train(mlp, x)
    assert 'NerfMlpTrainFn' in type(raw.grad_fn).__name__
    (raw * d).sum().backward()
    torch.cuda.synchronize()
    return mlp, raw.grad_fn.saved, d, raw.detach(), {id(p): p.grad.detach().clone() for p in mlp.parameters()}


class Chain:
    """float64 backward of NerfMlpTrainFn from the kernel's saved activations and masks: per nn.Linear (gW, gb) of the exact chain (unscaled), the
    mass chain (M', with the staging floor), tau and D; and per staged dZ the float64 values (for the subnormal census)"""

    def __init__(self, mlp, saved, d_raw, n):
        S, enc, pts, dirs, H, F, V = saved
        nt = (n + 127) // 128
        ic, icd = mlp.input_ch, mlp.input_ch_dirs
        dec = lambda img: decode(img, nt)[:n].double()
        self.pts, self.dirs = dec(pts)[:, :ic], dec(dirs)[:, :icd]
        self.H, self.F, self.V = [dec(h) for h in H], dec(F), dec(V)
        self.mlp, self.n = mlp, n
        d = d_raw[:n].double()
        self.s = head_scale(d)
        self.floor = 2.0 ** -25 / self.s / U16
        self.exact, self.mass, self.tau, self.staged = {}, {}, {}, {}
        for absolute in (False, True):
            self._run(d, absolute)
        D = max(dw_depth(n, 1), dw_depth(n, 2))
        self.bound = {k: (self.tau[k] + D * 2.0 ** -23) * self.mass[k][0] for k in self.exact}
        self.bound_b = {k: (self.tau[k] + D * 2.0 ** -23) * self.mass[k][1] for k in self.exact}

    def _run(self, d, absolute):
        mlp = self.mlp
        T = (lambda a: a.abs()) if absolute else (lambda a: a)
        Wm = lambda lin: T(w16(lin))
        st = (lambda v, live: v.abs() + self.floor * live) if absolute else (lambda v, live: v)
        out = self.mass if absolute else self.exact
        ones = torch.ones((self.n, 1), dtype=torch.float64, device='cuda')
        path = {}

        def grad(key, lin, dz, x, R, Ksum):
            out[key] = (dz.T @ T(x), dz.sum(0))
            self.tau[key] = (R + 1) * U16 + Ksum * GAMMA_TC
            if not absolute:
                self.staged[key] = dz

        z_rgb, z_a = st(d[:, :3], ones), st(d[:, 3:4], ones)
        grad('rgb', mlp.rgb_linear, z_rgb, self.V, 1, 0)
        m = (self.V > 0).double()
        zV = st((z_rgb @ Wm(mlp.rgb_linear)) * m, m)
        grad('views', mlp.views_linears[0], zV, torch.cat([self.F, self.dirs], 1), 2, 16)
        zF = st(zV @ Wm(mlp.views_linears[0])[:, :256], ones)
        grad('feature', mlp.feature_linear, zF, self.H[7], 3, 16 + 128)
        grad('alpha', mlp.alpha_linear, z_a, self.H[7], 1, 0)
        m = (self.H[7] > 0).double()
        z = st((zF @ Wm(mlp.feature_linear) + z_a @ Wm(mlp.alpha_linear)) * m, m)
        R, Ksum = 4, 16 + 128 + 272
        ic = mlp.input_ch
        for l in range(7, 0, -1):
            lin = mlp.pts_linears[l]
            skip = (l - 1) in mlp.skips
            grad(f'pts{l}', lin, z, torch.cat([self.pts, self.H[l - 1]], 1) if skip else self.H[l - 1], R, Ksum)
            m = (self.H[l - 1] > 0).double()
            Wl = Wm(lin)[:, ic:] if skip else Wm(lin)
            z = st((z @ Wl) * m, m)
            R, Ksum = R + 1, Ksum + 256
        grad('pts0', mlp.pts_linears[0], z, self.pts, R, Ksum)

    def lins(self):
        mlp = self.mlp
        return [(f'pts{l}', mlp.pts_linears[l]) for l in range(8)] + [('alpha', mlp.alpha_linear), ('feature', mlp.feature_linear),
                                                                        ('views', mlp.views_linears[0]), ('rgb', mlp.rgb_linear)]

    def check(self, grads, alter=None):
        """every weight and bias entry inside its bound; returns {layer: max err/bound}. alter(key, ref) may change a reference (sensitivity)"""
        out, bad = {}, []
        for key, lin in self.lins():
            gW, gb = grads[id(lin.weight)], grads[id(lin.bias)]
            refW, refb = self.exact[key]
            if alter is not None:
                refW = alter(key, refW.clone())
            okW, rW, kW = within(gW, refW, self.bound[key])
            okb, rb, _ = within(gb, refb, self.bound_b[key])
            out[key] = max(rW, rb)
            if not (okW and okb):
                bad.append((key, 'entry', divmod(kW, refW.shape[1]), rW, rb))
        return out, bad


def check_chain_forward(mlp, saved, raw, n):
    """every forward layer from the previous layer's decoded kernel output"""
    S, enc, pts, dirs, H, F, V = saved
    nt = (n + 127) // 128
    dec = lambda img: decode(img, nt)[:n]
    ic, icd, P = mlp.input_ch, mlp.input_ch_dirs, S.P
    p64, d64 = dec(pts)[:, :ic].double(), dec(dirs)[:, :icd].double()
    Hs = [dec(h) for h in H]
    out = {}
    x = p64
    for l in range(8):
        K = 64 * (P if l == 0 else (P + 4 if (l - 1) in mlp.skips else 4))
        z, b = fwd_ref(x, mlp.pts_linears[l], K)
        out[f'pts{l}'] = interval(Hs[l], z, b, True)
        x = torch.cat([p64, Hs[l].double()], 1) if l in mlp.skips else Hs[l].double()
    h7 = Hs[7].double()
    z, b = fwd_ref(h7, mlp.feature_linear, 256)
    out['feature'] = interval(dec(F), z, b, False)
    z, b = fwd_ref(torch.cat([dec(F).double(), d64], 1), mlp.views_linears[0], 320)
    out['views'] = interval(dec(V), z, b, True)
    z, b = fwd_ref(h7, mlp.alpha_linear, 256)
    out['alpha'] = within(raw[:n, 3:4], z, b)[:2]
    z, b = fwd_ref(dec(V).double(), mlp.rgb_linear, 128)
    out['rgb'] = within(raw[:n, :3], z, b)[:2]
    return out


@pytest.mark.gpu
@pytest.mark.parametrize('n', [1, 129, 300, 40000])
@pytest.mark.parametrize('kind', ['nerf', 'mip'])
def test_chain_entrywise(kind, n):
    """NerfMlpTrainFn end to end: each forward layer from the kernel's own previous output, then every weight and bias gradient entry against
    the float64 backward over the kernel's activations and masks (no ReLU-flip rejection is needed: the masks are the kernel's)"""
    mlp, saved, d, raw, grads = run_train_fn(kind, n, seed=1000 + n)
    fwd = check_chain_forward(mlp, saved, raw, n)
    bad = {k: v for k, v in fwd.items() if not v[0]}
    assert not bad, ('forward', bad)
    ch = Chain(mlp, saved, d, n)
    ratios, bad = ch.check(grads)
    REPORT.append(f'chain {kind} n={n}: forward max err/bound ' + ' '.join(f'{k}={v[1]:.3f}' for k, v in fwd.items())
                  + ' | gradients ' + ' '.join(f'{k}={v:.3f}' for k, v in ratios.items()))
    assert not bad, bad
    if n == 300:
        _chain_alterations_rejected(ch, grads, kind)


def _chain_alterations_rejected(ch, grads, kind):
    """the direction block's k_off moved by one column: the views weight reference with its 27 direction columns one column to the right"""
    def shift(key, ref):
        if key == 'views':
            blk = ref[:, 256:].clone()
            ref[:, 256:] = 0
            ref[:, 257:] = blk[:, :-1]
        return ref
    _, bad = ch.check(grads, alter=shift)
    assert any(b[0] == 'views' for b in bad), 'a shifted direction block went unnoticed'
    REPORT.append(f'sensitivity {kind}: direction block k_off + 1 rejected')


# ----------------------------------------------------------------------------------------------------------------------------- 5. sensitivity
@pytest.mark.gpu
def test_altered_references_are_rejected():
    """the assertions the kernels pass reject: the tg_dw reference without the last row of a ragged tile (129 rows: a 1-row tile; 300 rows:
    a 44-row tile), the dZ scale off by a factor of 2 (either way), and the forward reference with one bias entry moved by one fp16 ulp"""
    for n in (129, 300):
        for spec in (DW_CASES[0], DW_CASES[6]):
            (okW, _), (okb, _) = dw_case(spec, n, True, seed=5)
            assert okW and okb
            (okW, rW), (okb, rb) = dw_case(spec, n, True, seed=5, drop_last=True)
            assert not okW and not okb, ('dropped row went unnoticed', spec, n, rW, rb)
    for sc in (SCALE / 2, SCALE * 2):
        (okW, _), (okb, _) = dw_case(DW_CASES[2], 300, True, seed=6, scale=sc)
        assert not okW and not okb, ('scale', sc)
    mlp, _ = mlp_for('nerf')
    c = int(torch.argmax(mlp.pts_linears[1].bias.detach()))    # a positive bias: the dead rows' output is fp16(bias), one ulp from the altered one
    out = run_layer_cases('nerf', 40001, bias_shift=('pts1', c))
    assert not out['fwd pts1'][0], 'a bias one fp16 ulp off went unnoticed'
    assert all(v[0] for k, v in out.items() if k != 'fwd pts1')
    REPORT.append('sensitivity: dropped ragged row (n=129, 300), dZ scale x1/2 and x2, bias +1 fp16 ulp: all rejected')


# ----------------------------------------------------------------------------------------------------------------------------- 6. real gradient magnitudes
def _blender_rays(n, seed):
    """rays from cameras on a sphere of radius 4 looking at the origin (the Blender scenes' framing), directions spread over the image plane"""
    g = torch.Generator().manual_seed(seed)
    c = torch.nn.functional.normalize(torch.randn((n, 3), generator=g), dim=-1) * 4.0
    d = torch.nn.functional.normalize(-c + torch.randn((n, 3), generator=g) * 0.5, dim=-1)
    return c.cuda(), d.cuda()


def _capture(monkeypatch):
    from xrnerf_b200 import nerf_train as NT
    calls, orig = [], NT.run_mlp_train

    def wrapped(mlp, embedded):
        raw = orig(mlp, embedded)
        rec = {'mlp': mlp, 'node': raw.grad_fn, 'n': int(embedded.shape[0])}
        raw.register_hook(lambda g: rec.__setitem__('d_raw', g.detach().clone()))
        calls.append(rec)
        return raw
    monkeypatch.setattr(NT, 'run_mlp_train', wrapped)
    return calls


def _blender_step(kind):
    from xrnerf_b200 import registry as R
    torch.manual_seed(0)
    n = 4096
    o, d = _blender_rays(n, 1)
    tgt = torch.rand((1, n, 3), generator=torch.Generator().manual_seed(2)).cuda()
    if kind == 'nerf':
        net = R.build_network(dict(type='NerfNetwork', cfg=dict(phase='train', N_importance=128, is_perturb=False, chunk=1024 * 32, bs_data='rays_o'), mlp=NERF_MLP,
                                   mlp_fine=NERF_MLP, render=dict(type='NerfRender', white_bkgd=True, raw_noise_std=0))).cuda()
        t = torch.linspace(0., 1., 64, device='cuda')
        z = (2.0 * (1. - t) + 6.0 * t).expand(n, 64).contiguous()
        data = {'rays_o': o[None], 'rays_d': d[None], 'viewdirs': d[None], 'z_vals': z[None], 'pts': (o[:, None, :] + d[:, None, :] * z[:, :, None])[None], 'target_s': tgt}
    else:
        net = R.build_network(dict(type='MipNerfNetwork', cfg=dict(phase='train', ray_shape='cone', resample_padding=0.01, use_multiscale=False, coarse_loss_mult=0.1,
                                                                   num_levels=2, chunk=1024 * 32, bs_data='rays_o'), mlp=MIP_MLP,
                                   render=dict(type='MipNerfRender', white_bkgd=True, raw_noise_std=0, rgb_padding=0.001, density_bias=-1, density_activation='softplus'))).cuda()
        t = torch.linspace(0., 1., 129, device='cuda')
        z = (2.0 * (1. - t) + 6.0 * t).expand(n, 129).contiguous()
        data = {'rays_o': o[None], 'rays_d': d[None], 'viewdirs': d[None], 'radii': torch.full((1, n, 1), 1.2e-3, device='cuda'), 'z_vals': z[None], 'target_s': tgt}
    opt = torch.optim.Adam(net.parameters(), lr=5e-4)
    return net, data, opt


@pytest.mark.gpu
@pytest.mark.parametrize('kind', ['nerf', 'mip'])
def test_blender_train_step_gradients(kind, monkeypatch):
    """every weight and bias gradient of a Blender-sized train_step within 1e-2 relative L2 of the float64 backward over the kernel's own
    activations; the staged dZ census (fraction subnormal / zero in fp16, largest magnitude) is printed per layer"""
    calls = _capture(monkeypatch)
    net, data, opt = _blender_step(kind)
    out = net.train_step(data, opt)
    opt.zero_grad(set_to_none=True)
    out['loss'].backward()
    torch.cuda.synchronize()
    assert len(calls) == 2 and all('d_raw' in c for c in calls)
    refs, census, lines = {}, {}, []
    for c in calls:
        mlp, n = c['mlp'], c['n']
        ch = _exact_only(mlp, c['node'].saved, c['d_raw'], n)
        lines.append(f'{kind} call n={n}: staging scale 2^{int(math.log2(ch.s))}, |dL/draw| rms {float(c["d_raw"].double().pow(2).mean().sqrt()):.2e} max {float(c["d_raw"].abs().max()):.2e}')
        for key, lin in ch.lins():
            gW, gb = ch.exact[key]
            k = (id(mlp), key)
            if k in refs:
                refs[k] = (lin, refs[k][1] + gW, refs[k][2] + gb)
            else:
                refs[k] = (lin, gW, gb)
            v = ch.staged[key] * ch.s
            live = v != 0
            cnt, sub, zero, mx = census.get(k, (0, 0, 0, 0.0))
            census[k] = (cnt + int(live.sum()), sub + int((live & (v.abs() < 2.0 ** -14)).sum()), zero + int((live & (v.abs() <= 2.0 ** -25)).sum()),
                         max(mx, float(v.abs().max()) if v.numel() else 0.0))
    worst, bad = 0.0, []
    for k, (lin, gW, gb) in refs.items():
        rel = []
        for got, ref in ((lin.weight.grad, gW), (lin.bias.grad, gb)):
            r = float((got.double() - ref).norm() / ref.norm().clamp_min(1e-300))
            rel.append(r)
            if not r <= 1e-2:
                bad.append((k[1], r))
        cnt, sub, zero, mx = census[k]
        lines.append(f'  {k[1]:8s} staged dZ: subnormal {sub / max(cnt, 1):7.2%} zero {zero / max(cnt, 1):7.2%} max|dZ s| {mx:.2e} | rel L2 W {rel[0]:.2e} b {rel[1]:.2e}')
        worst = max(worst, *rel)
    REPORT.append(f'blender train_step {kind}: worst relative L2 {worst:.2e}')
    REPORT.extend(lines)
    print('\n'.join(lines))
    assert not bad, bad
    # measured, not derived: dZ shrinks on its way down the trunk, so the head's bound max < 2^13 keeps every layer far from fp16's overflow
    assert all(c[3] < 2.0 ** 15 for c in census.values()), census


class _exact_only(Chain):
    """the exact chain only (the Blender-sized rows make the mass chain needless: the test compares relative L2)"""

    def __init__(self, mlp, saved, d_raw, n):
        S, enc, pts, dirs, H, F, V = saved
        nt = (n + 127) // 128
        dec = lambda img: decode(img, nt)[:n].double()
        self.pts, self.dirs = dec(pts)[:, :mlp.input_ch], dec(dirs)[:, :mlp.input_ch_dirs]
        self.H, self.F, self.V = [dec(h) for h in H], dec(F), dec(V)
        self.mlp, self.n = mlp, n
        self.s = head_scale(d_raw[:n])
        self.exact, self.mass, self.tau, self.staged = {}, {}, {}, {}
        self._run(d_raw[:n].double(), False)


# ----------------------------------------------------------------------------------------------------------------------------- 7. argument validation
def _lib():
    from xrnerf_b200 import _C
    from xrnerf_b200 import nerf_train  # noqa: F401  (declares the argument types)
    _C.lib.xrb_last_error.restype = C.c_char_p
    return _C.lib


def _good_layer(a):
    """a descriptor that passes every check (forward pts1: 4 A blocks, 4 slabs of 256 x 64); never launched here"""
    from xrnerf_b200.nerf_train import TgLayer
    L = TgLayer()
    L.a_base[0], L.a_tile_stride[0], L.a_blk_off[0], L.a_n_blk[0], L.n_a = a, 4 * BLOCK, 0, 4, 1
    L.w = a
    for s in range(4):
        L.slab_w_off[s], L.slab_bytes[s], L.slab_n_sub[s], L.slab_a_blk0[s], L.slab_d_col[s], L.slab_first[s], L.slab_n_k[s] = s * 32768, 32768, 1, s, 0, int(s == 0), 4
    L.n_slabs, L.b_mn, L.mma_n, L.out_cols, L.epi, L.relu = 4, 0, 256, 256, 0, 1
    L.y, L.y_tile_stride = a, 4 * BLOCK
    L.n_rows = 1000
    return L


def test_tg_layer_argument_validation_without_gpu():
    """every XRB_REQUIRE of xrb_nerf_tg_layer, each violated alone on a descriptor that otherwise passes"""
    lib = _lib()
    _, a = host_buffer(1 << 16)
    assert lib.xrb_nerf_tg_layer(None, None) == -1 and b'null descriptor' in lib.xrb_last_error()

    def bad(msg, **kv):
        L = _good_layer(a)
        for k, v in kv.items():
            if '__' in k:
                f, i = k.split('__')
                getattr(L, f)[int(i)] = v
            else:
                setattr(L, k, v)
        assert lib.xrb_nerf_tg_layer(C.byref(L), None) == -1, kv
        assert msg.encode() in lib.xrb_last_error(), (kv, lib.xrb_last_error())

    for kv in (dict(n_rows=-1), dict(n_a=0), dict(n_a=3), dict(n_slabs=0), dict(n_slabs=11)):
        bad('bad sizes', **kv)
    L = _good_layer(a); L.w = None; L.n_rows = 0
    assert lib.xrb_nerf_tg_layer(C.byref(L), None) == 0                                  # no rows: nothing is read, not even the pointers
    bad('null pointer', w=None)
    bad('null pointer', a_base__0=None)
    for kv in (dict(epi=4), dict(epi=-1), dict(out_cols=8), dict(out_cols=272), dict(out_cols=200)):
        bad('bad epilogue', **kv)
    bad('MMA N must be', mma_n=32)
    bad('128-byte aligned', a_base__0=a + 64)
    bad('128-byte aligned', a_n_blk__0=0)
    bad('at most 6 input blocks', n_a=2, a_base__1=a, a_n_blk__1=3)
    for kv in (dict(slab_n_k__2=0), dict(slab_n_k__2=5), dict(slab_n_sub__2=0)):
        bad('slab K-steps', **kv)
    for kv in (dict(slab_bytes__1=32768 + 1024), dict(slab_bytes__1=16384 + 512), dict(slab_w_off__1=32768 + 64)):
        bad('slab size/offset', **kv)
    bad('outside the tile', slab_a_blk0__3=4)
    bad('outside the tile', slab_d_col__0=64)
    bad('implemented MMA shapes', mma_n=128, slab_d_col__0=64, slab_bytes__0=16384, slab_bytes__1=16384, slab_bytes__2=16384, slab_bytes__3=16384)
    bad('implemented MMA shapes', mma_n=64, b_mn=1, slab_d_col__0=32)
    # every MMA reads inside its slab: forward mma_n rows of 128 bytes; input gradient ((n_sub - 1) 4 + n_k) 2 KB
    bad('MMA reads past the slab', slab_bytes__2=16384)
    ig = dict(b_mn=1, mma_n=64, out_cols=64, epi=3)
    bad('MMA reads past the slab', **ig, slab_n_sub__0=4, slab_bytes__0=16384)                # an oversized n_k / n_sub would read stale ring data
    bad('MMA reads past the slab', **ig, slab_n_k__1=2, slab_bytes__1=2048)
    bad('output', epi=1, yf=None, yf_n=1)
    bad('output', epi=1, yf=a, yf_n=0)
    bad('output', epi=1, yf=a, yf_n=17)
    bad('output', y=None)
    bad('output', out_cols=16, mma_n=16, slab_bytes__0=2048, slab_bytes__1=2048, slab_bytes__2=2048, slab_bytes__3=2048)
    bad('mask image missing', epi=2, b_mn=1, mma_n=64, out_cols=64, x_base=None)


def test_tg_dw_argument_validation_without_gpu():
    """every XRB_REQUIRE of xrb_nerf_tg_dw, including k_cols <= 64 x_n_blk (wider columns would never be written)"""
    from xrnerf_b200.nerf_train import TgDw
    lib = _lib()
    _, a = host_buffer(1 << 16)
    assert lib.xrb_nerf_tg_dw(None, None) == -1 and b'null descriptor' in lib.xrb_last_error()

    def desc(**kv):
        D = TgDw(a, 4 * BLOCK, 0, a, 4 * BLOCK, 0, 4, 256, 256, 0, 256, a, a, 1000)
        for k, v in kv.items():
            setattr(D, k, v)
        return D

    def bad(msg, **kv):
        assert lib.xrb_nerf_tg_dw(C.byref(desc(**kv)), None) == -1, kv
        assert msg.encode() in lib.xrb_last_error(), (kv, lib.xrb_last_error())

    for kv in (dict(n_rows=-1), dict(N=0), dict(K=0), dict(x_n_blk=0), dict(x_n_blk=5), dict(k_off=-1), dict(k_cols=0), dict(k_off=1), dict(K=200)):
        bad('bad sizes', **kv)
    bad('k_cols wider than the input blocks', x_n_blk=3)
    bad('k_cols wider than the input blocks', x_n_blk=1, K=400, k_off=256, k_cols=65)
    assert lib.xrb_nerf_tg_dw(C.byref(desc(n_rows=0, z_base=None)), None) == 0
    bad('null pointer', z_base=None)
    bad('null pointer', x_base=None)
    bad('null pointer', dW=None)
    bad('128 or 256 columns', N=3, x_n_blk=3, k_cols=128)
    bad('N must be 128 or 256', N=64)


def test_tg_pack_argument_validation_without_gpu():
    """every XRB_REQUIRE of xrb_nerf_tg_pack_weights and xrb_nerf_tg_pack_draw"""
    lib = _lib()
    _, a = host_buffer(1 << 16)
    I = lambda *v: (C.c_int * len(v))(*v)
    w, s = C.c_void_p(a), C.c_void_p(a)

    def pw(W=w, N=256, K_in=63, n_pad=256, n_kb=1, col0=I(0), valid=I(63), slabs=s):
        return lib.xrb_nerf_tg_pack_weights(W, N, K_in, n_pad, n_kb, col0, valid, slabs, None)
    for kv in (dict(W=None), dict(slabs=None), dict(col0=None), dict(valid=None), dict(N=0), dict(n_pad=248), dict(N=3, n_pad=12), dict(n_kb=0),
               dict(n_kb=7, col0=I(*[0] * 7), valid=I(*[0] * 7))):
        assert pw(**kv) == -1 and b'bad arguments' in lib.xrb_last_error(), kv
    assert pw(slabs=C.c_void_p(a + 64)) == -1 and b'128-byte aligned' in lib.xrb_last_error()
    for col0, valid in ((-1, 10), (0, -1), (0, 65), (10, 54)):
        assert pw(col0=I(col0), valid=I(valid)) == -1 and b'outside the matrix' in lib.xrb_last_error(), (col0, valid)
    assert lib.xrb_nerf_tg_pack_draw(None, C.c_int64(-1), None, None, None, None) == -1 and b'negative' in lib.xrb_last_error()
    assert lib.xrb_nerf_tg_pack_draw(None, C.c_int64(0), None, None, None, None) == 0
    for args in ((None, s, s, s), (s, None, s, s), (s, s, None, s), (s, s, s, None)):
        assert lib.xrb_nerf_tg_pack_draw(args[0], C.c_int64(5), args[1], args[2], args[3], None) == -1 and b'null' in lib.xrb_last_error(), args
    assert lib.xrb_nerf_tg_pack_draw(C.c_void_p(a + 4), C.c_int64(5), s, s, s, None) == -1 and b'misaligned' in lib.xrb_last_error()
    assert lib.xrb_nerf_tg_pack_draw(s, C.c_int64(5), s, s, C.c_void_p(a + 2), None) == -1 and b'misaligned' in lib.xrb_last_error()
