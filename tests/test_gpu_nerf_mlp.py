"""GPU parity of the fused wgmma NerfMLP kernel (xrb_nerf_mlp_forward) against the fp32 path of the same module (library GEMMs, the
reference's arithmetic) and the numpy oracle. Tolerance for the fp16-operand / fp32-accumulate pipeline over 12 layers:
|err| <= 2e-2 * max|raw| (measured ~3e-3); composited rgb <= 5e-3."""
import numpy as np
import pytest
import torch
from cases import MIP_CFG, MIP_MLP, MIP_MODEL, NERF_MLP

pytestmark = pytest.mark.gpu


def _ref_fp32(mlp, emb):
    prev, mlp.fused_train = getattr(mlp, 'fused_train', True), False
    try:
        with torch.enable_grad():   # autograd on, fused training kernels off => nn.Linear: the library-GEMM fp32 path
            return mlp.batchify_run_mlp(emb.clone().requires_grad_(True)).detach()
    finally:
        mlp.fused_train = prev


def _emulated_kernel(mlp, emb):
    """csrc/nerf_mlp_tc.cu's own arithmetic, in torch, over every row: fp16 encodings and fp16 weights; per layer the fp32 products summed in fp32,
    rounded to fp16, plus the fp16 bias (__hadd2), then an fp16 ReLU on every layer but feature_linear; alpha = fp32 dot product of the fp16
    pts_linears.7 output with the fp32 alpha_linear weights, plus its bias; rgb = fp32 accumulator + fp32 bias. Only the order of the fp32 sums differs."""
    prev = torch.backends.cuda.matmul.allow_tf32
    torch.backends.cuda.matmul.allow_tf32 = False    # fp32 GEMMs on fp16 values: exact products, fp32 sums
    try:
        with torch.no_grad():
            acc = lambda lin, h: h.float() @ lin.weight.half().float().t()
            layer = lambda lin, h, relu: (lambda y: y.clamp_min(0) if relu else y)(acc(lin, h).half() + lin.bias.half())
            pts, views = torch.split(emb.half(), [mlp.input_ch, mlp.input_ch_dirs], dim=-1)
            h = pts
            for i, lin in enumerate(mlp.pts_linears):
                h = layer(lin, h, True)
                if i in mlp.skips:
                    h = torch.cat([pts, h], -1)
            alpha = h.float() @ mlp.alpha_linear.weight.float().t() + mlp.alpha_linear.bias.float()
            h = torch.cat([layer(mlp.feature_linear, h, False), views], -1)
            h = layer(mlp.views_linears[0], h, True)
            return torch.cat([acc(mlp.rgb_linear, h) + mlp.rgb_linear.bias.float(), alpha], -1)
    finally:
        torch.backends.cuda.matmul.allow_tf32 = prev


@pytest.mark.parametrize('n_rays,s', [(1, 1), (1, 127), (3, 43), (40, 64), (500, 192)])
def test_fused_nerf_mlp_matches_fp32_path(n_rays, s):
    from xrnerf_b200 import registry as R
    torch.manual_seed(0)
    mlp = R.build_mlp(NERF_MLP).cuda()
    pts = torch.rand((n_rays, s, 3), device='cuda') * 4 - 2
    vd = torch.nn.functional.normalize(torch.randn((n_rays, 3), device='cuda'), dim=-1)
    with torch.no_grad():
        data = mlp({'pts': pts, 'viewdirs': vd})
        emb = mlp.embedder({'pts': pts, 'viewdirs': vd})['embedded']
    raw = data['raw']
    assert raw.shape == (n_rays, s, 4) and torch.isfinite(raw).all()
    ref = _ref_fp32(mlp, emb).reshape(n_rays, s, 4)
    err = (raw - ref).abs().max().item()
    assert err <= 2e-2 * ref.abs().max().item() + 1e-3, err


def test_fused_nerf_mlp_vs_numpy_oracle_and_render():
    from oracle import nerf_oracle as O
    from xrnerf_b200 import registry as R
    torch.manual_seed(1)
    mlp = R.build_mlp(NERF_MLP).cuda()
    render = R.build_render(dict(type='NerfRender', white_bkgd=True, raw_noise_std=0))
    rng = np.random.default_rng(0)
    n, s = 64, 64
    o = (rng.random((n, 3)) * 0.2).astype(np.float32); d = rng.normal(0, 1, (n, 3)).astype(np.float32)
    vd = d / np.linalg.norm(d, axis=-1, keepdims=True)
    z = np.broadcast_to(np.linspace(2, 6, s, dtype=np.float32), (n, s)).copy()
    pts = o[:, None] + d[:, None] * z[..., None]
    sd = {k: v.detach().cpu().numpy() for k, v in mlp.state_dict().items()}
    raw_ref = O.nerf_mlp(sd, O.embed(pts, vd), 63, 27).reshape(n, s, 4)
    rgb_ref = O.nerf_render(raw_ref, z, d, white_bkgd=True)['rgb']
    t = lambda a: torch.from_numpy(np.ascontiguousarray(a)).cuda()
    with torch.no_grad():
        data = mlp({'pts': t(pts), 'viewdirs': t(vd)})
        data.update(z_vals=t(z), rays_d=t(d))
        _, ret = render(data, is_test=True)
    assert np.abs(data['raw'].cpu().numpy() - raw_ref).max() <= 2e-2 * np.abs(raw_ref).max() + 1e-3
    assert np.abs(ret['rgb'].cpu().numpy() - rgb_ref).max() <= 5e-3


def test_fused_mip_mlp_matches_fp32_path():
    from xrnerf_b200 import registry as R
    torch.manual_seed(2)
    mlp = R.build_mlp(MIP_MLP).cuda()
    n, s1 = 300, 129
    d = torch.randn((n, 3), device='cuda')
    data = dict(rays_o=torch.rand((n, 3), device='cuda') * 0.2, rays_d=d, viewdirs=torch.nn.functional.normalize(d, dim=-1), radii=torch.full((n, 1), 1e-3, device='cuda'),
                z_vals=torch.linspace(2, 6, s1, device='cuda').expand(n, s1).contiguous())
    with torch.no_grad():
        emb = mlp.embedder(dict(data))['embedded']
        raw = mlp(dict(data))['raw']
    assert raw.shape == (n, s1 - 1, 4)
    ref = _ref_fp32(mlp, emb).reshape(n, s1 - 1, 4)
    assert (raw - ref).abs().max().item() <= 2e-2 * ref.abs().max().item() + 1e-3


def test_weight_repack_on_update():
    from xrnerf_b200 import registry as R
    torch.manual_seed(3)
    mlp = R.build_mlp(NERF_MLP).cuda()
    pts = torch.rand((8, 16, 3), device='cuda'); vd = torch.nn.functional.normalize(torch.randn((8, 3), device='cuda'), dim=-1)
    with torch.no_grad():
        a = mlp({'pts': pts, 'viewdirs': vd})['raw'].clone()
        mlp.rgb_linear.bias.add_(1.0)
        b = mlp({'pts': pts, 'viewdirs': vd})['raw']
    assert torch.allclose(b[..., :3], a[..., :3] + 1.0, atol=1e-5) and torch.equal(a[..., 3], b[..., 3])


MIP_TEST_MODEL = dict(MIP_MODEL, cfg=dict(MIP_CFG, phase='test'))


def _mip_rays(n, seed):
    g = torch.Generator(device='cuda').manual_seed(seed)
    d = torch.randn((n, 3), device='cuda', generator=g)
    o = torch.rand((n, 3), device='cuda', generator=g) * 0.2
    return o, d, torch.nn.functional.normalize(d, dim=-1), torch.full((n, 1), 1.2e-3, device='cuda')


def test_mip_ipe_tile_images_are_the_fp16_rounding_of_mip_embed():
    """xrb_mip_ipe_tiles_rays == xrb_nerf_pack_embedded(xrb_mip_embed(...)) byte for byte (same fp32 expressions, one fp16 rounding); ragged last tile.
    Degrees (0, 16, 0, 4) take the specialised kernel, (0, 16, 0, 3) the generic one."""
    from xrnerf_b200 import _C
    n, s = 37, 19                         # 703 rows: 5 full tiles + a ragged one
    o, d, vd, radii = _mip_rays(n, 4)
    z = (2.0 + 4.0 * torch.rand((n, s + 1), device='cuda')).sort(dim=-1).values.contiguous()
    emb = torch.empty((n * s, 123), device='cuda')
    _C.check(_C.lib.xrb_mip_embed(_C.ptr(z), _C.ptr(o), _C.ptr(d), _C.ptr(radii.reshape(-1)), _C.ptr(vd), n, s, 0, 16, 0, 4, _C.ptr(emb), None, None, _C.stream()))
    nbytes = _C.lib.xrb_nerf_enc_image_bytes(n * s, 96)
    a = torch.zeros(nbytes, dtype=torch.uint8, device='cuda'); b = torch.full((nbytes,), 0xA5, dtype=torch.uint8, device='cuda')
    _C.check(_C.lib.xrb_nerf_pack_embedded(_C.ptr(emb), n * s, 96, 27, _C.ptr(a), _C.stream()))
    _C.check(_C.lib.xrb_mip_ipe_tiles_rays(_C.ptr(z), _C.ptr(o), _C.ptr(d), _C.ptr(radii.reshape(-1)), _C.ptr(vd), n, s, 0, 16, 0, 4, _C.ptr(b), _C.stream()))
    assert nbytes == 6 * 3 * 16384
    assert torch.equal(a.view(torch.float16), b.view(torch.float16))      # as fp16 VALUES: where exp(-y_var/2) < 2^-25 the specialised kernel writes +0 without evaluating sin (may be -0 above)
    emb3 = torch.empty((n * s, 117), device='cuda')                        # the generic-degree kernel: byte for byte
    _C.check(_C.lib.xrb_mip_embed(_C.ptr(z), _C.ptr(o), _C.ptr(d), _C.ptr(radii.reshape(-1)), _C.ptr(vd), n, s, 0, 16, 0, 3, _C.ptr(emb3), None, None, _C.stream()))
    a3 = torch.zeros(nbytes, dtype=torch.uint8, device='cuda')
    _C.check(_C.lib.xrb_nerf_pack_embedded(_C.ptr(emb3), n * s, 96, 21, _C.ptr(a3), _C.stream()))
    c = torch.full((nbytes,), 0x5A, dtype=torch.uint8, device='cuda')
    _C.check(_C.lib.xrb_mip_ipe_tiles_rays(_C.ptr(z), _C.ptr(o), _C.ptr(d), _C.ptr(radii.reshape(-1)), _C.ptr(vd), n, s, 0, 16, 0, 3, _C.ptr(c), _C.stream()))
    assert torch.equal(a3, c)


def test_posenc_tile_images_match_fp32_posenc():
    """xrb_nerf_posenc_tiles / _rays (specialised multires 10/4 kernel, and the generic one at 10/3) == fp16 rounding of xrb_nerf_posenc on pts = o + d*z
    formed by torch (GetPts). The specialised kernel uses sincosf where the fp32 kernel uses sinf / cosf: allow 1 fp16 ulp on < 0.1 % of the entries."""
    from xrnerf_b200 import _C
    n, s = 29, 21
    g = torch.Generator(device='cuda').manual_seed(9)
    o = torch.rand((n, 3), device='cuda', generator=g); d = torch.randn((n, 3), device='cuda', generator=g)
    vd = torch.nn.functional.normalize(d, dim=-1)
    z = (2.0 + 4.0 * torch.rand((n, s), device='cuda', generator=g)).sort(dim=-1).values.contiguous()
    pts = (o[:, None, :] + d[:, None, :] * z[:, :, None]).contiguous()
    nbytes = _C.lib.xrb_nerf_enc_image_bytes(n * s, 63)
    for generic in (False, True):
        multires_dirs = 3 if generic else 4                                 # 10/4 takes the specialised kernel, 10/3 the generic one
        input_ch_dirs = 3 + 6 * multires_dirs
        emb = torch.empty((n * s, 63 + input_ch_dirs), device='cuda')
        _C.check(_C.lib.xrb_nerf_posenc(_C.ptr(pts), _C.ptr(vd), n * s, s, 10, multires_dirs, _C.ptr(emb), _C.stream()))
        ref = torch.zeros(nbytes, dtype=torch.uint8, device='cuda')
        _C.check(_C.lib.xrb_nerf_pack_embedded(_C.ptr(emb), n * s, 63, input_ch_dirs, _C.ptr(ref), _C.stream()))
        ref16 = ref.view(torch.float16).float()
        for ray_mode in (False, True):
            img = torch.full((nbytes,), 0xA5, dtype=torch.uint8, device='cuda')
            if ray_mode:
                _C.check(_C.lib.xrb_nerf_posenc_tiles_rays(_C.ptr(o), _C.ptr(d), _C.ptr(z), _C.ptr(vd), n, s, 10, multires_dirs, _C.ptr(img), _C.stream()))
            else:
                _C.check(_C.lib.xrb_nerf_posenc_tiles(_C.ptr(pts), _C.ptr(vd), n * s, s, 10, multires_dirs, _C.ptr(img), _C.stream()))
            got = img.view(torch.float16).float()
            diff = (got - ref16).abs()
            assert diff.max().item() <= 1e-3, (generic, ray_mode)             # one fp16 ulp below 1.0 is 4.9e-4
            assert (diff > 0).float().mean().item() <= (0.0 if generic else 1e-3), (generic, ray_mode)


@pytest.mark.parametrize('ic,icd', [(63, 27), (96, 27)])
def test_pack_embedded_image_decodes_with_the_slab_layout(ic, icd):
    """xrb_nerf_pack_embedded's image read back with the layout nerf_mlp._slab documents, not with the kernels' own helpers: the point columns,
    then the direction columns from the last block on, hold embedded.half(); padding columns and the rows past the last one are +0.
    300 rows: two full tiles and a ragged one."""
    from xrnerf_b200 import _C
    n = 300
    g = torch.Generator(device='cuda').manual_seed(11)
    emb = torch.randn((n, ic + icd), device='cuda', generator=g)
    n_tiles, n_blk = (n + 127) // 128, (ic + 63) // 64 + 1
    nbytes = _C.lib.xrb_nerf_enc_image_bytes(n, ic)
    assert nbytes == n_tiles * n_blk * 16384
    img = torch.full((nbytes,), 0xA5, dtype=torch.uint8, device='cuda')
    _C.check(_C.lib.xrb_nerf_pack_embedded(_C.ptr(emb), n, ic, icd, _C.ptr(img), _C.stream()))
    r, k = np.meshgrid(np.arange(128), np.arange(64), indexing='ij')
    off = (r >> 3) * 1024 + (r & 7) * 128 + (((k >> 3) ^ (r & 7)) << 4) + (k & 7) * 2          # byte of element (r, k) of a block
    blocks = img.cpu().numpy().view(np.float16).reshape(n_tiles, n_blk, 8192)[:, :, off // 2]  # [tile, block, row, col]
    got = blocks.transpose(0, 2, 1, 3).reshape(n_tiles * 128, n_blk * 64)
    want = np.zeros_like(got)
    e = emb.half().cpu().numpy()
    want[:n, :ic] = e[:, :ic]
    want[:n, (n_blk - 1) * 64:(n_blk - 1) * 64 + icd] = e[:, ic:]
    assert np.array_equal(got.view(np.uint16), want.view(np.uint16))


def test_fused_mip_renderer_matches_registry_network():
    """MipNerfRenderer (IPE tile images -> wgmma MLP -> composite, 2 levels) vs MipNerfNetwork.forward(is_test=True) with the fp32 library-GEMM MLP.
    Tolerance: fp16-operand MLP over 12 layers, then two composites and a resampling that moves with the coarse weights: rgb 1e-2."""
    from xrnerf_b200 import registry as R
    from xrnerf_b200.nerf import MipNerfRenderer
    torch.manual_seed(5)
    net = R.build_network(MIP_TEST_MODEL).cuda()
    n, S = 200, 128
    o, d, vd, radii = _mip_rays(n, 6)
    with torch.no_grad():
        got = MipNerfRenderer(net, near=2.0, far=6.0, n_samples=S).render(o, d, vd, radii)
        t = torch.linspace(0., 1., S + 1, device='cuda')
        data = dict(rays_o=o, rays_d=d, viewdirs=vd, radii=radii, z_vals=(2.0 * (1. - t) + 6.0 * t).expand(n, S + 1).contiguous())
        net.mlp.fused = False
        ref = net.forward(data, is_test=True)
    assert set(got) == set(ref) == {'rgb', 'disp', 'acc', 'coarse_rgb', 'coarse_disp', 'coarse_acc'}
    for k in ('rgb', 'coarse_rgb', 'acc', 'coarse_acc'):
        assert (got[k] - ref[k]).abs().max().item() <= 1e-2, k


@pytest.mark.parametrize('cfg,n_rows', [(NERF_MLP, 1), (NERF_MLP, 129), (NERF_MLP, 2 * 296 * 128 + 77), (MIP_MLP, 128), (MIP_MLP, 2 * 296 * 128 + 300)])
def test_nerf_mlp_two_tiles_in_flight_matches_emulation_and_fp32(cfg, n_rows):
    """csrc/nerf_mlp_tc.cu (256-wide layers streamed as [256 x 32] K-half slabs with 64-byte swizzle, several tiles per CTA at the larger sizes), every row,
    against a torch emulation of its own fp16 arithmetic (<= 1e-3 of max|raw|) and the fp32 library path (2e-2)."""
    from xrnerf_b200 import registry as R
    from xrnerf_b200.nerf_mlp import nerf_mlp_forward
    torch.manual_seed(7)
    mlp = R.build_mlp(cfg).cuda()
    emb = torch.randn((n_rows, mlp.input_ch + mlp.input_ch_dirs), device='cuda').clamp_(-1, 1)
    image, bias = mlp._packed()
    out = nerf_mlp_forward(image, bias, emb, mlp.input_ch, mlp.input_ch_dirs)
    emu = _emulated_kernel(mlp, emb)
    torch.cuda.synchronize()
    assert out.shape == emu.shape == (n_rows, 4)
    assert (out - emu).abs().max().item() <= 1e-3 * emu.abs().max().item() + 1e-6
    ref = _ref_fp32(mlp, emb)
    assert (out - ref).abs().max().item() <= 2e-2 * ref.abs().max().item() + 1e-3
