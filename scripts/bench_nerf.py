"""Developer probe: tensor-pipe throughput of the fused wgmma NerfMLP kernel vs the fp32 library-GEMM path (config-3 shape)."""
import sys, os
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import torch
from xrnerf_b200 import registry as R
from xrnerf_b200.nerf_mlp import nerf_mlp_forward

MLP = dict(type='NerfMLP', skips=[4], netdepth=8, netwidth=256, netchunk=1024 * 32, output_ch=5, use_viewdirs=True, embedder=dict(type='BaseEmbedder', i_embed=0, multires=10, multires_dirs=4))


def timeit(fn, n=5, warm=2):
    for _ in range(warm):
        fn()
    torch.cuda.synchronize()
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    a.record()
    for _ in range(n):
        fn()
    b.record(); torch.cuda.synchronize()
    return a.elapsed_time(b) / n


mlp = R.build_mlp(MLP).cuda()
rows = 32768 * 64            # 32 768 rays x 64 samples
emb = torch.randn((rows, 90), device='cuda')
flop = rows * 593408 * 2
from xrnerf_b200 import _C
from xrnerf_b200.nerf_mlp import nerf_mlp_forward_tiles, pack_nerf_mlp
image, bias = pack_nerf_mlp(mlp)
t = timeit(lambda: nerf_mlp_forward(image, bias, emb, 63, 27))
print(f'fused wgmma NerfMLP (fp32 rows, packing included): {t:.3f} ms for {rows} rows -> {flop / t / 1e9:.1f} TFLOP/s ({rows / t / 1e3:.1f} Mrows/s)', flush=True)
enc = torch.empty(_C.lib.xrb_nerf_enc_image_bytes(rows, 63), dtype=torch.uint8, device='cuda')
_C.check(_C.lib.xrb_nerf_pack_embedded(_C.ptr(emb), rows, 63, 27, _C.ptr(enc), _C.stream()))
raw = torch.empty((rows, 4), device='cuda')
t = timeit(lambda: nerf_mlp_forward_tiles(image, bias, enc, rows, 63, 27, raw))
print(f'   MLP kernel alone (pre-packed encodings): {t:.3f} ms -> {flop / t / 1e9:.1f} TFLOP/s', flush=True)
z = torch.linspace(2, 6, 64, device='cuda').expand(32768, 64).contiguous(); o = torch.rand((32768, 3), device='cuda'); d = torch.nn.functional.normalize(torch.randn((32768, 3), device='cuda'), dim=-1)
t = timeit(lambda: _C.check(_C.lib.xrb_nerf_posenc_tiles_rays(_C.ptr(o), _C.ptr(d), _C.ptr(z), _C.ptr(d), 32768, 64, 10, 4, _C.ptr(enc), _C.stream())))
print(f'   posenc tile images (ray mode, 32768 x 64): {t:.3f} ms', flush=True)
z2 = torch.linspace(2, 6, 129, device='cuda').expand(32768, 129).contiguous(); rad = torch.full((32768,), 5e-4, device='cuda')
enc2 = torch.empty(_C.lib.xrb_nerf_enc_image_bytes(32768 * 128, 96), dtype=torch.uint8, device='cuda')
t = timeit(lambda: _C.check(_C.lib.xrb_mip_ipe_tiles_rays(_C.ptr(z2), _C.ptr(o), _C.ptr(d), _C.ptr(rad), _C.ptr(d), 32768, 128, 0, 16, 0, 4, _C.ptr(enc2), _C.stream())))
print(f'   IPE tile images (32768 x 128): {t:.3f} ms', flush=True)
if os.environ.get('XRB_SKIP_LIB'):
    sys.exit(0)
with torch.enable_grad():
    x = emb[:32768 * 8].clone().requires_grad_(True)
    t2 = timeit(lambda: mlp.batchify_run_mlp(x), n=3, warm=1)
print(f'library fp32 GEMM path: {t2:.3f} ms for {x.shape[0]} rows -> {x.shape[0] * 593408 * 2 / t2 / 1e9:.1f} TFLOP/s')
torch.backends.cuda.matmul.allow_tf32 = True
with torch.enable_grad():
    t3 = timeit(lambda: mlp.batchify_run_mlp(x), n=3, warm=1)
print(f'library TF32 GEMM path: {t3:.3f} ms -> {x.shape[0] * 593408 * 2 / t3 / 1e9:.1f} TFLOP/s')
