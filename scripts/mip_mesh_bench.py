"""Times Mip-NeRF mesh export on one GPU: NerfMLP.density_lattice with a MipNerfEmbedder (xrb_mip_density_lattice) at 256^3 and 512^3 with the
'cell' footprint, against the point encoder (xrb_mip_ipe_tiles_points) + nerf_mlp_forward on the same points (in 2^21-row chunks),
NerfMLP.density_grad per 2^20 points, and MipNerfNetwork.extract_mesh / extract_colored_mesh at 256^3 on the sine field of
tests/test_gpu_mip_mesh.py and on a default-initialised network. Every shape is run once before it is timed; medians of repeated calls, CUDA
events; the card, power limit and SM clock are read in the same run.

    python scripts/mip_mesh_bench.py [--reps 10]
"""
import argparse
import json
import math
import os
import subprocess
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, 'tests'))

MAC_DENSITY = 508160   # per point: pts_linears.0..7 (96x256 + 6 x 256x256 + 352x256) + alpha_linear
MAC_FULL = 610304      # the whole NerfMLP: + feature_linear, views_linears.0, rgb_linear


def card():
    q = subprocess.run(['nvidia-smi', '--query-gpu=name,power.limit,clocks.sm,clocks.max.sm', '--format=csv,noheader'], capture_output=True, text=True)
    return q.stdout.strip().splitlines()[0] if q.returncode == 0 else 'unknown'


def timed(fn, reps):
    fn()
    torch.cuda.synchronize()
    ts = []
    for _ in range(reps):
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        a.record(); fn(); b.record()
        torch.cuda.synchronize()
        ts.append(a.elapsed_time(b))
    return sorted(ts)[len(ts) // 2]


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--reps', type=int, default=10)
    args = ap.parse_args()
    assert torch.cuda.is_available(), 'needs a GPU'
    from test_gpu_mip_mesh import BOX, MIP_MLP, RGB_PADDING, _bands, _infer, _lattice_points, _sine_network
    from xrnerf_b200 import registry as R
    from xrnerf_b200.mesh import footprint_sigma
    from xrnerf_b200.registry.networks import MipNerfNetwork
    out = {'card_before': card()}
    torch.manual_seed(0)
    mlp = R.build_mlp(MIP_MLP).cuda()
    with torch.no_grad():
        for n in (256, 512):
            shape = (n, n, n)
            sigma = footprint_sigma('cell', shape, BOX)
            pts = _lattice_points(shape, BOX)
            dirs = torch.nn.functional.normalize(torch.randn_like(pts), dim=-1)
            t_lat = timed(lambda: mlp.density_lattice(shape, BOX, footprint='cell'), args.reps)
            ch = 1 << 21
            t_cmp = timed(lambda: [_infer(mlp, pts[i:i + ch], dirs[i:i + ch], sigma) for i in range(0, pts.shape[0], ch)], args.reps)
            npt = n ** 3
            out[f'lattice_{n}'] = dict(sigma=sigma, live_bands=int((_bands(sigma) > 0).sum()),
                                       density_lattice_ms=t_lat, encoder_plus_mlp_ms=t_cmp, lattice_tflops=2 * MAC_DENSITY * npt / t_lat * 1e-9,
                                       comparison_tflops=2 * MAC_FULL * npt / t_cmp * 1e-9)
            del pts, dirs
        p = (torch.rand((1 << 20, 3), device='cuda') * 3 - 1.5).contiguous()
        out['density_grad_2e20_ms'] = timed(lambda: mlp.density_grad(p, footprint=footprint_sigma('cell', (256,) * 3, BOX)), args.reps)
    default = MipNerfNetwork(dict(phase='test', ray_shape='cone', resample_padding=0.01, use_multiscale=False, coarse_loss_mult=0.1, num_levels=2, chunk=800,
                                  bs_data='rays_o'),
                             mlp=MIP_MLP, render=dict(type='MipNerfRender', white_bkgd=True, raw_noise_std=0, rgb_padding=RGB_PADDING, density_bias=-1,
                                                      density_activation='softplus')).cuda()
    for name, net, thr in (('sine', _sine_network(), math.log1p(math.exp(-1.0))), ('default_init', default, math.log1p(math.exp(-1.0 + 1e-3)))):
        v, f = net.extract_mesh(256, thr, footprint='cell')
        out[f'mesh_{name}_256'] = dict(V=int(v.shape[0]), F=int(f.shape[0]), extract_mesh_ms=timed(lambda: net.extract_mesh(256, thr, footprint='cell'), 3),
                                       extract_colored_mesh_ms=timed(lambda: net.extract_colored_mesh(256, thr, footprint='cell'), 3))
    out['card_after'] = card()
    print(json.dumps(out))


if __name__ == '__main__':
    main()
