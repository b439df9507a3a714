"""Times NeRF mesh export on one GPU: NerfMLP.density_lattice at 256^3 and 512^3 against the point encoder + nerf_mlp_forward on the same points
(in 2^21-row chunks), NerfMLP.density_grad per 2^20 points, and extract_mesh / extract_colored_mesh at 256^3 on an analytic field and on a
default-initialised network. Plain: NerfNetwork with BaseEmbedder (xrb_nerf_density_lattice against posenc_tiles + the MLP), on the octahedron field
of tests/test_gpu_nerf_mesh.py. --mip: MipNerfNetwork with MipNerfEmbedder at the 'cell' footprint (xrb_mip_density_lattice against
xrb_mip_ipe_tiles_points + the MLP), on the sine field of tests/test_gpu_mip_mesh.py. Every shape is run once before it is timed; medians of
repeated calls, CUDA events; the card, power limit and SM clock are read in the same run.

    python scripts/nerf_mesh_bench.py [--mip] [--reps 10]
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

# MACs per point: pts_linears.0..7 (ic x 256 + 6 x 256x256 + (256 + ic) x 256) + alpha_linear; FULL adds feature_linear, views_linears.0, rgb_linear
MAC_DENSITY = {False: 491264, True: 508160}   # ic = 63 / 96
MAC_FULL = {False: 593408, True: 610304}


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


def nerf_meshes():
    """[(name, network, threshold)] of the plain mode"""
    from cases import NERF_MLP
    from test_gpu_nerf_mesh import _octahedron_network
    from xrnerf_b200.registry.networks import NerfNetwork
    octahedron = _octahedron_network()
    default = NerfNetwork(dict(N_importance=0, chunk=1024, bs_data='rays_o', is_perturb=False), mlp=NERF_MLP,
                          render=dict(type='NerfRender', white_bkgd=False, raw_noise_std=0)).cuda()
    return [('octahedron', octahedron, 1e-9), ('default_init', default, 1e-3)]


def mip_meshes():
    """[(name, network, threshold)] of --mip"""
    from cases import MIP_MLP
    from test_gpu_mip_mesh import RGB_PADDING, _sine_network
    from xrnerf_b200.registry.networks import MipNerfNetwork
    default = MipNerfNetwork(dict(phase='test', ray_shape='cone', resample_padding=0.01, use_multiscale=False, coarse_loss_mult=0.1, num_levels=2, chunk=800,
                                  bs_data='rays_o'),
                             mlp=MIP_MLP, render=dict(type='MipNerfRender', white_bkgd=True, raw_noise_std=0, rgb_padding=RGB_PADDING, density_bias=-1,
                                                      density_activation='softplus')).cuda()
    return [('sine', _sine_network(), math.log1p(math.exp(-1.0))), ('default_init', default, math.log1p(math.exp(-1.0 + 1e-3)))]


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--mip', action='store_true', help='Mip-NeRF at the cell footprint')
    ap.add_argument('--reps', type=int, default=10)
    args = ap.parse_args()
    assert torch.cuda.is_available(), 'needs a GPU'
    import test_gpu_mip_mesh as tm
    import test_gpu_nerf_mesh as tn
    from cases import MIP_MLP, NERF_MLP
    from restate64 import lattice_points, mip_bands
    from xrnerf_b200 import registry as R
    from xrnerf_b200.mesh import footprint_sigma
    mip = args.mip
    box = tm.BOX if mip else ((-1.5,) * 3, (1.5,) * 3)
    fp = dict(footprint='cell') if mip else {}
    out = {'card_before': card()}
    torch.manual_seed(0)
    mlp = R.build_mlp(MIP_MLP if mip else NERF_MLP).cuda()
    with torch.no_grad():
        for n in (256, 512):
            shape = (n, n, n)
            sigma = footprint_sigma('cell', shape, box)
            pts = lattice_points(shape, box)
            dirs = torch.nn.functional.normalize(torch.randn_like(pts), dim=-1)
            t_lat = timed(lambda: mlp.density_lattice(shape, box, **fp), args.reps)
            infer = (lambda p, d: tm._infer(mlp, p, d, sigma)) if mip else (lambda p, d: tn._infer(mlp, p, d))
            ch = 1 << 21
            t_cmp = timed(lambda: [infer(pts[i:i + ch], dirs[i:i + ch]) for i in range(0, pts.shape[0], ch)], args.reps)
            npt = n ** 3
            r = dict(sigma=sigma, live_bands=int((mip_bands(sigma) > 0).sum())) if mip else {}
            r.update({'density_lattice_ms': t_lat, 'encoder_plus_mlp_ms' if mip else 'posenc_plus_mlp_ms': t_cmp,
                      'lattice_tflops': 2 * MAC_DENSITY[mip] * npt / t_lat * 1e-9, 'comparison_tflops': 2 * MAC_FULL[mip] * npt / t_cmp * 1e-9})
            out[f'lattice_{n}'] = r
            del pts, dirs
        p = (torch.rand((1 << 20, 3), device='cuda') * 3 - 1.5).contiguous()
        grad_fp = dict(footprint=footprint_sigma('cell', (256,) * 3, box)) if mip else {}
        out['density_grad_2e20_ms'] = timed(lambda: mlp.density_grad(p, **grad_fp), args.reps)
    for name, net, thr in (mip_meshes() if mip else nerf_meshes()):
        v, f = net.extract_mesh(256, thr, **fp)
        out[f'mesh_{name}_256'] = dict(V=int(v.shape[0]), F=int(f.shape[0]), extract_mesh_ms=timed(lambda: net.extract_mesh(256, thr, **fp), 3),
                                       extract_colored_mesh_ms=timed(lambda: net.extract_colored_mesh(256, thr, **fp), 3))
    out['card_after'] = card()
    print(json.dumps(out))


if __name__ == '__main__':
    main()
