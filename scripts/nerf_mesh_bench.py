"""Times NeRF mesh export on one GPU: NerfMLP.density_lattice at 256^3 and 512^3 against posenc_tiles + nerf_mlp_forward on the same points (in
2^21-row chunks), NerfMLP.density_grad per 2^20 points, and NerfNetwork.extract_colored_mesh on the octahedron field of tests/test_gpu_nerf_mesh.py
and on a default-initialised network. Medians of repeated calls, CUDA events; the card, power limit and SM clock are read in the same run.

    python scripts/nerf_mesh_bench.py [--reps 10]
"""
import argparse
import json
import os
import subprocess
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, 'tests'))

MAC_DENSITY = 491264   # per point: pts_linears.0..7 (63x256 + 6 x 256x256 + 319x256) + alpha_linear
MAC_FULL = 593408      # the whole NerfMLP: + feature_linear, views_linears.0, rgb_linear


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
    from test_gpu_nerf_mesh import NERF_MLP, _infer, _lattice_points, _octahedron_network
    from xrnerf_b200 import registry as R
    from xrnerf_b200.registry.networks import NerfNetwork
    out = {'card_before': card()}
    torch.manual_seed(0)
    mlp = R.build_mlp(NERF_MLP).cuda()
    box = ((-1.5,) * 3, (1.5,) * 3)
    with torch.no_grad():
        for n in (256, 512):
            pts = _lattice_points((n, n, n), box)
            dirs = torch.nn.functional.normalize(torch.randn_like(pts), dim=-1)
            t_lat = timed(lambda: mlp.density_lattice((n, n, n), box), args.reps)
            ch = 1 << 21
            t_cmp = timed(lambda: [_infer(mlp, pts[i:i + ch], dirs[i:i + ch]) for i in range(0, pts.shape[0], ch)], args.reps)
            npt = n ** 3
            out[f'lattice_{n}'] = dict(density_lattice_ms=t_lat, posenc_plus_mlp_ms=t_cmp, lattice_tflops=2 * MAC_DENSITY * npt / t_lat * 1e-9,
                                       comparison_tflops=2 * MAC_FULL * npt / t_cmp * 1e-9)
            del pts, dirs
        p = (torch.rand((1 << 20, 3), device='cuda') * 3 - 1.5).contiguous()
        out['density_grad_2e20_ms'] = timed(lambda: mlp.density_grad(p), args.reps)
    for name, net in (('octahedron', _octahedron_network()),
                      ('default_init', NerfNetwork(dict(N_importance=0, chunk=1024, bs_data='rays_o', is_perturb=False), mlp=NERF_MLP,
                                                   render=dict(type='NerfRender', white_bkgd=False, raw_noise_std=0)).cuda())):
        thr = 1e-9 if name == 'octahedron' else 1e-3
        v, f = net.extract_mesh(256, thr)
        out[f'mesh_{name}_256'] = dict(V=int(v.shape[0]), F=int(f.shape[0]), extract_mesh_ms=timed(lambda: net.extract_mesh(256, thr), 3),
                                       extract_colored_mesh_ms=timed(lambda: net.extract_colored_mesh(256, thr), 3))
    out['card_after'] = card()
    print(json.dumps(out))


if __name__ == '__main__':
    main()
