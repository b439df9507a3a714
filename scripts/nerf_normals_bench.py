"""NeRF / Mip-NeRF normal maps: val_step on one 800x800 Blender-intrinsics view with and without render_normals, and the tensor-core density gradient
(xrb_nerf_density_grad_rays / xrb_mip_density_grad_rays) against the training kernels' nerf_train.density_grad on the same rows. Medians of
alternated calls, timed with CUDA events; the card name, power limit and SM clock are read before and after the run (never set). Untrained
default-initialised weights. Both gradient paths are timed from positions: grad_tc_ms includes the ray encoder that forms the encoding image
(nerf_train.density_grad encodes its points itself); grad_kernel_ms is the gradient kernel alone on that image.

    python scripts/nerf_normals_bench.py [--mip] [--reps 7] [--grad-reps 21] [--rows 1048576]
"""
import argparse
import ctypes as C
import json
import os
import subprocess
import sys

import numpy as np
import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))


def card():
    try:
        q = subprocess.run(['nvidia-smi', '--query-gpu=name,power.limit,clocks.sm,clocks.max.sm', '--format=csv,noheader'], capture_output=True, text=True, timeout=30).stdout
        return q.strip().splitlines()[0]
    except Exception as e:   # noqa: BLE001
        return f'unknown ({e})'


def timed(fn):
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    a.record(); fn(); b.record(); b.synchronize()
    return a.elapsed_time(b)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--mip', action='store_true')
    ap.add_argument('--reps', type=int, default=7, help='alternated val_step pairs')
    ap.add_argument('--grad-reps', type=int, default=21, help='alternated gradient calls per path')
    ap.add_argument('--rows', type=int, default=1 << 20, help='rows of the gradient comparison')
    args = ap.parse_args()
    from xrnerf_b200 import _C, nerf_train, synth
    from xrnerf_b200 import registry as R
    from xrnerf_b200.nerf import density_grad_rays, encode_rays
    before = card()
    torch.manual_seed(0)
    emb = dict(type='MipNerfEmbedder', min_deg_point=0, max_deg_point=16, min_deg_view=0, max_deg_view=4, use_viewdirs=True, append_identity=True) if args.mip \
        else dict(type='BaseEmbedder', i_embed=0, multires=10, multires_dirs=4)
    mlp = dict(type='NerfMLP', skips=[4], netdepth=8, netwidth=256, netchunk=1024 * 32, output_ch=5, use_viewdirs=True, embedder=emb)
    if args.mip:
        model = dict(type='MipNerfNetwork', cfg=dict(phase='train', ray_shape='cone', resample_padding=0.01, use_multiscale=False, coarse_loss_mult=0.1, num_levels=2,
                                                     chunk=800, bs_data='rays_o'), mlp=mlp,
                     render=dict(type='MipNerfRender', white_bkgd=True, raw_noise_std=0, rgb_padding=0.001, density_bias=-1, density_activation='softplus'))
    else:
        model = dict(type='NerfNetwork', cfg=dict(phase='train', N_importance=128, is_perturb=False, chunk=1024 * 32, bs_data='rays_o'), mlp=mlp, mlp_fine=mlp,
                     render=dict(type='NerfRender', white_bkgd=True, raw_noise_std=0))
    net = R.build_network(model).cuda()
    H = W = 800
    n = H * W
    pose = synth.pose_spherical(30.0, -30.0, 4.0)
    c2w = (C.c_float * 12)(*[float(v) for v in pose[:3, :4].reshape(-1)])
    o, d, v = (torch.empty((n, 3), device='cuda') for _ in range(3))
    r = torch.empty((n, 1), device='cuda')
    _C.check(_C.lib.xrb_nerf_get_rays(c2w, H, W, float(synth.FOCAL), float(synth.FOCAL), W / 2.0, H / 2.0, 0, None, n, _C.ptr(o), _C.ptr(d), _C.ptr(v), _C.ptr(r), _C.stream()), 'get_rays')
    S = 129 if args.mip else 64
    t = torch.linspace(0., 1., S, device='cuda')
    z = (2.0 * (1 - t) + 6.0 * t)[None].expand(n, S).contiguous()
    view = {'rays_o': o, 'rays_d': d, 'viewdirs': v, 'z_vals': z, 'src_shape': torch.tensor([H, W, 3])}
    if args.mip:
        view['radii'] = r
    net.set_val_pipeline(lambda item: dict(view))
    data = {'poses': torch.zeros((1, 1, 4, 4))}
    res = {'with': [], 'without': [], 'tc': [], 'kernel': [], 'train': []}

    def step(flag):
        net.render_normals = flag
        net.val_step(dict(data))
    step(False); step(True)
    for _ in range(args.reps):
        res['without'].append(timed(lambda: step(False)))
        res['with'].append(timed(lambda: step(True)))
    # the gradient on the same rows: rays with S' samples each, n' S' = rows
    m = net.mlp if args.mip else net.mlp_fine
    s2 = 64
    nr = args.rows // s2
    zz = (2.0 * (1 - torch.linspace(0., 1., s2 + (1 if args.mip else 0), device='cuda')) + 6.0 * torch.linspace(0., 1., s2 + (1 if args.mip else 0), device='cuda'))
    zz = zz[None].expand(nr, -1).contiguous()
    oo, dd, vv, rr = o[:nr].contiguous(), d[:nr].contiguous(), v[:nr].contiguous(), r[:nr].reshape(-1).contiguous()
    rad = rr if args.mip else None
    enc = encode_rays(m, oo, dd, vv, zz, rad)
    with torch.no_grad():
        tm = 0.5 * (zz[:, :-1] + zz[:, 1:]) if args.mip else zz          # the same number of rows; the training path takes points
        pts = (oo[:, None] + dd[:, None] * tm[..., None]).reshape(-1, 3).contiguous()
        run_tc = lambda: density_grad_rays(m, encode_rays(m, oo, dd, vv, zz, rad), oo, dd, zz, rad)
        run_k = lambda: density_grad_rays(m, enc, oo, dd, zz, rad)
        run_tr = lambda: nerf_train.density_grad(m, pts, sigma=0.0 if args.mip else None)
        run_tc(); run_k(); run_tr()
        for _ in range(args.grad_reps):
            res['tc'].append(timed(run_tc))
            res['kernel'].append(timed(run_k))
            res['train'].append(timed(run_tr))
    med = {k: float(np.median(x)) for k, x in res.items()}
    print(json.dumps({'mode': 'mip' if args.mip else 'nerf', 'view': f'{H}x{W}', 'val_step_ms': med['without'], 'val_step_normals_ms': med['with'],
                      'grad_rows': nr * s2, 'grad_tc_ms': med['tc'], 'grad_kernel_ms': med['kernel'], 'density_grad_train_ms': med['train'], 'speedup': med['train'] / med['tc'],
                      'card_before': before, 'card_after': card(), 'reps': args.reps, 'grad_reps': args.grad_reps}))


if __name__ == '__main__':
    main()
