"""Depth and opacity supervision: the cost of the geometry terms in a training step.

  NGP: NgpTrainer.step at the bench shape (65 536 rays, T = 2^20, synthetic lego-like scene) with depth_weight = opacity_weight = 0 and with both > 0
       (composite forward with depth and alpha, the geometry loss, the geometry backward).
  NeRF / Mip-NeRF: a 4096-ray train_step + backward of the Blender configs with and without depth_loss_weight / opacity_loss_weight.

Medians of alternated runs, timed with CUDA events; the card name, power limit and SM clock are read in the same run (never set).

    python scripts/geom_supervision_bench.py [--reps 7] [--steps 20]
"""
import argparse
import json
import os
import subprocess
import sys

import numpy as np
import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), 'tests'))


def card():
    try:
        q = subprocess.run(['nvidia-smi', '--query-gpu=name,power.limit,clocks.sm,clocks.max.sm', '--format=csv,noheader'], capture_output=True, text=True, timeout=30).stdout
        return q.strip().splitlines()[0]
    except Exception as e:   # noqa: BLE001
        return f'unknown ({e})'


def timed(fn, steps):
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    a.record()
    for _ in range(steps):
        fn()
    b.record(); b.synchronize()
    return a.elapsed_time(b) / steps


def ngp(reps, steps):
    from xrnerf_b200 import synth
    from xrnerf_b200.ngp import NgpField
    from xrnerf_b200.train import NgpTrainer
    table, dens, color = synth.ngp_weights(seed=3, hash_range=0.5, mlp_gain=2.0)
    bf = torch.from_numpy(synth.bitfield_from_grid_numpy(synth.lego_like_density_grid(0))[0]).cuda()
    n = 65536
    o, d, _, _ = synth.ray_batch(n, seed=1)
    o, d = torch.from_numpy(o).cuda(), torch.from_numpy(d).cuda()
    tgt, bg = torch.rand((n, 3), device='cuda'), torch.zeros((n, 3), device='cuda')
    td, ta = torch.rand(n, device='cuda') + 0.5, torch.rand(n, device='cuda')
    trainers = {}
    for name, kw, step_kw in (('colour only', {}, {}), ('colour + depth + opacity', dict(depth_weight=1.0, opacity_weight=1.0), dict(target_depth=td, target_alpha=ta))):
        f = NgpField().cuda()
        with torch.no_grad():
            f.hash_params.copy_(torch.from_numpy(table)); f.density_params.copy_(torch.from_numpy(dens)); f.color_params.copy_(torch.from_numpy(color))
        tr = NgpTrainer(f, bf, n, target_batch_size=1 << 20, lr=0.0, **kw)
        for _ in range(3):
            tr.step(o, d, tgt, bg, next_rays=(o, d), **step_kw)
        trainers[name] = (tr, step_kw)
    ms = {k: [] for k in trainers}
    for _ in range(reps):
        for k, (tr, step_kw) in trainers.items():
            ms[k].append(timed(lambda: tr.step(o, d, tgt, bg, next_rays=(o, d), **step_kw), steps))
    return {k: float(np.median(v)) for k, v in ms.items()}


def nerf(kind, reps):
    from xrnerf_b200 import registry as R
    from cases import MIP_MLP, NERF_MLP, view_rays
    n = 4096
    o, d, v, r = view_rays(64, 64, seed=1)
    tgt = torch.rand((1, n, 3), device='cuda')
    out = {}
    for name, w in (('colour only', 0.0), ('colour + depth + opacity', 1.0)):
        torch.manual_seed(0)
        if kind == 'nerf':
            net = R.build_network(dict(type='NerfNetwork', cfg=dict(phase='train', N_importance=128, is_perturb=False, chunk=1024 * 32, bs_data='rays_o', depth_loss_weight=w,
                                                                    opacity_loss_weight=w), mlp=NERF_MLP, mlp_fine=NERF_MLP,
                                       render=dict(type='NerfRender', white_bkgd=True, raw_noise_std=0))).cuda()
            t = torch.linspace(0., 1., 64, device='cuda')
            z = (2.0 * (1. - t) + 6.0 * t).expand(n, 64).contiguous()
            data = {'rays_o': o[None], 'rays_d': d[None], 'viewdirs': v[None], 'z_vals': z[None], 'pts': (o[:, None, :] + d[:, None, :] * z[:, :, None])[None], 'target_s': tgt}
        else:
            net = R.build_network(dict(type='MipNerfNetwork', cfg=dict(phase='train', ray_shape='cone', resample_padding=0.01, use_multiscale=False, coarse_loss_mult=0.1,
                                                                       num_levels=2, chunk=1024 * 32, bs_data='rays_o', depth_loss_weight=w, opacity_loss_weight=w), mlp=MIP_MLP,
                                       render=dict(type='MipNerfRender', white_bkgd=True, raw_noise_std=0, rgb_padding=0.001, density_bias=-1,
                                                   density_activation='softplus'))).cuda()
            t = torch.linspace(0., 1., 129, device='cuda')
            z = (2.0 * (1. - t) + 6.0 * t).expand(n, 129).contiguous()
            data = {'rays_o': o[None], 'rays_d': d[None], 'viewdirs': v[None], 'radii': r[None], 'z_vals': z[None], 'target_s': tgt}
        data['target_depth'] = torch.rand((1, n, 1), device='cuda') + 3.0
        data['target_alpha'] = torch.ones((1, n, 1), device='cuda')
        opt = torch.optim.Adam(net.parameters(), lr=0.0)

        def step():
            res = net.train_step(dict(data), opt)
            opt.zero_grad(set_to_none=True)
            res['loss'].backward()
        for _ in range(2):
            step()
        out[name] = float(np.median([timed(step, 3) for _ in range(reps)]))
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--reps', type=int, default=7)
    ap.add_argument('--steps', type=int, default=20)
    args = ap.parse_args()
    assert torch.cuda.is_available(), 'this benchmark needs a CUDA device'
    res = {'card': card(), 'ngp_step_ms (65536 rays, T = 2^20)': ngp(args.reps, args.steps)}
    for kind in ('nerf', 'mip'):
        res[f'{kind}_train_step_ms (4096 rays, fwd + bwd)'] = nerf(kind, args.reps)
    print(json.dumps(res, indent=1))


if __name__ == '__main__':
    main()
