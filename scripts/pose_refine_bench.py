"""NGP camera pose refinement: the cost of the ray gradients and the pose update in a training step.

NgpTrainer.step at the bench shape (65 536 rays, T = 2^20, synthetic lego-like scene, rays of the 40 spiral 800 x 800 views drawn by NgpRaySource) without
ray_grad, and with ray_grad=True followed by NgpRaySource.pose_step (the field backward's INPUTS variant, the per-ray reduction, the per-image reduction, the
Exp-map autograd and the Adam step on the corrections). Also the field backward alone, with and without d_rows, on the same compacted rows.

Medians of alternated runs, timed with CUDA events; the card name, power limit and SM clock are read in the same run (never set).

    python scripts/pose_refine_bench.py [--reps 7] [--steps 20]
"""
import argparse
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


def timed(fn, steps):
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    a.record()
    for _ in range(steps):
        fn()
    b.record(); b.synchronize()
    return a.elapsed_time(b) / steps


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--reps', type=int, default=7)
    ap.add_argument('--steps', type=int, default=20)
    args = ap.parse_args()
    assert torch.cuda.is_available(), 'this benchmark needs a CUDA device'
    from xrnerf_b200 import synth
    from xrnerf_b200.data import NgpRaySource
    from xrnerf_b200.ngp import NgpField
    from xrnerf_b200.train import NgpTrainer
    table, dens, color = synth.ngp_weights(seed=3, hash_range=0.5, mlp_gain=2.0)
    bf = torch.from_numpy(synth.bitfield_from_grid_numpy(synth.lego_like_density_grid(0))[0]).cuda()
    n = 65536
    poses = synth.spiral_poses_ngp(40)
    K = [[synth.FOCAL, 0, 0.5 * synth.W], [0, synth.FOCAL, 0.5 * synth.H], [0, 0, 1]]
    src = NgpRaySource(poses, torch.rand(40, synth.H, synth.W, 4), K, refine_poses=True).cuda()
    batch = src.next_batch(n)
    o, d, tgt = batch['rays_o'], batch['rays_d'], batch['target_s']
    bg = torch.zeros((n, 3), device='cuda')
    trainers = {}
    for name, rg in (('step', False), ('step + ray_grad + pose_step', True)):
        f = NgpField().cuda()
        with torch.no_grad():
            f.hash_params.copy_(torch.from_numpy(table)); f.density_params.copy_(torch.from_numpy(dens)); f.color_params.copy_(torch.from_numpy(color))
        tr = NgpTrainer(f, bf, n, target_batch_size=1 << 20, lr=0.0, ray_grad=rg)

        def step(tr=tr, rg=rg):
            tr.step(o, d, tgt, bg, next_rays=(o, d))
            if rg:
                src.pose_step(batch, tr.grad_rays_o, tr.grad_rays_d)
        for _ in range(3):
            step()
        trainers[name] = (tr, step)
    ms = {k: [] for k in trainers}
    for _ in range(args.reps):
        for k, (_, step) in trainers.items():
            ms[k].append(timed(step, args.steps))
    res = {'card': card(), 'ngp_step_ms (65536 rays, T = 2^20)': {k: float(np.median(v)) for k, v in ms.items()}}
    # the field backward alone on the last step's compacted rows
    tr = trainers['step + ray_grad + pose_step'][0]
    torch.cuda.synchronize()
    s = tr.slots[tr.cur ^ 1]
    pts, dirs, n_dev = s.coords_c[:, :3], s.coords_c[:, 4:], s.cnt_c[1:2]
    bw = {'backward_rows': lambda: tr.f.backward_rows(pts, dirs, tr.draw, tr.grads, n_dev, 1),
          'backward_rows + d_rows': lambda: tr.f.backward_rows(pts, dirs, tr.draw, tr.grads, n_dev, 1, d_rows=tr.d_rows)}
    for fn in bw.values():
        fn()
    bms = {k: [] for k in bw}
    for _ in range(args.reps):
        for k, fn in bw.items():
            bms[k].append(timed(fn, args.steps))
    res['field_backward_ms (compacted rows: %d)' % int(s.cnt_c[1])] = {k: float(np.median(v)) for k, v in bms.items()}
    print(json.dumps(res, indent=1))


if __name__ == '__main__':
    main()
