"""NGP normal maps: the chain render with depth vs with normals, and the tensor-core density gradient (xrb_ngp_density_grad_tc) vs the CUDA-core one
(xrb_ngp_density_grad) on the same marched rows, in ray order and in bucketed order. Medians of alternated runs, timed with CUDA events; the card name,
power limit and SM clock are read in the same run (never set). --profile: one torch.profiler run instead, printing the time per kernel.

    python scripts/ngp_normals_bench.py [--reps 7] [--profile]
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


def timed(fn, reps):
    ts = []
    for _ in range(reps):
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        a.record(); fn(); b.record(); b.synchronize()
        ts.append(a.elapsed_time(b))
    return ts


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--reps', type=int, default=7)
    ap.add_argument('--profile', action='store_true')
    args = ap.parse_args()
    from xrnerf_b200 import _C, synth
    from xrnerf_b200.ngp import NgpField, NgpRenderer
    f = NgpField().cuda()
    table, dens, color = synth.ngp_weights(seed=3, hash_range=0.5, mlp_gain=2.0)
    with torch.no_grad():
        f.hash_params.copy_(torch.from_numpy(table)); f.density_params.copy_(torch.from_numpy(dens)); f.color_params.copy_(torch.from_numpy(color))
    bf = torch.from_numpy(synth.bitfield_from_grid_numpy(synth.lego_like_density_grid(0))[0]).cuda()
    o, d, _, poses = synth.ray_batch(65536, seed=1)
    vo, vd = synth.get_rays_ngp(poses[7])
    cases = {'bench batch 65536 rays': (torch.from_numpy(o).cuda(), torch.from_numpy(d).cuda(), 64),
             'one 800x800 view': (torch.from_numpy(np.ascontiguousarray(vo)).cuda(), torch.from_numpy(np.ascontiguousarray(vd)).cuda(), 64)}
    res = {'card': card()}
    prof = None
    if args.profile:
        prof = torch.profiler.profile(activities=[torch.profiler.ProfilerActivity.CUDA])
        prof.__enter__()
    for name, (ro, rd, budget) in cases.items():
        n = ro.shape[0]
        r = NgpRenderer(f, samples_per_ray_budget=budget)
        dp, nm = torch.empty(n, device='cuda'), torch.empty((n, 3), device='cuda')
        depth = lambda: r.render(ro, rd, bf, depth=dp)
        normals = lambda: r.render(ro, rd, bf, depth=dp, normals=nm)
        for fn in (depth, normals):
            fn(); fn()
        td, tn = [], []
        for _ in range(args.reps):
            td += timed(depth, 1); tn += timed(normals, 1)
        counters = r.render(ro, rd, bf, depth=dp, normals=nm)[3]
        rows = int(min(counters[1].item(), n * budget))
        res[name] = {'rays': n, 'rows': rows, 'render_depth_ms': float(np.median(td)), 'render_normals_ms': float(np.median(tn))}
        # the two gradient kernels on the same marched rows: ray order, and the chain's bucketed order (read back from its workspace)
        a256 = lambda b: (b + 255) // 256 * 256
        c0 = a256(_C.lib.xrb_rm_rays_sampler_workspace(n))
        ms = n * budget
        fl = r._ws[c0:c0 + ms * 12 * 4].view(torch.float32)
        coords = fl[:ms * 7].view(ms, 7)[:rows].clone()
        order = fl[ms * 11:ms * 12].view(torch.int32)[:rows].clone() if rows <= (1 << 21) else None
        pts = coords[:, :3]
        tc = lambda: f.density_grad_tc(pts, density=False)
        tco = (lambda: f.density_grad_tc(pts, density=False, order=order)) if order is not None else None
        cc = lambda: f.density_grad(pts)
        sorted_pts = pts[order.long()].contiguous() if order is not None else None
        ccs = (lambda: f.density_grad(sorted_pts)) if order is not None else None
        fns = [('grad_tc_ray_order_ms', tc), ('grad_cc_ray_order_ms', cc)] + ([('grad_tc_bucketed_ms', tco), ('grad_cc_bucketed_ms', ccs)] if order is not None else [])
        for _, fn in fns:
            fn()
        ts = {k: [] for k, _ in fns}
        for _ in range(args.reps):
            for k, fn in fns:
                ts[k] += timed(fn, 1)
        for k in ts:
            res[name][k] = float(np.median(ts[k]))
        torch.cuda.synchronize()
    if prof is not None:
        prof.__exit__(None, None, None)
        print(prof.key_averages().table(sort_by='cuda_time_total', row_limit=25))
    res['card_after'] = card()
    print(json.dumps(res))


if __name__ == '__main__':
    main()
