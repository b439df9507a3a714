"""Cost of depth on the two NGP render paths: NgpRenderer.render (march -> sample order -> field -> composite chain) and render_fused (single-launch
kernel), each timed with depth off and on, alternating, with CUDA events, on one stream.

Shapes: the bench shape (65 536-ray batches from the synthetic 40-view scene over the lego-like occupancy grid, 32 distinct batches cycled so the
inputs exceed L2) and one whole 800x800 view (640 000 rays). A round times `--calls` back-to-back calls per (shape, path, depth) cell; the cells of a
round run in alternating order and the report gives the median over `--rounds` rounds, with the card's name, power limit and SM clock (sampled by
nvidia-smi during the timed rounds). Afterwards, in a separate torch.profiler pass, the chain's composite kernel alone (composite_fwd_kernel<1> without
depth, <2> with), since that is the only kernel of the chain that depth changes.

    python scripts/depth_bench.py [--rounds 7] [--calls 40] [--json out.json]
"""
import argparse
import json
import os
import subprocess
import sys
import threading

import numpy as np
import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from xrnerf_b200 import synth  # noqa: E402
from xrnerf_b200.ngp import NgpField, NgpRenderer  # noqa: E402

N_RAYS, N_BATCHES, BUDGET = 65536, 32, 64


def gpu_info():
    q = 'name,power.limit,clocks.max.sm'
    try:
        out = subprocess.run(['nvidia-smi', f'--query-gpu={q}', '--format=csv,noheader,nounits', '-i', str(torch.cuda.current_device())], capture_output=True, text=True,
                             timeout=30).stdout.strip().split(', ')
        return {'name': out[0], 'power_limit_w': float(out[1]), 'sm_max_mhz': float(out[2])}
    except Exception as e:   # noqa: BLE001
        return {'name': torch.cuda.get_device_name(), 'error': repr(e)[:120]}


class ClockSampler:
    """SM clock sampled every 200 ms by nvidia-smi while the timed rounds run"""

    def start(self):
        self.rows = []
        self.proc = subprocess.Popen(['nvidia-smi', '--query-gpu=clocks.sm', '--format=csv,noheader,nounits', '-lms', '200', '-i', str(torch.cuda.current_device())],
                                     stdout=subprocess.PIPE, stderr=subprocess.DEVNULL, text=True)
        self.t = threading.Thread(target=lambda: self.rows.extend(line.strip() for line in self.proc.stdout), daemon=True)
        self.t.start()

    def stop(self):
        self.proc.terminate()
        try:
            self.proc.wait(timeout=5)
        except subprocess.TimeoutExpired:
            self.proc.kill()
            self.proc.wait()
        self.t.join(timeout=5)
        mhz = [float(r) for r in self.rows if r.replace('.', '').isdigit()]
        return {'sm_mhz_median': float(np.median(mhz)) if mhz else None, 'sm_mhz_min': min(mhz) if mhz else None, 'samples': len(mhz)}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--rounds', type=int, default=7)
    ap.add_argument('--calls', type=int, default=40)
    ap.add_argument('--json', default=None)
    a = ap.parse_args()
    assert torch.cuda.is_available(), 'depth_bench measures on a CUDA device'
    dev = torch.device('cuda')
    bf_np, _ = synth.bitfield_from_grid_numpy(synth.lego_like_density_grid(0))
    bf = torch.from_numpy(bf_np).to(dev)
    table, dens, color = synth.ngp_weights(seed=0)
    field = NgpField().to(dev)
    with torch.no_grad():
        field.hash_params.copy_(torch.from_numpy(table)); field.density_params.copy_(torch.from_numpy(dens)); field.color_params.copy_(torch.from_numpy(color))
    batches = [tuple(torch.from_numpy(x).to(dev) for x in synth.ray_batch(N_RAYS, seed=b)[:2]) for b in range(N_BATCHES)]
    view = tuple(torch.from_numpy(x).to(dev) for x in synth.get_rays_ngp(synth.spiral_poses_ngp(40)[7]))
    shapes = {'batch65536': batches, 'view800x800': [view]}
    r = NgpRenderer(field, samples_per_ray_budget=BUDGET)
    depth_out = {k: torch.empty(v[0][0].shape[0], device=dev) for k, v in shapes.items()}

    def run(shape, path, depth, calls):
        fn = r.render_fused if path == 'fused' else r.render
        d_ = depth_out[shape] if depth else None
        bs = shapes[shape]
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        for i in range(calls):
            fn(*bs[i % len(bs)], bf, depth=d_)
        e1.record()
        e1.synchronize()
        return e0.elapsed_time(e1) * 1e3 / calls   # us per call

    cells = [(s, p, dp) for s in shapes for p in ('chain', 'fused') for dp in (False, True)]
    for c in cells:                                   # warm-up: modules, workspaces, output buffers of every cell
        run(*c, calls=4)
    torch.cuda.synchronize()
    times = {c: [] for c in cells}
    clk = ClockSampler()
    clk.start()
    try:
        for k in range(a.rounds):
            order = cells if k % 2 == 0 else [(s, p, not dp) for (s, p, dp) in cells]   # depth off first, then on first, alternately
            for c in order:
                times[c].append(run(*c, calls=a.calls))
    finally:
        clocks = clk.stop()
    res = {'gpu': gpu_info(), 'clocks_during_timing': clocks, 'rounds': a.rounds, 'calls_per_round': a.calls, 'results': []}
    for s in shapes:
        n = shapes[s][0][0].shape[0]
        for p in ('chain', 'fused'):
            off, on = float(np.median(times[(s, p, False)])), float(np.median(times[(s, p, True)]))
            res['results'].append({'shape': s, 'path': p, 'rays': n, 'us_per_call_depth_off': off, 'us_per_call_depth_on': on,
                                   'depth_cost_pct': 100.0 * (on - off) / off, 'mrays_per_s_off': n / off, 'mrays_per_s_on': n / on,
                                   'spread_off_us': [min(times[(s, p, False)]), max(times[(s, p, False)])],
                                   'spread_on_us': [min(times[(s, p, True)]), max(times[(s, p, True)])]})
    from torch.profiler import ProfilerActivity, profile
    res['chain_composite_kernel_us'] = {}
    for s in shapes:
        per = {}
        for dp in (False, True):
            with profile(activities=[ProfilerActivity.CUDA]) as prof:
                run(s, 'chain', dp, calls=20)
                torch.cuda.synchronize()
            per['on' if dp else 'off'] = sum(e.device_time_total for e in prof.key_averages() if 'composite_fwd_kernel' in e.key) / 20
        res['chain_composite_kernel_us'][s] = per
    for x in res['results']:
        print('%-12s %-6s off %9.1f us  on %9.1f us  cost %+5.1f %%  (off %.1f..%.1f, on %.1f..%.1f)' % (
            x['shape'], x['path'], x['us_per_call_depth_off'], x['us_per_call_depth_on'], x['depth_cost_pct'], *x['spread_off_us'], *x['spread_on_us']))
    for s, per in res['chain_composite_kernel_us'].items():
        print('%-12s chain composite kernel alone: off %.1f us  on %.1f us' % (s, per['off'], per['on']))
    print(json.dumps({'gpu': res['gpu'], 'clocks_during_timing': clocks}))
    if a.json:
        with open(a.json, 'w') as fh:
            json.dump(res, fh, indent=1)


if __name__ == '__main__':
    main()
