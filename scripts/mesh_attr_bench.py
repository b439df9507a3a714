"""Cost of the mesh attributes: the field's density gradient (xrb_ngp_density_grad, NgpField.density_grad) and HashNerfNetwork.extract_colored_mesh.

  - density_grad next to run_density with impl 0 (CUDA cores) and impl 1 (wgmma) on the same points: (a) the vertices of the synthetic field's mesh at
    256^3 (its 70th-percentile level set) and (b) 2^20 uniform random points;
  - extract_colored_mesh next to extract_mesh at 256^3 on the same network.
Times are medians over `--reps` calls between CUDA events after `--warmup` calls, on one stream. The card's name, power limit and SM clock are read
with nvidia-smi in the same run.

    python scripts/mesh_attr_bench.py [--reps 20] [--warmup 3] [--json out.json]
"""
import argparse
import json
import math
import os
import subprocess
import sys

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from xrnerf_b200 import registry as R, synth  # noqa: E402
from xrnerf_b200.mesh import marching_cubes  # noqa: E402

MODEL = dict(   # configs/instant_ngp/nerf_blender_local01.py's model
    type='HashNerfNetwork', cfg=dict(phase='train', chunk=4096, bs_data='rays_o'),
    mlp=dict(type='HashNerfMLP', bound=1,
             embedder_pos=dict(n_input_dims=3, encoding_config=dict(otype='HashGrid', n_levels=16, n_features_per_level=2, log2_hashmap_size=19, base_resolution=16, interpolation='Linear')),
             embedder_dir=dict(n_input_dims=3, encoding_config=dict(otype='SphericalHarmonics', degree=4)),
             density_net=dict(n_input_dims=32, n_output_dims=16, network_config=dict(otype='FullyFusedMLP', activation='ReLU', output_activation='None', n_neurons=64, num_layers=1)),
             color_net=dict(n_output_dims=3, network_config=dict(otype='FullyFusedMLP', activation='ReLU', output_activation='None', n_neurons=64, num_layers=2))),
    sampler=dict(type='NGPGridSampler', update_grid_freq=16, update_block_size=5000000, n_rays_per_batch=4096, cone_angle_constant=0.00390625, near_distance=0.2,
                 target_batch_size=1 << 18, rgb_activation=2, density_activation=3),
    render=dict(type='HashNerfRender', bg_color=[0, 0, 0]))


def gpu_info():
    q = 'name,power.limit,clocks.sm,clocks.max.sm'
    out = subprocess.run(['nvidia-smi', f'--query-gpu={q}', '--format=csv,noheader', '-i', str(torch.cuda.current_device())], capture_output=True, text=True)
    return dict(zip(q.split(','), (v.strip() for v in out.stdout.strip().split(','))))


def time_ms(fn, reps, warmup):
    for _ in range(warmup):
        fn()
    ts = []
    for _ in range(reps):
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        a.record(); fn(); b.record()
        b.synchronize()
        ts.append(a.elapsed_time(b))
    return sorted(ts)[len(ts) // 2]


def point_case(field, pts, reps, warmup):
    return {'n': int(pts.shape[0]),
            'density_grad_ms': round(time_ms(lambda: field.density_grad(pts), reps, warmup), 4),
            'run_density_impl0_ms': round(time_ms(lambda: field.run_density(pts, impl=0), reps, warmup), 4),
            'run_density_impl1_ms': round(time_ms(lambda: field.run_density(pts, impl=1), reps, warmup), 4)}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--reps', type=int, default=20)
    ap.add_argument('--warmup', type=int, default=3)
    ap.add_argument('--json', default=None)
    a = ap.parse_args()
    assert torch.cuda.is_available(), 'mesh_attr_bench.py measures on the GPU'
    torch.cuda.set_device(0)
    net = R.build_network(MODEL).cuda()
    field = net.mlp.field
    table, dens, color = synth.ngp_weights(seed=3, hash_range=0.5, mlp_gain=2.0)
    with torch.no_grad():
        for p, v in ((field.hash_params, table), (field.density_params, dens), (field.color_params, color)):
            p.copy_(torch.from_numpy(v).cuda())
    result = {'gpu': gpu_info()}
    n = 256
    lat = field.density_lattice((n, n, n))
    raw = float(torch.quantile(lat.reshape(-1)[::97].float(), 0.7))
    verts, _ = marching_cubes(lat, raw)
    del lat
    result['mesh_vertices_256'] = point_case(field, verts, a.reps, a.warmup)
    pts = torch.rand((1 << 20, 3), generator=torch.Generator(device='cuda').manual_seed(7), device='cuda')
    result['random_2^20'] = point_case(field, pts, a.reps, a.warmup)
    sigma = math.exp(raw)   # the sampler's density activation is exponential
    result['extract_256'] = {'threshold_raw': round(raw, 4), 'V': int(verts.shape[0]),
                             'extract_mesh_ms': round(time_ms(lambda: net.extract_mesh(n, sigma), a.reps, a.warmup), 3),
                             'extract_colored_mesh_ms': round(time_ms(lambda: net.extract_colored_mesh(n, sigma), a.reps, a.warmup), 3)}
    result['gpu_after'] = gpu_info()
    print(json.dumps(result))
    if a.json:
        with open(a.json, 'w') as fh:
            json.dump(result, fh, indent=1)


if __name__ == '__main__':
    main()
