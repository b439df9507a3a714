"""Cost of the NGP mesh export: the field's density on a lattice (xrb_ngp_density_lattice) and marching cubes (xrb_mc_count, xrb_mc_emit).

At 256^3 and 512^3:
  - the density lattice, next to run_density on a position tensor holding the same points (the way to get the volume without the lattice entry);
  - xrb_mc_count (count + block-sum scan) and xrb_mc_emit, each on its own, on an analytic volume (a sphere plus smooth noise) and on the lattice
    of a synth.ngp_weights field at its 70th percentile;
  - V and F, and the marching-cubes bytes (volume read by each pass, the per-point word written and read, the mesh written) over kernel time, as a
    share of the H100 SXM's 3.35 TB/s HBM3.
Times are medians over `--reps` launches between CUDA events after `--warmup` launches, on one stream. The card's name, power limit and SM clock
are read with nvidia-smi in the same run.

    python scripts/mesh_bench.py [--reps 20] [--warmup 3] [--json out.json]
"""
import argparse
import json
import os
import subprocess
import sys

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from xrnerf_b200 import _C, synth  # noqa: E402
from xrnerf_b200.ngp import NgpField  # noqa: E402

HBM_BYTES_PER_S = 3.35e12


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


def analytic_volume(n):
    """sphere of radius 0.3 plus smooth noise, on the GPU"""
    g = torch.linspace(0, 1, n, device='cuda')
    z, y, x = torch.meshgrid(g, g, g, indexing='ij')
    r = torch.sqrt((x - 0.5) ** 2 + (y - 0.5) ** 2 + (z - 0.5) ** 2)
    return (0.3 - r + 0.03 * torch.sin(17 * x) * torch.sin(13 * y + 1) * torch.sin(11 * z + 2)).contiguous()


def mc_case(vol, thr, reps, warmup):
    nz, ny, nx = vol.shape
    lib, s = _C.lib, _C.stream()
    ws = torch.empty(lib.xrb_mc_workspace(nx, ny, nz), dtype=torch.uint8, device='cuda')
    counts = torch.zeros(2, dtype=torch.int32, device='cuda')
    box0, box1 = _C.float3((0, 0, 0)), _C.float3((1, 1, 1))
    count = lambda: _C.check(lib.xrb_mc_count(_C.f32(vol), nx, ny, nz, float(thr), _C.ptr(ws), _C.i32(counts), s), 'mc_count')
    count()
    V, F = (int(v) for v in counts.tolist())
    verts = torch.empty((V, 3), dtype=torch.float32, device='cuda')
    faces = torch.empty((F, 3), dtype=torch.int32, device='cuda')
    emit = lambda: _C.check(lib.xrb_mc_emit(_C.f32(vol), nx, ny, nz, float(thr), box0, box1, _C.ptr(ws), _C.f32(verts), _C.i32(faces), s), 'mc_emit')
    t_count, t_emit = time_ms(count, reps, warmup), time_ms(emit, reps, warmup)
    n = vol.numel()
    bytes_count = 4 * n + 4 * n               # volume read, point word written (the block sums are O(n / 256))
    bytes_emit = 4 * n + 4 * n + 12 * V + 12 * F
    total_ms = t_count + t_emit
    return {'V': V, 'F': F, 'count_ms': round(t_count, 4), 'emit_ms': round(t_emit, 4), 'bytes': bytes_count + bytes_emit,
            'GB_per_s': round((bytes_count + bytes_emit) / (total_ms * 1e-3) / 1e9, 1),
            'hbm_share': round((bytes_count + bytes_emit) / (total_ms * 1e-3) / HBM_BYTES_PER_S, 3)}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--reps', type=int, default=20)
    ap.add_argument('--warmup', type=int, default=3)
    ap.add_argument('--json', default=None)
    a = ap.parse_args()
    assert torch.cuda.is_available(), 'mesh_bench.py measures on the GPU'
    torch.cuda.set_device(0)
    field = NgpField().cuda()
    table, dens, color = synth.ngp_weights(seed=3, hash_range=0.5, mlp_gain=2.0)
    with torch.no_grad():
        for p, v in ((field.hash_params, table), (field.density_params, dens), (field.color_params, color)):
            p.copy_(torch.from_numpy(v).cuda())
    result = {'gpu': gpu_info(), 'sizes': {}}
    for n in (256, 512):
        r = {}
        r['density_lattice_ms'] = round(time_ms(lambda: field.density_lattice((n, n, n)), a.reps, a.warmup), 3)
        g = torch.linspace(0, 1, n, device='cuda')
        z, y, x = torch.meshgrid(g, g, g, indexing='ij')
        pts = torch.stack([x.reshape(-1), y.reshape(-1), z.reshape(-1)], 1).contiguous()
        del x, y, z
        r['run_density_ms'] = round(time_ms(lambda: field.run_density(pts), a.reps, a.warmup), 3)
        del pts
        vol = analytic_volume(n)
        r['mc_analytic'] = mc_case(vol, 0.0, a.reps, a.warmup)
        del vol
        lat = field.density_lattice((n, n, n))
        thr = float(torch.quantile(lat.reshape(-1)[::97].float(), 0.7))
        r['mc_field'] = dict(threshold=round(thr, 4), **mc_case(lat, thr, a.reps, a.warmup))
        del lat
        torch.cuda.empty_cache()
        result['sizes'][f'{n}^3'] = r
        print(json.dumps({f'{n}^3': r}), flush=True)
    result['gpu_after'] = gpu_info()
    print(json.dumps(result))
    if a.json:
        with open(a.json, 'w') as fh:
            json.dump(result, fh, indent=1)


if __name__ == '__main__':
    main()
