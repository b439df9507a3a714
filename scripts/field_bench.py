"""Isolated timings of the NGP chain's kernels on one 65 536-ray batch (CUDA events, L2 flushed between repetitions):
march (count+scan+emit), field (per gather plan), composite, and the single-launch kernel; then, per kernel (torch.profiler), the cost of
ordering the samples by position against the field on the same samples in ray order and in bucket order.
python scripts/field_bench.py [n_packed ...]"""
import os
import sys
import numpy as np
import torch
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from xrnerf_b200 import synth, _C
from xrnerf_b200.ngp import NgpField, NgpRenderer
import xrnerf_b200.raymarch_cuda as rm

dev = torch.device('cuda')
N = 65536
grid = synth.lego_like_density_grid(0)
bf_np, _ = synth.bitfield_from_grid_numpy(grid)
if os.environ.get('XRB_ALL_ONES'):
    bf_np = np.full_like(bf_np, 255)
bf = torch.from_numpy(bf_np).to(dev)
batches = [tuple(torch.from_numpy(x).to(dev) for x in synth.ray_batch(N, seed=b)[:2]) for b in range(8)]
table, dens, color = synth.ngp_weights(seed=0)
flush = torch.empty(256 << 20, dtype=torch.uint8, device=dev)
budget = 1024 if os.environ.get('XRB_ALL_ONES') else 64


def timed(fn, reps=10):
    ts = []
    for i in range(reps + 2):
        flush.zero_()
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record(); fn(i); e1.record(); torch.cuda.synchronize()
        if i >= 2:
            ts.append(e0.elapsed_time(e1) * 1e3)
    return float(np.median(ts)), float(np.min(ts))


cap = N * budget
coords = torch.zeros((cap, 7), device=dev); ridx = torch.zeros((N, 1), dtype=torch.int32, device=dev); ns = torch.zeros((N, 2), dtype=torch.int32, device=dev); cnt = torch.zeros(2, dtype=torch.int32, device=dev)


def march(i):
    cnt.zero_()
    o, d = batches[i % 8]
    rm.rays_sampler_api(o, d, bf, None, None, None, 0.0, 1.0, 0.05, 1.0 / 256, coords, ridx, ns, cnt)


print('march (memset + count + scan + emit) us: median %.1f min %.1f' % timed(march))
march(0); torch.cuda.synchronize()
S = int(cnt[1].item())
print('samples', S, 'per ray', S / N)
plans = [int(a) for a in sys.argv[1:]] or [0, 6, 7]
for npk in plans:
    f = NgpField(n_packed_levels=npk).to(dev)
    with torch.no_grad():
        f.hash_params.copy_(torch.from_numpy(table).to(dev)); f.density_params.copy_(torch.from_numpy(dens).to(dev)); f.color_params.copy_(torch.from_numpy(color).to(dev))
    f.refresh()
    torch.cuda.synchronize()
    print('n_packed=%d: cell image %.2f GB' % (npk, (f._cells.numel() if f._cells is not None else 0) / 1e9), flush=True)
    c = coords[:S]
    med, mn = timed(lambda i: f.run_mlp(c[:, :3], c[:, 4:]))
    print('field n_packed=%d: median %.1f us min %.1f us -> %.0f GB/s algorithmic (556 B/sample)' % (npk, med, mn, S * 556 / med / 1e3), flush=True)
    if os.environ.get('XRB_FIELD_ONLY'):
        continue
    med, mn = timed(lambda i: f.rebuild_cells())
    print('   cell image rebuild: %.1f us' % med)
    r = NgpRenderer(f, samples_per_ray_budget=budget)
    med, mn = timed(lambda i: r.render_fused(*batches[i % 8], bf))
    print('   fused single launch: median %.1f us min %.1f us' % (med, mn))
    med, mn = timed(lambda i: r.render(*batches[i % 8], bf))
    print('   chain (sequential launches): median %.1f us min %.1f us' % (med, mn))
    if npk != plans[-1]:
        continue
    # the same samples (same RNG call index) through the field in ray order (run_mlp on the march's rows) and inside the chain (bucket order)
    def per_kernel(fn, reps=10):
        from torch.profiler import profile, ProfilerActivity
        for i in range(2):
            fn(i)
        torch.cuda.synchronize()
        with profile(activities=[ProfilerActivity.CUDA]) as prof:
            for i in range(reps):
                flush.zero_()
                fn(i)
            torch.cuda.synchronize()
        return {e.key: e.device_time_total / reps for e in prof.key_averages() if e.device_time_total > 0}

    def ray_order(i):
        rm.reset_rng(ray_sampler=i)
        march(i)
        flush.zero_()
        n = min(int(cnt[1].item()), cap)
        f.run_mlp(coords[:n, :3], coords[:n, 4:])

    def bucket_order(i):
        r.calls = i
        r.render(*batches[i % 8], bf)

    name = lambda k, sub: [v for key, v in k.items() if sub in key]
    ka, kb = per_kernel(ray_order), per_kernel(bucket_order)
    print('   per kernel, us per batch (torch.profiler, L2 flushed before each batch):')
    for label, sub in (('memset (bucket counts, counters)', 'Memset'), ('order_key_kernel', 'order_key_kernel'), ('order_chunk_sum_kernel', 'order_chunk_sum_kernel'),
                       ('order_scan_kernel', 'order_scan_kernel'), ('order_scatter_kernel', 'order_scatter_kernel')):
        print('      %-34s %7.1f' % (label, sum(name(kb, sub))))
    order_us = sum(sum(name(kb, sub)) for sub in ('order_key_kernel', 'order_chunk_sum_kernel', 'order_scan_kernel', 'order_scatter_kernel'))
    fa, fb = sum(name(ka, 'ngp_field_tc_kernel')), sum(name(kb, 'ngp_field_tc_kernel'))
    print('      ordering kernels total              %7.1f' % order_us)
    print('      field, ray order                    %7.1f' % fa)
    print('      field, bucket order                 %7.1f  (ordering + field %.1f, %.2fx the ray-order field)' % (fb, order_us + fb, fa / (order_us + fb)))
