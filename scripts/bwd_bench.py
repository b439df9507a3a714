"""Isolated timing of the NGP field backward (wgmma) on the samples of one 65 536-ray batch.  python scripts/bwd_bench.py [n_packed]"""
import os
import sys
import numpy as np
import torch
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from xrnerf_b200 import synth
from xrnerf_b200.ngp import NgpField
import xrnerf_b200.raymarch_cuda as rm

dev = torch.device('cuda')
N = 65536
bf = torch.from_numpy(synth.bitfield_from_grid_numpy(synth.lego_like_density_grid(0))[0]).to(dev)
o, d = (torch.from_numpy(x).to(dev) for x in synth.ray_batch(N, seed=0)[:2])
cap = N * 64
coords = torch.zeros((cap, 7), device=dev); ridx = torch.zeros((N, 1), dtype=torch.int32, device=dev); ns = torch.zeros((N, 2), dtype=torch.int32, device=dev); cnt = torch.zeros(2, dtype=torch.int32, device=dev)
rm.rays_sampler_api(o, d, bf, None, None, None, 0.0, 1.0, 0.05, 1.0 / 256, coords, ridx, ns, cnt)
S = int(cnt[1].item())
c = coords[:S]
f = NgpField(n_packed_levels=int(sys.argv[1]) if len(sys.argv) > 1 else 6).to(dev)
f.refresh()
draw = torch.randn((S, 4), device=dev) * 1e-3
out = (torch.zeros_like(f.hash_params), torch.zeros_like(f.density_params), torch.zeros_like(f.color_params))
flush = torch.empty(256 << 20, dtype=torch.uint8, device=dev)
ts = []
for i in range(8):
    flush.zero_()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record(); f.backward_params(c[:, :3], c[:, 4:], draw, out=out, impl=int(os.environ.get('BWD_IMPL', '1'))); e1.record(); torch.cuda.synchronize()
    if i >= 2:
        ts.append(e0.elapsed_time(e1) * 1e3)
print('field backward impl=%s: %d samples, median %.1f us min %.1f us' % (os.environ.get('BWD_IMPL', '1'), S, np.median(ts), min(ts)), flush=True)
