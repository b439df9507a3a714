"""A few fused NGP training steps (for ncu launch lists / quick timing).  python scripts/train_probe.py [steps] [n_packed]"""
import os
import sys
import torch
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from xrnerf_b200 import synth
from xrnerf_b200.ngp import NgpField
from xrnerf_b200.train import NgpTrainer

dev = torch.device('cuda')
N = 65536
K = int(sys.argv[1]) if len(sys.argv) > 1 else 6
bf = torch.from_numpy(synth.bitfield_from_grid_numpy(synth.lego_like_density_grid(0))[0]).to(dev)
NB = int(os.environ.get('NB', '4'))
batches = [tuple(torch.from_numpy(x).to(dev) for x in synth.ray_batch(N, seed=b)[:2]) for b in range(NB)]
f = NgpField(n_packed_levels=int(sys.argv[2]) if len(sys.argv) > 2 else 6).to(dev)
PRE = int(os.environ.get('PRE', '0'))
if PRE:
    from xrnerf_b200.ngp import NgpRenderer
    rs = [NgpRenderer(f, samples_per_ray_budget=64) for _ in range(4)]
    sts = [torch.cuda.Stream(device=dev) for _ in range(4)]
    for i in range(16):
        with torch.cuda.stream(sts[i % 4]):
            (rs[i % 4].render_fused if PRE >= 2 and i % 2 else rs[i % 4].render)(*batches[i % NB], bf)
    torch.cuda.synchronize()
    if PRE >= 3:
        from xrnerf_b200 import _C
        tbl = torch.empty(24_400_000 // 4, dtype=torch.int32, device=dev).random_(); sink = torch.zeros(4, dtype=torch.int32, device=dev); nl = _C.C.c_int64(0)
        for _ in range(7):
            _C.check(_C.lib.xrb_micro_gather(_C.ptr(tbl), tbl.numel(), 4, 64, _C.C.byref(nl), _C.ptr(sink), _C.stream()))
        torch.cuda.synchronize()
    if PRE >= 4:
        hb = [tuple(t.cpu().pin_memory() for t in batches[i]) for i in range(4)]
        od = torch.empty((N, 3), device=dev); rh = torch.empty((N, 3)).pin_memory()
        for i in range(8):
            with torch.cuda.stream(sts[i % 4]):
                od.copy_(hb[i % 4][0], non_blocking=True); rh.copy_(rs[i % 4].render(od, batches[i % NB][1], bf)[0], non_blocking=True)
        torch.cuda.synchronize()
tr = NgpTrainer(f, bf, N, target_batch_size=1 << 20)
tgt = torch.rand((N, 3), device=dev); bg = torch.zeros((N, 3), device=dev)
if os.environ.get('SYNTH_W'):
    import numpy as np
    t_, d_, c_ = synth.ngp_weights(seed=0)
    with torch.no_grad():
        f.hash_params.copy_(torch.from_numpy(t_).to(dev)); f.density_params.copy_(torch.from_numpy(d_).to(dev)); f.color_params.copy_(torch.from_numpy(c_).to(dev))
    f.mark_dirty(); f.refresh()
for i in range(3):
    tr.step(*batches[i % NB], tgt, bg, next_rays=batches[(i + 1) % NB])
torch.cuda.synchronize()
e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
e0.record()
trained = torch.zeros((), dtype=torch.int64, device=dev)
import time
t0 = time.perf_counter()
for i in range(K):
    tr.step(*batches[i % NB], tgt, bg, next_rays=batches[(i + 1) % NB])
    if os.environ.get('COUNT'):
        trained += tr.trained_rays()
host = (time.perf_counter() - t0) / K * 1e3
e1.record(); torch.cuda.synchronize()
print('host issue %.3f ms/step' % host)
print('train step %.3f ms, compacted samples %d, trained rays %d' % (e0.elapsed_time(e1) / K, int(tr.compacted_samples()), int(tr.trained_rays())))
