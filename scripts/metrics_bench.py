"""Times SSIM scoring on one GPU: the xrb_ssim launch (tile + mean kernels, preallocated outputs and workspace) on one 800 x 800 x 3 pair and on a batch of
200 pairs, with and without the SSIM map, as CUDA events around each launch, warm, medians of --reps launches; its input bytes (two fp32 images per
pair, read once) over kernel time against the H100 SXM data sheet's 3.35 TB/s; metrics.validate_metrics on a 200-view val_step-shaped output as host
wall time including its one synchronisation; and, as a stand-in for the reference's scikit-image scoring (not installed here), the host path the
reference's ValidateHook takes per view: two device-to-host copies, numpy MSE / PSNR and a float64 scipy.ndimage.uniform_filter restatement of
structural_similarity, timed on --host-views views and scaled to 200. The card, power limit and SM clock are read in the same run.

    python scripts/metrics_bench.py [--reps 20] [--host-views 5]
"""
import argparse
import json
import os
import subprocess
import sys
import time

import numpy as np
import torch
from scipy.ndimage import uniform_filter

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

H = W = 800
CH = 3
VIEWS = 200
HBM_BYTES_PER_S = 3.35e12


def card():
    q = subprocess.run(['nvidia-smi', '--query-gpu=name,power.limit,clocks.sm,clocks.max.sm', '--format=csv,noheader'], capture_output=True, text=True)
    return q.stdout.strip().splitlines()[0] if q.returncode == 0 else 'unknown'


def host_ssim(x, y, R):
    """structural_similarity(x, y, multichannel=True, full=True)[1].mean() restated in float64 on scipy.ndimage.uniform_filter, the filter
    scikit-image calls"""
    x, y = x.astype(np.float64), y.astype(np.float64)
    C1, C2, cn = (0.01 * R) ** 2, (0.03 * R) ** 2, 49 / 48
    total = 0.0
    for c in range(x.shape[-1]):
        a, b = x[..., c], y[..., c]
        f = lambda t: uniform_filter(t, size=7, mode='reflect')                                          # noqa: E731
        ux, uy, uxx, uyy, uxy = f(a), f(b), f(a * a), f(b * b), f(a * b)
        vx, vy, vxy = cn * (uxx - ux * ux), cn * (uyy - uy * uy), cn * (uxy - ux * uy)
        total += (((2 * ux * uy + C1) * (2 * vxy + C2)) / ((ux ** 2 + uy ** 2 + C1) * (vx + vy + C2))).sum()
    return total / x.size


def time_launch(x, y, reps, full):
    """median ms of one xrb_ssim launch on x, y [n,H,W,C], CUDA events around each launch"""
    from xrnerf_b200 import _C
    n = x.shape[0]
    mf, mc = torch.empty(n, dtype=torch.float64, device='cuda'), torch.empty(n, dtype=torch.float64, device='cuda')
    smap = torch.empty_like(x) if full else None
    ws = torch.empty(int(_C.lib.xrb_ssim_workspace(n, H, W)), dtype=torch.uint8, device='cuda')
    args = (_C.f32(x), _C.f32(y), n, H, W, CH, 2.0, _C.ptr(mf), _C.ptr(mc), _C.f32(smap), _C.ptr(ws), ws.numel())

    def launch():
        _C.check(_C.lib.xrb_ssim(*args, _C.stream()), 'ssim')
    for _ in range(3):
        launch()
    times = []
    for _ in range(reps):
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        a.record(); launch(); b.record()
        b.synchronize()
        times.append(a.elapsed_time(b))
    return float(np.median(times))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--reps', type=int, default=20)
    ap.add_argument('--host-views', type=int, default=5)
    a = ap.parse_args()
    assert torch.cuda.is_available(), 'metrics_bench needs a GPU'
    from xrnerf_b200 import metrics
    out = {'card_before': card()}
    g = torch.Generator(device='cuda').manual_seed(0)
    gt = torch.rand((VIEWS, H, W, CH), device='cuda', generator=g)
    rgb = (gt + 0.05 * torch.randn((VIEWS, H, W, CH), device='cuda', generator=g)).clamp_(0, 1)
    pair_bytes = 2 * H * W * CH * 4
    for name, n in (('pair', 1), ('batch200', VIEWS)):
        for full in (False, True):
            ms = time_launch(rgb[:n], gt[:n], a.reps, full)
            key = name + ('_map' if full else '')
            out[key + '_ms'] = round(ms, 4)
            out[key + '_read_TBps'] = round(n * pair_bytes / (ms * 1e-3) / 1e12, 3)
            out[key + '_read_share_of_3.35TBps'] = round(n * pair_bytes / (ms * 1e-3) / HBM_BYTES_PER_S, 3)
    outputs = {'rgbs': list(rgb.unbind(0)), 'gt_imgs': list(gt.unbind(0))}
    metrics.validate_metrics(outputs)
    walls = []
    for _ in range(5):
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        res = metrics.validate_metrics(outputs)
        walls.append(time.perf_counter() - t0)
    out['validate_metrics_200_views_ms'] = round(1e3 * float(np.median(walls)), 2)
    host = []
    for i in range(a.host_views):
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        x, y = outputs['rgbs'][i].cpu().numpy(), outputs['gt_imgs'][i].cpu().numpy()
        mse = np.mean((x - y) ** 2)
        _ = -10. * np.log(mse) / np.log(np.array([10.]))
        s = host_ssim(x, y, 2.0)
        host.append(time.perf_counter() - t0)
        assert abs(s - res['ssim'][i]) <= 1e-10, (s, res['ssim'][i])
    out['host_standin_per_view_ms'] = round(1e3 * float(np.median(host)), 1)
    out['host_standin_200_views_ms_scaled'] = round(VIEWS * 1e3 * float(np.median(host)), 0)
    out['host_standin_views_timed'] = a.host_views
    out['cpu'] = os.cpu_count()
    out['card_after'] = card()
    print(json.dumps(out))


if __name__ == '__main__':
    main()
