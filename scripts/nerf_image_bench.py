"""Times whole-image inference of the dense networks on one GPU: NerfNetwork.val_step (NeRF, 64 + 128 samples) and MipNerfNetwork.val_step (2 x 128)
on one 800 x 800 view (640 000 rays, GPU-generated with xrb_nerf_get_rays, Blender intrinsics and a spiral pose), fused path (fused_inference = True,
ray batches of xrnerf_b200.nerf.ray_batch_size rays) against the reference-shaped chunk loop (fused_inference = False, chunk 32 768 rays), on the same
rays, z values and default-initialised weights, with the two paths' per-ray rgb differences; and the fused renderers with depth=True against depth=False on the same rays. The val pipeline hands
back precomputed rays, so the times are the render's. Every arm runs once before it is timed; the compared arms alternate; medians of CUDA events;
peak torch.cuda.max_memory_allocated above the allocation before the call; the card, power limit and SM clock are read before and after.

    python scripts/nerf_image_bench.py [--reps 5]
"""
import argparse
import ctypes as C
import json
import os
import subprocess
import sys

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

H = W = 800
NERF_MLP = dict(type='NerfMLP', skips=[4], netdepth=8, netwidth=256, netchunk=1024 * 32, output_ch=5, use_viewdirs=True,
                embedder=dict(type='BaseEmbedder', i_embed=0, multires=10, multires_dirs=4))
NERF = dict(type='NerfNetwork', cfg=dict(phase='train', N_importance=128, is_perturb=False, chunk=1024 * 32, bs_data='rays_o'), mlp=NERF_MLP, mlp_fine=NERF_MLP,
            render=dict(type='NerfRender', white_bkgd=True, raw_noise_std=0))
MIP = dict(type='MipNerfNetwork', cfg=dict(phase='train', ray_shape='cone', resample_padding=0.01, use_multiscale=False, coarse_loss_mult=0.1, num_levels=2,
                                          chunk=1024 * 32, bs_data='rays_o'),
           mlp=dict(type='NerfMLP', skips=[4], netdepth=8, netwidth=256, netchunk=1024 * 32, use_viewdirs=True,
                    embedder=dict(type='MipNerfEmbedder', min_deg_point=0, max_deg_point=16, min_deg_view=0, max_deg_view=4, use_viewdirs=True, append_identity=True)),
           render=dict(type='MipNerfRender', white_bkgd=True, raw_noise_std=0, rgb_padding=0.001, density_bias=-1, density_activation='softplus'))


def card():
    q = subprocess.run(['nvidia-smi', '--query-gpu=name,power.limit,clocks.sm,clocks.max.sm', '--format=csv,noheader'], capture_output=True, text=True)
    return q.stdout.strip().splitlines()[0] if q.returncode == 0 else 'unknown'


def view(mip):
    """one whole view: rays (+ radii), GetZvals(near 2, far 6, 64 or 129), and GetPts for the NeRF chunk loop"""
    from xrnerf_b200 import _C, synth
    n = H * W
    pose = synth.pose_spherical(30.0, -30.0, 4.0)
    c2w = (C.c_float * 12)(*[float(v) for v in pose[:3, :4].reshape(-1)])
    o, d, v = (torch.empty((n, 3), device='cuda') for _ in range(3))
    r = torch.empty((n, 1), device='cuda') if mip else None
    _C.check(_C.lib.xrb_nerf_get_rays(c2w, H, W, float(synth.FOCAL), float(synth.FOCAL), W / 2.0, H / 2.0, 0, None, n, _C.ptr(o), _C.ptr(d), _C.ptr(v), _C.ptr(r),
                                      _C.stream()), 'get_rays')
    s = 129 if mip else 64
    z = torch.empty((n, s), device='cuda')
    _C.check(_C.lib.xrb_nerf_zvals(n, s, 2.0, 6.0, 0, None, _C.ptr(z), _C.stream()), 'zvals')
    d_view = {'rays_o': o, 'rays_d': d, 'viewdirs': v, 'z_vals': z, 'src_shape': torch.tensor([H, W, 3])}
    if mip:
        d_view['radii'] = r
    else:
        d_view['pts'] = o[:, None] + d[:, None] * z[..., None]
    return d_view


def run_alternating(arms, reps):
    """arms: name -> fn; each run once, then `reps` rounds of every arm in turn -> name -> (median ms, peak extra bytes of the first timed call)"""
    times, peaks = {k: [] for k in arms}, {}
    for fn in arms.values():
        fn()
    for _ in range(reps):
        for k, fn in arms.items():
            torch.cuda.synchronize()
            base = torch.cuda.memory_allocated()
            torch.cuda.reset_peak_memory_stats()
            a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            a.record(); fn(); b.record()
            torch.cuda.synchronize()
            times[k].append(a.elapsed_time(b))
            peaks.setdefault(k, torch.cuda.max_memory_allocated() - base)
    return {k: (float(np.median(v)), peaks[k]) for k, v in times.items()}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--reps', type=int, default=5)
    args = ap.parse_args()
    assert torch.cuda.is_available(), 'needs a GPU'
    from xrnerf_b200 import registry as R
    from xrnerf_b200.nerf import MipNerfRenderer, NerfRenderer, bytes_per_ray, ray_batch_size
    out = {'card_before': card(), 'rays': H * W}
    for name, model, mip in (('nerf', NERF, False), ('mipnerf', MIP, True)):
        torch.manual_seed(0)
        net = R.build_network(model).cuda()
        d_view = view(mip)
        net.set_val_pipeline(lambda item: dict(d_view))
        image = torch.rand((1, 1, H, W, 3), device='cuda')
        rows = [128, 128] if mip else [64, 192]
        ic = 96 if mip else 63

        def val(fused):
            net.fused_inference = fused
            return net.val_step({'poses': torch.zeros((1, 1, 4, 4)), 'images': image})
        res = run_alternating({'fused': lambda: val(True), 'chunked': lambda: val(False)}, args.reps)
        tol = {'coarse_rgb': 1e-2, 'rgb': 1e-2} if mip else {'coarse_rgb': 2e-3, 'rgb': 5e-3}      # the renderer tests' tolerances
        with torch.no_grad():
            net.fused_inference = True
            a = net.batchify_forward(dict(d_view), is_test=True)
            net.fused_inference = False
            b = net.batchify_forward(dict(d_view), is_test=True)
        diff = {k: (a[k] - b[k]).abs().amax(-1) for k in tol}
        batch = ray_batch_size(rows, ic)
        agree = {k: dict(max_abs=float(v.max()), p999_abs=float(v.quantile(0.999)), rays_over_tolerance=int((v > tol[k]).sum()), tolerance=tol[k],
                         ray_batches_with_rays_over=sorted({int(i) // batch for i in torch.nonzero(v > tol[k]).flatten().tolist()}))
                 for k, v in diff.items()}
        r = MipNerfRenderer(net) if mip else NerfRenderer(net)
        rargs = (d_view['rays_o'], d_view['rays_d'], d_view['viewdirs']) + ((d_view['radii'],) if mip else ())
        dep = run_alternating({'depth_off': lambda: r.render(*rargs, z_vals=d_view['z_vals'], depth=False),
                               'depth_on': lambda: r.render(*rargs, z_vals=d_view['z_vals'], depth=True)}, args.reps)
        out[name] = dict(ray_batch=batch, bytes_per_ray=bytes_per_ray(rows, ic),
                         fused_ms=res['fused'][0], fused_rays_per_s=H * W / res['fused'][0] * 1e3, fused_peak_bytes=res['fused'][1],
                         chunked_ms=res['chunked'][0], chunked_rays_per_s=H * W / res['chunked'][0] * 1e3, chunked_peak_bytes=res['chunked'][1],
                         fused_vs_chunked=agree,
                         render_depth_off_ms=dep['depth_off'][0], render_depth_on_ms=dep['depth_on'][0])
        del net, d_view, r, a, b
        torch.cuda.empty_cache()
    out['card_after'] = card()
    print(json.dumps(out))


if __name__ == '__main__':
    main()
