"""GPU cross-check against the REFERENCE's own CUDA kernels (extensions/ngp_raymarch built unmodified for sm_90a by oracle/build_ref_cuda.py), through the identical
`raymarch_cuda` signatures. The bit-exact contract is defined on the un-contracted CPU build of the same sources (oracle/_ref, tests/test_gpu_raymarch.py): nvcc fuses
the reference's `o + t*d` into FMAs, so here the march may differ in a handful of samples and the tolerances say so. The reference side is recorded in tests/golden/ref_cuda_march.npz
(tests/golden/make_golden_ref_cuda.py), so the test needs neither the reference checkout nor its build."""
import os

import numpy as np
import pytest
import torch

pytestmark = pytest.mark.gpu
GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), 'golden', 'ref_cuda_march.npz')   # tests/golden/make_golden_ref_cuda.py
N_SAMPLED_RAYS = 256


@pytest.fixture(scope='module')
def ours():
    import xrnerf_b200.raymarch_cuda as m
    return m


def scene_rays():
    """the `scene` fixture's rays and bitfield (tests/conftest.py) on the GPU"""
    from xrnerf_b200 import synth
    bf, _ = synth.bitfield_from_grid_numpy(synth.lego_like_density_grid(0))
    o, d, _, _ = synth.ray_batch(4096, seed=1)
    return (torch.from_numpy(np.ascontiguousarray(o)).cuda(), torch.from_numpy(np.ascontiguousarray(d)).cuda(), torch.from_numpy(bf).cuda())


def march(mod, o, d, bf, ours_mod=None):
    n = o.shape[0]
    cap = n * 256
    md = torch.tensor([[0, 0, 0, 0, .5, .5, 1111., 1111., 0, 0, 0]], dtype=torch.float32, device='cuda')
    xf = torch.zeros((1, 4, 3), dtype=torch.float32, device='cuda'); ids = torch.zeros(n, dtype=torch.int32, device='cuda')
    coords = torch.zeros((cap, 7), dtype=torch.float32, device='cuda'); ridx = torch.zeros((n, 1), dtype=torch.int32, device='cuda')
    ns = torch.zeros((n, 2), dtype=torch.int32, device='cuda'); cnt = torch.zeros(2, dtype=torch.int32, device='cuda')
    if ours_mod is not None:
        ours_mod.reset_rng(ray_sampler=0)
    mod.rays_sampler_api(o, d, bf, md, ids, xf, 0.0, 1.0, 0.05, 1.0 / 256, coords, ridx, ns, cnt)
    torch.cuda.synchronize()
    return coords, ridx, ns, cnt


def composite(mod, coords, ns):
    """calc_rgb_influence_api of seeded raw values over the samples `coords` / `ns` of a march"""
    s = int(ns[:, 0].sum())
    raw = (torch.randn((s, 4), generator=torch.Generator().manual_seed(0)) * 0.5).cuda()   # drawn on the host: the same values on every GPU
    n = ns.shape[0]
    rgb = torch.zeros((n, 3), device='cuda'); alpha = torch.zeros((n, 1), device='cuda')
    mod.calc_rgb_influence_api(raw, coords[:s].contiguous(), ns, torch.tensor([0.1, 0.2, 0.3]), 2, 3, 0.0, 1.0, rgb, alpha)
    torch.cuda.synchronize()
    return rgb, alpha


def test_march_and_composite_agree_with_reference_cuda_kernels(ours):
    g = np.load(GOLDEN)
    o, d, bf = scene_rays()
    co, _, no, cnto = march(ours, o, d, bf, ours)
    a, b = g['counts'].astype(np.int64), no[:, 0].cpu().numpy().astype(np.int64)
    assert abs(int(g['total']) - int(cnto[1])) <= max(8, int(cnto[1]) // 2000)
    assert (a != b).mean() < 2e-3                              # per-ray counts: all but FMA-rounding cases
    bo, con = no[:, 1].cpu().numpy(), co.cpu().numpy()         # the reference's bases depend on atomic arrival order: compare ray by ray
    worst, off, compared = 0.0, 0, 0
    for i in g['rays']:
        k = int(a[i])
        if b[i] == k:
            worst = max(worst, float(np.abs(g['rows'][off:off + k] - con[bo[i]:bo[i] + k]).max())); compared += 1
        off += k
    assert compared >= N_SAMPLED_RAYS * 9 // 10
    assert worst <= 2e-6, worst                                 # positions differ by the FMA's one rounding at most
    # compositing of identical inputs (our march, seeded raw) through the reference kernel (recorded) and ours
    rgb, alpha = composite(ours, co, no)
    assert float(np.abs(g['rgb'] - rgb.cpu().numpy()).max()) <= 2e-5 and float(np.abs(g['alpha'] - alpha.cpu().numpy()).max()) <= 2e-5
