"""Records what the REFERENCE's own CUDA kernels (extensions/ngp_raymarch, built unmodified by oracle/build_ref_cuda.py) compute for the inputs of
tests/test_gpu_vs_ref_cuda.py, into tests/golden/ref_cuda_march.npz, so that the test needs neither the reference checkout nor its build.

    python tests/golden/make_golden_ref_cuda.py        # on a GPU, with oracle/_ref/cuda/raymarch_cuda_ref.so built

Stored: the reference march's per-ray sample counts and total, the sample rows of a fixed, seeded subset of rays (<= 256), and the reference
compositing (calc_rgb_influence_api) of seeded raw values over OUR march of the same rays."""
import os
import sys

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, 'tests'))

from test_gpu_vs_ref_cuda import N_SAMPLED_RAYS, composite, march, scene_rays   # noqa: E402


def main():
    from oracle import build_ref_cuda
    import xrnerf_b200.raymarch_cuda as ours
    ref = build_ref_cuda.load_module()
    assert ref is not None, 'oracle/_ref/cuda/raymarch_cuda_ref.so is not built'
    o, d, bf = scene_rays()
    cr, _, nr, cntr = march(ref, o, d, bf)          # first call of the process: the reference's static pcg32 is at its seed
    co, _, no, _ = march(ours, o, d, bf, ours)
    counts, base = nr[:, 0].cpu().numpy(), nr[:, 1].cpu().numpy()
    rays = np.sort(np.random.default_rng(17).choice(np.nonzero(counts > 0)[0], N_SAMPLED_RAYS, replace=False))
    crn = cr.cpu().numpy()
    rows = np.concatenate([crn[base[i]:base[i] + counts[i]] for i in rays])
    rgb, alpha = composite(ref, co, no)
    np.savez_compressed(os.path.join(ROOT, 'tests', 'golden', 'ref_cuda_march.npz'), counts=counts.astype(np.int32), total=np.int64(int(cntr[1])),
                        rays=rays.astype(np.int32), rows=rows.astype(np.float32), rgb=rgb.cpu().numpy(), alpha=alpha.cpu().numpy())


if __name__ == '__main__':
    main()
