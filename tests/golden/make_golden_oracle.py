"""Records what the REFERENCE's own raymarch kernels, compiled for CPU (oracle/_ref, built by oracle/Makefile where the reference checkout exists),
return for the cases of tests/test_oracle_vs_ref.py, into tests/golden/oracle_ref.npz. The test then compares the C port with these records and needs
neither the reference checkout nor its build.

    python tests/golden/make_golden_oracle.py
"""
import os
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, 'tests'))

import test_oracle_vs_ref as T   # noqa: E402


def main():
    from oracle.oracle import Port, Ref, build, have_ref
    from xrnerf_b200 import synth
    build()
    assert have_ref(), 'oracle/_ref is not built (needs the reference checkout)'
    port, ref, rec = Port(), Ref(serial=True), T.Record()
    grid = synth.lego_like_density_grid(0)
    bf, mean = synth.bitfield_from_grid_numpy(grid)
    o, d, img, poses = synth.ray_batch(4096, seed=1)
    s = dict(grid=grid, bitfield=bf, mean=mean, rays_o=o, rays_d=d, img_ids=img, poses=poses, metadata=synth.metadata_for(poses.shape[0]))   # tests/conftest.py `scene`
    marched = T.march(port, s)
    raw = T.raw_for_march(marched)
    T.case_march(ref, s, rec, T.march(ref, s))
    T.case_second_call(ref, s, rec)
    T.case_edge_rays(ref, s, rec)
    T.case_all_ones(ref, s, rec)
    T.case_compacted(ref, port, rec, marched, raw)
    for ra, da in [(2, 3), (3, 1), (0, 2), (1, 0)]:
        T.case_calc_rgb(ref, port, rec, marched, raw, ra, da)
    T.case_mark_untrained(ref, s, rec)
    T.case_grid_samples(ref, s, rec)
    T.case_splat_ema_bitfield(ref, port, s, rec)
    b, m = ref.update_bitfield(grid)
    rec.exact('scene_bitfield', np.asarray(b, np.uint8))
    rec.d['scene_mean'] = np.float64(m[0])
    np.savez_compressed(os.path.join(ROOT, 'tests', 'golden', 'oracle_ref.npz'), **rec.d)


if __name__ == '__main__':
    main()
