"""Records the REFERENCE's own host-side helpers (networks/utils/batching.py, transforms.py) on the inputs of tests/test_host_utils_vs_reference.py and the
state_dict layout of its NerfMLP (NeRF and Mip-NeRF embedders), imported unmodified through oracle/ref_import.py, into tests/golden/host_utils_ref.npz.

    python tests/golden/make_golden_host_utils.py      # where the reference checkout exists
"""
import os
import sys

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, 'tests'))

import test_host_utils_vs_reference as T   # noqa: E402


def main():
    from oracle import ref_import as R
    rb, rt = R.load('networks.utils.batching'), R.load('networks.utils.transforms')
    out = {}
    xs, data, lens, a, b = T.batching_inputs()
    for k, x in enumerate(xs):
        out[f'unfold_{k}'] = rb.unfold_batching(x).numpy()
    out['recover_shape'] = rt.recover_shape(data, lens).numpy()
    for k, v in rt.merge_ret(dict(a), dict(b)).items():
        out[f'merge_ret/{k}'] = v.numpy()
    mlpm = R.load('mlps.nerf_mlp'); R.load('embedders.base'); R.load('embedders.mipnerf_embedder')
    for c, cfg in enumerate(T.NERF_MLP_CFGS):
        torch.manual_seed(0)
        ref = mlpm.NerfMLP(**{k: (dict(v) if isinstance(v, dict) else v) for k, v in cfg.items()})
        sd = ref.state_dict()
        out[f'ckpt{c}/keys'] = np.array(list(sd))
        out[f'ckpt{c}/shapes'] = np.array([list(v.shape) + [0] * (2 - v.dim()) for v in sd.values()], np.int64)
        out[f'ckpt{c}/input_ch'] = np.array([ref.input_ch, ref.input_ch_dirs], np.int64)
        out[f'ckpt{c}/pts_linears.0.bias'] = sd['pts_linears.0.bias'].numpy()
    np.savez_compressed(os.path.join(ROOT, 'tests', 'golden', 'host_utils_ref.npz'), **out)


if __name__ == '__main__':
    main()
