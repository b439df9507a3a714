"""Records the `model` dict that each of the five reference config files of the three model families yields through xrnerf_b200.registry.load_config
(the reference's configs/*.py, read from its checkout), into tests/golden/reference_config_models.json, so that tests/test_registry.py builds the networks
from them without the reference checkout.

    python tests/golden/make_golden_configs.py /path/to/xrnerf      # a checkout of the reference
"""
import importlib.util
import json
import os
import sys

HERE = os.path.dirname(os.path.abspath(__file__))
CONFIGS = [('configs/nerf/nerf_blender_base01.py', 'NerfNetwork'), ('configs/nerf/nerf_llff_base01.py', 'NerfNetwork'), ('configs/instant_ngp/nerf_blender_local01.py', 'HashNerfNetwork'),
           ('configs/mipnerf/mipnerf_blender.py', 'MipNerfNetwork'), ('configs/mipnerf/mipnerf_multiscale.py', 'MipNerfNetwork')]   # every config of the three model families


def plain(x):
    if isinstance(x, dict):
        return {k: plain(v) for k, v in x.items()}
    if isinstance(x, (list, tuple)):
        return [plain(v) for v in x]
    return x


def main(ref_root):
    spec = importlib.util.spec_from_file_location('xrb_config', os.path.join(HERE, '..', '..', 'xrnerf_b200', 'registry', 'config.py'))
    m = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(m)
    out = []
    for p, t in CONFIGS:
        cfg = m.load_config(os.path.join(ref_root, p), dataname='lego')
        assert 'lego' in cfg.work_dir or 'lego' in str(cfg.get('basedata_cfg', ''))   # the dataname substitution reached the file
        out.append({'config': p, 'type': t, 'model': plain(dict(cfg.model))})
    with open(os.path.join(HERE, 'reference_config_models.json'), 'w') as fh:
        fh.write(json.dumps(out, indent=1) + '\n')


if __name__ == '__main__':
    main(sys.argv[1])
