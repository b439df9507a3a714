"""Host-side helpers of the networks against the REFERENCE's own functions, imported unmodified from the reference checkout by
tests/golden/make_golden_host_utils.py and recorded in tests/golden/host_utils_ref.npz:
batching.unfold_batching, transforms.recover_shape / merge_ret (networks/utils/batching.py:5-12, transforms.py:5-31), and NGPGridSampler.update_batch_rays
(samplers/ngp_grid_sampler.py:268-284, restated: the reference class imports its CUDA extension at module import)."""
import math
import os

import numpy as np
import torch

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), 'golden', 'host_utils_ref.npz')   # tests/golden/make_golden_host_utils.py
NERF_MLP_CFGS = [dict(skips=[4], netdepth=8, netwidth=256, output_ch=5, use_viewdirs=True, netchunk=1024 * 32, embedder=dict(type='BaseEmbedder', i_embed=0, multires=10, multires_dirs=4)),
                 dict(skips=[4], netdepth=8, netwidth=256, use_viewdirs=True, netchunk=1024 * 32,
                      embedder=dict(type='MipNerfEmbedder', min_deg_point=0, max_deg_point=16, min_deg_view=0, max_deg_view=4, use_viewdirs=True, append_identity=True))]


def batching_inputs():
    g = torch.Generator().manual_seed(0)
    xs = [torch.rand(shape, generator=g) for shape in [(1, 7, 3), (2, 5, 3), (3, 4), (6,), (1, 2, 4, 4)]]
    data = torch.rand((12, 3), generator=g)
    a = {k: torch.rand(5, generator=g) for k in ('rgb', 'disp', 'acc')}; b = {k: torch.rand(5, generator=g) for k in ('rgb', 'disp', 'acc')}
    return xs, data, torch.tensor([3, 4, 3]), a, b


def test_unfold_batching_recover_shape_merge_ret_match_reference():
    from xrnerf_b200.registry import networks as N
    G = np.load(GOLDEN)
    xs, data, lens, a, b = batching_inputs()
    for k, x in enumerate(xs):
        assert np.array_equal(N.unfold_batching(x).numpy(), G[f'unfold_{k}']), x.shape
    assert np.array_equal(N.recover_shape(data, lens).numpy(), G['recover_shape'])
    ours = N.merge_ret(dict(a), dict(b))
    assert set(ours) == {k.split('/')[1] for k in G.files if k.startswith('merge_ret/')}
    assert all(np.array_equal(ours[k].numpy(), G[f'merge_ret/{k}']) for k in ours)


def test_update_batch_rays_rule():
    """n_rays <- min(ceil128(int(n_rays * 2^18 / max(measured / 16, 1))), 2^18), every update_grid_freq-th step, then the counter is cleared."""
    from xrnerf_b200 import registry as R
    smp = R.build_sampler(dict(type='NGPGridSampler', update_grid_freq=16, update_block_size=5000000, n_rays_per_batch=4096, cone_angle_constant=0.00390625, near_distance=0.2,
                               target_batch_size=1 << 18, rgb_activation=2, density_activation=3))
    for measured, n0 in [(16 * 40000, 4096), (16 * 300000, 65536), (0, 4096), (16 * 262144, 262144)]:
        smp.n_rays_per_batch = n0
        smp.measured_batch_size = torch.tensor([measured], dtype=torch.int32)
        smp.set_iter(15)
        smp.update_batch_rays(True)
        m = max(measured / 16, 1)
        want = int(min(math.ceil(int(n0 * (1 << 18) / m) / 128) * 128, 1 << 18))
        assert smp.n_rays_per_batch == want and smp.measured_batch_size.item() == 0
        smp.n_rays_per_batch = n0
        smp.measured_batch_size = torch.tensor([measured], dtype=torch.int32)
        smp.set_iter(14)
        smp.update_batch_rays(True)
        assert smp.n_rays_per_batch == n0 and smp.measured_batch_size.item() == measured


def test_reference_nerf_mlp_checkpoints_load_into_registry_modules():
    """SURVEY 8f-4 (checkpoint compatibility): the state_dict of the REFERENCE's own NerfMLP (NeRF and Mip-NeRF embedders) has exactly our keys and shapes and loads
    with strict=True; the packed wgmma weight image is rebuilt from the loaded weights."""
    from xrnerf_b200 import registry as R
    from xrnerf_b200.nerf_mlp import pack_nerf_mlp
    G = np.load(GOLDEN)
    for c, cfg in enumerate(NERF_MLP_CFGS):
        keys, shapes = [str(k) for k in G[f'ckpt{c}/keys']], [tuple(int(x) for x in s if x) for s in G[f'ckpt{c}/shapes']]
        g = torch.Generator().manual_seed(c)
        sd_ref = {k: torch.randn(s, generator=g) for k, s in zip(keys, shapes)}   # the reference's layout; values: its pts_linears.0.bias, the rest seeded
        sd_ref['pts_linears.0.bias'] = torch.from_numpy(G[f'ckpt{c}/pts_linears.0.bias'])
        ours = R.build_mlp(dict(cfg, type='NerfMLP'))
        sd_ours = ours.state_dict()
        assert list(sd_ref) == list(sd_ours) and all(sd_ref[k].shape == sd_ours[k].shape for k in sd_ref)
        assert (ours.input_ch, ours.input_ch_dirs) == tuple(int(x) for x in G[f'ckpt{c}/input_ch'])
        ours.load_state_dict(sd_ref, strict=True)
        image, bias = pack_nerf_mlp(ours)
        assert torch.equal(bias[:256], sd_ref['pts_linears.0.bias']) and image.numel() > 1_000_000
