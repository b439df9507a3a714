"""CPU-only: the tcnn-shaped modules and the registry HashNerfMLP share tcnn's flat parameter layouts, so a checkpoint written by the reference
(state_dict keys `embedder_pos.params`, `embedder_dir.params`, `density_net.params`, `color_net.params`, /root/reference/xrnerf/models/mlps/hashnerf_mlp.py:36-45) loads into
both, and flat vectors round-trip through import_params / export_params (SURVEY §8f-4). Sizes are tcnn's: hash table 12 196 240 (16 levels x 2 features, T = 2^19, levels
back to back), density net 64*32 + 16*64, colour net 64*32 + 64*64 + 16*64 (outputs padded to 16, 31 inputs padded to 32)."""
import pytest
import torch


def _mods():
    import xrnerf_b200.tcnn as tcnn
    from xrnerf_b200.ngp import PER_LEVEL_SCALE
    enc = tcnn.Encoding(3, dict(otype='HashGrid', n_levels=16, n_features_per_level=2, log2_hashmap_size=19, base_resolution=16, per_level_scale=PER_LEVEL_SCALE))
    sh = tcnn.Encoding(3, dict(otype='SphericalHarmonics', degree=4))
    dnet = tcnn.Network(32, 16, dict(otype='FullyFusedMLP', activation='ReLU', output_activation='None', n_neurons=64, num_layers=1))
    cnet = tcnn.Network(31, 3, dict(otype='FullyFusedMLP', activation='ReLU', output_activation='None', n_neurons=64, num_layers=2))
    return enc, sh, dnet, cnet


def test_flat_param_sizes_and_roundtrip():
    enc, sh, dnet, cnet = _mods()
    assert enc.params.numel() == 12196240 and sh.params.numel() == 0 and dnet.params.numel() == 64 * 32 + 16 * 64 and cnet.params.numel() == 64 * 32 + 64 * 64 + 16 * 64
    assert enc.n_output_dims == 32 and sh.n_output_dims == 16
    g = torch.Generator().manual_seed(0)
    for m in (dnet, cnet):
        v = torch.randn(m.params.numel(), generator=g)
        m.import_params(v)
        assert torch.equal(m.export_params(), v) and m._shadow.version is None          # the fp16 working copy will be rebuilt
        with pytest.raises(ValueError):
            m.import_params(v[:-1])
    v = torch.rand(enc.params.numel(), generator=g) * 2e-4 - 1e-4
    enc.import_params(v.double())                                                          # any dtype is converted to the fp32 master
    assert enc.params.dtype == torch.float32 and torch.equal(enc.export_params(), v)


def test_reference_style_checkpoint_loads_into_modules_and_registry():
    """a `.pth` state_dict with the reference's keys (what mmcv's save_checkpoint writes for HashNerfNetwork.mlp) -> registry HashNerfMLP (strict) and -> the four
    tcnn-shaped modules; exporting from the registry module gives the same vectors back"""
    from xrnerf_b200 import registry as R
    enc, sh, dnet, cnet = _mods()
    g = torch.Generator().manual_seed(1)
    ckpt = {'embedder_pos.params': torch.rand(12196240, generator=g) * 2e-4 - 1e-4, 'embedder_dir.params': torch.zeros(0),
            'density_net.params': torch.randn(3072, generator=g) * 0.1, 'color_net.params': torch.randn(7168, generator=g) * 0.1}
    mlp = R.build_mlp(dict(type='HashNerfMLP', bound=1,
                           embedder_pos=dict(n_input_dims=3, encoding_config=dict(otype='HashGrid', n_levels=16, n_features_per_level=2, log2_hashmap_size=19, base_resolution=16, interpolation='Linear')),
                           embedder_dir=dict(n_input_dims=3, encoding_config=dict(otype='SphericalHarmonics', degree=4)),
                           density_net=dict(n_input_dims=32, n_output_dims=16, network_config=dict(otype='FullyFusedMLP', activation='ReLU', output_activation='None', n_neurons=64, num_layers=1)),
                           color_net=dict(n_input_dims=31, n_output_dims=3, network_config=dict(otype='FullyFusedMLP', activation='ReLU', output_activation='None', n_neurons=64, num_layers=2))))
    assert sorted(mlp.state_dict().keys()) == sorted(ckpt.keys())
    mlp.field._ver = 'stale-marker'
    missing = mlp.load_state_dict(ckpt, strict=True)
    assert not missing.missing_keys and not missing.unexpected_keys
    assert mlp.field._ver is None                                                           # load_state_dict marks the fp16 shadows / cell image / wgmma weight image dirty
    for m, k in ((enc, 'embedder_pos.params'), (dnet, 'density_net.params'), (cnet, 'color_net.params')):
        m.import_params(ckpt[k])
        assert torch.equal(m.export_params(), mlp.state_dict()[k])
    # the registry module's parameters ARE the fused field's (no copy): what the fused kernels train is what state_dict() saves
    assert mlp.field.hash_params.data_ptr() == mlp.embedder_pos.params.data_ptr() and mlp.field.color_params.data_ptr() == mlp.color_net.params.data_ptr()
