"""CPU checks of the host-side weight packers of the wgmma NerfMLP kernels (xrnerf_b200/nerf_mlp.py): the swizzled byte layouts the kernels'
shared-memory descriptors assume, and the stream image sizes / bias vector layout of csrc/nerf_mlp_tc.cu. No GPU needed."""
import numpy as np
import torch
from cases import MIP_MLP, NERF_MLP

from xrnerf_b200 import nerf_mlp as nm
from xrnerf_b200 import registry as R


def test_swizzle_128b_slab_layout():
    """K-major SWIZZLE_128B: element (n,k) of an [N,64] slab at (n>>3)*1024 + (n&7)*128 + (((k>>3) ^ (n&7))<<4) + (k&7)*2"""
    rng = np.random.default_rng(0)
    w = rng.integers(-1000, 1000, (128, 64)).astype(np.float32)
    b = nm._slab(w).view(np.float16)
    n, k = np.meshgrid(np.arange(128), np.arange(64), indexing='ij')
    off = ((n >> 3) * 1024 + (n & 7) * 128 + (((k >> 3) ^ (n & 7)) << 4) + (k & 7) * 2) // 2
    assert b.size == 128 * 64 and np.array_equal(b[off], w.astype(np.float16))
    assert len(np.unique(off)) == off.size                          # a bijection


def test_swizzle_64b_slab_layout():
    """K-major SWIZZLE_64B: element (n,k) of a [N,32] slab at (n>>3)*512 + (n&7)*64 + (((k>>3) ^ ((n>>1)&3))<<4) + (k&7)*2"""
    rng = np.random.default_rng(1)
    w = rng.integers(-1000, 1000, (256, 32)).astype(np.float32)
    b = nm._slab64(w).view(np.float16)
    n, k = np.meshgrid(np.arange(256), np.arange(32), indexing='ij')
    off = ((n >> 3) * 512 + (n & 7) * 64 + (((k >> 3) ^ ((n >> 1) & 3)) << 4) + (k & 7) * 2) // 2
    assert b.size == 256 * 32 and np.array_equal(b[off], w.astype(np.float16))
    assert len(np.unique(off)) == off.size


def test_stream_image_and_bias_vector():
    torch.manual_seed(0)
    for cfg, n_kb in ((NERF_MLP, [1, 4, 4, 4, 4, 5, 4, 4, 4]), (MIP_MLP, [2, 4, 4, 4, 4, 6, 4, 4, 4])):
        mlp = R.build_mlp(cfg)
        image, bias = nm.pack_nerf_mlp(mlp)
        # 256-wide layers: 2 slabs of 16 KB per K-block; views_linears.0: 5 slabs [128 x 64]; rgb_linear: 2 slabs [16 x 64]
        assert image.numel() == sum(n_kb) * 2 * 16384 + 5 * 16384 + 2 * 2048
        n_layer_bias = 9 * 256 + 128 + 16
        f32 = (n_layer_bias + 257 + 7) // 8 * 8
        assert bias.numel() == f32 + n_layer_bias // 2 and bias.dtype == torch.float32
        b = bias.numpy()
        assert np.array_equal(b[:256], mlp.pts_linears[0].bias.detach().numpy())
        assert np.array_equal(b[n_layer_bias:n_layer_bias + 256], mlp.alpha_linear.weight.detach().numpy()[0]) and b[n_layer_bias + 256] == mlp.alpha_linear.bias.item()
        h16 = b[f32:].view(np.float16)
        assert np.array_equal(h16[:n_layer_bias], b[:n_layer_bias].astype(np.float16))
        # first slab = K-half 0 of pts_linears.0 over the first 64 encoding columns, in the 64-byte-swizzle layout
        W0 = mlp.pts_linears[0].weight.detach().numpy()
        assert np.array_equal(image.numpy()[:16384], nm._slab64(np.ascontiguousarray(W0[:, :32])))
