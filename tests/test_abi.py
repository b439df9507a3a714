"""CPU-only: the C-ABI shared library builds/loads without a GPU and exports EVERY symbol include/xrnerf_b200.h declares;
argument validation paths (no kernel launch) return the documented error codes; the product package has no CPU fallback."""
import ctypes as C
import os
import re

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _declared():
    src = open(os.path.join(ROOT, 'include', 'xrnerf_b200.h')).read()
    src = re.sub(r'/\*.*?\*/', '', src, flags=re.S)
    return sorted(set(re.findall(r'\b(xrb_[a-z0-9_]+)\s*\(', src)))


def test_library_exports_every_declared_symbol():
    from xrnerf_b200 import build
    lib = C.CDLL(build.build())
    names = _declared()
    assert len(names) >= 40
    missing = [n for n in names if not hasattr(lib, n)]
    assert not missing, missing
    assert lib.xrb_abi_version() == 5 and lib.xrb_built_for_sm() == 90


def test_python_binding_covers_header():
    from xrnerf_b200 import _C
    assert sorted(_C.EXPORTS) == _declared()


def test_argument_validation_without_gpu():
    from xrnerf_b200 import _C
    lib = _C.lib
    lib.xrb_last_error.restype = C.c_char_p
    # negative sizes / null pointers are rejected before any CUDA call
    assert lib.xrb_rm_ema_grid_samples(None, -1, C.c_float(0.95), None, None) == -1
    assert b'negative' in lib.xrb_last_error()
    assert lib.xrb_rm_ema_grid_samples(None, 16, C.c_float(0.95), None, None) == -1
    assert lib.xrb_rm_rays_sampler(None, None, None, None, None, None, 0, 0, C.c_float(0), C.c_float(1), C.c_float(0.05), C.c_float(1 / 256), 9121, 0, None, None, None, None, None, None) == 0  # empty batch is a no-op
    cfg = _C.NgpConfig(16, 2, 19, 16, 1.38191288, 64, 1, 2)
    assert lib.xrb_tcnn_hashgrid_num_params(cfg) == 12196240
    bad = _C.NgpConfig(16, 4, 19, 16, 1.38191288, 64, 1, 2)   # n_features 4 is not implemented: loud, not silent
    assert lib.xrb_tcnn_hashgrid_num_params(bad) == -1 and b'unsupported' in lib.xrb_last_error()
    assert lib.xrb_nerf_sample_pdf(None, None, None, None, None, 4, 300, 128, None, None, None) == -2
    # NerfMLP: sizes / supported shapes / null pointers / alignment, all checked before any CUDA call
    assert lib.xrb_nerf_mlp_forward(None, None, None, -1, 63, 27, None, None) == -1
    assert lib.xrb_nerf_mlp_forward(None, None, None, 10, 50, 27, None, None) == -2
    assert lib.xrb_nerf_mlp_forward(None, None, None, 10, 60, 27, None, None) == -2 and b'(63,27) or (96,27)' in lib.xrb_last_error()
    assert lib.xrb_nerf_mlp_forward(None, None, None, 0, 63, 27, None, None) == 0                          # empty input is not an error
    assert lib.xrb_nerf_mlp_forward(None, None, None, 10, 63, 27, None, None) == -1 and b'null' in lib.xrb_last_error()
    buf = (C.c_char * 64)()
    a = C.addressof(buf)
    odd = C.c_void_p(a + 4)                                                                                  # not 16-byte aligned
    assert lib.xrb_nerf_mlp_forward(odd, odd, odd, 10, 63, 27, odd, None) == -1 and b'aligned' in lib.xrb_last_error()
    assert lib.xrb_mip_ipe_tiles_rays(None, None, None, None, None, 4, 8, 0, 30, 0, 4, None, None) == -1 and b'wider' in lib.xrb_last_error()   # 180 IPE columns do not fit two blocks
    assert lib.xrb_mip_ipe_tiles_rays(None, None, None, None, None, 0, 8, 0, 16, 0, 4, None, None) == 0
    assert lib.xrb_mip_ipe_tiles_rays(None, None, None, None, None, 4, 8, 0, 16, 0, 4, None, None) == -1
    assert lib.xrb_adam_ema_step(None, None, None, None, None, 8, C.c_float(1e-2), C.c_float(.9), C.c_float(.99), C.c_float(1e-15), C.c_float(0), 1, C.c_float(1), None, C.c_float(1.5), None) == -1
    assert lib.xrb_adam_ema_step(None, None, None, None, None, 0, C.c_float(1e-2), C.c_float(.9), C.c_float(.99), C.c_float(1e-15), C.c_float(0), 1, C.c_float(1), None, C.c_float(0.05), None) == 0
    assert lib.xrb_nerf_enc_image_bytes(129, 63) == 2 * 2 * 16384 and lib.xrb_nerf_enc_image_bytes(129, 96) == 2 * 3 * 16384


def test_peer_exchange_argument_validation_without_gpu():
    """xrb_peer_* (csrc/peer_adam.cu): the exchange layout is validated before any CUDA call"""
    from xrnerf_b200 import _C
    lib = _C.lib
    buf = (C.c_char * 4096)()
    a = (C.addressof(buf) + 255) & ~255

    def layout(world=2, rank=0, per=1024, n_table=2000, n_mlp=10, off_g16=128, off_gmlp=128 + 2 * 2048, off_t16=128 + 2 * 2048 + 48, base=(1, 1)):
        L = _C.PeerLayout(world, rank, (C.c_void_p * 8)(), off_g16, off_gmlp, off_t16, n_table, per, n_mlp)
        for p, b in enumerate(base):
            L.base[p] = a if b else None
        return L
    g = C.c_void_p(a)
    assert lib.xrb_peer_publish_grads(C.byref(layout(world=9)), g, g, 1, None) == -1 and b'world' in lib.xrb_last_error()
    assert lib.xrb_peer_publish_grads(C.byref(layout(rank=2)), g, g, 1, None) == -1
    assert lib.xrb_peer_publish_grads(C.byref(layout(per=1001)), g, g, 1, None) == -1 and b'multiple of 8' in lib.xrb_last_error()
    assert lib.xrb_peer_publish_grads(C.byref(layout(n_table=5000)), g, g, 1, None) == -1                       # the slices do not cover the table
    assert lib.xrb_peer_publish_grads(C.byref(layout(off_g16=64)), g, g, 1, None) == -1 and b'flags' in lib.xrb_last_error()
    assert lib.xrb_peer_publish_grads(C.byref(layout(off_t16=128 + 2 * 2048 + 50)), g, g, 1, None) == -1       # not 16-byte aligned
    assert lib.xrb_peer_publish_grads(C.byref(layout(base=(1, 0))), g, g, 1, None) == -1 and b'null block' in lib.xrb_last_error()
    assert lib.xrb_peer_publish_grads(C.byref(layout()), g, g, 0, None) == -1 and b'step' in lib.xrb_last_error()     # steps count from 1
    grp = _C.PeerMlpGroup(a, None, a, a, None, 8, 4)
    assert lib.xrb_peer_adam_step(C.byref(layout()), g, g, g, None, C.byref(grp), C.byref(grp), C.c_float(1e-2), C.c_float(.9), C.c_float(.99), C.c_float(1e-15), C.c_float(0), 1, C.c_float(0), 1,
                                  None) == -1 and b'outside the gradient block' in lib.xrb_last_error()          # g_off + n > n_mlp
    assert lib.xrb_peer_alloc(64, None, None) == -1 and lib.xrb_peer_open(None, None) == -1
    assert lib.xrb_peer_close(None) == 0 and lib.xrb_peer_free(None) == 0


def test_strided_or_wrong_dtype_tensors_are_rejected():
    """Round-1 W1: a Fortran-ordered rays_o (what `broadcast_to -> reshape -> astype` + torch.from_numpy gives) was handed to the kernels as a bare
    data_ptr() and silently rendered different rays. Every dense-row pointer now goes through _C.ptr, which refuses non-contiguous / wrong-dtype
    tensors with the library's bad-argument status; the high-level renderers copy strided rays instead of reinterpreting them."""
    import numpy as np
    import torch
    from xrnerf_b200 import _C, synth
    from xrnerf_b200.ngp import _rays
    base = np.broadcast_to(np.arange(3, dtype=np.float32), (10, 10, 3)).reshape(-1, 3).astype(np.float32)      # the round-1 construction
    t = torch.from_numpy(base)
    if not t.is_contiguous():                                                                                   # numpy keeps the broadcast's 'K' order here
        with pytest.raises(_C.XrbError, match='non-contiguous'):
            _C.ptr(t)
    f = torch.zeros(6, 3).t()                                                                                   # explicit strided view
    assert not f.is_contiguous()
    with pytest.raises(_C.XrbError, match='XRB_E_BADARG'):
        _C.ptr(f)
    with pytest.raises(_C.XrbError, match='expected torch.float32'):
        _C.f32(torch.zeros(4, dtype=torch.float64))
    with pytest.raises(_C.XrbError):
        _C.rows(torch.zeros(4, 7)[:, ::2])                                                                      # inner stride 2: not a row view
    p, stride = _C.rows(torch.zeros(5, 7)[:, 4:])                                                               # coords[:, 4:] is a legal row view
    assert stride == 7
    r = _rays(torch.zeros(3, 8).t()[:, :3])
    assert r.is_contiguous() and r.shape == (8, 3)
    with pytest.raises(_C.XrbError):
        _rays(torch.zeros(8, 3, dtype=torch.float64))
    o, d = synth.get_rays_ngp(synth.spiral_poses_ngp(40)[3], h=12, w=20)
    assert o.flags['C_CONTIGUOUS'] and d.flags['C_CONTIGUOUS'] and o.strides == (12, 4)


def test_cell_image_layout_and_validation_without_gpu():
    from xrnerf_b200 import _C
    lib = _C.lib
    cfg = _C.NgpConfig(16, 2, 19, 16, 1.38191288, 64, 1, 2)
    res = (C.c_uint32 * 16)()
    assert lib.xrb_tcnn_hashgrid_layout(cfg, None, None, res) == 0
    for n in range(0, 9):                                                                                       # (up to 13 levels may be packed; 9+ are GB-sized)
        assert lib.xrb_ngp_cell_image_bytes(cfg, n) == 32 * sum(int(r) ** 3 for r in list(res)[:n])           # one 32-byte record per grid cell
    assert lib.xrb_ngp_cell_image_bytes(cfg, 6) == 32 * (16 ** 3 + 23 ** 3 + 31 ** 3 + 43 ** 3 + 59 ** 3 + 81 ** 3)
    assert lib.xrb_ngp_build_cell_image(cfg, None, 0, None, None) == 0
    assert lib.xrb_ngp_build_cell_image(cfg, None, 14, None, None) == -1
    assert lib.xrb_ngp_build_cell_image(cfg, None, 5, None, None) == -1 and b'null' in lib.xrb_last_error()
    buf = (C.c_char * 256)()
    a = (C.addressof(buf) + 63) & ~63
    tab = _C.NgpTable(a, a + 4, 6)                                                                              # cell image not 32-byte aligned
    out = C.c_void_p(a)
    assert lib.xrb_ngp_mlp_forward(cfg, tab, None, None, out, out, 3, out, 3, 4, None, out, 1, None) == -1 and b'cell image' in lib.xrb_last_error()
    assert lib.xrb_ngp_mlp_forward(cfg, None, None, None, out, out, 3, out, 3, 4, None, out, 1, None) == -1
    assert lib.xrb_rm_update_bitfield(out, out, out, None, None) == -1                                          # scratch is the caller's
    assert lib.xrb_rm_update_bitfield_workspace() == 512 * 4


def test_no_cpu_fallback():
    import torch
    from xrnerf_b200 import _C
    from xrnerf_b200.ngp import NgpField
    f = NgpField()
    with pytest.raises(_C.XrbError):
        f.run_mlp(torch.rand(4, 3), torch.rand(4, 3))        # CPU tensors are refused, nothing silently falls back
    from xrnerf_b200 import registry as R
    e = R.BaseEmbedder(i_embed=0, multires=10, multires_dirs=4)
    with pytest.raises(_C.XrbError):
        e({'pts': torch.rand(2, 4, 3), 'viewdirs': torch.rand(2, 3)})
