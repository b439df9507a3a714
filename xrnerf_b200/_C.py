"""ctypes binding of libxrnerf_b200.so (the C ABI declared in include/xrnerf_b200.h).

The product path has NO CPU fallback: importing this module without the built CUDA library raises, and every call
checks the status code the library returns. torch is used only for device memory and streams.
"""
import ctypes as C
import os

import torch

_HERE = os.path.dirname(os.path.abspath(__file__))
LIB_PATH = os.path.join(_HERE, 'lib', 'libxrnerf_b200.so')

if not os.path.exists(LIB_PATH):
    raise ImportError(f'{LIB_PATH} is missing: run `python -m xrnerf_b200.build` (needs nvcc; cross-compiles for sm_90a without a GPU). '
                      'xrnerf_b200 has no CPU or PyTorch fallback for its kernels.')

lib = C.CDLL(LIB_PATH)


class NgpConfig(C.Structure):
    _fields_ = [('n_levels', C.c_int), ('n_features', C.c_int), ('log2_hashmap_size', C.c_int), ('base_resolution', C.c_int),
                ('per_level_scale', C.c_float), ('width', C.c_int), ('density_hidden', C.c_int), ('color_hidden', C.c_int)]


class NgpTable(C.Structure):
    """xrb_ngp_table: the fp16 hash table (tcnn layout) + its optional cell image (include/xrnerf_b200.h)"""
    _fields_ = [('table_fp16', C.c_void_p), ('cell_image', C.c_void_p), ('n_packed_levels', C.c_int)]


class PeerLayout(C.Structure):
    """xrb_peer_layout: the exchange blocks of all ranks as mapped in this process + the layout inside a block (include/xrnerf_b200.h)"""
    _fields_ = [('world', C.c_int), ('rank', C.c_int), ('base', C.c_void_p * 8), ('off_g16', C.c_size_t), ('off_gmlp', C.c_size_t), ('off_t16', C.c_size_t),
                ('n_table', C.c_int64), ('per', C.c_int64), ('n_mlp', C.c_int64)]


class PeerMlpGroup(C.Structure):
    """xrb_peer_mlp_group: one small parameter vector every rank updates identically"""
    _fields_ = [('param', C.c_void_p), ('param_fp16', C.c_void_p), ('exp_avg', C.c_void_p), ('exp_avg_sq', C.c_void_p), ('ema', C.c_void_p), ('n', C.c_int64), ('g_off', C.c_int64)]


P = C.c_void_p
_i, _f, _u64, _i64, _sz = C.c_int, C.c_float, C.c_uint64, C.c_int64, C.c_size_t
_cfg = C.POINTER(NgpConfig)
_tab = C.POINTER(NgpTable)

_SIGS = {
    'xrb_abi_version': (C.c_int, []),
    'xrb_built_for_sm': (C.c_int, []),
    'xrb_last_error': (C.c_char_p, []),
    'xrb_rm_generate_grid_samples': (_i, [P, _i, _i, _i, _f, _f, _f, _u64, _i64, P, P, P]),
    'xrb_rm_mark_untrained_density_grid': (_i, [P, P, _i, _i, _i, _i, P, P]),
    'xrb_rm_splat_grid_samples': (_i, [P, P, _i, _i, P, P]),
    'xrb_rm_ema_grid_samples': (_i, [P, _i, _f, P, P]),
    'xrb_rm_update_bitfield_workspace': (_sz, []),
    'xrb_rm_update_bitfield': (_i, [P, P, P, P, P]),
    'xrb_rm_rays_sampler_workspace': (_sz, [_i]),
    'xrb_rm_rays_sampler': (_i, [P, P, P, P, P, P, _i, _i, _f, _f, _f, _f, _u64, _i64, P, P, P, P, P, P]),
    'xrb_rm_compacted_coord_workspace': (_sz, [_i]),
    'xrb_rm_compacted_coord': (_i, [P, P, P, _i, _i, P, P, P, P, P, P]),
    'xrb_ngp_count_trained_rays': (_i, [P, P, _i, P, P]),
    'xrb_rm_calc_rgb_forward': (_i, [P, P, P, P, P, _i, _i, _i, P, P]),
    'xrb_rm_calc_rgb_backward': (_i, [P, P, P, P, P, P, _i, _i, _i, P, P]),
    'xrb_rm_calc_rgb_inference': (_i, [P, P, P, C.POINTER(C.c_float), _i, _i, _i, P, P, P]),
    'xrb_tcnn_hashgrid_num_params': (_i64, [_cfg]),
    'xrb_tcnn_density_num_params': (_i64, [_cfg]),
    'xrb_tcnn_color_num_params': (_i64, [_cfg]),
    'xrb_tcnn_hashgrid_layout': (_i, [_cfg, P, P, P]),
    'xrb_tcnn_cast_params': (_i, [P, P, _i64, P]),
    'xrb_ngp_weight_image_bytes': (_sz, [_cfg]),
    'xrb_ngp_pack_weights': (_i, [_cfg, P, P, P, P]),
    'xrb_ngp_cell_image_bytes': (_sz, [_cfg, _i]),
    'xrb_ngp_build_cell_image': (_i, [_cfg, P, _i, P, P]),
    'xrb_tcnn_hashgrid_forward': (_i, [_cfg, _tab, P, _i, _i, P, P]),
    'xrb_tcnn_sh4_forward': (_i, [P, _i, _i, P, P]),
    'xrb_tcnn_mlp_forward': (_i, [P, P, _i, _i, _i, _i, P, P]),
    'xrb_tcnn_hashgrid_backward': (_i, [_cfg, P, _i, _i, P, _f, P, P]),
    'xrb_tcnn_mlp_backward': (_i, [P, P, P, _i, _i, _i, _i, P, P, P]),
    'xrb_ngp_mlp_forward': (_i, [_cfg, _tab, P, P, P, P, _i, P, _i, _i, P, P, _i, P]),
    'xrb_ngp_density_forward': (_i, [_cfg, _tab, P, P, P, _i, _i, P, _i, P]),
    'xrb_ngp_density_grad': (_i, [_cfg, _tab, P, P, _i, _i, P, P, P]),
    'xrb_ngp_mlp_backward': (_i, [_cfg, _tab, P, P, P, _i, P, _i, P, _i, P, P, P, P]),
    'xrb_ngp_mlp_backward_tc': (_i, [_cfg, _tab, P, P, _i, P, _i, P, _i, P, P, P, P, P]),
    'xrb_adam_ema_step': (_i, [P, P, P, P, P, _i64, _f, _f, _f, _f, _f, _i, _f, P, _f, P]),
    'xrb_adam_ema_step_bf16grad': (_i, [P, P, P, P, P, _i64, _f, _f, _f, _f, _f, _i, _f, P, _f, P]),
    'xrb_pack_bf16': (_i, [P, P, _i64, P]),
    'xrb_peer_alloc': (_i, [_sz, C.POINTER(C.c_void_p), P]),
    'xrb_peer_open': (_i, [P, C.POINTER(C.c_void_p)]),
    'xrb_peer_close': (_i, [P]),
    'xrb_peer_free': (_i, [P]),
    'xrb_peer_publish_grads': (_i, [C.POINTER(PeerLayout), P, P, C.c_uint32, P]),
    'xrb_peer_adam_step': (_i, [C.POINTER(PeerLayout), P, P, P, P, C.POINTER(PeerMlpGroup), C.POINTER(PeerMlpGroup), _f, _f, _f, _f, _f, _i, _f, C.c_uint32, P]),
    'xrb_peer_status': (_i, [P, C.POINTER(C.c_uint32), P]),
    'xrb_ngp_huber5_grad': (_i, [P, P, _i64, _f, P, P, P]),
    'xrb_ngp_render_workspace': (_sz, [_i, _i]),
    'xrb_ngp_render_fused_workspace': (_sz, []),
    'xrb_ngp_render_fused': (_i, [_cfg, _tab, P, P, P, P, _i, _f, _f, _f, _f, _u64, _i64, C.POINTER(C.c_float), _i, _i, P, P, P, P, P]),
    'xrb_nerf_composite_forward': (_i, [P, P, P, _i, _i, _i, _i, _f, _f, _i, P, P, P, P, P]),
    'xrb_nerf_composite_forward_depth': (_i, [P, P, P, _i, _i, _i, _i, _f, _f, _i, P, P, P, P, P, P]),
    'xrb_nerf_composite_backward':(_i, [P, P, P, P, _i, _i, _i, _i, _f, _f, _i, P, P]),
    'xrb_nerf_sample_pdf': (_i, [P, P, P, P, P, _i, _i, _i, P, P, P]),
    'xrb_nerf_posenc': (_i, [P, P, _i64, _i, _i, _i, P, P]),
    'xrb_nerf_mlp_forward': (_i, [P, P, P, _i64, _i, _i, P, P]),
    'xrb_nerf_enc_image_bytes': (_sz, [_i64, _i]),
    'xrb_nerf_pack_embedded': (_i, [P, _i64, _i, _i, P, P]),
    'xrb_nerf_posenc_tiles': (_i, [P, P, _i64, _i, _i, _i, P, P]),
    'xrb_nerf_posenc_tiles_rays': (_i, [P, P, P, P, _i64, _i, _i, _i, P, P]),
    'xrb_mip_embed': (_i, [P, P, P, P, P, _i, _i, _i, _i, _i, _i, P, P, P, P]),
    'xrb_mip_ipe_tiles_rays': (_i, [P, P, P, P, P, _i64, _i, _i, _i, _i, _i, P, P]),
    'xrb_mip_resample': (_i, [P, P, P, _i, _i, _f, P, P]),
    'xrb_nerf_get_rays': (_i, [C.POINTER(C.c_float), _i, _i, _f, _f, _f, _f, _i, P, _i64, P, P, P, P, P]),
    'xrb_ngp_batch_sample': (_i, [P, P, _i, _i, _i, _f, _f, _f, _f, P, _i64, P, _u64, _i64, P, P, P, P, P, P, P]),
    'xrb_nerf_tg_layer': (_i, [P, P]),
    'xrb_nerf_tg_dw': (_i, [P, P]),
    'xrb_nerf_tg_pack_weights': (_i, [P, _i, _i, _i, _i, C.POINTER(C.c_int), C.POINTER(C.c_int), P, P]),
    'xrb_nerf_tg_pack_draw': (_i, [P, _i64, P, P, P, P]),
    'xrb_nerf_tg_grad_scale': (C.c_float, []),
    'xrb_micro_gather': (_i, [P, _i64, _i, _i, C.POINTER(C.c_int64), P, P]),
    'xrb_nerf_zvals': (_i, [_i64, _i, _f, _f, _i, P, P, P]),
    'xrb_ngp_render': (_i, [_cfg, _tab, P, P, P, P, _i, _i, _f, _f, _f, _f, _u64, _i64, C.POINTER(C.c_float), _i, _i, P, P, P, P, P, P, P, P]),
    'xrb_ngp_render_depth': (_i, [_cfg, _tab, P, P, P, P, _i, _i, _f, _f, _f, _f, _u64, _i64, C.POINTER(C.c_float), _i, _i, P, P, P, P, P, P, P, P, P]),
    'xrb_ngp_render_fused_depth': (_i, [_cfg, _tab, P, P, P, P, _i, _f, _f, _f, _f, _u64, _i64, C.POINTER(C.c_float), _i, _i, P, P, P, P, P, P]),
    'xrb_ngp_density_lattice_workspace': (_sz, []),
    'xrb_ngp_density_lattice': (_i, [_cfg, _tab, P, P, _i, _i, _i, C.POINTER(C.c_float), C.POINTER(C.c_float), P, _i, P, P]),
    'xrb_mc_workspace': (_sz, [_i, _i, _i]),
    'xrb_mc_count': (_i, [P, _i, _i, _i, _f, P, P, P]),
    'xrb_mc_emit': (_i, [P, _i, _i, _i, _f, C.POINTER(C.c_float), C.POINTER(C.c_float), P, P, P, P]),
    'xrb_nerf_density_lattice': (_i, [P, P, _i, _i, _i, _i, _i, C.POINTER(C.c_float), C.POINTER(C.c_float), P, P]),
    'xrb_nerf_posenc_grad': (_i, [P, _i64, _i, P, _i, P, P, P]),
    'xrb_mip_ipe_tiles_points': (_i, [P, P, _i64, _i, _f, _i, _i, _i, _i, P, P]),
    'xrb_mip_density_lattice': (_i, [P, P, _i, _i, _f, _i, _i, _i, C.POINTER(C.c_float), C.POINTER(C.c_float), P, P]),
    'xrb_mip_ipe_grad': (_i, [P, _i64, _f, _i, _i, P, _i, P, P, P]),
    'xrb_ssim_workspace': (_sz, [_i, _i, _i]),
    'xrb_ssim': (_i, [P, P, _i, _i, _i, _i, C.c_double, P, P, P, P, _sz, P]),
}

EXPORTS = sorted(_SIGS)  # every symbol the header declares and the library currently implements
for _name, (_res, _args) in _SIGS.items():
    _fn = getattr(lib, _name)
    _fn.restype = _res
    _fn.argtypes = _args


XRB_E_BADARG = -1


class XrbError(RuntimeError):
    pass


def check(status, what=''):
    if status != 0:
        raise XrbError(f'{what} failed with status {status}: {lib.xrb_last_error().decode()}')


def ptr(t, dtype=None):
    """Device (or host) pointer of a DENSE tensor; None -> NULL.

    The kernels index `base + i * row_width`: a strided view (e.g. a Fortran-ordered `rays_o` that `torch.from_numpy` made
    from a `broadcast_to(...).reshape(...)` array) would be read as different data without any error, so it is rejected here
    with the library's bad-argument status instead (the reference's Python wrappers assert contiguity the same way,
    /root/reference/xrnerf/models/renders/hashnerf_render.py:76-96). Row-strided inputs go through `rows()`."""
    if t is None:
        return None
    if not t.is_contiguous():
        raise XrbError(f'XRB_E_BADARG ({XRB_E_BADARG}): non-contiguous tensor (shape {tuple(t.shape)}, strides {tuple(t.stride())}) passed to a kernel that '
                       'reads dense rows; call .contiguous() first')
    if dtype is not None and t.dtype != dtype:
        raise XrbError(f'XRB_E_BADARG ({XRB_E_BADARG}): expected {dtype}, got {t.dtype}')
    return C.c_void_p(t.data_ptr())


def f32(t):
    return ptr(t, torch.float32)


def i32(t):
    return ptr(t, torch.int32)


def u8(t):
    return ptr(t, torch.uint8)


def rows(t):
    """(pointer, row stride in floats) of a [n, >=3] float32 view whose rows are dense but may be spaced (coords[:, :3], coords[:, 4:])."""
    if t.dtype != torch.float32 or t.dim() != 2 or t.stride(1) != 1 or t.stride(0) < t.shape[1]:
        raise XrbError(f'XRB_E_BADARG ({XRB_E_BADARG}): expected float32 rows with unit inner stride, got {t.dtype} shape {tuple(t.shape)} strides {tuple(t.stride())}')
    return C.c_void_p(t.data_ptr()), int(t.stride(0))


def stream():
    # naming the current device skips torch's device discovery, which costs more host time than the lookup itself (a training step makes ~10 of these)
    return C.c_void_p(torch.cuda.current_stream(torch.cuda.current_device()).cuda_stream)


def float3(v):
    arr = (C.c_float * 3)(*[float(x) for x in v])
    return arr


def require_cuda(*tensors):
    for t in tensors:
        if t is not None and not t.is_cuda:
            raise XrbError('xrnerf_b200 kernels need CUDA tensors; there is no CPU fallback')
