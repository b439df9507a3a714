"""NerfMLP / HashNerfMLP with the reference's kwargs, state_dict keys and data-dict protocol
(/root/reference/xrnerf/models/mlps/nerf_mlp.py:11-94, hashnerf_mlp.py:23-111)."""
import torch
import torch.nn.functional as F
from torch import nn

from . import builder
from .builder import MLPS
from ..ngp import NgpField, PER_LEVEL_SCALE


@MLPS.register_module()
class BaseMLP(nn.Module):
    def __init__(self, **kwarg):
        super().__init__()


@MLPS.register_module()
class NerfMLP(BaseMLP):
    """8x256 ReLU MLP with skip at layer 4 and a 128-wide view branch; parameters are nn.Linear modules with the reference's
    names (pts_linears.i, views_linears.0, feature_linear, alpha_linear, rgb_linear) so reference checkpoints load.

    Inference (no_grad) runs the whole chain in ONE persistent wgmma kernel (csrc/nerf_mlp_tc.cu; fp16 operands, fp32 accumulate).
    With autograd enabled (training) run_mlp is ONE autograd node whose forward and backward are wgmma kernels over fp16 tile images
    (xrnerf_b200/nerf_train.py, csrc/nerf_train.cu); `fused_train = False` (or an unsupported shape) falls back to nn.Linear under autograd."""

    def __init__(self, skips=[4], netdepth=8, netwidth=256, output_ch=4, use_viewdirs=True, netchunk=1024 * 32, embedder=None, fused=True, **kwarg):
        super().__init__()
        self.skips, self.chunk, self.use_viewdirs, self.fused = skips, netchunk, use_viewdirs, fused
        self.embedder = builder.build_embedder(embedder)
        D, W = netdepth, netwidth
        self.input_ch, self.input_ch_dirs = self.embedder.get_embed_ch()
        self.pts_linears = nn.ModuleList([nn.Linear(self.input_ch, W)] + [nn.Linear(W, W) if i not in self.skips else nn.Linear(W + self.input_ch, W) for i in range(D - 1)])
        if self.use_viewdirs:
            self.views_linears = nn.ModuleList([nn.Linear(self.input_ch_dirs + W, W // 2)])
            self.feature_linear = nn.Linear(W, W)
            self.alpha_linear = nn.Linear(W, 1)
            self.rgb_linear = nn.Linear(W // 2, 3)
        else:
            self.output_linear = nn.Linear(W, output_ch)

    def forward(self, data):
        data = self.embedder(data)
        out = self.batchify_run_mlp(data['embedded'])
        data['raw'] = torch.reshape(out, list(data['unflatten_shape']) + [out.shape[-1]])
        del data['unflatten_shape']
        return data

    # the packed wgmma weight image is keyed on Parameter._version, which writes through `.data` (EMAHook swap, load_state_dict, .to()) do not bump
    def mark_dirty(self):
        self._pack_ver = None

    def _apply(self, fn, *a, **kw):
        self._pack_ver = None
        return super()._apply(fn, *a, **kw)

    def _load_from_state_dict(self, *a, **kw):
        self._pack_ver = None
        return super()._load_from_state_dict(*a, **kw)

    def _fused_ok(self, x):
        from ..nerf_mlp import fused_shape
        return self.fused and not torch.is_grad_enabled() and x.is_cuda and fused_shape(self)

    def _is_mip(self):
        return hasattr(self.embedder, 'min_deg')

    def _mesh_check(self, x):
        """mesh export runs the fused kernels only, for the reference NeRF shape with the positional encoding of multires 10 (input channels (63, 27)) or
        the reference Mip-NeRF IPE (point degrees 0..16, view degrees 0..4: (96, 27)): anything else is an error"""
        from ..nerf_mlp import fused_shape
        e = self.embedder
        enc_ok = ((e.min_deg, e.max_deg, e.min_deg_view, e.max_deg_view) == (0, 16, 0, 4)) if self._is_mip() else (getattr(e, 'multires', None) == 10)
        if not (self.fused and x.is_cuda and fused_shape(self) and enc_ok):
            raise NotImplementedError('NerfMLP mesh export is implemented for the fused CUDA NerfMLP(netdepth=8, netwidth=256, skips=[4], use_viewdirs=True) '
                                      'with BaseEmbedder(multires=10, multires_dirs=4) (input channels (63, 27)) or MipNerfEmbedder(min_deg_point=0, '
                                      'max_deg_point=16, min_deg_view=0, max_deg_view=4) (input channels (96, 27)) on a CUDA device')

    def _footprint(self, footprint, shape=None, box=None):
        """the point query's sigma (Mip-NeRF), or None (NeRF): a MipNerfEmbedder needs a footprint, a BaseEmbedder takes none"""
        from ..mesh import footprint_sigma
        if not self._is_mip():
            if footprint is not None:
                raise ValueError('a BaseEmbedder NerfMLP is defined at points: footprint must be None')
            return None
        if footprint is None:
            raise NotImplementedError('a Mip-NeRF field is defined on conical frusta, and a point query needs a chosen footprint: pass footprint=sigma or \'cell\'')
        return footprint_sigma(footprint, shape, box)

    def density_lattice(self, shape, box, footprint=None):
        """Raw alpha on the lattice of shape (nz, ny, nx) over box = (box_min, box_max) -> CUDA f32[nz,ny,nx] (x fastest); lattice positions:
        xrb_nerf_density_lattice (include/xrnerf_b200.h). Each value is bit-identical to the inference raw[:, 3] (nerf_mlp_forward on the
        xrb_nerf_posenc_tiles encoding of the point).

        With a MipNerfEmbedder the field is a point query at footprint sigma (xrb_mip_density_lattice: the IPE of the isotropic Gaussian of standard
        deviation sigma at the point, bit-identical to nerf_mlp_forward on the xrb_mip_ipe_tiles_points encoding): `footprint` is sigma >= 0 in the
        rays' world frame, or 'cell' (mesh.footprint_sigma: the standard deviation of a uniform distribution over one lattice cell). A BaseEmbedder takes
        footprint=None."""
        from ..nerf_mlp import density_lattice
        w = self.pts_linears[0].weight
        self._mesh_check(w)
        shape = tuple(int(n) for n in shape)
        sigma = self._footprint(footprint, shape, box)
        image, bias = self._packed()
        out = torch.empty(shape, dtype=torch.float32, device=w.device)
        density_lattice(self, sigma, image, bias, shape, box, out)
        return out

    def density_grad(self, pts, footprint=None):
        """pts f32[n,3] in the frame the rays are given in -> (raw density f32[n], grad f32[n,3] = d(raw alpha)/d(position)). Computed with the training
        kernels (xrnerf_b200.nerf_train.density_grad: forward with saved activations, then the input gradients from alpha_linear down to the point
        encoding); that forward's density agrees with the inference kernel's, which density_lattice uses, to the fp16 tolerance, not bit for bit.
        With a MipNerfEmbedder, `footprint` is the point query's sigma >= 0 (required; 'cell' needs a lattice, so it is not accepted here); a
        BaseEmbedder takes footprint=None."""
        self._mesh_check(pts)
        sigma = self._footprint(footprint)
        from .. import nerf_train
        with torch.no_grad():
            return nerf_train.density_grad(self, pts.detach().reshape(-1, 3).contiguous().float(), sigma=sigma)

    def density_grad_rays(self, rays_o, rays_d, z_vals, radii=None, enc=None):
        """The raw density and its gradient at every sample of a set of rays -> (density f32[n*S], grad f32[n*S,3]), from one tensor-core kernel
        (xrb_nerf_density_grad_rays / xrb_mip_density_grad_rays, include/xrnerf_b200.h "NeRF / Mip-NeRF normal maps"): rays_o, rays_d f32[n,3];
        z_vals f32[n,S] (BaseEmbedder: positions o + d z) or, with a MipNerfEmbedder, f32[n,S+1] interval ends and radii f32[n] (positions: the
        frustum Gaussians' means). enc: the rows' encoding tile image (None: formed here by the renderer's encoder, xrnerf_b200.nerf.encode_rays).
        density is bit-identical to the inference kernel's raw[:, 3] on that image."""
        from ..nerf import density_grad_rays, encode_rays
        self._mesh_check(rays_o)
        o, d, z = (t.contiguous().float() for t in (rays_o, rays_d, z_vals))
        rad = None if radii is None else radii.reshape(-1).contiguous().float()
        n, s = z.shape[0], z.shape[1] - (1 if self._is_mip() else 0)
        if enc is None:
            enc = encode_rays(self, o, d, d, z, rad)
        density = torch.empty(n * s, dtype=torch.float32, device=o.device)
        grad = density_grad_rays(self, enc, o, d, z, rad, density)
        return density, grad

    def _packed(self, grad=False):
        """(weight image, bias) of pack_nerf_mlp, and with grad=True also pack_nerf_mlp_grad's image of the same weights; each is packed once per weight
        version (mark_dirty forgets both)"""
        ver = tuple(p._version for p in self.parameters()) + (self.pts_linears[0].weight.device,)
        if getattr(self, '_pack_ver', None) != ver:
            from ..nerf_mlp import pack_nerf_mlp
            self._pack = pack_nerf_mlp(self)
            self._pack_grad = None
            self._pack_ver = ver
        if not grad:
            return self._pack
        if self._pack_grad is None:
            from ..nerf_mlp import pack_nerf_mlp_grad
            self._pack_grad = pack_nerf_mlp_grad(self)
        return self._pack + (self._pack_grad,)

    def batchify_run_mlp(self, x):
        if self._fused_ok(x):   # inference: the whole 12-GEMM chain in one wgmma kernel, no chunking needed (activations never leave the SM)
            from ..nerf_mlp import nerf_mlp_forward
            image, bias = self._packed()
            return nerf_mlp_forward(image, bias, x, self.input_ch, self.input_ch_dirs)
        if self.fused and getattr(self, 'fused_train', True) and torch.is_grad_enabled() and x.is_cuda and any(p.requires_grad for p in self.parameters()):
            from .. import nerf_train
            if nerf_train.supported(self):   # training: every dense layer forward + backward as wgmma kernels over fp16 tile images (csrc/nerf_train.cu), one autograd node
                return nerf_train.run_mlp_train(self, x)
        if self.chunk is None:
            return self.run_mlp(x)
        return torch.cat([self.run_mlp(x[i:i + self.chunk]) for i in range(0, x.shape[0], self.chunk)], 0)

    def run_mlp(self, x):
        input_pts, input_views = torch.split(x, [self.input_ch, self.input_ch_dirs], dim=-1)
        h = input_pts
        for i, l in enumerate(self.pts_linears):
            h = F.relu(l(h))
            if i in self.skips:
                h = torch.cat([input_pts, h], -1)
        if self.use_viewdirs:
            alpha = self.alpha_linear(h)
            h = torch.cat([self.feature_linear(h), input_views], -1)
            for l in self.views_linears:
                h = F.relu(l(h))
            return torch.cat([self.rgb_linear(h), alpha], -1)
        return self.output_linear(h)


class _ParamHolder(nn.Module):
    """gives a flat parameter the reference's state_dict key `<name>.params` (tcnn modules expose exactly one `params`)"""

    def __init__(self, p):
        super().__init__()
        self.params = p


def _hidden(network_config):
    if 'n_hidden_layers' in network_config:
        return int(network_config['n_hidden_layers'])
    return int(network_config.get('num_layers', 5))  # SURVEY Q7: the reference's key is num_layers; tcnn's default would be 5


@MLPS.register_module()
class HashNerfMLP(BaseMLP):
    """state_dict keys: embedder_pos.params, embedder_dir.params (empty), density_net.params, color_net.params."""

    def __init__(self, bound=1, embedder_pos=None, embedder_dir=None, density_net=None, color_net=None, impl=1, **kwarg):
        super().__init__()
        enc = dict(embedder_pos['encoding_config'])
        if enc.get('otype') != 'HashGrid' or embedder_dir['encoding_config'].get('otype') != 'SphericalHarmonics' or int(embedder_dir['encoding_config'].get('degree', 4)) != 4:
            raise NotImplementedError('HashNerfMLP: HashGrid position encoding + SphericalHarmonics degree 4 (the reference config)')
        if int(density_net['n_output_dims']) != 16 or int(color_net['n_output_dims']) != 3:
            raise NotImplementedError('HashNerfMLP: density_net 16 outputs, color_net 3 outputs (the reference config)')
        field = NgpField(n_levels=int(enc.get('n_levels', 16)), n_features=int(enc.get('n_features_per_level', 2)), log2_hashmap_size=int(enc.get('log2_hashmap_size', 19)),
                              base_resolution=int(enc.get('base_resolution', 16)), per_level_scale=PER_LEVEL_SCALE,  # get_per_level_scale(1): ignores `bound` (Q6)
                              width=int(density_net['network_config'].get('n_neurons', 64)), density_hidden=_hidden(density_net['network_config']),
                              color_hidden=_hidden(color_net['network_config']), impl=impl)
        # not registered as a sub-module: its Parameters are the very objects held by the four tcnn-named holders below, so
        # state_dict()/load_state_dict() see exactly the reference's keys and .to()/.cuda() (in-place on .data) still moves them
        self.__dict__['field'] = field
        f = field
        self.embedder_pos = _ParamHolder(f.hash_params)
        self.embedder_dir = _ParamHolder(nn.Parameter(torch.zeros(0)))
        self.density_net = _ParamHolder(f.density_params)
        self.color_net = _ParamHolder(f.color_params)

    # the fused field caches fp16 shadows, the cell image and the wgmma weight image keyed on Parameter._version, which writes through `.data` (mmcv's EMAHook,
    # load_state_dict's copy_, .to()) do not bump: every such entry point marks the caches dirty (ADVICE r1, medium)
    def _apply(self, fn, *a, **kw):
        self.field.mark_dirty()
        return super()._apply(fn, *a, **kw)

    def _load_from_state_dict(self, *a, **kw):
        self.field.mark_dirty()
        return super()._load_from_state_dict(*a, **kw)

    def load_state_dict(self, *a, **kw):
        self.field.mark_dirty()
        return super().load_state_dict(*a, **kw)

    def mark_dirty(self):
        self.field.mark_dirty()

    def forward(self, data):
        shape = data['pts'].shape[:-1]
        out = self.run_mlp(data)
        data['raw'] = torch.reshape(out, list(shape) + [out.shape[-1]])
        return data

    def run_mlp(self, data):
        pts, viewdirs = data['pts'], data['viewdirs']
        if pts.dim() > viewdirs.dim():
            viewdirs = viewdirs[:, None].expand(pts.shape)
        pts, viewdirs = pts.reshape(-1, 3).detach(), viewdirs.reshape(-1, 3).detach()
        if pts.stride(-1) != 1:
            pts = pts.contiguous()
        if viewdirs.stride(-1) != 1:
            viewdirs = viewdirs.contiguous()
        return self.field(pts.float(), viewdirs.float())

    def run_density(self, pts_flat):
        return self.field.run_density(pts_flat.float() if pts_flat.stride(-1) == 1 else pts_flat.contiguous().float())
