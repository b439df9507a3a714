"""tcnn-shaped boundary (#2): the subset of `tinycudann`'s PyTorch API the reference's HashNerfMLP uses
(/root/reference/xrnerf/models/mlps/hashnerf_mlp.py:11, :36-45, :55-79, :107-111):

    tcnn.Encoding(n_input_dims, encoding_config)   -> module with .n_output_dims, .params, __call__([S,3] f32) -> [S,D] f16
    tcnn.Network(n_input_dims, n_output_dims, network_config) -> module with .params, __call__([S,Din]) -> [S,Dout] f16

so `import xrnerf_b200.tcnn as tcnn` lets the reference module run on these kernels. Each module owns one flat fp32
`params` nn.Parameter (tcnn's master-parameter layout: hash table levels back to back; MLP weight matrices W[out][in]
row-major, first/hidden/last) and a cached fp16 working copy refreshed when `params` changes.
Both modules are trainable like tcnn's: `params` receives gradients through torch.autograd (Encoding: table gradient by scatter; Network: input and
parameter gradients), in the dtypes tcnn's bindings use (fp16 activations and activation gradients, fp32 parameter gradients), so the reference's
`HashNerfMLP.run_mlp` (hashnerf_mlp.py:55-79) trains through them unchanged. The fused fast path (one kernel for encodings + both MLPs, wgmma forward and
backward) lives in xrnerf_b200.ngp.NgpField; these modules are the composable building blocks behind the same parameter layouts:
`export_params()` / `import_params()` move a flat tcnn parameter vector in and out (checkpoint compatibility, SURVEY §8f-4).
"""
import math

import torch
from torch import nn

from . import _C


def _n_hidden(network_config):
    # tcnn's key is n_hidden_layers; the reference's config writes `num_layers` (configs/instant_ngp/nerf_blender_local01.py:113,123).
    # SURVEY §8c / Appendix B Q7: accept both, read `num_layers` as the hidden-layer count.
    if 'n_hidden_layers' in network_config:
        return int(network_config['n_hidden_layers'])
    if 'num_layers' in network_config:
        return int(network_config['num_layers'])
    return 5  # tcnn default


class _Fp16Shadow:
    """fp16 working copy of an fp32 master parameter, re-cast only when the master changed."""

    def __init__(self):
        self.buf, self.version = None, None

    def get(self, p):
        if self.buf is None or self.buf.device != p.device or self.version != p._version or self.buf.numel() != p.numel():
            self.buf = torch.empty(p.numel(), dtype=torch.float16, device=p.device)
            _C.check(_C.lib.xrb_tcnn_cast_params(_C.ptr(p.detach()), _C.ptr(self.buf), p.numel(), _C.stream()), 'cast_params')
            self.version = p._version
        return self.buf


class _EncodingFn(torch.autograd.Function):
    """HashGrid forward = xrb_tcnn_hashgrid_forward; backward scatters dL/d enc into the fp32 table gradient (positions are not differentiated: the
    reference detaches them, hashnerf_mlp.py:58-59)."""

    @staticmethod
    def forward(ctx, mod, x, params):
        ctx.mod = mod
        ctx.save_for_backward(x)
        return mod._forward(x)

    @staticmethod
    def backward(ctx, g):
        mod = ctx.mod
        x, = ctx.saved_tensors
        d = torch.zeros_like(mod.params, dtype=torch.float32)
        g = g.contiguous().to(torch.float16)
        xp, xs = _C.rows(x)
        _C.check(_C.lib.xrb_tcnn_hashgrid_backward(mod.cfg, xp, xs, x.shape[0], _C.ptr(g), 1.0, _C.ptr(d), _C.stream()), 'hashgrid_backward')
        return None, None, d


class _NetworkFn(torch.autograd.Function):
    """FullyFusedMLP forward = xrb_tcnn_mlp_forward; backward = xrb_tcnn_mlp_backward (recomputes the hidden activations; dX fp16, dW fp32)."""

    @staticmethod
    def forward(ctx, mod, x16, params):
        ctx.mod = mod
        ctx.save_for_backward(x16)
        return mod._forward(x16)

    @staticmethod
    def backward(ctx, g):
        mod = ctx.mod
        x16, = ctx.saved_tensors
        n = x16.shape[0]
        g16 = torch.zeros((n, mod.out_pad), dtype=torch.float16, device=x16.device)
        g16[:, :g.shape[1]] = g
        d = torch.zeros_like(mod.params, dtype=torch.float32)
        dx = torch.empty((n, mod.in_pad), dtype=torch.float16, device=x16.device) if ctx.needs_input_grad[1] else None
        _C.check(_C.lib.xrb_tcnn_mlp_backward(_C.ptr(mod._shadow.get(mod.params)), _C.ptr(x16), _C.ptr(g16), n, mod.in_pad, mod.width, mod.n_hidden, _C.ptr(dx), _C.ptr(d),
                                              _C.stream()), 'mlp_backward')
        return None, dx, d


class _ParamIO:
    """flat-parameter import / export in tcnn's layout (`module.params` of the tcnn torch bindings; state_dict key `<name>.params`)"""

    def export_params(self):
        return self.params.detach().clone()

    def import_params(self, flat):
        flat = torch.as_tensor(flat)
        if flat.numel() != self.params.numel():
            raise ValueError(f'{type(self).__name__}: expected {self.params.numel()} parameters (tcnn layout), got {flat.numel()}')
        with torch.no_grad():
            self.params.copy_(flat.reshape(-1).to(self.params.dtype))
        self._shadow.version = None                      # the fp16 working copy is rebuilt on the next forward


class Encoding(nn.Module, _ParamIO):
    def __init__(self, n_input_dims, encoding_config, seed=1337):
        super().__init__()
        self.n_input_dims = int(n_input_dims)
        self.encoding_config = dict(encoding_config)
        otype = self.encoding_config.get('otype')
        self._shadow = _Fp16Shadow()
        if otype in ('HashGrid', 'Grid'):
            c = self.encoding_config
            self.cfg = _C.NgpConfig(int(c.get('n_levels', 16)), int(c.get('n_features_per_level', 2)), int(c.get('log2_hashmap_size', 19)),
                                    int(c.get('base_resolution', 16)), float(c.get('per_level_scale', 2.0)), 64, 1, 1)
            n = _C.lib.xrb_tcnn_hashgrid_num_params(self.cfg)
            if n < 0:
                raise _C.XrbError(_C.lib.xrb_last_error().decode())
            g = torch.Generator().manual_seed(seed)
            self.params = nn.Parameter((torch.rand(n, generator=g) * 2 - 1) * 1e-4)  # tcnn: U(-1e-4, 1e-4)
            self.n_output_dims = self.cfg.n_levels * self.cfg.n_features
            self.kind = 'hash'
        elif otype == 'SphericalHarmonics':
            if int(self.encoding_config.get('degree', 4)) != 4:
                raise NotImplementedError('SphericalHarmonics: only degree 4 (the reference config) is implemented')
            self.params = nn.Parameter(torch.zeros(0))
            self.n_output_dims = 16
            self.kind = 'sh'
        else:
            raise NotImplementedError(f'encoding otype {otype!r}')

    def forward(self, x):
        _C.require_cuda(x)
        x = x.detach().to(torch.float32)
        if x.stride(-1) != 1:
            x = x.contiguous()
        if self.kind == 'hash' and torch.is_grad_enabled() and self.params.requires_grad:
            return _EncodingFn.apply(self, x, self.params)
        return self._forward(x)

    def _forward(self, x):
        n = x.shape[0]
        out = torch.empty((n, self.n_output_dims), dtype=torch.float16, device=x.device)
        if self.kind == 'hash':
            tab = _C.NgpTable(self._shadow.get(self.params).data_ptr(), None, 0)
            xp, xs = _C.rows(x)
            _C.check(_C.lib.xrb_tcnn_hashgrid_forward(self.cfg, tab, xp, xs, n, _C.ptr(out), _C.stream()), 'hashgrid_forward')
        else:
            xp, xs = _C.rows(x)
            _C.check(_C.lib.xrb_tcnn_sh4_forward(xp, xs, n, _C.ptr(out), _C.stream()), 'sh4_forward')
        return out


class Network(nn.Module, _ParamIO):
    def __init__(self, n_input_dims, n_output_dims, network_config, seed=1337):
        super().__init__()
        self.n_input_dims, self.n_output_dims = int(n_input_dims), int(n_output_dims)
        self.network_config = dict(network_config)
        self.width = int(self.network_config.get('n_neurons', 64))
        self.n_hidden = _n_hidden(self.network_config)
        if self.network_config.get('activation', 'ReLU') != 'ReLU' or self.network_config.get('output_activation', 'None') != 'None':
            raise NotImplementedError('FullyFusedMLP: only ReLU hidden / None output activations (the reference config)')
        self.in_pad = (self.n_input_dims + 15) // 16 * 16   # tcnn.Network pads its input to a multiple of 16 with ones
        self.out_pad = (self.n_output_dims + 15) // 16 * 16
        if self.in_pad != 32 or self.width != 64 or self.out_pad != 16 or not (1 <= self.n_hidden <= 4):
            raise NotImplementedError('FullyFusedMLP: implemented for (<=32 in, 64 wide, <=16 out, 1..4 hidden layers)')
        shapes = [(self.width, self.in_pad)] + [(self.width, self.width)] * (self.n_hidden - 1) + [(self.out_pad, self.width)]
        g = torch.Generator().manual_seed(seed)
        mats = []
        for (o, i) in shapes:  # tcnn: Xavier-uniform per matrix
            s = math.sqrt(6.0 / (i + o))
            mats.append(((torch.rand(o, i, generator=g) * 2 - 1) * s).reshape(-1))
        self.params = nn.Parameter(torch.cat(mats))
        self._shadow = _Fp16Shadow()

    def forward(self, x):
        _C.require_cuda(x)
        n = x.shape[0]
        x = x.to(torch.float16)
        if x.shape[1] != self.in_pad:                    # tcnn.Network pads its input to a multiple of 16 with ones
            x = torch.cat([x, torch.ones((n, self.in_pad - x.shape[1]), dtype=torch.float16, device=x.device)], 1)
        x = x.contiguous()
        if torch.is_grad_enabled() and (self.params.requires_grad or x.requires_grad):
            return _NetworkFn.apply(self, x, self.params)[:, :self.n_output_dims]
        return self._forward(x.detach())[:, :self.n_output_dims]

    def _forward(self, x):
        n = x.shape[0]
        y = torch.empty((n, self.out_pad), dtype=torch.float16, device=x.device)
        _C.check(_C.lib.xrb_tcnn_mlp_forward(_C.ptr(self._shadow.get(self.params)), _C.ptr(x), n, self.in_pad, self.width, self.n_hidden, _C.ptr(y), _C.stream()),
                 'mlp_forward')
        return y
