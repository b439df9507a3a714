"""GPU parity of the tcnn-shaped boundary and of the fused HashNerfMLP field (CUDA-core impl 0 and wgmma impl 1) against
oracle/tcnn_oracle.c. Tolerances (stated, fp16 pipeline): encodings 1 fp16 ulp of the value range (2e-7 abs on 1e-4-scale
table entries), MLP outputs 2e-3 abs / 1e-2 rel (fp16 activations; accumulation order differs on tensor cores)."""
import numpy as np
import pytest
import torch
from cases import dev

pytestmark = pytest.mark.gpu


@pytest.fixture(scope='module')
def field_and_weights():
    from xrnerf_b200 import synth
    from xrnerf_b200.ngp import NgpField
    f = NgpField().cuda()
    # larger-than-default table values so the hash encoding actually matters in the outputs
    table, dens, color = synth.ngp_weights(seed=0, hash_range=0.5)
    with torch.no_grad():
        f.hash_params.copy_(dev(table)); f.density_params.copy_(dev(dens)); f.color_params.copy_(dev(color))
    return f, table, dens, color


def _pts(n, seed=0):
    rng = np.random.default_rng(seed)
    pts = rng.random((n, 3)).astype(np.float32)
    if n >= 3:
        pts[0] = 0.0; pts[1] = 1.0; pts[2] = [0.0, 1.0, 0.5]
    dirs = rng.random((n, 3)).astype(np.float32)
    return pts, dirs


def test_layout_matches_oracle(port, field_and_weights):
    import ctypes as C
    from xrnerf_b200 import _C
    f = field_and_weights[0]
    n, off, sc, res = port.hashgrid_layout()
    assert n == f.hash_params.numel() == 12196240
    o2 = (C.c_uint32 * 17)(); s2 = (C.c_float * 16)(); r2 = (C.c_uint32 * 16)()
    _C.check(_C.lib.xrb_tcnn_hashgrid_layout(f.cfg, o2, s2, r2))
    assert list(o2) == off.tolist() and list(r2) == res.tolist() and np.array_equal(np.array(list(s2), np.float32), sc)


def test_hashgrid_sh_mlp_modules(port, field_and_weights):
    import xrnerf_b200.tcnn as tcnn
    from xrnerf_b200.ngp import PER_LEVEL_SCALE
    f, table, dens, color = field_and_weights
    pts, dirs = _pts(5000)
    enc = tcnn.Encoding(3, dict(otype='HashGrid', n_levels=16, n_features_per_level=2, log2_hashmap_size=19, base_resolution=16, per_level_scale=PER_LEVEL_SCALE)).cuda()
    with torch.no_grad():
        enc.params.copy_(dev(table))
    e_gpu = enc(dev(pts)).detach().float().cpu().numpy()
    e_ref = port.hashgrid_forward(table, pts)
    assert e_gpu.shape == (5000, 32)
    assert np.abs(e_gpu - e_ref).max() <= 5e-4  # values up to 0.5 in fp16: 1 ulp = 2.4e-4
    sh = tcnn.Encoding(3, dict(otype='SphericalHarmonics', degree=4)).cuda()
    s_gpu = sh(dev(dirs)).float().cpu().numpy()
    assert np.abs(s_gpu - port.sh4(dirs)).max() <= 2e-3
    net = tcnn.Network(32, 16, dict(otype='FullyFusedMLP', activation='ReLU', output_activation='None', n_neurons=64, num_layers=1)).cuda()
    with torch.no_grad():
        net.params.copy_(dev(dens))
    x = e_ref.astype(np.float16)
    y_gpu = net(dev(x)).detach().float().cpu().numpy()
    y_ref = port.mlp_forward(dens, x.astype(np.float32), 64, 1)
    assert np.abs(y_gpu - y_ref).max() <= 2e-3 + 1e-2 * np.abs(y_ref).max()


@pytest.mark.parametrize('impl', [0, 1])
def test_gather_forms_are_bit_identical(field_and_weights, impl):
    """The cell image (one 256-bit record per grid cell) and the paired 64-bit loads return exactly the entries the 8 scalar gathers return, so the field
    output must not change by a single bit whichever levels are packed (0 = table only; 5 = the dense levels; 6, 7 = + the first hashed ones; 3 = a plan
    the static specialisation does not cover: run-time form)."""
    from xrnerf_b200.ngp import NgpField
    import xrnerf_b200.tcnn as tcnn
    from xrnerf_b200.ngp import PER_LEVEL_SCALE
    f0, table, dens, color = field_and_weights
    pts, dirs = _pts(70001, seed=9)
    pts[3] = [1.0, 0.0, 1.0]; pts[4] = [0.999999, 0.5, 1e-7]
    outs = []
    for npk in (0, 3, 5, 6, 7):
        f = NgpField(n_packed_levels=npk).cuda()
        with torch.no_grad():
            f.hash_params.copy_(dev(table)); f.density_params.copy_(dev(dens)); f.color_params.copy_(dev(color))
        outs.append((f.run_mlp(dev(pts), dev(dirs), impl=impl).clone(), f.run_density(dev(pts), impl=impl).clone()))
    for raw, den in outs[1:]:
        assert torch.equal(raw, outs[0][0]) and torch.equal(den, outs[0][1])
    if impl == 0:   # the stand-alone encoding reads the table only: it is the un-packed reference the cell image is checked against, entry by entry
        enc = tcnn.Encoding(3, dict(otype='HashGrid', n_levels=16, n_features_per_level=2, log2_hashmap_size=19, base_resolution=16, per_level_scale=PER_LEVEL_SCALE)).cuda()
        with torch.no_grad():
            enc.params.copy_(dev(table))
        e0 = enc(dev(pts))
        from xrnerf_b200 import _C
        f = NgpField(n_packed_levels=7).cuda()
        with torch.no_grad():
            f.hash_params.copy_(dev(table))
        f.refresh()
        e1 = torch.empty_like(e0)
        pts_d = dev(pts)
        xp, xs = _C.rows(pts_d)
        _C.check(_C.lib.xrb_tcnn_hashgrid_forward(f.cfg, f.tab, xp, xs, pts.shape[0], _C.ptr(e1), _C.stream()))
        assert torch.equal(e0, e1)


@pytest.mark.parametrize('impl', [0, 1])
def test_fused_field_vs_oracle(port, field_and_weights, impl):
    f, table, dens, color = field_and_weights
    for n in (1, 127, 128, 129, 5000, 40000):
        pts, dirs = _pts(n, seed=n)
        raw_ref = port.ngp_mlp_forward(table, dens, color, pts, dirs)
        raw = f.run_mlp(dev(pts), dev(dirs), impl=impl).cpu().numpy()
        assert raw.shape == (n, 4)
        assert np.isfinite(raw).all()
        err = np.abs(raw - raw_ref).max()
        assert err <= 2e-3 + 1e-2 * np.abs(raw_ref).max(), (impl, n, err)
        d_ref = port.ngp_density_forward(table, dens, pts)
        d = f.run_density(dev(pts), impl=impl).cpu().numpy().reshape(-1)
        assert np.abs(d - d_ref).max() <= 2e-3 + 1e-2 * np.abs(d_ref).max()


def test_fused_field_strided_views_and_impl_agreement(field_and_weights):
    f = field_and_weights[0]
    rng = np.random.default_rng(9)
    coords = dev(rng.random((10000, 7)).astype(np.float32))
    a = f.run_mlp(coords[:, :3], coords[:, 4:], impl=0)
    b = f.run_mlp(coords[:, :3], coords[:, 4:], impl=1)
    c = f.run_mlp(coords[:, :3].contiguous(), coords[:, 4:].contiguous(), impl=1)
    assert torch.equal(b, c)
    assert (a - b).abs().max().item() <= 2e-3 + 1e-2 * a.abs().max().item()


def test_deeper_networks(port):
    """n_hidden_layers up to 4 (tcnn's own default is 5 hidden layers when the reference's `num_layers` key is ignored, SURVEY Q7)."""
    from xrnerf_b200 import synth
    from xrnerf_b200.ngp import NgpField
    f = NgpField(density_hidden=2, color_hidden=3).cuda()
    table, dens, color = synth.ngp_weights(seed=2, dens_hidden=2, color_hidden=3, hash_range=0.5)
    with torch.no_grad():
        f.hash_params.copy_(dev(table)); f.density_params.copy_(dev(dens)); f.color_params.copy_(dev(color))
    pts, dirs = _pts(3000, seed=4)
    ref = port.ngp_mlp_forward(table, dens, color, pts, dirs, dens_hidden=2, color_hidden=3)
    for impl in (0, 1):
        raw = f.run_mlp(dev(pts), dev(dirs), impl=impl).cpu().numpy()
        assert np.abs(raw - ref).max() <= 3e-3 + 1e-2 * np.abs(ref).max()


@pytest.mark.parametrize('impl,n', [(0, 3000), (1, 3000), (1, 128), (1, 40001)])
def test_field_backward_vs_oracle(port, field_and_weights, impl, n):
    """gradients of the three parameter vectors: fp32 oracle backward on the fp16-rounded forward. impl 0 (CUDA cores) stages only dY in fp16 (x4096);
    impl 1 (wgmma: dX and dW as tensor-core instructions, dW accumulated in registers) rounds every layer's dZ to fp16 like tcnn does => 3e-3 relative to the
    largest gradient of each vector for both."""
    f, table, dens, color = field_and_weights
    pts, dirs = _pts(n, seed=21)
    rng = np.random.default_rng(2)
    draw = (rng.normal(0, 1, (n, 4)) * 1e-3).astype(np.float32)
    dt_ref, dd_ref, dc_ref = port.ngp_mlp_backward(table, dens, color, pts, dirs, draw)
    dt, dd, dc = f.backward_params(dev(pts), dev(dirs), dev(draw), impl=impl)
    for name, a, b in (('density', dd, dd_ref), ('color', dc, dc_ref), ('table', dt, dt_ref)):
        a = a.cpu().numpy()
        scale = np.abs(b).max()
        assert scale > 0
        err = np.abs(a - b)
        if impl == 0:
            assert err.max() <= 3e-3 * scale, (name, impl, n, err.max(), scale)
        else:
            # The tensor core sums a layer's products in another order than the oracle's sequential fma chain, so a pre-activation that is zero to within
            # ~1e-6 relative can land on the other side of ReLU: that sample's whole dZ element switches, which moves single dW entries by one term (measured:
            # 1 flip per ~5 M activations, 3.2e-3 of max at n = 40 001). The gradient is still the exact gradient of the forward this kernel's sibling
            # evaluates. A hash-table entry that only a few samples touch can therefore differ by a whole term (measured: 3 % of max on single entries). So: 3e-3 of
            # max in the L2 sense and for 99.9 % of the entries of every vector; no entry off by more than one sample's worth (the largest reference gradient).
            assert np.sqrt((err.astype(np.float64) ** 2).sum() / max((b.astype(np.float64) ** 2).sum(), 1e-300)) <= 3e-3, (name, n)
            assert np.quantile(err, 0.999) <= 3e-3 * scale and err.max() <= (2e-2 if name != 'table' else 1.0) * scale, (name, impl, n, err.max(), scale)
    if impl == 0:
        return
    # autograd bridge gives the same thing
    for p_ in (f.hash_params, f.density_params, f.color_params):
        p_.grad = None
    raw = f(dev(pts), dev(dirs))
    (raw * dev(draw)).sum().backward()
    assert torch.allclose(f.density_params.grad, dd, rtol=0, atol=1e-12 + 1e-6 * float(dd.abs().max()))


def test_adam_step_matches_torch():
    from xrnerf_b200 import _C
    torch.manual_seed(0)
    n = 100003
    p = torch.randn(n, device='cuda'); g = torch.randn(n, device='cuda') * 0.1
    ref = p.clone().requires_grad_(True)
    opt = torch.optim.Adam([ref], lr=1e-2, betas=(0.9, 0.99), eps=1e-15, weight_decay=1e-6)
    m = torch.zeros_like(p); v = torch.zeros_like(p); p16 = torch.empty(n, dtype=torch.float16, device='cuda')
    for step in range(1, 4):
        ref.grad = g.clone() * step
        opt.step()
        _C.check(_C.lib.xrb_adam_ema_step(_C.ptr(p), _C.ptr(p16), _C.ptr(g * step * 2.0), _C.ptr(m), _C.ptr(v), n, 1e-2, 0.9, 0.99, 1e-15, 1e-6, step, 2.0, None, 0.0,
                                          _C.stream()))
    assert torch.allclose(p, ref.detach(), rtol=1e-5, atol=1e-6)
    assert torch.equal(p16, p.half())


def test_adam_ema_step_matches_torch_and_mmcv_ema_rule():
    """xrb_adam_ema_step == torch.optim.Adam followed by mmcv's EMAHook.after_train_iter (buffer.mul_(1 - m).add_(m * param),
    m = min(momentum, (1 + iter) / (warm_up + iter)), buffers initialised as copies): configs/instant_ngp/nerf_blender_local01.py:24."""
    from xrnerf_b200 import _C
    torch.manual_seed(1)
    n = 70001
    p = torch.randn(n, device='cuda'); g = torch.randn(n, device='cuda') * 0.1
    ref = p.clone().requires_grad_(True)
    opt = torch.optim.Adam([ref], lr=1e-2, betas=(0.9, 0.99), eps=1e-15, weight_decay=1e-6)
    ema_ref = p.clone(); ema = p.clone()
    m = torch.zeros_like(p); v = torch.zeros_like(p)
    for step in range(1, 9):
        ref.grad = g.clone() * (1 + 0.1 * step)
        opt.step()
        it = step - 1
        mom = min(0.05, (1 + it) / (100 + it))
        ema_ref.mul_(1 - mom).add_(ref.detach(), alpha=mom)
        _C.check(_C.lib.xrb_adam_ema_step(_C.ptr(p), None, _C.ptr(g * (1 + 0.1 * step)), _C.ptr(m), _C.ptr(v), n, 1e-2, 0.9, 0.99, 1e-15, 1e-6, step, 1.0, _C.ptr(ema), mom, _C.stream()))
    assert torch.allclose(p, ref.detach(), rtol=1e-5, atol=1e-6)
    assert torch.allclose(ema, ema_ref, rtol=1e-5, atol=1e-6)


def test_tcnn_modules_train_like_the_fused_field(field_and_weights):
    """The reference's HashNerfMLP.run_mlp (hashnerf_mlp.py:55-79) written against `xrnerf_b200.tcnn` exactly as it is written against tinycudann, under
    torch.autograd: the parameter gradients of the four composable modules equal the fused field's backward (same arithmetic; fp16 activation gradients between
    the modules, as tcnn's bindings have): 5e-3 relative L2, 1e-2 of max per vector. Flat-parameter import/export feeds the modules."""
    import xrnerf_b200.tcnn as tcnn
    from xrnerf_b200.ngp import PER_LEVEL_SCALE
    f, table, dens, color = field_and_weights
    enc = tcnn.Encoding(3, dict(otype='HashGrid', n_levels=16, n_features_per_level=2, log2_hashmap_size=19, base_resolution=16, per_level_scale=PER_LEVEL_SCALE)).cuda()
    sh = tcnn.Encoding(3, dict(otype='SphericalHarmonics', degree=4)).cuda()
    dnet = tcnn.Network(32, 16, dict(otype='FullyFusedMLP', activation='ReLU', output_activation='None', n_neurons=64, num_layers=1)).cuda()
    cnet = tcnn.Network(31, 3, dict(otype='FullyFusedMLP', activation='ReLU', output_activation='None', n_neurons=64, num_layers=2)).cuda()
    enc.import_params(dev(table)); dnet.import_params(dev(dens)); cnet.import_params(dev(color))
    assert torch.equal(enc.export_params(), dev(table)) and torch.equal(cnet.export_params(), dev(color))
    n = 6000
    pts, dirs = _pts(n, seed=33)
    rng = np.random.default_rng(4)
    draw = dev((rng.normal(0, 1, (n, 4)) * 0.05).astype(np.float32))     # large enough for fp16 activation gradients
    h = enc(dev(pts))
    d_out = dnet(h)
    c_out = cnet(torch.cat([d_out[..., 1:], sh(dev(dirs))], dim=-1))
    out = torch.cat([c_out, d_out[..., :1]], -1).to(torch.float32).contiguous()
    raw_fused = f.run_mlp(dev(pts), dev(dirs), impl=0)
    assert float((out.detach() - raw_fused).abs().max()) <= 2e-3 + 1e-2 * float(raw_fused.abs().max())
    (out * draw).sum().backward()
    dt, dd, dc = f.backward_params(dev(pts), dev(dirs), draw, impl=0)
    for name, a, b in (('table', enc.params.grad, dt), ('density', dnet.params.grad, dd), ('color', cnet.params.grad, dc)):
        assert a is not None and a.dtype == torch.float32 and a.shape == b.shape
        err = (a - b).abs()
        assert float(torch.sqrt((err.double() ** 2).sum() / (b.double() ** 2).sum())) <= 5e-3, name
        assert float(err.max()) <= 1e-2 * float(b.abs().max()), (name, float(err.max()), float(b.abs().max()))
    # one optimiser step through the modules changes their output (they are trainable end to end)
    opt = torch.optim.Adam([enc.params, dnet.params, cnet.params], lr=1e-2)
    opt.step()
    assert not torch.equal(enc(dev(pts)), h.detach())
