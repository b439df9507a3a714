"""The NGP field (forward and backward, every kernel instantiation) against a float64 restatement of its arithmetic whose ReLU decisions are
proven stable, entry by entry.

Reference (numpy, float64; oracle/tcnn_oracle.c's network): W[out][in] row-major fp16 weights, ReLU hidden layers, fp16 activations,
colour input dout[1:16] ++ SH16 ++ 1.0, raw = (cout[0:3], dout[0]). Its inputs are the kernels' own bits: the encodings come from
xrb_tcnn_hashgrid_forward on the field's table (the field kernels call the same hash_level() and round with the same fp16 RNE) and the SH values
from xrb_tcnn_sh4_forward (the same sh4()). test_forward_within_derived_bound is what shows these are the values the field kernels use.

Forward error bound, propagated per unit and layer. z = W16 x in float64; the kernel's pre-activation differs from z by at most
    b = |W16| e_x + gamma (|W16| (|x| + e_x))
(e_x: bound on the kernel's input minus ours; gamma bounds fp32 accumulation of K exact fp16 x fp16 products: K 2^-22 on the tensor cores, whose
adder this covers, and K 2^-24 (1 + 2^-16) for the CUDA-core kernels' chain of K fma). Rounding and ReLU are monotone, so the kernel's activation
fp16(relu(.)) lies in [fp16(relu(z-b)), fp16(relu(z+b))]: it is within e_a = the larger distance from ours, a = fp16(relu(z)), to either end
(0 when they coincide). A sample is REJECTED when some hidden unit's decision a > 0 differs between z-b and z+b: only there can the kernel take
the other ReLU branch. Rejected samples get dL/draw = 0 on both sides, so they contribute exactly nothing to either gradient. The bound is a worst
case over 64-wide layers, so it grows with depth: the rejected fraction is about 1-20 % for the (1,1) and (1,2) networks and more for deeper
ones (measured per case and printed); at least a third of every batch must be stable.

Backward (float64, exact, on the stable samples, whose masks are the kernel's): dW = sum_s dZ (x) x, dX = W^T dZ, dL/denc scattered with
trilinear weights at tcnn's grid_index (restated here in numpy). The same chain on absolute values (|W|, |dZ|, |x|, the scatter of |dL/denc|)
gives each entry's contribution mass M. Every entry of the table, density and colour gradients must satisfy
    |g_kernel - g64| <= (tau + D 2^-23) M' + (1 + tau) E
  * tau = (R + 1) 2^-11 with R the fp16 roundings on a gradient's path: the wgmma kernel stages every layer's dZ in fp16 (R = number of linear
    layers: 4 for (1,1), 5 for (1,2)); the CUDA-core kernel stages only the dY its dW GEMM reads (R = 1; its dX chain and the table scatter are
    fp32). A staged value v comes back as v (1 + d) + h with |d| <= 2^-11 and |h| <= 2^-25 / 4096 (half the fp16 subnormal step at the 2^12
    staging scale), so to first order the final error is 2^-11 times the absolute chain of (|v| + 2^-26) at every staging point: M' is M with
    that floor (the epsilon of the bound) added to every live staged value. The "+1" covers fp32 accumulation along the dX chain
    (sum_l K_l 2^-22 < 2^-11 for these widths) and the second-order terms.
  * D bounds the depth of the fp32 sums into one entry: dW entries are per-tile partial sums (<= 128 samples, +64 for the tensor-core adder)
    added across <= ceil(n/128) tiles, D = 192 + ceil(n/128); a table entry receives its c contributions with atomics in any order, and each
    contribution carries <= 6 fp32 roundings from the trilinear weight, D = c + 8. (2^-23 is twice the fp32 unit roundoff.)
  * E = |dZ|^T e_x: the kernel's activations may differ from ours by e_x where the fp16 rounding of an activation is ambiguous.
Nothing in tau, D or the floor is fitted to a run.
"""
import time

import numpy as np
import pytest
import torch
from cases import dev, load_ngp_weights
from restate64 import GAMMA_TC, U16, Grid, f16, hashgrid_enc16, ngp_mats, ulp16

pytestmark = pytest.mark.gpu

SCALE = 4096.0              # staging scale of dZ / dY in both backward kernels
FLOOR = 2.0 ** -26          # (2^-25 / SCALE) / U16: the subnormal half-step at the staging scale, as a floor on the staged magnitude
REJECT_CEILING = 2.0 / 3.0  # a batch with more rejected samples than this does not test enough
GAMMA_FMA = 2.0 ** -24 * (1 + 2.0 ** -16)   # per-term accumulation bound of a K-term dot product as a chain of K fp32 fma (the CUDA-core kernels): K u / (1 - K u), K <= 64
REPORT = []


def _layer(W, x, ex, relu, gamma_unit, rnd=f16):
    aW = np.abs(W)
    z = x @ W.T
    b = ex @ aW.T + W.shape[1] * gamma_unit * ((np.abs(x) + ex) @ aW.T)
    act = (lambda v: np.maximum(v, 0.0)) if relu else (lambda v: v)
    a, lo, hi = rnd(act(z)), rnd(act(z - b)), rnd(act(z + b))
    flip = ((lo > 0) != (hi > 0)).any(1) if relu else np.zeros(z.shape[0], bool)
    # the kernel's activation is an fp16 value in [lo, hi] (rounding and ReLU are monotone): at most max(hi - a, a - lo) from ours, 0 when lo == hi
    ea = np.maximum(hi - a, a - lo)
    return a, ea, flip, z, b


class Forward:
    """float64 forward of the field with per-unit bounds: layer inputs (value, bound) and masks of both nets, raw64 and its bound, stable rows"""

    def __init__(self, dm, cm, enc, sh, gamma_unit=GAMMA_TC, rnd=f16):
        n = enc.shape[0]
        self.flip = np.zeros(n, bool)
        self.g = gamma_unit
        self.dxs, self.dmasks, dout, edout, zd, bd = self._net(dm, enc, np.zeros_like(enc), rnd)
        cin = np.concatenate([dout[:, 1:], sh, np.ones((n, 1))], 1)
        ecin = np.concatenate([edout[:, 1:], np.zeros((n, 17))], 1)
        self.cxs, self.cmasks, _, _, zc, bc = self._net(cm, cin, ecin, rnd)
        self.raw = np.concatenate([zc[:, :3], zd[:, :1]], 1)
        self.braw = np.concatenate([bc[:, :3], bd[:, :1]], 1)
        self.stable = ~self.flip

    def _net(self, mats, x, ex, rnd):
        xs, masks = [], []
        for W in mats[:-1]:
            xs.append((x, ex))
            x, ex, flip, _, _ = _layer(W, x, ex, True, self.g, rnd)
            self.flip |= flip
            masks.append(x > 0)
        xs.append((x, ex))
        y, ey, _, z, b = _layer(mats[-1], x, ex, False, self.g, rnd)
        return xs, masks, y, ey, z, b

    def check_raw(self, raw, cols=slice(0, 4)):
        """|raw_kernel - raw64| <= b + ulp16(|raw64| + b) on every row (the interval bound holds across a ReLU kink, so rows with an unstable
        decision are checked too, only more loosely); returns the largest err / bound"""
        r, b = self.raw[:, cols], self.braw[:, cols]
        bound = b + ulp16(np.abs(r) + b)
        err = np.abs(np.asarray(raw, np.float64).reshape(r.shape) - r)
        assert np.isfinite(raw).all()
        ratio = float((err / bound).max()) if err.size else 0.0
        assert ratio <= 1.0, ('forward outside the derived bound', ratio)
        return ratio


def _back(mats, xs, masks, gy, live, absolute):
    """gy: dL/d(output pre-activation) of one net. Returns (flat dW in tcnn order, flat E = |dZ|^T e_x, dL/d(input))"""
    T = np.abs if absolute else (lambda a: a)
    stage = (lambda v, lv: np.abs(v) + FLOOR * lv) if absolute else (lambda v, lv: v)
    dws, es = [None] * len(mats), [None] * len(mats)
    dz = stage(gy, live)
    for k in range(len(mats) - 1, -1, -1):
        x, ex = xs[k]
        dws[k] = dz.T @ T(x)
        es[k] = dz.T @ ex if absolute else None
        dx = dz @ T(mats[k])
        if k > 0:
            m = masks[k - 1]
            dz = stage(dx * m, m & live[:, :1])
    flat = np.concatenate([w.ravel() for w in dws])
    return flat, (np.concatenate([e.ravel() for e in es]) if absolute else None), dx


def field_chain(F, dm, cm, draw, rows, absolute):
    """exact backward (absolute=False) or its mass chain (True) -> (d_density, d_color, dL/denc, E_density, E_color)"""
    n = draw.shape[0]
    gy = np.zeros((n, 16)); gy[:, :3] = draw[:, :3]
    live = np.zeros((n, 16), bool); live[:, :3] = rows[:, None]
    dc, ec, gcin = _back(cm, F.cxs, F.cmasks, gy, live, absolute)
    gy = np.concatenate([draw[:, 3:4], gcin[:, :15]], 1)
    live = np.repeat(rows[:, None], 16, 1)
    dd, ed, genc = _back(dm, F.dxs, F.dmasks, gy, live, absolute)
    return dd, dc, genc, ed, ec


def within(name, got, ref, M, E, tau, depth, pre=None):
    """the per-entry assertion; returns (passes, largest err / bound, worst index)"""
    got = np.asarray(got, np.float64)
    bound = (tau + depth * 2.0 ** -23) * M + (1 + tau) * E
    if pre is not None:
        ref = ref + pre
        bound = bound + depth * 2.0 ** -23 * np.abs(pre)
    err = np.abs(got - ref)
    ratio = np.divide(err, bound, out=np.where(err > 0, np.inf, 0.0), where=bound > 0)
    k = int(np.argmax(ratio))
    return bool(np.isfinite(got).all() and ratio[k] <= 1.0), float(ratio[k]), k


# ----------------------------------------------------------------------------------------------------------------------------- fixtures
_WEIGHTS = {}


def _weights(dh, ch):
    if (dh, ch) not in _WEIGHTS:
        from xrnerf_b200 import synth
        _WEIGHTS[(dh, ch)] = synth.ngp_weights(seed=10 * dh + ch, dens_hidden=dh, color_hidden=ch, hash_range=0.5)
    return _WEIGHTS[(dh, ch)]


_FIELDS = {}


def field(dh, ch, npk):
    """NgpField with the (dh, ch) weights and `npk` levels in the cell image (one field per network shape, re-packed on demand)"""
    from xrnerf_b200.ngp import NgpField
    if (dh, ch) not in _FIELDS:
        _FIELDS.clear()
        _FIELDS[(dh, ch)] = load_ngp_weights(NgpField(density_hidden=dh, color_hidden=ch, n_packed_levels=npk).cuda(), _weights(dh, ch))
    f = _FIELDS[(dh, ch)]
    f.set_packed_levels(npk)
    f.refresh()
    assert f.n_packed == npk
    return f


@pytest.fixture(scope='module', autouse=True)
def _report():
    t0 = time.time()
    yield
    print(f'\n[field grad exact] wall {time.time() - t0:.1f} s')
    for line in REPORT:
        print('  ' + line)
    _FIELDS.clear()
    _CASES.clear()


def kernel_inputs(f, pts_d, dirs_d):
    """the bits the field kernels feed their networks: fp16 encodings (xrb_tcnn_hashgrid_forward on the field's table) and fp16 SH"""
    from xrnerf_b200 import _C
    n = pts_d.shape[0]
    sh = torch.empty((n, 16), dtype=torch.float16, device='cuda')
    dp, ds = _C.rows(dirs_d)
    _C.check(_C.lib.xrb_tcnn_sh4_forward(dp, ds, n, _C.ptr(sh), _C.stream()))
    return hashgrid_enc16(f, pts_d), sh.cpu().numpy().astype(np.float64)


def random_batch(n, seed):
    rng = np.random.default_rng(seed)
    pts = rng.random((n, 3)).astype(np.float32)
    dirs = rng.random((n, 3)).astype(np.float32)
    draw = (rng.normal(0, 1, (n, 4)) * 1e-3).astype(np.float32)
    return pts, dirs, draw


def contention_batch(grid, n=5000, seed=5):
    """n samples strictly inside ONE finest-level cell: every sample's atomics hit the same 8 entries per level"""
    rng = np.random.default_rng(seed)
    sc = np.float64(grid.scale[15])
    cell = np.array([1000, 1377, 642])
    pts = ((cell - 0.5 + rng.uniform(0.05, 0.95, (n, 3))) / sc).astype(np.float32)
    assert len(np.unique(grid.corners(15, pts)[0][:, 0])) == 1
    dirs = rng.random((n, 3)).astype(np.float32)
    draw = (rng.normal(0, 1, (n, 4)) * 1e-3).astype(np.float32)
    return pts, dirs, draw


def boundary_batch(grid, seed=6):
    """points exactly on cell boundaries (q = scale p + 0.5 an integer in fp32) with even and odd cell index on every level, dense and hashed
    (exercises the paired / swapped scatter and the dense-level wrap), plus every combination of 0 and 1 in the coordinates"""
    rng = np.random.default_rng(seed)
    rows = [[a, b, c] for a in (0.0, 1.0) for b in (0.0, 1.0) for c in (0.0, 1.0)]
    parity = set()
    for l in range(16):
        sc = np.float64(grid.scale[l])
        for k in rng.choice(np.arange(1, int(grid.res[l]) - 1), min(24, int(grid.res[l]) - 2), replace=False):
            # the fp32 value nearest (k - 0.5) / scale, or one of its neighbours, for which fma(scale, p, 0.5) is exactly k
            up = dn = np.float32((k - 0.5) / sc)
            cands = [up]
            for _ in range(4):
                up, dn = np.nextafter(up, np.float32(2)), np.nextafter(dn, np.float32(-1))
                cands += [up, dn]
            for p in cands:
                if np.float32(sc * np.float64(p) + 0.5) == k:
                    y, z = rng.random(2)
                    rows += [[p, y, z], [p, p, z], [p, p, p], [y, 1.0, p], [0.0, p, 1.0]]
                    parity.add((bool(grid.hashed[l]), int(k) & 1))
                    break
    assert parity == {(False, 0), (False, 1), (True, 0), (True, 1)}, parity
    pts = np.array(rows, np.float32)
    n = pts.shape[0]
    dirs = rng.random((n, 3)).astype(np.float32)
    dirs[:8] = pts[:8]
    draw = (rng.normal(0, 1, (n, 4)) * 1e-3).astype(np.float32)
    return pts, dirs, draw


class Case:
    """reference gradients, masses and depths of one batch on one field"""

    def __init__(self, f, pts, dirs, draw, impl, n_eff=None, pts_d=None, dirs_d=None):
        dh, ch = f.cfg.density_hidden, f.cfg.color_hidden
        table, dens, color = _weights(dh, ch)
        n_eff = pts.shape[0] if n_eff is None else n_eff
        pts, dirs, draw = pts[:n_eff], dirs[:n_eff], draw[:n_eff]
        pts_d = dev(pts) if pts_d is None else pts_d[:n_eff]
        dirs_d = dev(dirs) if dirs_d is None else dirs_d[:n_eff]
        self.grid = Grid(f.cfg)
        self.dm, self.cm = ngp_mats(dens, dh), ngp_mats(color, ch)
        enc, sh = kernel_inputs(f, pts_d, dirs_d) if n_eff else (np.zeros((0, 32)), np.zeros((0, 16)))
        self.F = F = Forward(self.dm, self.cm, enc, sh, GAMMA_TC if impl == 1 else GAMMA_FMA)
        self.n = n_eff
        self.rejected = float((~F.stable).mean()) if n_eff else 0.0
        rows = F.stable
        self.draw_masked = draw.copy()
        self.draw_masked[~rows] = 0.0
        d64 = self.draw_masked.astype(np.float64)
        self.dd, self.dc, genc, _, _ = field_chain(F, self.dm, self.cm, d64, rows, False)
        self.Md, self.Mc, agenc, self.Ed, self.Ec = field_chain(F, self.dm, self.cm, d64, rows, True)
        self.pts, self.rows, self.genc, self.agenc = pts, rows, genc, agenc
        self.dt, cnt = self.grid.scatter(pts, genc, rows)
        self.Mt, _ = self.grid.scatter(pts, agenc, rows)
        self.Dt = cnt + 8
        self.Dw = 192 + (n_eff + 127) // 128
        self.Et = np.zeros_like(self.Mt)

    def check(self, got, tau, pre=None, name=''):
        """every entry of the three vectors inside the bound; returns {vector: largest err / bound}"""
        out = {}
        for vec, g, ref, M, E, D in (('table', got[0], self.dt, self.Mt, self.Et, self.Dt), ('density', got[1], self.dd, self.Md, self.Ed, self.Dw),
                                     ('color', got[2], self.dc, self.Mc, self.Ec, self.Dw)):
            g = g.detach().cpu().numpy() if torch.is_tensor(g) else g
            p = None if pre is None else pre[vec]
            ok, ratio, k = within(vec, g, ref, M, E, tau, D, p)
            assert ok, (name, vec, 'entry', k, 'err/bound', ratio, 'kernel', float(g[k]), 'ref', float(ref[k] + (0 if p is None else p[k])), 'mass', float(M[k]))
            out[vec] = ratio
        if self.n >= 100:
            assert self.rejected <= REJECT_CEILING, (name, self.rejected)
            # not vacuous: most entries receive something (the colour output rows 3..15 and never-active hidden units receive nothing)
            assert (self.Mt > 0).sum() >= 128 and (self.Md > 0).mean() > 0.5 and (self.Mc > 0).mean() > 0.5
        return out


def tau_for(impl, dh, ch):
    layers = dh + 1 + ch + 1
    return (layers + 1) * U16 if impl == 1 else 2 * U16


def zeros_like_grads(f):
    return torch.zeros_like(f.hash_params), torch.zeros_like(f.density_params), torch.zeros_like(f.color_params)


def run_backward(f, pts_d, dirs_d, draw_d, impl, out=None, n=None, n_rows_dev=None):
    from xrnerf_b200 import _C
    out = zeros_like_grads(f) if out is None else out
    n = pts_d.shape[0] if n is None else n
    (pp, ps), (dp, ds) = _C.rows(pts_d), _C.rows(dirs_d)
    if impl == 1:
        _C.check(_C.lib.xrb_ngp_mlp_backward_tc(f.cfg, f.tab, _C.ptr(f._image), pp, ps, dp, ds, _C.f32(draw_d), n, None if n_rows_dev is None else _C.i32(n_rows_dev),
                                                _C.f32(out[0]), _C.f32(out[1]), _C.f32(out[2]), _C.stream()))
    else:
        assert n_rows_dev is None
        _C.check(_C.lib.xrb_ngp_mlp_backward(f.cfg, f.tab, _C.ptr(f._dens16), _C.ptr(f._color16), pp, ps, dp, ds, _C.f32(draw_d), n, _C.f32(out[0]), _C.f32(out[1]),
                                             _C.f32(out[2]), _C.stream()))
    torch.cuda.synchronize()
    return out


def report(name, case, ratios):
    REPORT.append(f'{name}: n={case.n} rejected={case.rejected:.4f} max err/bound ' + ' '.join(f'{k}={v:.3f}' for k, v in ratios.items()))


# ----------------------------------------------------------------------------------------------------------------------------- forward
@pytest.mark.parametrize('dh,ch', [(1, 1), (1, 2), (2, 3), (4, 4)])
def test_forward_within_derived_bound(dh, ch):
    """run_mlp and run_density, impl 0 (CUDA cores) and 1 (wgmma), packed levels 0/3/5/6/7: every sample's raw output within the bound
    propagated through the layers; the encodings the reference starts from are the same whatever the packing"""
    n = 20000
    pts, dirs, _ = random_batch(n, seed=100 + dh * 10 + ch)
    pts[:8] = [[a, b, c] for a in (0, 1) for b in (0, 1) for c in (0, 1)]
    pts_d, dirs_d = dev(pts), dev(dirs)
    _, dens, color = _weights(dh, ch)
    F = enc0 = None
    worst = 0.0
    for npk in (0, 3, 5, 6, 7):
        f = field(dh, ch, npk)
        enc, sh = kernel_inputs(f, pts_d, dirs_d)
        if F is None:
            enc0 = enc
            F = Forward(ngp_mats(dens, dh), ngp_mats(color, ch), enc, sh)
        assert np.array_equal(enc, enc0), npk
        for impl in (0, 1):
            worst = max(worst, F.check_raw(f.run_mlp(pts_d, dirs_d, impl=impl).cpu().numpy()))
            worst = max(worst, F.check_raw(f.run_density(pts_d, impl=impl).cpu().numpy(), cols=slice(3, 4)))
    REPORT.append(f'forward ({dh},{ch}): n={n} rejected={(~F.stable).mean():.4f} max err/bound={worst:.3f}')


# ----------------------------------------------------------------------------------------------------------------------------- backward
_CASES = {}
BACKWARD_CASES = [(1, (1, 1), 0), (1, (1, 1), 6), (1, (1, 1), 7), (1, (1, 2), 0), (1, (1, 2), 6), (1, (1, 2), 7),
                  (0, (1, 1), 6), (0, (1, 2), 6), (0, (2, 2), 6), (0, (1, 3), 6), (0, (2, 3), 6)]


def _expected_kernel(impl, dh, ch, npk):
    if impl == 1:   # the wgmma backward is specialised for "levels [0,6) packed, the rest hashed" only: 0 and 7 packed levels take NP = 0 (run-time gather form)
        return f'ngp_field_bwd_tc_kernel<{dh},{ch},{6 if npk == 6 else 0}>'
    return f'ngp_field_bwd_kernel<{dh},{ch}>'


@pytest.mark.parametrize('impl,shape,npk', BACKWARD_CASES, ids=[f'impl{i}-{s[0]}{s[1]}-np{p}' for i, s, p in BACKWARD_CASES])
def test_backward_entrywise(impl, shape, npk):
    """every instantiation of both backward kernels (test_every_backward_instantiation_runs checks which one each case launches), n = 40 001:
    table, density and colour gradients entry by entry"""
    dh, ch = shape
    f = field(dh, ch, npk)
    pts, dirs, draw = random_batch(40001, seed=7)
    if (dh, ch, impl) not in _CASES:   # the encodings do not depend on the packing (test_forward_within_derived_bound): one reference per network and path
        _CASES.clear()
        _CASES[(dh, ch, impl)] = Case(f, pts, dirs, draw, impl)
    case = _CASES[(dh, ch, impl)]
    got = run_backward(f, dev(pts), dev(dirs), dev(case.draw_masked), impl)
    ratios = case.check(got, tau_for(impl, dh, ch), name=_expected_kernel(impl, dh, ch, npk))
    report(f'backward {_expected_kernel(impl, dh, ch, npk)} np{npk}', case, ratios)
    if (impl, shape, npk) == (1, (1, 2), 6):
        _altered_references_are_rejected(case, got, tau_for(impl, dh, ch))


def test_every_backward_instantiation_runs():
    """one profiler trace over the cases of test_backward_entrywise: each launches the template instance it is named for (wgmma <1,1,0> <1,1,6>
    <1,2,0> <1,2,6>, CUDA cores (1,1) (1,2) (2,2) (1,3) (2,3))"""
    from torch.profiler import ProfilerActivity, profile
    pts, dirs, draw = (dev(a) for a in random_batch(300, seed=8))
    fields = {}
    for impl, (dh, ch), npk in BACKWARD_CASES:
        fields[(impl, dh, ch, npk)] = field(dh, ch, npk)
        run_backward(fields[(impl, dh, ch, npk)], pts, dirs, draw, impl)   # outside the trace: first launches load the module
    names = []
    for (impl, dh, ch, npk), f in fields.items():
        f.set_packed_levels(npk); f.refresh()
        torch.cuda.synchronize()
        with profile(activities=[ProfilerActivity.CUDA]) as prof:
            run_backward(f, pts, dirs, draw, impl)
        got = [e.name.replace(' ', '') for e in prof.events() if 'bwd' in e.name]
        want = _expected_kernel(impl, dh, ch, npk)
        assert any(want in k for k in got), (want, got)
        names.append(want)
    assert len(set(names)) == 9
    REPORT.append('kernels run: ' + ' '.join(sorted(set(names))))


def _altered_references_are_rejected(case, got, tau):
    """The assertion the kernel passes must reject (a) the reference without one stable sample's contribution on the finest-level entries it
    touches, and (b) the reference with one sample's x-adjacent corner pair swapped on one hashed level (what a wrong `swap` would do)."""
    g = got[0].cpu().numpy()
    grid = case.grid
    s = int(np.argmax(np.abs(case.genc[:, 30:32]).sum(1) * case.rows))
    assert case.rows[s]
    p = case.pts[s:s + 1]
    idx, w = grid.corners(15, p)
    ref, M = case.dt.copy(), case.Mt.copy()
    for c in range(8):
        for ft in range(2):
            ref[2 * idx[0, c] + ft] -= w[0, c] * case.genc[s, 30 + ft]
            M[2 * idx[0, c] + ft] -= w[0, c] * case.agenc[s, 30 + ft]
    assert not within('table', g, ref, np.maximum(M, 0), case.Et, tau, case.Dt)[0], 'removing a sample from the finest level went unnoticed'
    # (b): the hashed level and sample with the largest |w1 - w0| |g|
    best = None
    for l in np.nonzero(grid.hashed)[0]:
        idx, w = grid.corners(l, case.pts)
        gl = np.abs(case.genc[:, 2 * l]) * case.rows
        score = (np.abs(w[:, 1] - w[:, 0]) * gl)
        k = int(np.argmax(score))
        if best is None or score[k] > best[0]:
            best = (score[k], l, k, idx[k], w[k])
    _, l, s, idx, w = best
    ref, M = case.dt.copy(), case.Mt.copy()
    for yz in range(4):
        i0, i1, w0, w1 = idx[2 * yz], idx[2 * yz + 1], w[2 * yz], w[2 * yz + 1]
        for ft in range(2):
            gv, av = case.genc[s, 2 * l + ft], case.agenc[s, 2 * l + ft]
            ref[2 * i0 + ft] += (w1 - w0) * gv; ref[2 * i1 + ft] += (w0 - w1) * gv
            M[2 * i0 + ft] += (w1 - w0) * av; M[2 * i1 + ft] += (w0 - w1) * av
    assert not within('table', g, ref, np.maximum(M, 0), case.Et, tau, case.Dt)[0], 'a swapped corner pair went unnoticed'


@pytest.mark.parametrize('impl', [0, 1])
@pytest.mark.parametrize('n', [1, 127, 128, 129])
def test_backward_row_counts(impl, n):
    """partial, exact and one-over tiles (impl 1: the production instance <1,2,6>)"""
    f = field(1, 2, 6)
    pts, dirs, draw = random_batch(n, seed=1000 + n)
    case = Case(f, pts, dirs, draw, impl)
    got = run_backward(f, dev(pts), dev(dirs), dev(case.draw_masked), impl)
    report(f'backward impl{impl} (1,2) n={n}', case, case.check(got, tau_for(impl, 1, 2), name=f'n={n}'))


@pytest.mark.parametrize('impl', [0, 1])
@pytest.mark.parametrize('kind', ['contention', 'boundaries'])
def test_backward_edge_batches(impl, kind):
    """contention: 5000 samples in one finest-level cell (every atomic of a level on the same entries); boundaries: points exactly on cell
    boundaries with even and odd index on dense and hashed levels, and the corners of the unit cube"""
    f = field(1, 2, 6)
    pts, dirs, draw = (contention_batch if kind == 'contention' else boundary_batch)(Grid(f.cfg))
    case = Case(f, pts, dirs, draw, impl)
    got = run_backward(f, dev(pts), dev(dirs), dev(case.draw_masked), impl)
    report(f'backward impl{impl} (1,2) {kind}', case, case.check(got, tau_for(impl, 1, 2), name=kind))


@pytest.mark.parametrize('impl', [0, 1])
def test_backward_strided_rows_and_prefilled_out(impl):
    """pts / dirs as the stride-7 views coords[:, :3] / coords[:, 4:] the trainer passes, and gradients ACCUMULATED onto non-zero outputs"""
    f = field(1, 2, 6)
    n = 9000
    pts, dirs, draw = random_batch(n, seed=77)
    rng = np.random.default_rng(78)
    coords = rng.random((n, 7)).astype(np.float32)
    coords[:, :3] = pts; coords[:, 4:] = dirs
    coords_d = dev(coords)
    case = Case(f, pts, dirs, draw, impl, pts_d=coords_d[:, :3], dirs_d=coords_d[:, 4:])
    pre = {k: (rng.normal(0, 1, v.size) * np.abs(v).max()).astype(np.float32) for k, v in (('table', case.dt), ('density', case.dd), ('color', case.dc))}
    out = tuple(dev(pre[k]) for k in ('table', 'density', 'color'))
    got = run_backward(f, coords_d[:, :3], coords_d[:, 4:], dev(case.draw_masked), impl, out=out)
    report(f'backward impl{impl} (1,2) strided + prefilled', case,
           case.check(got, tau_for(impl, 1, 2), pre={k: v.astype(np.float64) for k, v in pre.items()}, name='prefilled'))


@pytest.mark.parametrize('count', [700, 0, -5, 1100])
def test_backward_device_row_count(count):
    """n_rows_dev (the compacted sample count the trainer leaves on the device): the kernel reads min(n, max(count, 0)) rows; the rows past
    the count are NaN in pts and dL/draw and must never be read"""
    f = field(1, 2, 6)
    n = 1000
    n_eff = min(n, max(count, 0))
    pts, dirs, draw = random_batch(n, seed=31)
    case = Case(f, pts, dirs, draw, 1, n_eff=n_eff)
    draw_k = draw.copy()
    draw_k[:n_eff] = case.draw_masked
    pts[n_eff:] = np.nan; draw_k[n_eff:] = np.nan
    got = run_backward(f, dev(pts), dev(dirs), dev(draw_k), 1, n=n, n_rows_dev=torch.tensor([count], dtype=torch.int32, device='cuda'))
    if n_eff == 0:
        assert all(float(g.abs().max()) == 0.0 for g in got)
        return
    report(f'backward <1,2,6> n_rows_dev={count}', case, case.check(got, tau_for(1, 1, 2), name=f'count={count}'))


# ----------------------------------------------------------------------------------------------------------------------------- stand-alone module backwards
def test_tcnn_hashgrid_backward_entrywise():
    """xrb_tcnn_hashgrid_backward (tcnn.Encoding's backward): fp16 dL/denc x grad_scale scattered into an accumulated fp32 table gradient"""
    from xrnerf_b200 import _C
    f = field(1, 2, 0)
    grid = Grid(f.cfg)
    pts, _, _ = random_batch(30000, seed=41)
    pts = np.concatenate([boundary_batch(grid)[0], contention_batch(grid, 2000)[0], pts])
    n = pts.shape[0]
    rng = np.random.default_rng(42)
    denc = rng.normal(0, 1, (n, 32)).astype(np.float16)
    denc[::97] = 0
    scale = 0.25
    g64 = denc.astype(np.float64) * scale
    rows = np.ones(n, bool)
    ref, cnt = grid.scatter(pts, g64, rows)
    M, _ = grid.scatter(pts, np.abs(g64), rows)
    pre = (rng.normal(0, 1, ref.size) * np.abs(ref).max()).astype(np.float32)
    out, pts_d, denc_d = dev(pre), dev(pts), dev(denc)
    xp, xs = _C.rows(pts_d)
    _C.check(_C.lib.xrb_tcnn_hashgrid_backward(f.cfg, xp, xs, n, _C.ptr(denc_d), scale, _C.f32(out), _C.stream()))
    ok, ratio, k = within('table', out.cpu().numpy(), ref, M, 0.0, U16, cnt + 8, pre.astype(np.float64))
    assert ok, (k, ratio)
    REPORT.append(f'tcnn hashgrid backward: n={n} max err/bound={ratio:.3f}')


@pytest.mark.parametrize('n_hidden', [1, 2])
def test_tcnn_mlp_backward_entrywise(n_hidden):
    """xrb_tcnn_mlp_backward (tcnn.Network's backward): dX (fp16) and the accumulated fp32 parameter gradient, against the same float64 chain"""
    from xrnerf_b200 import _C, synth
    n = 20001
    _, dens, _ = synth.ngp_weights(seed=50 + n_hidden, n_hash_params=8, dens_hidden=n_hidden)
    mats = ngp_mats(dens, n_hidden)
    rng = np.random.default_rng(51)
    x16 = rng.uniform(-1, 1, (n, 32)).astype(np.float16)
    x16[:, 31] = 1
    dy16 = (rng.normal(0, 1, (n, 16)) * 5e-2).astype(np.float16)
    # forward bound and rejection exactly as for the field (the input is exact)
    xs, masks, x, ex, flip = [], [], x16.astype(np.float64), np.zeros((n, 32)), np.zeros(n, bool)
    for W in mats[:-1]:
        xs.append((x, ex))
        x, ex, fl, _, _ = _layer(W, x, ex, True, GAMMA_FMA)
        flip |= fl
        masks.append(x > 0)
    xs.append((x, ex))
    rejected = float(flip.mean())
    assert rejected <= REJECT_CEILING
    dy16[flip] = 0
    rows = ~flip
    live = np.repeat(rows[:, None], 16, 1)
    dw, _, dx = _back(mats, xs, masks, dy16.astype(np.float64), live, False)
    Mw, Ew, Mx = _back(mats, xs, masks, dy16.astype(np.float64), live, True)
    pre = (rng.normal(0, 1, dw.size) * np.abs(dw).max()).astype(np.float32)
    p16, x_d, dy_d, d = dev(f16(dens).astype(np.float16)), dev(x16), dev(dy16), dev(pre)
    dx_k = torch.empty((n, 32), dtype=torch.float16, device='cuda')
    _C.check(_C.lib.xrb_tcnn_mlp_backward(_C.ptr(p16), _C.ptr(x_d), _C.ptr(dy_d), n, 32, 64, n_hidden, _C.ptr(dx_k), _C.f32(d), _C.stream()))
    tau = 2 * U16
    ok, r_w, k = within('params', d.cpu().numpy(), dw, Mw, Ew, tau, 192 + (n + 127) // 128, pre.astype(np.float64))
    assert ok, ('dW', k, r_w)
    # dX: the fp32 chain rounded once to fp16 (relative 2^-11, absolute 2^-25 below the normal range)
    got_dx = dx_k.cpu().numpy().astype(np.float64)[rows]
    bound = tau * Mx[rows] + 2.0 ** -25
    r_x = float((np.abs(got_dx - dx[rows]) / bound).max())
    assert r_x <= 1.0, ('dX', r_x)
    REPORT.append(f'tcnn mlp backward n_hidden={n_hidden}: n={n} rejected={rejected:.4f} max err/bound dW={r_w:.3f} dX={r_x:.3f}')
