"""The NGP training step's small kernels on their own: the 5 x Huber loss and its gradient, the bf16 gradient pack and the Adam + EMA step
that reads it (the sharded data-parallel path), the peer-memory Adam + EMA step against the local one, and the count of fully trained rays.
Each is checked bit for bit where its arithmetic is one fp32 expression, and against float64 within a stated bound where it is a sum."""
import numpy as np
import pytest
import torch
from cases import dev

pytestmark = pytest.mark.gpu


# ----------------------------------------------------------------------------------------------------------------------------- 5 x Huber
@pytest.mark.parametrize('n', [1, 255, 256, 257, 3 * 65536 + 5])
def test_huber5_grad_bits_and_loss(n):
    """gradient == the kernel's fp32 expression evaluated by numpy, bit for bit; loss == float64 5 * HuberLoss(sum) within
    n 2^-23 sum|terms| (fp32 terms summed in any order); the loss is ADDED to the accumulator's prior value"""
    from xrnerf_b200 import _C
    delta = np.float32(0.1)
    rng = np.random.default_rng(n)
    target = rng.random(n).astype(np.float32)
    rgb = (target + rng.normal(0, 0.15, n)).astype(np.float32)
    special = [(0.0, 0.0), (0.0, 0.1), (0.1, 0.0), (0.0, -0.1), (0.5, 0.5), (0.3, 0.0), (0.0, 0.75), (-0.1, 0.0)]   # |diff| = 0, exactly delta, beyond delta
    for k, (a, b) in enumerate(special[:n]):
        rgb[k], target[k] = np.float32(a), np.float32(b)
    if n >= 3:
        assert np.float32(rgb[1] - target[1]) == -delta and np.float32(rgb[2] - target[2]) == delta
    prior = 1.5
    grad = torch.full((n,), np.nan, dtype=torch.float32, device='cuda')
    loss = torch.tensor([prior], dtype=torch.float32, device='cuda')
    rgb_d, target_d = dev(rgb), dev(target)
    _C.check(_C.lib.xrb_ngp_huber5_grad(_C.ptr(rgb_d), _C.ptr(target_d), n, float(delta), _C.ptr(grad), _C.ptr(loss), _C.stream()))
    torch.cuda.synchronize()
    diff = rgb - target
    rel = np.abs(diff)
    with np.errstate(all='raise'):
        want = np.float32(5) * np.where(rel > delta, np.copysign(np.float32(1), diff), diff / delta).astype(np.float32)
    assert want.dtype == np.float32
    assert np.array_equal(grad.cpu().numpy().view(np.uint32), want.view(np.uint32))
    d64 = rgb.astype(np.float64) - target.astype(np.float64)
    r64 = np.abs(d64)
    terms = 5 * np.where(r64 > np.float64(delta), r64 - 0.5 * np.float64(delta), 0.5 / np.float64(delta) * r64 * r64)
    got = float(loss.item()) - prior
    bound = n * 2.0 ** -23 * np.abs(terms).sum() + np.spacing(np.float32(prior + terms.sum()))
    assert abs(got - terms.sum()) <= bound, (got, terms.sum(), bound)


# ----------------------------------------------------------------------------------------------------------------------------- bf16 pack
def _special_bits():
    bits = [0x3F808000, 0x3F818000, 0xBF808000, 0xBF818000,     # ties (low half 0x8000) with an even and an odd upper half, both signs
            0x3F807FFF, 0x3F808001,                             # just below / above a tie
            0x00000000, 0x80000000,                             # +-0
            0x00000001, 0x00008000, 0x00018000, 0x007FFFFF, 0x807FFFFF, 0x80008000,   # subnormals (incl. ties)
            0x7F800000, 0xFF800000,                             # +-inf
            0x7F7FFFFF, 0xFF7FFFFF, 0x7F7F8000, 0x7F7F7FFF,     # the largest finite values: round to inf / to the largest bf16
            0x7FC00000, 0xFFC00001, 0x7F800001, 0x7FBFFFFF]     # NaNs (quiet, negative, signalling)
    return np.array(bits, np.uint32).view(np.float32)


@pytest.mark.parametrize('n', [1, 2, 3, 4, 5, 1023, 4 * 65536 + 3])
def test_pack_bf16_bits_match_torch(n):
    """xrb_pack_bf16 == torch's round-to-nearest-even float -> bfloat16 conversion bit for bit, NaN as NaN, with the special values placed at the
    head and in the scalar tail of the vectorised loop"""
    from xrnerf_b200 import _C
    rng = np.random.default_rng(n)
    src = (rng.normal(0, 1, n) * np.exp2(rng.integers(-140, 120, n))).astype(np.float32)   # normal and subnormal magnitudes
    sp = _special_bits()
    m = min(n, sp.size)
    src[:m] = sp[:m]
    if n > 8:
        src[-3:] = sp[[0, 1, 16]]   # ties and the round-to-inf value in the tail elements
    src_d, dst = dev(src), torch.full((n,), -1, dtype=torch.int16, device='cuda')
    _C.check(_C.lib.xrb_pack_bf16(_C.ptr(src_d), _C.ptr(dst), n, _C.stream()))
    got = dst.cpu().numpy().view(np.uint16)
    want = torch.from_numpy(src).to(torch.bfloat16).view(torch.int16).numpy().view(np.uint16)
    nan = np.isnan(src)
    got_f = (got.astype(np.uint32) << 16).view(np.float32)
    assert np.isnan(got_f[nan]).all()
    assert np.array_equal(got[~nan], want[~nan])


# ----------------------------------------------------------------------------------------------------------------------------- Adam + EMA, bf16 gradient
def test_adam_ema_step_bf16grad():
    """4 steps with grad_div = 2, weight decay and EMA: float64 torch.optim.Adam + mmcv EMAHook agree at the fp32 Adam test's tolerance; the fp16
    shadow is the RNE rounding of the new parameters; the parameters (and moments, EMA) are bit-identical to xrb_adam_ema_step fed the same
    gradient widened to fp32"""
    from xrnerf_b200 import _C
    torch.manual_seed(3)
    n = 70003
    lr, b1, b2, eps, wd, div = 1e-2, 0.9, 0.99, 1e-15, 1e-6, 2.0
    p0 = torch.randn(n, device='cuda')
    a = {k: v.clone() for k, v in (('p', p0), ('m', torch.zeros_like(p0)), ('v', torch.zeros_like(p0)), ('ema', p0))}
    b = {k: v.clone() for k, v in a.items()}
    p16 = torch.empty(n, dtype=torch.float16, device='cuda'); p16b = torch.empty_like(p16)
    ref = p0.double().clone().requires_grad_(True)
    opt = torch.optim.Adam([ref], lr=lr, betas=(b1, b2), eps=eps, weight_decay=wd)
    ema_ref = p0.double().clone()
    for step in range(1, 5):
        g16 = (torch.randn(n, device='cuda') * 0.1 * step).to(torch.bfloat16)
        g16[:4] = torch.tensor([0.0, -0.0, 1e-40, -3e4], dtype=torch.bfloat16)   # zero, signed zero, a bf16 subnormal, a large value
        mom = min(0.05, step / (100 + step - 1))
        _C.check(_C.lib.xrb_adam_ema_step_bf16grad(_C.ptr(a['p']), _C.ptr(p16), _C.ptr(g16), _C.ptr(a['m']), _C.ptr(a['v']), n, lr, b1, b2, eps, wd, step, div,
                                                    _C.ptr(a['ema']), mom, _C.stream()))
        g32 = g16.float()
        _C.check(_C.lib.xrb_adam_ema_step(_C.ptr(b['p']), _C.ptr(p16b), _C.ptr(g32), _C.ptr(b['m']), _C.ptr(b['v']), n, lr, b1, b2, eps, wd, step, div,
                                          _C.ptr(b['ema']), mom, _C.stream()))
        ref.grad = g16.double() / div
        opt.step()
        ema_ref.mul_(1 - mom).add_(ref.detach(), alpha=mom)
        torch.cuda.synchronize()
        assert torch.equal(p16, a['p'].half())
    for k in a:
        assert torch.equal(a[k].view(torch.int32), b[k].view(torch.int32)), k
    assert torch.equal(p16, p16b)
    assert torch.allclose(a['p'].double(), ref.detach(), rtol=1e-5, atol=1e-6)
    assert torch.allclose(a['ema'].double(), ema_ref, rtol=1e-5, atol=1e-6)


# ----------------------------------------------------------------------------------------------------------------------------- peer Adam + EMA at world 1
def test_peer_adam_step_world1_bits_match_local_adam():
    """xrb_peer_publish_grads + xrb_peer_adam_step on one rank's own exchange block (world 1, no IPC mapping), 4 steps with weight decay and EMA:
    the table slice (8-wide path and scalar tail: n_table is not a multiple of 8) is bit-identical to xrb_adam_ema_step_bf16grad fed xrb_pack_bf16 of
    the same fp32 gradient, and both MLP groups to xrb_adam_ema_step on the fp32 gradient (master, moments, EMA, fp16 copies). Parameters have no
    exact zeros: the peer sum 0 + g turns a -0 gradient into +0, which weight decay would otherwise expose."""
    from xrnerf_b200 import _C
    from xrnerf_b200.train import _DevView, shard_range
    C = _C.C
    torch.manual_seed(5)
    n_table, n_mlp = (70003, (4099, 2055))
    _, _, per, padded = shard_range(n_table, 1, 0)
    lr, b1, b2, eps, wd = 1e-2, 0.9, 0.99, 1e-15, 1e-6
    a16 = lambda x: (x + 15) // 16 * 16   # noqa: E731
    off_g16 = 128
    off_gmlp = a16(off_g16 + 2 * padded)
    off_t16 = a16(off_gmlp + 4 * sum(n_mlp))
    own, handle = C.c_void_p(), (C.c_char * 64)()
    _C.check(_C.lib.xrb_peer_alloc(a16(off_t16 + 2 * padded), C.byref(own), handle), 'peer_alloc')
    try:
        layout = _C.PeerLayout(1, 0, (C.c_void_p * 8)(own.value), off_g16, off_gmlp, off_t16, n_table, per, sum(n_mlp))
        t16 = torch.as_tensor(_DevView(own.value + off_t16, padded, '<f2'), device='cuda')

        def state(n):
            p = torch.randn(n, device='cuda')
            p[p == 0] = 1.0
            return {'p': p, 'm': torch.zeros_like(p), 'v': torch.zeros_like(p), 'ema': p.clone(), 'p16': torch.empty(n, dtype=torch.float16, device='cuda')}
        peer = [state(n) for n in (n_table,) + n_mlp]
        local = [{k: v.clone() for k, v in s.items()} for s in peer]
        groups = [_C.PeerMlpGroup(_C.ptr(s['p']), _C.ptr(s['p16']), _C.ptr(s['m']), _C.ptr(s['v']), _C.ptr(s['ema']), s['p'].numel(), off)
                  for s, off in ((peer[1], 0), (peer[2], n_mlp[0]))]
        g16 = torch.empty(n_table, dtype=torch.bfloat16, device='cuda')
        for step in range(1, 5):
            g_table = torch.randn(n_table, device='cuda') * 0.1 * step
            g_mlp = torch.randn(sum(n_mlp), device='cuda') * 0.1 * step
            mom = min(0.05, step / (100 + step - 1))
            tp = peer[0]
            _C.check(_C.lib.xrb_peer_publish_grads(C.byref(layout), _C.ptr(g_table), _C.ptr(g_mlp), step, _C.stream()), 'peer_publish_grads')
            _C.check(_C.lib.xrb_peer_adam_step(C.byref(layout), _C.ptr(tp['p']), _C.ptr(tp['m']), _C.ptr(tp['v']), _C.ptr(tp['ema']), C.byref(groups[0]), C.byref(groups[1]),
                                               lr, b1, b2, eps, wd, step, mom, step, _C.stream()), 'peer_adam_step')
            _C.check(_C.lib.xrb_pack_bf16(_C.ptr(g_table), _C.ptr(g16), n_table, _C.stream()), 'pack_bf16')
            tl = local[0]
            _C.check(_C.lib.xrb_adam_ema_step_bf16grad(_C.ptr(tl['p']), _C.ptr(tl['p16']), _C.ptr(g16), _C.ptr(tl['m']), _C.ptr(tl['v']), n_table, lr, b1, b2, eps, wd, step, 1.0,
                                                        _C.ptr(tl['ema']), mom, _C.stream()), 'adam bf16')
            for s, g in zip(local[1:], (g_mlp[:n_mlp[0]], g_mlp[n_mlp[0]:])):
                _C.check(_C.lib.xrb_adam_ema_step(_C.ptr(s['p']), _C.ptr(s['p16']), _C.ptr(g), _C.ptr(s['m']), _C.ptr(s['v']), s['p'].numel(), lr, b1, b2, eps, wd, step, 1.0,
                                                  _C.ptr(s['ema']), mom, _C.stream()), 'adam')
        torch.cuda.synchronize()
        st = C.c_uint32(1)
        _C.check(_C.lib.xrb_peer_status(own, C.byref(st), _C.stream()), 'peer_status')
        assert st.value == 0
        for name, a, b in zip(('table', 'density', 'color'), peer, local):
            for k in ('p', 'm', 'v', 'ema'):
                assert torch.equal(a[k].view(torch.int32), b[k].view(torch.int32)), (name, k)
        assert torch.equal(t16[:n_table].view(torch.int16), local[0]['p'].half().view(torch.int16))
        for a, b in zip(peer[1:], local[1:]):
            assert torch.equal(a['p16'].view(torch.int16), b['p16'].view(torch.int16))
    finally:
        torch.cuda.synchronize()
        _C.check(_C.lib.xrb_peer_free(own), 'peer_free')


# ----------------------------------------------------------------------------------------------------------------------------- trained-ray count
def test_count_trained_rays_on_truncated_compaction():
    """xrb_rm_compacted_coord truncates a batch to T = 20 000 samples; xrb_ngp_count_trained_rays ADDS the number of rays whose every sample survived
    (n_rays = 3001, not a multiple of the 256-thread block), twice; both against numpy"""
    from xrnerf_b200 import _C
    n_rays, T = 3001, 20000
    rng = np.random.default_rng(12)
    counts = rng.integers(0, 16, n_rays).astype(np.int32)
    counts[rng.random(n_rays) < 0.1] = 0
    offs = np.concatenate([[0], np.cumsum(counts)[:-1]]).astype(np.int32)
    total = int(counts.sum())
    assert total > T
    numsteps = dev(np.stack([counts, offs], 1))
    coords = dev(rng.random((total, 7)).astype(np.float32))
    coords_c = torch.zeros((T, 7), dtype=torch.float32, device='cuda')
    numsteps_c = torch.full((n_rays, 2), -1, dtype=torch.int32, device='cuda')
    rc = torch.zeros(1, dtype=torch.int32, device='cuda'); sc = torch.zeros(1, dtype=torch.int32, device='cuda')
    ws = torch.empty(_C.lib.xrb_rm_compacted_coord_workspace(n_rays), dtype=torch.uint8, device='cuda')
    _C.check(_C.lib.xrb_rm_compacted_coord(None, _C.ptr(coords), _C.ptr(numsteps), n_rays, T, _C.ptr(coords_c), _C.ptr(numsteps_c), _C.ptr(rc), _C.ptr(sc), _C.ptr(ws),
                                           _C.stream()))
    accum = torch.tensor([7], dtype=torch.int64, device='cuda')
    for _ in range(2):
        _C.check(_C.lib.xrb_ngp_count_trained_rays(_C.ptr(numsteps), _C.ptr(numsteps_c), n_rays, _C.ptr(accum), _C.stream()))
    torch.cuda.synchronize()
    nc = numsteps_c.cpu().numpy()
    want_c = np.minimum(np.maximum(T - offs, 0), counts)      # the compaction keeps a ray's samples up to the T-th of the batch
    assert np.array_equal(nc[:, 0], want_c)
    trained = int((want_c == counts).sum())
    assert 0 < trained < n_rays and trained == int((nc[:, 0] == counts).sum())
    assert int(accum.item()) == 7 + 2 * trained
