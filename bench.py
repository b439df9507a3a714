#!/usr/bin/env python
"""bench.py — rays/sec of the Instant-NGP hot path (BASELINE.json configs[1]: lego-shaped scene, 65 536 rays per batch).

    python bench.py [--gpus N] [--steps K] [--warmup W] [--impl ours|reference]

A "step" is one pass of the hot path (ray march -> hash/SH encode -> tiny MLPs -> alpha compositing) over one batch of
65 536 synthetic Blender-shaped rays (800x800 spiral views, seeded lego-like occupancy grid, tcnn-default random weights).
  value      device-timed rays/s with the ray batches already resident in HBM (one CUDA-event pair around the K steps, max over
             ranks); inputs larger than L2: 96 distinct ray batches (151 MB) are cycled, nothing is flushed (the 24.4 MB fp16 hash
             table and its cell image are meant to stay L2-resident, as in production)
  e2e        the same metric through the public API with HOST (pinned) ray buffers: H2D of the rays and D2H of rgb+alpha
             inside the timed region
  roofline   dominant kernel (ngp_field_tc_kernel: hash gather + wgmma MLPs) timed live with CUDA events recorded inside the
             step; algorithmic bytes = 512 B gathered per sample (16 levels x 8 corners x 2 x fp16, SURVEY §8d) + 28 B coords in
             + 16 B raw out per sample
  cpu_baseline / --impl reference   the reference's own ngp_raymarch kernels compiled for CPU (oracle/_ref) for march and
             compositing + the C restatement of tcnn (oracle port) for the field, all host cores, on a bounded ray sample.
  reference_gpu / nerf.reference_torch_gpu_mlp   BASELINE.md B4 / B3: the reference's own CUDA kernels (built unmodified for sm_90a, oracle/build_ref_cuda.py) and its
             NerfMLP arithmetic on cuBLAS, timed per op on this GPU next to ours (rank 0, N = 1)
Steps are issued on `--pipeline` CUDA streams (default 8 batches in flight, each with its own workspace; stated in config.batches_in_flight): throughput, not latency.
Multi-GPU (torchrun): rays shard over ranks with no data-path collective (weak scaling: 65 536 rays per rank per step); the training arm's optimiser exchange runs over
NVLink peer memory (csrc/peer_adam.cu; --grad-comm).
"""
import argparse
import json
import os
import subprocess
import sys
import threading
import time

if '--impl' in sys.argv and 'reference' in sys.argv or not os.environ.get('WORLD_SIZE'):
    # the CPU legs use every host core; must happen before numpy / torch / the oracle load libgomp (see _omp_configure)
    os.environ['OMP_NUM_THREADS'] = str(os.cpu_count() or 1)
    os.environ.setdefault('OMP_PROC_BIND', 'close'); os.environ.setdefault('OMP_PLACES', 'cores'); os.environ.setdefault('OMP_DYNAMIC', 'false')

import numpy as np

ROOT = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, ROOT)

N_RAYS = 65536
BUDGET = 64          # max samples per ray the workspace is sized for (reference: 1024; measured mean is ~11-30)
N_BATCHES = 96       # distinct ray batches cycled through: 96 x 1.5 MiB of rays = 151 MB > 50 MB L2 (inputs larger than L2)
METRIC = 'rays/sec (inference render, Instant-NGP lego-shaped 800x800, 65536 rays/batch)'
WORKLOAD = 'instant-ngp lego-like synthetic (configs[1]): 65536 rays/batch from 40 spiral 800x800 views, occupancy-grid march + hash(16x2,T=2^19) + SH4 + MLP(64;1+2 hidden) + composite, forward'
BYTES_PER_SAMPLE = 512 + 28 + 16


def peaks():
    try:
        with open(os.path.join(ROOT, 'MEASURED_PEAKS.json')) as fh:
            p = json.load(fh)
        return float(p['hbm_gbs']), 'measured (MEASURED_PEAKS.json hbm_gbs)'
    except Exception:
        return 3350.0, 'H100 SXM data sheet (3.35 TB/s HBM3)'


def tensor_peak():
    try:
        with open(os.path.join(ROOT, 'MEASURED_PEAKS.json')) as fh:
            return float(json.load(fh)['bf16_tflops_sustained']), 'measured (MEASURED_PEAKS.json bf16_tflops_sustained; kernel timed inside a multi-kernel step)'
    except Exception:
        return 989.0, 'H100 SXM data sheet (989 TFLOP/s dense fp16 / bf16)'


class ClockSampler:
    """nvidia-smi clocks + throttle reasons sampled every 200 ms while the timed region runs."""

    def __init__(self, index):
        self.index, self.rows, self.proc = index, [], None

    def start(self):
        q = 'index,clocks.sm,clocks.max.sm,clocks_event_reasons.hw_slowdown,clocks_event_reasons.hw_thermal_slowdown,clocks_event_reasons.sw_thermal_slowdown,clocks_event_reasons.sw_power_cap'
        try:
            self.proc = subprocess.Popen(['nvidia-smi', f'--query-gpu={q}', '--format=csv,noheader,nounits', '-lms', '200', '-i', str(self.index)],
                                         stdout=subprocess.PIPE, stderr=subprocess.DEVNULL, text=True)
            self.t = threading.Thread(target=self._read, daemon=True)
            self.t.start()
        except Exception:
            self.proc = None

    def _read(self):
        for line in self.proc.stdout:
            self.rows.append([x.strip() for x in line.split(',')])

    def stop(self):
        if self.proc is None:
            return {'sm_mhz': None, 'sm_max_mhz': None, 'reasons': ['nvidia-smi unavailable']}
        time.sleep(0.25)
        self.proc.terminate()
        try:
            self.proc.wait(timeout=2)
        except Exception:
            self.proc.kill()
        sm = [float(r[1]) for r in self.rows if len(r) >= 7 and r[1].replace('.', '').isdigit()]
        mx = [float(r[2]) for r in self.rows if len(r) >= 7 and r[2].replace('.', '').isdigit()]
        names = ['hw_slowdown', 'hw_thermal_slowdown', 'sw_thermal_slowdown', 'sw_power_cap']
        reasons = sorted({names[i] for r in self.rows if len(r) >= 7 for i in range(4) if r[3 + i].lower().startswith('active')})
        return {'sm_mhz': float(np.median(sm)) if sm else None, 'sm_max_mhz': max(mx) if mx else None, 'reasons': reasons, 'samples': len(sm)}


def make_scene(rank, n_batches=N_BATCHES):
    from xrnerf_b200 import synth
    grid = synth.lego_like_density_grid(0)
    bf, _ = synth.bitfield_from_grid_numpy(grid)
    batches = [synth.ray_batch(N_RAYS, seed=1000 * rank + b)[:2] for b in range(n_batches)]
    table, dens, color = synth.ngp_weights(seed=0)
    return bf, batches, (table, dens, color)


# ------------------------------------------------------------------------------------------- CPU arm (oracle; timing only)
def _omp_configure():
    """libgomp reads its environment when it is first loaded: pin and size the team BEFORE anything that links it (numpy/torch/the oracle .so) is imported.
    torchrun exports OMP_NUM_THREADS=1, which round 1 overrode too late (VERDICT W8: 8.7 K ... 47 K rays/s for the same code)."""
    os.environ['OMP_NUM_THREADS'] = str(os.cpu_count() or 1)
    os.environ.setdefault('OMP_PROC_BIND', 'close')
    os.environ.setdefault('OMP_PLACES', 'cores')
    os.environ.setdefault('OMP_DYNAMIC', 'false')


def _omp_set_threads(k):
    import ctypes
    try:
        ctypes.CDLL('libgomp.so.1').omp_set_num_threads(int(k))
        return True
    except Exception:
        return False


_CPU_SCENE = {}


def cpu_reference_rate(sample_rays, reps=3, threads=None):
    """rays/s of the reference path on the host cores: reference march/composite kernels compiled for CPU (oracle/_ref) + C restatement of the tcnn field
    (oracle port), OpenMP with `threads` threads (default: all), best of `reps`."""
    from oracle import oracle as O
    if 'port' not in _CPU_SCENE:
        O.build()
        _CPU_SCENE['port'] = O.Port()
        _CPU_SCENE['ref'] = O.Ref(serial=False) if O.have_ref() else None
        _CPU_SCENE['scene'] = make_scene(0, 1)
    port, ref = _CPU_SCENE['port'], _CPU_SCENE['ref']
    use_ref = ref is not None
    bf, batches, (table, dens, color) = _CPU_SCENE['scene']
    cores = os.cpu_count() or 1
    threads = cores if threads is None else int(threads)
    _omp_set_threads(threads)
    o, d = batches[0][0][:sample_rays], batches[0][1][:sample_rays]
    m = ref or port
    best = None
    n_samples = 0
    for _ in range(reps):
        t0 = time.perf_counter()
        c, _, ns, cnt = m.rays_sampler(o, d, bf, sample_rays * BUDGET)
        coords = c[:cnt[1]]
        raw = port.ngp_mlp_forward(table, dens, color, np.ascontiguousarray(coords[:, :3]), np.ascontiguousarray(coords[:, 4:]))
        rgb_cpu, alpha_cpu = m.calc_rgb_inference(raw, coords, ns, np.zeros(3, np.float32))
        dt = time.perf_counter() - t0
        cpu_reference_rate.last = (np.asarray(rgb_cpu).copy(), np.asarray(alpha_cpu).copy(), np.asarray(ns)[:, 0].copy())
        best = dt if best is None else min(best, dt)
        n_samples = int(cnt[1])
    kind = 'reference' if use_ref else 'port'
    sample = (f'{sample_rays} rays of batch 0 ({n_samples} samples): march+composite = reference ngp_raymarch kernels compiled for CPU '
              f'(oracle/_ref, OpenMP), field = C restatement of tcnn (oracle port, OpenMP); {threads} threads (OMP_PROC_BIND=close, OMP_PLACES=cores), best of {reps}') if use_ref else \
             f'{sample_rays} rays of batch 0 ({n_samples} samples), plain-C oracle port, OpenMP, {threads} threads; best of {reps}'
    return sample_rays / best, threads, kind, sample, best


def cpu_thread_sweep(sample_rays, reps=3):
    """thread counts {1, 16, 64, all}: the fastest setting is the baseline, every setting is reported"""
    cores = os.cpu_count() or 1
    sweep = {}
    for k in sorted({1, min(16, cores), min(64, cores), cores}):
        r, _, kind, sample, best = cpu_reference_rate(sample_rays, reps=reps, threads=k)
        sweep[k] = (r, kind, sample, best)
    k_best = max(sweep, key=lambda k: sweep[k][0])
    r, kind, sample, best = sweep[k_best]
    return r, k_best, kind, sample + f'; thread sweep rays/s: ' + ', '.join(f'{k}: {v[0]:.0f}' for k, v in sweep.items()), best


def run_reference(args):
    rank = int(os.environ.get('RANK', '0'))
    if rank != 0:
        return
    t_start = time.time()
    sample_rays = 8192
    for _ in range(max(args.warmup, 1)):
        cpu_reference_rate(1024, reps=1)
    # thread sweep once (which team size is fastest on this box), then the timed steps at that setting
    _, k_best, kind, _, _ = cpu_thread_sweep(2048, reps=2)
    rates, per = [], []
    for _ in range(args.steps):
        r, cores, kind, sample, dt = cpu_reference_rate(sample_rays, reps=1, threads=k_best)
        rates.append(r); per.append(dt)
        if time.time() - t_start > 240:
            break
    value = float(np.median(rates))
    line = {
        'impl': 'reference', 'metric': METRIC, 'value': value, 'unit': 'rays/s', 'n_gpus': args.gpus, 'steps': len(rates), 'warmup': args.warmup,
        'ms_per_step': float(np.median(per) * 1e3), 'higher_is_better': True, 'scaling': 'weak', 'vs_baseline': None, 'dtype': 'f16', 'data': 'synthetic',
        'config': {'workload': WORKLOAD, 'note': f'each step = a bounded sample of {sample_rays} rays of the 65536-ray batch on the host cores; median over the steps; '
                                                 f'spread min {min(rates):.0f} / max {max(rates):.0f} rays/s'},
        'cpu_baseline': {'value': value, 'unit': 'rays/s', 'cores': cores, 'kind': kind, 'sample': sample + f'; team size chosen by a sweep over 1/16/64/all threads'},
        'e2e': {'value': value, 'unit': 'rays/s', 'h2d_bytes_per_step': 0, 'd2h_bytes_per_step': 0},
    }
    print(json.dumps(line), flush=True)


# ------------------------------------------------------------------------------------------- GPU reference leg (BASELINE.md B4)
def _torch_field_fp32(pts01, dirs01, hash_params, dens_params, color_params, chunk=1 << 18):
    """fp32 PyTorch restatement of HashNerfMLP.run_mlp (hashnerf_mlp.py:55-79) for the naive GPU path: tiny-cuda-nn is not in this image, so its hash grid (16 levels x 2,
    T = 2^19, base 16, scale 1.3819), SH degree 4 and the two bias-free ReLU MLPs (32-64-16, 32-64-64-16) are written with torch ops. Timing stand-in only (the parity
    oracle is oracle/tcnn_oracle.c); returns raw [n, 4] = (rgb, density)."""
    import torch
    dev = pts01.device
    L, T, base, pls = 16, 1 << 19, 16, 1.38191288
    scales, ress, offs, off = [], [], [0], 0
    for l in range(L):
        sc = float(np.float32(np.exp2(np.float32(l) * np.log2(np.float32(pls))) * base - 1.0))
        res = int(np.ceil(sc)) + 1
        n = min(((min(res ** 3, 0x7fffffff) + 7) // 8) * 8, T)
        scales.append(sc); ress.append(res); off += n; offs.append(off)
    table = hash_params.view(-1, 2)
    Wd = [dens_params[:64 * 32].view(64, 32), dens_params[64 * 32:].view(16, 64)]
    Wc = [color_params[:64 * 32].view(64, 32), color_params[64 * 32:64 * 32 + 64 * 64].view(64, 64), color_params[64 * 32 + 64 * 64:].view(16, 64)]
    out = torch.empty((pts01.shape[0], 4), dtype=torch.float32, device=dev)
    for a in range(0, pts01.shape[0], chunk):
        x, dd = pts01[a:a + chunk], dirs01[a:a + chunk]
        feats = []
        for l in range(L):
            hs, res = offs[l + 1] - offs[l], ress[l]
            p = x * scales[l] + 0.5
            fl = torch.floor(p)
            fr = p - fl
            g = fl.to(torch.int64)
            acc = 0
            for c in range(8):
                q = g + torch.tensor([c & 1, (c >> 1) & 1, (c >> 2) & 1], device=dev)
                w = torch.where(torch.tensor([bool(c & 1), bool(c & 2), bool(c & 4)], device=dev), fr, 1 - fr).prod(-1, keepdim=True)
                if res ** 3 <= hs:
                    idx = q[:, 0] + q[:, 1] * res + q[:, 2] * res * res
                else:
                    idx = (q[:, 0] ^ (q[:, 1] * 2654435761 & 0xffffffff) ^ (q[:, 2] * 805459861 & 0xffffffff)) & 0xffffffff
                acc = acc + w * table[offs[l] + idx % hs]
            feats.append(acc)
        enc = torch.cat(feats, -1)
        h = torch.relu(enc @ Wd[0].t()) @ Wd[1].t()
        v = dd * 2 - 1
        X, Y, Z = v[:, 0], v[:, 1], v[:, 2]
        xy, xz, yz, x2, y2, z2 = X * Y, X * Z, Y * Z, X * X, Y * Y, Z * Z
        sh = torch.stack([torch.full_like(X, 0.28209479177387814), -0.48860251190291987 * Y, 0.48860251190291987 * Z, -0.48860251190291987 * X, 1.0925484305920792 * xy,
                          -1.0925484305920792 * yz, 0.94617469575755997 * z2 - 0.31539156525251999, -1.0925484305920792 * xz, 0.54627421529603959 * (x2 - y2),
                          0.59004358992664352 * Y * (-3.0 * x2 + y2), 2.8906114426405538 * xy * Z, 0.45704579946446572 * Y * (1.0 - 5.0 * z2),
                          0.3731763325901154 * Z * (5.0 * z2 - 3.0), 0.45704579946446572 * X * (1.0 - 5.0 * z2), 1.4453057213202769 * Z * (x2 - y2),
                          0.59004358992664352 * X * (-x2 + 3.0 * y2)], -1)
        cin = torch.cat([h[:, 1:], sh, torch.ones_like(X)[:, None]], -1)
        c = torch.relu(torch.relu(cin @ Wc[0].t()) @ Wc[1].t()) @ Wc[2].t()
        out[a:a + chunk, :3] = c[:, :3]; out[a:a + chunk, 3] = h[:, 0]
    return out


def reference_gpu_leg(dev, bf, rays, field, ours_chain_ms, ours_field_ms):
    """BASELINE.md B4: the reference's own `raymarch_cuda` kernels, built unmodified for sm_90a (oracle/build_ref_cuda.py), timed on this GPU on the same 65 536-ray batch,
    occupancy grid and weights, with the calls and allocations of the reference's Python wrappers (rays_sampler.py:20-27 zero-fills coords for n_rays x 1024 samples on every
    call; every *_api ends in cudaDeviceSynchronize). Field: fp32 torch restatement (tcnn is not in the image). Per-op times next to ours through the identical signatures."""
    import torch
    sys.path.insert(0, ROOT)
    try:
        from oracle import build_ref_cuda
        ref = build_ref_cuda.load_module()
    except Exception as e:   # noqa: BLE001
        return {'unavailable': 'reference CUDA extension failed to load: ' + repr(e)[:160]}
    if ref is None:
        return {'unavailable': 'oracle/_ref/cuda/raymarch_cuda_ref.so not built (python oracle/build_ref_cuda.py where /root/reference exists)'}
    import xrnerf_b200.raymarch_cuda as ours
    o, d = rays
    n = o.shape[0]
    md = torch.tensor([[0, 0, 0, 0, .5, .5, 1111., 1111., 0, 0, 0]], dtype=torch.float32, device=dev)
    xf = torch.zeros((1, 4, 3), dtype=torch.float32, device=dev)
    ids = torch.zeros(n, dtype=torch.int32, device=dev)
    cap = n * BUDGET
    bg = torch.zeros(3, dtype=torch.float32)

    def timed(fn, reps=5):
        fn(); torch.cuda.synchronize()
        ts = []
        for _ in range(reps):
            a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            a.record(); fn(); b.record(); torch.cuda.synchronize()
            ts.append(a.elapsed_time(b))
        return float(np.median(ts))

    state = {}

    def march(mod, stock_alloc):
        def f():
            if mod is ours:
                ours.reset_rng(ray_sampler=0)
            m = n * 1024 if stock_alloc else cap
            coords = torch.zeros((m, 7), dtype=torch.float32, device=dev)
            ridx = torch.zeros((n, 1), dtype=torch.int32, device=dev); ns = torch.zeros((n, 2), dtype=torch.int32, device=dev); cnt = torch.zeros(2, dtype=torch.int32, device=dev)
            mod.rays_sampler_api(o, d, bf, md, ids, xf, 0.0, 1.0, 0.05, 1.0 / 256, coords, ridx, ns, cnt)
            state[mod] = (coords, ns, cnt)
        return f
    t_ref_march_stock = timed(march(ref, True), reps=3)
    t_ref_march = timed(march(ref, False))
    t_our_march = timed(march(ours, False))
    s_ref, s_our = int(state[ref][2][1]), int(state[ours][2][1])
    coords_r, ns_r, _ = state[ref]
    pts, dirs = coords_r[:s_ref, :3].contiguous(), coords_r[:s_ref, 4:7].contiguous()
    with torch.no_grad():
        hp, dp, cp = field.hash_params.detach().float(), field.density_params.detach().float(), field.color_params.detach().float()
        t_field_torch = timed(lambda: state.__setitem__('raw', _torch_field_fp32(pts, dirs, hp, dp, cp)), reps=3)
        raw_t = state['raw']
        raw_o = field.run_mlp(pts, dirs).float()
    field_err = float((raw_t - raw_o).abs().max())
    rgb = torch.zeros((n, 3), dtype=torch.float32, device=dev); alpha = torch.zeros((n, 1), dtype=torch.float32, device=dev)
    raw_c = raw_o.contiguous()
    coords_c = coords_r[:s_ref].contiguous()
    t_ref_comp = timed(lambda: ref.calc_rgb_influence_api(raw_c, coords_c, ns_r, bg, 2, 3, 0.0, 1.0, rgb, alpha))
    rgb_ref = rgb.clone()
    t_our_comp = timed(lambda: ours.calc_rgb_influence_api(raw_c, coords_c, ns_r, bg, 2, 3, 0.0, 1.0, rgb, alpha))
    comp_err = float((rgb - rgb_ref).abs().max())
    naive_ms = t_ref_march_stock + t_field_torch + t_ref_comp
    return {'value': n / (naive_ms * 1e-3), 'unit': 'rays/s', 'ms_per_batch': naive_ms,
            'what': 'naive GPU path on this GPU, one 65 536-ray batch, sequential: reference rays_sampler (stock wrapper: coords zero-filled for n_rays x 1024 samples = 1.88 GB per call) '
                    '+ fp32 torch restatement of the tcnn field (tcnn absent from the image) + reference calc_rgb_inference; reference kernels = extensions/ngp_raymarch built '
                    'unmodified for sm_90a (oracle/build_ref_cuda.py)',
            'per_op_ms': {'rays_sampler': {'reference_stock_wrapper': t_ref_march_stock, 'reference_kernel_same_capacity_as_ours': t_ref_march, 'ours': t_our_march},
                          'field': {'torch_fp32_restatement': t_field_torch, 'ours': ours_field_ms},
                          'calc_rgb_inference': {'reference': t_ref_comp, 'ours': t_our_comp}},
            'ours_same_batch_sequential_ms': ours_chain_ms, 'speedup_sequential': naive_ms / ours_chain_ms,
            'cross_check': {'samples_reference_kernel': s_ref, 'samples_ours': s_our, 'note': 'nvcc contracts the reference\'s o + t*d into FMAs (default -fmad=true); the bit-exact parity '
                            'contract is the un-contracted CPU build of the same sources (oracle/_ref), so a handful of samples may differ here',
                            'max_abs_raw_torch_vs_ours': field_err, 'max_abs_rgb_composite_ref_vs_ours': comp_err}}



def nerf_convention_rays(dev, n, seed, with_radii=False):
    """BASELINE-convention rays for the NeRF / Mip-NeRF arms (VERDICT W9): Blender spiral pose (pose_spherical(theta, -30, 4.0), load_blender.py:22-29,72-75), 800x800 f=1111.1 camera,
    GetRays + GetViewdirs conventions (create.py:205-245,:437-448) through xrb_nerf_get_rays on `n` random pixels; near 2 / far 6 (load.py:58-59)."""
    import torch
    from xrnerf_b200 import _C, synth
    rng = np.random.default_rng(seed)
    pose = synth.pose_spherical(float(rng.uniform(-180, 180)), -30.0, 4.0)
    pix = torch.from_numpy(rng.integers(0, 800 * 800, n).astype(np.int32)).to(dev)
    c2w = (_C.C.c_float * 12)(*[float(v) for v in pose[:3, :4].reshape(-1)])
    o = torch.empty((n, 3), device=dev); d = torch.empty((n, 3), device=dev); v = torch.empty((n, 3), device=dev)
    r = torch.empty((n, 1), device=dev) if with_radii else None
    _C.check(_C.lib.xrb_nerf_get_rays(c2w, 800, 800, float(synth.FOCAL), float(synth.FOCAL), 400.0, 400.0, 0, _C.ptr(pix), n, _C.ptr(o), _C.ptr(d), _C.ptr(v), _C.ptr(r), _C.stream()), 'get_rays')
    return (o, d, v, r) if with_radii else (o, d, v)


def psnr_obj(a, b, what):
    err = np.abs(np.asarray(a, np.float64) - np.asarray(b, np.float64))
    mse = float((err ** 2).mean())
    return {'rays': int(a.shape[0]), 'max_abs_rgb_err': float(err.max()), 'psnr_vs_ref_db': float(-10.0 * np.log10(max(mse, 1e-20))), 'against': what}


# ------------------------------------------------------------------------------------------- our arm
def dump_outputs(path, arrays):
    """What each timed path (chain_*, fused_*) returned for its last timed batch, one float32 .npy per array (n_samples: per-ray sample counts). The inputs
    are seeded, so two builds run with the same arguments can be compared array by array."""
    os.makedirs(path, exist_ok=True)
    for name, t in arrays.items():
        np.save(os.path.join(path, f'{name}.npy'), t.float().cpu().numpy())


def run_ours(args):
    import torch
    import torch.distributed as dist
    from xrnerf_b200 import _C
    from xrnerf_b200.ngp import NgpField, NgpRenderer

    world = int(os.environ.get('WORLD_SIZE', '1'))
    rank = int(os.environ.get('RANK', '0'))
    local = int(os.environ.get('LOCAL_RANK', '0'))
    if not torch.cuda.is_available():
        raise SystemExit('bench.py: no CUDA device; xrnerf_b200 has no CPU fallback (use --impl reference for the CPU arm)')
    torch.cuda.set_device(local)
    if world > 1:
        dist.init_process_group('nccl', device_id=torch.device('cuda', local))
    dev = torch.device('cuda', local)

    bf_np, batches, (table, dens, color) = make_scene(rank)
    bf = torch.from_numpy(bf_np).to(dev)
    field = NgpField().to(dev)
    with torch.no_grad():
        field.hash_params.copy_(torch.from_numpy(table).to(dev)); field.density_params.copy_(torch.from_numpy(dens).to(dev)); field.color_params.copy_(torch.from_numpy(color).to(dev))
    P = max(1, args.pipeline)   # batches in flight: step i runs on stream i % P with its own workspace, so the (latency-bound) march of
    renderers = [NgpRenderer(field, samples_per_ray_budget=BUDGET) for _ in range(P)]   # batch i+1 overlaps the field kernel of batch i
    streams = [torch.cuda.Stream(device=dev) for _ in range(P)]
    dev_batches = [(torch.from_numpy(o).to(dev), torch.from_numpy(d).to(dev)) for (o, d) in batches]
    host_batches = [(torch.from_numpy(o).pin_memory(), torch.from_numpy(d).pin_memory()) for (o, d) in batches[:8]]

    def barrier():
        if world > 1:
            dist.barrier()
        torch.cuda.synchronize()

    main = torch.cuda.current_stream()

    def fork():
        e = torch.cuda.Event(); e.record(main)
        for st in streams:
            st.wait_event(e)

    def join():
        for st in streams:
            e = torch.cuda.Event(); e.record(st); main.wait_event(e)

    # ---- device-resident arm
    K, W = args.steps, args.warmup
    WU = max(W, 2 * P)      # untimed warm-up steps actually run: at least two per stream, so that every stream's renderer has allocated its workspace / outputs
    evf = [(torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)) for _ in range(K)]
    fork()
    for i in range(WU):
        with torch.cuda.stream(streams[i % P]):
            renderers[i % P].render(*dev_batches[i % N_BATCHES], bf)
    join()
    barrier()
    clocks = ClockSampler(local)
    if rank == 0:
        clocks.start()
    counters_log = []
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record(main)
    fork()
    for i in range(K):
        st = streams[i % P]
        with torch.cuda.stream(st):
            for e in evf[i]:
                e.record(st)                          # materialise the cudaEvent_t handles
            out = renderers[i % P].render(*dev_batches[(W + i) % N_BATCHES], bf, profile_events=evf[i])
            counters_log.append(out[3].clone())
    join()
    e1.record(main)
    barrier()
    last_chain = {'rgb': out[0].clone(), 'alpha': out[1].clone(), 'n_samples': out[2][:, 0].clone()}   # the renderer reuses its output buffers
    field_ms = [a.elapsed_time(b) for a, b in evf]
    samples = [int(c[1].item()) for c in counters_log]
    total_ms = float(e0.elapsed_time(e1))
    t = torch.tensor([total_ms], dtype=torch.float64, device=dev)
    if world > 1:
        dist.all_reduce(t, op=dist.ReduceOp.MAX)
    total_ms_max = float(t.item())
    clk = clocks.stop() if rank == 0 else None

    # ---- isolated pass (P = 1, one stream): the dominant kernel timed ALONE, so that kernel_ms <= the step it is part of (round 1 recorded the events while three other
    # streams shared the SMs: kernel_share_of_step 1.06 > 1). Distinct batches every step (inputs > L2); event pair around the field kernel inside xrb_ngp_render and
    # around the whole 5-launch call.
    KI_ = min(K, 24)
    ev_f = [(torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)) for _ in range(KI_)]
    ev_c = [(torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)) for _ in range(KI_)]
    iso_cnt = []
    for i in range(3):
        renderers[0].render(*dev_batches[(i + 40) % N_BATCHES], bf)
    barrier()
    for i in range(KI_):
        for e in ev_f[i]:
            e.record(main)
        ev_c[i][0].record(main)
        out = renderers[0].render(*dev_batches[(i + 48) % N_BATCHES], bf, profile_events=ev_f[i])
        ev_c[i][1].record(main)
        iso_cnt.append(out[3].clone())
    barrier()
    iso_field_ms = float(np.median([a.elapsed_time(b) for a, b in ev_f]))
    iso_chain_ms = float(np.median([a.elapsed_time(b) for a, b in ev_c]))
    iso_samples = float(np.mean([int(c[1].item()) for c in iso_cnt]))

    # ---- the roof the gather actually runs under: random 4-byte reads from an L2-resident table of the hash table's size (xrb_micro_gather). Every read costs one 32-byte
    # sector; the rate is reported as sectors x 32 B / s next to the HBM copy peak the contract's roofline is quoted against.
    l2_roof = None
    try:
        tbl = torch.empty(24_400_000 // 4, dtype=torch.int32, device=dev).random_()
        sink = torch.zeros(4, dtype=torch.int32, device=dev)
        n_loads = _C.C.c_int64(0)
        res_roof = {}
        for wbytes in (4, 32):
            nrec = tbl.numel() * 4 // wbytes
            for _ in range(2):
                _C.check(_C.lib.xrb_micro_gather(_C.ptr(tbl), nrec, wbytes, 64, _C.C.byref(n_loads), _C.ptr(sink), _C.stream()), 'micro_gather')
            r0, r1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            r0.record(main)
            for _ in range(5):
                _C.check(_C.lib.xrb_micro_gather(_C.ptr(tbl), nrec, wbytes, 64, _C.C.byref(n_loads), _C.ptr(sink), _C.stream()), 'micro_gather')
            r1.record(main)
            torch.cuda.synchronize()
            res_roof[wbytes] = 5 * n_loads.value / (r0.elapsed_time(r1) * 1e-3)
        l2_roof = {'random_4B_loads_per_s': res_roof[4], 'random_32B_loads_per_s': res_roof[32], 'sector_GBs_at_4B': res_roof[4] * 32 / 1e9, 'sector_GBs_at_32B': res_roof[32] * 32 / 1e9,
                   'what': 'xrb_micro_gather: random reads from a 24.4 MB (L2-resident) table, 8 independent loads in flight per thread, SMs x 8 CTAs x 256 threads; one 32-byte sector per load'}
        del tbl
    except Exception as e:
        l2_roof = {'error': repr(e)[:200]}

    # ---- single-launch arm: the same K steps through xrb_ngp_render_fused (march + encode + wgmma MLPs + composite in ONE kernel per batch)
    evk = [(torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)) for _ in range(K)]
    fork()
    for i in range(WU):
        with torch.cuda.stream(streams[i % P]):
            renderers[i % P].render_fused(*dev_batches[i % N_BATCHES], bf)
    join()
    barrier()
    f0, f1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    f0.record(main)
    fork()
    ns_log = []
    kev = not os.environ.get('XRB_BENCH_NO_KEVENTS')
    th0 = time.perf_counter()
    for i in range(K):
        st = streams[i % P]
        with torch.cuda.stream(st):
            if kev:
                evk[i][0].record(st)
            outf = renderers[i % P].render_fused(*dev_batches[(W + i) % N_BATCHES], bf)
            if kev:
                evk[i][1].record(st)
            if i < P:
                ns_log.append(outf[2])   # per-ray sample counts of this batch; reduced AFTER the timed region (a first-use torch reduction costs ~20 ms of lazy module loading)
    th1 = time.perf_counter()
    join()
    f1.record(main)
    barrier()
    last_fused = {'rgb': outf[0].clone(), 'alpha': outf[1].clone(), 'n_samples': outf[2].clone()}
    if os.environ.get('XRB_BENCH_DEBUG') and kev:
        gaps = [evk[i][1].elapsed_time(evk[i + 1][0]) for i in range(K - 1)] if P == 1 else []
        kms = [a.elapsed_time(b) for a, b in evk]
        print('[bench] kernel ms: first 8', [round(x, 3) for x in kms[:8]], 'p50', round(float(np.median(kms)), 3), '| gaps ms first 8', [round(x, 3) for x in gaps[:8]], 'p50', round(float(np.median(gaps)), 3) if gaps else None, 'max', round(max(gaps), 3) if gaps else None, file=sys.stderr, flush=True)
    if os.environ.get('XRB_BENCH_DEBUG'):
        print(f'[bench] fused arm: host issue {1e3 * (th1 - th0) / K:.3f} ms/step, total wall {1e3 * (time.perf_counter() - th0) / K:.3f} ms/step', file=sys.stderr, flush=True)
    fused_total = torch.tensor([float(f0.elapsed_time(f1))], dtype=torch.float64, device=dev)
    if world > 1:
        dist.all_reduce(fused_total, op=dist.ReduceOp.MAX)
    fused_total_ms = float(fused_total.item())
    fused_kernel_ms = float(np.mean([a.elapsed_time(b) for a, b in evk])) if kev else fused_total_ms / K
    fused_samples = float(np.mean([float(x.sum().item()) for x in ns_log]))
    use_fused = args.path == 'fused' or (args.path == 'auto' and fused_total_ms < total_ms_max)
    if args.dump_outputs and rank == 0:   # both timed paths, whichever of them the headline reports
        dump_outputs(args.dump_outputs, {**{'chain_' + k: v for k, v in last_chain.items()}, **{'fused_' + k: v for k, v in last_fused.items()}})
    del last_chain, last_fused

    # ---- end-to-end arm: host (pinned) rays in, rgb+alpha out, every step, through the public API; P batches in flight
    slots = [dict(rgb_h=torch.empty((N_RAYS, 3), dtype=torch.float32).pin_memory(), alpha_h=torch.empty((N_RAYS, 1), dtype=torch.float32).pin_memory(),
                  o_d=torch.empty((N_RAYS, 3), dtype=torch.float32, device=dev), d_d=torch.empty((N_RAYS, 3), dtype=torch.float32, device=dev), done=None) for _ in range(P)]

    def e2e_step(i):
        sl, st = slots[i % P], streams[i % P]
        if sl['done'] is not None:
            sl['done'].synchronize()                 # the caller consumes the pixels of the batch that used this slot before reusing it
        o_h, d_h = host_batches[i % len(host_batches)]
        with torch.cuda.stream(st):
            sl['o_d'].copy_(o_h, non_blocking=True); sl['d_d'].copy_(d_h, non_blocking=True)
            rgb, alpha = (renderers[i % P].render_fused if use_fused else renderers[i % P].render)(sl['o_d'], sl['d_d'], bf)[:2]
            sl['rgb_h'].copy_(rgb, non_blocking=True); sl['alpha_h'].copy_(alpha, non_blocking=True)
            sl['done'] = torch.cuda.Event(); sl['done'].record(st)

    def e2e_drain():
        for sl in slots:
            if sl['done'] is not None:
                sl['done'].synchronize(); sl['done'] = None
    fork()
    for i in range(WU):
        e2e_step(i)
    e2e_drain()
    barrier()
    t0 = time.perf_counter()
    g0, g1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    g0.record(main)
    fork()
    for i in range(K):
        e2e_step(W + i)
    e2e_drain()
    join()
    g1.record(main)
    barrier()
    e2e_wall_ms = (time.perf_counter() - t0) * 1e3
    e2e_ms = torch.tensor([max(g0.elapsed_time(g1), 0.0)], dtype=torch.float64, device=dev)
    if world > 1:
        dist.all_reduce(e2e_ms, op=dist.ReduceOp.MAX)
    e2e_ms = float(e2e_ms.item())

    # ---- whole-image inference (SURVEY 8d C2 "full 640 000-ray images"): 800x800 spiral views rendered in pixel order, one call per image.
    # Placed before the training arm so that it renders the same (initial) weights as the batch arms.
    image_arm = None
    if not args.no_image:
        try:
            from xrnerf_b200 import synth as _synth
            poses = _synth.spiral_poses_ngp(40)
            n_views = 4
            views = []
            for v in range(n_views):
                o_np, d_np = _synth.get_rays_ngp(poses[(rank * n_views + v * 7) % 40])
                views.append((torch.from_numpy(o_np).to(dev), torch.from_numpy(d_np).to(dev)))
            n_img = views[0][0].shape[0]
            img_r = NgpRenderer(field, samples_per_ray_budget=BUDGET)
            res = {}
            for path in ('chain', 'fused'):
                fn = (lambda o_, d_: img_r.render_fused(o_, d_, bf)) if path == 'fused' else (lambda o_, d_: img_r.render(o_, d_, bf))
                for v in range(2):
                    fn(*views[v])
                barrier()
                i0, i1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                KI = 12
                ns_acc = torch.zeros((), dtype=torch.float64, device=dev)
                ns_acc += 0.0                                  # first-use kernels loaded before the timed region
                i0.record()
                for i in range(KI):
                    out_i = fn(*views[i % n_views])
                i1.record()
                barrier()
                im = torch.tensor([i0.elapsed_time(i1)], dtype=torch.float64, device=dev)
                if world > 1:
                    dist.all_reduce(im, op=dist.ReduceOp.MAX)
                for v in range(n_views):                       # samples of EVERY timed image (the views are cycled; counts re-measured outside the timed region)
                    ns_v = fn(*views[v])[2]
                    ns_acc += (ns_v[:, 0] if ns_v.dim() == 2 else ns_v).double().sum() * (KI // n_views)
                spr = float(ns_acc.item()) / (n_img * KI)
                ms_img = float(im.item()) / KI
                img_bytes = n_img * spr * (512 if path == 'fused' else BYTES_PER_SAMPLE) + n_img * 44          # gather (+ coords/raw round trip on the chain path) + ray I/O
                pk, _ = peaks()
                res[path] = {'value': world * n_img * KI / (float(im.item()) * 1e-3), 'unit': 'rays/s', 'ms_per_image': ms_img, 'samples_per_ray_mean': spr,
                             'roofline': {'bound': 'hbm', 'achieved': img_bytes / (ms_img * 1e-3) / 1e9, 'peak': pk, 'unit': 'GB/s', 'frac': img_bytes / (ms_img * 1e-3) / 1e9 / pk,
                                          'algorithmic_bytes_per_image': img_bytes, 'note': 'whole call(s) of one image; gather served by L1/L2 (coherent rays)'}}
            image_arm = dict(res, what='800x800 spiral views in pixel order (coherent rays), 640 000 rays per call, sequential calls on one stream; 4 distinct views cycled (61 MB of rays)')
        except Exception as e:   # an auxiliary arm must never take the headline line down
            image_arm = {'error': repr(e)[:300]}

    # ---- parity sample (N=1): this arm's render of the 4096 rays the CPU reference arm renders below, taken BEFORE the training arm updates the weights
    parity_gpu = {}
    if world == 1:
        prn = NgpRenderer(field, samples_per_ray_budget=BUDGET, bg=(0., 0., 0.))
        po, pd = dev_batches[0][0][:4096].contiguous(), dev_batches[0][1][:4096].contiguous()
        for path in ('chain', 'fused'):
            prn.calls = 0                                   # same jitter stream as the CPU arm's call 0 (pcg32 seed 9121, SURVEY Q9)
            if path == 'fused':
                rgb_g, _, ns_g = prn.render_fused(po, pd, bf)
            else:
                rgb_g, _, ns_g, _ = prn.render(po, pd, bf)
            torch.cuda.synchronize()
            ns_np = ns_g.cpu().numpy()
            parity_gpu[path] = (rgb_g.cpu().numpy().copy(), (ns_np[:, 0] if ns_np.ndim == 2 else ns_np).copy())

    # ---- training arm (BASELINE configs[4] shape: 65 536 rays per rank per step; march + compaction + field fwd/bwd (wgmma) + composite fwd/bwd + loss + gradient exchange +
    # fused Adam; device-resident batches, synthetic targets). T = 2^20 compacted samples so that NO ray of the batch is truncated away (the reference's 2^18 is sized for its
    # adaptive ~24 K-ray batches); `trained_rays_per_step` is counted on the device (rays whose every marched sample took part).
    train = None
    if not args.no_train:
        try:
            from xrnerf_b200.train import NgpTrainer
            T_TRAIN = 1 << 20
            tr = NgpTrainer(field, bf, N_RAYS, target_batch_size=T_TRAIN, grad_comm=args.grad_comm)
            tgt = torch.rand((N_RAYS, 3), device=dev); bgc = torch.zeros((N_RAYS, 3), device=dev)
            nb = lambda i: dev_batches[i % N_BATCHES]
            for i in range(max(W, 3)):
                tr.step(*nb(i), tgt, bgc, next_rays=nb(i + 1))
            barrier()
            t0e, t1e = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            torch.cuda.synchronize()
            trained0 = int(tr.trained_total.item())                     # batches prepared so far (warm-up + the first timed batch, prepared one step ahead)
            t0e.record()
            th_ = time.perf_counter()
            for i in range(K):
                tr.step(*nb(W + i), tgt, bgc, next_rays=nb(W + i + 1))
            host_issue_ms = (time.perf_counter() - th_) * 1e3 / K       # host time to ENQUEUE a step (no sync inside): above ms_per_step means the step is launch-bound
            t1e.record()
            barrier()
            tm = torch.tensor([t0e.elapsed_time(t1e)], dtype=torch.float64, device=dev)
            # K batches were prepared (one step ahead) inside the loop: their fully-trained ray count is what the device counter gained
            tsum = torch.tensor([float(int(tr.trained_total.item()) - trained0)], dtype=torch.float64, device=dev)
            if world > 1:
                dist.all_reduce(tm, op=dist.ReduceOp.MAX)
                dist.all_reduce(tsum, op=dist.ReduceOp.SUM)
            train = {'value': float(tsum.item()) / (float(tm.item()) * 1e-3), 'unit': 'rays/s (trained rays only)', 'ms_per_step': float(tm.item()) / K,
                     'rays_per_step': world * N_RAYS, 'trained_rays_per_step': float(tsum.item()) / K, 'target_batch_size': T_TRAIN,
                     'compacted_samples_per_step_rank0': int(tr.compacted_samples().item()), 'grad_comm': tr.grad_comm, 'host_issue_ms_per_step': host_issue_ms, 'field_backward': 'wgmma' if tr.bwd_impl == 1 else 'cuda cores',
                     'what': 'march + compaction (aux stream, one step ahead) | field fwd (wgmma) + composite fwd + Huber x5 + composite bwd + field bwd (wgmma dX/dW) + gradient exchange '
                             '+ Adam (world>1, grad_comm=peer: ONE optimiser kernel over NVLink peer memory - every rank sums all ranks\' bf16 gradients for its 1/N of the table, runs Adam on it and '
                             'stores the new fp16 values into every rank\'s working table, csrc/peer_adam.cu; grad_comm=sharded: NCCL bf16 reduce-scatter -> sharded Adam -> fp16 all-gather) + cell-image refresh'}
            if tr.px is not None:
                tr.px.check()                      # raises if a rank timed out inside the exchange kernels
                train['peer_exchange'] = 'ok'
                tr.close()
            del tr
        except Exception as e:   # an auxiliary arm must never take the headline line down
            import traceback
            train = {'error': repr(e)[:300], 'trace': traceback.format_exc()[-600:]}

    # ---- occupancy-grid update (ngp_grid_sampler.py:90-166; every 16 training steps): candidate cells -> density query -> splat -> EMA -> bitfield + mean
    grid_upd = None
    if not args.no_grid:
        try:
            from xrnerf_b200 import registry as R, synth
            from xrnerf_b200.registry.mlps import HashNerfMLP
            smp = R.build_sampler(dict(type='NGPGridSampler', update_grid_freq=16, update_block_size=5000000, n_rays_per_batch=4096, cone_angle_constant=0.00390625, near_distance=0.2,
                                       target_batch_size=1 << 18, rgb_activation=2, density_activation=3))
            poses = synth.spiral_poses_ngp(40)
            smp.set_data(dict(poses=poses, focal=np.full((40, 2), synth.FOCAL), aabb_scale=1, aabb_range=(0.0, 1.0), metadata=synth.metadata_for(40)), dict(H=800, W=800))
            smp.check_device({'rays_o': dev_batches[0][0]})

            class _Density:   # the sampler only needs run_density (hashnerf_mlp.py:107-111)
                def run_density(self, pts):
                    return field.run_density(pts)
            dm = _Density()
            M = 128 ** 3
            modes = {}
            for name, (nu, nn_) in (('warmup_phase_uniform_M', (M, 0)), ('steady_quarter_plus_quarter', (M // 4, M // 4))):
                for _ in range(2):
                    smp.update_density_grid_func(nu, nn_, dm)
                barrier()
                u0, u1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                KU = 5
                u0.record()
                for _ in range(KU):
                    smp.update_density_grid_func(nu, nn_, dm)
                u1.record()
                barrier()
                ms = u0.elapsed_time(u1) / KU
                n_q = nu + nn_
                # algorithmic HBM stream (SURVEY 8d): tmp zero-fill 64 MB + EMA read grid+tmp, write grid (192 MB) + bitfield pass reads level grids (64 MB) writes 2 MB
                # + per candidate 12+4 B written and read, 4 B density, 4 B splat atomic; the density query's gathers (512 B/cell) are L2 traffic
                stream_bytes = (64 + 192 + 66) * 2 ** 20 + n_q * (2 * 16 + 4 + 4)
                modes[name] = {'ms_per_update': ms, 'ms_per_training_step_amortised': ms / 16, 'candidate_cells': n_q, 'hbm_stream_bytes': stream_bytes,
                               'stream_gbs': stream_bytes / (ms * 1e-3) / 1e9}
            grid_upd = dict(modes, what='NGPGridSampler.update_density_grid_func: generate_grid_samples x2, density-only field (wgmma), splat (atomicMax), EMA, bitfield + cascade pooling + mean')
        except Exception as e:   # an auxiliary arm must never take the headline line down
            grid_upd = {'error': repr(e)[:300]}

    # ---- all-ones occupancy grid (SURVEY 8d C2(i): the first 256 training iterations, ngp_grid_sampler.py:168-174): every cell occupied, rays carry hundreds of samples
    all_ones = None
    if not args.no_image:
        try:
            n_ao = 8192
            bf_ones = torch.full_like(bf, 255)
            ao_r = NgpRenderer(field, samples_per_ray_budget=1024)
            res_ao = {}
            for path in ('chain', 'fused'):
                fn = (lambda o_, d_: ao_r.render_fused(o_, d_, bf_ones)) if path == 'fused' else (lambda o_, d_: ao_r.render(o_, d_, bf_ones))
                for i in range(2):
                    fn(dev_batches[i][0][:n_ao], dev_batches[i][1][:n_ao])
                barrier()
                a0, a1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                KA = 6
                a0.record()
                for i in range(KA):
                    out_a = fn(dev_batches[(i + 2) % N_BATCHES][0][:n_ao], dev_batches[(i + 2) % N_BATCHES][1][:n_ao])
                a1.record()
                barrier()
                ns_a = out_a[2]
                spr_a = float((ns_a[:, 0] if ns_a.dim() == 2 else ns_a).float().mean().item())
                ms_a = a0.elapsed_time(a1) / KA
                res_ao[path] = {'value': world * n_ao / (ms_a * 1e-3), 'unit': 'rays/s', 'ms_per_batch': ms_a, 'samples_per_ray_mean': spr_a, 'samples_per_s': world * n_ao * spr_a / (ms_a * 1e-3)}
            all_ones = dict(res_ao, what=f'all-ones bitfield, {n_ao}-ray batches (sample budget 1024 per ray on the chain path), sequential calls on one stream')
            del ao_r
        except Exception as e:
            all_ones = {'error': repr(e)[:300]}

    # ---- NeRF arm (BASELINE configs[2]: hierarchical 64 + 128, 800x800-shaped rays): fused wgmma NerfMLP path, device-resident rays
    nerf = None
    if not args.no_nerf:
        try:
            from xrnerf_b200 import registry as R
            from xrnerf_b200.nerf import NerfRenderer
            mlp_cfg = dict(type='NerfMLP', skips=[4], netdepth=8, netwidth=256, netchunk=1024 * 32, output_ch=5, use_viewdirs=True, embedder=dict(type='BaseEmbedder', i_embed=0, multires=10, multires_dirs=4))
            net = R.build_network(dict(type='NerfNetwork', cfg=dict(phase='test', N_importance=128, is_perturb=False, chunk=1024 * 32, bs_data='rays_o'), mlp=mlp_cfg, mlp_fine=mlp_cfg,
                                       render=dict(type='NerfRender', white_bkgd=True, raw_noise_std=0))).to(dev)
            nr = NerfRenderer(net, near=2.0, far=6.0, n_samples=64)
            n_nerf = 32768
            nerf_rays = [nerf_convention_rays(dev, n_nerf, 500 + 10 * rank + b) for b in range(8)]
            for _ in range(3):
                nr.render(*nerf_rays[0])
            barrier()
            n0, n1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            KN = max(3, min(K, 20))
            n0.record()
            for i in range(KN):
                nr.render(*nerf_rays[i % 8])
            n1.record()
            barrier()
            nm = torch.tensor([n0.elapsed_time(n1)], dtype=torch.float64, device=dev)
            if world > 1:
                dist.all_reduce(nm, op=dist.ReduceOp.MAX)
            rps = world * n_nerf * KN / (float(nm.item()) * 1e-3)
            flop_per_ray = (64 + 192) * 593408 * 2
            tpeak, tsrc = tensor_peak()
            # CPU baseline leg of this arm (rank 0, N=1): BASELINE configs[0] shape - 1024 rays x 64 samples, coarse network only - through the numpy oracle
            # (embed -> 12-layer NerfMLP -> composite; multi-threaded BLAS on the box's host cores). Checker code, timed only.
            nerf_cpu = None
            nerf_parity = None
            if world == 1:
                try:
                    from oracle import nerf_oracle as NO
                    sd = {k: v.detach().cpu().numpy() for k, v in net.state_dict().items()}
                    # parity of THIS arm on its own rays: 512 of the timed rays through the numpy restatement of the reference's hierarchical forward (fp32) vs the fused wgmma path (fp16 operands)
                    po, pd, pv = (t[:512].contiguous() for t in nerf_rays[0])
                    got = nr.render(po, pd, pv)
                    o_p, d_p, v_p = po.cpu().numpy(), pd.cpu().numpy(), pv.cpu().numpy()
                    z_p = np.broadcast_to(np.linspace(2, 6, 64, dtype=np.float32), (512, 64)).copy()
                    pts_p = o_p[:, None] + d_p[:, None] * z_p[..., None]
                    c_p = NO.nerf_render(NO.nerf_mlp(sd, NO.embed(pts_p, v_p), 63, 27, prefix='mlp.').reshape(512, 64, 4), z_p, d_p, white_bkgd=True)
                    z2_p, pts2_p, _ = NO.sample_pdf(z_p, c_p['weights'], o_p, d_p, 128)
                    f_p = NO.nerf_render(NO.nerf_mlp(sd, NO.embed(pts2_p, v_p), 63, 27, prefix='mlp_fine.').reshape(512, 192, 4), z2_p, d_p, white_bkgd=True)
                    nerf_parity = psnr_obj(got['rgb'].cpu().numpy(), f_p['rgb'], 'oracle/nerf_oracle.py (numpy fp32 restatement of NerfNetwork.forward, pinned to the reference by tests/golden)')
                    o_c = o_p.repeat(2, 0); d_c = d_p.repeat(2, 0)
                    z_c = np.broadcast_to(np.linspace(2, 6, 64, dtype=np.float32), (1024, 64)).copy()
                    best = None
                    for _ in range(2):
                        tc0 = time.perf_counter()
                        pts_c = o_c[:, None] + d_c[:, None] * z_c[..., None]
                        raw_c = NO.nerf_mlp(sd, NO.embed(pts_c, d_c), 63, 27, prefix='mlp.').reshape(1024, 64, 4)
                        NO.nerf_render(raw_c, z_c, d_c, white_bkgd=True)
                        dtc = time.perf_counter() - tc0
                        best = dtc if best is None else min(best, dtc)
                    nerf_cpu = {'value': 1024 / best, 'unit': 'rays/s', 'cores': os.cpu_count(), 'kind': 'port',
                                'sample': 'configs[0]: 1024 rays x 64 samples, coarse network only, numpy oracle (fp32, multi-threaded BLAS); best of 2'}
                except Exception as e:
                    nerf_cpu = {'error': repr(e)[:200]}
            # BASELINE.md B3 for the dominant op: the reference's NerfMLP.batchify_run_mlp arithmetic (nerf_mlp.py:70-94: 11 nn.Linear GEMMs + 2 cat per 32 768-row chunk, cuBLAS)
            # on this GPU, fp32 with TF32 off and on, against the single wgmma kernel on the same 2 097 152 embedded rows and weights
            torch_mlp = None
            if world == 1:
                try:
                    rows = 2097152
                    xe = torch.randn((rows, 90), dtype=torch.float32, device=dev)
                    res_t = {}
                    old_flags = (torch.backends.cuda.matmul.allow_tf32, torch.backends.cudnn.allow_tf32)
                    with torch.no_grad():
                        def timed_mlp(reps):
                            net.mlp.batchify_run_mlp(xe); torch.cuda.synchronize()
                            a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                            a.record()
                            for _ in range(reps):
                                out = net.mlp.batchify_run_mlp(xe)
                            b.record(); torch.cuda.synchronize()
                            return a.elapsed_time(b) / reps, out
                        t_tc, y_tc = timed_mlp(5)
                        net.mlp.fused = False
                        try:
                            for name, flag in (('fp32', False), ('tf32', True)):
                                torch.backends.cuda.matmul.allow_tf32 = flag; torch.backends.cudnn.allow_tf32 = flag
                                res_t[name], y_t = timed_mlp(2)
                                if not flag:
                                    err_t = float((y_t - y_tc).abs().max())
                        finally:
                            net.mlp.fused = True
                            torch.backends.cuda.matmul.allow_tf32, torch.backends.cudnn.allow_tf32 = old_flags
                    torch_mlp = {'rows': rows, 'ms': {'torch_nn_linear_fp32': res_t['fp32'], 'torch_nn_linear_tf32': res_t['tf32'], 'ours_wgmma_fp16': t_tc},
                                 'speedup_vs_fp32': res_t['fp32'] / t_tc, 'speedup_vs_tf32': res_t['tf32'] / t_tc, 'max_abs_diff_vs_fp32': err_t,
                                 'what': 'NerfMLP.batchify_run_mlp on 2 097 152 embedded rows (= 32 768 rays x 64 samples): the reference module\'s own arithmetic (nn.Linear chain, cat at the skip, '
                                         '32 768-row chunks, cuBLAS) vs the single wgmma kernel; same weights, CUDA events'}
                    del xe
                except Exception as e:   # noqa: BLE001
                    torch_mlp = {'error': repr(e)[:200]}
            nerf = {'value': rps, 'unit': 'rays/s', 'cpu_baseline': nerf_cpu, 'parity': nerf_parity, 'reference_torch_gpu_mlp': torch_mlp, 'rays': 'NeRF convention (GetRays on random pixels of Blender spiral poses, radius 4), near 2 / far 6', 'workload': 'vanilla NeRF hierarchical 64 coarse + 192 fine evaluations per ray (configs[2]), 32768-ray batches, inference',
                    'ms_per_batch': float(nm.item()) / KN, 'roofline': {'bound': 'tensor', 'achieved': rps * flop_per_ray / 1e12 / world, 'peak': tpeak, 'unit': 'TFLOP/s',
                                                                         'frac': rps * flop_per_ray / 1e12 / world / tpeak, 'flop_per_ray': flop_per_ray,
                                                                         'peak_source': tsrc}}
        except Exception as e:   # an auxiliary arm must never take the headline line down
            nerf = {'error': repr(e)[:300]}

    # ---- NeRF training step (configs[2], N_rand 4096 as configs/nerf/nerf_blender_base01.py): encoders / composite fwd+bwd / sample_pdf kernels + the 12 dense layers of both
    # networks forward AND backward as wgmma kernels over fp16 tile images (csrc/nerf_train.cu), torch.optim.Adam on the fp32 nn.Linear parameters
    nerf_train = None
    if not args.no_nerf:
        try:
            from xrnerf_b200 import registry as R
            mlp_cfg_t = dict(type='NerfMLP', skips=[4], netdepth=8, netwidth=256, netchunk=1024 * 32, output_ch=5, use_viewdirs=True, embedder=dict(type='BaseEmbedder', i_embed=0, multires=10, multires_dirs=4))
            tnet = R.build_network(dict(type='NerfNetwork', cfg=dict(phase='train', N_importance=128, is_perturb=False, chunk=1024 * 32, bs_data='rays_o'), mlp=mlp_cfg_t, mlp_fine=mlp_cfg_t,
                                        render=dict(type='NerfRender', white_bkgd=True, raw_noise_std=0))).to(dev)
            topt = torch.optim.Adam(tnet.parameters(), lr=5e-4, betas=(0.9, 0.999))
            n_t = 4096
            o_t, d_t, v_t = nerf_convention_rays(dev, n_t, 900 + rank)
            tt = torch.linspace(0., 1., 64, device=dev)
            z_t = (2.0 * (1. - tt) + 6.0 * tt).expand(n_t, 64).contiguous()
            tdata = {'rays_o': o_t[None], 'rays_d': d_t[None], 'viewdirs': v_t[None], 'z_vals': z_t[None], 'pts': (o_t[:, None, :] + d_t[:, None, :] * z_t[:, :, None])[None],
                     'target_s': torch.rand((1, n_t, 3), device=dev)}

            def tstep():
                out = tnet.train_step(dict(tdata), topt)
                topt.zero_grad(set_to_none=True); out['loss'].backward(); topt.step()
            for _ in range(2):
                tstep()
            barrier()
            q0, q1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            KT = 5
            q0.record()
            for _ in range(KT):
                tstep()
            q1.record()
            barrier()
            qm = torch.tensor([q0.elapsed_time(q1)], dtype=torch.float64, device=dev)
            if world > 1:
                dist.all_reduce(qm, op=dist.ReduceOp.MAX)
            nerf_train = {'value': world * n_t * KT / (float(qm.item()) * 1e-3), 'unit': 'rays/s', 'ms_per_step': float(qm.item()) / KT, 'rays_per_step_per_gpu': n_t,
                          'rows_per_step_per_gpu': n_t * (64 + 192), 'flop_per_step': 3 * n_t * (64 + 192) * 593408 * 2,
                          'tflops': 3 * n_t * (64 + 192) * 593408 * 2 / (float(qm.item()) / KT * 1e-3) / 1e12,
                          'what': 'NerfNetwork.train_step + Adam (per-rank, no gradient all-reduce in this arm): encoders / composite fwd+bwd / sample_pdf kernels; the dense layers of both '
                                  'networks forward + backward on wgmma (tile-image GEMM kernels: forward, input gradient with fused ReLU mask, weight gradient accumulated in registers)'}
            del tnet, topt, tdata
        except Exception as e:   # an auxiliary arm must never take the headline line down
            nerf_train = {'error': repr(e)[:300]}

    # ---- Mip-NeRF training step (configs[3]: 2 levels x 128 samples through the SAME MLP, loss = fine + 0.1 coarse, mipnerf.py:45-74), 4096 rays per step
    mip_train = None
    if not args.no_mip:
        try:
            from xrnerf_b200 import registry as R
            mtnet = R.build_network(dict(type='MipNerfNetwork', cfg=dict(phase='train', ray_shape='cone', resample_padding=0.01, use_multiscale=False, coarse_loss_mult=0.1, num_levels=2,
                                                                         chunk=1024 * 32, bs_data='rays_o'),
                                         mlp=dict(type='NerfMLP', skips=[4], netdepth=8, netwidth=256, netchunk=1024 * 32, use_viewdirs=True,
                                                  embedder=dict(type='MipNerfEmbedder', min_deg_point=0, max_deg_point=16, min_deg_view=0, max_deg_view=4, use_viewdirs=True, append_identity=True)),
                                         render=dict(type='MipNerfRender', white_bkgd=True, raw_noise_std=0, rgb_padding=0.001, density_bias=-1, density_activation='softplus'))).to(dev)
            mtopt = torch.optim.Adam(mtnet.parameters(), lr=5e-4, betas=(0.9, 0.999))
            n_mt = 4096
            o_m, d_m, v_m, r_m = nerf_convention_rays(dev, n_mt, 950 + rank, with_radii=True)
            tm_ = torch.linspace(0., 1., 129, device=dev)
            z_m = (2.0 * (1. - tm_) + 6.0 * tm_).expand(n_mt, 129).contiguous()
            mdata = {'rays_o': o_m[None], 'rays_d': d_m[None], 'viewdirs': v_m[None], 'radii': r_m[None], 'lossmult': torch.ones((1, n_mt, 1), device=dev), 'z_vals': z_m[None],
                     'target_s': torch.rand((1, n_mt, 3), device=dev)}

            def mstep():
                out = mtnet.train_step(dict(mdata), mtopt)
                mtopt.zero_grad(set_to_none=True); out['loss'].backward(); mtopt.step()
            for _ in range(2):
                mstep()
            barrier()
            w0, w1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            KMT = 5
            w0.record()
            for _ in range(KMT):
                mstep()
            w1.record()
            barrier()
            wm = torch.tensor([w0.elapsed_time(w1)], dtype=torch.float64, device=dev)
            if world > 1:
                dist.all_reduce(wm, op=dist.ReduceOp.MAX)
            mip_train = {'value': world * n_mt * KMT / (float(wm.item()) * 1e-3), 'unit': 'rays/s', 'ms_per_step': float(wm.item()) / KMT, 'rays_per_step_per_gpu': n_mt,
                         'rows_per_step_per_gpu': n_mt * 256, 'tflops': 3 * n_mt * 256 * 610304 * 2 / (float(wm.item()) / KMT * 1e-3) / 1e12,
                         'what': 'MipNerfNetwork.train_step + Adam: cast_rays + IPE + composite fwd/bwd + resample kernels; the MLP (both levels) forward + backward on wgmma tile-image GEMMs'}
            del mtnet, mtopt, mdata
        except Exception as e:
            import traceback
            mip_train = {'error': repr(e)[:300], 'trace': traceback.format_exc()[-500:]}

    # ---- Mip-NeRF arm (BASELINE configs[3]: 2 levels x 128 cone samples, IPE): the same wgmma NerfMLP on IPE tile images, device-resident rays
    mip = None
    if not args.no_mip:
        try:
            from xrnerf_b200 import registry as R
            from xrnerf_b200.nerf import MipNerfRenderer
            mnet = R.build_network(dict(type='MipNerfNetwork', cfg=dict(phase='test', ray_shape='cone', resample_padding=0.01, use_multiscale=False, coarse_loss_mult=0.1, num_levels=2,
                                                                        chunk=1024 * 32, bs_data='rays_o'),
                                        mlp=dict(type='NerfMLP', skips=[4], netdepth=8, netwidth=256, netchunk=1024 * 32, use_viewdirs=True,
                                                 embedder=dict(type='MipNerfEmbedder', min_deg_point=0, max_deg_point=16, min_deg_view=0, max_deg_view=4, use_viewdirs=True, append_identity=True)),
                                        render=dict(type='MipNerfRender', white_bkgd=True, raw_noise_std=0, rgb_padding=0.001, density_bias=-1, density_activation='softplus'))).to(dev)
            mr = MipNerfRenderer(mnet, near=2.0, far=6.0, n_samples=128)
            n_mip = 32768
            mip_rays = [nerf_convention_rays(dev, n_mip, 700 + 10 * rank + b, with_radii=True) for b in range(8)]   # radii = |dx| * 2/sqrt(12) from GetRays (create.py:237-243)
            for i in range(3):
                mr.render(*mip_rays[0])
            barrier()
            m0, m1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            KM = max(3, min(K, 20))
            m0.record()
            for i in range(KM):
                mr.render(*mip_rays[i % 8])
            m1.record()
            barrier()
            mm = torch.tensor([m0.elapsed_time(m1)], dtype=torch.float64, device=dev)
            if world > 1:
                dist.all_reduce(mm, op=dist.ReduceOp.MAX)
            mrps = world * n_mip * KM / (float(mm.item()) * 1e-3)
            mflop = 256 * 610304 * 2
            tpeak, tsrc = tensor_peak()
            mip_parity = None
            if world == 1:
                try:
                    from oracle import nerf_oracle as NO
                    sdm = {k: v.detach().cpu().numpy() for k, v in mnet.state_dict().items()}
                    po, pd, pv, pr = (t[:256].contiguous() for t in mip_rays[0])
                    got = mr.render(po, pd, pv, pr)
                    o_p, d_p, v_p, r_p = po.cpu().numpy(), pd.cpu().numpy(), pv.cpu().numpy(), pr.cpu().numpy()
                    z_p = np.broadcast_to(np.linspace(2, 6, 129, dtype=np.float32), (256, 129)).copy()
                    rgb_levels = []
                    for level in range(2):
                        if level > 0:
                            z_p = NO.resample_along_rays(z_p, w_p, 0.01)
                        means, covs = NO.cast_rays(z_p, o_p, d_p, r_p)
                        emb = np.concatenate([NO.integrated_pos_enc(means, covs, 0, 16).reshape(256 * 128, -1), np.repeat(NO.mip_pos_enc(v_p, 0, 4), 128, 0)], -1)
                        raw_p = NO.nerf_mlp(sdm, emb, 96, 27, prefix='mlp.').reshape(256, 128, 4)
                        rl = NO.nerf_render(raw_p, z_p, d_p, white_bkgd=True, rgb_padding=0.001, density_bias=-1.0, density_activation='softplus', mip=True)
                        w_p = rl['weights']; rgb_levels.append(rl['rgb'])
                    mip_parity = psnr_obj(got['rgb'].cpu().numpy(), rgb_levels[-1], 'oracle/nerf_oracle.py (numpy fp32 restatement of MipNerfNetwork.forward, pinned to the reference by tests/golden)')
                except Exception as e:
                    mip_parity = {'error': repr(e)[:300]}
            mip = {'value': mrps, 'unit': 'rays/s', 'parity': mip_parity, 'rays': 'NeRF convention with GetRays radii, near 2 / far 6', 'workload': 'Mip-NeRF 2 levels x 128 conical-frustum samples per ray, IPE 96 + 27 (configs[3]), 32768-ray batches, inference',
                   'ms_per_batch': float(mm.item()) / KM, 'roofline': {'bound': 'tensor', 'achieved': mrps * mflop / 1e12 / world, 'peak': tpeak, 'unit': 'TFLOP/s',
                                                                       'frac': mrps * mflop / 1e12 / world / tpeak, 'flop_per_ray': mflop,
                                                                       'peak_source': tsrc}}
        except Exception as e:   # an auxiliary arm must never take the headline line down
            mip = {'error': repr(e)[:300]}

    if rank == 0:
        peak, peak_src = peaks()
        f_ms_loaded = float(np.mean(field_ms))                      # the same kernel's events recorded while P-1 other batches shared the SMs (context only)
        s_mean = float(np.mean(samples))
        achieved = iso_samples * BYTES_PER_SAMPLE / (iso_field_ms * 1e-3) / 1e9
        if world == 1:
            cpu_rate, cores, kind, sample, _ = cpu_thread_sweep(4096, reps=3)
            cpu_reference_rate(4096, reps=1, threads=cores)          # leaves the 4096-ray render in cpu_reference_rate.last for the parity object
        else:
            cpu_rate, cores, kind, sample = None, os.cpu_count(), 'reference', 'measured at N=1 only'
        parity = None
        if world == 1:   # the CPU arm just rendered 4096 rays of batch 0 with the reference arithmetic: compare this arm's render of the same rays (checker only)
            rgb_cpu, alpha_cpu, ns_cpu = cpu_reference_rate.last
            parity = {'rays': 4096, 'against': kind + ' CPU arm (oracle), fp32 march/composite + fp16 tcnn-shaped field'}
            for path, (rgb_g, ns_g) in parity_gpu.items():
                err = np.abs(rgb_g - rgb_cpu)
                mse = float((err.astype(np.float64) ** 2).mean())
                parity[path] = {'max_abs_rgb_err': float(err.max()), 'psnr_vs_ref_db': float(-10.0 * np.log10(max(mse, 1e-20))), 'sample_counts_bit_exact': bool(np.array_equal(ns_g, ns_cpu))}
        # the roof the gather runs under, measured live (xrb_micro_gather): the field kernel's own sector count is not measured by this run
        l2_obj = {'bound': 'l2 sector rate (random 4-byte gather)', 'peak': l2_roof['sector_GBs_at_4B'], 'unit': 'GB/s of 32-byte sectors', 'peak_measured_live': l2_roof} \
            if l2_roof and 'error' not in l2_roof else l2_roof
        chain = {'value': world * N_RAYS * K / (total_ms_max * 1e-3), 'unit': 'rays/s', 'ms_per_step': total_ms_max / K, 'gpu_launches_per_step': 6,
                 'what': '6 launches per batch on one stream (memset, march count / scan / emit, field, composite), P batches in flight on P streams',
                 'roofline': {'kernel': 'xrb::ngp_field_tc_kernel<false>', 'bound': 'hbm', 'achieved': achieved, 'peak': peak, 'unit': 'GB/s', 'frac': achieved / peak,
                              'kernel_ms': iso_field_ms, 'kernel_share_of_step': iso_field_ms / iso_chain_ms, 'step_ms_sequential': iso_chain_ms,
                              'timing': 'isolated pass: one stream, one batch at a time, CUDA events around the kernel inside xrb_ngp_render and around the whole call, median of %d' % KI_,
                              'kernel_ms_with_other_batches_in_flight': f_ms_loaded, 'algorithmic_bytes_per_launch': iso_samples * BYTES_PER_SAMPLE, 'l2_gather_roofline': l2_obj}}
        f_bytes = fused_samples * 512 + N_RAYS * 44   # no coords[S,7] / raw[S,4] round trip: gather bytes + 44 B of ray I/O
        f_ach = f_bytes / (fused_kernel_ms * 1e-3) / 1e9
        fused = {'value': world * N_RAYS * K / (fused_total_ms * 1e-3), 'unit': 'rays/s', 'ms_per_step': fused_total_ms / K, 'gpu_launches_per_step': 1,
                 'what': 'ONE launch per batch (xrb_ngp_render_fused: warp-specialised march + hash encode + wgmma MLPs + segmented-scan composite), P batches in flight on P streams',
                 'roofline': {'kernel': 'xrb::ngp_render_fused_kernel', 'bound': 'hbm', 'achieved': f_ach, 'peak': peak, 'unit': 'GB/s', 'frac': f_ach / peak,
                              'kernel_ms': fused_kernel_ms, 'kernel_share_of_step': 1.0, 'kernel_ms_note': 'events around the launch while P-1 other launches share the SMs',
                              'algorithmic_bytes_per_launch': f_bytes}}
        ref_gpu = None
        if world == 1 and not args.no_ref_gpu:
            try:
                ref_gpu = reference_gpu_leg(dev, bf, dev_batches[0], field, iso_chain_ms, iso_field_ms)
            except Exception as e:   # noqa: BLE001
                ref_gpu = {'error': repr(e)[:300]}
        head = fused if use_fused else chain
        line = {
            'metric': METRIC, 'value': head['value'], 'unit': 'rays/s', 'n_gpus': world, 'steps': K, 'warmup': W,
            'ms_per_step': head['ms_per_step'], 'higher_is_better': True, 'scaling': 'weak', 'vs_baseline': None, 'dtype': 'f16', 'data': 'synthetic',
            'config': {'workload': WORKLOAD, 'rays_per_step_per_gpu': N_RAYS, 'samples_per_ray_mean': s_mean / N_RAYS, 'parallelism': f'ray-sharded x{world}, no data-path collective',
                       'l2': f'inputs larger than L2: {N_BATCHES} distinct ray batches = {N_BATCHES * N_RAYS * 24 / 1e6:.0f} MB cycled (L2 50 MB), nothing flushed; the 24.4 MB fp16 hash table and its '
                             f'{field._cells.numel() / 1e6 if field._cells is not None else 0:.0f} MB cell image (levels 0..{field.n_packed - 1}) stay L2-resident as in production',
                       'timing': 'one CUDA-event pair around the K steps on the launching stream, max over ranks', 'batches_in_flight': P, 'untimed_warmup_steps_run': WU,
                       'path': 'fused single launch' if use_fused else 'chain of 6 launches', 'path_selection': args.path, 'cell_image_levels': field.n_packed},
            'clocks': clk,
            'e2e': {'value': world * N_RAYS * K / (e2e_ms * 1e-3), 'unit': 'rays/s', 'h2d_bytes_per_step': N_RAYS * 24, 'd2h_bytes_per_step': N_RAYS * 16,
                    'ms_per_step': e2e_ms / K, 'host_wall_ms_per_step': e2e_wall_ms / K},
            'gpu_launches': head['gpu_launches_per_step'] * K,
            'roofline': dict(head['roofline'], peak_source=peak_src,
                             note='hash table (24.4 MB fp16) + cell image are L2-resident by design: DRAM traffic is far below the algorithmic bytes; the gather runs under the L2 sector rate '
                                  '(l2_gather_roofline: every 4-byte entry costs a 32-byte sector), not under the HBM copy peak this frac is quoted against'),
            'paths': {'chain': chain, 'fused': fused},
            'reference_gpu': ref_gpu,
            'cpu_baseline': {'value': cpu_rate, 'unit': 'rays/s', 'cores': cores, 'kind': kind, 'sample': sample},
            'parity': parity,
            'image': image_arm,
            'grid_update': grid_upd,
            'nerf': nerf,
            'nerf_train': nerf_train,
            'mip': mip,
            'mip_train': mip_train,
            'all_ones_grid': all_ones,
            'train': train,                                   # last on purpose: the driver keeps the tail of the line
        }
        print(json.dumps(line), flush=True)
    if world > 1:
        dist.destroy_process_group()


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--gpus', type=int, default=1)
    ap.add_argument('--steps', type=int, default=50)
    ap.add_argument('--warmup', type=int, default=5)
    ap.add_argument('--impl', default='ours', choices=['ours', 'reference'])
    ap.add_argument('--no-train', dest='no_train', action='store_true', help='skip the training arm')
    ap.add_argument('--no-nerf', dest='no_nerf', action='store_true', help='skip the vanilla-NeRF arm')
    ap.add_argument('--no-image', dest='no_image', action='store_true', help='skip the whole-image inference arm')
    ap.add_argument('--no-grid', dest='no_grid', action='store_true', help='skip the occupancy-grid update arm')
    ap.add_argument('--no-mip', dest='no_mip', action='store_true', help='skip the Mip-NeRF arm')
    ap.add_argument('--no-ref-gpu', dest='no_ref_gpu', action='store_true', help='skip the GPU reference leg (reference raymarch_cuda kernels built for sm_90a, BASELINE.md B4)')
    ap.add_argument('--path', default='auto', choices=['auto', 'chain', 'fused'], help='inference path of the headline/e2e numbers: 5-launch chain, single-launch fused kernel, or the faster of the two (both are always measured)')
    ap.add_argument('--grad-comm', dest='grad_comm', default='auto', choices=['auto', 'peer', 'sharded', 'allreduce'], help='gradient exchange of the training arm at world > 1 (peer: one optimiser kernel over NVLink peer memory, csrc/peer_adam.cu; auto: peer where CUDA IPC works, else sharded NCCL)')
    ap.add_argument('--pipeline', type=int, default=8, help='ray batches in flight (CUDA streams); 1 = strictly sequential steps')
    ap.add_argument('--dump-outputs', dest='dump_outputs', default=None, metavar='DIR',
                    help='after the timed steps, write rgb / alpha / n_samples of the last timed batch of the chain and the fused path as DIR/{chain,fused}_<name>.npy (float32)')
    args = ap.parse_args()
    args.warmup = max(args.warmup, 3) if args.impl == 'ours' else args.warmup
    if args.impl == 'reference':
        run_reference(args)
    else:
        run_ours(args)


if __name__ == '__main__':
    main()
