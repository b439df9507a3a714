"""CPU model (no GPU involved) of the NGP field kernel's gather cost per sample, for the samples of one bench batch (oracle march, 65 536 rays,
lego-like grid) evaluated in ray order and in spatially sorted orders. For every load instruction of hash_level (7 packed levels as 2 x 16 B,
hashed levels as 4 x 8 B plus 4 x 4 B on odd gx) it counts
  - distinct 128-B lines per warp instruction (L1 wavefronts), and
  - distinct 32-B sectors per window of consecutive samples (what an SM working on that window fetches from L2 with an ideal L1).
These are counts from addresses, not measurements.   python scripts/gather_model.py"""
import os
import sys
import time

import numpy as np

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from oracle import oracle as O          # noqa: E402
from xrnerf_b200 import synth           # noqa: E402

N = 65536
bf, _ = synth.bitfield_from_grid_numpy(synth.lego_like_density_grid(0))
o, d = synth.ray_batch(N, seed=1005)[:2]
t0 = time.time()
c, _, _, cnt = O.Port().rays_sampler(o, d, bf, N * 64)
S = int(cnt[1])
pts = np.ascontiguousarray(c[:S, :3]).astype(np.float32)
print(f'samples {S} ({S / N:.2f} per ray), oracle march {time.time() - t0:.0f} s')

# hash-grid layout of the default NgpField (16 levels, 2^19 entries, base 16, finest 2048); levels [0, NP) come from the cell image
pls = np.float32(2.0 ** (np.log2(2048 / 16) / 15))
offs, scales, ress = [], [], []
off = 0
for lv in range(16):
    sc = np.float32(np.exp2(np.float32(lv) * np.log2(pls)) * 16 - 1)
    res = int(np.ceil(sc)) + 1
    p = min(res ** 3, 0x7fffffff); p = min((p + 7) // 8 * 8, 1 << 19)
    offs.append(off); scales.append(sc); ress.append(res); off += p
NP = 7
cell_off = np.cumsum([0] + [ress[lv] ** 3 for lv in range(NP - 1)])
CELL_BASE = 1 << 40   # the cell image is a separate allocation


def level_addrs(P, lv):
    """(byte address[S], active[S]) of every load instruction of level lv"""
    q = (P * scales[lv] + np.float32(0.5)).astype(np.float32)
    g = np.floor(q).astype(np.int64).astype(np.uint64)
    gx, gy, gz = g[:, 0], g[:, 1], g[:, 2]
    res, M32, on = ress[lv], np.uint64(0xffffffff), np.ones(len(P), bool)
    if lv < NP:
        cx, cy, cz = (np.minimum(v, np.uint64(res - 1)) for v in (gx, gy, gz))
        a = CELL_BASE + (np.uint64(cell_off[lv]) + cx + np.uint64(res) * (cy + np.uint64(res) * cz)) * np.uint64(32)
        return [(a, on), (a + np.uint64(16), on)]
    mask = np.uint64((1 << 19) - 1)
    hy = [(gy * np.uint64(2654435761)) & M32, ((gy + np.uint64(1)) * np.uint64(2654435761)) & M32]
    hz = [(gz * np.uint64(805459861)) & M32, ((gz + np.uint64(1)) * np.uint64(805459861)) & M32]
    rows = [hy[0] ^ hz[0], hy[1] ^ hz[0], hy[0] ^ hz[1], hy[1] ^ hz[1]]
    odd = (gx & np.uint64(1)).astype(bool)
    out = [((np.uint64(offs[lv]) + (((gx ^ a) & mask) & ~np.uint64(1))) * np.uint64(4), on) for a in rows]
    out += [((np.uint64(offs[lv]) + (((gx + np.uint64(1)) ^ a) & mask)) * np.uint64(4), odd) for a in rows]
    return out


def lines_per_sample(P):
    """distinct 128-B lines per warp load instruction, summed over the instructions of all levels, per sample"""
    n = len(P) // 32 * 32
    tot = 0
    for lv in range(16):
        for a, act in level_addrs(P[:n], lv):
            key = np.where(act, a.astype(np.int64) >> 7, -1).reshape(-1, 32)
            key.sort(axis=1)
            tot += ((np.diff(key, axis=1) != 0).sum(1) + 1 - (key[:, 0] == -1)).sum()
    return tot / n


def window_sectors(P, w):
    """distinct 32-B sectors per sample within windows of w consecutive samples"""
    n = len(P) // w * w
    wid = (np.arange(n) // w).astype(np.int64)
    tot = 0
    for lv in range(16):
        keys = [np.where(act, (wid << 42) | ((a.astype(np.int64) >> 5) & ((1 << 42) - 1)), -1) for a, act in level_addrs(P[:n], lv)]
        tot += (np.unique(np.concatenate(keys)) >= 0).sum()
    return tot / n


def morton(P, bits):
    q = np.clip((P * (1 << bits)).astype(np.int64), 0, (1 << bits) - 1).astype(np.uint64)
    code = np.zeros(len(P), np.uint64)
    for b in range(bits):
        for k in range(3):
            code |= ((q[:, k] >> np.uint64(b)) & np.uint64(1)) << np.uint64(3 * b + k)
    return code


tie = np.random.default_rng(0).random(S)    # a bucket sort leaves the order inside a bucket arbitrary
orders = {'ray order': np.arange(S), 'Morton order, 10 bits/axis (full sort)': np.argsort(morton(pts, 10), kind='stable')}
for bits in (6, 7, 5):
    orders[f'{1 << bits}^3-bucket order'] = np.lexsort((tie, morton(pts, bits)))
print(f'| sample order | L1 lines / sample | L2 sectors / sample, 128-sample window | 256-sample window |')
print('|---|---|---|---|')
for name, perm in orders.items():
    P = pts[perm]
    print(f'| {name} | {lines_per_sample(P):.1f} | {window_sectors(P, 128):.1f} | {window_sectors(P, 256):.1f} |', flush=True)
