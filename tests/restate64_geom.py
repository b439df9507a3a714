"""Float64 restatements of the depth / opacity supervision kernels (include/xrnerf_b200.h, "Depth and opacity supervision"): the NeRF / Mip-NeRF
composite with depth, the NGP training composite with depth and alpha, and the geometry loss; the counterpart of tests/restate64.py for this feature."""
import numpy as np
import torch


def nerf_composite64(raw, z, rays_d, mip, white_bkgd, rgb_padding=0.0, density_bias=0.0, softplus=False):
    """the NeRF / Mip-NeRF composite (xrb_nerf_composite_forward_depth) in float64 torch: (rgb [n,3], depth [n] = sum of w * z (interval mid-points when mip),
    acc [n], sigma * delta [n,S]); differentiable in raw. NeRF's transmittance is the product of (1 - alpha + 1e-10), its last interval 1e10; Mip-NeRF's is
    exp(-sum of the earlier sigma * delta)."""
    raw, z, rays_d = raw.double(), z.double(), rays_d.double()
    dnorm = rays_d.norm(dim=-1, keepdim=True)
    if mip:
        dist, zk = z[:, 1:] - z[:, :-1], 0.5 * (z[:, 1:] + z[:, :-1])
    else:
        dist, zk = torch.cat([z[:, 1:] - z[:, :-1], torch.full_like(z[:, :1], 1e10)], 1), z
    a = raw[..., 3] + density_bias
    sd = (torch.nn.functional.softplus(a) if softplus else torch.relu(a)) * (dist * dnorm)
    alpha = 1.0 - torch.exp(-sd)
    if mip:
        T = torch.exp(-(torch.cumsum(sd, 1) - sd))
    else:
        T = torch.cumprod(torch.cat([torch.ones_like(alpha[:, :1]), 1.0 - alpha + 1e-10], 1), 1)[:, :-1]
    w = alpha * T
    c = torch.sigmoid(raw[..., :3]) * (1 + 2 * rgb_padding) - rgb_padding
    rgb, acc, depth = (w[..., None] * c).sum(1), w.sum(1), (w * zk).sum(1)
    if white_bkgd:
        rgb = rgb + (1.0 - acc)[:, None]
    return rgb, depth, acc, sd


NGP_MIN_DT = np.float32(np.float32(1.73205080757) / np.float32(1024))


def ngp_row_dt(coords):
    """the dt the NGP composite reads back from sample rows (unwarp_dt, fp32 as the kernel rounds it), float64 numpy"""
    c = coords.astype(np.float32)
    span = np.float32(NGP_MIN_DT * np.float32(128)) - NGP_MIN_DT
    return (c[:, 3] * span + NGP_MIN_DT).astype(np.float64)


def ngp_pad(numsteps_c, n_rows):
    """[n_rays, K] row indices of each ray's compacted samples (K: the longest ray; padding slots point at row n_rows) and the [n_rays, K] validity mask"""
    ns = np.asarray(numsteps_c, np.int64)
    K = max(1, int(ns[:, 0].max()))
    k = np.arange(K)[None, :]
    valid = k < ns[:, :1]
    idx = np.where(valid, ns[:, 1:2] + k, n_rows)
    return idx, valid


def ngp_composite64(raw, coords, numsteps, numsteps_c, bg, rays_o, rays_d, lo, hi):
    """the NGP training composite with geometry (MODE 4 of composite_fwd_kernel; rgb is MODE 0's) in float64 torch on the CPU, logistic colour and exponential
    density (the reference config's activations): (rgb [n,3], alpha [n], depth [n], per-sample (w, Ta, t, dt) [n,K] and the mask). raw: tensor [rows,4],
    differentiable. t_k is rebuilt from the row as row_t does, ((lo + x (hi - lo)) - o) . d / |d|^2."""
    idx, valid = ngp_pad(numsteps_c, coords.shape[0])
    rows = np.concatenate([coords.astype(np.float64), np.zeros((1, 7))], 0)[idx]                       # [n,K,7]
    dt = torch.from_numpy(np.where(valid, ngp_row_dt(rows.reshape(-1, 7)).reshape(idx.shape), 0.0))
    o, d = rays_o.astype(np.float64), rays_d.astype(np.float64)
    p = lo + rows[..., :3] * (hi - lo) - o[:, None, :]
    t = torch.from_numpy(np.where(valid, (p * d[:, None, :]).sum(-1) / (d * d).sum(-1)[:, None], 0.0))
    r = torch.cat([raw.double(), torch.zeros((1, 4), dtype=torch.float64)], 0)[torch.from_numpy(idx)]   # [n,K,4]
    m = torch.from_numpy(valid)
    alpha_k = torch.where(m, 1.0 - torch.exp(-torch.exp(r[..., 3]) * dt), torch.zeros_like(dt))
    Ta = torch.cumprod(1.0 - alpha_k, 1)
    Tb = torch.cat([torch.ones_like(Ta[:, :1]), Ta[:, :-1]], 1)
    w = alpha_k * Tb
    c = torch.sigmoid(r[..., :3])
    rgb = (w[..., None] * c).sum(1)
    whole = torch.from_numpy(np.asarray(numsteps_c)[:, 0] == np.asarray(numsteps)[:, 0])
    rgb = rgb + torch.where(whole[:, None], Ta[:, -1:] * torch.from_numpy(np.asarray(bg, np.float64)), torch.zeros_like(rgb))
    return rgb, 1.0 - Ta[:, -1], (w * t).sum(1), (w, Ta, t, dt), m


def geom_loss64(depth, alpha, target_depth, target_alpha, keep, wd, wa, mean):
    """xrb_geom_loss_grad in float64 numpy: (loss, grad_depth, grad_alpha); keep = the rays no truncation dropped (bool [n])"""
    depth, alpha, td, ta = (np.asarray(v, np.float64).reshape(-1) for v in (depth, alpha, target_depth, target_alpha))
    kd = keep & np.isfinite(td) & (td > 0)
    cd = max(int(kd.sum()), 1) if mean else 1
    ca = max(int(keep.sum()), 1) if mean else 1
    r = np.where(kd, depth - np.where(kd, td, 0.0), 0.0)
    ra = np.where(keep, alpha - ta, 0.0)
    loss = wd * np.abs(r).sum() / cd + wa * (ra * ra).sum() / ca
    return loss, wd * np.sign(r) / cd, 2.0 * wa * ra / ca
