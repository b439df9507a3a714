"""float64 restatements for NGP camera pose refinement (include/xrnerf_b200.h, "NGP camera pose refinement"): the ReLU masks of the tensor-core field with
proof of their stability, the field's input gradients dL/d(encoding) and dL/d(SH) down the fp16-staged backward chain, the SH derivative, the per-ray sum
of xrb_ngp_ray_grad and the ray generation xrb_ngp_pose_grad differentiates. As in restate64.py nothing here asserts a bound; each function also returns
the same chain on absolute values (the mass a test's bound multiplies).

The field's input gradients depend on its forward only through the ReLU masks: dX = W^T dZ masked by ReLU'(forward). A row whose every mask is proven
stable (the kernel cannot take the other branch anywhere) therefore has the kernel's masks, and its gradient differs from the float64 chain by the fp16
staging of dZ at each layer and fp32 accumulation only.
"""
import numpy as np

from restate64 import GAMMA_TC, f16

FLOOR = 2.0 ** -26          # (2^-25 / 4096) / 2^-11: half the fp16 subnormal step at the backward's 2^12 staging scale, as a floor on a staged magnitude


def _layer(W, x, ex, relu):
    """one layer of the forward with its interval: (fp16 activation, its bound, rows whose ReLU decision is not proven)"""
    aW = np.abs(W)
    z = x @ W.T
    b = ex @ aW.T + W.shape[1] * GAMMA_TC * ((np.abs(x) + ex) @ aW.T)
    act = (lambda v: np.maximum(v, 0.0)) if relu else (lambda v: v)
    a, lo, hi = f16(act(z)), f16(act(z - b)), f16(act(z + b))
    flip = ((lo > 0) != (hi > 0)).any(1) if relu else np.zeros(z.shape[0], bool)
    return a, np.maximum(hi - a, a - lo), flip


def field_masks(dm, cm, enc, sh):
    """(density masks, colour masks, stable rows) of the tensor-core field on the fp16 encodings enc [n,32] and SH values sh [n,16] (float64)"""
    flip = np.zeros(enc.shape[0], bool)

    def net(mats, x, ex):
        nonlocal flip
        masks = []
        for W in mats[:-1]:
            x, ex, fl = _layer(W, x, ex, True)
            flip |= fl
            masks.append(x > 0)
        y, ey, _ = _layer(mats[-1], x, ex, False)
        return masks, y, ey
    dmasks, dout, edout = net(dm, enc, np.zeros_like(enc))
    n = enc.shape[0]
    cmasks, _, _ = net(cm, np.concatenate([dout[:, 1:], sh, np.ones((n, 1))], 1), np.concatenate([edout[:, 1:], np.zeros((n, 17))], 1))
    return dmasks, cmasks, ~flip


def input_grads(dm, cm, dmasks, cmasks, draw, rows):
    """dL/d(encoding) [n,32] and dL/d(colour input) [n,32] of the fp16-staged backward chain (xrb_ngp_mlp_backward_tc: dZ staged in fp16 at every layer,
    the net inputs' gradients in fp32), in float64, for dL/draw [n,4] on `rows` (others 0); and both chains on absolute values with FLOOR added at every
    live staged value"""
    out = []
    for absolute in (False, True):
        T = np.abs if absolute else (lambda a: a)
        stage = (lambda v, live: np.abs(v) + FLOOR * live) if absolute else (lambda v, live: v)

        def back(mats, masks, gy, live):
            dz = stage(gy, live)
            for k in range(len(mats) - 1, -1, -1):
                dx = dz @ T(mats[k])
                if k > 0:
                    dz = stage(dx * masks[k - 1], masks[k - 1] & rows[:, None])
            return dx
        n = draw.shape[0]
        gy = np.zeros((n, 16)); gy[:, :3] = draw[:, :3]
        live = np.zeros((n, 16), bool); live[:, :3] = rows[:, None]
        gcin = back(cm, cmasks, gy, live)
        genc = back(dm, dmasks, np.concatenate([draw[:, 3:4], gcin[:, :15]], 1), np.repeat(rows[:, None], 16, 1))
        out += [genc, gcin]
    return out


_C = dict(c1=0.48860251190291987, c4=1.0925484305920792, c6=0.94617469575755997, c8=0.54627421529603959, c9=0.59004358992664352, c10=2.8906114426405538,
          c11=0.45704579946446572, c12=0.3731763325901154, c14=1.4453057213202769)


def sh4_jacobian(w):
    """d SH_k / d w [n,16,3] of tcnn's degree-4 SH on x = 2 w - 1 (csrc/ngp_field.cuh sh4), w the warped directions [n,3] (float64)"""
    c = _C
    x, y, z = (2.0 * np.asarray(w, np.float64) - 1.0).T
    J = np.zeros((x.size, 16, 3))
    J[:, 1, 1] = -c['c1']; J[:, 2, 2] = c['c1']; J[:, 3, 0] = -c['c1']
    J[:, 4, 0], J[:, 4, 1] = c['c4'] * y, c['c4'] * x
    J[:, 5, 1], J[:, 5, 2] = -c['c4'] * z, -c['c4'] * y
    J[:, 6, 2] = 2 * c['c6'] * z
    J[:, 7, 0], J[:, 7, 2] = -c['c4'] * z, -c['c4'] * x
    J[:, 8, 0], J[:, 8, 1] = 2 * c['c8'] * x, -2 * c['c8'] * y
    J[:, 9, 0], J[:, 9, 1] = -6 * c['c9'] * x * y, 3 * c['c9'] * (y * y - x * x)
    J[:, 10, 0], J[:, 10, 1], J[:, 10, 2] = c['c10'] * y * z, c['c10'] * x * z, c['c10'] * x * y
    J[:, 11, 1], J[:, 11, 2] = c['c11'] * (1 - 5 * z * z), -10 * c['c11'] * y * z
    J[:, 12, 2] = c['c12'] * (15 * z * z - 3)
    J[:, 13, 0], J[:, 13, 2] = c['c11'] * (1 - 5 * z * z), -10 * c['c11'] * x * z
    J[:, 14, 0], J[:, 14, 1], J[:, 14, 2] = 2 * c['c14'] * x * z, -2 * c['c14'] * y * z, c['c14'] * (x * x - y * y)
    J[:, 15, 0], J[:, 15, 1] = 3 * c['c9'] * (y * y - x * x), 6 * c['c9'] * x * y
    return 2.0 * J


def row_t64(coords, o, d, lo, diag):
    """t of each sample row (float64 of row_t's fp32 inputs): ((lo + c diag - o) . d) / |d|^2, coords [k,>=3], o / d [k,3]"""
    p = lo + np.asarray(coords[:, :3], np.float64) * diag - o
    return (p * d).sum(1) / (d * d).sum(1)


def ray_grad64(d_rows, coords, numsteps_c, rays_o, rays_d, lo, hi, scale):
    """xrb_ngp_ray_grad in float64 -> (grad_o, grad_d [n_rays,3], the same sums on absolute values)"""
    diag = float(np.float32(hi) - np.float32(lo))
    n = numsteps_c.shape[0]
    go, gd, mo, md = (np.zeros((n, 3)) for _ in range(4))
    for r in range(n):
        k, b = int(numsteps_c[r, 0]), int(numsteps_c[r, 1])
        if k == 0:
            continue
        rows = np.asarray(d_rows[b:b + k], np.float64)
        o = np.repeat(np.asarray(rays_o[r:r + 1], np.float64), k, 0); d = np.repeat(np.asarray(rays_d[r:r + 1], np.float64), k, 0)
        t = row_t64(coords[b:b + k], o, d, lo, diag)
        go[r] = scale * rows[:, :3].sum(0) / diag
        gd[r] = scale * ((t[:, None] * rows[:, :3]).sum(0) / diag + 0.5 * rows[:, 3:].sum(0))
        mo[r] = abs(scale) * np.abs(rows[:, :3]).sum(0) / diag
        md[r] = abs(scale) * ((np.abs(t)[:, None] * np.abs(rows[:, :3])).sum(0) / diag + 0.5 * np.abs(rows[:, 3:]).sum(0))
    return go, gd, mo, md


def ngp_rays64(poses, row_idx, H, W, fx, fy, cx, cy):
    """xrb_ngp_batch_sample's rays in float64 torch (differentiable in poses [I,4,3]): (o, unit d) [n,3] of the rows row_idx"""
    import torch
    img, pix = row_idx // (H * W), row_idx % (H * W)
    j, i = (pix // W).double(), (pix % W).double()
    x, y = (i + 0.5 - cx) / fx, (j + 0.5 - cy) / fy
    P = poses[img]
    d = x[:, None] * P[:, 0] + y[:, None] * P[:, 1] + P[:, 2]
    return P[:, 3], d / d.norm(dim=1, keepdim=True)
