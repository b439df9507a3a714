"""Image metrics on the device: SSIM (xrb_ssim, csrc/metrics.cu) and the per-view MSE / PSNR / SSIM summaries the reference's ValidateHook and TestHook
log (xrnerf/core/hooks/validation_hooks.py:101-151, test_hooks.py:39-89), computed from the networks' val_step / test_step outputs without copying the
views to the host.

data_range: the hooks call calculate_ssim(rgb, gt, data_range=gt.max() - gt.min()), which forwards it to scikit-image as `val_range=`, a keyword
scikit-image does not take, so scikit-image runs with data_range=None. The releases that accept that call take the range of the float dtype, (-1, 1):
R = 2. validate_metrics and TestMetrics default to that R = 2.0 to reproduce the hooks' numbers; R = 1.0 is the usual convention for [0, 1] images."""
import torch

from . import _C
from .registry.networks import img2mse, mse2psnr


def ssim(x, y, data_range, full=False):
    """SSIM of float32 CUDA images x, y of one shape, [H,W,C] or [n,H,W,C] (HWC, 1 <= C <= 4, H and W at least 7), with scikit-image's
    structural_similarity(x, y, multichannel=True, data_range=data_range) definition (include/xrnerf_b200.h, xrb_ssim).

    Returns float64 device tensors (ssim, mssim), shape [n] (0-d for one [H,W,C] image): ssim is the mean of the SSIM map over every entry (the
    reference's calculate_ssim), mssim its mean over the entries at least 3 pixels from the border (scikit-image's first return value). With full=True
    the float32 SSIM map, shaped like x, comes third. Strided inputs are copied; nothing is synchronised."""
    if x.shape != y.shape:
        raise ValueError(f'ssim: input images must have the same shape, got {tuple(x.shape)} and {tuple(y.shape)}')
    if x.dim() not in (3, 4):
        raise ValueError(f'ssim: expected [H,W,C] or [n,H,W,C] images, got shape {tuple(x.shape)}')
    if x.dtype != torch.float32 or y.dtype != torch.float32:
        raise _C.XrbError(f'XRB_E_BADARG ({_C.XRB_E_BADARG}): ssim takes float32 images, got {x.dtype} and {y.dtype}')
    _C.require_cuda(x, y)
    one = x.dim() == 3
    x4, y4 = (x[None], y[None]) if one else (x, y)
    x4, y4 = x4.contiguous(), y4.contiguous()
    n, h, w, c = x4.shape
    dev = x4.device
    mean_full = torch.empty(n, dtype=torch.float64, device=dev)
    mean_crop = torch.empty(n, dtype=torch.float64, device=dev)
    s_map = torch.empty(x4.shape, dtype=torch.float32, device=dev) if full else None
    ws = torch.empty(max(int(_C.lib.xrb_ssim_workspace(n, h, w)), 8), dtype=torch.uint8, device=dev)
    with torch.cuda.device(dev):
        _C.check(_C.lib.xrb_ssim(_C.f32(x4), _C.f32(y4), n, h, w, c, float(data_range), _C.ptr(mean_full), _C.ptr(mean_crop), _C.f32(s_map), _C.ptr(ws),
                                 ws.numel(), _C.stream()), 'ssim')
    if one:
        mean_full, mean_crop, s_map = mean_full[0], mean_crop[0], None if s_map is None else s_map[0]
    return (mean_full, mean_crop, s_map) if full else (mean_full, mean_crop)


def _view_scores(rgbs, gts, data_range):
    """[k, 3] float64 device tensor of (mse, psnr, ssim) per view: mse / psnr by img2mse / mse2psnr per view, SSIM by one launch per distinct view
    shape (one launch in all when the views share a shape)"""
    mse = torch.stack([img2mse(r, g) for r, g in zip(rgbs, gts)])
    s = torch.empty(len(rgbs), dtype=torch.float64, device=mse.device)
    for shape in dict.fromkeys(r.shape for r in rgbs):
        idx = [i for i, r in enumerate(rgbs) if r.shape == shape]
        s[idx] = ssim(torch.stack([rgbs[i] for i in idx]), torch.stack([gts[i] for i in idx]), data_range)[0]
    return torch.stack([mse.double(), mse2psnr(mse).double(), s], 1)


def _mean(v):
    return sum(v) / len(v)


def validate_metrics(outputs, data_range=2.0):
    """ValidateHook.after_val_iter on a val_step output: None when `rgbs` is empty or rgbs[0] and gt_imgs[0] differ in shape (the hook returns
    there), else {'mse', 'psnr', 'ssim': one Python float per view, 'average_mse', 'average_psnr', 'average_ssim'}. The ssim is calculate_ssim's
    mean over the whole SSIM map; data_range defaults to the R = 2 the hook's call ends up with (module docstring)."""
    rgbs, gts = outputs['rgbs'], outputs['gt_imgs']
    if len(rgbs) == 0 or rgbs[0].shape != gts[0].shape:
        return None
    scores = _view_scores(rgbs, [gts[i] for i in range(len(rgbs))], data_range).cpu().tolist()
    out = {k: [v[j] for v in scores] for j, k in enumerate(('mse', 'psnr', 'ssim'))}
    out.update({'average_' + k: _mean(out[k]) for k in ('mse', 'psnr', 'ssim')})
    return out


class TestMetrics:
    """TestHook: add() files each test_step output's view under scale idx % ndown; summary() scores every view (one SSIM launch per view size, one host sync) and
    returns {'average_mse', 'average_psnr', 'average_ssim': one float per scale, 'psnrs', 'ssims': {scale: [one float per view]}}, the last two
    being the dict the hook dumps as JSON. data_range as validate_metrics."""
    __test__ = False                                    # not a pytest class

    def __init__(self, ndown=1, data_range=2.0):
        self.ndown, self.data_range = int(ndown), data_range
        self.views = []                                 # (scale, rgb, gt_img) in arrival order

    def add(self, output):
        self.views.append((int(output['idx']) % self.ndown, output['rgb'], output['gt_img']))

    def summary(self):
        if not self.views:
            raise ValueError('TestMetrics.summary: no view was added')
        scores = _view_scores([v[1] for v in self.views], [v[2] for v in self.views], self.data_range).cpu().tolist()
        by_scale = {s: [sc for v, sc in zip(self.views, scores) if v[0] == s] for s in range(self.ndown)}
        empty = [s for s, v in by_scale.items() if not v]
        if empty:
            raise ValueError(f'TestMetrics.summary: no view at scale(s) {empty}')
        out = {'average_' + k: [_mean([v[j] for v in by_scale[s]]) for s in range(self.ndown)] for j, k in enumerate(('mse', 'psnr', 'ssim'))}
        out['psnrs'] = {s: [v[1] for v in by_scale[s]] for s in range(self.ndown)}
        out['ssims'] = {s: [v[2] for v in by_scale[s]] for s in range(self.ndown)}
        return out
