"""developer probe: NerfNetwork.train_step time (forward + backward, Blender settings: 4096 rays, 64 + 128 samples) on the tensor-core training path.
CUDA events around whole steps after warm-up; prints the GPU's name and power limit with the figure."""
import os
import subprocess
import sys

sys.path.insert(0, os.environ.get('XRB_PKG_ROOT') or os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import torch
from xrnerf_b200 import registry as R

NERF = dict(type='NerfMLP', skips=[4], netdepth=8, netwidth=256, netchunk=1024 * 32, output_ch=5, use_viewdirs=True, embedder=dict(type='BaseEmbedder', i_embed=0, multires=10, multires_dirs=4))
steps = int(sys.argv[1]) if len(sys.argv) > 1 else 20
torch.manual_seed(0)
net = R.build_network(dict(type='NerfNetwork', cfg=dict(phase='train', N_importance=128, is_perturb=False, chunk=1024 * 32, bs_data='rays_o'), mlp=NERF, mlp_fine=NERF,
                           render=dict(type='NerfRender', white_bkgd=True, raw_noise_std=0))).cuda()
opt = torch.optim.Adam(net.parameters(), lr=5e-4)
n = 4096
g = torch.Generator().manual_seed(1)
o = (torch.nn.functional.normalize(torch.randn((n, 3), generator=g), dim=-1) * 4).cuda()
d = torch.nn.functional.normalize(-o.cpu() + torch.randn((n, 3), generator=g) * 0.5, dim=-1).cuda()
t = torch.linspace(0., 1., 64, device='cuda')
z = (2.0 * (1. - t) + 6.0 * t).expand(n, 64).contiguous()
data = {'rays_o': o[None], 'rays_d': d[None], 'viewdirs': d[None], 'z_vals': z[None], 'pts': (o[:, None, :] + d[:, None, :] * z[:, :, None])[None], 'target_s': torch.rand((1, n, 3), device='cuda')}


def step():
    out = net.train_step(dict(data), opt)
    opt.zero_grad(set_to_none=True)
    out['loss'].backward()
    opt.step()


for _ in range(3):
    step()
torch.cuda.synchronize()
a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
a.record()
for _ in range(steps):
    step()
b.record()
torch.cuda.synchronize()
gpu = subprocess.run(['nvidia-smi', '--query-gpu=name,power.limit', '--format=csv,noheader'], capture_output=True, text=True).stdout.strip()
print(f'train_step (4096 rays, 64 + 128 samples): {a.elapsed_time(b) / steps:.3f} ms/step over {steps} steps | {gpu}', flush=True)
