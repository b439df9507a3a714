"""developer probe: NerfMLP tensor-core training vs the fp16-emulated autograd path for several row counts"""
import os, sys
import torch
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), 'tests'))
import test_gpu_nerf_train as T
from cases import NERF_MLP
from restate64 import emulated_fp16_forward
from xrnerf_b200 import registry as R

for n in [int(a) for a in sys.argv[1:]] or [128, 129, 256, 300, 384]:
    torch.manual_seed(n)
    mlp = R.build_mlp(dict(NERF_MLP)).cuda()
    x = torch.rand((n, 90), device='cuda') * 2 - 1
    g = torch.randn((n, 4), device='cuda') * 1e-3
    if os.environ.get('ONLY_RGB'):
        g[:, 3] = 0
    if os.environ.get('ONLY_ALPHA'):
        g[:, :3] = 0
    mlp.fused_train = False
    ref = T._grads(mlp, emulated_fp16_forward(mlp, x), g)
    mlp.fused_train = True
    ours = T._grads(mlp, mlp.batchify_run_mlp(x), g)
    out = []
    for k in ('rgb_linear.weight', 'views_linears.0.weight', 'feature_linear.weight', 'alpha_linear.weight', 'pts_linears.7.weight', 'pts_linears.7.bias', 'pts_linears.6.weight', 'pts_linears.5.weight', 'pts_linears.4.weight', 'pts_linears.0.weight'):
        e = (ours[k] - ref[k]).double()
        out.append('%s %.1e' % (k.replace('_linears', '').replace('_linear', ''), float(torch.sqrt((e ** 2).sum() / (ref[k].double() ** 2).sum()))))
    print(n, ' | '.join(out), flush=True)
