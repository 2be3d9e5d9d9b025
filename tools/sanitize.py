"""Small invocations of every kernel, meant to run under compute-sanitizer:
compute-sanitizer --tool memcheck python tools/sanitize.py"""
import os
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import torch

import cspn_b200
from cspn_b200 import _lib
from cspn_b200.synth import make_inputs, make_inputs_3d

for (B, C, H, W, n, algo) in [(2, 1, 100, 256, 6, 2), (1, 2, 48, 260, 60, 2), (1, 1, 700, 64, 4, 2), (1, 1, 41, 132, 5, 2),
                              (1, 1, 20, 18, 4, 0)]:
    g, d, s = [t.cuda() for t in make_inputs(1, B, C, H, W)]
    out = cspn_b200.propagate2d(g, d, s, n, '8sum', algo)
    torch.cuda.synchronize()
    print('2D', B, C, H, W, n, _lib.ALGO_NAMES[_lib.lib().cspn_last_algo()], _lib.lib().cspn_last_launches(), float(out.sum()), flush=True)

# chained strips (forced: the batches are small), incl. several passes, and the 3D kernels that gather from the raw guidance
os.environ['CSPN_B200_CHAIN'] = '1'
for (B, C, H, W, n) in [(3, 1, 100, 520, 12), (2, 2, 48, 300, 40), (2, 1, 33, 260, 31)]:
    g, d, s = [t.cuda() for t in make_inputs(4, B, C, H, W)]
    out = cspn_b200.propagate2d(g, d, s, n, '8sum', 2)
    torch.cuda.synchronize()
    print('2D chained', B, C, H, W, n, cspn_b200.describe_plan(B, C, H, W, n, 2)[:60], float(out.sum()), flush=True)
os.environ.pop('CSPN_B200_CHAIN')
for mode in ('26sum', '26sum_abs', 'paddle'):
    g3, f3 = [t.cuda() for t in make_inputs_3d(3, 2, 1, 5, 9, 24, signed=(mode == '26sum'))]
    out = cspn_b200.propagate3d(g3, f3, 3, mode)
    torch.cuda.synchronize()
    print('3D direct', mode, _lib.lib().cspn_last_launches(), float(out.sum()), flush=True)

g, d, s = [t.cuda() for t in make_inputs(2, 1, 1, 40, 64)]
g.requires_grad_(True); d.requires_grad_(True)
cspn_b200.Affinity_Propagate(5, 3, '8sum')(g, d, s).sum().backward()
torch.cuda.synchronize()
print('2D backward', float(g.grad.abs().sum()), float(d.grad.sum()), flush=True)

g3, f3 = [t.cuda() for t in make_inputs_3d(3, 1, 1, 6, 10, 16)]
g3.requires_grad_(True); f3.requires_grad_(True)
cspn_b200.Affinity_Propagate3D(3, 3, '26sum_abs')(g3, f3).sum().backward()
torch.cuda.synchronize()
print('3D fwd+bwd', float(g3.grad.abs().sum()), float(f3.grad.sum()), flush=True)

# 5x5x5 kernels (cspn3d_wide.cu): every norm, direct / vectorised and scalar paths, forward and backward
for mode in ('124sum', '124sum_abs', 'paddle'):
    for W in (16, 13):
        g5 = torch.rand(2, 124, 5, 7, W, device='cuda')
        f5 = torch.rand(2, 2, 5, 7, W, device='cuda')
        out = cspn_b200.propagate3d_k(g5, f5, 5, 3, mode)
        torch.cuda.synchronize()
        print('3D 5x5x5', mode, W, _lib.lib().cspn_last_launches(), float(out.sum()), flush=True)
        g5.requires_grad_(True); f5.requires_grad_(True)
        m = cspn_b200.Affinity_Propagate3DK(3, 5, mode)
        m._use_op = False
        m(g5, f5).sum().backward()
        torch.cuda.synchronize()
        print('3D 5x5x5 fwd+bwd', mode, W, float(g5.grad.abs().sum()), float(f5.grad.sum()), flush=True)
